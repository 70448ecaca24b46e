// conv_tc.cuh -- 3x3 convolution, padding 1, as an implicit GEMM on wgmma / TMA (sm_90a): the LPIPS VGG16 layers with C_in >= 64.
//
//   out[p, n] = sum_{tap, c} x[p + shift(tap), c] . Wp[n, tap * C_in + c]      M = pixels, N = C_out, K = 9 C_in, fp32 accumulate
//
// x is a bf16 NHWC activation, Wp the weights packed once at load to [C_out, 9 C_in] (K-major, bf16). The M tile of 128 pixels is a
// spatial block of 8 rows x 16 columns of one image. Its A operand for one (tap, 64-channel chunk) is ONE 4-D TMA load of the NHWC
// tensor at coordinates shifted by the tap's (dy, dx): the box lands in shared memory as 128 rows of 128 B, swizzled exactly as the
// GEMM's 2-D A tile, and the rows / columns outside the image arrive zero-filled, which is the padding. No im2col buffer exists.
// The kernel runs the encoder GEMM's kernel body (gemm_body in tc_gemm.cuh) on its cooperative schedule; this file supplies the
// pixel-tile decode, the tap-shifted A load and the epilogue. Tiles are persistent over (image, tile row, tile column, N block).
// Pixels of a partial tile (45 x 80, 22 x 40, ...) are computed on zeros and not stored.
//
// The data gradient of the same layer is the same kernel: dx = conv3x3(dy, W flipped and transposed), packed [C_in, 9 C_out].
// Epilogues (bf16 NHWC out, 16 B per lane after the quad transpose of tc_gemm.cuh):
//   CONV_BIAS_RELU  out = max(acc + bias, 0)                       forward
//   CONV_MASK       out = mask > 0 ? acc : 0                       data gradient into a layer whose input is a ReLU output (mask):
//                                                                  a select, so a non-finite value under a zero mask never passes
//   CONV_PLAIN      out = acc                                      data gradient into a max-pool output (lpips.cu finishes it), and
//                                                                  every data gradient of the VQGAN decoder (vqgan.cu)
//   CONV_BIAS       out = acc + bias                               the VQGAN decoder's convolutions (no activation after them)
//   CONV_BIAS_RESID out = acc + bias + resid                       its ResnetBlock's conv2, with the shortcut as a bf16 residual
#pragma once
#include "tc_gemm.cuh"

namespace aph {

enum : int { CONV_BIAS_RELU = 0, CONV_MASK = 1, CONV_PLAIN = 2, CONV_BIAS = 3, CONV_BIAS_RESID = 4 };
template <int EPI> constexpr bool conv_has_bias() { return EPI == CONV_BIAS_RELU || EPI == CONV_BIAS || EPI == CONV_BIAS_RESID; }
constexpr int CONV_TH = 8, CONV_TW = 16;   // the 128-pixel spatial tile

struct ConvShape { int N, H, W, Cin, Cout, tiles_y, tiles_x; };
struct ConvEpi {
  const float* bias = nullptr;   // [Cout] (CONV_BIAS_RELU, CONV_BIAS, CONV_BIAS_RESID)
  const bf16* mask = nullptr;    // bf16 NHWC [N,H,W,Cout] (CONV_MASK)
  const bf16* resid = nullptr;   // bf16 NHWC [N,H,W,Cout] (CONV_BIAS_RESID)
  bf16* out = nullptr;           // bf16 NHWC [N,H,W,Cout]
};

// A 32-column chunk of one pixel's output (all 32 lanes call it: shuffles). v[2 t + {0,1}] = accumulators at columns
// col0 + 8 t + 2 q + {0,1}; bb[t] their bias.
template <int EPI>
__device__ __forceinline__ void conv_store_bf16x32(const ConvEpi& epi, size_t pix, bool valid, int Cout, int col0, int q,
                                                   const float* v, const float2* bb) {
  const size_t off = pix * Cout + col0 + 8 * q;
  uint32_t w[4], m[4];
  if constexpr (EPI == CONV_MASK) {
    uint4 g = make_uint4(0u, 0u, 0u, 0u);
    if (valid) g = __ldg(reinterpret_cast<const uint4*>(epi.mask + off));
    m[0] = g.x; m[1] = g.y; m[2] = g.z; m[3] = g.w;
    quad_transpose(m, q);                                        // back to the accumulator layout
  }
  if constexpr (EPI == CONV_BIAS_RESID) load_bf16x8_acc(epi.resid, off, valid, q, m);
#pragma unroll
  for (int t = 0; t < 4; ++t) {
    const float v0 = v[2 * t], v1 = v[2 * t + 1];
    if (EPI == CONV_BIAS_RELU) {
      w[t] = pack_bf16(fmaxf(v0 + bb[t].x, 0.f), fmaxf(v1 + bb[t].y, 0.f));
    } else if (EPI == CONV_MASK) {
      const float2 h = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&m[t]));
      w[t] = pack_bf16(h.x > 0.f ? v0 : 0.f, h.y > 0.f ? v1 : 0.f);
    } else if (EPI == CONV_BIAS) {
      w[t] = pack_bf16(v0 + bb[t].x, v1 + bb[t].y);
    } else if (EPI == CONV_BIAS_RESID) {
      const float2 r = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&m[t]));
      w[t] = pack_bf16(v0 + bb[t].x + r.x, v1 + bb[t].y + r.y);
    } else {
      w[t] = pack_bf16(v0, v1);
    }
  }
  quad_transpose(w, q);
  if (valid) st_global_16(epi.out + off, w);
}

// The convolution as a gemm_body problem (tc_gemm.cuh). Tile = (image, tile row, tile column, N block), in row-major order;
// K block kb is (tap, 64-channel chunk) = (kb / cchunks, kb % cchunks).
template <int BN, int EPI>
struct ConvProblem {
  const ConvShape& cs;
  const ConvEpi& epi;
  using Elem = bf16;

  __device__ __forceinline__ int tiles_img() const { return cs.tiles_y * cs.tiles_x; }
  __device__ __forceinline__ int cchunks() const { return cs.Cin / GEMM_BK; }
  __device__ __forceinline__ int n_tiles() const { return cs.Cout / BN; }
  __device__ __forceinline__ int num_tiles() const { return cs.N * tiles_img() * n_tiles(); }
  __device__ __forceinline__ int k_blocks() const { return 9 * cchunks(); }
  __device__ __forceinline__ bool has_tile(int tile) const { return tile < num_tiles(); }

  struct Tile { int img, ty, tx, n_blk; };
  __device__ __forceinline__ Tile tile(int tile) const {
    const int m_blk = tile / n_tiles(), n_blk = tile - m_blk * n_tiles();
    const int img = m_blk / tiles_img(), r = m_blk - img * tiles_img(), ty = r / cs.tiles_x;
    return {img, ty, r - ty * cs.tiles_x, n_blk};
  }

  // the 8 x 16 x 64 box of x at the tile's pixels shifted by the tap's (dy, dx)
  __device__ __forceinline__ void load_a(void* dst, const CUtensorMap* map_x, uint64_t* bar, Tile t, int kb) const {
    const int tap = kb / cchunks(), ch = kb - tap * cchunks();
    tma_load_4d(dst, map_x, bar, ch * GEMM_BK, t.tx * CONV_TW + tap % 3 - 1, t.ty * CONV_TH + tap / 3 - 1, t.img);
  }

  __device__ __forceinline__ void epilogue(const float (&d)[1][BN / 2], Tile t, int row_in_tile, int col_in_tile, int lane) const {
    // rows row_in_tile and row_in_tile + 8 are columns x0, x0 + 8 of tile row y
    const int y = t.ty * CONV_TH + row_in_tile / CONV_TW, x0 = t.tx * CONV_TW + row_in_tile % CONV_TW, x1 = x0 + 8;
    const bool v0ok = y < cs.H && x0 < cs.W, v1ok = y < cs.H && x1 < cs.W;
    const size_t pix0 = ((size_t)t.img * cs.H + y) * cs.W + x0, pix1 = pix0 + 8;
#pragma unroll
    for (int j0 = 0; j0 < BN / 8; j0 += 4) {            // 32-column chunks
      const int col0 = t.n_blk * BN + 8 * j0;
      float2 bb[4];
      float v0[8], v1[8];
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        bb[i] = conv_has_bias<EPI>() ? __ldg(reinterpret_cast<const float2*>(epi.bias + col0 + 8 * i + col_in_tile)) : make_float2(0.f, 0.f);
        v0[2 * i] = d[0][4 * (j0 + i)]; v0[2 * i + 1] = d[0][4 * (j0 + i) + 1];
        v1[2 * i] = d[0][4 * (j0 + i) + 2]; v1[2 * i + 1] = d[0][4 * (j0 + i) + 3];
      }
      conv_store_bf16x32<EPI>(epi, pix0, v0ok, cs.Cout, col0, lane & 3, v0, bb);
      conv_store_bf16x32<EPI>(epi, pix1, v1ok, cs.Cout, col0, lane & 3, v1, bb);
    }
  }
};

template <int BN, int EPI>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
k_conv3x3_tc(const __grid_constant__ CUtensorMap map_x, const __grid_constant__ CUtensorMap map_w, ConvShape cs, ConvEpi epi) {
  gemm_body<BN, false>(map_x, map_w, ConvProblem<BN, EPI>{cs, epi});
}

// Launches the convolution on `st` (conv_tc.cu): x bf16 NHWC [N,H,W,Cin], wpack bf16 [Cout, 9 Cin]; Cin and Cout multiples of 64.
int launch_conv3x3(const void* x, const void* wpack, int N, int H, int W, int Cin, int Cout, int epi_kind, const ConvEpi& epi,
                   cudaStream_t st);

}  // namespace aph
