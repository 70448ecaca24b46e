// conv_tc.cuh -- 3x3 convolution, padding 1, as an implicit GEMM on wgmma / TMA (sm_90a): the LPIPS VGG16 layers with C_in >= 64.
//
//   out[p, n] = sum_{tap, c} x[p + shift(tap), c] . Wp[n, tap * C_in + c]      M = pixels, N = C_out, K = 9 C_in, fp32 accumulate
//
// x is a bf16 NHWC activation, Wp the weights packed once at load to [C_out, 9 C_in] (K-major, bf16). The M tile of 128 pixels is a
// spatial block of 8 rows x 16 columns of one image. Its A operand for one (tap, 64-channel chunk) is ONE 4-D TMA load of the NHWC
// tensor at coordinates shifted by the tap's (dy, dx): the box lands in shared memory as 128 rows of 128 B, swizzled exactly as the
// GEMM's 2-D A tile, and the rows / columns outside the image arrive zero-filled, which is the padding. No im2col buffer exists.
// The schedule is the encoder GEMM's cooperative one (tc_gemm.cuh: TMA producer warpgroup, two consumer warpgroups on rows
// 0-63 / 64-127, the same stage ring, barriers and wgmma wrappers); tiles are persistent over (image, tile row, tile column, N
// block). Pixels of a partial tile (45 x 80, 22 x 40, ...) are computed on zeros and not stored.
//
// The data gradient of the same layer is the same kernel: dx = conv3x3(dy, W flipped and transposed), packed [C_in, 9 C_out].
// Epilogues (bf16 NHWC out, 16 B per lane after the quad transpose of tc_gemm.cuh):
//   CONV_BIAS_RELU  out = max(acc + bias, 0)                       forward
//   CONV_MASK       out = mask > 0 ? acc : 0                       data gradient into a layer whose input is a ReLU output (mask):
//                                                                  a select, so a non-finite value under a zero mask never passes
//   CONV_PLAIN      out = acc                                      data gradient into a max-pool output (lpips.cu finishes it)
#pragma once
#include "tc_gemm.cuh"

namespace aph {

enum : int { CONV_BIAS_RELU = 0, CONV_MASK = 1, CONV_PLAIN = 2 };
constexpr int CONV_TH = 8, CONV_TW = 16;   // the 128-pixel spatial tile

struct ConvShape { int N, H, W, Cin, Cout, tiles_y, tiles_x; };
struct ConvEpi {
  const float* bias = nullptr;   // [Cout] (CONV_BIAS_RELU)
  const bf16* mask = nullptr;    // bf16 NHWC [N,H,W,Cout] (CONV_MASK)
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
#pragma unroll
  for (int t = 0; t < 4; ++t) {
    const float v0 = v[2 * t], v1 = v[2 * t + 1];
    if (EPI == CONV_BIAS_RELU) {
      w[t] = pack_bf16(fmaxf(v0 + bb[t].x, 0.f), fmaxf(v1 + bb[t].y, 0.f));
    } else if (EPI == CONV_MASK) {
      const float2 h = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&m[t]));
      w[t] = pack_bf16(h.x > 0.f ? v0 : 0.f, h.y > 0.f ? v1 : 0.f);
    } else {
      w[t] = pack_bf16(v0, v1);
    }
  }
  quad_transpose(w, q);
  if (valid) st_global_16(epi.out + off, w);
}

template <int BN, int EPI>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
k_conv3x3_tc(const __grid_constant__ CUtensorMap map_x, const __grid_constant__ CUtensorMap map_w, ConvShape cs, ConvEpi epi) {
  using L = GemmCfg<BN>;
  constexpr int STAGES = L::STAGES;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + L::BAR_OFFSET);
  uint64_t* empty_bar = full_bar + STAGES;

  const int wg = threadIdx.x >> 7, tid = threadIdx.x & 127;
  const int n_tiles = cs.Cout / BN, tiles_img = cs.tiles_y * cs.tiles_x;
  const int num_tiles = cs.N * tiles_img * n_tiles, cchunks = cs.Cin / GEMM_BK, k_blocks = 9 * cchunks;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&map_x); tma_prefetch_desc(&map_w);
    for (int i = 0; i < STAGES; ++i) { mbar_init(&full_bar[i], 1); mbar_init(&empty_bar[i], 2); }
    fence_barrier_init();
  }
  __syncthreads();

  if (wg == 0) {
    setmaxnreg_dec<40>();
    if (tid == 0) {
      // ===== TMA producer: per k block one shifted 8 x 16 x 64 box of x and one BN x 64 box of the packed weights
      const uint64_t pol_b = l2_policy_evict_last();
      uint32_t it = 0;
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        const int m_blk = tile / n_tiles, n_blk = tile - m_blk * n_tiles;
        const int img = m_blk / tiles_img, r = m_blk - img * tiles_img, ty = r / cs.tiles_x, tx = r - ty * cs.tiles_x;
        for (int kb = 0; kb < k_blocks; ++kb, ++it) {
          const int tap = kb / cchunks, ch = kb - tap * cchunks;
          const uint32_t s = it % STAGES, ph = (it / STAGES) & 1;
          mbar_wait(&empty_bar[s], ph ^ 1);
          uint8_t* sa = smem + s * L::STAGE_BYTES;
          mbar_expect_tx(&full_bar[s], L::STAGE_BYTES);
          tma_load_4d(sa, &map_x, &full_bar[s], ch * GEMM_BK, tx * CONV_TW + tap % 3 - 1, ty * CONV_TH + tap / 3 - 1, img);
          tma_load_2d_hint(sa + L::A_BYTES, &map_w, &full_bar[s], kb * GEMM_BK, n_blk * BN, pol_b);
        }
      }
    }
  } else {
    setmaxnreg_inc<232>();
    // ===== consumer warpgroup c: rows 64 c .. 64 c + 63 of every tile
    const int c = wg - 1, warp = tid >> 5, lane = tid & 31;
    const int row_in_tile = 64 * c + 16 * warp + (lane >> 2), col_in_tile = 2 * (lane & 3);
    // rows row_in_tile and row_in_tile + 8 are columns px, px + 8 of tile row py
    const int py = row_in_tile / CONV_TW, px = row_in_tile % CONV_TW;
    uint32_t it = 0;
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
      float d[BN / 2];
#pragma unroll
      for (int r = 0; r < BN / 2; ++r) d[r] = 0.f;
      for (int kb = 0; kb < k_blocks; ++kb, ++it) {
        const uint32_t s = it % STAGES, ph = (it / STAGES) & 1;
        mbar_wait(&full_bar[s], ph);
        const uint64_t ds = make_smem_desc(smem_u32(smem + s * L::STAGE_BYTES));
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < GEMM_BK / GEMM_UK; ++k)
          Wgmma<BN>::mma(d, ds + (uint64_t)(c * 512 + 2 * k), ds + (uint64_t)(L::A_BYTES / 16 + 2 * k), (kb | k) != 0);
        wgmma_commit();
        wgmma_wait<1>();
        if (kb > 0 && tid == 0) mbar_arrive(&empty_bar[(it - 1) % STAGES]);
      }
      wgmma_wait<0>();
      if (tid == 0) mbar_arrive(&empty_bar[(it - 1) % STAGES]);
      const int m_blk = tile / n_tiles, n_blk = tile - m_blk * n_tiles;
      const int img = m_blk / tiles_img, r = m_blk - img * tiles_img, ty = r / cs.tiles_x, tx = r - ty * cs.tiles_x;
      const int y = ty * CONV_TH + py, x0 = tx * CONV_TW + px, x1 = x0 + 8;
      const bool v0ok = y < cs.H && x0 < cs.W, v1ok = y < cs.H && x1 < cs.W;
      const size_t pix0 = ((size_t)img * cs.H + y) * cs.W + x0, pix1 = pix0 + 8;
#pragma unroll
      for (int j0 = 0; j0 < BN / 8; j0 += 4) {            // 32-column chunks
        const int col0 = n_blk * BN + 8 * j0;
        float2 bb[4];
        float v0[8], v1[8];
#pragma unroll
        for (int t = 0; t < 4; ++t) {
          bb[t] = (EPI == CONV_BIAS_RELU) ? __ldg(reinterpret_cast<const float2*>(epi.bias + col0 + 8 * t + col_in_tile)) : make_float2(0.f, 0.f);
          v0[2 * t] = d[4 * (j0 + t)]; v0[2 * t + 1] = d[4 * (j0 + t) + 1];
          v1[2 * t] = d[4 * (j0 + t) + 2]; v1[2 * t + 1] = d[4 * (j0 + t) + 3];
        }
        conv_store_bf16x32<EPI>(epi, pix0, v0ok, cs.Cout, col0, lane & 3, v0, bb);
        conv_store_bf16x32<EPI>(epi, pix1, v1ok, cs.Cout, col0, lane & 3, v1, bb);
      }
    }
  }
}

// Launches the convolution on `st`: x bf16 NHWC [N,H,W,Cin], wpack bf16 [Cout, 9 Cin]; Cin and Cout multiples of 64.
int launch_conv3x3(const void* x, const void* wpack, int N, int H, int W, int Cin, int Cout, int epi_kind, const ConvEpi& epi,
                   cudaStream_t st);

}  // namespace aph
