// cppn.cu -- the CPPN generator of cppn.py: a per-pixel MLP from the (x, y) coordinate to RGB, forward and weight gradient.
//
// Network (cppn.py:71-116): layer 0 is 2 -> NF, layers 1 .. L-1 are KH -> NF, the output layer is KH -> 3 with a sigmoid.
// KH = 2 NF for the activations `unbias` / `comp`, NF for `relu`:
//   unbias: t = atan(z), x = cat(t / 0.67, (t^2 - 0.45) / 0.396)      comp: t = atan(z), x = cat(t / 0.67, t^2 / 0.6)
//   relu:   x = (relu(z) - 0.4) / 0.58
// Weights are the nn.Conv2d storages, [out][in] (the 1x1 kernel dimensions dropped), read in place every call.
//
//   k_cppn_fwd    : one warp takes 16 pixels at a time through every layer with the activations in registers.
//   k_cppn_bwd    : a CTA of 4 warps takes a tile of 64 pixels: it recomputes the forward, keeping each layer's pre-activation
//                   z_l, then walks back through the layers. Per-CTA weight-gradient partials go to handle scratch.
//   k_cppn_reduce : sums the partials of every CTA in a fixed order into the parameter gradients (no float atomics: the
//                   gradient is bit-reproducible from run to run).
//
// Tensor cores. The hidden layers' products (forward z = x W^T, data gradient dx = dz W, weight gradient dW = dz^T x) run as
// mma.sync.m16n8k8 TF32 with fp32 accumulation; both operands are rounded by cvt.rna.tf32.f32 (round to nearest, ties away).
// mma.sync rather than wgmma: the matrices are small (N = NF down to 8, K = KH), the operands live in registers between layers
// (wgmma needs M = 64 per warpgroup and its B operand in shared memory), and at nf 24 the atan of every pre-activation costs
// about as many instructions as the MMAs.
// Layer 0 (K = 2), the output layer (N = 3), atan, the activations and the sigmoid run in fp32 with atanf / expf.
//
// Register layout. Element e of an m16n8 accumulator fragment is (row g + 8 (e >> 1), column 2 t + (e & 1)), g = lane / 4,
// t = lane % 4. The next product reads the same registers as its A fragment by letting physical k-column t stand for logical
// column 2 t and t + 4 for 2 t + 1 (B is loaded with the same permutation), so layer outputs never leave the thread between
// layers. The weight gradient needs the pixel index as the K dimension, which the fragments hold on g: dz_l and x_l go
// through shared memory for it.
//
// Where z_l lives in the backward: per warp [L][NF/8][32 lanes] float4 (64 NF L floats per CTA), in shared memory when it fits
// beside the staging buffers within CPPN_SMEM_CAP (nf 24: up to 14 layers, 61 KB at the default 10; nf 64: up to 3 layers),
// otherwise in handle scratch (one slot per resident CTA, mostly L2-resident). Nothing else goes to global memory but the
// coordinates, the image, its gradient and the partials.
//
// Wide nets (72 <= nf <= 256) do not fit that scheme: a warp's 16 pixels x KH activations would take KH / 2 registers per lane,
// and per-CTA weight-gradient partials 512 KB per layer. They run layer by layer over all pixels instead, every hidden-layer
// product a TF32 wgmma GEMM on the encoder GEMM's main loop (gemm_body, tc_gemm.cuh) with a CPPN epilogue:
//   k_cppnw_pack     : rounds the hidden weights to TF32 once per call into the handle: W' [NF][KH] and its transpose W'^T
//                      [KH][NF]. W' takes the input columns in the order x' = (a_0, s_0, a_1, s_1, ...) (a_j = atan(z_j) / 0.67,
//                      s_j its square term) so that one thread holds both halves of feature j: the forward epilogue writes
//                      them with one store, and the data-gradient epilogue applies act'(z_j) to both (relu: no reordering).
//   k_cppnw_l0       : layer 0 (K = 2) in fp32, then the activation: x_1 [P][KH].
//   k_cppnw_gemm FWD : z_l = x_l W'_l^T + b_l (M = pixels, N = NF, K = KH); the epilogue writes x_{l+1} = act(z_l), rounded to
//                      TF32 when a hidden layer reads it (the output layer reads it in fp32), and in the backward also z_l
//                      pixel-contiguous ([NF][P], the only thing the forward keeps).
//   k_cppnw_head     : the output layer and the sigmoid in fp32, a warp per pixel.
// The backward recomputes that forward with z_l kept, then walks down the layers:
//   k_cppnw_head_bwd : dz_out = dy y (1 - y), dx_L = dz_out W_out and dz_{L-1} = dx_L act'(z_{L-1}) in fp32, a warp per 16
//                      pixels; per-group partials of dW_out, db_out and db_{L-1}.
//   k_cppnw_actT     : x_l = act(z_{l-1}) again, rounded, pixel-contiguous and split into pixel chunks ([S][KHP][chunk]).
//   k_cppnw_gemm DW  : dW_l = dz_l^T x_l (M = NF, N = KH, K = pixels), split over S pixel chunks: partials [S][NF][KH].
//   k_cppnw_gemm DX  : dx_l = dz_l W'_l (M = pixels, N = KH, K = NF, B = W'^T); the epilogue forms dz_{l-1} = dx act'(z_{l-1})
//                      and writes it rounded as [P][NF] (the next DX operand) and [NF][P] (the next DW operand; layer 0's
//                      unrounded), with per-16-pixel partials of db_{l-1}.
//   k_cppnw_colsum   : every partial is summed in a fixed order (no float atomics: two backward calls are bit-identical).
//   k_cppnw_l0_bwd   : dW_0, db_0 in fp32 from dz_0.
// The rounding model is the narrow path's: both operands of every hidden-layer product rounded by cvt.rna, fp32 accumulation,
// layer 0 / the output layer / the activations in fp32. Scratch: one handle buffer, sized by cppnw_floats().
#include "tc_gemm.cuh"
#include <algorithm>
#include <math.h>

namespace aph {

constexpr int CPPN_MAX_LAYERS = 32;
constexpr int CPPN_WARPS = 4;
constexpr int CPPN_TP = CPPN_WARPS * 16;        // pixels per backward tile
constexpr size_t CPPN_SMEM_CAP = 112 * 1024;    // z_l stays in shared memory up to this CTA size (two CTAs per SM)
constexpr size_t CPPN_PARTIAL_CAP = 128u << 20; // bytes of weight-gradient partials (limits the grid at the largest nets)

enum { CPPN_UNBIAS = 0, CPPN_COMP = 1, CPPN_RELU = 2 };

struct CppnWeights {
  const float* w[CPPN_MAX_LAYERS + 1];
  const float* b[CPPN_MAX_LAYERS + 1];
};
struct CppnGradOut {
  float* p[2 * (CPPN_MAX_LAYERS + 1)];          // W0, b0, W1, b1, ... (the parameter order of the module)
  int off[2 * (CPPN_MAX_LAYERS + 1) + 1];       // start of each in the partial vector; off[2 L + 2] = total
};

// Offsets in the packed parameter vector: W0 [NF][2], b0, then per hidden layer W [NF][KH], b, then W_out [3][KH], b_out.
__host__ __device__ inline int cppn_off_w(int nf, int kh, int l) { return l == 0 ? 0 : 3 * nf + (l - 1) * (nf * kh + nf); }
__host__ __device__ inline int cppn_off_b(int nf, int kh, int l, int L) {
  return l == 0 ? 2 * nf : cppn_off_w(nf, kh, l) + (l == L ? 3 : nf) * kh;
}
__host__ __device__ inline int cppn_total(int nf, int kh, int L) { return cppn_off_b(nf, kh, L, L) + 3; }
// shared-memory row stride for n columns (n % 8 == 0): stride % 32 is 8 or 24, so the fragment loads [p = t][c = g] hit 32 banks
__host__ __device__ constexpr int cppn_stride(int n) { return n / 16 * 16 + 8; }

__device__ __forceinline__ uint32_t to_tf32(float x) {
  uint32_t r;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
  return r;
}
// c += A B, A 16x8 (registers in C-fragment order, see the header), B 8x8
__device__ __forceinline__ void mma_tf32(float (&c)[4], const float (&a)[4], uint32_t b0, uint32_t b1) {
  asm("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
      : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
      : "r"(to_tf32(a[0])), "r"(to_tf32(a[2])), "r"(to_tf32(a[1])), "r"(to_tf32(a[3])), "r"(b0), "r"(b1));
}
__device__ __forceinline__ void mma_tf32_raw(float (&c)[4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint32_t b0,
                                             uint32_t b1) {
  asm("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
      : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
      : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}
__device__ __forceinline__ void rmw(float* p, float v, bool first) { *p = first ? v : *p + v; }

template <int NF, bool RELU>
struct Cppn {
  static constexpr int NB = NF / 8;                // n-blocks of a layer's output
  static constexpr int KB = RELU ? NB : 2 * NB;    // k-blocks of a hidden layer's input
  static constexpr int KH = 8 * KB;

  // x = act(z); t = atan(z) (unused for relu). off / div: the second half's (t^2 - off) / div.
  __device__ static void act(const float (&z)[NB][4], float (&x)[KB][4], float (&t)[NB][4], float off, float div) {
#pragma unroll
    for (int j = 0; j < NB; ++j)
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        if (RELU) {
          x[j][e] = (fmaxf(z[j][e], 0.f) - 0.4f) / 0.58f;
        } else {
          const float a = atanf(z[j][e]);
          t[j][e] = a;
          x[j][e] = a / 0.67f;
          x[j + NB][e] = (a * a - off) / div;
        }
      }
  }

  // z = x W^T + b of a hidden layer, on tensor cores
  __device__ static void hidden(const float (&x)[KB][4], const float* __restrict__ W, const float* __restrict__ b, float (&z)[NB][4],
                                int g, int t) {
#pragma unroll
    for (int j = 0; j < NB; ++j) {
      const float2 bb = __ldg(reinterpret_cast<const float2*>(b + 8 * j + 2 * t));
      z[j][0] = bb.x; z[j][1] = bb.y; z[j][2] = bb.x; z[j][3] = bb.y;
    }
#pragma unroll
    for (int kb = 0; kb < KB; ++kb)
#pragma unroll
      for (int j = 0; j < NB; ++j) {
        const float2 w = __ldg(reinterpret_cast<const float2*>(W + (8 * j + g) * KH + 8 * kb + 2 * t));
        mma_tf32(z[j], x[kb], to_tf32(w.x), to_tf32(w.y));
      }
  }

  // Every layer but the output one. Stores z_l to zs[l] when zs is given. Leaves x = act(z_{L-1}), z = z_{L-1}, tt = atan(z).
  __device__ static void trunk(const float (&c0)[2], const float (&c1)[2], const CppnWeights& P, int L, float off, float div,
                               float (&x)[KB][4], float (&z)[NB][4], float (&tt)[NB][4], float4* zs, int g, int t, int lane) {
#pragma unroll
    for (int j = 0; j < NB; ++j)
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int o = 8 * j + 2 * t + (e & 1), r = e >> 1;
        z[j][e] = fmaf(__ldg(P.w[0] + 2 * o + 1), c1[r], fmaf(__ldg(P.w[0] + 2 * o), c0[r], __ldg(P.b[0] + o)));
      }
    for (int l = 1;; ++l) {
      if (zs) {
#pragma unroll
        for (int j = 0; j < NB; ++j) zs[((l - 1) * NB + j) * 32 + lane] = make_float4(z[j][0], z[j][1], z[j][2], z[j][3]);
      }
      act(z, x, tt, off, div);
      if (l == L) break;
      hidden(x, P.w[l], P.b[l], z, g, t);
    }
  }

  // the output layer in fp32: y[r][c] for the lane's rows g (r = 0) and g + 8 (r = 1); every lane of a quad gets all three
  __device__ static void head(const float (&x)[KB][4], const float* __restrict__ W, const float* __restrict__ b, int t,
                              float (&y)[2][3]) {
    float s[2][3] = {{0.f, 0.f, 0.f}, {0.f, 0.f, 0.f}};
#pragma unroll
    for (int kb = 0; kb < KB; ++kb)
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int k = 8 * kb + 2 * t + (e & 1), r = e >> 1;
#pragma unroll
        for (int c = 0; c < 3; ++c) s[r][c] = fmaf(x[kb][e], __ldg(W + c * KH + k), s[r][c]);
      }
#pragma unroll
    for (int r = 0; r < 2; ++r)
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        float v = s[r][c];
        v += __shfl_xor_sync(0xffffffffu, v, 1);
        v += __shfl_xor_sync(0xffffffffu, v, 2);
        y[r][c] = 1.f / (1.f + expf(-(v + __ldg(b + c))));
      }
  }
};

__device__ __forceinline__ float pick3(const float (&v)[3], int c) { return c == 0 ? v[0] : (c == 1 ? v[1] : v[2]); }

// coordinates of pixel p (planar [N,2,H,W]); out-of-range rows read 0 and are never written
__device__ __forceinline__ void load_coords(const float* __restrict__ coords, int64_t npix, int64_t hw, int64_t p, float& c0, float& c1) {
  c0 = c1 = 0.f;
  if (p < npix) {
    const int64_t n = p / hw, q = p - n * hw;
    c0 = __ldg(coords + 2 * n * hw + q);
    c1 = __ldg(coords + 2 * n * hw + hw + q);
  }
}

template <int NF, bool RELU>
__global__ void __launch_bounds__(128) k_cppn_fwd(const float* __restrict__ coords, int64_t npix, int64_t hw, int L, CppnWeights P,
                                                  float off, float div, float* __restrict__ out) {
  using N = Cppn<NF, RELU>;
  const int lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  const int64_t nwarps = (int64_t)gridDim.x * (blockDim.x >> 5);
  for (int64_t m = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); m * 16 < npix; m += nwarps) {
    float c0[2], c1[2];
    int64_t p[2] = {m * 16 + g, m * 16 + g + 8};
    load_coords(coords, npix, hw, p[0], c0[0], c1[0]);
    load_coords(coords, npix, hw, p[1], c0[1], c1[1]);
    float x[N::KB][4], z[N::NB][4], tt[N::NB][4], y[2][3];
    N::trunk(c0, c1, P, L, off, div, x, z, tt, nullptr, g, t, lane);
    N::head(x, P.w[L], P.b[L], t, y);
    if (t < 3) {
#pragma unroll
      for (int r = 0; r < 2; ++r)
        if (p[r] < npix) {
          const int64_t n = p[r] / hw, q = p[r] - n * hw;
          out[3 * n * hw + t * hw + q] = pick3(y[r], t);
        }
    }
  }
}

template <int NF, bool RELU>
__global__ void __launch_bounds__(128) k_cppn_bwd(const float* __restrict__ coords, int64_t npix, int64_t hw, int L, CppnWeights P,
                                                  float off, float div, const float* __restrict__ gout, float* __restrict__ zglob,
                                                  float* __restrict__ partial, int ptotal, int64_t ntiles) {
  using N = Cppn<NF, RELU>;
  constexpr int NB = N::NB, KB = N::KB, KH = N::KH;
  constexpr int SX = cppn_stride(KH), SZ = cppn_stride(NF);
  constexpr int OB = (NF + 15) / 16;
  extern __shared__ float4 smem4[];
  float* Xs = reinterpret_cast<float*>(smem4);          // [64][SX]: x_l of the tile
  float* DZs = Xs + CPPN_TP * SX;                        // [64][SZ]: dz_l of the tile
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, t = lane & 3;
  const size_t zslot = (size_t)CPPN_TP * NF * L / 4;    // float4 per CTA
  float4* zs = (zglob ? reinterpret_cast<float4*>(zglob) + blockIdx.x * zslot : reinterpret_cast<float4*>(DZs + CPPN_TP * SZ)) +
               (size_t)warp * (zslot / CPPN_WARPS);
  float* part = partial + (size_t)blockIdx.x * ptotal;
  const int row0 = warp * 16 + g;                        // this lane's tile rows: row0, row0 + 8

  for (int64_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    const bool first = tile == blockIdx.x;
    float c0[2], c1[2];
    const int64_t p[2] = {tile * CPPN_TP + row0, tile * CPPN_TP + row0 + 8};
    load_coords(coords, npix, hw, p[0], c0[0], c1[0]);
    load_coords(coords, npix, hw, p[1], c0[1], c1[1]);

    float dx[KB][4], zc[NB][4], tc[NB][4], y[2][3];
    {
      float x[KB][4];
      N::trunk(c0, c1, P, L, off, div, x, zc, tc, zs, g, t, lane);
      N::head(x, P.w[L], P.b[L], t, y);
      // output layer: dz_out = dy y (1 - y) (0 on rows past the frame, so they add nothing anywhere below)
      float dzo[2][3];
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        const int64_t n = p[r] / hw, q = p[r] - n * hw;
#pragma unroll
        for (int c = 0; c < 3; ++c) dzo[r][c] = p[r] < npix ? __ldg(gout + 3 * n * hw + c * hw + q) * (y[r][c] * (1.f - y[r][c])) : 0.f;
        if (t < 3) DZs[(row0 + 8 * r) * SZ + t] = pick3(dzo[r], t);
      }
      const float* Wo = P.w[L];
#pragma unroll
      for (int kb = 0; kb < KB; ++kb) {
        const int k = 8 * kb + 2 * t;
#pragma unroll
        for (int r = 0; r < 2; ++r) {
            *reinterpret_cast<float2*>(Xs + (row0 + 8 * r) * SX + k) = make_float2(x[kb][2 * r], x[kb][2 * r + 1]);
            dx[kb][2 * r + 0] = dzo[r][0] * __ldg(Wo + k) + dzo[r][1] * __ldg(Wo + KH + k) + dzo[r][2] * __ldg(Wo + 2 * KH + k);
            dx[kb][2 * r + 1] = dzo[r][0] * __ldg(Wo + k + 1) + dzo[r][1] * __ldg(Wo + KH + k + 1) + dzo[r][2] * __ldg(Wo + 2 * KH + k + 1);
          }
        }
    }
    __syncthreads();
    {  // dW_out [3][KH], db_out [3] in fp32
      const int ow = cppn_off_w(NF, KH, L), ob = cppn_off_b(NF, KH, L, L);
      for (int idx = tid; idx < 3 * KH + 3; idx += blockDim.x) {
        float s = 0.f;
        if (idx < 3 * KH) {
          const int c = idx / KH, k = idx - c * KH;
          for (int q = 0; q < CPPN_TP; ++q) s = fmaf(DZs[q * SZ + c], Xs[q * SX + k], s);
          rmw(part + ow + idx, s, first);
        } else {
          const int c = idx - 3 * KH;
          for (int q = 0; q < CPPN_TP; ++q) s += DZs[q * SZ + c];
          rmw(part + ob + c, s, first);
        }
      }
    }
    __syncthreads();

    for (int l = L - 1; l >= 0; --l) {
      float dz[NB][4];
#pragma unroll
      for (int j = 0; j < NB; ++j)
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const float zz = zc[j][e];
          if (RELU) dz[j][e] = zz > 0.f ? dx[j][e] / 0.58f : 0.f;
          else dz[j][e] = (dx[j][e] / 0.67f + dx[j + NB][e] * (2.f * tc[j][e]) / div) / (1.f + zz * zz);
        }
#pragma unroll
      for (int j = 0; j < NB; ++j)
#pragma unroll
        for (int r = 0; r < 2; ++r)
          *reinterpret_cast<float2*>(DZs + (row0 + 8 * r) * SZ + 8 * j + 2 * t) = make_float2(dz[j][2 * r], dz[j][2 * r + 1]);
      if (l > 0) {
        // data gradient dx_l = dz_l W_l (M = pixels, N = KH, K = NF)
        const float* W = P.w[l];
#pragma unroll
        for (int i = 0; i < KB; ++i) dx[i][0] = dx[i][1] = dx[i][2] = dx[i][3] = 0.f;
#pragma unroll
        for (int ko = 0; ko < NB; ++ko)
#pragma unroll
          for (int i = 0; i < KB; ++i)
            mma_tf32(dx[i], dz[ko], to_tf32(__ldg(W + (8 * ko + 2 * t) * KH + 8 * i + g)),
                     to_tf32(__ldg(W + (8 * ko + 2 * t + 1) * KH + 8 * i + g)));
        // x_l = act(z_{l-1}), staged for the weight gradient; z_{l-1} and its atan are the next step's
        float x[KB][4];
#pragma unroll
        for (int j = 0; j < NB; ++j) {
          const float4 v = zs[((l - 1) * NB + j) * 32 + lane];
          zc[j][0] = v.x; zc[j][1] = v.y; zc[j][2] = v.z; zc[j][3] = v.w;
        }
        N::act(zc, x, tc, off, div);
#pragma unroll
        for (int kb = 0; kb < KB; ++kb)
#pragma unroll
          for (int r = 0; r < 2; ++r)
            *reinterpret_cast<float2*>(Xs + (row0 + 8 * r) * SX + 8 * kb + 2 * t) = make_float2(x[kb][2 * r], x[kb][2 * r + 1]);
      } else if (t == 0) {
#pragma unroll
        for (int r = 0; r < 2; ++r) *reinterpret_cast<float2*>(Xs + (row0 + 8 * r) * SX) = make_float2(c0[r], c1[r]);
      }
      __syncthreads();
      if (l > 0) {
        // dW_l = dz_l^T x_l over the tile (M = NF padded to 16, N = KH, K = 64 pixels); db_l = column sums of dz_l
        const int ow = cppn_off_w(NF, KH, l), ob = cppn_off_b(NF, KH, l, L);
        for (int tl = warp; tl < OB * KB; tl += CPPN_WARPS) {
          const int o0 = (tl / KB) * 16 + g, o1 = o0 + 8, i0 = (tl % KB) * 8;
          float c[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
          for (int ks = 0; ks < CPPN_TP / 8; ++ks) {
            const int q0 = 8 * ks + t, q1 = q0 + 4;
            const uint32_t a0 = to_tf32(o0 < NF ? DZs[q0 * SZ + o0] : 0.f), a1 = to_tf32(o1 < NF ? DZs[q0 * SZ + o1] : 0.f);
            const uint32_t a2 = to_tf32(o0 < NF ? DZs[q1 * SZ + o0] : 0.f), a3 = to_tf32(o1 < NF ? DZs[q1 * SZ + o1] : 0.f);
            mma_tf32_raw(c, a0, a1, a2, a3, to_tf32(Xs[q0 * SX + i0 + g]), to_tf32(Xs[q1 * SX + i0 + g]));
          }
          if (o0 < NF) { rmw(part + ow + o0 * KH + i0 + 2 * t, c[0], first); rmw(part + ow + o0 * KH + i0 + 2 * t + 1, c[1], first); }
          if (o1 < NF) { rmw(part + ow + o1 * KH + i0 + 2 * t, c[2], first); rmw(part + ow + o1 * KH + i0 + 2 * t + 1, c[3], first); }
        }
        for (int o = tid; o < NF; o += blockDim.x) {
          float s = 0.f;
          for (int q = 0; q < CPPN_TP; ++q) s += DZs[q * SZ + o];
          rmw(part + ob + o, s, first);
        }
      } else {
        // layer 0 in fp32: dW_0 [NF][2], db_0 [NF]
        for (int idx = tid; idx < 3 * NF; idx += blockDim.x) {
          const int o = idx / 3, j = idx - 3 * o;
          float s = 0.f;
          if (j < 2) { for (int q = 0; q < CPPN_TP; ++q) s = fmaf(DZs[q * SZ + o], Xs[q * SX + j], s); }
          else { for (int q = 0; q < CPPN_TP; ++q) s += DZs[q * SZ + o]; }
          rmw(part + (j < 2 ? 2 * o + j : 2 * NF + o), s, first);
        }
      }
      __syncthreads();
    }
  }
}

// dparams = sum over the G CTAs' partials, in CTA order
__global__ void __launch_bounds__(256) k_cppn_reduce(const float* __restrict__ partial, int G, int ptotal, int ntensors, CppnGradOut o) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= ptotal) return;
  float s = 0.f;
  for (int c = 0; c < G; ++c) s += partial[(size_t)c * ptotal + i];
  int k = 0;
  while (k + 1 < ntensors && i >= o.off[k + 1]) ++k;
  o.p[k][i - o.off[k]] = s;
}

// ================= wide nets (72 <= nf <= 256): layer by layer, TF32 wgmma GEMMs =====================================
constexpr int CPPNW_CHUNK = 4096;       // least pixels per weight-gradient split
constexpr int CPPNW_MAX_SPLITS = 256;
constexpr int CPPNW_CH = 256;           // rows per k_cppnw_colsum block

__device__ __forceinline__ float rna(float x) { return __uint_as_float(to_tf32(x)); }
__device__ __forceinline__ float rna_if(float x, bool r) { return r ? rna(x) : x; }
// column of the original [out][in] weight that column i' of W' holds (x' = a_0, s_0, a_1, s_1, ...; relu: the identity)
__host__ __device__ __forceinline__ int cppnw_src_col(int ip, int nf, bool relu) { return relu ? ip : ((ip & 1) ? nf + (ip >> 1) : ip >> 1); }

enum { CW_FWD = 0, CW_DX = 1, CW_DW = 2 };

// Kernel arguments of the three GEMM kinds. Pixel-contiguous buffers ([NF][Ppad]) have rows `ld` = Ppad apart.
struct CppnWideArgs {
  int M, N;                       // output rows / valid columns
  int m_tiles, n_tiles, splits, kblocks, chunk;
  int nf, kh;
  int64_t npix, ld;
  float off, div;
  const float* bias;              // FWD: b_l
  float* x_out;                   // FWD: x_{l+1} [P][KH] in x' order
  int round_out;                  // FWD: x_{l+1} rounded; DX: dz_{l-1} rounded
  float* zT;                      // FWD: z_l [NF][Ppad] (backward only, else NULL)
  const float* zT_in;             // DX: z_{l-1} [NF][Ppad]
  float* dz_out;                  // DX: dz_{l-1} [Ppad][NF] (NULL for layer 0)
  float* dzT_out;                 // DX: dz_{l-1} [NF][Ppad]
  float* part;                    // DX: db_{l-1} partials [Ppad / 16][NF] (NULL for layer 0); DW: [S][NF][KH]
};

// The CPPN GEMMs as a gemm_body problem (cooperative schedule, fp32 operands rounded to TF32, mapped as 16-bit views).
// Tile = (split, m block, n block), n fastest. The B operand of DW is split-major ([S][KHP][chunk]), so the body's n block
// split * n_tiles + n selects the split's rows; A is offset by the split's pixels in load_a.
template <int BN, int EPI, bool RELU>
struct CppnProblem {
  const CppnWideArgs& a;
  using Elem = float;

  __device__ __forceinline__ int num_tiles() const { return a.splits * a.m_tiles * a.n_tiles; }
  __device__ __forceinline__ int k_blocks() const { return a.kblocks; }
  __device__ __forceinline__ bool has_tile(int tile) const { return tile < num_tiles(); }

  struct Tile { int m_blk, n_blk, split; };
  __device__ __forceinline__ Tile tile(int tile) const {
    const int per = a.m_tiles * a.n_tiles, s = tile / per, r = tile - s * per, m = r / a.n_tiles;
    return {m, s * a.n_tiles + (r - m * a.n_tiles), s};
  }
  // K coordinates of the 16-bit view: 64 per 32 fp32
  __device__ __forceinline__ void load_a(void* dst, const CUtensorMap* map_a, uint64_t* bar, Tile t, int kb) const {
    tma_load_2d(dst, map_a, bar, (t.split * (a.chunk / 32) + kb) * GEMM_BK, t.m_blk * GEMM_BM);
  }

  __device__ __forceinline__ void epilogue(const float (&d)[1][BN / 2], Tile t, int row_in_tile, int col_in_tile, int lane) const {
    const int row0 = t.m_blk * GEMM_BM + row_in_tile;
    const int n0 = (t.n_blk - t.split * a.n_tiles) * BN;
    if constexpr (EPI == CW_FWD) {
#pragma unroll
      for (int j = 0; j < BN / 8; ++j) {
        const int col = n0 + 8 * j + col_in_tile;
        if (col >= a.N) continue;
        const float2 bb = __ldg(reinterpret_cast<const float2*>(a.bias + col));
#pragma unroll
        for (int r = 0; r < 2; ++r) {
          const int row = row0 + 8 * r;
          if (row >= a.M) continue;
          const float z0 = d[0][4 * j + 2 * r] + bb.x, z1 = d[0][4 * j + 2 * r + 1] + bb.y;
          if (a.zT) { a.zT[(size_t)col * a.ld + row] = z0; a.zT[(size_t)(col + 1) * a.ld + row] = z1; }
          const bool rd = a.round_out;
          if (RELU) {
            *reinterpret_cast<float2*>(a.x_out + (size_t)row * a.kh + col) =
                make_float2(rna_if((fmaxf(z0, 0.f) - 0.4f) / 0.58f, rd), rna_if((fmaxf(z1, 0.f) - 0.4f) / 0.58f, rd));
          } else {
            const float t0 = atanf(z0), t1 = atanf(z1);
            *reinterpret_cast<float4*>(a.x_out + (size_t)row * a.kh + 2 * col) =
                make_float4(rna_if(t0 / 0.67f, rd), rna_if((t0 * t0 - a.off) / a.div, rd), rna_if(t1 / 0.67f, rd),
                            rna_if((t1 * t1 - a.off) / a.div, rd));
          }
        }
      }
    } else if constexpr (EPI == CW_DX) {
      // columns (col, col + 1) of dx are (a_f, s_f) of feature f = col / 2 (relu: features col, col + 1)
#pragma unroll
      for (int j = 0; j < BN / 8; ++j) {
        const int col = n0 + 8 * j + col_in_tile;
        const bool cv = col < a.N;
        float s0 = 0.f, s1 = 0.f;
#pragma unroll
        for (int r = 0; r < 2; ++r) {
          const int row = row0 + 8 * r;
          float dz0 = 0.f, dz1 = 0.f;
          if (cv && row < a.npix) {
            const float dx0 = d[0][4 * j + 2 * r], dx1 = d[0][4 * j + 2 * r + 1];
            if (RELU) {
              dz0 = __ldg(a.zT_in + (size_t)col * a.ld + row) > 0.f ? dx0 / 0.58f : 0.f;
              dz1 = __ldg(a.zT_in + (size_t)(col + 1) * a.ld + row) > 0.f ? dx1 / 0.58f : 0.f;
            } else {
              const float zz = __ldg(a.zT_in + (size_t)(col >> 1) * a.ld + row), tt = atanf(zz);
              dz0 = (dx0 / 0.67f + dx1 * (2.f * tt) / a.div) / (1.f + zz * zz);
            }
          }
          if (cv && row < a.M) {     // rows past the frame get zeros: the next products read them
            const bool rd = a.round_out;
            if (RELU) {
              a.dzT_out[(size_t)col * a.ld + row] = rna_if(dz0, rd);
              a.dzT_out[(size_t)(col + 1) * a.ld + row] = rna_if(dz1, rd);
              if (a.dz_out) *reinterpret_cast<float2*>(a.dz_out + (size_t)row * a.nf + col) = make_float2(rna(dz0), rna(dz1));
            } else {
              a.dzT_out[(size_t)(col >> 1) * a.ld + row] = rna_if(dz0, rd);
              if (a.dz_out) a.dz_out[(size_t)row * a.nf + (col >> 1)] = rna(dz0);
            }
          }
          s0 += dz0; s1 += dz1;
        }
        if (a.part) {       // db_{l-1}: the unrounded dz summed over this warp's 16 rows, in a fixed order
#pragma unroll
          for (int o = 4; o < 32; o <<= 1) {
            s0 += __shfl_xor_sync(0xffffffffu, s0, o);
            if (RELU) s1 += __shfl_xor_sync(0xffffffffu, s1, o);
          }
          if (lane < 4 && cv) {
            float* pr = a.part + (size_t)(t.m_blk * (GEMM_BM / 16) + (row_in_tile >> 4)) * a.nf;
            if (RELU) { pr[col] = s0; pr[col + 1] = s1; }
            else pr[col >> 1] = s0;
          }
        }
      }
    } else {   // CW_DW: this split's partial dW [NF][KH]
#pragma unroll
      for (int j = 0; j < BN / 8; ++j) {
        const int col = n0 + 8 * j + col_in_tile;
        if (col >= a.N) continue;
#pragma unroll
        for (int r = 0; r < 2; ++r) {
          const int row = row0 + 8 * r;
          if (row < a.M)
            *reinterpret_cast<float2*>(a.part + ((size_t)t.split * a.M + row) * a.N + col) = make_float2(d[0][4 * j + 2 * r], d[0][4 * j + 2 * r + 1]);
        }
      }
    }
  }
};

template <int BN, int EPI, bool RELU>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
k_cppnw_gemm(const __grid_constant__ CUtensorMap map_a, const __grid_constant__ CUtensorMap map_b, CppnWideArgs a) {
  gemm_body<BN, false>(map_a, map_b, CppnProblem<BN, EPI, RELU>{a});
}

// W' (and W'^T when wtp is given) of every hidden layer, rounded to TF32
__global__ void __launch_bounds__(256) k_cppnw_pack(CppnWeights P, int L, int nf, int kh, bool relu, float* __restrict__ wp,
                                                    float* __restrict__ wtp) {
  const int64_t per = (int64_t)nf * kh, n = (L - 1) * per;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int l = (int)(i / per), r = (int)(i - l * per), o = r / kh, ip = r - o * kh;
    const float v = rna(__ldg(P.w[l + 1] + (size_t)o * kh + cppnw_src_col(ip, nf, relu)));
    wp[i] = v;
    if (wtp) wtp[l * per + (int64_t)ip * nf + o] = v;
  }
}

// layer 0 in fp32 and its activation: x_1 [P][KH] in x' order; z_0 to zT when given
__global__ void __launch_bounds__(256) k_cppnw_l0(const float* __restrict__ coords, int64_t npix, int64_t hw, const float* __restrict__ W0,
                                                  const float* __restrict__ b0, int nf, int kh, bool relu, float off, float div, bool round,
                                                  float* __restrict__ x_out, float* __restrict__ zT, int64_t ld) {
  const int64_t n = npix * nf;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t p = i / nf;
    const int j = (int)(i - p * nf);
    float c0, c1;
    load_coords(coords, npix, hw, p, c0, c1);
    const float z = fmaf(__ldg(W0 + 2 * j + 1), c1, fmaf(__ldg(W0 + 2 * j), c0, __ldg(b0 + j)));
    if (zT) zT[(size_t)j * ld + p] = z;
    if (relu) {
      x_out[p * kh + j] = rna_if((fmaxf(z, 0.f) - 0.4f) / 0.58f, round);
    } else {
      const float t = atanf(z);
      *reinterpret_cast<float2*>(x_out + p * kh + 2 * j) = make_float2(rna_if(t / 0.67f, round), rna_if((t * t - off) / div, round));
    }
  }
}

// the output layer and the sigmoid in fp32, a warp per pixel; x_L in x' order, W_out read in place
__global__ void __launch_bounds__(256) k_cppnw_head(const float* __restrict__ x, int64_t npix, int64_t hw, const float* __restrict__ Wo,
                                                    const float* __restrict__ bo, int nf, int kh, bool relu, float* __restrict__ out) {
  const int lane = threadIdx.x & 31;
  const int64_t nw = (int64_t)gridDim.x * (blockDim.x >> 5);
  for (int64_t p = blockIdx.x * (int64_t)(blockDim.x >> 5) + (threadIdx.x >> 5); p < npix; p += nw) {
    float s[3] = {0.f, 0.f, 0.f};
    for (int ip = 2 * lane; ip < kh; ip += 64) {
      const float2 v = __ldg(reinterpret_cast<const float2*>(x + p * kh + ip));
      const int i0 = cppnw_src_col(ip, nf, relu), i1 = cppnw_src_col(ip + 1, nf, relu);
#pragma unroll
      for (int c = 0; c < 3; ++c) s[c] = fmaf(v.y, __ldg(Wo + c * kh + i1), fmaf(v.x, __ldg(Wo + c * kh + i0), s[c]));
    }
#pragma unroll
    for (int c = 0; c < 3; ++c) s[c] = warp_sum(s[c]);
    if (lane < 3) {
      const int64_t n = p / hw, q = p - n * hw;
      out[3 * n * hw + lane * hw + q] = 1.f / (1.f + expf(-(pick3(s, lane) + __ldg(bo + lane))));
    }
  }
}

// The output layer's backward, a warp per 16-pixel group (all Ppad / 16 groups: pixels past the frame write zeros). Lane
// takes features j = lane + 32 k. Writes dz_{L-1} ([Ppad][NF] rounded when dz_out is given, [NF][Ppad] rounded when
// round_dz) and the group's partial row: dW_out [3][KH] (original column order), db_out at 3 KH, db_{L-1} at 3 KH + 8.
__global__ void __launch_bounds__(256) k_cppnw_head_bwd(const float* __restrict__ x, int64_t npix, int64_t hw, int64_t ld,
                                                        const float* __restrict__ Wo, const float* __restrict__ bo,
                                                        const float* __restrict__ gout, const float* __restrict__ zT, int nf, int kh,
                                                        bool relu, float off, float div, bool round_dz, float* __restrict__ dz_out,
                                                        float* __restrict__ dzT, float* __restrict__ part, int pw) {
  const int lane = threadIdx.x & 31;
  const int64_t grp = blockIdx.x * (int64_t)(blockDim.x >> 5) + (threadIdx.x >> 5);
  float aw[3][2][8], ab[8], ao[3] = {0.f, 0.f, 0.f};
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    ab[k] = 0.f;
#pragma unroll
    for (int c = 0; c < 3; ++c) aw[c][0][k] = aw[c][1][k] = 0.f;
  }
  for (int q = 0; q < 16; ++q) {
    const int64_t p = grp * 16 + q;
    if (p >= npix) {
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        const int j = lane + 32 * k;
        if (j < nf) {
          dzT[(size_t)j * ld + p] = 0.f;
          if (dz_out) dz_out[p * nf + j] = 0.f;
        }
      }
      continue;
    }
    float xv[2][8], s[3] = {0.f, 0.f, 0.f};
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      const int j = lane + 32 * k;
      xv[0][k] = xv[1][k] = 0.f;
      if (j < nf) {
        if (relu) {
          xv[0][k] = __ldg(x + p * kh + j);
        } else {
          const float2 v = __ldg(reinterpret_cast<const float2*>(x + p * kh + 2 * j));
          xv[0][k] = v.x; xv[1][k] = v.y;
        }
#pragma unroll
        for (int c = 0; c < 3; ++c) {
          s[c] = fmaf(xv[0][k], __ldg(Wo + c * kh + j), s[c]);
          if (!relu) s[c] = fmaf(xv[1][k], __ldg(Wo + c * kh + nf + j), s[c]);
        }
      }
    }
    const int64_t n = p / hw, qq = p - n * hw;
    float dzo[3];
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const float y = 1.f / (1.f + expf(-(warp_sum(s[c]) + __ldg(bo + c))));
      dzo[c] = __ldg(gout + 3 * n * hw + c * hw + qq) * (y * (1.f - y));
      ao[c] += dzo[c];
    }
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      const int j = lane + 32 * k;
      if (j < nf) {
        const float dx0 = dzo[0] * __ldg(Wo + j) + dzo[1] * __ldg(Wo + kh + j) + dzo[2] * __ldg(Wo + 2 * kh + j);
        const float zz = __ldg(zT + (size_t)j * ld + p);
        float dz;
        if (relu) {
          dz = zz > 0.f ? dx0 / 0.58f : 0.f;
        } else {
          const float dx1 = dzo[0] * __ldg(Wo + nf + j) + dzo[1] * __ldg(Wo + kh + nf + j) + dzo[2] * __ldg(Wo + 2 * kh + nf + j);
          dz = (dx0 / 0.67f + dx1 * (2.f * atanf(zz)) / div) / (1.f + zz * zz);
        }
        dzT[(size_t)j * ld + p] = rna_if(dz, round_dz);
        if (dz_out) dz_out[p * nf + j] = rna(dz);
        ab[k] += dz;
#pragma unroll
        for (int c = 0; c < 3; ++c) {
          aw[c][0][k] = fmaf(dzo[c], xv[0][k], aw[c][0][k]);
          aw[c][1][k] = fmaf(dzo[c], xv[1][k], aw[c][1][k]);
        }
      }
    }
  }
  float* pr = part + grp * pw;
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    const int j = lane + 32 * k;
    if (j < nf) {
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        pr[c * kh + j] = aw[c][0][k];
        if (!relu) pr[c * kh + nf + j] = aw[c][1][k];
      }
      pr[3 * kh + 8 + j] = ab[k];
    }
  }
  if (lane < 3) pr[3 * kh + lane] = pick3(ao, lane);
}

// x_l = act(z_{l-1}) rounded, pixel-contiguous in the original column order and split-major: [S][KHP][chunk] (rows KH .. KHP
// of a split are never read into a stored column); pixels past the frame are zeros
__global__ void __launch_bounds__(256) k_cppnw_actT(const float* __restrict__ zT, int64_t npix, int64_t ld, int nf, int khp, int chunk,
                                                    bool relu, float off, float div, float* __restrict__ xT) {
  const int64_t n = (int64_t)nf * ld;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int j = (int)(i / ld);
    const int64_t p = i - j * ld, s = p / chunk, kl = p - s * chunk;
    float v0 = 0.f, v1 = 0.f;
    if (p < npix) {
      const float z = __ldg(zT + i);
      if (relu) {
        v0 = rna((fmaxf(z, 0.f) - 0.4f) / 0.58f);
      } else {
        const float t = atanf(z);
        v0 = rna(t / 0.67f); v1 = rna((t * t - off) / div);
      }
    }
    xT[(s * khp + j) * chunk + kl] = v0;
    if (!relu) xT[(s * khp + nf + j) * chunk + kl] = v1;
  }
}

// dW_0 [NF][2], db_0 from dz_0 [NF][Ppad] in fp32, a block per feature, summed in a fixed order
__global__ void __launch_bounds__(256) k_cppnw_l0_bwd(const float* __restrict__ dzT, const float* __restrict__ coords, int64_t npix,
                                                      int64_t hw, int64_t ld, float* __restrict__ dW0, float* __restrict__ db0) {
  __shared__ float sh[3][256];
  const int o = blockIdx.x, tid = threadIdx.x;
  float s0 = 0.f, s1 = 0.f, sb = 0.f;
  for (int64_t p = tid; p < npix; p += blockDim.x) {
    const float dz = __ldg(dzT + (size_t)o * ld + p);
    float c0, c1;
    load_coords(coords, npix, hw, p, c0, c1);
    s0 = fmaf(dz, c0, s0); s1 = fmaf(dz, c1, s1); sb += dz;
  }
  sh[0][tid] = s0; sh[1][tid] = s1; sh[2][tid] = sb;
  __syncthreads();
  for (int w = 128; w > 0; w >>= 1) {
    if (tid < w) for (int k = 0; k < 3; ++k) sh[k][tid] += sh[k][tid + w];
    __syncthreads();
  }
  if (tid == 0) { dW0[2 * o] = sh[0][0]; dW0[2 * o + 1] = sh[1][0]; db0[o] = sh[2][0]; }
}

// out[c] = sum over rows r of in[r][c] in a fixed order: block (32 columns x 8 row lanes) over CPPNW_CH rows. With tmp, one
// sum per row chunk goes to tmp[chunk][c]; without, the single chunk's sum goes to the segment of `seg` holding column c
// (a segment with a NULL pointer is not stored).
struct CppnSegs { float* p[4]; int off[5]; int n; };
__global__ void __launch_bounds__(256) k_cppnw_colsum(const float* __restrict__ in, int64_t rows, int cols, CppnSegs seg,
                                                      float* __restrict__ tmp) {
  __shared__ float sh[8][33];
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5, c = blockIdx.x * 32 + tx;
  const int64_t r0 = (int64_t)blockIdx.y * CPPNW_CH, r1 = r0 + CPPNW_CH < rows ? r0 + CPPNW_CH : rows;
  float s = 0.f;
  if (c < cols)
    for (int64_t r = r0 + ty; r < r1; r += 8) s += __ldg(in + r * cols + c);
  sh[ty][tx] = s;
  __syncthreads();
  if (ty == 0 && c < cols) {
    float v = sh[0][tx];
#pragma unroll
    for (int k = 1; k < 8; ++k) v += sh[k][tx];
    if (tmp) {
      tmp[(int64_t)blockIdx.y * cols + c] = v;
    } else {
      int k = 0;
      while (k + 1 < seg.n && c >= seg.off[k + 1]) ++k;
      if (seg.p[k]) seg.p[k][c - seg.off[k]] = v;
    }
  }
}

}  // namespace aph

using namespace aph;

struct aph_cppn {
  int nf, layers, act;
  Scratch partial, zbuf;     // nf <= 64
  Scratch wide;              // nf >= 72: every buffer of the wide path (cppnw_floats)
};

namespace {

struct CppnCall {
  aph_cppn* h;
  const float* coords;
  int64_t npix, hw;
  CppnWeights P;
  float off, div;
  cudaStream_t st;
};

CppnCall make_call(aph_cppn* h, const float* coords, int N, int H, int W, const float* const* params, void* stream) {
  CppnCall c;
  c.h = h; c.coords = coords;
  c.hw = (int64_t)H * W; c.npix = (int64_t)N * c.hw;
  for (int l = 0; l <= h->layers; ++l) { c.P.w[l] = params[2 * l]; c.P.b[l] = params[2 * l + 1]; }
  c.off = h->act == CPPN_UNBIAS ? 0.45f : 0.f;
  c.div = h->act == CPPN_UNBIAS ? 0.396f : 0.6f;
  c.st = (cudaStream_t)stream;
  return c;
}

template <int NF, bool RELU>
int cppn_fwd(const CppnCall& c, float* out) {
  const int64_t mtiles = (c.npix + 15) / 16;
  const int blocks = (int)std::min<int64_t>((mtiles + CPPN_WARPS - 1) / CPPN_WARPS, (int64_t)num_sms() * 16);
  k_cppn_fwd<NF, RELU><<<blocks, 32 * CPPN_WARPS, 0, c.st>>>(c.coords, c.npix, c.hw, c.h->layers, c.P, c.off, c.div, out);
  APH_LAUNCH_OK();
  return 0;
}

template <int NF, bool RELU>
int cppn_bwd(const CppnCall& c, const float* grad_out, float* const* dparams) {
  constexpr int KH = RELU ? NF : 2 * NF;
  aph_cppn* h = c.h;
  const int L = h->layers;
  const size_t stage = (size_t)CPPN_TP * (cppn_stride(KH) + cppn_stride(NF)) * sizeof(float);
  const size_t zbytes = (size_t)CPPN_TP * NF * L * sizeof(float);
  const bool z_in_smem = stage + zbytes <= CPPN_SMEM_CAP;
  const size_t smem = stage + (z_in_smem ? zbytes : 0);
  auto kern = k_cppn_bwd<NF, RELU>;
  if (int e = smem_at_least((const void*)kern, smem)) return e;
  int per_sm = 0;
  APH_CUDA_OK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, 32 * CPPN_WARPS, smem));
  APH_REQUIRE(per_sm > 0, "aph_cppn_bwd: the backward kernel does not fit on this device (%zu bytes of shared memory)", smem);
  const int ptotal = cppn_total(NF, KH, L);
  const int64_t ntiles = (c.npix + CPPN_TP - 1) / CPPN_TP;
  int64_t G = std::min<int64_t>(ntiles, (int64_t)per_sm * num_sms());
  G = std::max<int64_t>(1, std::min<int64_t>(G, (int64_t)(CPPN_PARTIAL_CAP / ((size_t)ptotal * sizeof(float)))));
  if (h->partial.grow((size_t)G * ptotal * sizeof(float), c.st)) return 1;
  float* zglob = nullptr;
  if (!z_in_smem) {
    if (h->zbuf.grow((size_t)G * zbytes, c.st)) return 1;
    zglob = h->zbuf.p;
  }
  kern<<<(int)G, 32 * CPPN_WARPS, smem, c.st>>>(c.coords, c.npix, c.hw, L, c.P, c.off, c.div, grad_out, zglob, h->partial.p, ptotal,
                                                ntiles);
  APH_LAUNCH_OK();
  CppnGradOut o;
  const int nt = 2 * (L + 1);
  for (int l = 0; l <= L; ++l) {
    o.p[2 * l] = dparams[2 * l];
    o.p[2 * l + 1] = dparams[2 * l + 1];
    o.off[2 * l] = cppn_off_w(NF, KH, l);
    o.off[2 * l + 1] = cppn_off_b(NF, KH, l, L);
  }
  o.off[nt] = ptotal;
  k_cppn_reduce<<<(ptotal + 255) / 256, 256, 0, c.st>>>(h->partial.p, (int)G, ptotal, nt, o);
  APH_LAUNCH_OK();
  return 0;
}

// ---- wide path, host side
// Geometry of one call. Pixels are padded to Ppad = S chunk: the weight gradient splits them into S chunks of `chunk` pixels
// (at least CPPNW_CHUNK, at most CPPNW_MAX_SPLITS chunks), and every pixel-contiguous buffer has Ppad columns.
struct WideGeom {
  int nf, kh, L;
  bool relu;
  int64_t P, Ppad, R;       // pixels, padded pixels, 16-pixel groups
  int chunk, S;
  int bnk, ntk, khp;        // GEMM tile width over KH, tiles, KH padded to them
  int pw;                   // width of a head partial row: dW_out [3][KH], db_out (8 slots), db_{L-1} [NF]
};

WideGeom wide_geom(int nf, int L, int act, int64_t P) {
  WideGeom g;
  g.nf = nf; g.L = L; g.relu = act == CPPN_RELU; g.kh = g.relu ? nf : 2 * nf; g.P = P;
  const int64_t per = (P + CPPNW_MAX_SPLITS - 1) / CPPNW_MAX_SPLITS;
  g.chunk = (int)std::max<int64_t>(CPPNW_CHUNK, (per + 127) / 128 * 128);
  g.S = (int)((P + g.chunk - 1) / g.chunk);
  g.Ppad = (int64_t)g.S * g.chunk;
  g.R = g.Ppad / 16;
  g.bnk = g.kh <= 128 ? 128 : 256;
  g.ntk = (g.kh + g.bnk - 1) / g.bnk;
  g.khp = g.ntk * g.bnk;
  g.pw = 3 * g.kh + 8 + nf;
  return g;
}

// Regions of the handle buffer, in floats (include/aphb200.h states the same sum): the forward uses the first three.
struct WideBufs { float *xa, *xb, *wp, *wtp, *zT, *xT, *dzT, *part, *tmp; };
constexpr int CPPNW_REGIONS = 9;
void cppnw_regions(const WideGeom& g, int64_t (&n)[CPPNW_REGIONS]) {
  const int64_t nk = (int64_t)g.nf * g.kh;
  n[0] = n[1] = g.Ppad * g.kh;                                      // x_l (and dz_l in the backward), ping-pong
  n[2] = n[3] = (g.L - 1) * nk;                                     // W', W'^T
  n[4] = (int64_t)g.L * g.nf * g.Ppad;                              // z_0 .. z_{L-1}
  n[5] = (int64_t)g.khp * g.Ppad;                                   // x_l split-major
  n[6] = (int64_t)g.nf * g.Ppad;                                    // dz_l pixel-contiguous
  n[7] = std::max<int64_t>(g.R * g.pw, (int64_t)g.S * nk);          // partials
  n[8] = 2 * ((g.R + CPPNW_CH - 1) / CPPNW_CH) * g.pw;              // column-sum passes
}
int64_t cppnw_floats(const WideGeom& g, bool bwd) {
  int64_t n[CPPNW_REGIONS], total = 0;
  cppnw_regions(g, n);
  for (int i = 0; i < (bwd ? CPPNW_REGIONS : 3); ++i) total += n[i];
  return total;
}

int cppnw_alloc(aph_cppn* h, const WideGeom& g, bool bwd, cudaStream_t st, WideBufs& b, const char* what) {
  const size_t need = (size_t)cppnw_floats(g, bwd) * sizeof(float);
  if (h->wide.grow(need, st)) {
    cudaGetLastError();          // a failed cudaMalloc is not sticky: clear it so that later launches are not blamed
    aph::set_error("%s: %zu bytes of device scratch could not be allocated (nf %d, %d layers, %lld pixels)", what, need, g.nf, g.L,
                   (long long)g.P);
    return 1;
  }
  int64_t n[CPPNW_REGIONS];
  cppnw_regions(g, n);
  float** dst[CPPNW_REGIONS] = {&b.xa, &b.xb, &b.wp, &b.wtp, &b.zT, &b.xT, &b.dzT, &b.part, &b.tmp};
  float* p = h->wide.p;
  for (int i = 0; i < CPPNW_REGIONS; ++i) {
    *dst[i] = (bwd || i < 3) ? p : nullptr;
    p += (bwd || i < 3) ? n[i] : 0;
  }
  return 0;
}

// one GEMM: A [a_rows][a_k] and B [b_rows][b_k] fp32 (rows a_ld / b_ld floats apart) through their 16-bit views
template <int BN, int EPI, bool RELU>
int cppnw_gemm(const float* A, int a_rows, int a_k, int64_t a_ld, const float* B, int b_rows, int b_k, int64_t b_ld, const CppnWideArgs& a,
               cudaStream_t st) {
  auto kern = k_cppnw_gemm<BN, EPI, RELU>;
  if (int e = smem_at_least((const void*)kern, GemmCfg<BN>::SMEM)) return e;
  CUtensorMap ma, mb;
  if (int e = make_tmap_bf16(&ma, A, a_rows, 2 * a_k, GEMM_BM, 2 * a_ld)) return e;
  if (int e = make_tmap_bf16(&mb, B, b_rows, 2 * b_k, BN, 2 * b_ld)) return e;
  const int tiles = a.splits * a.m_tiles * a.n_tiles;
  kern<<<std::min(tiles, num_sms()), GEMM_THREADS, (size_t)GemmCfg<BN>::SMEM, st>>>(ma, mb, a);
  APH_LAUNCH_OK();
  return 0;
}

template <int EPI, bool RELU>
int cppnw_gemm_bn(int bn, const float* A, int a_rows, int a_k, int64_t a_ld, const float* B, int b_rows, int b_k, int64_t b_ld,
                  const CppnWideArgs& a, cudaStream_t st) {
  return bn == 128 ? cppnw_gemm<128, EPI, RELU>(A, a_rows, a_k, a_ld, B, b_rows, b_k, b_ld, a, st)
                   : cppnw_gemm<256, EPI, RELU>(A, a_rows, a_k, a_ld, B, b_rows, b_k, b_ld, a, st);
}

int cppnw_colsum(const float* in, int64_t rows, int cols, const CppnSegs& seg, float* tmp, cudaStream_t st) {
  float* bufs[2] = {tmp, tmp + (rows + CPPNW_CH - 1) / CPPNW_CH * cols};
  int pi = 0;
  const unsigned gx = (unsigned)((cols + 31) / 32);
  while (rows > CPPNW_CH) {
    const int64_t nch = (rows + CPPNW_CH - 1) / CPPNW_CH;
    k_cppnw_colsum<<<dim3(gx, (unsigned)nch), 256, 0, st>>>(in, rows, cols, seg, bufs[pi]);
    APH_LAUNCH_OK();
    in = bufs[pi]; rows = nch; pi ^= 1;
  }
  k_cppnw_colsum<<<dim3(gx, 1), 256, 0, st>>>(in, rows, cols, seg, nullptr);
  APH_LAUNCH_OK();
  return 0;
}

CppnSegs segs1(float* p, int n) {
  CppnSegs s{};
  s.p[0] = p; s.off[0] = 0; s.off[1] = n; s.n = 1;
  return s;
}

// The forward of every layer but the output one: pack, layer 0, the hidden GEMMs. z_l goes to b.zT when `save`. Returns
// the buffer holding x_L in *xl (the other one is free).
template <bool RELU>
int cppnw_trunk(const CppnCall& c, const WideGeom& g, const WideBufs& b, bool save, float** xl) {
  const int L = g.L;
  if (L > 1) {
    k_cppnw_pack<<<stride_blocks((int64_t)(L - 1) * g.nf * g.kh, 8), 256, 0, c.st>>>(c.P, L, g.nf, g.kh, RELU, b.wp, save ? b.wtp : nullptr);
    APH_LAUNCH_OK();
  }
  k_cppnw_l0<<<stride_blocks(g.P * g.nf, 8), 256, 0, c.st>>>(c.coords, g.P, c.hw, c.P.w[0], c.P.b[0], g.nf, g.kh, RELU, c.off, c.div, L > 1, b.xa,
                                                             save ? b.zT : nullptr, g.Ppad);
  APH_LAUNCH_OK();
  float *x = b.xa, *y = b.xb;
  const int bnf = g.nf <= 128 ? 128 : 256;
  for (int l = 1; l < L; ++l) {
    CppnWideArgs a{};
    a.M = (int)g.P; a.N = g.nf; a.m_tiles = (int)((g.P + GEMM_BM - 1) / GEMM_BM); a.n_tiles = 1; a.splits = 1;
    a.kblocks = (g.kh + 31) / 32; a.nf = g.nf; a.kh = g.kh; a.npix = g.P; a.ld = g.Ppad; a.off = c.off; a.div = c.div;
    a.bias = c.P.b[l]; a.x_out = y; a.round_out = l + 1 < L; a.zT = save ? b.zT + (int64_t)l * g.nf * g.Ppad : nullptr;
    if (int e = cppnw_gemm_bn<CW_FWD, RELU>(bnf, x, (int)g.P, g.kh, g.kh, b.wp + (int64_t)(l - 1) * g.nf * g.kh, g.nf, g.kh, g.kh, a, c.st))
      return e;
    std::swap(x, y);
  }
  *xl = x;
  return 0;
}

template <bool RELU>
int cppn_fwd_wide(const CppnCall& c, float* out) {
  const WideGeom g = wide_geom(c.h->nf, c.h->layers, c.h->act, c.npix);
  WideBufs b;
  if (int e = cppnw_alloc(c.h, g, false, c.st, b, "aph_cppn_fwd")) return e;
  float* xl = nullptr;
  if (int e = cppnw_trunk<RELU>(c, g, b, false, &xl)) return e;
  k_cppnw_head<<<stride_blocks(g.P * 32, 8), 256, 0, c.st>>>(xl, g.P, c.hw, c.P.w[g.L], c.P.b[g.L], g.nf, g.kh, RELU, out);
  APH_LAUNCH_OK();
  return 0;
}

template <bool RELU>
int cppn_bwd_wide(const CppnCall& c, const float* grad_out, float* const* dparams) {
  const WideGeom g = wide_geom(c.h->nf, c.h->layers, c.h->act, c.npix);
  const int L = g.L, nf = g.nf, kh = g.kh;
  WideBufs b;
  if (int e = cppnw_alloc(c.h, g, true, c.st, b, "aph_cppn_bwd")) return e;
  float* x = nullptr;
  if (int e = cppnw_trunk<RELU>(c, g, b, true, &x)) return e;
  float* dz = x == b.xa ? b.xb : b.xa;     // dz_l [Ppad][NF] ping-pongs through the two activation buffers
  float* dz_other = x;
  // the output layer: dW_out, db_out, and dz_{L-1} with its db
  k_cppnw_head_bwd<<<(unsigned)(g.R / 8), 256, 0, c.st>>>(x, g.P, c.hw, g.Ppad, c.P.w[L], c.P.b[L], grad_out,
                                                          b.zT + (int64_t)(L - 1) * nf * g.Ppad, nf, kh, RELU, c.off, c.div, L > 1,
                                                          L > 1 ? dz : nullptr, b.dzT, b.part, g.pw);
  APH_LAUNCH_OK();
  {
    // partial row: dW_out | db_out | 5 unused slots | db_{L-1} (layer 0's db comes from k_cppnw_l0_bwd)
    CppnSegs sg{};
    sg.p[0] = dparams[2 * L]; sg.p[1] = dparams[2 * L + 1]; sg.p[2] = nullptr; sg.p[3] = L > 1 ? dparams[2 * L - 1] : nullptr;
    sg.off[0] = 0; sg.off[1] = 3 * kh; sg.off[2] = 3 * kh + 3; sg.off[3] = 3 * kh + 8; sg.off[4] = g.pw;
    sg.n = 4;
    if (int e = cppnw_colsum(b.part, g.R, g.pw, sg, b.tmp, c.st)) return e;
  }
  for (int l = L - 1; l >= 1; --l) {
    // dW_l = dz_l^T x_l over S pixel splits, then the fixed-order sum of the splits
    k_cppnw_actT<<<stride_blocks((int64_t)nf * g.Ppad, 8), 256, 0, c.st>>>(b.zT + (int64_t)(l - 1) * nf * g.Ppad, g.P, g.Ppad, nf, g.khp, g.chunk,
                                                                           RELU, c.off, c.div, b.xT);
    APH_LAUNCH_OK();
    CppnWideArgs w{};
    w.M = nf; w.N = kh; w.m_tiles = (nf + GEMM_BM - 1) / GEMM_BM; w.n_tiles = g.ntk; w.splits = g.S; w.kblocks = g.chunk / 32;
    w.chunk = g.chunk; w.nf = nf; w.kh = kh; w.npix = g.P; w.ld = g.Ppad; w.part = b.part;
    if (int e = cppnw_gemm_bn<CW_DW, false>(g.bnk, b.dzT, nf, (int)g.Ppad, g.Ppad, b.xT, g.S * g.khp, g.chunk, g.chunk, w, c.st)) return e;
    if (int e = cppnw_colsum(b.part, g.S, nf * kh, segs1(dparams[2 * l], nf * kh), b.tmp, c.st)) return e;
    // dx_l = dz_l W_l; its epilogue forms dz_{l-1} (and db_{l-1} partials above layer 0)
    CppnWideArgs a{};
    a.M = (int)g.Ppad; a.N = kh; a.m_tiles = (int)(g.Ppad / GEMM_BM); a.n_tiles = g.ntk; a.splits = 1; a.kblocks = (nf + 31) / 32;
    a.nf = nf; a.kh = kh; a.npix = g.P; a.ld = g.Ppad; a.off = c.off; a.div = c.div; a.round_out = l > 1;
    a.zT_in = b.zT + (int64_t)(l - 1) * nf * g.Ppad; a.dz_out = l > 1 ? dz_other : nullptr; a.dzT_out = b.dzT;
    a.part = l > 1 ? b.part : nullptr;
    if (int e = cppnw_gemm_bn<CW_DX, RELU>(g.bnk, dz, (int)g.Ppad, nf, nf, b.wtp + (int64_t)(l - 1) * nf * kh, kh, nf, nf, a, c.st)) return e;
    if (l > 1)
      if (int e = cppnw_colsum(b.part, g.R, nf, segs1(dparams[2 * l - 1], nf), b.tmp, c.st)) return e;
    std::swap(dz, dz_other);
  }
  k_cppnw_l0_bwd<<<nf, 256, 0, c.st>>>(b.dzT, c.coords, g.P, c.hw, g.Ppad, dparams[0], dparams[1]);
  APH_LAUNCH_OK();
  return 0;
}

#define APH_CPPN_DISPATCH(FN, ...)                                                                \
  switch (h->nf) {                                                                                \
    case 8: return h->act == CPPN_RELU ? FN<8, true>(__VA_ARGS__) : FN<8, false>(__VA_ARGS__);    \
    case 16: return h->act == CPPN_RELU ? FN<16, true>(__VA_ARGS__) : FN<16, false>(__VA_ARGS__); \
    case 24: return h->act == CPPN_RELU ? FN<24, true>(__VA_ARGS__) : FN<24, false>(__VA_ARGS__); \
    case 32: return h->act == CPPN_RELU ? FN<32, true>(__VA_ARGS__) : FN<32, false>(__VA_ARGS__); \
    case 40: return h->act == CPPN_RELU ? FN<40, true>(__VA_ARGS__) : FN<40, false>(__VA_ARGS__); \
    case 48: return h->act == CPPN_RELU ? FN<48, true>(__VA_ARGS__) : FN<48, false>(__VA_ARGS__); \
    case 56: return h->act == CPPN_RELU ? FN<56, true>(__VA_ARGS__) : FN<56, false>(__VA_ARGS__); \
    case 64: return h->act == CPPN_RELU ? FN<64, true>(__VA_ARGS__) : FN<64, false>(__VA_ARGS__); \
    default: return h->act == CPPN_RELU ? FN##_wide<true>(__VA_ARGS__) : FN##_wide<false>(__VA_ARGS__); \
  }

int check_call(const aph_cppn* h, const float* coords, int N, int H, int W, const float* const* params, const char* what) {
  APH_REQUIRE(h && coords && params && N > 0 && H > 0 && W > 0, "%s: bad arguments", what);
  for (int i = 0; i < 2 * (h->layers + 1); ++i) {
    APH_REQUIRE(params[i], "%s: parameter %d is NULL", what, i);
    APH_REQUIRE(((uintptr_t)params[i] & 7) == 0, "%s: parameter %d is not 8-byte aligned", what, i);
  }
  return 0;
}

}  // namespace

extern "C" int aph_cppn_create(aph_cppn** handle, int nf, int layers, int act) {
  APH_REQUIRE(handle, "aph_cppn_create: bad arguments");
  APH_REQUIRE(nf >= 8 && nf <= 256 && nf % 8 == 0, "aph_cppn_create: nf = %d is not supported: nf must be a multiple of 8 in [8, 256]", nf);
  APH_REQUIRE(layers >= 1 && layers <= CPPN_MAX_LAYERS, "aph_cppn_create: layers = %d is not supported: layers must be in [1, %d]",
              layers, CPPN_MAX_LAYERS);
  APH_REQUIRE(act == CPPN_UNBIAS || act == CPPN_COMP || act == CPPN_RELU,
              "aph_cppn_create: act = %d is not one of 0 (unbias), 1 (comp), 2 (relu)", act);
  aph_cppn* h = new aph_cppn();
  h->nf = nf; h->layers = layers; h->act = act;
  *handle = h;
  return 0;
}

extern "C" int aph_cppn_destroy(aph_cppn* h) {
  delete h;
  return 0;
}

extern "C" int64_t aph_cppn_bytes(const aph_cppn* h) { return h ? (int64_t)(h->partial.bytes + h->zbuf.bytes + h->wide.bytes) : 0; }

extern "C" int aph_cppn_fwd(aph_cppn* h, const float* coords, int N, int H, int W, const float* const* params, float* out,
                            void* stream) {
  if (int rc = check_call(h, coords, N, H, W, params, "aph_cppn_fwd")) return rc;
  APH_REQUIRE(out, "aph_cppn_fwd: bad arguments");
  const CppnCall c = make_call(h, coords, N, H, W, params, stream);
  APH_CPPN_DISPATCH(cppn_fwd, c, out);
}

extern "C" int aph_cppn_bwd(aph_cppn* h, const float* coords, int N, int H, int W, const float* const* params, const float* grad_out,
                            float* const* dparams, void* stream) {
  if (int rc = check_call(h, coords, N, H, W, params, "aph_cppn_bwd")) return rc;
  APH_REQUIRE(grad_out && dparams, "aph_cppn_bwd: bad arguments");
  for (int i = 0; i < 2 * (h->layers + 1); ++i) APH_REQUIRE(dparams[i], "aph_cppn_bwd: gradient %d is NULL", i);
  const CppnCall c = make_call(h, coords, N, H, W, params, stream);
  APH_CPPN_DISPATCH(cppn_bwd, c, grad_out, dparams);
}
