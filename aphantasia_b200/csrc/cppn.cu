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
#include "aph_common.cuh"
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

}  // namespace aph

using namespace aph;

struct aph_cppn {
  int nf, layers, act;
  Scratch partial, zbuf;
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
int cppn_fwd_t(const CppnCall& c, float* out) {
  const int64_t mtiles = (c.npix + 15) / 16;
  const int blocks = (int)std::min<int64_t>((mtiles + CPPN_WARPS - 1) / CPPN_WARPS, (int64_t)num_sms() * 16);
  k_cppn_fwd<NF, RELU><<<blocks, 32 * CPPN_WARPS, 0, c.st>>>(c.coords, c.npix, c.hw, c.h->layers, c.P, c.off, c.div, out);
  APH_LAUNCH_OK();
  return 0;
}

template <int NF, bool RELU>
int cppn_bwd_t(const CppnCall& c, const float* grad_out, float* const* dparams) {
  constexpr int KH = RELU ? NF : 2 * NF;
  aph_cppn* h = c.h;
  const int L = h->layers;
  const size_t stage = (size_t)CPPN_TP * (cppn_stride(KH) + cppn_stride(NF)) * sizeof(float);
  const size_t zbytes = (size_t)CPPN_TP * NF * L * sizeof(float);
  const bool z_in_smem = stage + zbytes <= CPPN_SMEM_CAP;
  const size_t smem = stage + (z_in_smem ? zbytes : 0);
  auto kern = k_cppn_bwd<NF, RELU>;
  APH_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
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
    default: APH_REQUIRE(false, "aph_cppn: nf = %d is not supported", h->nf);                     \
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

extern "C" int aph_cppn_create(int nf, int layers, int act, aph_cppn** handle) {
  APH_REQUIRE(handle, "aph_cppn_create: bad arguments");
  APH_REQUIRE(nf >= 8 && nf <= 64 && nf % 8 == 0, "aph_cppn_create: nf = %d is not supported: nf must be a multiple of 8 in [8, 64]", nf);
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
  if (h) {
    if (h->partial.p) cudaFree(h->partial.p);
    if (h->zbuf.p) cudaFree(h->zbuf.p);
    delete h;
  }
  return 0;
}

extern "C" int aph_cppn_fwd(aph_cppn* h, const float* coords, int N, int H, int W, const float* const* params, float* out,
                            void* stream) {
  if (int rc = check_call(h, coords, N, H, W, params, "aph_cppn_fwd")) return rc;
  APH_REQUIRE(out, "aph_cppn_fwd: bad arguments");
  const CppnCall c = make_call(h, coords, N, H, W, params, stream);
  APH_CPPN_DISPATCH(cppn_fwd_t, c, out);
}

extern "C" int aph_cppn_bwd(aph_cppn* h, const float* coords, int N, int H, int W, const float* const* params, const float* grad_out,
                            float* const* dparams, void* stream) {
  if (int rc = check_call(h, coords, N, H, W, params, "aph_cppn_bwd")) return rc;
  APH_REQUIRE(grad_out && dparams, "aph_cppn_bwd: bad arguments");
  for (int i = 0; i < 2 * (h->layers + 1); ++i) APH_REQUIRE(dparams[i], "aph_cppn_bwd: gradient %d is NULL", i);
  const CppnCall c = make_call(h, coords, N, H, W, params, stream);
  APH_CPPN_DISPATCH(cppn_bwd_t, c, grad_out, dparams);
}
