// vit_ops.cu -- the non-GEMM kernels of the CLIP ViT-B image encoder, forward and data-gradient.
//
// Restates OpenAI clip/model.py VisionTransformer (third-party; SURVEY.md A5): patchify (conv1 with
// stride = kernel is an im2col permutation), cls/pos embedding + ln_pre, LayerNorm (fp32 statistics),
// and their backward passes (no weight gradients). The attention core is in vit_attn_tc.cuh and vit_attn_stream.cuh.
// Token rows are sample-major: row = s*T + t.  Width D = 128*NCH (template), so rows live in registers.
// Included by vit.cu and text.cu: the non-template kernels are static so that each translation unit has its own copy.
#pragma once
#include "tc_gemm.cuh"

namespace aph {

// Runs the statement with `constexpr int NCH = D / 128` for the row-in-registers kernels below (width 512 is the text tower's).
#define NCH_CASE(K, ...) case K: { constexpr int NCH = K; __VA_ARGS__; } break;
#define NCH_DISPATCH(D, ...)                                                           \
  switch ((D) / 128) {                                                                 \
    NCH_CASE(1, __VA_ARGS__) NCH_CASE(2, __VA_ARGS__) NCH_CASE(4, __VA_ARGS__) NCH_CASE(6, __VA_ARGS__) NCH_CASE(8, __VA_ARGS__) \
    default: set_error("vit: unsupported width %d", (D)); return 2;                    \
  }
// The same with RN50x4's text width 640 (NCH = 5) added, for the kernels the text towers run: the shared block forward's
// LayerNorm, the text embedding and pooling. The image towers' own kernels keep NCH_DISPATCH: aph_vit_create refuses 640.
#define NCH_DISPATCH_TEXT(D, ...)                                                      \
  switch ((D) / 128) {                                                                 \
    NCH_CASE(1, __VA_ARGS__) NCH_CASE(2, __VA_ARGS__) NCH_CASE(4, __VA_ARGS__) NCH_CASE(5, __VA_ARGS__) \
    NCH_CASE(6, __VA_ARGS__) NCH_CASE(8, __VA_ARGS__)                                 \
    default: set_error("text: unsupported width %d", (D)); return 2;                   \
  }

// ---------------------------------------------------------------------------------------------
// images fp32 [S,3,side,side] -> patches bf16 [S*g*g, patch_k(p)], col = c*p*p + py*p + px  (conv1 weight layout); side >= R = p*g:
// conv1 reads the top-left R x R window. The columns >= 3 p^2 of a row are padding (zeroed at create) and never written here.
// PAIRS = false (p % 16 == 0, rows without padding): 8 columns per thread. PAIRS = true (any even p, e.g. 14): 2 columns per
// thread, so that neither a patch-row boundary nor the end of the 3 p^2 columns falls inside one thread's vector.
template <bool PAIRS>
static __global__ void __launch_bounds__(256) k_patchify(const float* __restrict__ img, bf16* __restrict__ out, int S, int p, int g, int side) {
  if (PAIRS) {
    const int R = side, P3 = 3 * p * p, Kp = patch_k(p);
    const size_t total = (size_t)S * g * g * P3 / 2;
    for (size_t idx = blockIdx.x * (size_t)blockDim.x + threadIdx.x; idx < total; idx += (size_t)gridDim.x * blockDim.x) {
      const size_t e = idx * 2;
      const int row = (int)(e / P3), col = (int)(e - (size_t)row * P3);
      const int s = row / (g * g), pr = row - s * g * g, gy = pr / g, gx = pr - gy * g;
      const int c = col / (p * p), rem = col - c * p * p, py = rem / p, px = rem - py * p;
      const float* src = img + (((size_t)s * 3 + c) * R + gy * p + py) * R + gx * p + px;
      // px and p are even: with an even side the pair is 8-byte aligned
      const float2 a = (R & 1) == 0 ? __ldg(reinterpret_cast<const float2*>(src)) : make_float2(__ldg(src), __ldg(src + 1));
      *reinterpret_cast<__nv_bfloat162*>(out + (size_t)row * Kp + col) = __floats2bfloat162_rn(a.x, a.y);
    }
    return;
  }
  const int R = side, Kp = 3 * p * p;
  const size_t total = (size_t)S * g * g * Kp / 8;
  for (size_t idx = blockIdx.x * (size_t)blockDim.x + threadIdx.x; idx < total; idx += (size_t)gridDim.x * blockDim.x) {
    const size_t e = idx * 8;
    const int row = (int)(e / Kp), col = (int)(e - (size_t)row * Kp);
    const int s = row / (g * g), pr = row - s * g * g, gy = pr / g, gx = pr - gy * g;
    const int c = col / (p * p), rem = col - c * p * p, py = rem / p, px = rem - py * p;
    const float* src = img + (((size_t)s * 3 + c) * R + gy * p + py) * R + gx * p + px;
    float4 a, b;
    if ((R & 3) == 0) { a = __ldg(reinterpret_cast<const float4*>(src)); b = __ldg(reinterpret_cast<const float4*>(src) + 1); }
    else {                                          // rows of a side that is not a multiple of 4 are not 16-byte aligned
      a = make_float4(__ldg(src), __ldg(src + 1), __ldg(src + 2), __ldg(src + 3));
      b = make_float4(__ldg(src + 4), __ldg(src + 5), __ldg(src + 6), __ldg(src + 7));
    }
    __nv_bfloat162 p0 = __floats2bfloat162_rn(a.x, a.y), p1 = __floats2bfloat162_rn(a.z, a.w);
    __nv_bfloat162 p2 = __floats2bfloat162_rn(b.x, b.y), p3 = __floats2bfloat162_rn(b.z, b.w);
    uint4 u; u.x = *reinterpret_cast<uint32_t*>(&p0); u.y = *reinterpret_cast<uint32_t*>(&p1);
    u.z = *reinterpret_cast<uint32_t*>(&p2); u.w = *reinterpret_cast<uint32_t*>(&p3);
    *reinterpret_cast<uint4*>(out + e) = u;
  }
}

// planes [n,R,R] -> [n,side,side] (side >= R): the window at the top left, zeros in the margin
static __global__ void __launch_bounds__(256) k_window_expand(const float* __restrict__ src, float* __restrict__ dst, int n, int R, int side) {
  const size_t total = (size_t)n * side * side;
  for (size_t idx = blockIdx.x * (size_t)blockDim.x + threadIdx.x; idx < total; idx += (size_t)gridDim.x * blockDim.x) {
    const size_t plane = idx / ((size_t)side * side);
    const int rem = (int)(idx - plane * side * side), y = rem / side, x = rem - y * side;
    dst[idx] = (y < R && x < R) ? __ldg(src + (plane * R + y) * R + x) : 0.f;
  }
}

static __global__ void __launch_bounds__(256) k_f32_to_bf16(const float* __restrict__ in, bf16* __restrict__ out, size_t n) {
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
    out[i] = __float2bfloat16_rn(in[i]);
}

// ---------------------------------------------------------------------------------------------
// LayerNorm row helpers: one warp per row, width D (multiple of 128), each lane holds D/32 values.

struct RowStats { float mean, rstd; };

template <int N>
__device__ __forceinline__ RowStats row_stats(const float (&v)[N], int D) {
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < N; ++i) s += v[i];
  const float mean = warp_sum(s) / (float)D;
  float q = 0.f;
#pragma unroll
  for (int i = 0; i < N; ++i) { const float d = v[i] - mean; q += d * d; }
  const float var = warp_sum(q) / (float)D;
  return {mean, rsqrtf(var + 1e-5f)};
}

// lane owns float4 chunks: element index of chunk k = (k*32 + lane)*4
template <int N>
__device__ __forceinline__ void load_row(const float* __restrict__ row, float (&v)[N], int lane) {
#pragma unroll
  for (int k = 0; k < N / 4; ++k) {
    const float4 a = *reinterpret_cast<const float4*>(row + (k * 32 + lane) * 4);
    v[4 * k] = a.x; v[4 * k + 1] = a.y; v[4 * k + 2] = a.z; v[4 * k + 3] = a.w;
  }
}
// bf16 row -> fp32 registers (same lane ownership as load_row: chunk k holds elements (k*32 + lane)*4 .. +3)
template <int N>
__device__ __forceinline__ void load_row(const bf16* __restrict__ row, float (&v)[N], int lane) {
#pragma unroll
  for (int k = 0; k < N / 4; ++k) {
    const uint2 u = *reinterpret_cast<const uint2*>(row + (k * 32 + lane) * 4);
    const float2 a = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&u.x)), b = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&u.y));
    v[4 * k] = a.x; v[4 * k + 1] = a.y; v[4 * k + 2] = b.x; v[4 * k + 3] = b.y;
  }
}
template <int N>
__device__ __forceinline__ void store_row_f32(float* __restrict__ row, const float (&v)[N], int lane) {
#pragma unroll
  for (int k = 0; k < N / 4; ++k)
    *reinterpret_cast<float4*>(row + (k * 32 + lane) * 4) = make_float4(v[4 * k], v[4 * k + 1], v[4 * k + 2], v[4 * k + 3]);
}
template <int N>
__device__ __forceinline__ void store_row_bf16(bf16* __restrict__ row, const float (&v)[N], int lane) {
#pragma unroll
  for (int k = 0; k < N / 4; ++k) {
    __nv_bfloat162 p0 = __floats2bfloat162_rn(v[4 * k], v[4 * k + 1]), p1 = __floats2bfloat162_rn(v[4 * k + 2], v[4 * k + 3]);
    uint2 u; u.x = *reinterpret_cast<uint32_t*>(&p0); u.y = *reinterpret_cast<uint32_t*>(&p1);
    *reinterpret_cast<uint2*>(row + (k * 32 + lane) * 4) = u;
  }
}

// e = [cls; tok] + pos (saved), x0 = ln_pre(e). tok fp32 [S*(T-1), D].
template <int NCH>
__global__ void __launch_bounds__(256) k_embed_lnpre(const float* __restrict__ tok, const float* __restrict__ cls,
                                                     const float* __restrict__ pos, const float* __restrict__ gamma,
                                                     const float* __restrict__ beta, float* __restrict__ e_out,
                                                     float* __restrict__ x0, float* __restrict__ mean_out, float* __restrict__ rstd_out,
                                                     int S, int T, int D) {
  const int row = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (row >= S * T) return;
  const int s = row / T, t = row - s * T;
  constexpr int N = 4 * NCH;
  const float* src = (t == 0) ? cls : tok + ((size_t)s * (T - 1) + (t - 1)) * D;
  float v[N], pz[N];
  load_row(src, v, lane);
  load_row(pos + (size_t)t * D, pz, lane);
  #pragma unroll
  for (int i = 0; i < N; ++i) v[i] += pz[i];
  store_row_f32(e_out + (size_t)row * D, v, lane);
  const RowStats st = row_stats(v, D);
  float gm[N], bt[N];
  load_row(gamma, gm, lane); load_row(beta, bt, lane);
  #pragma unroll
  for (int i = 0; i < N; ++i) v[i] = (v[i] - st.mean) * st.rstd * gm[i] + bt[i];
  store_row_f32(x0 + (size_t)row * D, v, lane);
  if (lane == 0) { mean_out[row] = st.mean; rstd_out[row] = st.rstd; }
}

// y = LN(x) as bf16, x and y [rows, D].
template <int NCH>
__global__ void __launch_bounds__(256) k_ln_fwd(const float* __restrict__ x, const float* __restrict__ gamma,
                                                const float* __restrict__ beta, bf16* __restrict__ y, float* __restrict__ mean_out,
                                                float* __restrict__ rstd_out, int rows, int D) {
  const int row = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (row >= rows) return;
  constexpr int N = 4 * NCH;
  float v[N], gm[N], bt[N];
  load_row(x + (size_t)row * D, v, lane);
  const RowStats st = row_stats(v, D);
  load_row(gamma, gm, lane); load_row(beta, bt, lane);
  #pragma unroll
  for (int i = 0; i < N; ++i) v[i] = (v[i] - st.mean) * st.rstd * gm[i] + bt[i];
  store_row_bf16(y + (size_t)row * D, v, lane);
  if (lane == 0) { mean_out[row] = st.mean; rstd_out[row] = st.rstd; }
}

// LayerNorm data-gradient for one row: returns dx in v (input: dy in v, x in xv).
template <int N>
__device__ __forceinline__ void ln_bwd_row(float (&v)[N], const float (&xv)[N], const float (&gm)[N], float mean, float rstd, int D) {
  float s1 = 0.f, s2 = 0.f;
#pragma unroll
  for (int i = 0; i < N; ++i) {
    const float xh = (xv[i] - mean) * rstd, dxh = v[i] * gm[i];
    s1 += dxh; s2 += dxh * xh;
  }
  s1 = warp_sum(s1) / (float)D; s2 = warp_sum(s2) / (float)D;
#pragma unroll
  for (int i = 0; i < N; ++i) {
    const float xh = (xv[i] - mean) * rstd, dxh = v[i] * gm[i];
    v[i] = rstd * (dxh - s1 - xh * s2);
  }
}

// mode 0: all rows: dx[row] (+)= LNbwd(dy[row]); writes dx (fp32) and dx_bf16.        (ln_1 / ln_2, ln_post on its S rows)
// mode 1: ln_1 of the last block, whose residual gradient lives on the cls rows only, compact in dcls [S, D]:
//         dx[row] = LNbwd(dy[row]) + (row = s*T ? dcls[s] : 0); writes every row of dx and dx_bf16, reads no dx.
// mode 2: ln_pre : dy = dx itself (all rows); writes only non-cls rows as bf16 into dtok [S*(T-1), D].
template <int NCH, typename DY = float>
__global__ void __launch_bounds__(256) k_ln_bwd(const DY* __restrict__ dy, const float* __restrict__ x, const float* __restrict__ mean,
                                                const float* __restrict__ rstd, const float* __restrict__ gamma,
                                                float* __restrict__ dx, bf16* __restrict__ dx_bf16, int rows, int T, int D,
                                                int mode, int accumulate, const float* __restrict__ dcls) {
  const int r = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (r >= rows) return;
  constexpr int N = 4 * NCH;
  const size_t row = (size_t)r;
  if (mode == 2 && (r % T) == 0) return;                           // the cls row has no patch behind it
  float v[N], xv[N], gm[N];
  load_row(dy + row * D, v, lane);
  load_row(x + row * D, xv, lane);
  load_row(gamma, gm, lane);
  ln_bwd_row(v, xv, gm, mean[row], rstd[row], D);
  if (mode == 2) {
    const int s = r / T, t = r - s * T;
    store_row_bf16(dx_bf16 + ((size_t)s * (T - 1) + (t - 1)) * D, v, lane);
    return;
  }
  if (mode == 1 ? (r % T) == 0 : accumulate != 0) {
    float a[N];
    load_row(mode == 1 ? dcls + (size_t)(r / T) * D : dx + row * D, a, lane);
    #pragma unroll
    for (int i = 0; i < N; ++i) v[i] += a[i];
  }
  store_row_f32(dx + row * D, v, lane);
  store_row_bf16(dx_bf16 + row * D, v, lane);
}

}  // namespace aph
