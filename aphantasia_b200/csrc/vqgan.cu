// vqgan.cu -- the VQGAN decoder handle (taming.modules.diffusionmodules.model.Decoder, eval mode, temb_ch = 0): forward and
// data gradient (d loss / d z) on bf16 NHWC activations. No weight gradients: the weights are constants of the handle.
//
//   conv_in 3x3 (z_channels -> ch ch_mult[-1]); mid: ResnetBlock, AttnBlock, ResnetBlock; per level, coarsest first:
//   num_res_blocks + 1 ResnetBlocks, each followed by an AttnBlock on the levels of attn_mask, then (all but the finest) nearest
//   x2 + conv 3x3; norm_out, swish, conv_out 3x3 (-> 3). Every norm is GroupNorm(32, C, eps 1e-6, affine), swish = x sigmoid(x).
//   ResnetBlock  y = shortcut(x) + conv2(swish(norm2(conv1(swish(norm1 x))))), shortcut = x or nin_shortcut (1x1) on a width change
//   AttnBlock    y = x + proj_out(softmax(q k^T C^-1/2) v), q, k, v = 1x1 convs of norm(x); one head of width C over the h w tokens
// Kernels (sm_90a):
//   3x3 convolutions  k_conv3x3_tc (conv_tc.cuh): forward CONV_BIAS, conv2 CONV_BIAS_RESID (+ the shortcut), data gradient CONV_PLAIN
//   1x1 convolutions  launch_gemm on [pixels, C]: nin_shortcut, q/k/v as one [3C, C] operand, proj_out
//   GroupNorm         k_gn_partials (per-(image, group, pixel chunk) sums, fixed order, no atomics), k_gn_finalize (the chunks in
//                     fp64, in chunk order), k_gn_apply (affine [+ swish] -> the conv's bf16 operand); backward: the same partials
//                     of g = dout swish'(y) gamma and g xhat, then k_gn_apply_bwd, which also adds the residual branch's gradient
//   attention         per image: S = Q K^T (fp32, keys padded to a multiple of 128), k_softmax_rows (P bf16, padded keys 0),
//                     O = P V; backward dP = dO V^T, dS = P (dP - rowsum(dO O)) C^-1/2 (k_attn_ds), dQ = dS K, dK = dS^T Q,
//                     dV = P^T dO, with the transposed operands written by k_vq_pad
//   upsample          k_unpool2 (nhwc.cu) at scale 1: nearest x2, materialised (TMA cannot address half-pixel strides); its
//                     adjoint k_pool2<POOL_SUM> (2 x 2 sum)
//   the ends          k_nchw_to_nhwc (z), k_nhwc_to_nchw (dz), conv_out as the fp32 SIMT pair k_conv_out_fwd / _bwd on the
//                     caller's fp32 NCHW image and its gradient
// The kernels that touch caller memory (the two conversions and conv_out) run outside the cached graphs; everything between them
// replays through one graph per latent shape, forward and backward.
#include "nhwc.cuh"
#include "encoder.cuh"
#include <memory>

namespace aph {

constexpr int VQ_G = 32;              // GroupNorm groups
constexpr int VQ_CHUNK = 256;         // pixels per GroupNorm partial
constexpr float VQ_EPS = 1e-6f;

__device__ __forceinline__ float swishf(float y) { return y * sigmoidf_(y); }
__device__ __forceinline__ float swish_grad(float y) {
  const float s = sigmoidf_(y);
  return s * (1.f + y * (1.f - s));
}

// ---- GroupNorm ------------------------------------------------------------------------------------------------------------
// x bf16 [N, HW, C]; group g holds channels [g C/32, (g + 1) C/32). Block (chunk, n) covers pixels [chunk VQ_CHUNK, + VQ_CHUNK)
// of image n: thread (lane pl, vector cv) sums 8 channels over every PL-th pixel; the block then adds, per group, its threads'
// sums in index order and writes part[((n * chunks + chunk) * 32 + g) * 2 + {0, 1}].
// BWD = false: the sums of x and x^2. BWD = true: of g = dout (swish ? swish'(y) : 1) gamma and of g xhat, xhat = (x - mean) rstd,
// y = gamma xhat + beta, with stats [N, 32, 2] = (mean, rstd) of the forward.
template <bool BWD>
__global__ void __launch_bounds__(256) k_gn_partials(const bf16* __restrict__ x, const bf16* __restrict__ dout, const float* __restrict__ stats,
                                                      const float* __restrict__ gamma, const float* __restrict__ beta, int swish, int HW,
                                                      int C, float* __restrict__ part) {
  extern __shared__ float red[];                       // [2][PL][C]
  const int C8 = C / 8, PL = 256 / C8, Cg = C / VQ_G, n = blockIdx.y, chunks = gridDim.x;
  const int pl = threadIdx.x / C8, cv = threadIdx.x - pl * C8;
  float s[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f}, q[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  if (pl < PL) {
    float mean[8], rstd[8], ga[8], be[8];
    if (BWD) {
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const int c = 8 * cv + j, g = c / Cg;
        mean[j] = stats[(n * VQ_G + g) * 2]; rstd[j] = stats[(n * VQ_G + g) * 2 + 1];
        ga[j] = gamma[c]; be[j] = beta[c];
      }
    }
    const int p1 = min(HW, (blockIdx.x + 1) * VQ_CHUNK);
    for (int p = blockIdx.x * VQ_CHUNK + pl; p < p1; p += PL) {
      const size_t off = ((size_t)n * HW + p) * C8 + cv;
      float v[8];
      unpack_bf16x8(__ldg(reinterpret_cast<const uint4*>(x) + off), v);
      if (!BWD) {
#pragma unroll
        for (int j = 0; j < 8; ++j) { s[j] += v[j]; q[j] = fmaf(v[j], v[j], q[j]); }
      } else {
        float d[8];
        unpack_bf16x8(__ldg(reinterpret_cast<const uint4*>(dout) + off), d);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const float xh = (v[j] - mean[j]) * rstd[j];
          const float g = d[j] * (swish ? swish_grad(fmaf(ga[j], xh, be[j])) : 1.f) * ga[j];
          s[j] += g; q[j] = fmaf(g, xh, q[j]);
        }
      }
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) { red[pl * C + 8 * cv + j] = s[j]; red[(PL + pl) * C + 8 * cv + j] = q[j]; }
  }
  __syncthreads();
  if (threadIdx.x < 2 * VQ_G) {
    const int k = threadIdx.x / VQ_G, g = threadIdx.x - k * VQ_G;
    float t = 0.f;
    for (int l = 0; l < PL; ++l)
      for (int c = g * Cg; c < (g + 1) * Cg; ++c) t += red[(k * PL + l) * C + c];
    part[(((size_t)n * chunks + blockIdx.x) * VQ_G + g) * 2 + k] = t;
  }
}

// out [N, 32, 2]: the partials of each (image, group) summed in chunk order in fp64, over count = HW C / 32 elements.
// BWD = false: (mean, rstd = 1 / sqrt(var + eps)), the biased variance as torch's; BWD = true: (mean g, mean g xhat).
template <bool BWD>
__global__ void __launch_bounds__(256) k_gn_finalize(const float* __restrict__ part, int N, int chunks, double count, float* __restrict__ out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N * VQ_G) return;
  const int n = i / VQ_G, g = i - n * VQ_G;
  double s = 0., q = 0.;
  for (int c = 0; c < chunks; ++c) {
    const float* p = part + (((size_t)n * chunks + c) * VQ_G + g) * 2;
    s += p[0]; q += p[1];
  }
  s /= count; q /= count;
  if (BWD) { out[2 * i] = (float)s; out[2 * i + 1] = (float)q; return; }
  const double var = fmax(q - s * s, 0.);
  out[2 * i] = (float)s;
  out[2 * i + 1] = (float)(1. / sqrt(var + (double)VQ_EPS));
}

// out = [swish](gamma (x - mean) rstd + beta), bf16 [N, HW, C]
__global__ void __launch_bounds__(256) k_gn_apply(const bf16* __restrict__ x, const float* __restrict__ stats, const float* __restrict__ gamma,
                                                   const float* __restrict__ beta, int swish, int N, int HW, int C, bf16* __restrict__ out) {
  const int C8 = C / 8, Cg = C / VQ_G;
  const size_t n_items = (size_t)N * HW * C8;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n_items; i += (size_t)gridDim.x * blockDim.x) {
    const int cv = (int)(i % C8), n = (int)(i / ((size_t)HW * C8));
    float v[8];
    unpack_bf16x8(__ldg(reinterpret_cast<const uint4*>(x) + i), v);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int c = 8 * cv + j, g = c / Cg;
      const float y = fmaf(gamma[c], (v[j] - stats[(n * VQ_G + g) * 2]) * stats[(n * VQ_G + g) * 2 + 1], beta[c]);
      v[j] = swish ? swishf(y) : y;
    }
    reinterpret_cast<uint4*>(out)[i] = pack_bf16x8(v);
  }
}

// dx = rstd (g - mean g - xhat mean(g xhat)) [+ resid], g as in k_gn_partials<true>; red [N, 32, 2] from k_gn_finalize<true>
__global__ void __launch_bounds__(256) k_gn_apply_bwd(const bf16* __restrict__ dout, const bf16* __restrict__ x, const float* __restrict__ stats,
                                                       const float* __restrict__ red, const float* __restrict__ gamma,
                                                       const float* __restrict__ beta, int swish, const bf16* __restrict__ resid, int N,
                                                       int HW, int C, bf16* __restrict__ dx) {
  const int C8 = C / 8, Cg = C / VQ_G;
  const size_t n_items = (size_t)N * HW * C8;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n_items; i += (size_t)gridDim.x * blockDim.x) {
    const int cv = (int)(i % C8), n = (int)(i / ((size_t)HW * C8));
    float v[8], d[8], r[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    unpack_bf16x8(__ldg(reinterpret_cast<const uint4*>(x) + i), v);
    unpack_bf16x8(__ldg(reinterpret_cast<const uint4*>(dout) + i), d);
    if (resid) unpack_bf16x8(__ldg(reinterpret_cast<const uint4*>(resid) + i), r);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int c = 8 * cv + j, ng = n * VQ_G + c / Cg;
      const float rs = stats[2 * ng + 1], xh = (v[j] - stats[2 * ng]) * rs;
      const float g = d[j] * (swish ? swish_grad(fmaf(gamma[c], xh, beta[c])) : 1.f) * gamma[c];
      v[j] = rs * (g - red[2 * ng] - xh * red[2 * ng + 1]) + r[j];
    }
    reinterpret_cast<uint4*>(dx)[i] = pack_bf16x8(v);
  }
}

// ---- residual add, layout conversions --------------------------------------------------------------------------------------
// out = a + b, bf16, n8 items of 8 elements
__global__ void __launch_bounds__(256) k_add_bf16(const bf16* __restrict__ a, const bf16* __restrict__ b, size_t n8, bf16* __restrict__ out) {
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n8; i += (size_t)gridDim.x * blockDim.x) {
    float u[8], v[8];
    unpack_bf16x8(__ldg(reinterpret_cast<const uint4*>(a) + i), u);
    unpack_bf16x8(__ldg(reinterpret_cast<const uint4*>(b) + i), v);
#pragma unroll
    for (int j = 0; j < 8; ++j) u[j] += v[j];
    reinterpret_cast<uint4*>(out)[i] = pack_bf16x8(u);
  }
}

// z fp32 [N, C, H, W] -> bf16 [N, H, W, C]
__global__ void __launch_bounds__(256) k_nchw_to_nhwc(const float* __restrict__ z, int N, int C, int HW, bf16* __restrict__ out) {
  const size_t n_items = (size_t)N * HW * C;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n_items; i += (size_t)gridDim.x * blockDim.x) {
    const int c = (int)(i % C);
    const size_t p = i / C;
    const int n = (int)(p / HW), hw = (int)(p - (size_t)n * HW);
    out[i] = __float2bfloat16(z[((size_t)n * C + c) * HW + hw]);
  }
}

// x bf16 [N, H, W, C] -> fp32 [N, C, H, W]
__global__ void __launch_bounds__(256) k_nhwc_to_nchw(const bf16* __restrict__ x, int N, int C, int HW, float* __restrict__ out) {
  const size_t n_items = (size_t)N * HW * C;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n_items; i += (size_t)gridDim.x * blockDim.x) {
    const int hw = (int)(i % HW);
    const size_t nc = i / HW;
    const int c = (int)(nc % C), n = (int)(nc / C);
    out[i] = __bfloat162float(x[((size_t)n * HW + hw) * C + c]);
  }
}

// ---- conv_out: C -> 3, 3x3, pad 1, fp32 SIMT ------------------------------------------------------------------------------
// sw [9][C][3] (tap-major, then channel, then output), staged in dynamic shared memory from w [3][C][3][3]
__device__ __forceinline__ void vq_stage_wout(const float* __restrict__ w, int C, float* sw) {
  for (int i = threadIdx.x; i < 27 * C; i += blockDim.x) {
    const int o = i % 3, r = i / 3, c = r % C, t = r / C;
    sw[i] = w[((size_t)o * C + c) * 9 + t];
  }
  __syncthreads();
}

// a bf16 [N, H, W, C] (swish(norm_out x)) -> out fp32 [N, 3, H, W] = conv + bias. One thread per pixel.
__global__ void __launch_bounds__(128) k_conv_out_fwd(const bf16* __restrict__ a, int N, int H, int W, int C, const float* __restrict__ w,
                                                      const float* __restrict__ b, float* __restrict__ out) {
  extern __shared__ float sw[];
  vq_stage_wout(w, C, sw);
  const size_t HW = (size_t)H * W, p = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (p >= (size_t)N * HW) return;
  const int n = (int)(p / HW), rem = (int)(p - n * HW), y = rem / W, x = rem - y * W;
  float acc[3] = {b[0], b[1], b[2]};
  for (int t = 0; t < 9; ++t) {
    const int yy = y + t / 3 - 1, xx = x + t % 3 - 1;
    if (yy < 0 || yy >= H || xx < 0 || xx >= W) continue;
    const uint4* src = reinterpret_cast<const uint4*>(a + (((size_t)n * H + yy) * W + xx) * C);
    const float* wt = sw + (size_t)t * C * 3;
    for (int cv = 0; cv < C / 8; ++cv) {
      float f[8];
      unpack_bf16x8(__ldg(src + cv), f);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float* wc = wt + (8 * cv + j) * 3;
        acc[0] = fmaf(f[j], wc[0], acc[0]); acc[1] = fmaf(f[j], wc[1], acc[1]); acc[2] = fmaf(f[j], wc[2], acc[2]);
      }
    }
  }
#pragma unroll
  for (int o = 0; o < 3; ++o) out[((size_t)n * 3 + o) * HW + rem] = acc[o];
}

// grad fp32 [N, 3, H, W] -> da bf16 [N, H, W, C]: pixel q gets sum over taps t and outputs o of grad[o, q - shift(t)] w[o, c, t].
__global__ void __launch_bounds__(128) k_conv_out_bwd(const float* __restrict__ grad, int N, int H, int W, int C, const float* __restrict__ w,
                                                      bf16* __restrict__ da) {
  extern __shared__ float sw[];
  vq_stage_wout(w, C, sw);
  const size_t HW = (size_t)H * W, p = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (p >= (size_t)N * HW) return;
  const int n = (int)(p / HW), rem = (int)(p - n * HW), y = rem / W, x = rem - y * W;
  float g[27];
#pragma unroll
  for (int t = 0; t < 9; ++t) {
    const int yy = y - (t / 3 - 1), xx = x - (t % 3 - 1);
    const bool ok = yy >= 0 && yy < H && xx >= 0 && xx < W;
#pragma unroll
    for (int o = 0; o < 3; ++o) g[3 * t + o] = ok ? grad[((size_t)n * 3 + o) * HW + (size_t)yy * W + xx] : 0.f;
  }
  uint4* dst = reinterpret_cast<uint4*>(da + p * C);
  for (int cv = 0; cv < C / 8; ++cv) {
    float f[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int c = 8 * cv + j;
      float s = 0.f;
#pragma unroll
      for (int t = 0; t < 9; ++t) {
        const float* wc = sw + ((size_t)t * C + c) * 3;
        s = fmaf(g[3 * t], wc[0], fmaf(g[3 * t + 1], wc[1], fmaf(g[3 * t + 2], wc[2], s)));
      }
      f[j] = s;
    }
    dst[cv] = pack_bf16x8(f);
  }
}

// ---- attention (one head of width C, T tokens per image, keys padded to Tp, a multiple of 128) ---------------------------
// TR = false: out [rpad, cols] = src rows [0, rows) of columns [0, cols) (row stride ld), zero in rows >= rows.
// TR = true:  out [cols, rpad] = the transpose of the same, zero in columns >= rows. 32 x 32 tiles through shared memory.
template <bool TR>
__global__ void __launch_bounds__(256) k_vq_pad(const bf16* __restrict__ src, int ld, int rows, int cols, int rpad, bf16* __restrict__ out) {
  __shared__ bf16 t[32][34];
  const int c0 = blockIdx.x * 32, r0 = blockIdx.y * 32, tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  for (int i = ty; i < 32; i += 8) {
    const int r = r0 + i, c = c0 + tx;
    const bf16 v = (r < rows && c < cols) ? src[(size_t)r * ld + c] : __float2bfloat16(0.f);
    if (TR) t[i][tx] = v;
    else if (r < rpad && c < cols) out[(size_t)r * cols + c] = v;
  }
  if (!TR) return;
  __syncthreads();
  for (int i = ty; i < 32; i += 8) {
    const int c = c0 + i, r = r0 + tx;
    if (c < cols && r < rpad) out[(size_t)c * rpad + r] = t[tx][i];
  }
}

// block-wide sum / max of 256 threads (every thread gets the result)
__device__ __forceinline__ float vq_block_reduce(float v, bool is_max) {
  __shared__ float r[8];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float u = __shfl_xor_sync(0xffffffffu, v, o);
    v = is_max ? fmaxf(v, u) : v + u;
  }
  __syncthreads();                                   // r may still be read by a previous call
  if ((threadIdx.x & 31) == 0) r[threadIdx.x >> 5] = v;
  __syncthreads();
  v = r[0];
  for (int i = 1; i < 8; ++i) v = is_max ? fmaxf(v, r[i]) : v + r[i];
  return v;
}

// P [T, Tp] bf16 = softmax over the T keys of scale S [T, Tp] (fp32); keys >= T get 0. One block per row.
__global__ void __launch_bounds__(256) k_softmax_rows(const float* __restrict__ S, int T, int Tp, float scale, bf16* __restrict__ P) {
  const float* s = S + (size_t)blockIdx.x * Tp;
  bf16* p = P + (size_t)blockIdx.x * Tp;
  float m = -INFINITY;
  for (int j = threadIdx.x; j < T; j += 256) m = fmaxf(m, s[j]);
  m = vq_block_reduce(m, true);
  float z = 0.f;
  for (int j = threadIdx.x; j < T; j += 256) z += __expf((s[j] - m) * scale);
  const float inv = 1.f / vq_block_reduce(z, false);
  for (int j = threadIdx.x; j < Tp; j += 256) p[j] = __float2bfloat16(j < T ? __expf((s[j] - m) * scale) * inv : 0.f);
}

// dS [T, Tp] bf16 = P (dP - rowsum(dO O)) scale, 0 on the padded keys. dO, O bf16 [T, C]. One block per row.
__global__ void __launch_bounds__(256) k_attn_ds(const bf16* __restrict__ P, const float* __restrict__ dP, const bf16* __restrict__ dO,
                                                 const bf16* __restrict__ O, int T, int Tp, int C, float scale, bf16* __restrict__ dS) {
  const size_t i = blockIdx.x;
  float d = 0.f;
  for (int c = threadIdx.x; c < C; c += 256) d = fmaf(__bfloat162float(dO[i * C + c]), __bfloat162float(O[i * C + c]), d);
  d = vq_block_reduce(d, false);
  for (int j = threadIdx.x; j < Tp; j += 256)
    dS[i * Tp + j] = __float2bfloat16(j < T ? __bfloat162float(P[i * Tp + j]) * (dP[i * Tp + j] - d) * scale : 0.f);
}

inline int vq_tpad(int T) { return (T + 127) / 128 * 128; }

// The attention's scratch for one image of up to T tokens: F fp32 [T, Tp]; A bf16 [T, Tp]; X bf16 [Tp, Tp]; Kc bf16 [Tp, C];
// Kt bf16 [C, Tp]
struct AttnScratch { float* F; bf16 *A, *X, *Kc, *Kt; };

static int vq_pad(bool tr, const bf16* src, int ld, int rows, int cols, int rpad, bf16* out, cudaStream_t st) {
  const dim3 grid((cols + 31) / 32, (rpad + 31) / 32);
  if (tr) k_vq_pad<true><<<grid, 256, 0, st>>>(src, ld, rows, cols, rpad, out);
  else k_vq_pad<false><<<grid, 256, 0, st>>>(src, ld, rows, cols, rpad, out);
  APH_LAUNCH_OK();
  return 0;
}

// forward of image n: qkv bf16 [T, 3C] (rows of that image) -> P [T, Tp] (kept for the backward), O [T, C]
static int attn_fwd_img(const bf16* qkv, int T, int C, bf16* P, bf16* O, const AttnScratch& s, cudaStream_t st) {
  const int Tp = vq_tpad(T);
  int e;
  if ((e = vq_pad(false, qkv + C, 3 * C, T, C, Tp, s.Kc, st))) return e;
  { GemmEpi ep; ep.out_f32 = s.F;
    if ((e = launch_gemm(qkv, s.Kc, GemmShape{T, Tp, C}, ep, st, 3 * C))) return e; }
  k_softmax_rows<<<T, 256, 0, st>>>(s.F, T, Tp, 1.f / sqrtf((float)C), P);
  APH_LAUNCH_OK();
  if ((e = vq_pad(true, qkv + 2 * C, 3 * C, T, C, Tp, s.Kt, st))) return e;
  GemmEpi ep; ep.out_bf16 = O;
  return launch_gemm(P, s.Kt, GemmShape{T, C, Tp}, ep, st);
}

// backward of image n: dO bf16 [T, C] -> dqkv bf16 [T, 3C], from qkv, P and O of the forward
static int attn_bwd_img(const bf16* qkv, const bf16* P, const bf16* O, const bf16* dO, int T, int C, bf16* dqkv, const AttnScratch& s,
                        cudaStream_t st) {
  const int Tp = vq_tpad(T);
  int e;
  if ((e = vq_pad(false, qkv + 2 * C, 3 * C, T, C, Tp, s.Kc, st))) return e;              // V [Tp, C]
  { GemmEpi ep; ep.out_f32 = s.F;                                                          // dP = dO V^T
    if ((e = launch_gemm(dO, s.Kc, GemmShape{T, Tp, C}, ep, st))) return e; }
  k_attn_ds<<<T, 256, 0, st>>>(P, s.F, dO, O, T, Tp, C, 1.f / sqrtf((float)C), s.A);
  APH_LAUNCH_OK();
  if ((e = vq_pad(true, qkv + C, 3 * C, T, C, Tp, s.Kt, st))) return e;                  // K^T [C, Tp]
  { GemmEpi ep; ep.out_bf16 = dqkv; ep.ld_out = 3 * C;                                     // dQ = dS K
    if ((e = launch_gemm(s.A, s.Kt, GemmShape{T, C, Tp}, ep, st))) return e; }
  if ((e = vq_pad(true, s.A, Tp, T, T, Tp, s.X, st))) return e;                           // dS^T [T, Tp]
  if ((e = vq_pad(true, qkv, 3 * C, T, C, Tp, s.Kt, st))) return e;                       // Q^T [C, Tp]
  { GemmEpi ep; ep.out_bf16 = dqkv + C; ep.ld_out = 3 * C;                                 // dK = dS^T Q
    if ((e = launch_gemm(s.X, s.Kt, GemmShape{T, C, Tp}, ep, st))) return e; }
  if ((e = vq_pad(true, P, Tp, T, T, Tp, s.X, st))) return e;                             // P^T [T, Tp]
  if ((e = vq_pad(true, dO, C, T, C, Tp, s.Kt, st))) return e;                            // dO^T [C, Tp]
  GemmEpi ep; ep.out_bf16 = dqkv + 2 * C; ep.ld_out = 3 * C;                               // dV = P^T dO
  return launch_gemm(s.X, s.Kt, GemmShape{T, C, Tp}, ep, st);
}

// ---- launch helpers --------------------------------------------------------------------------------------------------------
static int gn_fwd(const bf16* x, const float* gamma, const float* beta, int swish, int N, int HW, int C, float* part, float* stats,
                  bf16* out, cudaStream_t st) {
  const int chunks = (HW + VQ_CHUNK - 1) / VQ_CHUNK;
  const size_t smem = (size_t)2 * (256 / (C / 8)) * C * sizeof(float);
  if (int e = smem_at_least((const void*)k_gn_partials<false>, smem)) return e;
  k_gn_partials<false><<<dim3(chunks, N), 256, smem, st>>>(x, nullptr, nullptr, nullptr, nullptr, 0, HW, C, part);
  APH_LAUNCH_OK();
  k_gn_finalize<false><<<(N * VQ_G + 255) / 256, 256, 0, st>>>(part, N, chunks, (double)HW * (C / VQ_G), stats);
  APH_LAUNCH_OK();
  k_gn_apply<<<stride_blocks((size_t)N * HW * C / 8, 16), 256, 0, st>>>(x, stats, gamma, beta, swish, N, HW, C, out);
  APH_LAUNCH_OK();
  return 0;
}

// red: [N, 32, 2] scratch
static int gn_bwd(const bf16* dout, const bf16* x, const float* stats, const float* gamma, const float* beta, int swish, const bf16* resid,
                  int N, int HW, int C, float* part, float* red, bf16* dx, cudaStream_t st) {
  const int chunks = (HW + VQ_CHUNK - 1) / VQ_CHUNK;
  const size_t smem = (size_t)2 * (256 / (C / 8)) * C * sizeof(float);
  if (int e = smem_at_least((const void*)k_gn_partials<true>, smem)) return e;
  k_gn_partials<true><<<dim3(chunks, N), 256, smem, st>>>(x, dout, stats, gamma, beta, swish, HW, C, part);
  APH_LAUNCH_OK();
  k_gn_finalize<true><<<(N * VQ_G + 255) / 256, 256, 0, st>>>(part, N, chunks, (double)HW * (C / VQ_G), red);
  APH_LAUNCH_OK();
  k_gn_apply_bwd<<<stride_blocks((size_t)N * HW * C / 8, 16), 256, 0, st>>>(dout, x, stats, red, gamma, beta, swish, resid, N, HW, C, dx);
  APH_LAUNCH_OK();
  return 0;
}

static int add_bf16(const bf16* a, const bf16* b, size_t n, bf16* out, cudaStream_t st) {
  k_add_bf16<<<stride_blocks(n / 8, 16), 256, 0, st>>>(a, b, n / 8, out);
  APH_LAUNCH_OK();
  return 0;
}

static int conv_out(bool fwd, const void* in, int N, int H, int W, int C, const float* w, const float* b, void* out, cudaStream_t st) {
  const size_t smem = (size_t)27 * C * sizeof(float), n = (size_t)N * H * W;
  const void* k = fwd ? (const void*)k_conv_out_fwd : (const void*)k_conv_out_bwd;
  if (int e = smem_at_least(k, smem)) return e;
  if (fwd) k_conv_out_fwd<<<(unsigned)((n + 127) / 128), 128, smem, st>>>(reinterpret_cast<const bf16*>(in), N, H, W, C, w, b, reinterpret_cast<float*>(out));
  else k_conv_out_bwd<<<(unsigned)((n + 127) / 128), 128, smem, st>>>(reinterpret_cast<const float*>(in), N, H, W, C, w, reinterpret_cast<bf16*>(out));
  APH_LAUNCH_OK();
  return 0;
}

static int layout(bool to_nhwc, const void* in, int N, int C, int HW, void* out, cudaStream_t st) {
  const size_t n = (size_t)N * C * HW;
  if (to_nhwc) k_nchw_to_nhwc<<<stride_blocks(n, 16), 256, 0, st>>>(reinterpret_cast<const float*>(in), N, C, HW, reinterpret_cast<bf16*>(out));
  else k_nhwc_to_nchw<<<stride_blocks(n, 16), 256, 0, st>>>(reinterpret_cast<const bf16*>(in), N, C, HW, reinterpret_cast<float*>(out));
  APH_LAUNCH_OK();
  return 0;
}

// ---- the handle ------------------------------------------------------------------------------------------------------------
struct VqNorm { float *gamma = nullptr, *beta = nullptr, *stats = nullptr; };   // stats [N, 32, 2] of the saved forward

// One step of the decoder after conv_in. Its input is the previous step's `out` (conv_in's for the first); `scale` is the
// pixel count of its input map over the latent's (4^k after k upsamples).
struct VqOp {
  enum Kind { RES, ATTN, UP } kind;
  int cin, cout, scale;
  VqNorm n1, n2;                                   // RES: norm1, norm2; ATTN: norm (n1)
  bf16 *w1 = nullptr, *w1t = nullptr, *w2 = nullptr, *w2t = nullptr;   // RES: conv1, conv2; UP: conv (w1); packed both ways
  float *b1 = nullptr, *b2 = nullptr;
  bf16 *wn = nullptr, *wnt = nullptr;              // RES nin_shortcut [cout, cin] / [cin, cout]; ATTN q|k|v [3C, C] / [C, 3C]
  float* bn = nullptr;                             // their bias
  bf16 *wp = nullptr, *wpt = nullptr;              // ATTN proj_out [C, C] and its transpose
  float* bp = nullptr;
  bf16* h1 = nullptr;                              // RES: conv1's output; ATTN: qkv [P, 3C]
  bf16* o = nullptr;                               // ATTN: the attention output [P, C]
  bf16* P = nullptr;                               // ATTN: the probabilities [N, T, Tp]
  bf16* out = nullptr;                             // the step's output
};

struct VqImpl : Weights {
  aph_vqgan_config cfg;
  std::vector<VqOp> ops;
  bf16 *w_in = nullptr, *w_in_t = nullptr;
  float *b_in = nullptr, *w_out = nullptr, *b_out = nullptr;
  VqNorm norm_out;
  int c_top = 0, c_out = 0, up_total = 0;           // the latent's width, the finest map's width, the number of upsamples
  bf16 *zb = nullptr, *x0 = nullptr;                // z as bf16 NHWC; conv_in's output
  bf16 *sa = nullptr, *sb = nullptr, *g[2] = {};    // [S emax] each: temporaries and the backward's gradients
  bf16 *dqkv = nullptr;                             // [S T, 3 C_attn]
  AttnScratch as{};
  float *part = nullptr, *red = nullptr;
  size_t emax = 0;
  int last_N = -1, last_h = -1, last_w = -1;
  GraphCacheRef fwd_graphs, bwd_graphs;
};

static int vq_fwd_body(VqImpl* h, int N, int lh, int lw, cudaStream_t st) {
  int e;
  { ConvEpi c; c.bias = h->b_in; c.out = h->x0;
    if ((e = launch_conv3x3(h->zb, h->w_in, N, lh, lw, h->cfg.z_channels, h->c_top, CONV_BIAS, c, st))) return e; }
  const bf16* x = h->x0;
  int H = lh, W = lw;
  for (VqOp& op : h->ops) {
    const int HW = H * W, Pn = N * HW;
    if (op.kind == VqOp::RES) {
      if ((e = gn_fwd(x, op.n1.gamma, op.n1.beta, 1, N, HW, op.cin, h->part, op.n1.stats, h->sa, st))) return e;
      { ConvEpi c; c.bias = op.b1; c.out = op.h1;
        if ((e = launch_conv3x3(h->sa, op.w1, N, H, W, op.cin, op.cout, CONV_BIAS, c, st))) return e; }
      if ((e = gn_fwd(op.h1, op.n2.gamma, op.n2.beta, 1, N, HW, op.cout, h->part, op.n2.stats, h->sa, st))) return e;
      const bf16* sc = x;
      if (op.wn) {
        GemmEpi ep; ep.bias = op.bn; ep.out_bf16 = h->sb;
        if ((e = launch_gemm(x, op.wn, GemmShape{Pn, op.cout, op.cin}, ep, st))) return e;
        sc = h->sb;
      }
      ConvEpi c; c.bias = op.b2; c.resid = sc; c.out = op.out;
      if ((e = launch_conv3x3(h->sa, op.w2, N, H, W, op.cout, op.cout, CONV_BIAS_RESID, c, st))) return e;
    } else if (op.kind == VqOp::ATTN) {
      const int C = op.cin, T = HW, Tp = vq_tpad(T);     // the tokens: every pixel of the map
      if ((e = gn_fwd(x, op.n1.gamma, op.n1.beta, 0, N, HW, C, h->part, op.n1.stats, h->sa, st))) return e;
      { GemmEpi ep; ep.bias = op.bn; ep.out_bf16 = op.h1;
        if ((e = launch_gemm(h->sa, op.wn, GemmShape{Pn, 3 * C, C}, ep, st))) return e; }
      for (int n = 0; n < N; ++n)
        if ((e = attn_fwd_img(op.h1 + (size_t)n * T * 3 * C, T, C, op.P + (size_t)n * T * Tp, op.o + (size_t)n * T * C, h->as, st))) return e;
      { GemmEpi ep; ep.bias = op.bp; ep.out_bf16 = h->sb;
        if ((e = launch_gemm(op.o, op.wp, GemmShape{Pn, C, C}, ep, st))) return e; }
      if ((e = add_bf16(x, h->sb, (size_t)Pn * C, op.out, st))) return e;
    } else {
      H *= 2; W *= 2;
      if ((e = launch_unpool2(x, nullptr, N, H, W, op.cin, 1.f, h->sa, st))) return e;
      ConvEpi c; c.bias = op.b1; c.out = op.out;
      if ((e = launch_conv3x3(h->sa, op.w1, N, H, W, op.cin, op.cout, CONV_BIAS, c, st))) return e;
    }
    x = op.out;
  }
  return gn_fwd(x, h->norm_out.gamma, h->norm_out.beta, 1, N, H * W, h->c_out, h->part, h->norm_out.stats, h->sa, st);
}

// from d (swish(norm_out x)) in sa down to d (conv_in's input), which it leaves in sb
static int vq_bwd_body(VqImpl* h, int N, int lh, int lw, cudaStream_t st) {
  int H = lh << h->up_total, W = lw << h->up_total;
  int e, cur = 0;
  const bf16* xlast = h->ops.empty() ? h->x0 : h->ops.back().out;
  if ((e = gn_bwd(h->sa, xlast, h->norm_out.stats, h->norm_out.gamma, h->norm_out.beta, 1, nullptr, N, H * W, h->c_out, h->part, h->red,
                  h->g[cur], st))) return e;
  for (int i = (int)h->ops.size() - 1; i >= 0; --i) {
    const VqOp& op = h->ops[i];
    const bf16* x = i > 0 ? h->ops[i - 1].out : h->x0;
    const bf16* dy = h->g[cur];
    bf16* dx = h->g[cur ^ 1];
    if (op.kind == VqOp::UP) {
      ConvEpi c; c.out = h->sa;
      if ((e = launch_conv3x3(dy, op.w1t, N, H, W, op.cout, op.cin, CONV_PLAIN, c, st))) return e;
      if ((e = launch_pool2(POOL_SUM, h->sa, N, H, W, op.cin, dx, st))) return e;
      H /= 2; W /= 2;
    } else if (op.kind == VqOp::RES) {
      const int HW = H * W, Pn = N * HW;
      { ConvEpi c; c.out = h->sa;
        if ((e = launch_conv3x3(dy, op.w2t, N, H, W, op.cout, op.cout, CONV_PLAIN, c, st))) return e; }
      if ((e = gn_bwd(h->sa, op.h1, op.n2.stats, op.n2.gamma, op.n2.beta, 1, nullptr, N, HW, op.cout, h->part, h->red, h->sb, st))) return e;
      { ConvEpi c; c.out = h->sa;
        if ((e = launch_conv3x3(h->sb, op.w1t, N, H, W, op.cout, op.cin, CONV_PLAIN, c, st))) return e; }
      const bf16* r = dy;
      if (op.wn) {
        GemmEpi ep; ep.out_bf16 = h->sb;
        if ((e = launch_gemm(dy, op.wnt, GemmShape{Pn, op.cin, op.cout}, ep, st))) return e;
        r = h->sb;
      }
      if ((e = gn_bwd(h->sa, x, op.n1.stats, op.n1.gamma, op.n1.beta, 1, r, N, HW, op.cin, h->part, h->red, dx, st))) return e;
    } else {
      const int HW = H * W, Pn = N * HW, C = op.cin, T = HW, Tp = vq_tpad(T);
      { GemmEpi ep; ep.out_bf16 = h->sb;                                    // dO = dy proj_out
        if ((e = launch_gemm(dy, op.wpt, GemmShape{Pn, C, C}, ep, st))) return e; }
      for (int n = 0; n < N; ++n)
        if ((e = attn_bwd_img(op.h1 + (size_t)n * T * 3 * C, op.P + (size_t)n * T * Tp, op.o + (size_t)n * T * C, h->sb + (size_t)n * T * C,
                              T, C, h->dqkv + (size_t)n * T * 3 * C, h->as, st))) return e;
      { GemmEpi ep; ep.out_bf16 = h->sa;
        if ((e = launch_gemm(h->dqkv, op.wnt, GemmShape{Pn, C, 3 * C}, ep, st))) return e; }
      if ((e = gn_bwd(h->sa, x, op.n1.stats, op.n1.gamma, op.n1.beta, 0, dy, N, HW, C, h->part, h->red, dx, st))) return e;
    }
    cur ^= 1;
  }
  ConvEpi c; c.out = h->sb;
  return launch_conv3x3(h->g[cur], h->w_in_t, N, lh, lw, h->c_top, h->cfg.z_channels, CONV_PLAIN, c, st);
}

}  // namespace aph

using namespace aph;

extern "C" int aph_vqgan_create(aph_vqgan** out, const aph_vqgan_config* cfg) {
  APH_REQUIRE(out && cfg, "aph_vqgan_create: null argument");
  const int L = cfg->num_levels;
  APH_REQUIRE(L >= 1 && L <= 8, "aph_vqgan_create: num_levels %d outside [1, 8]", L);
  APH_REQUIRE(cfg->num_res_blocks >= 0 && cfg->max_batch > 0 && cfg->max_tokens > 0, "aph_vqgan_create: bad num_res_blocks / max_batch / max_tokens");
  APH_REQUIRE(cfg->max_tokens <= APH_VQGAN_MAX_TOKENS, "aph_vqgan_create: max_tokens %d above %d", cfg->max_tokens, APH_VQGAN_MAX_TOKENS);
  APH_REQUIRE(cfg->z_channels % 64 == 0 && cfg->z_channels > 0, "aph_vqgan_create: z_channels %d is not a multiple of 64", cfg->z_channels);
  APH_REQUIRE(cfg->out_ch == 3, "aph_vqgan_create: out_ch %d (3 only)", cfg->out_ch);
  for (int i = 0; i < L; ++i) {
    const int c = cfg->ch * cfg->ch_mult[i];
    APH_REQUIRE(c % 64 == 0 && c > 0 && c <= 2048, "aph_vqgan_create: level %d width %d is not a multiple of 64 in (0, 2048]", i, c);
    // the widths a 1x1 convolution or attention runs at (launch_gemm's N): a width change, or a level with attention
    const int prev = i == L - 1 ? c : cfg->ch * cfg->ch_mult[i + 1];
    APH_REQUIRE((prev == c && !(cfg->attn_mask >> i & 1)) || (c % 128 == 0 && prev % 128 == 0) || (i == L - 1 && c % 128 == 0),
                "aph_vqgan_create: level %d width %d (from %d): a nin_shortcut or attention width must be a multiple of 128", i, c, prev);
  }
  APH_REQUIRE(cfg->ch * cfg->ch_mult[L - 1] % 128 == 0, "aph_vqgan_create: the mid attention's width %d is not a multiple of 128",
              cfg->ch * cfg->ch_mult[L - 1]);
  std::unique_ptr<VqImpl> h(new VqImpl());
  h->cfg = *cfg;
  const size_t S = (size_t)cfg->max_batch, T = (size_t)cfg->max_tokens;
  int e = 0;
  auto norm = [&](const std::string& p, int C, VqNorm& nm) {
    e |= h->add_f32(p + ".weight", &nm.gamma, C); e |= h->add_f32(p + ".bias", &nm.beta, C);
    e |= h->alloc(&nm.stats, S * VQ_G * 2);
  };
  size_t attn_c = 0, attn_t = 0;     // the widest attention and its largest token count
  int block_in = cfg->ch * cfg->ch_mult[L - 1], scale = 1;
  h->c_top = block_in;
  h->emax = T * std::max(block_in, cfg->z_channels);
  e |= h->add_conv3x3("conv_in.weight", block_in, cfg->z_channels, &h->w_in, &h->w_in_t); e |= h->add_f32("conv_in.bias", &h->b_in, block_in);
  e |= h->alloc(&h->zb, S * T * cfg->z_channels); e |= h->alloc(&h->x0, S * T * block_in);
  auto res = [&](const std::string& p, int cin, int cout) {
    VqOp op{}; op.kind = VqOp::RES; op.cin = cin; op.cout = cout; op.scale = scale;
    norm(p + ".norm1", cin, op.n1); norm(p + ".norm2", cout, op.n2);
    e |= h->add_conv3x3(p + ".conv1.weight", cout, cin, &op.w1, &op.w1t); e |= h->add_f32(p + ".conv1.bias", &op.b1, cout);
    e |= h->add_conv3x3(p + ".conv2.weight", cout, cout, &op.w2, &op.w2t); e |= h->add_f32(p + ".conv2.bias", &op.b2, cout);
    if (cin != cout) { e |= h->add_bf16(p + ".nin_shortcut.weight", cout, cin, &op.wn, &op.wnt); e |= h->add_f32(p + ".nin_shortcut.bias", &op.bn, cout); }
    const size_t px = S * T * scale;
    e |= h->alloc(&op.h1, px * cout); e |= h->alloc(&op.out, px * cout);
    h->emax = std::max(h->emax, (size_t)T * scale * std::max(cin, cout));
    h->ops.push_back(op);
  };
  auto attn = [&](const std::string& p, int C) {
    if ((size_t)T * scale > APH_VQGAN_MAX_TOKENS) { set_error("aph_vqgan_create: attention over %zu tokens above %d", (size_t)T * scale, APH_VQGAN_MAX_TOKENS); e |= 2; return; }
    VqOp op{}; op.kind = VqOp::ATTN; op.cin = op.cout = C; op.scale = scale;
    norm(p + ".norm", C, op.n1);
    e |= h->add_bf16(p + ".qkv.weight", 3 * C, C, &op.wn, &op.wnt); e |= h->add_f32(p + ".qkv.bias", &op.bn, 3 * C);
    e |= h->add_bf16(p + ".proj_out.weight", C, C, &op.wp, &op.wpt); e |= h->add_f32(p + ".proj_out.bias", &op.bp, C);
    const size_t Tq = T * scale, px = S * Tq;
    e |= h->alloc(&op.h1, px * 3 * C); e |= h->alloc(&op.o, px * C); e |= h->alloc(&op.out, px * C);
    e |= h->alloc(&op.P, S * Tq * vq_tpad((int)Tq));
    attn_c = std::max(attn_c, (size_t)C); attn_t = std::max(attn_t, Tq);
    h->emax = std::max(h->emax, (size_t)Tq * C);
    h->ops.push_back(op);
  };
  res("mid.block_1", block_in, block_in);
  attn("mid.attn_1", block_in);
  res("mid.block_2", block_in, block_in);
  for (int i = L - 1; i >= 0; --i) {
    const int block_out = cfg->ch * cfg->ch_mult[i];
    const std::string p = "up." + std::to_string(i);
    for (int j = 0; j <= cfg->num_res_blocks; ++j) {
      res(p + ".block." + std::to_string(j), block_in, block_out);
      block_in = block_out;
      if (cfg->attn_mask >> i & 1) attn(p + ".attn." + std::to_string(j), block_in);
    }
    if (i > 0) {
      VqOp op{}; op.kind = VqOp::UP; op.cin = op.cout = block_in; op.scale = scale;
      e |= h->add_conv3x3(p + ".upsample.conv.weight", block_in, block_in, &op.w1, &op.w1t);
      e |= h->add_f32(p + ".upsample.conv.bias", &op.b1, block_in);
      scale *= 4;
      e |= h->alloc(&op.out, S * T * scale * block_in);
      h->emax = std::max(h->emax, (size_t)T * scale * block_in);
      h->ops.push_back(op);
      ++h->up_total;
    }
  }
  h->c_out = block_in;
  norm("norm_out", block_in, h->norm_out);
  e |= h->add_f32("conv_out.weight", &h->w_out, (size_t)3 * block_in * 9); e |= h->add_f32("conv_out.bias", &h->b_out, 3);
  e |= h->alloc(&h->sa, S * h->emax); e |= h->alloc(&h->sb, S * h->emax);
  e |= h->alloc(&h->g[0], S * h->emax); e |= h->alloc(&h->g[1], S * h->emax);
  // GroupNorm partials: chunks of the largest map, per image
  const size_t chunks = (T * scale + VQ_CHUNK - 1) / VQ_CHUNK;
  e |= h->alloc(&h->part, S * chunks * VQ_G * 2); e |= h->alloc(&h->red, S * VQ_G * 2);
  if (attn_c) {
    const size_t Tp = vq_tpad((int)attn_t);
    e |= h->alloc(&h->dqkv, S * attn_t * 3 * attn_c);
    e |= h->alloc(&h->as.F, attn_t * Tp); e |= h->alloc(&h->as.A, attn_t * Tp); e |= h->alloc(&h->as.X, Tp * Tp);
    e |= h->alloc(&h->as.Kc, Tp * attn_c); e |= h->alloc(&h->as.Kt, attn_c * Tp);
  }
  if (e) return 1;
  *out = reinterpret_cast<aph_vqgan*>(h.release());
  return 0;
}

extern "C" int aph_vqgan_destroy(aph_vqgan* h) {
  delete reinterpret_cast<VqImpl*>(h);
  return 0;
}

extern "C" int64_t aph_vqgan_bytes(const aph_vqgan* h) { return h ? reinterpret_cast<const VqImpl*>(h)->bytes : 0; }

extern "C" int aph_vqgan_load_tensor(aph_vqgan* h, const char* key, const float* data, int64_t numel, void* stream) {
  return load_tensor(reinterpret_cast<VqImpl*>(h), key, data, numel, (cudaStream_t)stream, "aph_vqgan_load_tensor");
}

extern "C" int aph_vqgan_finalize(aph_vqgan* h) { return finalize(reinterpret_cast<VqImpl*>(h), "aph_vqgan_finalize"); }

static int vq_check(const VqImpl* h, int N, int lh, int lw, const char* who) {
  APH_REQUIRE(h->finalized, "%s: weights not finalized", who);
  APH_REQUIRE(N > 0 && N <= h->cfg.max_batch, "%s: N=%d outside (0, max_batch=%d]", who, N, h->cfg.max_batch);
  APH_REQUIRE(lh > 0 && lw > 0 && (int64_t)lh * lw <= h->cfg.max_tokens, "%s: latent %d x %d above max_tokens=%d", who, lh, lw, h->cfg.max_tokens);
  return 0;
}

extern "C" int aph_vqgan_fwd(aph_vqgan* vq, const float* z, int N, int lh, int lw, float* out, int save_for_bwd, void* stream) {
  APH_REQUIRE(vq && z && out, "aph_vqgan_fwd: null argument");
  VqImpl* h = reinterpret_cast<VqImpl*>(vq);
  if (int e = vq_check(h, N, lh, lw, "aph_vqgan_fwd")) return e;
  cudaStream_t st = (cudaStream_t)stream;
  h->last_N = -1;
  if (int e = layout(true, z, N, h->cfg.z_channels, lh * lw, h->zb, st)) return e;
  if (int e = h->fwd_graphs.replay(N, lh << 16 | lw, st, [&]() { return vq_fwd_body(h, N, lh, lw, st); })) return e;
  if (int e = conv_out(true, h->sa, N, lh << h->up_total, lw << h->up_total, h->c_out, h->w_out, h->b_out, out, st)) return e;
  if (save_for_bwd) { h->last_N = N; h->last_h = lh; h->last_w = lw; }
  return 0;
}

extern "C" int aph_vqgan_bwd(aph_vqgan* vq, const float* grad_out, int N, int lh, int lw, float* grad_z, void* stream) {
  APH_REQUIRE(vq && grad_out && grad_z, "aph_vqgan_bwd: null argument");
  VqImpl* h = reinterpret_cast<VqImpl*>(vq);
  if (int e = vq_check(h, N, lh, lw, "aph_vqgan_bwd")) return e;
  APH_REQUIRE(h->last_N == N && h->last_h == lh && h->last_w == lw, "aph_vqgan_bwd: no saved forward for N=%d latent %d x %d", N, lh, lw);
  cudaStream_t st = (cudaStream_t)stream;
  if (int e = conv_out(false, grad_out, N, lh << h->up_total, lw << h->up_total, h->c_out, h->w_out, nullptr, h->sa, st)) return e;
  if (int e = h->bwd_graphs.replay(N, lh << 16 | lw, st, [&]() { return vq_bwd_body(h, N, lh, lw, st); })) return e;
  return layout(false, h->sb, N, h->cfg.z_channels, lh * lw, grad_z, st);
}

// ---- test entries (tests/test_vqgan_gpu.py) ----------------------------------------------------------------------------------
extern "C" int aph_vqgan_gn_test(int fwd, const void* x, const void* dout, const float* gamma, const float* beta, int swish, const void* resid,
                                 float* stats, void* out, int N, int HW, int C, void* stream) {
  APH_REQUIRE(x && gamma && beta && stats && out && (fwd || dout) && N > 0 && HW > 0, "aph_vqgan_gn_test: bad arguments");
  APH_REQUIRE(C % 64 == 0 && C > 0 && C <= 2048, "aph_vqgan_gn_test: C=%d is not a multiple of 64 in (0, 2048]", C);
  cudaStream_t st = (cudaStream_t)stream;
  StreamTemp<float> part, red;
  if (int e = part.alloc((size_t)N * ((HW + VQ_CHUNK - 1) / VQ_CHUNK) * VQ_G * 2, st)) return e;
  if (int e = red.alloc((size_t)N * VQ_G * 2, st)) return e;
  if (fwd) return gn_fwd(reinterpret_cast<const bf16*>(x), gamma, beta, swish, N, HW, C, part.p, stats, reinterpret_cast<bf16*>(out), st);
  return gn_bwd(reinterpret_cast<const bf16*>(dout), reinterpret_cast<const bf16*>(x), stats, gamma, beta, swish, reinterpret_cast<const bf16*>(resid),
                N, HW, C, part.p, red.p, reinterpret_cast<bf16*>(out), st);
}

extern "C" int aph_vqgan_conv_test(const void* x, const float* weight, const float* bias, const void* resid, void* out, int N, int H, int W,
                                   int Cin, int Cout, void* stream) {
  APH_REQUIRE(x && weight && bias && out, "aph_vqgan_conv_test: bad arguments");
  APH_REQUIRE(Cin % 64 == 0 && Cout % 64 == 0, "aph_vqgan_conv_test: C_in=%d and C_out=%d must be multiples of 64", Cin, Cout);
  cudaStream_t st = (cudaStream_t)stream;
  StreamTemp<bf16> wp;
  if (int r = wp.alloc((size_t)Cout * Cin * 9, st)) return r;
  if (int r = pack_conv3x3(weight, Cout, Cin, wp.p, nullptr, st)) return r;
  ConvEpi c; c.bias = bias; c.resid = reinterpret_cast<const bf16*>(resid); c.out = reinterpret_cast<bf16*>(out);
  return launch_conv3x3(x, wp.p, N, H, W, Cin, Cout, resid ? CONV_BIAS_RESID : CONV_BIAS, c, st);
}

// Nearest x2 upsample, bf16 NHWC, C % 8 == 0. fwd = 1: in [N,H,W,C] -> out [N,2H,2W,C]; fwd = 0: in = dy [N,2H,2W,C] -> out
// [N,H,W,C] = its adjoint, the sum of each 2 x 2 window.
extern "C" int aph_vqgan_up_test(int fwd, const void* in, void* out, int N, int H, int W, int C, void* stream) {
  APH_REQUIRE(in && out && N > 0 && H > 0 && W > 0 && C % 8 == 0 && C > 0, "aph_vqgan_up_test: bad arguments");
  const bf16* x = reinterpret_cast<const bf16*>(in);
  bf16* y = reinterpret_cast<bf16*>(out);
  cudaStream_t st = (cudaStream_t)stream;
  if (fwd) return launch_unpool2(x, nullptr, N, 2 * H, 2 * W, C, 1.f, y, st);
  return launch_pool2(POOL_SUM, x, N, 2 * H, 2 * W, C, y, st);
}

extern "C" int aph_vqgan_attn_test(int fwd, const void* qkv, const void* dout, void* out, int N, int T, int C, void* stream) {
  APH_REQUIRE(qkv && out && (fwd || dout) && N > 0 && T > 0 && T <= APH_VQGAN_MAX_TOKENS, "aph_vqgan_attn_test: bad arguments");
  APH_REQUIRE(C % 128 == 0 && C > 0, "aph_vqgan_attn_test: C=%d is not a multiple of 128", C);
  cudaStream_t st = (cudaStream_t)stream;
  const size_t Tp = vq_tpad(T);
  StreamTemp<float> F;
  StreamTemp<bf16> A, X, Kc, Kt, P, O;
  int e = F.alloc(T * Tp, st) | A.alloc(T * Tp, st) | X.alloc(Tp * Tp, st) | Kc.alloc(Tp * C, st) | Kt.alloc(Tp * C, st) |
          P.alloc(T * Tp, st) | O.alloc((size_t)T * C, st);
  if (e) return e;
  const AttnScratch s{F.p, A.p, X.p, Kc.p, Kt.p};
  const bf16* q = reinterpret_cast<const bf16*>(qkv);
  for (int n = 0; n < N; ++n) {
    const bf16* qn = q + (size_t)n * T * 3 * C;
    if (fwd) {
      if ((e = attn_fwd_img(qn, T, C, P.p, reinterpret_cast<bf16*>(out) + (size_t)n * T * C, s, st))) return e;
    } else {
      if ((e = attn_fwd_img(qn, T, C, P.p, O.p, s, st))) return e;
      if ((e = attn_bwd_img(qn, P.p, O.p, reinterpret_cast<const bf16*>(dout) + (size_t)n * T * C, T, C,
                            reinterpret_cast<bf16*>(out) + (size_t)n * T * 3 * C, s, st))) return e;
    }
  }
  return 0;
}

extern "C" int aph_vqgan_ends_test(int kind, const void* in, const float* weight, const float* bias, void* out, int N, int C, int H, int W,
                                   void* stream) {
  APH_REQUIRE(in && out && N > 0 && C > 0 && H > 0 && W > 0 && kind >= 0 && kind <= 3, "aph_vqgan_ends_test: bad arguments");
  cudaStream_t st = (cudaStream_t)stream;
  if (kind < 2) return layout(kind == 0, in, N, C, H * W, out, st);
  APH_REQUIRE(weight && (bias || kind == 3) && C % 8 == 0, "aph_vqgan_ends_test: conv_out needs weights and C %% 8 == 0");
  return conv_out(kind == 2, in, N, H, W, C, weight, bias, out, st);
}
