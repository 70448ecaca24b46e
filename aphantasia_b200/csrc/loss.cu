// loss.cu -- similarity loss (fused value + gradients) and the Adam update. fp32.
//
// aph_sim_fwd replaces sim_func(v1, v2, type) for type None/'cossim' and 'mix'
// (/root/reference/aphantasia/utils.py:276-282,295):
//     cos_s = <v1,v2_s> / (|v1| |v2_s|);   mix: f = cos - 0.25 * 2*asin(|v1^ - v2^_s| / 2)^2
//     value = mean_s f_s
// One warp per sample; gradients w.r.t. both operands are written in the same pass.
// aph_adam_step replaces torch.optim.Adam / AdamW's single-tensor update (/root/reference/clip_fft.py:108-115,295; adam.cuh).
#include "adam.cuh"
#include <algorithm>
#include <math.h>

namespace aph {

__global__ void __launch_bounds__(256) k_sim(const float* __restrict__ v1, int n1, const float* __restrict__ v2, int S, int D,
                                             int kind, float* __restrict__ value, float* __restrict__ g1, float* __restrict__ g2) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (warp >= S) return;
  const float* a = v1 + (size_t)(n1 == 1 ? 0 : warp) * D;
  const float* b = v2 + (size_t)warp * D;
  float dot = 0.f, na = 0.f, nb = 0.f;
  for (int i = lane; i < D; i += 32) { const float x = a[i], y = b[i]; dot += x * y; na += x * x; nb += y * y; }
  dot = warp_sum(dot); na = warp_sum(na); nb = warp_sum(nb);
  const float eps = 1e-8f;
  const float la = fmaxf(sqrtf(na), eps), lb = fmaxf(sqrtf(nb), eps);
  const float c = dot / (la * lb);
  float f = c, dfdc = 1.f;
  if (kind == APH_SIM_MIX) {
    // d^2 = |a^ - b^|^2 computed explicitly, as the reference does (F.normalize eps = 1e-12)
    const float ia = 1.f / fmaxf(sqrtf(na), 1e-12f), ib = 1.f / fmaxf(sqrtf(nb), 1e-12f);
    float d2 = 0.f;
    for (int i = lane; i < D; i += 32) { const float t = a[i] * ia - b[i] * ib; d2 += t * t; }
    d2 = warp_sum(d2);
    const float u = fminf(0.5f * sqrtf(d2), 1.f);
    const float as = asinf(u);
    f = c - 0.25f * fabsf(2.f * as * as);
    // f(c) = c - theta^2/8 with theta = 2 asin(u): df/dc = 1 + theta / (4 sin theta)
    const float theta = 2.f * as, st = sinf(theta);
    dfdc = 1.f + ((st > 1e-6f) ? theta / (4.f * st) : 0.25f);
  }
  const float invS = 1.f / (float)S;
  if (lane == 0) atomicAdd(value, f * invS);
  const float k = dfdc * invS;
  if (g2) {
    float* o = g2 + (size_t)warp * D;
    for (int i = lane; i < D; i += 32) o[i] = k * (a[i] / la - c * b[i] / lb) / lb;
  }
  if (g1) {
    if (n1 == 1) { for (int i = lane; i < D; i += 32) atomicAdd(&g1[i], k * (b[i] / lb - c * a[i] / la) / la); }
    else { float* o = g1 + (size_t)warp * D; for (int i = lane; i < D; i += 32) o[i] = k * (b[i] / lb - c * a[i] / la) / la; }
  }
}

__global__ void __launch_bounds__(256) k_adam(const float* __restrict__ g, size_t n, AdamArgs a) {
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) adam_elem(a, i, g[i]);
}

// ---- optional loss heads of the step (SURVEY 8 row f4) -----------------------------------------------------------
// derivat(img, mode='naiv') (/root/reference/aphantasia/utils.py:256-268, the only mode clip_fft.py:272 uses):
//   0.5 * (mean |img[..., x+1] - img[..., x]| + mean |img[..., y+1, :] - img[..., y, :]|)
// sums[0] / sums[1] accumulate the two absolute-difference sums in fp64; k_derivat_fin folds them into the value.
__global__ void __launch_bounds__(256) k_derivat_fwd(const float* __restrict__ img, int C, int H, int W, double* __restrict__ sums) {
  const size_t n = (size_t)C * H * W;
  double sx = 0., sy = 0.;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const int x = (int)(i % W), y = (int)((i / W) % H);
    const float v = img[i];
    if (x + 1 < W) sx += fabsf(img[i + 1] - v);
    if (y + 1 < H) sy += fabsf(img[i + W] - v);
  }
  block_atomic_add_d({sx, sy}, sums);
}
__global__ void k_derivat_fin(const double* __restrict__ sums, double nx, double ny, float* __restrict__ value) {
  *value = (float)(0.5 * (sums[0] / nx + sums[1] / ny));
}
__device__ __forceinline__ float sgnf(float d) { return (d > 0.f) ? 1.f : ((d < 0.f) ? -1.f : 0.f); }
// d value / d img, times the upstream gradient (a DEVICE scalar: no host sync)
__global__ void __launch_bounds__(256) k_derivat_bwd(const float* __restrict__ img, int C, int H, int W, const float* __restrict__ up,
                                                     float inv_nx, float inv_ny, float* __restrict__ grad) {
  const size_t n = (size_t)C * H * W;
  const float g = 0.5f * up[0];
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const int x = (int)(i % W), y = (int)((i / W) % H);
    const float v = img[i];
    float a = 0.f, b = 0.f;
    if (x > 0) a += sgnf(v - img[i - 1]);
    if (x + 1 < W) a -= sgnf(img[i + 1] - v);
    if (y > 0) b += sgnf(v - img[i - W]);
    if (y + 1 < H) b -= sgnf(img[i + W] - v);
    grad[i] = g * (a * inv_nx + b * inv_ny);
  }
}

// derivat(img, mode='sobel') (/root/reference/aphantasia/utils.py:262-264; cppn.py:291-292 --sharp):
//   mean |kornia.filters.spatial_gradient(img)|: the 3x3 Sobel pair normalised by 1/8, replicate padding, both directions,
//   the mean over the N C 2 H W outputs. sums[0] accumulates |gx| + |gy| in fp64; k_derivat_sobel_fin divides.
// gx (y, x) = (sum over the rows y-1, y, y+1 with weights 1, 2, 1 of p(., x+1) - p(., x-1)) / 8, indices clamped to the frame;
// gy is the same with the axes swapped.
__device__ __forceinline__ void sobel_at(const float* __restrict__ pl, int H, int W, int y, int x, float& gx, float& gy) {
  const int ym = max(y - 1, 0), yp = min(y + 1, H - 1), xm = max(x - 1, 0), xp = min(x + 1, W - 1);
  const float* rm = pl + (size_t)ym * W;
  const float* r0 = pl + (size_t)y * W;
  const float* rp = pl + (size_t)yp * W;
  gx = ((rm[xp] - rm[xm]) + 2.f * (r0[xp] - r0[xm]) + (rp[xp] - rp[xm])) * 0.125f;
  gy = ((rp[xm] - rm[xm]) + 2.f * (rp[x] - rm[x]) + (rp[xp] - rm[xp])) * 0.125f;
}
__global__ void __launch_bounds__(256) k_derivat_sobel_fwd(const float* __restrict__ img, int C, int H, int W, double* __restrict__ sums) {
  const size_t hw = (size_t)H * W, n = (size_t)C * hw;
  double s = 0.;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const size_t c = i / hw, q = i - c * hw;
    const int y = (int)(q / W), x = (int)(q - (size_t)y * W);
    float gx, gy;
    sobel_at(img + c * hw, H, W, y, x, gx, gy);
    s += fabsf(gx) + fabsf(gy);
  }
  block_atomic_add_d({s}, sums);
}
__global__ void k_derivat_sobel_fin(const double* __restrict__ sums, double n, float* __restrict__ value) { *value = (float)(sums[0] / n); }
// Adjoint: pixel (yy, xx) gathers sign(g) k from every output (y, x) within one pixel whose clamped tap lands on it (several
// taps of an edge output land on the same edge pixel), times upstream / (8 N C 2 H W). sign(0) = 0, as torch.abs's gradient.
__global__ void __launch_bounds__(256) k_derivat_sobel_bwd(const float* __restrict__ img, int C, int H, int W, const float* __restrict__ up,
                                                           float scale, float* __restrict__ grad) {
  const size_t hw = (size_t)H * W, n = (size_t)C * hw;
  const float g = up[0] * scale;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const size_t c = i / hw, q = i - c * hw;
    const int yy = (int)(q / W), xx = (int)(q - (size_t)yy * W);
    const float* pl = img + c * hw;
    float acc = 0.f;                       // integer-valued: exact
    for (int y = max(yy - 1, 0); y <= min(yy + 1, H - 1); ++y)
      for (int x = max(xx - 1, 0); x <= min(xx + 1, W - 1); ++x) {
        float gx, gy;
        sobel_at(pl, H, W, y, x, gx, gy);
        const float sx = sgnf(gx), sy = sgnf(gy);
        if (sx == 0.f && sy == 0.f) continue;
        for (int a = 0; a < 3; ++a) {
          if (min(max(y + a - 1, 0), H - 1) != yy) continue;
          for (int b = 0; b < 3; ++b) {
            if (min(max(x + b - 1, 0), W - 1) != xx) continue;
            // Sobel taps (row a, column b): x kernel (b - 1) (2 - |a - 1|), y kernel (a - 1) (2 - |b - 1|)
            acc += sx * (float)((b - 1) * (2 - abs(a - 1))) + sy * (float)((a - 1) * (2 - abs(b - 1)));
          }
        }
      }
    grad[i] = g * acc;
  }
}

// Linear head on the embeddings (the LAION aesthetic predictor of --aest is nn.Linear(512, 1), utils.py:402-413; clip_fft.py:255-256):
// out[s] = <emb_s, w> + b; one warp per sample.
__global__ void __launch_bounds__(256) k_head_fwd(const float* __restrict__ emb, int S, int D, const float* __restrict__ w,
                                                  const float* __restrict__ b, float* __restrict__ out) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (warp >= S) return;
  const float* e = emb + (size_t)warp * D;
  float acc = 0.f;
  for (int i = lane; i < D; i += 32) acc += e[i] * w[i];
  acc = warp_sum(acc);
  if (lane == 0) out[warp] = acc + (b ? b[0] : 0.f);
}
__global__ void __launch_bounds__(256) k_head_bwd(const float* __restrict__ g, const float* __restrict__ w, int S, int D, float* __restrict__ grad_emb) {
  const size_t n = (size_t)S * D;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
    grad_emb[i] = g[i / D] * w[i % D];
}

}  // namespace aph

using namespace aph;

extern "C" int aph_derivat_fwd(const float* img, int C, int H, int W, double* sums, float* value, void* stream) {
  APH_REQUIRE(img && sums && value && C > 0 && H > 1 && W > 1, "aph_derivat_fwd: bad arguments");
  cudaStream_t st = (cudaStream_t)stream;
  APH_CUDA_OK(cudaMemsetAsync(sums, 0, 2 * sizeof(double), st));
  const size_t n = (size_t)C * H * W;
  const int blocks = stride_blocks(n, 8);
  k_derivat_fwd<<<blocks, 256, 0, st>>>(img, C, H, W, sums);
  APH_LAUNCH_OK();
  k_derivat_fin<<<1, 1, 0, st>>>(sums, (double)C * H * (W - 1), (double)C * (H - 1) * W, value);
  APH_LAUNCH_OK();
  return 0;
}

extern "C" int aph_derivat_bwd(const float* img, int C, int H, int W, const float* upstream, float* grad_img, void* stream) {
  APH_REQUIRE(img && upstream && grad_img && C > 0 && H > 1 && W > 1, "aph_derivat_bwd: bad arguments");
  const size_t n = (size_t)C * H * W;
  const int blocks = stride_blocks(n, 8);
  k_derivat_bwd<<<blocks, 256, 0, (cudaStream_t)stream>>>(img, C, H, W, upstream, (float)(1.0 / ((double)C * H * (W - 1))),
                                                         (float)(1.0 / ((double)C * (H - 1) * W)), grad_img);
  APH_LAUNCH_OK();
  return 0;
}

extern "C" int aph_derivat_sobel_fwd(const float* img, int C, int H, int W, double* sums, float* value, void* stream) {
  APH_REQUIRE(img && sums && value && C > 0 && H > 0 && W > 0, "aph_derivat_sobel_fwd: bad arguments");
  cudaStream_t st = (cudaStream_t)stream;
  APH_CUDA_OK(cudaMemsetAsync(sums, 0, sizeof(double), st));
  const size_t n = (size_t)C * H * W;
  const int blocks = stride_blocks(n, 8);
  k_derivat_sobel_fwd<<<blocks, 256, 0, st>>>(img, C, H, W, sums);
  APH_LAUNCH_OK();
  k_derivat_sobel_fin<<<1, 1, 0, st>>>(sums, 2.0 * (double)n, value);
  APH_LAUNCH_OK();
  return 0;
}

extern "C" int aph_derivat_sobel_bwd(const float* img, int C, int H, int W, const float* upstream, float* grad_img, void* stream) {
  APH_REQUIRE(img && upstream && grad_img && C > 0 && H > 0 && W > 0, "aph_derivat_sobel_bwd: bad arguments");
  const size_t n = (size_t)C * H * W;
  const int blocks = stride_blocks(n, 8);
  k_derivat_sobel_bwd<<<blocks, 256, 0, (cudaStream_t)stream>>>(img, C, H, W, upstream, (float)(1.0 / (16.0 * (double)n)), grad_img);
  APH_LAUNCH_OK();
  return 0;
}

extern "C" int aph_head_fwd(const float* emb, int S, int D, const float* w, const float* b, float* out, void* stream) {
  APH_REQUIRE(emb && w && out && S > 0 && D > 0, "aph_head_fwd: bad arguments");
  k_head_fwd<<<(S * 32 + 255) / 256, 256, 0, (cudaStream_t)stream>>>(emb, S, D, w, b, out);
  APH_LAUNCH_OK();
  return 0;
}

extern "C" int aph_head_bwd(const float* grad_out, const float* w, int S, int D, float* grad_emb, void* stream) {
  APH_REQUIRE(grad_out && w && grad_emb && S > 0 && D > 0, "aph_head_bwd: bad arguments");
  const size_t n = (size_t)S * D;
  const int blocks = stride_blocks(n, 8);
  k_head_bwd<<<blocks, 256, 0, (cudaStream_t)stream>>>(grad_out, w, S, D, grad_emb);
  APH_LAUNCH_OK();
  return 0;
}

extern "C" int aph_sim_fwd(const float* v1, int n1, const float* v2, int S, int D, int kind, float* value, float* grad_v1,
                           float* grad_v2, void* stream) {
  APH_REQUIRE(v1 && v2 && value && S > 0 && D > 0, "aph_sim_fwd: bad arguments");
  APH_REQUIRE(n1 == 1 || n1 == S, "aph_sim_fwd: v1 rows (%d) must be 1 or S (%d)", n1, S);
  APH_REQUIRE(kind == APH_SIM_COS || kind == APH_SIM_MIX, "aph_sim_fwd: unknown kind %d", kind);
  cudaStream_t st = (cudaStream_t)stream;
  APH_CUDA_OK(cudaMemsetAsync(value, 0, sizeof(float), st));
  if (grad_v1 && n1 == 1) APH_CUDA_OK(cudaMemsetAsync(grad_v1, 0, (size_t)D * sizeof(float), st));
  const int blocks = (S * 32 + 255) / 256;
  k_sim<<<blocks, 256, 0, st>>>(v1, n1, v2, S, D, kind, value, grad_v1, grad_v2);
  APH_LAUNCH_OK();
  return 0;
}

extern "C" int aph_adam_step(float* p, const float* g, float* m, float* v, int64_t n, float lr, float b1, float b2, float eps,
                             int step, void* stream, float weight_decay, float* vmax) {
  APH_REQUIRE(p && g && m && v && n > 0 && step >= 1, "aph_adam_step: bad arguments");
  const int blocks = stride_blocks((size_t)n, 8);
  k_adam<<<blocks, 256, 0, (cudaStream_t)stream>>>(g, (size_t)n, make_adam(p, m, v, vmax, lr, b1, b2, eps, weight_decay, step));
  APH_LAUNCH_OK();
  return 0;
}
