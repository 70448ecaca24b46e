// sample.cu -- fused multi-crop sampler + transforms_fast, forward and backward (fp32, L2/HBM-bound).
//
// Replaces the per-crop Python loop of /root/reference/aphantasia/utils.py:243-253 (slice_imgs) with
// transforms_fast (/root/reference/aphantasia/transforms.py:165-170) applied per crop:
//   1. cut = canvas[oy:oy+cs, ox:ox+cs]; bicubic (A=-0.75, align_corners=True, taps clamped to the crop)
//      resize to size x size                                       (utils.py:248-249; SURVEY.md D2)
//   2. RandomPerspective hit: bilinear grid_sample(zeros, align_corners=False) of [img; ones],
//      out = img_s * mask_s                                        (torchvision _functional_tensor.py:545-576,672-698)
//   3. RandomErasing hit: rectangle -> 0                           (_functional_tensor.py:931-938)
//   4. rotate (always, even 0 deg): affine grid + the same masked grid_sample (transforms.py:80,
//      _functional_tensor.py:579-618)
//   5. (x - mean) / std with the CLIP constants                    (transforms.py:106-108)
// The stages are SEQUENTIAL resamplings of intermediate size x size images; stages 2-5 are evaluated by exact tap composition
// (rotate tap -> erase test -> perspective taps) on top of the resized crop, so every intermediate is the reference's intermediate.
//
// Default kernels (round 2):
//   forward : k_resize (stage 1, separable, into a library scratch image) + k_compose (stages 2-5, three channels per thread; optionally
//             also the encoder's bf16 patch operand, aph_sample_fwd_patches);
//   backward: k_bwd_warp_adjoint (perspective crops: rotation adjoint as a gather, perspective adjoint by global reductions into a
//             scratch image) + k_bwd_bicubic3 (every crop: rotation adjoint gathered inline, bicubic adjoint through per-warp strips
//             and 16-byte vector reductions into the canvas gradient).
// The round-1 one-kernel forms (one CTA per (crop, channel), the crop's resized image / gradient image in 196 KB of shared memory:
// k_sample_fwd, k_sample_bwd_cas, k_sample_bwd) and the atomic-free tile gather stay selectable (APH_SAMPLE_FWD_OLD, APH_SAMPLE_BWD_OLD,
// APH_SAMPLE_BWD_FIXED, APH_SAMPLE_BWD_GATHER) and are what tests/test_gpu_parity.py::test_sampler_backward_variants_agree compares.
#include "aph_common.cuh"
#include <stdlib.h>
#include <stdint.h>

namespace aph {

constexpr float kCubicA = -0.75f;
__device__ __forceinline__ float cubic1(float x) { return ((kCubicA + 2.f) * x - (kCubicA + 3.f)) * x * x + 1.f; }
__device__ __forceinline__ float cubic2(float x) { return ((kCubicA * x - 5.f * kCubicA) * x + 8.f * kCubicA) * x - 4.f * kCubicA; }

struct CropParams {
  int oy, ox, cs, flags;
  float pc[8];
  int ei, ej, eh, ew;
  float r00, r01, r10, r11;
  float rs[4];     // r.. / (size/2): the affine grid of the rotate stage in normalised coordinates (prescale())
  float ps[6];     // pc[0..5] / (size/2)
};

// divisions of the grid builders, hoisted out of the per-pixel code (one CTA = one crop)
__device__ __forceinline__ void prescale(CropParams& p, int size) {
  const float half = 0.5f * (float)size;
  p.rs[0] = p.r00 / half; p.rs[1] = p.r01 / half; p.rs[2] = p.r10 / half; p.rs[3] = p.r11 / half;
#pragma unroll
  for (int i = 0; i < 6; ++i) p.ps[i] = p.pc[i] / half;
}

__device__ __forceinline__ CropParams load_params(const float* __restrict__ row) {
  CropParams p;
  p.oy = (int)row[APH_F_OFFY]; p.ox = (int)row[APH_F_OFFX]; p.cs = (int)row[APH_F_CSIZE]; p.flags = (int)row[APH_F_FLAGS];
#pragma unroll
  for (int i = 0; i < 8; ++i) p.pc[i] = row[APH_F_PERSP + i];
  p.ei = (int)row[APH_F_ER_I]; p.ej = (int)row[APH_F_ER_J]; p.eh = (int)row[APH_F_ER_H]; p.ew = (int)row[APH_F_ER_W];
  p.r00 = row[APH_F_ROT]; p.r01 = row[APH_F_ROT + 1]; p.r10 = row[APH_F_ROT + 2]; p.r11 = row[APH_F_ROT + 3];
  if (!(p.flags & APH_FLAG_ERASE)) { p.eh = 0; p.ew = 0; }
  p.rs[0] = p.rs[1] = p.rs[2] = p.rs[3] = 0.f;
#pragma unroll
  for (int i = 0; i < 6; ++i) p.ps[i] = 0.f;
  return p;
}

// bicubic source index + 4 weights for output index i (align_corners=True)
__device__ __forceinline__ void cubic_taps(int i, float scale, int cs, int idx[4], float w[4]) {
  const float real = scale * (float)i;
  int i0 = (int)floorf(real);
  i0 = min(i0, cs - 1);
  float t = fminf(fmaxf(real - (float)i0, 0.f), 1.f);
  w[0] = cubic2(t + 1.f); w[1] = cubic1(t); w[2] = cubic1(1.f - t); w[3] = cubic2(2.f - t);
#pragma unroll
  for (int a = 0; a < 4; ++a) idx[a] = max(min(i0 - 1 + a, cs - 1), 0);
}

// bilinear grid_sample taps (align_corners=False, zeros padding) for normalised coords (gx, gy).
struct Bilin { int x0, y0; float w00, w01, w10, w11; };   // wYX; taps (y0,x0) (y0,x0+1) (y0+1,x0) (y0+1,x0+1)
__device__ __forceinline__ Bilin bilin_taps(float gx, float gy, int size) {
  const float ix = ((gx + 1.f) * (float)size - 1.f) * 0.5f;
  const float iy = ((gy + 1.f) * (float)size - 1.f) * 0.5f;
  const float fx = floorf(ix), fy = floorf(iy);
  Bilin b;
  b.x0 = (int)fx; b.y0 = (int)fy;
  const float tx = ix - fx, ty = iy - fy;
  b.w00 = (1.f - tx) * (1.f - ty); b.w01 = tx * (1.f - ty);
  b.w10 = (1.f - tx) * ty;         b.w11 = tx * ty;
  const bool xin0 = b.x0 >= 0 && b.x0 < size, xin1 = b.x0 + 1 >= 0 && b.x0 + 1 < size;
  const bool yin0 = b.y0 >= 0 && b.y0 < size, yin1 = b.y0 + 1 >= 0 && b.y0 + 1 < size;
  if (!(xin0 && yin0)) b.w00 = 0.f;
  if (!(xin1 && yin0)) b.w01 = 0.f;
  if (!(xin0 && yin1)) b.w10 = 0.f;
  if (!(xin1 && yin1)) b.w11 = 0.f;
  return b;
}

__device__ __forceinline__ Bilin rot_taps(const CropParams& p, int i, int j, int size) {
  const float half = 0.5f * (float)size;
  const float bx = (float)j + 0.5f - half, by = (float)i + 0.5f - half;
  const float gx = bx * p.rs[0] + by * p.rs[1];
  const float gy = bx * p.rs[2] + by * p.rs[3];
  return bilin_taps(gx, gy, size);
}

__device__ __forceinline__ Bilin persp_taps(const CropParams& p, int y, int x, int size) {
  const float bx = (float)x + 0.5f, by = (float)y + 0.5f;
  const float n1x = bx * p.ps[0] + by * p.ps[1] + p.ps[2];
  const float n1y = bx * p.ps[3] + by * p.ps[4] + p.ps[5];
  const float den = bx * p.pc[6] + by * p.pc[7] + 1.f;
  const float inv = __fdividef(1.f, den);          // MUFU.RCP (<= 2 ulp); forward and backward share these taps
  return bilin_taps(n1x * inv - 1.f, n1y * inv - 1.f, size);
}

// erase rectangle test; an unset flag is folded into an empty rectangle by load_params (eh = ew = 0)
__device__ __forceinline__ bool erased(const CropParams& p, int y, int x) {
  return (unsigned)(y - p.ei) < (unsigned)p.eh && (unsigned)(x - p.ej) < (unsigned)p.ew;
}

__device__ __forceinline__ float tap_dot(const float* __restrict__ A, const Bilin& b, int size) {
  float v = 0.f;
  if (b.w00 != 0.f) v += b.w00 * A[b.y0 * size + b.x0];
  if (b.w01 != 0.f) v += b.w01 * A[b.y0 * size + b.x0 + 1];
  if (b.w10 != 0.f) v += b.w10 * A[(b.y0 + 1) * size + b.x0];
  if (b.w11 != 0.f) v += b.w11 * A[(b.y0 + 1) * size + b.x0 + 1];
  return v;
}

// value of the post-perspective, post-erase image B at integer pixel (y, x)
template <bool PERSP, bool ERASE = true>
__device__ __forceinline__ float stageB(const float* __restrict__ A, const CropParams& p, int y, int x, int size) {
  if (ERASE && erased(p, y, x)) return 0.f;
  if (PERSP) {
    const Bilin b = persp_taps(p, y, x, size);
    const float mask = b.w00 + b.w01 + b.w10 + b.w11;
    return tap_dot(A, b, size) * mask;
  }
  return A[y * size + x];
}

__constant__ float c_inv_std[3] = {1.f / 0.26862954f, 1.f / 0.26130258f, 1.f / 0.27577711f};
__constant__ float c_shift[3] = {-0.48145466f / 0.26862954f, -0.4578275f / 0.26130258f, -0.40821073f / 0.27577711f};

// the rotate stage is the identity resampling (angle 0: theta = [[1, 0], [0, 1]])
__device__ __forceinline__ bool identity_rot(const CropParams& p) { return p.r00 == 1.f && p.r01 == 0.f && p.r10 == 0.f && p.r11 == 1.f; }

__constant__ float c_mean[3] = {0.48145466f, 0.4578275f, 0.40821073f};
__constant__ float c_std[3] = {0.26862954f, 0.26130258f, 0.27577711f};

// Per-CTA tap tables: the 4 bicubic taps (canvas offset, weight) of every output row and column, computed once
// (size entries each) instead of per pixel; wrap-around ('over*' frames) is folded into the stored canvas index.
constexpr int STRIP = 128;     // per-warp strip (floats) used by the separable bicubic stage
struct TapTables { int* xo; float* xw; int* yo; float* yw; };
__device__ __forceinline__ TapTables build_taps(float* base, const CropParams& p, int size, int H, int W, int pad_top, int pad_left, float scale) {
  TapTables t;
  t.xo = reinterpret_cast<int*>(base); t.xw = base + 4 * size; t.yo = reinterpret_cast<int*>(base + 8 * size); t.yw = base + 12 * size;
  for (int k = threadIdx.x; k < 2 * size; k += blockDim.x) {
    const bool isy = k >= size;
    const int o = isy ? k - size : k;
    int idx[4]; float w[4];
    cubic_taps(o, scale, p.cs, idx, w);
#pragma unroll
    for (int a = 0; a < 4; ++a) {
      if (isy) { int y = p.oy + idx[a] - pad_top; y %= H; if (y < 0) y += H; t.yo[4 * o + a] = y * W; t.yw[4 * o + a] = w[a]; }
      else { int x = p.ox + idx[a] - pad_left; x %= W; if (x < 0) x += W; t.xo[4 * o + a] = x; t.xw[4 * o + a] = w[a]; }
    }
  }
  return t;
}

// rotate tap -> erase test -> perspective taps on top of the resized image A, then the CLIP normalisation as one FMA
template <bool PERSP, bool ERASE = true>
__device__ __forceinline__ void fwd_compose(const float* __restrict__ A, const CropParams& p, int size, int warp, int lane, int nwarps,
                                            float inv_sd, float shift, float* __restrict__ o) {
  for (int i = warp; i < size; i += nwarps) {
    for (int j = lane; j < size; j += 32) {
      const Bilin b = rot_taps(p, i, j, size);
      const float mask = b.w00 + b.w01 + b.w10 + b.w11;
      float s = 0.f;
      if (b.w00 != 0.f) s += b.w00 * stageB<PERSP, ERASE>(A, p, b.y0, b.x0, size);
      if (b.w01 != 0.f) s += b.w01 * stageB<PERSP, ERASE>(A, p, b.y0, b.x0 + 1, size);
      if (b.w10 != 0.f) s += b.w10 * stageB<PERSP, ERASE>(A, p, b.y0 + 1, b.x0, size);
      if (b.w11 != 0.f) s += b.w11 * stageB<PERSP, ERASE>(A, p, b.y0 + 1, b.x0 + 1, size);
      o[i * size + j] = fmaf(s * mask, inv_sd, shift);
    }
  }
}

__global__ void __launch_bounds__(1024, 1)
k_sample_fwd(const float* __restrict__ canvas, int H, int W, int pad_top, int pad_left, const float* __restrict__ table,
             int size, int kind, float* __restrict__ out) {
  extern __shared__ float A[];
  const int crop = blockIdx.x / 3, ch = blockIdx.x - crop * 3;
  CropParams p = load_params(table + (size_t)crop * APH_CROP_PARAM_FLOATS);
  prescale(p, size);
  const float* cch = canvas + (size_t)ch * H * W;
  const float scale = (size > 1) ? (float)(p.cs - 1) / (float)(size - 1) : 0.f;
  const int n = size * size;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nwarps = blockDim.x >> 5;
  const TapTables tt = build_taps(A + ((n + 3) & ~3), p, size, H, W, pad_top, pad_left, scale);
  __syncthreads();
  // ---- stage 1: bicubic resize into shared memory (warp = output row), direct 16-tap form through the per-CTA tap tables.
  // (A vertical-first per-warp strip variant was slower here: two extra warp barriers
  // and a dependent shared-memory round trip per chunk outweigh the saved L1 wavefronts; the backward keeps its strip.)
  for (int i = warp; i < size; i += nwarps) {
    const int4 yo = *reinterpret_cast<const int4*>(tt.yo + 4 * i);
    const float4 wy = *reinterpret_cast<const float4*>(tt.yw + 4 * i);
    const float* r0 = cch + yo.x; const float* r1 = cch + yo.y; const float* r2 = cch + yo.z; const float* r3 = cch + yo.w;
    for (int j0 = 0; j0 < size; j0 += 32) {
      const int j = j0 + lane;
      const int jc = min(j, size - 1);
      const int4 xo = *reinterpret_cast<const int4*>(tt.xo + 4 * jc);
      const float4 wx = *reinterpret_cast<const float4*>(tt.xw + 4 * jc);
      const float v0 = wx.x * __ldg(r0 + xo.x) + wx.y * __ldg(r0 + xo.y) + wx.z * __ldg(r0 + xo.z) + wx.w * __ldg(r0 + xo.w);
      const float v1 = wx.x * __ldg(r1 + xo.x) + wx.y * __ldg(r1 + xo.y) + wx.z * __ldg(r1 + xo.z) + wx.w * __ldg(r1 + xo.w);
      const float v2 = wx.x * __ldg(r2 + xo.x) + wx.y * __ldg(r2 + xo.y) + wx.z * __ldg(r2 + xo.z) + wx.w * __ldg(r2 + xo.w);
      const float v3 = wx.x * __ldg(r3 + xo.x) + wx.y * __ldg(r3 + xo.y) + wx.z * __ldg(r3 + xo.z) + wx.w * __ldg(r3 + xo.w);
      float acc = wy.x * v0;
      acc += wy.y * v1; acc += wy.z * v2; acc += wy.w * v3;
      if (j < size) A[i * size + j] = acc;
    }
  }
  __syncthreads();
  // ---- stages 2-5 by tap composition (the perspective branch is CTA-uniform: specialised loops)
  float* o = out + ((size_t)crop * 3 + ch) * n;
  const float inv_sd = 1.f / c_std[ch], shift = -c_mean[ch] * inv_sd;
  if (kind == APH_TF_FAST) {
    const bool er = (p.flags & APH_FLAG_ERASE) != 0;      // CTA-uniform: crops without an erase hit (80 %) skip the rectangle test per tap
    if (p.flags & APH_FLAG_PERSP) { if (er) fwd_compose<true, true>(A, p, size, warp, lane, nwarps, inv_sd, shift, o); else fwd_compose<true, false>(A, p, size, warp, lane, nwarps, inv_sd, shift, o); }
    else if (identity_rot(p)) {
      // angle 0 (26 % of the draws, transforms.py:168) without a perspective hit: the rotate stage resamples every pixel at its own
      // centre (bilinear weights (1, 0, 0, 0) up to 1e-6 round-off, coverage 1), so stages 2-5 reduce to erase + normalise.
      for (int idx = threadIdx.x; idx < n; idx += blockDim.x) {
        const int y = idx / size, x = idx - y * size;
        o[idx] = erased(p, y, x) ? shift : fmaf(A[idx], inv_sd, shift);
      }
    }
    else if (er) fwd_compose<false, true>(A, p, size, warp, lane, nwarps, inv_sd, shift, o);
    else fwd_compose<false, false>(A, p, size, warp, lane, nwarps, inv_sd, shift, o);
  } else {
    const float a = (kind != APH_TF_NONE) ? inv_sd : 1.f, b = (kind != APH_TF_NONE) ? shift : 0.f;
    for (int idx = threadIdx.x; idx < n; idx += blockDim.x) o[idx] = fmaf(A[idx], a, b);
  }
}


// ---------------------------------------------------------------------------------------------
// Forward, two-kernel form (round 2). The one-kernel form above keeps the resized crop of ONE channel in 196 KB of shared memory and
// recomputes the rotate / perspective geometry per channel; it is instruction-issue bound (~295 thread instructions per pixel and
// channel). Here
//   k_resize : stage 1 alone, SEPARABLE -- a warp owns an output row: vertical 4-tap pass over the crop's columns (coalesced row
//              reads) into a per-warp strip, then the horizontal 4-tap pass out of the strip; 8 rows of state per CTA, 7 CTAs / SM.
//              Result A [S,3,size,size] goes to a library scratch buffer (L2 / HBM), or straight to the output for transform kinds
//              without a warp stage.
//   k_compose: stages 2-5 for ALL THREE channels of a pixel per thread: one evaluation of the rotate (and perspective) taps,
//              4 (16) gathers per channel from the scratch image through L1.
// The encoder's patch-embedding GEMM reads its A operand patch-major in bf16: [S*g*g, 3*p*p], row = s*g*g + gy*g + gx,
// col = c*p*p + py*p + px (conv1 weight layout, vit_ops.cuh k_patchify). With `patches` set the sampler's last stage writes that
// operand beside the fp32 batch (SURVEY 2.4 k10-k12), so the encoder does not re-read 4 bytes per pixel to produce it.
struct PatchOut { __nv_bfloat16* base; int p, g; };
__device__ __forceinline__ size_t patch_index(const PatchOut& po, int s, int c, int i, int j) {
  const int gy = i / po.p, py = i - gy * po.p, gx = j / po.p, px = j - gx * po.p;
  return ((size_t)(s * po.g + gy) * po.g + gx) * (size_t)(3 * po.p * po.p) + (size_t)(c * po.p + py) * po.p + px;
}

template <bool WRAP>
__global__ void __launch_bounds__(256)
k_resize(const float* __restrict__ canvas, int H, int W, int pad_top, int pad_left, const float* __restrict__ table, int size, int rows_per_cta,
         int cap, int kind, float* __restrict__ dst, PatchOut po) {
  extern __shared__ float rs[];
  int* xi = reinterpret_cast<int*>(rs);              // [4*size] crop-relative source columns of every output column
  float* xw = rs + 4 * size;                         // [4*size] their weights
  const int crop = blockIdx.x / 3, ch = blockIdx.x - crop * 3;
  __shared__ int s_oy, s_ox, s_cs;
  if (threadIdx.x == 0) { const float* row = table + (size_t)crop * APH_CROP_PARAM_FLOATS; s_oy = (int)row[APH_F_OFFY]; s_ox = (int)row[APH_F_OFFX]; s_cs = (int)row[APH_F_CSIZE]; }
  __syncthreads();
  CropParams p; p.oy = s_oy; p.ox = s_ox; p.cs = s_cs;
  const float* cch = canvas + (size_t)ch * H * W;
  const float scale = (size > 1) ? (float)(p.cs - 1) / (float)(size - 1) : 0.f;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int k = threadIdx.x; k < size; k += blockDim.x) {
    int idx[4]; float w[4];
    cubic_taps(k, scale, p.cs, idx, w);
#pragma unroll
    for (int a = 0; a < 4; ++a) { xi[4 * k + a] = idx[a]; xw[4 * k + a] = w[a]; }
  }
  __syncthreads();
  float* strip = rs + 8 * size + warp * cap;
  const int n = size * size;
  float* o = dst + ((size_t)crop * 3 + ch) * n;
  const float na = (kind == APH_TF_NORMALIZE) ? 1.f / c_std[ch] : 1.f, nb = (kind == APH_TF_NORMALIZE) ? -c_mean[ch] / c_std[ch] : 0.f;
  const int r_end = min(size, ((int)blockIdx.y + 1) * rows_per_cta);
  for (int i = blockIdx.y * rows_per_cta + warp; i < r_end; i += 8) {
    int yidx[4]; float wy[4];
    cubic_taps(i, scale, p.cs, yidx, wy);
    const float* rp[4];
#pragma unroll
    for (int a = 0; a < 4; ++a) {
      int y = p.oy + yidx[a] - pad_top;
      if (WRAP) { y %= H; if (y < 0) y += H; }
      rp[a] = cch + y * W + (WRAP ? 0 : p.ox - pad_left);
    }
    if (WRAP) {
      for (int x = lane; x < p.cs; x += 32) {
        int col = (p.ox + x - pad_left) % W; if (col < 0) col += W;
        float v = wy[0] * __ldg(rp[0] + col);
        v += wy[1] * __ldg(rp[1] + col); v += wy[2] * __ldg(rp[2] + col); v += wy[3] * __ldg(rp[3] + col);
        strip[x] = v;
      }
    } else {
#pragma unroll 4
      for (int x = lane; x < p.cs; x += 32) {
        float v = wy[0] * __ldg(rp[0] + x);
        v += wy[1] * __ldg(rp[1] + x); v += wy[2] * __ldg(rp[2] + x); v += wy[3] * __ldg(rp[3] + x);
        strip[x] = v;
      }
    }
    __syncwarp();
    for (int j = lane; j < size; j += 32) {
      const int4 xo = *reinterpret_cast<const int4*>(xi + 4 * j);
      const float4 wx = *reinterpret_cast<const float4*>(xw + 4 * j);
      float acc = wx.x * strip[xo.x];
      acc += wx.y * strip[xo.y]; acc += wx.z * strip[xo.z]; acc += wx.w * strip[xo.w];
      const float v = (kind == APH_TF_FAST) ? acc : fmaf(acc, na, nb);
      o[i * size + j] = v;
      if (kind != APH_TF_FAST && po.base) po.base[patch_index(po, crop, ch, i, j)] = __float2bfloat16_rn(v);
    }
    __syncwarp();
  }
}

// value of the post-perspective, post-erase image B at integer pixel (y, x) for the three channels
template <bool PERSP, bool ERASE>
__device__ __forceinline__ void stageB3(const float* __restrict__ A, int n, const CropParams& p, int y, int x, int size, float w, float (&acc)[3]) {
  if (ERASE && erased(p, y, x)) return;
  if (PERSP) {
    const Bilin b = persp_taps(p, y, x, size);
    const float mw = (b.w00 + b.w01 + b.w10 + b.w11) * w;
    const int o = b.y0 * size + b.x0;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const float* Ac = A + c * n;
      float v = 0.f;
      if (b.w00 != 0.f) v += b.w00 * __ldg(Ac + o);
      if (b.w01 != 0.f) v += b.w01 * __ldg(Ac + o + 1);
      if (b.w10 != 0.f) v += b.w10 * __ldg(Ac + o + size);
      if (b.w11 != 0.f) v += b.w11 * __ldg(Ac + o + size + 1);
      acc[c] += v * mw;
    }
  } else {
    const int o = y * size + x;
#pragma unroll
    for (int c = 0; c < 3; ++c) acc[c] += w * __ldg(A + c * n + o);
  }
}

template <bool PERSP, bool ERASE>
__device__ __forceinline__ void compose3(const float* __restrict__ A, int n, const CropParams& p, int i, int j, int size, float* __restrict__ o,
                                         const PatchOut& po, int crop) {
  const Bilin b = rot_taps(p, i, j, size);
  const float mask = b.w00 + b.w01 + b.w10 + b.w11;
  float acc[3] = {0.f, 0.f, 0.f};
  if (b.w00 != 0.f) stageB3<PERSP, ERASE>(A, n, p, b.y0, b.x0, size, b.w00, acc);
  if (b.w01 != 0.f) stageB3<PERSP, ERASE>(A, n, p, b.y0, b.x0 + 1, size, b.w01, acc);
  if (b.w10 != 0.f) stageB3<PERSP, ERASE>(A, n, p, b.y0 + 1, b.x0, size, b.w10, acc);
  if (b.w11 != 0.f) stageB3<PERSP, ERASE>(A, n, p, b.y0 + 1, b.x0 + 1, size, b.w11, acc);
  const int pix = i * size + j;
  const size_t pi = po.base ? patch_index(po, crop, 0, i, j) : 0;
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const float v = fmaf(acc[c] * mask, c_inv_std[c], c_shift[c]);
    o[c * n + pix] = v;
    if (po.base) po.base[pi + (size_t)c * po.p * po.p] = __float2bfloat16_rn(v);
  }
}

__global__ void __launch_bounds__(256)
k_compose(const float* __restrict__ Ag, const float* __restrict__ table, int size, float* __restrict__ out, PatchOut po) {
  const int crop = blockIdx.y, tiles_x = (size + 15) >> 4;
  const int ti = blockIdx.x / tiles_x, tj = blockIdx.x - ti * tiles_x;
  const int i = ti * 16 + (threadIdx.x >> 4), j = tj * 16 + (threadIdx.x & 15);
  __shared__ CropParams sp;                      // the crop's parameters are decoded once per CTA
  if (threadIdx.x == 0) { sp = load_params(table + (size_t)crop * APH_CROP_PARAM_FLOATS); prescale(sp, size); }
  __syncthreads();
  const CropParams p = sp;
  if (i >= size || j >= size) return;
  const int n = size * size;
  const float* A = Ag + (size_t)crop * 3 * n;
  float* o = out + (size_t)crop * 3 * n;
  const bool er = (p.flags & APH_FLAG_ERASE) != 0;
  if (p.flags & APH_FLAG_PERSP) { if (er) compose3<true, true>(A, n, p, i, j, size, o, po, crop); else compose3<true, false>(A, n, p, i, j, size, o, po, crop); }
  else if (identity_rot(p)) {
    const bool e = erased(p, i, j);
    const int pix = i * size + j;
    const size_t pi = po.base ? patch_index(po, crop, 0, i, j) : 0;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const float v = e ? c_shift[c] : fmaf(__ldg(A + c * n + pix), c_inv_std[c], c_shift[c]);
      o[c * n + pix] = v;
      if (po.base) po.base[pi + (size_t)c * po.p * po.p] = __float2bfloat16_rn(v);
    }
  }
  else if (er) compose3<false, true>(A, n, p, i, j, size, o, po, crop);
  else compose3<false, false>(A, n, p, i, j, size, o, po, crop);
}

// Shared-memory accumulation cell. fp32 atomicAdd on shared memory is a compare-and-swap loop on this architecture
// (SASS: ATOMS.CAST.SPIN, ~6 instructions and two dependent shared round trips per add; ncu: 31 % of the backward kernel's
// instructions, 44 % of its stall samples). The opt-in FIXED form (k_sample_bwd, APH_SAMPLE_BWD_FIXED=1) accumulates round(v * scale) with the native integer ATOMS.ADD instead; the
// scale is chosen per (crop, channel) from the block maximum so the sum cannot overflow, and the result is order-independent.
template <bool FIXED>
__device__ __forceinline__ void acc_add(float* __restrict__ cell, float v) {
  if (FIXED) atomicAdd(reinterpret_cast<int*>(cell), __float2int_rn(v));
  else atomicAdd(cell, v);
}

template <bool PERSP, bool FIXED, bool ERASE = true>
__device__ __forceinline__ void scatterB(float* __restrict__ gA, const CropParams& p, int y, int x, int size, float g) {
  if (ERASE && erased(p, y, x)) return;
  if (PERSP) {
    const Bilin b = persp_taps(p, y, x, size);
    const float gm = g * (b.w00 + b.w01 + b.w10 + b.w11);
    if (b.w00 != 0.f) acc_add<FIXED>(&gA[b.y0 * size + b.x0], gm * b.w00);
    if (b.w01 != 0.f) acc_add<FIXED>(&gA[b.y0 * size + b.x0 + 1], gm * b.w01);
    if (b.w10 != 0.f) acc_add<FIXED>(&gA[(b.y0 + 1) * size + b.x0], gm * b.w10);
    if (b.w11 != 0.f) acc_add<FIXED>(&gA[(b.y0 + 1) * size + b.x0 + 1], gm * b.w11);
  } else {
    acc_add<FIXED>(&gA[y * size + x], g);
  }
}

// adjoint of normalise -> rotate -> erase -> perspective: scatters grad_out of one (crop, channel) into the shared gradient
// image. `gscale` = 1/std (fp32 cells) or fixed_scale/std (integer cells).
template <bool PERSP, bool FIXED, bool ERASE = true>
__device__ __forceinline__ void bwd_compose(float* __restrict__ gA, const float* __restrict__ go, const CropParams& p, int size,
                                            int warp, int lane, int nwarps, float gscale) {
  for (int i = warp; i < size; i += nwarps) {
    float gnext = (lane < size) ? go[i * size + lane] : 0.f;
    for (int j = lane; j < size; j += 32) {
      const float graw = gnext;
      if (j + 32 < size) gnext = go[i * size + j + 32];            // next chunk's load overlaps this chunk's scatter
      const Bilin b = rot_taps(p, i, j, size);
      const float g = graw * gscale * (b.w00 + b.w01 + b.w10 + b.w11);
      if (g == 0.f) continue;
      if (b.w00 != 0.f) scatterB<PERSP, FIXED, ERASE>(gA, p, b.y0, b.x0, size, g * b.w00);
      if (b.w01 != 0.f) scatterB<PERSP, FIXED, ERASE>(gA, p, b.y0, b.x0 + 1, size, g * b.w01);
      if (b.w10 != 0.f) scatterB<PERSP, FIXED, ERASE>(gA, p, b.y0 + 1, b.x0, size, g * b.w10);
      if (b.w11 != 0.f) scatterB<PERSP, FIXED, ERASE>(gA, p, b.y0 + 1, b.x0 + 1, size, g * b.w11);
    }
  }
}

// block-wide maximum (all threads get it); `red` = 32 floats of shared scratch
__device__ __forceinline__ float block_max(float v, float* red) {
  v = warp_max(v);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  float m = (threadIdx.x & 31) < (blockDim.x >> 5) ? red[threadIdx.x & 31] : 0.f;
  return warp_max(m);
}

// bicubic adjoint of the shared gradient image gA into the canvas gradient. Per 32-pixel chunk of a gradient row the horizontal
// taps are first accumulated into a per-warp strip (the lanes' 4-tap windows overlap), then the strip is scattered to the 4
// source rows with COALESCED global red.add (4 x span instead of 16 x 32 scattered atomics per chunk).
template <bool FIXED>
__device__ __forceinline__ void bwd_bicubic(const float* __restrict__ gA, float* __restrict__ strip, const TapTables& tt, float* __restrict__ gc,
                                            int size, int warp, int lane, int nwarps, bool can_strip, float sscale, float inv_sscale) {
  for (int i = warp; i < size; i += nwarps) {
    const int4 yo = *reinterpret_cast<const int4*>(tt.yo + 4 * i);
    const float4 wy = *reinterpret_cast<const float4*>(tt.yw + 4 * i);
    const int yoff[4] = {yo.x, yo.y, yo.z, yo.w};
    const float wya[4] = {wy.x, wy.y, wy.z, wy.w};
    for (int j0 = 0; j0 < size; j0 += 32) {
      const int j = j0 + lane;
      const float g = (j < size) ? gA[i * size + j] : 0.f;
      const int jc = min(j, size - 1);
      const int4 xo = *reinterpret_cast<const int4*>(tt.xo + 4 * jc);
      const float4 wx = *reinterpret_cast<const float4*>(tt.xw + 4 * jc);
      const int xfirst = tt.xo[4 * j0], xlast = tt.xo[4 * min(j0 + 31, size - 1) + 3];
      const int span = xlast - xfirst + 1;
      if (can_strip && span <= STRIP) {
        if (g != 0.f) {
          const float gs = FIXED ? g * sscale : g;
          acc_add<FIXED>(&strip[xo.x - xfirst], gs * wx.x); acc_add<FIXED>(&strip[xo.y - xfirst], gs * wx.y);
          acc_add<FIXED>(&strip[xo.z - xfirst], gs * wx.z); acc_add<FIXED>(&strip[xo.w - xfirst], gs * wx.w);
        }
        __syncwarp();
        for (int x = lane; x < span; x += 32) {
          const float raw = strip[x];                                // all-zero bits in either representation = nothing landed here
          if (__float_as_int(raw) != 0) {
            strip[x] = 0.f;
            const float h = FIXED ? (float)__float_as_int(raw) * inv_sscale : raw;
#pragma unroll
            for (int a = 0; a < 4; ++a) atomicAdd(gc + yoff[a] + xfirst + x, wya[a] * h);
          }
        }
        __syncwarp();
      } else if (g != 0.f) {
#pragma unroll
        for (int a = 0; a < 4; ++a) {
          float* r = gc + yoff[a];
          const float gy = g * wya[a];
          atomicAdd(r + xo.x, gy * wx.x); atomicAdd(r + xo.y, gy * wx.y); atomicAdd(r + xo.z, gy * wx.z); atomicAdd(r + xo.w, gy * wx.w);
        }
      }
    }
  }
}

__global__ void __launch_bounds__(1024, 1)
k_sample_bwd(const float* __restrict__ grad_out, int H, int W, int pad_top, int pad_left, const float* __restrict__ table,
             int size, int kind, float* __restrict__ grad_canvas) {
  extern __shared__ float gA[];
  __shared__ float red[32];
  const int crop = blockIdx.x / 3, ch = blockIdx.x - crop * 3;
  CropParams p = load_params(table + (size_t)crop * APH_CROP_PARAM_FLOATS);
  prescale(p, size);
  const int n = size * size;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nwarps = blockDim.x >> 5;
  const float* go = grad_out + ((size_t)crop * 3 + ch) * n;
  const float inv_sd = (kind != APH_TF_NONE) ? 1.f / c_std[ch] : 1.f;
  const float scale = (size > 1) ? (float)(p.cs - 1) / (float)(size - 1) : 0.f;
  const TapTables tt = build_taps(gA + ((n + 3) & ~3), p, size, H, W, pad_top, pad_left, scale);
  float* strip = gA + ((n + 3) & ~3) + 16 * size + warp * STRIP;
  for (int x = lane; x < STRIP; x += 32) strip[x] = 0.f;           // the strip is re-zeroed as it is drained
  // block maximum of |grad_out| sizes the fixed-point scale (NaN / Inf -> INFINITY: fmaxf alone would drop a NaN); the same pass
  // clears (or, without transforms, fills) gA
  float amax = 0.f;
  if (kind == APH_TF_FAST) {
    for (int idx = threadIdx.x; idx < n; idx += blockDim.x) { const float a = fabsf(go[idx]); amax = (a <= 3e38f) ? fmaxf(amax, a) : INFINITY; gA[idx] = 0.f; }
  } else {
    for (int idx = threadIdx.x; idx < n; idx += blockDim.x) { const float v = go[idx] * inv_sd, a = fabsf(v); amax = (a <= 3e38f) ? fmaxf(amax, a) : INFINITY; gA[idx] = v; }
  }
  amax = block_max(amax, red);                                      // (contains the block barriers)
  if (amax == 0.f) return;                                          // nothing to add (block-uniform)
  float* gc = grad_canvas + (size_t)ch * H * W;
  const bool can_strip = (pad_top == 0 && pad_left == 0);
  if (!(amax < 1e30f)) {                                            // Inf / NaN upstream: poison this crop's footprint, as fp32 would
    for (int idx = threadIdx.x; idx < n; idx += blockDim.x) gA[idx] = __int_as_float(0x7fc00000);
    __syncthreads();
    bwd_bicubic<true>(gA, strip, tt, gc, size, warp, lane, nwarps, false, 1.f, 1.f);
    return;
  }
  float gmax = amax;                                                // bound on |gA| for the strip scale
  if (kind == APH_TF_FAST) {
    amax *= inv_sd;
    const bool persp = (p.flags & APH_FLAG_PERSP) != 0;
    // fan-in bound of one gradient cell: a rotation (area preserving) lands <= 8 weighted samples on a pixel, a perspective
    // warp of distortion <= 0.5 compresses area by far less than the extra 32x allowed here
    const float s1 = 2147483648.f / ((persp ? 512.f : 16.f) * amax);
    if (persp) bwd_compose<true, true>(gA, go, p, size, warp, lane, nwarps, inv_sd * s1);
    else bwd_compose<false, true>(gA, go, p, size, warp, lane, nwarps, inv_sd * s1);
    __syncthreads();
    const float inv_s1 = 1.f / s1;
    float m = 0.f;
    for (int idx = threadIdx.x; idx < n; idx += blockDim.x) {       // integer cells -> fp32 in place, and their maximum
      const float v = (float)__float_as_int(gA[idx]) * inv_s1;
      gA[idx] = v; m = fmaxf(m, fabsf(v));
    }
    gmax = block_max(m, red);
    if (gmax == 0.f) return;
  }
  // a strip cell sums <= 4 / min(scale, 1) horizontal taps of |weight| <= 1.2: 64x headroom covers crops down to size / 12
  const float s2 = 1073741824.f / (64.f * gmax);
  bwd_bicubic<true>(gA, strip, tt, gc, size, warp, lane, nwarps, can_strip && scale >= 0.08f, s2, 1.f / s2);
}

// Default backward: fp32 shared accumulation (compare-and-swap loops in SASS).
__global__ void __launch_bounds__(1024, 1)
k_sample_bwd_cas(const float* __restrict__ grad_out, int H, int W, int pad_top, int pad_left, const float* __restrict__ table,
             int size, int kind, float* __restrict__ grad_canvas, float gscale) {
  extern __shared__ float gA[];
  const int crop = blockIdx.x / 3, ch = blockIdx.x - crop * 3;
  CropParams p = load_params(table + (size_t)crop * APH_CROP_PARAM_FLOATS);
  prescale(p, size);
  const int n = size * size;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nwarps = blockDim.x >> 5;
  const float* go = grad_out + ((size_t)crop * 3 + ch) * n;
  // gscale: weight of this rank's shard in the all-reduced gradient (S_local / S under torchrun, 1 otherwise), folded in here
  const float inv_sd = ((kind != APH_TF_NONE) ? 1.f / c_std[ch] : 1.f) * gscale;
  const float scale = (size > 1) ? (float)(p.cs - 1) / (float)(size - 1) : 0.f;
  const TapTables tt = build_taps(gA + ((n + 3) & ~3), p, size, H, W, pad_top, pad_left, scale);
  float* strip = gA + ((n + 3) & ~3) + 16 * size + warp * STRIP;
  for (int x = lane; x < STRIP; x += 32) strip[x] = 0.f;           // the strip is re-zeroed as it is drained below
  if (kind == APH_TF_FAST && !(p.flags & APH_FLAG_PERSP) && identity_rot(p)) {
    // adjoint of the angle-0 fast path of the forward: erase mask + 1/std, no scatter
    for (int idx = threadIdx.x; idx < n; idx += blockDim.x) {
      const int y = idx / size, x = idx - y * size;
      gA[idx] = erased(p, y, x) ? 0.f : go[idx] * inv_sd;
    }
  } else if (kind == APH_TF_FAST) {
    for (int idx = threadIdx.x; idx < n; idx += blockDim.x) gA[idx] = 0.f;
    __syncthreads();
    const bool er = (p.flags & APH_FLAG_ERASE) != 0;
    if (p.flags & APH_FLAG_PERSP) { if (er) bwd_compose<true, false, true>(gA, go, p, size, warp, lane, nwarps, inv_sd); else bwd_compose<true, false, false>(gA, go, p, size, warp, lane, nwarps, inv_sd); }
    else if (er) bwd_compose<false, false, true>(gA, go, p, size, warp, lane, nwarps, inv_sd);
    else bwd_compose<false, false, false>(gA, go, p, size, warp, lane, nwarps, inv_sd);
  } else {
    for (int idx = threadIdx.x; idx < n; idx += blockDim.x) gA[idx] = go[idx] * inv_sd;
  }
  __syncthreads();
  // ---- bicubic adjoint. Per 32-pixel chunk of a gradient row the horizontal taps are first accumulated into a per-warp
  // strip (shared atomics, the lanes' 4-tap windows overlap), then the strip is scattered to the 4 source rows with
  // COALESCED global red.add (4 x span instead of 16 x 32 scattered atomics per chunk).
  float* gc = grad_canvas + (size_t)ch * H * W;
  const bool can_strip = (pad_top == 0 && pad_left == 0);
  for (int i = warp; i < size; i += nwarps) {
    const int4 yo = *reinterpret_cast<const int4*>(tt.yo + 4 * i);
    const float4 wy = *reinterpret_cast<const float4*>(tt.yw + 4 * i);
    const int yoff[4] = {yo.x, yo.y, yo.z, yo.w};
    const float wya[4] = {wy.x, wy.y, wy.z, wy.w};
    for (int j0 = 0; j0 < size; j0 += 32) {
      const int j = j0 + lane;
      const float g = (j < size) ? gA[i * size + j] : 0.f;
      const int jc = min(j, size - 1);
      const int4 xo = *reinterpret_cast<const int4*>(tt.xo + 4 * jc);
      const float4 wx = *reinterpret_cast<const float4*>(tt.xw + 4 * jc);
      const int xfirst = tt.xo[4 * j0], xlast = tt.xo[4 * min(j0 + 31, size - 1) + 3];
      const int span = xlast - xfirst + 1;
      if (can_strip && span <= STRIP) {
        if (g != 0.f) {
          atomicAdd(&strip[xo.x - xfirst], g * wx.x); atomicAdd(&strip[xo.y - xfirst], g * wx.y);
          atomicAdd(&strip[xo.z - xfirst], g * wx.z); atomicAdd(&strip[xo.w - xfirst], g * wx.w);
        }
        __syncwarp();
        for (int x = lane; x < span; x += 32) {
          const float h = strip[x];
          if (h != 0.f) {
            strip[x] = 0.f;
#pragma unroll
            for (int a = 0; a < 4; ++a) atomicAdd(gc + yoff[a] + xfirst + x, wya[a] * h);
          }
        }
        __syncwarp();
      } else if (g != 0.f) {
#pragma unroll
        for (int a = 0; a < 4; ++a) {
          float* r = gc + yoff[a];
          const float gy = g * wya[a];
          atomicAdd(r + xo.x, gy * wx.x); atomicAdd(r + xo.y, gy * wx.y); atomicAdd(r + xo.z, gy * wx.z); atomicAdd(r + xo.w, gy * wx.w);
        }
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------
// Atomic-free backward for un-wrapped frames (the script's default 'uniform' / 'central' aligns).
//   stage 1 (k_sample_bwd_stage1, transforms_fast only): rotate / erase / perspective adjoints per (crop, channel) in shared
//            memory, result gA [S,3,size,size] written to a library scratch buffer (L2-resident at these sizes);
//   stage 2 (k_sample_bwd_gather): one CTA owns a 16x64 canvas tile of one channel and walks the crops that cover it.
//            The bicubic adjoint is separable: per (tile, crop) the <= 5 contributing output rows / columns and their
//            weights (clamped border taps merged) are listed once, T = Wy^T gA is formed for the touched column range in
//            shared memory, then each pixel reduces Wx^T T. Every canvas pixel is written exactly once: deterministic,
//            no 457 M global atomics.
__global__ void __launch_bounds__(1024, 1)
k_sample_bwd_stage1(const float* __restrict__ grad_out, const float* __restrict__ table, int size, float* __restrict__ gA_out) {
  extern __shared__ float gA[];
  const int crop = blockIdx.x / 3, ch = blockIdx.x - crop * 3;
  CropParams p = load_params(table + (size_t)crop * APH_CROP_PARAM_FLOATS);
  prescale(p, size);
  const int n = size * size;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nwarps = blockDim.x >> 5;
  const float* go = grad_out + ((size_t)crop * 3 + ch) * n;
  for (int idx = threadIdx.x; idx < n; idx += blockDim.x) gA[idx] = 0.f;
  __syncthreads();
  const float inv_sd = 1.f / c_std[ch];
  if (p.flags & APH_FLAG_PERSP) bwd_compose<true, false>(gA, go, p, size, warp, lane, nwarps, inv_sd);
  else bwd_compose<false, false>(gA, go, p, size, warp, lane, nwarps, inv_sd);
  __syncthreads();
  float* o = gA_out + ((size_t)crop * 3 + ch) * n;
  for (int idx = threadIdx.x; idx < n; idx += blockDim.x) o[idx] = gA[idx];
}

constexpr int GT_H = 16, GT_W = 64, GT_CAP = 8, GT_TW = 80;

// lists the output indices whose (clamped) bicubic taps hit source index `rel`, with the summed weight
__device__ __forceinline__ int adjoint_taps(int rel, float scale, int cs, int size, int* idx_out, float* w_out) {
  int n = 0;
  const int lo = max(0, (int)ceilf((float)(rel - 2) / scale) - 1);
  const int hi = min(size - 1, (int)floorf((float)(rel + 2) / scale) + 1);
  for (int i = lo; i <= hi; ++i) {
    int idx[4]; float w[4];
    cubic_taps(i, scale, cs, idx, w);
    float ws = 0.f; bool hit = false;
#pragma unroll
    for (int a = 0; a < 4; ++a) if (idx[a] == rel) { ws += w[a]; hit = true; }
    if (hit && n < GT_CAP) { idx_out[n] = i; w_out[n] = ws; ++n; }
  }
  return n;
}

__global__ void __launch_bounds__(256)
k_sample_bwd_gather(const float* __restrict__ gsrc, float pre_scale_r, float pre_scale_g, float pre_scale_b, const float* __restrict__ table,
                    int S, int size, int H, int W, float* __restrict__ grad_canvas) {
  __shared__ int rowcnt[GT_H], rowi[GT_H][GT_CAP], colcnt[GT_W], colj[GT_W][GT_CAP];
  __shared__ float roww[GT_H][GT_CAP], colw[GT_W][GT_CAP], Tt[GT_H][GT_TW];
  const int tiles_x = (W + GT_W - 1) / GT_W;
  const int ch = blockIdx.y, y0 = (blockIdx.x / tiles_x) * GT_H, x0 = (blockIdx.x % tiles_x) * GT_W;
  const int t = threadIdx.x, tx = t & (GT_W - 1), tyg = t >> 6;          // thread owns column tx, rows tyg + 4 r
  const float pre = ch == 0 ? pre_scale_r : (ch == 1 ? pre_scale_g : pre_scale_b);
  const int n = size * size;
  float acc[4] = {0.f, 0.f, 0.f, 0.f};
  for (int crop = 0; crop < S; ++crop) {
    const float* row = table + (size_t)crop * APH_CROP_PARAM_FLOATS;
    const int oy = (int)row[APH_F_OFFY], ox = (int)row[APH_F_OFFX], cs = (int)row[APH_F_CSIZE];
    if (oy >= y0 + GT_H || oy + cs <= y0 || ox >= x0 + GT_W || ox + cs <= x0) continue;      // CTA-uniform
    const float scale = (size > 1) ? (float)(cs - 1) / (float)(size - 1) : 0.f;
    __syncthreads();
    if (t < GT_H) {
      const int rel = y0 + t - oy;
      rowcnt[t] = (rel >= 0 && rel < cs && y0 + t < H) ? adjoint_taps(rel, scale, cs, size, rowi[t], roww[t]) : 0;
    } else if (t >= 64 && t < 64 + GT_W) {
      const int c = t - 64, rel = x0 + c - ox;
      colcnt[c] = (rel >= 0 && rel < cs && x0 + c < W) ? adjoint_taps(rel, scale, cs, size, colj[c], colw[c]) : 0;
    }
    const int rx_lo = max(0, x0 - ox), rx_hi = min(cs - 1, x0 + GT_W - 1 - ox);
    const int jlo = max(0, (int)ceilf((float)(rx_lo - 2) / scale) - 1);
    const int jhi = min(size - 1, (int)floorf((float)(rx_hi + 2) / scale) + 1);
    const int nj = min(jhi - jlo + 1, GT_TW);
    __syncthreads();
    const float* g = gsrc + ((size_t)crop * 3 + ch) * n + jlo;
    for (int e = t; e < GT_H * nj; e += 256) {
      const int ty = e / nj, jj = e - ty * nj;
      float v = 0.f;
      const int cnt = rowcnt[ty];
      for (int a = 0; a < cnt; ++a) v += roww[ty][a] * __ldg(g + rowi[ty][a] * size + jj);
      Tt[ty][jj] = v;
    }
    __syncthreads();
    const int ccnt = colcnt[tx];
    if (ccnt > 0) {
#pragma unroll
      for (int r = 0; r < 4; ++r) {
        const int ty = tyg + 4 * r;
        if (rowcnt[ty] > 0) {
          float v = 0.f;
          for (int b = 0; b < ccnt; ++b) v += colw[tx][b] * Tt[ty][colj[tx][b] - jlo];
          acc[r] += v;
        }
      }
    }
  }
  if (x0 + tx < W) {
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      const int y = y0 + tyg + 4 * r;
      if (y < H) grad_canvas[((size_t)ch * H + y) * W + x0 + tx] = acc[r] * pre;
    }
  }
}

// ---------------------------------------------------------------------------------------------
// Backward, two-kernel form (round 2, default). The one-kernel form above (k_sample_bwd_cas) holds the gradient image of ONE
// channel in 196 KB of shared memory (one CTA per SM), re-derives the rotate / perspective geometry per channel and accumulates
// with fp32 shared atomics (compare-and-swap loops): ~420 thread instructions per pixel and channel, issue bound. Here
//   the adjoint of normalise -> rotate -> erase is a GATHER, 3 channels per thread: the rotate stage is a rigid rotation, so the
//   output pixels whose bilinear footprint covers source pixel (y, x) lie in the 3 x 3 block around R^T (y, x) (footprint
//   half-extent |cos| + |sin| <= sqrt 2 < 1.5). No atomics, no shared image;
//   k_bwd_warp_adjoint : perspective crops only (20 % of the draws): that gather, then the adjoint of the perspective resampling as
//                        12 global red.add per pixel into a library scratch image gA (kept all-zero between calls: its consumer
//                        clears what it reads). Crops whose rotate matrix is not a rotation (never drawn by the reference's sampler,
//                        accepted by the C ABI) take the complete scatter adjoint here;
//   k_bwd_bicubic3     : bicubic adjoint for all three channels of a (crop, 32-row band): the gradient row chunk comes from the scratch
//                        (perspective crops), from grad_out directly (angle 0, or no transforms) or from the rotation gather evaluated
//                        inline (the other 59 %); horizontal taps merge in per-warp strips, which drain to the four source rows as
//                        16-byte vector reductions (red.global.add.v4.f32). 19 KB of shared memory, 4 CTAs per SM.
__device__ __forceinline__ bool rigid_rot(const CropParams& p) {
  const float n0 = p.r00 * p.r00 + p.r10 * p.r10, n1 = p.r01 * p.r01 + p.r11 * p.r11, d = p.r00 * p.r01 + p.r10 * p.r11;
  return fabsf(n0 - 1.f) < 1e-3f && fabsf(n1 - 1.f) < 1e-3f && fabsf(d) < 1e-3f;
}

// gradient with respect to B(y, x) (the post-perspective, post-erase image the rotate stage samples) of sum(go * rotate(B)),
// unnormalised (no 1/std), for the three channels; go = this crop's [3, size, size] block of grad_out
__device__ __forceinline__ void rot_gather3(const float* __restrict__ go, int n, const CropParams& p, int y, int x, int size, float (&acc)[3]) {
  const float off = 0.5f * (float)size - 0.5f, fs = (float)size;
  const float sx = (float)x - off, sy = (float)y - off;
  // centre of the footprint in output coordinates: the forward samples at R b + off, b = (j, i) - off; R^-1 = R^T
  const int jr = __float2int_rn(fmaf(p.r00, sx, fmaf(p.r10, sy, off))), ir = __float2int_rn(fmaf(p.r01, sx, fmaf(p.r11, sy, off)));
  acc[0] = acc[1] = acc[2] = 0.f;
#pragma unroll
  for (int di = -1; di <= 1; ++di) {
    const int i = ir + di;
    if ((unsigned)i >= (unsigned)size) continue;
    const float by = (float)i - off;
    const float cx = fmaf(by, p.r01, off), cy = fmaf(by, p.r11, off);
#pragma unroll
    for (int dj = -1; dj <= 1; ++dj) {
      const int j = jr + dj;
      if ((unsigned)j >= (unsigned)size) continue;
      const float bx = (float)j - off;
      const float ix = fmaf(bx, p.r00, cx), iy = fmaf(bx, p.r10, cy);              // where output pixel (i, j) samples B
      const float wx = 1.f - fabsf(ix - (float)x), wy = 1.f - fabsf(iy - (float)y);
      if (wx > 0.f && wy > 0.f) {
        // coverage of (i, j): sum of its in-bounds tap weights (zeros padding of the [img; ones] stack), separable
        const float mx = __saturatef(fminf(ix + 1.f, fs - ix)), my = __saturatef(fminf(iy + 1.f, fs - iy));
        const float w = wx * wy * mx * my;
        const int o = i * size + j;
        acc[0] = fmaf(w, __ldg(go + o), acc[0]); acc[1] = fmaf(w, __ldg(go + n + o), acc[1]); acc[2] = fmaf(w, __ldg(go + 2 * n + o), acc[2]);
      }
    }
  }
}

// crops whose warp stages' adjoint goes through the scratch image (k_bwd_warp_adjoint writes, k_bwd_bicubic3 reads and clears)
__device__ __forceinline__ bool via_scratch(const CropParams& p) {
  return (p.flags & APH_FLAG_PERSP) || !(identity_rot(p) || rigid_rot(p));
}

// adds v[c] * (tap weights of b) into the three channel planes of a [3, size, size] gradient image
__device__ __forceinline__ void scatter3(float* __restrict__ g, int n, const Bilin& b, int size, const float (&v)[3]) {
  const int o = b.y0 * size + b.x0;
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    float* gc = g + c * n + o;
    if (b.w00 != 0.f) atomicAdd(gc, v[c] * b.w00);
    if (b.w01 != 0.f) atomicAdd(gc + 1, v[c] * b.w01);
    if (b.w10 != 0.f) atomicAdd(gc + size, v[c] * b.w10);
    if (b.w11 != 0.f) atomicAdd(gc + size + 1, v[c] * b.w11);
  }
}

constexpr int BB_ROWS = 32;     // gradient rows per CTA of k_bwd_bicubic3
constexpr int WA_ROWS = 8;      // rows per CTA of k_bwd_warp_adjoint (one per warp: the 20 % of crops it serves must still fill the machine)

__global__ void __launch_bounds__(256)
k_bwd_warp_adjoint(const float* __restrict__ grad_out, const float* __restrict__ table, int size, float gscale, float* __restrict__ gA_all) {
  const int crop = blockIdx.y;
  __shared__ CropParams sp;
  if (threadIdx.x == 0) { sp = load_params(table + (size_t)crop * APH_CROP_PARAM_FLOATS); prescale(sp, size); }
  __syncthreads();
  const CropParams& p = sp;
  if (!via_scratch(p)) return;
  const bool persp = (p.flags & APH_FLAG_PERSP) != 0, ident = identity_rot(p), rigid = ident || rigid_rot(p);
  const int n = size * size, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const float* go = grad_out + (size_t)crop * 3 * n;
  float* gA = gA_all + (size_t)crop * 3 * n;
  const float k0 = c_inv_std[0] * gscale, k1 = c_inv_std[1] * gscale, k2 = c_inv_std[2] * gscale;
  const int r_end = min(size, ((int)blockIdx.x + 1) * WA_ROWS);
  for (int y = blockIdx.x * WA_ROWS + warp; y < r_end; y += 8) {
    for (int x = lane; x < size; x += 32) {
      const int pix = y * size + x;
      if (rigid) {
        // (y, x) = a pixel of B: gather through the rotation, scatter through the perspective taps
        if (erased(p, y, x)) continue;
        float v[3];
        if (ident) { v[0] = __ldg(go + pix); v[1] = __ldg(go + n + pix); v[2] = __ldg(go + 2 * n + pix); }
        else rot_gather3(go, n, p, y, x, size, v);
        if (v[0] == 0.f && v[1] == 0.f && v[2] == 0.f) continue;
        const Bilin b = persp_taps(p, y, x, size);
        const float m = b.w00 + b.w01 + b.w10 + b.w11;
        v[0] *= k0 * m; v[1] *= k1 * m; v[2] *= k2 * m;
        scatter3(gA, n, b, size, v);
      } else {
        // (y, x) = an output pixel: the complete scatter adjoint rotate -> erase -> perspective
        const float g0 = __ldg(go + pix) * k0, g1 = __ldg(go + n + pix) * k1, g2 = __ldg(go + 2 * n + pix) * k2;
        const Bilin b = rot_taps(p, y, x, size);
        const float m = b.w00 + b.w01 + b.w10 + b.w11;
        const float wt[4] = {b.w00, b.w01, b.w10, b.w11};
#pragma unroll
        for (int t = 0; t < 4; ++t) {
          if (wt[t] == 0.f) continue;
          const int ty = b.y0 + (t >> 1), tx = b.x0 + (t & 1);
          if (erased(p, ty, tx)) continue;
          const float gw = wt[t] * m;
          float v[3] = {g0 * gw, g1 * gw, g2 * gw};
          if (persp) {
            const Bilin pb = persp_taps(p, ty, tx, size);
            const float pm = pb.w00 + pb.w01 + pb.w10 + pb.w11;
            v[0] *= pm; v[1] *= pm; v[2] *= pm;
            scatter3(gA, n, pb, size, v);
          } else {
            const int o = ty * size + tx;
            atomicAdd(gA + o, v[0]); atomicAdd(gA + n + o, v[1]); atomicAdd(gA + 2 * n + o, v[2]);
          }
        }
      }
    }
  }
}

__device__ __forceinline__ void red_add_v4(float* addr, float a, float b, float c, float d) {
  asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" :: "l"(addr), "f"(a), "f"(b), "f"(c), "f"(d) : "memory");
}

// VEC: canvas rows are 16-byte aligned (W % 4 == 0, aligned base, no wrap): strips are anchored at a multiple of 4 canvas columns
// FIXED: the strips accumulate round(v * 2^k) with the native integer shared atomic instead of the fp32 compare-and-swap loop; k is
// chosen per 32-pixel chunk from the warp maximum of |g| so that the 24 leading bits of the largest term survive and the sum of the
// <= 32 x 4 terms of a cell cannot overflow (cells sum <= 48 |g|max: taps have |w| <= 1.2, a clamped border pixel lands <= 1.5).
template <bool VEC, bool FIXED>
__global__ void __launch_bounds__(256, 4)
k_bwd_bicubic3(const float* __restrict__ grad_out, float* __restrict__ gA_all, int H, int W, int pad_top, int pad_left,
               const float* __restrict__ table, int size, int kind, float gscale, float* __restrict__ grad_canvas) {
  extern __shared__ __align__(16) float sm[];
  int* xo_t = reinterpret_cast<int*>(sm);        // [4*size] canvas column of every tap of every gradient column (wrap folded in)
  float* xw_t = sm + 4 * size;                   // [4*size] their weights
  __shared__ CropParams sp;
  const int crop = blockIdx.y;
  if (threadIdx.x == 0) sp = load_params(table + (size_t)crop * APH_CROP_PARAM_FLOATS);
  __syncthreads();
  const CropParams& p = sp;
  const int n = size * size;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const float scale = (size > 1) ? (float)(p.cs - 1) / (float)(size - 1) : 0.f;
  for (int k = threadIdx.x; k < size; k += blockDim.x) {
    int idx[4]; float w[4];
    cubic_taps(k, scale, p.cs, idx, w);
#pragma unroll
    for (int a = 0; a < 4; ++a) { int x = p.ox + idx[a] - pad_left; x %= W; if (x < 0) x += W; xo_t[4 * k + a] = x; xw_t[4 * k + a] = w[a]; }
  }
  float* strip = sm + 8 * size + warp * (3 * STRIP);
  for (int x = lane; x < 3 * STRIP; x += 32) strip[x] = 0.f;       // re-zeroed as they are drained
  __syncthreads();
  // where this crop's gradient rows come from (CTA-uniform)
  int mode;                                                        // 0: grad_out * pre, 1: + erase mask, 2: rotation gather inline, 3: scratch
  float pre[3];
  if (kind != APH_TF_FAST) { mode = 0; for (int c = 0; c < 3; ++c) pre[c] = (kind == APH_TF_NORMALIZE ? c_inv_std[c] : 1.f) * gscale; }
  else {
    for (int c = 0; c < 3; ++c) pre[c] = c_inv_std[c] * gscale;
    if (via_scratch(p)) { mode = 3; pre[0] = pre[1] = pre[2] = 1.f; }
    else mode = identity_rot(p) ? 1 : 2;
  }
  const float* src = grad_out + (size_t)crop * 3 * n;
  float* scr = gA_all + (size_t)crop * 3 * n;
  const bool can_strip = (pad_top == 0 && pad_left == 0);
  const size_t plane = (size_t)H * W;
  const int r_end = min(size, ((int)blockIdx.x + 1) * BB_ROWS);
  for (int i = blockIdx.x * BB_ROWS + warp; i < r_end; i += 8) {
    int yidx[4]; float wya[4]; int yoff[4];
    cubic_taps(i, scale, p.cs, yidx, wya);
#pragma unroll
    for (int a = 0; a < 4; ++a) { int y = p.oy + yidx[a] - pad_top; y %= H; if (y < 0) y += H; yoff[a] = y * W; }
    for (int j0 = 0; j0 < size; j0 += 32) {
      const int j = j0 + lane;
      float g[3] = {0.f, 0.f, 0.f};
      if (j < size) {
        const int o = i * size + j;
        if (mode == 3) {
          g[0] = scr[o]; g[1] = scr[n + o]; g[2] = scr[2 * n + o];
          if (g[0] != 0.f) scr[o] = 0.f;                           // the scratch image is all-zero again when this kernel is done
          if (g[1] != 0.f) scr[n + o] = 0.f;
          if (g[2] != 0.f) scr[2 * n + o] = 0.f;
        } else if (mode == 2) {
          if (!erased(p, i, j)) rot_gather3(src, n, p, i, j, size, g);
        } else if (!(mode == 1 && erased(p, i, j))) {
          g[0] = __ldg(src + o); g[1] = __ldg(src + n + o); g[2] = __ldg(src + 2 * n + o);
        }
        g[0] *= pre[0]; g[1] *= pre[1]; g[2] *= pre[2];
      }
      const int jc = min(j, size - 1);
      const int4 xo = *reinterpret_cast<const int4*>(xo_t + 4 * jc);
      const float4 wx = *reinterpret_cast<const float4*>(xw_t + 4 * jc);
      const int xfirst = xo_t[4 * j0], xlast = xo_t[4 * min(j0 + 31, size - 1) + 3];
      const int xbase = VEC ? (xfirst & ~3) : xfirst;
      const int span = xlast - xbase + 1;
      float fs_up = 1.f, fs_dn = 1.f;
      bool strip_ok = can_strip && span <= STRIP;
      if (FIXED && strip_ok) {
        const unsigned mbits = __reduce_max_sync(0xffffffffu, __float_as_uint(fmaxf(fmaxf(fabsf(g[0]), fabsf(g[1])), fabsf(g[2]))));
        if (mbits == 0u) continue;                                 // nothing in this chunk (warp-uniform)
        const int E = min(max((int)(mbits >> 23), 25), 254);       // |g| < 2^(E - 126)
        fs_up = __uint_as_float((unsigned)(278 - E) << 23);        // 2^(151 - E): cell sums stay below 2^31
        fs_dn = __uint_as_float((unsigned)(E - 24) << 23);         // its inverse
        if (mbits >= 0x7f800000u) strip_ok = false;                // Inf / NaN upstream: plain fp32 reductions propagate them
      }
      if (strip_ok) {
#pragma unroll
        for (int c = 0; c < 3; ++c) {
          if (g[c] != 0.f) {
            if (FIXED) {
              int* s = reinterpret_cast<int*>(strip) + c * STRIP - xbase;
              const float gs = g[c] * fs_up;
              atomicAdd(s + xo.x, __float2int_rn(gs * wx.x)); atomicAdd(s + xo.y, __float2int_rn(gs * wx.y));
              atomicAdd(s + xo.z, __float2int_rn(gs * wx.z)); atomicAdd(s + xo.w, __float2int_rn(gs * wx.w));
            } else {
              float* s = strip + c * STRIP - xbase;
              atomicAdd(s + xo.x, g[c] * wx.x); atomicAdd(s + xo.y, g[c] * wx.y); atomicAdd(s + xo.z, g[c] * wx.z); atomicAdd(s + xo.w, g[c] * wx.w);
            }
          }
        }
        __syncwarp();
        if (VEC) {
          if (4 * lane < span) {
#pragma unroll
            for (int c = 0; c < 3; ++c) {
              float4* sp4 = reinterpret_cast<float4*>(strip + c * STRIP) + lane;
              float4 h = *sp4;                                     // (all-zero bits = nothing landed here, in either representation)
              if (__float_as_uint(h.x) | __float_as_uint(h.y) | __float_as_uint(h.z) | __float_as_uint(h.w)) {
                *sp4 = make_float4(0.f, 0.f, 0.f, 0.f);
                if (FIXED) { h.x = (float)__float_as_int(h.x) * fs_dn; h.y = (float)__float_as_int(h.y) * fs_dn; h.z = (float)__float_as_int(h.z) * fs_dn; h.w = (float)__float_as_int(h.w) * fs_dn; }
                float* gc = grad_canvas + c * plane + xbase + 4 * lane;
#pragma unroll
                for (int a = 0; a < 4; ++a) red_add_v4(gc + yoff[a], wya[a] * h.x, wya[a] * h.y, wya[a] * h.z, wya[a] * h.w);
              }
            }
          }
        } else {
          for (int x = lane; x < span; x += 32) {
#pragma unroll
            for (int c = 0; c < 3; ++c) {
              float h = strip[c * STRIP + x];
              if (__float_as_uint(h) != 0u) {
                strip[c * STRIP + x] = 0.f;
                if (FIXED) h = (float)__float_as_int(h) * fs_dn;
                float* gc = grad_canvas + c * plane + xbase + x;
#pragma unroll
                for (int a = 0; a < 4; ++a) atomicAdd(gc + yoff[a], wya[a] * h);
              }
            }
          }
        }
        __syncwarp();
      } else {
#pragma unroll
        for (int c = 0; c < 3; ++c) {
          if (g[c] == 0.f) continue;
#pragma unroll
          for (int a = 0; a < 4; ++a) {
            float* r = grad_canvas + c * plane + yoff[a];
            const float gy = g[c] * wya[a];
            atomicAdd(r + xo.x, gy * wx.x); atomicAdd(r + xo.y, gy * wx.y); atomicAdd(r + xo.z, gy * wx.z); atomicAdd(r + xo.w, gy * wx.w);
          }
        }
      }
    }
  }
}

}  // namespace aph

using namespace aph;

static int check_sample_args(const char* who, int H, int W, int S, int size, int kind) {
  APH_REQUIRE(H > 0 && W > 0 && S >= 0 && size > 0, "%s: bad shape H=%d W=%d S=%d size=%d", who, H, W, S, size);
  APH_REQUIRE(((size_t)size * size + 4 + 16 * (size_t)size + 32 * STRIP) * sizeof(float) <= 227 * 1024, "%s: size=%d does not fit one CTA's shared memory (max 224)", who, size);
  APH_REQUIRE(kind >= APH_TF_NONE && kind <= APH_TF_FAST, "%s: unknown transform kind %d", who, kind);
  return 0;
}

static float* g_A = nullptr;           // resized crops [S,3,size,size] between k_resize and k_compose (library-owned scratch)
static size_t g_A_bytes = 0;

static int sample_fwd_impl(const float* canvas, int H, int W, int pad_top, int pad_left, const float* table, int S,
                           int size, int kind, float* out, PatchOut po, int* patches_written, void* stream);

extern "C" int aph_sample_fwd(const float* canvas, int H, int W, int pad_top, int pad_left, const float* table, int S,
                              int size, int kind, float* out, void* stream) {
  return sample_fwd_impl(canvas, H, W, pad_top, pad_left, table, S, size, kind, out, PatchOut{nullptr, 1, 1}, nullptr, stream);
}

extern "C" int aph_sample_fwd_patches(const float* canvas, int H, int W, int pad_top, int pad_left, const float* table, int S,
                                      int size, int kind, float* out, void* patches_bf16, int patch, int* patches_written, void* stream) {
  APH_REQUIRE(patches_bf16 && patches_written, "aph_sample_fwd_patches: null pointer");
  APH_REQUIRE(patch > 0 && size % patch == 0, "aph_sample_fwd_patches: size=%d is not a multiple of patch=%d", size, patch);
  *patches_written = 0;
  return sample_fwd_impl(canvas, H, W, pad_top, pad_left, table, S, size, kind, out,
                         PatchOut{reinterpret_cast<__nv_bfloat16*>(patches_bf16), patch, size / patch}, patches_written, stream);
}

static int sample_fwd_impl(const float* canvas, int H, int W, int pad_top, int pad_left, const float* table, int S,
                           int size, int kind, float* out, PatchOut po, int* patches_written, void* stream) {
  if (int e = check_sample_args("aph_sample_fwd", H, W, S, size, kind)) return e;
  if (S == 0) return 0;
  APH_REQUIRE(canvas && table && out, "aph_sample_fwd: null pointer");
  {
    // default: the two-kernel form (k_resize + k_compose); APH_SAMPLE_FWD_OLD=1 keeps the one-kernel form (also used when the crop
    // strips would not fit: canvases beyond ~6000 px on the short side)
    static int old_path = -1;
    if (old_path < 0) { const char* e = getenv("APH_SAMPLE_FWD_OLD"); old_path = (e && e[0] == '1') ? 1 : 0; }
    const int cap = ((H + 2 * pad_top < W + 2 * pad_left ? H + 2 * pad_top : W + 2 * pad_left) + 1 + 3) & ~3;     // crops never exceed the short side of the frame
    const size_t smem2 = ((size_t)8 * size + (size_t)8 * cap) * sizeof(float);
    if (!old_path && smem2 <= 200 * 1024) {
      cudaStream_t st = (cudaStream_t)stream;
      float* dst = out;
      if (kind == APH_TF_FAST) {
        const size_t need = (size_t)S * 3 * size * size * sizeof(float);
        if (need > g_A_bytes) {
          APH_CUDA_OK(cudaStreamSynchronize(st));
          if (g_A) cudaFree(g_A);
          g_A = nullptr; g_A_bytes = 0;
          APH_CUDA_OK(cudaMalloc(&g_A, need));
          g_A_bytes = need;
        }
        dst = g_A;
      }
      static size_t conf = 0;
      if (smem2 > conf) {
        APH_CUDA_OK(cudaFuncSetAttribute(k_resize<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem2));
        APH_CUDA_OK(cudaFuncSetAttribute(k_resize<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem2));
        conf = smem2;
      }
      const int rows_per_cta = 32;
      const dim3 g1(S * 3, (size + rows_per_cta - 1) / rows_per_cta);
      if (pad_top || pad_left) k_resize<true><<<g1, 256, smem2, st>>>(canvas, H, W, pad_top, pad_left, table, size, rows_per_cta, cap, kind, dst, po);
      else k_resize<false><<<g1, 256, smem2, st>>>(canvas, H, W, pad_top, pad_left, table, size, rows_per_cta, cap, kind, dst, po);
      APH_LAUNCH_OK();
      if (kind == APH_TF_FAST) {
        const int tiles = ((size + 15) / 16) * ((size + 15) / 16);
        k_compose<<<dim3(tiles, S), 256, 0, st>>>(g_A, table, size, out, po);
        APH_LAUNCH_OK();
      }
      if (patches_written) *patches_written = 1;
      return 0;
    }
  }
  const size_t smem = ((size_t)size * size + 4 + 16 * (size_t)size) * sizeof(float);   // no strips in the forward: the rest stays L1
  static size_t configured = 0;
  if (smem > configured) {
    APH_CUDA_OK(cudaFuncSetAttribute(k_sample_fwd, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    configured = smem;
  }
  k_sample_fwd<<<S * 3, 1024, smem, (cudaStream_t)stream>>>(canvas, H, W, pad_top, pad_left, table, size, kind, out);
  APH_LAUNCH_OK();
  return 0;
}

namespace aph {
__global__ void __launch_bounds__(256) k_scale_inplace(float* __restrict__ p, size_t n, float a) {
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) p[i] *= a;
}
}  // namespace aph

static float* g_gW = nullptr;          // warp-stage adjoint scratch [S,3,size,size] of the default backward (all-zero between calls)
static size_t g_gW_bytes = 0;
static float* g_gA = nullptr;          // stage-1 scratch [S,3,size,size] (library-owned: survives torch.cuda.empty_cache())
static size_t g_gA_bytes = 0;

static int sample_bwd_impl(const float* grad_out, int H, int W, int pad_top, int pad_left, const float* table, int S,
                           int size, int kind, float* grad_canvas, float gscale, void* stream);

extern "C" int aph_sample_bwd(const float* grad_out, int H, int W, int pad_top, int pad_left, const float* table, int S,
                              int size, int kind, float* grad_canvas, void* stream) {
  return sample_bwd_impl(grad_out, H, W, pad_top, pad_left, table, S, size, kind, grad_canvas, 1.f, stream);
}

extern "C" int aph_sample_bwd_scaled(const float* grad_out, int H, int W, int pad_top, int pad_left, const float* table, int S,
                                     int size, int kind, float gscale, float* grad_canvas, void* stream) {
  return sample_bwd_impl(grad_out, H, W, pad_top, pad_left, table, S, size, kind, grad_canvas, gscale, stream);
}

static int sample_bwd_impl(const float* grad_out, int H, int W, int pad_top, int pad_left, const float* table, int S,
                           int size, int kind, float* grad_canvas, float gscale, void* stream) {
  if (int e = check_sample_args("aph_sample_bwd", H, W, S, size, kind)) return e;
  APH_REQUIRE(grad_canvas, "aph_sample_bwd: null grad_canvas");
  // The atomic scatter is faster than this gather (per-(tile, crop) list building + 3 barriers dominate the gather),
  // so the gather is opt-in: APH_SAMPLE_BWD_GATHER=1 gives a bit-reproducible gradient.
  static int force_scatter = -1;
  if (force_scatter < 0) { const char* e = getenv("APH_SAMPLE_BWD_GATHER"); force_scatter = (e && e[0] == '1') ? 0 : 1; }
  // (crops never upsample by more than 1/0.9 when min(H, W) >= size, which bounds the adjoint tap lists of the gather kernel)
  if (S > 0 && pad_top == 0 && pad_left == 0 && !force_scatter && (H < W ? H : W) >= size) {
    // ---- atomic-free path: (stage 1) + tile gather
    APH_REQUIRE(grad_out && table, "aph_sample_bwd: null pointer");
    cudaStream_t st = (cudaStream_t)stream;
    const float* gsrc = grad_out;
    float pre[3] = {1.f, 1.f, 1.f};
    if (kind == APH_TF_FAST) {
      const size_t need = (size_t)S * 3 * size * size * sizeof(float);
      if (need > g_gA_bytes) {
        APH_CUDA_OK(cudaStreamSynchronize(st));
        if (g_gA) cudaFree(g_gA);
        g_gA = nullptr; g_gA_bytes = 0;
        APH_CUDA_OK(cudaMalloc(&g_gA, need));
        g_gA_bytes = need;
      }
      const size_t smem1 = (size_t)size * size * sizeof(float);
      static size_t configured1 = 0;
      if (smem1 > configured1) {
        APH_CUDA_OK(cudaFuncSetAttribute(k_sample_bwd_stage1, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem1));
        configured1 = smem1;
      }
      k_sample_bwd_stage1<<<S * 3, 1024, smem1, st>>>(grad_out, table, size, g_gA);
      APH_LAUNCH_OK();
      gsrc = g_gA;
    } else if (kind == APH_TF_NORMALIZE) {
      const float sd[3] = {0.26862954f, 0.26130258f, 0.27577711f};
      for (int c = 0; c < 3; ++c) pre[c] = 1.f / sd[c];
    }
    dim3 grid(((W + GT_W - 1) / GT_W) * ((H + GT_H - 1) / GT_H), 3);
    k_sample_bwd_gather<<<grid, 256, 0, st>>>(gsrc, pre[0] * gscale, pre[1] * gscale, pre[2] * gscale, table, S, size, H, W, grad_canvas);
    APH_LAUNCH_OK();
    return 0;
  }
  APH_CUDA_OK(cudaMemsetAsync(grad_canvas, 0, (size_t)3 * H * W * sizeof(float), (cudaStream_t)stream));
  if (S == 0) return 0;
  APH_REQUIRE(grad_out && table, "aph_sample_bwd: null pointer");
  // default: the two-kernel form (k_bwd_warp_adjoint + k_bwd_bicubic3); APH_SAMPLE_BWD_OLD=1 keeps the one-kernel form
  static int old_bwd = -1;
  if (old_bwd < 0) { const char* e = getenv("APH_SAMPLE_BWD_OLD"); const char* f = getenv("APH_SAMPLE_BWD_FIXED"); old_bwd = ((e && e[0] == '1') || (f && f[0] == '1')) ? 1 : 0; }
  if (!old_bwd) {
    cudaStream_t st = (cudaStream_t)stream;
    const size_t smem3 = ((size_t)8 * size + 8 * 3 * STRIP) * sizeof(float);
    static size_t configured3 = 48 * 1024;
    if (smem3 > configured3) {
      APH_CUDA_OK((cudaFuncSetAttribute(k_bwd_bicubic3<true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem3)));
      APH_CUDA_OK((cudaFuncSetAttribute(k_bwd_bicubic3<false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem3)));
      APH_CUDA_OK((cudaFuncSetAttribute(k_bwd_bicubic3<true, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem3)));
      APH_CUDA_OK((cudaFuncSetAttribute(k_bwd_bicubic3<false, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem3)));
      configured3 = smem3;
    }
    const bool vec = pad_top == 0 && pad_left == 0 && W % 4 == 0 && ((uintptr_t)grad_canvas & 15) == 0;
    const dim3 g3((size + BB_ROWS - 1) / BB_ROWS, S);
    // strips in integer fixed point (native shared atomic add) by default; APH_SAMPLE_STRIP_FP32=1: fp32 strips (compare-and-swap loops)
    static int fp32_strips = -1;
    if (fp32_strips < 0) { const char* e = getenv("APH_SAMPLE_STRIP_FP32"); fp32_strips = (e && e[0] == '1') ? 1 : 0; }
#define APH_BB(V, F, STREAM) k_bwd_bicubic3<V, F><<<g3, 256, smem3, STREAM>>>(grad_out, g_gW, H, W, pad_top, pad_left, table, size, kind, gscale, grad_canvas)
#define APH_BB_ANY(STREAM)                                                                           \
    do {                                                                                             \
      if (vec) { if (fp32_strips) APH_BB(true, false, STREAM); else APH_BB(true, true, STREAM); }    \
      else { if (fp32_strips) APH_BB(false, false, STREAM); else APH_BB(false, true, STREAM); }      \
      APH_LAUNCH_OK();                                                                               \
    } while (0)
    if (kind != APH_TF_FAST) { APH_BB_ANY(st); return 0; }
    const size_t need = (size_t)S * 3 * size * size * sizeof(float);
    if (need > g_gW_bytes) {
      APH_CUDA_OK(cudaStreamSynchronize(st));
      if (g_gW) cudaFree(g_gW);
      g_gW = nullptr; g_gW_bytes = 0;
      APH_CUDA_OK(cudaMalloc(&g_gW, need));
      g_gW_bytes = need;
      APH_CUDA_OK(cudaMemsetAsync(g_gW, 0, need, st));          // invariant: all-zero between calls (k_bwd_bicubic3 clears what it consumes)
    }
    const dim3 g1((size + WA_ROWS - 1) / WA_ROWS, S);
    // (running this chain on a side stream beside the other crops' bicubic adjoint was measured: no gain, 0.335 vs 0.333 ms -- removed)
    k_bwd_warp_adjoint<<<g1, 256, 0, st>>>(grad_out, table, size, gscale, g_gW);
    APH_LAUNCH_OK();
    APH_BB_ANY(st);
#undef APH_BB_ANY
#undef APH_BB
    APH_LAUNCH_OK();
    return 0;
  }
  const size_t smem = ((size_t)size * size + 4 + 16 * (size_t)size + 32 * STRIP) * sizeof(float);
  static size_t configured = 0;
  if (smem > configured) {
    APH_CUDA_OK(cudaFuncSetAttribute(k_sample_bwd, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    APH_CUDA_OK(cudaFuncSetAttribute(k_sample_bwd_cas, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    configured = smem;
  }
  // APH_SAMPLE_BWD_FIXED=1: integer fixed-point shared accumulation (order-independent shared stage). Measured equal to the
  // fp32 compare-and-swap kernel (0.581 vs 0.578 ms at C2, profiles/README.md), so the plain fp32 kernel stays the default.
  static int fixed = -1;
  if (fixed < 0) { const char* e = getenv("APH_SAMPLE_BWD_FIXED"); fixed = (e && e[0] == '1') ? 1 : 0; }
  if (fixed) {
    k_sample_bwd<<<S * 3, 1024, smem, (cudaStream_t)stream>>>(grad_out, H, W, pad_top, pad_left, table, size, kind, grad_canvas);
    APH_LAUNCH_OK();
    if (gscale != 1.f) { k_scale_inplace<<<num_sms() * 4, 256, 0, (cudaStream_t)stream>>>(grad_canvas, (size_t)3 * H * W, gscale); APH_LAUNCH_OK(); }
    return 0;
  }
  k_sample_bwd_cas<<<S * 3, 1024, smem, (cudaStream_t)stream>>>(grad_out, H, W, pad_top, pad_left, table, size, kind, grad_canvas, gscale);
  APH_LAUNCH_OK();
  return 0;
}
