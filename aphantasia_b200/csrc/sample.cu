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
// Kernels:
//   forward : k_resize (stage 1, separable, into a library scratch image; the direct 16-tap form for frames whose short side is too
//             long for its per-warp crop rows) + k_compose / k_compose_kornia (stages 2-5, three channels per thread; optionally also
//             the encoder's bf16 patch operand, aph_sample_fwd_patches);
//   backward: k_bwd_warp_adjoint (perspective crops: rotation adjoint as a gather, perspective adjoint by global reductions into a
//             scratch image) + k_bwd_bicubic3 (every crop: rotation adjoint gathered inline, bicubic adjoint through per-warp strips
//             and 16-byte vector reductions into the canvas gradient).
#include "aph_common.cuh"
#include <stdint.h>
#include <type_traits>

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
template <typename T> __device__ __forceinline__ Bilin pix_taps(T ix, T iy, int size);
__device__ __forceinline__ Bilin bilin_taps(float gx, float gy, int size) {
  const float ix = ((gx + 1.f) * (float)size - 1.f) * 0.5f;
  const float iy = ((gy + 1.f) * (float)size - 1.f) * 0.5f;
  return pix_taps<float>(ix, iy, size);
}

// bilinear taps at pixel-index coordinates (ix, iy); taps outside [0, size) get weight 0 (zeros padding, no renormalisation).
// T = double: the kornia stages' positions, whose fractions a float near 200 would quantise to 1.5e-5 pixel
template <typename T>
__device__ __forceinline__ Bilin pix_taps(T ix, T iy, int size) {
  const T fx = floor(ix), fy = floor(iy);
  Bilin b;
  b.x0 = (int)fx; b.y0 = (int)fy;
  const float tx = (float)(ix - fx), ty = (float)(iy - fy);
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

__constant__ float c_inv_std[3] = {1.f / 0.26862954f, 1.f / 0.26130258f, 1.f / 0.27577711f};
__constant__ float c_shift[3] = {-0.48145466f / 0.26862954f, -0.4578275f / 0.26130258f, -0.40821073f / 0.27577711f};

// the rotate stage is the identity resampling (angle 0: theta = [[1, 0], [0, 1]])
__device__ __forceinline__ bool identity_rot(const CropParams& p) { return p.r00 == 1.f && p.r01 == 0.f && p.r10 == 0.f && p.r11 == 1.f; }

__constant__ float c_mean[3] = {0.48145466f, 0.4578275f, 0.40821073f};
__constant__ float c_std[3] = {0.26862954f, 0.26130258f, 0.27577711f};

// ---------------------------------------------------------------------------------------------
// Forward in two kernels.
//   k_resize : stage 1 alone, SEPARABLE -- a warp owns an output row: vertical 4-tap pass over the crop's columns (coalesced row
//              reads) into a per-warp strip, then the horizontal 4-tap pass out of the strip; 8 rows of state per CTA, 7 CTAs / SM.
//              A frame whose short side is too long for that strip (above about 6400 - size px: ~6170 at size 224, ~5950 at 448)
//              takes the DIRECT form, launched with cap = 0 (no strip memory, 32 size bytes of tap tables): every output pixel reads its 16 taps straight from the canvas, four
//              horizontal taps per source row, then the vertical combination. It is a template parameter rather than a run-time
//              flag because the flag would cost the strip forms' output loop its unrolling.
//              Result A [S,3,size,size] goes to a library scratch buffer (L2 / HBM), or straight to the output for transform kinds
//              without a warp stage.
//   k_compose: stages 2-5 for ALL THREE channels of a pixel per thread: one evaluation of the rotate (and perspective) taps,
//              4 (16) gathers per channel from the scratch image through L1.
// The encoder's patch-embedding GEMM reads its A operand patch-major in bf16: [S*g*g, patch_k(p)], row = s*g*g + gy*g + gx,
// col = c*p*p + py*p + px (conv1 weight layout, vit_ops.cuh k_patchify; the columns >= 3 p^2 are zero padding, never written).
// With `patches` set the sampler's last stage writes that operand beside the fp32 batch (SURVEY 2.4 k10-k12), so the encoder
// does not re-read 4 bytes per pixel to produce it.
struct PatchOut { __nv_bfloat16* base; int p, g; };
__device__ __forceinline__ size_t patch_index(const PatchOut& po, int s, int c, int i, int j) {
  const int gy = i / po.p, py = i - gy * po.p, gx = j / po.p, px = j - gx * po.p;
  return ((size_t)(s * po.g + gy) * po.g + gx) * (size_t)patch_k(po.p) + (size_t)(c * po.p + py) * po.p + px;
}

// DIRECT is launched with WRAP = true: the wrap is a no-op on an unpadded frame
template <bool WRAP, bool DIRECT>
__global__ void __launch_bounds__(256)
k_resize(const float* __restrict__ canvas, int H, int W, int pad_top, int pad_left, const float* __restrict__ table, int size, int rows_per_cta,
         int cap, int kind, float* __restrict__ dst, PatchOut po) {
  extern __shared__ float rs[];
  int* xi = reinterpret_cast<int*>(rs);              // [4*size] source columns of every output column: crop-relative, or (direct) canvas
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
    for (int a = 0; a < 4; ++a) {
      int x = idx[a];
      if (DIRECT) { x = (p.ox + x - pad_left) % W; if (x < 0) x += W; }
      xi[4 * k + a] = x; xw[4 * k + a] = w[a];
    }
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
    if (DIRECT) {
      // no strip: the loop below reads all 16 taps from the canvas
    } else if (WRAP) {
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
      float acc;
      if (DIRECT) {
        const float v0 = wx.x * __ldg(rp[0] + xo.x) + wx.y * __ldg(rp[0] + xo.y) + wx.z * __ldg(rp[0] + xo.z) + wx.w * __ldg(rp[0] + xo.w);
        const float v1 = wx.x * __ldg(rp[1] + xo.x) + wx.y * __ldg(rp[1] + xo.y) + wx.z * __ldg(rp[1] + xo.z) + wx.w * __ldg(rp[1] + xo.w);
        const float v2 = wx.x * __ldg(rp[2] + xo.x) + wx.y * __ldg(rp[2] + xo.y) + wx.z * __ldg(rp[2] + xo.z) + wx.w * __ldg(rp[2] + xo.w);
        const float v3 = wx.x * __ldg(rp[3] + xo.x) + wx.y * __ldg(rp[3] + xo.y) + wx.z * __ldg(rp[3] + xo.z) + wx.w * __ldg(rp[3] + xo.w);
        acc = wy[0] * v0;
        acc += wy[1] * v1; acc += wy[2] * v2; acc += wy[3] * v3;
      } else {
        acc = wx.x * strip[xo.x];
        acc += wx.y * strip[xo.y]; acc += wx.z * strip[xo.z]; acc += wx.w * strip[xo.w];
      }
      const float v = (kind >= APH_TF_FAST) ? acc : fmaf(acc, na, nb);
      o[i * size + j] = v;
      if (kind < APH_TF_FAST && po.base) po.base[patch_index(po, crop, ch, i, j)] = __float2bfloat16_rn(v);
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

// ---------------------------------------------------------------------------------------------
// transforms_custom / transforms_elastic (reference transforms.py:147-163, kornia stages restated; DESIGN §1). On the resized crop
// A [3,size,size] and s = size + 8, c = (s - 1) / 2, every stage a resampling of an s x s image:
//   P = pad(4, 0.5) of A, then (elastic) the erase rectangle -> 0        (F.pad; torchvision RandomErasing on the padded image)
//   R(x, y) = bilinear(P, c + Rot (x - c, y - c)), zeros outside          (kornia warp_affine, align_corners=True: pixel space)
//   E(x, y) = bilinear(R, x k - 1/2, y k - 1/2), k = s / (s - 1)          (elastic_transform2d with zero noise: grid_sample,
//                                                                          align_corners=False, of the align_corners=True mesh)
//   J(x, y) = E(x - dx, y - dy), zeros outside                           (kornia translate by an integer shift)
//   out = (J - mean) / std
// k_compose_kornia evaluates the chain by exact tap composition for the three channels of one output pixel, as k_compose does for
// transforms_fast; nothing between A and the output is materialised.
constexpr int KPAD = 4;

// pixel of the padded (and erased) image P
__device__ __forceinline__ void padded3(const float* __restrict__ A, int n, const CropParams& p, int y, int x, int size, float w, float (&acc)[3]) {
  if (erased(p, y, x)) return;
  const int u = y - KPAD, v = x - KPAD;
  if ((unsigned)u >= (unsigned)size || (unsigned)v >= (unsigned)size) { acc[0] += 0.5f * w; acc[1] += 0.5f * w; acc[2] += 0.5f * w; return; }
  const int o = u * size + v;
#pragma unroll
  for (int c = 0; c < 3; ++c) acc[c] += w * __ldg(A + c * n + o);
}

// where pixel (yr, xr) of R samples P: the same expression rot_gather3 inverts in the backward
__device__ __forceinline__ Bilin kornia_rot_taps(const CropParams& p, int yr, int xr, int s) {
  const double off = 0.5 * s - 0.5;
  const double bx = xr - off, by = yr - off;
  return pix_taps<double>(fma(bx, (double)p.r00, fma(by, (double)p.r01, off)), fma(bx, (double)p.r10, fma(by, (double)p.r11, off)), s);
}

__device__ __forceinline__ void rotated3(const float* __restrict__ A, int n, const CropParams& p, int yr, int xr, int size, float w, float (&acc)[3]) {
  const int s = size + 2 * KPAD;
  const Bilin b = kornia_rot_taps(p, yr, xr, s);
  if (b.w00 != 0.f) padded3(A, n, p, b.y0, b.x0, size, w * b.w00, acc);
  if (b.w01 != 0.f) padded3(A, n, p, b.y0, b.x0 + 1, size, w * b.w01, acc);
  if (b.w10 != 0.f) padded3(A, n, p, b.y0 + 1, b.x0, size, w * b.w10, acc);
  if (b.w11 != 0.f) padded3(A, n, p, b.y0 + 1, b.x0 + 1, size, w * b.w11, acc);
}

// the elastic stretch along one axis: output index j samples x0 (weight w0) and x0 + 1 (weight w1); out-of-range taps weigh 0
__device__ __forceinline__ void stretch_taps(int j, int s, int& x0, float& w0, float& w1) {
  const double src = (double)j * s / (s - 1) - 0.5;
  const double f = floor(src);
  const float t = (float)(src - f);
  x0 = (int)f;
  w0 = ((unsigned)x0 < (unsigned)s) ? 1.f - t : 0.f;
  w1 = ((unsigned)(x0 + 1) < (unsigned)s) ? t : 0.f;
}

template <bool ELASTIC>
__global__ void __launch_bounds__(256)
k_compose_kornia(const float* __restrict__ Ag, const float* __restrict__ table, int size, float* __restrict__ out, PatchOut po) {
  const int s = size + 2 * KPAD;
  const int crop = blockIdx.y, tiles_x = (s + 15) >> 4;
  const int ti = blockIdx.x / tiles_x, tj = blockIdx.x - ti * tiles_x;
  const int i = ti * 16 + (threadIdx.x >> 4), j = tj * 16 + (threadIdx.x & 15);
  __shared__ CropParams sp;
  __shared__ int sd[2];
  if (threadIdx.x == 0) {
    const float* row = table + (size_t)crop * APH_CROP_PARAM_FLOATS;
    sp = load_params(row); sd[0] = (int)row[APH_F_JIT_DX]; sd[1] = (int)row[APH_F_JIT_DY];
  }
  __syncthreads();
  const CropParams p = sp;
  if (i >= s || j >= s) return;
  const int n = size * size;
  const float* A = Ag + (size_t)crop * 3 * n;
  float acc[3] = {0.f, 0.f, 0.f};
  const int ye = i - sd[1], xe = j - sd[0];                 // jitter: J(i, j) = E(i - dy, j - dx)
  if ((unsigned)ye < (unsigned)s && (unsigned)xe < (unsigned)s) {
    if (ELASTIC) {
      int y0, x0; float wy0, wy1, wx0, wx1;
      stretch_taps(ye, s, y0, wy0, wy1);
      stretch_taps(xe, s, x0, wx0, wx1);
      if (wy0 * wx0 != 0.f) rotated3(A, n, p, y0, x0, size, wy0 * wx0, acc);
      if (wy0 * wx1 != 0.f) rotated3(A, n, p, y0, x0 + 1, size, wy0 * wx1, acc);
      if (wy1 * wx0 != 0.f) rotated3(A, n, p, y0 + 1, x0, size, wy1 * wx0, acc);
      if (wy1 * wx1 != 0.f) rotated3(A, n, p, y0 + 1, x0 + 1, size, wy1 * wx1, acc);
    } else {
      rotated3(A, n, p, ye, xe, size, 1.f, acc);
    }
  }
  const int sn = s * s, pix = i * s + j;
  float* o = out + (size_t)crop * 3 * sn;
  // the encoder's patch operand holds the top-left (g p)^2 window: conv1 (kernel = stride = p) never reads the rest
  const bool in_window = po.base && i < po.p * po.g && j < po.p * po.g;
  const size_t pi = in_window ? patch_index(po, crop, 0, i, j) : 0;
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const float v = fmaf(acc[c], c_inv_std[c], c_shift[c]);
    o[c * sn + pix] = v;
    if (in_window) po.base[pi + (size_t)c * po.p * po.p] = __float2bfloat16_rn(v);
  }
}

// ---------------------------------------------------------------------------------------------
// Backward in two kernels.
//   The adjoint of normalise -> rotate -> erase is a GATHER, 3 channels per thread: the rotate stage is a rigid rotation, so the
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
// unnormalised (no 1/std), for the three channels; go = this crop's [3, size, size] block of grad_out.
// COVER: torchvision's rotate multiplies by the coverage of the [img; ones] stack; kornia's warp_affine (COVER = false) does not.
template <bool COVER = true>
__device__ __forceinline__ void rot_gather3(const float* __restrict__ go, int n, const CropParams& p, int y, int x, int size, float (&acc)[3]) {
  using P = typename std::conditional<COVER, float, double>::type;      // kornia's positions in double (see pix_taps)
  const P off = (P)0.5 * (P)size - (P)0.5;
  const float fs = (float)size;
  const P sx = (P)x - off, sy = (P)y - off;
  const P r00 = p.r00, r01 = p.r01, r10 = p.r10, r11 = p.r11;
  // centre of the footprint in output coordinates: the forward samples at R b + off, b = (j, i) - off; R^-1 = R^T
  const int jr = (int)rint(fma(r00, sx, fma(r10, sy, off))), ir = (int)rint(fma(r01, sx, fma(r11, sy, off)));
  acc[0] = acc[1] = acc[2] = 0.f;
#pragma unroll
  for (int di = -1; di <= 1; ++di) {
    const int i = ir + di;
    if ((unsigned)i >= (unsigned)size) continue;
    const P by = (P)i - off;
    const P cx = fma(by, r01, off), cy = fma(by, r11, off);
#pragma unroll
    for (int dj = -1; dj <= 1; ++dj) {
      const int j = jr + dj;
      if ((unsigned)j >= (unsigned)size) continue;
      const P bx = (P)j - off;
      const P ix = fma(bx, r00, cx), iy = fma(bx, r10, cy);                        // where output pixel (i, j) samples B
      const float wx = (float)(1 - fabs(ix - (P)x)), wy = (float)(1 - fabs(iy - (P)y));
      if (wx > 0.f && wy > 0.f) {
        // coverage of (i, j): sum of its in-bounds tap weights (zeros padding of the [img; ones] stack), separable
        float w = wx * wy;
        if (COVER) { w *= __saturatef(fminf((float)ix + 1.f, fs - (float)ix)); w *= __saturatef(fminf((float)iy + 1.f, fs - (float)iy)); }
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

constexpr int STRIP = 128;      // per-warp strip (floats per channel) of k_bwd_bicubic3
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

// transforms_custom / _elastic, backward first stage: the adjoints of normalise, jitter and (elastic) the stretch, as a gather into
// gR [S,3,s,s] = d loss / d R (the rotated image). The rest -- rotation adjoint, erase mask, pad border, bicubic adjoint -- runs in
// k_bwd_bicubic3 (mode 4). Every element of gR is written: the scratch carries nothing from one call to the next.
// Output index j of the stretch taps x0(j) and x0(j) + 1 with x0(j) in {j - 1, j}: R index r is reached from j in {r - 1, r, r + 1}.
__device__ __forceinline__ int stretch_adjoint(int r, int s, int (&js)[3], float (&ws)[3]) {
  int m = 0;
#pragma unroll
  for (int d = -1; d <= 1; ++d) {
    const int j = r + d;
    if ((unsigned)j >= (unsigned)s) continue;
    int x0; float w0, w1;
    stretch_taps(j, s, x0, w0, w1);
    const float w = (x0 == r ? w0 : 0.f) + (x0 + 1 == r ? w1 : 0.f);
    if (w != 0.f) { js[m] = j; ws[m] = w; ++m; }
  }
  return m;
}

template <bool ELASTIC>
__global__ void __launch_bounds__(256)
k_bwd_kornia_stage(const float* __restrict__ grad_out, const float* __restrict__ table, int size, float gscale, float* __restrict__ gR_all) {
  const int s = size + 2 * KPAD, sn = s * s, crop = blockIdx.y;
  const float* row = table + (size_t)crop * APH_CROP_PARAM_FLOATS;
  const int dx = (int)row[APH_F_JIT_DX], dy = (int)row[APH_F_JIT_DY];
  const float* go = grad_out + (size_t)crop * 3 * sn;
  float* gR = gR_all + (size_t)crop * 3 * sn;
  const float k0 = c_inv_std[0] * gscale, k1 = c_inv_std[1] * gscale, k2 = c_inv_std[2] * gscale;
  for (int pix = blockIdx.x * blockDim.x + threadIdx.x; pix < sn; pix += gridDim.x * blockDim.x) {
    const int yr = pix / s, xr = pix - yr * s;
    float a0 = 0.f, a1 = 0.f, a2 = 0.f;
    int jy[3], jx[3]; float wy[3], wx[3];
    int my = 1, mx = 1;
    if (ELASTIC) { my = stretch_adjoint(yr, s, jy, wy); mx = stretch_adjoint(xr, s, jx, wx); }
    else { jy[0] = yr; jx[0] = xr; wy[0] = wx[0] = 1.f; }
    for (int a = 0; a < my; ++a) {
      const int y = jy[a] + dy;                             // output row the jitter moved E's row jy to
      if ((unsigned)y >= (unsigned)s) continue;
      for (int b = 0; b < mx; ++b) {
        const int x = jx[b] + dx;
        if ((unsigned)x >= (unsigned)s) continue;
        const float w = wy[a] * wx[b];
        const int o = y * s + x;
        a0 = fmaf(w, __ldg(go + o), a0); a1 = fmaf(w, __ldg(go + sn + o), a1); a2 = fmaf(w, __ldg(go + 2 * sn + o), a2);
      }
    }
    gR[pix] = a0 * k0; gR[sn + pix] = a1 * k1; gR[2 * sn + pix] = a2 * k2;
  }
}

__device__ __forceinline__ void red_add_v4(float* addr, float a, float b, float c, float d) {
  asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" :: "l"(addr), "f"(a), "f"(b), "f"(c), "f"(d) : "memory");
}

// VEC: canvas rows are 16-byte aligned (W % 4 == 0, aligned base, no wrap): strips are anchored at a multiple of 4 canvas columns
// The strips accumulate in integer fixed point, round(v * 2^k), with the native integer shared atomic add: fp32 atomicAdd on shared
// memory is a compare-and-swap loop on this architecture (SASS: ATOMS.CAST.SPIN, ~6 instructions and two dependent shared round trips
// per add). k is chosen per 32-pixel chunk from the warp maximum of |g| so that the 24 leading bits of the largest term survive and the
// sum of the <= 32 x 4 terms of a cell cannot overflow (cells sum <= 48 |g|max: taps have |w| <= 1.2, a clamped border pixel lands
// <= 1.5). The scale follows the chunk's largest term, not an absolute bound, so small gradients keep their relative precision.
template <bool VEC>
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
  // 0: grad_out * pre, 1: + erase mask, 2: rotation gather inline, 3: scratch, 4: kornia rotation gather from gR (grad_out is
  // k_bwd_kornia_stage's [S,3,size+8,size+8] output) at the padded pixel, erase mask
  int mode;
  float pre[3];
  if (kind >= APH_TF_CUSTOM) { mode = 4; pre[0] = pre[1] = pre[2] = 1.f; }
  else if (kind != APH_TF_FAST) { mode = 0; for (int c = 0; c < 3; ++c) pre[c] = (kind == APH_TF_NORMALIZE ? c_inv_std[c] : 1.f) * gscale; }
  else {
    for (int c = 0; c < 3; ++c) pre[c] = c_inv_std[c] * gscale;
    if (via_scratch(p)) { mode = 3; pre[0] = pre[1] = pre[2] = 1.f; }
    else mode = identity_rot(p) ? 1 : 2;
  }
  const int ks = size + 2 * KPAD;
  const float* src = grad_out + (size_t)crop * 3 * (mode == 4 ? ks * ks : n);
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
        } else if (mode == 4) {
          if (!erased(p, i + KPAD, j + KPAD)) rot_gather3<false>(src, ks * ks, p, i + KPAD, j + KPAD, ks, g);
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
      if (strip_ok) {
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
            int* s = reinterpret_cast<int*>(strip) + c * STRIP - xbase;
            const float gs = g[c] * fs_up;
            atomicAdd(s + xo.x, __float2int_rn(gs * wx.x)); atomicAdd(s + xo.y, __float2int_rn(gs * wx.y));
            atomicAdd(s + xo.z, __float2int_rn(gs * wx.z)); atomicAdd(s + xo.w, __float2int_rn(gs * wx.w));
          }
        }
        __syncwarp();
        if (VEC) {
          if (4 * lane < span) {
#pragma unroll
            for (int c = 0; c < 3; ++c) {
              float4* sp4 = reinterpret_cast<float4*>(strip + c * STRIP) + lane;
              float4 h = *sp4;                                     // (all-zero bits = nothing landed here)
              if (__float_as_uint(h.x) | __float_as_uint(h.y) | __float_as_uint(h.z) | __float_as_uint(h.w)) {
                *sp4 = make_float4(0.f, 0.f, 0.f, 0.f);
                h.x = (float)__float_as_int(h.x) * fs_dn; h.y = (float)__float_as_int(h.y) * fs_dn; h.z = (float)__float_as_int(h.z) * fs_dn; h.w = (float)__float_as_int(h.w) * fs_dn;
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
                h = (float)__float_as_int(h) * fs_dn;
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

// Largest output side of the sampler: the largest crop side the image encoders take (RN50x64's 448; the kornia kinds write
// size + 8), and the largest the tests cover. Every launch below is sized from `size` at run time: k_resize's tap tables take
// 8 size floats of shared memory (14 KB at 448) and k_bwd_bicubic3's 8 size + 24 STRIP (17 KB); the grids grow with size.
constexpr int kMaxSampleSize = 448;

static int check_sample_args(const char* who, int H, int W, int S, int size, int kind) {
  APH_REQUIRE(H > 0 && W > 0 && S >= 0 && size > 0, "%s: bad shape H=%d W=%d S=%d size=%d", who, H, W, S, size);
  APH_REQUIRE(size <= kMaxSampleSize, "%s: size=%d is above %d, the largest crop side the image encoders take", who, size, kMaxSampleSize);
  APH_REQUIRE(kind >= APH_TF_NONE && kind <= APH_TF_ELASTIC, "%s: unknown transform kind %d", who, kind);
  return 0;
}

static Scratch& g_A = *new Scratch;    // resized crops [S,3,size,size] between k_resize and k_compose

static int sample_fwd_impl(const float* canvas, int H, int W, int pad_top, int pad_left, const float* table, int S,
                           int size, int kind, float* out, PatchOut po, void* stream);

extern "C" int aph_sample_fwd(const float* canvas, int H, int W, int pad_top, int pad_left, const float* table, int S,
                              int size, int kind, float* out, void* stream) {
  return sample_fwd_impl(canvas, H, W, pad_top, pad_left, table, S, size, kind, out, PatchOut{nullptr, 1, 1}, stream);
}

extern "C" int aph_sample_fwd_patches(const float* canvas, int H, int W, int pad_top, int pad_left, const float* table, int S,
                                      int size, int kind, float* out, void* patches_bf16, int patch, int* patches_written, void* stream) {
  APH_REQUIRE(patches_bf16 && patches_written, "aph_sample_fwd_patches: null pointer");
  APH_REQUIRE(patch > 0, "aph_sample_fwd_patches: patch=%d", patch);
  // the kornia kinds write size + 8: the operand is the top-left (grid * patch)^2 window conv1 reads
  const int side = size + (kind >= APH_TF_CUSTOM ? 2 * KPAD : 0);
  APH_REQUIRE(kind >= APH_TF_CUSTOM ? side >= patch : size % patch == 0, "aph_sample_fwd_patches: size=%d does not fit patch=%d", size, patch);
  if (int e = sample_fwd_impl(canvas, H, W, pad_top, pad_left, table, S, size, kind, out,
                              PatchOut{reinterpret_cast<__nv_bfloat16*>(patches_bf16), patch, side / patch}, stream)) return e;
  *patches_written = 1;
  return 0;
}

static int sample_fwd_impl(const float* canvas, int H, int W, int pad_top, int pad_left, const float* table, int S,
                           int size, int kind, float* out, PatchOut po, void* stream) {
  if (int e = check_sample_args("aph_sample_fwd", H, W, S, size, kind)) return e;
  if (S == 0) return 0;
  APH_REQUIRE(canvas && table && out, "aph_sample_fwd: null pointer");
  cudaStream_t st = (cudaStream_t)stream;
  int cap = ((H + 2 * pad_top < W + 2 * pad_left ? H + 2 * pad_top : W + 2 * pad_left) + 1 + 3) & ~3;     // crops never exceed the short side of the frame
  // k_resize holds one crop row per warp in shared memory, sized by the frame's short side; above about 6400 - size px (~6170 at
  // size 224, ~5950 at 448) that does not fit, and k_resize runs its direct form (cap = 0: the x tap tables alone)
  if (((size_t)8 * size + (size_t)8 * cap) * sizeof(float) > 200 * 1024) cap = 0;
  const size_t smem2 = ((size_t)8 * size + (size_t)8 * cap) * sizeof(float);
  float* dst = out;
  if (kind >= APH_TF_FAST) {
    if (int e = g_A.grow((size_t)S * 3 * size * size * sizeof(float), st)) return e;
    dst = g_A.p;
  }
  auto resize = k_resize<false, false>;
  if (pad_top || pad_left) resize = k_resize<true, false>;
  if (cap == 0) resize = k_resize<true, true>;
  if (int e = smem_at_least((const void*)resize, smem2)) return e;
  const int rows_per_cta = 32;
  const dim3 g1(S * 3, (size + rows_per_cta - 1) / rows_per_cta);
  resize<<<g1, 256, smem2, st>>>(canvas, H, W, pad_top, pad_left, table, size, rows_per_cta, cap, kind, dst, po);
  APH_LAUNCH_OK();
  if (kind == APH_TF_FAST) {
    const int tiles = ((size + 15) / 16) * ((size + 15) / 16);
    k_compose<<<dim3(tiles, S), 256, 0, st>>>(g_A.p, table, size, out, po);
    APH_LAUNCH_OK();
  } else if (kind >= APH_TF_CUSTOM) {
    const int s = size + 2 * KPAD, tiles = ((s + 15) / 16) * ((s + 15) / 16);
    if (kind == APH_TF_ELASTIC) k_compose_kornia<true><<<dim3(tiles, S), 256, 0, st>>>(g_A.p, table, size, out, po);
    else k_compose_kornia<false><<<dim3(tiles, S), 256, 0, st>>>(g_A.p, table, size, out, po);
    APH_LAUNCH_OK();
  }
  return 0;
}

static Scratch& g_gW = *new Scratch;   // warp-stage adjoint scratch [S,3,size,size] of the default backward (all-zero between calls)
static Scratch& g_gR = *new Scratch;   // kornia kinds: d loss / d rotated image [S,3,size+8,size+8], rewritten by every backward

extern "C" int aph_sample_bwd_scaled(const float* grad_out, int H, int W, int pad_top, int pad_left, const float* table, int S,
                                     int size, int kind, float gscale, float* grad_canvas, void* stream) {
  if (int e = check_sample_args("aph_sample_bwd_scaled", H, W, S, size, kind)) return e;
  APH_REQUIRE(grad_canvas, "aph_sample_bwd_scaled: null grad_canvas");
  cudaStream_t st = (cudaStream_t)stream;
  APH_CUDA_OK(cudaMemsetAsync(grad_canvas, 0, (size_t)3 * H * W * sizeof(float), st));
  if (S == 0) return 0;
  APH_REQUIRE(grad_out && table, "aph_sample_bwd_scaled: null pointer");
  const size_t smem3 = ((size_t)8 * size + 8 * 3 * STRIP) * sizeof(float);
  const bool vec = pad_top == 0 && pad_left == 0 && W % 4 == 0 && ((uintptr_t)grad_canvas & 15) == 0;
  const auto bicubic = vec ? k_bwd_bicubic3<true> : k_bwd_bicubic3<false>;
  if (int e = smem_at_least((const void*)bicubic, smem3)) return e;
  const float* bb_src = grad_out;
  if (kind >= APH_TF_CUSTOM) {
    // adjoints of normalise, jitter and the elastic stretch into gR (fully overwritten), then the rest in k_bwd_bicubic3 (mode 4)
    const int s = size + 2 * KPAD;
    if (int e = g_gR.grow((size_t)S * 3 * s * s * sizeof(float), st)) return e;
    const dim3 gk((s * s + 1023) / 1024, S);
    if (kind == APH_TF_ELASTIC) k_bwd_kornia_stage<true><<<gk, 256, 0, st>>>(grad_out, table, size, gscale, g_gR.p);
    else k_bwd_kornia_stage<false><<<gk, 256, 0, st>>>(grad_out, table, size, gscale, g_gR.p);
    APH_LAUNCH_OK();
    bb_src = g_gR.p;
  } else if (kind == APH_TF_FAST) {
    const size_t need = (size_t)S * 3 * size * size * sizeof(float);
    if (need > g_gW.bytes) {
      if (int e = g_gW.grow(need, st)) return e;
      APH_CUDA_OK(cudaMemsetAsync(g_gW.p, 0, need, st));        // invariant: all-zero between calls (k_bwd_bicubic3 clears what it consumes)
    }
    const dim3 g1((size + WA_ROWS - 1) / WA_ROWS, S);
    // (running this chain on a side stream beside the other crops' bicubic adjoint was measured: no gain, 0.335 vs 0.333 ms -- removed)
    k_bwd_warp_adjoint<<<g1, 256, 0, st>>>(grad_out, table, size, gscale, g_gW.p);
    APH_LAUNCH_OK();
  }
  const dim3 g3((size + BB_ROWS - 1) / BB_ROWS, S);
  bicubic<<<g3, 256, smem3, st>>>(bb_src, g_gW.p, H, W, pad_top, pad_left, table, size, kind, gscale, grad_canvas);
  APH_LAUNCH_OK();
  return 0;
}
