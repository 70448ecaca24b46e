// synth_dwt.cu -- wavelet-pyramid -> RGB synthesis and its backward (BASELINE config 3; HBM-bound, fp32).
//
// Replaces /root/reference/aphantasia/image.py:61-71 (dwt_image.inner): img = DWTInverse((Yl, [Yh_i * scale_i])),
// img * contrast / img.std(), fused with to_valid_rgb (image.py:21-28). DWTInverse is third-party
// (pytorch_wavelets 1.3.0, mode 'symmetric'; absent here -> restated from the published algorithm, SURVEY.md A7):
// per level, coarsest first, ll = SFB2D(ll_trimmed, (lh, hl, hh)) with
//   sfb1d(lo, hi) = conv_transpose(lo, rec_lo, stride 2, padding L-2) + conv_transpose(hi, rec_hi, stride 2, padding L-2)
// along rows then columns, i.e. out[Y][X] = sum_{a,b} g_r(a) g_c(b) band[(Y+L-2-a)/2][(X+L-2-b)/2] over the taps with even
// numerators inside the band, where (g_r, g_c) = (g0,g0) for ll, (g1,g0) for lh, (g0,g1) for hl, (g1,g1) for hh.
// One launch per level: k_dwt_level_fwd (thread = output pixel, (L/2)^2 taps x 4 bands from L1/L2) and its exact adjoint
// k_dwt_level_bwd (thread = coefficient position, L^2 taps of the output gradient, all 4 band gradients at once).
// The analysis of an image file (DWTForward, image.py:82-94) is separable: per level, finest first, k_dwt_afb_w filters along
// W (stride 2, L taps, symmetric extension) and k_dwt_afb_h along H into LL and the three bands.
#include "synth_common.cuh"
#include <vector>
#include <algorithm>

namespace aph {

constexpr int kMaxL = 40;       // filter taps (db20 = 40)
constexpr int kMaxLevels = 16;
struct Filt { float g0[kMaxL]; float g1[kMaxL]; int L; };

struct DwtPlanImpl : DeviceAllocs {
  int H, W, L, J;
  int lh[kMaxLevels], lw[kMaxLevels];      // band sizes, finest (level 1) first
  int oh[kMaxLevels], ow[kMaxLevels];      // output size of each level's synthesis: 2*l - L + 2
  Filt f;
  float* ll[kMaxLevels] = {};              // ll[i]: output of level i's synthesis (i = 0 is the image x_raw-sized scratch not used)
  float* dll[kMaxLevels] = {};             // gradient w.r.t. ll[i]
  float* gimg = nullptr; float* gx = nullptr;
};

// Half-sample symmetric extension of index j onto [0, n) (pytorch_wavelets mypad 'symmetric'): period 2n, so it also wraps
// lines shorter than the filter more than once.
__device__ __forceinline__ int sym_index(int j, int n) {
  const int per = 2 * n;
  j %= per;
  if (j < 0) j += per;
  return j < n ? j : per - 1 - j;
}

// Analysis along W (pytorch_wavelets afb1d, dim 3, mode 'symmetric'): x [3][h][w] -> rows [3][2][h][ow] = (lo, hi), with
// lo[k] = sum_t g0[t] x[sym(2k + t - pad)], hi with g1 (dec_lo[L-1-t] = rec_lo[t]), pad = (2 (ow - 1) - w + L) / 2.
__global__ void __launch_bounds__(256) k_dwt_afb_w(const float* __restrict__ x, int h, int w, float* __restrict__ rows, int ow, Filt f) {
  const int pad = (2 * (ow - 1) - w + f.L) / 2;
  const size_t total = (size_t)3 * h * ow;
  for (size_t idx = blockIdx.x * (size_t)blockDim.x + threadIdx.x; idx < total; idx += (size_t)gridDim.x * blockDim.x) {
    const int c = (int)(idx / ((size_t)h * ow));
    const int r = (int)(idx - (size_t)c * h * ow);
    const int y = r / ow, k = r - y * ow;
    const float* line = x + ((size_t)c * h + y) * w;
    float lo = 0.f, hi = 0.f;
    for (int t = 0; t < f.L; ++t) {
      const float v = __ldg(line + sym_index(2 * k + t - pad, w));
      lo += f.g0[t] * v; hi += f.g1[t] * v;
    }
    rows[(((size_t)c * 2 + 0) * h + y) * ow + k] = lo;
    rows[(((size_t)c * 2 + 1) * h + y) * ow + k] = hi;
  }
}

// Analysis along H of both halves: ll [3][oh][ow] and bands [3][3][oh][ow] * s in pytorch_wavelets' order (LH = H-high of the
// W-low half, HL = H-low of the W-high half, HH).
__global__ void __launch_bounds__(256) k_dwt_afb_h(const float* __restrict__ rows, int h, int ow, float* __restrict__ ll,
                                                   float* __restrict__ bands, float s, int oh, Filt f) {
  const int pad = (2 * (oh - 1) - h + f.L) / 2;
  const size_t total = (size_t)3 * oh * ow;
  for (size_t idx = blockIdx.x * (size_t)blockDim.x + threadIdx.x; idx < total; idx += (size_t)gridDim.x * blockDim.x) {
    const int c = (int)(idx / ((size_t)oh * ow));
    const int r = (int)(idx - (size_t)c * oh * ow);
    const int k = r / ow, l = r - k * ow;
    const float* lo = rows + (size_t)c * 2 * h * ow + l;
    const float* hi = lo + (size_t)h * ow;
    float a_ll = 0.f, a_lh = 0.f, a_hl = 0.f, a_hh = 0.f;
    for (int t = 0; t < f.L; ++t) {
      const size_t o = (size_t)sym_index(2 * k + t - pad, h) * ow;
      const float vl = __ldg(lo + o), vh = __ldg(hi + o);
      a_ll += f.g0[t] * vl; a_lh += f.g1[t] * vl; a_hl += f.g0[t] * vh; a_hh += f.g1[t] * vh;
    }
    ll[idx] = a_ll;
    bands[((size_t)(c * 3 + 0) * oh + k) * ow + l] = s * a_lh;
    bands[((size_t)(c * 3 + 1) * oh + k) * ow + l] = s * a_hl;
    bands[((size_t)(c * 3 + 2) * oh + k) * ow + l] = s * a_hh;
  }
}

// out [3][oh][ow] = SFB2D(ll [3][*][llw] (logical h x w), bands [3][3][h][w] * s)
__global__ void __launch_bounds__(256) k_dwt_level_fwd(const float* __restrict__ ll, int llh_alloc, int llw, const float* __restrict__ bands, float s,
                                                       int h, int w, float* __restrict__ out, int oh, int ow, Filt f,
                                                       double* __restrict__ stats) {
  const int p = f.L - 2;
  double s1 = 0., s2 = 0.;
  const size_t total = (size_t)3 * oh * ow;
  for (size_t idx = blockIdx.x * (size_t)blockDim.x + threadIdx.x; idx < total; idx += (size_t)gridDim.x * blockDim.x) {
    const int c = (int)(idx / ((size_t)oh * ow));
    const int r = (int)(idx - (size_t)c * oh * ow);
    const int Y = r / ow, X = r - Y * ow;
    const float* pll = ll + (size_t)c * llh_alloc * llw;
    const float* plh = bands + (size_t)(c * 3 + 0) * h * w;
    const float* phl = bands + (size_t)(c * 3 + 1) * h * w;
    const float* phh = bands + (size_t)(c * 3 + 2) * h * w;
    float acc = 0.f;
    for (int a = (Y + p) & 1; a < f.L; a += 2) {
      const int k = (Y + p - a) >> 1;
      if (Y + p - a < 0 || k >= h) continue;
      float r_ll = 0.f, r_lh = 0.f, r_hl = 0.f, r_hh = 0.f;      // column-filtered partial sums of row k
      for (int b = (X + p) & 1; b < f.L; b += 2) {
        const int l = (X + p - b) >> 1;
        if (X + p - b < 0 || l >= w) continue;
        const float c0 = f.g0[b], c1 = f.g1[b];
        r_ll += c0 * __ldg(pll + (size_t)k * llw + l);
        r_lh += c0 * __ldg(plh + (size_t)k * w + l);
        r_hl += c1 * __ldg(phl + (size_t)k * w + l);
        r_hh += c1 * __ldg(phh + (size_t)k * w + l);
      }
      acc += f.g0[a] * (r_ll + s * r_hl) + f.g1[a] * s * (r_lh + r_hh);
    }
    out[idx] = acc;
    if (stats) { s1 += acc; s2 += (double)acc * acc; }
  }
  if (stats) block_atomic_add_d({s1, s2}, stats);
}

// Adjoint: d_ll [3][llh_alloc][llw] (zero outside h x w), d_bands [3][3][h][w] (already multiplied by s) from d_out [3][oh][ow].
// With band.p / low.p set, Adam updates the band (and, at the coarsest level, Yl = d_ll's parameter) where its gradient is formed;
// dll / dbands may then be null and are not written.
__global__ void __launch_bounds__(256) k_dwt_level_bwd(const float* __restrict__ dout, int oh, int ow, float* __restrict__ dll, int llh_alloc,
                                                       int llw, float* __restrict__ dbands, float s, int h, int w, Filt f,
                                                       AdamArgs band, AdamArgs low) {
  const int p = f.L - 2;
  const size_t total = (size_t)3 * llh_alloc * llw;
  for (size_t idx = blockIdx.x * (size_t)blockDim.x + threadIdx.x; idx < total; idx += (size_t)gridDim.x * blockDim.x) {
    const int c = (int)(idx / ((size_t)llh_alloc * llw));
    const int r = (int)(idx - (size_t)c * llh_alloc * llw);
    const int k = r / llw, l = r - k * llw;
    if (k >= h || l >= w) { if (dll) dll[idx] = 0.f; continue; }      // rows / columns trimmed before the synthesis get no gradient
    const float* g = dout + (size_t)c * oh * ow;
    float a_ll = 0.f, a_lh = 0.f, a_hl = 0.f, a_hh = 0.f;
    for (int a = 0; a < f.L; ++a) {
      const int Y = 2 * k - p + a;
      if (Y < 0 || Y >= oh) continue;
      float r0 = 0.f, r1 = 0.f;                               // row Y of d_out filtered with g0 / g1 along x
      for (int b = 0; b < f.L; ++b) {
        const int X = 2 * l - p + b;
        if (X < 0 || X >= ow) continue;
        const float v = __ldg(g + (size_t)Y * ow + X);
        r0 += f.g0[b] * v; r1 += f.g1[b] * v;
      }
      a_ll += f.g0[a] * r0; a_lh += f.g1[a] * r0; a_hl += f.g0[a] * r1; a_hh += f.g1[a] * r1;
    }
    const size_t b0 = ((size_t)(c * 3) * h + k) * w + l, hw = (size_t)h * w;
    const float d0 = s * a_lh, d1 = s * a_hl, d2 = s * a_hh;
    if (dll) dll[idx] = a_ll;
    if (low.p) adam_elem(low, idx, a_ll);
    if (dbands) { dbands[b0] = d0; dbands[b0 + hw] = d1; dbands[b0 + 2 * hw] = d2; }
    if (band.p) { adam_elem(band, b0, d0); adam_elem(band, b0 + hw, d1); adam_elem(band, b0 + 2 * hw, d2); }
  }
}

// sum x, sum x^2 over n floats -> stats[0], stats[1] (fp64 atomics)
__global__ void __launch_bounds__(256) k_stats(const float* __restrict__ x, size_t n, double* __restrict__ stats) {
  double s1 = 0., s2 = 0.;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) { const float v = x[i]; s1 += v; s2 += (double)v * v; }
  block_atomic_add_d({s1, s2}, stats);
}
__global__ void k_fix_stats(double* stats, double n, double sigma) { stats[0] = 0.; stats[1] = sigma * sigma * (n - 1.0); stats[2] = 0.; }

}  // namespace aph

using namespace aph;

extern "C" int aph_dwt_plan_create(aph_dwt_plan** out, int H, int W, const float* rec_lo_host, const float* rec_hi_host, int L) {
  APH_REQUIRE(out && rec_lo_host && rec_hi_host, "aph_dwt_plan_create: null argument");
  APH_REQUIRE(L >= 2 && L <= kMaxL && L % 2 == 0, "aph_dwt_plan_create: filter length %d unsupported (even, <= %d)", L, kMaxL);
  APH_REQUIRE(H >= 2 && W >= 2, "aph_dwt_plan_create: bad size %dx%d", H, W);
  std::unique_ptr<DwtPlanImpl> p(new DwtPlanImpl());
  p->H = H; p->W = W; p->L = L;
  p->f.L = L;
  for (int i = 0; i < L; ++i) { p->f.g0[i] = rec_lo_host[i]; p->f.g1[i] = rec_hi_host[i]; }
  int J = 0; for (int m = std::min(H, W); m > 1; m >>= 1) ++J;      // floor(log2(min(H, W)))  (image.py:35-36)
  APH_REQUIRE(J >= 1 && J <= kMaxLevels, "aph_dwt_plan_create: %d levels unsupported", J);
  p->J = J;
  int h = H, w = W;
  for (int i = 0; i < J; ++i) { h = (h + L - 1) / 2; w = (w + L - 1) / 2; p->lh[i] = h; p->lw[i] = w; p->oh[i] = 2 * h - L + 2; p->ow[i] = 2 * w - L + 2; }
  // ll[i] (i >= 1) = output of level (i+1)'s synthesis = low-pass input of level i (0-based level index i-1); ll[J] is Yl itself
  for (int i = 1; i < J; ++i) {
    if (int e = p->alloc(&p->ll[i], (size_t)3 * p->oh[i] * p->ow[i])) return e;
    if (int e = p->alloc(&p->dll[i], (size_t)3 * p->oh[i] * p->ow[i])) return e;
  }
  const size_t n = (size_t)3 * p->oh[0] * p->ow[0];
  if (int e = p->alloc(&p->gimg, n)) return e;
  if (int e = p->alloc(&p->gx, n)) return e;
  *out = reinterpret_cast<aph_dwt_plan*>(p.release());
  return 0;
}

extern "C" int aph_dwt_plan_destroy(aph_dwt_plan* plan) {
  delete reinterpret_cast<DwtPlanImpl*>(plan);
  return 0;
}

extern "C" int aph_dwt_plan_levels(const aph_dwt_plan* plan, int* J, int* dims, int* out_hw) {
  APH_REQUIRE(plan && J, "aph_dwt_plan_levels: null argument");
  const DwtPlanImpl* p = reinterpret_cast<const DwtPlanImpl*>(plan);
  *J = p->J;
  if (dims) for (int i = 0; i < p->J; ++i) { dims[2 * i] = p->lh[i]; dims[2 * i + 1] = p->lw[i]; }
  if (out_hw) { out_hw[0] = p->oh[0]; out_hw[1] = p->ow[0]; }
  return 0;
}

// Ys: HOST array of J+1 device pointers {Yl [3,h_J,w_J], Yh_1 [3,3,h_1,w_1] (finest), ..., Yh_J}; scales: HOST [J].
extern "C" int aph_synth_dwt_fwd(aph_dwt_plan* plan, const float* const* Ys, const float* scales_host, float contrast,
                                 const float* colmat_host, int apply_sigmoid, float* x_raw, double* stats, float* out, void* stream) {
  APH_REQUIRE(plan && Ys && scales_host && x_raw && stats && out, "aph_synth_dwt_fwd: null pointer");
  DwtPlanImpl* p = reinterpret_cast<DwtPlanImpl*>(plan);
  cudaStream_t st = (cudaStream_t)stream;
  APH_CUDA_OK(cudaMemsetAsync(stats, 0, 4 * sizeof(double), st));
  const int J = p->J;
  for (int i = J - 1; i >= 0; --i) {                   // level index i (0 = finest); coarsest first
    const float* ll = (i == J - 1) ? Ys[0] : p->ll[i + 1];
    const int llh = (i == J - 1) ? p->lh[J - 1] : p->oh[i + 1], llw = (i == J - 1) ? p->lw[J - 1] : p->ow[i + 1];
    float* o = (i == 0) ? x_raw : p->ll[i];
    const size_t n = (size_t)3 * p->oh[i] * p->ow[i];
    k_dwt_level_fwd<<<stride_blocks(n, 16), 256, 0, st>>>(ll, llh, llw, Ys[i + 1], scales_host[i], p->lh[i], p->lw[i], o, p->oh[i], p->ow[i], p->f,
                                                          i == 0 ? stats : nullptr);
    APH_LAUNCH_OK();
  }
  const size_t hw = (size_t)p->oh[0] * p->ow[0];
  k_finish<true><<<stride_blocks(hw, 16), 256, 0, st>>>(x_raw, stats, out, hw, contrast, make_colmat(colmat_host), apply_sigmoid);
  APH_LAUNCH_OK();
  return 0;
}

extern "C" int aph_synth_dwt_bwd(aph_dwt_plan* plan, const float* grad_out, const float* out, const float* x_raw, double* stats,
                                 const float* scales_host, float contrast, const float* colmat_host, int apply_sigmoid,
                                 float* const* grad_Ys, void* stream, float* const* params, float* const* m, float* const* v,
                                 float* const* vmax, float lr, float b1, float b2, float eps, float weight_decay, int step) {
  APH_REQUIRE(plan && grad_out && x_raw && stats && scales_host && (grad_Ys || params), "aph_synth_dwt_bwd: null pointer");
  APH_REQUIRE(!params || (m && v && step >= 1), "aph_synth_dwt_bwd: bad Adam state");
  APH_REQUIRE(!apply_sigmoid || out, "aph_synth_dwt_bwd: sigmoid backward needs the saved output");
  DwtPlanImpl* p = reinterpret_cast<DwtPlanImpl*>(plan);
  cudaStream_t st = (cudaStream_t)stream;
  const size_t hw = (size_t)p->oh[0] * p->ow[0];
  APH_CUDA_OK(cudaMemsetAsync(stats + 2, 0, sizeof(double), st));
  k_finish_bwd<<<stride_blocks(hw, 16), 256, 0, st>>>(grad_out, out, x_raw, p->gimg, stats, hw, make_colmat(colmat_host), apply_sigmoid);
  APH_LAUNCH_OK();
  k_norm_bwd<<<stride_blocks(3 * hw, 16), 256, 0, st>>>(p->gimg, x_raw, stats, p->gx, 3 * hw, contrast, AdamArgs{});
  APH_LAUNCH_OK();
  const int J = p->J;
  for (int i = 0; i < J; ++i) {                        // finest first
    const float* dout = (i == 0) ? p->gx : p->dll[i];
    float* dll = (i == J - 1) ? (grad_Ys ? grad_Ys[0] : nullptr) : p->dll[i + 1];
    const int llh = (i == J - 1) ? p->lh[J - 1] : p->oh[i + 1], llw = (i == J - 1) ? p->lw[J - 1] : p->ow[i + 1];
    const size_t n = (size_t)3 * llh * llw;
    // Yl is params[0] and Yh_(i+1) is params[i + 1], as in Ys
    auto adam_of = [&](int t) { return params ? make_adam(params[t], m[t], v[t], vmax ? vmax[t] : nullptr, lr, b1, b2, eps, weight_decay, step)
                                              : AdamArgs{}; };
    k_dwt_level_bwd<<<stride_blocks(n, 16), 256, 0, st>>>(dout, p->oh[i], p->ow[i], dll, llh, llw, grad_Ys ? grad_Ys[i + 1] : nullptr,
                                                          scales_host[i], p->lh[i], p->lw[i], p->f, adam_of(i + 1),
                                                          i == J - 1 ? adam_of(0) : AdamArgs{});
    APH_LAUNCH_OK();
  }
  return 0;
}

// Analysis (image-file resume, aphantasia/image.py:82-94): DWTForward(J, mode 'symmetric') of img [3,H,W], finest level first;
// Ys as in aph_synth_dwt_fwd (written here), Yh_i multiplied by inv_scales_host[i]. Level i's LL lands in ll[i + 1], which
// holds the oh[i + 1] x ow[i + 1] >= lh[i] x lw[i] synthesis output of that level, and the last one in Yl.
// The row-filtered halves [3][2][h][ow] of each level go to a stream-ordered temporary of exactly that level's size, freed
// behind the level's two launches: the long-lived plan keeps nothing for the analysis, and no size formula can fall short
// when lines shorter than the filter make the levels grow (h -> (h + L - 1) / 2 > h for h < L - 1).
extern "C" int aph_dwt_analyze(aph_dwt_plan* plan, const float* img, const float* inv_scales_host, float* const* Ys, void* stream) {
  APH_REQUIRE(plan && img && inv_scales_host && Ys, "aph_dwt_analyze: null pointer");
  DwtPlanImpl* p = reinterpret_cast<DwtPlanImpl*>(plan);
  cudaStream_t st = (cudaStream_t)stream;
  const int J = p->J;
  const float* x = img;
  int h = p->H, w = p->W;
  for (int i = 0; i < J; ++i) {
    const int oh = p->lh[i], ow = p->lw[i];
    StreamTemp<float> rows;
    if (int e = rows.alloc((size_t)3 * 2 * h * ow, st)) return e;
    float* ll = (i == J - 1) ? Ys[0] : p->ll[i + 1];
    k_dwt_afb_w<<<stride_blocks((size_t)3 * h * ow, 16), 256, 0, st>>>(x, h, w, rows.p, ow, p->f);
    APH_LAUNCH_OK();
    k_dwt_afb_h<<<stride_blocks((size_t)3 * oh * ow, 16), 256, 0, st>>>(rows.p, h, ow, ll, Ys[i + 1], inv_scales_host[i], oh, p->f);
    APH_LAUNCH_OK();
    x = ll; h = oh; w = ow;
  }
  return 0;
}

// Direct RGB parameterisation (pixel_image, /root/reference/aphantasia/image.py:98-119): img = x * contrast / std(x), or
// x * contrast / 3.3 with fixcontrast; fused with to_valid_rgb like the spectral generators. x, out, grad_x: [3,H,W].
extern "C" int aph_pixel_fwd(const float* x, int64_t hw, float contrast, int fixcontrast, const float* colmat_host, int apply_sigmoid,
                             double* stats, float* out, void* stream) {
  APH_REQUIRE(x && stats && out && hw > 0, "aph_pixel_fwd: bad arguments");
  cudaStream_t st = (cudaStream_t)stream;
  APH_CUDA_OK(cudaMemsetAsync(stats, 0, 4 * sizeof(double), st));
  if (fixcontrast) k_fix_stats<<<1, 1, 0, st>>>(stats, 3.0 * (double)hw, 3.3);       // sigma := 3.3 (image.py:115)
  else k_stats<<<stride_blocks(3 * (size_t)hw, 16), 256, 0, st>>>(x, 3 * (size_t)hw, stats);
  APH_LAUNCH_OK();
  k_finish<true><<<stride_blocks((size_t)hw, 16), 256, 0, st>>>(x, stats, out, (size_t)hw, contrast, make_colmat(colmat_host), apply_sigmoid);
  APH_LAUNCH_OK();
  return 0;
}

extern "C" int aph_pixel_bwd(const float* grad_out, const float* out, const float* x, double* stats, int64_t hw, float contrast,
                             int fixcontrast, const float* colmat_host, int apply_sigmoid, float* grad_x, void* stream, float* params,
                             float* m, float* v, float* vmax, float lr, float b1, float b2, float eps, float weight_decay, int step) {
  APH_REQUIRE(grad_out && x && stats && grad_x && hw > 0, "aph_pixel_bwd: bad arguments");
  APH_REQUIRE(!params || (m && v && step >= 1), "aph_pixel_bwd: bad Adam state");
  APH_REQUIRE(!apply_sigmoid || out, "aph_pixel_bwd: sigmoid backward needs the saved output");
  cudaStream_t st = (cudaStream_t)stream;
  APH_CUDA_OK(cudaMemsetAsync(stats + 2, 0, sizeof(double), st));
  // g_img lands in grad_x, then is rewritten in place by the normalisation adjoint (with fixcontrast the std term vanishes), or,
  // with params, feeds the Adam update of params (which may be x itself) in that same pass
  k_finish_bwd<<<stride_blocks((size_t)hw, 16), 256, 0, st>>>(grad_out, out, fixcontrast ? nullptr : x, grad_x, stats, (size_t)hw,
                                                              make_colmat(colmat_host), apply_sigmoid);
  APH_LAUNCH_OK();
  k_norm_bwd<<<stride_blocks(3 * (size_t)hw, 16), 256, 0, st>>>(grad_x, x, stats, grad_x, 3 * (size_t)hw, contrast,
                                                                params ? make_adam(params, m, v, vmax, lr, b1, b2, eps, weight_decay, step)
                                                                       : AdamArgs{});
  APH_LAUNCH_OK();
  return 0;
}
