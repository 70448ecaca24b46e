// lpips.cu -- LPIPS (lpips v0.1, net='vgg', lpips=True, spatial=False) forward and data-gradient for clip_fft.py --sync.
//
//   x' = ((a x + b) - shift) / scale            a, b = 2, -1 with normalize=True, else 1, 0; per-channel scaling layer
//   VGG16 features[0:30]: 13 conv3x3 (pad 1, bias) + ReLU, max-pool 2x2 (floor) after relu1_2, relu2_2, relu3_3, relu4_3
//   taps t = relu1_2, relu2_2, relu3_3, relu4_3, relu5_3:  n = f / (|f|_2 over channels + 1e-10)
//   LPIPS[i] = sum_t mean_{h,w} sum_c lin_t[c] (n0 - n1)^2
//
// Kernels (all sm_90a):
//   conv1_1 (C_in = 3)   k_conv3in_fwd<1, 64, IN_LPIPS> (nhwc.cu): fp32 SIMT, fused with the input scaling, bias and ReLU -> bf16
//                        NHWC; k_conv3in_bwd<1, 64, IN_LPIPS>: fp32 SIMT, d canvas from the masked gradient of relu1_1
//   the other 12 convs   k_conv3x3_tc (conv_tc.cuh, launched by conv_tc.cu): implicit GEMM on wgmma, forward and data gradient
//   max-pool             k_pool2<POOL_MAX> (nhwc.cu; ties: the first element of the window in row-major order, as torch.max_pool2d)
//   head                 k_head_fwd: one warp per tap pixel, block partials in a fixed order (no float atomics), k_head_fin
//                        k_tap_bwd: per tap pixel, d head / d f0 (scaled by the upstream gradient read from a DEVICE pointer)
//                        + the max-pool adjoint of the layer above, then the ReLU mask of the tap as a select -> d pre-ReLU
//
// The handle keeps two activation arenas: the saved forward of in0 (for the backward) and the features of in1, which are cached
// under a caller-supplied key (clip_fft.py passes the same reference picture every step). Both grow to the largest shape seen and
// survive torch.cuda.empty_cache(). Every forward bumps a generation; a backward must name the generation it belongs to.
#include "nhwc.cuh"
#include "weights.cuh"

namespace aph {

constexpr int LP_CONVS = 13, LP_TAPS = 5;
constexpr int LP_HEAD_BLOCKS = 64;                                         // fixed reduction tree of the head, per (tap, image)
static const int kCin[LP_CONVS] = {3, 64, 64, 128, 128, 256, 256, 256, 512, 512, 512, 512, 512};
static const int kCout[LP_CONVS] = {64, 64, 128, 128, 256, 256, 256, 512, 512, 512, 512, 512, 512};
static const int kLevel[LP_CONVS] = {0, 0, 1, 1, 2, 2, 2, 3, 3, 3, 4, 4, 4};   // spatial level (pools before it)
static const int kFeatIdx[LP_CONVS] = {0, 2, 5, 7, 10, 12, 14, 17, 19, 21, 24, 26, 28};   // torchvision features.{i}
static const int kTapConv[LP_TAPS] = {1, 3, 6, 9, 12};                    // conv whose ReLU output is tap t
static inline int tap_of(int l) { for (int t = 0; t < LP_TAPS; ++t) if (kTapConv[t] == l) return t; return -1; }

// ---- the LPIPS head ----------------------------------------------------------------------------------------
// f0, f1 bf16 NHWC [N, HW, C] (one tap); lin [C]. One warp per pixel; block b of image n sums its warps' pixel values in a fixed
// order into part[n * LP_HEAD_BLOCKS + b] (double).
__global__ void __launch_bounds__(256) k_head_fwd(const bf16* __restrict__ f0, const bf16* __restrict__ f1, const float* __restrict__ lin,
                                                  int HW, int C, double* __restrict__ part) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, n = blockIdx.y;
  double acc = 0.;
  for (int p = blockIdx.x * 8 + warp; p < HW; p += LP_HEAD_BLOCKS * 8) {
    const bf16* a = f0 + ((size_t)n * HW + p) * C;
    const bf16* b = f1 + ((size_t)n * HW + p) * C;
    float s0 = 0.f, s1 = 0.f;
    for (int c = lane; c < C; c += 32) { const float u = __bfloat162float(a[c]), v = __bfloat162float(b[c]); s0 += u * u; s1 += v * v; }
    s0 = warp_sum(s0); s1 = warp_sum(s1);
    const float i0 = 1.f / (sqrtf(s0) + 1e-10f), i1 = 1.f / (sqrtf(s1) + 1e-10f);
    float d = 0.f;
    for (int c = lane; c < C; c += 32) { const float t = __bfloat162float(a[c]) * i0 - __bfloat162float(b[c]) * i1; d += lin[c] * t * t; }
    d = warp_sum(d);
    acc += (double)d;
  }
  __shared__ double red[8];
  if (lane == 0) red[warp] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    double s = 0.;
    for (int w = 0; w < 8; ++w) s += red[w];
    part[(size_t)n * LP_HEAD_BLOCKS + blockIdx.x] = s;
  }
}
// out[n] = sum_t (sum_b part[t][n][b]) / HW_t
struct HeadHW { int hw[LP_TAPS]; };
__global__ void k_head_fin(const double* __restrict__ part, int N, HeadHW hw, float* __restrict__ out) {
  const int n = blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= N) return;
  double v = 0.;
  for (int t = 0; t < LP_TAPS; ++t) {
    double s = 0.;
    for (int b = 0; b < LP_HEAD_BLOCKS; ++b) s += part[((size_t)t * N + n) * LP_HEAD_BLOCKS + b];
    v += s / (double)hw.hw[t];
  }
  out[n] = (float)v;
}

// d loss / d (pre-ReLU output of the tap's conv), one warp per tap pixel, C / 32 channels per lane:
//   g = [lin: d head / d f0 x up[n] / HW] + [dpool: the max-pool adjoint of dpool (bf16 [N, H/2, W/2, C])]
//   out = f0 > 0 ? g : 0          (f0 is the tap, the ReLU output; a select, never a multiply)
// d head / d f0 = gn / e - f (f . gn) / (e^2 |f|), gn = 2 lin (n0 - n1), e = |f| + 1e-10. At |f| = 0 the second term is
// singular (PyTorch gets NaN there); every channel of such a pixel is masked, so it is left out.
// lin == NULL: no head term; mask == 0: no select (the max-pool test entry).
__global__ void __launch_bounds__(256) k_tap_bwd(const bf16* __restrict__ f0, const bf16* __restrict__ f1, const float* __restrict__ lin,
                                                 const float* __restrict__ up, const bf16* __restrict__ dpool, int N, int H, int W, int C,
                                                 int mask, bf16* __restrict__ out) {
  const int lane = threadIdx.x & 31;
  const size_t HW = (size_t)H * W, n_pix = (size_t)N * HW;
  const int Ho = H / 2, Wo = W / 2;
  for (size_t p = (blockIdx.x * (size_t)blockDim.x + threadIdx.x) >> 5; p < n_pix; p += ((size_t)gridDim.x * blockDim.x) >> 5) {
    const int n = (int)(p / HW), rem = (int)(p - n * HW), y = rem / W, x = rem - y * W;
    const bf16* a = f0 + p * C;
    float k1 = 0.f, i0 = 0.f, i1 = 0.f, k2 = 0.f;
    if (lin) {
      const bf16* b = f1 + p * C;
      float s0 = 0.f, s1 = 0.f;
      for (int c = lane; c < C; c += 32) { const float u = __bfloat162float(a[c]), v = __bfloat162float(b[c]); s0 += u * u; s1 += v * v; }
      s0 = warp_sum(s0); s1 = warp_sum(s1);
      const float r0 = sqrtf(s0), e0 = r0 + 1e-10f;
      i0 = 1.f / e0; i1 = 1.f / (sqrtf(s1) + 1e-10f);
      k1 = up[n] / (float)HW;
      float dot = 0.f;                                         // f . gn
      for (int c = lane; c < C; c += 32) {
        const float u = __bfloat162float(a[c]);
        dot += u * 2.f * lin[c] * (u * i0 - __bfloat162float(b[c]) * i1);
      }
      dot = warp_sum(dot);
      k2 = r0 > 0.f ? dot * i0 * i0 / r0 : 0.f;
    }
    const bool in_pool = dpool && y < 2 * Ho && x < 2 * Wo;
    const int yo = y >> 1, xo = x >> 1, self = ((y & 1) << 1) | (x & 1);
    for (int c = lane; c < C; c += 32) {
      const float u = __bfloat162float(a[c]);
      float g = 0.f;
      if (lin) g = k1 * (2.f * lin[c] * (u * i0 - __bfloat162float(f1[p * C + c]) * i1) * i0 - u * k2);
      if (in_pool) {
        const bf16* w0 = f0 + (((size_t)n * H + 2 * yo) * W + 2 * xo) * C + c;
        const float v[4] = {__bfloat162float(w0[0]), __bfloat162float(w0[C]), __bfloat162float(w0[(size_t)W * C]),
                            __bfloat162float(w0[(size_t)W * C + C])};
        int am = 0;
#pragma unroll
        for (int k = 1; k < 4; ++k) if (v[k] > v[am]) am = k;
        if (am == self) g += __bfloat162float(dpool[(((size_t)n * Ho + yo) * Wo + xo) * C + c]);
      }
      out[p * C + c] = __float2bfloat16((!mask || u > 0.f) ? g : 0.f);
    }
  }
}

// ---- launchers ----------------------------------------------------------------------------------------------
static int launch_tap_bwd(const bf16* f0, const bf16* f1, const float* lin, const float* up, const bf16* dpool, int N, int H, int W,
                          int C, int mask, bf16* out, cudaStream_t st) {
  k_tap_bwd<<<stride_blocks((size_t)N * H * W * 32, 16), 256, 0, st>>>(f0, f1, lin, up, dpool, N, H, W, C, mask, out);
  APH_LAUNCH_OK();
  return 0;
}

// ---- the handle ---------------------------------------------------------------------------------------------
struct LpLayout {           // element offsets (bf16) of the 13 conv outputs and 4 pool outputs inside one arena
  size_t act[LP_CONVS], pool[4], total;
  int h[5], w[5];
  void plan(int N, int H, int W) {
    h[0] = H; w[0] = W;
    for (int k = 1; k < 5; ++k) { h[k] = h[k - 1] / 2; w[k] = w[k - 1] / 2; }
    size_t o = 0;
    auto take = [&](size_t n) { const size_t r = o; o += (n + 127) / 128 * 128; return r; };
    for (int l = 0; l < LP_CONVS; ++l) act[l] = take((size_t)N * h[kLevel[l]] * w[kLevel[l]] * kCout[l]);
    for (int t = 0; t < 4; ++t) pool[t] = take((size_t)N * h[t + 1] * w[t + 1] * kCout[kTapConv[t]]);
    total = o;
  }
};

}  // namespace aph

using namespace aph;

struct aph_lpips : Weights {
  float* w0 = nullptr;                      // conv1_1 fp32 [64][27]
  float* bias[LP_CONVS] = {};               // fp32 [Cout]
  bf16* wf[LP_CONVS] = {};                  // [Cout, 9 Cin] (l >= 1)
  bf16* wb[LP_CONVS] = {};                  // [Cin, 9 Cout] (l >= 1)
  float* lin[LP_TAPS] = {};                 // [C_t]
  Scratch main_arena, ref_arena, grads, part;
  int64_t generation = 0, saved_generation = -1;
  int sN = 0, sH = 0, sW = 0, s_norm = 0;   // shape of the saved forward
  uint64_t ref_key = 0;                     // 0 = the reference arena is not reusable
  int rN = 0, rH = 0, rW = 0;
};

static int vgg_forward(aph_lpips* h, const float* img, int N, int H, int W, int normalize, bf16* arena, const LpLayout& lay,
                       cudaStream_t st) {
  const float a = normalize ? 2.f : 1.f, b = normalize ? -1.f : 0.f;
  if (int r = launch_conv3in_fwd<1, 64, IN_LPIPS>(img, N, H, W, h->w0, h->bias[0], arena + lay.act[0], st, a, b)) return r;
  for (int l = 1; l < LP_CONVS; ++l) {
    const int lv = kLevel[l], tp = tap_of(l - 1);
    const bf16* in = (tp >= 0) ? arena + lay.pool[tp] : arena + lay.act[l - 1];
    ConvEpi e; e.bias = h->bias[l]; e.out = arena + lay.act[l];
    if (int r = launch_conv3x3(in, h->wf[l], N, lay.h[lv], lay.w[lv], kCin[l], kCout[l], CONV_BIAS_RELU, e, st)) return r;
    const int t = tap_of(l);
    if (t >= 0 && t < 4)
      if (int r = launch_pool2(POOL_MAX, arena + lay.act[l], N, lay.h[lv], lay.w[lv], kCout[l], arena + lay.pool[t], st)) return r;
  }
  return 0;
}

// Keys: torchvision's "features.{i}.weight" [Co,Ci,3,3] / "features.{i}.bias" [Co] for the 13 convolutions, and lpips'
// "lin{t}.model.1.weight" [1,C,1,1]. Other keys are refused (the Python loader drops the classifier and anything else).
extern "C" int aph_lpips_create(aph_lpips** out) {
  APH_REQUIRE(out, "aph_lpips_create: null handle pointer");
  std::unique_ptr<aph_lpips> h(new aph_lpips());
  int e = 0;
  for (int l = 0; l < LP_CONVS; ++l) {
    const std::string f = "features." + std::to_string(kFeatIdx[l]);
    if (l == 0) e |= h->add_f32(f + ".weight", &h->w0, 64 * 27);
    else e |= h->add_conv3x3(f + ".weight", kCout[l], kCin[l], &h->wf[l], &h->wb[l]);
    e |= h->add_f32(f + ".bias", &h->bias[l], kCout[l]);
  }
  for (int t = 0; t < LP_TAPS; ++t) e |= h->add_f32("lin" + std::to_string(t) + ".model.1.weight", &h->lin[t], kCout[kTapConv[t]]);
  if (e) return 1;
  *out = h.release();
  return 0;
}

extern "C" int aph_lpips_destroy(aph_lpips* h) {
  delete h;
  return 0;
}

extern "C" int aph_lpips_load_tensor(aph_lpips* h, const char* key, const float* data, int64_t numel, void* stream) {
  return load_tensor(h, key, data, numel, (cudaStream_t)stream, "aph_lpips_load_tensor");
}

extern "C" int aph_lpips_finalize(aph_lpips* h) {
  if (int e = finalize(h, "aph_lpips_finalize")) return e;
  h->ref_key = 0;           // new weights: cached reference features are void
  ++h->generation;
  return 0;
}

// in0, in1 fp32 NCHW [N,3,H,W]; out [N]. in1 may be NULL when ref_key is non-zero and equals the key of the cached reference
// features (same N, H, W); otherwise in1's features are computed and cached under ref_key (0: not reusable).
extern "C" int aph_lpips_fwd(aph_lpips* h, const float* in0, const float* in1, uint64_t ref_key, int N, int H, int W, int normalize,
                             float* out, int save_for_bwd, int64_t* generation, void* stream) {
  APH_REQUIRE(h && h->finalized, "aph_lpips_fwd: handle not finalized");
  APH_REQUIRE(in0 && out && N > 0, "aph_lpips_fwd: bad arguments");
  APH_REQUIRE(H >= 16 && W >= 16, "aph_lpips_fwd: images of %dx%d are below VGG16's 16x16 (four 2x2 max-pools)", H, W);
  cudaStream_t st = (cudaStream_t)stream;
  LpLayout lay;
  lay.plan(N, H, W);
  const bool reuse = ref_key != 0 && ref_key == h->ref_key && N == h->rN && H == h->rH && W == h->rW;
  APH_REQUIRE(reuse || in1, "aph_lpips_fwd: no reference image and no cached features under this key");
  ++h->generation;                                  // the main arena is about to change: any saved forward is void
  h->saved_generation = -1;
  if (int e = h->main_arena.grow(lay.total * sizeof(bf16), st)) return e;
  if (int e = h->part.grow((size_t)LP_TAPS * N * LP_HEAD_BLOCKS * sizeof(double), st)) return e;
  bf16* A = reinterpret_cast<bf16*>(h->main_arena.p);
  if (!reuse) {
    h->ref_key = 0;
    if (int e = h->ref_arena.grow(lay.total * sizeof(bf16), st)) return e;
    if (int e = vgg_forward(h, in1, N, H, W, normalize, reinterpret_cast<bf16*>(h->ref_arena.p), lay, st)) return e;
    h->ref_key = ref_key; h->rN = N; h->rH = H; h->rW = W;
  }
  const bf16* R = reinterpret_cast<const bf16*>(h->ref_arena.p);
  if (int e = vgg_forward(h, in0, N, H, W, normalize, A, lay, st)) return e;
  double* part = reinterpret_cast<double*>(h->part.p);
  HeadHW hw;
  for (int t = 0; t < LP_TAPS; ++t) {
    const int l = kTapConv[t], lv = kLevel[l];
    hw.hw[t] = lay.h[lv] * lay.w[lv];
    k_head_fwd<<<dim3(LP_HEAD_BLOCKS, N), 256, 0, st>>>(A + lay.act[l], R + lay.act[l], h->lin[t], hw.hw[t], kCout[l],
                                                         part + (size_t)t * N * LP_HEAD_BLOCKS);
    APH_LAUNCH_OK();
  }
  k_head_fin<<<(N + 127) / 128, 128, 0, st>>>(part, N, hw, out);
  APH_LAUNCH_OK();
  if (save_for_bwd) { h->saved_generation = h->generation; h->sN = N; h->sH = H; h->sW = W; h->s_norm = normalize; }
  if (generation) *generation = h->generation;
  return 0;
}

// grad_out [N] DEVICE (d loss / d LPIPS[n]) -> grad_in0 [N,3,H,W] (overwritten), from the forward of `generation`
// (save_for_bwd = 1). A later forward on the handle voids it: the call then fails and launches nothing.
extern "C" int aph_lpips_bwd(aph_lpips* h, const float* grad_out, int64_t generation, float* grad_in0, void* stream) {
  APH_REQUIRE(h && grad_out && grad_in0, "aph_lpips_bwd: bad arguments");
  APH_REQUIRE(h->saved_generation >= 0 && generation == h->saved_generation,
              "aph_lpips_bwd: the activations of forward %lld were overwritten by a later forward (saved: %lld)",
              (long long)generation, (long long)h->saved_generation);
  cudaStream_t st = (cudaStream_t)stream;
  const int N = h->sN, H = h->sH, W = h->sW;
  LpLayout lay;
  lay.plan(N, H, W);
  const size_t gmax = (size_t)N * H * W * 64;       // the largest gradient: relu1_x
  if (int e = h->grads.grow(2 * gmax * sizeof(bf16), st)) return e;
  bf16* G[2] = {reinterpret_cast<bf16*>(h->grads.p), reinterpret_cast<bf16*>(h->grads.p) + gmax};
  const bf16* A = reinterpret_cast<const bf16*>(h->main_arena.p);
  const bf16* R = reinterpret_cast<const bf16*>(h->ref_arena.p);
  int cur = 0;                                      // G[cur] holds d loss / d (pre-ReLU output of conv l)
  {
    const int l = LP_CONVS - 1, lv = kLevel[l];
    if (int e = launch_tap_bwd(A + lay.act[l], R + lay.act[l], h->lin[4], grad_out, nullptr, N, lay.h[lv], lay.w[lv], kCout[l], 1, G[cur], st)) return e;
  }
  for (int l = LP_CONVS - 1; l >= 1; --l) {
    const int lv = kLevel[l], tp = tap_of(l - 1);
    ConvEpi e;
    e.out = G[cur ^ 1];
    if (tp >= 0) {                                  // input = max-pool of tap tp: plain store, then adjoint + head + mask
      if (int r = launch_conv3x3(G[cur], h->wb[l], N, lay.h[lv], lay.w[lv], kCout[l], kCin[l], CONV_PLAIN, e, st)) return r;
      const int lb = l - 1, lvb = kLevel[lb];
      if (int r = launch_tap_bwd(A + lay.act[lb], R + lay.act[lb], h->lin[tp], grad_out, G[cur ^ 1], N, lay.h[lvb], lay.w[lvb],
                                 kCout[lb], 1, G[cur], st)) return r;
    } else {                                        // input = ReLU output of conv l - 1: mask in the epilogue
      e.mask = A + lay.act[l - 1];
      if (int r = launch_conv3x3(G[cur], h->wb[l], N, lay.h[lv], lay.w[lv], kCout[l], kCin[l], CONV_MASK, e, st)) return r;
      cur ^= 1;
    }
  }
  return launch_conv3in_bwd<1, 64, IN_LPIPS>(G[cur], N, H, W, h->w0, grad_in0, st, h->s_norm ? 2.f : 1.f);
}

// ---- test entries -------------------------------------------------------------------------------------------
// One 3x3 layer on caller buffers. weight fp32 [Cout, Cin, 3, 3] (packed here, as the loader does). fwd = 1: x bf16 NHWC
// [N,H,W,Cin] -> out = relu(conv(x) + bias) [N,H,W,Cout]. fwd = 0: x = dy [N,H,W,Cout] -> out = dx [N,H,W,Cin], selected by
// mask > 0 (mask bf16 [N,H,W,Cin]) when mask is not NULL.
extern "C" int aph_lpips_conv_test(int fwd, const void* x, const float* weight, const float* bias, const void* mask, void* out, int N,
                                   int H, int W, int Cin, int Cout, void* stream) {
  APH_REQUIRE(x && weight && out && (bias || !fwd), "aph_lpips_conv_test: bad arguments");
  APH_REQUIRE(Cin % 64 == 0 && Cout % 64 == 0, "aph_lpips_conv_test: C_in=%d and C_out=%d must be multiples of 64", Cin, Cout);
  cudaStream_t st = (cudaStream_t)stream;
  StreamTemp<bf16> wp;
  if (int r = wp.alloc((size_t)Cout * Cin * 9, st)) return r;
  if (int r = pack_conv3x3(weight, Cout, Cin, fwd ? wp.p : nullptr, fwd ? nullptr : wp.p, st)) return r;
  ConvEpi e;
  e.out = reinterpret_cast<bf16*>(out);
  if (fwd) {
    e.bias = bias;
    return launch_conv3x3(x, wp.p, N, H, W, Cin, Cout, CONV_BIAS_RELU, e, st);
  }
  e.mask = reinterpret_cast<const bf16*>(mask);
  return launch_conv3x3(x, wp.p, N, H, W, Cout, Cin, mask ? CONV_MASK : CONV_PLAIN, e, st);
}

// conv1_1 on caller buffers: weight fp32 [64,3,3,3], bias [64]. fwd = 1: img fp32 [N,3,H,W] -> out bf16 NHWC [N,H,W,64]
// (ReLU output, with the input scaling: normalize = 1 maps x to 2x - 1 first). fwd = 0: dz bf16 [N,H,W,64] (d pre-ReLU) ->
// out fp32 [N,3,H,W] = d loss / d img.
extern "C" int aph_lpips_conv0_test(int fwd, const void* in, const float* weight, const float* bias, void* out, int N, int H, int W,
                                    int normalize, void* stream) {
  APH_REQUIRE(in && weight && out && (bias || !fwd) && N > 0 && H > 0 && W > 0, "aph_lpips_conv0_test: bad arguments");
  cudaStream_t st = (cudaStream_t)stream;
  const float a = normalize ? 2.f : 1.f, b = normalize ? -1.f : 0.f;
  if (fwd) return launch_conv3in_fwd<1, 64, IN_LPIPS>(reinterpret_cast<const float*>(in), N, H, W, weight, bias, reinterpret_cast<bf16*>(out),
                                                      st, a, b);
  return launch_conv3in_bwd<1, 64, IN_LPIPS>(reinterpret_cast<const bf16*>(in), N, H, W, weight, reinterpret_cast<float*>(out), st, a);
}

// 2x2 max-pool on caller buffers, bf16 NHWC, C % 8 == 0. fwd = 1: out = pool(x) [N,H/2,W/2,C]. fwd = 0: out [N,H,W,C] = the
// adjoint of dy [N,H/2,W/2,C] (the window's first maximum of x gets dy, rows / columns dropped by floor mode get zero).
extern "C" int aph_lpips_pool_test(int fwd, const void* x, const void* dy, void* out, int N, int H, int W, int C, void* stream) {
  APH_REQUIRE(x && out && (fwd || dy) && C % 8 == 0 && H >= 2 && W >= 2, "aph_lpips_pool_test: bad arguments");
  cudaStream_t st = (cudaStream_t)stream;
  if (fwd) return launch_pool2(POOL_MAX, reinterpret_cast<const bf16*>(x), N, H, W, C, reinterpret_cast<bf16*>(out), st);
  return launch_tap_bwd(reinterpret_cast<const bf16*>(x), nullptr, nullptr, nullptr, reinterpret_cast<const bf16*>(dy), N, H, W, C, 0,
                        reinterpret_cast<bf16*>(out), st);
}
