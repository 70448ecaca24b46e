// vit_gemm.cu -- host side of the wgmma GEMM (tensor-map encoding, launch) + the exported test entry.
#include "tc_gemm.cuh"
#include <algorithm>
#include <atomic>
#include <initializer_list>
#include <string>
#include <vector>
#include <utility>

namespace aph {

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

// Encodes the tensor map of a bf16 tensor (or of the 16-bit view of an fp32 one) with the 128-byte swizzle the kernels' shared-memory
// tiles assume. Dimensions and box are innermost first; `strides` are the byte strides of the outer dimensions. Boxes that reach
// past the tensor's bounds arrive zero-filled.
static int encode_tmap(CUtensorMap* out, const void* base, std::initializer_list<int64_t> dims, std::initializer_list<int64_t> strides,
                       std::initializer_list<int> box) {
  static const EncodeTiledFn enc = [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    const bool ok = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess;
    return ok ? reinterpret_cast<EncodeTiledFn>(p) : nullptr;
  }();
  APH_REQUIRE(enc != nullptr, "cuTensorMapEncodeTiled not available from the driver");
  const int rank = (int)dims.size();
  cuuint64_t gdim[5], gstride[4];
  cuuint32_t gbox[5];
  const cuuint32_t estr[5] = {1, 1, 1, 1, 1};
  std::copy(dims.begin(), dims.end(), gdim);
  std::copy(strides.begin(), strides.end(), gstride);
  std::copy(box.begin(), box.end(), gbox);
  auto shape = [&] {                 // "tensor [S x T x cols], box [1 x 64 x 64]": outermost first
    std::string s = "tensor [";
    for (int i = rank - 1; i >= 0; --i) s += std::to_string(gdim[i]) + (i ? " x " : "], box [");
    for (int i = rank - 1; i >= 0; --i) s += std::to_string(gbox[i]) + (i ? " x " : "]");
    return s;
  };
  bool aligned = (reinterpret_cast<uintptr_t>(base) & 15) == 0;
  for (int i = 0; i < rank - 1; ++i) aligned = aligned && gstride[i] % 16 == 0;
  APH_REQUIRE(aligned, "tensor map of %s: base or stride not 16-byte aligned", shape().c_str());
  const CUresult r = enc(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, rank, const_cast<void*>(base), gdim, gstride, gbox, estr,
                         CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                         CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  APH_REQUIRE(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled failed: CUresult %d (%s)", (int)r, shape().c_str());
  return 0;
}

int make_tmap_bf16(CUtensorMap* out, const void* base, int rows, int K, int box_rows, int64_t row_stride) {
  if (row_stride == 0) row_stride = K;
  APH_REQUIRE(row_stride >= K, "tensor map: row stride %lld < K=%d", (long long)row_stride, K);
  return encode_tmap(out, base, {K, rows}, {row_stride * 2}, {GEMM_BK, box_rows});
}

// 3-D view [S][T][cols] of a token-major bf16 matrix [S*T, cols]: a box of `box_rows` tokens x 64 columns of ONE sample; rows past T
// are out of bounds in the T dimension and arrive zero-filled (the attention kernels rely on that for their padded tiles).
int make_tmap_bf16_tokens(CUtensorMap* out, const void* base, int cols, int T, int S, int box_rows) {
  return encode_tmap(out, base, {cols, T, S}, {(int64_t)cols * 2, (int64_t)T * cols * 2}, {64, box_rows, 1});
}

// 4-D view of an NHWC activation for the 3x3 convolution (conv_tc.cuh): the producer loads the box at coordinates shifted by the
// tap's (dy, dx), and the rows / columns outside the image arrive zero-filled, which is the convolution's padding 1.
int make_tmap_bf16_nhwc(CUtensorMap* out, const void* base, int N, int H, int W, int C, int box_h, int box_w) {
  return encode_tmap(out, base, {C, W, H, N}, {(int64_t)C * 2, (int64_t)W * C * 2, (int64_t)H * W * C * 2}, {64, box_w, box_h, 1});
}

// ---- optional per-launch event timing (bench.py's roofline: the GEMM kernel's real time inside a step)
static bool g_prof = false;
bool gemm_profiling_on() { return g_prof; }
static std::vector<std::pair<cudaEvent_t, cudaEvent_t>> g_prof_ev;
static std::vector<double> g_prof_flops;

// launches per (kernel variant, epilogue kind): variant 0 = the small-problem kernels (cooperative, 128 x 128 tiles, or 128 x 64
// where N % 128 == 64),
// 1 = the large-problem kernels (ping-pong 128 x 128 tiles, or cooperative 128 x 256 tiles for long K).
// Read by the tests to prove which kernel a shape really ran (aph_gemm_variant_launches).
static std::atomic<long long> g_variant_launches[2][EPI_KINDS];

template <int BN, bool PINGPONG, int EPI>
static int launch_cfg(const void* A, const void* B, GemmShape shp, const GemmEpi& epi, cudaStream_t st, int lda) {
  using L = GemmCfg<BN>;
  static_assert(L::SMEM <= 227 * 1024, "GEMM shared-memory budget");
  g_variant_launches[(PINGPONG || BN == 256) ? 1 : 0][EPI].fetch_add(1, std::memory_order_relaxed);
  if (int e = smem_at_least((const void*)k_gemm_bf16_tn<BN, PINGPONG, EPI>, L::SMEM)) return e;
  CUtensorMap ma, mb;
  if (int e = make_tmap_bf16(&ma, A, shp.M, shp.K, GEMM_BM, lda)) return e;
  if (int e = make_tmap_bf16(&mb, B, shp.N, shp.K, BN)) return e;
  const int tiles = ((shp.M + GEMM_BM - 1) / GEMM_BM) * (shp.N / BN);
  const int grid = tiles < num_sms() ? tiles : num_sms();
  cudaEvent_t e0 = nullptr, e1 = nullptr;
  if (g_prof) { cudaEventCreate(&e0); cudaEventCreate(&e1); cudaEventRecord(e0, st); }
  k_gemm_bf16_tn<BN, PINGPONG, EPI><<<grid, GEMM_THREADS, (size_t)L::SMEM, st>>>(ma, mb, shp, epi);
  APH_LAUNCH_OK();
  if (g_prof) { cudaEventRecord(e1, st); g_prof_ev.emplace_back(e0, e1); g_prof_flops.push_back(2.0 * shp.M * shp.N * shp.K); }
  return 0;
}

int launch_gemm(const void* A, const void* B, GemmShape shp, const GemmEpi& epi_in, cudaStream_t st, int lda) {
  APH_REQUIRE(A && B && shp.M > 0, "gemm: null operand or empty M");
  APH_REQUIRE(shp.K % GEMM_BK == 0 && shp.K > 0, "gemm: K=%d must be a positive multiple of %d", shp.K, GEMM_BK);
  APH_REQUIRE(shp.N % 64 == 0 && shp.N > 0, "gemm: N=%d must be a positive multiple of 64", shp.N);
  APH_REQUIRE(lda == 0 || lda >= shp.K, "gemm: lda=%d < K=%d", lda, shp.K);
  APH_REQUIRE((epi_in.ld_out == 0 || epi_in.ld_out >= shp.N) && (epi_in.ld_resid == 0 || epi_in.ld_resid >= shp.N),
              "gemm: output / residual row stride below N=%d", shp.N);
  GemmEpi epi = epi_in;                       // the kernel reads resolved strides
  if (epi.ld_out == 0) epi.ld_out = shp.N;
  if (epi.ld_resid == 0) epi.ld_resid = shp.N;
  // map the requested fusion onto one of the compiled epilogue kinds
  int kind = -1;
  const bool b = epi.bias, r = epi.resid, gi = epi.gelu_in, f = epi.out_f32, h = epi.out_bf16, pre = epi.out_pre, act = epi.act == 1, un = epi.unpatch_p > 0;
  const bool rb = epi.resid_bf16, mk = epi.mask, relu = epi.act == 2;
  APH_REQUIRE(!un || epi.ld_out == shp.N, "gemm: the un-patchify store takes no output stride");
  if (rb || mk || relu) {                     // the ResNet kinds: bf16 out, no other operand
    if (h && !f && !r && !gi && !pre && !un) {
      if (b && relu && !mk) kind = rb ? EPI_BIAS_RESID_RELU : EPI_BIAS_RELU;
      else if (!b && !relu && mk) kind = rb ? EPI_MASK_RESID : EPI_MASK;
    }
  }
  else if (un && f && !b && !r && !gi && !h && !pre && !act) kind = EPI_UNPATCH;
  else if (f && !h && !b && !r && !gi && !pre && !act) kind = EPI_F32;
  else if (h && !f && !b && !r && !gi && !pre && !act) kind = EPI_BF16;
  else if (h && !f && b && !r && !gi && !pre && !act) kind = EPI_BIAS_BF16;
  else if (h && !f && b && !r && !gi && pre && act) kind = EPI_BIAS_GELU;
  else if (f && !h && b && r && !gi && !pre && !act) kind = EPI_BIAS_RESID;
  else if (h && !f && !b && !r && gi && !pre && !act) kind = EPI_GELUGRAD_BF16;
  APH_REQUIRE(kind >= 0, "gemm: unsupported epilogue combination");
  const uintptr_t bf16_ptrs = reinterpret_cast<uintptr_t>(epi.out_bf16) | reinterpret_cast<uintptr_t>(epi.out_pre) | reinterpret_cast<uintptr_t>(epi.gelu_in) |
                              reinterpret_cast<uintptr_t>(epi.resid_bf16) | reinterpret_cast<uintptr_t>(epi.mask);
  APH_REQUIRE((bf16_ptrs & 15) == 0 && ((size_t)epi.ld_out * (f ? 4 : 2)) % 16 == 0 && ((size_t)epi.ld_resid * 4) % 16 == 0 &&
              ((size_t)lda * 2) % 16 == 0,
              "gemm: bf16 epilogue operands and row strides must be 16-byte aligned (8 columns are stored per lane)");
  // The ping-pong kernel overlaps one consumer's epilogue with the other's mainloop, which needs two tiles per SM in flight. It is
  // chosen when there are at least twice as many 128 x 128 tiles as SMs and K is short (K = 768 in the encoder), so that the
  // epilogue is a large share of a tile's time. With long K the mainloop dominates and the cooperative 128 x 256 tile wins: its
  // m64n256 MMAs read less shared memory per FLOP. Smaller problems (the final projection, the text tower) keep 128 x 128 tiles.
  // N % 128 == 64 (RN50's first stage at N = 64, the wide towers' zero-padded widths 192 and 320 and their multiples) runs the
  // small-problem schedule on 128 x 64 tiles, the tile the 3x3 convolution uses for those widths.
  const int m_tiles = (shp.M + GEMM_BM - 1) / GEMM_BM;
  const bool narrow = shp.N % 128 == 64;
  const bool pingpong = !narrow && m_tiles * (shp.N / 128) >= 2 * num_sms() && shp.K <= 1024;
  const bool wide = !pingpong && shp.N % 256 == 0 && m_tiles * (shp.N / 256) >= num_sms();
#define APH_GEMM_CASE(K) case K: return pingpong ? launch_cfg<128, true, K>(A, B, shp, epi, st, lda) \
                                                 : wide ? launch_cfg<256, false, K>(A, B, shp, epi, st, lda) : launch_cfg<128, false, K>(A, B, shp, epi, st, lda);
#define APH_GEMM_CASE_RN(K) case K: return narrow ? launch_cfg<64, false, K>(A, B, shp, epi, st, lda) : pingpong ? launch_cfg<128, true, K>(A, B, shp, epi, st, lda) \
                                                 : wide ? launch_cfg<256, false, K>(A, B, shp, epi, st, lda) : launch_cfg<128, false, K>(A, B, shp, epi, st, lda);
  APH_REQUIRE(!narrow || kind == EPI_BF16 || kind == EPI_BIAS_BF16 || kind >= EPI_BIAS_RELU,
              "gemm: N=%d (N %% 128 == 64) takes the bf16, bias-bf16 and ResNet epilogues only", shp.N);
  switch (kind) {
    APH_GEMM_CASE(EPI_F32) APH_GEMM_CASE_RN(EPI_BF16) APH_GEMM_CASE_RN(EPI_BIAS_BF16) APH_GEMM_CASE(EPI_BIAS_GELU)
    APH_GEMM_CASE(EPI_BIAS_RESID) APH_GEMM_CASE(EPI_GELUGRAD_BF16) APH_GEMM_CASE(EPI_UNPATCH)
    APH_GEMM_CASE_RN(EPI_BIAS_RELU) APH_GEMM_CASE_RN(EPI_BIAS_RESID_RELU) APH_GEMM_CASE_RN(EPI_MASK) APH_GEMM_CASE_RN(EPI_MASK_RESID)
  }
#undef APH_GEMM_CASE
#undef APH_GEMM_CASE_RN
  return 2;
}

}  // namespace aph

using namespace aph;

extern "C" int aph_gemm_bf16_tn(const void* A, const void* B, float* C, int M, int N, int K, void* stream) {
  APH_REQUIRE(C != nullptr, "aph_gemm_bf16_tn: null output");
  GemmEpi epi;
  epi.out_f32 = C;
  return launch_gemm(A, B, GemmShape{M, N, K}, epi, (cudaStream_t)stream);
}

// Test entry: the encoder's GEMM with any of its fused epilogues, on caller-supplied operands (tests/test_gpu_bench_config.py).
// Unused pointers are NULL; the combination selects the epilogue kind exactly as the encoder's own calls do.
extern "C" int aph_gemm_epi_test(const void* A, const void* B, int M, int N, int K, const float* bias, const float* resid,
                                 const void* gelu_in, int act, float* out_f32, void* out_bf16, void* out_pre,
                                 int unpatch_p, int unpatch_g, void* stream) {
  GemmEpi epi;
  epi.bias = bias; epi.resid = resid; epi.gelu_in = reinterpret_cast<const bf16*>(gelu_in); epi.act = act;
  epi.out_f32 = out_f32; epi.out_bf16 = reinterpret_cast<bf16*>(out_bf16); epi.out_pre = reinterpret_cast<bf16*>(out_pre);
  epi.unpatch_p = unpatch_p; epi.unpatch_g = unpatch_g;
  return launch_gemm(A, B, GemmShape{M, N, K}, epi, (cudaStream_t)stream);
}

// Same with row strides in elements (0 = dense) for A, the residual and the outputs (tests/test_vit_last_block_gpu.py).
extern "C" int aph_gemm_epi_strided_test(const void* A, int lda, const void* B, int M, int N, int K, const float* bias,
                                         const float* resid, int ld_resid, const void* gelu_in, int act, float* out_f32,
                                         void* out_bf16, void* out_pre, int ld_out, void* stream) {
  GemmEpi epi;
  epi.bias = bias; epi.resid = resid; epi.gelu_in = reinterpret_cast<const bf16*>(gelu_in); epi.act = act;
  epi.out_f32 = out_f32; epi.out_bf16 = reinterpret_cast<bf16*>(out_bf16); epi.out_pre = reinterpret_cast<bf16*>(out_pre);
  epi.ld_resid = ld_resid; epi.ld_out = ld_out;
  return launch_gemm(A, B, GemmShape{M, N, K}, epi, (cudaStream_t)stream, lda);
}

// The ResNet epilogues (rn.cu) on caller operands: relu = 1: out_bf16 = relu(acc + bias [+ resid_bf16]); relu = 0:
// out_bf16 = mask > 0 ? acc [+ resid_bf16] : 0. N a multiple of 64.
extern "C" int aph_gemm_rn_epi_test(const void* A, const void* B, int M, int N, int K, const float* bias, const void* resid_bf16,
                                    const void* mask, int relu, void* out_bf16, void* stream) {
  GemmEpi epi;
  epi.bias = bias; epi.resid_bf16 = reinterpret_cast<const bf16*>(resid_bf16); epi.mask = reinterpret_cast<const bf16*>(mask);
  epi.act = relu ? 2 : 0; epi.out_bf16 = reinterpret_cast<bf16*>(out_bf16);
  return launch_gemm(A, B, GemmShape{M, N, K}, epi, (cudaStream_t)stream);
}

// launches so far of kernel variant `variant` (0: the small-problem kernels, 1: the large-problem kernels) with
// epilogue kind `epi` (EPI_* order of tc_gemm.cuh: 0 f32, 1 bf16, 2 bias-bf16, 3 bias-gelu, 4 bias-resid, 5 gelugrad, 6 unpatch,
// 7 bias-relu, 8 bias-resid-relu, 9 mask, 10 mask-resid; -1 = all)
extern "C" int64_t aph_gemm_variant_launches(int variant, int epi) {
  if (variant < 0 || variant > 1 || epi >= EPI_KINDS) return -1;
  long long n = 0;
  for (int k = 0; k < EPI_KINDS; ++k) if (epi < 0 || epi == k) n += g_variant_launches[variant][k].load();
  return (int64_t)n;
}

// Profiling aid for bench.py: enable=1 starts recording a CUDA-event pair around every GEMM launch (on its stream);
// enable=0 stops, synchronises and returns the summed kernel time / FLOPs / launch count since it was enabled.
extern "C" int aph_prof_gemm(int enable, double* total_ms, double* total_flops, int* launches) {
  if (enable) { g_prof = true; g_prof_ev.clear(); g_prof_flops.clear(); return 0; }
  g_prof = false;
  double ms = 0., fl = 0.;
  for (size_t i = 0; i < g_prof_ev.size(); ++i) {
    APH_CUDA_OK(cudaEventSynchronize(g_prof_ev[i].second));
    float t = 0.f;
    APH_CUDA_OK(cudaEventElapsedTime(&t, g_prof_ev[i].first, g_prof_ev[i].second));
    ms += t; fl += g_prof_flops[i];
    cudaEventDestroy(g_prof_ev[i].first); cudaEventDestroy(g_prof_ev[i].second);
  }
  if (total_ms) *total_ms = ms;
  if (total_flops) *total_flops = fl;
  if (launches) *launches = (int)g_prof_ev.size();
  g_prof_ev.clear(); g_prof_flops.clear();
  return 0;
}
