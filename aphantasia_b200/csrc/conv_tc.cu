// conv_tc.cu -- launch_conv3x3: the k_conv3x3_tc instances (conv_tc.cuh) for every 3x3 convolution with C_in >= 64 of LPIPS, the
// ResNet towers and the VQGAN decoder. A module that holds these instances reserves 1 KB of static shared memory in every kernel
// it contains, so the element-wise NHWC kernels (nhwc.cu) live in a module of their own.
#include "conv_tc.cuh"

namespace aph {

template <int BN, int EPI>
static int conv_cfg(const void* x, const void* wpack, const ConvShape& cs, const ConvEpi& epi, cudaStream_t st) {
  using L = GemmCfg<BN>;
  static_assert(L::SMEM <= 227 * 1024, "conv shared-memory budget");
  if (int e = smem_at_least((const void*)k_conv3x3_tc<BN, EPI>, L::SMEM)) return e;
  CUtensorMap mx, mw;
  if (int e = make_tmap_bf16_nhwc(&mx, x, cs.N, cs.H, cs.W, cs.Cin, CONV_TH, CONV_TW)) return e;
  if (int e = make_tmap_bf16(&mw, wpack, cs.Cout, 9 * cs.Cin, BN)) return e;
  const int tiles = cs.N * cs.tiles_y * cs.tiles_x * (cs.Cout / BN);
  const int grid = tiles < num_sms() ? tiles : num_sms();
  k_conv3x3_tc<BN, EPI><<<grid, GEMM_THREADS, L::SMEM, st>>>(mx, mw, cs, epi);
  APH_LAUNCH_OK();
  return 0;
}

int launch_conv3x3(const void* x, const void* wpack, int N, int H, int W, int Cin, int Cout, int epi_kind, const ConvEpi& epi,
                   cudaStream_t st) {
  APH_REQUIRE(x && wpack && epi.out && N > 0 && H > 0 && W > 0, "conv3x3: null operand or empty shape");
  APH_REQUIRE(Cin % 64 == 0 && Cout % 64 == 0 && Cin > 0 && Cout > 0, "conv3x3: C_in=%d and C_out=%d must be multiples of 64", Cin, Cout);
  APH_REQUIRE((epi_kind != CONV_BIAS_RELU && epi_kind != CONV_BIAS && epi_kind != CONV_BIAS_RESID) || epi.bias,
              "conv3x3: the forward epilogues need a bias");
  APH_REQUIRE(epi_kind != CONV_BIAS_RESID || epi.resid, "conv3x3: the residual epilogue needs a residual");
  APH_REQUIRE(epi_kind != CONV_MASK || epi.mask, "conv3x3: the masked epilogue needs a mask");
  APH_REQUIRE(((reinterpret_cast<uintptr_t>(epi.out) | reinterpret_cast<uintptr_t>(epi.mask) | reinterpret_cast<uintptr_t>(epi.resid)) & 15) == 0,
              "conv3x3: output, mask and residual must be 16-byte aligned");
  const ConvShape cs{N, H, W, Cin, Cout, (H + CONV_TH - 1) / CONV_TH, (W + CONV_TW - 1) / CONV_TW};
  const bool wide = Cout % 128 == 0;
#define APH_CONV_CASE(K) case K: return wide ? conv_cfg<128, K>(x, wpack, cs, epi, st) : conv_cfg<64, K>(x, wpack, cs, epi, st);
  switch (epi_kind) {
    APH_CONV_CASE(CONV_BIAS_RELU) APH_CONV_CASE(CONV_MASK) APH_CONV_CASE(CONV_PLAIN) APH_CONV_CASE(CONV_BIAS) APH_CONV_CASE(CONV_BIAS_RESID)
  }
#undef APH_CONV_CASE
  set_error("conv3x3: unknown epilogue kind %d", epi_kind);
  return 2;
}

}  // namespace aph
