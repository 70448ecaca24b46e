// nhwc.cu -- the shared bf16 NHWC layers of nhwc.cuh: 2x2 window reduction and spread, and the 3-input-channel convolution pair.
//
//   k_pool2<OP>         LPIPS max-pool (MAX), the ResNet average pool (MEAN), the VQGAN upsample's adjoint (SUM over the 2H x 2W map)
//   k_unpool2           the ResNet average pool's adjoint (scale 0.25, optional ReLU select), the VQGAN nearest x2 upsample (scale 1:
//                       bf16 -> fp32 -> x 1 -> bf16 returns every finite value unchanged)
//   k_conv3in_fwd/_bwd  LPIPS conv1_1 <1, 64, IN_LPIPS> and the ResNet stems' conv1 <2, COUT, IN_RAW> (COUT = width / 2: 32 RN50 /
//                       RN101, 40 RN50x4, 48 RN50x16, 56 for width 112, 64 RN50x64), fp32 SIMT; the output row is 64 channels wide, zero above COUT
// The 3x3 tensor-core convolution's launcher is in conv_tc.cu.
#include "nhwc.cuh"

namespace aph {

// ---- 2x2 window reduction and spread: one thread per (pixel, 8 channels) ---------------------------------------------------
template <int OP>
__global__ void __launch_bounds__(256) k_pool2(const bf16* __restrict__ x, int N, int H, int W, int C, bf16* __restrict__ out) {
  const int Ho = H / 2, Wo = W / 2, C8 = C / 8;
  const size_t n_items = (size_t)N * Ho * Wo * C8;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n_items; i += (size_t)gridDim.x * blockDim.x) {
    const int cv = (int)(i % C8);
    const size_t po = i / C8;
    const int xo = (int)(po % Wo), yo = (int)((po / Wo) % Ho), n = (int)(po / ((size_t)Wo * Ho));
    const uint4* base = reinterpret_cast<const uint4*>(x + (((size_t)n * H + 2 * yo) * W + 2 * xo) * C) + cv;
    const size_t row = (size_t)W * C8, col = C8;
    float r[8], f[8];
    unpack_bf16x8(__ldg(base), r);
    const size_t offs[3] = {col, row, row + col};
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      unpack_bf16x8(__ldg(base + offs[k]), f);
#pragma unroll
      for (int j = 0; j < 8; ++j) r[j] = OP == POOL_MAX ? (f[j] > r[j] ? f[j] : r[j]) : r[j] + f[j];
    }
    if (OP == POOL_MEAN) {
#pragma unroll
      for (int j = 0; j < 8; ++j) r[j] *= 0.25f;
    }
    reinterpret_cast<uint4*>(out)[i] = pack_bf16x8(r);
  }
}

__global__ void __launch_bounds__(256) k_unpool2(const bf16* __restrict__ dy, const bf16* __restrict__ mask, int N, int H, int W, int C,
                                                 float scale, bf16* __restrict__ out) {
  const int Ho = H / 2, Wo = W / 2, C8 = C / 8;
  const size_t n_items = (size_t)N * H * W * C8;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n_items; i += (size_t)gridDim.x * blockDim.x) {
    const int cv = (int)(i % C8);
    const size_t p = i / C8;
    const int x = (int)(p % W), y = (int)((p / W) % H), n = (int)(p / ((size_t)W * H));
    float g[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    if (y < 2 * Ho && x < 2 * Wo) {
      unpack_bf16x8(__ldg(reinterpret_cast<const uint4*>(dy + (((size_t)n * Ho + y / 2) * Wo + x / 2) * C) + cv), g);
#pragma unroll
      for (int j = 0; j < 8; ++j) g[j] *= scale;
    }
    if (mask) {
      float m[8];
      unpack_bf16x8(__ldg(reinterpret_cast<const uint4*>(mask) + i), m);
#pragma unroll
      for (int j = 0; j < 8; ++j) g[j] = m[j] > 0.f ? g[j] : 0.f;
    }
    reinterpret_cast<uint4*>(out)[i] = pack_bf16x8(g);
  }
}

int launch_pool2(int op, const bf16* x, int N, int H, int W, int C, bf16* out, cudaStream_t st) {
  const int blocks = stride_blocks((size_t)N * (H / 2) * (W / 2) * (C / 8), 16);
  switch (op) {
    case POOL_MAX: k_pool2<POOL_MAX><<<blocks, 256, 0, st>>>(x, N, H, W, C, out); break;
    case POOL_MEAN: k_pool2<POOL_MEAN><<<blocks, 256, 0, st>>>(x, N, H, W, C, out); break;
    case POOL_SUM: k_pool2<POOL_SUM><<<blocks, 256, 0, st>>>(x, N, H, W, C, out); break;
    default: set_error("pool2: unknown op %d", op); return 2;
  }
  APH_LAUNCH_OK();
  return 0;
}

int launch_unpool2(const bf16* dy, const bf16* mask, int N, int H, int W, int C, float scale, bf16* out, cudaStream_t st) {
  k_unpool2<<<stride_blocks((size_t)N * H * W * (C / 8), 16), 256, 0, st>>>(dy, mask, N, H, W, C, scale, out);
  APH_LAUNCH_OK();
  return 0;
}

// ---- 3x3 convolution of a 3-channel fp32 NCHW image ----------------------------------------------------------------------------
// LPIPS's scaling layer (lpips v0.1)
__constant__ float c_lpips_shift[3] = {-.030f, -.088f, -.188f};
__constant__ float c_lpips_scale[3] = {.458f, .448f, .450f};

template <int IN>
__device__ __forceinline__ float conv3in_read(float v, float a, float b, int c) {
  return IN == IN_LPIPS ? (fmaf(a, v, b) - c_lpips_shift[c]) / c_lpips_scale[c] : v;
}

// One thread per output pixel: the 27 inputs in registers, then one fmaf chain of 27 taps per output channel.
template <int STRIDE, int COUT, int IN>
__global__ void __launch_bounds__(128) k_conv3in_fwd(const float* __restrict__ img, int N, int H, int W, float a, float b,
                                                     const float* __restrict__ w, const float* __restrict__ bias, bf16* __restrict__ out) {
  __shared__ float sw[COUT * 27], sb[COUT];
  for (int i = threadIdx.x; i < COUT * 27; i += blockDim.x) sw[i] = w[i];
  for (int i = threadIdx.x; i < COUT; i += blockDim.x) sb[i] = bias[i];
  __syncthreads();
  const int Ho = (H - 1) / STRIDE + 1, Wo = (W - 1) / STRIDE + 1;
  const size_t HWo = (size_t)Ho * Wo, plane = (size_t)H * W, p = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (p >= (size_t)N * HWo) return;
  const int n = (int)(p / HWo), rem = (int)(p - n * HWo), oy = rem / Wo, ox = rem - oy * Wo;
  float in[27];
#pragma unroll
  for (int c = 0; c < 3; ++c)
#pragma unroll
    for (int t = 0; t < 9; ++t) {
      const int y = STRIDE * oy + t / 3 - 1, x = STRIDE * ox + t % 3 - 1;
      in[c * 9 + t] = (y >= 0 && y < H && x >= 0 && x < W) ? conv3in_read<IN>(img[((size_t)n * 3 + c) * plane + (size_t)y * W + x], a, b, c)
                                                           : 0.f;
    }
  uint4* o = reinterpret_cast<uint4*>(out + p * 64);
#pragma unroll
  for (int g = 0; g < COUT / 8; ++g) {
    float acc[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float* wj = sw + (8 * g + j) * 27;
      float s = sb[8 * g + j];
#pragma unroll
      for (int k = 0; k < 27; ++k) s = fmaf(wj[k], in[k], s);
      acc[j] = fmaxf(s, 0.f);
    }
    o[g] = pack_bf16x8(acc);
  }
#pragma unroll
  for (int g = COUT / 8; g < 8; ++g) o[g] = make_uint4(0u, 0u, 0u, 0u);
}

// One thread per input pixel: output pixel (oy, ox) read it through tap (ky, kx) when STRIDE oy = y + 1 - ky and STRIDE ox = x + 1 - kx.
template <int STRIDE, int COUT, int IN>
__global__ void __launch_bounds__(128) k_conv3in_bwd(const bf16* __restrict__ dz, int N, int H, int W, float a, const float* __restrict__ w,
                                                     float* __restrict__ grad) {
  __shared__ float sw[COUT * 27];
  for (int i = threadIdx.x; i < COUT * 27; i += blockDim.x) sw[i] = w[i];
  __syncthreads();
  const int Ho = (H - 1) / STRIDE + 1, Wo = (W - 1) / STRIDE + 1;
  const size_t plane = (size_t)H * W, p = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (p >= (size_t)N * plane) return;
  const int n = (int)(p / plane), rem = (int)(p - n * plane), y = rem / W, x = rem - y * W;
  float g[3] = {0.f, 0.f, 0.f};
  for (int ky = 0; ky < 3; ++ky) {
    const int ty = y + 1 - ky;
    if (ty < 0 || ty % STRIDE || ty / STRIDE >= Ho) continue;
    for (int kx = 0; kx < 3; ++kx) {
      const int tx = x + 1 - kx;
      if (tx < 0 || tx % STRIDE || tx / STRIDE >= Wo) continue;
      const int t = ky * 3 + kx;
      const uint4* src = reinterpret_cast<const uint4*>(dz + (((size_t)n * Ho + ty / STRIDE) * Wo + tx / STRIDE) * 64);
#pragma unroll
      for (int v = 0; v < COUT / 8; ++v) {
        float f[8];
        unpack_bf16x8(__ldg(src + v), f);
#pragma unroll
        for (int j = 0; j < 8; j += 2) {
          const int co = 8 * v + j;
#pragma unroll
          for (int c = 0; c < 3; ++c) g[c] = fmaf(f[j], sw[co * 27 + c * 9 + t], fmaf(f[j + 1], sw[(co + 1) * 27 + c * 9 + t], g[c]));
        }
      }
    }
  }
#pragma unroll
  for (int c = 0; c < 3; ++c) grad[((size_t)n * 3 + c) * plane + rem] = IN == IN_LPIPS ? g[c] * a / c_lpips_scale[c] : g[c];
}

template <int STRIDE, int COUT, int IN>
int launch_conv3in_fwd(const float* img, int N, int H, int W, const float* w, const float* bias, bf16* out, cudaStream_t st, float a,
                       float b) {
  const size_t n = (size_t)N * ((H - 1) / STRIDE + 1) * ((W - 1) / STRIDE + 1);
  k_conv3in_fwd<STRIDE, COUT, IN><<<(unsigned)((n + 127) / 128), 128, 0, st>>>(img, N, H, W, a, b, w, bias, out);
  APH_LAUNCH_OK();
  return 0;
}

template <int STRIDE, int COUT, int IN>
int launch_conv3in_bwd(const bf16* dz, int N, int H, int W, const float* w, float* grad, cudaStream_t st, float a) {
  const size_t n = (size_t)N * H * W;
  k_conv3in_bwd<STRIDE, COUT, IN><<<(unsigned)((n + 127) / 128), 128, 0, st>>>(dz, N, H, W, a, w, grad);
  APH_LAUNCH_OK();
  return 0;
}

template int launch_conv3in_fwd<1, 64, IN_LPIPS>(const float*, int, int, int, const float*, const float*, bf16*, cudaStream_t, float, float);
template int launch_conv3in_bwd<1, 64, IN_LPIPS>(const bf16*, int, int, int, const float*, float*, cudaStream_t, float);
#define APH_STEM_INSTANCES(COUT)                                                                                                   \
  template int launch_conv3in_fwd<2, COUT, IN_RAW>(const float*, int, int, int, const float*, const float*, bf16*, cudaStream_t, float, \
                                                   float);                                                                        \
  template int launch_conv3in_bwd<2, COUT, IN_RAW>(const bf16*, int, int, int, const float*, float*, cudaStream_t, float);
APH_STEM_INSTANCES(32) APH_STEM_INSTANCES(40) APH_STEM_INSTANCES(48) APH_STEM_INSTANCES(56) APH_STEM_INSTANCES(64)
#undef APH_STEM_INSTANCES

}  // namespace aph
