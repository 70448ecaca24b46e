// nhwc.cuh -- the layers LPIPS (lpips.cu), the ResNet towers (rn.cu) and the VQGAN decoder (vqgan.cu) share on bf16 NHWC
// activations: 8-channel bf16 vectors, the 2x2 window reduction and spread, and the 3-input-channel convolution that reads a
// caller's fp32 NCHW image (kernels and launchers in nhwc.cu). The 3x3 tensor-core convolution comes with it (conv_tc.cuh).
#pragma once
#include "conv_tc.cuh"

namespace aph {

// 8 bf16 <-> 8 fp32, one 16-byte vector (channel order)
__device__ __forceinline__ void unpack_bf16x8(const uint4& u, float* f) {
  const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
  for (int h = 0; h < 4; ++h) {
    const float2 v = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&w[h]));
    f[2 * h] = v.x; f[2 * h + 1] = v.y;
  }
}
__device__ __forceinline__ uint4 pack_bf16x8(const float* f) {
  return make_uint4(pack_bf16(f[0], f[1]), pack_bf16(f[2], f[3]), pack_bf16(f[4], f[5]), pack_bf16(f[6], f[7]));
}

// 2x2 window reductions, in (0,0) (0,1) (1,0) (1,1) order: the first maximum wins (as torch.max_pool2d); the fp32 sum times 0.25;
// the fp32 sum
enum : int { POOL_MAX = 0, POOL_MEAN = 1, POOL_SUM = 2 };
// x [N,H,W,C] -> out [N,H/2,W/2,C] (floor: an odd last row / column is dropped), bf16 NHWC, C % 8 == 0
int launch_pool2(int op, const bf16* x, int N, int H, int W, int C, bf16* out, cudaStream_t st);
// out [N,H,W,C] = scale dy [N,H/2,W/2,C] on each pixel of its window (zero on the rows / columns floor mode drops), selected by
// mask [N,H,W,C] > 0 when mask is not null
int launch_unpool2(const bf16* dy, const bf16* mask, int N, int H, int W, int C, float scale, bf16* out, cudaStream_t st);

// How the 3-input-channel convolution reads its image: as is (the ResNet stem), or as LPIPS's input scaling
// ((a x + b - shift) / scale; normalize: a, b = 2, -1, else 1, 0), whose gradient is then d x' a / scale
enum : int { IN_RAW = 0, IN_LPIPS = 1 };
// 3x3 convolution, pad 1, stride STRIDE, 3 -> COUT channels, fp32 SIMT, one thread per pixel. w fp32 [COUT][3][3][3], bias [COUT].
// Forward: img fp32 NCHW [N,3,H,W] -> out bf16 NHWC [N,Ho,Wo,64] = relu(conv + bias), Ho = (H - 1) / STRIDE + 1, channels
// COUT-63 zero. Backward: dz bf16 NHWC [N,Ho,Wo,64] (d pre-ReLU; channels below COUT read) -> grad fp32 NCHW [N,3,H,W], overwritten.
// Instances: <1, 64, IN_LPIPS> (LPIPS conv1_1) and <2, 32, IN_RAW> (the ResNet stem's conv1).
template <int STRIDE, int COUT, int IN>
int launch_conv3in_fwd(const float* img, int N, int H, int W, const float* w, const float* bias, bf16* out, cudaStream_t st,
                       float a = 1.f, float b = 0.f);
template <int STRIDE, int COUT, int IN>
int launch_conv3in_bwd(const bf16* dz, int N, int H, int W, const float* w, float* grad, cudaStream_t st, float a = 1.f);

}  // namespace aph
