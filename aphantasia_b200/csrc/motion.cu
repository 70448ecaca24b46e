// motion.cu -- the per-frame camera motion of illustrip.py (forward only; fp32 data, fp64 coordinates).
//
// Replaces frame_transform's torchvision call (/root/reference/illustrip.py:136):
//     T.functional.affine(img, angle, shift, scale, shear, fill=0, interpolation=BILINEAR)
// which on a CUDA tensor is torchvision's tensor path: _gen_affine_grid (pixel-centre base grid, normalised by the
// image size), grid_sample(bilinear, padding 'zeros', align_corners=False) of the image with a ones-plane appended,
// and the fill blend out = sample(img) * sample(ones) + (1 - sample(ones)) * 0.
//
//   k_frame_affine : one thread per output pixel. The source point, the four taps and their weights are computed once
//                    and reused for every plane and for the mask (the ones-plane's sample = the sum of the in-frame
//                    weights); then out[p] = (sum of in-frame taps of plane p) * mask.
//
// Source point of output pixel (i, j), with the inverse matrix m of _get_inverse_affine_matrix:
//     x = j + 0.5 - W/2,  y = i + 0.5 - H/2   (the base grid)
//     ix = m0 x + m1 y + m2 + W/2 - 0.5,  iy = m3 x + m4 y + m5 + H/2 - 0.5   (grid_sample's unnormalisation)
// torchvision forms the same point in fp32 through the normalised grid (about 1e-4 pixel of rounding at 1280 columns). Here
// the point and its fractional offsets are formed in fp64 from the fp64 matrix and rounded once to fp32 weights, so the
// kernel sits within fp32 rounding of the exact transform.
#include "aph_common.cuh"
#include <algorithm>
#include <math.h>

namespace aph {

struct Affine2 { double a, b, c, d, e, f; };   // ix = a j + b i + c ;  iy = d j + e i + f  (pixel indices)

__global__ void __launch_bounds__(256) k_frame_affine(const float* __restrict__ in, int planes, int H, int W, Affine2 m,
                                                      float* __restrict__ out) {
  const size_t hw = (size_t)H * W;
  for (size_t pix = blockIdx.x * (size_t)blockDim.x + threadIdx.x; pix < hw; pix += (size_t)gridDim.x * blockDim.x) {
    const int i = (int)(pix / W), j = (int)(pix - (size_t)i * W);
    const double sx = m.a * j + m.b * i + m.c, sy = m.d * j + m.e * i + m.f;
    float wt[4] = {0.f, 0.f, 0.f, 0.f};
    size_t off[4] = {0, 0, 0, 0};
    unsigned inside = 0;                 // bit t: tap t lies in the frame (grid_sample reads it even at weight 0)
    float mask = 0.f;
    // a point at least one pixel outside the frame has no tap inside it (and may not fit an int)
    if (sx > -1.0 && sy > -1.0 && sx < (double)W && sy < (double)H) {
      const double x0d = floor(sx), y0d = floor(sy);
      const int x0 = (int)x0d, y0 = (int)y0d;
      // the fractional offsets are taken in fp64 and rounded once; the weights and sums are fp32, as in grid_sample
      const float fx1 = (float)(sx - x0d), fx0 = (float)((x0d + 1.0) - sx);
      const float fy1 = (float)(sy - y0d), fy0 = (float)((y0d + 1.0) - sy);
      // grid_sample's tap order and weights: nw, ne, sw, se
      const int tx[4] = {x0, x0 + 1, x0, x0 + 1}, ty[4] = {y0, y0, y0 + 1, y0 + 1};
      const float w4[4] = {fx0 * fy0, fx1 * fy0, fx0 * fy1, fx1 * fy1};
#pragma unroll
      for (int t = 0; t < 4; ++t) {
        if (tx[t] >= 0 && tx[t] < W && ty[t] >= 0 && ty[t] < H) {
          wt[t] = w4[t];
          off[t] = (size_t)ty[t] * W + tx[t];
          inside |= 1u << t;
          mask += w4[t];
        }
      }
    }
    for (int p = 0; p < planes; ++p) {
      const float* src = in + (size_t)p * hw;
      float v = 0.f;
#pragma unroll
      for (int t = 0; t < 4; ++t)
        if (inside & (1u << t)) v += __ldg(src + off[t]) * wt[t];
      out[(size_t)p * hw + pix] = v * mask;
    }
  }
}

}  // namespace aph

using namespace aph;

extern "C" int aph_affine_fwd(const float* in, int planes, int H, int W, const double* inv_matrix_host, float* out,
                              void* stream) {
  APH_REQUIRE(in && out && inv_matrix_host && planes > 0 && H > 0 && W > 0, "aph_affine_fwd: bad arguments");
  APH_REQUIRE(in != out, "aph_affine_fwd: the output must not alias the input");
  const double* t = inv_matrix_host;
  // fold the base grid's centring and grid_sample's unnormalisation into the matrix (see the header comment)
  const double cx = 0.5 - 0.5 * W, cy = 0.5 - 0.5 * H;
  Affine2 m;
  m.a = t[0]; m.b = t[1]; m.c = t[0] * cx + t[1] * cy + t[2] + 0.5 * W - 0.5;
  m.d = t[3]; m.e = t[4]; m.f = t[3] * cx + t[4] * cy + t[5] + 0.5 * H - 0.5;
  const size_t hw = (size_t)H * W;
  const int blocks = (int)std::min<size_t>((hw + 255) / 256, (size_t)num_sms() * 16);
  k_frame_affine<<<blocks, 256, 0, (cudaStream_t)stream>>>(in, planes, H, W, m, out);
  APH_LAUNCH_OK();
  return 0;
}
