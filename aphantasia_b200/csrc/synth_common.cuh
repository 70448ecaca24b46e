// synth_common.cuh -- the pointwise tail of every image generator (FFT, DWT, pixel) and of aph_valid_rgb_*: normalise by the
// global std, colour-decorrelate, sigmoid (to_valid_rgb, aphantasia/image.py:21-28 fused with image.py:68,174), and its adjoint.
//   k_finish<NORM> : out = sigmoid(Mn . (x * contrast / sigma)); without NORM, out = sigmoid(Mn . x) and stats is not read
//   k_finish_bwd   : g_img = Mn^T . (g * out * (1 - out)); accumulates sum g_img . x into stats[2]
//   k_norm_bwd     : g_x = adjoint of the normalisation, from stats (the FFT fuses it into its row pass, k_row_r2c)
#pragma once
#include "adam.cuh"
#include <math.h>

namespace aph {

struct ColMat { float m[9]; int use; };

template <bool NORM>
static __global__ void __launch_bounds__(256) k_finish(const float* __restrict__ x_raw, const double* __restrict__ stats,
                                                float* __restrict__ out, size_t hw, float contrast, ColMat cm, int sig) {
  float s = 1.f;
  if (NORM) {
    const double Nn = 3.0 * (double)hw;
    const double var = (stats[1] - stats[0] * stats[0] / Nn) / (Nn - 1.0);
    s = (float)((double)contrast / sqrt(var));
  }
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < hw; i += (size_t)gridDim.x * blockDim.x) {
    float a = x_raw[i], b = x_raw[hw + i], c = x_raw[2 * hw + i];
    if (NORM) { a *= s; b *= s; c *= s; }
    float o0 = a, o1 = b, o2 = c;
    if (cm.use) {
      o0 = cm.m[0] * a + cm.m[1] * b + cm.m[2] * c;
      o1 = cm.m[3] * a + cm.m[4] * b + cm.m[5] * c;
      o2 = cm.m[6] * a + cm.m[7] * b + cm.m[8] * c;
    }
    if (sig) { o0 = 1.f / (1.f + expf(-o0)); o1 = 1.f / (1.f + expf(-o1)); o2 = 1.f / (1.f + expf(-o2)); }
    out[i] = o0; out[hw + i] = o1; out[2 * hw + i] = o2;
  }
}

// g_img = Mn^T (g * out * (1-out)); optionally accumulates sum g_img * x into stats[2].
static __global__ void __launch_bounds__(256) k_finish_bwd(const float* __restrict__ g, const float* __restrict__ out,
                                                    const float* __restrict__ x_raw, float* __restrict__ gimg,
                                                    double* __restrict__ stats, size_t hw, ColMat cm, int sig) {
  double dot = 0.;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < hw; i += (size_t)gridDim.x * blockDim.x) {
    float g0 = g[i], g1 = g[hw + i], g2 = g[2 * hw + i];
    if (sig) {
      const float o0 = out[i], o1 = out[hw + i], o2 = out[2 * hw + i];
      g0 *= o0 * (1.f - o0); g1 *= o1 * (1.f - o1); g2 *= o2 * (1.f - o2);
    }
    float a = g0, b = g1, c = g2;
    if (cm.use) {
      a = cm.m[0] * g0 + cm.m[3] * g1 + cm.m[6] * g2;
      b = cm.m[1] * g0 + cm.m[4] * g1 + cm.m[7] * g2;
      c = cm.m[2] * g0 + cm.m[5] * g1 + cm.m[8] * g2;
    }
    gimg[i] = a; gimg[hw + i] = b; gimg[2 * hw + i] = c;
    if (x_raw) dot += (double)a * x_raw[i] + (double)b * x_raw[hw + i] + (double)c * x_raw[2 * hw + i];
  }
  if (x_raw) block_atomic_add_d({dot}, stats + 2);
}

// g_x = (c/sigma) (g_img - (x - mu) * dot / ((N-1) sigma^2))      (adjoint of img = x * c / std(x), SURVEY.md A1)
// With adam.p set, g_x updates that parameter instead of being written (adam.cuh); it may be x_raw itself (the pixel generator).
static __global__ void __launch_bounds__(256) k_norm_bwd(const float* gimg, const float* x_raw, const double* __restrict__ stats,
                                                  float* gx, size_t n, float contrast, AdamArgs adam) {   // gimg may alias gx
  const double Nn = (double)n;
  const double mu = stats[0] / Nn;
  const double var = (stats[1] - stats[0] * stats[0] / Nn) / (Nn - 1.0);
  const float c_sig = (float)((double)contrast / sqrt(var));
  const float kk = (float)(stats[2] / ((Nn - 1.0) * var));
  const float muf = (float)mu;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const float g = c_sig * (gimg[i] - (x_raw[i] - muf) * kk);
    if (adam.p) adam_elem(adam, i, g);
    else gx[i] = g;
  }
}

static inline ColMat make_colmat(const float* host) {
  ColMat cm; cm.use = host != nullptr;
  for (int i = 0; i < 9; ++i) cm.m[i] = host ? host[i] : 0.f;
  return cm;
}


}  // namespace aph
