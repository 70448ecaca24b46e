// adam.cuh -- the one Adam / AdamW element update of libaphb200.so. aph_adam_step runs it over a gradient in memory; the
// generators' backwards (FFT column pass, DWT level adjoints, pixel normalisation adjoint) run it where the parameter's
// gradient is formed, so that gradient is never written and re-read.
// torch.optim.Adam / AdamW semantics and order (single-tensor path): decoupled decay p *= 1 - lr wd (AdamW), then
//   m = b1 m + (1 - b1) g,  v = b2 v + (1 - b2) g^2,  [AMSGrad: vmax = max(vmax, v), v -> vmax in the denominator]
//   p -= lr / (1 - b1^t) * m / (sqrt(v) / sqrt(1 - b2^t) + eps)
#pragma once
#include "aph_common.cuh"
#include <math.h>

namespace aph {

// p == nullptr: no update. vmax == nullptr: no AMSGrad. decay = 1 - lr * weight_decay (1 for Adam).
struct AdamArgs { float* p; float* m; float* v; float* vmax; float step_size, b1, b2, eps, inv_sqrt_bc2, decay; };

__device__ __forceinline__ void adam_elem(const AdamArgs& a, size_t i, float g) {
  float p = a.p[i];
  if (a.decay != 1.f) p = __fmul_rn(p, a.decay);         // its own rounding, as torch's separate mul_ (never fused into the update)
  const float m = a.b1 * a.m[i] + (1.f - a.b1) * g;
  float v = a.b2 * a.v[i] + (1.f - a.b2) * g * g;
  a.m[i] = m; a.v[i] = v;
  if (a.vmax) { v = fmaxf(a.vmax[i], v); a.vmax[i] = v; }
  a.p[i] = p - a.step_size * m / (sqrtf(v) * a.inv_sqrt_bc2 + a.eps);
}

// The launch constants of one step t >= 1 (bias corrections in fp64 on the host, as torch computes them in Python floats).
static inline AdamArgs make_adam(float* p, float* m, float* v, float* vmax, float lr, float b1, float b2, float eps,
                                 float weight_decay, int step) {
  const double bc1 = 1.0 - pow((double)b1, step), bc2 = 1.0 - pow((double)b2, step);
  AdamArgs a;
  a.p = p; a.m = m; a.v = v; a.vmax = vmax;
  a.step_size = (float)(lr / bc1); a.b1 = b1; a.b2 = b2; a.eps = eps; a.inv_sqrt_bc2 = (float)(1.0 / sqrt(bc2));
  a.decay = (float)(1.0 - (double)lr * weight_decay);
  return a;
}

}  // namespace aph
