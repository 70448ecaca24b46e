// synth_fft.cu -- spectrum -> RGB synthesis and its backward (HBM/L2-bound; fp32).
//
// Replaces /root/reference/aphantasia/image.py:164-175 (fft_image.inner) fused with
// image.py:21-28 (to_valid_rgb.inner):
//     Z = scale * (P [+ shift]);  x = irfftn(Z, s=(H,W), norm='ortho');  img = x*contrast/std(x)
//     out = sigmoid(Mn . img)
// Semantics of the C2R transform (SURVEY.md A1): full complex inverse DFT along H first, then the
// half-spectrum inverse along W that drops Im of columns 0 and W/2.
//
// Kernels (all mixed-radix Stockham FFTs staged in shared memory, radices {2,3,4,5,7,11,13}):
//   k_col_fft   : one CTA = C adjacent spectrum columns of one channel, length-H complex DFT.
//                 fwd: loads scale*(P+shift) (C*8 B contiguous segments), writes T[ch][n1][k2].
//                 bwd: loads dT, forward DFT, writes dP = scale * dZ.
//   k_row_c2r   : one CTA = a few row PAIRS; two real rows are recovered from ONE complex length-W
//                 inverse DFT (z = a + i b); writes x_raw and accumulates sum x, sum x^2 (fp64).
//   k_finish<true> / k_finish_bwd (synth_common.cuh): the pointwise tail, out = sigmoid(Mn . (x*contrast/sigma)) and
//                 g_img = Mn^T . (g*out*(1-out)); accumulates sum g_img.x
//   k_row_r2c   : g_x = (c/sigma)(g_img - (x-mu) * dot/((N-1) sigma^2)) formed on load; two real rows
//                 per complex forward DFT; interior columns x2; writes dT.
//   k_row_rfft  : analysis row pass (image-file resume): plain load of the image, two real rows per complex forward DFT,
//                 writes T; k_col_fft<false> then finishes rfftn and multiplies by the analysis scale.
//   k_un_rgb    : uint8 HWC picture -> planar fp32 through the inverse colour matrix (un_rgb).
#include "synth_common.cuh"
#include <vector>
#include <algorithm>

namespace aph {

constexpr int kMaxStages = 16;
struct Radices { int n; int r[kMaxStages]; };

struct FftPlanImpl : DeviceAllocs {
  int H, W, Wh;
  Radices rh, rw;
  float2* twH = nullptr;   // exp(+2 pi i k / H), k in [0,H)
  float2* twW = nullptr;
  float2* T = nullptr;     // [3][H][Wh] complex scratch (column-transformed spectrum / its gradient)
  float*  gimg = nullptr;  // [3][H][W] scratch (dL/d img)
  int colC;                // columns per CTA in the column pass
  bool colSingle = false;  // single-buffer / in-register-stage column kernel (long columns)
  int rowP;                // row pairs per CTA in the row pass
  size_t smem_col, smem_row;
};

static bool factorize(int n, Radices& out) {
  out.n = 0;
  const int cand[] = {4, 2, 3, 5, 7, 11, 13};
  for (int c : cand) {
    while (n % c == 0) {
      if (out.n >= kMaxStages) return false;
      out.r[out.n++] = c; n /= c;
    }
  }
  return n == 1;
}

__device__ __forceinline__ float2 cmul(float2 a, float2 b) {
  return make_float2(a.x * b.x - a.y * b.y, a.x * b.y + a.y * b.x);
}

// One Stockham stage of radix R over `lines` lines of length N stored with stride LS (float2 elements).
// tw[k] = exp(+2 pi i k / N); CONJ selects the forward (sign -) transform.
template <int R, bool CONJ>
__device__ __forceinline__ void fft_stage(const float2* __restrict__ in, float2* __restrict__ out,
                                          const float2* __restrict__ tw, int N, int Ns, int lines, int LS) {
  const int nb = N / R;               // butterflies per line
  const int tstride = N / (Ns * R);   // twiddle index stride
  const int rstride = N / R;          // small-DFT twiddle stride
  for (int idx = threadIdx.x; idx < lines * nb; idx += blockDim.x) {
    const int line = idx / nb, j = idx - line * nb;
    const int k = j % Ns;
    const float2* src = in + line * LS;
    float2* dst = out + line * LS + (j - k) * R + k;
    float2 v[R];
#pragma unroll
    for (int r = 0; r < R; ++r) {
      float2 x = src[j + r * nb];
      if (r > 0) {
        float2 w = tw[r * k * tstride];
        if (CONJ) w.y = -w.y;
        x = cmul(x, w);
      }
      v[r] = x;
    }
    if (R == 2) {
      dst[0] = make_float2(v[0].x + v[1].x, v[0].y + v[1].y);
      dst[Ns] = make_float2(v[0].x - v[1].x, v[0].y - v[1].y);
    } else if (R == 4) {
      // inverse (sign +): multiply by +i ; forward: -i
      float2 a = make_float2(v[0].x + v[2].x, v[0].y + v[2].y);
      float2 b = make_float2(v[0].x - v[2].x, v[0].y - v[2].y);
      float2 c = make_float2(v[1].x + v[3].x, v[1].y + v[3].y);
      float2 d = make_float2(v[1].x - v[3].x, v[1].y - v[3].y);
      float2 id = CONJ ? make_float2(d.y, -d.x) : make_float2(-d.y, d.x);   // (+-i) * d
      dst[0] = make_float2(a.x + c.x, a.y + c.y);
      dst[Ns] = make_float2(b.x + id.x, b.y + id.y);
      dst[2 * Ns] = make_float2(a.x - c.x, a.y - c.y);
      dst[3 * Ns] = make_float2(b.x - id.x, b.y - id.y);
    } else {
#pragma unroll
      for (int q = 0; q < R; ++q) {
        float2 acc = v[0];
#pragma unroll
        for (int r = 1; r < R; ++r) {
          float2 w = tw[((r * q) % R) * rstride];
          if (CONJ) w.y = -w.y;
          float2 t = cmul(v[r], w);
          acc.x += t.x; acc.y += t.y;
        }
        dst[q * Ns] = acc;
      }
    }
  }
}

// Runs all stages; data starts in `a`; returns pointer to the buffer holding the result.
template <bool CONJ>
__device__ float2* fft_lines(float2* a, float2* b, const float2* tw, int N, const Radices& rad, int lines, int LS) {
  int Ns = 1;
  for (int s = 0; s < rad.n; ++s) {
    const int R = rad.r[s];
    switch (R) {
      case 2: fft_stage<2, CONJ>(a, b, tw, N, Ns, lines, LS); break;
      case 3: fft_stage<3, CONJ>(a, b, tw, N, Ns, lines, LS); break;
      case 4: fft_stage<4, CONJ>(a, b, tw, N, Ns, lines, LS); break;
      case 5: fft_stage<5, CONJ>(a, b, tw, N, Ns, lines, LS); break;
      case 7: fft_stage<7, CONJ>(a, b, tw, N, Ns, lines, LS); break;
      case 11: fft_stage<11, CONJ>(a, b, tw, N, Ns, lines, LS); break;
      default: fft_stage<13, CONJ>(a, b, tw, N, Ns, lines, LS); break;
    }
    __syncthreads();
    Ns *= R;
    float2* t = a; a = b; b = t;
  }
  return a;
}

// Single-buffer variant for long columns (H > ~750: 4K canvases). A Stockham stage reads and writes different positions of the
// SAME buffer, so every thread first pulls ALL inputs of its butterflies into registers, the block synchronises, then the outputs
// are written: one buffer instead of two lets a CTA hold 8 columns of 2160 complex values (64-byte global segments instead of the
// 16-byte ones the two-buffer kernel is reduced to at that length). Requires lines * N / R <= (36 / R) * blockDim butterflies per stage.
template <int R, bool CONJ>
__device__ __forceinline__ void fft_stage_inreg(float2* __restrict__ buf, const float2* __restrict__ tw, int N, int Ns, int lines, int LS) {
  constexpr int MAXB = 36 / R;
  const int nb = N / R, total = lines * nb;
  const int tstride = N / (Ns * R), rstride = N / R;
  float2 v[MAXB][R];
#pragma unroll
  for (int b = 0; b < MAXB; ++b) {
    const int idx = threadIdx.x + b * blockDim.x;
    if (idx < total) {
      const int line = idx / nb, j = idx - line * nb, k = j % Ns;
      const float2* src = buf + line * LS;
#pragma unroll
      for (int r = 0; r < R; ++r) {
        float2 x = src[j + r * nb];
        if (r > 0) { float2 w = tw[r * k * tstride]; if (CONJ) w.y = -w.y; x = cmul(x, w); }
        v[b][r] = x;
      }
    }
  }
  __syncthreads();
#pragma unroll
  for (int b = 0; b < MAXB; ++b) {
    const int idx = threadIdx.x + b * blockDim.x;
    if (idx < total) {
      const int line = idx / nb, j = idx - line * nb, k = j % Ns;
      float2* dst = buf + line * LS + (j - k) * R + k;
      if (R == 2) {
        dst[0] = make_float2(v[b][0].x + v[b][1].x, v[b][0].y + v[b][1].y);
        dst[Ns] = make_float2(v[b][0].x - v[b][1].x, v[b][0].y - v[b][1].y);
      } else if (R == 4) {
        const float2 a = make_float2(v[b][0].x + v[b][2].x, v[b][0].y + v[b][2].y), bb = make_float2(v[b][0].x - v[b][2].x, v[b][0].y - v[b][2].y);
        const float2 c = make_float2(v[b][1].x + v[b][3].x, v[b][1].y + v[b][3].y), d = make_float2(v[b][1].x - v[b][3].x, v[b][1].y - v[b][3].y);
        const float2 id = CONJ ? make_float2(d.y, -d.x) : make_float2(-d.y, d.x);
        dst[0] = make_float2(a.x + c.x, a.y + c.y); dst[Ns] = make_float2(bb.x + id.x, bb.y + id.y);
        dst[2 * Ns] = make_float2(a.x - c.x, a.y - c.y); dst[3 * Ns] = make_float2(bb.x - id.x, bb.y - id.y);
      } else {
#pragma unroll
        for (int q = 0; q < R; ++q) {
          float2 acc = v[b][0];
#pragma unroll
          for (int r = 1; r < R; ++r) {
            float2 w = tw[((r * q) % R) * rstride];
            if (CONJ) w.y = -w.y;
            const float2 t = cmul(v[b][r], w);
            acc.x += t.x; acc.y += t.y;
          }
          dst[q * Ns] = acc;
        }
      }
    }
  }
  __syncthreads();
}

template <bool CONJ>
__device__ void fft_lines_inreg(float2* buf, const float2* tw, int N, const Radices& rad, int lines, int LS) {
  int Ns = 1;
  for (int s = 0; s < rad.n; ++s) {
    const int R = rad.r[s];
    switch (R) {
      case 2: fft_stage_inreg<2, CONJ>(buf, tw, N, Ns, lines, LS); break;
      case 3: fft_stage_inreg<3, CONJ>(buf, tw, N, Ns, lines, LS); break;
      case 4: fft_stage_inreg<4, CONJ>(buf, tw, N, Ns, lines, LS); break;
      default: fft_stage_inreg<5, CONJ>(buf, tw, N, Ns, lines, LS); break;      // the plan only selects this kernel for 2-3-5-smooth H
    }
    Ns *= R;
  }
}

// ---------------------------------------------------------------------------------------------
// Column pass. FWD: in = params [3][H][Wh] complex (+scale, +shift), out = T. !FWD: in = dT, out = dP*scale.
// Adam state for the fused update (row f2 of SURVEY 8f): the backward's last pass already holds dP = scale * dZ in registers,
// so p / m / v are updated right there instead of writing dP, re-reading it in torch.optim.Adam's ~12 launches.
struct AdamArgs { float2* p; float2* m; float2* v; float step_size, b1, b2, eps, inv_sqrt_bc2; int on; };

__device__ __forceinline__ float adam_elem(float& p, float& m, float& v, float g, const AdamArgs& a) {
  m = a.b1 * m + (1.f - a.b1) * g;
  v = a.b2 * v + (1.f - a.b2) * g * g;
  p -= a.step_size * m / (sqrtf(v) * a.inv_sqrt_bc2 + a.eps);
  return p;
}

template <bool FWD, bool SINGLE = false>
__global__ void __launch_bounds__(SINGLE ? 512 : 256, SINGLE ? 1 : 2) k_col_fft(const float2* __restrict__ in, float2* __restrict__ out,
                                                 const float* __restrict__ scale, const float* __restrict__ shift,
                                                 int shift_mode, const float2* __restrict__ twg, int H, int Wh, int C,
                                                 Radices rad, AdamArgs adam) {
  extern __shared__ float2 smem[];
  const int LS = H + 1;
  float2* tw = smem;                 // [H]
  float2* bufA = tw + H;             // [C][LS]
  float2* bufB = bufA + C * LS;      // (unused by the single-buffer variant)
  const int tiles = (Wh + C - 1) / C;
  const int ch = blockIdx.x / tiles, k2base = (blockIdx.x % tiles) * C;
  const int cols = min(C, Wh - k2base);
  for (int i = threadIdx.x; i < H; i += blockDim.x) tw[i] = twg[i];
  const size_t plane = (size_t)H * Wh;
  for (int idx = threadIdx.x; idx < H * C; idx += blockDim.x) {
    const int k1 = idx / C, c = idx - k1 * C;
    float2 v = make_float2(0.f, 0.f);
    if (c < cols) {
      const size_t g = (size_t)k1 * Wh + k2base + c;
      v = in[ch * plane + g];
      if (FWD) {
        const float s = scale[g];
        float2 z = make_float2(s * v.x, s * v.y);
        if (shift_mode == 1) { const float sh = s * shift[g]; z.x += sh; z.y += sh; }
        else if (shift_mode == 2) { const float2 sh = reinterpret_cast<const float2*>(shift)[ch * plane + g]; z.x += s * sh.x; z.y += s * sh.y; }
        v = z;
      }
    }
    bufA[c * LS + k1] = v;
  }
  __syncthreads();
  float2* res = bufA;
  if (SINGLE) fft_lines_inreg<!FWD>(bufA, tw, H, rad, C, LS);
  else res = fft_lines<!FWD>(bufA, bufB, tw, H, rad, C, LS);
  for (int idx = threadIdx.x; idx < H * C; idx += blockDim.x) {
    const int n1 = idx / C, c = idx - n1 * C;
    if (c < cols) {
      const size_t g = (size_t)n1 * Wh + k2base + c;
      float2 v = res[c * LS + n1];
      if (!FWD) {
        const float s = scale[g]; v.x *= s; v.y *= s;
        if (adam.on) {
          float2 pp = adam.p[ch * plane + g], mm = adam.m[ch * plane + g], vv = adam.v[ch * plane + g];
          adam_elem(pp.x, mm.x, vv.x, v.x, adam); adam_elem(pp.y, mm.y, vv.y, v.y, adam);
          adam.p[ch * plane + g] = pp; adam.m[ch * plane + g] = mm; adam.v[ch * plane + g] = vv;
        }
      }
      if (out) out[ch * plane + g] = v;
    }
  }
}

// ---------------------------------------------------------------------------------------------
// Row pass, inverse: T [3][H][Wh] complex -> x_raw [3][H][W]; accumulates {sum x, sum x^2} in stats (fp64).
__global__ void __launch_bounds__(256) k_row_c2r(const float2* __restrict__ T, float* __restrict__ x_raw,
                                                 double* __restrict__ stats, const float2* __restrict__ twg,
                                                 int H, int W, int Wh, int P, float norm, Radices rad) {
  extern __shared__ float2 smem[];
  const int LS = W + 1;
  float2* tw = smem;
  float2* bufA = tw + W;
  float2* bufB = bufA + P * LS;
  const int pairs_per_ch = (H + 1) / 2;
  const int groups = (pairs_per_ch + P - 1) / P;
  const int ch = blockIdx.x / groups, pbase = (blockIdx.x % groups) * P;
  const int np = min(P, pairs_per_ch - pbase);
  for (int i = threadIdx.x; i < W; i += blockDim.x) tw[i] = twg[i];
  const bool even = (W % 2) == 0;
  for (int idx = threadIdx.x; idx < np * Wh; idx += blockDim.x) {
    const int p = idx / Wh, k = idx - p * Wh;
    const int r0 = 2 * (pbase + p), r1 = r0 + 1;
    float2 a = T[((size_t)ch * H + r0) * Wh + k];
    float2 b = (r1 < H) ? T[((size_t)ch * H + r1) * Wh + k] : make_float2(0.f, 0.f);
    const bool special = (k == 0) || (even && k == W / 2);
    if (special) { a.y = 0.f; b.y = 0.f; }       // C2R ignores Im of the DC / Nyquist columns
    float2* line = bufA + p * LS;
    line[k] = make_float2(a.x - b.y, a.y + b.x);                       // A + iB
    if (!special) line[W - k] = make_float2(a.x + b.y, b.x - a.y);     // conj(A) + i conj(B)
  }
  __syncthreads();
  float2* res = fft_lines<false>(bufA, bufB, tw, W, rad, np, LS);
  double s1 = 0., s2 = 0.;
  for (int idx = threadIdx.x; idx < np * W; idx += blockDim.x) {
    const int p = idx / W, n = idx - p * W;
    const int r0 = 2 * (pbase + p), r1 = r0 + 1;
    const float2 z = res[p * LS + n];
    const float a = z.x * norm, b = z.y * norm;
    x_raw[((size_t)ch * H + r0) * W + n] = a;
    s1 += a; s2 += (double)a * a;
    if (r1 < H) { x_raw[((size_t)ch * H + r1) * W + n] = b; s1 += b; s2 += (double)b * b; }
  }
  block_atomic_add_d({s1, s2}, stats);
}

// Row pass, forward (backward of the synthesis): builds g_x on load, writes dT [3][H][Wh] complex.
__global__ void __launch_bounds__(256) k_row_r2c(const float* __restrict__ gimg, const float* __restrict__ x_raw,
                                                 const double* __restrict__ stats, float2* __restrict__ dT,
                                                 const float2* __restrict__ twg, int H, int W, int Wh, int P,
                                                 float norm, float contrast, Radices rad) {
  extern __shared__ float2 smem[];
  const int LS = W + 1;
  float2* tw = smem;
  float2* bufA = tw + W;
  float2* bufB = bufA + P * LS;
  const int pairs_per_ch = (H + 1) / 2;
  const int groups = (pairs_per_ch + P - 1) / P;
  const int ch = blockIdx.x / groups, pbase = (blockIdx.x % groups) * P;
  const int np = min(P, pairs_per_ch - pbase);
  for (int i = threadIdx.x; i < W; i += blockDim.x) tw[i] = twg[i];
  const double Nn = 3.0 * H * W;
  const double mu = stats[0] / Nn;
  const double var = (stats[1] - stats[0] * stats[0] / Nn) / (Nn - 1.0);
  const float c_sig = (float)((double)contrast / sqrt(var));
  const float kk = (float)(stats[2] / ((Nn - 1.0) * var));      // dot / ((N-1) sigma^2)
  const float muf = (float)mu;
  for (int idx = threadIdx.x; idx < np * W; idx += blockDim.x) {
    const int p = idx / W, n = idx - p * W;
    const int r0 = 2 * (pbase + p), r1 = r0 + 1;
    const size_t i0 = ((size_t)ch * H + r0) * W + n;
    const float a = c_sig * (gimg[i0] - (x_raw[i0] - muf) * kk);
    float b = 0.f;
    if (r1 < H) { const size_t i1 = i0 + W; b = c_sig * (gimg[i1] - (x_raw[i1] - muf) * kk); }
    bufA[p * LS + n] = make_float2(a, b);
  }
  __syncthreads();
  float2* res = fft_lines<true>(bufA, bufB, tw, W, rad, np, LS);
  const bool even = (W % 2) == 0;
  for (int idx = threadIdx.x; idx < np * Wh; idx += blockDim.x) {
    const int p = idx / Wh, k = idx - p * Wh;
    const int r0 = 2 * (pbase + p), r1 = r0 + 1;
    const float2 z = res[p * LS + k];
    const float2 zc = res[p * LS + ((W - k) % W)];
    // A = (Z[k] + conj(Z[W-k]))/2 ; B = (Z[k] - conj(Z[W-k]))/(2i)
    const bool special = (k == 0) || (even && k == W / 2);
    const float f = (special ? 0.5f : 1.0f) * norm;               // interior columns are doubled
    float2 A = make_float2((z.x + zc.x) * f, (z.y - zc.y) * f);
    float2 B = make_float2((z.y + zc.y) * f, (zc.x - z.x) * f);
    dT[((size_t)ch * H + r0) * Wh + k] = A;
    if (r1 < H) dT[((size_t)ch * H + r1) * Wh + k] = B;
  }
}

// Row pass of the analysis rfftn(img, 'ortho'): the same two-rows-per-complex-DFT split as k_row_r2c, on a plain load of img
// [3][H][W] and without the adjoint's doubling of the interior columns: every column is A = (Z[k] + conj(Z[W-k])) / 2.
__global__ void __launch_bounds__(256) k_row_rfft(const float* __restrict__ img, float2* __restrict__ T, const float2* __restrict__ twg,
                                                  int H, int W, int Wh, int P, float norm, Radices rad) {
  extern __shared__ float2 smem[];
  const int LS = W + 1;
  float2* tw = smem;
  float2* bufA = tw + W;
  float2* bufB = bufA + P * LS;
  const int pairs_per_ch = (H + 1) / 2;
  const int groups = (pairs_per_ch + P - 1) / P;
  const int ch = blockIdx.x / groups, pbase = (blockIdx.x % groups) * P;
  const int np = min(P, pairs_per_ch - pbase);
  for (int i = threadIdx.x; i < W; i += blockDim.x) tw[i] = twg[i];
  for (int idx = threadIdx.x; idx < np * W; idx += blockDim.x) {
    const int p = idx / W, n = idx - p * W;
    const int r0 = 2 * (pbase + p), r1 = r0 + 1;
    const size_t i0 = ((size_t)ch * H + r0) * W + n;
    bufA[p * LS + n] = make_float2(img[i0], r1 < H ? img[i0 + W] : 0.f);
  }
  __syncthreads();
  float2* res = fft_lines<true>(bufA, bufB, tw, W, rad, np, LS);
  const float f = 0.5f * norm;
  for (int idx = threadIdx.x; idx < np * Wh; idx += blockDim.x) {
    const int p = idx / Wh, k = idx - p * Wh;
    const int r0 = 2 * (pbase + p), r1 = r0 + 1;
    const float2 z = res[p * LS + k];
    const float2 zc = res[p * LS + ((W - k) % W)];
    T[((size_t)ch * H + r0) * Wh + k] = make_float2((z.x + zc.x) * f, (z.y - zc.y) * f);
    if (r1 < H) T[((size_t)ch * H + r1) * Wh + k] = make_float2((z.y + zc.y) * f, (zc.x - z.x) * f);
  }
}

// un_rgb (aphantasia/image.py:185-197): uint8 HWC -> planar [3][H][W] = gain * Minv . ((x / 255 - mean) / std), in the
// reference's order of operations (divide, subtract, divide, 3x3 mix, gain).
__global__ void __launch_bounds__(256) k_un_rgb(const uint8_t* __restrict__ hwc, size_t hw, ColMat mi, float gain, float* __restrict__ out) {
  const float mean[3] = {0.48145466f, 0.4578275f, 0.40821073f}, std_[3] = {0.26862954f, 0.26130258f, 0.27577711f};
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < hw; i += (size_t)gridDim.x * blockDim.x) {
    float v[3];
#pragma unroll
    for (int c = 0; c < 3; ++c) v[c] = ((float)hwc[3 * i + c] / 255.f - mean[c]) / std_[c];
#pragma unroll
    for (int d = 0; d < 3; ++d) out[d * hw + i] = gain * (mi.m[3 * d] * v[0] + mi.m[3 * d + 1] * v[1] + mi.m[3 * d + 2] * v[2]);
  }
}

// ---------------------------------------------------------------------------------------------
}  // namespace aph

using namespace aph;

extern "C" int aph_fft_plan_create(aph_fft_plan** plan_out, int H, int W) {
  APH_REQUIRE(plan_out && H >= 2 && W >= 2, "aph_fft_plan_create: bad arguments H=%d W=%d", H, W);
  std::unique_ptr<FftPlanImpl> p(new FftPlanImpl());
  p->H = H; p->W = W; p->Wh = W / 2 + 1;
  APH_REQUIRE(factorize(H, p->rh) && factorize(W, p->rw), "aph_fft_plan_create: H=%d or W=%d has a prime factor > 13 (unsupported FFT length)",
              H, W);
  // tile sizes bounded by shared memory (<= ~100 KB so two CTAs fit per SM when possible, hard cap 200 KB)
  int C = 8;
  while (C > 1 && (size_t)(2 * C * (H + 1) + H) * sizeof(float2) > 100 * 1024) C >>= 1;
  p->colC = C;
  p->smem_col = (size_t)(2 * C * (H + 1) + H) * sizeof(float2);
  if (C < 8) {            // long columns: the single-buffer kernel keeps 8 columns (or as many as 48 values per thread allow) per CTA
    int C1 = 8;
    auto fits = [&](int c) {
      if ((size_t)(c * (H + 1) + H) * sizeof(float2) > 200 * 1024) return false;
      for (int i = 0; i < p->rh.n; ++i) { const int r = p->rh.r[i]; if (r > 5 || (long long)c * H / r > (long long)(36 / r) * 512) return false; }
      return true;
    };
    while (C1 > 1 && !fits(C1)) --C1;
    if (C1 > C) { p->colC = C1; p->colSingle = true; p->smem_col = (size_t)(C1 * (H + 1) + H) * sizeof(float2); }
  }
  int P = 2;
  while (P > 1 && (size_t)(2 * P * (W + 1) + W) * sizeof(float2) > 100 * 1024) P >>= 1;
  p->rowP = P;
  p->smem_row = (size_t)(2 * P * (W + 1) + W) * sizeof(float2);
  APH_REQUIRE(p->smem_col <= 220 * 1024 && p->smem_row <= 220 * 1024, "aph_fft_plan_create: H=%d W=%d exceeds the shared-memory FFT size", H, W);
  std::vector<float2> th(H), tw(W);
  for (int k = 0; k < H; ++k) { double a = 2.0 * M_PI * k / H; th[k] = make_float2((float)cos(a), (float)sin(a)); }
  for (int k = 0; k < W; ++k) { double a = 2.0 * M_PI * k / W; tw[k] = make_float2((float)cos(a), (float)sin(a)); }
  if (int e = p->alloc(&p->twH, H)) return e;
  if (int e = p->alloc(&p->twW, W)) return e;
  APH_CUDA_OK(cudaMemcpy(p->twH, th.data(), H * sizeof(float2), cudaMemcpyHostToDevice));
  APH_CUDA_OK(cudaMemcpy(p->twW, tw.data(), W * sizeof(float2), cudaMemcpyHostToDevice));
  if (int e = p->alloc(&p->T, (size_t)3 * H * p->Wh)) return e;
  if (int e = p->alloc(&p->gimg, (size_t)3 * H * W)) return e;
  if (p->colSingle) {
    if (int e = smem_at_least((const void*)k_col_fft<true, true>, p->smem_col)) return e;
    if (int e = smem_at_least((const void*)k_col_fft<false, true>, p->smem_col)) return e;
  } else {
    if (int e = smem_at_least((const void*)k_col_fft<true>, p->smem_col)) return e;
    if (int e = smem_at_least((const void*)k_col_fft<false>, p->smem_col)) return e;
  }
  for (const void* k : {(const void*)k_row_c2r, (const void*)k_row_r2c, (const void*)k_row_rfft})
    if (int e = smem_at_least(k, p->smem_row)) return e;
  *plan_out = reinterpret_cast<aph_fft_plan*>(p.release());
  return 0;
}

extern "C" int aph_fft_plan_destroy(aph_fft_plan* plan) {
  delete reinterpret_cast<FftPlanImpl*>(plan);
  return 0;
}

extern "C" int aph_synth_fft_fwd(aph_fft_plan* plan, const float* params, const float* scale, const float* shift,
                                 int shift_mode, float contrast, const float* colmat_host, int apply_sigmoid,
                                 float* x_raw, double* stats, float* out, void* stream) {
  APH_REQUIRE(plan && params && scale && x_raw && stats && out, "aph_synth_fft_fwd: null pointer");
  APH_REQUIRE(shift_mode == 0 || shift != nullptr, "aph_synth_fft_fwd: shift_mode=%d without shift", shift_mode);
  FftPlanImpl* p = reinterpret_cast<FftPlanImpl*>(plan);
  cudaStream_t st = (cudaStream_t)stream;
  const int H = p->H, W = p->W, Wh = p->Wh;
  APH_CUDA_OK(cudaMemsetAsync(stats, 0, 4 * sizeof(double), st));
  const int col_tiles = (Wh + p->colC - 1) / p->colC;
  if (p->colSingle) k_col_fft<true, true><<<3 * col_tiles, 512, p->smem_col, st>>>(reinterpret_cast<const float2*>(params), p->T, scale, shift,
                                                                                    shift_mode, p->twH, H, Wh, p->colC, p->rh, AdamArgs{});
  else k_col_fft<true><<<3 * col_tiles, 256, p->smem_col, st>>>(reinterpret_cast<const float2*>(params), p->T, scale, shift,
                                                               shift_mode, p->twH, H, Wh, p->colC, p->rh, AdamArgs{});
  APH_LAUNCH_OK();
  const int groups = ((H + 1) / 2 + p->rowP - 1) / p->rowP;
  const float norm = (float)(1.0 / sqrt((double)H * W));
  k_row_c2r<<<3 * groups, 256, p->smem_row, st>>>(p->T, x_raw, stats, p->twW, H, W, Wh, p->rowP, norm, p->rw);
  APH_LAUNCH_OK();
  const size_t hw = (size_t)H * W;
  const int blocks = stride_blocks(hw, 8);
  k_finish<true><<<blocks, 256, 0, st>>>(x_raw, stats, out, hw, contrast, make_colmat(colmat_host), apply_sigmoid);
  APH_LAUNCH_OK();
  return 0;
}

static int synth_fft_bwd_impl(aph_fft_plan* plan, const float* grad_out, const float* out, const float* x_raw,
                              double* stats, const float* scale, float contrast, const float* colmat_host,
                              int apply_sigmoid, float* grad_params, const AdamArgs& adam, void* stream) {
  APH_REQUIRE(plan && grad_out && x_raw && stats && scale && (grad_params || adam.on), "aph_synth_fft_bwd: null pointer");
  APH_REQUIRE(!apply_sigmoid || out, "aph_synth_fft_bwd: sigmoid backward needs the saved output");
  FftPlanImpl* p = reinterpret_cast<FftPlanImpl*>(plan);
  cudaStream_t st = (cudaStream_t)stream;
  const int H = p->H, W = p->W, Wh = p->Wh;
  const size_t hw = (size_t)H * W;
  APH_CUDA_OK(cudaMemsetAsync(stats + 2, 0, sizeof(double), st));
  const int blocks = stride_blocks(hw, 8);
  k_finish_bwd<<<blocks, 256, 0, st>>>(grad_out, out, x_raw, p->gimg, stats, hw, make_colmat(colmat_host), apply_sigmoid);
  APH_LAUNCH_OK();
  const int groups = ((H + 1) / 2 + p->rowP - 1) / p->rowP;
  const float norm = (float)(1.0 / sqrt((double)H * W));
  k_row_r2c<<<3 * groups, 256, p->smem_row, st>>>(p->gimg, x_raw, stats, p->T, p->twW, H, W, Wh, p->rowP, norm, contrast, p->rw);
  APH_LAUNCH_OK();
  const int col_tiles = (Wh + p->colC - 1) / p->colC;
  if (p->colSingle) k_col_fft<false, true><<<3 * col_tiles, 512, p->smem_col, st>>>(p->T, reinterpret_cast<float2*>(grad_params), scale, nullptr, 0,
                                                                                     p->twH, H, Wh, p->colC, p->rh, adam);
  else k_col_fft<false><<<3 * col_tiles, 256, p->smem_col, st>>>(p->T, reinterpret_cast<float2*>(grad_params), scale, nullptr, 0,
                                                                p->twH, H, Wh, p->colC, p->rh, adam);
  APH_LAUNCH_OK();
  return 0;
}

extern "C" int aph_synth_fft_bwd(aph_fft_plan* plan, const float* grad_out, const float* out, const float* x_raw,
                                 double* stats, const float* scale, float contrast, const float* colmat_host,
                                 int apply_sigmoid, float* grad_params, void* stream) {
  return synth_fft_bwd_impl(plan, grad_out, out, x_raw, stats, scale, contrast, colmat_host, apply_sigmoid, grad_params, AdamArgs{}, stream);
}

extern "C" int aph_synth_fft_bwd_adam(aph_fft_plan* plan, const float* grad_out, const float* out, const float* x_raw,
                                      double* stats, const float* scale, float contrast, const float* colmat_host,
                                      int apply_sigmoid, float* grad_params, float* params, float* m, float* v,
                                      float lr, float b1, float b2, float eps, int step, void* stream) {
  APH_REQUIRE(params && m && v && step >= 1, "aph_synth_fft_bwd_adam: bad Adam state");
  const double bc1 = 1.0 - pow((double)b1, step), bc2 = 1.0 - pow((double)b2, step);
  AdamArgs a;
  a.p = reinterpret_cast<float2*>(params); a.m = reinterpret_cast<float2*>(m); a.v = reinterpret_cast<float2*>(v);
  a.step_size = (float)(lr / bc1); a.b1 = b1; a.b2 = b2; a.eps = eps; a.inv_sqrt_bc2 = (float)(1.0 / sqrt(bc2)); a.on = 1;
  return synth_fft_bwd_impl(plan, grad_out, out, x_raw, stats, scale, contrast, colmat_host, apply_sigmoid, grad_params, a, stream);
}

// Analysis (image-file resume, aphantasia/image.py:208-220): spectrum [3,H,Wh,2] = ascale * rfftn(img [3,H,W], 'ortho'). The row
// pass writes the plan's T; the column pass is the synthesis backward's forward DFT, which already multiplies by a per-bin scale.
extern "C" int aph_fft_analyze(aph_fft_plan* plan, const float* img, const float* ascale, float* spectrum, void* stream) {
  APH_REQUIRE(plan && img && ascale && spectrum, "aph_fft_analyze: null pointer");
  FftPlanImpl* p = reinterpret_cast<FftPlanImpl*>(plan);
  cudaStream_t st = (cudaStream_t)stream;
  const int H = p->H, W = p->W, Wh = p->Wh;
  const int groups = ((H + 1) / 2 + p->rowP - 1) / p->rowP;
  const float norm = (float)(1.0 / sqrt((double)H * W));
  k_row_rfft<<<3 * groups, 256, p->smem_row, st>>>(img, p->T, p->twW, H, W, Wh, p->rowP, norm, p->rw);
  APH_LAUNCH_OK();
  const int col_tiles = (Wh + p->colC - 1) / p->colC;
  if (p->colSingle) k_col_fft<false, true><<<3 * col_tiles, 512, p->smem_col, st>>>(p->T, reinterpret_cast<float2*>(spectrum), ascale, nullptr, 0,
                                                                                     p->twH, H, Wh, p->colC, p->rh, AdamArgs{});
  else k_col_fft<false><<<3 * col_tiles, 256, p->smem_col, st>>>(p->T, reinterpret_cast<float2*>(spectrum), ascale, nullptr, 0,
                                                                p->twH, H, Wh, p->colC, p->rh, AdamArgs{});
  APH_LAUNCH_OK();
  return 0;
}

extern "C" int aph_un_rgb(const uint8_t* hwc, int H, int W, const float* inv_colmat_host, float gain, float* out, void* stream) {
  APH_REQUIRE(hwc && inv_colmat_host && out && H > 0 && W > 0, "aph_un_rgb: bad arguments");
  const size_t hw = (size_t)H * W;
  const int blocks = stride_blocks(hw, 8);
  k_un_rgb<<<blocks, 256, 0, (cudaStream_t)stream>>>(hwc, hw, make_colmat(inv_colmat_host), gain, out);
  APH_LAUNCH_OK();
  return 0;
}

extern "C" int aph_valid_rgb_fwd(const float* img, int64_t hw, const float* colmat_host, float* out, void* stream) {
  APH_REQUIRE(img && out && hw > 0, "aph_valid_rgb_fwd: bad arguments");
  const int blocks = stride_blocks((size_t)hw, 8);
  k_finish<false><<<blocks, 256, 0, (cudaStream_t)stream>>>(img, nullptr, out, (size_t)hw, 1.f, make_colmat(colmat_host), 1);
  APH_LAUNCH_OK();
  return 0;
}

extern "C" int aph_valid_rgb_bwd(const float* grad_out, const float* out, int64_t hw, const float* colmat_host,
                                 float* grad_img, void* stream) {
  APH_REQUIRE(grad_out && out && grad_img && hw > 0, "aph_valid_rgb_bwd: bad arguments");
  const int blocks = stride_blocks((size_t)hw, 8);
  k_finish_bwd<<<blocks, 256, 0, (cudaStream_t)stream>>>(grad_out, out, nullptr, grad_img, nullptr, (size_t)hw,
                                                         make_colmat(colmat_host), 1);
  APH_LAUNCH_OK();
  return 0;
}
