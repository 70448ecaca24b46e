// rng_replay.cu -- HOST code: exact native replay of the reference's per-crop random draws.
//
// The reference draws its sampling / augmentation randomness per crop from torch's default CPU generator and NumPy's
// legacy global RandomState, in a data-dependent order (/root/reference/aphantasia/utils.py:244-247, torchvision
// RandomPerspective / RandomErasing get_params, /root/reference/aphantasia/transforms.py:75). Replaying that order with
// ~10 Python-level torch calls per crop costs tens of milliseconds per step -- more than the whole GPU step. This file
// continues both Mersenne-Twister streams natively, bit-exactly (same tempering, same reload, same draw->value
// transformations as ATen's CPUGeneratorImpl and NumPy's legacy bounded integers), and writes the crop parameter table.
// The Python replay (aphantasia_b200/_rng.py) stays as the executable specification; tests require identical tables
// and identical generator states afterwards.
#include "aph_common.cuh"
#include <math.h>
#include <string.h>

namespace aph {

struct Mt {            // MT19937 core shared by both generators
  uint32_t s[624];
  static inline uint32_t mix(uint32_t u, uint32_t v) { return (((u & 0x80000000u) | (v & 0x7fffffffu)) >> 1) ^ ((v & 1u) ? 0x9908b0dfu : 0u); }
  void reload() {
    const int N = 624, M = 397;
    int i = 0;
    for (; i < N - M; ++i) s[i] = s[i + M] ^ mix(s[i], s[i + 1]);
    for (; i < N - 1; ++i) s[i] = s[i + M - N] ^ mix(s[i], s[i + 1]);
    s[N - 1] = s[M - 1] ^ mix(s[N - 1], s[0]);
  }
  static inline uint32_t temper(uint32_t y) {
    y ^= (y >> 11); y ^= (y << 7) & 0x9d2c5680u; y ^= (y << 15) & 0xefc60000u; y ^= (y >> 18);
    return y;
  }
};

// ATen CPUGeneratorImpl legacy state blob (torch.get_rng_state(), 5056 bytes):
//   uint64 seed; int32 left; int32 seeded; uint64 next; uint64 state[624]; double normal_x, normal_y, normal_rho;
//   int32 normal_is_valid; (+ float next_float_normal_sample; bool valid)
struct TorchGen {
  Mt mt; int left; uint64_t next; uint8_t* blob;
  explicit TorchGen(uint8_t* b) : blob(b) {
    int32_t l; memcpy(&l, b + 8, 4); left = l;
    memcpy(&next, b + 16, 8);
    for (int i = 0; i < 624; ++i) { uint64_t v; memcpy(&v, b + 24 + 8 * i, 8); mt.s[i] = (uint32_t)v; }
  }
  void store() {
    int32_t l = left; memcpy(blob + 8, &l, 4);
    memcpy(blob + 16, &next, 8);
    for (int i = 0; i < 624; ++i) { uint64_t v = mt.s[i]; memcpy(blob + 24 + 8 * i, &v, 8); }
  }
  inline uint32_t random() {                       // at::mt19937::operator()
    if (--left == 0) { mt.reload(); left = 624; next = 0; }
    return Mt::temper(mt.s[next++]);
  }
  inline float rand01() { return (float)(random() & ((1u << 24) - 1)) * (1.0f / 16777216.0f); }      // torch.rand(1)
  inline float uniform(float from, float to) { return fmaf(rand01(), to - from, from); }              // tensor.uniform_(from, to)
  inline int64_t randint(int64_t lo, int64_t hi) { return (int64_t)(random() % (uint64_t)(hi - lo)) + lo; }   // torch.randint(lo, hi, (1,))
};

struct NumpyGen {      // legacy RandomState: key[624], pos
  Mt mt; int pos;
  inline uint32_t next32() {
    if (pos == 624) { mt.reload(); pos = 0; }
    return Mt::temper(mt.s[pos++]);
  }
  inline uint32_t bounded_masked(uint32_t rng) {   // legacy randint(0, rng + 1): masked rejection on 32-bit draws
    uint32_t mask = rng;
    mask |= mask >> 1; mask |= mask >> 2; mask |= mask >> 4; mask |= mask >> 8; mask |= mask >> 16;
    uint32_t v;
    do { v = next32() & mask; } while (v > rng);
    return v;
  }
  inline double rand53() {                         // legacy random_sample / rand(): 53-bit double from two 32-bit draws
    const uint32_t a = next32() >> 5, b = next32() >> 6;
    return (a * 67108864.0 + b) / 9007199254740992.0;
  }
};

// 8x8 linear solve in double (partial pivoting); the system is the one torchvision's _get_perspective_coeffs builds.
static bool solve8(double a[8][8], double b[8], double x[8]) {
  for (int c = 0; c < 8; ++c) {
    int p = c;
    for (int r = c + 1; r < 8; ++r) if (fabs(a[r][c]) > fabs(a[p][c])) p = r;
    if (a[p][c] == 0.0) return false;
    if (p != c) { for (int k = 0; k < 8; ++k) { double t = a[c][k]; a[c][k] = a[p][k]; a[p][k] = t; } double t = b[c]; b[c] = b[p]; b[p] = t; }
    for (int r = c + 1; r < 8; ++r) {
      const double f = a[r][c] / a[c][c];
      if (f != 0.0) { for (int k = c; k < 8; ++k) a[r][k] -= f * a[c][k]; b[r] -= f * b[c]; }
    }
  }
  for (int r = 7; r >= 0; --r) {
    double acc = b[r];
    for (int k = r + 1; k < 8; ++k) acc -= a[r][k] * x[k];
    x[r] = acc / a[r][r];
  }
  return true;
}

// RandomErasing(p = 0.2, scale (0.02, 0.33), ratio (0.3, 3.3), value 0) on an image of side `side`: APH_FLAG_ERASE or 0
static int draw_erase(TorchGen& tg, float* row, int side) {
  if (!(tg.rand01() < 0.2f)) return 0;
  const double area = (double)side * side;
  const float lr0 = logf(0.3f), lr1 = logf(3.3f);          // torch.log(torch.tensor((0.3, 3.3))) in float32
  for (int it = 0; it < 10; ++it) {
    const double erase_area = area * (double)tg.uniform(0.02f, 0.33f);
    const double aspect = (double)(float)exp((double)tg.uniform(lr0, lr1));     // torch.exp on a float32 tensor
    const int h = (int)nearbyint(sqrt(erase_area * aspect)), w = (int)nearbyint(sqrt(erase_area / aspect));
    if (!(h < side && w < side)) continue;
    const int i = (int)tg.randint(0, side - h + 1), j = (int)tg.randint(0, side - w + 1);
    row[APH_F_ER_I] = (float)i; row[APH_F_ER_J] = (float)j; row[APH_F_ER_H] = (float)h; row[APH_F_ER_W] = (float)w;
    return APH_FLAG_ERASE;
  }
  return 0;
}

// np.random.choice(list(range(-30, 30)) + 20 * [0]) (transforms.py:160, 168): degrees
static double draw_angle(NumpyGen& ng) {
  const uint32_t idx = ng.bounded_masked(79);
  return idx < 60 ? (double)((int)idx - 30) : 0.0;
}

// transforms_custom / transforms_elastic (transforms.py:147-163) after slice_imgs' macro draw: [RandomErasing on the padded
// image (torch)], random_rotate's angle, [random_elastic: rand(2), randint(8, 64), rand()], jitter(8): dx, dy (all NumPy)
static void draw_kornia(TorchGen& tg, NumpyGen& ng, float* row, int size, bool elastic) {
  const int s = size + 8;
  int flags = APH_FLAG_ROT | APH_FLAG_JITTER;
  if (elastic) flags |= draw_erase(tg, row, s);
  const double angle = draw_angle(ng);
  const double rot = angle * (M_PI / 180.0);
  // kornia get_rotation_matrix2d (OpenCV convention) inverted: source = c + [[cos, -sin], [sin, cos]] (dest - c)
  row[APH_F_ROT] = (float)cos(rot); row[APH_F_ROT + 1] = (float)(-sin(rot)); row[APH_F_ROT + 2] = (float)sin(rot); row[APH_F_ROT + 3] = (float)cos(rot);
  row[APH_F_ANGLE] = (float)angle;
  if (elastic) {        // the noise is zero: alpha, kernel size and sigma are drawn but do not change the output
    ng.rand53(); ng.rand53();
    ng.bounded_masked(55);
    ng.rand53();
    flags |= APH_FLAG_ELASTIC;
  }
  row[APH_F_JIT_DX] = (float)ng.bounded_masked(7);
  row[APH_F_JIT_DY] = (float)ng.bounded_masked(7);
  row[APH_F_FLAGS] = (float)flags;
}

static void draw_fast(TorchGen& tg, NumpyGen& ng, float* row, int size) {
  int flags = 0;
  // RandomPerspective(0.33, p = 0.2)
  if (tg.rand01() < 0.2f) {
    const int half = size / 2, d = (int)(0.33 * half);
    int ex[4], ey[4];
    ex[0] = (int)tg.randint(0, d + 1);           ey[0] = (int)tg.randint(0, d + 1);                 // top-left
    ex[1] = (int)tg.randint(size - d - 1, size); ey[1] = (int)tg.randint(0, d + 1);                 // top-right
    ex[2] = (int)tg.randint(size - d - 1, size); ey[2] = (int)tg.randint(size - d - 1, size);       // bottom-right
    ex[3] = (int)tg.randint(0, d + 1);           ey[3] = (int)tg.randint(size - d - 1, size);       // bottom-left
    const int sx[4] = {0, size - 1, size - 1, 0}, sy[4] = {0, 0, size - 1, size - 1};
    double a[8][8], b[8], x[8];
    for (int i = 0; i < 4; ++i) {
      const double p1x = ex[i], p1y = ey[i], p2x = sx[i], p2y = sy[i];
      const double r0[8] = {p1x, p1y, 1, 0, 0, 0, -p2x * p1x, -p2x * p1y};
      const double r1[8] = {0, 0, 0, p1x, p1y, 1, -p2y * p1x, -p2y * p1y};
      memcpy(a[2 * i], r0, sizeof(r0)); memcpy(a[2 * i + 1], r1, sizeof(r1));
      b[2 * i] = p2x; b[2 * i + 1] = p2y;
    }
    if (solve8(a, b, x)) { for (int i = 0; i < 8; ++i) row[APH_F_PERSP + i] = (float)x[i]; flags |= APH_FLAG_PERSP; }
  }
  flags |= draw_erase(tg, row, size);
  // random_rotate_fast: np.random.choice(list(range(-30, 30)) + 20 * [0]), always applied
  const double angle = draw_angle(ng);
  const double rot = angle * (M_PI / 180.0);
  row[APH_F_ROT] = (float)cos(rot); row[APH_F_ROT + 1] = (float)sin(rot); row[APH_F_ROT + 2] = (float)(-sin(rot)); row[APH_F_ROT + 3] = (float)cos(rot);
  row[APH_F_ANGLE] = (float)angle;
  flags |= APH_FLAG_ROT;
  row[APH_F_FLAGS] = (float)flags;
}

}  // namespace aph

using namespace aph;

// torch_state: the 5056-byte blob of torch.get_rng_state() (updated in place); np_key[624] + *np_pos: NumPy's legacy
// MT19937 state (updated in place). rnd_size / rnd_offx / rnd_offy: the three [count] vectors slice_imgs draws first
// (utils.py:222-228; left to torch because 'central' uses randn). tables: [n_imgs][count][APH_CROP_PARAM_FLOATS].
extern "C" int aph_rng_crop_tables(uint8_t* torch_state, int64_t torch_state_bytes, uint32_t* np_key, int32_t* np_pos,
                                   const float* rnd_size, const float* rnd_offx, const float* rnd_offy, int count, int H, int W,
                                   int frame_h, int frame_w, int size, int kind, float macro, int n_imgs, float* tables) {
  APH_REQUIRE(torch_state && np_key && np_pos && rnd_size && rnd_offx && rnd_offy && tables, "aph_rng_crop_tables: null pointer");
  APH_REQUIRE(torch_state_bytes >= 24 + 624 * 8, "aph_rng_crop_tables: torch RNG state blob too small (%lld bytes)", (long long)torch_state_bytes);
  APH_REQUIRE(*np_pos >= 0 && *np_pos <= 624, "aph_rng_crop_tables: bad numpy MT position %d", *np_pos);
  TorchGen tg(torch_state);
  NumpyGen ng; memcpy(ng.mt.s, np_key, sizeof(ng.mt.s)); ng.pos = *np_pos;
  const int sz_max = H < W ? H : W;
  const float macro_min = 0.9f * (float)sz_max;               // 0.9 * sz_max[i] : python scalar * int64 tensor -> float32
  for (int im = 0; im < n_imgs; ++im) {
    for (int c = 0; c < count; ++c) {
      float* row = tables + ((size_t)im * count + c) * APH_CROP_PARAM_FLOATS;
      memset(row, 0, APH_CROP_PARAM_FLOATS * sizeof(float));
      const bool mac = tg.rand01() < macro;
      // map(x, a, b) = x * (b - a) + a evaluated in float32, two roundings (utils.py:219-220), then .int() truncation
      float span, lo;
      if (mac) { lo = macro_min; span = (float)sz_max - macro_min; } else { lo = (float)size; span = (float)(sz_max - size); }
      volatile float prod = rnd_size[c] * span;
      const int csize = (int)(prod + lo);
      volatile float px = rnd_offx[c] * (float)(frame_w - csize);
      volatile float py = rnd_offy[c] * (float)(frame_h - csize);
      row[APH_F_OFFY] = (float)(int)(py + 0.0f); row[APH_F_OFFX] = (float)(int)(px + 0.0f); row[APH_F_CSIZE] = (float)csize;
      row[APH_F_ROT] = 1.f; row[APH_F_ROT + 3] = 1.f;
      if (kind == APH_TF_FAST) draw_fast(tg, ng, row, size);
      else if (kind == APH_TF_CUSTOM || kind == APH_TF_ELASTIC) draw_kornia(tg, ng, row, size, kind == APH_TF_ELASTIC);
    }
  }
  tg.store();
  memcpy(np_key, ng.mt.s, sizeof(ng.mt.s)); *np_pos = ng.pos;
  return 0;
}
