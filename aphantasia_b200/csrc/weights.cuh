// weights.cuh -- what every weight-bearing handle (aph_vit, aph_text, aph_lpips) shares: its device allocations, freed with it,
// and the table of the state-dict tensors it takes, built at create time. One loader looks a key up in the table, checks its
// element count and lands it on the device; one finalize names the first tensor that never arrived. Defined in weights.cu.
#pragma once
#include "aph_common.cuh"
#include <string>
#include <vector>

namespace aph {

// How a tensor lands on the device:
//   W_F32      copied as it is;
//   W_BF16     the fp32 [rows, cols] source packed to bf16 as it is into w (row stride ld, 0 = cols) and/or transposed into
//              w_t [cols, rows]; an absent destination is null;
//   W_CONV3X3  a 3x3 convolution [rows = C_out, cols = C_in, 3, 3] packed into w [C_out][tap][C_in] (forward operand) and w_t
//              [C_in][tap][C_out] = flipped taps (data-gradient operand).
enum WeightKind { W_F32, W_BF16, W_CONV3X3 };

struct WeightEntry {
  std::string key;             // state-dict key, without the handle's prefix
  WeightKind kind;
  int64_t numel;
  float* f32;
  bf16 *w, *w_t;
  int rows, cols, ld;
  bool loaded;
};

struct Weights : DeviceAllocs {
  const char* prefix = "";     // a key prefix the loader accepts and drops ("visual." for the image tower); finalize names it
  std::vector<WeightEntry> table;
  bool finalized = false;      // every entry loaded, and nothing loaded since

  // Each allocates its destinations (null: none) and adds the entry.
  int add_f32(const std::string& key, float** dst, size_t n) {
    const int e = alloc(dst, n);
    table.push_back({key, W_F32, (int64_t)n, *dst, nullptr, nullptr, 0, 0, 0, false});
    return e;
  }
  int add_bf16(const std::string& key, int rows, int cols, bf16** w, bf16** w_t, int ld = 0) {
    const size_t n = (size_t)rows * (ld > 0 ? ld : cols);   // w_t of a padded w spans the pad rows too
    int e = 0;
    if (w) e |= alloc(w, n);
    if (w_t) e |= alloc(w_t, n);
    table.push_back({key, W_BF16, (int64_t)rows * cols, nullptr, w ? *w : nullptr, w_t ? *w_t : nullptr, rows, cols, ld, false});
    return e;
  }
  int add_conv3x3(const std::string& key, int co, int ci, bf16** w, bf16** w_t) {
    const size_t n = (size_t)co * ci * 9;
    int e = alloc(w, n);
    e |= alloc(w_t, n);
    table.push_back({key, W_CONV3X3, (int64_t)n, nullptr, *w, *w_t, co, ci, 0, false});
    return e;
  }
};

// `who` is the entry point the messages name. A load voids `finalized`.
int load_tensor(Weights* h, const char* key, const float* data, int64_t numel, cudaStream_t st, const char* who);
int finalize(Weights* h, const char* who);

// w fp32 [co, ci, 3, 3] -> wf / wb as W_CONV3X3 (either may be null)
int pack_conv3x3(const float* w, int co, int ci, bf16* wf, bf16* wb, cudaStream_t st);

}  // namespace aph
