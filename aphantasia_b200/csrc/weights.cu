// weights.cu -- the shared loader of the weight-bearing handles (weights.cuh) and the kernels that pack their weights.
#include "weights.cuh"
#include <algorithm>
#include <stdlib.h>
#include <string.h>

namespace aph {

// ld: row stride of the untransposed output (>= cols; the columns past cols are not written)
__global__ void __launch_bounds__(256) k_pack_weight(const float* __restrict__ in, bf16* __restrict__ out, int rows, int cols, int transpose, int ld) {
  const size_t n = (size_t)rows * cols;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const int r = (int)(i / cols), c = (int)(i - (size_t)r * cols);
    const bf16 v = __float2bfloat16_rn(in[i]);
    if (transpose) out[(size_t)c * rows + r] = v; else out[(size_t)r * ld + c] = v;
  }
}

// w fp32 [Co, Ci, 3, 3] -> forward operand wf [Co][tap][Ci] and data-gradient operand wb [Ci][tap][Co] = w[co][ci][8 - tap]
__global__ void k_pack_w(const float* __restrict__ w, int Co, int Ci, bf16* __restrict__ wf, bf16* __restrict__ wb) {
  const size_t n = (size_t)Co * Ci * 9;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const int t = (int)(i % 9), ci = (int)((i / 9) % Ci), co = (int)(i / (9 * (size_t)Ci));
    const bf16 v = __float2bfloat16(w[i]);
    if (wf) wf[((size_t)co * 9 + t) * Ci + ci] = v;
    if (wb) wb[((size_t)ci * 9 + (8 - t)) * Co + co] = v;
  }
}

static int pack(const float* src, bf16* dst, int rows, int cols, int transpose, int ld, cudaStream_t st) {
  k_pack_weight<<<stride_blocks((size_t)rows * cols, 16), 256, 0, st>>>(src, dst, rows, cols, transpose, ld > 0 ? ld : cols);
  APH_LAUNCH_OK();
  return 0;
}

int pack_conv3x3(const float* w, int co, int ci, bf16* wf, bf16* wb, cudaStream_t st) {
  k_pack_w<<<stride_blocks((size_t)co * ci * 9, 16), 256, 0, st>>>(w, co, ci, wf, wb);
  APH_LAUNCH_OK();
  return 0;
}

static int land(const WeightEntry& t, const float* data, cudaStream_t st) {
  switch (t.kind) {
    case W_F32:
      APH_CUDA_OK(cudaMemcpyAsync(t.f32, data, t.numel * sizeof(float), cudaMemcpyDeviceToDevice, st));
      return 0;
    case W_BF16:
      if (t.w)
        if (int e = pack(data, t.w, t.rows, t.cols, 0, t.ld, st)) return e;
      return t.w_t ? pack(data, t.w_t, t.rows, t.cols, 1, 0, st) : 0;
    case W_CONV3X3:
      return pack_conv3x3(data, t.rows, t.cols, t.w, t.w_t, st);
  }
  return 0;
}

int load_tensor(Weights* h, const char* key, const float* data, int64_t numel, cudaStream_t st, const char* who) {
  APH_REQUIRE(h && key && data, "%s: null argument", who);
  const size_t np = strlen(h->prefix);
  const char* k = strncmp(key, h->prefix, np) == 0 ? key + np : key;
  for (WeightEntry& t : h->table) {
    if (t.key != k) continue;
    APH_REQUIRE(numel == t.numel, "%s(%s): expected %lld elements, got %lld", who, key, (long long)t.numel, (long long)numel);
    if (int e = land(t, data, st)) return e;
    t.loaded = true;
    h->finalized = false;
    return 0;
  }
  // a residual block's key that no entry matched: say so when its index names no block of the handle
  static const char kBlocks[] = "transformer.resblocks.";
  if (strncmp(k, kBlocks, sizeof(kBlocks) - 1) == 0) {
    char* end = nullptr;
    const long li = strtol(k + sizeof(kBlocks) - 1, &end, 10);
    const std::string block = kBlocks + std::to_string(li) + ".";
    const bool known = std::any_of(h->table.begin(), h->table.end(), [&](const WeightEntry& t) { return t.key.rfind(block, 0) == 0; });
    APH_REQUIRE(*end == '.' && known, "%s: bad layer index in %s", who, key);
  }
  set_error("%s: unknown tensor %s", who, key);
  return 2;
}

int finalize(Weights* h, const char* who) {
  APH_REQUIRE(h, "%s: null handle", who);
  for (const WeightEntry& t : h->table) APH_REQUIRE(t.loaded, "%s: tensor %s%s was never loaded", who, h->prefix, t.key.c_str());
  h->finalized = true;
  return 0;
}

}  // namespace aph
