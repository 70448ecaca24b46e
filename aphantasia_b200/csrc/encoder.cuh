// encoder.cuh -- what the CLIP image tower (vit.cu) and text tower (text.cu) share: a handle's device allocations, the residual
// block's weights (allocated, loaded and checked from one table of its tensors) and the block's forward. Defined in vit.cu.
#pragma once
#include "vit_ops.cuh"
#include <map>
#include <string>
#include <vector>

namespace aph {

// One residual block's weights: LayerNorm affines and biases in fp32; the GEMMs' forward B operands [N, K] in bf16 and, for the
// image tower's data gradient, their transposes [K, N] (null in the text tower, which has no backward).
struct BlockW {
  float *ln1_w = nullptr, *ln1_b = nullptr, *ln2_w = nullptr, *ln2_b = nullptr;
  float *b_qkv = nullptr, *b_o = nullptr, *b_fc = nullptr, *b_proj = nullptr;
  bf16 *w_qkv = nullptr, *w_qkv_t = nullptr;     // [3D, D], [D, 3D]
  bf16 *w_o = nullptr, *w_o_t = nullptr;         // [D, D]
  bf16 *w_fc = nullptr, *w_fc_t = nullptr;       // [4D, D], [D, 4D]
  bf16 *w_proj = nullptr, *w_proj_t = nullptr;   // [D, 4D], [4D, D]
};

// The part of a tower's handle that both towers have. Its device allocations are freed with it.
struct Encoder {
  int64_t bytes = 0;                      // aph_vit_bytes / aph_text_bytes
  std::vector<void*> allocs;
  std::vector<BlockW> L;
  std::map<std::string, bool> loaded;     // state-dict keys, the image tower's without "visual."
  bool finalized = false;
  ~Encoder() { for (void* p : allocs) cudaFree(p); }
};

template <typename Tp>
int dev_alloc(Encoder* h, Tp** p, size_t count) {
  void* q = nullptr;
  APH_CUDA_OK(cudaMalloc(&q, count * sizeof(Tp)));
  h->allocs.push_back(q);
  h->bytes += (int64_t)(count * sizeof(Tp));
  *p = reinterpret_cast<Tp*>(q);
  return 0;
}

// `layers` blocks of width D; with dgrad, also the transposed operands of the data gradient
int alloc_blocks(Encoder* h, int layers, int D, bool dgrad);
// k = "transformer.resblocks.<i>.<field>" -> block i's slot (and its transpose when allocated). `key` is the caller's key and
// `who` the entry point, for the error messages.
int load_block_tensor(Encoder* h, const std::string& k, const char* key, const float* data, int64_t numel, int D, cudaStream_t st,
                      const char* who);
// every key of `want` and of the blocks was loaded; a missing one is named as prefix + key
int check_loaded(const Encoder* h, std::vector<std::string> want, const char* who, const char* prefix);

// fp32 [rows, cols] -> bf16 [rows, cols] (transpose = 0, row stride ld, 0 = cols) or bf16 [cols, rows] (transpose = 1)
int pack(const float* src, bf16* dst, int rows, int cols, int transpose, cudaStream_t st, int ld = 0);
int copy_f32(const float* src, float* dst, size_t n, cudaStream_t st);

// grid of the one-warp-per-row kernels
inline int rows_grid(int rows) { return (rows * 32 + 255) / 256; }

// One block's activations and LayerNorm statistics. x_out may be x_in (the text tower keeps no snapshots).
struct BlockIO {
  const float* x_in; float *x_mid, *x_out;
  bf16 *ln_out, *qkv, *attn_out, *h_pre, *h_act;
  float *mean1, *rstd1, *mean2, *rstd2;
};

typedef int (*AttnFwd)(const bf16* qkv, bf16* out, int S, int T, int D, int heads, cudaStream_t st);

// x_mid = x_in + out_proj(attn(qkv(ln_1 x_in))); x_out = x_mid + c_proj(QuickGELU(c_fc(ln_2 x_mid))) for S sequences of T tokens.
// ln_1, qkv and attention run on all S*T rows, out_proj and what follows on Mr rows. out_proj reads its rows of attn_out and
// x_in at row stride ld_tok (0: dense; the image tower's last block takes the class-token rows, Mr = S and ld_tok = T*D).
int block_fwd(const BlockW& w, const BlockIO& io, int S, int T, int Mr, int ld_tok, int D, int heads, AttnFwd attn, cudaStream_t st);

}  // namespace aph
