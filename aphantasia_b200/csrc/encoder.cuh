// encoder.cuh -- what the CLIP image tower (vit.cu) and text tower (text.cu) share: the residual block's weights, added to the
// handle's weight table (weights.cuh) block by block, and the block's forward. Defined in vit.cu.
#pragma once
#include "vit_ops.cuh"
#include "weights.cuh"
#include <functional>

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

// The part of a tower's handle that both towers have
struct Encoder : Weights {
  std::vector<BlockW> L;
};

// `layers` blocks of width D under "transformer.resblocks.<i>."; with dgrad, also the transposed operands of the data gradient
int add_blocks(Encoder* h, int layers, int D, bool dgrad);

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

// The image towers' CUDA-graph cache (struct GraphCache, vit.cu) for a handle defined elsewhere (the ResNet tower, rn.cu):
// replay() runs `body` through the cache exactly as the ViT's forward and backward do.
struct GraphCache;
struct GraphCacheRef : NoCopy {
  GraphCache* cache;
  GraphCacheRef();
  ~GraphCacheRef();
  int replay(int S, int flag, cudaStream_t& st, const std::function<int()>& body);
};

// The resident attention kernels (T <= 256, head dim 64) on qkv [S*T, 3D]: fwd writes out [S*T, D]; otherwise dout [S*T, D] in,
// dqkv [S*T, 3D] out. Defined in vit.cu.
int attn_resident(bool fwd, const bf16* qkv, const bf16* dout, bf16* out_or_dqkv, int S, int T, int D, int heads, cudaStream_t st);

}  // namespace aph
