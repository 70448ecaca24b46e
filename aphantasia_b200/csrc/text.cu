// text.cu -- CLIP text encoder handle (forward only): fp32 token embedding, packed bf16 layer weights, one set of
// activation buffers, built from the image tower's pieces (wgmma GEMM with fused epilogues, k_ln_fwd, tensor-core attention).
//
// Restates OpenAI clip/model.py CLIP.encode_text (third-party, SURVEY.md A5):
//   x = token_embedding[ids] + positional_embedding -> layers x { x += out_proj(causal MHA(ln_1 x)); x += c_proj(QuickGELU(c_fc(ln_2 x))) }
//   -> ln_final(x[s, argmax(ids[s])]) @ text_projection
// It runs a handful of times per script run (once per prompt, before the optimisation loop): no CUDA graph, nothing is
// saved for a backward pass, and each layer overwrites the previous one's activations.
#include "encoder.cuh"
#include "vit_attn_tc.cuh"

namespace aph {
namespace {

struct TextImpl : Encoder {
  aph_text_config cfg;
  // weights besides the blocks'
  float* tok_emb = nullptr;      // [vocab, D] fp32: a gather reads n*ctx rows of it once per call
  float* pos = nullptr;          // [ctx, D]
  float *lnf_w = nullptr, *lnf_b = nullptr;
  bf16* w_out = nullptr;         // text_projection^T [out, D]
  // activations, sized for max_batch * ctx rows
  float *x = nullptr, *x_mid = nullptr;   // residual stream fp32 [M, D], ping-pong within a layer
  bf16* ln_out = nullptr;        // [M, D]
  bf16* qkv = nullptr;           // [M, 3D]
  bf16* attn_out = nullptr;      // [M, D]
  bf16* h_pre = nullptr;         // [M, 4D] (the fused QuickGELU epilogue always writes its pre-activation)
  bf16* h_act = nullptr;         // [M, 4D]
  float *mean = nullptr, *rstd = nullptr;  // [M] LayerNorm statistics (written by k_ln_fwd, unused here)
  int* eot = nullptr;            // [max_batch] pooling position per sequence
  bf16* pooled = nullptr;        // [max_batch, D] ln_final of the pooled rows
};

// x[row] = token_embedding[ids[row]] + positional_embedding[row % ctx]; one warp per token row.
// An id outside [0, vocab) contributes a zero row instead of reading out of bounds.
template <int NCH>
__global__ void __launch_bounds__(256) k_text_embed(const int64_t* __restrict__ ids, const float* __restrict__ tok_emb,
                                                    const float* __restrict__ pos, float* __restrict__ x, int rows, int ctx, int D, int vocab) {
  const int row = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (row >= rows) return;
  constexpr int N = 4 * NCH;
  const long long id = ids[row];
  float v[N], pz[N];
  load_row(pos + (size_t)(row % ctx) * D, pz, lane);
  if (id >= 0 && id < vocab) load_row(tok_emb + (size_t)id * D, v, lane);
  else {
#pragma unroll
    for (int i = 0; i < N; ++i) v[i] = 0.f;
  }
#pragma unroll
  for (int i = 0; i < N; ++i) v[i] += pz[i];
  store_row_f32(x + (size_t)row * D, v, lane);
}

// eot[s] = first position of the largest id of sequence s (torch.argmax semantics); one warp per sequence.
__global__ void __launch_bounds__(256) k_text_eot(const int64_t* __restrict__ ids, int* __restrict__ eot, int n, int ctx) {
  const int s = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (s >= n) return;
  long long best = ids[(size_t)s * ctx];
  int bi = 0;
  for (int t = lane; t < ctx; t += 32) {
    const long long v = ids[(size_t)s * ctx + t];
    if (v > best) { best = v; bi = t; }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const long long ob = __shfl_xor_sync(0xffffffffu, best, o);
    const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
    if (ob > best || (ob == best && oi < bi)) { best = ob; bi = oi; }
  }
  if (lane == 0) eot[s] = bi;
}

// y[s] = ln_final(x[s * ctx + eot[s]]) as bf16 (the A operand of the projection GEMM); one warp per sequence.
template <int NCH>
__global__ void __launch_bounds__(256) k_text_pool_ln(const float* __restrict__ x, const int* __restrict__ eot, const float* __restrict__ gamma,
                                                      const float* __restrict__ beta, bf16* __restrict__ y, int n, int ctx, int D) {
  const int s = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (s >= n) return;
  constexpr int N = 4 * NCH;
  float v[N], gm[N], bt[N];
  load_row(x + ((size_t)s * ctx + eot[s]) * D, v, lane);
  const RowStats st = row_stats(v, D);
  load_row(gamma, gm, lane); load_row(beta, bt, lane);
#pragma unroll
  for (int i = 0; i < N; ++i) v[i] = (v[i] - st.mean) * st.rstd * gm[i] + bt[i];
  store_row_bf16(y + (size_t)s * D, v, lane);
}

// causal tensor-core attention: the image tower's forward kernel with the mask compiled in
template <int NW, int NT2>
int attn_causal_launch(const bf16* qkv, bf16* out, int S, int T, int D, int heads, cudaStream_t st) {
  if (int e = smem_at_least((const void*)k_attn_fwd_tc<NW, NT2, true>, attn_tc_fwd_smem<NW, NT2>())) return e;
  k_attn_fwd_tc<NW, NT2, true><<<S * heads, NW * 32, attn_tc_fwd_smem<NW, NT2>(), st>>>(qkv, out, T, D, heads);
  APH_LAUNCH_OK();
  return 0;
}

int attn_causal(const bf16* qkv, bf16* out, int S, int T, int D, int heads, cudaStream_t st) {
  if (T <= 32) return attn_causal_launch<4, 2>(qkv, out, S, T, D, heads, st);
  if (T <= 64) return attn_causal_launch<4, 4>(qkv, out, S, T, D, heads, st);
  if (T <= 112) return attn_causal_launch<8, 7>(qkv, out, S, T, D, heads, st);
  set_error("text attention: context %d > 112 unsupported", T);
  return 2;
}

}  // namespace

// the text tower's causal attention, for the test entry aph_attn_test (vit.cu)
int attn_causal_test(const bf16* qkv, bf16* out, int S, int T, int D, int heads, cudaStream_t st) {
  return attn_causal(qkv, out, S, T, D, heads, st);
}
}  // namespace aph

using namespace aph;

extern "C" int aph_text_create(aph_text** out, const aph_text_config* cfg) {
  APH_REQUIRE(out && cfg, "aph_text_create: null argument");
  const int w128 = cfg->width / 128;
  APH_REQUIRE(cfg->width % 128 == 0 && (w128 == 1 || w128 == 2 || w128 == 4 || w128 == 5 || w128 == 6 || w128 == 8),
              "aph_text_create: width %d unsupported (128, 256, 512, 640, 768, 1024)", cfg->width);
  APH_REQUIRE(cfg->heads * 64 == cfg->width, "aph_text_create: head dim must be 64 (width %d, heads %d)", cfg->width, cfg->heads);
  APH_REQUIRE(cfg->context > 0 && cfg->context <= 112, "aph_text_create: context %d outside [1, 112]", cfg->context);
  APH_REQUIRE(cfg->out_dim > 0 && cfg->out_dim % 128 == 0, "aph_text_create: out_dim %d must be a multiple of 128", cfg->out_dim);
  APH_REQUIRE(cfg->vocab > 0 && cfg->max_batch > 0 && cfg->layers > 0, "aph_text_create: vocab %d, max_batch %d, layers %d must be positive",
              cfg->vocab, cfg->max_batch, cfg->layers);
  std::unique_ptr<TextImpl> t(new TextImpl());
  t->cfg = *cfg;
  const int D = cfg->width, O = cfg->out_dim, B = cfg->max_batch;
  const size_t M = (size_t)B * cfg->context;
  int e = 0;
  e |= t->add_f32("token_embedding.weight", &t->tok_emb, (size_t)cfg->vocab * D);
  e |= t->add_f32("positional_embedding", &t->pos, (size_t)cfg->context * D);
  e |= t->add_f32("ln_final.weight", &t->lnf_w, D); e |= t->add_f32("ln_final.bias", &t->lnf_b, D);
  e |= t->add_bf16("text_projection", D, O, nullptr, &t->w_out);   // [D, out] -> [out, D]
  e |= add_blocks(t.get(), cfg->layers, D, false);
  e |= t->alloc(&t->x, M * D); e |= t->alloc(&t->x_mid, M * D); e |= t->alloc(&t->ln_out, M * D);
  e |= t->alloc(&t->qkv, M * 3 * D); e |= t->alloc(&t->attn_out, M * D);
  e |= t->alloc(&t->h_pre, M * 4 * D); e |= t->alloc(&t->h_act, M * 4 * D);
  e |= t->alloc(&t->mean, M); e |= t->alloc(&t->rstd, M);
  e |= t->alloc(&t->eot, (size_t)B); e |= t->alloc(&t->pooled, (size_t)B * D);
  if (e) return 1;
  *out = reinterpret_cast<aph_text*>(t.release());
  return 0;
}

extern "C" int aph_text_destroy(aph_text* text) {
  delete reinterpret_cast<TextImpl*>(text);
  return 0;
}

extern "C" int64_t aph_text_bytes(const aph_text* text) { return text ? reinterpret_cast<const TextImpl*>(text)->bytes : 0; }

extern "C" int aph_text_load_tensor(aph_text* text, const char* key, const float* data, int64_t numel, void* stream) {
  return load_tensor(reinterpret_cast<TextImpl*>(text), key, data, numel, (cudaStream_t)stream, "aph_text_load_tensor");
}

extern "C" int aph_text_finalize(aph_text* text) { return finalize(reinterpret_cast<TextImpl*>(text), "aph_text_finalize"); }

extern "C" int aph_text_fwd(aph_text* text, const int64_t* tokens, int n, float* emb, void* stream) {
  APH_REQUIRE(text && tokens && emb, "aph_text_fwd: null argument");
  TextImpl* t = reinterpret_cast<TextImpl*>(text);
  APH_REQUIRE(t->finalized, "aph_text_fwd: weights not finalized");
  APH_REQUIRE(n > 0 && n <= t->cfg.max_batch, "aph_text_fwd: n=%d outside (0, max_batch=%d]", n, t->cfg.max_batch);
  cudaStream_t st = (cudaStream_t)stream;
  const int D = t->cfg.width, C = t->cfg.context, H = t->cfg.heads, O = t->cfg.out_dim;
  const int M = n * C;
  int e;
  NCH_DISPATCH_TEXT(D, k_text_embed<NCH><<<rows_grid(M), 256, 0, st>>>(tokens, t->tok_emb, t->pos, t->x, M, C, D, t->cfg.vocab));
  APH_LAUNCH_OK();
  k_text_eot<<<rows_grid(n), 256, 0, st>>>(tokens, t->eot, n, C);
  APH_LAUNCH_OK();
  const BlockIO io{t->x, t->x_mid, t->x, t->ln_out, t->qkv, t->attn_out, t->h_pre, t->h_act, t->mean, t->rstd, t->mean, t->rstd};
  for (const BlockW& w : t->L)
    if ((e = block_fwd(w, io, n, C, M, 0, D, H, attn_causal, st))) return e;
  NCH_DISPATCH_TEXT(D, k_text_pool_ln<NCH><<<rows_grid(n), 256, 0, st>>>(t->x, t->eot, t->lnf_w, t->lnf_b, t->pooled, n, C, D));
  APH_LAUNCH_OK();
  GemmEpi ep; ep.out_f32 = emb;
  return launch_gemm(t->pooled, t->w_out, GemmShape{n, O, D}, ep, st);
}
