// vit.cu -- CLIP ViT image encoder handle (B/32, B/16, L/14): packed bf16 weights, activation arena, forward and
// data-gradient backward built from the wgmma GEMM (tc_gemm.cuh) and the kernels of vit_ops.cuh.
//
// Restates OpenAI clip/model.py VisionTransformer.forward (third-party, SURVEY.md A5):
//   conv1 (patch-embed GEMM) -> [cls; tok] + pos -> ln_pre -> 12 x { x += out_proj(MHA(ln_1 x)); x += c_proj(QuickGELU(c_fc(ln_2 x))) }
//   -> ln_post(x[:,0]) @ proj
// The residual stream is fp32; GEMM operands are bf16; every x_l is kept (out-of-place residual) so the
// LayerNorm backward can recompute x-hat. No weight gradients (the reference computes and discards them).
#include "encoder.cuh"
#include "vit_attn_tc.cuh"
#include "vit_attn_stream.cuh"
#include <set>

namespace aph {

bool gemm_profiling_on();      // vit_gemm.cu

// CUDA-graph cache of one direction of a handle (forward or backward): the ~90 launches of a call are replayed as one graph when
// the call repeats with the same batch size S and flag (the optimisation loop does). The first call with an S runs eagerly (lazy
// one-time initialisations are not capturable), the next one captures and instantiates, later ones replay; a small LRU.
struct GraphCache : NoCopy {
  struct Entry { int S; int flag; cudaGraphExec_t exec; unsigned long long stamp; int nodes; };
  std::vector<Entry> entries;
  std::set<int> warm;            // batch sizes that have run eagerly
  unsigned long long stamp = 0;
  int misses = 0;                // captures in a row that were never replayed
  ~GraphCache() { for (auto& e : entries) cudaGraphExecDestroy(e.exec); }

  // Runs `body`, which launches on `st`, through the cache.
  template <typename Body>
  int run(int S, int flag, cudaStream_t& st, Body body) {
    // GEMM profiling (aph_prof_gemm) records events around each launch, so it runs eagerly. A cache whose keys keep changing
    // would re-capture forever: after 6 never-replayed captures in a row it stays eager
    if (gemm_profiling_on() || misses > 6) return body();
    for (auto& e : entries)
      if (e.S == S && e.flag == flag) {
        e.stamp = ++stamp;
        misses = 0;
        APH_CUDA_OK(cudaGraphLaunch(e.exec, st));
        count_launch(e.nodes);         // kernels replayed by the graph
        return 0;
      }
    if (warm.insert(S).second) return body();
    // The caller's stream is often the legacy default stream (torch's default), which cannot be captured: record the launch
    // sequence on a private stream (`st` is what the body launches on -- capture enqueues nothing), replay on the caller's.
    static cudaStream_t cap = nullptr;
    if (!cap) APH_CUDA_OK(cudaStreamCreateWithFlags(&cap, cudaStreamNonBlocking));
    cudaStream_t user = st;
    st = cap;
    if (cudaStreamBeginCapture(cap, cudaStreamCaptureModeThreadLocal) != cudaSuccess) { cudaGetLastError(); st = user; return body(); }
    const int rc = body();
    cudaGraph_t graph = nullptr;
    const cudaError_t ce = cudaStreamEndCapture(cap, &graph);
    st = user;
    if (rc != 0 || ce != cudaSuccess || graph == nullptr) {
      if (graph) cudaGraphDestroy(graph);
      cudaGetLastError();
      if (rc != 0) return rc;
      return body();                                               // capture refused: stay eager
    }
    size_t nodes = 0;
    cudaGraphGetNodes(graph, nullptr, &nodes);
    g_launches.fetch_sub((long long)nodes, std::memory_order_relaxed);   // the capture pass enqueued nothing; the replay below counts
    cudaGraphExec_t exec = nullptr;
    if (cudaGraphInstantiate(&exec, graph, 0) != cudaSuccess) { cudaGraphDestroy(graph); cudaGetLastError(); return body(); }
    cudaGraphDestroy(graph);
    if (entries.size() >= 4) {                                     // evict the least recently used
      size_t lru = 0;
      for (size_t i = 1; i < entries.size(); ++i) if (entries[i].stamp < entries[lru].stamp) lru = i;
      cudaGraphExecDestroy(entries[lru].exec);
      entries.erase(entries.begin() + lru);
    }
    ++misses;
    entries.push_back({S, flag, exec, ++stamp, (int)nodes});
    APH_CUDA_OK(cudaGraphLaunch(exec, st));
    count_launch((int)nodes);
    return 0;
  }
};

struct VitImpl : Encoder {
  aph_vit_config cfg;
  int g, T, D, Kp;                // Kp = patch_k(patch): the patch operand's row length, 3 p^2 zero-padded to a multiple of 128
  // weights besides the blocks'
  bf16 *w_conv = nullptr, *w_conv_t = nullptr;   // [D, Kp], [Kp, D]; the pad columns / rows are zero
  float *cls = nullptr, *pos = nullptr, *lnpre_w = nullptr, *lnpre_b = nullptr, *lnpost_w = nullptr, *lnpost_b = nullptr;
  bf16 *w_out = nullptr, *w_out_t = nullptr;     // proj^T [out, D] (forward B operand), proj [D, out] (dgrad B operand)
  // activations (sized for max_batch)
  bf16* patches = nullptr;       // [S*g*g, Kp]; columns >= 3 p^2 zeroed at creation and never written
  float* tok = nullptr;          // [S*g*g, D]
  float* e = nullptr;            // [M, D] pre-ln_pre
  // Everything the caller gets comes from the cls rows s*T of the last block's output (ln_post reads x[:, 0]). So past its
  // attention (whose keys and values come from every token) the last block runs on the S cls rows only: its x_mid, x_out and
  // h_pre are compact [S, ...] and its residual gradient is dxc / dxc_bf.
  std::vector<float*> xs;        // 2*layers+1 residual-stream snapshots, fp32 [M, D]; the last two are [S, D]
  bf16* ln_out = nullptr;        // [M, D]
  std::vector<bf16*> qkv;        // per layer [M, 3D]
  bf16* attn_out = nullptr;      // [M, D]
  std::vector<bf16*> h_pre;      // per layer [M, 4D]; the last layer's is [S, 4D]
  bf16* h_act = nullptr;         // [M, 4D]
  float *st_mean = nullptr, *st_rstd = nullptr;   // LayerNorm statistics, slots of stat_off()
  bf16* cls_ln = nullptr;        // [S, D]
  float* emb_int = nullptr;      // [S, out] (copied to the caller's buffer outside the graph)
  // backward scratch
  bf16* d_emb = nullptr;         // [S, out]
  float* d_cls = nullptr;        // [S, D]
  float* dxc = nullptr;          // [S, D] residual gradient of the last block (cls rows)
  bf16* dxc_bf = nullptr;        // [S, D]
  float* dx = nullptr;           // [M, D]
  bf16* dx_bf = nullptr;         // [M, D]
  bf16* dh = nullptr;            // [M, 4D]
  bf16* d_ln = nullptr;          // [M, D] gradient entering a LayerNorm backward (bf16: it is the output of a bf16-operand GEMM and is consumed once)
  bf16* d_attn = nullptr;        // [M, D]
  bf16* d_attn_last = nullptr;   // [M, D] the last block's attention-output gradient: zeroed at creation, only rows s*T are ever
                                 // written, so every other row stays exactly zero (layers below overwrite all rows of d_attn)
  bf16* d_qkv = nullptr;         // [M, 3D]
  bf16* d_tok = nullptr;         // [S*g*g, D]
  float2* attn_stats = nullptr;  // [S*heads*T] (lse, delta) of the streaming attention backward (T > 256 only), reused by every layer
  int last_S = -1;
  GraphCache fwd_graphs, bwd_graphs;
};

// LayerNorm statistics slot k: 0 = ln_pre, 1 + 2l / 2 + 2l = ln_1 / ln_2 of layer l, 2 layers + 1 = ln_post. The slots below
// 2 layers hold max_batch*T rows; the last two (ln_2 of the last block and ln_post, cls rows only) hold max_batch rows.
static size_t stat_off(const VitImpl* v, int k) {
  const size_t Mmax = (size_t)v->cfg.max_batch * v->T, k2 = 2 * (size_t)v->cfg.layers;
  return (size_t)k < k2 ? k * Mmax : k2 * Mmax + (k - k2) * (size_t)v->cfg.max_batch;
}

int add_blocks(Encoder* h, int layers, int D, bool dgrad) {
  h->L.resize(layers);
  int e = 0;
  for (int i = 0; i < layers; ++i) {
    BlockW& l = h->L[i];
    const std::string p = "transformer.resblocks." + std::to_string(i) + ".";
    auto mat = [&](const char* key, int rows, int cols, bf16** w, bf16** w_t) { e |= h->add_bf16(p + key, rows, cols, w, dgrad ? w_t : nullptr); };
    auto vec = [&](const char* key, int n, float** v) { e |= h->add_f32(p + key, v, n); };
    vec("ln_1.weight", D, &l.ln1_w); vec("ln_1.bias", D, &l.ln1_b); vec("ln_2.weight", D, &l.ln2_w); vec("ln_2.bias", D, &l.ln2_b);
    mat("attn.in_proj_weight", 3 * D, D, &l.w_qkv, &l.w_qkv_t); vec("attn.in_proj_bias", 3 * D, &l.b_qkv);
    mat("attn.out_proj.weight", D, D, &l.w_o, &l.w_o_t); vec("attn.out_proj.bias", D, &l.b_o);
    mat("mlp.c_fc.weight", 4 * D, D, &l.w_fc, &l.w_fc_t); vec("mlp.c_fc.bias", 4 * D, &l.b_fc);
    mat("mlp.c_proj.weight", D, 4 * D, &l.w_proj, &l.w_proj_t); vec("mlp.c_proj.bias", D, &l.b_proj);
  }
  return e;
}

int block_fwd(const BlockW& w, const BlockIO& io, int S, int T, int Mr, int ld_tok, int D, int heads, AttnFwd attn, cudaStream_t st) {
  const int M = S * T;
  int e;
  NCH_DISPATCH_TEXT(D, k_ln_fwd<NCH><<<rows_grid(M), 256, 0, st>>>(io.x_in, w.ln1_w, w.ln1_b, io.ln_out, io.mean1, io.rstd1, M, D));
  APH_LAUNCH_OK();
  { GemmEpi ep; ep.bias = w.b_qkv; ep.out_bf16 = io.qkv;
    if ((e = launch_gemm(io.ln_out, w.w_qkv, GemmShape{M, 3 * D, D}, ep, st))) return e; }
  if ((e = attn(io.qkv, io.attn_out, S, T, D, heads, st))) return e;
  { GemmEpi ep; ep.bias = w.b_o; ep.resid = io.x_in; ep.ld_resid = ld_tok; ep.out_f32 = io.x_mid;
    if ((e = launch_gemm(io.attn_out, w.w_o, GemmShape{Mr, D, D}, ep, st, ld_tok))) return e; }
  NCH_DISPATCH_TEXT(D, k_ln_fwd<NCH><<<rows_grid(Mr), 256, 0, st>>>(io.x_mid, w.ln2_w, w.ln2_b, io.ln_out, io.mean2, io.rstd2, Mr, D));
  APH_LAUNCH_OK();
  { GemmEpi ep; ep.bias = w.b_fc; ep.out_pre = io.h_pre; ep.act = 1; ep.out_bf16 = io.h_act;
    if ((e = launch_gemm(io.ln_out, w.w_fc, GemmShape{Mr, 4 * D, D}, ep, st))) return e; }
  { GemmEpi ep; ep.bias = w.b_proj; ep.resid = io.x_mid; ep.out_f32 = io.x_out;
    if ((e = launch_gemm(io.h_act, w.w_proj, GemmShape{Mr, D, 4 * D}, ep, st))) return e; }
  return 0;
}

// The resident kernels (attn_dispatch) keep a head's keys in shared memory and serve T <= 256; longer sequences
// (ViT-L/14: T = 257) take the streaming kernels of vit_attn_stream.cuh, whose backward needs `stats` (attn_stats).
constexpr int kAttnResidentMaxT = 256;

static int vit_attn(bool fwd, const bf16* qkv, const bf16* dout, bf16* out_or_dqkv, float2* stats, int S, int T, int D, int heads,
                    cudaStream_t st) {
  if (T > kAttnResidentMaxT) return attn_stream(fwd, qkv, dout, out_or_dqkv, stats, S, T, D, heads, st);
  return attn_dispatch(fwd, qkv, dout, out_or_dqkv, S, T, D, heads, st);
}

static int vit_attn_fwd(const bf16* qkv, bf16* out, int S, int T, int D, int heads, cudaStream_t st) {
  return vit_attn(true, qkv, nullptr, out, nullptr, S, T, D, heads, st);
}

GraphCacheRef::GraphCacheRef() : cache(new GraphCache) {}
GraphCacheRef::~GraphCacheRef() { delete cache; }
int GraphCacheRef::replay(int S, int flag, cudaStream_t& st, const std::function<int()>& body) { return cache->run(S, flag, st, body); }

int attn_resident(bool fwd, const bf16* qkv, const bf16* dout, bf16* out_or_dqkv, int S, int T, int D, int heads, cudaStream_t st) {
  return attn_dispatch(fwd, qkv, dout, out_or_dqkv, S, T, D, heads, st);
}

static Scratch& g_win = *new Scratch;   // aph_vit_bwd_sized: the R x R window gradient before k_window_expand

}  // namespace aph

using namespace aph;

extern "C" int aph_vit_create(aph_vit** out, const aph_vit_config* cfg) {
  APH_REQUIRE(out && cfg, "aph_vit_create: null argument");
  APH_REQUIRE(cfg->width % 128 == 0 && (cfg->width / 128 == 1 || cfg->width / 128 == 2 || cfg->width / 128 == 6 || cfg->width / 128 == 8),
              "aph_vit_create: width %d unsupported (128, 256, 768, 1024)", cfg->width);
  APH_REQUIRE(cfg->heads * 64 == cfg->width, "aph_vit_create: head dim must be 64 (width %d, heads %d)", cfg->width, cfg->heads);
  APH_REQUIRE(cfg->patch >= 2 && cfg->patch % 2 == 0 && cfg->res % cfg->patch == 0, "aph_vit_create: res %d / patch %d (the patch must be even)",
              cfg->res, cfg->patch);
  APH_REQUIRE(cfg->out_dim % 128 == 0 && cfg->max_batch > 0 && cfg->layers > 0, "aph_vit_create: out_dim %d must be a multiple of 128", cfg->out_dim);
  std::unique_ptr<VitImpl> v(new VitImpl());
  v->cfg = *cfg;
  v->g = cfg->res / cfg->patch; v->T = v->g * v->g + 1; v->D = cfg->width; v->Kp = patch_k(cfg->patch);
  const int D = v->D, T = v->T, S = cfg->max_batch, Ly = cfg->layers, O = cfg->out_dim;
  const size_t M = (size_t)S * T, Mp = (size_t)S * v->g * v->g;
  v->prefix = "visual.";
  int e = 0;
  // weights. conv1 [D, 3, p, p] = [D, 3 p^2] goes into the first 3 p^2 columns (rows of the transpose) of [D, Kp] / [Kp, D];
  // proj [D, out] is the data gradient's B operand as it is, the forward's transposed
  e |= v->add_bf16("conv1.weight", D, 3 * cfg->patch * cfg->patch, &v->w_conv, &v->w_conv_t, v->Kp);
  e |= v->add_f32("class_embedding", &v->cls, D); e |= v->add_f32("positional_embedding", &v->pos, (size_t)T * D);
  e |= v->add_f32("ln_pre.weight", &v->lnpre_w, D); e |= v->add_f32("ln_pre.bias", &v->lnpre_b, D);
  e |= v->add_f32("ln_post.weight", &v->lnpost_w, D); e |= v->add_f32("ln_post.bias", &v->lnpost_b, D);
  e |= v->add_bf16("proj", D, O, &v->w_out_t, &v->w_out);
  e |= add_blocks(v.get(), Ly, D, true);
  // activations
  e |= v->alloc(&v->patches, Mp * v->Kp); e |= v->alloc(&v->tok, Mp * D); e |= v->alloc(&v->e, M * D);
  v->xs.resize(2 * Ly + 1);
  for (int i = 0; i <= 2 * Ly; ++i) e |= v->alloc(&v->xs[i], (i >= 2 * Ly - 1 ? (size_t)S : M) * D);
  e |= v->alloc(&v->ln_out, M * D); e |= v->alloc(&v->attn_out, M * D); e |= v->alloc(&v->h_act, M * 4 * D);
  v->qkv.resize(Ly); v->h_pre.resize(Ly);
  for (int i = 0; i < Ly; ++i) { e |= v->alloc(&v->qkv[i], M * 3 * D); e |= v->alloc(&v->h_pre[i], (i == Ly - 1 ? (size_t)S : M) * 4 * D); }
  e |= v->alloc(&v->st_mean, stat_off(v.get(), 2 * Ly + 2)); e |= v->alloc(&v->st_rstd, stat_off(v.get(), 2 * Ly + 2));
  e |= v->alloc(&v->cls_ln, (size_t)S * D); e |= v->alloc(&v->emb_int, (size_t)S * O);
  e |= v->alloc(&v->d_emb, (size_t)S * O); e |= v->alloc(&v->d_cls, (size_t)S * D);
  e |= v->alloc(&v->dxc, (size_t)S * D); e |= v->alloc(&v->dxc_bf, (size_t)S * D);
  e |= v->alloc(&v->dx, M * D); e |= v->alloc(&v->dx_bf, M * D); e |= v->alloc(&v->dh, M * 4 * D);
  e |= v->alloc(&v->d_ln, M * D); e |= v->alloc(&v->d_attn, M * D); e |= v->alloc(&v->d_attn_last, M * D);
  e |= v->alloc(&v->d_qkv, M * 3 * D); e |= v->alloc(&v->d_tok, Mp * D);
  if (T > kAttnResidentMaxT) e |= v->alloc(&v->attn_stats, M * cfg->heads);
  if (e) return 1;
  APH_CUDA_OK(cudaMemset(v->d_attn_last, 0, M * D * sizeof(bf16)));
  if (v->Kp != 3 * cfg->patch * cfg->patch) {   // the zero padding of the patch operand and of conv1's packed weights
    APH_CUDA_OK(cudaMemset(v->patches, 0, Mp * v->Kp * sizeof(bf16)));
    APH_CUDA_OK(cudaMemset(v->w_conv, 0, (size_t)D * v->Kp * sizeof(bf16)));
    APH_CUDA_OK(cudaMemset(v->w_conv_t, 0, (size_t)D * v->Kp * sizeof(bf16)));
  }
  APH_CUDA_OK(cudaDeviceSynchronize());     // the zeros are in place before any caller stream (blocking or not) can read them
  *out = reinterpret_cast<aph_vit*>(v.release());
  return 0;
}

extern "C" int aph_vit_destroy(aph_vit* vit) {
  delete reinterpret_cast<VitImpl*>(vit);
  return 0;
}

extern "C" int64_t aph_vit_bytes(const aph_vit* vit) { return vit ? reinterpret_cast<const VitImpl*>(vit)->bytes : 0; }

extern "C" int aph_vit_load_tensor(aph_vit* vit, const char* key, const float* data, int64_t numel, void* stream) {
  return load_tensor(reinterpret_cast<VitImpl*>(vit), key, data, numel, (cudaStream_t)stream, "aph_vit_load_tensor");
}

extern "C" int aph_vit_finalize(aph_vit* vit) { return finalize(reinterpret_cast<VitImpl*>(vit), "aph_vit_finalize"); }

static int vit_fwd_impl(aph_vit* vit, const float* images, int S, int side, float* emb, int save_for_bwd, void* stream);
static int vit_bwd_impl(aph_vit* vit, const float* grad_emb, int S, int side, float* grad_images, void* stream);

extern "C" int aph_vit_fwd(aph_vit* vit, const float* images, int S, float* emb, int save_for_bwd, void* stream) {
  APH_REQUIRE(vit && images && emb, "aph_vit_fwd: null argument");
  return vit_fwd_impl(vit, images, S, reinterpret_cast<VitImpl*>(vit)->cfg.res, emb, save_for_bwd, stream);
}

// images of side res <= side < res + patch (the 232-pixel batches of transforms_custom / _elastic): conv1 sees the top-left window
static int check_side(const aph_vit* vit, int side, const char* who) {
  const VitImpl* v = reinterpret_cast<const VitImpl*>(vit);
  APH_REQUIRE(side >= v->cfg.res && side < v->cfg.res + v->cfg.patch, "%s: side=%d outside [%d, %d)", who, side, v->cfg.res, v->cfg.res + v->cfg.patch);
  return 0;
}

extern "C" int aph_vit_fwd_sized(aph_vit* vit, const float* images, int S, int side, float* emb, int save_for_bwd, void* stream) {
  APH_REQUIRE(vit && images && emb, "aph_vit_fwd_sized: null argument");
  if (int e = check_side(vit, side, "aph_vit_fwd_sized")) return e;
  return vit_fwd_impl(vit, images, S, side, emb, save_for_bwd, stream);
}

extern "C" int aph_vit_bwd_sized(aph_vit* vit, const float* grad_emb, int S, int side, float* grad_images, void* stream) {
  APH_REQUIRE(vit && grad_emb && grad_images, "aph_vit_bwd_sized: null argument");
  if (int e = check_side(vit, side, "aph_vit_bwd_sized")) return e;
  return vit_bwd_impl(vit, grad_emb, S, side, grad_images, stream);
}

// The sampler can write the patch-embedding operand itself (aph_sample_fwd_patches): this is where it goes ...
extern "C" int aph_vit_patch_operand(aph_vit* vit, int S, void** patches_bf16, int* patch, int* grid) {
  APH_REQUIRE(vit && patches_bf16 && patch && grid, "aph_vit_patch_operand: null argument");
  VitImpl* v = reinterpret_cast<VitImpl*>(vit);
  APH_REQUIRE(v->finalized, "aph_vit_patch_operand: weights not finalized");
  APH_REQUIRE(S > 0 && S <= v->cfg.max_batch, "aph_vit_patch_operand: S=%d outside (0, max_batch=%d]", S, v->cfg.max_batch);
  *patches_bf16 = v->patches; *patch = v->cfg.patch; *grid = v->g;
  return 0;
}

// ... and the forward that consumes it as it is (no k_patchify: the fp32 images are not read)
extern "C" int aph_vit_fwd_prepatched(aph_vit* vit, int S, float* emb, int save_for_bwd, void* stream) {
  APH_REQUIRE(vit && emb, "aph_vit_fwd_prepatched: null argument");
  return vit_fwd_impl(vit, nullptr, S, 0, emb, save_for_bwd, stream);
}

static int vit_fwd_impl(aph_vit* vit, const float* images, int S, int side, float* emb, int save_for_bwd, void* stream) {
  VitImpl* v = reinterpret_cast<VitImpl*>(vit);
  APH_REQUIRE(v->finalized, "aph_vit_fwd: weights not finalized");
  APH_REQUIRE(S > 0 && S <= v->cfg.max_batch, "aph_vit_fwd: S=%d outside (0, max_batch=%d]", S, v->cfg.max_batch);
  cudaStream_t st = (cudaStream_t)stream;
  // The only kernels that touch caller-owned memory (k_patchify reads `images`, the last copy writes `emb`) run OUTSIDE the cached
  // graph, so the graph is keyed on the batch size alone: a caller whose tensors move every step (clip_fft.py:285 calls
  // torch.cuda.empty_cache() per step) still replays it.
  if (images) {
    const int g = v->g, Mp = S * g * g;
    const int p = v->cfg.patch;
    if (v->Kp == 3 * p * p) {                // rows without padding (p = 16, 32): 8 columns per thread
      const size_t n8 = (size_t)Mp * v->Kp / 8;
      k_patchify<false><<<stride_blocks(n8, 16), 256, 0, st>>>(images, v->patches, S, p, g, side);
    } else {                                 // padded rows (p = 14): pixel pairs
      const size_t n2 = (size_t)Mp * 3 * p * p / 2;
      k_patchify<true><<<stride_blocks(n2, 16), 256, 0, st>>>(images, v->patches, S, p, g, side);
    }
    APH_LAUNCH_OK();
  }
  const int rc = v->fwd_graphs.run(S, save_for_bwd, st, [&]() -> int {
  const int D = v->D, T = v->T, g = v->g, Ly = v->cfg.layers, O = v->cfg.out_dim, H = v->cfg.heads;
  const int M = S * T, Mp = S * g * g;
  int e;
  // patch embedding
  {
    GemmEpi ep; ep.out_f32 = v->tok;
    if ((e = launch_gemm(v->patches, v->w_conv, GemmShape{Mp, D, v->Kp}, ep, st))) return e;
    NCH_DISPATCH(D, k_embed_lnpre<NCH><<<rows_grid(M), 256, 0, st>>>(v->tok, v->cls, v->pos, v->lnpre_w, v->lnpre_b, v->e, v->xs[0],
                                                                       v->st_mean, v->st_rstd, S, T, D));
    APH_LAUNCH_OK();
  }
  for (int l = 0; l < Ly; ++l) {
    // the last block runs on the cls rows after attention: out_proj reads rows s*T of attn_out and x_in (stride T*D)
    const bool last = l == Ly - 1;
    const BlockIO io{v->xs[2 * l], v->xs[2 * l + 1], v->xs[2 * l + 2], v->ln_out, v->qkv[l], v->attn_out, v->h_pre[l], v->h_act,
                     v->st_mean + stat_off(v, 1 + 2 * l), v->st_rstd + stat_off(v, 1 + 2 * l),
                     v->st_mean + stat_off(v, 2 + 2 * l), v->st_rstd + stat_off(v, 2 + 2 * l)};
    if ((e = block_fwd(v->L[l], io, S, T, last ? S : M, last ? T * D : 0, D, H, vit_attn_fwd, st))) return e;
  }
  {
    float* meanp = v->st_mean + stat_off(v, 2 * Ly + 1); float* rstdp = v->st_rstd + stat_off(v, 2 * Ly + 1);
    NCH_DISPATCH(D, k_ln_fwd<NCH><<<rows_grid(S), 256, 0, st>>>(v->xs[2 * Ly], v->lnpost_w, v->lnpost_b, v->cls_ln, meanp, rstdp, S, D));
    APH_LAUNCH_OK();
    GemmEpi ep; ep.out_f32 = v->emb_int;
    if ((e = launch_gemm(v->cls_ln, v->w_out, GemmShape{S, O, D}, ep, st))) return e;
  }
  return 0;
  });
  if (rc) return rc;
  APH_CUDA_OK(cudaMemcpyAsync(emb, v->emb_int, (size_t)S * v->cfg.out_dim * sizeof(float), cudaMemcpyDeviceToDevice, st));
  v->last_S = save_for_bwd ? S : -1;
  return 0;
}

extern "C" int aph_vit_bwd(aph_vit* vit, const float* grad_emb, int S, float* grad_images, void* stream) {
  APH_REQUIRE(vit && grad_emb && grad_images, "aph_vit_bwd: null argument");
  return vit_bwd_impl(vit, grad_emb, S, reinterpret_cast<VitImpl*>(vit)->cfg.res, grad_images, stream);
}

static int vit_bwd_impl(aph_vit* vit, const float* grad_emb, int S, int side, float* grad_images, void* stream) {
  VitImpl* v = reinterpret_cast<VitImpl*>(vit);
  APH_REQUIRE(v->last_S == S, "aph_vit_bwd: no saved forward for S=%d (last saved S=%d)", S, v->last_S);
  cudaStream_t st = (cudaStream_t)stream;
  {   // caller-owned input: converted outside the cached graph (see aph_vit_fwd)
    const size_t n = (size_t)S * v->cfg.out_dim;
    k_f32_to_bf16<<<stride_blocks(n, 8), 256, 0, st>>>(grad_emb, v->d_emb, n);
    APH_LAUNCH_OK();
  }
  const int rc = v->bwd_graphs.run(S, 0, st, [&]() -> int {
  const int D = v->D, T = v->T, Ly = v->cfg.layers, O = v->cfg.out_dim, H = v->cfg.heads;
  const int M = S * T;
  int e;
  {
    GemmEpi ep; ep.out_f32 = v->d_cls;
    if ((e = launch_gemm(v->d_emb, v->w_out_t, GemmShape{S, D, O}, ep, st))) return e;
    // ln_post: the gradient reaching the last block is non-zero on its cls rows only; it is kept compact in dxc / dxc_bf
    float* meanp = v->st_mean + stat_off(v, 2 * Ly + 1); float* rstdp = v->st_rstd + stat_off(v, 2 * Ly + 1);
    NCH_DISPATCH(D, k_ln_bwd<NCH><<<rows_grid(S), 256, 0, st>>>(v->d_cls, v->xs[2 * Ly], meanp, rstdp, v->lnpost_w, v->dxc, v->dxc_bf,
                                                                S, T, D, 0, 0, (const float*)nullptr));
    APH_LAUNCH_OK();
  }
  for (int l = Ly - 1; l >= 0; --l) {
    const BlockW& w = v->L[l];
    // the last block's MLP and out_proj run on its S cls rows: their gradient is dxc; d out_proj lands on rows s*T of d_attn_last
    const bool last = l == Ly - 1;
    const int Mr = last ? S : M;
    float* gx = last ? v->dxc : v->dx; bf16* gx_bf = last ? v->dxc_bf : v->dx_bf; bf16* d_attn = last ? v->d_attn_last : v->d_attn;
    float* x_in = v->xs[2 * l]; float* x_mid = v->xs[2 * l + 1];
    float* mean1 = v->st_mean + stat_off(v, 1 + 2 * l); float* rstd1 = v->st_rstd + stat_off(v, 1 + 2 * l);
    float* mean2 = v->st_mean + stat_off(v, 2 + 2 * l); float* rstd2 = v->st_rstd + stat_off(v, 2 + 2 * l);
    // MLP branch: dh = (dx . W_proj) * gelu'(h); d_ln2 = dh . W_fc
    { GemmEpi ep; ep.gelu_in = v->h_pre[l]; ep.out_bf16 = v->dh;
      if ((e = launch_gemm(gx_bf, w.w_proj_t, GemmShape{Mr, 4 * D, D}, ep, st))) return e; }
    { GemmEpi ep; ep.out_bf16 = v->d_ln;
      if ((e = launch_gemm(v->dh, w.w_fc_t, GemmShape{Mr, D, 4 * D}, ep, st))) return e; }
    NCH_DISPATCH(D, k_ln_bwd<NCH, bf16><<<rows_grid(Mr), 256, 0, st>>>(v->d_ln, x_mid, mean2, rstd2, w.ln2_w, gx, gx_bf, Mr, T, D, 0, 1,
                                                                       (const float*)nullptr));
    APH_LAUNCH_OK();
    // attention branch: d_attn = dx . W_o; (dq,dk,dv) = attn'(...); d_ln1 = d_qkv . W_qkv
    { GemmEpi ep; ep.out_bf16 = d_attn; ep.ld_out = last ? T * D : 0;
      if ((e = launch_gemm(gx_bf, w.w_o_t, GemmShape{Mr, D, D}, ep, st))) return e; }
    if ((e = vit_attn(false, v->qkv[l], d_attn, v->d_qkv, v->attn_stats, S, T, D, H, st))) return e;
    { GemmEpi ep; ep.out_bf16 = v->d_ln;
      if ((e = launch_gemm(v->d_qkv, w.w_qkv_t, GemmShape{M, D, 3 * D}, ep, st))) return e; }
    // ln_1: back to all M rows; in the last block dx is written here for the first time (+ dxc on the cls rows)
    NCH_DISPATCH(D, k_ln_bwd<NCH, bf16><<<rows_grid(M), 256, 0, st>>>(v->d_ln, x_in, mean1, rstd1, w.ln1_w, v->dx, v->dx_bf, M, T, D,
                                                                      last ? 1 : 0, 1, (const float*)(last ? v->dxc : nullptr)));
    APH_LAUNCH_OK();
  }
  // ln_pre backward (cls rows dropped) and patch-embed data gradient scattered back to NCHW
  NCH_DISPATCH(D, k_ln_bwd<NCH><<<rows_grid(M), 256, 0, st>>>(v->dx, v->e, v->st_mean, v->st_rstd, v->lnpre_w, nullptr, v->d_tok, M, T, D, 2, 0,
                                                              (const float*)nullptr));
  APH_LAUNCH_OK();
  return 0;
  });
  if (rc) return rc;
  // caller-owned output: the patch-embed data gradient (un-patchify epilogue writes NCHW) is launched outside the graph
  { const int g = v->g, Mp = S * g * g, R = v->cfg.res;
    // a larger image (aph_vit_bwd_sized): the epilogue writes the R x R window into a scratch image, k_window_expand places it
    // and zeroes the margin, which conv1 never reads
    const bool sized = side != R;
    if (sized)
      if (int e = g_win.grow((size_t)S * 3 * R * R * sizeof(float), st)) return e;
    GemmEpi ep; ep.out_f32 = sized ? g_win.p : grad_images; ep.unpatch_p = v->cfg.patch; ep.unpatch_g = g;
    if (int e = launch_gemm(v->d_tok, v->w_conv_t, GemmShape{Mp, v->Kp, v->D}, ep, st)) return e;
    if (sized) {
      const size_t n = (size_t)S * 3 * side * side;
      k_window_expand<<<stride_blocks(n, 16), 256, 0, st>>>((const float*)g_win.p, grad_images,
                                                            S * 3, R, side);
      APH_LAUNCH_OK();
    }
  }
  return 0;
}

namespace aph { int attn_causal_test(const bf16* qkv, bf16* out, int S, int T, int D, int heads, cudaStream_t st); }   // text.cu

// Test entries (tests/test_encoder_kernels_gpu.py): the encoder's attention and LayerNorm kernels on caller-supplied operands,
// dispatched exactly as the encoder (and, for causal attention, the text tower) dispatches them. aph_attn_test covers the
// resident kernels (T <= 256, the image tower's dispatch below the streaming kernels); aph_attn_long_test covers the streaming
// kernels the encoder runs for T > 256, at any T >= 1.
extern "C" int aph_attn_test(int fwd, int causal, const void* qkv, const void* dout, void* out, int S, int T, int D, int heads, void* stream) {
  APH_REQUIRE(qkv && out && (fwd || dout), "aph_attn_test: null argument");
  APH_REQUIRE(S > 0 && T > 0 && heads > 0 && D == 64 * heads, "aph_attn_test: S=%d T=%d D=%d heads=%d (head dim must be 64)", S, T, D, heads);
  const bf16* q = reinterpret_cast<const bf16*>(qkv);
  cudaStream_t st = (cudaStream_t)stream;
  if (causal) {
    APH_REQUIRE(fwd, "aph_attn_test: causal attention has no backward");
    return attn_causal_test(q, reinterpret_cast<bf16*>(out), S, T, D, heads, st);
  }
  return attn_dispatch(fwd != 0, q, reinterpret_cast<const bf16*>(dout), reinterpret_cast<bf16*>(out), S, T, D, heads, st);
}

extern "C" int aph_attn_long_test(int fwd, const void* qkv, const void* dout, void* out, int S, int T, int D, int heads, void* stream) {
  APH_REQUIRE(qkv && out && (fwd || dout), "aph_attn_long_test: null argument");
  APH_REQUIRE(S > 0 && T > 0 && heads > 0 && D == 64 * heads, "aph_attn_long_test: S=%d T=%d D=%d heads=%d (head dim must be 64)", S, T, D, heads);
  cudaStream_t st = (cudaStream_t)stream;
  const bf16* q = reinterpret_cast<const bf16*>(qkv);
  if (fwd) return attn_stream(true, q, nullptr, reinterpret_cast<bf16*>(out), nullptr, S, T, D, heads, st);
  StreamTemp<float2> stats;                  // freed behind the two backward launches
  if (int e = stats.alloc((size_t)S * heads * T, st)) return e;
  return attn_stream(false, q, reinterpret_cast<const bf16*>(dout), reinterpret_cast<bf16*>(out), stats.p, S, T, D, heads, st);
}

extern "C" int aph_ln_fwd_test(const float* x, const float* gamma, const float* beta, void* y, float* mean, float* rstd, int rows, int D,
                               void* stream) {
  APH_REQUIRE(x && gamma && beta && y && mean && rstd && rows > 0 && D % 128 == 0, "aph_ln_fwd_test: null argument or rows=%d D=%d", rows, D);
  NCH_DISPATCH(D, k_ln_fwd<NCH><<<rows_grid(rows), 256, 0, (cudaStream_t)stream>>>(x, gamma, beta, reinterpret_cast<bf16*>(y), mean, rstd, rows, D));
  APH_LAUNCH_OK();
  return 0;
}

extern "C" int aph_ln_bwd_test(const void* dy, int dy_bf16, const float* x, const float* mean, const float* rstd, const float* gamma, float* dx,
                               void* dx_bf16, int rows, int T, int D, int mode, int accumulate, const float* dcls, void* stream) {
  APH_REQUIRE(dy && x && mean && rstd && gamma && dx_bf16 && rows > 0 && T > 0 && D % 128 == 0, "aph_ln_bwd_test: null argument or rows=%d T=%d D=%d",
              rows, T, D);
  APH_REQUIRE(mode >= 0 && mode <= 2 && (mode == 2 || dx) && (mode != 1 || dcls), "aph_ln_bwd_test: mode %d needs dx%s", mode,
              mode == 1 ? " and dcls" : "");
  cudaStream_t st = (cudaStream_t)stream;
  bf16* dxb = reinterpret_cast<bf16*>(dx_bf16);
  if (dy_bf16)
    NCH_DISPATCH(D, k_ln_bwd<NCH, bf16><<<rows_grid(rows), 256, 0, st>>>(reinterpret_cast<const bf16*>(dy), x, mean, rstd, gamma, dx, dxb,
                                                                         rows, T, D, mode, accumulate, dcls))
  else
    NCH_DISPATCH(D, k_ln_bwd<NCH><<<rows_grid(rows), 256, 0, st>>>(reinterpret_cast<const float*>(dy), x, mean, rstd, gamma, dx, dxb,
                                                                   rows, T, D, mode, accumulate, dcls))
  APH_LAUNCH_OK();
  return 0;
}
