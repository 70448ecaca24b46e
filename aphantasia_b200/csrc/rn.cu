// rn.cu -- CLIP ResNet image encoder handle (RN50, RN101, RN50x4, RN50x16, RN50x64): forward and data-gradient on bf16 NHWC
// activations.
//
// Restates CLIP's ModifiedResNet in eval mode, with every BatchNorm folded into the convolution before it (on the host, in
// float64: aphantasia_b200/clip fold_resnet_state_dict), so each convolution here carries a weight and a bias. For width w
// (64 RN50 / RN101, 80 RN50x4, 96 RN50x16, 128 RN50x64) and input resolution r = 32 g:
//   stem     conv 3x3 / 2 (3 -> w/2) + ReLU, conv 3x3 (w/2 -> w/2) + ReLU, conv 3x3 (w/2 -> w) + ReLU, avgpool 2
//   stages   layers[i] bottlenecks of planes w << i (x 4 out); the first block of stages 2-4 has stride 2. Bottleneck:
//            y = relu(conv3(pool(relu(conv2(relu(conv1 x))))) + id), pool = avgpool(stride) when stride > 1,
//            id = downsample(pool(x)) (1x1 conv) when the stride or the width changes, else x
//   attnpool g^2 tokens of the g x g map, their mean prepended (T = g^2 + 1), + positional embedding; w/2-head attention (head
//            dim 64) queried by token 0; c_proj of its output
// Every channel count runs rounded up to a multiple of 64 (rc64): the host fold zero-pads the weights and biases, so the padded
// channels are exactly 0 after every bias, ReLU, residual and pool. RN50: the stem's 32 -> 64; RN50x4: 40 -> 64, 80 -> 128 and
// planes 80 -> 128, 160 -> 192; RN50x16: 48 -> 64, 96 -> 128 and planes 96 -> 128; RN50x64 runs unpadded. The blocks' outputs
// (4 planes) are multiples of 64 for every width.
// Kernels (sm_90a):
//   stem conv 1         k_conv3in_fwd / k_conv3in_bwd<2, w/2, IN_RAW> (nhwc.cu): fp32 SIMT (3 input channels, stride 2); they
//                       read the caller's fp32 crops and write its fp32 crop gradient, outside the cached graphs. They write
//                       64-channel rows, zero above w/2, so the two other stem convolutions run on zero-padded weights
//   3x3 convolutions    k_conv3x3_tc (conv_tc.cuh), forward CONV_BIAS_RELU, data gradient CONV_MASK (select by the ReLU output)
//   1x1 convolutions    launch_gemm on the NHWC tensor viewed as [pixels, C], epilogues EPI_BIAS_RELU / EPI_BIAS_RESID_RELU /
//                       EPI_BIAS_BF16 forward, EPI_MASK / EPI_MASK_RESID / EPI_BF16 data gradient
//   average pool        k_pool2<POOL_MEAN> (nhwc.cu), and its adjoint k_unpool2 (scale 1/4) fused with the select of the ReLU
//                       output below it
//   attention pool      k_rn_tokens_fwd / _bwd, the q/k/v GEMM, attn_resident at T = g^2 + 1 (50, 82, 145, 197), c_proj on
//                       the token-0 rows
// The data gradient of a block's input is selected by that input being > 0 in the epilogue of the GEMM that writes it: every
// block input is a ReLU output, except the first block's, the stem's average pool of a ReLU output, which is 0 exactly where its
// four inputs are, whose gradient the stem's own ReLU select then drops anyway.
#include "nhwc.cuh"
#include "encoder.cuh"

namespace aph {

// the channel count a layer runs at: c rounded up to a multiple of 64 (the 3x3 convolution's and the GEMM's N and K granule)
constexpr int rc64(int c) { return (c + 63) / 64 * 64; }

// ---- attention-pool tokens ----------------------------------------------------------------------------------------------
// x bf16 [S*P, C] (the last block's output, pixel-major; P = g^2) -> tok bf16 [S*(P+1), C]: row 0 = mean of the P rows + pos[0],
// row 1 + i = x[i] + pos[1 + i]; pos fp32 [P+1, C]. One item per (sample, 8 channels); the sum runs in fp32 in pixel order.
__global__ void __launch_bounds__(256) k_rn_tokens_fwd(const bf16* __restrict__ x, const float* __restrict__ pos, int S, int C, int P,
                                                       bf16* __restrict__ tok) {
  const int C8 = C / 8, T = P + 1;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < (size_t)S * C8; i += (size_t)gridDim.x * blockDim.x) {
    const int cv = (int)(i % C8), s = (int)(i / C8);
    float sum[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f}, f[8];
    for (int r = 0; r < P; ++r) {
      unpack_bf16x8(__ldg(reinterpret_cast<const uint4*>(x + ((size_t)s * P + r) * C) + cv), f);
      const float* pp = pos + (size_t)(1 + r) * C + 8 * cv;
#pragma unroll
      for (int j = 0; j < 8; ++j) { sum[j] += f[j]; f[j] += pp[j]; }
      reinterpret_cast<uint4*>(tok + ((size_t)s * T + 1 + r) * C)[cv] = pack_bf16x8(f);
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) sum[j] = sum[j] * (1.f / P) + pos[8 * cv + j];
    reinterpret_cast<uint4*>(tok + (size_t)s * T * C)[cv] = pack_bf16x8(sum);
  }
}

// the adjoint: dz bf16 [S*P, C] = x > 0 ? dtok[1 + i] + dtok[0] / P : 0 (x, the last block's output, is a ReLU output: the
// select is that block's ReLU, so dz is the gradient its backward starts from)
__global__ void __launch_bounds__(256) k_rn_tokens_bwd(const bf16* __restrict__ dtok, const bf16* __restrict__ x, int S, int C, int P,
                                                       bf16* __restrict__ dz) {
  const int C8 = C / 8, T = P + 1;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < (size_t)S * P * C8; i += (size_t)gridDim.x * blockDim.x) {
    const int cv = (int)(i % C8);
    const size_t row = i / C8;
    const int s = (int)(row / P), r = (int)(row % P);
    float g0[8], g[8], m[8];
    unpack_bf16x8(__ldg(reinterpret_cast<const uint4*>(dtok + (size_t)s * T * C) + cv), g0);
    unpack_bf16x8(__ldg(reinterpret_cast<const uint4*>(dtok + ((size_t)s * T + 1 + r) * C) + cv), g);
    unpack_bf16x8(__ldg(reinterpret_cast<const uint4*>(x) + i), m);
#pragma unroll
    for (int j = 0; j < 8; ++j) g[j] = m[j] > 0.f ? g[j] + g0[j] * (1.f / P) : 0.f;
    reinterpret_cast<uint4*>(dz)[i] = pack_bf16x8(g);
  }
}

// emb [S, O] = acc + bias (c_proj's bias; the GEMM writes the fp32 product)
__global__ void __launch_bounds__(256) k_rn_emb(const float* __restrict__ acc, const float* __restrict__ bias, int S, int O, float* __restrict__ emb) {
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < (size_t)S * O; i += (size_t)gridDim.x * blockDim.x)
    emb[i] = acc[i] + bias[i % O];
}

static int tokens_fwd(const bf16* x, const float* pos, int S, int C, int grid, bf16* tok, cudaStream_t st) {
  k_rn_tokens_fwd<<<stride_blocks((size_t)S * C / 8, 16), 256, 0, st>>>(x, pos, S, C, grid * grid, tok);
  APH_LAUNCH_OK();
  return 0;
}
static int tokens_bwd(const bf16* dtok, const bf16* x, int S, int C, int grid, bf16* dz, cudaStream_t st) {
  k_rn_tokens_bwd<<<stride_blocks((size_t)S * grid * grid * C / 8, 16), 256, 0, st>>>(dtok, x, S, C, grid * grid, dz);
  APH_LAUNCH_OK();
  return 0;
}

// the stem's map side (stride-2 conv, pad 1) and the side after each 2x2 pool
inline int rn_stem_side(int side) { return (side - 1) / 2 + 1; }

// The stem's first convolution for width 2 * cout, on caller buffers: its output rows are 64 channels wide, zero above cout.
static int stem_fwd(int cout, const float* x, int N, int side, const float* w, const float* b, bf16* out, cudaStream_t st) {
  switch (cout) {
    case 32: return launch_conv3in_fwd<2, 32, IN_RAW>(x, N, side, side, w, b, out, st);
    case 40: return launch_conv3in_fwd<2, 40, IN_RAW>(x, N, side, side, w, b, out, st);
    case 48: return launch_conv3in_fwd<2, 48, IN_RAW>(x, N, side, side, w, b, out, st);
    case 56: return launch_conv3in_fwd<2, 56, IN_RAW>(x, N, side, side, w, b, out, st);
    case 64: return launch_conv3in_fwd<2, 64, IN_RAW>(x, N, side, side, w, b, out, st);
  }
  set_error("rn stem: %d output channels unsupported (32, 40, 48, 56, 64)", cout);
  return 2;
}
static int stem_bwd(int cout, const bf16* dz, int N, int side, const float* w, float* grad, cudaStream_t st) {
  switch (cout) {
    case 32: return launch_conv3in_bwd<2, 32, IN_RAW>(dz, N, side, side, w, grad, st);
    case 40: return launch_conv3in_bwd<2, 40, IN_RAW>(dz, N, side, side, w, grad, st);
    case 48: return launch_conv3in_bwd<2, 48, IN_RAW>(dz, N, side, side, w, grad, st);
    case 56: return launch_conv3in_bwd<2, 56, IN_RAW>(dz, N, side, side, w, grad, st);
    case 64: return launch_conv3in_bwd<2, 64, IN_RAW>(dz, N, side, side, w, grad, st);
  }
  set_error("rn stem: %d output channels unsupported (32, 40, 48, 56, 64)", cout);
  return 2;
}

struct RnBlock {
  int cin, planes, E, stride, hin, hout;   // channel counts as run (cin, planes rounded up to 64); E = 4 x the real planes;
                                           // hin: the input map and the 3x3 conv's; hout = hin / stride
  bool down;
  bf16 *w1 = nullptr, *w1_t = nullptr, *w2 = nullptr, *w2_t = nullptr, *w3 = nullptr, *w3_t = nullptr, *wd = nullptr, *wd_t = nullptr;
  float *b1 = nullptr, *b2 = nullptr, *b3 = nullptr, *bd = nullptr;
  bf16 *r1 = nullptr, *r2 = nullptr, *y = nullptr;   // saved: the two ReLU outputs [S hin^2, planes], the output [S hout^2, E]
};

struct RnImpl : Weights {
  aph_rn_config cfg;
  int D = 0;                     // 32 width: the attention pool's width
  int grid = 0, T = 0;           // the final map's side res / 32 and the attention pool's tokens grid^2 + 1
  int side_min = 0, side_max = 0;   // [res - 1, res + 30]: the input sides whose final map is grid x grid
  int SC = 0;                    // the stem's output channels as run, rc64(width)
  std::vector<RnBlock> blocks;
  float *stem_w1 = nullptr, *stem_b1 = nullptr, *stem_b2 = nullptr, *stem_b3 = nullptr;
  bf16 *stem_w2 = nullptr, *stem_w2_t = nullptr, *stem_w3 = nullptr, *stem_w3_t = nullptr;
  float *pos = nullptr, *b_qkv = nullptr, *b_c = nullptr;
  bf16 *w_qkv = nullptr, *w_qkv_t = nullptr, *w_c = nullptr, *w_c_t = nullptr;
  // activations, sized for max_batch at side side_max
  bf16 *s1 = nullptr, *s2 = nullptr, *s3 = nullptr, *sp = nullptr;   // stem ReLU outputs [S h1^2, 64] (s3: SC) and its pool [S h0^2, SC]
  bf16* scratch[6] = {};         // [S emax] each: forward temporaries and the backward's gradients
  size_t emax = 0;               // per-crop elements of the largest map (the stem's)
  bf16 *tok = nullptr, *qkv = nullptr, *attn = nullptr;                 // [S*T, D], [S*T, 3D], [S*T, D]
  bf16 *d_attn = nullptr, *d_qkv = nullptr, *d_tok = nullptr;           // d_attn: zeroed at creation, only rows s*T are written
  float* emb_int = nullptr;      // [S, out_dim]
  bf16* d_emb = nullptr;         // [S, out_dim]
  int last_S = -1, last_side = -1;
  GraphCacheRef fwd_graphs, bwd_graphs;
};

// Lays out the blocks' shapes for input side `side` (the weights' shapes do not depend on it)
static void rn_shapes(RnImpl* h, int side) {
  int hin = rn_stem_side(side) / 2, cin = h->SC;
  size_t b = 0;
  for (int i = 0; i < 4; ++i)
    for (int j = 0; j < h->cfg.layers[i]; ++j, ++b) {
      RnBlock& k = h->blocks[b];
      k.cin = cin; k.planes = rc64(h->cfg.width << i); k.E = 4 * (h->cfg.width << i); k.stride = (i > 0 && j == 0) ? 2 : 1;
      k.down = k.stride > 1 || cin != k.E;
      k.hin = hin; k.hout = hin / k.stride;
      hin = k.hout; cin = k.E;
    }
}

// the launches of the forward between the stem's first convolution (s1) and the fp32 product of c_proj (emb_int)
static int rn_fwd_body(RnImpl* h, int S, int side, cudaStream_t st) {
  const int h1 = rn_stem_side(side), D = h->D, T = h->T, SC = h->SC;
  int e;
  ConvEpi ce;
  ce.bias = h->stem_b2; ce.out = h->s2;
  if ((e = launch_conv3x3(h->s1, h->stem_w2, S, h1, h1, 64, 64, CONV_BIAS_RELU, ce, st))) return e;
  ce.bias = h->stem_b3; ce.out = h->s3;
  if ((e = launch_conv3x3(h->s2, h->stem_w3, S, h1, h1, 64, SC, CONV_BIAS_RELU, ce, st))) return e;
  if ((e = launch_pool2(POOL_MEAN, h->s3, S, h1, h1, SC, h->sp, st))) return e;
  const bf16* x = h->sp;
  for (const RnBlock& k : h->blocks) {
    const int P = k.planes, E = k.E, Min = S * k.hin * k.hin, Mo = S * k.hout * k.hout;
    { GemmEpi ep; ep.bias = k.b1; ep.act = 2; ep.out_bf16 = k.r1;
      if ((e = launch_gemm(x, k.w1, GemmShape{Min, P, k.cin}, ep, st))) return e; }
    { ConvEpi c; c.bias = k.b2; c.out = k.r2;
      if ((e = launch_conv3x3(k.r1, k.w2, S, k.hin, k.hin, P, P, CONV_BIAS_RELU, c, st))) return e; }
    const bf16* a3 = k.r2;
    const bf16* id = x;
    if (k.stride > 1) {
      if ((e = launch_pool2(POOL_MEAN, k.r2, S, k.hin, k.hin, P, h->scratch[0], st))) return e;
      a3 = h->scratch[0];
    }
    if (k.down) {
      const bf16* xin = x;
      if (k.stride > 1) {
        if ((e = launch_pool2(POOL_MEAN, x, S, k.hin, k.hin, k.cin, h->scratch[1], st))) return e;
        xin = h->scratch[1];
      }
      GemmEpi ep; ep.bias = k.bd; ep.out_bf16 = h->scratch[2];
      if ((e = launch_gemm(xin, k.wd, GemmShape{Mo, E, k.cin}, ep, st))) return e;
      id = h->scratch[2];
    }
    { GemmEpi ep; ep.bias = k.b3; ep.act = 2; ep.resid_bf16 = id; ep.out_bf16 = k.y;
      if ((e = launch_gemm(a3, k.w3, GemmShape{Mo, E, P}, ep, st))) return e; }
    x = k.y;
  }
  if ((e = tokens_fwd(x, h->pos, S, D, h->grid, h->tok, st))) return e;
  { GemmEpi ep; ep.bias = h->b_qkv; ep.out_bf16 = h->qkv;
    if ((e = launch_gemm(h->tok, h->w_qkv, GemmShape{S * T, 3 * D, D}, ep, st))) return e; }
  if ((e = attn_resident(true, h->qkv, nullptr, h->attn, S, T, D, h->cfg.heads, st))) return e;
  // only token 0 is queried: c_proj reads rows s*T of the attention output
  GemmEpi ep; ep.out_f32 = h->emb_int;
  return launch_gemm(h->attn, h->w_c, GemmShape{S, h->cfg.out_dim, D}, ep, st, T * D);
}

// the launches of the backward from d_emb down to d (pre-ReLU stem conv 1 output), which it leaves in scratch[3]
static int rn_bwd_body(RnImpl* h, int S, int side, cudaStream_t st) {
  const int h1 = rn_stem_side(side), D = h->D, T = h->T, SC = h->SC;
  bf16* const* g = h->scratch;
  int e;
  // attention pool: the attention-output gradient is non-zero on the token-0 rows only (d_attn's other rows stay zero)
  { GemmEpi ep; ep.out_bf16 = h->d_attn; ep.ld_out = T * D;
    if ((e = launch_gemm(h->d_emb, h->w_c_t, GemmShape{S, D, h->cfg.out_dim}, ep, st))) return e; }
  if ((e = attn_resident(false, h->qkv, h->d_attn, h->d_qkv, S, T, D, h->cfg.heads, st))) return e;
  { GemmEpi ep; ep.out_bf16 = h->d_tok;
    if ((e = launch_gemm(h->d_qkv, h->w_qkv_t, GemmShape{S * T, D, 3 * D}, ep, st))) return e; }
  int cur = 0;   // g[cur]: d loss / d (the block's pre-ReLU sum), i.e. its output gradient selected by its ReLU
  if ((e = tokens_bwd(h->d_tok, h->blocks.back().y, S, D, h->grid, g[cur], st))) return e;
  for (int b = (int)h->blocks.size() - 1; b >= 0; --b) {
    const RnBlock& k = h->blocks[b];
    const bf16* x = b > 0 ? h->blocks[b - 1].y : h->sp;
    const int P = k.planes, E = k.E, Min = S * k.hin * k.hin, Mo = S * k.hout * k.hout;
    const bf16* dz = g[cur];
    bf16 *R = g[2], *U = g[3], *P1 = g[4], *Dp = g[5];   // Dp: the downsample input's gradient before the pool adjoint
    const bf16* rg = dz;                                     // the identity's gradient
    if (k.down) {
      GemmEpi ep; ep.out_bf16 = k.stride > 1 ? Dp : R;
      if ((e = launch_gemm(dz, k.wd_t, GemmShape{Mo, k.cin, E}, ep, st))) return e;
      if (k.stride > 1 && (e = launch_unpool2(Dp, nullptr, S, k.hin, k.hin, k.cin, 0.25f, R, st))) return e;
      rg = R;
    }
    if (k.stride > 1) {                                      // conv3's input was pool(relu2): adjoint, then relu2's select
      GemmEpi ep; ep.out_bf16 = P1;
      if ((e = launch_gemm(dz, k.w3_t, GemmShape{Mo, P, E}, ep, st))) return e;
      if ((e = launch_unpool2(P1, k.r2, S, k.hin, k.hin, P, 0.25f, U, st))) return e;
    } else {
      GemmEpi ep; ep.mask = k.r2; ep.out_bf16 = U;
      if ((e = launch_gemm(dz, k.w3_t, GemmShape{Mo, P, E}, ep, st))) return e;
    }
    { ConvEpi c; c.mask = k.r1; c.out = P1;
      if ((e = launch_conv3x3(U, k.w2_t, S, k.hin, k.hin, P, P, CONV_MASK, c, st))) return e; }
    // the block input's gradient, selected by the input (a ReLU output; see the top of the file)
    { GemmEpi ep; ep.mask = x; ep.resid_bf16 = rg; ep.out_bf16 = g[cur ^ 1];
      if ((e = launch_gemm(P1, k.w1_t, GemmShape{Min, k.cin, P}, ep, st))) return e; }
    cur ^= 1;
  }
  // stem: the pool's adjoint with relu3's select, then conv3 and conv2 backward with the selects of relu2 and relu1
  if ((e = launch_unpool2(g[cur], h->s3, S, h1, h1, SC, 0.25f, g[4], st))) return e;
  ConvEpi c;
  c.mask = h->s2; c.out = g[2];
  if ((e = launch_conv3x3(g[4], h->stem_w3_t, S, h1, h1, SC, 64, CONV_MASK, c, st))) return e;
  c.mask = h->s1; c.out = g[3];
  return launch_conv3x3(g[2], h->stem_w2_t, S, h1, h1, 64, 64, CONV_MASK, c, st);
}

}  // namespace aph

using namespace aph;

extern "C" int aph_rn_create(aph_rn** out, const aph_rn_config* cfg) {
  APH_REQUIRE(out && cfg, "aph_rn_create: null argument");
  APH_REQUIRE(cfg->width % 16 == 0 && cfg->width >= 64 && cfg->width <= 128 && cfg->heads * 2 == cfg->width,
              "aph_rn_create: width %d, heads %d unsupported (width a multiple of 16 in [64, 128], heads = width / 2: head dim 64)",
              cfg->width, cfg->heads);
  APH_REQUIRE(cfg->layers[0] > 0 && cfg->layers[1] > 0 && cfg->layers[2] > 0 && cfg->layers[3] > 0, "aph_rn_create: empty stage");
  APH_REQUIRE(cfg->out_dim % 128 == 0 && cfg->out_dim > 0 && cfg->max_batch > 0, "aph_rn_create: out_dim %d must be a multiple of 128",
              cfg->out_dim);
  APH_REQUIRE(cfg->res % 32 == 0 && cfg->res >= 224 && cfg->res <= 448, "aph_rn_create: res %d is not a multiple of 32 in [224, 448]",
              cfg->res);
  std::unique_ptr<RnImpl> h(new RnImpl());
  h->cfg = *cfg;
  h->D = 32 * cfg->width;
  h->grid = cfg->res / 32; h->T = h->grid * h->grid + 1;
  h->side_min = cfg->res - 1; h->side_max = cfg->res + 30;
  h->SC = rc64(cfg->width);
  const int D = h->D, O = cfg->out_dim, T = h->T, C1 = cfg->width / 2, SC = h->SC;
  const size_t S = (size_t)cfg->max_batch, MT = S * T;
  h->blocks.resize(cfg->layers[0] + cfg->layers[1] + cfg->layers[2] + cfg->layers[3]);
  rn_shapes(h.get(), h->side_max);
  int e = 0;
  // weights (BN folded): 1x1 convolutions [Co, Ci] and their transposes, 3x3 packed both ways, biases fp32
  e |= h->add_f32("conv1.weight", &h->stem_w1, (size_t)C1 * 27); e |= h->add_f32("conv1.bias", &h->stem_b1, C1);
  e |= h->add_conv3x3("conv2.weight", 64, 64, &h->stem_w2, &h->stem_w2_t); e |= h->add_f32("conv2.bias", &h->stem_b2, 64);
  e |= h->add_conv3x3("conv3.weight", SC, 64, &h->stem_w3, &h->stem_w3_t); e |= h->add_f32("conv3.bias", &h->stem_b3, SC);
  {
    size_t b = 0;
    for (int i = 0; i < 4; ++i)
      for (int j = 0; j < cfg->layers[i]; ++j, ++b) {
        RnBlock& k = h->blocks[b];
        const std::string p = "layer" + std::to_string(i + 1) + "." + std::to_string(j) + ".";
        const int P = k.planes, E = k.E;
        e |= h->add_bf16(p + "conv1.weight", P, k.cin, &k.w1, &k.w1_t); e |= h->add_f32(p + "conv1.bias", &k.b1, P);
        e |= h->add_conv3x3(p + "conv2.weight", P, P, &k.w2, &k.w2_t); e |= h->add_f32(p + "conv2.bias", &k.b2, P);
        e |= h->add_bf16(p + "conv3.weight", E, P, &k.w3, &k.w3_t); e |= h->add_f32(p + "conv3.bias", &k.b3, E);
        if (k.down) { e |= h->add_bf16(p + "downsample.weight", E, k.cin, &k.wd, &k.wd_t); e |= h->add_f32(p + "downsample.bias", &k.bd, E); }
        e |= h->alloc(&k.r1, S * k.hin * k.hin * P); e |= h->alloc(&k.r2, S * k.hin * k.hin * P);
        e |= h->alloc(&k.y, S * k.hout * k.hout * E);
      }
  }
  e |= h->add_f32("attnpool.positional_embedding", &h->pos, (size_t)T * D);
  e |= h->add_bf16("attnpool.qkv.weight", 3 * D, D, &h->w_qkv, &h->w_qkv_t); e |= h->add_f32("attnpool.qkv.bias", &h->b_qkv, 3 * D);
  e |= h->add_bf16("attnpool.c_proj.weight", O, D, &h->w_c, &h->w_c_t); e |= h->add_f32("attnpool.c_proj.bias", &h->b_c, O);
  // activations
  const size_t h1 = rn_stem_side(h->side_max), h0 = h1 / 2;
  h->emax = h1 * h1 * SC;
  for (const RnBlock& k : h->blocks) {
    h->emax = std::max(h->emax, (size_t)k.hin * k.hin * std::max(k.cin, k.planes));
    h->emax = std::max(h->emax, (size_t)k.hout * k.hout * k.E);
  }
  e |= h->alloc(&h->s1, S * h1 * h1 * 64); e |= h->alloc(&h->s2, S * h1 * h1 * 64); e |= h->alloc(&h->s3, S * h1 * h1 * SC);
  e |= h->alloc(&h->sp, S * h0 * h0 * SC);
  for (bf16*& p : h->scratch) e |= h->alloc(&p, S * h->emax);
  e |= h->alloc(&h->tok, MT * D); e |= h->alloc(&h->qkv, MT * 3 * D); e |= h->alloc(&h->attn, MT * D);
  e |= h->alloc(&h->d_attn, MT * D); e |= h->alloc(&h->d_qkv, MT * 3 * D); e |= h->alloc(&h->d_tok, MT * D);
  e |= h->alloc(&h->emb_int, S * O); e |= h->alloc(&h->d_emb, S * O);
  if (e) return 1;
  APH_CUDA_OK(cudaMemset(h->d_attn, 0, MT * D * sizeof(bf16)));
  APH_CUDA_OK(cudaDeviceSynchronize());     // the zeros are in place before any caller stream (blocking or not) can read them
  *out = reinterpret_cast<aph_rn*>(h.release());
  return 0;
}

extern "C" int aph_rn_destroy(aph_rn* h) {
  delete reinterpret_cast<RnImpl*>(h);
  return 0;
}

extern "C" int64_t aph_rn_bytes(const aph_rn* h) { return h ? reinterpret_cast<const RnImpl*>(h)->bytes : 0; }

extern "C" int aph_rn_load_tensor(aph_rn* h, const char* key, const float* data, int64_t numel, void* stream) {
  return load_tensor(reinterpret_cast<RnImpl*>(h), key, data, numel, (cudaStream_t)stream, "aph_rn_load_tensor");
}

extern "C" int aph_rn_finalize(aph_rn* h) { return finalize(reinterpret_cast<RnImpl*>(h), "aph_rn_finalize"); }

static int rn_check(const RnImpl* h, int S, int side, const char* who) {
  APH_REQUIRE(h->finalized, "%s: weights not finalized", who);
  APH_REQUIRE(S > 0 && S <= h->cfg.max_batch, "%s: S=%d outside (0, max_batch=%d]", who, S, h->cfg.max_batch);
  APH_REQUIRE(side >= h->side_min && side <= h->side_max, "%s: side=%d outside [%d, %d] (the sides whose final map is %d x %d)", who,
              side, h->side_min, h->side_max, h->grid, h->grid);
  return 0;
}

extern "C" int aph_rn_fwd(aph_rn* rn, const float* x, int S, int side, float* emb, int save_for_bwd, void* stream) {
  APH_REQUIRE(rn && x && emb, "aph_rn_fwd: null argument");
  RnImpl* h = reinterpret_cast<RnImpl*>(rn);
  if (int e = rn_check(h, S, side, "aph_rn_fwd")) return e;
  cudaStream_t st = (cudaStream_t)stream;
  h->last_S = h->last_side = -1;
  rn_shapes(h, side);
  // the kernels that touch caller memory run outside the cached graph (see aph_vit_fwd)
  if (int e = stem_fwd(h->cfg.width / 2, x, S, side, h->stem_w1, h->stem_b1, h->s1, st)) return e;
  // the graph is keyed on the side alone: the forward's launches are the same with or without save_for_bwd
  if (int e = h->fwd_graphs.replay(S, side, st, [&]() { return rn_fwd_body(h, S, side, st); })) return e;
  const int O = h->cfg.out_dim;
  k_rn_emb<<<stride_blocks((size_t)S * O, 8), 256, 0, st>>>(h->emb_int, h->b_c, S, O, emb);
  APH_LAUNCH_OK();
  if (save_for_bwd) { h->last_S = S; h->last_side = side; }
  return 0;
}

extern "C" int aph_rn_bwd(aph_rn* rn, const float* grad_emb, int S, int side, float* grad_x, void* stream) {
  APH_REQUIRE(rn && grad_emb && grad_x, "aph_rn_bwd: null argument");
  RnImpl* h = reinterpret_cast<RnImpl*>(rn);
  if (int e = rn_check(h, S, side, "aph_rn_bwd")) return e;
  APH_REQUIRE(h->last_S == S && h->last_side == side, "aph_rn_bwd: no saved forward for S=%d side=%d (last saved: S=%d side=%d)", S, side,
              h->last_S, h->last_side);
  cudaStream_t st = (cudaStream_t)stream;
  rn_shapes(h, side);
  const size_t n = (size_t)S * h->cfg.out_dim;
  k_f32_to_bf16<<<stride_blocks(n, 8), 256, 0, st>>>(grad_emb, h->d_emb, n);
  APH_LAUNCH_OK();
  if (int e = h->bwd_graphs.replay(S, side, st, [&]() { return rn_bwd_body(h, S, side, st); })) return e;
  return stem_bwd(h->cfg.width / 2, h->scratch[3], S, side, h->stem_w1, grad_x, st);
}

// The forward's saved ReLU outputs, for a float64 backward that takes the CUDA forward's own selects: k = 0, 1, 2 the stem's
// [S, h1, h1, 64], [S, h1, h1, 64] and [S, h1, h1, SC] (channels from width / 2, resp. width, on zero), then 3 b + 3, 3 b + 4,
// 3 b + 5 block b's conv1 and conv2 outputs [S, hin, hin, P] (P = rc64(planes)) and its output [S, hout, hout, 4 planes], all
// bf16 NHWC at the side of the last forward. *ptr is the handle's buffer (valid until the
// next forward); *numel its element count at that side.
extern "C" int aph_rn_saved_test(aph_rn* rn, int k, void** ptr, int64_t* numel) {
  APH_REQUIRE(rn && ptr && numel, "aph_rn_saved_test: null argument");
  RnImpl* h = reinterpret_cast<RnImpl*>(rn);
  APH_REQUIRE(h->last_S > 0, "aph_rn_saved_test: no saved forward");
  const int nb = (int)h->blocks.size();
  APH_REQUIRE(k >= 0 && k < 3 + 3 * nb, "aph_rn_saved_test: k=%d outside [0, %d)", k, 3 + 3 * nb);
  rn_shapes(h, h->last_side);
  const int64_t S = h->last_S, h1 = rn_stem_side(h->last_side);
  if (k < 3) {
    *ptr = k == 0 ? h->s1 : k == 1 ? h->s2 : h->s3;
    *numel = S * h1 * h1 * (k == 2 ? h->SC : 64);
    return 0;
  }
  const RnBlock& b = h->blocks[(k - 3) / 3];
  const int j = (k - 3) % 3;
  *ptr = j == 0 ? b.r1 : j == 1 ? b.r2 : b.y;
  *numel = j < 2 ? S * b.hin * b.hin * b.planes : S * b.hout * b.hout * b.E;
  return 0;
}

// ---- test entries (tests/test_clip_resnet_gpu.py) ----------------------------------------------------------------
// Stem conv 1 on caller buffers, cout output channels (0: 32): weight fp32 [cout,3,3,3], bias [cout]. fwd = 1: in = crops fp32
// [N,3,side,side] -> out bf16 [N,h,h,64] (ReLU output; channels cout-63 zero), h = (side - 1) / 2 + 1; fwd = 0: in = dz bf16
// [N,h,h,64] -> out fp32 [N,3,side,side].
extern "C" int aph_rn_stem_test(int fwd, const void* in, const float* weight, const float* bias, void* out, int N, int side, void* stream,
                                int cout) {
  APH_REQUIRE(in && weight && out && (bias || !fwd) && N > 0 && side > 0, "aph_rn_stem_test: bad arguments");
  cudaStream_t st = (cudaStream_t)stream;
  if (cout == 0) cout = 32;
  if (fwd) return stem_fwd(cout, reinterpret_cast<const float*>(in), N, side, weight, bias, reinterpret_cast<bf16*>(out), st);
  return stem_bwd(cout, reinterpret_cast<const bf16*>(in), N, side, weight, reinterpret_cast<float*>(out), st);
}

// 2x2 average pool, bf16 NHWC, C % 8 == 0. fwd = 1: out [N,H/2,W/2,C] = pool(x); fwd = 0: x = dy [N,H/2,W/2,C] -> out [N,H,W,C]
// = its adjoint, selected by mask [N,H,W,C] > 0 when mask is not NULL.
extern "C" int aph_rn_pool_test(int fwd, const void* x, const void* mask, void* out, int N, int H, int W, int C, void* stream) {
  APH_REQUIRE(x && out && N > 0 && H >= 2 && W >= 2 && C % 8 == 0 && C > 0, "aph_rn_pool_test: bad arguments");
  cudaStream_t st = (cudaStream_t)stream;
  if (fwd) return launch_pool2(POOL_MEAN, reinterpret_cast<const bf16*>(x), N, H, W, C, reinterpret_cast<bf16*>(out), st);
  return launch_unpool2(reinterpret_cast<const bf16*>(x), reinterpret_cast<const bf16*>(mask), N, H, W, C, 0.25f, reinterpret_cast<bf16*>(out), st);
}

// Attention-pool tokens of a grid x grid map (grid 0: 7), P = grid^2, C % 8 == 0. fwd = 1: in = x bf16 [S*P, C], aux = pos fp32
// [P+1, C] -> out bf16 [S*(P+1), C]; fwd = 0: in = dtok bf16 [S*(P+1), C], aux = x bf16 [S*P, C] (the select) -> out bf16 [S*P, C].
extern "C" int aph_rn_tokens_test(int fwd, const void* in, const void* aux, void* out, int S, int C, void* stream, int grid) {
  if (grid == 0) grid = 7;
  APH_REQUIRE(in && aux && out && S > 0 && C % 8 == 0 && C > 0 && grid > 0, "aph_rn_tokens_test: bad arguments");
  cudaStream_t st = (cudaStream_t)stream;
  if (fwd) return tokens_fwd(reinterpret_cast<const bf16*>(in), reinterpret_cast<const float*>(aux), S, C, grid, reinterpret_cast<bf16*>(out), st);
  return tokens_bwd(reinterpret_cast<const bf16*>(in), reinterpret_cast<const bf16*>(aux), S, C, grid, reinterpret_cast<bf16*>(out), st);
}
