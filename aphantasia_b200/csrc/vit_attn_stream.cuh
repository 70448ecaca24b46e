// vit_attn_stream.cuh -- streaming tensor-core attention of the CLIP ViT for any sequence length (head dim 64), forward and
// backward. The image tower runs it for T > 256 (ViT-L/14: 16 x 16 patches + the class token = 257), where the resident
// kernels of vit_attn_tc.cuh, which keep a head's K and V (and, backward, its P and dS) in shared memory, no longer fit.
//
// softmax(Q K^T / 8) V per (sample, head). One CTA = 4 warps = one block of 64 query rows (forward, dQ) or of 64 keys (dK, dV);
// the other operand streams through shared memory in tiles of 64 rows, rows >= T zero-filled (load_tile64). Same operand
// layout as the resident kernels: qkv bf16 [S*T, 3*D] (q | k | v), out / dout bf16 [S*T, D], dqkv bf16 [S*T, 3*D].
//   forward : online softmax -- running row max and sum in registers (exp2, fp32); the accumulator O is rescaled by
//             exp2(m_old - m_new) whenever a key tile raises the max; keys >= T are masked to -inf.
//   backward: deterministic, no atomics: every output element is written by exactly one CTA, in a fixed summation order.
//     k_attn_bwd_stream_q  (per query block): pass 1 over the key tiles forms the row statistics lse = m + log2(sum) and
//                          delta = sum_j P_ij dP_ij (dP = dO V^T) online; pass 2 recomputes P and dS = P o (dP - delta) / 8
//                          and accumulates dQ = dS K. It saves (lse, delta) per row for the second kernel.
//     k_attn_bwd_stream_kv (per key block): walks the query tiles and recomputes P^T and dS^T from those statistics with
//                          the keys as the MMA rows, so dV = P^T dO and dK = dS^T Q accumulate in registers.
//   The statistics are recomputed by the backward rather than saved by the forward: the forward is also run without a
//   backward (save_for_bwd = 0, and the forward re-run of a stale backward), and one buffer of S * heads * T (lse, delta)
//   pairs, shared by all layers, is all the backward needs (the encoder handle owns it; about 6.6 MB at S = 200, ViT-L/14).
#pragma once
#include "vit_attn_tc.cuh"

namespace aph {

constexpr int kStreamRows = 64;                                    // query rows or keys per CTA and per streamed tile
constexpr size_t kStreamFwdSmem = (size_t)3 * kStreamRows * 128;  // Q, K, V tiles
constexpr size_t kStreamBwdSmem = (size_t)4 * kStreamRows * 128 + kStreamRows * sizeof(float2);   // 2 own + 2 streamed tiles, stats
static_assert(kStreamFwdSmem <= 48 * 1024 && kStreamBwdSmem <= 48 * 1024, "streaming attention: static shared memory above 48 KB");

__global__ void __launch_bounds__(128) k_attn_fwd_stream(const bf16* __restrict__ qkv, bf16* __restrict__ out, int T, int D, int heads) {
  __shared__ __align__(128) uint8_t sm[kStreamFwdSmem];
  uint8_t* Qs = sm; uint8_t* Ks = Qs + kStreamRows * 128; uint8_t* Vs = Ks + kStreamRows * 128;
  const int nb = (T + kStreamRows - 1) / kStreamRows;
  const int item = blockIdx.x / nb, q0 = (blockIdx.x - item * nb) * kStreamRows;
  const int s = item / heads, h = item - s * heads;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  const size_t ld = (size_t)3 * D;
  const bf16* base = qkv + (size_t)s * T * ld + h * 64;
  const uint32_t qs_a = smem_u32(Qs), ks_a = smem_u32(Ks), vs_a = smem_u32(Vs);
  const int r0 = warp * 16;
  const bool live = q0 + r0 < T;                                   // this warp has query rows (all warps take the barriers)
  load_tile64(Qs, base + (size_t)q0 * ld, ld, kStreamRows, T - q0, 128);
  uint32_t qa[4][4];
  float o[8][4];
  zero_acc(o);
  float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;       // l: this lane's share of the row sums
  for (int k0 = 0; k0 < T; k0 += kStreamRows) {
    if (k0 > 0) __syncthreads();                                   // the previous K / V tile is consumed
    load_tile64(Ks, base + D + (size_t)k0 * ld, ld, kStreamRows, T - k0, 128);
    load_tile64(Vs, base + 2 * D + (size_t)k0 * ld, ld, kStreamRows, T - k0, 128);
    __syncthreads();
    if (!live) continue;
    if (k0 == 0) load_a_frags(qa, qs_a, r0, lane);
    float c[8][4];
    float mx0 = -INFINITY, mx1 = -INFINITY;
#pragma unroll
    for (int n2 = 0; n2 < 4; ++n2) {
      qk_tile(c[2 * n2], c[2 * n2 + 1], qa, ks_a, n2 * 16, lane);
      mask_scale(c[2 * n2], c[2 * n2 + 1], k0 + n2 * 16, T, t, mx0, mx1);
    }
    // key k0 < T is in every tile, so the new maxima are finite; on the first tile m = -inf and the rescale factor is 0
    const float mn0 = fmaxf(m0, quad_max(mx0)), mn1 = fmaxf(m1, quad_max(mx1));
    const float a0 = exp2f(m0 - mn0), a1 = exp2f(m1 - mn1);
    m0 = mn0; m1 = mn1;
    l0 *= a0; l1 *= a1;
#pragma unroll
    for (int i = 0; i < 8; ++i) { o[i][0] *= a0; o[i][1] *= a0; o[i][2] *= a1; o[i][3] *= a1; }
    exp_rowsum(c, m0, m1, l0, l1);
    pv_acc<4>(o, c, vs_a, lane);
  }
  if (!live) return;
  const float i0 = 1.f / quad_sum(l0), i1 = 1.f / quad_sum(l1);
  store_frag(out, (size_t)s * T, D, h * 64, o, q0 + r0 + g, T, t, i0, i1);
}

// dQ and the row statistics of one query block. stats: float2 [S*heads, T] = (lse, delta) per query row (log2 domain).
__global__ void __launch_bounds__(128) k_attn_bwd_stream_q(const bf16* __restrict__ qkv, const bf16* __restrict__ dout, bf16* __restrict__ dqkv,
                                                           float2* __restrict__ stats, int T, int D, int heads) {
  __shared__ __align__(128) uint8_t sm[kStreamBwdSmem];
  uint8_t* Qs = sm; uint8_t* Gs = Qs + kStreamRows * 128; uint8_t* Ks = Gs + kStreamRows * 128; uint8_t* Vs = Ks + kStreamRows * 128;
  const int nb = (T + kStreamRows - 1) / kStreamRows;
  const int item = blockIdx.x / nb, q0 = (blockIdx.x - item * nb) * kStreamRows;
  const int s = item / heads, h = item - s * heads;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  const size_t ld = (size_t)3 * D;
  const bf16* base = qkv + (size_t)s * T * ld + h * 64;
  const uint32_t qs_a = smem_u32(Qs), gs_a = smem_u32(Gs), ks_a = smem_u32(Ks), vs_a = smem_u32(Vs);
  const int r0 = warp * 16, row0 = q0 + r0 + g, row1 = row0 + 8;
  const bool live = q0 + r0 < T;
  load_tile64(Qs, base + (size_t)q0 * ld, ld, kStreamRows, T - q0, 128);
  load_tile64(Gs, dout + ((size_t)s * T + q0) * D + h * 64, (size_t)D, kStreamRows, T - q0, 128);
  uint32_t qa[4][4], ga[4][4];
  // ---- pass 1: online row max, sum of exp and sum of exp * dP
  float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f, d0 = 0.f, d1 = 0.f;
  for (int k0 = 0; k0 < T; k0 += kStreamRows) {
    if (k0 > 0) __syncthreads();
    load_tile64(Ks, base + D + (size_t)k0 * ld, ld, kStreamRows, T - k0, 128);
    load_tile64(Vs, base + 2 * D + (size_t)k0 * ld, ld, kStreamRows, T - k0, 128);
    __syncthreads();
    if (!live) continue;
    if (k0 == 0) { load_a_frags(qa, qs_a, r0, lane); load_a_frags(ga, gs_a, r0, lane); }
    float c[8][4], e[8][4];
    float mx0 = -INFINITY, mx1 = -INFINITY;
#pragma unroll
    for (int n2 = 0; n2 < 4; ++n2) {
      qk_tile(c[2 * n2], c[2 * n2 + 1], qa, ks_a, n2 * 16, lane);
      qk_tile(e[2 * n2], e[2 * n2 + 1], ga, vs_a, n2 * 16, lane);
      mask_scale(c[2 * n2], c[2 * n2 + 1], k0 + n2 * 16, T, t, mx0, mx1);
    }
    const float mn0 = fmaxf(m0, quad_max(mx0)), mn1 = fmaxf(m1, quad_max(mx1));
    const float a0 = exp2f(m0 - mn0), a1 = exp2f(m1 - mn1);
    m0 = mn0; m1 = mn1;
    l0 *= a0; l1 *= a1; d0 *= a0; d1 *= a1;
#pragma unroll
    for (int n = 0; n < 8; ++n) {
      const float p0 = exp2f(c[n][0] - m0), p1 = exp2f(c[n][1] - m0), p2 = exp2f(c[n][2] - m1), p3 = exp2f(c[n][3] - m1);
      l0 += p0 + p1; l1 += p2 + p3;
      d0 += p0 * e[n][0] + p1 * e[n][1]; d1 += p2 * e[n][2] + p3 * e[n][3];
    }
  }
  float lse0 = 0.f, lse1 = 0.f, dl0 = 0.f, dl1 = 0.f;
  if (live) {
    l0 = quad_sum(l0); l1 = quad_sum(l1); d0 = quad_sum(d0); d1 = quad_sum(d1);
    lse0 = m0 + log2f(l0); lse1 = m1 + log2f(l1);
    dl0 = d0 / l0; dl1 = d1 / l1;                                  // delta_i = sum_j P_ij dP_ij
    float2* srow = stats + (size_t)item * T;
    if (t == 0 && row0 < T) srow[row0] = make_float2(lse0, dl0);
    if (t == 0 && row1 < T) srow[row1] = make_float2(lse1, dl1);
  }
  // ---- pass 2: P, dS (scaled by 1/8) and dQ = dS K
  float dq[8][4];
  zero_acc(dq);
  for (int k0 = 0; k0 < T; k0 += kStreamRows) {
    __syncthreads();
    load_tile64(Ks, base + D + (size_t)k0 * ld, ld, kStreamRows, T - k0, 128);
    load_tile64(Vs, base + 2 * D + (size_t)k0 * ld, ld, kStreamRows, T - k0, 128);
    __syncthreads();
    if (!live) continue;
#pragma unroll
    for (int n2 = 0; n2 < 4; ++n2) {
      float c0[4], c1[4], e0[4], e1[4];
      qk_tile(c0, c1, qa, ks_a, n2 * 16, lane);
      qk_tile(e0, e1, ga, vs_a, n2 * 16, lane);
      uint32_t da[4];
#pragma unroll
      for (int u = 0; u < 2; ++u) {
        const float* cc = u ? c1 : c0; const float* ee = u ? e1 : e0;
        const int cl = k0 + n2 * 16 + u * 8 + 2 * t;
        const float p0 = (cl < T) ? exp2f(cc[0] * kAttnScaleLog2 - lse0) : 0.f, p1 = (cl + 1 < T) ? exp2f(cc[1] * kAttnScaleLog2 - lse0) : 0.f;
        const float p2 = (cl < T) ? exp2f(cc[2] * kAttnScaleLog2 - lse1) : 0.f, p3 = (cl + 1 < T) ? exp2f(cc[3] * kAttnScaleLog2 - lse1) : 0.f;
        da[2 * u] = pack2(p0 * (ee[0] - dl0) * 0.125f, p1 * (ee[1] - dl0) * 0.125f);
        da[2 * u + 1] = pack2(p2 * (ee[2] - dl1) * 0.125f, p3 * (ee[3] - dl1) * 0.125f);
      }
      av_step(dq, da, ks_a, n2 * 16, lane);
    }
  }
  if (!live) return;
  store_frag(dqkv + (size_t)s * T * ld + h * 64, 0, ld, 0, dq, row0, T, t);
}

// dK and dV of one key block, from the statistics k_attn_bwd_stream_q saved. Each warp owns 16 keys as the rows of its MMAs:
// S^T = K Q^T and dP^T = V dO^T per streamed query tile, then dV += P^T dO and dK += dS^T Q straight from registers.
__global__ void __launch_bounds__(128) k_attn_bwd_stream_kv(const bf16* __restrict__ qkv, const bf16* __restrict__ dout, bf16* __restrict__ dqkv,
                                                            const float2* __restrict__ stats, int T, int D, int heads) {
  __shared__ __align__(128) uint8_t sm[kStreamBwdSmem];
  uint8_t* Ks = sm; uint8_t* Vs = Ks + kStreamRows * 128; uint8_t* Qs = Vs + kStreamRows * 128; uint8_t* Gs = Qs + kStreamRows * 128;
  float2* Ls = reinterpret_cast<float2*>(Gs + kStreamRows * 128);
  const int nb = (T + kStreamRows - 1) / kStreamRows;
  const int item = blockIdx.x / nb, k0 = (blockIdx.x - item * nb) * kStreamRows;
  const int s = item / heads, h = item - s * heads;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  const size_t ld = (size_t)3 * D;
  const bf16* base = qkv + (size_t)s * T * ld + h * 64;
  const bf16* gbase = dout + (size_t)s * T * D + h * 64;
  const float2* srow = stats + (size_t)item * T;
  const uint32_t ks_a = smem_u32(Ks), vs_a = smem_u32(Vs), qs_a = smem_u32(Qs), gs_a = smem_u32(Gs);
  const int r0 = warp * 16;
  const bool live = k0 + r0 < T;
  load_tile64(Ks, base + D + (size_t)k0 * ld, ld, kStreamRows, T - k0, 128);
  load_tile64(Vs, base + 2 * D + (size_t)k0 * ld, ld, kStreamRows, T - k0, 128);
  uint32_t ka[4][4], va[4][4];
  float dk[8][4], dv[8][4];
  zero_acc(dk); zero_acc(dv);
  for (int q0 = 0; q0 < T; q0 += kStreamRows) {
    if (q0 > 0) __syncthreads();
    load_tile64(Qs, base + (size_t)q0 * ld, ld, kStreamRows, T - q0, 128);
    load_tile64(Gs, gbase + (size_t)q0 * D, (size_t)D, kStreamRows, T - q0, 128);
    // query rows >= T: lse = +inf makes their P (and dS) exactly 0
    if (threadIdx.x < kStreamRows) Ls[threadIdx.x] = q0 + (int)threadIdx.x < T ? srow[q0 + threadIdx.x] : make_float2(INFINITY, 0.f);
    __syncthreads();
    if (!live) continue;
    if (q0 == 0) { load_a_frags(ka, ks_a, r0, lane); load_a_frags(va, vs_a, r0, lane); }
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
      float c0[4], c1[4], e0[4], e1[4];
      qk_tile(c0, c1, ka, qs_a, kk * 16, lane);                   // rows: keys r0 + g, + 8; columns: queries
      qk_tile(e0, e1, va, gs_a, kk * 16, lane);
      uint32_t pa[4], da[4];
#pragma unroll
      for (int u = 0; u < 2; ++u) {
        const float* cc = u ? c1 : c0; const float* ee = u ? e1 : e0;
        const int qc = kk * 16 + u * 8 + 2 * t;
        const float2 sa = Ls[qc], sb = Ls[qc + 1];
        const float p0 = exp2f(cc[0] * kAttnScaleLog2 - sa.x), p1 = exp2f(cc[1] * kAttnScaleLog2 - sb.x);
        const float p2 = exp2f(cc[2] * kAttnScaleLog2 - sa.x), p3 = exp2f(cc[3] * kAttnScaleLog2 - sb.x);
        pa[2 * u] = pack2(p0, p1); pa[2 * u + 1] = pack2(p2, p3);
        da[2 * u] = pack2(p0 * (ee[0] - sa.y) * 0.125f, p1 * (ee[1] - sb.y) * 0.125f);
        da[2 * u + 1] = pack2(p2 * (ee[2] - sa.y) * 0.125f, p3 * (ee[3] - sb.y) * 0.125f);
      }
      av_step(dv, pa, gs_a, kk * 16, lane);
      av_step(dk, da, qs_a, kk * 16, lane);
    }
  }
  if (!live) return;
  bf16* obase = dqkv + (size_t)s * T * ld + h * 64;
  const int key0 = k0 + r0 + g, key1 = key0 + 8;
#pragma unroll
  for (int dt = 0; dt < 8; ++dt) {
    const int col = dt * 8 + 2 * t;
    if (key0 < T) {
      *reinterpret_cast<__nv_bfloat162*>(obase + (size_t)key0 * ld + D + col) = __floats2bfloat162_rn(dk[dt][0], dk[dt][1]);
      *reinterpret_cast<__nv_bfloat162*>(obase + (size_t)key0 * ld + 2 * D + col) = __floats2bfloat162_rn(dv[dt][0], dv[dt][1]);
    }
    if (key1 < T) {
      *reinterpret_cast<__nv_bfloat162*>(obase + (size_t)key1 * ld + D + col) = __floats2bfloat162_rn(dk[dt][2], dk[dt][3]);
      *reinterpret_cast<__nv_bfloat162*>(obase + (size_t)key1 * ld + 2 * D + col) = __floats2bfloat162_rn(dv[dt][2], dv[dt][3]);
    }
  }
}

// Host launch: fwd = out bf16 [S*T, D]; backward = dqkv bf16 [S*T, 3*D] from dout, with stats float2 [S*heads*T] as scratch.
static int attn_stream(bool fwd, const bf16* qkv, const bf16* dout, bf16* out_or_dqkv, float2* stats, int S, int T, int D, int heads,
                       cudaStream_t st) {
  const size_t blocks = (size_t)S * heads * ((T + kStreamRows - 1) / kStreamRows);
  APH_REQUIRE(blocks < (1u << 31), "attention: S=%d T=%d heads=%d is too many blocks", S, T, heads);
  if (fwd) {
    k_attn_fwd_stream<<<(unsigned)blocks, 128, 0, st>>>(qkv, out_or_dqkv, T, D, heads);
    APH_LAUNCH_OK();
    return 0;
  }
  k_attn_bwd_stream_q<<<(unsigned)blocks, 128, 0, st>>>(qkv, dout, out_or_dqkv, stats, T, D, heads);
  APH_LAUNCH_OK();
  k_attn_bwd_stream_kv<<<(unsigned)blocks, 128, 0, st>>>(qkv, dout, out_or_dqkv, (const float2*)stats, T, D, heads);
  APH_LAUNCH_OK();
  return 0;
}

}  // namespace aph
