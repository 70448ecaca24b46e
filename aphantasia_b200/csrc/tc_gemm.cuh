// tc_gemm.cuh -- the wgmma / TMA GEMM of the CLIP ViT encoder (sm_90a).
//
//   C[M,N] = A[M,K] . B[N,K]^T      A, B bf16 row-major (K contiguous = "K-major"), fp32 accumulate in registers.
//
// Persistent, warp-specialised, one CTA of three warpgroups per SM, tile 128 x BN (BN = 128 or 256):
//   warpgroup 0 (1 lane)  TMA producer : cp.async.bulk.tensor.2d -> 128B-swizzled smem stages, mbarrier complete_tx
//   warpgroups 1, 2       consumers    : wgmma.mma_async with both operands read from shared memory through descriptors,
//                                        then the fused epilogue from registers
// Two consumer schedules (launch_gemm picks one from the shape):
//   cooperative  both consumers work on every tile, rows 0-63 / 64-127 (m64nBNk16); the producer runs ahead into the next
//                tile's stages while they store the current one. BN = 256 for large problems with long K, BN = 128 for
//                small problems.
//   ping-pong    BN = 128; each consumer owns every other tile whole (two m64n128k16 per k16) and the two take turns in the
//                main loop, so one stores its tile while the other's MMAs run (large problems with short K).
// The producer gives its registers to the consumers (setmaxnreg). Fused epilogues (struct GemmEpi): +bias, QuickGELU (saving
// the pre-activation), x gelu'(h) for the MLP backward, +fp32 residual, fp32 or bf16 outputs, and an NCHW "un-patchify" store
// for the patch-embed data gradient. bf16 outputs are stored 16 B per lane after an exchange inside each quad of lanes.
// Rows >= M are zero-filled by TMA on load and not stored. A, the residual and the outputs may have a row stride larger than
// their width (the encoder's last block reads and writes the class-token rows s*T of token-major matrices in place).
#pragma once
#include "aph_common.cuh"
#include <cuda.h>

namespace aph {

typedef __nv_bfloat16 bf16;

struct GemmEpi {
  const float* bias = nullptr;     // [N]
  const float* resid = nullptr;    // fp32 [M, N], added last
  const bf16* gelu_in = nullptr;   // bf16 [M, N]: acc *= quickgelu'(gelu_in)
  float* out_f32 = nullptr;        // fp32 [M, N] (or NCHW images when unpatch_p > 0)
  bf16* out_bf16 = nullptr;        // bf16 [M, N]
  bf16* out_pre = nullptr;         // bf16 [M, N] pre-activation (acc + bias), saved for backward
  int act = 0;                     // 1 = QuickGELU x*sigmoid(1.702x)
  int unpatch_p = 0;               // >0: out_f32 is [S,3,R,R]; row = s*g*g + gy*g + gx, col = c*p*p + py*p + px (cols >= 3p^2 dropped)
  int unpatch_g = 0;
  // row strides in elements, 0 = N (dense). ld_out covers out_f32 / out_bf16 / out_pre and gelu_in, which has the output's rows.
  // A strided output leaves the rows between its rows untouched (the encoder's last block writes only the class-token rows).
  int ld_resid = 0;
  int ld_out = 0;
};

struct GemmShape { int M, N, K; };

constexpr int GEMM_BM = 128;
constexpr int GEMM_BK = 64;       // 64 bf16 = 128 B = one swizzle-128B row
constexpr int GEMM_UK = 16;       // K per wgmma (bf16)
constexpr int GEMM_THREADS = 3 * 128;   // warpgroup 0: TMA producer; warpgroups 1-2: MMA + epilogue

// compile-time epilogue kinds (a runtime-flag epilogue is a long predicated body in the hot loop)
enum : int {
  EPI_F32 = 0,            // out_f32 = acc
  EPI_BF16 = 1,           // out_bf16 = acc
  EPI_BIAS_BF16 = 2,      // out_bf16 = acc + bias
  EPI_BIAS_GELU = 3,      // out_pre = bf16(acc + bias); out_bf16 = quickgelu(acc + bias)
  EPI_BIAS_RESID = 4,     // out_f32 = acc + bias + resid
  EPI_GELUGRAD_BF16 = 5,  // out_bf16 = acc * quickgelu'(gelu_in)
  EPI_UNPATCH = 6,        // out_f32[NCHW] = acc (patch-embed data gradient)
  EPI_KINDS = 7
};

// ---- raw PTX wrappers -------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  uint32_t done;
  do {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(done) : "r"(smem_u32(bar)), "r"(parity) : "memory");
  } while (!done);
}
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }

__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
// 2-D tile load: coordinates (x = element index along K, y = row)
__device__ __forceinline__ void tma_load_2d(void* dst, const CUtensorMap* m, uint64_t* bar, int x, int y) {
  asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
               ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(x), "r"(y) : "memory");
}
// 3-D tile load (x = column, y = token, z = sample); out-of-bounds tokens are zero-filled
__device__ __forceinline__ void tma_load_3d(uint32_t dst_saddr, const CUtensorMap* m, uint64_t* bar, int x, int y, int z) {
  asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
               ::"r"(dst_saddr), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(x), "r"(y), "r"(z) : "memory");
}
// 4-D tile load (x = channel, y = column, z = row, w = image) of an NHWC activation; coordinates may be negative or past the
// edge: those elements arrive zero-filled (the 3x3 convolution's padding, conv_tc.cuh)
__device__ __forceinline__ void tma_load_4d(void* dst, const CUtensorMap* m, uint64_t* bar, int x, int y, int z, int w) {
  asm volatile("cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
               ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(x), "r"(y), "r"(z), "r"(w) : "memory");
}
// same with an L2 eviction-priority hint (weights are re-read by every M tile: evict_last)
__device__ __forceinline__ void tma_load_2d_hint(void* dst, const CUtensorMap* m, uint64_t* bar, int x, int y, uint64_t policy) {
  asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1, {%3, %4}], [%2], %5;"
               ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(x), "r"(y), "l"(policy) : "memory");
}
__device__ __forceinline__ uint64_t l2_policy_evict_last() {
  uint64_t p;
  asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(p));
  return p;
}

// K-major, 128B-swizzled operand tile: rows of 128 B, 8-row groups 1024 B apart (SBO). sm_90 wgmma descriptor.
__device__ __forceinline__ uint64_t make_smem_desc(uint32_t saddr) {
  uint64_t d = 0;
  d |= (uint64_t)((saddr & 0x3FFFF) >> 4);        // start address, bits [0,14)
  d |= (uint64_t)1 << 16;                          // leading byte offset (unused for swizzled K-major)
  d |= (uint64_t)(1024 >> 4) << 32;                // stride byte offset, bits [32,46)
  d |= (uint64_t)1 << 62;                          // layout type: SWIZZLE_128B
  return d;
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N> __device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
template <int R> __device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(R)); }
template <int R> __device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(R)); }

// D[64 x BN] (+)= A[64 x 16] . B[BN x 16]^T, fp32 accumulators d[BN/2] in the m64nNk16 fragment layout
template <int BN> struct Wgmma;
#define APH_WG_REGS8(o) "+f"(d[o]), "+f"(d[o + 1]), "+f"(d[o + 2]), "+f"(d[o + 3]), "+f"(d[o + 4]), "+f"(d[o + 5]), "+f"(d[o + 6]), "+f"(d[o + 7])
template <> struct Wgmma<64> {      // the 64-channel layers of the LPIPS VGG (conv_tc.cuh)
  static __device__ __forceinline__ void mma(float (&d)[32], uint64_t da, uint64_t db, int acc) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, "
        "%24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, 0, 0;\n\t}"
        : APH_WG_REGS8(0), APH_WG_REGS8(8), APH_WG_REGS8(16), APH_WG_REGS8(24)
        : "l"(da), "l"(db), "r"(acc));
  }
};
template <> struct Wgmma<128> {
  static __device__ __forceinline__ void mma(float (&d)[64], uint64_t da, uint64_t db, int acc) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, "
        "%24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
        "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, 0, 0;\n\t}"
        : APH_WG_REGS8(0), APH_WG_REGS8(8), APH_WG_REGS8(16), APH_WG_REGS8(24), APH_WG_REGS8(32), APH_WG_REGS8(40), APH_WG_REGS8(48), APH_WG_REGS8(56)
        : "l"(da), "l"(db), "r"(acc));
  }
};
template <> struct Wgmma<256> {
  static __device__ __forceinline__ void mma(float (&d)[128], uint64_t da, uint64_t db, int acc) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %130, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n256k16.f32.bf16.bf16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, "
        "%24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
        "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, %68, %69, %70, %71, "
        "%72, %73, %74, %75, %76, %77, %78, %79, %80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, "
        "%96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, %112, %113, %114, %115, "
        "%116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127}, %128, %129, p, 1, 1, 0, 0;\n\t}"
        : APH_WG_REGS8(0), APH_WG_REGS8(8), APH_WG_REGS8(16), APH_WG_REGS8(24), APH_WG_REGS8(32), APH_WG_REGS8(40), APH_WG_REGS8(48), APH_WG_REGS8(56),
          APH_WG_REGS8(64), APH_WG_REGS8(72), APH_WG_REGS8(80), APH_WG_REGS8(88), APH_WG_REGS8(96), APH_WG_REGS8(104), APH_WG_REGS8(112), APH_WG_REGS8(120)
        : "l"(da), "l"(db), "r"(acc));
  }
};
#undef APH_WG_REGS8

// sigmoid(1.702 x) through ONE special-function op: 0.5 tanh(0.851 x) + 0.5 (tanh.approx: max rel. error 2^-11, far inside
// the bf16 rounding of the value it feeds); the epilogues of the MLP GEMMs are MUFU-limited otherwise (exp + rcp per element)
__device__ __forceinline__ float sigmoid1702(float x) {
  float t;
  asm("tanh.approx.f32 %0, %1;" : "=f"(t) : "f"(0.851f * x));
  return fmaf(0.5f, t, 0.5f);
}
__device__ __forceinline__ float quickgelu(float x) { return x * sigmoid1702(x); }
__device__ __forceinline__ float quickgelu_grad(float x) {
  const float s = sigmoid1702(x);
  return s * (1.f + 1.702f * x * (1.f - s));
}
__device__ __forceinline__ uint32_t pack_bf16(float lo, float hi) {
  __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&v);
}

template <int BN>
struct GemmCfg {
  static constexpr int A_BYTES = GEMM_BM * GEMM_BK * 2;
  static constexpr int B_BYTES = BN * GEMM_BK * 2;
  static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
  static constexpr int STAGES = (BN == 256) ? 4 : 6;              // 192 KB of operand stages either way
  static constexpr int BAR_OFFSET = STAGES * STAGE_BYTES;
  static constexpr int SMEM = BAR_OFFSET + 2 * STAGES * 8 + 1024;  // + alignment slack
};

// named barriers of the two consumer warpgroups (256 threads; id 0 is __syncthreads): consumer c syncs on 1 + c before its
// mainloop, the other consumer arrives on it
__device__ __forceinline__ void consumer_bar_sync(int id) { asm volatile("bar.sync %0, 256;" ::"r"(id) : "memory"); }
__device__ __forceinline__ void consumer_bar_arrive(int id) { asm volatile("bar.arrive %0, 256;" ::"r"(id) : "memory"); }

// epilogue kinds with bf16 outputs: stored 8 columns (16 B) per lane after a transpose inside each quad of lanes
template <int EPI>
constexpr bool epi_bf16_out() { return EPI == EPI_BF16 || EPI == EPI_BIAS_BF16 || EPI == EPI_BIAS_GELU || EPI == EPI_GELUGRAD_BF16; }

// two adjacent output columns (col, col + 1) of one row through an fp32-output epilogue of kind EPI (launch_gemm has resolved the
// strides: epi.ld_out and epi.ld_resid are never 0 here). out_row / res_row: the row's offsets, computed once per row and tile.
template <int EPI>
__device__ __forceinline__ void epi_store2(const GemmEpi& epi, size_t out_row, size_t res_row, int row, int col, float v0, float v1,
                                           float2 bb) {
  const size_t off = out_row + col;
  if (EPI == EPI_F32) {
    *reinterpret_cast<float2*>(epi.out_f32 + off) = make_float2(v0, v1);
  } else if (EPI == EPI_BIAS_RESID) {
    const float2 r = __ldg(reinterpret_cast<const float2*>(epi.resid + res_row + col));
    *reinterpret_cast<float2*>(epi.out_f32 + off) = make_float2(v0 + bb.x + r.x, v1 + bb.y + r.y);
  } else {   // EPI_UNPATCH: col = c*p*p + py*p + px with p even, so (col, col + 1) are adjacent pixels of one image row
    const int p = epi.unpatch_p, g = epi.unpatch_g, R = p * g;
    if (col >= 3 * p * p) return;    // the operand's zero padding up to patch_k(p) (p = 14): no pixel of this patch
    const int ch = col / (p * p), rem = col - ch * p * p, py = rem / p, px = rem - py * p;
    const int s = row / (g * g), pr = row - s * g * g, gy = pr / g, gx = pr - gy * g;
    *reinterpret_cast<float2*>(epi.out_f32 + (((size_t)s * 3 + ch) * R + gy * p + py) * R + gx * p + px) = make_float2(v0, v1);
  }
}

// one 16-byte store (written out: the compiler splits a uint4 assignment through a bf16 pointer into four 4-byte stores)
__device__ __forceinline__ void st_global_16(void* p, const uint32_t (&w)[4]) {
  asm volatile("st.global.v4.b32 [%0], {%1, %2, %3, %4};" ::"l"(p), "r"(w[0]), "r"(w[1]), "r"(w[2]), "r"(w[3]) : "memory");
}

// 4 x 4 transpose of 32-bit words over the 4 lanes of a quad (lane q = lane & 3): lane q's w[t] <-> lane t's w[q].
// In the accumulator layout lane q holds columns 8 t + 2 q, +1 (t = 0..3) of a 32-column chunk; after the transpose it holds the
// 8 contiguous columns 8 q .. 8 q + 7, and the reverse. Two exchange steps, one per bit of (q, t).
__device__ __forceinline__ void quad_transpose(uint32_t (&w)[4], int q) {
  const bool b0 = q & 1, b1 = q & 2;
#pragma unroll
  for (int p = 0; p < 2; ++p) {
    const uint32_t r = __shfl_xor_sync(0xffffffffu, b0 ? w[2 * p] : w[2 * p + 1], 1);
    if (b0) w[2 * p] = r; else w[2 * p + 1] = r;
  }
#pragma unroll
  for (int p = 0; p < 2; ++p) {
    const uint32_t r = __shfl_xor_sync(0xffffffffu, b1 ? w[p] : w[p + 2], 2);
    if (b1) w[p] = r; else w[p + 2] = r;
  }
}

// A 32-column chunk of one row through a bf16-output epilogue of kind EPI. v[2 t + {0,1}] = accumulators at columns
// col0 + 8 t + 2 q + {0,1}, bb[t] their bias. The math per element is that of the pairwise store; only the stores (and the
// gelu_in loads) are 16 B per lane, so that a warp writes whole 32 B sectors. All 32 lanes must call it (shuffles); rows >= M
// load and store nothing.
template <int EPI>
__device__ __forceinline__ void epi_store_bf16x32(const GemmEpi& epi, int row, bool valid, int col0, int q, const float* v,
                                                  const float2* bb) {
  const size_t off = (size_t)row * epi.ld_out + col0 + 8 * q;  // this lane's 8 columns after the transpose
  uint32_t w[4], w2[4];
  if constexpr (EPI == EPI_GELUGRAD_BF16) {
    uint4 g = make_uint4(0u, 0u, 0u, 0u);
    if (valid) g = __ldg(reinterpret_cast<const uint4*>(epi.gelu_in + off));
    w2[0] = g.x; w2[1] = g.y; w2[2] = g.z; w2[3] = g.w;
    quad_transpose(w2, q);                                     // back to the accumulator layout
  }
#pragma unroll
  for (int t = 0; t < 4; ++t) {
    float v0 = v[2 * t], v1 = v[2 * t + 1];
    if (EPI == EPI_BF16) {
      w[t] = pack_bf16(v0, v1);
    } else if (EPI == EPI_BIAS_BF16) {
      w[t] = pack_bf16(v0 + bb[t].x, v1 + bb[t].y);
    } else if (EPI == EPI_BIAS_GELU) {
      v0 += bb[t].x; v1 += bb[t].y;
      w2[t] = pack_bf16(v0, v1);
      w[t] = pack_bf16(quickgelu(v0), quickgelu(v1));
    } else {   // EPI_GELUGRAD_BF16
      const float2 h = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&w2[t]));
      w[t] = pack_bf16(v0 * quickgelu_grad(h.x), v1 * quickgelu_grad(h.y));
    }
  }
  quad_transpose(w, q);
  if (valid) st_global_16(epi.out_bf16 + off, w);
  if constexpr (EPI == EPI_BIAS_GELU) {
    quad_transpose(w2, q);
    if (valid) st_global_16(epi.out_pre + off, w2);
  }
}

// PINGPONG = false ("cooperative"): both consumer warpgroups work on every tile, rows 0-63 / 64-127, one m64nBNk16 per k16.
// PINGPONG = true: consumer warpgroup c owns the whole 128 x 128 tiles i = c, c + 2, ... of this CTA's schedule (two m64n128k16
// per k16: rows 0-63 and 64-127). Two named barriers hand the mainloop back and forth, so one warpgroup issues the MMAs of tile
// i while the other stores tile i - 1: the tensor pipe and the epilogue's HBM traffic overlap instead of taking turns.
template <int BN, bool PINGPONG, int EPI>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
k_gemm_bf16_tn(const __grid_constant__ CUtensorMap map_a, const __grid_constant__ CUtensorMap map_b, GemmShape shp, GemmEpi epi) {
  static_assert(BN == 128 || !PINGPONG, "the ping-pong schedule runs 128 x 128 tiles");
  using L = GemmCfg<BN>;
  constexpr int STAGES = L::STAGES;
  constexpr int MMAS = PINGPONG ? 2 : 1;          // m64 row blocks per consumer warpgroup and tile
  constexpr bool HAS_BIAS = (EPI == EPI_BIAS_BF16 || EPI == EPI_BIAS_GELU || EPI == EPI_BIAS_RESID);
  pdl_trigger();
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + L::BAR_OFFSET);
  uint64_t* empty_bar = full_bar + STAGES;

  const int wg = threadIdx.x >> 7, tid = threadIdx.x & 127;
  const int m_tiles = (shp.M + GEMM_BM - 1) / GEMM_BM, n_tiles = shp.N / BN;
  const int num_tiles = m_tiles * n_tiles, k_blocks = shp.K / GEMM_BK;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&map_a); tma_prefetch_desc(&map_b);
    for (int i = 0; i < STAGES; ++i) { mbar_init(&full_bar[i], 1); mbar_init(&empty_bar[i], PINGPONG ? 1 : 2); }
    fence_barrier_init();
  }
  __syncthreads();
  pdl_wait();                  // everything above overlapped the previous kernel's tail; operands are read from here on

  if (wg == 0) {
    setmaxnreg_dec<40>();
    if (tid == 0) {
      // ===== TMA producer: fills the stage ring in tile order (both schedules)
      const uint64_t pol_b = l2_policy_evict_last();      // B = weights: shared by all M tiles
      uint32_t it = 0;
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        const int m_blk = tile / n_tiles, n_blk = tile - m_blk * n_tiles;
        for (int kb = 0; kb < k_blocks; ++kb, ++it) {
          const uint32_t s = it % STAGES, ph = (it / STAGES) & 1;
          mbar_wait(&empty_bar[s], ph ^ 1);
          uint8_t* sa = smem + s * L::STAGE_BYTES;
          mbar_expect_tx(&full_bar[s], L::STAGE_BYTES);
          tma_load_2d(sa, &map_a, &full_bar[s], kb * GEMM_BK, m_blk * GEMM_BM);
          tma_load_2d_hint(sa + L::A_BYTES, &map_b, &full_bar[s], kb * GEMM_BK, n_blk * BN, pol_b);
        }
      }
    }
  } else {
    setmaxnreg_inc<232>();
    // ===== consumer warpgroup c
    const int c = wg - 1, warp = tid >> 5, lane = tid & 31;
    const int row_in_tile = (PINGPONG ? 0 : 64 * c) + 16 * warp + (lane >> 2), col_in_tile = 2 * (lane & 3);
    // this CTA's tiles are blockIdx.x + i * gridDim.x, i = 0, 1, ...; their stages follow each other in the ring (`it`)
    uint32_t it = PINGPONG ? c * k_blocks : 0;
    const int tile_step = (PINGPONG ? 2 : 1) * gridDim.x;
    // (the loop bounds compare rows with shp.M, a kernel parameter, rather than keep num_tiles in a register)
    for (int tile = blockIdx.x + (PINGPONG ? c * gridDim.x : 0); tile / n_tiles * GEMM_BM < shp.M; tile += tile_step) {
      // Ping-pong: wait until the other warpgroup has issued the previous tile. This also keeps every full-barrier wait below at
      // most one phase ahead of the barrier (the stage's previous use, in that tile or earlier, has already been waited for).
      if (PINGPONG && tile != (int)blockIdx.x) consumer_bar_sync(1 + c);
      float d[MMAS][BN / 2];
#pragma unroll
      for (int h = 0; h < MMAS; ++h)
#pragma unroll
        for (int r = 0; r < BN / 2; ++r) d[h][r] = 0.f;
      for (int kb = 0; kb < k_blocks; ++kb, ++it) {
        const uint32_t s = it % STAGES, ph = (it / STAGES) & 1;
        mbar_wait(&full_bar[s], ph);
        // one descriptor for the stage; offsets go into its (address >> 4) field: +2 per 16 bf16 along K inside the swizzle atom,
        // +512 per 64 rows of A, +A_BYTES / 16 for B
        const uint64_t ds = make_smem_desc(smem_u32(smem + s * L::STAGE_BYTES));
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < GEMM_BK / GEMM_UK; ++k)
#pragma unroll
          for (int h = 0; h < MMAS; ++h)
            Wgmma<BN>::mma(d[h], ds + (uint64_t)((PINGPONG ? h : c) * 512 + 2 * k), ds + (uint64_t)(L::A_BYTES / 16 + 2 * k), (kb | k) != 0);
        wgmma_commit();
        wgmma_wait<1>();                                 // the previous stage's MMAs have retired: hand that stage back
        if (kb > 0 && tid == 0) mbar_arrive(&empty_bar[(it - 1) % STAGES]);
      }
      if (PINGPONG && (tile + (int)gridDim.x) / n_tiles * GEMM_BM < shp.M) consumer_bar_arrive(1 + (c ^ 1));    // the other warpgroup may issue the next tile
      wgmma_wait<0>();
      if (tid == 0) mbar_arrive(&empty_bar[(it - 1) % STAGES]);
      if (PINGPONG) it += k_blocks;                    // skip the other warpgroup's tile
      const int m_blk = tile / n_tiles, n_blk = tile - m_blk * n_tiles;
      // ---- epilogue straight from the accumulator fragments: d[h][4j + {0,1}] = (row, col + {0,1}), d[h][4j + {2,3}] = (row + 8, ...)
#pragma unroll
      for (int h = 0; h < MMAS; ++h) {
        const int row0 = m_blk * GEMM_BM + 64 * h + row_in_tile, row1 = row0 + 8;
        if constexpr (epi_bf16_out<EPI>()) {
#pragma unroll
          for (int j0 = 0; j0 < BN / 8; j0 += 4) {        // 32-column chunks
            const int col0 = n_blk * BN + 8 * j0;
            float2 bb[4];
            float v0[8], v1[8];
#pragma unroll
            for (int t = 0; t < 4; ++t) {
              bb[t] = HAS_BIAS ? __ldg(reinterpret_cast<const float2*>(epi.bias + col0 + 8 * t + col_in_tile)) : make_float2(0.f, 0.f);
              v0[2 * t] = d[h][4 * (j0 + t)]; v0[2 * t + 1] = d[h][4 * (j0 + t) + 1];
              v1[2 * t] = d[h][4 * (j0 + t) + 2]; v1[2 * t + 1] = d[h][4 * (j0 + t) + 3];
            }
            epi_store_bf16x32<EPI>(epi, row0, row0 < shp.M, col0, lane & 3, v0, bb);
            epi_store_bf16x32<EPI>(epi, row1, row1 < shp.M, col0, lane & 3, v1, bb);
          }
        } else {
          const size_t out0 = (size_t)row0 * epi.ld_out, out1 = out0 + 8 * (size_t)epi.ld_out;
          const size_t res0 = (EPI == EPI_BIAS_RESID) ? (size_t)row0 * epi.ld_resid : 0, res1 = res0 + 8 * (size_t)epi.ld_resid;
#pragma unroll
          for (int j = 0; j < BN / 8; ++j) {
            const int col = n_blk * BN + 8 * j + col_in_tile;
            const float2 bb = HAS_BIAS ? __ldg(reinterpret_cast<const float2*>(epi.bias + col)) : make_float2(0.f, 0.f);
            if (row0 < shp.M) epi_store2<EPI>(epi, out0, res0, row0, col, d[h][4 * j], d[h][4 * j + 1], bb);
            if (row1 < shp.M) epi_store2<EPI>(epi, out1, res1, row1, col, d[h][4 * j + 2], d[h][4 * j + 3], bb);
          }
        }
      }
    }
  }
}

// ---- host side ---------------------------------------------------------------------------------
// 2-D bf16 tensor map: tensor [rows, K] with rows `row_stride` elements apart (K when 0), box [box_rows, 64] with 128B swizzle.
int make_tmap_bf16(CUtensorMap* out, const void* base, int rows, int K, int box_rows, int64_t row_stride = 0);
int make_tmap_bf16_tokens(CUtensorMap* out, const void* base, int cols, int T, int S, int box_rows);
// 4-D view {C, W, H, N} of a bf16 NHWC activation, box {64 channels, box_w columns, box_h rows, 1 image}, 128B swizzle
int make_tmap_bf16_nhwc(CUtensorMap* out, const void* base, int N, int H, int W, int C, int box_h, int box_w);
// Launches the GEMM on `st`. A: [M,K] with rows `lda` elements apart (K when 0), B: [N,K] device bf16. Requires K % 64 == 0,
// N % 128 == 0, and row strides that are multiples of 16 bytes.
int launch_gemm(const void* A, const void* B, GemmShape shp, const GemmEpi& epi, cudaStream_t st, int lda = 0);

}  // namespace aph
