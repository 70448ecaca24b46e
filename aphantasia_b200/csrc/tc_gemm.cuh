// tc_gemm.cuh -- the wgmma / TMA GEMM of the CLIP ViT encoder (sm_90a).
//
//   C[M,N] = A[M,K] . B[N,K]^T      A, B bf16 row-major (K contiguous = "K-major"), fp32 accumulate in registers.
//
// Persistent, warp-specialised, one CTA of three warpgroups per SM, tile 128 x BN (BN = 128 or 256):
//   warpgroup 0 (1 lane)  TMA producer : cp.async.bulk.tensor.2d -> 128B-swizzled smem stages, mbarrier complete_tx
//   warpgroups 1, 2       consumers    : rows 0-63 / 64-127 of the tile; wgmma.mma_async m64nBNk16 with both operands read
//                                        from shared memory through descriptors, then the fused epilogue from registers
// The producer gives its registers to the consumers (setmaxnreg) and runs ahead into the next tile's stages while the
// consumers store the current one. Fused epilogues (struct GemmEpi): +bias, QuickGELU (saving the pre-activation),
// x gelu'(h) for the MLP backward, +fp32 residual, fp32 or bf16 outputs, and an NCHW "un-patchify" store for the
// patch-embed data gradient. Rows >= M are zero-filled by TMA on load and not stored.
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
  int unpatch_p = 0;               // >0: out_f32 is [S,3,R,R]; row = s*g*g + gy*g + gx, col = c*p*p + py*p + px
  int unpatch_g = 0;
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

// two adjacent output columns (col, col + 1) of one row through the epilogue of kind EPI
template <int EPI>
__device__ __forceinline__ void epi_store2(const GemmEpi& epi, int N, int row, int col, float v0, float v1, float2 bb) {
  const size_t off = (size_t)row * N + col;
  if (EPI == EPI_F32) {
    *reinterpret_cast<float2*>(epi.out_f32 + off) = make_float2(v0, v1);
  } else if (EPI == EPI_BF16) {
    *reinterpret_cast<uint32_t*>(epi.out_bf16 + off) = pack_bf16(v0, v1);
  } else if (EPI == EPI_BIAS_BF16) {
    *reinterpret_cast<uint32_t*>(epi.out_bf16 + off) = pack_bf16(v0 + bb.x, v1 + bb.y);
  } else if (EPI == EPI_BIAS_GELU) {
    v0 += bb.x; v1 += bb.y;
    *reinterpret_cast<uint32_t*>(epi.out_pre + off) = pack_bf16(v0, v1);
    *reinterpret_cast<uint32_t*>(epi.out_bf16 + off) = pack_bf16(quickgelu(v0), quickgelu(v1));
  } else if (EPI == EPI_BIAS_RESID) {
    const float2 r = __ldg(reinterpret_cast<const float2*>(epi.resid + off));
    *reinterpret_cast<float2*>(epi.out_f32 + off) = make_float2(v0 + bb.x + r.x, v1 + bb.y + r.y);
  } else if (EPI == EPI_GELUGRAD_BF16) {
    const uint32_t u = __ldg(reinterpret_cast<const unsigned int*>(epi.gelu_in + off));
    const float2 h = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&u));
    *reinterpret_cast<uint32_t*>(epi.out_bf16 + off) = pack_bf16(v0 * quickgelu_grad(h.x), v1 * quickgelu_grad(h.y));
  } else {   // EPI_UNPATCH: col = c*p*p + py*p + px with p even, so (col, col + 1) are adjacent pixels of one image row
    const int p = epi.unpatch_p, g = epi.unpatch_g, R = p * g;
    const int ch = col / (p * p), rem = col - ch * p * p, py = rem / p, px = rem - py * p;
    const int s = row / (g * g), pr = row - s * g * g, gy = pr / g, gx = pr - gy * g;
    *reinterpret_cast<float2*>(epi.out_f32 + (((size_t)s * 3 + ch) * R + gy * p + py) * R + gx * p + px) = make_float2(v0, v1);
  }
}

template <int BN, int EPI>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
k_gemm_bf16_tn(const __grid_constant__ CUtensorMap map_a, const __grid_constant__ CUtensorMap map_b, GemmShape shp, GemmEpi epi) {
  using L = GemmCfg<BN>;
  constexpr int STAGES = L::STAGES;
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
    for (int i = 0; i < STAGES; ++i) { mbar_init(&full_bar[i], 1); mbar_init(&empty_bar[i], 2); }
    fence_barrier_init();
  }
  __syncthreads();
  pdl_wait();                  // everything above overlapped the previous kernel's tail; operands are read from here on

  if (wg == 0) {
    setmaxnreg_dec<40>();
    if (tid == 0) {
      // ===== TMA producer
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
    // ===== consumer warpgroup: rows 64*(wg-1) .. +63 of each tile
    const int warp = tid >> 5, lane = tid & 31;
    const int row_in_tile = 64 * (wg - 1) + 16 * warp + (lane >> 2), col_in_tile = 2 * (lane & 3);
    uint32_t it = 0;
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
      const int m_blk = tile / n_tiles, n_blk = tile - m_blk * n_tiles;
      float d[BN / 2];
#pragma unroll
      for (int i = 0; i < BN / 2; ++i) d[i] = 0.f;
      int prev = -1;
      for (int kb = 0; kb < k_blocks; ++kb, ++it) {
        const uint32_t s = it % STAGES, ph = (it / STAGES) & 1;
        mbar_wait(&full_bar[s], ph);
        const uint32_t sa = smem_u32(smem + s * L::STAGE_BYTES);
        const uint64_t da = make_smem_desc(sa + (wg - 1) * (64 * 128)), db = make_smem_desc(sa + L::A_BYTES);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < GEMM_BK / GEMM_UK; ++k)      // advance 16 bf16 = 32 B along K inside the swizzle atom: +2 in the (>>4) address field
          Wgmma<BN>::mma(d, da + (uint64_t)(2 * k), db + (uint64_t)(2 * k), (kb | k) != 0);
        wgmma_commit();
        wgmma_wait<1>();                                 // the previous stage's MMAs have retired: hand that stage back
        if (prev >= 0 && tid == 0) mbar_arrive(&empty_bar[prev]);
        prev = (int)s;
      }
      wgmma_wait<0>();
      if (prev >= 0 && tid == 0) mbar_arrive(&empty_bar[prev]);
      // ---- epilogue straight from the accumulator fragments: d[4j + {0,1}] = (row, col + {0,1}), d[4j + {2,3}] = (row + 8, ...)
      const int row0 = m_blk * GEMM_BM + row_in_tile, row1 = row0 + 8;
#pragma unroll
      for (int j = 0; j < BN / 8; ++j) {
        const int col = n_blk * BN + 8 * j + col_in_tile;
        const float2 bb = HAS_BIAS ? __ldg(reinterpret_cast<const float2*>(epi.bias + col)) : make_float2(0.f, 0.f);
        if (row0 < shp.M) epi_store2<EPI>(epi, shp.N, row0, col, d[4 * j], d[4 * j + 1], bb);
        if (row1 < shp.M) epi_store2<EPI>(epi, shp.N, row1, col, d[4 * j + 2], d[4 * j + 3], bb);
      }
    }
  }
}

// ---- host side ---------------------------------------------------------------------------------
// 2-D bf16 tensor map: tensor [rows, K] row-major, box [box_rows, 64] with 128B swizzle.
int make_tmap_bf16(CUtensorMap* out, const void* base, int rows, int K, int box_rows);
int make_tmap_bf16_tokens(CUtensorMap* out, const void* base, int cols, int T, int S, int box_rows);
// Launches the GEMM on `st`. A: [M,K], B: [N,K] device bf16. Requires K % 64 == 0, N % 128 == 0.
int launch_gemm(const void* A, const void* B, GemmShape shp, const GemmEpi& epi, cudaStream_t st);

}  // namespace aph
