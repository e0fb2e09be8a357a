// TMA / mbarrier / wgmma PTX wrappers shared by the tensor-core kernels (fd_tapgemm_tc.cu, fd_wgrad_tc.cu,
// fd_respair_tc.cu), sm_90a.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include "fd_common.cuh"
#include "fd_host.h"

namespace {

// ------------------------------------------------------------------ PTX wrappers
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "WAIT_LOOP:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      "@p bra WAIT_DONE;\n"
      "bra WAIT_LOOP;\n"
      "WAIT_DONE:\n"
      "}\n" ::"r"(smem_u32(bar)),
      "r"(parity)
      : "memory");
}
__device__ __forceinline__ void fence_barrier_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}

// ---- thread-block clusters
__device__ __forceinline__ uint32_t cluster_ctarank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
// every thread of every CTA of the cluster
__device__ __forceinline__ void cluster_sync() {
  asm volatile("barrier.cluster.arrive.release.aligned;\nbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}
// arrive on the barrier at `bar`'s offset in CTA `cta` of the cluster.  CTA-scope release: a .release.cluster arrive
// puts a MEMBAR.GPU in front of every call (DESIGN.md section 5)
__device__ __forceinline__ void mbar_arrive_cluster(uint64_t* bar, uint32_t cta) {
  asm volatile(
      "{\n.reg .b32 ra;\nmapa.shared::cluster.u32 ra, %0, %1;\nmbarrier.arrive.shared::cluster.b64 _, [ra];\n}"
      ::"r"(smem_u32(bar)), "r"(cta)
      : "memory");
}

// named barrier ID (id 0 is __syncthreads) of N threads, a multiple of 32
template <int ID, int N>
__device__ __forceinline__ void named_bar_sync() {
  asm volatile("bar.sync %0, %1;" ::"n"(ID), "n"(N) : "memory");
}
template <int ID, int N>
__device__ __forceinline__ void named_bar_arrive() {
  asm volatile("bar.arrive %0, %1;" ::"n"(ID), "n"(N) : "memory");
}

__device__ __forceinline__ void tma_load_4d(void* smem_dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1,
                                            int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
      ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c0), "r"(c1),
      "r"(c2), "r"(c3)
      : "memory");
}
__device__ __forceinline__ void tma_load_3d(void* smem_dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1,
                                            int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
      ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c0), "r"(c1),
      "r"(c2)
      : "memory");
}
__device__ __forceinline__ void tma_load_5d(void* smem_dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1,
                                            int c2, int c3, int c4) {
  asm volatile(
      "cp.async.bulk.tensor.5d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6, %7}], [%2];"
      ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c0), "r"(c1),
      "r"(c2), "r"(c3), "r"(c4)
      : "memory");
}
// the same box written at the same shared-memory offset of every CTA in `cta_mask`, completing bytes on the barrier at
// the same offset in each of them
__device__ __forceinline__ void tma_load_4d_multicast(void* smem_dst, const CUtensorMap* map, uint64_t* bar, int c0,
                                                      int c1, int c2, int c3, uint16_t cta_mask) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster"
      " [%0], [%1, {%4, %5, %6, %7}], [%2], %3;"
      ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "h"(cta_mask), "r"(c0),
      "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}
__device__ __forceinline__ void tma_load_3d_multicast(void* smem_dst, const CUtensorMap* map, uint64_t* bar, int c0,
                                                      int c1, int c2, uint16_t cta_mask) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster"
      " [%0], [%1, {%4, %5, %6}], [%2], %3;"
      ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "h"(cta_mask), "r"(c0),
      "r"(c1), "r"(c2)
      : "memory");
}
__device__ __forceinline__ void prefetch_tmap(const CUtensorMap* map) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(map)) : "memory");
}

// explicit shared-space ld/st (scratch addresses come from integer arithmetic, which would make the compiler fall back
// to generic LD/ST with their longer latency)
__device__ __forceinline__ float4 lds128(uint32_t addr) {
  float4 r;
  asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w) : "r"(addr) : "memory");
  return r;
}
// N (a multiple of 4) consecutive floats: from shared memory, and streaming from global memory (evict-first)
template <int N>
__device__ __forceinline__ void lds_f32(uint32_t addr, float (&v)[N]) {
#pragma unroll
  for (int q = 0; q < N; q += 4) {
    const float4 x = lds128(addr + 4u * q);
    v[q] = x.x; v[q + 1] = x.y; v[q + 2] = x.z; v[q + 3] = x.w;
  }
}
template <int N>
__device__ __forceinline__ void ldcs_f32(const float* p, float (&v)[N]) {
#pragma unroll
  for (int q = 0; q < N; q += 4) {
    const float4 x = __ldcs(reinterpret_cast<const float4*>(p + q));
    v[q] = x.x; v[q + 1] = x.y; v[q + 2] = x.z; v[q + 3] = x.w;
  }
}
__device__ __forceinline__ void sts32(uint32_t addr, float x) {
  asm volatile("st.shared.f32 [%0], %1;" ::"r"(addr), "f"(x) : "memory");
}
__device__ __forceinline__ void sts64(uint32_t addr, float x, float y) {
  asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(addr), "f"(x), "f"(y) : "memory");
}

// Register budget of a warp-specialised CTA of three warpgroups (384 threads: at most 168 registers per thread at launch):
// the producer warpgroup, which only issues TMA, hands its registers to the two consumer warpgroups, which hold the
// accumulators (128 x 40 + 256 x 232 = 64512 of the 65536 registers of an SM).  Every thread of a warpgroup executes it.
// Warps 0..7 are the consumers, warps 8..11 the producer warpgroup.
constexpr int FD_TC_CONSUMER_THREADS = 256;
constexpr int FD_TC_THREADS = FD_TC_CONSUMER_THREADS + 128;
constexpr int FD_TC_PRODUCER_WARP = FD_TC_CONSUMER_THREADS / 32;
__device__ __forceinline__ void producer_regs() { asm volatile("setmaxnreg.dec.sync.aligned.u32 40;" ::: "memory"); }
__device__ __forceinline__ void consumer_regs() { asm volatile("setmaxnreg.inc.sync.aligned.u32 232;" ::: "memory"); }

// Dynamic shared memory of one CTA per SM (227 KB on sm_90), and the pipeline ring that fills what the fixed parts of a
// kernel's layout leave: stages of `stage_bytes` in FD_TC_SMEM_BUDGET - `fixed_bytes`, at most FD_TC_MAX_STAGES.
constexpr int FD_TC_SMEM_BUDGET = 227 * 1024;
constexpr int FD_TC_MAX_STAGES = 8;
constexpr int fd_tc_ring_stages(int fixed_bytes, int stage_bytes) {
  const int n = (FD_TC_SMEM_BUDGET - fixed_bytes) / stage_bytes;
  return n > FD_TC_MAX_STAGES ? FD_TC_MAX_STAGES : n;
}

// ------------------------------------------------------------------ wgmma
__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wg_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from moving accesses of accumulator registers across a wgmma fence / wait
template <int R>
__device__ __forceinline__ void wg_fence_operand(float (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// Shared-memory matrix descriptor (PTX "matrix descriptor" of wgmma): start addr>>4 [0,14), LBO>>4 [16,30),
// SBO>>4 [32,46), swizzle mode [62,64) (1 = 128 B, 2 = 64 B, 3 = 32 B).  K-major swizzled operands: SBO = byte distance
// between groups of 8 rows, LBO unused (1).  MN-major swizzled operands: LBO = byte distance between swizzle atoms
// along M/N, SBO = byte distance between groups of 8 K rows.  The base-offset field stays 0: the swizzle is applied to
// the absolute shared-memory address bits, so a K-major operand may also start a whole number of rows into a
// swizzled tile written by TMA (the transposed GATE's tap shifts, fd_tapgemm_tc.cu: its tests run every dilation
// 1..8, whose tap offsets cover every row of the 8-row swizzle atom).
__device__ __forceinline__ uint64_t make_smem_desc(uint32_t smem_addr, uint32_t lbo_bytes, uint32_t sbo_bytes,
                                                   uint32_t swizzle_mode) {
  uint64_t d = 0;
  d |= (uint64_t)((smem_addr & 0x3FFFF) >> 4);
  d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFF) << 16;
  d |= (uint64_t)((sbo_bytes >> 4) & 0x3FFF) << 32;
  d |= (uint64_t)swizzle_mode << 62;
  return d;
}
// swizzle mode of a K-major operand whose rows are `row_bytes` long (128 / 64 / 32)
__host__ __device__ constexpr uint32_t swizzle_mode_for(int row_bytes) {
  return row_bytes == 128 ? 1u : row_bytes == 64 ? 2u : 3u;
}
// the TMA swizzle that writes what that descriptor reads; NONE for other row lengths, which encode_tiled refuses
CUtensorMapSwizzle tma_swizzle_for(int row_bytes) {
  return row_bytes == 128 ? CU_TENSOR_MAP_SWIZZLE_128B : row_bytes == 64 ? CU_TENSOR_MAP_SWIZZLE_64B
         : row_bytes == 32 ? CU_TENSOR_MAP_SWIZZLE_32B : CU_TENSOR_MAP_SWIZZLE_NONE;
}

// wgmma.mma_async m64nNk16, fp32 accumulators d[N/2] in the standard fragment layout (see frag_to_scratch), for
// PREC = FD_F16 / FD_BF16 and the widths N defined below; any other N does not compile.  ss: both operands from shared
// memory (TA / TB = 1: that operand is MN-major); rs: A from registers (the mma.m16n8k16 A fragment of the warp's 16
// rows), B K-major from shared memory.  Both add to d (scale-d is a predicate that is always true).
template <int N, int PREC>
struct Wgmma;

// Inline PTX names its operands by number.  The R = N/2 accumulators come first, as operands %0 .. %(R-1):
// FD_WG_REGS<R> lists them (each list extends the one before) and FD_ACC<R>(0) binds d[0] .. d[R-1] to them.
#define FD_ACC4(i) "+f"(d[i]), "+f"(d[(i) + 1]), "+f"(d[(i) + 2]), "+f"(d[(i) + 3])
#define FD_ACC8(i) FD_ACC4(i), FD_ACC4((i) + 4)
#define FD_ACC16(i) FD_ACC8(i), FD_ACC8((i) + 8)
#define FD_ACC32(i) FD_ACC16(i), FD_ACC16((i) + 16)
#define FD_ACC64(i) FD_ACC32(i), FD_ACC32((i) + 32)
#define FD_ACC100(i) FD_ACC64(i), FD_ACC32((i) + 64), FD_ACC4((i) + 96)
#define FD_ACC120(i) FD_ACC100(i), FD_ACC16((i) + 100), FD_ACC4((i) + 116)
#define FD_ACC128(i) FD_ACC64(i), FD_ACC64((i) + 64)
#define FD_WG_REGS8 "%0, %1, %2, %3, %4, %5, %6, %7"
#define FD_WG_REGS16 FD_WG_REGS8 ", %8, %9, %10, %11, %12, %13, %14, %15"
#define FD_WG_REGS32 FD_WG_REGS16 ", %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31"
#define FD_WG_REGS64                                                                                          \
  FD_WG_REGS32 ", %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47"             \
               ", %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63"
#define FD_WG_REGS100                                                                                         \
  FD_WG_REGS64 ", %64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79"             \
               ", %80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95"             \
               ", %96, %97, %98, %99"
#define FD_WG_REGS120                                                                                         \
  FD_WG_REGS100 ", %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111"                    \
                ", %112, %113, %114, %115, %116, %117, %118, %119"
#define FD_WG_REGS128 FD_WG_REGS120 ", %120, %121, %122, %123, %124, %125, %126, %127"

// Wgmma<N, PREC> for input type TY ("f16" / "bf16"); the operands after the accumulators are numbered R .. R + 4.
#define FD_WGMMA_TY(N, PREC, TY, R, R1, R2, R3, R4)                                                           \
  template <> struct Wgmma<N, PREC> {                                                                         \
    static_assert(2 * R == N && R1 == R + 1 && R2 == R + 2 && R3 == R + 3 && R4 == R + 4, "operand numbers"); \
    template <int TA, int TB>                                                                                 \
    static __device__ __forceinline__ void ss(float* d, uint64_t da, uint64_t db) {                           \
      asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, 1, 0;\n"                                                 \
                   "wgmma.mma_async.sync.aligned.m64n" #N "k16.f32." TY "." TY " {" FD_WG_REGS##R "}, "       \
                   "%" #R ", %" #R1 ", p, 1, 1, %" #R2 ", %" #R3 ";\n}\n"                                     \
                   : FD_ACC##R(0)                                                                             \
                   : "l"(da), "l"(db), "n"(TA), "n"(TB));                                                     \
    }                                                                                                         \
    static __device__ __forceinline__ void rs(float* d, const uint32_t (&a)[4], uint64_t db) {                \
      asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, 1, 0;\n"                                                 \
                   "wgmma.mma_async.sync.aligned.m64n" #N "k16.f32." TY "." TY " {" FD_WG_REGS##R "}, "       \
                   "{%" #R ", %" #R1 ", %" #R2 ", %" #R3 "}, %" #R4 ", p, 1, 1, 0;\n}\n"                      \
                   : FD_ACC##R(0)                                                                             \
                   : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db));                                    \
    }                                                                                                         \
  };
#define FD_WGMMA(N, R, R1, R2, R3, R4)                                                                        \
  FD_WGMMA_TY(N, FD_F16, "f16", R, R1, R2, R3, R4)                                                            \
  FD_WGMMA_TY(N, FD_BF16, "bf16", R, R1, R2, R3, R4)
FD_WGMMA(16, 8, 9, 10, 11, 12)
FD_WGMMA(32, 16, 17, 18, 19, 20)
FD_WGMMA(64, 32, 33, 34, 35, 36)
FD_WGMMA(128, 64, 65, 66, 67, 68)
FD_WGMMA(256, 128, 129, 130, 131, 132)
// N = 200 / 240: the time tiles of the transposed GATE (fd_tapgemm_tc.cu), which calls ss only, both operands K-major
FD_WGMMA(200, 100, 101, 102, 103, 104)
FD_WGMMA(240, 120, 121, 122, 123, 124)

// ------------------------------------------------------------------ accumulator fragments -> warp scratch
// A warp of a consumer warpgroup holds rows [16 w, 16 w + 16) of the 64-row wgmma tile; lane l holds d[i] at
//   row = l/4 + 8 ((i/2) % 2),  col = 8 (i/4) + 2 (l % 4) + (i % 2).
// The epilogues re-distribute a chunk of columns through a warp-private 16 x 32 fp32 scratch (2 KB; 16-byte chunks
// XOR-swizzled by row & 7) into whatever per-lane layout their global accesses want.
constexpr int FD_TC_SCRATCH_WARP_BYTES = 16 * 32 * 4;
constexpr int FD_TC_SCRATCH_BYTES = (FD_TC_CONSUMER_THREADS / 32) * FD_TC_SCRATCH_WARP_BYTES;   // all consumer warps
// Writes columns [c0, c0 + CW) of the fragment (d points at the tile's first register) to scratch columns
// [off, off + CW).
template <int CW>
__device__ __forceinline__ void frag_to_scratch(uint32_t scratch, const float* d, int c0, int off, int lane) {
#pragma unroll
  for (int i = 0; i < CW / 2; i += 2) {
    const int row = (lane >> 2) + 8 * ((i >> 1) & 1);
    const int col = off + 8 * (i >> 2) + 2 * (lane & 3);
    sts64(scratch + row * 128 + (((col >> 2) ^ (row & 7)) << 4) + (col & 3) * 4, d[c0 / 2 + i], d[c0 / 2 + i + 1]);
  }
}
// four consecutive scratch columns [4 chunk, 4 chunk + 4) of one row
__device__ __forceinline__ float4 scratch_ld4(uint32_t scratch, int row, int chunk) {
  return lds128(scratch + row * 128 + ((chunk ^ (row & 7)) << 4));
}

// ------------------------------------------------------------------ pipeline plumbing
// One k-block of the split-precision product on shared-memory operands: KSTEPS k16 steps, the descriptors moving
// STEP_BYTES per step.  The three products of a step are issued as activation lo x weight hi, activation hi x weight
// lo, then hi x hi: small terms first, the dominant hi x hi last; every three-product result depends on this order
// bit for bit.  NPL == 1 issues hi x hi only.  The operands are given by role; W_IS_A puts the weights on the wgmma
// A (M) side, and TA / TB are the MN-major flags of operands A and B.
template <class MMA, int NPL, int KSTEPS, int STEP_BYTES, bool W_IS_A = false, int TA = 0, int TB = 0>
__device__ __forceinline__ void split_mma(float* acc, uint64_t x_hi, uint64_t x_lo, uint64_t w_hi, uint64_t w_lo) {
  auto mma = [&](uint64_t x, uint64_t w) {
    if (W_IS_A) MMA::template ss<TA, TB>(acc, w, x);
    else MMA::template ss<TA, TB>(acc, x, w);
  };
#pragma unroll
  for (int k = 0; k < KSTEPS; ++k) {
    const uint64_t adv = (uint64_t)((k * STEP_BYTES) >> 4);
    if (NPL == 2) {
      mma(x_lo + adv, w_hi + adv);
      mma(x_hi + adv, w_lo + adv);
    }
    mma(x_hi + adv, w_hi + adv);
  }
}
// One k16 step of the same products with the activations in registers (MMA::rs, operand A) and the weights K-major
// in shared memory; `single` issues hi x hi only.
template <class MMA>
__device__ __forceinline__ void split_mma_rs(float* acc, const uint32_t (&x_hi)[4], const uint32_t (&x_lo)[4],
                                             uint64_t w_hi, uint64_t w_lo, bool single) {
  if (!single) {
    MMA::rs(acc, x_lo, w_hi);
    MMA::rs(acc, x_hi, w_lo);
  }
  MMA::rs(acc, x_hi, w_hi);
}

// Cursor of a full / empty barrier ring of `stages` stages: the stage the next access goes to and the phase parity of
// its barriers.  The producer waits for a stage to be empty, the consumers for it to be full.  Where `stages` is a
// compile-time constant it folds into the code as the constant would.
struct Ring {
  uint64_t* full;
  uint64_t* empty;
  int stages;
  int stage = 0;
  uint32_t phase = 0;
  __device__ __forceinline__ uint64_t* full_bar() const { return &full[stage]; }
  __device__ __forceinline__ void wait_full() const { mbar_wait(&full[stage], phase); }
  __device__ __forceinline__ void wait_empty() const { mbar_wait(&empty[stage], phase ^ 1); }
  __device__ __forceinline__ void next() {
    if (++stage == stages) { stage = 0; phase ^= 1; }
  }
  __device__ __forceinline__ void advance(int n) {   // n ring positions on
    stage += n;
    phase ^= (uint32_t)(stage / stages) & 1u;
    stage %= stages;
  }
};

// The mainloop of a consumer warpgroup of the cooperative kernels over `k_blocks` k-blocks, `group` of them per ring
// stage: one wgmma group per stage, issued by issue(stage, k-blocks in the stage), and one group kept in flight; lane
// 0 of each warp releases a stage once the group that read it has completed.  The accumulators start at zero.
template <int R, class Issue>
__device__ __forceinline__ void ring_mainloop(float (&acc)[R], Ring& ring, int k_blocks, int group, int lane,
                                              Issue&& issue) {
#pragma unroll
  for (int i = 0; i < R; ++i) acc[i] = 0.f;
  int prev_stage = -1;
  for (int kb = 0; kb < k_blocks; kb += group) {
    ring.wait_full();
    wg_fence_operand(acc);
    wg_fence();
    issue(ring.stage, min(group, k_blocks - kb));
    wg_commit();
    wg_wait<1>();
    wg_fence_operand(acc);
    if (prev_stage >= 0 && lane == 0) mbar_arrive(&ring.empty[prev_stage]);
    prev_stage = ring.stage;
    ring.next();
  }
  wg_wait<0>();
  wg_fence_operand(acc);
  if (prev_stage >= 0 && lane == 0) mbar_arrive(&ring.empty[prev_stage]);
}

// The ping-pong turn of the two consumer warpgroups of a CTA in a 2x1x1 cluster (fd_tapgemm_tc.cu).  The producer
// fills one ring for both warpgroups, unit by unit, each unit `k_blocks` stages; warpgroup 0 takes the 1st, 3rd, ...
// unit, warpgroup 1 the 2nd, 4th, ...  The mainloops run in turn: a warpgroup waits for its turn (named barrier
// 1 + wg) and passes it (named barrier 2 - wg) once it has committed the last wgmma group of its unit, so that its
// epilogue overlaps the other warpgroup's mainloop.  The turn also keeps a warpgroup from waiting on a full barrier
// more than one phase ahead of the ring.  A stage is refilled in both CTAs (the weights arrive by multicast), so it is
// released into both.
struct PingPong {
  Ring ring;
  int k_blocks;
  int wg;
  __device__ __forceinline__ PingPong(uint64_t* full, uint64_t* empty, int stages, int k_blocks_, int wg_)
      : ring{full, empty, stages}, k_blocks(k_blocks_), wg(wg_) {
    if (wg == 1) ring.advance(k_blocks);
  }
  // One unit's mainloop, the accumulators from zero; `first`: the warpgroup's first unit (no turn to wait for),
  // `pass`: the other warpgroup has a next unit.  issue(stage) issues the wgmma group of one stage; one group is kept
  // in flight, as in ring_mainloop.  The ring steps by advance(1): with next() the compiler unrolls this loop and
  // triples the code of a three-product stage.
  template <int R, class Issue>
  __device__ __forceinline__ void mainloop(float (&acc)[R], bool first, bool pass, int lane, Issue&& issue) {
    auto release = [&](int st) {
      if (lane == 0) { mbar_arrive_cluster(&ring.empty[st], 0); mbar_arrive_cluster(&ring.empty[st], 1); }
    };
    if (!first) wg == 0 ? named_bar_sync<1, 256>() : named_bar_sync<2, 256>();       // wait for the turn
#pragma unroll
    for (int i = 0; i < R; ++i) acc[i] = 0.f;
    int prev_stage = -1;
    for (int kb = 0; kb < k_blocks; ++kb) {
      ring.wait_full();
      wg_fence_operand(acc);
      wg_fence();
      issue(ring.stage);
      wg_commit();
      if (kb == k_blocks - 1 && pass) wg == 0 ? named_bar_arrive<2, 256>() : named_bar_arrive<1, 256>();   // pass it
      wg_wait<1>();
      wg_fence_operand(acc);
      if (prev_stage >= 0) release(prev_stage);
      prev_stage = ring.stage;
      ring.advance(1);
    }
    wg_wait<0>();
    wg_fence_operand(acc);
    if (prev_stage >= 0) release(prev_stage);
    ring.advance(k_blocks);   // past the other warpgroup's unit
  }
};

// Shared memory of a warp-specialised tensor-core kernel, from the 1024-byte aligned base: the ring of `stages` stages
// of `stage_bytes`, `bias_floats` floats of bias vectors, the full and empty barriers, the consumer warps' scratch
// (16-byte aligned: every preceding size is).
constexpr int fd_tc_frame_bytes(int stages, int stage_bytes, int bias_floats) {
  return 1024 /*align slack*/ + stages * stage_bytes + bias_floats * 4 + 2 * stages * 8 + FD_TC_SCRATCH_BYTES;
}
// ring stages of `stage_bytes` that fit next to the rest of that frame
constexpr int fd_tc_frame_stages(int stage_bytes, int bias_floats) {
  return fd_tc_ring_stages(fd_tc_frame_bytes(FD_TC_MAX_STAGES, 0, bias_floats), stage_bytes);
}
struct TcFrame {
  uint8_t* ring;
  float* bias;
  uint64_t* full;
  uint64_t* empty;
  float* scratch;
};
__device__ __forceinline__ TcFrame tc_frame(uint8_t* smem_raw, int stages, int stage_bytes, int bias_floats) {
  TcFrame f;
  f.ring = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  f.bias = reinterpret_cast<float*>(f.ring + stages * stage_bytes);
  f.full = reinterpret_cast<uint64_t*>(f.bias + bias_floats);
  f.empty = f.full + stages;
  f.scratch = reinterpret_cast<float*>(f.empty + stages);
  return f;
}
// The prologue: thread 0 initialises the ring's barriers (a full barrier completes on the producer's arrival and its
// transaction bytes, an empty barrier on `empty_arrivals` consumer warps), the producer thread prefetches the tensor
// maps, then the CTA -- or with CLUSTER the whole cluster, so that no CTA multicasts or arrives into a peer whose
// barriers are not initialised -- synchronises.
template <bool CLUSTER, class... Maps>
__device__ __forceinline__ void tc_prologue(const TcFrame& f, int stages, uint32_t empty_arrivals,
                                            const Maps*... maps) {
  if (threadIdx.x == 0) {
    for (int i = 0; i < stages; ++i) { mbar_init(&f.full[i], 1); mbar_init(&f.empty[i], empty_arrivals); }
    fence_barrier_init();
  }
  if (threadIdx.x / 32 == FD_TC_PRODUCER_WARP && threadIdx.x % 32 == 0) (prefetch_tmap(maps), ...);
  if (CLUSTER) cluster_sync();
  else __syncthreads();
}

// The producer's walk over the K segments of a tap-GEMM: segment s, k offset k0 inside it, and koff, the packed weight
// column of the segment's first k.
struct SegCursor {
  int s = 0, k0 = 0, koff = 0;
  __device__ __forceinline__ void next(int block_k, int k_len) {   // one k-block on; k_len of segment s
    k0 += block_k;
    if (k0 >= k_len) { koff += k_len; k0 = 0; ++s; }
  }
};

// ------------------------------------------------------------------ host side: tensor-map encoder entry point
typedef CUresult (*PFN_tmapEncodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                        const cuuint64_t*, const cuuint32_t*, const cuuint32_t*,
                                        CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion,
                                        CUtensorMapFloatOOBfill);

PFN_tmapEncodeTiled get_encode() {
  static PFN_tmapEncodeTiled fn = nullptr;
  if (fn == nullptr) {
    void* ptr = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &qres) == cudaSuccess &&
        qres == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<PFN_tmapEncodeTiled>(ptr);
  }
  return fn;
}

// A tensor map over 16-bit split planes (dims, byte strides and box innermost first); the swizzle follows the box's row
// length, so that it matches swizzle_mode_for of the operand the box lands in.
int encode_tiled(CUtensorMap* m, const uint16_t* ptr, int rank, const cuuint64_t* dims, const cuuint64_t* strides,
                 const cuuint32_t* box, const char* what) {
  PFN_tmapEncodeTiled enc = get_encode();
  FD_REQUIRE(enc != nullptr, "cuTensorMapEncodeTiled not available from the driver");
  const CUtensorMapSwizzle sw = tma_swizzle_for((int)box[0] * 2);
  FD_REQUIRE(sw != CU_TENSOR_MAP_SWIZZLE_NONE, "tensor map (%s): box rows of %u bytes (wgmma swizzles 128, 64 or 32)",
             what, box[0] * 2);
  FD_REQUIRE(rank >= 1 && rank <= 5, "tensor map (%s): rank %d (1..5)", what, rank);
  const cuuint32_t estr[5] = {1, 1, 1, 1, 1};   // one per dimension: every element of the box
  CUresult r = enc(m, CU_TENSOR_MAP_DATA_TYPE_UINT16, (cuuint32_t)rank, const_cast<uint16_t*>(ptr), dims, strides, box,
                   estr, CU_TENSOR_MAP_INTERLEAVE_NONE, sw, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  FD_REQUIRE(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled(%s) failed: %d (dims %llu x %llu x %llu x %llu, box %u x %u x %u x %u, ptr %p)",
             what, (int)r, (unsigned long long)dims[0], (unsigned long long)dims[1], (unsigned long long)dims[2],
             rank >= 4 ? (unsigned long long)dims[3] : 1ull, box[0], box[1], box[2], rank >= 4 ? box[3] : 1u,
             (const void*)ptr);
  return 0;
}

// Split planes [plane][B][T][C] (strides in elements) as the 4-D tensor (C, T, B, plane); box {box_c, box_rows, 1,
// box_planes}.
int planes_map(CUtensorMap* m, const uint16_t* ptr, int C, int T, int B, long long row_stride, long long item_stride,
               long long plane_stride, int box_c, int box_rows, int box_planes, const char* what) {
  const cuuint64_t dims[4] = {(cuuint64_t)C, (cuuint64_t)T, (cuuint64_t)B, 2};
  const cuuint64_t strides[3] = {(cuuint64_t)row_stride * 2, (cuuint64_t)item_stride * 2, (cuuint64_t)plane_stride * 2};
  const cuuint32_t box[4] = {(cuuint32_t)box_c, (cuuint32_t)box_rows, 1, (cuuint32_t)box_planes};
  return encode_tiled(m, ptr, 4, dims, strides, box, what);
}

// Packed weights [plane][N][K] as the 3-D tensor (K, N, plane); box {box_k, box_n, box_planes}.
int weights_map(CUtensorMap* m, const uint16_t* ptr, int N, int K, int box_k, int box_n, int box_planes,
                const char* what) {
  const cuuint64_t dims[3] = {(cuuint64_t)K, (cuuint64_t)N, 2};
  const cuuint64_t strides[2] = {(cuuint64_t)K * 2, (cuuint64_t)N * K * 2};
  const cuuint32_t box[3] = {(cuuint32_t)box_k, (cuuint32_t)box_n, (cuuint32_t)box_planes};
  return encode_tiled(m, ptr, 3, dims, strides, box, what);
}

// Launches a persistent kernel of FD_TC_THREADS threads: one CTA per SM, at most one per work unit, in clusters of
// `cluster` CTAs along x (the grid rounded down to a multiple of it, and capped at the clusters that fit on the device
// at once, so that no cluster waits for another to finish).  The dynamic shared-memory limit is an attribute of each
// kernel and device, set on the kernel's first launch on a device (the cache below is per Kern); `max_carveout` also
// asks for the largest shared-memory carveout.
template <auto Kern, typename... Args>
int fd_tc_launch(int smem_bytes, int work_units, cudaStream_t stream, bool max_carveout, int cluster,
                 const Args&... args) {
  static bool attr_set[FD_MAX_DEVICES] = {false};
  static int max_grid[FD_MAX_DEVICES];
  const int dev = fd_current_device();
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = cluster;
  attr[0].val.clusterDim.y = 1;
  attr[0].val.clusterDim.z = 1;
  cudaLaunchConfig_t cfg = {};
  cfg.blockDim = dim3(FD_TC_THREADS);
  cfg.dynamicSmemBytes = smem_bytes;
  cfg.stream = stream;
  cfg.attrs = attr;
  cfg.numAttrs = cluster > 1 ? 1 : 0;
  if (!attr_set[dev]) {
    FD_CHECK_CUDA(cudaFuncSetAttribute(Kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_bytes));
    if (max_carveout)
      FD_CHECK_CUDA(cudaFuncSetAttribute(Kern, cudaFuncAttributePreferredSharedMemoryCarveout,
                                         cudaSharedmemCarveoutMaxShared));
    const int sms = fd_device_sms(dev);
    max_grid[dev] = sms - sms % cluster;
    if (cluster > 1) {
      int clusters = 0;
      cfg.gridDim = dim3(max_grid[dev]);
      FD_CHECK_CUDA(cudaOccupancyMaxActiveClusters(&clusters, Kern, &cfg));
      FD_REQUIRE(clusters > 0, "no cluster of %d CTAs with %d bytes of shared memory fits on device %d", cluster,
                 smem_bytes, dev);
      if (clusters * cluster < max_grid[dev]) max_grid[dev] = clusters * cluster;
    }
    attr_set[dev] = true;
  }
  const int grid = work_units < max_grid[dev] ? work_units : max_grid[dev];
  cfg.gridDim = dim3(grid - grid % cluster);
  FD_CHECK_CUDA(cudaLaunchKernelEx(&cfg, Kern, args...));
  return 0;
}


}  // namespace
