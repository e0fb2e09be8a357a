// Fused NSF-HiFiGAN ResBlock1 pair on wgmma (sm_90a):
//
//     x' = x + c2( lrelu( c1( lrelu(x) ) ) )          (reference models.py:103-110, one iteration of the loop)
//
// in ONE kernel per (c1, c2) pair.  HBM traffic per element: 4 bytes in (split planes of lrelu(x)) + 4 bytes out,
// against 24 for the two separate tap-GEMM launches with an fp32 residual master.
//
//   * the activation tile is loaded ONCE with its halo (ROWS + (k1-1)*d1 rows, one TMA box per 64-channel block, hi
//     and lo planes in separate boxes); every conv tap reads the SAME shared-memory tile, shifted by whole rows: the A
//     operand of each wgmma comes from registers (ldmatrix with the row offset of the tap; the 128/64/32-byte swizzle
//     of the TMA-written tile is undone in the addresses), the weights are the K-major shared-memory operand;
//   * c1's output never leaves the SM: the consumer warpgroups apply bias + LeakyReLU to their accumulators, split
//     them into hi/lo planes and write them into a second swizzled shared-memory tile that is c2's A operand;
//   * the residual x is recovered from the input tile (LeakyReLU is invertible) and, with c2's bias, becomes the initial
//     value of c2's accumulators, so the input tile is free for the next tile's TMA load while GEMM2 runs;
//   * the output goes through the mid tile as a swizzled staging image and TMA stores.
// A tile is ROWS = 16384 / C rows (every tile holds the same number of elements whatever the channel count, so the
// per-tile latency chain and the (k-1)-row halo are amortised over 1024 rows at C = 16); each of the two consumer
// warpgroups owns ROWS / 128 blocks of 64 rows, i.e. 64 fp32 accumulators per thread at every width.  A weight stage
// is used by all blocks of the tile before it is released, so the pair's weights stream through L2 -> shared memory
// once per tile.
//
// Warp roles (persistent, one CTA per SM): 0..7 = two consumer warpgroups, 8 = weight TMA producer,
// 9 = activation-tile TMA producer (warps 8..11 form the producer warpgroup, which gives its registers to the consumers).
#include <cuda.h>
#include <cstring>
#include "fd_common.cuh"
#include "fd_host.h"
#include "fd_tc_ptx.cuh"

namespace {

struct FdResPairK {
  int B, T;
  int k1, d1, k2;
  int h1, h2;        // halos of c1 / c2 in rows
  int r_in, rb, nbox;   // rows of the input tile = nbox TMA boxes of rb rows (rb a multiple of 8)
  int r_out;         // valid output rows per tile = ROWS - (k2-1)
  int nstages;       // stages of the weight ring (what the input tile of this launch leaves free)
  int group;         // weight units per stage of the ring
  int single;        // one product (hi planes only)
  float inv_s1, inv_s2, s2;
  float in_slope_inv, out_slope, planes_scale;
  const float* b1;
  const float* b2;
  // weight units (tap, K slice of BKW channels) that hold non-zero weights, in order, and per listed unit one bit per
  // K16 step (bit i * (BKW/16) + ks): the time-folded C = 16 convs are block-sparse (fd_respair_desc.kmask1/2)
  int n1, n2, masked1, masked2;
  unsigned long long km1, km2;
  unsigned char ul1[64], ul2[64];
};

template <int C>
struct RpCfg {
  static constexpr int ROWS = 16384 / C;
  static constexpr int BPW = ROWS / 128;                  // 64-row blocks per consumer warpgroup
  static constexpr int BK_A = C >= 64 ? 64 : C;          // channels per shared-memory activation block
  static constexpr int NKB = C / BK_A;
  static constexpr int ROWB = BK_A * 2;                   // bytes per activation row
  static constexpr uint32_t SWZ_A = ROWB == 128 ? 7u : ROWB == 64 ? 3u : 1u;
  static constexpr int NBOX_MAX = (ROWS + 56 + 255) / 256;
  static constexpr int RIN_MAX = ROWS + 56 + 8 * (NBOX_MAX - 1);
  static constexpr int MID_ROWS = ROWS + 16;              // + zero rows read by the trailing taps of c2
  static constexpr int BKW = C == 128 ? 32 : BK_A;        // K extent of one weight unit
  static constexpr int WROWB = BKW * 2;
  static constexpr uint32_t SWIZZLE_W = swizzle_mode_for(WROWB);
  static constexpr int UNIT_BYTES = 2 * C * WROWB;        // [2 planes][C rows][BKW]
  static constexpr int UNITS_PER_TAP = C / BKW;
  static constexpr int GROUP_RAW = 16384 / UNIT_BYTES;
  static constexpr int GROUP = GROUP_RAW > 8 ? 8 : GROUP_RAW;   // weight units per 16 KB pipeline stage
  static constexpr int MID_PLANE_BYTES = MID_ROWS * ROWB;
  static constexpr int MID_KB_BYTES = 2 * MID_PLANE_BYTES;
  static constexpr int MID_BYTES = NKB * MID_KB_BYTES;     // c1 output; afterwards the staging image of the output
  static constexpr int HEAD_BYTES = 2048;                   // biases (2C floats <= 1 KB) + barriers, in front of the tiles
  static_assert(2 * C * 4 + (2 * FD_TC_MAX_STAGES + 2) * 8 <= HEAD_BYTES, "head region too small");
  // stages of the weight ring for an input tile of r_in rows: the ring takes what the tiles leave of FD_TC_SMEM_BUDGET
  static constexpr int stages_for(int r_in, int group) {
    return fd_tc_ring_stages(1024 + HEAD_BYTES + NKB * 2 * r_in * ROWB + MID_BYTES, group * UNIT_BYTES);
  }
  static_assert(stages_for(RIN_MAX, GROUP) >= 2, "weight ring needs two stages");
};

__device__ __forceinline__ uint32_t swz(uint32_t off, uint32_t mask) { return off ^ (((off >> 7) & mask) << 4); }

__device__ __forceinline__ void fence_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void ldsm_x4(uint32_t addr, uint32_t (&r)[4]) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(addr) : "memory");
}
__device__ __forceinline__ uint32_t lds_u32(uint32_t addr) {
  uint32_t r;
  asm volatile("ld.shared.u32 %0, [%1];" : "=r"(r) : "r"(addr) : "memory");
  return r;
}
__device__ __forceinline__ void sts_u32(uint32_t addr, uint32_t x) {
  asm volatile("st.shared.u32 [%0], %1;" ::"r"(addr), "r"(x) : "memory");
}
__device__ __forceinline__ void tma_store_4d(const CUtensorMap* map, uint32_t smem_src, int c0, int c1, int c2, int c3) {
  asm volatile("cp.async.bulk.tensor.4d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5}], [%1];"
               ::"l"(reinterpret_cast<uint64_t>(map)), "r"(smem_src), "r"(c0), "r"(c1), "r"(c2), "r"(c3) : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
__device__ __forceinline__ void bulk_wait_read0() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
__device__ __forceinline__ void bulk_wait0() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }

// One conv of the pair over the whole tile: acc[j] (block j of this warpgroup) += A(shifted rows) x W for every listed
// weight unit.  A comes from the swizzled activation tile at a_base (a_kb bytes per 64-channel block, a_plane bytes
// from the hi to the lo plane), tap t reads rows shifted by t * tap_rows.
template <int C, int PREC>
__device__ __forceinline__ void rp_gemm(float* acc, const FdResPairK& p, int units, const unsigned char* ul,
                                        unsigned long long km, bool masked, uint32_t a_base, uint32_t a_kb,
                                        uint32_t a_plane, int tap_rows, int row0, uint32_t w_s, int stage_bytes,
                                        Ring& ring, int lane) {
  using K = RpCfg<C>;
  using MMA = Wgmma<C, PREC>;
  constexpr int KS = K::BKW / 16;
  constexpr uint32_t SBO_W = 8 * K::WROWB;
  // ldmatrix x4 addresses of the A fragment: lane -> row (lane & 7) + 8 ((lane >> 3) & 1), 8-channel chunk lane >> 4
  const int lrow = row0 + (lane & 7) + 8 * ((lane >> 3) & 1);
  const int lchunk = lane >> 4;
  const bool single = p.single != 0;
  int ui = 0;
#pragma unroll 1
  for (int u0 = 0; u0 < units; u0 += p.group) {
    const int nb = min(p.group, units - u0);
    ring.wait_full();
    const uint32_t w_stage = w_s + ring.stage * stage_bytes;
#pragma unroll 1
    for (int g = 0; g < nb; ++g, ++ui) {
      const int u = masked ? (int)ul[ui] : ui;      // dense convs: no table look-up on the issue path
      const int tap = u / K::UNITS_PER_TAP, kw = u % K::UNITS_PER_TAP;
      const uint32_t kbits = masked ? (uint32_t)(km >> (ui * KS)) & ((1u << KS) - 1u) : ((1u << KS) - 1u);
      const uint32_t w_hi = w_stage + g * K::UNIT_BYTES;
      const uint64_t dw_hi = make_smem_desc(w_hi, 16, SBO_W, K::SWIZZLE_W);
      const uint64_t dw_lo = make_smem_desc(w_hi + C * K::WROWB, 16, SBO_W, K::SWIZZLE_W);
      const int row = lrow + tap * tap_rows;
#pragma unroll
      for (int k = 0; k < KS; ++k) {
        if (!((kbits >> k) & 1u)) continue;             // an all-zero K16 slice of this tap
        const int ch = kw * K::BKW + 16 * k;
        const uint32_t a_addr = a_base + (uint32_t)(ch / K::BK_A) * a_kb +
                                swz((uint32_t)row * K::ROWB + (uint32_t)((ch % K::BK_A) / 8 + lchunk) * 16, K::SWZ_A);
        uint32_t ahi[K::BPW][4], alo[K::BPW][4];
#pragma unroll
        for (int j = 0; j < K::BPW; ++j) {
          ldsm_x4(a_addr + (uint32_t)(j * 64 * K::ROWB), ahi[j]);
          if (!single) ldsm_x4(a_addr + a_plane + (uint32_t)(j * 64 * K::ROWB), alo[j]);
        }
        wg_fence();
        const uint64_t adv = (uint64_t)((k * 32) >> 4);   // 16 elements * 2 B along K inside the swizzle row
#pragma unroll
        for (int j = 0; j < K::BPW; ++j)
          split_mma_rs<MMA>(acc + j * (C / 2), ahi[j], alo[j], dw_hi + adv, dw_lo + adv, single);
      }
    }
    wg_commit();
    wg_wait<0>();
    __syncwarp();
    if (lane == 0) mbar_arrive(&ring.empty[ring.stage]);
    ring.next();
  }
}

template <int C, int PREC>
__global__ void __launch_bounds__(FD_TC_THREADS, 1)
fd_respair_tc_kernel(const __grid_constant__ CUtensorMap tm_in, const __grid_constant__ CUtensorMap tm_w1,
                     const __grid_constant__ CUtensorMap tm_w2, const __grid_constant__ CUtensorMap tm_out,
                     const __grid_constant__ CUtensorMap tm_out_last, const FdResPairK p) {
  using K = RpCfg<C>;
  constexpr int NACC = K::BPW * (C / 2);
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  float* bias_s = reinterpret_cast<float*>(smem);                  // b1 [C] | b2 * s2 [C]
  uint64_t* w_full = reinterpret_cast<uint64_t*>(bias_s + 2 * C);
  uint64_t* w_empty = w_full + FD_TC_MAX_STAGES;
  uint64_t* in_full = w_empty + FD_TC_MAX_STAGES;
  uint64_t* in_empty = in_full + 1;
  const int in_plane = p.r_in * K::ROWB;                           // multiple of the swizzle period (rows % 8 == 0)
  const int in_kb = 2 * in_plane;
  const int STAGE_BYTES_RT = p.group * K::UNIT_BYTES;
  uint8_t* in_s = smem + K::HEAD_BYTES;
  uint8_t* mid_s = in_s + K::NKB * in_kb;
  uint8_t* w_s = mid_s + K::MID_BYTES;

  const int warp = threadIdx.x / 32;
  const int lane = threadIdx.x % 32;
  const int tiles_t = (p.T + p.r_out - 1) / p.r_out;
  const int num_tiles = p.B * tiles_t;

  if (threadIdx.x == 0) {
    for (int i = 0; i < p.nstages; ++i) { mbar_init(&w_full[i], 1); mbar_init(&w_empty[i], FD_TC_CONSUMER_THREADS / 32); }
    mbar_init(in_full, 1); mbar_init(in_empty, FD_TC_CONSUMER_THREADS / 32);
    fence_barrier_init();
  }
  if (warp == FD_TC_PRODUCER_WARP && lane == 0) {
    prefetch_tmap(&tm_in); prefetch_tmap(&tm_w1); prefetch_tmap(&tm_w2); prefetch_tmap(&tm_out); prefetch_tmap(&tm_out_last);
  }
  // biases (b2 pre-multiplied by the weight prescale of c2); the 16 trailing rows of the mid tile are zero for the whole kernel
  for (int i = threadIdx.x; i < C; i += blockDim.x) { bias_s[i] = p.b1[i]; bias_s[C + i] = p.b2[i] * p.s2; }
  for (int i = threadIdx.x; i < K::NKB * 2 * K::ROWB; i += blockDim.x)      // 16 rows = ROWB 16-byte chunks per plane
    *reinterpret_cast<uint4*>(mid_s + (i / K::ROWB) * K::MID_PLANE_BYTES + K::ROWS * K::ROWB + (i % K::ROWB) * 16) =
        make_uint4(0, 0, 0, 0);
  __syncthreads();

  if (warp >= FD_TC_PRODUCER_WARP) producer_regs();
  if (warp == FD_TC_PRODUCER_WARP) {
    // =========================================================== weight producer (the pair's weights, once per tile)
    if (lane == 0) {
      Ring ring{w_full, w_empty, p.nstages};
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        for (int g2 = 0; g2 < 2; ++g2) {
          const CUtensorMap* tm = g2 == 0 ? &tm_w1 : &tm_w2;
          const int units = g2 == 0 ? p.n1 : p.n2;
          const unsigned char* ul = g2 == 0 ? p.ul1 : p.ul2;
          const bool pmasked = (g2 == 0 ? p.masked1 : p.masked2) != 0;
          for (int u0 = 0; u0 < units; u0 += p.group) {
            const int nb = min(p.group, units - u0);
            ring.wait_empty();
            mbar_expect_tx(ring.full_bar(), nb * K::UNIT_BYTES);
            uint8_t* slot = w_s + ring.stage * STAGE_BYTES_RT;
            for (int g = 0; g < nb; ++g) {
              const int u = pmasked ? (int)ul[u0 + g] : u0 + g;
              const int tap = u / K::UNITS_PER_TAP, kw = u % K::UNITS_PER_TAP;
              tma_load_3d(slot + g * K::UNIT_BYTES, tm, ring.full_bar(), tap * C + kw * K::BKW, 0, 0);
            }
            ring.next();
          }
        }
      }
    }
    return;
  }
  if (warp >= FD_TC_PRODUCER_WARP + 1) {
    // =========================================================== activation-tile producer
    if (warp == FD_TC_PRODUCER_WARP + 1 && lane == 0) {
      uint32_t it = 0;
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x, ++it) {
        const int b = tile / tiles_t, t0 = (tile % tiles_t) * p.r_out;
        mbar_wait(in_empty, (it & 1) ^ 1);
        mbar_expect_tx(in_full, K::NKB * 2 * p.r_in * K::ROWB);
        for (int kb = 0; kb < K::NKB; ++kb)
          for (int pl = 0; pl < 2; ++pl)
            for (int bx = 0; bx < p.nbox; ++bx)
              tma_load_4d(in_s + kb * in_kb + pl * in_plane + bx * p.rb * K::ROWB, &tm_in, in_full,
                          kb * K::BK_A, t0 - p.h2 - p.h1 + bx * p.rb, b, pl);
      }
    }
    return;
  }

  // =========================================================== consumers
  consumer_regs();
  const int wg = warp / 4, wq = warp % 4;
  const int blk0 = wg * K::BPW;                      // first 64-row block of this warpgroup
  const int frow = 16 * wq + (lane >> 2);            // fragment row inside a 64-row block (and + 8)
  const int fcol = 2 * (lane & 3);                   // fragment column inside an 8-column group
  const bool issuer = threadIdx.x == 0;              // issues the output TMA stores
  const uint32_t in_u = smem_u32(in_s), mid_u = smem_u32(mid_s), w_u = smem_u32(w_s);
  const float slope_mid = 0.1f;
  const float s2_neg = p.s2 * p.in_slope_inv;
  const float out_c = p.inv_s2 * p.planes_scale, out_cs = out_c * p.out_slope;
  float acc[NACC];
  Ring ring{w_full, w_empty, p.nstages};
  uint32_t it = 0;
  for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x, ++it) {
    const int b = tile / tiles_t, t0 = (tile % tiles_t) * p.r_out;

    // ---- GEMM1: mid rows m = block row, input tile rows m + tap * d1
#pragma unroll
    for (int i = 0; i < NACC; ++i) acc[i] = 0.f;
    mbar_wait(in_full, it & 1);
    rp_gemm<C, PREC>(acc, p, p.n1, p.ul1, p.km1, p.masked1 != 0, in_u, in_kb, in_plane, p.d1, blk0 * 64 + 16 * wq,
                     w_u, STAGE_BYTES_RT, ring, lane);
    wg_fence_operand(acc);

    // ---- epilogue 1: bias, LeakyReLU, zero outside [0,T), split planes -> mid tile (c2's A operand).  The mid tile is
    //      also the staging image of the previous tile's output: its TMA stores must have read it.
    if (issuer) bulk_wait_read0();
    named_bar_sync<1, FD_TC_CONSUMER_THREADS>();
#pragma unroll
    for (int j = 0; j < K::BPW; ++j) {
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int m = (blk0 + j) * 64 + frow + 8 * h;
        const int t = t0 - p.h2 + m;
        const bool ok = t >= 0 && t < p.T;
#pragma unroll
        for (int g8 = 0; g8 < C / 8; ++g8) {
          const int col = 8 * g8 + fcol;
          const float* a = acc + j * (C / 2) + 4 * g8 + 2 * h;
          const float y0 = fmaf(a[0], p.inv_s1, bias_s[col]);
          const float y1 = fmaf(a[1], p.inv_s1, bias_s[col + 1]);
          uint32_t hi, lo;
          fd_split2(ok ? fmaxf(y0, slope_mid * y0) : 0.f, ok ? fmaxf(y1, slope_mid * y1) : 0.f, PREC, hi, lo);
          const uint32_t off = (uint32_t)(col / K::BK_A) * K::MID_KB_BYTES +
                               swz((uint32_t)m * K::ROWB + (uint32_t)((col % K::BK_A) / 8) * 16, K::SWZ_A) +
                               (uint32_t)(col % 8) * 2;
          sts_u32(mid_u + off, hi);
          sts_u32(mid_u + K::MID_PLANE_BYTES + off, lo);
        }
      }
    }
    // ---- residual + c2 bias -> initial accumulators of GEMM2 (pre-scaled by the weight prescale of c2); output row r
    //      (time t0 + r) is input tile row r + h1 + h2
#pragma unroll
    for (int j = 0; j < K::BPW; ++j) {
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int n = (blk0 + j) * 64 + frow + 8 * h + p.h1 + p.h2;
#pragma unroll
        for (int g8 = 0; g8 < C / 8; ++g8) {
          const int col = 8 * g8 + fcol;
          const uint32_t off = (uint32_t)(col / K::BK_A) * in_kb +
                               swz((uint32_t)n * K::ROWB + (uint32_t)((col % K::BK_A) / 8) * 16, K::SWZ_A) +
                               (uint32_t)(col % 8) * 2;
          float a0, a1;
          fd_combine2(lds_u32(in_u + off), lds_u32(in_u + in_plane + off), PREC, a0, a1);
          // x = p >= 0 ? p : p / slope (the planes hold lrelu(x)); (x + b2) * s2 as one fma
          float* a = acc + j * (C / 2) + 4 * g8 + 2 * h;
          a[0] = fmaf(a0, a0 >= 0.f ? p.s2 : s2_neg, bias_s[C + col]);
          a[1] = fmaf(a1, a1 >= 0.f ? p.s2 : s2_neg, bias_s[C + col + 1]);
        }
      }
    }
    __syncwarp();
    if (lane == 0) mbar_arrive(in_empty);            // this warp is done with the input tile
    named_bar_sync<1, FD_TC_CONSUMER_THREADS>();     // the whole mid tile is written

    // ---- GEMM2: output rows r, mid rows r + tap
    rp_gemm<C, PREC>(acc, p, p.n2, p.ul2, p.km2, p.masked2 != 0, mid_u, K::MID_KB_BYTES, K::MID_PLANE_BYTES, 1,
                     blk0 * 64 + 16 * wq, w_u, STAGE_BYTES_RT, ring, lane);
    wg_fence_operand(acc);
    named_bar_sync<1, FD_TC_CONSUMER_THREADS>();     // every warpgroup is done reading the mid tile

    // ---- epilogue 2: lrelu(acc * inv_s2) * planes_scale -> split planes -> staging image (mid tile) -> TMA stores
#pragma unroll
    for (int j = 0; j < K::BPW; ++j) {
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int m = (blk0 + j) * 64 + frow + 8 * h;
#pragma unroll
        for (int g8 = 0; g8 < C / 8; ++g8) {
          const int col = 8 * g8 + fcol;
          const float* a = acc + j * (C / 2) + 4 * g8 + 2 * h;
          uint32_t hi, lo;      // lrelu(a * inv_s2) * planes_scale = max(a * c, a * c * slope), 0 <= slope <= 1
          fd_split2(fmaxf(a[0] * out_c, a[0] * out_cs), fmaxf(a[1] * out_c, a[1] * out_cs), PREC, hi, lo);
          const uint32_t off = (uint32_t)(col / K::BK_A) * K::MID_KB_BYTES +
                               swz((uint32_t)m * K::ROWB + (uint32_t)((col % K::BK_A) / 8) * 16, K::SWZ_A) +
                               (uint32_t)(col % 8) * 2;
          sts_u32(mid_u + off, hi);
          sts_u32(mid_u + K::MID_PLANE_BYTES + off, lo);
        }
      }
    }
    fence_async_smem();
    named_bar_sync<1, FD_TC_CONSUMER_THREADS>();
    if (issuer) {
      for (int j = 0; j < K::ROWS / 128; ++j) {
        const CUtensorMap* tm = j == K::ROWS / 128 - 1 ? &tm_out_last : &tm_out;
        for (int kb = 0; kb < K::NKB; ++kb)
          for (int pl = 0; pl < 2; ++pl)
            tma_store_4d(tm, mid_u + kb * K::MID_KB_BYTES + pl * K::MID_PLANE_BYTES + (uint32_t)(j * 128) * K::ROWB,
                         kb * K::BK_A, t0 + j * 128, b, pl);
      }
      bulk_commit();
    }
  }
  if (issuer) bulk_wait0();
}

// ------------------------------------------------------------------ host side
template <int C, int PREC>
int launch_respair(const fd_respair_desc& d, FdResPairK p, cudaStream_t stream) {
  using K = RpCfg<C>;
  // tile geometry: ROWS rows; the input tile is nbox TMA boxes of rb rows
  const int need = K::ROWS + (p.k1 - 1) * p.d1;
  p.nbox = (need + 255) / 256;
  p.rb = ((need + p.nbox - 1) / p.nbox + 7) / 8 * 8;
  p.r_in = p.nbox * p.rb;
  p.r_out = K::ROWS - (p.k2 - 1);
  FD_REQUIRE(p.r_in <= K::RIN_MAX && p.rb <= 256, "fd_respair_fwd: input tile of %d rows exceeds the shared-memory tile", p.r_in);
  // a stage of the ring holds 2 x GROUP weight units (32 KB) when at least two such stages fit: fewer, larger stages
  // mean fewer barrier round trips per tile
  p.group = K::stages_for(p.r_in, 2 * K::GROUP) >= 2 ? 2 * K::GROUP : K::GROUP;
  p.nstages = K::stages_for(p.r_in, p.group);
  // planes [2][B][T][C], one plane per box; weights [2][C][k C], both planes of a unit in one box
  const long long rs = C, is = (long long)p.T * C, ps = (long long)p.B * p.T * C;
  CUtensorMap tin, tw1, tw2, tout, tout_last;
  int rc = planes_map(&tin, d.in_planes, C, p.T, p.B, rs, is, ps, K::BK_A, p.rb, 1, "respair in");
  if (rc) return rc;
  rc = weights_map(&tw1, d.w1, C, p.k1 * C, K::BKW, C, 2, "respair w1");
  if (rc) return rc;
  rc = weights_map(&tw2, d.w2, C, p.k2 * C, K::BKW, C, 2, "respair w2");
  if (rc) return rc;
  rc = planes_map(&tout, d.out_planes, C, p.T, p.B, rs, is, ps, K::BK_A, 128, 1, "respair out");
  if (rc) return rc;
  rc = planes_map(&tout_last, d.out_planes, C, p.T, p.B, rs, is, ps, K::BK_A, 128 - (p.k2 - 1), 1, "respair out_last");
  if (rc) return rc;
  const int tiles = p.B * ((p.T + p.r_out - 1) / p.r_out);
  return fd_tc_launch<fd_respair_tc_kernel<C, PREC>>(FD_TC_SMEM_BUDGET, tiles, stream, true, 1, tin, tw1, tw2, tout,
                                                     tout_last, p);
}

template <int C>
int launch_respair_prec(const fd_respair_desc& d, const FdResPairK& p, cudaStream_t stream) {
  return (d.prec & 0xF) == FD_F16 ? launch_respair<C, FD_F16>(d, p, stream) : launch_respair<C, FD_BF16>(d, p, stream);
}

}  // namespace

extern "C" int fd_respair_supported(int C, int k1, int d1, int k2) {
  if (C != 16 && C != 32 && C != 64 && C != 128) return 0;
  if (k1 < 1 || k2 < 1 || (k1 & 1) == 0 || (k2 & 1) == 0 || d1 < 1) return 0;
  if (k2 - 1 > 16) return 0;                             // zero rows behind the mid tile
  if ((k1 - 1) * d1 > 56) return 0;                      // halo rows of the input tile
  if ((k2 - 1) / 2 > (k1 - 1) / 2 * d1) return 0;       // the residual rows must lie inside the input tile
  return 1;
}

extern "C" int fd_respair_fwd(const fd_respair_desc* d, void* stream) {
  FD_DEVICE_GUARD();
  FD_REQUIRE(d != nullptr, "fd_respair_fwd: null descriptor");
  FD_REQUIRE(fd_respair_supported(d->C, d->k1, d->d1, d->k2), "fd_respair_fwd: unsupported shape C=%d k1=%d d1=%d k2=%d",
             d->C, d->k1, d->d1, d->k2);
  FD_REQUIRE(d->B > 0 && d->T > 0, "fd_respair_fwd: bad shape B=%d T=%d", d->B, d->T);
  FD_REQUIRE(d->in_planes && d->w1 && d->w2 && d->b1 && d->b2 && d->out_planes, "fd_respair_fwd: null pointer");
  FD_REQUIRE(d->in_slope > 0.f && d->in_slope <= 1.f, "fd_respair_fwd: the input LeakyReLU slope must be in (0, 1] (it is inverted)");
  FD_REQUIRE(d->out_slope >= 0.f && d->out_slope <= 1.f, "fd_respair_fwd: the output LeakyReLU slope must be in [0, 1]");
  FD_REQUIRE((const void*)d->out_planes != (const void*)d->in_planes, "fd_respair_fwd: in-place is not supported (halo reads)");
  FdResPairK p;
  memset(&p, 0, sizeof(p));
  p.B = d->B; p.T = d->T; p.k1 = d->k1; p.d1 = d->d1; p.k2 = d->k2;
  p.h1 = (d->k1 - 1) / 2 * d->d1; p.h2 = (d->k2 - 1) / 2;
  p.single = (d->prec & FD_SINGLE) ? 1 : 0;
  p.inv_s1 = d->w1_inv_scale; p.inv_s2 = d->w2_inv_scale; p.s2 = 1.f / d->w2_inv_scale;
  p.in_slope_inv = 1.f / d->in_slope; p.out_slope = d->out_slope; p.planes_scale = d->planes_scale;
  p.b1 = d->b1; p.b2 = d->b2;
  {
    // weight units of BKW channels per tap (BKW as in RpCfg: 32 at C = 128, else min(C, 64)) and their K16 steps
    const int bkw = d->C == 128 ? 32 : (d->C >= 64 ? 64 : d->C), upt = d->C / bkw, ks = bkw / 16, kst = d->C / 16;
    FD_REQUIRE(d->k1 * upt <= 64 && d->k2 * upt <= 64, "fd_respair_fwd: more than 64 weight units (k1=%d k2=%d C=%d)", d->k1,
               d->k2, d->C);
    auto fill = [&](int k, unsigned long long kmask, unsigned char* ul, int& n, unsigned long long& km) {
      n = 0; km = 0;
      const bool masked = kmask != 0ull && k * kst <= 64;
      if (masked) {
        for (int u = 0; u < k * upt; ++u) {
          const unsigned bits = (unsigned)(kmask >> ((u / upt) * kst + (u % upt) * ks)) & ((1u << ks) - 1u);
          if (bits) { km |= (unsigned long long)bits << (n * ks); ul[n++] = (unsigned char)u; }
        }
      }
      if (n == 0) {                    // dense (or a mask without any set bit inside the conv)
        for (int u = 0; u < k * upt; ++u) ul[u] = (unsigned char)u;
        n = k * upt; km = 0;
        return false;
      }
      return true;
    };
    const bool m1 = fill(d->k1, d->kmask1, p.ul1, p.n1, p.km1), m2 = fill(d->k2, d->kmask2, p.ul2, p.n2, p.km2);
    p.masked1 = m1 ? 1 : 0; p.masked2 = m2 ? 1 : 0;
  }
  cudaStream_t st = (cudaStream_t)stream;
  int rc;
  fd_prof_begin(d->C == 128 ? 12 : d->C == 64 ? 13 : d->C == 32 ? 14 : 15, st);
  switch (d->C) {
    case 128: rc = launch_respair_prec<128>(*d, p, st); break;
    case 64: rc = launch_respair_prec<64>(*d, p, st); break;
    case 32: rc = launch_respair_prec<32>(*d, p, st); break;
    default: rc = launch_respair_prec<16>(*d, p, st); break;
  }
  fd_prof_end(st);
  if (rc == 0) fd_count_launch(1);
  return rc;
}
