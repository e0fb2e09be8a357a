// wgmma / TMA tap-GEMM for sm_90a.
//
//   D[b,t,n] = sum_seg sum_k  A_seg[b, t+shift_seg, c_off_seg+k] * W[n, koff_seg+k]
//
// A (activations) and W (packed weights) are stored as 16-bit split planes (see fd_common.cuh).
// One persistent CTA per SM, warp-specialised:
//   warp 8      : TMA producer  (the third warpgroup, warps 8..11, gives its registers to the consumers; cp.async.bulk.tensor, 128B/64B/32B swizzle, OOB rows zero-filled: that is how the
//                 conv zero padding and the time shift of each tap are realised; the hi and lo planes of an operand
//                 arrive in one box)
//   warps 0..7  : two consumer warpgroups.  Each issues wgmma.mma_async m64nBLOCK_Nk16 (three products per k16 step --
//                 lo*hi + hi*lo + hi*hi -- or one in single-product mode; fp32 accumulation in registers) and then runs
//                 the fused epilogue on its own accumulators: chunks of columns go through a warp-private shared-memory
//                 scratch into a layout with coalesced global accesses.
// Two schedules:
//   cooperative (LINEAR, MAG, GATE_BWD; fd_tapgemm_tc_kernel): the warpgroups share a 128-row tile, one 64-row half
//     each, and run the mainloop and then the epilogue together; the producer runs ahead into the next tile while the
//     consumers are in the epilogue.
//   ping-pong (GATE, RES_SKIP -- the WaveNet GEMMs; fd_tapgemm_pp_kernel): each warpgroup owns a whole 64-row tile and
//     the warpgroups take alternate tiles; their mainloops take turns at the tensor cores, so one warpgroup's epilogue
//     runs during the other's mainloop.  CTAs run in 2x1x1 clusters: the two CTAs of a pair work on adjacent 64-row
//     tiles with the same column tile and each stages half of the W box into both (TMA multicast), so W is read from
//     L2 once per 128 rows as in the cooperative schedule.
//   The sampler's GATE (three products, conditioner projection in the epilogue) runs the ping-pong schedule with the
//   operands swapped (fd_gate_t_kernel, "transposed GATE" below).
// Pipeline: smem full/empty ring between the producer and the consumers.
#include <cuda.h>
#include "fd_common.cuh"
#include "fd_host.h"
#include "fd_tc_ptx.cuh"

namespace {

constexpr int BLOCK_M = 128;   // rows of a cooperative tile; a ping-pong tile is one warpgroup's 64

// NPL = operand planes staged per k-block: 2 (hi + lo, three products) or 1 (hi only, one product: 11-bit (f16) /
// 8-bit (bf16) operand mantissas, the arithmetic of a plain half-precision tensor-core GEMM with fp32 accumulation).
template <int BLOCK_N, int BLOCK_K, int EPI, int NPL>
struct Cfg {
  static constexpr bool PP = EPI == FD_EPI_GATE || EPI == FD_EPI_RES_SKIP;   // ping-pong schedule
  static constexpr int ROWS = PP ? 64 : BLOCK_M;                            // A rows staged per k-block
  static constexpr int A_BYTES = ROWS * BLOCK_K * 2;
  static constexpr int W_BYTES = BLOCK_N * BLOCK_K * 2;
  // One pipeline stage holds GROUP consecutive k-blocks (64 K-elements worth): with narrow channel counts a k-block
  // is a single conv tap of 16 or 32 channels, and one barrier round trip per tap is what bounds the small-channel
  // vocoder stages.  hi and lo planes of an operand arrive in ONE TMA box (plane dimension = 2).  The WaveNet GEMMs
  // (GATE, RES_SKIP) take BLOCK_K 32 only where a 64-wide ring would have 2 stages (see pick_cfg), and then keep one
  // k-block per stage: the point is a deeper ring, not fewer barrier round trips.
  static constexpr int GROUP = BLOCK_K >= 64 || PP ? 1 : 64 / BLOCK_K;
  static constexpr int SUB_BYTES = NPL * (A_BYTES + W_BYTES);           // multiple of 1024 for every instantiation
  static constexpr int STAGE_BYTES = GROUP * SUB_BYTES;
  static constexpr int TX_BYTES = SUB_BYTES;                            // per k-block
  static constexpr int SWIZZLE_BYTES = BLOCK_K * 2;                       // 128 / 64 / 32
  static constexpr uint32_t SWIZZLE_MODE = swizzle_mode_for(SWIZZLE_BYTES);
  static constexpr uint32_t SBO = 8 * SWIZZLE_BYTES;
  static constexpr int BIAS_FLOATS = (EPI == FD_EPI_GATE ? 3 : 1) * BLOCK_N;   // one copy of the bias vectors
  static constexpr int BIAS_TOTAL = (PP ? 2 : 1) * BIAS_FLOATS;               // ping-pong: one copy per warpgroup
  static constexpr int NUM_STAGES = fd_tc_frame_stages(STAGE_BYTES, BIAS_TOTAL);
  static constexpr int SMEM_BYTES = fd_tc_frame_bytes(NUM_STAGES, STAGE_BYTES, BIAS_TOTAL);
  static_assert(NUM_STAGES >= 2, "pipeline needs at least two stages");
  static_assert(SMEM_BYTES <= FD_TC_SMEM_BUDGET, "shared memory");
};

// the per-column bias vectors of column tile n0 of item b into shared memory, by threads i0, i0 + step, ...
template <int BLOCK_N, int EPI>
__device__ __forceinline__ void stage_bias(const FdTapGemm& p, int b, int n0, float* bias_s, int i0, int step) {
  if (EPI == FD_EPI_GATE) {
    const size_t bo = (size_t)b * p.gbias_bstride + n0;
    for (int i = i0; i < BLOCK_N; i += step) {
      bias_s[i] = p.gbias_full[bo + i];
      bias_s[BLOCK_N + i] = p.gbias_lo[bo + i];
      bias_s[2 * BLOCK_N + i] = p.gbias_hi[bo + i];
    }
  } else {
    for (int i = i0; i < BLOCK_N; i += step)
      bias_s[i] = p.bias ? p.bias[(size_t)b * p.bias_bstride + n0 + i] : 0.f;
  }
}
template <int EPI>
__device__ __forceinline__ long long bias_key(const FdTapGemm& p, int b, int n0) {
  return EPI == FD_EPI_GATE ? (long long)b * p.gbias_bstride + n0 : (long long)b * p.bias_bstride + n0;
}

// The fused epilogue of one warp: its 16 rows (time steps rw0 .. rw0 + 15 of item b) x BLOCK_N columns (column tile
// n_tile) of the wgmma accumulator fragment `acc`; bias_s holds the tile's bias vectors, `my_scratch` is the warp's
// shared-memory scratch.
template <int BLOCK_N, int EPI, int PREC>
__device__ __forceinline__ void tile_epilogue(const FdTapGemm& p, const float* acc, int b, int n_tile, int rw0,
                                              const float* bias_s, uint32_t my_scratch, int lane) {
  const int n0 = n_tile * BLOCK_N;
  if constexpr (EPI == FD_EPI_GATE || EPI == FD_EPI_MAG) {
    // 16 gate columns and the matching 16 filter columns per step; lane -> row lane/2, 8 columns (lane % 2)
    constexpr int HALF = BLOCK_N / 2;       // gate columns | filter columns
    const uint32_t sb = smem_u32(bias_s);
    const int r = lane >> 1, sub = lane & 1;
    const int t = rw0 + r;
    const bool valid = t < p.T;
    const bool e_lo = t < p.dil, e_hi = t + p.dil >= p.T;
    const bool edge_any = __any_sync(0xffffffffu, valid && (e_lo || e_hi));
    const size_t zplane = (size_t)p.B * p.T * p.C, zrow = ((size_t)b * p.T + t) * p.C + (size_t)n_tile * HALF;
    const size_t yplane = (size_t)p.B * p.T * p.n_total, yrow = ((size_t)b * p.T + t) * p.n_total;
#pragma unroll
    for (int c = 0; c < HALF; c += 16) {
      frag_to_scratch<16>(my_scratch, acc, c, 0, lane);
      frag_to_scratch<16>(my_scratch, acc, HALF + c, 16, lane);
      __syncwarp();
      float g[8], f[8];
      {
        const float4 g0 = scratch_ld4(my_scratch, r, 2 * sub), g1 = scratch_ld4(my_scratch, r, 2 * sub + 1);
        const float4 f0 = scratch_ld4(my_scratch, r, 4 + 2 * sub), f1 = scratch_ld4(my_scratch, r, 5 + 2 * sub);
        g[0] = g0.x; g[1] = g0.y; g[2] = g0.z; g[3] = g0.w; g[4] = g1.x; g[5] = g1.y; g[6] = g1.z; g[7] = g1.w;
        f[0] = f0.x; f[1] = f0.y; f[2] = f0.z; f[3] = f0.w; f[4] = f1.x; f[5] = f1.y; f[6] = f1.z; f[7] = f1.w;
      }
      __syncwarp();
      const int cc = c + 8 * sub;            // gate column inside the tile's gate half
      if (valid) {
        if (EPI == FD_EPI_MAG) {
          fd_epi_mag<8, PREC>(p, b, t, n_tile * HALF + cc, g, f);
        } else {
          // the addend (conditioner projection, packed columns n0 + cc and n0 + HALF + cc of this row) is issued before
          // the shared-space bias loads; it is read once per launch, so it streams past L2 (evict-first).  The
          // zero-padding corrections of the first / last `dilation` rows are skipped by a warp vote where no lane
          // needs them.
          float add[2][8], bias[2][8], lo[2][8], hi[2][8], z[8];
          if (p.addend != nullptr) {
#pragma unroll
            for (int h = 0; h < 2; ++h) ldcs_f32(p.addend + yrow + n0 + h * HALF + cc, add[h]);
          }
#pragma unroll
          for (int h = 0; h < 2; ++h) lds_f32(sb + 4u * (h * HALF + cc), bias[h]);
          if (edge_any) {
#pragma unroll
            for (int h = 0; h < 2; ++h)
              if (e_lo) lds_f32(sb + 4u * (BLOCK_N + h * HALF + cc), lo[h]);
#pragma unroll
            for (int h = 0; h < 2; ++h)
              if (e_hi) lds_f32(sb + 4u * (2 * BLOCK_N + h * HALF + cc), hi[h]);
          }
          fd_epi_gate<8>(p, t, g, f, z, bias, add, lo, hi);
          if (p.y_planes != nullptr) {   // training: keep the pre-activations (packed column order: gates | filters per tile)
            const int ng = p.gate_tile == BLOCK_N ? n0 + cc : fd_gate_col(p, n_tile * HALF + cc);
            fd_store_planes<8>(p.y_planes, yplane, yrow + ng, g, PREC);
            fd_store_planes<8>(p.y_planes, yplane, yrow + ng + p.gate_tile / 2, f, PREC);
          }
          fd_store_planes<8>(p.out_planes, zplane, zrow + cc, z, PREC);
        }
      }
    }
  } else if constexpr (BLOCK_N >= 64) {
    // ---- LINEAR / RES_SKIP / GATE_BWD, coalescing epilogue: 32-column chunks; lane -> rows rbase + 4 r (r < 4),
    //      columns 4 (lane % 8) .. + 3 of the chunk, so that 8 lanes cover one 128-byte row segment
    const uint32_t bias_addr = smem_u32(bias_s);
    const int j4 = (lane & 7) * 4, rsub = lane >> 3;
    const int rbase = rw0 + rsub;                      // time index of row 0
    const FdRows<uint32_t> rows{(uint32_t)b * (uint32_t)p.T, rbase, 4,
                                rbase < p.T ? min(4, (p.T - rbase + 3) / 4) : 0};
#pragma unroll
    for (int c = 0; c < BLOCK_N; c += 32) {
      const int col = c + j4;                          // first of this lane's 4 columns inside the tile
      const int n = n0 + col;                          // global packed column
      frag_to_scratch<32>(my_scratch, acc, c, 0, lane);
      __syncwarp();
      float a[4][4];
#pragma unroll
      for (int r = 0; r < 4; ++r) {
        const float4 x = scratch_ld4(my_scratch, 4 * r + rsub, lane & 7);
        a[r][0] = x.x; a[r][1] = x.y; a[r][2] = x.z; a[r][3] = x.w;
      }
      __syncwarp();
      if constexpr (EPI == FD_EPI_GATE_BWD) {
        // the 4 lanes that share these columns are lane bits 3 and 4; the warp's 16 rows decide the edge flags
        FdColSums<4> s{};
        fd_epi_gate_bwd<4, 4, PREC>(p, rows, n, a, s);
        fd_gate_bwd_colsums<8>(p, s, rw0 < p.dil, rw0 + 16 + p.dil > p.T, rsub == 0, b, n);
      } else {
        float bias[4];
        lds_f32(bias_addr + 4u * col, bias);
        if constexpr (EPI == FD_EPI_RES_SKIP) fd_epi_res_skip<4, 4, PREC>(p, rows, n, n0 < p.C, a, bias);   // C % BLOCK_N == 0
        else fd_epi_linear<4, 4, PREC>(p, rows, n, a, bias);
      }
    }
  } else {
    // ---- LINEAR with narrow tiles (BLOCK_N <= 32; pick_cfg gives RES_SKIP and GATE_BWD no tile under 64 columns):
    //      row-owner epilogue; lane -> row lane/2, BLOCK_N/2 columns (lane % 2) in groups of 8
    static_assert(EPI == FD_EPI_LINEAR, "narrow tiles: LINEAR only");
    constexpr int PER = BLOCK_N / 2;
    frag_to_scratch<BLOCK_N>(my_scratch, acc, 0, 0, lane);
    __syncwarp();
    const int r = lane >> 1, sub = lane & 1;
    float v[PER];
#pragma unroll
    for (int q4 = 0; q4 < PER / 4; ++q4) {
      const float4 x = scratch_ld4(my_scratch, r, sub * (PER / 4) + q4);
      v[4 * q4] = x.x; v[4 * q4 + 1] = x.y; v[4 * q4 + 2] = x.z; v[4 * q4 + 3] = x.w;
    }
    __syncwarp();
    const int t = rw0 + r;
    const FdRows<uint32_t> row{(uint32_t)b * (uint32_t)p.T, t, 1, t < p.T ? 1 : 0};
#pragma unroll
    for (int h = 0; h < PER / 8; ++h) {
      const int cc = sub * PER + h * 8;
      float a[1][8], bias[8];
#pragma unroll
      for (int i = 0; i < 8; ++i) a[0][i] = v[h * 8 + i];
      lds_f32(smem_u32(bias_s) + 4u * cc, bias);
      fd_epi_linear<1, 8, PREC>(p, row, n0 + cc, a, bias);
    }
  }
}

// ------------------------------------------------------------------ cooperative schedule (LINEAR, MAG, GATE_BWD)
template <int BLOCK_N, int BLOCK_K, int EPI, int PREC, int NPL>
__global__ void __launch_bounds__(FD_TC_THREADS, 1)
fd_tapgemm_tc_kernel(const __grid_constant__ CUtensorMap tm_src0, const __grid_constant__ CUtensorMap tm_src1,
                     const __grid_constant__ CUtensorMap tm_w, const FdTapGemm p) {
  using C = Cfg<BLOCK_N, BLOCK_K, EPI, NPL>;
  static_assert(!C::PP, "GATE / RES_SKIP run the ping-pong schedule");
  using MMA = Wgmma<BLOCK_N, PREC>;
  extern __shared__ uint8_t smem_raw[];
  const TcFrame f = tc_frame(smem_raw, C::NUM_STAGES, C::STAGE_BYTES, C::BIAS_TOTAL);
  Ring ring{f.full, f.empty, C::NUM_STAGES};

  const int warp = threadIdx.x / 32;
  const int lane = threadIdx.x % 32;

  const int tiles_t = (p.T + BLOCK_M - 1) / BLOCK_M;
  const int num_m_tiles = p.B * tiles_t;
  const int num_n_tiles = p.n_total / BLOCK_N;
  const int num_tiles = num_m_tiles * num_n_tiles;
  int total_k_blocks = 0;
  for (int sI = 0; sI < p.num_seg; ++sI) total_k_blocks += p.seg[sI].k_len / BLOCK_K;

  tc_prologue<false>(f, C::NUM_STAGES, FD_TC_CONSUMER_THREADS / 32, &tm_src0, &tm_src1, &tm_w);

  if (warp >= FD_TC_PRODUCER_WARP) {
    // =========================================================== TMA producer
    producer_regs();
    if (warp == FD_TC_PRODUCER_WARP && lane == 0) {
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        const int m_tile = tile / num_n_tiles;
        // rotate the column tile with the row tile: with a grid that is a multiple of num_n_tiles every CTA would
        // otherwise see the same n-tile forever, and epilogue costs differ per n-tile (residual vs skip columns)
        const int n_tile = (tile % num_n_tiles + m_tile) % num_n_tiles;
        const int b = m_tile / tiles_t, t0 = (m_tile % tiles_t) * BLOCK_M;
        const int n0 = n_tile * BLOCK_N;
        SegCursor sc;
        for (int kb = 0; kb < total_k_blocks; kb += C::GROUP) {
          const int nb = min(C::GROUP, total_k_blocks - kb);
          ring.wait_empty();
          uint8_t* st = f.ring + ring.stage * C::STAGE_BYTES;
          mbar_expect_tx(ring.full_bar(), nb * C::TX_BYTES);
          for (int g = 0; g < nb; ++g) {
            const FdSeg sg = p.seg[sc.s];
            const CUtensorMap* tm = sg.src == 0 ? &tm_src0 : &tm_src1;
            uint8_t* sub = st + g * C::SUB_BYTES;
            tma_load_4d(sub, tm, ring.full_bar(), sg.c_off + sc.k0, t0 + sg.shift, b, 0);          // hi + lo planes
            const int kw = sc.koff + sc.k0 + p.w_kshift;
            tma_load_3d(sub + NPL * C::A_BYTES, &tm_w, ring.full_bar(), kw, n0, 0);                 // hi + lo planes
            sc.next(BLOCK_K, sg.k_len);
          }
          ring.next();
        }
      }
    }
    return;
  }

  // =========================================================== consumers: wgmma mainloop + epilogue
  consumer_regs();
  const int wg = warp / 4;                                   // rows [64 wg, 64 wg + 64) of the tile
  const int wq = warp % 4;                                   // 16-row slice of the warpgroup's 64 rows
  const uint32_t my_scratch = smem_u32(f.scratch) + warp * FD_TC_SCRATCH_WARP_BYTES;
  float* bias_s = f.bias;
  float acc[BLOCK_N / 2];
  long long staged_key = -1;                                 // which bias vectors shared memory holds
  for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
    const int m_tile = tile / num_n_tiles;
    const int n_tile = (tile % num_n_tiles + m_tile) % num_n_tiles;     // as in the producer
    const int b = m_tile / tiles_t, t0 = (m_tile % tiles_t) * BLOCK_M;
    const int n0 = n_tile * BLOCK_N;

    // stage the per-column bias vectors of this tile in shared memory; skipped while the CTA keeps seeing the same
    // columns / item -- with a single column tile that is once per launch
    if (EPI == FD_EPI_LINEAR && bias_key<EPI>(p, b, n0) != staged_key) {
      staged_key = bias_key<EPI>(p, b, n0);
      named_bar_sync<1, FD_TC_CONSUMER_THREADS>();
      stage_bias<BLOCK_N, EPI>(p, b, n0, bias_s, threadIdx.x, FD_TC_CONSUMER_THREADS);
      named_bar_sync<1, FD_TC_CONSUMER_THREADS>();
    }

    // ---- mainloop: 16 elements * 2 B along K inside the swizzle row per k16 step
    ring_mainloop(acc, ring, total_k_blocks, C::GROUP, lane, [&](int stage, int nb) {
      for (int g = 0; g < nb; ++g) {
        const uint32_t st = smem_u32(f.ring + stage * C::STAGE_BYTES + g * C::SUB_BYTES);
        const uint32_t wg_a = wg * 64 * C::SWIZZLE_BYTES;     // the warpgroup's 64 rows of a plane
        const uint64_t a_hi = make_smem_desc(st + wg_a, 16, C::SBO, C::SWIZZLE_MODE);
        const uint64_t a_lo = make_smem_desc(st + C::A_BYTES + wg_a, 16, C::SBO, C::SWIZZLE_MODE);
        const uint64_t w_hi = make_smem_desc(st + NPL * C::A_BYTES, 16, C::SBO, C::SWIZZLE_MODE);
        const uint64_t w_lo = make_smem_desc(st + NPL * C::A_BYTES + C::W_BYTES, 16, C::SBO, C::SWIZZLE_MODE);
        split_mma<MMA, NPL, BLOCK_K / 16, 32>(acc, a_hi, a_lo, w_hi, w_lo);
      }
    });

    tile_epilogue<BLOCK_N, EPI, PREC>(p, acc, b, n_tile, t0 + wg * 64 + wq * 16, bias_s, my_scratch, lane);
  }
}

// ------------------------------------------------------------------ ping-pong schedule (GATE, RES_SKIP)
// Work unit = (pair of adjacent 64-row tiles, column tile); cluster `pair` takes units pair, pair + num_pairs, ...
// and its two warpgroups take them in turn (warpgroup 0 the 1st, 3rd, ..., warpgroup 1 the 2nd, 4th, ...).  CTA
// `rank` of the pair computes row tile 2 m_pair + rank.  The producer fills the ring unit by unit in that order, and
// the warpgroups take their turns at the tensor cores (PingPong).
template <int BLOCK_N, int BLOCK_K, int EPI, int PREC, int NPL>
__global__ void __launch_bounds__(FD_TC_THREADS, 1)
fd_tapgemm_pp_kernel(const __grid_constant__ CUtensorMap tm_src0, const __grid_constant__ CUtensorMap tm_src1,
                     const __grid_constant__ CUtensorMap tm_w, const FdTapGemm p) {
  using C = Cfg<BLOCK_N, BLOCK_K, EPI, NPL>;
  static_assert(C::PP && C::GROUP == 1, "ping-pong schedule: GATE / RES_SKIP, one k-block per stage");
  using MMA = Wgmma<BLOCK_N, PREC>;
  extern __shared__ uint8_t smem_raw[];
  const TcFrame f = tc_frame(smem_raw, C::NUM_STAGES, C::STAGE_BYTES, C::BIAS_TOTAL);

  const int warp = threadIdx.x / 32;
  const int lane = threadIdx.x % 32;
  const int rank = (int)cluster_ctarank();
  const int pair = blockIdx.x / 2, num_pairs = gridDim.x / 2;

  const int tiles_t = (p.T + 63) / 64;
  const int num_m_tiles = p.B * tiles_t;
  const int num_n_tiles = p.n_total / BLOCK_N;
  const int num_units = (num_m_tiles + 1) / 2 * num_n_tiles;
  int total_k_blocks = 0;
  for (int sI = 0; sI < p.num_seg; ++sI) total_k_blocks += p.seg[sI].k_len / BLOCK_K;

  // a stage is refilled (in both CTAs: W arrives by multicast) once the consuming warpgroup of both CTAs is done
  tc_prologue<true>(f, C::NUM_STAGES, 2 * 4, &tm_src0, &tm_src1, &tm_w);

  if (warp >= FD_TC_PRODUCER_WARP) {
    // =========================================================== TMA producer
    producer_regs();
    if (warp == FD_TC_PRODUCER_WARP && lane == 0) {
      Ring ring{f.full, f.empty, C::NUM_STAGES};
      for (int u = pair; u < num_units; u += num_pairs) {
        const int m_pair = u / num_n_tiles;
        const int n_tile = (u % num_n_tiles + m_pair) % num_n_tiles;     // rotated as in the cooperative schedule
        // with an odd number of row tiles the second tile of the last pair lies past the end: that CTA still stages
        // its half of W for its peer, and loads the first tile's rows for a mainloop whose result it drops
        const int m_tile = min(2 * m_pair + rank, num_m_tiles - 1);
        const int b = m_tile / tiles_t, t0 = (m_tile % tiles_t) * 64;
        const int n0 = n_tile * BLOCK_N;
        SegCursor sc;
#pragma unroll 1                                     // (unrolled, it spills out of the producer's 40 registers)
        for (int kb = 0; kb < total_k_blocks; ++kb) {
          ring.wait_empty();
          uint8_t* st = f.ring + ring.stage * C::STAGE_BYTES;
          mbar_expect_tx(ring.full_bar(), C::TX_BYTES);   // own A box + both halves of W
          const FdSeg sg = p.seg[sc.s];
          tma_load_4d(st, sg.src == 0 ? &tm_src0 : &tm_src1, ring.full_bar(), sg.c_off + sc.k0, t0 + sg.shift, b, 0);
          // this CTA's half of the W box -- its plane (three products) or its BLOCK_N / 2 rows (one) -- into both CTAs
          tma_load_3d_multicast(st + NPL * C::A_BYTES + rank * (NPL * C::W_BYTES / 2), &tm_w, ring.full_bar(),
                                sc.koff + sc.k0 + p.w_kshift, n0 + (NPL == 1 ? rank * (BLOCK_N / 2) : 0),
                                NPL == 2 ? rank : 0, 0x3);
          sc.next(BLOCK_K, sg.k_len);
          ring.next();
        }
      }
    }
  } else {
    // =========================================================== consumers: one warpgroup per tile, in turn
    consumer_regs();
    const int wg = warp / 4;
    const int wq = warp % 4;                                 // 16-row slice of the tile
    const uint32_t my_scratch = smem_u32(f.scratch) + warp * FD_TC_SCRATCH_WARP_BYTES;
    float* my_bias = f.bias + wg * C::BIAS_FLOATS;
    float acc[BLOCK_N / 2];
    PingPong turn(f.full, f.empty, C::NUM_STAGES, total_k_blocks, wg);
    long long staged_key = -1;
    for (int u = pair + wg * num_pairs; u < num_units; u += 2 * num_pairs) {
      const int m_pair = u / num_n_tiles;
      const int n_tile = (u % num_n_tiles + m_pair) % num_n_tiles;     // as in the producer
      const int m_tile = 2 * m_pair + rank;
      const bool valid = m_tile < num_m_tiles;
      const int b = m_tile / tiles_t, t0 = (m_tile % tiles_t) * 64;
      const int n0 = n_tile * BLOCK_N;

      // this warpgroup's bias vectors, while the other warpgroup has the tensor cores
      if (valid && bias_key<EPI>(p, b, n0) != staged_key) {
        staged_key = bias_key<EPI>(p, b, n0);
        wg == 0 ? named_bar_sync<3, 128>() : named_bar_sync<4, 128>();
        stage_bias<BLOCK_N, EPI>(p, b, n0, my_bias, threadIdx.x % 128, 128);
        wg == 0 ? named_bar_sync<3, 128>() : named_bar_sync<4, 128>();
      }

      // `pass`: the other warpgroup has a next tile
      turn.mainloop(acc, u == pair, u + num_pairs < num_units, lane, [&](int stage) {
        const uint32_t st = smem_u32(f.ring + stage * C::STAGE_BYTES);
        const uint64_t a_hi = make_smem_desc(st, 16, C::SBO, C::SWIZZLE_MODE);
        const uint64_t a_lo = make_smem_desc(st + C::A_BYTES, 16, C::SBO, C::SWIZZLE_MODE);
        const uint64_t w_hi = make_smem_desc(st + NPL * C::A_BYTES, 16, C::SBO, C::SWIZZLE_MODE);
        const uint64_t w_lo = make_smem_desc(st + NPL * C::A_BYTES + C::W_BYTES, 16, C::SBO, C::SWIZZLE_MODE);
        split_mma<MMA, NPL, BLOCK_K / 16, 32>(acc, a_hi, a_lo, w_hi, w_lo);
      });

      if (valid) tile_epilogue<BLOCK_N, EPI, PREC>(p, acc, b, n_tile, t0 + wq * 16, my_bias, my_scratch, lane);
    }
  }
  __syncwarp();
  cluster_sync();   // neither CTA leaves while the other may still multicast into it or arrive on its barriers
}

// ------------------------------------------------------------------ transposed GATE (the sampler's GEMM1)
// GEMM1 with the conditioner projection hoisted out (three conv taps of the residual stream, K = 3C, the projection
// added in the epilogue) and three products, with the operands swapped: 64 packed W1 rows are the wgmma M side and
// BLOCK_T time steps the N side.  A stage holds one 32-channel block: the activation rows [t0 - d, t0 + BLOCK_T + d)
// once, and the three taps' W boxes.  Tap j reads the activation tile from row j d on -- a descriptor start address
// moved by j d rows (see make_smem_desc) -- so each activation row is staged once for all three taps instead of once
// per tap, and the W box per stage is 64 rows instead of 256.
// The W tensor map views the existing pack (tiles of gate_tile rows: gate_tile / 2 gates, then their filters) as
// (K, 8 rows, gate | filter, 8-row group, plane): a box lands as 16-row groups of 8 gate rows followed by the 8
// matching filter rows, so a thread's accumulator rows r and r + 8 are the gate and the filter of one channel and the
// gate needs no exchange between threads.  The bias tables and the conditioner projection keep W1's packed order.
// Schedule: that of fd_tapgemm_pp_kernel (ping-pong warpgroups, 2x1x1 clusters); a work unit is (time tile, pair of
// adjacent 64-row W tiles), CTA `rank` of the pair computes W tile 2 pair + rank, and each CTA multicasts one plane of
// the shared activation tile into both.
template <int BLOCK_T>
struct GateTCfg {
  static constexpr int BLOCK_K = 32;                      // 64-byte rows: a 64-wide ring would hold 2 stages
  static constexpr int ROW_BYTES = BLOCK_K * 2;
  static constexpr int ACT_ROWS = BLOCK_T + 16;           // the halo: dilations up to MAX_DIL
  static constexpr int MAX_DIL = (ACT_ROWS - BLOCK_T) / 2;
  static constexpr int ACT_PLANE = ACT_ROWS * ROW_BYTES;
  static constexpr int W_PLANE = 64 * ROW_BYTES;
  static constexpr int W_OFF = 2 * ACT_PLANE;             // then tap j's W box (hi plane, lo plane) at W_OFF + 2 j W_PLANE
  static constexpr int STAGE_BYTES = W_OFF + 3 * 2 * W_PLANE;
  static constexpr uint32_t SWIZZLE_MODE = swizzle_mode_for(ROW_BYTES);
  static constexpr uint32_t SBO = 8 * ROW_BYTES;
  static constexpr int NUM_STAGES = fd_tc_frame_stages(STAGE_BYTES, 0);
  static constexpr int SMEM_BYTES = fd_tc_frame_bytes(NUM_STAGES, STAGE_BYTES, 0);
  static_assert(ACT_ROWS <= 256, "one TMA box per plane");
  static_assert(ACT_PLANE % 512 == 0 && STAGE_BYTES % 1024 == 0, "planes start on 64 B swizzle atoms");
  static_assert(NUM_STAGES >= 3, "ring depth");
  static_assert(SMEM_BYTES <= FD_TC_SMEM_BUDGET, "shared memory");
};

// Epilogue of one warp: rows [16 wq, 16 wq + 16) of the tile are residual channels ch .. ch + 7 (gates, then
// filters); lane -> channel ch + lane / 4, times t0 + 8 c + 2 (lane % 4) + {0, 1}.  z goes through the warp's scratch,
// 32 time steps at a time, so that each lane stores the 8 channels of one time step (16 bytes per plane).
template <int BLOCK_T, int PREC>
__device__ __forceinline__ void gate_t_epilogue(const FdTapGemm& p, const float* acc, int b, int t0, int ch,
                                                uint32_t my_scratch, int lane) {
  const int half = p.gate_tile / 2;
  const int e = lane >> 2, q4 = lane & 3;
  const int n_g = fd_gate_col(p, ch) + e, n_f = n_g + half;   // packed columns of rows r, r + 8
  const size_t bo = (size_t)b * p.gbias_bstride;
  const float bias[2][1] = {{p.gbias_full[bo + n_g]}, {p.gbias_full[bo + n_f]}};
  const float lo[2][1] = {{p.gbias_lo[bo + n_g]}, {p.gbias_lo[bo + n_f]}};
  const float hi[2][1] = {{p.gbias_hi[bo + n_g]}, {p.gbias_hi[bo + n_f]}};
  const size_t row0 = (size_t)b * p.T;
  const size_t zplane = (size_t)p.B * p.T * p.C;
  constexpr int NG = BLOCK_T / 8;                          // 8-column groups of the fragment
  // The addend (read once per launch: it streams past L2, evict-first) of a 32-step chunk, (gate, filter) per step,
  // rows past T clamped.  The loads of chunk c + 1 are issued before chunk c is computed: issued next to their use,
  // each would wait out a DRAM round trip, and the epilogue would outlast the other warpgroup's mainloop.
  auto load_addend = [&](int c0, float (&a)[16]) {
#pragma unroll
    for (int i = 0; i < 16; ++i) a[i] = 0.f;
    if (p.addend == nullptr) return;
#pragma unroll
    for (int ci = 0; ci < 4; ++ci) {
      if (c0 + ci < NG) {
#pragma unroll
        for (int s = 0; s < 2; ++s) {
          const int t = min(t0 + 8 * (c0 + ci) + 2 * q4 + s, p.T - 1);
          const float* ad = p.addend + (row0 + t) * p.n_total;
          a[4 * ci + 2 * s] = __ldcs(ad + n_g);
          a[4 * ci + 2 * s + 1] = __ldcs(ad + n_f);
        }
      }
    }
  };
  float a_next[16];
  load_addend(0, a_next);
#pragma unroll
  for (int c0 = 0; c0 < NG; c0 += 4) {
    float a_cur[16];
#pragma unroll
    for (int i = 0; i < 16; ++i) a_cur[i] = a_next[i];
    if (c0 + 4 < NG) load_addend(c0 + 4, a_next);
#pragma unroll
    for (int ci = 0; ci < 4; ++ci) {
      if (c0 + ci < NG) {
#pragma unroll
        for (int s = 0; s < 2; ++s) {
          const int tl = 8 * ci + 2 * q4 + s;              // time step inside the 32-step chunk
          const int t = t0 + 8 * c0 + tl;
          float g[1] = {acc[4 * (c0 + ci) + s]}, f[1] = {acc[4 * (c0 + ci) + 2 + s]}, z[1];
          const float add[2][1] = {{a_cur[4 * ci + 2 * s]}, {a_cur[4 * ci + 2 * s + 1]}};
          fd_epi_gate<1>(p, t, g, f, z, bias, add, lo, hi);
          // scratch [32 steps][8 channels], the two 16-byte halves of a step swapped on every other group of 4 steps
          sts32(my_scratch + 4u * (tl * 8 + (((e >> 2) ^ ((tl >> 2) & 1)) << 2) + (e & 3)), z[0]);
        }
      }
    }
    __syncwarp();
    const int t = t0 + 8 * c0 + lane;
    if (lane < 8 * min(4, NG - c0) && t < p.T) {
      const uint32_t sw = (uint32_t)((lane >> 2) & 1);
      const float4 z0 = lds128(my_scratch + 4u * (lane * 8 + (sw << 2)));
      const float4 z1 = lds128(my_scratch + 4u * (lane * 8 + ((sw ^ 1u) << 2)));
      const float z[8] = {z0.x, z0.y, z0.z, z0.w, z1.x, z1.y, z1.z, z1.w};
      fd_store_planes<8>(p.out_planes, zplane, (row0 + t) * p.C + ch, z, PREC);
    }
    __syncwarp();
  }
}

template <int BLOCK_T, int PREC>
__global__ void __launch_bounds__(FD_TC_THREADS, 1)
fd_gate_t_kernel(const __grid_constant__ CUtensorMap tm_x, const __grid_constant__ CUtensorMap tm_w, const FdTapGemm p) {
  using C = GateTCfg<BLOCK_T>;
  using MMA = Wgmma<BLOCK_T, PREC>;
  extern __shared__ uint8_t smem_raw[];
  const TcFrame f = tc_frame(smem_raw, C::NUM_STAGES, C::STAGE_BYTES, 0);

  const int warp = threadIdx.x / 32;
  const int lane = threadIdx.x % 32;
  const int rank = (int)cluster_ctarank();
  const int pair = blockIdx.x / 2, num_pairs = gridDim.x / 2;

  const int d = p.dil;
  const int tiles_t = (p.T + BLOCK_T - 1) / BLOCK_T;
  const int num_wp = p.n_total / 128;                      // pairs of 64-row W tiles
  const int num_units = p.B * tiles_t * num_wp;
  const int k_blocks = p.C / C::BLOCK_K;

  tc_prologue<true>(f, C::NUM_STAGES, 2 * 4, &tm_x, &tm_w);

  if (warp >= FD_TC_PRODUCER_WARP) {
    // =========================================================== TMA producer
    producer_regs();
    if (warp == FD_TC_PRODUCER_WARP && lane == 0) {
      // both activation planes (one from each CTA of the pair) + this CTA's three W boxes
      const uint32_t tx = 2u * (uint32_t)(BLOCK_T + 2 * d) * C::ROW_BYTES + 3 * 2 * C::W_PLANE;
      const int half = p.gate_tile / 2;
      Ring ring{f.full, f.empty, C::NUM_STAGES};
      for (int u = pair; u < num_units; u += num_pairs) {
        const int tt = u / num_wp, wt = 2 * (u % num_wp) + rank;
        const int b = tt / tiles_t, t0 = (tt % tiles_t) * BLOCK_T;
        const int ch = wt * 32;                                         // first residual channel of the W tile
        const int g0 = ((ch / half) * p.gate_tile + ch % half) / 8;     // its first 8-row group of gate rows
#pragma unroll 1
        for (int kb = 0; kb < k_blocks; ++kb) {
          ring.wait_empty();
          uint8_t* st = f.ring + ring.stage * C::STAGE_BYTES;
          mbar_expect_tx(ring.full_bar(), tx);
          tma_load_4d_multicast(st + rank * C::ACT_PLANE, &tm_x, ring.full_bar(), kb * C::BLOCK_K, t0 - d, b, rank,
                                0x3);
#pragma unroll 1
          for (int j = 0; j < 3; ++j)
            tma_load_5d(st + C::W_OFF + j * 2 * C::W_PLANE, &tm_w, ring.full_bar(), j * p.C + kb * C::BLOCK_K, 0, 0,
                        g0, 0);
          ring.next();
        }
      }
    }
  } else {
    // =========================================================== consumers: one warpgroup per unit, in turn
    consumer_regs();
    const int wg = warp / 4;
    const int wq = warp % 4;
    const uint32_t my_scratch = smem_u32(f.scratch) + warp * FD_TC_SCRATCH_WARP_BYTES;
    float acc[BLOCK_T / 2];
    PingPong turn(f.full, f.empty, C::NUM_STAGES, k_blocks, wg);
    for (int u = pair + wg * num_pairs; u < num_units; u += 2 * num_pairs) {
      const int tt = u / num_wp, wt = 2 * (u % num_wp) + rank;
      const int b = tt / tiles_t, t0 = (tt % tiles_t) * BLOCK_T;

      turn.mainloop(acc, u == pair, u + num_pairs < num_units, lane, [&](int stage) {
        const uint32_t st = smem_u32(f.ring + stage * C::STAGE_BYTES);
#pragma unroll
        for (int j = 0; j < 3; ++j) {
          const uint32_t xa = st + (uint32_t)(j * d * C::ROW_BYTES);       // tap j: activation rows t0 - d + j d ...
          const uint64_t x_hi = make_smem_desc(xa, 16, C::SBO, C::SWIZZLE_MODE);
          const uint64_t x_lo = make_smem_desc(xa + C::ACT_PLANE, 16, C::SBO, C::SWIZZLE_MODE);
          const uint32_t wa = st + C::W_OFF + j * 2 * C::W_PLANE;
          const uint64_t w_hi = make_smem_desc(wa, 16, C::SBO, C::SWIZZLE_MODE);
          const uint64_t w_lo = make_smem_desc(wa + C::W_PLANE, 16, C::SBO, C::SWIZZLE_MODE);
          split_mma<MMA, 2, C::BLOCK_K / 16, 32, /*W_IS_A=*/true>(acc, x_hi, x_lo, w_hi, w_lo);
        }
      });

      gate_t_epilogue<BLOCK_T, PREC>(p, acc, b, t0, wt * 32 + wq * 8, my_scratch, lane);
    }
  }
  __syncwarp();
  cluster_sync();
}

// ------------------------------------------------------------------ host side
// The transposed GATE's time-tile width for p, or 0 where it does not apply (the other GEMMs, training's forward,
// which keeps the pre-activations, the conditioner in the K loop, one product, a halo past MAX_DIL): of the
// instantiated widths, the one that pads T least.
int gate_t_block(const FdTapGemm& p) {
  if (p.epi != FD_EPI_GATE || p.single || p.y_planes != nullptr || p.num_seg != 3 || p.w_kshift != 0) return 0;
  if (p.C % GateTCfg<200>::BLOCK_K != 0 || p.n_total != 2 * p.C || p.src_C[0] != p.C) return 0;
  if ((p.gate_tile != 256 && p.gate_tile != 128) || p.n_total % p.gate_tile != 0) return 0;
  for (int s = 0; s < 3; ++s)
    if (p.seg[s].src != 0 || p.seg[s].shift != (s - 1) * p.dil || p.seg[s].c_off != 0 || p.seg[s].k_len != p.C)
      return 0;
  int best = 0;
  long long best_pad = 0;
  for (const int bt : {200, 240}) {
    if (p.dil > (bt == 200 ? GateTCfg<200>::MAX_DIL : GateTCfg<240>::MAX_DIL)) continue;
    const long long pad = (long long)(p.T + bt - 1) / bt * bt;
    if (best == 0 || pad < best_pad || (pad == best_pad && bt > best)) { best = bt; best_pad = pad; }
  }
  return best;
}

template <int BLOCK_T, int PREC>
int launch_gate_t(const FdTapGemm& p, cudaStream_t stream) {
  using C = GateTCfg<BLOCK_T>;
  CUtensorMap tmx, tmw;
  // one plane of rows [t0 - d, t0 + BLOCK_T + d) per box
  int rc = planes_map(&tmx, p.src[0], p.src_C[0], p.T, p.B, p.src_rs[0], p.src_bs[0], p.src_ps[0], C::BLOCK_K,
                      BLOCK_T + 2 * p.dil, 1, "gate_t x");
  if (rc) return rc;
  // packed W1 [plane][n_total][k_total], row q gate_tile + h gate_tile / 2 + 8 g + e, as (K, e, h, 8-row group, plane)
  const int half = p.gate_tile / 2;
  const cuuint64_t K = (cuuint64_t)p.k_total;
  const cuuint64_t dims[5] = {K, 8, 2, (cuuint64_t)p.n_total / 8, 2};
  const cuuint64_t strides[4] = {K * 2, (cuuint64_t)half * K * 2, 8 * K * 2, (cuuint64_t)p.n_total * K * 2};
  const cuuint32_t box[5] = {(cuuint32_t)C::BLOCK_K, 8, 2, 4, 2};
  rc = encode_tiled(&tmw, p.w, 5, dims, strides, box, "gate_t w");
  if (rc) return rc;
  const int units = p.B * ((p.T + BLOCK_T - 1) / BLOCK_T) * (p.n_total / 128);
  return fd_tc_launch<fd_gate_t_kernel<BLOCK_T, PREC>>(C::SMEM_BYTES, 2 * units, stream, false, 2, tmx, tmw, p);
}

template <int BLOCK_N, int BLOCK_K, int EPI, int PREC, int NPL>
int launch_inst(const FdTapGemm& p, cudaStream_t stream) {
  using C = Cfg<BLOCK_N, BLOCK_K, EPI, NPL>;
  CUtensorMap tm0, tm1, tmw;   // the hi and lo planes of an operand arrive in one box
  int rc = planes_map(&tm0, p.src[0], p.src_C[0], p.T, p.B, p.src_rs[0], p.src_bs[0], p.src_ps[0], BLOCK_K, C::ROWS,
                      NPL, "tapgemm src0");
  if (rc) return rc;
  if (p.src[1] != nullptr) {
    rc = planes_map(&tm1, p.src[1], p.src_C[1], p.T, p.B, p.src_rs[1], p.src_bs[1], p.src_ps[1], BLOCK_K, C::ROWS, NPL,
                    "tapgemm src1");
    if (rc) return rc;
  } else {
    tm1 = tm0;
  }
  const int m_tiles = p.B * ((p.T + C::ROWS - 1) / C::ROWS), n_tiles = p.n_total / BLOCK_N;
  if constexpr (C::PP) {
    // a box is one CTA's half of the W tile: one plane (three products) or BLOCK_N / 2 rows (one product)
    rc = weights_map(&tmw, p.w, p.n_total, p.k_total, BLOCK_K, NPL == 2 ? BLOCK_N : BLOCK_N / 2, 1, "tapgemm w");
    if (rc) return rc;
    return fd_tc_launch<fd_tapgemm_pp_kernel<BLOCK_N, BLOCK_K, EPI, PREC, NPL>>(
        C::SMEM_BYTES, 2 * ((m_tiles + 1) / 2 * n_tiles), stream, false, 2, tm0, tm1, tmw, p);
  } else {
    rc = weights_map(&tmw, p.w, p.n_total, p.k_total, BLOCK_K, BLOCK_N, NPL, "tapgemm w");
    if (rc) return rc;
    return fd_tc_launch<fd_tapgemm_tc_kernel<BLOCK_N, BLOCK_K, EPI, PREC, NPL>>(C::SMEM_BYTES, m_tiles * n_tiles,
                                                                              stream, false, 1, tm0, tm1, tmw, p);
  }
}

template <int BLOCK_N, int BLOCK_K, int EPI>
int launch_cfg(const FdTapGemm& p, cudaStream_t stream) {
  if (p.single) {
    return p.prec == FD_F16 ? launch_inst<BLOCK_N, BLOCK_K, EPI, FD_F16, 1>(p, stream)
                            : launch_inst<BLOCK_N, BLOCK_K, EPI, FD_BF16, 1>(p, stream);
  }
  return p.prec == FD_F16 ? launch_inst<BLOCK_N, BLOCK_K, EPI, FD_F16, 2>(p, stream)
                          : launch_inst<BLOCK_N, BLOCK_K, EPI, FD_BF16, 2>(p, stream);
}

template <int BLOCK_N, int BLOCK_K>
int launch_epi(const FdTapGemm& p, cudaStream_t stream) {
  if (p.epi == FD_EPI_GATE) return launch_cfg<BLOCK_N, BLOCK_K, FD_EPI_GATE>(p, stream);
  if (p.epi == FD_EPI_MAG) return launch_cfg<BLOCK_N, BLOCK_K, FD_EPI_MAG>(p, stream);
  if (p.epi == FD_EPI_RES_SKIP) return launch_cfg<BLOCK_N, BLOCK_K, FD_EPI_RES_SKIP>(p, stream);
  if (p.epi == FD_EPI_GATE_BWD) return launch_cfg<BLOCK_N, BLOCK_K, FD_EPI_GATE_BWD>(p, stream);
  return launch_cfg<BLOCK_N, BLOCK_K, FD_EPI_LINEAR>(p, stream);
}

// choose (BLOCK_N, BLOCK_K) for a problem; bn = 0 if no tensor-core instantiation fits
void pick_cfg(const FdTapGemm& p, int* bn, int* bk) {
  *bn = 0; *bk = 0;
  bool all64 = true, all32 = true, all16 = true;
  for (int s = 0; s < p.num_seg; ++s) {
    if (p.seg[s].c_off % 16 != 0) return;
    all64 &= p.seg[s].k_len % 64 == 0;
    all32 &= p.seg[s].k_len % 32 == 0;
    all16 &= p.seg[s].k_len % 16 == 0;
  }
  const int k = all64 ? 64 : all32 ? 32 : all16 ? 16 : 0;
  if (k == 0) return;
  // GATE / RES_SKIP (the WaveNet GEMMs): where a ring of 64-wide k-blocks holds only 2 stages (three products at
  // BLOCK_N 256: 96 KB per stage), only one stage is ever refilled while the other is consumed.  BLOCK_K 32 halves the
  // stage and doubles the ring; the k16 order of the wgmma calls, and so every output bit, stays the same.  Measured
  // at the sampler shape (B=32, T=4000, C=512, H100 SXM at a 400 W power limit): GATE 3.76 -> 3.17 ms, RES_SKIP
  // 1.38 -> 1.28 ms per launch.  Single-product mode already has 4 stages of 48 KB at BLOCK_K 64, and went 1.34 ->
  // 1.42 ms (GATE) at BLOCK_K 32, so the switch is made only where the 64-wide ring is 2 deep.  (Those figures are for
  // the cooperative 128-row schedule; the ping-pong stage -- 64 rows of A, W, bias vectors per warpgroup, see Cfg --
  // has the same 2-deep 64-wide ring at BLOCK_N 256 with three products and 5 stages of 40 KB at BLOCK_K 32.)
  const int npl = p.single ? 1 : 2;
  auto wavenet_bk = [&](int n) {
    return fd_tc_frame_stages(npl * (64 + n) * 64 * 2, 2 * (p.epi == FD_EPI_GATE ? 3 : 1) * n) < 3 ? 32 : 64;
  };
  if (p.epi == FD_EPI_GATE || p.epi == FD_EPI_MAG) {
    const int n = p.gate_tile;
    if ((n != 256 && n != 128) || p.n_total % n != 0 || k != 64) return;
    *bn = n; *bk = p.epi == FD_EPI_GATE ? wavenet_bk(n) : 64;
    return;
  }
  int n = 256;
  // (GEMM2 with narrower column tiles was measured in round 2: 256 -> 0.406 ms, 128 -> 0.426 ms, 64 -> 0.667 ms per launch)
  while (n >= 16 && (p.n_total % n != 0 || (p.epi == FD_EPI_RES_SKIP && p.C % n != 0))) n >>= 1;
  if (n < 16) return;
  if (k == 64) {
    if (n < 64) return;
    // Wave quantisation (a persistent grid runs ceil(tiles / SMs) tile times; at the training shape, 157 row tiles, an N = 512
    // GEMM is 314 tiles of 256 columns = 3 waves for 2.12 waves of work) was tried against 128-column tiles for LINEAR /
    // GATE_BWD whenever the quantised time came out > 5 % better: same-box A/B of the training step 12.87 / 12.81 -> 12.81 /
    // 12.80 ms (one product), 19.84 / 20.07 -> 19.87 / 19.66 ms (three products) -- noise; left out.
    *bn = n; *bk = p.epi == FD_EPI_RES_SKIP ? wavenet_bk(n) : 64;
  } else if (k == 32) {
    if (p.epi != FD_EPI_LINEAR || n < 32) return;   // (GATE_BWD: BLOCK_K 64 only)
    *bn = n > 64 ? 64 : n; *bk = 32;
  } else {
    if (p.epi != FD_EPI_LINEAR) return;
    *bn = n > 32 ? 32 : n; *bk = 16;
  }
}

}  // namespace

int fd_tapgemm_tc_supported(const FdTapGemm& p) {
  int bn, bk;
  pick_cfg(p, &bn, &bk);
  if (bn == 0) return 0;
  for (int s = 0; s < 2; ++s)
    if (p.src[s] != nullptr && (p.src_rs[s] % 8 != 0 || p.src_bs[s] % 8 != 0 || p.src_ps[s] % 8 != 0)) return 0;
  if (p.k_total % 8 != 0) return 0;
  return 1;
}

int fd_tapgemm_tc_launch(const FdTapGemm& p, cudaStream_t stream) {
  int bn, bk;
  pick_cfg(p, &bn, &bk);
  // the epilogues index their outputs with 32-bit element offsets; GATE_BWD's are into the 2C-wide dy / y planes
  const long long width = p.epi == FD_EPI_GATE_BWD ? 2ll * p.n_total : p.n_total;
  FD_REQUIRE((long long)p.B * p.T * width < (1ll << 32),
             "tapgemm(tc): B*T*%lld = %lld exceeds the 32-bit element offsets of the epilogue", width,
             (long long)p.B * p.T * width);
  FD_REQUIRE(bn != 0 && fd_tapgemm_tc_supported(p),
             "tapgemm(tc): no tensor-core instantiation for n_total=%d k_total=%d epi=%d", p.n_total, p.k_total,
             p.epi);
  if (const int bt = gate_t_block(p)) {
    if (bt == 200) return p.prec == FD_F16 ? launch_gate_t<200, FD_F16>(p, stream) : launch_gate_t<200, FD_BF16>(p, stream);
    return p.prec == FD_F16 ? launch_gate_t<240, FD_F16>(p, stream) : launch_gate_t<240, FD_BF16>(p, stream);
  }
  if (bk == 64) {
    if (bn == 256) return launch_epi<256, 64>(p, stream);
    if (bn == 128) return launch_epi<128, 64>(p, stream);
    if (p.epi == FD_EPI_GATE_BWD) return launch_cfg<64, 64, FD_EPI_GATE_BWD>(p, stream);
    if (p.epi == FD_EPI_RES_SKIP) return launch_cfg<64, 64, FD_EPI_RES_SKIP>(p, stream);
    return launch_cfg<64, 64, FD_EPI_LINEAR>(p, stream);
  }
  if (p.epi == FD_EPI_GATE || p.epi == FD_EPI_RES_SKIP) {
    // pick_cfg takes BLOCK_K 32 for these only at BLOCK_N 256 with three products
    FD_REQUIRE(bk == 32 && bn == 256 && !p.single, "tapgemm(tc): no BLOCK_K=%d instantiation of epi=%d", bk, p.epi);
    if (p.epi == FD_EPI_GATE)
      return p.prec == FD_F16 ? launch_inst<256, 32, FD_EPI_GATE, FD_F16, 2>(p, stream)
                              : launch_inst<256, 32, FD_EPI_GATE, FD_BF16, 2>(p, stream);
    return p.prec == FD_F16 ? launch_inst<256, 32, FD_EPI_RES_SKIP, FD_F16, 2>(p, stream)
                            : launch_inst<256, 32, FD_EPI_RES_SKIP, FD_BF16, 2>(p, stream);
  }
  if (bk == 32) {
    FD_REQUIRE(p.epi == FD_EPI_LINEAR, "tapgemm(tc): BLOCK_K=32 only instantiated for the linear epilogue");
    if (bn == 64) return launch_cfg<64, 32, FD_EPI_LINEAR>(p, stream);
    return launch_cfg<32, 32, FD_EPI_LINEAR>(p, stream);
  }
  FD_REQUIRE(p.epi == FD_EPI_LINEAR, "tapgemm(tc): BLOCK_K=16 only instantiated for the linear epilogue");
  if (bn == 32) return launch_cfg<32, 16, FD_EPI_LINEAR>(p, stream);
  return launch_cfg<16, 16, FD_EPI_LINEAR>(p, stream);
}
