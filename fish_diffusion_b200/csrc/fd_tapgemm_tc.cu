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
// Pipeline: smem full/empty ring between the producer and the consumers.
#include <cuda.h>
#include "fd_common.cuh"
#include "fd_host.h"
#include "fd_tc_ptx.cuh"

namespace {

constexpr int BLOCK_M = 128;   // rows of a cooperative tile; a ping-pong tile is one warpgroup's 64

// ring stages of `stage_bytes` that fit next to the fixed parts of shared memory (bias vectors, barriers, scratch)
constexpr int ring_stages(int stage_bytes, int bias_floats) {
  return fd_tc_ring_stages(1024 /*align slack*/ + bias_floats * 4 + 2 * FD_TC_MAX_STAGES * 8 + FD_TC_SCRATCH_BYTES,
                           stage_bytes);
}

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
  static constexpr int NUM_STAGES = ring_stages(STAGE_BYTES, BIAS_TOTAL);
  static constexpr int SMEM_BYTES = 1024 /*align slack*/ + NUM_STAGES * STAGE_BYTES + BIAS_TOTAL * 4 +
                                    2 * NUM_STAGES * 8 + FD_TC_SCRATCH_BYTES;
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
  if (EPI == FD_EPI_GATE || EPI == FD_EPI_MAG) {
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
    const int halfg = p.gate_tile / 2;
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
          // the bias vectors are read with shared-space loads, and the zero-padding corrections of the first / last
          // `dilation` rows are skipped by a warp vote where no lane needs them
          float yg[8], yf[8], z[8];
          {
            // the addend (conditioner projection, packed columns n0 + cc and n0 + HALF + cc of this row) is issued
            // with the bias loads; it is read once per launch, so it streams past L2 (evict-first)
            float4 c0, c1, d0, d1;
            if (p.addend != nullptr) {
              const float* ad = p.addend + yrow + n0 + cc;
              c0 = __ldcs(reinterpret_cast<const float4*>(ad));
              c1 = __ldcs(reinterpret_cast<const float4*>(ad + 4));
              d0 = __ldcs(reinterpret_cast<const float4*>(ad + HALF));
              d1 = __ldcs(reinterpret_cast<const float4*>(ad + HALF + 4));
            }
            const float4 a0 = lds128(sb + 4u * cc), a1 = lds128(sb + 4u * cc + 16u);
            const float4 b0 = lds128(sb + 4u * (HALF + cc)), b1 = lds128(sb + 4u * (HALF + cc) + 16u);
            const float bg[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
            const float bf[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
            for (int i = 0; i < 8; ++i) {
              yg[i] = g[i] * p.acc_scale + bg[i];
              yf[i] = f[i] * p.acc_scale + bf[i];
            }
            if (p.addend != nullptr) {
              const float cg[8] = {c0.x, c0.y, c0.z, c0.w, c1.x, c1.y, c1.z, c1.w};
              const float cf[8] = {d0.x, d0.y, d0.z, d0.w, d1.x, d1.y, d1.z, d1.w};
#pragma unroll
              for (int i = 0; i < 8; ++i) { yg[i] += cg[i]; yf[i] += cf[i]; }
            }
          }
          if (edge_any) {
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              if (e == 0 ? e_lo : e_hi) {
                const uint32_t eb = sb + 4u * ((1 + e) * BLOCK_N + cc);
                const float4 a0 = lds128(eb), a1 = lds128(eb + 16u);
                const float4 b0 = lds128(eb + 4u * HALF), b1 = lds128(eb + 4u * HALF + 16u);
                const float eg[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
                const float ef[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
                for (int i = 0; i < 8; ++i) { yg[i] -= eg[i]; yf[i] -= ef[i]; }
              }
            }
          }
#pragma unroll
          for (int i = 0; i < 8; ++i) z[i] = fd_sigmoid(yg[i]) * fd_tanh(yf[i]);
          if (p.y_planes != nullptr) {   // training: keep the pre-activations (packed column order: gates | filters per tile)
            const int zc0 = n_tile * HALF + cc;
            const int ng = p.gate_tile == BLOCK_N ? n_tile * BLOCK_N + cc : (zc0 / halfg) * p.gate_tile + (zc0 % halfg);
            fd_store_planes<8>(p.y_planes, yplane, yrow + ng, yg, PREC);
            fd_store_planes<8>(p.y_planes, yplane, yrow + ng + halfg, yf, PREC);
          }
          fd_store_planes<8>(p.out_planes, zplane, zrow + cc, z, PREC);
        }
      }
    }
  } else if (BLOCK_N >= 64) {
    // ---- LINEAR / RES_SKIP / GATE_BWD, coalescing epilogue: 32-column chunks; lane -> rows rbase + 4 pp (pp < 4),
    //      columns 4 (lane % 8) .. + 3 of the chunk, so that 8 lanes cover one 128-byte row segment
    const uint32_t bias_addr = smem_u32(bias_s);
    const int j4 = (lane & 7) * 4, rsub = lane >> 3;
    const int rbase = rw0 + rsub;                      // time index of pass 0
    const int nrows = rbase < p.T ? min(4, (p.T - rbase + 3) / 4) : 0;   // rows rbase + 4 pp < T
    const uint32_t rowbase = (uint32_t)b * (uint32_t)p.T;
#pragma unroll
    for (int c = 0; c < BLOCK_N; c += 32) {
      const int col = c + j4;                          // first of this lane's 4 columns inside the tile
      const int n = n0 + col;                          // global packed column
      frag_to_scratch<32>(my_scratch, acc, c, 0, lane);
      __syncwarp();
      float4 a[4];
#pragma unroll
      for (int pp = 0; pp < 4; ++pp) a[pp] = scratch_ld4(my_scratch, 4 * pp + rsub, lane & 7);
      __syncwarp();
      if (EPI == FD_EPI_GATE_BWD) {
        // backward of z = sigmoid(g) tanh(f) fused into the dz GEMM (training): this lane's 4 channels n..n+3 of 4 rows
        const int half_g = p.gate_tile / 2;
        const uint32_t pg = (uint32_t)((n / half_g) * p.gate_tile + (n % half_g));     // packed gate column
        const uint32_t W2 = 2u * (uint32_t)p.C;
        const size_t yplane = (size_t)p.B * p.T * W2;
        const uint16_t* const y_lo = p.y_planes + yplane;
        uint16_t* const o_lo = p.out_planes + yplane;
        float sg4[4] = {0.f, 0.f, 0.f, 0.f}, sf4[4] = {0.f, 0.f, 0.f, 0.f};          // column sums over this lane's rows
        float e0g[4] = {0.f, 0.f, 0.f, 0.f}, e0f[4] = {0.f, 0.f, 0.f, 0.f}, e1g[4] = {0.f, 0.f, 0.f, 0.f}, e1f[4] = {0.f, 0.f, 0.f, 0.f};
        uint2 gh[4], gl[4], fh[4], fl[4];
        uint32_t eo4[4];
#pragma unroll
        for (int pp = 0; pp < 4; ++pp) {
          eo4[pp] = (rowbase + (uint32_t)min(rbase + pp * 4, p.T - 1)) * W2 + pg;
          gh[pp] = *reinterpret_cast<const uint2*>(p.y_planes + eo4[pp]);
          gl[pp] = *reinterpret_cast<const uint2*>(y_lo + eo4[pp]);
          fh[pp] = *reinterpret_cast<const uint2*>(p.y_planes + eo4[pp] + half_g);
          fl[pp] = *reinterpret_cast<const uint2*>(y_lo + eo4[pp] + half_g);
        }
#pragma unroll
        for (int pp = 0; pp < 4; ++pp) {
          if (pp >= nrows) break;
          float g[4], f[4];
          fd_combine2(gh[pp].x, gl[pp].x, PREC, g[0], g[1]);
          fd_combine2(gh[pp].y, gl[pp].y, PREC, g[2], g[3]);
          fd_combine2(fh[pp].x, fl[pp].x, PREC, f[0], f[1]);
          fd_combine2(fh[pp].y, fl[pp].y, PREC, f[2], f[3]);
          const float dzv[4] = {a[pp].x * p.acc_scale, a[pp].y * p.acc_scale, a[pp].z * p.acc_scale, a[pp].w * p.acc_scale};
          float dg[4], df[4];
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            const float sg = fd_sigmoid(g[i]), th = fd_tanh(f[i]);
            dg[i] = dzv[i] * th * sg * (1.f - sg);
            df[i] = dzv[i] * sg * (1.f - th * th);
          }
          uint32_t h0, l0, h1, l1;
          fd_split2(dg[0], dg[1], PREC, h0, l0);
          fd_split2(dg[2], dg[3], PREC, h1, l1);
          *reinterpret_cast<uint2*>(p.out_planes + eo4[pp]) = make_uint2(h0, h1);
          *reinterpret_cast<uint2*>(o_lo + eo4[pp]) = make_uint2(l0, l1);
          fd_split2(df[0], df[1], PREC, h0, l0);
          fd_split2(df[2], df[3], PREC, h1, l1);
          *reinterpret_cast<uint2*>(p.out_planes + eo4[pp] + half_g) = make_uint2(h0, h1);
          *reinterpret_cast<uint2*>(o_lo + eo4[pp] + half_g) = make_uint2(l0, l1);
          if (p.cs != nullptr) {
            const int tt = rbase + pp * 4;
            const bool in0 = tt < p.dil, in1 = tt + p.dil >= p.T;
#pragma unroll
            for (int i = 0; i < 4; ++i) {
              sg4[i] += dg[i]; sf4[i] += df[i];
              if (in0) { e0g[i] += dg[i]; e0f[i] += df[i]; }
              if (in1) { e1g[i] += dg[i]; e1f[i] += df[i]; }
            }
          }
        }
        if (p.cs != nullptr) {
          // rows of the 4 lanes that share these columns (lane bits 3,4), then one atomic per column and warp
          const bool edge0 = rw0 < p.dil, edge1 = rw0 + 16 + p.dil > p.T;     // warp-uniform
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            sg4[i] += __shfl_xor_sync(0xffffffffu, sg4[i], 8); sg4[i] += __shfl_xor_sync(0xffffffffu, sg4[i], 16);
            sf4[i] += __shfl_xor_sync(0xffffffffu, sf4[i], 8); sf4[i] += __shfl_xor_sync(0xffffffffu, sf4[i], 16);
            if (edge0) {
              e0g[i] += __shfl_xor_sync(0xffffffffu, e0g[i], 8); e0g[i] += __shfl_xor_sync(0xffffffffu, e0g[i], 16);
              e0f[i] += __shfl_xor_sync(0xffffffffu, e0f[i], 8); e0f[i] += __shfl_xor_sync(0xffffffffu, e0f[i], 16);
            }
            if (edge1) {
              e1g[i] += __shfl_xor_sync(0xffffffffu, e1g[i], 8); e1g[i] += __shfl_xor_sync(0xffffffffu, e1g[i], 16);
              e1f[i] += __shfl_xor_sync(0xffffffffu, e1f[i], 8); e1f[i] += __shfl_xor_sync(0xffffffffu, e1f[i], 16);
            }
          }
          if (rsub == 0) {
            float* const csb = p.cs + (size_t)b * W2 + pg;
#pragma unroll
            for (int i = 0; i < 4; ++i) {
              atomicAdd(csb + i, sg4[i] * p.cs_scale);
              atomicAdd(csb + half_g + i, sf4[i] * p.cs_scale);
            }
            if (p.cs_edge != nullptr && (edge0 || edge1)) {
              float* const ce0 = p.cs_edge + (size_t)b * W2 + pg;
              float* const ce1 = ce0 + (size_t)p.B * W2;
#pragma unroll
              for (int i = 0; i < 4; ++i) {
                if (edge0) { atomicAdd(ce0 + i, e0g[i] * p.cs_scale); atomicAdd(ce0 + half_g + i, e0f[i] * p.cs_scale); }
                if (edge1) { atomicAdd(ce1 + i, e1g[i] * p.cs_scale); atomicAdd(ce1 + half_g + i, e1f[i] * p.cs_scale); }
              }
            }
          }
        }
      } else if (EPI == FD_EPI_RES_SKIP) {
        // residual columns: x' = (x + y)/sqrt2 on the split planes; skip columns: fp32 accumulation.  32-bit element
        // offsets (checked on the host), rows past T clamped for the loads and skipped for the stores.
        const float4 bias4 = lds128(bias_addr + 4u * col);
        const bool is_res = n0 < p.C;
        const uint32_t cn = (uint32_t)(is_res ? n : n - p.C);
        const size_t plane = (size_t)p.B * p.T * p.C;
        uint32_t eo[4];
#pragma unroll
        for (int pp = 0; pp < 4; ++pp)
          eo[pp] = (rowbase + (uint32_t)min(rbase + pp * 4, p.T - 1)) * (uint32_t)p.C + cn;
        if (is_res) {
          if (!p.last_layer) {
            const uint16_t* const xlo = p.x_planes + plane;
            uint16_t* const xo = p.x_out_planes != nullptr ? p.x_out_planes : p.x_planes;
            uint16_t* const xo_lo = xo + plane;
            uint2 h2[4], l2[4];
#pragma unroll
            for (int pp = 0; pp < 4; ++pp) {
              h2[pp] = *reinterpret_cast<const uint2*>(p.x_planes + eo[pp]);
              l2[pp] = *reinterpret_cast<const uint2*>(xlo + eo[pp]);
            }
#pragma unroll
            for (int pp = 0; pp < 4; ++pp) {
              if (pp >= nrows) break;
              float x0, x1, x2, x3;
              fd_combine2(h2[pp].x, l2[pp].x, PREC, x0, x1);
              fd_combine2(h2[pp].y, l2[pp].y, PREC, x2, x3);
              x0 = (x0 + (a[pp].x * p.acc_scale + bias4.x)) * 0.70710678118654752440f;
              x1 = (x1 + (a[pp].y * p.acc_scale + bias4.y)) * 0.70710678118654752440f;
              x2 = (x2 + (a[pp].z * p.acc_scale + bias4.z)) * 0.70710678118654752440f;
              x3 = (x3 + (a[pp].w * p.acc_scale + bias4.w)) * 0.70710678118654752440f;
              uint32_t h0, l0, h1, l1;
              fd_split2(x0, x1, PREC, h0, l0);
              fd_split2(x2, x3, PREC, h1, l1);
              *reinterpret_cast<uint2*>(xo + eo[pp]) = make_uint2(h0, h1);
              *reinterpret_cast<uint2*>(xo_lo + eo[pp]) = make_uint2(l0, l1);
            }
          }
        } else {
          float4 sk[4];
          if (!p.first_layer) {
#pragma unroll
            for (int pp = 0; pp < 4; ++pp) sk[pp] = *reinterpret_cast<const float4*>(p.skip_f32 + eo[pp]);
          }
          uint16_t* const sk_lo = p.skip_planes + plane;
#pragma unroll
          for (int pp = 0; pp < 4; ++pp) {
            if (pp >= nrows) break;
            float y0 = a[pp].x * p.acc_scale + bias4.x, y1 = a[pp].y * p.acc_scale + bias4.y;
            float y2 = a[pp].z * p.acc_scale + bias4.z, y3 = a[pp].w * p.acc_scale + bias4.w;
            if (!p.first_layer) { y0 += sk[pp].x; y1 += sk[pp].y; y2 += sk[pp].z; y3 += sk[pp].w; }
            if (p.last_layer) {
              uint32_t h0, l0, h1, l1;
              fd_split2(y0 * p.skip_scale, y1 * p.skip_scale, PREC, h0, l0);
              fd_split2(y2 * p.skip_scale, y3 * p.skip_scale, PREC, h1, l1);
              *reinterpret_cast<uint2*>(p.skip_planes + eo[pp]) = make_uint2(h0, h1);
              *reinterpret_cast<uint2*>(sk_lo + eo[pp]) = make_uint2(l0, l1);
            } else {
              *reinterpret_cast<float4*>(p.skip_f32 + eo[pp]) = make_float4(y0, y1, y2, y3);
            }
          }
        }
      } else {
        // LINEAR (vocoder convs, WaveNet head / tail, data gradients): the operands of a chunk are folded kind by kind
        // into one pre-sum; element offsets are 32-bit (checked on the host) and rows past T are clamped for the loads
        // and skipped for the stores.
        const float4 bias4 = lds128(bias_addr + 4u * col);
        uint32_t eo[4];                                                     // element offset of this lane's 4 columns
#pragma unroll
        for (int pp = 0; pp < 4; ++pp)
          eo[pp] = (rowbase + (uint32_t)min(rbase + pp * 4, p.T - 1)) * (uint32_t)p.n_total + (uint32_t)n;
        float4 pre[4];
#pragma unroll
        for (int pp = 0; pp < 4; ++pp) pre[pp] = make_float4(0.f, 0.f, 0.f, 0.f);
        if (p.addend != nullptr) {
#pragma unroll
          for (int pp = 0; pp < 4; ++pp) {
            const float4 t4 = *reinterpret_cast<const float4*>(p.addend + eo[pp]);
            pre[pp].x += t4.x; pre[pp].y += t4.y; pre[pp].z += t4.z; pre[pp].w += t4.w;
          }
        }
        if (p.res_f32 != nullptr) {
#pragma unroll
          for (int pp = 0; pp < 4; ++pp) {
            const float4 t4 = *reinterpret_cast<const float4*>(p.res_f32 + eo[pp]);
            pre[pp].x += t4.x; pre[pp].y += t4.y; pre[pp].z += t4.z; pre[pp].w += t4.w;
          }
        }
        if (p.res_planes != nullptr) {
          const uint16_t* const lo_base = p.res_planes + (size_t)p.B * p.T * p.n_total;
#pragma unroll
          for (int pp = 0; pp < 4; ++pp) {
            const uint2 h2 = *reinterpret_cast<const uint2*>(p.res_planes + eo[pp]);
            const uint2 l2 = *reinterpret_cast<const uint2*>(lo_base + eo[pp]);
            float r0, r1, r2, r3;
            fd_combine2(h2.x, l2.x, PREC, r0, r1);
            fd_combine2(h2.y, l2.y, PREC, r2, r3);
            pre[pp].x += p.res_scale * r0; pre[pp].y += p.res_scale * r1;
            pre[pp].z += p.res_scale * r2; pre[pp].w += p.res_scale * r3;
          }
        }
        uint32_t mkbits = 0;
        if (p.row_mask != nullptr) {
#pragma unroll
          for (int pp = 0; pp < 4; ++pp)
            if (p.row_mask[rowbase + (uint32_t)min(rbase + pp * 4, p.T - 1)] != 0) mkbits |= 1u << pp;
        }
#pragma unroll
        for (int pp = 0; pp < 4; ++pp) {
          a[pp].x = (a[pp].x * p.acc_scale + bias4.x + pre[pp].x) * p.post_scale;
          a[pp].y = (a[pp].y * p.acc_scale + bias4.y + pre[pp].y) * p.post_scale;
          a[pp].z = (a[pp].z * p.acc_scale + bias4.z + pre[pp].z) * p.post_scale;
          a[pp].w = (a[pp].w * p.acc_scale + bias4.w + pre[pp].w) * p.post_scale;
        }
        if (p.out_f32 != nullptr && p.out_accum) {       // accumulate launches: one more batch of loads
#pragma unroll
          for (int pp = 0; pp < 4; ++pp) {
            const float4 o4 = *reinterpret_cast<const float4*>(p.out_f32 + eo[pp]);
            a[pp].x += o4.x; a[pp].y += o4.y; a[pp].z += o4.z; a[pp].w += o4.w;
          }
        }
        const float slope = p.act == FD_ACT_NONE ? 1.f : p.act == FD_ACT_RELU ? 0.f : p.act_slope;
        uint16_t* const out_lo = p.out_planes + (size_t)p.B * p.T * p.n_total;
#pragma unroll
        for (int pp = 0; pp < 4; ++pp) {
          if (pp >= nrows) break;
          if ((mkbits >> pp) & 1u) a[pp] = make_float4(0.f, 0.f, 0.f, 0.f);      // masked row: zeros everywhere
          if (p.out_f32 != nullptr) *reinterpret_cast<float4*>(p.out_f32 + eo[pp]) = a[pp];
          if (p.out_planes != nullptr) {
            uint32_t h0, l0, h1, l1;
            fd_split2(fd_act(a[pp].x * p.planes_scale, slope), fd_act(a[pp].y * p.planes_scale, slope), PREC, h0, l0);
            fd_split2(fd_act(a[pp].z * p.planes_scale, slope), fd_act(a[pp].w * p.planes_scale, slope), PREC, h1, l1);
            *reinterpret_cast<uint2*>(p.out_planes + eo[pp]) = make_uint2(h0, h1);
            *reinterpret_cast<uint2*>(out_lo + eo[pp]) = make_uint2(l0, l1);
          }
        }
      }
    }
  } else {
    // ---- LINEAR / RES_SKIP with narrow tiles (BLOCK_N <= 32): row-owner epilogue; lane -> row lane/2,
    //      BLOCK_N/2 columns (lane % 2)
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
    if (t < p.T) {
#pragma unroll
      for (int h = 0; h < PER / 8; ++h) {
        float v8[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) v8[i] = v[h * 8 + i];
        const int cc = sub * PER + h * 8;
        if (EPI == FD_EPI_LINEAR) fd_epi_linear<8, PREC>(p, b, t, n0 + cc, v8, bias_s, n0);
        else fd_epi_res_skip<8, PREC>(p, b, t, n0 + cc, v8, bias_s + cc);
      }
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
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint8_t* stage_base = smem;
  float* bias_s = reinterpret_cast<float*>(smem + C::NUM_STAGES * C::STAGE_BYTES);
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(bias_s + C::BIAS_TOTAL);
  uint64_t* empty_bar = full_bar + C::NUM_STAGES;
  float* scratch_s = reinterpret_cast<float*>(empty_bar + C::NUM_STAGES);   // 16-byte aligned (all preceding sizes are)

  const int warp = threadIdx.x / 32;
  const int lane = threadIdx.x % 32;

  const int tiles_t = (p.T + BLOCK_M - 1) / BLOCK_M;
  const int num_m_tiles = p.B * tiles_t;
  const int num_n_tiles = p.n_total / BLOCK_N;
  const int num_tiles = num_m_tiles * num_n_tiles;
  int total_k_blocks = 0;
  for (int sI = 0; sI < p.num_seg; ++sI) total_k_blocks += p.seg[sI].k_len / BLOCK_K;

  if (threadIdx.x == 0) {
    for (int i = 0; i < C::NUM_STAGES; ++i) { mbar_init(&full_bar[i], 1); mbar_init(&empty_bar[i], FD_TC_CONSUMER_THREADS / 32); }
    fence_barrier_init();
  }
  if (warp == FD_TC_PRODUCER_WARP && lane == 0) {
    prefetch_tmap(&tm_src0);
    prefetch_tmap(&tm_src1);
    prefetch_tmap(&tm_w);
  }
  __syncthreads();

  if (warp >= FD_TC_PRODUCER_WARP) {
    // =========================================================== TMA producer
    producer_regs();
    if (warp == FD_TC_PRODUCER_WARP && lane == 0) {
      int stage = 0; uint32_t phase = 0;
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        const int m_tile = tile / num_n_tiles;
        // rotate the column tile with the row tile: with a grid that is a multiple of num_n_tiles every CTA would
        // otherwise see the same n-tile forever, and epilogue costs differ per n-tile (residual vs skip columns)
        const int n_tile = (tile % num_n_tiles + m_tile) % num_n_tiles;
        const int b = m_tile / tiles_t, t0 = (m_tile % tiles_t) * BLOCK_M;
        const int n0 = n_tile * BLOCK_N;
        int s = 0, k0 = 0, koff = 0;                 // flattened (segment, k offset) iterator
        for (int kb = 0; kb < total_k_blocks; kb += C::GROUP) {
          const int nb = min(C::GROUP, total_k_blocks - kb);
          mbar_wait(&empty_bar[stage], phase ^ 1);
          uint8_t* st = stage_base + stage * C::STAGE_BYTES;
          mbar_expect_tx(&full_bar[stage], nb * C::TX_BYTES);
          for (int g = 0; g < nb; ++g) {
            const FdSeg sg = p.seg[s];
            const CUtensorMap* tm = sg.src == 0 ? &tm_src0 : &tm_src1;
            uint8_t* sub = st + g * C::SUB_BYTES;
            tma_load_4d(sub, tm, &full_bar[stage], sg.c_off + k0, t0 + sg.shift, b, 0);          // hi + lo planes
            const int kw = koff + k0 + p.w_kshift;
            tma_load_3d(sub + NPL * C::A_BYTES, &tm_w, &full_bar[stage], kw, n0, 0);               // hi + lo planes
            k0 += BLOCK_K;
            if (k0 >= sg.k_len) { koff += sg.k_len; k0 = 0; ++s; }
          }
          if (++stage == C::NUM_STAGES) { stage = 0; phase ^= 1; }
        }
      }
    }
    return;
  }

  // =========================================================== consumers: wgmma mainloop + epilogue
  consumer_regs();
  const int wg = warp / 4;                                   // rows [64 wg, 64 wg + 64) of the tile
  const int wq = warp % 4;                                   // 16-row slice of the warpgroup's 64 rows
  const uint32_t my_scratch = smem_u32(scratch_s) + warp * FD_TC_SCRATCH_WARP_BYTES;
  float acc[BLOCK_N / 2];
  int stage = 0; uint32_t phase = 0;
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
      asm volatile("bar.sync 1, %0;" ::"r"(FD_TC_CONSUMER_THREADS) : "memory");
      stage_bias<BLOCK_N, EPI>(p, b, n0, bias_s, threadIdx.x, FD_TC_CONSUMER_THREADS);
      asm volatile("bar.sync 1, %0;" ::"r"(FD_TC_CONSUMER_THREADS) : "memory");
    }

    // ---- mainloop: one wgmma group per ring stage, one group kept in flight; a stage is released once the group
    //      that read it has completed
#pragma unroll
    for (int i = 0; i < BLOCK_N / 2; ++i) acc[i] = 0.f;
    int prev_stage = -1;
    for (int kb = 0; kb < total_k_blocks; kb += C::GROUP) {
      const int nb = min(C::GROUP, total_k_blocks - kb);
      mbar_wait(&full_bar[stage], phase);
      wg_fence_operand(acc);
      wg_fence();
      for (int g = 0; g < nb; ++g) {
        const uint32_t st = smem_u32(stage_base + stage * C::STAGE_BYTES + g * C::SUB_BYTES);
        const uint32_t wg_a = wg * 64 * C::SWIZZLE_BYTES;     // the warpgroup's 64 rows of a plane
        const uint64_t a_hi = make_smem_desc(st + wg_a, 16, C::SBO, C::SWIZZLE_MODE);
        const uint64_t a_lo = make_smem_desc(st + C::A_BYTES + wg_a, 16, C::SBO, C::SWIZZLE_MODE);
        const uint64_t w_hi = make_smem_desc(st + NPL * C::A_BYTES, 16, C::SBO, C::SWIZZLE_MODE);
        const uint64_t w_lo = make_smem_desc(st + NPL * C::A_BYTES + C::W_BYTES, 16, C::SBO, C::SWIZZLE_MODE);
#pragma unroll
        for (int k = 0; k < BLOCK_K / 16; ++k) {
          const uint64_t adv = (uint64_t)((k * 32) >> 4);   // 16 elements * 2 B along K inside the swizzle row
          if (NPL == 2) {
            // small terms first, the dominant hi*hi product last
            MMA::template ss<0, 0>(acc, a_lo + adv, w_hi + adv, 1u);
            MMA::template ss<0, 0>(acc, a_hi + adv, w_lo + adv, 1u);
            MMA::template ss<0, 0>(acc, a_hi + adv, w_hi + adv, 1u);
          } else {
            MMA::template ss<0, 0>(acc, a_hi + adv, w_hi + adv, 1u);
          }
        }
      }
      wg_commit();
      wg_wait<1>();
      wg_fence_operand(acc);
      if (prev_stage >= 0 && lane == 0) mbar_arrive(&empty_bar[prev_stage]);
      prev_stage = stage;
      if (++stage == C::NUM_STAGES) { stage = 0; phase ^= 1; }
    }
    wg_wait<0>();
    wg_fence_operand(acc);
    if (prev_stage >= 0 && lane == 0) mbar_arrive(&empty_bar[prev_stage]);

    tile_epilogue<BLOCK_N, EPI, PREC>(p, acc, b, n_tile, t0 + wg * 64 + wq * 16, bias_s, my_scratch, lane);
  }
}

// ------------------------------------------------------------------ ping-pong schedule (GATE, RES_SKIP)
// Work unit = (pair of adjacent 64-row tiles, column tile); cluster `pair` takes units pair, pair + num_pairs, ...
// and its two warpgroups take them in turn (warpgroup 0 the 1st, 3rd, ..., warpgroup 1 the 2nd, 4th, ...).  CTA
// `rank` of the pair computes row tile 2 m_pair + rank.  The producer fills the ring unit by unit in that order, so the
// stages of a warpgroup's unit are the total_k_blocks ring positions after the previous unit's.  The mainloops run in
// turn: a warpgroup waits for its turn (named barrier 1 + wg), and passes it (named barrier 2 - wg) once it has
// issued the last wgmma group of its tile; its epilogue then overlaps the other warpgroup's mainloop.  The turn also
// keeps a warpgroup from waiting on a full barrier more than one phase ahead of the ring.
template <int BLOCK_N, int BLOCK_K, int EPI, int PREC, int NPL>
__global__ void __launch_bounds__(FD_TC_THREADS, 1)
fd_tapgemm_pp_kernel(const __grid_constant__ CUtensorMap tm_src0, const __grid_constant__ CUtensorMap tm_src1,
                     const __grid_constant__ CUtensorMap tm_w, const FdTapGemm p) {
  using C = Cfg<BLOCK_N, BLOCK_K, EPI, NPL>;
  static_assert(C::PP && C::GROUP == 1, "ping-pong schedule: GATE / RES_SKIP, one k-block per stage");
  using MMA = Wgmma<BLOCK_N, PREC>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint8_t* stage_base = smem;
  float* bias_s = reinterpret_cast<float*>(smem + C::NUM_STAGES * C::STAGE_BYTES);
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(bias_s + C::BIAS_TOTAL);
  uint64_t* empty_bar = full_bar + C::NUM_STAGES;
  float* scratch_s = reinterpret_cast<float*>(empty_bar + C::NUM_STAGES);   // 16-byte aligned (all preceding sizes are)

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

  if (threadIdx.x == 0) {
    // a stage is refilled (in both CTAs: W arrives by multicast) once the consuming warpgroup of both CTAs is done
    for (int i = 0; i < C::NUM_STAGES; ++i) { mbar_init(&full_bar[i], 1); mbar_init(&empty_bar[i], 2 * 4); }
    fence_barrier_init();
  }
  if (warp == FD_TC_PRODUCER_WARP && lane == 0) {
    prefetch_tmap(&tm_src0);
    prefetch_tmap(&tm_src1);
    prefetch_tmap(&tm_w);
  }
  cluster_sync();   // both CTAs' barriers are initialised before either multicasts or arrives into the other

  if (warp >= FD_TC_PRODUCER_WARP) {
    // =========================================================== TMA producer
    producer_regs();
    if (warp == FD_TC_PRODUCER_WARP && lane == 0) {
      int stage = 0; uint32_t phase = 0;
      for (int u = pair; u < num_units; u += num_pairs) {
        const int m_pair = u / num_n_tiles;
        const int n_tile = (u % num_n_tiles + m_pair) % num_n_tiles;     // rotated as in the cooperative schedule
        // with an odd number of row tiles the second tile of the last pair lies past the end: that CTA still stages
        // its half of W for its peer, and loads the first tile's rows for a mainloop whose result it drops
        const int m_tile = min(2 * m_pair + rank, num_m_tiles - 1);
        const int b = m_tile / tiles_t, t0 = (m_tile % tiles_t) * 64;
        const int n0 = n_tile * BLOCK_N;
        int s = 0, k0 = 0, koff = 0;                 // flattened (segment, k offset) iterator
#pragma unroll 1                                     // (unrolled, it spills out of the producer's 40 registers)
        for (int kb = 0; kb < total_k_blocks; ++kb) {
          mbar_wait(&empty_bar[stage], phase ^ 1);
          uint8_t* st = stage_base + stage * C::STAGE_BYTES;
          mbar_expect_tx(&full_bar[stage], C::TX_BYTES);   // own A box + both halves of W
          const FdSeg sg = p.seg[s];
          tma_load_4d(st, sg.src == 0 ? &tm_src0 : &tm_src1, &full_bar[stage], sg.c_off + k0, t0 + sg.shift, b, 0);
          // this CTA's half of the W box -- its plane (three products) or its BLOCK_N / 2 rows (one) -- into both CTAs
          tma_load_3d_multicast(st + NPL * C::A_BYTES + rank * (NPL * C::W_BYTES / 2), &tm_w, &full_bar[stage],
                                koff + k0 + p.w_kshift, n0 + (NPL == 1 ? rank * (BLOCK_N / 2) : 0),
                                NPL == 2 ? rank : 0, 0x3);
          k0 += BLOCK_K;
          if (k0 >= sg.k_len) { koff += sg.k_len; k0 = 0; ++s; }
          if (++stage == C::NUM_STAGES) { stage = 0; phase ^= 1; }
        }
      }
    }
  } else {
    // =========================================================== consumers: one warpgroup per tile, in turn
    consumer_regs();
    const int wg = warp / 4;
    const int wq = warp % 4;                                 // 16-row slice of the tile
    const uint32_t my_scratch = smem_u32(scratch_s) + warp * FD_TC_SCRATCH_WARP_BYTES;
    float* my_bias = bias_s + wg * C::BIAS_FLOATS;
    float acc[BLOCK_N / 2];
    int stage = 0; uint32_t phase = 0;
    auto advance = [&](int n) {                              // n ring positions on
      stage += n;
      phase ^= (uint32_t)(stage / C::NUM_STAGES) & 1u;
      stage %= C::NUM_STAGES;
    };
    auto release = [&](int st) {                             // the stage, in both CTAs
      if (lane == 0) { mbar_arrive_cluster(&empty_bar[st], 0); mbar_arrive_cluster(&empty_bar[st], 1); }
    };
    if (wg == 1) advance(total_k_blocks);
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

      if (u != pair) wg == 0 ? named_bar_sync<1, 256>() : named_bar_sync<2, 256>();   // wait for the turn
      const bool pass = u + num_pairs < num_units;            // the other warpgroup has a next tile
#pragma unroll
      for (int i = 0; i < BLOCK_N / 2; ++i) acc[i] = 0.f;
      int prev_stage = -1;
      for (int kb = 0; kb < total_k_blocks; ++kb) {
        mbar_wait(&full_bar[stage], phase);
        wg_fence_operand(acc);
        wg_fence();
        const uint32_t st = smem_u32(stage_base + stage * C::STAGE_BYTES);
        const uint64_t a_hi = make_smem_desc(st, 16, C::SBO, C::SWIZZLE_MODE);
        const uint64_t a_lo = make_smem_desc(st + C::A_BYTES, 16, C::SBO, C::SWIZZLE_MODE);
        const uint64_t w_hi = make_smem_desc(st + NPL * C::A_BYTES, 16, C::SBO, C::SWIZZLE_MODE);
        const uint64_t w_lo = make_smem_desc(st + NPL * C::A_BYTES + C::W_BYTES, 16, C::SBO, C::SWIZZLE_MODE);
#pragma unroll
        for (int k = 0; k < BLOCK_K / 16; ++k) {
          const uint64_t adv = (uint64_t)((k * 32) >> 4);   // 16 elements * 2 B along K inside the swizzle row
          if (NPL == 2) {
            // small terms first, the dominant hi*hi product last
            MMA::template ss<0, 0>(acc, a_lo + adv, w_hi + adv, 1u);
            MMA::template ss<0, 0>(acc, a_hi + adv, w_lo + adv, 1u);
            MMA::template ss<0, 0>(acc, a_hi + adv, w_hi + adv, 1u);
          } else {
            MMA::template ss<0, 0>(acc, a_hi + adv, w_hi + adv, 1u);
          }
        }
        wg_commit();
        if (kb == total_k_blocks - 1 && pass)                                   // pass the turn
          wg == 0 ? named_bar_arrive<2, 256>() : named_bar_arrive<1, 256>();
        wg_wait<1>();
        wg_fence_operand(acc);
        if (prev_stage >= 0) release(prev_stage);
        prev_stage = stage;
        advance(1);
      }
      wg_wait<0>();
      wg_fence_operand(acc);
      if (prev_stage >= 0) release(prev_stage);
      advance(total_k_blocks);                                // past the other warpgroup's tile

      if (valid) tile_epilogue<BLOCK_N, EPI, PREC>(p, acc, b, n_tile, t0 + wq * 16, my_bias, my_scratch, lane);
    }
  }
  __syncwarp();
  cluster_sync();   // neither CTA leaves while the other may still multicast into it or arrive on its barriers
}

// ------------------------------------------------------------------ host side
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
    return ring_stages(npl * (64 + n) * 64 * 2, 2 * (p.epi == FD_EPI_GATE ? 3 : 1) * n) < 3 ? 32 : 64;
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
