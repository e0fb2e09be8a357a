// Weight-gradient GEMM on wgmma straight from channels-last split planes (sm_90a), and the fd_wgrad_cl entry point,
// which also serves the SIMT twin (fd_tapgemm_simt.cu).
//
//   part[s][r][c] = acc_scale * sum_{b in split s} sum_t  ROW[b, t, r] * COL[b, t + shift(c), c]
//
// Time is the contraction axis, and in channels-last storage it is the SLOW axis of both operands.  Instead of
// transposing the activations, both operands are fed to the tensor core as MN-major shared-memory tiles: a TMA box
// of [64 time steps][64 channels] with the 128-byte swizzle is exactly one MN-major SW128 atom column (64 channels
// contiguous = one 128-byte row per time step, 8 rows per swizzle atom), so the wgmma instructions just set the
// transpose flags of both operands.  The conv-tap shift of a column segment is a TMA row coordinate (zero fill
// outside [0,T) = the conv zero padding), exactly as in the forward kernel.
//
// Work unit = (split s, 128-row tile, BLOCK_N-column tile); a unit accumulates over its items and all time blocks in
// registers and stores one fp32 partial; fd_reduce_batch sums the `splits` partials.  Warp roles and the pipeline are
// those of fd_tapgemm_tc.cu (a TMA producer warpgroup, two consumer warpgroups of 64 rows each, smem full/empty ring).
#include <cuda.h>
#include <cstring>
#include "fd_common.cuh"
#include "fd_host.h"
#include "fd_tc_ptx.cuh"

namespace {

constexpr int WG_BLOCK_M = 128;
constexpr int WG_BLOCK_K = 64;                 // time steps per pipeline stage
constexpr int WG_BOX_BYTES = 64 * 64 * 2;      // one plane of one [64 t][64 ch] box

template <int BLOCK_N, int NPL>
struct WgCfg {
  static constexpr int A_BOXES = WG_BLOCK_M / 64;
  static constexpr int W_BOXES = BLOCK_N / 64;
  static constexpr int A_BYTES = A_BOXES * NPL * WG_BOX_BYTES;
  static constexpr int W_BYTES = W_BOXES * NPL * WG_BOX_BYTES;
  static constexpr int STAGE_BYTES = A_BYTES + W_BYTES;
  static constexpr int NUM_STAGES = fd_tc_frame_stages(STAGE_BYTES, 0);
  static constexpr int SMEM_BYTES = fd_tc_frame_bytes(NUM_STAGES, STAGE_BYTES, 0);
  static_assert(NUM_STAGES >= 2, "pipeline needs at least two stages");
};

template <int BLOCK_N, int PREC, int NPL>
__global__ void __launch_bounds__(FD_TC_THREADS, 1)
fd_wgrad_tc_kernel(const __grid_constant__ CUtensorMap tm_row0, const __grid_constant__ CUtensorMap tm_row1,
                   const __grid_constant__ CUtensorMap tm_col0, const __grid_constant__ CUtensorMap tm_col1,
                   const FdWgradK p) {
  using C = WgCfg<BLOCK_N, NPL>;
  using MMA = Wgmma<BLOCK_N, PREC>;
  extern __shared__ uint8_t smem_raw[];
  const TcFrame f = tc_frame(smem_raw, C::NUM_STAGES, C::STAGE_BYTES, 0);
  Ring ring{f.full, f.empty, C::NUM_STAGES};

  const int warp = threadIdx.x / 32;
  const int lane = threadIdx.x % 32;
  const int tiles_per_split = p.m_tiles * p.n_tiles;
  const int num_units = p.splits * tiles_per_split;
  const int k_blocks = (p.T + WG_BLOCK_K - 1) / WG_BLOCK_K;

  tc_prologue<false>(f, C::NUM_STAGES, FD_TC_CONSUMER_THREADS / 32, &tm_row0, &tm_row1, &tm_col0, &tm_col1);

  if (warp >= FD_TC_PRODUCER_WARP) {
    // =========================================================== TMA producer
    producer_regs();
    if (warp == FD_TC_PRODUCER_WARP && lane == 0) {
      for (int unit = blockIdx.x; unit < num_units; unit += gridDim.x) {
        const int s = unit / tiles_per_split;
        const int tile = unit % tiles_per_split;
        const int r0 = (tile / p.n_tiles) * WG_BLOCK_M, c0 = (tile % p.n_tiles) * BLOCK_N;
        // resolve the 64-channel boxes of this tile once: (map, first channel, time shift)
        const CUtensorMap* a_map[C::A_BOXES]; int a_ch[C::A_BOXES];
        const CUtensorMap* w_map[C::W_BOXES]; int w_ch[C::W_BOXES], w_sh[C::W_BOXES];
#pragma unroll
        for (int i = 0; i < C::A_BOXES; ++i) {
          const int r = r0 + 64 * i;
          a_map[i] = &tm_row0; a_ch[i] = p.row_C[0];            // rows past R: a box entirely out of range reads zeros
          for (int g = 0; g < p.num_row_seg; ++g)
            if (r >= p.row_start[g] && r < p.row_start[g] + p.row_width[g]) {
              a_map[i] = p.row_src[g] == 0 ? &tm_row0 : &tm_row1;
              a_ch[i] = p.row_coff[g] + (r - p.row_start[g]);
            }
        }
#pragma unroll
        for (int i = 0; i < C::W_BOXES; ++i) {
          const int c = c0 + 64 * i;
          w_map[i] = &tm_col0; w_ch[i] = p.col_C[0]; w_sh[i] = 0;
          for (int g = 0; g < p.num_col_seg; ++g)
            if (c >= p.col_start[g] && c < p.col_start[g] + p.col_width[g]) {
              w_map[i] = p.col_src[g] == 0 ? &tm_col0 : &tm_col1;
              w_ch[i] = p.col_coff[g] + (c - p.col_start[g]);
              w_sh[i] = p.col_shift[g];
            }
        }
        const int b_end = min(p.B, (s + 1) * p.items_per_split);
        for (int b = s * p.items_per_split; b < b_end; ++b) {
          for (int kb = 0; kb < k_blocks; ++kb) {
            const int t0 = kb * WG_BLOCK_K;
            ring.wait_empty();
            uint8_t* st = f.ring + ring.stage * C::STAGE_BYTES;
            mbar_expect_tx(ring.full_bar(), C::STAGE_BYTES);
#pragma unroll
            for (int i = 0; i < C::A_BOXES; ++i)
              tma_load_4d(st + i * NPL * WG_BOX_BYTES, a_map[i], ring.full_bar(), a_ch[i], t0, b, 0);
#pragma unroll
            for (int i = 0; i < C::W_BOXES; ++i)
              tma_load_4d(st + C::A_BYTES + i * NPL * WG_BOX_BYTES, w_map[i], ring.full_bar(), w_ch[i], t0 + w_sh[i],
                          b, 0);
            ring.next();
          }
        }
      }
    }
    return;
  }

  // =========================================================== consumers: wgmma mainloop, fp32 partial tile
  consumer_regs();
  const int wg = warp / 4;                           // rows [64 wg, 64 wg + 64) of the tile = A box wg
  const int wq = warp % 4;
  const uint32_t my_scratch = smem_u32(f.scratch) + warp * FD_TC_SCRATCH_WARP_BYTES;
  const int j4 = (lane & 7) * 4, rsub = lane >> 3;
  // MN-major SW128 operands: LBO = distance between 64-channel atoms (the boxes), SBO = 8 time rows of 128 bytes
  constexpr uint32_t LBO = NPL * WG_BOX_BYTES, SBO = 1024;
  float acc[BLOCK_N / 2];
  for (int unit = blockIdx.x; unit < num_units; unit += gridDim.x) {
    const int s = unit / tiles_per_split;
    const int tile = unit % tiles_per_split;
    const int r0 = (tile / p.n_tiles) * WG_BLOCK_M, c0 = (tile % p.n_tiles) * BLOCK_N;
    const int n_items = min(p.B, (s + 1) * p.items_per_split) - s * p.items_per_split;
    ring_mainloop(acc, ring, n_items * k_blocks, 1, lane, [&](int stage, int) {
      const uint32_t st = smem_u32(f.ring + stage * C::STAGE_BYTES);
      const uint64_t a_hi = make_smem_desc(st + wg * NPL * WG_BOX_BYTES, LBO, SBO, 1);
      const uint64_t a_lo = make_smem_desc(st + wg * NPL * WG_BOX_BYTES + WG_BOX_BYTES, LBO, SBO, 1);
      const uint64_t w_hi = make_smem_desc(st + C::A_BYTES, LBO, SBO, 1);
      const uint64_t w_lo = make_smem_desc(st + C::A_BYTES + WG_BOX_BYTES, LBO, SBO, 1);
      // k16 steps of 16 time rows of 128 bytes
      split_mma<MMA, NPL, WG_BLOCK_K / 16, 16 * 128, false, 1, 1>(acc, a_hi, a_lo, w_hi, w_lo);
    });

    // ---- epilogue: 32-column chunks through the warp scratch; 8 lanes cover one 128-byte row segment
    float* const out = p.part + (size_t)s * p.R * p.Cc;
#pragma unroll
    for (int c = 0; c < BLOCK_N; c += 32) {
      frag_to_scratch<32>(my_scratch, acc, c, 0, lane);
      __syncwarp();
      float4 a[4];
#pragma unroll
      for (int pp = 0; pp < 4; ++pp) a[pp] = scratch_ld4(my_scratch, 4 * pp + rsub, lane & 7);
      __syncwarp();
      const int col = c0 + c + j4;
#pragma unroll
      for (int pp = 0; pp < 4; ++pp) {
        const int r = r0 + wg * 64 + wq * 16 + pp * 4 + rsub;
        if (r < p.R)
          *reinterpret_cast<float4*>(out + (size_t)r * p.Cc + col) =
              make_float4(a[pp].x * p.acc_scale, a[pp].y * p.acc_scale, a[pp].z * p.acc_scale, a[pp].w * p.acc_scale);
      }
    }
  }
}

// row and column maps: box = [NPL planes][64 t][64 ch], 128-byte swizzle; absent second sources alias the first
template <int BLOCK_N, int PREC, int NPL>
int launch_wg(const FdWgradK& p, const uint16_t* const* row_ptr, const uint16_t* const* col_ptr, cudaStream_t stream) {
  CUtensorMap tr[2], tc[2];
  for (int i = 0; i < 2; ++i) {
    const int ri = row_ptr[i] != nullptr ? i : 0, ci = col_ptr[i] != nullptr ? i : 0;
    const long long rows_T = (long long)p.T * p.row_C[ri], cols_T = (long long)p.T * p.col_C[ci];
    int rc = planes_map(&tr[i], row_ptr[ri], p.row_C[ri], p.T, p.B, p.row_C[ri], rows_T, p.B * rows_T, 64, WG_BLOCK_K,
                        NPL, "wgrad rows");
    if (rc) return rc;
    rc = planes_map(&tc[i], col_ptr[ci], p.col_C[ci], p.T, p.B, p.col_C[ci], cols_T, p.B * cols_T, 64, WG_BLOCK_K, NPL,
                    "wgrad columns");
    if (rc) return rc;
  }
  return fd_tc_launch<fd_wgrad_tc_kernel<BLOCK_N, PREC, NPL>>(WgCfg<BLOCK_N, NPL>::SMEM_BYTES,
                                                              p.splits * p.m_tiles * p.n_tiles, stream, false, 1, tr[0],
                                                              tr[1], tc[0], tc[1], p);
}

template <int BLOCK_N>
int launch_wg_prec(const FdWgradK& p, int prec, const uint16_t* const* row_ptr, const uint16_t* const* col_ptr,
                   cudaStream_t stream) {
  const bool single = (prec & FD_SINGLE) != 0;
  if ((prec & 0xF) == FD_F16)
    return single ? launch_wg<BLOCK_N, FD_F16, 1>(p, row_ptr, col_ptr, stream)
                  : launch_wg<BLOCK_N, FD_F16, 2>(p, row_ptr, col_ptr, stream);
  return single ? launch_wg<BLOCK_N, FD_BF16, 1>(p, row_ptr, col_ptr, stream)
                : launch_wg<BLOCK_N, FD_BF16, 2>(p, row_ptr, col_ptr, stream);
}

}  // namespace

// Segment validation and row / column resolution are shared by both back ends; only the width rule differs.
extern "C" int fd_wgrad_cl(const fd_wgrad_desc* d, void* stream) {
  FD_DEVICE_GUARD();
  FD_REQUIRE(d != nullptr, "fd_wgrad_cl: null descriptor");
  FD_REQUIRE(d->backend == FD_BACKEND_TC || d->backend == FD_BACKEND_SIMT, "fd_wgrad_cl: unknown backend %d",
             d->backend);
  FD_REQUIRE(d->B > 0 && d->T > 0 && d->splits > 0 && d->splits <= d->B, "fd_wgrad_cl: bad B=%d T=%d splits=%d", d->B,
             d->T, d->splits);
  FD_REQUIRE(d->num_row_seg >= 1 && d->num_row_seg <= 2 && d->num_col_seg >= 1 &&
                 d->num_col_seg <= FD_WGRAD_MAX_COL_SEG,
             "fd_wgrad_cl: segment counts out of range (%d rows, %d cols)", d->num_row_seg, d->num_col_seg);
  FD_REQUIRE(d->part != nullptr && d->row_src[0] != nullptr && d->col_src[0] != nullptr, "fd_wgrad_cl: null pointer");
  // tensor cores: whole 64-channel TMA boxes; SIMT twin: 8-channel vector loads
  const int unit = d->backend == FD_BACKEND_TC ? 64 : 8;
  FdWgradK p;
  memset(&p, 0, sizeof(p));
  p.B = d->B; p.T = d->T; p.splits = d->splits; p.items_per_split = (d->B + d->splits - 1) / d->splits;
  FD_REQUIRE((long long)(p.splits - 1) * p.items_per_split < d->B, "fd_wgrad_cl: splits=%d leaves an empty split", d->splits);
  for (int i = 0; i < 2; ++i) {
    p.row_C[i] = d->row_C[i]; p.col_C[i] = d->col_C[i];
    FD_REQUIRE((d->row_src[i] == nullptr || d->row_C[i] % 8 == 0) && (d->col_src[i] == nullptr || d->col_C[i] % 8 == 0),
               "fd_wgrad_cl: channel counts must be multiples of 8");
  }
  int R = 0, Cc = 0;
  for (int g = 0; g < d->num_row_seg; ++g) {
    const int src = d->row_seg_src[g];
    FD_REQUIRE((src == 0 || src == 1) && d->row_src[src] != nullptr, "fd_wgrad_cl: row segment %d has no source", g);
    FD_REQUIRE(d->row_seg_width[g] > 0 && d->row_seg_width[g] % unit == 0 && d->row_seg_coff[g] >= 0 &&
                   d->row_seg_coff[g] % 8 == 0 && d->row_seg_coff[g] + d->row_seg_width[g] <= d->row_C[src],
               "fd_wgrad_cl: row segment %d (coff %d width %d) must be a multiple of %d inside the source", g,
               d->row_seg_coff[g], d->row_seg_width[g], unit);
    p.row_src[g] = src; p.row_coff[g] = d->row_seg_coff[g]; p.row_start[g] = R; p.row_width[g] = d->row_seg_width[g];
    R += d->row_seg_width[g];
  }
  for (int g = 0; g < d->num_col_seg; ++g) {
    const int src = d->col_seg_src[g];
    FD_REQUIRE((src == 0 || src == 1) && d->col_src[src] != nullptr, "fd_wgrad_cl: column segment %d has no source", g);
    FD_REQUIRE(d->col_seg_width[g] > 0 && d->col_seg_width[g] % unit == 0 && d->col_seg_coff[g] >= 0 &&
                   d->col_seg_coff[g] % 8 == 0 && d->col_seg_coff[g] + d->col_seg_width[g] <= d->col_C[src],
               "fd_wgrad_cl: column segment %d (coff %d width %d) must be a multiple of %d inside the source", g,
               d->col_seg_coff[g], d->col_seg_width[g], unit);
    p.col_src[g] = src; p.col_shift[g] = d->col_seg_shift[g]; p.col_coff[g] = d->col_seg_coff[g];
    p.col_start[g] = Cc; p.col_width[g] = d->col_seg_width[g];
    Cc += d->col_seg_width[g];
  }
  p.R = R; p.Cc = Cc;
  p.num_row_seg = d->num_row_seg; p.num_col_seg = d->num_col_seg;
  p.part = d->part; p.acc_scale = d->acc_scale;
  cudaStream_t st = (cudaStream_t)stream;
  int rc;
  if (d->backend == FD_BACKEND_SIMT) {
    rc = fd_wgrad_simt_launch(p, d->row_src, d->col_src, d->prec, st);
  } else {
    p.m_tiles = (R + WG_BLOCK_M - 1) / WG_BLOCK_M;
    const int bn = Cc % 256 == 0 ? 256 : Cc % 128 == 0 ? 128 : 64;
    p.n_tiles = Cc / bn;
    if (bn == 256) rc = launch_wg_prec<256>(p, d->prec, d->row_src, d->col_src, st);
    else if (bn == 128) rc = launch_wg_prec<128>(p, d->prec, d->row_src, d->col_src, st);
    else rc = launch_wg_prec<64>(p, d->prec, d->row_src, d->col_src, st);
  }
  if (rc == 0) fd_count_launch(1);
  return rc;
}
