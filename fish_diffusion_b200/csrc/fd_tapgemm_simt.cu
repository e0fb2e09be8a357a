// SIMT fp32 twins of the tap-GEMM (same operands, same packed weights, same epilogues as the
// wgmma kernel in fd_tapgemm_tc.cu) and of the weight-gradient GEMM (fd_wgrad_tc.cu).  They exist
// (a) as the device-side check of the tensor-core kernels, (b) for shapes the tensor-core
// instantiations do not cover.  They are plain CUDA-core FFMA over (hi+lo) recombined operands,
// i.e. fp32 arithmetic on 22-bit (f16 planes) inputs.
#include "fd_common.cuh"

namespace {

constexpr int BM = 128;   // rows (time positions) per CTA
constexpr int BK = 16;    // k per smem stage
constexpr int APITCH = BM + 4;

template <int RUN, int EPI>
__global__ void __launch_bounds__(256) fd_tapgemm_simt_kernel(const FdTapGemm p) {
  constexpr int BN = 2 * RUN;
  constexpr int TXC = RUN / 4;       // threads along n
  constexpr int TYC = 256 / TXC;     // threads along m
  constexpr int RM = BM / TYC;       // rows per thread
  constexpr int BPITCH = BN + 4;

  __shared__ float As[BK][APITCH];
  __shared__ float Bs[BK][BPITCH];

  const int tid = threadIdx.x;
  const int tx = tid % TXC, ty = tid / TXC;
  const int tiles_t = (p.T + BM - 1) / BM;
  const int m_tile = blockIdx.x;
  const int b = m_tile / tiles_t;
  const int t0 = (m_tile % tiles_t) * BM;
  const int j = blockIdx.y;

  int run0, run1;
  if (EPI == FD_EPI_GATE || EPI == FD_EPI_MAG) {
    const int half = p.gate_tile / 2;
    const int zc0 = j * RUN;
    run0 = (zc0 / half) * p.gate_tile + (zc0 % half);
    run1 = run0 + half;
  } else {
    run0 = j * BN;
    run1 = run0 + RUN;
  }

  float acc[RM][8];
#pragma unroll
  for (int r = 0; r < RM; ++r)
#pragma unroll
    for (int c = 0; c < 8; ++c) acc[r][c] = 0.f;

  const size_t w_plane = (size_t)p.n_total * p.k_total;
  int koff = 0;
  for (int s = 0; s < p.num_seg; ++s) {
    const FdSeg sg = p.seg[s];
    const uint16_t* src = p.src[sg.src];
    const size_t a_plane = (size_t)p.src_ps[sg.src];
    const size_t a_rs = (size_t)p.src_rs[sg.src], a_bs = (size_t)p.src_bs[sg.src];
    for (int k0 = 0; k0 < sg.k_len; k0 += BK) {
      // ---- load A tile: 128 rows x 16 k
      {
        const int row = tid % BM, kh = tid / BM;   // kh in {0,1}
        const int t = t0 + row + sg.shift;
        float v[8];
        const int kk = k0 + kh * 8;
        if (t >= 0 && t < p.T && t0 + row < p.T && kk < sg.k_len) {
          const size_t off = (size_t)b * a_bs + (size_t)t * a_rs + sg.c_off + kk;
          if (p.single) fd_load_hi8(src, off, v, p.prec);
          else fd_load_planes<8>(src, a_plane, off, v, p.prec);
        } else {
#pragma unroll
          for (int i = 0; i < 8; ++i) v[i] = 0.f;
        }
#pragma unroll
        for (int i = 0; i < 8; ++i) As[kh * 8 + i][row] = v[i];
      }
      // ---- load W tile: BN rows x 16 k
      if (tid < BN * 2) {
        const int nl = tid % BN, kh = tid / BN;
        const int n = nl < RUN ? run0 + nl : run1 + (nl - RUN);
        const int kk = k0 + kh * 8;
        float v[8];
        if (n < p.n_total && kk < sg.k_len) {
          const size_t off = (size_t)n * p.k_total + koff + kk + p.w_kshift;
          if (p.single) fd_load_hi8(p.w, off, v, p.prec);
          else fd_load_planes<8>(p.w, w_plane, off, v, p.prec);
        } else {
#pragma unroll
          for (int i = 0; i < 8; ++i) v[i] = 0.f;
        }
#pragma unroll
        for (int i = 0; i < 8; ++i) Bs[kh * 8 + i][nl] = v[i];
      }
      __syncthreads();
#pragma unroll
      for (int k = 0; k < BK; ++k) {
        float a[RM], bv[8];
#pragma unroll
        for (int r = 0; r < RM; ++r) a[r] = As[k][ty * RM + r];
        float4 b0 = *reinterpret_cast<const float4*>(&Bs[k][tx * 4]);
        float4 b1 = *reinterpret_cast<const float4*>(&Bs[k][RUN + tx * 4]);
        bv[0] = b0.x; bv[1] = b0.y; bv[2] = b0.z; bv[3] = b0.w;
        bv[4] = b1.x; bv[5] = b1.y; bv[6] = b1.z; bv[7] = b1.w;
#pragma unroll
        for (int r = 0; r < RM; ++r)
#pragma unroll
          for (int c = 0; c < 8; ++c) acc[r][c] = fmaf(a[r], bv[c], acc[r][c]);
      }
      __syncthreads();
    }
    koff += sg.k_len;
  }

  // ---- epilogue
#pragma unroll
  for (int r = 0; r < RM; ++r) {
    const int t = t0 + ty * RM + r;
    if (t >= p.T) continue;
    float v0[4] = {acc[r][0], acc[r][1], acc[r][2], acc[r][3]};
    float v1[4] = {acc[r][4], acc[r][5], acc[r][6], acc[r][7]};
    const int n_a = run0 + tx * 4, n_b = run1 + tx * 4;
    if (EPI == FD_EPI_LINEAR) {
      const float* bias = p.bias ? p.bias + (size_t)b * p.bias_bstride : nullptr;
      if (n_a < p.n_total) fd_epi_linear<4>(p, b, t, n_a, v0, bias, 0);
      if (n_b < p.n_total) fd_epi_linear<4>(p, b, t, n_b, v1, bias, 0);
    } else if (EPI == FD_EPI_GATE) {
      if (n_a < p.n_total) {
        const size_t bo = (size_t)b * p.gbias_bstride;
        fd_epi_gate<4>(p, b, t, j * RUN + tx * 4, n_a, n_b, v0, v1,
                       p.gbias_full + bo + n_a, p.gbias_full + bo + n_b,
                       p.gbias_lo + bo + n_a, p.gbias_lo + bo + n_b,
                       p.gbias_hi + bo + n_a, p.gbias_hi + bo + n_b);
      }
    } else if (EPI == FD_EPI_MAG) {
      if (n_a < p.n_total) fd_epi_mag<4>(p, b, t, j * RUN + tx * 4, v0, v1);
    } else {
      const float* bias = p.bias + (size_t)b * p.bias_bstride;
      if (n_a < p.n_total) fd_epi_res_skip<4>(p, b, t, n_a, v0, bias + n_a);
      if (n_b < p.n_total) fd_epi_res_skip<4>(p, b, t, n_b, v1, bias + n_b);
    }
  }
}

template <int RUN>
int launch_run(const FdTapGemm& p, cudaStream_t stream) {
  const int tiles_t = (p.T + BM - 1) / BM;
  dim3 grid(p.B * tiles_t, 1, 1), block(256);
  if (p.epi == FD_EPI_GATE) {
    grid.y = (p.n_total / 2 + RUN - 1) / RUN;
    fd_tapgemm_simt_kernel<RUN, FD_EPI_GATE><<<grid, block, 0, stream>>>(p);
  } else if (p.epi == FD_EPI_MAG) {
    grid.y = (p.n_total / 2 + RUN - 1) / RUN;
    fd_tapgemm_simt_kernel<RUN, FD_EPI_MAG><<<grid, block, 0, stream>>>(p);
  } else if (p.epi == FD_EPI_RES_SKIP) {
    grid.y = (p.n_total + 2 * RUN - 1) / (2 * RUN);
    fd_tapgemm_simt_kernel<RUN, FD_EPI_RES_SKIP><<<grid, block, 0, stream>>>(p);
  } else {
    grid.y = (p.n_total + 2 * RUN - 1) / (2 * RUN);
    fd_tapgemm_simt_kernel<RUN, FD_EPI_LINEAR><<<grid, block, 0, stream>>>(p);
  }
  FD_CHECK_CUDA(cudaGetLastError());
  return 0;
}

// ---- weight gradient (fd_wgrad_cl): one CTA per (split, WG_R-row tile, WG_C-column tile) loops over the items of its
//      split and their time steps, WG_T steps at a time; both operands are staged [t][channel] in shared memory
constexpr int WG_R = 64, WG_C = 64, WG_T = 16;

__global__ void __launch_bounds__(256) fd_wgrad_simt_kernel(const FdWgradK p, const uint16_t* row0,
                                                            const uint16_t* row1, const uint16_t* col0,
                                                            const uint16_t* col1, int prec, int single) {
  static_assert(WG_R == WG_C, "rows and columns share the staging code");
  __shared__ __align__(16) float Rs[WG_T][WG_R + 4];
  __shared__ __align__(16) float Cs[WG_T][WG_C + 4];
  const int tid = threadIdx.x;
  const int s = blockIdx.z, r0 = blockIdx.y * WG_R, c0 = blockIdx.x * WG_C;

  // staging: threads [0,128) load rows, [128,256) columns; each thread one 8-channel group at one time step of a block.
  // Segment widths and starts are multiples of 8, so a group lies in one segment (or past the last one: zeros).
  const bool is_col = tid >= 128;
  const int grp = tid % 8, tl = (tid % 128) / 8;
  const int i = (is_col ? c0 : r0) + grp * 8;
  const uint16_t* src = nullptr;
  int C = 0, ch = 0, shift = 0;
  if (!is_col) {
    for (int g = 0; g < p.num_row_seg; ++g)
      if (i >= p.row_start[g] && i < p.row_start[g] + p.row_width[g]) {
        src = p.row_src[g] == 0 ? row0 : row1;
        C = p.row_C[p.row_src[g]]; ch = p.row_coff[g] + (i - p.row_start[g]);
      }
  } else {
    for (int g = 0; g < p.num_col_seg; ++g)
      if (i >= p.col_start[g] && i < p.col_start[g] + p.col_width[g]) {
        src = p.col_src[g] == 0 ? col0 : col1;
        C = p.col_C[p.col_src[g]]; ch = p.col_coff[g] + (i - p.col_start[g]); shift = p.col_shift[g];
      }
  }
  const size_t plane = (size_t)p.B * p.T * C;
  float* const dst = is_col ? &Cs[tl][grp * 8] : &Rs[tl][grp * 8];

  const int tx = tid % 16, ty = tid / 16;      // this thread's outputs: rows r0 + 4 ty .. +4, columns c0 + 4 tx .. +4
  float acc[4][4];
#pragma unroll
  for (int r = 0; r < 4; ++r)
#pragma unroll
    for (int c = 0; c < 4; ++c) acc[r][c] = 0.f;

  const int b_end = min(p.B, (s + 1) * p.items_per_split);
  for (int b = s * p.items_per_split; b < b_end; ++b) {
    for (int t0 = 0; t0 < p.T; t0 += WG_T) {
      const int t = t0 + tl, ts = t + shift;   // a column segment's tap shift reads zero outside [0,T)
      float v[8];
      if (src != nullptr && t < p.T && ts >= 0 && ts < p.T) {
        const size_t off = ((size_t)b * p.T + ts) * C + ch;
        if (single) fd_load_hi8(src, off, v, prec);
        else fd_load_planes<8>(src, plane, off, v, prec);
      } else {
#pragma unroll
        for (int k = 0; k < 8; ++k) v[k] = 0.f;
      }
      *reinterpret_cast<float4*>(dst) = make_float4(v[0], v[1], v[2], v[3]);
      *reinterpret_cast<float4*>(dst + 4) = make_float4(v[4], v[5], v[6], v[7]);
      __syncthreads();
#pragma unroll
      for (int k = 0; k < WG_T; ++k) {
        const float4 a = *reinterpret_cast<const float4*>(&Rs[k][ty * 4]);
        const float4 c = *reinterpret_cast<const float4*>(&Cs[k][tx * 4]);
        const float av[4] = {a.x, a.y, a.z, a.w}, cv[4] = {c.x, c.y, c.z, c.w};
#pragma unroll
        for (int r = 0; r < 4; ++r)
#pragma unroll
          for (int cc = 0; cc < 4; ++cc) acc[r][cc] = fmaf(av[r], cv[cc], acc[r][cc]);
      }
      __syncthreads();
    }
  }

  const int col = c0 + tx * 4;                 // Cc is a multiple of 8: a 4-column group is all in or all out
  if (col >= p.Cc) return;
  float* const out = p.part + (size_t)s * p.R * p.Cc;
#pragma unroll
  for (int r = 0; r < 4; ++r) {
    const int row = r0 + ty * 4 + r;
    if (row < p.R)
      *reinterpret_cast<float4*>(out + (size_t)row * p.Cc + col) = make_float4(
          acc[r][0] * p.acc_scale, acc[r][1] * p.acc_scale, acc[r][2] * p.acc_scale, acc[r][3] * p.acc_scale);
  }
}

}  // namespace

int fd_tapgemm_simt_launch(const FdTapGemm& p, cudaStream_t stream) {
  FD_REQUIRE(p.n_total % 4 == 0, "tapgemm(simt): n_total=%d must be a multiple of 4", p.n_total);
  FD_REQUIRE(p.k_total % 8 == 0 && p.w_kshift % 8 == 0,
             "tapgemm(simt): k_total=%d and w_kshift=%d must be multiples of 8", p.k_total, p.w_kshift);
  for (int s = 0; s < p.num_seg; ++s) {
    FD_REQUIRE(p.seg[s].k_len % 8 == 0 && p.seg[s].c_off % 8 == 0 && p.src_rs[p.seg[s].src] % 8 == 0 &&
                   p.src_bs[p.seg[s].src] % 8 == 0 && p.src_ps[p.seg[s].src] % 8 == 0,
               "tapgemm(simt): segment %d needs k_len/c_off/strides multiples of 8", s);
  }
  if (p.epi == FD_EPI_GATE || p.epi == FD_EPI_MAG) {
    const int half = p.gate_tile / 2;
    FD_REQUIRE(half > 0 && p.n_total % p.gate_tile == 0, "tapgemm(simt): bad gate_tile %d", p.gate_tile);
    if (half % 64 == 0) return launch_run<64>(p, stream);
    FD_REQUIRE(half % 16 == 0, "tapgemm(simt): gate_tile/2=%d must be a multiple of 16", half);
    return launch_run<16>(p, stream);
  }
  if (p.epi == FD_EPI_RES_SKIP) {
    FD_REQUIRE(p.C % 4 == 0 && p.n_total == 2 * p.C, "tapgemm(simt): res/skip needs n_total == 2C");
  }
  if (p.n_total >= 96) return launch_run<64>(p, stream);
  return launch_run<16>(p, stream);
}

int fd_wgrad_simt_launch(const FdWgradK& p, const uint16_t* const* row_ptr, const uint16_t* const* col_ptr, int prec,
                         cudaStream_t stream) {
  dim3 grid((p.Cc + WG_C - 1) / WG_C, (p.R + WG_R - 1) / WG_R, p.splits);
  fd_wgrad_simt_kernel<<<grid, 256, 0, stream>>>(p, row_ptr[0], row_ptr[1], col_ptr[0], col_ptr[1], prec & 0xF,
                                                 (prec & FD_SINGLE) != 0);
  FD_CHECK_CUDA(cudaGetLastError());
  return 0;
}
