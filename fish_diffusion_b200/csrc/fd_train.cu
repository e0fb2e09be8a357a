// Memory-bound kernels of the WaveNet training step (backward pass), and fd_wavenet_block_bwd, which issues the whole
// backward of one residual block on either back end (wavenet.py:106-120 differentiated by hand; checked against the
// reference's autograd in the tests).  Data gradients are tap-GEMM launches (fd_tapgemm_*.cu) on transposed packed
// weights with mirrored tap shifts; weight gradients are fd_wgrad_cl launches that read both operands straight from the
// channels-last planes, with time as the contraction axis.
#include <cstring>
#include "fd_common.cuh"
#include "fd_host.h"

namespace {

// grad (fp32 [n]) masked by the sign of the forward activation (planes): out planes = split(grad * (act > 0) * scale)
__global__ void k_relu_bwd(const float* __restrict__ grad, const uint16_t* __restrict__ act, uint16_t* __restrict__ out,
                           long long n, float scale, int prec) {
  const long long n4 = n / 4;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
    const long long e = i * 4;
    float a[4], g[4];
    fd_load_planes<4>(act, (size_t)n, (size_t)e, a, prec);
    fd_load_f32<4>(grad + e, g);
#pragma unroll
    for (int k = 0; k < 4; ++k) g[k] = a[k] > 0.f ? g[k] * scale : 0.f;
    fd_store_planes<4>(out, (size_t)n, (size_t)e, g, prec);
  }
}

// LeakyReLU backward with an optional addend (autograd of `x + c2(lrelu(c1(lrelu(x))))`, nsf_hifigan/models.py:103-110):
//   v = grad * (act > 0 ? 1 : slope) * scale + addend      act = planes of lrelu(x) (same sign as x)
// -> out_f32 and / or out_planes (either may be null, not both)
__global__ void k_lrelu_bwd(const float* __restrict__ grad, const uint16_t* __restrict__ act,
                            const float* __restrict__ addend, float* __restrict__ out_f32,
                            uint16_t* __restrict__ out_planes, long long n, float slope, float scale, int prec) {
  const long long n4 = n / 4;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
    const long long e = i * 4;
    float a[4], g[4];
    fd_load_planes<4>(act, (size_t)n, (size_t)e, a, prec);
    fd_load_f32<4>(grad + e, g);
#pragma unroll
    for (int k = 0; k < 4; ++k) g[k] = (a[k] > 0.f ? g[k] : g[k] * slope) * scale;
    if (addend != nullptr) {
      float r[4];
      fd_load_f32<4>(addend + e, r);
#pragma unroll
      for (int k = 0; k < 4; ++k) g[k] += r[k];
    }
    if (out_f32 != nullptr) fd_store_f32<4>(out_f32 + e, g);
    if (out_planes != nullptr) fd_store_planes<4>(out_planes, (size_t)n, (size_t)e, g, prec);
  }
}

// column sums per batch item: in (planes [2][B][T][N] or fp32 [B][T][N]) -> out[b][n] += scale * sum_t in[b,t,n]
// (out must be zero-initialised; fp32 atomics over the row chunks)
__global__ void k_colsum(const uint16_t* __restrict__ planes, const float* __restrict__ f32, float* __restrict__ out,
                         int B, int T, int N, float scale, int rows_per_block, int prec) {
  const int b = blockIdx.z;
  const int n = blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= N) return;
  const int t0 = blockIdx.y * rows_per_block;
  const int t1 = min(T, t0 + rows_per_block);
  const size_t plane = (size_t)B * T * N;
  float acc = 0.f;
  for (int t = t0; t < t1; ++t) {
    const size_t off = ((size_t)b * T + t) * N + n;
    acc += planes != nullptr ? fd_combine(planes[off], planes[plane + off], prec) : f32[off];
  }
  atomicAdd(out + (size_t)b * N + n, acc * scale);
}

// out[i] = scale * sum_b in[b][i]
__global__ void k_reduce_batch(const float* __restrict__ in, float* __restrict__ out, int B, long long n, float scale) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    float acc = 0.f;
    for (int b = 0; b < B; ++b) acc += in[(size_t)b * n + i];
    out[i] = acc * scale;
  }
}

inline int grid1d(long long work, int block = 256, int cap = 132 * 16) {
  long long g = (work + block - 1) / block;
  return (int)(g < 1 ? 1 : (g > cap ? cap : g));
}

}  // namespace

extern "C" {

int fd_relu_bwd(const float* grad, const uint16_t* act_planes, uint16_t* out_planes, long long n, float scale, int prec,
                void* stream) {
  FD_DEVICE_GUARD();
  FD_REQUIRE(n % 4 == 0, "fd_relu_bwd: n=%lld must be a multiple of 4", n);
  k_relu_bwd<<<grid1d(n / 4), 256, 0, (cudaStream_t)stream>>>(grad, act_planes, out_planes, n, scale, prec);
  FD_LAUNCHED();
  return 0;
}

int fd_lrelu_bwd(const float* grad, const uint16_t* act_planes, const float* addend, float* out_f32,
                 uint16_t* out_planes, long long n, float slope, float scale, int prec, void* stream) {
  FD_DEVICE_GUARD();
  FD_REQUIRE(n > 0 && n % 4 == 0, "fd_lrelu_bwd: n=%lld must be a positive multiple of 4", n);
  FD_REQUIRE(grad != nullptr && act_planes != nullptr && (out_f32 != nullptr || out_planes != nullptr),
             "fd_lrelu_bwd: grad, act_planes and at least one output are required");
  k_lrelu_bwd<<<grid1d(n / 4), 256, 0, (cudaStream_t)stream>>>(grad, act_planes, addend, out_f32, out_planes, n, slope,
                                                               scale, prec);
  FD_LAUNCHED();
  return 0;
}

int fd_colsum(const uint16_t* planes, const float* f32, float* out, int B, int T, int N, float scale, int prec,
              void* stream) {
  FD_DEVICE_GUARD();
  FD_REQUIRE((planes != nullptr) != (f32 != nullptr), "fd_colsum: exactly one of planes / f32 must be given");
  const int rows_per_block = 128;
  dim3 grid((N + 127) / 128, (T + rows_per_block - 1) / rows_per_block, B);
  k_colsum<<<grid, 128, 0, (cudaStream_t)stream>>>(planes, f32, out, B, T, N, scale, rows_per_block, prec);
  FD_LAUNCHED();
  return 0;
}

int fd_reduce_batch(const float* in, float* out, int B, long long n, float scale, void* stream) {
  FD_DEVICE_GUARD();
  k_reduce_batch<<<grid1d(n), 256, 0, (cudaStream_t)stream>>>(in, out, B, n, scale);
  FD_LAUNCHED();
  return 0;
}

int fd_wavenet_block_bwd(const fd_wavenet_bwd_desc* d, void* stream) {
  FD_DEVICE_GUARD();
  FD_REQUIRE(d != nullptr, "fd_wavenet_block_bwd: null descriptor");
  const int B = d->B, T = d->T, C = d->C, E = d->E, dil = d->dilation;
  // the tensor-core weight gradient takes 64-channel segments, its SIMT twin 8
  const int unit = d->backend == FD_BACKEND_TC ? 64 : 8;
  FD_REQUIRE(B > 0 && T > 0 && C % unit == 0 && E % unit == 0 && dil > 0,
             "fd_wavenet_block_bwd: bad shape B=%d T=%d C=%d E=%d (backend %d)", B, T, C, E, d->backend);
  const float inv_sqrt2 = 0.70710678118654752440f;
  int rc;
  // ---- dy = gate backward of dz = [dx_next | d_skip] . W2 and the column sums of dy, both in the GEMM's epilogue (K
  //      offset C selects the skip half of W2^T when there is no residual gradient)
  {
    fd_gemm_desc g;
    memset(&g, 0, sizeof(g));
    g.w = d->w2t; g.n_total = C; g.k_total = 2 * C; g.B = B; g.T = T;
    g.w_inv_scale = d->w2t_inv; g.res_scale = 1.f; g.post_scale = 1.f; g.planes_scale = 1.f;
    g.prec = d->prec; g.backend = d->backend;
    g.out_planes = d->dy;
    g.gate_y = d->y_planes; g.gate_tile = d->gate_tile; g.gate_dil = dil < T ? dil : T;
    g.gate_cs = d->cs_dy; g.gate_cs_edge = d->cs_edge; g.gate_cs_scale = d->inv_S;
    if (d->dx_next == nullptr) {
      g.src[0] = d->dskip; g.src_C[0] = C; g.num_seg = 1; g.w_kshift = C;
      g.seg_src[0] = 0; g.seg_shift[0] = 0; g.seg_coff[0] = 0; g.seg_klen[0] = C;
    } else {
      g.src[0] = d->dx_next; g.src_C[0] = C; g.src[1] = d->dskip; g.src_C[1] = C; g.num_seg = 2;
      g.seg_src[0] = 0; g.seg_klen[0] = C; g.seg_src[1] = 1; g.seg_klen[1] = C;
    }
    rc = fd_gemm_cl_fwd(&g, stream);
    if (rc) return rc;
  }
  // ---- gw2 = [dx_next ; d_skip]^T . z
  {
    fd_wgrad_desc w;
    memset(&w, 0, sizeof(w));
    w.col_src[0] = d->z_planes; w.col_C[0] = C; w.num_col_seg = 1; w.col_seg_width[0] = C;
    w.B = B; w.T = T; w.splits = d->splits2; w.part = d->part2; w.acc_scale = 1.f; w.prec = d->prec;
    w.backend = d->backend;
    float* out = d->gw2;
    int R = 2 * C;
    if (d->dx_next == nullptr) {
      FD_CHECK_CUDA(cudaMemsetAsync(d->gw2, 0, (size_t)C * C * sizeof(float), (cudaStream_t)stream));
      w.row_src[0] = d->dskip; w.row_C[0] = C; w.num_row_seg = 1; w.row_seg_width[0] = C;
      out = d->gw2 + (size_t)C * C; R = C;
    } else {
      w.row_src[0] = d->dx_next; w.row_C[0] = C; w.row_src[1] = d->dskip; w.row_C[1] = C; w.num_row_seg = 2;
      w.row_seg_src[0] = 0; w.row_seg_width[0] = C; w.row_seg_src[1] = 1; w.row_seg_width[1] = C;
    }
    rc = fd_wgrad_cl(&w, stream);
    if (rc) return rc;
    rc = fd_reduce_batch(d->part2, out, d->splits2, (long long)R * C, d->inv_S, stream);
    if (rc) return rc;
  }
  // ---- gw1 = dy^T . [x(t-d) | x(t) | x(t+d) | cond]
  {
    fd_wgrad_desc w;
    memset(&w, 0, sizeof(w));
    w.row_src[0] = d->dy; w.row_C[0] = 2 * C; w.num_row_seg = 1; w.row_seg_width[0] = 2 * C;
    w.col_src[0] = d->x_planes; w.col_C[0] = C; w.col_src[1] = d->cond_planes; w.col_C[1] = E; w.num_col_seg = 4;
    const int sh[3] = {-dil, 0, dil};
    for (int j = 0; j < 3; ++j) { w.col_seg_src[j] = 0; w.col_seg_shift[j] = sh[j]; w.col_seg_width[j] = C; }
    w.col_seg_src[3] = 1; w.col_seg_width[3] = E;
    w.B = B; w.T = T; w.splits = d->splits1; w.part = d->part1; w.acc_scale = 1.f; w.prec = d->prec;
    w.backend = d->backend;
    rc = fd_wgrad_cl(&w, stream);
    if (rc) return rc;
    rc = fd_reduce_batch(d->part1, d->gw1, d->splits1, (long long)2 * C * (3 * C + E), d->inv_S, stream);
    if (rc) return rc;
  }
  // ---- dx_l = conv^T(dy) + dx_next/sqrt2 (mirrored tap shifts, K = 6C)
  {
    fd_gemm_desc g;
    memset(&g, 0, sizeof(g));
    g.src[0] = d->dy; g.src_C[0] = 2 * C; g.w = d->w1t; g.n_total = C; g.k_total = 6 * C; g.B = B; g.T = T; g.num_seg = 3;
    const int sh[3] = {dil, 0, -dil};
    for (int j = 0; j < 3; ++j) { g.seg_src[j] = 0; g.seg_shift[j] = sh[j]; g.seg_klen[j] = 2 * C; }
    g.res_planes = d->dx_next; g.res_scale = inv_sqrt2; g.w_inv_scale = d->w1t_inv; g.post_scale = 1.f; g.planes_scale = 1.f;
    g.out_planes = d->dx_out; g.out_f32 = d->dx_f32; g.prec = d->prec; g.backend = d->backend;
    rc = fd_gemm_cl_fwd(&g, stream);
    if (rc) return rc;
  }
  if (d->d_cond != nullptr) {
    fd_gemm_desc g;
    memset(&g, 0, sizeof(g));
    g.src[0] = d->dy; g.src_C[0] = 2 * C; g.w = d->wct; g.n_total = E; g.k_total = 2 * C; g.B = B; g.T = T; g.num_seg = 1;
    g.seg_klen[0] = 2 * C;
    g.w_inv_scale = d->wct_inv * d->inv_S; g.res_scale = 1.f; g.post_scale = 1.f; g.planes_scale = 1.f;
    g.out_f32 = d->d_cond; g.out_accum = 1; g.prec = d->prec; g.backend = d->backend;
    rc = fd_gemm_cl_fwd(&g, stream);
    if (rc) return rc;
  }
  return fd_colsum(d->dx_out, nullptr, d->cs_dx, B, T, C, d->inv_S, d->prec & 0xF, stream);
}

}  // extern "C"
