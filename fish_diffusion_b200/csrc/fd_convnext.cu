// ConvNext diffusion denoiser (reference fish_diffusion/modules/convnext.py:54-91, 155-261): the fused block front
// (depthwise dilated k=7 conv + LayerNorm, fd_convnext_dwln_fwd) and the whole forward as one native call.  Every dense
// product runs through the LINEAR tap-GEMM (fd_conv_cl_fwd); the block front is the one part that is not a GEMM.
#include <cstring>
#include "fd_common.cuh"
#include "fd_host.h"

namespace {

// One CTA: DW_TT consecutive output steps of one item, one warp per step, all C channels.  The channels go in chunks of
// DW_CK (four per lane); for each chunk the CTA stages the u rows its 7 taps read -- u = mask(x + s + p), zero outside
// [0, T) -- once in shared memory, and each warp keeps its step's conv outputs of every chunk in registers, so that the
// LayerNorm statistics are two passes over values already on chip.
constexpr int DW_TT = 16;
constexpr int DW_CK = 128;
constexpr int DW_MAXCH = 8;                    // chunks held in registers: C <= 1024
constexpr int DW_THREADS = DW_TT * 32;
constexpr int DW_Q = DW_CK / 4;                // float4 slots of a staged row
constexpr int DW_SMEM_MAX = 7 * DW_TT * DW_CK * 4;

struct DwlnArgs {
  const uint16_t* x;      // residual stream planes [2][B][T][C]
  const float* p;         // condition projection fp32 [B][T][C]
  const float* s;         // step vectors, item b at s + b * s_bstride
  long long s_bstride;
  const uint8_t* mask;    // [B][T] or null
  const float* dw_w;      // [C][7]
  const float* dw_b;      // [C]
  const float* ln_w;      // [C]
  const float* ln_b;      // [C]
  uint16_t* out;          // planes [2][B][T][C]
  int B, T, C, dil, prec;
};

// Staged row r of a tile starting at t0 holds u at step t0 - 3d + (r / stp) d + r % stp, stp = min(d, DW_TT): for
// d < DW_TT that is the contiguous window [t0 - 3d, t0 + DW_TT + 3d), for d >= DW_TT the 7 disjoint windows of the
// taps.  Either way tap j of output row i reads staged row i + j stp.
__global__ void __launch_bounds__(DW_THREADS) k_convnext_dwln(const DwlnArgs a) {
  extern __shared__ float4 u4[];
  const long long tiles = (a.T + DW_TT - 1) / DW_TT;
  const long long b = blockIdx.x / tiles;
  const long long t0 = (blockIdx.x % tiles) * DW_TT;
  const long long d = a.dil;
  const int stp = (int)min(d, (long long)DW_TT);
  const int rows = DW_TT + 6 * stp;
  const int warp = threadIdx.x / 32, lane = threadIdx.x % 32;
  const size_t plane = (size_t)a.B * a.T * a.C;
  const size_t item = (size_t)b * a.T;
  const float* s = a.s + b * a.s_bstride;
  const int nch = (a.C + DW_CK - 1) / DW_CK;
  float v[DW_MAXCH][4];
#pragma unroll
  for (int ch = 0; ch < DW_MAXCH; ++ch) {
#pragma unroll
    for (int k = 0; k < 4; ++k) v[ch][k] = 0.f;
    if (ch < nch) {                                  // uniform over the CTA
      const int c0 = ch * DW_CK, cw = min(DW_CK, a.C - c0);
      __syncthreads();                               // the previous chunk's readers are done
      for (int i = threadIdx.x; i < rows * DW_Q; i += DW_THREADS) {
        const int r = i / DW_Q, q = i % DW_Q;
        const long long tt = t0 - 3 * d + (long long)(r / stp) * d + r % stp;
        float4 u = make_float4(0.f, 0.f, 0.f, 0.f);
        if (4 * q < cw && tt >= 0 && tt < a.T && (a.mask == nullptr || a.mask[item + tt] == 0)) {
          const int c = c0 + 4 * q;
          const size_t off = (item + tt) * a.C + c;
          float xv[4], pv[4], sv[4];
          fd_load_planes<4>(a.x, plane, off, xv, a.prec);
          fd_load_f32<4>(a.p + off, pv);
          fd_load_f32<4>(s + c, sv);
          u = make_float4((xv[0] + sv[0]) + pv[0], (xv[1] + sv[1]) + pv[1], (xv[2] + sv[2]) + pv[2],
                          (xv[3] + sv[3]) + pv[3]);
        }
        u4[i] = u;
      }
      __syncthreads();
      if (4 * lane < cw) {
        const int c = c0 + 4 * lane;
#pragma unroll
        for (int k = 0; k < 4; ++k) v[ch][k] = __ldg(a.dw_b + c + k);
#pragma unroll
        for (int j = 0; j < 7; ++j) {
          const float4 u = u4[(warp + j * stp) * DW_Q + lane];
          v[ch][0] = fmaf(__ldg(a.dw_w + (size_t)(c + 0) * 7 + j), u.x, v[ch][0]);
          v[ch][1] = fmaf(__ldg(a.dw_w + (size_t)(c + 1) * 7 + j), u.y, v[ch][1]);
          v[ch][2] = fmaf(__ldg(a.dw_w + (size_t)(c + 2) * 7 + j), u.z, v[ch][2]);
          v[ch][3] = fmaf(__ldg(a.dw_w + (size_t)(c + 3) * 7 + j), u.w, v[ch][3]);
        }
      }
    }
  }
  const long long t = t0 + warp;
  if (t >= a.T) return;                              // no barrier follows
  // LayerNorm over the C channels of step t (eps 1e-6, biased variance): mean, then the mean of squared deviations.
  // Lanes past C hold zeros and are left out of the second sum.
  float sum = 0.f;
#pragma unroll
  for (int ch = 0; ch < DW_MAXCH; ++ch)
#pragma unroll
    for (int k = 0; k < 4; ++k) sum += v[ch][k];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
  const float inv_c = 1.f / (float)a.C;
  const float mean = sum * inv_c;
  float sq = 0.f;
#pragma unroll
  for (int ch = 0; ch < DW_MAXCH; ++ch) {
    if (ch < nch && 4 * lane < min(DW_CK, a.C - ch * DW_CK)) {
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const float dv = v[ch][k] - mean;
        sq = fmaf(dv, dv, sq);
      }
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) sq += __shfl_xor_sync(0xffffffffu, sq, o);
  const float rstd = 1.f / sqrtf(sq * inv_c + 1e-6f);
#pragma unroll
  for (int ch = 0; ch < DW_MAXCH; ++ch) {
    const int c = ch * DW_CK + 4 * lane;
    if (ch < nch && c < a.C) {
      float y[4];
#pragma unroll
      for (int k = 0; k < 4; ++k) y[k] = (v[ch][k] - mean) * rstd * __ldg(a.ln_w + c + k) + __ldg(a.ln_b + c + k);
      fd_store_planes<4>(a.out, plane, (item + t) * a.C + c, y, a.prec);
    }
  }
}

int dwln(const DwlnArgs& a, cudaStream_t st) {
  FD_REQUIRE(a.x != nullptr && a.p != nullptr && a.s != nullptr && a.out != nullptr && a.dw_w != nullptr &&
                 a.dw_b != nullptr && a.ln_w != nullptr && a.ln_b != nullptr,
             "fd_convnext_dwln_fwd: null pointer");
  FD_REQUIRE(a.B > 0 && a.T > 0 && a.dil > 0 && a.s_bstride >= 0, "fd_convnext_dwln_fwd: bad shape B=%d T=%d dilation=%d",
             a.B, a.T, a.dil);
  FD_REQUIRE(a.C > 0 && a.C % 16 == 0 && a.C <= DW_MAXCH * DW_CK,
             "fd_convnext_dwln_fwd: C=%d must be a multiple of 16 and at most %d", a.C, DW_MAXCH * DW_CK);
  FD_REQUIRE(a.s_bstride % 4 == 0, "fd_convnext_dwln_fwd: step stride %lld must be a multiple of 4", a.s_bstride);
  const long long blocks = (long long)a.B * ((a.T + DW_TT - 1) / DW_TT);
  FD_REQUIRE(blocks < (1ll << 31), "fd_convnext_dwln_fwd: %lld time tiles exceed the grid", blocks);
  static bool attr_set[FD_MAX_DEVICES] = {false};
  const int dev = fd_current_device();
  if (!attr_set[dev]) {
    FD_CHECK_CUDA(cudaFuncSetAttribute(k_convnext_dwln, cudaFuncAttributeMaxDynamicSharedMemorySize, DW_SMEM_MAX));
    attr_set[dev] = true;
  }
  const int stp = a.dil < DW_TT ? a.dil : DW_TT;
  const int smem = (DW_TT + 6 * stp) * DW_CK * 4;
  k_convnext_dwln<<<(unsigned)blocks, DW_THREADS, smem, st>>>(a);
  FD_LAUNCHED();
  return 0;
}

// out = epilogue(in . W^T): one LINEAR tap-GEMM over channels-last planes (fd_conv_cl_fwd)
struct Linear {
  fd_conv_desc d;
  Linear(int B, int T, int prec, int backend) {
    memset(&d, 0, sizeof(d));
    d.B = B; d.T = T; d.ntaps = 1; d.post_scale = 1.f; d.planes_scale = 1.f; d.prec = prec; d.backend = backend;
  }
  int operator()(const uint16_t* in, int K, const uint16_t* w, float w_inv, const float* bias, int N, int act,
                 const uint8_t* mask, uint16_t* out_planes, float* out_f32, const uint16_t* res_planes, void* stream) {
    d.in_planes = in; d.Cin = K; d.w_planes = w; d.w_inv_scale = w_inv; d.bias = bias; d.N = N; d.act = act;
    d.row_mask = mask; d.out_planes = out_planes; d.out_f32 = out_f32; d.res_planes = res_planes;
    return fd_conv_cl_fwd(&d, stream);
  }
};

int check_desc(const fd_convnext_fwd_desc* d, const char* who) {
  FD_REQUIRE(d != nullptr, "%s: null descriptor", who);
  FD_REQUIRE(d->L >= 1 && d->L <= 64, "%s: L=%d out of range (1..64)", who, d->L);
  FD_REQUIRE(d->B > 0 && d->T > 0 && d->M > 0 && d->C > 0 && d->H > 0 && d->E > 0, "%s: bad shape", who);
  FD_REQUIRE(d->Bs == 1 || d->Bs == d->B, "%s: Bs=%d must be 1 or B=%d", who, d->Bs, d->B);
  return 0;
}

// conditioner_projection (Conv1x1 E->H, GELU, Conv1x1 H->C; convnext.py:177-181, 234), its output masked by cond_mask
// (:239-240), into the planes d->cpl
int cond_mlp(const fd_convnext_fwd_desc* d, void* stream) {
  FD_REQUIRE(d->cond_planes != nullptr && d->cpl != nullptr && d->h != nullptr,
             "fd_convnext: cond_planes and the cpl / h workspaces are required");
  Linear lin(d->B, d->T, d->prec, d->backend);
  int rc = lin(d->cond_planes, d->E, d->w_c1, d->w_c1_inv, d->b_c1, d->H, FD_ACT_GELU, nullptr, d->h, nullptr,
               nullptr, stream);
  if (rc) return rc;
  return lin(d->h, d->H, d->w_c2, d->w_c2_inv, d->b_c2, d->C, FD_ACT_NONE, d->cond_mask, d->cpl, nullptr, nullptr,
             stream);
}

// residual_layers[l].condition_projection(condition) without its bias (the bias rides with the step vector)
int cond_proj_layer(const fd_convnext_fwd_desc* d, int l, float* out, void* stream) {
  Linear lin(d->B, d->T, d->prec, d->backend);
  return lin(d->cpl, d->C, d->w_cp + (size_t)l * 2 * d->C * d->C, d->w_cp_inv[l], nullptr, d->C, FD_ACT_NONE, nullptr,
             nullptr, out, nullptr, stream);
}

}  // namespace

extern "C" {

int fd_convnext_dwln_fwd(const uint16_t* x_planes, const float* cond_proj, const float* step, long long step_bstride,
                         const uint8_t* x_mask, const float* dw_w, const float* dw_b, const float* ln_w,
                         const float* ln_b, uint16_t* out_planes, int B, int T, int C, int dilation, int prec,
                         void* stream) {
  FD_DEVICE_GUARD();
  DwlnArgs a{x_planes, cond_proj, step, step_bstride, x_mask, dw_w, dw_b, ln_w, ln_b, out_planes, B, T, C, dilation,
             prec & 0xF};
  return dwln(a, (cudaStream_t)stream);
}

int fd_convnext_cond_proj(const fd_convnext_fwd_desc* d, void* stream) {
  FD_DEVICE_GUARD();
  if (int rc = check_desc(d, "fd_convnext_cond_proj")) return rc;
  FD_REQUIRE(d->cond_proj != nullptr, "fd_convnext_cond_proj: cond_proj is required");
  int rc = cond_mlp(d, stream);
  for (int l = 0; l < d->L && rc == 0; ++l)
    rc = cond_proj_layer(d, l, d->cond_proj + (size_t)l * d->B * d->T * d->C, stream);
  return rc;
}

int fd_convnext_fwd(const fd_convnext_fwd_desc* d, void* stream) {
  FD_DEVICE_GUARD();
  if (int rc = check_desc(d, "fd_convnext_fwd")) return rc;
  FD_REQUIRE(d->cond_proj != nullptr || d->p != nullptr, "fd_convnext_fwd: without cond_proj the p workspace is required");
  const int B = d->B, T = d->T, M = d->M, C = d->C, H = d->H, L = d->L, Bs = d->Bs;
  cudaStream_t st = (cudaStream_t)stream;
  // step vectors: DiffusionEmbedding -> Linear(C->H) -> GELU -> Linear(H->C) (convnext.py:171-176, 233), then all L
  // diffusion_step_projections in one launch over the stacked [L*C][C] weights; b_step carries each layer's
  // diffusion_step_projection bias plus its condition_projection bias.  sv [Bs][L*C]
  int rc = fd_step_mlp(d->steps, d->emb_w0, d->emb_b0, d->emb_w1, d->emb_b1, d->s, d->mlp_ws, Bs, C, H, 2, st);
  if (rc) return rc;
  rc = fd_small_linear(d->s, d->w_step, d->b_step, d->sv, Bs, C, L * C, C, 0, st);
  if (rc) return rc;
  if (d->cond_proj == nullptr && (rc = cond_mlp(d, stream)) != 0) return rc;
  Linear lin(B, T, d->prec, d->backend);
  // head: gelu(input_projection(x)), masked (convnext.py:230-231, 236-237)
  rc = lin(d->x_planes, M, d->w_in, d->w_in_inv, d->b_in, C, FD_ACT_GELU, d->x_mask, d->xr, nullptr, nullptr, stream);
  if (rc) return rc;
  const long long s_bstride = Bs > 1 ? (long long)L * C : 0;
  for (int l = 0; l < L; ++l) {
    const float* p = d->p;
    if (d->cond_proj != nullptr) {
      p = d->cond_proj + (size_t)l * B * T * C;
    } else if ((rc = cond_proj_layer(d, l, d->p, stream)) != 0) {
      return rc;
    }
    // block front: LayerNorm(dwconv(mask(x + step + condition)))  (convnext.py:64-78)
    DwlnArgs a{d->xr, p, d->sv + (size_t)l * C, s_bstride, d->x_mask, d->dw_w + (size_t)l * C * 7,
               d->dw_b + (size_t)l * C, d->ln_w + (size_t)l * C, d->ln_b + (size_t)l * C, d->a, B, T, C,
               d->dilation[l], d->prec & 0xF};
    if ((rc = dwln(a, st)) != 0) return rc;
    // pwconv1 + GELU, then pwconv2 with gamma folded into its rows and bias, + residual, masked, in place (:79-89)
    rc = lin(d->a, C, d->w_pw1 + (size_t)l * 2 * H * C, d->w_pw1_inv[l], d->b_pw1 + (size_t)l * H, H, FD_ACT_GELU,
             nullptr, d->h, nullptr, nullptr, stream);
    if (rc) return rc;
    rc = lin(d->h, H, d->w_pw2 + (size_t)l * 2 * C * H, d->w_pw2_inv[l], d->b_pw2 + (size_t)l * C, C, FD_ACT_NONE,
             d->x_mask, d->xr, nullptr, d->xr, stream);
    if (rc) return rc;
  }
  // tail: Conv1x1(C->C), GELU, Conv1x1(C->M), masked (:201-206, 257-259)
  rc = lin(d->xr, C, d->w_o1, d->w_o1_inv, d->b_o1, C, FD_ACT_GELU, nullptr, d->a, nullptr, nullptr, stream);
  if (rc) return rc;
  return lin(d->a, C, d->w_o2, d->w_o2_inv, d->b_o2, M, FD_ACT_NONE, d->x_mask, nullptr, d->out, nullptr, stream);
}

}  // extern "C"
