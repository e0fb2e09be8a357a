// Layout/packing kernels, the WaveNet step-embedding path, and the sampler's fused elementwise updates.
// All of these are HBM-bound (or tiny): coalesced, vectorised, no tensor cores.
#include <curand_kernel.h>
#include "fd_common.cuh"
#include "fd_host.h"

namespace {

// ---------------------------------------------------------------------------------- layout kernels
// fp32 [B,C,T] -> planes [2][B][T][C] through a 32x33 smem tile (coalesced on both sides)
__global__ void k_split_ncw(const float* __restrict__ src, const uint8_t* __restrict__ mask,
                            uint16_t* __restrict__ planes, int B, int C, int T, int prec) {
  __shared__ float tile[32][33];
  const int b = blockIdx.z;
  const int c0 = blockIdx.y * 32, t0 = blockIdx.x * 32;
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int c = c0 + i, t = t0 + threadIdx.x;
    tile[i][threadIdx.x] = (c < C && t < T) ? src[((size_t)b * C + c) * T + t] : 0.f;
  }
  __syncthreads();
  const size_t plane = (size_t)B * T * C;
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int t = t0 + i, c = c0 + threadIdx.x;
    if (t < T && c < C) {
      float v = tile[threadIdx.x][i];
      if (mask != nullptr && mask[(size_t)b * T + t]) v = 0.f;
      uint16_t hi, lo;
      fd_split(v, prec, hi, lo);
      const size_t off = ((size_t)b * T + t) * C + c;
      planes[off] = hi;
      planes[plane + off] = lo;
    }
  }
}

__global__ void k_split_nwc(const float* __restrict__ src, const uint8_t* __restrict__ mask,
                            uint16_t* __restrict__ planes, long long rows, int C, float scale, int prec) {
  const long long n4 = rows * C / 4;
  const size_t plane = (size_t)rows * C;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n4;
       i += (long long)gridDim.x * blockDim.x) {
    const long long e = i * 4;
    float v[4];
    fd_load_f32<4>(src + e, v);
    const bool m = mask != nullptr && mask[e / C] != 0;
#pragma unroll
    for (int k = 0; k < 4; ++k) v[k] = m ? 0.f : v[k] * scale;
    fd_store_planes<4>(planes, plane, (size_t)e, v, prec);
  }
}

// out = split(lrelu((sum_i invlrelu(in_i)) * scale, out_slope)): the multi-receptive-field average + LeakyReLU that
// feeds the next upsampling stage (models.py:420,426-434), on plane tensors
struct MrfIn { const uint16_t* p[4]; };
__global__ void k_mrf_finish(MrfIn in, int num, uint16_t* __restrict__ out, long long n, float in_slope_inv,
                             float scale, float out_slope, int prec) {
  const long long n8 = n / 8;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n8;
       i += (long long)gridDim.x * blockDim.x) {
    const size_t e = (size_t)i * 8;
    float acc[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) acc[k] = 0.f;
    for (int s = 0; s < num; ++s) {
      float v[8];
      fd_load_planes<8>(in.p[s], (size_t)n, e, v, prec);
#pragma unroll
      for (int k = 0; k < 8; ++k) acc[k] += v[k] >= 0.f ? v[k] : v[k] * in_slope_inv;
    }
#pragma unroll
    for (int k = 0; k < 8; ++k) acc[k] = fd_act(acc[k] * scale, out_slope);
    fd_store_planes<8>(out, (size_t)n, e, acc, prec);
  }
}

// generic 2-D transpose of the two inner dims: src [B][R][S] -> dst [B][S][R]
__global__ void k_transpose(const float* __restrict__ src, float* __restrict__ dst, int R, int S) {
  __shared__ float tile[32][33];
  const int b = blockIdx.z;
  const int r0 = blockIdx.y * 32, s0 = blockIdx.x * 32;
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int r = r0 + i, s = s0 + threadIdx.x;
    tile[i][threadIdx.x] = (r < R && s < S) ? src[((size_t)b * R + r) * S + s] : 0.f;
  }
  __syncthreads();
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int s = s0 + i, r = r0 + threadIdx.x;
    if (s < S && r < R) dst[((size_t)b * S + s) * R + r] = tile[threadIdx.x][i];
  }
}

__global__ void k_pack_weight(const float* __restrict__ w, uint16_t* __restrict__ planes, long long n, float scale,
                              int prec) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n;
       i += (long long)gridDim.x * blockDim.x) {
    uint16_t hi, lo;
    fd_split(w[i] * scale, prec, hi, lo);
    planes[i] = hi;
    planes[n + i] = lo;
  }
}

// ---------------------------------------------------------------------------------- batched WaveNet weight packing
// All residual layers in two launches, reading the raw parameters (conv [2C][C][3], conditioner [2C][E], output
// projection [2C][C]) through device pointer tables: forward packs (gate/filter row interleave per column tile, taps
// and conditioner concatenated along K), the fp32 copy the gate-bias fold reads, and -- for training -- the transposed
// packs of the data-gradient GEMMs.  A training step repacks every step, so this replaces ~25 small launches per layer.
struct PackLayersArgs {
  const float* const* conv_w;
  const float* const* cond_w;
  const float* const* out_w;
  const float* scales;      // [2][L]: s1 (conv + conditioner), s2 (output projection)
  float* w1p_f32;           // [L][2C][KT]
  uint16_t* w1;             // [L][2][2C][KT]
  uint16_t* w2;             // [L][2][2C][C]
  uint16_t* w1t;            // [L][2][C][6C]   or null
  uint16_t* wct;            // [L][2][E][2C]   or null
  uint16_t* w2t;            // [L][2][C][2C]   or null (residual half carries 1/sqrt2)
  int L, C, E, half, prec;
};

__device__ __forceinline__ int packed_to_orig_row(int rp, int C, int half) {
  const int q = rp / (2 * half), w = rp % (2 * half);
  return w < half ? q * half + w : C + q * half + (w - half);
}

__global__ void k_pack_layers_w1(const PackLayersArgs a) {
  __shared__ float tile[32][33];
  const int l = blockIdx.z, C = a.C, E = a.E, KT = 3 * C + E, R = 2 * C;
  const int r0 = blockIdx.y * 32, k0 = blockIdx.x * 32;
  const float s1 = a.scales[l];
  const float* cw = a.conv_w[l];
  const float* dw = a.cond_w[l];
  const size_t pl1 = (size_t)R * KT;
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int rp = r0 + i, k = k0 + threadIdx.x;
    float v = 0.f;
    if (rp < R && k < KT) {
      const int ro = packed_to_orig_row(rp, C, a.half);
      v = k < 3 * C ? cw[((size_t)ro * C + (k % C)) * 3 + k / C] : dw[(size_t)ro * E + (k - 3 * C)];
      a.w1p_f32[((size_t)l * R + rp) * KT + k] = v;
      v *= s1;
      uint16_t hi, lo;
      fd_split(v, a.prec, hi, lo);
      const size_t o = (size_t)l * 2 * pl1 + (size_t)rp * KT + k;
      a.w1[o] = hi;
      a.w1[o + pl1] = lo;
    }
    tile[i][threadIdx.x] = v;
  }
  if (a.w1t == nullptr) return;
  __syncthreads();
  const size_t plt = (size_t)C * 6 * C, plc = (size_t)E * R;
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int k = k0 + i, rp = r0 + threadIdx.x;
    if (rp >= R || k >= KT) continue;
    uint16_t hi, lo;
    fd_split(tile[threadIdx.x][i], a.prec, hi, lo);
    if (k < 3 * C) {
      const int j = k / C, c = k % C;
      const size_t o = (size_t)l * 2 * plt + (size_t)c * 6 * C + (size_t)j * R + rp;
      a.w1t[o] = hi;
      a.w1t[o + plt] = lo;
    } else {
      const size_t o = (size_t)l * 2 * plc + (size_t)(k - 3 * C) * R + rp;
      a.wct[o] = hi;
      a.wct[o + plc] = lo;
    }
  }
}

__global__ void k_pack_layers_w2(const PackLayersArgs a) {
  __shared__ float tile[32][33];
  const int l = blockIdx.z, C = a.C, R = 2 * C;
  const int n0 = blockIdx.y * 32, c0 = blockIdx.x * 32;
  const float s2 = a.scales[a.L + l];
  const float* ow = a.out_w[l];
  const size_t pl = (size_t)R * C;
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int n = n0 + i, c = c0 + threadIdx.x;
    float v = 0.f;
    if (n < R && c < C) {
      v = ow[(size_t)n * C + c] * s2;
      uint16_t hi, lo;
      fd_split(v, a.prec, hi, lo);
      const size_t o = (size_t)l * 2 * pl + (size_t)n * C + c;
      a.w2[o] = hi;
      a.w2[o + pl] = lo;
    }
    tile[i][threadIdx.x] = v;
  }
  if (a.w2t == nullptr) return;
  __syncthreads();
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int c = c0 + i, n = n0 + threadIdx.x;
    if (n >= R || c >= C) continue;
    uint16_t hi, lo;
    fd_split(tile[threadIdx.x][i] * (n < C ? 0.70710678118654752440f : 1.f), a.prec, hi, lo);
    const size_t o = (size_t)l * 2 * pl + (size_t)c * R + n;
    a.w2t[o] = hi;
    a.w2t[o + pl] = lo;
  }
}

// ---------------------------------------------------------------------------------- step embedding
// wavenet.py:20-27: emb_j = exp(j * -(ln(1e4)/(half-1))) ; [sin(t*emb), cos(t*emb)]
__global__ void k_step_embed(const float* __restrict__ steps, float* __restrict__ emb, int Bs, int C) {
  const int half = C / 2;
  const float scale = logf(10000.f) / (float)(half - 1);
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < Bs * half; i += gridDim.x * blockDim.x) {
    const int bs = i / half, j = i % half;
    const float f = expf((float)j * -scale);
    const float a = steps[bs] * f;
    emb[(size_t)bs * C + j] = sinf(a);
    emb[(size_t)bs * C + half + j] = cosf(a);
  }
}

// y[bs][n] = act( sum_k x[bs][k] * w[n*w_pitch + k] + bias[n] ), one warp per n, all bs.
// act: 0 none, 1 Mish (x * tanh(softplus(x)), softplus threshold 20 as in torch), 2 exact GELU
__global__ void k_small_linear(const float* __restrict__ x, const float* __restrict__ w,
                               const float* __restrict__ bias, float* __restrict__ y, int Bs, int K, int N,
                               long long w_pitch, int act) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) / 32;
  const int lane = threadIdx.x % 32;
  if (warp >= N) return;
  const float* wr = w + (size_t)warp * w_pitch;
  for (int bs = 0; bs < Bs; ++bs) {
    const float* xr = x + (size_t)bs * K;
    float acc = 0.f;
    for (int k = lane; k < K; k += 32) acc = fmaf(xr[k], wr[k], acc);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    if (lane == 0) {
      float v = acc + (bias ? bias[warp] : 0.f);
      if (act == 1) {
        const float sp = v > 20.f ? v : log1pf(expf(v));
        v = v * tanhf(sp);
      } else if (act == 2) {
        v = fd_gelu(v);
      }
      y[(size_t)bs * N + warp] = v;
    }
  }
}

// gate bias tables: one warp per (l, bs, n); d laid out [Bs][L][C]
__global__ void k_gate_bias(const float* __restrict__ d, const float* __restrict__ w1p,
                            const float* __restrict__ bias_sum, float* __restrict__ gb_full,
                            float* __restrict__ gb_lo, float* __restrict__ gb_hi, int L, int Bs, int C, int KT) {
  const long long warp = (blockIdx.x * (long long)blockDim.x + threadIdx.x) / 32;
  const int lane = threadIdx.x % 32;
  const int N = 2 * C;
  if (warp >= (long long)L * Bs * N) return;
  const int n = warp % N;
  const int bs = (warp / N) % Bs;
  const int l = warp / ((long long)N * Bs);
  const float* wr = w1p + ((size_t)l * N + n) * KT;
  const float* dr = d + ((size_t)bs * L + l) * C;
  float a0 = 0.f, a1 = 0.f, a2 = 0.f;
  for (int c = lane; c < C; c += 32) {
    const float dv = dr[c];
    a0 = fmaf(wr[c], dv, a0);
    a1 = fmaf(wr[C + c], dv, a1);
    a2 = fmaf(wr[2 * C + c], dv, a2);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    a0 += __shfl_xor_sync(0xffffffffu, a0, o);
    a1 += __shfl_xor_sync(0xffffffffu, a1, o);
    a2 += __shfl_xor_sync(0xffffffffu, a2, o);
  }
  if (lane == 0) {
    const size_t o = ((size_t)l * Bs + bs) * N + n;
    gb_full[o] = bias_sum[(size_t)l * N + n] + ((a0 + a2) + a1);
    gb_lo[o] = a0;
    gb_hi[o] = a2;
  }
}

// ---------------------------------------------------------------------------------- sampler kernels
__global__ void k_ddpm_step(const float* __restrict__ x, const float* __restrict__ eps,
                            const float* __restrict__ noise, float* __restrict__ x_out,
                            uint16_t* __restrict__ x_planes, long long n, float c_recip, float c_recipm1, float c1,
                            float c2, float sigma, float clip_min, float clip_max, unsigned long long seed,
                            unsigned long long offset, unsigned long long subseq0, int prec) {
  const long long n4 = n / 4;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n4;
       i += (long long)gridDim.x * blockDim.x) {
    const long long e = i * 4;
    float xv[4], ev[4], nz[4];
    fd_load_f32<4>(x + e, xv);
    fd_load_f32<4>(eps + e, ev);
    if (noise != nullptr) {
      fd_load_f32<4>(noise + e, nz);
    } else if (sigma != 0.f) {
      curandStatePhilox4_32_10_t st;
      curand_init(seed, subseq0 + (unsigned long long)i, offset, &st);
      const float4 g = curand_normal4(&st);
      nz[0] = g.x; nz[1] = g.y; nz[2] = g.z; nz[3] = g.w;
    } else {
      nz[0] = nz[1] = nz[2] = nz[3] = 0.f;
    }
    float o[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      float x0 = c_recip * xv[k] - c_recipm1 * ev[k];
      x0 = fminf(fmaxf(x0, clip_min), clip_max);
      const float mean = c1 * x0 + c2 * xv[k];
      o[k] = mean + sigma * nz[k];
    }
    fd_store_f32<4>(x_out + e, o);
    if (x_planes != nullptr) fd_store_planes<4>(x_planes, (size_t)n, (size_t)e, o, prec);
  }
}

struct LincombArgs {
  const float* in[6];
  float coef[6];
  int nterms;
};
__global__ void k_lincomb(float* __restrict__ out, uint16_t* __restrict__ out_planes, LincombArgs a, long long n,
                          int prec) {
  const long long n4 = n / 4;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n4;
       i += (long long)gridDim.x * blockDim.x) {
    const long long e = i * 4;
    float acc[4] = {0.f, 0.f, 0.f, 0.f};
    for (int t = 0; t < a.nterms; ++t) {
      float v[4];
      fd_load_f32<4>(a.in[t] + e, v);
#pragma unroll
      for (int k = 0; k < 4; ++k) acc[k] = t == 0 ? a.coef[0] * v[k] : fmaf(a.coef[t], v[k], acc[k]);
    }
    if (out != nullptr) fd_store_f32<4>(out + e, acc);
    if (out_planes != nullptr) fd_store_planes<4>(out_planes, (size_t)n, (size_t)e, acc, prec);
  }
}

__global__ void k_affine_cl(const float* __restrict__ x, float* __restrict__ y, const float* __restrict__ scale,
                            const float* __restrict__ shift, int nparam, long long n, int C) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n;
       i += (long long)gridDim.x * blockDim.x) {
    const int c = nparam == 1 ? 0 : (int)(i % C);
    y[i] = x[i] * scale[c] + shift[c];
  }
}

__global__ void k_q_sample(const float* __restrict__ x, const float* __restrict__ noise, const float* __restrict__ a,
                           const float* __restrict__ s, float* __restrict__ y, long long n, long long per_item) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n;
       i += (long long)gridDim.x * blockDim.x) {
    const long long b = i / per_item;
    y[i] = a[b] * x[i] + s[b] * noise[i];
  }
}

__global__ void k_randn(float* __restrict__ out, long long n, unsigned long long seed, unsigned long long offset,
                        unsigned long long subseq0) {
  const long long n4 = (n + 3) / 4;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n4;
       i += (long long)gridDim.x * blockDim.x) {
    curandStatePhilox4_32_10_t st;
    curand_init(seed, subseq0 + (unsigned long long)i, offset, &st);
    const float4 g = curand_normal4(&st);
    const float v[4] = {g.x, g.y, g.z, g.w};
    for (int k = 0; k < 4; ++k)
      if (i * 4 + k < n) out[i * 4 + k] = v[k];
  }
}

__global__ void k_log_clamp(const float* __restrict__ x, float* __restrict__ y, long long n, float clip,
                            float out_scale) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n;
       i += (long long)gridDim.x * blockDim.x)
    y[i] = logf(fmaxf(x[i], clip)) * out_scale;
}

inline int grid_for(long long work, int block = 256, int cap = 132 * 16) {
  long long g = (work + block - 1) / block;
  if (g < 1) g = 1;
  if (g > cap) g = cap;
  return (int)g;
}

}  // namespace

int fd_small_linear(const float* x, const float* w, const float* bias, float* y, int Bs, int K, int N, long long w_pitch,
                    int act, cudaStream_t st) {
  k_small_linear<<<(unsigned)(((long long)N * 32 + 255) / 256), 256, 0, st>>>(x, w, bias, y, Bs, K, N, w_pitch, act);
  FD_LAUNCHED();
  return 0;
}

int fd_step_mlp(const float* steps, const float* w0, const float* b0, const float* w1, const float* b1, float* s_out,
                float* ws, int Bs, int C, int H, int act, cudaStream_t st) {
  FD_REQUIRE(C % 2 == 0 && C >= 4 && H > 0, "step mlp: bad C=%d H=%d", C, H);
  float* emb = ws;                 // [Bs][C]
  float* h = ws + (size_t)Bs * C;  // [Bs][H]
  k_step_embed<<<grid_for((long long)Bs * C / 2), 256, 0, st>>>(steps, emb, Bs, C);
  FD_LAUNCHED();
  int rc = fd_small_linear(emb, w0, b0, h, Bs, C, H, C, act, st);
  if (rc) return rc;
  return fd_small_linear(h, w1, b1, s_out, Bs, H, C, H, 0, st);
}

extern "C" {

int fd_split_ncw(const float* src, const uint8_t* mask, uint16_t* planes, int B, int C, int T, int prec,
                 void* stream) {
  FD_DEVICE_GUARD();
  FD_REQUIRE(B > 0 && C > 0 && T > 0, "fd_split_ncw: bad shape B=%d C=%d T=%d", B, C, T);
  dim3 grid((T + 31) / 32, (C + 31) / 32, B), block(32, 8);
  k_split_ncw<<<grid, block, 0, (cudaStream_t)stream>>>(src, mask, planes, B, C, T, prec);
  FD_LAUNCHED();
  return 0;
}

int fd_split_nwc(const float* src, const uint8_t* mask, uint16_t* planes, int B, int T, int C, float scale,
                 int prec, void* stream) {
  FD_DEVICE_GUARD();
  FD_REQUIRE(C % 4 == 0, "fd_split_nwc: C=%d must be a multiple of 4", C);
  const long long rows = (long long)B * T;
  k_split_nwc<<<grid_for(rows * C / 4), 256, 0, (cudaStream_t)stream>>>(src, mask, planes, rows, C, scale, prec);
  FD_LAUNCHED();
  return 0;
}

int fd_mrf_finish(const uint16_t* const* in, int num, uint16_t* out, long long n, float in_slope, float scale,
                  float out_slope, int prec, void* stream) {
  FD_DEVICE_GUARD();
  FD_REQUIRE(num >= 1 && num <= 4 && n % 8 == 0 && in_slope > 0.f, "fd_mrf_finish: num=%d n=%lld in_slope=%g", num, n, in_slope);
  MrfIn m;
  for (int i = 0; i < 4; ++i) m.p[i] = i < num ? in[i] : nullptr;
  k_mrf_finish<<<grid_for(n / 8), 256, 0, (cudaStream_t)stream>>>(m, num, out, n, 1.f / in_slope, scale, out_slope, prec);
  FD_LAUNCHED();
  return 0;
}

int fd_transpose_nwc_to_ncw(const float* src, float* dst, int B, int T, int C, void* stream) {
  FD_DEVICE_GUARD();
  dim3 grid((C + 31) / 32, (T + 31) / 32, B), block(32, 8);
  k_transpose<<<grid, block, 0, (cudaStream_t)stream>>>(src, dst, T, C);
  FD_LAUNCHED();
  return 0;
}

int fd_transpose_ncw_to_nwc(const float* src, float* dst, int B, int C, int T, void* stream) {
  FD_DEVICE_GUARD();
  dim3 grid((T + 31) / 32, (C + 31) / 32, B), block(32, 8);
  k_transpose<<<grid, block, 0, (cudaStream_t)stream>>>(src, dst, C, T);
  FD_LAUNCHED();
  return 0;
}

int fd_pack_weight(const float* w, uint16_t* planes, long long n_elems, float scale, int prec, void* stream) {
  FD_DEVICE_GUARD();
  k_pack_weight<<<grid_for(n_elems), 256, 0, (cudaStream_t)stream>>>(w, planes, n_elems, scale, prec);
  FD_LAUNCHED();
  return 0;
}

int fd_wavenet_pack_layers(const float* const* conv_w, const float* const* cond_w, const float* const* out_w,
                           const float* scales, float* w1p_f32, uint16_t* w1, uint16_t* w2, uint16_t* w1t, uint16_t* wct,
                           uint16_t* w2t, int L, int C, int E, int gate_half, int prec, void* stream) {
  FD_DEVICE_GUARD();
  FD_REQUIRE(L > 0 && C > 0 && E > 0 && gate_half > 0 && C % gate_half == 0, "fd_wavenet_pack_layers: bad shape");
  FD_REQUIRE(conv_w && cond_w && out_w && scales && w1p_f32 && w1 && w2, "fd_wavenet_pack_layers: null pointer");
  FD_REQUIRE((w1t == nullptr) == (wct == nullptr) && (w1t == nullptr) == (w2t == nullptr),
             "fd_wavenet_pack_layers: the transposed packs come all or none");
  PackLayersArgs a{conv_w, cond_w, out_w, scales, w1p_f32, w1, w2, w1t, wct, w2t, L, C, E, gate_half, prec};
  cudaStream_t st = (cudaStream_t)stream;
  const int KT = 3 * C + E;
  k_pack_layers_w1<<<dim3((KT + 31) / 32, (2 * C + 31) / 32, L), dim3(32, 8), 0, st>>>(a);
  FD_LAUNCHED();
  k_pack_layers_w2<<<dim3((C + 31) / 32, (2 * C + 31) / 32, L), dim3(32, 8), 0, st>>>(a);
  FD_LAUNCHED();
  return 0;
}

int fd_wavenet_step_mlp(const float* steps, const float* w0, const float* b0, const float* w1, const float* b1,
                        float* s_out, float* ws, int Bs, int C, void* stream) {
  FD_DEVICE_GUARD();
  return fd_step_mlp(steps, w0, b0, w1, b1, s_out, ws, Bs, C, 4 * C, 1, (cudaStream_t)stream);
}

int fd_wavenet_gate_bias(const float* s, const float* wd, const float* bd, const float* w1p, const float* bias_sum,
                         float* gb_full, float* gb_lo, float* gb_hi, float* ws, int L, int Bs, int C, int KT,
                         void* stream) {
  FD_DEVICE_GUARD();
  cudaStream_t st = (cudaStream_t)stream;
  // d[bs][l][c] = Wd[l][c][:] . s[bs] + bd[l][c]
  int rc = fd_small_linear(s, wd, bd, ws, Bs, C, L * C, C, 0, st);
  if (rc) return rc;
  const long long warps = (long long)L * Bs * 2 * C;
  k_gate_bias<<<(unsigned)((warps * 32 + 255) / 256), 256, 0, st>>>(ws, w1p, bias_sum, gb_full, gb_lo, gb_hi, L, Bs,
                                                                   C, KT);
  FD_LAUNCHED();
  return 0;
}

int fd_wavenet_gate_bias_from_d(const float* d, const float* w1p, const float* bias_sum, float* gb_full, float* gb_lo,
                                float* gb_hi, int L, int Bs, int C, int KT, void* stream) {
  FD_DEVICE_GUARD();
  const long long warps = (long long)L * Bs * 2 * C;
  k_gate_bias<<<(unsigned)((warps * 32 + 255) / 256), 256, 0, (cudaStream_t)stream>>>(d, w1p, bias_sum, gb_full, gb_lo,
                                                                                       gb_hi, L, Bs, C, KT);
  FD_LAUNCHED();
  return 0;
}

int fd_ddpm_step(const float* x, const float* eps, const float* noise, float* x_out, uint16_t* x_planes,
                 long long n, float c_recip, float c_recipm1, float c1, float c2, float sigma, float clip_min,
                 float clip_max, unsigned long long seed, unsigned long long offset, unsigned long long subseq0,
                 int prec, void* stream) {
  FD_DEVICE_GUARD();
  FD_REQUIRE(n % 4 == 0, "fd_ddpm_step: n=%lld must be a multiple of 4", n);
  k_ddpm_step<<<grid_for(n / 4), 256, 0, (cudaStream_t)stream>>>(x, eps, noise, x_out, x_planes, n, c_recip,
                                                                  c_recipm1, c1, c2, sigma, clip_min, clip_max, seed,
                                                                  offset, subseq0, prec);
  FD_LAUNCHED();
  return 0;
}

int fd_lincomb(float* out, uint16_t* out_planes, const float* const* host_in_ptrs, const float* host_coefs,
               int nterms, long long n, int prec, void* stream) {
  FD_DEVICE_GUARD();
  FD_REQUIRE(nterms >= 1 && nterms <= 6, "fd_lincomb: nterms=%d out of range", nterms);
  FD_REQUIRE(n % 4 == 0, "fd_lincomb: n=%lld must be a multiple of 4", n);
  LincombArgs a;
  a.nterms = nterms;
  for (int i = 0; i < nterms; ++i) { a.in[i] = host_in_ptrs[i]; a.coef[i] = host_coefs[i]; }
  k_lincomb<<<grid_for(n / 4), 256, 0, (cudaStream_t)stream>>>(out, out_planes, a, n, prec);
  FD_LAUNCHED();
  return 0;
}

int fd_affine_cl(const float* x, float* y, const float* scale, const float* shift, int nparam, long long rows,
                 int C, void* stream) {
  FD_DEVICE_GUARD();
  FD_REQUIRE(nparam == 1 || nparam == C, "fd_affine_cl: nparam=%d must be 1 or C=%d", nparam, C);
  k_affine_cl<<<grid_for(rows * C), 256, 0, (cudaStream_t)stream>>>(x, y, scale, shift, nparam, rows * C, C);
  FD_LAUNCHED();
  return 0;
}

int fd_q_sample(const float* x, const float* noise, const float* a, const float* s, float* y, int B,
                long long per_item, void* stream) {
  FD_DEVICE_GUARD();
  k_q_sample<<<grid_for(B * per_item), 256, 0, (cudaStream_t)stream>>>(x, noise, a, s, y, B * per_item, per_item);
  FD_LAUNCHED();
  return 0;
}

int fd_randn(float* out, long long n, unsigned long long seed, unsigned long long offset, unsigned long long subseq0,
             void* stream) {
  FD_DEVICE_GUARD();
  k_randn<<<grid_for((n + 3) / 4), 256, 0, (cudaStream_t)stream>>>(out, n, seed, offset, subseq0);
  FD_LAUNCHED();
  return 0;
}

int fd_log_clamp(const float* x, float* y, long long n, float clip, float out_scale, void* stream) {
  FD_DEVICE_GUARD();
  k_log_clamp<<<grid_for(n), 256, 0, (cudaStream_t)stream>>>(x, y, n, clip, out_scale);
  FD_LAUNCHED();
  return 0;
}

}  // extern "C"
