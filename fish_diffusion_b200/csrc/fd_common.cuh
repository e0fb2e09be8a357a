// fish-diffusion hot path, H100-native: shared device/host definitions.
//
// Storage format used by every GEMM-shaped kernel on the path ("split planes"):
//   an activation tensor of logical shape [B, T, C] (channels-last) is stored as two
//   16-bit planes  planes[2][B][T][C]  with  value = hi + lo,  hi = rn16(value),
//   lo = rn16(value - hi).  In FD_F16 mode that is a 22-bit mantissa (fp32-faithful for
//   |value| < 65504), in FD_BF16 mode a 16-bit mantissa with fp32 range.  The tensor-core
//   kernel multiplies  hi*hi + lo*hi + hi*lo  with fp32 accumulation (wgmma), the SIMT twin
//   multiplies (hi+lo)*(hi+lo) in fp32 FMA.  Same bytes per element as fp32.
#pragma once
#include <cuda_runtime.h>
#include <cuda_fp16.h>
#include <cuda_bf16.h>
#include <stdint.h>

#define FD_F16 0
#define FD_BF16 1
// flag or-ed into a `prec` argument of the GEMM entry points: multiply the hi planes only (one product)
#define FD_SINGLE 0x10

#define FD_MAX_SEG 16

// epilogue kinds
#define FD_EPI_LINEAR 0
#define FD_EPI_GATE 1
#define FD_EPI_RES_SKIP 2
#define FD_EPI_MAG 3
#define FD_EPI_GATE_BWD 4

// activation kinds (linear epilogue)
#define FD_ACT_NONE 0
#define FD_ACT_RELU 1
#define FD_ACT_LRELU 2
#define FD_ACT_GELU 3

struct FdSeg {
  int src;    // which source tensor (0/1)
  int shift;  // row (time) shift applied to the A operand: A row = t + shift (zero outside [0,T))
  int c_off;  // first channel of the source used by this segment
  int k_len;  // number of channels (K extent) of this segment; multiple of the K block
};

struct FdTapGemm {
  // ---- problem: D[b,t,n] = sum_seg sum_k src[seg.src][b, t+seg.shift, seg.c_off+k] * W[n, koff(seg)+k]
  int B, T;
  int n_total;   // output columns (rows of W)
  int k_total;   // sum of seg.k_len (row pitch of W)
  int num_seg;
  int prec;      // FD_F16 / FD_BF16
  int single;    // 1: one product over the hi planes (half-precision operands), 0: three split products
  FdSeg seg[FD_MAX_SEG];
  const uint16_t* src[2];   // split planes [2][B][T][src_C]
  int src_C[2];
  // element strides of the source views (row = time step, batch item, plane); the generic layout
  // [2][B][T][C] has rs = C, bs = T*C, ps = B*T*C.  Overlapping rows (rs < C) give framed views.
  long long src_rs[2], src_bs[2], src_ps[2];
  const uint16_t* w;        // split planes [2][n_total][k_total]
  float acc_scale;          // accumulators are multiplied by this (undoes power-of-two weight prescale)
  // K offset of the W operand (a multiple of 8): the K coordinate of W is  koff(seg) + k0 + w_kshift, which selects a
  // column block of a wider W (the skip half of W2^T in the last layer's dz GEMM)
  int w_kshift;
  int epi;

  // ---- FD_EPI_LINEAR:  y = acc*acc_scale + bias[n] + addend[b,t,n] + res[b,t,n];  y *= post_scale
  //      if out_f32:   v = accum ? out_f32 + y : y ;  out_f32 = v   (else v = y)
  //      if out_planes: planes = split(act(v * planes_scale)), act = none / relu / leaky-relu / exact GELU
  //      rows with row_mask[b,t] != 0 produce zeros.
  const float* bias;        // [n_total] or per item [B][n_total] with bias_bstride
  int bias_bstride;
  const float* addend;      // fp32 [B,T,n_total] or null
  const float* res_f32;     // fp32 [B,T,n_total] or null
  const uint16_t* res_planes;  // split planes [2][B][T][n_total] or null
  float res_scale;          // multiplies the res_planes term (gradient chains: dx_next / sqrt(2))
  float post_scale;
  float* out_f32;           // fp32 [B,T,n_total] or null
  int out_accum;
  uint16_t* out_planes;     // split planes [2][B][T][n_total] or null
  float planes_scale;
  int act;
  float act_slope;
  const uint8_t* row_mask;  // [B,T] or null

  // ---- FD_EPI_GATE (WaveNet GEMM1): column tile of width NT holds NT/2 gate columns followed by
  //      NT/2 filter columns for residual channels [tile*NT/2, (tile+1)*NT/2).
  //      y = acc*acc_scale + gbias_full[n] + addend[b,t,n] - (t<dil ? gbias_lo[n] : 0) - (t+dil>=T ? gbias_hi[n] : 0)
  //      z = sigmoid(y_gate) * tanh(y_filter)  -> out_planes [2][B][T][C]
  //      addend (or null): fp32 [B][T][n_total] in the packed column order of W1 -- the conditioner projection computed
  //      once per sampler call (fd_wavenet_cond_proj) when the GEMM runs the three tap segments only
  const float* gbias_full;  // [Bs][n_total]  (conv bias + cond bias + sum over 3 taps of W_tap.d)
  const float* gbias_lo;    // [Bs][n_total]  tap-0 (t-dil) contribution of the step vector
  const float* gbias_hi;    // [Bs][n_total]  tap-2 (t+dil) contribution
  int gbias_bstride;        // 0 => one step for the whole batch
  int dil;
  int gate_tile;            // NT (column tile the weights were packed for)

  // ---- FD_EPI_MAG (framed DFT): same column pairing as the gate epilogue (re | im per tile);
  //      out_planes[b,t,c] = split(sqrt(re^2 + im^2 + mag_eps) * mag_scale), channel count = C
  float mag_scale;
  float mag_eps;            // 1e-9 (pitch_adjustable_mel.py:85) or 0 (torchaudio Spectrogram(power=1), utils/audio.py:45)

  // ---- FD_EPI_RES_SKIP (WaveNet GEMM2): columns [0,C) residual, [C,2C) skip.
  //      x' = (x + y_res) / sqrt(2)  -> x planes updated in place
  //      skip: first_layer ? skip_f32 = y : skip_f32 += y ; last_layer: skip planes = split((skip_f32+y)*skip_scale)
  uint16_t* x_planes;       // [2][B][T][C] in/out
  uint16_t* x_out_planes;   // training: write the updated residual stream here instead of in place (or null)
  uint16_t* y_planes;       // training (GATE epilogue): pre-activations [2][B][T][2C] in packed column order (or null)
  float* skip_f32;          // [B,T,C]
  uint16_t* skip_planes;    // [2][B][T][C] (last layer only)
  float skip_scale;
  int first_layer, last_layer;
  int C;                    // residual channels

  // ---- FD_EPI_GATE_BWD (training): the accumulator is dz[b,t,c] (n_total = C columns); with the saved pre-activations
  //      y_planes [2][B][T][2C] (packed order, see FD_EPI_GATE) the epilogue writes the gradient of z = sigmoid(g) tanh(f)
  //      dy = (dz tanh(f) sg (1-sg) | dz sg (1-tanh(f)^2))  -> out_planes [2][B][T][2C] (packed order)
  //      and accumulates its column sums: cs[b][col] += cs_scale * sum_t dy,  cs_edge[0/1][b][col] += the same over the
  //      first / last `dil` steps of the item (bias gradient and rank-one step-vector term of dW1).  cs buffers are zeroed
  //      by the caller.
  float* cs;                // [B][2C] or null
  float* cs_edge;           // [2][B][2C] or null
  float cs_scale;
};

// Weight-gradient GEMM (fd_wgrad_cl), resolved by the entry point for both back ends:
//   part[s][r][c] = acc_scale * sum_{b in split s} sum_t ROW[b, t, r] * COL[b, t + shift(c), c]
// rows / columns are concatenated segments; segment g covers rows [row_start[g], row_start[g] + row_width[g]) and reads
// channels from row_coff[g] on of source row_src[g] (likewise for columns, plus a time shift).
#define FD_WGRAD_MAX_COL_SEG 8
struct FdWgradK {
  int B, T, R, Cc;
  int splits, items_per_split;
  int m_tiles, n_tiles;     // tile counts of the tensor-core kernel
  int num_row_seg, num_col_seg;
  int row_src[2], row_coff[2], row_start[2], row_width[2];
  int col_src[FD_WGRAD_MAX_COL_SEG], col_shift[FD_WGRAD_MAX_COL_SEG], col_coff[FD_WGRAD_MAX_COL_SEG],
      col_start[FD_WGRAD_MAX_COL_SEG], col_width[FD_WGRAD_MAX_COL_SEG];
  int row_C[2], col_C[2];
  float* part;
  float acc_scale;
};

// ------------------------------------------------------------------------------------------------
// split / combine
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ void fd_split(float v, int prec, uint16_t& hi, uint16_t& lo) {
  if (prec == FD_F16) {
    v = fminf(fmaxf(v, -65504.f), 65504.f);
    __half h = __float2half_rn(v);
    __half l = __float2half_rn(v - __half2float(h));
    hi = __half_as_ushort(h);
    lo = __half_as_ushort(l);
  } else {
    __nv_bfloat16 h = __float2bfloat16_rn(v);
    __nv_bfloat16 l = __float2bfloat16_rn(v - __bfloat162float(h));
    hi = __bfloat16_as_ushort(h);
    lo = __bfloat16_as_ushort(l);
  }
}

__device__ __forceinline__ float fd_h2f(uint16_t u, int prec) {
  if (prec == FD_F16) return __half2float(__ushort_as_half(u));
  return __uint_as_float(((uint32_t)u) << 16);
}

__device__ __forceinline__ float fd_combine(uint16_t hi, uint16_t lo, int prec) {
  return fd_h2f(hi, prec) + fd_h2f(lo, prec);
}

// two neighbouring channels from their plane words (low half-word -> a, high half-word -> b)
__device__ __forceinline__ void fd_combine2(uint32_t hi2, uint32_t lo2, int prec, float& a, float& b) {
  if (prec == FD_F16) {
    const float2 h = __half22float2(*reinterpret_cast<const __half2*>(&hi2));
    const float2 l = __half22float2(*reinterpret_cast<const __half2*>(&lo2));
    a = h.x + l.x; b = h.y + l.y;
  } else {
    a = __uint_as_float(hi2 << 16) + __uint_as_float(lo2 << 16);
    b = __uint_as_float(hi2 & 0xffff0000u) + __uint_as_float(lo2 & 0xffff0000u);
  }
}

// branch-free activation of the linear epilogue: slope = 1 (none), 0 (ReLU) or the LeakyReLU slope
__device__ __forceinline__ float fd_act(float w, float slope) { return fmaf(slope, fminf(w, 0.f), fmaxf(w, 0.f)); }

// exact GELU (torch's nn.GELU() / F.gelu default, approximate="none"): 0.5 x (1 + erf(x / sqrt 2)), erff, no tanh form
__device__ __forceinline__ float fd_gelu(float x) { return 0.5f * x * (1.f + erff(x * 0.70710678118654752440f)); }

// accurate-enough transcendental pieces (relative error ~1e-7; tanh.approx is 1e-3 and is NOT used)
__device__ __forceinline__ float fd_sigmoid(float x) { return __fdividef(1.f, 1.f + __expf(-x)); }
__device__ __forceinline__ float fd_tanh(float x) {
  // tanh(x) = 1 - 2/(1+exp(2x)); for tiny |x| use the odd series to keep relative accuracy
  float ax = fabsf(x);
  if (ax < 0.04f) { float x2 = x * x; return x * (1.f - x2 * (0.33333333f - 0.13333333f * x2)); }
  float e = __expf(2.f * ax);
  float r = 1.f - __fdividef(2.f, e + 1.f);
  return copysignf(r, x);
}

// backward of z = sigmoid(g) tanh(f) at one element: dz -> (dg, df); the GATE_BWD epilogue of both tap-GEMM kernels
__device__ __forceinline__ void fd_dgate(float dz, float g, float f, float& dg, float& df) {
  const float sg = fd_sigmoid(g), th = fd_tanh(f);
  dg = dz * th * sg * (1.f - sg);
  df = dz * sg * (1.f - th * th);
}

// ------------------------------------------------------------------------------------------------
// vector helpers: V consecutive channels (V = 4 or 8)
// ------------------------------------------------------------------------------------------------
// two neighbouring channels at once: ONE packed, saturating conversion per plane word (F2FP.SATFINITE.*.PACK_AB)
// instead of clamp + convert + pack per element.  a -> low half-word, b -> high half-word.  Bit-identical to fd_split
// for |v| <= 65504 (f16) / all finite v (bf16).
__device__ __forceinline__ void fd_split2(float a, float b, int prec, uint32_t& hi2, uint32_t& lo2) {
  if (prec == FD_F16) {
    asm("cvt.rn.satfinite.f16x2.f32 %0, %1, %2;" : "=r"(hi2) : "f"(b), "f"(a));
    const float2 hf = __half22float2(*reinterpret_cast<const __half2*>(&hi2));
    asm("cvt.rn.satfinite.f16x2.f32 %0, %1, %2;" : "=r"(lo2) : "f"(b - hf.y), "f"(a - hf.x));
  } else {
    asm("cvt.rn.satfinite.bf16x2.f32 %0, %1, %2;" : "=r"(hi2) : "f"(b), "f"(a));
    const float ha = __uint_as_float(hi2 << 16), hb = __uint_as_float(hi2 & 0xffff0000u);
    asm("cvt.rn.satfinite.bf16x2.f32 %0, %1, %2;" : "=r"(lo2) : "f"(b - hb), "f"(a - ha));
  }
}

template <int V>
__device__ __forceinline__ void fd_store_planes(uint16_t* planes, size_t plane_elems, size_t off,
                                                const float (&y)[V], int prec) {
  uint32_t hi[V / 2], lo[V / 2];
#pragma unroll
  for (int i = 0; i < V / 2; ++i) fd_split2(y[2 * i], y[2 * i + 1], prec, hi[i], lo[i]);
  if (V == 4) {
    *reinterpret_cast<uint2*>(planes + off) = make_uint2(hi[0], hi[1]);
    *reinterpret_cast<uint2*>(planes + plane_elems + off) = make_uint2(lo[0], lo[1]);
  } else {
    *reinterpret_cast<uint4*>(planes + off) = make_uint4(hi[0], hi[1], hi[2 % (V / 2)], hi[3 % (V / 2)]);
    *reinterpret_cast<uint4*>(planes + plane_elems + off) = make_uint4(lo[0], lo[1], lo[2 % (V / 2)], lo[3 % (V / 2)]);
  }
}

template <int V>
__device__ __forceinline__ void fd_load_planes(const uint16_t* planes, size_t plane_elems, size_t off,
                                               float (&y)[V], int prec) {
  uint32_t hi[4], lo[4];
  if (V == 4) {
    const uint2 a = *reinterpret_cast<const uint2*>(planes + off);
    const uint2 b = *reinterpret_cast<const uint2*>(planes + plane_elems + off);
    hi[0] = a.x; hi[1] = a.y; lo[0] = b.x; lo[1] = b.y;
  } else {
    const uint4 a = *reinterpret_cast<const uint4*>(planes + off);
    const uint4 b = *reinterpret_cast<const uint4*>(planes + plane_elems + off);
    hi[0] = a.x; hi[1] = a.y; hi[2] = a.z; hi[3] = a.w; lo[0] = b.x; lo[1] = b.y; lo[2] = b.z; lo[3] = b.w;
  }
#pragma unroll
  for (int i = 0; i < V / 2; ++i) fd_combine2(hi[i], lo[i], prec, y[2 * i], y[2 * i + 1]);
}

// hi plane only (single-product mode of the SIMT twin)
__device__ __forceinline__ void fd_load_hi8(const uint16_t* planes, size_t off, float (&y)[8], int prec) {
  const uint4 a = *reinterpret_cast<const uint4*>(planes + off);
  const uint32_t w[4] = {a.x, a.y, a.z, a.w};
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    y[2 * i] = fd_h2f((uint16_t)(w[i] & 0xffff), prec);
    y[2 * i + 1] = fd_h2f((uint16_t)(w[i] >> 16), prec);
  }
}

template <int V>
__device__ __forceinline__ void fd_load_f32(const float* p, float (&y)[V]) {
#pragma unroll
  for (int i = 0; i < V; i += 4) {
    float4 q = *reinterpret_cast<const float4*>(p + i);
    y[i] = q.x; y[i + 1] = q.y; y[i + 2] = q.z; y[i + 3] = q.w;
  }
}
template <int V>
__device__ __forceinline__ void fd_store_f32(float* p, const float (&y)[V]) {
#pragma unroll
  for (int i = 0; i < V; i += 4)
    *reinterpret_cast<float4*>(p + i) = make_float4(y[i], y[i + 1], y[i + 2], y[i + 3]);
}

// ------------------------------------------------------------------------------------------------
// Epilogues: one definition per kind, used by every tap-GEMM kernel (the wgmma kernels' wide and narrow column tiles
// and the SIMT twin).  A kernel maps its accumulators to a fragment of R rows x V consecutive columns of one item,
// loads the bias values of those columns its own way and passes them in; PREC is compile-time in the tensor-core
// kernel (-1: p.prec).
// ------------------------------------------------------------------------------------------------
// The rows of a fragment: time steps t0, t0 + dt, ..., t0 + (R - 1) dt of one item.  The first nrows lie inside the
// item and are stored; the loads of the others are clamped to its last step.  I is the type of the element offsets:
// 32-bit in the tensor-core kernel (its launch checks the output sizes), 64-bit in the SIMT twin.
template <typename I>
struct FdRows {
  I item;   // b * T
  int t0, dt, nrows;
  __device__ __forceinline__ I row(const FdTapGemm& p, int r) const { return item + (I)min(t0 + r * dt, p.T - 1); }
};

// packed column of gate channel c: column tiles of gate_tile hold gate_tile / 2 gates, then their filters
__device__ __forceinline__ int fd_gate_col(const FdTapGemm& p, int c) {
  const int half = p.gate_tile / 2;
  return (c / half) * p.gate_tile + c % half;
}

// LINEAR: columns [n, n + V) of the fragment's rows, `a` the raw accumulators.  All loads are issued before the
// first store.
//   y = (a*acc_scale + bias + (addend + res_f32 + res_scale*res_planes)) * post_scale;  y += out_f32 if out_accum;
//   rows with row_mask != 0 are zeros;  out_f32 = y,  out_planes = split(act(y * planes_scale)).
template <int R, int V, int PREC, typename I>
__device__ __forceinline__ void fd_epi_linear(const FdTapGemm& p, const FdRows<I>& rw, int n, float (&a)[R][V],
                                              const float (&bias)[V]) {
  const int prec = PREC < 0 ? p.prec : PREC;
  const size_t plane = (size_t)p.B * p.T * p.n_total;
  I off[R];
  float pre[R][V];
#pragma unroll
  for (int r = 0; r < R; ++r) {
    off[r] = rw.row(p, r) * (I)p.n_total + (I)n;
#pragma unroll
    for (int i = 0; i < V; ++i) pre[r][i] = 0.f;
  }
  if (p.addend != nullptr) {
#pragma unroll
    for (int r = 0; r < R; ++r) {
      float v[V];
      fd_load_f32<V>(p.addend + off[r], v);
#pragma unroll
      for (int i = 0; i < V; ++i) pre[r][i] += v[i];
    }
  }
  if (p.res_f32 != nullptr) {
#pragma unroll
    for (int r = 0; r < R; ++r) {
      float v[V];
      fd_load_f32<V>(p.res_f32 + off[r], v);
#pragma unroll
      for (int i = 0; i < V; ++i) pre[r][i] += v[i];
    }
  }
  if (p.res_planes != nullptr) {
#pragma unroll
    for (int r = 0; r < R; ++r) {
      float v[V];
      fd_load_planes<V>(p.res_planes, plane, off[r], v, prec);
#pragma unroll
      for (int i = 0; i < V; ++i) pre[r][i] += p.res_scale * v[i];
    }
  }
  uint32_t masked = 0;
  if (p.row_mask != nullptr) {
#pragma unroll
    for (int r = 0; r < R; ++r)
      if (p.row_mask[rw.row(p, r)] != 0) masked |= 1u << r;
  }
#pragma unroll
  for (int r = 0; r < R; ++r)
#pragma unroll
    for (int i = 0; i < V; ++i) a[r][i] = (a[r][i] * p.acc_scale + bias[i] + pre[r][i]) * p.post_scale;
  if (p.out_f32 != nullptr && p.out_accum) {
#pragma unroll
    for (int r = 0; r < R; ++r) {
      float v[V];
      fd_load_f32<V>(p.out_f32 + off[r], v);
#pragma unroll
      for (int i = 0; i < V; ++i) a[r][i] += v[i];
    }
  }
  const float slope = p.act == FD_ACT_NONE ? 1.f : p.act == FD_ACT_RELU ? 0.f : p.act_slope;
#pragma unroll
  for (int r = 0; r < R; ++r) {
    if (r >= rw.nrows) break;
    if ((masked >> r) & 1u) {
#pragma unroll
      for (int i = 0; i < V; ++i) a[r][i] = 0.f;
    }
    if (p.out_f32 != nullptr) fd_store_f32<V>(p.out_f32 + off[r], a[r]);
    if (p.out_planes != nullptr) {
      float v[V];
      if (p.act == FD_ACT_GELU) {   // uniform over the launch; the slope path below stays as it was
#pragma unroll
        for (int i = 0; i < V; ++i) v[i] = fd_gelu(a[r][i] * p.planes_scale);
      } else {
#pragma unroll
        for (int i = 0; i < V; ++i) v[i] = fd_act(a[r][i] * p.planes_scale, slope);
      }
      fd_store_planes<V>(p.out_planes, plane, off[r], v, prec);
    }
  }
}

// RES_SKIP (WaveNet GEMM2): packed columns [0, C) are the residual half, [C, 2C) the skip half; y = a*acc_scale + bias.
//   residual: x = (x + y) / sqrt(2) on the split planes (into x_out_planes if set); not in the last layer, whose
//   residual stream is not consumed;
//   skip: y += skip_f32 except in the first layer; the last layer writes split(y * skip_scale) to skip_planes, the
//   others y to skip_f32.
// is_res = n < C, passed in so that a kernel whose column tiles lie in one half can make it a warp-uniform branch.
template <int R, int V, int PREC, typename I>
__device__ __forceinline__ void fd_epi_res_skip(const FdTapGemm& p, const FdRows<I>& rw, int n, bool is_res,
                                                const float (&a)[R][V], const float (&bias)[V]) {
  const int prec = PREC < 0 ? p.prec : PREC;
  const size_t plane = (size_t)p.B * p.T * p.C;
  const I cn = (I)(is_res ? n : n - p.C);
  I off[R];
#pragma unroll
  for (int r = 0; r < R; ++r) off[r] = rw.row(p, r) * (I)p.C + cn;
  if (is_res) {
    if (p.last_layer) return;
    float x[R][V];
#pragma unroll
    for (int r = 0; r < R; ++r) fd_load_planes<V>(p.x_planes, plane, off[r], x[r], prec);
    uint16_t* const xo = p.x_out_planes != nullptr ? p.x_out_planes : p.x_planes;
#pragma unroll
    for (int r = 0; r < R; ++r) {
      if (r >= rw.nrows) break;
#pragma unroll
      for (int i = 0; i < V; ++i) x[r][i] = (x[r][i] + (a[r][i] * p.acc_scale + bias[i])) * 0.70710678118654752440f;
      fd_store_planes<V>(xo, plane, off[r], x[r], prec);
    }
  } else {
    float sk[R][V];
    if (!p.first_layer) {
#pragma unroll
      for (int r = 0; r < R; ++r) fd_load_f32<V>(p.skip_f32 + off[r], sk[r]);
    }
#pragma unroll
    for (int r = 0; r < R; ++r) {
      if (r >= rw.nrows) break;
      float y[V];
#pragma unroll
      for (int i = 0; i < V; ++i) {
        y[i] = a[r][i] * p.acc_scale + bias[i];
        if (!p.first_layer) y[i] += sk[r][i];
      }
      if (p.last_layer) {
#pragma unroll
        for (int i = 0; i < V; ++i) y[i] *= p.skip_scale;
        fd_store_planes<V>(p.skip_planes, plane, off[r], y, prec);
      } else {
        fd_store_f32<V>(p.skip_f32 + off[r], y);
      }
    }
  }
}

// GATE (WaveNet GEMM1) at time step t: g and f hold the raw accumulators of V gate columns and of their V filter
// columns and leave as the pre-activations
//   y = acc*acc_scale + bias + addend - [t < dil] lo - [t + dil >= T] hi;   z = sigmoid(y_gate) tanh(y_filter).
// bias, add, lo and hi hold the gate values in [0] and the filter values in [1]; add is read only where p.addend is
// set, lo and hi only where their condition holds.  The caller stores z (and y where training keeps it).
template <int V>
__device__ __forceinline__ void fd_epi_gate(const FdTapGemm& p, int t, float (&g)[V], float (&f)[V], float (&z)[V],
                                            const float (&bias)[2][V], const float (&add)[2][V],
                                            const float (&lo)[2][V], const float (&hi)[2][V]) {
#pragma unroll
  for (int i = 0; i < V; ++i) {
    g[i] = g[i] * p.acc_scale + bias[0][i];
    f[i] = f[i] * p.acc_scale + bias[1][i];
  }
  if (p.addend != nullptr) {
#pragma unroll
    for (int i = 0; i < V; ++i) { g[i] += add[0][i]; f[i] += add[1][i]; }
  }
  if (t < p.dil) {
#pragma unroll
    for (int i = 0; i < V; ++i) { g[i] -= lo[0][i]; f[i] -= lo[1][i]; }
  }
  if (t + p.dil >= p.T) {
#pragma unroll
    for (int i = 0; i < V; ++i) { g[i] -= hi[0][i]; f[i] -= hi[1][i]; }
  }
#pragma unroll
  for (int i = 0; i < V; ++i) z[i] = fd_sigmoid(g[i]) * fd_tanh(f[i]);
}

// GATE_BWD's column sums of dy over a lane's rows (gate columns in [0], filter columns in [1]): over all its rows, and
// over those among the first / last `dil` steps of the item
template <int V>
struct FdColSums {
  float all[2][V], lo[2][V], hi[2][V];
};

// GATE_BWD (training): the accumulators are dz at channels [n, n + V) (n_total = C).  With the saved pre-activations
// y_planes [2][B][T][2C] (packed order) the fragment's rows get dy = (dz tanh(f) sg (1-sg) | dz sg (1-tanh(f)^2)) in
// out_planes, and s (zero on entry) collects the column sums of dy.  All loads are issued before the first store.
template <int R, int V, int PREC, typename I>
__device__ __forceinline__ void fd_epi_gate_bwd(const FdTapGemm& p, const FdRows<I>& rw, int n, const float (&a)[R][V],
                                                FdColSums<V>& s) {
  const int prec = PREC < 0 ? p.prec : PREC;
  const int half = p.gate_tile / 2;
  const I w2 = 2 * (I)p.C, pg = (I)fd_gate_col(p, n);
  const size_t plane = (size_t)p.B * p.T * w2;
  I off[R];
  float g[R][V], f[R][V];
#pragma unroll
  for (int r = 0; r < R; ++r) {
    off[r] = rw.row(p, r) * w2 + pg;
    fd_load_planes<V>(p.y_planes, plane, off[r], g[r], prec);
    fd_load_planes<V>(p.y_planes, plane, off[r] + half, f[r], prec);
  }
  const bool sums = p.cs != nullptr || p.cs_edge != nullptr;
#pragma unroll
  for (int r = 0; r < R; ++r) {
    if (r >= rw.nrows) break;
    float dg[V], df[V];
#pragma unroll
    for (int i = 0; i < V; ++i) fd_dgate(a[r][i] * p.acc_scale, g[r][i], f[r][i], dg[i], df[i]);
    fd_store_planes<V>(p.out_planes, plane, off[r], dg, prec);
    fd_store_planes<V>(p.out_planes, plane, off[r] + half, df, prec);
    if (sums) {
      const int t = rw.t0 + r * rw.dt;
      const bool in_lo = t < p.dil, in_hi = t + p.dil >= p.T;
#pragma unroll
      for (int i = 0; i < V; ++i) {
        s.all[0][i] += dg[i]; s.all[1][i] += df[i];
        if (in_lo) { s.lo[0][i] += dg[i]; s.lo[1][i] += df[i]; }
        if (in_hi) { s.hi[0][i] += dg[i]; s.hi[1][i] += df[i]; }
      }
    }
  }
}

// GATE_BWD's column sums of item b, channels [n, n + V): the lanes lane ^ FIRST_XOR, lane ^ 2 FIRST_XOR, ... hold the
// same columns and are summed by an xor butterfly, then the lanes with `lead` add one atomic per column to cs and,
// where the warp's rows hold edge steps (warp-uniform edge_lo / edge_hi), to cs_edge.  Every lane of the warp calls it.
template <int FIRST_XOR, int V>
__device__ __forceinline__ void fd_gate_bwd_colsums(const FdTapGemm& p, FdColSums<V>& s, bool edge_lo, bool edge_hi,
                                                    bool lead, int b, int n) {
  if (p.cs == nullptr && p.cs_edge == nullptr) return;
  auto butterfly = [](float (&x)[2][V], int i) {
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
      for (int o = FIRST_XOR; o < 32; o *= 2) x[h][i] += __shfl_xor_sync(0xffffffffu, x[h][i], o);
  };
#pragma unroll
  for (int i = 0; i < V; ++i) {
    butterfly(s.all, i);
    if (edge_lo) butterfly(s.lo, i);
    if (edge_hi) butterfly(s.hi, i);
  }
  if (!lead) return;
  const int half = p.gate_tile / 2;
  const size_t w2 = 2 * (size_t)p.C, c = (size_t)b * w2 + fd_gate_col(p, n);
  if (p.cs != nullptr) {
#pragma unroll
    for (int i = 0; i < V; ++i) {
      atomicAdd(p.cs + c + i, s.all[0][i] * p.cs_scale);
      atomicAdd(p.cs + c + half + i, s.all[1][i] * p.cs_scale);
    }
  }
  if (p.cs_edge != nullptr && (edge_lo || edge_hi)) {
    float* const e0 = p.cs_edge + c;
    float* const e1 = e0 + (size_t)p.B * w2;
#pragma unroll
    for (int i = 0; i < V; ++i) {
      if (edge_lo) { atomicAdd(e0 + i, s.lo[0][i] * p.cs_scale); atomicAdd(e0 + half + i, s.lo[1][i] * p.cs_scale); }
      if (edge_hi) { atomicAdd(e1 + i, s.hi[0][i] * p.cs_scale); atomicAdd(e1 + half + i, s.hi[1][i] * p.cs_scale); }
    }
  }
}

// MAG (framed DFT): V real and V imaginary accumulators of row t, magnitudes of channels [zc0, zc0 + V)
template <int V, int PREC = -1>
__device__ __forceinline__ void fd_epi_mag(const FdTapGemm& p, int b, int t, int zc0,
                                           const float (&re)[V], const float (&im)[V]) {
  const int prec = PREC < 0 ? p.prec : PREC;   // compile-time in the tensor-core kernel
  float z[V];
#pragma unroll
  for (int i = 0; i < V; ++i) {
    const float r = re[i] * p.acc_scale, q = im[i] * p.acc_scale;
    z[i] = sqrtf(r * r + q * q + p.mag_eps) * p.mag_scale;
  }
  const size_t plane_elems = (size_t)p.B * p.T * p.C;
  const size_t off = ((size_t)b * p.T + t) * p.C + zc0;
  fd_store_planes<V>(p.out_planes, plane_elems, off, z, prec);
}

// ------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------
#ifdef __cplusplus
extern "C" {
#endif
void fd_set_error(const char* fmt, ...);
#ifdef __cplusplus
}
#endif

#define FD_CHECK_CUDA(expr)                                                                    \
  do {                                                                                         \
    cudaError_t _e = (expr);                                                                   \
    if (_e != cudaSuccess) {                                                                   \
      fd_set_error("%s:%d CUDA error %d (%s) in %s", __FILE__, __LINE__, (int)_e,              \
                   cudaGetErrorString(_e), #expr);                                             \
      return -1;                                                                               \
    }                                                                                          \
  } while (0)

#define FD_REQUIRE(cond, ...)                                                                  \
  do {                                                                                         \
    if (!(cond)) {                                                                             \
      fd_set_error(__VA_ARGS__);                                                               \
      return -2;                                                                               \
    }                                                                                          \
  } while (0)

int fd_tapgemm_simt_launch(const FdTapGemm& p, cudaStream_t stream);
int fd_tapgemm_tc_launch(const FdTapGemm& p, cudaStream_t stream);
int fd_tapgemm_tc_supported(const FdTapGemm& p);
int fd_wgrad_simt_launch(const FdWgradK& p, const uint16_t* const* row_ptr, const uint16_t* const* col_ptr, int prec,
                         cudaStream_t stream);
