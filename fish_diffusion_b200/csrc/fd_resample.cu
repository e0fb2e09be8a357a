// fd_resample.cu -- band-limited rational sample-rate conversion, fp32 [B][n_in] -> fp32 [B][n_out].
//
// Replaces librosa.resample on the host (reference nsf_hifigan.py:96, tools/diffusion/flask_api.py:42,53,
// modules/feature_extractors/base.py:25).  With O input and P output samples per common period, output q*P + p is
//     sum_i bank[i][p] * x[q*O - W + first[p] + i],   i in [0, count[p]),   x = 0 outside [0, len_b):
// bank[i][p] is tap first[p] + i of phase p, the zero tails of each phase's 2W + O taps are not stored.
// The filter bank is an argument (host-built, fish_diffusion_b200/mel.py); the kernel does not know the window.
//
// A CTA owns one item and RS_F consecutive periods.  It stages their F*O + 2W input samples in shared memory (16-byte
// loads where the whole vector lies inside the item, zero fill elsewhere), then each thread takes (phase, group of
// RS_R periods) tasks: every tap is loaded once through the read-only path and used for RS_R outputs from registers.
// The bank itself (up to ~240 KB at 44.1 k -> 16 k) stays in L1/L2.  Consecutive tasks are consecutive phases, so a
// warp reads one line of the tap-major bank per tap and the stores of one period are contiguous.  No atomics, no workspace; the sum runs in tap order, so an item's result does
// not depend on the batch it is in.
#include "fd_common.cuh"
#include "fd_host.h"

namespace {

constexpr int RS_THREADS = 256;
constexpr int RS_R = 4;                      // periods per task (accumulators per thread)
constexpr int RS_STAGE = 8192;               // target staged samples per CTA (32 KB)
constexpr int RS_SMEM_MAX = 48 * 1024;       // static limit of dynamic shared memory without an opt-in attribute

__host__ __device__ inline long long rs_out_len(long long n_in, long long O, long long P) { return (n_in * P + O - 1) / O; }

__global__ void __launch_bounds__(RS_THREADS)
k_resample(const float* __restrict__ wav, const long long* __restrict__ lens, float* __restrict__ out,
           const float* __restrict__ bank, const int* __restrict__ first, const int* __restrict__ count, long long n_in,
           long long n_out, int O, int P, int W, int F) {
  extern __shared__ __align__(16) float s_x[];
  const int b = blockIdx.y;
  const long long q0 = (long long)blockIdx.x * F;
  long long len = lens ? lens[b] : n_in;
  len = len < 0 ? 0 : (len > n_in ? n_in : len);
  const long long len_out = rs_out_len(len, O, P);
  float* __restrict__ o = out + (long long)b * n_out;
  const long long n_lo = q0 * P;
  long long n_hi = n_lo + (long long)F * P;
  if (n_hi > n_out) n_hi = n_out;
  if (n_lo >= len_out) {                     // the whole tile lies past the item's output: zeros, nothing to stage
    for (long long n = n_lo + threadIdx.x; n < n_hi; n += RS_THREADS) o[n] = 0.f;
    return;
  }

  // ---- stage x[q0*O - W, q0*O - W + F*O + 2W) at s_x[sh ...]; a0 is the 16-byte-aligned element at or below its start
  const long long item0 = (long long)b * n_in;           // element index of x[0] in wav
  const long long start = item0 + q0 * O - W;            // may be negative for the first tile of item 0
  const long long a0 = start & ~3LL;                     // floor to a multiple of 4 (two's complement)
  const int sh = (int)(start - a0);
  const int nstage = F * O + 2 * W + sh;
  const long long v_lo = item0, v_hi = item0 + len;      // valid element range of this item
  for (int i = threadIdx.x * 4; i < nstage; i += RS_THREADS * 4) {
    const long long a = a0 + i;
    float4 v;
    if (a >= v_lo && a + 4 <= v_hi) {
      v = __ldg(reinterpret_cast<const float4*>(wav + a));
    } else {
      v.x = (a >= v_lo && a < v_hi) ? __ldg(wav + a) : 0.f;
      v.y = (a + 1 >= v_lo && a + 1 < v_hi) ? __ldg(wav + a + 1) : 0.f;
      v.z = (a + 2 >= v_lo && a + 2 < v_hi) ? __ldg(wav + a + 2) : 0.f;
      v.w = (a + 3 >= v_lo && a + 3 < v_hi) ? __ldg(wav + a + 3) : 0.f;
    }
    *reinterpret_cast<float4*>(s_x + i) = v;
  }
  __syncthreads();

  const int ntask = P * (F / RS_R);
  for (int task = threadIdx.x; task < ntask; task += RS_THREADS) {
    const int p = task % P, rg = task / P;
    const int f = __ldg(first + p), c = __ldg(count + p);
    const float* __restrict__ h = bank + p;                 // tap-major: lanes (consecutive phases) read one line per tap
    const float* xs = s_x + sh + rg * RS_R * O + f;
    float acc[RS_R];
#pragma unroll
    for (int r = 0; r < RS_R; ++r) acc[r] = 0.f;
#pragma unroll 4
    for (int i = 0; i < c; ++i) {
      const float hv = __ldg(h + (long long)i * P);
#pragma unroll
      for (int r = 0; r < RS_R; ++r) acc[r] = fmaf(hv, xs[r * O + i], acc[r]);
    }
#pragma unroll
    for (int r = 0; r < RS_R; ++r) {
      const long long n = (q0 + rg * RS_R + r) * P + p;
      if (n < n_out) o[n] = n < len_out ? acc[r] : 0.f;
    }
  }
}

long long rs_gcd(long long a, long long b) {
  while (b) { const long long t = a % b; a = b; b = t; }
  return a;
}

}  // namespace

extern "C" {

long long fd_resample_out_len(long long n_in, int sr_in, int sr_out) {
  if (n_in < 0 || sr_in < 1 || sr_out < 1) {
    fd_set_error("fd_resample_out_len: n_in=%lld, sr_in=%d, sr_out=%d must be non-negative / positive", n_in, sr_in, sr_out);
    return -2;
  }
  const long long g = rs_gcd(sr_in, sr_out);
  return rs_out_len(n_in, sr_in / g, sr_out / g);
}

int fd_resample_fwd(const float* wav, const long long* lens, float* out, const float* bank, const int* first,
                    const int* count, int B, long long n_in, long long n_out, int O, int P, int W, int taps, void* stream) {
  FD_DEVICE_GUARD();
  FD_REQUIRE(O >= 1 && P >= 1, "fd_resample_fwd: O=%d and P=%d must be positive", O, P);
  FD_REQUIRE(rs_gcd(O, P) == 1, "fd_resample_fwd: O=%d and P=%d must be coprime (divide the rates by their gcd)", O, P);
  FD_REQUIRE(W >= 0 && taps == 2 * W + O, "fd_resample_fwd: taps=%d must equal 2*W+O = %d", taps, 2 * W + O);
  FD_REQUIRE(B >= 0 && B <= 65535 && n_in >= 0, "fd_resample_fwd: B=%d (at most 65535) and n_in=%lld must not be negative",
             B, n_in);
  FD_REQUIRE(n_out == rs_out_len(n_in, O, P), "fd_resample_fwd: n_out=%lld, but ceil(n_in*P/O) = %lld", n_out,
             rs_out_len(n_in, O, P));
  FD_REQUIRE(wav && out && bank && first && count, "fd_resample_fwd: wav, out, bank, first and count must not be NULL");
  FD_REQUIRE(((uintptr_t)wav & 15) == 0, "fd_resample_fwd: wav must be 16-byte aligned");
  if (B == 0 || n_out == 0) return 0;
  int F = RS_STAGE / O / RS_R * RS_R;
  if (F < RS_R) F = RS_R;
  const long long periods = (n_out + P - 1) / P;
  if (F > periods) F = (int)((periods + RS_R - 1) / RS_R * RS_R);
  const long long smem = ((long long)F * O + 2LL * W + 3 + 3) / 4 * 4 * (long long)sizeof(float);
  FD_REQUIRE(smem <= RS_SMEM_MAX, "fd_resample_fwd: O=%d, W=%d need %lld bytes of shared memory per CTA (limit %d): O is too "
             "large", O, W, smem, RS_SMEM_MAX);
  const long long gx = (periods + F - 1) / F;
  FD_REQUIRE(gx <= 0x7fffffffLL, "fd_resample_fwd: n_out=%lld is too long", n_out);
  k_resample<<<dim3((unsigned)gx, (unsigned)B), RS_THREADS, (size_t)smem, (cudaStream_t)stream>>>(
      wav, lens, out, bank, first, count, n_in, n_out, O, P, W, F);
  FD_LAUNCHED();
  return 0;
}

}  // extern "C"
