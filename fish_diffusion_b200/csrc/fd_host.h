// host-side helpers shared by the translation units of libfishdiff_b200.so
#pragma once
#include <cuda_runtime.h>
#include "../../include/fishdiff_b200.h"

extern "C" void fd_set_error(const char* fmt, ...);
void fd_count_launch(int n);
// per-launch device timing (fd_prof_enable): event pair around a launch; kind indexes fd_prof_collect's arrays
void fd_prof_begin(int kind, cudaStream_t st);
void fd_prof_end(cudaStream_t st);

// call right after a kernel launch inside an `int`-returning API function
#define FD_LAUNCHED()                                                                          \
  do {                                                                                         \
    fd_count_launch(1);                                                                        \
    cudaError_t _e = cudaGetLastError();                                                       \
    if (_e != cudaSuccess) {                                                                   \
      fd_set_error("%s:%d kernel launch failed: %s", __FILE__, __LINE__, cudaGetErrorString(_e)); \
      return -1;                                                                               \
    }                                                                                          \
  } while (0)

// ---- device handling.  The binding names the device its tensors live on (fd_set_device, thread-local); every entry
// point opens with FD_DEVICE_GUARD(), which makes that device current for the duration of the call and restores the
// caller's afterwards.  Per-device facts (SM count, max-dynamic-smem attribute of a kernel) are cached per device.
struct FdDeviceGuard {
  int prev = -1;
  bool switched = false;
  FdDeviceGuard();
  ~FdDeviceGuard();
};
#define FD_DEVICE_GUARD() FdDeviceGuard _fd_device_guard
constexpr int FD_MAX_DEVICES = 64;
int fd_current_device();          // cudaGetDevice (clamped to [0, FD_MAX_DEVICES))
int fd_device_sms(int dev);       // multiprocessor count, cached

// the step-vector kernels of fd_aux.cu, shared by the WaveNet and ConvNext forwards:
//   y[bs][n] = act(w[n * w_pitch + :] . x[bs] + bias[n])  (act 0 none, 1 Mish, 2 exact GELU; bias may be NULL)
int fd_small_linear(const float* x, const float* w, const float* bias, float* y, int Bs, int K, int N, long long w_pitch,
                    int act, cudaStream_t st);
//   s_out[Bs][C] = w1 . act(w0 . DiffusionEmbedding(steps) + b0) + b1,  w0 [H][C], w1 [C][H]; ws: Bs * (C + H) floats
int fd_step_mlp(const float* steps, const float* w0, const float* b0, const float* w1, const float* b1, float* s_out,
                float* ws, int Bs, int C, int H, int act, cudaStream_t st);
