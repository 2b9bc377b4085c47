// common.cuh -- shared host/device helpers of libb200gan (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdarg.h>
#include "../../include/b200gan.h"

namespace b200gan {

// thread-local error text behind b200gan_last_error()
void set_error(const char *fmt, ...);

#define B2_CHECK_ARG(cond, ...)                  \
  do {                                           \
    if (!(cond)) {                               \
      ::b200gan::set_error(__VA_ARGS__);         \
      return B200GAN_E_BAD_ARG;                  \
    }                                            \
  } while (0)

#define B2_UNSUPPORTED(...)                      \
  do {                                           \
    ::b200gan::set_error(__VA_ARGS__);           \
    return B200GAN_E_UNSUPPORTED;                \
  } while (0)

#define B2_CUDA(expr)                                                              \
  do {                                                                             \
    cudaError_t _e = (expr);                                                       \
    if (_e != cudaSuccess) {                                                       \
      ::b200gan::set_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), \
                           __FILE__, __LINE__);                                    \
      return B200GAN_E_CUDA;                                                       \
    }                                                                              \
  } while (0)

#define B2_LAUNCH_CHECK() B2_CUDA(cudaPeekAtLastError())

static inline cudaStream_t as_stream(void *s) { return reinterpret_cast<cudaStream_t>(s); }
static inline int64_t ceil_div64(int64_t a, int64_t b) { return (a + b - 1) / b; }
static inline int ceil_div(int a, int b) { return (a + b - 1) / b; }

// SMs of the current device (queried once per device ordinal): grid sizes, split counts and the tile-width choices are
// planned for it.  Host-only planning queries without a usable device assume the 132 SMs of an H100 SXM.
int num_sms();

// geometry checks shared by every conv entry point (fills nothing; validates P/Q)
int validate_geom(const b200gan_conv_geom *g);

// ---- device helpers ---------------------------------------------------------------------
// if-chains, not `switch`: a switch in an unrolled loop is lowered to one indirect branch (BRX) per element
__device__ __forceinline__ float apply_act(float v, int act, float slope) {
  if (act == B200GAN_ACT_NONE) return v;
  if (act == B200GAN_ACT_LRELU) return v > 0.f ? v : v * slope;
  if (act == B200GAN_ACT_RELU) return fmaxf(v, 0.f);
  if (act == B200GAN_ACT_TANH) return tanhf(v);
  return 1.f / (1.f + expf(-v));
}
// derivative of the activation expressed through its OUTPUT y
__device__ __forceinline__ float act_grad_from_out(float y, int act, float slope) {
  if (act == B200GAN_ACT_NONE) return 1.f;
  if (act == B200GAN_ACT_LRELU) return y > 0.f ? 1.f : slope;
  if (act == B200GAN_ACT_RELU) return y > 0.f ? 1.f : 0.f;
  if (act == B200GAN_ACT_TANH) return 1.f - y * y;
  return y * (1.f - y);
}
// round-to-nearest fp32 -> tf32 (10-bit mantissa), result kept in an fp32 container
__device__ __forceinline__ float round_tf32(float v) {
  uint32_t r;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(v));
  return __uint_as_float(r);
}
// reflection of index i into [0, n) (torch ReflectionPad2d: edge pixel not repeated)
__device__ __forceinline__ int reflect_idx(int i, int n) {
  if (i < 0) i = -i;
  if (i >= n) i = 2 * (n - 1) - i;
  return i;
}

}  // namespace b200gan
