// Shared helpers for the b200vc CUDA library (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <functional>

namespace b200vc {

// ---------------------------------------------------------------------------
// Error plumbing: every extern "C" entry returns 0 on success, <0 on failure
// and leaves a message retrievable through b200vc_last_error().
// ---------------------------------------------------------------------------
enum Status : int {
  kOk = 0,
  kErrInvalidArg = -1,
  kErrCuda = -2,
  kErrUnsupported = -3,
  kErrDriver = -4,
};

void set_last_error(const char* fmt, ...);

#define B200VC_CHECK_CUDA(expr)                                                  \
  do {                                                                           \
    cudaError_t _e = (expr);                                                     \
    if (_e != cudaSuccess) {                                                     \
      ::b200vc::set_last_error("%s:%d: %s failed: %s", __FILE__, __LINE__, #expr, \
                               cudaGetErrorString(_e));                          \
      return ::b200vc::kErrCuda;                                                 \
    }                                                                            \
  } while (0)

#define B200VC_REQUIRE(cond, ...)                        \
  do {                                                   \
    if (!(cond)) {                                       \
      ::b200vc::set_last_error(__VA_ARGS__);             \
      return ::b200vc::kErrInvalidArg;                   \
    }                                                    \
  } while (0)

#define B200VC_LAUNCH_CHECK()                                                    \
  do {                                                                           \
    cudaError_t _e = cudaGetLastError();                                         \
    if (_e != cudaSuccess) {                                                     \
      ::b200vc::set_last_error("%s:%d: kernel launch failed: %s", __FILE__,      \
                               __LINE__, cudaGetErrorString(_e));                \
      return ::b200vc::kErrCuda;                                                 \
    }                                                                            \
  } while (0)

// Launch counter (bench.py reports it as gpu_launches).
void count_launch(int n = 1);

// Launch-plan recording (b200vc_plan_* in b200vc.h): between b200vc_plan_begin and b200vc_plan_end every recordable entry
// point called on this thread is appended to the plan as a closure over its arguments instead of being launched;
// b200vc_plan_run replays the closures on a stream.  All pointer arguments of recordable entries are DEVICE pointers.
bool plan_recording();
void plan_push(std::function<int(void*)> step);
#define B200VC_RECORD(call)                                                          \
  do {                                                                               \
    if (::b200vc::plan_recording()) {                                                \
      ::b200vc::plan_push([=](void* stream) -> int { (void)stream; return call; });  \
      return ::b200vc::kOk;                                                          \
    }                                                                                \
  } while (0)

// ---------------------------------------------------------------------------
// Activation codes shared by all epilogues (also mirrored in _ffi.py).
// ---------------------------------------------------------------------------
enum Act : int {
  ACT_NONE = 0,
  ACT_RELU = 1,
  ACT_LRELU = 2,   // parameter = negative slope
  ACT_GELU = 3,    // exact erf GELU (torch default)
  ACT_TANH = 4,
  ACT_SIGMOID = 5,
  ACT_EXP = 6,
};

__device__ __forceinline__ float apply_act(float v, int act, float p) {
  switch (act) {
    case ACT_RELU: return fmaxf(v, 0.f);
    case ACT_LRELU: return v > 0.f ? v : v * p;
    case ACT_GELU: return 0.5f * v * (1.f + erff(v * 0.70710678118654752440f));
    case ACT_TANH: return tanhf(v);
    case ACT_SIGMOID: return 1.f / (1.f + expf(-v));
    case ACT_EXP: return expf(v);
    default: return v;
  }
}

// Round-to-nearest to TF32 precision (10-bit mantissa); the tensor core then sees exact operands.
__device__ __forceinline__ float round_tf32(float v) {
  uint32_t r;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(v));
  return __uint_as_float(r);
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

static inline int ceil_div(int a, int b) { return (a + b - 1) / b; }
static inline long long ceil_div_ll(long long a, long long b) { return (a + b - 1) / b; }

}  // namespace b200vc
