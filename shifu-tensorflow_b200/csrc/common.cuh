// Shared host/device helpers: error plumbing, activation table, small math.
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <stdint.h>
#include <stdio.h>
#include <string>
#include <type_traits>
#include <utility>

#include "../../include/shifu_b200.h"

namespace sb {

// ---- thread-local last error (sb_last_error) ----
std::string& last_error_ref();
int set_error(int code, const char* fmt, ...);

#define SB_CUDA(call)                                                                                       \
  do {                                                                                                      \
    cudaError_t _e = (call);                                                                                \
    if (_e != cudaSuccess)                                                                                  \
      return ::sb::set_error(SB_ERR_CUDA, "%s failed: %s (%s:%d)", #call, cudaGetErrorString(_e), __FILE__, \
                             __LINE__);                                                                     \
  } while (0)

#define SB_CHECK(cond, code, ...)                          \
  do {                                                     \
    if (!(cond)) return ::sb::set_error(code, __VA_ARGS__); \
  } while (0)

#define SB_TRY(expr)          \
  do {                        \
    int _s = (expr);          \
    if (_s != SB_OK) return _s; \
  } while (0)

// A device allocation of n T that is freed when its owner goes out of scope
template <typename T>
struct DevBuf {
  T* p = nullptr;
  DevBuf() = default;
  DevBuf(const DevBuf&) = delete;
  DevBuf& operator=(const DevBuf&) = delete;
  DevBuf(DevBuf&& o) noexcept : p(o.p) { o.p = nullptr; }
  DevBuf& operator=(DevBuf&& o) noexcept { std::swap(p, o.p); return *this; }
  ~DevBuf() { if (p) cudaFree(p); }
  int alloc(size_t n) {
    SB_CHECK(p == nullptr, SB_ERR_STATE, "DevBuf allocated twice");
    void* q = nullptr;
    SB_CUDA(cudaMalloc(&q, n * sizeof(T)));
    p = static_cast<T*>(q);
    return SB_OK;
  }
};

inline int round_up(int x, int m) { return (x + m - 1) / m * m; }
inline int64_t ceil_div64(int64_t a, int64_t b) { return (a + b - 1) / b; }

// cudaLaunchKernelEx with the optional programmatic-stream-serialization (PDL) attribute
template <typename... KArgs, typename... Args>
int launch_kernel(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, bool pdl, Args... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = st;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  at[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = at; cfg.numAttrs = pdl ? 1 : 0;
  SB_CUDA(cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...));
  return SB_OK;
}

// opt a kernel in to more than 48 KB of dynamic shared memory (once per process, outside of stream capture)
template <typename... KArgs>
int set_max_smem(void (*kernel)(KArgs...), int bytes) {
  SB_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes));
  return SB_OK;
}

// f(std::integral_constant<int, act>()): calls the instantiation of f for a run-time activation
template <typename F>
int with_act(int act, F&& f) {
  switch (act) {
    case SB_ACT_SIGMOID: return f(std::integral_constant<int, SB_ACT_SIGMOID>());
    case SB_ACT_TANH: return f(std::integral_constant<int, SB_ACT_TANH>());
    case SB_ACT_RELU: return f(std::integral_constant<int, SB_ACT_RELU>());
    case SB_ACT_LEAKYRELU: return f(std::integral_constant<int, SB_ACT_LEAKYRELU>());
    default: return f(std::integral_constant<int, SB_ACT_NONE>());
  }
}

// ---- activations (get_activation_fun, res/ssgd_monitor.py:74-88; tf.nn.leaky_relu alpha = 0.2) ----
#define SB_LEAKY_ALPHA 0.2f

__device__ __forceinline__ float sigmoidf_stable(float z) {
  // same two-branch form as the oracle; expf (not __expf) to stay within 1e-6 of fp32 libm
  if (z >= 0.f) return 1.f / (1.f + expf(-z));
  float e = expf(z);
  return e / (1.f + e);
}

__device__ __forceinline__ float act_apply(float z, int act) {
  switch (act) {
    case SB_ACT_SIGMOID: return sigmoidf_stable(z);
    case SB_ACT_TANH: return tanhf(z);
    case SB_ACT_RELU: return fmaxf(z, 0.f);
    case SB_ACT_LEAKYRELU: return z > 0.f ? z : z * SB_LEAKY_ALPHA;
    default: return z;  // SB_ACT_NONE
  }
}
// d act/dz written in terms of the activation OUTPUT a (TF's SigmoidGrad/TanhGrad/ReluGrad convention)
__device__ __forceinline__ float act_grad_from_out(float a, int act) {
  switch (act) {
    case SB_ACT_SIGMOID: return a * (1.f - a);
    case SB_ACT_TANH: return 1.f - a * a;
    case SB_ACT_RELU: return a > 0.f ? 1.f : 0.f;
    case SB_ACT_LEAKYRELU: return a > 0.f ? 1.f : SB_LEAKY_ALPHA;
    default: return 1.f;
  }
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// Column sums of a 32(lanes = rows) x 32(registers = columns) fp32 fragment.
// On return lane j holds sum over the 32 rows of column j.  31 shuffles instead of 160.
__device__ __forceinline__ float warp_colsum_32x32(float (&v)[32], int lane) {
#pragma unroll
  for (int half = 16; half >= 1; half >>= 1) {
    const bool upper = (lane & half) != 0;
#pragma unroll
    for (int i = 0; i < half; ++i) {
      float send = upper ? v[i] : v[i + half];
      float keep = upper ? v[i + half] : v[i];
      v[i] = keep + __shfl_xor_sync(0xffffffffu, send, half);
    }
  }
  return v[0];
}

// Sums of N_ column values over the 8 row groups of a warp (lane bits 2..4) of a wgmma accumulator fragment.  Every round
// sends half of the values that are still open to the partner lane and keeps the other half, so on return lane l holds
// the complete sums of the N_ / 8 values q N_ / 8 .. q N_ / 8 + N_ / 8 - 1, q = l / 4, in v[0 .. N_ / 8 - 1].
template <int LEN, int N_>
__device__ __forceinline__ void colsum_halve(float (&v)[N_], int lane, int m) {   // one round: v[0 .. 2 LEN) -> v[0 .. LEN)
  const bool upper = (lane & m) != 0;
#pragma unroll
  for (int i = 0; i < LEN; ++i) {
    const float send = upper ? v[i] : v[i + LEN];
    const float keep = upper ? v[i + LEN] : v[i];
    v[i] = keep + __shfl_xor_sync(0xffffffffu, send, m);
  }
}
template <int N_>
__device__ __forceinline__ void colsum_row_groups(float (&v)[N_], int lane) {
  static_assert(N_ % 8 == 0, "three halving rounds");
  colsum_halve<N_ / 2>(v, lane, 16);
  colsum_halve<N_ / 4>(v, lane, 8);
  colsum_halve<N_ / 8>(v, lane, 4);
}

}  // namespace sb
