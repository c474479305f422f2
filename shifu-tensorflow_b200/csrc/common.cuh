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

// element j (0..7) of 8 bf16 packed in a uint4, as fp32, from the words themselves (j a compile-time constant after
// unrolling): no byte view of the vector, so it stays in registers
__device__ __forceinline__ float bf16_of_u4(const uint4& v, int j) {
  const uint32_t w = (j >> 1) == 0 ? v.x : (j >> 1) == 1 ? v.y : (j >> 1) == 2 ? v.z : v.w;
  return __uint_as_float((j & 1) ? (w & 0xFFFF0000u) : (w << 16));
}

// ---- deterministic epilogues (DET = true instantiations, sb_trainer_set_deterministic) ----
// A reduction over the CTAs of a launch: each CTA stores its partial sums with plain stores into its own slots of the
// launch's workspace; the CTA that takes the last ticket adds the slots in ascending slot order and writes the result.
// The order of the adds is fixed by slot index, never by arrival.
//
// det_last_cta is called by the `nthreads` threads of the CTA that stored slots (named barrier `bar`; `leader` is one of
// them) after their slot stores.  It returns true in all of them in the last of the launch's `n_ctas` CTAs; that CTA has
// already put the ticket back to 0, so the next launch (or graph replay) needs no memset.
__device__ __forceinline__ bool det_last_cta(unsigned int* ticket, unsigned int n_ctas, int bar, int nthreads, bool leader) {
  __threadfence();   // this thread's slot stores are visible device-wide before the CTA takes its ticket
  asm volatile("bar.sync %0, %1;" ::"r"(bar), "r"(nthreads) : "memory");
  int mine = 0, last = 0;
  if (leader) mine = atomicAdd(ticket, 1u) == n_ctas - 1u ? 1 : 0;
  asm volatile(
      "{\n .reg .pred p, q;\n setp.ne.s32 p, %1, 0;\n bar.red.or.pred q, %2, %3, p;\n selp.s32 %0, 1, 0, q;\n}"
      : "=r"(last) : "r"(mine), "r"(bar), "r"(nthreads) : "memory");
  if (last) {
    if (leader) *ticket = 0u;   // every CTA of this launch has taken its ticket
    __threadfence();            // the other CTAs' slots are read after this (with ld.global.cg: not through L1)
  }
  return last != 0;
}

// det_last_cta + det_colsum_finish for the wgmma GEMMs' dA epilogues, called once after the tile loop.  Not inlined: the
// ordered sum's loop would otherwise be scheduled into a kernel whose registers the accumulator already fills.
static __device__ __noinline__ void det_colsum_tail(unsigned int* ticket, const float* slots, int n_slots, int N, float* dst, int bar,
                                             int nthreads, int tid);

// Ordered sum of column slots [n_slots][N] into dst[0, N) (dst[c] += sum over s of slots[s][c], s ascending)
__device__ __forceinline__ void det_colsum_finish(const float* slots, int n_slots, int N, float* dst, int tid, int nthreads) {
  for (int c = tid; c < N; c += nthreads) {
    float s = 0.f;
    for (int k = 0; k < n_slots; ++k) s += __ldcg(slots + static_cast<size_t>(k) * N + c);
    dst[c] += s;
  }
}

// Output layer's slots, per CTA: [loss sum, db_o, db_L[halves][H], dw_o[halves][H]] (halves = partial sums per column and
// CTA).  Ordered sum over CTAs, then halves, into the step scalar and the flat gradient; loss / bwd select the outputs.
__device__ __forceinline__ size_t det_out_stride(int H, int halves) { return 2 + 2 * static_cast<size_t>(halves) * H; }
__device__ __forceinline__ void det_out_finish(const float* ws, int n_ctas, int H, int halves, bool loss, bool bwd, float* loss_dst,
                                               float* g_bo, float* g_bL, float* g_wo, int tid, int nthreads) {
  const size_t stride = det_out_stride(H, halves);
  for (int j = tid; j < 2 + 2 * H; j += nthreads) {
    if (j == 0 ? !loss : !bwd) continue;
    size_t off;
    float* dst;
    int nh = halves;
    if (j < 2) { off = j; dst = j == 0 ? loss_dst : g_bo; nh = 1; }
    else if (j < 2 + H) { off = 2 + (j - 2); dst = g_bL + (j - 2); }
    else { off = 2 + static_cast<size_t>(halves) * H + (j - 2 - H); dst = g_wo + (j - 2 - H); }
    float s = 0.f;
    for (int b = 0; b < n_ctas; ++b)
      for (int h = 0; h < nh; ++h) s += __ldcg(ws + b * stride + off + static_cast<size_t>(h) * H);
    *dst += s;
  }
}

static __device__ __noinline__ void det_colsum_tail(unsigned int* ticket, const float* slots, int n_slots, int N, float* dst, int bar,
                                             int nthreads, int tid) {
  if (det_last_cta(ticket, gridDim.x, bar, nthreads, tid == 0)) det_colsum_finish(slots, n_slots, N, dst, tid, nthreads);
}

}  // namespace sb
