// Peer-memory link probe (2+ GPUs of one node): what the exchange kernels of csrc/xchg_p2p.cuh can expect from the fabric.
//   nvcc -O3 -gencode arch=compute_90a,code=sm_90a -o scripts/p2p_probe scripts/p2p_probe.cu && scripts/p2p_probe
// Prints: peer attributes, copy-engine bandwidth, SM-issued peer load / store bandwidth by grid size and bytes in flight,
// flag round trip (st.release.sys into the peer -> peer spins locally -> answers).
#include <cuda_runtime.h>
#include <cstdio>
#include <cstdlib>
#include <vector>

#define CK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { printf("CUDA error %s at %s:%d\n", cudaGetErrorString(e_), __FILE__, __LINE__); exit(1); } } while (0)

template <int U, bool SYS>
__global__ void __launch_bounds__(256) read_kernel(const float4* __restrict__ src, float4* __restrict__ sink, long long n4) {
  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
  const long long stride = static_cast<long long>(gridDim.x) * 256 * U;
  for (long long base = static_cast<long long>(blockIdx.x) * 256 * U + threadIdx.x; base < n4; base += stride) {
    float4 v[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const long long i = base + u * 256;
      if (i < n4) {
        if (SYS) asm volatile("ld.relaxed.sys.global.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v[u].x), "=f"(v[u].y), "=f"(v[u].z), "=f"(v[u].w) : "l"(src + i) : "memory");
        else v[u] = __ldg(src + i);
      } else v[u] = make_float4(0.f, 0.f, 0.f, 0.f);
    }
#pragma unroll
    for (int u = 0; u < U; ++u) { acc.x += v[u].x; acc.y += v[u].y; acc.z += v[u].z; acc.w += v[u].w; }
  }
  if (acc.x == 12345.f) sink[0] = acc;
}

template <int BYTES>
__global__ void __launch_bounds__(256) write_kernel(char* __restrict__ dst, long long nbytes) {
  const long long n = nbytes / BYTES;
  for (long long i = static_cast<long long>(blockIdx.x) * 256 + threadIdx.x; i < n; i += static_cast<long long>(gridDim.x) * 256) {
    if (BYTES == 16) reinterpret_cast<float4*>(dst)[i] = make_float4(1.f, 2.f, 3.f, 4.f);
    else reinterpret_cast<uint2*>(dst)[i] = make_uint2(1u, 2u);
  }
}

__device__ __forceinline__ unsigned long long gtime() { unsigned long long t; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t)); return t; }

// pinger (dev 0): for k = 1..n: store k into the peer's flag, wait until MY flag shows k.  ponger (dev 1): the mirror image.
__global__ void ping_kernel(unsigned int* peer_flag, unsigned int* my_flag, int n, unsigned long long* out_ns) {
  const unsigned long long t0 = gtime();
  for (int k = 1; k <= n; ++k) {
    asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(peer_flag), "r"(k) : "memory");
    unsigned int v;
    do { asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(my_flag) : "memory"); } while (static_cast<int>(v) < k);
  }
  *out_ns = gtime() - t0;
}
__global__ void pong_kernel(unsigned int* peer_flag, unsigned int* my_flag, int n) {
  for (int k = 1; k <= n; ++k) {
    unsigned int v;
    do { asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(my_flag) : "memory"); } while (static_cast<int>(v) < k);
    asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(peer_flag), "r"(k) : "memory");
  }
}
// the same round trip with the waiter POLLING THE PEER'S memory (what a pull-style flag would cost)
__global__ void ping_remote_poll_kernel(unsigned int* peer_word, unsigned int* my_word, int n, unsigned long long* out_ns) {
  const unsigned long long t0 = gtime();
  for (int k = 1; k <= n; ++k) {
    asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(my_word), "r"(k) : "memory");
    unsigned int v;
    do { asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(peer_word) : "memory"); } while (static_cast<int>(v) < k);
  }
  *out_ns = gtime() - t0;
}
__global__ void pong_remote_poll_kernel(unsigned int* peer_word, unsigned int* my_word, int n) {
  for (int k = 1; k <= n; ++k) {
    unsigned int v;
    do { asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(peer_word) : "memory"); } while (static_cast<int>(v) < k);
    asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(my_word), "r"(k) : "memory");
  }
}


int main() {
  int nd = 0;
  CK(cudaGetDeviceCount(&nd));
  printf("devices: %d\n", nd);
  if (nd < 2) { printf("need 2 devices\n"); return 0; }
  int can01 = 0, can10 = 0, rank = -1, atom = -1;
  CK(cudaDeviceCanAccessPeer(&can01, 0, 1));
  CK(cudaDeviceCanAccessPeer(&can10, 1, 0));
  cudaDeviceGetP2PAttribute(&rank, cudaDevP2PAttrPerformanceRank, 0, 1);
  cudaDeviceGetP2PAttribute(&atom, cudaDevP2PAttrNativeAtomicSupported, 0, 1);
  printf("canAccessPeer 0->1 %d 1->0 %d  performanceRank %d  nativeAtomics %d\n", can01, can10, rank, atom);
  CK(cudaSetDevice(0)); CK(cudaDeviceEnablePeerAccess(1, 0));
  CK(cudaSetDevice(1)); CK(cudaDeviceEnablePeerAccess(0, 0));
  const long long BIG = 256ll << 20;
  char *b0, *b1;
  CK(cudaSetDevice(0)); CK(cudaMalloc(&b0, BIG)); CK(cudaMemset(b0, 0, BIG));
  CK(cudaSetDevice(1)); CK(cudaMalloc(&b1, BIG)); CK(cudaMemset(b1, 0, BIG));
  CK(cudaDeviceSynchronize());
  CK(cudaSetDevice(0));
  cudaStream_t st; CK(cudaStreamCreate(&st));
  cudaEvent_t e0, e1; CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
  auto timed = [&](auto&& fn, int reps) {
    fn(); fn();
    CK(cudaStreamSynchronize(st));
    CK(cudaEventRecord(e0, st));
    for (int i = 0; i < reps; ++i) fn();
    CK(cudaEventRecord(e1, st));
    CK(cudaStreamSynchronize(st));
    float ms = 0; CK(cudaEventElapsedTime(&ms, e0, e1));
    return ms / reps;
  };
  const long long sizes[] = {1ll << 20, 4ll << 20, 16ll << 20, 256ll << 20};
  printf("\ncopy engine (cudaMemcpyPeerAsync 1 -> 0):\n");
  for (long long s : sizes) {
    const float ms = timed([&] { CK(cudaMemcpyPeerAsync(b0, 0, b1, 1, s, st)); }, 10);
    printf("  %6lld KB  %8.2f us  %7.1f GB/s\n", s >> 10, ms * 1e3, s / ms / 1e6);
  }
  const int grids[] = {37, 74, 148, 296, 592};
  printf("\nSM-issued peer LOADS (dev 0 reads dev 1), 256 threads, U float4 per thread in flight:\n");
  for (long long s : sizes) {
    for (int g : grids) {
      const long long n4 = s / 16;
      const float a = timed([&] { read_kernel<4, true><<<g, 256, 0, st>>>(reinterpret_cast<float4*>(b1), reinterpret_cast<float4*>(b0), n4); }, 10);
      const float b = timed([&] { read_kernel<8, true><<<g, 256, 0, st>>>(reinterpret_cast<float4*>(b1), reinterpret_cast<float4*>(b0), n4); }, 10);
      const float c = timed([&] { read_kernel<16, true><<<g, 256, 0, st>>>(reinterpret_cast<float4*>(b1), reinterpret_cast<float4*>(b0), n4); }, 10);
      const float d = timed([&] { read_kernel<8, false><<<g, 256, 0, st>>>(reinterpret_cast<float4*>(b1), reinterpret_cast<float4*>(b0), n4); }, 10);
      printf("  %6lld KB grid %3d  sys U=4 %7.2f us %6.1f GB/s | U=8 %7.2f us %6.1f GB/s | U=16 %7.2f us %6.1f GB/s | ldg U=8 %7.2f us %6.1f GB/s\n",
             s >> 10, g, a * 1e3, s / a / 1e6, b * 1e3, s / b / 1e6, c * 1e3, s / c / 1e6, d * 1e3, s / d / 1e6);
    }
  }
  printf("\nlocal loads for comparison (dev 0 reads dev 0):\n");
  for (long long s : sizes) {
    const long long n4 = s / 16;
    const float b = timed([&] { read_kernel<8, true><<<148, 256, 0, st>>>(reinterpret_cast<float4*>(b0), reinterpret_cast<float4*>(b0) + n4, n4 / 2); }, 10);
    printf("  %6lld KB grid 148 sys U=8 %7.2f us %6.1f GB/s\n", (s / 2) >> 10, b * 1e3, s / 2 / b / 1e6);
  }
  printf("\nSM-issued peer STORES (dev 0 writes dev 1):\n");
  for (long long s : sizes) {
    for (int g : grids) {
      const float a = timed([&] { write_kernel<16><<<g, 256, 0, st>>>(b1, s); }, 10);
      const float b = timed([&] { write_kernel<8><<<g, 256, 0, st>>>(b1, s); }, 10);
      printf("  %6lld KB grid %3d  16 B %7.2f us %6.1f GB/s | 8 B %7.2f us %6.1f GB/s\n", s >> 10, g, a * 1e3, s / a / 1e6, b * 1e3, s / b / 1e6);
    }
  }
  // flag round trips
  unsigned long long* out_ns;
  CK(cudaMallocHost(&out_ns, 8));
  cudaStream_t st1;
  CK(cudaSetDevice(1)); CK(cudaStreamCreate(&st1));
  unsigned int* f0 = reinterpret_cast<unsigned int*>(b0);
  unsigned int* f1 = reinterpret_cast<unsigned int*>(b1);
  const int n = 200;
  for (int mode = 0; mode < 2; ++mode) {
    CK(cudaSetDevice(0)); CK(cudaMemset(b0, 0, 256)); CK(cudaDeviceSynchronize());
    CK(cudaSetDevice(1)); CK(cudaMemset(b1, 0, 256)); CK(cudaDeviceSynchronize());
    if (mode == 0) {
      CK(cudaSetDevice(1)); pong_kernel<<<1, 1, 0, st1>>>(f0, f1, n);
      CK(cudaSetDevice(0)); ping_kernel<<<1, 1, 0, st>>>(f1, f0, n, out_ns);
    } else {
      CK(cudaSetDevice(1)); pong_remote_poll_kernel<<<1, 1, 0, st1>>>(f0, f1, n);
      CK(cudaSetDevice(0)); ping_remote_poll_kernel<<<1, 1, 0, st>>>(f1, f0, n, out_ns);
    }
    CK(cudaSetDevice(0)); CK(cudaStreamSynchronize(st));
    CK(cudaSetDevice(1)); CK(cudaStreamSynchronize(st1));
    printf("\nflag round trip (%s): %.2f us\n", mode == 0 ? "push: store into the peer, poll locally" : "pull: store locally, poll the peer's memory", *out_ns / 1e3 / n);
  }
  return 0;
}
