// fp32 CUDA-core GEMM with the same fused epilogues as gemm_tc.cuh - the SB_PREC_FP32 "parity mode":
// fp32 operands, fp32 FMA accumulation, i.e. the arithmetic TF-CPU performs for nn_layer
// (res/ssgd_monitor.py:57-71) and its gradients.  Generic strides, so no transposed copies are needed.
//   C(m,n) = sum_k A(m,k) * B(k,n),   A(m,k) = A[m*sAm + k*sAk],  B(k,n) = B[k*sBk + n*sBn]
#pragma once
#include "common.cuh"
#include "gemm_tc.cuh"  // EPI_* ids

namespace sb {

struct GemmF32Params {
  int M, N, K;
  const float* A; long long sAm, sAk;
  const float* B; long long sBk, sBn;
  int k_per_split;  // multiple of 16; gridDim.z splits
  const float* bias; int act;
  float* out; int ld_out;
  const float* aux; int ld_aux;
  float* colsum;
  float* accum; int ld_acc;
  const float* addend; int ld_add;   // EPI_FWD, nullable: added to the pre-activation (wide+deep: the embedding sum)
  float* det_ws; unsigned int* det_ticket;   // EPI_DA with DET: column-sum slots [row tile][N] and the launch's ticket
};

// DET (EPI_DA only): the column sums go to slot blockIdx.y (the row tile) and the last CTA adds the row tiles in order
template <int EPI, bool DET = false>
__global__ void __launch_bounds__(256)
gemm_f32_kernel(const GemmF32Params p) {
  static_assert(!DET || EPI == EPI_DA, "DET: dA column sums only");
  constexpr int BM = 64, BN = 64, BK = 16;
  __shared__ float As[BK][BM + 4];
  __shared__ float Bs[BK][BN + 4];
  __shared__ float red[16][BN];

  const int tid = threadIdx.x;
  const int tx = tid & 15, ty = tid >> 4;
  const int m0 = blockIdx.y * BM, n0 = blockIdx.x * BN;
  const int k_begin = blockIdx.z * p.k_per_split;
  const int k_end = min(p.K, k_begin + p.k_per_split);

  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;

  const bool a_k_contig = (p.sAk == 1);
  const bool b_n_contig = (p.sBn == 1);

  for (int k0 = k_begin; k0 < k_end; k0 += BK) {
    // ---- stage A tile [BM x BK] ----
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      int m, k;
      if (a_k_contig) { k = tid & 15; m = (tid >> 4) + 16 * i; }
      else { m = tid & 63; k = (tid >> 6) + 4 * i; }
      const int gm = m0 + m, gk = k0 + k;
      As[k][m] = (gm < p.M && gk < k_end) ? __ldg(p.A + gm * p.sAm + gk * p.sAk) : 0.f;
    }
    // ---- stage B tile [BK x BN] ----
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      int n, k;
      if (b_n_contig) { n = tid & 63; k = (tid >> 6) + 4 * i; }
      else { k = tid & 15; n = (tid >> 4) + 16 * i; }
      const int gn = n0 + n, gk = k0 + k;
      Bs[k][n] = (gn < p.N && gk < k_end) ? __ldg(p.B + gk * p.sBk + gn * p.sBn) : 0.f;
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < BK; ++k) {
      const float4 a = *reinterpret_cast<const float4*>(&As[k][ty * 4]);
      const float4 b = *reinterpret_cast<const float4*>(&Bs[k][tx * 4]);
      const float av[4] = {a.x, a.y, a.z, a.w};
      const float bv[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
    }
    __syncthreads();
  }

  // ---- epilogue ----
  float csum[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int gm = m0 + ty * 4 + i;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int gn = n0 + tx * 4 + j;
      if (gm >= p.M || gn >= p.N) continue;
      float v = acc[i][j];
      if constexpr (EPI == EPI_FWD) {
        if (p.addend != nullptr) v += __ldg(p.addend + static_cast<size_t>(gm) * p.ld_add + gn);
        v = act_apply(v + __ldg(p.bias + gn), p.act);
        p.out[static_cast<size_t>(gm) * p.ld_out + gn] = v;
      } else if constexpr (EPI == EPI_DA) {
        v *= act_grad_from_out(__ldg(p.aux + static_cast<size_t>(gm) * p.ld_aux + gn), p.act);
        p.out[static_cast<size_t>(gm) * p.ld_out + gn] = v;
        csum[j] += v;
      } else if constexpr (EPI == EPI_DW) {
        atomicAdd(p.accum + static_cast<size_t>(gm) * p.ld_acc + gn, v);
      } else {
        if (gridDim.z == 1) p.accum[static_cast<size_t>(gm) * p.ld_acc + gn] = v;
        else atomicAdd(p.accum + static_cast<size_t>(gm) * p.ld_acc + gn, v);
      }
    }
  }
  if constexpr (EPI == EPI_DA) {
    if (p.colsum != nullptr) {
#pragma unroll
      for (int j = 0; j < 4; ++j) red[ty][tx * 4 + j] = csum[j];
      __syncthreads();
      if (tid < BN) {
        float s = 0.f;
#pragma unroll
        for (int r = 0; r < 16; ++r) s += red[r][tid];
        if constexpr (DET) {
          if (n0 + tid < p.N) p.det_ws[static_cast<size_t>(blockIdx.y) * p.N + n0 + tid] = s;
        } else {
          if (n0 + tid < p.N) atomicAdd(p.colsum + n0 + tid, s);
        }
      }
      if constexpr (DET) {
        if (det_last_cta(p.det_ticket, gridDim.x * gridDim.y * gridDim.z, 0, 256, tid == 0))
          det_colsum_finish(p.det_ws, static_cast<int>(gridDim.y), p.N, p.colsum, tid, 256);
      }
    }
  }
}

template <int EPI, bool DET = false>
int launch_gemm_f32(GemmF32Params p, int split_k, cudaStream_t st) {
  const int total_kb = (p.K + 15) / 16;
  if (split_k < 1) split_k = 1;
  if (split_k > total_kb) split_k = total_kb > 0 ? total_kb : 1;
  const int kb_per = (total_kb + split_k - 1) / split_k;
  split_k = kb_per > 0 ? (total_kb + kb_per - 1) / kb_per : 1;
  p.k_per_split = kb_per * 16;
  dim3 grid((p.N + 63) / 64, (p.M + 63) / 64, split_k);
  gemm_f32_kernel<EPI, DET><<<grid, 256, 0, st>>>(p);
  SB_CUDA(cudaGetLastError());
  return SB_OK;
}

}  // namespace sb
