// The forward of a small SB_PREC_FP32 batch in one launch: every hidden layer and the sigmoid output unit for up to
// SMALL_ROWS rows.  It gives the bits of the batched fp32 path (gemm_f32_kernel<EPI_FWD> per hidden layer, then
// out_layer_kernel<float>), so a model may pick either by row count without changing a score:
//   - hidden element (r, n): one fmaf chain over k = 0, 1, ..., K - 1, then fmaf(0, 0, acc) up to the next multiple of
//     16 (gemm_f32's zero-padded K tail, which turns an accumulated -0 into +0), then act_apply(acc + b_n);
//   - score of row r: lane-strided fmaf partials over j = lane, lane + 32, ..., warp_sum, + b_o, sigmoidf_stable.
// Layout: a grid of SR_CLUSTER-CTA clusters.  Cluster c owns rows [SR_ROWS c, SR_ROWS (c + 1)) and carries them through
// every layer; its CTAs split each layer's output columns in blocks of SR_COLS.  A layer's activations go through a
// global scratch buffer (two of them, alternating), and the cluster meets at a release / acquire cluster barrier between
// layers.  Clusters never wait on each other.
// Inside a CTA a k-block of SR_KB rows of W (SR_COLS columns) and of the cluster's activations is staged by cp.async
// into a ring of SR_STAGES slots, so that the L2 / HBM latency of W hides behind the FMA chains.  Thread t owns column
// t % SR_COLS and the four rows 4 (t / SR_COLS) .. + 3 of the cluster's group.
#pragma once
#include "common.cuh"
#include "ptx.cuh"

namespace sb {

constexpr int SR_CLUSTER = 8;     // CTAs per cluster (the portable maximum)
constexpr int SR_ROWS = 8;        // rows per cluster
constexpr int SR_COLS = 128;      // output columns per CTA and column block
constexpr int SR_THREADS = 256;   // SR_COLS columns x 2 groups of 4 rows
constexpr int SR_KB = 16;         // k per ring slot (gemm_f32's K tile, so the zero-padded tail matches)
constexpr int SR_STAGES = 8;
constexpr int SMALL_ROWS = 128;   // sb_model_* score batches of up to this many rows of an fp32 model here
constexpr int SR_SMEM = SR_STAGES * (SR_KB * SR_COLS + SR_ROWS * SR_KB) * static_cast<int>(sizeof(float));
static_assert(SR_THREADS == 2 * SR_COLS && SR_ROWS == 8 && SR_KB % 4 == 0, "thread layout");

struct ScoreRowsParams {
  int rows, F, L;
  const float* X;          // [rows, F] device
  const float* theta;      // flat parameters (W_l [in, out] row-major, b_l, ..., w_o, b_o)
  float* act[2];           // scratch [SMALL_ROWS, ld_act], 16-byte aligned rows
  int ld_act;              // multiple of 4, >= every hidden width
  float* yhat;             // [rows] device
  int out[SB_MAX_HIDDEN], act_fn[SB_MAX_HIDDEN];
  long long w_off[SB_MAX_HIDDEN + 1], b_off[SB_MAX_HIDDEN + 1];
};

__global__ void __cluster_dims__(SR_CLUSTER, 1, 1) __launch_bounds__(SR_THREADS)
score_rows_kernel(const ScoreRowsParams p) {
  extern __shared__ __align__(16) float sr_smem[];
  float* Ws = sr_smem;                                    // [SR_STAGES][SR_KB][SR_COLS]
  float* As = sr_smem + SR_STAGES * SR_KB * SR_COLS;      // [SR_STAGES][SR_ROWS][SR_KB]
  const int tid = threadIdx.x;
  const int rank = static_cast<int>(cluster_ctarank());
  const int r0 = (blockIdx.x / SR_CLUSTER) * SR_ROWS;
  const int nr = min(SR_ROWS, p.rows - r0);
  const int c = tid % SR_COLS, g = tid / SR_COLS;         // column in the block, row group (warp-uniform)
  const bool group_live = 4 * g < nr;

  int K = p.F;
  for (int l = 0; l < p.L; ++l) {
    const int N = p.out[l];
    const float* W = p.theta + p.w_off[l];
    const float* src = l == 0 ? p.X : p.act[(l - 1) & 1];
    float* dst = p.act[l & 1];
    const int nkb = (K + SR_KB - 1) / SR_KB;
    for (int n0 = rank * SR_COLS; n0 < N; n0 += SR_CLUSTER * SR_COLS) {   // uniform over the CTA
      // k-block kb of W[:, n0 .. n0 + SR_COLS) and of the cluster's rows of A_{l-1} into ring slot kb % SR_STAGES
      auto issue = [&](int kb) {
        if (kb < nkb) {
          const int s = kb % SR_STAGES, k0 = kb * SR_KB;
          float* ws = Ws + s * SR_KB * SR_COLS;
#pragma unroll
          for (int j = 0; j < SR_KB * SR_COLS / SR_THREADS; ++j) {
            const int i = tid + j * SR_THREADS, k = i / SR_COLS, cc = i % SR_COLS;
            const bool ok = k0 + k < K && n0 + cc < N;
            cp_async_ca4(smem_u32(ws + i), ok ? W + static_cast<size_t>(k0 + k) * N + n0 + cc : W, ok ? 4u : 0u);
          }
          float* as = As + s * SR_ROWS * SR_KB;
          if (l == 0) {         // the caller's rows: any F, so 4-byte copies
            if (tid < SR_ROWS * SR_KB) {
              const int r = tid / SR_KB, k = tid % SR_KB;
              const bool ok = r < nr && k0 + k < K;
              cp_async_ca4(smem_u32(as + tid), ok ? src + static_cast<size_t>(r0 + r) * K + k0 + k : src, ok ? 4u : 0u);
            }
          } else if (tid < SR_ROWS * SR_KB / 4) {   // scratch written by the cluster's CTAs: 16-byte copies through L2
            const int r = tid / (SR_KB / 4), k = 4 * (tid % (SR_KB / 4));
            const int left = K - (k0 + k);
            const uint32_t bytes = r < nr && left > 0 ? 4u * static_cast<uint32_t>(min(left, 4)) : 0u;
            cp_async_cg16(smem_u32(as + r * SR_KB + k), bytes ? src + static_cast<size_t>(r0 + r) * p.ld_act + k0 + k : src, bytes);
          }
        }
        cp_async_commit();
      };
      for (int kb = 0; kb < SR_STAGES - 1; ++kb) issue(kb);
      float acc[4] = {0.f, 0.f, 0.f, 0.f};
      for (int kb = 0; kb < nkb; ++kb) {
        cp_async_wait<SR_STAGES - 2>();
        __syncthreads();                   // slot kb is complete for every thread; slot kb - 1 is read by none
        issue(kb + SR_STAGES - 1);
        if (group_live) {
          const int s = kb % SR_STAGES;
          const float* ws = Ws + s * SR_KB * SR_COLS + c;
          const float* as = As + (s * SR_ROWS + 4 * g) * SR_KB;
#pragma unroll
          for (int k = 0; k < SR_KB; k += 4) {
            float4 a[4];
#pragma unroll
            for (int r = 0; r < 4; ++r) a[r] = *reinterpret_cast<const float4*>(as + r * SR_KB + k);
            const float w0 = ws[(k + 0) * SR_COLS], w1 = ws[(k + 1) * SR_COLS];
            const float w2 = ws[(k + 2) * SR_COLS], w3 = ws[(k + 3) * SR_COLS];
#pragma unroll
            for (int r = 0; r < 4; ++r) {
              acc[r] = fmaf(a[r].x, w0, acc[r]);
              acc[r] = fmaf(a[r].y, w1, acc[r]);
              acc[r] = fmaf(a[r].z, w2, acc[r]);
              acc[r] = fmaf(a[r].w, w3, acc[r]);
            }
          }
        }
      }
      cp_async_wait<0>();
      __syncthreads();                     // the ring is free for the next column block / layer
      const int n = n0 + c;
      if (group_live && n < N) {
        const float b = __ldg(p.theta + p.b_off[l] + n);
#pragma unroll
        for (int r = 0; r < 4; ++r)
          if (4 * g + r < nr) dst[static_cast<size_t>(r0 + 4 * g + r) * p.ld_act + n] = act_apply(acc[r] + b, p.act_fn[l]);
      }
    }
    cluster_sync_release_acquire();        // A_l of the cluster's rows is complete
    K = N;
  }

  // output unit: warp w of CTA 0 scores the cluster's row w
  const int warp = tid / 32, lane = tid % 32;
  if (rank == 0 && warp < nr) {
    const float* a = p.act[(p.L - 1) & 1] + static_cast<size_t>(r0 + warp) * p.ld_act;
    const float* wo = p.theta + p.w_off[p.L];
    float z = 0.f;
    for (int j = lane; j < K; j += 32) z = fmaf(__ldcg(a + j), __ldg(wo + j), z);
    z = warp_sum(z) + __ldg(p.theta + p.b_off[p.L]);
    if (lane == 0) p.yhat[r0 + warp] = sigmoidf_stable(z);
  }
}

}  // namespace sb
