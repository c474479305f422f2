// Bagged-model scoring (sb_ensemble_*, DESIGN §6h): the statistics of K member scores per row.
//
// ensemble_stats_kernel reads the members' scores of one row chunk, slot g = member g's scores [rows] at slots + g * ld,
// and writes, for each row r,
//   scores[r, g]  member g's score, row-major [rows, K] (the slots transposed)
//   stats[r, 0..3] = {mean, max, min, median}:
//     mean    ((s_0 + s_1) + ...) + s_{K-1} in fp32, in member order, then / (float)K
//     max     the first member score in member order that no later one exceeds (v > m replaces m), min likewise
//     median  the members' scores sorted by value, equal values in member order: K odd the middle one, K even
//             (a + b) * 0.5f of the two middle ones
//     a NaN among the K scores makes all four the quiet NaN 0x7fc00000.
// Either output may be null.  One thread per row; the block's rows are staged in shared memory as a column of K values
// per thread (v[g][t]: a warp's reads of one member are 32 consecutive words), so the statistics read no register
// array by a dynamic index: the median takes each value's rank by counting, O(K^2) compares.  Both outputs leave the
// block as one contiguous run each ([rows of the block, K] and [rows of the block, 4]), stored by consecutive threads.
//
// ensemble_stat_kernel writes one of the four statistics of each row as a contiguous column [rows]: the ensemble's
// sensitivity and reason codes (DESIGN §6j) form it for every pair row of a piece.  Both kernels take the statistics
// from ensemble_row_stats, the one definition of them.
#pragma once
#include "common.cuh"

namespace sb {

constexpr int ENS_THREADS = 128;    // rows per block

// the statistics of thread t's row, v[0 .. K-1][t] (the definitions above) -> st[4 t .. 4 t + 3] = mean, max, min, median
__device__ __forceinline__ void ensemble_row_stats(const float (*v)[ENS_THREADS], int t, int K, float* st) {
  float sum = v[0][t], mx = v[0][t], mn = v[0][t];
  bool nan = isnan(v[0][t]);
  for (int g = 1; g < K; ++g) {
    const float x = v[g][t];
    nan |= isnan(x);
    sum += x;
    if (x > mx) mx = x;
    if (x < mn) mn = x;
  }
  // rank of member i: the values below it, plus the equal ones of lower members (a total order, so the ranks are
  // 0 .. K-1 once no value is NaN)
  const int lo = (K - 1) / 2, hi = K / 2;
  float a = 0.f, b = 0.f;
  for (int i = 0; i < K; ++i) {
    const float x = v[i][t];
    int rank = 0;
    for (int j = 0; j < K; ++j) {
      const float y = v[j][t];
      rank += (y < x || (y == x && j < i)) ? 1 : 0;
    }
    if (rank == lo) a = x;
    if (rank == hi) b = x;
  }
  const float qnan = __int_as_float(0x7fc00000);
  st[4 * t + 0] = nan ? qnan : sum / static_cast<float>(K);
  st[4 * t + 1] = nan ? qnan : mx;
  st[4 * t + 2] = nan ? qnan : mn;
  st[4 * t + 3] = nan ? qnan : (lo == hi ? a : (a + b) * 0.5f);
}

__global__ void __launch_bounds__(ENS_THREADS)
ensemble_stats_kernel(const float* __restrict__ slots, long long ld, int K, int rows, float* __restrict__ scores,
                      float* __restrict__ stats) {
  __shared__ float v[SB_ENSEMBLE_MAX][ENS_THREADS];
  __shared__ float st[ENS_THREADS * 4];
  const int t = threadIdx.x;
  const long long r0 = static_cast<long long>(blockIdx.x) * ENS_THREADS;
  const int nr = rows - r0 < ENS_THREADS ? static_cast<int>(rows - r0) : ENS_THREADS;
  for (int g = 0; g < K; ++g) v[g][t] = t < nr ? __ldg(slots + g * ld + r0 + t) : 0.f;
  __syncthreads();
  if (scores != nullptr)
    for (int i = t; i < nr * K; i += ENS_THREADS) scores[r0 * K + i] = v[i % K][i / K];
  if (stats == nullptr) return;
  if (t < nr) ensemble_row_stats(v, t, K, st);
  __syncthreads();
  for (int i = t; i < nr * 4; i += ENS_THREADS) stats[r0 * 4 + i] = st[i];
}

// out[r] = statistic `stat` (SB_STAT_MEAN / MAX / MIN / MEDIAN) of row r's K member scores, slots as ensemble_stats_kernel
// reads them.  Each thread reads back only its own column of v and its own four words of st.
__global__ void __launch_bounds__(ENS_THREADS)
ensemble_stat_kernel(const float* __restrict__ slots, long long ld, int K, int rows, int stat, float* __restrict__ out) {
  __shared__ float v[SB_ENSEMBLE_MAX][ENS_THREADS];
  __shared__ float st[ENS_THREADS * 4];
  const int t = threadIdx.x;
  const long long r0 = static_cast<long long>(blockIdx.x) * ENS_THREADS;
  if (r0 + t >= rows) return;
  for (int g = 0; g < K; ++g) v[g][t] = __ldg(slots + g * ld + r0 + t);
  ensemble_row_stats(v, t, K, st);
  out[r0 + t] = st[4 * t + stat];
}

}  // namespace sb
