// Model performance over scored rows (sb_perf_*, DESIGN §6i): ROC AUC, PR AUC, KS and operating points from one sort.
//
// Each added row becomes a 32-bit key and a 32-bit payload (perf_add_kernel):
//   key      the score's bits mapped so that a DESCENDING score is an ASCENDING key (-0 folded into +0): a positive score
//            u -> ~u & 0x7fffffff, a negative one keeps its bits.  +inf -> 0x007fffff, +0 -> 0x7fffffff, -inf -> 0xff800000.
//   payload  the weight's bits (valid weights are >= 0, -0 becomes +0), with the label in the sign bit.
// The same pass counts the invalid rows of each kind and adds the keys' four 8-bit digit histograms to the handle's.
//
// Sort (perf_sort_pass_kernel): a stable LSD radix sort of the (key, payload) pairs, 8-bit digits, one launch per digit
// whose histogram does not put every key in one bin.  A launch takes tiles of PERF_TILE pairs in the order of a tile
// counter.  Each warp ranks its 512 pairs by digit with __match_any_sync (in element order, so the ranking is stable),
// the tile's digit counts go into a decoupled look-back over the tiles (status words: flag in bits 62..63, count below),
// and the tile is reordered in shared memory so that each digit's pairs leave it as one coalesced run.
//
// Runs (perf_runs_kernel<false> -> perf_tile_scan_kernel -> perf_runs_kernel<true>): a run head is a key that differs
// from its predecessor.  Each thread takes PERF_ITEMS consecutive sorted pairs; the tile's counts (heads, positives,
// negatives) and weight sums (fp64) are formed in a fixed order: serially within a thread, serially over the threads of a
// tile, serially over the tiles.  The weighted prefix at element i is fl(E_tile + fl(B_thread + a_i)), each of E, B and a
// the serial sum of what precedes it, so the cumulative weight sums are the same bits on every run and never decrease
// along the table (every step adds a value >= 0 to the very value the next level starts from).  The last pair of each
// run writes the run table: t_j, TP_j, FP_j (int64), WTP_j, WFP_j (fp64).
//
// Summary (perf_summary_kernel -> perf_summary_final_kernel): every run's terms (A2 in int64, the weighted-AUC and AP sums
// in fp64, the KS maxima with the first run that attains them), strided over a fixed grid, summed over each block by a
// fixed tree and over the blocks in order.  Points (perf_points_kernel): one thread per level, a binary search over the
// monotone run table.
#pragma once
#include "common.cuh"

namespace sb {

constexpr int PERF_THREADS = 256;                        // threads of the sort and run kernels: one per digit
constexpr int PERF_ITEMS = 16;                           // pairs per thread
constexpr int PERF_TILE = PERF_THREADS * PERF_ITEMS;     // pairs per tile
constexpr int PERF_ADD_THREADS = 512;
constexpr int PERF_SUM_BLOCKS = 264;                     // summary partials (fixed: the sums' order depends on m only)
constexpr unsigned long long PERF_AGG = 1ull << 62, PERF_PREFIX = 2ull << 62, PERF_VALUE = PERF_AGG - 1;

// per tile of the run kernels: counts and weight sums (totals after the up pass, exclusive prefixes after the scan)
struct PerfTile {
  long long heads, pos, neg;
  double wp, wn;
};

// summary partials of one block (and, after perf_summary_final_kernel, of the whole table)
struct PerfPart {
  unsigned long long a2;     // sum_j n_j (2 TP_{j-1} + p_j)
  double wauc;               // sum_j (WFP_j - WFP_{j-1}) (WTP_{j-1} + WTP_j) / 2
  double ap, wap;            // sum_j p_j TP_j / (TP_j + FP_j); weighted: runs with wp_j > 0
  unsigned long long ks;     // max_j |TP_j N - FP_j P| and the first j attaining it
  long long ks_j;
  double wks;                // max_j |WTP_j Wn - WFP_j Wp| and the first j
  long long wks_j;
};

struct PerfResult {
  PerfPart a;
  float ks_t, wks_t;         // t_j of the two KS maxima
};

__device__ __forceinline__ uint32_t perf_key(float s) {
  uint32_t u = __float_as_uint(s);
  if (u == 0x80000000u) u = 0u;
  return (u & 0x80000000u) ? u : (~u & 0x7fffffffu);
}

__device__ __forceinline__ float perf_score(uint32_t k) {
  return __uint_as_float((k & 0x80000000u) ? k : (~k & 0x7fffffffu));
}

// rows [0, rows) of one add: scores s[r * stride], labels y[r], weights w[r] (null: 1) -> keys / pay at the same r;
// hist [4][256] += the keys' digit counts; bad[0..2] += rows with a NaN score / a label other than 0 or 1 / a negative or
// non-finite weight
__global__ void __launch_bounds__(PERF_ADD_THREADS)
perf_add_kernel(const float* __restrict__ s, long long stride, const float* __restrict__ y, const float* __restrict__ w, long long rows,
                uint32_t* __restrict__ keys, uint32_t* __restrict__ pay, unsigned int* __restrict__ hist,
                unsigned long long* __restrict__ bad) {
  __shared__ unsigned int h[4 * 256];
  __shared__ unsigned int nb[3];
  for (int i = threadIdx.x; i < 4 * 256; i += blockDim.x) h[i] = 0u;
  if (threadIdx.x < 3) nb[threadIdx.x] = 0u;
  __syncthreads();
  unsigned int b0 = 0, b1 = 0, b2 = 0;
  for (long long r = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; r < rows;
       r += static_cast<long long>(gridDim.x) * blockDim.x) {
    const float sv = __ldg(s + r * stride);
    const float yv = __ldg(y + r);
    const float wv = w != nullptr ? __ldg(w + r) : 1.f;
    const bool pos = yv == 1.f;
    b0 += isnan(sv) ? 1u : 0u;
    b1 += (pos || yv == 0.f) ? 0u : 1u;
    b2 += (wv >= 0.f && !isinf(wv)) ? 0u : 1u;
    const uint32_t k = perf_key(sv);
    keys[r] = k;
    pay[r] = (wv == 0.f ? 0u : __float_as_uint(wv)) | (pos ? 0x80000000u : 0u);
#pragma unroll
    for (int d = 0; d < 4; ++d) atomicAdd(&h[d * 256 + ((k >> (8 * d)) & 255u)], 1u);
  }
  if (b0) atomicAdd(&nb[0], b0);
  if (b1) atomicAdd(&nb[1], b1);
  if (b2) atomicAdd(&nb[2], b2);
  __syncthreads();
  for (int i = threadIdx.x; i < 4 * 256; i += blockDim.x)
    if (h[i]) atomicAdd(hist + i, h[i]);
  if (threadIdx.x < 3 && nb[threadIdx.x]) atomicAdd(bad + threadIdx.x, static_cast<unsigned long long>(nb[threadIdx.x]));
}

// exclusive prefix of v over the PERF_THREADS threads of the block (all of them call it); tmp: PERF_THREADS / 32 words
__device__ __forceinline__ unsigned int perf_block_excl(unsigned int v, unsigned int* tmp) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  unsigned int x = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const unsigned int u = __shfl_up_sync(0xffffffffu, x, o);
    if (lane >= o) x += u;
  }
  if (lane == 31) tmp[wid] = x;
  __syncthreads();
  unsigned int before = 0;
  for (int i = 0; i < wid; ++i) before += tmp[i];
  __syncthreads();
  return before + x - v;
}

// One stable scatter pass of the LSD sort on digit `shift` / 8.  dhist: the 256 counts of this digit over all n keys.
// status [tiles][256] and *tile_ctr are zero at launch.
__global__ void __launch_bounds__(PERF_THREADS)
perf_sort_pass_kernel(const uint32_t* __restrict__ kin, const uint32_t* __restrict__ pin, uint32_t* __restrict__ kout,
                      uint32_t* __restrict__ pout, long long n, int shift, const unsigned int* __restrict__ dhist,
                      unsigned long long* status, unsigned int* tile_ctr) {
  constexpr int WARPS = PERF_THREADS / 32;
  __shared__ uint32_t sk[PERF_TILE], sp[PERF_TILE];
  __shared__ unsigned int wh[WARPS][256];   // per warp: running digit counts, then the warp's offset within the tile
  __shared__ unsigned int texcl[256];       // the tile's first local slot of each digit
  __shared__ long long gofs[256];           // global slot of local slot 0 of each digit's run in the tile
  __shared__ unsigned int tmp[WARPS];
  __shared__ unsigned int tile_s;
  const int t = threadIdx.x, lane = t & 31, wid = t >> 5;
  for (int i = t; i < WARPS * 256; i += PERF_THREADS) (&wh[0][0])[i] = 0u;
  if (t == 0) tile_s = atomicAdd(tile_ctr, 1u);
  __syncthreads();
  const long long tile = tile_s;
  const long long base = tile * PERF_TILE + static_cast<long long>(wid) * (32 * PERF_ITEMS) + lane;
  uint32_t k[PERF_ITEMS], p[PERF_ITEMS];
  unsigned int rk[PERF_ITEMS];
#pragma unroll
  for (int i = 0; i < PERF_ITEMS; ++i) {
    const long long idx = base + 32 * i;
    k[i] = idx < n ? kin[idx] : 0u;
    p[i] = idx < n ? pin[idx] : 0u;
  }
  unsigned int lt;
  asm("mov.u32 %0, %%lanemask_lt;" : "=r"(lt));
  // warp ranking in element order (item i of lane l is element base + 32 i: items outer, lanes inner)
#pragma unroll
  for (int i = 0; i < PERF_ITEMS; ++i) {
    const bool valid = base + 32 * i < n;
    const unsigned int d = valid ? (k[i] >> shift) & 255u : 256u;
    const unsigned int peers = __match_any_sync(0xffffffffu, d);
    const unsigned int pre = valid ? wh[wid][d] : 0u;
    __syncwarp();
    if (valid && (peers & lt) == 0u) wh[wid][d] = pre + __popc(peers);
    __syncwarp();
    rk[i] = pre + __popc(peers & lt);
  }
  __syncthreads();
  // thread t owns digit t: the warps' offsets, the tile's count, and its place among the tiles
  unsigned int cnt = 0;
  for (int v = 0; v < WARPS; ++v) {
    const unsigned int c = wh[v][t];
    wh[v][t] = cnt;
    cnt += c;
  }
  volatile unsigned long long* st = status + tile * 256 + t;
  *st = (tile == 0 ? PERF_PREFIX : PERF_AGG) | cnt;
  const unsigned int ex = perf_block_excl(cnt, tmp);
  const unsigned int dbase = perf_block_excl(__ldg(dhist + t), tmp);
  texcl[t] = ex;
  unsigned long long before = 0;
  if (tile > 0) {
    for (long long j = tile - 1;; --j) {
      const volatile unsigned long long* q = status + j * 256 + t;
      unsigned long long v;
      do { v = *q; } while ((v >> 62) == 0ull);
      before += v & PERF_VALUE;
      if ((v >> 62) == 2ull) break;
    }
    *st = PERF_PREFIX | (before + cnt);
  }
  gofs[t] = static_cast<long long>(dbase) + static_cast<long long>(before) - ex;
  __syncthreads();
#pragma unroll
  for (int i = 0; i < PERF_ITEMS; ++i) {
    if (base + 32 * i < n) {
      const unsigned int d = (k[i] >> shift) & 255u;
      const unsigned int at = texcl[d] + wh[wid][d] + rk[i];
      sk[at] = k[i];
      sp[at] = p[i];
    }
  }
  __syncthreads();
  const long long left = n - tile * PERF_TILE;
  const int nt = left < PERF_TILE ? static_cast<int>(left) : PERF_TILE;
  for (int j = t; j < nt; j += PERF_THREADS) {
    const uint32_t kk = sk[j];
    const long long o = gofs[(kk >> shift) & 255u] + j;
    kout[o] = kk;
    pout[o] = sp[j];
  }
}

// The run pass over the sorted pairs.  DOWN = false: tiles[b] = the tile's totals.  DOWN = true: tiles[b] holds the
// tile's exclusive prefixes (perf_tile_scan_kernel); each run's last pair writes its row of the run table.  Both
// passes form the same per-thread and per-tile sums in the same order.  keys / pay are readable up to a whole tile.
template <bool DOWN>
__global__ void __launch_bounds__(PERF_THREADS)
perf_runs_kernel(const uint32_t* __restrict__ keys, const uint32_t* __restrict__ pay, long long n, PerfTile* __restrict__ tiles,
                 float* __restrict__ rt, long long* __restrict__ rtp, long long* __restrict__ rfp, double* __restrict__ rwtp,
                 double* __restrict__ rwfp) {
  __shared__ long long sh[PERF_THREADS + 1], spos[PERF_THREADS + 1], sneg[PERF_THREADS + 1];
  __shared__ double swp[PERF_THREADS + 1], swn[PERF_THREADS + 1];
  const int t = threadIdx.x;
  const long long i0 = static_cast<long long>(blockIdx.x) * PERF_TILE + static_cast<long long>(t) * PERF_ITEMS;
  uint32_t k[PERF_ITEMS], p[PERF_ITEMS];
#pragma unroll
  for (int v = 0; v < PERF_ITEMS / 4; ++v) {
    const uint4 a = __ldg(reinterpret_cast<const uint4*>(keys + i0) + v);
    const uint4 b = __ldg(reinterpret_cast<const uint4*>(pay + i0) + v);
    k[4 * v] = a.x; k[4 * v + 1] = a.y; k[4 * v + 2] = a.z; k[4 * v + 3] = a.w;
    p[4 * v] = b.x; p[4 * v + 1] = b.y; p[4 * v + 2] = b.z; p[4 * v + 3] = b.w;
  }
  const uint32_t prev = i0 > 0 && i0 <= n ? __ldg(keys + i0 - 1) : ~k[0];
  const uint32_t next = i0 + PERF_ITEMS < n ? __ldg(keys + i0 + PERF_ITEMS) : 0u;
  int h = 0, np = 0, nn = 0;
  double wp = 0.0, wn = 0.0;
#pragma unroll
  for (int i = 0; i < PERF_ITEMS; ++i) {
    if (i0 + i < n) {
      h += k[i] != (i ? k[i - 1] : prev) ? 1 : 0;
      const bool pos = (p[i] >> 31) != 0u;
      const double wv = static_cast<double>(__uint_as_float(p[i] & 0x7fffffffu));
      if (pos) { ++np; wp += wv; } else { ++nn; wn += wv; }
    }
  }
  sh[t] = h; spos[t] = np; sneg[t] = nn; swp[t] = wp; swn[t] = wn;
  __syncthreads();
  if (t == 0) {   // exclusive prefixes over the threads, in thread order; slot PERF_THREADS: the tile's totals
    long long ah = 0, ap = 0, an = 0;
    double awp = 0.0, awn = 0.0;
    for (int j = 0; j <= PERF_THREADS; ++j) {
      const long long ch = sh[j], cp = spos[j], cn = sneg[j];
      const double cwp = swp[j], cwn = swn[j];
      sh[j] = ah; spos[j] = ap; sneg[j] = an; swp[j] = awp; swn[j] = awn;
      if (j == PERF_THREADS) break;
      ah += ch; ap += cp; an += cn; awp += cwp; awn += cwn;
    }
    if (!DOWN) tiles[blockIdx.x] = PerfTile{sh[PERF_THREADS], spos[PERF_THREADS], sneg[PERF_THREADS], swp[PERF_THREADS], swn[PERF_THREADS]};
  }
  if (!DOWN) return;
  __syncthreads();
  const PerfTile e = tiles[blockIdx.x];
  long long run = e.heads + sh[t] - 1, tp = e.pos + spos[t], fp = e.neg + sneg[t];
  const double bwp = swp[t], bwn = swn[t];
  wp = 0.0; wn = 0.0;
#pragma unroll
  for (int i = 0; i < PERF_ITEMS; ++i) {
    if (i0 + i < n) {
      run += k[i] != (i ? k[i - 1] : prev) ? 1 : 0;
      const bool pos = (p[i] >> 31) != 0u;
      const double wv = static_cast<double>(__uint_as_float(p[i] & 0x7fffffffu));
      if (pos) { ++tp; wp += wv; } else { ++fp; wn += wv; }
      const bool tail = i0 + i == n - 1 || (i + 1 < PERF_ITEMS ? k[i + 1] : next) != k[i];
      if (tail) {
        rt[run] = perf_score(k[i]);
        rtp[run] = tp;
        rfp[run] = fp;
        rwtp[run] = e.wp + (bwp + wp);
        rwfp[run] = e.wn + (bwn + wn);
      }
    }
  }
}

// tiles[0, n_tiles): totals -> exclusive prefixes, summed serially in tile order; *total = the grand totals
__global__ void __launch_bounds__(PERF_THREADS)
perf_tile_scan_kernel(PerfTile* __restrict__ tiles, long long n_tiles, PerfTile* __restrict__ total) {
  __shared__ PerfTile c[PERF_THREADS];
  PerfTile a{0, 0, 0, 0.0, 0.0};   // meaningful in thread 0
  for (long long b0 = 0; b0 < n_tiles; b0 += PERF_THREADS) {
    const int nb = n_tiles - b0 < PERF_THREADS ? static_cast<int>(n_tiles - b0) : PERF_THREADS;
    if (threadIdx.x < nb) c[threadIdx.x] = tiles[b0 + threadIdx.x];
    __syncthreads();
    if (threadIdx.x == 0) {
      for (int j = 0; j < nb; ++j) {
        const PerfTile v = c[j];
        c[j] = a;
        a.heads += v.heads; a.pos += v.pos; a.neg += v.neg; a.wp += v.wp; a.wn += v.wn;
      }
    }
    __syncthreads();
    if (threadIdx.x < nb) tiles[b0 + threadIdx.x] = c[threadIdx.x];
    __syncthreads();
  }
  if (threadIdx.x == 0) *total = a;
}

__device__ __forceinline__ void perf_combine(PerfPart& a, const PerfPart& b) {
  a.a2 += b.a2;
  a.wauc += b.wauc;
  a.ap += b.ap;
  a.wap += b.wap;
  if (b.ks > a.ks || (b.ks == a.ks && b.ks_j < a.ks_j)) { a.ks = b.ks; a.ks_j = b.ks_j; }
  if (b.wks > a.wks || (b.wks == a.wks && b.wks_j < a.wks_j)) { a.wks = b.wks; a.wks_j = b.wks_j; }
}

// runs j = blockIdx.x * PERF_THREADS + t + k * gridDim.x * PERF_THREADS, summed in that order per thread, then over the
// block's threads by a fixed tree -> parts[blockIdx.x].  m >= 1.
__global__ void __launch_bounds__(PERF_THREADS)
perf_summary_kernel(const long long* __restrict__ rtp, const long long* __restrict__ rfp, const double* __restrict__ rwtp,
                    const double* __restrict__ rwfp, long long m, PerfPart* __restrict__ parts) {
  __shared__ PerfPart sp[PERF_THREADS];
  const long long P = rtp[m - 1], N = rfp[m - 1];
  const double Wp = rwtp[m - 1], Wn = rwfp[m - 1];
  PerfPart a{0ull, 0.0, 0.0, 0.0, 0ull, m, 0.0, m};
  for (long long j = static_cast<long long>(blockIdx.x) * PERF_THREADS + threadIdx.x; j < m;
       j += static_cast<long long>(gridDim.x) * PERF_THREADS) {
    const long long tp = rtp[j], fp = rfp[j], tp0 = j ? rtp[j - 1] : 0, fp0 = j ? rfp[j - 1] : 0;
    const double wtp = rwtp[j], wfp = rwfp[j], wtp0 = j ? rwtp[j - 1] : 0.0, wfp0 = j ? rwfp[j - 1] : 0.0;
    const long long pj = tp - tp0, nj = fp - fp0;
    a.a2 += static_cast<unsigned long long>(nj) * static_cast<unsigned long long>(2 * tp0 + pj);
    a.wauc += (wfp - wfp0) * (wtp0 + wtp) * 0.5;
    if (pj > 0) a.ap += static_cast<double>(pj) * (static_cast<double>(tp) / static_cast<double>(tp + fp));
    const double wpj = wtp - wtp0;
    if (wpj > 0.0) a.wap += wpj * (wtp / (wtp + wfp));
    const long long d = tp * N - fp * P;
    const unsigned long long ad = static_cast<unsigned long long>(d < 0 ? -d : d);
    if (ad > a.ks || (ad == a.ks && j < a.ks_j)) { a.ks = ad; a.ks_j = j; }
    const double wd = fabs(wtp * Wn - wfp * Wp);
    if (wd > a.wks || (wd == a.wks && j < a.wks_j)) { a.wks = wd; a.wks_j = j; }
  }
  sp[threadIdx.x] = a;
  __syncthreads();
  for (int s = PERF_THREADS / 2; s > 0; s >>= 1) {
    if (threadIdx.x < s) perf_combine(sp[threadIdx.x], sp[threadIdx.x + s]);
    __syncthreads();
  }
  if (threadIdx.x == 0) parts[blockIdx.x] = sp[0];
}

// parts[0, n) -> out->a, in part order (one thread), with the thresholds of the two KS maxima
__global__ void perf_summary_final_kernel(const PerfPart* __restrict__ parts, int n, const float* __restrict__ rt,
                                          PerfResult* __restrict__ out) {
  PerfPart a = parts[0];
  for (int b = 1; b < n; ++b) perf_combine(a, parts[b]);
  out->a = a;
  out->ks_t = rt[a.ks_j];
  out->wks_t = rt[a.wks_j];
}

// One operating point per level (thread), m >= 1.  axis SB_PERF_ACTION_RATE / RECALL / FPR: the first run whose
// num_j / den >= level (num: TP+FP, TP or FP, weighted or not; den: the matching total, > 0); SB_PERF_SCORE: the last run
// with t_j >= level, or the empty point {+inf, 0, 0, 0, 0} when there is none.
__global__ void perf_points_kernel(const float* __restrict__ rt, const long long* __restrict__ rtp, const long long* __restrict__ rfp,
                                   const double* __restrict__ rwtp, const double* __restrict__ rwfp, long long m, int axis,
                                   int weighted, double den, const double* __restrict__ levels, int n, sb_perf_point* __restrict__ out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const double lv = levels[i];
  long long j;
  if (axis == SB_PERF_SCORE) {
    if (!(static_cast<double>(rt[0]) >= lv)) {
      out[i] = sb_perf_point{__int_as_float(0x7f800000), 0, 0, 0.0, 0.0};
      return;
    }
    long long lo = 0, hi = m - 1;
    while (lo < hi) {
      const long long mid = lo + (hi - lo + 1) / 2;
      if (static_cast<double>(rt[mid]) >= lv) lo = mid; else hi = mid - 1;
    }
    j = lo;
  } else {
    long long lo = 0, hi = m - 1;
    while (lo < hi) {
      const long long mid = lo + (hi - lo) / 2;
      double num;
      if (weighted) num = axis == SB_PERF_ACTION_RATE ? rwtp[mid] + rwfp[mid] : axis == SB_PERF_RECALL ? rwtp[mid] : rwfp[mid];
      else num = static_cast<double>(axis == SB_PERF_ACTION_RATE ? rtp[mid] + rfp[mid] : axis == SB_PERF_RECALL ? rtp[mid] : rfp[mid]);
      if (num / den >= lv) hi = mid; else lo = mid + 1;
    }
    j = lo;
  }
  out[i] = sb_perf_point{rt[j], rtp[j], rfp[j], rwtp[j], rwfp[j]};
}

}  // namespace sb
