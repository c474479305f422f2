// extern "C" surface of the performance handle (sb_perf_*): exact ranking metrics of scored rows from one radix sort
// (DESIGN §6i, kernels in perf.cuh).  See include/shifu_b200.h for the definitions.
#include <algorithm>
#include <cmath>
#include <limits>
#include <memory>
#include "net.cuh"
#include "perf.cuh"

using namespace sb;

constexpr long long PERF_MAX_ROWS = 2147483647LL;   // 2^31 - 1 rows per handle: every count fits the int64 formulas
constexpr long long PERF_STAGE_ROWS = 1 << 20;      // host rows go through a device staging of this many (s, y, w)

struct sb_perf {
  int device = -1, sms = 0;
  cudaStream_t stream = nullptr;
  cudaEvent_t ev_after = nullptr;      // the point of after_stream an add is queued behind
  long long rows = 0, cap = 0;         // rows held; pair capacity (a multiple of PERF_TILE)
  long long sorted = 0, m = 0;         // rows the run table describes, its runs
  long long P = 0, N = 0;              // the table's totals (its last row)
  double Wp = 0.0, Wn = 0.0;
  int cur = 0;                         // keys[cur] / pay[cur] hold the rows; the other pair is the sort's double buffer
  uint32_t* keys[2] = {nullptr, nullptr};
  uint32_t* pay[2] = {nullptr, nullptr};
  unsigned long long* status = nullptr;   // [cap / PERF_TILE][256]: the sort's look-back words
  PerfTile* tiles = nullptr;              // [cap / PERF_TILE]
  long long run_cap = 0;
  float* rt = nullptr;                    // the run table [run_cap]
  long long *rtp = nullptr, *rfp = nullptr;
  double *rwtp = nullptr, *rwfp = nullptr;
  unsigned int* hist = nullptr;           // [4][256] digit counts of every key held
  unsigned long long* bad = nullptr;      // [3] invalid rows: NaN score, bad label, bad weight
  unsigned int* tile_ctr = nullptr;
  PerfPart* parts = nullptr;              // [PERF_SUM_BLOCKS]
  PerfResult* result = nullptr;
  PerfTile* total = nullptr;
  float* stage = nullptr;                 // [3][PERF_STAGE_ROWS], at the first add that reads host memory
  long long pt_cap = 0;                   // sb_perf_points' levels and points on the device
  double* d_levels = nullptr;
  sb_perf_point* d_points = nullptr;
  long long bytes = 0;                    // device bytes held (sb_debug_perf_bytes)

  // stream-ordered allocations, so that growing on an asynchronous add needs no host synchronise
  template <typename T> int alloc(T** p, long long n) {
    void* q = nullptr;
    SB_CUDA(cudaMallocAsync(&q, sizeof(T) * static_cast<size_t>(n), stream));
    *p = static_cast<T*>(q);
    bytes += static_cast<long long>(sizeof(T)) * n;
    return SB_OK;
  }
  template <typename T> void release(T** p, long long n) {
    if (*p == nullptr) return;
    cudaFreeAsync(*p, stream);
    bytes -= static_cast<long long>(sizeof(T)) * n;
    *p = nullptr;
  }
  void release_runs() {
    release(&rt, run_cap); release(&rtp, run_cap); release(&rfp, run_cap); release(&rwtp, run_cap); release(&rwfp, run_cap);
    run_cap = 0;
  }
  ~sb_perf() {
    if (!stream) return;
    cudaSetDevice(device);
    const long long nt = cap / PERF_TILE;
    for (int b = 0; b < 2; ++b) { release(&keys[b], cap); release(&pay[b], cap); }
    release(&status, nt * 256); release(&tiles, nt);
    release_runs();
    release(&hist, 4 * 256); release(&bad, 3); release(&tile_ctr, 1); release(&parts, PERF_SUM_BLOCKS);
    release(&result, 1); release(&total, 1); release(&stage, 3 * PERF_STAGE_ROWS);
    release(&d_levels, pt_cap); release(&d_points, pt_cap);
    cudaStreamSynchronize(stream);
    if (ev_after) cudaEventDestroy(ev_after);
    cudaStreamDestroy(stream);
  }
};

// capacity for `need` rows: grows by half at least, keeps the rows held (copied into the new pair 0)
static int perf_reserve(sb_perf* p, long long need) {
  if (need <= p->cap) return SB_OK;
  long long c = std::max(need, p->cap + p->cap / 2);
  c = (c + PERF_TILE - 1) / PERF_TILE * PERF_TILE;
  const long long nt = c / PERF_TILE, old_nt = p->cap / PERF_TILE;
  sb_perf q;                           // the new buffers, owned by q until they are swapped in
  q.stream = p->stream;
  q.device = p->device;
  int s = SB_OK;
  for (int b = 0; b < 2 && s == SB_OK; ++b) {
    s = q.alloc(&q.keys[b], c);
    if (s == SB_OK) s = q.alloc(&q.pay[b], c);
  }
  if (s == SB_OK) s = q.alloc(&q.status, nt * 256);
  if (s == SB_OK) s = q.alloc(&q.tiles, nt);
  if (s == SB_OK && p->rows > 0) {
    const size_t b = sizeof(uint32_t) * static_cast<size_t>(p->rows);
    if (cudaMemcpyAsync(q.keys[0], p->keys[p->cur], b, cudaMemcpyDeviceToDevice, p->stream) != cudaSuccess ||
        cudaMemcpyAsync(q.pay[0], p->pay[p->cur], b, cudaMemcpyDeviceToDevice, p->stream) != cudaSuccess)
      s = set_error(SB_ERR_CUDA, "copying %lld rows into the grown buffers failed", p->rows);
  }
  if (s != SB_OK) {
    for (int b = 0; b < 2; ++b) { q.release(&q.keys[b], c); q.release(&q.pay[b], c); }
    q.release(&q.status, nt * 256); q.release(&q.tiles, nt);
    q.stream = nullptr;                // q's destructor must not tear down p's stream
    return s;
  }
  for (int b = 0; b < 2; ++b) {
    p->release(&p->keys[b], p->cap); p->release(&p->pay[b], p->cap);
    std::swap(p->keys[b], q.keys[b]); std::swap(p->pay[b], q.pay[b]);
  }
  p->release(&p->status, old_nt * 256); p->release(&p->tiles, old_nt);
  std::swap(p->status, q.status); std::swap(p->tiles, q.tiles);
  p->bytes += q.bytes;
  q.stream = nullptr;
  p->cur = 0;
  p->cap = c;
  return SB_OK;
}

// Synchronous: refuses a handle that holds invalid rows, then sorts the rows and builds the run table if rows arrived
// since the last time
static int perf_prepare(sb_perf* p) {
  SB_CUDA(cudaSetDevice(p->device));
  unsigned long long bad[3];
  SB_CUDA(cudaMemcpyAsync(bad, p->bad, sizeof(bad), cudaMemcpyDeviceToHost, p->stream));
  SB_CUDA(cudaStreamSynchronize(p->stream));
  SB_CHECK(bad[0] + bad[1] + bad[2] == 0, SB_ERR_INVALID,
           "the handle holds invalid rows: %llu with a NaN score, %llu with a label other than 0 or 1, %llu with a negative "
           "or non-finite weight (sb_perf_reset forgets them)", bad[0], bad[1], bad[2]);
  if (p->sorted == p->rows) return SB_OK;
  const long long n = p->rows;
  const long long nt = (n + PERF_TILE - 1) / PERF_TILE;
  unsigned int hist[4 * 256];
  SB_CUDA(cudaMemcpyAsync(hist, p->hist, sizeof(hist), cudaMemcpyDeviceToHost, p->stream));
  SB_CUDA(cudaStreamSynchronize(p->stream));
  for (int d = 0; d < 4; ++d) {
    bool one_bin = false;
    for (int b = 0; b < 256; ++b) one_bin |= hist[d * 256 + b] == static_cast<unsigned int>(n);
    if (one_bin) continue;             // this digit leaves the order as it is
    SB_CUDA(cudaMemsetAsync(p->status, 0, sizeof(unsigned long long) * 256 * static_cast<size_t>(nt), p->stream));
    SB_CUDA(cudaMemsetAsync(p->tile_ctr, 0, sizeof(unsigned int), p->stream));
    SB_TRY(launch_kernel(perf_sort_pass_kernel, dim3(static_cast<unsigned>(nt)), dim3(PERF_THREADS), 0, p->stream, false,
                         static_cast<const uint32_t*>(p->keys[p->cur]), static_cast<const uint32_t*>(p->pay[p->cur]),
                         p->keys[p->cur ^ 1], p->pay[p->cur ^ 1], n, 8 * d, static_cast<const unsigned int*>(p->hist + 256 * d),
                         p->status, p->tile_ctr));
    p->cur ^= 1;
  }
  if (p->run_cap < p->cap) {
    p->release_runs();
    SB_TRY(p->alloc(&p->rt, p->cap)); SB_TRY(p->alloc(&p->rtp, p->cap)); SB_TRY(p->alloc(&p->rfp, p->cap));
    SB_TRY(p->alloc(&p->rwtp, p->cap)); SB_TRY(p->alloc(&p->rwfp, p->cap));
    p->run_cap = p->cap;
  }
  const uint32_t* k = p->keys[p->cur];
  const uint32_t* w = p->pay[p->cur];
  SB_TRY(launch_kernel(perf_runs_kernel<false>, dim3(static_cast<unsigned>(nt)), dim3(PERF_THREADS), 0, p->stream, false, k, w, n,
                       p->tiles, p->rt, p->rtp, p->rfp, p->rwtp, p->rwfp));
  SB_TRY(launch_kernel(perf_tile_scan_kernel, dim3(1), dim3(PERF_THREADS), 0, p->stream, false, p->tiles, nt, p->total));
  SB_TRY(launch_kernel(perf_runs_kernel<true>, dim3(static_cast<unsigned>(nt)), dim3(PERF_THREADS), 0, p->stream, false, k, w, n,
                       p->tiles, p->rt, p->rtp, p->rfp, p->rwtp, p->rwfp));
  PerfTile tot;
  SB_CUDA(cudaMemcpyAsync(&tot, p->total, sizeof(tot), cudaMemcpyDeviceToHost, p->stream));
  SB_CUDA(cudaStreamSynchronize(p->stream));
  p->m = tot.heads;
  p->P = p->N = 0;
  p->Wp = p->Wn = 0.0;
  if (p->m > 0) {                      // the totals are the table's last row (the metrics' denominators)
    const long long j = p->m - 1;
    SB_CUDA(cudaMemcpyAsync(&p->P, p->rtp + j, sizeof(long long), cudaMemcpyDeviceToHost, p->stream));
    SB_CUDA(cudaMemcpyAsync(&p->N, p->rfp + j, sizeof(long long), cudaMemcpyDeviceToHost, p->stream));
    SB_CUDA(cudaMemcpyAsync(&p->Wp, p->rwtp + j, sizeof(double), cudaMemcpyDeviceToHost, p->stream));
    SB_CUDA(cudaMemcpyAsync(&p->Wn, p->rwfp + j, sizeof(double), cudaMemcpyDeviceToHost, p->stream));
    SB_CUDA(cudaStreamSynchronize(p->stream));
  }
  p->sorted = n;
  return SB_OK;
}

extern "C" {

int sb_perf_create(int device, int64_t reserve_rows, sb_perf_t** out) {
  SB_CHECK(out, SB_ERR_INVALID, "out is null");
  *out = nullptr;
  SB_CHECK(reserve_rows >= 0 && reserve_rows <= PERF_MAX_ROWS, SB_ERR_INVALID, "reserve_rows = %lld outside [0, 2^31 - 1]",
           static_cast<long long>(reserve_rows));
  std::unique_ptr<sb_perf> p(new sb_perf());
  SB_TRY(check_device(device, &p->sms));
  p->device = device;
  SB_CUDA(cudaStreamCreateWithFlags(&p->stream, cudaStreamNonBlocking));
  SB_CUDA(cudaEventCreateWithFlags(&p->ev_after, cudaEventDisableTiming));
  SB_TRY(p->alloc(&p->hist, 4 * 256));
  SB_TRY(p->alloc(&p->bad, 3));
  SB_TRY(p->alloc(&p->tile_ctr, 1));
  SB_TRY(p->alloc(&p->parts, PERF_SUM_BLOCKS));
  SB_TRY(p->alloc(&p->result, 1));
  SB_TRY(p->alloc(&p->total, 1));
  SB_CUDA(cudaMemsetAsync(p->hist, 0, sizeof(unsigned int) * 4 * 256, p->stream));
  SB_CUDA(cudaMemsetAsync(p->bad, 0, sizeof(unsigned long long) * 3, p->stream));
  SB_TRY(perf_reserve(p.get(), reserve_rows));
  SB_CUDA(cudaStreamSynchronize(p->stream));
  *out = p.release();
  return SB_OK;
}

int sb_perf_destroy(sb_perf_t* p) {
  delete p;
  return SB_OK;
}

int sb_perf_reset(sb_perf_t* p) {
  SB_CHECK(p, SB_ERR_STATE, "performance handle not initialized.");
  SB_CUDA(cudaSetDevice(p->device));
  SB_CUDA(cudaMemsetAsync(p->hist, 0, sizeof(unsigned int) * 4 * 256, p->stream));
  SB_CUDA(cudaMemsetAsync(p->bad, 0, sizeof(unsigned long long) * 3, p->stream));
  p->rows = p->sorted = p->m = p->P = p->N = 0;
  p->Wp = p->Wn = 0.0;
  return SB_OK;
}

int sb_perf_add(sb_perf_t* p, const float* scores, int32_t score_stride, const float* y, const float* w, int64_t rows,
                void* after_stream) {
  SB_CHECK(p, SB_ERR_STATE, "performance handle not initialized.");
  SB_CHECK(scores && y, SB_ERR_INVALID, "scores and y must not be null");
  SB_CHECK(rows >= 0, SB_ERR_INVALID, "rows = %lld < 0", static_cast<long long>(rows));
  SB_CHECK(score_stride >= 1, SB_ERR_INVALID, "score_stride = %d < 1", score_stride);
  SB_CHECK(rows <= PERF_MAX_ROWS - p->rows, SB_ERR_INVALID, "%lld rows held + %lld added exceed 2^31 - 1 rows per handle", p->rows,
           static_cast<long long>(rows));
  if (rows == 0) return SB_OK;
  // host memory (pageable, pinned or managed) is read through a staging copy
  const int ds = ptr_device(scores), dy = ptr_device(y), dw = w ? ptr_device(w) : p->device;
  for (int d : {ds, dy, dw})
    SB_CHECK(d < 0 || d == p->device, SB_ERR_INVALID, "a device pointer on device %d, the handle is on device %d", d, p->device);
  const bool on_device = ds >= 0 && dy >= 0 && dw >= 0;
  SB_CUDA(cudaSetDevice(p->device));
  if (after_stream) {
    SB_CUDA(cudaEventRecord(p->ev_after, static_cast<cudaStream_t>(after_stream)));
    SB_CUDA(cudaStreamWaitEvent(p->stream, p->ev_after, 0));
  }
  SB_TRY(perf_reserve(p, p->rows + rows));
  const long long sp = score_stride;
  auto add = [&](const float* s, long long stride, const float* yy, const float* ww, long long r0, long long c) {
    const long long grid = std::min<long long>((c + PERF_ADD_THREADS - 1) / PERF_ADD_THREADS, 4LL * p->sms);
    return launch_kernel(perf_add_kernel, dim3(static_cast<unsigned>(grid)), dim3(PERF_ADD_THREADS), 0, p->stream, false, s, stride,
                         yy, ww, c, p->keys[p->cur] + p->rows + r0, p->pay[p->cur] + p->rows + r0, p->hist, p->bad);
  };
  if (on_device) {
    SB_TRY(add(scores, sp, y, w, 0, rows));
  } else {
    if (!p->stage) SB_TRY(p->alloc(&p->stage, 3 * PERF_STAGE_ROWS));
    float* ss = p->stage;
    float* sy = ss + PERF_STAGE_ROWS;
    float* sw = sy + PERF_STAGE_ROWS;
    for (long long r0 = 0; r0 < rows; r0 += PERF_STAGE_ROWS) {
      const long long c = std::min<long long>(rows - r0, PERF_STAGE_ROWS);
      SB_CUDA(cudaMemcpy2DAsync(ss, sizeof(float), scores + r0 * sp, sizeof(float) * sp, sizeof(float), static_cast<size_t>(c),
                                cudaMemcpyDefault, p->stream));
      SB_CUDA(cudaMemcpyAsync(sy, y + r0, sizeof(float) * c, cudaMemcpyDefault, p->stream));
      if (w) SB_CUDA(cudaMemcpyAsync(sw, w + r0, sizeof(float) * c, cudaMemcpyDefault, p->stream));
      SB_TRY(add(ss, 1, sy, w ? sw : nullptr, r0, c));
    }
    SB_CUDA(cudaStreamSynchronize(p->stream));
  }
  p->rows += rows;
  return SB_OK;
}

int sb_perf_summary_get(sb_perf_t* p, sb_perf_summary* out) {
  SB_CHECK(p, SB_ERR_STATE, "performance handle not initialized.");
  SB_CHECK(out, SB_ERR_INVALID, "out is null");
  SB_TRY(perf_prepare(p));
  const double qnan = std::numeric_limits<double>::quiet_NaN();
  sb_perf_summary s;
  s.rows = p->rows; s.pos = p->P; s.neg = p->N; s.n_distinct = p->m; s.w_pos = p->Wp; s.w_neg = p->Wn;
  s.auc = s.w_auc = s.ap = s.w_ap = s.ks = s.w_ks = qnan;
  s.ks_score = s.w_ks_score = std::numeric_limits<float>::quiet_NaN();
  if (p->m > 0) {
    const int G = static_cast<int>(std::min<long long>(PERF_SUM_BLOCKS, (p->m + PERF_THREADS - 1) / PERF_THREADS));
    SB_TRY(launch_kernel(perf_summary_kernel, dim3(G), dim3(PERF_THREADS), 0, p->stream, false, static_cast<const long long*>(p->rtp),
                         static_cast<const long long*>(p->rfp), static_cast<const double*>(p->rwtp),
                         static_cast<const double*>(p->rwfp), p->m, p->parts));
    SB_TRY(launch_kernel(perf_summary_final_kernel, dim3(1), dim3(1), 0, p->stream, false, static_cast<const PerfPart*>(p->parts), G,
                         static_cast<const float*>(p->rt), p->result));
    PerfResult r;
    SB_CUDA(cudaMemcpyAsync(&r, p->result, sizeof(r), cudaMemcpyDeviceToHost, p->stream));
    SB_CUDA(cudaStreamSynchronize(p->stream));
    const long long pn = p->P * p->N;
    const double wpn = p->Wp * p->Wn;
    if (pn > 0) {
      s.auc = static_cast<double>(r.a.a2) / static_cast<double>(2 * pn);
      s.ks = static_cast<double>(r.a.ks) / static_cast<double>(pn);
      s.ks_score = r.ks_t;
    }
    if (p->P > 0) s.ap = r.a.ap / static_cast<double>(p->P);
    if (wpn > 0.0) {
      s.w_auc = r.a.wauc / wpn;
      s.w_ks = r.a.wks / wpn;
      s.w_ks_score = r.wks_t;
    }
    if (p->Wp > 0.0) s.w_ap = r.a.wap / p->Wp;
  }
  *out = s;
  return SB_OK;
}

int sb_perf_points(sb_perf_t* p, int32_t axis, int32_t weighted, const double* levels, int32_t n, sb_perf_point* out) {
  SB_CHECK(p, SB_ERR_STATE, "performance handle not initialized.");
  SB_CHECK(axis >= SB_PERF_ACTION_RATE && axis <= SB_PERF_SCORE, SB_ERR_INVALID, "unknown axis %d", axis);
  SB_CHECK(n >= 0, SB_ERR_INVALID, "n = %d < 0", n);
  SB_CHECK(n == 0 || (levels && out), SB_ERR_INVALID, "levels and out must not be null");
  for (int i = 0; i < n; ++i) {
    SB_CHECK(!std::isnan(levels[i]), SB_ERR_INVALID, "level %d is NaN", i);
    SB_CHECK(axis == SB_PERF_SCORE || (levels[i] >= 0.0 && levels[i] <= 1.0), SB_ERR_INVALID, "level %d = %g outside [0, 1]", i,
             levels[i]);
  }
  SB_TRY(perf_prepare(p));
  if (n == 0) return SB_OK;
  double den = 1.0;
  if (axis != SB_PERF_SCORE) {
    den = weighted ? (axis == SB_PERF_ACTION_RATE ? p->Wp + p->Wn : axis == SB_PERF_RECALL ? p->Wp : p->Wn)
                   : static_cast<double>(axis == SB_PERF_ACTION_RATE ? p->P + p->N : axis == SB_PERF_RECALL ? p->P : p->N);
    SB_CHECK(den > 0.0, SB_ERR_INVALID, "the %s%s total is 0: the axis is undefined", weighted ? "weighted " : "",
             axis == SB_PERF_ACTION_RATE ? "row" : axis == SB_PERF_RECALL ? "positive" : "negative");
  }
  if (p->m == 0) {                     // score axis of an empty handle: every point is the empty point
    for (int i = 0; i < n; ++i) out[i] = sb_perf_point{std::numeric_limits<float>::infinity(), 0, 0, 0.0, 0.0};
    return SB_OK;
  }
  if (n > p->pt_cap) {                 // kept for the next call: an allocation here would synchronise the device
    p->release(&p->d_levels, p->pt_cap); p->release(&p->d_points, p->pt_cap);
    p->pt_cap = 0;
    SB_TRY(p->alloc(&p->d_levels, n)); SB_TRY(p->alloc(&p->d_points, n));
    p->pt_cap = n;
  }
  SB_CUDA(cudaMemcpyAsync(p->d_levels, levels, sizeof(double) * n, cudaMemcpyHostToDevice, p->stream));
  SB_TRY(launch_kernel(perf_points_kernel, dim3(static_cast<unsigned>((n + 127) / 128)), dim3(128), 0, p->stream, false,
                       static_cast<const float*>(p->rt), static_cast<const long long*>(p->rtp), static_cast<const long long*>(p->rfp),
                       static_cast<const double*>(p->rwtp), static_cast<const double*>(p->rwfp), p->m, static_cast<int>(axis),
                       weighted ? 1 : 0, den, static_cast<const double*>(p->d_levels), static_cast<int>(n), p->d_points));
  SB_CUDA(cudaMemcpyAsync(out, p->d_points, sizeof(sb_perf_point) * n, cudaMemcpyDeviceToHost, p->stream));
  SB_CUDA(cudaStreamSynchronize(p->stream));
  return SB_OK;
}

int sb_perf_sync(sb_perf_t* p) {
  SB_CHECK(p, SB_ERR_STATE, "performance handle not initialized.");
  SB_CUDA(cudaSetDevice(p->device));
  SB_CUDA(cudaStreamSynchronize(p->stream));
  return SB_OK;
}

void* sb_perf_stream(sb_perf_t* p) { return p ? reinterpret_cast<void*>(p->stream) : nullptr; }

int sb_debug_perf_runs(sb_perf_t* p, float* t, int64_t* tp, int64_t* fp, double* wtp, double* wfp, int64_t cap, int64_t* n_runs) {
  SB_CHECK(p, SB_ERR_STATE, "performance handle not initialized.");
  SB_CHECK(n_runs && cap >= 0, SB_ERR_INVALID, "null n_runs or cap < 0");
  SB_TRY(perf_prepare(p));
  const size_t c = static_cast<size_t>(std::min<long long>(cap, p->m));
  if (c > 0) {
    if (t) SB_CUDA(cudaMemcpyAsync(t, p->rt, sizeof(float) * c, cudaMemcpyDeviceToHost, p->stream));
    if (tp) SB_CUDA(cudaMemcpyAsync(tp, p->rtp, sizeof(int64_t) * c, cudaMemcpyDeviceToHost, p->stream));
    if (fp) SB_CUDA(cudaMemcpyAsync(fp, p->rfp, sizeof(int64_t) * c, cudaMemcpyDeviceToHost, p->stream));
    if (wtp) SB_CUDA(cudaMemcpyAsync(wtp, p->rwtp, sizeof(double) * c, cudaMemcpyDeviceToHost, p->stream));
    if (wfp) SB_CUDA(cudaMemcpyAsync(wfp, p->rwfp, sizeof(double) * c, cudaMemcpyDeviceToHost, p->stream));
    SB_CUDA(cudaStreamSynchronize(p->stream));
  }
  *n_runs = p->m;
  return SB_OK;
}

int sb_debug_perf_bytes(sb_perf_t* p, int64_t* out) {
  SB_CHECK(p, SB_ERR_STATE, "performance handle not initialized.");
  SB_CHECK(out, SB_ERR_INVALID, "null argument");
  *out = p->bytes;
  return SB_OK;
}

}  // extern "C"
