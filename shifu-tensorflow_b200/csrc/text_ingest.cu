// sb_text_parse: '|'-delimited normalised text -> fp32 feature matrix / target / weight on the GPU
// (replaces the per-cell Python float() loop of load_data, res/ssgd_monitor.py:387-419).  See text_parse.cuh.
#include <string.h>
#include <vector>
#include "common.cuh"
#include "text_parse.cuh"

namespace sb {

constexpr int NL_CHUNK = 16384;   // bytes per block in the newline passes (256 threads x 64 B)

// pass 1: newlines per 16 KB chunk
static __global__ void __launch_bounds__(256) count_newlines_kernel(const unsigned char* __restrict__ text, long long n,
                                                                    int* __restrict__ chunk_counts) {
  const long long base = static_cast<long long>(blockIdx.x) * NL_CHUNK + threadIdx.x * 64;
  int cnt = 0;
  if (base < n) {
#pragma unroll
    for (int q = 0; q < 4; ++q) {           // text is padded to a multiple of 16 KB, 16-byte loads are always in bounds
      const uint4 v = __ldg(reinterpret_cast<const uint4*>(text + base) + q);
      const unsigned int w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int b = 0; b < 4; ++b) {
          const long long p = base + q * 16 + i * 4 + b;
          cnt += (p < n && ((w[i] >> (8 * b)) & 0xFFu) == '\n') ? 1 : 0;
        }
    }
  }
  cnt = static_cast<int>(warp_sum(static_cast<float>(cnt)) + 0.5f);
  __shared__ int part[8];
  if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = cnt;
  __syncthreads();
  if (threadIdx.x == 0) {
    int s = 0;
    for (int i = 0; i < 8; ++i) s += part[i];
    chunk_counts[blockIdx.x] = s;
  }
}

// pass 2: line_start[k + 1] = position after the k-th newline (line_start[0] = 0 is written by the host)
static __global__ void __launch_bounds__(256) line_offsets_kernel(const unsigned char* __restrict__ text, long long n,
                                                                  const long long* __restrict__ chunk_base_line,
                                                                  long long* __restrict__ line_start) {
  const long long base = static_cast<long long>(blockIdx.x) * NL_CHUNK + threadIdx.x * 64;
  int cnt = 0;
  unsigned long long mask = 0;   // bit i set: byte i of this thread's 64 is a newline
  if (base < n) {
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const uint4 v = __ldg(reinterpret_cast<const uint4*>(text + base) + q);
      const unsigned int w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int b = 0; b < 4; ++b) {
          const int idx = q * 16 + i * 4 + b;
          if (base + idx < n && ((w[i] >> (8 * b)) & 0xFFu) == '\n') { mask |= 1ull << idx; ++cnt; }
        }
    }
  }
  // exclusive scan of cnt over the block
  __shared__ int sc[256];
  sc[threadIdx.x] = cnt;
  __syncthreads();
  for (int off = 1; off < 256; off <<= 1) {
    const int v = (threadIdx.x >= off) ? sc[threadIdx.x - off] : 0;
    __syncthreads();
    sc[threadIdx.x] += v;
    __syncthreads();
  }
  long long k = chunk_base_line[blockIdx.x] + (sc[threadIdx.x] - cnt);
  while (mask) {
    const int idx = __ffsll(static_cast<long long>(mask)) - 1;
    mask &= mask - 1;
    line_start[k + 1] = base + idx + 1;
    ++k;
  }
}

struct ParseArgs {
  const unsigned char* text;
  const long long* line_start;
  long long n_lines;
  const int* col_map;
  int n_map, n_feat;
  unsigned char delim;
  float *X, *y, *w;
  CellFlag* flags;
  long long flag_cap;
  unsigned long long* n_flags;
};

SB_HD void flag_cell(const ParseArgs& a, long long row, int slot, long long off, int len) {
#if defined(__CUDA_ARCH__)
  const unsigned long long i = atomicAdd(a.n_flags, 1ull);
#else
  const unsigned long long i = (*a.n_flags)++;
#endif
  if (static_cast<long long>(i) < a.flag_cap) { a.flags[i].row = row; a.flags[i].slot = slot; a.flags[i].len = len; a.flags[i].offset = off; }
}

// one line: shared by the device kernel and the host test hook
SB_HD void parse_line(const ParseArgs& a, long long row) {
  const long long start = a.line_start[row], end = a.line_start[row + 1] - 1;   // [start, end) excludes the '\n'
  NumState st;
  num_reset(st);
  int field = 0, n_feat_seen = 0;
  bool target_seen = false;
  int role = (a.n_map > 0) ? a.col_map[0] : SB_COL_SKIP;
  long long cell_start = start;
  float wv = 1.0f;
  auto finish = [&](long long pos) {
    if (role != SB_COL_SKIP) {
      float v;
      const bool ok = num_finish(st, &v);
      if (role >= 0) {
        ++n_feat_seen;
        if (ok) a.X[row * a.n_feat + role] = v; else flag_cell(a, row, role, cell_start, static_cast<int>(pos - cell_start));
      } else if (role == SB_COL_TARGET) {
        target_seen = true;
        if (ok) a.y[row] = v; else flag_cell(a, row, role, cell_start, static_cast<int>(pos - cell_start));
      } else {  // weight: negative -> 1.0 (ssgd_monitor.py:414-416)
        if (ok) wv = (v < 0.0f) ? 1.0f : v; else flag_cell(a, row, role, cell_start, static_cast<int>(pos - cell_start));
      }
    }
    ++field;
    role = (field < a.n_map) ? a.col_map[field] : SB_COL_SKIP;
    num_reset(st);
    cell_start = pos + 1;
  };
  long long pos = start;
  while (pos < end) {
    const long long cb = pos & ~15ll;
#if defined(__CUDA_ARCH__)
    const uint4 v = __ldg(reinterpret_cast<const uint4*>(a.text + cb));
    const unsigned int wd[4] = {v.x, v.y, v.z, v.w};
#else
    unsigned int wd[4];
    memcpy(wd, a.text + cb, 16);
#endif
#pragma unroll
    for (int b = 0; b < 16; ++b) {
      const long long p = cb + b;
      if (p < pos || p >= end) continue;
      const unsigned char c = static_cast<unsigned char>((wd[b >> 2] >> (8 * (b & 3))) & 0xFFu);
      if (c == a.delim) finish(p);
      else if (role != SB_COL_SKIP) num_feed(st, c);
    }
    pos = cb + 16;
  }
  finish(end);   // last cell of the line
  a.w[row] = wv; // no weight column / column beyond the line -> 1.0 (ssgd_monitor.py:412-419)
  if (n_feat_seen != a.n_feat || !target_seen) flag_cell(a, row, -100, start, static_cast<int>(end - start));
}

static __global__ void __launch_bounds__(128) parse_lines_kernel(const ParseArgs a) {
  const long long row = blockIdx.x * 128ll + threadIdx.x;
  if (row < a.n_lines) parse_line(a, row);
}

}  // namespace sb

using namespace sb;

static_assert(sizeof(sb_cell_flag) == sizeof(CellFlag), "flag layout");

// rows of a row-major fp32 matrix picked by index (train / valid split of the parsed set, on the device)
static __global__ void __launch_bounds__(256) gather_rows_kernel(const float* __restrict__ src, int n_cols, const long long* __restrict__ rows,
                                                                 long long n, float* __restrict__ dst) {
  const long long total = n * n_cols;
  for (long long i = blockIdx.x * 256ll + threadIdx.x; i < total; i += gridDim.x * 256ll) {
    const long long r = i / n_cols;
    dst[i] = __ldg(src + rows[r] * n_cols + (i - r * n_cols));
  }
}

static int check_args(const char* text, int64_t n_bytes, const int32_t* col_map, int32_t n_map, int32_t n_feat, const void* X, const void* y,
                      const void* w, int64_t* n_rows_out, int64_t* n_flags_out) {
  SB_CHECK(text && col_map && X && y && w && n_rows_out && n_flags_out, SB_ERR_INVALID, "null argument");
  SB_CHECK(n_bytes > 0 && n_map > 0 && n_feat > 0, SB_ERR_INVALID, "empty input");
  SB_CHECK(text[n_bytes - 1] == '\n', SB_ERR_INVALID, "text must end with a newline");
  // parse_line stores a feature cell at X[row * n_feat + role] unchecked: every role must name a column of X, and each
  // column exactly once (a repeated index would leave another column silently 0 with no line flagged)
  SB_CHECK(n_feat <= n_map, SB_ERR_INVALID, "col_map has %d entries, fewer than n_feat=%d features", n_map, n_feat);
  std::vector<char> seen(static_cast<size_t>(n_feat), 0);
  int n_seen = 0, n_target = 0, n_weight = 0;
  for (int32_t c = 0; c < n_map; ++c) {
    const int32_t r = col_map[c];
    SB_CHECK(r >= SB_COL_WEIGHT && r < n_feat, SB_ERR_INVALID, "col_map[%d] = %d outside [%d, n_feat=%d)", c, r, SB_COL_WEIGHT,
             n_feat);
    if (r >= 0) {
      SB_CHECK(!seen[static_cast<size_t>(r)], SB_ERR_INVALID, "col_map[%d]: feature %d is mapped twice", c, r);
      seen[static_cast<size_t>(r)] = 1;
      ++n_seen;
    } else if (r == SB_COL_TARGET) {
      ++n_target;
    } else if (r == SB_COL_WEIGHT) {
      ++n_weight;
    }
  }
  SB_CHECK(n_seen == n_feat, SB_ERR_INVALID, "col_map maps %d of n_feat=%d features", n_seen, n_feat);
  SB_CHECK(n_target == 1, SB_ERR_INVALID, "col_map has %d target columns, needs exactly one", n_target);
  SB_CHECK(n_weight <= 1, SB_ERR_INVALID, "col_map has %d weight columns, at most one", n_weight);
  return SB_OK;
}

// keep != nullptr: the parsed arrays stay on the device (keep[0..2] = X, y, w; caller frees with sb_device_free) and
// nothing but the flags travels back; kernel_ms (nullable) = device time of the three parsing kernels
static int text_parse_impl(const char* text, int64_t n_bytes, char delim, const int32_t* col_map, int32_t n_map, int32_t n_feat, float* X,
                           float* y, float* w, int64_t max_rows, int64_t* n_rows_out, sb_cell_flag* flags, int64_t flag_cap,
                           int64_t* n_flags_out, int device, float** keep, float* kernel_ms);

extern "C" {

int sb_text_parse(const char* text, int64_t n_bytes, char delim, const int32_t* col_map, int32_t n_map, int32_t n_feat, float* X,
                  float* y, float* w, int64_t max_rows, int64_t* n_rows_out, sb_cell_flag* flags, int64_t flag_cap,
                  int64_t* n_flags_out, int device) {
  SB_TRY(check_args(text, n_bytes, col_map, n_map, n_feat, X, y, w, n_rows_out, n_flags_out));
  return text_parse_impl(text, n_bytes, delim, col_map, n_map, n_feat, X, y, w, max_rows, n_rows_out, flags, flag_cap, n_flags_out, device,
                         nullptr, nullptr);
}

int sb_text_parse_device(const char* text, int64_t n_bytes, char delim, const int32_t* col_map, int32_t n_map, int32_t n_feat,
                         float** dX, float** dy, float** dw, int64_t* n_rows_out, sb_cell_flag* flags, int64_t flag_cap,
                         int64_t* n_flags_out, int device, float* kernel_ms_out) {
  SB_TRY(check_args(text, n_bytes, col_map, n_map, n_feat, dX, dy, dw, n_rows_out, n_flags_out));
  float* keep[3] = {nullptr, nullptr, nullptr};
  SB_TRY(text_parse_impl(text, n_bytes, delim, col_map, n_map, n_feat, nullptr, nullptr, nullptr, INT64_MAX, n_rows_out, flags, flag_cap,
                         n_flags_out, device, keep, kernel_ms_out));
  *dX = keep[0]; *dy = keep[1]; *dw = keep[2];
  return SB_OK;
}

int sb_device_free(void* p) {
  if (p) SB_CUDA(cudaFree(p));
  return SB_OK;
}

int sb_device_alloc_f32(float** out, int64_t n, int device) {
  SB_CHECK(out && n > 0, SB_ERR_INVALID, "bad argument");
  SB_CUDA(cudaSetDevice(device));
  void* q = nullptr;
  SB_CUDA(cudaMalloc(&q, sizeof(float) * static_cast<size_t>(n)));
  *out = static_cast<float*>(q);
  return SB_OK;
}

int sb_device_patch_f32(float* d_base, int64_t index, float value) {
  SB_CHECK(d_base && index >= 0, SB_ERR_INVALID, "bad argument");
  SB_CUDA(cudaMemcpy(d_base + index, &value, sizeof(float), cudaMemcpyHostToDevice));
  return SB_OK;
}

int sb_device_read_f32(const float* d_src, int64_t n, float* host_out) {
  SB_CHECK(d_src && host_out && n >= 0, SB_ERR_INVALID, "bad argument");
  SB_CUDA(cudaMemcpy(host_out, d_src, sizeof(float) * static_cast<size_t>(n), cudaMemcpyDeviceToHost));
  return SB_OK;
}

int sb_device_gather_rows(const float* d_src, int32_t n_cols, const int64_t* rows_host, int64_t n, float* d_dst, int device) {
  SB_CHECK(d_src && rows_host && d_dst && n_cols > 0 && n >= 0, SB_ERR_INVALID, "bad argument");
  if (n == 0) return SB_OK;
  SB_CUDA(cudaSetDevice(device));
  long long* d_rows = nullptr;
  SB_CUDA(cudaMalloc(&d_rows, sizeof(long long) * static_cast<size_t>(n)));
  cudaError_t e = cudaMemcpy(d_rows, rows_host, sizeof(long long) * static_cast<size_t>(n), cudaMemcpyHostToDevice);
  if (e == cudaSuccess) {
    long long blocks = (n * n_cols + 255) / 256;
    if (blocks > 132 * 32) blocks = 132 * 32;
    gather_rows_kernel<<<static_cast<unsigned>(blocks), 256>>>(d_src, n_cols, d_rows, n, d_dst);
    e = cudaGetLastError();
    if (e == cudaSuccess) e = cudaDeviceSynchronize();
  }
  cudaFree(d_rows);
  SB_CHECK(e == cudaSuccess, SB_ERR_CUDA, "gather_rows failed: %s", cudaGetErrorString(e));
  return SB_OK;
}

}  // extern "C"

static int text_parse_impl(const char* text, int64_t n_bytes, char delim, const int32_t* col_map, int32_t n_map, int32_t n_feat, float* X,
                           float* y, float* w, int64_t max_rows, int64_t* n_rows_out, sb_cell_flag* flags, int64_t flag_cap,
                           int64_t* n_flags_out, int device, float** keep, float* kernel_ms) {
  int n_dev = 0;
  SB_CHECK(cudaGetDeviceCount(&n_dev) == cudaSuccess && n_dev > 0, SB_ERR_CUDA,
           "no CUDA device available; this library has no CPU fallback");
  SB_CUDA(cudaSetDevice(device));
  const long long n_chunks = (n_bytes + NL_CHUNK - 1) / NL_CHUNK;
  const size_t padded = static_cast<size_t>(n_chunks) * NL_CHUNK + 16;
  unsigned char* d_text = nullptr;
  int* d_counts = nullptr;
  long long *d_base = nullptr, *d_lines = nullptr;
  int* d_map = nullptr;
  float *dX = nullptr, *dy = nullptr, *dw = nullptr;
  CellFlag* d_flags = nullptr;
  unsigned long long* d_nflags = nullptr;
  int s = SB_OK;
  cudaEvent_t ev[2] = {nullptr, nullptr};
  float k_ms = 0.f;
  auto cleanup = [&]() {
    cudaFree(d_text); cudaFree(d_counts); cudaFree(d_base); cudaFree(d_lines); cudaFree(d_map);
    cudaFree(dX); cudaFree(dy); cudaFree(dw); cudaFree(d_flags); cudaFree(d_nflags);
    if (ev[0]) cudaEventDestroy(ev[0]);
    if (ev[1]) cudaEventDestroy(ev[1]);
  };
  auto tick = [&](int i) { if (kernel_ms) { if (!ev[i]) cudaEventCreate(&ev[i]); cudaEventRecord(ev[i], 0); } };
  auto tock = [&]() { if (kernel_ms) { float m = 0.f; cudaEventSynchronize(ev[1]); cudaEventElapsedTime(&m, ev[0], ev[1]); k_ms += m; } };
#define SB_G(call) do { cudaError_t e_ = (call); if (e_ != cudaSuccess) { cleanup(); return set_error(SB_ERR_CUDA, "%s failed: %s", #call, cudaGetErrorString(e_)); } } while (0)
  SB_G(cudaMalloc(&d_text, padded));
  SB_G(cudaMemset(d_text + n_bytes, 0, padded - n_bytes));
  SB_G(cudaMemcpy(d_text, text, n_bytes, cudaMemcpyHostToDevice));
  SB_G(cudaMalloc(&d_counts, sizeof(int) * n_chunks));
  tick(0);
  count_newlines_kernel<<<static_cast<unsigned>(n_chunks), 256>>>(d_text, n_bytes, d_counts);
  tick(1); tock();
  std::vector<int> counts(static_cast<size_t>(n_chunks));
  SB_G(cudaMemcpy(counts.data(), d_counts, sizeof(int) * n_chunks, cudaMemcpyDeviceToHost));
  std::vector<long long> base(static_cast<size_t>(n_chunks));
  long long n_lines = 0;
  for (long long i = 0; i < n_chunks; ++i) { base[i] = n_lines; n_lines += counts[i]; }
  if (n_lines > max_rows) { cleanup(); return set_error(SB_ERR_INVALID, "%lld lines exceed max_rows=%lld", n_lines, (long long)max_rows); }
  SB_G(cudaMalloc(&d_base, sizeof(long long) * n_chunks));
  SB_G(cudaMemcpy(d_base, base.data(), sizeof(long long) * n_chunks, cudaMemcpyHostToDevice));
  SB_G(cudaMalloc(&d_lines, sizeof(long long) * (n_lines + 1)));
  SB_G(cudaMemset(d_lines, 0, sizeof(long long)));
  tick(0);
  line_offsets_kernel<<<static_cast<unsigned>(n_chunks), 256>>>(d_text, n_bytes, d_base, d_lines);
  tick(1); tock();
  SB_G(cudaMalloc(&d_map, sizeof(int) * n_map));
  SB_G(cudaMemcpy(d_map, col_map, sizeof(int) * n_map, cudaMemcpyHostToDevice));
  SB_G(cudaMalloc(&dX, sizeof(float) * n_lines * n_feat));
  SB_G(cudaMemset(dX, 0, sizeof(float) * n_lines * n_feat));
  SB_G(cudaMalloc(&dy, sizeof(float) * n_lines));
  SB_G(cudaMemset(dy, 0, sizeof(float) * n_lines));
  SB_G(cudaMalloc(&dw, sizeof(float) * n_lines));
  const long long cap = flag_cap > 0 ? flag_cap : 1;
  SB_G(cudaMalloc(&d_flags, sizeof(CellFlag) * cap));
  SB_G(cudaMalloc(&d_nflags, sizeof(unsigned long long)));
  SB_G(cudaMemset(d_nflags, 0, sizeof(unsigned long long)));
  ParseArgs a = {d_text, d_lines, n_lines, d_map, n_map, n_feat, static_cast<unsigned char>(delim), dX, dy, dw, d_flags,
                 flags ? flag_cap : 0, d_nflags};
  tick(0);
  if (n_lines > 0) parse_lines_kernel<<<static_cast<unsigned>((n_lines + 127) / 128), 128>>>(a);
  tick(1);
  SB_G(cudaGetLastError());
  SB_G(cudaDeviceSynchronize());
  tock();
  if (kernel_ms) *kernel_ms = k_ms;
  if (keep == nullptr) {
    SB_G(cudaMemcpy(X, dX, sizeof(float) * n_lines * n_feat, cudaMemcpyDeviceToHost));
    SB_G(cudaMemcpy(y, dy, sizeof(float) * n_lines, cudaMemcpyDeviceToHost));
    SB_G(cudaMemcpy(w, dw, sizeof(float) * n_lines, cudaMemcpyDeviceToHost));
  }
  unsigned long long nf = 0;
  SB_G(cudaMemcpy(&nf, d_nflags, sizeof(nf), cudaMemcpyDeviceToHost));
  if (flags && nf > 0) {
    const unsigned long long m = nf < static_cast<unsigned long long>(flag_cap) ? nf : flag_cap;
    SB_G(cudaMemcpy(flags, d_flags, sizeof(CellFlag) * m, cudaMemcpyDeviceToHost));
  }
#undef SB_G
  if (keep != nullptr) { keep[0] = dX; keep[1] = dy; keep[2] = dw; dX = dy = dw = nullptr; }   // ownership moves to the caller
  cleanup();
  *n_rows_out = n_lines;
  *n_flags_out = static_cast<int64_t>(nf);
  return s;
}

extern "C" {

// TEST HOOK: the identical state machine (text_parse.cuh / parse_line) executed on the host, so that the number
// parsing can be checked against Python's float() in the CPU test-suite.  Not a product path.
int sb_debug_text_parse_host(const char* text, int64_t n_bytes, char delim, const int32_t* col_map, int32_t n_map, int32_t n_feat,
                             float* X, float* y, float* w, int64_t max_rows, int64_t* n_rows_out, sb_cell_flag* flags,
                             int64_t flag_cap, int64_t* n_flags_out) {
  SB_TRY(check_args(text, n_bytes, col_map, n_map, n_feat, X, y, w, n_rows_out, n_flags_out));
  std::vector<unsigned char> padded(static_cast<size_t>(n_bytes) + 32, 0);
  memcpy(padded.data(), text, static_cast<size_t>(n_bytes));
  std::vector<long long> lines(1, 0);
  for (int64_t i = 0; i < n_bytes; ++i)
    if (text[i] == '\n') lines.push_back(i + 1);
  const long long n_lines = static_cast<long long>(lines.size()) - 1;
  SB_CHECK(n_lines <= max_rows, SB_ERR_INVALID, "%lld lines exceed max_rows=%lld", n_lines, (long long)max_rows);
  unsigned long long nf = 0;
  std::vector<CellFlag> dummy(1);
  ParseArgs a = {padded.data(), lines.data(), n_lines, col_map, n_map, n_feat, static_cast<unsigned char>(delim), X, y, w,
                 flags ? reinterpret_cast<CellFlag*>(flags) : dummy.data(), flags ? flag_cap : 0, &nf};
  for (long long i = 0; i < n_lines; ++i) for (int j = 0; j < n_feat; ++j) X[i * n_feat + j] = 0.f;
  for (long long r = 0; r < n_lines; ++r) { y[r] = 0.f; parse_line(a, r); }
  *n_rows_out = n_lines;
  *n_flags_out = static_cast<int64_t>(nf);
  return SB_OK;
}

}  // extern "C"
