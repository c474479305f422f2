// extern "C" surface of the scorers: the model (sb_model_*: scores, compute(), column sensitivity, reason codes) and the
// bagged ensemble (sb_ensemble_*, DESIGN §6h / §6j).  Both hold a ScoreCore: their members' nets, one forward of the
// members, the chunk loops, the compute() queue, the sensitivity loop and the launch routes.  See include/shifu_b200.h
// for the contract.
#include <string.h>
#include <algorithm>
#include <atomic>
#include <chrono>
#include <cmath>
#include <condition_variable>
#include <functional>
#include <memory>
#include "ensemble.cuh"
#include "net.cuh"
#include "savedmodel.h"
#include "score_rows.cuh"
#include "sensitivity.cuh"

using namespace sb;

// compute() (sb_model_score_row_f64) callers on one handle share device batches of up to MB_ROWS rows: the tensor-core
// kernels' tile height.  plan_gemm / plan_gemm_pp depend on M only through ceil(M / 128) and the grid size, so every GEMM
// plan of <= 128 rows is the one-row plan, and rows never interact in the forward GEMMs, the load or the output kernels:
// a row's score does not depend on which rows shared its batch.
static const int MB_ROWS = 128;
static_assert(SMALL_ROWS >= MB_ROWS, "an fp32 micro-batch is one score_rows_kernel launch");

struct RowWaiter {            // one compute() call, on its caller's stack
  float* out = nullptr;       // its result, RowQueue::words floats
  int status = SB_OK;
  std::string err;            // the leader's error text, re-raised in the caller's thread
  bool done = false;
};

// The compute() queue of a model (one score per row) or an ensemble (K scores and four statistics per row): concurrent
// callers on one handle share device batches of up to MB_ROWS rows.  No thread of its own: the first caller that finds
// no batch in flight leads, running every queued row in batches until the queue is empty; the others wait for their
// result.  A batch is run by the owner's run(b, rows): the rows of stage[b] -> res[b] [rows, words].
struct RowQueue {
  using Run = std::function<int(int, int)>;
  int F = 0, words = 1;
  std::mutex q_mu;
  std::condition_variable q_cv;
  float* stage[2] = {nullptr, nullptr};       // pinned [MB_ROWS, F]: one buffer fills while the other's batch runs
  float* res[2] = {nullptr, nullptr};         // pinned [MB_ROWS, words]
  RowWaiter* waiters[2][MB_ROWS] = {};
  int fill[2] = {0, 0};       // rows queued in a buffer
  int writers[2] = {0, 0};    // callers still converting their row into it
  int cur = 0;                // the buffer that takes new rows
  bool leading = false;
  int hold_k = 0, hold_ms = 0;                // sb_debug_model_hold
  std::atomic<long long> batches{0}, rows{0}, max_fill{0};   // since creation: batches run, their rows, the largest

  int alloc(int F_, int words_) {
    F = F_; words = words_;
    for (int b = 0; b < 2; ++b) {
      SB_CUDA(cudaHostAlloc(reinterpret_cast<void**>(&stage[b]), sizeof(float) * MB_ROWS * F, cudaHostAllocDefault));
      SB_CUDA(cudaHostAlloc(reinterpret_cast<void**>(&res[b]), sizeof(float) * MB_ROWS * words, cudaHostAllocDefault));
    }
    return SB_OK;
  }
  ~RowQueue() {
    for (int b = 0; b < 2; ++b) {
      if (stage[b]) cudaFreeHost(stage[b]);
      if (res[b]) cudaFreeHost(res[b]);
    }
  }

  // one row of F doubles (cast to float as TensorflowModel.java:64-68 casts it) -> out[words]
  int submit(const double* row, float* out, const Run& run) {
    RowWaiter me;
    me.out = out;
    std::unique_lock<std::mutex> lk(q_mu);
    q_cv.wait(lk, [&] { return fill[cur] < MB_ROWS; });
    const int b = cur, slot = fill[b]++;
    waiters[b][slot] = &me;
    ++writers[b];
    lk.unlock();
    float* f = stage[b] + static_cast<size_t>(slot) * F;
    for (int i = 0; i < F; ++i) f[i] = static_cast<float>(row[i]);
    lk.lock();
    if (--writers[b] == 0) q_cv.notify_all();
    while (!me.done) {
      if (!leading) {           // no batch in flight: lead (a lone caller is scored at once)
        leading = true;
        lead(lk, run);
        leading = false;
        q_cv.notify_all();
      } else {
        q_cv.wait(lk);
      }
    }
    lk.unlock();
    if (me.status != SB_OK) return set_error(me.status, "%s", me.err.c_str());
    return SB_OK;
  }

 private:
  // The leader (q_mu held through lk): runs the queued rows in batches until the queue is empty, and publishes each
  // caller's result and status.
  void lead(std::unique_lock<std::mutex>& lk, const Run& run) {
    while (fill[cur] > 0) {
      if (hold_k > 0) {         // sb_debug_model_hold: this batch waits for hold_k rows or the timeout
        const int k = hold_k;
        hold_k = 0;
        q_cv.wait_until(lk, std::chrono::steady_clock::now() + std::chrono::milliseconds(hold_ms), [&] { return fill[cur] >= k; });
      }
      const int b = cur;
      q_cv.wait(lk, [&] { return writers[b] == 0; });
      const int n = fill[b];
      cur ^= 1;                 // new rows go to the other buffer (empty: its batch was published before this one began)
      q_cv.notify_all();
      lk.unlock();
      const int s = run(b, n);
      const std::string err = s == SB_OK ? std::string() : last_error_ref();
      lk.lock();
      for (int i = 0; i < n; ++i) {
        RowWaiter* w = waiters[b][i];
        w->status = s;
        if (s == SB_OK) memcpy(w->out, res[b] + static_cast<size_t>(i) * words, sizeof(float) * words);
        else w->err = err;
        w->done = true;
      }
      fill[b] = 0;
      ++batches;
      rows += n;
      if (n > max_fill) max_fill = n;
      q_cv.notify_all();
    }
  }
};

static const int MODEL_CHUNK_ROWS = 16384;        // fp32 parity mode
static const int MODEL_CHUNK_ROWS_BF16 = 65536;   // bf16: bigger GEMMs per launch (workspace ~0.8 GB at 2000 cols)

static int model_chunk_rows(int precision) {
  return precision == SB_PREC_FP32 ? MODEL_CHUNK_ROWS : (precision == SB_PREC_BF16 ? MODEL_CHUNK_ROWS_BF16 : MODEL_CHUNK_ROWS_BF16 / 2);
}

// The scorer's load: `rows` staged fp32 rows X (weights w; nullptr weighs every row 1) described in the net's own slot, then
// load_batch_kernel into its layer-0 operand (Xb / Xf).  Scoring reads no descriptor field or step scalar besides what the
// load reads (the output layer runs without the loss).
static int load_rows(Net& n, const float* X, const float* w, int rows) {
  const StepIn in{n.desc, n.scal};
  const Batch b = host_batch(n, X, nullptr, w, rows);
  SB_TRY(write_desc(n.stream, in, &b, 0.f, 1.f, 0, nullptr));
  return n.enqueue_load(in, rows);
}

// One scoring member: a net and, in fp32, score_rows_kernel's activation buffers
struct Member {
  Net net;
  DevBuf<float> sr_act;       // fp32: score_rows_kernel's two activation buffers [SMALL_ROWS, sr_ld]
  int sr_ld = 0;

  // with input_from set, the net runs on that net's stream and reads its input staging
  int init(sb_net_desc d, const float* flat, int64_t n, int device, const Net* input_from) {
    d.max_batch = model_chunk_rows(d.precision);
    net.input_from = input_from;
    SB_TRY(net.init(&d, device, false));
    SB_CHECK(n == net.n_params, SB_ERR_INVALID, "expected %lld params, got %lld", (long long)net.n_params, (long long)n);
    SB_CUDA(cudaMemcpyAsync(net.theta, flat, sizeof(float) * n, cudaMemcpyHostToDevice, net.stream));
    SB_TRY(net.refresh_shadows());
    if (!net.tc()) {
      int widest = 1;
      for (int l = 0; l < net.L; ++l) widest = std::max(widest, net.layers[l].out);
      sr_ld = round_up(widest, 4);
      SB_TRY(sr_act.alloc(static_cast<size_t>(2) * SMALL_ROWS * sr_ld));
      SB_TRY(set_max_smem(score_rows_kernel, SR_SMEM));
    }
    SB_CUDA(cudaStreamSynchronize(net.stream));
    return SB_OK;
  }

  // The forward of `rows` (<= max_batch) device rows to scores dOut (device), queued on the net's stream.  An fp32 batch of
  // <= SMALL_ROWS rows is one score_rows_kernel launch that reads dX; any other batch runs the hidden-layer and output
  // launches, which read the operand load_rows filled (through member 0).  Both give the same bits.
  int enqueue(const float* dX, int rows, float* dOut) {
    Net& n = net;
    if (!n.tc() && rows <= SMALL_ROWS) {
      ScoreRowsParams p = {};
      p.rows = rows; p.F = n.F; p.L = n.L;
      p.X = dX; p.theta = n.theta;
      p.act[0] = sr_act.p; p.act[1] = sr_act.p + static_cast<size_t>(SMALL_ROWS) * sr_ld; p.ld_act = sr_ld;
      p.yhat = dOut;
      for (int l = 0; l < n.L; ++l) { p.out[l] = n.layers[l].out; p.act_fn[l] = n.layers[l].act; }
      for (int l = 0; l <= n.L; ++l) { p.w_off[l] = n.layers[l].w_off; p.b_off[l] = n.layers[l].b_off; }
      const int clusters = (rows + SR_ROWS - 1) / SR_ROWS;
      score_rows_kernel<<<clusters * SR_CLUSTER, SR_THREADS, SR_SMEM, n.stream>>>(p);
      SB_CUDA(cudaGetLastError());
      n.mark("score_rows");
      return SB_OK;
    }
    const StepIn in{n.desc, n.scal};
    SB_TRY(n.enqueue_hidden_forward(in, rows));
    return n.enqueue_out(in, rows, false, false, dOut, nullptr);
  }
};

// Column sensitivity's and reason codes' buffers (guarded by ScoreCore::mu), allocated by the first call and grown when a
// call needs more.  Only z is per member; the rest serves every member.
struct SensBufs {
  std::vector<DevBuf<float>> z;   // member g's layer-0 pre-activations of a row chunk [R, ld_out_0(g)]
  std::vector<size_t> z_n;
  DevBuf<double> acc;         // running sums [list position][w d^2, w d], then sum w
  DevBuf<int> cols;           // the column list and its values
  DevBuf<float> vals;
  DevBuf<float> d;            // the deltas of one piece [R, piece columns] (max_batch)
  DevBuf<float> stat;         // ensemble: the statistic of a piece's pair scores [max_batch], laid out like a model's yhat
  size_t acc_n = 0, cols_n = 0, vals_n = 0;
  DevBuf<float> reason_d;     // reason codes' running top k of a row chunk [R, k], best first
  DevBuf<int> reason_pos;
  size_t reason_d_n = 0, reason_pos_n = 0;
};

// What a model and an ensemble share.  Member 0 owns the stream and the input staging (stX, Xb / Xf); members 1 .. K-1
// borrow both (Net::input_from).  A chunk's results are outs[i] [max_batch, outs[i].words] on the device: a model's
// scores (1 word per row), or an ensemble's scores (K words) and statistics (4 words); a compute() row gets the words of
// every output, in order.
struct ScoreCore {
  struct Output { float* d = nullptr; int words = 0; };
  std::mutex mu;              // device work on the stream
  std::vector<std::unique_ptr<Member>> members;
  float* slots = nullptr;     // ensemble: [K, max_batch], member g's scores of a chunk at slots + g * max_batch
  Output outs[2];
  int n_outs = 0;
  RowQueue q;                 // compute()
  cudaGraphExec_t mb_graph = nullptr;         // tensor-core modes: the forward of MB_ROWS staged rows
  std::atomic<long long> st[SB_DEBUG_MSTAT_WORDS] = {};   // a model's counters (the first three words are the queue's)
  std::string routes;         // the launches of the last forward, "+"-joined (sb_debug_*_routes; guarded by mu)
  SensBufs sens;              // sensitivity and reason codes (freed after the destructor's wait)

  Net& lead() { return members[0]->net; }
  const Net& lead() const { return members[0]->net; }
  void wait() {
    if (members.empty() || !lead().stream) return;
    cudaSetDevice(lead().device);
    cudaStreamSynchronize(lead().stream);
  }
  ~ScoreCore() {
    wait();
    if (mb_graph) cudaGraphExecDestroy(mb_graph);
    while (!members.empty()) members.pop_back();   // member 0 last: the others run on its stream
  }

  int add_member(const sb_net_desc& d, const float* flat, int64_t n, int device) {
    std::unique_ptr<Member> m(new Member());
    SB_TRY(m->init(d, flat, n, device, members.empty() ? nullptr : &lead()));
    members.push_back(std::move(m));
    return SB_OK;
  }

  // f() with every member's launches kept in routes
  template <typename F>
  int routed(const F& f) {
    routes.clear();
    for (auto& m : members) m->net.marks = &routes;
    const int s = f();
    for (auto& m : members) m->net.marks = nullptr;
    return s;
  }

  // The forward of `rows` (<= max_batch) device rows dX into dst[i] (output i, nullable for an ensemble), queued on the
  // stream.  Tensor-core modes and fp32 chunks of more than SMALL_ROWS rows load the rows once through member 0; then every
  // member runs its forward, a model's straight into dst[0], an ensemble's into its slot, read by ensemble_stats_kernel.
  // Every scoring path comes through here.  Called with mu held.
  int forward(const float* dX, int rows, float* const* dst) {
    return routed([&]() -> int {
      Net& n0 = lead();
      const bool layered = n0.tc() || rows > SMALL_ROWS;
      if (layered) SB_TRY(load_rows(n0, dX, nullptr, rows));
      for (size_t g = 0; g < members.size(); ++g) {
        SB_TRY(members[g]->enqueue(dX, rows, slots ? slots + g * n0.max_batch : dst[0]));
        if (!layered) ++st[SB_DEBUG_MSTAT_SMALL_LAUNCHES];
      }
      if (!slots) return SB_OK;
      SB_TRY(launch_kernel(ensemble_stats_kernel, dim3(static_cast<unsigned>((rows + ENS_THREADS - 1) / ENS_THREADS)),
                           dim3(ENS_THREADS), 0, n0.stream, false, static_cast<const float*>(slots),
                           static_cast<long long>(n0.max_batch), static_cast<int>(members.size()), rows, dst[0], dst[1]));
      n0.mark("ensemble_stats");
      return SB_OK;
    });
  }

  // rows of host or device memory X, through the staging area in max_batch chunks, each chunk synchronised; output i to
  // host[i] [rows, outs[i].words] (host or device memory; nullable for an ensemble)
  int score(const float* X, int64_t rows, float* const* host) {
    std::lock_guard<std::mutex> lk(mu);
    Net& n = lead();
    SB_CUDA(cudaSetDevice(n.device));
    for (int64_t r0 = 0; r0 < rows; r0 += n.max_batch) {
      const int c = static_cast<int>(rows - r0 < n.max_batch ? rows - r0 : n.max_batch);
      SB_CUDA(cudaMemcpyAsync(n.stX, X + r0 * n.F, sizeof(float) * c * static_cast<size_t>(n.F), cudaMemcpyDefault, n.stream));
      float* dst[2] = {};
      for (int i = 0; i < n_outs; ++i) dst[i] = host[i] ? outs[i].d : nullptr;
      SB_TRY(forward(n.stX, c, dst));
      for (int i = 0; i < n_outs; ++i)
        if (host[i])
          SB_CUDA(cudaMemcpyAsync(host[i] + r0 * outs[i].words, outs[i].d, sizeof(float) * c * outs[i].words, cudaMemcpyDefault,
                                  n.stream));
      SB_CUDA(cudaStreamSynchronize(n.stream));
    }
    return SB_OK;
  }

  // device rows dX to device outputs dev[i] [rows, outs[i].words] (nullable for an ensemble), queued on the stream
  int score_device(const float* dX, int64_t rows, float* const* dev) {
    std::lock_guard<std::mutex> lk(mu);
    Net& n = lead();
    SB_CUDA(cudaSetDevice(n.device));
    for (int64_t r0 = 0; r0 < rows; r0 += n.max_batch) {
      const int c = static_cast<int>(rows - r0 < n.max_batch ? rows - r0 : n.max_batch);
      float* dst[2] = {};
      for (int i = 0; i < n_outs; ++i) dst[i] = dev[i] ? dev[i] + r0 * outs[i].words : nullptr;
      SB_TRY(forward(dX + r0 * n.F, c, dst));
    }
    return SB_OK;
  }

  // One compute() batch: rows of staging buffer b -> q.res[b] [rows, q.words].  A tensor-core batch runs the forward of
  // MB_ROWS rows captured once, its pad rows zero-filled; only the real rows are copied back, an output as wide as the
  // row in one copy.
  int run_micro_batch(int b, int rows) {
    std::lock_guard<std::mutex> lk(mu);
    Net& n = lead();
    SB_CUDA(cudaSetDevice(n.device));
    float* const dst[2] = {outs[0].d, outs[1].d};
    if (n.tc() && !mb_graph) {  // captured once, so that a micro-batch is one launch
      cudaGraph_t g = nullptr;
      SB_CUDA(cudaStreamBeginCapture(n.stream, cudaStreamCaptureModeThreadLocal));
      const int s = forward(n.stX, MB_ROWS, dst);
      const cudaError_t e = cudaStreamEndCapture(n.stream, &g);
      if (s != SB_OK) { if (g) cudaGraphDestroy(g); return s; }
      SB_CHECK(e == cudaSuccess, SB_ERR_CUDA, "cudaStreamEndCapture failed: %s", cudaGetErrorString(e));
      const cudaError_t ei = cudaGraphInstantiate(&mb_graph, g, 0);
      cudaGraphDestroy(g);
      SB_CHECK(ei == cudaSuccess, SB_ERR_CUDA, "cudaGraphInstantiate failed: %s", cudaGetErrorString(ei));
    }
    const size_t row_bytes = sizeof(float) * n.F;
    SB_CUDA(cudaMemcpyAsync(n.stX, q.stage[b], row_bytes * rows, cudaMemcpyHostToDevice, n.stream));
    if (n.tc()) {
      if (rows < MB_ROWS) SB_CUDA(cudaMemsetAsync(n.stX + static_cast<size_t>(rows) * n.F, 0, row_bytes * (MB_ROWS - rows), n.stream));
      SB_CUDA(cudaGraphLaunch(mb_graph, n.stream));
      ++st[SB_DEBUG_MSTAT_GRAPH];
    } else {
      SB_TRY(forward(n.stX, rows, dst));
      ++st[SB_DEBUG_MSTAT_SMALL];
    }
    float* res = q.res[b];
    for (int i = 0; i < n_outs; ++i) {
      const size_t w = sizeof(float) * outs[i].words;
      if (outs[i].words == q.words)
        SB_CUDA(cudaMemcpyAsync(res, outs[i].d, w * rows, cudaMemcpyDeviceToHost, n.stream));
      else
        SB_CUDA(cudaMemcpy2DAsync(res, sizeof(float) * q.words, outs[i].d, w, w, rows, cudaMemcpyDeviceToHost, n.stream));
      res += outs[i].words;
    }
    SB_CUDA(cudaStreamSynchronize(n.stream));
    return SB_OK;
  }

  // one row of F doubles -> out[q.words]
  int submit(const double* row, float* out) {
    return q.submit(row, out, [this](int b, int rows) { return run_micro_batch(b, rows); });
  }

  int sync() {
    SB_CUDA(cudaStreamSynchronize(lead().stream));
    return SB_OK;
  }

  int get_routes(char* out, int32_t cap) {
    SB_CHECK(out && cap > 0, SB_ERR_INVALID, "route buffer of %d bytes", cap);
    std::lock_guard<std::mutex> lk(mu);
    snprintf(out, static_cast<size_t>(cap), "%s", routes.empty() ? "none" : routes.c_str());
    return SB_OK;
  }

  long long bytes() const {
    long long b = 0;
    for (const auto& m : members) b += static_cast<long long>(m->net.dalloc_bytes);
    return b;
  }
};

// ================================================================================================
// model
// ================================================================================================
struct sb_model : ScoreCore {};

static int model_from_desc(const sb_net_desc& d, const float* flat, int64_t n, int device, sb_model_t** out) {
  std::unique_ptr<sb_model> m(new sb_model());
  SB_TRY(m->add_member(d, flat, n, device));
  m->outs[0] = {m->lead().yhat, 1};
  m->n_outs = 1;
  SB_TRY(m->q.alloc(m->lead().F, 1));
  *out = m.release();
  return SB_OK;
}

// A SavedModel directory -> the topology (at `precision`) and flat parameters of a scoring model; host work only.  The
// null checks mirror TensorflowModel.init (TensorflowModel.java:147-166).
static int read_scoring_model(const char* saved_model_dir, const char* input_name, const char* output_name, const char* tag,
                              int precision, sb_net_desc* d, std::vector<float>* flat) {
  SB_CHECK(saved_model_dir && saved_model_dir[0], SB_ERR_INVALID, "Model path is null");
  SB_CHECK(input_name && input_name[0], SB_ERR_INVALID, "Input names is null");
  SB_CHECK(output_name && output_name[0], SB_ERR_INVALID, "Output names is null");
  SB_CHECK(tag && tag[0], SB_ERR_INVALID, "Tags is null");
  memset(d, 0, sizeof(*d));
  int32_t out_act = SB_ACT_SIGMOID;
  int64_t np = 0;
  SB_TRY(sb_savedmodel_read(saved_model_dir, input_name, output_name, tag, d, &out_act, nullptr, 0, &np));
  SB_CHECK(out_act == SB_ACT_SIGMOID, SB_ERR_FORMAT, "output layer must be a sigmoid unit");
  flat->assign(static_cast<size_t>(np), 0.f);
  SB_TRY(sb_savedmodel_read(saved_model_dir, input_name, output_name, tag, d, &out_act, flat->data(), np, &np));
  d->precision = precision;
  d->max_batch = 1;
  return SB_OK;
}

extern "C" {

int sb_model_create(const sb_net_desc* desc, const float* flat_params, int64_t n, int device, sb_model_t** out) {
  SB_CHECK(out && flat_params, SB_ERR_INVALID, "null argument");
  *out = nullptr;
  sb_net_desc d = *desc;
  if (d.max_batch <= 0) d.max_batch = 1;
  SB_TRY(validate_desc(&d));
  return model_from_desc(d, flat_params, n, device, out);
}

int sb_model_load(const char* saved_model_dir, const char* input_name, const char* output_name, const char* tag,
                  int device, int precision, sb_model_t** out) {
  SB_CHECK(out, SB_ERR_INVALID, "out is null");
  *out = nullptr;
  sb_net_desc d;
  std::vector<float> flat;
  SB_TRY(read_scoring_model(saved_model_dir, input_name, output_name, tag, precision, &d, &flat));
  return model_from_desc(d, flat.data(), static_cast<int64_t>(flat.size()), device, out);
}

int sb_model_destroy(sb_model_t* m) {
  delete m;
  return SB_OK;
}

int32_t sb_model_n_features(const sb_model_t* m) { return m ? m->lead().F : 0; }
int32_t sb_model_n_layers(const sb_model_t* m) { return m ? m->lead().L + 1 : 0; }

int sb_model_score(sb_model_t* m, const float* X, int64_t rows, float* out) {
  SB_CHECK(m, SB_ERR_STATE, "TF model not initialized.");
  SB_CHECK(X && out, SB_ERR_INVALID, "null argument");
  if (rows <= 0) return SB_OK;
  return m->score(X, rows, &out);
}

int sb_model_score_row_f64(sb_model_t* m, const double* row, int32_t n, double* out) {
  SB_CHECK(m, SB_ERR_STATE, "TF model not initialized.");
  SB_CHECK(row && out, SB_ERR_INVALID, "null argument");
  SB_CHECK(n == m->lead().F, SB_ERR_INVALID, "expected %d features, got %d", m->lead().F, n);
  float v = 0.f;
  SB_TRY(m->submit(row, &v));
  *out = static_cast<double>(v);
  return SB_OK;
}

int sb_model_score_device(sb_model_t* m, const float* dX, int64_t rows, float* dOut) {
  SB_CHECK(m, SB_ERR_STATE, "TF model not initialized.");
  SB_CHECK(dX && dOut, SB_ERR_INVALID, "null argument");
  return m->score_device(dX, rows, &dOut);
}

}  // extern "C"

// Rows per row chunk for C list positions: max_batch / (C + 1), so that a row chunk's pairs fit one piece, but at least 64
// (more columns go in several pieces) and at most max_batch / 2
static int sens_chunk_rows(int max_batch, int C) {
  long long r = max_batch / (static_cast<long long>(C) + 1);
  if (r < 64) r = 64;
  if (r > max_batch / 2) r = max_batch / 2;
  return static_cast<int>(r > 0 ? r : 1);
}

template <typename T>
static int sens_grow(DevBuf<T>* b, size_t* cap, size_t n) {
  if (n <= *cap) return SB_OK;
  *b = DevBuf<T>();
  *cap = 0;
  SB_TRY(b->alloc(n));
  *cap = n;
  return SB_OK;
}

// Column sensitivity's pieces (sensitivity.cuh, DESIGN §6f / §6j), called with m->mu held.  Rows go in row chunks of R rows
// (sens_chunk_rows); a row chunk is loaded once through member 0 and each member's z0 is computed once, and its list
// positions go in pieces of up to max_batch / R - 1 columns.  A piece is, per member in member order, one forward of
// R (columns + 1) pair rows through its layers 1..L and output unit; a model's pair scores land in n.yhat, an
// ensemble's in its slots, of which ensemble_stat_kernel forms statistic `stat` as one column.  After each piece,
// piece(y, r0, rc, k0, ck, wd) consumes that column (pair p = slot * rc + r; wd: the chunk's weights): the sums and
// deltas of sensitivity, or the top-k merge of reason codes.
template <typename Piece>
static int sens_forward(ScoreCore* m, int stat, const float* X, const float* w, int64_t rows, int C, const Piece& piece) {
  Net& n = m->lead();
  const int K = static_cast<int>(m->members.size());
  const int R = sens_chunk_rows(n.max_batch, C);
  const int Cp = n.max_batch / R - 1;
  SensBufs& sb = m->sens;
  sb.z.resize(static_cast<size_t>(K));
  sb.z_n.resize(static_cast<size_t>(K));
  using PerturbFn = void (*)(SensParams);
  std::vector<SensParams> sp(static_cast<size_t>(K));
  std::vector<PerturbFn> perturb(static_cast<size_t>(K));
  std::vector<const char*> perturb_name(static_cast<size_t>(K));
  for (int g = 0; g < K; ++g) {
    Net& ng = m->members[g]->net;
    const Layer& l0 = ng.layers[0];
    SB_TRY(sens_grow(&sb.z[g], &sb.z_n[g], static_cast<size_t>(R) * l0.ld_out));
    SensParams& p = sp[g];
    p = {};
    p.F = ng.F; p.N = l0.out; p.ld = l0.ld_out;
    p.X = n.stX;
    p.z = sb.z[g].p;
    p.act = l0.act;
    if (ng.tc()) {
      p.bias = ng.theta + l0.b_off;
      p.Wn = l0.Wn; p.w_ps = ng.Wn_ps[0];
      p.out = ng.A[0]; p.out_ps = ng.A_ps[0];
    } else {
      p.W32 = ng.theta + l0.w_off;
      p.out32 = ng.Af[0];
    }
    perturb[g] = !ng.tc() ? sens_perturb_kernel<false, 1>
                 : ng.nparts == 3 ? sens_perturb_kernel<true, 3>
                 : ng.nparts == 2 ? sens_perturb_kernel<true, 2> : sens_perturb_kernel<true, 1>;
    perturb_name[g] = !ng.tc() ? "sens_perturb<fp32>"
                      : ng.nparts == 3 ? "sens_perturb<bf16x3>"
                      : ng.nparts == 2 ? "sens_perturb<bf16x2>" : "sens_perturb<bf16>";
  }
  if (m->slots && !sb.stat.p) SB_TRY(sb.stat.alloc(static_cast<size_t>(n.max_batch)));
  float* const y = m->slots ? sb.stat.p : n.yhat;
  const size_t row_bytes = sizeof(float) * n.F;
  for (int64_t r0 = 0; r0 < rows; r0 += R) {
    const int rc = static_cast<int>(rows - r0 < R ? rows - r0 : R);
    SB_CUDA(cudaMemcpyAsync(n.stX, X + r0 * n.F, row_bytes * rc, cudaMemcpyDefault, n.stream));
    if (w) SB_CUDA(cudaMemcpyAsync(n.stW, w + r0, sizeof(float) * rc, cudaMemcpyDefault, n.stream));
    const float* wd = w ? n.stW : n.ones;
    m->routes.clear();
    SB_TRY(load_rows(n, n.stX, wd, rc));
    for (int g = 0; g < K; ++g) {
      Net& ng = m->members[g]->net;
      SB_TRY(ng.enqueue_layer0_pre(StepIn{ng.desc, ng.scal}, rc, sb.z[g].p, ng.layers[0].ld_out));
      sp[g].R = rc;
    }
    const std::string prefix = m->routes;
    for (int k0 = 0; k0 < C; k0 += Cp) {
      const int ck = C - k0 < Cp ? C - k0 : Cp;
      const int pairs = rc * (ck + 1);
      m->routes = prefix;
      for (int g = 0; g < K; ++g) {
        Net& ng = m->members[g]->net;
        const StepIn in{ng.desc, ng.scal};
        sp[g].cols = sb.cols.p + k0; sp[g].vals = sb.vals.p + k0;
        const dim3 grid(static_cast<unsigned>((sp[g].N + 255) / 256), static_cast<unsigned>(ck + 1),
                        static_cast<unsigned>((rc + SENS_ROWS - 1) / SENS_ROWS));
        SB_TRY(launch_kernel(perturb[g], grid, dim3(32, 8), 0, ng.stream, false, sp[g]));
        ng.mark(perturb_name[g]);
        SB_TRY(ng.enqueue_hidden_forward(in, pairs, nullptr, nullptr, nullptr, 0, 1));
        SB_TRY(ng.enqueue_out(in, pairs, false, false, m->slots ? m->slots + static_cast<size_t>(g) * n.max_batch : n.yhat, nullptr));
      }
      if (m->slots) {
        SB_TRY(launch_kernel(ensemble_stat_kernel, dim3(static_cast<unsigned>((pairs + ENS_THREADS - 1) / ENS_THREADS)),
                             dim3(ENS_THREADS), 0, n.stream, false, static_cast<const float*>(m->slots),
                             static_cast<long long>(n.max_batch), K, pairs, stat, y));
        n.mark("ensemble_stat");
      }
      SB_TRY(piece(static_cast<const float*>(y), r0, rc, k0, ck, wd));
    }
  }
  return SB_OK;
}

// cols / n_cols / values as sb_model_sensitivity takes them -> the column list and its values (cl, vl)
static int sens_list(const Net& n, const int32_t* cols, int32_t n_cols, const float* values, std::vector<int32_t>* cl,
                     std::vector<float>* vl) {
  SB_CHECK((cols == nullptr && n_cols == 0) || (cols != nullptr && n_cols >= 1), SB_ERR_INVALID,
           "cols / n_cols: a list of n_cols >= 1 columns, or NULL and 0 for every column (got %s and %d)", cols ? "a list" : "NULL",
           n_cols);
  const int C = cols ? n_cols : n.F;
  cl->resize(static_cast<size_t>(C));
  vl->resize(static_cast<size_t>(C));
  for (int k = 0; k < C; ++k) {
    (*cl)[k] = cols ? cols[k] : k;
    SB_CHECK((*cl)[k] >= 0 && (*cl)[k] < n.F, SB_ERR_INVALID, "cols[%d] = %d outside [0, %d)", k, (*cl)[k], n.F);
    (*vl)[k] = values ? values[k] : 0.f;
    SB_CHECK(std::isfinite((*vl)[k]), SB_ERR_INVALID, "values[%d] = %g is not finite", k, static_cast<double>((*vl)[k]));
  }
  return SB_OK;
}

// the column list and its values to the device (with m->mu held); the running sums are sized with them
static int sens_upload_list(ScoreCore* m, const std::vector<int32_t>& cl, const std::vector<float>& vl) {
  Net& n = m->lead();
  SensBufs& sb = m->sens;
  const size_t list_n = cl.size();
  SB_TRY(sens_grow(&sb.acc, &sb.acc_n, 2 * list_n + 1));
  SB_TRY(sens_grow(&sb.cols, &sb.cols_n, list_n));
  SB_TRY(sens_grow(&sb.vals, &sb.vals_n, list_n));
  SB_CUDA(cudaMemcpyAsync(sb.cols.p, cl.data(), sizeof(int32_t) * list_n, cudaMemcpyHostToDevice, n.stream));
  SB_CUDA(cudaMemcpyAsync(sb.vals.p, vl.data(), sizeof(float) * list_n, cudaMemcpyHostToDevice, n.stream));
  return SB_OK;
}

// sb_model_sensitivity / sb_ensemble_sensitivity after the handle's checks (stat: an ensemble's statistic)
static int sensitivity(ScoreCore* m, int stat, const float* X, const float* w, int64_t rows, const int32_t* cols, int32_t n_cols,
                       const float* values, double* sum_sq, double* sum, double* w_sum, float* deltas) {
  SB_CHECK(X && sum_sq && sum && w_sum, SB_ERR_INVALID, "null argument");
  SB_CHECK(rows >= 0, SB_ERR_INVALID, "rows = %lld < 0", static_cast<long long>(rows));
  Net& n = m->lead();
  std::vector<int32_t> cl;
  std::vector<float> vl;
  SB_TRY(sens_list(n, cols, n_cols, values, &cl, &vl));
  const int C = static_cast<int>(cl.size());
  for (int k = 0; k < C; ++k) sum_sq[k] = sum[k] = 0.0;
  *w_sum = 0.0;
  if (rows == 0) return SB_OK;
  std::lock_guard<std::mutex> lk(m->mu);
  SB_CUDA(cudaSetDevice(n.device));
  SensBufs& sb = m->sens;
  const size_t list_n = static_cast<size_t>(C);
  SB_TRY(sens_upload_list(m, cl, vl));
  SB_CUDA(cudaMemsetAsync(sb.acc.p, 0, sizeof(double) * (2 * list_n + 1), n.stream));
  if (!sb.d.p) SB_TRY(sb.d.alloc(static_cast<size_t>(n.max_batch)));
  // per piece: d and the sums (sens_reduce_kernel), and the piece's deltas copied out when asked
  const auto reduce = [&](const float* y, int64_t r0, int rc, int k0, int ck, const float* wd) -> int {
    SB_TRY(launch_kernel(sens_reduce_kernel, dim3(static_cast<unsigned>(ck + 1)), dim3(SENS_REDUCE_THREADS), 0, n.stream, false, y,
                         wd, rc, ck, k0, deltas ? sb.d.p : nullptr, ck, sb.acc.p, k0 == 0 ? 1 : 0, 2LL * C));
    n.mark("sens_reduce");
    if (deltas)
      SB_CUDA(cudaMemcpy2DAsync(deltas + r0 * C + k0, sizeof(float) * C, sb.d.p, sizeof(float) * ck, sizeof(float) * ck, rc,
                                cudaMemcpyDefault, n.stream));
    return SB_OK;
  };
  SB_TRY(m->routed([&] { return sens_forward(m, stat, X, w, rows, C, reduce); }));
  std::vector<double> acc(2 * list_n + 1);
  SB_CUDA(cudaMemcpyAsync(acc.data(), sb.acc.p, sizeof(double) * acc.size(), cudaMemcpyDeviceToHost, n.stream));
  SB_CUDA(cudaStreamSynchronize(n.stream));
  for (int k = 0; k < C; ++k) { sum_sq[k] = acc[2 * k]; sum[k] = acc[2 * k + 1]; }
  *w_sum = acc[2 * list_n];
  return SB_OK;
}

// sb_model_reason_codes / sb_ensemble_reason_codes after the handle's checks (stat: an ensemble's statistic)
static int reason_codes(ScoreCore* m, int stat, const float* X, int64_t rows, const int32_t* cols, int32_t n_cols,
                        const float* values, int32_t k, int32_t order, int32_t* pos, float* d, float* scores) {
  SB_CHECK(X && pos && d, SB_ERR_INVALID, "null argument");
  SB_CHECK(rows >= 0, SB_ERR_INVALID, "rows = %lld < 0", static_cast<long long>(rows));
  Net& n = m->lead();
  std::vector<int32_t> cl;
  std::vector<float> vl;
  SB_TRY(sens_list(n, cols, n_cols, values, &cl, &vl));
  const int C = static_cast<int>(cl.size());
  SB_CHECK(k >= 1 && k <= C && k <= SENS_TOPK_MAX_K, SB_ERR_INVALID, "k = %d outside [1, min(%d list positions, %d)]", k, C,
           SENS_TOPK_MAX_K);
  SB_CHECK(order == SB_REASON_RAISE || order == SB_REASON_LOWER || order == SB_REASON_MAGNITUDE, SB_ERR_INVALID,
           "order = %d is not SB_REASON_RAISE, SB_REASON_LOWER or SB_REASON_MAGNITUDE", order);
  if (rows == 0) return SB_OK;
  std::lock_guard<std::mutex> lk(m->mu);
  SB_CUDA(cudaSetDevice(n.device));
  SensBufs& sb = m->sens;
  SB_TRY(sens_upload_list(m, cl, vl));
  const size_t run_n = static_cast<size_t>(sens_chunk_rows(n.max_batch, C)) * k;
  SB_TRY(sens_grow(&sb.reason_d, &sb.reason_d_n, run_n));
  SB_TRY(sens_grow(&sb.reason_pos, &sb.reason_pos_n, run_n));
  // per piece: merge its deltas into each row's running top k (reset by the chunk's first piece); after the chunk's last
  // piece, copy the chunk's top k and base scores out
  const auto merge = [&](const float* y, int64_t r0, int rc, int k0, int ck, const float*) -> int {
    const unsigned warps = static_cast<unsigned>(std::min((ck + 31) / 32, SENS_TOPK_WARPS));
    SB_TRY(launch_kernel(sens_topk_kernel, dim3(static_cast<unsigned>(rc)), dim3(32, warps), 0, n.stream, false, y, rc, ck, k0,
                         static_cast<int>(k), static_cast<int>(order), k0 == 0 ? 1 : 0, sb.reason_d.p, sb.reason_pos.p));
    n.mark("sens_topk");
    if (k0 + ck < C) return SB_OK;
    const size_t out_n = static_cast<size_t>(rc) * k;
    SB_CUDA(cudaMemcpyAsync(pos + r0 * k, sb.reason_pos.p, sizeof(int32_t) * out_n, cudaMemcpyDefault, n.stream));
    SB_CUDA(cudaMemcpyAsync(d + r0 * k, sb.reason_d.p, sizeof(float) * out_n, cudaMemcpyDefault, n.stream));
    if (scores) SB_CUDA(cudaMemcpyAsync(scores + r0, y, sizeof(float) * rc, cudaMemcpyDefault, n.stream));
    return SB_OK;
  };
  SB_TRY(m->routed([&] { return sens_forward(m, stat, X, nullptr, rows, C, merge); }));
  SB_CUDA(cudaStreamSynchronize(n.stream));
  return SB_OK;
}

extern "C" {

int sb_model_sensitivity(sb_model_t* m, const float* X, const float* w, int64_t rows, const int32_t* cols, int32_t n_cols,
                         const float* values, double* sum_sq, double* sum, double* w_sum, float* deltas) {
  SB_CHECK(m, SB_ERR_STATE, "TF model not initialized.");
  return sensitivity(m, SB_STAT_MEAN, X, w, rows, cols, n_cols, values, sum_sq, sum, w_sum, deltas);
}

int sb_model_reason_codes(sb_model_t* m, const float* X, int64_t rows, const int32_t* cols, int32_t n_cols, const float* values,
                          int32_t k, int32_t order, int32_t* pos, float* d, float* scores) {
  SB_CHECK(m, SB_ERR_STATE, "TF model not initialized.");
  return reason_codes(m, SB_STAT_MEAN, X, rows, cols, n_cols, values, k, order, pos, d, scores);
}

int sb_model_sync(sb_model_t* m) {
  SB_CHECK(m, SB_ERR_STATE, "TF model not initialized.");
  return m->sync();
}
void* sb_model_stream(sb_model_t* m) { return m ? reinterpret_cast<void*>(m->lead().stream) : nullptr; }

int sb_debug_model_batch_stats(sb_model_t* m, int64_t* stats, int32_t n_stats) {
  SB_CHECK(m, SB_ERR_STATE, "TF model not initialized.");
  SB_CHECK(stats && n_stats >= SB_DEBUG_MSTAT_WORDS, SB_ERR_INVALID, "stats needs %d words, got %d", SB_DEBUG_MSTAT_WORDS, n_stats);
  for (int i = 0; i < SB_DEBUG_MSTAT_WORDS; ++i) stats[i] = m->st[i].load();
  stats[SB_DEBUG_MSTAT_BATCHES] = m->q.batches.load();
  stats[SB_DEBUG_MSTAT_ROWS] = m->q.rows.load();
  stats[SB_DEBUG_MSTAT_MAX_FILL] = m->q.max_fill.load();
  return SB_OK;
}

int sb_debug_model_routes(sb_model_t* m, char* out, int32_t cap) {
  SB_CHECK(m, SB_ERR_STATE, "TF model not initialized.");
  return m->get_routes(out, cap);
}

int sb_debug_model_hold(sb_model_t* m, int32_t k, int32_t timeout_ms) {
  SB_CHECK(m, SB_ERR_STATE, "TF model not initialized.");
  SB_CHECK(k >= 0 && k <= MB_ROWS && timeout_ms >= 0, SB_ERR_INVALID, "k = %d outside [0, %d] or timeout_ms = %d < 0", k, MB_ROWS,
           timeout_ms);
  std::lock_guard<std::mutex> lk(m->q.q_mu);
  m->q.hold_k = k;
  m->q.hold_ms = timeout_ms;
  return SB_OK;
}

int sb_debug_model_bytes(sb_model_t* m, int64_t* out) {
  SB_CHECK(m, SB_ERR_STATE, "TF model not initialized.");
  SB_CHECK(out, SB_ERR_INVALID, "null argument");
  *out = static_cast<int64_t>(m->bytes());
  return SB_OK;
}

}  // extern "C"

// ================================================================================================
// ensemble: K member models on one stream that share one staged copy of the rows (DESIGN §6h)
// ================================================================================================
struct sb_ensemble : ScoreCore {};

// the flat parameter count of a topology (what Net::init lays out)
static long long desc_param_count(const sb_net_desc& d) {
  long long np = 0;
  int prev = d.n_features;
  for (int l = 0; l <= d.n_hidden; ++l) {
    const int out = l < d.n_hidden ? d.hidden[l] : 1;
    np += static_cast<long long>(prev) * out + out;
    prev = out;
  }
  return np;
}

// K checked descriptors (n_features and precision shared) and their parameters -> an ensemble
static int ensemble_from_descs(const std::vector<sb_net_desc>& ds, const float* const* flats, const int64_t* n_params, int device,
                               sb_ensemble_t** out) {
  std::unique_ptr<sb_ensemble> e(new sb_ensemble());
  const int K = static_cast<int>(ds.size());
  for (int g = 0; g < K; ++g) SB_TRY(e->add_member(ds[g], flats[g], n_params[g], device));
  Net& n0 = e->lead();
  SB_TRY(n0.dalloc(&e->slots, static_cast<size_t>(K) * n0.max_batch));
  SB_TRY(n0.dalloc(&e->outs[0].d, static_cast<size_t>(n0.max_batch) * K));
  SB_TRY(n0.dalloc(&e->outs[1].d, static_cast<size_t>(n0.max_batch) * 4));
  e->outs[0].words = K;
  e->outs[1].words = 4;
  e->n_outs = 2;
  SB_TRY(e->q.alloc(n0.F, K + 4));
  SB_CUDA(cudaStreamSynchronize(n0.stream));
  *out = e.release();
  return SB_OK;
}

static int check_ensemble_k(int32_t k) {
  SB_CHECK(k >= 1 && k <= SB_ENSEMBLE_MAX, SB_ERR_INVALID, "k = %d members outside [1, %d]", k, SB_ENSEMBLE_MAX);
  return SB_OK;
}

static int check_ensemble_members(const std::vector<sb_net_desc>& ds) {
  for (size_t g = 1; g < ds.size(); ++g) {
    SB_CHECK(ds[g].n_features == ds[0].n_features, SB_ERR_INVALID, "member %d has %d features, member 0 has %d", static_cast<int>(g),
             ds[g].n_features, ds[0].n_features);
    SB_CHECK(ds[g].precision == ds[0].precision, SB_ERR_INVALID, "member %d has precision %d, member 0 has %d", static_cast<int>(g),
             ds[g].precision, ds[0].precision);
  }
  return SB_OK;
}

extern "C" {

int sb_ensemble_create(const sb_net_desc* descs, const float* const* flats, const int64_t* n_params, int32_t k, int device,
                       sb_ensemble_t** out) {
  SB_CHECK(out, SB_ERR_INVALID, "out is null");
  *out = nullptr;
  SB_TRY(check_ensemble_k(k));
  SB_CHECK(descs && flats && n_params, SB_ERR_INVALID, "null argument");
  std::vector<sb_net_desc> ds(descs, descs + k);
  for (int g = 0; g < k; ++g) {
    SB_CHECK(flats[g], SB_ERR_INVALID, "flats[%d] is null", g);
    if (ds[g].max_batch <= 0) ds[g].max_batch = 1;
    SB_TRY(validate_desc(&ds[g]));
    const long long np = desc_param_count(ds[g]);
    SB_CHECK(n_params[g] == np, SB_ERR_INVALID, "member %d: expected %lld params, got %lld", g, np, static_cast<long long>(n_params[g]));
  }
  SB_TRY(check_ensemble_members(ds));
  return ensemble_from_descs(ds, flats, n_params, device, out);
}

int sb_ensemble_load(const char* const* dirs, int32_t k, const char* input_name, const char* output_name, const char* tag,
                     int device, int precision, sb_ensemble_t** out) {
  SB_CHECK(out, SB_ERR_INVALID, "out is null");
  *out = nullptr;
  SB_TRY(check_ensemble_k(k));
  SB_CHECK(dirs, SB_ERR_INVALID, "dirs is null");
  std::vector<sb_net_desc> ds(static_cast<size_t>(k));
  std::vector<std::vector<float>> flat(static_cast<size_t>(k));
  for (int g = 0; g < k; ++g) SB_TRY(read_scoring_model(dirs[g], input_name, output_name, tag, precision, &ds[g], &flat[g]));
  SB_TRY(check_ensemble_members(ds));
  std::vector<const float*> fp(static_cast<size_t>(k));
  std::vector<int64_t> np(static_cast<size_t>(k));
  for (int g = 0; g < k; ++g) { fp[g] = flat[g].data(); np[g] = static_cast<int64_t>(flat[g].size()); }
  return ensemble_from_descs(ds, fp.data(), np.data(), device, out);
}

int sb_ensemble_destroy(sb_ensemble_t* e) {
  delete e;
  return SB_OK;
}

int32_t sb_ensemble_size(const sb_ensemble_t* e) { return e ? static_cast<int32_t>(e->members.size()) : 0; }

// the argument checks every scoring entry point shares
static int check_ensemble_score(const sb_ensemble* e, const float* X, int64_t rows, const float* scores, const float* stats) {
  SB_CHECK(e, SB_ERR_STATE, "TF ensemble not initialized.");
  SB_CHECK(X, SB_ERR_INVALID, "X is null");
  SB_CHECK(scores || stats, SB_ERR_INVALID, "scores and stats are both null");
  SB_CHECK(rows >= 0, SB_ERR_INVALID, "rows = %lld < 0", static_cast<long long>(rows));
  return SB_OK;
}

int sb_ensemble_score(sb_ensemble_t* e, const float* X, int64_t rows, float* scores, float* stats) {
  SB_TRY(check_ensemble_score(e, X, rows, scores, stats));
  if (rows == 0) return SB_OK;
  float* const host[2] = {scores, stats};
  return e->score(X, rows, host);
}

int sb_ensemble_score_device(sb_ensemble_t* e, const float* dX, int64_t rows, float* dScores, float* dStats) {
  SB_TRY(check_ensemble_score(e, dX, rows, dScores, dStats));
  float* const dev[2] = {dScores, dStats};
  return e->score_device(dX, rows, dev);
}

int sb_ensemble_score_row_f64(sb_ensemble_t* e, const double* row, int32_t n, double* out) {
  SB_CHECK(e, SB_ERR_STATE, "TF ensemble not initialized.");
  SB_CHECK(row && out, SB_ERR_INVALID, "null argument");
  SB_CHECK(n == e->q.F, SB_ERR_INVALID, "expected %d features, got %d", e->q.F, n);
  float v[SB_ENSEMBLE_MAX + 4];
  SB_TRY(e->submit(row, v));
  for (int i = 0; i < e->q.words; ++i) out[i] = static_cast<double>(v[i]);
  return SB_OK;
}

static int check_ensemble_stat(const sb_ensemble* e, int32_t stat) {
  SB_CHECK(e, SB_ERR_STATE, "TF ensemble not initialized.");
  SB_CHECK(stat >= SB_STAT_MEAN && stat <= SB_STAT_MEDIAN, SB_ERR_INVALID,
           "stat = %d is not SB_STAT_MEAN, SB_STAT_MAX, SB_STAT_MIN or SB_STAT_MEDIAN", stat);
  return SB_OK;
}

int sb_ensemble_sensitivity(sb_ensemble_t* e, int32_t stat, const float* X, const float* w, int64_t rows, const int32_t* cols,
                            int32_t n_cols, const float* values, double* sum_sq, double* sum, double* w_sum, float* deltas) {
  SB_TRY(check_ensemble_stat(e, stat));
  return sensitivity(e, stat, X, w, rows, cols, n_cols, values, sum_sq, sum, w_sum, deltas);
}

int sb_ensemble_reason_codes(sb_ensemble_t* e, int32_t stat, const float* X, int64_t rows, const int32_t* cols, int32_t n_cols,
                             const float* values, int32_t k, int32_t order, int32_t* pos, float* d, float* scores) {
  SB_TRY(check_ensemble_stat(e, stat));
  return reason_codes(e, stat, X, rows, cols, n_cols, values, k, order, pos, d, scores);
}

int sb_ensemble_sync(sb_ensemble_t* e) {
  SB_CHECK(e, SB_ERR_STATE, "TF ensemble not initialized.");
  return e->sync();
}

void* sb_ensemble_stream(sb_ensemble_t* e) { return e ? reinterpret_cast<void*>(e->lead().stream) : nullptr; }

int sb_debug_ensemble_routes(sb_ensemble_t* e, char* out, int32_t cap) {
  SB_CHECK(e, SB_ERR_STATE, "TF ensemble not initialized.");
  return e->get_routes(out, cap);
}

int sb_debug_ensemble_bytes(sb_ensemble_t* e, int64_t* out) {
  SB_CHECK(e, SB_ERR_STATE, "TF ensemble not initialized.");
  SB_CHECK(out, SB_ERR_INVALID, "null argument");
  *out = e->bytes();
  return SB_OK;
}

}  // extern "C"
