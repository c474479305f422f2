// extern "C" surface of libshifu_b200.so: the trainer, its step-trace and exchange test hooks, and the library-wide calls
// (version, devices, host allocation, NCCL id).  The scorers are in score.cu, the performance handle in perf.cu, and the
// kernel-level test hooks in net.cu.
// See include/shifu_b200.h for the contract and the reference call each entry point replaces.
#include <math.h>
#include <stdlib.h>
#include <cmath>
#include <string.h>
#include <algorithm>
#include <memory>
#include <random>
#include "net.cuh"
#include "savedmodel.h"
#include "xchg_p2p.cuh"

using namespace sb;

// ================================================================================================
// trainer
// ================================================================================================
enum { G_STEP = 0, G_ACC = 1, G_KINDS = 2 };

// A captured graph: `steps` consecutive steps (1, or RUN_S for sb_trainer_run_resident) of `kind` over `rows`-row batches
// of feed `feed`, reading the descriptor slots of ring set `set`
struct GraphKey {
  int rows, kind;
  Feed feed;
  int steps, set;
  bool operator<(const GraphKey& o) const {
    return std::tie(rows, kind, feed, steps, set) < std::tie(o.rows, o.kind, o.feed, o.steps, o.set);
  }
};

struct sb_trainer {
  Net net;
  sb_net_desc desc;
  OptHyper hyper;
  float lr = 0.f;
  float initial_accumulator = 0.1f;   // Adagrad / FTRL: start value of s1 (sb_trainer_set_optimizer_params)
  int rank = 0, world = 1;
  NcclComm comm = nullptr;
  float *grad = nullptr, *s1 = nullptr, *s2 = nullptr, *acc = nullptr;
  int n_acc = 0;
  float grad_out_scale = 1.f;  // what sb_trainer_get_grads multiplies the raw buffer by
  long long global_step = 0;
  float* h_scal = nullptr;  // pinned + mapped [SCAL_COUNT]: written by the tail kernel of every step
  float* d_hscal = nullptr; // device-side alias of h_scal
  // loss curve: (loss sum, n_nz) of the last HIST update steps, ring indexed by global_step % HIST, pinned + mapped
  enum { HIST = 8192 };
  float2* h_hist = nullptr;
  float2* d_hist = nullptr;
  float2* hist_slot(long long step) { return d_hist ? d_hist + (step % HIST) : nullptr; }
  // Resident training set.  dsX / dsXb live in HBM, or, when the set does not fit there (or force_host, the test hook
  // sb_debug_force_host_set), in mapped pinned host memory (ds_host) that the steps read over PCIe; y, w and P are always
  // in HBM.
  float *dsX = nullptr, *dsY = nullptr, *dsW = nullptr;   // dsX only in fp32 mode
  __nv_bfloat16* dsXb = nullptr;                           // bf16 mode: the set in GEMM-operand form [ds_rows, ldF]
  long long ds_ps = 0;                                     // part stride of dsXb (elements)
  int* dsP = nullptr;                                      // prefix counts of non-zero weights [ds_rows + 1]
  long long ds_rows = 0;
  bool ds_host = false, force_host = false;
  int* ds_iota = nullptr;   // bf16 set in host memory: the identity order its steps gather through without a row order
  // Batch buffers: where gather_batch_kernel puts a step's rows (Xb; fp32 mode: the net's Xf), labels and weights.  Entry
  // 0's Xb is the net's own.  Entry 1 exists for a bf16 set in host memory only: inside a run_resident graph its streamed
  // steps fetch the rows of step k + 1 on fetch_stream into the other buffer while step k runs, on fetch_ctas CTAs, with
  // step k's GEMM grids planned for the remaining SMs.  Step k of a captured graph (k = 0 outside graphs) reads buffer
  // k & 1 if its feed is STREAMED and buffer 0 otherwise; a RESIDENT step reads the set itself at desc->row0 (slot).
  struct BatchBuf { __nv_bfloat16* Xb = nullptr; float *y = nullptr, *w = nullptr; };
  BatchBuf bufs[2];
  const BatchBuf& batch_buf(Feed feed, int k) const { return bufs[feed == Feed::STREAMED ? (k & 1) : 0]; }
  cudaStream_t fetch_stream = nullptr;
  cudaEvent_t ev_fork = nullptr, ev_fetched = nullptr;
  int fetch_ctas = 16;
  // row order of the resident set (sb_trainer_set_row_order): the resident entry points address logical row r as row
  // ord[r] (int32 on the device, the only per-row memory an order costs); ord_n == 0: physical order
  int* ord = nullptr;
  long long ord_n = 0, ord_cap = 0;
  std::map<GraphKey, cudaGraphExec_t> graphs;
  std::map<std::pair<int, Feed>, int> kernels_per_step;   // (rows, feed) of a captured single G_STEP step
  // peer-memory exchange (xchg_p2p.cuh): the net's parameter arena [theta | s1 | s2 | shadows | gradient | P2PFlags] is
  // ONE exported allocation; `xch` aliases it
  void* xch = nullptr;
  long long xch_n4 = 0;            // float4 count of the padded gradient
  long long grad_off = 0, flags_off = 0;   // byte offsets of the gradient / flag block inside the arena
  P2PFlags* flags = nullptr;
  P2PPeers* d_peers = nullptr;     // device table of every rank's arena
  std::vector<void*> peer_bases;   // opened IPC mappings (to close)
  bool p2p_ready = false;
  bool peers_share_device = false; // in-process replicas on this device (tests): see enqueue_xchg and plan_dw1
  bool grad_sharded = false;       // the reduced gradient of the last step lives in slices on its owners (sb_trainer_get_grads gathers)
  bool master_stale = false;       // sharded updates ran since the fp32 master / state were last gathered from their owners
  unsigned int epoch = 0;
  unsigned int* h_err = nullptr;   // pinned + mapped: a peer that never arrived (xchg_p2p.cuh), 0 = none
  unsigned int* d_herr = nullptr;
  unsigned long long xchg_timeout_ns = 300ull * 1000000000ull;
  int xchg_blocks = 0;             // grid cap of the exchange kernels (0 = one block per SM)
  // slot table of the exchange (fixed for the trainer's life: it defines who owns which run): slot 0 = every layer but
  // hidden layer 0, slots 1..x_chunks = row chunks of hidden layer 0 (the last one also carries b_0)
  int x_chunks = 1, x_slots = 2;
  int x_chunk_rows = 0;            // rows of W_0 per slot chunk (128-row multiple; the last chunk may be shorter)
  int x_begin[SB_XCHG_SLOTS] = {}, x_end[SB_XCHG_SLOTS] = {};
  cudaEvent_t ev_x[SB_XCHG_SLOTS] = {};   // exchange of slot s complete (recorded on its comm stream)
  cudaEvent_t ev_c[SB_XCHG_SLOTS] = {};   // dW_0 chunk c complete on the main stream / tail of the main stream
  bool ll_ready = false;           // the LL exchange (xchg_ll_kernel) is usable: plain bf16, world > 1, buffers in the arena
  long long llg_off = 0, lls_off = 0;
  // streams and events of the step schedule (enqueue_step_backward)
  cudaStream_t side = nullptr;               // dW GEMMs run here, concurrently with the dA chain on the net's stream
  cudaStream_t xstream[2] = {};              // the exchange launches behind dW_0's row chunks alternate between these
  std::vector<cudaEvent_t> ev_dz;            // ev_dz[l]: dZ_l is complete on the net's stream
  cudaEvent_t ev_join = nullptr;
  cudaEvent_t ev_da_done = nullptr;          // the last dA GEMM (last reader of the bf16 weight shadows) is complete
  // pipelined host-buffer steps (sb_trainer_step_async): second staging slot + copy stream, so the H2D of batch i+1
  // overlaps the compute of batch i
  cudaStream_t copy_stream = nullptr;
  float *st2X = nullptr, *st2Y = nullptr, *st2W = nullptr;
  cudaEvent_t ev_copied[2] = {nullptr, nullptr}, ev_consumed[2] = {nullptr, nullptr};
  bool copy_ready = false;   // every piece of the second slot exists
  unsigned long long async_steps = 0;
  // Descriptor ring: two sets of RUN_S (descriptor, scalar) slots; set 0 slot 0 is the net's own.  sb_trainer_run_resident
  // captures RUN_S steps per graph (kernel -> kernel edges instead of a graph turn-around between steps).  Prefetched
  // launches (bf16-resident and ordered steps) alternate between the sets: the descriptors of launch i+1 are written on
  // `prep` while launch i still runs, so set_batch_kernel leaves the critical path.  Every other user of a slot writes
  // set 0 (host-batch steps, forward paths) or the last prefetched set (update-only launches) on the main stream.
  enum { RUN_S = 4 };
  BatchDesc* ring_desc[2][RUN_S] = {};
  float* ring_scal[2][RUN_S] = {};
  cudaStream_t prep = nullptr;
  cudaEvent_t ev_prep[2] = {nullptr, nullptr}, ev_pos[2] = {nullptr, nullptr};
  unsigned long long prefetches = 0;   // prefetched launches so far: launch i uses set i & 1
  // Fine-tuning (sb_trainer_set_fixed_layers): whether W_l / b_l of layer l = 0..L train, and the same as bit masks of the
  // frozen ones (what the peers compare).  dA_l (l >= 1) runs only for l > l_min, the lowest hidden layer with a parameter
  // that trains (L: none), since it exists to make dZ_{l-1} for dW and bias gradients at or below layer l - 1.
  std::vector<char> w_trains, b_trains;
  int l_min = 0;
  unsigned long long frozen_w = 0, frozen_b = 0;
  bool started = false;    // a step ran or was captured: sb_trainer_set_deterministic is refused from here on
  bool have_pos = false;   // ev_pos[] of the previous prefetched launch is valid (no step on set 0 since)
  int last_set = 0;        // the set of the last prefetched launch
  StepIn slot(int set, int k, Feed feed = Feed::HOST) const {
    const Operand0 x0 = feed == Feed::RESIDENT ? Operand0{dsXb, ds_ps, static_cast<int>(ds_rows), true}
                                               : Operand0{batch_buf(feed, k).Xb, net.Xb_ps};
    return StepIn{ring_desc[set][k], ring_scal[set][k], feed, x0};
  }
  // y / w of batch buffer 0 and, for a bf16 set in host memory (`streamed`), all of buffer 1; kept once made
  int alloc_batch_bufs(bool streamed) {
    for (int i = 0; i < (streamed ? 2 : 1); ++i) {
      if (i == 1 && !bufs[1].Xb) SB_TRY(net.dalloc(&bufs[1].Xb, static_cast<size_t>(net.Xb_ps) * net.nparts));
      if (!bufs[i].y) SB_TRY(net.dalloc(&bufs[i].y, net.max_batch));
      if (!bufs[i].w) SB_TRY(net.dalloc(&bufs[i].w, net.max_batch));
    }
    return SB_OK;
  }

  // Releases what the trainer created.  Pointers into the net's allocations (ring_desc, ring_scal, grad, flags, xch, s1,
  // s2, acc, st2*) are freed by `net`, the first member and so the last destroyed.
  ~sb_trainer() {
    drop_step_graphs();
    auto destroy_event = [](cudaEvent_t e) { if (e) cudaEventDestroy(e); };
    for (cudaEvent_t e : ev_dz) destroy_event(e);
    destroy_event(ev_join);
    destroy_event(ev_da_done);
    for (int i = 0; i < SB_XCHG_SLOTS; ++i) { destroy_event(ev_x[i]); destroy_event(ev_c[i]); }
    destroy_event(ev_fork);
    destroy_event(ev_fetched);
    for (int i = 0; i < 2; ++i) {
      destroy_event(ev_copied[i]); destroy_event(ev_consumed[i]);
      destroy_event(ev_prep[i]); destroy_event(ev_pos[i]);
    }
    if (prep) cudaStreamSynchronize(prep);
    for (cudaStream_t s : {xstream[0], xstream[1], side, prep, copy_stream, fetch_stream}) if (s) cudaStreamDestroy(s);
    if (h_scal) cudaFreeHost(h_scal);
    if (h_err) cudaFreeHost(h_err);
    if (h_hist) cudaFreeHost(h_hist);
    close_peer_mappings();   // before the net frees the arena they were opened against
    if (d_peers) cudaFree(d_peers);
    free_dataset();
    if (comm) { NcclApi* api = nccl_api(); if (api) api->CommDestroy(comm); }
  }

  void drop_step_graphs() {   // captured steps carry the exchange and the resident set they were captured with
    for (auto& kv : graphs) cudaGraphExecDestroy(kv.second);
    graphs.clear();
  }
  void free_dataset() {
    void* x = dsXb ? static_cast<void*>(dsXb) : static_cast<void*>(dsX);
    if (x) { if (ds_host) cudaFreeHost(x); else cudaFree(x); }
    ds_host = false;
    if (ds_iota) cudaFree(ds_iota);
    ds_iota = nullptr;
    if (dsP) cudaFree(dsP);
    if (dsY) cudaFree(dsY);
    if (dsW) cudaFree(dsW);
    dsX = dsY = dsW = nullptr; dsXb = nullptr; dsP = nullptr; ds_rows = 0;
    drop_row_order();
  }
  void drop_row_order() {
    if (ord) cudaFree(ord);
    ord = nullptr;
    ord_n = ord_cap = 0;
  }
  long long resident_len() const { return ord_n > 0 ? ord_n : ds_rows; }   // what resident offsets are checked against
  // resident steps gather their batch into Xb / Xf first: through the row order, or, from a bf16 set in host memory, whose
  // rows layer 0's GEMMs cannot read by TMA, through the row order or the identity order ds_iota
  bool streamed() const { return ds_host && dsXb; }
  bool gathers() const { return ord_n > 0 || streamed(); }
  // the feed of a resident step: the fp32 set (in HBM or host memory) is read in place through the host-batch graph
  Feed resident_feed() const {
    return streamed() ? Feed::STREAMED : ord_n > 0 ? Feed::ORDERED : dsXb ? Feed::RESIDENT : Feed::HOST;
  }
  void close_peer_mappings() {
    for (void* p : peer_bases) cudaIpcCloseMemHandle(p);
    peer_bases.clear();
  }
};

static int create_event(cudaEvent_t* e) {   // (no-op if it exists: a retry after a failure creates what is missing)
  if (!*e) SB_CUDA(cudaEventCreateWithFlags(e, cudaEventDisableTiming));
  return SB_OK;
}

static float lr_for_step(const sb_trainer* t, long long step /*1-based*/) {
  if (t->hyper.kind == SB_OPT_ADAM) {
    const double b1 = t->hyper.beta1, b2 = t->hyper.beta2;
    return static_cast<float>(t->lr * sqrt(1.0 - pow(b2, static_cast<double>(step))) / (1.0 - pow(b1, static_cast<double>(step))));
  }
  return t->lr;
}

// an update: advances the step count and the exchange round; -> the update's learning rate
static float begin_update(sb_trainer* t) {
  ++t->global_step;
  ++t->epoch;
  return lr_for_step(t, t->global_step);
}

// rows [off, off + rows) of the resident set, through the row order if one is set, for step k of a graph.  step >= 0
// names the step of a run in the error message.
static int resident_batch(const sb_trainer* t, long long off, int rows, int step, int k, Batch* b) {
  SB_CHECK(t->ds_rows > 0, SB_ERR_STATE, "no resident dataset loaded");
  const long long len = t->resident_len();
  if (off < 0 || rows <= 0 || off + rows > len) {
    char at[32] = "";
    if (step >= 0) snprintf(at, sizeof(at), "step %d: ", step);
    return set_error(SB_ERR_INVALID, "%srows [%lld, %lld) outside the resident set of %lld %s", at, off, off + rows, len,
                     t->ord_n > 0 ? "rows of the row order" : "rows");
  }
  SB_CHECK(rows <= t->net.max_batch, SB_ERR_INVALID, "rows=%d outside (0, max_batch=%d]", rows, t->net.max_batch);
  *b = Batch{};
  b->feed = t->resident_feed();
  b->rows = rows;
  if (b->feed == Feed::ORDERED || b->feed == Feed::STREAMED) {   // gather_batch_kernel counts n_nz and fills y / w
    b->y = t->batch_buf(b->feed, k).y; b->w = t->batch_buf(b->feed, k).w;
    b->order = (t->ord_n > 0 ? t->ord : t->ds_iota) + off;
    return SB_OK;
  }
  b->y = t->dsY + off; b->w = t->dsW + off;
  if (b->feed == Feed::RESIDENT) {
    b->row0 = static_cast<int>(off);
    b->nz_prefix = t->dsP;
  } else {
    b->X = t->dsX + off * t->net.F;
  }
  return SB_OK;
}

static int enqueue_allreduce(sb_trainer* t, float* buf) {
  if (t->world <= 1) return SB_OK;
  NcclApi* api = nccl_api();
  SB_CHECK(api && t->comm, SB_ERR_NCCL, "no gradient exchange configured: world = %d but neither an NCCL communicator (nccl_id) nor a "
           "peer table (sb_trainer_set_peer_handles / _pointers) exists", t->world);
  int r = api->AllReduce(buf, buf, static_cast<size_t>(t->net.n_params), NCCL_FLOAT32, NCCL_SUM, t->comm, t->net.stream);
  SB_CHECK(r == 0, SB_ERR_NCCL, "ncclAllReduce failed: %s", api->GetErrorString(r));
  return SB_OK;
}

// The update kernels of every optimizer group (opt_group) and, for the exchange, world size: every launch, the carveout
// setting and the preload read these tables.
static void (*const optimizer_kernels[OPT_GROUPS])(const OptWork*, const BatchDesc*, OptHyper, float*, const float*, float*, float*,
                                                   const float*, float*, unsigned long long*) = {
    optimizer_kernel<OPT_BASE>, optimizer_kernel<OPT_EXT>, optimizer_kernel<OPT_RPROP>};
static const char* const opt_group_names[OPT_GROUPS] = {"base", "ext", "rprop"};
enum { XCHG_WORLDS = 4 };   // world <= 2 / 4 / 8 / 16
static void (*const xchg_update_kernels[OPT_GROUPS][XCHG_WORLDS])(const XchgParams) = {
    {xchg_update_kernel<2, OPT_BASE>, xchg_update_kernel<4, OPT_BASE>, xchg_update_kernel<8, OPT_BASE>, xchg_update_kernel<16, OPT_BASE>},
    {xchg_update_kernel<2, OPT_EXT>, xchg_update_kernel<4, OPT_EXT>, xchg_update_kernel<8, OPT_EXT>, xchg_update_kernel<16, OPT_EXT>},
    {xchg_update_kernel<2, OPT_RPROP>, xchg_update_kernel<4, OPT_RPROP>, xchg_update_kernel<8, OPT_RPROP>, xchg_update_kernel<16, OPT_RPROP>}};
static void (*const xchg_ll_kernels[OPT_GROUPS][XCHG_WORLDS])(const LLParams) = {
    {xchg_ll_kernel<2, OPT_BASE>, xchg_ll_kernel<4, OPT_BASE>, xchg_ll_kernel<8, OPT_BASE>, xchg_ll_kernel<16, OPT_BASE>},
    {xchg_ll_kernel<2, OPT_EXT>, xchg_ll_kernel<4, OPT_EXT>, xchg_ll_kernel<8, OPT_EXT>, xchg_ll_kernel<16, OPT_EXT>},
    {xchg_ll_kernel<2, OPT_RPROP>, xchg_ll_kernel<4, OPT_RPROP>, xchg_ll_kernel<8, OPT_RPROP>, xchg_ll_kernel<16, OPT_RPROP>}};
static const char* const xchg_update_names[XCHG_WORLDS] = {"xchg_update<2>", "xchg_update<4>", "xchg_update<8>", "xchg_update<16>"};
static const char* const xchg_ll_names[XCHG_WORLDS] = {"xchg_ll<2>", "xchg_ll<4>", "xchg_ll<8>", "xchg_ll<16>"};

// route (nullable, sb_debug_optimizer): appends "+"-joined "optimizer<base|ext|rprop>@<main|side>[w0,w1)" for the launch
static int enqueue_optimizer(sb_trainer* t, const StepIn& in, const float* g, int w0 = 0, int w1 = -1, cudaStream_t st = nullptr,
                             bool publish_scalars = false, bool pdl = false, std::string* route = nullptr) {
  Net& n = t->net;
  if (w1 < 0) w1 = n.n_work;
  if (!st) st = n.stream;
  if (w1 <= w0) return SB_OK;
  const int grp = opt_group(t->hyper.kind);
  // pdl = false: plain dependency (runs after a stream join / on the comm stream)
  SB_TRY(launch_kernel(optimizer_kernels[grp], dim3(static_cast<unsigned>(w1 - w0)), dim3(256), 0, st, pdl, n.work + w0, in.desc, t->hyper,
                       n.theta, g, n.s1, n.s2, in.scal, publish_scalars ? t->d_hscal : static_cast<float*>(nullptr),
                       n.next_trace(st == n.stream ? "opt" : "opt_side")));
  n.mark("optimizer");
  if (route) {
    char r[64];
    snprintf(r, sizeof(r), "%soptimizer<%s>@%s[%d,%d)", route->empty() ? "" : "+", opt_group_names[grp],
             st == n.stream ? "main" : "side", w0, w1);
    *route += r;
  }
  return SB_OK;
}

// slots of the sharded exchange: bit 0 = A (every layer but hidden layer 0), bits 1.. = the row chunks of hidden layer 0
enum { XSEG_A = 1 };
static int xseg_all(const sb_trainer* t) { return (1 << t->x_slots) - 1; }

static XchgParams xchg_params(sb_trainer* t, const BatchDesc* desc) {
  Net& n = t->net;
  XchgParams p;
  memset(&p, 0, sizeof(p));
  p.peers = t->d_peers;
  p.rank = t->rank; p.world = t->world;
  p.s1_off = static_cast<long long>(n.s1_off); p.s2_off = static_cast<long long>(n.s2_off);
  p.grad_off = t->grad_off; p.flags_off = t->flags_off;
  p.work = n.work;
  p.n_slots = t->x_slots;
  for (int sl = 0; sl < t->x_slots; ++sl) { p.slot_begin[sl] = t->x_begin[sl]; p.slot_end[sl] = t->x_end[sl]; }
  p.desc = desc;
  p.hyper = t->hyper;
  p.host_err = t->d_herr;
  p.timeout_ns = t->xchg_timeout_ns;
  static const bool fence_sys = getenv("SB_XCHG_FENCE_SYS") != nullptr;
  p.fence_gpu = fence_sys ? 0 : 1;
  return p;
}

// grid of an exchange launch over the slots of `slot_mask`
static int xchg_grid(const sb_trainer* t, int slot_mask, bool alone) {
  int runs = 0, all_runs = 0;      // owned runs of the launch (the largest share) / runs of the launch
  for (int sl = 0; sl < t->x_slots; ++sl)
    if ((slot_mask >> sl) & 1) {
      runs += (t->x_end[sl] - t->x_begin[sl] + t->world - 1) / t->world;
      all_runs += t->x_end[sl] - t->x_begin[sl];
    }
  const int U = t->world <= 2 ? 2 : 1;      // runs per block iteration of the update phase (xchg_update_kernel)
  const int want = std::max((runs + U - 1) / U, (all_runs - runs + 3) / 4);   // ... and 4 per iteration of the gather phase
  // one block per SM and launch.  A GEMM CTA takes a whole SM (registers and shared memory, gemm_tc.cuh), so exchange
  // blocks run only on SMs no GEMM CTA holds and otherwise wait for GEMM CTAs to leave - those never wait for an exchange,
  // so this cannot deadlock, only be slow.  The schedule below was tuned where an exchange block fitted beside a GEMM CTA;
  // on H100 it has not been measured with more than one GPU.
  // (alone: nothing but other exchange launches runs beside this one - two blocks per SM, all loads of a phase in one round)
  int grid = t->xchg_blocks > 0 ? t->xchg_blocks : (alone ? 2 : 1) * t->net.num_sms;
  if (t->peers_share_device && grid > 32) grid = 32;    // replicas on ONE device: leave registers to the replica being waited for
  if (grid > want) grid = want;
  if (grid < 1) grid = 1;
  return grid;
}

// the exchange kernel of the world size and optimizer group; *kernel names it (the same name for every group)
static int launch_xchg(sb_trainer* t, const XchgParams& p, dim3 g, dim3 b, cudaStream_t st, bool pdl, const char** kernel) {
  const int grp = opt_group(t->hyper.kind), wi = t->world <= 2 ? 0 : t->world <= 4 ? 1 : t->world <= 8 ? 2 : 3;
  // plain bf16: the LL protocol (flags inside the data) needs fewer fabric round trips than the flag-and-pull kernel
  if (t->ll_ready) {
    LLParams lp;
    lp.x = p; lp.llg_off = t->llg_off; lp.lls_off = t->lls_off; lp.n4 = t->xch_n4;
    SB_TRY(launch_kernel(xchg_ll_kernels[grp][wi], g, b, 0, st, pdl, lp));
    *kernel = xchg_ll_names[wi];
  } else {
    SB_TRY(launch_kernel(xchg_update_kernels[grp][wi], g, b, 0, st, pdl, p));
    *kernel = xchg_update_names[wi];
  }
  return SB_OK;
}

// reduce-scatter -> owner update -> all-gather of the operands for the given segments (xchg_p2p.cuh); `g` must be t->grad.
// grid > 0 replaces the grid rule (sb_debug_exchange).
static int enqueue_xchg(sb_trainer* t, const StepIn& in, int slot_mask, cudaStream_t st, bool publish_scalars, bool pdl,
                        bool alone = false, int grid = 0) {
  Net& n = t->net;
  XchgParams p = xchg_params(t, in.desc);
  p.slot_mask = slot_mask;
  p.scal = publish_scalars ? in.scal : nullptr;
  p.host_scal = publish_scalars ? t->d_hscal : nullptr;
  char nm[24];
  if (slot_mask == XSEG_A) snprintf(nm, sizeof(nm), "xchg_A");
  else if ((slot_mask & (slot_mask - 1)) == 0) snprintf(nm, sizeof(nm), "xchg_B%d", __builtin_ctz(slot_mask) - 1);
  else snprintf(nm, sizeof(nm), "xchg");
  p.trace = n.next_trace(nm);
  if (grid <= 0) grid = xchg_grid(t, slot_mask, alone);
  const dim3 g(static_cast<unsigned>(grid)), b(256);
  const char* kernel;
  SB_TRY(launch_xchg(t, p, g, b, st, pdl, &kernel));
  n.mark(kernel);
  t->master_stale = true;
  t->grad_sharded = true;
  return SB_OK;
}

// before the host reads theta / s1 / s2: pull the runs other ranks own from their owners (no-op unless sharded updates ran)
static int gather_master(sb_trainer* t) {
  if (!t->p2p_ready || !t->master_stale || t->world <= 1) return SB_OK;
  Net& n = t->net;
  SB_CUDA(cudaStreamSynchronize(n.stream));     // my last exchange kernel has seen every peer's done flag
  XchgParams p = xchg_params(t, n.desc);
  gather_master_kernel<<<n.n_work, 256, 0, n.stream>>>(p, 0);
  SB_CUDA(cudaGetLastError());
  SB_CUDA(cudaStreamSynchronize(n.stream));
  t->master_stale = false;
  return SB_OK;
}

// `to` waits for everything enqueued on `from` so far
static int join_streams(cudaStream_t to, cudaStream_t from, cudaEvent_t e) {
  SB_CUDA(cudaEventRecord(e, from));
  SB_CUDA(cudaStreamWaitEvent(to, e, 0));
  return SB_OK;
}

// The single-GPU step's split tail: layer 0's runs on the main stream, PDL-chained behind dW_0 and publishing the step
// scalars; the other runs on the side stream once the last dA GEMM (ev_da_done, recorded by the caller) no longer reads
// their shadows; then the main stream joins the side stream.
static int enqueue_split_tail(sb_trainer* t, const StepIn& in, const float* g, std::string* route = nullptr) {
  Net& n = t->net;
  // the layer-0 optimizer publishes the step scalars, or the other layers' one when layer 0 has nothing that trains
  const bool l0_runs = n.work_end[0] > n.work_begin[0];
  SB_TRY(enqueue_optimizer(t, in, g, n.work_begin[0], n.work_end[0], n.stream, true, true, route));
  // the other layers' shadows are read by the dA GEMMs on the main stream: update them only after the last one
  SB_CUDA(cudaStreamWaitEvent(t->side, t->ev_da_done, 0));
  SB_TRY(enqueue_optimizer(t, in, g, n.work_end[0], n.n_work, t->side, !l0_runs, false, route));
  return join_streams(n.stream, t->side, t->ev_join);
}

// Where dW_1 runs, and the SM budget (grid cap) of dW_0 / dW_1, in a tensor-core step with more than one hidden layer:
//   BESIDE  on the side stream, at the same time as dW_0 on the main stream;
//   FRONT   on the main stream in front of dW_0;
//   BEHIND  on the main stream behind dW_0.
enum Dw1At { DW1_BESIDE, DW1_FRONT, DW1_BEHIND };
struct Dw1Plan {
  Dw1At at;
  int sms[2];
};

static Dw1Plan plan_dw1(const sb_trainer* t, int rows, bool split_tail, bool xsched) {
  const Net& n = t->net;
  const int S = n.num_sms;
  Dw1Plan d = {DW1_BESIDE, {S, S}};
  // peer exchange: in front of dW_0, so that slot A's exchange hides behind dW_0's chunks; replicas that share a device
  // put it behind, as cover for the last chunk's exchange
  if (xsched) {
    d.at = t->peers_share_device ? DW1_BEHIND : DW1_FRONT;
    return d;
  }
  // dW_1 (side stream) and dW_0 (main stream) run at the same time, one CTA per SM each.  If their natural grids do not
  // fit the machine together, dW_1's second wave only starts when dW_0's CTAs exit.
  const Layer& l0 = n.layers[0];
  const Layer& l1 = n.layers[1];
  const int kx = round_up(rows, 64) * pairs_of(n.nparts);
  const int ms = n.dw_max_split();
  const GemmPlan n0 = plan_gemm(l0.in, l0.out, kx, S, true, ms);
  const GemmPlan n1 = plan_gemm(l1.in, l1.out, kx, S, true, ms);
  if (n0.grid + n1.grid <= S) return d;
  // single-GPU tail: dW_1 runs IN FRONT of dW_0 on the main stream instead of beside it - side by side the two persistent
  // grids take turns on the SMs; small layers (cfg1) stay side by side.  Only when dW_0 alone fills every SM: on one H100,
  // cfg2 (dW_0 = 128 tiles on 132 SMs, budget split below) measured within 1 % of both dW_1 in front and the natural
  // grids, while moving dW_1 in front once dW_0 fills >= 90 % of the SMs made cfg1 4 % slower.  A dW_0 on 128 x 256 tiles
  // (plan_gemm; cfg2) also takes dW_1 in front: beside it, dW_1's CTAs only get SMs as dW_0 ends and then hold them while
  // layer 0's optimizer runs (one H100 SXM, 700 W: the optimizer took 32 us sharing the SMs, 13 us after dW_1 in front;
  // cfg2 +0.9 %)
  if (split_tail && (n0.grid == S || n0.bn == 256)) {
    d.at = DW1_FRONT;
    return d;
  }
  // compare, in k-blocks per CTA, "natural grids, dW_1 finishing after dW_0" against "dW_1 on a third of the SMs, dW_0
  // on the rest" and take the shorter
  const GemmPlan b1 = plan_gemm(l1.in, l1.out, kx, S / 3, true, ms);
  const GemmPlan b0 = plan_gemm(l0.in, l0.out, kx, S - b1.grid, true, ms);
  auto waves = [&](const GemmPlan& pl, const Layer& ly, int sms) {   // k-blocks one CTA works through
    const int tiles = ((ly.in + 127) / 128) * ((ly.out + pl.bn - 1) / pl.bn) * pl.split_k;
    return ((tiles + sms - 1) / sms) * pl.kb_per_split;
  };
  const int t_nat = waves(n0, l0, S) + waves(n1, l1, S);
  const int t0 = waves(b0, l0, S - b1.grid);
  const int t1 = waves(b1, l1, S / 3);
  if ((t0 > t1 ? t0 : t1) < t_nat) { d.sms[1] = S / 3; d.sms[0] = S - b1.grid; }
  return d;
}

// The step's backward pass and tail, in launch order.
static int enqueue_step_backward(sb_trainer* t, const StepIn& in, int rows, int kind) {
  Net& n = t->net;
  float* g = t->grad;
  const int L = n.L, S = n.num_sms;
  // frozen layers (sb_trainer_set_fixed_layers): dW_l only where W_l trains, dA_l only where something at or below layer
  // l - 1 needs dZ_{l-1}.  With nothing frozen both are always true.
  auto dw = [&](int l) { return t->w_trains[static_cast<size_t>(l)] != 0; };
  auto da = [&](int l) { return l > t->l_min; };
  if (!n.tc()) {
    for (int l = L - 1; l >= 0; --l) {            // fp32: one stream
      if (dw(l)) SB_TRY(n.enqueue_dw(in, l, rows, g, n.stream, false, S));
      if (l > 0 && da(l)) SB_TRY(n.enqueue_da(l, rows, g));
    }
  } else {
    // Single GPU, one update per mini-batch: no exchange, so nothing needs ALL gradients at once.  dW_0 runs on the main
    // stream behind the last dA GEMM and is followed (PDL) by the optimizer of layer 0 alone; the side stream updates the
    // other layers right after their dW GEMMs; the two streams only join at the end of the graph.
    const bool split_tail = kind == G_STEP && (t->world == 1 || t->p2p_ready) && L > 1;
    // Peer exchange (world > 1): one exchange launch costs several fabric round trips however little data it moves
    // (xchg_p2p.cuh) - hidden when a GEMM follows it, exposed in full behind the last GEMM:
    //   main:  ... dA_1 -> dW_1 -> dW_0 chunk 0 -> dW_0 chunk 1 | wait A, B0, B1 | next step
    //   side:  ... dW_2 ...     A ------------->
    //   comm:                             B0 ---------------->    B1 ------>
    // A (every layer but hidden layer 0) and B0 run beside dW_0's chunks, only B1 - half of layer 0 - is exposed, on an
    // otherwise idle GPU, where an exchange kernel is faster than beside a GEMM.
    // Replicas that share ONE device (tests) put dW_1 BEHIND dW_0 instead, as cover for B1, and launch A on the side
    // stream behind it: with three exchange launches of both replicas waiting beside each other's persistent GEMMs, dW_1
    // in front stopped making progress within the exchange timeout.
    // Every exchange launch of the step is joined into the main stream before the step ends.  A rank's exchange only ends
    // once every peer has read the gradient runs it owns of this rank (xchg_p2p.cuh), so the next step's layer-0 forward
    // GEMM may clear the gradient buffer.
    const bool xsched = split_tail && t->world > 1;
    Dw1Plan d1 = L > 1 ? plan_dw1(t, rows, split_tail, xsched) : Dw1Plan{DW1_BESIDE, {S, S}};
    if (L > 1 && !(dw(0) && dw(1))) {
      // dW_0 or dW_1 frozen: the other one has the SMs to itself.  Without dW_0 (and without the exchange, which keeps its
      // plan) dW_1 is the last GEMM: in front, PDL-chained on the main stream.
      d1.sms[0] = d1.sms[1] = S;
      if (!xsched && !dw(0)) d1.at = DW1_FRONT;
    }
    // the exchange's slot A publishes the step scalars when there are no layer-0 chunks (W_0 frozen)
    const bool a_publishes = t->x_chunks == 0;
    bool side_used = false;     // a launch went to the side stream (which the end of the step then joins)
    // dW_l and dA_l both consume dZ_l and are independent of each other: the dW GEMMs go to the side stream and overlap
    // the dA chain
    for (int l = L - 1; l >= 1; --l) {
      if ((l > 1 || d1.at == DW1_BESIDE) && dw(l)) {
        SB_TRY(join_streams(t->side, n.stream, t->ev_dz[l]));
        SB_TRY(n.enqueue_dw(in, l, rows, g, t->side, false, l == 1 ? d1.sms[1] : S));
        side_used = true;
      }
      if (da(l)) SB_TRY(n.enqueue_da(l, rows, g));
    }
    if (split_tail) SB_CUDA(cudaEventRecord(t->ev_da_done, n.stream));
    if (L == 1) {
      if (dw(0)) {
        SB_TRY(join_streams(t->side, n.stream, t->ev_dz[0]));
        SB_TRY(n.enqueue_dw(in, 0, rows, g, t->side, false, S));
        side_used = true;
      }
    } else {
      if (d1.at == DW1_FRONT) {
        // dW_0's last exchange then runs on an idle GPU; the side stream's next launch (slot A's exchange, or the
        // optimizer of the other layers) waits for dW_1
        if (dw(1)) SB_TRY(n.enqueue_dw(in, 1, rows, g, n.stream, true, d1.sms[1]));
        SB_TRY(join_streams(t->side, n.stream, t->ev_c[0]));
        side_used = true;
        if (xsched) {
          SB_TRY(enqueue_xchg(t, in, XSEG_A, t->side, a_publishes, false));
          SB_CUDA(cudaEventRecord(t->ev_x[0], t->side));
        }
      }
      // dW_0 has nothing to overlap with (no dA_0): PDL-chained on the main stream right behind the last GEMM it starts
      // earlier than as a cross-stream launch.  With the peer exchange it is cut into the slot chunks (each a contiguous
      // slice of the flat gradient) and each chunk's exchange overlaps the GEMMs that follow it.
      if (xsched && in.feed != Feed::SPARSE) {
        for (int c = 0; c < t->x_chunks; ++c) {
          const int r0 = c * t->x_chunk_rows, r1 = std::min(r0 + t->x_chunk_rows, n.layers[0].in);
          SB_TRY(n.enqueue_dw(in, 0, rows, g, n.stream, true, d1.sms[0], r0, r1, t->x_chunks > 1 ? c : -1));
          cudaStream_t cs = t->xstream[c & 1];
          SB_TRY(join_streams(cs, n.stream, t->ev_c[1 + c]));
          // the last chunk publishes the step scalars; no GEMM follows it unless dW_1 does
          const bool last = c == t->x_chunks - 1;
          SB_TRY(enqueue_xchg(t, in, 1 << (1 + c), cs, last, false, last && d1.at != DW1_BEHIND));
          SB_CUDA(cudaEventRecord(t->ev_x[1 + c], cs));
        }
      } else if (dw(0)) {
        SB_TRY(n.enqueue_dw(in, 0, rows, g, n.stream, true, d1.sms[0]));
      }
      if (d1.at == DW1_BEHIND) {
        if (dw(1)) SB_TRY(n.enqueue_dw(in, 1, rows, g, n.stream, true, d1.sms[1]));
        SB_TRY(join_streams(t->side, n.stream, t->ev_c[0]));
        side_used = true;
        SB_TRY(enqueue_xchg(t, in, XSEG_A, t->side, a_publishes, false));
        SB_CUDA(cudaEventRecord(t->ev_x[0], t->side));
      }
    }
    if (xsched) {
      // whatever follows on the main stream (the next step's layer-0 forward, or the end of the graph) needs hidden
      // layer 0.  A wide+deep step's layer-0 dW is not cut into the slot chunks: it is exchanged here, behind everything.
      if (in.feed == Feed::SPARSE) {
        if (t->x_chunks > 0) SB_TRY(enqueue_xchg(t, in, xseg_all(t) & ~XSEG_A, n.stream, true, false));
      } else {
        for (int c = 0; c < t->x_chunks; ++c) SB_CUDA(cudaStreamWaitEvent(n.stream, t->ev_x[1 + c], 0));
      }
      SB_CUDA(cudaStreamWaitEvent(n.stream, t->ev_x[0], 0));
      return SB_OK;
    }
    if (split_tail) return enqueue_split_tail(t, in, g);
    if (side_used) SB_TRY(join_streams(n.stream, t->side, t->ev_join));
  }
  if (kind == G_STEP) {
    if (t->world > 1 && t->p2p_ready) {
      // (fp32 mode or one hidden layer: no split tail) one launch handles both segments
      SB_TRY(enqueue_xchg(t, in, xseg_all(t), n.stream, true, false));
    } else {
      SB_TRY(enqueue_allreduce(t, g));
      SB_TRY(enqueue_optimizer(t, in, g, 0, -1, nullptr, true, false));
    }
  } else {
    const long long np = n.n_params;
    axpy_kernel<<<static_cast<unsigned>((np + 255) / 256), 256, 0, n.stream>>>(t->acc, g, np, in.scal, t->d_hscal);
    SB_CUDA(cudaGetLastError());
    n.mark("accumulate");
  }
  return SB_OK;
}

// first kernel of an ordered step, in load_batch_kernel's place: the batch's rows of the resident set through the order
// slice in.desc->order into batch buffer bb (fp32 mode: X into Xf) and the step scalars; clears clear[0, clear_n) on the
// way.  On stream st (null: the main stream, PDL-chained, at most 16 blocks per SM), else on st with at most `ctas` blocks
static int enqueue_gather(sb_trainer* t, const StepIn& in, const sb_trainer::BatchBuf& bb, int rows, float* clear,
                          long long clear_n, cudaStream_t st = nullptr, int ctas = 0) {
  Net& n = t->net;
  GatherParams p = {};
  p.desc = in.desc;
  p.rows = rows; p.F = n.F; p.ldF = n.ldF; p.np = n.nparts;
  p.src_b = t->dsXb; p.src_ps = t->ds_ps; p.Xb = bb.Xb; p.Xb_ps = n.Xb_ps;
  p.src_f = t->dsX; p.Xf = n.Xf;
  p.src_y = t->dsY; p.src_w = t->dsW; p.y = bb.y; p.w = bb.w;
  p.scal = in.scal;
  p.zero_buf = clear; p.zero_n = clear_n;
  p.trace = n.next_trace(st ? "fetch_batch" : "gather_batch");
  const long long units = static_cast<long long>(rows) * (n.tc() ? n.ldF / 8 : (n.F + 3) / 4);
  const long long cap = st ? ctas : static_cast<long long>(n.num_sms) * 16;
  const long long blocks = std::max(1LL, std::min((units + 255) / 256, cap));
  const dim3 g(static_cast<unsigned>(blocks));
  const bool pdl = st == nullptr;
  if (!st) st = n.stream;
  if (n.tc()) SB_TRY(launch_kernel(gather_batch_kernel<true>, g, dim3(256), 0, st, pdl, p));
  else SB_TRY(launch_kernel(gather_batch_kernel<false>, g, dim3(256), 0, st, pdl, p));
  n.mark(n.tc() ? "gather_batch<bf16>" : "gather_batch<fp32>");
  return SB_OK;
}

// The first kernel of a step or forward, by feed: HOST / SPARSE load_batch_kernel, ORDERED (and a streamed forward)
// gather_batch_kernel into batch buffer 0 (t: its trainer), RESIDENT none (layer 0 reads the set by TMA; set_batch_kernel
// already published n_nz).  Clears clear[0, clear_n) on the way.
static int enqueue_first(Net& n, sb_trainer* t, const StepIn& in, int rows, float* clear, long long clear_n) {
  if (in.feed == Feed::RESIDENT) return SB_OK;
  if (in.feed == Feed::ORDERED || in.feed == Feed::STREAMED) return enqueue_gather(t, in, t->bufs[0], rows, clear, clear_n);
  return n.enqueue_load(in, rows, clear, clear_n);
}

// A streamed step k of a graph of `steps` reads batch buffer k & 1.  Step 0's rows are fetched first, on the main stream
// with the whole GPU; the rows of step k + 1 are fetched on fetch_stream while step k runs (forked behind step k - 1,
// the last reader of that buffer), and step k + 1 waits for them.  The fetch clears no gradient: step k still
// accumulates into it.
static int enqueue_streamed_fetch(sb_trainer* t, int set, int k, int steps, int rows) {
  Net& n = t->net;
  if (k == 0) SB_TRY(enqueue_gather(t, t->slot(set, 0, Feed::STREAMED), t->batch_buf(Feed::STREAMED, 0), rows, nullptr, 0));
  else SB_CUDA(cudaStreamWaitEvent(n.stream, t->ev_fetched, 0));
  if (k + 1 < steps) {
    SB_TRY(join_streams(t->fetch_stream, n.stream, t->ev_fork));
    SB_TRY(enqueue_gather(t, t->slot(set, k + 1, Feed::STREAMED), t->batch_buf(Feed::STREAMED, k + 1), rows, nullptr, 0,
                          t->fetch_stream, t->fetch_ctas));
    SB_CUDA(cudaEventRecord(t->ev_fetched, t->fetch_stream));
  }
  return SB_OK;
}

// the body of one step as a sequence of stream operations (captured into a CUDA graph)
static int enqueue_step_body(sb_trainer* t, const StepIn& in, int rows, int kind) {
  Net& n = t->net;
  n.trace_k = 0;
  float4* clear = nullptr;
  long long clear_n4 = 0;
  if (in.feed == Feed::RESIDENT || in.feed == Feed::STREAMED) {
    // no first kernel to clear the gradient buffer.  It is first written by the last forward layer's epilogue, so with
    // more than one hidden layer the layer-0 forward GEMM clears it (its producer warpgroup's idle warps, beside the main
    // loop) instead of a memset node at the head of the chain.
    if (n.L > 1) {
      clear = reinterpret_cast<float4*>(t->grad);   // cudaMalloc'ed, padded to xch_n4 float4
      clear_n4 = t->xch_n4;
    } else {
      SB_CUDA(cudaMemsetAsync(t->grad, 0, sizeof(float) * n.n_params, n.stream));
    }
  }
  if (in.feed != Feed::STREAMED) SB_TRY(enqueue_first(n, t, in, rows, t->grad, n.n_params));   // also clears the step scalars
  bool fused_out = false;
  SB_TRY(n.enqueue_hidden_forward(in, rows, t->grad, &fused_out, clear, clear_n4));
  if (!fused_out) SB_TRY(n.enqueue_out(in, rows, true, true, nullptr, t->grad));
  return enqueue_step_backward(t, in, rows, kind);
}

static int get_graph(sb_trainer* t, const GraphKey& key, cudaGraphExec_t* out) {
  auto it = t->graphs.find(key);
  if (it != t->graphs.end()) { *out = it->second; return SB_OK; }
  Net& n = t->net;
  t->started = true;
  n.launches = 0;
  cudaGraph_t g = nullptr;
  SB_CUDA(cudaStreamBeginCapture(n.stream, cudaStreamCaptureModeThreadLocal));
  int s = SB_OK;
  // a streamed graph of several steps overlaps each fetch with the previous step: its GEMM grids leave fetch_ctas SMs free
  const int sms = n.num_sms;
  const bool overlap = key.feed == Feed::STREAMED && key.steps > 1;
  if (overlap) n.num_sms = sms - t->fetch_ctas;
  for (int k = 0; k < key.steps && s == SB_OK; ++k) {
    // (SB_STEP_TRACE: of a run, an interior step is the one traced - it starts behind the previous step's tail, as most
    // steps of a run do)
    n.trace_on = key.steps == 1 || k == 1;
    if (key.feed == Feed::STREAMED) s = enqueue_streamed_fetch(t, key.set, k, key.steps, key.rows);
    if (s == SB_OK) s = enqueue_step_body(t, t->slot(key.set, k, key.feed), key.rows, key.kind);
  }
  n.num_sms = sms;
  n.trace_on = true;
  cudaError_t e = cudaStreamEndCapture(n.stream, &g);
  if (s != SB_OK) { if (g) cudaGraphDestroy(g); return s; }
  SB_CHECK(e == cudaSuccess, SB_ERR_CUDA, "cudaStreamEndCapture failed: %s", cudaGetErrorString(e));
  cudaGraphExec_t ge = nullptr;
  SB_CUDA(cudaGraphInstantiate(&ge, g, 0));
  cudaGraphDestroy(g);
  t->graphs[key] = ge;
  if (key.steps == 1 && key.kind == G_STEP && key.feed != Feed::SPARSE)
    t->kernels_per_step[{key.rows, key.feed}] = n.launches + 1;  // + set_batch_kernel
  *out = ge;
  return SB_OK;
}

// A prefetched launch writes the descriptors of ring set `set` = prefetches & 1 on `prep`:
//   prefetch_begin(t, set);  write_desc(t->prep, t->slot(set, k), ...) ...;  prefetch_end(t, set);  graph launch
// Set s was last read by the prefetched launch two back and by whatever followed it on the main stream before the previous
// prefetched launch (update-only launches write the last set there): ev_pos[s ^ 1], recorded right before that launch,
// covers both.  Without one (have_pos false: the first prefetched launch, or a step on set 0 since), join the main stream's
// current position.
static int prefetch_begin(sb_trainer* t, int set) {
  if (!t->have_pos) SB_CUDA(cudaEventRecord(t->ev_pos[set ^ 1], t->net.stream));
  SB_CUDA(cudaStreamWaitEvent(t->prep, t->ev_pos[set ^ 1], 0));
  return SB_OK;
}

static int prefetch_end(sb_trainer* t, int set) {
  SB_CUDA(cudaEventRecord(t->ev_prep[set], t->prep));
  SB_CUDA(cudaEventRecord(t->ev_pos[set], t->net.stream));
  SB_CUDA(cudaStreamWaitEvent(t->net.stream, t->ev_prep[set], 0));
  t->have_pos = true;
  t->last_set = set;
  ++t->prefetches;
  return SB_OK;
}

// A deterministic trainer with more than one rank needs the peer-memory exchange, which adds the ranks' gradients in rank
// order; NCCL's all-reduce promises no summation order.
static int check_det_exchange(const sb_trainer* t) {
  SB_CHECK(!t->net.det || t->world == 1 || t->p2p_ready, SB_ERR_STATE,
           "deterministic trainer (rank %d of %d) has no peer table: the NCCL all-reduce does not fix its summation order, so "
           "deterministic training across ranks needs sb_trainer_set_peer_handles / _pointers", t->rank, t->world);
  return SB_OK;
}

// One step over batch `b`: bf16-resident and ordered steps are prefetched, every other step writes set 0 on the main stream
static int run_step(sb_trainer* t, const Batch& b, int kind) {
  Net& n = t->net;
  SB_TRY(check_det_exchange(t));
  t->started = true;
  SB_CHECK(b.rows > 0 && b.rows <= n.max_batch, SB_ERR_INVALID, "rows=%d outside (0, max_batch=%d]", b.rows, n.max_batch);
  SB_CUDA(cudaSetDevice(n.device));
  const bool prefetch = b.feed == Feed::RESIDENT || b.feed == Feed::ORDERED || b.feed == Feed::STREAMED;
  const int set = prefetch ? static_cast<int>(t->prefetches & 1) : 0;
  cudaGraphExec_t ge = nullptr;
  SB_TRY(get_graph(t, GraphKey{b.rows, kind, b.feed, 1, set}, &ge));
  const float gscale = 1.f / static_cast<float>(t->world);
  const float lr_t = kind == G_STEP ? begin_update(t) : t->lr;
  float2* hist = kind == G_STEP ? t->hist_slot(t->global_step) : nullptr;
  if (prefetch) {
    SB_TRY(prefetch_begin(t, set));
    SB_TRY(write_desc(t->prep, t->slot(set, 0), &b, lr_t, gscale, t->epoch, hist));
    SB_TRY(prefetch_end(t, set));
  } else {
    t->have_pos = false;
    SB_TRY(write_desc(n.stream, t->slot(0, 0), &b, lr_t, gscale, t->epoch, hist));
  }
  SB_CUDA(cudaGraphLaunch(ge, n.stream));
  // the step's tail kernel (optimizer / accumulate) wrote (loss sum, n_nz) into h_scal; visible after a stream sync
  if (kind == G_ACC) ++t->n_acc;
  t->grad_out_scale = (kind == G_STEP) ? gscale : 1.f;
  return SB_OK;
}

// The forward of one batch on the main stream: its descriptor into slot `in`, the feed's first kernel, the hidden layers and
// the output layer (do_loss: + the loss sum into in.scal), scores to yhat_dst (nullable).
static int enqueue_forward(Net& n, sb_trainer* t, StepIn in, const Batch& b, unsigned int epoch, bool do_loss, float* yhat_dst) {
  in.feed = b.feed;
  SB_TRY(write_desc(n.stream, in, &b, 0.f, 1.f, epoch, nullptr));
  SB_TRY(enqueue_first(n, t, in, b.rows, nullptr, 0));
  SB_TRY(n.enqueue_hidden_forward(in, b.rows));
  return n.enqueue_out(in, b.rows, do_loss, false, yhat_dst, nullptr);
}

// forward (+ loss if loss_sum != nullptr) over any number of rows in max_batch chunks: stage(r0, c, &b) stages rows
// [r0, r0 + c) and describes them in b; out nullable.
// (Slot set 0: these host-driven paths are not captured.  A step queues its descriptor writes ahead of its graph on the
// main stream, and every forward path synchronises that stream before it returns, so no descriptor prefetch overlaps them.)
template <typename Stage>
static int forward_chunks(sb_trainer* t, int64_t rows, Stage stage, float* out, double* loss_sum, double* nnz) {
  Net& n = t->net;
  SB_CUDA(cudaSetDevice(n.device));
  const StepIn in{n.desc, n.scal};
  float h[SCAL_COUNT];
  for (int64_t r0 = 0; r0 < rows; r0 += n.max_batch) {
    const int c = static_cast<int>(rows - r0 < n.max_batch ? rows - r0 : n.max_batch);
    Batch b;
    SB_TRY(stage(r0, c, &b));
    SB_TRY(enqueue_forward(n, t, in, b, 0, loss_sum != nullptr, n.yhat));
    if (out) SB_CUDA(cudaMemcpyAsync(out + r0, n.yhat, sizeof(float) * c, cudaMemcpyDefault, n.stream));
    if (loss_sum) SB_CUDA(cudaMemcpyAsync(h, in.scal, sizeof(h), cudaMemcpyDeviceToHost, n.stream));
    SB_CUDA(cudaStreamSynchronize(n.stream));
    if (loss_sum) { *loss_sum += h[SCAL_LOSS_SUM]; *nnz += h[SCAL_NNZ]; }
  }
  return SB_OK;
}

// an NCCL failure on another rank (peer died, transport error) is reported asynchronously: surface it at every point where
// the host waits for the device instead of hanging in the next collective
static int poll_nccl(sb_trainer* t) {
  if (!t->comm) return SB_OK;
  NcclApi* api = nccl_api();
  if (!api || !api->CommGetAsyncError) return SB_OK;
  int err = 0;
  if (api->CommGetAsyncError(t->comm, &err) == 0 && err != 0)
    return set_error(SB_ERR_NCCL, "NCCL asynchronous error on rank %d: %s", t->rank, api->GetErrorString(err));
  return SB_OK;
}

// a peer that never arrived at the exchange (xchg_p2p.cuh) left a note in mapped host memory
static int poll_xchg(sb_trainer* t) {
  if (!t->h_err) return SB_OK;
  const unsigned int e = *reinterpret_cast<volatile unsigned int*>(t->h_err);
  if (e == 0) return SB_OK;
  return set_error(SB_ERR_NCCL, "gradient exchange timed out on rank %d: rank %u did not reach slot %u of the exchange within %.0f s "
                   "(peer process dead or stuck); this trainer is no longer usable", t->rank, (e - 1) & 15u, (e - 1) >> 4,
                   t->xchg_timeout_ns * 1e-9);
}

static int finish_loss(sb_trainer* t, float* loss_out) {
  SB_CUDA(cudaStreamSynchronize(t->net.stream));
  SB_TRY(poll_nccl(t));
  SB_TRY(poll_xchg(t));
  if (loss_out) {
    const float nnz = t->h_scal[SCAL_NNZ];
    *loss_out = nnz > 0.f ? t->h_scal[SCAL_LOSS_SUM] / nnz : 0.f;
  }
  return SB_OK;
}

static int stage_host_batch(sb_trainer* t, const float* X, const float* y, const float* w, int rows) {
  Net& n = t->net;
  SB_CHECK(X && y, SB_ERR_INVALID, "X and y must not be null");
  SB_CHECK(rows > 0 && rows <= n.max_batch, SB_ERR_INVALID, "rows=%d outside (0, max_batch=%d]", rows, n.max_batch);
  SB_CUDA(cudaSetDevice(n.device));
  SB_CUDA(cudaMemcpyAsync(n.stX, X, sizeof(float) * rows * static_cast<size_t>(n.F), cudaMemcpyHostToDevice, n.stream));
  SB_CUDA(cudaMemcpyAsync(n.stY, y, sizeof(float) * rows, cudaMemcpyHostToDevice, n.stream));
  if (w) SB_CUDA(cudaMemcpyAsync(n.stW, w, sizeof(float) * rows, cudaMemcpyHostToDevice, n.stream));
  return SB_OK;
}

extern "C" {

const char* sb_version(void) { return "shifu_b200 0.1 (sm_90a)"; }
const char* sb_last_error(void) { return last_error_ref().c_str(); }

int sb_device_count(void) {
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess) return set_error(SB_ERR_CUDA, "cudaGetDeviceCount failed");
  int ok = 0;
  for (int i = 0; i < n; ++i) {
    cudaDeviceProp p;
    if (cudaGetDeviceProperties(&p, i) == cudaSuccess && p.major == 9 && p.minor == 0) ++ok;
  }
  return ok;
}

int sb_device_mem_info(int device, uint64_t* free_bytes, uint64_t* total_bytes) {
  SB_CHECK(free_bytes && total_bytes, SB_ERR_INVALID, "null argument");
  SB_CUDA(cudaSetDevice(device));
  size_t f = 0, t = 0;
  SB_CUDA(cudaMemGetInfo(&f, &t));
  *free_bytes = f; *total_bytes = t;
  return SB_OK;
}

int sb_host_alloc(void** ptr, uint64_t bytes) {
  SB_CHECK(ptr, SB_ERR_INVALID, "ptr is null");
  SB_CUDA(cudaHostAlloc(ptr, bytes, cudaHostAllocDefault));
  return SB_OK;
}
int sb_host_free(void* ptr) {
  SB_CUDA(cudaFreeHost(ptr));
  return SB_OK;
}

int sb_nccl_unique_id(void* out128) {
  SB_CHECK(out128, SB_ERR_INVALID, "out is null");
  NcclApi* api = nccl_api();
  SB_CHECK(api, SB_ERR_NCCL, "libnccl.so.2 could not be loaded");
  NcclUniqueId id;
  int r = api->GetUniqueId(&id);
  SB_CHECK(r == 0, SB_ERR_NCCL, "ncclGetUniqueId failed: %s", api->GetErrorString(r));
  memcpy(out128, &id, sizeof(id));
  return SB_OK;
}

// Optimizer state that does not start at 0 (the arena's value): Adagrad's and FTRL's accum start at initial_accumulator,
// RMSProp's ms at 1 (TF's RMSPropOptimizer creates its `rms` slot with a ones initializer), RPROP's step size at the
// learning rate (torch.optim.Rprop's lr).  Every rank fills its whole state, so the runs a rank owns in the peer exchange
// start there as well.
static int fill_initial_state(sb_trainer* t) {
  Net& n = t->net;
  const int k = t->hyper.kind;
  if (opt_group(k) == OPT_RPROP) {
    fill_kernel<<<static_cast<unsigned>((n.n_params + 255) / 256), 256, 0, n.stream>>>(n.s2, t->lr, n.n_params);
    SB_CUDA(cudaGetLastError());
    return SB_OK;
  }
  if (k != SB_OPT_ADAGRAD && k != SB_OPT_FTRL && k != SB_OPT_RMSPROP) return SB_OK;
  const float v = k == SB_OPT_RMSPROP ? 1.f : t->initial_accumulator;
  fill_kernel<<<static_cast<unsigned>((n.n_params + 255) / 256), 256, 0, n.stream>>>(n.s1, v, n.n_params);
  SB_CUDA(cudaGetLastError());
  return SB_OK;
}

// Exchange slots over the work table: hidden layer 0 in row chunks of W_0 (128-row multiples; runs are 1024 parameters, so
// chunk borders fall on run borders when out % 8 == 0), the last chunk also carries b_0; everything else is slot 0.  With
// W_0 frozen there are no chunks, and slot 0 also carries b_0 if it trains.
static void set_exchange_slots(sb_trainer* t) {
  const Net& n = t->net;
  const Layer& l0 = n.layers[0];
  if (!t->w_trains[0]) {
    t->x_chunk_rows = 0;
    t->x_chunks = 0;
    t->x_slots = 1;
    t->x_begin[0] = n.work_begin[0]; t->x_end[0] = n.n_work;
    return;
  }
  int chunks = 2;
  if (!n.tc() || (l0.out % 8) != 0 || l0.in < 256 * chunks) chunks = 1;
  const int cr = round_up((l0.in + chunks - 1) / chunks, 128);
  chunks = (l0.in + cr - 1) / cr;           // (rounding to 128 rows may need fewer chunks)
  t->x_chunk_rows = cr;
  t->x_chunks = chunks;
  t->x_slots = 1 + chunks;
  t->x_begin[0] = n.work_end[0]; t->x_end[0] = n.n_work;
  for (int c = 0; c < chunks; ++c) {
    const long long e0 = static_cast<long long>(c) * cr * l0.out, e1 = static_cast<long long>(c + 1) * cr * l0.out;
    t->x_begin[1 + c] = n.work_begin[0] + static_cast<int>(e0 / 1024);
    t->x_end[1 + c] = (c == chunks - 1) ? n.work_end[0] : n.work_begin[0] + static_cast<int>(e1 / 1024);
  }
}

int sb_trainer_create(const sb_net_desc* desc, int device, const void* nccl_id, int rank, int world, sb_trainer_t** out) {
  SB_CHECK(out, SB_ERR_INVALID, "out is null");
  *out = nullptr;
  SB_TRY(validate_desc(desc));
  SB_CHECK(world >= 1 && rank >= 0 && rank < world, SB_ERR_INVALID, "bad rank/world %d/%d", rank, world);
  // world > 1 without an NCCL id: the ranks live in one process (sb_trainer_set_peer_pointers is then the only exchange)
  std::unique_ptr<sb_trainer> t(new sb_trainer());
  t->desc = *desc;
  t->rank = rank; t->world = world;
  t->lr = desc->learning_rate;
  t->hyper.kind = desc->optimizer;
  t->hyper.rho = desc->rho; t->hyper.eps = desc->epsilon;
  t->hyper.beta1 = desc->beta1; t->hyper.beta2 = desc->beta2; t->hyper.momentum = desc->momentum;
  t->hyper.l1 = 0.f; t->hyper.l2 = 0.f;
  {
    // parameter count is needed for the size of the gradient buffer that lives behind the parameters in the arena
    long long np = 0; int prev = desc->n_features;
    for (int l = 0; l <= desc->n_hidden; ++l) { const int out = l < desc->n_hidden ? desc->hidden[l] : 1; np += static_cast<long long>(prev) * out + out; prev = out; }
    t->xch_n4 = (np + 3) / 4;
    t->net.arena_extra_bytes = static_cast<size_t>(t->xch_n4) * 16 + sizeof(P2PFlags);
    // LL exchange buffers (xchg_p2p.cuh): gbuf = world regions, sbuf = one, of n4 entries x 32 bytes
    if (world > 1 && desc->precision == SB_PREC_BF16) {
      t->ll_ready = true;
      t->net.arena_extra_bytes += 256 + static_cast<size_t>(world + 1) * static_cast<size_t>(t->xch_n4) * 32;
    }
  }
  // from here on, a failed step returns and `t` releases whatever exists
  SB_TRY(t->net.init(desc, device, true));
  t->bufs[0].Xb = t->net.Xb;
  // see Net::init: no L1 / shared-memory re-partition between the kernels of a step
  write_desc_max_shared();
  for (auto k : optimizer_kernels) cudaFuncSetAttribute(k, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
  cudaFuncSetAttribute(axpy_kernel, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
  Net& n = t->net;
  // streams and events of the step schedule; the side stream's CTAs are scheduled behind the main chain's
  int prio_least = 0, prio_greatest = 0;
  SB_CUDA(cudaDeviceGetStreamPriorityRange(&prio_least, &prio_greatest));
  SB_CUDA(cudaStreamCreateWithPriority(&t->side, cudaStreamNonBlocking, prio_least));
  t->ev_dz.assign(n.L, nullptr);
  for (auto& e : t->ev_dz) SB_TRY(create_event(&e));
  SB_TRY(create_event(&t->ev_join));
  SB_TRY(create_event(&t->ev_da_done));
  for (auto& x : t->xstream) SB_CUDA(cudaStreamCreateWithFlags(&x, cudaStreamNonBlocking));
  // gradient + exchange flags behind the parameters, in the arena a single IPC handle exports
  t->xch = n.arena;
  t->grad_off = static_cast<long long>(n.extra_off);
  t->flags_off = t->grad_off + t->xch_n4 * 16;
  t->grad = reinterpret_cast<float*>(n.arena + t->grad_off);
  t->flags = reinterpret_cast<P2PFlags*>(n.arena + t->flags_off);
  if (t->ll_ready) {
    t->llg_off = (t->flags_off + static_cast<long long>(sizeof(P2PFlags)) + 255) / 256 * 256;
    t->lls_off = t->llg_off + static_cast<long long>(world) * t->xch_n4 * 32;
    // entries carry the epoch of the exchange that wrote them; epochs start at 1
    SB_CUDA(cudaMemset(n.arena + t->llg_off, 0, static_cast<size_t>(world + 1) * static_cast<size_t>(t->xch_n4) * 32));
  }
  t->s1 = n.s1; t->s2 = n.s2;
  SB_TRY(fill_initial_state(t.get()));
  SB_TRY(n.dalloc(&t->acc, n.n_params));
  SB_CUDA(cudaHostAlloc(reinterpret_cast<void**>(&t->h_err), sizeof(unsigned int) * 4, cudaHostAllocMapped));
  SB_CUDA(cudaHostGetDevicePointer(reinterpret_cast<void**>(&t->d_herr), t->h_err, 0));
  memset(t->h_err, 0, sizeof(unsigned int) * 4);
  if (const char* e = getenv("SB_XCHG_TIMEOUT_S")) t->xchg_timeout_ns = static_cast<unsigned long long>(atof(e) * 1e9);
  if (const char* e = getenv("SB_XCHG_BLOCKS")) t->xchg_blocks = atoi(e);
  // CTAs of a streamed step's overlapped fetch (DESIGN §6e measures the choice); a value outside [1, SMs / 2] keeps it
  if (const char* e = getenv("SB_FETCH_CTAS")) {
    const int k = atoi(e);
    if (k >= 1 && k <= t->net.num_sms / 2) t->fetch_ctas = k;
  }
  t->w_trains.assign(static_cast<size_t>(n.L + 1), 1);
  t->b_trains.assign(static_cast<size_t>(n.L + 1), 1);
  set_exchange_slots(t.get());
  for (int i = 0; i < SB_XCHG_SLOTS; ++i) {
    SB_TRY(create_event(&t->ev_x[i]));
    SB_TRY(create_event(&t->ev_c[i]));
  }
  SB_CUDA(cudaHostAlloc(reinterpret_cast<void**>(&t->h_scal), sizeof(float) * SCAL_COUNT, cudaHostAllocMapped));
  memset(t->h_scal, 0, sizeof(float) * SCAL_COUNT);
  SB_CUDA(cudaHostAlloc(reinterpret_cast<void**>(&t->h_hist), sizeof(float2) * sb_trainer::HIST, cudaHostAllocMapped));
  SB_CUDA(cudaHostGetDevicePointer(reinterpret_cast<void**>(&t->d_hist), t->h_hist, 0));
  memset(t->h_hist, 0, sizeof(float2) * sb_trainer::HIST);
  t->ring_desc[0][0] = n.desc;
  t->ring_scal[0][0] = n.scal;
  for (int set = 0; set < 2; ++set) {
    for (int k = set == 0 ? 1 : 0; k < sb_trainer::RUN_S; ++k) {
      SB_TRY(n.dalloc(&t->ring_desc[set][k], 1));
      SB_TRY(n.dalloc(&t->ring_scal[set][k], SCAL_COUNT));
    }
    SB_TRY(create_event(&t->ev_prep[set]));
    SB_TRY(create_event(&t->ev_pos[set]));
  }
  SB_CUDA(cudaStreamCreateWithFlags(&t->prep, cudaStreamNonBlocking));
  SB_CUDA(cudaHostGetDevicePointer(reinterpret_cast<void**>(&t->d_hscal), t->h_scal, 0));
  if (world > 1 && nccl_id != nullptr) {
    NcclApi* api = nccl_api();
    SB_CHECK(api, SB_ERR_NCCL, "libnccl.so.2 could not be loaded");
    NcclUniqueId id;
    memcpy(&id, nccl_id, sizeof(id));
    int r = api->CommInitRank(&t->comm, world, id, rank);
    SB_CHECK(r == 0, SB_ERR_NCCL, "ncclCommInitRank failed: %s", api->GetErrorString(r));
  }
  SB_CUDA(cudaStreamSynchronize(n.stream));
  *out = t.release();
  return SB_OK;
}

int sb_trainer_ipc_handle(sb_trainer_t* t, void* out64) {
  SB_CHECK(t && out64, SB_ERR_INVALID, "null argument");
  static_assert(sizeof(cudaIpcMemHandle_t) == SB_IPC_HANDLE_BYTES, "IPC handle size");
  SB_CUDA(cudaSetDevice(t->net.device));
  cudaIpcMemHandle_t h;
  SB_CUDA(cudaIpcGetMemHandle(&h, t->xch));
  memcpy(out64, &h, sizeof(h));
  return SB_OK;
}

// CUDA loads kernels lazily, at their first launch, and that load may synchronise the device: behind an exchange kernel that
// is still spinning for a peer whose work the same host thread has not queued yet (replicas in one process), the load - and
// with it the thread - would never return.  Everything a non-captured path launches around an exchange is loaded up front.
static int preload_exchange_kernels() {
  cudaFuncAttributes a;
  for (const auto& row : xchg_update_kernels)
    for (auto k : row) SB_CUDA(cudaFuncGetAttributes(&a, k));
  for (const auto& row : xchg_ll_kernels)
    for (auto k : row) SB_CUDA(cudaFuncGetAttributes(&a, k));
  SB_CUDA(cudaFuncGetAttributes(&a, gather_master_kernel));
  SB_TRY(write_desc_preload());
  SB_CUDA(cudaFuncGetAttributes(&a, scale_kernel));
  SB_CUDA(cudaFuncGetAttributes(&a, zero_f32_kernel));
  SB_CUDA(cudaFuncGetAttributes(&a, axpy_kernel));
  return SB_OK;
}

// peers' exchange allocations -> device table; bases[rank] is ignored (own allocation)
static int install_peer_table(sb_trainer* t, void* const* bases) {
  SB_TRY(preload_exchange_kernels());
  // every rank must freeze the same parameters (sb_trainer_set_fixed_layers): the slot tables define who owns which run.
  // Read each peer's masks from its flag block and refuse a mismatch instead of exchanging with it.
  for (int q = 0; q < t->world; ++q) {
    if (q == t->rank) continue;
    unsigned long long theirs[2] = {};
    const char* at = static_cast<const char*>(bases[q]) + t->flags_off + offsetof(P2PFlags, frozen);
    SB_CUDA(cudaMemcpyAsync(theirs, at, sizeof(theirs), cudaMemcpyDefault, t->net.stream));
    SB_CUDA(cudaStreamSynchronize(t->net.stream));
    if (theirs[0] != t->frozen_w || theirs[1] != t->frozen_b) {
      t->close_peer_mappings();
      return set_error(SB_ERR_INVALID, "rank %d fixes other parameters than rank %d (frozen W / b layer masks %#llx / %#llx vs "
                       "%#llx / %#llx): every rank needs the same sb_trainer_set_fixed_layers", q, t->rank, theirs[0], theirs[1],
                       t->frozen_w, t->frozen_b);
    }
  }
  P2PPeers hp;
  memset(&hp, 0, sizeof(hp));
  for (int q = 0; q < t->world; ++q) hp.base[q] = static_cast<char*>((q == t->rank) ? t->xch : bases[q]);
  if (!t->d_peers) SB_CUDA(cudaMalloc(&t->d_peers, sizeof(P2PPeers)));
  SB_CUDA(cudaMemcpy(t->d_peers, &hp, sizeof(hp), cudaMemcpyHostToDevice));
  t->drop_step_graphs();
  t->p2p_ready = true;
  return SB_OK;
}

int sb_trainer_set_peer_handles(sb_trainer_t* t, const void* handles, int32_t n_handles) {
  SB_CHECK(t && handles, SB_ERR_INVALID, "null argument");
  SB_CHECK(n_handles == t->world && t->world <= SB_MAX_RANKS, SB_ERR_INVALID, "expected %d handles (<= %d), got %d", t->world,
           SB_MAX_RANKS, n_handles);
  SB_CUDA(cudaSetDevice(t->net.device));
  SB_CUDA(cudaStreamSynchronize(t->net.stream));
  t->close_peer_mappings();
  t->p2p_ready = false;
  void* bases[SB_MAX_RANKS] = {};
  for (int q = 0; q < t->world; ++q) {
    if (q == t->rank) continue;
    cudaIpcMemHandle_t h;
    memcpy(&h, static_cast<const char*>(handles) + static_cast<size_t>(q) * sizeof(h), sizeof(h));
    cudaError_t e = cudaIpcOpenMemHandle(&bases[q], h, cudaIpcMemLazyEnablePeerAccess);
    if (e != cudaSuccess) {
      cudaGetLastError();
      t->close_peer_mappings();   // all or nothing: a half-mapped table must never be used
      return set_error(SB_ERR_CUDA, "cudaIpcOpenMemHandle(rank %d) failed: %s (no P2P path / separate IPC namespace?)", q,
                       cudaGetErrorString(e));
    }
    t->peer_bases.push_back(bases[q]);
  }
  return install_peer_table(t, bases);
}

int sb_trainer_clear_peer_handles(sb_trainer_t* t) {
  SB_CHECK(t, SB_ERR_INVALID, "null trainer");
  SB_CUDA(cudaSetDevice(t->net.device));
  SB_CUDA(cudaStreamSynchronize(t->net.stream));
  t->close_peer_mappings();
  if (t->p2p_ready) t->drop_step_graphs();
  t->p2p_ready = false;
  return SB_OK;
}

void* sb_trainer_exchange_base(sb_trainer_t* t) { return t ? t->xch : nullptr; }

int sb_trainer_set_peer_pointers(sb_trainer_t* t, void* const* bases, int32_t n) {
  SB_CHECK(t && bases, SB_ERR_INVALID, "null argument");
  SB_CHECK(n == t->world && t->world <= SB_MAX_RANKS, SB_ERR_INVALID, "expected %d pointers (<= %d), got %d", t->world,
           SB_MAX_RANKS, n);
  SB_CUDA(cudaSetDevice(t->net.device));
  SB_CUDA(cudaStreamSynchronize(t->net.stream));
  for (int q = 0; q < t->world; ++q) {
    if (q == t->rank) continue;
    SB_CHECK(bases[q] != nullptr, SB_ERR_INVALID, "pointer of rank %d is null", q);
    cudaPointerAttributes at;
    SB_CUDA(cudaPointerGetAttributes(&at, bases[q]));
    SB_CHECK(at.type == cudaMemoryTypeDevice, SB_ERR_INVALID, "pointer of rank %d is not device memory", q);
    if (at.device == t->net.device) t->peers_share_device = true;
    if (at.device != t->net.device) {
      int can = 0;
      SB_CUDA(cudaDeviceCanAccessPeer(&can, t->net.device, at.device));
      SB_CHECK(can, SB_ERR_CUDA, "device %d cannot access device %d (no P2P path)", t->net.device, at.device);
      cudaError_t e = cudaDeviceEnablePeerAccess(at.device, 0);
      if (e != cudaSuccess && e != cudaErrorPeerAccessAlreadyEnabled) return set_error(SB_ERR_CUDA, "cudaDeviceEnablePeerAccess failed: %s", cudaGetErrorString(e));
      cudaGetLastError();
    }
  }
  t->close_peer_mappings();
  return install_peer_table(t, bases);
}

int sb_trainer_destroy(sb_trainer_t* t) {
  if (!t) return SB_OK;
  cudaSetDevice(t->net.device);
  cudaStreamSynchronize(t->net.stream);
  delete t;
  return SB_OK;
}

int64_t sb_trainer_param_count(const sb_trainer_t* t) { return t ? t->net.n_params : 0; }

int sb_trainer_set_params(sb_trainer_t* t, const float* flat, int64_t n) {
  SB_CHECK(t && flat, SB_ERR_INVALID, "null argument");
  SB_CHECK(n == t->net.n_params, SB_ERR_INVALID, "expected %lld params, got %lld", (long long)t->net.n_params, (long long)n);
  SB_CUDA(cudaSetDevice(t->net.device));
  SB_CUDA(cudaMemcpyAsync(t->net.theta, flat, sizeof(float) * n, cudaMemcpyHostToDevice, t->net.stream));
  SB_TRY(t->net.refresh_shadows());
  SB_CUDA(cudaStreamSynchronize(t->net.stream));
  return SB_OK;   // (optimizer state is untouched: a sharded trainer keeps each run's state on its owner)
}

int sb_trainer_get_params(sb_trainer_t* t, float* flat, int64_t n) {
  SB_CHECK(t && flat, SB_ERR_INVALID, "null argument");
  SB_CHECK(n == t->net.n_params, SB_ERR_INVALID, "expected %lld params, got %lld", (long long)t->net.n_params, (long long)n);
  SB_CUDA(cudaSetDevice(t->net.device));
  SB_TRY(gather_master(t));
  SB_CUDA(cudaMemcpyAsync(flat, t->net.theta, sizeof(float) * n, cudaMemcpyDeviceToHost, t->net.stream));
  SB_CUDA(cudaStreamSynchronize(t->net.stream));
  return SB_OK;
}

int sb_trainer_init_xavier(sb_trainer_t* t, uint64_t seed) {
  SB_CHECK(t, SB_ERR_INVALID, "null trainer");
  // xavier_initializer() (uniform) on weights and biases, res/ssgd_monitor.py:59-68
  std::vector<float> flat(static_cast<size_t>(t->net.n_params));
  std::mt19937_64 rng(seed);
  for (const Layer& ly : t->net.layers) {
    const double lw = sqrt(6.0 / (ly.in + ly.out)), lb = sqrt(3.0 / ly.out);
    std::uniform_real_distribution<double> uw(-lw, lw), ub(-lb, lb);
    for (long long i = 0; i < static_cast<long long>(ly.in) * ly.out; ++i) flat[ly.w_off + i] = static_cast<float>(uw(rng));
    for (int i = 0; i < ly.out; ++i) flat[ly.b_off + i] = static_cast<float>(ub(rng));
  }
  return sb_trainer_set_params(t, flat.data(), t->net.n_params);
}

int sb_trainer_get_grads(sb_trainer_t* t, float* flat, int64_t n) {
  SB_CHECK(t && flat, SB_ERR_INVALID, "null argument");
  SB_CHECK(n == t->net.n_params, SB_ERR_INVALID, "expected %lld grads, got %lld", (long long)t->net.n_params, (long long)n);
  SB_CUDA(cudaSetDevice(t->net.device));
  if (t->p2p_ready && t->grad_sharded && t->world > 1) {
    // sharded exchange: every owner kept the reduced gradient of its runs; collect them (overwrites this rank's own
    // contributions, which the next step clears anyway)
    SB_CUDA(cudaStreamSynchronize(t->net.stream));
    gather_master_kernel<<<t->net.n_work, 256, 0, t->net.stream>>>(xchg_params(t, t->net.desc), 1);
    SB_CUDA(cudaGetLastError());
  }
  SB_CUDA(cudaMemcpyAsync(flat, t->grad, sizeof(float) * n, cudaMemcpyDeviceToHost, t->net.stream));
  SB_CUDA(cudaStreamSynchronize(t->net.stream));
  const float gs = t->grad_out_scale;
  if (gs != 1.f) for (int64_t i = 0; i < n; ++i) flat[i] *= gs;
  // a frozen parameter's gradient is 0 (a dA or output-layer epilogue that runs for the layers below may have written the
  // bias gradient of a frozen layer; no update reads it)
  for (size_t l = 0; l < t->net.layers.size(); ++l) {
    const Layer& ly = t->net.layers[l];
    if (!t->w_trains[l]) std::fill(flat + ly.w_off, flat + ly.w_off + static_cast<long long>(ly.in) * ly.out, 0.f);
    if (!t->b_trains[l]) std::fill(flat + ly.b_off, flat + ly.b_off + ly.out, 0.f);
  }
  return SB_OK;
}

int sb_trainer_step(sb_trainer_t* t, const float* X, const float* y, const float* w, int32_t rows, float* loss_out) {
  SB_CHECK(t, SB_ERR_INVALID, "null trainer");
  SB_TRY(stage_host_batch(t, X, y, w, rows));
  SB_TRY(run_step(t, host_batch(t->net, t->net.stX, t->net.stY, w ? t->net.stW : nullptr, rows), G_STEP));
  return finish_loss(t, loss_out);
}

// ---- wide+deep (BASELINE config 4): hidden layer 0 = [dense | one-hot]; the step feeds (dense block, index matrix) ----
int sb_trainer_set_sparse(sb_trainer_t* t, int32_t n_dense, int32_t n_onehot, int32_t n_cat) {
  SB_CHECK(t, SB_ERR_INVALID, "null trainer");
  SB_CHECK(!t->net.det, SB_ERR_STATE, "wide+deep on a deterministic trainer: the embedding gradient is scatter-added with "
           "red.global (embed_scatter_kernel), whose summation order is not fixed");
  return t->net.set_sparse(n_dense, n_onehot, n_cat);
}

int sb_trainer_set_deterministic(sb_trainer_t* t, int32_t on) {
  SB_CHECK(t, SB_ERR_INVALID, "null trainer");
  Net& n = t->net;
  if ((on != 0) == n.det) return SB_OK;
  SB_CHECK(!t->started && t->n_acc == 0 && t->global_step == 0, SB_ERR_STATE,
           "sb_trainer_set_deterministic after the first step or graph capture: set it right after sb_trainer_create");
  SB_CHECK(!t->p2p_ready, SB_ERR_STATE, "sb_trainer_set_deterministic after the peer exchange was set up: set it first");
  if (!on) { n.det = false; return SB_OK; }
  SB_CHECK(n.n_cat == 0, SB_ERR_STATE, "deterministic training of a wide+deep trainer: the embedding gradient is scatter-added "
           "with red.global (embed_scatter_kernel), whose summation order is not fixed");
  return n.enable_det();
}

int sb_trainer_set_optimizer_params(sb_trainer_t* t, float initial_accumulator, float l1, float l2) {
  SB_CHECK(t, SB_ERR_INVALID, "null trainer");
  const int k = t->hyper.kind;
  SB_CHECK(k == SB_OPT_ADAGRAD || k == SB_OPT_FTRL, SB_ERR_INVALID,
           "optimizer %d reads none of initial_accumulator, l1, l2 (Adagrad and FTRL do)", k);
  SB_CHECK(initial_accumulator > 0.f && std::isfinite(initial_accumulator), SB_ERR_INVALID,
           "initial_accumulator must be > 0 (got %g)", initial_accumulator);
  SB_CHECK(l1 >= 0.f && l2 >= 0.f && std::isfinite(l1) && std::isfinite(l2), SB_ERR_INVALID,
           "l1 and l2 must be >= 0 (got %g, %g)", l1, l2);
  SB_CHECK(k == SB_OPT_FTRL || (l1 == 0.f && l2 == 0.f), SB_ERR_INVALID, "Adagrad has no l1 / l2 (got %g, %g)", l1, l2);
  SB_CHECK(!t->started && t->n_acc == 0 && t->global_step == 0, SB_ERR_STATE,
           "sb_trainer_set_optimizer_params after the first step or graph capture: set it right after sb_trainer_create");
  SB_CUDA(cudaSetDevice(t->net.device));
  t->initial_accumulator = initial_accumulator;
  t->hyper.l1 = l1; t->hyper.l2 = l2;
  SB_TRY(fill_initial_state(t));
  SB_CUDA(cudaStreamSynchronize(t->net.stream));
  return SB_OK;
}

int sb_trainer_set_fixed_layers(sb_trainer_t* t, const int32_t* layers, int32_t n, int32_t fix_bias) {
  SB_CHECK(t, SB_ERR_INVALID, "null trainer");
  SB_CHECK(n >= 0, SB_ERR_INVALID, "n = %d must be >= 0", n);
  SB_CHECK(n == 0 || layers, SB_ERR_INVALID, "layers is null");
  Net& net = t->net;
  const int nl = net.L + 1;                    // layers 1..L hidden, L + 1 the output layer
  std::vector<char> w(static_cast<size_t>(nl), 1), b(static_cast<size_t>(nl), 1);
  for (int i = 0; i < n; ++i) {
    const int x = layers[i];
    SB_CHECK(x >= 1 && x <= nl, SB_ERR_INVALID, "fixed layer %d outside [1, %d] (hidden layers 1..%d, output layer %d)", x, nl,
             nl - 1, nl);
    SB_CHECK(w[static_cast<size_t>(x - 1)], SB_ERR_INVALID, "fixed layer %d listed twice", x);
    w[static_cast<size_t>(x - 1)] = 0;
    if (fix_bias) b[static_cast<size_t>(x - 1)] = 0;
  }
  int l_min = net.L;
  for (int l = net.L - 1; l >= 0; --l)
    if (w[static_cast<size_t>(l)] || b[static_cast<size_t>(l)]) l_min = l;
  const bool any = l_min < net.L || w[static_cast<size_t>(net.L)] || b[static_cast<size_t>(net.L)];
  SB_CHECK(any, SB_ERR_INVALID, "every parameter is fixed: nothing would train");
  SB_CHECK(!t->started && t->n_acc == 0 && t->global_step == 0, SB_ERR_STATE,
           "sb_trainer_set_fixed_layers after the first step or graph capture: set it right after sb_trainer_create");
  SB_CHECK(!t->p2p_ready, SB_ERR_STATE, "sb_trainer_set_fixed_layers after the peer exchange was set up: set it first");
  SB_CUDA(cudaSetDevice(net.device));
  SB_TRY(net.set_trainable(w, b));
  t->w_trains = w; t->b_trains = b;
  t->l_min = l_min;
  t->frozen_w = t->frozen_b = 0;
  for (int l = 0; l < nl; ++l) {
    if (!w[static_cast<size_t>(l)]) t->frozen_w |= 1ull << l;
    if (!b[static_cast<size_t>(l)]) t->frozen_b |= 1ull << l;
  }
  set_exchange_slots(t);
  // the peers compare the masks when their tables are set (install_peer_table)
  const unsigned long long masks[2] = {t->frozen_w, t->frozen_b};
  SB_CUDA(cudaMemcpyAsync(t->flags->frozen, masks, sizeof(masks), cudaMemcpyHostToDevice, net.stream));
  SB_CUDA(cudaStreamSynchronize(net.stream));
  return SB_OK;
}

static int stage_sparse_batch(Net& n, const float* Xd, const int32_t* idx, const float* y, const float* w, int rows) {
  SB_CHECK(n.n_cat > 0, SB_ERR_STATE, "sb_trainer_set_sparse has not been called");
  SB_CHECK(Xd && idx, SB_ERR_INVALID, "Xd and idx must not be null");
  SB_CHECK(rows > 0 && rows <= n.max_batch, SB_ERR_INVALID, "rows=%d outside (0, max_batch=%d]", rows, n.max_batch);
  SB_TRY(check_sparse_idx(idx, static_cast<long long>(rows) * n.n_cat, n.n_onehot));
  SB_CUDA(cudaSetDevice(n.device));
  SB_CUDA(cudaMemcpyAsync(n.stX, Xd, sizeof(float) * rows * static_cast<size_t>(n.n_dense), cudaMemcpyHostToDevice, n.stream));
  SB_CUDA(cudaMemcpyAsync(n.idx, idx, sizeof(int32_t) * rows * static_cast<size_t>(n.n_cat), cudaMemcpyHostToDevice, n.stream));
  if (y) SB_CUDA(cudaMemcpyAsync(n.stY, y, sizeof(float) * rows, cudaMemcpyHostToDevice, n.stream));
  if (w) SB_CUDA(cudaMemcpyAsync(n.stW, w, sizeof(float) * rows, cudaMemcpyHostToDevice, n.stream));
  return SB_OK;
}

int sb_trainer_step_sparse(sb_trainer_t* t, const float* Xd, const int32_t* idx, const float* y, const float* w, int32_t rows,
                           float* loss_out) {
  SB_CHECK(t && y, SB_ERR_INVALID, "null argument");
  SB_TRY(stage_sparse_batch(t->net, Xd, idx, y, w, rows));
  SB_TRY(run_step(t, host_batch(t->net, t->net.stX, t->net.stY, w ? t->net.stW : nullptr, rows, Feed::SPARSE), G_STEP));
  return finish_loss(t, loss_out);
}

// forward (+ loss: y != nullptr) over any number of sparse rows; out / loss accumulators nullable
static int forward_sparse(sb_trainer* t, const float* Xd, const int32_t* idx, const float* y, const float* w, int64_t rows,
                          float* out, double* loss_sum, double* nnz) {
  Net& n = t->net;
  return forward_chunks(t, rows, [&](int64_t r0, int c, Batch* b) -> int {
    SB_TRY(stage_sparse_batch(n, Xd + r0 * n.n_dense, idx + r0 * n.n_cat, y ? y + r0 : nullptr, (y && w) ? w + r0 : nullptr, c));
    *b = host_batch(n, n.stX, n.stY, (y && w) ? n.stW : nullptr, c, Feed::SPARSE);
    return SB_OK;
  }, out, loss_sum, nnz);
}

int sb_trainer_predict_sparse(sb_trainer_t* t, const float* Xd, const int32_t* idx, int64_t rows, float* out) {
  SB_CHECK(t && out, SB_ERR_INVALID, "null argument");
  return forward_sparse(t, Xd, idx, nullptr, nullptr, rows, out, nullptr, nullptr);
}

int sb_trainer_eval_loss_sparse(sb_trainer_t* t, const float* Xd, const int32_t* idx, const float* y, const float* w, int64_t rows,
                                float* loss_out) {
  SB_CHECK(t && y && loss_out && rows > 0, SB_ERR_INVALID, "bad argument");
  double ls = 0, nz = 0;
  SB_TRY(forward_sparse(t, Xd, idx, y, w, rows, nullptr, &ls, &nz));
  *loss_out = nz > 0 ? static_cast<float>(ls / nz) : 0.f;
  return SB_OK;
}

int sb_trainer_step_async(sb_trainer_t* t, const float* X, const float* y, const float* w, int32_t rows) {
  SB_CHECK(t && X && y, SB_ERR_INVALID, "null argument");
  Net& n = t->net;
  SB_CHECK(rows > 0 && rows <= n.max_batch, SB_ERR_INVALID, "rows=%d outside (0, max_batch=%d]", rows, n.max_batch);
  SB_CUDA(cudaSetDevice(n.device));
  if (!t->copy_ready) {
    if (!t->copy_stream) SB_CUDA(cudaStreamCreateWithFlags(&t->copy_stream, cudaStreamNonBlocking));
    if (!t->st2X) SB_TRY(n.dalloc(&t->st2X, static_cast<size_t>(n.max_batch) * n.F));
    if (!t->st2Y) SB_TRY(n.dalloc(&t->st2Y, n.max_batch));
    if (!t->st2W) SB_TRY(n.dalloc(&t->st2W, n.max_batch));
    for (int i = 0; i < 2; ++i) {
      SB_TRY(create_event(&t->ev_copied[i]));
      SB_TRY(create_event(&t->ev_consumed[i]));
    }
    SB_CUDA(cudaStreamSynchronize(n.stream));   // the zero-fill of the new staging buffers ran on the main stream
    t->copy_ready = true;
  }
  const int slot = static_cast<int>(t->async_steps & 1);
  float* sx = slot ? t->st2X : n.stX;
  float* sy = slot ? t->st2Y : n.stY;
  float* sw = slot ? t->st2W : n.stW;
  // the slot is free once the step that consumed it two calls ago has finished
  if (t->async_steps >= 2) SB_CUDA(cudaStreamWaitEvent(t->copy_stream, t->ev_consumed[slot], 0));
  SB_CUDA(cudaMemcpyAsync(sx, X, sizeof(float) * rows * static_cast<size_t>(n.F), cudaMemcpyHostToDevice, t->copy_stream));
  SB_CUDA(cudaMemcpyAsync(sy, y, sizeof(float) * rows, cudaMemcpyHostToDevice, t->copy_stream));
  if (w) SB_CUDA(cudaMemcpyAsync(sw, w, sizeof(float) * rows, cudaMemcpyHostToDevice, t->copy_stream));
  SB_CUDA(cudaEventRecord(t->ev_copied[slot], t->copy_stream));
  SB_CUDA(cudaStreamWaitEvent(n.stream, t->ev_copied[slot], 0));
  SB_TRY(run_step(t, host_batch(n, sx, sy, w ? sw : nullptr, rows), G_STEP));
  SB_CUDA(cudaEventRecord(t->ev_consumed[slot], n.stream));
  ++t->async_steps;
  return SB_OK;
}

int sb_trainer_accumulate(sb_trainer_t* t, const float* X, const float* y, const float* w, int32_t rows, float* loss_out) {
  SB_CHECK(t, SB_ERR_INVALID, "null trainer");
  SB_TRY(stage_host_batch(t, X, y, w, rows));
  SB_TRY(run_step(t, host_batch(t->net, t->net.stX, t->net.stY, w ? t->net.stW : nullptr, rows), G_ACC));
  return finish_loss(t, loss_out);
}

static int apply_accumulated_impl(sb_trainer_t* t, int64_t total_pushes);

int sb_trainer_apply_accumulated(sb_trainer_t* t) {
  SB_CHECK(t, SB_ERR_INVALID, "null trainer");
  SB_CHECK(t->n_acc > 0, SB_ERR_STATE, "no accumulated gradients");
  return apply_accumulated_impl(t, static_cast<int64_t>(t->world) * t->n_acc);
}

int sb_trainer_apply_accumulated_mean(sb_trainer_t* t, int64_t total_pushes) {
  SB_CHECK(t, SB_ERR_INVALID, "null trainer");
  SB_CHECK(total_pushes > 0, SB_ERR_INVALID, "total_pushes must be > 0");
  return apply_accumulated_impl(t, total_pushes);
}

static int apply_accumulated_impl(sb_trainer_t* t, int64_t total_pushes) {
  Net& n = t->net;
  SB_CUDA(cudaSetDevice(n.device));
  const float gscale = 1.f / static_cast<float>(total_pushes);
  const float lr_t = begin_update(t);
  // the last prefetched set: the next descriptor prefetch writes the other one, possibly while this update runs
  const StepIn in = t->slot(t->last_set, 0);
  SB_TRY(write_desc(n.stream, in, nullptr, lr_t, gscale, t->epoch, nullptr));
  // exchange + apply through the (IPC-exported) gradient buffer; it then holds the applied mean for sb_trainer_get_grads
  SB_CUDA(cudaMemcpyAsync(t->grad, t->acc, sizeof(float) * n.n_params, cudaMemcpyDeviceToDevice, n.stream));
  if (t->world > 1 && t->p2p_ready) {
    SB_TRY(enqueue_xchg(t, in, xseg_all(t), n.stream, false, false));
  } else {
    SB_TRY(enqueue_allreduce(t, t->grad));
    SB_TRY(enqueue_optimizer(t, in, t->grad));
  }
  const long long np = n.n_params;
  scale_kernel<<<static_cast<unsigned>((np + 255) / 256), 256, 0, n.stream>>>(t->grad, in.desc, np);
  SB_CUDA(cudaGetLastError());
  t->grad_out_scale = 1.f;  // scale_kernel already applied 1/(world * n_acc)
  zero_f32_kernel<<<static_cast<unsigned>((np + 255) / 256), 256, 0, n.stream>>>(t->acc, np);   // (a preloaded kernel, see preload_exchange_kernels)
  SB_CUDA(cudaGetLastError());
  // queued, not waited for (like a step): with a peer exchange inside, a host thread that drives several replicas must be able
  // to queue the update on all of them before any can complete; everything that reads the result synchronises the stream
  t->n_acc = 0;
  return SB_OK;
}

// Where sb_trainer_load_dataset puts the set's rows (X in GEMM-operand form; y, w and the prefix counts always go to HBM):
// in HBM if they fit beside what the trainer still allocates after the load, else in mapped pinned host memory.  The
// reserve counts, besides the set's 12 bytes per row of y, w and P: a row order of every row (4 bytes per row), the
// conversion windows, batch y / w, and once more what the net allocated for its step buffers - the margin for what is
// sized like them later (the deterministic workspaces, graph instantiation, the validation forward's chunks).
static int place_dataset(sb_trainer* t, int64_t n_rows, size_t x_bytes, size_t win_bytes, bool* host) {
  const Net& n = t->net;
  size_t free_b = 0, total_b = 0;
  SB_CUDA(cudaMemGetInfo(&free_b, &total_b));
  const size_t reserve = 16 * static_cast<size_t>(n_rows) + win_bytes + 8 * static_cast<size_t>(n.max_batch) + n.dalloc_bytes;
  *host = t->force_host || x_bytes + reserve > free_b;
  return SB_OK;
}

// X / y / w of load_dataset, eval_loss and predict may be HOST or DEVICE pointers (unified addressing: the copies use
// cudaMemcpyDefault); the GPU text ingest hands over device arrays so that the parsed set never visits the host
int sb_trainer_load_dataset(sb_trainer_t* t, const float* X, const float* y, const float* w, int64_t n_rows) {
  SB_CHECK(t && X && y, SB_ERR_INVALID, "null argument");
  SB_CHECK(n_rows > 0 && n_rows < (1ll << 31), SB_ERR_INVALID, "n_rows must be in (0, 2^31)");
  Net& n = t->net;
  SB_CUDA(cudaSetDevice(n.device));
  SB_CUDA(cudaStreamSynchronize(n.stream));
  t->drop_step_graphs();   // captured steps carry tensor maps of the old set
  t->free_dataset();
  // X is converted through a bounded fp32 window (and, for a set in host memory, a bf16 window) so that a 100+ GB set
  // never needs a second full copy
  const int64_t win = 32768, wrows = win < n_rows ? win : n_rows;
  const size_t part_elems = static_cast<size_t>(n_rows) * n.ldF;
  const size_t x_bytes = n.tc() ? sizeof(__nv_bfloat16) * part_elems * n.nparts : sizeof(float) * static_cast<size_t>(n_rows) * n.F;
  const size_t win_bytes = n.tc() ? static_cast<size_t>(wrows) * (sizeof(float) * n.F + sizeof(__nv_bfloat16) * n.ldF * n.nparts) : 0;
  bool host = false;
  SB_TRY(place_dataset(t, n_rows, x_bytes, win_bytes, &host));
  void* xs = nullptr;
  if (host) {
    // mapped + portable: with unified addressing the host address is also the address kernels read it at
    const cudaError_t e = cudaHostAlloc(&xs, x_bytes, cudaHostAllocMapped | cudaHostAllocPortable);
    if (e != cudaSuccess) {
      cudaGetLastError();
      return set_error(SB_ERR_CUDA, "the resident set does not fit in device memory and %zu bytes of pinned host memory for its "
                       "%lld rows could not be allocated: %s", x_bytes, (long long)n_rows, cudaGetErrorString(e));
    }
  } else {
    SB_CUDA(cudaMalloc(&xs, x_bytes));
  }
  t->ds_host = host;
  if (n.tc()) t->dsXb = static_cast<__nv_bfloat16*>(xs);
  else t->dsX = static_cast<float*>(xs);
  SB_CUDA(cudaMalloc(&t->dsY, sizeof(float) * n_rows));
  SB_CUDA(cudaMalloc(&t->dsW, sizeof(float) * n_rows));
  SB_CUDA(cudaMemcpyAsync(t->dsY, y, sizeof(float) * n_rows, cudaMemcpyDefault, n.stream));
  if (w) {
    SB_CUDA(cudaMemcpyAsync(t->dsW, w, sizeof(float) * n_rows, cudaMemcpyDefault, n.stream));
  } else {
    fill_kernel<<<static_cast<unsigned>((n_rows + 255) / 256), 256, 0, n.stream>>>(t->dsW, 1.f, n_rows);
    SB_CUDA(cudaGetLastError());
  }
  if (n.tc()) {
    // keep the set in the form the layer-0 GEMMs consume (bf16, row pitch ldF; split modes: nparts such arrays),
    // converted once here.  In HBM it is read by TMA every step; in host memory gather_batch_kernel copies each batch's
    // rows into Xb.  A host set is converted in a device window and copied out part by part, so it holds the same bits.
    t->ds_ps = static_cast<long long>(part_elems);
    DevBuf<float> tmp;
    DevBuf<__nv_bfloat16> wb;
    SB_TRY(tmp.alloc(static_cast<size_t>(wrows) * n.F));
    const long long wps = host ? wrows * n.ldF : t->ds_ps;   // part stride of the cast's destination
    if (host) {
      SB_TRY(wb.alloc(static_cast<size_t>(wps) * n.nparts));
      SB_CUDA(cudaMemsetAsync(wb.p, 0, sizeof(__nv_bfloat16) * wps * n.nparts, n.stream));   // pad columns (never written)
    } else {
      SB_CUDA(cudaMemsetAsync(t->dsXb, 0, x_bytes, n.stream));
    }
    for (int64_t r0 = 0; r0 < n_rows; r0 += win) {
      const int64_t c = n_rows - r0 < win ? n_rows - r0 : win;
      SB_CUDA(cudaMemcpyAsync(tmp.p, X + r0 * n.F, sizeof(float) * c * n.F, cudaMemcpyDefault, n.stream));
      __nv_bfloat16* dst = host ? wb.p : t->dsXb + r0 * n.ldF;
      cast_bf16_kernel<<<static_cast<unsigned>((c * n.F + 255) / 256), 256, 0, n.stream>>>(tmp.p, static_cast<int>(c), n.F,
                                                                                           dst, n.ldF, n.nparts, wps);
      SB_CUDA(cudaGetLastError());
      for (int k = 0; host && k < n.nparts; ++k)
        SB_CUDA(cudaMemcpyAsync(t->dsXb + k * t->ds_ps + r0 * n.ldF, wb.p + k * wps, sizeof(__nv_bfloat16) * c * n.ldF,
                                cudaMemcpyDefault, n.stream));
      SB_CUDA(cudaStreamSynchronize(n.stream));   // X may be pageable: the window is reused
    }
    std::vector<int> prefix(static_cast<size_t>(n_rows) + 1);
    prefix[0] = 0;
    std::vector<float> w_host;
    const float* wh = w;
    if (ptr_device(w) >= 0) {    // 4 bytes per row: the only part of a device-resident set the host looks at
      w_host.resize(static_cast<size_t>(n_rows));
      SB_CUDA(cudaMemcpy(w_host.data(), w, sizeof(float) * n_rows, cudaMemcpyDeviceToHost));
      wh = w_host.data();
    }
    for (int64_t i = 0; i < n_rows; ++i) prefix[i + 1] = prefix[i] + ((wh == nullptr || wh[i] != 0.f) ? 1 : 0);
    SB_CUDA(cudaMalloc(&t->dsP, sizeof(int) * (n_rows + 1)));
    SB_CUDA(cudaMemcpyAsync(t->dsP, prefix.data(), sizeof(int) * (n_rows + 1), cudaMemcpyHostToDevice, n.stream));
    SB_CUDA(cudaStreamSynchronize(n.stream));
    if (host) {
      // (4 bytes per row, inside the reserve's row order)
      for (int64_t i = 0; i < n_rows; ++i) prefix[i] = static_cast<int>(i);
      SB_CUDA(cudaMalloc(&t->ds_iota, sizeof(int) * n_rows));
      SB_CUDA(cudaMemcpy(t->ds_iota, prefix.data(), sizeof(int) * n_rows, cudaMemcpyHostToDevice));
      // the streamed steps' batch buffers and the fetch branch
      SB_TRY(t->alloc_batch_bufs(true));
      if (!t->fetch_stream) SB_CUDA(cudaStreamCreateWithFlags(&t->fetch_stream, cudaStreamNonBlocking));
      SB_TRY(create_event(&t->ev_fork));
      SB_TRY(create_event(&t->ev_fetched));
    }
  } else {
    SB_CUDA(cudaMemcpyAsync(t->dsX, X, sizeof(float) * n_rows * n.F, cudaMemcpyDefault, n.stream));
  }
  SB_CUDA(cudaStreamSynchronize(n.stream));
  t->ds_rows = n_rows;
  return SB_OK;
}

int sb_debug_force_host_set(sb_trainer_t* t, int32_t on) {
  SB_CHECK(t, SB_ERR_INVALID, "null trainer");
  SB_CHECK(on == 0 || on == 1, SB_ERR_INVALID, "on = %d: 0 or 1", on);
  t->force_host = on != 0;
  return SB_OK;
}

int sb_trainer_dataset_on_host(const sb_trainer_t* t) { return t && t->ds_rows > 0 && t->ds_host ? 1 : 0; }

static int resident_step(sb_trainer_t* t, int64_t row_offset, int32_t rows, int kind) {
  SB_CHECK(t, SB_ERR_INVALID, "null trainer");
  Batch b;
  SB_TRY(resident_batch(t, row_offset, rows, -1, 0, &b));
  return run_step(t, b, kind);
}

int sb_trainer_run_resident(sb_trainer_t* t, const int64_t* row_offsets, int32_t n_steps, int32_t rows) {
  SB_CHECK(t && row_offsets, SB_ERR_INVALID, "null argument");
  SB_CHECK(n_steps >= 0, SB_ERR_INVALID, "n_steps must be >= 0");
  SB_CHECK(t->ds_rows > 0, SB_ERR_STATE, "no resident dataset loaded");
  Net& n = t->net;
  SB_CHECK(rows > 0 && rows <= n.max_batch, SB_ERR_INVALID, "rows=%d outside (0, max_batch=%d]", rows, n.max_batch);
  Batch b;
  for (int i = 0; i < n_steps; ++i) SB_TRY(resident_batch(t, row_offsets[i], rows, i, 0, &b));
  constexpr int S = sb_trainer::RUN_S;
  int i = 0;
  SB_TRY(check_det_exchange(t));
  const Feed feed = t->resident_feed();
  if (feed != Feed::HOST) {      // (the fp32 set without an order runs one host-batch graph per step, not prefetched)
    SB_CUDA(cudaSetDevice(n.device));
    const float gscale = 1.f / static_cast<float>(t->world);
    for (; i + S <= n_steps; i += S) {
      const int set = static_cast<int>(t->prefetches & 1);
      cudaGraphExec_t ge = nullptr;
      SB_TRY(get_graph(t, GraphKey{rows, G_STEP, feed, S, set}, &ge));
      SB_TRY(prefetch_begin(t, set));
      for (int k = 0; k < S; ++k) {
        SB_TRY(resident_batch(t, row_offsets[i + k], rows, i + k, k, &b));
        const float lr_t = begin_update(t);
        SB_TRY(write_desc(t->prep, t->slot(set, k), &b, lr_t, gscale, t->epoch, t->hist_slot(t->global_step)));
      }
      SB_TRY(prefetch_end(t, set));
      SB_CUDA(cudaGraphLaunch(ge, n.stream));
      t->grad_out_scale = gscale;
    }
  }
  for (; i < n_steps; ++i) SB_TRY(resident_step(t, row_offsets[i], rows, G_STEP));
  return SB_OK;
}

int sb_trainer_step_resident(sb_trainer_t* t, int64_t row_offset, int32_t rows, float* loss_out) {
  SB_TRY(resident_step(t, row_offset, rows, G_STEP));
  return finish_loss(t, loss_out);
}
int sb_trainer_step_resident_async(sb_trainer_t* t, int64_t row_offset, int32_t rows) {
  return resident_step(t, row_offset, rows, G_STEP);
}
int sb_trainer_accumulate_resident(sb_trainer_t* t, int64_t row_offset, int32_t rows, float* loss_out) {
  SB_TRY(resident_step(t, row_offset, rows, G_ACC));
  return finish_loss(t, loss_out);
}
int sb_trainer_loss_resident(sb_trainer_t* t, int64_t row_offset, int32_t rows, float* loss_out) {
  SB_CHECK(t && loss_out, SB_ERR_INVALID, "null argument");
  Batch b;
  SB_TRY(resident_batch(t, row_offset, rows, -1, 0, &b));
  Net& n = t->net;
  SB_CUDA(cudaSetDevice(n.device));
  t->have_pos = false;
  const StepIn in = t->slot(0, 0, b.feed);      // (see forward_chunks)
  SB_TRY(enqueue_forward(n, t, in, b, t->epoch, true, nullptr));
  float h[SCAL_COUNT];
  SB_CUDA(cudaMemcpyAsync(h, in.scal, sizeof(h), cudaMemcpyDeviceToHost, n.stream));
  SB_CUDA(cudaStreamSynchronize(n.stream));
  *loss_out = h[SCAL_NNZ] > 0.f ? h[SCAL_LOSS_SUM] / h[SCAL_NNZ] : 0.f;
  return SB_OK;
}

int sb_trainer_broadcast_state(sb_trainer_t* t, int32_t root) {
  SB_CHECK(t, SB_ERR_INVALID, "null trainer");
  if (t->world <= 1) return SB_OK;
  SB_CHECK(root >= 0 && root < t->world, SB_ERR_INVALID, "root %d outside [0, %d)", root, t->world);
  NcclApi* api = nccl_api();
  SB_CHECK(api && t->comm, SB_ERR_NCCL, "no NCCL communicator");
  Net& n = t->net;
  SB_CUDA(cudaSetDevice(n.device));
  DevBuf<long long> d_step;
  SB_TRY(d_step.alloc(1));
  SB_CUDA(cudaMemcpyAsync(d_step.p, &t->global_step, sizeof(long long), cudaMemcpyHostToDevice, n.stream));
  int r = api->Broadcast(n.theta, n.theta, static_cast<size_t>(n.n_params), NCCL_FLOAT32, root, t->comm, n.stream);
  if (r == 0) r = api->Broadcast(t->s1, t->s1, static_cast<size_t>(n.n_params), NCCL_FLOAT32, root, t->comm, n.stream);
  if (r == 0) r = api->Broadcast(t->s2, t->s2, static_cast<size_t>(n.n_params), NCCL_FLOAT32, root, t->comm, n.stream);
  if (r == 0) r = api->Broadcast(d_step.p, d_step.p, 1, NCCL_INT64, root, t->comm, n.stream);
  SB_CHECK(r == 0, SB_ERR_NCCL, "ncclBroadcast failed: %s", api->GetErrorString(r));
  long long step = 0;
  SB_CUDA(cudaMemcpyAsync(&step, d_step.p, sizeof(long long), cudaMemcpyDeviceToHost, n.stream));
  SB_TRY(n.refresh_shadows());
  SB_CUDA(cudaStreamSynchronize(n.stream));
  t->global_step = step;
  return poll_nccl(t);
}

int sb_trainer_loss_history(sb_trainer_t* t, int64_t first_step, int32_t n, float* out) {
  SB_CHECK(t && out, SB_ERR_INVALID, "null argument");
  SB_CHECK(n >= 0 && first_step >= 1 && first_step + n - 1 <= t->global_step, SB_ERR_INVALID,
           "steps [%lld, %lld] outside [1, global_step=%lld]", (long long)first_step, (long long)(first_step + n - 1), (long long)t->global_step);
  SB_CHECK(t->global_step - first_step < sb_trainer::HIST, SB_ERR_INVALID, "only the last %d steps are kept", (int)sb_trainer::HIST);
  SB_CUDA(cudaSetDevice(t->net.device));
  SB_CUDA(cudaStreamSynchronize(t->net.stream));
  SB_TRY(poll_nccl(t));
  for (int i = 0; i < n; ++i) {
    const float2 v = t->h_hist[(first_step + i) % sb_trainer::HIST];
    out[i] = v.y > 0.f ? v.x / v.y : 0.f;
  }
  return SB_OK;
}

int sb_trainer_last_loss(sb_trainer_t* t, float* loss_out) {
  SB_CHECK(t && loss_out, SB_ERR_INVALID, "null argument");
  return finish_loss(t, loss_out);
}
int sb_trainer_sync(sb_trainer_t* t) {
  SB_CHECK(t, SB_ERR_INVALID, "null trainer");
  SB_CUDA(cudaStreamSynchronize(t->net.stream));
  SB_TRY(poll_nccl(t));
  SB_TRY(poll_xchg(t));
  return SB_OK;
}
void* sb_trainer_stream(sb_trainer_t* t) { return t ? reinterpret_cast<void*>(t->net.stream) : nullptr; }

int sb_trainer_kernels_per_step(sb_trainer_t* t, int32_t rows) {
  SB_CHECK(t, SB_ERR_INVALID, "null trainer");
  cudaGraphExec_t ge;
  const Feed feed = t->resident_feed();   // the path resident steps take now (no set loaded: host-batch steps)
  SB_TRY(get_graph(t, GraphKey{rows, G_STEP, feed, 1, 0}, &ge));
  return t->kernels_per_step[{rows, feed}];
}

int sb_trainer_set_row_order(sb_trainer_t* t, const int64_t* rows, int64_t n) {
  SB_CHECK(t, SB_ERR_INVALID, "null trainer");
  SB_CHECK((rows == nullptr && n == 0) || (rows != nullptr && n >= 1 && n < (1ll << 31)), SB_ERR_INVALID,
           "row order of %lld rows (%s list): give 1 <= n < 2^31 rows, or NULL and 0 for the physical order", (long long)n,
           rows ? "non-null" : "null");
  SB_CHECK(t->ds_rows > 0, SB_ERR_STATE, "no resident dataset loaded");
  std::vector<int> h(static_cast<size_t>(n));
  for (int64_t i = 0; i < n; ++i) {
    SB_CHECK(rows[i] >= 0 && rows[i] < t->ds_rows, SB_ERR_INVALID, "row order entry %lld = %lld outside the resident set of %lld rows",
             (long long)i, (long long)rows[i], (long long)t->ds_rows);
    h[static_cast<size_t>(i)] = static_cast<int>(rows[i]);
  }
  Net& net = t->net;
  SB_CUDA(cudaSetDevice(net.device));
  // steps already queued read the current order (and batch buffer 0) when they run; the graphs read the order through the
  // descriptor, so neither a new buffer nor new contents need a new capture
  SB_CUDA(cudaStreamSynchronize(net.stream));
  if (n == 0) { t->drop_row_order(); return SB_OK; }
  SB_TRY(t->alloc_batch_bufs(false));
  if (n > t->ord_cap) {
    t->drop_row_order();
    SB_CUDA(cudaMalloc(&t->ord, sizeof(int) * n));
    t->ord_cap = n;
  }
  SB_CUDA(cudaMemcpyAsync(t->ord, h.data(), sizeof(int) * n, cudaMemcpyHostToDevice, net.stream));
  SB_CUDA(cudaStreamSynchronize(net.stream));
  t->ord_n = n;
  return SB_OK;
}

// forward (+ loss: y != nullptr) over any number of host or device rows; out / loss accumulators nullable
static int forward_rows(sb_trainer* t, const float* X, const float* y, const float* w, int64_t rows, float* out,
                        double* loss_sum, double* nnz) {
  Net& n = t->net;
  return forward_chunks(t, rows, [&](int64_t r0, int c, Batch* b) -> int {
    SB_CUDA(cudaMemcpyAsync(n.stX, X + r0 * n.F, sizeof(float) * c * static_cast<size_t>(n.F), cudaMemcpyDefault, n.stream));
    if (y) {
      SB_CUDA(cudaMemcpyAsync(n.stY, y + r0, sizeof(float) * c, cudaMemcpyDefault, n.stream));
      if (w) SB_CUDA(cudaMemcpyAsync(n.stW, w + r0, sizeof(float) * c, cudaMemcpyDefault, n.stream));
    }
    *b = host_batch(n, n.stX, n.stY, (y && w) ? n.stW : nullptr, c);
    return SB_OK;
  }, out, loss_sum, nnz);
}

int sb_trainer_eval_loss(sb_trainer_t* t, const float* X, const float* y, const float* w, int64_t rows, float* loss_out) {
  SB_CHECK(t && X && y && loss_out, SB_ERR_INVALID, "null argument");
  SB_CHECK(rows > 0, SB_ERR_INVALID, "rows must be > 0");
  double ls = 0, nz = 0;
  SB_TRY(forward_rows(t, X, y, w, rows, nullptr, &ls, &nz));
  *loss_out = nz > 0 ? static_cast<float>(ls / nz) : 0.f;
  return SB_OK;
}

int sb_trainer_predict(sb_trainer_t* t, const float* X, int64_t rows, float* out) {
  SB_CHECK(t && X && out, SB_ERR_INVALID, "null argument");
  SB_CHECK(rows > 0, SB_ERR_INVALID, "rows must be > 0");
  return forward_rows(t, X, nullptr, nullptr, rows, out, nullptr, nullptr);
}

// ---- checkpoint: flat blob {magic, version, n_params, global_step, optimizer, theta, s1, s2} ----
static const uint64_t CKPT_MAGIC = 0x5348494655423230ull;  // "SHIFUB20"

int sb_trainer_save_checkpoint(sb_trainer_t* t, const char* path) {
  SB_CHECK(t && path, SB_ERR_INVALID, "null argument");
  Net& n = t->net;
  SB_CUDA(cudaSetDevice(n.device));
  SB_TRY(gather_master(t));
  std::vector<float> buf(static_cast<size_t>(n.n_params) * 3);
  SB_CUDA(cudaMemcpyAsync(buf.data(), n.theta, sizeof(float) * n.n_params, cudaMemcpyDeviceToHost, n.stream));
  SB_CUDA(cudaMemcpyAsync(buf.data() + n.n_params, t->s1, sizeof(float) * n.n_params, cudaMemcpyDeviceToHost, n.stream));
  SB_CUDA(cudaMemcpyAsync(buf.data() + 2 * n.n_params, t->s2, sizeof(float) * n.n_params, cudaMemcpyDeviceToHost, n.stream));
  SB_CUDA(cudaStreamSynchronize(n.stream));
  std::string tmp = std::string(path) + ".tmp";
  FILE* f = fopen(tmp.c_str(), "wb");
  SB_CHECK(f, SB_ERR_IO, "cannot open %s for writing", tmp.c_str());
  uint64_t hdr[5] = {CKPT_MAGIC, 1, static_cast<uint64_t>(n.n_params), static_cast<uint64_t>(t->global_step),
                     static_cast<uint64_t>(t->hyper.kind)};
  bool ok = fwrite(hdr, sizeof(hdr), 1, f) == 1 && fwrite(buf.data(), sizeof(float), buf.size(), f) == buf.size();
  ok = (fclose(f) == 0) && ok;
  SB_CHECK(ok, SB_ERR_IO, "short write to %s", tmp.c_str());
  SB_CHECK(rename(tmp.c_str(), path) == 0, SB_ERR_IO, "rename to %s failed", path);
  return SB_OK;
}

int sb_trainer_load_checkpoint(sb_trainer_t* t, const char* path) {
  SB_CHECK(t && path, SB_ERR_INVALID, "null argument");
  Net& n = t->net;
  FILE* f = fopen(path, "rb");
  SB_CHECK(f, SB_ERR_IO, "cannot open %s", path);
  uint64_t hdr[5];
  std::vector<float> buf(static_cast<size_t>(n.n_params) * 3);
  bool ok = fread(hdr, sizeof(hdr), 1, f) == 1;
  ok = ok && hdr[0] == CKPT_MAGIC && hdr[2] == static_cast<uint64_t>(n.n_params);
  ok = ok && fread(buf.data(), sizeof(float), buf.size(), f) == buf.size();
  fclose(f);
  SB_CHECK(ok, SB_ERR_FORMAT, "%s is not a checkpoint of this network", path);
  SB_CHECK(hdr[4] == static_cast<uint64_t>(t->hyper.kind), SB_ERR_FORMAT,
           "%s was written by optimizer %d, this trainer uses optimizer %d: the saved optimizer state does not apply", path,
           static_cast<int>(hdr[4]), t->hyper.kind);
  SB_CUDA(cudaSetDevice(n.device));
  SB_CUDA(cudaMemcpyAsync(n.theta, buf.data(), sizeof(float) * n.n_params, cudaMemcpyHostToDevice, n.stream));
  SB_CUDA(cudaMemcpyAsync(t->s1, buf.data() + n.n_params, sizeof(float) * n.n_params, cudaMemcpyHostToDevice, n.stream));
  SB_CUDA(cudaMemcpyAsync(t->s2, buf.data() + 2 * n.n_params, sizeof(float) * n.n_params, cudaMemcpyHostToDevice, n.stream));
  SB_TRY(n.refresh_shadows());
  SB_CUDA(cudaStreamSynchronize(n.stream));
  t->global_step = static_cast<long long>(hdr[3]);
  return SB_OK;
}

int64_t sb_trainer_global_step(const sb_trainer_t* t) { return t ? t->global_step : 0; }

int sb_trainer_export_savedmodel(sb_trainer_t* t, const char* export_dir) {
  SB_CHECK(t && export_dir, SB_ERR_INVALID, "null argument");
  std::vector<float> flat(static_cast<size_t>(t->net.n_params));
  SB_TRY(sb_trainer_get_params(t, flat.data(), t->net.n_params));
  return sb_savedmodel_write(export_dir, &t->desc, flat.data(), t->net.n_params);
}

// ================================================================================================
// step-timeline test hook (the kernel-level hooks are in net.cu, beside the step's GEMM launches)
// ================================================================================================
int sb_debug_step_trace(sb_trainer_t* t, uint64_t* stamps, int32_t cap_kernels, char* names, int32_t names_cap, int32_t* n_kernels) {
  SB_CHECK(t && stamps && n_kernels, SB_ERR_INVALID, "null argument");
  Net& n = t->net;
  SB_CHECK(n.step_trace != nullptr, SB_ERR_STATE, "create the trainer with SB_STEP_TRACE=1 in the environment");
  SB_CUDA(cudaSetDevice(n.device));
  SB_CUDA(cudaStreamSynchronize(n.stream));
  const int k = n.trace_n < cap_kernels ? n.trace_n : cap_kernels;
  SB_CUDA(cudaMemcpy(stamps, n.step_trace, sizeof(uint64_t) * 16 * k, cudaMemcpyDeviceToHost));
  *n_kernels = k;
  if (names && names_cap > 0) {
    std::string all;
    for (int i = 0; i < k; ++i) { if (i) all += ','; all += n.trace_names[i]; }
    snprintf(names, names_cap, "%s", all.c_str());
  }
  return SB_OK;
}

// ================================================================================================
// exchange test hooks: a rank's raw arena buffers, one exchange launch as a step queues it, the ownership tables
// ================================================================================================
// The input-stage buffers of sb_debug_trainer_buffer (SB_DEBUG_BUF_BATCH_X .. _DS_P): one device range per part, laid
// out one behind the other on the host
static int input_buffer(sb_trainer* t, int which, void* host, int64_t count, bool write) {
  Net& n = t->net;
  struct Range { void* dev; long long elems; };
  std::vector<Range> rs;
  size_t esz = sizeof(float);
  const bool bf = n.tc();
  const bool resident = which >= SB_DEBUG_BUF_DS_X;
  SB_CHECK(!resident || t->ds_rows > 0, SB_ERR_STATE, "buffer %d: no resident dataset loaded", which);
  const long long ds = t->ds_rows;
  switch (which) {
    case SB_DEBUG_BUF_BATCH_X:
      if (bf) {
        const int ldx = n.n_cat > 0 ? n.ldD : n.ldF;
        esz = sizeof(uint16_t);
        for (int k = 0; k < n.nparts; ++k) rs.push_back({n.Xb + k * n.Xb_ps, static_cast<long long>(n.max_batch) * ldx});
      } else {
        rs.push_back({n.Xf, static_cast<long long>(n.max_batch) * n.F});
      }
      break;
    case SB_DEBUG_BUF_BATCH_Y: rs.push_back({t->gathers() ? t->bufs[0].y : n.stY, n.max_batch}); break;
    case SB_DEBUG_BUF_BATCH_W: rs.push_back({t->gathers() ? t->bufs[0].w : n.stW, n.max_batch}); break;
    case SB_DEBUG_BUF_SCAL: rs.push_back({t->slot(0, 0).scal, SCAL_COUNT}); break;
    case SB_DEBUG_BUF_DS_X:
      if (bf) {
        esz = sizeof(uint16_t);
        for (int k = 0; k < n.nparts; ++k) rs.push_back({t->dsXb + k * t->ds_ps, ds * n.ldF});
      } else {
        rs.push_back({t->dsX, ds * n.F});
      }
      break;
    case SB_DEBUG_BUF_DS_Y: rs.push_back({t->dsY, ds}); break;
    case SB_DEBUG_BUF_DS_W: rs.push_back({t->dsW, ds}); break;
    default:   // SB_DEBUG_BUF_DS_P
      SB_CHECK(t->dsP, SB_ERR_STATE, "buffer %d: the fp32 resident set has no prefix counts", which);
      esz = sizeof(int);
      rs.push_back({t->dsP, ds + 1});
  }
  long long total = 0;
  for (const Range& r : rs) total += r.elems;
  SB_CHECK(count == total, SB_ERR_INVALID, "buffer %d: expected %lld values, got %lld", which, total, (long long)count);
  SB_CUDA(cudaSetDevice(n.device));
  SB_CUDA(cudaStreamSynchronize(n.stream));
  char* h = static_cast<char*>(host);
  for (const Range& r : rs) {
    const size_t bytes = esz * static_cast<size_t>(r.elems);
    // (cudaMemcpyDefault: the resident set may be in host memory)
    if (write) SB_CUDA(cudaMemcpyAsync(r.dev, h, bytes, cudaMemcpyHostToDevice, n.stream));
    else SB_CUDA(cudaMemcpyAsync(h, r.dev, bytes, cudaMemcpyDefault, n.stream));
    h += bytes;
  }
  SB_CUDA(cudaStreamSynchronize(n.stream));
  return SB_OK;
}

int sb_debug_trainer_buffer(sb_trainer_t* t, int32_t which, void* host, int64_t n, int32_t write) {
  const bool input = which >= SB_DEBUG_BUF_BATCH_X && which <= SB_DEBUG_BUF_DS_P;
  SB_CHECK((which >= SB_DEBUG_BUF_THETA && which < SB_DEBUG_BUF_SHADOW + SB_MAX_HIDDEN) || input, SB_ERR_INVALID,
           "buffer %d is not a buffer id", which);
  SB_CHECK(write >= 0 && write <= 2 && (write != 2 || which == SB_DEBUG_BUF_THETA), SB_ERR_INVALID,
           "write = %d: 0 reads, 1 writes, 2 writes theta and refreshes the shadows", write);
  SB_CHECK(write == 0 || which < SB_DEBUG_BUF_DS_X, SB_ERR_INVALID, "buffer %d (the resident set) is read-only", which);
  SB_CHECK(t && host, SB_ERR_INVALID, "null argument");
  Net& net = t->net;
  if (input) return input_buffer(t, which, host, n, write != 0);
  SB_CHECK(which < SB_DEBUG_BUF_SHADOW + net.L, SB_ERR_INVALID, "buffer %d outside [0, %d)", which, SB_DEBUG_BUF_SHADOW + net.L);
  if (which < SB_DEBUG_BUF_SHADOW) {
    SB_CHECK(n == net.n_params, SB_ERR_INVALID, "expected %lld floats, got %lld", (long long)net.n_params, (long long)n);
    float* dev = which == SB_DEBUG_BUF_THETA ? net.theta : which == SB_DEBUG_BUF_S1 ? net.s1 : which == SB_DEBUG_BUF_S2 ? net.s2 : t->grad;
    SB_CUDA(cudaSetDevice(net.device));
    SB_CUDA(cudaStreamSynchronize(net.stream));
    if (write) SB_CUDA(cudaMemcpyAsync(dev, host, sizeof(float) * n, cudaMemcpyHostToDevice, net.stream));
    else SB_CUDA(cudaMemcpyAsync(host, dev, sizeof(float) * n, cudaMemcpyDeviceToHost, net.stream));
    if (write == 2) SB_TRY(net.refresh_shadows());
  } else {
    const int l = which - SB_DEBUG_BUF_SHADOW;
    SB_CHECK(net.tc(), SB_ERR_STATE, "layer %d has no bf16 shadow in fp32 mode", l);
    const Layer& ly = net.layers[l];
    const long long part = static_cast<long long>(ly.in) * ly.ld_out;
    SB_CHECK(n == part * net.nparts, SB_ERR_INVALID, "expected %d x %d x %d bf16 values, got %lld", net.nparts, ly.in, ly.ld_out,
             (long long)n);
    SB_CUDA(cudaSetDevice(net.device));
    SB_CUDA(cudaStreamSynchronize(net.stream));
    for (int k = 0; k < net.nparts; ++k) {
      uint16_t* h = static_cast<uint16_t*>(host) + k * part;
      __nv_bfloat16* d = ly.Wn + k * net.Wn_ps[l];
      if (write) SB_CUDA(cudaMemcpyAsync(d, h, sizeof(uint16_t) * part, cudaMemcpyHostToDevice, net.stream));
      else SB_CUDA(cudaMemcpyAsync(h, d, sizeof(uint16_t) * part, cudaMemcpyDeviceToHost, net.stream));
    }
  }
  SB_CUDA(cudaStreamSynchronize(net.stream));
  return SB_OK;
}

int sb_debug_first_kernel(sb_trainer_t* t, const float* X, const float* y, const float* w, const int32_t* idx, int64_t row_offset,
                          int32_t rows, int32_t clear, char* route, int32_t route_cap) {
  SB_CHECK(clear == 0 || clear == 1, SB_ERR_INVALID, "clear = %d: 0 or 1", clear);
  SB_CHECK(route_cap >= 0 && (route != nullptr || route_cap == 0), SB_ERR_INVALID, "route_cap %d without a buffer", route_cap);
  SB_CHECK(X != nullptr || (y == nullptr && w == nullptr && idx == nullptr), SB_ERR_INVALID,
           "resident rows (X null) take no y, w or idx");
  SB_CHECK(X == nullptr || (y != nullptr && row_offset == 0), SB_ERR_INVALID, "host rows need y and take no row_offset");
  SB_CHECK(t, SB_ERR_INVALID, "null trainer");
  Net& n = t->net;
  Batch b;
  if (X == nullptr) {
    SB_TRY(resident_batch(t, row_offset, rows, -1, 0, &b));
  } else if (n.n_cat > 0) {   // as sb_trainer_step_sparse
    SB_TRY(stage_sparse_batch(n, X, idx, y, w, rows));
    b = host_batch(n, n.stX, n.stY, w ? n.stW : nullptr, rows, Feed::SPARSE);
  } else {                    // as sb_trainer_step
    SB_CHECK(idx == nullptr, SB_ERR_INVALID, "idx on a trainer without sb_trainer_set_sparse");
    SB_TRY(stage_host_batch(t, X, y, w, rows));
    b = host_batch(n, n.stX, n.stY, w ? n.stW : nullptr, rows);
  }
  SB_CUDA(cudaSetDevice(n.device));
  // as run_step for a batch it does not prefetch: set 0 written on the main stream, then what enqueue_step_body queues
  // ahead of layer 0
  const StepIn in = t->slot(0, 0, b.feed);
  t->have_pos = false;
  SB_TRY(write_desc(n.stream, in, &b, t->lr, 1.f / static_cast<float>(t->world), t->epoch, nullptr));
  std::string r;
  n.marks = &r;
  const int s = enqueue_first(n, t, in, b.rows, clear ? t->grad : nullptr, clear ? n.n_params : 0);
  n.marks = nullptr;
  SB_TRY(s);
  SB_CUDA(cudaStreamSynchronize(n.stream));
  if (route_cap > 0) snprintf(route, static_cast<size_t>(route_cap), "%s", r.empty() ? "none" : r.c_str());
  return SB_OK;
}

int sb_debug_exchange(sb_trainer_t* t, int32_t slot_mask, float gscale, int32_t grid, int32_t alone, float* lr_t_out,
                      int32_t* grid_out, char* route, int32_t route_cap) {
  SB_CHECK(t, SB_ERR_INVALID, "null trainer");
  SB_CHECK(t->world > 1 && t->p2p_ready, SB_ERR_STATE, "no peers configured (world = %d): set the peer table first", t->world);
  SB_CHECK(slot_mask > 0 && (slot_mask & ~xseg_all(t)) == 0, SB_ERR_INVALID, "slot mask 0x%x outside 0x%x (%d slots)", slot_mask,
           xseg_all(t), t->x_slots);
  SB_CHECK(std::isfinite(gscale) && gscale >= 0.f, SB_ERR_INVALID, "gscale %g is not a finite value >= 0", gscale);
  SB_CHECK(grid >= 0 && grid <= 65535, SB_ERR_INVALID, "grid %d outside [0, 65535]", grid);
  SB_CHECK(route_cap >= 0 && (route != nullptr || route_cap == 0), SB_ERR_INVALID, "route_cap %d without a buffer", route_cap);
  Net& n = t->net;
  SB_CUDA(cudaSetDevice(n.device));
  // as a step: the descriptor of this update (step count, lr_t, gradient scale, epoch), then the exchange on the main stream.
  // Nothing here waits for the device - the peers' launches are still to be queued by the same host thread.
  const float lr_t = begin_update(t);
  const float gs = gscale > 0.f ? gscale : 1.f / static_cast<float>(t->world);
  const StepIn in = t->slot(t->last_set, 0);    // (as apply_accumulated)
  SB_TRY(write_desc(n.stream, in, nullptr, lr_t, gs, t->epoch, nullptr));
  if (grid <= 0) grid = xchg_grid(t, slot_mask, alone != 0);
  n.last_kernel = nullptr;
  SB_TRY(enqueue_xchg(t, in, slot_mask, n.stream, false, false, alone != 0, grid));
  t->grad_out_scale = gs;
  if (lr_t_out) *lr_t_out = lr_t;
  if (grid_out) *grid_out = grid;
  if (route_cap > 0) snprintf(route, static_cast<size_t>(route_cap), "%s", n.last_kernel ? n.last_kernel : "");
  return SB_OK;
}

int sb_debug_optimizer(sb_trainer_t* t, float gscale, int32_t tail, float* lr_t_out, char* route, int32_t route_cap) {
  SB_CHECK(t, SB_ERR_INVALID, "null trainer");
  SB_CHECK(std::isfinite(gscale) && gscale >= 0.f, SB_ERR_INVALID, "gscale %g is not a finite value >= 0", gscale);
  SB_CHECK(tail == 0 || tail == 1, SB_ERR_INVALID, "tail = %d: 0 runs one pass over the work table, 1 the split tail", tail);
  SB_CHECK(tail == 0 || t->net.L > 1, SB_ERR_INVALID, "the split tail needs two hidden layers (the net has %d)", t->net.L);
  SB_CHECK(route_cap >= 0 && (route != nullptr || route_cap == 0), SB_ERR_INVALID, "route_cap %d without a buffer", route_cap);
  SB_CHECK(t->world == 1, SB_ERR_STATE, "world = %d: a peer update is sb_debug_exchange, an NCCL rank needs its communicator",
           t->world);
  Net& n = t->net;
  SB_CUDA(cudaSetDevice(n.device));
  // as a single-GPU update: the descriptor (step count, lr_t, gradient scale, epoch), then the optimizer as
  // apply_accumulated and the non-split step queue it (tail = 0) or as the step's split tail (tail = 1)
  const float lr_t = begin_update(t);
  const float gs = gscale > 0.f ? gscale : 1.f / static_cast<float>(t->world);
  const StepIn in = t->slot(t->last_set, 0);    // (as apply_accumulated)
  SB_TRY(write_desc(n.stream, in, nullptr, lr_t, gs, t->epoch, nullptr));
  std::string r;
  if (tail) {
    SB_CUDA(cudaEventRecord(t->ev_da_done, n.stream));     // no dA GEMM here to record it
    SB_TRY(enqueue_split_tail(t, in, t->grad, &r));
  } else {
    SB_TRY(enqueue_optimizer(t, in, t->grad, 0, -1, nullptr, true, false, &r));
  }
  t->grad_out_scale = gs;
  if (lr_t_out) *lr_t_out = lr_t;
  if (route_cap > 0) snprintf(route, static_cast<size_t>(route_cap), "%s", r.c_str());
  return SB_OK;
}

int sb_debug_exchange_layout(sb_trainer_t* t, int32_t* info, int32_t info_cap, int64_t* work, int64_t work_cap, int32_t* n_work) {
  SB_CHECK(t && info && n_work, SB_ERR_INVALID, "null argument");
  SB_CHECK(info_cap >= SB_DEBUG_XINFO_WORDS, SB_ERR_INVALID, "info needs %d words, got %d", SB_DEBUG_XINFO_WORDS, info_cap);
  Net& n = t->net;
  SB_CHECK(work == nullptr || work_cap >= static_cast<int64_t>(n.n_work) * SB_DEBUG_XWORK_WORDS, SB_ERR_INVALID,
           "work needs %lld words, got %lld", static_cast<long long>(n.n_work) * SB_DEBUG_XWORK_WORDS, (long long)work_cap);
  *n_work = n.n_work;
  memset(info, 0, sizeof(int32_t) * SB_DEBUG_XINFO_WORDS);
  info[0] = t->x_slots; info[1] = n.num_sms; info[2] = t->ll_ready; info[3] = t->peers_share_device;
  info[4] = t->rank; info[5] = t->world; info[6] = n.nparts;
  for (int s = 0; s < SB_XCHG_SLOTS; ++s) { info[8 + s] = t->x_begin[s]; info[16 + s] = t->x_end[s]; }
  if (work == nullptr) return SB_OK;
  std::vector<OptWork> wk(static_cast<size_t>(n.n_work));
  SB_CUDA(cudaSetDevice(n.device));
  SB_CUDA(cudaStreamSynchronize(n.stream));
  SB_CUDA(cudaMemcpy(wk.data(), n.work, sizeof(OptWork) * wk.size(), cudaMemcpyDeviceToHost));
  for (int i = 0; i < n.n_work; ++i) {
    int64_t* o = work + static_cast<size_t>(i) * SB_DEBUG_XWORK_WORDS;
    int layer = -1;
    for (int l = 0; l < n.L; ++l) if (wk[i].Wn != nullptr && wk[i].Wn == n.layers[l].Wn) layer = l;
    o[0] = wk[i].off; o[1] = wk[i].count; o[2] = wk[i].out_dim; o[3] = wk[i].mat_off;
    o[4] = wk[i].ld_out; o[5] = wk[i].np; o[6] = layer; o[7] = wk[i].part_stride;
  }
  return SB_OK;
}

}  // extern "C"
