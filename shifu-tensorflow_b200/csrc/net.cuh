// Device-side network state shared by the trainer and the scorer: parameters, bf16 shadow weights,
// activation workspace, and the enqueue_* routines that put the step's kernels on a stream.
#pragma once
#include <vector>
#include <map>
#include <mutex>
#include "common.cuh"
#include "gemm_tc.cuh"
#include "gemm_f32.cuh"
#include "kernels.cuh"
#include "nccl_dyn.h"

namespace sb {

struct Layer {
  int in, out, act;
  long long w_off, b_off;              // offsets into the flat parameter vector
  __nv_bfloat16* Wn = nullptr;  // bf16 shadow of W [in, ld_out] (row-major like the fp32 master)
  int ld_in = 0, ld_out = 0;
};

// Where layer 0 of a step gets its batch:
//   HOST      fp32 rows at desc->X (the staging area, or the fp32 resident set): load_batch_kernel fills Xb / Xf
//   SPARSE    wide+deep: dense block + index matrix, hidden layer 0's one-hot block via the embedding
//   RESIDENT  layer 0's GEMMs read their A operand by TMA from the resident set (StepIn::x0) at row offset desc->row0
//   ORDERED   resident rows through the row order: gather_batch_kernel fills Xb / Xf, layer 0 reads them
//   STREAMED  rows of a bf16 set in mapped host memory: gather_batch_kernel fetches them over PCIe into one of two batch
//             buffers, in a run_resident graph one step ahead, beside the previous step's GEMMs (capi.cu, DESIGN §6e)
enum class Feed { HOST, SPARSE, RESIDENT, ORDERED, STREAMED };

// Layer 0's bf16 A operand in tensor-core modes: nparts arrays `ps` elements apart, whose tensor maps span `rows` rows
// (0: the batch rows).  at_row0: the TMA row coordinate is offset by desc->row0 (the resident set, read in place).
struct Operand0 { const __nv_bfloat16* p = nullptr; long long ps = 0; int rows = 0; bool at_row0 = false; };

// What one step's launches read: its descriptor / scalar slot, its feed and layer 0's operand (unset: the net's own Xb,
// Net::layer0).  The trainer takes the slots of its captured steps from a ring of descriptor sets (capi.cu).
struct StepIn {
  BatchDesc* desc = nullptr;
  float* scal = nullptr;
  Feed feed = Feed::HOST;
  Operand0 x0;
};

// One step's batch: everything set_batch_kernel reads besides the update's scalars (write_desc)
struct Batch {
  Feed feed = Feed::HOST;
  const float *X = nullptr, *y = nullptr, *w = nullptr;
  int row0 = 0;                     // RESIDENT: first row in the resident set
  const int* nz_prefix = nullptr;   // RESIDENT: n_nz is published from the set's prefix counts
  const int* order = nullptr;       // ORDERED: the batch's slice of the row order
  int rows = 0;
};

inline int pairs_of(int np) { return np == 3 ? 6 : (np == 2 ? 3 : 1); }

struct Net {
  int device = 0, num_sms = 132;
  cudaStream_t stream = nullptr;
  std::vector<int> work_begin, work_end;     // optimizer work-table range of layer l (0..L)
  int F = 0, L = 0;             // features, hidden layers
  std::vector<Layer> layers;    // L hidden + 1 output (out = 1)
  long long n_params = 0;
  int precision = SB_PREC_FP32, loss = SB_LOSS_MSE;
  // tensor-core modes keep every GEMM operand as `nparts` bf16 arrays (1 = plain bf16; 3 = SB_PREC_FP32_TC; 2 = BF16X2),
  // see GemmTcParams in gemm_tc.cuh.  Part k of a buffer lies k * <buffer>_ps elements behind part 0.
  int nparts = 1;
  bool tc() const { return precision != SB_PREC_FP32; }
  long long Xb_ps = 0;                       // part strides (elements)
  std::vector<long long> A_ps, Wn_ps;        // A_ps[l] also applies to dZ[l]
  int max_batch = 0, ldB = 0, ldF = 0;
  bool training = false;

  // Parameter arena: ONE allocation [theta fp32 | s1 | s2 (training) | bf16 weight shadows | extra], so that a trainer can
  // export everything the peer-memory exchange touches with a single CUDA-IPC handle (xchg_p2p.cuh).  `arena_extra_bytes`
  // is set by the trainer BEFORE init(): room for its gradient buffer and flag block behind the parameters.
  char* arena = nullptr;
  size_t arena_bytes = 0, arena_extra_bytes = 0;
  // Set BEFORE init() on an ensemble member (score.cu sb_ensemble): the net runs on input_from's stream and uses its input
  // staging (stX, Xb / Xf) instead of creating its own; input_from must have the same F and max_batch and outlive it.
  const Net* input_from = nullptr;
  size_t s1_off = 0, s2_off = 0, shadow_off = 0, extra_off = 0;   // byte offsets inside the arena (theta at 0)
  float* theta = nullptr;
  float *s1 = nullptr, *s2 = nullptr;      // optimizer state (training only)
  // bf16 workspace
  __nv_bfloat16* Xb = nullptr;             // current batch as bf16 [rows, ldF]
  std::vector<__nv_bfloat16*> A, dZ;       // A_l, dZ_l as bf16 [rows, ld_out_l]
  // fp32 workspace
  float* Xf = nullptr;
  std::vector<float*> Af, dZf;
  float *yhat = nullptr, *ones = nullptr;
  BatchDesc* desc = nullptr;               // the net's own descriptor / scalar slot (set 0, slot 0 of a trainer's ring)
  float* scal = nullptr;
  float *stX = nullptr, *stY = nullptr, *stW = nullptr;  // H2D staging (device)
  // The optimizer's work table: the runs of every parameter that trains (all of them unless set_trainable froze some).
  // work_all / n_work_all: every run, which the shadow refresh walks.
  OptWork* work = nullptr;
  int n_work = 0;
  OptWork* work_all = nullptr;
  int n_work_all = 0;
  OptWork* work_part = nullptr;            // the table's storage once set_trainable left parameters out
  int build_work(const std::vector<char>& w_trains, const std::vector<char>& b_trains, std::vector<OptWork>* wk,
                 std::vector<int>* begin, std::vector<int>* end) const;
  // Freeze parameters (fine-tuning, sb_trainer_set_fixed_layers): the work table and work_begin / work_end keep only the runs
  // of W_l where w_trains[l] and of b_l where b_trains[l] (l = 0..L).  Frozen runs are never updated or shadow-refreshed by
  // a step.
  int set_trainable(const std::vector<char>& w_trains, const std::vector<char>& b_trains);
  int launches = 0;  // kernels enqueued since last reset (for gpu_launches accounting)
  // SB_STEP_TRACE=1: every GEMM of a step stamps %globaltimer milestones of its CTA 0 into 16 slots (debug timeline)
  unsigned long long* step_trace = nullptr;
  int trace_k = 0;
  std::vector<std::string> trace_names;
  bool trace_on = true;
  int trace_n = 0;                 // kernels of the last traced step
  // name = role (+ layer, + ".chunk"); GEMMs append "@MxNxK" so that a reader needs no knowledge of the launch order
  unsigned long long* next_trace(const char* name, int layer = -1, int M = 0, int N = 0, int K = 0, int chunk = -1) {
    if (!step_trace || !trace_on || trace_k >= 32) return nullptr;
    if (static_cast<int>(trace_names.size()) <= trace_k) trace_names.resize(trace_k + 1);
    std::string nm = name;
    if (layer >= 0) nm += std::to_string(layer);
    if (chunk >= 0) nm += "." + std::to_string(chunk);
    if (M > 0) nm += "@" + std::to_string(M) + "x" + std::to_string(N) + "x" + std::to_string(K);
    trace_names[trace_k] = nm;
    trace_n = trace_k + 1;
    return step_trace + 16 * (trace_k++);
  }
  // every launch of an enqueue_* routine: `kernel` names the kernel and tile it launched (sb_debug_gemm_layer reports it)
  const char* last_kernel = nullptr;
  std::string* marks = nullptr;   // non-null: every launch's name is appended, "+"-joined (sb_debug_first_kernel,
                                  // sb_debug_model_routes)
  void mark(const char* kernel) {
    ++launches; last_kernel = kernel;
    if (marks) { if (!marks->empty()) *marks += '+'; *marks += kernel; }
  }

  std::vector<void*> allocs;
  size_t dalloc_bytes = 0;   // what dalloc allocated so far
  template <typename T> int dalloc(T** p, size_t n) {
    void* q = nullptr;
    SB_CUDA(cudaMalloc(&q, n * sizeof(T) + 256));
    allocs.push_back(q);
    dalloc_bytes += n * sizeof(T) + 256;
    SB_CUDA(cudaMemsetAsync(q, 0, n * sizeof(T) + 256, stream));
    *p = reinterpret_cast<T*>(q);
    return SB_OK;
  }

  Net() = default;
  Net(const Net&) = delete;
  Net& operator=(const Net&) = delete;
  ~Net();   // waits for the stream, frees every allocation and the stream
  int init(const sb_net_desc* d, int device_, bool training_);
  int refresh_shadows();
  // forward through the hidden layers (A_0 = current batch -> A_L).  The load kernel clears clear[0, clear_n) on the way.
  int enqueue_load(const StepIn& in, int rows, float* clear = nullptr, long long clear_n = 0);
  // grad != nullptr (training step): the last hidden layer's GEMM also runs the output layer, the loss and the output
  // backward in its epilogue when h_L <= 128; *fused_out tells the caller whether enqueue_out is still needed.  clear
  // (resident steps): the layer-0 GEMM's idle producer warps clear clear[0, clear_n4) beside its main loop.  first > 0
  // starts at hidden layer `first`, whose input A_{first-1} the caller has written (sb_model_sensitivity: layer 0's
  // rank-1 updates).
  int enqueue_hidden_forward(const StepIn& in, int rows, float* grad = nullptr, bool* fused_out = nullptr, float4* clear = nullptr,
                             long long clear_n4 = 0, int first = 0);
  // wide+deep first layer (oracle/wide_deep.py): hidden layer 0 = [n_dense numeric columns | n_onehot one-hot columns of
  // n_cat categorical columns]; a SPARSE step feeds (dense block, index matrix) and evaluates the one-hot block as an
  // embedding gather / scatter-add.  F = n_dense + n_onehot, the parameters are those of the dense net.
  int n_dense = 0, n_onehot = 0, n_cat = 0, ldD = 0;
  int* idx = nullptr;                        // [max_batch, n_cat] staged indices
  float* E = nullptr;                        // [max_batch, ld_out_0] embedding sums
  int set_sparse(int n_dense_, int n_onehot_, int n_cat_);
  int enqueue_embed(int rows, bool scatter, float* grad, cudaStream_t st);
  // layer 0's A operand of a step over `rows` batch rows: in.x0, or, unset, Xb
  Operand0 layer0(const StepIn& in, int rows) const {
    return in.x0.p ? Operand0{in.x0.p, in.x0.ps, in.x0.rows ? in.x0.rows : rows, in.x0.at_row0} : Operand0{Xb, Xb_ps, rows};
  }
  int enqueue_out(const StepIn& in, int rows, bool do_loss, bool do_bwd, float* yhat_dst, float* grad);
  // layer 0's pre-activation of the batch's rows to fp32 z [rows, ld_z] (sb_model_sensitivity): tensor-core modes
  // X W0 from the bf16 parts by the fp32-store GEMM (every part pair, fp32 accumulator stored as it is, no bias), fp32
  // mode X W0 + b0 by the fp32 GEMM
  int enqueue_layer0_pre(const StepIn& in, int rows, float* z, int ld_z);
  bool f32_attrs = false;                  // the fp32-store GEMM's shared-memory opt-in is done
  // Backward pass, one GEMM per call; the trainer's step schedule (enqueue_step_backward, capi.cu) puts them on streams.
  // dW_l[r0, r1) rows of W_l (r1 < 0: all) += A_{l-1}^T dZ_l on `st`, its grid capped at `sms` (tensor-core modes; `pdl`:
  // launched with programmatic dependent launch); layer 0 of a sparse step also scatter-adds the embedding rows' gradient.
  int enqueue_dw(const StepIn& in, int l, int rows, float* grad, cudaStream_t st, bool pdl, int sms, int r0 = 0, int r1 = -1,
                 int chunk = -1);
  // dZ_{l-1} = (dZ_l W_l^T) .* act'(A_{l-1}) and the bias gradient of layer l-1, on the main stream
  int enqueue_da(int l, int rows, float* grad);

  // Deterministic training (sb_trainer_set_deterministic, DESIGN §6b).  Every launch that sums over CTAs runs its DET
  // instantiation: partials into the launch site's own slots, the last CTA adds them in slot order.  dW GEMMs keep their
  // red.global epilogue with split-K capped at 2 (two addends onto a zeroed element: 0 + a + b == 0 + b + a).
  bool det = false;
  float* det_out_ws = nullptr;            // output layer (fused or not): [CTA][2 + 4 h_L]
  std::vector<float*> det_col_ws;         // det_col_ws[l], dA_l (l >= 1): column-sum slots [64-row tile][in_l]
  unsigned int* det_tickets = nullptr;    // [L]: 0 = output layer, l = dA_l
  int enable_det();                       // allocates the workspaces for max_batch rows (once)
  int dw_max_split() const { return det ? 2 : 0; }
};

// The only writer of a step descriptor: batch `b` (nullptr: an update without a batch), the update's scalars and the
// step's slot in the loss history, into slot `in` on stream `st`
int write_desc(cudaStream_t st, const StepIn& in, const Batch* b, float lr_t, float gscale, unsigned int epoch, float2* hist);
// set_batch_kernel is static (one copy per translation unit): these reach the copy write_desc launches.  The trainer keeps
// it in the step's shared-memory carve-out (see Net::init) and loads it before an exchange (preload_exchange_kernels).
void write_desc_max_shared();
int write_desc_preload();
// a batch of fp32 rows on the device (the staging area, or the fp32 resident set); w == nullptr weighs every row 1
Batch host_batch(const Net& n, const float* X, const float* y, const float* w, int rows, Feed feed = Feed::HOST);

int validate_desc(const sb_net_desc* d);
// makes `device` current if it is an sm_90 device (SB_ERR_CUDA when there is none)
int check_device(int device, int* num_sms);
// the device a pointer lives on, or -1 for host memory (pageable, pinned or managed) and for nullptr
int ptr_device(const void* p);
// a wide+deep index matrix of n entries: each a one-hot column in [0, n_onehot) or -1 (missing); anything else is
// SB_ERR_INVALID (a negative index other than -1 is not "missing", and a numpy caller would read it as a row from the end)
int check_sparse_idx(const int32_t* idx, long long n, int n_onehot);

}  // namespace sb
