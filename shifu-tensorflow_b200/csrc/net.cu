// Net: device state + kernel sequencing for the tabular-DNN forward / backward.
// Mirrors generate_from_modelconf + model (res/ssgd_monitor.py:91-144) as a list of fused launches.
// Also the kernel-level test hooks (sb_debug_gemm_*, sb_debug_out_layer, sb_debug_embed), so that every GEMM kernel is
// compiled in this one translation unit.
#include <stdarg.h>
#include <stdlib.h>
#include <string.h>
#include <algorithm>
#include <limits>
#include "net.cuh"
#include "gemm_dw.cuh"
#include "gemm_fwd_out.cuh"
#include "gemm_pp.cuh"
#include "gemm_wide.cuh"

namespace sb {

std::string& last_error_ref() {
  thread_local std::string e;
  return e;
}
int set_error(int code, const char* fmt, ...) {
  char buf[1024];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof(buf), fmt, ap);
  va_end(ap);
  last_error_ref() = buf;
  return code;
}

PFN_encodeTiled get_encode_tiled() {
  static PFN_encodeTiled fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<PFN_encodeTiled>(p);
  }
  return fn;
}

int make_tmaps_bf16(CUtensorMap* out3, const void* base, long long part_stride, int np, int rows, int cols, int ld, int box_rows) {
  for (int k = 0; k < (np > 1 ? np : 1); ++k)
    SB_TRY(make_tmap_bf16(out3 + k, static_cast<const __nv_bfloat16*>(base) + k * part_stride, rows, cols, ld, box_rows));
  return SB_OK;
}

void set_part_pairs(GemmTcParams* p, int np) {
  p->np = np > 1 ? np : 1;
  int n = 0;
  // smallest products first: they are added to a still small accumulator
  for (int sum = p->np - 1; sum >= 0; --sum)
    for (int i = 0; i <= sum; ++i) { p->pair_a[n] = static_cast<unsigned char>(i); p->pair_b[n] = static_cast<unsigned char>(sum - i); ++n; }
  p->n_pairs = n;
}

int make_tmap_bf16(CUtensorMap* out, const void* base, int rows, int cols, int ld, int box_rows) {
  PFN_encodeTiled enc = get_encode_tiled();
  SB_CHECK(enc != nullptr, SB_ERR_CUDA, "cuTensorMapEncodeTiled not available from the driver");
  SB_CHECK(rows > 0 && cols > 0 && (ld % 8) == 0 && (reinterpret_cast<uintptr_t>(base) & 15) == 0, SB_ERR_INVALID,
           "tensor map: bad geometry rows=%d cols=%d ld=%d", rows, cols, ld);
  cuuint64_t gdim[2] = {static_cast<cuuint64_t>(cols), static_cast<cuuint64_t>(rows)};
  cuuint64_t gstr[1] = {static_cast<cuuint64_t>(ld) * 2};
  cuuint32_t box[2] = {64u, static_cast<cuuint32_t>(box_rows)};
  cuuint32_t estr[2] = {1u, 1u};
  CUresult r = enc(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(base), gdim, gstr, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  SB_CHECK(r == CUDA_SUCCESS, SB_ERR_CUDA, "cuTensorMapEncodeTiled failed (%d) rows=%d cols=%d ld=%d box_rows=%d",
           static_cast<int>(r), rows, cols, ld, box_rows);
  return SB_OK;
}

// Tile configuration (persistent grid, one CTA per SM, 128 x BN tiles):
//   - BN = 128 (64 for a layer at most 64 wide).  The plain-bf16 forward and dA GEMMs are planned apart (plan_gemm_pp,
//     gemm_pp.cuh): two warpgroups per CTA with whole tiles each, 128 or 64 rows.  The fused output layer
//     (gemm_fwd_out.cuh) is planned apart: it needs whole rows of A_L in one CTA, so it takes 64 x h_L tiles (h_L <= 256,
//     the two consumer warpgroups split the columns: 64 accumulator registers per thread) and ceil(rows / 64) CTAs -
//     twice the CTAs a 128-row tile would give the narrow last layer;
//   - split-K (dW GEMMs, reduction over the batch; allow_split): fill the machine but keep >= 8 k-blocks per split;
//   - dW GEMMs take 128 x 256 tiles (gemm_dw.cuh) where that costs nothing in parallelism: the same grid as the 128-wide
//     plan, no more k-blocks x tile width per CTA, and >= 32 k-blocks per split.  The wider tile reads fewer shared-memory
//     operand bytes per flop, but needs twice the split-K factor for the same grid - twice the red.global traffic into
//     the gradient - and a split of few k-blocks is mostly the ring's fill and drain.
GemmPlan plan_gemm(int M, int N, int K, int num_sms, bool allow_split, int max_split) {
  const int total_kb = (K + 63) / 64;
  auto tiles_of = [&](int bn) { return ((M + 127) / 128) * ((N + bn - 1) / bn); };
  auto plan = [&](int bn) {
    const int tiles = tiles_of(bn);
    int split = 1;
    if (allow_split) {
      split = num_sms / tiles;
      const int cap = total_kb / 8;
      if (split > cap) split = cap;
      if (max_split > 0 && split > max_split) split = max_split;
      if (split < 1) split = 1;
    }
    if (split > total_kb) split = total_kb;
    GemmPlan pl = {};
    pl.bn = bn;
    pl.kb_per_split = (total_kb + split - 1) / split;
    pl.split_k = (total_kb + pl.kb_per_split - 1) / pl.kb_per_split;
    const int work = tiles * pl.split_k;
    pl.grid = work < num_sms ? work : num_sms;
    return pl;
  };
  // k-blocks x tile width one CTA works through (whole waves of work items)
  auto cost = [&](const GemmPlan& pl) {
    const long long work = static_cast<long long>(tiles_of(pl.bn)) * pl.split_k;
    return (work + pl.grid - 1) / pl.grid * pl.kb_per_split * pl.bn;
  };
  const GemmPlan pl = plan(N <= 64 ? 64 : 128);
  if (allow_split && N > 128) {
    const GemmPlan wide = plan(256);
    if (wide.grid == pl.grid && cost(wide) <= cost(pl) && wide.kb_per_split >= 32) return wide;
  }
  return pl;
}

int validate_desc(const sb_net_desc* d) {
  SB_CHECK(d != nullptr, SB_ERR_INVALID, "net desc is null");
  SB_CHECK(d->n_features > 0, SB_ERR_INVALID, "n_features must be > 0 (got %d)", d->n_features);
  SB_CHECK(d->n_hidden >= 1 && d->n_hidden <= SB_MAX_HIDDEN, SB_ERR_INVALID, "n_hidden must be in [1,%d] (got %d)",
           SB_MAX_HIDDEN, d->n_hidden);
  for (int l = 0; l < d->n_hidden; ++l) {
    SB_CHECK(d->hidden[l] > 0, SB_ERR_INVALID, "hidden[%d] must be > 0", l);
    SB_CHECK(d->acts[l] >= SB_ACT_NONE && d->acts[l] <= SB_ACT_LEAKYRELU, SB_ERR_INVALID, "acts[%d] invalid", l);
  }
  SB_CHECK(d->max_batch > 0, SB_ERR_INVALID, "max_batch must be > 0");
  SB_CHECK(d->precision >= SB_PREC_FP32 && d->precision <= SB_PREC_BF16X2, SB_ERR_INVALID, "precision invalid");
  SB_CHECK(d->loss == SB_LOSS_MSE || d->loss == SB_LOSS_SIGMOID_CE, SB_ERR_INVALID, "loss invalid");
  SB_CHECK((d->optimizer >= SB_OPT_ADADELTA && d->optimizer <= SB_OPT_FTRL) || d->optimizer == SB_OPT_RPROP, SB_ERR_INVALID,
           "optimizer invalid");
  if (d->optimizer == SB_OPT_RMSPROP) {   // (only the optimizer that reads them: other descriptors may leave them at 0)
    SB_CHECK(d->rho >= 0.f && d->rho <= 1.f, SB_ERR_INVALID, "RMSProp decay (rho) must be in [0, 1] (got %g)", d->rho);
    SB_CHECK(d->momentum >= 0.f, SB_ERR_INVALID, "RMSProp momentum must be >= 0 (got %g)", d->momentum);
    SB_CHECK(d->epsilon >= 0.f, SB_ERR_INVALID, "RMSProp epsilon must be >= 0 (got %g)", d->epsilon);
  }
  return SB_OK;
}

int check_device(int device, int* num_sms) {
  int n = 0;
  cudaError_t e = cudaGetDeviceCount(&n);
  SB_CHECK(e == cudaSuccess && n > 0, SB_ERR_CUDA, "no CUDA device available (%s); this library has no CPU fallback",
           cudaGetErrorString(e));
  SB_CHECK(device >= 0 && device < n, SB_ERR_INVALID, "device %d out of range [0,%d)", device, n);
  cudaDeviceProp prop;
  SB_CUDA(cudaGetDeviceProperties(&prop, device));
  SB_CHECK(prop.major == 9 && prop.minor == 0, SB_ERR_CUDA, "device %d is sm_%d%d; this library is built for sm_90a only",
           device, prop.major, prop.minor);
  *num_sms = prop.multiProcessorCount;
  SB_CUDA(cudaSetDevice(device));
  return SB_OK;
}

int ptr_device(const void* p) {
  if (!p) return -1;
  cudaPointerAttributes at;
  if (cudaPointerGetAttributes(&at, p) != cudaSuccess) { cudaGetLastError(); return -1; }
  return at.type == cudaMemoryTypeDevice ? at.device : -1;
}

int Net::init(const sb_net_desc* d, int device_, bool training_) {
  SB_TRY(validate_desc(d));
  SB_TRY(check_device(device_, &num_sms));
  device = device_;
  training = training_;
  const bool want_trace = getenv("SB_STEP_TRACE") != nullptr;
  // the main chain is the critical path: its CTAs are scheduled ahead of the trainer's side stream's (dW GEMMs, second
  // optimizer)
  if (input_from) {
    SB_CHECK(input_from->F == d->n_features && input_from->max_batch == d->max_batch && input_from->device == device_,
             SB_ERR_INVALID, "a net that borrows input staging needs the lender's features, max_batch and device");
    stream = input_from->stream;
  } else {
    int prio_least = 0, prio_greatest = 0;
    SB_CUDA(cudaDeviceGetStreamPriorityRange(&prio_least, &prio_greatest));
    SB_CUDA(cudaStreamCreateWithPriority(&stream, cudaStreamNonBlocking, prio_greatest));
  }
  F = d->n_features;
  L = d->n_hidden;
  precision = d->precision;
  nparts = precision == SB_PREC_FP32_TC ? 3 : (precision == SB_PREC_BF16X2 ? 2 : 1);
  loss = d->loss;
  max_batch = d->max_batch;
  ldB = round_up(max_batch, 8);
  ldF = round_up(F, 8);
  layers.resize(L + 1);
  long long off = 0;
  int prev = F;
  for (int l = 0; l <= L; ++l) {
    Layer& ly = layers[l];
    ly.in = prev;
    ly.out = (l < L) ? d->hidden[l] : 1;
    ly.act = (l < L) ? d->acts[l] : SB_ACT_SIGMOID;
    ly.w_off = off; off += static_cast<long long>(ly.in) * ly.out;
    ly.b_off = off; off += ly.out;
    ly.ld_in = round_up(ly.in, 8);
    ly.ld_out = round_up(ly.out, 8);
    prev = ly.out;
  }
  n_params = off;
  const bool bf = tc();
  {
    auto align256 = [](size_t b) { return (b + 255) & ~static_cast<size_t>(255); };
    const size_t vec_bytes = align256(static_cast<size_t>(n_params) * sizeof(float) + 64);
    size_t at = vec_bytes;                       // theta at 0
    if (training) { s1_off = at; at += vec_bytes; s2_off = at; at += vec_bytes; }
    shadow_off = at;
    std::vector<size_t> wn_off(L, 0);
    Wn_ps.assign(L, 0);
    if (bf)
      for (int l = 0; l < L; ++l) {
        const size_t part = align256(static_cast<size_t>(layers[l].in) * layers[l].ld_out * sizeof(__nv_bfloat16));
        wn_off[l] = at; at += part * nparts;
        Wn_ps[l] = static_cast<long long>(part / sizeof(__nv_bfloat16));
      }
    extra_off = at;
    at += align256(arena_extra_bytes);
    arena_bytes = at;
    void* q = nullptr;
    SB_CUDA(cudaMalloc(&q, arena_bytes));
    allocs.push_back(q);
    SB_CUDA(cudaMemsetAsync(q, 0, arena_bytes, stream));
    arena = static_cast<char*>(q);
    theta = reinterpret_cast<float*>(arena);
    if (training) { s1 = reinterpret_cast<float*>(arena + s1_off); s2 = reinterpret_cast<float*>(arena + s2_off); }
    if (bf)
      for (int l = 0; l < L; ++l) layers[l].Wn = reinterpret_cast<__nv_bfloat16*>(arena + wn_off[l]);
  }
  SB_TRY(dalloc(&scal, SCAL_COUNT));
  SB_TRY(dalloc(&desc, 1));
  if (want_trace) SB_TRY(dalloc(&step_trace, 32 * 16));
  SB_TRY(dalloc(&yhat, max_batch));
  SB_TRY(dalloc(&ones, max_batch));
  if (input_from) stX = input_from->stX;
  else SB_TRY(dalloc(&stX, static_cast<size_t>(max_batch) * F));
  SB_TRY(dalloc(&stY, max_batch));
  SB_TRY(dalloc(&stW, max_batch));
  fill_kernel<<<(max_batch + 255) / 256, 256, 0, stream>>>(ones, 1.f, max_batch);

  if (bf) {
    Xb_ps = static_cast<long long>(max_batch) * ldF;
    if (input_from) Xb = input_from->Xb;
    else SB_TRY(dalloc(&Xb, static_cast<size_t>(Xb_ps) * nparts));
    A.assign(L, nullptr); dZ.assign(L, nullptr); A_ps.assign(L, 0);
    for (int l = 0; l < L; ++l) {
      Layer& ly = layers[l];
      A_ps[l] = static_cast<long long>(max_batch) * ly.ld_out;
      SB_TRY(dalloc(&A[l], static_cast<size_t>(A_ps[l]) * nparts));
      if (training) SB_TRY(dalloc(&dZ[l], static_cast<size_t>(A_ps[l]) * nparts));
    }
  } else {
    if (input_from) Xf = input_from->Xf;
    else SB_TRY(dalloc(&Xf, static_cast<size_t>(max_batch) * F));
    Af.assign(L, nullptr); dZf.assign(L, nullptr);
    for (int l = 0; l < L; ++l) {
      SB_TRY(dalloc(&Af[l], static_cast<size_t>(max_batch) * layers[l].out));
      if (training) SB_TRY(dalloc(&dZf[l], static_cast<size_t>(max_batch) * layers[l].out));
    }
  }

  // optimizer / shadow-refresh work table: runs of <= 1024 consecutive parameters
  const std::vector<char> all(static_cast<size_t>(L + 1), 1);
  std::vector<OptWork> wk;
  SB_TRY(build_work(all, all, &wk, &work_begin, &work_end));
  n_work = static_cast<int>(wk.size());
  SB_TRY(dalloc(&work, wk.size()));
  SB_CUDA(cudaMemcpyAsync(work, wk.data(), wk.size() * sizeof(OptWork), cudaMemcpyHostToDevice, stream));
  SB_CUDA(cudaStreamSynchronize(stream));
  work_all = work; n_work_all = n_work;

  // opt in to > 48 KB dynamic shared memory once, outside of any stream capture
  if (bf) {
    SB_TRY((set_gemm_tc_attrs<EPI_FWD, false, true>()));
    SB_TRY(set_gemm_fwd_out_attrs());
    SB_TRY(set_gemm_pp_attrs());
    SB_TRY(set_gemm_wide_attrs());
    SB_TRY((set_gemm_tc_attrs<EPI_DA, false, false>()));
    SB_TRY((set_gemm_tc_attrs<EPI_DW, true, true>()));
    SB_TRY(set_gemm_dw_attrs());
    // keep the SMs in the GEMMs' shared-memory carve-out for every kernel of the step, so that no launch in the chain
    // has to re-partition L1 / shared memory
    const int co = cudaSharedmemCarveoutMaxShared;
    cudaFuncSetAttribute(load_batch_kernel<true>, cudaFuncAttributePreferredSharedMemoryCarveout, co);
    cudaFuncSetAttribute(gather_batch_kernel<true>, cudaFuncAttributePreferredSharedMemoryCarveout, co);
    cudaFuncSetAttribute(out_layer_kernel<__nv_bfloat16>, cudaFuncAttributePreferredSharedMemoryCarveout, co);
    cudaFuncSetAttribute(out_layer_kernel<__nv_bfloat16, true>, cudaFuncAttributePreferredSharedMemoryCarveout, co);
  }
  return SB_OK;
}

Net::~Net() {
  if (!stream && allocs.empty()) return;    // init never got to the device
  cudaSetDevice(device);
  if (stream) cudaStreamSynchronize(stream);
  for (void* p : allocs) cudaFree(p);
  if (stream && !input_from) cudaStreamDestroy(stream);
}

int check_sparse_idx(const int32_t* idx, long long n, int n_onehot) {
  for (long long i = 0; i < n; ++i)
    SB_CHECK(idx[i] >= -1 && idx[i] < n_onehot, SB_ERR_INVALID, "idx[%lld] = %d outside [-1, n_onehot=%d)", i, idx[i], n_onehot);
  return SB_OK;
}

int Net::set_sparse(int n_dense_, int n_onehot_, int n_cat_) {
  SB_CHECK(n_dense_ >= 1 && n_onehot_ >= 1 && n_cat_ >= 1, SB_ERR_INVALID, "wide+deep needs >= 1 dense, one-hot and categorical column");
  SB_CHECK(n_dense_ + n_onehot_ == F, SB_ERR_INVALID, "n_dense (%d) + n_onehot (%d) must equal n_features (%d): the sparse path evaluates "
           "the SAME first layer", n_dense_, n_onehot_, F);
  SB_CUDA(cudaSetDevice(device));
  n_dense = n_dense_; n_onehot = n_onehot_; n_cat = n_cat_;
  ldD = round_up(n_dense, 8);
  if (!idx) SB_TRY(dalloc(&idx, static_cast<size_t>(max_batch) * n_cat));
  if (!E) SB_TRY(dalloc(&E, static_cast<size_t>(max_batch) * layers[0].ld_out));
  SB_CUDA(cudaStreamSynchronize(stream));
  return SB_OK;
}

// Slot workspaces of the deterministic epilogues, one per launch site, sized for max_batch rows: the output layer has at
// most max(2 SMs + 2, max_batch / 32) CTAs (fused: one per SM; out_layer_rows_kernel: ~2 per SM; out_layer_kernel: 32
// rows each) of 2 + 4 h_L slots; dA_l has one slot row per 64-row tile (the smallest dA tile) and column of in_l.
// Reuse: a site's slots and ticket are written and read only by that site's launch, and all of a site's launches go to
// the net's main stream, where two of them are always separated by complete kernels:
//   - PDL: griddepcontrol.launch_dependents lets the next kernel START early, but every kernel of the chain executes
//     griddepcontrol.wait before its first global access, and that returns only once the preceding grid has completed
//     and flushed its memory - the last CTA's ordered sum included.  So the next launch of the same site cannot store
//     into the slots while the last CTA still reads them.
//   - The dW side stream runs beside the dA chain, but the dW GEMMs use no workspace (red.global with split-K <= 2).
//   - set_batch_kernel on the prep stream writes the next step's descriptor and scalars, never a slot or a ticket.
//   - eval_loss / loss_resident use the output layer's site on the same main stream, behind or ahead of whole steps.
// The ticket is put back to 0 by the last CTA of each launch, so a graph replay starts from 0 without a memset node.
int Net::enable_det() {
  if (det_tickets) { det = true; return SB_OK; }
  SB_CUDA(cudaSetDevice(device));
  const Layer& hl = layers[L - 1];
  const long long ctas = std::max<long long>(2LL * num_sms + 2, (max_batch + 31) / 32);
  SB_TRY(dalloc(&det_out_ws, static_cast<size_t>(ctas) * (2 + 4 * static_cast<size_t>(hl.out))));
  det_col_ws.assign(L, nullptr);
  for (int l = 1; l < L; ++l)
    SB_TRY(dalloc(&det_col_ws[l], static_cast<size_t>((max_batch + 63) / 64) * layers[l - 1].out));
  SB_TRY(dalloc(&det_tickets, static_cast<size_t>(L)));
  SB_CUDA(cudaStreamSynchronize(stream));
  det = true;
  return SB_OK;
}

int Net::enqueue_embed(int rows, bool scatter, float* grad, cudaStream_t st) {
  const Layer& l0 = layers[0];
  EmbedParams p = {};
  p.rows = rows; p.n_cat = n_cat; p.H = l0.out;
  p.idx = idx;
  p.np = nparts; p.ldW = tc() ? l0.ld_out : l0.out;
  if (tc()) { p.We = l0.Wn + static_cast<size_t>(n_dense) * l0.ld_out; p.We_ps = Wn_ps[0]; }
  else p.We32 = theta + l0.w_off + static_cast<long long>(n_dense) * l0.out;
  p.E = E; p.ldE = l0.ld_out;
  if (scatter) {
    if (tc()) { p.dZ = dZ[0]; p.dZ_ps = A_ps[0]; p.ld_dZ = l0.ld_out; }
    else { p.dZ32 = dZf[0]; p.ld_dZ = l0.out; }
    p.gWe = grad + l0.w_off + static_cast<long long>(n_dense) * l0.out;
    SB_TRY(launch_kernel(embed_scatter_kernel, dim3((rows + 7) / 8), dim3(256), 0, st, false, p));
    mark("embed_scatter");
  } else {
    SB_TRY(launch_kernel(embed_gather_kernel, dim3((rows + 7) / 8), dim3(256), 0, st, false, p));
    mark("embed_gather");
  }
  return SB_OK;
}

// The runs of every parameter that trains (w_trains[l] / b_trains[l]: W_l / b_l of layer l = 0..L), layer by layer; the
// range of layer l goes to [(*begin)[l], (*end)[l]).  A tensor-core net keeps W_l (shadow-backed) and b_l in separate
// runs; fp32 mode puts W_l and b_l, which lie next to each other, into one stretch of runs when both train.
int Net::build_work(const std::vector<char>& w_trains, const std::vector<char>& b_trains, std::vector<OptWork>* out,
                    std::vector<int>* begin, std::vector<int>* end) const {
  std::vector<OptWork>& wk = *out;
  wk.clear();
  auto add_runs = [&](long long o, long long n, const Layer* mat) {
    for (long long s = 0; s < n; s += 1024) {
      OptWork w = {};
      w.off = o + s; w.count = static_cast<int>(n - s < 1024 ? n - s : 1024);
      w.np = 1;
      if (mat) {
        w.out_dim = mat->out; w.mat_off = mat->w_off; w.Wn = mat->Wn; w.ld_out = mat->ld_out;
        w.np = nparts; w.part_stride = Wn_ps[static_cast<size_t>(mat - layers.data())];
      }
      wk.push_back(w);
    }
  };
  begin->assign(L + 1, 0); end->assign(L + 1, 0);
  for (int l = 0; l <= L; ++l) {
    const Layer& ly = layers[l];
    const long long nw = static_cast<long long>(ly.in) * ly.out;
    // the 16-byte path (SB_RUN_IS_VEC) stores 4 shadow elements at once: they are 8-byte aligned only when ld_out % 4 == 0
    SB_CHECK(!tc() || l == L || ly.ld_out % 4 == 0, SB_ERR_STATE, "layer %d: shadow row pitch %d is not a multiple of 4", l, ly.ld_out);
    (*begin)[l] = static_cast<int>(wk.size());
    if (tc() && l < L) {
      if (w_trains[l]) add_runs(ly.w_off, nw, &ly);
      if (b_trains[l]) add_runs(ly.b_off, ly.out, nullptr);
    } else if (w_trains[l] && b_trains[l]) {
      add_runs(ly.w_off, nw + ly.out, nullptr);
    } else {
      if (w_trains[l]) add_runs(ly.w_off, nw, nullptr);
      if (b_trains[l]) add_runs(ly.b_off, ly.out, nullptr);
    }
    (*end)[l] = static_cast<int>(wk.size());
  }
  return SB_OK;
}

int Net::set_trainable(const std::vector<char>& w_trains, const std::vector<char>& b_trains) {
  SB_CUDA(cudaSetDevice(device));
  std::vector<OptWork> wk;
  SB_TRY(build_work(w_trains, b_trains, &wk, &work_begin, &work_end));
  n_work = static_cast<int>(wk.size());
  const bool every = std::all_of(w_trains.begin(), w_trains.end(), [](char c) { return c != 0; }) &&
                     std::all_of(b_trains.begin(), b_trains.end(), [](char c) { return c != 0; });
  if (every) {                       // everything trains: the table init() built
    work = work_all;
    return SB_OK;
  }
  if (!work_part) SB_TRY(dalloc(&work_part, static_cast<size_t>(n_work_all)));
  work = work_part;
  if (n_work > 0) SB_CUDA(cudaMemcpyAsync(work, wk.data(), wk.size() * sizeof(OptWork), cudaMemcpyHostToDevice, stream));
  SB_CUDA(cudaStreamSynchronize(stream));
  return SB_OK;
}

int Net::refresh_shadows() {
  if (!tc()) return SB_OK;
  shadow_refresh_kernel<<<n_work_all, 256, 0, stream>>>(work_all, theta);
  SB_CUDA(cudaGetLastError());
  return SB_OK;
}

int write_desc(cudaStream_t st, const StepIn& in, const Batch* b, float lr_t, float gscale, unsigned int epoch, float2* hist) {
  static const Batch none{};
  const Batch& x = b ? *b : none;
  return launch_kernel(set_batch_kernel, dim3(1), dim3(1), 0, st, false, in.desc, x.X, x.y, x.w, lr_t, gscale, epoch, x.row0,
                       x.nz_prefix, x.rows, in.scal, hist, x.order);
}

void write_desc_max_shared() {
  cudaFuncSetAttribute(set_batch_kernel, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
}

int write_desc_preload() {
  cudaFuncAttributes a;
  SB_CUDA(cudaFuncGetAttributes(&a, set_batch_kernel));
  return SB_OK;
}

Batch host_batch(const Net& n, const float* X, const float* y, const float* w, int rows, Feed feed) {
  Batch b;
  b.feed = feed;
  b.X = X; b.y = y; b.w = w ? w : n.ones;
  b.rows = rows;
  return b;
}

int Net::enqueue_load(const StepIn& in, int rows, float* clear, long long clear_n) {
  const int Fx = in.feed == Feed::SPARSE ? n_dense : F;        // a sparse step stages only the dense block
  const int ldx = in.feed == Feed::SPARSE ? ldD : ldF;
  const long long units = static_cast<long long>(rows) * (ldx / 8);
  long long blocks = (units + 255) / 256;
  const long long cap = static_cast<long long>(num_sms) * 16;
  if (blocks > cap) blocks = cap;
  if (blocks < 1) blocks = 1;
  // first kernel of the step: its stream predecessor is set_batch_kernel (a kernel), so PDL applies here too
  if (tc())
    SB_TRY(launch_kernel(load_batch_kernel<true>, dim3(static_cast<unsigned>(blocks)), dim3(256), 0, stream, true,
                         static_cast<const BatchDesc*>(in.desc), rows, Fx, Xb, ldx, static_cast<float*>(nullptr), in.scal, clear,
                         clear_n, nparts, Xb_ps));
  else
    SB_TRY(launch_kernel(load_batch_kernel<false>, dim3(static_cast<unsigned>(blocks)), dim3(256), 0, stream, true,
                         static_cast<const BatchDesc*>(in.desc), rows, Fx, static_cast<__nv_bfloat16*>(nullptr), ldx, Xf, in.scal,
                         clear, clear_n, 1, 0ll));
  mark(tc() ? "load_batch<bf16>" : "load_batch<fp32>");
  if (in.feed == Feed::SPARSE) SB_TRY(enqueue_embed(rows, false, nullptr, stream));
  return SB_OK;
}

int Net::enqueue_hidden_forward(const StepIn& in, int rows, float* grad, bool* fused_out, float4* clear, long long clear_n4,
                                int first) {
  if (fused_out) *fused_out = false;
  for (int l = first; l < L; ++l) {
    Layer& ly = layers[l];
    const bool sp0 = (l == 0) && in.feed == Feed::SPARSE;       // wide+deep: contract the dense columns only, add the embedding sums
    const int k_in = sp0 ? n_dense : ly.in;
    const int ld_k = sp0 ? ldD : ly.ld_in;
    if (tc()) {
      // Z = A_{l-1}[rows,in] (K-major) x W_l[in,out] (MN-major B operand: n contiguous)
      TmapSet tm;
      const Operand0 a = (l == 0) ? layer0(in, rows) : Operand0{A[l - 1], A_ps[l - 1], rows};
      SB_TRY(make_tmaps_bf16(tm.b, ly.Wn, Wn_ps[l], nparts, k_in, ly.out, ly.ld_out, 64));
      GemmTcParams p = {};
      set_part_pairs(&p, nparts);
      p.M = rows; p.N = ly.out; p.K = k_in;
      if (sp0) { p.addend = E; p.ld_add = ly.ld_out; }
      p.bias = theta + ly.b_off; p.act = ly.act;
      p.out = A[l]; p.ld_out = ly.ld_out; p.out_ps = A_ps[l];
      p.a_rows = a.at_row0 ? in.desc : nullptr;
      if (l == L - 1 && grad != nullptr && training && ly.out <= FWD_OUT_MAX_N && p.addend == nullptr) {
        // K2 + K3 + K4 + output backward in one kernel (gemm_fwd_out.cuh): 64-row tiles of whole rows of A_L
        FwdOutTmaps ft;
        SB_TRY(make_tmaps_bf16(ft.a, a.p, a.ps, nparts, a.rows, k_in, ld_k, 64));
        for (int i = 0; i < 3; ++i) ft.b[i] = tm.b[i];
        SB_TRY(make_tmaps_bf16(ft.o, dZ[l], A_ps[l], nparts, rows, ly.out, ly.ld_out, 64));
        const int tiles = (rows + 63) / 64;
        const int grid = tiles < num_sms ? tiles : num_sms;
        Layer& ol = layers[L];
        p.wo = theta + ol.w_off; p.bo = theta + ol.b_off;
        p.desc = in.desc; p.scal = in.scal; p.loss = loss;
        p.g_wo = grad + ol.w_off; p.g_bo = grad + ol.b_off; p.g_bL = grad + ly.b_off;
        if (det) { p.det_ws = det_out_ws; p.det_ticket = det_tickets; }
        p.trace = next_trace("fwd_out", l, rows, ly.out, k_in);
        SB_TRY(launch_gemm_fwd_out(grid, ft, p, stream, true));
        if (fused_out) *fused_out = true;
        mark("gemm_fwd_out");
        continue;
      }
      if (l == 0) { p.zero_buf = clear; p.zero_n4 = clear_n4; }
      p.trace = next_trace("fwd", l, rows, ly.out, k_in);
      if (nparts == 1 && p.addend == nullptr) {    // plain bf16: the ping-pong kernel
        const PpPlan pp = plan_gemm_pp(rows, ly.out, k_in, num_sms, true);
        PpTmaps pt;
        SB_TRY(make_tmap_bf16(&pt.a, a.p, a.rows, k_in, ld_k, pp.bm_wg));
        pt.b = tm.b[0];
        SB_TRY(make_tmap_bf16(&pt.o, A[l], rows, ly.out, ly.ld_out, pp.bm_wg));
        if (pp.bn == 256) {
          SB_TRY(launch_gemm_wide(pp, pt, p, stream, true));
          mark("gemm_wide");
        } else {
          SB_TRY(launch_gemm_pp<EPI_FWD>(pp, pt, p, stream, true));
          mark("gemm_pp<FWD>");
        }
      } else {
        const GemmPlan pl = plan_gemm(rows, ly.out, round_up(k_in, 64) * pairs_of(nparts), num_sms, false);
        SB_TRY(make_tmaps_bf16(tm.a, a.p, a.ps, nparts, a.rows, k_in, ld_k, 128));
        SB_TRY((launch_gemm_tc<EPI_FWD, false, true>(pl, tm, p, stream, true)));
        mark(pl.bn == 64 ? "gemm_tc<64,FWD,GENERIC>" : "gemm_tc<128,FWD,GENERIC>");
      }
    } else {
      GemmF32Params p = {};
      p.M = rows; p.N = ly.out; p.K = k_in;
      p.A = (l == 0) ? Xf : Af[l - 1]; p.sAm = k_in; p.sAk = 1;
      if (sp0) { p.addend = E; p.ld_add = ly.ld_out; }
      p.B = theta + ly.w_off; p.sBk = ly.out; p.sBn = 1;
      p.bias = theta + ly.b_off; p.act = ly.act;
      p.out = Af[l]; p.ld_out = ly.out;
      SB_TRY(launch_gemm_f32<EPI_FWD>(p, 1, stream));
      mark("gemm_f32<FWD>");
    }
  }
  return SB_OK;
}

int Net::enqueue_out(const StepIn& in, int rows, bool do_loss, bool do_bwd, float* yhat_dst, float* grad) {
  Layer& hl = layers[L - 1];
  Layer& ol = layers[L];
  OutLayerParams p = {};
  p.rows = rows; p.H = hl.out;
  p.wo = theta + ol.w_off; p.bo = theta + ol.b_off;
  p.desc = in.desc; p.scal = in.scal; p.loss = loss; p.act = hl.act;
  p.do_bwd = do_bwd ? 1 : 0; p.do_loss = do_loss ? 1 : 0;
  p.yhat = yhat_dst;
  p.trace = next_trace("out_layer");
  if (do_bwd) {
    p.g_wo = grad + ol.w_off; p.g_bo = grad + ol.b_off; p.g_bL = grad + hl.b_off;
  }
  const bool d = det && (do_loss || do_bwd);   // the DET instantiations (slots + last-CTA sum) when anything is summed
  if (d) { p.det_ws = det_out_ws; p.det_ticket = det_tickets; }
  const int grid = (rows + 31) / 32;
  const char* kernel;
  if (tc()) {
    p.A = A[L - 1]; p.ldA = hl.ld_out;
    p.np = nparts; p.a_ps = A_ps[L - 1]; p.dz_ps = A_ps[L - 1];
    if (do_bwd) { p.dZ = dZ[L - 1]; p.ld_dZ = hl.ld_out; }
    if (hl.out <= 1024) {
      // one-pass kernel: rows per block sized for ~2 blocks per SM, at least one row per warp
      int rpb = (rows + 2 * num_sms - 1) / (2 * num_sms);
      rpb = ((rpb + 7) / 8) * 8;
      if (rpb < 8) rpb = 8;
      const dim3 g((rows + rpb - 1) / rpb);
      static const char* const names[2][3] = {{"out_layer_rows<1>", "out_layer_rows<2>", "out_layer_rows<4>"},
                                              {"out_layer_rows<1,DET>", "out_layer_rows<2,DET>", "out_layer_rows<4,DET>"}};
      const int nch = hl.out <= 256 ? 0 : (hl.out <= 512 ? 1 : 2);
      kernel = names[d ? 1 : 0][nch];
      if (d) {
        if (nch == 0) SB_TRY(launch_kernel(out_layer_rows_kernel<1, true>, g, dim3(256), 0, stream, true, p, rpb));
        else if (nch == 1) SB_TRY(launch_kernel(out_layer_rows_kernel<2, true>, g, dim3(256), 0, stream, true, p, rpb));
        else SB_TRY(launch_kernel(out_layer_rows_kernel<4, true>, g, dim3(256), 0, stream, true, p, rpb));
      } else if (nch == 0) SB_TRY(launch_kernel(out_layer_rows_kernel<1>, g, dim3(256), 0, stream, true, p, rpb));
      else if (nch == 1) SB_TRY(launch_kernel(out_layer_rows_kernel<2>, g, dim3(256), 0, stream, true, p, rpb));
      else SB_TRY(launch_kernel(out_layer_rows_kernel<4>, g, dim3(256), 0, stream, true, p, rpb));
    } else if (d) {
      SB_TRY(launch_kernel(out_layer_kernel<__nv_bfloat16, true>, dim3(grid), dim3(256), 0, stream, true, p));
      kernel = "out_layer<bf16,DET>";
    } else {
      SB_TRY(launch_kernel(out_layer_kernel<__nv_bfloat16>, dim3(grid), dim3(256), 0, stream, true, p));
      kernel = "out_layer<bf16>";
    }
  } else {
    p.A = Af[L - 1]; p.ldA = hl.out;
    if (do_bwd) { p.dZ = dZf[L - 1]; p.ld_dZ = hl.out; }
    if (d) SB_TRY(launch_kernel(out_layer_kernel<float, true>, dim3(grid), dim3(256), 0, stream, true, p));
    else SB_TRY(launch_kernel(out_layer_kernel<float>, dim3(grid), dim3(256), 0, stream, true, p));
    kernel = d ? "out_layer<float,DET>" : "out_layer<float>";
  }
  SB_CUDA(cudaGetLastError());
  mark(kernel);
  return SB_OK;
}

int Net::enqueue_layer0_pre(const StepIn& in, int rows, float* z, int ld_z) {
  const Layer& ly = layers[0];
  if (!tc()) {
    GemmF32Params p = {};
    p.M = rows; p.N = ly.out; p.K = ly.in;
    p.A = Xf; p.sAm = ly.in; p.sAk = 1;
    p.B = theta + ly.w_off; p.sBk = ly.out; p.sBn = 1;
    p.bias = theta + ly.b_off; p.act = SB_ACT_NONE;
    p.out = z; p.ld_out = ld_z;
    SB_TRY(launch_gemm_f32<EPI_FWD>(p, 1, stream));
    mark("gemm_f32<FWD>");
    return SB_OK;
  }
  if (!f32_attrs) {
    SB_TRY((set_gemm_tc_attrs<EPI_F32, false, true>()));
    f32_attrs = true;
  }
  const Operand0 a = layer0(in, rows);
  const GemmPlan pl = plan_gemm(rows, ly.out, round_up(ly.in, 64) * pairs_of(nparts), num_sms, false);
  TmapSet tm;
  SB_TRY(make_tmaps_bf16(tm.a, a.p, a.ps, nparts, a.rows, ly.in, ly.ld_in, 128));
  SB_TRY(make_tmaps_bf16(tm.b, ly.Wn, Wn_ps[0], nparts, ly.in, ly.out, ly.ld_out, 64));
  GemmTcParams p = {};
  set_part_pairs(&p, nparts);
  p.M = rows; p.N = ly.out; p.K = ly.in;
  p.accum = z; p.ld_acc = ld_z;
  SB_TRY((launch_gemm_tc<EPI_F32, false, true>(pl, tm, p, stream, true)));
  mark(pl.bn == 64 ? "gemm_tc<64,F32>" : "gemm_tc<128,F32>");
  return SB_OK;
}

int Net::enqueue_dw(const StepIn& in, int l, int rows, float* grad, cudaStream_t st, bool pdl, int sms, int r0, int r1, int chunk) {
  Layer& ly = layers[l];
  const bool sp0 = (l == 0) && in.feed == Feed::SPARSE;         // wide+deep: dW of the dense rows by GEMM, of the embedding rows by scatter-add
  const int in_rows = sp0 ? n_dense : ly.in;
  if (r1 < 0) r1 = in_rows;
  if (sp0) SB_TRY(enqueue_embed(rows, true, grad, st));
  if (!tc()) {
    GemmF32Params p = {};
    p.M = in_rows; p.N = ly.out; p.K = rows;
    p.A = (l == 0) ? Xf : Af[l - 1]; p.sAm = 1; p.sAk = in_rows;
    p.B = dZf[l]; p.sBk = ly.out; p.sBn = 1;
    p.accum = grad + ly.w_off; p.ld_acc = ly.out;
    const int tiles = ((p.M + 63) / 64) * ((p.N + 63) / 64);
    int split = (2 * num_sms) / (tiles > 0 ? tiles : 1);
    const int cap = (rows + 63) / 64;
    if (split > cap) split = cap;
    if (det && split > 2) split = 2;   // at most two atomic addends per element (see dw_max_split)
    SB_TRY(launch_gemm_f32<EPI_DW>(p, split, st));
    mark("gemm_f32<DW>");
    return SB_OK;
  }
  // dW_l[in,out] += sum_rows A_{l-1}[rows,in] (MN-major A) * dZ_l[rows,out] (MN-major B), split-K over rows
  const int ld_k = sp0 ? ldD : ly.ld_in;
  const Operand0 a = (l == 0) ? layer0(in, rows) : Operand0{A[l - 1], A_ps[l - 1], rows};
  const GemmPlan pl = plan_gemm(r1 - r0, ly.out, round_up(rows, 64) * pairs_of(nparts), sms, true, dw_max_split());
  TmapSet tm;
  // resident set: rows past the batch end are real rows of other batches; the B operand (dZ_l, extent = rows) is
  // zero-filled there, so they contribute nothing
  SB_TRY(make_tmaps_bf16(tm.a, a.p + r0, a.ps, nparts, a.rows, r1 - r0, ld_k, 64));
  SB_TRY(make_tmaps_bf16(tm.b, dZ[l], A_ps[l], nparts, rows, ly.out, ly.ld_out, 64));
  GemmTcParams p = {};
  set_part_pairs(&p, nparts);
  p.M = r1 - r0; p.N = ly.out; p.K = rows;
  p.a_rows = a.at_row0 ? in.desc : nullptr;
  p.accum = grad + ly.w_off + static_cast<long long>(r0) * ly.out; p.ld_acc = ly.out;
  p.acc_vec4 = (ly.out % 4 == 0 && ly.w_off % 4 == 0) ? 1 : 0;
  p.trace = next_trace("dW", l, r1 - r0, ly.out, rows, chunk);
  if (pl.bn == 256) {
    SB_TRY(launch_gemm_dw(pl, tm, p, st, pdl));
    mark("gemm_dw");
  } else {
    SB_TRY((launch_gemm_tc<EPI_DW, true, true>(pl, tm, p, st, pdl)));
    mark(pl.bn == 64 ? "gemm_tc<64,DW>" : "gemm_tc<128,DW>");
  }
  return SB_OK;
}

int Net::enqueue_da(int l, int rows, float* grad) {
  Layer& ly = layers[l];
  Layer& pl = layers[l - 1];
  if (!tc()) {
    GemmF32Params p = {};
    p.M = rows; p.N = ly.in; p.K = ly.out;
    p.A = dZf[l]; p.sAm = ly.out; p.sAk = 1;
    p.B = theta + ly.w_off; p.sBk = 1; p.sBn = ly.out;
    p.act = pl.act;
    p.aux = Af[l - 1]; p.ld_aux = pl.out;
    p.out = dZf[l - 1]; p.ld_out = pl.out;
    p.colsum = grad + pl.b_off;
    if (det) {
      p.det_ws = det_col_ws[l]; p.det_ticket = det_tickets + l;
      SB_TRY((launch_gemm_f32<EPI_DA, true>(p, 1, stream)));
    } else {
      SB_TRY(launch_gemm_f32<EPI_DA>(p, 1, stream));
    }
    mark("gemm_f32<DA>");
    return SB_OK;
  }
  // dZ_{l-1}[rows,in] = (dZ_l[rows,out] (K-major) x W_l[in,out] (K-major B: k = out contiguous)) .* act'(A_{l-1})
  GemmTcParams p = {};
  set_part_pairs(&p, nparts);
  p.M = rows; p.N = ly.in; p.K = ly.out;
  p.act = pl.act;
  p.aux = A[l - 1]; p.ld_aux = pl.ld_out; p.aux_ps = A_ps[l - 1];
  p.out = dZ[l - 1]; p.ld_out = pl.ld_out; p.out_ps = A_ps[l - 1];
  p.colsum = grad + pl.b_off;
  p.trace = next_trace("dA", l, rows, ly.in, ly.out);
  if (det) { p.det_ws = det_col_ws[l]; p.det_ticket = det_tickets + l; }
  if (nparts == 1) {                           // plain bf16: the ping-pong kernel
    const PpPlan pp = plan_gemm_pp(rows, ly.in, ly.out, num_sms, false);
    PpTmaps pt;
    SB_TRY(make_tmap_bf16(&pt.a, dZ[l], rows, ly.out, ly.ld_out, pp.bm_wg));
    SB_TRY(make_tmap_bf16(&pt.b, ly.Wn, ly.in, ly.out, ly.ld_out, pp.bn));
    SB_TRY(make_tmap_bf16(&pt.o, dZ[l - 1], rows, ly.in, pl.ld_out, pp.bm_wg));
    SB_TRY(make_tmap_bf16(&pt.x, A[l - 1], rows, ly.in, pl.ld_out, pp.bm_wg));
    SB_TRY(launch_gemm_pp<EPI_DA>(pp, pt, p, stream, true));
    mark("gemm_pp<DA>");
  } else {
    const GemmPlan gp = plan_gemm(rows, ly.in, round_up(ly.out, 64) * pairs_of(nparts), num_sms, false);
    TmapSet tm;
    SB_TRY(make_tmaps_bf16(tm.a, dZ[l], A_ps[l], nparts, rows, ly.out, ly.ld_out, 128));
    SB_TRY(make_tmaps_bf16(tm.b, ly.Wn, Wn_ps[l], nparts, ly.in, ly.out, ly.ld_out, gp.bn));
    SB_TRY((launch_gemm_tc<EPI_DA, false, false>(gp, tm, p, stream, true)));
    mark(gp.bn == 64 ? "gemm_tc<64,DA,GENERIC>" : "gemm_tc<128,DA,GENERIC>");
  }
  return SB_OK;
}

// ================================================================================================
// kernel-level test hooks: one GEMM of the step on fp32 host operands, through the launches above
// ================================================================================================
template <typename T>
static int alloc_filled(DevBuf<T>* b, size_t n, int byte = 0) {
  SB_TRY(b->alloc(n));
  SB_CUDA(cudaMemset(b->p, byte, sizeof(T) * n));
  return SB_OK;
}

// fp32 host [rows, cols] -> np bf16 parts (bf16_residual, the step's split) into a device buffer: rows of ld elements, parts
// ps elements apart; the pad columns are left as they are
static int upload_parts(__nv_bfloat16* dst, const float* src, int rows, int cols, int ld, int np, long long ps) {
  const long long n = static_cast<long long>(rows) * cols;
  DevBuf<float> f32;
  SB_TRY(f32.alloc(n));
  SB_CUDA(cudaMemcpy(f32.p, src, sizeof(float) * n, cudaMemcpyHostToDevice));
  cast_bf16_kernel<<<static_cast<unsigned>((n + 255) / 256), 256>>>(f32.p, rows, cols, dst, ld, np, ps);
  SB_CUDA(cudaGetLastError());
  return SB_OK;
}

// fp32 host [rows, cols] -> np bf16 parts on the device, each [rows, round_up(cols, 8)] with zero padding, one behind the other
static int upload_bf16(DevBuf<__nv_bfloat16>* dst, const float* src, int rows, int cols, int np = 1) {
  const int ld = round_up(cols, 8);
  const long long ps = static_cast<long long>(rows) * ld;
  SB_TRY(alloc_filled(dst, static_cast<size_t>(ps) * np));
  return upload_parts(dst->p, src, rows, cols, ld, np, ps);
}

// np bf16 parts of part_stride elements on the device, rows of round_up(cols, 8) -> fp32 host [np, rows, cols] (widening
// is exact); raw keeps every part's bits, padding included
static int download_bf16(float* dst, const __nv_bfloat16* src, int rows, int cols, int np, long long part_stride,
                         std::vector<uint16_t>& raw) {
  const int ld = round_up(cols, 8);
  raw.resize(static_cast<size_t>(part_stride) * np);
  SB_CUDA(cudaMemcpy(raw.data(), src, sizeof(uint16_t) * raw.size(), cudaMemcpyDeviceToHost));
  for (int k = 0; k < np; ++k)
    for (int r = 0; r < rows; ++r)
      for (int c = 0; c < cols; ++c) {
        const uint32_t u = static_cast<uint32_t>(raw[static_cast<size_t>(k * part_stride) + static_cast<size_t>(r) * ld + c]) << 16;
        memcpy(dst + (static_cast<size_t>(k) * rows + r) * cols + c, &u, 4);
      }
  return SB_OK;
}

static int sync_hook(const char* kernel) {
  const cudaError_t e = cudaDeviceSynchronize();
  SB_CHECK(e == cudaSuccess, SB_ERR_CUDA, "%s failed: %s", kernel, cudaGetErrorString(e));
  return SB_OK;
}

// average device milliseconds per launch over `iters` back-to-back launches after `warmup` ones (CUDA events on the
// legacy stream)
template <typename Launch>
static int time_launches(Launch&& launch, int warmup, int iters, float* ms_out) {
  struct Events {
    cudaEvent_t e[2] = {};
    ~Events() { for (cudaEvent_t x : e) if (x) cudaEventDestroy(x); }
  } ev;
  SB_CUDA(cudaEventCreate(&ev.e[0]));
  SB_CUDA(cudaEventCreate(&ev.e[1]));
  for (int i = 0; i < warmup; ++i) SB_TRY(launch());
  SB_CUDA(cudaEventRecord(ev.e[0], 0));
  for (int i = 0; i < iters; ++i) SB_TRY(launch());
  SB_CUDA(cudaEventRecord(ev.e[1], 0));
  SB_CUDA(cudaEventSynchronize(ev.e[1]));
  float ms = 0.f;
  SB_CUDA(cudaEventElapsedTime(&ms, ev.e[0], ev.e[1]));
  *ms_out = ms / iters;
  return SB_OK;
}

static int debug_gemm_impl(const float* A, const float* B, float* D, int32_t M, int32_t N, int32_t K, int32_t split_k,
                           int32_t a_mn, int32_t b_mn, int32_t cfg_cg, int32_t cfg_bn, int device, int iters, float* ms_out) {
  SB_CHECK(cfg_cg == 0 || (cfg_cg == 1 && (cfg_bn == 64 || cfg_bn == 128 || (cfg_bn == 256 && a_mn && b_mn))), SB_ERR_INVALID,
           "tile configuration cg=%d bn=%d not instantiated for this layout (bn=256: MM only)", cfg_cg, cfg_bn);
  SB_CHECK(A && B && D && M > 0 && N > 0 && K > 0, SB_ERR_INVALID, "bad argument");
  SB_CHECK((a_mn == 0 && b_mn == 0) || (a_mn == 0 && b_mn == 1) || (a_mn == 1 && b_mn == 1), SB_ERR_INVALID,
           "layout combination not instantiated (use KK, KM or MM)");
  int sms = 0;
  SB_TRY(check_device(device, &sms));
  // stored shapes: K-major [R, K]; MN-major [K, R]
  const int a_rows = a_mn ? K : M, a_cols = a_mn ? M : K;
  const int b_rows = b_mn ? K : N, b_cols = b_mn ? N : K;
  const int lda = round_up(a_cols, 8), ldb = round_up(b_cols, 8);
  DevBuf<__nv_bfloat16> dA, dB;
  DevBuf<float> dD;
  SB_TRY(upload_bf16(&dA, A, a_rows, a_cols));
  SB_TRY(upload_bf16(&dB, B, b_rows, b_cols));
  SB_TRY(alloc_filled(&dD, static_cast<size_t>(M) * N));
  GemmPlan pl = plan_gemm(M, N, K, sms, false);
  if (cfg_cg > 0) pl.bn = cfg_bn;  // explicit tile configuration requested by the test
  {
    const int total_kb = (K + 63) / 64;
    int want = split_k < 1 ? 1 : (split_k > total_kb ? total_kb : split_k);
    pl.kb_per_split = (total_kb + want - 1) / want;
    pl.split_k = (total_kb + pl.kb_per_split - 1) / pl.kb_per_split;
    const int work = ((M + 127) / 128) * ((N + pl.bn - 1) / pl.bn) * pl.split_k;
    pl.grid = work < sms ? work : sms;
  }
  TmapSet tms;
  SB_TRY(make_tmap_bf16(&tms.a[0], dA.p, a_rows, a_cols, lda, a_mn ? 64 : 128));
  SB_TRY(make_tmap_bf16(&tms.b[0], dB.p, b_rows, b_cols, ldb, b_mn ? 64 : pl.bn));
  GemmTcParams p = {};
  p.M = M; p.N = N; p.K = K;
  p.accum = dD.p; p.ld_acc = N;
  p.acc_vec4 = (N % 4 == 0) ? 1 : 0;
  // 256-wide tiles (MM, the dW layout, only): the dW kernel, whose red.add into the zeroed D is the product
  if (pl.bn == 256) {
    SB_TRY(set_gemm_dw_attrs());
    SB_TRY(launch_gemm_dw(pl, tms, p, 0));
  } else if (!a_mn && !b_mn) {
    SB_TRY((set_gemm_tc_attrs<EPI_F32, false, false>()));
    SB_TRY((launch_gemm_tc<EPI_F32, false, false>(pl, tms, p, 0)));
  } else if (!a_mn) {
    SB_TRY((set_gemm_tc_attrs<EPI_F32, false, true>()));
    SB_TRY((launch_gemm_tc<EPI_F32, false, true>(pl, tms, p, 0)));
  } else {
    SB_TRY((set_gemm_tc_attrs<EPI_F32, true, true>()));
    SB_TRY((launch_gemm_tc<EPI_F32, true, true>(pl, tms, p, 0)));
  }
  if (iters > 0) {
    // benchmark with the REAL epilogue of the layout's use: KM -> forward (bias + relu -> bf16), KK -> dA
    // (act' * , bf16 store, column sums), MM -> dW (fp32 red.add)
    const int ldn = round_up(N, 8);
    DevBuf<float> d_bias, d_colsum;
    DevBuf<__nv_bfloat16> d_out, d_aux;
    SB_TRY(alloc_filled(&d_bias, N));
    SB_TRY(alloc_filled(&d_colsum, N));
    SB_TRY(d_out.alloc(static_cast<size_t>(M) * ldn));
    SB_TRY(alloc_filled(&d_aux, static_cast<size_t>(M) * ldn, 0x3f));
    GemmTcParams q = p;
    q.bias = d_bias.p; q.act = SB_ACT_RELU; q.out = d_out.p; q.ld_out = ldn; q.aux = d_aux.p; q.ld_aux = ldn; q.colsum = d_colsum.p;
    // KM / KK: the kernel the step plans for the shape
    const PpPlan pp = plan_gemm_pp(M, N, K, sms, !a_mn && b_mn);
    PpTmaps pt;
    if (!a_mn) {
      SB_TRY(make_tmap_bf16(&pt.a, dA.p, a_rows, a_cols, lda, pp.bm_wg));
      SB_TRY(make_tmap_bf16(&pt.b, dB.p, b_rows, b_cols, ldb, b_mn ? 64 : pp.bn));
      SB_TRY(make_tmap_bf16(&pt.o, d_out.p, M, N, ldn, pp.bm_wg));
      SB_TRY(make_tmap_bf16(&pt.x, d_aux.p, M, N, ldn, pp.bm_wg));
    }
    auto real = [&]() -> int {
      if (!a_mn && !b_mn) return launch_gemm_pp<EPI_DA>(pp, pt, q, 0, false);
      if (!a_mn) return pp.bn == 256 ? launch_gemm_wide(pp, pt, q, 0, false) : launch_gemm_pp<EPI_FWD>(pp, pt, q, 0, false);
      if (pl.bn == 256) return launch_gemm_dw(pl, tms, q, 0, false);
      return launch_gemm_tc<EPI_DW, true, true>(pl, tms, q, 0, false);
    };
    SB_TRY((a_mn ? set_gemm_tc_attrs<EPI_DW, true, true>() : set_gemm_pp_attrs()));
    if (pp.bn == 256) SB_TRY(set_gemm_wide_attrs());
    SB_TRY(time_launches(real, 3, iters, ms_out));
    if (getenv("SB_GEMM_TRACE")) {
      // one more launch with %globaltimer stamps from CTA 0 (ns relative to kernel entry), and the host-visible
      // launch-to-completion time of a single isolated launch
      DevBuf<unsigned long long> d_tr;
      SB_TRY(alloc_filled(&d_tr, 16));
      q.trace = d_tr.p;
      SB_CUDA(cudaDeviceSynchronize());
      float one = 0.f;
      SB_TRY(time_launches(real, 0, 1, &one));
      unsigned long long h[16];
      SB_CUDA(cudaMemcpy(h, d_tr.p, sizeof(h), cudaMemcpyDeviceToHost));
      if (a_mn)
        fprintf(stderr, "[trace] M=%d N=%d K=%d bn=%d split=%d single-launch %.2f us | ns since entry:", M, N, K, pl.bn, pl.split_k,
                one * 1e3f);
      else
        fprintf(stderr, "[trace] M=%d N=%d K=%d ping-pong bm_wg=%d bn=%d single-launch %.2f us | ns since entry:", M, N, K, pp.bm_wg,
                pp.bn, one * 1e3f);
      const char* nm[9] = {"entry", "setup", "deps", "tma0", "land0", "mma_done", "acc_ready", "epi_done", "exit"};
      for (int i = 1; i < 9; ++i) fprintf(stderr, " %s=%lld", nm[i], (long long)(h[i] - h[0]));
      fprintf(stderr, "\n");
    }
  }
  SB_TRY(sync_hook("gemm_tc_kernel"));
  SB_CUDA(cudaMemcpy(D, dD.p, sizeof(float) * M * N, cudaMemcpyDeviceToHost));
  return SB_OK;
}
}  // namespace sb

using namespace sb;

extern "C" {

int sb_debug_gemm_bf16_cfg(const float* A, const float* B, float* D, int32_t M, int32_t N, int32_t K, int32_t split_k,
                           int32_t a_mn, int32_t b_mn, int32_t cfg_cg, int32_t cfg_bn, int device) {
  return debug_gemm_impl(A, B, D, M, N, K, split_k, a_mn, b_mn, cfg_cg, cfg_bn, device, 0, nullptr);
}
int sb_debug_gemm_bench(const float* A, const float* B, float* D, int32_t M, int32_t N, int32_t K, int32_t split_k,
                        int32_t a_mn, int32_t b_mn, int32_t cfg_cg, int32_t cfg_bn, int device, int32_t iters, float* ms_out) {
  SB_CHECK(iters > 0 && ms_out, SB_ERR_INVALID, "iters / ms_out");
  return debug_gemm_impl(A, B, D, M, N, K, split_k, a_mn, b_mn, cfg_cg, cfg_bn, device, iters, ms_out);
}

// One forward, dA or dW GEMM of a training step, launched by the step's own Net::enqueue_* code on a Net built so that the
// GEMM is one of its layers (see shifu_b200.h)
int sb_debug_gemm_layer(int32_t kind, int32_t precision, const float* A, const float* W, const float* bias, const float* aux,
                        const float* addend, float* out, float* colsum, float* grad, int32_t* guard, char* route,
                        int32_t route_cap, int32_t M, int32_t N, int32_t K, int32_t a_rows, int32_t row0, int32_t act,
                        int32_t r0, int32_t r1, int32_t sms, int64_t clear_n4, int device) {
  enum { FWD = 0, DA = 1, DW = 2 };
  SB_CHECK(kind >= FWD && kind <= DW, SB_ERR_INVALID, "kind=%d (0 forward, 1 dA, 2 dW)", kind);
  SB_CHECK(precision >= SB_PREC_FP32 && precision <= SB_PREC_BF16X2, SB_ERR_INVALID, "precision=%d invalid", precision);
  SB_CHECK(act >= SB_ACT_NONE && act <= SB_ACT_LEAKYRELU, SB_ERR_INVALID, "act=%d invalid", act);
  SB_CHECK(M > 0 && N > 0 && K > 0, SB_ERR_INVALID, "M=%d N=%d K=%d", M, N, K);
  SB_CHECK(A && W && guard && (route == nullptr || route_cap > 0), SB_ERR_INVALID, "null argument");
  SB_CHECK(kind != FWD || (bias && out), SB_ERR_INVALID, "the forward GEMM needs bias and out");
  SB_CHECK(kind != DA || (aux && out && colsum), SB_ERR_INVALID, "the dA GEMM needs aux, out and colsum");
  SB_CHECK(kind != DW || grad, SB_ERR_INVALID, "the dW GEMM needs grad");
  SB_CHECK(addend == nullptr || kind == FWD, SB_ERR_INVALID, "an addend belongs to the forward GEMM only");
  const bool tc = precision != SB_PREC_FP32;
  const int rows = kind == DW ? K : M;                  // batch rows
  SB_CHECK(row0 >= 0 && static_cast<long long>(row0) + rows <= a_rows, SB_ERR_INVALID, "rows %d..%d outside the %d rows of A",
           row0, row0 + rows - 1, a_rows);
  const bool resident = row0 != 0 || a_rows != rows;
  SB_CHECK(!resident || (tc && kind != DA && addend == nullptr), SB_ERR_INVALID,
           "a resident batch is read by the layer-0 forward / dW GEMMs of a dense tensor-core step only");
  if (kind == DW) {
    SB_CHECK(r0 >= 0 && r0 < r1 && r1 <= M && r0 % 8 == 0, SB_ERR_INVALID, "rows r0=%d .. r1=%d of the %d-row gradient "
             "(r0 a multiple of 8)", r0, r1, M);
    SB_CHECK(tc || (r0 == 0 && r1 == M), SB_ERR_INVALID, "the fp32 dW GEMM has no row chunks");
  }
  SB_CHECK(clear_n4 >= 0 && (clear_n4 == 0 || (kind == FWD && tc)), SB_ERR_INVALID,
           "clear_n4=%lld: the tensor-core forward GEMM only", static_cast<long long>(clear_n4));
  SB_CHECK(sms >= 0, SB_ERR_INVALID, "sms=%d", sms);
  int dev_sms = 0;
  SB_TRY(check_device(device, &dev_sms));
  SB_CHECK(sms <= dev_sms, SB_ERR_INVALID, "sms=%d above the %d SMs", sms, dev_sms);

  // the net: forward = layer 0 (F = K, hidden [N]; a sparse step contracts the K dense columns of F = K + 1), dA = layer 1
  // (hidden [N, K]), dW = layer 0 (F = M, hidden [N]).  64 rows past the batch in every activation part are guard rows.
  sb_net_desc d = {};
  d.n_features = kind == FWD ? (addend ? K + 1 : K) : (kind == DA ? 8 : M);
  d.n_hidden = kind == DA ? 2 : 1;
  d.hidden[0] = N; d.acts[0] = kind == DW ? SB_ACT_NONE : act;
  d.hidden[1] = K; d.acts[1] = SB_ACT_NONE;
  d.loss = SB_LOSS_MSE; d.optimizer = SB_OPT_SGD;
  d.max_batch = kind == DW ? K : M + 64;
  d.precision = precision;
  constexpr int GUARD = 256;                            // floats behind the gradient / the cleared buffer
  const uint32_t S32 = 0x7f7f7f7fu;                     // sentinels: fp32 3.4e38, bf16 3.4e38
  const uint16_t S16 = 0x7f7f;
  DevBuf<__nv_bfloat16> res;
  DevBuf<float> g, clr;
  Net net;                                              // (destroyed first: waits for its stream)
  SB_TRY(net.init(&d, device, true));
  if (sms > 0) net.num_sms = sms;
  const int np = net.nparts;
  if (addend) SB_TRY(net.set_sparse(K, 1, 1));
  const Layer& l0 = net.layers[0];
  // parameters: W and bias into theta, the bf16 shadows from there (set_params)
  std::vector<float> theta(static_cast<size_t>(net.n_params), 0.f);
  if (kind == FWD) {
    std::copy(W, W + static_cast<size_t>(K) * N, theta.begin() + l0.w_off);
    std::copy(bias, bias + N, theta.begin() + l0.b_off);
  } else if (kind == DA) {
    std::copy(W, W + static_cast<size_t>(N) * K, theta.begin() + net.layers[1].w_off);
  }
  SB_CUDA(cudaMemcpy(net.theta, theta.data(), sizeof(float) * theta.size(), cudaMemcpyHostToDevice));
  BatchDesc hd = {};
  hd.row0 = row0;
  SB_CUDA(cudaMemcpy(net.desc, &hd, sizeof(hd), cudaMemcpyHostToDevice));
  // the batch operand of layer 0: the staged batch, or the resident set
  StepIn in{net.desc, net.scal, resident ? Feed::RESIDENT : addend ? Feed::SPARSE : Feed::HOST};
  if (kind != DA) {
    const int cols = kind == FWD ? K : M;
    if (resident) {
      const long long ps = static_cast<long long>(a_rows) * net.ldF;
      SB_TRY(alloc_filled(&res, static_cast<size_t>(ps) * np));
      SB_TRY(upload_parts(res.p, A, a_rows, cols, net.ldF, np, ps));
      in.x0 = Operand0{res.p, ps, a_rows, true};
    } else if (tc) {
      SB_TRY(upload_parts(net.Xb, A, rows, cols, addend ? net.ldD : net.ldF, np, net.Xb_ps));
    } else {
      SB_CUDA(cudaMemcpy(net.Xf, A, sizeof(float) * rows * cols, cudaMemcpyHostToDevice));
    }
  }
  if (addend)
    SB_CUDA(cudaMemcpy2D(net.E, sizeof(float) * l0.ld_out, addend, sizeof(float) * N, sizeof(float) * N, M, cudaMemcpyHostToDevice));
  if (kind == DA) {     // dZ_1 [M, K], A_0 [M, N]
    if (tc) {
      SB_TRY(upload_parts(net.dZ[1], A, M, K, net.layers[1].ld_out, np, net.A_ps[1]));
      SB_TRY(upload_parts(net.A[0], aux, M, N, l0.ld_out, np, net.A_ps[0]));
    } else {
      SB_CUDA(cudaMemcpy(net.dZf[1], A, sizeof(float) * M * K, cudaMemcpyHostToDevice));
      SB_CUDA(cudaMemcpy(net.Af[0], aux, sizeof(float) * M * N, cudaMemcpyHostToDevice));
    }
  }
  if (kind == DW) {     // dZ_0 [K, N]
    if (tc) SB_TRY(upload_parts(net.dZ[0], W, K, N, l0.ld_out, np, net.A_ps[0]));
    else SB_CUDA(cudaMemcpy(net.dZf[0], W, sizeof(float) * K * N, cudaMemcpyHostToDevice));
  }
  // the output, with its guard rows and pad columns, filled with the sentinel
  void* outp = nullptr;
  size_t out_bytes = 0;
  if (kind != DW) {
    outp = tc ? static_cast<void*>(kind == FWD ? net.A[0] : net.dZ[0]) : static_cast<void*>(kind == FWD ? net.Af[0] : net.dZf[0]);
    out_bytes = tc ? sizeof(__nv_bfloat16) * net.A_ps[0] * np : sizeof(float) * static_cast<size_t>(net.max_batch) * N;
    SB_CUDA(cudaMemset(outp, 0x7f, out_bytes));
  }
  // the gradient: the in/out region (dA: the column sums = layer 0's bias slot; dW: rows r0 .. r1 - 1 of W_0's slot) holds
  // the caller's values, everything else and GUARD floats behind it the sentinel
  const size_t g_n = static_cast<size_t>(net.n_params) + GUARD;
  std::vector<float> hg(g_n);
  {
    float s;
    memcpy(&s, &S32, 4);
    std::fill(hg.begin(), hg.end(), s);
  }
  auto in_region = [&](size_t i) {
    if (kind == DA) return i >= static_cast<size_t>(l0.b_off) && i < static_cast<size_t>(l0.b_off) + N;
    return i >= static_cast<size_t>(r0) * N && i < static_cast<size_t>(r1) * N;    // W_0 at offset 0
  };
  if (kind == DA) std::copy(colsum, colsum + N, hg.begin() + l0.b_off);
  if (kind == DW) std::copy(grad + static_cast<size_t>(r0) * N, grad + static_cast<size_t>(r1) * N, hg.begin() + static_cast<size_t>(r0) * N);
  if (kind != FWD) {
    SB_TRY(g.alloc(g_n));
    SB_CUDA(cudaMemcpy(g.p, hg.data(), sizeof(float) * g_n, cudaMemcpyHostToDevice));
  }
  const size_t clr_n = clear_n4 > 0 ? static_cast<size_t>(clear_n4) * 4 + GUARD : 0;
  if (clear_n4 > 0) SB_TRY(alloc_filled(&clr, clr_n, 0x7f));
  SB_CUDA(cudaDeviceSynchronize());     // the uploads above ran on the legacy stream, the net launches on its own

  SB_TRY(net.refresh_shadows());
  net.launches = 0;
  if (kind == FWD) SB_TRY(net.enqueue_hidden_forward(in, M, nullptr, nullptr, reinterpret_cast<float4*>(clr.p), clear_n4));
  else if (kind == DA) SB_TRY(net.enqueue_da(1, M, g.p));
  else SB_TRY(net.enqueue_dw(in, 0, K, g.p, net.stream, false, sms > 0 ? sms : dev_sms, r0, r1));
  SB_CHECK(net.launches == 1 && net.last_kernel != nullptr, SB_ERR_STATE, "%d GEMM launches", net.launches);
  SB_TRY(sync_hook(net.last_kernel));
  if (route) {
    strncpy(route, net.last_kernel, static_cast<size_t>(route_cap) - 1);
    route[route_cap - 1] = '\0';
  }

  int32_t changed = 0;
  if (kind != DW) {
    if (tc) {
      std::vector<uint16_t> h;
      SB_TRY(download_bf16(out, static_cast<const __nv_bfloat16*>(outp), M, N, np, net.A_ps[0], h));
      // pad columns of a batch row may hold what the kernels store beyond N: forward the parts of act(0) (the tile is 0
      // there), dA +-0
      const uint16_t a0 = kind == FWD && act == SB_ACT_SIGMOID ? 0x3f00 : 0;     // bf16(0.5)
      const int ld = l0.ld_out;
      for (int k = 0; k < np; ++k)
        for (int r = 0; r < M + 64; ++r)
          for (int c = (r < M ? N : 0); c < ld; ++c) {
            const uint16_t v = h[static_cast<size_t>(k * net.A_ps[0]) + static_cast<size_t>(r) * ld + c];
            const uint16_t want = k == 0 ? a0 : 0;
            const bool legit = r < M && (v == want || (want == 0 && v == 0x8000));
            if (v != S16 && !legit) ++changed;
          }
    } else {
      std::vector<uint32_t> h(static_cast<size_t>(M + 64) * N);
      SB_CUDA(cudaMemcpy(h.data(), outp, sizeof(uint32_t) * h.size(), cudaMemcpyDeviceToHost));
      memcpy(out, h.data(), sizeof(float) * M * N);
      for (size_t i = static_cast<size_t>(M) * N; i < h.size(); ++i) changed += h[i] != S32;
    }
  }
  if (kind != FWD) {
    SB_CUDA(cudaMemcpy(hg.data(), g.p, sizeof(float) * g_n, cudaMemcpyDeviceToHost));
    for (size_t i = 0; i < g_n; ++i) {
      uint32_t u;
      memcpy(&u, &hg[i], 4);
      if (!in_region(i) && u != S32) ++changed;
    }
    if (kind == DA) std::copy(hg.begin() + l0.b_off, hg.begin() + l0.b_off + N, colsum);
    else std::copy(hg.begin() + static_cast<size_t>(r0) * N, hg.begin() + static_cast<size_t>(r1) * N, grad + static_cast<size_t>(r0) * N);
  }
  if (clear_n4 > 0) {
    std::vector<uint32_t> h(clr_n);
    SB_CUDA(cudaMemcpy(h.data(), clr.p, sizeof(uint32_t) * clr_n, cudaMemcpyDeviceToHost));
    for (size_t i = 0; i < clr_n; ++i) changed += i < clr_n - GUARD ? h[i] != 0u : h[i] != S32;
  }
  *guard = changed;
  return SB_OK;
}

int sb_debug_gemm_epilogue(const float* A, const float* W, const float* bias, const float* aux, float* out, float* colsum,
                           int32_t M, int32_t N, int32_t K, int32_t da, int32_t act, int32_t bm_wg, int device,
                           int32_t iters, float* ms_out) {
  SB_CHECK(A && W && out && M > 0 && N > 0 && K > 0 && (da == 0 || da == 1), SB_ERR_INVALID, "bad argument");
  SB_CHECK(da ? aux != nullptr : bias != nullptr, SB_ERR_INVALID, "the forward GEMM needs a bias, the dA GEMM an aux matrix");
  SB_CHECK(act >= SB_ACT_NONE && act <= SB_ACT_LEAKYRELU, SB_ERR_INVALID, "act invalid");
  SB_CHECK(bm_wg == 0 || bm_wg == 64 || bm_wg == 128 || bm_wg == PP_TILE_WIDE, SB_ERR_INVALID,
           "bm_wg must be 0, 64, 128 or %d (got %d)", PP_TILE_WIDE, bm_wg);
  SB_CHECK(!(da && bm_wg == PP_TILE_WIDE), SB_ERR_INVALID, "the %d-wide tile is for the forward GEMM only", PP_TILE_WIDE);
  SB_CHECK(iters >= 0 && (iters == 0 || ms_out != nullptr), SB_ERR_INVALID, "iters / ms_out");
  int sms = 0;
  SB_TRY(check_device(device, &sms));
  // stored shapes: A [M, K]; W [K, N] (forward, MN-major operand) or [N, K] (dA, K-major operand)
  const int w_rows = da ? N : K, w_cols = da ? K : N;
  const int lda = round_up(K, 8), ldw = round_up(w_cols, 8), ldn = round_up(N, 8);
  DevBuf<__nv_bfloat16> dA, dW, d_out, d_aux;
  DevBuf<float> d_bias, d_col;
  SB_TRY(upload_bf16(&dA, A, M, K));
  SB_TRY(upload_bf16(&dW, W, w_rows, w_cols));
  SB_TRY(alloc_filled(&d_out, static_cast<size_t>(M) * ldn));
  SB_TRY(aux ? upload_bf16(&d_aux, aux, M, N) : alloc_filled(&d_aux, static_cast<size_t>(M) * ldn));
  SB_TRY(alloc_filled(&d_bias, N));
  SB_TRY(alloc_filled(&d_col, N));
  if (bias) SB_CUDA(cudaMemcpy(d_bias.p, bias, sizeof(float) * N, cudaMemcpyHostToDevice));
  const PpPlan pp = plan_gemm_pp(M, N, K, sms, da == 0, bm_wg);
  PpTmaps pt;
  SB_TRY(make_tmap_bf16(&pt.a, dA.p, M, K, lda, pp.bm_wg));
  SB_TRY(make_tmap_bf16(&pt.b, dW.p, w_rows, w_cols, ldw, da ? pp.bn : 64));
  SB_TRY(make_tmap_bf16(&pt.o, d_out.p, M, N, ldn, pp.bm_wg));
  SB_TRY(make_tmap_bf16(&pt.x, d_aux.p, M, N, ldn, pp.bm_wg));
  GemmTcParams p = {};
  p.M = M; p.N = N; p.K = K;
  p.act = act; p.bias = d_bias.p; p.colsum = colsum ? d_col.p : nullptr;
  auto launch = [&]() {
    if (da) return launch_gemm_pp<EPI_DA>(pp, pt, p, 0, false);
    return pp.bn == 256 ? launch_gemm_wide(pp, pt, p, 0, false) : launch_gemm_pp<EPI_FWD>(pp, pt, p, 0, false);
  };
  const char* kernel = pp.bn == 256 ? "gemm_wide_kernel" : "gemm_pp_kernel";
  SB_TRY(pp.bn == 256 ? set_gemm_wide_attrs() : set_gemm_pp_attrs());
  SB_TRY(launch());
  SB_TRY(sync_hook(kernel));
  std::vector<uint16_t> h;
  SB_TRY(download_bf16(out, d_out.p, M, N, 1, static_cast<long long>(M) * ldn, h));
  if (colsum) SB_CUDA(cudaMemcpy(colsum, d_col.p, sizeof(float) * N, cudaMemcpyDeviceToHost));
  if (iters > 0) {
    SB_TRY(time_launches(launch, 3, iters, ms_out));
    SB_TRY(sync_hook(kernel));
  }
  return SB_OK;
}

int sb_debug_gemm_fwd_out(const float* A, const float* W, const float* bias, const float* wo, float bo, const float* y,
                          const float* w, float* dZ, float* g_bL, float* g_wo, float* g_bo, float* loss_sum, int32_t* guard,
                          int32_t M, int32_t N, int32_t K, int32_t a_rows, int32_t row0, int32_t act, int32_t loss,
                          int32_t np, int32_t grid, int device) {
  SB_CHECK(A && W && bias && wo && y && w && dZ && g_bL && g_wo && g_bo && loss_sum && guard, SB_ERR_INVALID, "null argument");
  SB_CHECK(M > 0 && K > 0 && N >= 1 && N <= FWD_OUT_MAX_N, SB_ERR_INVALID, "M=%d K=%d N=%d (N must be 1..%d)", M, K, N,
           FWD_OUT_MAX_N);
  SB_CHECK(np >= 1 && np <= 3, SB_ERR_INVALID, "np=%d outside 1..3", np);
  SB_CHECK(loss == SB_LOSS_MSE || loss == SB_LOSS_SIGMOID_CE, SB_ERR_INVALID, "loss invalid");
  SB_CHECK(act >= SB_ACT_NONE && act <= SB_ACT_LEAKYRELU, SB_ERR_INVALID, "act invalid");
  SB_CHECK(grid >= 0, SB_ERR_INVALID, "grid=%d", grid);
  SB_CHECK(row0 >= 0 && static_cast<long long>(row0) + M <= a_rows, SB_ERR_INVALID, "rows %d..%d outside the %d rows of A", row0,
           row0 + M - 1, a_rows);
  int sms = 0;
  SB_TRY(check_device(device, &sms));
  SB_CHECK(grid <= sms, SB_ERR_INVALID, "grid=%d above the %d SMs", grid, sms);
  // the step's layout: parts one after the other, rows of ld = round_up(cols, 8) elements; dZ has 64 guard rows per part
  const int lda = round_up(K, 8), ldn = round_up(N, 8), dz_rows = M + 64;
  const long long a_ps = static_cast<long long>(a_rows) * lda, w_ps = static_cast<long long>(K) * ldn;
  const long long dz_ps = static_cast<long long>(dz_rows) * ldn;
  DevBuf<__nv_bfloat16> dA, dW, d_dz;
  DevBuf<float> d_vec, d_yw;
  DevBuf<BatchDesc> d_desc;
  SB_TRY(upload_bf16(&dA, A, a_rows, K, np));
  SB_TRY(upload_bf16(&dW, W, K, N, np));
  SB_TRY(alloc_filled(&d_dz, static_cast<size_t>(dz_ps) * np, 0x7f));   // every element the bf16 sentinel 0x7f7f
  // [bias N][w_o N][db_L N][dw_o N][b_o][db_o][scal SCAL_COUNT]
  float nnz = 0.f;
  for (int r = 0; r < M; ++r) nnz += (w[r] != 0.f) ? 1.f : 0.f;
  std::vector<float> h_vec(4 * N + 2 + SCAL_COUNT, 0.f);
  std::copy(bias, bias + N, h_vec.begin());
  std::copy(wo, wo + N, h_vec.begin() + N);
  std::copy(g_bL, g_bL + N, h_vec.begin() + 2 * N);
  std::copy(g_wo, g_wo + N, h_vec.begin() + 3 * N);
  h_vec[4 * N] = bo;
  h_vec[4 * N + 1] = *g_bo;
  h_vec[4 * N + 2 + SCAL_LOSS_SUM] = *loss_sum;
  h_vec[4 * N + 2 + SCAL_NNZ] = nnz;
  SB_TRY(d_vec.alloc(h_vec.size()));
  SB_CUDA(cudaMemcpy(d_vec.p, h_vec.data(), sizeof(float) * h_vec.size(), cudaMemcpyHostToDevice));
  float* d_bias = d_vec.p;
  float* d_wo = d_vec.p + N;
  float* d_gbL = d_vec.p + 2 * N;
  float* d_gwo = d_vec.p + 3 * N;
  float* d_bo = d_vec.p + 4 * N;
  float* d_gbo = d_bo + 1;
  float* d_scal = d_bo + 2;
  SB_TRY(d_yw.alloc(2 * static_cast<size_t>(M)));
  SB_CUDA(cudaMemcpy(d_yw.p, y, sizeof(float) * M, cudaMemcpyHostToDevice));
  SB_CUDA(cudaMemcpy(d_yw.p + M, w, sizeof(float) * M, cudaMemcpyHostToDevice));
  BatchDesc h_desc = {};
  h_desc.y = d_yw.p; h_desc.w = d_yw.p + M; h_desc.gscale = 1.f; h_desc.row0 = row0;
  SB_TRY(d_desc.alloc(1));
  SB_CUDA(cudaMemcpy(d_desc.p, &h_desc, sizeof(BatchDesc), cudaMemcpyHostToDevice));
  // the launch of Net::enqueue_hidden_forward's fused branch
  const bool resident = row0 != 0 || a_rows != M;
  FwdOutTmaps ft;
  SB_TRY(make_tmaps_bf16(ft.a, dA.p, a_ps, np, a_rows, K, lda, 64));
  SB_TRY(make_tmaps_bf16(ft.b, dW.p, w_ps, np, K, N, ldn, 64));
  SB_TRY(make_tmaps_bf16(ft.o, d_dz.p, dz_ps, np, M, N, ldn, 64));
  GemmTcParams p = {};
  set_part_pairs(&p, np);
  p.M = M; p.N = N; p.K = K;
  p.bias = d_bias; p.act = act;
  p.a_rows = resident ? d_desc.p : nullptr;
  p.wo = d_wo; p.bo = d_bo;
  p.desc = d_desc.p; p.scal = d_scal; p.loss = loss;
  p.g_wo = d_gwo; p.g_bo = d_gbo; p.g_bL = d_gbL;
  const int tiles = (M + 63) / 64;
  const int step_grid = tiles < sms ? tiles : sms;
  SB_TRY(set_gemm_fwd_out_attrs());
  SB_TRY(launch_gemm_fwd_out(grid > 0 ? grid : step_grid, ft, p, 0, false));
  SB_TRY(sync_hook("gemm_fwd_out_kernel"));
  std::vector<uint16_t> h;
  SB_TRY(download_bf16(dZ, d_dz.p, M, N, np, dz_ps, h));
  SB_CUDA(cudaMemcpy(h_vec.data(), d_vec.p, sizeof(float) * h_vec.size(), cudaMemcpyDeviceToHost));
  int32_t changed = 0;
  for (int k = 0; k < np; ++k)
    for (int r = 0; r < dz_rows; ++r)
      for (int c = 0; c < ldn; ++c) {
        const uint16_t v = h[static_cast<size_t>(k * dz_ps) + static_cast<size_t>(r) * ldn + c];
        // the bulk tensor store writes a row's last 16-byte piece whole, so the pad columns of a batch row may receive
        // the tile's +-0 beyond N; anything else, or any write into the guard rows, is counted
        if ((r >= M || c >= N) && v != 0x7f7f && (r >= M || (v & 0x7fff) != 0)) ++changed;
      }
  *guard = changed;
  std::copy(h_vec.begin() + 2 * N, h_vec.begin() + 3 * N, g_bL);
  std::copy(h_vec.begin() + 3 * N, h_vec.begin() + 4 * N, g_wo);
  *g_bo = h_vec[4 * N + 1];
  *loss_sum = h_vec[4 * N + 2 + SCAL_LOSS_SUM];
  return SB_OK;
}

// The output layer of a step launched by Net::enqueue_out on a Net whose last hidden layer holds A_L (see shifu_b200.h)
int sb_debug_out_layer(int32_t precision, int32_t det, int32_t do_loss, int32_t do_bwd, const float* A, const float* wo, float bo,
                       const float* y, const float* w, float* yhat, float* dZ, float* g_bL, float* g_wo, float* g_bo,
                       float* loss_sum, int32_t* guard, int32_t* repeat_same, char* route, int32_t route_cap, int32_t M, int32_t H,
                       int32_t act, int32_t loss, int32_t sms, int device) {
  SB_CHECK(precision >= SB_PREC_FP32 && precision <= SB_PREC_BF16X2, SB_ERR_INVALID, "precision=%d invalid", precision);
  SB_CHECK((det == 0 || det == 1) && (do_loss == 0 || do_loss == 1) && (do_bwd == 0 || do_bwd == 1), SB_ERR_INVALID,
           "det=%d do_loss=%d do_bwd=%d (each 0 or 1)", det, do_loss, do_bwd);
  SB_CHECK(do_loss || !do_bwd, SB_ERR_INVALID, "do_bwd needs do_loss: the backward starts from the loss gradient");
  SB_CHECK(M >= 1 && M <= (1 << 30) && H >= 1 && H <= (1 << 20), SB_ERR_INVALID, "M=%d H=%d", M, H);
  SB_CHECK(act >= SB_ACT_NONE && act <= SB_ACT_LEAKYRELU, SB_ERR_INVALID, "act=%d invalid", act);
  SB_CHECK(loss == SB_LOSS_MSE || loss == SB_LOSS_SIGMOID_CE, SB_ERR_INVALID, "loss=%d invalid", loss);
  SB_CHECK(A && wo && guard && (route == nullptr || route_cap > 0), SB_ERR_INVALID, "null argument");
  SB_CHECK(!do_loss || (y && w && loss_sum), SB_ERR_INVALID, "the loss needs y, w and loss_sum");
  SB_CHECK(!do_bwd || (dZ && g_bL && g_wo && g_bo), SB_ERR_INVALID, "the backward needs dZ, g_bL, g_wo and g_bo");
  SB_CHECK(do_loss || yhat, SB_ERR_INVALID, "a score (do_loss = 0) needs yhat");
  SB_CHECK(sms >= 0, SB_ERR_INVALID, "sms=%d", sms);
  int dev_sms = 0;
  SB_TRY(check_device(device, &dev_sms));
  SB_CHECK(sms <= dev_sms, SB_ERR_INVALID, "sms=%d above the %d SMs", sms, dev_sms);

  // the net: F = 8, hidden [H] with A_L = A_0; 64 rows past the batch in every activation part are guard rows
  sb_net_desc d = {};
  d.n_features = 8; d.n_hidden = 1;
  d.hidden[0] = H; d.acts[0] = act;
  d.loss = loss; d.optimizer = SB_OPT_SGD;
  d.max_batch = M + 64;
  d.precision = precision;
  constexpr int GUARD = 256;                            // floats behind the gradient
  const uint32_t S32 = 0x7f7f7f7fu;                     // sentinels: fp32 3.4e38, bf16 3.4e38
  const uint16_t S16 = 0x7f7f;
  const float qnan = std::numeric_limits<float>::quiet_NaN();
  float s32;
  memcpy(&s32, &S32, 4);
  DevBuf<float> g, d_yh, d_yw;
  Net net;                                              // (destroyed first: waits for its stream)
  SB_TRY(net.init(&d, device, true));
  if (det) SB_TRY(net.enable_det());
  if (sms > 0) net.num_sms = sms;
  const bool tc = net.tc();
  const int np = net.nparts;
  const Layer& hl = net.layers[0];
  const Layer& ol = net.layers[1];
  const int rows_all = M + 64, ld = tc ? hl.ld_out : H;
  std::vector<float> theta(static_cast<size_t>(net.n_params), 0.f);
  std::copy(wo, wo + H, theta.begin() + ol.w_off);
  theta[static_cast<size_t>(ol.b_off)] = bo;
  SB_CUDA(cudaMemcpy(net.theta, theta.data(), sizeof(float) * theta.size(), cudaMemcpyHostToDevice));
  // A_L: every part's pad columns and the 64 rows past M hold NaN, which a result can only show if the kernel reads them
  if (tc) {
    SB_CUDA(cudaMemset(net.A[0], 0xff, sizeof(__nv_bfloat16) * static_cast<size_t>(net.A_ps[0]) * np));
    SB_TRY(upload_parts(net.A[0], A, M, H, ld, np, net.A_ps[0]));
  } else {
    SB_CUDA(cudaMemset(net.Af[0], 0xff, sizeof(float) * static_cast<size_t>(rows_all) * H));
    SB_CUDA(cudaMemcpy(net.Af[0], A, sizeof(float) * static_cast<size_t>(M) * H, cudaMemcpyHostToDevice));
  }
  // y / w: the caller's rows, NaN behind them; all NaN for a score, which must not read them
  std::vector<float> hyw(2 * static_cast<size_t>(rows_all), qnan);
  float nnz = 0.f;
  if (do_loss) {
    std::copy(y, y + M, hyw.begin());
    std::copy(w, w + M, hyw.begin() + rows_all);
    for (int r = 0; r < M; ++r) nnz += w[r] != 0.f ? 1.f : 0.f;
  }
  SB_TRY(d_yw.alloc(hyw.size()));
  SB_CUDA(cudaMemcpy(d_yw.p, hyw.data(), sizeof(float) * hyw.size(), cudaMemcpyHostToDevice));
  BatchDesc hd = {};
  hd.y = d_yw.p; hd.w = d_yw.p + rows_all; hd.gscale = 1.f;
  SB_CUDA(cudaMemcpy(net.desc, &hd, sizeof(hd), cudaMemcpyHostToDevice));
  // the step scalars: the loss sum in/out and n_nz; the other words (and both, for a score) must keep what they hold
  float hscal[SCAL_COUNT];
  std::fill(hscal, hscal + SCAL_COUNT, s32);
  hscal[SCAL_NNZ] = do_loss ? nnz : qnan;
  if (do_loss) hscal[SCAL_LOSS_SUM] = *loss_sum;
  // the flat gradient: the g_bL, g_wo, g_bo slots (contiguous: b_0, w_o, b_o) in/out on a backward, the rest and GUARD
  // floats behind it the sentinel
  const size_t g_n = static_cast<size_t>(net.n_params) + GUARD;
  const size_t io0 = static_cast<size_t>(hl.b_off), io1 = static_cast<size_t>(ol.b_off) + 1;
  std::vector<float> hg(g_n, s32);
  if (do_bwd) {
    std::copy(g_bL, g_bL + H, hg.begin() + hl.b_off);
    std::copy(g_wo, g_wo + H, hg.begin() + ol.w_off);
    hg[static_cast<size_t>(ol.b_off)] = *g_bo;
  }
  SB_TRY(g.alloc(g_n));
  SB_TRY(d_yh.alloc(rows_all));
  void* dz_dev = tc ? static_cast<void*>(net.dZ[0]) : static_cast<void*>(net.dZf[0]);
  const size_t dz_bytes = tc ? sizeof(__nv_bfloat16) * static_cast<size_t>(net.A_ps[0]) * np : sizeof(float) * static_cast<size_t>(rows_all) * H;
  // one launch from the initial values -> the raw bits of [gradient | scalars | yhat | dZ]
  const size_t o_scal = g_n * 4, o_yh = o_scal + sizeof(hscal), o_dz = o_yh + sizeof(float) * rows_all;
  std::vector<char> res, first;
  StepIn in;
  in.desc = net.desc; in.scal = net.scal;
  auto launch = [&](std::vector<char>& out) -> int {
    SB_CUDA(cudaMemcpy(g.p, hg.data(), sizeof(float) * g_n, cudaMemcpyHostToDevice));
    SB_CUDA(cudaMemcpy(net.scal, hscal, sizeof(hscal), cudaMemcpyHostToDevice));
    SB_CUDA(cudaMemset(d_yh.p, 0x7f, sizeof(float) * rows_all));
    SB_CUDA(cudaMemset(dz_dev, 0x7f, dz_bytes));
    SB_CUDA(cudaDeviceSynchronize());     // the uploads ran on the legacy stream, the net launches on its own
    net.launches = 0;
    SB_TRY(net.enqueue_out(in, M, do_loss != 0, do_bwd != 0, yhat ? d_yh.p : nullptr, g.p));
    SB_CHECK(net.launches == 1 && net.last_kernel != nullptr, SB_ERR_STATE, "%d output-layer launches", net.launches);
    SB_TRY(sync_hook(net.last_kernel));
    out.resize(o_dz + dz_bytes);
    SB_CUDA(cudaMemcpy(out.data(), g.p, sizeof(float) * g_n, cudaMemcpyDeviceToHost));
    SB_CUDA(cudaMemcpy(out.data() + o_scal, net.scal, sizeof(hscal), cudaMemcpyDeviceToHost));
    SB_CUDA(cudaMemcpy(out.data() + o_yh, d_yh.p, sizeof(float) * rows_all, cudaMemcpyDeviceToHost));
    SB_CUDA(cudaMemcpy(out.data() + o_dz, dz_dev, dz_bytes, cudaMemcpyDeviceToHost));
    return SB_OK;
  };
  // DET: a second launch on the same net (its slots and ticket as the first one left them) from the same initial values
  SB_TRY(launch(res));
  if (det) {
    first.swap(res);
    SB_TRY(launch(res));
  }
  if (repeat_same) *repeat_same = det ? (res == first ? 1 : 0) : -1;
  if (route) {
    strncpy(route, net.last_kernel, static_cast<size_t>(route_cap) - 1);
    route[route_cap - 1] = '\0';
  }

  int32_t changed = 0;
  auto u32_at = [&](size_t byte) { uint32_t u; memcpy(&u, res.data() + byte, 4); return u; };
  for (size_t i = 0; i < g_n; ++i)
    if (!(do_bwd && i >= io0 && i < io1) && u32_at(4 * i) != S32) ++changed;
  for (int i = 0; i < SCAL_COUNT; ++i) {
    uint32_t want;
    memcpy(&want, hscal + i, 4);
    if (!(do_loss && i == SCAL_LOSS_SUM) && u32_at(o_scal + 4 * i) != want) ++changed;
  }
  for (int r = M; r < rows_all; ++r) changed += u32_at(o_yh + 4 * static_cast<size_t>(r)) != S32;
  if (yhat) memcpy(yhat, res.data() + o_yh, sizeof(float) * M);
  if (do_bwd) {
    memcpy(g_bL, res.data() + 4 * hl.b_off, sizeof(float) * H);
    memcpy(g_wo, res.data() + 4 * ol.w_off, sizeof(float) * H);
    memcpy(g_bo, res.data() + 4 * ol.b_off, sizeof(float));
  }
  if (do_loss) memcpy(loss_sum, res.data() + o_scal + 4 * SCAL_LOSS_SUM, sizeof(float));
  // dZ: a backward writes the batch rows' H columns; a batch row's pad columns may hold the sentinel or the +-0 of the
  // 16-byte piece that reaches into them; nothing else changes (a score or an eval: nothing at all)
  if (tc) {
    const uint16_t* h = reinterpret_cast<const uint16_t*>(res.data() + o_dz);
    for (int k = 0; k < np; ++k)
      for (int r = 0; r < rows_all; ++r)
        for (int c = 0; c < ld; ++c) {
          const uint16_t v = h[static_cast<size_t>(k * net.A_ps[0]) + static_cast<size_t>(r) * ld + c];
          if (do_bwd && r < M && c < H) {
            const uint32_t u = static_cast<uint32_t>(v) << 16;
            memcpy(dZ + (static_cast<size_t>(k) * M + r) * H + c, &u, 4);
          } else if (v != S16 && !(do_bwd && r < M && (v & 0x7fff) == 0)) {
            ++changed;
          }
        }
  } else {
    for (size_t i = 0; i < static_cast<size_t>(rows_all) * H; ++i)
      if (do_bwd && i < static_cast<size_t>(M) * H) memcpy(dZ + i, res.data() + o_dz + 4 * i, 4);
      else changed += u32_at(o_dz + 4 * i) != S32;
  }
  *guard = changed;
  return SB_OK;
}

// The wide+deep embedding gather / scatter-add of a sparse step launched by Net::enqueue_embed (see shifu_b200.h)
int sb_debug_embed(int32_t precision, int32_t scatter, const float* We, const int32_t* idx, const float* dZ, float* out,
                   int32_t* guard, int32_t rows, int32_t H, int32_t n_onehot, int32_t n_cat, int device) {
  SB_CHECK(precision >= SB_PREC_FP32 && precision <= SB_PREC_BF16X2, SB_ERR_INVALID, "precision=%d invalid", precision);
  SB_CHECK(scatter == 0 || scatter == 1, SB_ERR_INVALID, "scatter=%d (0 gather, 1 scatter-add)", scatter);
  SB_CHECK(rows >= 1 && rows <= (1 << 24) && H >= 1 && H <= (1 << 16) && n_onehot >= 1 && n_onehot <= (1 << 24) && n_cat >= 1 &&
           n_cat <= 4096, SB_ERR_INVALID, "rows=%d H=%d n_onehot=%d n_cat=%d", rows, H, n_onehot, n_cat);
  SB_CHECK(idx && out && guard, SB_ERR_INVALID, "null argument");
  SB_CHECK(scatter ? dZ != nullptr : We != nullptr, SB_ERR_INVALID, "the gather needs We, the scatter-add dZ");
  SB_TRY(check_sparse_idx(idx, static_cast<long long>(rows) * n_cat, n_onehot));
  SB_CHECK(static_cast<long long>(3 + n_onehot) * H < (1LL << 31), SB_ERR_INVALID, "W_0 of %d x %d elements", 3 + n_onehot, H);
  int dev_sms = 0;
  SB_TRY(check_device(device, &dev_sms));

  // the net: n_dense = 3 dense columns ahead of the n_onehot embedding rows of W_0, hidden [H]; 64 guard rows past the batch
  constexpr int N_DENSE = 3, GUARD = 256;
  sb_net_desc d = {};
  d.n_features = N_DENSE + n_onehot; d.n_hidden = 1;
  d.hidden[0] = H; d.acts[0] = SB_ACT_NONE;
  d.loss = SB_LOSS_MSE; d.optimizer = SB_OPT_SGD;
  d.max_batch = rows + 64;
  d.precision = precision;
  const uint32_t S32 = 0x7f7f7f7fu;
  const float qnan = std::numeric_limits<float>::quiet_NaN();
  float s32;
  memcpy(&s32, &S32, 4);
  DevBuf<float> g;
  Net net;                                              // (destroyed first: waits for its stream)
  SB_TRY(net.init(&d, device, true));
  SB_TRY(net.set_sparse(N_DENSE, n_onehot, n_cat));
  const bool tc = net.tc();
  const int np = net.nparts;
  const Layer& l0 = net.layers[0];
  const int rows_all = rows + 64;
  const size_t e0 = static_cast<size_t>(l0.w_off) + static_cast<size_t>(N_DENSE) * H, e1 = e0 + static_cast<size_t>(n_onehot) * H;
  // theta: W_e's rows; W_d's rows, b_0 and the output layer NaN, so that a gather reading outside W_e shows it.  The bf16
  // shadow parts from there, as set_params makes them.
  std::vector<float> theta(static_cast<size_t>(net.n_params), qnan);
  if (We) std::copy(We, We + (e1 - e0), theta.begin() + e0);
  else std::fill(theta.begin() + e0, theta.begin() + e1, 0.f);
  SB_CUDA(cudaMemcpy(net.theta, theta.data(), sizeof(float) * theta.size(), cudaMemcpyHostToDevice));
  SB_CUDA(cudaDeviceSynchronize());     // a pageable copy may still be landing when cudaMemcpy returns; the refresh runs
  SB_TRY(net.refresh_shadows());        // on the net's own stream
  SB_CUDA(cudaMemcpy(net.idx, idx, sizeof(int32_t) * static_cast<size_t>(rows) * n_cat, cudaMemcpyHostToDevice));
  int32_t changed = 0;
  if (!scatter) {
    // E [rows_all, ld_out]: the sentinel everywhere; the gather writes the batch rows' H columns only
    const int ldE = l0.ld_out;
    const size_t e_n = static_cast<size_t>(rows_all) * ldE;
    SB_CUDA(cudaMemset(net.E, 0x7f, sizeof(float) * e_n));
    SB_CUDA(cudaDeviceSynchronize());
    net.launches = 0;
    SB_TRY(net.enqueue_embed(rows, false, nullptr, net.stream));
    SB_CHECK(net.launches == 1, SB_ERR_STATE, "%d embedding launches", net.launches);
    SB_TRY(sync_hook(net.last_kernel));
    std::vector<uint32_t> h(e_n);
    SB_CUDA(cudaMemcpy(h.data(), net.E, sizeof(float) * e_n, cudaMemcpyDeviceToHost));
    for (int r = 0; r < rows_all; ++r)
      for (int c = 0; c < ldE; ++c) {
        const uint32_t v = h[static_cast<size_t>(r) * ldE + c];
        if (r < rows && c < H) memcpy(out + static_cast<size_t>(r) * H + c, &v, 4);
        else changed += v != S32;
      }
  } else {
    // dZ_0: the caller's rows as the step stores them (np bf16 parts, or fp32); pad columns and guard rows NaN
    if (tc) {
      SB_CUDA(cudaMemset(net.dZ[0], 0xff, sizeof(__nv_bfloat16) * static_cast<size_t>(net.A_ps[0]) * np));
      SB_TRY(upload_parts(net.dZ[0], dZ, rows, H, l0.ld_out, np, net.A_ps[0]));
    } else {
      SB_CUDA(cudaMemset(net.dZf[0], 0xff, sizeof(float) * static_cast<size_t>(rows_all) * H));
      SB_CUDA(cudaMemcpy(net.dZf[0], dZ, sizeof(float) * static_cast<size_t>(rows) * H, cudaMemcpyHostToDevice));
    }
    // the flat gradient: W_e's rows in/out, W_d's rows, b_0, the output layer and GUARD floats behind the sentinel
    const size_t g_n = static_cast<size_t>(net.n_params) + GUARD;
    std::vector<float> hg(g_n, s32);
    std::copy(out, out + (e1 - e0), hg.begin() + e0);
    SB_TRY(g.alloc(g_n));
    SB_CUDA(cudaMemcpy(g.p, hg.data(), sizeof(float) * g_n, cudaMemcpyHostToDevice));
    SB_CUDA(cudaDeviceSynchronize());
    net.launches = 0;
    SB_TRY(net.enqueue_embed(rows, true, g.p, net.stream));
    SB_CHECK(net.launches == 1, SB_ERR_STATE, "%d embedding launches", net.launches);
    SB_TRY(sync_hook(net.last_kernel));
    SB_CUDA(cudaMemcpy(hg.data(), g.p, sizeof(float) * g_n, cudaMemcpyDeviceToHost));
    for (size_t i = 0; i < g_n; ++i) {
      uint32_t u;
      memcpy(&u, &hg[i], 4);
      if ((i < e0 || i >= e1) && u != S32) ++changed;
    }
    std::copy(hg.begin() + e0, hg.begin() + e1, out);
  }
  *guard = changed;
  return SB_OK;
}

}  // extern "C"
