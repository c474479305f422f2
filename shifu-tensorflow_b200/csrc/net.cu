// Net: device state + kernel sequencing for the tabular-DNN forward / backward.
// Mirrors generate_from_modelconf + model (res/ssgd_monitor.py:91-144) as a list of fused launches.
#include <stdarg.h>
#include <stdlib.h>
#include <string.h>
#include <algorithm>
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
GemmPlan plan_gemm(int M, int N, int K, int num_sms, bool allow_split) {
  const int total_kb = (K + 63) / 64;
  auto tiles_of = [&](int bn) { return ((M + 127) / 128) * ((N + bn - 1) / bn); };
  auto plan = [&](int bn) {
    const int tiles = tiles_of(bn);
    int split = 1;
    if (allow_split) {
      split = num_sms / tiles;
      const int cap = total_kb / 8;
      if (split > cap) split = cap;
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
  SB_CHECK(d->optimizer >= SB_OPT_ADADELTA && d->optimizer <= SB_OPT_MOMENTUM, SB_ERR_INVALID, "optimizer invalid");
  return SB_OK;
}

static int check_device(int device, int* num_sms) {
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
  return SB_OK;
}

int Net::init(const sb_net_desc* d, int device_, bool training_) {
  SB_TRY(validate_desc(d));
  SB_TRY(check_device(device_, &num_sms));
  device = device_;
  training = training_;
  const bool want_trace = getenv("SB_STEP_TRACE") != nullptr;
  SB_CUDA(cudaSetDevice(device));
  // the main chain is the critical path: its CTAs are scheduled ahead of the trainer's side stream's (dW GEMMs, second
  // optimizer)
  int prio_least = 0, prio_greatest = 0;
  SB_CUDA(cudaDeviceGetStreamPriorityRange(&prio_least, &prio_greatest));
  SB_CUDA(cudaStreamCreateWithPriority(&stream, cudaStreamNonBlocking, prio_greatest));
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
  SB_TRY(dalloc(&stX, static_cast<size_t>(max_batch) * F));
  SB_TRY(dalloc(&stY, max_batch));
  SB_TRY(dalloc(&stW, max_batch));
  fill_kernel<<<(max_batch + 255) / 256, 256, 0, stream>>>(ones, 1.f, max_batch);

  if (bf) {
    Xb_ps = static_cast<long long>(max_batch) * ldF;
    SB_TRY(dalloc(&Xb, static_cast<size_t>(Xb_ps) * nparts));
    A.assign(L, nullptr); dZ.assign(L, nullptr); A_ps.assign(L, 0);
    for (int l = 0; l < L; ++l) {
      Layer& ly = layers[l];
      A_ps[l] = static_cast<long long>(max_batch) * ly.ld_out;
      SB_TRY(dalloc(&A[l], static_cast<size_t>(A_ps[l]) * nparts));
      if (training) SB_TRY(dalloc(&dZ[l], static_cast<size_t>(A_ps[l]) * nparts));
    }
  } else {
    SB_TRY(dalloc(&Xf, static_cast<size_t>(max_batch) * F));
    Af.assign(L, nullptr); dZf.assign(L, nullptr);
    for (int l = 0; l < L; ++l) {
      SB_TRY(dalloc(&Af[l], static_cast<size_t>(max_batch) * layers[l].out));
      if (training) SB_TRY(dalloc(&dZf[l], static_cast<size_t>(max_batch) * layers[l].out));
    }
  }

  // optimizer / shadow-refresh work table: runs of <= 1024 consecutive parameters
  std::vector<OptWork> wk;
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
  work_begin.assign(L + 1, 0); work_end.assign(L + 1, 0);
  for (int l = 0; l <= L; ++l) {
    Layer& ly = layers[l];
    work_begin[l] = static_cast<int>(wk.size());
    if (bf && l < L) {
      add_runs(ly.w_off, static_cast<long long>(ly.in) * ly.out, &ly);
      add_runs(ly.b_off, ly.out, nullptr);
    } else {
      add_runs(ly.w_off, static_cast<long long>(ly.in) * ly.out + ly.out, nullptr);
    }
    work_end[l] = static_cast<int>(wk.size());
  }
  n_work = static_cast<int>(wk.size());
  SB_TRY(dalloc(&work, wk.size()));
  SB_CUDA(cudaMemcpyAsync(work, wk.data(), wk.size() * sizeof(OptWork), cudaMemcpyHostToDevice, stream));
  SB_CUDA(cudaStreamSynchronize(stream));

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
    cudaFuncSetAttribute(out_layer_kernel<__nv_bfloat16>, cudaFuncAttributePreferredSharedMemoryCarveout, co);
  }
  return SB_OK;
}

void Net::destroy() {
  if (stream) cudaStreamSynchronize(stream);
  for (void* p : allocs) cudaFree(p);
  allocs.clear();
  if (stream) cudaStreamDestroy(stream);
  stream = nullptr;
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

int Net::refresh_shadows() {
  if (!tc()) return SB_OK;
  shadow_refresh_kernel<<<n_work, 256, 0, stream>>>(work, theta);
  SB_CUDA(cudaGetLastError());
  return SB_OK;
}

int Net::enqueue_load(const StepIn& in, int rows, float* clear, long long clear_n) {
  const int Fx = in.sparse ? n_dense : F;        // a sparse step stages only the dense block
  const int ldx = in.sparse ? ldD : ldF;
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
  mark("load_batch");
  if (in.sparse) SB_TRY(enqueue_embed(rows, false, nullptr, stream));
  return SB_OK;
}

int Net::enqueue_hidden_forward(const StepIn& in, int rows, float* grad, bool* fused_out, float4* clear, long long clear_n4) {
  if (fused_out) *fused_out = false;
  for (int l = 0; l < L; ++l) {
    Layer& ly = layers[l];
    const bool sp0 = (l == 0) && in.sparse;       // wide+deep: contract the dense columns only, add the embedding sums
    const int k_in = sp0 ? n_dense : ly.in;
    const int ld_k = sp0 ? ldD : ly.ld_in;
    if (tc()) {
      // Z = A_{l-1}[rows,in] (K-major) x W_l[in,out] (MN-major B operand: n contiguous)
      TmapSet tm;
      const bool res0 = (l == 0) && in.resident;
      const __nv_bfloat16* src = (l == 0) ? (res0 ? resident_Xb : Xb) : A[l - 1];
      const long long src_ps = (l == 0) ? (res0 ? resident_ps : Xb_ps) : A_ps[l - 1];
      const int src_rows = res0 ? static_cast<int>(resident_rows) : rows;
      SB_TRY(make_tmaps_bf16(tm.b, ly.Wn, Wn_ps[l], nparts, k_in, ly.out, ly.ld_out, 64));
      GemmTcParams p = {};
      set_part_pairs(&p, nparts);
      p.M = rows; p.N = ly.out; p.K = k_in;
      if (sp0) { p.addend = E; p.ld_add = ly.ld_out; }
      p.bias = theta + ly.b_off; p.act = ly.act;
      p.out = A[l]; p.ld_out = ly.ld_out; p.out_ps = A_ps[l];
      p.a_rows = res0 ? in.desc : nullptr;
      if (l == L - 1 && grad != nullptr && training && ly.out <= FWD_OUT_MAX_N && p.addend == nullptr) {
        // K2 + K3 + K4 + output backward in one kernel (gemm_fwd_out.cuh): 64-row tiles of whole rows of A_L
        FwdOutTmaps ft;
        SB_TRY(make_tmaps_bf16(ft.a, src, src_ps, nparts, src_rows, k_in, ld_k, 64));
        for (int i = 0; i < 3; ++i) ft.b[i] = tm.b[i];
        SB_TRY(make_tmaps_bf16(ft.o, dZ[l], A_ps[l], nparts, rows, ly.out, ly.ld_out, 64));
        const int tiles = (rows + 63) / 64;
        const int grid = tiles < num_sms ? tiles : num_sms;
        Layer& ol = layers[L];
        p.wo = theta + ol.w_off; p.bo = theta + ol.b_off;
        p.desc = in.desc; p.scal = in.scal; p.loss = loss;
        p.g_wo = grad + ol.w_off; p.g_bo = grad + ol.b_off; p.g_bL = grad + ly.b_off;
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
        SB_TRY(make_tmap_bf16(&pt.a, src, src_rows, k_in, ld_k, pp.bm_wg));
        pt.b = tm.b[0];
        SB_TRY(make_tmap_bf16(&pt.o, A[l], rows, ly.out, ly.ld_out, pp.bm_wg));
        if (pp.bn == 256) SB_TRY(launch_gemm_wide(pp, pt, p, stream, true));
        else SB_TRY(launch_gemm_pp<EPI_FWD>(pp, pt, p, stream, true));
      } else {
        const GemmPlan pl = plan_gemm(rows, ly.out, round_up(k_in, 64) * pairs_of(nparts), num_sms, false);
        SB_TRY(make_tmaps_bf16(tm.a, src, src_ps, nparts, src_rows, k_in, ld_k, 128));
        SB_TRY((launch_gemm_tc<EPI_FWD, false, true>(pl, tm, p, stream, true)));
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
    }
    mark("gemm_fwd");
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
  const int grid = (rows + 31) / 32;
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
      if (hl.out <= 256) SB_TRY(launch_kernel(out_layer_rows_kernel<1>, g, dim3(256), 0, stream, true, p, rpb));
      else if (hl.out <= 512) SB_TRY(launch_kernel(out_layer_rows_kernel<2>, g, dim3(256), 0, stream, true, p, rpb));
      else SB_TRY(launch_kernel(out_layer_rows_kernel<4>, g, dim3(256), 0, stream, true, p, rpb));
    } else {
      SB_TRY(launch_kernel(out_layer_kernel<__nv_bfloat16>, dim3(grid), dim3(256), 0, stream, true, p));
    }
  } else {
    p.A = Af[L - 1]; p.ldA = hl.out;
    if (do_bwd) { p.dZ = dZf[L - 1]; p.ld_dZ = hl.out; }
    SB_TRY(launch_kernel(out_layer_kernel<float>, dim3(grid), dim3(256), 0, stream, true, p));
  }
  SB_CUDA(cudaGetLastError());
  mark("out_layer");
  return SB_OK;
}

int Net::enqueue_dw(const StepIn& in, int l, int rows, float* grad, cudaStream_t st, bool pdl, int sms, int r0, int r1, int chunk) {
  Layer& ly = layers[l];
  const bool sp0 = (l == 0) && in.sparse;         // wide+deep: dW of the dense rows by GEMM, of the embedding rows by scatter-add
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
    SB_TRY(launch_gemm_f32<EPI_DW>(p, split, st));
    mark("gemm_dw");
    return SB_OK;
  }
  // dW_l[in,out] += sum_rows A_{l-1}[rows,in] (MN-major A) * dZ_l[rows,out] (MN-major B), split-K over rows
  const bool res0 = (l == 0) && in.resident;
  const int ld_k = sp0 ? ldD : ly.ld_in;
  const __nv_bfloat16* ap = (l == 0) ? (res0 ? resident_Xb : Xb) : A[l - 1];
  const long long ap_ps = (l == 0) ? (res0 ? resident_ps : Xb_ps) : A_ps[l - 1];
  const GemmPlan pl = plan_gemm(r1 - r0, ly.out, round_up(rows, 64) * pairs_of(nparts), sms, true);
  TmapSet tm;
  // resident set: rows past the batch end are real rows of other batches; the B operand (dZ_l, extent = rows) is
  // zero-filled there, so they contribute nothing
  SB_TRY(make_tmaps_bf16(tm.a, ap + r0, ap_ps, nparts, res0 ? static_cast<int>(resident_rows) : rows, r1 - r0, ld_k, 64));
  SB_TRY(make_tmaps_bf16(tm.b, dZ[l], A_ps[l], nparts, rows, ly.out, ly.ld_out, 64));
  GemmTcParams p = {};
  set_part_pairs(&p, nparts);
  p.M = r1 - r0; p.N = ly.out; p.K = rows;
  p.a_rows = res0 ? in.desc : nullptr;
  p.accum = grad + ly.w_off + static_cast<long long>(r0) * ly.out; p.ld_acc = ly.out;
  p.acc_vec4 = (ly.out % 4 == 0 && ly.w_off % 4 == 0) ? 1 : 0;
  p.trace = next_trace("dW", l, r1 - r0, ly.out, rows, chunk);
  if (pl.bn == 256) SB_TRY(launch_gemm_dw(pl, tm, p, st, pdl));
  else SB_TRY((launch_gemm_tc<EPI_DW, true, true>(pl, tm, p, st, pdl)));
  mark("gemm_dw");
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
    SB_TRY(launch_gemm_f32<EPI_DA>(p, 1, stream));
    mark("gemm_da");
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
  if (nparts == 1) {                           // plain bf16: the ping-pong kernel
    const PpPlan pp = plan_gemm_pp(rows, ly.in, ly.out, num_sms, false);
    PpTmaps pt;
    SB_TRY(make_tmap_bf16(&pt.a, dZ[l], rows, ly.out, ly.ld_out, pp.bm_wg));
    SB_TRY(make_tmap_bf16(&pt.b, ly.Wn, ly.in, ly.out, ly.ld_out, pp.bn));
    SB_TRY(make_tmap_bf16(&pt.o, dZ[l - 1], rows, ly.in, pl.ld_out, pp.bm_wg));
    SB_TRY(make_tmap_bf16(&pt.x, A[l - 1], rows, ly.in, pl.ld_out, pp.bm_wg));
    SB_TRY(launch_gemm_pp<EPI_DA>(pp, pt, p, stream, true));
  } else {
    const GemmPlan gp = plan_gemm(rows, ly.in, round_up(ly.out, 64) * pairs_of(nparts), num_sms, false);
    TmapSet tm;
    SB_TRY(make_tmaps_bf16(tm.a, dZ[l], A_ps[l], nparts, rows, ly.out, ly.ld_out, 128));
    SB_TRY(make_tmaps_bf16(tm.b, ly.Wn, Wn_ps[l], nparts, ly.in, ly.out, ly.ld_out, gp.bn));
    SB_TRY((launch_gemm_tc<EPI_DA, false, false>(gp, tm, p, stream, true)));
  }
  mark("gemm_da");
  return SB_OK;
}
}  // namespace sb
