// HBM-bound kernels of the step: mini-batch load/cast/transpose (K1), output layer + loss + its
// backward (K3/K4), fused multi-tensor optimizer (K7), gradient accumulation.
#pragma once
#include "common.cuh"
#include "ptx.cuh"

namespace sb {

// Where the current mini-batch lives (HBM-resident training set or the H2D staging area).
// Written by set_batch_kernel right before the captured step graph runs, so the graph itself
// never changes (res/ssgd_monitor.py:272-276 builds the same feed_dict from x_batch[i]).
struct BatchDesc {
  const float* X;  // [rows, F] row-major fp32
  const float* y;  // [rows]
  const float* w;  // [rows]
  float lr_t;      // Adam: lr * sqrt(1-b2^t)/(1-b1^t); others: lr
  float gscale;    // 1/world (and 1/n_accumulated for the epoch-sync schedule)
  unsigned int epoch;  // exchange round (flag value of the peer-memory all-reduce)
  int row0;            // first row of the batch inside the bf16 HBM-resident set (TMA row-coordinate offset)
  float2* hist;        // nullable: slot of this step in the pinned-host loss history (loss sum, n_nz), written by the step's tail
  const int* order;    // ordered resident steps (gather_batch_kernel): the batch's slice of the row order, row r = order[r]
};

// nz_prefix != nullptr (bf16 resident set): the batch is consumed by TMA straight from the resident set, there is no
// load kernel, so this kernel also publishes n_nz = #{w != 0 in the batch} from the prefix counts built at load time
// and clears the loss accumulator.
static __global__ void set_batch_kernel(BatchDesc* d, const float* X, const float* y, const float* w, float lr_t, float gscale,
                                        unsigned int epoch = 0, int row0 = 0, const int* nz_prefix = nullptr, int rows = 0,
                                        float* scal = nullptr, float2* hist = nullptr, const int* order = nullptr) {
  d->X = X; d->y = y; d->w = w; d->lr_t = lr_t; d->gscale = gscale; d->epoch = epoch; d->row0 = row0; d->hist = hist;
  d->order = order;
  if (nz_prefix != nullptr) {
    scal[1] = static_cast<float>(nz_prefix[row0 + rows] - nz_prefix[row0]);  // SCAL_NNZ
    scal[0] = 0.f;                                                           // SCAL_LOSS_SUM
  }
}

// Split-precision modes: the value whose bf16 rounding is part `part` of x (part 0: x itself; part k: x minus the first k
// parts).  x = bf16(r_0) + bf16(r_1) + ... with r_0 = x, r_{k+1} = r_k - bf16(r_k).
__device__ __forceinline__ float bf16_residual(float x, int part) {
  for (int i = 0; i < part; ++i) x -= __bfloat162float(__float2bfloat16_rn(x));
  return x;
}

// step scalars (device): [0] = sum_i w_i * per-row loss, [1] = n_nz (count of non-zero weights)
enum { SCAL_LOSS_SUM = 0, SCAL_NNZ = 1, SCAL_COUNT = 4 };

// ------------------------------------------------------------------------------------------------
// K1 mini-batch load.  fp32 rows of the current batch -> the operand buffer of the layer-0 GEMMs:
// (bf16 mode) row-major bf16 [rows, ldF] - the SAME buffer feeds the forward GEMM (K-major) and the dW
// GEMM (MN-major), so no transposed copy exists; (fp32 mode) fp32 copy into the batch buffer.
// HBM-bound: each thread moves 8 consecutive columns (2 x 16 B loads -> one 16 B store).
// Block 0 additionally counts the non-zero sample weights of the batch (n_nz of
// SUM_BY_NONZERO_WEIGHTS, res/ssgd_monitor.py:129).
// ------------------------------------------------------------------------------------------------
template <bool BF16>
__global__ void __launch_bounds__(256)
load_batch_kernel(const BatchDesc* __restrict__ desc, int rows, int F, __nv_bfloat16* __restrict__ Xb, int ldF,
                  float* __restrict__ Xf, float* __restrict__ scal, float* __restrict__ zero_buf, long long zero_n,
                  int np = 1, long long part_stride = 0) {
  pdl_wait();
  pdl_launch_dependents();
  // the step's gradient buffer is accumulated with atomics: clear it here (replaces a memset node in the graph)
  for (long long i = blockIdx.x * 256ll + threadIdx.x; i < zero_n; i += gridDim.x * 256ll) zero_buf[i] = 0.f;
  const float* __restrict__ X = desc->X;
  const int groups = ldF >> 3;  // 8-column groups per row (ldF is a multiple of 8)
  const long long total = static_cast<long long>(rows) * groups;
  const bool vec = ((F & 7) == 0) && ((reinterpret_cast<uintptr_t>(X) & 15) == 0);
  for (long long u = blockIdx.x * 256ll + threadIdx.x; u < total; u += gridDim.x * 256ll) {
    const int r = static_cast<int>(u / groups), c = static_cast<int>(u % groups) * 8;
    float v[8];
    if (vec) {
      const float4 a = __ldg(reinterpret_cast<const float4*>(X + static_cast<size_t>(r) * F + c));
      const float4 b = __ldg(reinterpret_cast<const float4*>(X + static_cast<size_t>(r) * F + c + 4));
      v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
    } else {
#pragma unroll
      for (int j = 0; j < 8; ++j) v[j] = (c + j < F) ? __ldg(X + static_cast<size_t>(r) * F + c + j) : 0.f;
    }
    if constexpr (BF16) {
      for (int part = 0; part < np; ++part) {      // np > 1: split-precision parts (bf16_residual)
        uint4 o;
        o.x = pack_bf16x2(bf16_residual(v[0], part), bf16_residual(v[1], part));
        o.y = pack_bf16x2(bf16_residual(v[2], part), bf16_residual(v[3], part));
        o.z = pack_bf16x2(bf16_residual(v[4], part), bf16_residual(v[5], part));
        o.w = pack_bf16x2(bf16_residual(v[6], part), bf16_residual(v[7], part));
        *reinterpret_cast<uint4*>(Xb + part * part_stride + static_cast<size_t>(r) * ldF + c) = o;
      }
    } else {
      if (vec) {
        *reinterpret_cast<float4*>(Xf + static_cast<size_t>(r) * F + c) = make_float4(v[0], v[1], v[2], v[3]);
        *reinterpret_cast<float4*>(Xf + static_cast<size_t>(r) * F + c + 4) = make_float4(v[4], v[5], v[6], v[7]);
      } else {
#pragma unroll
        for (int j = 0; j < 8; ++j)
          if (c + j < F) Xf[static_cast<size_t>(r) * F + c + j] = v[j];
      }
    }
  }
  if (blockIdx.x == 0) {
    const float* __restrict__ w = desc->w;
    float cnt = 0.f;
    for (int i = threadIdx.x; i < rows; i += 256) cnt += (__ldg(w + i) != 0.f) ? 1.f : 0.f;
    cnt = warp_sum(cnt);
    __shared__ float part[8];
    if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = cnt;
    __syncthreads();
    if (threadIdx.x == 0) {
      float t = 0.f;
      for (int i = 0; i < 8; ++i) t += part[i];
      scal[SCAL_NNZ] = t;
      scal[SCAL_LOSS_SUM] = 0.f;
    }
  }
}

// ------------------------------------------------------------------------------------------------
// K3+K4 (+ output-layer backward): y_hat = sigmoid(A_L w_o + b_o); loss = sum w (y_hat-y)^2 / n_nz
// (res/ssgd_monitor.py:121,129) or the sigmoid-CE variant; d z_hat; then the rank-1 backward
//   dZ_L[r,j] = dz_r * w_o[j] * act'(A_L[r,j])     (row-major, bf16 or fp32)
//   dw_o[j] += sum_r dz_r A_L[r,j],  db_o += sum_r dz_r,  db_L[j] += sum_r dZ_L[r,j]
// out = 1 is GEMV-class: CUDA cores, one pass over A_L.  Each block owns 32 rows.
// ------------------------------------------------------------------------------------------------
struct OutLayerParams {
  int rows, H, ldA;          // A_L is [rows, ldA] with H valid columns
  const void* A;             // bf16 or fp32
  const float* wo;           // [H]
  const float* bo;           // [1]
  const BatchDesc* desc;     // y, w
  float* scal;               // SCAL_*
  int loss, act;             // sb_loss, activation of hidden layer L
  int do_bwd;                // 0: forward (+loss) only
  int do_loss;               // 0: scores only (no y / w access)
  float* yhat;               // nullable [rows]
  void* dZ; int ld_dZ;       // [rows, ld_dZ] bf16 or fp32
  float* g_wo; float* g_bo; float* g_bL;  // gradient slots (atomic accumulate)
  unsigned long long* trace;              // debug timeline (nullable): [0] entry, [2] deps resolved (block 0), [10] last exit
  int np;                                 // bf16 parts per value of A / dZ (split-precision modes; 0 or 1 = plain)
  long long a_ps, dz_ps;                  // element stride between parts
  float* det_ws;                          // DET instantiations only (common.cuh, det_last_cta): slots and ticket
  unsigned int* det_ticket;
};

// in-graph kernel span for the step timeline: begin = block 0's stamp after griddepcontrol.wait, end = atomicMax over blocks
__device__ __forceinline__ void trace_begin(unsigned long long* trace, bool entry) {
  if (trace != nullptr && blockIdx.x == 0 && threadIdx.x == 0) trace[entry ? 0 : 2] = globaltimer_ns();
}
__device__ __forceinline__ void trace_end(unsigned long long* trace) {
  if (trace != nullptr && threadIdx.x == 0) atomicMax(trace + 10, static_cast<unsigned long long>(globaltimer_ns()));
}

// ------------------------------------------------------------------------------------------------
// Ordered resident steps (sb_trainer_set_row_order): the first kernel of the step, in load_batch_kernel's place and with
// its duties (clear the gradient buffer, publish n_nz and the cleared loss sum).  Row r of the batch is row
// desc->order[r] of the resident set.  Tensor-core modes copy that row's np bf16 parts, pad columns included, into Xb as
// they are, so Xb holds what load_batch_kernel writes for the same rows; fp32 mode copies the fp32 row into Xf.  y and w
// are gathered into the batch buffers the descriptor points the loss at.  HBM-bound: 16-byte vectors; block 0 counts the
// non-zero weights in load_batch_kernel's order.
// ------------------------------------------------------------------------------------------------
struct GatherParams {
  const BatchDesc* desc;
  int rows, F, ldF, np;
  const __nv_bfloat16* src_b; long long src_ps;   // tensor-core modes: the resident set [n, ldF], np parts src_ps apart
  __nv_bfloat16* Xb; long long Xb_ps;             // -> [rows, ldF] parts
  const float* src_f; float* Xf;                  // fp32 mode: the resident set [n, F] -> [rows, F]
  const float* src_y; const float* src_w;         // labels / weights of the resident set [n]
  float* y; float* w;                             // -> [rows]
  float* scal;
  float* zero_buf; long long zero_n;
  unsigned long long* trace;
};

template <bool BF16>
__global__ void __launch_bounds__(256)
gather_batch_kernel(const GatherParams p) {
  trace_begin(p.trace, true);
  pdl_wait();
  pdl_launch_dependents();
  trace_begin(p.trace, false);
  const long long stride = gridDim.x * 256ll, tid0 = blockIdx.x * 256ll + threadIdx.x;
  for (long long i = tid0; i < p.zero_n; i += stride) p.zero_buf[i] = 0.f;
  const int* __restrict__ order = p.desc->order;
  if constexpr (BF16) {
    const int groups = p.ldF >> 3;   // 8-element vectors per row (ldF is a multiple of 8)
    const long long total = static_cast<long long>(p.rows) * groups;
    for (long long u = tid0; u < total; u += stride) {
      const int r = static_cast<int>(u / groups), c = static_cast<int>(u % groups) * 8;
      const size_t s = static_cast<size_t>(__ldg(order + r)) * p.ldF + c, d = static_cast<size_t>(r) * p.ldF + c;
      for (int part = 0; part < p.np; ++part)
        *reinterpret_cast<uint4*>(p.Xb + part * p.Xb_ps + d) = __ldg(reinterpret_cast<const uint4*>(p.src_b + part * p.src_ps + s));
    }
  } else {
    const bool vec = ((p.F & 3) == 0) && ((reinterpret_cast<uintptr_t>(p.src_f) & 15) == 0);
    const int groups = vec ? (p.F >> 2) : p.F;   // 4-float vectors (or single floats) per row
    const long long total = static_cast<long long>(p.rows) * groups;
    for (long long u = tid0; u < total; u += stride) {
      const int r = static_cast<int>(u / groups), c = static_cast<int>(u % groups);
      const size_t s = static_cast<size_t>(__ldg(order + r)) * p.F, d = static_cast<size_t>(r) * p.F;
      if (vec) reinterpret_cast<float4*>(p.Xf + d)[c] = __ldg(reinterpret_cast<const float4*>(p.src_f + s) + c);
      else p.Xf[d + c] = __ldg(p.src_f + s + c);
    }
  }
  for (long long r = tid0; r < p.rows; r += stride) {
    const int s = __ldg(order + r);
    p.y[r] = __ldg(p.src_y + s);
    p.w[r] = __ldg(p.src_w + s);
  }
  if (blockIdx.x == 0) {
    float cnt = 0.f;
    for (int i = threadIdx.x; i < p.rows; i += 256) cnt += (__ldg(p.src_w + __ldg(order + i)) != 0.f) ? 1.f : 0.f;
    cnt = warp_sum(cnt);
    __shared__ float part[8];
    if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = cnt;
    __syncthreads();
    if (threadIdx.x == 0) {
      float t = 0.f;
      for (int i = 0; i < 8; ++i) t += part[i];
      p.scal[SCAL_NNZ] = t;
      p.scal[SCAL_LOSS_SUM] = 0.f;
    }
  }
  trace_end(p.trace);
}

template <typename T> __device__ __forceinline__ float ld_as_float(const T* p);
template <> __device__ __forceinline__ float ld_as_float<float>(const float* p) { return __ldg(p); }
template <> __device__ __forceinline__ float ld_as_float<__nv_bfloat16>(const __nv_bfloat16* p) { return __bfloat162float(*p); }
template <typename T> __device__ __forceinline__ void st_from_float(T* p, float v);
template <> __device__ __forceinline__ void st_from_float<float>(float* p, float v) { *p = v; }
template <> __device__ __forceinline__ void st_from_float<__nv_bfloat16>(__nv_bfloat16* p, float v) { *p = __float2bfloat16_rn(v); }

// DET: the per-block loss sum, db_o and the two row halves' dw_o / db_L go to the block's slots (det_out_finish, halves = 2)
template <typename T, bool DET = false>
__global__ void __launch_bounds__(256)
out_layer_kernel(const OutLayerParams p) {
  trace_begin(p.trace, true);
  pdl_wait();
  pdl_launch_dependents();
  trace_begin(p.trace, false);
  __shared__ float dz_row[32];
  __shared__ float blk_red[8];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int r0 = blockIdx.x * 32;
  const T* __restrict__ A = reinterpret_cast<const T*>(p.A);
  const float bo = __ldg(p.bo);
  const float nnz = p.do_loss ? p.scal[SCAL_NNZ] : 1.f;
  const float inv_nnz = nnz > 0.f ? 1.f / nnz : 0.f;

  // ---- phase 1: one warp per row (4 rows per warp) ----
  float loss_part = 0.f;
  for (int i = 0; i < 4; ++i) {
    const int rl = warp * 4 + i, r = r0 + rl;
    float z = 0.f;
    if (r < p.rows) {
      const T* ar = A + static_cast<size_t>(r) * p.ldA;
      for (int j = lane; j < p.H; j += 32) {
        float a = ld_as_float<T>(ar + j);
        for (int part = 1; part < p.np; ++part) a += ld_as_float<T>(ar + part * p.a_ps + j);
        z = fmaf(a, __ldg(p.wo + j), z);
      }
    }
    z = warp_sum(z) + bo;
    if (lane == 0) {
      float dz = 0.f;
      if (r < p.rows) {
        const float yh = sigmoidf_stable(z);
        if (p.yhat) p.yhat[r] = yh;
        if (p.do_loss) {
          const float y = __ldg(p.desc->y + r), w = __ldg(p.desc->w + r);
          if (p.loss == SB_LOSS_MSE) {
            const float d = yh - y;
            loss_part += w * d * d;
            dz = 2.f * w * d * yh * (1.f - yh) * inv_nnz;
          } else {
            loss_part += w * (fmaxf(z, 0.f) - z * y + log1pf(expf(-fabsf(z))));
            dz = w * (yh - y) * inv_nnz;
          }
        }
      }
      dz_row[rl] = dz;
    }
  }
  if (p.do_loss) {
    if (lane == 0) blk_red[warp] = loss_part;
    __syncthreads();
    if (tid == 0) {
      float s = 0.f;
      for (int i = 0; i < 8; ++i) s += blk_red[i];
      if constexpr (DET) p.det_ws[blockIdx.x * det_out_stride(p.H, 2)] = s;
      else atomicAdd(p.scal + SCAL_LOSS_SUM, s);
    }
  }
  float* const slots = DET ? p.det_ws + blockIdx.x * det_out_stride(p.H, 2) : nullptr;
  auto det_finish = [&]() {
    if (det_last_cta(p.det_ticket, gridDim.x, 0, 256, tid == 0))
      det_out_finish(p.det_ws, static_cast<int>(gridDim.x), p.H, 2, p.do_loss != 0, p.do_bwd != 0, p.scal + SCAL_LOSS_SUM, p.g_bo,
                     p.g_bL, p.g_wo, tid, 256);
  };
  if (!p.do_bwd) {
    if constexpr (DET) det_finish();
    trace_end(p.trace);
    return;
  }
  __syncthreads();

  // ---- phase 2: rank-1 backward over column chunks of 128 ----
  float dbo = 0.f;
  if (tid < 32) {
    dbo = warp_sum(dz_row[tid]);
    if (tid == 0) {
      if constexpr (DET) slots[1] = dbo;
      else atomicAdd(p.g_bo, dbo);
    }
  }
  T* __restrict__ dZ = reinterpret_cast<T*>(p.dZ);
  for (int c0 = 0; c0 < p.H; c0 += 128) {
    const int cl = tid & 127, j = c0 + cl;  // column handled by this thread
    const int rh = tid >> 7;                // row half: rows rh*16 .. rh*16+15
    float s_dw = 0.f, s_db = 0.f;
    const float woj = (j < p.H) ? __ldg(p.wo + j) : 0.f;
    for (int i = 0; i < 16; ++i) {
      const int rl = rh * 16 + i, r = r0 + rl;
      float g = 0.f;
      if (r < p.rows && j < p.H) {
        float a = ld_as_float<T>(A + static_cast<size_t>(r) * p.ldA + j);
        for (int part = 1; part < p.np; ++part) a += ld_as_float<T>(A + part * p.a_ps + static_cast<size_t>(r) * p.ldA + j);
        const float dz = dz_row[rl];
        g = dz * woj * act_grad_from_out(a, p.act);
        s_dw = fmaf(dz, a, s_dw);
        s_db += g;
        st_from_float<T>(dZ + static_cast<size_t>(r) * p.ld_dZ + j, g);
        for (int part = 1; part < p.np; ++part)
          st_from_float<T>(dZ + part * p.dz_ps + static_cast<size_t>(r) * p.ld_dZ + j, bf16_residual(g, part));
      }
    }
    if (j < p.H) {
      if constexpr (DET) {
        slots[2 + rh * p.H + j] = s_db;
        slots[2 + (2 + rh) * p.H + j] = s_dw;
      } else {
        atomicAdd(p.g_wo + j, s_dw);
        atomicAdd(p.g_bL + j, s_db);
      }
    }
  }
  if constexpr (DET) det_finish();
  trace_end(p.trace);
}

// bf16 variant of the kernel above for H <= 256 * NCH: ONE pass over A_L.  A warp owns whole rows (rows w, w+8, ... of
// the block's slice); lane i owns columns [256 c + 8 i, +8) of every 256-column chunk c of every row, moved with 16-byte
// loads / stores.  Because the lane <-> column mapping is the same for every row, the row's dot product is one xor-shuffle
// reduction and the dw_o / db_L column sums stay in registers over all rows of the warp; a block reduces them through
// shared memory and issues ONE atomic per column (the 32-rows-per-block kernel above reads A_L twice with 2-byte
// accesses).
// DET: the block's sums go to its slots (det_out_finish, halves = 1) instead of one atomic per column
template <int NCH, bool DET = false>
__global__ void __launch_bounds__(256)
out_layer_rows_kernel(const OutLayerParams p, int rows_per_block) {
  trace_begin(p.trace, true);
  pdl_wait();
  pdl_launch_dependents();
  trace_begin(p.trace, false);
  __shared__ float red[2][8][256];
  __shared__ float red_s[2][8];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const __nv_bfloat16* __restrict__ A = reinterpret_cast<const __nv_bfloat16*>(p.A);
  __nv_bfloat16* __restrict__ dZ = reinterpret_cast<__nv_bfloat16*>(p.dZ);
  const float bo = __ldg(p.bo);
  const float nnz = p.do_loss ? p.scal[SCAL_NNZ] : 1.f;
  const float inv_nnz = nnz > 0.f ? 1.f / nnz : 0.f;
  float wo[NCH][8], s_dw[NCH][8], s_db[NCH][8];
#pragma unroll
  for (int c = 0; c < NCH; ++c)
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      const int j = c * 256 + lane * 8 + k;
      wo[c][k] = (j < p.H) ? __ldg(p.wo + j) : 0.f;
      s_dw[c][k] = 0.f; s_db[c][k] = 0.f;
    }
  float loss_part = 0.f, dz_sum = 0.f;
  const int r_begin = blockIdx.x * rows_per_block;
  const int r_end = min(p.rows, r_begin + rows_per_block);
  for (int r = r_begin + warp; r < r_end; r += 8) {
    float a[NCH][8];
    float z = 0.f;
#pragma unroll
    for (int c = 0; c < NCH; ++c) {
      const int col0 = c * 256 + lane * 8;
      uint4 raw = make_uint4(0, 0, 0, 0);
      if (col0 < p.ldA && col0 < p.H) raw = *reinterpret_cast<const uint4*>(A + static_cast<size_t>(r) * p.ldA + col0);
#pragma unroll
      for (int k = 0; k < 8; ++k) {   // pad columns of A_L hold act(0), not 0
        if constexpr (DET) a[c][k] = (col0 + k < p.H) ? bf16_of_u4(raw, k) : 0.f;   // no byte view of raw: registers only
        else a[c][k] = (col0 + k < p.H) ? __bfloat162float(reinterpret_cast<const __nv_bfloat16*>(&raw)[k]) : 0.f;
      }
      for (int part = 1; part < p.np; ++part) {       // split-precision modes: add the lower parts
        uint4 lo = make_uint4(0, 0, 0, 0);
        if (col0 < p.ldA && col0 < p.H) lo = *reinterpret_cast<const uint4*>(A + part * p.a_ps + static_cast<size_t>(r) * p.ldA + col0);
#pragma unroll
        for (int k = 0; k < 8; ++k) {
          if constexpr (DET) a[c][k] += (col0 + k < p.H) ? bf16_of_u4(lo, k) : 0.f;
          else a[c][k] += (col0 + k < p.H) ? __bfloat162float(reinterpret_cast<const __nv_bfloat16*>(&lo)[k]) : 0.f;
        }
      }
#pragma unroll
      for (int k = 0; k < 8; ++k) z = fmaf(a[c][k], wo[c][k], z);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) z += __shfl_xor_sync(0xffffffffu, z, o);
    z += bo;
    const float yh = sigmoidf_stable(z);
    if (p.yhat && lane == 0) p.yhat[r] = yh;
    float dz = 0.f;
    if (p.do_loss) {
      const float y = __ldg(p.desc->y + r), w = __ldg(p.desc->w + r);
      if (p.loss == SB_LOSS_MSE) {
        const float d = yh - y;
        loss_part += w * d * d;
        dz = 2.f * w * d * yh * (1.f - yh) * inv_nnz;
      } else {
        loss_part += w * (fmaxf(z, 0.f) - z * y + log1pf(expf(-fabsf(z))));
        dz = w * (yh - y) * inv_nnz;
      }
    }
    if (p.do_bwd) {
      dz_sum += dz;
#pragma unroll
      for (int c = 0; c < NCH; ++c) {
        const int col0 = c * 256 + lane * 8;
        float g[8];
#pragma unroll
        for (int k = 0; k < 8; ++k) {
          g[k] = dz * wo[c][k] * act_grad_from_out(a[c][k], p.act);   // wo = 0 beyond H -> g = 0 in pad columns
          s_db[c][k] += g[k];
          s_dw[c][k] = fmaf(dz, a[c][k], s_dw[c][k]);
        }
        if (col0 < p.ld_dZ && col0 < p.H) {
          const int np = p.np > 1 ? p.np : 1;
          for (int part = 0; part < np; ++part) {
            uint4 o;
            o.x = pack_bf16x2(bf16_residual(g[0], part), bf16_residual(g[1], part));
            o.y = pack_bf16x2(bf16_residual(g[2], part), bf16_residual(g[3], part));
            o.z = pack_bf16x2(bf16_residual(g[4], part), bf16_residual(g[5], part));
            o.w = pack_bf16x2(bf16_residual(g[6], part), bf16_residual(g[7], part));
            *reinterpret_cast<uint4*>(dZ + part * p.dz_ps + static_cast<size_t>(r) * p.ld_dZ + col0) = o;
          }
        }
      }
    }
  }
  // block reduction: scalars first, then one 256-column chunk at a time
  if (lane == 0) { red_s[0][warp] = loss_part; red_s[1][warp] = dz_sum; }
  __syncthreads();
  if (tid == 0) {
    float l = 0.f, d = 0.f;
    for (int i = 0; i < 8; ++i) { l += red_s[0][i]; d += red_s[1][i]; }
    if constexpr (DET) {
      float* slots = p.det_ws + blockIdx.x * det_out_stride(p.H, 1);
      slots[0] = l;
      slots[1] = d;
    } else {
      if (p.do_loss) atomicAdd(p.scal + SCAL_LOSS_SUM, l);
      if (p.do_bwd) atomicAdd(p.g_bo, d);
    }
  }
  auto det_finish = [&]() {
    if (det_last_cta(p.det_ticket, gridDim.x, 0, 256, tid == 0))
      det_out_finish(p.det_ws, static_cast<int>(gridDim.x), p.H, 1, p.do_loss != 0, p.do_bwd != 0, p.scal + SCAL_LOSS_SUM, p.g_bo,
                     p.g_bL, p.g_wo, tid, 256);
  };
  if (!p.do_bwd) {
    if constexpr (DET) det_finish();
    trace_end(p.trace);
    return;
  }
#pragma unroll
  for (int c = 0; c < NCH; ++c) {
    if (c * 256 >= p.H) break;
    __syncthreads();
#pragma unroll
    for (int k = 0; k < 8; ++k) { red[0][warp][lane * 8 + k] = s_dw[c][k]; red[1][warp][lane * 8 + k] = s_db[c][k]; }
    __syncthreads();
    const int j = c * 256 + tid;
    if (j < p.H) {
      float dw = 0.f, db = 0.f;
#pragma unroll
      for (int i = 0; i < 8; ++i) { dw += red[0][i][tid]; db += red[1][i][tid]; }
      if constexpr (DET) {
        float* slots = p.det_ws + blockIdx.x * det_out_stride(p.H, 1);
        slots[2 + j] = db;
        slots[2 + p.H + j] = dw;
      } else {
        atomicAdd(p.g_wo + j, dw);
        atomicAdd(p.g_bL + j, db);
      }
    }
  }
  if constexpr (DET) det_finish();
  trace_end(p.trace);
}

// ------------------------------------------------------------------------------------------------
// K7 fused multi-tensor optimizer over the flat parameter vector (TF 1.x kernel forms: ApplyAdadelta
// res/ssgd_monitor.py:138, ApplyAdam res/ssgd.py:57, ApplyGradientDescent res/ssgd_monitor_bk.py:81,
// ApplyMomentum, ApplyAdagrad, ApplyRMSProp, ApplyFtrl; and iRPROP- as torch.optim.Rprop computes it).  Reads the
// (all-reduced) gradient once, updates fp32 master weights + state, and in bf16 mode refreshes the bf16 shadow of every
// hidden-layer weight matrix in the same pass.
// ------------------------------------------------------------------------------------------------
struct OptHyper {
  int kind;
  float rho, eps, beta1, beta2, momentum;   // rho = RMSProp decay as well
  float l1, l2;                             // FTRL
};

// Optimizer groups: every kernel that applies the update is instantiated once per group and launched for the optimizer's
// group, so the reference's four run without the later cases in their switch: with one switch of all seven, the larger
// update cost the peer exchange kernels spills (ptxas -v, DESIGN.md section 5).  RPROP has a group of its own: as a fourth
// case of the EXT switch it slowed FTRL's optimizer pass at cfg2 from 21.0 to 24.3 us and RMSProp's from 19.5 to 21.1
// (scripts/bench_optimizer.py, H100 SXM 80 GB at 700 W).
enum OptGroup { OPT_BASE = 0, OPT_EXT = 1, OPT_RPROP = 2, OPT_GROUPS = 3 };
inline int opt_group(int kind) {   // the one place that maps an sb_optimizer to its group
  return kind == SB_OPT_RPROP ? OPT_RPROP : kind >= SB_OPT_ADAGRAD ? OPT_EXT : OPT_BASE;
}

// the state streams each optimizer has (HBM-bound passes touch only those): SGD none, Momentum and Adagrad s1, the others
// (RPROP included) s1 + s2
template <int G>
__device__ __forceinline__ bool opt_uses_s1(int kind) { return G != OPT_BASE || kind != SB_OPT_SGD; }
template <int G>
__device__ __forceinline__ bool opt_uses_s2(int kind) {
  return G != OPT_BASE ? kind != SB_OPT_ADAGRAD : (kind == SB_OPT_ADAM || kind == SB_OPT_ADADELTA);
}

// correctly rounded sqrtf and true divisions throughout (no rsqrtf, no fast-math): the fp32 oracle bounds stay tight
template <int G>
__device__ __forceinline__ float opt_update(const OptHyper& h, float lr_t, float theta, float g, float& s1, float& s2) {
  if constexpr (G == OPT_RPROP) {   // iRPROP- in torch.optim.Rprop's order: s1 = prev (the last gradient, 0 after a sign
                                     // flip), s2 = step size; lr_t is unused (the learning rate is only s2's start value)
    const float p = g * s1;   // a product that underflows to 0 counts as no change, as in torch
    s2 = fminf(fmaxf(s2 * (p > 0.f ? 1.2f : (p < 0.f ? 0.5f : 1.f)), 1e-6f), 50.f);
    s1 = p < 0.f ? 0.f : g;   // a sign flip: no move this step, and no flip next step
    return s1 > 0.f ? theta - s2 : (s1 < 0.f ? theta + s2 : theta);   // g = +-0: theta keeps its bits
  }
  if constexpr (G == OPT_EXT) {
    switch (h.kind) {
      case SB_OPT_ADAGRAD:   // s1 = accum
        s1 = s1 + g * g;
        return theta - lr_t * g / sqrtf(s1);
      case SB_OPT_RMSPROP:   // s1 = ms, s2 = mom (not centered)
        s1 = s1 + (g * g - s1) * (1.f - h.rho);
        s2 = h.momentum * s2 + lr_t * g / sqrtf(s1 + h.eps);
        return theta - s2;
      default: {             // SB_OPT_FTRL: s1 = accum, s2 = linear (lr_power = -0.5, no l2 shrinkage)
        const float a = s1 + g * g;
        const float sa = sqrtf(a);
        s2 = s2 + (g - (sa - sqrtf(s1)) / lr_t * theta);
        s1 = a;
        const float q = sa / lr_t + 2.f * h.l2;
        return fabsf(s2) > h.l1 ? (copysignf(h.l1, s2) - s2) / q : 0.f;
      }
    }
  }
  switch (h.kind) {
    case SB_OPT_SGD:
      return theta - lr_t * g;
    case SB_OPT_MOMENTUM:
      s1 = s1 * h.momentum + g;
      return theta - lr_t * s1;
    case SB_OPT_ADAM:
      s1 = s1 + (g - s1) * (1.f - h.beta1);
      s2 = s2 + (g * g - s2) * (1.f - h.beta2);
      return theta - lr_t * s1 / (sqrtf(s2) + h.eps);
    default: {  // SB_OPT_ADADELTA
      s1 = s1 * h.rho + g * g * (1.f - h.rho);
      const float upd = sqrtf(s2 + h.eps) / sqrtf(s1 + h.eps) * g;
      s2 = s2 * h.rho + upd * upd * (1.f - h.rho);
      return theta - upd * lr_t;
    }
  }
}

// One work item per block: a run of <= 1024 consecutive parameters.  Runs that lie inside a hidden-layer
// weight matrix also refresh its bf16 shadow W [in, ld_out] (row-major, the layout both the forward GEMM
// (MN-major B operand) and the dA GEMM (K-major B operand) consume).
struct OptWork {
  long long off;          // flat offset of the first element of the run
  int count;              // elements in this run (<= 1024)
  int out_dim;            // > 0: run lies in a weight matrix with this many columns
  long long mat_off;      // flat offset of that matrix
  __nv_bfloat16* Wn;      // shadow base (nullptr: no shadow)
  int ld_out;             // a multiple of 4 (Net::build_work): the 16-byte path's shadow stores are 8-byte aligned
  int np;                 // bf16 parts of the shadow (split-precision modes; 1 = plain)
  long long part_stride;  // elements between parts
};

// A run takes the 16-byte path (one thread = 4 consecutive parameters) when its parameters, and the elements of its shadow,
// come in aligned fours: 4 consecutive elements of a shadow-backed run never straddle a row (out_dim % 4 == 0).
// optimizer_kernel tests the macro: the bool an inlined function returns stays a value the kernel branches on (byte moves,
// another block layout), which made its Adagrad / RMSProp / FTRL / RPROP passes over the other layers ~0.8 us slower.  The
// exchange kernels test it through run_is_vec, whose kept value leaves them fewer registers and spills than the macro
// (xchg_ll<2, *>: 70-74 registers instead of 78-80).
#define SB_RUN_IS_VEC(wk) \
  (((wk).off & 3) == 0 && ((wk).count & 3) == 0 && ((wk).Wn == nullptr || (((wk).out_dim & 3) == 0 && (((wk).off - (wk).mat_off) & 3) == 0)))
__device__ __forceinline__ bool run_is_vec(const OptWork& wk) { return SB_RUN_IS_VEC(wk); }
// element offset inside one part of the shadow of flat parameter idx of a shadow-backed run
__device__ __forceinline__ long long shadow_at(const OptWork& wk, long long idx) {
  const long long m = idx - wk.mat_off;
  const long long r = m / wk.out_dim;
  return r * wk.ld_out + (m - r * wk.out_dim);
}

// store 4 / 1 updated weights into the bf16 shadow (all of its parts)
__device__ __forceinline__ void shadow_store4(const OptWork& wk, long long at, const float4& t) {
  for (int part = 0; part < wk.np; ++part) {
    uint2 o;
    o.x = pack_bf16x2(bf16_residual(t.x, part), bf16_residual(t.y, part));
    o.y = pack_bf16x2(bf16_residual(t.z, part), bf16_residual(t.w, part));
    *reinterpret_cast<uint2*>(wk.Wn + part * wk.part_stride + at) = o;
  }
}
__device__ __forceinline__ void shadow_store1(const OptWork& wk, long long at, float t) {
  for (int part = 0; part < wk.np; ++part) wk.Wn[part * wk.part_stride + at] = __float2bfloat16_rn(bf16_residual(t, part));
}

// The update of parameter idx (opt_apply1) or of the 4 from idx (opt_apply4, 16-byte path) and its write-back: theta, the
// state streams the optimizer has and every part of the shadow.  th, g, a, b are the loaded theta, the unscaled gradient (or
// the sum over ranks), s1 and s2 (0 where the optimizer has no such stream).  Returns the new theta.
template <int G>
__device__ __forceinline__ float4 opt_apply4(const OptHyper& h, float lr_t, float gs, const OptWork& wk, long long idx, float4 th,
                                             float4 g, float4 a, float4 b, float* theta, float* s1, float* s2) {
  float4 t;
  t.x = opt_update<G>(h, lr_t, th.x, g.x * gs, a.x, b.x);
  t.y = opt_update<G>(h, lr_t, th.y, g.y * gs, a.y, b.y);
  t.z = opt_update<G>(h, lr_t, th.z, g.z * gs, a.z, b.z);
  t.w = opt_update<G>(h, lr_t, th.w, g.w * gs, a.w, b.w);
  *reinterpret_cast<float4*>(theta + idx) = t;
  if (opt_uses_s1<G>(h.kind)) *reinterpret_cast<float4*>(s1 + idx) = a;
  if (opt_uses_s2<G>(h.kind)) *reinterpret_cast<float4*>(s2 + idx) = b;
  if (wk.Wn != nullptr) shadow_store4(wk, shadow_at(wk, idx), t);
  return t;
}
template <int G>
__device__ __forceinline__ float opt_apply1(const OptHyper& h, float lr_t, float gs, const OptWork& wk, long long idx, float th,
                                            float g, float a, float b, float* theta, float* s1, float* s2) {
  const float t = opt_update<G>(h, lr_t, th, g * gs, a, b);
  theta[idx] = t;
  if (opt_uses_s1<G>(h.kind)) s1[idx] = a;
  if (opt_uses_s2<G>(h.kind)) s2[idx] = b;
  if (wk.Wn != nullptr) shadow_store1(wk, shadow_at(wk, idx), t);
  return t;
}

// The last kernel of a step publishes the step scalars (loss sum, n_nz) and the step's loss-history slot straight into
// mapped pinned host memory: a posted PCIe write off the critical path instead of a D2H copy node between two steps.
__device__ __forceinline__ void publish_step_scalars(const float* scal, float* host_scal, const BatchDesc* desc) {
  if (host_scal != nullptr && blockIdx.x == 0 && threadIdx.x < SCAL_COUNT) {
    host_scal[threadIdx.x] = scal[threadIdx.x];
    if (threadIdx.x == 0 && desc->hist != nullptr) *desc->hist = make_float2(scal[SCAL_LOSS_SUM], scal[SCAL_NNZ]);   // loss curve
    __threadfence_system();
  }
}

template <int G>
static __global__ void __launch_bounds__(256)
optimizer_kernel(const OptWork* __restrict__ work, const BatchDesc* __restrict__ desc, OptHyper h,
                 float* __restrict__ theta, const float* __restrict__ grad, float* __restrict__ s1, float* __restrict__ s2,
                 const float* __restrict__ scal = nullptr, float* __restrict__ host_scal = nullptr,
                 unsigned long long* __restrict__ trace = nullptr) {
  if (trace != nullptr && blockIdx.x == 0 && threadIdx.x == 0) trace[0] = globaltimer_ns();   // debug timeline: entry
  pdl_wait();
  pdl_launch_dependents();
  if (trace != nullptr && blockIdx.x == 0 && threadIdx.x == 0) trace[2] = globaltimer_ns();   // dependencies resolved
  publish_step_scalars(scal, host_scal, desc);
  const OptWork wk = work[blockIdx.x];
  const float lr_t = desc->lr_t, gs = desc->gscale;
  // HBM-bound: only touch the state streams the optimizer actually has
  const bool use_s1 = opt_uses_s1<G>(h.kind);
  const bool use_s2 = opt_uses_s2<G>(h.kind);
  if (SB_RUN_IS_VEC(wk)) {
    // one thread = 4 consecutive parameters (a full 1024-run = 256 threads x float4)
    const int e = threadIdx.x * 4;
    if (e < wk.count) {
      const long long idx = wk.off + e;
      const float4 th = *reinterpret_cast<const float4*>(theta + idx);
      const float4 g = *reinterpret_cast<const float4*>(grad + idx);
      const float4 a = use_s1 ? *reinterpret_cast<const float4*>(s1 + idx) : make_float4(0.f, 0.f, 0.f, 0.f);
      const float4 b = use_s2 ? *reinterpret_cast<const float4*>(s2 + idx) : make_float4(0.f, 0.f, 0.f, 0.f);
      opt_apply4<G>(h, lr_t, gs, wk, idx, th, g, a, b, theta, s1, s2);
    }
    trace_end(trace);
    return;
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int e = threadIdx.x + 256 * i;
    if (e < wk.count) {
      const long long idx = wk.off + e;
      const float a = use_s1 ? s1[idx] : 0.f, b = use_s2 ? s2[idx] : 0.f;
      opt_apply1<G>(h, lr_t, gs, wk, idx, theta[idx], grad[idx], a, b, theta, s1, s2);
    }
  }
  trace_end(trace);
}

// Refresh the bf16 shadows from the fp32 master without touching state (after set_params / restore).
static __global__ void __launch_bounds__(256)
shadow_refresh_kernel(const OptWork* __restrict__ work, const float* __restrict__ theta) {
  const OptWork wk = work[blockIdx.x];
  if (wk.Wn == nullptr) return;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int e = threadIdx.x + 256 * i;
    if (e < wk.count) {
      const long long idx = wk.off + e;
      shadow_store1(wk, shadow_at(wk, idx), theta[idx]);
    }
  }
}

// ------------------------------------------------------------------------------------------------
// Wide+deep first layer (BASELINE config 4; spec + CPU oracle in oracle/wide_deep.py): Shifu's one-hot normalisation turns
// C categorical columns into n_onehot 0/1 columns of the reference's first dense layer (res/ssgd_monitor.py:57-71).  With
// idx[r, c] = the global one-hot column that is 1 for categorical column c of row r (-1 = missing), the one-hot block of
//     Z_0 = [X_dense | X_onehot] W_0 + b_0
// is a gather-sum of rows of W_e = W_0[n_dense:], and its gradient a scatter-add of dZ_0 rows.  Both read the SAME operand
// precision as the dense path (bf16 shadow / its parts, or fp32), so the sparse evaluation equals the dense layer on the
// materialised one-hot matrix up to fp32 summation order.  HBM/L2-bound: one warp per row, 16-byte accesses.
// ------------------------------------------------------------------------------------------------
struct EmbedParams {
  int rows, n_cat, H;              // H = width of hidden layer 0
  const int* idx;                  // [rows, n_cat]
  const __nv_bfloat16* We;         // bf16 modes: shadow rows of W_e [n_onehot, ldW] (part 0); nullptr in fp32 mode
  long long We_ps; int np;         // parts
  const float* We32;               // fp32 mode: master rows [n_onehot, ldW]
  int ldW;
  float* E; int ldE;               // gather: out [rows, ldE] fp32
  const __nv_bfloat16* dZ; long long dZ_ps; int ld_dZ;   // scatter: dZ_0 (bf16 modes) ...
  const float* dZ32;               // ... or fp32
  float* gWe;                      // scatter: gradient rows of W_e [n_onehot, H] fp32 (flat gradient, ld = H)
};

static __global__ void __launch_bounds__(256) embed_gather_kernel(const EmbedParams p) {
  pdl_wait();
  pdl_launch_dependents();
  const int lane = threadIdx.x & 31;
  const int r = blockIdx.x * 8 + (threadIdx.x >> 5);
  if (r >= p.rows) return;
  for (int c0 = lane * 8; c0 < p.H; c0 += 256) {       // 8 columns per lane per pass
    float acc[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) acc[k] = 0.f;
    for (int c = 0; c < p.n_cat; ++c) {
      const int j = __ldg(p.idx + static_cast<size_t>(r) * p.n_cat + c);
      if (j < 0) continue;
      if (p.We != nullptr) {
        for (int part = 0; part < p.np; ++part) {
          const __nv_bfloat16* src = p.We + part * p.We_ps + static_cast<size_t>(j) * p.ldW + c0;
          if (c0 + 8 <= p.H && (p.ldW & 7) == 0) {
            const uint4 raw = __ldg(reinterpret_cast<const uint4*>(src));
            const __nv_bfloat16* h = reinterpret_cast<const __nv_bfloat16*>(&raw);
#pragma unroll
            for (int k = 0; k < 8; ++k) acc[k] += __bfloat162float(h[k]);
          } else {
            for (int k = 0; k < 8; ++k)
              if (c0 + k < p.H) acc[k] += __bfloat162float(src[k]);
          }
        }
      } else {
        const float* src = p.We32 + static_cast<size_t>(j) * p.ldW + c0;
        for (int k = 0; k < 8; ++k)
          if (c0 + k < p.H) acc[k] += __ldg(src + k);
      }
    }
    float* dst = p.E + static_cast<size_t>(r) * p.ldE + c0;
    for (int k = 0; k < 8; ++k)
      if (c0 + k < p.H) dst[k] = acc[k];
  }
}

static __global__ void __launch_bounds__(256) embed_scatter_kernel(const EmbedParams p) {
  pdl_wait();
  pdl_launch_dependents();
  const int lane = threadIdx.x & 31;
  const int r = blockIdx.x * 8 + (threadIdx.x >> 5);
  if (r >= p.rows) return;
  for (int c0 = lane * 4; c0 < p.H; c0 += 128) {       // 4 columns per lane per pass -> red.global.add.v4.f32
    float g[4] = {0.f, 0.f, 0.f, 0.f};
    for (int k = 0; k < 4; ++k) {
      if (c0 + k >= p.H) break;
      if (p.dZ != nullptr) {
        for (int part = 0; part < p.np; ++part) g[k] += __bfloat162float(p.dZ[part * p.dZ_ps + static_cast<size_t>(r) * p.ld_dZ + c0 + k]);
      } else {
        g[k] = p.dZ32[static_cast<size_t>(r) * p.ld_dZ + c0 + k];
      }
    }
    for (int c = 0; c < p.n_cat; ++c) {
      const int j = __ldg(p.idx + static_cast<size_t>(r) * p.n_cat + c);
      if (j < 0) continue;
      float* dst = p.gWe + static_cast<size_t>(j) * p.H + c0;
      if (c0 + 4 <= p.H && (p.H & 3) == 0 && (reinterpret_cast<uintptr_t>(p.gWe) & 15) == 0) red_add_v4_f32(dst, g[0], g[1], g[2], g[3]);
      else
        for (int k = 0; k < 4; ++k)
          if (c0 + k < p.H) red_add_f32(dst + k, g[k]);
    }
  }
}

// acc += g  (epoch-sync schedule: ConditionalAccumulator.apply_grad, res/ssgd_monitor.py:136-141)
static __global__ void axpy_kernel(float* __restrict__ acc, const float* __restrict__ g, long long n,
                                   const float* __restrict__ scal = nullptr, float* __restrict__ host_scal = nullptr) {
  const long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  if (i < n) acc[i] += g[i];
  if (host_scal != nullptr && i < SCAL_COUNT) {   // tail kernel of an accumulate step: publish (loss sum, n_nz) to the host
    host_scal[i] = scal[i];
    __threadfence_system();
  }
}
// p[0..n) = 0, 16 bytes per thread where aligned (clears the step's gradient buffer on the side stream)
static __global__ void __launch_bounds__(256) zero_f32_kernel(float* __restrict__ p, long long n) {
  const long long n4 = ((reinterpret_cast<uintptr_t>(p) & 15) == 0) ? (n >> 2) : 0;
  for (long long i = blockIdx.x * 256ll + threadIdx.x; i < n4; i += gridDim.x * 256ll)
    reinterpret_cast<float4*>(p)[i] = make_float4(0.f, 0.f, 0.f, 0.f);
  for (long long i = n4 * 4 + blockIdx.x * 256ll + threadIdx.x; i < n; i += gridDim.x * 256ll) p[i] = 0.f;
}
static __global__ void scale_kernel(float* __restrict__ g, const BatchDesc* __restrict__ desc, long long n) {
  const long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  if (i < n) g[i] *= desc->gscale;
}
static __global__ void fill_kernel(float* __restrict__ p, float v, long long n) {
  const long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  if (i < n) p[i] = v;
}
// f32 -> bf16 with arbitrary leading dims (test hook operand staging)
static __global__ void cast_bf16_kernel(const float* __restrict__ src, int rows, int cols, __nv_bfloat16* __restrict__ dst, int ld,
                                        int np = 1, long long part_stride = 0) {
  const long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  if (i < static_cast<long long>(rows) * cols) {
    const int r = static_cast<int>(i / cols), c = static_cast<int>(i % cols);
    for (int part = 0; part < np; ++part)
      dst[part * part_stride + static_cast<size_t>(r) * ld + c] = __float2bfloat16_rn(bf16_residual(src[i], part));
  }
}

}  // namespace sb
