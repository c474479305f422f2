// The skeleton shared by the wgmma GEMM kernels (gemm_tc.cuh, gemm_pp.cuh, gemm_wide.cuh, gemm_dw.cuh, gemm_fwd_out.cuh):
// the TMA producer, the shared-memory operand ring, the consumers' k-block loop, kernel entry and exit.  The kernels add
// their tile enumeration, the boxes they load per k-block and their epilogues.
//
// Persistent, one CTA per SM, 384 threads = three warpgroups:
//   warps 8..11: the producer warpgroup.  One thread fills a STAGES-deep ring of 128-byte-swizzled TMA boxes, one k-block
//                (64 of K) per stage, in the order the consumers read them: it waits until the stage is empty, announces
//                the stage's bytes on its `full` mbarrier and issues the boxes, whose arrival the TMA engine signals on
//                that barrier.  The other three warps clear GemmTcParams::zero_buf when it is set.  The group gives its
//                registers to the consumers (setmaxnreg 40 / 232).
//   warps 0..7 : two consumer warpgroups.  Per k-block a group waits on `full`, issues its wgmma and keeps one wgmma group in
//                flight; once the group before it has retired, one thread of the warpgroup arrives on that stage's `empty`
//                mbarrier, which completes when every warpgroup that reads the stage has arrived.
// M / N / K tails need no code on the load side: TMA zero-fills out-of-bounds box elements.
// Trace (GemmTcParams::trace, stamps of CTA 0): [0] entry, [1] setup done, [2] dependencies resolved, [3] first TMA issued,
// [4] first stage landed, [5] MMAs of the first tile issued, [6] its accumulator complete, [7] first epilogue done, [8]
// exit ([3] and [7] are stamped by the kernels); [10] the latest exit over ALL CTAs (%globaltimer only grows, so atomicMax needs no reset
// between steps).  The in-graph kernel span is [2] .. [10].
#pragma once
#include <cuda.h>
#include "common.cuh"
#include "ptx.cuh"
#include "kernels.cuh"

namespace sb {

struct GemmTcParams {
  int M, N, K;
  int kb_per_split;  // k-blocks (of 64) per split
  int split_k;       // number of splits actually used (all non-empty)
  // EPI_FWD
  const float* bias;  // [N]
  int act;            // FWD: activation applied; DA: activation whose derivative is applied
  __nv_bfloat16* out;  // [M, ld_out] row-major (FWD, DA)
  int ld_out;
  // EPI_DA
  const __nv_bfloat16* aux;  // activation output A_{l-1} [M, ld_aux]
  int ld_aux;
  float* colsum;  // [N] fp32, atomically accumulated (bias gradient), nullable
  // EPI_DW / EPI_F32
  float* accum;  // [M, ld_acc] fp32
  int ld_acc;
  int acc_vec4;  // 1 if 16-byte aligned rows -> red.global.add.v4.f32
  // fused output layer (gemm_fwd_out_kernel: output layer + loss + its backward, res/ssgd_monitor.py:121,129)
  const float* wo;          // [N] output-layer weights (fp32)
  const float* bo;          // [1]
  const BatchDesc* desc;    // y, w of the current batch
  float* scal;              // SCAL_LOSS_SUM / SCAL_NNZ
  int loss;                 // sb_loss
  float *g_wo, *g_bo, *g_bL;  // gradient slots: dw_o [N], db_o [1], db_L [N]
  const BatchDesc* a_rows;  // non-null: operand A lives in the HBM-resident set; add a_rows->row0 to its row coordinate
  // optional: the producer warpgroup's idle warps clear this buffer (16-byte units) beside the main loop.  Used by the
  // layer-0 forward GEMM of a resident step to clear the step's gradient buffer (no memset node on the chain).
  float4* zero_buf;
  long long zero_n4;
  unsigned long long* trace;  // debug: CTA 0 writes %globaltimer stamps of its pipeline milestones (nullable)
  // Split-precision modes (SB_PREC_FP32_TC / SB_PREC_BF16X2, net.cuh): every fp32 operand value is held as np bf16 PARTS
  // v = p0 + p1 (+ p2) in np equally shaped arrays; the contraction is then a plain bf16 GEMM over an EXTENDED K axis that
  // walks the part pairs (a_i, b_j) with i + j < np one after the other, all accumulating into the same fp32 tile:
  //   np = 2 : a0b0 + a0b1 + a1b0                        (relative error ~2^-17 per product)
  //   np = 3 : a0b0 + a0b1 + a1b0 + a0b2 + a1b1 + a2b0   (~2^-24: fp32-class, what TF-CPU's fp32 GEMM delivers)
  // The MMA issuer does not know about it; the TMA producer picks the pair's tensor maps per k-block.
  int np;                     // parts per value in `out` / `aux` (1 = plain bf16)
  int n_pairs;                // part pairs accumulated (1, 3 or 6); 0 is read as 1
  unsigned char pair_a[6], pair_b[6];
  long long out_ps, aux_ps;   // element stride between consecutive parts of `out` / `aux`
  // EPI_FWD, nullable: fp32 [M, ld_add] added to the pre-activation before bias + activation.  Wide+deep first layer:
  // the sum of the embedding rows of the row's categorical values, i.e. the one-hot block of Z_0 = X W_0 evaluated as a
  // gather (oracle/wide_deep.py) while this GEMM contracts only the dense columns.
  const float* addend;
  int ld_add;
  // DET instantiations only (common.cuh, det_last_cta): the launch's slot workspace and ticket
  float* det_ws;
  unsigned int* det_ticket;
};

// Geometry of a ring GEMM: stages of A_BYTES + B_BYTES (one k-block) in the 227 KB of dynamic shared memory a block may
// have, as many as fit beside the kernel's FIXED_BYTES (1024 B of alignment slack, barriers, epilogue buffers), at most 8.
template <int A_BYTES_, int B_BYTES_, int FIXED_BYTES_>
struct RingCfg {
  static constexpr int BK = 64;              // 64 bf16 = 128 B = one swizzle row
  static constexpr int THREADS = 384;
  static constexpr int PRODUCER_WARP = 8;    // first warp of the producer warpgroup
  // per-thread registers after setmaxnreg: 2 x 128 x 232 + 128 x 40 <= 64 K
  static constexpr int CONSUMER_REGS = 232;
  static constexpr int PRODUCER_REGS = 40;
  static constexpr int A_BYTES = A_BYTES_, B_BYTES = B_BYTES_, FIXED_BYTES = FIXED_BYTES_;
  static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
  static constexpr int RING_BUDGET = 232448 - FIXED_BYTES;
  static constexpr int STAGES = RING_BUDGET / STAGE_BYTES > 8 ? 8 : RING_BUDGET / STAGE_BYTES;
  static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + FIXED_BYTES;
};

// Shared-memory addresses: the stages from the 1024-byte-aligned start of dynamic shared memory (SWIZZLE_128B), the
// kernel's buffers from end(), and bar_offset bytes past end() full[STAGES], empty[STAGES], then the kernel's own
// barriers (8 B each).
template <class Cfg>
struct Ring {
  uint32_t base, bars;
  __device__ __forceinline__ Ring(const uint8_t* smem, uint32_t bar_offset)
      : base((smem_u32(smem) + 1023u) & ~1023u), bars(base + Cfg::STAGES * Cfg::STAGE_BYTES + bar_offset) {}
  __device__ __forceinline__ uint32_t end() const { return base + Cfg::STAGES * Cfg::STAGE_BYTES; }
  __device__ __forceinline__ uint32_t a(int s) const { return base + s * Cfg::STAGE_BYTES; }
  __device__ __forceinline__ uint32_t b(int s) const { return a(s) + Cfg::A_BYTES; }
  __device__ __forceinline__ uint32_t full(int s) const { return bars + 8u * s; }
  __device__ __forceinline__ uint32_t empty(int s) const { return bars + 8u * (Cfg::STAGES + s); }
  __device__ __forceinline__ uint32_t bar(int i) const { return bars + 8u * (2 * Cfg::STAGES + i); }
};

// Stage and phase parity of a ring position.
template <int STAGES>
struct RingPos {
  int stage = 0;
  uint32_t phase = 0;
  __device__ __forceinline__ void advance() {
    if (++stage == STAGES) { stage = 0; phase ^= 1u; }
  }
  // the position of the n-th k-block the producer has issued
  __device__ __forceinline__ static RingPos at(int n) {
    RingPos r;
    r.stage = n % STAGES;
    r.phase = static_cast<uint32_t>(n / STAGES) & 1u;
    return r;
  }
};

// tracing: CTA 0 of a launch with a trace buffer, evaluated once by ring_enter (evaluated at every stamp, it costs the
// 128 x 128 dA ping-pong kernel a spill)
__device__ __forceinline__ void ring_stamp(const GemmTcParams& p, bool tracing, int slot) {
  if (tracing) p.trace[slot] = globaltimer_ns();
}

// Kernel entry.  Thread 0 initialises the barriers: `empty` expects empty_arrivals (one per warpgroup that reads a stage),
// the kernel's own n_own_bars barriers one arrival.  (Not the producer thread: its predicate would stay live across the
// consumer code.)  Everything before the PDL wait overlaps the previous kernel's tail; from there on global memory written
// by it is touched.  Returns whether this CTA stamps the trace.
template <class Cfg>
__device__ __forceinline__ bool ring_enter(const Ring<Cfg>& ring, uint32_t empty_arrivals, int n_own_bars, const void* tm_a,
                                           const void* tm_b, const GemmTcParams& p) {
  const bool tracing = p.trace != nullptr && blockIdx.x == 0;
  if (threadIdx.x == 0) ring_stamp(p, tracing, 0);
  if (threadIdx.x == 0) {
    tma_prefetch_desc(tm_a);
    tma_prefetch_desc(tm_b);
    for (int s = 0; s < Cfg::STAGES; ++s) {
      mbar_init(ring.full(s), 1);   // the producer's arrive.expect_tx
      mbar_init(ring.empty(s), empty_arrivals);
    }
    for (int i = 0; i < n_own_bars; ++i) mbar_init(ring.bar(i), 1);
    fence_barrier_init();
  }
  __syncthreads();
  if (threadIdx.x == 0) ring_stamp(p, tracing, 1);
  pdl_wait();
  pdl_launch_dependents();
  if (threadIdx.x == 0) ring_stamp(p, tracing, 2);
  return tracing;
}

__device__ __forceinline__ void ring_exit(const GemmTcParams& p, bool tracing) {
  __syncthreads();
  if (threadIdx.x == 0) {
    ring_stamp(p, tracing, 8);
    if (p.trace != nullptr) atomicMax(p.trace + 10, static_cast<unsigned long long>(globaltimer_ns()));
  }
}

// The producer thread's step for one k-block at ring position pos (advanced past it): wait until the stage is empty,
// announce its bytes on its `full` barrier, then boxes(full_bar, a_dst, b_dst) issues the k-block's TMA loads into it.
template <class Cfg, class Boxes>
__device__ __forceinline__ void ring_issue(const Ring<Cfg>& ring, RingPos<Cfg::STAGES>& pos, Boxes&& boxes) {
  mbar_wait(ring.empty(pos.stage), pos.phase ^ 1u);
  const uint32_t fb = ring.full(pos.stage);
  mbar_arrive_expect_tx(fb, Cfg::STAGE_BYTES);
  boxes(fb, ring.a(pos.stage), ring.b(pos.stage));
  pos.advance();
}

// The rest of the producer warpgroup, after the producer thread: its other three warps clear GemmTcParams::zero_buf.
template <class Cfg>
__device__ __forceinline__ void ring_producer_tail(const GemmTcParams& p) {
  if ((threadIdx.x >> 5) > Cfg::PRODUCER_WARP && p.zero_buf != nullptr) {
    // (read by nobody before the next kernel boundary)
    const float4 z4 = make_float4(0.f, 0.f, 0.f, 0.f);
    const long long zt = static_cast<long long>(threadIdx.x) - 32 * (Cfg::PRODUCER_WARP + 1), zn = 32 * 3;
    for (long long i = static_cast<long long>(blockIdx.x) * zn + zt; i < p.zero_n4; i += static_cast<long long>(gridDim.x) * zn)
      p.zero_buf[i] = z4;
  }
  __syncwarp();   // the whole warp reaches the final block barrier together (bar.sync counts warps, not lanes)
}

struct RingNoOp {
  __device__ __forceinline__ void operator()() const {}
};

// One consumer warpgroup's main loop: n_kb k-blocks from ring position pos (which it advances past them) into acc.  MI
// blocks of 64 rows of A, from a_off into the stage and 8 KB apart (the next 64 rows of a K-major box, the next MN atom of
// MN-major ones), times the N columns of B from b_off: MI wgmma.m64nNk16 per 16 of K.  `releaser` is the one thread of the
// warpgroup that arrives on a stage's `empty` barrier once the wgmma group that read it has retired.  issued() runs when
// the last k-block is issued, before its wgmma group retires.  first_tile: stamps 4 to 6.
template <int N, bool A_MN, bool B_MN, class Cfg, int MI, class Issued = RingNoOp>
__device__ __forceinline__ void ring_mma(const Ring<Cfg>& ring, RingPos<Cfg::STAGES>& pos, int n_kb, float (&acc)[MI][N / 2],
                                         uint32_t a_off, uint32_t b_off, bool releaser, bool first_tile,
                                         const GemmTcParams& p, bool tracing, Issued&& issued = Issued()) {
  // descriptor steps for 16 elements along K: K-major = 32 B inside the swizzle row; MN-major = 16 rows of 128 B
  constexpr uint32_t a_kstep = A_MN ? (2048u >> 4) : (32u >> 4);
  constexpr uint32_t b_kstep = B_MN ? (2048u >> 4) : (32u >> 4);
  int prev_stage = -1;
  for (int kb = 0; kb < n_kb; ++kb) {
    mbar_wait(ring.full(pos.stage), pos.phase);  // the stage's TMA bytes have landed
    if (kb == 0 && first_tile && threadIdx.x == 0) ring_stamp(p, tracing, 4);
    const uint32_t sa = ring.a(pos.stage) + a_off, sb = ring.b(pos.stage) + b_off;
    const uint64_t da = A_MN ? make_mnmajor_sw128_desc(sa, 8192u) : make_kmajor_sw128_desc(sa);
    const uint64_t db = B_MN ? make_mnmajor_sw128_desc(sb, 8192u) : make_kmajor_sw128_desc(sb);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < Cfg::BK / 16; ++k) {
#pragma unroll
      for (int mi = 0; mi < MI; ++mi)
        wgmma_bf16<N, A_MN ? 1 : 0, B_MN ? 1 : 0>(acc[mi], da + (8192u >> 4) * mi + a_kstep * k, db + b_kstep * k,
                                                  (kb > 0 || k > 0) ? 1u : 0u);
    }
    wgmma_commit();
    wgmma_wait<1>();   // the previous k-block's wgmma group has finished reading its stage
    if (prev_stage >= 0 && releaser) mbar_arrive(ring.empty(prev_stage));
    prev_stage = pos.stage;
    pos.advance();
  }
  issued();
  wgmma_wait<0>();
  if (prev_stage >= 0 && releaser) mbar_arrive(ring.empty(prev_stage));
  if (first_tile && threadIdx.x == 0) { ring_stamp(p, tracing, 5); ring_stamp(p, tracing, 6); }
}

}  // namespace sb
