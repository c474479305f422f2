// The dW GEMMs of the tensor-core step that the planner puts on 128 x 256 tiles (plan_gemm), with split-K over the batch:
//
//   dW_l[in, out] += sum_rows A_{l-1}[rows, in] * dZ_l[rows, out]      A, B bf16 MN-major, fp32 red.add into the gradient
//
// Tile: one CTA owns 128 x 256 of dW_l and a range of k-blocks (one split).  Producer warpgroup, operand ring, main loop,
// kernel entry and exit: gemm_ring.cuh.  Warpgroup g multiplies rows 64 g .. 64 g + 63 of the tile with wgmma.m64n256k16
// (128 fp32 accumulator registers per thread).  The epilogue is an fp32 red.global.add of the accumulator in the wgmma
// fragment layout, straight from registers: no shared-memory staging (the thread-owns-row epilogue of gemm_tc.cuh would
// need it, and with 128 accumulator registers it does not fit), so the whole of shared memory goes to ring stages (48 KB
// per stage, 4 stages).  Split-precision modes (np > 1) walk an extended K axis of part pairs: only the producer's choice
// of tensor map depends on it.  128- and 64-wide dW tiles stay on gemm_tc.cuh: measured on one H100 SXM (700 W), its
// row-coalesced red.v4 (64 contiguous bytes per row) beats this fragment-layout one (32 bytes per row) on the high-split
// shapes those tiles get.
#pragma once
#include "gemm_tc.cuh"

namespace sb {

// shared memory besides the ring: 1024 B of alignment slack and the ring's barriers
struct GemmDwCfg : RingCfg<128 * 64 * 2, 256 * 64 * 2, 1024 + 256> {
  static constexpr int BM = 128, BN = 256;
};
static_assert(GemmDwCfg::STAGES >= 2, "operand ring");

static __global__ void __launch_bounds__(GemmDwCfg::THREADS, 1)
gemm_dw_kernel(const __grid_constant__ TmapSet tms, const GemmTcParams p) {
  using Cfg = GemmDwCfg;
  constexpr int BM = Cfg::BM, BN = Cfg::BN, BK = Cfg::BK;

  extern __shared__ uint8_t smem_raw[];
  const Ring<Cfg> ring(smem_raw, 0);

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const bool tracing = ring_enter(ring, 2, 0, &tms.a[0], &tms.b[0], p);   // one empty arrival per consumer warpgroup

  const int n_pairs = p.n_pairs > 0 ? p.n_pairs : 1;
  const int tiles_m = (p.M + BM - 1) / BM;
  const int tiles_n = (p.N + BN - 1) / BN;
  const int n_tiles = tiles_m * tiles_n;
  const int n_work = n_tiles * p.split_k;
  const int part_kb = (p.K + BK - 1) / BK;         // k-blocks of ONE part pair
  const int total_kb = part_kb * n_pairs;          // extended K axis: the pairs one after the other
  const int w_first = blockIdx.x;

  if (warp >= Cfg::PRODUCER_WARP) {
    asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(Cfg::PRODUCER_REGS));
    if (warp == Cfg::PRODUCER_WARP && lane == 0) {
      RingPos<Cfg::STAGES> pos;
      const int a_row0 = (p.a_rows != nullptr) ? p.a_rows->row0 : 0;  // batch position inside the resident set
      for (int w = w_first; w < n_work; w += gridDim.x) {
        const int tile = w % n_tiles, ks = w / n_tiles;
        const int m0 = (tile / tiles_n) * BM, n0 = (tile % tiles_n) * BN;
        const int kb0 = ks * p.kb_per_split;
        const int kb1 = min(total_kb, kb0 + p.kb_per_split);
        for (int kbx = kb0; kbx < kb1; ++kbx) {
          const int pp = (n_pairs > 1) ? kbx / part_kb : 0;     // which part pair this k-block belongs to
          const int kb = kbx - pp * part_kb;
          const CUtensorMap* tmA = &tms.a[n_pairs > 1 ? p.pair_a[pp] : 0];
          const CUtensorMap* tmB = &tms.b[n_pairs > 1 ? p.pair_b[pp] : 0];
          ring_issue(ring, pos, [&](uint32_t fb, uint32_t sa, uint32_t sb) {
            // 64(MN) x 64(K) boxes, 8 KB each, side by side along MN; the rows of the batch are K here
#pragma unroll
            for (int i = 0; i < BM / 64; ++i) tma_load_2d(sa + i * 8192, tmA, fb, m0 + i * 64, kb * BK + a_row0);
#pragma unroll
            for (int i = 0; i < BN / 64; ++i) tma_load_2d(sb + i * 8192, tmB, fb, n0 + i * 64, kb * BK);
          });
          if (kbx == kb0 && w == w_first) ring_stamp(p, tracing, 3);  // first TMA issued
        }
      }
    }
    ring_producer_tail<Cfg>(p);
  } else {
    // ================= consumer warpgroups (warps 0..7): MMA, then the red.add of the tile =================
    asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(Cfg::CONSUMER_REGS));
    const int wg = warp >> 2;                  // rows 64 wg .. 64 wg + 63 of the tile
    const uint32_t a_wg_off = static_cast<uint32_t>(wg) * 8192u;   // this warpgroup's 64-wide MN atom of the A stage
    // Fragment (ptx.cuh, wgmma_bf16): lane l holds for n8 block i the columns 8 i + 2 (l % 4) + 0/1 of row r and of row
    // r + 8.  One shuffle with the neighbour lane l ^ 1 gives each lane four consecutive columns of one row: even lanes
    // columns 8 i + 2 (l & 2) .. + 3 of row r, odd lanes the same columns of row r + 8.  A warp's red.v4 then covers 16
    // rows x 32 contiguous bytes (whole sectors).
    const bool odd = (lane & 1) != 0;
    const int frag_row = wg * 64 + (warp & 3) * 16 + (lane >> 2) + (odd ? 8 : 0);
    const int frag_col = 2 * (lane & 2);
    float acc_mi[1][BN / 2];
    float (&acc)[BN / 2] = acc_mi[0];
    RingPos<Cfg::STAGES> pos;
    for (int w = w_first; w < n_work; w += gridDim.x) {
      const int tile = w % n_tiles, ks = w / n_tiles;
      const int tm = tile / tiles_n, tn = tile % tiles_n;
      const int kb0 = ks * p.kb_per_split;
      const int kb1 = min(total_kb, kb0 + p.kb_per_split);

      ring_mma<BN, true, true>(ring, pos, kb1 - kb0, acc_mi, a_wg_off, 0u, (warp & 3) == 0 && lane == 0, w == w_first, p, tracing);

      const int row = tm * BM + frag_row;
      const int col0 = tn * BN + frag_col;
      float* gp = p.accum + static_cast<size_t>(row) * p.ld_acc + col0;
      // vector path: 16-byte aligned gradient rows and the tile's columns all inside N (warp-uniform)
      const bool vec = p.acc_vec4 && tn * BN + BN <= p.N;
#pragma unroll
      for (int i = 0; i < BN / 8; ++i) {
        const float s0 = odd ? acc[4 * i] : acc[4 * i + 2];
        const float s1 = odd ? acc[4 * i + 1] : acc[4 * i + 3];
        const float r0 = __shfl_xor_sync(0xffffffffu, s0, 1);
        const float r1 = __shfl_xor_sync(0xffffffffu, s1, 1);
        const float v0 = odd ? r0 : acc[4 * i], v1 = odd ? r1 : acc[4 * i + 1];
        const float v2 = odd ? acc[4 * i + 2] : r0, v3 = odd ? acc[4 * i + 3] : r1;
        if (row < p.M) {
          if (vec) {
            red_add_v4_f32(gp + 8 * i, v0, v1, v2, v3);
          } else {
            const int c = col0 + 8 * i;
            if (c < p.N) red_add_f32(gp + 8 * i, v0);
            if (c + 1 < p.N) red_add_f32(gp + 8 * i + 1, v1);
            if (c + 2 < p.N) red_add_f32(gp + 8 * i + 2, v2);
            if (c + 3 < p.N) red_add_f32(gp + 8 * i + 3, v3);
          }
        }
      }
      if (w == w_first && threadIdx.x == 0) ring_stamp(p, tracing, 7);  // first tile's epilogue done
    }
  }
  ring_exit(p, tracing);
}

// tms: the part maps of A_{l-1} (MN-major, box 64 x 64) and dZ_l (MN-major, box 64 x 64)
static inline int launch_gemm_dw(const GemmPlan& pl, const TmapSet& tms, GemmTcParams p, cudaStream_t st, bool pdl = false) {
  if (p.np < 1) p.np = 1;
  if (p.n_pairs < 1) p.n_pairs = 1;
  p.split_k = pl.split_k;
  p.kb_per_split = pl.kb_per_split;
  if (pl.bn != 256) return set_error(SB_ERR_INVALID, "gemm_dw has 128 x 256 tiles only (bn=%d)", pl.bn);
  return launch_kernel(gemm_dw_kernel, pl.grid, GemmDwCfg::THREADS, GemmDwCfg::SMEM_BYTES, st, pdl, tms, p);
}

// opt in to > 48 KB dynamic shared memory (once per process, outside of stream capture)
static inline int set_gemm_dw_attrs() { return set_max_smem(gemm_dw_kernel, GemmDwCfg::SMEM_BYTES); }

}  // namespace sb
