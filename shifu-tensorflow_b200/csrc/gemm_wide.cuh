// The plain-bf16 forward GEMMs that the planner (plan_gemm_pp) puts on 128 x 256 tiles:
//   A_l = act(A_{l-1} W_l + b_l)      A K-major [rows, in], B = W_l [in, out] MN-major
//
// Producer warpgroup, operand ring, main loop, kernel entry and exit: gemm_ring.cuh.  A stage holds one k-block of the
// tile: A as one K-major box of 64 (K) x 128 rows (16 KB), B as four MN-major 64 x 64 boxes (32 KB).  Both consumer
// warpgroups work on the same tile: warpgroup g multiplies rows 64 g .. 64 g + 63 with wgmma.m64n256k16 (128 fp32
// accumulator registers per thread, the gemm_dw.cuh layout).  Per k16 step that is one m64n256k16 per warpgroup instead
// of the two m64n128k16 of a 128 x 128 ping-pong tile: 27 % fewer operand bytes through shared memory per flop.
// Epilogue, in the wgmma fragment layout as in gemm_pp.cuh: bias (loaded before the main loop, staged in shared memory
// after it) + activation, bf16 pairs into the 128 x 256 epilogue buffer (four 128 x 64 tiles in the 128-byte swizzle of
// the output tensor map), then cp.async.bulk.tensor stores.  The epilogue is not hidden behind a main loop, but the
// producer keeps filling the ring with the next tile's k-blocks meanwhile, and the stores are only waited on (for their
// reads of the buffer) before the next tile's epilogue rewrites it.
// M / N / K tails: TMA zero fill on the load side, tensor-map clipping on the store side.
#pragma once
#include "gemm_pp.cuh"

namespace sb {

// besides the ring: align slack, barriers, bias [BN] fp32, the epilogue buffer (BM x BN bf16): 3 stages of 48 KB
struct GemmWideCfg : RingCfg<128 * 64 * 2, 256 * 64 * 2, 1024 + 256 + 256 * 4 + 128 * 256 * 2> {
  static constexpr int BM = 128, BN = 256;
  static constexpr int X_TILE = BM * 128;   // one BM x 64 bf16 swizzled tile
};
static_assert(GemmWideCfg::STAGES >= 3, "operand ring");

template <int ACT>
__global__ void __launch_bounds__(GemmWideCfg::THREADS, 1)
gemm_wide_kernel(const __grid_constant__ PpTmaps tms, const GemmTcParams p) {
  using Cfg = GemmWideCfg;
  constexpr int BM = Cfg::BM, BN = Cfg::BN, BK = Cfg::BK;

  extern __shared__ uint8_t smem_raw[];
  const Ring<Cfg> ring(smem_raw, Cfg::BN * Cfg::BM * 2);
  const uint32_t xs = ring.end();               // epilogue buffer (1024-byte aligned)
  const uint32_t bias_s = ring.bars + 256u;     // [BN] fp32

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const bool tracing = ring_enter(ring, 2, 0, &tms.a, &tms.b, p);   // one empty arrival per consumer warpgroup

  const int tiles_m = (p.M + BM - 1) / BM;
  const int tiles_n = (p.N + BN - 1) / BN;
  const int n_tiles = tiles_m * tiles_n;
  const int kb_n = (p.K + BK - 1) / BK;

  if (warp >= Cfg::PRODUCER_WARP) {
    asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(Cfg::PRODUCER_REGS));
    if (warp == Cfg::PRODUCER_WARP && lane == 0) {
      RingPos<Cfg::STAGES> pos;
      const int a_row0 = (p.a_rows != nullptr) ? p.a_rows->row0 : 0;  // batch position inside the resident set
      for (int t = blockIdx.x; t < n_tiles; t += gridDim.x) {
        const int m0 = (t / tiles_n) * BM, n0 = (t % tiles_n) * BN;
        for (int kb = 0; kb < kb_n; ++kb) {
          ring_issue(ring, pos, [&](uint32_t fb, uint32_t sa, uint32_t sb) {
            tma_load_2d(sa, &tms.a, fb, kb * BK, m0 + a_row0);
#pragma unroll
            for (int j = 0; j < BN / 64; ++j) tma_load_2d(sb + j * 8192, &tms.b, fb, n0 + j * 64, kb * BK);
          });
          if (kb == 0 && t == static_cast<int>(blockIdx.x)) ring_stamp(p, tracing, 3);  // first TMA issued
        }
      }
    }
    ring_producer_tail<Cfg>(p);
  } else {
    // ================= consumer warpgroups (warps 0..7): both on every tile of the CTA =================
    asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(Cfg::CONSUMER_REGS));
    const int g = warp >> 2;                       // rows 64 g .. 64 g + 63 of the tile
    const int ct = static_cast<int>(threadIdx.x);  // 0 .. 255
    // named barrier 2: the 256 consumer threads
    auto bar_consumers = [&]() { asm volatile("bar.sync 2, 256;" ::: "memory"); };
    const int r0 = 64 * g + (warp & 3) * 16 + (lane >> 2);   // fragment rows r0, r0 + 8
    const int c0 = 2 * (lane & 3);                           // fragment columns c0 + 8 i + {0, 1}
    // byte offset of the bf16 pair at (row r, column c) of the buffer: tile c / 64, 16-byte piece swizzled by r % 8
    auto xaddr = [&](int r, int c) {
      return xs + static_cast<uint32_t>((c >> 6) * Cfg::X_TILE + r * 128 + ((((c & 63) >> 3) ^ (r & 7)) << 4) + (c & 7) * 2);
    };

    float acc_mi[1][BN / 2];
    float (&acc)[BN / 2] = acc_mi[0];
    RingPos<Cfg::STAGES> pos;
    for (int t = blockIdx.x; t < n_tiles; t += gridDim.x) {
      const bool first = t == static_cast<int>(blockIdx.x);
      const int m0 = (t / tiles_n) * BM, n0 = (t % tiles_n) * BN;
      const int nx = min(BN / 64, (p.N - n0 + 63) / 64);   // 64-column tiles inside N
      const float bv = (n0 + ct < p.N) ? __ldg(p.bias + n0 + ct) : 0.f;   // lands during the main loop

      ring_mma<BN, false, true>(ring, pos, kb_n, acc_mi, static_cast<uint32_t>(g) * 8192u, 0u, (ct & 127) == 0, first, p,
                                tracing);

      // the previous tile's epilogue has read the bias (bar_consumers before its stores): stage this tile's
      asm volatile("st.shared.f32 [%0], %1;" ::"r"(bias_s + ct * 4u), "f"(bv) : "memory");
      if (ct == 0) tma_store_wait_read<0>();   // the previous tile's stores have read the buffer
      bar_consumers();
#pragma unroll
      for (int i = 0; i < BN / 8; ++i) {
        const int c = c0 + 8 * i;
        float2 b;
        asm volatile("ld.shared.v2.f32 {%0, %1}, [%2];" : "=f"(b.x), "=f"(b.y) : "r"(bias_s + c * 4u) : "memory");
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const float v0 = act_apply(acc[4 * i + 2 * h] + b.x, ACT);
          const float v1 = act_apply(acc[4 * i + 2 * h + 1] + b.y, ACT);
          asm volatile("st.shared.b32 [%0], %1;" ::"r"(xaddr(r0 + 8 * h, c)), "r"(pack_bf16x2(v0, v1)) : "memory");
        }
      }
      fence_proxy_async();   // generic-proxy writes -> visible to the TMA engine
      bar_consumers();       // the tile is complete in the buffer
      if (ct == 0) {
        for (int x = 0; x < nx; ++x) tma_store_2d(&tms.o, xs + x * Cfg::X_TILE, n0 + x * 64, m0);
        tma_store_commit();
      }
      if (first && ct == 0) ring_stamp(p, tracing, 7);  // first tile's epilogue done
    }
    if (ct == 0) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");   // the last tile is in global memory
  }
  ring_exit(p, tracing);
}

// tensor maps: a with 128-row boxes, b MN-major 64 x 64 boxes, o with 128-row boxes (the plan's bm_wg = 128)
static int launch_gemm_wide(const PpPlan& pl, const PpTmaps& tms, const GemmTcParams& p, cudaStream_t st, bool pdl) {
  if (pl.bm_wg != GemmWideCfg::BM || pl.bn != GemmWideCfg::BN)
    return set_error(SB_ERR_INVALID, "gemm_wide has 128 x 256 tiles only (bm_wg=%d bn=%d)", pl.bm_wg, pl.bn);
  return with_act(p.act, [&](auto ACT) {
    return launch_kernel(gemm_wide_kernel<ACT>, pl.grid, GemmWideCfg::THREADS, GemmWideCfg::SMEM_BYTES, st, pdl, tms, p);
  });
}

// opt in to > 48 KB dynamic shared memory (once per process, outside of stream capture)
static int set_gemm_wide_attrs() {
  for (int act = SB_ACT_NONE; act <= SB_ACT_LEAKYRELU; ++act)
    SB_TRY(with_act(act, [&](auto ACT) { return set_max_smem(gemm_wide_kernel<ACT>, GemmWideCfg::SMEM_BYTES); }));
  return SB_OK;
}

}  // namespace sb
