// Ping-pong wgmma / TMA GEMM for the plain-bf16 forward and dA GEMMs of a training step and the forward GEMMs of scoring:
//   EPI_FWD : A_l      = act(A_{l-1} W_l + b_l)                 A K-major [rows, in], B = W_l [in, out] MN-major
//   EPI_DA  : dZ_{l-1} = (dZ_l W_l^T) * act'(A_{l-1}),  db_{l-1} += column sums     A K-major [rows, out], B = W_l K-major
//
// Producer warpgroup, operand ring, main loop, kernel entry and exit: gemm_ring.cuh.  The producer fills the ring with the
// k-blocks of the CTA's tiles in tile order.
//   warps 0..7 : two consumer warpgroups.  Each owns WHOLE tiles of BM_WG x BN: the CTA's tiles alternate between them
//                (local tile 0, 2, 4, ... -> group 0; 1, 3, 5, ... -> group 1).  A group skips the other's k-blocks when it
//                advances its ring position.  An ordered pair of named barriers makes the groups take turns issuing their
//                main loops, so one group's wgmma run while the other runs its epilogue: the tensor cores are not idle
//                for the length of an epilogue, and the epilogue no longer shares the SM with its own group's next fill.
// Accumulator: BM_WG / 64 wgmma.m64nBNk16 per k16 step (128 registers per thread at 128 x 128).
// Epilogues run in the wgmma fragment layout (thread = warp w of the group, lane l: rows 64 mi + 16 w + l / 4 (+ 8),
// columns 8 i + 2 (l % 4) + {0, 1}); nothing fp32 is staged through shared memory.  Each group has one epilogue buffer of
// BM_WG x BN bf16: BN / 64 tiles of BM_WG x 64 in the 128-byte swizzle the output tensor map expects.  A bf16 pair per
// thread and n8 block is a conflict-free 4-byte access in that layout.
//   forward: bias (staged in shared memory before the main loop) + activation in place, bf16 pairs into the buffer,
//            cp.async.bulk.tensor stores
//   dA     : A_{l-1}'s tile arrives by TMA into the buffer during the main loop, act' is applied to the accumulator and
//            dZ_{l-1} is written over A_{l-1} in place, then stored by TMA.  Column sums: each thread adds its rows, a
//            reduce-scatter over the warp's 8 row groups (colsum_row_groups), one shared-memory slot per warp, the 4 warps
//            added in a fixed order (a step's result does not depend on warp timing), one red.global per column and tile.
// M / N / K tails: TMA zero fill on the load side (so out-of-range accumulator rows and columns are 0 and add nothing to the
// column sums), tensor-map clipping on the store side.
#pragma once
#include "gemm_tc.cuh"

namespace sb {

// tensor maps of one ping-pong GEMM (plain bf16: one part per operand)
struct PpTmaps {
  CUtensorMap a;   // K-major: box 64 (K) x BM_WG rows
  CUtensorMap b;   // forward: MN-major, box 64 (N) x 64 (K); dA: K-major, box 64 (K) x BN rows
  CUtensorMap o;   // output [M, N] bf16: box 64 columns x BM_WG rows (store)
  CUtensorMap x;   // dA: A_{l-1} [M, N] bf16, same box (load)
};

// besides the ring: align slack, barriers, bias [group][BN], column sums [group][parity][warp][BN], the two epilogue
// buffers (X_BYTES each)
template <int BM_WG, int BN>
struct GemmPpCfg : RingCfg<BM_WG * 64 * 2, BN * 64 * 2, 1024 + 256 + 2 * BN * 4 + 16 * BN * 4 + 2 * BM_WG * BN * 2> {
  static_assert(BM_WG == 64 || BM_WG == 128, "warpgroup tile rows");
  static_assert(BN == 64 || BN == 128, "tile N");
  static_assert(GemmPpCfg::STAGES >= 4, "operand ring");
  static constexpr int X_TILE = BM_WG * 128;               // one BM_WG x 64 bf16 swizzled tile
  static constexpr int X_BYTES = X_TILE * (BN / 64);       // one group's epilogue buffer
};

// DET (dA only): a tile's column sums are stored into slot m0 / BM_WG (its row tile) of p.det_ws [row tile][N] instead of
// red.global, and the CTA that arrives last adds the row tiles in ascending order into p.colsum (common.cuh, det_last_cta)
template <int BM_WG, int BN, int EPI, int ACT, bool DET = false>
__global__ void __launch_bounds__(GemmPpCfg<BM_WG, BN>::THREADS, 1)
gemm_pp_kernel(const __grid_constant__ PpTmaps tms, const GemmTcParams p) {
  static_assert(EPI == EPI_FWD || EPI == EPI_DA, "forward or dA");
  static_assert(!DET || EPI == EPI_DA, "DET: dA column sums only");
  using Cfg = GemmPpCfg<BM_WG, BN>;
  constexpr int BK = Cfg::BK, MI = BM_WG / 64;
  constexpr bool B_MN = EPI == EPI_FWD;

  extern __shared__ uint8_t smem_raw[];
  const Ring<Cfg> ring(smem_raw, 2 * Cfg::X_BYTES);
  const uint32_t xs_base = ring.end();                                // [group] epilogue buffers (1024-byte aligned)
  const uint32_t sm_bias = ring.bars + 256u;                          // [group][BN] fp32
  const uint32_t sm_col = sm_bias + 2u * BN * 4u;                     // [group][tile parity][warp][BN] fp32
  auto aux_bar = [&](int g) { return ring.bar(g); };

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  // empty: one arrival, by the warpgroup that owns the tile; two own barriers: aux_bar(0), aux_bar(1)
  const bool tracing = ring_enter(ring, 1, 2, &tms.a, &tms.b, p);

  const int tiles_m = (p.M + BM_WG - 1) / BM_WG;
  const int tiles_n = (p.N + BN - 1) / BN;
  const int n_tiles = tiles_m * tiles_n;
  const int kb_n = (p.K + BK - 1) / BK;

  if (warp >= Cfg::PRODUCER_WARP) {
    asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(Cfg::PRODUCER_REGS));
    if (warp == Cfg::PRODUCER_WARP && lane == 0) {
      RingPos<Cfg::STAGES> pos;
      const int a_row0 = (p.a_rows != nullptr) ? p.a_rows->row0 : 0;  // batch position inside the resident set
      for (int t = blockIdx.x; t < n_tiles; t += gridDim.x) {
        const int m0 = (t / tiles_n) * BM_WG, n0 = (t % tiles_n) * BN;
        for (int kb = 0; kb < kb_n; ++kb) {
          ring_issue(ring, pos, [&](uint32_t fb, uint32_t sa, uint32_t sb) {
            tma_load_2d(sa, &tms.a, fb, kb * BK, m0 + a_row0);
            if constexpr (B_MN) {
#pragma unroll
              for (int j = 0; j < BN / 64; ++j) tma_load_2d(sb + j * 8192, &tms.b, fb, n0 + j * 64, kb * BK);
            } else {
              tma_load_2d(sb, &tms.b, fb, kb * BK, n0);
            }
          });
          if (kb == 0 && t == static_cast<int>(blockIdx.x)) ring_stamp(p, tracing, 3);  // first TMA issued
        }
      }
    }
    ring_producer_tail<Cfg>(p);
  } else {
    // ================= consumer warpgroups: whole tiles, alternating =================
    asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(Cfg::CONSUMER_REGS));
    const int g = warp >> 2;                      // this group's tiles: local tile g, g + 2, ...
    const int gt = static_cast<int>(threadIdx.x) & 127;
    const bool xthread = gt == 0;                 // issues the group's epilogue TMA and its ring releases
    // named barriers: 2 + g = this group's 128 threads; 4 + g = "group g may issue its main loop" (group g syncs, the other
    // group arrives once it has issued the main loop of the tile before)
    auto bar_wg = [&]() { asm volatile("bar.sync %0, 128;" ::"r"(2 + g) : "memory"); };
    const uint32_t xs = xs_base + static_cast<uint32_t>(g) * Cfg::X_BYTES;
    const uint32_t bias_s = sm_bias + static_cast<uint32_t>(g) * BN * 4u;
    const uint32_t col_w = sm_col + static_cast<uint32_t>(g * 8 + (warp & 3)) * BN * 4u;   // this warp's column-sum slots
    const int r0 = (warp & 3) * 16 + (lane >> 2);   // fragment rows r0 + 8 h + 64 mi
    const int c0 = 2 * (lane & 3);                  // fragment columns c0 + 8 i + {0, 1}
    // byte offset of the bf16 pair at (row r, column c) of the group's buffer: tile c / 64, 16-byte piece swizzled by r % 8
    auto xaddr = [&](int r, int c) {
      return xs + static_cast<uint32_t>((c >> 6) * Cfg::X_TILE + r * 128 + ((((c & 63) >> 3) ^ (r & 7)) << 4) + (c & 7) * 2);
    };
    const bool do_cols = EPI == EPI_DA && p.colsum != nullptr;

    float acc[MI][BN / 2];
    for (int lt = g;; lt += 2) {
      const int t = static_cast<int>(blockIdx.x) + lt * static_cast<int>(gridDim.x);
      if (t >= n_tiles) break;
      const int it = lt >> 1;                      // tiles this group has done
      const int m0 = (t / tiles_n) * BM_WG, n0 = (t % tiles_n) * BN;
      const int nx = min(BN / 64, (p.N - n0 + 63) / 64);   // 64-column tiles inside N

      // ---------- before the main loop: the buffer is free once this group's previous stores have read it ----------
      if (xthread) tma_store_wait_read<0>();
      if constexpr (EPI == EPI_FWD) {
        for (int j = gt; j < BN; j += 128) {
          const float bv = (n0 + j < p.N) ? __ldg(p.bias + n0 + j) : 0.f;
          asm volatile("st.shared.f32 [%0], %1;" ::"r"(bias_s + j * 4u), "f"(bv) : "memory");
        }
        bar_wg();   // bias staged; every thread may now overwrite the buffer
      } else {
        if (xthread) {   // A_{l-1}'s tile, landing during the main loop
          mbar_arrive_expect_tx(aux_bar(g), static_cast<uint32_t>(nx * Cfg::X_TILE));
          for (int x = 0; x < nx; ++x) tma_load_2d(xs + x * Cfg::X_TILE, &tms.x, aux_bar(g), n0 + x * 64, m0);
        }
      }

      // ---------- main loop, in turn with the other group ----------
      if (lt >= 1) asm volatile("bar.sync %0, 256;" ::"r"(4 + g) : "memory");
      RingPos<Cfg::STAGES> pos = RingPos<Cfg::STAGES>::at(lt * kb_n);   // after the k-blocks of every earlier tile of the CTA
      ring_mma<BN, false, B_MN>(ring, pos, kb_n, acc, 0u, 0u, xthread, lt == 0, p, tracing, [&] {
        // the other group's next tile (local tile lt + 1) may issue now
        if (t + static_cast<int>(gridDim.x) < n_tiles) asm volatile("bar.arrive %0, 256;" ::"r"(4 + (g ^ 1)) : "memory");
      });

      // ---------- epilogue in the fragment layout ----------
      if constexpr (EPI == EPI_FWD) {
#pragma unroll
        for (int i = 0; i < BN / 8; ++i) {
          const int c = c0 + 8 * i;
          float2 b;
          asm volatile("ld.shared.v2.f32 {%0, %1}, [%2];" : "=f"(b.x), "=f"(b.y) : "r"(bias_s + c * 4u) : "memory");
#pragma unroll
          for (int mi = 0; mi < MI; ++mi) {
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              const float v0 = act_apply(acc[mi][4 * i + 2 * h] + b.x, ACT);
              const float v1 = act_apply(acc[mi][4 * i + 2 * h + 1] + b.y, ACT);
              asm volatile("st.shared.b32 [%0], %1;" ::"r"(xaddr(64 * mi + r0 + 8 * h, c)), "r"(pack_bf16x2(v0, v1)) : "memory");
            }
          }
        }
      } else {
        mbar_wait(aux_bar(g), static_cast<uint32_t>(it) & 1u);   // A_{l-1}'s tile has landed
        const uint32_t cb = col_w + static_cast<uint32_t>(it & 1) * 4u * BN * 4u;
#pragma unroll
        for (int x = 0; x < BN / 64; ++x) {   // one 64-column tile at a time (keeps the column sums at 16 registers)
          float cs[16];   // per column pair of the thread in this tile: the sum over its rows
#pragma unroll
          for (int i = 0; i < 8; ++i) {
            const int c = 64 * x + c0 + 8 * i;
            float s0 = 0.f, s1 = 0.f;
#pragma unroll
            for (int mi = 0; mi < MI; ++mi) {
#pragma unroll
              for (int h = 0; h < 2; ++h) {
                const uint32_t a = xaddr(64 * mi + r0 + 8 * h, c);
                uint32_t raw;
                asm volatile("ld.shared.b32 %0, [%1];" : "=r"(raw) : "r"(a) : "memory");
                const float x0 = __uint_as_float(raw << 16), x1 = __uint_as_float(raw & 0xFFFF0000u);   // bf16 pair -> fp32
                const float v0 = acc[mi][32 * x + 4 * i + 2 * h] * act_grad_from_out(x0, ACT);
                const float v1 = acc[mi][32 * x + 4 * i + 2 * h + 1] * act_grad_from_out(x1, ACT);
                asm volatile("st.shared.b32 [%0], %1;" ::"r"(a), "r"(pack_bf16x2(v0, v1)) : "memory");
                s0 += v0;
                s1 += v1;
              }
            }
            cs[2 * i] = s0;
            cs[2 * i + 1] = s1;
          }
          if (do_cols) {
            colsum_row_groups(cs, lane);
            // values 2 q, 2 q + 1 (q = lane / 4) = the column pair 8 q + c0 of this tile
            const uint32_t col = static_cast<uint32_t>(64 * x + c0 + 8 * (lane >> 2));
            asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(cb + col * 4u), "f"(cs[0]), "f"(cs[1]) : "memory");
          }
        }
      }
      fence_proxy_async();   // generic-proxy writes -> visible to the TMA engine
      bar_wg();              // the tile is complete in the buffer; the column sums of every warp are in
      if (xthread) {
        for (int x = 0; x < nx; ++x) tma_store_2d(&tms.o, xs + x * Cfg::X_TILE, n0 + x * 64, m0);
        tma_store_commit();
      }
      if (do_cols) {
        // the 4 warps' sums in a fixed order, one red.global per column and tile; the slots of this parity are rewritten two
        // tiles later, after the next bar_wg
        const uint32_t cb = col_w + static_cast<uint32_t>((it & 1) * 4 - (warp & 3)) * BN * 4u;   // warp 0's slot
        for (int j = gt; j < BN; j += 128) {
          float v = 0.f;
#pragma unroll
          for (int w = 0; w < 4; ++w) {
            float x;
            asm volatile("ld.shared.f32 %0, [%1];" : "=f"(x) : "r"(cb + (w * BN + j) * 4u) : "memory");
            v += x;
          }
          if constexpr (DET) {
            if (n0 + j < p.N) p.det_ws[(t / tiles_n) * p.N + n0 + j] = v;   // row tile t / tiles_n (< 2^31 slots)
          } else {
            if (n0 + j < p.N && v != 0.f) red_add_f32(p.colsum + n0 + j, v);
          }
        }
      }
      if (lt == 0 && threadIdx.x == 0) ring_stamp(p, tracing, 7);  // first tile's epilogue done
    }
    if constexpr (DET) {
      // both consumer groups (named barrier 1, unused by the main loop) have stored the slots of all their tiles
      // (nothing of the tile loop stays live for this: the predicate and the slot count come from the parameters)
      if (p.colsum != nullptr)
        det_colsum_tail(p.det_ticket, p.det_ws, (p.M + BM_WG - 1) / BM_WG, p.N, p.colsum, 1, 256, static_cast<int>(threadIdx.x));
    }
    if (xthread) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");   // the last tiles are in global memory
  }
  ring_exit(p, tracing);
}

// ------------------------------------------------------------------ host side
struct PpPlan {
  int bm_wg;   // rows of one warpgroup's tile: 128, or 64 when 128-row tiles would leave warpgroups without a tile;
               // 128 = the CTA's rows for the 128 x 256 forward tile (bn = 256)
  int bn;      // 64 / 128: gemm_pp_kernel; 256: gemm_wide_kernel (gemm_wide.cuh, forward only)
  int grid;
};

// PP_TILE_WIDE as the forced tile: the 128 x 256 forward tile of gemm_wide.cuh
constexpr int PP_TILE_WIDE = 256;

// tile = 0: chosen from the shape; 64 / 128 force the ping-pong kernel's warpgroup tile rows, PP_TILE_WIDE the 128 x 256
// forward tile (the caller rejects it for dA).
// Forward GEMMs go on 128 x 256 tiles when N > 128 (a narrower layer would fill half the tile with zeros), there are at
// least 7/8 as many such tiles as SMs, no more waves of them than of 128 x 128 tiles (each counted twice: a 256-wide
// tile is two 128-wide ones), and the main loop is long (>= 16 k-blocks), so that the exposed epilogue is a small share of
// a tile.  cfg2's forward 0 and 1 qualify (256 and 128 tiles on 132 SMs; one H100 SXM at 400 W, relu: 8192 x 1024 x 2000
// 71.0 -> 64.3 us, 8192 x 512 x 1024 18.0 -> 17.2 us), cfg1's largest does not (4096 x 512 x 1000, 64 tiles: 11.9 us on
// ping-pong, 15.1 us wide), nor cfg2's forward 2 (8192 x 256 x 512, 64 tiles: 7.8 vs 10.5 us).
// Otherwise (ping-pong) a CTA needs two tiles for both of its warpgroups to have work, so with no more 128-row tiles than
// SMs 64-row tiles give each CTA two to four.  Except when 128-row tiles still cover nearly every SM and the main loop is
// long (>= 8 k-blocks): there the taller tile's operand reuse wins over the overlapped epilogue (one H100 SXM, 132 SMs:
// 4096 x 512 x 1000 takes 11.7 us with 128-row tiles, 13.2 us with 64; 8192 x 256 x 512 7.6 vs 9.1 us; 4096 x 512 x 256,
// 4 k-blocks, 7.8 vs 7.4 us).
static inline PpPlan plan_gemm_pp(int M, int N, int K, int num_sms, bool fwd, int tile = 0) {
  PpPlan pl = {};
  const int tiles_m = (M + 127) / 128, kb = (K + 63) / 64;
  const int wide_tiles = tiles_m * ((N + 255) / 256), narrow_tiles = tiles_m * ((N + 127) / 128);
  const bool wide = fwd && N > 128 && 8 * wide_tiles >= 7 * num_sms && kb >= 16 &&
                    2 * ((wide_tiles + num_sms - 1) / num_sms) <= (narrow_tiles + num_sms - 1) / num_sms;
  if (tile == PP_TILE_WIDE || (tile == 0 && wide)) {
    pl.bm_wg = 128;
    pl.bn = 256;
    pl.grid = wide_tiles < num_sms ? wide_tiles : num_sms;
    return pl;
  }
  pl.bn = N <= 64 ? 64 : 128;
  const int tiles_n = (N + pl.bn - 1) / pl.bn;
  const int tiles128 = tiles_m * tiles_n;
  const bool tall = tiles128 > num_sms || (8 * tiles128 >= 7 * num_sms && kb >= 8);
  pl.bm_wg = tile > 0 ? tile : (tall ? 128 : 64);
  const int tiles = ((M + pl.bm_wg - 1) / pl.bm_wg) * tiles_n;
  pl.grid = tiles < num_sms ? tiles : num_sms;
  return pl;
}

// f(integral_constant BM_WG, integral_constant BN) for a plan's tile shape
template <typename F>
static int with_pp_shape(int bm_wg, int bn, F&& f) {
  using std::integral_constant;
  if (bm_wg == 128 && bn == 128) return f(integral_constant<int, 128>(), integral_constant<int, 128>());
  if (bm_wg == 128 && bn == 64) return f(integral_constant<int, 128>(), integral_constant<int, 64>());
  if (bm_wg == 64 && bn == 128) return f(integral_constant<int, 64>(), integral_constant<int, 128>());
  if (bm_wg == 64 && bn == 64) return f(integral_constant<int, 64>(), integral_constant<int, 64>());
  return set_error(SB_ERR_INVALID, "no gemm_pp instantiation for bm_wg=%d bn=%d", bm_wg, bn);
}

// tensor maps (pl.bm_wg-row boxes) must have been made for the same plan.  A dA launch with p.det_ws set runs the DET
// instantiation (p.det_ws: [ceil(M / bm_wg)][N] floats).
template <int EPI>
static int launch_gemm_pp(const PpPlan& pl, const PpTmaps& tms, const GemmTcParams& p, cudaStream_t st, bool pdl) {
  return with_pp_shape(pl.bm_wg, pl.bn, [&](auto BM_WG, auto BN) {
    return with_act(p.act, [&](auto ACT) {
      using Cfg = GemmPpCfg<BM_WG, BN>;
      if constexpr (EPI == EPI_DA)
        if (p.det_ws != nullptr)
          return launch_kernel(gemm_pp_kernel<BM_WG, BN, EPI, ACT, true>, pl.grid, Cfg::THREADS, Cfg::SMEM_BYTES, st, pdl, tms, p);
      return launch_kernel(gemm_pp_kernel<BM_WG, BN, EPI, ACT>, pl.grid, Cfg::THREADS, Cfg::SMEM_BYTES, st, pdl, tms, p);
    });
  });
}

// opt in to > 48 KB dynamic shared memory (once per process, outside of stream capture)
static int set_gemm_pp_attrs() {
  for (int bm_wg : {64, 128})
    for (int bn : {64, 128})
      for (int act = SB_ACT_NONE; act <= SB_ACT_LEAKYRELU; ++act)
        SB_TRY(with_pp_shape(bm_wg, bn, [&](auto BM_WG, auto BN) {
          return with_act(act, [&](auto ACT) {
            const int bytes = GemmPpCfg<BM_WG, BN>::SMEM_BYTES;
            SB_TRY(set_max_smem(gemm_pp_kernel<BM_WG, BN, EPI_FWD, ACT>, bytes));
            SB_TRY(set_max_smem(gemm_pp_kernel<BM_WG, BN, EPI_DA, ACT, true>, bytes));
            return set_max_smem(gemm_pp_kernel<BM_WG, BN, EPI_DA, ACT>, bytes);
          });
        }));
  return SB_OK;
}

}  // namespace sb
