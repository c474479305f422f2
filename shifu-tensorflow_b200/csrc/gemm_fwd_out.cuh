// Last hidden layer of a TRAINING step with the output layer fused into its epilogue (K2 + K3 + K4 + output backward in
// one kernel, res/ssgd_monitor.py:121,129; h_L = N <= 256, so one CTA holds whole rows of A_L):
//   a     = act(A_{L-1} W_L + b_L)                 fp32, never rounded, never leaves the registers
//   z     = a . w_o + b_o,  y_hat = sigmoid(z),  loss term,  dz
//   dZ_L  = dz * w_o * act'(a)  -> bf16 (or its split-precision parts), by TMA store
//   db_L / dw_o column sums, db_o and the loss sum by atomics into the flat gradient / the step scalars
//
// Tile: 64 rows x BN (BN = 64 | 128 | 256 >= N).  The 64-row tile puts twice as many CTAs on the machine as a 128-row one
// (cfg2: 128 of 132 SMs at 8192 rows), and the two consumer warpgroups split N instead of M: warpgroup g multiplies the
// same 64 rows against columns g BN/2 .. g BN/2 + BN/2 - 1 with wgmma.m64n(BN/2)k16, so its accumulator is BN/4 registers
// per thread (64 at BN = 256).  The epilogue runs in the wgmma fragment layout itself - no fp32 staging through shared
// memory: thread (warp w of the group, lane l) holds rows 16 w + l/4 and +8 at the column pairs 8 i + 2 (l % 4).
//   row dot products  : per-thread partials, shuffle over the 4 lanes of a row, the two warpgroups' halves through shared
//                       memory (one consumer barrier)
//   column sums       : each thread adds its two rows, a reduce-scatter over the 8 row groups of the warp (3 shuffle
//                       rounds that halve the data each time), red.shared into the warp's own slots; the 4 slots are
//                       added in a fixed order and flushed to the flat gradient once per CTA (as are the loss sum and
//                       db_o), so a step's result does not depend on warp timing
//   dZ_L              : bf16 pairs into BN/64 128-byte-swizzled 64 x 64 tiles (the output tensor map's layout; conflict
//                       free for the fragment), one cp.async.bulk.tensor store per tile
// Producer warpgroup, operand ring, main loop, kernel entry and exit: gemm_ring.cuh.
#pragma once
#include "gemm_tc.cuh"

namespace sb {

// tensor maps of the split-precision parts (np = 1: index 0 only); one kernel parameter of 1152 B
struct FwdOutTmaps {
  CUtensorMap a[3];   // A_{L-1} [rows, K] K-major: box 64 (K) x 64 rows
  CUtensorMap b[3];   // W_L [K, N] MN-major: box 64 (N) x 64 (K)
  CUtensorMap o[3];   // dZ_L [rows, N]: box 64 columns x 64 rows (store)
};

// widest tile: the widest last hidden layer whose GEMM also runs the output layer
constexpr int FWD_OUT_MAX_N = 256;

// besides the ring: align slack, barriers, bias + w_o, the two column-sum arrays per warp of a group, z partials
// [tile parity][group][64], loss / db_o per warp of group 0, dZ_L staging tiles (X_BYTES)
template <int BN>
struct FwdOutCfg : RingCfg<64 * 64 * 2, BN * 64 * 2, 1024 + 256 + 2 * BN * 4 + 4 * 2 * BN * 4 + 2 * 2 * 64 * 4 + 32 + 64 * BN * 2> {
  static_assert(BN == 64 || BN == 128 || BN == 256, "tile N");
  static_assert(FwdOutCfg::STAGES >= 4, "operand ring");
  static constexpr int BM = 64;
  static constexpr int WN = BN / 2;                 // columns of one consumer warpgroup
  static constexpr int X_BYTES = BM * BN * 2;       // dZ_L staging tiles
  static constexpr int EPI_THREADS = 256;           // the two consumer warpgroups
};

// DET: the CTA's loss sum, db_o, db_L and dw_o go to its slots of p.det_ws (common.cuh, det_out_finish with halves = 1)
// and the CTA that arrives last adds the CTAs in ascending order
template <int BN, int ACT, bool DET = false>
__global__ void __launch_bounds__(FwdOutCfg<BN>::THREADS, 1)
gemm_fwd_out_kernel(const __grid_constant__ FwdOutTmaps tms, const GemmTcParams p) {
  using Cfg = FwdOutCfg<BN>;
  constexpr int BM = Cfg::BM, BK = Cfg::BK, WN = Cfg::WN;

  extern __shared__ uint8_t smem_raw[];
  const Ring<Cfg> ring(smem_raw, Cfg::X_BYTES);
  const uint32_t xs_base = ring.end();                                // dZ_L staging tiles (1024-byte aligned)
  const uint32_t sm_vec = ring.bars + 256u;                           // [bias BN][w_o BN] fp32, 0 beyond N
  const uint32_t sm_col = sm_vec + 2u * BN * 4u;                      // [warp & 3][db_L BN][dw_o BN] fp32 column sums
  const uint32_t sm_z = sm_col + 4u * 2u * BN * 4u;                   // z partials [tile parity][group][64 rows]
  const uint32_t sm_lw = sm_z + 2u * 2u * BM * 4u;                    // [warp][loss, db_o] of group 0

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const bool tracing = ring_enter(ring, 2, 0, &tms.a[0], &tms.b[0], p);   // one empty arrival per consumer warpgroup

  const int np = p.np > 0 ? p.np : 1;
  const int n_pairs = p.n_pairs > 0 ? p.n_pairs : 1;
  const int tiles = (p.M + BM - 1) / BM;
  const int part_kb = (p.K + BK - 1) / BK;         // k-blocks of ONE part pair
  const int total_kb = part_kb * n_pairs;          // extended K axis: the pairs one after the other

  if (warp >= Cfg::PRODUCER_WARP) {
    asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(Cfg::PRODUCER_REGS));
    if (warp == Cfg::PRODUCER_WARP && lane == 0) {
      RingPos<Cfg::STAGES> pos;
      const int a_row0 = (p.a_rows != nullptr) ? p.a_rows->row0 : 0;  // batch position inside the resident set
      for (int t = blockIdx.x; t < tiles; t += gridDim.x) {
        for (int kbx = 0; kbx < total_kb; ++kbx) {
          const int pp = (n_pairs > 1) ? kbx / part_kb : 0;     // which part pair this k-block belongs to
          const int kb = kbx - pp * part_kb;
          const CUtensorMap* tmA = &tms.a[n_pairs > 1 ? p.pair_a[pp] : 0];
          const CUtensorMap* tmB = &tms.b[n_pairs > 1 ? p.pair_b[pp] : 0];
          ring_issue(ring, pos, [&](uint32_t fb, uint32_t sa, uint32_t sb) {
            tma_load_2d(sa, tmA, fb, kb * BK, t * BM + a_row0);
#pragma unroll
            for (int j = 0; j < BN / 64; ++j) tma_load_2d(sb + j * 8192, tmB, fb, j * 64, kb * BK);
          });
          if (kbx == 0 && t == static_cast<int>(blockIdx.x)) ring_stamp(p, tracing, 3);  // first TMA issued
        }
      }
    }
    ring_producer_tail<Cfg>(p);
  } else {
    // ================= consumer warpgroups (warps 0..7): MMA, then the fused epilogue of the tile =================
    asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(Cfg::CONSUMER_REGS));
    const int wg = warp >> 2;                 // columns wg WN .. wg WN + WN - 1 of the tile
    const int et = static_cast<int>(threadIdx.x);
    auto bar_all = [&]() { asm volatile("bar.sync 1, %0;" ::"n"(Cfg::EPI_THREADS) : "memory"); };
    const bool xthread = (warp == 0 && lane == 0);   // issues the dZ_L stores
    auto lds = [](uint32_t a) { float v; asm volatile("ld.shared.f32 %0, [%1];" : "=f"(v) : "r"(a) : "memory"); return v; };
    auto lds2 = [](uint32_t a) {
      float2 v;
      asm volatile("ld.shared.v2.f32 {%0, %1}, [%2];" : "=f"(v.x), "=f"(v.y) : "r"(a) : "memory");
      return v;
    };
    auto sts = [](uint32_t a, float v) { asm volatile("st.shared.f32 [%0], %1;" ::"r"(a), "f"(v) : "memory"); };
    // bias and w_o staged once (broadcast ld.shared in the epilogue), column sums cleared
    for (int j = et; j < 2 * BN; j += Cfg::EPI_THREADS) {
      const int col = j < BN ? j : j - BN;
      const float* src = j < BN ? p.bias : p.wo;
      sts(sm_vec + static_cast<uint32_t>(j) * 4u, col < p.N ? __ldg(src + col) : 0.f);
    }
    for (int j = et; j < 4 * 2 * BN; j += Cfg::EPI_THREADS) sts(sm_col + static_cast<uint32_t>(j) * 4u, 0.f);
    bar_all();
    const float b_o = __ldg(p.bo);
    const float nnz = p.scal[SCAL_NNZ];
    const float inv_nnz = nnz > 0.f ? 1.f / nnz : 0.f;
    float loss_acc = 0.f, dz_acc = 0.f;   // this warp's loss / db_o contributions over all its tiles (group 0 only)

    // fragment: rows r0 = 16 (warp & 3) + lane / 4 and r0 + 8; n8 block i holds columns c0 + 8 i + {0, 1}
    const int r0 = (warp & 3) * 16 + (lane >> 2);
    const int c0 = wg * WN + 2 * (lane & 3);
    float acc_mi[1][WN / 2];
    float (&acc)[WN / 2] = acc_mi[0];
    // This group's B columns: the next 64-wide MN atom(s), or for WN = 32 the second half of the 128-byte swizzle rows
    // (the swizzle is a function of the address, so a start 64 B into the row reads columns 32..63).
    const uint32_t b_wg_off = WN >= 64 ? static_cast<uint32_t>(wg) * (WN / 64) * 8192u : static_cast<uint32_t>(wg) * 64u;
    RingPos<Cfg::STAGES> pos;
    int it = 0;
    for (int t = blockIdx.x; t < tiles; t += gridDim.x, ++it) {
      const int row0 = t * BM + r0, row1 = row0 + 8;
      const bool ok0 = row0 < p.M, ok1 = row1 < p.M;
      // per-row label / weight fetched before the main loop
      const float y0 = ok0 ? __ldg(p.desc->y + row0) : 0.f, w0 = ok0 ? __ldg(p.desc->w + row0) : 0.f;
      const float y1 = ok1 ? __ldg(p.desc->y + row1) : 0.f, w1 = ok1 ? __ldg(p.desc->w + row1) : 0.f;

      ring_mma<WN, false, true>(ring, pos, total_kb, acc_mi, 0u, b_wg_off, (warp & 3) == 0 && lane == 0, it == 0, p, tracing);

      // ---------- (1) a = act(acc + bias), 0 beyond N;  (2) row partials of a . w_o ----------
      float zp0 = 0.f, zp1 = 0.f;
#pragma unroll
      for (int i = 0; i < WN / 8; ++i) {
        const int c = c0 + 8 * i;
        const float2 b = lds2(sm_vec + static_cast<uint32_t>(c) * 4u);
        const float2 wo = lds2(sm_vec + static_cast<uint32_t>(BN + c) * 4u);
        acc[4 * i + 0] = act_apply(acc[4 * i + 0] + b.x, ACT);
        acc[4 * i + 1] = act_apply(acc[4 * i + 1] + b.y, ACT);
        acc[4 * i + 2] = act_apply(acc[4 * i + 2] + b.x, ACT);
        acc[4 * i + 3] = act_apply(acc[4 * i + 3] + b.y, ACT);
        if (p.N < BN) {
          if (c >= p.N) { acc[4 * i + 0] = 0.f; acc[4 * i + 2] = 0.f; }
          if (c + 1 >= p.N) { acc[4 * i + 1] = 0.f; acc[4 * i + 3] = 0.f; }
        }
        zp0 = fmaf(acc[4 * i + 0], wo.x, zp0); zp0 = fmaf(acc[4 * i + 1], wo.y, zp0);
        zp1 = fmaf(acc[4 * i + 2], wo.x, zp1); zp1 = fmaf(acc[4 * i + 3], wo.y, zp1);
      }
#pragma unroll
      for (int m = 1; m <= 2; m <<= 1) {
        zp0 += __shfl_xor_sync(0xffffffffu, zp0, m);
        zp1 += __shfl_xor_sync(0xffffffffu, zp1, m);
      }
      const uint32_t zs = sm_z + static_cast<uint32_t>(it & 1) * (2u * BM * 4u);   // [group][64]
      if ((lane & 3) == 0) {
        sts(zs + static_cast<uint32_t>(wg * BM + r0) * 4u, zp0);
        sts(zs + static_cast<uint32_t>(wg * BM + r0 + 8) * 4u, zp1);
      }
      if (xthread) tma_store_wait_read<0>();   // the previous tile's dZ_L stores have read the staging tiles
      bar_all();
      const float z0 = lds(zs + static_cast<uint32_t>(r0) * 4u) + lds(zs + static_cast<uint32_t>(BM + r0) * 4u) + b_o;
      const float z1 = lds(zs + static_cast<uint32_t>(r0 + 8) * 4u) + lds(zs + static_cast<uint32_t>(BM + r0 + 8) * 4u) + b_o;

      // ---------- (3) per row: y_hat, loss term, dz (a rolled loop over the two rows: one copy of the code) ----------
      float dz0 = 0.f, dz1 = 0.f;
#pragma unroll 1
      for (int h = 0; h < 2; ++h) {
        const float z = h ? z1 : z0, y = h ? y1 : y0, wgt = h ? w1 : w0;
        float dz = 0.f, lossv = 0.f;
        if (h ? ok1 : ok0) {
          const float yh = sigmoidf_stable(z);
          if (p.loss == SB_LOSS_MSE) {
            const float d = yh - y;
            lossv = wgt * d * d;
            dz = 2.f * wgt * d * yh * (1.f - yh) * inv_nnz;
          } else {
            lossv = wgt * (fmaxf(z, 0.f) - z * y + log1pf(expf(-fabsf(z))));
            dz = wgt * (yh - y) * inv_nnz;
          }
        }
        if (h) dz1 = dz; else dz0 = dz;
        if (wg == 0 && (lane & 3) == 0) { loss_acc += lossv; dz_acc += dz; }   // each row once
      }

      // ---------- (4) g = dz w_o act'(a) (replaces a in acc), column sums of g and dz a over the two rows ----------
      float sdb[WN / 4], sdw[WN / 4];
#pragma unroll
      for (int i = 0; i < WN / 8; ++i) {
        const float2 wo = lds2(sm_vec + static_cast<uint32_t>(BN + c0 + 8 * i) * 4u);
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const float w = e ? wo.y : wo.x;
          const float a0 = acc[4 * i + e], a1 = acc[4 * i + 2 + e];
          const float g0 = dz0 * w * act_grad_from_out(a0, ACT);
          const float g1 = dz1 * w * act_grad_from_out(a1, ACT);
          sdb[2 * i + e] = g0 + g1;
          sdw[2 * i + e] = a0 * dz0 + a1 * dz1;
          acc[4 * i + e] = g0;
          acc[4 * i + 2 + e] = g1;
        }
      }
      // ---------- (5) over the warp's 16 rows, then into the warp's slots (one writer per address) ----------
      colsum_row_groups(sdb, lane);
      colsum_row_groups(sdw, lane);
      const uint32_t cw = sm_col + static_cast<uint32_t>(warp & 3) * 2u * BN * 4u;
#pragma unroll
      for (int j = 0; j < WN / 32; ++j) {
        const int k = (lane >> 2) * (WN / 32) + j;   // value index 2 i + e of the thread's columns
        const uint32_t col = static_cast<uint32_t>(c0 + 8 * (k >> 1) + (k & 1));
        asm volatile("red.shared.add.f32 [%0], %1;" ::"r"(cw + col * 4u), "f"(sdb[j]) : "memory");
        asm volatile("red.shared.add.f32 [%0], %1;" ::"r"(cw + (BN + col) * 4u), "f"(sdw[j]) : "memory");
      }

      // ---------- (6) dZ_L: bf16, TMA store.  Split modes: part k = bf16 of the residual after parts 0..k-1 (acc keeps
      //            the residual) ----------
#pragma unroll 1
      for (int part = 0; part < np; ++part) {
        if (part > 0) {
#pragma unroll
          for (int j = 0; j < WN / 2; ++j) acc[j] -= __bfloat162float(__float2bfloat16_rn(acc[j]));
          if (xthread) tma_store_wait_read<0>();   // the previous part's stores have read the staging tiles
          bar_all();
        }
#pragma unroll
        for (int i = 0; i < WN / 8; ++i) {
          const int c = c0 + 8 * i;   // tile column; 64 x 64 tile c / 64, 16-byte piece (c % 64) / 8, swizzled by row
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int r = r0 + 8 * h;
            const uint32_t a = xs_base + static_cast<uint32_t>((c >> 6) * 8192 + r * 128 + ((((c & 63) >> 3) ^ (r & 7)) << 4) + (c & 7) * 2);
            asm volatile("st.shared.b32 [%0], %1;" ::"r"(a), "r"(pack_bf16x2(acc[4 * i + 2 * h], acc[4 * i + 2 * h + 1])) : "memory");
          }
        }
        fence_proxy_async();   // generic-proxy writes -> visible to the TMA engine
        bar_all();
        if (xthread) {
#pragma unroll
          for (int x = 0; x < BN / 64; ++x)
            if (x * 64 < p.N) tma_store_2d(&tms.o[part], xs_base + x * 8192, x * 64, t * BM);
          tma_store_commit();
        }
      }
      if (it == 0 && threadIdx.x == 0) ring_stamp(p, tracing, 7);  // first tile's epilogue done
    }
    // loss sum and db_o: one atomic pair per CTA; db_L / dw_o: one red.global per column and CTA (warps added in order)
    if (wg == 0) {
      const float ls = warp_sum(loss_acc), ds = warp_sum(dz_acc);
      if (lane == 0) { sts(sm_lw + warp * 8u, ls); sts(sm_lw + warp * 8u + 4u, ds); }
    }
    bar_all();
    if (et == 0) {
      float ls = 0.f, ds = 0.f;
      for (int w = 0; w < 4; ++w) { ls += lds(sm_lw + w * 8u); ds += lds(sm_lw + w * 8u + 4u); }
      if constexpr (DET) {
        float* slots = p.det_ws + blockIdx.x * det_out_stride(p.N, 1);
        slots[0] = ls;
        slots[1] = ds;
      } else {
        atomicAdd(p.scal + SCAL_LOSS_SUM, ls);
        atomicAdd(p.g_bo, ds);
      }
    }
    for (int j = et; j < BN && j < p.N; j += Cfg::EPI_THREADS) {
      float db = 0.f, dw = 0.f;
      for (int w = 0; w < 4; ++w) {
        db += lds(sm_col + static_cast<uint32_t>(w * 2 * BN + j) * 4u);
        dw += lds(sm_col + static_cast<uint32_t>(w * 2 * BN + BN + j) * 4u);
      }
      if constexpr (DET) {
        float* slots = p.det_ws + blockIdx.x * det_out_stride(p.N, 1);
        slots[2 + j] = db;
        slots[2 + p.N + j] = dw;
      } else {
        if (db != 0.f) red_add_f32(p.g_bL + j, db);
        if (dw != 0.f) red_add_f32(p.g_wo + j, dw);
      }
    }
    if constexpr (DET) {
      if (det_last_cta(p.det_ticket, gridDim.x, 1, Cfg::EPI_THREADS, et == 0))
        det_out_finish(p.det_ws, static_cast<int>(gridDim.x), p.N, 1, true, true, p.scal + SCAL_LOSS_SUM, p.g_bo, p.g_bL, p.g_wo, et,
                       Cfg::EPI_THREADS);
    }
    if (xthread) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");   // the last tiles are in global memory
  }
  ring_exit(p, tracing);
}

// ------------------------------------------------------------------ host side
// f(integral_constant BN): the narrowest tile that holds a whole row of A_L (N <= 256); one CTA per SM and 64-row tile
template <typename F>
static int with_fwd_out_bn(int N, F&& f) {
  SB_CHECK(N <= FWD_OUT_MAX_N, SB_ERR_INVALID, "fused output layer: last hidden layer %d wider than %d", N, FWD_OUT_MAX_N);
  if (N <= 64) return f(std::integral_constant<int, 64>());
  if (N <= 128) return f(std::integral_constant<int, 128>());
  return f(std::integral_constant<int, 256>());
}

static int launch_gemm_fwd_out(int grid, const FwdOutTmaps& tms, const GemmTcParams& p, cudaStream_t st, bool pdl) {
  return with_fwd_out_bn(p.N, [&](auto BN) {
    return with_act(p.act, [&](auto ACT) {
      if (p.det_ws != nullptr)   // DET: p.det_ws holds grid x (2 + 2 N) floats
        return launch_kernel(gemm_fwd_out_kernel<BN, ACT, true>, grid, FwdOutCfg<BN>::THREADS, FwdOutCfg<BN>::SMEM_BYTES, st, pdl, tms, p);
      return launch_kernel(gemm_fwd_out_kernel<BN, ACT>, grid, FwdOutCfg<BN>::THREADS, FwdOutCfg<BN>::SMEM_BYTES, st, pdl, tms, p);
    });
  });
}

// opt in to > 48 KB dynamic shared memory (once per process, outside of stream capture)
static int set_gemm_fwd_out_attrs() {
  for (int n : {64, 128, 256})
    for (int act = SB_ACT_NONE; act <= SB_ACT_LEAKYRELU; ++act)
      SB_TRY(with_fwd_out_bn(n, [&](auto BN) {
        return with_act(act, [&](auto ACT) {
          SB_TRY(set_max_smem(gemm_fwd_out_kernel<BN, ACT, true>, FwdOutCfg<BN>::SMEM_BYTES));
          return set_max_smem(gemm_fwd_out_kernel<BN, ACT>, FwdOutCfg<BN>::SMEM_BYTES);
        });
      }));
  return SB_OK;
}

}  // namespace sb
