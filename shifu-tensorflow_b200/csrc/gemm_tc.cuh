// wgmma / TMA dense-layer GEMM for sm_90a with fused epilogues.
//
//   D[M,N] = sum_k A(m,k) * B(n,k)      A, B bf16, fp32 accumulation in registers
//
// Each operand is consumed in the layout it already has in HBM - no transposed copies anywhere:
//   K-major  : element (r,k) at r*ld + k   (row-major [M|N, K]);  TMA box 64(K) x rows, wgmma K-major descriptor
//   MN-major : element (r,k) at k*ld + r   (row-major [K, M|N]);  TMA boxes 64(MN) x 64(K), wgmma MN-major descriptor
//
// One kernel covers every dense contraction of the tabular-DNN step (the TF ops behind nn_layer,
// res/ssgd_monitor.py:57-71, and their gradients built by opt.minimize, :142):
//   EPI_FWD : Z = A_{l-1} W_l        A K-major [rows,in], B = W_l [in,out] MN-major; +bias, activation -> A_l (bf16)
//   EPI_DA  : dA = dZ_l W_l^T        A K-major [rows,out], B = W_l [in,out] K-major; *act'(A_{l-1}) -> dZ_{l-1},
//                                    column sums -> db_{l-1}
//   EPI_DW  : dW_l = A_{l-1}^T dZ_l  A = A_{l-1} [rows,in] MN-major, B = dZ_l [rows,out] MN-major; split-K over the
//                                    batch, fp32 red.add into the flat gradient (128 x 256 tiles: gemm_dw.cuh)
//   EPI_F32 : plain fp32 store (kernel-level parity test hook)
// Here EPI_FWD / EPI_DA are the split-precision parts and the wide+deep addend (GENERIC); the plain-bf16 forward and dA
// GEMMs are gemm_pp.cuh, the last hidden GEMM of a training step with the output layer fused into its epilogue is
// gemm_fwd_out.cuh.
//
// Tile: one CTA owns 128 x BN (BN = 64 | 128).  Producer warpgroup, operand ring, main loop, kernel entry and exit:
// gemm_ring.cuh.  Warpgroup g multiplies rows 64 g .. 64 g + 63 of the tile with wgmma.m64nBNk16, then both run the
// epilogue while the producer runs ahead into the next tile.  The epilogue is written thread-owns-row: warp w takes the
// 32 rows of quarter w & 3 and every other 32-column chunk (parity w >> 2).  The accumulator reaches that layout through a
// padded 128 x 64 fp32 block in shared memory, one 64-column block at a time.
#pragma once
#include "gemm_ring.cuh"

namespace sb {

enum { EPI_FWD = 0, EPI_DA = 1, EPI_DW = 2, EPI_F32 = 3 };

// tensor maps of the parts of both operands (one kernel parameter, 768 B)
struct TmapSet {
  CUtensorMap a[3];
  CUtensorMap b[3];
};

// shared memory besides the ring: align slack, barriers, epilogue scratch, bias, per-warp transpose tiles (TR_BYTES),
// column-sum accumulators, accumulator block (ACC_BYTES)
template <int BN>
struct GemmTcCfg : RingCfg<128 * 64 * 2, BN * 64 * 2, 1024 + 256 + 2048 + 2048 + 8 * 2048 + 4096 + 128 * (64 + 4) * 4> {
  static_assert(BN == 64 || BN == 128, "tile N");
  static_assert(GemmTcCfg::STAGES >= 2, "operand ring");
  static constexpr int BM = 128;
  // accumulator staging block: 128 rows x 64 fp32 columns, rows padded by 16 B so that both the fragment stores and the
  // row-wise 16-byte loads are free of bank conflicts
  static constexpr int ACC_LD = 64 + 4;
  static constexpr int ACC_BYTES = BM * ACC_LD * 4;
  static constexpr int TR_BYTES = 8 * 2048;
  static constexpr int EPI_THREADS = 256;   // the two consumer warpgroups
};

// ---- epilogue element functions, specialised per activation so the switch is hoisted out of the element loop
template <int ACT>
__device__ __forceinline__ void epi_fwd_chunk(float (&v)[32], const float (&b)[32]) {
#pragma unroll
  for (int j = 0; j < 32; ++j) v[j] = act_apply(v[j] + b[j], ACT);
}
template <int ACT>
__device__ __forceinline__ void epi_da_chunk(float (&v)[32], const __nv_bfloat16* ah) {
#pragma unroll
  for (int j = 0; j < 32; ++j) v[j] *= act_grad_from_out(__bfloat162float(ah[j]), ACT);
}

// GENERIC = true adds the cold features at compile time: split-precision part stores / loads (np > 1) and the fp32 addend
// of the wide+deep first layer.  EPI_FWD / EPI_DA are instantiated with it only.
// DET (dA only, deterministic training): each epilogue warp stores its column sums into its own shared-memory slot
// (plain st.shared instead of red.shared), the 4 warps of a column are added in warp order, the tile's sums go to row
// tile tm of p.det_ws [tiles_m][N], and the CTA that arrives last adds the row tiles in order (common.cuh, det_last_cta).
template <int BN, int EPI, bool A_MN, bool B_MN, bool GENERIC = false, bool DET = false>
__global__ void __launch_bounds__(GemmTcCfg<BN>::THREADS, 1)
gemm_tc_kernel(const __grid_constant__ TmapSet tms, const GemmTcParams p) {
  static_assert(!DET || EPI == EPI_DA, "DET: dA column sums only");
  using Cfg = GemmTcCfg<BN>;
  const int act_sel = p.act;
  constexpr int BM = Cfg::BM, BK = Cfg::BK;

  extern __shared__ uint8_t smem_raw[];
  const Ring<Cfg> ring(smem_raw, Cfg::ACC_BYTES);
  const uint32_t accs_base = ring.end();            // accumulator staging block
  const uint32_t scratch = ring.bar(0) + 16u;

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
            if constexpr (A_MN) {
#pragma unroll
              for (int i = 0; i < BM / 64; ++i)  // 64(MN) x 64(K) boxes, 8 KB each, side by side along MN
                tma_load_2d(sa + i * 8192, tmA, fb, m0 + i * 64, kb * BK + a_row0);   // rows of the set = K here
            } else {
              tma_load_2d(sa, tmA, fb, kb * BK, m0 + a_row0);
            }
            if constexpr (B_MN) {
#pragma unroll
              for (int i = 0; i < BN / 64; ++i) tma_load_2d(sb + i * 8192, tmB, fb, n0 + i * 64, kb * BK);
            } else {
              tma_load_2d(sb, tmB, fb, kb * BK, n0);
            }
          });
          if (kbx == kb0 && w == w_first) ring_stamp(p, tracing, 3);  // first TMA issued
        }
      }
    }
    ring_producer_tail<Cfg>(p);
  } else {
    // ================= consumer warpgroups (warps 0..7): MMA, then the epilogue of the tile =================
    asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(Cfg::CONSUMER_REGS));
    const int wg = warp >> 2;                  // MMA: rows 64 wg .. 64 wg + 63 of the tile
    const int quarter = warp & 3;              // epilogue: rows 32 quarter .. 32 quarter + 31 of the tile
    const int half = (warp >> 2) & 1;          // epilogue: which of the two warps sharing the quarter (chunk parity)
    const int et = static_cast<int>(threadIdx.x);   // 0 .. EPI_THREADS-1 over all consumer warps
    constexpr int ET = Cfg::EPI_THREADS;
    auto bar_all = [&]() { asm volatile("bar.sync 1, %0;" ::"n"(Cfg::EPI_THREADS) : "memory"); };    // every consumer warp
    // EPI_FWD: the tile's bias staged in shared memory (broadcast ld.shared instead of dependent global loads)
    const uint32_t sm_vec = scratch + 2048u;   // [tile parity][bias BN floats]
    // Coalescing: the epilogue hands thread t the 32 columns of ROW t, so a direct 16-byte access per thread touches 32
    // different rows (32 L1 wavefronts per instruction).  Every global access of the epilogue therefore goes through a
    // warp-private 32 x 64 B tile in shared memory (16-byte pieces XOR-swizzled by row pair -> conflict-free on both
    // sides): on the global side lane l handles piece (l & 3) of rows 8 i + (l >> 2), i = 0..3, i.e. four lanes cover
    // 64 contiguous bytes of a row and one instruction touches 8 rows instead of 32.
    const uint32_t sm_stage = sm_vec + 2048u + static_cast<uint32_t>(warp) * 2048u;
    // Column sums (bias gradients) are accumulated per CTA in shared memory and flushed to the flat gradient ONCE per tile
    // and column: one red.global per column per 128 rows instead of one per 32 rows (with one red per warp and chunk, the
    // wide dA GEMMs wait on the L2 atomic units).
    // layout: [buffer (tile parity)][BN] floats; DET: [buffer][quarter][BN] (8 BN floats = the 4096 bytes at BN = 128)
    const uint32_t sm_col = sm_vec + 2048u + static_cast<uint32_t>(Cfg::TR_BYTES);
    static_assert(!DET || 8 * BN * 4 <= 4096, "DET column-sum slots");
    const int rt = quarter * 32 + lane;                                   // row of this thread inside the CTA's 128 rows
    auto col_slot = [&](int buf, int j) { return sm_col + static_cast<uint32_t>((buf * BN + j) * 4); };
    auto red_shared = [](uint32_t a, float v) { asm volatile("red.shared.add.f32 [%0], %1;" ::"r"(a), "f"(v) : "memory"); };
    if constexpr (EPI == EPI_DA && !DET) {
      for (int j = et; j < 2 * BN; j += ET) asm volatile("st.shared.f32 [%0], %1;" ::"r"(sm_col + static_cast<uint32_t>(j) * 4u), "f"(0.f) : "memory");
      bar_all();
    }
    // DET: after every epilogue warp has stored its sums of tile `it`: the 4 quarters in order, one slot store per column
    // into row tile tm_ of p.det_ws (every column < N of the tile is written by all 4 quarters, so no clearing is needed)
    auto flush_cols_det = [&](int it_, int tm_, int tn_) {
      bar_all();
      for (int j = et; j < BN; j += ET) {
        const int col = tn_ * BN + j;
        float vsum = 0.f;
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          float x;
          asm volatile("ld.shared.f32 %0, [%1];" : "=f"(x) : "r"(sm_col + static_cast<uint32_t>(((it_ & 1) * 4 + q) * BN + j) * 4u) : "memory");
          vsum += x;
        }
        if (col < p.N) p.det_ws[static_cast<size_t>(tm_) * p.N + col] = vsum;
      }
    };
    // after every epilogue warp has added its sums of tile `it`: one thread per column flushes and clears buffer it & 1
    auto flush_cols = [&](int it_, int tn_, float* dst) {
      bar_all();
      for (int j = et; j < BN; j += ET) {
        const int col = tn_ * BN + j;
        float vsum;
        asm volatile("ld.shared.f32 %0, [%1];" : "=f"(vsum) : "r"(col_slot(it_ & 1, j)) : "memory");
        asm volatile("st.shared.f32 [%0], %1;" ::"r"(col_slot(it_ & 1, j)), "f"(0.f) : "memory");
        if (col < p.N && vsum != 0.f) red_add_f32(dst + col, vsum);
      }
    };
    const int lrow = lane >> 2, lpc = lane & 3;
    auto stg = [&](int r, int pc) { return sm_stage + static_cast<uint32_t>(r) * 64u + static_cast<uint32_t>((pc ^ ((r >> 1) & 3)) << 4); };
    auto sts4 = [](uint32_t a, const uint4& v) {
      asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(a), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
    };
    auto lds4 = [](uint32_t a) {
      uint4 v;
      asm volatile("ld.shared.v4.b32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(a) : "memory");
      return v;
    };
    auto row_to_lanes = [&](const uint4 (&mine)[4], uint4 (&out)[4]) {   // thread-owns-row -> lane-coalesced
#pragma unroll
      for (int q = 0; q < 4; ++q) sts4(stg(lane, q), mine[q]);
      __syncwarp();
#pragma unroll
      for (int i = 0; i < 4; ++i) out[i] = lds4(stg(8 * i + lrow, lpc));
      __syncwarp();
    };
    auto lanes_to_row = [&](const uint4 (&in)[4], uint4 (&mine)[4]) {    // lane-coalesced -> thread-owns-row
#pragma unroll
      for (int i = 0; i < 4; ++i) sts4(stg(8 * i + lrow, lpc), in[i]);
      __syncwarp();
#pragma unroll
      for (int q = 0; q < 4; ++q) mine[q] = lds4(stg(lane, q));
      __syncwarp();
    };

    // ---- accumulator: registers of the wgmma fragment, handed to the epilogue one 64-column block at a time
    float acc_mi[1][BN / 2];
    float (&acc)[BN / 2] = acc_mi[0];
    // write columns 64 j .. 64 j + 63 of the fragment to the staging block (every consumer warp calls this together; the
    // first barrier waits for the readers of the previous block).  j selects among unrolled copies so that acc[] stays in
    // registers.
    auto stage_block = [&](int j) {
      bar_all();
      const int r0 = wg * 64 + (warp & 3) * 16 + (lane >> 2);
#pragma unroll
      for (int jj = 0; jj < BN / 64; ++jj) {
        if (jj == j) {
#pragma unroll
          for (int i = 0; i < 8; ++i) {
            const int n8 = jj * 8 + i;
            const uint32_t col = static_cast<uint32_t>(8 * i + 2 * (lane & 3));
            const uint32_t a0 = accs_base + (static_cast<uint32_t>(r0) * Cfg::ACC_LD + col) * 4u;
            const uint32_t a1 = a0 + 8u * Cfg::ACC_LD * 4u;
            asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(a0), "f"(acc[4 * n8]), "f"(acc[4 * n8 + 1]) : "memory");
            asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(a1), "f"(acc[4 * n8 + 2]), "f"(acc[4 * n8 + 3]) : "memory");
          }
        }
      }
      bar_all();
    };
    // chunk c (32 columns; its block c / 2 is staged): row rt of this thread
    auto acc_ld = [&](int c, uint32_t (&raw)[32]) {
      const uint32_t a = accs_base + (static_cast<uint32_t>(rt) * Cfg::ACC_LD + static_cast<uint32_t>((c & 1) * 32)) * 4u;
#pragma unroll
      for (int q = 0; q < 8; ++q)
        asm volatile("ld.shared.v4.b32 {%0, %1, %2, %3}, [%4];"
                     : "=r"(raw[4 * q]), "=r"(raw[4 * q + 1]), "=r"(raw[4 * q + 2]), "=r"(raw[4 * q + 3])
                     : "r"(a + 16u * q) : "memory");
    };

    // this warpgroup's 64 rows of the A stage: K-major = 64 rows of 128 B further; MN-major = the second 64-wide MN atom
    const uint32_t a_wg_off = static_cast<uint32_t>(wg) * 8192u;
    RingPos<Cfg::STAGES> pos;
    int it = 0;
    for (int w = w_first; w < n_work; w += gridDim.x, ++it) {
      const int tile = w % n_tiles, ks = w / n_tiles;
      const int tm = tile / tiles_n, tn = tile % tiles_n;
      const int kb0 = ks * p.kb_per_split;
      const int kb1 = min(total_kb, kb0 + p.kb_per_split);
      const int row = tm * BM + quarter * 32 + lane;  // output row of this thread
      const bool row_ok = row < p.M;
      // operands of the epilogue that do not depend on the accumulator are fetched BEFORE the main loop: the A_{l-1} tiles
      // of the dA epilogue
      // dA epilogue without TMA staging: A_{l-1} of EVERY chunk this warp will handle is fetched before the main loop and
      // kept in registers as a shift queue, so that one L2 / HBM latency is paid per tile instead of one per chunk
      constexpr int AUXQ = EPI == EPI_DA ? (BN / 64 > 0 ? BN / 64 : 1) : 1;
      uint4 aux_q[AUXQ][4];
      const int row_base = tm * BM + quarter * 32;   // first row of this warp's 32
      // store a 32 x 64 B tile held one-row-per-thread (4 pieces each) to a row-major bf16 matrix, coalesced
      auto store_rows_bf16 = [&](const uint4 (&mine)[4], __nv_bfloat16* base, int ld, int col0_, bool all_cols) {
        uint4 oc[4];
        row_to_lanes(mine, oc);
        const int gc = col0_ + 8 * lpc;
        if (all_cols || gc < ld) {
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            const int gr = row_base + 8 * i + lrow;
            if (gr < p.M) *reinterpret_cast<uint4*>(base + static_cast<size_t>(gr) * ld + gc) = oc[i];
          }
        }
      };
      // split-precision output: part 0 = bf16(v), part k = bf16(v - sum of the previous parts); np = 1 is the plain store.
      // x is left untouched (the residual of part k is re-derived from x: at most two extra cvt + sub per element).
      auto store_parts = [&](const float (&x)[32], __nv_bfloat16* base, long long ps, int ld, int col0_, bool all_cols) {
        const int np_ = GENERIC ? p.np : 1;
#pragma unroll 1
        for (int part = 0; part < np_; ++part) {
          auto res = [&](float r) {
            if constexpr (GENERIC) {
              for (int i = 0; i < part; ++i) r -= __bfloat162float(__float2bfloat16_rn(r));
            }
            return r;
          };
          uint4 o[4];
#pragma unroll
          for (int q = 0; q < 4; ++q) {
            o[q].x = pack_bf16x2(res(x[q * 8 + 0]), res(x[q * 8 + 1]));
            o[q].y = pack_bf16x2(res(x[q * 8 + 2]), res(x[q * 8 + 3]));
            o[q].z = pack_bf16x2(res(x[q * 8 + 4]), res(x[q * 8 + 5]));
            o[q].w = pack_bf16x2(res(x[q * 8 + 6]), res(x[q * 8 + 7]));
          }
          store_rows_bf16(o, base + part * ps, ld, col0_, all_cols);
        }
      };
      auto load_aux = [&](int c, uint4 (&a)[4], int part = 0) {   // lane-coalesced fetch of chunk c of A_{l-1}; zeros outside
#pragma unroll
        for (int i = 0; i < 4; ++i) a[i] = make_uint4(0, 0, 0, 0);
        const int gc = tn * BN + c * 32 + 8 * lpc;
        if (c < BN / 32 && tn * BN + c * 32 < p.N && gc < p.ld_aux) {
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            const int gr = row_base + 8 * i + lrow;
            if (gr < p.M) a[i] = __ldg(reinterpret_cast<const uint4*>(p.aux + part * p.aux_ps + static_cast<size_t>(gr) * p.ld_aux + gc));
          }
        }
      };
      if constexpr (EPI == EPI_DA) {
#pragma unroll
        for (int i = 0; i < AUXQ; ++i) load_aux(half + 2 * i, aux_q[i]);
      }
      // blocks of 64 columns this tile really has (the same number for every warp: the block loop contains barriers)
      const int tile_cols = (p.N - tn * BN) < BN ? (p.N - tn * BN) : BN;
      const int nblk = (tile_cols + 63) / 64;
      const uint32_t sm_bias = sm_vec + static_cast<uint32_t>(it & 1) * (BN * 4u);   // EPI_FWD: this tile's bias, double-buffered
      if constexpr (EPI == EPI_FWD) {
        // (a warp reaches this barrier only after finishing the previous tile, so buffer it & 1 is no longer read)
#pragma unroll
        for (int j = et; j < BN; j += ET) {
          const int col = tn * BN + j;
          const float bv = (col < p.N) ? __ldg(p.bias + col) : 0.f;
          asm volatile("st.shared.f32 [%0], %1;" ::"r"(sm_bias + static_cast<uint32_t>(j) * 4u), "f"(bv) : "memory");
        }
        bar_all();
      }

      ring_mma<BN, A_MN, B_MN>(ring, pos, kb1 - kb0, acc_mi, a_wg_off, 0u, (warp & 3) == 0 && lane == 0, w == w_first, p, tracing);

#pragma unroll 1
      for (int c = half; (c >> 1) < nblk; c += 2) {
        stage_block(c >> 1);
        const int col0 = tn * BN + c * 32;
        if (col0 >= p.N) continue;  // whole chunk out of range (warp-uniform)
        uint32_t raw[32];
        acc_ld(c, raw);
        float v[32];
#pragma unroll
        for (int j = 0; j < 32; ++j) v[j] = __uint_as_float(raw[j]);
        const bool full = col0 + 32 <= p.N;  // warp-uniform fast path

        if constexpr (EPI == EPI_FWD) {
          if (GENERIC && p.addend != nullptr && row_ok) {
            const float* ad = p.addend + static_cast<size_t>(row) * p.ld_add + col0;
            if (full && (p.ld_add & 3) == 0) {
#pragma unroll
              for (int q = 0; q < 8; ++q) {
                const float4 a4 = __ldg(reinterpret_cast<const float4*>(ad) + q);
                v[4 * q] += a4.x; v[4 * q + 1] += a4.y; v[4 * q + 2] += a4.z; v[4 * q + 3] += a4.w;
              }
            } else {
#pragma unroll
              for (int j = 0; j < 32; ++j)
                if (col0 + j < p.N) v[j] += __ldg(ad + j);
            }
          }
          float b[32];   // staged before the main loop (0 beyond N)
#pragma unroll
          for (int q = 0; q < 8; ++q)
            asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];"
                         : "=f"(b[4 * q]), "=f"(b[4 * q + 1]), "=f"(b[4 * q + 2]), "=f"(b[4 * q + 3])
                         : "r"(sm_bias + static_cast<uint32_t>(c * 32 + 4 * q) * 4u));
          switch (act_sel) {
            case SB_ACT_RELU: epi_fwd_chunk<SB_ACT_RELU>(v, b); break;
            case SB_ACT_SIGMOID: epi_fwd_chunk<SB_ACT_SIGMOID>(v, b); break;
            case SB_ACT_TANH: epi_fwd_chunk<SB_ACT_TANH>(v, b); break;
            case SB_ACT_LEAKYRELU: epi_fwd_chunk<SB_ACT_LEAKYRELU>(v, b); break;
            default: epi_fwd_chunk<SB_ACT_NONE>(v, b); break;
          }
        } else if constexpr (EPI == EPI_DA) {
          // multiply by act'(A_{l-1}[row, col]) read as bf16
          uint4 a4[4];
          lanes_to_row(aux_q[0], a4);
#pragma unroll
          for (int i = 0; i + 1 < AUXQ; ++i) {
#pragma unroll
            for (int k = 0; k < 4; ++k) aux_q[i][k] = aux_q[i + 1][k];
          }
          __nv_bfloat16* ah = reinterpret_cast<__nv_bfloat16*>(a4);
          if (GENERIC && p.np > 1 && (act_sel == SB_ACT_SIGMOID || act_sel == SB_ACT_TANH)) {
            // act' needs the VALUE of A_{l-1}: add the lower parts (fetched here, not prefetched: the split modes are the
            // parity modes).  relu / leaky relu only look at the sign, which part 0 carries.
            float af[32];
#pragma unroll
            for (int j = 0; j < 32; ++j) af[j] = __bfloat162float(ah[j]);
            for (int part = 1; part < p.np; ++part) {
              uint4 lo_l[4], lo_r[4];
              load_aux(c, lo_l, part);
              lanes_to_row(lo_l, lo_r);
              const __nv_bfloat16* lh = reinterpret_cast<const __nv_bfloat16*>(lo_r);
#pragma unroll
              for (int j = 0; j < 32; ++j) af[j] += __bfloat162float(lh[j]);
            }
#pragma unroll
            for (int j = 0; j < 32; ++j) v[j] *= act_grad_from_out(af[j], act_sel);
          } else
          switch (act_sel) {
            case SB_ACT_RELU: epi_da_chunk<SB_ACT_RELU>(v, ah); break;
            case SB_ACT_SIGMOID: epi_da_chunk<SB_ACT_SIGMOID>(v, ah); break;
            case SB_ACT_TANH: epi_da_chunk<SB_ACT_TANH>(v, ah); break;
            case SB_ACT_LEAKYRELU: epi_da_chunk<SB_ACT_LEAKYRELU>(v, ah); break;
            default: break;
          }
          if (!row_ok || !full) {
#pragma unroll
            for (int j = 0; j < 32; ++j)
              if (!row_ok || col0 + j >= p.N) v[j] = 0.f;
          }
        }

        if constexpr (EPI == EPI_FWD || EPI == EPI_DA) {
          // row-major bf16 (ld_out is a multiple of 8, pad columns belong to the buffer); split modes: np part arrays
          store_parts(v, p.out, p.out_ps, p.ld_out, col0, full);
          if constexpr (EPI == EPI_DA) {
            if (p.colsum != nullptr) {
              // bias gradient: per-column sum over this warp's 32 rows, accumulated per CTA in shared memory
              const float s = warp_colsum_32x32(v, lane);
              if constexpr (DET)   // this warp's own slot: one writer per address
                asm volatile("st.shared.f32 [%0], %1;" ::"r"(sm_col + static_cast<uint32_t>(((it & 1) * 4 + quarter) * BN + c * 32 + lane) * 4u),
                             "f"(s) : "memory");
              else
                red_shared(col_slot(it & 1, c * 32 + lane), s);     // columns beyond N / rows beyond M were zeroed above
            }
          }
        } else if constexpr (EPI == EPI_DW) {
          if (p.acc_vec4 && full) {
            // fp32 rows are 128 B per 32-column chunk: two 64-byte halves through the transpose tile, then
            // red.global.add.v4.f32 with four lanes per 64 contiguous bytes
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              uint4 mine[4], oc[4];
#pragma unroll
              for (int q = 0; q < 4; ++q)
                mine[q] = make_uint4(__float_as_uint(v[16 * h + 4 * q]), __float_as_uint(v[16 * h + 4 * q + 1]),
                                     __float_as_uint(v[16 * h + 4 * q + 2]), __float_as_uint(v[16 * h + 4 * q + 3]));
              row_to_lanes(mine, oc);
#pragma unroll
              for (int i = 0; i < 4; ++i) {
                const int gr = row_base + 8 * i + lrow;
                if (gr < p.M)
                  red_add_v4_f32(p.accum + static_cast<size_t>(gr) * p.ld_acc + col0 + 16 * h + 4 * lpc, __uint_as_float(oc[i].x),
                                 __uint_as_float(oc[i].y), __uint_as_float(oc[i].z), __uint_as_float(oc[i].w));
              }
            }
          } else if (row_ok) {
            float* gp = p.accum + static_cast<size_t>(row) * p.ld_acc + col0;
#pragma unroll
            for (int j = 0; j < 32; ++j)
              if (col0 + j < p.N) red_add_f32(gp + j, v[j]);
          }
        } else {  // EPI_F32
          if (row_ok) {
            float* gp = p.accum + static_cast<size_t>(row) * p.ld_acc + col0;
            if (p.split_k == 1) {
#pragma unroll
              for (int j = 0; j < 32; ++j)
                if (col0 + j < p.N) gp[j] = v[j];
            } else {
#pragma unroll
              for (int j = 0; j < 32; ++j)
                if (col0 + j < p.N) red_add_f32(gp + j, v[j]);
            }
          }
        }
      }
      if constexpr (DET) {
        if (p.colsum != nullptr) flush_cols_det(it, tm, tn);
      } else if constexpr (EPI == EPI_DA) {
        if (p.colsum != nullptr) flush_cols(it, tn, p.colsum);
      }
      if (w == w_first && threadIdx.x == 0) ring_stamp(p, tracing, 7);  // first tile's epilogue done
    }
    if constexpr (DET) {
      // (named barrier 1 = every consumer warp; dA runs without split-K, so the work items are the tiles)
      if (p.colsum != nullptr) det_colsum_tail(p.det_ticket, p.det_ws, (p.M + BM - 1) / BM, p.N, p.colsum, 1, ET, et);
    }
  }
  ring_exit(p, tracing);
}

// ------------------------------------------------------------------ host side
typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
PFN_encodeTiled get_encode_tiled();

// Tensor map of a row-major bf16 matrix [rows, cols] with leading dimension ld (elements):
// box = 64 columns x box_rows rows, 128-byte swizzle.  cols/rows are the LOGICAL extents (TMA zero-fills beyond
// them), ld*2 must be a multiple of 16 bytes.  K-major operand: box_rows = rows one CTA stages (128 for A,
// BN for B); MN-major operand: 64.
int make_tmap_bf16(CUtensorMap* out, const void* base, int rows, int cols, int ld, int box_rows);
// the same map for each of np part arrays that lie part_stride ELEMENTS apart (np = 1: just the one)
int make_tmaps_bf16(CUtensorMap* out3, const void* base, long long part_stride, int np, int rows, int cols, int ld, int box_rows);
// fills n_pairs / pair_a / pair_b of p for np parts per operand
void set_part_pairs(GemmTcParams* p, int np);

// Tile configuration chosen per problem.
struct GemmPlan {
  int bn;            // 64 / 128; 256 for dW GEMMs only (gemm_dw.cuh)
  int split_k, kb_per_split;
  int grid;          // CTAs to launch
};
// max_split > 0 caps the split-K factor (deterministic training: 2, see Net::enqueue_dw)
GemmPlan plan_gemm(int M, int N, int K, int num_sms, bool allow_split, int max_split = 0);

template <int EPI, bool A_MN, bool B_MN>
int launch_gemm_tc(const GemmPlan& pl, const TmapSet& tms, GemmTcParams p, cudaStream_t st, bool pdl = false) {
  if (p.np < 1) p.np = 1;
  if (p.n_pairs < 1) p.n_pairs = 1;
  p.split_k = pl.split_k;
  p.kb_per_split = pl.kb_per_split;
  // forward / dA: split-precision parts or an fp32 addend, the GENERIC instantiations (plain bf16 is gemm_pp.cuh)
  constexpr bool GENERIC = EPI == EPI_FWD || EPI == EPI_DA;
  if constexpr (EPI == EPI_DA) {
    if (p.det_ws != nullptr) {   // deterministic training: p.det_ws holds [ceil(M / 128)][N] floats
      if (pl.bn == 64)
        return launch_kernel(gemm_tc_kernel<64, EPI, A_MN, B_MN, true, true>, pl.grid, GemmTcCfg<64>::THREADS,
                             GemmTcCfg<64>::SMEM_BYTES, st, pdl, tms, p);
      if (pl.bn == 128)
        return launch_kernel(gemm_tc_kernel<128, EPI, A_MN, B_MN, true, true>, pl.grid, GemmTcCfg<128>::THREADS,
                             GemmTcCfg<128>::SMEM_BYTES, st, pdl, tms, p);
      return set_error(SB_ERR_INVALID, "no gemm_tc instantiation for bn=%d", pl.bn);
    }
  }
  if (pl.bn == 64)
    return launch_kernel(gemm_tc_kernel<64, EPI, A_MN, B_MN, GENERIC>, pl.grid, GemmTcCfg<64>::THREADS, GemmTcCfg<64>::SMEM_BYTES,
                         st, pdl, tms, p);
  if (pl.bn == 128)
    return launch_kernel(gemm_tc_kernel<128, EPI, A_MN, B_MN, GENERIC>, pl.grid, GemmTcCfg<128>::THREADS,
                         GemmTcCfg<128>::SMEM_BYTES, st, pdl, tms, p);
  return set_error(SB_ERR_INVALID, "no gemm_tc instantiation for bn=%d", pl.bn);
}

// opt in to > 48 KB dynamic shared memory (once per process per instantiation, outside of stream capture)
template <int EPI, bool A_MN, bool B_MN>
int set_gemm_tc_attrs() {
  constexpr bool GENERIC = EPI == EPI_FWD || EPI == EPI_DA;
  if constexpr (EPI == EPI_DA) {
    SB_TRY((set_max_smem(gemm_tc_kernel<64, EPI, A_MN, B_MN, true, true>, GemmTcCfg<64>::SMEM_BYTES)));
    SB_TRY((set_max_smem(gemm_tc_kernel<128, EPI, A_MN, B_MN, true, true>, GemmTcCfg<128>::SMEM_BYTES)));
  }
  SB_TRY(set_max_smem(gemm_tc_kernel<64, EPI, A_MN, B_MN, GENERIC>, GemmTcCfg<64>::SMEM_BYTES));
  return set_max_smem(gemm_tc_kernel<128, EPI, A_MN, B_MN, GENERIC>, GemmTcCfg<128>::SMEM_BYTES);
}

}  // namespace sb
