// Column sensitivity (sb_model_sensitivity, DESIGN §6f): how far a model's score moves when one input column is replaced
// by a value.  Replacing column c of a row changes one term of layer 0's pre-activation,
//   z0' = z0 + (v - x_c) W0[c, :],
// so z0 is computed once per row and every (row, column) pair is a rank-1 update of it followed by layers 1..L.
//
// A piece of pair rows is column-major: pair p = slot * R + r (R = the piece's rows), slot 0 = the base slot (the row
// itself, delta 0), slot k + 1 = list position k0 + k of the piece.  The base slot's score comes out of the same launches
// as the perturbed scores, so a pair whose column already holds the value gets exactly the base row's score.
//   sens_perturb_kernel  z0 (fp32, [R, ld_z]) -> A0' of every pair, stored as layer 0's forward epilogue stores A0
//   sens_reduce_kernel   the pair scores -> d = s(base) - s(pair) per (row, column), and the fp64 sums of w d^2 and w d
//   sens_topk_kernel     the pair scores -> each row's running top k of d (sb_model_reason_codes, DESIGN §6g)
#pragma once
#include "common.cuh"
#include "kernels.cuh"

namespace sb {

struct SensParams {
  int R;                       // rows of the piece (= of its row chunk)
  int F;                       // columns of X
  int N, ld;                   // layer 0's width and the row pitch of z0 and of A0' (tensor-core modes; fp32 A0' is dense)
  const float* X;              // [R, F] fp32 rows as staged for layer 0
  const float* z;              // [R, ld] fp32 pre-activations (without the bias in tensor-core modes)
  const float* bias;           // nullable: added after the update (tensor-core modes)
  const int* cols;             // [slots - 1] column of each perturbed slot
  const float* vals;           // [slots - 1] its value
  int act;
  // tensor-core modes: W0's bf16 shadow parts [in, ld] and A0' as np bf16 parts; fp32: W0 [in, N] and A0' [pairs, N]
  const __nv_bfloat16* Wn; long long w_ps;
  __nv_bfloat16* out; long long out_ps;
  const float* W32;
  float* out32;
};

constexpr int SENS_ROWS = 32;   // rows one thread of sens_perturb_kernel walks with one W0 row group in registers

// the bf16 part `part` of x as the load kernel splits it (load_batch_kernel)
__device__ __forceinline__ float sens_part(float x, int part) { return __bfloat162float(__float2bfloat16_rn(bf16_residual(x, part))); }

// grid (ceil(groups / 32), slots, ceil(R / SENS_ROWS)), block (32, 8): thread x owns the 8-column group g of slot y and
// walks rows ty, ty + 8, ... of its row block with that group of W0[c, :] held in registers (read once per column and row
// block; W0 is L2-resident).  Every access is 16 bytes wide where the layout allows it.
template <bool TC, int NP>
__global__ void __launch_bounds__(256) sens_perturb_kernel(const SensParams p) {
  static_assert(NP >= 1 && NP <= 3 && (TC || NP == 1), "bf16 parts");
  const int groups = (p.N + 7) / 8;
  const int g = blockIdx.x * 32 + threadIdx.x;
  const int slot = blockIdx.y;
  if (g >= groups) return;
  const int c0 = g * 8;
  const int col = slot > 0 ? p.cols[slot - 1] : 0;
  const float v = slot > 0 ? p.vals[slot - 1] : 0.f;
  constexpr int np = NP;
  // W0[c, c0 .. c0 + 8) per part (fp32: one "part"); zero beyond N
  float w[NP][8];
#pragma unroll
  for (int b = 0; b < NP; ++b)
#pragma unroll
    for (int j = 0; j < 8; ++j) w[b][j] = 0.f;
  if (slot > 0) {
    if constexpr (TC) {
#pragma unroll
      for (int b = 0; b < np; ++b) {
        const uint4 u = __ldg(reinterpret_cast<const uint4*>(p.Wn + b * p.w_ps + static_cast<size_t>(col) * p.ld + c0));
#pragma unroll
        for (int j = 0; j < 8; ++j) w[b][j] = bf16_of_u4(u, j);
      }
    } else {
#pragma unroll
      for (int j = 0; j < 8; ++j) w[0][j] = c0 + j < p.N ? __ldg(p.W32 + static_cast<size_t>(col) * p.N + c0 + j) : 0.f;
    }
  }
  float bias[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) bias[j] = (p.bias != nullptr && c0 + j < p.N) ? __ldg(p.bias + c0 + j) : 0.f;
  const int r_end = min(p.R, static_cast<int>(blockIdx.z + 1) * SENS_ROWS);
  for (int r = blockIdx.z * SENS_ROWS + threadIdx.y; r < r_end; r += 8) {
    // delta of column c as layer 0's GEMM saw it.  Tensor-core modes multiply part a of x with part b of W for
    // a + b < np, so the column's term changes by sum_b W_b (sum_{a < np - b} (v_a - x_a)).  Each difference is made +0
    // when it is zero, so a value equal to x (+0 against -0 included) gives the base slot's arithmetic.
    float dx[NP];
#pragma unroll
    for (int b = 0; b < NP; ++b) dx[b] = 0.f;
    bool moved = false;
    if (slot > 0) {
      const float x = __ldg(p.X + static_cast<size_t>(r) * p.F + col);
      if constexpr (TC) {
        float dp[NP];
#pragma unroll
        for (int a = 0; a < np; ++a) {
          const float d = sens_part(v, a) - sens_part(x, a);
          dp[a] = d == 0.f ? 0.f : d;
        }
#pragma unroll
        for (int b = 0; b < np; ++b)
#pragma unroll
          for (int a = 0; a < np - b; ++a) dx[b] += dp[a];
      } else {
        const float d = v - x;
        dx[0] = d == 0.f ? 0.f : d;
      }
#pragma unroll
      for (int b = 0; b < NP; ++b) moved = moved || dx[b] != 0.f;
    }
    const float* zr = p.z + static_cast<size_t>(r) * p.ld + c0;
    float zz[8];
    const float4 z0 = __ldg(reinterpret_cast<const float4*>(zr));
    const float4 z1 = __ldg(reinterpret_cast<const float4*>(zr) + 1);
    zz[0] = z0.x; zz[1] = z0.y; zz[2] = z0.z; zz[3] = z0.w; zz[4] = z1.x; zz[5] = z1.y; zz[6] = z1.z; zz[7] = z1.w;
    float a[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      float t = zz[j];
      if (moved) {
        if constexpr (TC) {
          float dlt = w[np - 1][j] * dx[np - 1];
#pragma unroll
          for (int b = np - 2; b >= 0; --b) dlt = fmaf(w[b][j], dx[b], dlt);
          t += dlt;
        } else {
          t = fmaf(dx[0], w[0][j], t);
        }
      }
      a[j] = c0 + j < p.N ? act_apply(t + bias[j], p.act) : 0.f;   // pad columns: 0 (no tensor map reads them)
    }
    const size_t pr = static_cast<size_t>(slot) * p.R + r;   // the pair row
    if constexpr (TC) {
#pragma unroll
      for (int part = 0; part < np; ++part) {
        uint4 o;
        o.x = pack_bf16x2(bf16_residual(a[0], part), bf16_residual(a[1], part));
        o.y = pack_bf16x2(bf16_residual(a[2], part), bf16_residual(a[3], part));
        o.z = pack_bf16x2(bf16_residual(a[4], part), bf16_residual(a[5], part));
        o.w = pack_bf16x2(bf16_residual(a[6], part), bf16_residual(a[7], part));
        *reinterpret_cast<uint4*>(p.out + part * p.out_ps + pr * p.ld + c0) = o;
      }
    } else {
      float* o = p.out32 + pr * p.N + c0;
      if ((p.N & 3) == 0 && c0 + 8 <= p.N) {
        reinterpret_cast<float4*>(o)[0] = make_float4(a[0], a[1], a[2], a[3]);
        reinterpret_cast<float4*>(o)[1] = make_float4(a[4], a[5], a[6], a[7]);
      } else {
#pragma unroll
        for (int j = 0; j < 8; ++j)
          if (c0 + j < p.N) o[j] = a[j];
      }
    }
  }
}

constexpr int SENS_REDUCE_THREADS = 256;

// block k < C: column k of the piece.  d[r] = yhat[r] - yhat[(k + 1) R + r] goes to D[r * ldD + k] (D nullable); the
// block's w d^2 and w d are summed in fp64 in a fixed order (thread t takes rows t, t + 256, ... in turn, then a fixed
// shared-memory tree) and added to acc[2 (k0 + k)] / acc[2 (k0 + k) + 1].  Block C (when add_w): sum w into acc[w_slot].
// The launches of one call are stream-ordered and each slot has one writer per launch, so the running sums are added in
// row-chunk order.
__global__ void __launch_bounds__(SENS_REDUCE_THREADS)
sens_reduce_kernel(const float* __restrict__ yhat, const float* __restrict__ w, int R, int C, int k0, float* __restrict__ D,
                   int ldD, double* __restrict__ acc, int add_w, long long w_slot) {
  __shared__ double s2[SENS_REDUCE_THREADS], s1[SENS_REDUCE_THREADS];
  const int k = blockIdx.x, t = threadIdx.x;
  double a2 = 0.0, a1 = 0.0;
  if (k < C) {
    const float* ys = yhat + static_cast<size_t>(k + 1) * R;
    for (int r = t; r < R; r += SENS_REDUCE_THREADS) {
      const float d = yhat[r] - ys[r];
      if (D != nullptr) D[static_cast<size_t>(r) * ldD + k] = d;
      const double wd = static_cast<double>(w[r]) * static_cast<double>(d);
      a2 += wd * static_cast<double>(d);
      a1 += wd;
    }
  } else {
    if (!add_w) return;
    for (int r = t; r < R; r += SENS_REDUCE_THREADS) a1 += static_cast<double>(w[r]);
  }
  s2[t] = a2; s1[t] = a1;
  __syncthreads();
  for (int h = SENS_REDUCE_THREADS / 2; h > 0; h >>= 1) {
    if (t < h) { s2[t] += s2[t + h]; s1[t] += s1[t + h]; }
    __syncthreads();
  }
  if (t == 0) {
    if (k < C) {
      acc[2 * static_cast<size_t>(k0 + k)] += s2[0];
      acc[2 * static_cast<size_t>(k0 + k) + 1] += s1[0];
    } else {
      acc[w_slot] += s1[0];
    }
  }
}

constexpr int SENS_TOPK_MAX_K = 32;      // one running entry per lane
constexpr int SENS_TOPK_WARPS = 8;       // most warps per row

// The reason-code order as one unsigned 64-bit key, larger = ranks first: the high word maps the float key (d, -d or
// |d| for SB_REASON_RAISE / LOWER / MAGNITUDE) to an order-preserving integer with -0 made +0 and NaN below -inf; the
// low word is ~pos, so equal keys rank by the smaller list position.  Every entry is > 0; 0 is an empty slot.
__device__ __forceinline__ unsigned long long topk_key(float d, int order, int pos) {
  const float f = order == SB_REASON_RAISE ? d : order == SB_REASON_LOWER ? -d : fabsf(d);
  unsigned u = __float_as_uint(f);
  if ((u << 1) == 0u) u = 0u;                                   // -0 -> +0
  u = (u & 0x80000000u) ? ~u : (u | 0x80000000u);
  if (f != f) u = 0u;
  return (static_cast<unsigned long long>(u) << 32) | (0xFFFFFFFFu - static_cast<unsigned>(pos));
}

// one compare-exchange of a warp bitonic network with the lane `lane ^ s`: this lane keeps the larger (key, d) entry when
// keep_max, else the smaller.  Keys are distinct unless both are empty.
__device__ __forceinline__ void topk_cx(unsigned long long& key, float& d, int s, bool keep_max) {
  const unsigned long long pk = __shfl_xor_sync(0xFFFFFFFFu, key, s);
  const float pd = __shfl_xor_sync(0xFFFFFFFFu, d, s);
  if (keep_max ? pk > key : pk < key) { key = pk; d = pd; }
}

// a bitonic sequence over the warp's lanes -> sorted, largest key in lane 0
__device__ __forceinline__ void topk_bitonic_merge(unsigned long long& key, float& d, int lane) {
#pragma unroll
  for (int s = 16; s > 0; s >>= 1) topk_cx(key, d, s, (lane & s) == 0);
}

// `key` (sorted, lane 0 first) := the 32 largest of itself and the sorted list `ok` / `od` (lane 0 first), sorted
__device__ __forceinline__ void topk_merge(unsigned long long& key, float& d, unsigned long long ok, float od, int lane) {
  ok = __shfl_sync(0xFFFFFFFFu, ok, 31 - lane);                 // ascending: max(key[i], ok[31 - i]) is bitonic and holds
  od = __shfl_sync(0xFFFFFFFFu, od, 31 - lane);                 // the 32 largest of the union
  if (ok > key) { key = ok; d = od; }
  topk_bitonic_merge(key, d, lane);
}

// grid (R), block (32, W), W <= SENS_TOPK_WARPS: block r merges the piece's C deltas d = yhat[r] - yhat[(j + 1) R + r]
// (j < C, list position k0 + j; the fp32 expression of sens_reduce_kernel) into row r's running top k, run_d / run_pos
// [R, k] sorted best first (first: the running list starts empty).  Warp w takes columns w * 32 + lane, w * 32 + 32 W +
// lane, ...; a batch of 32 whose best key does not beat the warp's k-th is skipped, otherwise it is sorted by a warp
// bitonic network and merged into the warp's list.  Warp 0 then merges the other warps' lists from shared memory.  The
// order is total and each merge keeps the k best of the union, so the result does not depend on the piece boundaries or
// on the order the columns are taken in.
__global__ void __launch_bounds__(32 * SENS_TOPK_WARPS)
sens_topk_kernel(const float* __restrict__ yhat, int R, int C, int k0, int k, int order, int first, float* __restrict__ run_d,
                 int* __restrict__ run_pos) {
  __shared__ unsigned long long s_key[SENS_TOPK_WARPS][32];
  __shared__ float s_d[SENS_TOPK_WARPS][32];
  const int r = blockIdx.x, lane = threadIdx.x, wp = threadIdx.y, W = blockDim.y;
  const size_t o = static_cast<size_t>(r) * k + lane;
  unsigned long long key = 0;
  float d = 0.f;
  if (wp == 0 && !first && lane < k) {
    d = run_d[o];
    key = topk_key(d, order, run_pos[o]);
  }
  const float base = yhat[r];
  for (int j0 = wp * 32; j0 < C; j0 += 32 * W) {
    const int j = j0 + lane;
    unsigned long long ck = 0;
    float cd = 0.f;
    if (j < C) {
      cd = base - yhat[static_cast<size_t>(j + 1) * R + r];
      ck = topk_key(cd, order, k0 + j);
    }
    const unsigned long long kth = __shfl_sync(0xFFFFFFFFu, key, k - 1);
    if (!__any_sync(0xFFFFFFFFu, ck > kth)) continue;
#pragma unroll
    for (int size = 2; size <= 32; size <<= 1)                  // sort the batch, largest key in lane 0
#pragma unroll
      for (int s = size / 2; s > 0; s >>= 1) topk_cx(ck, cd, s, ((lane & s) == 0) == ((lane & size) == 0));
    topk_merge(key, d, ck, cd, lane);
  }
  if (W > 1) {
    s_key[wp][lane] = key;
    s_d[wp][lane] = d;
    __syncthreads();
    if (wp != 0) return;
    for (int v = 1; v < W; ++v) topk_merge(key, d, s_key[v][lane], s_d[v][lane], lane);
  }
  if (lane < k) {
    run_d[o] = d;
    run_pos[o] = static_cast<int>(0xFFFFFFFFu - static_cast<unsigned>(key));
  }
}

}  // namespace sb
