// Host-side launch of gemm_tc_kernel: picks the instantiation for a GemmPlan, sets the cluster attribute for CTA pairs.
#pragma once
#include "gemm_tc.cuh"

namespace sb {

template <int BN, int EPI, bool A_MN, bool B_MN, int CG, bool GENERIC = false>
static int launch_gemm_tc_one(const GemmPlan& pl, const TmapSet& tms, const GemmTcParams& p, cudaStream_t st,
                              bool pdl) {
  using Cfg = GemmTcCfg<BN, CG>;
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(static_cast<unsigned>(pl.grid));
  cfg.blockDim = dim3(Cfg::THREADS);
  cfg.dynamicSmemBytes = Cfg::SMEM_BYTES;
  cfg.stream = st;
  cudaLaunchAttribute at[2];
  int na = 0;
  if (CG == 2) {
    at[na].id = cudaLaunchAttributeClusterDimension;
    at[na].val.clusterDim.x = 2; at[na].val.clusterDim.y = 1; at[na].val.clusterDim.z = 1;
    ++na;
  }
  if (pdl) {
    at[na].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    at[na].val.programmaticStreamSerializationAllowed = 1;
    ++na;
  }
  cfg.attrs = at;
  cfg.numAttrs = na;
  SB_CUDA(cudaLaunchKernelEx(&cfg, gemm_tc_kernel<BN, EPI, A_MN, B_MN, CG, GENERIC>, tms, p));
  return SB_OK;
}

template <int EPI, bool A_MN, bool B_MN>
int launch_gemm_tc(const GemmPlan& pl, const TmapSet& tms, GemmTcParams p, cudaStream_t st, bool pdl = false) {
  if (p.np < 1) p.np = 1;
  if (p.n_pairs < 1) p.n_pairs = 1;
  p.split_k = pl.split_k;
  p.kb_per_split = pl.kb_per_split;
  // forward / dA: split-precision parts or an fp32 addend, the GENERIC instantiations (plain bf16 is gemm_pp.cuh)
  constexpr bool GENERIC = EPI == EPI_FWD || EPI == EPI_DA;
  if (pl.cg == 1 && pl.bn == 64) return launch_gemm_tc_one<64, EPI, A_MN, B_MN, 1, GENERIC>(pl, tms, p, st, pdl);
  if (pl.cg == 1 && pl.bn == 128) return launch_gemm_tc_one<128, EPI, A_MN, B_MN, 1, GENERIC>(pl, tms, p, st, pdl);
  if constexpr (EPI == EPI_F32) {   // CTA pairs: the tile-configuration hook's (the planner does not pick them)
  if (pl.cg == 2 && pl.bn == 128) return launch_gemm_tc_one<128, EPI, A_MN, B_MN, 2>(pl, tms, p, st, pdl);
  if (pl.cg == 2 && pl.bn == 256) return launch_gemm_tc_one<256, EPI, A_MN, B_MN, 2>(pl, tms, p, st, pdl);
  }
  return set_error(SB_ERR_INVALID, "no gemm_tc instantiation for cg=%d bn=%d", pl.cg, pl.bn);
}

// opt in to > 48 KB dynamic shared memory (once per process per instantiation, outside of stream capture)
template <int EPI, bool A_MN, bool B_MN>
int set_gemm_tc_attrs() {
  constexpr bool GENERIC = EPI == EPI_FWD || EPI == EPI_DA;
#define SB_ATTR(BN, CG)                                                                                                     \
  SB_CUDA(cudaFuncSetAttribute(gemm_tc_kernel<BN, EPI, A_MN, B_MN, CG, GENERIC>, cudaFuncAttributeMaxDynamicSharedMemorySize, \
                               GemmTcCfg<BN, CG>::SMEM_BYTES))
  SB_ATTR(64, 1); SB_ATTR(128, 1);
  if constexpr (EPI == EPI_F32) { SB_ATTR(128, 2); SB_ATTR(256, 2); }
#undef SB_ATTR
  return SB_OK;
}

// box rows of the tensor map of a K-major B operand / tile geometry helpers
inline int plan_box_rows_b(const GemmPlan& pl) { return pl.bn / pl.cg; }

}  // namespace sb
