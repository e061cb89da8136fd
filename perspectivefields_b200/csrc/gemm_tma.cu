// The TMA -> wgmma engine's kernel instantiations and their host dispatcher: the only translation unit that compiles
// gemm_tma.cuh, so the rest of the library builds without the engine's device code and reaches it through gemm_tma_launch.
#include "gemm_tma.cuh"

namespace pf {

template <int BN, int MODE, int KB, bool PP = false, int NP = 3>
inline cudaError_t gemm_tma_launch_bn(const TmaMaps& maps, const TmaGemmParams& p, int sm_count, cudaStream_t st, const PredTail* pred) {
  using Cfg = TmaCfg<BN, MODE, KB, PP, NP>;   // (the > 48 KB shared-memory opt-in is per device: gemm_tma_configure_device, at pf_create)
  const int tiles_x = MODE == MODE_HALO ? cdiv(p.W, kHtTileW) : 0, tiles_y = MODE == MODE_HALO ? cdiv(p.H, kHtTileH) : 0;
  const long long m_tiles = MODE == MODE_GEMM ? cdiv(p.M, Cfg::kTileM) : (long long)p.B * tiles_x * tiles_y;
  const long long total = m_tiles * cdiv(p.N, BN) * p.groups;
  const unsigned grid = (unsigned)(total < sm_count ? total : sm_count);
  // resident-weight mode (single chunk, one N tile) assumes every tile of a CTA uses the same weights: one group per launch
  // (a fused prediction tail is per group as well: same decomposition)
  if (MODE == MODE_HALO && ((p.Cin == 64 && 9 * (64 / KB) <= Cfg::kStages && (p.groups > 1 || cdiv(p.N, BN) > 1)) || pred)) {
    cudaError_t last = cudaSuccess;
    for (int g = 0; g < p.groups; ++g)
      for (int nt = 0; nt < cdiv(p.N, BN); ++nt) {
        TmaGemmParams q = p;     // fold group g / N tile nt into the offsets of a single-group, single-tile launch
        q.groups = 1;
        q.a_c0 = p.a_c0 + g * p.a_gc;
        q.bias = p.bias ? p.bias + (long long)g * p.bias_gstride : nullptr;
        q.c_coff = p.c_coff + g * p.c_gcoff; q.s_coff = p.s_coff + g * p.s_gcoff;
        q.r_coff = p.r_coff + g * p.r_gcoff; q.r2_coff = p.r2_coff + g * p.r2_gcoff;
        q.b_row0 = g * p.N;
        if (pred) { q.pred_w = pred[g].w; q.pred_b = pred[g].b; q.pred_out = pred[g].out; q.pred_nc = pred[g].nc; q.pred_mode = pred[g].mode; }
        if (cdiv(p.N, BN) > 1) return cudaErrorInvalidValue;   // (not needed by the network: conv_fuse_conv1 has one N tile)
        const unsigned gr = (unsigned)(m_tiles < sm_count ? m_tiles : sm_count);
        last = launch_pdl(gemm_tma_kernel<BN, MODE, KB, false, NP>, dim3(gr), dim3(kTmaThreads), Cfg::kSmemBytes, st, maps, q, tiles_x, tiles_y);
        if (last != cudaSuccess) return last;
      }
    return last;
  }
  return launch_pdl(gemm_tma_kernel<BN, MODE, KB, PP, NP>, dim3(grid), dim3(kTmaThreads), Cfg::kSmemBytes, st, maps, p, tiles_x, tiles_y);
}

template <int NP>
inline cudaError_t gemm_tma_configure_np() {
  cudaError_t e = cudaSuccess;
#define PF_TMA_CFG(BN_, MODE_, KB_)                                                                                          \
  if (e == cudaSuccess) e = cudaFuncSetAttribute(gemm_tma_kernel<BN_, MODE_, KB_, false, NP>, cudaFuncAttributeMaxDynamicSharedMemorySize, TmaCfg<BN_, MODE_, KB_, false, NP>::kSmemBytes);
  PF_TMA_VARIANTS(PF_TMA_CFG)
#undef PF_TMA_CFG
#define PF_TMA_CFG_PP(BN_, KB_)                                                                                               \
  if (e == cudaSuccess) e = cudaFuncSetAttribute(gemm_tma_kernel<BN_, MODE_GEMM, KB_, true, NP>, cudaFuncAttributeMaxDynamicSharedMemorySize, TmaCfg<BN_, MODE_GEMM, KB_, true, NP>::kSmemBytes);
  PF_TMA_PINGPONG_VARIANTS(PF_TMA_CFG_PP)
#undef PF_TMA_CFG_PP
  return e;
}
cudaError_t gemm_tma_configure_device(int np) {
  return np == 1 ? gemm_tma_configure_np<1>() : (np == 3 ? gemm_tma_configure_np<3>() : cudaErrorInvalidValue);
}

template <int NP>
inline int tma_stages_np(int mode, int bn, int kb, bool pp) {
#define PF_TMA_NS(BN_, MODE_, KB_) if (!pp && mode == MODE_ && bn == BN_ && kb == KB_) return TmaCfg<BN_, MODE_, KB_, false, NP>::kStages;
  PF_TMA_VARIANTS(PF_TMA_NS)
#undef PF_TMA_NS
#define PF_TMA_NS_PP(BN_, KB_) if (pp && mode == MODE_GEMM && bn == BN_ && kb == KB_) return TmaCfg<BN_, MODE_GEMM, KB_, true, NP>::kStages;
  PF_TMA_PINGPONG_VARIANTS(PF_TMA_NS_PP)
#undef PF_TMA_NS_PP
  return 0;
}
int tma_stages(int mode, int bn, int kb, bool pp, int np) {
  return np == 1 ? tma_stages_np<1>(mode, bn, kb, pp) : (np == 3 ? tma_stages_np<3>(mode, bn, kb, pp) : 0);
}

// Every case gemm_tma_check rejects would otherwise launch something that computes a different result (a K tail, a prediction
// tail or phase layout the tile width does not implement) or that gemm_tma_launch_bn refuses after the fact (resident weights
// over several N tiles).  Whether the weights are resident depends on the ring depth, so on np: the one-product ring is deeper.
const char* gemm_tma_check(int mode, const TmaGemmParams& p, int bn, int kb, bool pred, bool pp, int np) {
  const int ns = tma_stages(mode, bn, kb, pp, np);
  if (!ns) return pp ? "no ping-pong engine instantiation for this (mode, bn, kb)" : "no engine instantiation for this (mode, bn, kb)";
  if (mode == MODE_GEMM) return p.K % kb ? "GEMM mode: K must be a multiple of the K step" : nullptr;
  if (p.phase4 && (p.N != 128 || bn != 128)) return "phase4 needs N = 128 in one 128-wide tile";
  if (pred && bn != (p.phase4 ? 128 : 32)) return "the fused prediction tail needs N = 32 (phase4: 128) in one tile";
  const bool resident = p.Cin == 64 && 9 * (64 / kb) <= ns;
  if ((resident || pred) && cdiv(p.N, bn) > 1) return "resident weights (Cin = 64) and the prediction tail need one N tile per launch";
  return nullptr;
}

template <int NP>
inline cudaError_t gemm_tma_launch_np(int mode, const TmaMaps& maps, const TmaGemmParams& p, int bn, int kb, bool pp, int sm_count, cudaStream_t st,
                                      const PredTail* pred) {
#define PF_TMA_CASE(BN_, MODE_, KB_) if (!pp && mode == MODE_ && bn == BN_ && kb == KB_) return gemm_tma_launch_bn<BN_, MODE_, KB_, false, NP>(maps, p, sm_count, st, pred);
  PF_TMA_VARIANTS(PF_TMA_CASE)
#undef PF_TMA_CASE
#define PF_TMA_CASE_PP(BN_, KB_) if (pp && mode == MODE_GEMM && bn == BN_ && kb == KB_) return gemm_tma_launch_bn<BN_, MODE_GEMM, KB_, true, NP>(maps, p, sm_count, st, pred);
  PF_TMA_PINGPONG_VARIANTS(PF_TMA_CASE_PP)
#undef PF_TMA_CASE_PP
  return cudaErrorInvalidValue;
}
cudaError_t gemm_tma_launch(int mode, const TmaMaps& maps, const TmaGemmParams& p, int bn, int kb, bool pp, int np, int sm_count, cudaStream_t st,
                            const PredTail* pred) {
  if (np == 1) return gemm_tma_launch_np<1>(mode, maps, p, bn, kb, pp, sm_count, st, pred);
  if (np == 3) return gemm_tma_launch_np<3>(mode, maps, p, bn, kb, pp, sm_count, st, pred);
  return cudaErrorInvalidValue;
}

}  // namespace pf
