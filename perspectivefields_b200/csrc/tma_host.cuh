// Host side of the TMA engine: tensor-map construction (cuTensorMapEncodeTiled through the runtime's driver entry point,
// so libcuda is not linked) and the launcher of gemm_tma_kernel.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>

#include <cstdlib>
#include <string>

#include "gemm_tma.cuh"

namespace pf {

typedef CUresult (*PFN_tensorMapEncodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                             const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                             CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

inline PFN_tensorMapEncodeTiled tma_encoder() {
  static PFN_tensorMapEncodeTiled fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess)
      fn = (PFN_tensorMapEncodeTiled)p;
  }
  return fn;
}

// bf16 tensor [rows][ld] (row-major); box = box_rows x kb elements (kb = 32: 64 B rows, SWIZZLE_64B; kb = 64: 128 B rows,
// SWIZZLE_128B).  `cols` = logical row length.
inline const char* tma_map_2d(CUtensorMap* m, const void* base, long long cols, long long rows, long long ld, int box_rows, int kb) {
  PFN_tensorMapEncodeTiled enc = tma_encoder();
  if (!enc) return "cuTensorMapEncodeTiled entry point not available";
  cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
  cuuint64_t strides[1] = {(cuuint64_t)ld * 2};
  cuuint32_t box[2] = {(cuuint32_t)kb, (cuuint32_t)box_rows};
  cuuint32_t es[2] = {1, 1};
  if (((uintptr_t)base & 15) || (strides[0] & 15) || box_rows < 1 || box_rows > 256) return "tma_map_2d: alignment / box";
  CUresult r = enc(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(base), dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                   kb == 32 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? nullptr : "cuTensorMapEncodeTiled (2d) failed";
}

// bf16 NHWC tensor [B][H][W][ld]; box = 1 x 18 x 10 x 64 channels (128 B), SWIZZLE_128B: one halo chunk.
inline const char* tma_map_halo(CUtensorMap* m, const void* base, int B, int H, int W, int ld) {
  PFN_tensorMapEncodeTiled enc = tma_encoder();
  if (!enc) return "cuTensorMapEncodeTiled entry point not available";
  cuuint64_t dims[4] = {(cuuint64_t)ld, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)B};
  cuuint64_t strides[3] = {(cuuint64_t)ld * 2, (cuuint64_t)W * ld * 2, (cuuint64_t)H * W * ld * 2};
  cuuint32_t box[4] = {64, (cuuint32_t)kHtHaloW, (cuuint32_t)kHtHaloH, 1};
  cuuint32_t es[4] = {1, 1, 1, 1};
  if (((uintptr_t)base & 15) || (strides[0] & 15)) return "tma_map_halo: alignment";
  CUresult r = enc(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, const_cast<void*>(base), dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                   CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? nullptr : "cuTensorMapEncodeTiled (halo) failed";
}

// N tile: fewest tiles of <= 256 columns, then the narrowest multiple of 32 covering N (halo mode: powers of two only).
inline int tma_pick_bn(int N, int mode) {
  const int tiles = cdiv(N, 256);
  int bn = cdiv(cdiv(N, tiles), 32) * 32;
  if (mode == MODE_HALO) bn = bn <= 32 ? 32 : (bn <= 64 ? 64 : (bn <= 128 ? 128 : 256));
  return bn;
}

// GEMM mode with the number of rows known.  The widest tile moves the fewest operand bytes per output column, so it wins whenever
// the tiles fill the machine.  A launch that leaves most SMs idle (stage-4 / spatially reduced layers: 25 row tiles) is faster
// with narrower tiles spread over more SMs: pick the width that minimises waves x time per tile, with a K step of 16 costing the
// larger of its MMA time (3 products x 128 x BN x 16 at 4096 bf16 FLOP per clock and SM, the H100 SXM data-sheet peak) and
// its operand loads (1.6 clk per operand row), plus a fixed ~3000 clk per tile.  Results do not depend on the choice (same K
// order per output).
inline int tma_pick_bn_gemm(long long M, int N, int K, int sm_count) {
  const int base = tma_pick_bn(N, MODE_GEMM);
  const long long mt = cdivl(M, 128);
  if (mt * cdiv(N, base) * 4 > 3LL * sm_count) return base;
  int best = base;
  double best_cost = 1e30;
  for (int bn = base; bn >= 32; bn -= 32) {
    const long long tiles = mt * cdiv(N, bn);
    const double waves = (double)cdivl(tiles, sm_count);
    const double mma = 3.0 * bn, load = 1.6 * (128 + bn);
    const double cost = waves * ((K / 16) * (mma > load ? mma : load) + 3000.0);
    if (cost < best_cost - 1e-9) { best_cost = cost; best = bn; }
  }
  return best;
}

// K elements per pipeline step: 64 for narrow tiles when K allows it (halo mode: BN <= 128; GEMM mode, whose stages also
// hold the A tile: BN <= 64), else 32
inline int tma_pick_kb(int bn, int K, int mode) {
  const int lim = mode == MODE_HALO ? 128 : 64;
  return (bn <= lim && K % 64 == 0) ? 64 : 32;
}

// (bn, kb) of one launch: GEMM mode with the row count and SM count known (tma_pick_bn_gemm), halo mode from N alone.
// K = the GEMM's K (halo mode: 9 x Cin).  Chosen once per launch: the B-map boxes and the launched instantiation both follow it.
inline void tma_pick_tile(int mode, long long M, int N, int K, int sm_count, int& bn, int& kb) {
  bn = mode == MODE_GEMM ? tma_pick_bn_gemm(M, N, K, sm_count) : tma_pick_bn(N, mode);
  kb = tma_pick_kb(bn, K, mode);
}

// GEMM-mode schedule on top of (bn, kb): ping-pong (64-row tiles, one warpgroup's epilogue under the other's main loop) or
// cooperative (128-row tiles, both warpgroups on one tile).  Ping-pong for K <= 512 when the 64-row tiles fill every CTA with
// at least two.  Measured per launch on the C2 forward (H100 80GB HBM3, 400 W; tools/launch_floors.py), this rule saved about
// 1 ms per step against the cooperative schedule.  Ping-pong on every launch was slower on the wide short-K ConvNeXt stage-0
// pw1 (M = 204800, K = 96).
constexpr int kPingPongKMax = 512;
inline bool tma_pick_pingpong(long long M, int N, int K, int bn, int sm_count) {
  return K <= kPingPongKMax && cdivl(M, 64) * cdiv(N, bn) >= 2LL * sm_count;
}

struct PredTail { const float* w; const float* b; float* out; int nc, mode; };   // per group, see TmaGemmParams::pred_*

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

// every instantiation the dispatcher below can reach: X(BN, MODE, KB).  Each one exists with three products and with one (the
// bf16 precision mode picks the same tiles).
#define PF_TMA_VARIANTS(X)                                                                                                  \
  X(256, MODE_GEMM, 32) X(224, MODE_GEMM, 32) X(192, MODE_GEMM, 32) X(160, MODE_GEMM, 32) X(128, MODE_GEMM, 32) X(96, MODE_GEMM, 32) \
  X(64, MODE_GEMM, 32) X(32, MODE_GEMM, 32) X(64, MODE_GEMM, 64) X(32, MODE_GEMM, 64)                                        \
  X(256, MODE_HALO, 32) X(128, MODE_HALO, 64) X(64, MODE_HALO, 64) X(32, MODE_HALO, 64)
// the GEMM-mode (bn, kb) pairs above, in the ping-pong schedule: X(BN, KB)
#define PF_TMA_PINGPONG_VARIANTS(X)                                                                                         \
  X(256, 32) X(224, 32) X(192, 32) X(160, 32) X(128, 32) X(96, 32) X(64, 32) X(32, 32) X(64, 64) X(32, 64)

// cudaFuncAttributeMaxDynamicSharedMemorySize is a per-device (per-context) attribute: called once for every device an engine is
// created on (pf_create) and every product count np (3 or 1) -- not behind a process-wide flag.
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
inline cudaError_t gemm_tma_configure_device(int np) {
  return np == 1 ? gemm_tma_configure_np<1>() : (np == 3 ? gemm_tma_configure_np<3>() : cudaErrorInvalidValue);
}

// ring depth of an instantiation, 0 if PF_TMA_VARIANTS (pp: PF_TMA_PINGPONG_VARIANTS) does not list it or np is not 3 or 1
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
inline int tma_stages(int mode, int bn, int kb, bool pp, int np) {
  return np == 1 ? tma_stages_np<1>(mode, bn, kb, pp) : (np == 3 ? tma_stages_np<3>(mode, bn, kb, pp) : 0);
}

// Why the (bn, kb) instantiation with np products cannot compute p: nullptr when it can.  Every case here would otherwise launch
// something that computes a different result (a K tail, a prediction tail or phase layout the tile width does not implement) or
// that gemm_tma_launch_bn refuses after the fact (resident weights over several N tiles).  Whether the weights are resident
// depends on the ring depth, so on np: the one-product ring is deeper.
inline const char* gemm_tma_check(int mode, const TmaGemmParams& p, int bn, int kb, bool pred, bool pp, int np) {
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
// np = bf16 products per output: 3 (split precision) or 1 (bf16 precision mode)
inline cudaError_t gemm_tma_launch(int mode, const TmaMaps& maps, const TmaGemmParams& p, int bn, int kb, bool pp, int np, int sm_count, cudaStream_t st,
                                   const PredTail* pred = nullptr) {
  if (np == 1) return gemm_tma_launch_np<1>(mode, maps, p, bn, kb, pp, sm_count, st, pred);
  if (np == 3) return gemm_tma_launch_np<3>(mode, maps, p, bn, kb, pp, sm_count, st, pred);
  return cudaErrorInvalidValue;
}

}  // namespace pf
