// Host side of the TMA engine: the launch parameters it shares with gemm_tma_kernel (gemm_tma.cuh), tensor-map construction
// (cuTensorMapEncodeTiled through the runtime's driver entry point, so libcuda is not linked), the tile pickers, the list of
// instantiations and the launcher, which gemm_tma.cu compiles together with the kernel.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>

#include <cstdlib>
#include <string>

#include "tc_ptx.cuh"

namespace pf {

constexpr int MODE_GEMM = 0, MODE_HALO = 1;

struct TmaGemmParams {
  int M;                    // MODE_GEMM: rows
  int B, H, W;              // MODE_HALO: images, spatial size (output == input)
  int Cin;                  // MODE_HALO: input channels per group (multiple of 64);  MODE_GEMM: K
  int N, K;
  int a_c0, a_gc;           // channel coordinate of the first input channel in A's tensor map, step per group
  int c_split, a2_c0;       // MODE_HALO dual source: input channels >= c_split come from the A2 maps at a2_c0 + (ci - c_split); 0 = off
  int groups;
  int b_row0;               // first row of this launch's weights in the B tensor map (resident-weight launches fold the group in)
  // epilogue:  v = acc + bias;  v = act(v);  v *= gamma;  v += relu?(res);  v += res2
  const float* bias; int bias_mode, bias_gstride;
  int act; const float* gamma;
  const float* res;  int ldr, r_coff, r_gcoff, res_relu;
  const float* res2; int ldr2, r2_coff, r2_gcoff;
  float* C; int ldc, c_coff, c_gcoff;                                           // fp32 output (may be null)
  __nv_bfloat16* Shi; __nv_bfloat16* Slo; int lds, s_coff, s_gcoff, split_relu; // split output (may be null)
  // MODE_HALO, N = 32 (conv_fuse_conv1): fused prediction tail -- 1x1 conv 32 -> pred_nc (gravity_head.py:175 /
  // latitude_head.py:174) + F.normalize (pred_mode 1, gravity_head.py:192-193) or clamp to [-1,1] (pred_mode 2,
  // latitude_head.py:191-192), written NCHW to pred_out; replaces the separate pred_tail_kernel pass over conv1's output
  const float* pred_w; const float* pred_b; float* pred_out; int pred_nc, pred_mode;
  // MODE_HALO, N = BN = 128: the four 32-column chunks are the four output phases (py, px) of a convolution composed with the
  // bilinear x2 upsample in front of it (weights.py:_compose_up2_conv3): chunk ph, low-res pixel (y, x) -> pixel
  // (2y + ph/2, 2x + ph%2) of the 2H x 2W output, 32 channels.  C / S / the prediction tail are addressed on that grid.
  int phase4;
};

struct TmaMaps {   // passed by value as a __grid_constant__ kernel parameter
  CUtensorMap a_hi, a_lo, a2_hi, a2_lo, b_hi, b_lo;
};

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

// every instantiation the dispatcher (gemm_tma_launch) can reach: X(BN, MODE, KB).  Each one exists with three products and
// with one (the bf16 precision mode picks the same tiles).
#define PF_TMA_VARIANTS(X)                                                                                                  \
  X(256, MODE_GEMM, 32) X(224, MODE_GEMM, 32) X(192, MODE_GEMM, 32) X(160, MODE_GEMM, 32) X(128, MODE_GEMM, 32) X(96, MODE_GEMM, 32) \
  X(64, MODE_GEMM, 32) X(32, MODE_GEMM, 32) X(64, MODE_GEMM, 64) X(32, MODE_GEMM, 64)                                        \
  X(256, MODE_HALO, 32) X(128, MODE_HALO, 64) X(64, MODE_HALO, 64) X(32, MODE_HALO, 64)
// the GEMM-mode (bn, kb) pairs above, in the ping-pong schedule: X(BN, KB)
#define PF_TMA_PINGPONG_VARIANTS(X)                                                                                         \
  X(256, 32) X(224, 32) X(192, 32) X(160, 32) X(128, 32) X(96, 32) X(64, 32) X(32, 32) X(64, 64) X(32, 64)

// cudaFuncAttributeMaxDynamicSharedMemorySize is a per-device (per-context) attribute: called once for every device an engine is
// created on (pf_create) and every product count np (3 or 1) -- not behind a process-wide flag.
cudaError_t gemm_tma_configure_device(int np);
// ring depth of an instantiation, 0 if PF_TMA_VARIANTS (pp: PF_TMA_PINGPONG_VARIANTS) does not list it or np is not 3 or 1
int tma_stages(int mode, int bn, int kb, bool pp, int np);
// Why the (bn, kb) instantiation with np products cannot compute p: nullptr when it can.
const char* gemm_tma_check(int mode, const TmaGemmParams& p, int bn, int kb, bool pred, bool pp, int np);
// np = bf16 products per output: 3 (split precision) or 1 (bf16 precision mode)
cudaError_t gemm_tma_launch(int mode, const TmaMaps& maps, const TmaGemmParams& p, int bn, int kb, bool pp, int np, int sm_count, cudaStream_t st,
                            const PredTail* pred = nullptr);

}  // namespace pf
