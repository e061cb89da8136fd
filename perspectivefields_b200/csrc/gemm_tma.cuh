// TMA -> wgmma engine: persistent, warp-specialised, TMA producer running ahead of the MMA warpgroups through an mbarrier ring.
//
// All GEMM operands arrive PRE-SPLIT: activations as two bf16 planes (hi = bf16(x), lo = bf16(x - hi)) written by the
// producing kernel's epilogue, weights as hi/lo planes split at load time.  Each product costs three bf16 MMAs
// (lo*hi + hi*lo + hi*hi, fp32 accumulation) -- see DESIGN.md "precision"; the opt-in bf16 mode (NP = 1) loads the hi planes
// only and costs one (hi*hi).  The epilogue writes both split planes in either mode.  Nothing is converted here: tiles go
// HBM/L2 --TMA--> swizzled shared memory --wgmma--> registers --> fused epilogue --> HBM.
//
//   MODE_GEMM : C[M,N] = A[M,K] W[N,K]^T.     A tiles 128 x KB by 2-D TMA, NS-stage ring.
//   MODE_HALO : 3x3 / stride 1 / pad 1 convolution, 16 x 8 pixel tiles.  One 4-D TMA per 64-channel chunk loads the
//               18 x 10 input halo (OOB = zero padding) as [180 pixels][128 B] SWIZZLE_128B; the A operand of filter tap
//               (ky,kx) is a shifted view of it (start + (ky*10+kx)*128 B, SBO = 1280 B).  Weights stream through an NS-stage
//               ring of KB-wide K steps.
//
//   warpgroup 0 : warp 0 = TMA producer (B ring; in MODE_GEMM also A), warp 1 = MODE_HALO halo (A) producer
//   warpgroups 1, 2 : MMA + epilogue.  Two schedules:
//     cooperative (PP = false): both work on one 128 x BN tile, rows 0-63 and 64-127 (wgmma M = 64 per warpgroup); each
//                     accumulates its 64 x BN block in registers and runs the fused epilogue on it.
//     ping-pong (PP = true, MODE_GEMM): tiles are 64 x BN and each warpgroup owns every other tile of the CTA's sequence, so one
//                     warpgroup's epilogue (HBM traffic) overlaps the other's main loop (tensor cores).  A ring stage belongs to
//                     the warpgroup whose tile it holds.  B is loaded once per 64 rows instead of 128: this pays on short K,
//                     where the epilogue is a large share of a tile's time.  Same K order per output as the cooperative schedule.
//
// Epilogue (fused): + bias | border-class bias, ReLU / GELU, layer scale, + relu?(residual), + second residual; writes the
// fp32 tensor and/or the bf16 hi/lo planes (optionally rectified) that the next GEMM will TMA-load.  Residual loads and both kinds
// of store move through the warpgroup's shared-memory staging rows as whole row segments.
#pragma once
#include <cuda.h>

#include "tc_ptx.cuh"
#include "tma_host.cuh"

namespace pf {

constexpr int kTmaThreads = 384;   // warpgroup 0: producers;  warpgroups 1-2: MMA + epilogue
constexpr int kHaloBytes = 180 * 128;   // one bf16 plane of an 18 x 10 pixel x 64 channel halo (what one TMA box delivers)

// KB = K elements per pipeline step: 32 (64 B rows, SWIZZLE_64B) for wide tiles, 64 (128 B rows, SWIZZLE_128B) for narrow ones
// where a 32-wide step would be shorter than the barrier round trip that feeds it.
// NP = bf16 products per output: 3 (lo*hi + hi*lo + hi*hi on hi / lo planes, fp32-accurate) or 1 (hi*hi only: the opt-in
// bf16 precision mode).  With one product only the hi planes are loaded, so a stage holds half the bytes and the ring is deeper.
template <int BN, int MODE, int KB, bool PP = false, int NP = 3> struct TmaCfg {
  static_assert(KB == 32 || KB == 64, "KB");
  static_assert(BN % 32 == 0 && BN <= 256, "BN");
  static_assert(!PP || MODE == MODE_GEMM, "the ping-pong schedule is a GEMM-mode schedule");
  static_assert(NP == 1 || NP == 3, "NP");
  static constexpr int kPlanes = NP == 3 ? 2 : 1;               // bf16 planes loaded per operand: hi + lo, or hi
  static constexpr int kTileM = PP ? 64 : 128;                  // MODE_GEMM: rows per tile
  static constexpr int kBPlane = BN * KB * 2;                   // bf16 plane of one K step of B
  static constexpr int kAPlane = kTileM * KB * 2;               // MODE_GEMM: plane of a kTileM x KB A tile
  static constexpr int kStage = (MODE == MODE_GEMM ? kPlanes * kAPlane : 0) + kPlanes * kBPlane;
  static constexpr int kABuf = kPlanes * kHtPlaneBytes;         // MODE_HALO: the halo planes of one chunk (1024 B multiples)
  // epilogue staging: each MMA warpgroup moves its accumulators through shared memory 64 columns at a time so that one thread
  // then holds 32 consecutive columns of one row (row pitch 68 floats: the row-wise float4 reads are free of bank conflicts)
  static constexpr int kAccPitch = 68;
  static constexpr int kAccStage = 2 * 64 * kAccPitch * 4;
  static constexpr int kBudget = 225 * 1024 - kAccStage - (MODE == MODE_HALO ? 2 * kABuf : 0);
  static constexpr int kStagesRaw = kBudget / kStage;
  static constexpr int kStages = kStagesRaw > 16 ? 16 : kStagesRaw;
  static constexpr int kSmemBytes = (MODE == MODE_HALO ? 2 * kABuf : 0) + kStages * kStage + kAccStage + 512 + 1024;
  static_assert(kStages >= 2, "ring too shallow");
  static_assert(kSmemBytes <= 227 * 1024, "shared memory per block");
};

// ------------------------------------------------------------------------------------------------ TMA PTX
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;\n" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void tma_load_2d(uint32_t dst, const CUtensorMap* map, uint32_t bar, int c0, int c1) {
  asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];\n"
               ::"r"(dst), "l"(reinterpret_cast<uint64_t>(map)), "r"(bar), "r"(c0), "r"(c1) : "memory");
}
__device__ __forceinline__ void tma_load_4d(uint32_t dst, const CUtensorMap* map, uint32_t bar, int c0, int c1, int c2, int c3) {
  asm volatile("cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];\n"
               ::"r"(dst), "l"(reinterpret_cast<uint64_t>(map)), "r"(bar), "r"(c0), "r"(c1), "r"(c2), "r"(c3) : "memory");
}
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* map) {
  asm volatile("prefetch.tensormap [%0];\n" ::"l"(reinterpret_cast<uint64_t>(map)) : "memory");
}

template <int BN, int MODE, int KB, bool PP = false, int NP = 3>
__global__ void __launch_bounds__(kTmaThreads, 1) gemm_tma_kernel(const __grid_constant__ TmaMaps maps, const TmaGemmParams p, int tiles_x, int tiles_y) {
  using Cfg = TmaCfg<BN, MODE, KB, PP, NP>;
  constexpr bool kLo = NP == 3;               // the lo planes are loaded and multiplied
  constexpr int NS = Cfg::kStages;
  constexpr int SPC = 9 * (64 / KB);          // MODE_HALO: pipeline steps per 64-channel chunk (9 taps x 64 / KB)
  constexpr int kConsumerWarps = PP ? 4 : 8;   // warps that release a ring stage: its warpgroup (ping-pong) or both
  extern __shared__ unsigned char smem_dyn[];
  const uint32_t raw = smem_u32(smem_dyn);
  const uint32_t sbase = (raw + 1023u) & ~1023u;
  unsigned char* sm = smem_dyn + (sbase - raw);
  const uint32_t a_base = sbase;                                                  // MODE_HALO: 2 halo buffers
  const uint32_t ring = sbase + (MODE == MODE_HALO ? 2 * Cfg::kABuf : 0);         // NS stages
  const uint32_t acc_base = ring + NS * Cfg::kStage;                              // epilogue staging, one half per MMA warpgroup
  const uint32_t bars = acc_base + Cfg::kAccStage;
  auto full_b = [&](int s) { return bars + 8u * s; };
  auto empty_b = [&](int s) { return bars + 8u * (NS + s); };
  auto full_a = [&](int i) { return bars + 8u * (2 * NS + i); };
  auto empty_a = [&](int i) { return bars + 8u * (2 * NS + 2 + i); };
  auto order_b = [&](int w) { return bars + 8u * (2 * NS + 4 + w); };   // ping-pong: warpgroup w has issued a tile's main loop

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int n_tiles = cdiv(p.N, BN);
  const int m_tiles = MODE == MODE_GEMM ? cdiv(p.M, Cfg::kTileM) : p.B * tiles_x * tiles_y;
  const int total_tiles = m_tiles * n_tiles * p.groups;
  const int nchunks = MODE == MODE_HALO ? p.Cin / 64 : 0;
  const int nk = MODE == MODE_GEMM ? p.K / KB : nchunks * SPC;
  // MODE_HALO with a single chunk whose 9 taps fit the ring (conv_fuse_conv1): the weights are loaded once per CTA and stay
  // resident for all of its tiles instead of being re-streamed from L2 for every tile.
  const bool b_resident = MODE == MODE_HALO && nchunks == 1 && SPC <= NS;

  if (tid == 0) {
    tma_prefetch_desc(&maps.a_hi); tma_prefetch_desc(&maps.b_hi);
    if (kLo) { tma_prefetch_desc(&maps.a_lo); tma_prefetch_desc(&maps.b_lo); }
    for (int s = 0; s < NS; ++s) { mbar_init(full_b(s), 1); mbar_init(empty_b(s), kConsumerWarps); }
    for (int i = 0; i < 2; ++i) { mbar_init(full_a(i), 1); mbar_init(empty_a(i), kConsumerWarps); mbar_init(order_b(i), 4); }
    fence_mbar_init();
  }
  __syncthreads();
  // everything above (barrier init, descriptor prefetch) overlaps the tail of the previous kernel of the stream when this one
  // was launched with programmatic stream serialisation; from here on its results are read
  pdl_wait();
  pdl_launch();

  // tile id -> (m tile, group, n tile); n fastest so that CTAs running together share the A tile / halo in L2
  auto decode = [&](int tile, int& mt, int& g, int& n0) {
    n0 = (tile % n_tiles) * BN;
    tile /= n_tiles;
    g = tile % p.groups;
    mt = tile / p.groups;
  };

  if (warp < 4) {
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;\n");
    if (warp == 0 && lane == 0) {
      // ===================================================================== TMA producer: B ring (+ A tiles in MODE_GEMM)
      int it = 0;
      for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
        int mt, g, n0;
        decode(tile, mt, g, n0);
        const int brow = p.b_row0 + g * p.N + n0;
        if (b_resident && it > 0) break;     // resident weights: loaded with the first tile only (one group / N tile per launch)
        for (int kc = 0; kc < nk; ++kc, ++it) {
          const int s = it % NS;
          mbar_wait(empty_b(s), ((it / NS) & 1) ^ 1);
          mbar_expect_tx(full_b(s), Cfg::kStage);
          const uint32_t st = ring + s * Cfg::kStage;
          int kcol;
          if (MODE == MODE_GEMM) {
            kcol = kc * KB;
            tma_load_2d(st, &maps.a_hi, full_b(s), p.a_c0 + g * p.a_gc + kcol, mt * Cfg::kTileM);
            if (kLo) tma_load_2d(st + Cfg::kAPlane, &maps.a_lo, full_b(s), p.a_c0 + g * p.a_gc + kcol, mt * Cfg::kTileM);
          } else {
            const int c = kc / SPC, u = kc - c * SPC;
            kcol = KB == 32 ? (u >> 1) * p.Cin + c * 64 + (u & 1) * 32 : u * p.Cin + c * 64;
          }
          const uint32_t bdst = st + (MODE == MODE_GEMM ? Cfg::kPlanes * Cfg::kAPlane : 0);
          tma_load_2d(bdst, &maps.b_hi, full_b(s), kcol, brow);
          if (kLo) tma_load_2d(bdst + Cfg::kBPlane, &maps.b_lo, full_b(s), kcol, brow);
        }
      }
    } else if (MODE == MODE_HALO && warp == 1 && lane == 0) {
      // ===================================================================== MODE_HALO: halo (A) producer
      int ita = 0;
      for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
        int mt, g, n0;
        decode(tile, mt, g, n0);
        const int tx = mt % tiles_x, ty = (mt / tiles_x) % tiles_y, bimg = mt / (tiles_x * tiles_y);
        for (int c = 0; c < nchunks; ++c, ++ita) {
          const int buf = ita & 1;
          mbar_wait(empty_a(buf), ((ita >> 1) & 1) ^ 1);
          mbar_expect_tx(full_a(buf), Cfg::kPlanes * kHaloBytes);
          const uint32_t dst = a_base + buf * Cfg::kABuf;
          const int ci = c * 64;
          if (p.c_split > 0 && ci >= p.c_split) {
            tma_load_4d(dst, &maps.a2_hi, full_a(buf), p.a2_c0 + ci - p.c_split, tx * kHtTileW - 1, ty * kHtTileH - 1, bimg);
            if (kLo) tma_load_4d(dst + kHtPlaneBytes, &maps.a2_lo, full_a(buf), p.a2_c0 + ci - p.c_split, tx * kHtTileW - 1, ty * kHtTileH - 1, bimg);
          } else {
            tma_load_4d(dst, &maps.a_hi, full_a(buf), p.a_c0 + g * p.a_gc + ci, tx * kHtTileW - 1, ty * kHtTileH - 1, bimg);
            if (kLo) tma_load_4d(dst + kHtPlaneBytes, &maps.a_lo, full_a(buf), p.a_c0 + g * p.a_gc + ci, tx * kHtTileW - 1, ty * kHtTileH - 1, bimg);
          }
        }
      }
    }
    return;
  }

  // ======================================================================= MMA + epilogue warpgroups
  asm volatile("setmaxnreg.inc.sync.aligned.u32 232;\n");
  const int wg = (warp >> 2) - 1;                 // cooperative: 0 = tile rows 0-63, 1 = rows 64-127;  ping-pong: CTA-local tile parity
  const int wt = tid & 127;                       // thread within the warpgroup
  float* stage = reinterpret_cast<float*>(sm + (acc_base - sbase)) + wg * 64 * Cfg::kAccPitch;
  // epilogue ownership: row `erow` of this warpgroup's 64, 32-column half `eh` of each 64-column staging round
  const int erow = wt & 63, eh = wt >> 6;
  const int r = PP ? erow : wg * 64 + erow;       // row of the tile
  constexpr int kTileStep = PP ? 2 : 1;           // ping-pong: this warpgroup's tiles are CTA-local tiles wg, wg + 2, ...
  float acc[BN / 2];
  int it = 0, ita = 0;
  for (int tl = PP ? wg : 0, tile = blockIdx.x + tl * gridDim.x; tile < total_tiles; tile += kTileStep * gridDim.x, tl += kTileStep) {
    int mt, g, n0;
    decode(tile, mt, g, n0);
    if (PP) {
      it = tl * nk;                               // the producer fills nk stages per tile in CTA-local tile order
      // main loops alternate: tile tl starts once the other warpgroup has issued tile tl - 1 (its completion (tl - 1) / 2).  This
      // also keeps a warpgroup's full-barrier waits within one ring round of the producer, which their parity needs.
      if (tl > 0) mbar_wait(order_b(wg ^ 1), ((tl - 1) >> 1) & 1);
    }
    // ---------------- main loop: per k16 of a K step, one m64nBNk16 wgmma per product (lo*hi, hi*lo, hi*hi; NP = 1: hi*hi), one commit group per
    // step; the stage of the previous step is released once that step's group has completed (one group stays in flight under the
    // next wait).  The B plane is contiguous in 8-row groups, so one descriptor spans all BN weight rows.
    int prev_s = -1, prev_buf = -1;
    fence_regs(acc);
    for (int kc = 0; kc < nk; ++kc, ++it) {
      const int s = it % NS;
      uint32_t a_hi, a_lo;
      bool chunk_end = false;
      int buf = 0;
      if (MODE == MODE_HALO) {
        const int c = kc / SPC, u = kc - c * SPC;
        const int tap = KB == 32 ? (u >> 1) : u, ky = tap / 3, kx = tap - ky * 3;
        buf = ita & 1;
        if (u == 0) mbar_wait(full_a(buf), (ita >> 1) & 1);
        // this warpgroup's 64 pixels are image rows 8 wg .. 8 wg + 7 of the tile
        a_hi = a_base + buf * Cfg::kABuf + ((ky + 8 * wg) * kHtHaloW + kx) * 128 + (KB == 32 ? (u & 1) * 64 : 0);
        a_lo = a_hi + kHtPlaneBytes;
        chunk_end = u == SPC - 1;
      } else {
        a_hi = ring + s * Cfg::kStage + (PP ? 0 : wg * 64 * KB * 2);
        a_lo = a_hi + Cfg::kAPlane;
      }
      const int sb = b_resident ? kc : s;                                   // resident weights: step kc lives in slot kc
      if (!b_resident || tl == 0) mbar_wait(full_b(sb), b_resident ? 0 : ((it / NS) & 1));
      const uint32_t b_hi = ring + sb * Cfg::kStage + (MODE == MODE_GEMM ? Cfg::kPlanes * Cfg::kAPlane : 0);
      const uint64_t dah = MODE == MODE_HALO ? ht_a_desc(a_hi) : wgmma_tile_desc<KB>(a_hi);
      const uint64_t dbh = wgmma_tile_desc<KB>(b_hi);
      wgmma_fence();
      if (kLo) {
        const uint64_t dal = MODE == MODE_HALO ? ht_a_desc(a_lo) : wgmma_tile_desc<KB>(a_lo);
        const uint64_t dbl = wgmma_tile_desc<KB>(b_hi + Cfg::kBPlane);
#pragma unroll
        for (int kk = 0; kk < KB / 16; ++kk) {
          const uint32_t first = (kc | kk) ? 1u : 0u;
          wgmma_bf16<BN>(acc, dal + 2 * kk, dbh + 2 * kk, first);
          wgmma_bf16<BN>(acc, dah + 2 * kk, dbl + 2 * kk, 1u);
          wgmma_bf16<BN>(acc, dah + 2 * kk, dbh + 2 * kk, 1u);
        }
      } else {
#pragma unroll
        for (int kk = 0; kk < KB / 16; ++kk) wgmma_bf16<BN>(acc, dah + 2 * kk, dbh + 2 * kk, (kc | kk) ? 1u : 0u);
      }
      wgmma_commit();
      wgmma_wait<1>();
      if (lane == 0 && prev_s >= 0) {
        if (!b_resident) mbar_arrive(empty_b(prev_s));
        if (MODE == MODE_HALO && prev_buf >= 0) mbar_arrive(empty_a(prev_buf));
      }
      prev_s = s;
      prev_buf = chunk_end ? buf : -1;
      if (MODE == MODE_HALO && chunk_end) ++ita;
    }
    if (PP && lane == 0) mbar_arrive(order_b(wg));
    wgmma_wait<0>();
    fence_regs(acc);
    if (lane == 0 && prev_s >= 0) {
      if (!b_resident) mbar_arrive(empty_b(prev_s));
      if (MODE == MODE_HALO && prev_buf >= 0) mbar_arrive(empty_a(prev_buf));
    }

    // ---------------- epilogue
    long long m;
    bool valid;
    int cls_off = 0;
    int bimg = 0, oy = 0, ox = 0, oy0 = 0, ox0 = 0;
    if (MODE == MODE_GEMM) {
      m = (long long)mt * Cfg::kTileM + r;
      valid = m < p.M;
    } else {
      const int tx = mt % tiles_x, ty = (mt / tiles_x) % tiles_y;
      bimg = mt / (tiles_x * tiles_y);
      oy0 = ty * kHtTileH; ox0 = tx * kHtTileW;
      oy = oy0 + (r >> 3); ox = ox0 + (r & 7);
      valid = oy < p.H && ox < p.W;
      m = ((long long)bimg * p.H + oy) * p.W + ox;
      if (p.bias_mode == 2) {
        const int ry = oy == 0 ? 0 : (oy == p.H - 1 ? 2 : 1);
        const int rx = ox == 0 ? 0 : (ox == p.W - 1 ? 2 : 1);
        cls_off = (ry * 3 + rx) * p.N;
      }
    }
    const float* __restrict__ bias = p.bias ? p.bias + (long long)g * p.bias_gstride : nullptr;
    // global row of staging row rr of this warpgroup (MODE_HALO: its pixel), and whether it exists
    auto stage_row = [&](int rr, long long& mr) -> bool {
      if (MODE == MODE_GEMM) {
        mr = (long long)mt * Cfg::kTileM + (PP ? 0 : wg * 64) + rr;
        return mr < p.M;
      }
      const int rt = wg * 64 + rr, py = oy0 + (rt >> 3), px = ox0 + (rt & 7);
      mr = ((long long)bimg * p.H + py) * p.W + px;
      return py < p.H && px < p.W;
    };
    // accumulator fragment of m64nNk16: register 4 jb + 2 h + e holds row 16 (wt / 32) + lane / 4 + 8 h, column 8 jb + 2 (lane % 4) + e
    const int frow = (wt >> 5) * 16 + (lane >> 2), fcol = 2 * (lane & 3);
#pragma unroll
    for (int rd = 0; rd < (BN + 63) / 64; ++rd) {
      named_bar_sync(1 + wg, 128);                // the previous round's (or tile's) rows have been read
#pragma unroll
      for (int jb = 0; jb < 8; ++jb) {
        const int cb = rd * 8 + jb;
        if (cb < BN / 8) {
          float* d0 = stage + frow * Cfg::kAccPitch + jb * 8 + fcol;
          *reinterpret_cast<float2*>(d0) = make_float2(acc[4 * cb], acc[4 * cb + 1]);
          *reinterpret_cast<float2*>(d0 + 8 * Cfg::kAccPitch) = make_float2(acc[4 * cb + 2], acc[4 * cb + 3]);
        }
      }
      named_bar_sync(1 + wg, 128);
      const int ch = 2 * rd + eh;                 // this thread's 32-column chunk (warp-uniform)
      const bool own = ch < BN / 32;              // (the last round of a BN % 64 == 32 tile has one chunk)
      const bool ph4 = MODE == MODE_HALO && BN == 128 && p.phase4;
      // fp32 output and split planes outside phase mode go out through shared memory (staged stores below)
      const bool staged_split = p.Shi && !ph4;
      const int nb = n0 + ch * 32;
      const bool chunk_ok = own && nb < p.N;     // warp-uniform
      const bool live = valid && chunk_ok;
      const float* srow = stage + erow * Cfg::kAccPitch + eh * 32;   // this thread's 32 columns of the staging rows
      float o[32];
      if (own) {
#pragma unroll
        for (int j = 0; j < 32; j += 4) {
          const float4 t = *reinterpret_cast<const float4*>(srow + j);
          o[j] = t.x; o[j + 1] = t.y; o[j + 2] = t.z; o[j + 3] = t.w;
        }
      }
      if (live) {
        if (p.bias_mode) {
#pragma unroll
          for (int j = 0; j < 32; j += 4) {
            const float4 bv = __ldg(reinterpret_cast<const float4*>(bias + cls_off + nb + j));
            o[j] += bv.x; o[j + 1] += bv.y; o[j + 2] += bv.z; o[j + 3] += bv.w;
          }
        }
        if (p.act == 1) {
#pragma unroll
          for (int j = 0; j < 32; ++j) o[j] = fmaxf(o[j], 0.f);
        } else if (p.act == 2) {
#pragma unroll
          for (int j = 0; j < 32; ++j) o[j] = gelu_erf(o[j]);
        }
        if (p.gamma) {
#pragma unroll
          for (int j = 0; j < 32; j += 4) {
            const float4 gv = __ldg(reinterpret_cast<const float4*>(p.gamma + nb + j));
            o[j] *= gv.x; o[j + 1] *= gv.y; o[j + 2] *= gv.z; o[j + 3] *= gv.w;
          }
        }
      }
      // Residuals.  A thread's 32 columns are 128 B of one row, so reading them from registers makes every warp-wide load touch
      // 32 lines for 16 B each.  The warpgroup reads the round's 64 rows x 64 columns into the staging area instead (free once
      // every thread has read its accumulators), as whole 256 B row segments: 16 lanes per row, 2 rows per instruction.  The
      // rows a tile stores are its own, so in-place launches (res == C) still read every residual before it is overwritten.
      auto stage_in = [&](const float* src, int ld, int coff) {
        named_bar_sync(1 + wg, 128);              // every thread has read what the staging area holds
        float4 v[8];
#pragma unroll
        for (int t = 0; t < 8; ++t) {
          const int i = wt + 128 * t, col = rd * 64 + (i & 15) * 4;
          long long mr;
          v[t] = make_float4(0.f, 0.f, 0.f, 0.f);
          if (col < BN && n0 + col < p.N && stage_row(i >> 4, mr)) v[t] = *reinterpret_cast<const float4*>(src + mr * ld + coff + n0 + col);
        }
#pragma unroll
        for (int t = 0; t < 8; ++t) {
          const int i = wt + 128 * t;
          *reinterpret_cast<float4*>(stage + (i >> 4) * Cfg::kAccPitch + (i & 15) * 4) = v[t];
        }
        named_bar_sync(1 + wg, 128);
      };
      if (p.res) {
        stage_in(p.res, p.ldr, p.r_coff + g * p.r_gcoff);
        if (live) {
#pragma unroll
          for (int j = 0; j < 32; j += 4) {
            float4 rv = *reinterpret_cast<const float4*>(srow + j);
            if (p.res_relu) { rv.x = fmaxf(rv.x, 0.f); rv.y = fmaxf(rv.y, 0.f); rv.z = fmaxf(rv.z, 0.f); rv.w = fmaxf(rv.w, 0.f); }
            o[j] += rv.x; o[j + 1] += rv.y; o[j + 2] += rv.z; o[j + 3] += rv.w;
          }
        }
      }
      if (p.res2) {
        stage_in(p.res2, p.ldr2, p.r2_coff + g * p.r2_gcoff);
        if (live) {
#pragma unroll
          for (int j = 0; j < 32; j += 4) {
            const float4 rv = *reinterpret_cast<const float4*>(srow + j);
            o[j] += rv.x; o[j + 1] += rv.y; o[j + 2] += rv.z; o[j + 3] += rv.w;
          }
        }
      }
      // output row / first output column of this chunk (phase mode: hi-res pixel of phase `ch`, channels 0-31)
      const long long mo = ph4 ? ((long long)bimg * 2 * p.H + 2 * oy + (ch >> 1)) * (2 * p.W) + 2 * ox + (ch & 1) : m;
      if (MODE == MODE_HALO && (BN == 32 || BN == 128) && p.pred_w && live) {
        float v0 = __ldg(p.pred_b), v1 = p.pred_nc > 1 ? __ldg(p.pred_b + 1) : 0.f;
#pragma unroll
        for (int j = 0; j < 32; j += 4) {
          const float4 w0 = __ldg(reinterpret_cast<const float4*>(p.pred_w + j));
          v0 = fmaf(o[j], w0.x, v0); v0 = fmaf(o[j + 1], w0.y, v0); v0 = fmaf(o[j + 2], w0.z, v0); v0 = fmaf(o[j + 3], w0.w, v0);
          if (p.pred_nc > 1) {
            const float4 w1 = __ldg(reinterpret_cast<const float4*>(p.pred_w + 32 + j));
            v1 = fmaf(o[j], w1.x, v1); v1 = fmaf(o[j + 1], w1.y, v1); v1 = fmaf(o[j + 2], w1.z, v1); v1 = fmaf(o[j + 3], w1.w, v1);
          }
        }
        const long long HWl = (long long)p.H * p.W * (ph4 ? 4 : 1);
        const long long bi = mo / HWl, pix = mo - bi * HWl;
        float* po = p.pred_out + bi * p.pred_nc * HWl + pix;
        if (p.pred_mode == 1) {
          const float nrm = fmaxf(sqrtf(v0 * v0 + v1 * v1), 1e-12f);
          po[0] = v0 / nrm; po[HWl] = v1 / nrm;
        } else {
          po[0] = fminf(fmaxf(v0, -1.f), 1.f);
        }
      }
      // Phase-mode stores (conv1's four output phases: rows are not one dense box).  A thread owns one row of the chunk (128 B of
      // fp32, 64 B per bf16 plane); storing it 16 bytes at a time makes every warp-wide store touch 32 half-filled sectors.  The
      // two lanes of an x-adjacent pixel pair exchange halves so that each store instruction writes 32 contiguous bytes per pair.
      if (ph4 && chunk_ok && (p.C || p.Shi)) {
        const bool odd = lane & 1;
        const bool valid_p = __shfl_xor_sync(0xffffffffu, (int)valid, 1) != 0;
        const long long mo_p = mo + (odd ? -2 : 2);                       // the partner's hi-res pixel (same image row, x +- 1)
        const long long moA = odd ? mo_p : mo, moB = odd ? mo : mo_p;     // row A = the even lane's, row B = the odd lane's
        const bool vA = odd ? valid_p : valid, vB = odd ? valid : valid_p;
        if (p.C) {
          float* cA = p.C + moA * p.ldc + p.c_coff + g * p.c_gcoff + (odd ? 4 : 0);
          float* cB = p.C + moB * p.ldc + p.c_coff + g * p.c_gcoff + (odd ? 4 : 0);
#pragma unroll
          for (int t = 0; t < 4; ++t) {      // float4 slots 2t (even lane) and 2t + 1 (odd lane) of both rows
            float k[4], rr[4];
#pragma unroll
            for (int e = 0; e < 4; ++e) {
              k[e] = odd ? o[8 * t + 4 + e] : o[8 * t + e];
              rr[e] = __shfl_xor_sync(0xffffffffu, odd ? o[8 * t + e] : o[8 * t + 4 + e], 1);
            }
            if (vA) *reinterpret_cast<float4*>(cA + 8 * t) = odd ? make_float4(rr[0], rr[1], rr[2], rr[3]) : make_float4(k[0], k[1], k[2], k[3]);
            if (vB) *reinterpret_cast<float4*>(cB + 8 * t) = odd ? make_float4(k[0], k[1], k[2], k[3]) : make_float4(rr[0], rr[1], rr[2], rr[3]);
          }
        }
        if (p.Shi) {
          const long long sA = moA * p.lds + p.s_coff + g * p.s_gcoff + (odd ? 8 : 0);
          const long long sB = moB * p.lds + p.s_coff + g * p.s_gcoff + (odd ? 8 : 0);
#pragma unroll
          for (int t = 0; t < 2; ++t) {      // 8-column slots 2t (even lane) and 2t + 1 (odd lane) of both rows
            float k[8], rr[8];
#pragma unroll
            for (int e = 0; e < 8; ++e) {
              const float mine = odd ? o[16 * t + 8 + e] : o[16 * t + e], give = odd ? o[16 * t + e] : o[16 * t + 8 + e];
              k[e] = p.split_relu ? fmaxf(mine, 0.f) : mine;
              rr[e] = __shfl_xor_sync(0xffffffffu, p.split_relu ? fmaxf(give, 0.f) : give, 1);
            }
            uint4 kh, kl, rh, rl;
            split_bf16x2(k[0], k[1], kh.x, kl.x); split_bf16x2(k[2], k[3], kh.y, kl.y);
            split_bf16x2(k[4], k[5], kh.z, kl.z); split_bf16x2(k[6], k[7], kh.w, kl.w);
            split_bf16x2(rr[0], rr[1], rh.x, rl.x); split_bf16x2(rr[2], rr[3], rh.y, rl.y);
            split_bf16x2(rr[4], rr[5], rh.z, rl.z); split_bf16x2(rr[6], rr[7], rh.w, rl.w);
            if (vA) {
              *reinterpret_cast<uint4*>(p.Shi + sA + 16 * t) = odd ? rh : kh;
              *reinterpret_cast<uint4*>(p.Slo + sA + 16 * t) = odd ? rl : kl;
            }
            if (vB) {
              *reinterpret_cast<uint4*>(p.Shi + sB + 16 * t) = odd ? kh : rh;
              *reinterpret_cast<uint4*>(p.Slo + sB + 16 * t) = odd ? kl : rl;
            }
          }
        }
      }
      // fp32 output: the round's results go back to the staging rows (free once every thread has read them), and the warpgroup
      // stores whole 256 B row segments: 16 lanes per row, 2 rows per instruction, instead of 16 B pieces of 32 rows.
      if (p.C && !ph4) {
        named_bar_sync(1 + wg, 128);              // every thread has read what the staging area holds
        if (own) {
          float* drow = stage + erow * Cfg::kAccPitch + eh * 32;
#pragma unroll
          for (int j = 0; j < 32; j += 4) *reinterpret_cast<float4*>(drow + j) = make_float4(o[j], o[j + 1], o[j + 2], o[j + 3]);
        }
        named_bar_sync(1 + wg, 128);
        float* cbase = p.C + p.c_coff + g * p.c_gcoff + n0;
#pragma unroll
        for (int t = 0; t < 8; ++t) {
          const int i = wt + 128 * t, col = rd * 64 + (i & 15) * 4;
          long long mr;
          if (col < BN && n0 + col < p.N && stage_row(i >> 4, mr))
            *reinterpret_cast<float4*>(cbase + mr * p.ldc + col) = *reinterpret_cast<const float4*>(stage + (i >> 4) * Cfg::kAccPitch + (i & 15) * 4);
        }
      }
      // Split planes: a thread's 32 columns are 64 B per plane, so stores from registers leave every 128 B line half written by
      // two warps (measured on H100: 3x slower than fp32 stores of the same bytes).  The round's bf16 hi / lo values go to
      // shared memory instead (the fp32 staging area, free once every thread has read it: 64 rows x 128 B per plane, 16 B
      // pieces XOR-swizzled by row), and the warpgroup stores whole 128 B row segments: 8 lanes per row, 4 rows per instruction.
      if (staged_split) {
        named_bar_sync(1 + wg, 128);              // every thread has read what the staging area holds
        unsigned char* sS = reinterpret_cast<unsigned char*>(stage);
        if (own) {
#pragma unroll
          for (int t = 0; t < 4; ++t) {           // 8-column pieces eh * 4 + t of row erow
            uint4 h, l;
            float k[8];
#pragma unroll
            for (int e = 0; e < 8; ++e) k[e] = p.split_relu ? fmaxf(o[8 * t + e], 0.f) : o[8 * t + e];
            split_bf16x2(k[0], k[1], h.x, l.x); split_bf16x2(k[2], k[3], h.y, l.y);
            split_bf16x2(k[4], k[5], h.z, l.z); split_bf16x2(k[6], k[7], h.w, l.w);
            const int off = erow * 128 + (((eh * 4 + t) ^ (erow & 7)) << 4);
            *reinterpret_cast<uint4*>(sS + off) = h;
            *reinterpret_cast<uint4*>(sS + 64 * 128 + off) = l;
          }
        }
        named_bar_sync(1 + wg, 128);
#pragma unroll
        for (int i = wt; i < 2 * 64 * 8; i += 128) {
          const int lo_plane = i >> 9, rr = (i >> 3) & 63, pc = i & 7;
          const int col = rd * 64 + pc * 8;       // column within the tile
          long long mr;
          if (col >= BN || n0 + col >= p.N || !stage_row(rr, mr)) continue;
          const uint4 v = *reinterpret_cast<const uint4*>(sS + lo_plane * 64 * 128 + rr * 128 + ((pc ^ (rr & 7)) << 4));
          *reinterpret_cast<uint4*>((lo_plane ? p.Slo : p.Shi) + mr * p.lds + p.s_coff + g * p.s_gcoff + n0 + col) = v;
        }
      }
    }
  }
}

}  // namespace pf
