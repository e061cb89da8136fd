// Spatial-reduction attention core on the tensor cores: softmax(q k^T / 8) v, 100 keys, head_dim 64
// (mix_transformers.py:127-131), split-precision bf16x3 products (lo*hi + hi*lo + hi*hi, fp32 accumulate) for both
// q k^T and p v, fp32 softmax.
//
//   block = 4 warps (3 blocks per SM), one (image, head); the bf16 hi/lo planes of the head's K and V are staged once in shared memory
//   (keys padded 100 -> 112, rows of 128 B, 16 B chunks XOR-swizzled for conflict-free ldmatrix); the block then loops over
//   passes of 64 queries (16 per warp); passes per block are chosen so that the grid is about one resident wave.  Per warp and tile: S = q k^T (mma.sync.m16n8k16, 4 k-steps x 14 key tiles x 3),
//   row softmax in registers (quad shuffles), O = P V (7 k-steps x 8 tiles x 3; P re-used from the S accumulators as the A
//   operand, V through ldmatrix.trans), normalise, store fp32 and/or split planes.
//
//   NP = 1 (the opt-in bf16 precision mode): K and V are staged as hi planes only (28 KB per block), Q fragments are hi only,
//   and each product is one mma.sync (hi*hi) with P rounded to bf16 once.  The softmax stays fp32.
#pragma once
#include "common.cuh"

namespace pf {

constexpr int kAmKeys = 100, kAmKeysPad = 112, kAmD = 64, kAmQTile = 64, kAmThreads = 128;   // 4 warps x 16 queries per pass
constexpr int kAmPlane = kAmKeysPad * kAmD * 2;      // bytes of one bf16 plane (K or V, hi or lo)
constexpr int kAmSmem = 4 * kAmPlane;                // K_hi, K_lo, V_hi, V_lo = 57344 B
template <int NP> constexpr int am_smem() { return NP == 3 ? kAmSmem : 2 * kAmPlane; }   // NP = 1: K_hi, V_hi

__device__ __forceinline__ void ldmatrix_x4_trans(uint32_t addr, uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];\n"
               : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3) : "r"(addr));
}

// q and kv arrive as bf16 hi/lo planes (written by the q / kv GEMM epilogues): K and V are copied into shared memory
// with cp.async (no conversion work), Q fragments are read as bf16 pairs; the 1/8 scale is applied to S in fp32 (a power of
// two: identical to scaling q).
// KEYS: the key count (100: every stage at a 320 x 320 working size); 0 = the run-time count `nkv_rt` (at most kAmKeysPad).
template <int NP = 3, int KEYS = kAmKeys>
__global__ void __launch_bounds__(kAmThreads) attention_mma_kernel(const __nv_bfloat16* __restrict__ q_hi, const __nv_bfloat16* __restrict__ q_lo,
                                                                   const __nv_bfloat16* __restrict__ kv_hi, const __nv_bfloat16* __restrict__ kv_lo,
                                                                   float* __restrict__ out,
                                                                   __nv_bfloat16* __restrict__ shi, __nv_bfloat16* __restrict__ slo, int N, int C,
                                                                   int tiles_per_block, int nkv_rt) {
  static_assert(NP == 1 || NP == 3, "NP");
  static_assert(KEYS >= 0 && KEYS <= kAmKeysPad, "KEYS");
  const int nkv = KEYS ? KEYS : nkv_rt;
  constexpr bool kLo = NP == 3;
  constexpr int kPl = kLo ? 2 : 1;                    // planes per operand (K, V): hi + lo, or hi
  pdl_wait();
  pdl_launch();
  extern __shared__ __align__(128) unsigned char sm_raw[];
  const uint32_t sK_hi = smem_u32(sm_raw), sK_lo = sK_hi + kAmPlane, sV_hi = sK_hi + kPl * kAmPlane, sV_lo = sV_hi + kAmPlane;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int b = blockIdx.z, h = blockIdx.y;
  // ---- stage K and V of this (image, head): [key][64] rows of 128 B, chunk (16 B) index ^= key & 7
  {
    // 2 kPl planes (K_hi, K_lo, V_hi, V_lo; NP = 1: K_hi, V_hi) x 112 keys x 8 chunks of 16 B
    const long long kvo = (long long)b * nkv * 2 * C + h * kAmD;
    for (int i = tid; i < 2 * kPl * kAmKeysPad * 8; i += kAmThreads) {
      const int plane = i / (kAmKeysPad * 8), j = i % (kAmKeysPad * 8), key = j >> 3, c = j & 7;
      const uint32_t dst = sK_hi + plane * kAmPlane + (uint32_t)key * 128u + (uint32_t)((c ^ (key & 7)) << 4);
      const bool valid = key < nkv;    // keys nkv..111: zero fill (src-size 0)
      const int lo = plane % kPl, isv = plane / kPl;
      const __nv_bfloat16* src = (lo ? kv_lo : kv_hi) + kvo + (long long)(valid ? key : 0) * 2 * C + (isv ? C : 0) + c * 8;
      cp_async16(dst, src, valid);
    }
    cp_async_commit();
    cp_async_wait<0>();
  }
  __syncthreads();

  const int g = lane >> 2, t = lane & 3;
  for (int it = 0; it < tiles_per_block; ++it) {
    const int q0 = (blockIdx.x * tiles_per_block + it) * kAmQTile + warp * 16;   // first query row of this warp
    if (q0 >= N) break;                                                         // warp-uniform
    const int r0 = q0 + g, r1 = q0 + g + 8;
    // ---- Q fragments, hi / lo
    uint32_t qh[4][4], ql[4][4];
    const long long o0 = ((long long)b * N + (r0 < N ? r0 : N - 1)) * C + h * kAmD, o1 = ((long long)b * N + (r1 < N ? r1 : N - 1)) * C + h * kAmD;
#pragma unroll
    for (int ks = 0; ks < 4; ++ks) {
      const int c0 = ks * 16 + 2 * t;
      qh[ks][0] = __ldg(reinterpret_cast<const uint32_t*>(q_hi + o0 + c0));
      qh[ks][1] = __ldg(reinterpret_cast<const uint32_t*>(q_hi + o1 + c0));
      qh[ks][2] = __ldg(reinterpret_cast<const uint32_t*>(q_hi + o0 + c0 + 8));
      qh[ks][3] = __ldg(reinterpret_cast<const uint32_t*>(q_hi + o1 + c0 + 8));
      if (kLo) {
        ql[ks][0] = __ldg(reinterpret_cast<const uint32_t*>(q_lo + o0 + c0));
        ql[ks][1] = __ldg(reinterpret_cast<const uint32_t*>(q_lo + o1 + c0));
        ql[ks][2] = __ldg(reinterpret_cast<const uint32_t*>(q_lo + o0 + c0 + 8));
        ql[ks][3] = __ldg(reinterpret_cast<const uint32_t*>(q_lo + o1 + c0 + 8));
      }
    }
    // ---- S = Q K^T : 16 x 112
    float s[14][4];
#pragma unroll
    for (int nt = 0; nt < 14; ++nt) { s[nt][0] = s[nt][1] = s[nt][2] = s[nt][3] = 0.f; }
#pragma unroll
    for (int ks = 0; ks < 4; ++ks) {
#pragma unroll
      for (int np = 0; np < 7; ++np) {
        // two key tiles (16 keys) x 16 d: matrices (keys 0-7, d 0-7), (keys 0-7, d 8-15), (keys 8-15, d 0-7), (keys 8-15, d 8-15)
        const int key = np * 16 + (lane & 7) + ((lane >> 4) << 3);
        const int chunk = ks * 2 + ((lane >> 3) & 1);
        const uint32_t off = (uint32_t)key * 128u + (uint32_t)((chunk ^ (key & 7)) << 4);
        uint32_t bh0, bh1, bh2, bh3;
        ldmatrix_x4(sK_hi + off, bh0, bh1, bh2, bh3);
        if (kLo) {
          uint32_t bl0, bl1, bl2, bl3;
          ldmatrix_x4(sK_lo + off, bl0, bl1, bl2, bl3);
          mma_bf16_16816(s[2 * np], ql[ks], bh0, bh1);
          mma_bf16_16816(s[2 * np], qh[ks], bl0, bl1);
          mma_bf16_16816(s[2 * np], qh[ks], bh0, bh1);
          mma_bf16_16816(s[2 * np + 1], ql[ks], bh2, bh3);
          mma_bf16_16816(s[2 * np + 1], qh[ks], bl2, bl3);
          mma_bf16_16816(s[2 * np + 1], qh[ks], bh2, bh3);
        } else {
          mma_bf16_16816(s[2 * np], qh[ks], bh0, bh1);
          mma_bf16_16816(s[2 * np + 1], qh[ks], bh2, bh3);
        }
      }
    }
    // ---- softmax over the nkv valid keys (rows r0: regs 0,1 ; r1: regs 2,3), fp32
    float m0 = -INFINITY, m1 = -INFINITY;
#pragma unroll
    for (int nt = 0; nt < 14; ++nt) {
      const int k0 = nt * 8 + 2 * t;
      s[nt][0] *= 0.125f; s[nt][1] *= 0.125f; s[nt][2] *= 0.125f; s[nt][3] *= 0.125f;
      if (k0 >= nkv) { s[nt][0] = -INFINITY; s[nt][2] = -INFINITY; }
      if (k0 + 1 >= nkv) { s[nt][1] = -INFINITY; s[nt][3] = -INFINITY; }
      m0 = fmaxf(m0, fmaxf(s[nt][0], s[nt][1]));
      m1 = fmaxf(m1, fmaxf(s[nt][2], s[nt][3]));
    }
    m0 = fmaxf(m0, __shfl_xor_sync(0xffffffffu, m0, 1)); m0 = fmaxf(m0, __shfl_xor_sync(0xffffffffu, m0, 2));
    m1 = fmaxf(m1, __shfl_xor_sync(0xffffffffu, m1, 1)); m1 = fmaxf(m1, __shfl_xor_sync(0xffffffffu, m1, 2));
    float l0 = 0.f, l1 = 0.f;
#pragma unroll
    for (int nt = 0; nt < 14; ++nt) {
      s[nt][0] = expf(s[nt][0] - m0); s[nt][1] = expf(s[nt][1] - m0);
      s[nt][2] = expf(s[nt][2] - m1); s[nt][3] = expf(s[nt][3] - m1);
      l0 += s[nt][0] + s[nt][1];
      l1 += s[nt][2] + s[nt][3];
    }
    l0 += __shfl_xor_sync(0xffffffffu, l0, 1); l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
    l1 += __shfl_xor_sync(0xffffffffu, l1, 1); l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
    // ---- O = P V : 16 x 64, P taken from the S accumulators (A fragment of k-step j = key tiles 2j, 2j+1)
    float o[8][4];
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) { o[nt][0] = o[nt][1] = o[nt][2] = o[nt][3] = 0.f; }
#pragma unroll
    for (int j = 0; j < 7; ++j) {
      uint32_t ph[4], pl[4];
      split_bf16x2(s[2 * j][0], s[2 * j][1], ph[0], pl[0]);
      split_bf16x2(s[2 * j][2], s[2 * j][3], ph[1], pl[1]);
      split_bf16x2(s[2 * j + 1][0], s[2 * j + 1][1], ph[2], pl[2]);
      split_bf16x2(s[2 * j + 1][2], s[2 * j + 1][3], ph[3], pl[3]);
#pragma unroll
      for (int np = 0; np < 4; ++np) {
        // V[key][d] rows = k: transposed 8x8 loads: (k 0-7, d 0-7), (k 8-15, d 0-7), (k 0-7, d 8-15), (k 8-15, d 8-15)
        const int key = j * 16 + (lane & 7) + (((lane >> 3) & 1) << 3);
        const int chunk = np * 2 + (lane >> 4);
        const uint32_t off = (uint32_t)key * 128u + (uint32_t)((chunk ^ (key & 7)) << 4);
        uint32_t vh0, vh1, vh2, vh3;
        ldmatrix_x4_trans(sV_hi + off, vh0, vh1, vh2, vh3);
        if (kLo) {
          uint32_t vl0, vl1, vl2, vl3;
          ldmatrix_x4_trans(sV_lo + off, vl0, vl1, vl2, vl3);
          mma_bf16_16816(o[2 * np], pl, vh0, vh1);
          mma_bf16_16816(o[2 * np], ph, vl0, vl1);
          mma_bf16_16816(o[2 * np], ph, vh0, vh1);
          mma_bf16_16816(o[2 * np + 1], pl, vh2, vh3);
          mma_bf16_16816(o[2 * np + 1], ph, vl2, vl3);
          mma_bf16_16816(o[2 * np + 1], ph, vh2, vh3);
        } else {
          mma_bf16_16816(o[2 * np], ph, vh0, vh1);
          mma_bf16_16816(o[2 * np + 1], ph, vh2, vh3);
        }
      }
    }
    // ---- normalise and store (row r0: regs 0,1 ; row r1: regs 2,3 ; columns nt*8 + 2t, +1)
    const float i0 = 1.0f / l0, i1 = 1.0f / l1;
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) {
      const int d = nt * 8 + 2 * t;
      if (r0 < N) {
        const long long oi = ((long long)b * N + r0) * C + h * kAmD + d;
        const float x = o[nt][0] * i0, y = o[nt][1] * i0;
        if (out) *reinterpret_cast<float2*>(out + oi) = make_float2(x, y);
        if (shi) { uint32_t hh, ll; split_bf16x2(x, y, hh, ll); *reinterpret_cast<uint32_t*>(shi + oi) = hh; *reinterpret_cast<uint32_t*>(slo + oi) = ll; }
      }
      if (r1 < N) {
        const long long oi = ((long long)b * N + r1) * C + h * kAmD + d;
        const float x = o[nt][2] * i1, y = o[nt][3] * i1;
        if (out) *reinterpret_cast<float2*>(out + oi) = make_float2(x, y);
        if (shi) { uint32_t hh, ll; split_bf16x2(x, y, hh, ll); *reinterpret_cast<uint32_t*>(shi + oi) = hh; *reinterpret_cast<uint32_t*>(slo + oi) = ll; }
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------------------
// Key-block path: more than kAmKeysPad keys (working sizes other than 320 x 320: (H/32) * (W/32) keys, up to kAmMaxKeys).
// Same block (4 warps, one (image, head), 16 queries per warp and pass) and the same staging, with
// K and V resident in shared memory for all keys (padded to 16): 4 planes x 256 keys x 128 B = 128 KB at NP = 3, half at NP = 1.
// The warp loops over blocks of 64 keys with an online (running-max) fp32 softmax: S of one key block is 8 tiles (32 registers
// per thread instead of 4 * keys / 8), the running output O is rescaled by exp(m_old - m_new) before each block's P V.
constexpr int kAmMaxKeys = 256, kAmKeyBlock = 64;
template <int NP> constexpr int am_kb_smem(int nkv_pad) { return 2 * (NP == 3 ? 2 : 1) * nkv_pad * kAmD * 2; }
constexpr int kAmKbSmemMax = am_kb_smem<3>(kAmMaxKeys);   // 131072 B

template <int NP>
__global__ void __launch_bounds__(kAmThreads) attention_mma_kb_kernel(const __nv_bfloat16* __restrict__ q_hi, const __nv_bfloat16* __restrict__ q_lo,
                                                                      const __nv_bfloat16* __restrict__ kv_hi, const __nv_bfloat16* __restrict__ kv_lo,
                                                                      float* __restrict__ out, __nv_bfloat16* __restrict__ shi, __nv_bfloat16* __restrict__ slo,
                                                                      int N, int C, int tiles_per_block, int nkv) {
  static_assert(NP == 1 || NP == 3, "NP");
  constexpr bool kLo = NP == 3;
  constexpr int kPl = kLo ? 2 : 1;
  pdl_wait();
  pdl_launch();
  extern __shared__ __align__(128) unsigned char sm_raw[];
  const int kpad = (nkv + 15) & ~15;
  const uint32_t plane = (uint32_t)kpad * 128u;
  const uint32_t sK_hi = smem_u32(sm_raw), sK_lo = sK_hi + plane, sV_hi = sK_hi + kPl * plane, sV_lo = sV_hi + plane;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int b = blockIdx.z, h = blockIdx.y;
  {
    const long long kvo = (long long)b * nkv * 2 * C + h * kAmD;
    for (int i = tid; i < 2 * kPl * kpad * 8; i += kAmThreads) {
      const int pl = i / (kpad * 8), j = i % (kpad * 8), key = j >> 3, c = j & 7;
      const uint32_t dst = sK_hi + pl * plane + (uint32_t)key * 128u + (uint32_t)((c ^ (key & 7)) << 4);
      const bool valid = key < nkv;
      const int lo = pl % kPl, isv = pl / kPl;
      const __nv_bfloat16* src = (lo ? kv_lo : kv_hi) + kvo + (long long)(valid ? key : 0) * 2 * C + (isv ? C : 0) + c * 8;
      cp_async16(dst, src, valid);
    }
    cp_async_commit();
    cp_async_wait<0>();
  }
  __syncthreads();

  const int g = lane >> 2, t = lane & 3;
  for (int it = 0; it < tiles_per_block; ++it) {
    const int q0 = (blockIdx.x * tiles_per_block + it) * kAmQTile + warp * 16;
    if (q0 >= N) break;                                                         // warp-uniform
    const int r0 = q0 + g, r1 = q0 + g + 8;
    uint32_t qh[4][4], ql[4][4];
    const long long o0 = ((long long)b * N + (r0 < N ? r0 : N - 1)) * C + h * kAmD, o1 = ((long long)b * N + (r1 < N ? r1 : N - 1)) * C + h * kAmD;
#pragma unroll
    for (int ks = 0; ks < 4; ++ks) {
      const int c0 = ks * 16 + 2 * t;
      qh[ks][0] = __ldg(reinterpret_cast<const uint32_t*>(q_hi + o0 + c0));
      qh[ks][1] = __ldg(reinterpret_cast<const uint32_t*>(q_hi + o1 + c0));
      qh[ks][2] = __ldg(reinterpret_cast<const uint32_t*>(q_hi + o0 + c0 + 8));
      qh[ks][3] = __ldg(reinterpret_cast<const uint32_t*>(q_hi + o1 + c0 + 8));
      if (kLo) {
        ql[ks][0] = __ldg(reinterpret_cast<const uint32_t*>(q_lo + o0 + c0));
        ql[ks][1] = __ldg(reinterpret_cast<const uint32_t*>(q_lo + o1 + c0));
        ql[ks][2] = __ldg(reinterpret_cast<const uint32_t*>(q_lo + o0 + c0 + 8));
        ql[ks][3] = __ldg(reinterpret_cast<const uint32_t*>(q_lo + o1 + c0 + 8));
      }
    }
    float o[8][4];
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) { o[nt][0] = o[nt][1] = o[nt][2] = o[nt][3] = 0.f; }
    float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;    // running max (quad-uniform) and this thread's partial sums
    // every key block holds at least one valid key (kb0 < kpad <= nkv + 15): its row maxima are finite
    for (int kb0 = 0; kb0 < kpad; kb0 += kAmKeyBlock) {
      // ---- S = Q K^T : 16 x 64 (16-key tiles at or past kpad are skipped; warp-uniform)
      float s[8][4];
#pragma unroll
      for (int nt = 0; nt < 8; ++nt) { s[nt][0] = s[nt][1] = s[nt][2] = s[nt][3] = 0.f; }
#pragma unroll
      for (int ks = 0; ks < 4; ++ks) {
#pragma unroll
        for (int np = 0; np < 4; ++np) {
          if (kb0 + np * 16 >= kpad) break;
          const int key = kb0 + np * 16 + (lane & 7) + ((lane >> 4) << 3);
          const int chunk = ks * 2 + ((lane >> 3) & 1);
          const uint32_t off = (uint32_t)key * 128u + (uint32_t)((chunk ^ (key & 7)) << 4);
          uint32_t bh0, bh1, bh2, bh3;
          ldmatrix_x4(sK_hi + off, bh0, bh1, bh2, bh3);
          if (kLo) {
            uint32_t bl0, bl1, bl2, bl3;
            ldmatrix_x4(sK_lo + off, bl0, bl1, bl2, bl3);
            mma_bf16_16816(s[2 * np], ql[ks], bh0, bh1);
            mma_bf16_16816(s[2 * np], qh[ks], bl0, bl1);
            mma_bf16_16816(s[2 * np], qh[ks], bh0, bh1);
            mma_bf16_16816(s[2 * np + 1], ql[ks], bh2, bh3);
            mma_bf16_16816(s[2 * np + 1], qh[ks], bl2, bl3);
            mma_bf16_16816(s[2 * np + 1], qh[ks], bh2, bh3);
          } else {
            mma_bf16_16816(s[2 * np], qh[ks], bh0, bh1);
            mma_bf16_16816(s[2 * np + 1], qh[ks], bh2, bh3);
          }
        }
      }
      // ---- online softmax (fp32): block maxima, rescale of the running state, exponentials
      float x0 = -INFINITY, x1 = -INFINITY;
#pragma unroll
      for (int nt = 0; nt < 8; ++nt) {
        const int k0 = kb0 + nt * 8 + 2 * t;
        s[nt][0] *= 0.125f; s[nt][1] *= 0.125f; s[nt][2] *= 0.125f; s[nt][3] *= 0.125f;
        if (k0 >= nkv) { s[nt][0] = -INFINITY; s[nt][2] = -INFINITY; }
        if (k0 + 1 >= nkv) { s[nt][1] = -INFINITY; s[nt][3] = -INFINITY; }
        x0 = fmaxf(x0, fmaxf(s[nt][0], s[nt][1]));
        x1 = fmaxf(x1, fmaxf(s[nt][2], s[nt][3]));
      }
      x0 = fmaxf(x0, __shfl_xor_sync(0xffffffffu, x0, 1)); x0 = fmaxf(x0, __shfl_xor_sync(0xffffffffu, x0, 2));
      x1 = fmaxf(x1, __shfl_xor_sync(0xffffffffu, x1, 1)); x1 = fmaxf(x1, __shfl_xor_sync(0xffffffffu, x1, 2));
      const float n0 = fmaxf(m0, x0), n1 = fmaxf(m1, x1);
      const float a0 = expf(m0 - n0), a1 = expf(m1 - n1);      // 0 for the first block (m = -inf)
      m0 = n0; m1 = n1;
      l0 *= a0; l1 *= a1;
#pragma unroll
      for (int nt = 0; nt < 8; ++nt) {
        s[nt][0] = expf(s[nt][0] - m0); s[nt][1] = expf(s[nt][1] - m0);
        s[nt][2] = expf(s[nt][2] - m1); s[nt][3] = expf(s[nt][3] - m1);
        l0 += s[nt][0] + s[nt][1];
        l1 += s[nt][2] + s[nt][3];
        o[nt][0] *= a0; o[nt][1] *= a0; o[nt][2] *= a1; o[nt][3] *= a1;
      }
      // ---- O += P V over this key block
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        if (kb0 + j * 16 >= kpad) break;
        uint32_t ph[4], pl[4];
        split_bf16x2(s[2 * j][0], s[2 * j][1], ph[0], pl[0]);
        split_bf16x2(s[2 * j][2], s[2 * j][3], ph[1], pl[1]);
        split_bf16x2(s[2 * j + 1][0], s[2 * j + 1][1], ph[2], pl[2]);
        split_bf16x2(s[2 * j + 1][2], s[2 * j + 1][3], ph[3], pl[3]);
#pragma unroll
        for (int np = 0; np < 4; ++np) {
          const int key = kb0 + j * 16 + (lane & 7) + (((lane >> 3) & 1) << 3);
          const int chunk = np * 2 + (lane >> 4);
          const uint32_t off = (uint32_t)key * 128u + (uint32_t)((chunk ^ (key & 7)) << 4);
          uint32_t vh0, vh1, vh2, vh3;
          ldmatrix_x4_trans(sV_hi + off, vh0, vh1, vh2, vh3);
          if (kLo) {
            uint32_t vl0, vl1, vl2, vl3;
            ldmatrix_x4_trans(sV_lo + off, vl0, vl1, vl2, vl3);
            mma_bf16_16816(o[2 * np], pl, vh0, vh1);
            mma_bf16_16816(o[2 * np], ph, vl0, vl1);
            mma_bf16_16816(o[2 * np], ph, vh0, vh1);
            mma_bf16_16816(o[2 * np + 1], pl, vh2, vh3);
            mma_bf16_16816(o[2 * np + 1], ph, vl2, vl3);
            mma_bf16_16816(o[2 * np + 1], ph, vh2, vh3);
          } else {
            mma_bf16_16816(o[2 * np], ph, vh0, vh1);
            mma_bf16_16816(o[2 * np + 1], ph, vh2, vh3);
          }
        }
      }
    }
    l0 += __shfl_xor_sync(0xffffffffu, l0, 1); l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
    l1 += __shfl_xor_sync(0xffffffffu, l1, 1); l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
    const float i0 = 1.0f / l0, i1 = 1.0f / l1;
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) {
      const int d = nt * 8 + 2 * t;
      if (r0 < N) {
        const long long oi = ((long long)b * N + r0) * C + h * kAmD + d;
        const float x = o[nt][0] * i0, y = o[nt][1] * i0;
        if (out) *reinterpret_cast<float2*>(out + oi) = make_float2(x, y);
        if (shi) { uint32_t hh, ll; split_bf16x2(x, y, hh, ll); *reinterpret_cast<uint32_t*>(shi + oi) = hh; *reinterpret_cast<uint32_t*>(slo + oi) = ll; }
      }
      if (r1 < N) {
        const long long oi = ((long long)b * N + r1) * C + h * kAmD + d;
        const float x = o[nt][2] * i1, y = o[nt][3] * i1;
        if (out) *reinterpret_cast<float2*>(out + oi) = make_float2(x, y);
        if (shi) { uint32_t hh, ll; split_bf16x2(x, y, hh, ll); *reinterpret_cast<uint32_t*>(shi + oi) = hh; *reinterpret_cast<uint32_t*>(slo + oi) = ll; }
      }
    }
  }
}

inline cudaError_t attention_mma_configure_device() {   // per-device shared-memory opt-in (pf_create)
  cudaError_t e = cudaFuncSetAttribute(attention_mma_kernel<3>, cudaFuncAttributeMaxDynamicSharedMemorySize, kAmSmem);
  if (e == cudaSuccess) e = cudaFuncSetAttribute(attention_mma_kernel<3, 0>, cudaFuncAttributeMaxDynamicSharedMemorySize, kAmSmem);
  if (e == cudaSuccess) e = cudaFuncSetAttribute(attention_mma_kb_kernel<3>, cudaFuncAttributeMaxDynamicSharedMemorySize, kAmKbSmemMax);
  if (e == cudaSuccess) e = cudaFuncSetAttribute(attention_mma_kb_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, am_kb_smem<1>(kAmMaxKeys));
  return e;   // (the single-block NP = 1 instantiations use 28 KB: no opt-in)
}

template <int NP>
inline cudaError_t attention_mma_launch_np(float* out, dim3 grid, int N, int C, int tpb, cudaStream_t st, SplitT sp, SplitT qs, SplitT kvs, int nkv) {
  if (nkv != kAmKeys)   // run-time key count (<= kAmKeysPad)
    return launch_pdl(attention_mma_kernel<NP, 0>, grid, dim3(kAmThreads), am_smem<NP>(), st, qs.hi, qs.lo, kvs.hi, kvs.lo, out, sp.hi, sp.lo, N, C, tpb, nkv);
  return launch_pdl(attention_mma_kernel<NP>, grid, dim3(kAmThreads), am_smem<NP>(), st, qs.hi, qs.lo, kvs.hi, kvs.lo, out, sp.hi, sp.lo, N, C, tpb, nkv);
}

// resident blocks per SM of the key-block kernel (228 KB of shared memory per SM, 1 KB of it reserved per block; at most 4)
inline int attention_kb_blocks_per_sm(int nkv, int np) {
  const int smem = (np == 3 ? am_kb_smem<3>((nkv + 15) & ~15) : am_kb_smem<1>((nkv + 15) & ~15)) + 1024;
  const int b = (228 * 1024) / smem;
  return b < 1 ? 1 : (b > 4 ? 4 : b);
}

// qs / kvs: q and kv as split planes with row pitch C / 2C; the result goes to the split planes sp and / or the fp32 tensor out
// (either may be empty).  np = bf16 products per output: 3 (split precision) or 1 (bf16 precision mode: only the hi planes of
// qs / kvs are read).  nkv: keys per image (kv holds nkv rows per image): 100 = the 320 x 320 kernel; other counts up to
// kAmKeysPad run the single-block kernel with a run-time count, larger ones (up to kAmMaxKeys) the key-block kernel.
inline cudaError_t attention_mma_launch(float* out, int B, int N, int C, int heads, cudaStream_t st, SplitT sp, SplitT qs, SplitT kvs, int np = 3,
                                        int nkv = kAmKeys) {
  if (!qs.hi || !kvs.hi || qs.ld != C || kvs.ld != 2 * C) return cudaErrorInvalidValue;
  if (nkv < 1 || nkv > kAmMaxKeys || (np != 1 && np != 3)) return cudaErrorInvalidValue;
  const int tiles = cdiv(N, kAmQTile);
  if (nkv > kAmKeysPad) {
    // one resident wave of 132 SMs x the blocks per SM the key-block kernel's shared memory allows
    int tpb = (tiles * heads * B) / (132 * attention_kb_blocks_per_sm(nkv, np));
    tpb = tpb < 1 ? 1 : (tpb > tiles ? tiles : tpb);
    const dim3 grid(cdiv(tiles, tpb), heads, B);
    const int kpad = (nkv + 15) & ~15;
    if (np == 1) return launch_pdl(attention_mma_kb_kernel<1>, grid, dim3(kAmThreads), am_kb_smem<1>(kpad), st, qs.hi, qs.lo, kvs.hi, kvs.lo, out, sp.hi, sp.lo, N, C, tpb, nkv);
    return launch_pdl(attention_mma_kb_kernel<3>, grid, dim3(kAmThreads), am_kb_smem<3>(kpad), st, qs.hi, qs.lo, kvs.hi, kvs.lo, out, sp.hi, sp.lo, N, C, tpb, nkv);
  }
  // passes per block: the grid should be about one resident wave (132 SMs x 3 blocks); the K/V staging of a block is
  // amortised over tpb * 64 queries
  int tpb = (tiles * heads * B) / 396;
  tpb = tpb < 1 ? 1 : (tpb > tiles ? tiles : tpb);
  dim3 grid(cdiv(tiles, tpb), heads, B);
  if (np == 1) return attention_mma_launch_np<1>(out, grid, N, C, tpb, st, sp, qs, kvs, nkv);
  return attention_mma_launch_np<3>(out, grid, N, C, tpb, st, sp, qs, kvs, nkv);
}

}  // namespace pf
