// CUDA-core kernels of the inference path: the ParamNet stem, LayerNorm, depthwise convs,
// x2 bilinear upsample, prediction tails and the ParamNet pooling/regression tail.  All activations NHWC fp32.
#pragma once
#include "common.cuh"

namespace pf {

// =====================================================================================================
// Direct fp32 convolution for the ParamNet (ConvNeXt) stem, conv4x4/4 p0 3->96 (+bias), convnext.py:88-91
// (K = KH*KW*3 = 48 is too small for the MMA tile).
// in : [B, H, W, ldin] (first 3 channels used); w: [(ky,kx,ci)][COUT]; out: [B, OH, OW, COUT].
// Block = PIX_PER_BLOCK output pixels of one row x COUT channels; thread = 1 channel x PPT pixels.
template <int KH, int KW, int STRIDE, int PAD, int COUT, int PPT, int PGROUPS>
__global__ void __launch_bounds__(COUT* PGROUPS) stem_conv_kernel(const float* __restrict__ in, int ldin, int B, int H, int W,
                                                                  const float* __restrict__ w, const float* __restrict__ bias,
                                                                  float* __restrict__ out, int OH, int OW) {
  constexpr int PIX = PPT * PGROUPS;                   // output pixels per block (along x)
  constexpr int IN_W = (PIX - 1) * STRIDE + KW;        // input columns needed
  __shared__ float s_in[KH][IN_W][3];
  const int tiles_x = cdiv(OW, PIX);
  int bid = blockIdx.x;
  const int tx = bid % tiles_x; bid /= tiles_x;
  const int oy = bid % OH; const int b = bid / OH;
  const int ox0 = tx * PIX;
  const int iy0 = oy * STRIDE - PAD, ix0 = ox0 * STRIDE - PAD;
  for (int i = threadIdx.x; i < KH * IN_W * 3; i += blockDim.x) {
    const int c = i % 3, x = (i / 3) % IN_W, y = i / (3 * IN_W);
    const int iy = iy0 + y, ix = ix0 + x;
    float v = 0.f;
    if ((unsigned)iy < (unsigned)H && (unsigned)ix < (unsigned)W) v = __ldg(in + ((long long)(b * H + iy) * W + ix) * ldin + c);
    s_in[y][x][c] = v;
  }
  __syncthreads();
  const int co = threadIdx.x % COUT, pg = threadIdx.x / COUT;
  float acc[PPT];
  const float bv = bias ? __ldg(bias + co) : 0.f;
#pragma unroll
  for (int j = 0; j < PPT; ++j) acc[j] = bv;
#pragma unroll 1
  for (int ky = 0; ky < KH; ++ky) {
#pragma unroll
    for (int kx = 0; kx < KW; ++kx) {
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        const float wv = __ldg(w + ((ky * KW + kx) * 3 + c) * COUT + co);
#pragma unroll
        for (int j = 0; j < PPT; ++j) acc[j] = fmaf(s_in[ky][(pg * PPT + j) * STRIDE + kx][c], wv, acc[j]);
      }
    }
  }
#pragma unroll
  for (int j = 0; j < PPT; ++j) {
    const int ox = ox0 + pg * PPT + j;
    if (ox < OW) out[((long long)(b * OH + oy) * OW + ox) * COUT + co] = acc[j];
  }
}

template <int KH, int KW, int STRIDE, int PAD, int COUT>
inline cudaError_t stem_conv_launch(const float* in, int ldin, int B, int H, int W, const float* w, const float* bias,
                                    float* out, cudaStream_t st) {
  constexpr int PPT = 4, PGROUPS = (COUT == 64) ? 4 : 2;
  const int OH = (H + 2 * PAD - KH) / STRIDE + 1, OW = (W + 2 * PAD - KW) / STRIDE + 1;
  const int tiles_x = cdiv(OW, PPT * PGROUPS);
  stem_conv_kernel<KH, KW, STRIDE, PAD, COUT, PPT, PGROUPS><<<B * OH * tiles_x, COUT * PGROUPS, 0, st>>>(in, ldin, B, H, W, w, bias, out, OH, OW);
  return cudaGetLastError();
}

// =====================================================================================================
// LayerNorm over the channel dimension of [rows, C] (nn.LayerNorm / F.layer_norm, biased variance, eps inside
// the sqrt) -- mix_transformers.py:199-200,247,120,457 and convnext.py:172-182 (both data formats reduce to this
// in NHWC).  One warp per row; two-pass (mean, then centred variance) in registers.
// NR independent rows per lane group are in flight at once (all their loads are issued before the first reduction): with one row
// per warp the kernel was bound by the latency of that single load, not by bandwidth.  Index arithmetic is 32-bit in float4 units
// (rows * C / 4 < 2^32, checked by the launcher).
template <int MAXQ, int LANES, int NR>   // float4 quads per lane; LANES (32 or 16) lanes cooperate on one row: lane owns quads lane + LANES*i
__global__ void __launch_bounds__(256) layernorm_kernel(const float* __restrict__ in, float* __restrict__ out, long long rows_ll, int C,
                                                        const float* __restrict__ gw, const float* __restrict__ gb, float eps,
                                                        __nv_bfloat16* __restrict__ shi, __nv_bfloat16* __restrict__ slo,
                                                        __nv_bfloat16* __restrict__ phi, __nv_bfloat16* __restrict__ plo, int RH, int RW, int sr) {
  pdl_wait();
  pdl_launch();
  constexpr int RPW = 32 / LANES;       // lane groups (rows) per warp
  const unsigned lane = threadIdx.x & (LANES - 1);
  const unsigned rows = (unsigned)rows_ll;
  const unsigned row0 = ((blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5)) * RPW + ((threadIdx.x & 31) / LANES)) * NR;
  const unsigned Q = (unsigned)C >> 2;
  const float inv_c = 1.0f / (float)C;
  const float4* __restrict__ in4 = reinterpret_cast<const float4*>(in);
  float4 v[NR][MAXQ];
  float s[NR], q[NR];
#pragma unroll
  for (int j = 0; j < NR; ++j) {
    const bool ok = row0 + j < rows;
    const unsigned xb = (ok ? row0 + j : 0u) * Q;
    s[j] = 0.f;
#pragma unroll
    for (int i = 0; i < MAXQ; ++i) {
      const unsigned qd = lane + LANES * i;
      v[j][i] = make_float4(0.f, 0.f, 0.f, 0.f);
      if (ok && qd < Q) v[j][i] = __ldg(in4 + (xb + qd));
      s[j] += (v[j][i].x + v[j][i].y) + (v[j][i].z + v[j][i].w);
    }
  }
#pragma unroll
  for (int o = LANES / 2; o > 0; o >>= 1)
#pragma unroll
    for (int j = 0; j < NR; ++j) s[j] += __shfl_xor_sync(0xffffffffu, s[j], o);
#pragma unroll
  for (int j = 0; j < NR; ++j) {
    s[j] *= inv_c;                      // mean
    q[j] = 0.f;
#pragma unroll
    for (int i = 0; i < MAXQ; ++i) {
      if (lane + LANES * i < Q) {
        const float a = v[j][i].x - s[j], b = v[j][i].y - s[j], c = v[j][i].z - s[j], d = v[j][i].w - s[j];
        q[j] = fmaf(a, a, q[j]); q[j] = fmaf(b, b, q[j]); q[j] = fmaf(c, c, q[j]); q[j] = fmaf(d, d, q[j]);
      }
    }
  }
#pragma unroll
  for (int o = LANES / 2; o > 0; o >>= 1)
#pragma unroll
    for (int j = 0; j < NR; ++j) q[j] += __shfl_xor_sync(0xffffffffu, q[j], o);
  // optional second copy in PATCH order for a k = s = sr convolution that follows (spatial-reduction conv of the attention,
  // mix_transformers.py:112-117; ConvNeXt downsample 2x2/2, convnext.py:93-99): token (b, y, x) of an RH x RW map goes to row
  // (b, y / sr, x / sr), columns ((y % sr) * sr + x % sr) * C + c -- the im2col matrix of that convolution, written by the
  // producer instead of a separate gather kernel
#pragma unroll
  for (int j = 0; j < NR; ++j) {
    const unsigned row = row0 + j;
    if (row >= rows) break;
    const float mean = s[j];
    const float rstd = 1.0f / sqrtf(fmaf(q[j], inv_c, eps));
    unsigned pb = 0;
    if (phi) {
      const unsigned uRH = (unsigned)RH, uRW = (unsigned)RW, usr = (unsigned)sr;
      const unsigned x = row % uRW, t = row / uRW, y = t % uRH, b = t / uRH;
      const unsigned ORH = uRH / usr, ORW = uRW / usr;
      pb = (((b * ORH + y / usr) * ORW + x / usr) * (usr * usr) + (y % usr) * usr + x % usr) * Q;
    }
    const unsigned ob = row * Q;
#pragma unroll
    for (int i = 0; i < MAXQ; ++i) {
      const unsigned qd = lane + LANES * i;
      if (qd < Q) {
        const float4 w = __ldg(reinterpret_cast<const float4*>(gw) + qd), b = __ldg(reinterpret_cast<const float4*>(gb) + qd);
        const float4 y = make_float4((v[j][i].x - mean) * rstd * w.x + b.x, (v[j][i].y - mean) * rstd * w.y + b.y,
                                     (v[j][i].z - mean) * rstd * w.z + b.z, (v[j][i].w - mean) * rstd * w.w + b.w);
        if (out) reinterpret_cast<float4*>(out)[ob + qd] = y;
        if (shi || phi) {
          uint2 h, l;
          split_bf16x2(y.x, y.y, h.x, l.x);
          split_bf16x2(y.z, y.w, h.y, l.y);
          if (shi) { reinterpret_cast<uint2*>(shi)[ob + qd] = h; reinterpret_cast<uint2*>(slo)[ob + qd] = l; }
          if (phi) { reinterpret_cast<uint2*>(phi)[pb + qd] = h; reinterpret_cast<uint2*>(plo)[pb + qd] = l; }
        }
      }
    }
  }
}

#ifndef PF_LN_NR3
#define PF_LN_NR3 1            // rows in flight per lane group for C > 128 (C <= 128: 4 rows)
#endif
inline cudaError_t layernorm_launch(const float* in, float* out, long long rows, int C, const float* w, const float* b, float eps,
                                    cudaStream_t st, SplitT sp = SplitT(), SplitT patch = SplitT(), int RH = 0, int RW = 0, int sr = 0) {
  if (C % 4 || C > 768 || rows * (C / 4) >= (1LL << 32)) return cudaErrorInvalidValue;
  if (patch.hi && (RH < 1 || RW < 1 || sr < 1 || RH % sr || RW % sr || rows % ((long long)RH * RW))) return cudaErrorInvalidValue;
  // rows per block = 8 warps x (32 / LANES) lane groups x NR rows in flight per group
  if (C <= 64) return launch_pdl(layernorm_kernel<1, 16, 4>, dim3((unsigned)cdivl(rows, 64)), dim3(256), 0, st, in, out, rows, C, w, b, eps, sp.hi, sp.lo, patch.hi, patch.lo, RH, RW, sr);
  if (C <= 128) return launch_pdl(layernorm_kernel<1, 32, 4>, dim3((unsigned)cdivl(rows, 32)), dim3(256), 0, st, in, out, rows, C, w, b, eps, sp.hi, sp.lo, patch.hi, patch.lo, RH, RW, sr);
  if (C <= 384) return launch_pdl(layernorm_kernel<3, 32, PF_LN_NR3>, dim3((unsigned)cdivl(rows, 8 * PF_LN_NR3)), dim3(256), 0, st, in, out, rows, C, w, b, eps, sp.hi, sp.lo, patch.hi, patch.lo, RH, RW, sr);
  return launch_pdl(layernorm_kernel<6, 32, PF_LN_NR3>, dim3((unsigned)cdivl(rows, 8 * PF_LN_NR3)), dim3(256), 0, st, in, out, rows, C, w, b, eps, sp.hi, sp.lo, patch.hi, patch.lo, RH, RW, sr);
}

// =====================================================================================================
// Depthwise 3x3 conv (pad 1) + bias + GELU(erf) on NHWC -- Mix-FFN middle, mix_transformers.py:51-52,502-508.
// w: [9][C], thread = 4 channels of one pixel.
#ifndef PF_DW3_PX
#define PF_DW3_PX 4            // output pixels per thread along x (x 2 rows x 4 channels)
#endif
#ifndef PF_DW3_HOIST
#define PF_DW3_HOIST 1          // 0: weights loaded row by row
#endif
#ifndef PF_DW3_MINBLOCKS
#define PF_DW3_MINBLOCKS 2     // (3 blocks per SM = 80 registers, with spills)
#endif
// Index arithmetic is 32-bit in units of float4 (4 channels): o00 = pixel (y0, x0) of the thread's tile, neighbours at +- W*C/4 and
// +- C/4 (modular unsigned arithmetic: an index is only dereferenced when its row / column predicate holds).  The 64-bit
// per-load address chains of a first version were a third of its executed instructions.
__global__ void __launch_bounds__(256, PF_DW3_MINBLOCKS) dwconv3x3_gelu_kernel(const float* __restrict__ in, float* __restrict__ out, int B, int H, int W, int C,
                                                             const float* __restrict__ w, const float* __restrict__ bias,
                                                             __nv_bfloat16* __restrict__ shi = nullptr, __nv_bfloat16* __restrict__ slo = nullptr) {
  pdl_wait();
  pdl_launch();
  // thread = 4 channels x (2 rows x PX consecutive pixels): 4 (PX + 2) activation + 9 weight loads (float4) for 2 PX outputs
  constexpr int PX = PF_DW3_PX;
  const unsigned C4 = (unsigned)C >> 2, XG = ((unsigned)W + PX - 1) / PX, YG = ((unsigned)H + 1) >> 1;
  const unsigned total = (unsigned)B * YG * XG * C4;      // B H W C / 4 < 2^31, checked by Fwd::dw3_gelu (pf_b200.cu): 32-bit index math
  const unsigned rs = (unsigned)W * C4;                   // row stride in float4
  const float4* __restrict__ in4 = reinterpret_cast<const float4*>(in);
  const float4* __restrict__ w4 = reinterpret_cast<const float4*>(w);
  for (unsigned i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    const unsigned c4 = i % C4;
    unsigned r = i / C4;
    const unsigned xg = r % XG; r /= XG;
    const int y0 = (int)(r % YG) * 2; const unsigned b = r / YG;
    const int x0 = (int)xg * PX;
    const unsigned o00 = ((b * (unsigned)H + (unsigned)y0) * (unsigned)W + (unsigned)x0) * C4 + c4;
    bool cv[PX + 2];
#pragma unroll
    for (int j = 0; j < PX + 2; ++j) cv[j] = (unsigned)(x0 - 1 + j) < (unsigned)W;
    const float4 bv = __ldg(reinterpret_cast<const float4*>(bias) + c4);
    float4 acc[2][PX];
#pragma unroll
    for (int p = 0; p < PX; ++p) acc[0][p] = acc[1][p] = bv;
    float4 k[9];
#pragma unroll
    for (int t = 0; t < 9; ++t) k[t] = __ldg(w4 + ((unsigned)t * C4 + c4));
#if PF_DW3_HOIST
    // all 4 (PX + 2) loads are issued before the first FMA (rows outside the image contribute zeros): one exposed memory latency
    // per tile instead of one per input row
    float4 a[4][PX + 2];
#pragma unroll
    for (int ry = 0; ry < 4; ++ry) {
      const bool rv = (unsigned)(y0 + ry - 1) < (unsigned)H;
      const unsigned rb = o00 + (unsigned)(ry - 1) * rs - C4;     // (iy, x0 - 1)
#pragma unroll
      for (int j = 0; j < PX + 2; ++j) {
        a[ry][j] = make_float4(0.f, 0.f, 0.f, 0.f);
        if (rv && cv[j]) a[ry][j] = __ldg(in4 + (rb + (unsigned)j * C4));
      }
    }
#pragma unroll
    for (int ry = 0; ry < 4; ++ry) {
#pragma unroll
      for (int oy = 0; oy < 2; ++oy) {
        const int ky = ry - oy;
        if (ky < 0 || ky > 2) continue;
#pragma unroll
        for (int kx = 0; kx < 3; ++kx) {
          const float4 kk = k[ky * 3 + kx];
#pragma unroll
          for (int p = 0; p < PX; ++p) {
            acc[oy][p].x = fmaf(a[ry][p + kx].x, kk.x, acc[oy][p].x); acc[oy][p].y = fmaf(a[ry][p + kx].y, kk.y, acc[oy][p].y);
            acc[oy][p].z = fmaf(a[ry][p + kx].z, kk.z, acc[oy][p].z); acc[oy][p].w = fmaf(a[ry][p + kx].w, kk.w, acc[oy][p].w);
          }
        }
      }
    }
#else
#pragma unroll
    for (int ry = 0; ry < 4; ++ry) {          // input rows y0-1 .. y0+2
      const int iy = y0 + ry - 1;
      if ((unsigned)iy >= (unsigned)H) continue;
      const unsigned rb = o00 + (unsigned)(ry - 1) * rs - C4;     // (iy, x0 - 1)
      float4 a[PX + 2];
#pragma unroll
      for (int j = 0; j < PX + 2; ++j) {
        a[j] = make_float4(0.f, 0.f, 0.f, 0.f);
        if (cv[j]) a[j] = __ldg(in4 + (rb + (unsigned)j * C4));
      }
#pragma unroll
      for (int oy = 0; oy < 2; ++oy) {        // this input row is filter row ky = ry - oy of output row y0 + oy
        const int ky = ry - oy;
        if (ky < 0 || ky > 2) continue;
#pragma unroll
        for (int kx = 0; kx < 3; ++kx) {
          const float4 kk = k[ky * 3 + kx];
#pragma unroll
          for (int p = 0; p < PX; ++p) {
            acc[oy][p].x = fmaf(a[p + kx].x, kk.x, acc[oy][p].x); acc[oy][p].y = fmaf(a[p + kx].y, kk.y, acc[oy][p].y);
            acc[oy][p].z = fmaf(a[p + kx].z, kk.z, acc[oy][p].z); acc[oy][p].w = fmaf(a[p + kx].w, kk.w, acc[oy][p].w);
          }
        }
      }
    }
#endif
#pragma unroll
    for (int oy = 0; oy < 2; ++oy) {
      if (y0 + oy >= H) break;
#pragma unroll
      for (int p = 0; p < PX; ++p) {
        if (!cv[p + 1]) break;                 // x0 + p < W
        const float4 o = make_float4(gelu_erf(acc[oy][p].x), gelu_erf(acc[oy][p].y), gelu_erf(acc[oy][p].z), gelu_erf(acc[oy][p].w));
        const unsigned oi = o00 + (unsigned)oy * rs + (unsigned)p * C4;
        if (out) reinterpret_cast<float4*>(out)[oi] = o;
        if (shi) {
          uint2 h, l;
          split_bf16x2(o.x, o.y, h.x, l.x);
          split_bf16x2(o.z, o.w, h.y, l.y);
          reinterpret_cast<uint2*>(shi)[oi] = h;
          reinterpret_cast<uint2*>(slo)[oi] = l;
        }
      }
    }
  }
}

// Depthwise 7x7 conv (pad 3) + bias on NHWC -- ConvNeXt block head, convnext.py:28-30,48.  w: [49][C].
// thread = 4 channels x (2 rows x 8 consecutive pixels): per input row 14 activation loads serve both output rows; 98 weight +
// 112 activation loads (16 B) for 3136 FMAs, which balances the L1 path against the FMA pipe (one row x 4 pixels was L1-bound 2.4x)
#ifndef PF_DW7_PX
#define PF_DW7_PX 4            // output pixels per thread along x (x 2 rows x 4 channels); A/B: 4 px at 2 blocks / SM 0.78 ms, 8 px at 1 block 0.84 ms
#endif
#ifndef PF_DW7_MINBLOCKS
#define PF_DW7_MINBLOCKS 2
#endif
__global__ void __launch_bounds__(256, PF_DW7_MINBLOCKS) dwconv7x7_kernel(const float* __restrict__ in, float* __restrict__ out, int B, int H, int W, int C,
                                                        const float* __restrict__ w, const float* __restrict__ bias) {
  pdl_wait();
  pdl_launch();
  constexpr int PX = PF_DW7_PX;
  const unsigned C4 = (unsigned)C >> 2, XG = ((unsigned)W + PX - 1) / PX, YG = ((unsigned)H + 1) >> 1;
  const unsigned total = (unsigned)B * YG * XG * C4;
  const unsigned rs = (unsigned)W * C4;                   // row stride in float4 (32-bit index arithmetic as dwconv3x3_gelu_kernel, bound checked by pn_dw_launch)
  const float4* __restrict__ in4 = reinterpret_cast<const float4*>(in);
  const float4* __restrict__ w4 = reinterpret_cast<const float4*>(w);
  for (unsigned i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    const unsigned c4 = i % C4;
    unsigned r = i / C4;
    const unsigned xg = r % XG; r /= XG;
    const int y0 = (int)(r % YG) * 2; const unsigned b = r / YG;
    const int x0 = (int)xg * PX;
    const unsigned o00 = ((b * (unsigned)H + (unsigned)y0) * (unsigned)W + (unsigned)x0) * C4 + c4;
    bool cv[PX + 6];
#pragma unroll
    for (int j = 0; j < PX + 6; ++j) cv[j] = (unsigned)(x0 - 3 + j) < (unsigned)W;
    const float4 bv = __ldg(reinterpret_cast<const float4*>(bias) + c4);
    float4 acc[2][PX];
#pragma unroll
    for (int oy = 0; oy < 2; ++oy)
#pragma unroll
      for (int p = 0; p < PX; ++p) acc[oy][p] = bv;
#pragma unroll
    for (int ry = 0; ry < 8; ++ry) {          // input rows y0-3 .. y0+4
      const int iy = y0 + ry - 3;
      if ((unsigned)iy >= (unsigned)H) continue;
      const unsigned rb = o00 + (unsigned)(ry - 3) * rs - 3u * C4;     // (iy, x0 - 3)
      float4 a[PX + 6];
#pragma unroll
      for (int j = 0; j < PX + 6; ++j) {
        a[j] = make_float4(0.f, 0.f, 0.f, 0.f);
        if (cv[j]) a[j] = __ldg(in4 + (rb + (unsigned)j * C4));
      }
#pragma unroll
      for (int oy = 0; oy < 2; ++oy) {        // this input row is filter row ky = ry - oy of output row y0 + oy
        const int ky = ry - oy;
        if (ky < 0 || ky > 6) continue;
#pragma unroll
        for (int kx = 0; kx < 7; ++kx) {
          const float4 k = __ldg(w4 + ((unsigned)(ky * 7 + kx) * C4 + c4));
#pragma unroll
          for (int p = 0; p < PX; ++p) {
            acc[oy][p].x = fmaf(a[p + kx].x, k.x, acc[oy][p].x); acc[oy][p].y = fmaf(a[p + kx].y, k.y, acc[oy][p].y);
            acc[oy][p].z = fmaf(a[p + kx].z, k.z, acc[oy][p].z); acc[oy][p].w = fmaf(a[p + kx].w, k.w, acc[oy][p].w);
          }
        }
      }
    }
#pragma unroll
    for (int oy = 0; oy < 2; ++oy) {
      if (y0 + oy >= H) break;
#pragma unroll
      for (int p = 0; p < PX; ++p) {
        if (!cv[p + 3]) break;                 // x0 + p < W
        reinterpret_cast<float4*>(out)[o00 + (unsigned)oy * rs + (unsigned)p * C4] = acc[oy][p];
      }
    }
  }
}

// =====================================================================================================
// Bilinear x2 upsample, align_corners=False (decode_head.py:284-286, gravity_head.py:172): taps {0.25, 0.75},
// edges clamped.  ATen: src = 0.5*(dst+0.5)-0.5 clamped at 0, i1 = min(i0+1, in-1).  NHWC, float4 per thread.
// `in` channel pitch/offset (ldi, icoff) select one head's half of a 512-channel tensor.
// thread = 4 channels x (2 output rows x 4 output columns) = the outputs of two neighbouring low-res pixels of one row: 12
// float4 loads (3 rows x 4 columns, clamped) for 32 results, separable (horizontal, then vertical) -- a third of the loads and
// half of the instructions of the one-output-pixel-per-thread version.  out[2i] = 0.25 in[i-1] + 0.75 in[i], out[2i+1] =
// 0.75 in[i] + 0.25 in[i+1]; at the clamped edges both taps are the same pixel and fmaf(0.75, a, 0.25 a) returns a exactly.
// Index arithmetic is 32-bit in float4 units (B H W ldi / 4 and 4 B H W ldo / 4 < 2^31, checked by Fwd::up2x in pf_b200.cu).
inline long long upsample2x_threads(int B, int H, int W, int C) { return (long long)B * H * ((W + 1) / 2) * (C / 4); }
__global__ void __launch_bounds__(256) upsample2x_kernel(const float* __restrict__ in, int ldi, int icoff, float* __restrict__ out, int ldo, int ocoff,
                                                         int B, int H, int W, int C, __nv_bfloat16* __restrict__ shi = nullptr, __nv_bfloat16* __restrict__ slo = nullptr) {
  pdl_wait();
  pdl_launch();
  const unsigned C4 = (unsigned)C >> 2, JG = ((unsigned)W + 1) >> 1, li4 = (unsigned)ldi >> 2, lo4 = (unsigned)ldo >> 2;
  const unsigned total = (unsigned)B * H * JG * C4;
  const unsigned OW = 2u * W;
  const float4* __restrict__ in4 = reinterpret_cast<const float4*>(in + icoff);
  const unsigned oc4 = (unsigned)ocoff >> 2;
  for (unsigned i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    const unsigned c4 = i % C4;
    unsigned r = i / C4;
    const unsigned jg = r % JG; r /= JG;
    const int iy = (int)(r % (unsigned)H); const unsigned b = r / (unsigned)H;
    const int j0 = (int)jg * 2;
    const bool two = j0 + 1 < W;                                       // second low-res column of the pair exists (odd W: not in the last group)
    const int cx[4] = {j0 > 0 ? j0 - 1 : 0, j0, j0 + 1 < W ? j0 + 1 : W - 1, j0 + 2 < W ? j0 + 2 : W - 1};
    const int cy[3] = {iy > 0 ? iy - 1 : 0, iy, iy + 1 < H ? iy + 1 : H - 1};
    float4 t[3][4];
#pragma unroll
    for (int ry = 0; ry < 3; ++ry) {
      const unsigned rb = ((b * (unsigned)H + (unsigned)cy[ry]) * (unsigned)W) * li4 + c4;
      float4 v[4];
#pragma unroll
      for (int k = 0; k < 4; ++k) v[k] = __ldg(in4 + (rb + (unsigned)cx[k] * li4));
#define PF_UP_LERP(d, lo_, hi_)                                                                                 \
  d.x = fmaf(0.75f, hi_.x, 0.25f * lo_.x); d.y = fmaf(0.75f, hi_.y, 0.25f * lo_.y);                             \
  d.z = fmaf(0.75f, hi_.z, 0.25f * lo_.z); d.w = fmaf(0.75f, hi_.w, 0.25f * lo_.w);
      PF_UP_LERP(t[ry][0], v[0], v[1])        // output column 2 j0     : 0.25 in[j0-1] + 0.75 in[j0]
      PF_UP_LERP(t[ry][1], v[2], v[1])        //               2 j0 + 1 : 0.75 in[j0]   + 0.25 in[j0+1]
      PF_UP_LERP(t[ry][2], v[1], v[2])        //               2 j0 + 2 : 0.25 in[j0]   + 0.75 in[j0+1]
      PF_UP_LERP(t[ry][3], v[3], v[2])        //               2 j0 + 3 : 0.75 in[j0+1] + 0.25 in[j0+2]
    }
    const unsigned ob = ((b * 2u * (unsigned)H + 2u * (unsigned)iy) * OW + 4u * jg) * lo4 + oc4 + c4;     // output pixel (2 iy, 4 jg)
#pragma unroll
    for (int oy = 0; oy < 2; ++oy) {
#pragma unroll
      for (int p = 0; p < 4; ++p) {
        if (p >= 2 && !two) break;
        float4 o;
        if (oy == 0) { PF_UP_LERP(o, t[0][p], t[1][p]) } else { PF_UP_LERP(o, t[2][p], t[1][p]) }
        const unsigned oi = ob + ((unsigned)oy * OW + (unsigned)p) * lo4;
        if (out) reinterpret_cast<float4*>(out)[oi] = o;
        if (shi) {
          uint2 h, l;
          split_bf16x2(o.x, o.y, h.x, l.x);
          split_bf16x2(o.z, o.w, h.y, l.y);
          reinterpret_cast<uint2*>(shi)[oi] = h;
          reinterpret_cast<uint2*>(slo)[oi] = l;
        }
      }
    }
#undef PF_UP_LERP
  }
}

// =====================================================================================================
// Patch gather on split planes: dst[m][(ky,kx,c)] = src[b, oy*stride - pad + ky, ox*stride - pad + kx, c] (zero outside),
// for the few strided convolutions (overlap patch embed 3x3/2, spatial-reduction k = s = R, ConvNeXt downsample 2x2/2)
// so that they run on the same TMA GEMM kernel.  16 B (8 channels) per thread per plane.
__global__ void __launch_bounds__(256) im2col_split_kernel(const __nv_bfloat16* __restrict__ shi, const __nv_bfloat16* __restrict__ slo, int lds,
                                                           __nv_bfloat16* __restrict__ dhi, __nv_bfloat16* __restrict__ dlo,
                                                           int B, int H, int W, int C, int OH, int OW, int KH, int stride, int pad) {
  pdl_wait();
  pdl_launch();
  const int C8 = C >> 3;
  const long long total = (long long)B * OH * OW * KH * KH * C8;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int c8 = (int)(i % C8);
    long long r = i / C8;
    const int kx = (int)(r % KH); r /= KH;
    const int ky = (int)(r % KH); r /= KH;
    const int ox = (int)(r % OW); r /= OW;
    const int oy = (int)(r % OH); const int b = (int)(r / OH);
    const int iy = oy * stride - pad + ky, ix = ox * stride - pad + kx;
    uint4 h = make_uint4(0, 0, 0, 0), l = h;
    if ((unsigned)iy < (unsigned)H && (unsigned)ix < (unsigned)W) {
      const long long si = ((long long)(b * H + iy) * W + ix) * lds + c8 * 8;
      h = __ldg(reinterpret_cast<const uint4*>(shi + si));
      l = __ldg(reinterpret_cast<const uint4*>(slo + si));
    }
    reinterpret_cast<uint4*>(dhi)[i] = h;
    reinterpret_cast<uint4*>(dlo)[i] = l;
  }
}

// Patch gather for the 7x7 stems (patch_embed1: stride 4, ll_enc: stride 2; pad 3) straight from the normalised input
// x0 [B,IH,IW,4] fp32 (b,g,r,0) (the net size): dst[m][(ky*7+kx)*3 + c] split into bf16 hi/lo, K padded 147 -> 160 with zeros, so that the
// stems run on the TMA GEMM engine too.  One thread = one output pixel x 8 consecutive K columns (16 B per plane).
// (A one-pixel-per-thread variant -- 49 float4 loads, 40 16-byte stores into the thread's own 320-byte row -- executed a third of
// the instructions but every store instruction of a warp touched 32 different rows.)
inline long long stem_gather_threads(int B, int OH, int OW) { return (long long)B * OH * OW * 20; }
__global__ void __launch_bounds__(256) stem_gather_kernel(const float* __restrict__ x0, __nv_bfloat16* __restrict__ dhi, __nv_bfloat16* __restrict__ dlo,
                                                          int B, int OH, int OW, int stride, int IH, int IW) {
  pdl_wait();
  pdl_launch();
  constexpr int KP = 160, KQ = KP / 8;
  const unsigned total = (unsigned)B * OH * OW * KQ;
  for (unsigned i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    const int kq = (int)(i % KQ);
    unsigned m = i / KQ;
    const int ox = (int)(m % (unsigned)OW); unsigned t = m / (unsigned)OW;
    const int oy = (int)(t % (unsigned)OH); const unsigned b = t / (unsigned)OH;
    const int iy0 = oy * stride - 3, ix0 = ox * stride - 3;
    const unsigned pb = ((b * (unsigned)IH + (unsigned)iy0) * (unsigned)IW + (unsigned)ix0) * 4u;     // float index of pixel (iy0, ix0), dereferenced where valid
    float v[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      const int k = kq * 8 + e;
      float val = 0.f;
      if (k < 147) {
        const int tap = k / 3, c = k - tap * 3;
        const int ky = tap / 7, kx = tap - ky * 7;
        if ((unsigned)(iy0 + ky) < (unsigned)IH && (unsigned)(ix0 + kx) < (unsigned)IW) val = __ldg(x0 + (pb + (unsigned)((ky * IW + kx) * 4 + c)));
      }
      v[e] = val;
    }
    uint4 h, l;
    split_bf16x2(v[0], v[1], h.x, l.x); split_bf16x2(v[2], v[3], h.y, l.y);
    split_bf16x2(v[4], v[5], h.z, l.z); split_bf16x2(v[6], v[7], h.w, l.w);
    reinterpret_cast<uint4*>(dhi)[i] = h;
    reinterpret_cast<uint4*>(dlo)[i] = l;
  }
}

// fp32 = hi + lo (debug taps / tests)
__global__ void __launch_bounds__(256) merge_split_kernel(const __nv_bfloat16* __restrict__ hi, const __nv_bfloat16* __restrict__ lo, float* __restrict__ out, long long n) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = __bfloat162float(hi[i]) + __bfloat162float(lo[i]);
}
// fp32 -> split planes (tests)
__global__ void __launch_bounds__(256) split_kernel(const float* __restrict__ in, __nv_bfloat16* __restrict__ hi, __nv_bfloat16* __restrict__ lo, long long n, int relu) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) store_split1(hi, lo, i, relu ? fmaxf(in[i], 0.f) : in[i]);
}

// =====================================================================================================
// Prediction tail: 1x1 conv 32 -> NC (gravity_head.py:175 / latitude_head.py:174) fused with the head's
// inference epilogue: mode 1 = F.normalize over the 2 channels (gravity_head.py:192-193, eps 1e-12),
// mode 2 = clamp to [-1, 1] (latitude_head.py:191-192), mode 0 = raw logits (classification variant).
// in: [npix, ldi] NHWC (32 channels at offset icoff); out: NCHW [B, NC, HW].  One thread per pixel; weights [NC][32] + bias in smem.
__global__ void __launch_bounds__(128) pred_tail_kernel(const float* __restrict__ in, int ldi, int icoff, const float* __restrict__ w,
                                                        const float* __restrict__ bias, float* __restrict__ out, int B, int HW, int NC, int mode) {
  extern __shared__ float s_w[];  // [NC][32] then [NC]
  for (int i = threadIdx.x; i < NC * 33; i += blockDim.x) s_w[i] = i < NC * 32 ? __ldg(w + i) : __ldg(bias + i - NC * 32);
  __syncthreads();
  const long long pix = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (pix >= (long long)B * HW) return;
  float f[32];
#pragma unroll
  for (int d = 0; d < 32; d += 4) {
    const float4 t = __ldg(reinterpret_cast<const float4*>(in + pix * ldi + icoff + d));
    f[d] = t.x; f[d + 1] = t.y; f[d + 2] = t.z; f[d + 3] = t.w;
  }
  const int b = (int)(pix / HW), r = (int)(pix % HW);
  float* o = out + (long long)b * NC * HW + r;
  if (mode == 1) {
    float v0 = s_w[64], v1 = s_w[65];
#pragma unroll
    for (int d = 0; d < 32; ++d) { v0 = fmaf(f[d], s_w[d], v0); v1 = fmaf(f[d], s_w[32 + d], v1); }
    const float nrm = fmaxf(sqrtf(v0 * v0 + v1 * v1), 1e-12f);
    o[0] = v0 / nrm; o[HW] = v1 / nrm;
  } else {
    for (int c = 0; c < NC; ++c) {
      float v = s_w[NC * 32 + c];
#pragma unroll
      for (int d = 0; d < 32; ++d) v = fmaf(f[d], s_w[c * 32 + d], v);
      if (mode == 2) v = fminf(fmaxf(v, -1.f), 1.f);
      o[(long long)c * HW] = v;
    }
  }
}

// =====================================================================================================
// Border ring of conv_fuse_conv1 (gravity_head.py:171-175 / latitude_head.py:170-174).  The engine evaluates
// conv3x3(bilinear_x2(c0)) as four phase convolutions on the 160x160 grid (weights.py:_compose_up2_conv3); that identity holds
// wherever neither the upsample's index clamp nor the convolution's zero padding is involved, i.e. everywhere except the two
// outermost rows / columns of the 320x320 output.  This kernel recomputes those 2544 pixels per image directly in fp32:
// u = bilinear_x2(c0) sampled on the fly (align_corners=False: src = max(0, (i + 0.5) / 2 - 0.5), neighbour index clamped),
// zero outside the image, 3x3 taps, + bias, ReLU; then (regression heads) the same fused prediction tail as the GEMM epilogue.
// c0: split planes [B, H, W, 128] (gravity channels 0-63, latitude 64-127); wf: [2][9][64][32] fp32; out NHWC [B, 2H, 2W, 64].
// Block = 64 ring pixels x both heads; warp w -> head w / 4, pixels (w % 4) * 16 .. + 16; lane = output channel.  Per filter tap the
// block stages the tap's weights and the upsampled inputs of its pixels (16 lanes read the 128 channels of one source pixel:
// coalesced 256-byte rows -- with one pixel per lane every 16-byte load pulled its own 32-byte sector and the kernel was bound by
// L2 sector traffic), then each lane accumulates its channel for 16 pixels from broadcast 16-byte reads of the inputs.
constexpr int kRingPx = 64;
__host__ __device__ inline int conv1_ring_count(int H2, int W2) { return 4 * W2 + 4 * (H2 - 4); }
__global__ void __launch_bounds__(256) conv1_ring_kernel(const __nv_bfloat16* __restrict__ chi, const __nv_bfloat16* __restrict__ clo, int H, int W,
                                                         const float* __restrict__ wf, const float* __restrict__ bias, float* __restrict__ out,
                                                         const float* __restrict__ pg_w, const float* __restrict__ pg_b, float* __restrict__ pg_out,
                                                         const float* __restrict__ pl_w, const float* __restrict__ pl_b, float* __restrict__ pl_out) {
  extern __shared__ __align__(16) float s_ring[];
  float* sU = s_ring;                        // [64 px][128 ch]; after the last tap: conv1 outputs [64 px][65] for the prediction tail
  float* sW = s_ring + 128 * kRingPx;        // [2][64 ci][32 o]
  __shared__ int s_y[kRingPx], s_x[kRingPx];
  const int H2 = 2 * H, W2 = 2 * W, ring = conv1_ring_count(H2, W2);
  const int b = blockIdx.y, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  if (tid < kRingPx) {
    const int r = blockIdx.x * kRingPx + tid;
    int y = -1, x = -1;
    if (r < 4 * W2) { const int k = r / W2; y = k < 2 ? k : H2 - 4 + k; x = r - k * W2; }
    else if (r < ring) { const int q = r - 4 * W2, k = q & 3; y = 2 + (q >> 2); x = k < 2 ? k : W2 - 4 + k; }
    s_y[tid] = y; s_x[tid] = x;
  }
  const int g = warp >> 2, pq = warp & 3;
  float acc[16];
#pragma unroll
  for (int j = 0; j < 16; ++j) acc[j] = 0.f;
  for (int tap = 0; tap < 9; ++tap) {
    __syncthreads();
    // weights of this tap: [2][64][32] <- wf[g][tap][ci][o]
    for (int i = tid; i < 2 * 64 * 8; i += 256) {
      const int gg = i / 512, rem = i % 512;
      reinterpret_cast<float4*>(sW)[i] = __ldg(reinterpret_cast<const float4*>(wf + ((long long)(gg * 9 + tap) * 64) * 32) + rem);
    }
    // upsampled input of this tap: 64 px x 16 channel octets (the 16 octets of a pixel on consecutive lanes)
    const int ky = tap / 3 - 1, kx = tap % 3 - 1;
    for (int i = tid; i < kRingPx * 16; i += 256) {
      const int c8 = i & 15, px = i >> 4;
      const int y = s_y[px] + ky, x = s_x[px] + kx;
      float u[8];
#pragma unroll
      for (int e = 0; e < 8; ++e) u[e] = 0.f;
      if (s_y[px] >= 0 && y >= 0 && y < H2 && x >= 0 && x < W2) {
        const float sy = fmaxf((y + 0.5f) * 0.5f - 0.5f, 0.f), sx = fmaxf((x + 0.5f) * 0.5f - 0.5f, 0.f);
        const int y0 = (int)sy, x0 = (int)sx;
        const int y1 = min(y0 + 1, H - 1), x1 = min(x0 + 1, W - 1);
        const float ly = sy - y0, lx = sx - x0;
        const float cw[4] = {(1.f - ly) * (1.f - lx), (1.f - ly) * lx, ly * (1.f - lx), ly * lx};
        const int yy[4] = {y0, y0, y1, y1}, xx[4] = {x0, x1, x0, x1};
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const unsigned o = ((unsigned)(b * H + yy[k]) * (unsigned)W + (unsigned)xx[k]) * 16u + (unsigned)c8;      // uint4 units
          const uint4 h = __ldg(reinterpret_cast<const uint4*>(chi) + o), l = __ldg(reinterpret_cast<const uint4*>(clo) + o);
          const uint32_t hw[4] = {h.x, h.y, h.z, h.w}, lw[4] = {l.x, l.y, l.z, l.w};
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            const float v0 = __uint_as_float(hw[e] << 16) + __uint_as_float(lw[e] << 16);
            const float v1 = __uint_as_float(hw[e] & 0xffff0000u) + __uint_as_float(lw[e] & 0xffff0000u);
            u[2 * e] = fmaf(cw[k], v0, u[2 * e]); u[2 * e + 1] = fmaf(cw[k], v1, u[2 * e + 1]);
          }
        }
      }
      float4* d = reinterpret_cast<float4*>(sU + px * 128 + c8 * 8);
      d[0] = make_float4(u[0], u[1], u[2], u[3]);
      d[1] = make_float4(u[4], u[5], u[6], u[7]);
    }
    __syncthreads();
    const float* su = sU + (pq * 16) * 128 + g * 64;
    const float* sw = sW + g * 64 * 32 + lane;
#pragma unroll 2
    for (int c4 = 0; c4 < 16; ++c4) {
      const float w0 = sw[(4 * c4) * 32], w1 = sw[(4 * c4 + 1) * 32], w2 = sw[(4 * c4 + 2) * 32], w3 = sw[(4 * c4 + 3) * 32];
#pragma unroll
      for (int j = 0; j < 16; ++j) {
        const float4 uv = *reinterpret_cast<const float4*>(su + j * 128 + 4 * c4);      // same address on every lane: broadcast
        acc[j] = fmaf(uv.x, w0, acc[j]); acc[j] = fmaf(uv.y, w1, acc[j]);
        acc[j] = fmaf(uv.z, w2, acc[j]); acc[j] = fmaf(uv.w, w3, acc[j]);
      }
    }
  }
  // bias + ReLU, conv1 output (when kept: 128 contiguous bytes per pixel and head), rectified features to shared memory for the tail
  __syncthreads();                                 // every warp is done reading sU
  float* sV = sU;                                  // [64 px][65]
  const float bv = __ldg(bias + g * 32 + lane);
#pragma unroll
  for (int j = 0; j < 16; ++j) {
    const int px = pq * 16 + j, y = s_y[px], x = s_x[px];
    const float v = fmaxf(acc[j] + bv, 0.f);
    if (y >= 0 && out) out[(((long long)b * H2 + y) * W2 + x) * 64 + g * 32 + lane] = v;
    sV[px * 65 + g * 32 + lane] = v;
  }
  if (!pg_w) return;
  __syncthreads();
  // fused prediction tail of the regression heads: 1x1 conv 32 -> 2 (gravity) / 1 (latitude), bias first then channels in order
  // (the fma chain of pred_tail_kernel), normalise / clamp
  if (tid < kRingPx && s_y[tid] >= 0) {
    const float* f = sV + tid * 65;
    float v0 = __ldg(pg_b), v1 = __ldg(pg_b + 1), vl = __ldg(pl_b);
#pragma unroll 8
    for (int c = 0; c < 32; ++c) {
      v0 = fmaf(f[c], __ldg(pg_w + c), v0);
      v1 = fmaf(f[c], __ldg(pg_w + 32 + c), v1);
      vl = fmaf(f[32 + c], __ldg(pl_w + c), vl);
    }
    const long long HW2 = (long long)H2 * W2, pix = (long long)s_y[tid] * W2 + s_x[tid];
    const float nrm = fmaxf(sqrtf(v0 * v0 + v1 * v1), 1e-12f);
    float* po = pg_out + (long long)b * 2 * HW2 + pix;
    po[0] = v0 / nrm; po[HW2] = v1 / nrm;
    pl_out[(long long)b * HW2 + pix] = fminf(fmaxf(vl, -1.f), 1.f);
  }
}
constexpr int kRingSmem = (128 * kRingPx + 2 * 64 * 32) * 4;

// Bin decode shared by the two classification kernels (utils/utils.py:114-130 and :148-162).
__device__ __forceinline__ void decode_bin_store(float* __restrict__ field, int b, int r, int HW, int NC, int bi, int is_gravity) {
  if (is_gravity) {
    // angle = (bin * (360/(NC-1)) - 180) / 180 * pi ; bin NC-1 -> (0, 0).  torch evaluates this in fp32 on an int64
    // tensor promoted to float: bin*5.0 - 180 exact in fp32, then /180*pi.
    float* o = field + (long long)b * 2 * HW + r;
    if (bi == NC - 1) { o[0] = 0.f; o[HW] = 0.f; }
    else {
      const float ang = ((float)bi * gravity_bin_deg(NC) - 180.0f) / 180.0f * 3.14159265358979323846f;
      o[0] = cosf(ang); o[HW] = sinf(ang);
    }
  } else {
    const float bin = latitude_bin_deg(NC);
    field[(long long)b * HW + r] = (-90.0f + (float)bi * bin) + bin * 0.5f;
  }
}

// Sub-bin decode (DESIGN.md section 1, "Sub-bin decode"): the argmax bin bi moved to p = bi + delta, delta in [-1/2, 1/2] the
// vertex of the parabola through l0 = l(bi) and the logits lm / lp of its two neighbours, then decode_bin_store's formulas at p.
// subbin_neighbours gives the neighbours' classes: the up head's direction bins 0 .. NC-2 form a circle (bin NC-1, no direction,
// is never a neighbour and is not refined); the latitude head's are bi -+ 1, clamped, and its two pole bins are not refined.
// Unrefined bins return bi itself, so every class read is in range.  delta = 0 gives decode_bin_store's value bit for bit.
__device__ __forceinline__ int2 subbin_neighbours(int NC, int bi, int is_gravity) {
  if (!is_gravity) return make_int2(max(bi - 1, 0), min(bi + 1, NC - 1));
  if (bi >= NC - 1) return make_int2(bi, bi);
  return make_int2(bi == 0 ? NC - 2 : bi - 1, bi == NC - 2 ? 0 : bi + 1);
}
__device__ __forceinline__ void subbin_decode_store(float* __restrict__ field, int b, int r, int HW, int NC, int bi, float l0, float lm, float lp,
                                                    int is_gravity) {
  // a, b >= 0 for a true maximum; non-finite logits (and a flat top, a + b = 0) give delta = 0.  The products and sums below are
  // rounded one at a time, as the fp32 oracle evaluates them (no fma contraction).
  const float da = l0 - lm, db = l0 - lp, s = da + db;
  float delta = (isfinite(da) && isfinite(db) && s > 0.0f) ? __fdiv_rn(da - db, 2.0f * s) : 0.0f;
  if (!is_gravity && (bi == 0 || bi == NC - 1)) delta = 0.0f;
  const float p = (float)bi + delta;
  if (is_gravity) {
    float* o = field + (long long)b * 2 * HW + r;
    if (bi == NC - 1) { o[0] = 0.f; o[HW] = 0.f; }
    else {
      const float ang = __fmul_rn(__fdiv_rn(__fsub_rn(__fmul_rn(p, gravity_bin_deg(NC)), 180.0f), 180.0f), 3.14159265358979323846f);
      o[0] = cosf(ang); o[HW] = sinf(ang);
    }
  } else {
    const float bin = latitude_bin_deg(NC);
    field[(long long)b * HW + r] = __fadd_rn(__fadd_rn(-90.0f, __fmul_rn(p, bin)), bin * 0.5f);
  }
}

// Classification variant: argmax over channels + bin decode (gravity_head.py:243-244 + utils.py:114-130;
// latitude_head.py:205-208 + utils.py:148-162).  logits NCHW [B, NC, HW] -> field [B, 2 or 1, HW].
// torch.argmax returns the FIRST maximal index; strict '>' reproduces that.
// kRefine: the sub-bin decode instead, reading the winner's two neighbour planes after the pass.
template <bool kRefine>
__global__ void __launch_bounds__(256) argmax_decode_kernel(const float* __restrict__ logits, float* __restrict__ field, int B, int HW, int NC, int is_gravity) {
  const long long pix = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (pix >= (long long)B * HW) return;
  const int b = (int)(pix / HW), r = (int)(pix % HW);
  const float* lp = logits + (long long)b * NC * HW + r;
  float best = lp[0];
  int bi = 0;
  for (int c = 1; c < NC; ++c) {
    const float v = __ldg(lp + (long long)c * HW);
    if (v > best) { best = v; bi = c; }
  }
  if constexpr (kRefine) {
    const int2 nb = subbin_neighbours(NC, bi, is_gravity);
    subbin_decode_store(field, b, r, HW, NC, bi, best, __ldg(lp + (long long)nb.x * HW), __ldg(lp + (long long)nb.y * HW), is_gravity);
  } else {
    decode_bin_store(field, b, r, HW, NC, bi, is_gravity);
  }
}

// Head confidence (DESIGN.md section 1): conf = max_c softmax(l)_c = 1 / sum_c exp(l_c - l_max) in fp32 over all NC classes.
// Online form: a running maximum m and the sum s of exp(l_c - m), rescaled by exp(m_old - m) when the maximum grows.
__device__ __forceinline__ void conf_update(float v, float& m, float& s) {
  if (v > m) { s = s * expf(m - v) + 1.0f; m = v; }
  else s += expf(v - m);
}
// merge another running pair (om, os) into (m, s), the own pair first
__device__ __forceinline__ void conf_merge(float& m, float& s, float om, float os) {
  const float mm = fmaxf(m, om);
  s = s * expf(m - mm) + os * expf(om - mm);
  m = mm;
}
// argmax_decode_kernel plus the confidence, in one pass over the logits (the logits are read once).  conf: [B, HW].
// kRefine: as argmax_decode_kernel's; conf does not depend on it.  The sum runs in pred_argmax_decode_kernel's order: four
// running pairs over the classes c = j, j + 4, ... (j = 0..3), merged as its quad shuffles merge them, ((0, 1), (2, 3)), so
// that both "decode_only" settings return the same confidence bit for bit.
template <bool kRefine>
__global__ void __launch_bounds__(256) argmax_conf_decode_kernel(const float* __restrict__ logits, float* __restrict__ field, float* __restrict__ conf,
                                                                 int B, int HW, int NC, int is_gravity) {
  const long long pix = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (pix >= (long long)B * HW) return;
  const int b = (int)(pix / HW), r = (int)(pix % HW);
  const float* lp = logits + (long long)b * NC * HW + r;
  float best = lp[0];
  int bi = 0;
  float cm[4] = {-INFINITY, -INFINITY, -INFINITY, -INFINITY}, cs[4] = {0.0f, 0.0f, 0.0f, 0.0f};
  for (int c0 = 0; c0 < NC; c0 += 4) {
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int c = c0 + j;
      if (c < NC) {
        const float v = __ldg(lp + (long long)c * HW);
        if (v > best) { best = v; bi = c; }
        conf_update(v, cm[j], cs[j]);
      }
    }
  }
  conf_merge(cm[0], cs[0], cm[1], cs[1]);
  conf_merge(cm[2], cs[2], cm[3], cs[3]);
  conf_merge(cm[0], cs[0], cm[2], cs[2]);
  conf[pix] = 1.0f / cs[0];
  if constexpr (kRefine) {
    const int2 nb = subbin_neighbours(NC, bi, is_gravity);
    subbin_decode_store(field, b, r, HW, NC, bi, best, __ldg(lp + (long long)nb.x * HW), __ldg(lp + (long long)nb.y * HW), is_gravity);
  } else {
    decode_bin_store(field, b, r, HW, NC, bi, is_gravity);
  }
}

// Classification heads WITHOUT the logits (SURVEY.md 8f-3, option "decode_only"): 1x1 prediction conv 32 -> NC
// (gravity_head.py:175 / latitude_head.py:174), argmax over the NC logits and bin decode in one pass; the 73 / 180-channel
// logit tensors (103.6 MB per image) are never written.  Four lanes (a quad) share one pixel: lane q evaluates the classes
// c = q, q + 4, ... with the SAME fma chain as pred_tail_kernel (bias first, then channels 0..31 in order: bit-identical logits,
// hence the same argmax as the default path), keeps its first maximum, and the quad's winner is found with two warp shuffles
// (larger logit wins, the lower class index on ties = torch.argmax's first maximal index).
// in: [npix, ldi] NHWC (32 channels at icoff); weights [NC][32] + bias staged in shared memory with rows padded to 36 floats
// (the four lanes of a quad read four different rows with 16-byte loads: no bank conflict).
// kConf: also the head confidence into conf [B, HW]: each lane keeps a running (max, sum) over its classes (conf_update), and the
// quad merges the pairs with the same two shuffles, s = s1 exp(m1 - m) + s2 exp(m2 - m).  kConf = false does not read conf.
// kRefine: the sub-bin decode.  The two neighbour logits are recomputed from f[] with the same fma chain (bit-identical to the
// logits the separate path reads): lanes q = 0, 2 evaluate the lower neighbour, q = 1, 3 the upper one, and lane 0, which stores,
// takes the upper one from lane 1.  The winner is lane 0's, broadcast to the quad (with NaN logits the lanes' winners can differ).
template <bool kConf, bool kRefine>
__global__ void __launch_bounds__(256) pred_argmax_decode_kernel(const float* __restrict__ in, int ldi, int icoff, const float* __restrict__ w,
                                                                 const float* __restrict__ bias, float* __restrict__ field, int B, int HW, int NC,
                                                                 int is_gravity, float* __restrict__ conf) {
  extern __shared__ __align__(16) float s_pw[];  // [NC][36] then [NC]
  for (int i = threadIdx.x; i < NC * 32; i += blockDim.x) s_pw[(i >> 5) * 36 + (i & 31)] = __ldg(w + i);
  float* s_b = s_pw + NC * 36;
  for (int i = threadIdx.x; i < NC; i += blockDim.x) s_b[i] = __ldg(bias + i);
  __syncthreads();
  const int q = threadIdx.x & 3;
  const long long npix = (long long)B * HW;
  const long long stride = (long long)gridDim.x * (blockDim.x >> 2);
  const long long pix_last = npix - 1;
  // (every lane of a warp runs the same number of iterations: the shuffles below need the full quad)
  const long long iters = (npix + stride - 1) / stride;
  long long pix = (long long)blockIdx.x * (blockDim.x >> 2) + (threadIdx.x >> 2);
  for (long long it = 0; it < iters; ++it, pix += stride) {
    const bool live = pix <= pix_last;
    const long long pc = live ? pix : pix_last;
    float f[32];
#pragma unroll
    for (int d = 0; d < 32; d += 4) {
      const float4 t = __ldg(reinterpret_cast<const float4*>(in + pc * ldi + icoff + d));
      f[d] = t.x; f[d + 1] = t.y; f[d + 2] = t.z; f[d + 3] = t.w;
    }
    float best = -INFINITY, cm = -INFINITY, cs = 0.0f;
    int bi = 0x7fffffff;
    for (int c = q; c < NC; c += 4) {
      const float4* wr = reinterpret_cast<const float4*>(s_pw + c * 36);
      float v = s_b[c];
#pragma unroll
      for (int d4 = 0; d4 < 8; ++d4) {
        const float4 ww = wr[d4];
        v = fmaf(f[4 * d4], ww.x, v); v = fmaf(f[4 * d4 + 1], ww.y, v); v = fmaf(f[4 * d4 + 2], ww.z, v); v = fmaf(f[4 * d4 + 3], ww.w, v);
      }
      if (v > best || bi == 0x7fffffff) { best = v; bi = c; }      // strict '>': first maximal index of this lane's classes
      if constexpr (kConf) conf_update(v, cm, cs);
    }
#pragma unroll
    for (int o = 1; o < 4; o <<= 1) {
      const float ov = __shfl_xor_sync(0xffffffffu, best, o);
      const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
      if (ov > best || (ov == best && oi < bi)) { best = ov; bi = oi; }
      if constexpr (kConf) {
        const float om = __shfl_xor_sync(0xffffffffu, cm, o), os = __shfl_xor_sync(0xffffffffu, cs, o);
        conf_merge(cm, cs, om, os);
      }
    }
    float lm = 0.0f, lp = 0.0f;
    if constexpr (kRefine) {
      const int2 nb = subbin_neighbours(NC, __shfl_sync(0xffffffffu, bi, 0, 4), is_gravity);
      const float4* wr = reinterpret_cast<const float4*>(s_pw + ((q & 1) ? nb.y : nb.x) * 36);
      float v = s_b[(q & 1) ? nb.y : nb.x];
#pragma unroll
      for (int d4 = 0; d4 < 8; ++d4) {
        const float4 ww = wr[d4];
        v = fmaf(f[4 * d4], ww.x, v); v = fmaf(f[4 * d4 + 1], ww.y, v); v = fmaf(f[4 * d4 + 2], ww.z, v); v = fmaf(f[4 * d4 + 3], ww.w, v);
      }
      lm = v;
      lp = __shfl_xor_sync(0xffffffffu, v, 1);
    }
    if (live && q == 0) {
      if constexpr (kRefine) subbin_decode_store(field, (int)(pix / HW), (int)(pix % HW), HW, NC, bi, best, lm, lp, is_gravity);
      else decode_bin_store(field, (int)(pix / HW), (int)(pix % HW), HW, NC, bi, is_gravity);
      if constexpr (kConf) conf[pix] = 1.0f / cs;
    }
  }
}

// =====================================================================================================
// Flip test-time augmentation (DESIGN.md section 1, "Flip test-time augmentation"; option "flip_tta").  The network ran on 2n
// slots: slot i is image i, slot n + i its mirror x[:, ::-1].  The merges below write n outputs at the working size H x W; b is
// read at column W - 1 - x for output column x (M(b)).  Every merge is a sum, then a scale, rounded one at a time (no fma
// contraction), and the up vector's x component enters as an exact negation: merge(mirror) is the mirror of merge bit for bit.

// Regression heads: g2 [2n, 2, HW] (normalised up vectors), l2 [2n, 1, HW] (clamped sin-latitude) -> g [n, 2, HW], l [n, 1, HW]:
//   g = normalize(a + M(b) * (-1, 1)) with F.normalize's rule v / max(|v|, 1e-12);  l = (a + M(b)) * 0.5.
__global__ void __launch_bounds__(256) flip_merge_reg_kernel(const float* __restrict__ g2, const float* __restrict__ l2, float* __restrict__ g,
                                                             float* __restrict__ l, int n, int H, int W) {
  const int HW = H * W;
  const int pix = blockIdx.x * blockDim.x + threadIdx.x;
  if (pix >= n * HW) return;
  const int i = pix / HW, r = pix - i * HW, y = r / W, x = r - y * W;
  const int rb = y * W + (W - 1 - x);
  const float* ga = g2 + (size_t)i * 2 * HW + r;
  const float* gb = g2 + (size_t)(n + i) * 2 * HW + rb;
  const float vx = __fsub_rn(__ldg(ga), __ldg(gb)), vy = __fadd_rn(__ldg(ga + HW), __ldg(gb + HW));
  const float nrm = fmaxf(__fsqrt_rn(__fadd_rn(__fmul_rn(vx, vx), __fmul_rn(vy, vy))), 1e-12f);
  float* go = g + (size_t)i * 2 * HW + r;
  go[0] = __fdiv_rn(vx, nrm);
  go[HW] = __fdiv_rn(vy, nrm);
  l[pix] = __fmul_rn(__fadd_rn(__ldg(l2 + (size_t)i * HW + r), __ldg(l2 + (size_t)(n + i) * HW + rb)), 0.5f);
}

// Class of the mirrored direction: up-direction bin c (angle 5c - 180 degrees for NC = 73) becomes 180 degrees minus that
// angle, bin (3 (NC - 1) / 2 - c) mod (NC - 1) = (36 - c) mod 72; the no-direction bin NC - 1 and every latitude class stay.
__host__ __device__ inline int flip_class(int c, int NC, int is_gravity) {
  if (!is_gravity || c >= NC - 1) return c;
  const int m = NC - 1;
  return (m + m / 2 - c) % m;
}
// the 1x1 prediction conv of one class on one pixel's 32 features: bias first, then channels 0..31 in order (pred_tail_kernel's
// fma chain, so the logits equal the unmerged path's bit for bit); wr: the class's weight row (16-byte aligned), b its bias
__device__ __forceinline__ float pred_logit(const float* f, const float* wr, float b) {
  const float4* w4 = reinterpret_cast<const float4*>(wr);
  float v = b;
#pragma unroll
  for (int d4 = 0; d4 < 8; ++d4) {
    const float4 ww = w4[d4];
    v = fmaf(f[4 * d4], ww.x, v); v = fmaf(f[4 * d4 + 1], ww.y, v); v = fmaf(f[4 * d4 + 2], ww.z, v); v = fmaf(f[4 * d4 + 3], ww.w, v);
  }
  return v;
}

// Classification heads, from the features: per output pixel (i, y, x) the 1x1 prediction conv 32 -> NC of conv1 features
// (32 channels at icoff of [2n * HW, ldi] NHWC) at slot i, pixel (y, x) (a) and at slot n + i, pixel (y, W - 1 - x) (b), and the
// merged logits (a_c + b_P(c)) * 0.5, P = flip_class.  The threads, weights and reductions are pred_argmax_decode_kernel's: a quad
// per pixel, lane q on the classes q, q + 4, ...; weights [NC][36] + bias in shared memory.
// kDecode = false: the merged logits to out [n, NC, HW] (the decode and confidence kernels then run on them unchanged).
// kDecode = true ("decode_only"): no logits are written; argmax (first maximal index), kRefine's sub-bin decode and kConf's
// confidence of the merged logits, in pred_argmax_decode_kernel's order, to out = the field [n, 2 or 1, HW] and conf [n, HW].
template <bool kDecode, bool kConf, bool kRefine>
__global__ void __launch_bounds__(256) pred_flip_kernel(const float* __restrict__ in, int ldi, int icoff, const float* __restrict__ w,
                                                        const float* __restrict__ bias, float* __restrict__ out, float* __restrict__ conf, int n, int H,
                                                        int W, int NC, int is_gravity) {
  extern __shared__ __align__(16) float s_pw[];  // [NC][36] then [NC]
  for (int i = threadIdx.x; i < NC * 32; i += blockDim.x) s_pw[(i >> 5) * 36 + (i & 31)] = __ldg(w + i);
  float* s_b = s_pw + NC * 36;
  for (int i = threadIdx.x; i < NC; i += blockDim.x) s_b[i] = __ldg(bias + i);
  __syncthreads();
  const int q = threadIdx.x & 3;
  const int HW = H * W;
  const long long npix = (long long)n * HW;
  const long long stride = (long long)gridDim.x * (blockDim.x >> 2);
  const long long pix_last = npix - 1;
  const long long iters = (npix + stride - 1) / stride;     // (the same on every lane: the shuffles need the full quad)
  long long pix = (long long)blockIdx.x * (blockDim.x >> 2) + (threadIdx.x >> 2);
  for (long long it = 0; it < iters; ++it, pix += stride) {
    const bool live = pix <= pix_last;
    const long long pc = live ? pix : pix_last;
    const int i = (int)(pc / HW), r = (int)(pc - (long long)i * HW), y = r / W, x = r - y * W;
    const long long pb = (long long)(n + i) * HW + y * W + (W - 1 - x);
    float fa[32], fb[32];
#pragma unroll
    for (int d = 0; d < 32; d += 4) {
      const float4 t = __ldg(reinterpret_cast<const float4*>(in + pc * ldi + icoff + d));
      fa[d] = t.x; fa[d + 1] = t.y; fa[d + 2] = t.z; fa[d + 3] = t.w;
      const float4 u = __ldg(reinterpret_cast<const float4*>(in + pb * ldi + icoff + d));
      fb[d] = u.x; fb[d + 1] = u.y; fb[d + 2] = u.z; fb[d + 3] = u.w;
    }
    auto merged = [&](int c) {
      const int p = flip_class(c, NC, is_gravity);
      return __fmul_rn(__fadd_rn(pred_logit(fa, s_pw + c * 36, s_b[c]), pred_logit(fb, s_pw + p * 36, s_b[p])), 0.5f);
    };
    if constexpr (!kDecode) {
      float* o = out + (long long)i * NC * HW + r;
      for (int c = q; c < NC; c += 4) {
        const float v = merged(c);
        if (live) o[(long long)c * HW] = v;
      }
    } else {
      float best = -INFINITY, cm = -INFINITY, cs = 0.0f;
      int bi = 0x7fffffff;
      for (int c = q; c < NC; c += 4) {
        const float v = merged(c);
        if (v > best || bi == 0x7fffffff) { best = v; bi = c; }
        if constexpr (kConf) conf_update(v, cm, cs);
      }
#pragma unroll
      for (int o = 1; o < 4; o <<= 1) {
        const float ov = __shfl_xor_sync(0xffffffffu, best, o);
        const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
        if (ov > best || (ov == best && oi < bi)) { best = ov; bi = oi; }
        if constexpr (kConf) {
          const float om = __shfl_xor_sync(0xffffffffu, cm, o), os = __shfl_xor_sync(0xffffffffu, cs, o);
          conf_merge(cm, cs, om, os);
        }
      }
      float lm = 0.0f, lp = 0.0f;
      if constexpr (kRefine) {
        const int2 nb = subbin_neighbours(NC, __shfl_sync(0xffffffffu, bi, 0, 4), is_gravity);
        lm = merged((q & 1) ? nb.y : nb.x);
        lp = __shfl_xor_sync(0xffffffffu, lm, 1);
      }
      if (live && q == 0) {
        if constexpr (kRefine) subbin_decode_store(out, i, r, HW, NC, bi, best, lm, lp, is_gravity);
        else decode_bin_store(out, i, r, HW, NC, bi, is_gravity);
        if constexpr (kConf) conf[pix] = 1.0f / cs;
      }
    }
  }
}

// =====================================================================================================
// ParamNet input: cat(pred_gravity, pred_latitude) (param_network.py:47-49 / 194-197), optionally the nearest
// IH x IW -> OH x OW sub-sample F.interpolate(images, (OH, OW)) (ATen nearest: src = floor(dst * (float)in / out), clamped).
// NCHW fields at the net size IH x IW -> NHWC [B,OH,OW,4].
__global__ void __launch_bounds__(256) pack_fields_kernel(const float* __restrict__ grav, const float* __restrict__ lat, float* __restrict__ out, int B, int IH,
                                                          int IW, int OH, int OW) {
  const long long total = (long long)B * OH * OW;
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int x = (int)(i % OW), y = (int)((i / OW) % OH), b = (int)(i / ((long long)OH * OW));
  const int sy = (int)floorf((float)y * ((float)IH / (float)OH)), sx = (int)floorf((float)x * ((float)IW / (float)OW));
  const long long IHW = (long long)IH * IW;
  const int sp = min(sy, IH - 1) * IW + min(sx, IW - 1);
  const float g0 = __ldg(grav + (long long)b * 2 * IHW + sp);
  const float g1 = __ldg(grav + (long long)b * 2 * IHW + IHW + sp);
  const float l0 = __ldg(lat + (long long)b * IHW + sp);
  reinterpret_cast<float4*>(out)[i] = make_float4(g0, g1, l0, 0.f);
}

// ParamNet tail: global average pool -> LayerNorm(768, eps 1e-6) -> Linear 768->5 (convnext.py:144-151), then
// the parameter scaling of param_network.py:54-67 (centered) / :205-220 (uncentered).  One block per image.
// params out: [B][8] = roll, pitch, vfov|general_vfov, rel_cx, rel_cy, rel_focal, raw2, 0
// kind 1 (ParamNet): vfov = x2*90, rel_focal = 1/2/tan(x2) (sic), cx = cy = 0.
// kind 2 (ParamNetConvNextRegress): general_vfov = x2*90, cx = x3, cy = x4, rel_focal = closed-form root of
//   cos(gvfov) = (p^2+q^2-1)/(2pq), p^2 = f^2+cx^2+(cy+.5)^2, q^2 = f^2+cx^2+(cy-.5)^2 (utils.py:47-91 solves the
//   same equation with scipy fsolve from f=1.5 and takes abs()).
// raw (optional, NULL to skip): [B][5] = x0..x4, the head's outputs before the scaling (the training branch's prediction).
__global__ void __launch_bounds__(256) param_tail_kernel(const float* __restrict__ feat, int HW, const float* __restrict__ nw, const float* __restrict__ nb,
                                                         const float* __restrict__ hw, const float* __restrict__ hb, float* __restrict__ params,
                                                         float* __restrict__ raw, int kind) {
  constexpr int C = 768;
  __shared__ float s_x[C];
  __shared__ float s_red[8];
  __shared__ float s_out[5];
  const int b = blockIdx.x, tid = threadIdx.x;
  const float* f = feat + (long long)b * HW * C;
  for (int c = tid; c < C; c += 256) {
    float s = 0.f;
    for (int p = 0; p < HW; ++p) s += f[(long long)p * C + c];
    s_x[c] = s / (float)HW;
  }
  __syncthreads();
  float s = 0.f;
  for (int c = tid; c < C; c += 256) s += s_x[c];
  s = warp_sum(s);
  if ((tid & 31) == 0) s_red[tid >> 5] = s;
  __syncthreads();
  float mean = 0.f;
  for (int i = 0; i < 8; ++i) mean += s_red[i];
  mean /= (float)C;
  __syncthreads();
  float q = 0.f;
  for (int c = tid; c < C; c += 256) { const float d = s_x[c] - mean; q = fmaf(d, d, q); }
  q = warp_sum(q);
  if ((tid & 31) == 0) s_red[tid >> 5] = q;
  __syncthreads();
  float var = 0.f;
  for (int i = 0; i < 8; ++i) var += s_red[i];
  const float rstd = 1.0f / sqrtf(var / (float)C + 1e-6f);
  __syncthreads();
  for (int c = tid; c < C; c += 256) s_x[c] = (s_x[c] - mean) * rstd * nw[c] + nb[c];
  __syncthreads();
  const int warp = tid >> 5, lane = tid & 31;
  if (warp < 5) {
    float a = 0.f;
    for (int c = lane; c < C; c += 32) a = fmaf(s_x[c], hw[warp * C + c], a);
    a = warp_sum(a);
    if (lane == 0) s_out[warp] = a + hb[warp];
  }
  __syncthreads();
  if (tid == 0) {
    float* o = params + b * 8;
    const float x0 = s_out[0], x1 = s_out[1], x2 = s_out[2], x3 = s_out[3], x4 = s_out[4];
    if (raw) { float* r = raw + b * 5; r[0] = x0; r[1] = x1; r[2] = x2; r[3] = x3; r[4] = x4; }
    o[0] = x0 * 90.0f; o[1] = x1 * 90.0f; o[2] = x2 * 90.0f; o[6] = x2; o[7] = 0.f;
    if (kind == 1) {
      o[3] = 0.f; o[4] = 0.f;
      o[5] = 1.0f / 2.0f / tanf(x2);
    } else {
      o[3] = x3; o[4] = x4;
      const double cx = (double)x3, cy = (double)x4;
      const double gv = (double)o[2] * (3.14159265358979323846 / 180.0);
      const double c = cos(gv), s2 = 1.0 - c * c;
      double A;
      if (s2 < 1e-300) A = INFINITY;
      else {
        const double D = 1.0 - s2 * (1.0 + 4.0 * c * c * cy * cy);
        const double rt = sqrt(fmax(D, 0.0));
        A = (c >= 0.0 ? (1.0 + rt) : (1.0 - rt)) / (2.0 * s2);
      }
      const double f2 = A - cx * cx - cy * cy - 0.25;
      o[5] = (float)sqrt(f2);   // NaN when the equation has no real root (fsolve does not converge there either)
    }
  }
}

}  // namespace pf
