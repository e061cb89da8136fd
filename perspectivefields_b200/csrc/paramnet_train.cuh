// CUDA-core kernels of ParamNet training (pf_param_train_forward / pf_param_backward): the backward of the ConvNeXt-T
// layers that are not GEMMs, the operand transposes that feed the weight-gradient GEMMs, and the deterministic reductions.
//
// Every parameter gradient is a sum over pixels.  None of them uses atomics: a kernel writes one partial sum per block of
// rows (a fixed partition that depends on the shapes only), and reduce_partials_kernel adds the partials in a fixed order.
// Repeated calls on the same inputs are therefore bit-identical.
#pragma once
#include "common.cuh"

namespace pf {

// out[l] = sum over p < P of part[p * L + l], p ascending within each of 8 interleaved groups, then the 8 groups in order.
__global__ void __launch_bounds__(256) reduce_partials_kernel(const float* __restrict__ part, int P, long long L, float* __restrict__ out) {
  __shared__ float s[8][33];
  const int lane = threadIdx.x & 31, g = threadIdx.x >> 5;
  const long long l = (long long)blockIdx.x * 32 + lane;
  float a = 0.f;
  if (l < L)
    for (int p = g; p < P; p += 8) a += part[(long long)p * L + l];
  s[g][lane] = a;
  __syncthreads();
  if (g == 0 && l < L) {
    float t = s[0][lane];
    for (int i = 1; i < 8; ++i) t += s[i][lane];
    out[l] = t;
  }
}

// part[p][c] = sum of src[r][c] over the rows r of block p (rows p * rpb .. p * rpb + rpb - 1 of R)
__global__ void __launch_bounds__(256) colsum_partial_kernel(const float* __restrict__ src, long long R, int C, long long rpb, float* __restrict__ part) {
  __shared__ float s[8][33];
  const int lane = threadIdx.x & 31, g = threadIdx.x >> 5;
  const int c = blockIdx.y * 32 + lane;
  const long long r0 = (long long)blockIdx.x * rpb, r1 = r0 + rpb < R ? r0 + rpb : R;
  float a = 0.f;
  if (c < C)
    for (long long r = r0 + g; r < r1; r += 8) a += src[r * C + c];
  s[g][lane] = a;
  __syncthreads();
  if (g == 0 && c < C) {
    float t = s[0][lane];
    for (int i = 1; i < 8; ++i) t += s[i][lane];
    part[(long long)blockIdx.x * C + c] = t;
  }
}

// Transposed split copy of a [R x C] row-major operand for the weight-gradient GEMM (reduction over R):
// element (r, c) -> offset (r / chunk) * sS + c * sC + r % chunk of both bf16 planes; rows R .. Rp - 1 are zero.
// Source: fp32 (src, ld) or, with SPLIT_SRC, the hi / lo planes its producer wrote (value = hi + lo).  OP 1 applies the exact-erf
// GELU on the way (the hidden activation of a ConvNeXt block from its pre-activation).
template <bool SPLIT_SRC, int OP>
__global__ void __launch_bounds__(256) transpose_split_kernel(const float* __restrict__ src, const __nv_bfloat16* __restrict__ shi,
                                                              const __nv_bfloat16* __restrict__ slo, int ld, long long R, long long Rp, int C,
                                                              int chunk, long long sS, long long sC, __nv_bfloat16* __restrict__ hi,
                                                              __nv_bfloat16* __restrict__ lo) {
  __shared__ float t[32][33];
  const long long r0 = (long long)blockIdx.x * 32;
  const int c0 = blockIdx.y * 32;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  for (int i = ty; i < 32; i += 8) {
    const long long r = r0 + i;
    const int c = c0 + tx;
    float v = 0.f;
    if (r < R && c < C) {
      const long long o = r * ld + c;
      v = SPLIT_SRC ? __bfloat162float(shi[o]) + __bfloat162float(slo[o]) : src[o];
      if (OP == 1) v = 0.5f * v * (1.0f + erff(v * 0.70710678118654752440f));
    }
    t[i][tx] = v;
  }
  __syncthreads();
  for (int i = ty; i < 32; i += 8) {
    const int c = c0 + i;
    const long long r = r0 + tx;
    if (c < C && r < Rp) store_split1(hi, lo, (r / chunk) * sS + c * sC + r % chunk, t[tx][i]);
  }
}

// du = dh * GELU'(u), GELU'(u) = Phi(u) + u phi(u) (exact erf), written over u; also the bf16 split planes of du
__global__ void __launch_bounds__(256) gelu_bwd_kernel(const float* __restrict__ dh, float* __restrict__ u, long long n,
                                                       __nv_bfloat16* __restrict__ hi, __nv_bfloat16* __restrict__ lo) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const float x = u[i];
    const float d = 0.5f * (1.0f + erff(x * 0.70710678118654752440f)) + x * 0.39894228040143267794f * expf(-0.5f * x * x);
    const float v = dh[i] * d;
    u[i] = v;
    if (hi) store_split1(hi, lo, i, v);
  }
}

// bf16 split planes of src [R x C] (optionally times scale[c])
__global__ void __launch_bounds__(256) scale_split_kernel(const float* __restrict__ src, const float* __restrict__ scale, long long n, int C,
                                                          __nv_bfloat16* __restrict__ hi, __nv_bfloat16* __restrict__ lo) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    store_split1(hi, lo, i, scale ? src[i] * scale[i % C] : src[i]);
}

__global__ void __launch_bounds__(256) add_inplace_kernel(float* __restrict__ a, const float* __restrict__ b, long long n) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) a[i] += b[i];
}

// pwconv2 gradients from G = dy^T h [C][K] (dy: gradient of the block output, h: hidden activation) and sdy[c] = sum_r dy[r][c]:
// out = x + gamma * (h W^T + b), so dW = gamma G, db = gamma sdy, dgamma = sum_k W[c][k] G[c][k] + b[c] sdy[c].  One warp per c.
__global__ void __launch_bounds__(256) pw2_grads_kernel(const float* __restrict__ G, const float* __restrict__ sdy, int C, int K,
                                                        const float* __restrict__ gamma, const __nv_bfloat16* __restrict__ whi,
                                                        const __nv_bfloat16* __restrict__ wlo, const float* __restrict__ b,
                                                        float* __restrict__ dW, float* __restrict__ db, float* __restrict__ dgamma) {
  const int c = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (c >= C) return;
  const float gc = gamma[c];
  float a = 0.f;
  for (int k = lane; k < K; k += 32) {
    const long long o = (long long)c * K + k;
    const float g = G[o];
    dW[o] = gc * g;
    a = fmaf(__bfloat162float(whi[o]) + __bfloat162float(wlo[o]), g, a);
  }
  a = warp_sum(a);
  if (lane == 0) {
    db[c] = gc * sdy[c];
    dgamma[c] = fmaf(b[c], sdy[c], a);
  }
}

// LayerNorm backward over the channels of [R x C] rows (C <= 768, eps inside the sqrt): dx = rstd (g - mean(g) - xhat mean(g xhat))
// with g = dy * w; dx is written (not accumulated).  Block p handles rows p * rpb ..; its partial sums of dy * xhat (dweight) and dy
// (dbias) go to part[p][0 .. C) and part[p][C .. 2C).
constexpr int kLnBwdMaxPer = 24;   // channels per lane: 768 / 32
__global__ void __launch_bounds__(256) ln_bwd_kernel(const float* __restrict__ x, const float* __restrict__ dy, long long R, int C,
                                                     const float* __restrict__ w, float eps, long long rpb, float* __restrict__ dx,
                                                     float* __restrict__ part) {
  __shared__ float s[2 * 768];
  const int lane = threadIdx.x & 31, wp = threadIdx.x >> 5;
  const int per = C / 32;
  const float inv_c = 1.0f / (float)C;
  float aw[kLnBwdMaxPer], ab[kLnBwdMaxPer];
#pragma unroll
  for (int i = 0; i < kLnBwdMaxPer; ++i) { aw[i] = 0.f; ab[i] = 0.f; }
  const long long r0 = (long long)blockIdx.x * rpb, r1 = r0 + rpb < R ? r0 + rpb : R;
  for (long long r = r0 + wp; r < r1; r += 8) {
    const float* xr = x + r * C;
    const float* gr = dy + r * C;
    float xv[kLnBwdMaxPer], gv[kLnBwdMaxPer];
    float sm = 0.f;
#pragma unroll
    for (int i = 0; i < kLnBwdMaxPer; ++i)
      if (i < per) { xv[i] = xr[lane + 32 * i]; sm += xv[i]; }
    const float mean = warp_sum(sm) * inv_c;
    float q = 0.f;
#pragma unroll
    for (int i = 0; i < kLnBwdMaxPer; ++i)
      if (i < per) { const float d = xv[i] - mean; q = fmaf(d, d, q); }
    const float rstd = 1.0f / sqrtf(fmaf(warp_sum(q), inv_c, eps));
    float s1 = 0.f, s2 = 0.f;
#pragma unroll
    for (int i = 0; i < kLnBwdMaxPer; ++i)
      if (i < per) {
        const int c = lane + 32 * i;
        const float xh = (xv[i] - mean) * rstd, d = gr[c];
        aw[i] = fmaf(d, xh, aw[i]);
        ab[i] += d;
        gv[i] = d * w[c];
        s1 += gv[i];
        s2 = fmaf(gv[i], xh, s2);
        xv[i] = xh;
      }
    s1 = warp_sum(s1) * inv_c;
    s2 = warp_sum(s2) * inv_c;
#pragma unroll
    for (int i = 0; i < kLnBwdMaxPer; ++i)
      if (i < per) dx[r * C + lane + 32 * i] = rstd * (gv[i] - s1 - xv[i] * s2);
  }
  // warps' partials in warp order
  for (int k = 0; k < 8; ++k) {
    if (wp == k)
#pragma unroll
      for (int i = 0; i < kLnBwdMaxPer; ++i)
        if (i < per) {
          const int c = lane + 32 * i;
          s[c] = k ? s[c] + aw[i] : aw[i];
          s[C + c] = k ? s[C + c] + ab[i] : ab[i];
        }
    __syncthreads();
  }
  for (int c = threadIdx.x; c < 2 * C; c += 256) part[(long long)blockIdx.x * 2 * C + c] = s[c];
}

// Depthwise 7x7 (pad 3) weight and bias gradients: dW[tap][c] = sum over pixels of dt[b, y, x, c] x[b, y + ky - 3, x + kx - 3, c],
// db[c] = sum dt.  Block (p, channel block of 32): image rows p * rpb .. (over all images: row index b * H + y); warp k takes one
// contiguous run of columns of every row and slides a 7-wide register window of x along it, so each input value is loaded once
// per filter row instead of once per tap.  Partials part[p][tap * C + c] (tap 49 = bias), combined over the warps in order.
__global__ void __launch_bounds__(256) dw7_wgrad_kernel(const float* __restrict__ x, const float* __restrict__ dt, int B, int H, int W, int C,
                                                        int rpb, float* __restrict__ part) {
  __shared__ float s[50][32];
  const int lane = threadIdx.x & 31, wp = threadIdx.x >> 5;
  const int c = blockIdx.y * 32 + lane;
  float acc[50];
#pragma unroll
  for (int i = 0; i < 50; ++i) acc[i] = 0.f;
  const int row0 = blockIdx.x * rpb, row1 = min(row0 + rpb, B * H);
  const int seg = (W + 7) / 8, xs = wp * seg, xe = min(W, xs + seg);
  if (c < C && xs < xe)
    for (int row = row0; row < row1; ++row) {
      const int b = row / H, y = row - b * H;
      const float* xb = x + (long long)b * H * W * C + c;
      const float* gr = dt + (long long)row * W * C + c;
      for (int xx = xs; xx < xe; ++xx) acc[49] += gr[(long long)xx * C];
#pragma unroll
      for (int ky = 0; ky < 7; ++ky) {
        const int iy = y + ky - 3;
        if ((unsigned)iy >= (unsigned)H) continue;
        const float* xr = xb + (long long)iy * W * C;
        float win[7];
#pragma unroll
        for (int k = 0; k < 7; ++k) {
          const int ix = xs + k - 3;
          win[k] = (unsigned)ix < (unsigned)W ? xr[(long long)ix * C] : 0.f;
        }
        for (int xx = xs; xx < xe; ++xx) {
          const float g = gr[(long long)xx * C];
#pragma unroll
          for (int kx = 0; kx < 7; ++kx) acc[ky * 7 + kx] = fmaf(g, win[kx], acc[ky * 7 + kx]);
#pragma unroll
          for (int k = 0; k < 6; ++k) win[k] = win[k + 1];
          const int ix = xx + 4;
          win[6] = ix < W ? xr[(long long)ix * C] : 0.f;
        }
      }
    }
  for (int k = 0; k < 8; ++k) {
    if (wp == k)
#pragma unroll
      for (int i = 0; i < 50; ++i) s[i][lane] = k ? s[i][lane] + acc[i] : acc[i];
    __syncthreads();
  }
  for (int i = threadIdx.x; i < 50 * 32; i += 256) {
    const int tap = i >> 5, cc = blockIdx.y * 32 + (i & 31);
    if (cc < C) part[(long long)blockIdx.x * 50 * C + tap * C + cc] = s[tap][i & 31];
  }
}

// ParamNet stem (4x4 / stride 4, 3 -> 96) weight and bias gradients from dS [B, OH, OW, 96] and the packed input [B, 4 OH, 4 OW, 4]:
// dW[(ky, kx, ci)][co] (the engine's stem layout), db[co].  Block (p, co block): output rows p * rpb .. ; partials
// part[p][j * 96 + co], j = 48 for the bias.
__global__ void __launch_bounds__(256) stem_wgrad_kernel(const float* __restrict__ pin, const float* __restrict__ dS, int B, int OH, int OW, int rpb,
                                                         float* __restrict__ part) {
  __shared__ float s[49][32];
  const int lane = threadIdx.x & 31, wp = threadIdx.x >> 5;
  const int co = blockIdx.y * 32 + lane;
  float acc[49];
#pragma unroll
  for (int i = 0; i < 49; ++i) acc[i] = 0.f;
  const int row0 = blockIdx.x * rpb, row1 = min(row0 + rpb, B * OH);
  const int W = OW * 4;
  for (int row = row0; row < row1; ++row) {
    const int b = row / OH, oy = row - b * OH;
    for (int ox = wp; ox < OW; ox += 8) {
      const float g = dS[((long long)row * OW + ox) * 96 + co];
      acc[48] += g;
#pragma unroll
      for (int ky = 0; ky < 4; ++ky) {
        const float4* pr = reinterpret_cast<const float4*>(pin + (((long long)b * OH * 4 + oy * 4 + ky) * W + ox * 4) * 4);
#pragma unroll
        for (int kx = 0; kx < 4; ++kx) {
          const float4 v = __ldg(pr + kx);
          const int j = (ky * 4 + kx) * 3;
          acc[j] = fmaf(g, v.x, acc[j]); acc[j + 1] = fmaf(g, v.y, acc[j + 1]); acc[j + 2] = fmaf(g, v.z, acc[j + 2]);
        }
      }
    }
  }
  for (int k = 0; k < 8; ++k) {
    if (wp == k)
#pragma unroll
      for (int i = 0; i < 49; ++i) s[i][lane] = k ? s[i][lane] + acc[i] : acc[i];
    __syncthreads();
  }
  for (int i = threadIdx.x; i < 49 * 32; i += 256) {
    const int j = i >> 5;
    part[(long long)blockIdx.x * 49 * 96 + j * 96 + blockIdx.y * 32 + (i & 31)] = s[j][i & 31];
  }
}

// stem data gradient: dpin[b, 4 oy + ky, 4 ox + kx, ci] = sum_co dS[b, oy, ox, co] w[(ky, kx, ci)][co]; one thread per (pixel, j < 48).
// The patches do not overlap, so every input element is written once (channel 3 of the packed input is left alone).
__global__ void __launch_bounds__(256) stem_dgrad_kernel(const float* __restrict__ dS, const float* __restrict__ w, int B, int OH, int OW,
                                                         float* __restrict__ dpin) {
  const long long total = (long long)B * OH * OW * 48;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int j = (int)(i % 48);
    const long long pix = i / 48;
    const int ox = (int)(pix % OW), oy = (int)((pix / OW) % OH), b = (int)(pix / ((long long)OW * OH));
    const float* g = dS + pix * 96;
    const float* wr = w + j * 96;
    float a = 0.f;
    for (int co = 0; co < 96; ++co) a = fmaf(g[co], wr[co], a);
    const int ky = j / 12, kx = (j / 3) % 4, ci = j % 3;
    dpin[(((long long)b * OH * 4 + oy * 4 + ky) * (OW * 4) + ox * 4 + kx) * 4 + ci] = a;
  }
}

// Gradient of pack_fields_kernel: dpin [B, OH, OW, 4] -> d gravity [B, 2, IH, IW], d latitude [B, 1, IH, IW].  Source pixel
// (sy, sx) collects every output pixel whose nearest source it is (the forward's formula), rows then columns ascending; a source
// no output picks gets zero.
__global__ void __launch_bounds__(256) unpack_fields_grad_kernel(const float* __restrict__ dpin, int B, int IH, int IW, int OH, int OW,
                                                                 float* __restrict__ dgrav, float* __restrict__ dlat) {
  const long long total = (long long)B * IH * IW;
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int sx = (int)(i % IW), sy = (int)((i / IW) % IH), b = (int)(i / ((long long)IH * IW));
  const float fy = (float)IH / (float)OH, fx = (float)IW / (float)OW;
  auto src_y = [&](int y) { return min((int)floorf((float)y * fy), IH - 1); };
  auto src_x = [&](int x) { return min((int)floorf((float)x * fx), IW - 1); };
  // candidates: y with y * fy within one of sy (the floor is monotone in y)
  const int ylo = max(0, (int)((float)sy / fy) - 2), yhi = min(OH - 1, (int)((float)(sy + 1) / fy) + 2);
  const int xlo = max(0, (int)((float)sx / fx) - 2), xhi = min(OW - 1, (int)((float)(sx + 1) / fx) + 2);
  float g0 = 0.f, g1 = 0.f, l0 = 0.f;
  for (int y = ylo; y <= yhi; ++y) {
    if (src_y(y) != sy) continue;
    for (int x = xlo; x <= xhi; ++x) {
      if (src_x(x) != sx) continue;
      const float4 v = reinterpret_cast<const float4*>(dpin)[((long long)b * OH + y) * OW + x];
      g0 += v.x; g1 += v.y; l0 += v.z;
    }
  }
  const long long IHW = (long long)IH * IW, sp = (long long)sy * IW + sx;
  dgrav[(long long)b * 2 * IHW + sp] = g0;
  dgrav[(long long)b * 2 * IHW + IHW + sp] = g1;
  dlat[(long long)b * IHW + sp] = l0;
}

// Gradient of the 2x2 / stride 2 patch matrix [B * (H/2) * (W/2), 4 C] (column ((y % 2) * 2 + x % 2) * C + c) back to the
// [B, H, W, C] map it was gathered from: a permutation, the patches do not overlap.
__global__ void __launch_bounds__(256) col2im2_kernel(const float* __restrict__ dP, int B, int H, int W, int C, float* __restrict__ out) {
  const long long total = (long long)B * H * W * C;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % C);
    const long long pix = i / C;
    const int x = (int)(pix % W), y = (int)((pix / W) % H), b = (int)(pix / ((long long)W * H));
    const long long prow = ((long long)b * (H / 2) + y / 2) * (W / 2) + x / 2;
    out[i] = dP[prow * 4 * C + ((y % 2) * 2 + x % 2) * C + c];
  }
}

// Backward of param_tail_kernel's pool -> LayerNorm(768) -> Linear 768 -> 5 for one pair per block, from draw [B][5] (the gradient
// of the raw head outputs).  dx[b][p][c] = dfeat[c] / HW for every pixel p; per-pair partials part[b][...] of the tail parameters
// in the order norm.w (768), norm.b (768), head.w (5 x 768), head.b (5).
constexpr int kTailGrads = 768 * 2 + 5 * 768 + 5;
__global__ void __launch_bounds__(256) param_tail_bwd_kernel(const float* __restrict__ feat, int HW, const float* __restrict__ nw,
                                                             const float* __restrict__ nb, const float* __restrict__ hw, const float* __restrict__ draw,
                                                             float* __restrict__ dx, float* __restrict__ part) {
  constexpr int C = 768;
  __shared__ float s_x[C], s_d[C];
  __shared__ float s_red[8];
  __shared__ float s_g[5];
  const int b = blockIdx.x, tid = threadIdx.x;
  const float* f = feat + (long long)b * HW * C;
  for (int c = tid; c < C; c += 256) {
    float s = 0.f;
    for (int p = 0; p < HW; ++p) s += f[(long long)p * C + c];
    s_x[c] = s / (float)HW;
  }
  if (tid < 5) s_g[tid] = draw[b * 5 + tid];
  __syncthreads();
  auto block_sum = [&](float v) {
    v = warp_sum(v);
    if ((tid & 31) == 0) s_red[tid >> 5] = v;
    __syncthreads();
    float t = 0.f;
    for (int i = 0; i < 8; ++i) t += s_red[i];
    __syncthreads();
    return t;
  };
  float s = 0.f;
  for (int c = tid; c < C; c += 256) s += s_x[c];
  const float mean = block_sum(s) / (float)C;
  float q = 0.f;
  for (int c = tid; c < C; c += 256) { const float d = s_x[c] - mean; q = fmaf(d, d, q); }
  const float rstd = 1.0f / sqrtf(block_sum(q) / (float)C + 1e-6f);
  float* pp = part + (long long)b * kTailGrads;
  if (tid < 5) pp[2 * C + 5 * C + tid] = s_g[tid];                    // d head.b
  float s1 = 0.f, s2 = 0.f;
  for (int c = tid; c < C; c += 256) {
    const float xh = (s_x[c] - mean) * rstd;
    const float fo = xh * nw[c] + nb[c];                               // the head's input
    float df = 0.f;
    for (int k = 0; k < 5; ++k) {
      df = fmaf(s_g[k], hw[k * C + c], df);
      pp[2 * C + k * C + c] = s_g[k] * fo;                             // d head.w
    }
    pp[c] = df * xh;            // d norm.w
    pp[C + c] = df;             // d norm.b
    const float g = df * nw[c];
    s_d[c] = g;
    s1 += g;
    s2 = fmaf(g, xh, s2);
    s_x[c] = xh;
  }
  s1 = block_sum(s1) / (float)C;
  s2 = block_sum(s2) / (float)C;
  __syncthreads();
  for (int c = tid; c < C; c += 256) s_d[c] = rstd * (s_d[c] - s1 - s_x[c] * s2) / (float)HW;
  __syncthreads();
  float* dxb = dx + (long long)b * HW * C;
  for (long long i = tid; i < (long long)HW * C; i += 256) dxb[i] = s_d[i % C];
}

}  // namespace pf
