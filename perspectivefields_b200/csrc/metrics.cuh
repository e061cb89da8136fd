// Scoring of predictions against ground-truth perspective fields: the reference's bin encoders (utils/utils.py:94-146), the
// heads' training losses (gravity_head.py:199-235, latitude_head.py:221-254, persformer_heads/loss_fns.py:5-43) and this
// project's per-image field errors (DESIGN.md section 1).  Every reduction writes per-block partials (fp64 sums, integer
// counts) and a final pass sums them in a fixed order: two identical calls give bit-identical results, and no floating-point
// atomic decides a value.
#pragma once
#include <stdint.h>

#include "common.cuh"

namespace pf {

constexpr int kMetThreads = 256;

// Deterministic block sum (fixed shuffle tree, then the warps' partials in order by warp 0).  Every thread gets the result.
template <class T>
__device__ __forceinline__ T block_sum(T v, T* sh) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
  __syncthreads();   // sh may still be read by the previous call
  if (lane == 0) sh[warp] = v;
  __syncthreads();
  if (warp == 0) {
    v = lane < nw ? sh[lane] : T(0);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
    if (lane == 0) sh[32] = v;
  }
  __syncthreads();
  return sh[32];
}

// ------------------------------------------------------------------------------------------------------------- encoders
// encode_bin (utils.py:94-111) in float32 in the reference's order, every step an explicit round-to-nearest operation so that
// nvcc contracts nothing: atan2(y, x) / pi_f * 180 + 180, remainder by 360, / (360 / (NB - 1)), round half to even; bin NB - 1
// wraps to 0 and an all-zero vector gets NB - 1.
__device__ __forceinline__ long long encode_gravity_bin(float x, float y, int NB) {
  if (x == 0.f && y == 0.f) return NB - 1;
  float a = __fadd_rn(__fmul_rn(__fdiv_rn(atan2f(y, x), 3.14159265358979323846f), 180.f), 180.f);
  a = fmodf(a, 360.f);
  if (a < 0.f) a = __fadd_rn(a, 360.f);   // torch.remainder's sign rule (a >= 0 here except for rounding)
  long long b = (long long)rintf(__fdiv_rn(a, gravity_bin_deg(NB)));
  return b == NB - 1 ? 0 : b;
}
// encode_bin_latitude (utils.py:133-146): bucketize(right=False) against float32 arange(-90, 90, 180 / NC)[1:], torch's
// lower-bound search (a NaN latitude lands in the last class, as there).
__device__ __forceinline__ long long encode_latitude_bin(float v, int NC) {
  const float step = latitude_bin_deg(NC);
  int lo = 0, hi = NC - 1;
  while (lo < hi) {
    const int mid = lo + ((hi - lo) >> 1);
    const float b = __fadd_rn(-90.f, __fmul_rn((float)(mid + 1), step));
    if (!(b >= v)) lo = mid + 1; else hi = mid;
  }
  return lo;
}

struct EncodeArgs {
  int n, H, W;
  const float* up; long long us_img, us_row, us_col, us_comp;   // element strides
  const float* lat; long long ls_img, ls_row, ls_col;
  int lat_rad;         // lat holds radians (else degrees)
  int gc, lc;          // 2 / 1: regression targets (float32), else the class counts of the encoders (int64 labels)
  void* gt_g; void* gt_l;
};

// One thread per pixel: gt_g [n, 2, H, W] float32 (the up vector's (x, y)) or [n, H, W] int64; gt_l [n, 1, H, W] float32
// sin(latitude) or [n, H, W] int64.
__global__ void __launch_bounds__(kMetThreads) encode_fields_kernel(EncodeArgs a) {
  const long long HW = (long long)a.H * a.W;
  const long long q = (long long)blockIdx.x * kMetThreads + threadIdx.x;
  if (q >= (long long)a.n * HW) return;
  const long long b = q / HW, r = q - b * HW, y = r / a.W, x = r - y * a.W;
  if (a.up) {
    const float* u = a.up + b * a.us_img + y * a.us_row + x * a.us_col;
    const float ux = u[0], uy = u[a.us_comp];
    if (a.gc == 2) {
      float* o = (float*)a.gt_g + b * 2 * HW + r;
      o[0] = ux; o[HW] = uy;
    } else {
      ((long long*)a.gt_g)[q] = encode_gravity_bin(ux, uy, a.gc);
    }
  }
  if (a.lat) {
    float v = a.lat[b * a.ls_img + y * a.ls_row + x * a.ls_col];
    if (a.lc == 1) {
      const double rad = a.lat_rad ? (double)v : (double)v * (3.14159265358979323846 / 180.0);
      ((float*)a.gt_l)[q] = (float)sin(rad);
    } else {
      if (a.lat_rad) v = __fmul_rn(v, (float)(180.0 / 3.14159265358979323846));   // torch.rad2deg in float32
      ((long long*)a.gt_l)[q] = encode_latitude_bin(v, a.lc);
    }
  }
}

// ------------------------------------------------------------------------------------------------------ cross-entropy
// F.cross_entropy(logits, labels, reduction="mean", ignore_index) of both classification heads in one launch.  One thread owns
// 4 consecutive pixels and walks the C channel planes (stride H*W) with 16-byte streaming loads, keeping an online max and sum
// of exp in fp32 and picking up the target logit in the same pass: every logit is read from HBM once.  A logit of -inf adds
// nothing (exp(-inf) = 0, also while the running max is still -inf).  The pixel's loss is (max - target) + log(sum): the
// difference is exact for the argmax target, so a confident pixel keeps log(sum)'s precision whatever the logits' magnitude.
// A label that is neither the ignore value nor in [0, C) contributes NaN (never an out-of-bounds read).
constexpr int kCePix = 4, kCeUnroll = 8;
struct CeHead {
  const float* logits;       // [n, C, HW], 16-byte aligned
  const long long* labels;   // [n, HW]
  int C, ignore;
  int blocks;                // blocks of this head
};

__global__ void __launch_bounds__(kMetThreads) cross_entropy_kernel(CeHead g, CeHead l, int n, int HW, double* psum, long long* pcnt) {
  __shared__ double shd[33];
  __shared__ long long shl[33];
  const bool grav = (int)blockIdx.x < g.blocks;
  const CeHead h = grav ? g : l;
  const int blk = grav ? blockIdx.x : blockIdx.x - g.blocks;
  const long long q = ((long long)blk * kMetThreads + threadIdx.x) * kCePix;
  double sum = 0.0;
  long long cnt = 0;
  if (q < (long long)n * HW) {
    const long long b = q / HW, r = q - b * HW;
    const float4* p = reinterpret_cast<const float4*>(h.logits + b * h.C * HW + r);
    const long long hw4 = HW / 4;
    long long lab[kCePix];
#pragma unroll
    for (int k = 0; k < kCePix; ++k) lab[k] = h.labels[q + k];
    float m[kCePix], s[kCePix], xt[kCePix];
#pragma unroll
    for (int k = 0; k < kCePix; ++k) { m[k] = -INFINITY; s[k] = 0.f; xt[k] = 0.f; }
    for (int c0 = 0; c0 < h.C; c0 += kCeUnroll) {
      float4 v[kCeUnroll];
#pragma unroll
      for (int j = 0; j < kCeUnroll; ++j)
        if (c0 + j < h.C) v[j] = __ldcs(p + (long long)(c0 + j) * hw4);
#pragma unroll
      for (int j = 0; j < kCeUnroll; ++j) {
        if (c0 + j >= h.C) break;
        const float e[kCePix] = {v[j].x, v[j].y, v[j].z, v[j].w};
#pragma unroll
        for (int k = 0; k < kCePix; ++k) {
          const float t = e[k] == -INFINITY ? 0.f : __expf(-fabsf(e[k] - m[k]));   // exp(min - max); 0 while m is -inf
          s[k] = e[k] > m[k] ? s[k] * t + 1.f : s[k] + t;
          m[k] = fmaxf(m[k], e[k]);
          if (lab[k] == c0 + j) xt[k] = e[k];
        }
      }
    }
#pragma unroll
    for (int k = 0; k < kCePix; ++k) {
      if (lab[k] == h.ignore) continue;
      const bool ok = lab[k] >= 0 && lab[k] < h.C;
      sum += ok ? (double)((m[k] - xt[k]) + logf(s[k])) : (double)NAN;
      ++cnt;
    }
  }
  sum = block_sum(sum, shd);
  cnt = block_sum(cnt, shl);
  if (threadIdx.x == 0) { psum[blockIdx.x] = sum; pcnt[blockIdx.x] = cnt; }
}

// ------------------------------------------------------------------------------------------------------ regression losses
// One pass over the regression heads' predictions and targets (gravity [n, 2, H, W], latitude [n, 1, H, W]):
//   msgil_norm_loss (loss_fns.py:27-43): at scale s the pixels of the ::2^s grid are compared with their neighbours two grid
//     steps (2 * 2^s pixels) below and to the right; |d(p) - d(q)| with d = pred - target, counted where both masks hold.  Each
//     scale keeps its own sum and count.  Masks: gravity |t| > 1e-5 on both channels (gravity_head.py:206-207), latitude all.
//   the L2 terms: masked sum of |pred - t|^2 over the gravity pixels; sum of (pred - t)^2 over every latitude pixel.
// Per block: 10 fp64 sums (gravity scales 0-3, latitude scales 0-3, gravity L2, latitude L2) and 9 counts (gravity scales,
// latitude scales, gravity L2 pixels) as planes [quantity][block].
constexpr int kRegSums = 10, kRegCounts = 9, kRegPix = 16;
struct RegArgs { const float* pg; const float* tg; const float* pl; const float* tl; int n, H, W; };

__device__ __forceinline__ bool grav_valid(const float* t, long long HW) {
  const float a = t[0], b = t[HW];
  return __fsqrt_rn(__fadd_rn(__fmul_rn(a, a), __fmul_rn(b, b))) > 1e-5f;
}

__global__ void __launch_bounds__(kMetThreads) regression_loss_kernel(RegArgs a, int nblocks, double* psum, long long* pcnt) {
  __shared__ double shd[33];
  __shared__ long long shl[33];
  const long long HW = (long long)a.H * a.W;
  double sums[kRegSums];
  long long cnts[kRegCounts];
#pragma unroll
  for (int k = 0; k < kRegSums; ++k) sums[k] = 0.0;
#pragma unroll
  for (int k = 0; k < kRegCounts; ++k) cnts[k] = 0;
  for (int it = 0; it < kRegPix; ++it) {   // kRegPix coalesced rows of pixels per block amortise its 19 block reductions
    const long long q = ((long long)blockIdx.x * kRegPix + it) * kMetThreads + threadIdx.x;
    if (q >= (long long)a.n * HW) break;
    const long long b = q / HW, r = q - b * HW;
    const int y = (int)(r / a.W), x = (int)(r - (long long)y * a.W);
    const float* pg = a.pg + b * 2 * HW + r;
    const float* tg = a.tg + b * 2 * HW + r;
    const float* pl = a.pl + b * HW + r;
    const float* tl = a.tl + b * HW + r;
    const float d0 = __fsub_rn(pg[0], tg[0]), d1 = __fsub_rn(pg[HW], tg[HW]), dl = __fsub_rn(pl[0], tl[0]);
    const bool mp = grav_valid(tg, HW);
    if (mp) { sums[8] += (double)__fadd_rn(__fmul_rn(d0, d0), __fmul_rn(d1, d1)); cnts[8] += 1; }
    sums[9] += (double)__fmul_rn(dl, dl);
#pragma unroll
    for (int s = 0; s < 4; ++s) {
      const int step = 1 << s;
      if ((y & (step - 1)) || (x & (step - 1))) break;   // not on this scale's grid (nor on any coarser one)
#pragma unroll
      for (int dir = 0; dir < 2; ++dir) {
        const bool in = dir == 0 ? y + 2 * step < a.H : x + 2 * step < a.W;
        if (!in) continue;
        const long long o = dir == 0 ? 2LL * step * a.W : 2LL * step;
        const float el = __fsub_rn(pl[o], tl[o]);
        sums[4 + s] += (double)fabsf(__fsub_rn(dl, el));
        cnts[4 + s] += 1;
        if (mp && grav_valid(tg + o, HW)) {
          const float e0 = __fsub_rn(pg[o], tg[o]), e1 = __fsub_rn(pg[o + HW], tg[o + HW]);
          sums[s] += (double)fabsf(__fsub_rn(d0, e0)) + (double)fabsf(__fsub_rn(d1, e1));
          cnts[s] += 2;
        }
      }
    }
  }
#pragma unroll
  for (int k = 0; k < kRegSums; ++k) {
    const double v = block_sum(sums[k], shd);
    if (threadIdx.x == 0) psum[(long long)k * nblocks + blockIdx.x] = v;
  }
#pragma unroll
  for (int k = 0; k < kRegCounts; ++k) {
    const long long v = block_sum(cnts[k], shl);
    if (threadIdx.x == 0) pcnt[(long long)k * nblocks + blockIdx.x] = v;
  }
}

// Fixed-order sum of plane k of a [quantity][nblocks] partials array (each thread a strided serial sum, then block_sum).
template <class T>
__device__ __forceinline__ T sum_plane(const T* p, int k, int nblocks, T* sh) {
  T v = T(0);
  for (int i = threadIdx.x; i < nblocks; i += blockDim.x) v += p[(long long)k * nblocks + i];
  return block_sum(v, sh);
}

// The losses dicts' values (one block):
//   mode 0 (classification): out[0] = loss_gravity, out[1] = loss_latitude (sum / count * weight; NaN for no counted pixel).
//   mode 1 (regression): gravity-msg-normal-loss, gravity-l2-loss, latitude-msg-normal-loss, latitude-l2-loss.
__global__ void __launch_bounds__(kMetThreads) loss_finish_kernel(int mode, int nblocks_g, int nblocks, const double* psum, const long long* pcnt,
                                                                  long long lat_pixels, float wg, float wl, float* out) {
  __shared__ double shd[33];
  __shared__ long long shl[33];
  if (mode == 0) {
    // the partials of the two heads lie one after the other: plane 0 of the gravity blocks, then of the latitude blocks
    const double sg = sum_plane(psum, 0, nblocks_g, shd), sl = sum_plane(psum + nblocks_g, 0, nblocks - nblocks_g, shd);
    const long long cg = sum_plane(pcnt, 0, nblocks_g, shl), cl = sum_plane(pcnt + nblocks_g, 0, nblocks - nblocks_g, shl);
    if (threadIdx.x == 0) {
      out[0] = (float)(sg / (double)cg * (double)wg);
      out[1] = (float)(sl / (double)cl * (double)wl);
    }
    return;
  }
  double msg_g = 0.0, msg_l = 0.0;
  for (int s = 0; s < 4; ++s) {
    const double sg = sum_plane(psum, s, nblocks, shd), sl = sum_plane(psum, 4 + s, nblocks, shd);
    const long long cg = sum_plane(pcnt, s, nblocks, shl), cl = sum_plane(pcnt, 4 + s, nblocks, shl);
    msg_g += sg / ((double)cg + 1e-8);
    msg_l += sl / ((double)cl + 1e-8);
  }
  const double l2g = sum_plane(psum, 8, nblocks, shd), l2l = sum_plane(psum, 9, nblocks, shd);
  const long long cg = sum_plane(pcnt, 8, nblocks, shl);
  if (threadIdx.x == 0) {
    out[0] = (float)(0.1 * msg_g * (double)wg);
    out[1] = (float)(l2g / (double)cg * (double)wg);
    out[2] = (float)(0.1 * msg_l * (double)wl);
    out[3] = (float)(l2l / (double)lat_pixels * (double)wl);
  }
}

// ------------------------------------------------------------------------------------------------------ field errors
// Per-pixel errors of the predictions at the original size against ground truth (this project's rule, DESIGN.md section 1):
//   up: atan2(|p x g|, p . g) in degrees, valid where g is finite and |g| > 1e-5 (and the mask holds); a prediction that is not
//       finite or has |p| <= 1e-5 (the decoder's "no direction" bin) counts as 180.
//   latitude: |p - g| in degrees, valid where g is finite (and the mask holds); a non-finite prediction counts as +inf.
// Maps hold NaN at invalid pixels.  A block owns kFeTile pixels of one image and writes fp64 sums and integer counts (valid
// pixels, then pixels under each threshold) per field as planes [field][quantity][block].
constexpr int kFeTile = 16 * kMetThreads, kFeMaxThr = 8, kFeSelThreads = 1024;   // 16 pixels per thread amortise the 20 block sums
struct FeImage {
  int H, W;
  long long pu_off, pu_sr, pu_sc, pu_sk;   // predicted up: offset and element strides (row, column, component)
  long long pl_off;                        // predicted latitude [H, W]
  long long gu_off, gu_sr, gu_sc, gu_sk;
  long long gl_off;
  long long mask_off;                      // bytes, -1: none
  long long map_off;                       // first pixel of this image in the maps
  int block0, nblk;                        // its blocks in the error pass
};
struct FeArgs {
  const FeImage* im; int n, nblocks;
  const float* pu; const float* pl; const float* gu; const float* gl; const unsigned char* mask;
  int lat_rad, T;
  double thr[kFeMaxThr];
  float* map_up; float* map_lat;
  double* psum;          // [2][nblocks]
  int* pcnt;             // [2][1 + T][nblocks]
};

__global__ void __launch_bounds__(kMetThreads) field_errors_kernel(FeArgs a) {
  __shared__ double shd[33];
  __shared__ int shi[33];
  int lo = 0, hi = a.n - 1;   // the image this block belongs to: the last one with block0 <= blockIdx.x
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (a.im[mid].block0 <= (int)blockIdx.x) lo = mid; else hi = mid - 1;
  }
  const FeImage d = a.im[lo];
  const long long HW = (long long)d.H * d.W;
  const long long t0 = (long long)((int)blockIdx.x - d.block0) * kFeTile;
  double sum[2] = {0.0, 0.0};
  int cnt[2][1 + kFeMaxThr] = {};
#pragma unroll 4
  for (int i = 0; i < kFeTile / kMetThreads; ++i) {
    const long long r = t0 + i * kMetThreads + threadIdx.x;
    if (r >= HW) break;
    const int y = (int)(r / d.W), x = (int)(r - (long long)y * d.W);
    const bool m = d.mask_off < 0 || a.mask[d.mask_off + r] != 0;
    float e[2];
    {
      const float* g = a.gu + d.gu_off + y * d.gu_sr + x * d.gu_sc;
      const double gx = g[0], gy = g[d.gu_sk];
      const bool ok = m && isfinite(gx) && isfinite(gy) && sqrt(gx * gx + gy * gy) > 1e-5;
      if (ok) {
        const float* p = a.pu + d.pu_off + y * d.pu_sr + x * d.pu_sc;
        const double px = p[0], py = p[d.pu_sk];
        if (isfinite(px) && isfinite(py) && sqrt(px * px + py * py) > 1e-5)
          e[0] = (float)(atan2(fabs(px * gy - py * gx), px * gx + py * gy) * (180.0 / 3.14159265358979323846));
        else
          e[0] = 180.f;
      } else {
        e[0] = NAN;
      }
    }
    {
      double g = a.gl[d.gl_off + r];
      if (a.lat_rad) g = g * (180.0 / 3.14159265358979323846);
      if (m && isfinite(g)) {
        const double p = a.pl[d.pl_off + r];
        e[1] = isfinite(p) ? (float)fabs(p - g) : INFINITY;
      } else {
        e[1] = NAN;
      }
    }
    a.map_up[d.map_off + r] = e[0];
    a.map_lat[d.map_off + r] = e[1];
#pragma unroll
    for (int f = 0; f < 2; ++f) {
      if (e[f] != e[f]) continue;
      sum[f] += (double)e[f];
      cnt[f][0] += 1;
#pragma unroll
      for (int k = 0; k < kFeMaxThr; ++k)
        if (k < a.T && (double)e[f] < a.thr[k]) cnt[f][1 + k] += 1;
    }
  }
#pragma unroll
  for (int f = 0; f < 2; ++f) {
    const double s = block_sum(sum[f], shd);
    if (threadIdx.x == 0) a.psum[(long long)f * a.nblocks + blockIdx.x] = s;
#pragma unroll
    for (int k = 0; k < 1 + kFeMaxThr; ++k) {
      if (k > a.T) break;
      const int c = block_sum(cnt[f][k], shi);
      if (threadIdx.x == 0) a.pcnt[((long long)f * (1 + a.T) + k) * a.nblocks + blockIdx.x] = c;
    }
  }
}

// One block per (image, field): the statistics from the partials (fixed order), then the median as the mean of the order
// statistics (count - 1) / 2 and count / 2 of the valid (non-NaN) map values.  The errors are >= 0, so their float bit patterns
// are ordered: a radix select over 4 digits of 8 bits finds the lower one; the upper one is the same value unless the lower one
// was the last of its equals, and then it is the least value above it.
struct FeOut { long long* count; double* mean; double* median; double* fraction; };

__global__ void __launch_bounds__(kFeSelThreads) field_stats_kernel(FeArgs a, FeOut o) {
  __shared__ double shd[33];
  __shared__ int shi[33];
  __shared__ unsigned hist[256];
  __shared__ unsigned sel_bin, sel_eq, next_up;
  __shared__ long long sel_k;
  const int i = blockIdx.x, f = blockIdx.y;
  const FeImage d = a.im[i];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  double s = 0.0;
  for (int b = threadIdx.x; b < d.nblk; b += blockDim.x) s += a.psum[(long long)f * a.nblocks + d.block0 + b];
  s = block_sum(s, shd);
  long long cnt = 0;
  for (int k = 0; k <= a.T; ++k) {
    int c = 0;
    for (int b = threadIdx.x; b < d.nblk; b += blockDim.x) c += a.pcnt[((long long)f * (1 + a.T) + k) * a.nblocks + d.block0 + b];
    c = block_sum(c, shi);
    if (k == 0) cnt = c;
    else if (threadIdx.x == 0) o.fraction[((long long)f * a.n + i) * a.T + (k - 1)] = (double)c / (double)cnt;
  }
  const long long oi = (long long)f * a.n + i;
  if (threadIdx.x == 0) { o.count[oi] = cnt; o.mean[oi] = s / (double)cnt; }
  if (cnt == 0) {
    if (threadIdx.x == 0) o.median[oi] = NAN;
    return;
  }
  const float* map = (f == 0 ? a.map_up : a.map_lat) + d.map_off;
  const long long HW = (long long)d.H * d.W;
  const long long k1 = (cnt - 1) / 2, k2 = cnt / 2;
  unsigned prefix = 0, pmask = 0;
  long long k = k1;
  for (int shift = 24; shift >= 0; shift -= 8) {
    for (int b = threadIdx.x; b < 256; b += blockDim.x) hist[b] = 0;
    __syncthreads();
    // errors cluster in a few bins (the leading digit has a handful of values): lanes with the same bin add once, by their leader
    for (long long r0 = 0; r0 < HW; r0 += blockDim.x) {
      const long long r = r0 + threadIdx.x;
      unsigned key = 256u;
      if (r < HW) {
        const float e = map[r];
        const unsigned u = __float_as_uint(e);
        if (e == e && (u & pmask) == prefix) key = (u >> shift) & 255u;
      }
      const unsigned peers = __match_any_sync(0xffffffffu, key);
      if (key < 256u && __ffs(peers) - 1 == lane) atomicAdd(&hist[key], (unsigned)__popc(peers));
    }
    __syncthreads();
    if (warp == 0) {   // lane l owns bins 8l .. 8l + 7: scan the lanes' totals, the lane holding rank k resolves the bin
      unsigned c[8], tot = 0;
#pragma unroll
      for (int j = 0; j < 8; ++j) { c[j] = hist[8 * lane + j]; tot += c[j]; }
      unsigned inc = tot;
#pragma unroll
      for (int ofs = 1; ofs < 32; ofs <<= 1) {
        const unsigned t = __shfl_up_sync(0xffffffffu, inc, ofs);
        if (lane >= ofs) inc += t;
      }
      const long long exc = (long long)(inc - tot);
      if (exc <= k && k < (long long)inc) {
        long long rr = k - exc;
        int j = 0;
        while (rr >= (long long)c[j]) { rr -= c[j]; ++j; }
        sel_bin = 8 * lane + j; sel_k = rr; sel_eq = c[j];
      }
    }
    __syncthreads();
    prefix |= sel_bin << shift;
    pmask |= 255u << shift;
    k = sel_k;
    __syncthreads();
  }
  const float v1 = __uint_as_float(prefix);
  float v2 = v1;
  if (k2 != k1 && k + 1 >= (long long)sel_eq) {
    if (threadIdx.x == 0) next_up = 0xffffffffu;
    __syncthreads();
    unsigned best = 0xffffffffu;
    for (long long r = threadIdx.x; r < HW; r += blockDim.x) {
      const float e = map[r];
      const unsigned u = __float_as_uint(e);
      if (e == e && u > prefix && u < best) best = u;
    }
    atomicMin(&next_up, best);
    __syncthreads();
    v2 = __uint_as_float(next_up);
  }
  if (threadIdx.x == 0) o.median[oi] = ((double)v1 + (double)v2) * 0.5;
}

}  // namespace pf
