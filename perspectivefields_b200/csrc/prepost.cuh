// HBM-bound ends of the path: Pillow-exact uint8 resize + normalisation (pre) and resample-to-original (post).
#pragma once
#include <math.h>

#include <vector>

#include "common.cuh"

namespace pf {

// =====================================================================================================
// Pre-process.  Reference: perspectivefields.py:38-46 (PIL.Image.resize((320,320), BILINEAR) on uint8) and
// :234-236 ((x - pixel_mean) / pixel_std).  Pillow's resampler (src/libImaging/Resample.c, third-party) is an
// antialiased separable triangle filter with 22-bit fixed-point coefficients, horizontal pass first, each pass
// rounded to uint8.  The coefficient tables are built on the host in double precision exactly as Pillow's
// precompute_coeffs/normalize_coeffs_8bpc do; the kernel is pure integer arithmetic and therefore bit-exact.
constexpr int kPrecisionBits = 32 - 8 - 2;

struct ResampleTable {  // host-side, for one (in_size -> out_size) axis
  int in_size = 0, ksize = 0;
  std::vector<int> bounds;  // [out_size][2] = (xmin, count)
  std::vector<int> coeffs;  // [out_size][ksize]
};

inline ResampleTable make_resample_table(int in_size, int out_size) {
  ResampleTable t;
  t.in_size = in_size;
  const double scale = (double)in_size / (double)out_size;
  const double filterscale = scale < 1.0 ? 1.0 : scale;
  const double support = 1.0 * filterscale;  // bilinear (triangle) filter support = 1
  t.ksize = (int)ceil(support) * 2 + 1;
  t.bounds.assign((size_t)out_size * 2, 0);
  t.coeffs.assign((size_t)out_size * t.ksize, 0);
  std::vector<double> k((size_t)t.ksize);
  const double ss = 1.0 / filterscale;
  for (int xx = 0; xx < out_size; ++xx) {
    const double center = (xx + 0.5) * scale;
    int xmin = (int)(center - support + 0.5);
    if (xmin < 0) xmin = 0;
    int xmax = (int)(center + support + 0.5);
    if (xmax > in_size) xmax = in_size;
    const int n = xmax - xmin;
    double ww = 0.0;
    for (int x = 0; x < n; ++x) {
      double a = (x + xmin - center + 0.5) * ss;
      if (a < 0.0) a = -a;
      const double w = a < 1.0 ? 1.0 - a : 0.0;
      k[x] = w;
      ww += w;
    }
    for (int x = 0; x < n; ++x) {
      double v = k[x];
      if (ww != 0.0) v /= ww;
      t.coeffs[(size_t)xx * t.ksize + x] = v < 0 ? (int)(-0.5 + v * (1 << kPrecisionBits)) : (int)(0.5 + v * (1 << kPrecisionBits));
    }
    t.bounds[2 * xx] = xmin;
    t.bounds[2 * xx + 1] = n;
  }
  return t;
}

struct PreImage {          // per image, device-visible
  long long offset;        // byte offset of the HWC uint8 image in the input blob
  int H, W;
  int ksx, ksy;            // table widths
  const int* bx; const int* cx;   // horizontal tables (depend on W)
  const int* by; const int* cy;   // vertical tables   (depend on H)
};

constexpr int kPreRows = 8;        // output rows per block
constexpr int kPreMaxW = 640;      // widest working size (block = one thread per output column)
constexpr int kPreSmemBytes = 200 * 1024;   // budget of the horizontally resampled rows: 213 rows of 320 columns, 106 of 640

// grid = (OH / kPreRows, n_images), block = OW threads (one per output column); OH = net height, OW = net width.
// dyn smem = rows_needed * OW * 3 bytes for the horizontally resampled input rows of this tile.
// out: [n, OH, OW, 4] fp32 NHWC, channels (b, g, r, 0), value = (u8 - mean[c]) / std[c].
__global__ void __launch_bounds__(kPreMaxW) preprocess_kernel(const unsigned char* __restrict__ blob, const PreImage* __restrict__ imgs, float* __restrict__ out,
                                                              float m0, float m1, float m2, float s0, float s1, float s2, int max_rows, int OH, int OW) {
  extern __shared__ unsigned char s_h[];  // [rows][OW][3]
  const PreImage im = imgs[blockIdx.y];
  const int oy0 = blockIdx.x * kPreRows;
  const int x = threadIdx.x;
  const unsigned char* src = blob + im.offset;
  const int xmin = im.bx[2 * x], xn = im.bx[2 * x + 1];
  const int* kx = im.cx + (long long)x * im.ksx;
  for (int r0 = 0; r0 < kPreRows;) {
    // process as many output rows as fit in smem (normally all kPreRows at once)
    int rcount = 0;
    const int in_first = im.by[2 * (oy0 + r0)];
    int in_last = in_first;
    while (r0 + rcount < kPreRows) {
      const int o = oy0 + r0 + rcount;
      const int last = im.by[2 * o] + im.by[2 * o + 1];
      if (last - in_first > max_rows && rcount > 0) break;
      in_last = last;
      ++rcount;
    }
    const int nrows = in_last - in_first;
    // horizontal pass: input rows [in_first, in_last) -> uint8 [nrows][OW][3]
    for (int r = 0; r < nrows; ++r) {
      const unsigned char* row = src + ((long long)(in_first + r) * im.W + xmin) * 3;
      int a0 = 1 << (kPrecisionBits - 1), a1 = a0, a2 = a0;
      for (int t = 0; t < xn; ++t) {
        const int k = kx[t];
        a0 += row[3 * t] * k; a1 += row[3 * t + 1] * k; a2 += row[3 * t + 2] * k;
      }
      unsigned char* d = s_h + (r * OW + x) * 3;
      d[0] = (unsigned char)min(max(a0 >> kPrecisionBits, 0), 255);
      d[1] = (unsigned char)min(max(a1 >> kPrecisionBits, 0), 255);
      d[2] = (unsigned char)min(max(a2 >> kPrecisionBits, 0), 255);
    }
    __syncthreads();
    // vertical pass
    for (int rr = 0; rr < rcount; ++rr) {
      const int o = oy0 + r0 + rr;
      const int ymin = im.by[2 * o] - in_first, yn = im.by[2 * o + 1];
      const int* ky = im.cy + (long long)o * im.ksy;
      int a0 = 1 << (kPrecisionBits - 1), a1 = a0, a2 = a0;
      for (int t = 0; t < yn; ++t) {
        const int k = ky[t];
        const unsigned char* d = s_h + ((ymin + t) * OW + x) * 3;
        a0 += d[0] * k; a1 += d[1] * k; a2 += d[2] * k;
      }
      const float v0 = (float)min(max(a0 >> kPrecisionBits, 0), 255);
      const float v1 = (float)min(max(a1 >> kPrecisionBits, 0), 255);
      const float v2 = (float)min(max(a2 >> kPrecisionBits, 0), 255);
      reinterpret_cast<float4*>(out)[((long long)blockIdx.y * OH + o) * OW + x] =
          make_float4((v0 - m0) / s0, (v1 - m1) / s1, (v2 - m2) / s2, 0.f);
    }
    __syncthreads();
    r0 += rcount;
  }
}

// Lower entry (perspectivefields.py:223-236 called directly): images already resized, fp32 CHW [n,3,H,W] (the net size).
__global__ void __launch_bounds__(256) normalize_chw_kernel(const float* __restrict__ in, float* __restrict__ out, int n, int H, int W,
                                                            float m0, float m1, float m2, float s0, float s1, float s2) {
  const long long HW = (long long)H * W, total = (long long)n * HW;
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const long long b = i / HW, p = i % HW;
  const float* s = in + b * 3 * HW + p;
  reinterpret_cast<float4*>(out)[i] = make_float4((s[0] - m0) / s0, (s[HW] - m1) / s1, (s[2 * HW] - m2) / s2, 0.f);
}

// =====================================================================================================
// Post-process.  Reference: gravity_head.py:237-261, latitude_head.py:195-219, utils/utils.py:483-507.
// The fields arrive at the net size SH x SW (DATALOADER.RESIZE, the heads' image_size; 320 x 320 in every shipped config):
//   gravity : vec * (W/SW, H/SH) -> bilinear (align_corners=False, no antialias) to (H, W) -> F.normalize(dim=0)
//   latitude: bilinear to (H, W) -> asin -> rad2deg          (regression)   |  bilinear of decoded degrees (classification)
// ATen upsample_bilinear2d: scale = (float)SH / out; src = scale*(dst+0.5)-0.5, clamped at 0; i1 = i0 + (i0 < SH - 1).
struct PostImage {
  int H, W;
  long long g_off;  // float offset of this image's [2,H,W] block in the gravity_original blob
  long long l_off;  // float offset of this image's [H,W] block in the latitude_original blob
  long long pix0;   // first global output-pixel index of this image (prefix sum of H*W)
};

// asin for |x| <= 1, branch-free (Cephes-style): |x| <= 1/2: x + x z P(z), z = x^2; else pi/2 - 2 (s + s z P(z)), z = (1 - |x|)/2,
// s = sqrt z.  Max error 1.7e-7 rad against float64 asin over 4e6 samples incl. the end points (tests/test_host_logic.py repeats
// the check on these coefficients); libm's asinf costs ~3x the instructions and made this kernel instruction-bound.
__device__ __forceinline__ float fast_asinf(float x) {
  const float a = fabsf(x);
  const bool big = a > 0.5f;
  const float z = big ? (1.0f - a) * 0.5f : a * a;
  const float s = big ? z * rsqrtf(fmaxf(z, 1e-30f)) : a;       // sqrt z (z = 0 at |x| = 1 stays 0); rsqrt.approx: 2^-22 relative
  float p = 4.2163199048e-2f;
  p = fmaf(p, z, 2.4181311049e-2f);
  p = fmaf(p, z, 4.5470025998e-2f);
  p = fmaf(p, z, 7.4953002686e-2f);
  p = fmaf(p, z, 1.6666752422e-1f);
  float r = fmaf(s * z, p, s);
  r = big ? 1.5707963267948966f - (r + r) : r;
  return copysignf(r, x);
}

// Block = (band of kPostBand output rows, image).  Per group of kPostRows output rows the block first interpolates VERTICALLY:
// for each of the SW source columns it stores (gravity x * W/320, gravity y * H/320, latitude) blended between the two source
// rows as ONE float4 in shared memory; then every thread produces 4 consecutive output pixels of one row from two 16-byte
// shared-memory taps per pixel (per-column index / weight tables, built once per block), normalises the up-vector
// (v * rsqrt(max(|v|^2, 1e-24)) == v / max(|v|, 1e-12)), applies asin + rad2deg and writes three 16-byte streaming stores.
// A straightforward version needs ~160 instructions per pixel and is instruction-bound; this one needs ~45 and is bound by
// its 12 B/pixel of stores.
// The interpolation is evaluated as hx * (hy v00 + ly v10) + lx * (hy v01 + ly v11): ATen's bilinear kernel nests the two axes the
// other way round (same weights, same products; the results differ by fp32 rounding only, ~1e-7 relative).
constexpr int kPostRows = 4, kPostBand = 16, kPostThreads = 256, kPostMaxW = 3072;
// dynamic shared memory: the source-row buffer (kPostRows x (SW + 1) float4; 20.6 KB at SW = 320) + 8 B per output column
inline int post_smem_bytes(int SW, int max_wp) { return kPostRows * (SW + 1) * 16 + max_wp * 8; }
constexpr int kPostSmemMax = kPostRows * (kPreMaxW + 1) * 16 + kPostMaxW * 8;   // 65600 B
__global__ void __launch_bounds__(kPostThreads) postprocess_kernel(const float* __restrict__ vec, const float* __restrict__ lat, const PostImage* __restrict__ imgs,
                                                                   float* __restrict__ g_out, float* __restrict__ l_out, int lat_is_sin, int SH, int SW) {
  extern __shared__ __align__(16) unsigned char s_dyn[];
  float4* s_v = reinterpret_cast<float4*>(s_dyn);    // [kPostRows][SW + 1] vertically interpolated source rows (+1: tap xa + 1 of the last column)
  const int SW1 = SW + 1;
  const PostImage im = imgs[blockIdx.y];
  const int band0 = blockIdx.x * kPostBand;
  if (band0 >= im.H) return;
  const int W4 = (im.W + 3) >> 2, Wp = W4 * 4;
  int* s_xa = reinterpret_cast<int*>(s_v + kPostRows * SW1);   // per output column: int xa, float lx  (W entries each, W padded to 4)
  float* s_lx = reinterpret_cast<float*>(s_xa) + Wp;
  const int tid = threadIdx.x;
  const float sch = (float)SH / (float)im.H, scw = (float)SW / (float)im.W;
  const bool tab = Wp <= kPostMaxW;       // wider images: indices / weights are recomputed per pixel instead
  for (int x = tid; tab && x < Wp; x += kPostThreads) {
    const int xc = min(x, im.W - 1);
    const float sx = fmaxf(scw * ((float)xc + 0.5f) - 0.5f, 0.f);
    const int xa = min((int)sx, SW - 1);
    s_xa[x] = xa;
    s_lx[x] = sx - (float)xa;
  }
  const long long SHW = (long long)SH * SW;
  const float* v0 = vec + (long long)blockIdx.y * 2 * SHW;
  const float* v1 = v0 + SHW;
  const float* lp = lat + (long long)blockIdx.y * SHW;
  // the reference scales the field before resampling: vec * [[W/SW],[H/SH]] (float32 tensor built from python doubles)
  const float fx = (float)((double)im.W / (double)SW), fy = (float)((double)im.H / (double)SH);
  const long long HW = (long long)im.H * im.W;
  const bool vec_ok = (im.W & 3) == 0 && (im.g_off & 3) == 0 && ((im.g_off + HW) & 3) == 0 && (im.l_off & 3) == 0;
  const int band1 = min(band0 + kPostBand, im.H);
  // work items of one row group: (row rr, column group g), rr-major; thread `tid` starts at item tid and advances by 256
  const int g_start = tid % W4, r_start = tid / W4, g_step = kPostThreads % W4, r_step = kPostThreads / W4;
  for (int r0 = band0; r0 < band1; r0 += kPostRows) {
    __syncthreads();     // (the previous group's readers are done; the column tables are complete)
    for (int i = tid; i < kPostRows * SW; i += kPostThreads) {
      const int rr = i / SW, x = i - rr * SW;
      const int y = min(r0 + rr, im.H - 1);
      const float sy = fmaxf(sch * ((float)y + 0.5f) - 0.5f, 0.f);
      const int y0 = min((int)sy, SH - 1);
      const int y1 = y0 + (y0 < SH - 1);
      const float ly = sy - (float)y0, hy = 1.f - ly;
      const int i0 = y0 * SW + x, i1 = y1 * SW + x;
      const float4 t = make_float4(hy * (__ldg(v0 + i0) * fx) + ly * (__ldg(v0 + i1) * fx), hy * (__ldg(v1 + i0) * fy) + ly * (__ldg(v1 + i1) * fy),
                                   hy * __ldg(lp + i0) + ly * __ldg(lp + i1), 0.f);
      s_v[rr * SW1 + x] = t;
      if (x == SW - 1) s_v[rr * SW1 + SW] = t;      // tap xa + 1 of the last column (its weight lx is 0 there)
    }
    __syncthreads();
    const int rows = min(kPostRows, band1 - r0);
    for (int rr = r_start, g = g_start; rr < rows;) {
      const int x0 = g * 4;
      int xa[4];
      float lx[4];
      if (tab) {
        const int4 xa4 = *reinterpret_cast<const int4*>(s_xa + x0);
        const float4 lx4 = *reinterpret_cast<const float4*>(s_lx + x0);
        xa[0] = xa4.x; xa[1] = xa4.y; xa[2] = xa4.z; xa[3] = xa4.w;
        lx[0] = lx4.x; lx[1] = lx4.y; lx[2] = lx4.z; lx[3] = lx4.w;
      } else {
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const float sx = fmaxf(scw * ((float)min(x0 + j, im.W - 1) + 0.5f) - 0.5f, 0.f);
          xa[j] = min((int)sx, SW - 1);
          lx[j] = sx - (float)xa[j];
        }
      }
      float ogx[4], ogy[4], ol[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float4 a = s_v[rr * SW1 + xa[j]], b = s_v[rr * SW1 + xa[j] + 1];
        const float hx = 1.f - lx[j];
        const float gx = hx * a.x + lx[j] * b.x;
        const float gy = hx * a.y + lx[j] * b.y;
        float lv = hx * a.z + lx[j] * b.z;
        const float inv = rsqrtf(fmaxf(fmaf(gx, gx, gy * gy), 1e-24f));     // F.normalize: v / max(|v|, 1e-12)
        ogx[j] = gx * inv; ogy[j] = gy * inv;
        if (lat_is_sin) lv = fast_asinf(lv) * (180.0f / 3.14159265358979323846f);
        ol[j] = lv;
      }
      const long long p = (long long)(r0 + rr) * im.W + x0;
      float* gp = g_out + im.g_off + p;
      float* lpo = l_out + im.l_off + p;
      if (vec_ok) {
        __stcs(reinterpret_cast<float4*>(gp), make_float4(ogx[0], ogx[1], ogx[2], ogx[3]));
        __stcs(reinterpret_cast<float4*>(gp + HW), make_float4(ogy[0], ogy[1], ogy[2], ogy[3]));
        __stcs(reinterpret_cast<float4*>(lpo), make_float4(ol[0], ol[1], ol[2], ol[3]));
      } else {
        for (int j = 0; j < 4 && x0 + j < im.W; ++j) { gp[j] = ogx[j]; gp[HW + j] = ogy[j]; lpo[j] = ol[j]; }
      }
      g += g_step; rr += r_step;
      if (g >= W4) { g -= W4; ++rr; }
    }
  }
}

// =====================================================================================================
// Camera parameters -> dense perspective fields (SURVEY.md 8f-1): PanoCam.get_up_general / get_lat_general
// (utils/panocam.py:451-556), what callers evaluate right after the inference path (utils/utils.py:367-385).
// One thread per pixel, float64 arithmetic like the numpy reference, float32 results; the kernel is bound by its stores.
//   up  [H, W, 2] (x, y): unit vector from the pixel centre (j + .5, i + .5) to the vertical vanishing point, flipped by
//                sign(elevation); the constant (-sin roll, -cos roll) when elevation == 0 exactly (:488)
//   lat [H, W] degrees: ray ((dx, dy, f) / f) rotated by roll, then elevation; -atan2(y_w, hypot(x_w, z_w)); dx / dy sample
//                linspace(-cx, W - cx, W) INCLUDING both end points (:534-539: spacing W / (W - 1), not pixel centres)
struct CamImage {
  int H, W;
  double f, cx, cy;           // focal length in pixels, principal point in pixels
  double sr, cr, se, ce;      // sin / cos of roll and elevation (computed on the host in float64)
  double sgn;                 // sign(elevation): +1, -1 or 0 (0 selects the constant field)
  int vp;                     // 1: the up field points to (vpx, vpy) instead (PanoCam.get_up's far point at elevation 0)
  double vpx, vpy;
  long long up_off, lat_off;  // float offsets of this image's blocks in the output blobs
};
constexpr int kCamChunk = 24;   // images per launch (the descriptors travel as a kernel parameter)
struct CamBatch { CamImage im[kCamChunk]; };

// atan2(y, h) in DEGREES for h >= 0 (Cephes-style atanf: three ranges, odd polynomial on |r| <= tan(pi/8)); the range offset is
// added by the same fma that converts to degrees, so the result is rounded once.  Max error 7.2e-6 degrees incl. that final
// rounding (ulp(90)/2 = 3.8e-6), checked against float64 atan2 in tests/test_host_logic.py.
__device__ __forceinline__ float fast_atan2_deg(float y, float h) {
  const float a = fabsf(y);
  const bool hi = a > 2.414213562373095f * h, mid = !hi && a > 0.4142135623730950f * h;
  const float num = hi ? -h : (mid ? a - h : a), den = hi ? a : (mid ? a + h : h);
  const float r = num / den;
  const float z = r * r;
  float p = 8.05374449538e-2f;
  p = fmaf(p, z, -1.38776856032e-1f);
  p = fmaf(p, z, 1.99777106478e-1f);
  p = fmaf(p, z, -3.33329491539e-1f);
  const float pr = fmaf(r * z, p, r);
  const float off = hi ? 90.0f : (mid ? 45.0f : 0.0f);              // exact in float32
  const float deg = fmaf(pr, 57.29577951308232f, off);             // one rounding (the constant's own error: 1e-8 relative)
  return copysignf(deg, y);
}

// One thread = 4 consecutive pixels of one row.  The pixel -> ray map is linear: its three world components are evaluated in
// float64 for the thread's FIRST pixel (x_j = linspace sample: 1e-16 relative, like the numpy reference), rounded to float32
// and advanced by float32 steps for the other three (the steps are ~1/f: their rounding is 1e-10 absolute); square root,
// division and arctangent are float32 (fast_atan2_deg): float64 square roots, divisions and arctangents per pixel would make
// the kernel bound by conversions and special-function operations instead of its stores.
__global__ void __launch_bounds__(256) camera_fields_kernel(const __grid_constant__ CamBatch batch, float* __restrict__ up, float* __restrict__ lat) {
  const CamImage& c = batch.im[blockIdx.y];
  const int W4 = (c.W + 3) >> 2;
  const long long q = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= (long long)c.H * W4) return;
  const int i = (int)(q / W4), j0 = (int)(q - (long long)i * W4) * 4;
  const long long p0 = (long long)i * c.W + j0;
  const int nj = min(4, c.W - j0);
  if (up) {
    float o[8];
    if (c.sgn == 0.0) {
#pragma unroll
      for (int k = 0; k < 4; ++k) { o[2 * k] = (float)(-c.sr); o[2 * k + 1] = (float)(-c.cr); }
    } else {
      const double vvp_x = c.vp ? c.vpx : (c.sr * c.ce * c.f) / -c.se + c.cx, vvp_y = c.vp ? c.vpy : (c.cr * c.ce * c.f) / -c.se + c.cy;
      const float vy = (float)((vvp_y - ((double)i + 0.5)) * c.sgn);
      const float vx0 = (float)((vvp_x - ((double)j0 + 0.5)) * c.sgn), dvx = (float)(-c.sgn);    // pixel k: vx0 + k * dvx
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const float vx = fmaf((float)k, dvx, vx0);
        const float inv = rsqrtf(fmaf(vx, vx, vy * vy));
        o[2 * k] = vx * inv; o[2 * k + 1] = vy * inv;
      }
    }
    float* dst = up + c.up_off + 2 * p0;
    if (nj == 4 && ((c.up_off + 2 * p0) & 3) == 0) {
      __stcs(reinterpret_cast<float4*>(dst), make_float4(o[0], o[1], o[2], o[3]));
      __stcs(reinterpret_cast<float4*>(dst) + 1, make_float4(o[4], o[5], o[6], o[7]));
    } else {
      for (int k = 0; k < nj; ++k) *reinterpret_cast<float2*>(dst + 2 * k) = make_float2(o[2 * k], o[2 * k + 1]);
    }
  }
  if (lat) {
    // numpy.linspace(start, stop, num): start + k * ((stop - start) / (num - 1)), last sample = stop exactly
    const double x0 = (-c.W / 2.0) - (c.cx - (c.W / 2.0)), x1 = (c.W / 2.0) - (c.cx - (c.W / 2.0));
    const double y0 = (-c.H / 2.0) - (c.cy - (c.H / 2.0)), y1 = (c.H / 2.0) - (c.cy - (c.H / 2.0));
    const double sx = c.W == 1 ? 0.0 : (x1 - x0) / (double)(c.W - 1);
    const double dy = c.H == 1 ? y0 : (i == c.H - 1 ? y1 : (double)i * ((y1 - y0) / (double)(c.H - 1)) + y0);
    const double y = dy / c.f, rf = 1.0 / c.f;
    // world ray = R_elevation R_roll (x, y, 1):  xw = x cr - y sr;  yw = x ce sr + y ce cr - se;  zw = x se sr + y se cr + ce
    const double bx = -y * c.sr, by = y * c.ce * c.cr - c.se, bz = y * c.se * c.cr + c.ce;
    const double ax = c.cr, ay = c.ce * c.sr, az = c.se * c.sr;
    float o[4];
    if (j0 + 4 >= c.W) {
      // the thread that holds the row's last pixel (linspace's exact end point): float64 per pixel
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const int j = min(j0 + k, c.W - 1);
        const double dx = j == c.W - 1 ? (c.W == 1 ? x0 : x1) : fma((double)j, sx, x0);
        const double x = dx * rf;
        const float xw = (float)fma(x, ax, bx), yw = (float)fma(x, ay, by), zw = (float)fma(x, az, bz);
        o[k] = -fast_atan2_deg(yw, sqrtf(fmaf(xw, xw, zw * zw)));
      }
    } else {
      const double x = fma((double)j0, sx, x0) * rf, xs = sx * rf;          // first pixel and the step between pixels
      const float xw0 = (float)fma(x, ax, bx), yw0 = (float)fma(x, ay, by), zw0 = (float)fma(x, az, bz);
      const float dxw = (float)(xs * ax), dyw = (float)(xs * ay), dzw = (float)(xs * az);
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const float xw = fmaf((float)k, dxw, xw0), yw = fmaf((float)k, dyw, yw0), zw = fmaf((float)k, dzw, zw0);
        o[k] = -fast_atan2_deg(yw, sqrtf(fmaf(xw, xw, zw * zw)));
      }
    }
    float* dst = lat + c.lat_off + p0;
    if (nj == 4 && ((c.lat_off + p0) & 3) == 0) __stcs(reinterpret_cast<float4*>(dst), make_float4(o[0], o[1], o[2], o[3]));
    else for (int k = 0; k < nj; ++k) dst[k] = o[k];
  }
}

// =====================================================================================================
// ResizeTransform.apply_image as a stand-alone device transform (perspectivefields.py:34-67; `model.aug.apply_image`).
//   uint8: Pillow's two-pass antialiased triangle filter, integer arithmetic, bit-exact (same tables / rounding as
//          preprocess_kernel, arbitrary target size): horizontal pass [H,W,3] -> [H,new_w,3], vertical pass -> [new_h,new_w,3].
__global__ void __launch_bounds__(256) resize_u8_h_kernel(const unsigned char* __restrict__ src, int H, int W, int OW, const int* __restrict__ bounds,
                                                          const int* __restrict__ coeffs, int ks, unsigned char* __restrict__ dst) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)H * OW) return;
  const int y = (int)(i / OW), x = (int)(i - (long long)y * OW);
  const int xmin = bounds[2 * x], xn = bounds[2 * x + 1];
  const int* k = coeffs + (long long)x * ks;
  const unsigned char* row = src + ((long long)y * W + xmin) * 3;
  int a0 = 1 << (kPrecisionBits - 1), a1 = a0, a2 = a0;
  for (int t = 0; t < xn; ++t) { const int kk = k[t]; a0 += row[3 * t] * kk; a1 += row[3 * t + 1] * kk; a2 += row[3 * t + 2] * kk; }
  unsigned char* d = dst + i * 3;
  d[0] = (unsigned char)min(max(a0 >> kPrecisionBits, 0), 255);
  d[1] = (unsigned char)min(max(a1 >> kPrecisionBits, 0), 255);
  d[2] = (unsigned char)min(max(a2 >> kPrecisionBits, 0), 255);
}
__global__ void __launch_bounds__(256) resize_u8_v_kernel(const unsigned char* __restrict__ src, int H, int OW, int OH, const int* __restrict__ bounds,
                                                          const int* __restrict__ coeffs, int ks, unsigned char* __restrict__ dst) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)OH * OW) return;
  const int y = (int)(i / OW), x = (int)(i - (long long)y * OW);
  const int ymin = bounds[2 * y], yn = bounds[2 * y + 1];
  const int* k = coeffs + (long long)y * ks;
  int a0 = 1 << (kPrecisionBits - 1), a1 = a0, a2 = a0;
  for (int t = 0; t < yn; ++t) {
    const int kk = k[t];
    const unsigned char* s = src + ((long long)(ymin + t) * OW + x) * 3;
    a0 += s[0] * kk; a1 += s[1] * kk; a2 += s[2] * kk;
  }
  unsigned char* d = dst + i * 3;
  d[0] = (unsigned char)min(max(a0 >> kPrecisionBits, 0), 255);
  d[1] = (unsigned char)min(max(a1 >> kPrecisionBits, 0), 255);
  d[2] = (unsigned char)min(max(a2 >> kPrecisionBits, 0), 255);
  (void)H;
}
//   float32: F.interpolate(mode="bilinear", align_corners=False) without antialias (ATen upsample_bilinear2d: scale = in / out,
//          src = scale * (dst + 0.5) - 0.5 clamped at 0, i1 = i0 + (i0 < in - 1)); HWC with C channels.  Also the cv2.resize
//          (INTER_LINEAR) of the visualisation hand-off (demo/demo.py:41-51), which uses the same sampling positions.
__global__ void __launch_bounds__(256) resize_f32_kernel(const float* __restrict__ src, int H, int W, int C, int OH, int OW, float* __restrict__ dst) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)OH * OW * C) return;
  const int c = (int)(i % C);
  const long long pix = i / C;
  const int x = (int)(pix % OW), y = (int)(pix / OW);
  const float sch = (float)H / (float)OH, scw = (float)W / (float)OW;
  const float sy = fmaxf(sch * ((float)y + 0.5f) - 0.5f, 0.f), sx = fmaxf(scw * ((float)x + 0.5f) - 0.5f, 0.f);
  const int y0 = min((int)sy, H - 1), x0 = min((int)sx, W - 1);
  const int y1 = y0 + (y0 < H - 1), x1 = x0 + (x0 < W - 1);
  const float ly = sy - (float)y0, lx = sx - (float)x0, hy = 1.f - ly, hx = 1.f - lx;
  const float v00 = __ldg(src + ((long long)y0 * W + x0) * C + c), v01 = __ldg(src + ((long long)y0 * W + x1) * C + c);
  const float v10 = __ldg(src + ((long long)y1 * W + x0) * C + c), v11 = __ldg(src + ((long long)y1 * W + x1) * C + c);
  dst[i] = hy * (hx * v00 + lx * v01) + ly * (hx * v10 + lx * v11);
}

// Write-only bandwidth probe (bench.py: the roofline of the store-bound write-out kernels): 16-byte streaming stores, grid-stride.
__global__ void __launch_bounds__(256) fill_stream_kernel(float4* __restrict__ dst, long long n4, float v) {
  const float4 val = make_float4(v, v, v, v);
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) __stcs(dst + i, val);
}

}  // namespace pf
