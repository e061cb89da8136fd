// Upright warp: straighten images from their camera parameters (this project's rule, DESIGN.md section 1 "Upright warp";
// restated on the CPU in tests/oracle_rectify.py).
//
// Input camera per image: roll r, pitch e, f_rel (from the general vfov and principal point, general_vfov_to_focal's closed
// form), cx_rel, cy_rel; F = f_rel H, cx = (cx_rel + 1/2) W, cy = (cy_rel + 1/2) H, ray c = ((x - cx) / F, (y - cy) / F, 1) at
// pixel-centre coordinates (pixel (i, j) at (j + 1/2, i + 1/2)), world ray R_x(e) R_z(r) c (get_lat_general's rotation order).
// Output camera: roll 0, pitch e_o (0, or e with keep_pitch), centred principal point, size H_o x W_o, focal F_o ("same" f_rel H_o,
// a vfov, or "fill": the smallest F_o >= f_rel H_o that keeps the canvas corners inside the input).  An output pixel centre x'
// maps to the input homogeneous point M x' with M = K R_z(-r) R_x(e_o - e) K_o^-1, valid iff its z > 0 and it lies in
// [0, W] x [0, H].
//
// Two kernels, chained with programmatic dependent launch and enqueued without synchronisation: rectify_setup_kernel (one thread
// per image: parameters from device memory -> status, output camera, M) and rectify_warp_kernel (every output pixel of every image,
// grid.y = image).  "fill_common" (one zoom for the whole call: the largest "fill" F_o / H_o of the usable images, times each H_o)
// replaces the setup by rectify_setup_common_kernel, one block that reduces the zoom and then writes every image's setup.
#pragma once
#include <math.h>
#include <stdint.h>

#include "common.cuh"

namespace pf {

constexpr int kRectFocalSame = 0, kRectFocalVfov = 1, kRectFocalFill = 2;
constexpr int kRectCommonThreads = 256;
constexpr int kRectThreads = 256, kRectPix = 4;   // 4 consecutive output pixels (of the image's flat H_o * W_o range) per thread
constexpr double kRectPi = 3.14159265358979323846;

struct RectImage {
  int H, W, Ho, Wo;
  long long in_off, out_off;   // bytes of the [H, W, C] input / [H_o, W_o, C] output
  long long mask_off;          // bytes of the uint8 [H_o, W_o] mask, -1: none
  long long map_off;           // floats of the float32 [H_o, W_o, 2] map, -1: none
};
struct RectMap {
  double m[9];                 // row-major: input (X, Y, Z) = M (x', y', 1) at output pixel-centre coordinates
  int ok;                      // 0: status 2, every sample invalid
};
struct RectArgs {
  const RectImage* im; RectMap* map; int n;
  const double* params;        // [n][5] roll, pitch, general vfov (degrees), cx_rel, cy_rel
  double* camera;              // [n][5] the output camera in the same form
  int* status;
  int keep_pitch, focal_mode;
  double vfov;                 // degrees, focal_mode kRectFocalVfov
  const unsigned char* in; unsigned char* out; unsigned char* mask; float* xy;
  unsigned char fill[3];
};

// general_vfov_to_focal (panocam.py, DESIGN.md section 4) at h = 1: with c = cos(gvfov), A = f^2 + cx^2 + cy^2 + 1/4,
// 4 (c^2 - 1) A^2 + 4 A - (1 + 4 c^2 cy^2) = 0, the root with sign(2A - 1) = sign(c)
__device__ __forceinline__ double rect_focal_rel(double cx, double cy, double gvfov_rad) {
  const double c = cos(gvfov_rad);
  const double a2 = 4.0 * (c * c - 1.0), a1 = 4.0, a0 = -(1.0 + 4.0 * c * c * cy * cy);
  const double disc = sqrt(fmax(a1 * a1 - 4.0 * a2 * a0, 0.0));
  double A;
  if (fabs(a2) < 1e-300) {
    A = -a0 / a1;
  } else {
    const double r1 = (-a1 + disc) / (2.0 * a2), r2 = (-a1 - disc) / (2.0 * a2);
    const double s1 = 2.0 * r1 - 1.0;
    const double sg1 = (s1 > 0.0) - (s1 < 0.0), sgc = (c > 0.0) - (c < 0.0);
    A = sg1 == sgc ? r1 : r2;
  }
  return sqrt(A - cx * cx - cy * cy - 0.25);
}

// ------------------------------------------------------------------------------------------------------------ setup
// Image i's setup.  kFillZoom: return its "fill" F_o / H_o (0 when its parameters are unusable) and write nothing.  kCommon: write it
// at F_o = fo_rel H_o, with the status of its own "fill" focal length.  Neither: the focal mode's F_o.
template <bool kFillZoom = false, bool kCommon = false>
__device__ __forceinline__ double rect_setup_image(const RectArgs& a, int i, double fo_rel = 0.0) {
  const RectImage d = a.im[i];
  const double* p = a.params + 5LL * i;
  const double roll = p[0], pitch = p[1], gv = p[2], cxr = p[3], cyr = p[4];
  const double d2r = kRectPi / 180.0, r2d = 180.0 / kRectPi;
  double f = NAN;
  bool ok = isfinite(roll) && isfinite(pitch) && isfinite(gv) && isfinite(cxr) && isfinite(cyr) && gv > 0.0 && gv < 180.0;
  if (ok) f = rect_focal_rel(cxr, cyr, gv * d2r);
  ok = ok && isfinite(f) && f > 0.0;
  RectMap& mp = a.map[i];
  double* cam = a.camera + 5LL * i;
  if (!ok) {
    if constexpr (kFillZoom) return 0.0;
    for (int k = 0; k < 9; ++k) mp.m[k] = NAN;
    mp.ok = 0;
    for (int k = 0; k < 5; ++k) cam[k] = NAN;
    a.status[i] = 2;
    return 0.0;
  }
  const double H = d.H, W = d.W, Ho = d.Ho, Wo = d.Wo;
  const double F = f * H, cx = (cxr + 0.5) * W, cy = (cyr + 0.5) * H;
  const double r = roll * d2r, e = pitch * d2r, eo = a.keep_pitch ? e : 0.0;
  double sr, cr, sd, cd;
  sincos(r, &sr, &cr);
  sincos(eo - e, &sd, &cd);
  // R = R_z(-r) R_x(eo - e);  R_z(-r) = [[cr, sr, 0], [-sr, cr, 0], [0, 0, 1]],  R_x(d) = [[1, 0, 0], [0, cd, -sd], [0, sd, cd]]
  const double R[9] = {cr, sr * cd, -sr * sd,
                       -sr, cr * cd, -cr * sd,
                       0.0, sd, cd};
  const double Fs = f * Ho;
  double Fo = Fs;
  int status = 0;
  if (a.focal_mode == kRectFocalVfov && !kFillZoom && !kCommon) {
    Fo = Ho / (2.0 * tan(a.vfov * d2r / 2.0));
  } else if (a.focal_mode == kRectFocalFill || kFillZoom || kCommon) {
    // the input rectangle as four half-spaces n_k . c >= 0 of input rays; a canvas corner (a, b) relative to the centre has the
    // ray p + t q with p = R (0, 0, 1), q = R (a, b, 0), t = 1 / F_o
    const double nrm[4][3] = {{F, 0.0, cx}, {-F, 0.0, W - cx}, {0.0, F, cy}, {0.0, -F, H - cy}};
    const double px = R[2], py = R[5], pz = R[8];
    bool inside = true;
    double tmax = INFINITY;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const double np = nrm[k][0] * px + nrm[k][1] * py + nrm[k][2] * pz;
      inside = inside && np > 0.0;
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const double ca = (q & 1) ? Wo / 2.0 : -Wo / 2.0, cb = (q & 2) ? Ho / 2.0 : -Ho / 2.0;
        const double qx = R[0] * ca + R[1] * cb, qy = R[3] * ca + R[4] * cb, qz = R[6] * ca + R[7] * cb;
        const double nq = nrm[k][0] * qx + nrm[k][1] * qy + nrm[k][2] * qz;
        if (nq < 0.0) tmax = fmin(tmax, np / -nq);
      }
    }
    if (!inside) status = 1;
    else if (tmax < INFINITY) Fo = fmax(Fs, 1.0 / tmax);
  }
  if constexpr (kFillZoom) return Fo / Ho;
  if constexpr (kCommon) Fo = fo_rel * Ho;
  // M = K R K_o^-1 with K = [[F, 0, cx], [0, F, cy], [0, 0, 1]], K_o^-1 = [[1/Fo, 0, -Wo/(2Fo)], [0, 1/Fo, -Ho/(2Fo)], [0, 0, 1]]
  double KR[9];
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    KR[c] = F * R[c] + cx * R[6 + c];
    KR[3 + c] = F * R[3 + c] + cy * R[6 + c];
    KR[6 + c] = R[6 + c];
  }
  const double iF = 1.0 / Fo, ox = -(Wo / 2.0) / Fo, oy = -(Ho / 2.0) / Fo;
#pragma unroll
  for (int rr = 0; rr < 3; ++rr) {
    mp.m[3 * rr + 0] = KR[3 * rr + 0] * iF;
    mp.m[3 * rr + 1] = KR[3 * rr + 1] * iF;
    mp.m[3 * rr + 2] = KR[3 * rr + 0] * ox + KR[3 * rr + 1] * oy + KR[3 * rr + 2];
  }
  mp.ok = 1;
  cam[0] = 0.0;
  cam[1] = eo * r2d;
  cam[2] = 2.0 * atan(Ho / (2.0 * Fo)) * r2d;
  cam[3] = 0.0;
  cam[4] = 0.0;
  a.status[i] = status;
  return Fo / Ho;
}

// One thread per image: "same", a vfov, or "fill"
__global__ void __launch_bounds__(128) rectify_setup_kernel(RectArgs a) {
  pdl_wait();      // params may come from the previous kernel on the stream (e.g. the camera fit)
  pdl_launch();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= a.n) return;
  rect_setup_image(a, i);
}

// "fill_common", one block for the whole call: f_o = the largest "fill" F_o / H_o of the usable images (a maximum: the same bits
// in any order), then every image written at F_o = f_o H_o with its own "fill" status.  A larger focal length keeps a filled
// canvas filled, since every corner constraint has the form t <= bound.
__global__ void __launch_bounds__(kRectCommonThreads) rectify_setup_common_kernel(RectArgs a) {
  __shared__ double shm[kRectCommonThreads / 32];
  pdl_wait();
  pdl_launch();
  double fo = 0.0;
  for (int i = threadIdx.x; i < a.n; i += blockDim.x) fo = fmax(fo, rect_setup_image<true>(a, i));
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) fo = fmax(fo, __shfl_xor_sync(0xffffffffu, fo, o));
  if ((threadIdx.x & 31) == 0) shm[threadIdx.x >> 5] = fo;
  __syncthreads();
  for (int w = 0; w < kRectCommonThreads / 32; ++w) fo = fmax(fo, shm[w]);
  for (int i = threadIdx.x; i < a.n; i += blockDim.x) rect_setup_image<false, true>(a, i, fo);
}

// ------------------------------------------------------------------------------------------------------------ warp
// grid = (pixel blocks of the largest output, images).  A thread maps kRectPix consecutive output pixels and stages their bytes
// (image, mask) in its slot of the warp's span in shared memory; the warp then writes the span as contiguous 16-byte stores (full
// sectors) when it is aligned and whole.  The map is written directly, two pixels per 16-byte store when aligned.
__device__ __forceinline__ void rect_store_span(unsigned char* dst, const unsigned char* span, int bytes_per_thread, int lane, int nj,
                                                bool full) {
  if (full && ((uintptr_t)dst & 15) == 0) {
    const uint4* s = reinterpret_cast<const uint4*>(span);
    uint4* o = reinterpret_cast<uint4*>(dst);
    for (int q = lane; q < 2 * bytes_per_thread; q += 32) __stcs(o + q, s[q]);   // 32 * bytes_per_thread / 16 vectors
  } else {
    const int nb = nj * (bytes_per_thread / kRectPix);
    for (int b = 0; b < nb; ++b) dst[lane * bytes_per_thread + b] = span[lane * bytes_per_thread + b];
  }
}

template <int C, bool kNearest>
__global__ void __launch_bounds__(kRectThreads) rectify_warp_kernel(RectArgs a) {
  __shared__ __align__(16) unsigned char s_im[kRectThreads / 32][32 * kRectPix * C];
  __shared__ __align__(16) unsigned char s_mk[kRectThreads / 32][32 * kRectPix];
  pdl_wait();      // the maps are written by rectify_setup_kernel
  pdl_launch();
  const RectImage d = a.im[blockIdx.y];
  const long long HW = (long long)d.Ho * d.Wo;
  const long long p0 = ((long long)blockIdx.x * kRectThreads + threadIdx.x) * kRectPix;
  const long long pw = p0 - (long long)(threadIdx.x & 31) * kRectPix;     // first pixel of this warp
  if (pw >= HW) return;                                                   // whole warps only: the stores below need all lanes
  const int nj = p0 < HW ? (int)min((long long)kRectPix, HW - p0) : 0;
  const int lane = threadIdx.x & 31, wp = threadIdx.x >> 5;
  const RectMap& mp = a.map[blockIdx.y];
  double m[9];
#pragma unroll
  for (int k = 0; k < 9; ++k) m[k] = mp.m[k];
  const bool ok = mp.ok != 0;
  const unsigned char* src = a.in + d.in_off;
  unsigned char* px = &s_im[wp][lane * kRectPix * C];
  unsigned char* mk = &s_mk[wp][lane * kRectPix];
  float uv[2 * kRectPix];
  int i = (int)(min(p0, HW - 1) / d.Wo), j = (int)(min(p0, HW - 1) - (long long)i * d.Wo);
  const double Wd = d.W, Hd = d.H;
#pragma unroll
  for (int k = 0; k < kRectPix; ++k) {
    const double x = j + 0.5, y = i + 0.5;
    const double X = m[0] * x + m[1] * y + m[2], Y = m[3] * x + m[4] * y + m[5], Z = m[6] * x + m[7] * y + m[8];
    const double u = X / Z, v = Y / Z;
    const bool valid = ok && k < nj && Z > 0.0 && u >= 0.0 && u <= Wd && v >= 0.0 && v <= Hd;
    uv[2 * k] = valid ? (float)u : NAN;
    uv[2 * k + 1] = valid ? (float)v : NAN;
    mk[k] = valid;
    if (!valid) {
#pragma unroll
      for (int c = 0; c < C; ++c) px[k * C + c] = a.fill[c];
    } else if (kNearest) {
      const int xi = (int)fmin(fmax(floor((u - 0.5) + 0.5), 0.0), Wd - 1.0);
      const int yi = (int)fmin(fmax(floor((v - 0.5) + 0.5), 0.0), Hd - 1.0);
      const unsigned char* q = src + ((long long)yi * d.W + xi) * C;
#pragma unroll
      for (int c = 0; c < C; ++c) px[k * C + c] = __ldg(q + c);
    } else {
      const double s = u - 0.5, t = v - 0.5;
      const double fs = floor(s), ft = floor(t);
      const double fx = s - fs, fy = t - ft;
      const int x0 = (int)fmin(fmax(fs, 0.0), Wd - 1.0), x1 = (int)fmin(fmax(fs + 1.0, 0.0), Wd - 1.0);
      const int y0 = (int)fmin(fmax(ft, 0.0), Hd - 1.0), y1 = (int)fmin(fmax(ft + 1.0, 0.0), Hd - 1.0);
      const unsigned char* r0 = src + (long long)y0 * d.W * C;
      const unsigned char* r1 = src + (long long)y1 * d.W * C;
#pragma unroll
      for (int c = 0; c < C; ++c) {
        const double top = (double)__ldg(r0 + x0 * C + c) * (1.0 - fx) + (double)__ldg(r0 + x1 * C + c) * fx;
        const double bot = (double)__ldg(r1 + x0 * C + c) * (1.0 - fx) + (double)__ldg(r1 + x1 * C + c) * fx;
        const double val = rint(top * (1.0 - fy) + bot * fy);
        px[k * C + c] = (unsigned char)fmin(fmax(val, 0.0), 255.0);
      }
    }
    if (++j == d.Wo) { j = 0; ++i; }
  }
  const bool full = pw + 32 * kRectPix <= HW;       // warp-uniform
  __syncwarp();
  rect_store_span(a.out + d.out_off + pw * C, s_im[wp], kRectPix * C, lane, nj, full);
  if (d.mask_off >= 0) rect_store_span(a.mask + d.mask_off + pw, s_mk[wp], kRectPix, lane, nj, full);
  if (d.map_off >= 0) {
    float* o = a.xy + d.map_off + 2 * p0;
    if (nj == kRectPix && ((uintptr_t)o & 15) == 0) {
#pragma unroll
      for (int k = 0; k < kRectPix; k += 2) __stcs(reinterpret_cast<float4*>(o + 2 * k), make_float4(uv[2 * k], uv[2 * k + 1], uv[2 * k + 2], uv[2 * k + 3]));
    } else {
#pragma unroll
      for (int k = 0; k < 2 * kRectPix; ++k)
        if (k < 2 * nj) o[k] = uv[k];
    }
  }
}

}  // namespace pf
