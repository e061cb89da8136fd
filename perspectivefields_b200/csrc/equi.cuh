// Panorama -> pinhole views: PanoCam.crop_equi / PanoCam(path).get_image (perspective2d/utils/panocam.py:121-249), batched.  One
// launch crops up to kEquiChunk views of one equirectangular panorama (uint8 or float32, 1 or 3 channels).  Also the rotation
// warp of whole panoramas that levels them (rotate_panoramas_kernel, DESIGN.md section 1 "Panorama levelling").
#pragma once
#include <math.h>

#include <type_traits>

#include "common.cuh"
#include "pano.cuh"

namespace pf {

// Geometry per output pixel (i, j) of a view (DESIGN.md section 1), float64 with explicit round-to-nearest intrinsics (no fma
// contraction), in this order:
//   ray (x, y, 1) = ((j - W/2) / f, (i - H/2) / f, 1), x right, y down, z forward;
//   roll:      x' = x cr - y sr,        y' = x sr + y cr
//   elevation: y'' = y' ce - se,        z'' = y' se + ce
//   azimuth:   x''' = x' ca + z'' sa,   z''' = -(x' sa) + z'' ca
//   theta = atan2(x''', z'''), phi = -asin(y'' / |p|) with |p| = sqrt((x'''^2 + y''^2) + z'''^2)
//   panorama pixel u = (theta + pi) * (Wp / 2pi), v = (pi/2 - phi) * (Hp / pi)   (pixel k is sampled at k)
// then the panorama sampler of pano.cuh (bilinear: columns wrap, rows clamp, float64 weights) or the nearest pixel
// (floor(u + 1/2) mod Wp, clamp(floor(v + 1/2), 0, Hp - 1)).
struct EquiView {            // device copy of one pf_equi_view, with what the host precomputes once per view
  int H, W;
  double f, u0, v0;          // focal length in pixels, W / 2, H / 2
  double cr, sr, ce, se, ca, sa;
  long long off;             // byte offset of the view's [H, W, C] crop in im
};
struct EquiMap {
  int Hp, Wp, C;             // panorama size and channels (1 or 3)
  int nearest, swap_rb;      // nearest-pixel sampling; output channel c reads input channel 2 - c
  double su, sv;             // Wp / 2pi, Hp / pi
};
constexpr int kEquiChunk = 24;             // views per launch (the descriptors travel as a kernel parameter, < 4 KB)
struct EquiBatch { EquiView v[kEquiChunk]; };
constexpr int kEquiThreads = 256, kEquiPix = 4;   // 4 consecutive pixels (of the view's flat H*W range) per thread

__device__ __forceinline__ void equi_forward(const EquiView& v, const EquiMap& m, int i, int j, double& u, double& w) {
  const double x = pd(ps((double)j, v.u0), v.f), y = pd(ps((double)i, v.v0), v.f);
  const double xr = ps(pm(x, v.cr), pm(y, v.sr)), yr = pa(pm(x, v.sr), pm(y, v.cr));
  const double ye = ps(pm(yr, v.ce), v.se), ze = pa(pm(yr, v.se), v.ce);
  const double xa = pa(pm(xr, v.ca), pm(ze, v.sa)), za = pa(-pm(xr, v.sa), pm(ze, v.ca));
  const double n = __dsqrt_rn(pa(pa(pm(xa, xa), pm(ye, ye)), pm(za, za)));
  u = pm(pa(atan2(xa, za), M_PI), m.su);
  w = pm(ps(M_PI / 2, -asin(pd(ye, n))), m.sv);
}

// Input element -> the float64 value the sampler weighs.  kUnit (get_image): torchvision's ToTensor, p / 255 in float32.
template <typename Tin, bool kUnit>
__device__ __forceinline__ double equi_in(const Tin* p) {
  if constexpr (kUnit) return (double)__fdiv_rn((float)__ldg(p), 255.f);
  else return (double)__ldg(p);
}
// float64 sample -> output element: the sampler's float32 result cast back to the input dtype (uint8: truncated); kUnit: then
// ToPILImage's mul(255).byte() in float32.
template <typename Tin, bool kUnit>
__device__ __forceinline__ auto equi_out(double s) {
  const float s32 = (float)s;
  if constexpr (std::is_same<Tin, float>::value) return s32;
  else if constexpr (kUnit) return (unsigned char)(int)fminf(fmaxf(__fmul_rn(s32, 255.f), 0.f), 255.f);
  else return (unsigned char)(int)fminf(fmaxf(s32, 0.f), 255.f);
}

// grid = (pixel blocks of the largest view, views of the chunk).  A thread samples kEquiPix consecutive pixels into its slot of
// the warp's span in shared memory (nothing per pixel stays live in registers across the float64 atan2 / asin calls); the warp
// then writes its 32 * kEquiPix pixels as contiguous 16-byte stores (full sectors) when the span is aligned.
template <typename Tin, bool kUnit>
__global__ void __launch_bounds__(kEquiThreads) equi_views_kernel(const __grid_constant__ EquiBatch batch, const __grid_constant__ EquiMap m,
                                                                  const Tin* __restrict__ pano, unsigned char* __restrict__ im) {
  using Tout = decltype(equi_out<Tin, kUnit>(0.0));
  constexpr int kMaxBytes = 3 * (int)sizeof(Tout) * kEquiPix;      // per thread
  __shared__ __align__(16) unsigned char s_st[kEquiThreads / 32][32 * kMaxBytes];
  const EquiView& v = batch.v[blockIdx.y];
  const long long HW = (long long)v.H * v.W;
  const long long p0 = ((long long)blockIdx.x * kEquiThreads + threadIdx.x) * kEquiPix;
  const long long pw = p0 - (long long)(threadIdx.x & 31) * kEquiPix;     // first pixel of this warp
  if (pw >= HW) return;                                                   // (whole warps only: the staging below needs all lanes)
  const int nj = p0 < HW ? (int)min((long long)kEquiPix, HW - p0) : 0;
  const int C = m.C, bpp = C * (int)sizeof(Tout);
  const int lane = threadIdx.x & 31, wp = threadIdx.x >> 5;
  Tout* px = reinterpret_cast<Tout*>(&s_st[wp][lane * kEquiPix * bpp]);   // this thread's pixels, [kEquiPix][C]
  int i = (int)(min(p0, HW - 1) / v.W), j = (int)(min(p0, HW - 1) - (long long)i * v.W);
#pragma unroll
  for (int k = 0; k < kEquiPix; ++k) {
    if (k < nj) {
      double u, w;
      equi_forward(v, m, i, j, u, w);
      if (!m.nearest) {
        const PanoTaps t = pano_taps(u, w, m.Hp, m.Wp);
        const Tin* r0 = pano + t.y0 * m.Wp * C;
        const Tin* r1 = pano + t.y1 * m.Wp * C;
#pragma unroll
        for (int c = 0; c < 3; ++c) {
          if (c >= C) break;
          const int ci = m.swap_rb ? 2 - c : c;
          const double s = pano_lerp(t, equi_in<Tin, kUnit>(r0 + t.x0 * C + ci), equi_in<Tin, kUnit>(r0 + t.x1 * C + ci),
                                     equi_in<Tin, kUnit>(r1 + t.x0 * C + ci), equi_in<Tin, kUnit>(r1 + t.x1 * C + ci));
          px[k * C + c] = equi_out<Tin, kUnit>(s);
        }
      } else {
        long long x = (long long)floor(pa(u, 0.5)) % m.Wp;
        if (x < 0) x += m.Wp;
        const long long y = (long long)fmin(fmax(floor(pa(w, 0.5)), 0.0), (double)(m.Hp - 1));
        const Tin* q = pano + (y * m.Wp + x) * C;
#pragma unroll
        for (int c = 0; c < 3; ++c) {
          if (c >= C) break;
          px[k * C + c] = equi_out<Tin, kUnit>(equi_in<Tin, kUnit>(q + (m.swap_rb ? 2 - c : c)));
        }
      }
    }
    if (++j == v.W) { j = 0; ++i; }
  }
  unsigned char* dst = im + v.off;
  const bool full = pw + 32 * kEquiPix <= HW;       // warp-uniform
  if (full && ((uintptr_t)(dst + pw * bpp) & 15) == 0) {
    __syncwarp();
    const uint4* src = reinterpret_cast<const uint4*>(s_st[wp]);
    uint4* d = reinterpret_cast<uint4*>(dst + pw * bpp);
    for (int q = lane; q < 2 * kEquiPix * bpp; q += 32) __stcs(d + q, src[q]);      // 32 * kEquiPix * bpp / 16 vectors
  } else {
    Tout* d = reinterpret_cast<Tout*>(dst) + p0 * C;
#pragma unroll
    for (int k = 0; k < kEquiPix; ++k)
#pragma unroll
      for (int c = 0; c < 3; ++c)
        if (k < nj && c < C) d[k * C + c] = px[k * C + c];
  }
}

// ------------------------------------------------------------------------------------------------------ panorama rotation
// out(d) = P(R d) for each panorama of a list (DESIGN.md section 1, "Panorama levelling"): output pixel (i, j) is the direction
// theta = 2 pi j / Wp - pi, phi = pi/2 - pi i / Hp, d = (cos phi sin theta, -sin phi, cos phi cos theta); R d (float64) maps back
// by the crop rule (u = (theta' + pi) Wp / 2pi, v = (pi/2 - phi') Hp / pi) and is sampled by the panorama sampler (bilinear, or
// the nearest pixel as equi_views_kernel takes it).  uint8 output is rounded to nearest (half to even) and clamped, float32 output
// is the sample rounded to float32.  Optional map: float32 (u, v) per output pixel.
struct RotPano {             // device copy of one pf_rotate_pano
  int Hp, Wp;
  long long in_off, out_off, map_off;   // elements of the input / output panorama, floats of the map (-1: none)
};
struct RotArgs {
  const RotPano* pano; const double* R;   // [n] descriptors, [n][9] rotations (row-major)
  const void* in; void* out; float* map;
  int C, nearest;
};
// A block covers kRotRows rows x kRotCols columns: sin / cos of theta once per column and of phi once per row into shared memory;
// each warp takes kRotRows / 8 rows of 32 lanes x kEquiPix consecutive pixels and writes each row span as equi_views_kernel does.
constexpr int kRotThreads = 256, kRotCols = 32 * kEquiPix, kRotRows = 16;

template <typename T>
__global__ void __launch_bounds__(kRotThreads) rotate_panoramas_kernel(const RotArgs a) {
  constexpr int kMaxBytes = 3 * (int)sizeof(T) * kEquiPix;      // per thread
  __shared__ __align__(16) unsigned char s_st[kRotThreads / 32][32 * kMaxBytes];
  __shared__ double s_col[kRotCols][2], s_row[kRotRows][2];
  const RotPano d = a.pano[blockIdx.y];
  const int tiles_x = (d.Wp + kRotCols - 1) / kRotCols;
  const int i0 = (int)(blockIdx.x / tiles_x) * kRotRows, j0 = (int)(blockIdx.x % tiles_x) * kRotCols;
  if (i0 >= d.Hp) return;   // (whole blocks)
  const double Wd = d.Wp, Hd = d.Hp;
  if (threadIdx.x < kRotCols) {
    const double t = 2.0 * M_PI * (double)(j0 + (int)threadIdx.x) / Wd - M_PI;
    sincos(t, &s_col[threadIdx.x][0], &s_col[threadIdx.x][1]);
  } else if (threadIdx.x < kRotCols + kRotRows) {
    const int r = threadIdx.x - kRotCols;
    const double f = M_PI / 2.0 - M_PI * (double)(i0 + r) / Hd;
    sincos(f, &s_row[r][0], &s_row[r][1]);
  }
  double R[9];
#pragma unroll
  for (int k = 0; k < 9; ++k) R[k] = __ldg(a.R + 9LL * blockIdx.y + k);
  __syncthreads();
  const int C = a.C, bpp = C * (int)sizeof(T);
  const int lane = threadIdx.x & 31, wp = threadIdx.x >> 5;
  const T* src = reinterpret_cast<const T*>(a.in) + d.in_off;
  T* px = reinterpret_cast<T*>(&s_st[wp][lane * kEquiPix * bpp]);   // this thread's pixels, [kEquiPix][C]
  const int jl = lane * kEquiPix, nj = max(0, min(kEquiPix, d.Wp - (j0 + jl)));
  const bool full = j0 + kRotCols <= d.Wp;   // warp-uniform
#pragma unroll 1
  for (int rr = wp; rr < kRotRows; rr += kRotThreads / 32) {
    const int i = i0 + rr;
    if (i >= d.Hp) break;   // (warp-uniform)
    const double sf = s_row[rr][0], cf = s_row[rr][1];
#pragma unroll
    for (int k = 0; k < kEquiPix; ++k) {
      if (k >= nj) break;
      const double st = s_col[jl + k][0], ct = s_col[jl + k][1];
      const double dx = cf * st, dy = -sf, dz = cf * ct;
      const double x = R[0] * dx + R[1] * dy + R[2] * dz, y = R[3] * dx + R[4] * dy + R[5] * dz, z = R[6] * dx + R[7] * dy + R[8] * dz;
      const double n = sqrt(x * x + y * y + z * z);
      const double u = (atan2(x, z) + M_PI) * (Wd / (2.0 * M_PI)), w = (M_PI / 2.0 + asin(y / n)) * (Hd / M_PI);
      if (d.map_off >= 0) *reinterpret_cast<float2*>(a.map + d.map_off + 2 * ((long long)i * d.Wp + j0 + jl + k)) = make_float2((float)u, (float)w);
      if (!a.nearest) {
        const PanoTaps t = pano_taps(u, w, d.Hp, d.Wp);
        const T* r0 = src + t.y0 * d.Wp * C;
        const T* r1 = src + t.y1 * d.Wp * C;
#pragma unroll
        for (int c = 0; c < 3; ++c) {
          if (c >= C) break;
          const double s = pano_lerp(t, (double)__ldg(r0 + t.x0 * C + c), (double)__ldg(r0 + t.x1 * C + c), (double)__ldg(r1 + t.x0 * C + c),
                                     (double)__ldg(r1 + t.x1 * C + c));
          if constexpr (std::is_same<T, float>::value) px[k * C + c] = (float)s;
          else px[k * C + c] = (unsigned char)fmin(fmax(rint(s), 0.0), 255.0);
        }
      } else {
        long long x = (long long)floor(u + 0.5) % d.Wp;
        if (x < 0) x += d.Wp;
        const long long y = (long long)fmin(fmax(floor(w + 0.5), 0.0), Hd - 1.0);
        const T* q = src + (y * d.Wp + x) * C;
#pragma unroll
        for (int c = 0; c < 3; ++c)
          if (c < C) px[k * C + c] = __ldg(q + c);
      }
    }
    const long long p0 = (long long)i * d.Wp + j0;   // first pixel of the warp's span
    T* dst = reinterpret_cast<T*>(a.out) + d.out_off + p0 * C;
    __syncwarp();
    if (full && ((uintptr_t)dst & 15) == 0) {
      const uint4* s = reinterpret_cast<const uint4*>(s_st[wp]);
      uint4* o = reinterpret_cast<uint4*>(dst);
      for (int q = lane; q < 2 * kEquiPix * bpp; q += 32) __stcs(o + q, s[q]);   // 32 * kEquiPix * bpp / 16 vectors
    } else {
#pragma unroll
      for (int k = 0; k < kEquiPix; ++k)
#pragma unroll
        for (int c = 0; c < 3; ++c)
          if (k < nj && c < C) dst[(jl + k) * C + c] = px[k * C + c];
    }
    __syncwarp();   // the staging span is rewritten by the next row
  }
}

}  // namespace pf
