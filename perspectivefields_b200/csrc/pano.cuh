// Panorama -> perspective / distorted views with their ground-truth fields: PanoCam.crop_distortion
// (perspective2d/utils/panocam.py:559-752), batched.  One launch crops up to kPanoChunk views of one equirectangular uint8 panorama.
#pragma once
#include <math.h>

#include "common.cuh"

namespace pf {

// Geometry per output pixel (i, j) of a view, float64 in the reference's order of operations (every + - * / below is an explicit
// round-to-nearest intrinsic, so nvcc never contracts a pair into an fma the numpy reference does not perform):
//   camera plane (j - u0) / f, -((i - v0) / f) -> unit sphere of the Unified Spherical Model (alpha = xi + sqrt(1 + (1 - xi^2) r^2),
//   or xi where the root is imaginary: np.real(csqrt(.)) of a negative argument is 0) -> rot_az (rot_roll^T (rot_el p)), applied
//   as the reference's three 3x3 products -> ntheta = atan2(x, z), nphi = atan2(y, sqrt(z^2 + x^2)) -> panorama pixel
//   nx = (1/ax)(ntheta - bx), ny = (1/ay)(nphi - by).
// up: the point (nx, ny - 1e-5) projected back into the view minus the pixel itself, with the reference's Y = sin(nphi) (not
//   sin(nphi_end)), then sklearn's normalize (a vector shorter than 10 eps is left unscaled).  The difference is ~1e-5 px or less
//   against coordinates of hundreds of px, so the whole chain is float64.
// im: bilinear sample of the panorama at (ny, nx) (the project's sampler rule, DESIGN.md section 5: columns wrap, rows clamp,
//   float64 weights and sum, clipped and truncated to uint8), 0 outside the catadioptric disk when xi > 1 and f < fmin.
// offset / status: the horizon row at column W // 2 from the zero crossings of nphi (the last x-block of the grid).
struct PanoView {            // device copy of one pf_pano_view plus what the host precomputes once per view
  int H, W;
  double f, xi, one_m_xi2, u0, v0;
  double rel[9], rroll[9], raz[9];       // rot_el, rot_roll, rot_az (row-major, as the reference builds them)
  double r2, ci0, ci1;                   // catadioptric disk: radius^2 and centre (round-half-even(H/2), round-half-even(W/2))
  int masked;                            // xi > 1 and f < fmin
  long long im_off, fld_off;             // byte offset of [H,W,3] in im; float offset of [H,W] blocks ([H,W,2] blocks: 2 * fld_off)
};
struct PanoMap {             // panorama constants of :666-687 (host, float64)
  double ax, bx, iax, ay, by, iay;
  int Hp, Wp;
};
constexpr int kPanoChunk = 12;             // views per launch (the descriptors travel as a kernel parameter, < 4 KB)
struct PanoBatch { PanoView v[kPanoChunk]; };
constexpr int kPanoThreads = 256, kPanoPix = 4;   // 4 consecutive pixels (of the view's flat H*W range) per thread
constexpr double kUpTiny = 10.0 * 2.220446049250313e-16;   // sklearn.preprocessing._handle_zeros_in_scale: norms < 10 eps -> 1

__device__ __forceinline__ double pm(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ double pa(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ double ps(double a, double b) { return __dsub_rn(a, b); }
__device__ __forceinline__ double pd(double a, double b) { return __ddiv_rn(a, b); }

// The project's panorama sampler (DESIGN.md section 1), shared with equi_views_kernel: taps and weights of a bilinear sample at
// panorama pixel (nx, ny) in pixel-index units; columns wrap (x1 = (x0 + 1) mod Wp), rows clamp (ny to [0, Hp - 1], y1 <= Hp - 1).
struct PanoTaps {
  long long x0, x1, y0, y1;
  double wx, hx, wy, hy;
};
__device__ __forceinline__ PanoTaps pano_taps(double nx, double ny, int Hp, int Wp) {
  PanoTaps t;
  const double xf = floor(nx);
  t.wx = ps(nx, xf); t.hx = ps(1.0, t.wx);
  t.x0 = (long long)xf % Wp;
  if (t.x0 < 0) t.x0 += Wp;
  t.x1 = t.x0 + 1 == Wp ? 0 : t.x0 + 1;
  const double nyc = fmin(fmax(ny, 0.0), (double)(Hp - 1));
  const double yf = floor(nyc);
  t.wy = ps(nyc, yf); t.hy = ps(1.0, t.wy);
  t.y0 = (long long)yf;
  t.y1 = t.y0 + 1 < Hp ? t.y0 + 1 : t.y0;
  return t;
}
// (1 - wy) ((1 - wx) p00 + wx p01) + wy ((1 - wx) p10 + wx p11), float64, in that order
__device__ __forceinline__ double pano_lerp(const PanoTaps& t, double p00, double p01, double p10, double p11) {
  return pa(pm(t.hy, pa(pm(t.hx, p00), pm(t.wx, p01))), pm(t.wy, pa(pm(t.hx, p10), pm(t.wx, p11))));
}

// out = M p (transpose: M^T p); each row summed left to right, (m0 x + m1 y) + m2 z
__device__ __forceinline__ void pano_rot(const double* M, bool transpose, double& x, double& y, double& z) {
  double o[3];
#pragma unroll
  for (int r = 0; r < 3; ++r) {
    const double m0 = transpose ? M[r] : M[3 * r], m1 = transpose ? M[3 + r] : M[3 * r + 1], m2 = transpose ? M[6 + r] : M[3 * r + 2];
    o[r] = pa(pa(pm(m0, x), pm(m1, y)), pm(m2, z));
  }
  x = o[0]; y = o[1]; z = o[2];
}

// :596-664: (ntheta, nphi) of pixel (i, j)
__device__ __forceinline__ void pano_forward(const PanoView& v, int i, int j, double& ntheta, double& nphi) {
  const double xc = pd(ps((double)j, v.u0), v.f);
  const double yc = -pd(ps((double)i, v.v0), v.f);
  const double aux = pa(pm(xc, xc), pm(yc, yc));
  const double t = pa(1.0, pm(v.one_m_xi2, aux));
  const double alpha = pa(v.xi, t >= 0.0 ? __dsqrt_rn(t) : 0.0);
  const double acd = pd(alpha, pa(aux, 1.0));
  double x = pm(xc, acd), y = pm(yc, acd), z = ps(acd, v.xi);
  pano_rot(v.rel, false, x, y, z);
  pano_rot(v.rroll, true, x, y, z);
  pano_rot(v.raz, false, x, y, z);
  ntheta = atan2(x, z);
  nphi = atan2(y, __dsqrt_rn(pa(pm(z, z), pm(x, x))));
}

__device__ __forceinline__ int pano_sign(double x) { return (x > 0.0) - (x < 0.0); }

// :709-722 for view v -> offset (nan when there is no crossing or an assertion fails) and status 0 / 1 / 2
__device__ void pano_offset(const PanoView& v, double* offset, int* status) {
  __shared__ int s_count, s_first;
  if (threadIdx.x == 0) { s_count = 0; s_first = 0x7fffffff; }
  __syncthreads();
  const int jc = v.W / 2;
  for (int r = threadIdx.x; r < v.H - 1; r += blockDim.x) {
    double t0, p0, t1, p1;
    pano_forward(v, r, jc, t0, p0);
    pano_forward(v, r + 1, jc, t1, p1);
    if (pano_sign(p0) != pano_sign(p1)) { atomicAdd(&s_count, 1); atomicMin(&s_first, r); }
  }
  __syncthreads();
  if (threadIdx.x != 0) return;
  double off = __longlong_as_double(0x7ff8000000000000LL);
  int st = 0;
  if (s_count > 0) {
    st = s_count >= 2 ? 1 : 0;
    const int r = s_first;
    double t, c0, c1;
    pano_forward(v, r, jc, t, c0);
    pano_forward(v, r + 1, jc, t, c1);
    if (!(c0 >= 0.0) || !(c1 <= 0.0)) {
      st = 2;
    } else {
      const double dy = ps(c1, c0), q = pd(c0, dy);
      if (!(q <= 1.0)) st = 2;
      else off = ps((double)r, q);
    }
  }
  if (offset) *offset = off;
  if (status) *status = st;
}

// grid = (pixel blocks of the largest view + 1, views of the chunk); the last x-block of every view computes its offset.
// Stores: ntheta / nphi / lat one float4 per thread, up / xy two float4 per thread (as camera_fields_kernel); the crop's 12 bytes
// per thread are staged in shared memory so that a warp writes its 384 contiguous bytes as 24 16-byte stores (full sectors).
__global__ void __launch_bounds__(kPanoThreads) pano_views_kernel(const __grid_constant__ PanoBatch batch, const __grid_constant__ PanoMap m,
                                                                  const unsigned char* __restrict__ pano, unsigned char* __restrict__ im,
                                                                  float* __restrict__ ntheta_o, float* __restrict__ nphi_o, float* __restrict__ up_o,
                                                                  float* __restrict__ lat_o, float* __restrict__ xy_o, double* __restrict__ offset,
                                                                  int* __restrict__ status, int view0) {
  __shared__ __align__(16) unsigned char s_im[kPanoThreads / 32][32 * 3 * kPanoPix];
  const PanoView& v = batch.v[blockIdx.y];
  if (blockIdx.x == gridDim.x - 1) {
    if (offset || status) pano_offset(v, offset ? offset + view0 + blockIdx.y : nullptr, status ? status + view0 + blockIdx.y : nullptr);
    return;
  }
  const long long HW = (long long)v.H * v.W;
  const long long p0 = ((long long)blockIdx.x * kPanoThreads + threadIdx.x) * kPanoPix;
  const long long pw = p0 - (long long)(threadIdx.x & 31) * kPanoPix;     // first pixel of this warp
  if (pw >= HW) return;                                                   // (whole warps only: the staging below needs all lanes)
  const int nj = p0 < HW ? (int)min((long long)kPanoPix, HW - p0) : 0;
  unsigned char px[3 * kPanoPix];
  float th[kPanoPix], ph[kPanoPix], upv[2 * kPanoPix], xyv[2 * kPanoPix];
  int i = (int)(min(p0, HW - 1) / v.W), j = (int)(min(p0, HW - 1) - (long long)i * v.W);
#pragma unroll
  for (int k = 0; k < kPanoPix; ++k) {
    px[3 * k] = px[3 * k + 1] = px[3 * k + 2] = 0;
    th[k] = ph[k] = upv[2 * k] = upv[2 * k + 1] = xyv[2 * k] = xyv[2 * k + 1] = 0.f;
    if (k < nj) {
      double ntheta, nphi;
      pano_forward(v, i, j, ntheta, nphi);
      const double nx = pm(m.iax, ps(ntheta, m.bx)), ny = pm(m.iay, ps(nphi, m.by));
      th[k] = (float)ntheta; ph[k] = (float)nphi; xyv[2 * k] = (float)nx; xyv[2 * k + 1] = (float)ny;
      if (im) {
        const bool inside = !v.masked || pa(pm(ps((double)i, v.ci0), ps((double)i, v.ci0)), pm(ps((double)j, v.ci1), ps((double)j, v.ci1))) < v.r2;
        if (inside) {
          const PanoTaps t = pano_taps(nx, ny, m.Hp, m.Wp);
          const unsigned char* r0 = pano + t.y0 * m.Wp * 3;
          const unsigned char* r1 = pano + t.y1 * m.Wp * 3;
#pragma unroll
          for (int c = 0; c < 3; ++c) {
            const double s = pano_lerp(t, __ldg(r0 + t.x0 * 3 + c), __ldg(r0 + t.x1 * 3 + c), __ldg(r1 + t.x0 * 3 + c), __ldg(r1 + t.x1 * 3 + c));
            px[3 * k + c] = (unsigned char)(int)fmin(fmax(s, 0.0), 255.0);
          }
        }
      }
      if (up_o) {
        // :723-750
        const double te = pa(pm(nx, m.ax), m.bx), pe = pa(pm(ps(ny, 1e-5), m.ay), m.by);
        double st, ct, sp, cp;
        sincos(te, &st, &ct);
        sincos(pe, &sp, &cp);
        double x = pm(cp, st), y = sin(nphi), z = pm(cp, ct);
        pano_rot(v.raz, true, x, y, z);
        pano_rot(v.rroll, false, x, y, z);
        pano_rot(v.rel, true, x, y, z);
        const double n = __dsqrt_rn(pa(pa(pm(x, x), pm(y, y)), pm(z, z)));
        const double den = pa(pm(v.xi, n), z);
        const double ux = ps(pa(pd(pm(x, v.f), den), v.u0), (double)j);
        const double uy = ps(pa(pd(pm(-y, v.f), den), v.v0), (double)i);
        double len = __dsqrt_rn(pa(pm(ux, ux), pm(uy, uy)));
        if (len < kUpTiny) len = 1.0;
        upv[2 * k] = (float)pd(ux, len); upv[2 * k + 1] = (float)pd(uy, len);
      }
    }
    if (++j == v.W) { j = 0; ++i; }
  }
  const bool full = pw + 32 * kPanoPix <= HW;       // warp-uniform
  if (im) {
    unsigned char* dst = im + v.im_off;
    if (full && ((uintptr_t)(dst + pw * 3) & 15) == 0) {
      const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
      uint32_t* s = reinterpret_cast<uint32_t*>(&s_im[w][lane * 3 * kPanoPix]);
#pragma unroll
      for (int q = 0; q < 3; ++q)
        s[q] = (uint32_t)px[4 * q] | ((uint32_t)px[4 * q + 1] << 8) | ((uint32_t)px[4 * q + 2] << 16) | ((uint32_t)px[4 * q + 3] << 24);
      __syncwarp();
      if (lane < 24) __stcs(reinterpret_cast<uint4*>(dst + pw * 3) + lane, reinterpret_cast<const uint4*>(s_im[w])[lane]);
    } else {
#pragma unroll
      for (int k = 0; k < 3 * kPanoPix; ++k)
        if (k < 3 * nj) dst[p0 * 3 + k] = px[k];
    }
  }
  if (nj == 0) return;
  const long long f0 = v.fld_off + p0;
  float* outs1[3] = {ntheta_o, nphi_o, lat_o};
  const float* vals1[3] = {th, ph, ph};
#pragma unroll
  for (int o = 0; o < 3; ++o) {
    if (!outs1[o]) continue;
    float* d = outs1[o] + f0;
    if (nj == kPanoPix && ((uintptr_t)d & 15) == 0) __stcs(reinterpret_cast<float4*>(d), make_float4(vals1[o][0], vals1[o][1], vals1[o][2], vals1[o][3]));
    else {
#pragma unroll
      for (int k = 0; k < kPanoPix; ++k)
        if (k < nj) d[k] = vals1[o][k];
    }
  }
  float* outs2[2] = {up_o, xy_o};
  const float* vals2[2] = {upv, xyv};
#pragma unroll
  for (int o = 0; o < 2; ++o) {
    if (!outs2[o]) continue;
    float* d = outs2[o] + 2 * f0;
    if (nj == kPanoPix && ((uintptr_t)d & 15) == 0) {
      __stcs(reinterpret_cast<float4*>(d), make_float4(vals2[o][0], vals2[o][1], vals2[o][2], vals2[o][3]));
      __stcs(reinterpret_cast<float4*>(d) + 1, make_float4(vals2[o][4], vals2[o][5], vals2[o][6], vals2[o][7]));
    } else {
#pragma unroll
      for (int k = 0; k < 2 * kPanoPix; ++k)
        if (k < 2 * nj) d[k] = vals2[o][k];
    }
  }
}

}  // namespace pf
