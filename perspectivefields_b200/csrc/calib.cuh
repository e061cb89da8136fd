// Camera parameters from perspective fields: a batched Levenberg-Marquardt fit of roll, pitch, focal length and (optionally) the
// principal point to predicted up and latitude fields (this project's rule, DESIGN.md section 1 "Camera fit"; restated on the
// CPU in tests/oracle_calib.py).
//
// theta = (roll r, pitch e, s = ln f_rel, cx_rel, cy_rel); F = f_rel H, cx = (cx_rel + 1/2) W, cy = (cy_rel + 1/2) H.  The model
// is what camera_fields_kernel (prepost.cuh) draws, in float64:
//   up at the pixel centre (x, y):  u = (-sin r cos e F + sin e (cx - x), -cos r cos e F + sin e (cy - y))  (unnormalised)
//   latitude (radians): -atan2(yw, hypot(xw, zw)) of the ray (dx, dy, F) / F on get_lat_general's linspace grid, rotated by
//                       roll, then pitch.
// Residuals: r_u = atan2(u x p, u . p) where the prediction p is finite with |p| > 1e-5; r_l = rad(l_pred) - l where l_pred
// is finite; both under the optional mask.  Cost C = 1/2 sum delta^2 rho((r / delta)^2) (scipy's least_squares with
// f_scale = delta: rho(z) = z, or Huber's 2 sqrt(z) - 1 above 1), IRLS weights w = rho'.
//
// Three kernels, chained with programmatic dependent launch and enqueued without synchronisation: fit_init_kernel (the
// start), then max_iterations pairs of fit_pass_kernel (one cost evaluation: C, A = sum w J^T J and g = sum w J^T r at the
// candidate, as per-block fp64 partials) and fit_step_kernel (reduce the partials in a fixed order, accept or reject, solve the
// damped normal equations by Cholesky, write the next candidate or the result).  Images that have stopped cost their pass
// blocks one early exit.  No floating-point atomic decides a value: repeated calls are bit-identical.
#pragma once
#include <stdint.h>

#include "common.cuh"
#include "metrics.cuh"

namespace pf {

constexpr int kFitThreads = 256, kFitTile = 16 * kFitThreads;   // pass: 16 pixels per thread amortise the block reduction
constexpr int kFitQ = 22;                                        // partials per block: C, count, g[5], A[15] (upper triangle)
constexpr int kFitStepWarps = 8;
constexpr int kFitRunning = -1;
constexpr double kFitLambda0 = 1e-3, kFitCostRtol = 1e-12, kFitStepRtol = 1e-12, kFitLambdaMax = 1e16, kFitUpMin = 1e-5;
constexpr double kPi = 3.14159265358979323846;

__host__ __device__ constexpr int fit_nq(int P) { return 2 + P + P * (P + 1) / 2; }

struct FitImage {
  int H, W;
  long long up_off, up_sr, up_sc, up_sk;   // predicted up: element offset and strides (row, column, component)
  long long lat_off;                       // latitude [H, W] row-major, degrees
  long long mask_off;                      // bytes, -1: none
  int block0, nblk;                        // its blocks in the pass
  double init[5];                          // roll, pitch (radians), f_rel, cx_rel, cy_rel; NaN roll: the closed-form start
};
struct FitState {
  double theta[5], cand[5];   // accepted parameters, the candidate the next pass evaluates
  double A[15], g[5], C;      // at theta
  double lambda;
  int evals, status;          // cost evaluations so far; kFitRunning, or the final status
};
struct FitArgs {
  const FitImage* im; FitState* st; int n, nblocks;
  const float* up; const float* lat; const unsigned char* mask;
  double huber;               // 0: least squares
  int max_iter;
  double* part;               // [kFitQ][nblocks]
  double* params; double* cost; int* iters; int* status;
};

// The image whose blocks contain blockIdx.x (the last one with block0 <= blockIdx.x)
__device__ __forceinline__ int fit_image_of_block(const FitArgs& a) {
  int lo = 0, hi = a.n - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (a.im[mid].block0 <= (int)blockIdx.x) lo = mid; else hi = mid - 1;
  }
  return lo;
}

__device__ __forceinline__ bool up_usable(double px, double py) {
  return isfinite(px) && isfinite(py) && sqrt(px * px + py * py) > kFitUpMin;
}

// ------------------------------------------------------------------------------------------------------------ start
// One block of 64 threads per image, one thread per pixel of the 8 x 8 window of rows H/2 - 4 .. H/2 + 3 and the same columns
// around W/2 (clipped to the image):
//   roll0 = atan2(-sum px^, -sum py^) of the unit predictions (at the principal point up = (-sin r, -cos r));
//   pitch0 = the window's mean latitude (latitude = pitch at the principal point);
//   f0 = 1 / (H mean |grad l|), central differences where the four neighbours are valid (|grad l| = 1 / F there).
// A term without a valid pixel falls back to roll 0, pitch 0, vfov 60 degrees.
__global__ void __launch_bounds__(64) fit_init_kernel(FitArgs a, int principal_point) {
  __shared__ double shd[33];
  __shared__ int shi[33];
  pdl_wait();
  pdl_launch();
  const int i = blockIdx.x;
  const FitImage d = a.im[i];
  double th[5];
  if (!isnan(d.init[0])) {
    th[0] = d.init[0]; th[1] = d.init[1]; th[2] = log(d.init[2]);
    th[3] = principal_point ? d.init[3] : 0.0; th[4] = principal_point ? d.init[4] : 0.0;
  } else {
    const int y = d.H / 2 - 4 + (threadIdx.x >> 3), x = d.W / 2 - 4 + (threadIdx.x & 7);
    double sx = 0.0, sy = 0.0, sl = 0.0, sg = 0.0;
    int nu = 0, nl = 0, ng = 0;
    if (y >= 0 && y < d.H && x >= 0 && x < d.W) {
      auto ok = [&](int yy, int xx) { return d.mask_off < 0 || a.mask[d.mask_off + (long long)yy * d.W + xx] != 0; };
      auto lat = [&](int yy, int xx) { return (double)a.lat[d.lat_off + (long long)yy * d.W + xx] * (kPi / 180.0); };
      if (ok(y, x)) {
        const float* p = a.up + d.up_off + y * d.up_sr + x * d.up_sc;
        const double px = p[0], py = p[d.up_sk];
        if (up_usable(px, py)) {
          const double nn = sqrt(px * px + py * py);
          sx = px / nn; sy = py / nn; nu = 1;
        }
        const double l0 = lat(y, x);
        if (isfinite(l0)) {
          sl = l0; nl = 1;
          if (y > 0 && y < d.H - 1 && x > 0 && x < d.W - 1 && ok(y, x + 1) && ok(y, x - 1) && ok(y + 1, x) && ok(y - 1, x)) {
            const double r = lat(y, x + 1), l = lat(y, x - 1), b = lat(y + 1, x), t = lat(y - 1, x);
            if (isfinite(r) && isfinite(l) && isfinite(b) && isfinite(t)) {
              const double gx = 0.5 * (r - l), gy = 0.5 * (b - t);
              sg = sqrt(gx * gx + gy * gy); ng = 1;
            }
          }
        }
      }
    }
    sx = block_sum(sx, shd); sy = block_sum(sy, shd); sl = block_sum(sl, shd); sg = block_sum(sg, shd);
    nu = block_sum(nu, shi); nl = block_sum(nl, shi); ng = block_sum(ng, shi);
    th[0] = nu ? atan2(-sx, -sy) : 0.0;
    th[1] = nl ? sl / nl : 0.0;
    th[2] = (ng && sg > 0.0) ? log(1.0 / ((double)d.H * (sg / ng))) : log(1.0 / (2.0 * tan(kPi / 6.0)));
    th[3] = th[4] = 0.0;
  }
  if (threadIdx.x == 0) {
    FitState& s = a.st[i];
    for (int k = 0; k < 5; ++k) s.cand[k] = s.theta[k] = th[k];
    s.C = 0.0; s.lambda = kFitLambda0; s.evals = 0; s.status = kFitRunning;
  }
}

// ------------------------------------------------------------------------------------------------------------ pass
template <int P>
__device__ __forceinline__ void fit_accumulate(double (&acc)[fit_nq(P)], double r, const double (&J)[P], double huber) {
  const double ar = fabs(r);
  double c = r * r, w = 1.0;
  if (huber > 0.0 && ar > huber) { c = 2.0 * huber * ar - huber * huber; w = huber / ar; }
  acc[0] += c;
  acc[1] += 1.0;
#pragma unroll
  for (int k = 0; k < P; ++k) acc[2 + k] += w * J[k] * r;
  int q = 2 + P;
#pragma unroll
  for (int k = 0; k < P; ++k) {
    const double wk = w * J[k];
#pragma unroll
    for (int m = k; m < P; ++m) acc[q++] += wk * J[m];
  }
}

// Blocks of kFitTile pixels, each within one image.  Writes plane q of the partials: 0 = sum delta^2 rho (2 C), 1 = residual
// count, 2 .. 1 + P = g, then A's upper triangle row by row.
template <int P>
__global__ void __launch_bounds__(kFitThreads) fit_pass_kernel(FitArgs a) {
  constexpr int NQ = fit_nq(P);
  __shared__ double shq[kFitThreads / 32][NQ];
  pdl_wait();
  pdl_launch();
  const int img = fit_image_of_block(a);
  if (a.st[img].status != kFitRunning) return;   // stopped: A, g and C of the accepted point are kept in the state
  const FitImage d = a.im[img];
  double th[5];
#pragma unroll
  for (int k = 0; k < 5; ++k) th[k] = a.st[img].cand[k];
  const double F = exp(th[2]) * d.H, cx = (th[3] + 0.5) * d.W, cy = (th[4] + 0.5) * d.H;
  double sr, cr, se, ce;
  sincos(th[0], &sr, &cr);
  sincos(th[1], &se, &ce);
  const double Hd = d.H, Wd = d.W;
  // get_lat_general's grid: linspace((-W/2) - (cx - W/2), (W/2) - (cx - W/2), W), last sample exact (camera_fields_kernel)
  const double x0 = (-Wd / 2.0) - (cx - Wd / 2.0), x1 = (Wd / 2.0) - (cx - Wd / 2.0), sxg = (x1 - x0) / (Wd - 1.0);
  const double y0 = (-Hd / 2.0) - (cy - Hd / 2.0), y1 = (Hd / 2.0) - (cy - Hd / 2.0), syg = (y1 - y0) / (Hd - 1.0);
  const double rF = 1.0 / F;
  double acc[NQ];
#pragma unroll
  for (int q = 0; q < NQ; ++q) acc[q] = 0.0;
  const long long HW = (long long)d.H * d.W;
  const long long t0 = (long long)((int)blockIdx.x - d.block0) * kFitTile;
#pragma unroll 1
  for (int it = 0; it < kFitTile / kFitThreads; ++it) {
    const long long q = t0 + it * kFitThreads + threadIdx.x;
    if (q >= HW) break;
    if (d.mask_off >= 0 && a.mask[d.mask_off + q] == 0) continue;
    const int y = (int)(q / d.W), x = (int)(q - (long long)y * d.W);
    {
      const float* p = a.up + d.up_off + y * d.up_sr + x * d.up_sc;
      const double px = p[0], py = p[d.up_sk];
      if (up_usable(px, py)) {
        const double ex = cx - ((double)x + 0.5), ey = cy - ((double)y + 0.5);
        const double ux = -sr * ce * F + se * ex, uy = -cr * ce * F + se * ey;
        const double u2 = ux * ux + uy * uy;
        if (u2 > 0.0) {
          const double r = atan2(ux * py - uy * px, ux * px + uy * py);
          // r = angle(p) - angle(u):  dr = -(ux duy - uy dux) / |u|^2
          double dux[P], duy[P], J[P];
          dux[0] = -cr * ce * F;          duy[0] = sr * ce * F;
          dux[1] = sr * se * F + ce * ex; duy[1] = cr * se * F + ce * ey;
          dux[2] = -sr * ce * F;          duy[2] = -cr * ce * F;
          if constexpr (P == 5) { dux[3] = se * Wd; duy[3] = 0.0; dux[4] = 0.0; duy[4] = se * Hd; }
          const double iu2 = 1.0 / u2;
#pragma unroll
          for (int k = 0; k < P; ++k) J[k] = -(ux * duy[k] - uy * dux[k]) * iu2;
          fit_accumulate<P>(acc, r, J, a.huber);
        }
      }
    }
    {
      const double lp = a.lat[d.lat_off + q];
      if (isfinite(lp)) {
        const double dx = x == d.W - 1 ? x1 : fma((double)x, sxg, x0), dy = y == d.H - 1 ? y1 : fma((double)y, syg, y0);
        const double xx = dx * rF, yy = dy * rF;
        const double xw = xx * cr - yy * sr;
        const double yw = xx * (ce * sr) + yy * (ce * cr) - se;
        const double zw = xx * (se * sr) + yy * (se * cr) + ce;
        const double h = sqrt(xw * xw + zw * zw);
        const double r = lp * (kPi / 180.0) + atan2(yw, h);
        // l = -atan2(yw, h), |ray|^2 = n2:  dl = -(dyw - yw (x dx + y dy) / n2) / h;  J = -dl
        const double c = yw / (1.0 + xx * xx + yy * yy), ih = 1.0 / h;
        double J[P];
        J[0] = (xx * (ce * cr) - yy * (ce * sr)) * ih;
        J[1] = (-xx * (se * sr) - yy * (se * cr) - ce) * ih;
        J[2] = (-(yw + se) + c * (xx * xx + yy * yy)) * ih;
        if constexpr (P == 5) {
          J[3] = (-(Wd * rF) * (ce * sr) + c * xx * (Wd * rF)) * ih;
          J[4] = (-(Hd * rF) * (ce * cr) + c * yy * (Hd * rF)) * ih;
        }
        fit_accumulate<P>(acc, r, J, a.huber);
      }
    }
  }
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int q = 0; q < NQ; ++q) {
    double v = acc[q];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
    if (lane == 0) shq[warp][q] = v;
  }
  __syncthreads();
  if (threadIdx.x < NQ) {
    double v = 0.0;
#pragma unroll
    for (int w = 0; w < kFitThreads / 32; ++w) v += shq[w][threadIdx.x];
    a.part[(long long)threadIdx.x * a.nblocks + blockIdx.x] = v;
  }
}

// ------------------------------------------------------------------------------------------------------------ step
__device__ __forceinline__ double wrap_pi(double v) {   // into (-pi, pi]
  return v - 2.0 * kPi * ceil((v - kPi) / (2.0 * kPi));
}

// (M) x = b for a P x P symmetric matrix given as its upper triangle (row by row); false if M is not positive definite
template <int P>
__device__ __forceinline__ bool cholesky_solve(const double (&M)[P * (P + 1) / 2], const double (&b)[P], double (&x)[P]) {
  double L[P][P];
  auto up = [&](int i, int j) {   // M[i][j], i <= j
    return M[i * P - i * (i - 1) / 2 + (j - i)];
  };
  for (int i = 0; i < P; ++i) {
    for (int j = 0; j <= i; ++j) {
      double s = up(j, i);
      for (int k = 0; k < j; ++k) s -= L[i][k] * L[j][k];
      if (i == j) {
        if (!(s > 0.0)) return false;
        L[i][i] = sqrt(s);
      } else {
        L[i][j] = s / L[j][j];
      }
    }
  }
  double y[P];
  for (int i = 0; i < P; ++i) {
    double s = b[i];
    for (int k = 0; k < i; ++k) s -= L[i][k] * y[k];
    y[i] = s / L[i][i];
  }
  for (int i = P - 1; i >= 0; --i) {
    double s = y[i];
    for (int k = i + 1; k < P; ++k) s -= L[k][i] * x[k];
    x[i] = s / L[i][i];
  }
  return true;
}

template <int P>
__device__ void fit_finish(const FitArgs& a, int i, FitState& s, int status) {
  double* o = a.params + 5LL * i;
  if (status == 2) {
    for (int k = 0; k < 5; ++k) o[k] = NAN;
    a.cost[i] = NAN;
  } else {
    double r = s.theta[0], e = wrap_pi(s.theta[1]);
    if (fabs(e) > kPi / 2.0) { e = wrap_pi(kPi - e); r += kPi; }   // (r + pi, pi - e) draws the same fields
    r = wrap_pi(r);
    o[0] = r * (180.0 / kPi); o[1] = e * (180.0 / kPi); o[2] = exp(s.theta[2]); o[3] = s.theta[3]; o[4] = s.theta[4];
    a.cost[i] = s.C;
  }
  a.iters[i] = s.evals;
  a.status[i] = status;
  s.status = status;
}

// One warp per image: the partials of its last pass summed in a fixed order (lane-strided serial sums, then a shuffle tree),
// then lane 0 runs one step of the loop.
template <int P>
__global__ void __launch_bounds__(32 * kFitStepWarps) fit_step_kernel(FitArgs a) {
  constexpr int NQ = fit_nq(P), NA = P * (P + 1) / 2;
  pdl_wait();
  pdl_launch();
  const int lane = threadIdx.x & 31;
  const int i = blockIdx.x * kFitStepWarps + (threadIdx.x >> 5);
  if (i >= a.n) return;
  FitState& s = a.st[i];
  if (s.status != kFitRunning) return;
  const FitImage d = a.im[i];
  double v[NQ];
#pragma unroll
  for (int q = 0; q < NQ; ++q) {
    double t = 0.0;
    for (int b = lane; b < d.nblk; b += 32) t += a.part[(long long)q * a.nblocks + d.block0 + b];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) t += __shfl_down_sync(0xffffffffu, t, o);
    v[q] = t;
  }
  if (lane != 0) return;
  const double Cc = 0.5 * v[0];
  s.evals += 1;
  if (s.evals == 1) {   // the start
    bool bad = v[1] < (double)P;
    for (int k = 0, q = 0; k < P; q += P - k, ++k) bad = bad || v[2 + P + q] == 0.0;   // diagonal of A
    if (bad) { fit_finish<P>(a, i, s, 2); return; }
    s.C = Cc;
    for (int k = 0; k < P; ++k) { s.theta[k] = s.cand[k]; s.g[k] = v[2 + k]; }
    for (int k = 0; k < NA; ++k) s.A[k] = v[2 + P + k];
  } else if (Cc < s.C) {   // accept
    const bool done = s.C - Cc <= kFitCostRtol * s.C;
    s.C = Cc;
    for (int k = 0; k < P; ++k) { s.theta[k] = s.cand[k]; s.g[k] = v[2 + k]; }
    for (int k = 0; k < NA; ++k) s.A[k] = v[2 + P + k];
    s.lambda /= 10.0;
    if (done) { fit_finish<P>(a, i, s, 0); return; }
  } else {                 // reject: keep theta, A, g
    s.lambda *= 10.0;
    if (s.lambda > kFitLambdaMax) { fit_finish<P>(a, i, s, 0); return; }
  }
  double M[NA], g[P], delta[P];
  for (int k = 0; k < P; ++k) g[k] = -s.g[k];
  bool ok = false;
  while (s.lambda <= kFitLambdaMax) {
    for (int k = 0; k < NA; ++k) M[k] = s.A[k];
    for (int k = 0, q = 0; k < P; q += P - k, ++k) M[q] = s.A[q] + s.lambda * s.A[q];
    if ((ok = cholesky_solve<P>(M, g, delta))) break;
    s.lambda *= 10.0;
  }
  if (!ok) { fit_finish<P>(a, i, s, 0); return; }
  bool small = true;
  for (int k = 0; k < P; ++k) small = small && fabs(delta[k]) <= kFitStepRtol * (1.0 + fabs(s.theta[k]));
  if (small) { fit_finish<P>(a, i, s, 0); return; }
  if (s.evals >= a.max_iter) { fit_finish<P>(a, i, s, 1); return; }
  for (int k = 0; k < P; ++k) s.cand[k] = s.theta[k] + delta[k];
}

}  // namespace pf
