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
// f_scale = delta: rho(z) = z, or Huber's 2 sqrt(z) - 1 above 1), IRLS weights w = rho'.  With per-residual weights v (maps of
// the up and latitude residuals, pf_fit_camera_weighted) a residual also needs a finite v > 0; it adds v delta^2 rho to 2 C and
// has the IRLS weight v rho' (the Huber threshold applies to the unweighted r).
//
// Three kernels, chained with programmatic dependent launch and enqueued without synchronisation: fit_init_kernel (the
// start), then max_iterations pairs of fit_pass_kernel (one cost evaluation: C, A = sum w J^T J and g = sum w J^T r at the
// candidate, as per-block fp64 partials) and fit_step_kernel (reduce the partials in a fixed order, accept or reject, solve the
// damped normal equations by Cholesky, write the next candidate or the result).  Images that have stopped cost their pass
// blocks one early exit.  No floating-point atomic decides a value: repeated calls are bit-identical.
//
// Groups of images with shared intrinsics (pf_fit_camera_groups, "shared intrinsics" below) reuse the start and the pass, and
// replace the step by fit_reduce_kernel (each image's sums) and fit_group_step_kernel (one Schur-complement step per group).
//
// Panorama levelling (pf_fit_panorama, "panorama levelling" below) fits one tilt to all views cropped from a panorama: the pass
// in terms of each view's world up direction v (fit_pass_kernel<3, kW, true>), fit_reduce_kernel, then fit_pano_step_kernel.
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
  long long uw_off, lw_off;                // weights of the up / latitude residuals, [H, W] row-major floats; -1: none
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
  const float* wt;            // base of the weight maps (FitImage::uw_off / lw_off)
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

// A residual weight that keeps its residual: finite and > 0 (NaN, infinities, zero and negative weights drop it)
__device__ __forceinline__ bool weight_usable(float w) { return w > 0.0f && w < INFINITY; }

// Weight of pixel q of a [H, W] weight map at off (-1: none, weight 1); 0 when unusable (the residual is dropped)
__device__ __forceinline__ double fit_weight(const FitArgs& a, long long off, long long q) {
  if (off < 0) return 1.0;
  const float t = a.wt[off + q];
  return weight_usable(t) ? (double)t : 0.0;
}

// ------------------------------------------------------------------------------------------------------------ start
// One block of 64 threads per image, one thread per pixel of the 8 x 8 window of rows H/2 - 4 .. H/2 + 3 and the same columns
// around W/2 (clipped to the image):
//   roll0 = atan2(-sum px^, -sum py^) of the unit predictions (at the principal point up = (-sin r, -cos r));
//   pitch0 = the window's mean latitude (latitude = pitch at the principal point);
//   f0 = 1 / (H mean |grad l|), central differences where the four neighbours are valid (|grad l| = 1 / F there).
// A term without a valid pixel falls back to roll 0, pitch 0, vfov 60 degrees.  With weights, a pixel counts for the roll term only
// where its up weight is usable, for the pitch and gradient terms (the four neighbours included) only where its latitude weight is.
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
      auto okl = [&](int yy, int xx) { return ok(yy, xx) && (d.lw_off < 0 || weight_usable(a.wt[d.lw_off + (long long)yy * d.W + xx])); };
      auto lat = [&](int yy, int xx) { return (double)a.lat[d.lat_off + (long long)yy * d.W + xx] * (kPi / 180.0); };
      if (ok(y, x)) {
        const float* p = a.up + d.up_off + y * d.up_sr + x * d.up_sc;
        const double px = p[0], py = p[d.up_sk];
        if (up_usable(px, py) && (d.uw_off < 0 || weight_usable(a.wt[d.uw_off + (long long)y * d.W + x]))) {
          const double nn = sqrt(px * px + py * py);
          sx = px / nn; sy = py / nn; nu = 1;
        }
        const double l0 = lat(y, x);
        if (isfinite(l0) && okl(y, x)) {
          sl = l0; nl = 1;
          if (y > 0 && y < d.H - 1 && x > 0 && x < d.W - 1 && okl(y, x + 1) && okl(y, x - 1) && okl(y + 1, x) && okl(y - 1, x)) {
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
// kW: the residual has weight v (> 0, finite): v c and v w in place of c and w.  Both products are exact for v = 1, and so is
// the fused v c + acc[0] the compiler makes of the first: unit weights add the unweighted terms bit for bit.
template <int P, bool kW = false>
__device__ __forceinline__ void fit_accumulate(double (&acc)[fit_nq(P)], double r, const double (&J)[P], double huber, double v = 1.0) {
  const double ar = fabs(r);
  double c = r * r, w = 1.0;
  if (huber > 0.0 && ar > huber) { c = 2.0 * huber * ar - huber * huber; w = huber / ar; }
  if constexpr (kW) { c = v * c; w = v * w; }
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
// count, 2 .. 1 + P = g, then A's upper triangle row by row.  kW: the launch has weight maps (an image without one has v = 1).
// kV (P = 3, the panorama fit below): the model in terms of the world up direction v in camera coordinates, cand[0 .. 2] = v,
// with fixed intrinsics F = init[2] (pixels), cx = (init[3] + 1/2) W, cy = (init[4] + 1/2) H; g and A are taken with respect to v.
template <int P, bool kW = false, bool kV = false>
__global__ void __launch_bounds__(kFitThreads) fit_pass_kernel(FitArgs a) {
  static_assert(!kV || P == 3, "the v model has three parameters");
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
  const double F = kV ? d.init[2] : exp(th[2]) * d.H;
  const double cx = ((kV ? d.init[3] : th[3]) + 0.5) * d.W, cy = ((kV ? d.init[4] : th[4]) + 0.5) * d.H;
  double sr = 0.0, cr = 0.0, se = 0.0, ce = 0.0;
  if constexpr (!kV) {
    sincos(th[0], &sr, &cr);
    sincos(th[1], &se, &ce);
  }
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
    // (the weighted instantiation computes each residual and its Jacobian row in the same blocks as the unweighted one and only
    // then reads the weight, so that the compiler makes the same instructions of them: unit weights and 0 / 1 weight maps give
    // the unweighted and the masked sums bit for bit)
    {
      const float* p = a.up + d.up_off + y * d.up_sr + x * d.up_sc;
      const double px = p[0], py = p[d.up_sk];
      if (up_usable(px, py)) {
        const double ex = cx - ((double)x + 0.5), ey = cy - ((double)y + 0.5);
        double ux, uy;
        if constexpr (kV) { ux = F * th[0] + th[2] * ex; uy = F * th[1] + th[2] * ey; }
        else { ux = -sr * ce * F + se * ex; uy = -cr * ce * F + se * ey; }
        const double u2 = ux * ux + uy * uy;
        if (u2 > 0.0) {
          const double r = atan2(ux * py - uy * px, ux * px + uy * py);
          // r = angle(p) - angle(u):  dr = -(ux duy - uy dux) / |u|^2
          double dux[P], duy[P], J[P];
          if constexpr (kV) {   // u = F (vx, vy) + vz (ex, ey)
            dux[0] = F;   duy[0] = 0.0;
            dux[1] = 0.0; duy[1] = F;
            dux[2] = ex;  duy[2] = ey;
          } else {
            dux[0] = -cr * ce * F;          duy[0] = sr * ce * F;
            dux[1] = sr * se * F + ce * ex; duy[1] = cr * se * F + ce * ey;
            dux[2] = -sr * ce * F;          duy[2] = -cr * ce * F;
          }
          if constexpr (P == 5) { dux[3] = se * Wd; duy[3] = 0.0; dux[4] = 0.0; duy[4] = se * Hd; }
          const double iu2 = 1.0 / u2;
#pragma unroll
          for (int k = 0; k < P; ++k) J[k] = -(ux * duy[k] - uy * dux[k]) * iu2;
          if constexpr (kW) {
            const double v = fit_weight(a, d.uw_off, q);
            if (v > 0.0) fit_accumulate<P, true>(acc, r, J, a.huber, v);
          } else {
            fit_accumulate<P>(acc, r, J, a.huber);
          }
        }
      }
    }
    {
      const double lp = a.lat[d.lat_off + q];
      if (isfinite(lp)) {
        const double dx = x == d.W - 1 ? x1 : fma((double)x, sxg, x0), dy = y == d.H - 1 ? y1 : fma((double)y, syg, y0);
        const double xx = dx * rF, yy = dy * rF;
        if constexpr (kV) {
          // l = atan2(v . c, |v x c|) for the ray c = (xx, yy, 1); along the sphere dl = c . dv / |v x c|, J = -dl
          const double s = th[0] * xx + th[1] * yy + th[2];
          const double qx = th[1] - th[2] * yy, qy = th[2] * xx - th[0], qz = th[0] * yy - th[1] * xx;
          const double h = sqrt(qx * qx + qy * qy + qz * qz), ih = 1.0 / h;
          const double r = lp * (kPi / 180.0) - atan2(s, h);
          const double J[P] = {-xx * ih, -yy * ih, -ih};
          if constexpr (kW) {
            const double v = fit_weight(a, d.lw_off, q);
            if (v > 0.0) fit_accumulate<P, true>(acc, r, J, a.huber, v);
          } else {
            fit_accumulate<P>(acc, r, J, a.huber);
          }
          continue;
        }
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
        if constexpr (kW) {
          const double v = fit_weight(a, d.lw_off, q);
          if (v > 0.0) fit_accumulate<P, true>(acc, r, J, a.huber, v);
        } else {
          fit_accumulate<P>(acc, r, J, a.huber);
        }
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

// The partials of image d's last pass summed in a fixed order by one warp: lane-strided serial sums, then a shuffle tree.
// Lane 0 holds the NQ sums.
template <int P>
__device__ __forceinline__ void fit_reduce_partials(const FitArgs& a, const FitImage& d, int lane, double (&v)[fit_nq(P)]) {
#pragma unroll
  for (int q = 0; q < fit_nq(P); ++q) {
    double t = 0.0;
    for (int b = lane; b < d.nblk; b += 32) t += a.part[(long long)q * a.nblocks + d.block0 + b];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) t += __shfl_down_sync(0xffffffffu, t, o);
    v[q] = t;
  }
}

// One warp per image: the partials of its last pass summed (fit_reduce_partials), then lane 0 runs one step of the loop.
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
  fit_reduce_partials<P>(a, d, lane, v);
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

// ------------------------------------------------------------------------------------------------------ shared intrinsics
// Groups of images from one camera (DESIGN.md section 1, "Shared intrinsics"): per-image roll and pitch, one s = ln f_rel (and
// cx_rel, cy_rel with principal_point) per group.  The pass is fit_pass_kernel's; fit_reduce_kernel writes each running
// image's sums, and fit_group_step_kernel (one block per group) takes one Levenberg-Marquardt step on the group's joint
// normal equations by a Schur complement on the shared parameters.  An image's FitState keeps its own theta (the shared
// entries equal the group's, bit for bit), A, g and C_i at the accepted point; status 2 marks a dropped member.
constexpr int kFitGroupThreads = 256;

struct FitGroupState {
  double shared[3], cand[3];   // accepted (s, cx_rel, cy_rel) and the candidate's
  double C, lambda;            // C_G at the accepted point
  int evals, status;           // cost evaluations of the group so far; kFitRunning, or the group's final status
};
struct FitGroups {
  const int* off;              // [ngroups + 1]: group G's members are mem[off[G] .. off[G + 1] - 1]
  const int* mem;              // [n] image indices, in index order within each group
  FitGroupState* gs;           // [ngroups]
  double* sums;                // [n][kFitQ]: each running image's sums of its last pass
  int ngroups;
};

// Entry (i, j), i <= j, of a P x P upper triangle stored row by row
__host__ __device__ constexpr int fit_up(int P, int i, int j) { return i * P - i * (i - 1) / 2 + (j - i); }

// Deterministic block sum of N values per thread (fixed shuffle trees, then the warps' partials in warp order); every thread
// gets the same bits.  sh: [blockDim.x / 32][N] doubles in shared memory.
template <int N>
__device__ __forceinline__ void fit_block_sum(double (&v)[N], double* sh) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
#pragma unroll
  for (int q = 0; q < N; ++q)
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v[q] += __shfl_down_sync(0xffffffffu, v[q], o);
  __syncthreads();   // sh may still be read by the previous call
  if (lane == 0)
#pragma unroll
    for (int q = 0; q < N; ++q) sh[warp * N + q] = v[q];
  __syncthreads();
#pragma unroll
  for (int q = 0; q < N; ++q) {
    double t = sh[q];
    for (int w = 1; w < nw; ++w) t += sh[w * N + q];
    v[q] = t;
  }
}

// The damped local block B = A[ll] + lambda diag A[ll] of one image by Cholesky, kept as L's off-diagonal entry and the
// reciprocals of its diagonal (two divisions per factorisation, none per solve): false if B is not positive definite
struct FitLocal {
  double r00, l10, r11;
  __device__ __forceinline__ bool factor(const double* A, int P, double lambda) {
    return factor2(A[0] + lambda * A[0], A[1], A[P] + lambda * A[P]);
  }
  __device__ __forceinline__ bool factor2(double b00, double b01, double b11) {   // B given by its entries
    if (!(b00 > 0.0)) return false;
    r00 = 1.0 / sqrt(b00);
    l10 = b01 * r00;
    const double t = b11 - l10 * l10;
    if (!(t > 0.0)) return false;
    r11 = 1.0 / sqrt(t);
    return true;
  }
  __device__ __forceinline__ void solve(double b0, double b1, double& x0, double& x1) const {   // B x = b
    const double y0 = b0 * r00, y1 = (b1 - l10 * y0) * r11;
    x1 = y1 * r11;
    x0 = (y0 - l10 * x1) * r00;
  }
};

// One thread per group: the shared entries of the start are the mean, in index order, of the members' starts
__global__ void __launch_bounds__(128) fit_group_init_kernel(FitArgs a, FitGroups g) {
  pdl_wait();
  pdl_launch();
  const int G = blockIdx.x * blockDim.x + threadIdx.x;
  if (G >= g.ngroups) return;
  const int m0 = g.off[G], m1 = g.off[G + 1];
  double sh[3];
  for (int k = 0; k < 3; ++k) {
    double t = a.st[g.mem[m0]].cand[2 + k];
    for (int j = m0 + 1; j < m1; ++j) t += a.st[g.mem[j]].cand[2 + k];
    sh[k] = t / (double)(m1 - m0);
  }
  for (int j = m0; j < m1; ++j) {
    FitState& s = a.st[g.mem[j]];
    for (int k = 0; k < 3; ++k) s.cand[2 + k] = s.theta[2 + k] = sh[k];
  }
  FitGroupState& gs = g.gs[G];
  for (int k = 0; k < 3; ++k) gs.shared[k] = gs.cand[k] = sh[k];
  gs.C = 0.0; gs.lambda = kFitLambda0; gs.evals = 0; gs.status = kFitRunning;
}

// One warp per image: the sums of a running image's last pass (fit_reduce_partials) into g.sums
template <int P>
__global__ void __launch_bounds__(32 * kFitStepWarps) fit_reduce_kernel(FitArgs a, FitGroups g) {
  constexpr int NQ = fit_nq(P);
  pdl_wait();
  pdl_launch();
  const int lane = threadIdx.x & 31;
  const int i = blockIdx.x * kFitStepWarps + (threadIdx.x >> 5);
  if (i >= a.n || a.st[i].status != kFitRunning) return;
  const FitImage d = a.im[i];
  double v[NQ];
  fit_reduce_partials<P>(a, d, lane, v);
  if (lane == 0)
#pragma unroll
    for (int q = 0; q < NQ; ++q) g.sums[(long long)i * kFitQ + q] = v[q];
}

// One block per group: accept or reject the candidate on C_G, then solve (A + lambda diag A) delta = -g over the group's
// parameters (locals l = roll, pitch of each member; shared s = K entries) by a Schur complement on the shared block:
//   S = D_lambda - sum E_i^T B_i^-1 E_i,  b = -g_s + sum E_i^T B_i^-1 g_l,i,  S ds = b,  dl_i = B_i^-1 (-g_l,i - E_i ds).
// Each thread takes members off[G] + threadIdx.x, + blockDim.x, ...; the sums over members are fixed-order block sums, and
// every thread solves the K x K system on the same bits.
template <int P>
__global__ void __launch_bounds__(kFitGroupThreads, 1) fit_group_step_kernel(FitArgs a, FitGroups g) {
  constexpr int K = P - 2, NK = K * (K + 1) / 2;
  constexpr int OD = 0, OG = NK, OS = NK + K, OB = 2 * NK + K, OF = 2 * NK + 2 * K, NR = OF + 1;   // sums of the lambda loop
  __shared__ double shr[kFitGroupThreads / 32 * NR];
  pdl_wait();
  pdl_launch();
  FitGroupState& gs = g.gs[blockIdx.x];
  if (gs.status != kFitRunning) return;
  const int m0 = g.off[blockIdx.x], m1 = g.off[blockIdx.x + 1];
  const int evals = gs.evals + 1;
  double lambda = gs.lambda, C = gs.C, th[K], cs[K];
#pragma unroll
  for (int c = 0; c < K; ++c) { th[c] = gs.shared[c]; cs[c] = gs.cand[c]; }
  auto accept = [&](FitState& s, const double* v) {
    s.C = 0.5 * v[0];
#pragma unroll
    for (int k = 0; k < P; ++k) { s.theta[k] = s.cand[k]; s.g[k] = v[2 + k]; }
#pragma unroll
    for (int k = 0; k < P * (P + 1) / 2; ++k) s.A[k] = v[2 + P + k];
  };
  // One step; returns the group's final status, or kFitRunning.  gs is written only after the first block sum, when every
  // thread has read it.
  const int status = [&]() -> int {
    if (evals == 1) {   // the start: drop members without a usable local block, then check what is left
      double r[3 + K] = {};   // residuals, C_G, members kept, diag D
      for (int j = m0 + (int)threadIdx.x; j < m1; j += blockDim.x) {
        const int i = g.mem[j];
        FitState& s = a.st[i];
        const double* v = g.sums + (long long)i * kFitQ;
        if (v[1] < 2.0 || v[2 + P + fit_up(P, 0, 0)] == 0.0 || v[2 + P + fit_up(P, 1, 1)] == 0.0) { s.status = 2; continue; }
        r[0] += v[1]; r[1] += 0.5 * v[0]; r[2] += 1.0;
#pragma unroll
        for (int c = 0; c < K; ++c) r[3 + c] += v[2 + P + fit_up(P, 2 + c, 2 + c)];
        accept(s, v);
      }
      fit_block_sum<3 + K>(r, shr);
      bool bad = r[2] == 0.0 || r[0] < 2.0 * r[2] + K;
#pragma unroll
      for (int c = 0; c < K; ++c) bad = bad || r[3 + c] == 0.0;
      if (bad) return 2;
      C = r[1];
    } else {
      double r[1] = {0.0};
      for (int j = m0 + (int)threadIdx.x; j < m1; j += blockDim.x) {
        const int i = g.mem[j];
        if (a.st[i].status == kFitRunning) r[0] += 0.5 * g.sums[(long long)i * kFitQ];
      }
      fit_block_sum<1>(r, shr);
      if (r[0] < C) {   // accept
        const bool done = C - r[0] <= kFitCostRtol * C;
        C = r[0];
        for (int j = m0 + (int)threadIdx.x; j < m1; j += blockDim.x) {
          const int i = g.mem[j];
          FitState& s = a.st[i];
          if (s.status == kFitRunning) accept(s, g.sums + (long long)i * kFitQ);
        }
#pragma unroll
        for (int c = 0; c < K; ++c) th[c] = cs[c];
        lambda /= 10.0;
        if (done) return 0;
      } else {          // reject: keep theta, A, g
        lambda *= 10.0;
        if (lambda > kFitLambdaMax) return 0;
      }
    }
    double ds[K];
    bool ok = false;
    while (lambda <= kFitLambdaMax) {
      double r[NR] = {};   // D (upper triangle), g_s, sum E^T B^-1 E (upper triangle), sum E^T B^-1 g_l, members with B not PD
      for (int j = m0 + (int)threadIdx.x; j < m1; j += blockDim.x) {
        const FitState& s = a.st[g.mem[j]];
        if (s.status != kFitRunning) continue;
#pragma unroll
        for (int c = 0, q = 0; c < K; ++c) {
          r[OG + c] += s.g[2 + c];
#pragma unroll
          for (int e = c; e < K; ++e, ++q) r[OD + q] += s.A[fit_up(P, 2 + c, 2 + e)];
        }
        FitLocal B;
        if (!B.factor(s.A, P, lambda)) { r[OF] += 1.0; continue; }
        double X0[K], X1[K], y0, y1;
        B.solve(s.g[0], s.g[1], y0, y1);
#pragma unroll
        for (int c = 0; c < K; ++c) B.solve(s.A[fit_up(P, 0, 2 + c)], s.A[fit_up(P, 1, 2 + c)], X0[c], X1[c]);
#pragma unroll
        for (int c = 0, q = 0; c < K; ++c) {
          const double e0 = s.A[fit_up(P, 0, 2 + c)], e1 = s.A[fit_up(P, 1, 2 + c)];
          r[OB + c] += e0 * y0 + e1 * y1;
#pragma unroll
          for (int e = c; e < K; ++e, ++q) r[OS + q] += e0 * X0[e] + e1 * X1[e];
        }
      }
      fit_block_sum<NR>(r, shr);
      if (r[OF] == 0.0) {
        double S[NK], b[K];
#pragma unroll
        for (int c = 0, q = 0; c < K; ++c) {
          b[c] = -r[OG + c] + r[OB + c];
#pragma unroll
          for (int e = c; e < K; ++e, ++q) S[q] = (e == c ? r[OD + q] + lambda * r[OD + q] : r[OD + q]) - r[OS + q];
        }
        if ((ok = cholesky_solve<K>(S, b, ds))) break;
      }
      lambda *= 10.0;
    }
    if (!ok) return 0;
    double big[1] = {0.0};   // members with a local step above the tolerance
    for (int j = m0 + (int)threadIdx.x; j < m1; j += blockDim.x) {
      FitState& s = a.st[g.mem[j]];
      if (s.status != kFitRunning) continue;
      FitLocal B;
      B.factor(s.A, P, lambda);   // positive definite: the same bits passed above
      double b0 = -s.g[0], b1 = -s.g[1], x0, x1;
#pragma unroll
      for (int c = 0; c < K; ++c) { b0 -= s.A[fit_up(P, 0, 2 + c)] * ds[c]; b1 -= s.A[fit_up(P, 1, 2 + c)] * ds[c]; }
      B.solve(b0, b1, x0, x1);
      if (!(fabs(x0) <= kFitStepRtol * (1.0 + fabs(s.theta[0])) && fabs(x1) <= kFitStepRtol * (1.0 + fabs(s.theta[1])))) big[0] += 1.0;
      s.cand[0] = s.theta[0] + x0; s.cand[1] = s.theta[1] + x1;
#pragma unroll
      for (int c = 0; c < K; ++c) s.cand[2 + c] = th[c] + ds[c];
    }
    fit_block_sum<1>(big, shr);
    bool small = big[0] == 0.0;
#pragma unroll
    for (int c = 0; c < K; ++c) small = small && fabs(ds[c]) <= kFitStepRtol * (1.0 + fabs(th[c]));
    if (small) return 0;
    if (evals >= a.max_iter) return 1;
    if (threadIdx.x == 0) {
#pragma unroll
      for (int c = 0; c < K; ++c) { gs.shared[c] = th[c]; gs.cand[c] = th[c] + ds[c]; }
      gs.C = C; gs.lambda = lambda; gs.evals = evals;
    }
    return kFitRunning;
  }();
  if (status == kFitRunning) return;
  for (int j = m0 + (int)threadIdx.x; j < m1; j += blockDim.x) {   // finish: every member, dropped ones with status 2
    const int i = g.mem[j];
    FitState& s = a.st[i];
    s.evals = evals;
    fit_finish<P>(a, i, s, s.status == 2 ? 2 : status);
  }
  if (threadIdx.x == 0) { gs.evals = evals; gs.status = status; }
}

// ------------------------------------------------------------------------------------------------------ camera tracks
// Sequences of evenly spaced video frames (DESIGN.md section 1, "Camera tracks"): the grouped fit's parameters and residuals,
// each frame's cost divided by its residual count M_t (fixed: validity does not depend on theta), plus a random-walk prior
// 1/2 sum_t ((r_t+1 - r_t) / sr)^2 + ((e_t+1 - e_t) / se)^2 on neighbouring frames (the angles in radians, sr and se the numbers
// given in degrees).  The start is fit_group_init_kernel's, then fit_seq_init_kernel unwraps the roll starts along each
// sequence; the pass and fit_reduce_kernel are reused, and fit_seq_step_kernel takes one Levenberg-Marquardt step per sequence.
// A frame's FitState keeps its own C_t (unscaled), theta, and A / M_t, g / M_t at the accepted point (zero when M_t = 0).
constexpr int kFitSeqRow = 22;   // per-frame workspace doubles: B (3), E (2 K), g_l (2), the pivot's factor (3), z (2 (K + 1))

struct FitSeqs {
  FitGroups g;                   // the sequences as groups: members in frame order, state, each frame's sums
  double* work;                  // [n][kFitSeqRow], row j for the member at position j of g.mem
  double wr, we;                 // prior weights 1 / sr^2, 1 / se^2
};

// One thread per sequence: each roll start moved by a multiple of 2 pi to within pi of its (moved) predecessor's
__global__ void __launch_bounds__(128) fit_seq_init_kernel(FitArgs a, FitSeqs q) {
  pdl_wait();
  pdl_launch();
  const int G = blockIdx.x * blockDim.x + threadIdx.x;
  if (G >= q.g.ngroups) return;
  double prev = a.st[q.g.mem[q.g.off[G]]].theta[0];
  for (int j = q.g.off[G] + 1; j < q.g.off[G + 1]; ++j) {
    FitState& s = a.st[q.g.mem[j]];
    const double r = s.theta[0] - 2.0 * kPi * rint((s.theta[0] - prev) / (2.0 * kPi));
    s.theta[0] = s.cand[0] = r;
    prev = r;
  }
}

// One block per sequence.  Accept or reject the candidate on C_S, then solve (A + lambda diag A) delta = -g: the locals form a
// block-tridiagonal matrix T (diagonal blocks A_t[ll] / M_t + the prior's W = diag(wr, we) once per neighbour, off-diagonal
// blocks -W), eliminated from the K shared unknowns by a Schur complement.  The block threads prepare each frame's row (B_t,
// E_t = A_t[ls] / M_t, g_l,t with the prior's gradient) and the fixed-order block sums D and g_s; thread 0 then runs the block
// LDL^T recursion along the chain with K + 1 right-hand sides (g_l, E):
//   P_0 = B_0,  P_t = B_t - W P_t-1^-1 W,  z_t = rhs_t + W P_t-1^-1 z_t-1,  rhs^T T^-1 rhs' = sum_t z_t^T P_t^-1 z'_t,
// solves S ds = b with S = D_lambda - E^T T^-1 E, b = -g_s + E^T T^-1 g_l, and sweeps back dl_t = P_t^-1 (z'_t + W dl_t+1)
// with z'_t = -z_g,t - Z_t ds.
template <int P>
__global__ void __launch_bounds__(kFitGroupThreads, 1) fit_seq_step_kernel(FitArgs a, FitSeqs q) {
  constexpr int K = P - 2, NK = K * (K + 1) / 2, NA = P * (P + 1) / 2;
  constexpr int RB = 0, RE = 3, RG = 3 + 2 * K, RF = 5 + 2 * K, RZ = 8 + 2 * K;   // row offsets
  static_assert(RZ + 2 * (K + 1) <= kFitSeqRow, "row too short");
  constexpr int NC = 2 + K, NS = NK + K, NSH = NC > NS ? NC : NS;   // the two block sums' widths, the scratch's
  __shared__ double shr[kFitGroupThreads / 32 * NSH];
  __shared__ int sh_status;
  pdl_wait();
  pdl_launch();
  const FitGroups& g = q.g;
  FitGroupState& gs = g.gs[blockIdx.x];
  if (gs.status != kFitRunning) return;
  const int m0 = g.off[blockIdx.x], m1 = g.off[blockIdx.x + 1], m = m1 - m0;
  const int evals = gs.evals + 1;
  const double wr = q.wr, we = q.we;
  double lambda = gs.lambda, C = gs.C, th[K], cs[K];
#pragma unroll
  for (int c = 0; c < K; ++c) { th[c] = gs.shared[c]; cs[c] = gs.cand[c]; }
  auto accept = [&](FitState& s, const double* v) {   // v: the frame's sums
    const double M = v[1];
    s.C = 0.5 * v[0];
#pragma unroll
    for (int k = 0; k < P; ++k) { s.theta[k] = s.cand[k]; s.g[k] = M > 0.0 ? v[2 + k] / M : 0.0; }
#pragma unroll
    for (int k = 0; k < NA; ++k) s.A[k] = M > 0.0 ? v[2 + P + k] / M : 0.0;
  };
  const int status = [&]() -> int {
    // C_S at the candidate: sum C_t / M_t, plus the prior on the pair (t, t + 1) by the thread of t; at the start also the
    // residual count and D's diagonal
    double r[NC] = {};
    for (int j = m0 + (int)threadIdx.x; j < m1; j += blockDim.x) {
      const double* v = g.sums + (long long)g.mem[j] * kFitQ;
      const double M = v[1];
      if (M > 0.0) r[0] += 0.5 * v[0] / M;
      if (j + 1 < m1) {
        const double dr = a.st[g.mem[j + 1]].cand[0] - a.st[g.mem[j]].cand[0], de = a.st[g.mem[j + 1]].cand[1] - a.st[g.mem[j]].cand[1];
        r[0] += 0.5 * (dr * dr * wr + de * de * we);
      }
      if (evals == 1) {
        r[1] += M;
#pragma unroll
        for (int c = 0; c < K; ++c) r[2 + c] += M > 0.0 ? v[2 + P + fit_up(P, 2 + c, 2 + c)] / M : 0.0;
      }
    }
    static_assert(NC <= NSH, "scratch too small for the cost sum");
    fit_block_sum<NC>(r, shr);
    bool acc = true, done = false;
    if (evals == 1) {   // the start
      bool bad = r[1] < 2.0 + K;
#pragma unroll
      for (int c = 0; c < K; ++c) bad = bad || r[2 + c] == 0.0;
      if (m == 1) {
        const double* v = g.sums + (long long)g.mem[m0] * kFitQ;
        bad = bad || v[2 + P + fit_up(P, 0, 0)] == 0.0 || v[2 + P + fit_up(P, 1, 1)] == 0.0;
      }
      if (bad) return 2;
      C = r[0];
    } else if (r[0] < C) {   // accept
      done = C - r[0] <= kFitCostRtol * C;
      C = r[0];
#pragma unroll
      for (int c = 0; c < K; ++c) th[c] = cs[c];
      lambda /= 10.0;
    } else {                 // reject: keep theta, A, g
      acc = false;
      lambda *= 10.0;
      if (lambda > kFitLambdaMax) return 0;
    }
    if (acc)
      for (int j = m0 + (int)threadIdx.x; j < m1; j += blockDim.x) accept(a.st[g.mem[j]], g.sums + (long long)g.mem[j] * kFitQ);
    if (done) return 0;
    __syncthreads();   // every frame's accepted theta before the prior's gradient reads its neighbours'
    // each frame's row, and the sums D (upper triangle) and g_s
    double r2[NS] = {};
    for (int j = m0 + (int)threadIdx.x; j < m1; j += blockDim.x) {
      const FitState& s = a.st[g.mem[j]];
      double* row = q.work + (long long)j * kFitSeqRow;
      const double nb = (double)((j > m0) + (j + 1 < m1));
      double gl0 = s.g[0], gl1 = s.g[1];
      if (j > m0) { const FitState& o = a.st[g.mem[j - 1]]; gl0 += wr * (s.theta[0] - o.theta[0]); gl1 += we * (s.theta[1] - o.theta[1]); }
      if (j + 1 < m1) { const FitState& o = a.st[g.mem[j + 1]]; gl0 += wr * (s.theta[0] - o.theta[0]); gl1 += we * (s.theta[1] - o.theta[1]); }
      row[RB] = s.A[fit_up(P, 0, 0)] + nb * wr; row[RB + 1] = s.A[fit_up(P, 0, 1)]; row[RB + 2] = s.A[fit_up(P, 1, 1)] + nb * we;
#pragma unroll
      for (int c = 0; c < K; ++c) { row[RE + c] = s.A[fit_up(P, 0, 2 + c)]; row[RE + K + c] = s.A[fit_up(P, 1, 2 + c)]; }
      row[RG] = gl0; row[RG + 1] = gl1;
#pragma unroll
      for (int c = 0, k = 0; c < K; ++c) {
        r2[NK + c] += s.g[2 + c];
#pragma unroll
        for (int e = c; e < K; ++e, ++k) r2[k] += s.A[fit_up(P, 2 + c, 2 + e)];
      }
    }
    static_assert(NS <= NSH, "scratch too small for the D and g_s sums");
    fit_block_sum<NS>(r2, shr);   // (its first barrier also orders the rows before thread 0 reads them)
    if (threadIdx.x == 0) {
      int st = kFitRunning;
      double ds[K];
      bool ok = false;
      while (lambda <= kFitLambdaMax) {
        double S[NK], b[K], up[2][K + 1];
        for (int k = 0; k < NK; ++k) S[k] = 0.0;
        for (int c = 0; c < K; ++c) b[c] = 0.0;
        FitLocal Pp{}, Pt{};
        bool pd = true;
        for (int t = 0; t < m && pd; ++t) {   // forward: factor P_t, z_t, u_t = P_t^-1 z_t
          double* row = q.work + (long long)(m0 + t) * kFitSeqRow;
          double b00 = row[RB] + lambda * row[RB], b01 = row[RB + 1], b11 = row[RB + 2] + lambda * row[RB + 2];
          double z[2][K + 1];
          z[0][0] = row[RG]; z[1][0] = row[RG + 1];
#pragma unroll
          for (int c = 0; c < K; ++c) { z[0][1 + c] = row[RE + c]; z[1][1 + c] = row[RE + K + c]; }
          if (t > 0) {
            double x0, x1, y0, y1;
            Pp.solve(wr, 0.0, x0, x1);   // P_t-1^-1 W, column by column
            Pp.solve(0.0, we, y0, y1);
            b00 -= wr * x0; b01 -= wr * y0; b11 -= we * y1;
#pragma unroll
            for (int k = 0; k <= K; ++k) { z[0][k] += wr * up[0][k]; z[1][k] += we * up[1][k]; }
          }
          if (!(pd = Pt.factor2(b00, b01, b11))) break;
#pragma unroll
          for (int k = 0; k <= K; ++k) Pt.solve(z[0][k], z[1][k], up[0][k], up[1][k]);
#pragma unroll
          for (int c = 0, k = 0; c < K; ++c) {
            b[c] += z[0][1 + c] * up[0][0] + z[1][1 + c] * up[1][0];
#pragma unroll
            for (int e = c; e < K; ++e, ++k) S[k] += z[0][1 + c] * up[0][1 + e] + z[1][1 + c] * up[1][1 + e];
          }
          row[RF] = Pt.r00; row[RF + 1] = Pt.l10; row[RF + 2] = Pt.r11;
#pragma unroll
          for (int k = 0; k <= K; ++k) { row[RZ + k] = z[0][k]; row[RZ + K + 1 + k] = z[1][k]; }
          Pp = Pt;
        }
        if (pd) {
#pragma unroll
          for (int c = 0, k = 0; c < K; ++c) {
            b[c] = -r2[NK + c] + b[c];
#pragma unroll
            for (int e = c; e < K; ++e, ++k) S[k] = (e == c ? r2[k] + lambda * r2[k] : r2[k]) - S[k];
          }
          if ((ok = cholesky_solve<K>(S, b, ds))) break;
        }
        lambda *= 10.0;
      }
      if (!ok) {
        st = 0;
      } else {
        bool small = true;
#pragma unroll
        for (int c = 0; c < K; ++c) small = small && fabs(ds[c]) <= kFitStepRtol * (1.0 + fabs(th[c]));
        double n0 = 0.0, n1 = 0.0;   // W dl_t+1
        for (int t = m - 1; t >= 0; --t) {   // backward: dl_t, the candidate
          const double* row = q.work + (long long)(m0 + t) * kFitSeqRow;
          FitLocal Pf;
          Pf.r00 = row[RF]; Pf.l10 = row[RF + 1]; Pf.r11 = row[RF + 2];
          double z0 = -row[RZ] + n0, z1 = -row[RZ + K + 1] + n1, x0, x1;
#pragma unroll
          for (int c = 0; c < K; ++c) { z0 -= row[RZ + 1 + c] * ds[c]; z1 -= row[RZ + K + 2 + c] * ds[c]; }
          Pf.solve(z0, z1, x0, x1);
          FitState& s = a.st[g.mem[m0 + t]];
          small = small && fabs(x0) <= kFitStepRtol * (1.0 + fabs(s.theta[0])) && fabs(x1) <= kFitStepRtol * (1.0 + fabs(s.theta[1]));
          s.cand[0] = s.theta[0] + x0; s.cand[1] = s.theta[1] + x1;
#pragma unroll
          for (int c = 0; c < K; ++c) s.cand[2 + c] = th[c] + ds[c];
          n0 = wr * x0; n1 = we * x1;
        }
        if (small) st = 0;
        else if (evals >= a.max_iter) st = 1;
        else {
#pragma unroll
          for (int c = 0; c < K; ++c) { gs.shared[c] = th[c]; gs.cand[c] = th[c] + ds[c]; }
          gs.C = C; gs.lambda = lambda; gs.evals = evals;
        }
      }
      sh_status = st;
    }
    __syncthreads();
    return sh_status;
  }();
  if (status == kFitRunning) return;
  for (int j = m0 + (int)threadIdx.x; j < m1; j += blockDim.x) {   // finish every frame
    const int i = g.mem[j];
    FitState& s = a.st[i];
    s.evals = evals;
    fit_finish<P>(a, i, s, status);
  }
  if (threadIdx.x == 0) { gs.evals = evals; gs.status = status; }
}

// ------------------------------------------------------------------------------------------------------ panorama levelling
// Views cropped from one panorama share its tilt (DESIGN.md section 1, "Panorama levelling"): theta = (psi, phi), T = Z(psi) X(phi),
// the panorama's up direction g = T^T n = (-sin psi, -cos psi cos phi, cos psi sin phi) for n = (0, -1, 0), and view k (crop
// rotation A_k) sees the world up direction v_k = A_k^T g.  The pass is fit_pass_kernel<3, kW, true> (sums with respect to v),
// fit_reduce_kernel writes each view's sums, and fit_pano_step_kernel (one warp per panorama) takes one Levenberg-Marquardt step
// on A = sum D_k^T A_k D_k, g = sum D_k^T g_k with D_k = A_k^T dg/dtheta, then writes each member's next v_k.
struct FitPanoState {
  double theta[2], cand[2];   // accepted (psi, phi) and the candidate the next pass evaluates
  double A[3], g[2], C;       // at theta (A: upper triangle)
  double lambda;
  int evals, status;
};
struct FitPanos {
  const int* off;             // [npano + 1]: panorama P's views are mem[off[P] .. off[P + 1] - 1]
  const int* mem;             // [n] view indices, in index order within each panorama
  const double* rot;          // [n][9] A_k row-major
  const double* init;         // [npano][2] start (psi, phi), radians
  FitPanoState* ps;           // [npano]
  double* sums;               // [n][kFitQ]: each view's sums of its last pass (fit_reduce_kernel)
  int npano;
  double* angles; double* up; double* R; double* cost; int* iters; int* status;   // outputs [npano][2], [3], [9], [1] ...
};

// g(theta) and its derivatives dg[m][k] = d g_m / d theta_k
__device__ __forceinline__ void pano_gravity(const double (&th)[2], double (&gv)[3], double (&dg)[3][2]) {
  double sp, cp, sf, cf;
  sincos(th[0], &sp, &cp);
  sincos(th[1], &sf, &cf);
  gv[0] = -sp; gv[1] = -cp * cf; gv[2] = cp * sf;
  dg[0][0] = -cp;      dg[0][1] = 0.0;
  dg[1][0] = sp * cf;  dg[1][1] = cp * sf;
  dg[2][0] = -sp * sf; dg[2][1] = cp * cf;
}

// The member views of panorama P taken by lanes lane, lane + 32, ...: candidate v_k = A_k^T g(th), or the final status
__device__ __forceinline__ void pano_members(const FitArgs& a, const FitPanos& p, int P, int lane, const double (&th)[2], int status) {
  double gv[3], dg[3][2];
  pano_gravity(th, gv, dg);
  for (int j = p.off[P] + lane; j < p.off[P + 1]; j += 32) {
    const int i = p.mem[j];
    FitState& s = a.st[i];
    if (status == kFitRunning) {
      const double* M = p.rot + 9LL * i;
#pragma unroll
      for (int c = 0; c < 3; ++c) s.cand[c] = M[c] * gv[0] + M[3 + c] * gv[1] + M[6 + c] * gv[2];
    }
    s.status = status;
  }
}

// One warp per panorama: the start (init, or psi = phi = 0) and every member's v_k
__global__ void __launch_bounds__(32 * kFitStepWarps) fit_pano_init_kernel(FitArgs a, FitPanos p) {
  pdl_wait();
  pdl_launch();
  const int P = blockIdx.x * kFitStepWarps + (threadIdx.x >> 5);
  if (P >= p.npano) return;
  const double th[2] = {p.init[2 * P], p.init[2 * P + 1]};
  pano_members(a, p, P, threadIdx.x & 31, th, kFitRunning);
  if ((threadIdx.x & 31) == 0) {
    FitPanoState& s = p.ps[P];
    for (int k = 0; k < 2; ++k) s.theta[k] = s.cand[k] = th[k];
    s.C = 0.0; s.lambda = kFitLambda0; s.evals = 0; s.status = kFitRunning;
  }
}

// (psi, phi) -> outputs: the pair with |psi| <= 90 degrees and phi in (-180, 180] ((psi, phi) and (180 - psi, phi + 180) give the
// same g), g, and R = the smallest rotation with R n = g: I cos a + [w]x + w w^T / (1 + cos a) for w = n x g, cos a = n . g (180
// degrees about x when g = -n)
__device__ void pano_finish(const FitPanos& p, int P, const FitPanoState& s, int status) {
  double* ang = p.angles + 2LL * P;
  double* up = p.up + 3LL * P;
  double* R = p.R + 9LL * P;
  if (status == 2) {
    ang[0] = ang[1] = NAN;
    for (int k = 0; k < 3; ++k) up[k] = NAN;
    for (int k = 0; k < 9; ++k) R[k] = NAN;
    p.cost[P] = NAN;
  } else {
    double psi = wrap_pi(s.theta[0]), phi = s.theta[1];
    if (fabs(psi) > kPi / 2.0) { psi = wrap_pi(kPi - psi); phi += kPi; }
    phi = wrap_pi(phi);
    const double th[2] = {psi, phi};
    double gv[3], dg[3][2];
    pano_gravity(th, gv, dg);
    ang[0] = psi * (180.0 / kPi); ang[1] = phi * (180.0 / kPi);
    for (int k = 0; k < 3; ++k) up[k] = gv[k];
    const double c = -gv[1], wx = -gv[2], wz = gv[0];   // n = (0, -1, 0): w = n x g = (-gz, 0, gx)
    if (1.0 + c > 0.0) {
      const double q = 1.0 / (1.0 + c);
      R[0] = c + wx * wx * q; R[1] = -wz;  R[2] = wx * wz * q;
      R[3] = wz;              R[4] = c;    R[5] = -wx;
      R[6] = wx * wz * q;     R[7] = wx;   R[8] = c + wz * wz * q;
    } else {
      for (int k = 0; k < 9; ++k) R[k] = 0.0;
      R[0] = 1.0; R[4] = -1.0; R[8] = -1.0;
    }
    p.cost[P] = s.C;
  }
  p.iters[P] = s.evals;
  p.status[P] = status;
}

// One warp per panorama: the members' sums at the candidate chained through D_k (lane-strided serial sums, then a shuffle tree:
// a fixed order), then lane 0 runs fit_step_kernel's step on the 2 x 2 system, and the lanes write the members' next v_k.
__global__ void __launch_bounds__(32 * kFitStepWarps) fit_pano_step_kernel(FitArgs a, FitPanos p) {
  pdl_wait();
  pdl_launch();
  const int lane = threadIdx.x & 31;
  const int P = blockIdx.x * kFitStepWarps + (threadIdx.x >> 5);
  if (P >= p.npano) return;
  FitPanoState& s = p.ps[P];
  if (s.status != kFitRunning) return;
  double gv[3], dg[3][2];
  pano_gravity(s.cand, gv, dg);
  double r[7] = {};   // 2 C, count, g[2], A[3]
  for (int j = p.off[P] + lane; j < p.off[P + 1]; j += 32) {
    const int i = p.mem[j];
    const double* v = p.sums + (long long)i * kFitQ;
    const double* M = p.rot + 9LL * i;
    double D[3][2];
#pragma unroll
    for (int c = 0; c < 3; ++c)
#pragma unroll
      for (int k = 0; k < 2; ++k) D[c][k] = M[c] * dg[0][k] + M[3 + c] * dg[1][k] + M[6 + c] * dg[2][k];
    const double Av[3][3] = {{v[5], v[6], v[7]}, {v[6], v[8], v[9]}, {v[7], v[9], v[10]}};
    double AD[3][2];
#pragma unroll
    for (int c = 0; c < 3; ++c)
#pragma unroll
      for (int k = 0; k < 2; ++k) AD[c][k] = Av[c][0] * D[0][k] + Av[c][1] * D[1][k] + Av[c][2] * D[2][k];
    r[0] += v[0];
    r[1] += v[1];
#pragma unroll
    for (int k = 0; k < 2; ++k) r[2 + k] += D[0][k] * v[2] + D[1][k] * v[3] + D[2][k] * v[4];
    r[4] += D[0][0] * AD[0][0] + D[1][0] * AD[1][0] + D[2][0] * AD[2][0];
    r[5] += D[0][0] * AD[0][1] + D[1][0] * AD[1][1] + D[2][0] * AD[2][1];
    r[6] += D[0][1] * AD[0][1] + D[1][1] * AD[1][1] + D[2][1] * AD[2][1];
  }
#pragma unroll
  for (int q = 0; q < 7; ++q)
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) r[q] += __shfl_down_sync(0xffffffffu, r[q], o);
  int status = kFitRunning;
  double cand[2] = {0.0, 0.0};
  if (lane == 0) {
    status = [&]() -> int {
      const double Cc = 0.5 * r[0];
      s.evals += 1;
      if (s.evals == 1) {   // the start
        if (r[1] < 2.0 || r[4] == 0.0 || r[6] == 0.0) return 2;
        s.C = Cc;
        for (int k = 0; k < 2; ++k) { s.theta[k] = s.cand[k]; s.g[k] = r[2 + k]; }
        for (int k = 0; k < 3; ++k) s.A[k] = r[4 + k];
      } else if (Cc < s.C) {   // accept
        const bool done = s.C - Cc <= kFitCostRtol * s.C;
        s.C = Cc;
        for (int k = 0; k < 2; ++k) { s.theta[k] = s.cand[k]; s.g[k] = r[2 + k]; }
        for (int k = 0; k < 3; ++k) s.A[k] = r[4 + k];
        s.lambda /= 10.0;
        if (done) return 0;
      } else {                 // reject: keep theta, A, g
        s.lambda *= 10.0;
        if (s.lambda > kFitLambdaMax) return 0;
      }
      double M[3], g[2] = {-s.g[0], -s.g[1]}, delta[2];
      bool ok = false;
      while (s.lambda <= kFitLambdaMax) {
        M[0] = s.A[0] + s.lambda * s.A[0]; M[1] = s.A[1]; M[2] = s.A[2] + s.lambda * s.A[2];
        if ((ok = cholesky_solve<2>(M, g, delta))) break;
        s.lambda *= 10.0;
      }
      if (!ok) return 0;
      if (fabs(delta[0]) <= kFitStepRtol * (1.0 + fabs(s.theta[0])) && fabs(delta[1]) <= kFitStepRtol * (1.0 + fabs(s.theta[1]))) return 0;
      if (s.evals >= a.max_iter) return 1;
      for (int k = 0; k < 2; ++k) s.cand[k] = s.theta[k] + delta[k];
      return kFitRunning;
    }();
    if (status != kFitRunning) { pano_finish(p, P, s, status); s.status = status; }
    cand[0] = s.cand[0]; cand[1] = s.cand[1];
  }
  status = __shfl_sync(0xffffffffu, status, 0);
  cand[0] = __shfl_sync(0xffffffffu, cand[0], 0);
  cand[1] = __shfl_sync(0xffffffffu, cand[1], 0);
  pano_members(a, p, P, lane, cand, status);
}

}  // namespace pf
