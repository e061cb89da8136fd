// Perspective-field overlays: the reference's draw_perspective_fields / draw_up_field / draw_latitude_field
// (perspective2d/utils/utils.py:165-430, drawn through utils/visualizer.py:192-279 with matplotlib), rasterised on the device.
// One launch renders up to kDrawChunk canvases (each with its own size); a CTA owns one kDrawTW x kDrawTH tile of one canvas.
//
// The rendering rule (this project's; parity with matplotlib's Agg is unpinned, DESIGN.md section 1).  Canvas coordinates are
// pixels, pixel (i, j) covers [j, j+1] x [i, i+1]; every pixel is the average of 4 x 4 samples at (j + (a + .5)/4, i + (b + .5)/4),
// each composited in float32 in this order over the image's RGB:
//   fill   the latitude v (bilinear in its node cell: contourf puts the values on the nodes (j, i), so the contoured domain is
//          [0, W-1] x [0, H-1] and the last column / row strip gets neither fill nor lines) in band k, lev[k] <= v < lev[k+1]
//          (the last band includes lev[18] = pi/2), composited at alpha_fill with band k's colour;
//   lines  every level k with |v - lev[k]| <= lw/2 * |grad v| (the cell's analytic gradient), in increasing k, composited at
//          alpha_line with line k's colour;
//   arrows opaque, the union of the quiver polygons (tail at the lattice point, shaft width w; see draw_arrow_hit), over the
//          lines: in the reference's own rendering (assets/vancouver/pred_pers.png) fully covered shaft pixels stay pure
//          green where they cross the horizon line.
// The 16 samples are summed pairwise (a pixel whose samples agree averages to exactly their value) and rounded half to even.
// Every pixel is read and written by one thread, so the output may alias the input.
#pragma once
#include <stdint.h>

#include "common.cuh"

namespace pf {

constexpr int kDrawTW = 32, kDrawTH = 8, kDrawThreads = kDrawTW * kDrawTH;   // one thread per pixel of the tile
constexpr int kDrawLevels = 19;                                               // linspace(-pi/2, pi/2, 19): 18 bands
constexpr int kDrawChunk = 24;                                                // canvases per launch (descriptors < 4 KB)
constexpr float kDrawHalfLine = 0.5f * 5.0f * 100.0f / 72.0f;                 // linewidths=5 pt at 100 dpi, half of it in px

struct DrawCanvas {          // device copy of one pf_draw_canvas plus what the host derives from it
  int H, W, tiles_x;
  int draw_lat, draw_up;
  int sx, sy, nx, ny;                     // arrow lattice: steps W // density, H // density and counts
  float len, w;                           // arrow length factor sqrt(W^2 + H^2) // arrow_inv_len; shaft width in px
  float rgb[3];                           // arrow colour, 0..255
  float alpha_fill, alpha_line;
  long long img_off, out_off, lat_off, up_off;
  long long us_row, us_col, us_comp;      // up-field element strides
};
struct DrawBatch { DrawCanvas c[kDrawChunk]; };
struct DrawStyle {           // the seismic colours of the bands and lines (0..255) and the levels, built on the host
  float lev[kDrawLevels];
  float band[kDrawLevels - 1][3];
  float line[kDrawLevels][3];
};

// Sample (rx, ry) relative to an arrow's tail; (dx, dy) the unit direction; inv = 1 / (k w) with k the short-arrow scale;
// lp = the polygon's length in units of k w, or < 0 for the hexagon of a vector shorter than one shaft width.
// Upper half (|b|, the polygon is symmetric) of quiver's polygon (0, .5) (lp-3.5, .5) (lp-5, 1.5) (lp, 0): inside the tip's
// edges b <= 0.3 (lp - a), behind the shaft's start a >= 0, and in front of the barb's back edge where b > .5.
__device__ __forceinline__ bool draw_arrow_hit(float rx, float ry, float4 d, float2 s) {
  const float a = (rx * d.z + ry * d.w) * s.x, b = fabsf(ry * d.z - rx * d.w) * s.x;
  if (s.y < 0.f) {                        // regular hexagon of circumradius 1/2, one vertex along the direction
    const float apo = 0.4330127018922193f;
    return b <= apo && fmaf(0.8660254037844386f, fabsf(a), 0.5f * b) <= apo;
  }
  const float lp = s.y;
  if (b > 0.3f * (lp - a)) return false;
  return b <= 0.5f ? a >= 0.f : a >= lp - 3.5f - 1.5f * (b - 0.5f);
}

__global__ void __launch_bounds__(kDrawThreads) draw_fields_kernel(const __grid_constant__ DrawBatch batch, const __grid_constant__ DrawStyle st,
                                                                   const uint8_t* img, uint8_t* out, const float* __restrict__ lat,
                                                                   const float* __restrict__ up) {
  __shared__ float4 s_pos[kDrawThreads];  // tail x, y; unit direction x, y
  __shared__ float2 s_shape[kDrawThreads];
  __shared__ int s_n;
  const DrawCanvas& c = batch.c[blockIdx.y];
  const int ty = blockIdx.x / c.tiles_x, tx = blockIdx.x - ty * c.tiles_x;
  const int x0 = tx * kDrawTW, y0 = ty * kDrawTH;
  if (y0 >= c.H) return;                  // (whole CTA) tiles past a smaller canvas of the chunk
  const int j = x0 + (threadIdx.x % kDrawTW), i = y0 + (threadIdx.x / kDrawTW);
  const bool px = i < c.H && j < c.W;
  const float fj = (float)j, fi = (float)i;

  // arrows: every CTA scans the lattice in chunks of kDrawThreads and keeps those whose box meets its tile
  unsigned hits = 0;                      // bit 4 b + a: sample (a, b) is inside an arrow
  if (c.draw_up) {
    const int N = c.nx * c.ny;
    for (int a0 = 0; a0 < N; a0 += kDrawThreads) {
      if (threadIdx.x == 0) s_n = 0;
      __syncthreads();
      const int q = a0 + threadIdx.x;
      if (q < N) {
        const int ay = q / c.nx, ax = q - ay * c.nx;
        const float tailx = (float)(ax * c.sx), taily = (float)(ay * c.sy);
        const float* u = up + c.up_off + (long long)(ay * c.sy) * c.us_row + (long long)(ax * c.sx) * c.us_col;
        const float ux = u[0] * c.len, uy = u[c.us_comp] * c.len;
        const float len = sqrtf(fmaf(ux, ux, uy * uy));
        const float l = len / c.w;        // length in shaft widths
        float dx = 1.f, dy = 0.f;         // atan2(0, 0) = 0: a zero vector's hexagon has a vertex along +x
        if (len > 0.f) { dx = ux / len; dy = uy / len; }
        float inv, lp, reach;
        if (l < 1.f) { inv = 1.f / c.w; lp = -1.f; reach = 0.5f * c.w; }
        else if (l < 5.f) { inv = 5.f / len; lp = 5.f; reach = len + 0.3f * len; }   // the l = 5 polygon scaled by l / 5
        else { inv = 1.f / c.w; lp = l; reach = len + 1.5f * c.w; }
        // conservative box: the polygon lies within `reach` of the tail
        if (tailx + reach >= (float)x0 && tailx - reach <= (float)(x0 + kDrawTW) && taily + reach >= (float)y0 &&
            taily - reach <= (float)(y0 + kDrawTH)) {
          const int slot = atomicAdd(&s_n, 1);
          s_pos[slot] = make_float4(tailx, taily, dx, dy);
          s_shape[slot] = make_float2(inv, lp);
        }
      }
      __syncthreads();
      const int n = s_n;
      if (px) {
        for (int k = 0; k < n; ++k) {
          const float4 d = s_pos[k];
          const float2 s = s_shape[k];
#pragma unroll
          for (int b = 0; b < 4; ++b)
#pragma unroll
            for (int a = 0; a < 4; ++a)
              if (draw_arrow_hit(fj + (a + 0.5f) * 0.25f - d.x, fi + (b + 0.5f) * 0.25f - d.y, d, s)) hits |= 1u << (4 * b + a);
        }
      }
      __syncthreads();                    // s_n / the list are rewritten by the next chunk
    }
  }
  if (!px) return;

  const long long p = (long long)i * c.W + j;
  const uint8_t* src = img + c.img_off + 3 * p;
  const float im[3] = {(float)src[0], (float)src[1], (float)src[2]};
  const bool dom = c.draw_lat && j < c.W - 1 && i < c.H - 1;
  float v00 = 0.f, v01 = 0.f, v10 = 0.f, v11 = 0.f;
  if (dom) {
    const float* l0 = lat + c.lat_off + p;
    v00 = l0[0]; v01 = l0[1]; v10 = l0[c.W]; v11 = l0[c.W + 1];
  }
  const float lev0 = st.lev[0], levN = st.lev[kDrawLevels - 1];
  const float inv_step = (float)(kDrawLevels - 1) / (levN - lev0);
  float rows[4][3];
#pragma unroll
  for (int b = 0; b < 4; ++b) {
    float smp[4][3];
#pragma unroll
    for (int a = 0; a < 4; ++a) {
      float col[3] = {im[0], im[1], im[2]};
      float v = 0.f, g = 0.f;
      if (dom) {
        const float fx = (a + 0.5f) * 0.25f, fy = (b + 0.5f) * 0.25f;
        const float top = fmaf(fx, v01 - v00, v00), bot = fmaf(fx, v11 - v10, v10);
        v = fmaf(fy, bot - top, top);
        const float gx = fmaf(fy, (v11 - v10) - (v01 - v00), v01 - v00), gy = fmaf(fx, (v11 - v01) - (v10 - v00), v10 - v00);
        g = kDrawHalfLine * sqrtf(fmaf(gx, gx, gy * gy));
        if (v >= lev0 && v <= levN) {
          int k = min(max((int)((v - lev0) * inv_step), 0), kDrawLevels - 2);
          if (v < st.lev[k]) --k;                                   // the table decides at the boundaries
          else if (k < kDrawLevels - 2 && v >= st.lev[k + 1]) ++k;
#pragma unroll
          for (int ch = 0; ch < 3; ++ch) col[ch] = fmaf(c.alpha_fill, st.band[k][ch] - col[ch], col[ch]);
        }
      }
      if (dom && v == v) {
        // only the levels within g of v can hold the sample (one level of slack each side for the float rounding)
        // (clamped in float: g may be infinite)
        const int klo = (int)fmaxf(floorf((v - g - lev0) * inv_step) - 1.f, 0.f);
        const int khi = (int)fminf(floorf((v + g - lev0) * inv_step) + 1.f, (float)(kDrawLevels - 1));
        for (int k = klo; k <= khi; ++k) {
          if (fabsf(v - st.lev[k]) <= g) {
#pragma unroll
            for (int ch = 0; ch < 3; ++ch) col[ch] = fmaf(c.alpha_line, st.line[k][ch] - col[ch], col[ch]);
          }
        }
      }
      const bool arrow = hits >> (4 * b + a) & 1u;
#pragma unroll
      for (int ch = 0; ch < 3; ++ch) smp[a][ch] = arrow ? c.rgb[ch] : col[ch];
    }
#pragma unroll
    for (int ch = 0; ch < 3; ++ch) rows[b][ch] = (smp[0][ch] + smp[1][ch]) + (smp[2][ch] + smp[3][ch]);
  }
  uint8_t* dst = out + c.out_off + 3 * p;
#pragma unroll
  for (int ch = 0; ch < 3; ++ch) {
    const float m = ((rows[0][ch] + rows[1][ch]) + (rows[2][ch] + rows[3][ch])) * (1.f / 16.f);
    dst[ch] = (uint8_t)min(max(__float2int_rn(m), 0), 255);
  }
}

}  // namespace pf
