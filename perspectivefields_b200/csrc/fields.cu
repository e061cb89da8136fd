// Batched calls on images and fields, outside the network: panorama and equirectangular crops, field drawing, scoring against
// ground truth, the camera fit and the upright warp (C ABI: include/pf_b200.h).  Each runs on the caller's device pointers and stream.
#include <algorithm>
#include <cmath>
#include <cstring>

#include "host.h"
#include "calib.cuh"
#include "draw.cuh"
#include "equi.cuh"
#include "metrics.cuh"
#include "pano.cuh"
#include "rectify.cuh"

using namespace pf;

extern "C" {

// PanoCam.crop_distortion (utils/panocam.py:559-752) for n views of one panorama: the host builds each view's rotation matrices
// (:617-655), minimal focal length and disk (:592-594, :696-705) in float64 once; one launch per kPanoChunk views.
int pf_pano_views(int device, const uint8_t* pano, int pano_h, int pano_w, const pf_pano_view* views, int n, uint8_t* im, float* ntheta,
                  float* nphi, float* up, float* lat, float* xy, double* offset, int32_t* status, void* stream) {
  if (!pano || !views || n < 1) return fail(PF_ERR_ARG, "pf_pano_views: null panorama / views or n < 1");
  if (pano_h < 2 || pano_w < 2) return fail(PF_ERR_ARG, "pf_pano_views: panorama of %dx%d (needs at least 2x2)", pano_h, pano_w);
  if (!im && !ntheta && !nphi && !up && !lat && !xy && !offset && !status) return fail(PF_ERR_ARG, "pf_pano_views: no output");
  for (int i = 0; i < n; ++i) {
    const pf_pano_view& c = views[i];
    if (c.height < 1 || c.width < 1) return fail(PF_ERR_ARG, "pf_pano_views: view %d has size %dx%d", i, c.height, c.width);
    if (!std::isfinite(c.f) || !(c.f > 0.0) || !std::isfinite(c.xi) || !std::isfinite(c.az) || !std::isfinite(c.el) || !std::isfinite(c.roll))
      return fail(PF_ERR_ARG, "pf_pano_views: view %d: f must be finite and > 0, xi and the angles finite (f %g, xi %g)", i, c.f, c.xi);
    if (c.im_offset < 0 || c.field_offset < 0) return fail(PF_ERR_ARG, "pf_pano_views: view %d has a negative offset", i);
  }
  CU(cudaSetDevice(device));
  PanoMap m{};
  m.Hp = pano_h; m.Wp = pano_w;
  m.ax = (M_PI - -M_PI) / ((pano_w - 1.0) - 0);   // :680-687, python's own expressions
  m.bx = M_PI - m.ax * (pano_w - 1.0);
  m.iax = 1.0 / m.ax;
  m.ay = (-M_PI / 2.0 - M_PI / 2.0) / ((pano_h - 1.0) - 0);
  m.by = M_PI / 2.0 - m.ay * 0;
  m.iay = 1.0 / m.ay;
  auto rad = [](double deg) { return deg * M_PI / 180; };
  for (int i0 = 0; i0 < n; i0 += kPanoChunk) {
    const int cnt = n - i0 < kPanoChunk ? n - i0 : kPanoChunk;
    PanoBatch b{};
    long long max_px = 1;
    for (int i = 0; i < cnt; ++i) {
      const pf_pano_view& c = views[i0 + i];
      PanoView& o = b.v[i];
      o.H = c.height; o.W = c.width;
      o.f = c.f; o.xi = c.xi; o.one_m_xi2 = 1 - c.xi * c.xi;
      o.u0 = c.width / 2.0; o.v0 = c.height / 2.0;
      const double ce = cos(rad(c.el)), se = sin(rad(c.el)), ca = cos(rad(c.az)), sa = sin(rad(c.az)), cr = cos(rad(c.roll)), sr = sin(rad(c.roll));
      const double rel[9] = {1.0, 0.0, 0.0, 0.0, ce, -se, 0.0, se, ce};
      const double raz[9] = {ca, 0.0, sa, 0.0, 1.0, 0.0, -sa, 0.0, ca};
      const double rroll[9] = {cr, -sr, 0.0, sr, cr, 0.0, 0.0, 0.0, 1.0};
      memcpy(o.rel, rel, sizeof rel); memcpy(o.raz, raz, sizeof raz); memcpy(o.rroll, rroll, sizeof rroll);
      // minfocal(u0, v0, xi, 1, 1) (:64-70): NaN unless xi > 1, and f < NaN is false
      const double fmin = sqrt(-(1 - c.xi * c.xi) * ((1 - o.u0) * (1 - o.u0) + (1 - o.v0) * (1 - o.v0))) * 1.0001;
      o.masked = c.f < fmin;
      const double r = sqrt(-(c.f * c.f) / (1 - c.xi * c.xi));   // diskradius (:18-19)
      o.r2 = r * r;
      o.ci0 = nearbyint(c.height / 2.0); o.ci1 = nearbyint(c.width / 2.0);   // np.round: half to even (the default rounding mode)
      o.im_off = c.im_offset; o.fld_off = c.field_offset;
      const long long px = (long long)c.height * c.width;
      if (px > max_px) max_px = px;
    }
    const dim3 grid((unsigned)cdivl(max_px, (long long)kPanoThreads * kPanoPix) + 1, (unsigned)cnt);
    LAUNCHED((pano_views_kernel<<<grid, kPanoThreads, 0, (cudaStream_t)stream>>>(b, m, pano, im, ntheta, nphi, up, lat, xy, offset, status, i0),
              cudaGetLastError()));
  }
  return PF_OK;
}

// PanoCam.crop_equi / get_image (utils/panocam.py:121-249) for n views of one panorama: the host computes each view's fov_x
// (:216-218, the wrapper's own expression), focal length and the sines and cosines of its angles once; one launch per kEquiChunk views.
int pf_equi_views(int device, const void* pano, int pano_h, int pano_w, int channels, int dtype, const pf_equi_view* views, int n, int mode,
                  int out_kind, int swap_rb, void* im, void* stream) {
  if (!pano || !views || !im || n < 1) return fail(PF_ERR_ARG, "pf_equi_views: null panorama / views / im or n < 1");
  if (pano_h < 1 || pano_w < 1) return fail(PF_ERR_ARG, "pf_equi_views: panorama of %dx%d", pano_h, pano_w);
  if (channels != 1 && channels != 3) return fail(PF_ERR_ARG, "pf_equi_views: %d channels (1 or 3)", channels);
  if (dtype != PF_EQUI_U8 && dtype != PF_EQUI_F32) return fail(PF_ERR_ARG, "pf_equi_views: unknown dtype %d", dtype);
  if (mode != PF_EQUI_BILINEAR && mode != PF_EQUI_NEAREST) return fail(PF_ERR_ARG, "pf_equi_views: unknown mode %d", mode);
  if (out_kind != PF_EQUI_CAST && out_kind != PF_EQUI_UNIT) return fail(PF_ERR_ARG, "pf_equi_views: unknown out_kind %d", out_kind);
  if (out_kind == PF_EQUI_UNIT && dtype != PF_EQUI_U8) return fail(PF_ERR_ARG, "pf_equi_views: the unit path needs a uint8 panorama");
  if (swap_rb != 0 && (swap_rb != 1 || channels != 3)) return fail(PF_ERR_ARG, "pf_equi_views: swap_rb must be 0, or 1 with 3 channels");
  const int esize = dtype == PF_EQUI_F32 ? 4 : 1;
  std::vector<double> fov_x(n);
  for (int i = 0; i < n; ++i) {
    const pf_equi_view& c = views[i];
    if (c.height < 1 || c.width < 1) return fail(PF_ERR_ARG, "pf_equi_views: view %d has size %dx%d", i, c.height, c.width);
    if (!std::isfinite(c.azimuth) || !std::isfinite(c.elevation) || !std::isfinite(c.roll))
      return fail(PF_ERR_ARG, "pf_equi_views: view %d: non-finite angle", i);
    if (!std::isfinite(c.vfov) || !(c.vfov > 0.0 && c.vfov < 180.0) || !std::isfinite(c.ar) || !(c.ar > 0.0))
      return fail(PF_ERR_ARG, "pf_equi_views: view %d: vfov %g must lie in (0, 180) and ar %g be finite and > 0", i, c.vfov, c.ar);
    fov_x[i] = 2 * atan(tan(c.vfov * M_PI / 180.0 / 2) * c.ar) * 180 / M_PI;
    if (!(fov_x[i] > 0.0 && fov_x[i] < 180.0)) return fail(PF_ERR_ARG, "pf_equi_views: view %d: fov_x %g must lie in (0, 180)", i, fov_x[i]);
    if (c.offset < 0 || c.offset % esize != 0) return fail(PF_ERR_ARG, "pf_equi_views: view %d: offset %lld (>= 0, a multiple of %d)", i,
                                                          (long long)c.offset, esize);
  }
  CU(cudaSetDevice(device));
  EquiMap m{};
  m.Hp = pano_h; m.Wp = pano_w; m.C = channels;
  m.nearest = mode == PF_EQUI_NEAREST; m.swap_rb = swap_rb;
  m.su = pano_w / (2 * M_PI); m.sv = pano_h / M_PI;
  for (int i0 = 0; i0 < n; i0 += kEquiChunk) {
    const int cnt = n - i0 < kEquiChunk ? n - i0 : kEquiChunk;
    EquiBatch b{};
    long long max_px = 1;
    for (int i = 0; i < cnt; ++i) {
      const pf_equi_view& c = views[i0 + i];
      EquiView& o = b.v[i];
      o.H = c.height; o.W = c.width;
      o.f = c.width / (2 * tan(fov_x[i0 + i] * M_PI / 180 / 2));
      o.u0 = c.width / 2.0; o.v0 = c.height / 2.0;
      const double roll = c.roll / 180 * M_PI, el = c.elevation / 180 * M_PI, az = c.azimuth / 180 * M_PI;   // the wrapper's rot dict
      o.cr = cos(roll); o.sr = sin(roll); o.ce = cos(el); o.se = sin(el); o.ca = cos(az); o.sa = sin(az);
      o.off = c.offset;
      const long long px = (long long)c.height * c.width;
      if (px > max_px) max_px = px;
    }
    const dim3 grid((unsigned)cdivl(max_px, (long long)kEquiThreads * kEquiPix), (unsigned)cnt);
    cudaStream_t st = (cudaStream_t)stream;
    unsigned char* out = (unsigned char*)im;
    if (dtype == PF_EQUI_F32)
      LAUNCHED((equi_views_kernel<float, false><<<grid, kEquiThreads, 0, st>>>(b, m, (const float*)pano, out), cudaGetLastError()));
    else if (out_kind == PF_EQUI_UNIT)
      LAUNCHED((equi_views_kernel<unsigned char, true><<<grid, kEquiThreads, 0, st>>>(b, m, (const unsigned char*)pano, out), cudaGetLastError()));
    else
      LAUNCHED((equi_views_kernel<unsigned char, false><<<grid, kEquiThreads, 0, st>>>(b, m, (const unsigned char*)pano, out), cudaGetLastError()));
  }
  return PF_OK;
}

// ----------------------------------------------------------------------------------------------- batched feature calls
static long long align256(long long b) { return (b + 255) / 256 * 256; }

// A caller-provided workspace carved into 256-byte-aligned sections, in the order they are added: at[k] is the byte offset of
// section k; the first holds the per-image descriptors (upload_descriptors)
struct WsLayout {
  long long at[4] = {}, total = 0;
  int count = 0;
  WsLayout& add(long long bytes) { at[count++] = total; total += align256(bytes); return *this; }
};

static int check_workspace(const char* fn, const void* ws, int64_t bytes, long long need) {
  if (bytes < need) return fail(PF_ERR_WORKSPACE, "%s: workspace %lld B < required %lld B", fn, (long long)bytes, need);
  if (((uintptr_t)ws & 255) != 0) return fail(PF_ERR_ARG, "%s: workspace must be 256-byte aligned", fn);
  return PF_OK;
}

static int upload_descriptors(const void* d, size_t bytes, void* ws, cudaStream_t st) {
  CU(cudaMemcpyAsync(ws, d, bytes, cudaMemcpyHostToDevice, st));
  return PF_OK;
}

// The per-image offset rule of the batched calls: a required offset is >= 0; an optional one is -1 (absent) or >= 0, and then
// the buffer it points into must be given
static int check_offsets(const char* fn, int i, std::initializer_list<long long> required,
                         std::initializer_list<std::pair<long long, const void*>> optional = {}) {
  for (const long long o : required)
    if (o < 0) return fail(PF_ERR_ARG, "%s: image %d has a negative offset", fn, i);
  for (const auto& [o, buf] : optional) {
    if (o < -1) return fail(PF_ERR_ARG, "%s: image %d has a negative offset", fn, i);
    if (o >= 0 && !buf) return fail(PF_ERR_ARG, "%s: image %d has an offset into a NULL buffer", fn, i);
  }
  return PF_OK;
}

// matplotlib's "seismic" map as the 256-entry table it samples (LinearSegmentedColormap.from_list: anchors at 0, 1/4, 1/2, 3/4, 1,
// linear interpolation at i / 255), and t -> entry min(floor(256 t), 255); levels linspace(-pi/2, pi/2, 19).
static DrawStyle draw_style() {
  static const double anchors[5][3] = {{0.0, 0.0, 0.3}, {0.0, 0.0, 1.0}, {1.0, 1.0, 1.0}, {1.0, 0.0, 0.0}, {0.5, 0.0, 0.0}};
  auto seismic = [&](double t, int ch) {
    const int e = std::min((int)std::floor(256.0 * t), 255);
    const double x = e / 255.0;
    const int s = std::min((int)(x * 4.0), 3);
    const double dist = (x - s / 4.0) / 0.25;
    return 255.0 * (dist * (anchors[s + 1][ch] - anchors[s][ch]) + anchors[s][ch]);
  };
  DrawStyle st{};
  const int nb = kDrawLevels - 1;
  for (int k = 0; k < kDrawLevels; ++k) {
    st.lev[k] = (float)(k == nb ? M_PI / 2 : -M_PI / 2 + k * (M_PI / nb));
    for (int ch = 0; ch < 3; ++ch) {
      st.line[k][ch] = (float)seismic((double)k / nb, ch);
      if (k < nb) st.band[k][ch] = (float)seismic((k + 0.5) / nb, ch);
    }
  }
  return st;
}

int pf_draw_fields(int device, const pf_draw_canvas* cs, int n, const uint8_t* img, uint8_t* out, const float* lat, const float* up, void* stream) {
  if (!cs || n < 1 || !img || !out) return fail(PF_ERR_ARG, "pf_draw_fields: null canvases / img / out or n < 1");
  auto unit = [](float x) { return std::isfinite(x) && x >= 0.f && x <= 1.f; };
  for (int i = 0; i < n; ++i) {
    const pf_draw_canvas& c = cs[i];
    if (c.height < 1 || c.width < 1 || (long long)c.height * c.width >= (1LL << 31))
      return fail(PF_ERR_ARG, "pf_draw_fields: canvas %d has size %dx%d", i, c.height, c.width);
    TRY(check_offsets("pf_draw_fields", i, {c.img_offset, c.out_offset}));
    if (!unit(c.alpha_fill) || !unit(c.alpha_line)) return fail(PF_ERR_ARG, "pf_draw_fields: canvas %d: alphas must lie in [0, 1]", i);
    if (c.draw_lat && (!lat || c.lat_offset < 0)) return fail(PF_ERR_ARG, "pf_draw_fields: canvas %d draws the latitude without a latitude map", i);
    if (c.draw_up) {
      if (!up || c.up_offset < 0 || c.up_stride[0] < 0 || c.up_stride[1] < 0 || c.up_stride[2] < 0)
        return fail(PF_ERR_ARG, "pf_draw_fields: canvas %d draws arrows without an up field, or with a negative offset / stride", i);
      if (c.density < 1 || c.arrow_inv_len < 1 || c.width / c.density < 1 || c.height / c.density < 1)
        return fail(PF_ERR_ARG, "pf_draw_fields: canvas %d (%dx%d): density %d and arrow_inv_len %d must be >= 1 and leave W // density, "
                    "H // density >= 1", i, c.height, c.width, c.density, c.arrow_inv_len);
      if (!unit(c.arrow_rgb[0]) || !unit(c.arrow_rgb[1]) || !unit(c.arrow_rgb[2])) return fail(PF_ERR_ARG, "pf_draw_fields: canvas %d: arrow colour outside [0, 1]", i);
    }
  }
  CU(cudaSetDevice(device));
  const DrawStyle st = draw_style();
  for (int i0 = 0; i0 < n; i0 += kDrawChunk) {
    const int cnt = n - i0 < kDrawChunk ? n - i0 : kDrawChunk;
    DrawBatch b{};
    long long max_tiles = 1;
    for (int i = 0; i < cnt; ++i) {
      const pf_draw_canvas& c = cs[i0 + i];
      DrawCanvas& o = b.c[i];
      o.H = c.height; o.W = c.width;
      o.tiles_x = cdiv(c.width, kDrawTW);
      o.draw_lat = c.draw_lat != 0; o.draw_up = c.draw_up != 0;
      o.alpha_fill = c.alpha_fill; o.alpha_line = c.alpha_line;
      o.img_off = c.img_offset; o.out_off = c.out_offset; o.lat_off = c.lat_offset; o.up_off = c.up_offset;
      o.us_row = c.up_stride[0]; o.us_col = c.up_stride[1]; o.us_comp = c.up_stride[2];
      if (o.draw_up) {
        o.sx = c.width / c.density; o.sy = c.height / c.density;
        o.nx = cdiv(c.width, o.sx); o.ny = cdiv(c.height, o.sy);
        // np.sqrt(W^2 + H^2) // arrow_inv_len with Python's float floor division
        const double diag = std::sqrt((double)c.width * c.width + (double)c.height * c.height), q = c.arrow_inv_len;
        const double mod = std::fmod(diag, q), div = (diag - mod) / q;
        double fl = std::floor(div);
        if (div - fl > 0.5) fl += 1.0;
        o.len = (float)fl;
        const double sq = std::sqrt((double)o.nx * o.ny);                        // quiver's default width: 0.06 span / clip(sqrt(N), 8, 25)
        o.w = (float)(0.06 * c.width / std::min(std::max(sq, 8.0), 25.0));
        for (int ch = 0; ch < 3; ++ch) o.rgb[ch] = 255.f * c.arrow_rgb[ch];
      }
      const long long tiles = (long long)o.tiles_x * cdiv(c.height, kDrawTH);
      if (tiles > max_tiles) max_tiles = tiles;
    }
    const dim3 grid((unsigned)max_tiles, (unsigned)cnt);
    LAUNCHED((draw_fields_kernel<<<grid, kDrawThreads, 0, (cudaStream_t)stream>>>(b, st, img, out, lat, up), cudaGetLastError()));
  }
  return PF_OK;
}

// ----------------------------------------------------------------------------------------------- scoring (metrics.cuh)
static bool gravity_classes_ok(int c) { return c == 2 || c >= 3; }
static bool latitude_classes_ok(int c) { return c >= 1; }

int pf_encode_fields(int device, int n, int H, int W, const float* up, const int64_t* up_stride, const float* lat, const int64_t* lat_stride,
                     int lat_rad, int gravity_classes, int latitude_classes, void* gt_gravity, void* gt_latitude, void* stream) {
  if (n < 1 || H < 1 || W < 1 || (long long)n * H * W >= (1LL << 40)) return fail(PF_ERR_ARG, "pf_encode_fields: bad batch %d x %d x %d", n, H, W);
  if (!up && !lat) return fail(PF_ERR_ARG, "pf_encode_fields: neither an up nor a latitude field");
  if (up && (!up_stride || !gt_gravity || !gravity_classes_ok(gravity_classes)))
    return fail(PF_ERR_ARG, "pf_encode_fields: the up field needs strides, an output and gravity_classes 2 or >= 3 (got %d)", gravity_classes);
  if (lat && (!lat_stride || !gt_latitude || !latitude_classes_ok(latitude_classes)))
    return fail(PF_ERR_ARG, "pf_encode_fields: the latitude field needs strides, an output and latitude_classes >= 1 (got %d)", latitude_classes);
  if (lat_rad != 0 && lat_rad != 1) return fail(PF_ERR_ARG, "pf_encode_fields: lat_rad must be 0 or 1");
  EncodeArgs a{};
  a.n = n; a.H = H; a.W = W; a.up = up; a.lat = lat; a.lat_rad = lat_rad; a.gc = gravity_classes; a.lc = latitude_classes;
  a.gt_g = gt_gravity; a.gt_l = gt_latitude;
  if (up) { a.us_img = up_stride[0]; a.us_row = up_stride[1]; a.us_col = up_stride[2]; a.us_comp = up_stride[3]; }
  if (lat) { a.ls_img = lat_stride[0]; a.ls_row = lat_stride[1]; a.ls_col = lat_stride[2]; }
  CU(cudaSetDevice(device));
  const long long px = (long long)n * H * W;
  LAUNCHED((encode_fields_kernel<<<(unsigned)cdivl(px, kMetThreads), kMetThreads, 0, (cudaStream_t)stream>>>(a), cudaGetLastError()));
  return PF_OK;
}

// Blocks of the loss passes: classification (gravity, latitude) or regression (one pass over both heads)
static void loss_blocks(int n, int H, int W, int gc, long long* bg, long long* bl) {
  const long long px = (long long)n * H * W;
  if (gc == 2) { *bg = cdivl(px, (long long)kMetThreads * kRegPix); *bl = 0; }
  else { *bg = cdivl(px / kCePix, kMetThreads); *bl = *bg; }
}
int64_t pf_head_losses_workspace(int n, int H, int W, int gravity_classes, int latitude_classes) {
  if (n < 1 || H < 1 || W < 1) return fail(PF_ERR_ARG, "pf_head_losses_workspace: bad batch %d x %d x %d", n, H, W);
  if (!((gravity_classes == 2 && latitude_classes == 1) || (gravity_classes >= 3 && latitude_classes >= 2)))
    return fail(PF_ERR_ARG, "pf_head_losses_workspace: heads %d / %d: both regression (2 / 1) or both classification", gravity_classes, latitude_classes);
  long long bg, bl;
  loss_blocks(n, H, W, gravity_classes, &bg, &bl);
  return gravity_classes == 2 ? align256(bg * kRegSums * 8) + align256(bg * kRegCounts * 8) : align256((bg + bl) * 8) * 2;
}

int pf_head_losses(int device, int n, int H, int W, int gravity_classes, const float* pred_gravity, const void* gt_gravity, int latitude_classes,
                   const float* pred_latitude, const void* gt_latitude, int gravity_ignore, int latitude_ignore, float gravity_weight,
                   float latitude_weight, float* losses, void* workspace, int64_t workspace_bytes, void* stream) {
  const int64_t need = pf_head_losses_workspace(n, H, W, gravity_classes, latitude_classes);
  if (need < 0) return (int)need;
  if (!pred_gravity || !gt_gravity || !pred_latitude || !gt_latitude || !losses || !workspace)
    return fail(PF_ERR_ARG, "pf_head_losses: null prediction / target / losses / workspace");
  TRY(check_workspace("pf_head_losses", workspace, workspace_bytes, need));
  const bool cls = gravity_classes != 2;
  if (cls && (((long long)H * W) % kCePix != 0 || ((uintptr_t)pred_gravity & 15) || ((uintptr_t)pred_latitude & 15)))
    return fail(PF_ERR_ARG, "pf_head_losses: classification logits need H * W %% 4 == 0 and 16-byte aligned planes");
  if (cls && ((long long)latitude_classes * H * W >= (1LL << 40))) return fail(PF_ERR_ARG, "pf_head_losses: logits too large");
  CU(cudaSetDevice(device));
  cudaStream_t st = (cudaStream_t)stream;
  long long bg, bl;
  loss_blocks(n, H, W, gravity_classes, &bg, &bl);
  double* psum = (double*)workspace;
  const int HW = H * W;
  if (cls) {
    long long* pcnt = (long long*)((char*)workspace + align256((bg + bl) * 8));
    const CeHead g{pred_gravity, (const long long*)gt_gravity, gravity_classes, gravity_ignore, (int)bg};
    const CeHead l{pred_latitude, (const long long*)gt_latitude, latitude_classes, latitude_ignore, (int)bl};
    LAUNCHED((cross_entropy_kernel<<<(unsigned)(bg + bl), kMetThreads, 0, st>>>(g, l, n, HW, psum, pcnt), cudaGetLastError()));
    LAUNCHED((loss_finish_kernel<<<1, kMetThreads, 0, st>>>(0, (int)bg, (int)(bg + bl), psum, pcnt, 0, gravity_weight, latitude_weight, losses),
              cudaGetLastError()));
  } else {
    long long* pcnt = (long long*)((char*)workspace + align256(bg * kRegSums * 8));
    const RegArgs a{pred_gravity, (const float*)gt_gravity, pred_latitude, (const float*)gt_latitude, n, H, W};
    LAUNCHED((regression_loss_kernel<<<(unsigned)bg, kMetThreads, 0, st>>>(a, (int)bg, psum, pcnt), cudaGetLastError()));
    LAUNCHED((loss_finish_kernel<<<1, kMetThreads, 0, st>>>(1, (int)bg, (int)bg, psum, pcnt, (long long)n * HW, gravity_weight, latitude_weight, losses),
              cudaGetLastError()));
  }
  return PF_OK;
}

// Workspace layout of pf_field_errors: device descriptors | fp64 sums [2][blocks] | counts [2][1 + 8][blocks] | maps if not given
static int field_errors_layout(const pf_field_image* im, int n, int with_maps, WsLayout* lay, long long* blocks_out = nullptr,
                               long long* pixels_out = nullptr) {
  if (!im || n < 1) return fail(PF_ERR_ARG, "pf_field_errors: null images or n < 1");
  long long blocks = 0, pixels = 0;
  for (int i = 0; i < n; ++i) {
    if (im[i].height < 1 || im[i].width < 1 || (long long)im[i].height * im[i].width >= (1LL << 31))
      return fail(PF_ERR_ARG, "pf_field_errors: image %d has size %dx%d", i, im[i].height, im[i].width);
    const long long hw = (long long)im[i].height * im[i].width;
    blocks += cdivl(hw, kFeTile);
    pixels += hw;
  }
  if (blocks >= (1LL << 31)) return fail(PF_ERR_ARG, "pf_field_errors: too many pixels");
  lay->add((long long)n * sizeof(FeImage)).add(2 * blocks * 8).add(2LL * (1 + kFeMaxThr) * blocks * 4).add(with_maps ? 0 : 2 * pixels * 4);
  if (blocks_out) *blocks_out = blocks;
  if (pixels_out) *pixels_out = pixels;
  return PF_OK;
}
int64_t pf_field_errors_workspace(const pf_field_image* images, int n, int with_maps) {
  WsLayout lay;
  TRY(field_errors_layout(images, n, with_maps, &lay));
  return lay.total;
}

int pf_field_errors(int device, const pf_field_image* images, int n, const float* pred_up, const float* pred_lat, const float* gt_up,
                    const float* gt_lat, const uint8_t* mask, int lat_rad, const double* thresholds, int n_thresholds, float* up_maps,
                    float* lat_maps, int64_t* count, double* mean, double* median, double* fraction, void* workspace,
                    int64_t workspace_bytes, void* stream) {
  if ((up_maps == nullptr) != (lat_maps == nullptr)) return fail(PF_ERR_ARG, "pf_field_errors: give both maps or neither");
  WsLayout lay;
  long long blocks, pixels;
  TRY(field_errors_layout(images, n, up_maps != nullptr, &lay, &blocks, &pixels));
  if (!pred_up || !pred_lat || !gt_up || !gt_lat || !count || !mean || !median || !workspace)
    return fail(PF_ERR_ARG, "pf_field_errors: null field / output / workspace");
  if (n_thresholds < 0 || n_thresholds > kFeMaxThr || (n_thresholds > 0 && (!thresholds || !fraction)))
    return fail(PF_ERR_ARG, "pf_field_errors: %d thresholds (0 to %d, with a fraction output)", n_thresholds, kFeMaxThr);
  for (int k = 0; k < n_thresholds; ++k)
    if (std::isnan(thresholds[k])) return fail(PF_ERR_ARG, "pf_field_errors: threshold %d is NaN", k);
  if (lat_rad != 0 && lat_rad != 1) return fail(PF_ERR_ARG, "pf_field_errors: lat_rad must be 0 or 1");
  TRY(check_workspace("pf_field_errors", workspace, workspace_bytes, lay.total));
  std::vector<FeImage> d(n);
  long long block0 = 0, map_off = 0;
  for (int i = 0; i < n; ++i) {
    const pf_field_image& c = images[i];
    TRY(check_offsets("pf_field_errors", i, {c.pred_up_offset, c.pred_lat_offset, c.gt_up_offset, c.gt_lat_offset}, {{c.mask_offset, mask}}));
    FeImage& o = d[i];
    o.H = c.height; o.W = c.width;
    o.pu_off = c.pred_up_offset; o.pu_sr = c.pred_up_stride[0]; o.pu_sc = c.pred_up_stride[1]; o.pu_sk = c.pred_up_stride[2];
    o.pl_off = c.pred_lat_offset;
    o.gu_off = c.gt_up_offset; o.gu_sr = c.gt_up_stride[0]; o.gu_sc = c.gt_up_stride[1]; o.gu_sk = c.gt_up_stride[2];
    o.gl_off = c.gt_lat_offset;
    o.mask_off = c.mask_offset;
    o.map_off = map_off;
    const long long hw = (long long)c.height * c.width;
    o.block0 = (int)block0; o.nblk = (int)cdivl(hw, kFeTile);
    block0 += o.nblk; map_off += hw;
  }
  CU(cudaSetDevice(device));
  cudaStream_t st = (cudaStream_t)stream;
  char* ws = (char*)workspace;
  FeArgs a{};
  a.im = (const FeImage*)ws; a.n = n; a.nblocks = (int)blocks;
  a.pu = pred_up; a.pl = pred_lat; a.gu = gt_up; a.gl = gt_lat; a.mask = mask;
  a.lat_rad = lat_rad; a.T = n_thresholds;
  for (int k = 0; k < n_thresholds; ++k) a.thr[k] = thresholds[k];
  a.map_up = up_maps ? up_maps : (float*)(ws + lay.at[3]);
  a.map_lat = lat_maps ? lat_maps : (float*)(ws + lay.at[3]) + pixels;
  a.psum = (double*)(ws + lay.at[1]); a.pcnt = (int*)(ws + lay.at[2]);
  TRY(upload_descriptors(d.data(), d.size() * sizeof(d[0]), ws, st));
  LAUNCHED((field_errors_kernel<<<(unsigned)blocks, kMetThreads, 0, st>>>(a), cudaGetLastError()));
  const FeOut o{(long long*)count, mean, median, fraction};
  LAUNCHED((field_stats_kernel<<<dim3((unsigned)n, 2), kFeSelThreads, 0, st>>>(a, o), cudaGetLastError()));
  return PF_OK;
}

// ----------------------------------------------------------------------------------------------- camera fit (calib.cuh)
// Workspace layout of pf_fit_camera: device descriptors | per-image state | fp64 partials [kFitQ][pass blocks]
constexpr int kFitMaxIterations = 1000;
static int fit_layout(const pf_fit_image* im, int n, WsLayout* lay, long long* blocks_out = nullptr) {
  if (!im || n < 1) return fail(PF_ERR_ARG, "pf_fit_camera: null images or n < 1");
  long long blocks = 0;
  for (int i = 0; i < n; ++i) {
    if (im[i].height < 3 || im[i].width < 3 || (long long)im[i].height * im[i].width >= (1LL << 31))
      return fail(PF_ERR_ARG, "pf_fit_camera: image %d has size %dx%d (3x3 at least)", i, im[i].height, im[i].width);
    blocks += cdivl((long long)im[i].height * im[i].width, kFitTile);
  }
  if (blocks >= (1LL << 31)) return fail(PF_ERR_ARG, "pf_fit_camera: too many pixels");
  lay->add((long long)n * sizeof(FitImage)).add((long long)n * sizeof(FitState)).add((long long)kFitQ * blocks * 8);
  if (blocks_out) *blocks_out = blocks;
  return PF_OK;
}
int64_t pf_fit_camera_workspace(const pf_fit_image* images, int n) {
  WsLayout lay;
  TRY(fit_layout(images, n, &lay));
  return lay.total;
}

// Enables programmatic dependent launch for the calling thread while alive (the fit's kernels wait on their predecessor with
// griddepcontrol.wait before their first global access)
struct PdlScope {
  explicit PdlScope(bool on) { pdl_enabled() = on; }
  ~PdlScope() { pdl_enabled() = false; }
};

int pf_fit_camera(int device, const pf_fit_image* images, int n, const float* up_base, const float* lat_base, const uint8_t* mask_base,
                  int principal_point, double huber, int max_iterations, double* params, double* cost, int32_t* iterations,
                  int32_t* status, void* workspace, int64_t workspace_bytes, void* stream) {
  WsLayout lay;
  long long blocks;
  TRY(fit_layout(images, n, &lay, &blocks));
  if (!up_base || !lat_base || !params || !cost || !iterations || !status || !workspace)
    return fail(PF_ERR_ARG, "pf_fit_camera: null field / output / workspace");
  if (principal_point != 0 && principal_point != 1) return fail(PF_ERR_ARG, "pf_fit_camera: principal_point must be 0 or 1");
  if (!(huber == 0.0 || (std::isfinite(huber) && huber > 0.0)))
    return fail(PF_ERR_ARG, "pf_fit_camera: huber must be 0 (least squares) or finite and > 0, got %g", huber);
  if (max_iterations < 1 || max_iterations > kFitMaxIterations)
    return fail(PF_ERR_ARG, "pf_fit_camera: max_iterations %d outside 1 .. %d", max_iterations, kFitMaxIterations);
  TRY(check_workspace("pf_fit_camera", workspace, workspace_bytes, lay.total));
  std::vector<FitImage> d(n);
  long long block0 = 0;
  for (int i = 0; i < n; ++i) {
    const pf_fit_image& c = images[i];
    TRY(check_offsets("pf_fit_camera", i, {c.up_offset, c.lat_offset}, {{c.mask_offset, mask_base}}));
    if (c.up_stride[0] < 0 || c.up_stride[1] < 0 || c.up_stride[2] < 0) return fail(PF_ERR_ARG, "pf_fit_camera: image %d has a negative stride", i);
    if (!std::isnan(c.init[0])) {
      bool fin = true;
      for (int k = 0; k < 5; ++k) fin = fin && std::isfinite(c.init[k]);
      if (!fin || !(c.init[2] > 0.0)) return fail(PF_ERR_ARG, "pf_fit_camera: image %d: init must be finite with f_rel > 0 (or a NaN roll)", i);
    }
    FitImage& o = d[i];
    o.H = c.height; o.W = c.width;
    o.up_off = c.up_offset; o.up_sr = c.up_stride[0]; o.up_sc = c.up_stride[1]; o.up_sk = c.up_stride[2];
    o.lat_off = c.lat_offset;
    o.mask_off = c.mask_offset;
    for (int k = 0; k < 5; ++k) o.init[k] = c.init[k];
    o.block0 = (int)block0; o.nblk = (int)cdivl((long long)c.height * c.width, kFitTile);
    block0 += o.nblk;
  }
  CU(cudaSetDevice(device));
  cudaStream_t st = (cudaStream_t)stream;
  char* ws = (char*)workspace;
  FitArgs a{};
  a.im = (const FitImage*)ws; a.st = (FitState*)(ws + lay.at[1]); a.n = n; a.nblocks = (int)blocks;
  a.up = up_base; a.lat = lat_base; a.mask = mask_base;
  a.huber = huber; a.max_iter = max_iterations;
  a.part = (double*)(ws + lay.at[2]);
  a.params = params; a.cost = cost; a.iters = iterations; a.status = status;
  TRY(upload_descriptors(d.data(), d.size() * sizeof(d[0]), ws, st));
  const PdlScope pdl(!sync_debug());
  const dim3 pass_grid((unsigned)blocks), step_grid((unsigned)cdiv(n, kFitStepWarps));
  LAUNCHED(launch_pdl(fit_init_kernel, dim3(n), dim3(64), 0, st, a, principal_point));
  for (int it = 0; it < max_iterations; ++it) {
    if (principal_point) {
      LAUNCHED(launch_pdl(fit_pass_kernel<5>, pass_grid, dim3(kFitThreads), 0, st, a));
      LAUNCHED(launch_pdl(fit_step_kernel<5>, step_grid, dim3(32 * kFitStepWarps), 0, st, a));
    } else {
      LAUNCHED(launch_pdl(fit_pass_kernel<3>, pass_grid, dim3(kFitThreads), 0, st, a));
      LAUNCHED(launch_pdl(fit_step_kernel<3>, step_grid, dim3(32 * kFitStepWarps), 0, st, a));
    }
  }
  return PF_OK;
}

// ----------------------------------------------------------------------------------------------- upright warp (rectify.cuh)
// Workspace layout of pf_rectify_views: device descriptors | per-image maps
static int rectify_layout(const pf_rectify_image* im, int n, WsLayout* lay) {
  if (!im || n < 1) return fail(PF_ERR_ARG, "pf_rectify_views: null images or n < 1");
  if (n > 65535) return fail(PF_ERR_ARG, "pf_rectify_views: %d images (at most 65535 per call)", n);
  for (int i = 0; i < n; ++i) {
    const pf_rectify_image& c = im[i];
    if (c.height < 1 || c.width < 1 || (long long)c.height * c.width >= (1LL << 31))
      return fail(PF_ERR_ARG, "pf_rectify_views: image %d has input size %dx%d", i, c.height, c.width);
    if (c.out_height < 1 || c.out_width < 1 || (long long)c.out_height * c.out_width >= (1LL << 31))
      return fail(PF_ERR_ARG, "pf_rectify_views: image %d has output size %dx%d", i, c.out_height, c.out_width);
  }
  lay->add((long long)n * sizeof(RectImage)).add((long long)n * sizeof(RectMap));
  return PF_OK;
}
int64_t pf_rectify_workspace(const pf_rectify_image* images, int n) {
  WsLayout lay;
  TRY(rectify_layout(images, n, &lay));
  return lay.total;
}

int pf_rectify_views(int device, const pf_rectify_image* images, int n, const uint8_t* in_base, uint8_t* out_base, uint8_t* mask_base,
                     float* map_base, int channels, const double* params, int keep_pitch, int focal_mode, double vfov, int sampler,
                     const int32_t* fill, double* camera, int32_t* status, void* workspace, int64_t workspace_bytes, void* stream) {
  WsLayout lay;
  TRY(rectify_layout(images, n, &lay));
  if (!in_base || !out_base || !params || !camera || !status || !workspace)
    return fail(PF_ERR_ARG, "pf_rectify_views: null input / output / params / camera / status / workspace");
  if (channels != 1 && channels != 3) return fail(PF_ERR_ARG, "pf_rectify_views: %d channels (1 or 3)", channels);
  if (keep_pitch != 0 && keep_pitch != 1) return fail(PF_ERR_ARG, "pf_rectify_views: keep_pitch must be 0 or 1");
  if (focal_mode != PF_RECTIFY_SAME && focal_mode != PF_RECTIFY_VFOV && focal_mode != PF_RECTIFY_FILL)
    return fail(PF_ERR_ARG, "pf_rectify_views: unknown focal mode %d", focal_mode);
  if (focal_mode == PF_RECTIFY_VFOV && !(std::isfinite(vfov) && vfov > 0.0 && vfov < 180.0))
    return fail(PF_ERR_ARG, "pf_rectify_views: vfov %g must lie in (0, 180) degrees", vfov);
  if (sampler != PF_RECTIFY_BILINEAR && sampler != PF_RECTIFY_NEAREST) return fail(PF_ERR_ARG, "pf_rectify_views: unknown sampler %d", sampler);
  unsigned char fv[3] = {0, 0, 0};
  for (int c = 0; fill && c < channels; ++c) {
    if (fill[c] < 0 || fill[c] > 255) return fail(PF_ERR_ARG, "pf_rectify_views: fill[%d] = %d outside 0 .. 255", c, fill[c]);
    fv[c] = (unsigned char)fill[c];
  }
  TRY(check_workspace("pf_rectify_views", workspace, workspace_bytes, lay.total));
  std::vector<RectImage> d(n);
  long long max_px = 1;
  for (int i = 0; i < n; ++i) {
    const pf_rectify_image& c = images[i];
    TRY(check_offsets("pf_rectify_views", i, {c.in_offset, c.out_offset}, {{c.mask_offset, mask_base}, {c.map_offset, map_base}}));
    RectImage& o = d[i];
    o.H = c.height; o.W = c.width; o.Ho = c.out_height; o.Wo = c.out_width;
    o.in_off = c.in_offset; o.out_off = c.out_offset; o.mask_off = c.mask_offset; o.map_off = c.map_offset;
    max_px = std::max(max_px, (long long)c.out_height * c.out_width);
  }
  if (cdivl(max_px, (long long)kRectThreads * kRectPix) >= (1LL << 31)) return fail(PF_ERR_ARG, "pf_rectify_views: output too large");
  CU(cudaSetDevice(device));
  cudaStream_t st = (cudaStream_t)stream;
  char* ws = (char*)workspace;
  RectArgs a{};
  a.im = (const RectImage*)ws; a.map = (RectMap*)(ws + lay.at[1]); a.n = n;
  a.params = params; a.camera = camera; a.status = status;
  a.keep_pitch = keep_pitch; a.focal_mode = focal_mode; a.vfov = vfov;
  a.in = in_base; a.out = out_base; a.mask = mask_base; a.xy = map_base;
  for (int c = 0; c < 3; ++c) a.fill[c] = fv[c];
  TRY(upload_descriptors(d.data(), d.size() * sizeof(d[0]), ws, st));
  const PdlScope pdl(!sync_debug());
  LAUNCHED(launch_pdl(rectify_setup_kernel, dim3((unsigned)cdiv(n, 128)), dim3(128), 0, st, a));
  const dim3 grid((unsigned)cdivl(max_px, (long long)kRectThreads * kRectPix), (unsigned)n);
  const bool nearest = sampler == PF_RECTIFY_NEAREST;
  if (channels == 3)
    LAUNCHED(nearest ? launch_pdl(rectify_warp_kernel<3, true>, grid, dim3(kRectThreads), 0, st, a)
                     : launch_pdl(rectify_warp_kernel<3, false>, grid, dim3(kRectThreads), 0, st, a));
  else
    LAUNCHED(nearest ? launch_pdl(rectify_warp_kernel<1, true>, grid, dim3(kRectThreads), 0, st, a)
                     : launch_pdl(rectify_warp_kernel<1, false>, grid, dim3(kRectThreads), 0, st, a));
  return PF_OK;
}

}  // extern "C"
