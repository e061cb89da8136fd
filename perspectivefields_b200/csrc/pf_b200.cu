// libpf_b200.so -- C ABI (include/pf_b200.h) and forward orchestration of the H100-native (sm_90a) PerspectiveFields
// inference engine.  One engine per device; pf_forward enqueues the whole graph of
// perspective2d/perspectivefields.py:223-272 on the caller's stream.
#include <cctype>
#include <cmath>
#include <cstring>
#include <mutex>

#include "engine.h"
#include "attention_mma.cuh"
#include "layers.cuh"
#include "prepost.cuh"

// ----------------------------------------------------------------------------------------------- shared state (host.h)
namespace pf {

static thread_local std::string g_err;
std::atomic<long long> g_launches{0};
char g_crumb[96] = "";
thread_local KernelProf* tl_kp = nullptr;

int fail(int code, const char* fmt, ...) {
  char buf[1024];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof(buf), fmt, ap);
  va_end(ap);
  g_err = buf;
  return code;
}

int configure_device(int device) {
  static std::mutex mu;
  static std::vector<char> done;
  std::lock_guard<std::mutex> lock(mu);
  if (device < (int)done.size() && done[device]) return PF_OK;
  CU(gemm_tma_configure_device(3));
  CU(gemm_tma_configure_device(1));
  CU(attention_mma_configure_device());
  CU(cudaFuncSetAttribute(conv1_ring_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kRingSmem));
  CU(cudaFuncSetAttribute(preprocess_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kPreSmemBytes));
  CU(cudaFuncSetAttribute(postprocess_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kPostSmemMax));
  if (device >= (int)done.size()) done.resize(device + 1, 0);
  done[device] = 1;
  return PF_OK;
}
int configure_current_device() {
  int dev = 0;
  CU(cudaGetDevice(&dev));
  return configure_device(dev);
}

}  // namespace pf

// ----------------------------------------------------------------------------------------------- weight lookup
int get_w(pf_engine* e, const std::string& name, int dtype, long long numel, const void** out) {
  auto it = e->weights.find(name);
  if (it == e->weights.end()) return fail(PF_ERR_WEIGHT, "missing weight '%s'", name.c_str());
  if (it->second.dtype != dtype) return fail(PF_ERR_WEIGHT, "weight '%s': wrong dtype", name.c_str());
  if (it->second.numel != numel) return fail(PF_ERR_WEIGHT, "weight '%s': numel %lld, expected %lld", name.c_str(), it->second.numel, numel);
  *out = it->second.p;
  return PF_OK;
}
int get_f(pf_engine* e, const std::string& n, long long numel, const float** out) { return get_w(e, n, PF_F32, numel, (const void**)out); }
static int get_gemm(pf_engine* e, const std::string& n, long long N, long long K, long long nbias, GemmW* g, int groups = 1) {
  TRY(get_w(e, n + ".whi", PF_BF16, groups * N * K, (const void**)&g->hi));
  TRY(get_w(e, n + ".wlo", PF_BF16, groups * N * K, (const void**)&g->lo));
  TRY(get_f(e, n + ".b", groups * nbias, &g->b));
  return PF_OK;
}
static int get_ln(pf_engine* e, const std::string& n, int C, LnW* l) {
  TRY(get_f(e, n + ".w", C, &l->w));
  TRY(get_f(e, n + ".b", C, &l->b));
  return PF_OK;
}

static int resolve_weights(pf_engine* e) {
  char nm[128];
  TRY(get_gemm(e, "embed1g", 64, 160, 64, &e->embed1g));
  TRY(get_gemm(e, "llencg", 64, 160, 64, &e->llencg));
  for (int s = 0; s < 4; ++s) {
    const int C = kMitDims[s];
    snprintf(nm, sizeof nm, "embed%d.ln", s + 1);
    TRY(get_ln(e, nm, C, &e->embed_ln[s]));
    if (s > 0) {
      snprintf(nm, sizeof nm, "embed%d", s + 1);
      TRY(get_gemm(e, nm, C, 9LL * kMitDims[s - 1], C, &e->embed[s]));
    }
    e->blocks[s].resize(kMitDepths[s]);
    for (int i = 0; i < kMitDepths[s]; ++i) {
      MitBlockW& b = e->blocks[s][i];
      char p[64];
      snprintf(p, sizeof p, "s%d.b%d.", s + 1, i);
      std::string P(p);
      TRY(get_ln(e, P + "ln1", C, &b.ln1));
      TRY(get_gemm(e, P + "q", C, C, C, &b.q));
      if (kMitSr[s] > 1) {
        TRY(get_gemm(e, P + "sr", C, (long long)kMitSr[s] * kMitSr[s] * C, C, &b.sr));
        TRY(get_ln(e, P + "srln", C, &b.srln));
      }
      TRY(get_gemm(e, P + "kv", 2 * C, C, 2 * C, &b.kv));
      TRY(get_gemm(e, P + "proj", C, C, C, &b.proj));
      TRY(get_ln(e, P + "ln2", C, &b.ln2));
      TRY(get_gemm(e, P + "fc1", 4 * C, C, 4 * C, &b.fc1));
      TRY(get_f(e, P + "dw.w", 9LL * 4 * C, &b.dw_w));
      TRY(get_f(e, P + "dw.b", 4 * C, &b.dw_b));
      TRY(get_gemm(e, P + "fc2", C, 4 * C, C, &b.fc2));
    }
    snprintf(nm, sizeof nm, "s%d.norm", s + 1);
    TRY(get_ln(e, nm, C, &e->stage_norm[s]));
  }
  for (int l = 0; l < 4; ++l) {
    snprintf(nm, sizeof nm, "head.proc%d", l + 1);
    TRY(get_gemm(e, nm, 512, 9LL * kMitDims[l], 9 * 512, &e->proc[l]));
  }
  for (int f = 0; f < 4; ++f)
    for (int u = 0; u < 2; ++u) {
      if (f == 3 && u == 0) continue;  // fusion4 has resConfUnit2 only (gravity_head.py:102)
      for (int c = 0; c < 2; ++c) {
        snprintf(nm, sizeof nm, "head.f%d.u%d.c%d", f + 1, u + 1, c + 1);
        TRY(get_gemm(e, nm, 256, 2304, 256, &e->rcu[f][u][c], 2));
      }
    }
  TRY(get_gemm(e, "head.conv0", 64, 9 * 320, 64, &e->conv0, 2));
  TRY(get_gemm(e, "head.conv1p", 128, 9 * 64, 128, &e->conv1p, 2));
  TRY(get_f(e, "head.conv1f.w", 2LL * 9 * 64 * 32, &e->conv1f_w));
  TRY(get_f(e, "head.conv1f.b", 64, &e->conv1f_b));
  TRY(get_f(e, "head.pred_g.w", 32LL * e->desc.gravity_classes, &e->pred_g_w));
  TRY(get_f(e, "head.pred_g.b", e->desc.gravity_classes, &e->pred_g_b));
  TRY(get_f(e, "head.pred_l.w", 32LL * e->desc.latitude_classes, &e->pred_l_w));
  TRY(get_f(e, "head.pred_l.b", e->desc.latitude_classes, &e->pred_l_b));
  if (e->desc.param_net != PF_PARAM_NONE) {
    TRY(get_f(e, "pn.stem.w", 48 * 96, &e->pn_stem_w));
    TRY(get_f(e, "pn.stem.b", 96, &e->pn_stem_b));
    TRY(get_ln(e, "pn.stem.ln", 96, &e->pn_stem_ln));
    for (int k = 1; k < 4; ++k) {
      snprintf(nm, sizeof nm, "pn.ds%d.ln", k);
      TRY(get_ln(e, nm, kCnxDims[k - 1], &e->pn_ds_ln[k]));
      snprintf(nm, sizeof nm, "pn.ds%d", k);
      TRY(get_gemm(e, nm, kCnxDims[k], 4LL * kCnxDims[k - 1], kCnxDims[k], &e->pn_ds[k]));
    }
    for (int s = 0; s < 4; ++s) {
      const int C = kCnxDims[s];
      e->pn_blocks[s].resize(kCnxDepths[s]);
      e->pn_train.pw1_t[s].resize(kCnxDepths[s]);     // (filled by resolve_train_weights; sized here for the sizing dry runs)
      e->pn_train.pw2_t[s].resize(kCnxDepths[s]);
      e->pn_train.dw_rot[s].resize(kCnxDepths[s], nullptr);
      for (int j = 0; j < kCnxDepths[s]; ++j) {
        CnxBlockW& b = e->pn_blocks[s][j];
        char p[64];
        snprintf(p, sizeof p, "pn.s%d.b%d.", s, j);
        std::string P(p);
        TRY(get_f(e, P + "dw.w", 49LL * C, &b.dw_w));
        TRY(get_f(e, P + "dw.b", C, &b.dw_b));
        TRY(get_ln(e, P + "ln", C, &b.ln));
        TRY(get_gemm(e, P + "pw1", 4 * C, C, 4 * C, &b.pw1));
        TRY(get_gemm(e, P + "pw2", C, 4 * C, C, &b.pw2));
        TRY(get_f(e, P + "gamma", C, &b.gamma));
      }
    }
    TRY(get_ln(e, "pn.norm", 768, &e->pn_norm));
    TRY(get_f(e, "pn.head.w", 5 * 768, &e->pn_head_w));
    TRY(get_f(e, "pn.head.b", 5, &e->pn_head_b));
  }
  return PF_OK;
}

// ----------------------------------------------------------------------------------------------- Fwd members that launch graph kernels
int Fwd::tap_split(const char* name, const SplitT& t, long long numel) {
  if (!e->debug) return PF_OK;
  float* cp = ar.f(numel);
  if (dry) return PF_OK;
  snprintf(g_crumb, sizeof g_crumb, "%s", name);
  LAUNCHED((merge_split_kernel<<<(unsigned)cdivl(numel, 256), 256, 0, st>>>(t.hi, t.lo, cp, numel), cudaGetLastError()));
  e->taps.push_back({name, {cp, numel}});
  return PF_OK;
}
int Fwd::tconv_gather(const SplitT& A, int B, int H, int W, int Cin, int KH, int stride, int pad, const GemmW& w, int N, const Epi& o) {
  const int OH = (H + 2 * pad - KH) / stride + 1, OW = (W + 2 * pad - KH) / stride + 1;
  const long long M = (long long)B * OH * OW;
  const int K = KH * KH * Cin;
  const long long m = ar.mark();
  SplitT col = salloc(M, K);
  if (!dry) {
    if (Cin % 8) return fail(PF_ERR_ARG, "tconv_gather: Cin %% 8");
    LAUNCHED(launch_pdl(im2col_split_kernel, dim3(ew_grid(M * K / 8)), dim3(256), 0, st, A.hi, A.lo, A.ld, col.hi, col.lo, B, H, W, Cin, OH, OW, KH, stride, pad));
  }
  int r = tgemm(col, M, K, 0, w, N, o);
  ar.release(m);
  return r;
}
// The shapes layernorm_launch accepts, checked before the launch (the launcher itself fails after the launch counter has moved):
// C a multiple of 4 up to 768 and rows * C / 4 < 2^32 (the kernel's float4 indices are 32-bit); the patch order needs an RH x RW
// map that sr divides and whose images tile the rows.
static int ln_check(long long rows, int C, bool patch, int RH, int RW, int sr) {
  if (rows < 1 || C < 4 || C % 4 || C > 768 || rows * (C / 4) >= (1LL << 32)) return fail(PF_ERR_ARG, "LayerNorm: %lld rows of %d channels", rows, C);
  if (patch && (RH < 1 || RW < 1 || sr < 1 || RH % sr || RW % sr || rows % ((long long)RH * RW)))
    return fail(PF_ERR_ARG, "LayerNorm: patch order of %lld rows as %dx%d maps with sr %d", rows, RH, RW, sr);
  return PF_OK;
}
int Fwd::ln_split(const float* x, const SplitT& y, long long rows, int C, const LnW& w, float eps, float* yf) {
  TRY(ln_check(rows, C, false, 0, 0, 0));
  if (dry) return PF_OK;
  LAUNCHED(layernorm_launch(x, yf, rows, C, w.w, w.b, eps, st, y));
  return PF_OK;
}
int Fwd::ln_split_patch(const float* x, const SplitT& y, const SplitT& patch, long long rows, int C, const LnW& w, float eps, int RH, int RW, int sr, float* yf) {
  TRY(ln_check(rows, C, true, RH, RW, sr));
  if (dry) return PF_OK;
  LAUNCHED(layernorm_launch(x, yf, rows, C, w.w, w.b, eps, st, y, patch, RH, RW, sr));
  return PF_OK;
}
int Fwd::ln(const float* x, float* y, long long rows, int C, const LnW& w, float eps) {
  TRY(ln_check(rows, C, false, 0, 0, 0));
  if (dry) return PF_OK;
  LAUNCHED(layernorm_launch(x, y, rows, C, w.w, w.b, eps, st));
  return PF_OK;
}

// The element-wise kernels below form their indices in 32-bit arithmetic, most of them unsigned in float4 units, and the
// grid-stride loops advance an unsigned counter by one grid of threads: every index a kernel forms stays below 2^31, which also
// keeps that counter from wrapping.
static bool fits31(long long n) { return n >= 0 && n < (1LL << 31); }

int Fwd::dw3_gelu(const float* x, float* y, const SplitT& s, int H, int W, int C, const float* w, const float* b) {
  if (n < 1 || H < 1 || W < 1 || C < 4 || C % 4 || !fits31((long long)n * H * W * (C / 4)))
    return fail(PF_ERR_ARG, "dwconv3x3_gelu: %d images of %dx%d x %d channels", n, H, W, C);
  if (dry) return PF_OK;
  LAUNCHED(launch_pdl(dwconv3x3_gelu_kernel, dim3(ew_grid((long long)n * ((H + 1) / 2) * ((W + PF_DW3_PX - 1) / PF_DW3_PX) * (C / 4))), dim3(256), 0, st,
                      x, y, n, H, W, C, w, b, s.hi, s.lo));
  return PF_OK;
}
int Fwd::up2x(const float* x, int ldi, int icoff, float* y, int ldo, int ocoff, const SplitT& s, int H, int W, int C) {
  if (n < 1 || H < 1 || W < 1 || C < 4 || (C | ldi | icoff | ldo | ocoff) % 4 || icoff < 0 || ocoff < 0 || icoff + C > ldi || ocoff + C > ldo ||
      !fits31((long long)n * H * W * (ldi / 4)) || !fits31(4LL * n * H * W * (ldo / 4)))
    return fail(PF_ERR_ARG, "upsample2x: %d images of %dx%d, channels %d..%d of %d -> %d..%d of %d", n, H, W, icoff, icoff + C - 1, ldi, ocoff, ocoff + C - 1, ldo);
  if (dry) return PF_OK;
  LAUNCHED(launch_pdl(upsample2x_kernel, dim3(ew_grid(upsample2x_threads(n, H, W, C))), dim3(256), 0, st, x, ldi, icoff, y, ldo, ocoff, n, H, W, C, s.hi, s.lo));
  return PF_OK;
}
int Fwd::stem_gather(const float* x0, const SplitT& col, int IH, int IW, int stride) {
  const int OH = (IH - 1) / stride + 1, OW = (IW - 1) / stride + 1;     // 7 x 7, pad 3
  if (n < 1 || IH < 1 || IW < 1 || (stride != 2 && stride != 4) || !fits31(4LL * n * IH * IW) || !fits31(stem_gather_threads(n, OH, OW)))
    return fail(PF_ERR_ARG, "stem_gather: %d images of %dx%d, stride %d", n, IH, IW, stride);
  if (dry) return PF_OK;
  LAUNCHED(launch_pdl(stem_gather_kernel, dim3(ew_grid(stem_gather_threads(n, OH, OW))), dim3(256), 0, st, x0, col.hi, col.lo, n, OH, OW, stride, IH, IW));
  return PF_OK;
}
int Fwd::pn_stem(const float* pin, int SH, int SW, const float* w, const float* b, float* out) {
  if (n < 1 || SH < 4 || SW < 4 || !fits31(4LL * n * SH * SW)) return fail(PF_ERR_ARG, "ParamNet stem: %d images of %dx%d", n, SH, SW);
  if (dry) return PF_OK;
  LAUNCHED((stem_conv_launch<4, 4, 4, 0, 96>(pin, 4, n, SH, SW, w, b, out, st)));
  return PF_OK;
}
int Fwd::pack_fields(const float* grav, const float* lat, int IH, int IW, int OH, int OW, float* out) {
  if (n < 1 || IH < 1 || IW < 1 || OH < 1 || OW < 1 || !fits31((long long)IH * IW) || !fits31((long long)n * OH * OW))
    return fail(PF_ERR_ARG, "pack_fields: %d images of %dx%d -> %dx%d", n, IH, IW, OH, OW);
  if (dry) return PF_OK;
  LAUNCHED((pack_fields_kernel<<<(unsigned)cdivl((long long)n * OH * OW, 256), 256, 0, st>>>(grav, lat, out, n, IH, IW, OH, OW), cudaGetLastError()));
  return PF_OK;
}
int Fwd::param_tail(const float* feat, int HW, const LnW& norm, const float* hw, const float* hb, int kind, float* params, float* raw) {
  if (n < 1 || HW < 1 || (kind != PF_PARAM_CENTERED && kind != PF_PARAM_UNCENTERED) || !fits31(8LL * n))
    return fail(PF_ERR_ARG, "param_tail: %d images of %d pixels, kind %d", n, HW, kind);
  if (dry) return PF_OK;
  LAUNCHED((param_tail_kernel<<<n, 256, 0, st>>>(feat, HW, norm.w, norm.b, hw, hb, params, raw, kind), cudaGetLastError()));
  return PF_OK;
}
int Fwd::pred_tail(const float* in, int ldi, int icoff, const float* w, const float* b, float* out, int HW, int NC, int mode) {
  // weights and bias in shared memory (NC * 33 floats); mode 1 normalises the two channels of an up vector
  if (n < 1 || HW < 1 || NC < 1 || NC > 256 || mode < 0 || mode > 2 || (mode == 1 && NC != 2) || (ldi | icoff) % 4 || icoff < 0 || icoff + 32 > ldi ||
      !fits31((long long)n * HW))
    return fail(PF_ERR_ARG, "pred_tail: %d images of %d pixels, %d classes, mode %d, channels %d.. of %d", n, HW, NC, mode, icoff, ldi);
  if (dry) return PF_OK;
  LAUNCHED((pred_tail_kernel<<<(unsigned)cdivl((long long)n * HW, 128), 128, NC * 33 * 4, st>>>(in, ldi, icoff, w, b, out, n, HW, NC, mode), cudaGetLastError()));
  return PF_OK;
}

// ----------------------------------------------------------------------------------------------- the forward graph
constexpr long long kTableSlabBytes = 8LL << 20;   // ~370 tables of a 2048-pixel axis; reset (after a stream sync) when full
static int get_table(pf_engine* e, int in_size, int out_size, pf_engine::DevTable* out, cudaStream_t st) {
  auto it = e->tables.find({in_size, out_size});
  if (it == e->tables.end()) {
    ResampleTable t = make_resample_table(in_size, out_size);
    const long long nb = (long long)t.bounds.size() * sizeof(int), nc = (long long)t.coeffs.size() * sizeof(int);
    const long long need = ((nb + 255) & ~255LL) + ((nc + 255) & ~255LL);
    if (need > kTableSlabBytes) return fail(PF_ERR_ARG, "image axis of %d pixels is too long for the resize tables", in_size);
    if (e->table_off + need > kTableSlabBytes) {
      // slab full: earlier forwards on this stream may still read the old tables and the pinned mirror may still be the source
      // of an in-flight copy -> drain the stream once, then start over
      CU(cudaStreamSynchronize(st));
      e->tables.clear();
      e->table_off = 0;
    }
    pf_engine::DevTable d{};
    d.ksize = t.ksize;
    const long long o0 = e->table_off, o1 = o0 + ((nb + 255) & ~255LL);
    memcpy(e->table_host + o0, t.bounds.data(), nb);
    memcpy(e->table_host + o1, t.coeffs.data(), nc);
    d.bounds = (int*)(e->table_dev + o0);
    d.coeffs = (int*)(e->table_dev + o1);
    CU(cudaMemcpyAsync(e->table_dev + o0, e->table_host + o0, need, cudaMemcpyHostToDevice, st));
    e->table_off += need;
    it = e->tables.emplace(std::make_pair(in_size, out_size), d).first;
  }
  *out = it->second;
  return PF_OK;
}

static int pre_rows_needed(int H, int OH) {  // input rows one block of kPreRows output rows may need
  const double scale = (double)H / OH;
  const double support = scale < 1.0 ? 1.0 : scale;
  return (int)(kPreRows * scale) + 2 * (int)ceil(support) + 3;
}
static int pre_max_smem_rows(int OW) { return kPreSmemBytes / (OW * 3); }   // resampled rows that fit the shared-memory budget

// ----------------------------------------------------------------------------------------------- shared graph sections
// uint8 HWC (any size) or pre-resized fp32 CHW -> x0 [n,NH,NW,4] fp32 normalised (NH x NW: the engine's working size)
static int fwd_preprocess(Fwd& F, const pf_batch* bt, float*& x0, PreImage*& d_pre, PostImage*& d_post) {
  pf_engine* e = F.e;
  const pf_model_desc& D = e->desc;
  const int n = F.n;
  const bool dry = F.dry;
  cudaStream_t st = F.st;
  Arena& ar = F.ar;
  const int NH = e->net_h, NW = e->net_w;
  const int max_rows = pre_max_smem_rows(NW);
  // ---------------- pre-process: uint8 HWC (any size) -> [n,NH,NW,4] fp32 normalised -------------------
  x0 = ar.f((long long)n * NH * NW * 4);
  d_pre = (PreImage*)ar.alloc((long long)n * sizeof(PreImage));
  d_post = (PostImage*)ar.alloc((long long)n * sizeof(PostImage));
  if (!dry) {
    if (bt->images_u8) {
      std::vector<PreImage> pre(n);
      int max_h = 1;
      for (int i = 0; i < n; ++i) {
        const int H = bt->height[i], W = bt->width[i];
        if (H < 1 || W < 1) return fail(PF_ERR_ARG, "image %d has size %dx%d", i, H, W);
        pf_engine::DevTable tx, ty;
        TRY(get_table(e, W, NW, &tx, st));
        TRY(get_table(e, H, NH, &ty, st));
        if (ty.ksize + 1 > max_rows) return fail(PF_ERR_ARG, "image %d is too tall (%d rows) for the resize kernel", i, H);
        pre[i] = PreImage{bt->image_offset[i], H, W, tx.ksize, ty.ksize, tx.bounds, tx.coeffs, ty.bounds, ty.coeffs};
        if (H > max_h) max_h = H;
      }
      CU(cudaMemcpyAsync(d_pre, pre.data(), n * sizeof(PreImage), cudaMemcpyHostToDevice, st));
      int rows = pre_rows_needed(max_h, NH);
      if (rows > max_rows) rows = max_rows;
      const int smem = rows * NW * 3;
      LAUNCHED((preprocess_kernel<<<dim3(NH / kPreRows, n), NW, smem, st>>>(bt->images_u8, d_pre, x0, D.pixel_mean[0], D.pixel_mean[1],
                                                                           D.pixel_mean[2], D.pixel_std[0], D.pixel_std[1], D.pixel_std[2], rows, NH, NW),
                cudaGetLastError()));
    } else {
      const long long total = (long long)n * NH * NW;
      LAUNCHED((normalize_chw_kernel<<<(unsigned)cdivl(total, 256), 256, 0, st>>>(bt->images_chw, x0, n, NH, NW, D.pixel_mean[0], D.pixel_mean[1],
                                                                                 D.pixel_mean[2], D.pixel_std[0], D.pixel_std[1], D.pixel_std[2]),
                cudaGetLastError()));
    }
  }
  return PF_OK;
}

// resample of the (decoded) SH x SW fields (the net size) to the original sizes: one launch for all images of the batch
static int launch_postprocess(const float* vec, const float* lat, int n, int SH, int SW, const int32_t* height, const int32_t* width, const int64_t* g_off,
                              const int64_t* l_off, float* g_out, float* l_out, int lat_is_sin, PostImage* d_post, cudaStream_t st) {
  std::vector<PostImage> post(n);
  long long total = 0;
  int max_h = 1, max_wp = 4;
  for (int i = 0; i < n; ++i) {
    if (height[i] < 1 || width[i] < 1) return fail(PF_ERR_ARG, "image %d has size %dx%d", i, height[i], width[i]);
    post[i] = PostImage{height[i], width[i], g_off[i], l_off[i], total};
    total += (long long)height[i] * width[i];
    if (height[i] > max_h) max_h = height[i];
    const int wp = (width[i] + 3) / 4 * 4;
    if (wp <= kPostMaxW && wp > max_wp) max_wp = wp;    // (wider images take the table-less path of the kernel)
  }
  CU(cudaMemcpyAsync(d_post, post.data(), n * sizeof(PostImage), cudaMemcpyHostToDevice, st));
  const int smem = post_smem_bytes(SW, max_wp);
  LAUNCHED((postprocess_kernel<<<dim3((unsigned)cdiv(max_h, kPostBand), (unsigned)n), kPostThreads, smem, st>>>(vec, lat, d_post, g_out, l_out, lat_is_sin, SH, SW),
            cudaGetLastError()));
  return PF_OK;
}

// prediction 1x1 convs (+ normalise / clamp) -> NCHW outputs, then argmax decode (classification) and resample to the
// original resolutions.  conv1_out: [n,NH,NW,64] fp32 (gravity head channels 0-31, latitude head 32-63).
static int fwd_tails_post(Fwd& F, const pf_batch* bt, const float* conv1_out, PostImage* d_post, bool pred_done = false) {
  pf_engine* e = F.e;
  const pf_model_desc& D = e->desc;
  const int n = F.n;
  const bool dry = F.dry;
  cudaStream_t st = F.st;
  Arena& ar = F.ar;
  const int HW = e->net_h * e->net_w;
  const bool cls_g = D.gravity_classes != 2, cls_l = D.latitude_classes != 1;
  const bool fused_decode = e->decode_only && (cls_g || cls_l);
  if (e->decode_only && cls_g != cls_l) return fail(PF_ERR_ARG, "decode_only needs both heads to be classification heads");
  const float* vec = dry ? nullptr : bt->pred_gravity;
  const float* lat = dry ? nullptr : bt->pred_latitude;
  if (e->debug) {
    // debug taps: the raw prediction-conv outputs before normalise / clamp (oracle taps g.raw / l.raw)
    float* rg = ar.f((long long)n * D.gravity_classes * HW);
    float* rl = ar.f((long long)n * D.latitude_classes * HW);
    TRY(F.pred_tail(conv1_out, 64, 0, e->pred_g_w, e->pred_g_b, rg, HW, D.gravity_classes, 0));
    TRY(F.pred_tail(conv1_out, 64, 32, e->pred_l_w, e->pred_l_b, rl, HW, D.latitude_classes, 0));
    TRY(F.tap("head.raw_g", rg, (long long)n * D.gravity_classes * HW));
    TRY(F.tap("head.raw_l", rl, (long long)n * D.latitude_classes * HW));
  }
  if (fused_decode) {
    // option "decode_only": 1x1 conv + argmax + bin decode in one kernel; pred_gravity / pred_latitude hold the decoded fields
    if (!dry) {
      const unsigned grid = ew_grid((long long)n * HW * 4);
      LAUNCHED((pred_argmax_decode_kernel<<<grid, 256, D.gravity_classes * 37 * 4, st>>>(conv1_out, 64, 0, e->pred_g_w, e->pred_g_b, bt->pred_gravity, n, HW,
                                                                                      D.gravity_classes, 1), cudaGetLastError()));
      LAUNCHED((pred_argmax_decode_kernel<<<grid, 256, D.latitude_classes * 37 * 4, st>>>(conv1_out, 64, 32, e->pred_l_w, e->pred_l_b, bt->pred_latitude, n, HW,
                                                                                       D.latitude_classes, 0), cudaGetLastError()));
    }
  } else {
    // prediction tails -> NCHW outputs (returned to the caller)
    if (!pred_done) {
      TRY(F.pred_tail(conv1_out, 64, 0, e->pred_g_w, e->pred_g_b, dry ? nullptr : bt->pred_gravity, HW, D.gravity_classes, D.gravity_classes == 2 ? 1 : 0));
      TRY(F.pred_tail(conv1_out, 64, 32, e->pred_l_w, e->pred_l_b, dry ? nullptr : bt->pred_latitude, HW, D.latitude_classes, D.latitude_classes == 1 ? 2 : 0));
    }
    if (cls_g) {
      float* dv = ar.f((long long)n * 2 * HW);
      if (!dry) LAUNCHED((argmax_decode_kernel<<<(unsigned)cdivl((long long)n * HW, 256), 256, 0, st>>>(bt->pred_gravity, dv, n, HW, D.gravity_classes, 1), cudaGetLastError()));
      vec = dv;
    }
    if (cls_l) {
      float* dl = ar.f((long long)n * HW);
      if (!dry) LAUNCHED((argmax_decode_kernel<<<(unsigned)cdivl((long long)n * HW, 256), 256, 0, st>>>(bt->pred_latitude, dl, n, HW, D.latitude_classes, 0), cudaGetLastError()));
      lat = dl;
    }
  }
  // ---------------- post-process to the original resolutions ------------------------------------------------
  if (!dry)
    TRY(launch_postprocess(vec, lat, n, e->net_h, e->net_w, bt->height, bt->width, bt->gravity_original_offset, bt->latitude_original_offset, bt->gravity_original,
                           bt->latitude_original, cls_l ? 0 : 1, d_post, st));
  return PF_OK;
}
// =============================================================================================== the forward graph
// The whole network on the TMA -> wgmma engine: every GEMM input is a pre-split bf16 hi/lo tensor written by its producer
// (LayerNorm, attention, depthwise conv, upsample, stem gather, or the previous GEMM's epilogue).
static int run_forward(Fwd& F, const pf_batch* bt) {
  pf_engine* e = F.e;
  const pf_model_desc& D = e->desc;
  const int n = F.n;
  const bool dry = F.dry;
  cudaStream_t st = F.st;
  Arena& ar = F.ar;
  using Epi = Fwd::Epi;
  // working size NH x NW: the MiT stage grids are NH/4 x NW/4 ... NH/32 x NW/32, the attention key count of every stage is
  // (NH/32) * (NW/32) (100 at 320 x 320), the head levels run at NH/32 x NW/32 ... NH/2 x NW/2
  const int NH = e->net_h, NW = e->net_w;
  int RH[4], RW[4];
  for (int s = 0; s < 4; ++s) { RH[s] = NH >> (s + 2); RW[s] = NW >> (s + 2); }
  const int nkv = RH[3] * RW[3];

  float* x0; PreImage* d_pre; PostImage* d_post;
  {
    NvtxRange r_("pf:preprocess");
    TRY(fwd_preprocess(F, bt, x0, d_pre, d_post));
  }
  TRY(F.tap("pre", x0, (long long)n * NH * NW * 4));

  NvtxRange* sect = new NvtxRange("pf:ll_enc");
  struct SectGuard { NvtxRange*& p; ~SectGuard() { delete p; } } sect_guard{sect};
  auto section = [&](const char* name) { delete sect; sect = nullptr; sect = new NvtxRange(name); };
  SplitT cfeat[4];
  for (int s = 0; s < 4; ++s) cfeat[s] = F.salloc((long long)n * RH[s] * RW[s], kMitDims[s]);
  const int LH = NH / 2, LW = NW / 2;                 // low-level encoder / conv_fuse_conv0 grid
  SplitT ll = F.salloc((long long)n * LH * LW, 64);
  {   // conv7x7/2 (+ folded BN + ReLU) as patch gather + TMA GEMM (K = 147 padded to 160)
    const long long m = ar.mark();
    const long long M = (long long)n * LH * LW;
    SplitT col = F.salloc(M, 160);
    TRY(F.stem_gather(x0, col, NH, NW, 2));
    Epi o; o.S = ll; o.act = 1;
    TRY(F.tgemm(col, M, 160, 0, e->llencg, 64, o));
    ar.release(m);
  }
  TRY(F.tap_split("ll", ll, (long long)n * LH * LW * 64));

  // ---------------- MiT-B3 encoder ---------------------------------------------------------------------------
  for (int s = 0; s < 4; ++s) {
    { char nm[32]; snprintf(nm, sizeof nm, "pf:mit.stage%d", s + 1); section(nm); }
    const int C = kMitDims[s], N = RH[s] * RW[s], heads = kMitHeads[s], sr = kMitSr[s];
    const long long rows = (long long)n * N;
    const long long m = ar.mark();
    float* x = ar.f(rows * C);
    float* tf = ar.f(rows * C);                      // patch-embed conv output (before its LayerNorm)
    SplitT t1 = F.salloc(rows, C);                   // LayerNorm output (GEMM input only)
    SplitT t1p;                                      // the same in patch order [n*nkv, sr*sr*C]: A operand of the spatial-reduction conv
    if (sr > 1) t1p = F.salloc((long long)n * nkv, sr * sr * C);
    SplitT q = F.salloc(rows, C);                    // q and kv leave their GEMMs as split planes: the attention core's MMA operands
    SplitT a = F.salloc(rows, C);                    // attention output
    float* t2f = ar.f((long long)n * nkv * C);
    SplitT t2 = F.salloc((long long)n * nkv, C);
    SplitT kv = F.salloc((long long)n * nkv, 2 * C);
    float* h1 = ar.f(rows * 4 * C);
    SplitT h2 = F.salloc(rows, 4 * C);
    if (s == 0) {
      const long long mm = ar.mark();
      SplitT col = F.salloc(rows, 160);
      TRY(F.stem_gather(x0, col, NH, NW, 4));
      Epi o; o.C = tf; o.ldc = C;
      TRY(F.tgemm(col, rows, 160, 0, e->embed1g, 64, o));
      ar.release(mm);
    } else {
      Epi o; o.C = tf; o.ldc = C;
      TRY(F.tconv_gather(cfeat[s - 1], n, RH[s - 1], RW[s - 1], kMitDims[s - 1], 3, 2, 1, e->embed[s], C, o));
    }
    TRY(F.ln(tf, x, rows, C, e->embed_ln[s], 1e-5f));
    TRY(F.tapf(x, rows * C, "mit.s%d.embed", s + 1));
    for (int i = 0; i < kMitDepths[s]; ++i) {
      const MitBlockW& b = e->blocks[s][i];
      if (sr > 1) TRY(F.ln_split_patch(x, t1, t1p, rows, C, b.ln1, 1e-6f, RH[s], RW[s], sr));     // + the sr conv's im2col matrix
      else TRY(F.ln_split(x, t1, rows, C, b.ln1, 1e-6f));
      Epi oq, okv; oq.S = q; okv.S = kv;
      if (sr > 1) {
        { Epi o; o.C = t2f; o.ldc = C; TRY(F.tgemm(t1p, (long long)n * nkv, sr * sr * C, 0, b.sr, C, o)); }
        TRY(F.ln_split(t2f, t2, (long long)n * nkv, C, b.srln, 1e-5f));
        TRY(F.tgemm(t2, (long long)n * nkv, C, 0, b.kv, 2 * C, okv));
      }
      TRY(F.tgemm(t1, rows, C, 0, b.q, C, oq));
      if (sr == 1) TRY(F.tgemm(t1, rows, C, 0, b.kv, 2 * C, okv));
      if (!dry) LAUNCHED(attention_mma_launch(nullptr, n, N, C, heads, st, a, q, kv, F.np(), nkv));
      { Epi o; o.C = x; o.ldc = C; o.res = x; o.ldr = C; TRY(F.tgemm(a, rows, C, 0, b.proj, C, o)); }
      TRY(F.tapf(x, rows * C, "mit.s%d.b%d.attn", s + 1, i));
      TRY(F.ln_split(x, t1, rows, C, b.ln2, 1e-6f));
      { Epi o; o.C = h1; o.ldc = 4 * C; TRY(F.tgemm(t1, rows, C, 0, b.fc1, 4 * C, o)); }
      TRY(F.dw3_gelu(h1, nullptr, h2, RH[s], RW[s], 4 * C, b.dw_w, b.dw_b));
      { Epi o; o.C = x; o.ldc = C; o.res = x; o.ldr = C; TRY(F.tgemm(h2, rows, 4 * C, 0, b.fc2, C, o)); }
      TRY(F.tapf(x, rows * C, "mit.s%d.b%d", s + 1, i));
    }
    TRY(F.ln_split(x, cfeat[s], rows, C, e->stage_norm[s], 1e-6f));
    { char nm[32]; snprintf(nm, sizeof nm, "mit.c%d", s + 1); TRY(F.tap_split(nm, cfeat[s], rows * C)); }
    ar.release(m);
  }

  // ---------------- decoder heads (group 0 = gravity, group 1 = latitude, side by side in the channel dimension) ----
  float* conv1_out = ar.f((long long)n * NH * NW * 64);
  bool fuse_pred = false;
  {
    const long long m = ar.mark();
    float* fused = nullptr;       // fp32 top-down feature of the previous level, upsampled to this level's resolution
    SplitT fused_s;               // level 1 only: the final fused feature at LH x LW, split (input of conv_fuse_conv0)
    for (int lvl = 4; lvl >= 1; --lvl) {
      { char nm[32]; snprintf(nm, sizeof nm, "pf:heads.level%d", lvl); section(nm); }
      const int rh = RH[lvl - 1], rw = RW[lvl - 1], Cin = kMitDims[lvl - 1];
      const long long px = (long long)n * rh * rw;
      float* t = ar.f(px * 512);
      SplitT rt = F.salloc(px, 512);        // relu(t)
      SplitT u = F.salloc(px, 512);         // rectified conv1 outputs
      float* v = ar.f(px * 512);
      SplitT rv = F.salloc(px, 512);        // relu(v)
      float* w2 = ar.f(px * 512);
      {   // composed linear_c{lvl} o linear_c{lvl}_proc (both heads: N = 512), border-class bias
        Epi o; o.C = t; o.ldc = 512; o.S = rt; o.split_relu = 1; o.bias_mode = 2;
        TRY(F.thalo(cfeat[lvl - 1], 0, 0, nullptr, 0, 0, n, rh, rw, Cin, e->proc[lvl - 1], 512, 1, 0, o));
        TRY(F.tapf(t, px * 512, "head.proc%d", lvl));
      }
      auto rcu = [&](const SplitT& A, const GemmW& w, Epi o) {
        o.c_gcoff = 256; o.s_gcoff = 256; o.r_gcoff = 256; o.r2_gcoff = 256;
        return F.thalo(A, 0, 256, nullptr, 0, 0, n, rh, rw, 256, w, 256, 2, 256, o);
      };
      const float* of = t;
      const SplitT* os = &rt;
      if (lvl < 4) {
        { Epi o; o.S = u; o.act = 1; TRY(rcu(rt, e->rcu[lvl - 1][0][0], o)); }
        { Epi o; o.C = v; o.ldc = 512; o.S = rv; o.split_relu = 1; o.res = t; o.ldr = 512; o.res_relu = 1; o.res2 = fused; o.ldr2 = 512;
          TRY(rcu(u, e->rcu[lvl - 1][0][1], o)); }
        of = v; os = &rv;
      }
      { Epi o; o.S = u; o.act = 1; TRY(rcu(*os, e->rcu[lvl - 1][1][0], o)); }
      { Epi o; o.C = w2; o.ldc = 512; o.res = of; o.ldr = 512; o.res_relu = 1; TRY(rcu(u, e->rcu[lvl - 1][1][1], o)); }
      if (lvl > 1) {
        float* up = ar.f(px * 4 * 512);
        TRY(F.up2x(w2, 512, 0, up, 512, 0, SplitT(), rh, rw, 512));
        fused = up;
        TRY(F.tapf(up, px * 4 * 512, "head.fusion%d", lvl));
      } else {
        fused_s = F.salloc(px * 4, 512);
        TRY(F.up2x(w2, 512, 0, nullptr, 512, 0, fused_s, rh, rw, 512));
        TRY(F.tap_split("head.fusion1", fused_s, px * 4 * 512));
      }
    }
    // conv_fuse_conv0 on cat([fused, ll]) -> ReLU ; x2 ; conv_fuse_conv1 -> ReLU
    // regression heads: the 1x1 prediction conv + normalise / clamp run inside conv_fuse_conv1's epilogue (conv1's own output is
    // then only materialised for the debug taps); classification heads (73 / 180 logits) keep the separate tail kernel
    section("pf:heads.fuse_convs");
    fuse_pred = D.gravity_classes == 2 && D.latitude_classes == 1;
    const bool keep_conv1 = !fuse_pred || e->debug;   // (not `o.C != nullptr`: the sizing dry run has null pointers)
    PredTail pt[2] = {{e->pred_g_w, e->pred_g_b, dry ? nullptr : bt->pred_gravity, 2, 1}, {e->pred_l_w, e->pred_l_b, dry ? nullptr : bt->pred_latitude, 1, 2}};
    // x2 upsample folded into conv1's weights: conv1 runs on the LH x LW grid with N = 4 output phases x 32 (no upsampled
    // tensor); the two outermost output rows / columns, where the identity does not hold, are recomputed by conv1_ring_kernel
    SplitT c0s = F.salloc((long long)n * LH * LW, 128);
    {
      Epi o; o.S = c0s; o.s_gcoff = 64; o.act = 1;
      TRY(F.thalo(fused_s, 0, 256, &ll, 256, 0, n, LH, LW, 320, e->conv0, 64, 2, 64, o));
      TRY(F.tap_split("head.conv0", c0s, (long long)n * LH * LW * 128));
    }
    Epi o; o.ldc = 64; o.c_gcoff = 32; o.act = 1; o.phase4 = 1;
    if (keep_conv1) o.C = conv1_out;
    TRY(F.thalo(c0s, 0, 64, nullptr, 0, 0, n, LH, LW, 64, e->conv1p, 128, 2, 128, o, fuse_pred ? pt : nullptr));
    if (!dry) {
      const dim3 grid((unsigned)cdiv(conv1_ring_count(NH, NW), kRingPx), (unsigned)n);
      LAUNCHED((conv1_ring_kernel<<<grid, 256, kRingSmem, st>>>(c0s.hi, c0s.lo, LH, LW, e->conv1f_w, e->conv1f_b, keep_conv1 ? conv1_out : nullptr,
                                                               fuse_pred ? e->pred_g_w : nullptr, e->pred_g_b, bt->pred_gravity,
                                                               fuse_pred ? e->pred_l_w : nullptr, e->pred_l_b, bt->pred_latitude), cudaGetLastError()));
    }
    if (keep_conv1) TRY(F.tap("head.conv1", conv1_out, (long long)n * NH * NW * 64));
    ar.release(m);
  }
  section("pf:tails_postprocess");
  TRY(fwd_tails_post(F, bt, conv1_out, d_post, fuse_pred));

  // ---------------- ParamNet (ConvNeXt-T on the predicted fields) -------------------------------------------
  if (D.param_net != PF_PARAM_NONE) {
    section("pf:paramnet");
    TRY(fwd_paramnet(F, dry ? nullptr : bt->pred_gravity, dry ? nullptr : bt->pred_latitude, dry ? nullptr : bt->params, nullptr));
  }
  return PF_OK;
}

// ParamNet (ConvNeXt-T) on fields at the working size, the last section of pf_forward (on the heads' outputs) and all of
// pf_param_forward (on the caller's fields): grav [n,2,NH,NW] up vectors, lat [n,1,NH,NW] sin(latitude) -> params [n,8]
// (pf_batch.params layout) and, when raw is non-NULL, the head's five outputs before any scaling as [n,5].
int fwd_paramnet(Fwd& F, const float* grav, const float* lat, float* params, float* raw, const PnSaved* sv) {
  pf_engine* e = F.e;
  const pf_model_desc& D = e->desc;
  const int n = F.n;
  const bool dry = F.dry;
  cudaStream_t st = F.st;
  Arena& ar = F.ar;
  using Epi = Fwd::Epi;
  const int NH = e->net_h, NW = e->net_w;
  {
    if (D.gravity_classes != 2 || D.latitude_classes != 1) return fail(PF_ERR_ARG, "ParamNet needs regression heads");
    // centered: ConvNeXt on the fields at the net size; uncentered: nearest resample to INPUT_SIZE x INPUT_SIZE first
    const bool centered = D.param_net == PF_PARAM_CENTERED;
    const int SH = centered ? NH : D.param_input_size, SW = centered ? NW : D.param_input_size;
    float* pin = sv ? sv->pin : ar.f((long long)n * SH * SW * 4);
    TRY(F.pack_fields(grav, lat, NH, NW, SH, SW, pin));
    int rh = SH / 4, rw = SW / 4;
    float* x = sv ? sv->xs[0][0] : ar.f((long long)n * rh * rw * 96);
    float* stem = sv ? sv->stem_pre : x;
    TRY(F.pn_stem(pin, SH, SW, e->pn_stem_w, e->pn_stem_b, stem));
    TRY(F.ln(stem, x, (long long)n * rh * rw, 96, e->pn_stem_ln, 1e-6f));
    for (int s = 0; s < 4; ++s) {
      const int C = kCnxDims[s];
      if (s > 0) {
        const int r2h = rh / 2, r2w = rw / 2;
        SplitT y = F.salloc((long long)n * r2h * r2w, 4 * kCnxDims[s - 1]);      // LayerNorm output written directly as the 2x2/2 conv's im2col matrix
        TRY(F.ln_split_patch(x, SplitT(), y, (long long)n * rh * rw, kCnxDims[s - 1], e->pn_ds_ln[s], 1e-6f, rh, rw, 2));
        float* xn = sv ? sv->xs[s][0] : ar.f((long long)n * r2h * r2w * C);
        Epi o; o.C = xn; o.ldc = C;
        TRY(F.tgemm(y, (long long)n * r2h * r2w, 4 * kCnxDims[s - 1], 0, e->pn_ds[s], C, o));
        x = xn; rh = r2h; rw = r2w;
      }
      const long long rows = (long long)n * rh * rw;
      float* yf = ar.f(rows * C);
      SplitT y = F.salloc(rows, C);
      SplitT h = F.salloc(rows, 4 * C);
      for (int j = 0; j < kCnxDepths[s]; ++j) {
        const CnxBlockW& b = e->pn_blocks[s][j];
        TRY(pn_dw_launch(F, x, yf, rh, rw, C, b.dw_w, b.dw_b));
        TRY(F.ln_split(yf, y, rows, C, b.ln, 1e-6f));
        { Epi o; o.S = h; o.act = 2; TRY(F.tgemm(y, rows, C, 0, b.pw1, 4 * C, o)); }
        float* xo = sv ? sv->xs[s][j + 1] : x;     // training keeps every block's input: out of place, same arithmetic
        { Epi o; o.C = xo; o.ldc = C; o.res = x; o.ldr = C; o.gamma = b.gamma; TRY(F.tgemm(h, rows, 4 * C, 0, b.pw2, C, o)); }
        x = xo;
      }
      TRY(F.tapf(x, rows * C, "cnx.s%d", s));
    }
    if (!dry && !params) return fail(PF_ERR_ARG, "params output is NULL");
    TRY(F.param_tail(x, rh * rw, e->pn_norm, e->pn_head_w, e->pn_head_b, D.param_net, params, raw));
  }
  return PF_OK;
}

int pn_dw_launch(Fwd& F, const float* x, float* y, int rh, int rw, int C, const float* w, const float* b) {
  if (F.n < 1 || rh < 1 || rw < 1 || C < 4 || C % 4 || !fits31((long long)F.n * rh * rw * (C / 4)))
    return fail(PF_ERR_ARG, "dwconv7x7: %d images of %dx%d x %d channels", F.n, rh, rw, C);
  if (!F.dry) LAUNCHED(launch_pdl(dwconv7x7_kernel, dim3(ew_grid((long long)F.n * ((rh + 1) / 2) * ((rw + PF_DW7_PX - 1) / PF_DW7_PX) * (C / 4))), dim3(256), 0, F.st,
                                  x, y, F.n, rh, rw, C, w, b));
  return PF_OK;
}

// ----------------------------------------------------------------------------------------------- C ABI
extern "C" {

int pf_abi_version(void) { return PF_ABI_VERSION; }
const char* pf_last_error(void) { return g_err.c_str(); }
int64_t pf_kernel_launch_count(void) { return g_launches.load(); }

// a working size the engine supports: H and W multiples of 32 in [64, 640] (the smallest head level is then at least 2 x 2, which
// the border-class bias needs) with at most kAmMaxKeys attention keys (H/32) * (W/32)
static bool net_size_ok(int h, int w) {
  return h >= 64 && w >= 64 && h <= 640 && w <= 640 && h % 32 == 0 && w % 32 == 0 && (h / 32) * (w / 32) <= kAmMaxKeys;
}

int pf_create(int device, const pf_model_desc* desc, pf_handle* out) { return pf_create_sized(device, desc, kNet, kNet, out); }

int pf_create_sized(int device, const pf_model_desc* desc, int net_h, int net_w, pf_handle* out) {
  if (!desc || !out) return fail(PF_ERR_ARG, "pf_create: null argument");
  if (!net_size_ok(net_h, net_w))
    return fail(PF_ERR_ARG, "pf_create: working size %dx%d: height and width must be multiples of 32 in [64, 640] with (H/32)*(W/32) <= %d", net_h, net_w, kAmMaxKeys);
  if (!((desc->gravity_classes == 2 || desc->gravity_classes == 73) && (desc->latitude_classes == 1 || desc->latitude_classes == 180)))
    return fail(PF_ERR_ARG, "pf_create: unsupported head widths %d/%d", desc->gravity_classes, desc->latitude_classes);
  if (desc->param_net < 0 || desc->param_net > 2) return fail(PF_ERR_ARG, "pf_create: bad param_net");
  if (desc->param_net == PF_PARAM_UNCENTERED && (desc->param_input_size < 32 || desc->param_input_size > kNet || desc->param_input_size % 32))
    return fail(PF_ERR_ARG, "pf_create: param_input_size must be a multiple of 32 in [32, 320]");
  int count = 0;
  CU(cudaGetDeviceCount(&count));
  if (device < 0 || device >= count) return fail(PF_ERR_CUDA, "pf_create: no CUDA device %d (found %d)", device, count);
  CU(cudaSetDevice(device));
  cudaDeviceProp prop;
  CU(cudaGetDeviceProperties(&prop, device));
  if (prop.major != 9 || prop.minor != 0) return fail(PF_ERR_CUDA, "pf_create: device %d is sm_%d%d; this library is built for sm_90a only", device, prop.major, prop.minor);
  TRY(configure_device(device));
  pf_engine* e = new pf_engine();
  e->device = device;
  e->sm_count = prop.multiProcessorCount;
  e->desc = *desc;
  e->net_h = net_h;
  e->net_w = net_w;
  if (cudaMalloc(&e->table_dev, kTableSlabBytes) != cudaSuccess || cudaMallocHost(&e->table_host, kTableSlabBytes) != cudaSuccess) {
    const int r = fail(PF_ERR_CUDA, "pf_create: resize-table slab: %s", cudaGetErrorString(cudaGetLastError()));
    cudaFree(e->table_dev);
    delete e;
    return r;
  }
  *out = e;
  return PF_OK;
}

int pf_destroy(pf_handle h) {
  if (!h) return PF_OK;
  cudaSetDevice(h->device);
  cudaFree(h->table_dev);
  cudaFreeHost(h->table_host);
  for (auto& r : h->prof) { cudaEventDestroy(r.a); cudaEventDestroy(r.b); }
  for (auto ev : h->ev_pool) cudaEventDestroy(ev);
  for (auto ev : h->kp.pool) cudaEventDestroy(ev);
  delete h;
  return PF_OK;
}

int pf_set_weight(pf_handle h, const char* name, const void* dev_ptr, int64_t numel, int dtype) {
  if (!h || !name || !dev_ptr) return fail(PF_ERR_ARG, "pf_set_weight: null argument");
  if (((uintptr_t)dev_ptr & 15) != 0) return fail(PF_ERR_ARG, "pf_set_weight: '%s' is not 16-byte aligned", name);
  h->weights[name] = WeightRef{dev_ptr, numel, dtype};
  h->finalized = false;
  return PF_OK;
}

int pf_finalize(pf_handle h) {
  if (!h) return fail(PF_ERR_ARG, "pf_finalize: null handle");
  TRY(resolve_weights(h));
  h->finalized = true;
  return PF_OK;
}

int64_t pf_workspace_bytes(pf_handle h, int n, int max_h) {
  if (!h || n < 1) return fail(PF_ERR_ARG, "pf_workspace_bytes: bad argument");
  Fwd F{h, Arena{}, nullptr, true, n};
  F.ar.dry = true;
  F.ar.keep = h->debug;
  (void)max_h;
  int r = run_forward(F, nullptr);
  if (r != PF_OK) return r;
  return F.ar.peak + 4096;
}

int pf_forward(pf_handle h, const pf_batch* bt, void* workspace, int64_t workspace_bytes, void* stream) {
  if (!h || !bt || !workspace) return fail(PF_ERR_ARG, "pf_forward: null argument");
  if (!h->finalized) return fail(PF_ERR_WEIGHT, "pf_forward: pf_finalize has not succeeded");
  if (bt->n < 1) return fail(PF_ERR_ARG, "pf_forward: empty batch");
  if ((bt->images_u8 != nullptr) == (bt->images_chw != nullptr)) return fail(PF_ERR_ARG, "pf_forward: exactly one of images_u8 / images_chw");
  if (bt->images_u8 && !bt->image_offset) return fail(PF_ERR_ARG, "pf_forward: image_offset is NULL");
  if (!bt->height || !bt->width || !bt->pred_gravity || !bt->pred_latitude || !bt->gravity_original || !bt->latitude_original ||
      !bt->gravity_original_offset || !bt->latitude_original_offset)
    return fail(PF_ERR_ARG, "pf_forward: null input/output pointer");
  CU(cudaSetDevice(h->device));
  Fwd F{h, Arena{}, (cudaStream_t)stream, false, bt->n};
  F.ar.base = (char*)workspace;
  F.ar.cap = workspace_bytes;
  F.ar.keep = h->debug;
  {  // capacity check with a dry run (cheap: no launches)
    Fwd T{h, Arena{}, nullptr, true, bt->n};
    T.ar.dry = true; T.ar.keep = h->debug;
    TRY(run_forward(T, nullptr));
    if (T.ar.peak > workspace_bytes) return fail(PF_ERR_WORKSPACE, "pf_forward: workspace %lld B < required %lld B", (long long)workspace_bytes, T.ar.peak);
  }
  if (((uintptr_t)workspace & 255) != 0) return fail(PF_ERR_ARG, "pf_forward: workspace must be 256-byte aligned");
  h->taps.clear();
  h->kp.st = (cudaStream_t)stream;
  tl_kp = &h->kp;
  pdl_enabled() = h->use_pdl && !h->kp.on && !h->profile && !sync_debug();   // (event records between launches defeat it anyway)
  const int r = run_forward(F, bt);
  pdl_enabled() = false;
  tl_kp = nullptr;
  return r;
}

// ParamNet alone on the caller's fields: the sizing dry run of fwd_paramnet (no launches)
static int param_peak(pf_handle h, int n, long long* peak) {
  Fwd T{h, Arena{}, nullptr, true, n};
  T.ar.dry = true;
  T.ar.keep = h->debug;
  TRY(fwd_paramnet(T, nullptr, nullptr, nullptr, nullptr));
  *peak = T.ar.peak;
  return PF_OK;
}

int64_t pf_param_workspace_bytes(pf_handle h, int n) {
  if (!h || n < 1) return fail(PF_ERR_ARG, "pf_param_workspace_bytes: bad argument");
  if (h->desc.param_net == PF_PARAM_NONE) return fail(PF_ERR_ARG, "pf_param_workspace_bytes: this model has no ParamNet");
  long long peak = 0;
  TRY(param_peak(h, n, &peak));
  return peak + 4096;
}

int pf_param_forward(pf_handle h, int n, const float* gravity, const float* latitude, float* params, float* raw, void* workspace,
                     int64_t workspace_bytes, void* stream) {
  if (!h) return fail(PF_ERR_ARG, "pf_param_forward: null handle");
  if (!h->finalized) return fail(PF_ERR_WEIGHT, "pf_param_forward: pf_finalize has not succeeded");
  if (h->desc.param_net == PF_PARAM_NONE) return fail(PF_ERR_ARG, "pf_param_forward: this model has no ParamNet");
  if (n < 1) return fail(PF_ERR_ARG, "pf_param_forward: n = %d, at least 1 pair of fields is needed", n);
  if (!gravity || !latitude || !params || !workspace) return fail(PF_ERR_ARG, "pf_param_forward: null gravity / latitude / params / workspace");
  long long peak = 0;
  TRY(param_peak(h, n, &peak));
  if (peak > workspace_bytes) return fail(PF_ERR_ARG, "pf_param_forward: workspace %lld B < required %lld B", (long long)workspace_bytes, peak);
  if (((uintptr_t)workspace & 255) != 0) return fail(PF_ERR_ARG, "pf_param_forward: workspace must be 256-byte aligned");
  CU(cudaSetDevice(h->device));
  Fwd F{h, Arena{}, (cudaStream_t)stream, false, n};
  F.ar.base = (char*)workspace;
  F.ar.cap = workspace_bytes;
  F.ar.keep = h->debug;
  h->taps.clear();
  h->kp.st = (cudaStream_t)stream;
  tl_kp = &h->kp;
  pdl_enabled() = h->use_pdl && !h->kp.on && !h->profile && !sync_debug();
  int r;
  {
    NvtxRange r_("pf:paramnet");
    r = fwd_paramnet(F, gravity, latitude, params, raw);
  }
  pdl_enabled() = false;
  tl_kp = nullptr;
  return r;
}

int pf_profile_enable(pf_handle h, int on) {
  if (!h) return fail(PF_ERR_ARG, "null handle");
  h->profile = on != 0;
  // `on` > 1: pre-create the CUDA events for that many GEMM launches now, so none is created inside a timed region
  while (on > 1 && (long long)h->ev_pool.size() < 2LL * on) {
    cudaEvent_t ev;
    CU(cudaEventCreate(&ev));
    h->ev_pool.push_back(ev);
  }
  return PF_OK;
}
int pf_profile_kernels_enable(pf_handle h, int max_launches) {
  if (!h) return fail(PF_ERR_ARG, "null handle");
  CU(cudaSetDevice(h->device));
  KernelProf& kp = h->kp;
  kp.on = max_launches > 0;
  kp.used = 0;
  kp.recs.clear();
  while ((long long)kp.pool.size() < 2LL * max_launches) {
    cudaEvent_t ev;
    CU(cudaEventCreate(&ev));
    kp.pool.push_back(ev);
  }
  return PF_OK;
}
// text table "kernel,launches,ms\n" aggregated over the launches recorded since pf_profile_kernels_enable; the caller must have
// synchronised the stream.  Returns the number of bytes written (excluding the terminating NUL) or a negative status.
int pf_profile_kernels_read(pf_handle h, char* buf, int cap) {
  if (!h || !buf || cap < 1) return fail(PF_ERR_ARG, "pf_profile_kernels_read: bad argument");
  std::map<std::string, std::pair<int, double>> agg;
  std::vector<std::string> order;
  for (const auto& r : h->kp.recs) {
    float ms = 0.f;
    CU(cudaEventElapsedTime(&ms, r.a, r.b));
    const char* c = r.expr;
    while (*c == '(' || *c == ' ') ++c;
    const char* e = c;
    while (*e && (isalnum((unsigned char)*e) || *e == '_')) ++e;
    std::string name(c, e);
    if (name == "launch_pdl" && *e == '(') {   // launch_pdl(kernel, grid, ...): the kernel is the first argument
      c = e + 1;
      e = c;
      while (*e && (isalnum((unsigned char)*e) || *e == '_')) ++e;
      name.assign(c, e);
    }
    // template arguments of direct kernel launches distinguish the variants (e.g. stem_conv_launch<4, 4, 4, 0, 96>)
    if (*e == '<' && e[1] != '<') { const char* t = strchr(e, '>'); if (t) name.append(e, t + 1); }
    auto it = agg.find(name);
    if (it == agg.end()) { order.push_back(name); it = agg.emplace(name, std::make_pair(0, 0.0)).first; }
    it->second.first += 1;
    it->second.second += ms;
  }
  std::string out = "kernel,launches,ms\n";
  for (const auto& n : order) {
    char line[256];
    snprintf(line, sizeof line, "%s,%d,%.4f\n", n.c_str(), agg[n].first, agg[n].second);
    out += line;
  }
  if ((int)out.size() + 1 > cap) return fail(PF_ERR_ARG, "pf_profile_kernels_read: buffer too small (%d needed)", (int)out.size() + 1);
  memcpy(buf, out.c_str(), out.size() + 1);
  h->kp.used = 0;
  h->kp.recs.clear();
  return (int)out.size();
}
int pf_set_option(pf_handle h, const char* name, int value) {
  if (!h || !name) return fail(PF_ERR_ARG, "pf_set_option: null argument");
  if (!strcmp(name, "decode_only")) { h->decode_only = value != 0; return PF_OK; }
  if (!strcmp(name, "pdl")) { h->use_pdl = value != 0; return PF_OK; }
  if (!strcmp(name, "bf16")) { h->bf16 = value != 0; return PF_OK; }
  return fail(PF_ERR_ARG, "pf_set_option: unknown option '%s'", name);
}
// out[cfg*3 + {0,1,2}] = {milliseconds, algorithmic FLOPs, launches} per GEMM engine configuration (7 configs),
// accumulated since the last read; the caller must have synchronised the stream.
int pf_profile_read(pf_handle h, double* out9) {
  if (!h || !out9) return fail(PF_ERR_ARG, "pf_profile_read: null argument");
  for (int i = 0; i < 21; ++i) out9[i] = 0.0;
  FILE* csv = nullptr;
  if (const char* path = getenv("PF_PROFILE_CSV")) {   // optional per-launch dump
    csv = fopen(path, "w");
    if (csv) fprintf(csv, "engine_cfg,M,N,K,Cin,KH,stride,groups,ms,algorithmic_tflops\n");
  }
  for (auto& r : h->prof) {
    float ms = 0.f;
    CU(cudaEventSynchronize(r.b));
    CU(cudaEventElapsedTime(&ms, r.a, r.b));
    if (csv) fprintf(csv, "%d,%d,%d,%d,%d,%d,%d,%d,%.4f,%.1f\n", r.cfg, r.M, r.N, r.K, r.Cin, r.KH, r.stride, r.groups, ms, r.flops / (ms * 1e9));
    out9[r.cfg * 3 + 0] += ms;
    out9[r.cfg * 3 + 1] += r.flops;
    out9[r.cfg * 3 + 2] += 1.0;
    h->ev_pool.push_back(r.a);
    h->ev_pool.push_back(r.b);
  }
  if (csv) fclose(csv);
  h->prof.clear();
  return PF_OK;
}

int pf_debug_enable(pf_handle h, int on) {
  if (!h) return fail(PF_ERR_ARG, "null handle");
  h->debug = on != 0;
  h->taps.clear();
  return PF_OK;
}
int pf_debug_count(pf_handle h) { return h ? (int)h->taps.size() : 0; }
const char* pf_debug_name(pf_handle h, int i) { return (h && i >= 0 && i < (int)h->taps.size()) ? h->taps[i].first.c_str() : ""; }
int64_t pf_debug_numel(pf_handle h, const char* name) {
  if (!h || !name) return -1;
  for (auto& t : h->taps) if (t.first == name) return t.second.second;
  return -1;
}
int pf_debug_copy(pf_handle h, const char* name, float* dst, int64_t numel, void* stream) {
  if (!h || !name || !dst) return fail(PF_ERR_ARG, "pf_debug_copy: null argument");
  for (auto& t : h->taps)
    if (t.first == name) {
      if (numel != t.second.second) return fail(PF_ERR_ARG, "pf_debug_copy: '%s' has %lld elements", name, t.second.second);
      CU(cudaMemcpyAsync(dst, t.second.first, numel * 4, cudaMemcpyDeviceToDevice, (cudaStream_t)stream));
      return PF_OK;
    }
  return fail(PF_ERR_ARG, "pf_debug_copy: no tap '%s'", name);
}

}  // extern "C"

// ----------------------------------------------------------------------------------------------- single-operator entry points
int op_engine(pf_engine& e, bool bf16) {
  TRY(configure_current_device());
  CU(cudaGetDevice(&e.device));
  CU(cudaDeviceGetAttribute(&e.sm_count, cudaDevAttrMultiProcessorCount, e.device));
  e.bf16 = bf16;
  return PF_OK;
}

static bool al16(const void* p) { return ((uintptr_t)p & 15) == 0; }

// a host array copied into the op's scratch on its stream
template <class T>
static int op_upload(Fwd& F, const T* src, size_t count, T** dst) {
  *dst = (T*)F.ar.alloc((long long)(count * sizeof(T)));
  if (!F.dry) CU(cudaMemcpyAsync(*dst, src, count * sizeof(T), cudaMemcpyHostToDevice, F.st));
  return PF_OK;
}

extern "C" {

int pf_op_conv_gemm(const float* x, int B, int H, int W, int Cin, const void* whi, const void* wlo, const float* bias, int N, int KH, int KW,
                    int stride, int pad, int in_relu, int act, const float* res, int res_relu, float* y, void* stream) {
  // split the input the way a producer kernel would, then run the same helpers the forward graph uses
  if (!x || !whi || !wlo || !y) return fail(PF_ERR_ARG, "pf_op_conv_gemm: null argument");
  if (KH != KW) return fail(PF_ERR_ARG, "pf_op_conv_gemm: square filters only");
  const GemmW w{(const __nv_bfloat16*)whi, (const __nv_bfloat16*)wlo, bias};
  Fwd::Epi o;
  o.C = y; o.ldc = N; o.act = act; o.res = res; o.ldr = N; o.res_relu = res_relu;
  return op_run("pf_op_conv_gemm", B, stream, [&](Fwd& F) -> int {
    const long long nx = (long long)B * H * W * Cin;
    SplitT A = F.salloc((long long)B * H * W, Cin);
    if (!F.dry) LAUNCHED((split_kernel<<<(unsigned)cdivl(nx, 256), 256, 0, F.st>>>(x, A.hi, A.lo, nx, in_relu), cudaGetLastError()));
    if (KH == 3 && stride == 1 && pad == 1 && Cin % 64 == 0) return F.thalo(A, 0, 0, nullptr, 0, 0, B, H, W, Cin, w, N, 1, 0, o);
    if (KH == 1 && stride == 1 && pad == 0) return F.tgemm(A, (long long)B * H * W, Cin, 0, w, N, o);
    return F.tconv_gather(A, B, H, W, Cin, KH, stride, pad, w, N, o);
  });
}
static int op_tma(pf_tma_op* op, void* stream, bool bf16) {
  if (!op || !op->a_hi || !op->a_lo || !op->w_hi || !op->w_lo) return fail(PF_ERR_ARG, "pf_op_tma: null argument");
  const pf_tma_op& q = *op;
  if (q.mode != MODE_GEMM && q.mode != MODE_HALO) return fail(PF_ERR_ARG, "pf_op_tma: mode %d", q.mode);
  if (!q.C && !q.s_hi) return fail(PF_ERR_ARG, "pf_op_tma: no output (C and S are both NULL)");
  if (!q.s_hi != !q.s_lo || !q.a2_hi != !q.a2_lo) return fail(PF_ERR_ARG, "pf_op_tma: a split pair needs both planes");
  if (q.bias_mode < 0 || q.bias_mode > 2 || q.act < 0 || q.act > 2) return fail(PF_ERR_ARG, "pf_op_tma: bias_mode %d / act %d", q.bias_mode, q.act);
  if (q.groups < 1 || q.groups > 2 || q.N < 1) return fail(PF_ERR_ARG, "pf_op_tma: groups %d, N %d", q.groups, q.N);
  if (q.npred != 0 && q.npred != q.groups) return fail(PF_ERR_ARG, "pf_op_tma: npred must be 0 or groups");
  if (q.mode == MODE_GEMM && (q.groups != 1 || q.a2_hi || q.phase4 || q.npred || q.M < 1 || q.M > INT32_MAX))
    return fail(PF_ERR_ARG, "pf_op_tma: GEMM mode runs one group of 1..2^31-1 rows without A2, phase4 or prediction tail");
  if (q.mode == MODE_HALO && (q.B < 1 || q.H < 1 || q.W < 1)) return fail(PF_ERR_ARG, "pf_op_tma: image size %dx%dx%d", q.B, q.H, q.W);
  pf_engine tmp;
  TRY(op_engine(tmp, bf16));
  Fwd F{&tmp, Arena{}, (cudaStream_t)stream, false, q.B};
  if (q.force_sched < 0 || q.force_sched > 2 || (q.force_sched && q.mode != MODE_GEMM)) return fail(PF_ERR_ARG, "pf_op_tma: force_sched %d", q.force_sched);
  F.force_bn = q.force_bn; F.force_kb = q.force_kb; F.force_sched = q.force_sched;
  const SplitT A{(__nv_bfloat16*)q.a_hi, (__nv_bfloat16*)q.a_lo, q.lda};
  const SplitT A2{(__nv_bfloat16*)q.a2_hi, (__nv_bfloat16*)q.a2_lo, q.lda2};
  const GemmW w{(const __nv_bfloat16*)q.w_hi, (const __nv_bfloat16*)q.w_lo, q.bias};
  Fwd::Epi o;
  o.C = q.C; o.ldc = q.ldc; o.c_coff = q.c_coff; o.c_gcoff = q.c_gcoff;
  o.S = SplitT{(__nv_bfloat16*)q.s_hi, (__nv_bfloat16*)q.s_lo, q.lds}; o.s_coff = q.s_coff; o.s_gcoff = q.s_gcoff; o.split_relu = q.split_relu;
  o.act = q.act; o.gamma = q.gamma;
  o.res = q.res; o.ldr = q.ldr; o.r_coff = q.r_coff; o.r_gcoff = q.r_gcoff; o.res_relu = q.res_relu;
  o.res2 = q.res2; o.ldr2 = q.ldr2; o.r2_coff = q.r2_coff; o.r2_gcoff = q.r2_gcoff;
  o.bias_mode = q.bias_mode; o.phase4 = q.phase4;
  PredTail pt[2];
  for (int g = 0; g < q.npred; ++g) {
    const pf_tma_pred& s = q.pred[g];
    if (!s.w || !s.b || !s.out || !(s.mode == 1 ? s.nc == 2 : (s.mode == 2 && s.nc == 1))) return fail(PF_ERR_ARG, "pf_op_tma: prediction tail %d", g);
    pt[g] = PredTail{s.w, s.b, s.out, s.nc, s.mode};
  }
  op->picked_bn = op->picked_kb = op->picked_sched = 0;
  const int r = q.mode == MODE_GEMM ? F.tgemm(A, q.M, q.K, q.a_c0, w, q.N, o)
                                    : F.thalo(A, q.a_c0, q.a_gc, q.a2_hi ? &A2 : nullptr, q.c_split, q.a2_c0, q.B, q.H, q.W, q.Cin, w, q.N, q.groups,
                                              q.bias_gstride, o, q.npred ? pt : nullptr);
  if (r == PF_OK) { op->picked_bn = F.picked_bn; op->picked_kb = F.picked_kb; op->picked_sched = F.picked_sched; }
  return r;
}
int pf_op_tma(pf_tma_op* op, void* stream) { return op_tma(op, stream, false); }
int pf_op_tma_bf16(pf_tma_op* op, void* stream) { return op_tma(op, stream, true); }
int pf_op_conv1_ring(const void* c_hi, const void* c_lo, int B, int H, int W, const float* wf, const float* bias, float* out,
                     const float* pg_w, const float* pg_b, float* pg_out, const float* pl_w, const float* pl_b, float* pl_out, void* stream) {
  if (!c_hi || !c_lo || !wf || !bias) return fail(PF_ERR_ARG, "pf_op_conv1_ring: null argument");
  const bool tail = pg_w || pg_b || pg_out || pl_w || pl_b || pl_out;
  if (tail && !(pg_w && pg_b && pg_out && pl_w && pl_b && pl_out)) return fail(PF_ERR_ARG, "pf_op_conv1_ring: the prediction tail needs all six pointers");
  if (!out && !tail) return fail(PF_ERR_ARG, "pf_op_conv1_ring: no output");
  // the ring is the two outermost rows / columns of the 2H x 2W output: it needs two of each
  if (B < 1 || H < 2 || W < 2) return fail(PF_ERR_ARG, "pf_op_conv1_ring: needs B >= 1 and H, W >= 2 (got %dx%dx%d)", B, H, W);
  TRY(configure_current_device());
  const dim3 grid((unsigned)cdiv(conv1_ring_count(2 * H, 2 * W), kRingPx), (unsigned)B);
  LAUNCHED((conv1_ring_kernel<<<grid, 256, kRingSmem, (cudaStream_t)stream>>>((const __nv_bfloat16*)c_hi, (const __nv_bfloat16*)c_lo, H, W, wf, bias, out,
                                                                             pg_w, pg_b, pg_out, pl_w, pl_b, pl_out), cudaGetLastError()));
  return PF_OK;
}
int pf_tma_pick_tile(int mode, int64_t M, int N, int K, int sm_count, int* bn, int* kb) {
  if (!bn || !kb || (mode != MODE_GEMM && mode != MODE_HALO) || N < 1 || K < 1 || sm_count < 1) return fail(PF_ERR_ARG, "pf_tma_pick_tile: bad argument");
  tma_pick_tile(mode, M, N, K, sm_count, *bn, *kb);
  return PF_OK;
}
int pf_camera_fields(int device, const pf_camera* cams, int n, float* up, float* lat, void* stream) {
  return pf_camera_fields_vp(device, cams, nullptr, n, up, lat, stream);
}
int pf_camera_fields_vp(int device, const pf_camera* cams, const double* vp, int n, float* up, float* lat, void* stream) {
  if (!cams || n < 1 || (!up && !lat)) return fail(PF_ERR_ARG, "pf_camera_fields: bad argument");
  if (vp) {
    for (int i = 0; i < n; ++i)
      if (std::isfinite(vp[2 * i]) != std::isfinite(vp[2 * i + 1]))
        return fail(PF_ERR_ARG, "pf_camera_fields_vp: image %d: a vanishing point needs two finite coordinates (or two NaN)", i);
  }
  CU(cudaSetDevice(device));
  for (int i0 = 0; i0 < n; i0 += kCamChunk) {
    const int m = n - i0 < kCamChunk ? n - i0 : kCamChunk;
    CamBatch b{};
    long long max_q = 1;
    for (int i = 0; i < m; ++i) {
      const pf_camera& c = cams[i0 + i];
      if (c.height < 1 || c.width < 1 || !(c.focal_rel != 0.0)) return fail(PF_ERR_ARG, "pf_camera_fields: image %d: size %dx%d, focal %g", i0 + i, c.height, c.width, c.focal_rel);
      if ((c.up_offset & 1) != 0) return fail(PF_ERR_ARG, "pf_camera_fields: up_offset must be even (8-byte stores)");
      CamImage& o = b.im[i];
      o.H = c.height; o.W = c.width;
      o.f = c.focal_rel * c.height;
      o.cx = (c.cx_rel + 0.5) * c.width; o.cy = (c.cy_rel + 0.5) * c.height;
      o.sr = sin(c.roll); o.cr = cos(c.roll); o.se = sin(c.elevation); o.ce = cos(c.elevation);
      o.sgn = c.elevation > 0 ? 1.0 : (c.elevation < 0 ? -1.0 : 0.0);
      o.vp = vp && std::isfinite(vp[2 * (i0 + i)]);
      if (o.vp) { o.vpx = vp[2 * (i0 + i)]; o.vpy = vp[2 * (i0 + i) + 1]; o.sgn = 1.0; }
      o.up_off = c.up_offset; o.lat_off = c.lat_offset;
      const long long qd = (long long)c.height * ((c.width + 3) / 4);
      if (qd > max_q) max_q = qd;
    }
    const dim3 grid((unsigned)cdivl(max_q, 256), (unsigned)m);
    LAUNCHED((camera_fields_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(b, up, lat), cudaGetLastError()));
  }
  return PF_OK;
}

int pf_op_resize_u8(const uint8_t* img, int H, int W, int new_h, int new_w, uint8_t* out, void* stream) {
  if (!img || !out || H < 1 || W < 1 || new_h < 1 || new_w < 1) return fail(PF_ERR_ARG, "pf_op_resize_u8: bad argument");
  if (H == new_h && W == new_w) {   // Pillow returns a copy when the size does not change
    CU(cudaMemcpyAsync(out, img, (size_t)H * W * 3, cudaMemcpyDeviceToDevice, (cudaStream_t)stream));
    return PF_OK;
  }
  const ResampleTable tx = make_resample_table(W, new_w), ty = make_resample_table(H, new_h);
  return op_run("pf_op_resize_u8", 1, stream, [&](Fwd& F) -> int {
    int *bx, *cx, *by, *cy;
    TRY(op_upload(F, tx.bounds.data(), tx.bounds.size(), &bx));
    TRY(op_upload(F, tx.coeffs.data(), tx.coeffs.size(), &cx));
    TRY(op_upload(F, ty.bounds.data(), ty.bounds.size(), &by));
    TRY(op_upload(F, ty.coeffs.data(), ty.coeffs.size(), &cy));
    unsigned char* tmp = (unsigned char*)F.ar.alloc((long long)H * new_w * 3);
    if (F.dry) return PF_OK;
    // Pillow runs the horizontal pass first (over the rows the vertical pass needs: all of them here), each pass rounded to uint8
    LAUNCHED((resize_u8_h_kernel<<<(unsigned)cdivl((long long)H * new_w, 256), 256, 0, F.st>>>(img, H, W, new_w, bx, cx, tx.ksize, tmp), cudaGetLastError()));
    LAUNCHED((resize_u8_v_kernel<<<(unsigned)cdivl((long long)new_h * new_w, 256), 256, 0, F.st>>>(tmp, H, new_w, new_h, by, cy, ty.ksize, out), cudaGetLastError()));
    return PF_OK;
  });
}
int pf_op_resize_f32(const float* img, int H, int W, int C, int new_h, int new_w, float* out, void* stream) {
  if (!img || !out || H < 1 || W < 1 || C < 1 || new_h < 1 || new_w < 1) return fail(PF_ERR_ARG, "pf_op_resize_f32: bad argument");
  LAUNCHED((resize_f32_kernel<<<(unsigned)cdivl((long long)new_h * new_w * C, 256), 256, 0, (cudaStream_t)stream>>>(img, H, W, C, new_h, new_w, out), cudaGetLastError()));
  return PF_OK;
}
int pf_op_argmax_decode(const float* logits, float* field, int B, int HW, int NC, int is_gravity, void* stream) {
  if (!logits || !field || B < 1 || HW < 1 || NC < 1) return fail(PF_ERR_ARG, "pf_op_argmax_decode: bad argument");
  LAUNCHED((argmax_decode_kernel<<<(unsigned)cdivl((long long)B * HW, 256), 256, 0, (cudaStream_t)stream>>>(logits, field, B, HW, NC, is_gravity), cudaGetLastError()));
  return PF_OK;
}
int pf_op_pred_argmax_decode(const float* feat, int ld, int coff, const float* w, const float* bias, float* field, int B, int HW, int NC, int is_gravity,
                             void* stream) {
  if (!feat || !w || !bias || !field || B < 1 || HW < 1 || NC < 1 || NC > 256 || (ld & 3) || (coff & 3)) return fail(PF_ERR_ARG, "pf_op_pred_argmax_decode: bad argument");
  LAUNCHED((pred_argmax_decode_kernel<<<ew_grid((long long)B * HW * 4), 256, NC * 37 * 4, (cudaStream_t)stream>>>(feat, ld, coff, w, bias, field, B, HW, NC, is_gravity),
            cudaGetLastError()));
  return PF_OK;
}
int pf_op_postprocess(const float* vec, const float* lat, int n, const int32_t* height, const int32_t* width, float* gravity_original,
                      const int64_t* gravity_original_offset, float* latitude_original, const int64_t* latitude_original_offset, int lat_is_sin,
                      void* stream) {
  return pf_op_postprocess_sized(vec, lat, n, kNet, kNet, height, width, gravity_original, gravity_original_offset, latitude_original, latitude_original_offset,
                                 lat_is_sin, stream);
}
int pf_op_postprocess_sized(const float* vec, const float* lat, int n, int net_h, int net_w, const int32_t* height, const int32_t* width, float* gravity_original,
                            const int64_t* gravity_original_offset, float* latitude_original, const int64_t* latitude_original_offset, int lat_is_sin,
                            void* stream) {
  if (!vec || !lat || n < 1 || !height || !width || !gravity_original || !gravity_original_offset || !latitude_original || !latitude_original_offset)
    return fail(PF_ERR_ARG, "pf_op_postprocess: bad argument");
  if (!net_size_ok(net_h, net_w)) return fail(PF_ERR_ARG, "pf_op_postprocess: unsupported working size %dx%d", net_h, net_w);
  return op_run("pf_op_postprocess", n, stream, [&](Fwd& F) -> int {
    PostImage* d_post = (PostImage*)F.ar.alloc((long long)n * sizeof(PostImage));
    if (F.dry) return PF_OK;
    return launch_postprocess(vec, lat, n, net_h, net_w, height, width, gravity_original_offset, latitude_original_offset, gravity_original,
                              latitude_original, lat_is_sin, d_post, F.st);
  });
}

int pf_op_fill_stream(float* dst, int64_t numel, float value, void* stream) {
  if (!dst || numel < 4 || (numel & 3) || ((uintptr_t)dst & 15)) return fail(PF_ERR_ARG, "pf_op_fill_stream: bad argument");
  LAUNCHED((fill_stream_kernel<<<132 * 16, 256, 0, (cudaStream_t)stream>>>(reinterpret_cast<float4*>(dst), numel / 4, value), cudaGetLastError()));
  return PF_OK;
}
static int op_attention_tc(const float* q, const float* kv, float* out, int B, int N, int C, int heads, void* stream, int np, int nkv = kAmKeys) {
  if (!q || !kv || !out || C != heads * kAmD) return fail(PF_ERR_ARG, "pf_op_attention_tc: head_dim must be 64");
  if (B < 1 || N < 1 || nkv < 1 || nkv > kAmMaxKeys) return fail(PF_ERR_ARG, "pf_op_attention_tc: B %d, N %d, %d keys (1..%d)", B, N, nkv, kAmMaxKeys);
  return op_run("pf_op_attention_tc", B, stream, [&](Fwd& F) -> int {
    const long long nq = (long long)B * N * C, nkve = (long long)B * nkv * 2 * C;
    SplitT qs = F.salloc((long long)B * N, C), kvs = F.salloc((long long)B * nkv, 2 * C), as = F.salloc((long long)B * N, C);
    if (F.dry) return PF_OK;
    LAUNCHED((split_kernel<<<(unsigned)cdivl(nq, 256), 256, 0, F.st>>>(q, qs.hi, qs.lo, nq, 0), cudaGetLastError()));
    LAUNCHED((split_kernel<<<(unsigned)cdivl(nkve, 256), 256, 0, F.st>>>(kv, kvs.hi, kvs.lo, nkve, 0), cudaGetLastError()));
    LAUNCHED(attention_mma_launch(nullptr, B, N, C, heads, F.st, as, qs, kvs, np, nkv));
    LAUNCHED((merge_split_kernel<<<(unsigned)cdivl(nq, 256), 256, 0, F.st>>>(as.hi, as.lo, out, nq), cudaGetLastError()));
    return PF_OK;
  });
}
int pf_op_attention_tc(const float* q, const float* kv, float* out, int B, int N, int C, int heads, void* stream) {
  return op_attention_tc(q, kv, out, B, N, C, heads, stream, 3);
}
int pf_op_attention_tc_bf16(const float* q, const float* kv, float* out, int B, int N, int C, int heads, void* stream) {
  return op_attention_tc(q, kv, out, B, N, C, heads, stream, 1);
}
int pf_op_attention_tc_keys(const float* q, const float* kv, float* out, int B, int N, int NKV, int C, int heads, int bf16, void* stream) {
  return op_attention_tc(q, kv, out, B, N, C, heads, stream, bf16 ? 1 : 3, NKV);
}
// The forward graph's CUDA-core kernels, each through the Fwd helper the graph launches it with (same grid, block and arguments).
int pf_op_layernorm(const float* x, float* y, int64_t rows, int C, const float* w, const float* b, float eps, void* stream) {
  return pf_op_layernorm_ex(x, y, nullptr, nullptr, nullptr, nullptr, rows, C, w, b, eps, 0, 0, 0, stream);
}
int pf_op_layernorm_ex(const float* x, float* y, void* hi, void* lo, void* phi, void* plo, int64_t rows, int C, const float* w, const float* b,
                       float eps, int RH, int RW, int sr, void* stream) {
  if (!x || !w || !b || !hi != !lo || !phi != !plo || (!y && !hi && !phi)) return fail(PF_ERR_ARG, "pf_op_layernorm_ex: null input, half a split pair or no output");
  if (!al16(x) || !al16(y) || !al16(w) || !al16(b) || !al16(hi) || !al16(lo) || !al16(phi) || !al16(plo)) return fail(PF_ERR_ARG, "pf_op_layernorm_ex: unaligned pointer");
  if (!(eps > 0.f)) return fail(PF_ERR_ARG, "pf_op_layernorm_ex: eps %g", eps);
  const SplitT s{(__nv_bfloat16*)hi, (__nv_bfloat16*)lo, C}, p{(__nv_bfloat16*)phi, (__nv_bfloat16*)plo, C};
  const LnW lw{w, b};
  return op_run("pf_op_layernorm_ex", 1, stream, [&](Fwd& F) {
    if (phi) return F.ln_split_patch(x, s, p, rows, C, lw, eps, RH, RW, sr, y);
    if (hi) return F.ln_split(x, s, rows, C, lw, eps, y);
    return F.ln(x, y, rows, C, lw, eps);
  });
}
int pf_op_dwconv3x3_gelu(const float* x, float* y, int B, int H, int W, int C, const float* w, const float* bias, void* stream) {
  return pf_op_dwconv3x3_gelu_ex(x, B, H, W, C, w, bias, y, nullptr, nullptr, stream);
}
int pf_op_dwconv3x3_gelu_ex(const float* x, int B, int H, int W, int C, const float* w, const float* bias, float* y, void* hi, void* lo, void* stream) {
  if (!x || !w || !bias || !hi != !lo || (!y && !hi)) return fail(PF_ERR_ARG, "pf_op_dwconv3x3_gelu_ex: null input, half a split pair or no output");
  if (!al16(x) || !al16(w) || !al16(bias) || !al16(y) || !al16(hi) || !al16(lo)) return fail(PF_ERR_ARG, "pf_op_dwconv3x3_gelu_ex: unaligned pointer");
  const SplitT s{(__nv_bfloat16*)hi, (__nv_bfloat16*)lo, C};
  return op_run("pf_op_dwconv3x3_gelu_ex", B, stream, [&](Fwd& F) { return F.dw3_gelu(x, y, s, H, W, C, w, bias); });
}
int pf_op_dwconv7x7(const float* x, float* y, int B, int H, int W, int C, const float* w, const float* bias, void* stream) {
  if (!x || !y || !w || !bias) return fail(PF_ERR_ARG, "pf_op_dwconv7x7: null argument");
  if (!al16(x) || !al16(y) || !al16(w) || !al16(bias)) return fail(PF_ERR_ARG, "pf_op_dwconv7x7: unaligned pointer");
  return op_run("pf_op_dwconv7x7", B, stream, [&](Fwd& F) { return pn_dw_launch(F, x, y, H, W, C, w, bias); });
}
int pf_op_upsample2x(const float* x, float* y, int B, int H, int W, int C, void* stream) {
  return pf_op_upsample2x_ex(x, C, 0, y, C, 0, nullptr, nullptr, B, H, W, C, stream);
}
int pf_op_upsample2x_ex(const float* x, int ldi, int icoff, float* y, int ldo, int ocoff, void* hi, void* lo, int B, int H, int W, int C, void* stream) {
  if (!x || !hi != !lo || (!y && !hi)) return fail(PF_ERR_ARG, "pf_op_upsample2x_ex: null input, half a split pair or no output");
  if (!al16(x) || !al16(y) || !al16(hi) || !al16(lo)) return fail(PF_ERR_ARG, "pf_op_upsample2x_ex: unaligned pointer");
  const SplitT s{(__nv_bfloat16*)hi, (__nv_bfloat16*)lo, ldo};
  return op_run("pf_op_upsample2x_ex", B, stream, [&](Fwd& F) { return F.up2x(x, ldi, icoff, y, ldo, ocoff, s, H, W, C); });
}
int pf_op_stem_gather(const float* x0, int B, int IH, int IW, int stride, void* hi, void* lo, void* stream) {
  if (!x0 || !hi || !lo) return fail(PF_ERR_ARG, "pf_op_stem_gather: null argument");
  if (!al16(hi) || !al16(lo)) return fail(PF_ERR_ARG, "pf_op_stem_gather: unaligned pointer");
  const SplitT col{(__nv_bfloat16*)hi, (__nv_bfloat16*)lo, 160};
  return op_run("pf_op_stem_gather", B, stream, [&](Fwd& F) { return F.stem_gather(x0, col, IH, IW, stride); });
}
int pf_op_pn_stem(const float* pin, int B, int SH, int SW, const float* w, const float* b, float* out, void* stream) {
  if (!pin || !w || !b || !out) return fail(PF_ERR_ARG, "pf_op_pn_stem: null argument");
  return op_run("pf_op_pn_stem", B, stream, [&](Fwd& F) { return F.pn_stem(pin, SH, SW, w, b, out); });
}
int pf_op_pack_fields(const float* grav, const float* lat, int B, int IH, int IW, int OH, int OW, float* out, void* stream) {
  if (!grav || !lat || !out) return fail(PF_ERR_ARG, "pf_op_pack_fields: null argument");
  if (!al16(out)) return fail(PF_ERR_ARG, "pf_op_pack_fields: unaligned output");
  return op_run("pf_op_pack_fields", B, stream, [&](Fwd& F) { return F.pack_fields(grav, lat, IH, IW, OH, OW, out); });
}
int pf_op_param_tail(const float* feat, int n, int HW, const float* nw, const float* nb, const float* hw, const float* hb, int kind, float* params, float* raw,
                     void* stream) {
  if (!feat || !nw || !nb || !hw || !hb || !params) return fail(PF_ERR_ARG, "pf_op_param_tail: null argument");
  const LnW norm{nw, nb};
  return op_run("pf_op_param_tail", n, stream, [&](Fwd& F) { return F.param_tail(feat, HW, norm, hw, hb, kind, params, raw); });
}
int pf_op_pred_tail(const float* feat, int ld, int coff, const float* w, const float* b, float* out, int B, int HW, int NC, int mode, void* stream) {
  if (!feat || !w || !b || !out) return fail(PF_ERR_ARG, "pf_op_pred_tail: null argument");
  if (!al16(feat)) return fail(PF_ERR_ARG, "pf_op_pred_tail: unaligned input");
  return op_run("pf_op_pred_tail", B, stream, [&](Fwd& F) { return F.pred_tail(feat, ld, coff, w, b, out, HW, NC, mode); });
}
int pf_op_preprocess(const uint8_t* img, int H, int W, const float* mean3, const float* std3, float* y, void* stream) {
  return pf_op_preprocess_sized(img, H, W, kNet, kNet, mean3, std3, y, stream);
}
int pf_op_preprocess_sized(const uint8_t* img, int H, int W, int net_h, int net_w, const float* mean3, const float* std3, float* y, void* stream) {
  if (!img || !mean3 || !std3 || !y || H < 1 || W < 1) return fail(PF_ERR_ARG, "pf_op_preprocess: bad argument");
  if (!net_size_ok(net_h, net_w)) return fail(PF_ERR_ARG, "pf_op_preprocess: unsupported working size %dx%d", net_h, net_w);
  // standalone tables (not cached): test entry point only
  const ResampleTable tx = make_resample_table(W, net_w), ty = make_resample_table(H, net_h);
  const int max_rows = pre_max_smem_rows(net_w);
  if (ty.ksize + 1 > max_rows) return fail(PF_ERR_ARG, "image too tall");
  const int rows = std::min(pre_rows_needed(H, net_h), max_rows);
  return op_run("pf_op_preprocess", 1, stream, [&](Fwd& F) -> int {
    int *bx, *cx, *by, *cy;
    TRY(op_upload(F, tx.bounds.data(), tx.bounds.size(), &bx));
    TRY(op_upload(F, tx.coeffs.data(), tx.coeffs.size(), &cx));
    TRY(op_upload(F, ty.bounds.data(), ty.bounds.size(), &by));
    TRY(op_upload(F, ty.coeffs.data(), ty.coeffs.size(), &cy));
    const PreImage pi{0, H, W, tx.ksize, ty.ksize, bx, cx, by, cy};
    PreImage* d;
    TRY(op_upload(F, &pi, 1, &d));
    if (F.dry) return PF_OK;
    LAUNCHED((preprocess_kernel<<<dim3(net_h / kPreRows, 1), net_w, rows * net_w * 3, F.st>>>(img, d, y, mean3[0], mean3[1], mean3[2], std3[0], std3[1], std3[2],
                                                                                         rows, net_h, net_w),
              cudaGetLastError()));
    return PF_OK;
  });
}

}  // extern "C"
