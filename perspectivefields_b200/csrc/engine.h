// The engine and its launch helper, shared by the translation units that launch through it (pf_b200.cu: the forward graph,
// paramnet_train.cu: ParamNet training).  Internal: not part of the C ABI.
#pragma once
#include <cuda.h>

#include <cstdarg>
#include <cstdio>
#include <map>
#include <string>
#include <unordered_map>
#include <vector>

#include "common.cuh"
#include "host.h"
#include "tma_host.cuh"

using namespace pf;

// ----------------------------------------------------------------------------------------------- model constants
static const int kMitDims[4] = {64, 128, 320, 512};
static const int kMitHeads[4] = {1, 2, 5, 8};
static const int kMitDepths[4] = {3, 4, 18, 3};
static const int kMitSr[4] = {8, 4, 2, 1};
static const int kCnxDims[4] = {96, 192, 384, 768};
static const int kCnxDepths[4] = {3, 3, 9, 3};

struct WeightRef { const void* p; long long numel; int dtype; };
struct GemmW { const __nv_bfloat16* hi = nullptr; const __nv_bfloat16* lo = nullptr; const float* b = nullptr; };
struct LnW { const float* w = nullptr; const float* b = nullptr; };

struct MitBlockW { LnW ln1, srln, ln2; GemmW q, sr, kv, proj, fc1, fc2; const float* dw_w; const float* dw_b; };
struct CnxBlockW { const float* dw_w; const float* dw_b; LnW ln; GemmW pw1, pw2; const float* gamma; };

struct Arena {
  char* base = nullptr;
  long long cap = 0, off = 0, peak = 0;
  bool dry = false, keep = false;  // keep: debug mode, never recycle
  void* alloc(long long bytes) {
    off = (off + 255) & ~255LL;
    void* p = dry ? nullptr : base + off;
    off += bytes;
    if (off > peak) peak = off;
    return p;
  }
  float* f(long long n) { return (float*)alloc(n * 4); }
  long long mark() const { return off; }
  void release(long long m) { if (!keep) off = m; }
};

struct pf_engine {
  int device = 0;
  pf_model_desc desc{};
  int net_h = kNet, net_w = kNet;     // working size (DATALOADER.RESIZE = [net_h, net_w]): multiples of 32 in [64, 640] (pf_create_sized)
  bool finalized = false;
  std::unordered_map<std::string, WeightRef> weights;
  // resolved weights
  LnW embed_ln[4], stage_norm[4];
  GemmW embed[4];  // [1..3] used
  GemmW embed1g, llencg;  // 7x7 stems as [64][160] GEMMs
  std::vector<MitBlockW> blocks[4];
  GemmW proc[4];   // composed linear_c{l} o linear_c{l}_proc, both heads side by side (N = 512), index lvl-1
  GemmW rcu[4][2][2];  // [fusion-1][unit-1][conv-1], grouped over the two heads
  GemmW conv0;
  GemmW conv1p;                       // conv_fuse_conv1 composed with the x2 upsample in front of it: 4 phases x 32 outputs per head
  const float *conv1f_w, *conv1f_b;   // plain fp32 conv_fuse_conv1 [head][tap][ci][o] / bias, for the border-ring kernel
  bool use_pdl = true;                // option "pdl": programmatic dependent launch of the graph's kernels (common.cuh)
  bool decode_only = false;           // option "decode_only": classification heads return decoded fields, logits are never written
  bool subbin = false;                // option "subbin": classification heads decode their argmax bin to a sub-bin position
  bool flip_tta = false;              // option "flip_tta": the network also runs on every image's mirror; the heads' outputs are merged
  const float *pred_g_w, *pred_g_b, *pred_l_w, *pred_l_b;
  const float *pn_stem_w, *pn_stem_b;
  LnW pn_stem_ln, pn_ds_ln[4], pn_norm;
  GemmW pn_ds[4];
  std::vector<CnxBlockW> pn_blocks[4];
  const float *pn_head_w, *pn_head_b;
  // ParamNet training only (pf_param_backward, resolved there): transposed split copies of the GEMM weights for the data
  // gradients, the depthwise kernels rotated by 180 degrees and a zero bias for the depthwise data gradient
  struct PnTrainW { GemmW ds_t[4]; std::vector<GemmW> pw1_t[4], pw2_t[4]; std::vector<const float*> dw_rot[4]; const float* zero = nullptr; } pn_train;
  // Pillow resample tables, cached per (input size, output size) in one device slab owned by the engine (bump allocation; built on the host
  // into a pinned mirror of the slab and copied with cudaMemcpyAsync on the caller's stream: no allocation and no
  // synchronising copy inside pf_forward)
  struct DevTable { int ksize; int* bounds; int* coeffs; };
  std::map<std::pair<int, int>, DevTable> tables;
  char* table_dev = nullptr;
  char* table_host = nullptr;       // pinned
  long long table_off = 0;
  long long table_resets = 0;       // times the slab was full and started over (pf_resize_table_stats)
  KernelProf kp;                    // pf_profile_kernels_*
  // per-launch profiling of the GEMM engine (bench.py roofline leg): CUDA events on the launch stream
  // tensor maps are pure functions of (pointer, shape, box): cached across calls (the arena hands out the same addresses for the
  // same batch size), which takes cuTensorMapEncodeTiled (~5 us each, ~1800 per forward) off the launch path
  struct MapKey {
    const void* base; long long d0, d1, d2; int kind, box, kb;
    bool operator==(const MapKey& o) const { return base == o.base && d0 == o.d0 && d1 == o.d1 && d2 == o.d2 && kind == o.kind && box == o.box && kb == o.kb; }
  };
  struct MapKeyHash {
    size_t operator()(const MapKey& k) const {
      size_t h = std::hash<const void*>()(k.base);
      for (long long v : {k.d0, k.d1, k.d2, (long long)k.kind, (long long)k.box, (long long)k.kb}) h = h * 1000003u ^ std::hash<long long>()(v);
      return h;
    }
  };
  std::unordered_map<MapKey, CUtensorMap, MapKeyHash> map_cache;
  bool bf16 = false;          // option "bf16": every tensor-core product is one bf16 MMA (hi * hi) instead of three; read per launch
  int sm_count = 132;
  bool profile = false;
  struct ProfRec { cudaEvent_t a, b; double flops; int cfg; int M, N, K, KH, stride, groups, Cin; };
  std::vector<ProfRec> prof;
  std::vector<cudaEvent_t> ev_pool;   // events are created once and recycled: no create/destroy inside a timed region
  // debug taps
  bool debug = false;
  std::vector<std::pair<std::string, std::pair<const float*, long long>>> taps;
};

// ----------------------------------------------------------------------------------------------- weight lookup
int get_w(pf_engine* e, const std::string& name, int dtype, long long numel, const void** out);
int get_f(pf_engine* e, const std::string& n, long long numel, const float** out);

// ----------------------------------------------------------------------------------------------- op helpers
struct Fwd {
  pf_engine* e;
  Arena ar;
  cudaStream_t st;
  bool dry;
  int n;

  // debug taps: snapshot the tensor into a private buffer (many intermediates are updated in place later)
  int tap(const char* name, const float* p, long long numel) {
    if (!e->debug) return PF_OK;
    float* cp = ar.f(numel);
    if (dry) return PF_OK;
    snprintf(g_crumb, sizeof g_crumb, "%s", name);
    if (sync_debug()) fprintf(stderr, "[pf tap] %s cp=%p (+%lld of cap %lld) p=%p numel=%lld\n", name, (void*)cp, (long long)((char*)cp - ar.base), ar.cap, (const void*)p, numel);
    CU(cudaMemcpyAsync(cp, p, numel * 4, cudaMemcpyDeviceToDevice, st));
    if (sync_debug()) CU(cudaDeviceSynchronize());
    e->taps.push_back({name, {cp, numel}});
    return PF_OK;
  }
  int tapf(const float* p, long long numel, const char* fmt, ...) {
    if (!e->debug) return PF_OK;
    char buf[96];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof buf, fmt, ap);
    va_end(ap);
    return tap(buf, p, numel);
  }

  // ------------------------------------------------------------------------------------------ TMA engine helpers
  SplitT salloc(long long pixels, int ld) {
    SplitT t;
    t.hi = (__nv_bfloat16*)ar.alloc(pixels * ld * 2);
    t.lo = (__nv_bfloat16*)ar.alloc(pixels * ld * 2);
    t.ld = ld;
    return t;
  }
  int tap_split(const char* name, const SplitT& t, long long numel);
  // (two names so that the per-kernel profile separates the GEMM-mode and halo-mode launches)
  static cudaError_t gemm_tma_gemm_mode(const TmaMaps& maps, const TmaGemmParams& p, int bn, int kb, bool pp, int np, int sms, cudaStream_t st, const PredTail* pred) {
    return gemm_tma_launch(MODE_GEMM, maps, p, bn, kb, pp, np, sms, st, pred);
  }
  static cudaError_t gemm_tma_halo_mode(const TmaMaps& maps, const TmaGemmParams& p, int bn, int kb, bool pp, int np, int sms, cudaStream_t st, const PredTail* pred) {
    return gemm_tma_launch(MODE_HALO, maps, p, bn, kb, pp, np, sms, st, pred);
  }
  // bf16 products per output of the tensor-core launches: 3 (split precision) or 1 (option "bf16")
  int np() const { return e->bf16 ? 1 : 3; }
  int force_bn = 0, force_kb = 0;     // pf_op_tma: tile override (0 = the dispatcher's choice)
  int force_sched = 0;                // pf_op_tma: GEMM-mode schedule override (0 = the dispatcher's choice, 1 cooperative, 2 ping-pong)
  int picked_bn = 0, picked_kb = 0, picked_sched = 0;   // (bn, kb, schedule) of the last TMA launch
  // the one place a launch's (bn, kb) and schedule are chosen: tgemm / thalo build the A and B maps with them and hand them to
  // launch_tma.  pp: the ping-pong schedule (GEMM mode only).
  int pick_tile(int mode, const TmaGemmParams& p, const PredTail* pred, int& bn, int& kb, bool& pp) {
    tma_pick_tile(mode, p.M, p.N, p.K, e->sm_count, bn, kb);
    if (force_bn) { bn = force_bn; kb = tma_pick_kb(bn, p.K, mode); }
    if (force_kb) kb = force_kb;
    pp = mode == MODE_GEMM && (force_sched ? force_sched == 2 : tma_pick_pingpong(p.M, p.N, p.K, bn, e->sm_count));
    if (const char* msg = gemm_tma_check(mode, p, bn, kb, pred != nullptr, pp, np())) return fail(PF_ERR_ARG, "TMA engine, %s (bn %d, kb %d): %s", mode == MODE_GEMM ? "GEMM mode" : "halo mode", bn, kb, msg);
    picked_bn = bn; picked_kb = kb; picked_sched = mode == MODE_GEMM ? (pp ? 2 : 1) : 0;
    return PF_OK;
  }
  int launch_tma(int mode, const TmaMaps& maps, const TmaGemmParams& p, int bn, int kb, bool pp, const PredTail* pred = nullptr) {
    if (e->profile) {
      pf_engine::ProfRec r{};
      for (cudaEvent_t* ev : {&r.a, &r.b}) {
        if (e->ev_pool.empty()) { CU(cudaEventCreate(ev)); }
        else { *ev = e->ev_pool.back(); e->ev_pool.pop_back(); }
      }
      const double Mrows = mode == MODE_GEMM ? (double)p.M : (double)p.B * p.H * p.W;
      r.flops = 2.0 * Mrows * (double)p.N * (double)p.K * (double)p.groups;
      r.cfg = mode == MODE_GEMM ? 5 : 6;
      r.M = (int)Mrows; r.N = p.N; r.K = p.K; r.KH = mode == MODE_GEMM ? 1 : 3; r.stride = 1; r.groups = p.groups; r.Cin = p.Cin;
      CU(cudaEventRecord(r.a, st));
      if (mode == MODE_GEMM) LAUNCHED(gemm_tma_gemm_mode(maps, p, bn, kb, pp, np(), e->sm_count, st, pred));
      else LAUNCHED(gemm_tma_halo_mode(maps, p, bn, kb, pp, np(), e->sm_count, st, pred));
      CU(cudaEventRecord(r.b, st));
      e->prof.push_back(r);
      return PF_OK;
    }
    if (mode == MODE_GEMM) LAUNCHED(gemm_tma_gemm_mode(maps, p, bn, kb, pp, np(), e->sm_count, st, pred));
    else LAUNCHED(gemm_tma_halo_mode(maps, p, bn, kb, pp, np(), e->sm_count, st, pred));
    return PF_OK;
  }
  struct Epi {   // epilogue options of one TMA GEMM / conv
    float* C = nullptr; int ldc = 0, c_coff = 0, c_gcoff = 0;
    SplitT S; int s_coff = 0, s_gcoff = 0, split_relu = 0;
    int act = 0; const float* gamma = nullptr;
    const float* res = nullptr; int ldr = 0, r_coff = 0, r_gcoff = 0, res_relu = 0;
    const float* res2 = nullptr; int ldr2 = 0, r2_coff = 0, r2_gcoff = 0;
    int bias_mode = 1;
    int phase4 = 0;   // halo mode, N = 128: columns are 4 output phases x 32 channels of a 2H x 2W output (TmaGemmParams::phase4)
  };
  static void fill_epi(TmaGemmParams& p, const GemmW& w, const Epi& o, int bias_gstride) {
    p.bias = w.b; p.bias_mode = w.b ? o.bias_mode : 0; p.bias_gstride = bias_gstride;
    p.act = o.act; p.gamma = o.gamma;
    p.res = o.res; p.ldr = o.ldr; p.r_coff = o.r_coff; p.r_gcoff = o.r_gcoff; p.res_relu = o.res_relu;
    p.res2 = o.res2; p.ldr2 = o.ldr2; p.r2_coff = o.r2_coff; p.r2_gcoff = o.r2_gcoff;
    p.C = o.C; p.ldc = o.ldc; p.c_coff = o.c_coff; p.c_gcoff = o.c_gcoff;
    p.Shi = o.S.hi; p.Slo = o.S.lo; p.lds = o.S.ld; p.s_coff = o.s_coff; p.s_gcoff = o.s_gcoff; p.split_relu = o.split_relu;
    p.phase4 = o.phase4;
  }
  // cached tensor-map constructors
  template <class F>
  const char* cached_map(CUtensorMap* out, const pf_engine::MapKey& key, F&& make) {
    auto it = e->map_cache.find(key);
    if (it != e->map_cache.end()) { *out = it->second; return nullptr; }
    const char* msg = make(out);
    if (!msg) {
      if (e->map_cache.size() > 20000) e->map_cache.clear();
      e->map_cache.emplace(key, *out);
    }
    return msg;
  }
  const char* map2d(CUtensorMap* m, const void* base, long long cols, long long rows, long long ld, int box_rows, int kb) {
    return cached_map(m, pf_engine::MapKey{base, cols, rows, ld, 0, box_rows, kb}, [&](CUtensorMap* o) { return tma_map_2d(o, base, cols, rows, ld, box_rows, kb); });
  }
  const char* map_halo(CUtensorMap* m, const void* base, int B, int H, int W, int ld) {
    return cached_map(m, pf_engine::MapKey{base, ((long long)B << 32) | (unsigned)H, W, ld, 3, 0, 0}, [&](CUtensorMap* o) { return tma_map_halo(o, base, B, H, W, ld); });
  }
  // C[M, N] = A[M, K] W^T : A = split planes with row pitch A.ld, first channel a_c0
  int tgemm(const SplitT& A, long long M, int K, int a_c0, const GemmW& w, int N, const Epi& o) {
    if (dry) return PF_OK;
    if (K % 32 || N % 32 || A.ld % 8) return fail(PF_ERR_ARG, "tgemm: K/N must be multiples of 32");
    if (o.res2 || o.bias_mode == 2) return fail(PF_ERR_ARG, "tgemm: second residual / border-class bias are halo-mode features");
    TmaGemmParams p{};
    p.M = (int)M; p.Cin = K; p.N = N; p.K = K; p.a_c0 = a_c0; p.groups = 1;
    fill_epi(p, w, o, 0);
    TmaMaps maps{};
    int bn, kb;
    bool pp;
    TRY(pick_tile(MODE_GEMM, p, nullptr, bn, kb, pp));
    const char* msg = nullptr;
    const int a_rows = pp ? 64 : 128;     // A box = one tile's rows
    if (!msg) msg = map2d(&maps.a_hi, A.hi, A.ld, M, A.ld, a_rows, kb);
    if (!msg) msg = map2d(&maps.a_lo, A.lo, A.ld, M, A.ld, a_rows, kb);
    if (!msg) msg = map2d(&maps.b_hi, w.hi, K, N, K, bn, kb);
    if (!msg) msg = map2d(&maps.b_lo, w.lo, K, N, K, bn, kb);
    if (msg) return fail(PF_ERR_CUDA, "%s", msg);
    maps.a2_hi = maps.a_hi; maps.a2_lo = maps.a_lo;
    return launch_tma(MODE_GEMM, maps, p, bn, kb, pp);
  }
  // 3x3 / stride 1 / pad 1 convolution on split NHWC planes (optionally a second source for channels >= c_split)
  int thalo(const SplitT& A, int a_c0, int a_gc, const SplitT* A2, int c_split, int a2_c0, int B, int H, int W, int Cin, const GemmW& w, int N,
            int groups, int bias_gstride, const Epi& o, const PredTail* pred = nullptr) {
    if (dry) return PF_OK;
    if (Cin % 64 || N % 32 || (A2 && c_split % 64)) return fail(PF_ERR_ARG, "thalo: Cin must be a multiple of 64, N of 32");
    // the nine border classes (weights.py:_compose_proc) assume a pixel is never both the first and the last of a row / column
    if (w.b && o.bias_mode == 2 && (H < 2 || W < 2)) return fail(PF_ERR_ARG, "thalo: border-class bias needs H, W >= 2 (got %dx%d)", H, W);
    TmaGemmParams p{};
    p.B = B; p.H = H; p.W = W; p.Cin = Cin; p.N = N; p.K = 9 * Cin; p.a_c0 = a_c0; p.a_gc = a_gc; p.groups = groups;
    p.c_split = A2 ? c_split : 0; p.a2_c0 = a2_c0;
    fill_epi(p, w, o, bias_gstride);
    TmaMaps maps{};
    int bn, kb;
    bool pp;
    TRY(pick_tile(MODE_HALO, p, pred, bn, kb, pp));
    const char* msg = nullptr;
    if (!msg) msg = map_halo(&maps.a_hi, A.hi, B, H, W, A.ld);
    if (!msg) msg = map_halo(&maps.a_lo, A.lo, B, H, W, A.ld);
    if (A2) {
      if (!msg) msg = map_halo(&maps.a2_hi, A2->hi, B, H, W, A2->ld);
      if (!msg) msg = map_halo(&maps.a2_lo, A2->lo, B, H, W, A2->ld);
    } else { maps.a2_hi = maps.a_hi; maps.a2_lo = maps.a_lo; }
    if (!msg) msg = map2d(&maps.b_hi, w.hi, p.K, (long long)groups * N, p.K, bn, kb);
    if (!msg) msg = map2d(&maps.b_lo, w.lo, p.K, (long long)groups * N, p.K, bn, kb);
    if (msg) return fail(PF_ERR_CUDA, "%s", msg);
    return launch_tma(MODE_HALO, maps, p, bn, kb, pp, pred);
  }
  // strided / patchifying convolution = patch gather on split planes + TMA GEMM
  int tconv_gather(const SplitT& A, int B, int H, int W, int Cin, int KH, int stride, int pad, const GemmW& w, int N, const Epi& o);
  int ln_split(const float* x, const SplitT& y, long long rows, int C, const LnW& w, float eps, float* yf = nullptr);
  // LayerNorm whose output is (also) written in patch order for a k = s = sr convolution on the RH x RW map (y may be empty)
  int ln_split_patch(const float* x, const SplitT& y, const SplitT& patch, long long rows, int C, const LnW& w, float eps, int RH, int RW, int sr,
                     float* yf = nullptr);
  int ln(const float* x, float* y, long long rows, int C, const LnW& w, float eps);
  // The graph's other CUDA-core kernels (layers.cuh) on the n images of this pass.  Each helper is the only place its kernel is
  // launched from, and it rejects (PF_ERR_ARG, also in the sizing dry run) a shape whose indices would leave the 32-bit range the
  // kernel computes them in.
  // depthwise 3x3 + GELU on [n, H, W, C]: fp32 y and / or split planes s (the graph writes the planes only)
  int dw3_gelu(const float* x, float* y, const SplitT& s, int H, int W, int C, const float* w, const float* b);
  // x2 bilinear upsample of channels icoff .. icoff + C - 1 of [n, H, W, ldi] into channels ocoff .. of [n, 2H, 2W, ldo]: fp32 y
  // and / or split planes s (pitch ldo as well)
  int up2x(const float* x, int ldi, int icoff, float* y, int ldo, int ocoff, const SplitT& s, int H, int W, int C);
  // 7x7 / stride (2 or 4) / pad 3 patch matrix of x0 [n, IH, IW, 4] (channels 0-2) as split planes [n * OH * OW][160]
  int stem_gather(const float* x0, const SplitT& col, int IH, int IW, int stride);
  // ParamNet stem conv 4x4 / 4, 3 -> 96, on pin [n, SH, SW, 4] -> out [n, SH / 4, SW / 4, 96]
  int pn_stem(const float* pin, int SH, int SW, const float* w, const float* b, float* out);
  // ParamNet input: fields [n, 2 | 1, IH, IW] nearest-resampled to [n, OH, OW, 4]
  int pack_fields(const float* grav, const float* lat, int IH, int IW, int OH, int OW, float* out);
  // ParamNet tail on feat [n, HW, 768]: params [n][8], raw [n][5] (may be NULL); kind = PF_PARAM_CENTERED / _UNCENTERED
  int param_tail(const float* feat, int HW, const LnW& norm, const float* hw, const float* hb, int kind, float* params, float* raw);
  // 1x1 conv 32 -> NC on channels icoff .. icoff + 31 of [n * HW, ldi] -> NCHW out; mode 0 raw, 1 normalise (NC 2), 2 clamp
  int pred_tail(const float* in, int ldi, int icoff, const float* w, const float* b, float* out, int HW, int NC, int mode);
  // option "flip_tta": the n merged outputs of the 2n slots (image i in slot i, its mirror in slot n + i) at the working size H x W.
  // Regression heads: g2 [2n, 2, HW] / l2 [2n, 1, HW] head outputs -> g [n, 2, HW] / l [n, 1, HW]
  int flip_merge_reg(const float* g2, const float* l2, float* g, float* l, int H, int W);
  // classification head of NC classes from channels icoff .. icoff + 31 of conv1 features [2n * HW, ldi]: decode = false writes the
  // merged logits [n, NC, HW] to out; decode = true the decoded field (argmax, or sub-bin with refine) to out and, when conf is not
  // NULL, the confidence [n, HW]
  int flip_pred(const float* in, int ldi, int icoff, const float* w, const float* b, float* out, float* conf, int H, int W, int NC, int is_gravity,
                bool decode, bool refine);
};


// ----------------------------------------------------------------------------------------------- graph sections
// What ParamNet training keeps from its forward for the backward (pf_param_train_forward -> pf_param_backward): the packed input,
// the stem's pre-LayerNorm output and the residual stream before and after every block (xs[s][j] = input of block j of stage s,
// xs[s][depth] = the stage's output).  Everything else is recomputed.
struct PnSaved {
  float* pin = nullptr;
  float* stem_pre = nullptr;
  float* xs[4][10] = {};
};
int fwd_paramnet(Fwd& F, const float* grav, const float* lat, float* params, float* raw, const PnSaved* sv = nullptr);
// depthwise 7x7 convolution of the F.n images [rh, rw, C] (the forward's kernel; ParamNet training runs its data gradient with it);
// rejects the shapes Fwd::dw3_gelu rejects
int pn_dw_launch(Fwd& F, const float* x, float* y, int rh, int rw, int C, const float* w, const float* b);

// ----------------------------------------------------------------------------------------------- single-operator entry points
// A temporary engine for the current device: the device's kernels configured, its id and SM count filled in.
int op_engine(pf_engine& e, bool bf16 = false);

// Runs body(Fwd&) once on a temporary engine: a dry run sizes the scratch, which is then allocated, filled with 0xFF bytes (NaN:
// a read of memory no kernel wrote poisons the result) and handed to the real run on the caller's stream; the stream is
// synchronised before the scratch is freed.
template <class Body>
int op_run(const char* name, int n, void* stream, Body body, bool bf16 = false) {
  pf_engine tmp;
  TRY(op_engine(tmp, bf16));
  Fwd T{&tmp, Arena{}, nullptr, true, n};
  T.ar.dry = true;
  TRY(body(T));
  const long long bytes = T.ar.peak + 4096;
  cudaStream_t st = (cudaStream_t)stream;
  struct Scratch { char* p = nullptr; ~Scratch() { cudaFree(p); } } scratch;
  CU(cudaMalloc(&scratch.p, bytes));
  Fwd F{&tmp, Arena{}, st, false, n};
  F.ar.base = scratch.p; F.ar.cap = bytes;
  const cudaError_t me = cudaMemsetAsync(scratch.p, 0xFF, bytes, st);
  int r = me == cudaSuccess ? body(F) : fail(PF_ERR_CUDA, "%s: %s", name, cudaGetErrorString(me));
  const cudaError_t se = cudaStreamSynchronize(st);
  if (r == PF_OK && se != cudaSuccess) r = fail(PF_ERR_CUDA, "%s: %s", name, cudaGetErrorString(se));
  return r;
}
