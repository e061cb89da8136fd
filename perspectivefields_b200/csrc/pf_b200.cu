// libpf_b200.so -- C ABI (include/pf_b200.h) and forward orchestration of the H100-native (sm_90a) PerspectiveFields
// inference engine.  One engine per device; pf_forward enqueues the whole graph of
// perspective2d/perspectivefields.py:223-272 on the caller's stream.
#include "../../include/pf_b200.h"

#include <cuda_runtime.h>
#include <nvtx3/nvToolsExt.h>

#include <atomic>
#include <cctype>
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <mutex>
#include <string>
#include <functional>
#include <unordered_map>
#include <vector>

#include "common.cuh"
#include "tma_host.cuh"
#include "attention_mma.cuh"
#include "layers.cuh"
#include "prepost.cuh"
#include "pano.cuh"
#include "equi.cuh"
#include "draw.cuh"
#include "metrics.cuh"
#include "calib.cuh"
#include "rectify.cuh"
#include "comm.cuh"
#include "jpeg.cuh"
#include "paramnet_train.cuh"

using namespace pf;

// ----------------------------------------------------------------------------------------------- errors
static thread_local std::string g_err;
static std::atomic<long long> g_launches{0};

static int fail(int code, const char* fmt, ...) {
  char buf[1024];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof(buf), fmt, ap);
  va_end(ap);
  g_err = buf;
  return code;
}
#define CU(expr)                                                                                    \
  do {                                                                                              \
    cudaError_t e__ = (expr);                                                                       \
    if (e__ != cudaSuccess) return fail(PF_ERR_CUDA, "%s: %s (%s:%d)", #expr, cudaGetErrorString(e__), __FILE__, __LINE__); \
  } while (0)
// PF_SYNC_DEBUG=1 in the environment: synchronise after every launch so that a device fault is reported at the launch that
// caused it (debugging aid; never set in production)
static char g_crumb[96] = "";   // name of the last debug tap taken (breadcrumb for the error text)
static bool sync_debug() {
  static int v = -1;
  if (v < 0) v = getenv("PF_SYNC_DEBUG") ? 1 : 0;
  return v == 1;
}
// pf_profile_kernels_*: a CUDA-event pair around EVERY launch of the forward graph (in-pipeline time per kernel, bench.py's
// "per_kernel" table).  Off by default: the event records cost a few percent, so bench.py uses a separate pass for it.
// The state lives in the engine; the launch macro reaches it through a thread-local pointer that pf_forward sets for the
// duration of the call (operator entry points run with it unset).
struct KernelProf {
  bool on = false;
  cudaStream_t st = nullptr;
  std::vector<cudaEvent_t> pool;
  size_t used = 0;
  struct Rec { const char* expr; cudaEvent_t a, b; };
  std::vector<Rec> recs;
  cudaEvent_t next() { return used < pool.size() ? pool[used++] : nullptr; }
};
static thread_local KernelProf* tl_kp = nullptr;
#define LAUNCHED(expr)                                                                              \
  do {                                                                                              \
    KernelProf* kp__ = tl_kp;                                                                       \
    cudaEvent_t ka__ = (kp__ && kp__->on) ? kp__->next() : nullptr;                                 \
    if (ka__) cudaEventRecord(ka__, kp__->st);                                                      \
    cudaError_t e__ = (expr);                                                                       \
    g_launches.fetch_add(1, std::memory_order_relaxed);                                             \
    if (ka__) {                                                                                     \
      cudaEvent_t kb__ = kp__->next();                                                              \
      if (kb__) { cudaEventRecord(kb__, kp__->st); kp__->recs.push_back({#expr, ka__, kb__}); }     \
    }                                                                                               \
    if (e__ == cudaSuccess && sync_debug()) e__ = cudaDeviceSynchronize();                          \
    if (e__ != cudaSuccess) return fail(PF_ERR_CUDA, "%s: %s (%s:%d, after tap '%s')", #expr, cudaGetErrorString(e__), __FILE__, __LINE__, g_crumb); \
  } while (0)
// NVTX range per section of the forward graph (visible in Nsight Systems / ncu --nvtx; a few ns when no tool is attached)
struct NvtxRange {
  explicit NvtxRange(const char* name) { nvtxRangePushA(name); }
  ~NvtxRange() { nvtxRangePop(); }
};
#define TRY(expr)                \
  do {                           \
    int r__ = (expr);            \
    if (r__ != PF_OK) return r__; \
  } while (0)

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
static int get_w(pf_engine* e, const std::string& name, int dtype, long long numel, const void** out) {
  auto it = e->weights.find(name);
  if (it == e->weights.end()) return fail(PF_ERR_WEIGHT, "missing weight '%s'", name.c_str());
  if (it->second.dtype != dtype) return fail(PF_ERR_WEIGHT, "weight '%s': wrong dtype", name.c_str());
  if (it->second.numel != numel) return fail(PF_ERR_WEIGHT, "weight '%s': numel %lld, expected %lld", name.c_str(), it->second.numel, numel);
  *out = it->second.p;
  return PF_OK;
}
static int get_f(pf_engine* e, const std::string& n, long long numel, const float** out) { return get_w(e, n, PF_F32, numel, (const void**)out); }
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
  int tap_split(const char* name, const SplitT& t, long long numel) {
    if (!e->debug) return PF_OK;
    float* cp = ar.f(numel);
    if (dry) return PF_OK;
    snprintf(g_crumb, sizeof g_crumb, "%s", name);
    LAUNCHED((merge_split_kernel<<<(unsigned)cdivl(numel, 256), 256, 0, st>>>(t.hi, t.lo, cp, numel), cudaGetLastError()));
    e->taps.push_back({name, {cp, numel}});
    return PF_OK;
  }
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
  int tconv_gather(const SplitT& A, int B, int H, int W, int Cin, int KH, int stride, int pad, const GemmW& w, int N, const Epi& o) {
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
  int ln_split(const float* x, const SplitT& y, long long rows, int C, const LnW& w, float eps, float* yf = nullptr) {
    if (dry) return PF_OK;
    LAUNCHED(layernorm_launch(x, yf, rows, C, w.w, w.b, eps, st, y));
    return PF_OK;
  }
  // LayerNorm whose output is (also) written in patch order for a k = s = sr convolution on the RH x RW map (y may be empty)
  int ln_split_patch(const float* x, const SplitT& y, const SplitT& patch, long long rows, int C, const LnW& w, float eps, int RH, int RW, int sr) {
    if (dry) return PF_OK;
    LAUNCHED(layernorm_launch(x, nullptr, rows, C, w.w, w.b, eps, st, y, patch, RH, RW, sr));
    return PF_OK;
  }
  int ln(const float* x, float* y, long long rows, int C, const LnW& w, float eps) {
    if (dry) return PF_OK;
    LAUNCHED(layernorm_launch(x, y, rows, C, w.w, w.b, eps, st));
    return PF_OK;
  }
};

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
    if (!dry) {
      const unsigned grid = (unsigned)cdivl((long long)n * HW, 128);
      LAUNCHED((pred_tail_kernel<<<grid, 128, D.gravity_classes * 33 * 4, st>>>(conv1_out, 64, 0, e->pred_g_w, e->pred_g_b, rg, n, HW, D.gravity_classes, 0), cudaGetLastError()));
      LAUNCHED((pred_tail_kernel<<<grid, 128, D.latitude_classes * 33 * 4, st>>>(conv1_out, 64, 32, e->pred_l_w, e->pred_l_b, rl, n, HW, D.latitude_classes, 0), cudaGetLastError()));
    }
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
    if (!dry && !pred_done) {
      const unsigned grid = (unsigned)cdivl((long long)n * HW, 128);
      LAUNCHED((pred_tail_kernel<<<grid, 128, D.gravity_classes * 33 * 4, st>>>(conv1_out, 64, 0, e->pred_g_w, e->pred_g_b, bt->pred_gravity, n, HW,
                                                                             D.gravity_classes, D.gravity_classes == 2 ? 1 : 0), cudaGetLastError()));
      LAUNCHED((pred_tail_kernel<<<grid, 128, D.latitude_classes * 33 * 4, st>>>(conv1_out, 64, 32, e->pred_l_w, e->pred_l_b, bt->pred_latitude, n, HW,
                                                                              D.latitude_classes, D.latitude_classes == 1 ? 2 : 0), cudaGetLastError()));
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
// What ParamNet training keeps from its forward for the backward (pf_param_train_forward -> pf_param_backward): the packed input,
// the stem's pre-LayerNorm output and the residual stream before and after every block (xs[s][j] = input of block j of stage s,
// xs[s][depth] = the stage's output).  Everything else is recomputed.
struct PnSaved {
  float* pin = nullptr;
  float* stem_pre = nullptr;
  float* xs[4][10] = {};
};
static int fwd_paramnet(Fwd& F, const float* grav, const float* lat, float* params, float* raw, const PnSaved* sv = nullptr);
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
    if (!dry) LAUNCHED(launch_pdl(stem_gather_kernel, dim3(ew_grid(stem_gather_threads(n, LH, LW))), dim3(256), 0, st, x0, col.hi, col.lo, n, LH, LW, 2, NH, NW));
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
      if (!dry) LAUNCHED(launch_pdl(stem_gather_kernel, dim3(ew_grid(stem_gather_threads(n, RH[0], RW[0]))), dim3(256), 0, st, x0, col.hi, col.lo, n, RH[0], RW[0], 4, NH, NW));
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
      if (!dry) LAUNCHED(launch_pdl(dwconv3x3_gelu_kernel, dim3(ew_grid((long long)n * ((RH[s] + 1) / 2) * ((RW[s] + PF_DW3_PX - 1) / PF_DW3_PX) * C)), dim3(256), 0, st, h1, nullptr, n, RH[s], RW[s], 4 * C, b.dw_w, b.dw_b, h2.hi, h2.lo));
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
        if (!dry) LAUNCHED(launch_pdl(upsample2x_kernel, dim3(ew_grid(upsample2x_threads(n, rh, rw, 512))), dim3(256), 0, st, w2, 512, 0, up, 512, 0, n, rh, rw, 512, nullptr, nullptr));
        fused = up;
        TRY(F.tapf(up, px * 4 * 512, "head.fusion%d", lvl));
      } else {
        fused_s = F.salloc(px * 4, 512);
        if (!dry) LAUNCHED(launch_pdl(upsample2x_kernel, dim3(ew_grid(upsample2x_threads(n, rh, rw, 512))), dim3(256), 0, st, w2, 512, 0, nullptr, 512, 0, n, rh, rw, 512, fused_s.hi, fused_s.lo));
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
static int fwd_paramnet(Fwd& F, const float* grav, const float* lat, float* params, float* raw, const PnSaved* sv) {
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
    if (!dry) LAUNCHED((pack_fields_kernel<<<(unsigned)cdivl((long long)n * SH * SW, 256), 256, 0, st>>>(grav, lat, pin, n, NH, NW, SH, SW), cudaGetLastError()));
    int rh = SH / 4, rw = SW / 4;
    float* x = sv ? sv->xs[0][0] : ar.f((long long)n * rh * rw * 96);
    float* stem = sv ? sv->stem_pre : x;
    if (!dry) LAUNCHED((stem_conv_launch<4, 4, 4, 0, 96>(pin, 4, n, SH, SW, e->pn_stem_w, e->pn_stem_b, stem, st)));
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
        if (!dry) LAUNCHED(launch_pdl(dwconv7x7_kernel, dim3(ew_grid((long long)n * ((rh + 1) / 2) * ((rw + PF_DW7_PX - 1) / PF_DW7_PX) * (C / 4))), dim3(256), 0, st, x, yf, n, rh, rw, C, b.dw_w, b.dw_b));
        TRY(F.ln_split(yf, y, rows, C, b.ln, 1e-6f));
        { Epi o; o.S = h; o.act = 2; TRY(F.tgemm(y, rows, C, 0, b.pw1, 4 * C, o)); }
        float* xo = sv ? sv->xs[s][j + 1] : x;     // training keeps every block's input: out of place, same arithmetic
        { Epi o; o.C = xo; o.ldc = C; o.res = x; o.ldr = C; o.gamma = b.gamma; TRY(F.tgemm(h, rows, 4 * C, 0, b.pw2, C, o)); }
        x = xo;
      }
      TRY(F.tapf(x, rows * C, "cnx.s%d", s));
    }
    if (!dry) {
      if (!params) return fail(PF_ERR_ARG, "params output is NULL");
      LAUNCHED((param_tail_kernel<<<n, 256, 0, st>>>(x, rh * rw, e->pn_norm.w, e->pn_norm.b, e->pn_head_w, e->pn_head_b, params, raw, D.param_net), cudaGetLastError()));
    }
  }
  return PF_OK;
}

// ----------------------------------------------------------------------------------------------- ParamNet training
// The fields' size at the ConvNeXt input (centred: the working size; uncentred: INPUT_SIZE square)
static void pn_input_size(const pf_engine* e, int* SH, int* SW) {
  const bool centered = e->desc.param_net == PF_PARAM_CENTERED;
  *SH = centered ? e->net_h : e->desc.param_input_size;
  *SW = centered ? e->net_w : e->desc.param_input_size;
}

// The saved activations sit at the start of the workspace, so the training forward and the backward find them at the same place.
static void pn_saved_alloc(Fwd& F, PnSaved& sv) {
  int SH, SW;
  pn_input_size(F.e, &SH, &SW);
  const long long n = F.n;
  sv.pin = F.ar.f(n * SH * SW * 4);
  int rh = SH / 4, rw = SW / 4;
  sv.stem_pre = F.ar.f(n * rh * rw * 96);
  for (int s = 0; s < 4; ++s) {
    if (s > 0) { rh /= 2; rw /= 2; }
    for (int j = 0; j <= kCnxDepths[s]; ++j) sv.xs[s][j] = F.ar.f(n * rh * rw * kCnxDims[s]);
  }
}

// Gradient buffer of pf_param_backward: one fp32 tensor per ParamNet parameter in the engine's layout, back to back in this order
// (a parameter's weight and bias are adjacent: the reductions write both at once).
struct PnGradEntry { std::string name; long long off, numel; };
static const std::vector<PnGradEntry>& pn_grad_layout() {
  static const std::vector<PnGradEntry> v = [] {
    std::vector<PnGradEntry> out;
    long long off = 0;
    auto add = [&](const std::string& nm, long long k) { out.push_back({nm, off, k}); off += k; };
    add("pn.stem.w", 48 * 96); add("pn.stem.b", 96); add("pn.stem.ln.w", 96); add("pn.stem.ln.b", 96);
    char nm[64];
    for (int s = 0; s < 4; ++s) {
      const int C = kCnxDims[s];
      if (s > 0) {
        const int Cp = kCnxDims[s - 1];
        snprintf(nm, sizeof nm, "pn.ds%d.", s);
        std::string P(nm);
        add(P + "ln.w", Cp); add(P + "ln.b", Cp); add(P + "w", 4LL * Cp * C); add(P + "b", C);
      }
      for (int j = 0; j < kCnxDepths[s]; ++j) {
        snprintf(nm, sizeof nm, "pn.s%d.b%d.", s, j);
        std::string P(nm);
        add(P + "dw.w", 49LL * C); add(P + "dw.b", C); add(P + "ln.w", C); add(P + "ln.b", C);
        add(P + "pw1.w", 4LL * C * C); add(P + "pw1.b", 4 * C); add(P + "pw2.w", 4LL * C * C); add(P + "pw2.b", C); add(P + "gamma", C);
      }
    }
    add("pn.norm.w", 768); add("pn.norm.b", 768); add("pn.head.w", 5 * 768); add("pn.head.b", 5);
    return out;
  }();
  return v;
}
static long long pn_grad_numel() { const auto& v = pn_grad_layout(); return v.back().off + v.back().numel; }
static long long pn_goff(const std::string& name) {
  static const std::unordered_map<std::string, long long> m = [] {
    std::unordered_map<std::string, long long> r;
    for (const auto& g : pn_grad_layout()) r[g.name] = g.off;
    return r;
  }();
  return m.at(name);
}

static int resolve_train_weights(pf_engine* e) {
  auto& T = e->pn_train;
  char nm[96];
  for (int s = 1; s < 4; ++s) {
    const long long numel = 4LL * kCnxDims[s - 1] * kCnxDims[s];
    snprintf(nm, sizeof nm, "pn.ds%d.t", s);
    std::string P(nm);
    TRY(get_w(e, P + ".whi", PF_BF16, numel, (const void**)&T.ds_t[s].hi));
    TRY(get_w(e, P + ".wlo", PF_BF16, numel, (const void**)&T.ds_t[s].lo));
  }
  for (int s = 0; s < 4; ++s) {
    const int C = kCnxDims[s];
    T.pw1_t[s].assign(kCnxDepths[s], GemmW());
    T.pw2_t[s].assign(kCnxDepths[s], GemmW());
    T.dw_rot[s].assign(kCnxDepths[s], nullptr);
    for (int j = 0; j < kCnxDepths[s]; ++j) {
      snprintf(nm, sizeof nm, "pn.s%d.b%d.", s, j);
      std::string P(nm);
      for (int k = 0; k < 2; ++k) {
        GemmW& g = k ? T.pw2_t[s][j] : T.pw1_t[s][j];
        const std::string q = P + (k ? "pw2t" : "pw1t");
        TRY(get_w(e, q + ".whi", PF_BF16, 4LL * C * C, (const void**)&g.hi));
        TRY(get_w(e, q + ".wlo", PF_BF16, 4LL * C * C, (const void**)&g.lo));
      }
      TRY(get_f(e, P + "dw.wr", 49LL * C, &T.dw_rot[s][j]));
    }
  }
  TRY(get_f(e, "pn.zero", 768, &T.zero));
  return PF_OK;
}

static int pn_reduce(Fwd& F, const float* part, int P, long long L, float* out) {
  if (!F.dry) LAUNCHED((reduce_partials_kernel<<<(unsigned)cdivl(L, 32), 256, 0, F.st>>>(part, P, L, out), cudaGetLastError()));
  return PF_OK;
}
// out[c] = sum over the R rows of src [R x C]
static int pn_colsum(Fwd& F, const float* src, long long R, int C, float* out) {
  const long long rpb = std::max(256LL, cdivl(R, 2048));
  const int P = (int)cdivl(R, rpb);
  const long long m = F.ar.mark();
  float* part = F.ar.f((long long)P * C);
  if (!F.dry) LAUNCHED((colsum_partial_kernel<<<dim3(P, cdiv(C, 32)), 256, 0, F.st>>>(src, R, C, rpb, part), cudaGetLastError()));
  TRY(pn_reduce(F, part, P, C, out));
  F.ar.release(m);
  return PF_OK;
}
// LayerNorm backward: dx (written) and the weight / bias gradients at g, g + C
static int pn_ln_bwd(Fwd& F, const float* x, const float* dy, long long R, int C, const float* w, float* dx, float* g) {
  const long long rpb = std::max(64LL, cdivl(R, 2048));
  const int P = (int)cdivl(R, rpb);
  const long long m = F.ar.mark();
  float* part = F.ar.f((long long)P * 2 * C);
  if (!F.dry) LAUNCHED((ln_bwd_kernel<<<P, 256, 0, F.st>>>(x, dy, R, C, w, 1e-6f, rpb, dx, part), cudaGetLastError()));
  TRY(pn_reduce(F, part, P, 2LL * C, g));
  F.ar.release(m);
  return PF_OK;
}

// Weight gradient dW[N x K] = sum over R rows of dY[r][n] X[r][k] on the GEMM engine: the rows are cut into S chunks, each chunk is
// one group of a grouped GEMM-mode launch (A = dY^T [N][S chunk], B = X^T [S][K][chunk], both transposed split copies), which writes
// per-chunk partials [S][N][K]; pn_reduce adds them in order.  S is chosen from the shapes so that the launch fills the SMs.
struct WgPlan { int S, chunk; long long Rp; };
static WgPlan pn_wg_plan(const pf_engine* e, long long R, int N, int K) {
  const int bn = tma_pick_bn(K, MODE_GEMM);
  const long long tiles = (long long)cdiv(N, 128) * cdiv(K, bn);
  long long S = cdivl(2LL * e->sm_count, tiles);
  S = std::min(S, std::max(1LL, R / 1024));
  S = std::max(1LL, std::min(S, 256LL));
  WgPlan p;
  p.chunk = (int)(cdivl(cdivl(R, S), 64) * 64);
  p.S = (int)cdivl(R, p.chunk);
  p.Rp = (long long)p.S * p.chunk;
  return p;
}
// transposed split copy of [R x C] (fp32 src with row pitch ld, or split planes ssrc): layout A [C][Rp], layout B [S][C][chunk]
static int pn_tsplit(Fwd& F, const float* src, const SplitT* ssrc, int ld, long long R, int C, const WgPlan& pl, bool layout_b, int op, SplitT& out) {
  out = F.salloc(pl.Rp, C);
  if (F.dry) return PF_OK;
  const long long sS = layout_b ? (long long)C * pl.chunk : pl.chunk, sC = layout_b ? pl.chunk : pl.Rp;
  const dim3 grid((unsigned)cdivl(pl.Rp, 32), (unsigned)cdiv(C, 32));
  if (ssrc) LAUNCHED((transpose_split_kernel<true, 0><<<grid, 256, 0, F.st>>>(nullptr, ssrc->hi, ssrc->lo, ld, R, pl.Rp, C, pl.chunk, sS, sC, out.hi, out.lo), cudaGetLastError()));
  else if (op == 1) LAUNCHED((transpose_split_kernel<false, 1><<<grid, 256, 0, F.st>>>(src, nullptr, nullptr, ld, R, pl.Rp, C, pl.chunk, sS, sC, out.hi, out.lo), cudaGetLastError()));
  else LAUNCHED((transpose_split_kernel<false, 0><<<grid, 256, 0, F.st>>>(src, nullptr, nullptr, ld, R, pl.Rp, C, pl.chunk, sS, sC, out.hi, out.lo), cudaGetLastError()));
  return PF_OK;
}
static int pn_wgrad(Fwd& F, const SplitT& aT, const SplitT& bT, int N, int K, const WgPlan& pl, float* part) {
  TmaGemmParams p{};
  p.M = N; p.N = K; p.K = pl.chunk; p.Cin = pl.chunk; p.a_gc = pl.chunk; p.groups = pl.S;
  p.C = part; p.ldc = K; p.c_gcoff = N * K;
  const int bn = tma_pick_bn(K, MODE_GEMM), kb = tma_pick_kb(bn, pl.chunk, MODE_GEMM);
  // (checked in the sizing dry run too, so that a shape the engine cannot run fails before anything is launched)
  if (const char* msg = gemm_tma_check(MODE_GEMM, p, bn, kb, false, false, F.np())) return fail(PF_ERR_ARG, "weight-gradient GEMM (bn %d, kb %d): %s", bn, kb, msg);
  if (F.dry) return PF_OK;
  TmaMaps maps{};
  const char* msg = F.map2d(&maps.a_hi, aT.hi, pl.Rp, N, pl.Rp, 128, kb);
  if (!msg) msg = F.map2d(&maps.a_lo, aT.lo, pl.Rp, N, pl.Rp, 128, kb);
  if (!msg) msg = F.map2d(&maps.b_hi, bT.hi, pl.chunk, (long long)pl.S * K, pl.chunk, bn, kb);
  if (!msg) msg = F.map2d(&maps.b_lo, bT.lo, pl.chunk, (long long)pl.S * K, pl.chunk, bn, kb);
  if (msg) return fail(PF_ERR_CUDA, "%s", msg);
  maps.a2_hi = maps.a_hi; maps.a2_lo = maps.a_lo;
  F.picked_bn = bn; F.picked_kb = kb; F.picked_sched = 1;
  return F.launch_tma(MODE_GEMM, maps, p, bn, kb, false);
}
static int pn_wgrad_full(Fwd& F, const float* dy, int ldy, const SplitT* xs, const float* xf, int op, int ldx, long long R, int N, int K, float* out,
                         WgPlan* plan = nullptr) {
  const long long m = F.ar.mark();
  const WgPlan pl = pn_wg_plan(F.e, R, N, K);
  if (plan) *plan = pl;
  SplitT aT, bT;
  TRY(pn_tsplit(F, dy, nullptr, ldy, R, N, pl, false, 0, aT));
  TRY(pn_tsplit(F, xf, xs, ldx, R, K, pl, true, op, bT));
  float* part = F.ar.f((long long)pl.S * N * K);
  TRY(pn_wgrad(F, aT, bT, N, K, pl, part));
  TRY(pn_reduce(F, part, pl.S, (long long)N * K, out));
  F.ar.release(m);
  return PF_OK;
}

static int pn_dw_launch(Fwd& F, const float* x, float* y, int rh, int rw, int C, const float* w, const float* b) {
  if (!F.dry) LAUNCHED(launch_pdl(dwconv7x7_kernel, dim3(ew_grid((long long)F.n * ((rh + 1) / 2) * ((rw + PF_DW7_PX - 1) / PF_DW7_PX) * (C / 4))), dim3(256), 0, F.st,
                                  x, y, F.n, rh, rw, C, w, b));
  return PF_OK;
}

// Image rows per block of the depthwise and stem weight-gradient kernels: at most 1024 partials, one row each while that suffices
static int pn_rows_per_block(int rows) { return std::max(1, cdiv(rows, 1024)); }

// depthwise 7x7 weight and bias gradients of the F.n images [rh, rw, C]: out [50][C] (49 taps, then the bias)
static int pn_dw7_wgrad(Fwd& F, const float* xin, const float* dt, int rh, int rw, int C, float* out, int* rpb_out = nullptr) {
  const int rows = F.n * rh, rpb = pn_rows_per_block(rows), np_ = cdiv(rows, rpb);
  if (rpb_out) *rpb_out = rpb;
  const long long m = F.ar.mark();
  float* part = F.ar.f((long long)np_ * 50 * C);
  if (!F.dry) LAUNCHED((dw7_wgrad_kernel<<<dim3(np_, C / 32), 256, 0, F.st>>>(xin, dt, F.n, rh, rw, C, rpb, part), cudaGetLastError()));
  TRY(pn_reduce(F, part, np_, 50LL * C, out));
  F.ar.release(m);
  return PF_OK;
}

static int pn_pw2_grads(Fwd& F, const float* G, const float* sdy, int C, int K, const float* gamma, const GemmW& w2, float* dW, float* db, float* dgamma) {
  if (!F.dry) LAUNCHED((pw2_grads_kernel<<<cdiv(C, 8), 256, 0, F.st>>>(G, sdy, C, K, gamma, w2.hi, w2.lo, w2.b, dW, db, dgamma), cudaGetLastError()));
  return PF_OK;
}
static int pn_gelu_bwd(Fwd& F, const float* dh, float* u, long long n, __nv_bfloat16* hi, __nv_bfloat16* lo) {
  if (!F.dry) LAUNCHED((gelu_bwd_kernel<<<ew_grid(n), 256, 0, F.st>>>(dh, u, n, hi, lo), cudaGetLastError()));
  return PF_OK;
}
static int pn_scale_split(Fwd& F, const float* src, const float* scale, long long n, int C, const SplitT& out) {
  if (!F.dry) LAUNCHED((scale_split_kernel<<<ew_grid(n), 256, 0, F.st>>>(src, scale, n, C, out.hi, out.lo), cudaGetLastError()));
  return PF_OK;
}
static int pn_col2im2(Fwd& F, const float* dP, int rh, int rw, int C, float* out) {
  if (!F.dry) LAUNCHED((col2im2_kernel<<<ew_grid((long long)F.n * rh * rw * C), 256, 0, F.st>>>(dP, F.n, rh, rw, C, out), cudaGetLastError()));
  return PF_OK;
}

// One ConvNeXt block backward: dx holds d loss / d(block output) and becomes d loss / d(block input).  Recomputes dwconv -> LN ->
// pwconv1 from the saved input.
static int pn_block_bwd(Fwd& F, int s, int j, const float* xin, float* dx, int rh, int rw, float* grads) {
  pf_engine* e = F.e;
  Arena& ar = F.ar;
  const bool dry = F.dry;
  cudaStream_t st = F.st;
  const int C = kCnxDims[s];
  const long long R = (long long)F.n * rh * rw;
  const CnxBlockW& b = e->pn_blocks[s][j];
  const auto& T = e->pn_train;
  char nm[64];
  snprintf(nm, sizeof nm, "pn.s%d.b%d.", s, j);
  const std::string P(nm);
  const long long m0 = ar.mark();
  float* t = ar.f(R * C);
  TRY(pn_dw_launch(F, xin, t, rh, rw, C, b.dw_w, b.dw_b));
  SplitT ys = F.salloc(R, C);
  TRY(F.ln_split(t, ys, R, C, b.ln, 1e-6f));
  float* u = ar.f(R * 4 * C);                     // pwconv1 output before the GELU
  { Fwd::Epi o; o.C = u; o.ldc = 4 * C; TRY(F.tgemm(ys, R, C, 0, b.pw1, 4 * C, o)); }
  // pwconv2 and gamma from G = dx^T GELU(u) and the column sums of dx
  {
    const long long m1 = ar.mark();
    float* G = ar.f(4LL * C * C);
    float* sdx = ar.f(C);
    TRY(pn_wgrad_full(F, dx, C, nullptr, u, 1, 4 * C, R, C, 4 * C, G));
    TRY(pn_colsum(F, dx, R, C, sdx));
    TRY(pn_pw2_grads(F, G, sdx, C, 4 * C, b.gamma, b.pw2, grads + pn_goff(P + "pw2.w"), grads + pn_goff(P + "pw2.b"), grads + pn_goff(P + "gamma")));
    ar.release(m1);
  }
  // dh = (gamma dx) W2, then du = dh GELU'(u), written over u
  {
    const long long m1 = ar.mark();
    SplitT dz = F.salloc(R, C);
    TRY(pn_scale_split(F, dx, b.gamma, R * C, C, dz));
    float* dh = ar.f(R * 4 * C);
    { Fwd::Epi o; o.C = dh; o.ldc = 4 * C; TRY(F.tgemm(dz, R, C, 0, T.pw2_t[s][j], 4 * C, o)); }
    TRY(pn_gelu_bwd(F, dh, u, R * 4 * C, nullptr, nullptr));
    ar.release(m1);
  }
  // pwconv1 weight and bias
  TRY(pn_wgrad_full(F, u, 4 * C, &ys, nullptr, 0, C, R, 4 * C, C, grads + pn_goff(P + "pw1.w")));
  TRY(pn_colsum(F, u, R, 4 * C, grads + pn_goff(P + "pw1.b")));
  // dy = du W1
  float* dy = ar.f(R * C);
  {
    const long long m1 = ar.mark();
    SplitT du = F.salloc(R, 4 * C);
    TRY(pn_scale_split(F, u, nullptr, R * 4 * C, 4 * C, du));
    Fwd::Epi o; o.C = dy; o.ldc = C;
    TRY(F.tgemm(du, R, 4 * C, 0, T.pw1_t[s][j], C, o));
    ar.release(m1);
  }
  float* dt = ar.f(R * C);
  TRY(pn_ln_bwd(F, t, dy, R, C, b.ln.w, dt, grads + pn_goff(P + "ln.w")));
  // depthwise 7x7: weight and bias, then the data gradient (the forward kernel with the rotated kernel) added to the residual's
  TRY(pn_dw7_wgrad(F, xin, dt, rh, rw, C, grads + pn_goff(P + "dw.w")));
  TRY(pn_dw_launch(F, dt, dy, rh, rw, C, T.dw_rot[s][j], T.zero));
  if (!dry) LAUNCHED((add_inplace_kernel<<<ew_grid(R * C), 256, 0, st>>>(dx, dy, R * C), cudaGetLastError()));
  ar.release(m0);
  return PF_OK;
}

// Downsample s (LayerNorm, then the 2x2 / stride 2 conv) backward: dxn = d loss / d(its output) -> dprev = d loss / d(its input xprev)
static int pn_downsample_bwd(Fwd& F, int s, const float* xprev, int rh, int rw, const float* dxn, float* dprev, float* grads) {
  pf_engine* e = F.e;
  Arena& ar = F.ar;
  const int Cp = kCnxDims[s - 1], C = kCnxDims[s];
  const long long R = (long long)F.n * rh * rw, R2 = R / 4;
  char nm[64];
  snprintf(nm, sizeof nm, "pn.ds%d.", s);
  const std::string P(nm);
  const long long m0 = ar.mark();
  SplitT patch = F.salloc(R2, 4 * Cp);
  TRY(F.ln_split_patch(xprev, SplitT(), patch, R, Cp, e->pn_ds_ln[s], 1e-6f, rh, rw, 2));
  TRY(pn_wgrad_full(F, dxn, C, &patch, nullptr, 0, 4 * Cp, R2, C, 4 * Cp, grads + pn_goff(P + "w")));
  TRY(pn_colsum(F, dxn, R2, C, grads + pn_goff(P + "b")));
  float* dln = ar.f(R * Cp);
  {
    const long long m1 = ar.mark();
    SplitT d = F.salloc(R2, C);
    TRY(pn_scale_split(F, dxn, nullptr, R2 * C, C, d));
    float* dP = ar.f(R2 * 4 * Cp);
    Fwd::Epi o; o.C = dP; o.ldc = 4 * Cp;
    TRY(F.tgemm(d, R2, C, 0, e->pn_train.ds_t[s], 4 * Cp, o));
    TRY(pn_col2im2(F, dP, rh, rw, Cp, dln));
    ar.release(m1);
  }
  TRY(pn_ln_bwd(F, xprev, dln, R, Cp, e->pn_ds_ln[s].w, dprev, grads + pn_goff(P + "ln.w")));
  ar.release(m0);
  return PF_OK;
}

// tail (pool -> LayerNorm(768) -> head) backward of the F.n pairs: dx [n, HW, 768] and the tail's gradients at g (norm.w, norm.b,
// head.w, head.b: kTailGrads values)
static int pn_tail_bwd(Fwd& F, const float* feat, int HW, const float* nw, const float* nb, const float* hw, const float* draw, float* dx, float* g) {
  const long long m = F.ar.mark();
  float* part = F.ar.f((long long)F.n * kTailGrads);
  if (!F.dry) LAUNCHED((param_tail_bwd_kernel<<<F.n, 256, 0, F.st>>>(feat, HW, nw, nb, hw, draw, dx, part), cudaGetLastError()));
  TRY(pn_reduce(F, part, F.n, kTailGrads, g));
  F.ar.release(m);
  return PF_OK;
}

// stem weight and bias gradients from the packed input [n, 4 OH, 4 OW, 4] and dS [n, OH, OW, 96]: out [49][96] (48 weight rows
// (ky, kx, ci), then the bias)
static int pn_stem_wgrad(Fwd& F, const float* pin, const float* dS, int OH, int OW, float* out, int* rpb_out = nullptr) {
  const int rows = F.n * OH, rpb = pn_rows_per_block(rows), np_ = cdiv(rows, rpb);
  if (rpb_out) *rpb_out = rpb;
  const long long m = F.ar.mark();
  float* part = F.ar.f((long long)np_ * 49 * 96);
  if (!F.dry) LAUNCHED((stem_wgrad_kernel<<<dim3(np_, 3), 256, 0, F.st>>>(pin, dS, F.n, OH, OW, rpb, part), cudaGetLastError()));
  TRY(pn_reduce(F, part, np_, 49LL * 96, out));
  F.ar.release(m);
  return PF_OK;
}
static int pn_stem_dgrad(Fwd& F, const float* dS, const float* w, int OH, int OW, float* dpin) {
  if (!F.dry) LAUNCHED((stem_dgrad_kernel<<<ew_grid((long long)F.n * OH * OW * 48), 256, 0, F.st>>>(dS, w, F.n, OH, OW, dpin), cudaGetLastError()));
  return PF_OK;
}
// backward of the nearest resize of the fields IH x IW -> OH x OW (pack_fields_kernel)
static int pn_fields_grad(Fwd& F, const float* dpin, int IH, int IW, int OH, int OW, float* dgrav, float* dlat) {
  if (!F.dry)
    LAUNCHED((unpack_fields_grad_kernel<<<(unsigned)cdivl((long long)F.n * IH * IW, 256), 256, 0, F.st>>>(dpin, F.n, IH, IW, OH, OW, dgrav, dlat), cudaGetLastError()));
  return PF_OK;
}

// ParamNet backward from draw [n, 5] (d loss / d raw head outputs) over the activations pf_param_train_forward saved: every
// parameter gradient into grads (pn_grad_layout, overwritten) and, when dgrav / dlat are non-NULL, the fields' gradients.
static int bwd_paramnet(Fwd& F, const PnSaved& sv, const float* draw, float* grads, float* dgrav, float* dlat) {
  pf_engine* e = F.e;
  Arena& ar = F.ar;
  const int n = F.n;
  int SH, SW;
  pn_input_size(e, &SH, &SW);
  int rh[4], rw[4];
  rh[0] = SH / 4; rw[0] = SW / 4;
  for (int s = 1; s < 4; ++s) { rh[s] = rh[s - 1] / 2; rw[s] = rw[s - 1] / 2; }
  float* dx = ar.f((long long)n * rh[3] * rw[3] * 768);
  TRY(pn_tail_bwd(F, sv.xs[3][kCnxDepths[3]], rh[3] * rw[3], e->pn_norm.w, e->pn_norm.b, e->pn_head_w, draw, dx, grads + pn_goff("pn.norm.w")));
  for (int s = 3; s >= 0; --s) {
    for (int j = kCnxDepths[s] - 1; j >= 0; --j) TRY(pn_block_bwd(F, s, j, sv.xs[s][j], dx, rh[s], rw[s], grads));
    if (s > 0) {
      float* dprev = ar.f((long long)n * rh[s - 1] * rw[s - 1] * kCnxDims[s - 1]);
      TRY(pn_downsample_bwd(F, s, sv.xs[s - 1][kCnxDepths[s - 1]], rh[s - 1], rw[s - 1], dx, dprev, grads));
      dx = dprev;
    }
  }
  // stem: LayerNorm, then the 4x4 / stride 4 conv
  const long long R0 = (long long)n * rh[0] * rw[0];
  float* dstem = ar.f(R0 * 96);
  TRY(pn_ln_bwd(F, sv.stem_pre, dx, R0, 96, e->pn_stem_ln.w, dstem, grads + pn_goff("pn.stem.ln.w")));
  TRY(pn_stem_wgrad(F, sv.pin, dstem, rh[0], rw[0], grads + pn_goff("pn.stem.w")));
  if (dgrav) {
    float* dpin = ar.f((long long)n * SH * SW * 4);
    TRY(pn_stem_dgrad(F, dstem, e->pn_stem_w, rh[0], rw[0], dpin));
    TRY(pn_fields_grad(F, dpin, e->net_h, e->net_w, SH, SW, dgrav, dlat));
  }
  return PF_OK;
}

// the two training passes, each starting with the saved activations at the bottom of the workspace
static int pn_train_pass(Fwd& F, bool backward, const float* grav, const float* lat, float* raw, const float* draw, float* grads, float* dgrav, float* dlat) {
  PnSaved sv;
  pn_saved_alloc(F, sv);
  if (backward) return bwd_paramnet(F, sv, draw, grads, dgrav, dlat);
  float* params = F.ar.f((long long)F.n * 8);
  return fwd_paramnet(F, grav, lat, params, raw, &sv);
}
static int pn_train_peak(pf_handle h, int n, long long* peak) {
  *peak = 0;
  for (int b = 0; b < 2; ++b) {
    Fwd T{h, Arena{}, nullptr, true, n};
    T.ar.dry = true;
    TRY(pn_train_pass(T, b == 1, nullptr, nullptr, nullptr, nullptr, nullptr, b == 1 ? (float*)1 : nullptr, nullptr));
    *peak = std::max(*peak, T.ar.peak);
  }
  return PF_OK;
}

// ----------------------------------------------------------------------------------------------- C ABI
extern "C" {

int pf_abi_version(void) { return PF_ABI_VERSION; }
const char* pf_last_error(void) { return g_err.c_str(); }
int64_t pf_kernel_launch_count(void) { return g_launches.load(); }

// The opt-in for more than 48 KB of dynamic shared memory is a per-device attribute of each kernel: set for every kernel of the
// library on every device an engine (or an operator entry point) uses, once per device and thread-safe.
static int configure_device(int device) {
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
static int configure_current_device() {
  int dev = 0;
  CU(cudaGetDevice(&dev));
  return configure_device(dev);
}

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

static int pn_train_check(const char* fn, pf_handle h, int n, void* workspace, int64_t workspace_bytes) {
  if (!h) return fail(PF_ERR_ARG, "%s: null handle", fn);
  if (!h->finalized) return fail(PF_ERR_WEIGHT, "%s: pf_finalize has not succeeded", fn);
  if (h->desc.param_net == PF_PARAM_NONE) return fail(PF_ERR_ARG, "%s: this model has no ParamNet", fn);
  if (n < 1) return fail(PF_ERR_ARG, "%s: n = %d, at least 1 pair of fields is needed", fn, n);
  if (!workspace) return fail(PF_ERR_ARG, "%s: null workspace", fn);
  long long peak = 0;
  TRY(pn_train_peak(h, n, &peak));
  if (peak > workspace_bytes) return fail(PF_ERR_ARG, "%s: workspace %lld B < required %lld B", fn, (long long)workspace_bytes, peak);
  if (((uintptr_t)workspace & 255) != 0) return fail(PF_ERR_ARG, "%s: workspace must be 256-byte aligned", fn);
  return PF_OK;
}

int64_t pf_param_train_workspace_bytes(pf_handle h, int n) {
  if (!h || n < 1) return fail(PF_ERR_ARG, "pf_param_train_workspace_bytes: bad argument");
  if (!h->finalized) return fail(PF_ERR_WEIGHT, "pf_param_train_workspace_bytes: pf_finalize has not succeeded");
  if (h->desc.param_net == PF_PARAM_NONE) return fail(PF_ERR_ARG, "pf_param_train_workspace_bytes: this model has no ParamNet");
  long long peak = 0;
  TRY(pn_train_peak(h, n, &peak));
  return peak + 4096;
}

int pf_param_train_forward(pf_handle h, int n, const float* gravity, const float* latitude, float* raw, void* workspace, int64_t workspace_bytes,
                           void* stream) {
  TRY(pn_train_check("pf_param_train_forward", h, n, workspace, workspace_bytes));
  if (!gravity || !latitude || !raw) return fail(PF_ERR_ARG, "pf_param_train_forward: null gravity / latitude / raw");
  CU(cudaSetDevice(h->device));
  Fwd F{h, Arena{}, (cudaStream_t)stream, false, n};
  F.ar.base = (char*)workspace;
  F.ar.cap = workspace_bytes;
  NvtxRange r_("pf:paramnet_train_forward");
  return pn_train_pass(F, false, gravity, latitude, raw, nullptr, nullptr, nullptr, nullptr);
}

int pf_param_backward(pf_handle h, int n, const float* draw, float* grads, float* grad_gravity, float* grad_latitude, void* workspace,
                      int64_t workspace_bytes, void* stream) {
  TRY(pn_train_check("pf_param_backward", h, n, workspace, workspace_bytes));
  if (!draw || !grads) return fail(PF_ERR_ARG, "pf_param_backward: null draw / grads");
  if ((grad_gravity == nullptr) != (grad_latitude == nullptr)) return fail(PF_ERR_ARG, "pf_param_backward: grad_gravity and grad_latitude are both NULL or both set");
  TRY(resolve_train_weights(h));
  CU(cudaSetDevice(h->device));
  Fwd F{h, Arena{}, (cudaStream_t)stream, false, n};
  F.ar.base = (char*)workspace;
  F.ar.cap = workspace_bytes;
  NvtxRange r_("pf:paramnet_backward");
  return pn_train_pass(F, true, nullptr, nullptr, nullptr, draw, grads, grad_gravity, grad_latitude);
}

int64_t pf_param_grad_numel(void) { return pn_grad_numel(); }

int pf_param_grad_entry(int i, const char** name, int64_t* offset, int64_t* numel) {
  const auto& v = pn_grad_layout();
  if (i < 0 || i >= (int)v.size() || !name || !offset || !numel) return fail(PF_ERR_ARG, "pf_param_grad_entry: bad argument");
  *name = v[i].name.c_str();
  *offset = v[i].off;
  *numel = v[i].numel;
  return PF_OK;
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

// ---- multi-GPU gather (NCCL point-to-point; SURVEY.md 8e) ---------------------------------------------------
#define NCCL_TRY(expr)                                                                                              \
  do {                                                                                                              \
    int r__ = (expr);                                                                                               \
    if (r__ != kNcclSuccess) return fail(PF_ERR_CUDA, "%s: %s", #expr, api.GetErrorString ? api.GetErrorString(r__) : "NCCL error"); \
  } while (0)
int pf_comm_unique_id(void* id128) {
  if (!id128) return fail(PF_ERR_ARG, "pf_comm_unique_id: null argument");
  const NcclApi& api = nccl_api();
  if (api.error) return fail(PF_ERR_CUDA, "%s", api.error);
  static_assert(sizeof(NcclUniqueId) == 128, "ncclUniqueId is 128 bytes");
  NCCL_TRY(api.GetUniqueId((NcclUniqueId*)id128));
  return PF_OK;
}
int pf_comm_create(int device, int rank, int nranks, const void* id128, pf_comm_handle* out) {
  if (!id128 || !out || nranks < 1 || rank < 0 || rank >= nranks) return fail(PF_ERR_ARG, "pf_comm_create: bad argument");
  const NcclApi& api = nccl_api();
  if (api.error) return fail(PF_ERR_CUDA, "%s", api.error);
  CU(cudaSetDevice(device));
  NcclUniqueId id;
  memcpy(&id, id128, sizeof id);
  pf_comm* c = new pf_comm();
  c->device = device; c->rank = rank; c->nranks = nranks;
  const int r = api.CommInitRank(&c->comm, nranks, id, rank);
  if (r != kNcclSuccess) { delete c; return fail(PF_ERR_CUDA, "ncclCommInitRank: %s", api.GetErrorString(r)); }
  *out = c;
  return PF_OK;
}
int pf_comm_destroy(pf_comm_handle c) {
  if (!c) return PF_OK;
  const NcclApi& api = nccl_api();
  cudaSetDevice(c->device);
  if (c->comm && api.CommDestroy) api.CommDestroy(c->comm);
  delete c;
  return PF_OK;
}
int pf_gather(pf_comm_handle c, int root, int count, void* const* dev_ptrs, const int64_t* bytes, const int32_t* peer, void* stream) {
  if (!c || count < 0 || root < 0 || root >= c->nranks || (count > 0 && (!dev_ptrs || !bytes))) return fail(PF_ERR_ARG, "pf_gather: bad argument");
  if (c->rank == root && count > 0 && !peer) return fail(PF_ERR_ARG, "pf_gather: the root needs the source rank of every segment");
  const NcclApi& api = nccl_api();
  CU(cudaSetDevice(c->device));
  if (count == 0) return PF_OK;
  NCCL_TRY(api.GroupStart());
  for (int i = 0; i < count; ++i) {
    int r;
    if (c->rank == root) {
      if (peer[i] < 0 || peer[i] >= c->nranks || peer[i] == root) { api.GroupEnd(); return fail(PF_ERR_ARG, "pf_gather: segment %d comes from rank %d", i, peer[i]); }
      r = api.Recv(dev_ptrs[i], (size_t)bytes[i], kNcclUint8, peer[i], c->comm, (cudaStream_t)stream);
    } else {
      r = api.Send(dev_ptrs[i], (size_t)bytes[i], kNcclUint8, root, c->comm, (cudaStream_t)stream);
    }
    if (r != kNcclSuccess) { api.GroupEnd(); return fail(PF_ERR_CUDA, "ncclSend/Recv: %s", api.GetErrorString(r)); }
  }
  NCCL_TRY(api.GroupEnd());
  return PF_OK;
}

// ---- decode front-end (nvJPEG; SURVEY.md 8f-2) ------------------------------------------------------------------
int pf_jpeg_create(int device, int max_threads, pf_jpeg_handle* out) {
  if (!out) return fail(PF_ERR_ARG, "pf_jpeg_create: null argument");
  const NvjpegApi& api = nvjpeg_api();
  if (api.error) return fail(PF_ERR_CUDA, "%s", api.error);
  CU(cudaSetDevice(device));
  pf_jpeg* j = new pf_jpeg();
  j->device = device;
  if (api.CreateSimple(&j->handle) != NVJPEG_STATUS_SUCCESS) { delete j; return fail(PF_ERR_CUDA, "nvjpegCreateSimple failed"); }
  int nt = max_threads > 0 ? max_threads : (int)std::thread::hardware_concurrency() / 2;
  nt = nt < 1 ? 1 : (nt > 32 ? 32 : nt);
  j->workers.resize(nt);
  bool ok = cudaEventCreateWithFlags(&j->start, cudaEventDisableTiming) == cudaSuccess;
  for (auto& w : j->workers) {
    ok = ok && api.StateCreate(j->handle, &w.state) == NVJPEG_STATUS_SUCCESS;
    ok = ok && cudaStreamCreateWithFlags(&w.stream, cudaStreamNonBlocking) == cudaSuccess;
    ok = ok && cudaEventCreateWithFlags(&w.done, cudaEventDisableTiming) == cudaSuccess;
  }
  if (!ok) { pf_jpeg_destroy(j); return fail(PF_ERR_CUDA, "pf_jpeg_create: decoder state / stream creation failed"); }
  *out = j;
  return PF_OK;
}
int pf_jpeg_destroy(pf_jpeg_handle j) {
  if (!j) return PF_OK;
  const NvjpegApi& api = nvjpeg_api();
  cudaSetDevice(j->device);
  for (auto& w : j->workers) {
    if (w.stream) cudaStreamSynchronize(w.stream);
    if (w.state) api.StateDestroy(w.state);
    if (w.stream) cudaStreamDestroy(w.stream);
    if (w.done) cudaEventDestroy(w.done);
  }
  if (j->start) cudaEventDestroy(j->start);
  if (j->handle) api.Destroy(j->handle);
  delete j;
  return PF_OK;
}
int pf_jpeg_info(pf_jpeg_handle j, const uint8_t* data, int64_t length, int32_t* height, int32_t* width) {
  if (!j || !data || length < 4 || !height || !width) return fail(PF_ERR_ARG, "pf_jpeg_info: bad argument");
  const NvjpegApi& api = nvjpeg_api();
  int nc = 0, ws[NVJPEG_MAX_COMPONENT] = {0}, hs[NVJPEG_MAX_COMPONENT] = {0};
  nvjpegChromaSubsampling_t ss;
  if (api.GetImageInfo(j->handle, data, (size_t)length, &nc, &ss, ws, hs) != NVJPEG_STATUS_SUCCESS) return fail(PF_ERR_ARG, "pf_jpeg_info: not a decodable JPEG stream");
  *height = hs[0]; *width = ws[0];
  return PF_OK;
}
int pf_jpeg_decode_batch(pf_jpeg_handle j, int n, const uint8_t* const* data, const int64_t* length, const int32_t* height, const int32_t* width,
                         uint8_t* blob, const int64_t* offset, void* stream) {
  if (!j || n < 1 || !data || !length || !height || !width || !blob || !offset) return fail(PF_ERR_ARG, "pf_jpeg_decode_batch: bad argument");
  const NvjpegApi& api = nvjpeg_api();
  CU(cudaSetDevice(j->device));
  cudaStream_t st = (cudaStream_t)stream;
  // the workers' streams start after everything already queued on the caller's stream (the blob may be in use by an earlier forward)
  CU(cudaEventRecord(j->start, st));
  const int nt = (int)j->workers.size() < n ? (int)j->workers.size() : n;
  std::atomic<int> next{0}, failed{-1};
  auto work = [&](int t) {
    cudaSetDevice(j->device);
    pf_jpeg::Worker& w = j->workers[t];
    cudaStreamWaitEvent(w.stream, j->start, 0);
    for (int i = next.fetch_add(1); i < n; i = next.fetch_add(1)) {
      nvjpegImage_t dst{};
      dst.channel[0] = blob + offset[i];
      dst.pitch[0] = (size_t)width[i] * 3;
      if (api.Decode(j->handle, w.state, data[i], (size_t)length[i], NVJPEG_OUTPUT_BGRI, &dst, w.stream) != NVJPEG_STATUS_SUCCESS) failed.store(i);
    }
    cudaEventRecord(w.done, w.stream);
  };
  std::vector<std::thread> threads;
  for (int t = 1; t < nt; ++t) threads.emplace_back(work, t);
  work(0);
  for (auto& th : threads) th.join();
  for (int t = 0; t < nt; ++t) CU(cudaStreamWaitEvent(st, j->workers[t].done, 0));
  if (failed.load() >= 0) return fail(PF_ERR_ARG, "pf_jpeg_decode_batch: image %d could not be decoded", failed.load());
  return PF_OK;
}

// ---- single-operator entry points ------------------------------------------------------------------------
int pf_op_conv_gemm(const float* x, int B, int H, int W, int Cin, const void* whi, const void* wlo, const float* bias, int N, int KH, int KW,
                    int stride, int pad, int in_relu, int act, const float* res, int res_relu, float* y, void* stream) {
  // split the input the way a producer kernel would, then run the same helpers the forward graph uses
  if (!x || !whi || !wlo || !y) return fail(PF_ERR_ARG, "pf_op_conv_gemm: null argument");
  if (KH != KW) return fail(PF_ERR_ARG, "pf_op_conv_gemm: square filters only");
  TRY(configure_current_device());
  cudaStream_t st = (cudaStream_t)stream;
  int dev = 0;
  CU(cudaGetDevice(&dev));
  cudaDeviceProp prop;
  CU(cudaGetDeviceProperties(&prop, dev));
  pf_engine tmp;
  tmp.device = dev;
  tmp.sm_count = prop.multiProcessorCount;
  const int OH = (H + 2 * pad - KH) / stride + 1, OW = (W + 2 * pad - KW) / stride + 1;
  const long long nx = (long long)B * H * W * Cin;
  const long long colb = (long long)B * OH * OW * KH * KW * Cin * 4 + (1 << 20);
  char* scratch = nullptr;
  CU(cudaMalloc(&scratch, nx * 4 + colb + 4096));
  Fwd F{&tmp, Arena{}, st, false, B};
  F.ar.base = scratch; F.ar.cap = nx * 4 + colb + 4096;
  SplitT A = F.salloc((long long)B * H * W, Cin);
  int r = PF_OK;
  {
    cudaError_t le = (split_kernel<<<(unsigned)cdivl(nx, 256), 256, 0, st>>>(x, A.hi, A.lo, nx, in_relu), cudaGetLastError());
    g_launches.fetch_add(1, std::memory_order_relaxed);
    if (le != cudaSuccess) r = fail(PF_ERR_CUDA, "split_kernel: %s", cudaGetErrorString(le));
  }
  GemmW w{(const __nv_bfloat16*)whi, (const __nv_bfloat16*)wlo, bias};
  Fwd::Epi o;
  o.C = y; o.ldc = N; o.act = act; o.res = res; o.ldr = N; o.res_relu = res_relu;
  if (r == PF_OK) {
    if (KH == 3 && stride == 1 && pad == 1 && Cin % 64 == 0) r = F.thalo(A, 0, 0, nullptr, 0, 0, B, H, W, Cin, w, N, 1, 0, o);
    else if (KH == 1 && stride == 1 && pad == 0) r = F.tgemm(A, (long long)B * H * W, Cin, 0, w, N, o);
    else r = F.tconv_gather(A, B, H, W, Cin, KH, stride, pad, w, N, o);
  }
  cudaError_t se = cudaStreamSynchronize(st);
  cudaFree(scratch);
  if (r != PF_OK) return r;
  if (se != cudaSuccess) return fail(PF_ERR_CUDA, "pf_op_conv_gemm: %s", cudaGetErrorString(se));
  return PF_OK;
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
  TRY(configure_current_device());
  int dev = 0;
  CU(cudaGetDevice(&dev));
  cudaDeviceProp prop;
  CU(cudaGetDeviceProperties(&prop, dev));
  pf_engine tmp;
  tmp.device = dev;
  tmp.sm_count = prop.multiProcessorCount;
  tmp.bf16 = bf16;
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
}  // extern "C"

// ParamNet backward pieces, one host helper of bwd_paramnet each: a temporary engine for the current device, scratch sized by a
// dry run of the same body and filled with 0xFF bytes (NaN: a read of memory no kernel wrote poisons the result), a sync at the end.
template <class Body>
static int pn_op_run(const char* name, int n, void* stream, Body body) {
  TRY(configure_current_device());
  pf_engine tmp;
  CU(cudaGetDevice(&tmp.device));
  CU(cudaDeviceGetAttribute(&tmp.sm_count, cudaDevAttrMultiProcessorCount, tmp.device));
  Fwd T{&tmp, Arena{}, nullptr, true, n};
  T.ar.dry = true;
  TRY(body(T));
  const long long bytes = T.ar.peak + 4096;
  cudaStream_t st = (cudaStream_t)stream;
  char* scratch = nullptr;
  CU(cudaMalloc(&scratch, bytes));
  Fwd F{&tmp, Arena{}, st, false, n};
  F.ar.base = scratch; F.ar.cap = bytes;
  const cudaError_t me = cudaMemsetAsync(scratch, 0xFF, bytes, st);
  int r = me == cudaSuccess ? body(F) : fail(PF_ERR_CUDA, "%s: %s", name, cudaGetErrorString(me));
  const cudaError_t se = cudaStreamSynchronize(st);
  cudaFree(scratch);
  if (r == PF_OK && se != cudaSuccess) r = fail(PF_ERR_CUDA, "%s: %s", name, cudaGetErrorString(se));
  return r;
}
static bool al16(const void* p) { return ((uintptr_t)p & 15) == 0; }

extern "C" {

int pf_op_pn_wgrad(const float* dy, int ldy, const float* x, const void* x_hi, const void* x_lo, int op, int ldx, int64_t R, int N, int K, float* out,
                   int* S, int* chunk, void* stream) {
  if (!dy || !out || !S || !chunk) return fail(PF_ERR_ARG, "pf_op_pn_wgrad: null argument");
  if (!x_hi != !x_lo || !x == !x_hi) return fail(PF_ERR_ARG, "pf_op_pn_wgrad: the source is x or the pair x_hi / x_lo");
  if ((op != 0 && op != 1) || (op == 1 && !x)) return fail(PF_ERR_ARG, "pf_op_pn_wgrad: op %d (1, the GELU, needs the fp32 source)", op);
  if (R < 1 || R > INT32_MAX || N < 1 || K < 1 || ldy < N || ldx < K) return fail(PF_ERR_ARG, "pf_op_pn_wgrad: R %lld, N %d, K %d, ldy %d, ldx %d", (long long)R, N, K, ldy, ldx);
  const SplitT xs{(__nv_bfloat16*)x_hi, (__nv_bfloat16*)x_lo, ldx};
  WgPlan pl{};
  const int r = pn_op_run("pf_op_pn_wgrad", 1, stream, [&](Fwd& F) { return pn_wgrad_full(F, dy, ldy, x ? nullptr : &xs, x, op, ldx, R, N, K, out, &pl); });
  *S = pl.S;
  *chunk = pl.chunk;
  return r;
}
int pf_op_pn_colsum(const float* src, int64_t R, int C, float* out, void* stream) {
  if (!src || !out || R < 1 || C < 1) return fail(PF_ERR_ARG, "pf_op_pn_colsum: bad argument");
  return pn_op_run("pf_op_pn_colsum", 1, stream, [&](Fwd& F) { return pn_colsum(F, src, R, C, out); });
}
int pf_op_pn_ln_bwd(const float* x, const float* dy, int64_t R, int C, const float* w, float* dx, float* g, void* stream) {
  if (!x || !dy || !w || !dx || !g) return fail(PF_ERR_ARG, "pf_op_pn_ln_bwd: null argument");
  if (R < 1 || C < 32 || C > 768 || C % 32) return fail(PF_ERR_ARG, "pf_op_pn_ln_bwd: R %lld, C %d (a multiple of 32 up to 768)", (long long)R, C);
  return pn_op_run("pf_op_pn_ln_bwd", 1, stream, [&](Fwd& F) { return pn_ln_bwd(F, x, dy, R, C, w, dx, g); });
}
int pf_op_pn_dw7_bwd(const float* x, const float* dt, int B, int H, int W, int C, const float* w_rot, float* dw, float* dx, int* rows_per_block, void* stream) {
  if (!x || !dt || !w_rot || !dw || !dx) return fail(PF_ERR_ARG, "pf_op_pn_dw7_bwd: null argument");
  if (!al16(x) || !al16(dt) || !al16(w_rot) || !al16(dx)) return fail(PF_ERR_ARG, "pf_op_pn_dw7_bwd: x, dt, w_rot and dx must be 16-byte aligned");
  if (B < 1 || H < 1 || W < 1 || C < 32 || C % 32 || (long long)B * H * W * C > INT32_MAX)
    return fail(PF_ERR_ARG, "pf_op_pn_dw7_bwd: B %d, H %d, W %d, C %d (a multiple of 32)", B, H, W, C);
  return pn_op_run("pf_op_pn_dw7_bwd", B, stream, [&](Fwd& F) {
    float* zero = F.ar.f(C);
    if (!F.dry) CU(cudaMemsetAsync(zero, 0, (size_t)C * 4, F.st));
    TRY(pn_dw7_wgrad(F, x, dt, H, W, C, dw, rows_per_block));
    return pn_dw_launch(F, dt, dx, H, W, C, w_rot, zero);
  });
}
int pf_op_pn_stem_bwd(const float* pin, const float* dS, const float* w, int B, int OH, int OW, float* dw, float* dpin, int* rows_per_block, void* stream) {
  if (!pin || !dS || !w || !dw || !dpin) return fail(PF_ERR_ARG, "pf_op_pn_stem_bwd: null argument");
  if (!al16(pin)) return fail(PF_ERR_ARG, "pf_op_pn_stem_bwd: pin must be 16-byte aligned");
  if (B < 1 || OH < 1 || OW < 1) return fail(PF_ERR_ARG, "pf_op_pn_stem_bwd: B %d, OH %d, OW %d", B, OH, OW);
  return pn_op_run("pf_op_pn_stem_bwd", B, stream, [&](Fwd& F) {
    TRY(pn_stem_wgrad(F, pin, dS, OH, OW, dw, rows_per_block));
    return pn_stem_dgrad(F, dS, w, OH, OW, dpin);
  });
}
int pf_op_pn_fields_grad(const float* dpin, int B, int IH, int IW, int OH, int OW, float* dgrav, float* dlat, void* stream) {
  if (!dpin || !dgrav || !dlat) return fail(PF_ERR_ARG, "pf_op_pn_fields_grad: null argument");
  if (!al16(dpin)) return fail(PF_ERR_ARG, "pf_op_pn_fields_grad: dpin must be 16-byte aligned");
  if (B < 1 || IH < 1 || IW < 1 || OH < 1 || OW < 1) return fail(PF_ERR_ARG, "pf_op_pn_fields_grad: B %d, %dx%d -> %dx%d", B, IH, IW, OH, OW);
  return pn_op_run("pf_op_pn_fields_grad", B, stream, [&](Fwd& F) { return pn_fields_grad(F, dpin, IH, IW, OH, OW, dgrav, dlat); });
}
int pf_op_pn_tail_bwd(const float* feat, int n, int HW, const float* nw, const float* nb, const float* hw, const float* draw, float* dx, float* grads, void* stream) {
  if (!feat || !nw || !nb || !hw || !draw || !dx || !grads) return fail(PF_ERR_ARG, "pf_op_pn_tail_bwd: null argument");
  if (n < 1 || HW < 1) return fail(PF_ERR_ARG, "pf_op_pn_tail_bwd: n %d, HW %d", n, HW);
  return pn_op_run("pf_op_pn_tail_bwd", n, stream, [&](Fwd& F) { return pn_tail_bwd(F, feat, HW, nw, nb, hw, draw, dx, grads); });
}
int pf_op_pn_pw2_grads(const float* G, const float* sdy, int C, int K, const float* gamma, const void* w_hi, const void* w_lo, const float* b, float* dW, float* db,
                       float* dgamma, void* stream) {
  if (!G || !sdy || !gamma || !w_hi || !w_lo || !b || !dW || !db || !dgamma) return fail(PF_ERR_ARG, "pf_op_pn_pw2_grads: null argument");
  if (C < 1 || K < 1) return fail(PF_ERR_ARG, "pf_op_pn_pw2_grads: C %d, K %d", C, K);
  const GemmW w2{(const __nv_bfloat16*)w_hi, (const __nv_bfloat16*)w_lo, b};
  return pn_op_run("pf_op_pn_pw2_grads", 1, stream, [&](Fwd& F) { return pn_pw2_grads(F, G, sdy, C, K, gamma, w2, dW, db, dgamma); });
}
int pf_op_pn_gelu_bwd(const float* dh, float* u, int64_t n, void* hi, void* lo, void* stream) {
  if (!dh || !u || n < 1 || !hi != !lo) return fail(PF_ERR_ARG, "pf_op_pn_gelu_bwd: bad argument");
  return pn_op_run("pf_op_pn_gelu_bwd", 1, stream, [&](Fwd& F) { return pn_gelu_bwd(F, dh, u, n, (__nv_bfloat16*)hi, (__nv_bfloat16*)lo); });
}
int pf_op_pn_scale_split(const float* src, const float* scale, int64_t n, int C, void* hi, void* lo, void* stream) {
  if (!src || !hi || !lo || n < 1 || C < 1 || n % C) return fail(PF_ERR_ARG, "pf_op_pn_scale_split: bad argument");
  const SplitT out{(__nv_bfloat16*)hi, (__nv_bfloat16*)lo, C};
  return pn_op_run("pf_op_pn_scale_split", 1, stream, [&](Fwd& F) { return pn_scale_split(F, src, scale, n, C, out); });
}
int pf_op_pn_col2im2(const float* dP, int B, int H, int W, int C, float* out, void* stream) {
  if (!dP || !out || B < 1 || H < 2 || W < 2 || H % 2 || W % 2 || C < 1) return fail(PF_ERR_ARG, "pf_op_pn_col2im2: bad argument");
  return pn_op_run("pf_op_pn_col2im2", B, stream, [&](Fwd& F) { return pn_col2im2(F, dP, H, W, C, out); });
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

static int upload_table(const ResampleTable& t, int** bounds, int** coeffs) {
  CU(cudaMalloc(bounds, t.bounds.size() * 4));
  CU(cudaMalloc(coeffs, t.coeffs.size() * 4));
  CU(cudaMemcpy(*bounds, t.bounds.data(), t.bounds.size() * 4, cudaMemcpyHostToDevice));
  CU(cudaMemcpy(*coeffs, t.coeffs.data(), t.coeffs.size() * 4, cudaMemcpyHostToDevice));
  return PF_OK;
}
int pf_op_resize_u8(const uint8_t* img, int H, int W, int new_h, int new_w, uint8_t* out, void* stream) {
  if (!img || !out || H < 1 || W < 1 || new_h < 1 || new_w < 1) return fail(PF_ERR_ARG, "pf_op_resize_u8: bad argument");
  cudaStream_t st = (cudaStream_t)stream;
  if (H == new_h && W == new_w) {   // Pillow returns a copy when the size does not change
    CU(cudaMemcpyAsync(out, img, (size_t)H * W * 3, cudaMemcpyDeviceToDevice, st));
    return PF_OK;
  }
  ResampleTable tx = make_resample_table(W, new_w), ty = make_resample_table(H, new_h);
  int *bx = nullptr, *cx = nullptr, *by = nullptr, *cy = nullptr;
  unsigned char* tmp = nullptr;
  int r = upload_table(tx, &bx, &cx);
  if (r == PF_OK) r = upload_table(ty, &by, &cy);
  if (r == PF_OK && cudaMalloc(&tmp, (size_t)H * new_w * 3) != cudaSuccess) r = fail(PF_ERR_CUDA, "pf_op_resize_u8: cudaMalloc");
  if (r == PF_OK) {
    // Pillow runs the horizontal pass first (over the rows the vertical pass needs: all of them here), each pass rounded to uint8
    cudaError_t le = (resize_u8_h_kernel<<<(unsigned)cdivl((long long)H * new_w, 256), 256, 0, st>>>(img, H, W, new_w, bx, cx, tx.ksize, tmp), cudaGetLastError());
    if (le == cudaSuccess) le = (resize_u8_v_kernel<<<(unsigned)cdivl((long long)new_h * new_w, 256), 256, 0, st>>>(tmp, H, new_w, new_h, by, cy, ty.ksize, out), cudaGetLastError());
    g_launches.fetch_add(2, std::memory_order_relaxed);
    if (le == cudaSuccess) le = cudaStreamSynchronize(st);
    if (le != cudaSuccess) r = fail(PF_ERR_CUDA, "pf_op_resize_u8: %s", cudaGetErrorString(le));
  }
  cudaFree(bx); cudaFree(cx); cudaFree(by); cudaFree(cy); cudaFree(tmp);
  return r;
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
  if (!vec || !lat || n < 1 || !height || !width || !gravity_original || !gravity_original_offset || !latitude_original || !latitude_original_offset)
    return fail(PF_ERR_ARG, "pf_op_postprocess: bad argument");
  return pf_op_postprocess_sized(vec, lat, n, kNet, kNet, height, width, gravity_original, gravity_original_offset, latitude_original, latitude_original_offset,
                                 lat_is_sin, stream);
}
int pf_op_postprocess_sized(const float* vec, const float* lat, int n, int net_h, int net_w, const int32_t* height, const int32_t* width, float* gravity_original,
                            const int64_t* gravity_original_offset, float* latitude_original, const int64_t* latitude_original_offset, int lat_is_sin,
                            void* stream) {
  if (!vec || !lat || n < 1 || !height || !width || !gravity_original || !gravity_original_offset || !latitude_original || !latitude_original_offset)
    return fail(PF_ERR_ARG, "pf_op_postprocess: bad argument");
  if (!net_size_ok(net_h, net_w)) return fail(PF_ERR_ARG, "pf_op_postprocess: unsupported working size %dx%d", net_h, net_w);
  TRY(configure_current_device());
  PostImage* d_post = nullptr;
  CU(cudaMalloc(&d_post, n * sizeof(PostImage)));
  int r = launch_postprocess(vec, lat, n, net_h, net_w, height, width, gravity_original_offset, latitude_original_offset, gravity_original, latitude_original,
                             lat_is_sin, d_post, (cudaStream_t)stream);
  cudaError_t se = cudaStreamSynchronize((cudaStream_t)stream);
  cudaFree(d_post);
  if (r == PF_OK && se != cudaSuccess) r = fail(PF_ERR_CUDA, "pf_op_postprocess: %s", cudaGetErrorString(se));
  return r;
}

int pf_op_fill_stream(float* dst, int64_t numel, float value, void* stream) {
  if (!dst || numel < 4 || (numel & 3) || ((uintptr_t)dst & 15)) return fail(PF_ERR_ARG, "pf_op_fill_stream: bad argument");
  LAUNCHED((fill_stream_kernel<<<132 * 16, 256, 0, (cudaStream_t)stream>>>(reinterpret_cast<float4*>(dst), numel / 4, value), cudaGetLastError()));
  return PF_OK;
}
int pf_op_layernorm(const float* x, float* y, int64_t rows, int C, const float* w, const float* b, float eps, void* stream) {
  LAUNCHED(layernorm_launch(x, y, rows, C, w, b, eps, (cudaStream_t)stream));
  return PF_OK;
}
static int op_attention_tc(const float* q, const float* kv, float* out, int B, int N, int C, int heads, void* stream, int np, int nkv = kAmKeys) {
  if (!q || !kv || !out || C != heads * kAmD) return fail(PF_ERR_ARG, "pf_op_attention_tc: head_dim must be 64");
  if (B < 1 || N < 1 || nkv < 1 || nkv > kAmMaxKeys) return fail(PF_ERR_ARG, "pf_op_attention_tc: B %d, N %d, %d keys (1..%d)", B, N, nkv, kAmMaxKeys);
  TRY(configure_current_device());
  cudaStream_t st = (cudaStream_t)stream;
  int dev = 0;
  CU(cudaGetDevice(&dev));
  cudaDeviceProp prop;
  CU(cudaGetDeviceProperties(&prop, dev));
  pf_engine tmp;
  tmp.device = dev;
  tmp.sm_count = prop.multiProcessorCount;
  const long long nq = (long long)B * N * C, nkve = (long long)B * nkv * 2 * C;
  char* scratch = nullptr;
  CU(cudaMalloc(&scratch, (2 * nq + nkve) * 4 + 8192));
  Fwd F{&tmp, Arena{}, st, false, B};
  F.ar.base = scratch; F.ar.cap = (2 * nq + nkve) * 4 + 8192;
  SplitT qs = F.salloc((long long)B * N, C), kvs = F.salloc((long long)B * nkv, 2 * C), as = F.salloc((long long)B * N, C);
  int r = PF_OK;
  cudaError_t le = (split_kernel<<<(unsigned)cdivl(nq, 256), 256, 0, st>>>(q, qs.hi, qs.lo, nq, 0), cudaGetLastError());
  if (le == cudaSuccess) le = (split_kernel<<<(unsigned)cdivl(nkve, 256), 256, 0, st>>>(kv, kvs.hi, kvs.lo, nkve, 0), cudaGetLastError());
  if (le != cudaSuccess) r = fail(PF_ERR_CUDA, "split_kernel: %s", cudaGetErrorString(le));
  if (r == PF_OK) {
    le = attention_mma_launch(nullptr, B, N, C, heads, st, as, qs, kvs, np, nkv);
    if (le != cudaSuccess) r = fail(PF_ERR_CUDA, "attention_mma_launch: %s", cudaGetErrorString(le));
  }
  if (r == PF_OK) {
    le = (merge_split_kernel<<<(unsigned)cdivl(nq, 256), 256, 0, st>>>(as.hi, as.lo, out, nq), cudaGetLastError());
    if (le != cudaSuccess) r = fail(PF_ERR_CUDA, "merge_split_kernel: %s", cudaGetErrorString(le));
  }
  cudaError_t se = cudaStreamSynchronize(st);
  cudaFree(scratch);
  if (r == PF_OK && se != cudaSuccess) r = fail(PF_ERR_CUDA, "pf_op_attention_tc: %s", cudaGetErrorString(se));
  return r;
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
int pf_op_dwconv3x3_gelu(const float* x, float* y, int B, int H, int W, int C, const float* w, const float* bias, void* stream) {
  if (C % 4) return fail(PF_ERR_ARG, "C %% 4");
  LAUNCHED(launch_pdl(dwconv3x3_gelu_kernel, dim3(ew_grid((long long)B * ((H + 1) / 2) * ((W + PF_DW3_PX - 1) / PF_DW3_PX) * (C / 4))), dim3(256), 0, (cudaStream_t)stream, x, y, B, H, W, C, w, bias, nullptr, nullptr));
  return PF_OK;
}
int pf_op_dwconv7x7(const float* x, float* y, int B, int H, int W, int C, const float* w, const float* bias, void* stream) {
  if (C % 4) return fail(PF_ERR_ARG, "C %% 4");
  LAUNCHED(launch_pdl(dwconv7x7_kernel, dim3(ew_grid((long long)B * ((H + 1) / 2) * ((W + PF_DW7_PX - 1) / PF_DW7_PX) * (C / 4))), dim3(256), 0, (cudaStream_t)stream, x, y, B, H, W, C, w, bias));
  return PF_OK;
}
int pf_op_upsample2x(const float* x, float* y, int B, int H, int W, int C, void* stream) {
  if (C % 4) return fail(PF_ERR_ARG, "C %% 4");
  LAUNCHED(launch_pdl(upsample2x_kernel, dim3(ew_grid(upsample2x_threads(B, H, W, C))), dim3(256), 0, (cudaStream_t)stream, x, C, 0, y, C, 0, B, H, W, C, nullptr, nullptr));
  return PF_OK;
}
int pf_op_preprocess(const uint8_t* img, int H, int W, const float* mean3, const float* std3, float* y, void* stream) {
  return pf_op_preprocess_sized(img, H, W, kNet, kNet, mean3, std3, y, stream);
}
int pf_op_preprocess_sized(const uint8_t* img, int H, int W, int net_h, int net_w, const float* mean3, const float* std3, float* y, void* stream) {
  if (!img || !mean3 || !std3 || !y || H < 1 || W < 1) return fail(PF_ERR_ARG, "pf_op_preprocess: bad argument");
  if (!net_size_ok(net_h, net_w)) return fail(PF_ERR_ARG, "pf_op_preprocess: unsupported working size %dx%d", net_h, net_w);
  TRY(configure_current_device());
  // standalone tables (not cached): test entry point only
  ResampleTable tx = make_resample_table(W, net_w), ty = make_resample_table(H, net_h);
  const int max_rows = pre_max_smem_rows(net_w);
  if (ty.ksize + 1 > max_rows) return fail(PF_ERR_ARG, "image too tall");
  int *bx, *cx, *by, *cy;
  PreImage* d;
  CU(cudaMalloc(&bx, tx.bounds.size() * 4)); CU(cudaMalloc(&cx, tx.coeffs.size() * 4));
  CU(cudaMalloc(&by, ty.bounds.size() * 4)); CU(cudaMalloc(&cy, ty.coeffs.size() * 4));
  CU(cudaMalloc(&d, sizeof(PreImage)));
  CU(cudaMemcpy(bx, tx.bounds.data(), tx.bounds.size() * 4, cudaMemcpyHostToDevice));
  CU(cudaMemcpy(cx, tx.coeffs.data(), tx.coeffs.size() * 4, cudaMemcpyHostToDevice));
  CU(cudaMemcpy(by, ty.bounds.data(), ty.bounds.size() * 4, cudaMemcpyHostToDevice));
  CU(cudaMemcpy(cy, ty.coeffs.data(), ty.coeffs.size() * 4, cudaMemcpyHostToDevice));
  PreImage pi{0, H, W, tx.ksize, ty.ksize, bx, cx, by, cy};
  CU(cudaMemcpy(d, &pi, sizeof pi, cudaMemcpyHostToDevice));
  int rows = pre_rows_needed(H, net_h);
  if (rows > max_rows) rows = max_rows;
  const int smem = rows * net_w * 3;
  LAUNCHED((preprocess_kernel<<<dim3(net_h / kPreRows, 1), net_w, smem, (cudaStream_t)stream>>>(img, d, y, mean3[0], mean3[1], mean3[2], std3[0], std3[1], std3[2], rows,
                                                                                                 net_h, net_w),
            cudaGetLastError()));
  CU(cudaStreamSynchronize((cudaStream_t)stream));
  cudaFree(bx); cudaFree(cx); cudaFree(by); cudaFree(cy); cudaFree(d);
  return PF_OK;
}

}  // extern "C"
