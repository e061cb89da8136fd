// ParamNet training (C ABI: include/pf_b200.h): the training forward, the ConvNeXt-T backward into the gradient buffer, and the
// single-operator entry points that run one piece of the backward each.  The only translation unit that compiles
// paramnet_train.cuh.
#include <algorithm>

#include "engine.h"
#include "paramnet_train.cuh"

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

static bool al16(const void* p) { return ((uintptr_t)p & 15) == 0; }

extern "C" {

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

// The pf_op_pn_* entry points: one host helper of bwd_paramnet each, run through op_run.
int pf_op_pn_wgrad(const float* dy, int ldy, const float* x, const void* x_hi, const void* x_lo, int op, int ldx, int64_t R, int N, int K, float* out,
                   int* S, int* chunk, void* stream) {
  if (!dy || !out || !S || !chunk) return fail(PF_ERR_ARG, "pf_op_pn_wgrad: null argument");
  if (!x_hi != !x_lo || !x == !x_hi) return fail(PF_ERR_ARG, "pf_op_pn_wgrad: the source is x or the pair x_hi / x_lo");
  if ((op != 0 && op != 1) || (op == 1 && !x)) return fail(PF_ERR_ARG, "pf_op_pn_wgrad: op %d (1, the GELU, needs the fp32 source)", op);
  if (R < 1 || R > INT32_MAX || N < 1 || K < 1 || ldy < N || ldx < K) return fail(PF_ERR_ARG, "pf_op_pn_wgrad: R %lld, N %d, K %d, ldy %d, ldx %d", (long long)R, N, K, ldy, ldx);
  const SplitT xs{(__nv_bfloat16*)x_hi, (__nv_bfloat16*)x_lo, ldx};
  WgPlan pl{};
  const int r = op_run("pf_op_pn_wgrad", 1, stream, [&](Fwd& F) { return pn_wgrad_full(F, dy, ldy, x ? nullptr : &xs, x, op, ldx, R, N, K, out, &pl); });
  *S = pl.S;
  *chunk = pl.chunk;
  return r;
}
int pf_op_pn_colsum(const float* src, int64_t R, int C, float* out, void* stream) {
  if (!src || !out || R < 1 || C < 1) return fail(PF_ERR_ARG, "pf_op_pn_colsum: bad argument");
  return op_run("pf_op_pn_colsum", 1, stream, [&](Fwd& F) { return pn_colsum(F, src, R, C, out); });
}
int pf_op_pn_ln_bwd(const float* x, const float* dy, int64_t R, int C, const float* w, float* dx, float* g, void* stream) {
  if (!x || !dy || !w || !dx || !g) return fail(PF_ERR_ARG, "pf_op_pn_ln_bwd: null argument");
  if (R < 1 || C < 32 || C > 768 || C % 32) return fail(PF_ERR_ARG, "pf_op_pn_ln_bwd: R %lld, C %d (a multiple of 32 up to 768)", (long long)R, C);
  return op_run("pf_op_pn_ln_bwd", 1, stream, [&](Fwd& F) { return pn_ln_bwd(F, x, dy, R, C, w, dx, g); });
}
int pf_op_pn_dw7_bwd(const float* x, const float* dt, int B, int H, int W, int C, const float* w_rot, float* dw, float* dx, int* rows_per_block, void* stream) {
  if (!x || !dt || !w_rot || !dw || !dx) return fail(PF_ERR_ARG, "pf_op_pn_dw7_bwd: null argument");
  if (!al16(x) || !al16(dt) || !al16(w_rot) || !al16(dx)) return fail(PF_ERR_ARG, "pf_op_pn_dw7_bwd: x, dt, w_rot and dx must be 16-byte aligned");
  if (B < 1 || H < 1 || W < 1 || C < 32 || C % 32 || (long long)B * H * W * C > INT32_MAX)
    return fail(PF_ERR_ARG, "pf_op_pn_dw7_bwd: B %d, H %d, W %d, C %d (a multiple of 32)", B, H, W, C);
  return op_run("pf_op_pn_dw7_bwd", B, stream, [&](Fwd& F) {
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
  return op_run("pf_op_pn_stem_bwd", B, stream, [&](Fwd& F) {
    TRY(pn_stem_wgrad(F, pin, dS, OH, OW, dw, rows_per_block));
    return pn_stem_dgrad(F, dS, w, OH, OW, dpin);
  });
}
int pf_op_pn_fields_grad(const float* dpin, int B, int IH, int IW, int OH, int OW, float* dgrav, float* dlat, void* stream) {
  if (!dpin || !dgrav || !dlat) return fail(PF_ERR_ARG, "pf_op_pn_fields_grad: null argument");
  if (!al16(dpin)) return fail(PF_ERR_ARG, "pf_op_pn_fields_grad: dpin must be 16-byte aligned");
  if (B < 1 || IH < 1 || IW < 1 || OH < 1 || OW < 1) return fail(PF_ERR_ARG, "pf_op_pn_fields_grad: B %d, %dx%d -> %dx%d", B, IH, IW, OH, OW);
  return op_run("pf_op_pn_fields_grad", B, stream, [&](Fwd& F) { return pn_fields_grad(F, dpin, IH, IW, OH, OW, dgrav, dlat); });
}
int pf_op_pn_tail_bwd(const float* feat, int n, int HW, const float* nw, const float* nb, const float* hw, const float* draw, float* dx, float* grads, void* stream) {
  if (!feat || !nw || !nb || !hw || !draw || !dx || !grads) return fail(PF_ERR_ARG, "pf_op_pn_tail_bwd: null argument");
  if (n < 1 || HW < 1) return fail(PF_ERR_ARG, "pf_op_pn_tail_bwd: n %d, HW %d", n, HW);
  return op_run("pf_op_pn_tail_bwd", n, stream, [&](Fwd& F) { return pn_tail_bwd(F, feat, HW, nw, nb, hw, draw, dx, grads); });
}
int pf_op_pn_pw2_grads(const float* G, const float* sdy, int C, int K, const float* gamma, const void* w_hi, const void* w_lo, const float* b, float* dW, float* db,
                       float* dgamma, void* stream) {
  if (!G || !sdy || !gamma || !w_hi || !w_lo || !b || !dW || !db || !dgamma) return fail(PF_ERR_ARG, "pf_op_pn_pw2_grads: null argument");
  if (C < 1 || K < 1) return fail(PF_ERR_ARG, "pf_op_pn_pw2_grads: C %d, K %d", C, K);
  const GemmW w2{(const __nv_bfloat16*)w_hi, (const __nv_bfloat16*)w_lo, b};
  return op_run("pf_op_pn_pw2_grads", 1, stream, [&](Fwd& F) { return pn_pw2_grads(F, G, sdy, C, K, gamma, w2, dW, db, dgamma); });
}
int pf_op_pn_gelu_bwd(const float* dh, float* u, int64_t n, void* hi, void* lo, void* stream) {
  if (!dh || !u || n < 1 || !hi != !lo) return fail(PF_ERR_ARG, "pf_op_pn_gelu_bwd: bad argument");
  return op_run("pf_op_pn_gelu_bwd", 1, stream, [&](Fwd& F) { return pn_gelu_bwd(F, dh, u, n, (__nv_bfloat16*)hi, (__nv_bfloat16*)lo); });
}
int pf_op_pn_scale_split(const float* src, const float* scale, int64_t n, int C, void* hi, void* lo, void* stream) {
  if (!src || !hi || !lo || n < 1 || C < 1 || n % C) return fail(PF_ERR_ARG, "pf_op_pn_scale_split: bad argument");
  const SplitT out{(__nv_bfloat16*)hi, (__nv_bfloat16*)lo, C};
  return op_run("pf_op_pn_scale_split", 1, stream, [&](Fwd& F) { return pn_scale_split(F, src, scale, n, C, out); });
}
int pf_op_pn_col2im2(const float* dP, int B, int H, int W, int C, float* out, void* stream) {
  if (!dP || !out || B < 1 || H < 2 || W < 2 || H % 2 || W % 2 || C < 1) return fail(PF_ERR_ARG, "pf_op_pn_col2im2: bad argument");
  return op_run("pf_op_pn_col2im2", B, stream, [&](Fwd& F) { return pn_col2im2(F, dP, H, W, C, out); });
}

}  // extern "C"
