// Common device helpers for the sm_90a kernels of the PerspectiveFields inference path.
#pragma once
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace pf {

constexpr int kNet = 320;  // network working resolution (every shipped config: DATALOADER.RESIZE = [320, 320])

__host__ __device__ inline int cdiv(int a, int b) { return (a + b - 1) / b; }
__host__ __device__ inline long long cdivl(long long a, long long b) { return (a + b - 1) / b; }

// grid of a 256-thread grid-stride launch over `total` items
inline unsigned ew_grid(long long total) {
  long long g = cdivl(total, 256);
  const long long cap = 132LL * 32;
  return (unsigned)(g < cap ? (g > 0 ? g : 1) : cap);
}

// Bin widths in degrees of the gravity (NC - 1 angle bins plus the "no direction" bin NC - 1) and latitude classes, shared by
// the decoders of layers.cuh and the encoders of metrics.cuh (utils/utils.py:94-162).
__host__ __device__ __forceinline__ float gravity_bin_deg(int NC) { return 360.0f / (float)(NC - 1); }
__host__ __device__ __forceinline__ float latitude_bin_deg(int NC) { return 180.0f / (float)NC; }

// ---------------------------------------------------------------- programmatic dependent launch (PDL)
// The forward graph is ~450 dependent launches of 10-60 us kernels.  Kernels launched with
// cudaLaunchAttributeProgrammaticStreamSerialization may begin (block scheduling, prologue: barrier init,
// descriptor prefetch) while the previous kernel of the stream is still draining; pdl_wait() (griddepcontrol.wait) then blocks
// until that kernel has completed and its memory is visible -- every kernel launched that way calls it before its first global
// access.  It is a no-op for ordinary launches.  pdl_launch() lets the NEXT kernel's launch proceed as early as possible.
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_launch() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

inline bool& pdl_enabled() {   // set per pf_forward call from the engine option "pdl"
  static thread_local bool on = false;
  return on;
}
template <class... KArgs, class... Args>
inline cudaError_t launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args&&... args) {
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = st;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  at[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = at;
  cfg.numAttrs = pdl_enabled() ? 1 : 0;
  return cudaLaunchKernelEx(&cfg, kernel, KArgs(args)...);
}

// ---------------------------------------------------------------- bf16 hi/lo split of an fp32 value
// x ~= hi + lo with hi = bf16(x), lo = bf16(x - hi): 16 significant bits.  A product a*b is then
// evaluated on the tensor cores as a_hi*b_hi + a_lo*b_hi + a_hi*b_lo (fp32 accumulate), relative error
// ~2^-17 per product instead of 2^-9 (bf16) or 2^-11 (tf32).  See DESIGN.md "precision".
__device__ __forceinline__ void split_bf16x2(float a, float b, uint32_t& hi, uint32_t& lo) {
  __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
  float2 hf = __bfloat1622float2(h);
  __nv_bfloat162 l = __floats2bfloat162_rn(a - hf.x, b - hf.y);
  hi = *reinterpret_cast<uint32_t*>(&h);
  lo = *reinterpret_cast<uint32_t*>(&l);
}

// A "split tensor": the two bf16 planes of an fp32 activation tensor, NHWC with `ld` channels per pixel.  GEMM inputs are
// always stored this way by their producer so that the wgmma kernels can TMA-load them without any conversion.
struct SplitT {
  __nv_bfloat16* hi = nullptr;
  __nv_bfloat16* lo = nullptr;
  int ld = 0;
};
__device__ __forceinline__ void store_split1(__nv_bfloat16* hi, __nv_bfloat16* lo, long long idx, float v) {
  const __nv_bfloat16 h = __float2bfloat16_rn(v);
  hi[idx] = h;
  lo[idx] = __float2bfloat16_rn(v - __bfloat162float(h));
}

// ---------------------------------------------------------------- async copy / ldmatrix / mma wrappers
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src, bool valid) {
  int sz = valid ? 16 : 0;  // src-size 0 -> zero fill
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;\n" ::"r"(dst), "l"(src), "r"(sz));
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;\n" ::"n"(N)); }

__device__ __forceinline__ void ldmatrix_x4(uint32_t addr, uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];\n"
               : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3) : "r"(addr));
}

// D(16x8,f32) += A(16x16,bf16,row) * B(16x8,bf16,col)
__device__ __forceinline__ void mma_bf16_16816(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

// exact-erf GELU (nn.GELU default; mix_transformers.py:20, convnext.py:52):  0.5 x (1 + erf(x / sqrt 2)).
// erf(z) = sign(z) (1 - erfc|z|) with erfc|z| = 2^q(|z|): q = degree-8 polynomial fitted (weighted minimax, float64) to
// log2 erfc on [0, 4.2] (erfc(4.2) = 3e-9: clamped beyond), evaluated by Horner FMAs + ONE ex2 -- 14 instructions against ~45
// (and two MUFU operations) for libm's branch-free erff.  GELU error over all x: 4.4e-7 absolute, 1.1e-7 relative to max(|x|, 1)
// -- the same as the fp32 rounding of the erff route (both checked against scipy in float64; tests/test_host_logic.py repeats
// the check on the coefficients below).  PF_GELU_LIBM selects erff.
__device__ __forceinline__ float gelu_erf(float x) {
#ifdef PF_GELU_LIBM
  return 0.5f * x * (1.0f + erff(x * 0.70710678118654752440f));
#else
  const float z = fminf(fabsf(x) * 0.70710678118654752440f, 4.2f);
  float q = -3.6446916055865586e-05f;
  q = fmaf(q, z, 0.00037918094312772155f);
  q = fmaf(q, z, -0.0012955267447978258f);
  q = fmaf(q, z, -0.0010598527733236551f);
  q = fmaf(q, z, 0.028478290885686874f);
  q = fmaf(q, z, -0.14857476949691772f);
  q = fmaf(q, z, -0.9183977246284485f);
  q = fmaf(q, z, -1.6279100179672241f);
  q = fmaf(q, z, -0.99999997195662971f);                        // (2.8043370292607506e-08 - 1): ex2 below returns erfc / 2
  float h;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(h) : "f"(q));       // erfc(|x| / sqrt 2) / 2
  return fmaf(x, 0.5f, fabsf(x) * (0.5f - h));                  // x/2 + |x| erf(|x| / sqrt 2) / 2
#endif
}

// 2^x on the special-function unit (2 ulp; results below 2^-126 flush to zero -- softmax weights that small do not matter)
__device__ __forceinline__ float ex2_approx(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

}  // namespace pf
