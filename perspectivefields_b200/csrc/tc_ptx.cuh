// wgmma / mbarrier PTX wrappers and the shared-memory matrix descriptors of the sm_90a tensor-core kernels
// (gemm_tma.cuh: persistent TMA -> wgmma engine).
//
// Every mbarrier wait is bounded (clock64 watchdog -> __trap) so that a protocol bug aborts the launch instead of
// hanging the device.
#pragma once
#include "common.cuh"

namespace pf {

// Halo tile of the 3x3 / stride 1 / pad 1 convolutions: a CTA owns a 16 x 8 output-pixel tile (128 rows, two wgmma M = 64
// halves of 8 image rows each) and stages the 18 x 10 input halo of one 64-channel chunk once in shared memory (bf16 hi + lo
// planes, 128 B per pixel, SWIZZLE_128B).  The A operand of filter tap (ky, kx) is a SHIFTED VIEW of that pixel array:
//     start address = plane + (ky*10 + kx) * 128 B,   8-row groups (= 8 pixels of one image row) SBO = 10 * 128 B apart
// The swizzle is a function of the absolute shared-memory address on both sides (TMA writes and wgmma reads), so a view that
// starts at any 128 B boundary reads the pattern the TMA wrote with base offset 0 (checked on H100: setting the base offset to
// (start >> 7) & 7 gives wrong halo convolutions).
constexpr int kHtTileH = 16, kHtTileW = 8;                 // output tile (rows x cols) = 128 pixels
constexpr int kHtHaloW = kHtTileW + 2, kHtHaloH = kHtTileH + 2;
constexpr int kHtHaloPix = kHtHaloW * kHtHaloH;            // 180
constexpr int kHtPlaneBytes = 23 * 1024;                   // 180 x 128 B rounded up to a 1024 B multiple

// ------------------------------------------------------------------------------------------- mbarrier
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;\n" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];\n" ::"r"(bar) : "memory");
}
__device__ __forceinline__ uint32_t mbar_try_wait(uint32_t bar, uint32_t parity) {
  uint32_t ok;
  asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}\n"
               : "=r"(ok) : "r"(bar), "r"(parity) : "memory");
  return ok;
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;
  const long long t0 = clock64();
  while (!mbar_try_wait(bar, parity)) {
    if (clock64() - t0 > 4000000000LL) __trap();  // ~2 s: protocol bug, abort instead of hanging the GPU
  }
}
__device__ __forceinline__ void fence_mbar_init() { asm volatile("fence.mbarrier_init.release.cluster;\n" ::: "memory"); }
// named barrier over `count` threads (id 0 is __syncthreads)
__device__ __forceinline__ void named_bar_sync(int id, int count) { asm volatile("bar.sync %0, %1;\n" ::"r"(id), "r"(count) : "memory"); }

// ------------------------------------------------------------------------------------------- wgmma
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;\n" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;\n" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;\n" ::"n"(N) : "memory"); }
// keeps the compiler from moving accesses of accumulator registers across the asynchronous MMAs that own them
template <int R>
__device__ __forceinline__ void fence_regs(float (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// D[64 x N] (+)= A[64 x 16] * B[N x 16]^T, bf16 operands from shared-memory descriptors (both K-major), fp32 accumulators in the
// N / 2 registers d[0 .. N/2) of the issuing warpgroup.  scale_d = 0 overwrites D.  One instruction covers the whole N: the A slice
// is read from shared memory once per product instead of once per 64 columns.  N = 32 .. 256 in steps of 32 (the engine's tile widths).
#define PF_R8(i) "+f"(d[i]), "+f"(d[i + 1]), "+f"(d[i + 2]), "+f"(d[i + 3]), "+f"(d[i + 4]), "+f"(d[i + 5]), "+f"(d[i + 6]), "+f"(d[i + 7])
template <int N> struct Wgmma;
template <> struct Wgmma<32> {
  static __device__ __forceinline__ void mma(float* d, uint64_t adesc, uint64_t bdesc, uint32_t scale_d) {
    asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 {"
      "%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15"
      "}, %16, %17, p, 1, 1, 0, 0;\n\t}\n"
      : PF_R8(0), PF_R8(8)
      : "l"(adesc), "l"(bdesc), "r"(scale_d));
  }
};
template <> struct Wgmma<64> {
  static __device__ __forceinline__ void mma(float* d, uint64_t adesc, uint64_t bdesc, uint32_t scale_d) {
    asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 {"
      "%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31"
      "}, %32, %33, p, 1, 1, 0, 0;\n\t}\n"
      : PF_R8(0), PF_R8(8), PF_R8(16), PF_R8(24)
      : "l"(adesc), "l"(bdesc), "r"(scale_d));
  }
};
template <> struct Wgmma<96> {
  static __device__ __forceinline__ void mma(float* d, uint64_t adesc, uint64_t bdesc, uint32_t scale_d) {
    asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %50, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n96k16.f32.bf16.bf16 {"
      "%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,"
      "%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47"
      "}, %48, %49, p, 1, 1, 0, 0;\n\t}\n"
      : PF_R8(0), PF_R8(8), PF_R8(16), PF_R8(24), PF_R8(32), PF_R8(40)
      : "l"(adesc), "l"(bdesc), "r"(scale_d));
  }
};
template <> struct Wgmma<128> {
  static __device__ __forceinline__ void mma(float* d, uint64_t adesc, uint64_t bdesc, uint32_t scale_d) {
    asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 {"
      "%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,"
      "%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63"
      "}, %64, %65, p, 1, 1, 0, 0;\n\t}\n"
      : PF_R8(0), PF_R8(8), PF_R8(16), PF_R8(24), PF_R8(32), PF_R8(40), PF_R8(48), PF_R8(56)
      : "l"(adesc), "l"(bdesc), "r"(scale_d));
  }
};
template <> struct Wgmma<160> {
  static __device__ __forceinline__ void mma(float* d, uint64_t adesc, uint64_t bdesc, uint32_t scale_d) {
    asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %82, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n160k16.f32.bf16.bf16 {"
      "%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,"
      "%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63,"
      "%64,%65,%66,%67,%68,%69,%70,%71,%72,%73,%74,%75,%76,%77,%78,%79"
      "}, %80, %81, p, 1, 1, 0, 0;\n\t}\n"
      : PF_R8(0), PF_R8(8), PF_R8(16), PF_R8(24), PF_R8(32), PF_R8(40), PF_R8(48), PF_R8(56), PF_R8(64), PF_R8(72)
      : "l"(adesc), "l"(bdesc), "r"(scale_d));
  }
};
template <> struct Wgmma<192> {
  static __device__ __forceinline__ void mma(float* d, uint64_t adesc, uint64_t bdesc, uint32_t scale_d) {
    asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %98, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n192k16.f32.bf16.bf16 {"
      "%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,"
      "%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63,"
      "%64,%65,%66,%67,%68,%69,%70,%71,%72,%73,%74,%75,%76,%77,%78,%79,%80,%81,%82,%83,%84,%85,%86,%87,%88,%89,%90,%91,%92,%93,%94,%95"
      "}, %96, %97, p, 1, 1, 0, 0;\n\t}\n"
      : PF_R8(0), PF_R8(8), PF_R8(16), PF_R8(24), PF_R8(32), PF_R8(40), PF_R8(48), PF_R8(56), PF_R8(64), PF_R8(72), PF_R8(80), PF_R8(88)
      : "l"(adesc), "l"(bdesc), "r"(scale_d));
  }
};
template <> struct Wgmma<224> {
  static __device__ __forceinline__ void mma(float* d, uint64_t adesc, uint64_t bdesc, uint32_t scale_d) {
    asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %114, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n224k16.f32.bf16.bf16 {"
      "%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,"
      "%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63,"
      "%64,%65,%66,%67,%68,%69,%70,%71,%72,%73,%74,%75,%76,%77,%78,%79,%80,%81,%82,%83,%84,%85,%86,%87,%88,%89,%90,%91,%92,%93,%94,%95,"
      "%96,%97,%98,%99,%100,%101,%102,%103,%104,%105,%106,%107,%108,%109,%110,%111"
      "}, %112, %113, p, 1, 1, 0, 0;\n\t}\n"
      : PF_R8(0), PF_R8(8), PF_R8(16), PF_R8(24), PF_R8(32), PF_R8(40), PF_R8(48), PF_R8(56), PF_R8(64), PF_R8(72), PF_R8(80), PF_R8(88), PF_R8(96), PF_R8(104)
      : "l"(adesc), "l"(bdesc), "r"(scale_d));
  }
};
template <> struct Wgmma<256> {
  static __device__ __forceinline__ void mma(float* d, uint64_t adesc, uint64_t bdesc, uint32_t scale_d) {
    asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %130, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n256k16.f32.bf16.bf16 {"
      "%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,"
      "%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63,"
      "%64,%65,%66,%67,%68,%69,%70,%71,%72,%73,%74,%75,%76,%77,%78,%79,%80,%81,%82,%83,%84,%85,%86,%87,%88,%89,%90,%91,%92,%93,%94,%95,"
      "%96,%97,%98,%99,%100,%101,%102,%103,%104,%105,%106,%107,%108,%109,%110,%111,%112,%113,%114,%115,%116,%117,%118,%119,%120,%121,%122,%123,%124,%125,%126,%127"
      "}, %128, %129, p, 1, 1, 0, 0;\n\t}\n"
      : PF_R8(0), PF_R8(8), PF_R8(16), PF_R8(24), PF_R8(32), PF_R8(40), PF_R8(48), PF_R8(56), PF_R8(64), PF_R8(72), PF_R8(80), PF_R8(88), PF_R8(96), PF_R8(104), PF_R8(112), PF_R8(120)
      : "l"(adesc), "l"(bdesc), "r"(scale_d));
  }
};
#undef PF_R8
template <int N>
__device__ __forceinline__ void wgmma_bf16(float* d, uint64_t adesc, uint64_t bdesc, uint32_t scale_d) { Wgmma<N>::mma(d, adesc, bdesc, scale_d); }

// K-major SWIZZLE_128B (kb = 64: 128 B rows, 8-row groups 1024 B apart) or SWIZZLE_64B (kb = 32: 64 B rows, 512 B apart) descriptor
// of a tile that starts on a swizzle-pattern boundary.  Advancing K by 16 elements is +32 B of start address (+2 in the field).
template <int KB>
__device__ __forceinline__ uint64_t wgmma_tile_desc(uint32_t smem_addr) {
  constexpr uint64_t sbo = KB == 32 ? 512 : 1024, layout = KB == 32 ? 2 : 1;
  return (uint64_t)((smem_addr >> 4) & 0x3FFFu) | ((uint64_t)1 << 16) | ((sbo >> 4) << 32) | (layout << 62);
}
// halo view: 128 B rows, SWIZZLE_128B, 8-row groups kHtHaloW * 128 B apart, start anywhere on a 128 B boundary
__device__ __forceinline__ uint64_t ht_a_desc(uint32_t smem_addr) {
  return (uint64_t)((smem_addr >> 4) & 0x3FFFu) | ((uint64_t)1 << 16) | ((uint64_t)((kHtHaloW * 128) >> 4) << 32) |
         ((uint64_t)1 << 62);
}

}  // namespace pf
