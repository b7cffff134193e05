// Thin inline-PTX wrappers for the sm_90a features the kernels use:
// mbarrier, TMA (cp.async.bulk.tensor), wgmma (warpgroup MMA with shared-memory descriptors).
// Descriptor bit layouts follow the PTX ISA "Matrix Descriptor Format" table of wgmma.
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

namespace vb {

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

// ------------------------------------------------------------------ mbarrier
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_barrier_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
// Non-blocking probe (mbarrier.test_wait returns at once; try_wait may suspend the thread for a system-dependent time,
// which is wrong for a thread that polls SEVERAL barriers in turn).
__device__ __forceinline__ bool mbar_test_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.test_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
// Bounded wait: a pipeline bug must end in a trap (test failure), never in a hung GPU.  The clock is consulted only every
// 4096 failed probes.  No printf here or in mbar_wait_relaxed: these waits sit in kernels that issue wgmma, and any function
// call in such a kernel (vprintf is one) makes ptxas serialise all of its wgmma instructions (C7510).  `tag` names the
// wait for a reader of the source.
#ifndef VB_WAIT_TIMEOUT_CYCLES
#define VB_WAIT_TIMEOUT_CYCLES (4000000000ll)  // ~2 s at 1.9 GHz
#endif
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity, int tag = 0) {
  (void)tag;
  if (mbar_try_wait(bar, parity)) return;
  long long t0 = 0;
  for (uint32_t spins = 1;; ++spins) {
    if (mbar_try_wait(bar, parity)) return;
    if ((spins & 4095u) == 0u) {
      const long long now = clock64();
      if (t0 == 0) t0 = now;
      if (now - t0 > VB_WAIT_TIMEOUT_CYCLES) __trap();
    }
  }
}
// Same, for waits that are usually long (a producer ahead of its consumers): after a few failed probes the warp sleeps between probes instead of burning the issue slots the epilogue warps need.
__device__ __forceinline__ void mbar_wait_relaxed(uint64_t* bar, uint32_t parity, int tag = 0) {
  (void)tag;
  for (int i = 0; i < 4; ++i)
    if (mbar_try_wait(bar, parity)) return;
  long long t0 = 0;
  for (uint32_t spins = 1;; ++spins) {
    __nanosleep(32);
    if (mbar_try_wait(bar, parity)) return;
    if ((spins & 4095u) == 0u) {
      const long long now = clock64();
      if (t0 == 0) t0 = now;
      if (now - t0 > VB_WAIT_TIMEOUT_CYCLES) __trap();
    }
  }
}

__device__ __forceinline__ void fence_proxy_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}

// ------------------------------------------------------------------ TMA loads (tile mode, mbarrier completion)
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
__device__ __forceinline__ void tma_load_2d(void* dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
__device__ __forceinline__ void tma_load_3d(void* dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
      ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}
__device__ __forceinline__ void tma_load_4d(void* dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1, int c2,
                                            int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
      ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}

// ------------------------------------------------------------------ wgmma
// Shared-memory matrix descriptor (64 bit):
//   [0,14)  start address >> 4      [16,30) leading-dim byte offset >> 4
//   [32,46) stride-dim byte offset >> 4      [49,52) base offset (0: tiles are 1024 B aligned)
//   [62,64) layout: 1 = SWIZZLE_128B
// K-major SW128 tile [rows x 64 fp16] (as TMA writes it with CU_TENSOR_MAP_SWIZZLE_128B): rows 128 B apart, 8-row groups
// 1024 B apart (SBO); a K step of 16 elements advances the start address by 32 B.  MN-major SW128 (V of attention,
// [keys x 64 dims]): the same bytes read transposed; a K step of 16 keys advances the start address by 2048 B.
__device__ __forceinline__ uint64_t make_desc_sw128(uint32_t smem_addr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((smem_addr & 0x3FFFFu) >> 4);
  d |= static_cast<uint64_t>((lbo_bytes >> 4) & 0x3FFFu) << 16;
  d |= static_cast<uint64_t>((sbo_bytes >> 4) & 0x3FFFu) << 32;
  d |= static_cast<uint64_t>(1) << 62;
  return d;
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// register budget of the calling warpgroup (warp-specialised kernels: producers give registers to the MMA warpgroups)
template <int R>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(R)); }
template <int R>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(R)); }
// keeps the compiler from moving accesses of accumulator registers across the asynchronous MMAs that own them
template <int N>
__device__ __forceinline__ void fence_regs(float (&r)[N]) {
#pragma unroll
  for (int i = 0; i < N; ++i) asm volatile("" : "+f"(r[i])::"memory");
}

// D[64 x N] (+)= A[smem desc, 64 x 16] * B[smem desc, 16 x N], both K-major; scale_d = 0 overwrites D; N any multiple
// of 32 up to 256, fp16 or bf16 operands.  Accumulator fragment of thread (warp w, lane l) of the warpgroup:
// d[4 i + e] = D[16 w + l / 4][8 i + 2 (l % 4) + e], d[4 i + 2 + e] = D[16 w + l / 4 + 8][8 i + 2 (l % 4) + e], e in {0, 1}.
// The descriptors and scale_d are operands %0 .. %2 (read-write only so that they precede the accumulators), so the
// accumulator list of every N is %3 .. %(N/2 + 2): a prefix of the 16-register blocks below.
#define VB_R16_0 "%3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18"
#define VB_R16_1 ", %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34"
#define VB_R16_2 ", %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50"
#define VB_R16_3 ", %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66"
#define VB_R16_4 ", %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, %80, %81, %82"
#define VB_R16_5 ", %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, %96, %97, %98"
#define VB_R16_6 ", %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, %112, %113, %114"
#define VB_R16_7 ", %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127, %128, %129, %130"
#define VB_D16(b)                                                                                                      \
  "+f"(d[b + 0]), "+f"(d[b + 1]), "+f"(d[b + 2]), "+f"(d[b + 3]), "+f"(d[b + 4]), "+f"(d[b + 5]), "+f"(d[b + 6]),      \
      "+f"(d[b + 7]), "+f"(d[b + 8]), "+f"(d[b + 9]), "+f"(d[b + 10]), "+f"(d[b + 11]), "+f"(d[b + 12]),               \
      "+f"(d[b + 13]), "+f"(d[b + 14]), "+f"(d[b + 15])
#define VB_WGMMA_SS(N, T, REGS, ...)                                                                                   \
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %2, 0;\n\t"                                                      \
               "wgmma.mma_async.sync.aligned.m64n" #N "k16.f32." T "." T " {" REGS "}, %0, %1, p, 1, 1, 0, 0;\n\t}" \
               : "+l"(da), "+l"(db), "+r"(scale_d), __VA_ARGS__)
#define VB_WGMMA_SS_T(N, REGS, ...)                                                                                    \
  do {                                                                                                                 \
    if constexpr (BF16) VB_WGMMA_SS(N, "bf16", REGS, __VA_ARGS__);                                                     \
    else VB_WGMMA_SS(N, "f16", REGS, __VA_ARGS__);                                                                     \
  } while (0)
template <int N, bool BF16>
__device__ __forceinline__ void wgmma_ss(float (&d)[N / 2], uint64_t da, uint64_t db, int scale_d) {
  static_assert(N >= 32 && N <= 256 && N % 32 == 0, "wgmma_ss: N must be a multiple of 32 in [32, 256]");
  if constexpr (N == 32) VB_WGMMA_SS_T(32, VB_R16_0, VB_D16(0));
  else if constexpr (N == 64) VB_WGMMA_SS_T(64, VB_R16_0 VB_R16_1, VB_D16(0), VB_D16(16));
  else if constexpr (N == 96) VB_WGMMA_SS_T(96, VB_R16_0 VB_R16_1 VB_R16_2, VB_D16(0), VB_D16(16), VB_D16(32));
  else if constexpr (N == 128)
    VB_WGMMA_SS_T(128, VB_R16_0 VB_R16_1 VB_R16_2 VB_R16_3, VB_D16(0), VB_D16(16), VB_D16(32), VB_D16(48));
  else if constexpr (N == 160)
    VB_WGMMA_SS_T(160, VB_R16_0 VB_R16_1 VB_R16_2 VB_R16_3 VB_R16_4, VB_D16(0), VB_D16(16), VB_D16(32), VB_D16(48),
                  VB_D16(64));
  else if constexpr (N == 192)
    VB_WGMMA_SS_T(192, VB_R16_0 VB_R16_1 VB_R16_2 VB_R16_3 VB_R16_4 VB_R16_5, VB_D16(0), VB_D16(16), VB_D16(32),
                  VB_D16(48), VB_D16(64), VB_D16(80));
  else if constexpr (N == 224)
    VB_WGMMA_SS_T(224, VB_R16_0 VB_R16_1 VB_R16_2 VB_R16_3 VB_R16_4 VB_R16_5 VB_R16_6, VB_D16(0), VB_D16(16),
                  VB_D16(32), VB_D16(48), VB_D16(64), VB_D16(80), VB_D16(96));
  else
    VB_WGMMA_SS_T(256, VB_R16_0 VB_R16_1 VB_R16_2 VB_R16_3 VB_R16_4 VB_R16_5 VB_R16_6 VB_R16_7, VB_D16(0), VB_D16(16),
                  VB_D16(32), VB_D16(48), VB_D16(64), VB_D16(80), VB_D16(96), VB_D16(112));
}
#undef VB_WGMMA_SS_T
#undef VB_WGMMA_SS
#undef VB_D16
#undef VB_R16_0
#undef VB_R16_1
#undef VB_R16_2
#undef VB_R16_3
#undef VB_R16_4
#undef VB_R16_5
#undef VB_R16_6
#undef VB_R16_7

__device__ __forceinline__ void wgmma_m64n128_f16(float (&d)[64], uint64_t da, uint64_t db, int scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
      "%64, %65, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(da), "l"(db), "r"(scale_d));
}

// The register-A form (A = 64 x 16 fp16 in the mma.m16n8k16 A layout: a[0] = rows l/4, k 2(l%4) + {0,1}; a[1] = rows
// l/4 + 8; a[2], a[3] = the same at k + 8) with B MN-major (transposed).
__device__ __forceinline__ void wgmma_m64n64_f16_rs_tb(float (&d)[32], const uint32_t (&a)[4], uint64_t db, int scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %37, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, "
      "{%32, %33, %34, %35}, %36, p, 1, 1, 1;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db), "r"(scale_d));
}

// ------------------------------------------------------------------ misc math
// x * sigmoid(x) with two MUFU operations (ex2, rcp) and no IEEE division sequence; relative error ~2^-22, far below
// the fp16 rounding of every tensor this is stored to
__device__ __forceinline__ float silu_f(float x) {
  float e, r;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(x * -1.4426950408889634f));
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(1.0f + e));
  return x * r;
}
__device__ __forceinline__ float gelu_erf_f(float x) { return 0.5f * x * (1.0f + erff(x * 0.70710678118654752f)); }
// erf-GELU via Abramowitz-Stegun 7.1.26 (|erf error| <= 1.5e-7; measured |gelu error| <= 4.3e-7, below the
// fp16 rounding of the output): erfc(a) = poly(t) * exp(-a^2), t = 1/(1 + p a), a = |x|/sqrt(2).
// gelu(x) = x<0 ? h*erfc : x - h*erfc with h = x/2.  2 MUFU + ~13 FMA-pipe operations.
__device__ __forceinline__ float gelu_erf_fast(float x) {
  const float ax = fabsf(x) * 0.70710678118654752f;
  float t;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(t) : "f"(fmaf(0.3275911f, ax, 1.0f)));
  float poly = fmaf(t, 1.061405429f, -1.453152027f);
  poly = fmaf(t, poly, 1.421413741f);
  poly = fmaf(t, poly, -0.284496736f);
  poly = fmaf(t, poly, 0.254829592f);
  float e;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(ax * (ax * -1.4426950408889634f)));
  const float r = (0.5f * x) * ((poly * t) * e);   // h * erfc(|x|/sqrt2)
  return x < 0.0f ? r : x - r;
}
// value * gelu(gate) with the constants of gelu_erf_fast folded (sqrt(1/2) into p, 1/2 into the polynomial):
// 13 FMA-pipe operations + 2 MUFU per element.
__device__ __forceinline__ float geglu_fast(float v, float x) {
  float t;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(t) : "f"(fmaf(fabsf(x), 0.23164190f, 1.0f)));
  float poly = fmaf(t, 0.5307027145f, -0.7265760135f);
  poly = fmaf(t, poly, 0.7107068705f);
  poly = fmaf(t, poly, -0.142248368f);
  poly = fmaf(t, poly, 0.127414796f);
  float e;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"((x * -0.72134752044f) * x));
  const float w = (poly * t) * e;          // erfc(|x|/sqrt2) / 2
  const float vx = v * x;
  const float r = vx * w;
  return x < 0.0f ? r : vx - r;
}
__device__ __forceinline__ float ex2_f(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

}  // namespace vb
