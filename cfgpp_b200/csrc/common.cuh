// cfgpp_b200 — shared device-side PTX wrappers for sm_90a (wgmma / mma.sync / TMA / mbarrier).
// Everything here is raw inline PTX; no CUTLASS/CuTe dependency.
#pragma once
#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

namespace cfgpp {

#define CFGPP_DEVICE __device__ __forceinline__

CFGPP_DEVICE uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

// ----------------------------------------------------------------------------------------------
// programmatic dependent launch (PDL): every kernel of the step is launched with the programmatic-stream-
// serialization attribute. pdl_launch_dependents() lets the next kernel's CTAs start (and run their prologue:
// barrier init, descriptor prefetch) as soon as SM resources free up; pdl_wait() blocks until the
// preceding kernel has fully completed and its writes are visible — it must precede the first global access.
// ----------------------------------------------------------------------------------------------
CFGPP_DEVICE void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
CFGPP_DEVICE void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

// ----------------------------------------------------------------------------------------------
// mbarrier
// ----------------------------------------------------------------------------------------------
CFGPP_DEVICE void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
CFGPP_DEVICE void fence_barrier_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
CFGPP_DEVICE void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
               : "memory");
}
CFGPP_DEVICE void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
// Non-blocking probe (used by polling state machines): returns after the default, short, hardware time-out.
CFGPP_DEVICE uint32_t mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t"
      ".reg .pred P1;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 P1, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, P1;\n\t"
      "}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok;
}
#ifndef CFGPP_MBAR_SLEEP_NS
#define CFGPP_MBAR_SLEEP_NS 1000000
#endif
// Probe with a suspend-time hint: the thread may sleep in hardware for up to ~1 ms waiting for the phase, instead
// of spinning through the issue stage (a consumer may wait for a whole main loop of TMA loads).
CFGPP_DEVICE uint32_t mbar_try_wait_sleep(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t"
      ".reg .pred P1;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 P1, [%1], %2, %3;\n\t"
      "selp.u32 %0, 1, 0, P1;\n\t"
      "}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity), "r"(CFGPP_MBAR_SLEEP_NS)
      : "memory");
  return ok;
}
// Wait for the phase with the given parity to complete. A wait that lasts > ~2 s of SM clocks can only be
// a pipeline bug; trap (surfaces as a launch failure) instead of hanging the GPU.
CFGPP_DEVICE void mbar_wait(uint64_t* bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;
  const long long t0 = clock64();
#if CFGPP_MBAR_SLEEP_NS > 0
  while (!mbar_try_wait_sleep(bar, parity)) {
#else
  while (!mbar_try_wait(bar, parity)) {
#endif
    if (clock64() - t0 > 4000000000LL) {
      printf("cfgpp: mbarrier wait timeout (block %d thread %d bar 0x%x parity %u)\n", blockIdx.x, threadIdx.x,
             smem_u32(bar), parity);
      __trap();
    }
  }
}

// The same wait with the same time-out, but trapping without the printf report: any function call (printf) in a kernel
// that issues wgmma makes ptxas serialise every wgmma of that kernel.
CFGPP_DEVICE void mbar_wait_nocall(uint64_t* bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;
  const long long t0 = clock64();
  while (!mbar_try_wait(bar, parity)) {
    if (clock64() - t0 > 4000000000LL) __trap();
  }
}

// ----------------------------------------------------------------------------------------------
// TMA (cp.async.bulk.tensor) loads, completion on an mbarrier
// ----------------------------------------------------------------------------------------------
CFGPP_DEVICE void tma_prefetch_desc(const CUtensorMap* map) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(map)) : "memory");
}
CFGPP_DEVICE void tma_load_2d(void* smem_dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
CFGPP_DEVICE void tma_load_3d(void* smem_dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
      ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c0), "r"(c1),
      "r"(c2)
      : "memory");
}
CFGPP_DEVICE void tma_load_4d(void* smem_dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1, int c2,
                              int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], "
      "[%2];" ::"r"(smem_u32(smem_dst)),
      "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}
// im2col load through a rank-4 im2col map (host.h make_tmap_im2col_f16): the pixel walk starts at box coordinate
// (w, h) of image n, channels [c, c + channels_per_pixel); every pixel read is shifted by (off_w, off_h).
CFGPP_DEVICE void tma_load_im2col_4d(void* smem_dst, const CUtensorMap* map, uint64_t* bar, int c, int w, int h, int n,
                                     uint16_t off_w, uint16_t off_h) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.im2col.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], "
      "[%2], {%7, %8};" ::"r"(smem_u32(smem_dst)),
      "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c), "r"(w), "r"(h), "r"(n), "h"(off_w), "h"(off_h)
      : "memory");
}

// TMA store smem -> global (bulk async-group completion)
CFGPP_DEVICE void tma_store_2d(const CUtensorMap* map, const void* smem_src, int c0, int c1) {
  asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];" ::"l"(
                   reinterpret_cast<uint64_t>(map)),
               "r"(smem_u32(smem_src)), "r"(c0), "r"(c1)
               : "memory");
}
CFGPP_DEVICE void tma_store_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
CFGPP_DEVICE void tma_store_wait_read0() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
CFGPP_DEVICE void tma_store_wait0() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }
CFGPP_DEVICE void named_bar_sync(int id, int nthreads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}
CFGPP_DEVICE void named_bar_arrive(int id, int nthreads) {
  asm volatile("bar.arrive %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}

// generic-proxy smem writes -> visible to the async proxy (wgmma / TMA reads)
CFGPP_DEVICE void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// ----------------------------------------------------------------------------------------------
// warpgroup register reallocation (setmaxnreg): the producer warpgroup gives registers back so the two MMA / epilogue
// warpgroups can hold a 64 x 256 fp32 accumulator each. Executed by all warps of a warpgroup.
// ----------------------------------------------------------------------------------------------
template <uint32_t N>
CFGPP_DEVICE void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(N)); }
template <uint32_t N>
CFGPP_DEVICE void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(N)); }

// ----------------------------------------------------------------------------------------------
// wgmma (sm_90a warpgroup MMA): D[64 x N] (+)= A[64 x 16] * B[N x 16]^T, fp16 in, fp32 accumulate in registers.
// Both operands come from shared memory through matrix descriptors (K-major, 128B swizzle).
// ----------------------------------------------------------------------------------------------
CFGPP_DEVICE void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
CFGPP_DEVICE void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
CFGPP_DEVICE void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from moving accumulator reads / writes across the asynchronous wgmma window
template <int N>
CFGPP_DEVICE void fence_acc(float (&d)[N]) {
#pragma unroll
  for (int i = 0; i < N; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
// the same for A fragments a register-A wgmma reads: they stay live (unreused) until the wait that retires it
template <int N>
CFGPP_DEVICE void fence_acc(uint32_t (&a)[N]) {
#pragma unroll
  for (int i = 0; i < N; ++i) asm volatile("" : "+r"(a[i])::"memory");
}

// Shared-memory matrix descriptor (sm_90 wgmma), 128B swizzle, K-major operand whose K extent per tile row is exactly
// one 128-byte swizzle atom (64 fp16). Rows are 128 B apart; 8-row groups are 1024 B apart (SBO).
//   bits [0,14)  start address >> 4        bits [16,30) leading byte offset >> 4 (unused for swizzled K-major: 1)
//   bits [32,46) stride byte offset >> 4   bits [62,64) layout type: 1 = SWIZZLE_128B
// Advancing 16 fp16 (32 B) along K inside the atom is +2 in the start-address field.
CFGPP_DEVICE uint64_t make_wgmma_desc_sw128(uint32_t smem_addr) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((smem_addr >> 4) & 0x3FFF);
  d |= static_cast<uint64_t>(1) << 16;
  d |= static_cast<uint64_t>(1024 >> 4) << 32;
  d |= static_cast<uint64_t>(1) << 62;
  return d;
}

// D[64 x N] (+)= A * B^T from two smem descriptors; scale_d = 0 overwrites D. One instruction per N (inline asm needs
// literal operand lists), for the tile widths the GEMM instantiates.
#define CFGPP_D8(i) "+f"(d[i]), "+f"(d[i + 1]), "+f"(d[i + 2]), "+f"(d[i + 3]), "+f"(d[i + 4]), "+f"(d[i + 5]), \
                    "+f"(d[i + 6]), "+f"(d[i + 7])
template <int N>
CFGPP_DEVICE void wgmma_f16(float (&d)[N / 2], uint64_t a_desc, uint64_t b_desc, uint32_t scale_d);
template <>
CFGPP_DEVICE void wgmma_f16<64>(float (&d)[32], uint64_t a_desc, uint64_t b_desc, uint32_t scale_d) {
  asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %34, 0;\nwgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 {"
               "%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,"
               "%27,%28,%29,%30,%31"
               "}, %32, %33, p, 1, 1, 0, 0;\n}\n"
               : CFGPP_D8(0), CFGPP_D8(8), CFGPP_D8(16), CFGPP_D8(24)
               : "l"(a_desc), "l"(b_desc), "r"(scale_d)
               : "memory");
}
template <>
CFGPP_DEVICE void wgmma_f16<128>(float (&d)[64], uint64_t a_desc, uint64_t b_desc, uint32_t scale_d) {
  asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %66, 0;\nwgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 {"
               "%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,"
               "%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,"
               "%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63"
               "}, %64, %65, p, 1, 1, 0, 0;\n}\n"
               : CFGPP_D8(0), CFGPP_D8(8), CFGPP_D8(16), CFGPP_D8(24), CFGPP_D8(32), CFGPP_D8(40), CFGPP_D8(48), CFGPP_D8(56)
               : "l"(a_desc), "l"(b_desc), "r"(scale_d)
               : "memory");
}
template <>
CFGPP_DEVICE void wgmma_f16<160>(float (&d)[80], uint64_t a_desc, uint64_t b_desc, uint32_t scale_d) {
  asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %82, 0;\nwgmma.mma_async.sync.aligned.m64n160k16.f32.f16.f16 {"
               "%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,"
               "%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,"
               "%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63,%64,%65,%66,%67,%68,%69,%70,%71,%72,%73,%74,%75,%76,"
               "%77,%78,%79"
               "}, %80, %81, p, 1, 1, 0, 0;\n}\n"
               : CFGPP_D8(0), CFGPP_D8(8), CFGPP_D8(16), CFGPP_D8(24), CFGPP_D8(32), CFGPP_D8(40), CFGPP_D8(48), CFGPP_D8(56), CFGPP_D8(64), CFGPP_D8(72)
               : "l"(a_desc), "l"(b_desc), "r"(scale_d)
               : "memory");
}
template <>
CFGPP_DEVICE void wgmma_f16<256>(float (&d)[128], uint64_t a_desc, uint64_t b_desc, uint32_t scale_d) {
  asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %130, 0;\nwgmma.mma_async.sync.aligned.m64n256k16.f32.f16.f16 {"
               "%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,"
               "%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,"
               "%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63,%64,%65,%66,%67,%68,%69,%70,%71,%72,%73,%74,%75,%76,"
               "%77,%78,%79,%80,%81,%82,%83,%84,%85,%86,%87,%88,%89,%90,%91,%92,%93,%94,%95,%96,%97,%98,%99,%100,"
               "%101,%102,%103,%104,%105,%106,%107,%108,%109,%110,%111,%112,%113,%114,%115,%116,%117,%118,%119,%120,"
               "%121,%122,%123,%124,%125,%126,%127"
               "}, %128, %129, p, 1, 1, 0, 0;\n}\n"
               : CFGPP_D8(0), CFGPP_D8(8), CFGPP_D8(16), CFGPP_D8(24), CFGPP_D8(32), CFGPP_D8(40), CFGPP_D8(48), CFGPP_D8(56), CFGPP_D8(64), CFGPP_D8(72), CFGPP_D8(80), CFGPP_D8(88), CFGPP_D8(96), CFGPP_D8(104), CFGPP_D8(112), CFGPP_D8(120)
               : "l"(a_desc), "l"(b_desc), "r"(scale_d)
               : "memory");
}

// MN-major 128B-swizzle descriptor: the operand's rows run along K, each row holding 64 fp16 of N contiguously (a
// [K rows x 64] tile as TMA writes it with SWIZZLE_128B, e.g. V for O += P V). 8-row K groups are 1024 B apart. The N
// extent of one row is the whole swizzle atom, so the stride between atoms along N is never applied; both offset fields
// carry the 1024 B group stride. Advancing 16 rows along K (2048 B) is +128 in the start-address field.
CFGPP_DEVICE uint64_t make_wgmma_desc_sw128_mn(uint32_t smem_addr) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((smem_addr >> 4) & 0x3FFF);
  d |= static_cast<uint64_t>(1024 >> 4) << 16;
  d |= static_cast<uint64_t>(1024 >> 4) << 32;
  d |= static_cast<uint64_t>(1) << 62;
  return d;
}

// D[64 x 64] += A[64 x 16] * B[16 x 64], A from registers (the m16n8k16 A fragment of each warp's 16 rows: a[0] / a[1]
// rows r / r + 8 at columns 2 (lane % 4) + {0, 1}, a[2] / a[3] the same rows 8 columns on), B an MN-major smem
// descriptor (imm-trans-b = 1).
CFGPP_DEVICE void wgmma_f16_rs_tb64(float (&d)[32], const uint32_t (&a)[4], uint64_t b_desc, uint32_t scale_d) {
  asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %37, 0;\nwgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 {"
               "%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,"
               "%27,%28,%29,%30,%31"
               "}, {%32,%33,%34,%35}, %36, p, 1, 1, 1;\n}\n"
               : CFGPP_D8(0), CFGPP_D8(8), CFGPP_D8(16), CFGPP_D8(24)
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b_desc), "r"(scale_d)
               : "memory");
}
#undef CFGPP_D8

// ----------------------------------------------------------------------------------------------
// warp-level tensor-core MMA (mma.sync m16n8k16) and ldmatrix, used by the attention kernel
// ----------------------------------------------------------------------------------------------
CFGPP_DEVICE void ldmatrix_x4(uint32_t addr, uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];"
               : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3)
               : "r"(addr));
}
CFGPP_DEVICE void ldmatrix_x4_trans(uint32_t addr, uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0, %1, %2, %3}, [%4];"
               : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3)
               : "r"(addr));
}
// D (fp32, 16 x 8) += A (fp16, 16 x 16, row) * B (fp16, 16 x 8, col)
CFGPP_DEVICE void mma_16816(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, "
      "{%0, %1, %2, %3};"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

// ----------------------------------------------------------------------------------------------
// misc math
// ----------------------------------------------------------------------------------------------
CFGPP_DEVICE unsigned long long globaltimer_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}

// SiLU with the fast divide (<= 2 ulp in fp32; the result is rounded to fp16 by every caller)
CFGPP_DEVICE float silu_f(float x) { return __fdividef(x, 1.0f + __expf(-x)); }
CFGPP_DEVICE float gelu_erf_f(float x) { return 0.5f * x * (1.0f + erff(x * 0.70710678118654752440f)); }
// Exact (erf) GELU through Abramowitz-Stegun 7.1.26: erf(z) = 1 - (a1 t + .. + a5 t^5) exp(-z^2), t = 1/(1 + p z), z >= 0.
// |error| <= 4.2e-7 absolute on the GELU value over [-8, 8] in fp32 (rel-L2 8e-8 on N(0, 1.5) inputs; libdevice erff
// itself is ~1e-7), three orders below the fp16 rounding every caller applies to the result. For x < 0 the form
// 1 + erf(z) = q avoids the cancellation. 14 instructions (two MUFU) instead of the 27 of erff with its range selects:
// the GEGLU epilogue is issue bound on this function.
CFGPP_DEVICE float gelu_erf_fast_f(float x) {
  const float az = fabsf(x) * 0.70710678118654752440f;
  const float t = __fdividef(1.0f, fmaf(0.3275911f, az, 1.0f));
  float e;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(-az * az * 1.4426950408889634f));
  float p = 1.061405429f;
  p = fmaf(p, t, -1.453152027f);
  p = fmaf(p, t, 1.421413741f);
  p = fmaf(p, t, -0.284496736f);
  p = fmaf(p, t, 0.254829592f);
  const float q = p * t * e;
  return 0.5f * x * (x >= 0.f ? 2.0f - q : q);
}

CFGPP_DEVICE float fast_exp2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

CFGPP_DEVICE uint32_t pack_half2(float a, float b) {
  __half2 h = __floats2half2_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&h);
}

}  // namespace cfgpp
