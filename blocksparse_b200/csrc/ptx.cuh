// Thin inline-PTX wrappers for the Hopper (sm_90a) features the tensor-core kernels use:
// mbarrier, TMA (cp.async.bulk.tensor) and warpgroup MMA (wgmma.mma_async) with its shared-memory
// matrix descriptor.  No CUTLASS: bit layouts follow the PTX ISA ("Matrix Descriptor Format" of the
// asynchronous warpgroup-level matrix instructions).
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace ptx {

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

// ---- mbarrier -------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_mbar_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}\n"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
// Bounded wait: a barrier that does not flip within g_wait_timeout_ns of wall clock (default 2 s, host-settable
// through bsmm_set_wait_timeout_ms) is a protocol bug or a starved kernel.  The first wait that gives up records
// code 100 in g_wait_error and -- unless trapping is disabled -- executes `trap`, so that the launch FAILS (the
// next CUDA call of the host returns a fault) instead of completing with partially written outputs.
__device__ unsigned long long g_wait_timeout_ns = 2000000000ull;
__device__ int g_wait_trap = 1;
__device__ int g_wait_error = 0;
__device__ __noinline__ void wait_timed_out() {
  g_wait_error = 100;
  __threadfence_system();
  if (g_wait_trap) asm volatile("trap;");
}
__device__ __forceinline__ uint64_t globaltimer_ns() {
  uint64_t t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}
__device__ __forceinline__ bool mbar_wait(uint64_t* bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return true;
  const uint64_t t0 = globaltimer_ns();
  for (;;) {
#pragma unroll 1
    for (int i = 0; i < 64; ++i)
      if (mbar_try_wait(bar, parity)) return true;
    if (globaltimer_ns() - t0 > g_wait_timeout_ns) {
      wait_timed_out();
      return false;
    }
  }
}

// ---- TMA ---------------------------------------------------------------------------------
__device__ __forceinline__ void prefetch_tensormap(const void* tmap) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(tmap)) : "memory");
}
__device__ __forceinline__ void tma_load_2d(uint32_t smem_dst, const void* tmap, uint64_t* bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      ::"r"(smem_dst), "l"(reinterpret_cast<uint64_t>(tmap)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}

// TMA load delivered to every CTA of `mask` (thread-block cluster) at the same CTA-relative shared-memory offset; each
// destination's mbarrier at the same offset receives the complete_tx for the bytes that landed there.
__device__ __forceinline__ void tma_load_2d_mc(uint32_t smem_dst, const void* tmap, uint64_t* bar, int c0, int c1, uint16_t mask) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes.multicast::cluster [%0], [%1, {%3, %4}], [%2], %5;"
      ::"r"(smem_dst), "l"(reinterpret_cast<uint64_t>(tmap)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "h"(mask)
      : "memory");
}

// ---- thread-block clusters ------------------------------------------------------------------
__device__ __forceinline__ uint32_t cluster_ctarank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
__device__ __forceinline__ void cluster_sync() {
  asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}

// ---- register reallocation between warpgroups --------------------------------------------
// Executed by every warp of a warpgroup: lowers (dec) or raises (inc) its per-thread register limit to R (a multiple
// of 8 in [24, 256]); an inc blocks until the registers released by a dec are free.
template <int R> __device__ __forceinline__ void setmaxnreg_dec() {
  asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(R));
}
template <int R> __device__ __forceinline__ void setmaxnreg_inc() {
  asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(R));
}

// ---- wgmma ---------------------------------------------------------------------------------
// Swizzle modes of the wgmma matrix descriptor (bits 62-63).
enum : uint32_t { SWZ_NONE = 0, SWZ_128B = 1, SWZ_64B = 2, SWZ_32B = 3 };
// Swizzle mode whose span equals a row of `row_bytes` (32, 64 or 128): the layout TMA writes with the matching
// CU_TENSOR_MAP_SWIZZLE_*.
__host__ __device__ constexpr uint32_t swz_for_row(int row_bytes) {
  return row_bytes == 128 ? SWZ_128B : row_bytes == 64 ? SWZ_64B : SWZ_32B;
}

// Shared-memory matrix descriptor:
//   [ 0,14) start address >> 4      [16,30) leading-dimension byte offset >> 4
//   [32,46) stride-dimension byte offset >> 4   [49,52) base offset (0: tiles aligned to the swizzle repeat)
//   [62,64) swizzle mode
// Swizzled K-major operands: rows of one swizzle span, SBO = distance between 8-row groups, LBO unused; a K=16 step
// advances the start address by 32 bytes.  Swizzled MN-major operands: atoms of (span) MN elements x 8 K rows,
// SBO = distance between 8-row K groups, LBO = distance between atoms along MN.
__device__ __forceinline__ uint64_t make_desc(uint32_t saddr, uint32_t lbo_bytes, uint32_t sbo_bytes, uint32_t swizzle) {
  uint64_t d = 0;
  d |= (uint64_t)((saddr & 0x3FFFF) >> 4);
  d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFF) << 16;
  d |= (uint64_t)((sbo_bytes >> 4) & 0x3FFF) << 32;
  d |= (uint64_t)(swizzle & 3) << 62;
  return d;
}

__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N> __device__ __forceinline__ void wg_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}
// Keeps the compiler from moving accumulator reads / writes across wgmma issue and wait.
template <int R> __device__ __forceinline__ void wg_fence_regs(float (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// D[64 x N] (fp32, registers) += A[64 x 16] * B[16 x N], both operands in shared memory (descriptors).
// TA / TB: 0 = K-major, 1 = MN-major.  Accumulator layout (per warp w of the warpgroup, lane l):
//   d[4j + 2h + e] = D[16w + l/4 + 8h][8j + 2(l%4) + e]
#define BSMM_WG_OPS8(o)  "+f"(d[o + 0]), "+f"(d[o + 1]), "+f"(d[o + 2]), "+f"(d[o + 3]), \
                         "+f"(d[o + 4]), "+f"(d[o + 5]), "+f"(d[o + 6]), "+f"(d[o + 7])
#define BSMM_WG_TAIL(bf, n)                                                                                      \
  "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\t"                                                               \
  "wgmma.mma_async.sync.aligned.m64n" #n "k16.f32." bf "." bf " "

template <bool BF16, int TA, int TB>
__device__ __forceinline__ void wgmma_n16(float (&d)[8], uint64_t a, uint64_t b) {
  if constexpr (BF16)
    asm volatile(BSMM_WG_TAIL("bf16", 16) "{%0,%1,%2,%3,%4,%5,%6,%7}, %8, %9, p, 1, 1, %10, %11;\n\t}\n"
                 : BSMM_WG_OPS8(0) : "l"(a), "l"(b), "n"(TA), "n"(TB));
  else
    asm volatile(BSMM_WG_TAIL("f16", 16) "{%0,%1,%2,%3,%4,%5,%6,%7}, %8, %9, p, 1, 1, %10, %11;\n\t}\n"
                 : BSMM_WG_OPS8(0) : "l"(a), "l"(b), "n"(TA), "n"(TB));
}
template <bool BF16, int TA, int TB>
__device__ __forceinline__ void wgmma_n32(float (&d)[16], uint64_t a, uint64_t b) {
  if constexpr (BF16)
    asm volatile(BSMM_WG_TAIL("bf16", 32)
                 "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15}, %16, %17, p, 1, 1, %18, %19;\n\t}\n"
                 : BSMM_WG_OPS8(0), BSMM_WG_OPS8(8) : "l"(a), "l"(b), "n"(TA), "n"(TB));
  else
    asm volatile(BSMM_WG_TAIL("f16", 32)
                 "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15}, %16, %17, p, 1, 1, %18, %19;\n\t}\n"
                 : BSMM_WG_OPS8(0), BSMM_WG_OPS8(8) : "l"(a), "l"(b), "n"(TA), "n"(TB));
}
template <bool BF16, int TA, int TB>
__device__ __forceinline__ void wgmma_n64(float (&d)[32], uint64_t a, uint64_t b) {
  if constexpr (BF16)
    asm volatile(BSMM_WG_TAIL("bf16", 64)
                 "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,"
                 "%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, %32, %33, p, 1, 1, %34, %35;\n\t}\n"
                 : BSMM_WG_OPS8(0), BSMM_WG_OPS8(8), BSMM_WG_OPS8(16), BSMM_WG_OPS8(24)
                 : "l"(a), "l"(b), "n"(TA), "n"(TB));
  else
    asm volatile(BSMM_WG_TAIL("f16", 64)
                 "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,"
                 "%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, %32, %33, p, 1, 1, %34, %35;\n\t}\n"
                 : BSMM_WG_OPS8(0), BSMM_WG_OPS8(8), BSMM_WG_OPS8(16), BSMM_WG_OPS8(24)
                 : "l"(a), "l"(b), "n"(TA), "n"(TB));
}
template <bool BF16, int TA, int TB>
__device__ __forceinline__ void wgmma_n128(float (&d)[64], uint64_t a, uint64_t b) {
  if constexpr (BF16)
    asm volatile(BSMM_WG_TAIL("bf16", 128)
                 "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,"
                 "%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,"
                 "%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,"
                 "%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63}, %64, %65, p, 1, 1, %66, %67;\n\t}\n"
                 : BSMM_WG_OPS8(0), BSMM_WG_OPS8(8), BSMM_WG_OPS8(16), BSMM_WG_OPS8(24),
                   BSMM_WG_OPS8(32), BSMM_WG_OPS8(40), BSMM_WG_OPS8(48), BSMM_WG_OPS8(56)
                 : "l"(a), "l"(b), "n"(TA), "n"(TB));
  else
    asm volatile(BSMM_WG_TAIL("f16", 128)
                 "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,"
                 "%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,"
                 "%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,"
                 "%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63}, %64, %65, p, 1, 1, %66, %67;\n\t}\n"
                 : BSMM_WG_OPS8(0), BSMM_WG_OPS8(8), BSMM_WG_OPS8(16), BSMM_WG_OPS8(24),
                   BSMM_WG_OPS8(32), BSMM_WG_OPS8(40), BSMM_WG_OPS8(48), BSMM_WG_OPS8(56)
                 : "l"(a), "l"(b), "n"(TA), "n"(TB));
}
template <bool BF16, int TA, int TB>
__device__ __forceinline__ void wgmma_n192(float (&d)[96], uint64_t a, uint64_t b) {
  if constexpr (BF16)
    asm volatile(BSMM_WG_TAIL("bf16", 192)
                 "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,"
                 "%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,"
                 "%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,"
                 "%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63,"
                 "%64,%65,%66,%67,%68,%69,%70,%71,%72,%73,%74,%75,%76,%77,%78,%79,"
                 "%80,%81,%82,%83,%84,%85,%86,%87,%88,%89,%90,%91,%92,%93,%94,%95}, %96, %97, p, 1, 1, %98, %99;\n\t}\n"
                 : BSMM_WG_OPS8(0), BSMM_WG_OPS8(8), BSMM_WG_OPS8(16), BSMM_WG_OPS8(24),
                   BSMM_WG_OPS8(32), BSMM_WG_OPS8(40), BSMM_WG_OPS8(48), BSMM_WG_OPS8(56),
                   BSMM_WG_OPS8(64), BSMM_WG_OPS8(72), BSMM_WG_OPS8(80), BSMM_WG_OPS8(88)
                 : "l"(a), "l"(b), "n"(TA), "n"(TB));
  else
    asm volatile(BSMM_WG_TAIL("f16", 192)
                 "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,"
                 "%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,"
                 "%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,"
                 "%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63,"
                 "%64,%65,%66,%67,%68,%69,%70,%71,%72,%73,%74,%75,%76,%77,%78,%79,"
                 "%80,%81,%82,%83,%84,%85,%86,%87,%88,%89,%90,%91,%92,%93,%94,%95}, %96, %97, p, 1, 1, %98, %99;\n\t}\n"
                 : BSMM_WG_OPS8(0), BSMM_WG_OPS8(8), BSMM_WG_OPS8(16), BSMM_WG_OPS8(24),
                   BSMM_WG_OPS8(32), BSMM_WG_OPS8(40), BSMM_WG_OPS8(48), BSMM_WG_OPS8(56),
                   BSMM_WG_OPS8(64), BSMM_WG_OPS8(72), BSMM_WG_OPS8(80), BSMM_WG_OPS8(88)
                 : "l"(a), "l"(b), "n"(TA), "n"(TB));
}
template <bool BF16, int TA, int TB>
__device__ __forceinline__ void wgmma_n256(float (&d)[128], uint64_t a, uint64_t b) {
  if constexpr (BF16)
    asm volatile(BSMM_WG_TAIL("bf16", 256)
                 "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,"
                 "%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,"
                 "%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,"
                 "%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63,"
                 "%64,%65,%66,%67,%68,%69,%70,%71,%72,%73,%74,%75,%76,%77,%78,%79,"
                 "%80,%81,%82,%83,%84,%85,%86,%87,%88,%89,%90,%91,%92,%93,%94,%95,"
                 "%96,%97,%98,%99,%100,%101,%102,%103,%104,%105,%106,%107,%108,%109,%110,%111,"
                 "%112,%113,%114,%115,%116,%117,%118,%119,%120,%121,%122,%123,%124,%125,%126,%127}, %128, %129, p, 1, 1, %130, %131;\n\t}\n"
                 : BSMM_WG_OPS8(0), BSMM_WG_OPS8(8), BSMM_WG_OPS8(16), BSMM_WG_OPS8(24),
                   BSMM_WG_OPS8(32), BSMM_WG_OPS8(40), BSMM_WG_OPS8(48), BSMM_WG_OPS8(56),
                   BSMM_WG_OPS8(64), BSMM_WG_OPS8(72), BSMM_WG_OPS8(80), BSMM_WG_OPS8(88),
                   BSMM_WG_OPS8(96), BSMM_WG_OPS8(104), BSMM_WG_OPS8(112), BSMM_WG_OPS8(120)
                 : "l"(a), "l"(b), "n"(TA), "n"(TB));
  else
    asm volatile(BSMM_WG_TAIL("f16", 256)
                 "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,"
                 "%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,"
                 "%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,"
                 "%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63,"
                 "%64,%65,%66,%67,%68,%69,%70,%71,%72,%73,%74,%75,%76,%77,%78,%79,"
                 "%80,%81,%82,%83,%84,%85,%86,%87,%88,%89,%90,%91,%92,%93,%94,%95,"
                 "%96,%97,%98,%99,%100,%101,%102,%103,%104,%105,%106,%107,%108,%109,%110,%111,"
                 "%112,%113,%114,%115,%116,%117,%118,%119,%120,%121,%122,%123,%124,%125,%126,%127}, %128, %129, p, 1, 1, %130, %131;\n\t}\n"
                 : BSMM_WG_OPS8(0), BSMM_WG_OPS8(8), BSMM_WG_OPS8(16), BSMM_WG_OPS8(24),
                   BSMM_WG_OPS8(32), BSMM_WG_OPS8(40), BSMM_WG_OPS8(48), BSMM_WG_OPS8(56),
                   BSMM_WG_OPS8(64), BSMM_WG_OPS8(72), BSMM_WG_OPS8(80), BSMM_WG_OPS8(88),
                   BSMM_WG_OPS8(96), BSMM_WG_OPS8(104), BSMM_WG_OPS8(112), BSMM_WG_OPS8(120)
                 : "l"(a), "l"(b), "n"(TA), "n"(TB));
}
// D[64 x 64] (fp32, registers) += A[64 x 16] * B[16 x 64] with A in registers: four b32 per thread, each two 16-bit
// elements, low half first.  Fragment layout (PTX ISA, register fragment of matrix A for .f16 / .bf16 wgmma):
//   a[h + 2i] = A[16w + l/4 + 8h][8i + 2(l%4) + {0,1}]      (h, i in {0, 1})
// i.e. the accumulator layout above for the two 8-column groups j = 2kk, 2kk + 1 of a K = 16 slice: a[r] packs
// d[8kk + 2r], d[8kk + 2r + 1].  B comes from shared memory (TB: 0 = K-major, 1 = MN-major).
template <bool BF16, int TB>
__device__ __forceinline__ void wgmma_rs_n64(float (&d)[32], const uint32_t (&a)[4], uint64_t b) {
  if constexpr (BF16)
    asm volatile(BSMM_WG_TAIL("bf16", 64)
                 "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,"
                 "%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, {%32,%33,%34,%35}, %36, p, 1, 1, %37;\n\t}\n"
                 : BSMM_WG_OPS8(0), BSMM_WG_OPS8(8), BSMM_WG_OPS8(16), BSMM_WG_OPS8(24)
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b), "n"(TB));
  else
    asm volatile(BSMM_WG_TAIL("f16", 64)
                 "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,"
                 "%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, {%32,%33,%34,%35}, %36, p, 1, 1, %37;\n\t}\n"
                 : BSMM_WG_OPS8(0), BSMM_WG_OPS8(8), BSMM_WG_OPS8(16), BSMM_WG_OPS8(24)
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b), "n"(TB));
}
// N = 16, 32, 64, 128, 192 or 256 dispatch
template <bool BF16, int TA, int TB, int N>
__device__ __forceinline__ void wgmma(float (&d)[N / 2], uint64_t a, uint64_t b) {
  if constexpr (N == 16) wgmma_n16<BF16, TA, TB>(d, a, b);
  else if constexpr (N == 32) wgmma_n32<BF16, TA, TB>(d, a, b);
  else if constexpr (N == 64) wgmma_n64<BF16, TA, TB>(d, a, b);
  else if constexpr (N == 128) wgmma_n128<BF16, TA, TB>(d, a, b);
  else if constexpr (N == 192) wgmma_n192<BF16, TA, TB>(d, a, b);
  else wgmma_n256<BF16, TA, TB>(d, a, b);
}

// D[64 x N] (fp32, registers, N = 32, 64 or 128) = A[64 x 32] * B[32 x N] (+ D when scale_d != 0), fp8 operands: AT / BT = 0 for e4m3,
// 1 for e5m2. fp8 wgmma takes no transpose flags, so both operands are K-major. Accumulator layout as above.
#define BSMM_WG8_N32(types)                                                                                      \
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"                                               \
               "wgmma.mma_async.sync.aligned.m64n32k32.f32." types " "                                          \
               "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15}, %16, %17, p, 1, 1;\n\t}\n"             \
               : BSMM_WG_OPS8(0), BSMM_WG_OPS8(8) : "l"(a), "l"(b), "r"(scale_d))
#define BSMM_WG8_N64(types)                                                                                      \
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"                                               \
               "wgmma.mma_async.sync.aligned.m64n64k32.f32." types " "                                          \
               "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,"                                        \
               "%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, %32, %33, p, 1, 1;\n\t}\n"    \
               : BSMM_WG_OPS8(0), BSMM_WG_OPS8(8), BSMM_WG_OPS8(16), BSMM_WG_OPS8(24)                           \
               : "l"(a), "l"(b), "r"(scale_d))
#define BSMM_WG8_N128(types)                                                                                     \
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"                                               \
               "wgmma.mma_async.sync.aligned.m64n128k32.f32." types " "                                         \
               "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,"                                        \
               "%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,"                               \
               "%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,"                               \
               "%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63}, %64, %65, p, 1, 1;\n\t}\n"    \
               : BSMM_WG_OPS8(0), BSMM_WG_OPS8(8), BSMM_WG_OPS8(16), BSMM_WG_OPS8(24),                          \
                 BSMM_WG_OPS8(32), BSMM_WG_OPS8(40), BSMM_WG_OPS8(48), BSMM_WG_OPS8(56)                         \
               : "l"(a), "l"(b), "r"(scale_d))
template <int AT, int BT>
__device__ __forceinline__ void wgmma_fp8_n32(float (&d)[16], uint64_t a, uint64_t b, int scale_d) {
  if constexpr (AT == 0 && BT == 0) BSMM_WG8_N32("e4m3.e4m3");
  else if constexpr (AT == 0) BSMM_WG8_N32("e4m3.e5m2");
  else if constexpr (BT == 0) BSMM_WG8_N32("e5m2.e4m3");
  else BSMM_WG8_N32("e5m2.e5m2");
}
template <int AT, int BT>
__device__ __forceinline__ void wgmma_fp8_n64(float (&d)[32], uint64_t a, uint64_t b, int scale_d) {
  if constexpr (AT == 0 && BT == 0) BSMM_WG8_N64("e4m3.e4m3");
  else if constexpr (AT == 0) BSMM_WG8_N64("e4m3.e5m2");
  else if constexpr (BT == 0) BSMM_WG8_N64("e5m2.e4m3");
  else BSMM_WG8_N64("e5m2.e5m2");
}
template <int AT, int BT>
__device__ __forceinline__ void wgmma_fp8_n128(float (&d)[64], uint64_t a, uint64_t b, int scale_d) {
  if constexpr (AT == 0 && BT == 0) BSMM_WG8_N128("e4m3.e4m3");
  else if constexpr (AT == 0) BSMM_WG8_N128("e4m3.e5m2");
  else if constexpr (BT == 0) BSMM_WG8_N128("e5m2.e4m3");
  else BSMM_WG8_N128("e5m2.e5m2");
}
template <int AT, int BT, int N>
__device__ __forceinline__ void wgmma_fp8(float (&d)[N / 2], uint64_t a, uint64_t b, int scale_d) {
  if constexpr (N == 32) wgmma_fp8_n32<AT, BT>(d, a, b, scale_d);
  else if constexpr (N == 64) wgmma_fp8_n64<AT, BT>(d, a, b, scale_d);
  else wgmma_fp8_n128<AT, BT>(d, a, b, scale_d);
}
#undef BSMM_WG8_N128
#undef BSMM_WG8_N64
#undef BSMM_WG8_N32
#undef BSMM_WG_TAIL
#undef BSMM_WG_OPS8

}  // namespace ptx
