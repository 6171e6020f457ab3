// Shared device helpers for the sm_90a kernels of libln3b200: mbarrier, TMA (cp.async.bulk.tensor),
// wgmma inline-PTX wrappers and the shared-memory matrix descriptor encoder.  Bit layouts follow the
// PTX ISA "asynchronous warpgroup level matrix" section (the fields CUTLASS names GmmaDescriptor).
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

namespace ln3 {

static constexpr int kWarp = 32;

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

__device__ __forceinline__ uint32_t lane_id() { return threadIdx.x & 31; }

__device__ __forceinline__ bool elect_one() {
  uint32_t pred = 0;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "elect.sync _|p, 0xffffffff;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}\n"
      : "=r"(pred));
  return pred != 0;
}

// ------------------------------------------------------------------ mbarrier
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_barrier_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)),
               "r"(bytes)
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
// Bounded wait: a protocol bug becomes a trap (sticky CUDA error the host reports) instead of a hung GPU.
// The poll loop is just try_wait (which suspends the thread for a hardware time slice) + a spin counter:
// reading clock64() in every iteration made a waiting producer / MMA warp issue several extra instructions
// per poll on the scheduler it shares with the math warps.
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  uint32_t spins = 0;
  while (!mbar_try_wait(bar, parity)) {
    if (++spins == (1u << 26)) {
      printf("ln3: mbarrier timeout block=(%d,%d,%d) thread=%d parity=%u\n", blockIdx.x,
             blockIdx.y, blockIdx.z, threadIdx.x, parity);
      __trap();
    }
  }
}

// mbar_wait without the diagnostic printf, for loops that keep a wgmma group in flight across the wait: a function
// call there (vprintf) makes ptxas serialise every wgmma of the kernel (C7510).  A timeout still traps.
__device__ __forceinline__ void mbar_wait_silent(uint64_t* bar, uint32_t parity) {
  uint32_t spins = 0;
  while (!mbar_try_wait(bar, parity)) {
    if (++spins == (1u << 26)) __trap();
  }
}

// try_wait with an explicit suspend-time hint (ns): the thread may sleep in hardware until the phase completes or the
// time limit passes, instead of returning after the (short, implementation-defined) default slice -- a waiting warp
// then stops feeding try_wait / branch pairs into the issue slots and the MIO queue of the math warps it shares a
// scheduler with.
__device__ __forceinline__ bool mbar_try_wait_hint(uint64_t* bar, uint32_t parity, uint32_t ns) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2, %3;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}\n"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity), "r"(ns)
      : "memory");
  return ok != 0;
}
__device__ __forceinline__ void mbar_wait_hint(uint64_t* bar, uint32_t parity, uint32_t ns) {
  uint32_t spins = 0;
  while (!mbar_try_wait_hint(bar, parity, ns)) {
    if (++spins == (1u << 22)) {
      printf("ln3: mbarrier timeout block=(%d,%d,%d) thread=%d parity=%u\n", blockIdx.x, blockIdx.y, blockIdx.z,
             threadIdx.x, parity);
      __trap();
    }
  }
}

// ------------------------------------------------------------------ TMA
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
__device__ __forceinline__ void tma_load_2d(void* smem_dst, const CUtensorMap* m, uint64_t* bar,
                                            int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4}], [%2];" ::"r"(smem_u32(smem_dst)),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
// 1-D bulk copy global -> shared (no tensor map): `bytes` % 16 == 0, 16-byte aligned addresses; completion is
// counted in bytes on `bar` (pair with mbar_arrive_expect_tx).
__device__ __forceinline__ void bulk_load_1d(void* smem_dst, const void* gsrc, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                   smem_u32(smem_dst)),
               "l"(gsrc), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}
__device__ __forceinline__ void tma_load_3d(void* smem_dst, const CUtensorMap* m, uint64_t* bar,
                                            int c0, int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4, %5}], [%2];" ::"r"(smem_u32(smem_dst)),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}

// smem -> global tile store (bulk async group); rows / columns outside the tensor are clipped.
__device__ __forceinline__ void tma_store_2d(const void* smem_src, const CUtensorMap* m, int c0, int c1) {
  asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];" ::"l"(
                   reinterpret_cast<uint64_t>(m)),
               "r"(smem_u32(smem_src)), "r"(c0), "r"(c1)
               : "memory");
}
__device__ __forceinline__ void tma_store_3d(const void* smem_src, const CUtensorMap* m, int c0, int c1, int c2) {
  asm volatile("cp.async.bulk.tensor.3d.global.shared::cta.bulk_group [%0, {%2, %3, %4}], [%1];" ::"l"(
                   reinterpret_cast<uint64_t>(m)),
               "r"(smem_u32(smem_src)), "r"(c0), "r"(c1), "r"(c2)
               : "memory");
}
__device__ __forceinline__ void tma_store_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
// all of this thread's bulk stores have finished READING their smem source
__device__ __forceinline__ void tma_store_wait_read() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
__device__ __forceinline__ void tma_store_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }

// ------------------------------------------------------------------ wgmma (warpgroup MMA)
// Every wgmma of a warpgroup is preceded by wgmma_fence() (orders the accumulator / A registers written by
// ordinary instructions), issued, committed as one group and waited for before its registers are read.
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// Keeps the compiler from moving accesses of an accumulator across the asynchronous MMA that owns it.
__device__ __forceinline__ void reg_fence(float& r) { asm volatile("" : "+f"(r)::"memory"); }
// D[64 x 128] (fp32, registers) (+)= A[smem desc] * B[smem desc]^T, both K-major bf16.  scale_d = 0: D = A * B.
__device__ __forceinline__ void wgmma_m64n128k16_ss(float* d, uint64_t desc_a, uint64_t desc_b, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, 0, 0;\n\t}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(desc_a), "l"(desc_b), "r"(scale_d));
}
// D[64 x 128] (fp32, registers) (+)= A[smem desc] * B[smem desc]^T, both K-major e4m3 (32 bytes of K per
// instruction: +2 in the descriptor per step).  fp8 wgmma has no transpose operands.  scale_d = 0: D = A * B.
__device__ __forceinline__ void wgmma_m64n128k32_e4m3_ss(float* d, uint64_t desc_a, uint64_t desc_b, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k32.f32.e4m3.e4m3 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1;\n\t}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(desc_a), "l"(desc_b), "r"(scale_d));
}
// D[64 x 64] (fp32) (+)= A[registers: m16n8k16-style A fragments, 16 rows per warp] * B[smem desc], B MN-major
// (a row-major K x N tile, N contiguous, transposed by the instruction).  scale_d = 0: D = A * B.
__device__ __forceinline__ void wgmma_m64n64k16_rs_tb(float* d, const uint32_t* a, uint64_t desc_b, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %37, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, {%32, %33, %34, %35}, %36, p, 1, 1, 1;\n\t}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(desc_b), "r"(scale_d));
}
// D[64 x 8] (fp32) (+)= A[registers, as above] * B[smem desc], B MN-major.  scale_d = 0: D = A * B.
__device__ __forceinline__ void wgmma_m64n8k16_rs_tb(float* d, const uint32_t* a, uint64_t desc_b, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %9, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n8k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3}, {%4, %5, %6, %7}, %8, p, 1, 1, 1;\n\t}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(desc_b), "r"(scale_d));
}

// Shared-memory matrix descriptor (64 bit):
//   [0,14)  start address >> 4        [16,30) leading-dim byte offset >> 4
//   [32,46) stride-dim byte offset>>4 [49,52) base offset     [62,64) layout: 1 = 128B swizzle
// K-major, SWIZZLE_128B tile whose rows are 128 bytes (64 bf16): 8-row groups are `sbo` bytes apart (1024 for
// a dense tile); LBO is unused for swizzled K-major operands.  A K step of 16 elements inside the 128-byte row
// advances the start address by 32 bytes (+2 in the descriptor).
// MN-major, SWIZZLE_128B: 64 MN-elements (128 B) contiguous, k-rows 128 B apart, 8-k-row groups `sbo` bytes
// apart, further 64-element MN groups `lbo` bytes apart.  A K step of 16 rows advances 2048 bytes (+128).
// Tiles start on a 1024-byte boundary (the swizzle pattern repeats every 8 rows of 128 bytes).
__device__ __forceinline__ uint64_t make_smem_desc_sw128(uint32_t smem_addr, uint32_t lbo_bytes,
                                                         uint32_t sbo_bytes) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((smem_addr & 0x3FFFF) >> 4);
  d |= static_cast<uint64_t>((lbo_bytes >> 4) & 0x3FFF) << 16;
  d |= static_cast<uint64_t>((sbo_bytes >> 4) & 0x3FFF) << 32;
  d |= static_cast<uint64_t>(1) << 62;
  return d;
}
// The same descriptor without swizzle (layout 0): the operand is a grid of 8 x 16-byte core matrices, each 128
// contiguous bytes.  K-major: `lbo` bytes between the two core matrices of a k16 step (K direction), `sbo` bytes
// between 8-row groups (M / N direction).  An MN-major operand 8 elements wide has one core matrix per 8 k-rows.
__device__ __forceinline__ uint64_t make_smem_desc_plain(uint32_t smem_addr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((smem_addr & 0x3FFFF) >> 4);
  d |= static_cast<uint64_t>((lbo_bytes >> 4) & 0x3FFF) << 16;
  d |= static_cast<uint64_t>((sbo_bytes >> 4) & 0x3FFF) << 32;
  return d;
}

__device__ __forceinline__ int ld_acquire_gpu(const int* p) {
  int v;
  asm volatile("ld.acquire.gpu.global.s32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}

// One elected lane of the (converged) warp.
__device__ __forceinline__ bool elect_one_sync() {
  uint32_t pred;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "elect.sync _|p, 0xffffffff;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}\n"
      : "=r"(pred));
  return pred != 0;
}
__device__ __forceinline__ void named_bar_sync(int id, int nthreads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}
__device__ __forceinline__ void named_bar_arrive(int id, int nthreads) {
  asm volatile("bar.arrive %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}
// Move registers between the warpgroups of a CTA (every thread of the warpgroup executes it): a warpgroup that
// only issues TMA gives registers back, the MMA warpgroups take them.
template <int N>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(N)); }
template <int N>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(N)); }
// fp32 pairs held in one 64-bit value; fma2 evaluates both lanes with scalar FMAs (same rounding as the
// packed form: one fma.rn per lane).
__device__ __forceinline__ uint64_t pk2(float lo, float hi) {
  uint64_t d;
  asm("mov.b64 %0, {%1, %2};" : "=l"(d) : "f"(lo), "f"(hi));
  return d;
}
__device__ __forceinline__ void upk2(uint64_t v, float& lo, float& hi) {
  asm("mov.b64 {%0, %1}, %2;" : "=f"(lo), "=f"(hi) : "l"(v));
}
__device__ __forceinline__ float fast_exp2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ uint64_t fma2(uint64_t a, uint64_t b, uint64_t c) {
  float a0, a1, b0, b1, c0, c1;
  upk2(a, a0, a1);
  upk2(b, b0, b1);
  upk2(c, c0, c1);
  return pk2(fmaf(a0, b0, c0), fmaf(a1, b1, c1));
}

// ------------------------------------------------------------------ 32-byte global accesses
// Eight consecutive fp32 / 32-bit words as two 128-bit accesses (32-byte aligned addresses).
__device__ __forceinline__ void ldg256_na(const void* p, float* v) {
  asm volatile("ld.global.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];"
               : "=f"(v[0]), "=f"(v[1]), "=f"(v[2]), "=f"(v[3]) : "l"(p));
  asm volatile("ld.global.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4+16];"
               : "=f"(v[4]), "=f"(v[5]), "=f"(v[6]), "=f"(v[7]) : "l"(p));
}
// L2 evict_last forms: the fp32 residual stream is read and re-written by three passes per block with GEMM
// operand streams in between; marking its lines evict_last keeps them in L2.
__device__ __forceinline__ void ldg256_na_el(const void* p, float* v) {
  asm volatile(
      "{\n\t.reg .b64 pol;\n\t"
      "createpolicy.fractional.L2::evict_last.b64 pol, 1.0;\n\t"
      "ld.global.L1::no_allocate.L2::cache_hint.v4.f32 {%0,%1,%2,%3}, [%8], pol;\n\t"
      "ld.global.L1::no_allocate.L2::cache_hint.v4.f32 {%4,%5,%6,%7}, [%8+16], pol;\n\t}\n"
      : "=f"(v[0]), "=f"(v[1]), "=f"(v[2]), "=f"(v[3]), "=f"(v[4]), "=f"(v[5]), "=f"(v[6]), "=f"(v[7])
      : "l"(p));
}
__device__ __forceinline__ void stg256_f32_el(void* p, const float* v) {
  asm volatile(
      "{\n\t.reg .b64 pol;\n\t"
      "createpolicy.fractional.L2::evict_last.b64 pol, 1.0;\n\t"
      "st.global.L2::cache_hint.v4.f32 [%0], {%1,%2,%3,%4}, pol;\n\t"
      "st.global.L2::cache_hint.v4.f32 [%0+16], {%5,%6,%7,%8}, pol;\n\t}\n" ::"l"(p),
      "f"(v[0]), "f"(v[1]), "f"(v[2]), "f"(v[3]), "f"(v[4]), "f"(v[5]), "f"(v[6]), "f"(v[7])
      : "memory");
}
__device__ __forceinline__ void stg256_f32(void* p, const float* v) {
  asm volatile("st.global.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(p), "f"(v[0]), "f"(v[1]), "f"(v[2]), "f"(v[3])
               : "memory");
  asm volatile("st.global.v4.f32 [%0+16], {%1,%2,%3,%4};" ::"l"(p), "f"(v[4]), "f"(v[5]), "f"(v[6]), "f"(v[7])
               : "memory");
}

// ------------------------------------------------------------------ math
__device__ __forceinline__ float gelu_erf(float x) {
  return 0.5f * x * (1.0f + erff(x * 0.70710678118654752440f));
}
// GELU(x) = x * Phi(x) with erfc by Abramowitz-Stegun 7.1.26 (|error| <= 1.5e-7):
//   erfc(z) = t(a1 + t(a2 + t(a3 + t(a4 + t a5)))) exp(-z^2),  t = 1/(1 + p z),  z = |x|/sqrt2
//   GELU(x) = relu(x) - |x| * 0.5 erfc(z)          (both signs of x)
// Written with s = |x| * sqrt(log2(e)/2) so that exp(-z^2) = 2^(-s*s), the 0.5 folded into the a_i, and
// raw MUFU rcp/ex2 (.ftz: no range fix-up code): 5 FMUL + 5 FFMA + FMNMX + FADD + 2 MUFU per element,
// against ~25 for the __fdividef/__expf form and ~40 for erff.  Used where the result is rounded to bf16.
__device__ __forceinline__ float rcp_approx_ftz(float x) {
  float y;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ float ex2_approx_ftz(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ float gelu_erf_fast(float x) {
  constexpr float kS = 0.84932180028801904272f;                 // sqrt(log2(e) / 2)
  constexpr float kP = 0.3275911f * 0.70710678118654752440f / kS;  // p * z = kP * s
  const float s = fabsf(x) * kS;
  const float t = rcp_approx_ftz(fmaf(kP, s, 1.f));
  float q = fmaf(t, 0.5f * 1.061405429f, 0.5f * -1.453152027f);
  q = fmaf(t, q, 0.5f * 1.421413741f);
  q = fmaf(t, q, 0.5f * -0.284496736f);
  q = fmaf(t, q, 0.5f * 0.254829592f);
  const float e = ex2_approx_ftz(s * -s);
  const float w = (q * t) * (e * x);                            // x * 0.5 erfc(z), sign of x
  return fmaxf(x, 0.f) - fabsf(w);
}
// erf-GELU for the fc1 epilogue of the GEMM, two elements at a time on the FMA pipe and WITHOUT the MUFU:
// GELU(x) = x * Phi(x),  Phi(x) = sat(0.5 + x * Q(min(x^2, 16))),  Q an even polynomial of degree
// 8 in u = x^2 fitted (x^2-weighted Chebyshev least squares on |x| <= 4) to (Phi(x) - 0.5) / x.  fma.sat clamps
// Phi to [0, 1], which is also the right limit for |x| > 4 (x Q(16) = +-0.49997 |x| / 4).
// Error (fp32 evaluation, |x| <= 8): |abs| <= 1.1e-5 for |x| < 4, relative <= 5e-4 where |GELU| > 0.01, and GELU is
// flushed to 0 below x = -4 (true value > -1.3e-4): all below the bf16 rounding of the stored result (2^-9).
__device__ __forceinline__ void gelu_erf_poly2(float& a, float& b) {
  const uint64_t x = pk2(a, b);
  uint64_t u = fma2(x, x, pk2(0.f, 0.f));
  float u0, u1;
  upk2(u, u0, u1);
  u = pk2(fminf(u0, 16.f), fminf(u1, 16.f));
  uint64_t q = pk2(6.4972029061e-11f, 6.4972029061e-11f);
  q = fma2(q, u, pk2(-5.8924924216e-09f, -5.8924924216e-09f));
  q = fma2(q, u, pk2(2.3887849765e-07f, 2.3887849765e-07f));
  q = fma2(q, u, pk2(-5.7769494275e-06f, -5.7769494275e-06f));
  q = fma2(q, u, pk2(9.4159107405e-05f, 9.4159107405e-05f));
  q = fma2(q, u, pk2(-1.1085928497e-03f, -1.1085928497e-03f));
  q = fma2(q, u, pk2(9.8028649727e-03f, 9.8028649727e-03f));
  q = fma2(q, u, pk2(-6.6304471162e-02f, -6.6304471162e-02f));
  q = fma2(q, u, pk2(3.9887112041e-01f, 3.9887112041e-01f));
  float q0, q1, p0, p1;
  upk2(q, q0, q1);
  asm("fma.rn.sat.f32 %0, %1, %2, 0f3F000000;" : "=f"(p0) : "f"(a), "f"(q0));
  asm("fma.rn.sat.f32 %0, %1, %2, 0f3F000000;" : "=f"(p1) : "f"(b), "f"(q1));
  a *= p0;
  b *= p1;
}
__device__ __forceinline__ float gelu_tanh(float x) {
  const float k0 = 0.7978845608028654f, k1 = 0.044715f;
  return 0.5f * x * (1.0f + tanhf(k0 * (x + k1 * x * x * x)));
}
__device__ __forceinline__ float silu(float x) { return x / (1.0f + __expf(-x)); }
// CLIP's QuickGELU: x * sigmoid(1.702 x)  (transformers `quick_gelu`, open_clip `QuickGELU`)
__device__ __forceinline__ float quick_gelu(float x) { return x / (1.0f + __expf(-1.702f * x)); }

__device__ __forceinline__ uint32_t pack_bf16x2(float lo, float hi) {
  __nv_bfloat162 t = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&t);
}

// ------------------------------------------------------------------ fp8 (e4m3) block quantisation
// The 1 x 128 block format of include/ln3b200.h: s = fp32(absmax / 448) (IEEE division), code = e4m3 of fp32(x / s)
// rounded to nearest even with saturation to +-448 (cvt.rn.satfinite); an all-zero block has s = 0 and zero codes.
__device__ __forceinline__ float fp8_block_scale(float absmax) { return __fdiv_rn(absmax, 448.0f); }
// two e4m3 codes, `lo` in the low byte
__device__ __forceinline__ uint16_t fp8_code2(float lo, float hi, float s) {
  if (s == 0.f) return 0;
  uint16_t r;
  asm("cvt.rn.satfinite.e4m3x2.f32 %0, %1, %2;" : "=h"(r) : "f"(__fdiv_rn(hi, s)), "f"(__fdiv_rn(lo, s)));
  return r;
}

// ------------------------------------------------------------------ legacy warp-level TF32 MMA
__device__ __forceinline__ uint32_t to_tf32(float x) {
  uint32_t r;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
  return r;
}
// D (16x8, fp32) += A (16x8, tf32, row) * B (8x8, tf32, col).  Lane = 4g + t holds
//   A: a0 (g, t)  a1 (g+8, t)  a2 (g, t+4)  a3 (g+8, t+4);   B: b0 (k=t, n=g)  b1 (k=t+4, n=g)
//   D: d0 (g, 2t)  d1 (g, 2t+1)  d2 (g+8, 2t)  d3 (g+8, 2t+1)
__device__ __forceinline__ void mma_tf32(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}


}  // namespace ln3
