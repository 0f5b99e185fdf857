// Thin inline-PTX wrappers for sm_90a: mbarrier, 1-D bulk async copy (TMA engine), warpgroup MMA (wgmma)
// and shared-memory matrix descriptors.
#pragma once
#include <cstdint>
#include <cuda_runtime.h>

namespace adn {

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

// One lane of a converged warp (elect.sync): keeps the surrounding code warp-uniform for the compiler.
__device__ __forceinline__ bool elect_one() {
  uint32_t pred;
  asm volatile("{\n\t.reg .pred p;\n\telect.sync _|p, 0xffffffff;\n\tselp.b32 %0, 1, 0, p;\n\t}" : "=r"(pred));
  return pred != 0;
}

__device__ __forceinline__ void st_shared_v4(uint32_t addr, uint32_t x, uint32_t y, uint32_t z, uint32_t w) {
  asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(x), "r"(y), "r"(z), "r"(w) : "memory");
}

__device__ __forceinline__ float4 ld_shared_f4(uint32_t addr) {
  float4 v;
  asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(addr));
  return v;
}

// Named CTA barriers (bar.sync / bar.arrive with an explicit participant count).
__device__ __forceinline__ void named_bar_sync(int id, int nthreads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}
__device__ __forceinline__ void named_bar_arrive(int id, int nthreads) {
  asm volatile("bar.arrive %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}

// ------------------------------------------------------------------------------------ mbarrier
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_fence_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("{\n\t.reg .b64 st;\n\tmbarrier.arrive.shared::cta.b64 st, [%0];\n\t}" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("{\n\t.reg .b64 st;\n\tmbarrier.arrive.expect_tx.shared::cta.b64 st, [%0], %1;\n\t}" ::"r"(smem_u32(bar)),
               "r"(bytes)
               : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  // the suspend-time hint lets the hardware park the thread instead of spinning through the issue slots
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2, %3;\n\t"
      "selp.b32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity), "r"(0x989680u)
      : "memory");
  return ok != 0;
}

// Device-side watchdog: every wait is bounded so a protocol bug can never hang the GPU.
// On timeout the kernel records the site in *err_flag and traps (the launch then reports an error).  Inlined: a call
// in a kernel that reallocates registers between warpgroups (setmaxnreg) makes ptxas's register allocation fail.
#ifndef ADN_WATCHDOG_CYCLES
#define ADN_WATCHDOG_CYCLES (4000000000ll)  // ~2 s at 1.98 GHz
#endif
static __device__ __forceinline__ void mbar_wait_slow(uint64_t* bar, uint32_t parity, int* err_flag, int site) {
  const long long t0 = clock64();
  while (!mbar_try_wait(bar, parity)) {
    if (clock64() - t0 > ADN_WATCHDOG_CYCLES) {
      if (err_flag) atomicExch(err_flag, 0x1000 + site);
      __threadfence_system();
      asm volatile("trap;");
    }
  }
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity, int* err_flag, int site) {
  if (mbar_try_wait(bar, parity)) return;
  mbar_wait_slow(bar, parity, err_flag, site);
}

// --------------------------------------------------------------------------- async bulk copy
// 1-D bulk copy global -> shared through the TMA engine (SASS: UBLKCP), completion on an mbarrier.
__device__ __forceinline__ void bulk_g2s(void* smem_dst, const void* gmem_src, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                   smem_u32(smem_dst)),
               "l"(gmem_src), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}
// 1-D bulk copy shared -> global through the TMA engine (bulk async-group completion).
__device__ __forceinline__ void bulk_s2g(void* gmem_dst, const void* smem_src, uint32_t bytes) {
  asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(gmem_dst), "r"(smem_u32(smem_src)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
__device__ __forceinline__ void bulk_wait_read_all() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
__device__ __forceinline__ void bulk_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }

// generic-proxy writes (any state space) -> visible to subsequent async-proxy (TMA) accesses
__device__ __forceinline__ void fence_proxy_async_all() { asm volatile("fence.proxy.async;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}

// Register reallocation between warpgroups (all threads of a warpgroup execute it).
template <int N>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(N)); }
template <int N>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(N)); }

// ------------------------------------------------------------------------------------ wgmma
// Warpgroup MMA (sm_90a): D[64 x 128] (fp32, registers) += A[64 x 16] * B[128 x 16]^T, B (and, in the first form, A) bf16
// K-major in shared memory, issued by all 128 threads of a warpgroup.  Accumulator fragment of thread t (warp w = t / 32, lane l):
// d[4 i + j] is row 16 w + l / 4 + 8 (j >> 1), column 8 i + 2 (l % 4) + (j & 1).
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }

// accumulate == 0: D = A * B (the registers' previous contents are ignored).
__device__ __forceinline__ void wgmma_m64n128_bf16(float (&d)[64], uint64_t a_desc, uint64_t b_desc, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
      "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
      "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
      "%64, %65, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),
        "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]),
        "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]),
        "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]),
        "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]),
        "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]),
        "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]),
        "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(a_desc), "l"(b_desc), "r"(accumulate)
      : "memory");
}

// The same MMA with A from registers (SASS: HGMMA with a register A operand).  Fragment of thread t (warp w, lane l):
// a[0] = A[16 w + l / 4][2 (l % 4) + {0, 1}], a[1] = the same columns of row + 8, a[2] / a[3] = columns + 8 of those rows,
// bf16 pairs, lower column in the low half.  For columns 16 j .. 16 j + 15 of a finished accumulator d that is
// a = {bf16x2(d[8j], d[8j+1]), bf16x2(d[8j+2], d[8j+3]), bf16x2(d[8j+4], d[8j+5]), bf16x2(d[8j+6], d[8j+7])}: a layer's
// output feeds the next layer's MMAs without leaving the registers.
__device__ __forceinline__ void wgmma_m64n128_bf16_rs(float (&d)[64], const uint32_t (&a)[4], uint64_t b_desc, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %69, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
      "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
      "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
      "{%64, %65, %66, %67}, %68, p, 1, 1, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),
        "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]),
        "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]),
        "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]),
        "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]),
        "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]),
        "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]),
        "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b_desc), "r"(accumulate)
      : "memory");
}

// Shared-memory matrix descriptor (sm_90 wgmma), K-major operand, 128-byte swizzle, bf16:
// rows are 128 B (64 elements) apart, groups of 8 rows are 1024 B apart (SBO), the 16-byte chunk
// index is XORed with (row % 8) by the hardware.  Tile base must be 1024-byte aligned; a K step of 16
// elements advances the start address by 32 bytes.
//   bits [0,14)  start address >> 4        bits [16,30) leading byte offset >> 4 (unused for swizzled K-major: 1)
//   bits [32,46) stride byte offset >> 4   bits [62,64) layout type: 1 = SWIZZLE_128B
__device__ __forceinline__ uint64_t make_desc_sw128(uint32_t smem_addr_bytes) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((smem_addr_bytes & 0x3FFFF) >> 4);
  d |= static_cast<uint64_t>(1) << 16;
  d |= static_cast<uint64_t>(1024 >> 4) << 32;
  d |= static_cast<uint64_t>(1) << 62;
  return d;
}

// The same descriptor for the 64-byte swizzle: rows are 64 B (32 elements) apart, groups of 8 rows 512 B apart (SBO), the
// 16-byte chunk index is XORed with (row % 8) / 2.  Tile base 512-byte aligned; a K step of 16 elements advances the
// start address by 32 bytes.  Layout type (bits [62,64)) 2 = SWIZZLE_64B.
__device__ __forceinline__ uint64_t make_desc_sw64(uint32_t smem_addr_bytes) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((smem_addr_bytes & 0x3FFFF) >> 4);
  d |= static_cast<uint64_t>(1) << 16;
  d |= static_cast<uint64_t>(512 >> 4) << 32;
  d |= static_cast<uint64_t>(2) << 62;
  return d;
}

// Byte offset of element (row, col) inside one [rows x 64] bf16 K-major SWIZZLE_128B block.
__host__ __device__ __forceinline__ uint32_t sw128_offset(uint32_t row, uint32_t col) {
  const uint32_t chunk = (col >> 3) ^ (row & 7);
  return (row >> 3) * 1024u + (row & 7) * 128u + chunk * 16u + (col & 7) * 2u;
}

// Byte offset of element (row, col) inside one [rows x 32] bf16 K-major SWIZZLE_64B block.
__host__ __device__ __forceinline__ uint32_t sw64_offset(uint32_t row, uint32_t col) {
  const uint32_t chunk = (col >> 3) ^ ((row >> 1) & 3);
  return (row >> 3) * 512u + (row & 7) * 64u + chunk * 16u + (col & 7) * 2u;
}

}  // namespace adn
