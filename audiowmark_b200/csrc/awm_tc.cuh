// awm_tc.cuh -- Hopper (sm_90a) plumbing used by the tensor-core kernels of this library: mbarriers, the bulk-copy engine
// (TMA, 1-D form) and warpgroup MMA (wgmma), as thin inline-PTX wrappers, plus the shared-memory operand layout the kernels
// build by hand.
//
// Operand layout (K-major, no swizzle -- "interleaved" canonical layout of the wgmma shared-memory descriptor): an operand of
// R rows (M or N) and K columns of 16-bit elements is stored as 8 x 8 core matrices of 128 contiguous bytes (8 rows x 16 bytes);
// core matrices that are neighbours in the row direction lie SBO = 128 bytes apart, neighbours in the K direction LBO = R * 16
// bytes apart (one "slab" of 8 K-columns for all rows):
//     byte offset of element (r, k) = (k / 8) * (R * 16) + (r / 8) * 128 + (r % 8) * 16 + (k % 8) * 2
// One wgmma of f16 inputs consumes K = 16, i.e. two slabs; the descriptor of K-step j starts at slab 2 j, that of rows r0 .. at
// byte (r0 / 8) * 128 of the slab.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace awm { namespace tc {

__device__ __forceinline__ uint32_t smem_u32 (const void *p) { return (uint32_t) __cvta_generic_to_shared (p); }

// ---- mbarrier ----------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init (uint64_t *bar, uint32_t count)
{
  asm volatile ("mbarrier.init.shared::cta.b64 [%0], %1;" :: "r"(smem_u32 (bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_mbar_init() { asm volatile ("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_arrive (uint64_t *bar)
{
  asm volatile ("mbarrier.arrive.shared::cta.b64 _, [%0];" :: "r"(smem_u32 (bar)) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx (uint64_t *bar, uint32_t bytes)
{
  asm volatile ("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" :: "r"(smem_u32 (bar)), "r"(bytes) : "memory");
}
// spin until the phase with the given parity has completed (a fresh barrier passes a wait on parity 1)
__device__ __forceinline__ void mbar_wait (uint64_t *bar, uint32_t parity)
{
  const uint32_t addr = smem_u32 (bar);
  uint32_t done;
  do
    {
      asm volatile ("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                    : "=r"(done) : "r"(addr), "r"(parity) : "memory");
    }
  while (!done);
}
// the same for warps that wait for work which takes microseconds (the MMA warpgroup, FFT warps waiting for a free A buffer):
// try_wait with a suspend-time hint parks the thread in hardware until the phase completes or the hint (nanoseconds) runs out, so
// a waiting warp wakes up at once when its barrier flips but takes next to no issue slots from the FFT warps meanwhile
__device__ __forceinline__ void mbar_wait_relaxed (uint64_t *bar, uint32_t parity, uint32_t suspend_ns = 20000)
{
  const uint32_t addr = smem_u32 (bar);
  uint32_t done;
  do
    {
      asm volatile ("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2, %3;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                    : "=r"(done) : "r"(addr), "r"(parity), "r"(suspend_ns) : "memory");
    }
  while (!done);
}
// make generic-proxy writes to shared memory (st.shared) visible to the async proxy (wgmma / bulk copies read through it)
__device__ __forceinline__ void fence_proxy_async() { asm volatile ("fence.proxy.async.shared::cta;" ::: "memory"); }

// ---- TMA, 1-D bulk copy global -> shared, completion counted in bytes on an mbarrier (SASS: UBLKCP) ------------------------------
__device__ __forceinline__ void bulk_load (void *smem_dst, const void *gmem_src, uint32_t bytes, uint64_t *bar)
{
  asm volatile ("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                :: "r"(smem_u32 (smem_dst)), "l"(gmem_src), "r"(bytes), "r"(smem_u32 (bar)) : "memory");
}

// ---- wgmma (sm_90a warpgroup MMA) -------------------------------------------------------------------------------------------------
// shared-memory matrix descriptor, K-major, no swizzle: start address, LBO (K direction), SBO (row direction), all >> 4;
// base offset (bits 49..51) and layout type (bits 62..63) = 0
__device__ __forceinline__ uint64_t smem_desc_kmajor (uint32_t smem_addr, uint32_t lbo_bytes, uint32_t sbo_bytes)
{
  return uint64_t ((smem_addr >> 4) & 0x3fff) | (uint64_t ((lbo_bytes >> 4) & 0x3fff) << 16) | (uint64_t ((sbo_bytes >> 4) & 0x3fff) << 32);
}
__device__ __forceinline__ void wgmma_fence() { asm volatile ("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile ("wgmma.commit_group.sync.aligned;" ::: "memory"); }
// wait until at most `Pending` committed wgmma groups of this thread are still in flight
template <int Pending>
__device__ __forceinline__ void wgmma_wait() { asm volatile ("wgmma.wait_group.sync.aligned %0;" :: "n"(Pending) : "memory"); }
// keeps the compiler from touching accumulator registers across the asynchronous MMA (reads after the wait stay after it)
__device__ __forceinline__ void wgmma_fence_operand (float& r) { asm volatile ("" : "+f"(r) :: "memory"); }

// D (+)= A[smem] * B[smem]^T for a 64 x 96 tile, K = 16, fp16 inputs, fp32 accumulators; the whole warpgroup (4 aligned warps)
// issues it together.  Accumulator fragment of thread t (warp wi = t / 32, lane l): d[4 q + 2 h + c] holds row 16 wi + l / 4 + 8 h,
// column 8 q + 2 (l % 4) + c.
__device__ __forceinline__ void wgmma_m64n96k16_f16 (float (&d)[48], uint64_t desc_a, uint64_t desc_b, bool accumulate)
{
  asm volatile ("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %50, 0;\n\t"
                "wgmma.mma_async.sync.aligned.m64n96k16.f32.f16.f16 "
                "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, "
                "%24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47}, "
                "%48, %49, p, 1, 1, 0, 0;\n\t}"
                : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
                  "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
                  "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
                  "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
                  "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
                  "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47])
                : "l"(desc_a), "l"(desc_b), "r"(accumulate ? 1u : 0u) : "memory");
}

// byte offset of element (r, k) of an R-row operand in the layout described at the top of this file
__host__ __device__ constexpr uint32_t operand_offset (int R, int r, int k)
{
  return uint32_t (k >> 3) * uint32_t (R * 16) + uint32_t (r >> 3) * 128u + uint32_t (r & 7) * 16u + uint32_t (k & 7) * 2u;
}

} } // namespace awm::tc
