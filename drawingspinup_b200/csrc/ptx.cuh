// Thin inline-PTX wrappers for the sm_90a features the convolution kernel uses:
// cp.async, proxy fences and warpgroup MMA (wgmma) with shared-memory operand descriptors.
#pragma once
#include <cuda_fp16.h>
#include <stdint.h>

namespace dsu {

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
    return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

// ---------------------------------------------------------------- async copies
// 16-byte cp.async with zero fill when src_bytes == 0 (LDGSTS).
__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src, uint32_t src_bytes) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(src_bytes) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

__device__ __forceinline__ uint4 ld_shared_v4(uint32_t addr) {
    uint4 v;
    asm volatile("ld.shared.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(addr) : "memory");
    return v;
}
__device__ __forceinline__ void st_shared_v4(uint32_t addr, const uint4& v) {
    asm volatile("st.shared.v4.u32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}

// generic-proxy smem writes (st.shared, cp.async) -> visible to the async proxy (wgmma operand reads)
__device__ __forceinline__ void fence_proxy_async_smem() {
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}

// Read-only 128-bit global load under a predicate, zeros otherwise (no branch, no dependence on a dummy address).
__device__ __forceinline__ uint4 ldg128_if(const void* ptr, bool ok) {
    uint4 v;
    asm("{\n\t.reg .pred p;\n\tsetp.ne.u32 p, %5, 0;\n\tmov.u32 %0, 0;\n\tmov.u32 %1, 0;\n\tmov.u32 %2, 0;\n\tmov.u32 %3, 0;\n\t"
        "@p ld.global.nc.v4.u32 {%0, %1, %2, %3}, [%4];\n\t}"
        : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w)
        : "l"(ptr), "r"(static_cast<uint32_t>(ok)));
    return v;
}

// ---------------------------------------------------------------- wgmma
// Shared-memory matrix descriptor, K-major operand, 128-byte swizzle: rows of 128 B (64 fp16 of K), 8-row groups
// `sbo_bytes` apart, the 16-byte chunk c of row r at r * 128 + ((c ^ (r & 7)) << 4) inside a 1024-byte aligned atom.
// Adding 2 to the descriptor (32 bytes) steps to the next K16 slice of the row.
__device__ __forceinline__ uint64_t wgmma_desc_sw128(uint32_t smem_addr, uint32_t sbo_bytes) {
    uint64_t d = 0;
    d |= static_cast<uint64_t>((smem_addr >> 4) & 0x3FFFu);
    d |= static_cast<uint64_t>(1) << 16;                 // leading byte offset: unused for swizzled K-major operands
    d |= static_cast<uint64_t>((sbo_bytes >> 4) & 0x3FFFu) << 32;
    d |= static_cast<uint64_t>(1) << 62;                 // SWIZZLE_128B
    return d;
}

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }

// D[64 x N] += A[64 x 16] * B[16 x N]; fp16 operands from shared memory (both K-major), fp32 accumulators in registers.
// Thread t of the warpgroup holds d[i] = D[16 * (t / 32) + (t % 32) / 4 + 8 * ((i >> 1) & 1)][8 * (i >> 2) + 2 * (t % 4) + (i & 1)].
template <int N>
struct Wgmma;

template <>
struct Wgmma<32> {
    __device__ __forceinline__ static void mma(float* d, uint64_t a, uint64_t b) {
        asm volatile(
            "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\t"
            "wgmma.mma_async.sync.aligned.m64n32k16.f32.f16.f16 "
            "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1, 0, 0;\n\t}"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
              "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
            : "l"(a), "l"(b));
    }
};

template <>
struct Wgmma<64> {
    __device__ __forceinline__ static void mma(float* d, uint64_t a, uint64_t b) {
        asm volatile(
            "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\t"
            "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 "
            "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
            "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, 0, 0;\n\t}"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
              "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
              "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
              "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
            : "l"(a), "l"(b));
    }
};

template <>
struct Wgmma<128> {
    __device__ __forceinline__ static void mma(float* d, uint64_t a, uint64_t b) {
        asm volatile(
            "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\t"
            "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 "
            "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, 0, 0;\n\t}"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
              "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
              "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
              "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
              "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
              "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
              "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
              "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
            : "l"(a), "l"(b));
    }
};

}  // namespace dsu
