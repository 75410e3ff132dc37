// TMA / mbarrier / wgmma PTX wrappers and descriptor helpers shared by the tensor-core kernels (sm_90a)
// (conv_tc.cu: forward / data gradient; wgrad_tc.cu: weight gradient).
#pragma once
#include <cuda_bf16.h>
#include <stdint.h>

namespace svb {

// ------------------------------------------------------------------ PTX wrappers
__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t *bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t *bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t *bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t *bar, uint32_t parity) {
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
__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t parity) {
    // bounded spin: a lost arrival (bad descriptor, wrong byte count) must surface as a launch
    // failure through the C ABI, never as a hung GPU
    const long long t_start = clock64();
    uint32_t spins = 0;
    while (!mbar_try_wait(bar, parity)) {
        if ((++spins & 0x3FFu) == 0 && clock64() - t_start > 4000000000LL) __trap();
    }
}
__device__ __forceinline__ void bulk_g2s(void *dst_smem, const void *src_gmem, uint32_t bytes, uint64_t *bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                     smem_u32(dst_smem)),
                 "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}
// L2 prefetch of a contiguous global span (16-byte aligned, a multiple of 16 bytes); nothing lands in shared memory
__device__ __forceinline__ void bulk_prefetch_l2(const void *src_gmem, uint32_t bytes) {
    asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(src_gmem), "r"(bytes) : "memory");
}
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
// generic-proxy global writes -> visible to later bulk copies (async proxy) that read them
__device__ __forceinline__ void fence_proxy_async_global() { asm volatile("fence.proxy.async.global;" ::: "memory"); }
// named barrier over the first `threads` threads of the CTA (id 0 is __syncthreads)
__device__ __forceinline__ void named_bar_sync(uint32_t id, uint32_t threads) {
    asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(threads) : "memory");
}

// SWIZZLE_128B shared-memory matrix descriptor of wgmma (sm_90).  Rows are 128 bytes; 8-row groups (1024 B atoms)
// are SBO apart; within an atom the 16-byte chunk index is XORed with (row & 7) of the absolute shared-memory address,
// so a descriptor may start at any 128-byte row (a conv tap is a row shift).  hi word is constant per operand
// (SBO = 1024 B, base offset 0, layout 1 = SWIZZLE_128B); lo word carries the start address and the leading byte
// offset (K-major: unused; MN-major: distance between 64-element blocks of M or N).
__device__ __forceinline__ uint32_t desc_hi_sw128() { return 64u | (1u << 30); }
__device__ __forceinline__ uint32_t desc_lo(uint32_t saddr, uint32_t lbo16 = 1u) { return ((saddr >> 4) & 0x3FFFu) | (lbo16 << 16); }
__device__ __forceinline__ uint64_t desc64(uint32_t lo, uint32_t hi) { return ((uint64_t)hi << 32) | lo; }

// wgmma issue / completion.  A warpgroup (4 consecutive warps, the first a multiple of 4) issues every wgmma together;
// the accumulator fragment of m64nN is N / 2 fp32 registers per thread: row 16 * (warp % 4) + lane / 4 (+ 8), column
// 8 * j + 2 * (lane % 4) (+ 1) in d[4 j + {0, 1, 2, 3}] = {(r, c), (r, c + 1), (r + 8, c), (r + 8, c + 1)}.
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_keep(float *d) {   // the accumulator registers stay live across the async MMAs
#pragma unroll
    for (int i = 0; i < N / 2; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// d (m64 x N fp32) (+)= A (64 x K) * B (K x N); TA / TB = 1: operand is MN-major (bf16 only), 0: K-major.
// scale_d = 0 overwrites the accumulator.
#define SVB_F8(i) "+f"(d[i]), "+f"(d[i + 1]), "+f"(d[i + 2]), "+f"(d[i + 3]), "+f"(d[i + 4]), "+f"(d[i + 5]), "+f"(d[i + 6]), "+f"(d[i + 7])
#define SVB_F16 SVB_F8(0), SVB_F8(8)
#define SVB_F32 SVB_F16, SVB_F8(16), SVB_F8(24)
#define SVB_F48 SVB_F32, SVB_F8(32), SVB_F8(40)
#define SVB_F64 SVB_F48, SVB_F8(48), SVB_F8(56)
#define SVB_D16 "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}"
#define SVB_D32 "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}"
#define SVB_D48 "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47}"
#define SVB_D64 "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}"
template <int TA, int TB>
__device__ __forceinline__ void wgmma_bf16_n32(float *d, uint64_t da, uint64_t db, uint32_t scale_d) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\twgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 " SVB_D16
                 ", %16, %17, p, 1, 1, %19, %20;\n\t}"
                 : SVB_F16 : "l"(da), "l"(db), "r"(scale_d), "n"(TA), "n"(TB));
}
__device__ __forceinline__ void wgmma_tf32_n32(float *d, uint64_t da, uint64_t db, uint32_t scale_d) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\twgmma.mma_async.sync.aligned.m64n32k8.f32.tf32.tf32 " SVB_D16
                 ", %16, %17, p, 1, 1;\n\t}"
                 : SVB_F16 : "l"(da), "l"(db), "r"(scale_d));
}
template <int TA, int TB>
__device__ __forceinline__ void wgmma_bf16_n64(float *d, uint64_t da, uint64_t db, uint32_t scale_d) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\twgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 " SVB_D32
                 ", %32, %33, p, 1, 1, %35, %36;\n\t}"
                 : SVB_F32 : "l"(da), "l"(db), "r"(scale_d), "n"(TA), "n"(TB));
}
__device__ __forceinline__ void wgmma_tf32_n64(float *d, uint64_t da, uint64_t db, uint32_t scale_d) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\twgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 " SVB_D32
                 ", %32, %33, p, 1, 1;\n\t}"
                 : SVB_F32 : "l"(da), "l"(db), "r"(scale_d));
}
template <int TA, int TB>
__device__ __forceinline__ void wgmma_bf16_n96(float *d, uint64_t da, uint64_t db, uint32_t scale_d) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %50, 0;\n\twgmma.mma_async.sync.aligned.m64n96k16.f32.bf16.bf16 " SVB_D48
                 ", %48, %49, p, 1, 1, %51, %52;\n\t}"
                 : SVB_F48 : "l"(da), "l"(db), "r"(scale_d), "n"(TA), "n"(TB));
}
__device__ __forceinline__ void wgmma_tf32_n96(float *d, uint64_t da, uint64_t db, uint32_t scale_d) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %50, 0;\n\twgmma.mma_async.sync.aligned.m64n96k8.f32.tf32.tf32 " SVB_D48
                 ", %48, %49, p, 1, 1;\n\t}"
                 : SVB_F48 : "l"(da), "l"(db), "r"(scale_d));
}
template <int TA, int TB>
__device__ __forceinline__ void wgmma_bf16_n128(float *d, uint64_t da, uint64_t db, uint32_t scale_d) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\twgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 " SVB_D64
                 ", %64, %65, p, 1, 1, %67, %68;\n\t}"
                 : SVB_F64 : "l"(da), "l"(db), "r"(scale_d), "n"(TA), "n"(TB));
}
__device__ __forceinline__ void wgmma_tf32_n128(float *d, uint64_t da, uint64_t db, uint32_t scale_d) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\twgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 " SVB_D64
                 ", %64, %65, p, 1, 1;\n\t}"
                 : SVB_F64 : "l"(da), "l"(db), "r"(scale_d));
}

template <int N, int TA = 0, int TB = 0>
__device__ __forceinline__ void wgmma_bf16(float *d, uint64_t da, uint64_t db, uint32_t scale_d) {
    static_assert(N == 32 || N == 64 || N == 96 || N == 128, "wgmma_bf16: N");
    if (N == 32) wgmma_bf16_n32<TA, TB>(d, da, db, scale_d);
    else if (N == 64) wgmma_bf16_n64<TA, TB>(d, da, db, scale_d);
    else if (N == 96) wgmma_bf16_n96<TA, TB>(d, da, db, scale_d);
    else wgmma_bf16_n128<TA, TB>(d, da, db, scale_d);
}
template <int N>
__device__ __forceinline__ void wgmma_tf32(float *d, uint64_t da, uint64_t db, uint32_t scale_d) {
    static_assert(N == 32 || N == 64 || N == 96 || N == 128, "wgmma_tf32: N");
    if (N == 32) wgmma_tf32_n32(d, da, db, scale_d);
    else if (N == 64) wgmma_tf32_n64(d, da, db, scale_d);
    else if (N == 96) wgmma_tf32_n96(d, da, db, scale_d);
    else wgmma_tf32_n128(d, da, db, scale_d);
}

__device__ __forceinline__ float to_tf32(float x) {
    uint32_t r;
    asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
    return __uint_as_float(r);
}

}  // namespace svb
