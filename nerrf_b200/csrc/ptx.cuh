// sm_90a PTX wrappers shared by the kernels: shared-memory addresses, mbarriers, async copies (cp.async and the bulk
// copy engine), proxy fences, named barriers and the wgmma pieces (shared-memory descriptor, register-A MMAs, the bf16
// term split of fp32 values and the swizzled K-major operand layout).
#pragma once
#include <cuda_bf16.h>
#include <stdint.h>

namespace nerrf {

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

// ---------------------------------------------------------------- mbarriers
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
    asm volatile("{\n\t.reg .b64 st;\n\tmbarrier.arrive.shared::cta.b64 st, [%0];\n\t}" ::"r"(bar) : "memory");
}
// arrive (count 1) and add `bytes` to the phase's pending transaction count: the phase completes when the
// arrival count AND the byte count are both satisfied
__device__ __forceinline__ void mbar_arrive_expect_tx(uint32_t bar, uint32_t bytes) {
    asm volatile("{\n\t.reg .b64 st;\n\tmbarrier.arrive.expect_tx.shared::cta.b64 st, [%0], %1;\n\t}" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint32_t bar, uint32_t parity) {
    uint32_t done;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(done)
        : "r"(bar), "r"(parity)
        : "memory");
    return done != 0;
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
    while (!mbar_try_wait(bar, parity)) {
    }
}
// for roles that have slack: poll with a sleep so they do not burn the issue slots the busy warps need
__device__ __forceinline__ void mbar_wait_relaxed(uint32_t bar, uint32_t parity) {
    while (!mbar_try_wait(bar, parity)) __nanosleep(400);
}
// bounded: a protocol bug ends in a trap (launch error), never in a hung GPU
__device__ __forceinline__ void mbar_wait_bounded(uint32_t bar, uint32_t parity) {
    for (uint32_t spin = 0; !mbar_try_wait(bar, parity); ++spin) {
        if (spin > (1u << 16)) __nanosleep(64);
        if (spin > (1u << 26)) __trap();
    }
}

// ---------------------------------------------------------------- async copies
// bulk async copy global -> shared (the non-tensor TMA path, SASS UBLKCP): `bytes` (multiple of 16) from a 16-byte
// aligned global address to a 16-byte aligned shared address; completion is signalled on `bar` as complete_tx(bytes)
__device__ __forceinline__ void bulk_g2s(uint32_t smem_dst, const void* gsrc, uint32_t bytes, uint32_t bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(smem_dst), "l"(gsrc), "r"(bytes), "r"(bar)
                 : "memory");
}
// bulk prefetch of `bytes` (multiple of 16) from a 16-byte aligned global address into L2, no completion signal
__device__ __forceinline__ void bulk_prefetch_l2(const void* gsrc, uint32_t bytes) {
    asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(gsrc), "r"(bytes) : "memory");
}
__device__ __forceinline__ void cp_async16(uint32_t smem_dst, const void* gsrc) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_dst), "l"(gsrc) : "memory");
}
// predicated 16-byte async copy (no branch)
__device__ __forceinline__ void cp_async16_pred(uint32_t smem_dst, const void* gsrc, bool pred) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "setp.ne.b32 p, %2, 0;\n\t"
        "@p cp.async.cg.shared.global [%0], [%1], 16;\n\t}"
        ::"r"(smem_dst), "l"(gsrc), "r"((uint32_t)pred)
        : "memory");
}
// ---------------------------------------------------------------- L2 eviction-priority hints
// A policy (createpolicy, applied to every access that carries it) is passed to the .L2::cache_hint form of an access.
// The operand ends up in a uniform register: pass a value that is the same in every lane, or ptxas emits a loop over
// the distinct values.  Hints only change which lines L2 evicts first, never the data an access returns.  createpolicy
// is volatile so that it is issued where the policy is used instead of holding two registers for the whole kernel.
__device__ __forceinline__ uint64_t l2_policy_evict_first() {
    uint64_t p;
    asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p));
    return p;
}
__device__ __forceinline__ uint64_t l2_policy_evict_normal() {
    uint64_t p;
    asm volatile("createpolicy.fractional.L2::evict_normal.b64 %0, 1.0;" : "=l"(p));
    return p;
}
__device__ __forceinline__ void bulk_g2s_hint(uint32_t smem_dst, const void* gsrc, uint32_t bytes, uint32_t bar, uint64_t pol) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;"
                 ::"r"(smem_dst), "l"(gsrc), "r"(bytes), "r"(bar), "l"(pol)
                 : "memory");
}
__device__ __forceinline__ void bulk_prefetch_l2_hint(const void* gsrc, uint32_t bytes, uint64_t pol) {
    asm volatile("cp.async.bulk.prefetch.L2.global.L2::cache_hint [%0], %1, %2;" ::"l"(gsrc), "r"(bytes), "l"(pol) : "memory");
}
__device__ __forceinline__ void cp_async16_pred_hint(uint32_t smem_dst, const void* gsrc, bool pred, uint64_t pol) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "setp.ne.b32 p, %2, 0;\n\t"
        "@p cp.async.cg.shared.global.L2::cache_hint [%0], [%1], 16, %3;\n\t}"
        ::"r"(smem_dst), "l"(gsrc), "r"((uint32_t)pred), "l"(pol)
        : "memory");
}
// read-only loads that do not allocate in L1, and a store, with an L2 policy
__device__ __forceinline__ float2 ld_nc_na_hint(const float2* p, uint64_t pol) {
    float2 v;
    asm("ld.global.nc.L1::no_allocate.L2::cache_hint.v2.f32 {%0, %1}, [%2], %3;" : "=f"(v.x), "=f"(v.y) : "l"(p), "l"(pol));
    return v;
}
__device__ __forceinline__ float4 ld_nc_na_hint(const float4* p, uint64_t pol) {
    float4 v;
    asm("ld.global.nc.L1::no_allocate.L2::cache_hint.v4.f32 {%0, %1, %2, %3}, [%4], %5;"
                 : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(p), "l"(pol));
    return v;
}
__device__ __forceinline__ void st_hint(float2* p, float2 v, uint64_t pol) {
    asm volatile("st.global.L2::cache_hint.v2.f32 [%0], {%1, %2}, %3;" ::"l"(p), "f"(v.x), "f"(v.y), "l"(pol) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

// ---------------------------------------------------------------- fences and barriers
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async_all() { asm volatile("fence.proxy.async;" ::: "memory"); }
__device__ __forceinline__ void named_bar(int id, int nthreads) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory"); }

// ---------------------------------------------------------------- register reallocation
// setmaxnreg: sets the per-thread register count of the executing warpgroup (all four warps execute it).  dec returns
// registers to the CTA's pool; inc waits until the pool holds enough.  N is a multiple of 8 in [24, 256].
template <int N>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(N) : "memory"); }
template <int N>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(N) : "memory"); }

// ---------------------------------------------------------------- wgmma
// shared-memory matrix descriptor (sm_90): K-major, SWIZZLE_128B, 8-row groups 1024 B apart (SBO); the leading byte
// offset is unused for swizzled K-major operands.  A K step inside the 128-byte swizzle atom advances the start address
// by 32 bytes (the atom itself is 1024-byte aligned).
__device__ __forceinline__ uint64_t make_b_desc(uint32_t smem_addr) {
    uint64_t d = 0;
    d |= (uint64_t)((smem_addr >> 4) & 0x3FFF);          // start address
    d |= (uint64_t)1 << 16;                               // LBO (unused)
    d |= (uint64_t)(1024 >> 4) << 32;                     // SBO = 1024 B
    d |= (uint64_t)1 << 62;                               // SWIZZLE_128B
    return d;
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_wait_all() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }
// D[64 x 32] (+)= A[64 x 16] (bf16 register fragment) . B[16 x 32] (bf16, K-major shared memory), fp32 accumulate
__device__ __forceinline__ void wgmma_rs(float (&d)[16], const uint32_t (&a)[4], uint64_t b_desc, uint32_t accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "setp.ne.b32 p, %21, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, "
        "{%16, %17, %18, %19}, %20, p, 1, 1, 0;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b_desc), "r"(accumulate)
        : "memory");
}
// D[64 x 64] (+)= A[64 x 16] (bf16 register fragment) . B[16 x 64] (bf16, K-major shared memory), fp32 accumulate
__device__ __forceinline__ void wgmma_rs(float (&d)[32], const uint32_t (&a)[4], uint64_t b_desc, uint32_t accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "setp.ne.b32 p, %37, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, "
        "{%32, %33, %34, %35}, %36, p, 1, 1, 0;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
          "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
          "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b_desc), "r"(accumulate)
        : "memory");
}

// split fp32 values into NS bf16 terms of the running residual; pairs packed (first element low)
template <int NS>
__device__ __forceinline__ void split_pair(float a, float b, uint32_t (&parts)[NS]) {
#pragma unroll
    for (int p = 0; p < NS; ++p) {
        const __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
        parts[p] = *reinterpret_cast<const uint32_t*>(&h);
        if (p + 1 < NS) {
            const float2 f = __bfloat1622float2(h);
            a -= f.x; b -= f.y;                        // exact: the residual is representable in fp32
        }
    }
}

// byte offset of the bf16 element (row r, K index k) inside one bf16 term of a K-major SWIZZLE_128B tile of ROWS rows
// (what wgmma reads): 64-wide K blocks of ROWS 128-byte rows, 16-byte chunks XOR-swizzled by the row
template <int ROWS>
__device__ __forceinline__ uint32_t sw128_offset(int r, int k) {
    const int kb = k >> 6, col = k & 63;
    const int chunk = col >> 3;                            // 16-byte chunk in the 128-byte row
    return (uint32_t)(kb * (ROWS * 128) + r * 128 + (((chunk ^ (r & 7)) << 4) | ((col & 7) << 1)));
}

}  // namespace nerrf
