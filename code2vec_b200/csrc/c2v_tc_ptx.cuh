// c2v_tc_ptx.cuh -- raw PTX wrappers shared by the sm_90a tensor-core kernels: mbarrier, proxy fences,
// cp.async.bulk (TMA), wgmma (warpgroup MMA) and its shared-memory matrix descriptors.
#pragma once
#include <cuda_fp16.h>

#include <type_traits>

#include "c2v_common.cuh"

#ifndef C2V_SPIN_NS
#define C2V_SPIN_NS 64
#endif

namespace c2v {

// Passes of the fp16 tensor-core GEMMs, the last template argument of every kernel that has both (named types, so that
// profiles tell the instantiations apart).  ThreePass (the default): both operands split into fp16 hi + lo, three MMAs
// per k-step, hi.hi + lo.hi + hi.lo, fp32-accurate.  OnePass (C2V_MATMUL_TF32): hi.hi only -- 10 explicit mantissa bits
// per operand, TF32-class -- with the lo halves neither converted, loaded nor multiplied.
struct ThreePass {};
struct OnePass {};
template <class P> constexpr bool one_pass = std::is_same<P, OnePass>::value;

// ------------------------------------------------------------------------------------
// PTX wrappers
// ------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint32_t bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
// Wait for the phase with the given parity; a watchdog turns a protocol bug into a trap instead of a hung GPU.
// A bare try_wait returns after ~30 cycles, so a waiting warp re-polls ~30x per microsecond and takes issue slots from
// the warps that have work: a short nanosleep between polls (C2V_SPIN_NS) keeps the wake-up latency low.
#ifndef C2V_WAIT_HINT_NS
#define C2V_WAIT_HINT_NS 0
#endif
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity, long long *status) {
    uint32_t ok = 0;
    long long t0 = 0;
    for (uint32_t spins = 0;; ++spins) {
#if C2V_WAIT_HINT_NS > 0
        asm volatile("{\n\t.reg .pred p;\n\t"
                     "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2, %3;\n\t"
                     "selp.u32 %0, 1, 0, p;\n\t}"
                     : "=r"(ok) : "r"(bar), "r"(parity), "r"((uint32_t)C2V_WAIT_HINT_NS) : "memory");
#else
        asm volatile("{\n\t.reg .pred p;\n\t"
                     "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
                     "selp.u32 %0, 1, 0, p;\n\t}"
                     : "=r"(ok) : "r"(bar), "r"(parity) : "memory");
#endif
        if (ok) break;
#if C2V_SPIN_NS > 0
        __nanosleep(C2V_SPIN_NS);
#endif
#ifndef C2V_NO_WATCHDOG                               // (compute-sanitizer slows kernels 100x: build the variant without it)
        if ((spins & 0x3ff) == 0x3ff) {
            const long long now = clock64();
            if (t0 == 0) t0 = now;
            else if (now - t0 > 4000000000LL) {           // ~2 s: certainly a deadlock
                status[1] = 0xDEAD0000LL | (long long)(bar & 0xffff);
                __threadfence();
                __trap();
            }
        }
#endif
    }
}
__device__ __forceinline__ bool elect_one() {
    uint32_t pred;
    asm volatile("{\n\t.reg .pred P;\n\telect.sync _|P, 0xffffffff;\n\tselp.u32 %0, 1, 0, P;\n\t}" : "=r"(pred));
    return pred != 0;
}
__device__ __forceinline__ void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void bulk_copy_g2s(uint32_t dst, const void *src, uint32_t bytes, uint32_t bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(dst), "l"(src), "r"(bytes), "r"(bar) : "memory");
}

// K-major 128-byte-swizzled shared-memory matrix descriptor of wgmma (Hopper GMMA descriptor):
// start>>4 [0,14) | LBO>>4 [16,30) (unused for swizzled K-major, 1) | SBO>>4 [32,46) = 1024 B (stride between 8-row
// groups) | base offset [49,52) = 0 (tiles are 1024-B aligned) | layout [62,64) = 1 (SWIZZLE_128B).  The k-steps of a
// 64-wide k-block advance the start address by 32 B inside the swizzle atom.
__device__ __forceinline__ uint64_t wgmma_desc(uint32_t saddr) {
    return (uint64_t)((saddr & 0x3FFFFu) >> 4) | (1ull << 16) | ((uint64_t)(1024 >> 4) << 32) | (1ull << 62);
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from moving accesses to an accumulator register across the asynchronous MMA that writes it
__device__ __forceinline__ void fence_operand(float &r) { asm volatile("" : "+f"(r)::"memory"); }
// d[O .. O+63] (+)= A[64 x 16] . B[128 x 16]^T, both fp16 K-major in shared memory, fp32 accumulation (one warpgroup)
template <int O, int N>
__device__ __forceinline__ void wgmma_m64n128(float (&d)[N], uint64_t adesc, uint64_t bdesc, int scale_d) {
    static_assert(O + 64 <= N, "accumulator fragment");
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 "
                 "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, 0, 0;\n\t}"
                 : "+f"(d[O + 0]), "+f"(d[O + 1]), "+f"(d[O + 2]), "+f"(d[O + 3]), "+f"(d[O + 4]), "+f"(d[O + 5]), "+f"(d[O + 6]), "+f"(d[O + 7]), "+f"(d[O + 8]), "+f"(d[O + 9]), "+f"(d[O + 10]), "+f"(d[O + 11]), "+f"(d[O + 12]), "+f"(d[O + 13]), "+f"(d[O + 14]), "+f"(d[O + 15]), "+f"(d[O + 16]), "+f"(d[O + 17]), "+f"(d[O + 18]), "+f"(d[O + 19]), "+f"(d[O + 20]), "+f"(d[O + 21]), "+f"(d[O + 22]), "+f"(d[O + 23]), "+f"(d[O + 24]), "+f"(d[O + 25]), "+f"(d[O + 26]), "+f"(d[O + 27]), "+f"(d[O + 28]), "+f"(d[O + 29]), "+f"(d[O + 30]), "+f"(d[O + 31]), "+f"(d[O + 32]), "+f"(d[O + 33]), "+f"(d[O + 34]), "+f"(d[O + 35]), "+f"(d[O + 36]), "+f"(d[O + 37]), "+f"(d[O + 38]), "+f"(d[O + 39]), "+f"(d[O + 40]), "+f"(d[O + 41]), "+f"(d[O + 42]), "+f"(d[O + 43]), "+f"(d[O + 44]), "+f"(d[O + 45]), "+f"(d[O + 46]), "+f"(d[O + 47]), "+f"(d[O + 48]), "+f"(d[O + 49]), "+f"(d[O + 50]), "+f"(d[O + 51]), "+f"(d[O + 52]), "+f"(d[O + 53]), "+f"(d[O + 54]), "+f"(d[O + 55]), "+f"(d[O + 56]), "+f"(d[O + 57]), "+f"(d[O + 58]), "+f"(d[O + 59]), "+f"(d[O + 60]), "+f"(d[O + 61]), "+f"(d[O + 62]), "+f"(d[O + 63])
                 : "l"(adesc), "l"(bdesc), "r"(scale_d));
}
// d (+)= A[64 x 16] . B[64 x 16]^T, fp16 in shared memory, fp32 accumulation (one warpgroup).  TA / TB = 1: the operand is
// MN-major (the 64 M / N elements of one k are contiguous), described by wgmma_desc_mn
template <int TA, int TB>
__device__ __forceinline__ void wgmma_m64n64(float (&d)[32], uint64_t adesc, uint64_t bdesc, int scale_d) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 "
                 "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, %35, %36;\n\t}"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
                 : "l"(adesc), "l"(bdesc), "r"(scale_d), "n"(TA), "n"(TB));
}
// MN-major 128-byte-swizzled descriptor: LBO = byte stride between 64-element MN groups, SBO = 1024 B between 8-row K
// groups; a k-step of 16 rows advances the start address by 2 KB
__device__ __forceinline__ uint64_t wgmma_desc_mn(uint32_t saddr, uint32_t lbo_bytes) {
    return (uint64_t)((saddr & 0x3FFFFu) >> 4) | ((uint64_t)(lbo_bytes >> 4) << 16) | ((uint64_t)(1024 >> 4) << 32) | (1ull << 62);
}
__device__ __forceinline__ void red_add_v2(float *addr, float x, float y) {
    asm volatile("red.relaxed.gpu.global.add.v2.f32 [%0], {%1, %2};" ::"l"(addr), "f"(x), "f"(y) : "memory");
}
__device__ __forceinline__ float4 ldg_nc_v4(const float4 *p) {
    float4 v;
    asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0, %1, %2, %3}, [%4];"
                 : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(p));
    return v;
}
__device__ __forceinline__ void sts_v2(uint32_t addr, uint32_t a, uint32_t b) {
    asm volatile("st.shared.v2.b32 [%0], {%1, %2};" ::"r"(addr), "r"(a), "r"(b) : "memory");
}
__device__ __forceinline__ uint32_t pack_h2(__half2 h) { return *reinterpret_cast<uint32_t *>(&h); }

// byte offset of fp16 element (row, k) inside a [rows x 64] K-major SWIZZLE_128B tile
__host__ __device__ __forceinline__ uint32_t sw128_offset(int row, int k) {
    return (uint32_t)((row >> 3) * 1024 + (row & 7) * 128 + ((((k >> 3) ^ (row & 7)) & 7) << 4) + (k & 7) * 2);
}

// In-place transpose-reduce across the 32 lanes of a warp: on entry lane i holds v[0..31]
// (32 columns of its row); on exit v[0] of lane i is the sum over all 32 lanes of column i.
// 31 shuffles instead of 32 x 5.
__device__ __forceinline__ void butterfly_reduce32(float (&v)[32], int lane) {
#pragma unroll
    for (int off = 16; off >= 1; off >>= 1) {
        const bool upper = (lane & off) != 0;
#pragma unroll
        for (int j = 0; j < off; ++j) {
            const float send = upper ? v[j] : v[j + off];
            const float keep = upper ? v[j + off] : v[j];
            v[j] = keep + __shfl_xor_sync(0xffffffffu, send, off);
        }
    }
}

__device__ __forceinline__ float rcp_approx(float x) {
    float r;
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
    return r;
}
__device__ __forceinline__ float ex2_approx(float x) {
    float r;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
    return r;
}
// tanh(v) given w = 2*log2(e)*v :  1 - 2/(2^w + 1); 2^w = inf -> 1, 2^w = 0 -> -1.  Two MUFU ops,
// absolute error ~2e-7 (same formula as tanh_accurate, constants folded into gamma/beta).
__device__ __forceinline__ float tanh_from_scaled(float w) {
    return fmaf(-2.0f, rcp_approx(ex2_approx(w) + 1.0f), 1.0f);
}
__device__ __forceinline__ void named_bar_sync(int id, int nthreads) {
    asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}


}  // namespace c2v
