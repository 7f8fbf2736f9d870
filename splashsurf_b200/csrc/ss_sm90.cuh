// ss_sm90.cuh -- the sm_90a building blocks of the reconstruct path.
//
//  * FP32 pairs: the level-set folds handle two candidates / two grid points at a time as one `ss_f2` value.  Hopper has no
//    packed FP32 instruction, so each pair operation is two scalar IEEE-754 single operations rounded to nearest (FADD / FMUL /
//    FFMA) -- explicit intrinsics, never contracted or reassociated, so the results stay bit-identical to the reference.
//  * bulk asynchronous copies (TMA engine, 1-D form): cp.async.bulk.shared::cluster.global with mbarrier completion.  A run of
//    particle records is contiguous in HBM, so one elected lane moves a whole run with one instruction and no register
//    staging; the consumers wait on the mbarrier phase.
//
// Under SS_HOST_EMUL (tests/emul/cuda_emul.h: the CPU executor of the CUDA sources) the same entry points are plain C++.
#pragma once
#include <stdint.h>

// ------------------------------------------------------------------ FP32 pairs ----
struct ss_f2 { float lo, hi; };
__device__ __forceinline__ ss_f2 ss_pack(float lo, float hi) { return ss_f2{ lo, hi }; }
__device__ __forceinline__ void ss_unpack(ss_f2 v, float &lo, float &hi) { lo = v.lo; hi = v.hi; }
__device__ __forceinline__ ss_f2 ss_fma2(ss_f2 a, ss_f2 b, ss_f2 c) { return ss_f2{ __fmaf_rn(a.lo, b.lo, c.lo), __fmaf_rn(a.hi, b.hi, c.hi) }; }
__device__ __forceinline__ ss_f2 ss_add2(ss_f2 a, ss_f2 b) { return ss_f2{ __fadd_rn(a.lo, b.lo), __fadd_rn(a.hi, b.hi) }; }
__device__ __forceinline__ ss_f2 ss_mul2(ss_f2 a, ss_f2 b) { return ss_f2{ __fmul_rn(a.lo, b.lo), __fmul_rn(a.hi, b.hi) }; }

#ifndef SS_HOST_EMUL
// ------------------------------------------------------------------ mbarrier + bulk copy ----
__device__ __forceinline__ uint32_t ss_smem_addr(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void ss_mbar_init(unsigned long long *bar, uint32_t arrivals) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(ss_smem_addr(bar)), "r"(arrivals) : "memory");
}
// makes the initialised barrier visible to the async proxy (TMA engine)
__device__ __forceinline__ void ss_mbar_fence_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
// orders this thread's earlier generic-proxy accesses of shared memory before later async-proxy (bulk copy) accesses
__device__ __forceinline__ void ss_fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void ss_mbar_arrive_expect_tx(unsigned long long *bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(ss_smem_addr(bar)), "r"(bytes) : "memory");
}
// global -> shared bulk copy; dst, src and bytes must be multiples of 16
__device__ __forceinline__ void ss_bulk_g2s(void *dst_smem, const void *src_gmem, uint32_t bytes, unsigned long long *bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(ss_smem_addr(dst_smem)), "l"(src_gmem), "r"(bytes), "r"(ss_smem_addr(bar)) : "memory");
}
__device__ __forceinline__ void ss_mbar_wait(unsigned long long *bar, uint32_t parity) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "SS_MBAR_WAIT_%=:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra SS_MBAR_DONE_%=;\n"
        "bra SS_MBAR_WAIT_%=;\n"
        "SS_MBAR_DONE_%=:\n"
        "}\n" ::"r"(ss_smem_addr(bar)), "r"(parity) : "memory");
}

#else   // ------------------------------------------------------------------ CPU executor ----
// the copy happens at issue (a legal completion order); the barrier only checks the byte accounting of the caller
static inline void ss_mbar_init(unsigned long long *bar, uint32_t) { *bar = 0; }
static inline void ss_mbar_fence_init() {}
static inline void ss_fence_proxy_async() {}
static inline void ss_mbar_arrive_expect_tx(unsigned long long *bar, uint32_t bytes) { *bar += bytes; }
static inline void ss_bulk_g2s(void *dst, const void *src, uint32_t bytes, unsigned long long *bar) {
    if ((bytes & 15u) || ((uintptr_t)dst & 15u) || ((uintptr_t)src & 15u)) { fprintf(stderr, "emul: misaligned bulk copy (%p <- %p, %u bytes)\n", dst, src, bytes); abort(); }
    memcpy(dst, src, bytes);
    *bar -= bytes;
}
static inline void ss_mbar_wait(unsigned long long *bar, uint32_t) {
    if (*bar != 0) { fprintf(stderr, "emul: mbarrier wait with %lld bytes outstanding (expect_tx does not match the copies issued)\n", (long long)*bar); abort(); }
}
// the phase clocks of instrumented kernels count nanoseconds here
static inline long long clock64() { return (long long)std::chrono::duration_cast<std::chrono::nanoseconds>(std::chrono::steady_clock::now().time_since_epoch()).count(); }
#endif
