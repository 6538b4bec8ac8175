// rl_devmem.cuh — the few global-memory primitives the maintenance and CRDT kernels use, in two forms: the real ones
// (ld.global.cg / st.global.cg / atom.cas.b128, as in rl_kernels.cuh) and plain host ones for tests/emu/cuda_shim.h
// (RL_SHIM: one thread after the other) and tests/emu/cuda_simt.h (RL_SIMT: fibers; the kernels' warp-level branches run).
#pragma once
#include <stdint.h>

#if !defined(RL_SHIM) && !defined(RL_SIMT)
__device__ __forceinline__ ulonglong2 rlm_ld(const void* p) { return __ldcg(reinterpret_cast<const ulonglong2*>(p)); }
__device__ __forceinline__ void rlm_st(void* p, unsigned long long a, unsigned long long b) {
    __stcg(reinterpret_cast<ulonglong2*>(p), make_ulonglong2(a, b));
}
// 128-bit compare-and-swap (PTX atom.cas.b128, sm_90+) — the instruction the hot path claims rows with
__device__ __forceinline__ ulonglong2 rlm_cas128(void* addr, ulonglong2 cmp, ulonglong2 val) {
    ulonglong2 old;
    asm volatile(
        "{\n\t"
        ".reg .b128 c, v, o;\n\t"
        "mov.b128 c, {%3, %4};\n\t"
        "mov.b128 v, {%5, %6};\n\t"
        "atom.global.cas.b128 o, [%2], c, v;\n\t"
        "mov.b128 {%0, %1}, o;\n\t"
        "}\n"
        : "=l"(old.x), "=l"(old.y)
        : "l"(addr), "l"(cmp.x), "l"(cmp.y), "l"(val.x), "l"(val.y)
        : "memory");
    return old;
}
#else
inline ulonglong2 rlm_ld(const void* p) { return *reinterpret_cast<const ulonglong2*>(p); }
inline void rlm_st(void* p, unsigned long long a, unsigned long long b) { *reinterpret_cast<ulonglong2*>(p) = make_ulonglong2(a, b); }
inline ulonglong2 rlm_cas128(void* addr, ulonglong2 cmp, ulonglong2 val) {
    ulonglong2* p = reinterpret_cast<ulonglong2*>(addr);
    const ulonglong2 old = *p;
    if (old.x == cmp.x && old.y == cmp.y) *p = val;
    return old;
}
#endif

// 64-bit load that bypasses L1 (other threads' atomics on the word are visible)
#if !defined(RL_SHIM) && !defined(RL_SIMT)
__device__ __forceinline__ unsigned long long rlm_ld64(const void* p) { return __ldcg(reinterpret_cast<const unsigned long long*>(p)); }
#else
inline unsigned long long rlm_ld64(const void* p) { return *reinterpret_cast<const unsigned long long*>(p); }
#endif

// atomic OR of a 32-bit word; returns the old value
#if !defined(RL_SHIM) && !defined(RL_SIMT)
__device__ __forceinline__ unsigned rlm_or(unsigned* p, unsigned v) { return atomicOr(p, v); }
#else
inline unsigned rlm_or(unsigned* p, unsigned v) {
    const unsigned o = *p;
    *p = o | v;
    return o;
}
#endif
