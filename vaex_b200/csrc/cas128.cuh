// cas128.cuh — 16-byte pairs updated with one 128-bit compare-and-swap (atom.global.cas.b128, sm_90+): the (order key, global row)
// state of first.cu and statistic.cu's FIRST, and the (cell, value) slots of nunique.cu's table.
#pragma once
#include "common.cuh"

namespace b200 {

struct U128 {
    unsigned long long lo, hi;
};

// one 16-byte L2 load (never served from L1): the pair is read consistently enough for the CAS to validate
__device__ __forceinline__ U128 load128(const unsigned long long *p) {
    U128 v;
    asm volatile("ld.global.cg.v2.u64 {%0, %1}, [%2];" : "=l"(v.lo), "=l"(v.hi) : "l"(p) : "memory");
    return v;
}

__device__ __forceinline__ U128 cas128(unsigned long long *addr, U128 cmp, U128 val) {
    U128 old;
    asm volatile("{\n\t"
                 ".reg .b128 d, b, c;\n\t"
                 "mov.b128 b, {%2, %3};\n\t"
                 "mov.b128 c, {%4, %5};\n\t"
                 "atom.global.cas.b128 d, [%6], b, c;\n\t"
                 "mov.b128 {%0, %1}, d;\n\t"
                 "}"
                 : "=l"(old.lo), "=l"(old.hi)
                 : "l"(cmp.lo), "l"(cmp.hi), "l"(val.lo), "l"(val.hi), "l"(addr)
                 : "memory");
    return old;
}

__device__ __forceinline__ bool less128(const U128 &a, const U128 &b) { return a.lo < b.lo || (a.lo == b.lo && a.hi < b.hi); }

// lower the pair at `st` to `kr` when `kr` is lexicographically smaller
__device__ __forceinline__ void cas128_min(unsigned long long *st, U128 kr) {
    U128 cur = load128(st);
    while (less128(kr, cur)) {
        const U128 old = cas128(st, cur, kr);
        if (old.lo == cur.lo && old.hi == cur.hi)
            break;
        cur = old;
    }
}

// monotone map of a double to u64 so that `<` on doubles is `<` on keys; -0.0 == +0.0
__device__ __forceinline__ unsigned long long order_key_f64(double d) {
    if (d == 0.0)
        d = 0.0;
    const unsigned long long b = (unsigned long long)__double_as_longlong(d);
    return (b >> 63) ? ~b : (b | 0x8000000000000000ULL);
}

} // namespace b200
