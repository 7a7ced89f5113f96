// device_utils.cuh — typed loads, bit-exact bin-index math and atomic cell updates (sm_90a).
#pragma once
#include "common.cuh"

namespace b200 {

// ---- streaming loads: the row columns are read exactly once, the grid must stay L2-resident ------
// ld.global.cs = evict-first; keeps the 8 GB column stream from pushing the grid out of the 50 MB L2.
__device__ __forceinline__ uint4 ldcs128(const void *p) { return __ldcs(reinterpret_cast<const uint4 *>(p)); }
__device__ __forceinline__ uint2 ldcs64(const void *p) { return __ldcs(reinterpret_cast<const uint2 *>(p)); }
__device__ __forceinline__ unsigned ldcs32(const void *p) { return __ldcs(reinterpret_cast<const unsigned *>(p)); }

__device__ __forceinline__ uint64_t bswap(uint64_t v, int isz) {
    switch (isz) {
    case 8: {
        uint32_t lo = (uint32_t)v, hi = (uint32_t)(v >> 32);
        return ((uint64_t)__byte_perm(lo, 0, 0x0123) << 32) | __byte_perm(hi, 0, 0x0123);
    }
    case 4: return __byte_perm((uint32_t)v, 0, 0x0123);
    case 2: return __byte_perm((uint32_t)v, 0, 0x4401) & 0xffffu;
    default: return v;
    }
}

// R consecutive rows (R = 4) of an `isz`-byte column as zero-extended raw bits.
// VEC: all column pointers are 16-byte aligned and base % 4 == 0, so one 128-bit (isz 4), two 128-bit
// (isz 8), one 64-bit (isz 2) or one 32-bit (isz 1) load covers the four rows.
template <bool VEC>
__device__ __forceinline__ void load4_raw(const void *data, int isz, long long base, int nv, uint64_t r[4]) {
    const char *p = static_cast<const char *>(data) + base * isz;
    if (VEC && nv == 4) {
        switch (isz) {
        case 8: {
            uint4 a = ldcs128(p), b = ldcs128(p + 16);
            r[0] = ((uint64_t)a.y << 32) | a.x;
            r[1] = ((uint64_t)a.w << 32) | a.z;
            r[2] = ((uint64_t)b.y << 32) | b.x;
            r[3] = ((uint64_t)b.w << 32) | b.z;
            break;
        }
        case 4: {
            uint4 a = ldcs128(p);
            r[0] = a.x, r[1] = a.y, r[2] = a.z, r[3] = a.w;
            break;
        }
        case 2: {
            uint2 a = ldcs64(p);
            r[0] = a.x & 0xffffu, r[1] = a.x >> 16, r[2] = a.y & 0xffffu, r[3] = a.y >> 16;
            break;
        }
        default: {
            unsigned a = ldcs32(p);
            r[0] = a & 0xffu, r[1] = (a >> 8) & 0xffu, r[2] = (a >> 16) & 0xffu, r[3] = a >> 24;
            break;
        }
        }
    } else {
#pragma unroll
        for (int j = 0; j < 4; j++) {
            r[j] = 0;
            if (j < nv) {
                switch (isz) {
                case 8: r[j] = __ldcs(reinterpret_cast<const unsigned long long *>(p) + j); break;
                case 4: r[j] = __ldcs(reinterpret_cast<const unsigned *>(p) + j); break;
                case 2: r[j] = __ldcs(reinterpret_cast<const unsigned short *>(p) + j); break;
                default: r[j] = __ldcs(reinterpret_cast<const unsigned char *>(p) + j); break;
                }
            }
        }
    }
}

// 4 mask bytes (VEC: one 32-bit load)
template <bool VEC>
__device__ __forceinline__ void load4_mask(const uint8_t *mask, long long base, int nv, unsigned m[4]) {
    if (VEC && nv == 4) {
        unsigned a = ldcs32(mask + base);
        m[0] = a & 0xffu, m[1] = (a >> 8) & 0xffu, m[2] = (a >> 16) & 0xffu, m[3] = a >> 24;
    } else {
#pragma unroll
        for (int j = 0; j < 4; j++)
            m[j] = j < nv ? __ldcs(mask + base + j) : 0u;
    }
}

// ---- raw bits -> value ---------------------------------------------------------------------------
__device__ __forceinline__ bool raw_isnan(int dt, uint64_t r) {
    if (dt == B200_F64)
        return (r & 0x7fffffffffffffffULL) > 0x7ff0000000000000ULL;
    if (dt == B200_F32)
        return ((uint32_t)r & 0x7fffffffu) > 0x7f800000u;
    return false;
}
// `double value_double = value` (src/binners.cpp:25): exact for every type but (u)int64 (round-to-nearest-even)
__device__ __forceinline__ double raw_to_double(int dt, uint64_t r) {
    switch (dt) {
    case B200_F64: return __longlong_as_double((long long)r);
    case B200_F32: return (double)__uint_as_float((uint32_t)r);
    case B200_I64: return __ll2double_rn((long long)r);
    case B200_I32: return (double)(int32_t)(uint32_t)r;
    case B200_I16: return (double)(int16_t)(uint16_t)r;
    case B200_I8: return (double)(int8_t)(uint8_t)r;
    case B200_U64: return __ull2double_rn(r);
    default: return (double)(uint32_t)r; // u32/u16/u8/bool: zero-extended already
    }
}
// integer types -> sign/zero-extended 64-bit pattern
__device__ __forceinline__ uint64_t raw_to_i64bits(int dt, uint64_t r) {
    switch (dt) {
    case B200_I32: return (uint64_t)(int64_t)(int32_t)(uint32_t)r;
    case B200_I16: return (uint64_t)(int64_t)(int16_t)(uint16_t)r;
    case B200_I8: return (uint64_t)(int64_t)(int8_t)(uint8_t)r;
    default: return r;
    }
}
// x86 cvttsd2si semantics (what the reference binary does for float -> int64): NaN / out of range -> INT64_MIN
__device__ __forceinline__ long long f64_to_i64_x86(double x) {
    if (!(x == x) || x >= 9223372036854775808.0 || x < -9223372036854775808.0)
        return (long long)0x8000000000000000ULL;
    return __double2ll_rz(x);
}
// gcc's x86-64 double -> uint64 sequence: below 2^63 cvttsd2si as above, else cvttsd2si(x - 2^63) ^ 2^63; so >= 2^64 -> 0
__device__ __forceinline__ unsigned long long f64_to_u64_x86(double x) {
    if (x >= 9223372036854775808.0)
        return (unsigned long long)f64_to_i64_x86(x - 9223372036854775808.0) ^ 0x8000000000000000ULL;
    return (unsigned long long)f64_to_i64_x86(x);
}

// ---- BinnerScalar::to_bins, bit-exact (src/binners.cpp:13-57) -------------------------------------
// scaled = (double(v) - vmin) * scale_v, scale_v = 1./(vmax-vmin) precomputed on the host in IEEE double.
// __dsub_rn/__dmul_rn are never contracted into FMA, matching the reference build (x86-64 baseline, no FMA).
__device__ __forceinline__ unsigned long long scalar_index(double v, bool masked, double vmin, double scale, double bins_d, unsigned long long bins) {
    double scaled = __dmul_rn(__dsub_rn(v, vmin), scale);
    if (scaled != scaled || masked)
        return 0ull;
    if (scaled < 0.0)
        return 1ull;
    if (scaled >= 1.0)
        return bins + 2ull;
    return (unsigned long long)(long long)(__double2int_rz(__dmul_rn(scaled, bins_d)) + 2);
}

// The ONE branch-free form every specialised float kernel (fast.cu, ringcount.cu, tilesort.cu) uses; bit-identical to
// scalar_index above for unmasked rows (tests/test_gpu_parity.py::test_bin_edges_bit_exact, test_bin_index_sweep_all_fp32).
// Reference: nan -> 0; scaled < 0 -> 1; scaled >= 1 -> bins+2; else (int)(scaled*bins)+2.
// With t = RN(scaled*bins): scaled < 0 <=> t < 0 and scaled >= 1 <=> t >= bins (RN is monotone, and for scaled < 1 the
// product rounds to at most `bins`, which lands in the same cell bins+2), and floor(t) == trunc(t) on [0, bins).  So ONE
// saturating round-down conversion + an integer clamp reproduce the three range branches; only NaN needs its own test.
// Returns cell - 1 in [-1, bins+1] so that callers fold the "+1" into the constant sum(stride):
//   clamp(i, -1, bins) + 1 == max(min(i, bins) + 1, 0): VIMNMX + VIADDMNMX (DPX), no overflow (min first).
__device__ __forceinline__ int bin_cell_m1(double v, double vmin, double scale, double bins_d, unsigned bins) {
    const double scaled = __dmul_rn(__dsub_rn(v, vmin), scale);
    const int i = __double2int_rd(__dmul_rn(scaled, bins_d)); // saturates; NaN -> 0 (fixed up below)
    const int c = __viaddmax_s32(min(i, (int)bins), 1, 0);
    return scaled != scaled ? -1 : c;
}
__device__ __forceinline__ unsigned bin_index(double v, double vmin, double scale, double bins_d, unsigned bins) {
    return (unsigned)(bin_cell_m1(v, vmin, scale, bins_d, bins) + 1);
}

// ---- BinnerOrdinal::to_bins (src/binner_ordinal.cpp:20-176) ---------------------------------------
__device__ __forceinline__ long long ordinal_value(int dt, uint64_t r, long long min_value, bool flip) {
    long long value;
    switch (dt) {
    case B200_F64: value = f64_to_i64_x86(__dsub_rn(__longlong_as_double((long long)r), __ll2double_rn(min_value))); break;
    case B200_F32: value = f64_to_i64_x86((double)__fsub_rn(__uint_as_float((uint32_t)r), __ll2float_rn(min_value))); break;
    default: value = (long long)(raw_to_i64bits(dt, r) - (uint64_t)min_value); break;
    }
    if (flip) // FlipEndian quirk: the flip is applied to the int64 difference (:28-30)
        value = (long long)bswap((uint64_t)value, 8);
    return value;
}
__device__ __forceinline__ unsigned long long ordinal_index(long long value, bool masked, long long n, bool allow_other, bool invert) {
    bool oob = value < 0 || value >= n;
    if (allow_other) {
        if (masked)
            return (unsigned long long)(n + 1);
        if (oob)
            return (unsigned long long)n;
    } else if (masked || oob) {
        return (unsigned long long)n;
    }
    return (unsigned long long)(invert ? n - 1 - value : value);
}

// ---- atomic cell updates -------------------------------------------------------------------------
// float max/min on raw IEEE storage with integer atomics: non-negative floats order like signed ints,
// negative floats order inversely as unsigned ints.  Works with the +-inf initial fill and is order independent.
__device__ __forceinline__ void atomic_max_f32(float *addr, float v) {
    if (!(__float_as_uint(v) >> 31))
        atomicMax(reinterpret_cast<int *>(addr), __float_as_int(v));
    else
        atomicMin(reinterpret_cast<unsigned *>(addr), __float_as_uint(v));
}
__device__ __forceinline__ void atomic_min_f32(float *addr, float v) {
    if (!(__float_as_uint(v) >> 31))
        atomicMin(reinterpret_cast<int *>(addr), __float_as_int(v));
    else
        atomicMax(reinterpret_cast<unsigned *>(addr), __float_as_uint(v));
}
__device__ __forceinline__ void atomic_max_f64(double *addr, double v) {
    unsigned long long b = (unsigned long long)__double_as_longlong(v);
    if (!(b >> 63))
        atomicMax(reinterpret_cast<long long *>(addr), (long long)b);
    else
        atomicMin(reinterpret_cast<unsigned long long *>(addr), b);
}
__device__ __forceinline__ void atomic_min_f64(double *addr, double v) {
    unsigned long long b = (unsigned long long)__double_as_longlong(v);
    if (!(b >> 63))
        atomicMin(reinterpret_cast<long long *>(addr), (long long)b);
    else
        atomicMax(reinterpret_cast<unsigned long long *>(addr), b);
}

// pow(b, moment) for the small integer moments vaex uses (var/skew/kurtosis: 1..4); generic pow otherwise
__device__ __forceinline__ double pow_moment(double b, unsigned m) {
    switch (m) {
    case 0: return 1.0;
    case 1: return b;
    case 2: return b * b;
    case 3: return b * b * b;
    case 4: {
        double b2 = b * b;
        return b2 * b2;
    }
    default: return pow(b, (double)m);
    }
}
// the same for integer grids, where the power is truncated to an integer: for m >= 5 repeated multiplication instead of pow
// (pow may be 2 ulp off), exact while |b|^m < 2^53
__device__ __forceinline__ double pow_moment_int(double b, unsigned m) {
    if (m <= 4)
        return pow_moment(b, m);
    double r = b;
    for (unsigned i = 1; i < m; i++)
        r *= b;
    return r;
}

// splitmix64 finaliser (src/hash.hpp:40-45)
__host__ __device__ __forceinline__ uint64_t hash64(uint64_t x) {
    x = (x ^ (x >> 30)) * 0xbf58476d1ce4e5b9ULL;
    x = (x ^ (x >> 27)) * 0x94d049bb133111ebULL;
    x = x ^ (x >> 31);
    return x;
}
// key widening per type (src/hash.hpp:50-152): raw zero-extended bits -> canonical 64-bit key pattern
__host__ __device__ __forceinline__ uint64_t key_canon(int dt, uint64_t r) {
    switch (dt) {
    case B200_I32: return (uint64_t)(int64_t)(int32_t)(uint32_t)r;
    case B200_I16: return (uint64_t)(int64_t)(int16_t)(uint16_t)r;
    case B200_I8: return (uint64_t)(int64_t)(int8_t)(uint8_t)r;
    default: return r;
    }
}
// hash of the canonical pattern: 8/16-bit ints and bool use std::hash identity in the reference
__host__ __device__ __forceinline__ uint64_t key_hash(int dt, uint64_t canon) {
    switch (dt) {
    case B200_I16:
    case B200_I8:
    case B200_U16:
    case B200_U8:
    case B200_BOOL: return canon;
    default: return hash64(canon);
    }
}

} // namespace b200
