// device_utils.cuh — typed loads, bit-exact bin-index math and atomic cell updates (sm_90a).
#pragma once
#include "common.cuh"

namespace b200 {

// ---- streaming loads: the row columns are read exactly once, the grid must stay L2-resident ------
// ld.global.cs = evict-first; keeps the 8 GB column stream from pushing the grid out of the 50 MB L2.
__device__ __forceinline__ uint4 ldcs128(const void *p) { return __ldcs(reinterpret_cast<const uint4 *>(p)); }
__device__ __forceinline__ uint2 ldcs64(const void *p) { return __ldcs(reinterpret_cast<const uint2 *>(p)); }
__device__ __forceinline__ unsigned ldcs32(const void *p) { return __ldcs(reinterpret_cast<const unsigned *>(p)); }

// 4 consecutive elements of a float / double column from element i (16-byte aligned): one or two 128-bit loads
template <typename T>
__device__ __forceinline__ void ldcs4(const void *p, long long i, T out[4]);
template <>
__device__ __forceinline__ void ldcs4<float>(const void *p, long long i, float out[4]) {
    const uint4 a = ldcs128(static_cast<const float *>(p) + i);
    out[0] = __uint_as_float(a.x), out[1] = __uint_as_float(a.y), out[2] = __uint_as_float(a.z), out[3] = __uint_as_float(a.w);
}
template <>
__device__ __forceinline__ void ldcs4<double>(const void *p, long long i, double out[4]) {
    const uint4 *q = reinterpret_cast<const uint4 *>(static_cast<const double *>(p) + i);
    const uint4 a = __ldcs(q), b = __ldcs(q + 1);
    out[0] = __longlong_as_double(((long long)a.y << 32) | a.x), out[1] = __longlong_as_double(((long long)a.w << 32) | a.z);
    out[2] = __longlong_as_double(((long long)b.y << 32) | b.x), out[3] = __longlong_as_double(((long long)b.w << 32) | b.z);
}

// ---- one element of an `isz`-byte (1, 2, 4 or 8) array as zero-extended raw bits -------------------------------------------------
// ldcs1_raw is for the row columns above (read once, evict-first); load1_raw is a plain load for data that is read through an
// index, read again or worth keeping in L2.
__device__ __forceinline__ uint64_t load1_raw(const void *p, int isz, long long i) {
    switch (isz) {
    case 8: return static_cast<const unsigned long long *>(p)[i];
    case 4: return static_cast<const unsigned *>(p)[i];
    case 2: return static_cast<const unsigned short *>(p)[i];
    default: return static_cast<const unsigned char *>(p)[i];
    }
}
__device__ __forceinline__ uint64_t ldcs1_raw(const void *p, int isz, long long i) {
    switch (isz) {
    case 8: return __ldcs(static_cast<const unsigned long long *>(p) + i);
    case 4: return __ldcs(static_cast<const unsigned *>(p) + i);
    case 2: return __ldcs(static_cast<const unsigned short *>(p) + i);
    default: return __ldcs(static_cast<const unsigned char *>(p) + i);
    }
}
// the low `isz` bytes of v
__host__ __device__ __forceinline__ void store1_raw(void *p, int isz, long long i, uint64_t v) {
    switch (isz) {
    case 8: static_cast<unsigned long long *>(p)[i] = v; break;
    case 4: static_cast<unsigned *>(p)[i] = (unsigned)v; break;
    case 2: static_cast<unsigned short *>(p)[i] = (unsigned short)v; break;
    default: static_cast<unsigned char *>(p)[i] = (unsigned char)v; break;
    }
}

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
// the 32-bit cvttsd2si (numpy's float -> int8/int16/int32/uint8/uint16 loops go through it): NaN / out of range -> INT32_MIN
__device__ __forceinline__ int f64_to_i32_x86(double x) {
    if (!(x == x) || x >= 2147483648.0 || x < -2147483648.0)
        return (int)0x80000000u;
    return __double2int_rz(x);
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

// ---- BinnerTime: numpy's datetime64 astype('M8[R]') on raw int64 ticks (B200_BINNER_TIME) ---------------------------------------
// floor(n / d) for a divisor d >= 1 known only at run time, without a 64-bit division per row: for 0 <= u < 2^63,
// floor(u / d) = umulhi(u, magic) >> shift with l = ceil(log2 d), magic = ceil(2^(63 + l) / d) (< 2^64), shift = l - 1 (the error
// of magic / 2^(63 + l) against 1 / d is below 2^-l / 2^63, too small to carry u / d over the next integer).  magic = 0: d = 1.
struct Divisor {
    unsigned long long magic;
    int shift;
};
inline Divisor make_divisor(unsigned long long d) {
    Divisor v{0, 0};
    if (d <= 1)
        return v;
    int l = 0;
    while (l < 64 && (1ull << l) < d)
        l++;
    const unsigned __int128 num = (unsigned __int128)1 << (63 + l);
    v.magic = (unsigned long long)((num + d - 1) / d);
    v.shift = l - 1;
    return v;
}
// floor division towards -inf: with s = n >> 63 (all ones for n < 0), n ^ s = -n - 1 >= 0 and floor(n / d) = ~floor((-n - 1) / d)
__device__ __forceinline__ long long floor_div(long long n, const Divisor &d) {
    const unsigned long long s = (unsigned long long)(n >> 63), u = (unsigned long long)n ^ s;
    const unsigned long long q = d.magic ? __umul64hi(u, d.magic) >> d.shift : u;
    return (long long)(q ^ s);
}
// the same for a compile-time divisor (the compiler's own multiply-high)
template <unsigned long long D>
__device__ __forceinline__ long long floor_div(long long n) {
    const unsigned long long s = (unsigned long long)(n >> 63);
    return (long long)((((unsigned long long)n ^ s) / D) ^ s);
}

// days since 1970-01-01 <-> proleptic Gregorian (year, month), 400-year eras of 146097 days counted from 0000-03-01
__device__ __forceinline__ long long days_from_months(long long months) { // months since 1970-01 -> day of the month's first day
    const long long yq = floor_div<12>(months);
    const unsigned m = (unsigned)(months - yq * 12);     // 0 = January
    const long long y = yq + 1970 - (m < 2);             // March-based year
    const long long era = floor_div<400>(y);
    const unsigned yoe = (unsigned)(y - era * 400);      // [0, 399]
    const unsigned mp = m < 2 ? m + 10 : m - 2;          // 0 = March
    const unsigned doe = yoe * 365 + yoe / 4 - yoe / 100 + (153 * mp + 2) / 5;
    return era * 146097 + (long long)doe - 719468;
}
__device__ __forceinline__ long long months_from_days(long long days, bool years) { // -> months (or years) since 1970
    const long long q = floor_div<146097>(days); // days + 719468 could overflow: shift the remainder instead
    const unsigned z = (unsigned)(days - q * 146097) + 719468;
    const long long era = q + z / 146097;
    const unsigned doe = z % 146097;                                              // [0, 146096]
    const unsigned yoe = (doe - doe / 1460 + doe / 36524 - doe / 146096) / 365;   // [0, 399]
    const unsigned doy = doe - (365 * yoe + yoe / 4 - yoe / 100);                 // [0, 365], from March 1
    const unsigned mp = (5 * doy + 2) / 153;                                      // 0 = March
    const long long y = era * 400 + yoe + (mp >= 10) - 1970;
    return years ? y : y * 12 + (mp < 10 ? mp + 2 : mp - 10);
}

// How a unit U becomes a resolution R.  Linear units (W .. ns) scale by one factor: p = floor(t * mul / div), one of mul, div 1.
// CIVIL_IN (U = Y or M, R linear): t is first turned into the day its period starts on; CIVIL_OUT (U linear, R = M or Y): the
// day count t * mul / div is turned into months or years.  Y <-> M is linear (x 12).  Multiplication wraps, as numpy's does.
enum { TIME_CIVIL_IN = 1, TIME_CIVIL_OUT = 2, TIME_YEARS = 4 };
struct TimeSteps {
    int mode;
    unsigned long long mul;
    Divisor div;
};
// unit and resolution: b200_time_unit codes, both valid
inline TimeSteps time_steps(int unit, int res) {
    // nanoseconds per tick of W .. ns; Y and M have none
    static const unsigned long long ns[B200_TIME_NUNITS] = {0, 0, 604800000000000ull, 86400000000000ull, 3600000000000ull, 60000000000ull,
                                                           1000000000ull, 1000000ull, 1000ull, 1ull};
    const bool civil_u = unit <= B200_TIME_M, civil_r = res <= B200_TIME_M;
    TimeSteps s{0, 1, make_divisor(1)};
    unsigned long long from, to;
    if (civil_u && civil_r) { // months <-> years
        from = unit == B200_TIME_Y ? 12 : 1;
        to = res == B200_TIME_Y ? 12 : 1;
    } else {
        s.mode = civil_u ? TIME_CIVIL_IN | (unit == B200_TIME_Y ? TIME_YEARS : 0) : civil_r ? TIME_CIVIL_OUT | (res == B200_TIME_Y ? TIME_YEARS : 0) : 0;
        from = ns[civil_u ? B200_TIME_D : unit];
        to = ns[civil_r ? B200_TIME_D : res];
    }
    if (to >= from)
        s.div = make_divisor(to / from);
    else
        s.mul = from / to;
    return s;
}
__device__ __forceinline__ long long time_period(long long t, const TimeSteps &s) {
    if (s.mode & TIME_CIVIL_IN)
        t = days_from_months((s.mode & TIME_YEARS) ? (long long)((unsigned long long)t * 12) : t);
    long long p = floor_div((long long)((unsigned long long)t * s.mul), s.div);
    if (s.mode & TIME_CIVIL_OUT)
        p = months_from_days(p, (s.mode & TIME_YEARS) != 0);
    return p;
}
// the bin of one row: NaT and masked rows give -1 (the null cell through ordinal_index), like the reference's NaT // every
__device__ __forceinline__ long long time_bin(long long t, bool masked, const TimeSteps &s, long long begin, const Divisor &every) {
    if (masked || t == (long long)0x8000000000000000ULL)
        return -1;
    return floor_div((long long)((unsigned long long)time_period(t, s) - (unsigned long long)begin), every);
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
