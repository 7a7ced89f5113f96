// refvalue.cuh — how the reference's legacy statistics (vaexfast statisticNd, driven by TaskPartStatistic.process,
// vaex/cpu.py:510-611) see a column's values: every block is cast to one compute class, float64 or float32 (`as_flat_array`,
// vaex/utils.py:691-695), and byte-swapped blocks give the values of their native twin.  Shared by minmax.cu and statistic.cu.
#pragma once
#include <type_traits>

#include "device_utils.cuh"

namespace b200 {

// numpy astype(C) of one element of native type T, C = double or float: round-to-nearest-even where the class cannot hold the
// value exactly (int64 / uint64 -> double, 32/64-bit integers -> float), exact otherwise
template <typename C, typename T>
__device__ __forceinline__ C class_value(T v) {
    if constexpr (std::is_same<C, double>::value) {
        if constexpr (std::is_same<T, long long>::value)
            return __ll2double_rn(v);
        else if constexpr (std::is_same<T, unsigned long long>::value)
            return __ull2double_rn(v);
        else
            return (double)v;
    } else {
        if constexpr (std::is_same<T, double>::value)
            return __double2float_rn(v);
        else if constexpr (std::is_same<T, long long>::value)
            return __ll2float_rn(v);
        else if constexpr (std::is_same<T, unsigned long long>::value)
            return __ull2float_rn(v);
        else if constexpr (std::is_same<T, int>::value)
            return __int2float_rn(v);
        else if constexpr (std::is_same<T, unsigned>::value)
            return __uint2float_rn(v);
        else
            return (float)v; // float itself, and 8/16-bit integers (exact)
    }
}

// the reference's cast + widening for one element of a column that is alone in its call: float64 and int64 compute in float64,
// everything else in float32 (vaex/cpu.py:527-541)
template <typename T>
__device__ __forceinline__ double ref_value(T v) {
    if constexpr (std::is_same<T, double>::value || std::is_same<T, long long>::value)
        return class_value<double>(v);
    else
        return (double)class_value<float>(v);
}

template <typename T>
__device__ __forceinline__ T swap_bytes(T v) {
    if constexpr (sizeof(T) == 8) {
        unsigned long long b;
        memcpy(&b, &v, 8);
        b = bswap(b, 8);
        memcpy(&v, &b, 8);
    } else if constexpr (sizeof(T) == 4) {
        unsigned b;
        memcpy(&b, &v, 4);
        b = __byte_perm(b, 0, 0x0123);
        memcpy(&v, &b, 4);
    } else if constexpr (sizeof(T) == 2) {
        unsigned short b;
        memcpy(&b, &v, 2);
        b = (unsigned short)((b >> 8) | (b << 8));
        memcpy(&v, &b, 2);
    }
    return v;
}

// class_value of a native-order element held as zero-extended raw bits (load4_raw) of b200_dtype `dt`
template <typename C>
__device__ __forceinline__ C raw_class_value(int dt, uint64_t r) {
    switch (dt) {
    case B200_F64: return class_value<C>(__longlong_as_double((long long)r));
    case B200_F32: return class_value<C>(__uint_as_float((uint32_t)r));
    case B200_I64: return class_value<C>((long long)r);
    case B200_I32: return class_value<C>((int)(uint32_t)r);
    case B200_I16: return class_value<C>((short)(uint16_t)r);
    case B200_I8: return class_value<C>((signed char)(uint8_t)r);
    case B200_U64: return class_value<C>((unsigned long long)r);
    case B200_U32: return class_value<C>((unsigned)r);
    case B200_U16: return class_value<C>((unsigned short)r);
    default: return class_value<C>((unsigned char)r); // uint8, bool (0 / 1)
    }
}

} // namespace b200
