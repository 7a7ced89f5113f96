// binby_index.cuh — flat grid index of 4 consecutive rows: every Binner::to_bins fused (src/agg.hpp:106-124).
#pragma once
#include "binby.cuh"
#include "device_utils.cuh"
#include "settable.cuh"

namespace b200 {

template <bool VEC>
__device__ __forceinline__ void binby_indices(const DevBinner *__restrict__ binners, int nb, long long base, int nv, unsigned long long idx[4]) {
#pragma unroll
    for (int j = 0; j < 4; j++)
        idx[j] = 0;
    for (int i = 0; i < nb; i++) {
        const DevBinner &b = binners[i];
        uint64_t r[4];
        unsigned m[4] = {0, 0, 0, 0};
        load4_raw<VEC>(b.data, b.isz, base, nv, r);
        if (b.mask)
            load4_mask<VEC>(b.mask, base, nv, m);
        if (b.kind == B200_BINNER_SCALAR) {
#pragma unroll
            for (int j = 0; j < 4; j++) {
                uint64_t raw = b.byteswap ? bswap(r[j], b.isz) : r[j];
                double v = raw_to_double(b.dtype, raw);
                idx[j] += scalar_index(v, m[j] == 1, b.vmin, b.scale, b.bins_d, b.bins) * b.stride;
            }
        } else if (b.kind == B200_BINNER_ORDINAL) {
#pragma unroll
            for (int j = 0; j < 4; j++) {
                long long value = ordinal_value(b.dtype, r[j], b.min_value, b.byteswap != 0);
                idx[j] += ordinal_index(value, m[j] == 1, b.ordinal_count, b.allow_other != 0, b.invert != 0) * b.stride;
            }
        } else if (b.kind == B200_BINNER_TIME) {
#pragma unroll
            for (int j = 0; j < 4; j++) {
                const long long t = (long long)(b.byteswap ? bswap(r[j], 8) : r[j]);
                idx[j] += ordinal_index(time_bin(t, m[j] == 1, b.time, b.min_value, b.every), false, b.ordinal_count, false, false) * b.stride;
            }
        } else { // B200_BINNER_HASH: HashMapUnique.map (vaex/hash.py:193-214) + BinnerOrdinal
#pragma unroll
            for (int j = 0; j < 4; j++) {
                const uint64_t raw = b.byteswap ? bswap(r[j], b.isz) : r[j];
                long long value;
                if (j >= nv)
                    value = -1;
                else if (m[j] == 1)
                    value = b.null_ordinal;
                else if (raw_isnan(b.dtype, raw))
                    value = b.nan_ordinal;
                else
                    value = set_ordinal(b.table, b.table_mask, b.sentinel_ordinal, key_canon(b.dtype, raw));
                idx[j] += ordinal_index(value, false, b.ordinal_count, b.allow_other != 0, b.invert != 0) * b.stride;
            }
        }
    }
}

} // namespace b200
