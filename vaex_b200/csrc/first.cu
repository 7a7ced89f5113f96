// first.cu — AggFirstPrimitive (first / last by an order column) on the device.
// Reference: src/agg_first.cpp:115-165 (aggregate), :19-26 (initial_fill), :61-114 (get_result).
//
// The reference keeps (value, order, cell_masked) per cell and replaces them when the new order is strictly
// smaller (first) / larger (last); ties keep the row seen first.  Sequential row order is the tie-break, so the
// device version reduces the lexicographic pair (order_key, global_row) with ONE 128-bit compare-and-swap per
// candidate row (atom.global.cas.b128, sm_90+), then a second pass over the chunk lets the unique winning row of
// each cell deposit its value.  Both passes recompute the flat index from the binner columns (cheaper than
// materialising 8 B/row of indices).
#include "binby_index.cuh"
#include "cas128.cuh"

namespace b200 {

namespace {

constexpr int kThreads = 256;

// monotone map of an order value to u64 so that `<` on the original type is `<` on the key; -0.0 == +0.0
__device__ __forceinline__ unsigned long long order_key(int dt, uint64_t raw) {
    switch (dt) {
    case B200_F64:
    case B200_F32: return order_key_f64(raw_to_double(dt, raw));
    case B200_I64:
    case B200_I32:
    case B200_I16:
    case B200_I8: return raw_to_i64bits(dt, raw) ^ 0x8000000000000000ULL;
    default: return raw;
    }
}

// shared by both passes: validity + (key,row) of row j
struct Cand {
    bool valid;
    U128 kr;
    uint64_t value_raw, order_raw;
};

template <bool VEC>
__device__ __forceinline__ void candidates(const FirstParams &p, long long base, int nv, Cand c[4]) {
    uint64_t v[4], o[4] = {0, 0, 0, 0};
    load4_raw<VEC>(p.data, p.isz, base, nv, v);
    if (p.order)
        load4_raw<VEC>(p.order, p.isz2, base, nv, o);
#pragma unroll
    for (int j = 0; j < 4; j++) {
        const long long i = base + j; // chunk-local row
        bool valid = j < nv;
        // reference quirk kept for parity: the mask is indexed inside the current 1024-row block
        // WITHOUT the block offset (src/agg_first.cpp:131, `data_mask_ptr[j]`)
        if (valid && p.mask)
            valid = p.mask[i & 1023] == 1;
        uint64_t vr = p.byteswap ? bswap(v[j], p.isz) : v[j];
        uint64_t orr;
        if (p.order) {
            orr = p.byteswap ? bswap(o[j], p.isz2) : o[j];
        } else {
            // DataType2 value_order = offset + j, flipped too when FlipEndian (:134-138)
            orr = (uint64_t)i;
            if (p.isz2 < 8)
                orr &= (1ULL << (8 * p.isz2)) - 1;
            if (p.dtype2 == B200_F64)
                orr = (uint64_t)__double_as_longlong(__ll2double_rn(i));
            else if (p.dtype2 == B200_F32)
                orr = __float_as_uint(__ll2float_rn(i));
            else if (p.dtype2 == B200_BOOL)
                orr = i != 0;
            if (p.byteswap)
                orr = bswap(orr, p.isz2);
        }
        if (valid && (raw_isnan(p.dtype, vr) || raw_isnan(p.dtype2, orr)))
            valid = false;
        unsigned long long key = order_key(p.dtype2, orr);
        if (p.invert)
            key = ~key;
        c[j].valid = valid;
        c[j].kr = U128{key, (unsigned long long)(p.row_offset + i)};
        c[j].value_raw = vr;
        c[j].order_raw = orr;
    }
}

template <bool VEC>
__global__ void __launch_bounds__(kThreads) k_first_select(const __grid_constant__ FirstParams p) {
    const long long step = (long long)gridDim.x * kThreads * 4;
    for (long long base = ((long long)blockIdx.x * kThreads + threadIdx.x) * 4; base < p.nrows; base += step) {
        const long long left = p.nrows - base;
        const int nv = left < 4 ? (int)left : 4;
        unsigned long long idx[4];
        binby_indices<VEC>(p.b, p.nb, base, nv, idx);
        Cand c[4];
        candidates<VEC>(p, base, nv, c);
#pragma unroll
        for (int j = 0; j < 4; j++) {
            if (!c[j].valid)
                continue;
            cas128_min(p.state + 2 * idx[j], c[j].kr);
        }
    }
}

__device__ __forceinline__ void store_raw(void *arr, int isz, unsigned long long i, uint64_t raw) {
    switch (isz) {
    case 8: static_cast<unsigned long long *>(arr)[i] = raw; break;
    case 4: static_cast<unsigned *>(arr)[i] = (unsigned)raw; break;
    case 2: static_cast<unsigned short *>(arr)[i] = (unsigned short)raw; break;
    default: static_cast<unsigned char *>(arr)[i] = (unsigned char)raw; break;
    }
}

template <bool VEC>
__global__ void __launch_bounds__(kThreads) k_first_deposit(const __grid_constant__ FirstParams p) {
    const long long step = (long long)gridDim.x * kThreads * 4;
    for (long long base = ((long long)blockIdx.x * kThreads + threadIdx.x) * 4; base < p.nrows; base += step) {
        const long long left = p.nrows - base;
        const int nv = left < 4 ? (int)left : 4;
        unsigned long long idx[4];
        binby_indices<VEC>(p.b, p.nb, base, nv, idx);
        Cand c[4];
        candidates<VEC>(p, base, nv, c);
#pragma unroll
        for (int j = 0; j < 4; j++) {
            if (!c[j].valid)
                continue;
            U128 cur = load128(p.state + 2 * idx[j]);
            if (cur.lo == c[j].kr.lo && cur.hi == c[j].kr.hi) { // exactly one row of the whole job matches
                store_raw(p.grid, p.isz, idx[j], c[j].value_raw);
                store_raw(p.order_grid, p.isz2, idx[j], c[j].order_raw);
                p.cell_masked[idx[j]] = 0;
            }
        }
    }
}

// get_result fold of the reference (src/agg_first.cpp:68-99) as a merge of two device aggregators
__global__ void k_merge_first(unsigned long long *dstate, const unsigned long long *sstate, void *dgrid, const void *sgrid, void *dorder,
                              const void *sorder, uint8_t *dmask, const uint8_t *smask, int isz, int isz2, uint64_t n) {
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
        if (smask[i] == 1)
            continue;
        U128 s{sstate[2 * i], sstate[2 * i + 1]}, d{dstate[2 * i], dstate[2 * i + 1]};
        if (dmask[i] == 1 || less128(s, d)) {
            dstate[2 * i] = s.lo;
            dstate[2 * i + 1] = s.hi;
            dmask[i] = 0;
            switch (isz) {
            case 8: static_cast<unsigned long long *>(dgrid)[i] = static_cast<const unsigned long long *>(sgrid)[i]; break;
            case 4: static_cast<unsigned *>(dgrid)[i] = static_cast<const unsigned *>(sgrid)[i]; break;
            case 2: static_cast<unsigned short *>(dgrid)[i] = static_cast<const unsigned short *>(sgrid)[i]; break;
            default: static_cast<unsigned char *>(dgrid)[i] = static_cast<const unsigned char *>(sgrid)[i]; break;
            }
            switch (isz2) {
            case 8: static_cast<unsigned long long *>(dorder)[i] = static_cast<const unsigned long long *>(sorder)[i]; break;
            case 4: static_cast<unsigned *>(dorder)[i] = static_cast<const unsigned *>(sorder)[i]; break;
            case 2: static_cast<unsigned short *>(dorder)[i] = static_cast<const unsigned short *>(sorder)[i]; break;
            default: static_cast<unsigned char *>(dorder)[i] = static_cast<const unsigned char *>(sorder)[i]; break;
            }
        }
    }
}

} // namespace

int launch_first(b200_ctx *ctx, cudaStream_t stream, const FirstParams &p, bool vec) {
    if (p.nrows <= 0)
        return B200_OK;
    long long want = (p.nrows + (long long)kThreads * 4 - 1) / ((long long)kThreads * 4);
    long long cap = (long long)ctx->sm_count * 4;
    int blocks = (int)(want < cap ? want : cap);
    if (vec) {
        k_first_select<true><<<blocks, kThreads, 0, stream>>>(p);
        k_first_deposit<true><<<blocks, kThreads, 0, stream>>>(p);
    } else {
        k_first_select<false><<<blocks, kThreads, 0, stream>>>(p);
        k_first_deposit<false><<<blocks, kThreads, 0, stream>>>(p);
    }
    B200_CUDA(cudaGetLastError());
    return B200_OK;
}

int launch_merge_first(cudaStream_t stream, b200_agg *dst, const b200_agg *src) {
    uint64_t n = dst->cells;
    if (!n)
        return B200_OK;
    int blocks = (int)((n + 255) / 256 < kSmCount * 8 ? (n + 255) / 256 : kSmCount * 8);
    k_merge_first<<<blocks, 256, 0, stream>>>(static_cast<unsigned long long *>(dst->state), static_cast<const unsigned long long *>(src->state), dst->grid,
                                              src->grid, dst->order, src->order, dst->cell_masked, src->cell_masked, dtype_size(dst->dtype),
                                              dtype_size(dst->dtype2), n);
    B200_CUDA(cudaGetLastError());
    return B200_OK;
}

} // namespace b200
