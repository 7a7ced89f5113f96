// nunique.cu — AggNUniquePrimitive on the device: number of distinct values per grid cell.
// Reference: src/agg_nunique.cpp:57-86 (aggregate: one counter<T> per cell; a row outside the selection is skipped, a masked
// row counts as null, NaN as nan, anything else is inserted into the cell's hash map), :16-42 (get_result).
//
// The reference owns `cells` separate hash maps.  Here ONE open-addressing table holds the distinct (cell, value) pairs of the
// whole grid — 16-byte slots claimed with one 128-bit compare-and-swap (atom.global.cas.b128, as in first.cu) — and three
// planes of per-cell counters (distinct pairs, NaN rows, null rows) are bumped on the side; get_result folds them with the
// reference's formula.  The table never overflows inside a kernel: the host sizes it for (pairs so far + rows of the batch)
// before every launch and rehashes when it has to grow.
#include "binby_index.cuh"
#include "cas128.cuh"

namespace b200 {

namespace {

constexpr int kThreads = 256;
constexpr unsigned long long kEmpty = ~0ull;

// true when (cell, canon) was not in the table yet
__device__ __forceinline__ bool pair_insert(unsigned long long *table, unsigned long long mask, unsigned long long cell, unsigned long long canon) {
    unsigned long long h = hash64(canon ^ hash64(cell)) & mask;
    while (true) {
        U128 cur = load128(table + 2 * h);
        if (cur.lo == kEmpty) {
            cur = cas128(table + 2 * h, U128{kEmpty, kEmpty}, U128{cell, canon});
            if (cur.lo == kEmpty)
                return true;
        }
        if (cur.lo == cell && cur.hi == canon)
            return false;
        h = (h + 1) & mask;
    }
}

template <bool VEC>
__global__ void __launch_bounds__(kThreads) k_nunique(const __grid_constant__ NUniqueParams p) {
    const long long end = p.row0 + p.nrows;
    const long long step = (long long)gridDim.x * kThreads * 4;
    unsigned fresh = 0;
    for (long long base = p.row0 + ((long long)blockIdx.x * kThreads + threadIdx.x) * 4; base < end; base += step) {
        const long long left = end - base;
        const int nv = left < 4 ? (int)left : 4;
        unsigned long long idx[4];
        binby_indices<VEC>(p.b, p.nb, base, nv, idx);
        uint64_t r[4];
        unsigned valid[4] = {1, 1, 1, 1}, use[4] = {1, 1, 1, 1};
        load4_raw<VEC>(p.data, p.isz, base, nv, r);
        if (p.valid)
            load4_mask<VEC>(p.valid, base, nv, valid);
        if (p.selection)
            load4_mask<VEC>(p.selection, base, nv, use);
#pragma unroll
        for (int j = 0; j < 4; j++) {
            if (j >= nv || !use[j])
                continue; // not in the selection / filter: not even a null (src/agg_nunique.cpp:67-68)
            if (!valid[j]) {
                atomicAdd(p.null_rows + idx[j], 1ull);
                continue;
            }
            const uint64_t raw = p.byteswap ? bswap(r[j], p.isz) : r[j];
            if (raw_isnan(p.dtype, raw)) {
                atomicAdd(p.nan_rows + idx[j], 1ull);
                continue;
            }
            if (pair_insert(p.table, p.tmask, idx[j], key_canon(p.dtype, raw))) {
                atomicAdd(p.distinct + idx[j], 1ull);
                fresh++;
            }
        }
    }
    // pairs added by this launch: one atomic per warp on the shared total (same-address atomics serialise in the L2)
#pragma unroll
    for (int o = 16; o > 0; o >>= 1)
        fresh += __shfl_xor_sync(0xffffffffu, fresh, o);
    if ((threadIdx.x & 31) == 0 && fresh)
        atomicAdd(p.total, (unsigned long long)fresh);
}

__global__ void k_nunique_rehash(const unsigned long long *old_table, unsigned long long old_cap, unsigned long long *table, unsigned long long mask) {
    for (unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; i < old_cap; i += (unsigned long long)gridDim.x * blockDim.x) {
        const unsigned long long cell = old_table[2 * i];
        if (cell != kEmpty)
            pair_insert(table, mask, cell, old_table[2 * i + 1]);
    }
}

} // namespace

int launch_nunique(b200_ctx *ctx, cudaStream_t stream, const NUniqueParams &p, bool vec) {
    if (p.nrows <= 0)
        return B200_OK;
    long long want = (p.nrows + (long long)kThreads * 4 - 1) / ((long long)kThreads * 4);
    long long cap = (long long)ctx->sm_count * 8;
    int blocks = (int)(want < cap ? want : cap);
    if (vec)
        k_nunique<true><<<blocks, kThreads, 0, stream>>>(p);
    else
        k_nunique<false><<<blocks, kThreads, 0, stream>>>(p);
    B200_CUDA(cudaGetLastError());
    return B200_OK;
}

int launch_nunique_rehash(cudaStream_t stream, const unsigned long long *old_table, unsigned long long old_cap, unsigned long long *table, unsigned long long cap) {
    if (!old_cap)
        return B200_OK;
    unsigned long long want = (old_cap + 255) / 256;
    int blocks = (int)(want < kSmCount * 8ull ? want : kSmCount * 8ull);
    k_nunique_rehash<<<blocks, 256, 0, stream>>>(old_table, old_cap, table, cap - 1);
    B200_CUDA(cudaGetLastError());
    return B200_OK;
}

} // namespace b200
