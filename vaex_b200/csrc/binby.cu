// binby.cu — the fused binned-aggregation kernel: Grid::bin_ + Binner::to_bins + Aggregator::aggregate
// of the reference (src/agg.hpp:106-137) as ONE pass over the row columns.
//
// Data layout in HBM
//   columns : flat native-dtype arrays (device resident or staged per chunk), optional uint8 masks
//   grids   : one flat array per aggregator, dim 0 (first binner) fastest — the reference's strides
//             (src/agg.hpp:67-72) — int64 for counts, upcast<T> for sums, T for min/max.
//
// Work decomposition
//   persistent grid (SMs x resident CTAs), grid-stride loop, 4 consecutive rows per thread per step so a
//   warp covers 128 consecutive rows: every column is read with 128-bit ld.global.cs (evict-first, the grid
//   stays in L2), fp64 index math replicates the reference bit for bit, then one RED per (row, aggregator).
//   Small grids (all aggregators' private copies fit in shared memory) are privatised per CTA — with several
//   per-warp-group copies to cut same-address contention — and flushed with one global RED per non-empty cell.
//
// Bound: the scatter.  Large grids issue one L2 RED per row per aggregator; L1TEX/LSU retires ~1 scattered lane
// per clock per SM, so rows/s <= 132 SMs x f_SM / n_aggs — well below the HBM stream rate for 8-12 B rows.
#include <stdlib.h>

#include "binby_index.cuh"

namespace b200 {

namespace {

constexpr int kThreads = 256;

template <bool SMEM>
__device__ __forceinline__ void apply_agg(const DevAgg &a, char *cells, unsigned long long idx, uint64_t raw) {
    switch (a.op) {
    case B200_AGG_COUNT:
        if (SMEM)
            atomicAdd(reinterpret_cast<unsigned *>(cells) + idx, 1u);
        else
            atomicAdd(reinterpret_cast<unsigned long long *>(cells) + idx, 1ull);
        break;
    case B200_AGG_SUM:
    case B200_AGG_SUM_MOMENT:
        if (a.cell_dtype == B200_F64) {
            double b = raw_to_double(a.dtype, raw);
            if (a.op == B200_AGG_SUM_MOMENT)
                b = pow_moment(b, a.moment);
            atomicAdd(reinterpret_cast<double *>(cells) + idx, b);
        } else {
            unsigned long long b = raw_to_i64bits(a.dtype, raw);
            if (a.op == B200_AGG_SUM_MOMENT) {
                // `a += pow(b, moment)` on an integer grid is evaluated in double (src/agg_sum.cpp:159).  Each row's power is
                // converted the way the reference's x86-64 build converts (out of range: INT64_MIN, uint64 >= 2^64: 0) and the
                // integers are summed exactly, mod 2^64: bit-exact while a cell's running sum stays below 2^53 (DESIGN §3)
                if (a.cell_dtype == B200_I64)
                    b = (unsigned long long)f64_to_i64_x86(pow_moment_int(__ll2double_rn((long long)b), a.moment));
                else
                    b = f64_to_u64_x86(pow_moment_int(__ull2double_rn(b), a.moment));
            }
            atomicAdd(reinterpret_cast<unsigned long long *>(cells) + idx, b);
        }
        break;
    case B200_AGG_MIN:
    case B200_AGG_MAX: {
        const bool mx = a.op == B200_AGG_MAX;
        switch (a.cell_dtype) {
        case B200_F64: {
            double v = __longlong_as_double((long long)raw);
            mx ? atomic_max_f64(reinterpret_cast<double *>(cells) + idx, v) : atomic_min_f64(reinterpret_cast<double *>(cells) + idx, v);
            break;
        }
        case B200_F32: {
            float v = __uint_as_float((uint32_t)raw);
            mx ? atomic_max_f32(reinterpret_cast<float *>(cells) + idx, v) : atomic_min_f32(reinterpret_cast<float *>(cells) + idx, v);
            break;
        }
        case B200_I64: {
            long long v = (long long)raw;
            mx ? atomicMax(reinterpret_cast<long long *>(cells) + idx, v) : atomicMin(reinterpret_cast<long long *>(cells) + idx, v);
            break;
        }
        case B200_U64: mx ? atomicMax(reinterpret_cast<unsigned long long *>(cells) + idx, raw) : atomicMin(reinterpret_cast<unsigned long long *>(cells) + idx, raw); break;
        case B200_I32: {
            int v = (int)(long long)raw_to_i64bits(a.dtype, raw);
            mx ? atomicMax(reinterpret_cast<int *>(cells) + idx, v) : atomicMin(reinterpret_cast<int *>(cells) + idx, v);
            break;
        }
        default: {
            unsigned v = (unsigned)raw;
            mx ? atomicMax(reinterpret_cast<unsigned *>(cells) + idx, v) : atomicMin(reinterpret_cast<unsigned *>(cells) + idx, v);
            break;
        }
        }
        break;
    }
    default: break;
    }
}

// flush one private shared-memory cell into the global grid
__device__ __forceinline__ void flush_cell(const DevAgg &a, const char *scells, unsigned long long idx) {
    char *g = static_cast<char *>(a.grid);
    if (a.op == B200_AGG_COUNT) {
        unsigned c = reinterpret_cast<const unsigned *>(scells)[idx];
        if (c)
            atomicAdd(reinterpret_cast<unsigned long long *>(g) + idx, (unsigned long long)c);
        return;
    }
    if (a.smem_cell == 8) {
        unsigned long long v = reinterpret_cast<const unsigned long long *>(scells)[idx];
        if (v == a.init_bits)
            return;
        if (a.op == B200_AGG_SUM || a.op == B200_AGG_SUM_MOMENT) {
            if (a.cell_dtype == B200_F64)
                atomicAdd(reinterpret_cast<double *>(g) + idx, __longlong_as_double((long long)v));
            else
                atomicAdd(reinterpret_cast<unsigned long long *>(g) + idx, v);
        } else {
            DevAgg t = a; // min/max: re-apply the private extreme as one more "row"
            apply_agg<false>(t, g, idx, v);
        }
    } else {
        unsigned v = reinterpret_cast<const unsigned *>(scells)[idx];
        if (v == (unsigned)a.init_bits)
            return;
        const bool mx = a.op == B200_AGG_MAX;
        if (a.cell_dtype == B200_F32) {
            float f = __uint_as_float(v);
            mx ? atomic_max_f32(reinterpret_cast<float *>(g) + idx, f) : atomic_min_f32(reinterpret_cast<float *>(g) + idx, f);
        } else if (a.cell_dtype == B200_I32) {
            mx ? atomicMax(reinterpret_cast<int *>(g) + idx, (int)v) : atomicMin(reinterpret_cast<int *>(g) + idx, (int)v);
        } else {
            mx ? atomicMax(reinterpret_cast<unsigned *>(g) + idx, v) : atomicMin(reinterpret_cast<unsigned *>(g) + idx, v);
        }
    }
}

template <bool VEC, bool SMEM>
__global__ void __launch_bounds__(kThreads) k_binby(const __grid_constant__ BinParams p) {
    extern __shared__ __align__(16) char smem[];
    char *my_copy = nullptr;
    if (SMEM) {
        // initialise every private copy with the aggregators' identity elements
        for (int k = 0; k < p.na; k++) {
            const DevAgg &a = p.a[k];
            for (int c = 0; c < p.smem_copies; c++) {
                char *cp = smem + (size_t)c * p.smem_copy_bytes + a.smem_off;
                if (a.smem_cell == 8) {
                    for (unsigned long long i = threadIdx.x; i < p.cells; i += kThreads)
                        reinterpret_cast<unsigned long long *>(cp)[i] = a.op == B200_AGG_COUNT ? 0ull : a.init_bits;
                } else {
                    for (unsigned long long i = threadIdx.x; i < p.cells; i += kThreads)
                        reinterpret_cast<unsigned *>(cp)[i] = a.op == B200_AGG_COUNT ? 0u : (unsigned)a.init_bits;
                }
            }
        }
        __syncthreads();
        my_copy = smem + (size_t)((threadIdx.x >> 5) % p.smem_copies) * p.smem_copy_bytes;
    }

    const long long step = (long long)gridDim.x * kThreads * 4;
    for (long long base = ((long long)blockIdx.x * kThreads + threadIdx.x) * 4; base < p.nrows; base += step) {
        const long long left = p.nrows - base;
        const int nv = left < 4 ? (int)left : 4;
        unsigned long long idx[4];
        binby_indices<VEC>(p.b, p.nb, base, nv, idx);

        for (int k = 0; k < p.na; k++) {
            const DevAgg &a = p.a[k];
            uint64_t r[4] = {0, 0, 0, 0};
            unsigned m[4] = {1, 1, 1, 1};
            if (a.data)
                load4_raw<VEC>(a.data, a.isz, base, nv, r);
            if (a.mask)
                load4_mask<VEC>(a.mask, base, nv, m);
            char *cells = SMEM ? my_copy + a.smem_off : static_cast<char *>(a.grid);
#pragma unroll
            for (int j = 0; j < 4; j++) {
                uint64_t raw = a.byteswap ? bswap(r[j], a.isz) : r[j];
                // aggregator mask convention: 1 = use the row; NaN values never count (src/agg_count.cpp:49-60)
                bool use = j < nv && m[j] == 1 && !(a.data && raw_isnan(a.dtype, raw));
                if (use)
                    apply_agg<SMEM>(a, cells, idx[j], raw);
            }
        }
    }

    if (SMEM) {
        __syncthreads();
        for (int k = 0; k < p.na; k++) {
            const DevAgg &a = p.a[k];
            for (int c = 0; c < p.smem_copies; c++) {
                const char *cp = smem + (size_t)c * p.smem_copy_bytes + a.smem_off;
                for (unsigned long long i = threadIdx.x; i < p.cells; i += kThreads)
                    flush_cell(a, cp, i);
            }
        }
    }
}

__global__ void k_fill64(unsigned long long *p, uint64_t n, unsigned long long v) {
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x)
        p[i] = v;
}
__global__ void k_fill32(unsigned *p, uint64_t n, unsigned v) {
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x)
        p[i] = v;
}
__global__ void k_fill16(unsigned short *p, uint64_t n, unsigned short v) {
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x)
        p[i] = v;
}

// Aggregator::merge (src/agg_count.cpp:15-23, src/agg_sum.cpp:69-76, src/agg_minmax.cpp:19-27)
__global__ void k_merge(int op, int cell_dtype, void *dst, const void *src, uint64_t n) {
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
        if (op == B200_AGG_COUNT || op == B200_AGG_SUM || op == B200_AGG_SUM_MOMENT) {
            if (cell_dtype == B200_F64)
                static_cast<double *>(dst)[i] += static_cast<const double *>(src)[i];
            else
                static_cast<unsigned long long *>(dst)[i] += static_cast<const unsigned long long *>(src)[i];
        } else {
            const bool mx = op == B200_AGG_MAX;
#define MM(T)                                                                                                                  \
    {                                                                                                                          \
        T a = static_cast<T *>(dst)[i], b = static_cast<const T *>(src)[i];                                                   \
        static_cast<T *>(dst)[i] = mx ? (a < b ? b : a) : (b < a ? b : a);                                                    \
    }
            switch (cell_dtype) {
            case B200_F64: MM(double) break;
            case B200_F32: MM(float) break;
            case B200_I64: MM(long long) break;
            case B200_U64: MM(unsigned long long) break;
            case B200_I32: MM(int) break;
            default: MM(unsigned) break;
            }
#undef MM
        }
    }
}

template <bool VEC, bool SMEM>
int launch_variant(b200_ctx *ctx, cudaStream_t stream, const BinParams &p) {
    size_t smem = SMEM ? (size_t)p.smem_copies * p.smem_copy_bytes : 0;
    auto kern = k_binby<VEC, SMEM>;
    if (smem > 48 * 1024)
        B200_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    int per_sm = 0;
    B200_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, kThreads, smem));
    if (per_sm < 1)
        per_sm = 1;
    long long want = (p.nrows + (long long)kThreads * 4 - 1) / ((long long)kThreads * 4);
    long long cap = (long long)ctx->sm_count * per_sm;
    int blocks = (int)(want < cap ? want : cap);
    if (blocks < 1)
        blocks = 1;
    kern<<<blocks, kThreads, smem, stream>>>(p);
    B200_CUDA(cudaGetLastError());
    return B200_OK;
}

} // namespace

int try_launch_fast(b200_ctx *ctx, Slot *slot, const BinParams &bp, bool vec, bool *taken);          // fast.cu
int try_launch_ringcount(b200_ctx *ctx, Slot *slot, const BinParams &bp, bool vec, bool *taken);     // ringcount.cu

int launch_binby(b200_ctx *ctx, Slot *slot, const BinParams &p, bool vec) {
    if (p.nrows <= 0)
        return B200_OK;
    if (p.nrows >= (1ll << 38)) { // the shared-memory sub-histograms count in 32 bits per CTA: >= 132 CTAs keep a CTA's share below 2^31
        set_error("b200_bin: %lld rows in one call (the limit is 2^38; an H100 holds < 2^38 rows of any column)", (long long)p.nrows);
        return B200_ERR_INVALID;
    }
    cudaStream_t stream = slot->stream;
    // B200_DISABLE_FAST=1 forces the descriptor-driven kernel (A/B measurements, parity tests of both kernels)
    static const bool disable_fast = getenv("B200_DISABLE_FAST") && atoi(getenv("B200_DISABLE_FAST")) != 0;
    if (!disable_fast) {
        bool taken = false;
        B200_CHECK(try_launch_ringcount(ctx, slot, p, vec, &taken));
        if (taken)
            return B200_OK;
        B200_CHECK(try_launch_fast(ctx, slot, p, vec, &taken));
        if (taken)
            return B200_OK;
    }
    if (p.smem_copies > 0)
        return vec ? launch_variant<true, true>(ctx, stream, p) : launch_variant<false, true>(ctx, stream, p);
    return vec ? launch_variant<true, false>(ctx, stream, p) : launch_variant<false, false>(ctx, stream, p);
}

int launch_fill(cudaStream_t stream, void *ptr, int cell_dtype, uint64_t cells, uint64_t bits) {
    if (!cells)
        return B200_OK;
    int blocks = (int)((cells + 255) / 256 < kSmCount * 8 ? (cells + 255) / 256 : kSmCount * 8);
    if (dtype_size(cell_dtype) == 8)
        k_fill64<<<blocks, 256, 0, stream>>>(static_cast<unsigned long long *>(ptr), cells, bits);
    else
        k_fill32<<<blocks, 256, 0, stream>>>(static_cast<unsigned *>(ptr), cells, (unsigned)bits);
    B200_CUDA(cudaGetLastError());
    return B200_OK;
}

// n elements of `isz` bytes (1, 2, 4 or 8), each set to the low bytes of `bits`
int launch_fill_elems(cudaStream_t stream, void *ptr, int isz, uint64_t n, uint64_t bits) {
    if (!n)
        return B200_OK;
    const int blocks = (int)((n + 255) / 256 < kSmCount * 8 ? (n + 255) / 256 : kSmCount * 8);
    switch (isz) {
    case 8: k_fill64<<<blocks, 256, 0, stream>>>(static_cast<unsigned long long *>(ptr), n, bits); break;
    case 4: k_fill32<<<blocks, 256, 0, stream>>>(static_cast<unsigned *>(ptr), n, (unsigned)bits); break;
    case 2: k_fill16<<<blocks, 256, 0, stream>>>(static_cast<unsigned short *>(ptr), n, (unsigned short)bits); break;
    default: B200_CUDA(cudaMemsetAsync(ptr, (int)(bits & 0xff), n, stream)); break;
    }
    B200_CUDA(cudaGetLastError());
    return B200_OK;
}

int launch_merge(cudaStream_t stream, int op, int cell_dtype, void *dst, const void *src, uint64_t cells) {
    if (!cells)
        return B200_OK;
    int blocks = (int)((cells + 255) / 256 < kSmCount * 8 ? (cells + 255) / 256 : kSmCount * 8);
    k_merge<<<blocks, 256, 0, stream>>>(op, cell_dtype, dst, src, cells);
    B200_CUDA(cudaGetLastError());
    return B200_OK;
}

} // namespace b200
