// binby.cuh — kernel parameter blocks shared by the binby kernels and the C-ABI layer.
#pragma once
#include <stdlib.h>

#include <algorithm>
#include <type_traits>

#include "common.cuh"
#include "device_utils.cuh"
#include "settable.cuh"

namespace b200 {

struct DevBinner {
    int kind, dtype, isz, byteswap, allow_other, invert;
    double vmin, scale, bins_d;
    unsigned long long bins;
    long long ordinal_count, min_value;
    unsigned long long stride;
    const void *data;
    const uint8_t *mask;
    // B200_BINNER_HASH: finalized set table
    const SetSlot *table;
    unsigned long long table_mask;
    long long nan_ordinal;      // -1 when the set saw no NaN
    long long null_ordinal;     // -1 when the set saw no null (masked rows then fall into the null cell)
    long long sentinel_ordinal; // ordinal of the key whose pattern equals SET_EMPTY, -1 if absent
    // B200_BINNER_TIME (time_period in device_utils.cuh): begin = min_value, N = ordinal_count
    TimeSteps time;
    Divisor every;
};

struct DevAgg {
    int op, dtype, isz, byteswap, cell_dtype, smem_off; // smem_off: byte offset of this grid in the CTA's private copy
    unsigned moment;
    int smem_cell; // bytes per cell in the shared-memory copy (COUNT: 4, else the device cell size)
    unsigned long long init_bits; // identity element of the device cell (0, +-inf, numeric limits)
    const void *data;
    const uint8_t *mask;
    void *grid;
};

struct BinParams {
    int nb, na;
    long long nrows;
    unsigned long long cells;
    int smem_copies;     // 0 = global atomics; >= 1: number of per-warp-group private copies in shared memory
    int smem_copy_bytes; // bytes of one private copy (all aggregators)
    DevBinner b[B200_MAX_BINNERS];
    DevAgg a[B200_MAX_AGGS];
};

// FIRST/LAST (first.cu)
struct FirstParams {
    int nb;
    long long nrows, row_offset;
    DevBinner b[B200_MAX_BINNERS];
    int dtype, isz, dtype2, isz2, byteswap, invert;
    const void *data;
    const void *order;
    const uint8_t *mask;
    void *grid;                 // value cells (dtype)
    void *order_grid;           // order cells (dtype2)
    unsigned long long *state;  // {key,row} pairs, 16 B aligned
    uint8_t *cell_masked;
};

// ---- specialised float-key paths (ringcount.cu, fast.cu, tilesort.cu), picked by launch_binby --------------------------------
// 1-3 scalar binners over one float type, native byte order, no masks.  The first 120 bytes of FastParams and RingParams: no
// padding, so the kernels' parameter offsets are those of the flat structs this replaced.
struct FloatKeys {
    const void *x[3];
    double vmin[3], scale[3], bins_d[3];
    unsigned bins[3];
    unsigned stride[3];
};

struct FastParams : FloatKeys {
    long long nrows;
    unsigned cells;
    const void *v;                      // value column or null
    unsigned long long *count_star;     // nullable grids (global)
    unsigned long long *vcount;
    double *vsum;
    double *vm2;
    int smem_copies;                    // > 0: privatise in shared memory (u32 counts, f64 sums)
};

// a b200_bin call the float-key kernels can take: keys, count(*) / count(v) / sum(v) / sum(v^2) of at most one value column
struct FloatPlan {
    FastParams p;
    int xdtype; // B200_F32 / B200_F64, every key column
    int nd;     // key columns, 1..3
    int vdtype; // of the value column, -1 without one
};

// ringcount.cu: parts of <= kRingTileCells cells (192 KB of u32 counters in k_ring_count, one of them the pad cell), <= kRingParts
constexpr unsigned kRingTileCells = 49151;
constexpr int kRingParts = 64;

// Each launches one variant for the plan.  The ring pair and the region sort set *taken = false, with no error, when their
// scratch or part geometry does not work out for this grid: the caller then takes the next kernel.
int launch_ringcount(b200_ctx *ctx, Slot *slot, const FloatPlan &f, bool *taken);
int launch_fast(b200_ctx *ctx, cudaStream_t stream, const FloatPlan &f, size_t smem);
int launch_tilesort(b200_ctx *ctx, Slot *slot, const FloatPlan &f, bool *taken);

// Calls fn(T(), std::integral_constant<int, ND>()) with the plan's key type (float / double) and dimension count.
template <typename F>
int with_keys(const FloatPlan &f, F &&fn) {
    auto nd = [&](auto t) {
        switch (f.nd) {
        case 1: return fn(t, std::integral_constant<int, 1>());
        case 2: return fn(t, std::integral_constant<int, 2>());
        default: return fn(t, std::integral_constant<int, 3>());
        }
    };
    return f.xdtype == B200_F32 ? nd(float()) : nd(double());
}

// Grid-stride kernels: one CTA per `rows_per_cta` rows, at most as many as are resident on all SMs at once.
template <typename P>
int launch_persistent(b200_ctx *ctx, cudaStream_t stream, void (*kern)(P), int threads, size_t smem, long long rows_per_cta, const P &p) {
    if (smem > 48 * 1024)
        B200_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    int per_sm = 0;
    B200_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, threads, smem));
    const long long want = (p.nrows + rows_per_cta - 1) / rows_per_cta, cap = (long long)ctx->sm_count * std::max(per_sm, 1);
    kern<<<(int)std::max(std::min(want, cap), 1ll), threads, smem, stream>>>(p);
    B200_CUDA(cudaGetLastError());
    return B200_OK;
}

// tuning knobs of the region sort, read per call (tests shrink them to reach every variant with small inputs)
inline long long env_ll(const char *name, long long dflt) {
    const char *e = getenv(name);
    return e && *e ? atoll(e) : dflt;
}

// Grows slot->scratch (partition scratch) to at least `need` bytes; the old block is freed once the slot's stream has drained.
// *room = false, with no error set, when cudaMalloc refuses: the caller then takes another kernel.
int slot_scratch(Slot *slot, size_t need, bool *room);

// NUNIQUE (nunique.cu)
struct NUniqueParams {
    int nb;
    long long row0, nrows;
    DevBinner b[B200_MAX_BINNERS];
    int dtype, isz, byteswap;
    const void *data;
    const uint8_t *valid;      // 1 = value present (nullable)
    const uint8_t *selection;  // 1 = row takes part (nullable)
    unsigned long long *table; // 2 u64 per slot: {cell, canonical value bits}; empty = {~0, ~0}
    unsigned long long tmask;
    unsigned long long *distinct, *nan_rows, *null_rows; // cells each
    unsigned long long *total;
};

int launch_binby(b200_ctx *ctx, Slot *slot, const BinParams &p, bool vec);
int launch_nunique(b200_ctx *ctx, cudaStream_t stream, const NUniqueParams &p, bool vec);
int launch_nunique_rehash(cudaStream_t stream, const unsigned long long *old_table, unsigned long long old_cap, unsigned long long *table, unsigned long long cap);
int launch_first(b200_ctx *ctx, cudaStream_t stream, const FirstParams &p, bool vec);
int launch_fill(cudaStream_t stream, void *ptr, int cell_dtype, uint64_t cells, uint64_t bits);
int launch_fill_elems(cudaStream_t stream, void *ptr, int isz, uint64_t n, uint64_t bits);
int launch_merge(cudaStream_t stream, int op, int cell_dtype, void *dst, const void *src, uint64_t cells);
// the FIRST/LAST state merged into an aggregator: another aggregator's buffers, or copies of them on this device
struct FirstGrids {
    const void *grid, *state, *order;
    const uint8_t *cell_masked;
};
int launch_merge_first(cudaStream_t stream, b200_agg *dst, const FirstGrids &src);

} // namespace b200
