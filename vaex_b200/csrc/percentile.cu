// percentile.cu — the finish of df.percentile_approx / df.median_approx (vaex/dataframe.py:1675-1754) on an int64 count grid that is
// already in device memory: the cumulative sum along the percentile axis, vaexfast.grid_find_edges (src/vaexfast.cpp:1680-1719) for
// the floor and the ceil target of every percentage, and the linear interpolation between the two edges.
//
// Grid layout (the aggregator's, edges=True): first dimension fastest, the percentile axis last and slowest with stride S = the cells
// of the binby grid.  Every binby axis is sliced [2:-1] and the percentile axis [1:] (P + 2 entries: underflow, P bins, overflow).
//
// grid_find_edges walks cum[] for the last index `left` with every cum[1..left] below the target and then `right` up to the first
// cum[right] not below it, both capped at P + 1.  cum[] is non-decreasing, so with c = the number of entries below the target,
// left = max(c - 1, 0) and right = min(c, P + 1): a count and the cum values at those two indices replace the search.  The reference
// compares cum.astype(float64) with the target, so the count compares the rounded double too; cum itself stays exact int64.
//
// Every double operation is one IEEE operation in the order numpy evaluates the reference's expression (__d*_rn: no contraction),
// so the result is bit-identical to the reference wherever the reference reads inside its grid (0 and 1 binby dimensions).
#include "common.cuh"
#include "scan.cuh"

#include <limits.h>
#include <math.h>

#include <algorithm>

namespace b200 {
namespace {

constexpr int kPctMax = 8;              // percentages per launch; a longer list takes one launch per group of kPctMax
constexpr long long kPctCellMin = 2048; // output cells from which one thread per cell (k_pct_cell) beats one CTA per cell

struct PctArgs {
    const long long *grid;
    long long S;     // stride of the percentile axis: the binby grid's cells, edges included
    long long cells; // sliced binby cells (the output's cells per percentage)
    int ndim;        // binby dimensions
    int plen;        // P + 2: the sliced percentile axis
    long long n[B200_MAX_BINNERS - 1];      // sliced size of each binby dimension
    long long stride[B200_MAX_BINNERS - 1]; // its stride in the grid
    double lb, span, axis;                  // axis = P - 1, the reference's shape[-1] - 3
    double pct[kPctMax];
    int integral[kPctMax];
    int npct; // valid entries of pct[] in this launch
    double *out; // out[k * cells + cell] for the launch's k-th percentage
};

// address of sliced percentile entry 0 (the underflow cell) of a sliced binby cell, first binner fastest
__device__ __forceinline__ const long long *cell_row(const PctArgs &a, long long cell) {
    long long off = a.S;
    for (int d = 0; d < a.ndim; d++) {
        const long long i = cell % a.n[d];
        cell /= a.n[d];
        off += (i + 2) * a.stride[d];
    }
    return a.grid + off;
}

// values = (total + 1) * p / 100. (0 for an empty cell).  An integral p multiplies in int64 first (NEP 50), wrapping like numpy.
__device__ __forceinline__ double target_value(long long total, double p, int integral) {
    if (total == 0)
        return 0.0;
    if (integral) {
        const long long prod = (long long)((unsigned long long)(total + 1) * (unsigned long long)(long long)p);
        return __ddiv_rn(__ll2double_rn(prod), 100.0);
    }
    return __ddiv_rn(__dmul_rn(__ll2double_rn(total + 1), p), 100.0);
}

// lb + (e - 0.5) * span / axis
__device__ __forceinline__ double edge_x(const PctArgs &a, long long e) {
    return __dadd_rn(a.lb, __ddiv_rn(__dmul_rn(__dsub_rn(__ll2double_rn(e), 0.5), a.span), a.axis));
}

// calculate_x of the reference for one target: c entries below it, `below` = the last cum below it, `above` = the first cum not below
__device__ __forceinline__ double calc_x(const PctArgs &a, double t, int c, long long below, long long above) {
    const long long left = c > 0 ? c - 1 : 0, right = c < a.plen - 1 ? c : a.plen - 1;
    const double vl = __ll2double_rn(c > 0 ? below : above), vr = __ll2double_rn(c < a.plen ? above : below);
    double denom = __dsub_rn(vr, vl);
    if (denom == 0.0)
        denom = 1.0;
    const double u = __ddiv_rn(__dsub_rn(t, vl), denom);
    const double xl = edge_x(a, left), xr = edge_x(a, right);
    return __dadd_rn(xl, __dmul_rn(__dsub_rn(xr, xl), u));
}

// x1 + (x2 - x1) * (values - floor(values))
__device__ __forceinline__ double finish(const PctArgs &a, double v, double tf, double tc, int cf, long long bf, long long af, int cc, long long bc,
                                         long long ac) {
    const double x1 = calc_x(a, tf, cf, bf, af), x2 = calc_x(a, tc, cc, bc, ac);
    return __dadd_rn(x1, __dmul_rn(__dsub_rn(x2, x1), __dsub_rn(v, tf)));
}

// one thread per binby cell: a warp reads 32 adjacent cells at every step of the percentile axis
template <int NP>
__global__ void __launch_bounds__(256) k_pct_cell(const PctArgs a) {
    const long long step = (long long)gridDim.x * blockDim.x;
    for (long long cell = blockIdx.x * (long long)blockDim.x + threadIdx.x; cell < a.cells; cell += step) {
        const long long *row = cell_row(a, cell);
        long long total = 0;
#pragma unroll 8
        for (int j = 0; j < a.plen; j++)
            total += row[(long long)j * a.S];
        double v[NP], t[2 * NP];
        int c[2 * NP];
        long long below[2 * NP], above[2 * NP];
#pragma unroll
        for (int k = 0; k < NP; k++) {
            v[k] = k < a.npct ? target_value(total, a.pct[k], a.integral[k]) : 0.0;
            t[2 * k] = floor(v[k]);
            t[2 * k + 1] = ceil(v[k]);
        }
#pragma unroll
        for (int q = 0; q < 2 * NP; q++) {
            c[q] = 0;
            below[q] = above[q] = 0;
        }
        long long cum = 0;
#pragma unroll 4
        for (int j = 0; j < a.plen; j++) {
            cum += row[(long long)j * a.S];
            const double cd = __ll2double_rn(cum);
#pragma unroll
            for (int q = 0; q < 2 * NP; q++) {
                if (cd < t[q]) {
                    c[q]++;
                    below[q] = cum;
                } else if (c[q] == j) {
                    above[q] = cum;
                }
            }
        }
#pragma unroll
        for (int k = 0; k < NP; k++)
            if (k < a.npct)
                a.out[k * a.cells + cell] = finish(a, v[k], t[2 * k], t[2 * k + 1], c[2 * k], below[2 * k], above[2 * k], c[2 * k + 1],
                                                   below[2 * k + 1], above[2 * k + 1]);
    }
}

constexpr int kPctItems = 4; // consecutive entries per thread and tile in k_pct_block
constexpr int kPctWarps = kScanThreads / 32;

// one CTA per binby cell: the percentile axis in tiles of kScanThreads * kPctItems, a block scan per tile with the prefix carried
// over, each thread's counts and edge values kept across tiles and reduced over the CTA at the end
template <int NP>
__global__ void __launch_bounds__(kScanThreads) k_pct_block(const PctArgs a) {
    __shared__ int s_c[kPctWarps][2 * NP];
    __shared__ long long s_below[kPctWarps][2 * NP], s_above[kPctWarps][2 * NP];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (long long cell = blockIdx.x; cell < a.cells; cell += gridDim.x) {
        const long long *row = cell_row(a, cell);
        long long part = 0;
        for (int j = threadIdx.x; j < a.plen; j += kScanThreads)
            part += row[(long long)j * a.S];
        long long total;
        block_exclusive_i64(part, &total);
        __syncthreads(); // the scan's shared sums are reused below
        double v[NP], t[2 * NP];
        int c[2 * NP];
        long long below[2 * NP], above[2 * NP];
#pragma unroll
        for (int k = 0; k < NP; k++) {
            v[k] = k < a.npct ? target_value(total, a.pct[k], a.integral[k]) : 0.0;
            t[2 * k] = floor(v[k]);
            t[2 * k + 1] = ceil(v[k]);
        }
#pragma unroll
        for (int q = 0; q < 2 * NP; q++) {
            c[q] = 0;
            below[q] = LLONG_MIN;
            above[q] = LLONG_MAX;
        }
        long long carry = 0;
        for (int base = 0; base < a.plen; base += kScanThreads * kPctItems) {
            const int j0 = base + threadIdx.x * kPctItems;
            long long r[kPctItems], s = 0;
#pragma unroll
            for (int i = 0; i < kPctItems; i++) {
                r[i] = j0 + i < a.plen ? row[(long long)(j0 + i) * a.S] : 0;
                s += r[i];
            }
            long long tile;
            long long cum = carry + block_exclusive_i64(s, &tile);
            __syncthreads();
            carry += tile;
#pragma unroll
            for (int i = 0; i < kPctItems; i++) {
                if (j0 + i < a.plen) {
                    cum += r[i];
                    const double cd = __ll2double_rn(cum);
#pragma unroll
                    for (int q = 0; q < 2 * NP; q++) {
                        if (cd < t[q]) {
                            c[q]++;
                            below[q] = max(below[q], cum);
                        } else {
                            above[q] = min(above[q], cum);
                        }
                    }
                }
            }
        }
#pragma unroll
        for (int q = 0; q < 2 * NP; q++) {
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) {
                c[q] += __shfl_xor_sync(0xffffffffu, c[q], o);
                below[q] = max(below[q], __shfl_xor_sync(0xffffffffu, below[q], o));
                above[q] = min(above[q], __shfl_xor_sync(0xffffffffu, above[q], o));
            }
            if (lane == 0) {
                s_c[warp][q] = c[q];
                s_below[warp][q] = below[q];
                s_above[warp][q] = above[q];
            }
        }
        __syncthreads();
        if (threadIdx.x < NP && threadIdx.x < a.npct) {
            const int k = threadIdx.x;
            int cf = 0, cc = 0;
            long long bf = LLONG_MIN, bc = LLONG_MIN, af = LLONG_MAX, ac = LLONG_MAX;
            for (int w = 0; w < kPctWarps; w++) {
                cf += s_c[w][2 * k];
                cc += s_c[w][2 * k + 1];
                bf = max(bf, s_below[w][2 * k]);
                bc = max(bc, s_below[w][2 * k + 1]);
                af = min(af, s_above[w][2 * k]);
                ac = min(ac, s_above[w][2 * k + 1]);
            }
            const double vk = target_value(total, a.pct[k], a.integral[k]);
            a.out[k * a.cells + cell] = finish(a, vk, floor(vk), ceil(vk), cf, bf, af, cc, bc, ac);
        }
        __syncthreads();
    }
}

template <int NP>
int launch_np(const PctArgs &a, int sm_count, cudaStream_t st) {
    if (a.cells >= kPctCellMin) {
        const long long blocks = std::min<long long>((a.cells + 255) / 256, (long long)sm_count * 8);
        k_pct_cell<NP><<<(unsigned)blocks, 256, 0, st>>>(a);
    } else {
        const long long blocks = std::min<long long>(a.cells, (long long)sm_count * 8);
        k_pct_block<NP><<<(unsigned)blocks, kScanThreads, 0, st>>>(a);
    }
    B200_CUDA(cudaGetLastError());
    return B200_OK;
}

int launch(const PctArgs &a, int sm_count, cudaStream_t st) {
    if (a.npct <= 1)
        return launch_np<1>(a, sm_count, st);
    if (a.npct <= 2)
        return launch_np<2>(a, sm_count, st);
    if (a.npct <= 4)
        return launch_np<4>(a, sm_count, st);
    return launch_np<8>(a, sm_count, st);
}

} // namespace
} // namespace b200

using namespace b200;

extern "C" int b200_grid_percentile(b200_ctx *ctx, int slot, const int64_t *grid, int ndim, const int64_t *sizes, double lb, double span,
                                    const double *pct, const uint8_t *integral, int npct, int memspace_out, double *out) {
    if (!grid || !sizes || ndim < 1 || ndim > B200_MAX_BINNERS || npct < 0 || (npct && (!pct || !integral)) ||
        (memspace_out != B200_MEM_HOST && memspace_out != B200_MEM_DEVICE)) {
        set_error("b200_grid_percentile: invalid argument");
        return B200_ERR_INVALID;
    }
    CallFrame call(ctx, slot, B200_MEM_DEVICE, 0, "b200_grid_percentile");
    B200_CHECK(call.rc);
    PctArgs a = {};
    a.grid = reinterpret_cast<const long long *>(grid);
    a.ndim = ndim - 1;
    a.S = 1;
    a.cells = 1;
    for (int d = 0; d < ndim - 1; d++) {
        if (sizes[d] < 4) {
            set_error("b200_grid_percentile: binby dimension %d has %lld cells; with edges it needs at least 4", d, (long long)sizes[d]);
            return B200_ERR_INVALID;
        }
        a.n[d] = sizes[d] - 3;
        a.stride[d] = a.S;
        a.cells *= a.n[d];
        a.S *= sizes[d];
    }
    const int64_t pfull = sizes[ndim - 1];
    if (pfull < 4 || pfull - 1 > INT_MAX) {
        set_error("b200_grid_percentile: the percentile axis has %lld cells; with edges it needs 4 to 2^31", (long long)pfull);
        return B200_ERR_INVALID;
    }
    a.plen = (int)(pfull - 1);
    a.lb = lb;
    a.span = span;
    a.axis = (double)(pfull - 4);
    if (!npct || !a.cells)
        return B200_OK;
    if (!out) {
        set_error("b200_grid_percentile: invalid argument (out is null)");
        return B200_ERR_INVALID;
    }
    B200_CHECK(b200_ctx_sync(ctx, -1)); // the grid may have been written on any slot
    cudaStream_t st = call.st;
    double *dout;
    B200_CHECK(call.out(out, (size_t)a.cells * npct * sizeof(double), memspace_out == B200_MEM_DEVICE, &dout));
    for (int k0 = 0; k0 < npct; k0 += kPctMax) {
        a.npct = std::min(kPctMax, npct - k0);
        for (int k = 0; k < a.npct; k++) {
            a.pct[k] = pct[k0 + k];
            a.integral[k] = integral[k0 + k] != 0;
        }
        a.out = dout + (size_t)k0 * a.cells;
        B200_CHECK(launch(a, ctx->sm_count, st));
    }
    return call.finish(true);
}
