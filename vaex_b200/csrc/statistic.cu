// statistic.cu — the legacy statistics on the device: df.cov / df.correlation / binned df.minmax and the limits pre-pass
// (TaskStatistic, vaex/tasks.py:288-470 -> TaskPartStatistic.process, vaex/cpu.py:510-611 -> vaexfast statisticNd,
// src/vaexfast.cpp:1061-1278).
//
// What is restated bit for bit:
//   * every column is cast to the compute class T (float or double, refvalue.cuh); byte-swapped columns give their native values;
//   * a row masked in any column is dropped from every selection; a selection keeps the rows its mask marks;
//   * binning is statisticNd's, not BinnerScalar's: minima and scale = 1/(max-min) are T, scaled = (v-min)*scale is T (no FMA);
//     without edges a row is kept when 0 <= scaled < 1 and its bin is (int)(scaled*size), a product taken in double except for
//     exactly two dimensions, where it is T; with edges NaN -> 0, < 0 -> 1, >= 1 -> size-1, else (int)(scaled*(size-3))+2 in double;
//   * the grid is C order with the first binby dimension slowest and the op's fields last.
// Accumulators: counts are u64 (exact), sums and products fp64 with __dadd_rn / __dmul_rn semantics (atomicAdd is a correctly
// rounded add; only the order differs from the reference), min/max the sign-split integer atomics of device_utils.cuh, FIRST the
// (order key, global row) 128-bit CAS of cas128.cuh (as first.cu) followed by a deposit pass.  COV keeps the diagonal and one triangle only.
//
// Three accumulation strategies, picked on the host per call:
//   k_stat_reg    no binby, one selection: per-thread registers, warp + block reduction, one global atomic per field per block;
//   k_stat_smem   the whole (selections x cells x fields) accumulator fits in shared memory: a block-private copy, flushed once;
//   k_stat_global otherwise: atomics on the device accumulator.
// FIRST always runs k_stat_first<T, false> (select) + k_stat_first<T, true> (deposit) on the device accumulator.
//
// df.mode's count (vaex/dataframe.py:2006-2034 -> vaex.legacy.TaskHistogram, vaex/legacy.py:22-110 -> vaexfast histogram2d /
// histogram3d / histogramNd, src/vaexfast.cpp:577-600, 818-860, 939-965) is an ADD1 grid of class double built by
// b200_stat_create_histogram.  Two dimensions bin exactly like statisticNd of class double without edges, so they run the statistic
// rule; three or more run the kBinHist rule of histogram3d / histogramNd: a row is kept when min <= v < max and its bin is
// (int)((v-min)*scale) with scale = size/(max-min).  A bin index that rounds up to `size` goes to the last bin, as statisticNd's
// does, and a NaN index (an infinite minimum) drops the row.  Histograms whose 32-bit counts fit shared memory run k_stat_count_smem,
// the others k_stat_global; k_stat_mode is the per-cell argmax finish.
#include <algorithm>
#include <cmath>
#include <vector>

#include "cas128.cuh"
#include "refvalue.cuh"

namespace b200 {
namespace {

constexpr int kThreads = 256;
constexpr size_t kSmemBudget = 96 * 1024;
constexpr size_t kSmemPerSm = 200 * 1024; // of an H100 SM's 228 KB, what the histogram count's CTAs share

enum BinRule { kBinStat, kBinHist }; // statisticNd's bins, or histogram3d / histogramNd's

struct StatCol {
    const void *data;
    const uint8_t *mask; // 1 = masked
    int dt, isz, swap;
};

struct StatParams {
    StatCol bin[B200_MAX_BINNERS];
    StatCol w[B200_STAT_MAX_WEIGHTS];
    const uint8_t *sel[B200_STAT_MAX_SELECTIONS]; // non-zero = keep; NULL = all rows
    double minv[B200_MAX_BINNERS], maxv[B200_MAX_BINNERS], scale[B200_MAX_BINNERS]; // values of class T
    int size[B200_MAX_BINNERS];
    long long stride[B200_MAX_BINNERS]; // in cells
    int ndim, nw, nsel, edges, vec;
    int nc, K; // counts per cell, 8-byte slots per cell (counts first, then fp64 sums / min,max / FIRST state)
    long long nrows, row_offset, cells;
    unsigned long long *acc;
};

__host__ __device__ constexpr int cov_pairs(int n) { return n * (n + 1) / 2; }
__host__ __device__ constexpr int pair_index(int n, int i, int j) { return i * n - i * (i - 1) / 2 + (j - i); } // i <= j

template <typename T>
__device__ __forceinline__ T sub_rn(T a, T b) {
    if constexpr (std::is_same<T, double>::value)
        return __dsub_rn(a, b);
    else
        return __fsub_rn(a, b);
}
template <typename T>
__device__ __forceinline__ T mul_rn(T a, T b) {
    if constexpr (std::is_same<T, double>::value)
        return __dmul_rn(a, b);
    else
        return __fmul_rn(a, b);
}
template <typename T>
__device__ __forceinline__ int trunc_int(T a) {
    if constexpr (std::is_same<T, double>::value)
        return __double2int_rz(a);
    else
        return __float2int_rz(a);
}

// statisticNd's (or, kBinHist, histogram3d / histogramNd's) bin of one value along dimension d; -1 = outside (no edges)
template <typename T, int RULE>
__device__ __forceinline__ int stat_bin(const StatParams &p, int d, T v) {
    const int size = p.size[d];
    if constexpr (RULE == kBinHist) {
        if (!(v >= (T)p.minv[d] && v < (T)p.maxv[d]))
            return -1;
        const T f = mul_rn<T>(sub_rn<T>(v, (T)p.minv[d]), (T)p.scale[d]);
        // (v-min) can round up to max-min, so f can reach `size`: the reference then writes past its row, here the row lands in
        // the last bin.  An infinite minimum gives inf * 0 = NaN, where the reference indexes with INT_MIN: the row is dropped.
        if (f != f)
            return -1;
        return min(trunc_int<T>(f), size - 1);
    }
    const T scaled = mul_rn<T>(sub_rn<T>(v, (T)p.minv[d]), (T)p.scale[d]);
    int b;
    if (p.edges) {
        if (scaled != scaled)
            return 0;
        if (scaled < (T)0)
            return 1;
        if (scaled >= (T)1)
            return size - 1;
        b = __double2int_rz(__dmul_rn((double)scaled, (double)(size - 3))) + 2;
    } else {
        if (!(scaled >= (T)0 && scaled < (T)1))
            return -1;
        b = p.ndim == 2 ? trunc_int<T>(mul_rn<T>(scaled, (T)size)) : __double2int_rz(__dmul_rn((double)scaled, (double)size));
    }
    // scaled < 1 can still round scaled*size up to `size` (the float product of two dimensions, large sizes): the reference then
    // writes past its grid; here such a row lands in the last bin
    return min(b, size - 1);
}

template <typename T>
__device__ __forceinline__ double col_value(const StatCol &c, uint64_t r) {
    return (double)raw_class_value<T>(c.dt, c.swap ? bswap(r, c.isz) : r);
}

// four consecutive rows of a column (128-bit loads when every pointer of the call is 16-byte aligned)
template <typename T>
__device__ __forceinline__ void load4_values(const StatParams &p, const StatCol &c, long long base, int nv, double out[4]) {
    uint64_t r[4];
    if (p.vec)
        load4_raw<true>(c.data, c.isz, base, nv, r);
    else
        load4_raw<false>(c.data, c.isz, base, nv, r);
#pragma unroll
    for (int j = 0; j < 4; j++)
        out[j] = col_value<T>(c, r[j]);
}

__device__ __forceinline__ void drop_masked(const StatParams &p, const StatCol &c, long long base, int nv, bool ok[4]) {
    if (!c.mask)
        return;
    unsigned m[4];
    if (p.vec)
        load4_mask<true>(c.mask, base, nv, m);
    else
        load4_mask<false>(c.mask, base, nv, m);
#pragma unroll
    for (int j = 0; j < 4; j++)
        ok[j] = ok[j] && !m[j];
}

// flat cell of four rows and whether each takes part at all (inside the grid, unmasked in every column)
template <typename T, int RULE>
__device__ __forceinline__ void rows4(const StatParams &p, long long base, int nv, long long idx[4], bool ok[4]) {
#pragma unroll
    for (int j = 0; j < 4; j++)
        idx[j] = 0, ok[j] = j < nv;
    for (int d = 0; d < p.ndim; d++) {
        uint64_t r[4];
        if (p.vec)
            load4_raw<true>(p.bin[d].data, p.bin[d].isz, base, nv, r);
        else
            load4_raw<false>(p.bin[d].data, p.bin[d].isz, base, nv, r);
#pragma unroll
        for (int j = 0; j < 4; j++) {
            const uint64_t b = p.bin[d].swap ? bswap(r[j], p.bin[d].isz) : r[j];
            const int k = stat_bin<T, RULE>(p, d, raw_class_value<T>(p.bin[d].dt, b));
            ok[j] = ok[j] && k >= 0;
            idx[j] += p.stride[d] * (long long)max(k, 0);
        }
        drop_masked(p, p.bin[d], base, nv, ok);
    }
    for (int c = 0; c < p.nw; c++)
        drop_masked(p, p.w[c], base, nv, ok);
}

__device__ __forceinline__ bool selected(const StatParams &p, int s, long long row) { return !p.sel[s] || p.sel[s][row]; }

__device__ __forceinline__ bool isnan_d(double v) { return v != v; }

// the op's update of one cell with one row, through atomics (shared or global memory)
// NT > 0: the row's first NT weight values are in `wv`; NT == 0 (COV with more than 4 weights): they are loaded per row
template <typename T, int OP, int NT>
__device__ __forceinline__ void apply_atomic(const StatParams &p, unsigned long long *a, const double *wv, long long row) {
    double *f = reinterpret_cast<double *>(a);
    if constexpr (OP == B200_STAT_ADD1) {
        atomicAdd(a, 1ull);
    } else if constexpr (OP == B200_STAT_COUNT) {
        if (!isnan_d(wv[0]))
            atomicAdd(a, 1ull);
    } else if constexpr (OP == B200_STAT_MIN_MAX) {
        const double v = wv[0];
        if (!isnan_d(v)) {
            if (v < f[0] || (v == 0.0 && f[0] == 0.0))
                atomic_min_f64(f, v);
            if (v > f[1] || (v == 0.0 && f[1] == 0.0))
                atomic_max_f64(f + 1, v);
        }
    } else if constexpr (OP == B200_STAT_MOMENTS_01 || OP == B200_STAT_MOMENTS_012) {
        const double v = wv[0];
        if (!isnan_d(v)) {
            atomicAdd(a, 1ull);
            atomicAdd(f + 1, v);
            if constexpr (OP == B200_STAT_MOMENTS_012)
                atomicAdd(f + 2, __dmul_rn(v, v));
        }
    } else if constexpr (OP == B200_STAT_COV) {
        const int n = NT ? NT : p.nw, P = cov_pairs(n), nc = p.nc;
        auto val = [&](int i) { return NT ? wv[i] : col_value<T>(p.w[i], ldcs1_raw(p.w[i].data, p.w[i].isz, row)); };
        for (int i = 0; i < n; i++) {
            const double x = val(i);
            if (isnan_d(x))
                continue;
            atomicAdd(a + i, 1ull);
            atomicAdd(f + nc + i, x);
            for (int j = i; j < n; j++) {
                const double y = j == i ? x : val(j);
                if (isnan_d(y))
                    continue;
                const int q = n + pair_index(n, i, j);
                atomicAdd(a + q, 1ull);
                atomicAdd(f + nc + q, __dmul_rn(x, y));
            }
        }
        (void)P;
    }
}

// the weights of four rows held in registers
template <typename T, int NT>
__device__ __forceinline__ void weights4(const StatParams &p, long long base, int nv, double wv[][4]) {
#pragma unroll
    for (int c = 0; c < NT; c++)
        if (c < p.nw)
            load4_values<T>(p, p.w[c], base, nv, wv[c]);
}

template <typename T, int OP, int NT, int RULE>
__device__ __forceinline__ void bin_rows_atomic(const StatParams &p, unsigned long long *acc) {
    constexpr int W = NT > 0 ? NT : 1;
    const long long step = (long long)gridDim.x * kThreads * 4;
    for (long long base = ((long long)blockIdx.x * kThreads + threadIdx.x) * 4; base < p.nrows; base += step) {
        const long long left = p.nrows - base;
        const int nv = left < 4 ? (int)left : 4;
        long long idx[4];
        bool ok[4];
        rows4<T, RULE>(p, base, nv, idx, ok);
        double wv[W][4];
        if constexpr (NT > 0)
            weights4<T, NT>(p, base, nv, wv);
#pragma unroll
        for (int j = 0; j < 4; j++) {
            if (!ok[j])
                continue;
            double w[W];
#pragma unroll
            for (int c = 0; c < W; c++)
                w[c] = NT > 0 ? wv[c][j] : 0.0;
            for (int s = 0; s < p.nsel; s++)
                if (selected(p, s, base + j))
                    apply_atomic<T, OP, NT>(p, acc + ((long long)s * p.cells + idx[j]) * p.K, w, base + j);
        }
    }
}

__device__ __forceinline__ unsigned long long init_slot(const StatParams &p, int op, int k) {
    if (op == B200_STAT_MIN_MAX)
        return k == 0 ? 0x7ff0000000000000ULL : 0xfff0000000000000ULL; // (+inf, -inf): StatOpMinMax.init
    return 0;
}

template <typename T, int OP, int NT, int RULE>
__global__ void __launch_bounds__(kThreads) k_stat_global(const __grid_constant__ StatParams p) {
    bin_rows_atomic<T, OP, NT, RULE>(p, p.acc);
}

// the histogram's ADD1 count with one selection in a block-private grid of 32-bit counts (half the shared memory of k_stat_smem's
// 64-bit slots, so mode's default 64 x 256 grid fits), flushed once into the 64-bit device grid.  The host picks it only when no
// CTA can see 2^32 rows.
template <int RULE>
__global__ void __launch_bounds__(kThreads) k_stat_count_smem(const __grid_constant__ StatParams p) {
    extern __shared__ unsigned scount[];
    for (long long i = threadIdx.x; i < p.cells; i += kThreads)
        scount[i] = 0;
    __syncthreads();
    const long long step = (long long)gridDim.x * kThreads * 4;
    for (long long base = ((long long)blockIdx.x * kThreads + threadIdx.x) * 4; base < p.nrows; base += step) {
        const long long left = p.nrows - base;
        const int nv = left < 4 ? (int)left : 4;
        long long idx[4];
        bool ok[4];
        rows4<double, RULE>(p, base, nv, idx, ok);
#pragma unroll
        for (int j = 0; j < 4; j++)
            if (ok[j] && selected(p, 0, base + j))
                atomicAdd(scount + idx[j], 1u);
    }
    __syncthreads();
    for (long long i = threadIdx.x; i < p.cells; i += kThreads)
        if (scount[i])
            atomicAdd(p.acc + i, (unsigned long long)scount[i]);
}

// mode's finish: one thread per cell of axes 1.. walks axis 0 (coalesced across cells) and keeps its first maximum, as np.argmax;
// an all-zero cell gives NaN
__global__ void __launch_bounds__(kThreads) k_stat_mode(const unsigned long long *counts, int n0, long long cells, const double *centers, double *out) {
    for (long long c = (long long)blockIdx.x * kThreads + threadIdx.x; c < cells; c += (long long)gridDim.x * kThreads) {
        unsigned long long best = 0;
        int at = 0;
        for (int m = 0; m < n0; m++) {
            const unsigned long long v = counts[(long long)m * cells + c];
            if (v > best)
                best = v, at = m;
        }
        out[c] = best ? centers[at] : __longlong_as_double(0x7ff8000000000000LL);
    }
}

template <typename T, int OP, int NT, int RULE>
__global__ void __launch_bounds__(kThreads) k_stat_smem(const __grid_constant__ StatParams p) {
    extern __shared__ unsigned long long sacc[];
    const long long n = (long long)p.nsel * p.cells * p.K;
    for (long long i = threadIdx.x; i < n; i += kThreads)
        sacc[i] = init_slot(p, OP, (int)(i % p.K));
    __syncthreads();
    bin_rows_atomic<T, OP, NT, RULE>(p, sacc);
    __syncthreads();
    for (long long i = threadIdx.x; i < n; i += kThreads) {
        const unsigned long long v = sacc[i];
        const int k = (int)(i % p.K);
        if (v == init_slot(p, OP, k))
            continue;
        if (OP == B200_STAT_MIN_MAX)
            k == 0 ? atomic_min_f64(reinterpret_cast<double *>(p.acc + i), __longlong_as_double(v))
                   : atomic_max_f64(reinterpret_cast<double *>(p.acc + i), __longlong_as_double(v));
        else if (k < p.nc)
            atomicAdd(p.acc + i, v);
        else
            atomicAdd(reinterpret_cast<double *>(p.acc + i), __longlong_as_double(v));
    }
}

// min / max that order -0.0 below +0.0 (the rule of the sign-split atomics)
__device__ __forceinline__ double min0(double a, double b) { return (b < a || (b == a && signbit(b))) ? b : a; }
__device__ __forceinline__ double max0(double a, double b) { return (b > a || (b == a && !signbit(b))) ? b : a; }

template <int OP, int NT>
struct RegShape {
    static constexpr int nc = OP == B200_STAT_COV ? NT + cov_pairs(NT) : (OP == B200_STAT_MIN_MAX ? 0 : 1);
    static constexpr int ns = OP == B200_STAT_COV ? NT + cov_pairs(NT) : (OP == B200_STAT_MOMENTS_01 ? 1 : OP == B200_STAT_MOMENTS_012 ? 2 : 0);
};

// no binby, one selection: every row lands in the one cell, so each thread keeps the cell in registers
template <typename T, int OP, int NT>
__global__ void __launch_bounds__(kThreads) k_stat_reg(const __grid_constant__ StatParams p) {
    constexpr int NC = RegShape<OP, NT>::nc, NS = RegShape<OP, NT>::ns, W = NT;
    unsigned long long c[NC > 0 ? NC : 1];
    double s[NS > 0 ? NS : 1];
    double lo = INFINITY, hi = -INFINITY;
#pragma unroll
    for (int k = 0; k < NC; k++)
        c[k] = 0;
#pragma unroll
    for (int k = 0; k < NS; k++)
        s[k] = 0.0;
    const long long step = (long long)gridDim.x * kThreads * 4;
    for (long long base = ((long long)blockIdx.x * kThreads + threadIdx.x) * 4; base < p.nrows; base += step) {
        const long long left = p.nrows - base;
        const int nv = left < 4 ? (int)left : 4;
        bool ok[4];
#pragma unroll
        for (int j = 0; j < 4; j++)
            ok[j] = j < nv;
        for (int k = 0; k < p.nw; k++)
            drop_masked(p, p.w[k], base, nv, ok);
        double wv[W][4];
        weights4<T, NT>(p, base, nv, wv);
#pragma unroll
        for (int j = 0; j < 4; j++) {
            if (!ok[j] || !selected(p, 0, base + j))
                continue;
            if constexpr (OP == B200_STAT_ADD1) {
                c[0]++;
            } else if constexpr (OP == B200_STAT_COUNT) {
                c[0] += !isnan_d(wv[0][j]);
            } else if constexpr (OP == B200_STAT_MIN_MAX) {
                const double v = wv[0][j];
                if (!isnan_d(v))
                    lo = min0(lo, v), hi = max0(hi, v);
            } else if constexpr (OP == B200_STAT_MOMENTS_01 || OP == B200_STAT_MOMENTS_012) {
                const double v = wv[0][j];
                if (!isnan_d(v)) {
                    c[0]++;
                    s[0] = __dadd_rn(s[0], v);
                    if constexpr (OP == B200_STAT_MOMENTS_012)
                        s[1] = __dadd_rn(s[1], __dmul_rn(v, v));
                }
            } else if constexpr (OP == B200_STAT_COV) {
#pragma unroll
                for (int i = 0; i < NT; i++) {
                    const double x = wv[i][j];
                    const bool xi = !isnan_d(x);
                    c[i] += xi;
                    s[i] = xi ? __dadd_rn(s[i], x) : s[i];
#pragma unroll
                    for (int k = i; k < NT; k++) {
                        const double y = wv[k][j];
                        const bool both = xi && !isnan_d(y);
                        const int q = NT + pair_index(NT, i, k);
                        c[q] += both;
                        s[q] = both ? __dadd_rn(s[q], __dmul_rn(x, y)) : s[q];
                    }
                }
            }
        }
    }
    // warp, then block: one global update per field per block
#pragma unroll
    for (int o = 16; o; o >>= 1) {
#pragma unroll
        for (int k = 0; k < NC; k++)
            c[k] += __shfl_xor_sync(0xffffffffu, c[k], o);
#pragma unroll
        for (int k = 0; k < NS; k++)
            s[k] = __dadd_rn(s[k], __shfl_xor_sync(0xffffffffu, s[k], o));
        if (OP == B200_STAT_MIN_MAX) {
            lo = min0(lo, __shfl_xor_sync(0xffffffffu, lo, o));
            hi = max0(hi, __shfl_xor_sync(0xffffffffu, hi, o));
        }
    }
    constexpr int KR = OP == B200_STAT_MIN_MAX ? 2 : NC + NS;
    __shared__ unsigned long long red[kThreads / 32][KR];
    const int warp = threadIdx.x >> 5;
    if ((threadIdx.x & 31) == 0) {
        if (OP == B200_STAT_MIN_MAX) {
            red[warp][0] = (unsigned long long)__double_as_longlong(lo);
            red[warp][1] = (unsigned long long)__double_as_longlong(hi);
        } else {
#pragma unroll
            for (int k = 0; k < NC; k++)
                red[warp][k] = c[k];
#pragma unroll
            for (int k = 0; k < NS; k++)
                red[warp][NC + k] = (unsigned long long)__double_as_longlong(s[k]);
        }
    }
    __syncthreads();
    const int k = threadIdx.x;
    if (k >= KR)
        return;
    if (OP == B200_STAT_MIN_MAX) {
        double v = __longlong_as_double(red[0][k]);
        for (int w = 1; w < kThreads / 32; w++)
            v = k == 0 ? min0(v, __longlong_as_double(red[w][k])) : max0(v, __longlong_as_double(red[w][k]));
        if (k == 0 && v < INFINITY)
            atomic_min_f64(reinterpret_cast<double *>(p.acc), v);
        if (k == 1 && v > -INFINITY)
            atomic_max_f64(reinterpret_cast<double *>(p.acc) + 1, v);
    } else if (k < NC) {
        unsigned long long v = 0;
        for (int w = 0; w < kThreads / 32; w++)
            v += red[w][k];
        if (v)
            atomicAdd(p.acc + k, v);
    } else {
        double v = 0.0;
        for (int w = 0; w < kThreads / 32; w++)
            v = __dadd_rn(v, __longlong_as_double(red[w][k]));
        atomicAdd(reinterpret_cast<double *>(p.acc) + k, v);
    }
}

// ---- FIRST: (order key, global row) minimum per cell, then the winning row deposits its value and order ----------------------
template <typename T, bool DEPOSIT>
__global__ void __launch_bounds__(kThreads) k_stat_first(const __grid_constant__ StatParams p) {
    const long long step = (long long)gridDim.x * kThreads * 4;
    for (long long base = ((long long)blockIdx.x * kThreads + threadIdx.x) * 4; base < p.nrows; base += step) {
        const long long left = p.nrows - base;
        const int nv = left < 4 ? (int)left : 4;
        long long idx[4];
        bool ok[4];
        rows4<T, kBinStat>(p, base, nv, idx, ok);
        double wv[2][4];
        weights4<T, 2>(p, base, nv, wv);
#pragma unroll
        for (int j = 0; j < 4; j++) {
            const double order = wv[1][j];
            if (!ok[j] || !(order < INFINITY)) // NaN and +inf orders never beat the initial +inf
                continue;
            const U128 kr{order_key_f64(order), (unsigned long long)(p.row_offset + base + j)};
            for (int s = 0; s < p.nsel; s++) {
                if (!selected(p, s, base + j))
                    continue;
                unsigned long long *st = p.acc + ((long long)s * p.cells + idx[j]) * p.K;
                if (DEPOSIT) {
                    const U128 cur = load128(st);
                    if (cur.lo == kr.lo && cur.hi == kr.hi) {
                        st[2] = (unsigned long long)__double_as_longlong(wv[0][j]);
                        st[3] = (unsigned long long)__double_as_longlong(order);
                    }
                    continue;
                }
                cas128_min(st, kr);
            }
        }
    }
}

__global__ void k_stat_fill(unsigned long long *acc, long long n, int K, int op) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const int k = (int)(i % K);
        unsigned long long v = 0;
        if (op == B200_STAT_MIN_MAX)
            v = k == 0 ? 0x7ff0000000000000ULL : 0xfff0000000000000ULL;
        else if (op == B200_STAT_FIRST) // {order key, row} = max, value NaN, order +inf: StatOpFirst.init
            v = k < 2 ? ~0ULL : (k == 2 ? 0x7ff8000000000000ULL : 0x7ff0000000000000ULL);
        acc[i] = v;
    }
}

template <typename Kern>
int launch(Kern k, b200_ctx *ctx, cudaStream_t st, const StatParams &p, int per_sm, size_t smem) {
    if (smem > 48 * 1024)
        B200_CUDA(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    const long long want = (p.nrows + 4LL * kThreads - 1) / (4LL * kThreads);
    const int blocks = (int)std::max<long long>(1, std::min<long long>(want, (long long)ctx->sm_count * per_sm));
    k<<<blocks, kThreads, smem, st>>>(p);
    B200_CUDA(cudaGetLastError());
    return B200_OK;
}

enum Strategy { kReg, kSmem, kGlobal, kFirst, kCountSmem };

template <typename T, int OP, int NT, int RULE = kBinStat>
int launch_op(b200_ctx *ctx, cudaStream_t st, const StatParams &p, Strategy s) {
    const size_t bytes = (size_t)p.nsel * p.cells * p.K * 8;
    if constexpr (OP != B200_STAT_FIRST) {
        if (s == kReg) {
            if constexpr (NT > 0)
                return launch(k_stat_reg<T, OP, NT>, ctx, st, p, 8, 0);
        } else if (s == kSmem) {
            if constexpr (RULE == kBinStat) // histograms count in k_stat_count_smem
                return launch(k_stat_smem<T, OP, NT, RULE>, ctx, st, p, bytes > 48 * 1024 ? 2 : 4, bytes);
        } else if (s == kCountSmem) {
            if constexpr (OP == B200_STAT_ADD1) {
                const size_t sbytes = (size_t)p.cells * 4;
                return launch(k_stat_count_smem<RULE>, ctx, st, p, (int)std::max<size_t>(1, std::min<size_t>(8, kSmemPerSm / sbytes)), sbytes);
            }
        } else {
            return launch(k_stat_global<T, OP, NT, RULE>, ctx, st, p, 8, 0);
        }
    } else {
        B200_CHECK(launch(k_stat_first<T, false>, ctx, st, p, 8, 0));
        return launch(k_stat_first<T, true>, ctx, st, p, 8, 0);
    }
    set_error("b200_stat_bin: no kernel for this op and strategy");
    return B200_ERR_UNSUPPORTED;
}

template <typename T>
int launch_class(b200_ctx *ctx, cudaStream_t st, const StatParams &p, int op, Strategy s) {
    switch (op) {
    case B200_STAT_ADD1: return launch_op<T, B200_STAT_ADD1, 2>(ctx, st, p, s);
    case B200_STAT_COUNT: return launch_op<T, B200_STAT_COUNT, 2>(ctx, st, p, s);
    case B200_STAT_MIN_MAX: return launch_op<T, B200_STAT_MIN_MAX, 2>(ctx, st, p, s);
    case B200_STAT_MOMENTS_01: return launch_op<T, B200_STAT_MOMENTS_01, 2>(ctx, st, p, s);
    case B200_STAT_MOMENTS_012: return launch_op<T, B200_STAT_MOMENTS_012, 2>(ctx, st, p, s);
    case B200_STAT_FIRST: return launch_op<T, B200_STAT_FIRST, 2>(ctx, st, p, s);
    default: // COV: up to four weights are held in registers for four rows at a time, more are read per row
        switch (p.nw) {
        case 1: return launch_op<T, B200_STAT_COV, 1>(ctx, st, p, s);
        case 2: return launch_op<T, B200_STAT_COV, 2>(ctx, st, p, s);
        case 3: return launch_op<T, B200_STAT_COV, 3>(ctx, st, p, s);
        case 4: return launch_op<T, B200_STAT_COV, 4>(ctx, st, p, s);
        default: return launch_op<T, B200_STAT_COV, 0>(ctx, st, p, s);
        }
    }
}

int op_fields(int op, int nw) {
    switch (op) {
    case B200_STAT_ADD1:
    case B200_STAT_COUNT: return 1;
    case B200_STAT_MIN_MAX:
    case B200_STAT_MOMENTS_01:
    case B200_STAT_FIRST: return 2;
    case B200_STAT_MOMENTS_012: return 3;
    default: return 2 * nw + 2 * nw * nw;
    }
}

} // namespace
} // namespace b200

using namespace b200;

struct b200_stat {
    b200_ctx *ctx = nullptr;
    int op = 0, cls = 0, ndim = 0, edges = 0, nw = 0, nsel = 0;
    int nc = 0, K = 0; // device layout per cell (see StatParams)
    bool hist = false;   // b200_stat_create_histogram: df.mode's count
    int rule = kBinStat; // its bin rule
    bool empty = false;  // histogram2d with a non-finite limit counts nothing
    int64_t sizes[B200_MAX_BINNERS] = {};
    double minv[B200_MAX_BINNERS] = {}, maxv[B200_MAX_BINNERS] = {}, scale[B200_MAX_BINNERS] = {};
    long long stride[B200_MAX_BINNERS] = {};
    long long cells = 1;
    DevBuf<unsigned long long> acc;
    size_t bytes = 0;
    cudaEvent_t chain = nullptr; // FIRST: select + deposit pairs of different slots must not interleave
    std::mutex chain_mu;

    ~b200_stat() {
        if (chain)
            cudaEventDestroy(chain);
    }
};

static int stat_fill(b200_stat *s, cudaStream_t st) {
    const long long n = (long long)(s->bytes / 8);
    k_stat_fill<<<(int)std::min<long long>((n + 255) / 256, kSmCount * 4), 256, 0, st>>>(s->acc, n, s->K, s->op);
    B200_CUDA(cudaGetLastError());
    return B200_OK;
}

extern "C" {

int b200_stat_create(b200_ctx *ctx, int op, int cls, int ndim, const int64_t *sizes, const double *minima, const double *maxima, int edges,
                     int nweights, int nselections, b200_stat **out) {
    if (!ctx || !out || op < B200_STAT_ADD1 || op > B200_STAT_FIRST || (cls != B200_F64 && cls != B200_F32) || ndim < 0 || nweights < 0 ||
        nselections < 1 || (ndim && (!sizes || !minima || !maxima))) {
        set_error("b200_stat_create: invalid argument");
        return B200_ERR_INVALID;
    }
    if (ndim > B200_MAX_BINNERS || nweights > B200_STAT_MAX_WEIGHTS || nselections > B200_STAT_MAX_SELECTIONS) {
        set_error("b200_stat_create: at most %d dimensions, %d weights and %d selections", B200_MAX_BINNERS, B200_STAT_MAX_WEIGHTS,
                  B200_STAT_MAX_SELECTIONS);
        return B200_ERR_UNSUPPORTED;
    }
    const int need = op == B200_STAT_ADD1 ? 0 : op == B200_STAT_FIRST ? 2 : 1;
    if (nweights < need) {
        set_error("b200_stat_create: op %d needs %d weight(s), got %d", op, need, nweights);
        return B200_ERR_INVALID;
    }
    std::unique_ptr<b200_stat, int (*)(b200_stat *)> s(new b200_stat, b200_stat_destroy);
    s->ctx = ctx, s->op = op, s->cls = cls, s->ndim = ndim, s->edges = edges != 0, s->nw = nweights, s->nsel = nselections;
    for (int d = ndim - 1; d >= 0; d--) { // C order: the first dimension is the slowest
        if (sizes[d] < 1 || sizes[d] > (1LL << 30) || (edges && sizes[d] < 3)) {
            set_error("b200_stat_create: invalid size %lld of dimension %d", (long long)sizes[d], d);
            return B200_ERR_INVALID;
        }
        s->sizes[d] = sizes[d];
        s->stride[d] = s->cells;
        if (s->cells > (1LL << 40) / sizes[d]) {
            set_error("b200_stat_create: grid too large");
            return B200_ERR_INVALID;
        }
        s->cells *= sizes[d];
        // statisticNd_: minima / maxima cast to T, scale = 1 / (max - min) in T (src/vaexfast.cpp:1186-1188, 1444-1445)
        if (cls == B200_F32) {
            const float lo = (float)minima[d], hi = (float)maxima[d];
            volatile float diff = hi - lo;
            s->minv[d] = lo, s->scale[d] = (float)(1.0f / diff);
        } else {
            volatile double diff = maxima[d] - minima[d];
            s->minv[d] = minima[d], s->scale[d] = 1.0 / diff;
        }
    }
    const int n = nweights;
    switch (op) {
    case B200_STAT_ADD1:
    case B200_STAT_COUNT: s->nc = 1, s->K = 1; break;
    case B200_STAT_MIN_MAX: s->nc = 0, s->K = 2; break;
    case B200_STAT_MOMENTS_01: s->nc = 1, s->K = 2; break;
    case B200_STAT_MOMENTS_012: s->nc = 1, s->K = 3; break;
    case B200_STAT_COV: s->nc = n + cov_pairs(n), s->K = 2 * s->nc; break;
    default: s->nc = 0, s->K = 4; break;
    }
    s->bytes = (size_t)nselections * s->cells * s->K * 8;
    B200_CUDA(cudaSetDevice(ctx->device));
    B200_CHECK(s->acc.alloc(ctx, s->bytes, "b200_stat_create"));
    B200_CUDA(cudaEventCreateWithFlags(&s->chain, cudaEventDisableTiming));
    cudaStream_t st = ctx->slots[0]->stream;
    B200_CHECK(stat_fill(s.get(), st));
    B200_CUDA(cudaStreamSynchronize(st));
    *out = s.release();
    return B200_OK;
}

int b200_stat_create_histogram(b200_ctx *ctx, int ndim, const int64_t *sizes, const double *minima, const double *maxima, b200_stat **out) {
    if (!ctx || !out || ndim < 2 || ndim > B200_MAX_BINNERS || !sizes || !minima || !maxima) {
        set_error("b200_stat_create_histogram: invalid argument (2 to %d dimensions)", B200_MAX_BINNERS);
        return B200_ERR_INVALID;
    }
    for (int d = 1; ndim > 3 && d < ndim; d++)
        if (sizes[d] != sizes[0]) { // histogramNd scales block e by count_sizes[e] but strides it by axis ndim-1-e
            set_error("b200_stat_create_histogram: %d dimensions need equal sizes (histogramNd mixes up the axes of unequal ones)", ndim);
            return B200_ERR_UNSUPPORTED;
        }
    b200_stat *raw = nullptr;
    B200_CHECK(b200_stat_create(ctx, B200_STAT_ADD1, B200_F64, ndim, sizes, minima, maxima, 0, 0, 1, &raw));
    raw->hist = true;
    raw->rule = ndim == 2 ? kBinStat : kBinHist;
    for (int d = 0; d < ndim; d++) {
        raw->maxv[d] = maxima[d];
        raw->empty |= ndim == 2 && !(std::isfinite(minima[d]) && std::isfinite(maxima[d])); // src/vaexfast.cpp:582-583
        if (ndim > 2) {
            volatile double diff = maxima[d] - minima[d]; // histogram3d / histogramNd: scale = size / (max - min)
            raw->scale[d] = (double)sizes[d] / diff;
        }
    }
    *out = raw;
    return B200_OK;
}

int b200_stat_mode(b200_stat *s, const double *centers, double *out) {
    if (!s || !s->hist || !centers || !out) {
        set_error("b200_stat_mode: invalid argument (a histogram of b200_stat_create_histogram, centers and out)");
        return B200_ERR_INVALID;
    }
    b200_ctx *ctx = s->ctx;
    B200_CUDA(cudaSetDevice(ctx->device));
    B200_CHECK(b200_ctx_sync(ctx, -1)); // the grid may have been written on any slot
    Slot *sl = ctx->slots[0];
    std::lock_guard<std::mutex> lock(sl->mu);
    cudaStream_t st = sl->stream;
    const int n0 = (int)s->sizes[0];
    const long long cells = s->cells / n0;
    DevBuf<double> dev;
    B200_CHECK(dev.alloc(ctx, (size_t)(n0 + cells) * sizeof(double), "b200_stat_mode", st));
    B200_CUDA(cudaMemcpyAsync(dev, centers, (size_t)n0 * sizeof(double), cudaMemcpyHostToDevice, st));
    const long long blocks = std::max<long long>(1, std::min<long long>((cells + kThreads - 1) / kThreads, (long long)ctx->sm_count * 8));
    k_stat_mode<<<(unsigned)blocks, kThreads, 0, st>>>(s->acc, n0, cells, dev, dev + n0);
    B200_CUDA(cudaGetLastError());
    B200_CUDA(cudaMemcpyAsync(out, dev + n0, (size_t)cells * sizeof(double), cudaMemcpyDeviceToHost, st));
    B200_CUDA(cudaStreamSynchronize(st));
    return B200_OK;
}

int b200_stat_destroy(b200_stat *s) {
    if (!s)
        return B200_OK;
    cudaSetDevice(s->ctx->device);
    for (Slot *sl : s->ctx->slots)
        cudaStreamSynchronize(sl->stream);
    delete s;
    return B200_OK;
}

int b200_stat_fields(const b200_stat *s) { return s ? op_fields(s->op, s->nw) : B200_ERR_INVALID; }

int b200_stat_reset(b200_stat *s) {
    if (!s) {
        set_error("b200_stat_reset: null");
        return B200_ERR_INVALID;
    }
    B200_CUDA(cudaSetDevice(s->ctx->device));
    B200_CHECK(b200_ctx_sync(s->ctx, -1));
    cudaStream_t st = s->ctx->slots[0]->stream;
    B200_CHECK(stat_fill(s, st));
    B200_CUDA(cudaStreamSynchronize(st));
    return B200_OK;
}

int b200_stat_bin(b200_stat *s, int slot, const b200_stat_column *binby, const b200_stat_column *weights, const uint8_t *const *selections,
                  int64_t nrows, int64_t row_offset, int memspace, uint32_t flags) {
    if (!s || nrows < 0 || (s->ndim && !binby) || (s->nw && !weights)) {
        set_error("b200_stat_bin: invalid argument");
        return B200_ERR_INVALID;
    }
    CallFrame call(s->ctx, slot, memspace, flags, "b200_stat_bin");
    B200_CHECK(call.rc);
    for (int i = 0; i < s->ndim + s->nw; i++) {
        const b200_stat_column &c = i < s->ndim ? binby[i] : weights[i - s->ndim];
        if (c.dtype < 0 || c.dtype >= B200_NDTYPE || (nrows && !c.data)) {
            set_error("b200_stat_bin: invalid column %d", i);
            return B200_ERR_INVALID;
        }
    }
    if (nrows == 0 || s->empty)
        return B200_OK;
    b200_ctx *ctx = s->ctx;
    cudaStream_t st = call.st;
    for (int i = 0; i < s->ndim + s->nw; i++) {
        const b200_stat_column &c = i < s->ndim ? binby[i] : weights[i - s->ndim];
        call.plan(c.data, (size_t)nrows * dtype_size(c.dtype));
        if (c.mask)
            call.plan(c.mask, (size_t)nrows);
    }
    for (int k = 0; selections && k < s->nsel; k++)
        if (selections[k])
            call.plan(selections[k], (size_t)nrows);
    B200_CHECK(call.commit());

    StatParams p;
    memset(&p, 0, sizeof p);
    bool vec = true;
    auto dev = [&](const void *h) {
        const void *d = call.dev(h);
        if (d && (reinterpret_cast<uintptr_t>(d) & 15))
            vec = false;
        return d;
    };
    auto col = [&](const b200_stat_column &c) {
        StatCol r;
        r.data = dev(c.data);
        r.mask = static_cast<const uint8_t *>(dev(c.mask));
        r.dt = c.dtype;
        r.isz = dtype_size(c.dtype);
        r.swap = c.byteswap && r.isz > 1;
        return r;
    };
    for (int d = 0; d < s->ndim; d++) {
        p.bin[d] = col(binby[d]);
        p.minv[d] = s->minv[d], p.maxv[d] = s->maxv[d], p.scale[d] = s->scale[d], p.size[d] = (int)s->sizes[d], p.stride[d] = s->stride[d];
    }
    for (int k = 0; k < s->nw; k++)
        p.w[k] = col(weights[k]);
    for (int k = 0; selections && k < s->nsel; k++)
        p.sel[k] = static_cast<const uint8_t *>(dev(selections[k]));
    p.ndim = s->ndim, p.nw = s->nw, p.nsel = s->nsel, p.edges = s->edges, p.vec = vec;
    p.nc = s->nc, p.K = s->K;
    p.nrows = nrows, p.row_offset = row_offset, p.cells = s->cells;
    p.acc = s->acc;

    Strategy strat;
    if (s->hist) {
        strat = (size_t)s->cells * 4 <= kSmemBudget && nrows < (1LL << 32) ? kCountSmem : kGlobal;
        const int rc = s->rule == kBinHist ? launch_op<double, B200_STAT_ADD1, 2, kBinHist>(ctx, st, p, strat)
                                           : launch_op<double, B200_STAT_ADD1, 2, kBinStat>(ctx, st, p, strat);
        B200_CHECK(rc);
        return call.finish();
    }
    if (s->op == B200_STAT_FIRST)
        strat = kFirst;
    else if (s->ndim == 0 && s->nsel == 1 && (s->op != B200_STAT_COV || s->nw <= 4))
        strat = kReg;
    else if (s->bytes <= kSmemBudget)
        strat = kSmem;
    else
        strat = kGlobal;
    int rc;
    if (strat == kFirst) {
        std::lock_guard<std::mutex> chain(s->chain_mu);
        B200_CUDA(cudaStreamWaitEvent(st, s->chain, 0));
        rc = s->cls == B200_F64 ? launch_class<double>(ctx, st, p, s->op, strat) : launch_class<float>(ctx, st, p, s->op, strat);
        B200_CHECK(rc);
        B200_CUDA(cudaEventRecord(s->chain, st));
    } else {
        rc = s->cls == B200_F64 ? launch_class<double>(ctx, st, p, s->op, strat) : launch_class<float>(ctx, st, p, s->op, strat);
        B200_CHECK(rc);
    }
    return call.finish();
}

int b200_stat_read(b200_stat *s, double *out) {
    if (!s || !out) {
        set_error("b200_stat_read: invalid argument");
        return B200_ERR_INVALID;
    }
    B200_CUDA(cudaSetDevice(s->ctx->device));
    B200_CHECK(b200_ctx_sync(s->ctx, -1));
    std::vector<unsigned long long> h(s->bytes / 8);
    B200_CUDA(cudaMemcpy(h.data(), s->acc, s->bytes, cudaMemcpyDeviceToHost));
    const int F = op_fields(s->op, s->nw), K = s->K, nc = s->nc, n = s->nw;
    auto dbl = [](unsigned long long b) {
        double d;
        memcpy(&d, &b, 8);
        return d;
    };
    const long long total = (long long)s->nsel * s->cells;
    for (long long c = 0; c < total; c++) {
        const unsigned long long *a = h.data() + c * K;
        double *o = out + c * F;
        switch (s->op) {
        case B200_STAT_ADD1:
        case B200_STAT_COUNT: o[0] = (double)a[0]; break;
        case B200_STAT_MIN_MAX: o[0] = dbl(a[0]), o[1] = dbl(a[1]); break;
        case B200_STAT_MOMENTS_012: o[2] = dbl(a[2]); // fall through
        case B200_STAT_MOMENTS_01: o[0] = (double)a[0], o[1] = dbl(a[1]); break;
        case B200_STAT_FIRST: o[0] = dbl(a[2]), o[1] = dbl(a[3]); break;
        default: // COV: per-column counts and sums, then the N x N pair counts and products, mirrored from one triangle
            for (int i = 0; i < n; i++) {
                o[i] = (double)a[i];
                o[n + i] = dbl(a[nc + i]);
                for (int j = i; j < n; j++) {
                    const int q = n + pair_index(n, i, j);
                    o[2 * n + i * n + j] = o[2 * n + j * n + i] = (double)a[q];
                    o[2 * n + n * n + i * n + j] = o[2 * n + n * n + j * n + i] = dbl(a[nc + q]);
                }
            }
        }
    }
    return B200_OK;
}

} // extern "C"
