// mutinfo.cu — the finish of df.mutual_information (vaex/dataframe.py:685-819) on an int64 count grid that is already in device
// memory: for every binby cell, kld.mutual_information (vaex/kld.py:13-21) of that cell's MI sub-grid, with the marginals of
// vaex.utils.disjoined (vaex/utils.py:172-195).
//
// Grid layout (the aggregator's, edges=True): first dimension fastest, the d MI axes first, the binby axes after them.  Every axis is
// sliced [2:-1] (count(..., edges=False)).  Because the MI axes are the fastest, one binby cell's MI block, edges included, is one
// contiguous run of block = Π(m_k + 3) counts; the edge counts inside it are skipped.
//
// Per cell: N = Σc over the interior, the exact int64 marginals M_k[j], q_k[j] = M_k[j] / N, and
//     MI = Σ_{c > 0} P · log(P / Q),   P = c / N,   Q = Π_k q_k[j_k]
// Q is the reference's product of marginals normalised by its own sum: that sum is Π_k Σ_j M_k[j] = N^d exactly, so each factor is
// normalised instead and no rounded N^d enters.  An empty cell gives 0.0 (the reference's mask is empty), d = 1 gives exactly 0.0
// (P and Q are the same division).  Both regimes reduce in a fixed tree without floating-point atomics, and the regime follows from
// the shape alone, so a grid gives the same bits on every run.  The error bound against the reference is in DESIGN.md section 3.
#include "common.cuh"
#include "scan.cuh"

#include <limits.h>
#include <math.h>

#include <algorithm>

namespace b200 {
namespace {

constexpr long long kMiCellMin = 256;          // binby cells from which one CTA per cell (k_mi_cell) is used, ...
constexpr long long kMiCellBlockMax = 1 << 16; // ... when one cell's block holds at most this many counts ...
constexpr int kMiCellMargMax = 2048;           // ... and its marginals fit 16 KB of shared memory
constexpr int kMiChunk = kScanThreads * 16;    // counts per CTA in the split regime
constexpr size_t kMiSmemMax = 48 * 1024;       // dynamic + static shared memory of k_mi_marg without an opt-in: the marginals it
                                               // privatises must fit beside its static block_sum scratch; more go to L2 atomics
constexpr long long kMaxGridY = 65535;

struct MiArgs {
    const long long *grid;
    int d;                                 // MI axes: the first d axes of the grid
    int nb;                                // binby axes
    long long len[B200_MAX_BINNERS];       // MI axis k with its edges: m_k + 3
    int moff[B200_MAX_BINNERS + 1];        // offset of axis k's marginal; moff[d] = Σ m_k
    long long block;                       // Π len[k]: the counts of one binby cell, contiguous
    long long n[B200_MAX_BINNERS];         // sliced size of binby axis j
    long long stride[B200_MAX_BINNERS];    // its stride in the grid
    long long cells;                       // sliced binby cells
    double *out;                           // out[cell], first binner fastest
};

__device__ __forceinline__ const long long *cell_block(const MiArgs &a, long long cell) {
    long long off = 0;
    for (int j = 0; j < a.nb; j++) {
        const long long i = cell % a.n[j];
        cell /= a.n[j];
        off += (i + 2) * a.stride[j];
    }
    return a.grid + off;
}

// the marginal slot of every MI axis for count t of a block; false for a count in an edge row (NaN, underflow, overflow)
template <typename I>
__device__ __forceinline__ bool interior(const MiArgs &a, I t, int idx[B200_MAX_BINNERS]) {
    bool in = true;
#pragma unroll
    for (int k = 0; k < B200_MAX_BINNERS; k++) {
        if (k < a.d) {
            const I l = (I)a.len[k];
            const I j = t % l;
            t /= l;
            in &= j >= 2 && j < l - 1;
            idx[k] = a.moff[k] + (int)j - 2;
        }
    }
    return in;
}

template <typename I>
__device__ __forceinline__ long long add_marginals(const MiArgs &a, const long long *blk, I t0, I t1, long long *marg) {
    long long part = 0;
    for (I t = t0 + threadIdx.x; t < t1; t += kScanThreads) {
        const long long c = blk[t];
        int idx[B200_MAX_BINNERS];
        if (c != 0 && interior(a, t, idx)) {
            part += c;
#pragma unroll
            for (int k = 0; k < B200_MAX_BINNERS; k++)
                if (k < a.d)
                    atomicAdd(reinterpret_cast<unsigned long long *>(marg + idx[k]), (unsigned long long)c);
        }
    }
    return part;
}

// Σ P·log(P/Q) over this thread's counts of [t0, t1); q = the cell's normalised marginals
template <typename I>
__device__ __forceinline__ double add_terms(const MiArgs &a, const long long *blk, I t0, I t1, const double *q, double Nd) {
    double acc = 0.0;
    for (I t = t0 + threadIdx.x; t < t1; t += kScanThreads) {
        const long long c = blk[t];
        int idx[B200_MAX_BINNERS];
        if (c > 0 && interior(a, t, idx)) {
            const double P = __ll2double_rn(c) / Nd;
            double Q = q[idx[0]];
#pragma unroll
            for (int k = 1; k < B200_MAX_BINNERS; k++)
                if (k < a.d)
                    Q *= q[idx[k]];
            if (Q > 0.0)
                acc += P * log(P / Q);
        }
    }
    return acc;
}

// many small cells: one CTA per binby cell, the marginals as exact integers in shared memory, then converted in place to q; the
// block is read twice, the second time from L1 / L2
__global__ void __launch_bounds__(kScanThreads) k_mi_cell(const MiArgs a) {
    extern __shared__ long long s_marg[];
    double *s_q = reinterpret_cast<double *>(s_marg);
    const int msum = a.moff[a.d];
    const unsigned block = (unsigned)a.block;
    for (long long cell = blockIdx.x; cell < a.cells; cell += gridDim.x) {
        for (int i = threadIdx.x; i < msum; i += kScanThreads)
            s_marg[i] = 0;
        __syncthreads();
        const long long *blk = cell_block(a, cell);
        const long long N = block_sum(add_marginals<unsigned>(a, blk, 0u, block, s_marg));
        if (N == 0) {
            if (threadIdx.x == 0)
                a.out[cell] = 0.0;
            continue;
        }
        const double Nd = __ll2double_rn(N);
        for (int i = threadIdx.x; i < msum; i += kScanThreads)
            s_q[i] = __ll2double_rn(s_marg[i]) / Nd;
        __syncthreads();
        const double mi = block_sum(add_terms<unsigned>(a, blk, 0u, block, s_q, Nd));
        if (threadIdx.x == 0)
            a.out[cell] = mi;
    }
}

// few large cells, pass 1: chunk blockIdx.x of every cell adds its counts to the cell's int64 marginals and total in global scratch
// (integer atomics: exact in any order), privatised in shared memory when they fit
__global__ void __launch_bounds__(kScanThreads) k_mi_marg(const MiArgs a, long long *gmarg, long long *gN, int priv) {
    extern __shared__ long long s_marg[];
    const int msum = a.moff[a.d];
    const long long t0 = (long long)blockIdx.x * kMiChunk, t1 = min(a.block, t0 + kMiChunk);
    for (long long cell = blockIdx.y; cell < a.cells; cell += gridDim.y) {
        long long *g = gmarg + cell * msum;
        if (priv) {
            for (int i = threadIdx.x; i < msum; i += kScanThreads)
                s_marg[i] = 0;
            __syncthreads();
        }
        const long long part = block_sum(add_marginals<long long>(a, cell_block(a, cell), t0, t1, priv ? s_marg : g));
        if (threadIdx.x == 0 && part != 0)
            atomicAdd(reinterpret_cast<unsigned long long *>(gN + cell), (unsigned long long)part);
        if (priv) {
            for (int i = threadIdx.x; i < msum; i += kScanThreads)
                if (s_marg[i] != 0)
                    atomicAdd(reinterpret_cast<unsigned long long *>(g + i), (unsigned long long)s_marg[i]);
            __syncthreads();
        }
    }
}

// pass 2: the marginals become q = M / N in place (same 8 bytes per entry)
__global__ void __launch_bounds__(kScanThreads) k_mi_norm(const MiArgs a, long long *gmarg, const long long *gN) {
    const long long msum = a.moff[a.d], n = a.cells * msum;
    for (long long i = blockIdx.x * (long long)kScanThreads + threadIdx.x; i < n; i += (long long)gridDim.x * kScanThreads) {
        const long long N = gN[i / msum];
        reinterpret_cast<double *>(gmarg)[i] = N ? __ll2double_rn(gmarg[i]) / __ll2double_rn(N) : 0.0;
    }
}

// pass 3: every chunk's Σ P·log(P/Q) in a fixed tree, one partial per (cell, chunk)
__global__ void __launch_bounds__(kScanThreads) k_mi_terms(const MiArgs a, const double *gq, const long long *gN, double *partial, long long chunks) {
    const int msum = a.moff[a.d];
    const long long t0 = (long long)blockIdx.x * kMiChunk, t1 = min(a.block, t0 + kMiChunk);
    for (long long cell = blockIdx.y; cell < a.cells; cell += gridDim.y) {
        const long long N = gN[cell];
        double s = 0.0;
        if (N != 0) // uniform over the CTA
            s = block_sum(add_terms<long long>(a, cell_block(a, cell), t0, t1, gq + cell * msum, __ll2double_rn(N)));
        if (threadIdx.x == 0)
            partial[cell * chunks + blockIdx.x] = s;
    }
}

// pass 4: one CTA per cell sums its partials in chunk order per thread, then the fixed tree
__global__ void __launch_bounds__(kScanThreads) k_mi_final(const MiArgs a, const double *partial, long long chunks) {
    for (long long cell = blockIdx.x; cell < a.cells; cell += gridDim.x) {
        double acc = 0.0;
        for (long long i = threadIdx.x; i < chunks; i += kScanThreads)
            acc += partial[cell * chunks + i];
        const double mi = block_sum(acc);
        if (threadIdx.x == 0)
            a.out[cell] = mi;
    }
}

// the split regime's scratch comes from the context's block cache (a fresh allocation per call costs more than the finish) and goes
// back once the stream has finished with it
int launch(b200_ctx *ctx, const MiArgs &a, cudaStream_t st) {
    const int sm_count = ctx->sm_count;
    const int msum = a.moff[a.d];
    if (a.cells >= kMiCellMin && a.block <= kMiCellBlockMax && msum <= kMiCellMargMax) {
        const long long blocks = std::min<long long>(a.cells, (long long)sm_count * 8);
        k_mi_cell<<<(unsigned)blocks, kScanThreads, msum * sizeof(long long), st>>>(a);
        B200_CUDA(cudaGetLastError());
        return B200_OK;
    }
    const long long chunks = (a.block + kMiChunk - 1) / kMiChunk;
    if (chunks > INT_MAX) {
        set_error("b200_grid_mutual_information: %lld counts per binby cell are too many", a.block);
        return B200_ERR_INVALID;
    }
    static size_t marg_static = 0; // k_mi_marg's static shared memory (block_sum's warp sums), read once
    if (!marg_static) {
        cudaFuncAttributes attr;
        B200_CUDA(cudaFuncGetAttributes(&attr, k_mi_marg));
        marg_static = attr.sharedSizeBytes ? attr.sharedSizeBytes : 1;
    }
    const int priv = (size_t)msum * sizeof(long long) + marg_static <= kMiSmemMax;
    const size_t marg_bytes = (size_t)a.cells * msum * 8, n_bytes = (size_t)a.cells * 8, part_bytes = (size_t)a.cells * chunks * 8;
    DevBuf<char> scratch;
    B200_CHECK(scratch.alloc(ctx, marg_bytes + n_bytes + part_bytes, "b200_grid_mutual_information", st));
    long long *gmarg = reinterpret_cast<long long *>(scratch.get()), *gN = reinterpret_cast<long long *>(scratch + marg_bytes);
    double *partial = reinterpret_cast<double *>(scratch + marg_bytes + n_bytes);
    B200_CUDA(cudaMemsetAsync(scratch, 0, marg_bytes + n_bytes, st));
    const dim3 g((unsigned)chunks, (unsigned)std::min(a.cells, kMaxGridY));
    k_mi_marg<<<g, kScanThreads, priv ? msum * sizeof(long long) : 0, st>>>(a, gmarg, gN, priv);
    const long long norm_blocks = std::min<long long>((a.cells * msum + kScanThreads - 1) / kScanThreads, (long long)sm_count * 8);
    k_mi_norm<<<(unsigned)norm_blocks, kScanThreads, 0, st>>>(a, gmarg, gN);
    k_mi_terms<<<g, kScanThreads, 0, st>>>(a, reinterpret_cast<const double *>(gmarg), gN, partial, chunks);
    k_mi_final<<<(unsigned)std::min(a.cells, kMaxGridY), kScanThreads, 0, st>>>(a, partial, chunks);
    B200_CUDA(cudaGetLastError());
    B200_CUDA(cudaStreamSynchronize(st));
    return B200_OK;
}

} // namespace
} // namespace b200

using namespace b200;

extern "C" int b200_grid_mutual_information(b200_ctx *ctx, int slot, const int64_t *grid, int ndim, const int64_t *sizes, int dimension,
                                            int memspace_out, double *out) {
    if (!grid || !sizes || dimension < 1 || ndim < dimension || ndim > B200_MAX_BINNERS || (memspace_out != B200_MEM_HOST && memspace_out != B200_MEM_DEVICE)) {
        set_error("b200_grid_mutual_information: invalid argument");
        return B200_ERR_INVALID;
    }
    CallFrame call(ctx, slot, B200_MEM_DEVICE, 0, "b200_grid_mutual_information");
    B200_CHECK(call.rc);
    MiArgs a = {};
    a.grid = reinterpret_cast<const long long *>(grid);
    a.d = dimension;
    a.nb = ndim - dimension;
    a.block = 1;
    long long msum = 0, stride = 1;
    for (int k = 0; k < ndim; k++) {
        if (sizes[k] < 4 || sizes[k] > INT_MAX || stride > LLONG_MAX / sizes[k]) {
            set_error("b200_grid_mutual_information: axis %d has %lld cells; with edges it needs 4 to 2^31, and the grid fewer than 2^63", k,
                      (long long)sizes[k]);
            return B200_ERR_INVALID;
        }
        if (k < dimension) {
            a.len[k] = sizes[k];
            a.moff[k] = (int)msum;
            msum += sizes[k] - 3;
        } else {
            a.n[k - dimension] = sizes[k] - 3;
            a.stride[k - dimension] = stride;
        }
        stride *= sizes[k];
        if (k == dimension - 1)
            a.block = stride;
    }
    if (msum > INT_MAX) {
        set_error("b200_grid_mutual_information: %lld marginal entries are too many", msum);
        return B200_ERR_INVALID;
    }
    a.moff[dimension] = (int)msum;
    a.cells = 1;
    for (int j = 0; j < a.nb; j++)
        a.cells *= a.n[j];
    if (!out) {
        set_error("b200_grid_mutual_information: invalid argument (out is null)");
        return B200_ERR_INVALID;
    }
    B200_CHECK(b200_ctx_sync(ctx, -1)); // the grid may have been written on any slot
    B200_CHECK(call.out(out, (size_t)a.cells * sizeof(double), memspace_out == B200_MEM_DEVICE, &a.out));
    B200_CHECK(launch(ctx, a, call.st));
    return call.finish(true);
}
