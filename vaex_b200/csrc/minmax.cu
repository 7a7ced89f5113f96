// minmax.cu — the limits pre-pass: df.minmax(expression) on the device (SURVEY.md section 8f row 1).
//
// Reference: DataFrame.minmax -> TaskStatistic(OP_MIN_MAX) (vaex/dataframe.py:1519-1528) -> TaskPartStatistic.process
// (vaex/cpu.py:513-606) -> vaexfast.statisticNd with op_min_max (src/vaexfast.cpp:1089-1101, 1167-1290):
//   * rows masked in the column are dropped; NaN never wins (`value < min`, `value > max` from (+inf, -inf));
//   * the column is cast to float64 when it is float64 or int64 and to FLOAT32 otherwise (as_flat_array, vaex/cpu.py:519-531):
//     int32 / uint32 / uint64 values are rounded to fp32, int64 to fp64 — part of the observable result, reproduced here with
//     round-to-nearest-even conversions;
//   * byte-swapped columns give the values of their native twin (float32 columns are astype'd to native, float64 columns are
//     read through functor_double_to_native).
// One streaming pass: 128-bit loads (evict-first), four in flight per thread, compile-time dtype; 8 B/row for a float64 column,
// nothing but the two doubles written.  The (min, max) pair is folded with order-independent integer atomics on IEEE storage.
#include <algorithm>

#include "binby.cuh"
#include "refvalue.cuh"

namespace b200 {
namespace {

constexpr int kThreads = 256;

template <typename T, bool SWAP, bool MASK>
__global__ void __launch_bounds__(kThreads) k_minmax(const T *__restrict__ data, const uint8_t *__restrict__ mask, long long nrows, double *out) {
    constexpr int V = 16 / sizeof(T); // elements per 128-bit load
    double lo = INFINITY, hi = -INFINITY;
    auto take = [&](T raw, long long i) {
        if (MASK && mask[i])
            return;
        const double v = ref_value<T>(SWAP ? swap_bytes<T>(raw) : raw);
        if (v < lo)
            lo = v;
        if (v > hi)
            hi = v;
    };
    // scalar head up to the first 16-byte boundary, vector body, scalar tail
    const uintptr_t addr = reinterpret_cast<uintptr_t>(data);
    long long head = (long long)(((16 - (addr & 15)) & 15) / sizeof(T));
    if (head > nrows)
        head = nrows;
    const long long nvec = (nrows - head) / V;
    const long long tid = (long long)blockIdx.x * kThreads + threadIdx.x, nthreads = (long long)gridDim.x * kThreads;
    if (tid < head)
        take(data[tid], tid);
    const uint4 *vec = reinterpret_cast<const uint4 *>(data + head);
    auto take_vec = [&](const uint4 &q, long long j) {
        T e[V];
        memcpy(e, &q, 16);
#pragma unroll
        for (int k = 0; k < V; k++)
            take(e[k], head + j * V + k);
    };
    long long j = tid;
    for (; j + 3 * nthreads < nvec; j += 4 * nthreads) { // four independent 128-bit loads in flight
        const uint4 a = __ldcs(vec + j), b = __ldcs(vec + j + nthreads), c = __ldcs(vec + j + 2 * nthreads), d = __ldcs(vec + j + 3 * nthreads);
        take_vec(a, j);
        take_vec(b, j + nthreads);
        take_vec(c, j + 2 * nthreads);
        take_vec(d, j + 3 * nthreads);
    }
    for (; j < nvec; j += nthreads)
        take_vec(__ldcs(vec + j), j);
    const long long tail0 = head + nvec * V;
    if (tail0 + tid < nrows)
        take(data[tail0 + tid], tail0 + tid);

#pragma unroll
    for (int o = 16; o; o >>= 1) {
        lo = fmin(lo, __shfl_xor_sync(0xffffffffu, lo, o));
        hi = fmax(hi, __shfl_xor_sync(0xffffffffu, hi, o));
    }
    __shared__ double slo[kThreads / 32], shi[kThreads / 32];
    if ((threadIdx.x & 31) == 0) {
        slo[threadIdx.x >> 5] = lo;
        shi[threadIdx.x >> 5] = hi;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        for (int w = 1; w < kThreads / 32; w++) {
            lo = fmin(lo, slo[w]);
            hi = fmax(hi, shi[w]);
        }
        if (lo < INFINITY)
            atomic_min_f64(out, lo);
        if (hi > -INFINITY)
            atomic_max_f64(out + 1, hi);
    }
}

template <typename T>
int launch_t(int sm_count, cudaStream_t st, const void *data, const uint8_t *mask, long long nrows, bool swap, double *out) {
    const long long want = (nrows / (16 / sizeof(T)) + kThreads - 1) / kThreads;
    const int blocks = (int)std::max<long long>(1, std::min<long long>(want, (long long)sm_count * 8));
    const T *d = static_cast<const T *>(data);
    if (swap && sizeof(T) > 1) {
        if (mask)
            k_minmax<T, true, true><<<blocks, kThreads, 0, st>>>(d, mask, nrows, out);
        else
            k_minmax<T, true, false><<<blocks, kThreads, 0, st>>>(d, mask, nrows, out);
    } else {
        if (mask)
            k_minmax<T, false, true><<<blocks, kThreads, 0, st>>>(d, mask, nrows, out);
        else
            k_minmax<T, false, false><<<blocks, kThreads, 0, st>>>(d, mask, nrows, out);
    }
    B200_CUDA(cudaGetLastError());
    return B200_OK;
}

} // namespace
} // namespace b200

using namespace b200;

extern "C" int b200_minmax(b200_ctx *ctx, int slot, int dtype, int byteswap, const void *data, const uint8_t *mask, int64_t nrows, int memspace,
                           double *out) {
    if (!ctx || slot < 0 || slot >= ctx->nslots || dtype < 0 || dtype >= B200_NDTYPE || !out || (nrows && !data)) {
        set_error("b200_minmax: invalid argument");
        return B200_ERR_INVALID;
    }
    B200_CUDA(cudaSetDevice(ctx->device));
    Slot *sl = ctx->slots[slot];
    std::lock_guard<std::mutex> guard(sl->mu);
    Stager stg{ctx, sl, memspace};
    const int isz = dtype_size(dtype);
    stg.plan(data, (size_t)nrows * isz);
    if (mask)
        stg.plan(mask, (size_t)nrows);
    B200_CHECK(stg.commit());
    double init[2] = {INFINITY, -INFINITY}; // StatOpMinMax.init (vaex/tasks.py)
    double *d = static_cast<double *>(sl->dscratch);
    B200_CUDA(cudaMemcpyAsync(d, init, sizeof init, cudaMemcpyHostToDevice, sl->stream));
    if (nrows) {
        const void *dd = stg.dev(data);
        const uint8_t *dm = static_cast<const uint8_t *>(stg.dev(mask));
        const bool sw = byteswap != 0;
        int rc = B200_OK;
        switch (dtype) {
        case B200_F64: rc = launch_t<double>(ctx->sm_count, sl->stream, dd, dm, nrows, sw, d); break;
        case B200_F32: rc = launch_t<float>(ctx->sm_count, sl->stream, dd, dm, nrows, sw, d); break;
        case B200_I64: rc = launch_t<long long>(ctx->sm_count, sl->stream, dd, dm, nrows, sw, d); break;
        case B200_I32: rc = launch_t<int>(ctx->sm_count, sl->stream, dd, dm, nrows, sw, d); break;
        case B200_I16: rc = launch_t<short>(ctx->sm_count, sl->stream, dd, dm, nrows, sw, d); break;
        case B200_I8: rc = launch_t<signed char>(ctx->sm_count, sl->stream, dd, dm, nrows, sw, d); break;
        case B200_U64: rc = launch_t<unsigned long long>(ctx->sm_count, sl->stream, dd, dm, nrows, sw, d); break;
        case B200_U32: rc = launch_t<unsigned>(ctx->sm_count, sl->stream, dd, dm, nrows, sw, d); break;
        case B200_U16: rc = launch_t<unsigned short>(ctx->sm_count, sl->stream, dd, dm, nrows, sw, d); break;
        default: rc = launch_t<unsigned char>(ctx->sm_count, sl->stream, dd, dm, nrows, sw, d); break; // uint8, bool (0 / 1)
        }
        B200_CHECK(rc);
    }
    B200_CUDA(cudaMemcpyAsync(out, d, sizeof init, cudaMemcpyDeviceToHost, sl->stream));
    B200_CUDA(cudaStreamSynchronize(sl->stream));
    return B200_OK;
}
