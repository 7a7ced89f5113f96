// scan.cuh — exclusive scans in place: u32 counters in one CTA (shared by the radix sort of radix.cuh and the filter compaction
// of expr.cu: n is a few million at most), and int64 values of any length over many CTAs (list.cu).
#pragma once
#include "common.cuh"

namespace b200 {

// total (optional) receives the sum of all counters
static __global__ void __launch_bounds__(1024) k_scan_u32(unsigned *a, unsigned long long n, unsigned long long *total = nullptr) {
    __shared__ unsigned warp_sums[32];
    __shared__ unsigned long long carry;
    if (threadIdx.x == 0)
        carry = 0;
    __syncthreads();
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (unsigned long long base = 0; base < n; base += 1024) {
        const unsigned long long i = base + threadIdx.x;
        const unsigned v = i < n ? a[i] : 0u;
        unsigned x = v;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const unsigned y = __shfl_up_sync(0xffffffffu, x, o);
            if (lane >= o)
                x += y;
        }
        if (lane == 31)
            warp_sums[warp] = x;
        __syncthreads();
        if (warp == 0) {
            unsigned w = warp_sums[lane];
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const unsigned y = __shfl_up_sync(0xffffffffu, w, o);
                if (lane >= o)
                    w += y;
            }
            warp_sums[lane] = w;
        }
        __syncthreads();
        const unsigned long long before = carry + (warp ? warp_sums[warp - 1] : 0u) + x - v;
        if (i < n)
            a[i] = (unsigned)before;
        __syncthreads();
        if (threadIdx.x == 1023)
            carry = before + v;
        __syncthreads();
    }
    if (total && threadIdx.x == 0)
        *total = carry;
}

// ---- exclusive scan of int64 values in place, any length (the string list's byte offsets: totals past 2^32) ------------------
// Tiles of 2048 values: a pass writes every tile's sum, the sums are scanned the same way (recursively; 2^32 values need three
// levels), and a second pass scans every tile and adds its tile's offset.
constexpr int kScanThreads = 256, kScanItems = 8;
constexpr unsigned long long kScanTile = (unsigned long long)kScanThreads * kScanItems;

// exclusive prefix of one value per thread over the block; *total = the block's sum
static __device__ __forceinline__ long long block_exclusive_i64(long long v, long long *total) {
    __shared__ long long warp_sums[kScanThreads / 32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    long long x = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const long long y = __shfl_up_sync(0xffffffffu, x, o);
        if (lane >= o)
            x += y;
    }
    if (lane == 31)
        warp_sums[warp] = x;
    __syncthreads();
    long long before = 0, all = 0;
#pragma unroll
    for (int w = 0; w < kScanThreads / 32; w++) {
        const long long s = warp_sums[w];
        before += w < warp ? s : 0;
        all += s;
    }
    *total = all;
    return before + x - v;
}

// sum of one value per thread over a kScanThreads block in a fixed tree (xor butterfly per warp, then the warp sums in warp order),
// so a floating-point sum is the same bits on every run; every thread receives it.  Ends with a barrier: callable in a loop.
template <typename T>
static __device__ __forceinline__ T block_sum(T v) {
    __shared__ T warp_sums[kScanThreads / 32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1)
        v += __shfl_xor_sync(0xffffffffu, v, o);
    if (lane == 0)
        warp_sums[warp] = v;
    __syncthreads();
    T all = warp_sums[0];
#pragma unroll
    for (int w = 1; w < kScanThreads / 32; w++)
        all += warp_sums[w];
    __syncthreads();
    return all;
}

static __global__ void __launch_bounds__(kScanThreads) k_scan_i64_sums(const long long *a, unsigned long long n, long long *sums) {
    const unsigned long long i0 = blockIdx.x * kScanTile + (unsigned long long)threadIdx.x * kScanItems;
    long long s = 0;
#pragma unroll
    for (int k = 0; k < kScanItems; k++)
        s += i0 + k < n ? a[i0 + k] : 0;
    long long total;
    block_exclusive_i64(s, &total);
    if (threadIdx.x == 0)
        sums[blockIdx.x] = total;
}

static __global__ void __launch_bounds__(kScanThreads) k_scan_i64_apply(long long *a, unsigned long long n, const long long *tile_offsets) {
    const unsigned long long i0 = blockIdx.x * kScanTile + (unsigned long long)threadIdx.x * kScanItems;
    long long r[kScanItems], s = 0;
#pragma unroll
    for (int k = 0; k < kScanItems; k++) {
        r[k] = i0 + k < n ? a[i0 + k] : 0;
        s += r[k];
    }
    long long total;
    long long x = block_exclusive_i64(s, &total) + (tile_offsets ? tile_offsets[blockIdx.x] : 0);
#pragma unroll
    for (int k = 0; k < kScanItems; k++) {
        if (i0 + k < n)
            a[i0 + k] = x;
        x += r[k];
    }
}

// tile sums of every level of scan_i64(n): the caller provides them and keeps them until the scan has run
static inline unsigned long long scan_i64_sums(unsigned long long n) {
    unsigned long long total = 0;
    for (; n > kScanTile; n = (n + kScanTile - 1) / kScanTile)
        total += (n + kScanTile - 1) / kScanTile;
    return total;
}

static inline int scan_i64(long long *a, unsigned long long n, long long *sums, cudaStream_t st) {
    if (n <= kScanTile) {
        k_scan_i64_apply<<<1, kScanThreads, 0, st>>>(a, n, nullptr);
        B200_CUDA(cudaGetLastError());
        return B200_OK;
    }
    const unsigned long long tiles = (n + kScanTile - 1) / kScanTile;
    k_scan_i64_sums<<<(unsigned)tiles, kScanThreads, 0, st>>>(a, n, sums);
    B200_CUDA(cudaGetLastError());
    B200_CHECK(scan_i64(sums, tiles, sums + tiles, st));
    k_scan_i64_apply<<<(unsigned)tiles, kScanThreads, 0, st>>>(a, n, sums);
    B200_CUDA(cudaGetLastError());
    return B200_OK;
}

} // namespace b200
