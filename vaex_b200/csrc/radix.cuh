// radix.cuh — stable LSD radix sort of (64-bit key, 64-bit payload) pairs, one driver (radix_sort) for every device sort: the
// ordered_set finalisation and the index_hash row ranges (hashset.cu), the argsort (sort.cu) and the list aggregator (list.cu).
#pragma once
#include <algorithm>

#include "common.cuh"
#include "scan.cuh"

namespace b200 {

// ---- LSD radix sort of (64-bit sort key, 64-bit payload) pairs, 8 bits per pass, stable --------------------------------------
// Replaces round 1's bitonic network (210 launches for 2^20 entries) + a 24 MB download + a host loop.  One pass = per-block digit
// histograms (digit-major), one exclusive scan over the 256 x nblocks matrix, a stable scatter.  `from_val`: the digit comes from
// the payload's upper word instead of the key.
constexpr int kRadixThreads = 256;

// A block sorts a TILE of `tiles` consecutive sub-tiles of 256 pairs (in order, so the pass stays stable); the tile size grows
// with n so that the 256 x nblocks histogram the single-CTA scan walks stays below ~2^19 counters (it was one 256-pair block per
// CTA: 1M counters and 0.9 ms of scan per pass for 1e6 keys — the whole finalisation time of groupby pass 1).
static inline unsigned radix_tiles(unsigned long long n) {
    unsigned long long t = 16;
    while ((n + t * kRadixThreads - 1) / (t * kRadixThreads) > 2048)
        t *= 2;
    return (unsigned)t;
}
static inline unsigned radix_blocks(unsigned long long n) {
    const unsigned long long per = (unsigned long long)radix_tiles(n) * kRadixThreads;
    return (unsigned)((n + per - 1) / per);
}

static __global__ void __launch_bounds__(kRadixThreads) k_radix_hist(const unsigned long long *key, const unsigned long long *val, unsigned long long n, int shift,
                                                              int from_val, unsigned *hist, unsigned nblk, unsigned tiles) {
    __shared__ unsigned h[256];
    h[threadIdx.x] = 0;
    __syncthreads();
    const unsigned long long base = (unsigned long long)blockIdx.x * tiles * kRadixThreads;
    for (unsigned j = 0; j < tiles; j++) {
        const unsigned long long i = base + (unsigned long long)j * kRadixThreads + threadIdx.x;
        if (i < n) {
            const unsigned long long x = from_val ? (val[i] >> 32) : key[i];
            atomicAdd(&h[(x >> shift) & 255u], 1u);
        }
    }
    __syncthreads();
    hist[(unsigned long long)threadIdx.x * nblk + blockIdx.x] = h[threadIdx.x];
}

static __global__ void __launch_bounds__(kRadixThreads) k_radix_scatter(const unsigned long long *key, const unsigned long long *val, unsigned long long *key_out,
                                                                 unsigned long long *val_out, unsigned long long n, int shift, int from_val,
                                                                 const unsigned *hist, unsigned nblk, unsigned tiles) {
    __shared__ unsigned wcnt[kRadixThreads / 32][256];
    __shared__ unsigned run[256]; // pairs of this digit the earlier sub-tiles of the block already placed (thread t owns digit t)
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    run[threadIdx.x] = hist[(unsigned long long)threadIdx.x * nblk + blockIdx.x];
    const unsigned long long base = (unsigned long long)blockIdx.x * tiles * kRadixThreads;
    for (unsigned j = 0; j < tiles; j++) {
        if (base + (unsigned long long)j * kRadixThreads >= n)
            break; // uniform
        for (int w = 0; w < kRadixThreads / 32; w++)
            wcnt[w][threadIdx.x] = 0;
        __syncthreads();
        const unsigned long long i = base + (unsigned long long)j * kRadixThreads + threadIdx.x;
        const bool live = i < n;
        unsigned long long k = 0, v = 0;
        unsigned d = 0;
        if (live) {
            k = key[i];
            v = val[i];
            d = (unsigned)(((from_val ? (v >> 32) : k) >> shift) & 255u);
        }
        const unsigned act = __ballot_sync(0xffffffffu, live);
        unsigned lrank = 0;
        if (live) {
            const unsigned m = __match_any_sync(act, d);
            lrank = __popc(m & ((1u << lane) - 1u));
            if (lrank == 0)
                wcnt[warp][d] = __popc(m);
        }
        __syncthreads();
        unsigned total = 0;
        { // exclusive prefix over the warps, per digit (thread t owns digit t)
            for (int w = 0; w < kRadixThreads / 32; w++) {
                const unsigned t = wcnt[w][threadIdx.x];
                wcnt[w][threadIdx.x] = total;
                total += t;
            }
        }
        __syncthreads();
        if (live) {
            const unsigned long long pos = (unsigned long long)run[d] + wcnt[warp][d] + lrank;
            key_out[pos] = k;
            val_out[pos] = v;
        }
        __syncthreads();
        run[threadIdx.x] += total;
    }
}

// the histogram scratch radix_sort needs for n pairs
static inline size_t radix_scratch_bytes(unsigned long long n) { return (size_t)256 * 4 * std::max(radix_blocks(n), 1u); }

// every byte of x through its highest non-zero one: the byte set that orders values in [0, x]
static inline unsigned radix_bytes_through(unsigned long long x) {
    unsigned bytes = 0;
    for (int b = 0; b < 8 && (x >> (8 * b)); b++)
        bytes |= 1u << b;
    return bytes;
}

// Enqueues on `st` a stable LSD sort of the n pairs (key[i], val[i]): one pass for every bit b of key_bytes, on key byte b, least
// significant first, then one for every bit b (0-3) of val_bytes, on byte b of val >> 32.  Each pass moves the pairs between
// (key, val) and (key_alt, val_alt); on return key / val point at the sorted pairs and key_alt / val_alt at the other two arrays.
// hist holds radix_scratch_bytes(n).  Nothing is allocated and nothing is synchronised: the caller orders what follows on `st`.
static inline int radix_sort(unsigned long long n, unsigned key_bytes, unsigned val_bytes, unsigned long long *&key, unsigned long long *&val,
                             unsigned long long *&key_alt, unsigned long long *&val_alt, unsigned *hist, cudaStream_t st) {
    if (n < 2)
        return B200_OK;
    const unsigned nblk = radix_blocks(n), tiles = radix_tiles(n);
    for (int pass = 0; pass < 12; pass++) {
        const int from_val = pass >= 8, b = from_val ? pass - 8 : pass;
        if (!(((from_val ? val_bytes : key_bytes) >> b) & 1u))
            continue;
        k_radix_hist<<<nblk, kRadixThreads, 0, st>>>(key, val, n, 8 * b, from_val, hist, nblk, tiles);
        k_scan_u32<<<1, 1024, 0, st>>>(hist, 256ull * nblk);
        k_radix_scatter<<<nblk, kRadixThreads, 0, st>>>(key, val, key_alt, val_alt, n, 8 * b, from_val, hist, nblk, tiles);
        B200_CUDA(cudaGetLastError());
        std::swap(key, key_alt);
        std::swap(val, val_alt);
    }
    return B200_OK;
}


} // namespace b200
