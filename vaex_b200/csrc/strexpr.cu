// strexpr.cu — vaex's string predicates and measures over an arrow string column, the string calls of a device expression.
//
// Reference: the StringSequenceBase methods that vaex's str_* functions call (vaex/functions.py str_equals, str_startswith, ...):
// equals / equals2 / startswith / endswith / find (src/superstring.hpp:130-268), len and byte_length (src/superstring.hpp:1434-1438
// over str_len of src/string_utils.hpp:310-326), and the literal branches of search and count (src/strings.cpp:31-110).  Every one
// reads row i through its offsets (view(i)), null or not; only the two equals look at the null mask.  One call writes one bool or
// int64 column to device memory on the slot's stream; vaex_b200/expression.py feeds it to b200_eval as an ordinary input.  Like the
// gathers of take.cu it reads and writes device memory only: the caller stages the string buffers on the slot's stream.
//
// Kernels: one thread per row, with coalesced offset loads.  count also has a form with one warp per row, which the call picks when
// the mean row length bytes / rows is long (DESIGN.md §4).
#include <algorithm>
#include <stdlib.h>
#include <string.h>

#include "common.cuh"

namespace b200 {
namespace {

// the mean row length (bytes) from which count runs one warp per row (measured on the H100, DESIGN.md §4)
constexpr long long kWarpScanMinMean = 128;

struct StrCol {
    const void *off; // nrows + 1 offsets of `isz` bytes
    int isz;
    const unsigned char *bytes; // the byte at offset value 0 (the buffer the offsets index)
    const uint8_t *nulls; // 1 = null, may be null
};

struct StrParams {
    StrCol a, b;
    const unsigned char *pat;
    long long plen, start, end; // end = INT64_MAX: to the end of the row (the reference's till_end, which gives the same window)
    long long nrows;
    void *out;
};

struct Row {
    const unsigned char *s;
    long long len;
};

__device__ __forceinline__ long long offset_at(const StrCol &c, long long i) {
    return c.isz == 4 ? (long long)__ldg(static_cast<const int *>(c.off) + i) : __ldg(static_cast<const long long *>(c.off) + i);
}

__device__ __forceinline__ Row row_at(const StrCol &c, long long r) {
    const long long a = offset_at(c, r), b = offset_at(c, r + 1);
    return Row{c.bytes + a, b > a ? b - a : 0};
}

__device__ __forceinline__ bool bytes_equal(const unsigned char *x, const unsigned char *y, long long n) {
    for (long long k = 0; k < n; k++)
        if (__ldg(x + k) != __ldg(y + k))
            return false;
    return true;
}

// the bytes a UTF-8 lead byte steps over (src/string_utils.hpp:310-326); a lead byte >= 0xF8 steps one byte here, where the
// reference does not move and never ends
__device__ __forceinline__ int utf8_step(unsigned char c) { return c < 0x80 ? 1 : c < 0xE0 ? 2 : c < 0xF0 ? 3 : c < 0xF8 ? 4 : 1; }

// str_len: code points by the lead-byte rule; a sequence cut off by the end of the row counts once
__device__ long long utf8_len(const unsigned char *s, long long len) {
    long long p = 0, n = 0;
    while (p < len) {
        p += utf8_step(__ldg(s + p));
        n++;
    }
    return n;
}

// utf8_index_to_byte_offset (src/superstring.hpp:77-95): the byte offset of code point `index`, which can pass `len` when the row
// ends inside a sequence; a negative index gives 0
__device__ long long utf8_index_to_byte(const unsigned char *s, long long len, long long index) {
    long long p = 0;
    while (p < len && index > 0) {
        p += utf8_step(__ldg(s + p));
        index--;
    }
    return p;
}

// utf8_slice_neg_index_to_byte_offset (src/superstring.hpp:56-75): the byte offset of code point str_len + index
__device__ long long utf8_neg_index_to_byte(const unsigned char *s, long long len, long long index) {
    return utf8_index_to_byte(s, len, utf8_len(s, len) + index);
}

// StringSequenceBase::find's window (src/superstring.hpp:161-197): [*lo, *lo + *n) of the row, false when the search does not run
__device__ __forceinline__ bool find_window(const StrParams &p, const Row &x, long long *lo, long long *n) {
    const long long bs = utf8_index_to_byte(x.s, x.len, p.start);
    long long be;
    if (p.end > x.len)
        be = x.len;
    else if (p.end < 0)
        be = utf8_neg_index_to_byte(x.s, x.len, p.end);
    else
        be = utf8_index_to_byte(x.s, x.len, p.end);
    if (!(bs < x.len && be > bs))
        return false;
    *lo = bs;
    *n = min(be - bs, x.len - bs); // string_view::substr clamps the count
    return true;
}

__device__ __forceinline__ bool match_at(const StrParams &p, const unsigned char *s, unsigned char first) {
    return __ldg(s) == first && bytes_equal(s + 1, p.pat + 1, p.plen - 1);
}

// ---- one thread per row -----------------------------------------------------------------------------------------------------
// the first (or with Last, the last) start of the pattern in s[0, n), -1 when there is none; an empty pattern is found at 0 (at n)
template <bool Last> __device__ long long search_thread(const StrParams &p, const unsigned char *s, long long n) {
    if (p.plen > n)
        return -1;
    if (p.plen == 0)
        return Last ? n : 0;
    const unsigned char first = __ldg(p.pat);
    if (Last) {
        for (long long k = n - p.plen; k >= 0; k--)
            if (match_at(p, s + k, first))
                return k;
    } else {
        for (long long k = 0; k <= n - p.plen; k++)
            if (match_at(p, s + k, first))
                return k;
    }
    return -1;
}

template <int OP> __device__ __forceinline__ long long eval_row(const StrParams &p, long long r) {
    const Row x = row_at(p.a, r);
    switch (OP) {
    case B200_EX_STR_EQUALS:
        return !(p.a.nulls && p.a.nulls[r]) && x.len == p.plen && bytes_equal(x.s, p.pat, p.plen);
    case B200_EX_STR_EQUALS2: {
        const bool na = p.a.nulls && p.a.nulls[r], nb = p.b.nulls && p.b.nulls[r];
        if (na || nb)
            return na && nb;
        const Row y = row_at(p.b, r);
        return x.len == y.len && bytes_equal(x.s, y.s, x.len);
    }
    case B200_EX_STR_STARTSWITH: return x.len >= p.plen && bytes_equal(x.s, p.pat, p.plen);
    case B200_EX_STR_ENDSWITH: return x.len >= p.plen && bytes_equal(x.s + (x.len - p.plen), p.pat, p.plen);
    case B200_EX_STR_CONTAINS: return search_thread<false>(p, x.s, x.len) >= 0;
    case B200_EX_STR_COUNT: { // non-overlapping: every match moves the search past itself (plen >= 1, checked by the call)
        long long n = 0, k = 0, f;
        while ((f = search_thread<false>(p, x.s + k, x.len - k)) >= 0) {
            n++;
            k += f + p.plen;
        }
        return n;
    }
    case B200_EX_STR_FIND:
    case B200_EX_STR_RFIND: {
        long long lo, n;
        if (!find_window(p, x, &lo, &n))
            return -1;
        return search_thread<OP == B200_EX_STR_RFIND>(p, x.s + lo, n);
    }
    case B200_EX_STR_LEN: return utf8_len(x.s, x.len);
    default: return x.len; // byte_length
    }
}

template <int OP> __global__ void __launch_bounds__(256) k_str_thread(const __grid_constant__ StrParams p) {
    for (long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x; r < p.nrows; r += (long long)gridDim.x * blockDim.x) {
        const long long v = eval_row<OP>(p, r);
        if (OP == B200_EX_STR_COUNT || OP == B200_EX_STR_FIND || OP == B200_EX_STR_RFIND || OP == B200_EX_STR_LEN || OP == B200_EX_STR_BYTE_LENGTH)
            static_cast<long long *>(p.out)[r] = v;
        else
            static_cast<uint8_t *>(p.out)[r] = (uint8_t)v;
    }
}

// ---- one warp per row: count on long rows ------------------------------------------------------------------------------------
// Lane l tests the start position base + l of a 32-wide window (first byte, then the rest); the ballot gives the window's matches in
// order and every lane counts them greedily, so the count is the non-overlapping one of the thread form.  On the H100 this beats the
// thread form for count only, and only on long rows: contains / find / rfind stop at their first match and stay one thread per row.
__global__ void __launch_bounds__(256) k_count_warp(const __grid_constant__ StrParams p) {
    const int lane = threadIdx.x & 31;
    const long long nwarps = (long long)gridDim.x * (blockDim.x >> 5);
    const unsigned char first = __ldg(p.pat);
    for (long long r = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5; r < p.nrows; r += nwarps) {
        const Row x = row_at(p.a, r);
        const long long last = x.len - p.plen; // the last start position
        long long next = 0, c = 0;
        for (long long base = 0; base <= last; base += 32) {
            const long long k = base + lane;
            unsigned m = __ballot_sync(0xffffffffu, k <= last && match_at(p, x.s + k, first));
            while (m) { // a match counts when it starts after the previous one ended
                const long long k2 = base + __ffs(m) - 1;
                m &= m - 1;
                if (k2 >= next) {
                    c++;
                    next = k2 + p.plen;
                }
            }
        }
        if (lane == 0)
            static_cast<long long *>(p.out)[r] = c;
    }
}

int str_blocks(b200_ctx *ctx, unsigned long long threads) {
    const unsigned long long want = (threads + 255) / 256;
    return (int)std::min<unsigned long long>(std::max<unsigned long long>(want, 1), (unsigned long long)ctx->sm_count * 16);
}

template <int OP> void launch(b200_ctx *ctx, cudaStream_t st, const StrParams &p, bool warp) {
    if (OP == B200_EX_STR_COUNT && warp) {
        k_count_warp<<<str_blocks(ctx, (unsigned long long)p.nrows * 32), 256, 0, st>>>(p);
        return;
    }
    k_str_thread<OP><<<str_blocks(ctx, (unsigned long long)p.nrows), 256, 0, st>>>(p);
}

} // namespace
} // namespace b200

using namespace b200;

extern "C" int b200_str_eval(b200_ctx *ctx, int slot, int op, const void *offsets, int offset_isz, const uint8_t *bytes, const uint8_t *nulls,
                             const void *offsets2, int offset2_isz, const uint8_t *bytes2, const uint8_t *nulls2, const uint8_t *pattern,
                             int64_t plen, int64_t start, int64_t end, int64_t nrows, int64_t nbytes, void *out_device) {
    const bool two = op == B200_EX_STR_EQUALS2;
    if (op < B200_EX_STR_EQUALS || op > B200_EX_STR_BYTE_LENGTH || nrows < 0 || plen < 0 || (plen && !pattern) || (offset_isz != 4 && offset_isz != 8) ||
        (nrows && (!offsets || !out_device)) || (two && (!offsets2 || (offset2_isz != 4 && offset2_isz != 8)))) {
        set_error("b200_str_eval: invalid argument (op %d, %lld rows, pattern of %lld bytes)", op, (long long)nrows, (long long)plen);
        return B200_ERR_INVALID;
    }
    if (op == B200_EX_STR_COUNT && plen == 0) {
        set_error("b200_str_eval: str_count of an empty pattern (the reference never ends on it)");
        return B200_ERR_INVALID;
    }
    if (!nrows)
        return B200_OK;
    Slot *sl;
    B200_CHECK(device_slot(ctx, slot, "b200_str_eval", &sl));
    std::lock_guard<std::mutex> g(sl->mu);
    StrParams p;
    memset(&p, 0, sizeof p);
    p.a = StrCol{offsets, offset_isz, bytes, nulls};
    if (two)
        p.b = StrCol{offsets2, offset2_isz, bytes2, nulls2};
    p.pat = pattern;
    p.plen = plen;
    p.start = start;
    p.end = end;
    p.nrows = nrows;
    p.out = out_device;
    // B200_STR_SCAN=thread|warp forces the form of count (tools/bench_str_expr.py measures both); the call picks by the mean row
    // length, which the caller's offsets give without a read of the device
    const char *force = getenv("B200_STR_SCAN");
    const bool warp = force ? strcmp(force, "warp") == 0 : nbytes / nrows >= kWarpScanMinMean;
    cudaStream_t st = sl->stream;
    switch (op) {
    case B200_EX_STR_EQUALS: launch<B200_EX_STR_EQUALS>(ctx, st, p, warp); break;
    case B200_EX_STR_EQUALS2: launch<B200_EX_STR_EQUALS2>(ctx, st, p, warp); break;
    case B200_EX_STR_STARTSWITH: launch<B200_EX_STR_STARTSWITH>(ctx, st, p, warp); break;
    case B200_EX_STR_ENDSWITH: launch<B200_EX_STR_ENDSWITH>(ctx, st, p, warp); break;
    case B200_EX_STR_CONTAINS: launch<B200_EX_STR_CONTAINS>(ctx, st, p, warp); break;
    case B200_EX_STR_COUNT: launch<B200_EX_STR_COUNT>(ctx, st, p, warp); break;
    case B200_EX_STR_FIND: launch<B200_EX_STR_FIND>(ctx, st, p, warp); break;
    case B200_EX_STR_RFIND: launch<B200_EX_STR_RFIND>(ctx, st, p, warp); break;
    case B200_EX_STR_LEN: launch<B200_EX_STR_LEN>(ctx, st, p, warp); break;
    default: launch<B200_EX_STR_BYTE_LENGTH>(ctx, st, p, warp); break;
    }
    B200_CUDA(cudaGetLastError());
    return B200_OK;
}
