// take.cu — the row gather of df.join: out[i] = src[index[i]] for up to 16 fixed-width columns in one launch (b200_take), and the
// same gather for arrow string columns (b200_take_strings).
//
// Reference: vaex/join.py:286 (`right_dataset.take(lookup, masked=...)`: the right's columns moved to the left's rows), :214
// (`left.take(lookup_left)`: the left's rows repeated for the right's duplicates) and :218-222 (the inner join's matched left rows).
// An index < 0 is a row without a match: its value is zero and its validity 0.  An index >= the source length is a bug in the
// caller (the reference fills its lookup with iinfo.max so that such a bug crashes, join.py:178-181): the call fails instead of
// reading past the column.
//
// Bound: every output row reads its index once and one random source item per column.  A source that fits in L2 (50 MB on an H100)
// is read at L2 rate; beyond that each 1-8 byte item costs a 32-byte HBM sector.
#include <algorithm>

#include "device_utils.cuh"
#include "scan.cuh"
#include "strings.cuh"

namespace b200 {
namespace {

constexpr int kTakeMaxCols = 16;
constexpr unsigned kOutOfRange = 1u << kTakeMaxCols; // flag word: bit c = column c has a missing row, this bit = an index past the end

struct TakeParams {
    const void *src[kTakeMaxCols];
    const uint8_t *src_mask[kTakeMaxCols]; // 1 = missing, may be null
    void *dst[kTakeMaxCols];
    uint8_t *dst_valid[kTakeMaxCols]; // 1 = valid, may be null
    int isz[kTakeMaxCols];
    int ncols;
};

__device__ __forceinline__ long long load_index(const void *index, int isz, long long i) {
    switch (isz) {
    case 1: return static_cast<const signed char *>(index)[i];
    case 2: return static_cast<const short *>(index)[i];
    case 4: return static_cast<const int *>(index)[i];
    default: return static_cast<const long long *>(index)[i];
    }
}

// one thread per output row (grid-stride); the per-thread flag bits are OR-ed over the warp and written with one atomic per warp
__global__ void __launch_bounds__(256) k_take(const void *__restrict__ index, int index_isz, long long n, long long src_len, TakeParams p,
                                              unsigned *flags) {
    unsigned bits = 0;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const long long idx = load_index(index, index_isz, i);
        const bool bad = idx >= src_len;
        bits |= bad ? kOutOfRange : 0u;
        const bool none = idx < 0 || bad;
        for (int c = 0; c < p.ncols; c++) {
            const bool missing = none || (p.src_mask[c] && p.src_mask[c][idx]);
            store1_raw(p.dst[c], p.isz[c], i, none ? 0 : load1_raw(p.src[c], p.isz[c], idx)); // a miss's index may be out of range
            if (p.dst_valid[c])
                p.dst_valid[c][i] = missing ? 0 : 1;
            bits |= missing ? 1u << c : 0u;
        }
    }
    bits = __reduce_or_sync(0xffffffffu, bits);
    if ((threadIdx.x & 31) == 0 && bits)
        atomicOr(flags, bits);
}

// ---- strings --------------------------------------------------------------------------------------------------------------
struct TakeStrSrc {
    const void *offsets; // src_len + 1 entries of offset_isz bytes
    int offset_isz;
    const unsigned char *bytes; // the byte of offset value `base`
    long long base;
    const uint8_t *mask; // 1 = missing, may be null
};

__device__ __forceinline__ long long load_offset(const TakeStrSrc &s, long long i) {
    return s.offset_isz == 4 ? (long long)static_cast<const int *>(s.offsets)[i] : static_cast<const long long *>(s.offsets)[i];
}

// pass 1: every output row's length (0 when missing) into len[i], its validity, and the flag word
__global__ void __launch_bounds__(256) k_take_str_len(const void *__restrict__ index, int index_isz, long long n, long long src_len, TakeStrSrc s,
                                                      long long *len, uint8_t *valid, unsigned *flags) {
    unsigned bits = 0;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const long long idx = load_index(index, index_isz, i);
        const bool bad = idx >= src_len;
        const bool missing = idx < 0 || bad || (s.mask && s.mask[idx]);
        bits |= (bad ? kOutOfRange : 0u) | (missing ? 1u : 0u);
        len[i] = missing ? 0 : load_offset(s, idx + 1) - load_offset(s, idx);
        if (valid)
            valid[i] = missing ? 0 : 1;
    }
    bits = __reduce_or_sync(0xffffffffu, bits);
    if ((threadIdx.x & 31) == 0 && bits)
        atomicOr(flags, bits);
}

// pass 3, after the scan: G threads copy one row's string to its output offset (copy_string of strings.cuh)
template <int G>
__global__ void __launch_bounds__(256) k_take_str_copy(const void *__restrict__ index, int index_isz, long long n, TakeStrSrc s, const long long *off,
                                                       char *out) {
    const int lane = threadIdx.x % G;
    const long long groups = (long long)gridDim.x * (256 / G);
    for (long long i = ((long long)blockIdx.x * 256 + threadIdx.x) / G; i < n; i += groups) {
        const long long o = off[i], len = off[i + 1] - o;
        if (len)
            copy_string<G>(out + o, reinterpret_cast<const char *>(s.bytes) + (load_offset(s, load_index(index, index_isz, i)) - s.base), len, lane);
    }
}

int take_blocks(b200_ctx *ctx, unsigned long long threads) {
    const unsigned long long want = (threads + 255) / 256;
    return (int)std::min<unsigned long long>(std::max<unsigned long long>(want, 1), (unsigned long long)ctx->sm_count * 16);
}

bool index_size_ok(int isz) { return isz == 1 || isz == 2 || isz == 4 || isz == 8; }

} // namespace

// the gathers (and the argsort of sort.cu) read and write device memory only (the caller stages a host column once, not once per
// call), so they need no call frame: the slot's stream, under the slot's lock, with the device set
int device_slot(b200_ctx *ctx, int slot, const char *what, Slot **out) {
    if (!ctx || slot < 0 || slot >= ctx->nslots) {
        set_error("%s: invalid slot %d", what, slot);
        return B200_ERR_INVALID;
    }
    B200_CUDA(cudaSetDevice(ctx->device));
    *out = ctx->slots[slot];
    return B200_OK;
}

} // namespace b200

using namespace b200;

extern "C" {

int b200_take(b200_ctx *ctx, int slot, const void *index, int index_isz, int64_t n, int ncols, const void *const *src, const int32_t *src_isz,
              const uint8_t *const *src_masks, int64_t src_len, void *const *dst, uint8_t *const *dst_valid, int32_t *missing_out) {
    if (n < 0 || src_len < 0 || ncols < 1 || ncols > kTakeMaxCols || !index_size_ok(index_isz) || (n && !index) || !src || !src_isz || !dst ||
        !missing_out) {
        set_error("b200_take: invalid argument");
        return B200_ERR_INVALID;
    }
    TakeParams p;
    memset(&p, 0, sizeof p);
    p.ncols = ncols;
    for (int c = 0; c < ncols; c++) {
        if (!index_size_ok(src_isz[c]) || (src_len && !src[c]) || (n && !dst[c])) {
            set_error("b200_take: column %d is invalid", c);
            return B200_ERR_INVALID;
        }
        p.isz[c] = src_isz[c];
        p.src[c] = src[c];
        p.src_mask[c] = src_masks ? src_masks[c] : nullptr;
        p.dst[c] = dst[c];
        p.dst_valid[c] = dst_valid ? dst_valid[c] : nullptr;
        missing_out[c] = 0;
    }
    if (!n)
        return B200_OK;
    Slot *sl;
    B200_CHECK(device_slot(ctx, slot, "b200_take", &sl));
    std::lock_guard<std::mutex> g(sl->mu);
    DevBuf<unsigned> d_flags;
    B200_CHECK(d_flags.alloc(ctx, 4, "b200_take", sl->stream));
    B200_CUDA(cudaMemsetAsync(d_flags, 0, 4, sl->stream));
    k_take<<<take_blocks(ctx, (unsigned long long)n), 256, 0, sl->stream>>>(index, index_isz, n, src_len, p, d_flags);
    B200_CUDA(cudaGetLastError());
    unsigned flags = 0;
    B200_CUDA(cudaMemcpyAsync(&flags, d_flags, 4, cudaMemcpyDeviceToHost, sl->stream));
    B200_CUDA(cudaStreamSynchronize(sl->stream));
    if (flags & kOutOfRange) {
        set_error("b200_take: an index is >= the source length %lld", (long long)src_len);
        return B200_ERR_INVALID;
    }
    for (int c = 0; c < ncols; c++)
        missing_out[c] = (flags >> c) & 1;
    return B200_OK;
}

int b200_take_strings(b200_ctx *ctx, int slot, const void *index, int index_isz, int64_t n, const void *offsets, int offset_isz, const uint8_t *bytes,
                      const uint8_t *src_mask, int64_t src_len, int64_t *offsets_out, uint8_t *bytes_out, uint8_t *valid_out, int64_t capacity,
                      int64_t *size_needed, int32_t *missing_out) {
    if (n < 0 || src_len < 0 || capacity < 0 || !index_size_ok(index_isz) || (offset_isz != 4 && offset_isz != 8) || (n && !index) || !offsets ||
        !offsets_out || !size_needed || !missing_out) {
        set_error("b200_take_strings: invalid argument");
        return B200_ERR_INVALID;
    }
    *size_needed = 0;
    *missing_out = 0;
    Slot *sl;
    B200_CHECK(device_slot(ctx, slot, "b200_take_strings", &sl));
    std::lock_guard<std::mutex> g(sl->mu);
    cudaStream_t st = sl->stream;
    // the byte range the source uses: offsets[0] .. offsets[src_len] (a sliced arrow array's offsets do not start at 0)
    long long first = 0, last = 0;
    B200_CUDA(cudaMemcpyAsync(&first, offsets, offset_isz, cudaMemcpyDeviceToHost, st));
    B200_CUDA(cudaMemcpyAsync(&last, static_cast<const char *>(offsets) + src_len * offset_isz, offset_isz, cudaMemcpyDeviceToHost, st));
    B200_CUDA(cudaStreamSynchronize(st));
    if (offset_isz == 4)
        first = (int)first, last = (int)last;
    if (last < first || (last > first && !bytes)) {
        set_error("b200_take_strings: offsets[%lld] (%lld) < offsets[0] (%lld) or no bytes", (long long)src_len, last, first);
        return B200_ERR_INVALID;
    }
    TakeStrSrc s;
    s.offsets = offsets;
    s.offset_isz = offset_isz;
    s.bytes = last > first ? bytes + first : nullptr;
    s.base = first;
    s.mask = src_mask;
    DevBuf<unsigned> d_flags;
    B200_CHECK(d_flags.alloc(ctx, 4, "b200_take_strings", st));
    B200_CUDA(cudaMemsetAsync(d_flags, 0, 4, st));
    B200_CUDA(cudaMemsetAsync(offsets_out + n, 0, 8, st));
    if (n) {
        k_take_str_len<<<take_blocks(ctx, (unsigned long long)n), 256, 0, st>>>(index, index_isz, n, src_len, s, (long long *)offsets_out, valid_out, d_flags);
        B200_CUDA(cudaGetLastError());
    }
    DevBuf<long long> tile_sums;
    if (const unsigned long long ns = scan_i64_sums((unsigned long long)n + 1))
        B200_CHECK(tile_sums.alloc(ctx, ns * 8, "b200_take_strings", st));
    B200_CHECK(scan_i64((long long *)offsets_out, (unsigned long long)n + 1, tile_sums, st));
    unsigned flags = 0;
    long long total = 0;
    B200_CUDA(cudaMemcpyAsync(&flags, d_flags, 4, cudaMemcpyDeviceToHost, st));
    B200_CUDA(cudaMemcpyAsync(&total, offsets_out + n, 8, cudaMemcpyDeviceToHost, st));
    B200_CUDA(cudaStreamSynchronize(st));
    if (flags & kOutOfRange) {
        set_error("b200_take_strings: an index is >= the source length %lld", (long long)src_len);
        return B200_ERR_INVALID;
    }
    *size_needed = total;
    *missing_out = flags & 1;
    if (total && bytes_out && total <= capacity) {
        // a group of threads per string, sized by the mean length: short strings must not leave most of a warp idle
        const long long mean = total / std::max<int64_t>(n, 1);
        const long long *off = (const long long *)offsets_out;
        char *out = (char *)bytes_out;
        if (mean > 256)
            k_take_str_copy<32><<<take_blocks(ctx, (unsigned long long)n * 32), 256, 0, st>>>(index, index_isz, n, s, off, out);
        else if (mean > 32)
            k_take_str_copy<8><<<take_blocks(ctx, (unsigned long long)n * 8), 256, 0, st>>>(index, index_isz, n, s, off, out);
        else
            k_take_str_copy<4><<<take_blocks(ctx, (unsigned long long)n * 4), 256, 0, st>>>(index, index_isz, n, s, off, out);
        B200_CUDA(cudaGetLastError());
        B200_CUDA(cudaStreamSynchronize(st));
    }
    return B200_OK;
}

} // extern "C"
