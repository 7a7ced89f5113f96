// sort.cu — the argsort of df.sort (vaex/dataframe.py:4694-4745: pa.compute.sort_indices over the `by` columns), on the device.
//
// Every key row becomes an unsigned, order-preserving field: the value bits (sign bit flipped for signed integers; for floats -0.0
// made +0.0, then all bits of negatives and the sign bit of positives flipped; bool and unsigned integers as they are; inverted
// when the key is descending) under a class field (value 0 < NaN < null) that is never inverted, so NaN and null stay last in
// either direction, as arrow's are.  A NaN or null row's value bits are zero: every NaN equals every other NaN.
//
// The fields of all keys, least significant first (the last key's value, its class, the previous key's value, ...), are packed
// greedily into 64-bit words.  Each word is one round, last word first: an encode kernel reads the keys through the current
// permutation (one gather per round; the first round starts from the identity) and reduces the AND / OR of all words, then a
// stable LSD radix sort (radix.cuh) carries the permutation along — over the bytes that vary only.  Two int32 keys are one word and
// one round; a float key whose rows hold no NaN or null sorts on its value bytes alone.
//
// Bound: a round reads the keys once through the permutation (random reads when it is not the first) and writes 16 bytes per row;
// a radix pass reads 8 (histogram) + 16 bytes and writes 16 per row.  The scatter's positions are 32-bit: n < 2^32.
#include <algorithm>

#include "device_utils.cuh"
#include "radix.cuh"

namespace b200 {
namespace {

constexpr int kSortFields = 2 * B200_SORT_MAX_KEYS;

struct EncodeParams {
    const void *data[B200_SORT_MAX_KEYS];
    const uint8_t *mask[B200_SORT_MAX_KEYS]; // 1 = null, may be null
    int dtype[B200_SORT_MAX_KEYS];
    int byteswap[B200_SORT_MAX_KEYS];
    int descending[B200_SORT_MAX_KEYS];
    int nat_is_null[B200_SORT_MAX_KEYS];
    int class_bits[B200_SORT_MAX_KEYS];
    // the fields of this round's word
    int nfields;
    int fkey[kSortFields];
    int fclass[kSortFields]; // 1 = the key's class field, 0 = its value field
    int fshift[kSortFields];
};

__host__ __device__ inline int value_bits(int dtype) { return dtype == B200_BOOL ? 1 : 8 * dtype_size(dtype); }

// the class (0 value, 1 NaN, 2 null) and the order-preserving value bits of key k at row r
__device__ __forceinline__ int encode_key(const EncodeParams &p, int k, long long r, unsigned long long *value) {
    const int dt = p.dtype[k], bits = value_bits(dt);
    const unsigned long long full = bits == 64 ? ~0ull : (1ull << bits) - 1ull, top = 1ull << (bits - 1);
    const int isz = dtype_size(dt);
    unsigned long long v = load1_raw(p.data[k], isz, r);
    if (p.byteswap[k])
        v = bswap(v, isz);
    int cls = p.mask[k] && p.mask[k][r] ? 2 : 0;
    switch (dt) {
    case B200_F64:
    case B200_F32: {
        const unsigned long long mag = v & (full >> 1), inf = dt == B200_F64 ? 0x7ff0000000000000ull : 0x7f800000ull;
        if (!cls && mag > inf)
            cls = 1;
        if (!mag)
            v = 0; // -0.0 == +0.0
        v = (v & top) ? (~v & full) : (v | top);
        break;
    }
    case B200_I64:
        if (p.nat_is_null[k] && v == 0x8000000000000000ull)
            cls = 2; // NaT of a datetime column without a mask: arrow's null
        v ^= top;
        break;
    case B200_I32:
    case B200_I16:
    case B200_I8: v ^= top; break;
    case B200_BOOL: v = v != 0; break;
    default: break;
    }
    *value = cls ? 0 : p.descending[k] ? (~v & full) : v;
    return cls;
}

// one thread per row (grid-stride): word[i] = the round's fields of row perm[i] (i in the first round, which also writes the
// identity payload); the AND and OR of every word, one atomic pair per warp
__global__ void __launch_bounds__(256) k_sort_encode(const __grid_constant__ EncodeParams p, long long n, long long *payload, int first,
                                                     unsigned long long *word, unsigned long long *andor) {
    unsigned long long a = ~0ull, o = 0;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        long long r = i;
        if (first)
            payload[i] = i;
        else
            r = payload[i];
        unsigned long long w = 0;
        for (int f = 0; f < p.nfields; f++) {
            const int k = p.fkey[f];
            unsigned long long v;
            const int cls = encode_key(p, k, r, &v);
            // class field: value 0, NaN 1, null the all-ones of its width (1 bit when a key has only one of NaN / null)
            const unsigned long long x = p.fclass[f] ? (cls == 0 ? 0ull : cls == 2 ? (1ull << p.class_bits[k]) - 1ull : 1ull) : v;
            w |= x << p.fshift[f];
        }
        word[i] = w;
        a &= w;
        o |= w;
    }
    for (int s = 16; s; s >>= 1) {
        a &= __shfl_xor_sync(0xffffffffu, a, s);
        o |= __shfl_xor_sync(0xffffffffu, o, s);
    }
    if ((threadIdx.x & 31) == 0) {
        atomicAnd(andor, a);
        atomicOr(andor + 1, o);
    }
}

int sort_blocks(b200_ctx *ctx, long long n) {
    const long long want = (n + 255) / 256;
    return (int)std::min<long long>(std::max<long long>(want, 1), (long long)ctx->sm_count * 16);
}

// the keys' fields packed into 64-bit words, least significant first: a field never straddles two words
struct SortPlan {
    int nwords = 0;
    int word_of[2 * B200_SORT_MAX_KEYS];
    int nfields = 0;
    int fkey[2 * B200_SORT_MAX_KEYS], fclass[2 * B200_SORT_MAX_KEYS], fshift[2 * B200_SORT_MAX_KEYS];
};

SortPlan plan_fields(int nkeys, const b200_sort_key *keys, const int *class_bits) {
    SortPlan pl;
    int used = 64;
    auto add = [&](int k, int cls, int bits) {
        if (used + bits > 64) {
            pl.nwords++;
            used = 0;
        }
        pl.fkey[pl.nfields] = k, pl.fclass[pl.nfields] = cls, pl.fshift[pl.nfields] = used, pl.word_of[pl.nfields] = pl.nwords - 1;
        pl.nfields++;
        used += bits;
    };
    for (int k = nkeys - 1; k >= 0; k--) {
        add(k, 0, value_bits(keys[k].dtype));
        if (class_bits[k])
            add(k, 1, class_bits[k]);
    }
    return pl;
}

} // namespace
} // namespace b200

using namespace b200;

extern "C" {

int b200_argsort(b200_ctx *ctx, int slot, int nkeys, const b200_sort_key *keys, int64_t nrows, int64_t *perm_out, uint32_t flags) {
    if (nkeys < 1 || nkeys > B200_SORT_MAX_KEYS || !keys || nrows < 0 || (nrows && !perm_out) || flags) {
        set_error("b200_argsort: invalid argument");
        return B200_ERR_INVALID;
    }
    if ((unsigned long long)nrows > B200_SORT_MAX_ROWS) {
        set_error("b200_argsort: %lld rows exceed the limit of %llu rows of one sort", (long long)nrows, (unsigned long long)B200_SORT_MAX_ROWS);
        return B200_ERR_INVALID;
    }
    EncodeParams p;
    memset(&p, 0, sizeof p);
    for (int k = 0; k < nkeys; k++) {
        const b200_sort_key &K = keys[k];
        if (K.dtype < 0 || K.dtype >= B200_NDTYPE || (nrows && !K.data) || (K.nat_is_null && K.dtype != B200_I64)) {
            set_error("b200_argsort: key %d is invalid", k);
            return B200_ERR_INVALID;
        }
        p.data[k] = K.data, p.mask[k] = K.mask, p.dtype[k] = K.dtype, p.byteswap[k] = K.byteswap != 0, p.descending[k] = K.descending != 0;
        p.nat_is_null[k] = K.nat_is_null != 0;
        const bool nan = dtype_is_float(K.dtype), null = K.mask || K.nat_is_null;
        p.class_bits[k] = nan && null ? 2 : nan || null ? 1 : 0;
    }
    if (nrows == 0)
        return B200_OK;
    const SortPlan pl = plan_fields(nkeys, keys, p.class_bits);
    Slot *sl;
    B200_CHECK(device_slot(ctx, slot, "b200_argsort", &sl));
    std::lock_guard<std::mutex> g(sl->mu);
    cudaStream_t st = sl->stream;
    const unsigned long long n = (unsigned long long)nrows;
    // scratch: word A | word B | payload B (payload A is perm_out) | radix histograms | AND / OR
    const size_t off_hist = 3 * n * 8, off_andor = off_hist + align_up(radix_scratch_bytes(n), 256);
    DevBuf<char> work;
    B200_CHECK(work.alloc(ctx, off_andor + 16, "b200_argsort", st));
    unsigned long long *win = reinterpret_cast<unsigned long long *>(work.get()), *wout = win + n;
    unsigned long long *pin = reinterpret_cast<unsigned long long *>(perm_out), *pout = wout + n;
    unsigned *hist = reinterpret_cast<unsigned *>(work + off_hist);
    unsigned long long *andor = reinterpret_cast<unsigned long long *>(work + off_andor);
    const unsigned long long init[2] = {~0ull, 0ull};
    for (int w = 0; w < pl.nwords; w++) {
        p.nfields = 0;
        for (int f = 0; f < pl.nfields; f++)
            if (pl.word_of[f] == w) {
                p.fkey[p.nfields] = pl.fkey[f], p.fclass[p.nfields] = pl.fclass[f], p.fshift[p.nfields] = pl.fshift[f];
                p.nfields++;
            }
        B200_CUDA(cudaMemcpyAsync(andor, init, 16, cudaMemcpyHostToDevice, st));
        k_sort_encode<<<sort_blocks(ctx, nrows), 256, 0, st>>>(p, nrows, reinterpret_cast<long long *>(pin), w == 0, win, andor);
        B200_CUDA(cudaGetLastError());
        unsigned long long h[2];
        B200_CUDA(cudaMemcpyAsync(h, andor, 16, cudaMemcpyDeviceToHost, st));
        B200_CUDA(cudaStreamSynchronize(st));
        // a byte every row shares orders nothing
        const unsigned long long varying = h[0] ^ h[1];
        unsigned bytes = 0;
        for (int b = 0; b < 8; b++)
            bytes |= ((varying >> (8 * b)) & 255u) ? 1u << b : 0u;
        B200_CHECK(radix_sort(n, bytes, 0, win, pin, wout, pout, hist, st));
    }
    if (pin != reinterpret_cast<unsigned long long *>(perm_out))
        B200_CUDA(cudaMemcpyAsync(perm_out, pin, n * 8, cudaMemcpyDeviceToDevice, st));
    B200_CUDA(cudaStreamSynchronize(st));
    return B200_OK;
}

} // extern "C"
