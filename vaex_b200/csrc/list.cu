// list.cu — AggList_<dtype>: per cell the list of the rows' values (SURVEY.md section 8f row 4).
//
// Reference: AggListPrimitive (src/agg_list.cpp:5-127): `grids` must be 1; aggregate() appends every valid, non-NaN value to its
// cell's std::vector, counts NaN values (unless dropnan) and null rows (data mask == 0, unless dropnull) per cell; get_result()
// returns offsets[cells + 1] + flat values: a cell's values in arrival order, then one NaN per counted NaN, then one (unwritten)
// slot per counted null — handed to vaex.arrow.convert.list_from_arrays.
// Device design: nothing cell-shaped is kept.  Every b200_bin call appends one record per row — key = cell * 4 + category (0 value,
// 1 NaN, 2 null; skipped rows get the all-ones key), payload = the value's bits — to a growing pair of device arrays, at positions
// reserved per call, so arrival order is (call, row) order.  Finishing = one stable LSD radix sort of the records by key (radix.cuh,
// only the bytes that vary) + a per-cell count + a scan: the sorted payloads ARE the flat values.
//
// AggList_string (AggListString, src/agg_list.cpp:122-222): per cell the strings in arrival order, a null string pushed as a null AT
// ITS ARRIVAL POSITION unless dropnull (:190-195); dropnan has no effect and the data mask is never read (AggBaseString stores it,
// src/agg_base.hpp:192-199).  Device design: the same record log — key = cell (dropped nulls: the skip key), payload = the
// record's index | null << 63 — plus, per call, the call's byte range appended to a device pool and, per record, where its string
// starts there.  Finishing = the same sort + count, then an int64 scan of the sorted records' lengths (the output string offsets)
// and a gather of the bytes by groups of threads with 16-byte stores.
#include <algorithm>

#include "binby.cuh"
#include "binby_index.cuh"
#include "radix.cuh"
#include "scan.cuh"
#include "strings.cuh"

namespace b200 {

struct ListParams {
    int nb;
    long long nrows;
    DevBinner b[B200_MAX_BINNERS];
    int dtype, isz, byteswap, dropnan, dropnull;
    const void *data;
    const uint8_t *mask; // aggregator convention: 1 = use the row, 0 = null row
    unsigned long long *keys, *vals;
    unsigned long long base;
    unsigned long long skip_key; // cells * 4: sorts behind every real record, costs no extra radix pass
};

struct ListStrParams {
    int nb, dropnull;
    long long nrows;
    DevBinner b[B200_MAX_BINNERS];
    const long long *offsets; // the call's offsets[nrows + 1] (absolute: the string of row r starts at offsets[r] - base)
    const uint8_t *valid;     // 1 = string present, 0 = null (nullable)
    long long base;
    unsigned long long *keys, *vals, *starts;
    unsigned long long rbase;    // first record of the call
    unsigned long long pbase;    // where the call's byte range starts in the pool
    unsigned long long skip_key; // cells: sorts behind every real record
};

namespace {

template <bool VEC>
__global__ void __launch_bounds__(256) k_list_append(const __grid_constant__ ListParams p) {
    const long long step = (long long)gridDim.x * 256 * 4;
    for (long long base = ((long long)blockIdx.x * 256 + threadIdx.x) * 4; base < p.nrows; base += step) {
        const long long left = p.nrows - base;
        const int nv = left < 4 ? (int)left : 4;
        unsigned long long idx[4];
        binby_indices<VEC>(p.b, p.nb, base, nv, idx);
        uint64_t r[4] = {0, 0, 0, 0};
        unsigned m[4] = {1, 1, 1, 1};
        load4_raw<VEC>(p.data, p.isz, base, nv, r);
        // REFERENCE QUIRK, kept (golden vectors from the compiled reference pin it): AggListPrimitive::aggregate runs per 1024-row
        // block of a bin() call with the block offset applied to the data but NOT to the mask (src/agg_list.cpp:96-97), so row r of
        // a call is judged by mask[r % 1024] — the same slip as AggFirst (src/agg_first.cpp:131).  base is a multiple of 4.
        if (p.mask)
            load4_mask<VEC>(p.mask, base & 1023, nv, m);
#pragma unroll
        for (int j = 0; j < 4; j++) {
            if (j >= nv)
                break;
            const uint64_t raw = p.byteswap ? bswap(r[j], p.isz) : r[j];
            unsigned long long key;
            if (m[j] == 1) {
                if (!raw_isnan(p.dtype, raw))
                    key = idx[j] * 4 + 0;
                else
                    key = p.dropnan ? p.skip_key : idx[j] * 4 + 1;
            } else {
                key = (m[j] == 0 && !p.dropnull) ? idx[j] * 4 + 2 : p.skip_key;
            }
            p.keys[p.base + base + j] = key;
            p.vals[p.base + base + j] = raw;
        }
    }
}

// shift: 2 for the numeric records (cell * 4 + category), 0 for the string records (cell)
__global__ void k_list_count(const unsigned long long *keys, unsigned long long n, unsigned *counts, unsigned long long cells, int shift) {
    for (unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (unsigned long long)gridDim.x * blockDim.x) {
        const unsigned long long k = keys[i];
        if ((k >> shift) < cells)
            atomicAdd(counts + (k >> shift), 1u);
    }
}

__global__ void k_list_values(const unsigned long long *keys, const unsigned long long *vals, unsigned long long total, int dtype, int isz, void *out) {
    for (unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (unsigned long long)gridDim.x * blockDim.x) {
        const unsigned cat = (unsigned)(keys[i] & 3ull);
        unsigned long long v = vals[i];
        if (cat == 1) // std::numeric_limits<T>::quiet_NaN()
            v = dtype == B200_F64 ? 0x7ff8000000000000ull : 0x7fc00000ull;
        else if (cat == 2)
            v = 0; // the reference leaves these slots unwritten
        switch (isz) {
        case 8: static_cast<unsigned long long *>(out)[i] = v; break;
        case 4: static_cast<unsigned *>(out)[i] = (unsigned)v; break;
        case 2: static_cast<unsigned short *>(out)[i] = (unsigned short)v; break;
        default: static_cast<unsigned char *>(out)[i] = (unsigned char)v; break;
        }
    }
}

int nblocks_for(unsigned long long n) {
    const unsigned long long b = (n + 255) / 256;
    return (int)std::max<unsigned long long>(1, std::min<unsigned long long>(b, kSmCount * 16ull));
}

// ---- AggList_string ----------------------------------------------------------------------------------------------------------
constexpr unsigned long long kNullBit = 1ull << 63;

template <bool VEC>
__global__ void __launch_bounds__(256) k_list_str_append(const __grid_constant__ ListStrParams p) {
    const long long step = (long long)gridDim.x * 256 * 4;
    for (long long base = ((long long)blockIdx.x * 256 + threadIdx.x) * 4; base < p.nrows; base += step) {
        const long long left = p.nrows - base;
        const int nv = left < 4 ? (int)left : 4;
        unsigned long long idx[4];
        binby_indices<VEC>(p.b, p.nb, base, nv, idx);
#pragma unroll
        for (int j = 0; j < 4; j++) {
            if (j >= nv)
                break;
            const long long row = base + j;
            const bool null = p.valid && p.valid[row] == 0;
            const unsigned long long rec = p.rbase + (unsigned long long)row;
            // src/agg_list.cpp:190-195: a null is pushed where it arrives unless dropnull; no other row is ever dropped
            p.keys[rec] = null && p.dropnull ? p.skip_key : idx[j];
            p.vals[rec] = rec | (null ? kNullBit : 0ull);
            p.starts[rec] = p.pbase + (unsigned long long)(p.offsets[row] - p.base);
        }
    }
}

// length of every kept record's string in sorted order (0 for a null: StringList::push_null pushes an empty string, src/superstring.hpp:729-734)
__global__ void k_list_str_len(const unsigned long long *vals, const unsigned long long *starts, unsigned long long total, long long *len) {
    for (unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (unsigned long long)gridDim.x * blockDim.x) {
        const unsigned long long v = vals[i], rec = v & ~kNullBit;
        len[i] = (v & kNullBit) ? 0 : (long long)(starts[rec + 1] - starts[rec]);
    }
}

// 16 bytes of the byte stream that starts `mis` (1..15) bytes into the aligned word `a`, followed by `b`
__device__ __forceinline__ uint4 shift16(uint4 a, uint4 b, int mis) {
    const int q = mis >> 2;
    const unsigned r = (unsigned)(mis & 3) * 8;
    const unsigned w0 = q == 0 ? a.x : q == 1 ? a.y : q == 2 ? a.z : a.w;
    const unsigned w1 = q == 0 ? a.y : q == 1 ? a.z : q == 2 ? a.w : b.x;
    const unsigned w2 = q == 0 ? a.z : q == 1 ? a.w : q == 2 ? b.x : b.y;
    const unsigned w3 = q == 0 ? a.w : q == 1 ? b.x : q == 2 ? b.y : b.z;
    const unsigned w4 = q == 0 ? b.x : q == 1 ? b.y : q == 2 ? b.z : b.w;
    return make_uint4(__funnelshift_r(w0, w1, r), __funnelshift_r(w1, w2, r), __funnelshift_r(w2, w3, r), __funnelshift_r(w3, w4, r));
}

// G threads copy one string: single bytes up to the first 16-byte boundary of the destination, then 16-byte stores (16-byte loads
// when source and destination are equally misaligned, else two aligned loads and a funnel shift), then the last bytes.  The source
// reads may run up to 16 bytes past the string: the pool is allocated with that much slack.
template <int G>
__device__ __forceinline__ void copy_string(char *dst, const char *src, long long len, int lane) {
    const long long head = min(len, (long long)((16 - (reinterpret_cast<uintptr_t>(dst) & 15)) & 15));
    for (long long c = lane; c < head; c += G)
        dst[c] = src[c];
    const long long chunks = (len - head) >> 4;
    uint4 *d = reinterpret_cast<uint4 *>(dst + head);
    const char *s = src + head;
    const int mis = (int)(reinterpret_cast<uintptr_t>(s) & 15);
    const uint4 *s4 = reinterpret_cast<const uint4 *>(s - mis);
    if (mis == 0) {
        for (long long c = lane; c < chunks; c += G)
            d[c] = __ldg(s4 + c);
    } else {
        for (long long c = lane; c < chunks; c += G)
            d[c] = shift16(__ldg(s4 + c), __ldg(s4 + c + 1), mis);
    }
    for (long long c = head + chunks * 16 + lane; c < len; c += G)
        dst[c] = src[c];
}

template <int G>
__global__ void __launch_bounds__(256) k_list_str_gather(const unsigned long long *vals, const unsigned long long *starts, const long long *off,
                                                         unsigned long long total, const char *pool, char *out, uint8_t *valid) {
    const int lane = threadIdx.x % G;
    const unsigned long long groups = (unsigned long long)gridDim.x * (256 / G);
    for (unsigned long long i = ((unsigned long long)blockIdx.x * 256 + threadIdx.x) / G; i < total; i += groups) {
        const unsigned long long v = vals[i];
        if (lane == 0)
            valid[i] = (v & kNullBit) ? 0 : 1;
        const long long o = off[i], len = off[i + 1] - o;
        if (len)
            copy_string<G>(out + o, pool + starts[v & ~kNullBit], len, lane);
    }
}

} // namespace

// room for `more` records (and, for strings, `more_bytes` pool bytes); caller holds a->nmu.  Growth synchronises the device: other
// slots may be appending into the old arrays
static int list_reserve(b200_agg *a, uint64_t more, uint64_t more_bytes) {
    const bool str = a->op == B200_AGG_LIST_STRING;
    if (a->list_n + more > a->list_cap) {
        B200_CUDA(cudaDeviceSynchronize());
        const uint64_t cap = std::max<uint64_t>((a->list_n + more) * 2, 1u << 16);
        unsigned long long *nk = nullptr, *nv = nullptr, *ns = nullptr;
        B200_CUDA(cudaMalloc(&nk, cap * 8));
        B200_CUDA(cudaMalloc(&nv, cap * 8));
        if (str)
            B200_CUDA(cudaMalloc(&ns, (cap + 1) * 8));
        if (a->list_n) {
            B200_CUDA(cudaMemcpy(nk, a->list_keys, a->list_n * 8, cudaMemcpyDeviceToDevice));
            B200_CUDA(cudaMemcpy(nv, a->list_vals, a->list_n * 8, cudaMemcpyDeviceToDevice));
            if (str)
                B200_CUDA(cudaMemcpy(ns, a->list_starts, a->list_n * 8, cudaMemcpyDeviceToDevice));
        }
        cudaFree(a->list_keys);
        cudaFree(a->list_vals);
        cudaFree(a->list_starts);
        a->list_keys = nk, a->list_vals = nv, a->list_starts = ns, a->list_cap = cap;
    }
    if (str && (a->lstr_pool_n + more_bytes + 16 > a->lstr_pool_cap || !a->lstr_pool)) {
        B200_CUDA(cudaDeviceSynchronize());
        const uint64_t cap = std::max<uint64_t>((a->lstr_pool_n + more_bytes) * 2 + 16, 1u << 20); // + 16: the gather's read slack
        char *np = nullptr;
        B200_CUDA(cudaMalloc(&np, cap));
        if (a->lstr_pool_n)
            B200_CUDA(cudaMemcpy(np, a->lstr_pool, a->lstr_pool_n, cudaMemcpyDeviceToDevice));
        cudaFree(a->lstr_pool);
        a->lstr_pool = np, a->lstr_pool_cap = cap;
    }
    return B200_OK;
}

// one b200_bin call: reserve nrows records, append (api.cu calls this for B200_AGG_LIST aggregators)
int bin_list(b200_ctx *ctx, Slot *sl, b200_agg *a, const DevBinner *db, int nbinners, const void *data, const uint8_t *mask, int64_t nrows, bool vec) {
    unsigned long long base;
    {
        std::lock_guard<std::mutex> g(a->nmu);
        B200_CHECK(list_reserve(a, (uint64_t)nrows, 0));
        base = a->list_n;
        a->list_n += (uint64_t)nrows;
        a->list_sorted = false;
    }
    ListParams p;
    memset(&p, 0, sizeof p);
    p.nb = nbinners;
    p.nrows = nrows;
    memcpy(p.b, db, sizeof(DevBinner) * nbinners);
    p.dtype = a->dtype;
    p.isz = dtype_size(a->dtype);
    p.byteswap = a->byteswap && p.isz > 1;
    p.dropnan = (a->moment & 1) != 0; // AggList_<T>(grid, grids, threads, dropnan, dropnull): carried in `moment` like NUNIQUE's flags
    p.dropnull = (a->moment & 2) != 0;
    p.data = data;
    p.mask = mask;
    p.keys = a->list_keys;
    p.vals = a->list_vals;
    p.base = base;
    p.skip_key = a->cells * 4;
    const bool v = vec && !(reinterpret_cast<uintptr_t>(data) & 15) && !(reinterpret_cast<uintptr_t>(mask) & 15);
    const int blocks = nblocks_for(((unsigned long long)nrows + 3) / 4);
    if (v)
        k_list_append<true><<<blocks, 256, 0, sl->stream>>>(p);
    else
        k_list_append<false><<<blocks, 256, 0, sl->stream>>>(p);
    B200_CUDA(cudaGetLastError());
    (void)ctx;
    return B200_OK;
}

// one b200_bin call of a B200_AGG_LIST_STRING aggregator: reserve nrows records and the call's bytes, append both.  The pool copy
// and the append kernel are enqueued under the aggregator's lock, so a growth on another slot (which synchronises the device
// before it frees the old arrays) can never run between reading the pointers and using them.
int bin_list_string(b200_ctx *ctx, Slot *sl, b200_agg *a, const DevBinner *db, int nbinners, const StrInput &in, int64_t nrows, bool vec) {
    std::lock_guard<std::mutex> g(a->nmu);
    B200_CHECK(list_reserve(a, (uint64_t)nrows, (uint64_t)in.nbytes));
    ListStrParams p;
    memset(&p, 0, sizeof p);
    p.nb = nbinners;
    p.nrows = nrows;
    memcpy(p.b, db, sizeof(DevBinner) * nbinners);
    p.dropnull = (a->moment & 2) != 0; // bit 0, dropnan, has no effect on strings (src/agg_list.cpp:122-222 never reads it)
    p.offsets = in.offsets;
    p.valid = in.masks;
    p.base = in.base;
    p.keys = a->list_keys;
    p.vals = a->list_vals;
    p.starts = a->list_starts;
    p.rbase = a->list_n;
    p.pbase = a->lstr_pool_n;
    p.skip_key = a->cells;
    if (in.nbytes)
        B200_CUDA(cudaMemcpyAsync(a->lstr_pool + a->lstr_pool_n, in.bytes, (size_t)in.nbytes, cudaMemcpyDeviceToDevice, sl->stream));
    const int blocks = nblocks_for(((unsigned long long)nrows + 3) / 4);
    if (vec)
        k_list_str_append<true><<<blocks, 256, 0, sl->stream>>>(p);
    else
        k_list_str_append<false><<<blocks, 256, 0, sl->stream>>>(p);
    B200_CUDA(cudaGetLastError());
    a->list_n += (uint64_t)nrows;
    a->lstr_pool_n += (uint64_t)in.nbytes;
    a->list_sorted = false;
    (void)ctx;
    return B200_OK;
}

// sorts the records once (stable LSD radix sort on the bytes of the key that can differ, keys <= maxkey) and counts the kept ones
// per cell: list_counts = exclusive offsets per cell, list_total = the kept records (they lead the sorted arrays).  Both list kinds
// finish through here.  Caller holds a->nmu, every slot synchronised.
static int list_sort_count(b200_agg *a, cudaStream_t st, unsigned long long maxkey, int cell_shift) {
    const uint64_t n = a->list_n;
    if (!a->list_sorted && n > 1) {
        if (n >= (1ull << 32)) {
            set_error("AggList: more than 2^32 rows are not supported");
            return B200_ERR_UNSUPPORTED;
        }
        const unsigned nblk = radix_blocks(n), tiles = radix_tiles(n);
        unsigned long long *kb = nullptr, *vb = nullptr;
        unsigned *hist = nullptr;
        B200_CUDA(cudaMalloc(&kb, n * 8));
        B200_CUDA(cudaMalloc(&vb, n * 8));
        B200_CUDA(cudaMalloc(&hist, (size_t)256 * nblk * 4));
        unsigned long long *kin = a->list_keys, *vin = a->list_vals, *kout = kb, *vout = vb;
        for (int shift = 0; shift < 64 && (maxkey >> shift); shift += 8) {
            k_radix_hist<<<nblk, kRadixThreads, 0, st>>>(kin, vin, n, shift, 0, hist, nblk, tiles);
            k_scan_u32<<<1, 1024, 0, st>>>(hist, 256ull * nblk);
            k_radix_scatter<<<nblk, kRadixThreads, 0, st>>>(kin, vin, kout, vout, n, shift, 0, hist, nblk, tiles);
            B200_CUDA(cudaGetLastError());
            std::swap(kin, kout);
            std::swap(vin, vout);
        }
        B200_CUDA(cudaStreamSynchronize(st));
        if (kin != a->list_keys) { // an odd number of passes: the sorted records sit in the scratch arrays, which have n entries
            B200_CUDA(cudaMemcpy(a->list_keys, kin, n * 8, cudaMemcpyDeviceToDevice));
            B200_CUDA(cudaMemcpy(a->list_vals, vin, n * 8, cudaMemcpyDeviceToDevice));
        }
        cudaFree(kb);
        cudaFree(vb);
        cudaFree(hist);
    }
    a->list_sorted = true;
    // per-cell counts -> offsets (kept on the device until read)
    const size_t cn = (size_t)a->cells + 1;
    if (!a->list_counts)
        B200_CUDA(cudaMalloc((void **)&a->list_counts, cn * 4));
    B200_CUDA(cudaMemsetAsync(a->list_counts, 0, cn * 4, st));
    if (n)
        k_list_count<<<nblocks_for(n), 256, 0, st>>>(a->list_keys, n, a->list_counts, a->cells, cell_shift);
    unsigned long long *d_total = nullptr;
    B200_CUDA(cudaMalloc((void **)&d_total, 8));
    k_scan_u32<<<1, 1024, 0, st>>>(a->list_counts, cn, d_total);
    B200_CUDA(cudaGetLastError());
    unsigned long long total = 0;
    B200_CUDA(cudaMemcpyAsync(&total, d_total, 8, cudaMemcpyDeviceToHost, st));
    B200_CUDA(cudaStreamSynchronize(st));
    cudaFree(d_total);
    a->list_total = total;
    return B200_OK;
}

// the string elements of the sorted records: int64 offsets (a scan of the lengths), the bytes gathered from the pool, validity
static int list_string_gather(b200_agg *a, cudaStream_t st) {
    const uint64_t total = a->list_total;
    cudaFree(a->lstr_off);
    cudaFree(a->lstr_bytes);
    cudaFree(a->lstr_valid);
    a->lstr_off = nullptr, a->lstr_bytes = nullptr, a->lstr_valid = nullptr, a->lstr_nbytes = 0;
    B200_CUDA(cudaMalloc((void **)&a->lstr_off, (total + 1) * 8));
    B200_CUDA(cudaMalloc((void **)&a->lstr_valid, total ? total : 1));
    B200_CUDA(cudaMemsetAsync(a->lstr_off + total, 0, 8, st));
    if (total) {
        // the record after the last one closes the pool
        B200_CUDA(cudaMemcpyAsync(a->list_starts + a->list_n, &a->lstr_pool_n, 8, cudaMemcpyHostToDevice, st));
        k_list_str_len<<<nblocks_for(total), 256, 0, st>>>(a->list_vals, a->list_starts, total, a->lstr_off);
        B200_CUDA(cudaGetLastError());
    }
    B200_CHECK(scan_i64(a->lstr_off, total + 1, st));
    long long nbytes = 0;
    B200_CUDA(cudaMemcpyAsync(&nbytes, a->lstr_off + total, 8, cudaMemcpyDeviceToHost, st));
    B200_CUDA(cudaStreamSynchronize(st));
    a->lstr_nbytes = (uint64_t)nbytes;
    B200_CUDA(cudaMalloc((void **)&a->lstr_bytes, a->lstr_nbytes ? a->lstr_nbytes : 1));
    if (total) {
        // a group of threads per string, sized by the mean length: short strings must not leave most of a warp idle
        const uint64_t mean = a->lstr_nbytes / total;
        if (mean > 256)
            k_list_str_gather<32><<<nblocks_for(total * 32), 256, 0, st>>>(a->list_vals, a->list_starts, a->lstr_off, total, a->lstr_pool, a->lstr_bytes, a->lstr_valid);
        else if (mean > 32)
            k_list_str_gather<8><<<nblocks_for(total * 8), 256, 0, st>>>(a->list_vals, a->list_starts, a->lstr_off, total, a->lstr_pool, a->lstr_bytes, a->lstr_valid);
        else
            k_list_str_gather<4><<<nblocks_for(total * 4), 256, 0, st>>>(a->list_vals, a->list_starts, a->lstr_off, total, a->lstr_pool, a->lstr_bytes, a->lstr_valid);
        B200_CUDA(cudaGetLastError());
    }
    B200_CUDA(cudaStreamSynchronize(st));
    return B200_OK;
}

} // namespace b200

using namespace b200;

extern "C" {

/* sorts the records and reports the length of the flat value array (offsets[cells]); every slot is synchronised first.  String
 * lists also gather their elements here (b200_agg_list_string_bytes / _read hand them out). */
int b200_agg_list_finish(b200_agg *a, int64_t *total_out) {
    if (!a || (a->op != B200_AGG_LIST && a->op != B200_AGG_LIST_STRING) || !total_out) {
        set_error("b200_agg_list_finish: not a list aggregator");
        return B200_ERR_INVALID;
    }
    B200_CUDA(cudaSetDevice(a->ctx->device));
    B200_CHECK(b200_ctx_sync(a->ctx, -1));
    std::lock_guard<std::mutex> g(a->nmu);
    cudaStream_t st = a->ctx->slots[0]->stream;
    if (a->op == B200_AGG_LIST) {
        // keys are cell * 4 + category (skipped rows: cells * 4): only the bytes that can differ are sorted on
        B200_CHECK(list_sort_count(a, st, a->cells * 4 + 3, 2));
    } else {
        B200_CHECK(list_sort_count(a, st, a->cells, 0)); // keys are cells, skipped rows: cells
        B200_CHECK(list_string_gather(a, st));
    }
    *total_out = (int64_t)a->list_total;
    return B200_OK;
}

/* after b200_agg_list_finish: offsets_out = int64[cells + 1], values_out = total elements of the aggregator's dtype */
int b200_agg_list_read(b200_agg *a, int64_t *offsets_out, void *values_out) {
    if (!a || a->op != B200_AGG_LIST || !offsets_out || !a->list_sorted || !a->list_counts) {
        set_error("b200_agg_list_read: call b200_agg_list_finish first");
        return B200_ERR_STATE;
    }
    B200_CUDA(cudaSetDevice(a->ctx->device));
    std::lock_guard<std::mutex> g(a->nmu);
    cudaStream_t st = a->ctx->slots[0]->stream;
    const size_t cn = (size_t)a->cells + 1;
    std::vector<unsigned> off(cn);
    B200_CUDA(cudaMemcpyAsync(off.data(), a->list_counts, cn * 4, cudaMemcpyDeviceToHost, st));
    const int isz = dtype_size(a->dtype);
    void *d_out = nullptr;
    if (a->list_total && values_out) {
        B200_CUDA(cudaMalloc(&d_out, a->list_total * isz));
        k_list_values<<<nblocks_for(a->list_total), 256, 0, st>>>(a->list_keys, a->list_vals, a->list_total, a->dtype, isz, d_out);
        B200_CUDA(cudaGetLastError());
        B200_CUDA(cudaMemcpyAsync(values_out, d_out, a->list_total * isz, cudaMemcpyDeviceToHost, st));
    }
    B200_CUDA(cudaStreamSynchronize(st));
    cudaFree(d_out);
    for (size_t i = 0; i < cn; i++)
        offsets_out[i] = (int64_t)off[i];
    return B200_OK;
}

/* after b200_agg_list_finish of a string list: the bytes of all its elements */
int b200_agg_list_string_bytes(b200_agg *a, int64_t *nbytes_out) {
    if (!a || a->op != B200_AGG_LIST_STRING || !nbytes_out || !a->list_sorted || !a->lstr_off) {
        set_error("b200_agg_list_string_bytes: call b200_agg_list_finish on a string list aggregator first");
        return B200_ERR_STATE;
    }
    *nbytes_out = (int64_t)a->lstr_nbytes;
    return B200_OK;
}

/* after b200_agg_list_finish of a string list (host buffers, each nullable): list_offsets int64[cells + 1], str_offsets
 * int64[total + 1], bytes[nbytes], valid uint8[total] (1 = string, 0 = null) */
int b200_agg_list_string_read(b200_agg *a, int64_t *list_offsets_out, int64_t *str_offsets_out, uint8_t *bytes_out, uint8_t *valid_out) {
    if (!a || a->op != B200_AGG_LIST_STRING || !a->list_sorted || !a->list_counts || !a->lstr_off) {
        set_error("b200_agg_list_string_read: call b200_agg_list_finish on a string list aggregator first");
        return B200_ERR_STATE;
    }
    B200_CUDA(cudaSetDevice(a->ctx->device));
    std::lock_guard<std::mutex> g(a->nmu);
    cudaStream_t st = a->ctx->slots[0]->stream;
    const size_t cn = (size_t)a->cells + 1;
    std::vector<unsigned> off(list_offsets_out ? cn : 0);
    if (list_offsets_out)
        B200_CUDA(cudaMemcpyAsync(off.data(), a->list_counts, cn * 4, cudaMemcpyDeviceToHost, st));
    if (str_offsets_out)
        B200_CUDA(cudaMemcpyAsync(str_offsets_out, a->lstr_off, (a->list_total + 1) * 8, cudaMemcpyDeviceToHost, st));
    if (bytes_out && a->lstr_nbytes)
        B200_CUDA(cudaMemcpyAsync(bytes_out, a->lstr_bytes, a->lstr_nbytes, cudaMemcpyDeviceToHost, st));
    if (valid_out && a->list_total)
        B200_CUDA(cudaMemcpyAsync(valid_out, a->lstr_valid, a->list_total, cudaMemcpyDeviceToHost, st));
    B200_CUDA(cudaStreamSynchronize(st));
    for (size_t i = 0; i < off.size(); i++)
        list_offsets_out[i] = (int64_t)off[i];
    return B200_OK;
}

} // extern "C"
