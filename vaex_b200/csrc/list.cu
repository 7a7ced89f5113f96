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
        store1_raw(out, isz, i, v);
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

// room for `more` records (and, for strings, `more_bytes` pool bytes); caller holds a->nmu.  Growth synchronises the device first:
// every append into the old arrays was enqueued under a->nmu, on any slot, so once the device has drained and the copies on `st` have
// finished, no stream can still touch the old blocks.
static int list_reserve(b200_agg *a, cudaStream_t st, uint64_t more, uint64_t more_bytes) {
    const bool str = a->op == B200_AGG_LIST_STRING;
    if (a->list_n + more > a->list_cap) {
        B200_CUDA(cudaDeviceSynchronize());
        const uint64_t cap = std::max<uint64_t>((a->list_n + more) * 2, 1u << 16);
        DevBuf<unsigned long long> nk, nv, ns;
        B200_CHECK(nk.alloc(a->ctx, cap * 8, "AggList", st));
        B200_CHECK(nv.alloc(a->ctx, cap * 8, "AggList", st));
        if (str)
            B200_CHECK(ns.alloc(a->ctx, (cap + 1) * 8, "AggList", st));
        if (a->list_n) {
            B200_CUDA(cudaMemcpyAsync(nk, a->list_keys, a->list_n * 8, cudaMemcpyDeviceToDevice, st));
            B200_CUDA(cudaMemcpyAsync(nv, a->list_vals, a->list_n * 8, cudaMemcpyDeviceToDevice, st));
            if (str)
                B200_CUDA(cudaMemcpyAsync(ns, a->list_starts, a->list_n * 8, cudaMemcpyDeviceToDevice, st));
            B200_CUDA(cudaStreamSynchronize(st));
        }
        nk.unbind(), nv.unbind(), ns.unbind();
        a->list_keys = std::move(nk), a->list_vals = std::move(nv), a->list_starts = std::move(ns), a->list_cap = cap;
    }
    if (str && (a->lstr_pool_n + more_bytes + 16 > a->lstr_pool_cap || !a->lstr_pool)) {
        B200_CUDA(cudaDeviceSynchronize());
        const uint64_t cap = std::max<uint64_t>((a->lstr_pool_n + more_bytes) * 2 + 16, 1u << 20); // + 16: the gather's read slack
        DevBuf<char> np;
        B200_CHECK(np.alloc(a->ctx, cap, "AggList_string", st));
        if (a->lstr_pool_n) {
            B200_CUDA(cudaMemcpyAsync(np, a->lstr_pool, a->lstr_pool_n, cudaMemcpyDeviceToDevice, st));
            B200_CUDA(cudaStreamSynchronize(st));
        }
        np.unbind();
        a->lstr_pool = std::move(np), a->lstr_pool_cap = cap;
    }
    return B200_OK;
}

// one b200_bin call: reserve nrows records, append (api.cu calls this for B200_AGG_LIST aggregators).  The append is enqueued under
// the aggregator's lock, like bin_list_string's.
int bin_list(b200_ctx *ctx, Slot *sl, b200_agg *a, const DevBinner *db, int nbinners, const void *data, const uint8_t *mask, int64_t nrows, bool vec) {
    std::lock_guard<std::mutex> g(a->nmu);
    B200_CHECK(list_reserve(a, sl->stream, (uint64_t)nrows, 0));
    const unsigned long long base = a->list_n;
    a->list_n += (uint64_t)nrows;
    a->list_sorted = false;
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
    B200_CHECK(list_reserve(a, sl->stream, (uint64_t)nrows, (uint64_t)in.nbytes));
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
        DevBuf<unsigned long long> kb, vb;
        DevBuf<unsigned> hist;
        B200_CHECK(kb.alloc(a->ctx, n * 8, "b200_agg_list_finish", st));
        B200_CHECK(vb.alloc(a->ctx, n * 8, "b200_agg_list_finish", st));
        B200_CHECK(hist.alloc(a->ctx, radix_scratch_bytes(n), "b200_agg_list_finish", st));
        unsigned long long *kin = a->list_keys, *vin = a->list_vals, *kout = kb, *vout = vb;
        B200_CHECK(radix_sort(n, radix_bytes_through(maxkey), 0, kin, vin, kout, vout, hist, st));
        if (kin != a->list_keys) { // an odd number of passes: the sorted records sit in the scratch arrays, which have n entries
            B200_CUDA(cudaMemcpyAsync(a->list_keys, kin, n * 8, cudaMemcpyDeviceToDevice, st));
            B200_CUDA(cudaMemcpyAsync(a->list_vals, vin, n * 8, cudaMemcpyDeviceToDevice, st));
        }
        B200_CUDA(cudaStreamSynchronize(st));
    }
    a->list_sorted = true;
    // per-cell counts -> offsets (kept on the device until read)
    const size_t cn = (size_t)a->cells + 1;
    if (!a->list_counts)
        B200_CHECK(a->list_counts.alloc(a->ctx, cn * 4, "b200_agg_list_finish"));
    B200_CUDA(cudaMemsetAsync(a->list_counts, 0, cn * 4, st));
    if (n)
        k_list_count<<<nblocks_for(n), 256, 0, st>>>(a->list_keys, n, a->list_counts, a->cells, cell_shift);
    DevBuf<unsigned long long> d_total;
    B200_CHECK(d_total.alloc(a->ctx, 8, "b200_agg_list_finish", st));
    k_scan_u32<<<1, 1024, 0, st>>>(a->list_counts, cn, d_total);
    B200_CUDA(cudaGetLastError());
    unsigned long long total = 0;
    B200_CUDA(cudaMemcpyAsync(&total, d_total, 8, cudaMemcpyDeviceToHost, st));
    B200_CUDA(cudaStreamSynchronize(st));
    a->list_total = total;
    return B200_OK;
}

// the string elements of the sorted records: int64 offsets (a scan of the lengths), the bytes gathered from the pool, validity
// (the previous outputs are replaced under a->nmu with every slot synchronised, and their readers synchronise before they unlock)
static int list_string_gather(b200_agg *a, cudaStream_t st) {
    const uint64_t total = a->list_total;
    a->lstr_bytes.reset();
    a->lstr_nbytes = 0;
    B200_CHECK(a->lstr_off.alloc(a->ctx, (total + 1) * 8, "b200_agg_list_finish"));
    B200_CHECK(a->lstr_valid.alloc(a->ctx, total, "b200_agg_list_finish"));
    B200_CUDA(cudaMemsetAsync(a->lstr_off + total, 0, 8, st));
    if (total) {
        // the record after the last one closes the pool
        B200_CUDA(cudaMemcpyAsync(a->list_starts + a->list_n, &a->lstr_pool_n, 8, cudaMemcpyHostToDevice, st));
        k_list_str_len<<<nblocks_for(total), 256, 0, st>>>(a->list_vals, a->list_starts, total, a->lstr_off);
        B200_CUDA(cudaGetLastError());
    }
    DevBuf<long long> tile_sums;
    if (const unsigned long long ns = scan_i64_sums(total + 1))
        B200_CHECK(tile_sums.alloc(a->ctx, ns * 8, "b200_agg_list_finish", st));
    B200_CHECK(scan_i64(a->lstr_off, total + 1, tile_sums, st));
    long long nbytes = 0;
    B200_CUDA(cudaMemcpyAsync(&nbytes, a->lstr_off + total, 8, cudaMemcpyDeviceToHost, st));
    B200_CUDA(cudaStreamSynchronize(st));
    a->lstr_nbytes = (uint64_t)nbytes;
    B200_CHECK(a->lstr_bytes.alloc(a->ctx, a->lstr_nbytes, "b200_agg_list_finish"));
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
    DevBuf<> d_out;
    if (a->list_total && values_out) {
        B200_CHECK(d_out.alloc(a->ctx, a->list_total * isz, "b200_agg_list_read", st));
        k_list_values<<<nblocks_for(a->list_total), 256, 0, st>>>(a->list_keys, a->list_vals, a->list_total, a->dtype, isz, d_out);
        B200_CUDA(cudaGetLastError());
        B200_CUDA(cudaMemcpyAsync(values_out, d_out, a->list_total * isz, cudaMemcpyDeviceToHost, st));
    }
    B200_CUDA(cudaStreamSynchronize(st));
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
