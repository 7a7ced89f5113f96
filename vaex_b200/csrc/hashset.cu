// hashset.cu — device ordered_set: the reference's hash-map ordinal encoder
// (src/hash_primitives.hpp:437-725 ordered_set on hash_base :41-330, hash functors src/hash.hpp:40-152).
//
// Reference semantics reproduced (for the sequential, chunks-in-order run of the reference):
//   * a key's shard is hash<T>(key) % nmaps; its shard-local ordinal is its insertion rank in that shard, i.e.
//     the rank of its FIRST occurrence in (update call, row) order (_update :98-295 buckets rows in order and
//     flushes bucket by bucket; add_new :471-479 assigns map.size()).
//   * NaN / null live in shard 0 and take the next shard-0 ordinal at the END of the update call that first
//     sees them (:264-287; null before NaN when use_offsets, NaN before null otherwise; add_nan/add_null :454-468).
//   * global ordinal = shard-local ordinal + offsets[shard] (src/hash.hpp:337-353).
// Device design: one open-addressing table {key, first-occurrence tag} filled with atomicCAS + atomicMin
// (tag = call_seq << 40 | row).  Ordinals are materialised lazily: compact -> bitonic sort by (shard, tag) ->
// position in the sorted list IS the global ordinal -> build a {key, ordinal} probe table (one 16-byte sector
// per probe) used by map_ordinal / isin and by the fused B200_BINNER_HASH binner.
#include <algorithm>

#include "binby.cuh"
#include "device_utils.cuh"
#include "radix.cuh"
#include "scan.cuh"
#include "settable.cuh"
#include "strings.cuh"

namespace b200 {
struct StrLog {
    unsigned long long hash, off;
    unsigned len, pad;
};
} // namespace b200

struct b200_set {
    b200_ctx *ctx = nullptr;
    int dtype = 0, nmaps = 1;
    int64_t limit = -1;
    b200::DevBuf<b200::SetSlot> table; // insert table: first = tag
    uint64_t cap = 0;
    b200::DevBuf<unsigned long long> counts; // counter<T> mode (src/hash_primitives.hpp:344-433): occurrences per slot, parallel to `table`
    bool counting = false;
    bool hold_count_pass = false; // merge: keys are inserted first, the other set's counts are added afterwards
    b200::DevBuf<unsigned long long> d_ctr; // see CTR_*
    int64_t seq = 0;
    bool dirty = true;
    // finalized view
    b200::DevBuf<b200::SetSlot> probe; // first = global ordinal
    uint64_t probe_cap = 0;
    b200::DevBuf<long long> d_offsets; // nmaps
    std::vector<uint64_t> h_keys;      // canonical patterns in ordinal order (special slots hold 0); filled lazily from d_keys_ord
    bool h_keys_valid = false;
    b200::DevBuf<unsigned long long> d_keys_ord; // n_entries canonical patterns in ordinal order (device)
    uint64_t n_entries = 0;                      // keys + NaN + null slots
    int64_t max_call_rows = 0;                   // largest update so far: bounds the row part of every tag
    // string keys (ordered_set_string): the table's key is the reference's 64-bit string hash; the bytes of every distinct key live
    // in `pool`, described by `log` (one record per key, in claim order); slot_log[table slot] = index of the key's record
    bool strings = false;
    b200::DevBuf<char> pool;
    uint64_t pool_cap = 0;
    b200::DevBuf<b200::StrLog> log;
    b200::DevBuf<unsigned> slot_log;           // parallel to `table`
    b200::DevBuf<unsigned long long> d_strctr;  // [0] records in `log`, [1] bytes used in `pool`
    b200::DevBuf<unsigned long long> d_str_off; // finalized: pool offset of the key with ordinal i
    b200::DevBuf<unsigned> d_str_len;
    std::vector<int64_t> h_offsets;
    int64_t n_keys = 0, nan_count = 0, null_count = 0;
    int64_t nan_value = 0x7fffffff, null_value = 0x7fffffff; // src/hash_primitives.hpp:447
    int64_t sentinel_ordinal = -1;
    // index_hash<T> (`indexing`, src/hash_primitives.hpp:731-1040): the table's `first` holds the key's smallest global row (biased,
    // see index_bias); every non-NaN, non-null row is appended to a row log {canonical key, global row}; the first map_index_duplicates
    // after a change sorts the log by (table slot, row) into per-slot ranges: primary row first, then the overflow in row order
    bool indexing = false;
    b200::DevBuf<unsigned long long> log_key;
    b200::DevBuf<long long> log_row;
    uint64_t log_n = 0, log_cap = 0;
    int64_t row_min = INT64_MAX, row_max = INT64_MIN;
    bool idx_sorted = false;
    b200::DevBuf<long long> idx_rows; // the log's rows sorted by (slot, row)
    b200::DevBuf<uint2> idx_seg;      // per table slot (+1: the key whose pattern is SET_EMPTY): [begin, end) in idx_rows
    std::mutex mu;
};

namespace b200 {

enum { CTR_COUNT = 0, CTR_OVERFLOW, CTR_NAN_COUNT, CTR_NULL_COUNT, CTR_NAN_TAG, CTR_NULL_TAG, CTR_SENTINEL_TAG, CTR_CURSOR, CTR_SENTINEL_COUNT, CTR_STR_ERROR /* 1: hash == empty pattern, 2: two strings share a 64-bit hash */,
       CTR_NAN_MAX, CTR_NULL_MAX, CTR_LOG /* index mode: largest biased NaN / null row, rows in the log */, CTR_N };

namespace {

constexpr unsigned long long kTagLowMask = (1ULL << 40) - 1;

// index mode keeps rows as unsigned tags: flipping the sign bit makes unsigned order the signed order of the rows (a negative
// start_index works), and 0 — the bias of INT64_MIN — stands for "no row" in the NaN / null maxima
__host__ __device__ __forceinline__ unsigned long long index_bias(long long row) { return (unsigned long long)row ^ (1ull << 63); }
__host__ __device__ __forceinline__ long long index_unbias(unsigned long long tag) { return (long long)(tag ^ (1ull << 63)); }

// hash_base::_update (src/hash_primitives.hpp:98-295).  from_keys: ordered_set::create (:486-537) where row i IS the ordinal.
__global__ void __launch_bounds__(256) k_set_insert(SetSlot *table, unsigned long long mask, unsigned long long *ctr, int dtype,
                                                    int isz, const void *keys, const uint8_t *masks, long long row0, long long nrows,
                                                    unsigned long long tag_base, int skip_keys, long long from_keys_null_index, int from_keys,
                                                    unsigned long long nan_low, unsigned long long null_low) {
    bool dead = false;
    unsigned it = 0;
    // NaN / null bookkeeping is accumulated per thread and published once (same-address atomics serialise in the L2)
    unsigned long long n_nan = 0, n_null = 0, t_nan = ~0ull, t_null = ~0ull;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < nrows; i += (long long)gridDim.x * blockDim.x) {
        // once the table overflowed this launch will be redone after a growth: stop inserting (and stop altogether on a redo,
        // whose NaN/null rows were already counted)
        if (!dead && (it++ % kPollRows) == 0 && overflow_seen(ctr + CTR_OVERFLOW))
            dead = true;
        if (dead && (skip_keys & 2))
            return;
        const long long row = row0 + i;
        uint64_t raw = ldcs1_raw(keys, isz, row);
        bool isnull = from_keys ? (row == from_keys_null_index) : (masks && masks[row]);
        if (isnull) {
            if (!(skip_keys & 2)) { // bit 1: this range is being redone after a table growth — specials were already counted
                n_null++;
                t_null = min(t_null, from_keys ? (unsigned long long)row : (tag_base | null_low));
            }
            continue;
        }
        if (raw_isnan(dtype, raw)) {
            if (!(skip_keys & 2)) {
                n_nan++;
                t_nan = min(t_nan, from_keys ? (unsigned long long)row : (tag_base | nan_low));
            }
            continue;
        }
        if ((skip_keys & 1) || dead)
            continue;
        unsigned long long canon = key_canon(dtype, raw);
        unsigned long long tag = tag_base + (unsigned long long)row; // == tag_base | row for an ordered set (row < 2^40)
        if (canon == SET_EMPTY) {
            atomicMin(ctr + CTR_SENTINEL_TAG, tag);
            continue;
        }
        if (!set_insert(table, mask, canon, tag)) { // the host grows the table and redoes this range
            overflow_raise(ctr + CTR_OVERFLOW);
            dead = true;
        }
    }
    if (n_null) {
        atomicAdd(ctr + CTR_NULL_COUNT, n_null);
        atomicMin(ctr + CTR_NULL_TAG, t_null);
    }
    if (n_nan) {
        atomicAdd(ctr + CTR_NAN_COUNT, n_nan);
        atomicMin(ctr + CTR_NAN_TAG, t_nan);
    }
}

// counter<T>::add_new / add_existing (src/hash_primitives.hpp:377-386): one occurrence per row.  Runs AFTER the insert pass of
// the same rows succeeded, so every key is present and the pass is not repeated when the table grows.
__global__ void __launch_bounds__(256) k_set_count(const SetSlot *table, unsigned long long mask, unsigned long long *counts, unsigned long long *ctr, int dtype,
                                                   int isz, const void *keys, const uint8_t *masks, const unsigned long long *weights, long long nrows) {
    unsigned long long n_sent = 0;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < nrows; i += (long long)gridDim.x * blockDim.x) {
        const uint64_t raw = ldcs1_raw(keys, isz, i);
        if ((masks && masks[i]) || raw_isnan(dtype, raw))
            continue; // NaN / null occurrences are counted by k_set_insert
        const unsigned long long w = weights ? weights[i] : 1ull;
        const unsigned long long canon = key_canon(dtype, raw);
        if (canon == SET_EMPTY) {
            n_sent += w;
            continue;
        }
        const unsigned long long h = set_slot(table, mask, canon); // present: the insert pass of these rows succeeded
        if (h != ~0ull)
            atomicAdd(counts + h, w);
    }
    if (n_sent)
        atomicAdd(ctr + CTR_SENTINEL_COUNT, n_sent);
}

// counts in ordinal order: slot -> ordinal through the finalized probe table
__global__ void k_counts_gather(const SetSlot *table, unsigned long long cap, const unsigned long long *counts, const SetSlot *probe, unsigned long long pmask,
                                unsigned long long *out) {
    for (unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; i < cap; i += (unsigned long long)gridDim.x * blockDim.x) {
        const unsigned long long k = table[i].key;
        if (k == SET_EMPTY)
            continue;
        const unsigned long long h = set_slot(probe, pmask, k); // present: every key of the table is in the probe table
        if (h != ~0ull)
            out[probe[h].first] = counts[i];
    }
}

__global__ void k_set_init(SetSlot *table, unsigned long long cap) {
    for (unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; i < cap; i += (unsigned long long)gridDim.x * blockDim.x) {
        table[i].key = SET_EMPTY;
        table[i].first = 0xFFFFFFFFFFFFFFFFULL;
    }
}

__global__ void k_set_rehash(const SetSlot *old, unsigned long long old_cap, SetSlot *table, unsigned long long mask, const unsigned long long *old_counts,
                             unsigned long long *counts, const unsigned *old_aux = nullptr, unsigned *aux = nullptr) {
    for (unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; i < old_cap; i += (unsigned long long)gridDim.x * blockDim.x) {
        unsigned long long k = old[i].key;
        if (k == SET_EMPTY)
            continue;
        const unsigned long long h = set_claim(table, mask, k);
        table[h].first = old[i].first;
        if (counts)
            counts[h] = old_counts[i];
        if (aux)
            aux[h] = old_aux[i];
    }
}

// occupied slots -> dense arrays (unordered): sort key = first-occurrence tag, payload = shard << 32 | index into ckey
__global__ void k_set_compact(const SetSlot *table, unsigned long long cap, unsigned long long *ctr, unsigned long long *ckey, unsigned long long *ctag,
                              unsigned long long *cval, int dtype, int nmaps) {
    const unsigned lane = threadIdx.x & 31;
    for (unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; i < cap; i += (unsigned long long)gridDim.x * blockDim.x) {
        const ulonglong2 slot = *reinterpret_cast<const ulonglong2 *>(table + i);
        const bool occ = slot.x != SET_EMPTY;
        // one cursor bump per warp, not per occupied slot (same-address atomics serialise in the L2)
        const unsigned act = __activemask();
        const unsigned m = __ballot_sync(act, occ);
        unsigned long long base = 0;
        const int leader = __ffs(m) - 1;
        if (occ && (int)lane == leader)
            base = atomicAdd(ctr + CTR_CURSOR, (unsigned long long)__popc(m));
        base = __shfl_sync(act, base, leader < 0 ? 0 : leader);
        if (occ && ckey) { // ckey == nullptr: counting pass only
            const unsigned long long pos = base + __popc(m & ((1u << lane) - 1u));
            ckey[pos] = slot.x;
            ctag[pos] = slot.y;
            cval[pos] = ((key_hash(dtype, slot.x) % (unsigned long long)nmaps) << 32) | pos;
        }
    }
}

// after the sort: position == global ordinal.  Gathers the keys into ordinal order, builds the {key, ordinal} probe table, notes
// where every shard starts and where the special entries (indices >= n_table of the compacted arrays) ended up.
__global__ void k_set_finish(const unsigned long long *val, const unsigned long long *ckey, unsigned long long E, unsigned long long n_table, int sent_idx,
                             int nan_idx, int null_idx, SetSlot *probe, unsigned long long pmask, unsigned long long *keys_ord, long long *shard_first,
                             long long *special_ord) {
    for (unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; i < E; i += (unsigned long long)gridDim.x * blockDim.x) {
        const unsigned long long v = val[i];
        const unsigned shard = (unsigned)(v >> 32);
        const unsigned long long src = v & 0xffffffffull;
        if (i == 0 || (unsigned)(val[i - 1] >> 32) != shard)
            shard_first[shard] = (long long)i;
        unsigned long long k = ckey[src];
        if (src >= n_table) {
            const int which = (int)(src - n_table);
            if (which == sent_idx) {
                special_ord[0] = (long long)i;
            } else {
                special_ord[which == nan_idx ? 1 : 2] = (long long)i;
                keys_ord[i] = 0;
                continue; // NaN / null: not a key of the probe table
            }
            keys_ord[i] = k;
            continue; // the key whose pattern equals SET_EMPTY cannot live in the table either
        }
        keys_ord[i] = k;
        probe[set_claim(probe, pmask, k)].first = i;
    }
}

// ordered_set::_map_ordinal (src/hash_primitives.hpp:624-691).  out_isz selects int8/16/32/64; out_isz == 0: isin (uint8)
__global__ void __launch_bounds__(256) k_set_map(const SetSlot *probe, unsigned long long mask, long long sentinel_ordinal, long long nan_ordinal, int dtype,
                                                 int isz, const void *keys, long long nrows, void *out, int out_isz) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < nrows; i += (long long)gridDim.x * blockDim.x) {
        uint64_t raw = ldcs1_raw(keys, isz, i);
        long long v = raw_isnan(dtype, raw) ? nan_ordinal : set_ordinal(probe, mask, sentinel_ordinal, key_canon(dtype, raw));
        if (out_isz)
            store1_raw(out, out_isz, i, (uint64_t)v);
        else
            static_cast<unsigned char *>(out)[i] = v >= 0;
    }
}

// fused ordinal lookup of up to B200_MAX_COMBINE key columns -> one int64 group code (vaex/groupby.py:526-584)
struct CombineParams {
    int nkeys;
    const SetSlot *probe[B200_MAX_COMBINE];
    unsigned long long mask[B200_MAX_COMBINE];
    long long sentinel[B200_MAX_COMBINE], nan_ord[B200_MAX_COMBINE], null_ord[B200_MAX_COMBINE], mult[B200_MAX_COMBINE];
    int dtype[B200_MAX_COMBINE], isz[B200_MAX_COMBINE];
    const void *keys[B200_MAX_COMBINE];
    const uint8_t *masks[B200_MAX_COMBINE];
};

__global__ void __launch_bounds__(256) k_set_combine(const __grid_constant__ CombineParams p, long long nrows, long long *out) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < nrows; i += (long long)gridDim.x * blockDim.x) {
        long long acc = 0;
        bool missing = false;
        for (int k = 0; k < p.nkeys; k++) {
            long long o;
            if (p.masks[k] && p.masks[k][i]) {
                o = p.null_ord[k];
            } else {
                const uint64_t raw = ldcs1_raw(p.keys[k], p.isz[k], i);
                o = raw_isnan(p.dtype[k], raw) ? p.nan_ord[k] : set_ordinal(p.probe[k], p.mask[k], p.sentinel[k], key_canon(p.dtype[k], raw));
            }
            missing |= o < 0;
            acc += o * p.mult[k];
        }
        out[i] = missing ? -1 : acc;
    }
}

// update(..., return_values=True): per row the shard-local ordinal and the shard (src/hash_primitives.hpp:139-176)
__global__ void __launch_bounds__(256) k_set_values(const SetSlot *probe, unsigned long long mask, long long sentinel_ordinal, long long nan_ordinal,
                                                    long long null_ordinal, int dtype, int isz, int nmaps, const long long *offsets, const void *keys,
                                                    const uint8_t *masks, long long nrows, long long *out_values, short *out_map) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < nrows; i += (long long)gridDim.x * blockDim.x) {
        uint64_t raw = ldcs1_raw(keys, isz, i);
        if (masks && masks[i]) {
            out_values[i] = null_ordinal;
            out_map[i] = 0;
        } else if (raw_isnan(dtype, raw)) {
            out_values[i] = nan_ordinal;
            out_map[i] = 0;
        } else {
            unsigned long long canon = key_canon(dtype, raw);
            int shard = (int)(key_hash(dtype, canon) % (unsigned long long)nmaps);
            long long g = set_ordinal(probe, mask, sentinel_ordinal, canon);
            out_values[i] = g - offsets[shard];
            out_map[i] = (short)shard;
        }
    }
}

inline int nblocks(unsigned long long n, int threads = 256) {
    unsigned long long b = (n + threads - 1) / threads;
    return (int)(b < kSmCount * 8ull ? (b ? b : 1) : kSmCount * 8ull);
}

// Tables, sort scratch and probe tables come from the context's block cache (DevBuf, common.cuh): a groupby builds and drops a set
// per key column and pass, and cudaMalloc / cudaFree synchronise the device and contend with the feeder threads' copies.
//
// The table and its parallel arrays (counts, slot log, string log), built at `cap` slots and rehashed from the current ones.  The old
// blocks go back to the cache once `st` has drained: every launch that touches a set's table, pool or logs runs under s->mu and its
// stream is synchronised before the lock is released, so no other stream can still touch them.
int set_grow(b200_set *s, cudaStream_t st, uint64_t new_cap = 0) {
    const uint64_t old_cap = s->cap, cap = new_cap > old_cap ? new_cap : old_cap * 4;
    DevBuf<SetSlot> table;
    DevBuf<unsigned long long> counts;
    DevBuf<unsigned> slot_log;
    DevBuf<StrLog> log;
    B200_CHECK(table.alloc(s->ctx, cap * sizeof(SetSlot), "ordered_set table", st));
    if (s->counting) {
        B200_CHECK(counts.alloc(s->ctx, cap * sizeof(unsigned long long), "ordered_set table", st));
        B200_CUDA(cudaMemsetAsync(counts, 0, cap * sizeof(unsigned long long), st));
    }
    if (s->strings) { // one record per key at most: the log is as long as the table
        B200_CHECK(slot_log.alloc(s->ctx, cap * sizeof(unsigned), "ordered_set table", st));
        B200_CHECK(log.alloc(s->ctx, cap * sizeof(StrLog), "ordered_set table", st));
    }
    k_set_init<<<nblocks(cap), 256, 0, st>>>(table, cap);
    B200_CUDA(cudaGetLastError());
    if (old_cap) {
        k_set_rehash<<<nblocks(old_cap), 256, 0, st>>>(s->table, old_cap, table, cap - 1, s->counts, counts, s->slot_log, slot_log);
        B200_CUDA(cudaGetLastError());
        if (s->strings)
            B200_CUDA(cudaMemcpyAsync(log, s->log, old_cap * sizeof(StrLog), cudaMemcpyDeviceToDevice, st));
        B200_CUDA(cudaStreamSynchronize(st));
    }
    table.unbind(), counts.unbind(), slot_log.unbind(), log.unbind();
    s->table = std::move(table), s->counts = std::move(counts), s->slot_log = std::move(slot_log), s->log = std::move(log);
    s->cap = cap;
    return B200_OK;
}

// room for the worst case of a call that inserts `nrows` rows: every row a new key, capped at 2^22 slots = 64 MB.  One growth step
// up front avoids the grow-and-redo cascade 4K -> 16K -> ... (five allocations and rehashes) on big inputs; growth on demand covers
// the rest
int set_reserve(b200_set *s, cudaStream_t st, int64_t nrows) {
    const uint64_t known = s->dirty ? 0 : (uint64_t)s->n_keys; // exact only right after a finalisation
    const uint64_t target = std::min<uint64_t>((known + (uint64_t)nrows) * 2, 1ull << 22);
    uint64_t want = s->cap;
    while (want < target)
        want <<= 1;
    return want > s->cap ? set_grow(s, st, want) : B200_OK;
}

int read_ctr(b200_set *s, cudaStream_t st, unsigned long long *h) {
    B200_CUDA(cudaMemcpyAsync(h, s->d_ctr, sizeof(unsigned long long) * CTR_N, cudaMemcpyDeviceToHost, st));
    B200_CUDA(cudaStreamSynchronize(st));
    return B200_OK;
}

// Runs one insert pass until the table holds it: pass(redo) enqueues the pass on `st` and returns its launch status.  When a
// thread's insert overflowed, the table grows four-fold and the pass runs again with redo = 2: key inserts are idempotent (CAS claim
// + atomicMin of the tag), while a pass's NaN / null counting is not and is skipped on a redo.  The loop ends when the pass fits or
// when set_grow cannot allocate the larger table.
template <typename Pass>
int set_insert_pass(b200_set *s, cudaStream_t st, Pass &&pass) {
    unsigned long long h[CTR_N];
    for (int redo = 0;; redo = 2) {
        B200_CHECK(pass(redo));
        B200_CHECK(read_ctr(s, st, h));
        if (!h[CTR_OVERFLOW])
            return B200_OK;
        unsigned long long zero = 0;
        B200_CUDA(cudaMemcpyAsync(s->d_ctr + CTR_OVERFLOW, &zero, sizeof zero, cudaMemcpyHostToDevice, st));
        B200_CHECK(set_grow(s, st));
    }
}

// the shard of a key is key_hash(dtype, key) % nmaps; a string set's table key already IS the reference's string hash, and the
// 16-bit integer types use the identity there too (src/hash.hpp:50-152)
static int shard_dtype(const b200_set *s) { return s->strings ? B200_U16 : s->dtype; }

// lazily materialise ordinals; caller holds s->mu.  Everything stays on the device: compact -> radix sort by first-occurrence tag
// (only the bytes that vary) -> stable radix pass(es) by shard -> position == global ordinal (src/hash.hpp:337-353) -> keys in
// ordinal order + {key, ordinal} probe table.  The host learns nmaps shard starts and three special ordinals; key_array() copies
// the ordered keys on demand (ensure_host_keys).
int set_finalize(b200_set *s) {
    if (!s->dirty)
        return B200_OK;
    B200_CUDA(cudaSetDevice(s->ctx->device));
    cudaStream_t st = s->ctx->slots[0]->stream;
    unsigned long long h[CTR_N];
    unsigned long long zero = 0;
    // the insert kernel keeps no fill counter (see kMaxProbe in settable.cuh): count the occupied slots first, then compact them
    B200_CUDA(cudaMemcpyAsync(s->d_ctr + CTR_CURSOR, &zero, sizeof zero, cudaMemcpyHostToDevice, st));
    k_set_compact<<<nblocks(s->cap), 256, 0, st>>>(s->table, s->cap, s->d_ctr, nullptr, nullptr, nullptr, shard_dtype(s), s->nmaps);
    B200_CHECK(read_ctr(s, st, h));
    h[CTR_COUNT] = h[CTR_CURSOR];
    B200_CUDA(cudaMemcpyAsync(s->d_ctr + CTR_CURSOR, &zero, sizeof zero, cudaMemcpyHostToDevice, st));
    const bool has_nan = h[CTR_NAN_COUNT] > 0, has_null = h[CTR_NULL_COUNT] > 0, has_sent = h[CTR_SENTINEL_TAG] != 0xFFFFFFFFFFFFFFFFULL;
    const unsigned long long n_table = h[CTR_COUNT];
    const unsigned long long E = n_table + has_nan + has_null + has_sent;
    if (E >= (1ull << 32)) {
        set_error("ordered_set: more than 2^32 distinct keys are not supported");
        return B200_ERR_UNSUPPORTED;
    }
    // one allocation: ckey | tag A | val A | tag B | val B | radix histograms | shard starts | special ordinals
    const size_t en = (size_t)(E ? E : 1);
    const size_t off_hist = 5 * en * 8, off_first = off_hist + align_up(radix_scratch_bytes(E), 256), off_spec = off_first + align_up((size_t)s->nmaps * 8, 256);
    DevBuf<char> work;
    B200_CHECK(work.alloc(s->ctx, off_spec + 256, "set_finalize", st));
    unsigned long long *ckey = reinterpret_cast<unsigned long long *>(work.get()), *tagA = ckey + en, *valA = tagA + en, *tagB = valA + en, *valB = tagB + en;
    unsigned *hist = reinterpret_cast<unsigned *>(work + off_hist);
    long long *d_first = reinterpret_cast<long long *>(work + off_first), *d_spec = reinterpret_cast<long long *>(work + off_spec);
    if (n_table)
        k_set_compact<<<nblocks(s->cap), 256, 0, st>>>(s->table, s->cap, s->d_ctr, ckey, tagA, valA, shard_dtype(s), s->nmaps);
    // the special entries ride along behind the table's keys: [key == SET_EMPTY pattern] [NaN] [null]; NaN / null live in shard 0
    unsigned long long xk[3], xt[3], xv[3];
    int ne = 0, sent_idx = -1, nan_idx = -1, null_idx = -1;
    // NaN / null sort behind every row of the call that first saw them (row part kTagLowMask - 1 / kTagLowMask, see
    // set_insert_device): keep that order but with a small row part, so that the sort can skip the empty high bytes
    auto special_tag = [&](unsigned long long tag) {
        const unsigned long long low = tag & kTagLowMask;
        if (low < kTagLowMask - 1)
            return tag; // from_keys: the tag is the row itself
        return (tag & ~kTagLowMask) | ((unsigned long long)s->max_call_rows + (low - (kTagLowMask - 1)));
    };
    if (has_sent) {
        sent_idx = ne;
        xk[ne] = SET_EMPTY, xt[ne] = h[CTR_SENTINEL_TAG], xv[ne] = ((key_hash(shard_dtype(s), SET_EMPTY) % (unsigned long long)s->nmaps) << 32) | (n_table + ne);
        ne++;
    }
    if (has_nan) {
        nan_idx = ne;
        xk[ne] = 0, xt[ne] = special_tag(h[CTR_NAN_TAG]), xv[ne] = n_table + ne;
        ne++;
    }
    if (has_null) {
        null_idx = ne;
        xk[ne] = 0, xt[ne] = special_tag(h[CTR_NULL_TAG]), xv[ne] = n_table + ne;
        ne++;
    }
    if (ne) {
        B200_CUDA(cudaMemcpyAsync(ckey + n_table, xk, 8 * ne, cudaMemcpyHostToDevice, st));
        B200_CUDA(cudaMemcpyAsync(tagA + n_table, xt, 8 * ne, cudaMemcpyHostToDevice, st));
        B200_CUDA(cudaMemcpyAsync(valA + n_table, xv, 8 * ne, cudaMemcpyHostToDevice, st));
    }
    unsigned long long *tin = tagA, *vin = valA, *tout = tagB, *vout = valB;
    // tags are (call sequence << 40 | row): only the bytes that can differ are sorted on, then (stable) the shard bytes of the
    // payload.  The NaN / null tags were moved just behind the largest row (see `special_tag`), so the row part stays below max_low.
    const unsigned long long max_low = (unsigned long long)s->max_call_rows + 2, max_seq = (unsigned long long)(s->seq > 0 ? s->seq - 1 : 0);
    const unsigned tag_bytes = (radix_bytes_through(max_low) & 0x1fu) | (radix_bytes_through(max_seq) & 0x7u) << 5;
    B200_CHECK(radix_sort(E, tag_bytes, radix_bytes_through((unsigned)(s->nmaps - 1)) & 0x3u, tin, vin, tout, vout, hist, st));
    // probe table + keys in ordinal order
    // (every reader of the previous probe table / key array holds s->mu or ran on a stream that has been synchronised since)
    B200_CHECK(b200_ctx_sync(s->ctx, -1));
    s->probe.reset();
    s->d_keys_ord.reset();
    uint64_t pc = 16;
    while (pc < 2 * (n_table + 1))
        pc <<= 1;
    B200_CHECK(s->probe.alloc(s->ctx, pc * sizeof(SetSlot), "set_finalize"));
    s->probe_cap = pc;
    B200_CHECK(s->d_keys_ord.alloc(s->ctx, en * 8, "set_finalize"));
    k_set_init<<<nblocks(pc), 256, 0, st>>>(s->probe, pc);
    B200_CUDA(cudaMemsetAsync(d_first, 0xff, (size_t)s->nmaps * 8, st)); // -1: shard without keys
    B200_CUDA(cudaMemsetAsync(d_spec, 0xff, 3 * 8, st));
    if (E)
        k_set_finish<<<nblocks(E), 256, 0, st>>>(vin, ckey, E, n_table, sent_idx, nan_idx, null_idx, s->probe, pc - 1, s->d_keys_ord, d_first, d_spec);
    B200_CUDA(cudaGetLastError());
    std::vector<long long> first(s->nmaps);
    long long spec[3];
    B200_CUDA(cudaMemcpyAsync(first.data(), d_first, (size_t)s->nmaps * 8, cudaMemcpyDeviceToHost, st));
    B200_CUDA(cudaMemcpyAsync(spec, d_spec, sizeof spec, cudaMemcpyDeviceToHost, st));
    B200_CUDA(cudaStreamSynchronize(st));

    s->n_entries = E;
    s->h_keys.clear();
    s->h_keys_valid = false;
    s->nan_count = (int64_t)h[CTR_NAN_COUNT];
    s->null_count = (int64_t)h[CTR_NULL_COUNT];
    s->nan_value = has_nan ? spec[1] : 0x7fffffff;
    s->null_value = has_null ? spec[2] : 0x7fffffff;
    s->sentinel_ordinal = has_sent ? spec[0] : -1;
    s->n_keys = (int64_t)(n_table + has_sent);
    // offsets[m] = where shard m starts; an empty shard starts where the next non-empty one does (src/hash.hpp:337-353)
    s->h_offsets.assign(s->nmaps, 0);
    long long next = (long long)E;
    for (int m = s->nmaps - 1; m >= 0; m--) {
        if (first[m] >= 0)
            next = first[m];
        s->h_offsets[m] = next;
    }
    if (!s->d_offsets)
        B200_CHECK(s->d_offsets.alloc(s->ctx, sizeof(long long) * s->nmaps, "set_finalize"));
    B200_CUDA(cudaMemcpyAsync(s->d_offsets, s->h_offsets.data(), sizeof(long long) * s->nmaps, cudaMemcpyHostToDevice, st));
    B200_CUDA(cudaStreamSynchronize(st));
    s->dirty = false;
    return B200_OK;
}

// key_array() / merge need the ordered keys on the host: one download per finalisation, on demand; caller holds s->mu
int ensure_host_keys(b200_set *s) {
    B200_CHECK(set_finalize(s));
    if (s->h_keys_valid)
        return B200_OK;
    s->h_keys.assign(s->n_entries, 0);
    if (s->n_entries) {
        cudaStream_t st = s->ctx->slots[0]->stream;
        B200_CUDA(cudaMemcpyAsync(s->h_keys.data(), s->d_keys_ord, s->n_entries * 8, cudaMemcpyDeviceToHost, st));
        B200_CUDA(cudaStreamSynchronize(st));
    }
    s->h_keys_valid = true;
    return B200_OK;
}

int64_t set_count_locked(b200_set *s) { return s->n_keys + (s->nan_count > 0) + (s->null_count > 0); }

// insert rows [0, nrows) of device arrays; caller holds s->mu
int set_insert_device(b200_set *s, cudaStream_t st, const void *d_keys, const uint8_t *d_masks, int64_t nrows, bool use_offsets, bool from_keys,
                      int64_t from_keys_null_index, int64_t start_index = 0) {
    int skip_keys = 0;
    if (s->limit >= 0) { // hash_primitives.hpp:237-249: a full set skips the whole flush of this call
        B200_CHECK(set_finalize(s));
        if (set_count_locked(s) >= s->limit)
            skip_keys = 1;
    }
    const unsigned long long tag_base = s->indexing ? index_bias(start_index) : from_keys ? 0ull : ((unsigned long long)s->seq << 40);
    s->seq++;
    s->max_call_rows = std::max<int64_t>(s->max_call_rows, nrows);
    const unsigned long long first_low = kTagLowMask - 1, second_low = kTagLowMask;
    const unsigned long long null_low = use_offsets ? first_low : second_low;
    const unsigned long long nan_low = use_offsets ? second_low : first_low;
    const int isz = dtype_size(s->dtype);
    const int64_t sub = 1ll << 26;
    B200_CHECK(set_reserve(s, st, nrows));
    for (int64_t row0 = 0; row0 < nrows; row0 += sub) {
        const int64_t n = std::min<int64_t>(sub, nrows - row0);
        B200_CHECK(set_insert_pass(s, st, [&](int redo) -> int {
            k_set_insert<<<nblocks((unsigned long long)n), 256, 0, st>>>(s->table, s->cap - 1, s->d_ctr, s->dtype, isz, d_keys, d_masks, row0, n, tag_base,
                                                                         skip_keys | redo, from_keys_null_index, from_keys ? 1 : 0, nan_low, null_low);
            B200_CUDA(cudaGetLastError());
            return B200_OK;
        }));
    }
    if (s->counting && !s->hold_count_pass && !skip_keys && nrows) {
        k_set_count<<<nblocks((unsigned long long)nrows), 256, 0, st>>>(s->table, s->cap - 1, s->counts, s->d_ctr, s->dtype, isz, d_keys, d_masks, nullptr, nrows);
        B200_CUDA(cudaGetLastError());
        // finalisation, counts() and growth run on slot 0's stream: the counts must be complete before any of them looks
        B200_CUDA(cudaStreamSynchronize(st));
    }
    B200_CUDA(cudaGetLastError());
    s->dirty = true;
    return B200_OK;
}

// ---- index_hash<T> (src/hash_primitives.hpp:731-1040) ----------------------------------------------------------------------------

// the row log of one update: every non-NaN, non-null row appends {canonical key, global row} (one cursor bump per warp); NaN / null
// rows raise the largest biased NaN / null row.  Runs once per update, after its insert pass succeeded.
__global__ void __launch_bounds__(256) k_index_log(unsigned long long *ctr, int dtype, int isz, const void *keys, const uint8_t *masks, long long nrows,
                                                   long long start, unsigned long long *log_key, long long *log_row) {
    const unsigned lane = threadIdx.x & 31;
    unsigned long long nan_max = 0, null_max = 0;
    for (long long base = (long long)blockIdx.x * blockDim.x; base < nrows; base += (long long)gridDim.x * blockDim.x) {
        const long long i = base + threadIdx.x; // every lane of a warp runs the same iterations: the ballot below sees all 32
        bool keep = false;
        unsigned long long canon = 0;
        if (i < nrows) {
            const uint64_t raw = ldcs1_raw(keys, isz, i);
            if (masks && masks[i])
                null_max = max(null_max, index_bias(start + i));
            else if (raw_isnan(dtype, raw))
                nan_max = max(nan_max, index_bias(start + i));
            else
                keep = true, canon = key_canon(dtype, raw);
        }
        const unsigned m = __ballot_sync(0xffffffffu, keep);
        unsigned long long pos = 0;
        if (lane == 0 && m)
            pos = atomicAdd(ctr + CTR_LOG, (unsigned long long)__popc(m));
        pos = __shfl_sync(0xffffffffu, pos, 0) + __popc(m & ((1u << lane) - 1u));
        if (keep) {
            log_key[pos] = canon;
            log_row[pos] = start + i;
        }
    }
    if (nan_max)
        atomicMax(ctr + CTR_NAN_MAX, nan_max);
    if (null_max)
        atomicMax(ctr + CTR_NULL_MAX, null_max);
}

// the slot of a key (~0ull: absent); the key whose pattern is SET_EMPTY lives outside the table, at slot `cap`
__device__ __forceinline__ unsigned long long index_slot(const SetSlot *table, unsigned long long mask, unsigned long long canon) {
    return canon == SET_EMPTY ? mask + 1 : set_slot(table, mask, canon);
}

// radix input: sort key = row - row_min, payload = slot << 32 (the shard-pass layout of radix.cuh: from_val digits)
__global__ void k_index_sort_keys(const SetSlot *table, unsigned long long mask, const unsigned long long *log_key, const long long *log_row,
                                  unsigned long long n, long long row_min, unsigned long long *key, unsigned long long *val) {
    for (unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (unsigned long long)gridDim.x * blockDim.x) {
        key[i] = (unsigned long long)(log_row[i] - row_min);
        val[i] = index_slot(table, mask, log_key[i]) << 32;
    }
}

// sorted by (slot, row): rows back to global rows, and every slot's [begin, end)
__global__ void k_index_segments(const unsigned long long *key, const unsigned long long *val, unsigned long long n, long long row_min, long long *rows,
                                 uint2 *seg) {
    for (unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (unsigned long long)gridDim.x * blockDim.x) {
        const unsigned long long slot = val[i] >> 32;
        rows[i] = (long long)key[i] + row_min;
        if (i == 0 || (val[i - 1] >> 32) != slot)
            seg[slot].x = (unsigned)i;
        if (i == n - 1 || (val[i + 1] >> 32) != slot)
            seg[slot].y = (unsigned)(i + 1);
    }
}

// looked-up row of one key: NaN -> the NaN row, masked -> the null row (each -1 and "unknown" when absent), else the primary row
struct IndexSpecials {
    long long nan_row, null_row, sent_row; // -1: absent
    bool sent_present;
};
__device__ __forceinline__ IndexSpecials index_specials(const unsigned long long *ctr) {
    IndexSpecials x;
    x.nan_row = ctr[CTR_NAN_COUNT] ? index_unbias(ctr[CTR_NAN_MAX]) : -1;
    x.null_row = ctr[CTR_NULL_COUNT] ? index_unbias(ctr[CTR_NULL_MAX]) : -1;
    x.sent_present = ctr[CTR_SENTINEL_TAG] != ~0ull;
    x.sent_row = x.sent_present ? index_unbias(ctr[CTR_SENTINEL_TAG]) : -1;
    return x;
}

// index_hash::map_index_write / map_index_with_mask_write (src/hash_primitives.hpp:793-889): out_isz 1/2/4/8 truncates like the
// reference's assignment into an int8..int64 array
__global__ void __launch_bounds__(256) k_index_map(const SetSlot *table, unsigned long long mask, const unsigned long long *ctr, int dtype, int isz,
                                                   const void *keys, const uint8_t *masks, long long nrows, void *out, int out_isz, int *unknown) {
    const IndexSpecials sp = index_specials(ctr);
    bool unk = false;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < nrows; i += (long long)gridDim.x * blockDim.x) {
        const uint64_t raw = ldcs1_raw(keys, isz, i);
        long long v;
        if (raw_isnan(dtype, raw)) {
            v = sp.nan_row;
            unk |= v == -1;
        } else if (masks && masks[i]) {
            v = sp.null_row;
            unk |= v == -1;
        } else {
            const unsigned long long canon = key_canon(dtype, raw);
            bool found;
            if (canon == SET_EMPTY) {
                found = sp.sent_present;
                v = sp.sent_row;
            } else {
                unsigned long long first;
                found = set_lookup(table, mask, canon, &first);
                v = found ? index_unbias(first) : -1;
            }
            unk |= !found;
        }
        store1_raw(out, out_isz, i, (uint64_t)v);
    }
    if (unk)
        *unknown = 1;
}

// the overflow range of a left row's key: [begin + 1, end) of its slot (the primary row is excluded); NaN and masked rows have none
__device__ __forceinline__ uint2 index_overflow(const SetSlot *table, unsigned long long mask, const uint2 *seg, int dtype, int isz, const void *keys,
                                                const uint8_t *masks, long long i) {
    const uint64_t raw = ldcs1_raw(keys, isz, i);
    if ((masks && masks[i]) || raw_isnan(dtype, raw))
        return make_uint2(0, 0);
    const unsigned long long slot = index_slot(table, mask, key_canon(dtype, raw));
    if (slot == ~0ull)
        return make_uint2(0, 0);
    const uint2 r = seg[slot];
    return r.y > r.x + 1 ? make_uint2(r.x + 1, r.y) : make_uint2(0, 0);
}

// index_hash::map_index_duplicates (src/hash_primitives.hpp:939-985): pass 1 counts every left row's extra matches (cnt[nrows] = 0,
// so the exclusive scan leaves the total there) and notes where its range starts in the sorted rows; pass 2 writes the pairs
// (start + i, overflow row), grouped by left row in left-row order
__global__ void __launch_bounds__(256) k_index_dup_count(const SetSlot *table, unsigned long long mask, const uint2 *seg, int dtype, int isz, const void *keys,
                                                         const uint8_t *masks, long long nrows, long long *cnt, unsigned *begin) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i <= nrows; i += (long long)gridDim.x * blockDim.x) {
        if (i == nrows) {
            cnt[i] = 0;
            continue;
        }
        const uint2 r = index_overflow(table, mask, seg, dtype, isz, keys, masks, i);
        cnt[i] = (long long)(r.y - r.x);
        begin[i] = r.x;
    }
}

// one thread per OUTPUT pair, not per left row: a key with millions of rows would otherwise leave one thread writing them all while
// the grid idles.  The pair's left row is the last i with off[i] <= o (rows without pairs have off[i] == off[i + 1]).
__global__ void __launch_bounds__(256) k_index_dup_write(const long long *rows, const long long *off, const unsigned *begin, long long nrows, long long total,
                                                         long long start, long long *left, long long *right) {
    for (long long o = (long long)blockIdx.x * blockDim.x + threadIdx.x; o < total; o += (long long)gridDim.x * blockDim.x) {
        long long lo = 0, hi = nrows; // invariant: off[lo] <= o < off[hi]
        while (hi - lo > 1) {
            const long long mid = lo + ((hi - lo) >> 1);
            if (__ldg(off + mid) <= o)
                lo = mid;
            else
                hi = mid;
        }
        left[o] = start + lo;
        right[o] = rows[begin[lo] + (o - off[lo])];
    }
}

// merge: every key of the other table enters with its primary row (atomicMin keeps the smaller); on overflow the host grows the
// table and redoes the pass (idempotent)
__global__ void __launch_bounds__(256) k_index_merge_table(const SetSlot *other, unsigned long long other_cap, SetSlot *table, unsigned long long mask,
                                                           unsigned long long *ctr) {
    for (unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; i < other_cap; i += (unsigned long long)gridDim.x * blockDim.x) {
        const SetSlot s = other[i];
        if (s.key == SET_EMPTY)
            continue;
        if (!set_insert(table, mask, s.key, s.first)) {
            overflow_raise(ctr + CTR_OVERFLOW);
            return;
        }
    }
}

// merge: the other index's counters join this one's (its log was appended behind this one's)
__global__ void k_index_merge_ctr(unsigned long long *ctr, const unsigned long long *other) {
    atomicAdd(ctr + CTR_NAN_COUNT, other[CTR_NAN_COUNT]);
    atomicAdd(ctr + CTR_NULL_COUNT, other[CTR_NULL_COUNT]);
    atomicAdd(ctr + CTR_LOG, other[CTR_LOG]);
    atomicMin(ctr + CTR_SENTINEL_TAG, other[CTR_SENTINEL_TAG]);
    atomicMax(ctr + CTR_NAN_MAX, other[CTR_NAN_MAX]);
    atomicMax(ctr + CTR_NULL_MAX, other[CTR_NULL_MAX]);
}

// room for `need` log rows; caller holds s->mu
int index_log_reserve(b200_set *s, cudaStream_t st, uint64_t need) {
    if (need <= s->log_cap)
        return B200_OK;
    const uint64_t cap = std::max<uint64_t>({need, s->log_cap * 2, 1ull << 16});
    DevBuf<unsigned long long> key;
    DevBuf<long long> row;
    B200_CHECK(key.alloc(s->ctx, cap * 8, "index_hash row log", st));
    B200_CHECK(row.alloc(s->ctx, cap * 8, "index_hash row log", st));
    if (s->log_n) {
        B200_CUDA(cudaMemcpyAsync(key, s->log_key, s->log_n * 8, cudaMemcpyDeviceToDevice, st));
        B200_CUDA(cudaMemcpyAsync(row, s->log_row, s->log_n * 8, cudaMemcpyDeviceToDevice, st));
    }
    B200_CUDA(cudaStreamSynchronize(st));
    key.unbind(), row.unbind();
    s->log_key = std::move(key), s->log_row = std::move(row);
    s->log_cap = cap;
    return B200_OK;
}

// distinct keys (table + the SET_EMPTY pattern) and the counters, refreshed after a change; caller holds s->mu
int index_stats(b200_set *s, cudaStream_t st, unsigned long long *h) {
    if (s->dirty) {
        unsigned long long zero = 0;
        B200_CUDA(cudaMemcpyAsync(s->d_ctr + CTR_CURSOR, &zero, sizeof zero, cudaMemcpyHostToDevice, st));
        k_set_compact<<<nblocks(s->cap), 256, 0, st>>>(s->table, s->cap, s->d_ctr, nullptr, nullptr, nullptr, s->dtype, s->nmaps);
        B200_CUDA(cudaGetLastError());
    }
    B200_CHECK(read_ctr(s, st, h));
    if (s->dirty) {
        s->n_keys = (int64_t)(h[CTR_CURSOR] + (h[CTR_SENTINEL_TAG] != ~0ull));
        s->dirty = false;
    }
    s->nan_count = (int64_t)h[CTR_NAN_COUNT];
    s->null_count = (int64_t)h[CTR_NULL_COUNT];
    return B200_OK;
}

// the log sorted by (slot, row) into per-slot ranges, after a change; caller holds s->mu
int index_sort(b200_set *s, cudaStream_t st) {
    if (s->idx_sorted)
        return B200_OK;
    const unsigned long long E = s->log_n, nslots = s->cap + 1;
    B200_CHECK(s->idx_seg.alloc(s->ctx, nslots * sizeof(uint2), "index_hash ranges"));
    B200_CUDA(cudaMemsetAsync(s->idx_seg, 0, nslots * sizeof(uint2), st));
    B200_CHECK(s->idx_rows.alloc(s->ctx, (E ? E : 1) * 8, "index_hash ranges"));
    if (E) {
        const size_t off_hist = 4 * E * 8;
        DevBuf<char> work;
        B200_CHECK(work.alloc(s->ctx, off_hist + radix_scratch_bytes(E), "index_hash sort", st));
        unsigned long long *tin = reinterpret_cast<unsigned long long *>(work.get()), *vin = tin + E, *tout = vin + E, *vout = tout + E;
        unsigned *hist = reinterpret_cast<unsigned *>(work + off_hist);
        k_index_sort_keys<<<nblocks(E), 256, 0, st>>>(s->table, s->cap - 1, s->log_key, s->log_row, E, s->row_min, tin, vin);
        B200_CUDA(cudaGetLastError());
        // LSD: the row bytes that vary, then (stable) the slot bytes
        const unsigned long long row_span = (unsigned long long)(s->row_max - s->row_min);
        B200_CHECK(radix_sort(E, radix_bytes_through(row_span), radix_bytes_through(s->cap) & 0xfu, tin, vin, tout, vout, hist, st));
        k_index_segments<<<nblocks(E), 256, 0, st>>>(tin, vin, E, s->row_min, s->idx_rows, s->idx_seg);
        B200_CUDA(cudaGetLastError());
        B200_CUDA(cudaStreamSynchronize(st));
    }
    s->idx_sorted = true;
    return B200_OK;
}

// b200_set_update of an index: the insert pass, then the row log; the frame's inputs are staged
int index_update(b200_set *s, CallFrame &call, const void *d_keys, const uint8_t *d_masks, int64_t nrows, int64_t start_index) {
    if (s->log_n + (uint64_t)nrows >= (1ull << 32)) {
        set_error("b200_index_update: an index_hash holds at most 2^32 rows");
        return B200_ERR_UNSUPPORTED;
    }
    if (!nrows)
        return B200_OK;
    cudaStream_t st = call.st;
    B200_CHECK(index_log_reserve(s, st, s->log_n + (uint64_t)nrows));
    B200_CHECK(set_insert_device(s, st, d_keys, d_masks, nrows, true, false, -1, start_index));
    k_index_log<<<nblocks((unsigned long long)nrows), 256, 0, st>>>(s->d_ctr, s->dtype, dtype_size(s->dtype), d_keys, d_masks, nrows, start_index, s->log_key,
                                                                    s->log_row);
    B200_CUDA(cudaGetLastError());
    unsigned long long h[CTR_N];
    B200_CHECK(read_ctr(s, st, h));
    s->log_n = h[CTR_LOG];
    s->row_min = std::min<int64_t>(s->row_min, start_index);
    s->row_max = std::max<int64_t>(s->row_max, start_index + nrows - 1);
    s->idx_sorted = false;
    return B200_OK;
}

// b200_set_merge of one other index, under the sequential rule: the union of both indexes' rows, primary = the smallest row, NaN /
// null row = the largest; caller holds both locks
int index_merge_one(b200_set *s, b200_set *o, cudaStream_t st) {
    if (s->log_n + o->log_n >= (1ull << 32)) {
        set_error("b200_index_merge: an index_hash holds at most 2^32 rows");
        return B200_ERR_UNSUPPORTED;
    }
    unsigned long long h[CTR_N], ho[CTR_N];
    B200_CHECK(index_stats(s, st, h));
    B200_CHECK(index_stats(o, st, ho));
    uint64_t want = s->cap;
    while (want < 2 * (uint64_t)(s->n_keys + o->n_keys))
        want <<= 1;
    if (want > s->cap)
        B200_CHECK(set_grow(s, st, want));
    B200_CHECK(set_insert_pass(s, st, [&](int) -> int {
        k_index_merge_table<<<nblocks(o->cap), 256, 0, st>>>(o->table, o->cap, s->table, s->cap - 1, s->d_ctr);
        B200_CUDA(cudaGetLastError());
        return B200_OK;
    }));
    B200_CHECK(index_log_reserve(s, st, s->log_n + o->log_n));
    if (o->log_n) {
        B200_CUDA(cudaMemcpyAsync(s->log_key + s->log_n, o->log_key, o->log_n * 8, cudaMemcpyDeviceToDevice, st));
        B200_CUDA(cudaMemcpyAsync(s->log_row + s->log_n, o->log_row, o->log_n * 8, cudaMemcpyDeviceToDevice, st));
    }
    k_index_merge_ctr<<<1, 1, 0, st>>>(s->d_ctr, o->d_ctr);
    B200_CUDA(cudaGetLastError());
    B200_CHECK(read_ctr(s, st, h));
    s->log_n = h[CTR_LOG];
    s->row_min = std::min(s->row_min, o->row_min);
    s->row_max = std::max(s->row_max, o->row_max);
    s->dirty = true;
    s->idx_sorted = false;
    return B200_OK;
}

// what set_map_common does for an index: map_index (out = rows of out_isz bytes, *unknown) or map_index_duplicates (out = the left
// rows, right = the right rows, written when *total <= capacity)
struct IndexLookup {
    const uint8_t *masks;
    int32_t *unknown;
    bool duplicates;
    int64_t start;
    int64_t *right;
    int64_t capacity;
    int64_t *total;
};

// caller holds s->mu; the frame's result rule applies (the entry point finishes it, waiting: the table may grow once the lock is
// released)
int index_lookup(b200_set *s, CallFrame &call, const void *keys, int64_t nrows, void *out, int out_isz, const IndexLookup &ix) {
    cudaStream_t st = call.st;
    const int isz = dtype_size(s->dtype);
    call.plan(keys, (size_t)nrows * isz);
    if (ix.masks)
        call.plan(ix.masks, (size_t)nrows);
    B200_CHECK(call.commit());
    const void *d_keys = call.dev(keys);
    const uint8_t *d_masks = ix.masks ? static_cast<const uint8_t *>(call.dev(ix.masks)) : nullptr;
    if (!ix.duplicates) {
        void *d_out;
        int *d_unknown;
        B200_CHECK(call.out(out, (size_t)nrows * out_isz, call.result_on_device(out), &d_out));
        B200_CHECK(call.out(ix.unknown, sizeof(int32_t), false, &d_unknown));
        B200_CUDA(cudaMemsetAsync(d_unknown, 0, sizeof(int32_t), st));
        k_index_map<<<nblocks((unsigned long long)nrows), 256, 0, st>>>(s->table, s->cap - 1, s->d_ctr, s->dtype, isz, d_keys, d_masks, nrows, d_out, out_isz,
                                                                       d_unknown);
        B200_CUDA(cudaGetLastError());
        return B200_OK;
    }
    B200_CHECK(index_sort(s, st));
    const unsigned long long n1 = (unsigned long long)nrows + 1;
    const unsigned long long n_off = n1 + scan_i64_sums(n1);
    DevBuf<long long> off;
    B200_CHECK(off.alloc(s->ctx, n_off * 8 + (size_t)nrows * 4, "b200_index_duplicates", st));
    unsigned *begin = reinterpret_cast<unsigned *>(off + n_off);
    k_index_dup_count<<<nblocks(n1), 256, 0, st>>>(s->table, s->cap - 1, s->idx_seg, s->dtype, isz, d_keys, d_masks, nrows, off, begin);
    B200_CUDA(cudaGetLastError());
    B200_CHECK(scan_i64(off, n1, off + n1, st));
    long long n_out = 0;
    B200_CUDA(cudaMemcpyAsync(&n_out, off + nrows, 8, cudaMemcpyDeviceToHost, st));
    B200_CUDA(cudaStreamSynchronize(st));
    *ix.total = n_out;
    if (n_out && n_out <= ix.capacity) {
        long long *d_left, *d_right;
        B200_CHECK(call.out(out, (size_t)n_out * 8, call.result_on_device(out), &d_left));
        B200_CHECK(call.out(ix.right, (size_t)n_out * 8, call.result_on_device(ix.right), &d_right));
        k_index_dup_write<<<nblocks((unsigned long long)n_out), 256, 0, st>>>(s->idx_rows, off, begin, nrows, n_out, ix.start, d_left, d_right);
        B200_CUDA(cudaGetLastError());
    }
    return B200_OK;
}

} // namespace

// used by the C-ABI layer for B200_BINNER_HASH
int set_fill_binner(b200_set *s, DevBinner &b) {
    std::lock_guard<std::mutex> g(s->mu);
    B200_CHECK(set_finalize(s));
    b.table = s->probe;
    b.table_mask = s->probe_cap - 1;
    b.nan_ordinal = s->nan_count > 0 ? s->nan_value : -1;
    b.null_ordinal = s->null_count > 0 ? s->null_value : -1;
    b.sentinel_ordinal = s->sentinel_ordinal;
    return B200_OK;
}

} // namespace b200

using namespace b200;

extern "C" {

// ordered_set, counter (`counting`) and ordered_set_string (`strings`): a failure leaves nothing behind and *out untouched
static int set_create(b200_ctx *ctx, int dtype, int nmaps, int64_t limit, bool counting, bool strings, b200_set **out) {
    if (!ctx || !out || dtype < 0 || dtype >= B200_NDTYPE || nmaps < 1 || nmaps > 32767) {
        set_error("b200_set_create: invalid argument");
        return B200_ERR_INVALID;
    }
    B200_CUDA(cudaSetDevice(ctx->device));
    std::unique_ptr<b200_set, int (*)(b200_set *)> s(new b200_set, b200_set_destroy);
    s->ctx = ctx;
    s->dtype = dtype;
    s->nmaps = nmaps;
    s->limit = limit;
    s->counting = counting;
    s->strings = strings;
    cudaStream_t st = ctx->slots[0]->stream;
    B200_CHECK(set_grow(s.get(), st, 1ull << 12));
    unsigned long long init[CTR_N] = {0, 0, 0, 0, ~0ull, ~0ull, ~0ull, 0, 0, 0};
    B200_CHECK(s->d_ctr.alloc(ctx, sizeof init, "b200_set_create"));
    B200_CUDA(cudaMemcpyAsync(s->d_ctr, init, sizeof init, cudaMemcpyHostToDevice, st));
    if (strings) {
        B200_CHECK(s->d_strctr.alloc(ctx, 16, "b200_strset_create"));
        B200_CUDA(cudaMemsetAsync(s->d_strctr, 0, 16, st));
    }
    B200_CUDA(cudaStreamSynchronize(st));
    *out = s.release();
    return B200_OK;
}

int b200_set_create(b200_ctx *ctx, int dtype, int nmaps, int64_t limit, b200_set **out) { return set_create(ctx, dtype, nmaps, limit, false, false, out); }

// counter_<T>(nmaps) (src/hash_primitives.cpp:36-43): an ordered set that also counts the occurrences of every key
int b200_counter_create(b200_ctx *ctx, int dtype, int nmaps, b200_set **out) { return set_create(ctx, dtype, nmaps, -1, true, false, out); }

// counter::counts (src/hash_primitives.hpp:387-413) in the ordinal order of key_array(); the NaN / null slots hold their counts
int b200_set_counts(b200_set *s, int64_t *out) {
    if (!s || !out || !s->counting) {
        set_error("b200_set_counts: not a counter");
        return B200_ERR_INVALID;
    }
    B200_CUDA(cudaSetDevice(s->ctx->device));
    std::lock_guard<std::mutex> g(s->mu);
    B200_CHECK(set_finalize(s));
    cudaStream_t st = s->ctx->slots[0]->stream;
    const size_t n = (size_t)s->n_entries;
    if (!n)
        return B200_OK;
    DevBuf<unsigned long long> d_out;
    B200_CHECK(d_out.alloc(s->ctx, n * 8, "b200_set_counts", st));
    B200_CUDA(cudaMemsetAsync(d_out, 0, n * 8, st));
    k_counts_gather<<<nblocks(s->cap), 256, 0, st>>>(s->table, s->cap, s->counts, s->probe, s->probe_cap - 1, d_out);
    B200_CUDA(cudaGetLastError());
    B200_CUDA(cudaMemcpyAsync(out, d_out, n * 8, cudaMemcpyDeviceToHost, st));
    unsigned long long h[CTR_N];
    B200_CHECK(read_ctr(s, st, h));
    if (s->nan_count > 0)
        out[s->nan_value] = s->nan_count;
    if (s->null_count > 0)
        out[s->null_value] = s->null_count;
    if (s->sentinel_ordinal >= 0)
        out[s->sentinel_ordinal] = (int64_t)h[CTR_SENTINEL_COUNT];
    return B200_OK;
}

int b200_set_destroy(b200_set *s) {
    if (!s)
        return B200_OK;
    cudaSetDevice(s->ctx->device);
    for (Slot *sl : s->ctx->slots) // the blocks go back to the cache: nothing in flight may still touch them
        cudaStreamSynchronize(sl->stream);
    delete s;
    return B200_OK;
}

int b200_set_update(b200_set *s, int slot, const void *keys, const uint8_t *masks, int64_t nrows, int64_t start_index, int return_values,
                    int64_t *out_values, int16_t *out_map_index, int memspace, uint32_t flags) {
    if (!s || nrows < 0 || (nrows && !keys)) {
        set_error("b200_set_update: invalid argument");
        return B200_ERR_INVALID;
    }
    if (s->limit >= 0 && return_values) {
        set_error("Cannot combine limit with return_inverse"); // hash_primitives.hpp:102-104
        return B200_ERR_STATE;
    }
    if (s->indexing && return_values) {
        set_error("b200_set_update: an index_hash returns no values");
        return B200_ERR_INVALID;
    }
    if (nrows >= (1ll << 40) - 2) {
        set_error("b200_set_update: more than 2^40 rows in one call");
        return B200_ERR_UNSUPPORTED;
    }
    CallFrame call(s->ctx, slot, memspace, flags, "b200_set_update");
    B200_CHECK(call.rc);
    std::lock_guard<std::mutex> g(s->mu);
    cudaStream_t st = call.st;
    const size_t isz = dtype_size(s->dtype);
    call.plan(keys, (size_t)nrows * isz);
    if (masks)
        call.plan(masks, (size_t)nrows);
    B200_CHECK(call.commit());
    const void *d_keys = call.dev(keys);
    const uint8_t *d_masks = masks ? static_cast<const uint8_t *>(call.dev(masks)) : nullptr;
    if (s->indexing) {
        B200_CHECK(index_update(s, call, d_keys, d_masks, nrows, start_index));
        return call.finish(true); // the table may grow once the lock is released
    }
    const bool use_offsets = return_values || start_index != -1;
    B200_CHECK(set_insert_device(s, st, d_keys, d_masks, nrows, use_offsets, false, -1));
    if (return_values && nrows) {
        B200_CHECK(set_finalize(s));
        long long *d_vals;
        short *d_map;
        B200_CHECK(call.out(out_values, sizeof(long long) * nrows, false, &d_vals));
        B200_CHECK(call.out(out_map_index, sizeof(short) * nrows, false, &d_map));
        k_set_values<<<nblocks((unsigned long long)nrows), 256, 0, st>>>(s->probe, s->probe_cap - 1, s->sentinel_ordinal, s->nan_value, s->null_value, s->dtype,
                                                                       (int)isz, s->nmaps, s->d_offsets, d_keys, d_masks, nrows, d_vals, d_map);
        B200_CUDA(cudaGetLastError());
    }
    return call.finish();
}

int b200_set_from_keys(b200_ctx *ctx, int dtype, const void *keys, int64_t nkeys, int64_t null_index, int64_t nan_count, int64_t null_count,
                       b200_set **out) {
    b200_set *s = nullptr;
    B200_CHECK(b200_set_create(ctx, dtype, 1, -1, &s));
    int rc = B200_OK;
    {
        CallFrame call(ctx, 0, B200_MEM_HOST, 0, "b200_set_from_keys");
        std::lock_guard<std::mutex> g(s->mu);
        call.plan(keys, (size_t)nkeys * dtype_size(dtype));
        rc = call.rc ? call.rc : call.commit();
        if (!rc && nkeys)
            rc = set_insert_device(s, call.st, call.dev(keys), nullptr, nkeys, true, true, null_index);
        if (!rc)
            rc = set_finalize(s);
        if (!rc) {
            // ordered_set::create validation (src/hash_primitives.hpp:504-530)
            const char *msg = nullptr;
            if (nan_count == 0 && s->nan_count != 0)
                msg = "NaN found in data, while claiming there should be none";
            else if (nan_count != 0 && s->nan_count == 0)
                msg = "no NaN found in data, while claiming there should be";
            else if (null_count == 0 && s->null_count != 0)
                msg = "null found in data, while claiming there should be none";
            else if (null_count != 0 && s->null_count == 0)
                msg = "no null found in data, while claiming there should be";
            else if (null_count != 0 && s->null_value != null_index)
                msg = "null_value does not match expected value";
            else if (set_count_locked(s) != nkeys)
                msg = "key array length does not match expected length (duplicate keys)";
            if (msg) {
                set_error("%s", msg);
                rc = B200_ERR_STATE;
            } else {
                s->nan_count = nan_count;
                s->null_count = null_count;
            }
        }
        if (!rc)
            rc = call.finish();
    }
    if (rc) {
        b200_set_destroy(s);
        return rc;
    }
    *out = s;
    return B200_OK;
}

// ordered_set::merge (src/hash_primitives.hpp:693-720).  The reference appends unseen keys in the other map's
// hopscotch iteration order (container-internal); here they are appended in the other set's ORDINAL order —
// a documented, deterministic deviation (merging distinct sets does not occur in the reference's own flow:
// TaskPartHashmapUniqueCreate.ideal_splits() == 1, vaex/cpu.py:362-364).
int b200_set_merge(b200_set *s, b200_set *const *others, int nothers) {
    if (!s) {
        set_error("b200_set_merge: null set");
        return B200_ERR_INVALID;
    }
    for (int i = 0; i < nothers; i++) {
        if (others[i]->indexing != s->indexing || (s->indexing && (others[i] == s || others[i]->ctx->device != s->ctx->device))) {
            set_error("b200_set_merge: invalid argument");
            return B200_ERR_INVALID;
        }
        if (others[i]->nmaps != s->nmaps || others[i]->dtype != s->dtype) {
            set_error("cannot merge with an unequal maps");
            return B200_ERR_STATE;
        }
    }
    B200_CUDA(cudaSetDevice(s->ctx->device));
    for (int i = 0; i < nothers; i++) {
        b200_set *o = others[i];
        if (s->indexing) {
            CallFrame call(s->ctx, 0, B200_MEM_HOST, 0, "b200_set_merge");
            B200_CHECK(call.rc);
            std::scoped_lock g(s->mu, o->mu);
            B200_CHECK(index_merge_one(s, o, call.st));
            B200_CHECK(call.finish(true));
            continue;
        }
        std::vector<uint64_t> keys, weights;
        std::vector<int64_t> o_counts;
        int64_t o_nan, o_null;
        if (s->counting && o->counting) { // counter::merge adds the other's counts (src/hash_primitives.hpp:414-432)
            o_counts.resize(std::max<int64_t>(b200_set_count(o), 1));
            B200_CHECK(b200_set_counts(o, o_counts.data()));
        }
        {
            std::lock_guard<std::mutex> g(o->mu);
            B200_CHECK(ensure_host_keys(o));
            keys.reserve(o->h_keys.size());
            for (size_t k = 0; k < o->h_keys.size(); k++)
                if ((int64_t)k != o->nan_value && (int64_t)k != o->null_value) {
                    keys.push_back(o->h_keys[k]);
                    if (!o_counts.empty())
                        weights.push_back((uint64_t)o_counts[k]);
                }
            o_nan = o->nan_count;
            o_null = o->null_count;
        }
        CallFrame call(s->ctx, 0, B200_MEM_HOST, 0, "b200_set_merge");
        B200_CHECK(call.rc);
        std::lock_guard<std::mutex> g(s->mu);
        // feed canonical patterns as a 64-bit column of a same-hash dtype: U64 for hashed types keeps hash64(canon)
        // identical; identity-hashed small ints also stay identical because key_hash(dtype, canon) == canon there.
        int saved = s->dtype;
        call.plan(keys.data(), keys.size() * 8);
        if (!weights.empty())
            call.plan(weights.data(), weights.size() * 8);
        B200_CHECK(call.commit());
        // canonical patterns re-enter through a raw 64-bit view; key_canon(U64) is the identity and the shard hash is
        // evaluated from s->dtype at finalize, so only the column width differs.
        s->dtype = B200_U64;
        s->hold_count_pass = true;
        int rc = keys.empty() ? B200_OK : set_insert_device(s, call.st, call.dev(keys.data()), nullptr, (int64_t)keys.size(), false, false, -1);
        s->hold_count_pass = false;
        if (!rc && s->counting && !weights.empty()) {
            k_set_count<<<nblocks(keys.size()), 256, 0, call.st>>>(s->table, s->cap - 1, s->counts, s->d_ctr, B200_U64, 8, call.dev(keys.data()), nullptr,
                                                                   static_cast<const unsigned long long *>(call.dev(weights.data())), (long long)keys.size());
            if (cudaGetLastError() != cudaSuccess)
                rc = B200_ERR_CUDA;
        }
        s->dtype = saved;
        B200_CHECK(rc);
        // nan/null: counts add up; a special first seen through a merge takes the next shard-0 ordinal
        unsigned long long h[CTR_N];
        B200_CHECK(read_ctr(s, call.st, h));
        const unsigned long long tag_base = (unsigned long long)(s->seq - (keys.empty() ? 0 : 1)) << 40;
        if (keys.empty())
            s->seq++;
        if (o_nan) {
            h[CTR_NAN_COUNT] += (unsigned long long)o_nan;
            if (h[CTR_NAN_TAG] == ~0ull)
                h[CTR_NAN_TAG] = tag_base | (kTagLowMask - 1);
        }
        if (o_null) {
            h[CTR_NULL_COUNT] += (unsigned long long)o_null;
            if (h[CTR_NULL_TAG] == ~0ull)
                h[CTR_NULL_TAG] = tag_base | kTagLowMask;
        }
        B200_CUDA(cudaMemcpyAsync(s->d_ctr, h, sizeof h, cudaMemcpyHostToDevice, call.st));
        B200_CHECK(call.finish(true));
        s->dirty = true;
    }
    return B200_OK;
}

#define SET_GETTER(name, expr)                                                                                                 \
    int64_t b200_set_##name(b200_set *s) {                                                                                     \
        if (!s)                                                                                                                \
            return -1;                                                                                                         \
        std::lock_guard<std::mutex> g(s->mu);                                                                                  \
        if (set_finalize(s))                                                                                                   \
            return -1;                                                                                                         \
        return (expr);                                                                                                         \
    }
SET_GETTER(count, set_count_locked(s))
SET_GETTER(nan_count, s->nan_count)
SET_GETTER(null_count, s->null_count)
SET_GETTER(nan_index, s->nan_value)
SET_GETTER(null_index, s->null_value)

int b200_set_nmaps(const b200_set *s) { return s ? s->nmaps : -1; }
int b200_set_dtype(const b200_set *s) { return s ? s->dtype : -1; }

int b200_set_offsets(b200_set *s, int64_t *out) {
    std::lock_guard<std::mutex> g(s->mu);
    B200_CHECK(set_finalize(s));
    for (int m = 0; m < s->nmaps; m++)
        out[m] = s->h_offsets[m];
    return B200_OK;
}

// hash_base::key_array (src/hash_primitives.hpp:302-328): NaN slot holds NaN, null slot holds (T)-1
int b200_set_key_array(b200_set *s, void *out) {
    std::lock_guard<std::mutex> g(s->mu);
    B200_CHECK(ensure_host_keys(s));
    const int isz = dtype_size(s->dtype);
    for (size_t i = 0; i < s->h_keys.size(); i++) {
        uint64_t bits = s->h_keys[i];
        if (s->nan_count > 0 && (int64_t)i == s->nan_value)
            bits = s->dtype == B200_F64 ? 0x7ff8000000000000ULL : 0x7fc00000u;
        if (s->null_count > 0 && (int64_t)i == s->null_value) {
            if (s->dtype == B200_F64)
                bits = 0xbff0000000000000ULL; // -1.0
            else if (s->dtype == B200_F32)
                bits = 0xbf800000u;
            else if (s->dtype == B200_BOOL)
                bits = 1;
            else
                bits = ~0ull;
        }
        store1_raw(out, isz, i, bits);
    }
    return B200_OK;
}

int b200_set_ordinal_dtype(b200_set *s) {
    int64_t size = b200_set_count(s);
    if (size < (1 << 7))
        return B200_I8;
    if (size < (1 << 15))
        return B200_I16;
    if (size < (1ll << 31))
        return B200_I32;
    return B200_I64;
}

// out: nrows results of out_isz bytes (0: isin's one byte) in host or device memory (CallFrame::result_on_device)
// ix: an index_hash lookup (index_lookup)
static int set_map_common(b200_set *s, int slot, const void *keys, int64_t nrows, void *out, int out_isz, int memspace, uint32_t flags, const char *name,
                          const IndexLookup *ix = nullptr) {
    if (!s || nrows < 0 || s->indexing != (ix != nullptr)) {
        set_error("%s: invalid argument", name);
        return B200_ERR_INVALID;
    }
    CallFrame call(s->ctx, slot, memspace, flags, name);
    B200_CHECK(call.rc);
    if (!nrows)
        return B200_OK;
    std::lock_guard<std::mutex> g(s->mu);
    if (ix) {
        B200_CHECK(index_lookup(s, call, keys, nrows, out, out_isz, *ix));
        return call.finish(true); // the table may grow once the lock is released
    }
    B200_CHECK(set_finalize(s));
    const size_t isz = dtype_size(s->dtype);
    const size_t osz = out_isz ? out_isz : 1;
    call.plan(keys, (size_t)nrows * isz);
    B200_CHECK(call.commit());
    void *d_out;
    B200_CHECK(call.out(out, nrows * osz, call.result_on_device(out), &d_out));
    k_set_map<<<nblocks((unsigned long long)nrows), 256, 0, call.st>>>(s->probe, s->probe_cap - 1, s->sentinel_ordinal, s->nan_count > 0 ? s->nan_value : -1,
                                                                     s->dtype, (int)isz, call.dev(keys), nrows, d_out, out_isz);
    B200_CUDA(cudaGetLastError());
    return call.finish();
}

int b200_set_map_ordinal(b200_set *s, int slot, const void *keys, int64_t nrows, void *out, int memspace, uint32_t flags) {
    int od = b200_set_ordinal_dtype(s);
    return set_map_common(s, slot, keys, nrows, out, dtype_size(od), memspace, flags, "b200_set_map_ordinal");
}

// ordered_set::isin (src/hash_primitives.hpp:539-565); NaN is "in" iff the set saw a NaN
int b200_set_isin(b200_set *s, int slot, const void *keys, int64_t nrows, uint8_t *out, int memspace, uint32_t flags) {
    return set_map_common(s, slot, keys, nrows, out, 0, memspace, flags, "b200_set_isin");
}

int b200_set_combine(b200_ctx *ctx, int slot, int nkeys, b200_set *const *sets, const void *const *keys, const uint8_t *const *masks,
                     const int64_t *multipliers, int64_t nrows, int64_t *out, int memspace, uint32_t flags) {
    if (nkeys < 1 || nkeys > B200_MAX_COMBINE || !sets || !keys || !multipliers || nrows < 0 || (nrows && !out)) {
        set_error("b200_set_combine: invalid argument");
        return B200_ERR_INVALID;
    }
    // flags are not read: a MIXED call waits for its stream whatever they say
    (void)flags;
    CallFrame call(ctx, slot, memspace, 0, "b200_set_combine");
    B200_CHECK(call.rc);
    if (!nrows)
        return B200_OK;
    CombineParams p;
    memset(&p, 0, sizeof p);
    p.nkeys = nkeys;
    for (int k = 0; k < nkeys; k++) {
        b200_set *s = sets[k];
        if (!s || s->ctx != ctx || !keys[k]) {
            set_error("b200_set_combine: key %d: set / column missing or from another context", k);
            return B200_ERR_INVALID;
        }
        std::lock_guard<std::mutex> g(s->mu);
        B200_CHECK(set_finalize(s));
        p.probe[k] = s->probe;
        p.mask[k] = s->probe_cap - 1;
        p.sentinel[k] = s->sentinel_ordinal;
        p.nan_ord[k] = s->nan_count > 0 ? s->nan_value : -1;
        p.null_ord[k] = s->null_count > 0 ? s->null_value : -1;
        p.mult[k] = multipliers[k];
        p.dtype[k] = s->dtype;
        p.isz[k] = (int)dtype_size(s->dtype);
    }
    for (int k = 0; k < nkeys; k++) {
        call.plan(keys[k], (size_t)nrows * p.isz[k]);
        if (masks && masks[k])
            call.plan(masks[k], (size_t)nrows);
    }
    B200_CHECK(call.commit());
    for (int k = 0; k < nkeys; k++) {
        p.keys[k] = call.dev(keys[k]);
        p.masks[k] = masks && masks[k] ? static_cast<const uint8_t *>(call.dev(masks[k])) : nullptr;
    }
    long long *d_out;
    B200_CHECK(call.out(out, nrows * 8, call.result_on_device(out), &d_out));
    k_set_combine<<<nblocks((unsigned long long)nrows), 256, 0, call.st>>>(p, nrows, d_out);
    B200_CUDA(cudaGetLastError());
    return call.finish();
}

// hash_base::bytes_used (src/hash_primitives.hpp:62-69): sum over maps of size * (sizeof(key) + sizeof(value))
size_t b200_set_bytes(b200_set *s) {
    std::lock_guard<std::mutex> g(s->mu);
    if (set_finalize(s))
        return 0;
    return (size_t)s->n_keys * (dtype_size(s->dtype) + 8);
}

// ---- index_hash<T> ----------------------------------------------------------------------------------------------------------------

// index_hash_<T>(nmaps) (src/hash_primitives.cpp:57-75)
int b200_index_create(b200_ctx *ctx, int dtype, int nmaps, b200_set **out) {
    b200_set *s = nullptr;
    B200_CHECK(set_create(ctx, dtype, nmaps, -1, false, false, &s));
    s->indexing = true;
    *out = s;
    return B200_OK;
}

static bool index_check(const b200_set *s, const char *name) {
    if (!s || !s->indexing || s->strings) {
        set_error("%s: not an index_hash", name);
        return false;
    }
    return true;
}

// hash_base::_update (src/hash_primitives.hpp:98-295) with index_hash::add_new / add_existing (:776-788), through b200_set_update
int b200_index_update(b200_set *s, int slot, const void *keys, const uint8_t *masks, int64_t nrows, int64_t start_index, int memspace, uint32_t flags) {
    if (!index_check(s, "b200_index_update"))
        return B200_ERR_INVALID;
    return b200_set_update(s, slot, keys, masks, nrows, start_index, 0, nullptr, nullptr, memspace, flags);
}

// index_hash::merge (src/hash_primitives.hpp:987-1031), through b200_set_merge
int b200_index_merge(b200_set *s, b200_set *const *others, int nothers) {
    if (!index_check(s, "b200_index_merge"))
        return B200_ERR_INVALID;
    return b200_set_merge(s, others, nothers);
}

// index_hash::map_index_write / map_index_with_mask_write (src/hash_primitives.hpp:793-889)
int b200_index_map(b200_set *s, int slot, const void *keys, const uint8_t *masks, int64_t nrows, void *out, int out_isz, int32_t *unknown, int memspace,
                   uint32_t flags) {
    if (!index_check(s, "b200_index_map"))
        return B200_ERR_INVALID;
    if (nrows < 0 || (nrows && (!keys || !out)) || !unknown || (out_isz != 1 && out_isz != 2 && out_isz != 4 && out_isz != 8)) {
        set_error("b200_index_map: invalid argument");
        return B200_ERR_INVALID;
    }
    *unknown = 0;
    IndexLookup ix{masks, unknown, false, 0, nullptr, 0, nullptr};
    return set_map_common(s, slot, keys, nrows, out, out_isz, memspace, flags, "b200_index_map", &ix);
}

// index_hash::map_index_duplicates (src/hash_primitives.hpp:939-985; the masked form :891-937 is not bound)
int b200_index_duplicates(b200_set *s, int slot, const void *keys, const uint8_t *masks, int64_t nrows, int64_t start_index, int64_t *left_out,
                          int64_t *right_out, int64_t capacity, int64_t *total, int memspace, uint32_t flags) {
    if (!index_check(s, "b200_index_duplicates"))
        return B200_ERR_INVALID;
    if (nrows < 0 || (nrows && !keys) || !total || capacity < 0 || (capacity && (!left_out || !right_out))) {
        set_error("b200_index_duplicates: invalid argument");
        return B200_ERR_INVALID;
    }
    *total = 0;
    IndexLookup ix{masks, nullptr, true, start_index, right_out, capacity, total};
    return set_map_common(s, slot, keys, nrows, left_out, 8, memspace, flags, "b200_index_duplicates", &ix);
}

// out[B200_INDEX_INFO_N]: the scalar getters (bind_common, src/hash_primitives.cpp:4-25, and index_hash :750-759, :1037)
int b200_index_info(b200_set *s, int64_t *out) {
    if (!index_check(s, "b200_index_info") || !out)
        return B200_ERR_INVALID;
    B200_CUDA(cudaSetDevice(s->ctx->device));
    std::lock_guard<std::mutex> g(s->mu);
    unsigned long long h[CTR_N];
    B200_CHECK(index_stats(s, s->ctx->slots[0]->stream, h));
    const int64_t specials = (s->nan_count > 0) + (s->null_count > 0);
    out[B200_INDEX_LENGTH] = (int64_t)s->log_n + specials;
    out[B200_INDEX_COUNT] = s->n_keys + specials;
    out[B200_INDEX_HAS_DUPLICATES] = (int64_t)s->log_n > s->n_keys;
    out[B200_INDEX_NAN_COUNT] = s->nan_count;
    out[B200_INDEX_NULL_COUNT] = s->null_count;
    out[B200_INDEX_NAN_ROW] = s->nan_count ? index_unbias(h[CTR_NAN_MAX]) : -1;
    out[B200_INDEX_NULL_ROW] = s->null_count ? index_unbias(h[CTR_NULL_MAX]) : -1;
    out[B200_INDEX_BYTES] = (int64_t)(s->cap * sizeof(SetSlot) + s->log_cap * 16);
    return B200_OK;
}

// hash_base::extract (src/hash_primitives.hpp:330-341): every distinct key (canonical pattern, host), its primary row and its shard;
// *n_out = their number, written to the arrays when it is at most `capacity`
int b200_index_extract(b200_set *s, uint64_t *keys_out, int64_t *rows_out, int16_t *shard_out, int64_t capacity, int64_t *n_out) {
    if (!index_check(s, "b200_index_extract") || !n_out || capacity < 0 || (capacity && (!keys_out || !rows_out || !shard_out)))
        return B200_ERR_INVALID;
    B200_CUDA(cudaSetDevice(s->ctx->device));
    std::lock_guard<std::mutex> g(s->mu);
    cudaStream_t st = s->ctx->slots[0]->stream;
    unsigned long long h[CTR_N];
    B200_CHECK(index_stats(s, st, h));
    const bool has_sent = h[CTR_SENTINEL_TAG] != ~0ull;
    const uint64_t n = (uint64_t)s->n_keys - has_sent;
    *n_out = s->n_keys;
    if ((uint64_t)s->n_keys > (uint64_t)capacity)
        return B200_OK;
    if (n) {
        DevBuf<unsigned long long> work;
        B200_CHECK(work.alloc(s->ctx, n * 24, "b200_index_extract", st));
        unsigned long long zero = 0;
        B200_CUDA(cudaMemcpyAsync(s->d_ctr + CTR_CURSOR, &zero, sizeof zero, cudaMemcpyHostToDevice, st));
        k_set_compact<<<nblocks(s->cap), 256, 0, st>>>(s->table, s->cap, s->d_ctr, work, work + n, work + 2 * n, s->dtype, s->nmaps);
        B200_CUDA(cudaGetLastError());
        std::vector<unsigned long long> v(n);
        B200_CUDA(cudaMemcpyAsync(keys_out, work, n * 8, cudaMemcpyDeviceToHost, st));
        B200_CUDA(cudaMemcpyAsync(rows_out, work + n, n * 8, cudaMemcpyDeviceToHost, st));
        B200_CUDA(cudaMemcpyAsync(v.data(), work + 2 * n, n * 8, cudaMemcpyDeviceToHost, st));
        B200_CUDA(cudaStreamSynchronize(st));
        for (uint64_t i = 0; i < n; i++) {
            rows_out[i] = index_unbias((unsigned long long)rows_out[i]);
            shard_out[i] = (int16_t)(v[i] >> 32);
        }
    }
    if (has_sent) {
        keys_out[n] = SET_EMPTY;
        rows_out[n] = index_unbias(h[CTR_SENTINEL_TAG]);
        shard_out[n] = (int16_t)(key_hash(s->dtype, SET_EMPTY) % (unsigned long long)s->nmaps);
    }
    return B200_OK;
}

uint64_t b200_hash64(uint64_t x) { return hash64(x); }

} // extern "C"

// =====================================================================================================================================
// string keys: ordered_set_string (SURVEY.md section 8f row 3; src/hash_string.hpp:56-180 update, ordered_set<> :437-560)
// =====================================================================================================================================
// Reference: shard = std::hash<string_view>(key) % nmaps (libstdc++'s 64-bit Murmur-2, seed 0xc70f6907), ordinal = insertion rank
// in the shard, nulls join shard 0 at the end of the update call that first sees one, key_array() = the shards' strings back to
// back.  Device design: the set's table is keyed by that 64-bit hash (so shards and ordinals come out of the SAME finalisation as
// the numeric sets); the thread that claims a slot appends the key's bytes to a pool and logs {hash, offset, length}; a second
// kernel re-probes every row and compares its bytes with the pooled key, so two strings that share a 64-bit hash are DETECTED
// (error, never a silent merge).  Strings arrive in the arrow large_string layout (int64 offsets + bytes) plus a byte mask.
namespace b200 {
namespace {

__device__ __forceinline__ unsigned long long murmur64(const unsigned char *p, unsigned long long len) {
    const unsigned long long mul = (0xc6a4a793ull << 32) + 0x5bd1e995ull;
    unsigned long long h = 0xc70f6907ull ^ (len * mul);
    const unsigned long long body = len & ~7ull;
    for (unsigned long long i = 0; i < body; i += 8) {
        unsigned long long d = 0;
#pragma unroll
        for (int b = 0; b < 8; b++) // unaligned little-endian load
            d |= (unsigned long long)p[i + b] << (8 * b);
        d *= mul;
        d ^= d >> 47;
        d *= mul;
        h ^= d;
        h *= mul;
    }
    if (len & 7) {
        unsigned long long d = 0;
        for (unsigned b = 0; b < (len & 7); b++)
            d |= (unsigned long long)p[body + b] << (8 * b);
        h ^= d;
        h *= mul;
    }
    h ^= h >> 47;
    h *= mul;
    h ^= h >> 47;
    return h;
}

__global__ void __launch_bounds__(256) k_str_insert(SetSlot *table, unsigned long long mask, unsigned long long *ctr, unsigned long long *strctr, StrLog *log,
                                                    char *pool, unsigned *slot_log, const long long *offsets, const unsigned char *bytes, const uint8_t *masks,
                                                    long long base, long long row0, long long nrows, unsigned long long tag_base, int skip,
                                                    unsigned long long null_low) {
    unsigned long long n_null = 0, t_null = ~0ull;
    bool dead = false;
    unsigned it = 0;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < nrows; i += (long long)gridDim.x * blockDim.x) {
        if (!dead && (it++ % kPollRows) == 0 && overflow_seen(ctr + CTR_OVERFLOW))
            dead = true;
        if (dead && (skip & 2))
            return;
        const long long row = row0 + i;
        if (masks && masks[row]) {
            if (!(skip & 2)) {
                n_null++;
                t_null = min(t_null, tag_base | null_low);
            }
            continue;
        }
        if (dead)
            continue;
        const long long b = offsets[row] - base, e = offsets[row + 1] - base;
        const unsigned long long len = (unsigned long long)(e - b);
        const unsigned long long h = murmur64(bytes + b, len);
        if (h == SET_EMPTY) { // one pattern in 2^64 is the table's "empty" marker
            ctr[CTR_STR_ERROR] = 1;
            continue;
        }
        const unsigned long long tag = tag_base | (unsigned long long)row;
        auto pool_key = [&](unsigned long long slot) { // this thread owns the new key: pool its bytes, log it
            const unsigned long long li = atomicAdd(strctr + 0, 1ull), po = atomicAdd(strctr + 1, len);
            for (unsigned long long c = 0; c < len; c++)
                pool[po + c] = (char)bytes[b + c];
            log[li].hash = h, log[li].off = po, log[li].len = (unsigned)len;
            slot_log[slot] = (unsigned)li;
        };
        if (!set_insert(table, mask, h, tag, pool_key)) {
            overflow_raise(ctr + CTR_OVERFLOW);
            dead = true;
        }
    }
    if (n_null) {
        atomicAdd(ctr + CTR_NULL_COUNT, n_null);
        atomicMin(ctr + CTR_NULL_TAG, t_null);
    }
}

__device__ __forceinline__ bool bytes_equal(const char *a, const unsigned char *b, unsigned long long len) {
    for (unsigned long long c = 0; c < len; c++)
        if ((unsigned char)a[c] != b[c])
            return false;
    return true;
}

// every row against the pooled bytes of the key its hash selected: a mismatch is a 64-bit hash collision
__global__ void __launch_bounds__(256) k_str_verify(const SetSlot *table, unsigned long long mask, unsigned long long *ctr, const StrLog *log, const char *pool,
                                                    const unsigned *slot_log, const long long *offsets, const unsigned char *bytes, const uint8_t *masks,
                                                    long long base, long long nrows) {
    for (long long row = (long long)blockIdx.x * blockDim.x + threadIdx.x; row < nrows; row += (long long)gridDim.x * blockDim.x) {
        if (masks && masks[row])
            continue;
        const long long b = offsets[row] - base;
        const unsigned long long len = (unsigned long long)(offsets[row + 1] - offsets[row]);
        const unsigned long long h = murmur64(bytes + b, len);
        if (h == SET_EMPTY)
            continue;
        const unsigned long long pos = set_slot(table, mask, h);
        if (pos == ~0ull)
            continue; // cannot happen after a successful insert pass
        const StrLog r = log[slot_log[pos]];
        if (r.len != len || !bytes_equal(pool + r.off, bytes + b, len))
            ctr[CTR_STR_ERROR] = 2;
    }
}

// finalized view: ordinal -> where the key's bytes are
__global__ void k_str_index(const StrLog *log, unsigned long long nlog, const SetSlot *probe, unsigned long long pmask, unsigned long long *str_off, unsigned *str_len) {
    for (unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; i < nlog; i += (unsigned long long)gridDim.x * blockDim.x) {
        const long long ord = set_ordinal(probe, pmask, -1, log[i].hash);
        if (ord >= 0) {
            str_off[ord] = log[i].off;
            str_len[ord] = log[i].len;
        }
    }
}

// ordered_set<>::map_ordinal for strings (+ the (local ordinal, shard) pair of update(return_values=True))
__global__ void __launch_bounds__(256) k_str_map(const SetSlot *probe, unsigned long long pmask, const unsigned long long *str_off, const unsigned *str_len,
                                                 const char *pool, long long null_ordinal, int nmaps, const long long *shard_offsets, const long long *offsets,
                                                 const unsigned char *bytes, const uint8_t *masks, long long base, long long nrows, long long *out,
                                                 short *out_map_index, int local_values) {
    for (long long row = (long long)blockIdx.x * blockDim.x + threadIdx.x; row < nrows; row += (long long)gridDim.x * blockDim.x) {
        long long ord;
        int shard = 0;
        if (masks && masks[row]) {
            ord = null_ordinal;
        } else {
            const long long b = offsets[row] - base;
            const unsigned long long len = (unsigned long long)(offsets[row + 1] - offsets[row]);
            const unsigned long long h = murmur64(bytes + b, len);
            shard = (int)(h % (unsigned long long)nmaps);
            ord = set_ordinal(probe, pmask, -1, h);
            if (ord >= 0 && (str_len[ord] != len || !bytes_equal(pool + str_off[ord], bytes + b, len)))
                ord = -1; // same hash, different string: not a member
        }
        if (local_values && ord >= 0)
            ord -= shard_offsets[shard];
        out[row] = ord;
        if (out_map_index)
            out_map_index[row] = (short)shard;
    }
}

__global__ void k_str_gather(const unsigned long long *str_off, const unsigned *str_len, const unsigned *out_off, const char *pool, unsigned long long n, char *out) {
    for (unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (unsigned long long)gridDim.x * blockDim.x) {
        const char *src = pool + str_off[i];
        char *dst = out + out_off[i];
        for (unsigned c = 0; c < str_len[i]; c++)
            dst[c] = src[c];
    }
}

int str_finalize(b200_set *s) { // caller holds s->mu
    const bool was_dirty = s->dirty;
    B200_CHECK(set_finalize(s));
    if (!was_dirty && s->d_str_off)
        return B200_OK;
    cudaStream_t st = s->ctx->slots[0]->stream;
    // the previous index (if any) is replaced right after set_finalize synchronised every slot: nothing can still touch it
    const size_t en = (size_t)(s->n_entries ? s->n_entries : 1);
    B200_CHECK(s->d_str_off.alloc(s->ctx, en * 8, "ordered_set_string"));
    B200_CHECK(s->d_str_len.alloc(s->ctx, en * 4, "ordered_set_string"));
    B200_CUDA(cudaMemsetAsync(s->d_str_off, 0, en * 8, st));
    B200_CUDA(cudaMemsetAsync(s->d_str_len, 0, en * 4, st));
    unsigned long long sc[2];
    B200_CUDA(cudaMemcpyAsync(sc, s->d_strctr, 16, cudaMemcpyDeviceToHost, st));
    B200_CUDA(cudaStreamSynchronize(st));
    if (sc[0])
        k_str_index<<<nblocks(sc[0]), 256, 0, st>>>(s->log, sc[0], s->probe, s->probe_cap - 1, s->d_str_off, s->d_str_len);
    B200_CUDA(cudaGetLastError());
    B200_CUDA(cudaStreamSynchronize(st));
    return B200_OK;
}

int str_check_error(b200_set *s, cudaStream_t st) {
    unsigned long long h[CTR_N];
    B200_CHECK(read_ctr(s, st, h));
    if (h[CTR_STR_ERROR]) {
        set_error(h[CTR_STR_ERROR] == 2 ? "ordered_set_string: two different strings share one 64-bit hash (std::hash collision); refusing to merge them"
                                        : "ordered_set_string: a string hashes to the reserved empty pattern");
        // the refusal belongs to this call only: later calls that do not repeat the offending string must still succeed
        unsigned long long zero = 0;
        B200_CUDA(cudaMemcpyAsync(s->d_ctr + CTR_STR_ERROR, &zero, sizeof zero, cudaMemcpyHostToDevice, st));
        B200_CUDA(cudaStreamSynchronize(st));
        return B200_ERR_UNSUPPORTED;
    }
    return B200_OK;
}

} // namespace
} // namespace b200

extern "C" {

int b200_strset_create(b200_ctx *ctx, int nmaps, int64_t limit, b200_set **out) {
    if (limit >= 0) {
        set_error("ordered_set_string: limit is not supported");
        return B200_ERR_UNSUPPORTED;
    }
    return set_create(ctx, B200_U64, nmaps, -1, false, true, out);
}

int b200_strset_update(b200_set *s, int slot, const int64_t *offsets, const uint8_t *bytes, const uint8_t *masks, int64_t nrows, int return_values,
                       int64_t *out_values, int16_t *out_map_index, int memspace) {
    if (!s || !s->strings || nrows < 0 || (nrows && !offsets)) {
        set_error("b200_strset_update: invalid argument");
        return B200_ERR_INVALID;
    }
    if (nrows >= (1ll << 40) - 2) {
        set_error("b200_strset_update: more than 2^40 rows in one call");
        return B200_ERR_UNSUPPORTED;
    }
    CallFrame call(s->ctx, slot, memspace, 0, "b200_strset_update");
    B200_CHECK(call.rc);
    std::lock_guard<std::mutex> g(s->mu);
    cudaStream_t st = call.st;
    StrInput in;
    B200_CHECK(stage_strings(call, offsets, bytes, masks, nrows, &in));
    B200_CHECK(set_reserve(s, st, nrows));
    {
        unsigned long long sc[2];
        B200_CUDA(cudaMemcpyAsync(sc, s->d_strctr, 16, cudaMemcpyDeviceToHost, st));
        B200_CUDA(cudaStreamSynchronize(st));
        const uint64_t need = sc[1] + (uint64_t)in.nbytes + 16;
        if (need > s->pool_cap) { // the old pool goes back once `st` has drained (see set_grow)
            const uint64_t cap = std::max<uint64_t>(need + need / 2, 1u << 20);
            DevBuf<char> np;
            B200_CHECK(np.alloc(s->ctx, cap, "b200_strset_update", st));
            if (s->pool) {
                B200_CUDA(cudaMemcpyAsync(np, s->pool, sc[1], cudaMemcpyDeviceToDevice, st));
                B200_CUDA(cudaStreamSynchronize(st));
            }
            np.unbind();
            s->pool = std::move(np);
            s->pool_cap = cap;
        }
    }
    const unsigned long long tag_base = (unsigned long long)s->seq << 40;
    s->seq++;
    s->max_call_rows = std::max<int64_t>(s->max_call_rows, nrows);
    if (nrows) {
        B200_CHECK(set_insert_pass(s, st, [&](int redo) -> int {
            k_str_insert<<<nblocks((unsigned long long)nrows), 256, 0, st>>>(s->table, s->cap - 1, s->d_ctr, s->d_strctr, s->log, s->pool, s->slot_log, in.offsets,
                                                                           in.bytes, in.masks, in.base, 0, nrows, tag_base, redo, kTagLowMask - 1);
            B200_CUDA(cudaGetLastError());
            return B200_OK;
        }));
        k_str_verify<<<nblocks((unsigned long long)nrows), 256, 0, st>>>(s->table, s->cap - 1, s->d_ctr, s->log, s->pool, s->slot_log, in.offsets, in.bytes, in.masks,
                                                                       in.base, nrows);
        B200_CUDA(cudaGetLastError());
    }
    // dirty before the error check: a refused call still inserted its other new strings (all but the offending one), and the
    // next finalisation must see them
    s->dirty = true;
    B200_CHECK(str_check_error(s, st));
    if (return_values && nrows) {
        B200_CHECK(str_finalize(s));
        long long *d_vals;
        short *d_map;
        B200_CHECK(call.out(out_values, sizeof(long long) * nrows, false, &d_vals));
        B200_CHECK(call.out(out_map_index, sizeof(short) * nrows, false, &d_map));
        k_str_map<<<nblocks((unsigned long long)nrows), 256, 0, st>>>(s->probe, s->probe_cap - 1, s->d_str_off, s->d_str_len, s->pool,
                                                                    s->null_count > 0 ? s->null_value : -1, s->nmaps, s->d_offsets, in.offsets, in.bytes, in.masks,
                                                                    in.base, nrows, d_vals, d_map, 1);
        B200_CUDA(cudaGetLastError());
    }
    return call.finish(true);
}

/* out: nrows int64 ordinals (-1: not a member; nulls map to the null ordinal), written to host memory or, with out_is_device, to a
 * device buffer on the slot's stream */
int b200_strset_map_ordinal(b200_set *s, int slot, const int64_t *offsets, const uint8_t *bytes, const uint8_t *masks, int64_t nrows, int64_t *out,
                            int memspace, int out_is_device) {
    if (!s || !s->strings || nrows < 0 || (nrows && (!offsets || !out))) {
        set_error("b200_strset_map_ordinal: invalid argument");
        return B200_ERR_INVALID;
    }
    CallFrame call(s->ctx, slot, memspace, 0, "b200_strset_map_ordinal");
    B200_CHECK(call.rc);
    if (!nrows)
        return B200_OK;
    std::lock_guard<std::mutex> g(s->mu);
    B200_CHECK(str_finalize(s));
    StrInput in;
    B200_CHECK(stage_strings(call, offsets, bytes, masks, nrows, &in));
    long long *d_out;
    B200_CHECK(call.out(out, sizeof(long long) * nrows, out_is_device != 0, &d_out));
    k_str_map<<<nblocks((unsigned long long)nrows), 256, 0, call.st>>>(s->probe, s->probe_cap - 1, s->d_str_off, s->d_str_len, s->pool,
                                                                     s->null_count > 0 ? s->null_value : -1, s->nmaps, s->d_offsets, in.offsets, in.bytes,
                                                                     in.masks, in.base, nrows, d_out, nullptr, 0);
    B200_CUDA(cudaGetLastError());
    return call.finish(true);
}

/* key_array(): first the byte count, then offsets (int64[count + 1]) + bytes in ordinal order; the null slot is an empty string */
int b200_strset_key_bytes(b200_set *s, int64_t *nbytes_out) {
    if (!s || !s->strings || !nbytes_out) {
        set_error("b200_strset_key_bytes: invalid argument");
        return B200_ERR_INVALID;
    }
    B200_CUDA(cudaSetDevice(s->ctx->device));
    std::lock_guard<std::mutex> g(s->mu);
    B200_CHECK(str_finalize(s));
    std::vector<unsigned> len(s->n_entries);
    if (s->n_entries)
        B200_CUDA(cudaMemcpy(len.data(), s->d_str_len, s->n_entries * 4, cudaMemcpyDeviceToHost));
    int64_t total = 0;
    for (unsigned v : len)
        total += v;
    *nbytes_out = total;
    return B200_OK;
}

int b200_strset_key_array(b200_set *s, int64_t *offsets_out, uint8_t *bytes_out) {
    if (!s || !s->strings || !offsets_out) {
        set_error("b200_strset_key_array: invalid argument");
        return B200_ERR_INVALID;
    }
    B200_CUDA(cudaSetDevice(s->ctx->device));
    std::lock_guard<std::mutex> g(s->mu);
    B200_CHECK(str_finalize(s));
    const uint64_t n = s->n_entries;
    std::vector<unsigned> len(n), off(n + 1, 0);
    if (n)
        B200_CUDA(cudaMemcpy(len.data(), s->d_str_len, n * 4, cudaMemcpyDeviceToHost));
    uint64_t total = 0;
    for (uint64_t i = 0; i < n; i++) {
        offsets_out[i] = (int64_t)total;
        off[i] = (unsigned)total;
        total += len[i];
    }
    offsets_out[n] = (int64_t)total;
    if (total >= (1ull << 32)) {
        set_error("ordered_set_string.key_array: more than 4 GB of keys");
        return B200_ERR_UNSUPPORTED;
    }
    if (!total || !bytes_out)
        return B200_OK;
    cudaStream_t st = s->ctx->slots[0]->stream;
    DevBuf<unsigned> d_off;
    DevBuf<char> d_bytes;
    B200_CHECK(d_off.alloc(s->ctx, (n + 1) * 4, "b200_strset_key_array", st));
    B200_CHECK(d_bytes.alloc(s->ctx, total, "b200_strset_key_array", st));
    B200_CUDA(cudaMemcpyAsync(d_off, off.data(), (n + 1) * 4, cudaMemcpyHostToDevice, st));
    k_str_gather<<<nblocks(n), 256, 0, st>>>(s->d_str_off, s->d_str_len, d_off, s->pool, n, d_bytes);
    B200_CUDA(cudaGetLastError());
    B200_CUDA(cudaMemcpyAsync(bytes_out, d_bytes, total, cudaMemcpyDeviceToHost, st));
    B200_CUDA(cudaStreamSynchronize(st));
    return B200_OK;
}

} // extern "C"
