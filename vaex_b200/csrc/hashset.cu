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
    std::mutex mu;
};

namespace b200 {

enum { CTR_COUNT = 0, CTR_OVERFLOW, CTR_NAN_COUNT, CTR_NULL_COUNT, CTR_NAN_TAG, CTR_NULL_TAG, CTR_SENTINEL_TAG, CTR_CURSOR, CTR_SENTINEL_COUNT, CTR_STR_ERROR /* 1: hash == empty pattern, 2: two strings share a 64-bit hash */, CTR_N };

namespace {

constexpr unsigned long long kTagLowMask = (1ULL << 40) - 1;

__device__ __forceinline__ uint64_t load_raw1(const void *data, int isz, long long i) {
    switch (isz) {
    case 8: return __ldcs(static_cast<const unsigned long long *>(data) + i);
    case 4: return __ldcs(static_cast<const unsigned *>(data) + i);
    case 2: return __ldcs(static_cast<const unsigned short *>(data) + i);
    default: return __ldcs(static_cast<const unsigned char *>(data) + i);
    }
}

// insert (or touch) one key; returns false when the table is too full.  "Too full" is detected by PROBE LENGTH, not by a fill
// counter: one shared counter bumped per new key serialises in the L2 (one update at a time to one address), while a
// linear-probing table at load <= 0.5 practically never needs more than
// kMaxProbe steps and one past ~0.85 quickly does.  The bound also makes every probe loop finite by construction.
constexpr int kMaxProbe = 96;
__device__ __forceinline__ bool table_insert(SetSlot *table, unsigned long long mask, unsigned long long canon, unsigned long long tag) {
    unsigned long long h = hash64(canon) & mask;
    for (int step = 0; step < kMaxProbe; step++) {
        // ONE 16-byte L2 load per probe: key and tag share a sector.  A stale tag is harmless: tags only decrease, so at worst the
        // atomicMin below is issued although it changes nothing
        const ulonglong2 slot = __ldcg(reinterpret_cast<const ulonglong2 *>(table + h));
        unsigned long long k = slot.x;
        unsigned long long first = slot.y;
        if (k == SET_EMPTY) {
            k = atomicCAS(&table[h].key, SET_EMPTY, canon);
            if (k == SET_EMPTY)
                k = canon;
            first = ~0ull;
        }
        if (k == canon) {
            if (tag < first)
                atomicMin(&table[h].first, tag);
            return true;
        }
        h = (h + 1) & mask;
    }
    return false;
}

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
        // whose NaN/null rows were already counted); the flag is polled every 32 rows per thread
        if (!dead && (it++ & 31) == 0 && *reinterpret_cast<volatile unsigned long long *>(ctr + CTR_OVERFLOW))
            dead = true;
        if (dead && (skip_keys & 2))
            return;
        const long long row = row0 + i;
        uint64_t raw = load_raw1(keys, isz, row);
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
        unsigned long long tag = tag_base | (unsigned long long)row;
        if (canon == SET_EMPTY) {
            atomicMin(ctr + CTR_SENTINEL_TAG, tag);
            continue;
        }
        if (!table_insert(table, mask, canon, tag)) {
            // raise the flag ONCE (millions of plain stores to one address serialise in the L2) and stop: the host grows the table
            // and redoes this range
            if (!*reinterpret_cast<volatile unsigned long long *>(ctr + CTR_OVERFLOW))
                ctr[CTR_OVERFLOW] = 1ull;
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
        const uint64_t raw = load_raw1(keys, isz, i);
        if ((masks && masks[i]) || raw_isnan(dtype, raw))
            continue; // NaN / null occurrences are counted by k_set_insert
        const unsigned long long w = weights ? weights[i] : 1ull;
        const unsigned long long canon = key_canon(dtype, raw);
        if (canon == SET_EMPTY) {
            n_sent += w;
            continue;
        }
        // the key is present (the insert pass of these rows succeeded); a rehash may have placed it further than kMaxProbe from its
        // home slot, so the probe is bounded by the empty slot only
        unsigned long long h = hash64(canon) & mask;
        while (true) {
            const unsigned long long k = table[h].key;
            if (k == canon) {
                atomicAdd(counts + h, w);
                break;
            }
            if (k == SET_EMPTY)
                break;
            h = (h + 1) & mask;
        }
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
        unsigned long long h = hash64(k) & pmask;
        while (probe[h].key != k)
            h = (h + 1) & pmask;
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
        unsigned long long h = hash64(k) & mask;
        while (atomicCAS(&table[h].key, SET_EMPTY, k) != SET_EMPTY)
            h = (h + 1) & mask;
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
        unsigned long long h = hash64(k) & pmask;
        while (atomicCAS(&probe[h].key, SET_EMPTY, k) != SET_EMPTY)
            h = (h + 1) & pmask;
        probe[h].first = i;
    }
}

__device__ __forceinline__ long long probe_lookup(const SetSlot *probe, unsigned long long mask, long long sentinel_ordinal, unsigned long long canon) {
    if (canon == SET_EMPTY)
        return sentinel_ordinal;
    unsigned long long h = hash64(canon) & mask;
    while (true) {
        const ulonglong2 s = __ldg(reinterpret_cast<const ulonglong2 *>(probe + h));
        if (s.x == canon)
            return (long long)s.y;
        if (s.x == SET_EMPTY)
            return -1;
        h = (h + 1) & mask;
    }
}

// ordered_set::_map_ordinal (src/hash_primitives.hpp:624-691).  out_isz selects int8/16/32/64; out_isz == 0: isin (uint8)
__global__ void __launch_bounds__(256) k_set_map(const SetSlot *probe, unsigned long long mask, long long sentinel_ordinal, long long nan_ordinal, int dtype,
                                                 int isz, const void *keys, long long nrows, void *out, int out_isz) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < nrows; i += (long long)gridDim.x * blockDim.x) {
        uint64_t raw = load_raw1(keys, isz, i);
        long long v = raw_isnan(dtype, raw) ? nan_ordinal : probe_lookup(probe, mask, sentinel_ordinal, key_canon(dtype, raw));
        switch (out_isz) {
        case 0: static_cast<unsigned char *>(out)[i] = v >= 0; break;
        case 1: static_cast<signed char *>(out)[i] = (signed char)v; break;
        case 2: static_cast<short *>(out)[i] = (short)v; break;
        case 4: static_cast<int *>(out)[i] = (int)v; break;
        default: static_cast<long long *>(out)[i] = v; break;
        }
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
                const uint64_t raw = load_raw1(p.keys[k], p.isz[k], i);
                o = raw_isnan(p.dtype[k], raw) ? p.nan_ord[k] : probe_lookup(p.probe[k], p.mask[k], p.sentinel[k], key_canon(p.dtype[k], raw));
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
        uint64_t raw = load_raw1(keys, isz, i);
        if (masks && masks[i]) {
            out_values[i] = null_ordinal;
            out_map[i] = 0;
        } else if (raw_isnan(dtype, raw)) {
            out_values[i] = nan_ordinal;
            out_map[i] = 0;
        } else {
            unsigned long long canon = key_canon(dtype, raw);
            int shard = (int)(key_hash(dtype, canon) % (unsigned long long)nmaps);
            long long g = probe_lookup(probe, mask, sentinel_ordinal, canon);
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

int read_ctr(b200_set *s, cudaStream_t st, unsigned long long *h) {
    B200_CUDA(cudaMemcpyAsync(h, s->d_ctr, sizeof(unsigned long long) * CTR_N, cudaMemcpyDeviceToHost, st));
    B200_CUDA(cudaStreamSynchronize(st));
    return B200_OK;
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
    // the insert kernel keeps no fill counter (see table_insert): count the occupied slots first, then compact them
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
    const unsigned nblk = radix_blocks(E);
    const size_t en = (size_t)(E ? E : 1);
    const size_t off_hist = 5 * en * 8, off_first = off_hist + align_up((size_t)256 * (nblk ? nblk : 1) * 4, 256), off_spec = off_first + align_up((size_t)s->nmaps * 8, 256);
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
    auto pass = [&](int shift, int from_val) -> int {
        k_radix_hist<<<nblk, kRadixThreads, 0, st>>>(tin, vin, E, shift, from_val, hist, nblk, radix_tiles(E));
        k_scan_u32<<<1, 1024, 0, st>>>(hist, 256ull * nblk);
        k_radix_scatter<<<nblk, kRadixThreads, 0, st>>>(tin, vin, tout, vout, E, shift, from_val, hist, nblk, radix_tiles(E));
        B200_CUDA(cudaGetLastError());
        std::swap(tin, tout);
        std::swap(vin, vout);
        return B200_OK;
    };
    if (E > 1) {
        // tags are (call sequence << 40 | row): only the bytes that can differ are sorted on.  The NaN / null tags were moved just
        // behind the largest row (see `special_tag`), so the row part stays below max_low.
        const unsigned long long max_low = (unsigned long long)s->max_call_rows + 2, max_seq = (unsigned long long)(s->seq > 0 ? s->seq - 1 : 0);
        for (int shift = 0; shift < 40 && (max_low >> shift); shift += 8)
            B200_CHECK(pass(shift, 0));
        for (int shift = 0; shift < 24 && (max_seq >> shift); shift += 8)
            B200_CHECK(pass(40 + shift, 0));
        for (int shift = 0; shift < 16 && ((unsigned)(s->nmaps - 1) >> shift); shift += 8)
            B200_CHECK(pass(shift, 1));
    }
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
                      int64_t from_keys_null_index) {
    unsigned long long h[CTR_N];
    int skip_keys = 0;
    if (s->limit >= 0) { // hash_primitives.hpp:237-249: a full set skips the whole flush of this call
        B200_CHECK(set_finalize(s));
        if (set_count_locked(s) >= s->limit)
            skip_keys = 1;
    }
    const unsigned long long tag_base = from_keys ? 0ull : ((unsigned long long)s->seq << 40);
    s->seq++;
    s->max_call_rows = std::max<int64_t>(s->max_call_rows, nrows);
    const unsigned long long first_low = kTagLowMask - 1, second_low = kTagLowMask;
    const unsigned long long null_low = use_offsets ? first_low : second_low;
    const unsigned long long nan_low = use_offsets ? second_low : first_low;
    const int isz = dtype_size(s->dtype);
    const int64_t sub = 1ll << 26;
    // size the table for the call up front (every row could be a new key, capped at 2^22 slots = 64 MB): avoids the
    // grow-and-redo cascade 4K -> 16K -> ... on big inputs; further growth still happens on demand
    {
        uint64_t want = s->cap;
        const uint64_t known = s->dirty ? 0 : (uint64_t)s->n_keys; // exact only right after a finalisation; growth on demand covers the rest
        const uint64_t target = std::min<uint64_t>((known + (uint64_t)nrows) * 2, 1ull << 22);
        while (want < target)
            want <<= 1;
        if (s->cap < want)
            B200_CHECK(set_grow(s, st, want)); // one step (the cascade 4K -> 16K -> ... cost five allocations and rehashes)
    }
    int redo = 0;
    for (int64_t row0 = 0; row0 < nrows;) {
        int64_t n = std::min<int64_t>(sub, nrows - row0);
        k_set_insert<<<nblocks((unsigned long long)n), 256, 0, st>>>(s->table, s->cap - 1, s->d_ctr, s->dtype, isz, d_keys, d_masks, row0, n,
                                                                     tag_base, skip_keys | redo, from_keys_null_index, from_keys ? 1 : 0, nan_low, null_low);
        B200_CUDA(cudaGetLastError());
        B200_CHECK(read_ctr(s, st, h));
        if (h[CTR_OVERFLOW]) {
            unsigned long long zero = 0;
            B200_CUDA(cudaMemcpyAsync(s->d_ctr + CTR_OVERFLOW, &zero, sizeof zero, cudaMemcpyHostToDevice, st));
            B200_CHECK(set_grow(s, st));
            redo = 2; // redo this range: key inserts are idempotent (CAS claim + atomicMin of the tag); NaN/null counting is not
            continue;
        }
        redo = 0;
        row0 += n;
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
    for (int i = 0; i < nothers; i++)
        if (others[i]->nmaps != s->nmaps || others[i]->dtype != s->dtype) {
            set_error("cannot merge with an unequal maps");
            return B200_ERR_STATE;
        }
    B200_CUDA(cudaSetDevice(s->ctx->device));
    for (int i = 0; i < nothers; i++) {
        b200_set *o = others[i];
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
        switch (isz) {
        case 8: static_cast<uint64_t *>(out)[i] = bits; break;
        case 4: static_cast<uint32_t *>(out)[i] = (uint32_t)bits; break;
        case 2: static_cast<uint16_t *>(out)[i] = (uint16_t)bits; break;
        default: static_cast<uint8_t *>(out)[i] = (uint8_t)bits; break;
        }
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
static int set_map_common(b200_set *s, int slot, const void *keys, int64_t nrows, void *out, int out_isz, int memspace, uint32_t flags, const char *name) {
    if (!s || nrows < 0) {
        set_error("%s: invalid argument", name);
        return B200_ERR_INVALID;
    }
    CallFrame call(s->ctx, slot, memspace, flags, name);
    B200_CHECK(call.rc);
    if (!nrows)
        return B200_OK;
    std::lock_guard<std::mutex> g(s->mu);
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
        if (!dead && (it++ & 31) == 0 && *reinterpret_cast<volatile unsigned long long *>(ctr + CTR_OVERFLOW))
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
        unsigned long long pos = hash64(h) & mask;
        bool done = false;
        for (int step = 0; step < kMaxProbe && !done; step++) {
            const ulonglong2 slot = __ldcg(reinterpret_cast<const ulonglong2 *>(table + pos));
            unsigned long long k = slot.x, first = slot.y;
            if (k == SET_EMPTY) {
                k = atomicCAS(&table[pos].key, SET_EMPTY, h);
                if (k == SET_EMPTY) { // this thread owns the new key: pool its bytes, log it
                    k = h;
                    first = ~0ull;
                    const unsigned long long li = atomicAdd(strctr + 0, 1ull), po = atomicAdd(strctr + 1, len);
                    for (unsigned long long c = 0; c < len; c++)
                        pool[po + c] = (char)bytes[b + c];
                    log[li].hash = h, log[li].off = po, log[li].len = (unsigned)len;
                    slot_log[pos] = (unsigned)li;
                }
            }
            if (k == h) {
                if (tag < first)
                    atomicMin(&table[pos].first, tag);
                done = true;
            } else {
                pos = (pos + 1) & mask;
            }
        }
        if (!done) {
            if (!*reinterpret_cast<volatile unsigned long long *>(ctr + CTR_OVERFLOW))
                ctr[CTR_OVERFLOW] = 1ull;
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
        unsigned long long pos = hash64(h) & mask;
        while (true) {
            const unsigned long long k = table[pos].key;
            if (k == h) {
                const StrLog r = log[slot_log[pos]];
                if (r.len != len || !bytes_equal(pool + r.off, bytes + b, len))
                    ctr[CTR_STR_ERROR] = 2;
                break;
            }
            if (k == SET_EMPTY)
                break; // cannot happen after a successful insert pass
            pos = (pos + 1) & mask;
        }
    }
}

// finalized view: ordinal -> where the key's bytes are
__global__ void k_str_index(const StrLog *log, unsigned long long nlog, const SetSlot *probe, unsigned long long pmask, unsigned long long *str_off, unsigned *str_len) {
    for (unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; i < nlog; i += (unsigned long long)gridDim.x * blockDim.x) {
        const long long ord = probe_lookup(probe, pmask, -1, log[i].hash);
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
            ord = probe_lookup(probe, pmask, -1, h);
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
    // room for the worst case of this call: every row a new key
    {
        uint64_t want = s->cap;
        const uint64_t known = s->dirty ? 0 : (uint64_t)s->n_keys;
        const uint64_t target = std::min<uint64_t>((known + (uint64_t)nrows) * 2, 1ull << 22);
        while (want < target)
            want <<= 1;
        if (s->cap < want)
            B200_CHECK(set_grow(s, st, want)); // one step (the cascade 4K -> 16K -> ... cost five allocations and rehashes)
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
    unsigned long long h[CTR_N];
    int redo = 0;
    for (int attempt = 0; nrows && attempt < 64; attempt++) {
        k_str_insert<<<nblocks((unsigned long long)nrows), 256, 0, st>>>(s->table, s->cap - 1, s->d_ctr, s->d_strctr, s->log, s->pool, s->slot_log, in.offsets, in.bytes,
                                                                       in.masks, in.base, 0, nrows, tag_base, redo, kTagLowMask - 1);
        B200_CUDA(cudaGetLastError());
        B200_CHECK(read_ctr(s, st, h));
        if (!h[CTR_OVERFLOW])
            break;
        unsigned long long zero = 0;
        B200_CUDA(cudaMemcpyAsync(s->d_ctr + CTR_OVERFLOW, &zero, sizeof zero, cudaMemcpyHostToDevice, st));
        B200_CHECK(set_grow(s, st));
        redo = 2; // inserts are idempotent; the nulls of this call were already counted
    }
    if (nrows) {
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
