// settable.cuh — the key table of the ordered sets, counters, index_hash and ordered_set_string (hashset.cu), also probed by the
// fused B200_BINNER_HASH binner (binby_index.cuh) and by the expressions' _ordinal_values (expr.cu).
//
// An open-addressing table of 16-byte SetSlot {key, first}; SET_EMPTY marks a free slot.  A key's home slot is hash64(key) & mask
// and a collision steps linearly to (h + 1) & mask.  The functions below are the only code that computes a home slot or steps a
// probe; each keeps the memory access its callers need (see each one).
#pragma once
#include "device_utils.cuh"

namespace b200 {

#define SET_EMPTY 0xFFFFFFFFFFFFFFFFULL
struct SetSlot {
    unsigned long long key;   // canonical 64-bit key pattern
    unsigned long long first; // pass 1: (chunk_seq << 40 | row) of the first occurrence; after finalize: global ordinal
};

// An insert gives up when the table is too full.  "Too full" is detected by PROBE LENGTH, not by a fill counter: one shared counter
// bumped per new key serialises in the L2 (one update at a time to one address), while a linear-probing table at load <= 0.5
// practically never needs more than kMaxProbe steps and one past ~0.85 quickly does.  The bound also makes every insert finite.
constexpr int kMaxProbe = 96;

__device__ __forceinline__ unsigned long long set_home(const unsigned long long key, const unsigned long long mask) { return hash64(key) & mask; }
__device__ __forceinline__ unsigned long long set_step(const unsigned long long h, const unsigned long long mask) { return (h + 1) & mask; }

// A table no thread writes during the call (a finalized probe table, an index's table during a lookup): ONE 16-byte read-only load
// per step, key and value share a sector.  true and *value = the key's `first` when the key is there.
__device__ __forceinline__ bool set_lookup(const SetSlot *table, unsigned long long mask, unsigned long long key, unsigned long long *value) {
    unsigned long long h = set_home(key, mask);
    while (true) {
        const ulonglong2 s = __ldg(reinterpret_cast<const ulonglong2 *>(table + h));
        if (s.x == key) {
            *value = s.y;
            return true;
        }
        if (s.x == SET_EMPTY)
            return false;
        h = set_step(h, mask);
    }
}

// ordered_set::_map_ordinal (src/hash_primitives.hpp:624-691) on a finalized probe table: the key's global ordinal, -1 when absent.
// The key whose pattern is SET_EMPTY cannot live in the table: its ordinal is passed in.
__device__ __forceinline__ long long set_ordinal(const SetSlot *probe, unsigned long long mask, long long sentinel_ordinal, unsigned long long canon) {
    if (canon == SET_EMPTY)
        return sentinel_ordinal;
    unsigned long long ord;
    return set_lookup(probe, mask, canon, &ord) ? (long long)ord : -1;
}

// The slot of a key, ~0ull when absent, with plain 8-byte key loads.  Bounded by the empty slot only: a rehash may have placed a
// key further than kMaxProbe from its home slot.
__device__ __forceinline__ unsigned long long set_slot(const SetSlot *table, unsigned long long mask, unsigned long long key) {
    unsigned long long h = set_home(key, mask);
    while (true) {
        const unsigned long long k = table[h].key;
        if (k == key)
            return h;
        if (k == SET_EMPTY)
            return ~0ull;
        h = set_step(h, mask);
    }
}

// Claims the first free slot on the probe path of a key known not to be in the table (a rehash, the build of a probe table) and
// returns it; the caller fills `first`.
__device__ __forceinline__ unsigned long long set_claim(SetSlot *table, unsigned long long mask, unsigned long long key) {
    unsigned long long h = set_home(key, mask);
    while (atomicCAS(&table[h].key, SET_EMPTY, key) != SET_EMPTY)
        h = set_step(h, mask);
    return h;
}

struct NoClaimHook {
    __device__ void operator()(unsigned long long) const {}
};

// Inserts (or touches) a key with its first-occurrence tag: the slot's `first` keeps the smallest tag.  false when kMaxProbe steps
// found neither the key nor a free slot: the table is too full.  on_claim(slot) runs once per new key, in the thread whose CAS
// claimed its slot, before the tag is stored.
template <typename OnClaim = NoClaimHook>
__device__ __forceinline__ bool set_insert(SetSlot *table, unsigned long long mask, unsigned long long key, unsigned long long tag, OnClaim on_claim = {}) {
    unsigned long long h = set_home(key, mask);
    for (int step = 0; step < kMaxProbe; step++) {
        // ONE 16-byte L2 load per probe: key and tag share a sector.  A stale tag is harmless: tags only decrease, so at worst the
        // atomicMin below is issued although it changes nothing
        const ulonglong2 slot = __ldcg(reinterpret_cast<const ulonglong2 *>(table + h));
        unsigned long long k = slot.x;
        unsigned long long first = slot.y;
        if (k == SET_EMPTY) {
            k = atomicCAS(&table[h].key, SET_EMPTY, key);
            if (k == SET_EMPTY) {
                k = key;
                on_claim(h);
            }
            first = ~0ull;
        }
        if (k == key) {
            if (tag < first)
                atomicMin(&table[h].first, tag);
            return true;
        }
        h = set_step(h, mask);
    }
    return false;
}

// The overflow flag of an inserting kernel.  Once any thread's insert failed the host grows the table and redoes the pass, so the
// other threads stop too: each polls the flag once every kPollRows of its rows, in the kernel's own row-loop condition
// (`(it++ % kPollRows) == 0 && overflow_seen(flag)`; with the row count inside a helper the compiler branches around the poll
// instead of predicating it).
constexpr unsigned kPollRows = 32;
__device__ __forceinline__ bool overflow_seen(const unsigned long long *flag) { return *reinterpret_cast<const volatile unsigned long long *>(flag); }

// Raises the flag once: millions of plain stores to one address serialise in the L2.
__device__ __forceinline__ void overflow_raise(unsigned long long *flag) {
    if (!overflow_seen(flag))
        *flag = 1ull;
}

} // namespace b200
