// common.cuh — shared device/host helpers for libb200agg (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include <map>
#include <memory>
#include <mutex>
#include <string>
#include <utility>
#include <vector>

#include "../../include/b200agg.h"

namespace b200 {

// SMs of an H100 SXM: sizes the grid-stride launches that have no context at hand (fills, merges)
constexpr int kSmCount = 132;

// ---- error plumbing ----------------------------------------------------------------------------
void set_error(const char *fmt, ...);
int cuda_fail(cudaError_t e, const char *what, const char *file, int line);

#define B200_CUDA(expr)                                                                                                        \
    do {                                                                                                                       \
        cudaError_t e__ = (expr);                                                                                              \
        if (e__ != cudaSuccess)                                                                                                \
            return ::b200::cuda_fail(e__, #expr, __FILE__, __LINE__);                                                          \
    } while (0)

#define B200_CHECK(expr)                                                                                                       \
    do {                                                                                                                       \
        int rc__ = (expr);                                                                                                     \
        if (rc__ != B200_OK)                                                                                                   \
            return rc__;                                                                                                       \
    } while (0)

// ---- dtype tables ------------------------------------------------------------------------------
__host__ __device__ inline int dtype_size(int dt) {
    switch (dt) {
    case B200_F64:
    case B200_I64:
    case B200_U64: return 8;
    case B200_F32:
    case B200_I32:
    case B200_U32: return 4;
    case B200_I16:
    case B200_U16: return 2;
    default: return 1;
    }
}
__host__ __device__ inline bool dtype_is_float(int dt) { return dt == B200_F64 || dt == B200_F32; }
__host__ __device__ inline bool dtype_is_signed(int dt) { return dt == B200_I64 || dt == B200_I32 || dt == B200_I16 || dt == B200_I8; }
// upcast<T> of the reference (src/agg_sum.cpp:6-62): bool counts as signed
__host__ __device__ inline int dtype_upcast(int dt) {
    if (dtype_is_float(dt))
        return B200_F64;
    if (dtype_is_signed(dt) || dt == B200_BOOL)
        return B200_I64;
    return B200_U64;
}
// device cell type for min/max grids: 8/16-bit integers are held as 32-bit (no narrow atomics); widened back on read
__host__ __device__ inline int dtype_minmax_cell(int dt) {
    switch (dt) {
    case B200_I16:
    case B200_I8: return B200_I32;
    case B200_U16:
    case B200_U8:
    case B200_BOOL: return B200_U32;
    default: return dt;
    }
}

// ---- device-side context objects ---------------------------------------------------------------
struct Slot {
    cudaStream_t stream = nullptr;
    cudaEvent_t h2d_done = nullptr;
    void *stage = nullptr; // device staging arena for host chunks
    size_t stage_cap = 0;
    // host-chunk ingestion: a ring of kBounce page-locked pieces of kBouncePiece bytes.  The calling thread memcpy's a host column
    // piece by piece into the ring and every piece travels to the arena with its own asynchronous copy, so the call returns without
    // waiting for the device (the caller's buffer is only valid during the call, vaex/cpu.py:708-710).  The ring is small on
    // purpose (16 MB a slot whatever the chunk size): the pieces stay in the host's last-level cache between the memcpy that writes
    // them and the DMA that reads them, and no chunk-sized page-locked allocation is ever made.
    static constexpr int kBounceMax = 16;
    void *bounce[kBounceMax] = {};
    size_t bounce_cap[kBounceMax] = {};
    cudaEvent_t bounce_done[kBounceMax] = {};
    unsigned bounce_next = 0;
    // wall-clock nanoseconds of the host-chunk path on this slot (b200_ctx_host_stats): waiting for a ring piece, memcpy into it,
    // enqueueing its copy, the whole of the HOST call; pieces and calls
    uint64_t host_ns[4] = {0, 0, 0, 0}, host_pieces = 0, host_calls = 0;
    void *scratch = nullptr; // partition scratch (ringcount pool + list tables, tilesort buckets)
    size_t scratch_cap = 0;
    // the last ringcount batch on this slot, for b200_ctx_path_stats (device pointers into `scratch`)
    const unsigned *ring_len = nullptr, *ring_ctl = nullptr;
    size_t ring_lists = 0;
    uint64_t ring_rows = 0, ring_memset_bytes = 0, ring_chunk_entries = 0;
    // B200_RING_EVENTS=1: events around the memset, K1 and K2 of the last ringcount batch (b200_ctx_ring_times); created on first use
    cudaEvent_t ring_ev[4] = {};
    bool ring_timed = false;
    std::mutex mu;
};

// ---- device memory -----------------------------------------------------------------------------
// The context's block cache (api.cu), called only by DevBuf.  ctx_alloc takes a cached block of the size class or cudaMalloc's one;
// when the device is full it gives the cache back and retries, and reports B200_ERR_NOMEM naming `what` and the size.
int ctx_alloc(b200_ctx *ctx, void **out, size_t bytes, const char *what);
void ctx_release(b200_ctx *ctx, void *p, size_t bytes);

// One block of device memory from the context's cache, owned by exactly one handle: the block goes back to the cache, filed under the
// size it was allocated with, when the handle is reset, assigned to or destroyed.  A handle bound to a stream waits for that stream
// first: per-call temporaries are bound to the stream that uses them, so an early return cannot hand a block that a kernel or copy
// still uses to the next caller.  Unbound handles belong to objects whose *_destroy synchronises every slot before deleting them.
template <typename T = void> class DevBuf {
  public:
    DevBuf() = default;
    DevBuf(DevBuf &&o) noexcept { *this = std::move(o); }
    DevBuf &operator=(DevBuf &&o) noexcept {
        if (this != &o) {
            reset();
            ctx_ = o.ctx_, ptr_ = o.ptr_, bytes_ = o.bytes_, stream_ = o.stream_, bound_ = o.bound_;
            o.ptr_ = nullptr;
        }
        return *this;
    }
    ~DevBuf() { reset(); }

    int alloc(b200_ctx *ctx, size_t bytes, const char *what) { return alloc(ctx, bytes, what, nullptr, false); }
    int alloc(b200_ctx *ctx, size_t bytes, const char *what, cudaStream_t st) { return alloc(ctx, bytes, what, st, true); }
    // the bound stream has been synchronised and the block now belongs to an object
    void unbind() { bound_ = false; }
    void reset() {
        if (!ptr_)
            return;
        if (bound_)
            cudaStreamSynchronize(stream_);
        ctx_release(ctx_, ptr_, bytes_);
        ptr_ = nullptr;
    }
    T *get() const { return static_cast<T *>(ptr_); }
    operator T *() const { return get(); }

  private:
    int alloc(b200_ctx *ctx, size_t bytes, const char *what, cudaStream_t st, bool bound) {
        reset();
        B200_CHECK(ctx_alloc(ctx, &ptr_, bytes, what));
        ctx_ = ctx, bytes_ = bytes, stream_ = st, bound_ = bound;
        return B200_OK;
    }
    b200_ctx *ctx_ = nullptr;
    void *ptr_ = nullptr;
    size_t bytes_ = 0;
    cudaStream_t stream_ = nullptr;
    bool bound_ = false;
};

} // namespace b200

struct b200_ctx {
    int device = 0;
    int nslots = 0;
    int sm_count = b200::kSmCount;
    size_t smem_optin = 0;
    size_t l2_bytes = 50u << 20; // cudaDeviceProp::l2CacheSize (50 MB on an H100)
    std::vector<b200::Slot *> slots;
    // Grid cache: an aggregation pass creates its aggregators and destroys them when the result has been read (vaex builds a task
    // part per pass), and cudaMalloc / cudaFree synchronise the device and take the driver's allocation lock, which stalls while
    // 16-32 feeder threads are enqueueing copies.  Released grids are kept by exact size (bounded) and handed to the next pass.
    std::mutex cache_mu;
    std::multimap<size_t, void *> cache;
    size_t cache_bytes = 0;
    size_t live_bytes = 0; // handed out and not yet returned (b200_ctx_mem_stats)
};

struct b200_agg {
    b200_ctx *ctx = nullptr;
    int op = 0, dtype = 0, dtype2 = 0, byteswap = 0;
    uint32_t moment = 0;
    uint64_t cells = 0;
    int cell_dtype = 0;        // device cell type of `grid`
    b200::DevBuf<> grid;       // cells * dtype_size(cell_dtype)
    b200::DevBuf<> state;      // FIRST/LAST: cells * 16 B {u64 order key, u64 global row}
    b200::DevBuf<> order;      // FIRST/LAST: cells * dtype_size(dtype2) raw order values
    b200::DevBuf<uint8_t> cell_masked; // FIRST/LAST
    cudaEvent_t chain = nullptr;       // FIRST/LAST: completion of the previous select+deposit pair on this grid (any slot)
    std::mutex chain_mu;
    // NUNIQUE: `grid` holds three planes of `cells` u64 (distinct pairs, NaN rows, null rows); the distinct (cell, value) pairs
    // live in one open-addressing table of 16-byte slots
    b200::DevBuf<unsigned long long> ntable;
    uint64_t ncap = 0;                       // slots (power of two)
    b200::DevBuf<unsigned long long> ntotal; // device counter: pairs in the table
    uint64_t npairs = 0;                     // host copy, refreshed after every launch
    std::mutex nmu;                          // growth needs the table to itself
    // LIST (list.cu): one record per row {cell * 4 + category, value bits}, appended per call, sorted when the result is asked for
    b200::DevBuf<unsigned long long> list_keys, list_vals;
    b200::DevBuf<unsigned> list_counts; // after finish: exclusive offsets per cell (+ the total)
    uint64_t list_n = 0, list_cap = 0, list_total = 0;
    bool list_sorted = false;
    // LIST_STRING (list.cu): the same records (key = cell, payload = record index | null << 63); every call appends its byte range
    // to `lstr_pool` and list_starts[i] is where record i's string starts there (list_cap + 1 entries: the last one closes the pool)
    b200::DevBuf<unsigned long long> list_starts;
    b200::DevBuf<char> lstr_pool;
    uint64_t lstr_pool_n = 0, lstr_pool_cap = 0;
    // after finish: int64 string offsets[list_total + 1], the gathered bytes, one validity byte per element
    b200::DevBuf<long long> lstr_off;
    b200::DevBuf<char> lstr_bytes;
    b200::DevBuf<uint8_t> lstr_valid;
    uint64_t lstr_nbytes = 0;

    ~b200_agg() {
        if (chain)
            cudaEventDestroy(chain);
    }
};

namespace b200 {

// The frame of one per-slot library call: how it reads the caller's memory, where its results land and when it may return.
// Construction checks the slot (B200_ERR_INVALID naming the call, in `rc`), sets the device and takes the slot's lock for the
// frame's lifetime.  The slot lock is taken before any set, aggregator or statistic lock, in every call.
//
// Inputs, two-phase: plan() every column, then commit() stages the host ones into the slot's arena in one allocation and dev()
// gives each column's device pointer.  HOST columns go through the slot's page-locked bounce ring (Slot::bounce); MIXED columns
// are classified one by one and the host ones are copied straight from the caller's buffers; DEVICE columns are used in place.
// Results: out() gives the device pointer a result is written to, the caller's own or a temporary copied back by finish().
//
// The return rule, applied by finish(): the call waits for the slot's stream when a result goes to host memory, when MIXED
// inputs were copied straight from the caller's host buffers and B200_FLAG_ASYNC_HOST does not keep them alive (they are valid
// only during the call, vaex/cpu.py:708-710), or when the call asks to wait.  HOST inputs were memcpy'd into the bounce ring and
// DEVICE inputs stay the caller's: nothing of the caller's is read after return, so the next chunk (this slot or another)
// overlaps this one's copies and kernels.
class CallFrame {
  public:
    CallFrame(b200_ctx *ctx, int slot, int memspace, uint32_t flags, const char *call);
    ~CallFrame();
    CallFrame(const CallFrame &) = delete;
    CallFrame &operator=(const CallFrame &) = delete;

    int rc = B200_OK; // check before anything else: nothing is locked unless it is B200_OK
    b200_ctx *const ctx;
    Slot *sl = nullptr;
    cudaStream_t st = nullptr;

    // whether an input column lives on the device: every column of a DEVICE call, none of a HOST call, each on its own in MIXED
    bool on_device(const void *p) const;
    // whether a result pointer lives on the device: every one of a DEVICE call, each on its own otherwise
    bool result_on_device(const void *p) const;
    void plan(const void *p, size_t bytes);
    int commit();
    const void *dev(const void *p) const;
    // the device pointer `bytes` of a result are written to: `p` itself when on_device, otherwise a temporary on the slot's
    // stream that finish() copies to `p`
    template <typename T> int out(void *p, size_t bytes, bool on_device, T **dev) {
        if (on_device) {
            *dev = static_cast<T *>(p);
            return B200_OK;
        }
        DevBuf<> buf;
        B200_CHECK(buf.alloc(ctx, bytes, call_, st));
        *dev = static_cast<T *>(buf.get());
        results_.push_back(Result{p, bytes, std::move(buf)});
        return B200_OK;
    }
    int finish(bool wait = false);

  private:
    struct Entry {
        const void *host;
        size_t bytes;
        void *dev;
    };
    struct Result {
        void *host;
        size_t bytes;
        DevBuf<> buf;
    };
    const char *call_;
    int memspace_;
    bool async_host_;
    std::unique_lock<std::mutex> lock_;
    uint64_t t0_ = 0;
    std::vector<Entry> entries_;
    std::vector<Result> results_;
};

int slot_reserve(b200_ctx *ctx, Slot *s, size_t bytes);
// the slot of a call that reads and writes device memory only and so needs no CallFrame (take.cu, sort.cu): checks the slot
// (B200_ERR_INVALID naming `what`) and sets the device; the caller takes the slot's lock
int device_slot(b200_ctx *ctx, int slot, const char *what, Slot **out);

inline size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

} // namespace b200
