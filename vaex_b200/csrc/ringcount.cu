// ringcount.cu — count(*) on grids that do not fit in shared memory WITHOUT one L2 atomic per row (the headline path).
//
// Why two kernels: a direct kernel issues one RED per row, and the L2 retires only a fixed number of sector operations per clock
// chip-wide, loads included, which caps the 2-D 1024^2 count far below the HBM stream rate.  Shared-memory atomics retire
// several times more lanes per clock, but a 1027^2 grid is 4 MB even with 32-bit counters.  So the grid is
// cut into <= 32 (else 64) GRID TILES ("parts") of <= 49151 cells and the rows are partitioned by part first.  A part is every
// 32nd (64th) row of the grid along the outermost key when ceil(rows / parts) grid rows fit one part (INTERLEAVED parts: a
// crowded distribution spreads evenly over them), else a contiguous range of the index:
//
//   K1 k_ring_partition  every WARP is autonomous.  The keys of the NEXT 256-row group are loaded into registers (128-bit,
//                        evict-first loads) while the current group is placed, and the group after that is bulk-prefetched
//                        into L2 (one cp.async.bulk.prefetch per key column).
//                        Per row: the bit-exact fp64 bin index, the part (outer cell mod parts, or idx / tile_cells by one
//                        IMAD.HI), ONE shared-memory atomic
//                        on the (warp, part) counter whose return value is the row's slot in that part's RING (96 entries), and
//                        one 16-bit store of the local cell index into the ring.  Every 256 rows the rings that hold a full
//                        LINE (64 entries = 128 bytes) append it to the part's current CHUNK in global memory — half a warp per
//                        line: one LDS.64 + one coalesced STG.64 per lane — and slide the <= 32 entries behind it to the front.
//                        There is no scan, no scatter pass and no copy-out pass.  (Flushing 16-entry granules from the owner
//                        lanes instead would cost divergent 16-byte shared-memory accesses.)
//                        Chunks (512..2048 entries) come from ONE pool: a warp reserves 32 chunks with one global atomic and
//                        hands them to its parts with a ballot; the chunks of a (warp, part) form a linked list (next[]), its
//                        head and entry count go to head[] / len[], every warp adds its entry counts to the part totals at exit.
//                        No table is memset: K1 writes every entry of them K2 reads.  No per-part bucket provisioning, no
//                        overflow fallback, and 2 B/row of scratch whatever the distribution.
//   K2 k_ring_count      one persistent CTA per SM takes a contiguous share of the (part, warp) lists (balanced by entry count,
//                        from K1's part totals: every warp sees the same row distribution), keeps the part's u32 histogram in <= 192 KB of shared
//                        memory, walks the lists with 128-bit loads + one ATOMS per entry, and flushes the non-zero cells with one
//                        RED.ADD.64 each when the part changes (1-2 flushes per CTA).
//
// HBM traffic: 8 B/row of columns + 2 B/row written + 2 B/row read.  Exact integer counts, same grid layout, any distribution:
// a ring that fills up inside one 256-row group (> 32 rows of a warp in one part on top of a full leftover) sends the excess rows
// to direct REDs.
#include <math.h>

#include <algorithm>
#include <type_traits>

#include "binby.cuh"
#include "device_utils.cuh"

namespace b200 {

struct RingParams : FloatKeys {
    unsigned stride_sum;          // sum(stride): bin_cell_m1 returns cell - 1
    float clamp_lo[3], clamp_hi[3]; // CLAMPED variant (fp32 keys): see bin_cell_m2_clamped
    long long row0, nrows;        // this batch
    unsigned cells;
    unsigned tile_cells;          // cells per part (<= 49151): local cell index < tile_cells < 2^16; tile_cells is the pad entry
    // contiguous parts: part = idx / tile_cells, local = idx % tile_cells
    unsigned neg_tile_cells;      // 2^32 - tile_cells: local = idx + part * neg_tile_cells in one IMAD
    unsigned magic;               // part == __umulhi(idx, magic) for every idx < cells (verified on the host)
    // interleaved parts (`interleaved` != 0): with c the cell of the outermost key (the last one, stride outer_stride),
    // part = c mod nparts_pad, local = (c / nparts_pad) * outer_stride + (idx - c * outer_stride)
    int interleaved;
    unsigned outer_stride;
    unsigned inner_sum;           // stride_sum - outer_stride
    unsigned part_shift;          // log2(nparts_pad)
    int nparts;
    int nparts_pad;               // 32 * PPL
    unsigned chunk_shift;         // chunk = 1 << chunk_shift entries (9..11)
    unsigned nchunks_cap;         // chunks in the pool
    unsigned nlists_w;            // warps of K1 (lists per part)
    // Only the control block is memset; K1 writes every other table entry that K2 reads
    unsigned short *pool;         // chunk c = pool + (c << chunk_shift)
    unsigned *next;               // per chunk: next chunk of the same (warp, part) list; kNone = last   (set when the chunk opens)
    unsigned short *unused;       // per chunk: entries at the tail that were never written              (0 when it opens)
    unsigned *head;               // [warp][nparts_pad]: first chunk of the list; kNone = empty            (kNone at K1's start)
    unsigned *len;                // [warp][nparts_pad]: entries in the list (pads included)               (at K1's exit)
    unsigned *ctl;                // control block (memset 0): [0] pool cursor in chunks, [kPartTotals + part] entries of a part
    unsigned long long *grid;
};

namespace {

constexpr int kGroupRows = 256;   // rows between two ring flushes: 8 per lane
constexpr int kGran = 16;         // entries per lane and step in k_ring_count
constexpr unsigned kLine = 64;    // entries a ring flush moves: one 128-byte line
constexpr int kLineLanes = kLine / 8; // lanes that move one line with 16 bytes each
constexpr unsigned kSuper = 32;   // chunks a warp reserves from the pool at a time
constexpr unsigned kNone = 0xFFFFFFFFu;
constexpr int kCountThreads = 1024;
constexpr int kPartTotals = 64;   // ctl[kPartTotals + part]: entries of a part (pads included), summed by K1's warps
constexpr size_t kCtlBytes = (kPartTotals + kRingParts) * 4;

// CLAMPED index for fp32 keys: halves the load on the conversion pipe (F2F.F64.F32 + F2I.F64 per key on the quarter-rate XU
// pipe).  The cell is a monotone function of the key (every step of
// the reference formula is monotone and correctly rounded).  The host finds by bisection over the fp32 values
//   clamp_lo = the largest fp32 whose cell is 1 (underflow), clamp_hi = the smallest fp32 whose cell is bins+2 (overflow)
// and checks floor(t(clamp_lo)) == -1 and floor(t(clamp_hi)) == bins with the reference formula.  Then for every non-NaN key
// v' = min(max(v, clamp_lo), clamp_hi) has the same cell as v and -1 <= floor(t(v')) <= bins, so no integer clamp is needed and
// the floor can be taken with one round-down addition of 1.5 * 2^52 (low word of the sum) instead of a conversion.
// Returns cell - 2; NaN -> -2.
__device__ __forceinline__ int bin_cell_m2_clamped(float v, float lo, float hi, double vmin, double scale, double bins_d) {
    const float vc = fminf(fmaxf(v, lo), hi); // NaN -> lo (replaced below)
    const double t = __dmul_rn(__dmul_rn(__dsub_rn((double)vc, vmin), scale), bins_d);
    const int i = __double2loint(__dadd_rd(t, 6755399441055744.0));
    return v != v ? -2 : i;
}

// cell - 2 (CLAMPED) or cell - 1 of key d: the index is the sum of these times the strides, plus 2 (or 1) x stride_sum
template <typename T, bool CLAMPED>
__device__ __forceinline__ int key_cell(const RingParams &p, T v, int d) {
    if constexpr (CLAMPED)
        return bin_cell_m2_clamped(v, p.clamp_lo[d], p.clamp_hi[d], p.vmin[d], p.scale[d], p.bins_d[d]);
    else
        return bin_cell_m1((double)v, p.vmin[d], p.scale[d], p.bins_d[d], p.bins[d]);
}

// one row: bit-exact index, part, ONE shared-memory atomic for the slot, one 16-bit store.
// ILV: parts interleaved by the outermost key's cell (its value mod 32 * PPL) instead of contiguous ranges of the index: the rows
// of a crowded distribution spread over all parts, so fewer lanes of a warp rank into the same counter at once.
template <typename T, int ND, int RING, int RSTRIDE, bool CLAMPED, int PPL, bool ILV>
__device__ __forceinline__ void place_row(const RingParams &p, const T (&v)[ND], unsigned *cnt, unsigned short *ring, unsigned &idx, unsigned &slot_out,
                                          unsigned &worst) {
    constexpr unsigned kBase = CLAMPED ? 2 : 1;
    unsigned id, part, local;
    if constexpr (ILV) {
        constexpr unsigned kShift = PPL == 1 ? 5 : 6;
        unsigned inner = kBase * p.inner_sum;
#pragma unroll
        for (int d = 0; d < ND - 1; d++)
            inner += (unsigned)key_cell<T, CLAMPED>(p, v[d], d) * p.stride[d];
        const unsigned c = (unsigned)key_cell<T, CLAMPED>(p, v[ND - 1], ND - 1) + kBase;
        id = c * p.outer_stride + inner;
        part = c & ((1u << kShift) - 1u);
        local = (c >> kShift) * p.outer_stride + inner;
    } else {
        id = kBase * p.stride_sum;
#pragma unroll
        for (int d = 0; d < ND; d++)
            id += (unsigned)key_cell<T, CLAMPED>(p, v[d], d) * p.stride[d];
        part = __umulhi(id, p.magic);
    }
    idx = id;
    const unsigned slot = atomicAdd(cnt + part, 1u);
    slot_out = slot;
    worst = max(worst, slot);
    if constexpr (!ILV)
        local = id + part * p.neg_tile_cells; // after the atomic: one register less live across it
    if (slot < (unsigned)RING)
        ring[part * RSTRIDE + slot] = (unsigned short)local;
}

// the grid cell of entry `local` (< tile_cells) of `part`: one division for interleaved parts
__device__ __forceinline__ unsigned long long grid_cell(const RingParams &p, unsigned part, unsigned local) {
    if (!p.interleaved)
        return (unsigned long long)part * p.tile_cells + local;
    const unsigned q = local / p.outer_stride;
    return (unsigned long long)((q << p.part_shift) | part) * p.outer_stride + (local - q * p.outer_stride);
}

// one group of 256 rows (8 per lane) whose keys the caller already holds in registers (loaded one group ahead).
// Returns the largest slot a row of this lane was given (>= RING: that row did not fit, see `overflow`).
template <typename T, int ND, int RING, int RSTRIDE, bool CLAMPED, int PPL, bool ILV>
__device__ __forceinline__ unsigned group_rows_regs(const RingParams &p, const T (&c)[2][ND][4], unsigned *cnt, unsigned short *ring, unsigned idx[8],
                                                    unsigned slots[8]) {
    unsigned worst = 0;
#pragma unroll
    for (int q = 0; q < 2; q++)
#pragma unroll
        for (int j = 0; j < 4; j++) {
            T v[ND];
#pragma unroll
            for (int d = 0; d < ND; d++)
                v[d] = c[q][d][j];
            place_row<T, ND, RING, RSTRIDE, CLAMPED, PPL, ILV>(p, v, cnt, ring, idx[q * 4 + j], slots[q * 4 + j], worst);
        }
    return worst;
}

// the ragged end of the batch: global loads with bounds; slots[] = kNone marks rows that do not exist
template <typename T, int ND, int RING, int RSTRIDE, bool CLAMPED, int PPL, bool ILV>
__device__ __forceinline__ unsigned group_rows_tail(const RingParams &p, long long gbase, long long tend, int lane, unsigned *cnt, unsigned short *ring,
                                                    unsigned idx[8], unsigned slots[8]) {
    unsigned worst = 0;
#pragma unroll
    for (int q = 0; q < 2; q++)
#pragma unroll
        for (int j = 0; j < 4; j++) {
            const long long row = gbase + q * 128 + lane * 4 + j;
            idx[q * 4 + j] = 0;
            slots[q * 4 + j] = kNone;
            if (row < tend) {
                T v[ND];
#pragma unroll
                for (int d = 0; d < ND; d++)
                    v[d] = __ldcs(static_cast<const T *>(p.x[d]) + row);
                place_row<T, ND, RING, RSTRIDE, CLAMPED, PPL, ILV>(p, v, cnt, ring, idx[q * 4 + j], slots[q * 4 + j], worst);
            }
        }
    return worst;
}

// shared memory of one warp: [rings: 32*PPL parts x (RING + 8) u16] [counters: 32*PPL u32] [flush map: 32 x {position, owner}]
// A ring holds < 64 entries left over from the last flush + the new ones of one group; a flush moves whole LINES of 64 entries
// (128 bytes).  With <= 32 new entries per part and group the ring never fills (the busiest part of the headline workload takes
// 19 +- 4 of a group's 256 rows); rows that find it full go to direct REDs.
constexpr int kRing = 96;
constexpr int kRingStride = kRing + 8; // 208 bytes: 16-byte aligned rows that rotate over the banks
template <int PPL>
struct RingLayout {
    static constexpr size_t kRingBytes = 32ull * PPL * kRingStride * 2;
    static constexpr size_t kCntBytes = 32ull * PPL * 4 + 256; // + the flush's (write position, owner) map
    static constexpr size_t kPerWarp = kRingBytes + kCntBytes;
    // two CTAs per SM; 24 warps per SM leave 85 registers per thread: the two key sets + the placement fit without spills
    static constexpr int kWarps = std::min<int>(12, (113 * 1024 - 512) / kPerWarp);
};

// state of the parts a lane owns (parts lane, lane+32, ...): where the next granule goes
template <int PPL>
struct Owner {
    unsigned wpos[PPL]; // next entry to write (pool entry index); == wend: the current chunk is full / there is none yet
    unsigned wend[PPL];
    unsigned cur[PPL];  // current chunk id (kNone: none yet)
    unsigned total[PPL]; // entries written to this list so far
};

template <typename T, int ND, int PPL, int WARPS, bool CLAMPED, bool ILV>
__global__ void __launch_bounds__(WARPS * 32, 2) k_ring_partition(const __grid_constant__ RingParams p) {
    using L = RingLayout<PPL>;
    constexpr int RING = kRing, RSTRIDE = kRingStride;
    static_assert(RING - kLine <= kLine && (RSTRIDE * 2) % 16 == 0, "ring geometry");
    extern __shared__ __align__(128) unsigned char dyn_smem[];

    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    unsigned char *mine = dyn_smem + (size_t)warp * L::kPerWarp;
    unsigned short *const ring = reinterpret_cast<unsigned short *>(mine); // [32*PPL][RING + 8]
    unsigned *const cnt = reinterpret_cast<unsigned *>(mine + L::kRingBytes);
    uint2 *const fmap = reinterpret_cast<uint2 *>(cnt + 32 * PPL); // [32] {pool entry index, owner lane} of the lines of one flush
#pragma unroll
    for (int k = 0; k < PPL; k++)
        cnt[lane + 32 * k] = 0;
    __syncwarp();

    const unsigned cshift = p.chunk_shift, csize = 1u << cshift;
    const long long wglobal = (long long)blockIdx.x * WARPS + warp, wtotal = (long long)gridDim.x * WARPS;
#pragma unroll
    for (int k = 0; k < PPL; k++) // empty lists until their first chunk opens (the owner lane overwrites its own entry)
        p.head[(unsigned long long)wglobal * p.nparts_pad + lane + 32 * k] = kNone;

    Owner<PPL> own;
#pragma unroll
    for (int k = 0; k < PPL; k++)
        own.wpos[k] = own.wend[k] = 0, own.cur[k] = kNone, own.total[k] = 0;
    // the warp's reservation in the pool: chunks [sc_next, sc_end) are free; lane 0 holds the NEXT reservation (prefetched)
    unsigned sc_next = 0, sc_end = 0, sn_pref = 0;
    if (lane == 0)
        sn_pref = atomicAdd(p.ctl, kSuper);

    // ---- flush: every ring that holds a full LINE (64 entries = 128 bytes) appends it to its chunk list -------------------------
    // The owners (lane l owns parts l, l+32) do the bookkeeping in parallel: chunk switch, write position, counter.  Then the warp
    // moves the lines, FOUR parts per step: a quarter-warp copies one line with one LDS.128 + one coalesced STG.128 per lane and
    // slides the <= 32 entries behind it to the ring's front.  `final`: the incomplete last line too, padded with entries ==
    // tile_cells (k_ring_count's spare cell).
    auto flush = [&](bool final) {
#pragma unroll
        for (int k = 0; k < PPL; k++) {
            const int part = lane + 32 * k;
            unsigned n = min(cnt[part], (unsigned)RING); // rows past RING went to direct REDs
            if (final && n > 0 && n < kLine) {
                for (unsigned e = n; e < kLine; e++)
                    ring[part * RSTRIDE + e] = (unsigned short)p.tile_cells;
                n = kLine;
            }
            const bool has = n >= kLine; // cnt of parts >= nparts stays 0
            const bool need = has && own.wpos[k] == own.wend[k];
            // hand out chunks (rare: once per chunk per part); warp-uniform bookkeeping, ids in lane order
            unsigned newid = kNone;
            const unsigned mneed = __ballot_sync(0xffffffffu, need);
            if (mneed) {
                const unsigned sn = __shfl_sync(0xffffffffu, sn_pref, 0);
                const unsigned i = __popc(mneed & ((1u << lane) - 1u)), tot = __popc(mneed), avail = sc_end - sc_next;
                if (need)
                    newid = i < avail ? sc_next + i : sn + (i - avail);
                if (tot >= avail) { // the current reservation is used up: switch to the prefetched one, prefetch another
                    sc_next = sn + (tot - avail);
                    sc_end = sn + kSuper;
                    if (lane == 0)
                        sn_pref = atomicAdd(p.ctl, kSuper);
                } else {
                    sc_next += tot;
                }
            }
            unsigned wp = kNone; // pool entry index where this part's line goes
            if (has) {
                if (need && newid < p.nchunks_cap) { // open the next chunk of this list
                    if (own.cur[k] == kNone)
                        p.head[(unsigned long long)wglobal * p.nparts_pad + part] = newid;
                    else
                        p.next[own.cur[k]] = newid;
                    p.next[newid] = kNone; // the list's last chunk until the next one opens; full until the final flush says otherwise
                    p.unused[newid] = 0;
                    own.cur[k] = newid;
                    own.wpos[k] = newid << cshift;
                    own.wend[k] = own.wpos[k] + csize;
                }
                if (own.wpos[k] != own.wend[k]) {
                    wp = own.wpos[k];
                    own.wpos[k] += kLine;
                    own.total[k] += kLine;
                } else { // pool exhausted: cannot happen (sized for the worst case); stay exact anyway
                    for (unsigned e = 0; e < kLine; e++) {
                        const unsigned c = ring[part * RSTRIDE + e];
                        if (c < p.tile_cells)
                            atomicAdd(p.grid + grid_cell(p, part, c), 1ull);
                    }
                }
                cnt[part] = n - kLine;
            }
            // the owners publish {write position, lane} in rank order; then every group of kLineLanes lanes moves one line
            const unsigned m = __ballot_sync(0xffffffffu, has);
            if (m) {
                const int nl = __popc(m);
                if (has)
                    fmap[__popc(m & ((1u << lane) - 1u))] = make_uint2(wp, (unsigned)lane);
                __syncwarp();
                const int grp = lane / kLineLanes, gl = lane % kLineLanes;
                for (int j = grp; j < nl; j += 32 / kLineLanes) {
                    const uint2 e = fmap[j];
                    uint4 *r = reinterpret_cast<uint4 *>(ring + (e.y + 32 * k) * RSTRIDE);
                    const uint4 w = r[gl];
                    uint4 up = make_uint4(0, 0, 0, 0);
                    if (gl < (RING - (int)kLine) / 8)
                        up = r[kLineLanes + gl];
                    if (e.x != kNone)
                        reinterpret_cast<uint4 *>(p.pool + e.x)[gl] = w;
                    if (gl < (RING - (int)kLine) / 8)
                        r[gl] = up; // the entries behind the line slide to the front (each lane rewrites the 16 bytes it read)
                }
                __syncwarp();
            }
        }
    };
    // rows that found their ring full (slot >= RING) go straight to the grid; `slots` are the atomics' return values of one group
    auto overflow = [&](const unsigned idx[8], const unsigned slots[8]) {
#pragma unroll
        for (int r = 0; r < 8; r++)
            if (slots[r] >= (unsigned)RING && slots[r] != kNone)
                atomicAdd(p.grid + idx[r], 1ull);
    };

    // ---- complete groups of 256 rows: the keys of the NEXT group are loaded into registers (128-bit, evict-first) while the
    // current one is placed: two register sets, the loop is unrolled by two so that no copy is needed.  (Staging them through shared
    // memory instead would add shared-memory traffic to a kernel bound by the shared-memory pipe.)
    const long long ngroups = p.nrows / kGroupRows;
    auto load = [&](long long g, T (&dst)[2][ND][4]) {
        const long long r0 = p.row0 + g * kGroupRows + lane * 4;
#pragma unroll
        for (int q = 0; q < 2; q++)
#pragma unroll
            for (int d = 0; d < ND; d++)
                ldcs4<T>(p.x[d], r0 + q * 128, dst[q][d]);
    };
    // the warp's group two turns ahead goes into L2 with one bulk prefetch per key column (lane d: column d).  The register
    // loads reach only one group ahead; without this the warp has no load in flight once they land, and HBM sees too few
    // requests (3.72 -> 3.55 ms per 1e9 rows on an H100 80GB HBM3 at 700 W; three turns ahead gained nothing).  Columns are
    // 16-byte aligned and batches start on a 256-row boundary, so every group is 16-byte aligned.
    constexpr long long kPrefetch = 2;
    auto prefetch = [&](long long g) {
        if (lane < ND && g < ngroups) {
            const T *src = static_cast<const T *>(p.x[lane]) + p.row0 + g * kGroupRows;
            asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(src), "r"((unsigned)(kGroupRows * sizeof(T))) : "memory");
        }
    };
    auto place = [&](const T (&c)[2][ND][4]) {
        unsigned idx[8], slots[8];
        const unsigned worst = group_rows_regs<T, ND, RING, RSTRIDE, CLAMPED, PPL, ILV>(p, c, cnt, ring, idx, slots);
        __syncwarp();
        flush(false);
        if (__any_sync(0xffffffffu, worst >= (unsigned)RING))
            overflow(idx, slots);
        __syncwarp();
    };
    {
        T ca[2][ND][4], cb[2][ND][4];
        long long g = wglobal;
        if (g < ngroups)
            load(g, ca);
        while (g < ngroups) {
            prefetch(g + kPrefetch * wtotal);
            if (g + wtotal < ngroups)
                load(g + wtotal, cb);
            place(ca);
            g += wtotal;
            if (g >= ngroups)
                break;
            prefetch(g + kPrefetch * wtotal);
            if (g + wtotal < ngroups)
                load(g + wtotal, ca);
            place(cb);
            g += wtotal;
        }
    }
    // ---- the ragged end (< 256 rows), taken by the warp whose turn it is ------------------------------------------------------------
    if (ngroups * kGroupRows < p.nrows && ngroups % wtotal == wglobal) {
        unsigned idx[8], slots[8];
        const unsigned worst = group_rows_tail<T, ND, RING, RSTRIDE, CLAMPED, PPL, ILV>(p, p.row0 + ngroups * kGroupRows, p.row0 + p.nrows, lane, cnt, ring, idx, slots);
        __syncwarp();
        flush(false);
        if (__any_sync(0xffffffffu, worst >= (unsigned)RING))
            overflow(idx, slots);
        __syncwarp();
    }
    // ---- the incomplete last lines, then the list descriptors of every part (0 for the empty ones) and the part totals ---------
    flush(true);
#pragma unroll
    for (int k = 0; k < PPL; k++) {
        const int part = lane + 32 * k;
        if (own.cur[k] != kNone)
            p.unused[own.cur[k]] = (unsigned short)(own.wend[k] - own.wpos[k]);
        p.len[(unsigned long long)wglobal * p.nparts_pad + part] = own.total[k];
        if (own.total[k])
            atomicAdd(p.ctl + kPartTotals + part, own.total[k]);
    }
}

// ---- K2 -------------------------------------------------------------------------------------------------------------------
// The lists are laid out in the order (part, warp); CTA b takes the b-th of gridDim.x equal shares of that sequence measured in
// entries, assuming the entries of a part are spread evenly over its warps (they are: the warps take row tiles round-robin).
__global__ void __launch_bounds__(kCountThreads, 1) k_ring_count(const __grid_constant__ RingParams p) {
    extern __shared__ __align__(16) unsigned hist[];
    __shared__ unsigned long long s_part_entries[kRingParts + 1]; // exclusive prefix over parts
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int nparts = p.nparts, npad = p.nparts_pad;
    const unsigned W = p.nlists_w;
    // prefix over the part totals K1 left in the control block: one warp, lane l scans parts l and l + 32
    if (warp == 0) {
        unsigned long long a = lane < nparts ? p.ctl[kPartTotals + lane] : 0, b = lane + 32 < nparts ? p.ctl[kPartTotals + lane + 32] : 0;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const unsigned long long ua = __shfl_up_sync(0xffffffffu, a, o), ub = __shfl_up_sync(0xffffffffu, b, o);
            if (lane >= o)
                a += ua, b += ub;
        }
        b += __shfl_sync(0xffffffffu, a, 31);
        s_part_entries[lane + 1] = a;
        s_part_entries[lane + 33] = b;
        if (lane == 0)
            s_part_entries[0] = 0;
    }
    __syncthreads();
    const unsigned long long total = s_part_entries[nparts];
    const unsigned long long lo = total * blockIdx.x / gridDim.x, hi = total * (blockIdx.x + 1) / gridDim.x;
    if (lo >= hi)
        return;
    const unsigned tc = p.tile_cells;
    const unsigned cshift = p.chunk_shift, csize = 1u << cshift;
    for (int part = 0; part < nparts; part++) {
        const unsigned long long b = s_part_entries[part], e = s_part_entries[part + 1];
        if (e <= lo || b >= hi || e == b)
            continue;
        // the warps [w0, w1) of this part whose lists fall into [lo, hi): boundaries computed identically by both neighbours
        const unsigned long long n = e - b;
        const unsigned w0 = lo <= b ? 0u : (unsigned)(((lo - b) * W) / n);
        const unsigned w1 = hi >= e ? W : (unsigned)(((hi - b) * W) / n);
        if (w0 >= w1)
            continue;
        for (int i = tid; i < (int)(tc / 4 + 1); i += kCountThreads)
            reinterpret_cast<uint4 *>(hist)[i] = make_uint4(0, 0, 0, 0);
        __syncthreads();
        for (unsigned w = w0 + warp; w < w1; w += kCountThreads / 32) {
            unsigned id = p.head[(unsigned long long)w * npad + part];
            while (id != kNone) {
                const unsigned nx = p.next[id];
                const unsigned valid = csize - p.unused[id];
                const uint4 *src = reinterpret_cast<const uint4 *>(p.pool + ((unsigned long long)id << cshift));
                // a chunk = csize/512 steps of 32 lanes x 16 entries; all loads of a chunk are issued before the first atomic
                uint4 v[8];
#pragma unroll
                for (int s = 0; s < 4; s++) {
                    const unsigned off = s * 512 + lane * kGran;
                    if (off < valid) {
                        v[2 * s] = __ldcs(src + (off >> 3));
                        v[2 * s + 1] = __ldcs(src + (off >> 3) + 1);
                    }
                }
#pragma unroll
                for (int s = 0; s < 4; s++) {
                    const unsigned off = s * 512 + lane * kGran;
                    if (off < valid) {
                        const unsigned wd[8] = {v[2 * s].x, v[2 * s].y, v[2 * s].z, v[2 * s].w, v[2 * s + 1].x, v[2 * s + 1].y, v[2 * s + 1].z, v[2 * s + 1].w};
#pragma unroll
                        for (int k = 0; k < 8; k++) {
                            atomicAdd(hist + (wd[k] & 0xffffu), 1u); // pads carry tile_cells: the spare cell, never flushed
                            atomicAdd(hist + (wd[k] >> 16), 1u);
                        }
                    }
                }
                id = nx;
            }
        }
        __syncthreads();
        for (int i = tid; i < (int)tc; i += kCountThreads) {
            const unsigned c = hist[i];
            if (c) {
                const unsigned long long cell = grid_cell(p, (unsigned)part, (unsigned)i);
                if (cell < p.cells)
                    atomicAdd(p.grid + cell, (unsigned long long)c);
            }
        }
        __syncthreads();
    }
}

// CTAs of k_ring_partition for `nrows` rows: at least ~8 groups per warp so that the per-(warp, part) partial chunks stay a small
// share of the scratch, at most two per SM
long long partition_ctas(long long nrows, int warps, int sm_count) {
    const long long ngroups = (nrows + kGroupRows - 1) / kGroupRows;
    return std::max(std::min<long long>((ngroups / 8 + warps - 1) / warps, (long long)sm_count * 2), 1ll);
}

int launch_partition(const FloatPlan &f, bool clamped, long long ctas, cudaStream_t st, const RingParams &p) {
    return with_keys(f, [&](auto t, auto nd) {
        using T = decltype(t);
        constexpr int ND = decltype(nd)::value;
        auto go = [&](auto ppl) -> int {
            constexpr int PPL = decltype(ppl)::value, WARPS = RingLayout<PPL>::kWarps;
            constexpr bool kF32 = std::is_same<T, float>::value;
            auto kern = p.interleaved ? (clamped ? k_ring_partition<T, ND, PPL, WARPS, kF32, true> : k_ring_partition<T, ND, PPL, WARPS, false, true>)
                                      : (clamped ? k_ring_partition<T, ND, PPL, WARPS, kF32, false> : k_ring_partition<T, ND, PPL, WARPS, false, false>);
            constexpr size_t dyn = RingLayout<PPL>::kPerWarp * WARPS;
            B200_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)dyn));
            kern<<<(int)ctas, WARPS * 32, dyn, st>>>(p);
            B200_CUDA(cudaGetLastError());
            return B200_OK;
        };
        return p.nparts_pad == 32 ? go(std::integral_constant<int, 1>()) : go(std::integral_constant<int, 2>());
    });
}

// ---- host side of the CLAMPED index (see bin_cell_m2_clamped) ---------------------------------------------------------------
// the reference formula, evaluated exactly like src/binners.cpp:13-57 does (IEEE double, no contraction: volatile keeps every
// intermediate rounded to double whatever the host compiler flags)
double ref_t(float v, double vmin, double scale, double bins_d) {
    volatile double d = (double)v - vmin;
    volatile double s = d * scale;
    volatile double t = s * bins_d;
    return t;
}
// cell of a non-NaN key
long long ref_cell(float v, double vmin, double scale, double bins_d, unsigned bins) {
    volatile double d = (double)v - vmin;
    volatile double s = d * scale;
    if (s < 0)
        return 1;
    if (s >= 1)
        return (long long)bins + 2;
    volatile double t = s * bins_d;
    return (long long)(int)t + 2;
}
// fp32 values in increasing order <-> integers in increasing order (-inf .. +inf, NaNs excluded)
int float_order(float f) {
    int b;
    memcpy(&b, &f, 4);
    return b >= 0 ? b : (int)(0x80000000u - (unsigned)b);
}
float order_float(int o) {
    const int b = o >= 0 ? o : (int)(0x80000000u - (unsigned)o);
    float f;
    memcpy(&f, &b, 4);
    return f;
}
// the clamp bounds of one dimension; false when the construction does not apply (then the plain index runs)
bool clamp_bounds(double vmin, double scale, double bins_d, unsigned bins, float *lo_out, float *hi_out) {
    const int omin = float_order(-INFINITY), omax = float_order(INFINITY);
    auto first_with_cell_at_least = [&](long long c) { // smallest order o in [omin, omax] with cell >= c; omax + 1 if none
        long long lo = omin, hi = (long long)omax + 1;
        while (lo < hi) {
            const long long mid = lo + (hi - lo) / 2;
            if (ref_cell(order_float((int)mid), vmin, scale, bins_d, bins) >= c)
                hi = mid;
            else
                lo = mid + 1;
        }
        return lo;
    };
    const long long o_in = first_with_cell_at_least(2), o_over = first_with_cell_at_least((long long)bins + 2);
    if (o_in <= omin || o_over > omax || o_in >= o_over)
        return false; // no underflow value, no overflow value, or no value in range
    const float lo = order_float((int)(o_in - 1)), hi = order_float((int)o_over);
    if (!(lo > -INFINITY) || !(hi < INFINITY))
        return false;
    const double tlo = ref_t(lo, vmin, scale, bins_d), thi = ref_t(hi, vmin, scale, bins_d);
    // floor(t(lo)) == -1 and floor(t(hi)) == bins: every clamped key then has -1 <= floor(t) <= bins by monotonicity
    if (!(tlo >= -1.0 && tlo < 0.0) || !(thi >= bins_d && thi < bins_d + 1.0))
        return false;
    *lo_out = lo;
    *hi_out = hi;
    return true;
}

// part == __umulhi(idx, magic) for all idx < cells?  Both sides are monotone step functions of idx, so it suffices to check the
// last index of every part and the first index of the next one.
bool magic_exact(unsigned cells, unsigned tile_cells, unsigned magic) {
    for (unsigned long long k = 0; k * tile_cells < cells; k++) {
        const unsigned long long first = k * tile_cells, last = std::min<unsigned long long>(first + tile_cells, cells) - 1;
        if ((unsigned)((first * magic) >> 32) != k || (unsigned)((last * magic) >> 32) != k)
            return false;
    }
    return true;
}

} // namespace

// Scratch (pool + list tables) lives in the slot; grown on demand.
int launch_ringcount(b200_ctx *ctx, Slot *slot, const FloatPlan &f, bool *taken) {
    *taken = false;
    const long long nrows = f.p.nrows;
    const unsigned long long cells = f.p.cells;
    RingParams p;
    memset(&p, 0, sizeof p);
    static_cast<FloatKeys &>(p) = f.p;
    for (int i = 0; i < f.nd; i++)
        p.stride_sum += p.stride[i];
    bool clamped = f.xdtype == B200_F32;
    for (int i = 0; i < f.nd && clamped; i++)
        clamped = clamp_bounds(p.vmin[i], p.scale[i], p.bins_d[i], p.bins[i], &p.clamp_lo[i], &p.clamp_hi[i]);
    // As few parts as possible (32, else 64): the ring memory of k_ring_partition scales with the parts per lane.  At either count,
    // parts interleaved by the outermost key's cell when ceil(its cells / parts) rows of the grid fit one part: a crowded
    // distribution then spreads over all parts instead of a few central ones, which both ranks the rows with fewer same-counter
    // conflicts in k_ring_partition and gives k_ring_count parts of even size.  Otherwise (a huge inner dimension) contiguous
    // ranges of the index, tile_cells nudged upwards until the one-instruction division is exact.
    const unsigned long long outer_cells = (unsigned long long)p.bins[f.nd - 1] + 3, outer_stride = p.stride[f.nd - 1];
    unsigned tile_cells = 0, magic = 0;
    int np = 32;
    bool interleaved = false;
    for (; np <= kRingParts && !tile_cells; np *= 2) {
        const unsigned long long ilv_cells = (outer_cells + np - 1) / np * outer_stride;
        if (outer_cells * outer_stride == cells && ilv_cells <= kRingTileCells) {
            tile_cells = (unsigned)ilv_cells;
            interleaved = true;
            break;
        }
        unsigned long long tcells = ((cells + np - 1) / np + 7) / 8 * 8;
        for (int tries = 0; tries < 64 && tcells <= kRingTileCells; tries++, tcells += 8) {
            const unsigned m = (unsigned)((1ull << 32) / tcells) + 1u;
            if (magic_exact((unsigned)cells, (unsigned)tcells, m)) {
                tile_cells = (unsigned)tcells;
                magic = m;
                break;
            }
        }
        if (tile_cells)
            break;
    }
    if (!tile_cells)
        return B200_OK;
    p.cells = (unsigned)cells;
    p.tile_cells = tile_cells;
    if (interleaved) {
        p.interleaved = 1;
        p.outer_stride = (unsigned)outer_stride;
        p.inner_sum = p.stride_sum - p.outer_stride;
        p.nparts = (int)std::min<unsigned long long>(np, outer_cells);
        p.nparts_pad = np;
        p.part_shift = np == 32 ? 5 : 6;
    } else {
        p.neg_tile_cells = 0u - tile_cells;
        p.magic = magic;
        p.nparts = (int)((cells + tile_cells - 1) / tile_cells);
        p.nparts_pad = p.nparts <= 32 ? 32 : 64;
    }
    p.grid = f.p.count_star;

    // batches of <= 2^30 rows (32-bit entry counts), EQUAL in size: a 2^30 + remainder split paid the fixed cost of a pass (memsets,
    // one histogram flush per SM and part) for a small second batch
    const long long nbatch = (nrows + (1ll << 30) - 1) >> 30;
    const long long batch = std::min<long long>(nrows, (((nrows + nbatch - 1) / nbatch) + 255) & ~255ll);
    const int warps = p.nparts_pad == 32 ? RingLayout<1>::kWarps : RingLayout<2>::kWarps; // per CTA of k_ring_partition
    const long long nwarps = partition_ctas(batch, warps, ctx->sm_count) * warps;
    // chunk size: about a quarter of a (warp, part) list, within 512..2048 entries
    unsigned cshift = 9;
    while (cshift < 11 && (unsigned long long)batch / ((unsigned long long)nwarps * p.nparts) >= (8ull << cshift))
        cshift++;
    p.chunk_shift = cshift;
    p.nlists_w = (unsigned)nwarps;
    // every list wastes less than one chunk, every warp less than one reservation (+ its prefetched one)
    const unsigned long long nchunks = ((unsigned long long)batch >> cshift) + (unsigned long long)nwarps * (p.nparts + 2 * kSuper) + 2 * kSuper;
    if ((nchunks << cshift) >= (1ull << 32))
        return B200_OK;
    p.nchunks_cap = (unsigned)nchunks;
    const size_t lists = (size_t)nwarps * p.nparts_pad;
    // layout: [ctl] (zeroed before every batch)  [len | unused | head | next] (written by k_ring_partition)  [pool]
    const size_t zero_end = align_up(kCtlBytes, 256), off_len = zero_end, off_unused = align_up(off_len + lists * 4, 256);
    const size_t off_head = align_up(off_unused + nchunks * 2, 256), off_next = align_up(off_head + lists * 4, 256);
    const size_t off_pool = align_up(off_next + nchunks * 4, 256);
    bool room = false;
    B200_CHECK(slot_scratch(slot, off_pool + (nchunks << cshift) * 2, &room));
    if (!room) // not enough memory for the pool: the direct RED kernel takes the call
        return B200_OK;
    char *base = static_cast<char *>(slot->scratch);
    p.ctl = reinterpret_cast<unsigned *>(base);
    p.len = reinterpret_cast<unsigned *>(base + off_len);
    p.unused = reinterpret_cast<unsigned short *>(base + off_unused);
    p.head = reinterpret_cast<unsigned *>(base + off_head);
    p.next = reinterpret_cast<unsigned *>(base + off_next);
    p.pool = reinterpret_cast<unsigned short *>(base + off_pool);
    cudaStream_t st = slot->stream;
    B200_CUDA(cudaFuncSetAttribute(k_ring_count, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)((kRingTileCells + 1) * 4)));
    const size_t hist_bytes = ((size_t)tile_cells / 4 + 1) * 16;
    // B200_RING_EVENTS=1: events around the memsets, K1 and K2 of every batch; b200_ctx_ring_times reads those of the last one
    const bool timed = env_ll("B200_RING_EVENTS", 0) == 1;
    if (timed && !slot->ring_ev[0])
        for (cudaEvent_t &e : slot->ring_ev)
            B200_CUDA(cudaEventCreate(&e));
    slot->ring_timed = timed;
    for (long long r0 = 0; r0 < nrows; r0 += batch) {
        p.row0 = r0;
        p.nrows = std::min<long long>(batch, nrows - r0);
        if (timed)
            B200_CUDA(cudaEventRecord(slot->ring_ev[0], st));
        B200_CUDA(cudaMemsetAsync(base, 0, zero_end, st));
        if (timed)
            B200_CUDA(cudaEventRecord(slot->ring_ev[1], st));
        const long long ctas = partition_ctas(p.nrows, warps, ctx->sm_count);
        B200_CHECK(launch_partition(f, clamped, ctas, st, p));
        if (timed)
            B200_CUDA(cudaEventRecord(slot->ring_ev[2], st));
        const long long w = ctas * warps;
        p.nlists_w = (unsigned)w; // the last batch may launch fewer warps; its lists are the first w rows of head[] / len[]
        k_ring_count<<<ctx->sm_count, kCountThreads, hist_bytes, st>>>(p);
        B200_CUDA(cudaGetLastError());
        if (timed)
            B200_CUDA(cudaEventRecord(slot->ring_ev[3], st));
        slot->ring_len = p.len, slot->ring_ctl = p.ctl, slot->ring_lists = (size_t)w * p.nparts_pad;
        slot->ring_rows = (uint64_t)p.nrows, slot->ring_memset_bytes = zero_end, slot->ring_chunk_entries = 1u << cshift;
    }
    *taken = true;
    return B200_OK;
}

} // namespace b200
