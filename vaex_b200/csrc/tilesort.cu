// tilesort.cu — binned count/sum/sum-of-squares over grids that do not fit in the L2 (config C3: 256^3 cells x 3 aggregators
// = 417 MB of accumulators).
//
// With direct scatter every row touches up to three random 32-byte sectors of HBM (fill + write-back).  Packing the three
// accumulators of a cell into one 32-byte record (an earlier "interleaved record" variant) brought that to one sector and
// stayed bound by random sector traffic.  Here the rows of a batch are first SORTED BY GRID REGION (k_sort_partition: a
// warp-autonomous counting sort carrying {cell index u32, value f64} = 12 bytes per row), and the regions are
// then applied one after another (k_sort_apply) — the part of the grids a region covers is <= 16 MB and stays in the 50 MB
// L2, so the REDs never go to HBM and the pass is bound by the L2 request rate
// instead of random DRAM sectors.
//
// Results are identical to fast.cu / the generic kernel for the counts; fp sums differ only by atomic ordering (as they do
// between any two runs of those kernels).  Reference semantics: src/binners.cpp:13-57 (index), src/agg_count.cpp:53-57,
// src/agg_sum.cpp:98-127 (NaN values skipped).
#include <algorithm>

#include "binby.cuh"
#include "device_utils.cuh"

namespace b200 {

struct SortParams {
    FastParams f;
    long long row0, nrows;   // batch
    int shift;               // region = cell index >> shift
    int nparts;
    unsigned *bidx;          // nparts * cap cell indices (0xFFFFFFFF = padding)
    double *bval;            // nparts * cap values (only with a value column)
    unsigned long long cap;
    unsigned *cursors;       // entries reserved per region (may run past cap)
};

namespace {

constexpr int kRounds = 16;
constexpr int kWarpTile = 32 * kRounds; // rows sorted per warp at a time
constexpr int kMaxParts = 128;
constexpr int kWarps = 8;
constexpr unsigned kChunk = 512;        // bucket entries a warp reserves at a time (>= kWarpTile)
constexpr unsigned kNone = 0xFFFFFFFFu, kOver = 0xFFFFFFFEu;
constexpr unsigned long long kNone64 = ~0ull;
constexpr unsigned kPadIdx = 0xFFFFFFFFu;
constexpr int kSlice = 2048;            // bucket entries per k_sort_apply CTA: small, so that the CTAs resident at any moment
                                        // (132 x 8) span only a few regions and their cells stay in the L2

// 4 rows of a float / double column, widened to double
template <typename T>
__device__ __forceinline__ void load4(const void *p, long long i, double out[4]);
template <>
__device__ __forceinline__ void load4<float>(const void *p, long long i, double out[4]) {
    float a[4];
    ldcs4<float>(p, i, a);
    out[0] = (double)a[0], out[1] = (double)a[1], out[2] = (double)a[2], out[3] = (double)a[3];
}
template <>
__device__ __forceinline__ void load4<double>(const void *p, long long i, double out[4]) { ldcs4<double>(p, i, out); }

__device__ __forceinline__ void l2_prefetch(const void *p, unsigned bytes) {
    asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(p), "r"(bytes) : "memory");
}

template <bool HASV>
__device__ __forceinline__ void apply_row(const FastParams &f, unsigned idx, double v) {
    if (f.count_star)
        atomicAdd(f.count_star + idx, 1ull);
    if (HASV && v == v) { // NaN values are skipped (src/agg_count.cpp:53-57, src/agg_sum.cpp:118-121)
        if (f.vcount)
            atomicAdd(f.vcount + idx, 1ull);
        if (f.vsum)
            atomicAdd(f.vsum + idx, v);
        if (f.vm2)
            atomicAdd(f.vm2 + idx, v * v);
    }
}

template <bool HASV>
__host__ __device__ constexpr size_t warp_bytes() {
    return kWarpTile * sizeof(unsigned) + (HASV ? kWarpTile * sizeof(double) : 0) + kMaxParts * sizeof(unsigned long long) + 3 * kMaxParts * sizeof(unsigned);
}

template <typename T, int ND, typename TV, bool HASV, int PPL>
__global__ void __launch_bounds__(kWarps * 32, 2) k_sort_partition(const __grid_constant__ SortParams p) {
    // every warp is autonomous: sort 512 rows by region in shared memory, append each
    // segment to the region's bucket inside a chunk of kChunk entries the warp owns
    extern __shared__ __align__(16) unsigned char dyn_smem[];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    unsigned char *mine = dyn_smem + (size_t)warp * warp_bytes<HASV>();
    double *stage_val = reinterpret_cast<double *>(mine);
    unsigned char *q = mine + (HASV ? kWarpTile * sizeof(double) : 0);
    unsigned long long *dst = reinterpret_cast<unsigned long long *>(q);
    unsigned *stage_idx = reinterpret_cast<unsigned *>(q + kMaxParts * 8);
    unsigned *seg = stage_idx + kWarpTile;
    unsigned *cbase = seg + kMaxParts;
    unsigned *cused = cbase + kMaxParts;
    const FastParams &f = p.f;
    unsigned *const bidx = p.bidx;
    double *const bval = p.bval;
    const unsigned long long cap = p.cap;
    const int nparts = p.nparts, shift = p.shift;
    for (int i = lane; i < kMaxParts; i += 32) {
        seg[i] = 0;
        cbase[i] = kNone;
        cused[i] = 0;
    }
    __syncwarp();

    const long long ntiles = (p.nrows + kWarpTile - 1) / kWarpTile, nfull = p.nrows / kWarpTile;
    const long long wglobal = (long long)blockIdx.x * kWarps + warp, wtotal = (long long)gridDim.x * kWarps;
    for (long long tile = wglobal; tile < ntiles; tile += wtotal) {
        const long long tbase = p.row0 + tile * kWarpTile;
        const long long tend = min(p.row0 + p.nrows, tbase + kWarpTile);
        const int nvalid = (int)(tend - tbase);
        unsigned idxs[kRounds], packed[kRounds]; // packed: region | slot << 7; kNone = no row
        double vals[HASV ? kRounds : 1];
        // ---- 1. load, bit-exact index, rank inside (warp, region) ----------------------------------------------------------
#pragma unroll
        for (int qd = 0; qd < kRounds / 4; qd++) {
            const long long r0 = tbase + qd * 128 + lane * 4;
            double c[ND][4], vv[4] = {0, 0, 0, 0};
            if (r0 + 4 <= tend) {
#pragma unroll
                for (int d = 0; d < ND; d++)
                    load4<T>(f.x[d], r0, c[d]);
                if (HASV)
                    load4<TV>(f.v, r0, vv);
            } else {
#pragma unroll
                for (int j = 0; j < 4; j++) {
#pragma unroll
                    for (int d = 0; d < ND; d++)
                        c[d][j] = r0 + j < tend ? (double)__ldcs(static_cast<const T *>(f.x[d]) + r0 + j) : 0.0;
                    if (HASV)
                        vv[j] = r0 + j < tend ? (double)__ldcs(static_cast<const TV *>(f.v) + r0 + j) : 0.0;
                }
            }
#pragma unroll
            for (int j = 0; j < 4; j++) {
                unsigned idx = 0;
#pragma unroll
                for (int d = 0; d < ND; d++)
                    idx += bin_index(c[d][j], f.vmin[d], f.scale[d], f.bins_d[d], f.bins[d]) * f.stride[d];
                if (r0 + j < tend) {
                    const unsigned part = idx >> shift;
                    const unsigned slot = atomicAdd(seg + part, 1u);
                    idxs[qd * 4 + j] = idx;
                    packed[qd * 4 + j] = part | (slot << 7);
                } else {
                    idxs[qd * 4 + j] = 0;
                    packed[qd * 4 + j] = kNone;
                }
                if (HASV)
                    vals[qd * 4 + j] = vv[j];
            }
        }
        if (lane == 0 && tile + wtotal < nfull) {
            // pull the NEXT tile's columns into the L2 while this one is sorted (not earlier: a line prefetched a whole tile ahead
            // is evicted again before it is used): the next loads then wait for an L2 hit instead of HBM
            const long long nb = tbase + wtotal * kWarpTile;
#pragma unroll
            for (int d = 0; d < ND; d++)
                l2_prefetch(static_cast<const T *>(f.x[d]) + nb, kWarpTile * sizeof(T));
            if (HASV)
                l2_prefetch(static_cast<const TV *>(f.v) + nb, kWarpTile * sizeof(TV));
        }
        __syncwarp();
        // ---- 2. exclusive scan of the per-region counts; place each segment in the warp's current chunk --------------------
        {
            unsigned v[PPL], s = 0;
#pragma unroll
            for (int k = 0; k < PPL; k++) {
                const int i = lane * PPL + k;
                v[k] = i < nparts ? seg[i] : 0;
                s += v[k];
            }
            unsigned incl = s;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const unsigned n = __shfl_up_sync(0xffffffffu, incl, o);
                if (lane >= o)
                    incl += n;
            }
            unsigned run = incl - s;
            bool fresh[PPL];
            unsigned any = 0;
#pragma unroll
            for (int k = 0; k < PPL; k++) {
                const int i = lane * PPL + k;
                fresh[k] = i < nparts && v[k] && cbase[i] != kOver && (cbase[i] == kNone || cused[i] + v[k] > kChunk);
                any |= fresh[k];
            }
            if (__any_sync(0xffffffffu, any)) {
#pragma unroll
                for (int k = 0; k < PPL; k++) {
                    unsigned need = __ballot_sync(0xffffffffu, fresh[k]);
                    while (need) {
                        const int src = __ffs(need) - 1;
                        need &= need - 1;
                        const int part = src * PPL + k;
                        const unsigned ob = cbase[part], ou = cused[part];
                        if (ob != kNone) // pad the tail of the old chunk
                            for (unsigned e = ou + lane; e < kChunk; e += 32)
                                bidx[(unsigned long long)part * cap + ob + e] = kPadIdx;
                        unsigned nb = 0;
                        if (lane == 0) {
                            nb = atomicAdd(p.cursors + part, (unsigned)kChunk);
                            if ((unsigned long long)nb + kChunk > cap)
                                nb = kOver; // bucket exhausted: this (warp, region) applies its rows directly from now on
                        }
                        nb = __shfl_sync(0xffffffffu, nb, 0);
                        __syncwarp();
                        if (lane == 0) {
                            cbase[part] = nb;
                            cused[part] = 0;
                        }
                        __syncwarp();
                    }
                }
            }
#pragma unroll
            for (int k = 0; k < PPL; k++) {
                const int i = lane * PPL + k;
                if (i < nparts) {
                    seg[i] = run;
                    unsigned long long d = kNone64;
                    if (v[k] && cbase[i] != kOver) {
                        d = (unsigned long long)i * cap + cbase[i] + cused[i] - run; // entry index of stage[0] if it belonged to region i
                        cused[i] += v[k];
                    }
                    dst[i] = d;
                }
                run += v[k];
            }
        }
        __syncwarp();
        // ---- 3. scatter the tile into the warp's stage, sorted by region ----------------------------------------------------
#pragma unroll
        for (int r = 0; r < kRounds; r++) {
            const unsigned pk = packed[r];
            if (pk != kNone) {
                const unsigned pos = seg[pk & 127u] + (pk >> 7);
                stage_idx[pos] = idxs[r];
                if (HASV)
                    stage_val[pos] = vals[r];
            }
        }
        __syncwarp();
        // ---- 4. append every segment to its bucket (consecutive lanes -> consecutive entries of one segment) ----------------
        for (int i = lane; i < nvalid; i += 32) {
            const unsigned e = stage_idx[i];
            const unsigned long long d = dst[e >> shift];
            if (d != kNone64) {
                bidx[d + i] = e;
                if (HASV)
                    bval[d + i] = stage_val[i];
            } else {
                apply_row<HASV>(f, e, HASV ? stage_val[i] : 0.0);
            }
        }
        __syncwarp();
        for (int i = lane; i < kMaxParts; i += 32)
            seg[i] = 0;
        __syncwarp();
    }
    // pad the open chunks so that every reserved chunk is completely written
    for (int part = 0; part < nparts; part++) {
        const unsigned ob = cbase[part], ou = cused[part];
        if (ob != kNone && ob != kOver)
            for (unsigned e = ou + lane; e < kChunk; e += 32)
                bidx[(unsigned long long)part * cap + ob + e] = kPadIdx;
    }
}

template <bool HASV>
__global__ void __launch_bounds__(256) k_sort_apply(const __grid_constant__ SortParams p, int nslices) {
    // CTAs are numbered region-major, so the CTAs in flight at any time work on a handful of neighbouring regions
    const int part = blockIdx.x / nslices, slice = blockIdx.x % nslices;
    unsigned long long n = p.cursors[part];
    if (n > p.cap) // chunks past cap were refused (those rows were applied directly); cap is a multiple of kChunk
        n = p.cap;
    const unsigned long long begin = (unsigned long long)slice * kSlice;
    if (begin >= n)
        return;
    const unsigned *bi = p.bidx + (unsigned long long)part * p.cap + begin;
    const double *bv = HASV ? p.bval + (unsigned long long)part * p.cap + begin : nullptr;
    const int cnt = (int)min((unsigned long long)kSlice, n - begin);
    const unsigned cells = p.f.cells;
    constexpr int kPer = kSlice / 256;
    unsigned idx[kPer];
    double val[HASV ? kPer : 1];
#pragma unroll
    for (int k = 0; k < kPer; k++) { // all loads first: 8 independent requests in flight per thread
        const int i = k * 256 + threadIdx.x;
        idx[k] = i < cnt ? __ldcs(bi + i) : kPadIdx;
        if (HASV)
            val[k] = i < cnt ? __ldcs(bv + i) : 0.0;
    }
#pragma unroll
    for (int k = 0; k < kPer; k++)
        if (idx[k] < cells) // skips chunk padding
            apply_row<HASV>(p.f, idx[k], HASV ? val[k] : 0.0);
}

int launch_partition(const FloatPlan &f, int sm_count, cudaStream_t st, const SortParams &p) {
    const long long ntiles = (p.nrows + kWarpTile * kWarps - 1) / (kWarpTile * kWarps);
    const int blocks = (int)std::min<long long>(ntiles, (long long)sm_count * 2);
    return with_keys(f, [&](auto t, auto nd) {
        using T = decltype(t);
        constexpr int ND = decltype(nd)::value;
        auto go = [&](auto tv, auto hasv) -> int {
            using TV = decltype(tv);
            constexpr bool HASV = decltype(hasv)::value;
            constexpr size_t dyn = warp_bytes<HASV>() * kWarps;
            // (the region count is 33..64 by construction, up to 128 when a region would exceed its byte budget)
            auto kern = p.nparts <= 64 ? k_sort_partition<T, ND, TV, HASV, 2> : k_sort_partition<T, ND, TV, HASV, 4>;
            B200_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)dyn));
            kern<<<blocks, kWarps * 32, dyn, st>>>(p);
            B200_CUDA(cudaGetLastError());
            return B200_OK;
        };
        if (!p.f.v)
            return go(double(), std::false_type());
        return f.vdtype == B200_F32 ? go(float(), std::true_type()) : go(double(), std::true_type());
    });
}

} // namespace

int launch_tilesort(b200_ctx *ctx, Slot *slot, const FloatPlan &f, bool *taken) {
    *taken = false;
    const FastParams &fp = f.p;
    const unsigned long long region_bytes = (unsigned long long)env_ll("B200_TILESORT_REGION_KB", 16 << 10) << 10;
    const int naggs = (fp.count_star != nullptr) + (fp.vcount != nullptr) + (fp.vsum != nullptr) + (fp.vm2 != nullptr);
    const unsigned long long cells = fp.cells;
    // regions: as few as possible (<= 64 keeps two regions per lane in the scan) with <= 16 MB of accumulators each (a third of the L2)
    int shift = 0;
    while ((((cells - 1) >> shift) + 1) > 64)
        shift++;
    if (shift > 0 && ((unsigned long long)naggs * 8ull << shift) > region_bytes && (((cells - 1) >> (shift - 1)) + 1) <= kMaxParts)
        shift--;
    if (((unsigned long long)naggs * 8ull << shift) > region_bytes * 3 / 2)
        return B200_OK;
    const int nparts = (int)(((cells - 1) >> shift) + 1);
    SortParams p;
    memset(&p, 0, sizeof p);
    p.f = fp;
    p.shift = shift;
    p.nparts = nparts;
    const long long batch = std::min<long long>(fp.nrows, 1ll << 27);
    const unsigned long long cap = (((unsigned long long)batch * 4 / nparts + 65536) + kChunk - 1) / kChunk * kChunk;
    const size_t entry = 4 + (fp.v ? 8 : 0);
    bool room = false;
    B200_CHECK(slot_scratch(slot, 4096 + (size_t)nparts * cap * entry, &room));
    if (!room) // no room for the buckets: the caller scatters directly
        return B200_OK;
    char *base = static_cast<char *>(slot->scratch);
    p.cursors = reinterpret_cast<unsigned *>(base);
    p.bval = reinterpret_cast<double *>(base + 4096); // the 8-byte entries first (alignment)
    p.bidx = reinterpret_cast<unsigned *>(base + 4096 + (fp.v ? (size_t)nparts * cap * 8 : 0));
    p.cap = cap;
    cudaStream_t st = slot->stream;
    const int nslices = (int)((cap + kSlice - 1) / kSlice);
    for (long long r0 = 0; r0 < fp.nrows; r0 += batch) {
        p.row0 = r0;
        p.nrows = std::min<long long>(batch, fp.nrows - r0);
        B200_CUDA(cudaMemsetAsync(p.cursors, 0, 4096, st));
        B200_CHECK(launch_partition(f, ctx->sm_count, st, p));
        const long long ctas = (long long)nparts * nslices;
        if (fp.v)
            k_sort_apply<true><<<(unsigned)ctas, 256, 0, st>>>(p, nslices);
        else
            k_sort_apply<false><<<(unsigned)ctas, 256, 0, st>>>(p, nslices);
        B200_CUDA(cudaGetLastError());
    }
    *taken = true;
    return B200_OK;
}

} // namespace b200
