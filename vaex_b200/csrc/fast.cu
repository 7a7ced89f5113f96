// fast.cu — compile-time specialised binby kernels for the configurations BASELINE.json is quoted on:
//   all binners BinnerScalar over the SAME float type T (fp32 / fp64, native byte order, no masks), ND = 1..3,
//   aggregators drawn from { count(*), count(v), sum(v), sum(v^2) } over at most one value column v (fp32 / fp64).
// That covers df.count / df.sum / df.mean / df.std(binby=[...]) on float columns (configs C1, C2, C3, C5).  Everything
// else takes the descriptor-driven kernel in binby.cu; both are bit-identical on the cases they share (tests).
//
// Why a second kernel: the generic one spends several times more instructions per row on runtime dtype/op dispatch and
// 64-bit index math.  The bound that remains is the scatter itself: one RED per row per aggregator, retired by the L2 at a
// fixed chip-wide rate whatever the operand width.
//
// Load pattern: two 128-bit loads per column per step, the second one 32 lanes further on, so every warp-level LDG.128 is a
// dense 512-byte segment (fully coalesced, evict-first).
#include "binby.cuh"
#include "device_utils.cuh"

namespace b200 {

namespace {

constexpr int kThreads = 256;

template <typename T>
__device__ __forceinline__ double widen(T v);
template <>
__device__ __forceinline__ double widen<float>(float v) { return (double)v; }
template <>
__device__ __forceinline__ double widen<double>(double v) { return v; }

// R consecutive elements starting at element index i (16-byte aligned): R = 4 for float, 2 for double.  One 128-bit load per
// column and half-step whatever T (ldcs4 reads 4 doubles with two), so that both loads of a warp are dense 512-byte segments.
template <typename T>
struct Vec;
template <>
struct Vec<float> {
    static constexpr int R = 4;
    float v[4];
    __device__ __forceinline__ void load(const void *p, long long i) {
        uint4 a = __ldcs(reinterpret_cast<const uint4 *>(static_cast<const float *>(p) + i));
        v[0] = __uint_as_float(a.x), v[1] = __uint_as_float(a.y), v[2] = __uint_as_float(a.z), v[3] = __uint_as_float(a.w);
    }
};
template <>
struct Vec<double> {
    static constexpr int R = 2;
    double v[2];
    __device__ __forceinline__ void load(const void *p, long long i) {
        uint4 a = __ldcs(reinterpret_cast<const uint4 *>(static_cast<const double *>(p) + i));
        v[0] = __longlong_as_double(((long long)a.y << 32) | a.x), v[1] = __longlong_as_double(((long long)a.w << 32) | a.z);
    }
};

template <typename TV, bool SMEM>
__device__ __forceinline__ void scatter(const FastParams &p, unsigned idx, bool has_v, TV vraw, unsigned *s_count, unsigned *s_vcount, double *s_vsum,
                                        double *s_vm2) {
    if (p.count_star) {
        if (SMEM)
            atomicAdd(s_count + idx, 1u);
        else
            atomicAdd(p.count_star + idx, 1ull);
    }
    if (has_v) {
        const double v = widen<TV>(vraw);
        if (v == v) { // NaN values are skipped by count(v) / sum(v) (src/agg_count.cpp:53-57, src/agg_sum.cpp:118-121)
            if (p.vcount) {
                if (SMEM)
                    atomicAdd(s_vcount + idx, 1u);
                else
                    atomicAdd(p.vcount + idx, 1ull);
            }
            if (p.vsum)
                atomicAdd((SMEM ? s_vsum : p.vsum) + idx, v);
            if (p.vm2)
                atomicAdd((SMEM ? s_vm2 : p.vm2) + idx, v * v); // pow(v, 2)
        }
    }
}

template <typename T, int ND, typename TV, bool HASV, bool SMEM>
__global__ void __launch_bounds__(kThreads) k_binby_fast(const __grid_constant__ FastParams p) {
    extern __shared__ __align__(16) char smem[];
    unsigned *s_count = nullptr, *s_vcount = nullptr;
    double *s_vsum = nullptr, *s_vm2 = nullptr;
    if (SMEM) {
        // layout of one private copy: [vsum f64][vm2 f64][count u32][vcount u32]; `smem_copies` copies, one per warp group
        const size_t c = p.cells;
        const size_t copy_bytes = ((p.vsum ? 8 * c : 0) + (p.vm2 ? 8 * c : 0) + (p.count_star ? 4 * c : 0) + (p.vcount ? 4 * c : 0) + 15) / 16 * 16;
        for (size_t i = threadIdx.x; i < copy_bytes * p.smem_copies / 4; i += kThreads)
            reinterpret_cast<unsigned *>(smem)[i] = 0u;
        __syncthreads();
        char *base = smem + copy_bytes * ((threadIdx.x >> 5) % p.smem_copies);
        if (p.vsum) {
            s_vsum = reinterpret_cast<double *>(base);
            base += 8 * c;
        }
        if (p.vm2) {
            s_vm2 = reinterpret_cast<double *>(base);
            base += 8 * c;
        }
        if (p.count_star) {
            s_count = reinterpret_cast<unsigned *>(base);
            base += 4 * c;
        }
        if (p.vcount)
            s_vcount = reinterpret_cast<unsigned *>(base);
    }

    constexpr int R = Vec<T>::R;           // rows per 128-bit load of a binner column
    constexpr int SPAN = 32 * R;           // rows one warp-level load covers
    constexpr int ROWS_PER_WARP_STEP = 2 * SPAN;
    const int lane = threadIdx.x & 31;
    const long long warp_global = ((long long)blockIdx.x * kThreads + threadIdx.x) >> 5;
    const long long nwarps = ((long long)gridDim.x * kThreads) >> 5;
    const long long full_steps = p.nrows / ROWS_PER_WARP_STEP;

    for (long long s = warp_global; s < full_steps; s += nwarps) {
        const long long base = s * ROWS_PER_WARP_STEP + (long long)lane * R;
        Vec<T> c[ND][2];
#pragma unroll
        for (int d = 0; d < ND; d++) {
            c[d][0].load(p.x[d], base);
            c[d][1].load(p.x[d], base + SPAN);
        }
        TV vv[2][R];
        if (HASV) {
            // the value column may be wider/narrower than T: load element-wise vectors of R rows
            if (sizeof(TV) == sizeof(T)) {
                Vec<TV> a, b;
                a.load(p.v, base);
                b.load(p.v, base + SPAN);
#pragma unroll
                for (int j = 0; j < R; j++) {
                    vv[0][j] = a.v[j < Vec<TV>::R ? j : 0];
                    vv[1][j] = b.v[j < Vec<TV>::R ? j : 0];
                }
            } else {
#pragma unroll
                for (int h = 0; h < 2; h++)
#pragma unroll
                    for (int j = 0; j < R; j++)
                        vv[h][j] = __ldcs(static_cast<const TV *>(p.v) + base + h * SPAN + j);
            }
        }
#pragma unroll
        for (int h = 0; h < 2; h++) {
#pragma unroll
            for (int j = 0; j < R; j++) {
                unsigned idx = 0;
#pragma unroll
                for (int d = 0; d < ND; d++)
                    idx += bin_index(widen<T>(c[d][h].v[j]), p.vmin[d], p.scale[d], p.bins_d[d], p.bins[d]) * p.stride[d];
                scatter<TV, SMEM>(p, idx, HASV, HASV ? vv[h][j] : TV(0), s_count, s_vcount, s_vsum, s_vm2);
            }
        }
    }
    // ragged tail (< ROWS_PER_WARP_STEP rows): one row per thread of the first CTAs
    const long long tail0 = full_steps * ROWS_PER_WARP_STEP;
    for (long long i = tail0 + (long long)blockIdx.x * kThreads + threadIdx.x; i < p.nrows; i += (long long)gridDim.x * kThreads) {
        unsigned idx = 0;
#pragma unroll
        for (int d = 0; d < ND; d++)
            idx += bin_index(widen<T>(__ldcs(static_cast<const T *>(p.x[d]) + i)), p.vmin[d], p.scale[d], p.bins_d[d], p.bins[d]) * p.stride[d];
        scatter<TV, SMEM>(p, idx, HASV, HASV ? __ldcs(static_cast<const TV *>(p.v) + i) : TV(0), s_count, s_vcount, s_vsum, s_vm2);
    }

    if (SMEM) {
        __syncthreads();
        const size_t c = p.cells;
        const size_t copy_bytes = ((p.vsum ? 8 * c : 0) + (p.vm2 ? 8 * c : 0) + (p.count_star ? 4 * c : 0) + (p.vcount ? 4 * c : 0) + 15) / 16 * 16;
        for (unsigned i = threadIdx.x; i < p.cells; i += kThreads) {
            unsigned long long n0 = 0, n1 = 0;
            double a = 0, b = 0;
            for (int k = 0; k < p.smem_copies; k++) {
                char *base = smem + copy_bytes * k;
                if (p.vsum) {
                    a += reinterpret_cast<double *>(base)[i];
                    base += 8 * c;
                }
                if (p.vm2) {
                    b += reinterpret_cast<double *>(base)[i];
                    base += 8 * c;
                }
                if (p.count_star) {
                    n0 += reinterpret_cast<unsigned *>(base)[i];
                    base += 4 * c;
                }
                if (p.vcount)
                    n1 += reinterpret_cast<unsigned *>(base)[i];
            }
            if (p.count_star && n0)
                atomicAdd(p.count_star + i, n0);
            if (p.vcount && n1)
                atomicAdd(p.vcount + i, n1);
            if (p.vsum && a != 0.0)
                atomicAdd(p.vsum + i, a);
            if (p.vm2 && b != 0.0)
                atomicAdd(p.vm2 + i, b);
        }
    }
}

} // namespace

// smem > 0: f.p.smem_copies private copies of that many bytes in all
int launch_fast(b200_ctx *ctx, cudaStream_t stream, const FloatPlan &f, size_t smem) {
    return with_keys(f, [&](auto t, auto nd) {
        using T = decltype(t);
        constexpr int ND = decltype(nd)::value;
        auto go = [&](auto tv, auto hasv) {
            using TV = decltype(tv);
            constexpr bool HASV = decltype(hasv)::value;
            auto kern = smem ? k_binby_fast<T, ND, TV, HASV, true> : k_binby_fast<T, ND, TV, HASV, false>;
            return launch_persistent(ctx, stream, kern, kThreads, smem, kThreads * 2 * Vec<T>::R, f.p);
        };
        if (!f.p.v)
            return go(float(), std::false_type());
        return f.vdtype == B200_F32 ? go(float(), std::true_type()) : go(double(), std::true_type());
    });
}

} // namespace b200
