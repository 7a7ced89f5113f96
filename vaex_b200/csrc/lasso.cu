// lasso.cu — the point-in-polygon test of a lasso selection, one bool per row.
//
// Reference: SelectionLasso.evaluate (vaex/selections.py:172-201) calls vaexfast.pnpoly (src/vaexfast.cpp:1856-1874): a row is
// tested only when its squared distance to the polygon's mean is below radius^2, then by the crossing-number rule over every edge
// (i, j = i - 1).  Every operation here is the reference's, one IEEE rounding each and no FMA (__dsub_rn / __dmul_rn / __ddiv_rn /
// __dadd_rn): GCC folds pow(d, 2) into d * d, and the x86-64 build it is compared with has no FMA.
//
// Two loops over the edges (vaex_b200/selections.py picks one from the vertex count):
//   plain   every row tests every edge, in the reference's order;
//   banded  the host sorts the edges into bands of y: band b lists every edge whose [min(vy), max(vy)] meets the rows the band
//           function below maps to b.  An edge can toggle a row only when min(vy) <= ty < max(vy), and the parity does not depend on
//           the order in which the toggles come, so a row that tests only its band's edges gets the same answer bit for bit.  The
//           host assigns the edges with the same band function, so a row on a band boundary lands in a band that lists it.
// Edges are 4 doubles each (x_i, y_i, x_j, y_j), a band's edges stored together; every pointer is device memory.
#include <algorithm>
#include <string.h>

#include "common.cuh"
#include "device_utils.cuh"

namespace b200 {
namespace {

struct LassoParams {
    const double *x, *y; // nrows float64 each
    long long nrows;
    const double *edges; // 4 doubles an edge
    long long nedges;    // plain: the edges tested by every row
    const int *band_start; // banded: nbands + 1 offsets into edges
    int nbands;
    double band_lo, band_hi, band_scale; // band(ty) = clamp((int)((ty - lo) * scale), 0, nbands - 1) for lo <= ty < hi
    double meanx, meany, radius_squared;
    uint8_t *out;
};

__device__ __forceinline__ double load_f64(const double *p, long long i) { return __longlong_as_double((long long)load1_raw(p, 8, i)); }

// the crossing test of vaexfast's pnpoly for one edge
__device__ __forceinline__ bool crosses(const double *edges, long long e, double tx, double ty) {
    const double xi = load_f64(edges, 4 * e), yi = load_f64(edges, 4 * e + 1);
    const double xj = load_f64(edges, 4 * e + 2), yj = load_f64(edges, 4 * e + 3);
    if ((yi > ty) == (yj > ty))
        return false;
    return tx < __dadd_rn(__ddiv_rn(__dmul_rn(__dsub_rn(xj, xi), __dsub_rn(ty, yi)), __dsub_rn(yj, yi)), xi);
}

template <bool BANDED> __global__ void __launch_bounds__(256) k_lasso(const __grid_constant__ LassoParams p) {
    for (long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x; r < p.nrows; r += (long long)gridDim.x * blockDim.x) {
        const double tx = __longlong_as_double((long long)ldcs1_raw(p.x, 8, r));
        const double ty = __longlong_as_double((long long)ldcs1_raw(p.y, 8, r));
        const double dx = __dsub_rn(tx, p.meanx), dy = __dsub_rn(ty, p.meany);
        bool c = false;
        if (__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)) < p.radius_squared) {
            long long e0 = 0, e1 = p.nedges;
            if (BANDED) {
                e0 = e1 = 0; // outside [lo, hi) no edge can toggle
                if (ty >= p.band_lo && ty < p.band_hi) {
                    const int b = min(max((int)__dmul_rn(__dsub_rn(ty, p.band_lo), p.band_scale), 0), p.nbands - 1);
                    e0 = (long long)load1_raw(p.band_start, 4, b);
                    e1 = (long long)load1_raw(p.band_start, 4, b + 1);
                }
            }
            for (long long e = e0; e < e1; e++)
                c ^= crosses(p.edges, e, tx, ty);
        }
        store1_raw(p.out, 1, r, c);
    }
}

int lasso_blocks(b200_ctx *ctx, long long rows) {
    const long long want = (rows + 255) / 256;
    return (int)std::min<long long>(std::max<long long>(want, 1), (long long)ctx->sm_count * 16);
}

} // namespace
} // namespace b200

using namespace b200;

extern "C" int b200_lasso(b200_ctx *ctx, int slot, const double *x, const double *y, int64_t nrows, const double *edges, int64_t nedges,
                          const int32_t *band_start, int32_t nbands, double band_lo, double band_hi, double band_scale, double meanx, double meany,
                          double radius, uint8_t *out_device) {
    if (nrows < 0 || nedges < 0 || nbands < 0 || (nrows && (!x || !y || !out_device)) || (nedges && !edges) || (nbands && !band_start)) {
        set_error("b200_lasso: invalid argument (%lld rows, %lld edges, %d bands)", (long long)nrows, (long long)nedges, (int)nbands);
        return B200_ERR_INVALID;
    }
    if (!nrows)
        return B200_OK;
    Slot *sl;
    B200_CHECK(device_slot(ctx, slot, "b200_lasso", &sl));
    std::lock_guard<std::mutex> g(sl->mu);
    LassoParams p;
    memset(&p, 0, sizeof p);
    p.x = x;
    p.y = y;
    p.nrows = nrows;
    p.edges = edges;
    p.nedges = nedges;
    p.band_start = band_start;
    p.nbands = nbands;
    p.band_lo = band_lo;
    p.band_hi = band_hi;
    p.band_scale = band_scale;
    p.meanx = meanx;
    p.meany = meany;
    p.radius_squared = radius * radius; // `double radius_squared = radius*radius` (src/vaexfast.cpp:1857)
    p.out = out_device;
    if (nbands)
        k_lasso<true><<<lasso_blocks(ctx, nrows), 256, 0, sl->stream>>>(p);
    else
        k_lasso<false><<<lasso_blocks(ctx, nrows), 256, 0, sl->stream>>>(p);
    B200_CUDA(cudaGetLastError());
    return B200_OK;
}
