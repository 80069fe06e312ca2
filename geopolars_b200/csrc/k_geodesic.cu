// k_geodesic.cu — GeoSeries::geodesic_length (geoseries.rs:52-58, impl :216-218; accessor docstring
// georust/geoseries.py:128-166; method names py-geopolars/src/geo.rs:64-67): length in metres of (lon, lat)
// degree geometries under three metrics:
//   haversine  geo 0.27 haversine_distance.rs (mean earth radius 6 371 008.8 m)              (recalled)
//   vincenty   geo 0.27 vincenty_distance.rs (WGS84, 1e-12 tolerance, 100 iterations; a segment that does
//              not converge — near-antipodal — makes the row null, the reference returns Err)   (recalled)
//   geodesic   Karney's inverse problem (arXiv:1109.4448) as implemented by geographiclib and its Rust port
//              geographiclib-rs that geo calls: order-6 series, Newton on alp1 with bisection fallback, astroid
//              starting guess near the antipode (geodesic.cuh, the distance-only instantiation).
// Geometry rules are euclidean_length's (exterior ring for polygons).  One warp per geometry, lanes stride
// over segments; transcendental-bound (tens to hundreds of FP64 flops and 10+ sin/cos/atan2 per segment), not
// HBM-bound.  f64 results; tolerance vs the oracle 1e-9 relative (libm vs CUDA math differ in the last ulps).
#include <math.h>

#include "common.cuh"
#include "geodesic.cuh"
#include "haversine.cuh"
#include "output.cuh"

namespace gpl {

template <int METHOD>
__device__ __forceinline__ double range_geodesic(const double2 *__restrict__ xy, int64_t c0, int64_t c1, int lane, bool &ok) {
    double s = 0.0;
    for (int64_t i = c0 + lane; i < c1 - 1; i += 32) {
        const double2 p = xy[i], q = xy[i + 1];
        double d = 0.0;
        if (METHOD == 1) d = haversine_distance(p, q);
        else if (METHOD == 2) {
            if (!vincenty_distance(p, q, &d)) ok = false, d = 0.0;
        } else d = karney_distance(p, q);
        s += d;
    }
    return s;
}
template <int METHOD>
__global__ void __launch_bounds__(128) k_geodesic_length(int type, int64_t n_geoms, const double2 *__restrict__ xy,
                                                         const int64_t *__restrict__ geom_off, const int64_t *__restrict__ part_off,
                                                         const int64_t *__restrict__ ring_off, const uint8_t *__restrict__ validity,
                                                         double *__restrict__ out, uint8_t *__restrict__ out_valid) {
    const int lane = threadIdx.x & 31;
    int64_t warp = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
    const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t g = warp; g < n_geoms; g += nwarps) {
        double s = 0.0;
        bool ok = true;
        switch (type) {
        case GPL_LINESTRING: s = range_geodesic<METHOD>(xy, geom_off[g], geom_off[g + 1], lane, ok); break;
        case GPL_MULTILINESTRING:
            for (int64_t l = geom_off[g]; l < geom_off[g + 1]; ++l) s += range_geodesic<METHOD>(xy, ring_off[l], ring_off[l + 1], lane, ok);
            break;
        case GPL_POLYGON:
            if (geom_off[g + 1] > geom_off[g]) s = range_geodesic<METHOD>(xy, ring_off[geom_off[g]], ring_off[geom_off[g] + 1], lane, ok);
            break;
        case GPL_MULTIPOLYGON:
            for (int64_t p = geom_off[g]; p < geom_off[g + 1]; ++p)
                if (part_off[p + 1] > part_off[p]) s += range_geodesic<METHOD>(xy, ring_off[part_off[p]], ring_off[part_off[p] + 1], lane, ok);
            break;
        default: break;
        }
        s = warp_sum(s);
        ok = __all_sync(0xffffffffu, ok);
        if (lane == 0) {
            out[g] = ok ? s : nan("");
            out_valid[g] = (ok && bit_get(validity, g)) ? 1 : 0;  // a null row stays null (area / length / x / y do the same)
        }
    }
}

}  // namespace gpl

using namespace gpl;

extern "C" int gpl_geodesic_length(gpl_ctx *ctx, const gpl_array *in, int method, double *out, uint8_t *out_validity, int mem) {
    GPL_REQUIRE(ctx && in && out, GPL_ERR_INVALID_ARG, "gpl_geodesic_length: NULL argument");
    GPL_REQUIRE(method >= 0 && method <= 2, GPL_ERR_INVALID_ARG,
                "Geodesic calculation method not valid. Use one of geodesic, haversine or vincenty");
    GPL_TRY(check_mem(mem, "gpl_geodesic_length"));
    GPL_CUDA(cudaSetDevice(ctx->device));
    const int64_t n = in->n_geoms;
    if (n == 0) return GPL_OK;
    RowOut<double> res;
    ValidOut valid;
    GPL_TRY(res.get(ctx, out, n, mem));
    GPL_TRY(valid.get(ctx, out_validity, n, mem, true));
    const double2 *xy = reinterpret_cast<const double2 *>(in->xy);
    const int grid = warp_grid(n, 4);
    if (method == 0) GPL_LAUNCH(ctx, k_geodesic_length<0>, grid, 128, 0, in->type, n, xy, in->geom_off, in->part_off, in->ring_off, in->validity, res.p, valid.p);
    else if (method == 1) GPL_LAUNCH(ctx, k_geodesic_length<1>, grid, 128, 0, in->type, n, xy, in->geom_off, in->part_off, in->ring_off, in->validity, res.p, valid.p);
    else GPL_LAUNCH(ctx, k_geodesic_length<2>, grid, 128, 0, in->type, n, xy, in->geom_off, in->part_off, in->ring_off, in->validity, res.p, valid.p);
    GPL_TRY(valid.deliver(ctx));
    return res.deliver(ctx);
}
