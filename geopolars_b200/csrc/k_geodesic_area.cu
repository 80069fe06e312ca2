// k_geodesic_area.cu — geo 0.27 GeodesicArea (geodesic_area_signed / geodesic_area_unsigned / geodesic_perimeter, recalled) for
// (lon, lat) degree columns on WGS84: Karney's polygon area (arXiv:1109.4448 §6) through geographiclib's PolygonArea.  Each
// ring is PolygonArea over its vertices with the closing edge always added; the edge terms S12 are summed in double-double
// with the prime-meridian transits and the sum is reduced modulo the ellipsoid's area (reduceArea).  DESIGN.md §4.17.
//
// Two passes, because the per-edge inverse solve costs thousands of FP64 operations and a variable number of Newton steps:
//   k_geodesic_edges  one thread per edge of every ring of the column: s12, S12 and the transit (-1, 0, 1) to scratch
//                     (17 B per edge); an edge with a non-finite endpoint or |lat| > 90 gets s12 = NaN, which nulls its row.
//   k_geodesic_rows   one warp per row: lanes stride over each ring's edges, every lane keeps a double-double, the lanes are
//                     combined in a fixed tree and lane 0 reduces the ring and combines rings and polygons.  A closed ring
//                     leaves out its zero-length closing edge, so it sums exactly what the same ring unclosed sums.
// A row's result depends only on its own edges (the lane of an edge is its index within the ring modulo 32), never on the
// launch grid or on the other rows of the call.
#include <math.h>

#include "common.cuh"
#include "geodesic.cuh"
#include "output.cuh"

namespace gpl {

// edges per pass: the scratch of one pass is at most 17 B * kMaxEdgesPerPass (1.1 GiB); larger columns run in row chunks
constexpr int64_t kMaxEdgesPerPass = 1LL << 26;

/* geographiclib AngNormalize: x reduced to [-180, 180] */
__device__ __forceinline__ double kang_normalize(double x) {
    double y = remainder(x, 360.0);
    return fabs(y) == 180.0 ? copysign(180.0, x) : y;
}
/* PolygonArea transit: 1 or -1 when the edge lon1 -> lon2 crosses the prime meridian eastwards or westwards, else 0 */
__device__ __forceinline__ int ktransit(double lon1, double lon2) {
    double e, lon12 = kang_diff(lon1, lon2, &e);
    lon1 = kang_normalize(lon1);
    lon2 = kang_normalize(lon2);
    return lon12 > 0 && ((lon1 < 0 && lon2 >= 0) || (lon1 > 0 && lon2 == 0)) ? 1 : (lon12 < 0 && lon1 >= 0 && lon2 < 0 ? -1 : 0);
}

/* geographiclib Accumulator: s = s[0] + s[1] exactly representable sums (Shewchuk) */
struct dd_t {
    double hi, lo;
};
__device__ __forceinline__ void dd_add(dd_t &s, double y) {
    double u, z = ksum(y, s.lo, &u);
    s.hi = ksum(z, s.hi, &s.lo);
    if (s.hi == 0) s.hi = u;
    else s.lo = s.lo + u;
}
__device__ __forceinline__ void dd_add(dd_t &s, dd_t t) {
    dd_add(s, t.hi);
    dd_add(s, t.lo);
}

/* PolygonArea reduceArea: the clockwise sum reduced modulo area0, half an area0 added for an odd transit count, converted to
 * counter-clockwise positive unless `reverse`; signed: (-area0/2, area0/2], unsigned: [0, area0) */
__device__ __forceinline__ double kreduce_area(dd_t a, int crossings, bool reverse, bool sign, double area0) {
    a.hi = remainder(a.hi, area0);
    dd_add(a, 0.0);
    if (crossings & 1) dd_add(a, (a.hi < 0 ? 1 : -1) * area0 / 2);
    if (!reverse) a.hi = -a.hi, a.lo = -a.lo;
    if (sign) {
        if (a.hi > area0 / 2) dd_add(a, -area0);
        else if (a.hi <= -area0 / 2) dd_add(a, area0);
    } else {
        if (a.hi >= area0) dd_add(a, -area0);
        else if (a.hi < 0) dd_add(a, area0);
    }
    return 0.0 + a.hi;
}

__global__ void __launch_bounds__(128) k_geodesic_edges(const double2 *__restrict__ xy, const int64_t *__restrict__ ring_off, int64_t r0,
                                                        int64_t r1, int64_t c0, int64_t c1, double *__restrict__ s12_out,
                                                        double *__restrict__ S12_out, int8_t *__restrict__ transit_out) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = c0 + blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < c1; i += stride) {
        int64_t lo = r0, hi = r1 - 1; /* the last ring r with ring_off[r] <= i (empty rings share their start with the next) */
        while (lo < hi) {
            const int64_t mid = (lo + hi + 1) >> 1;
            if (ring_off[mid] <= i) lo = mid;
            else hi = mid - 1;
        }
        const int64_t j = i + 1 < ring_off[lo + 1] ? i + 1 : ring_off[lo];
        const double2 p = xy[i], q = xy[j];
        double s12 = nan(""), S12 = 0.0;
        int tr = 0;
        if (isfinite(p.x) && isfinite(p.y) && isfinite(q.x) && isfinite(q.y) && fabs(p.y) <= 90.0 && fabs(q.y) <= 90.0) {
            s12 = karney_inverse(p, q, &S12);
            tr = ktransit(p.x, q.x);
        }
        s12_out[i - c0] = s12;
        S12_out[i - c0] = S12;
        transit_out[i - c0] = (int8_t)tr;
    }
}

/* one ring's (area, perimeter) from its edges [e0, e1) of the scratch; the result is valid in lane 0 */
__device__ __forceinline__ void ring_area(const double *__restrict__ s12, const double *__restrict__ S12, const int8_t *__restrict__ tr,
                                          int64_t e0, int64_t e1, int lane, bool reverse, bool sign, double area0, double &area,
                                          double &perimeter, bool &ok) {
    dd_t A = {0.0, 0.0}, P = {0.0, 0.0};
    int cross = 0;
    for (int64_t e = e0 + lane; e < e1; e += 32) {
        const double s = s12[e];
        if (isnan(s)) ok = false;
        dd_add(P, s);
        dd_add(A, S12[e]);
        cross += tr[e];
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        dd_t a2, p2;
        a2.hi = __shfl_down_sync(0xffffffffu, A.hi, o), a2.lo = __shfl_down_sync(0xffffffffu, A.lo, o);
        p2.hi = __shfl_down_sync(0xffffffffu, P.hi, o), p2.lo = __shfl_down_sync(0xffffffffu, P.lo, o);
        cross += __shfl_down_sync(0xffffffffu, cross, o);
        if (lane < o) dd_add(A, a2), dd_add(P, p2);
    }
    if (e1 - e0 < 2) { /* PolygonArea of fewer than 2 points: 0 */
        area = 0.0, perimeter = 0.0;
        return;
    }
    area = kreduce_area(A, cross, reverse, sign, area0);
    perimeter = 0.0 + P.hi;
}

/* the edges of ring r in the scratch.  A closed ring (last coordinate == first) leaves out its last edge, the zero-length one
 * from the repeated vertex back to the first: adding a zero to a lane's double-double can renormalise it and move the result
 * by an ulp, and without that edge a closed ring and the same ring unclosed sum the same edges in the same lanes */
__device__ __forceinline__ void ring_edges(const double2 *__restrict__ xy, const int64_t *__restrict__ ring_off, int64_t r, int64_t c0,
                                           int64_t &e0, int64_t &e1) {
    const int64_t k0 = ring_off[r], k1 = ring_off[r + 1];
    e0 = k0 - c0, e1 = k1 - c0;
    if (k1 - k0 >= 2) {
        const double2 a = xy[k0], b = xy[k1 - 1];
        if (a.x == b.x && a.y == b.y) e1 -= 1;
    }
}

/* geo's geodesic_area for one polygon (rings [q0, q1)): exterior counter-clockwise positive, holes clockwise positive and
 * combined by magnitude; perimeter over every ring */
__device__ __forceinline__ void polygon_area(const double2 *__restrict__ xy, const int64_t *__restrict__ ring_off, int64_t c0, int64_t q0,
                                             int64_t q1, const double *s12, const double *S12, const int8_t *tr, int lane, bool sign,
                                             double area0, double &area, double &perimeter, bool &ok) {
    area = 0.0, perimeter = 0.0;
    if (q1 <= q0) return;
    double outer, holes = 0.0, per;
    int64_t e0, e1;
    ring_edges(xy, ring_off, q0, c0, e0, e1);
    ring_area(s12, S12, tr, e0, e1, lane, false, sign, area0, outer, perimeter, ok);
    for (int64_t r = q0 + 1; r < q1; ++r) {
        double h;
        ring_edges(xy, ring_off, r, c0, e0, e1);
        ring_area(s12, S12, tr, e0, e1, lane, true, sign, area0, h, per, ok);
        holes += fabs(h);
        perimeter += per;
    }
    if (outer < 0.0 && holes > 0.0) holes = -holes;
    area = outer - holes;
}

/* rows [g0, g1) of a Polygon / MultiPolygon column; the scratch holds the edges from coordinate c0 on */
__global__ void __launch_bounds__(128) k_geodesic_rows(int type, int64_t g0, int64_t g1, const double2 *__restrict__ xy,
                                                       const int64_t *__restrict__ geom_off,
                                                       const int64_t *__restrict__ part_off, const int64_t *__restrict__ ring_off,
                                                       const uint8_t *__restrict__ validity, int64_t c0, const double *__restrict__ s12,
                                                       const double *__restrict__ S12, const int8_t *__restrict__ tr, int sign,
                                                       double *__restrict__ area_out, double *__restrict__ perim_out,
                                                       uint8_t *__restrict__ valid_out) {
    const int lane = threadIdx.x & 31;
    const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    const double area0 = 4 * kPi * [] {
        const kg_t G = kwgs84();
        return kc2(&G);
    }();
    for (int64_t g = g0 + ((blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5); g < g1; g += nwarps) {
        double a = 0.0, p = 0.0;
        bool ok = true;
        if (type == GPL_POLYGON) {
            polygon_area(xy, ring_off, c0, geom_off[g], geom_off[g + 1], s12, S12, tr, lane, sign != 0, area0, a, p, ok);
        } else {
            for (int64_t k = geom_off[g]; k < geom_off[g + 1]; ++k) {
                double ak, pk;
                polygon_area(xy, ring_off, c0, part_off[k], part_off[k + 1], s12, S12, tr, lane, sign != 0, area0, ak, pk, ok);
                a += ak, p += pk;
            }
        }
        ok = __all_sync(0xffffffffu, ok) && bit_get(validity, g);
        if (lane == 0) {
            if (area_out) area_out[g] = ok ? a : nan("");
            if (perim_out) perim_out[g] = ok ? p : nan("");
            valid_out[g] = ok ? 1 : 0;
        }
    }
}

/* Point / LineString / MultiPoint / MultiLineString rows: area and perimeter 0 (geo's zero impls); null when the row is null or a
 * coordinate is non-finite or has |lat| > 90 */
__global__ void __launch_bounds__(128) k_geodesic_zero_rows(int type, int64_t n, const double2 *__restrict__ xy,
                                                            const int64_t *__restrict__ geom_off, const int64_t *__restrict__ ring_off,
                                                            const uint8_t *__restrict__ validity, double *__restrict__ area_out,
                                                            double *__restrict__ perim_out, uint8_t *__restrict__ valid_out) {
    const int lane = threadIdx.x & 31;
    const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t g = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5; g < n; g += nwarps) {
        int64_t k0, k1;
        if (type == GPL_POINT) k0 = g, k1 = g + 1;
        else if (type == GPL_MULTILINESTRING) k0 = ring_off[geom_off[g]], k1 = ring_off[geom_off[g + 1]];
        else k0 = geom_off[g], k1 = geom_off[g + 1];
        bool ok = true;
        for (int64_t k = k0 + lane; k < k1; k += 32) {
            const double2 c = xy[k];
            if (!(isfinite(c.x) && isfinite(c.y) && fabs(c.y) <= 90.0)) ok = false;
        }
        ok = __all_sync(0xffffffffu, ok) && bit_get(validity, g);
        if (lane == 0) {
            if (area_out) area_out[g] = ok ? 0.0 : nan("");
            if (perim_out) perim_out[g] = ok ? 0.0 : nan("");
            valid_out[g] = ok ? 1 : 0;
        }
    }
}

/* first ring and first coordinate of row g, for g in [0, n], of a Polygon / MultiPolygon column */
__global__ void k_row_starts(int type, int64_t n, const int64_t *__restrict__ geom_off, const int64_t *__restrict__ part_off,
                             const int64_t *__restrict__ ring_off, int64_t *__restrict__ first_ring, int64_t *__restrict__ first_coord) {
    for (int64_t g = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; g <= n; g += (int64_t)gridDim.x * blockDim.x) {
        const int64_t r = type == GPL_POLYGON ? geom_off[g] : part_off[geom_off[g]];
        first_ring[g] = r;
        first_coord[g] = ring_off[r];
    }
}

/* Polygon / MultiPolygon rows: the edge pass and the row pass over row chunks of at most kMaxEdgesPerPass edges (one chunk
 * unless the column is larger; a single row with more edges is a chunk of its own) */
static int geodesic_area_polygons(gpl_ctx *ctx, const gpl_array *in, int sign, double *area, double *perim, uint8_t *vb) {
    const int64_t n = in->n_geoms;
    const double2 *xy = reinterpret_cast<const double2 *>(in->xy);
    Scratch<int64_t> rs, cs;
    GPL_TRY(rs.get(ctx, (size_t)n + 1));
    GPL_TRY(cs.get(ctx, (size_t)n + 1));
    GPL_LAUNCH(ctx, k_row_starts, (int)std::min<int64_t>(ceil_div(n + 1, 256), (int64_t)kSMs * 8), 256, 0, in->type, n, in->geom_off,
               in->part_off, in->ring_off, rs.p, cs.p);
    int64_t ends[4];
    GPL_CUDA(cudaMemcpyAsync(&ends[0], rs.p, sizeof(int64_t), cudaMemcpyDeviceToHost, ctx->stream));
    GPL_CUDA(cudaMemcpyAsync(&ends[1], rs.p + n, sizeof(int64_t), cudaMemcpyDeviceToHost, ctx->stream));
    GPL_CUDA(cudaMemcpyAsync(&ends[2], cs.p, sizeof(int64_t), cudaMemcpyDeviceToHost, ctx->stream));
    GPL_CUDA(cudaMemcpyAsync(&ends[3], cs.p + n, sizeof(int64_t), cudaMemcpyDeviceToHost, ctx->stream));
    GPL_CUDA(cudaStreamSynchronize(ctx->stream));
    std::vector<int64_t> row_ring, row_coord;  // filled only when the column needs more than one pass
    if (ends[3] - ends[2] > kMaxEdgesPerPass) {
        row_ring.resize((size_t)n + 1);
        row_coord.resize((size_t)n + 1);
        GPL_CUDA(cudaMemcpyAsync(row_ring.data(), rs.p, sizeof(int64_t) * (n + 1), cudaMemcpyDeviceToHost, ctx->stream));
        GPL_CUDA(cudaMemcpyAsync(row_coord.data(), cs.p, sizeof(int64_t) * (n + 1), cudaMemcpyDeviceToHost, ctx->stream));
        GPL_CUDA(cudaStreamSynchronize(ctx->stream));
    }
    Scratch<double> s12, S12;
    Scratch<int8_t> tr;
    const size_t cap = (size_t)std::min<int64_t>(ends[3] - ends[2], kMaxEdgesPerPass);
    for (int64_t g0 = 0; g0 < n;) {
        int64_t g1 = n, r0 = ends[0], r1 = ends[1], c0 = ends[2], c1 = ends[3];
        if (!row_coord.empty()) {
            // the longest run of rows from g0 whose edges fit, at least one row
            g1 = std::upper_bound(row_coord.begin() + g0 + 1, row_coord.end(), row_coord[g0] + kMaxEdgesPerPass) - row_coord.begin() - 1;
            g1 = std::max(g1, g0 + 1);
            r0 = row_ring[g0], r1 = row_ring[g1], c0 = row_coord[g0], c1 = row_coord[g1];
        }
        const size_t edges = (size_t)(c1 - c0);
        if (s12.p == nullptr || edges > cap) {
            GPL_TRY(s12.get(ctx, std::max(edges, cap)));
            GPL_TRY(S12.get(ctx, std::max(edges, cap)));
            GPL_TRY(tr.get(ctx, std::max(edges, cap)));
        }
        if (edges > 0) {
            const int grid = (int)std::max<int64_t>(1, std::min<int64_t>(ceil_div((int64_t)edges, 128), (int64_t)kSMs * 16));
            GPL_LAUNCH(ctx, k_geodesic_edges, grid, 128, 0, xy, in->ring_off, r0, r1, c0, c1, s12.p, S12.p, tr.p);
        }
        GPL_LAUNCH(ctx, k_geodesic_rows, warp_grid(g1 - g0, 4), 128, 0, in->type, g0, g1, xy, in->geom_off, in->part_off, in->ring_off,
                   in->validity, c0, s12.p, S12.p, tr.p, sign, area, perim, vb);
        g0 = g1;
    }
    return GPL_OK;
}

}  // namespace gpl

using namespace gpl;

extern "C" int gpl_geodesic_area(gpl_ctx *ctx, const gpl_array *in, int sign, double *area, double *perimeter, uint8_t *out_validity,
                                 int mem) {
    GPL_REQUIRE(ctx && in, GPL_ERR_INVALID_ARG, "gpl_geodesic_area: NULL argument");
    GPL_REQUIRE(area || perimeter, GPL_ERR_INVALID_ARG, "gpl_geodesic_area: area and perimeter are both NULL");
    GPL_REQUIRE(sign == 0 || sign == 1, GPL_ERR_INVALID_ARG, "gpl_geodesic_area: sign must be 0 (unsigned) or 1 (signed), got %d", sign);
    GPL_TRY(check_mem(mem, "gpl_geodesic_area"));
    GPL_REQUIRE(known_type(in->type), GPL_ERR_INVALID_TYPE,
                "gpl_geodesic_area: unsupported geometry type %s", type_name(in->type));
    GPL_CUDA(cudaSetDevice(ctx->device));
    const int64_t n = in->n_geoms;
    if (n == 0) return GPL_OK;
    RowOut<double> ra, rp;
    ValidOut valid;
    GPL_TRY(ra.get(ctx, area, n, mem));
    GPL_TRY(rp.get(ctx, perimeter, n, mem));
    GPL_TRY(valid.get(ctx, out_validity, n, mem, true));
    if (is_area(in->type)) {
        GPL_TRY(geodesic_area_polygons(ctx, in, sign, ra.p, rp.p, valid.p));
    } else {
        GPL_LAUNCH(ctx, k_geodesic_zero_rows, warp_grid(n, 4), 128, 0, in->type, n, reinterpret_cast<const double2 *>(in->xy), in->geom_off,
                   in->ring_off, in->validity, ra.p, rp.p, valid.p);
    }
    GPL_TRY(valid.deliver(ctx));
    GPL_TRY(ra.deliver(ctx));
    return rp.deliver(ctx);
}
