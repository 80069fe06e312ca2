// k_geo_join.cu — great-circle (haversine) distance for (lon, lat) degree POINT columns, in metres: the row-wise op
// gpl_haversine_distance, and the distance-within and nearest joins whose distance is exactly that op's f64 value for the
// row pair (haversine.cuh; geo 0.27 HaversineDistance is Point x Point only, and so is everything here).  DESIGN.md §4.15
// states the contract and the exactness argument.
//
// Index (gpl_geo_index_build): the eligible right rows (non-null, finite, |lat| <= 90, |lon| <= 360) are listed in a G x G
// grid (join_grid.cuh) over (longitude wrapped into [-180, 180), latitude).  A point is a degenerate box, so a row is in
// exactly one cell.  A cell item is one 32-byte record: lon and lat as given, cos(lat * DEG) and the row id, so an
// evaluation reads nothing else.  The wrapped longitude only chooses the cell.
//
// Window (geo_window): the cells that can hold a row within D of a left point: the latitude band [lat - delta, lat + delta]
// and, unless the band reaches a pole, the longitudes within asin(sin delta / cos lat) of the point, split in two column
// ranges when it passes +-180.  delta = D / R widened by kGeoRel and kGeoAbs; above kGeoWholeDelta the whole grid is walked.
// Every item of the window is evaluated exactly (items are points: there is no cheaper bound to filter on).
//
// Kernels: persistent warps, one lane per left point, the next tile of left points in flight while one is evaluated.
//   k_geo_within<MODE>  MODE 0 counts the rows with d <= D, MODE 1 writes (rhs, d) at the row's offsets; with Drow != NULL
//                       the matches are the rows with d == Drow[i] (the tied rows of the nearest join).
//   k_geo_nearest       windows of growing radius until the minimum found lies inside the window just walked.
// Pair lists go through pair_list and the per-row sort of join_host.cuh.
#include <math.h>

#include <algorithm>
#include <cmath>
#include <memory>

#include "common.cuh"
#include "haversine.cuh"
#include "join_grid.cuh"
#include "join_host.cuh"
#include "output.cuh"
#include "scan.cuh"

namespace gpl {

// lon, lat as given (degrees), cos(lat * DEG) and the row id: two 16-byte loads per evaluation
struct __align__(16) GeoItem {
    double lon, lat, cos_lat;
    long long row;
};

}  // namespace gpl

struct gpl_geo_index {
    gpl_ctx *ctx = nullptr;
    int64_t n_rows = 0, n_r = 0, n_items = 0, bytes = 0;
    gpl::JoinGrid jg{0.0, 0.0, 0.0, 0.0, 0};
    int32_t gx = 0, gy = 0;                  // cells in use per axis (1 when the rows share one meridian / parallel)
    double ux0 = 0.0, uy0 = 0.0, ux1 = 0.0, uy1 = 0.0;
    double r0 = 0.0;                         // first radius of the nearest search, metres: about one cell
    int32_t *cell_start = nullptr;           // g*g + 1
    gpl::GeoItem *items = nullptr;
    unsigned long long *counters = nullptr;  // [0] exact evaluations of the last pass (stats only)
};

namespace gpl {

constexpr int kGeoWarps = 8;  // warps per CTA
// The window's slack (DESIGN.md §4.15 "Exactness").  delta = (D / R)(1 + kGeoRel) + kGeoAbs radians: kGeoAbs covers the
// absolute error of a computed distance (a few 1e-15 rad, from sin of a longitude difference near 360 degrees and cos of a
// latitude near a pole) and the rounding of the window edges with a factor of about 100 to spare, kGeoRel the relative error
// of the evaluation and of sin, cos, asin and the divisions in the window with a factor above 30.
constexpr double kGeoRel = 0x1p-36;
constexpr double kGeoAbs = 1e-12;
// Above this delta (radians) the whole grid is walked.  Below it a row outside the window has a true angle > delta <= 1, where
// asin(sqrt(a)) is well conditioned (a <= 0.23 at the window's edge); rows near the antipode, where the computed distance is
// only good to about 1e-8 rad, are then at an angle near pi >> 1 and cannot come out <= D.
constexpr double kGeoWholeDelta = 1.0;
constexpr double kGeoPoleMargin = 1e-9;  // radians: a band that comes this close to a pole takes every longitude
constexpr double kGeoLonPad = 1e-9;      // degrees: rounding of the wrap and of the longitude edges (<= 360 * 2^-52)
constexpr double kHalfPi = 1.57079632679489661923;

struct GeoView {
    JoinGrid jg;
    int32_t gx, gy;
    double ux0, uy0, ux1, uy1;
    const int32_t *cell_start;
    const GeoItem *items;
};
static GeoView view_of(const gpl_geo_index *idx) {
    return GeoView{idx->jg, idx->gx, idx->gy, idx->ux0, idx->uy0, idx->ux1, idx->uy1, idx->cell_start, idx->items};
}

// rows that take part, on either side: false for a NaN or infinite coordinate (so for an empty point too)
__device__ __forceinline__ bool geo_eligible(double2 p) { return fabs(p.y) <= 90.0 && fabs(p.x) <= 360.0; }
// longitude into [-180, 180); exact for |lon| <= 360 (Sterbenz)
__device__ __forceinline__ double geo_wrap(double lon) { return lon >= 180.0 ? lon - 360.0 : (lon < -180.0 ? lon + 360.0 : lon); }

// ---- build --------------------------------------------------------------------------------------------------------------
// one thread per right row: eligibility and the degenerate box (wrapped lon, lat)
__global__ void __launch_bounds__(256) k_geo_rows(const double2 *__restrict__ xy, const uint8_t *__restrict__ valid, int64_t n,
                                                  double *__restrict__ box4, uint8_t *__restrict__ has, unsigned long long *__restrict__ ctr) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    bool ok = false;
    if (i < n) {
        const double2 p = xy[i];
        ok = bit_get(valid, i) && geo_eligible(p);
        const double wl = geo_wrap(p.x);
        box4[4 * i] = wl, box4[4 * i + 1] = p.y, box4[4 * i + 2] = wl, box4[4 * i + 3] = p.y;
        has[i] = ok ? 1 : 0;
    }
    const unsigned m = __ballot_sync(0xffffffffu, ok);
    if ((threadIdx.x & 31) == 0 && m) atomicAdd(ctr, (unsigned long long)__popc(m));
}
// cell items -> records
__global__ void __launch_bounds__(256) k_geo_items(const int32_t *__restrict__ rows, int64_t n_items, const double2 *__restrict__ xy,
                                                   GeoItem *__restrict__ items) {
    const int64_t k = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (k >= n_items) return;
    const int32_t j = rows[k];
    const double2 q = xy[j];
    items[k] = GeoItem{q.x, q.y, cos(q.y * DEG), (long long)j};  // the cos haversine_distance computes for this row
}

// ---- window --------------------------------------------------------------------------------------------------------------
// Grid rows cy0 .. cy1 and, in each, the columns cx0 .. cx1 counted without wrapping: a column index >= gx stands for
// column - gx.  cx1 - cx0 < gx always, so no cell is listed twice.  Empty when cy0 > cy1.
struct GeoWindow {
    int32_t cy0, cy1, cx0, cx1;
    bool whole;  // every cell of the grid
};
// the window of the longitudes >= east_from or <= west_to (an interval that passes +-180)
__device__ __forceinline__ void geo_split(const GeoView &v, double east_from, double west_to, GeoWindow &w) {
    const bool east = east_from <= v.ux1, west = west_to >= v.ux0;  // else that part holds no row
    const int32_t ce = jg_cell(east_from, v.jg.x0, v.jg.inv_w, v.jg.g), cw = jg_cell(west_to, v.jg.x0, v.jg.inv_w, v.jg.g);
    if (east && west) {
        // jg_cell clamps and a cell can be wider than the gap between the two parts: when they meet in cell space the
        // union is the whole row of cells, once
        if (cw >= ce) w.cx0 = 0, w.cx1 = v.gx - 1;
        else w.cx0 = ce, w.cx1 = v.gx + cw;
    } else if (east) w.cx0 = ce, w.cx1 = v.gx - 1;
    else if (west) w.cx0 = 0, w.cx1 = cw;
    else w.cy1 = w.cy0 - 1;
}
// cos1 = cos(p.y * DEG); D >= 0 or +inf
__device__ __forceinline__ GeoWindow geo_window(const GeoView &v, double2 p, double cos1, double D) {
    GeoWindow w{0, -1, 0, -1, false};
    if (v.jg.g == 0) return w;
    const double delta = (D / kMeanEarthRadius) * (1.0 + kGeoRel) + kGeoAbs;
    if (!(delta <= kGeoWholeDelta)) {
        w.cy1 = v.gy - 1, w.cx1 = v.gx - 1, w.whole = true;
        return w;
    }
    const double dlat = delta / DEG * (1.0 + kGeoRel);
    const double lat_lo = p.y - dlat, lat_hi = p.y + dlat;
    if (lat_lo > v.uy1 || lat_hi < v.uy0) return w;
    w.cy0 = jg_cell(lat_lo, v.jg.y0, v.jg.inv_h, v.jg.g), w.cy1 = jg_cell(lat_hi, v.jg.y0, v.jg.inv_h, v.jg.g);
    if (fabs(p.y) * DEG + delta >= kHalfPi - kGeoPoleMargin) {  // the cap reaches a pole: every longitude
        w.cx1 = v.gx - 1;
        return w;
    }
    const double ratio = sin(delta) / cos1 * (1.0 + kGeoRel);
    const double dlon = asin(fmin(ratio, 1.0)) / DEG * (1.0 + kGeoRel) + kGeoLonPad;  // <= 90 + pad
    const double wl = geo_wrap(p.x), lo = wl - dlon, hi = wl + dlon;
    if (lo < -180.0) geo_split(v, lo + 360.0, hi, w);
    else if (hi >= 180.0) geo_split(v, lo, hi - 360.0, w);
    else if (lo > v.ux1 || hi < v.ux0) w.cy1 = w.cy0 - 1;
    else w.cx0 = jg_cell(lo, v.jg.x0, v.jg.inv_w, v.jg.g), w.cx1 = jg_cell(hi, v.jg.x0, v.jg.inv_w, v.jg.g);
    return w;
}
// f(row, d) for every item of the window, d = haversine_distance(p, row) bit for bit; returns the number of evaluations.
// The cells of one grid row and a column range are contiguous in the item array: at most two runs per grid row.
template <class F>
__device__ __forceinline__ unsigned long long geo_walk(const GeoView &v, const GeoWindow &w, double2 p, double cos1, F &&f) {
    unsigned long long evals = 0;
    for (int32_t cy = w.cy0; cy <= w.cy1; ++cy) {
        const int64_t base = (int64_t)cy * v.jg.g;
        for (int run = 0; run < 2; ++run) {
            const int32_t a = run == 0 ? w.cx0 : 0, b = run == 0 ? min(w.cx1, v.gx - 1) : w.cx1 - v.gx;
            if (b < a) continue;
            const int32_t k1 = v.cell_start[base + b + 1];
            for (int32_t k = v.cell_start[base + a]; k < k1; ++k) {
                const double2 *rec = reinterpret_cast<const double2 *>(v.items + k);
                const double2 q = __ldg(rec), cr = __ldg(rec + 1);
                f((int32_t)__double_as_longlong(cr.y), haversine_with_cos(p, cos1, q, cr.x));
            }
            evals += (unsigned long long)(k1 - v.cell_start[base + a]);
        }
    }
    return evals;
}

// ---- query kernels ----------------------------------------------------------------------------------------------------------
// MODE 0 writes the match count of each left row.  MODE 1 writes (rhs, d) into the row's slots [off[i], off[i+1]) in the order
// found (k_sort_rows_* orders them) and adds to *bad each row whose write pass found a different number of matches than its
// count pass; both passes evaluate the same pairs with the same routine, so the host treats bad != 0 as an internal error.
template <int MODE>
__global__ void __launch_bounds__(kGeoWarps * 32) k_geo_within(GeoView v, const double2 *__restrict__ pts, const uint8_t *__restrict__ pvalid,
                                                               int64_t n, double D, const double *__restrict__ Drow, int32_t *__restrict__ cnt,
                                                               const int64_t *__restrict__ off, int32_t *__restrict__ raw_rhs,
                                                               double *__restrict__ raw_d, unsigned long long *__restrict__ ctr,
                                                               unsigned long long *__restrict__ bad) {
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const int64_t nwarps = (int64_t)gridDim.x * kGeoWarps;
    unsigned long long evals = 0;
    int64_t t0 = ((int64_t)blockIdx.x * kGeoWarps + wid) * 32;
    double2 nxt = make_double2(0.0, 0.0);
    if (t0 + lane < n) nxt = __ldcs(pts + t0 + lane);  // lane-contiguous: 512 B per warp-wide load
    for (; t0 < n; t0 += nwarps * 32) {
        const int64_t i = t0 + lane;
        const double2 p = nxt;
        if (t0 + nwarps * 32 + lane < n) nxt = __ldcs(pts + t0 + nwarps * 32 + lane);  // next tile in flight
        const double Di = (Drow && i < n) ? Drow[i] : D;
        const bool live = i < n && bit_get(pvalid, i) && geo_eligible(p) && Di >= 0.0;  // a NaN Drow: the row has no match
        int32_t got = 0;
        if (live) {
            const double cos1 = cos(p.y * DEG);
            const int64_t b = MODE == 1 ? off[i] : 0, e = MODE == 1 ? off[i + 1] : 0;
            evals += geo_walk(v, geo_window(v, p, cos1, Di), p, cos1, [&](int32_t j, double d) {
                if (!(Drow ? d == Di : d <= Di)) return;
                if (MODE == 1 && b + got < e) {
                    raw_rhs[b + got] = j;
                    if (raw_d) raw_d[b + got] = d;
                }
                ++got;
            });
        }
        if (i < n) {
            if (MODE == 0) cnt[i] = got;
            else if (got != off[i + 1] - off[i]) atomicAdd(bad, 1ULL);
        }
    }
    __syncwarp();
    evals = (unsigned long long)warp_sum((double)evals);
    if (lane == 0 && evals) atomicAdd(ctr, evals);
}

// Nearest: a window of radius Dw holds every row with computed distance <= Dw, so once the minimum U found in it is <= Dw the
// minimum, its lowest row and its ties are final.  Otherwise the next window is the one at U (which holds that row, so it is
// the last), or twice as wide when nothing was found, up to max_distance and then the whole grid.
__global__ void __launch_bounds__(kGeoWarps * 32) k_geo_nearest(GeoView v, const double2 *__restrict__ pts, const uint8_t *__restrict__ pvalid,
                                                                int64_t n, double maxd, double r0, int32_t *__restrict__ nid,
                                                                double *__restrict__ dist, int32_t *__restrict__ ntied,
                                                                unsigned long long *__restrict__ ctr) {
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const int64_t nwarps = (int64_t)gridDim.x * kGeoWarps;
    const double inf = __longlong_as_double(0x7ff0000000000000LL);
    unsigned long long evals = 0;
    int64_t t0 = ((int64_t)blockIdx.x * kGeoWarps + wid) * 32;
    double2 nxt = make_double2(0.0, 0.0);
    if (t0 + lane < n) nxt = __ldcs(pts + t0 + lane);
    for (; t0 < n; t0 += nwarps * 32) {
        const int64_t i = t0 + lane;
        const double2 p = nxt;
        if (t0 + nwarps * 32 + lane < n) nxt = __ldcs(pts + t0 + nwarps * 32 + lane);
        int32_t best = -1, ties = 0;
        double U = inf;
        if (i < n && bit_get(pvalid, i) && geo_eligible(p) && v.jg.g > 0) {
            const double cos1 = cos(p.y * DEG);
            double Dw = fmin(r0, maxd);
            for (;;) {
                best = -1, ties = 0, U = inf;
                const GeoWindow w = geo_window(v, p, cos1, Dw);
                evals += geo_walk(v, w, p, cos1, [&](int32_t j, double d) {  // a NaN distance compares false twice
                    if (d < U) U = d, best = j, ties = 1;
                    else if (d == U) best = min(best, j), ++ties;
                });
                if (U <= Dw) break;
                if (w.whole || Dw >= maxd) {  // nothing is left to look at
                    if (!(U <= maxd)) best = -1, ties = 0;
                    break;
                }
                Dw = fmin(U < inf ? U : 2.0 * Dw, maxd);
            }
        }
        if (i < n) {
            nid[i] = best;
            if (dist) dist[i] = best >= 0 ? U : nan("");
            if (ntied) ntied[i] = ties;
        }
    }
    __syncwarp();
    evals = (unsigned long long)warp_sum((double)evals);
    if (lane == 0 && evals) atomicAdd(ctr, evals);
}

// row-wise: one thread per row
__global__ void __launch_bounds__(256) k_haversine_rows(int64_t n, const double2 *__restrict__ a, const uint8_t *__restrict__ av,
                                                        const double2 *__restrict__ b, const uint8_t *__restrict__ bv, double *__restrict__ out,
                                                        uint8_t *__restrict__ out_valid) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= n) return;
    const double2 p = a[i], q = b[i];
    const bool valid = bit_get(av, i) && bit_get(bv, i) && !(isnan(p.x) && isnan(p.y)) && !(isnan(q.x) && isnan(q.y));  // null or empty
    out[i] = valid ? haversine_distance(p, q) : nan("");
    out_valid[i] = valid ? 1 : 0;
}

static int geo_grid(int64_t n) { return (int)std::max<int64_t>(1, std::min<int64_t>(ceil_div(n, kGeoWarps * 32), (int64_t)kSMs * 8)); }

static int check_geo_left(const gpl_array *lhs, const char *join) {
    GPL_REQUIRE(lhs->type == GPL_POINT, GPL_ERR_INVALID_TYPE, "%s: the left side must be Point (found %s)", join, type_name(lhs->type));
    GPL_REQUIRE(lhs->n_geoms <= 0x7fffffffLL, GPL_ERR_UNSUPPORTED, "%s: at most 2^31 - 1 left rows per call (got %lld)", join,
                (long long)lhs->n_geoms);
    return GPL_OK;
}

// one pass of k_geo_within over the left points (device buffers).  raw_rhs == NULL: counts; else the matches at off.
static int geo_within_run(gpl_ctx *ctx, const gpl_geo_index *idx, const gpl_array *lhs, double D, const double *Drow, int32_t *cnt,
                          const int64_t *off, int32_t *raw_rhs, double *raw_d) {
    GPL_CUDA(cudaMemsetAsync(idx->counters, 0, sizeof(unsigned long long), ctx->stream));
    const int64_t n = lhs->n_geoms;
    if (n == 0) return GPL_OK;
    Scratch<unsigned long long> bad_d;
    GPL_TRY(bad_d.get(ctx, 1));
    GPL_CUDA(cudaMemsetAsync(bad_d.p, 0, sizeof(unsigned long long), ctx->stream));
    const GeoView v = view_of(idx);
    const double2 *pts = reinterpret_cast<const double2 *>(lhs->xy);
    if (raw_rhs == nullptr)
        GPL_LAUNCH(ctx, k_geo_within<0>, geo_grid(n), kGeoWarps * 32, 0, v, pts, lhs->validity, n, D, Drow, cnt, nullptr, nullptr, nullptr,
                   idx->counters, bad_d.p);
    else
        GPL_LAUNCH(ctx, k_geo_within<1>, geo_grid(n), kGeoWarps * 32, 0, v, pts, lhs->validity, n, D, Drow, nullptr, off, raw_rhs, raw_d,
                   idx->counters, bad_d.p);
    unsigned long long bad = 0;
    GPL_CUDA(cudaMemcpyAsync(&bad, bad_d.p, sizeof(bad), cudaMemcpyDeviceToHost, ctx->stream));
    GPL_CUDA(cudaStreamSynchronize(ctx->stream));  // bad_d returns to the cache when this scope ends
    GPL_REQUIRE(bad == 0, GPL_ERR_CUDA, "great-circle join: the write pass found a different number of matches than the count pass on %llu rows",
                bad);
    return GPL_OK;
}

static int geo_nearest_run(gpl_ctx *ctx, const gpl_geo_index *idx, const gpl_array *lhs, double maxd, int32_t *nid, double *dist,
                           int32_t *ntied) {
    GPL_CUDA(cudaMemsetAsync(idx->counters, 0, sizeof(unsigned long long), ctx->stream));
    const int64_t n = lhs->n_geoms;
    if (n == 0) return GPL_OK;
    GPL_LAUNCH(ctx, k_geo_nearest, geo_grid(n), kGeoWarps * 32, 0, view_of(idx), reinterpret_cast<const double2 *>(lhs->xy), lhs->validity, n,
               maxd, idx->r0, nid, dist, ntied, idx->counters);
    return GPL_OK;
}

}  // namespace gpl

using namespace gpl;

extern "C" int gpl_haversine_distance(gpl_ctx *ctx, const gpl_array *lhs, const gpl_array *rhs, double *out, uint8_t *out_validity, int mem) {
    GPL_REQUIRE(ctx && lhs && rhs && out, GPL_ERR_INVALID_ARG, "gpl_haversine_distance: NULL argument");
    GPL_TRY(check_mem(mem, "gpl_haversine_distance"));
    GPL_REQUIRE(lhs->type == GPL_POINT && rhs->type == GPL_POINT, GPL_ERR_INVALID_TYPE,
                "haversine_distance: both sides must be Point (found %s x %s)", type_name(lhs->type), type_name(rhs->type));
    GPL_TRY(require_same_length(lhs, rhs, "haversine_distance"));
    GPL_CUDA(cudaSetDevice(ctx->device));
    const int64_t n = lhs->n_geoms;
    if (n == 0) return GPL_OK;
    RowOut<double> res;
    ValidOut valid;
    GPL_TRY(res.get(ctx, out, n, mem));
    GPL_TRY(valid.get(ctx, out_validity, n, mem, true));
    GPL_LAUNCH(ctx, k_haversine_rows, (int)ceil_div(n, 256), 256, 0, n, reinterpret_cast<const double2 *>(lhs->xy), lhs->validity,
               reinterpret_cast<const double2 *>(rhs->xy), rhs->validity, res.p, valid.p);
    GPL_TRY(valid.deliver(ctx));
    return res.deliver(ctx);
}

extern "C" void gpl_geo_index_free(gpl_geo_index *idx) {
    if (!idx) return;
    gpl_ctx *ctx = idx->ctx;
    ctx->release(idx->cell_start);
    ctx->release(idx->items);
    ctx->release(idx->counters);
    delete idx;
}

extern "C" int gpl_geo_index_build(gpl_ctx *ctx, const gpl_array *rhs, gpl_geo_index **out) {
    GPL_REQUIRE(ctx && rhs && out, GPL_ERR_INVALID_ARG, "gpl_geo_index_build: NULL argument");
    GPL_REQUIRE(rhs->type == GPL_POINT, GPL_ERR_INVALID_TYPE, "great-circle join: the right side must be Point (found %s)",
                type_name(rhs->type));
    GPL_REQUIRE(rhs->n_geoms <= 0x7fffffffLL, GPL_ERR_UNSUPPORTED, "great-circle join: at most 2^31 - 1 right rows (got %lld)",
                (long long)rhs->n_geoms);
    GPL_CUDA(cudaSetDevice(ctx->device));
    // freed on every early return; released to the caller at the end
    std::unique_ptr<gpl_geo_index, void (*)(gpl_geo_index *)> idx(new gpl_geo_index(), gpl_geo_index_free);
    idx->ctx = ctx;
    const int64_t n = idx->n_rows = rhs->n_geoms;
    Scratch<unsigned long long> counters;
    GPL_TRY(counters.get(ctx, 2));
    idx->counters = counters.take();
    GPL_CUDA(cudaMemsetAsync(idx->counters, 0, 2 * sizeof(unsigned long long), ctx->stream));
    size_t bytes = 2 * sizeof(unsigned long long);
    if (n > 0) {
        const double2 *xy = reinterpret_cast<const double2 *>(rhs->xy);
        Scratch<double> box4;
        Scratch<uint8_t> has;
        GPL_TRY(box4.get(ctx, (size_t)n * 4));
        GPL_TRY(has.get(ctx, (size_t)n));
        GPL_LAUNCH(ctx, k_geo_rows, (int)ceil_div(n, 256), 256, 0, xy, rhs->validity, n, box4.p, has.p, idx->counters + 1);
        unsigned long long n_r = 0;
        GPL_CUDA(cudaMemcpyAsync(&n_r, idx->counters + 1, sizeof(n_r), cudaMemcpyDeviceToHost, ctx->stream));
        GPL_CUDA(cudaStreamSynchronize(ctx->stream));
        idx->n_r = (int64_t)n_r;
        if (n_r > 0) {
            GridBuild grid;
            GPL_TRY(join_grid_build(ctx, box4.p, has.p, n, idx->n_r, "great-circle join", grid));
            const JoinGrid &jg = idx->jg = grid.jg;
            idx->ux0 = grid.ux0, idx->uy0 = grid.uy0, idx->ux1 = grid.ux1, idx->uy1 = grid.uy1;
            // rows on one meridian (parallel) map every longitude (latitude) to cell 0: one column (row) of cells
            idx->gx = jg.inv_w == 0.0 ? 1 : jg.g;
            idx->gy = jg.inv_h == 0.0 ? 1 : jg.g;
            // the wider side of a cell, as metres along a meridian; a grid of one cell is walked whole at once
            const double cell_deg = std::max(idx->gx > 1 ? (idx->ux1 - idx->ux0) / jg.g : 0.0, idx->gy > 1 ? (idx->uy1 - idx->uy0) / jg.g : 0.0);
            idx->r0 = cell_deg > 0.0 ? cell_deg * DEG * kMeanEarthRadius : HUGE_VAL;
            const int64_t n_items = idx->n_items = grid.n_items;
            idx->cell_start = grid.cell_start.take();
            Scratch<GeoItem> items;
            GPL_TRY(items.get(ctx, (size_t)n_items + 1));
            idx->items = items.take();
            bytes += sizeof(int32_t) * ((size_t)jg.g * jg.g + 1) + sizeof(GeoItem) * (size_t)n_items;
            if (n_items > 0) GPL_LAUNCH(ctx, k_geo_items, (int)ceil_div(n_items, 256), 256, 0, grid.items.p, n_items, xy, idx->items);
            GPL_CUDA(cudaStreamSynchronize(ctx->stream));  // grid.items returns to the cache when this scope ends
        }
    }
    idx->bytes = (int64_t)bytes;
    GPL_CUDA(cudaStreamSynchronize(ctx->stream));
    *out = idx.release();
    return GPL_OK;
}

extern "C" int gpl_geo_index_stats(gpl_ctx *ctx, const gpl_geo_index *idx, int64_t *out8) {
    GPL_REQUIRE(ctx && idx && out8, GPL_ERR_INVALID_ARG, "gpl_geo_index_stats: NULL argument");
    GPL_CUDA(cudaSetDevice(ctx->device));
    unsigned long long evals = 0;
    GPL_CUDA(cudaMemcpyAsync(&evals, idx->counters, sizeof(evals), cudaMemcpyDeviceToHost, ctx->stream));
    GPL_CUDA(cudaStreamSynchronize(ctx->stream));
    out8[0] = idx->n_r;
    out8[1] = idx->n_rows - idx->n_r;
    out8[2] = idx->jg.g;
    out8[3] = idx->gx;
    out8[4] = idx->gy;
    out8[5] = idx->n_items;
    out8[6] = idx->bytes;
    out8[7] = (int64_t)evals;
    return GPL_OK;
}

static int check_geo_distance(double D) {
    GPL_REQUIRE(std::isfinite(D) && D >= 0.0, GPL_ERR_INVALID_ARG, "great-circle dwithin join: distance must be finite and >= 0 (got %g)", D);
    return GPL_OK;
}
static int check_geo_max_distance(double maxd) {
    GPL_REQUIRE(maxd >= 0.0, GPL_ERR_INVALID_ARG, "great-circle nearest join: max_distance must be >= 0 or +inf (got %g)", maxd);
    return GPL_OK;
}

extern "C" int gpl_geo_dwithin_count(gpl_ctx *ctx, const gpl_geo_index *idx, const gpl_array *lhs, double distance, int32_t *count, int mem) {
    GPL_REQUIRE(ctx && idx && lhs && (count || lhs->n_geoms == 0), GPL_ERR_INVALID_ARG, "gpl_geo_dwithin_count: NULL argument");
    GPL_TRY(check_mem(mem, "gpl_geo_dwithin_count"));
    GPL_TRY(check_geo_left(lhs, "great-circle dwithin join"));
    GPL_TRY(check_geo_distance(distance));
    GPL_CUDA(cudaSetDevice(ctx->device));
    RowOut<int32_t> res;
    GPL_TRY(res.get(ctx, count, lhs->n_geoms, mem));
    GPL_TRY(geo_within_run(ctx, idx, lhs, distance, nullptr, res.p, nullptr, nullptr, nullptr));
    return res.deliver(ctx);
}

extern "C" int gpl_geo_dwithin_join_pairs(gpl_ctx *ctx, const gpl_geo_index *idx, const gpl_array *lhs, double distance, int with_distance,
                                          gpl_pairs **out) {
    GPL_REQUIRE(ctx && idx && lhs && out, GPL_ERR_INVALID_ARG, "gpl_geo_dwithin_join_pairs: NULL argument");
    *out = nullptr;
    GPL_TRY(check_geo_left(lhs, "great-circle dwithin join"));
    GPL_TRY(check_geo_distance(distance));
    GPL_CUDA(cudaSetDevice(ctx->device));
    auto count = [&](int32_t *cnt) { return geo_within_run(ctx, idx, lhs, distance, nullptr, cnt, nullptr, nullptr, nullptr); };
    auto write = [&](const int64_t *off, int32_t *raw, double *raw_d) {
        return geo_within_run(ctx, idx, lhs, distance, nullptr, nullptr, off, raw, raw_d);
    };
    return pair_list(ctx, lhs->n_geoms, with_distance != 0, out, count, write);
}

extern "C" int gpl_geo_nearest_join(gpl_ctx *ctx, const gpl_geo_index *idx, const gpl_array *lhs, double max_distance, int32_t *nearest_id,
                                    double *distance, int32_t *n_tied, int mem) {
    GPL_REQUIRE(ctx && idx && lhs && (nearest_id || lhs->n_geoms == 0), GPL_ERR_INVALID_ARG, "gpl_geo_nearest_join: NULL argument");
    GPL_TRY(check_mem(mem, "gpl_geo_nearest_join"));
    GPL_TRY(check_geo_left(lhs, "great-circle nearest join"));
    GPL_TRY(check_geo_max_distance(max_distance));
    GPL_CUDA(cudaSetDevice(ctx->device));
    return dense_outputs(ctx, lhs->n_geoms, mem, nearest_id, distance, n_tied, [&](int32_t *nid, double *dist, int32_t *ntied) {
        return geo_nearest_run(ctx, idx, lhs, max_distance, nid, dist, ntied);
    });
}

extern "C" int gpl_geo_nearest_join_pairs(gpl_ctx *ctx, const gpl_geo_index *idx, const gpl_array *lhs, double max_distance, gpl_pairs **out,
                                          double *distance, int mem) {
    GPL_REQUIRE(ctx && idx && lhs && out, GPL_ERR_INVALID_ARG, "gpl_geo_nearest_join_pairs: NULL argument");
    *out = nullptr;
    GPL_TRY(check_mem(mem, "gpl_geo_nearest_join_pairs"));
    GPL_TRY(check_geo_left(lhs, "great-circle nearest join"));
    GPL_TRY(check_geo_max_distance(max_distance));
    GPL_CUDA(cudaSetDevice(ctx->device));
    const int64_t n = lhs->n_geoms;
    Scratch<int32_t> ids;
    Scratch<double> dist;  // the dense distance: the write pass collects the rows at exactly that distance
    auto count = [&](int32_t *cnt) -> int {
        GPL_TRY(ids.get(ctx, (size_t)n));
        GPL_TRY(dist.get(ctx, (size_t)n));
        GPL_TRY(geo_nearest_run(ctx, idx, lhs, max_distance, ids.p, dist.p, cnt));
        if (distance) GPL_TRY(deliver(ctx, distance, dist.p, sizeof(double) * (size_t)n, mem));
        return GPL_OK;
    };
    auto write = [&](const int64_t *off, int32_t *raw, double *) {
        return geo_within_run(ctx, idx, lhs, 0.0, dist.p, nullptr, off, raw, nullptr);
    };
    return pair_list(ctx, n, false, out, count, write);
}
