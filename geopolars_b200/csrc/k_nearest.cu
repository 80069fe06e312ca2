// k_nearest.cu — nearest-geometry join of a POINT column against any geometry column (GeoPandas' sjoin_nearest,
// rstar's nearest_neighbor): for each point, the right rows at the smallest distance, where the distance is exactly
// the f64 value gpl_distance returns for that row pair.  DESIGN.md §4.12 states the contract and the exactness argument.
//
// Index (gpl_nearest_index_build): every right row is classified as
//   excluded    null, no envelope (envelope_raw) or a non-finite coordinate: never matches;
//   grid        the box of ALL its coordinates (holes included) bounds its computed distance from below and the
//               distance to its first coordinate (the representative vertex) bounds it from above, both up to tau;
//   everywhere  a row with an empty member, an empty ring or a 1-coordinate linestring / ring: its computed distance
//               is not bounded by its box (0 everywhere, or geo's 1.19e-7 point rule), so every query evaluates it.
// Grid rows are listed in a G x G grid over their union box (join_grid.cuh, G = ceil(sqrt(|R|)) capped at 2048) as
// 32-byte sector records (the row's box), with the row id and the representative vertex in parallel arrays.
//
// Query (k_nearest): persistent warps, one lane per point, 32 points per tile.
//   phase 1 (per lane): a ring search around the point's cell lowers U = min(max_distance, dist(rep_j) + tau) over the
//     listed rows until the unsearched cells lie further than U + 2 tau; a second walk over the same window enqueues
//     every row with box distance lb_j <= U + tau into the warp's shared-memory queue, from the single cell that holds
//     the point of the row's box nearest to the query point (so each row is enqueued once).
//   phase 2 (whole warp): the queue is drained with the warp-cooperative routines of point_dist.cuh (Point and
//     MultiPoint rows: one lane per pair), the everywhere rows are evaluated for the tile's points without queueing,
//     and each lane reduces its own results to (min distance, lowest id, ties).
//   overflow: the queue is shared by the warp's 32 points; a lane whose push finds it full is flagged and
//     k_nearest_overflow redoes that point with one warp, streaming the candidates instead of queueing them.  A warp whose
//     points have more than 256 candidates in all therefore sends some of them there (a speed cliff, not a wrong answer).
// Pairs: the dense pass gives n_tied, a scan gives offsets, the same kernels in MODE 1 write the tied rows and
// k_nearest_sort_pairs orders each point's rows.
#include <math.h>
#include <string.h>

#include <algorithm>
#include <cmath>

#include "common.cuh"
#include "join_grid.cuh"
#include "point_dist.cuh"
#include "scan.cuh"

struct gpl_nearest_index {
    gpl_ctx *ctx = nullptr;
    int32_t type = GPL_MISSING;
    const double2 *xy = nullptr;
    const int64_t *go = nullptr, *po = nullptr, *ro = nullptr;
    int64_t n_rows = 0, n_r = 0, n_every = 0, n_items = 0, bytes = 0;
    gpl::JoinGrid jg{0.0, 0.0, 0.0, 0.0, 0};
    int32_t gx = 0, gy = 0;                                   // cells in use per axis (1 when the box has no width / height)
    double ux0 = 0.0, uy0 = 0.0, ux1 = 0.0, uy1 = 0.0, cw = 0.0, ch = 0.0, M = 0.0;
    int32_t *cell_start = nullptr;                           // g*g + 1
    double2 *recs = nullptr;                                 // 2 per item: (x0, y0), (x1, y1) of the row's box
    double2 *item_rep = nullptr;                             // representative vertex of the item's row
    int32_t *item_row = nullptr;
    int32_t *every = nullptr;                                // the everywhere rows
    unsigned long long *counters = nullptr;                  // [0] exact evaluations, [1] overflow points (last pass; shared
                                                             // by concurrent queries of this index: stats only)
};

namespace gpl {

constexpr int kNnWarps = 8;    // warps per CTA
constexpr int kNnQueue = 256;  // queued (point, row) pairs per warp

struct NearestView {
    int type;
    const double2 *xy;
    const int64_t *go, *po, *ro;
    JoinGrid jg;
    int32_t gx, gy;
    double ux0, uy0, ux1, uy1, cw, ch, M;
    const int32_t *cell_start;
    const double2 *recs, *item_rep;
    const int32_t *item_row, *every;
    int32_t n_every;
};

static NearestView view_of(const gpl_nearest_index *idx) {
    return NearestView{idx->type, idx->xy, idx->go, idx->po, idx->ro, idx->jg, idx->gx, idx->gy, idx->ux0, idx->uy0, idx->ux1, idx->uy1,
                       idx->cw, idx->ch, idx->M, idx->cell_start, idx->recs, idx->item_rep, idx->item_row, idx->every,
                       (int32_t)idx->n_every};
}

// ---- build --------------------------------------------------------------------------------------------------------------
// one thread per row: class (0 excluded, 1 grid, 2 everywhere), box of all coordinates, representative vertex
__global__ void __launch_bounds__(256) k_nearest_classify(int type, int64_t n, const double2 *__restrict__ xy, const int64_t *__restrict__ go,
                                                          const int64_t *__restrict__ po, const int64_t *__restrict__ ro,
                                                          const uint8_t *__restrict__ valid, const uint8_t *__restrict__ has_env,
                                                          double *__restrict__ box4, double2 *__restrict__ rep, uint8_t *__restrict__ cls,
                                                          uint8_t *__restrict__ grid_has, unsigned long long *__restrict__ ctr) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    uint8_t c = 0;
    if (i < n && bit_get(valid, i) && has_env[i]) {
        int64_t c0 = 0, c1 = 0;
        bool irregular = false;
        switch (type) {
        case GPL_POINT: c0 = i, c1 = i + 1; break;
        case GPL_LINESTRING:
        case GPL_MULTIPOINT:
            c0 = go[i], c1 = go[i + 1];
            irregular = type == GPL_LINESTRING && c1 - c0 < 2;
            break;
        case GPL_MULTILINESTRING:
            c0 = ro[go[i]], c1 = ro[go[i + 1]];
            for (int64_t m = go[i]; m < go[i + 1]; ++m) irregular = irregular || ro[m + 1] - ro[m] < 2;
            break;
        case GPL_POLYGON:
            c0 = ro[go[i]], c1 = ro[go[i + 1]];
            irregular = go[i + 1] <= go[i];
            for (int64_t r = go[i]; r < go[i + 1]; ++r) irregular = irregular || ro[r + 1] - ro[r] < 2;
            break;
        default:  // GPL_MULTIPOLYGON
            c0 = ro[po[go[i]]], c1 = ro[po[go[i + 1]]];
            for (int64_t q = go[i]; q < go[i + 1]; ++q) {
                irregular = irregular || po[q + 1] <= po[q];
                for (int64_t r = po[q]; r < po[q + 1]; ++r) irregular = irregular || ro[r + 1] - ro[r] < 2;
            }
            break;
        }
        const double inf = __longlong_as_double(0x7ff0000000000000LL);
        double x0 = inf, y0 = inf, x1 = -inf, y1 = -inf;
        bool finite = c1 > c0;
        for (int64_t k = c0; k < c1; ++k) {
            const double2 q = xy[k];
            finite = finite && isfinite(q.x) && isfinite(q.y);
            x0 = fmin(x0, q.x), y0 = fmin(y0, q.y), x1 = fmax(x1, q.x), y1 = fmax(y1, q.y);
        }
        if (finite) {
            c = irregular ? 2 : 1;
            box4[4 * i] = x0, box4[4 * i + 1] = y0, box4[4 * i + 2] = x1, box4[4 * i + 3] = y1;
            rep[i] = xy[c0];
        }
    }
    if (i < n) cls[i] = c, grid_has[i] = c == 1 ? 1 : 0;
    const unsigned m1 = __ballot_sync(0xffffffffu, c == 1), m2 = __ballot_sync(0xffffffffu, c == 2);
    if ((threadIdx.x & 31) == 0) {
        if (m1) atomicAdd(ctr, (unsigned long long)__popc(m1));
        if (m2) atomicAdd(ctr + 1, (unsigned long long)__popc(m2));
    }
}
// everywhere rows -> list (their order is irrelevant: every query evaluates all of them)
__global__ void k_nearest_every(const uint8_t *__restrict__ cls, int64_t n, unsigned long long *__restrict__ cursor, int32_t *__restrict__ every) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i < n && cls[i] == 2) every[atomicAdd(cursor, 1ULL)] = (int32_t)i;
}
// cell items -> sector records + parallel arrays
__global__ void k_nearest_records(const int32_t *__restrict__ items, int64_t n_items, const double *__restrict__ box4,
                                  const double2 *__restrict__ rep, double2 *__restrict__ recs, double2 *__restrict__ item_rep) {
    const int64_t k = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (k >= n_items) return;
    const int32_t j = items[k];
    recs[2 * k] = make_double2(box4[4 * j], box4[4 * j + 1]);
    recs[2 * k + 1] = make_double2(box4[4 * j + 2], box4[4 * j + 3]);
    item_rep[k] = rep[j];
}

// ---- query: shared device pieces -------------------------------------------------------------------------------------------
// exactly gpl_distance(point p, row j) (k_pairs.cu: k_point_point_dist, k_point_ls_dist, k_poly_point<1>, k_distance_multi
// with member_distance's point arms); warp cooperative except for Point / MultiPoint rows
__device__ __forceinline__ double row_distance(const NearestView &v, int64_t j, double2 p, int lane) {
    const double big = 1.7976931348623157e308;
    switch (v.type) {
    case GPL_POINT: return pt_dist(p, v.xy[j]);
    case GPL_LINESTRING: return point_ls_distance(v.xy, v.go[j], v.go[j + 1] - v.go[j], p, lane);
    case GPL_POLYGON: return point_polygon_distance(Side{GPL_POLYGON, v.xy, v.go, nullptr, v.ro}, j, p, lane);
    case GPL_MULTIPOINT: {
        double d = big;
        for (int64_t q = v.go[j]; q < v.go[j + 1]; ++q) d = fmin(d, pt_dist(p, v.xy[q]));
        return d;
    }
    case GPL_MULTILINESTRING: {
        double d = big;
        for (int64_t m = v.go[j]; m < v.go[j + 1]; ++m) d = fmin(d, point_ls_distance(v.xy, v.ro[m], v.ro[m + 1] - v.ro[m], p, lane));
        return d;
    }
    default: {  // GPL_MULTIPOLYGON: POLYGON view over the parts
        double d = big;
        const Side s{GPL_POLYGON, v.xy, v.po, nullptr, v.ro};
        for (int64_t q = v.go[j]; q < v.go[j + 1]; ++q) d = fmin(d, point_polygon_distance(s, q, p, lane));
        return d;
    }
    }
}
__device__ __forceinline__ bool lane_rows(int type) { return type == GPL_POINT || type == GPL_MULTIPOINT; }

// Euclidean distance from p to the closed box (CUDA hypot: <= 2 ulp; DESIGN.md §4.12 folds it into tau)
__device__ __forceinline__ double box_dist(double2 p, double x0, double y0, double x1, double y1) {
    return hypot(fmax(fmax(x0 - p.x, p.x - x1), 0.0), fmax(fmax(y0 - p.y, p.y - y1), 0.0));
}
__device__ __forceinline__ double slack(const NearestView &v, double2 p) {
    return 0x1p-40 * fmax(v.M, fmax(fabs(p.x), fabs(p.y)));
}
__device__ __forceinline__ int32_t cell_x(const NearestView &v, double x) { return jg_cell(x, v.jg.x0, v.jg.inv_w, v.jg.g); }
__device__ __forceinline__ int32_t cell_y(const NearestView &v, double y) { return jg_cell(y, v.jg.y0, v.jg.inv_h, v.jg.g); }

// the cells at Chebyshev distance r from (cxp, cyp) inside the used grid
template <class F>
__device__ __forceinline__ void visit_ring(const NearestView &v, int32_t cxp, int32_t cyp, int32_t r, F &&f) {
    const int32_t ylo = max(cyp - r, 0), yhi = min(cyp + r, v.gy - 1);
    for (int32_t cy = ylo; cy <= yhi; ++cy) {
        const bool full = cy == cyp - r || cy == cyp + r;
        const int32_t step = full ? 1 : 2 * r;
        for (int32_t cx = full ? cxp - r : cxp - r; cx <= cxp + r; cx += step) {
            if (cx >= 0 && cx < v.gx) f(cx, cy, (int64_t)cy * v.jg.g + cx);
        }
    }
}

// phase 1a: the ring search.  Lowers U with the upper bounds of the listed rows and returns the radius after which every
// unsearched cell lies further than U + 2 tau from p.
__device__ __forceinline__ int32_t search_radius(const NearestView &v, double2 p, double tau, int32_t cxp, int32_t cyp, double &U) {
    for (int32_t r = 0;; ++r) {
        visit_ring(v, cxp, cyp, r, [&](int32_t, int32_t, int64_t c) {
            const int32_t k1 = v.cell_start[c + 1];
            for (int32_t k = v.cell_start[c]; k < k1; ++k) {
                const double2 q = v.item_rep[k];
                U = fmin(U, hypot(q.x - p.x, q.y - p.y) + tau);
            }
        });
        // distance from p to the unsearched cells: one box per side that still has cells (cell edges ux0 + k * cw)
        const double inf = __longlong_as_double(0x7ff0000000000000LL);
        double B = inf;
        bool more = false;
        if (cxp + r + 1 < v.gx) more = true, B = fmin(B, box_dist(p, v.ux0 + (cxp + r + 1) * v.cw, v.uy0, v.ux1, v.uy1));
        if (cxp - r - 1 >= 0) more = true, B = fmin(B, box_dist(p, v.ux0, v.uy0, v.ux0 + (cxp - r) * v.cw, v.uy1));
        if (cyp + r + 1 < v.gy) more = true, B = fmin(B, box_dist(p, v.ux0, v.uy0 + (cyp + r + 1) * v.ch, v.ux1, v.uy1));
        if (cyp - r - 1 >= 0) more = true, B = fmin(B, box_dist(p, v.ux0, v.uy0, v.ux1, v.uy0 + (cyp - r) * v.ch));
        if (!more || B - 2.0 * tau > U) return r;
    }
}
// phase 1b test of item k listed in cell (cx, cy): lb <= U + tau, and this cell holds the box point nearest to p
__device__ __forceinline__ bool is_candidate(const NearestView &v, int32_t k, double2 p, double lim, int32_t cx, int32_t cy) {
    const double2 lo = v.recs[2 * (int64_t)k], hi = v.recs[2 * (int64_t)k + 1];  // one 32-byte sector
    if (!(box_dist(p, lo.x, lo.y, hi.x, hi.y) <= lim)) return false;
    return cell_x(v, fmin(fmax(p.x, lo.x), hi.x)) == cx && cell_y(v, fmin(fmax(p.y, lo.y), hi.y)) == cy;
}

// ---- query kernels ----------------------------------------------------------------------------------------------------------
// MODE 0: nearest_id / distance / n_tied per point (flag[i] = 1: left to the overflow kernel)
// MODE 1: the tied rows of each point into raw_rhs[off[i] ..off[i+1]) (unsorted)
template <int MODE>
__global__ void __launch_bounds__(kNnWarps * 32) k_nearest(NearestView v, const double2 *__restrict__ pts, const uint8_t *__restrict__ pvalid,
                                                          int64_t n, double maxd, int32_t *__restrict__ nid, double *__restrict__ dist,
                                                          int32_t *__restrict__ ntied, const int64_t *__restrict__ off,
                                                          int32_t *__restrict__ raw_rhs, uint8_t *__restrict__ flag,
                                                          unsigned long long *__restrict__ ctr) {
    __shared__ int32_t s_row[kNnWarps][kNnQueue];
    __shared__ double s_d[kNnWarps][kNnQueue];
    __shared__ uint8_t s_own[kNnWarps][kNnQueue];
    __shared__ double2 s_pt[kNnWarps][32];
    __shared__ uint8_t s_over[kNnWarps][32];
    __shared__ int s_qn[kNnWarps];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const int64_t nwarps = (int64_t)gridDim.x * kNnWarps;
    const bool grid = v.jg.g > 0;
    unsigned long long evals = 0;
    int64_t t0 = ((int64_t)blockIdx.x * kNnWarps + wid) * 32;
    double2 nxt = make_double2(0.0, 0.0);
    if (t0 + lane < n) nxt = __ldcs(pts + t0 + lane);  // lane-contiguous: 512 B per warp-wide load
    for (; t0 < n; t0 += nwarps * 32) {
        const int64_t i = t0 + lane;
        const double2 p = nxt;
        if (t0 + nwarps * 32 + lane < n) nxt = __ldcs(pts + t0 + nwarps * 32 + lane);  // next tile in flight
        const bool valid = i < n && bit_get(pvalid, i) && isfinite(p.x) && isfinite(p.y);
        if (lane == 0) s_qn[wid] = 0;
        s_pt[wid][lane] = p;
        __syncwarp();
        bool over = false;
        if (valid) {
            auto push = [&](int32_t row) {
                if (over) return;
                const int s = atomicAdd(&s_qn[wid], 1);
                if (s < kNnQueue) s_row[wid][s] = row, s_own[wid][s] = (uint8_t)lane;
                else over = true;
            };
            if (grid) {
                const double tau = slack(v, p);
                const int32_t cxp = cell_x(v, p.x), cyp = cell_y(v, p.y);
                double U = maxd;
                const int32_t rs = search_radius(v, p, tau, cxp, cyp, U);
                const double lim = U + tau;
                for (int32_t r = 0; r <= rs && !over; ++r)
                    visit_ring(v, cxp, cyp, r, [&](int32_t cx, int32_t cy, int64_t c) {
                        const int32_t k1 = v.cell_start[c + 1];
                        for (int32_t k = v.cell_start[c]; k < k1 && !over; ++k)
                            if (is_candidate(v, k, p, lim, cx, cy)) push(v.item_row[k]);
                    });
            }
        }
        s_over[wid][lane] = over ? 1 : 0;
        __syncwarp();
        const int nq = min(s_qn[wid], kNnQueue);
        // phase 2: exact distances of the queued pairs
        if (lane_rows(v.type)) {
            for (int e = lane; e < nq; e += 32) {
                const int own = s_own[wid][e];
                if (s_over[wid][own]) continue;
                s_d[wid][e] = row_distance(v, s_row[wid][e], s_pt[wid][own], lane);
                ++evals;
            }
        } else {
            for (int e = 0; e < nq; ++e) {
                const int own = s_own[wid][e];
                if (s_over[wid][own]) continue;
                const double d = row_distance(v, s_row[wid][e], s_pt[wid][own], lane);
                if (lane == 0) s_d[wid][e] = d, ++evals;
            }
        }
        __syncwarp();
        // each lane: its own entries -> (min distance <= maxd, lowest row at it, number of rows at it)
        double best = __longlong_as_double(0x7ff0000000000000LL);
        int32_t id = 0x7fffffff, cnt = 0;
        auto take = [&](double d, int32_t j) {
            if (!(d <= maxd)) return;
            if (d < best || cnt == 0) best = d, id = j, cnt = 1;
            else if (d == best) ++cnt, id = min(id, j);
        };
        // the everywhere rows, once per tile with the whole warp (never queued: they would fill the queue 32 times over)
        const unsigned live = __ballot_sync(0xffffffffu, valid && !over);
        for (int32_t e = 0; e < v.n_every; ++e) {
            const int32_t j = v.every[e];
            for (unsigned m = live; m; m &= m - 1) {
                const int l = __ffs(m) - 1;
                const double d = row_distance(v, j, s_pt[wid][l], lane);
                if (lane == l) take(d, j), ++evals;
            }
        }
        if (valid && !over) {
            for (int e = 0; e < nq; ++e)
                if (s_own[wid][e] == lane) take(s_d[wid][e], s_row[wid][e]);
        }
        if (i < n) {
            flag[i] = over ? 1 : 0;
            if (MODE == 0 && !over) {
                nid[i] = cnt ? id : -1;
                if (dist) dist[i] = cnt ? best : nan("");
                if (ntied) ntied[i] = cnt;
            }
        }
        if (MODE == 1) {
            const bool wr = i < n && cnt > 0;
            const int64_t b = wr ? off[i] : 0, cap = wr ? off[i + 1] - b : 0;
            int64_t w = 0;
            for (int e = 0; e < nq && wr; ++e)
                if (s_own[wid][e] == lane && s_d[wid][e] == best && w < cap) raw_rhs[b + w++] = s_row[wid][e];
            const unsigned tied_live = __ballot_sync(0xffffffffu, wr);
            for (int32_t e = 0; e < v.n_every && tied_live; ++e) {  // the everywhere rows at the best distance
                const int32_t j = v.every[e];
                for (unsigned m = tied_live; m; m &= m - 1) {
                    const int l = __ffs(m) - 1;
                    const double d = row_distance(v, j, s_pt[wid][l], lane);
                    if (lane == l && d == best && w < cap) raw_rhs[b + w++] = j;
                }
            }
        }
        __syncwarp();  // the queue is reused by the next tile
    }
    evals = (unsigned long long)warp_sum((double)evals);
    if (lane == 0 && evals) atomicAdd(ctr, evals);
}

// the flagged points, one warp per point: candidates are streamed, not queued.  MODE 1 writes the rows at dist_in[i].
template <int MODE>
__global__ void __launch_bounds__(256) k_nearest_overflow(NearestView v, const double2 *__restrict__ pts, int64_t n, double maxd,
                                                          const uint8_t *__restrict__ flag, int32_t *__restrict__ nid,
                                                          double *__restrict__ dist, int32_t *__restrict__ ntied,
                                                          const double *__restrict__ dist_in, const int64_t *__restrict__ off,
                                                          int32_t *__restrict__ raw_rhs, unsigned long long *__restrict__ ctr) {
    const int lane = threadIdx.x & 31;
    const int64_t warp = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5, nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    const int64_t n_blocks = (n + 31) >> 5;
    unsigned long long evals = 0, points = 0;
    for (int64_t blk = warp; blk < n_blocks; blk += nwarps) {
        unsigned todo = __ballot_sync(0xffffffffu, (blk << 5) + lane < n && flag[(blk << 5) + lane] != 0);
        while (todo) {
            const int64_t i = (blk << 5) + __ffs(todo) - 1;
            todo &= todo - 1;
            ++points;
            const double2 p = pts[i];
            double best = __longlong_as_double(0x7ff0000000000000LL);
            int32_t id = 0x7fffffff, cnt = 0;
            const double target = MODE == 1 ? dist_in[i] : 0.0;
            const int64_t b = MODE == 1 ? off[i] : 0, cap = MODE == 1 ? off[i + 1] - b : 0;
            int64_t w = 0;
            auto consider = [&](int32_t j) {  // warp-uniform
                const double d = row_distance(v, j, p, lane);
                ++evals;
                if (!(d <= maxd)) return;
                if (MODE == 0) {
                    if (d < best || cnt == 0) best = d, id = j, cnt = 1;
                    else if (d == best) ++cnt, id = min(id, j);
                } else if (d == target && w < cap) {
                    if (lane == 0) raw_rhs[b + w] = j;
                    ++w;
                }
            };
            for (int32_t e = 0; e < v.n_every; ++e) consider(v.every[e]);
            if (v.jg.g > 0) {
                const double tau = slack(v, p);
                const int32_t cxp = cell_x(v, p.x), cyp = cell_y(v, p.y);
                double U = maxd;
                const int32_t rs = search_radius(v, p, tau, cxp, cyp, U);
                const double lim = U + tau;
                for (int32_t r = 0; r <= rs; ++r)
                    visit_ring(v, cxp, cyp, r, [&](int32_t cx, int32_t cy, int64_t c) {
                        const int32_t k0 = v.cell_start[c], k1 = v.cell_start[c + 1];
                        for (int32_t kb = k0; kb < k1; kb += 32) {
                            const int32_t k = kb + lane;
                            const bool cand = k < k1 && is_candidate(v, k, p, lim, cx, cy);
                            const int32_t row = cand ? v.item_row[k] : 0;
                            unsigned m = __ballot_sync(0xffffffffu, cand);
                            while (m) {
                                const int src = __ffs(m) - 1;
                                m &= m - 1;
                                consider(__shfl_sync(0xffffffffu, row, src));
                            }
                        }
                    });
            }
            if (MODE == 0 && lane == 0) {
                nid[i] = cnt ? id : -1;
                if (dist) dist[i] = cnt ? best : nan("");
                if (ntied) ntied[i] = cnt;
            }
        }
    }
    if (lane == 0 && (evals || points)) {
        atomicAdd(ctr, evals);
        atomicAdd(ctr + 1, points);
    }
}

// each point's tied rows in ascending order: rank sort of the segment (rows of a point are distinct)
__global__ void __launch_bounds__(256) k_nearest_sort_pairs(int64_t n, const int64_t *__restrict__ off, const int32_t *__restrict__ raw,
                                                            uint64_t *__restrict__ lhs, uint64_t *__restrict__ rhs) {
    const int lane = threadIdx.x & 31;
    const int64_t warp = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5, nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t i = warp; i < n; i += nwarps) {
        const int64_t b = off[i], e = off[i + 1];
        for (int64_t k = b + lane; k < e; k += 32) {
            const int32_t j = raw[k];
            int64_t rank = 0;
            for (int64_t m = b; m < e; ++m) rank += raw[m] < j;
            lhs[b + rank] = (uint64_t)i;
            rhs[b + rank] = (uint64_t)j;
        }
    }
}

static const char *type_name_nn(int t) {
    switch (t) {
    case GPL_POINT: return "Point";
    case GPL_LINESTRING: return "LineString";
    case GPL_POLYGON: return "Polygon";
    case GPL_MULTIPOINT: return "MultiPoint";
    case GPL_MULTILINESTRING: return "MultiLineString";
    case GPL_MULTIPOLYGON: return "MultiPolygon";
    default: return "Unknown";
    }
}

int envelope_raw(gpl_ctx *ctx, const gpl_array *in, double *out4_dev, uint8_t *valid_bytes_dev);
int deliver(gpl_ctx *ctx, void *dst, const void *src_dev, size_t bytes, int mem);

static int nn_grid(int64_t n) { return (int)std::max<int64_t>(1, std::min<int64_t>(ceil_div(n, kNnWarps * 32), (int64_t)kSMs * 8)); }

// one pass over the points (device buffers).  MODE 0 fills nid / dist / ntied; MODE 1 writes raw_rhs at off.
static int nearest_run(gpl_ctx *ctx, const gpl_nearest_index *idx, const double2 *pts, const uint8_t *pvalid, int64_t n, double maxd,
                       int32_t *nid, double *dist, int32_t *ntied, const int64_t *off, int32_t *raw_rhs) {
    GPL_CUDA(cudaMemsetAsync(idx->counters, 0, 2 * sizeof(unsigned long long), ctx->stream));
    if (n == 0) return GPL_OK;
    Scratch<uint8_t> flag;
    GPL_TRY(flag.get(ctx, (size_t)n));
    const NearestView v = view_of(idx);
    const int ogrid = (int)std::max<int64_t>(1, std::min<int64_t>(ceil_div(ceil_div(n, 32), 8), (int64_t)kSMs * 16));
    if (raw_rhs == nullptr) {
        GPL_LAUNCH(ctx, k_nearest<0>, nn_grid(n), kNnWarps * 32, 0, v, pts, pvalid, n, maxd, nid, dist, ntied, nullptr, nullptr, flag.p,
                   idx->counters);
        GPL_LAUNCH(ctx, k_nearest_overflow<0>, ogrid, 256, 0, v, pts, n, maxd, flag.p, nid, dist, ntied, nullptr, nullptr, nullptr,
                   idx->counters);
    } else {
        GPL_LAUNCH(ctx, k_nearest<1>, nn_grid(n), kNnWarps * 32, 0, v, pts, pvalid, n, maxd, nullptr, nullptr, nullptr, off, raw_rhs, flag.p,
                   idx->counters);
        GPL_LAUNCH(ctx, k_nearest_overflow<1>, ogrid, 256, 0, v, pts, n, maxd, flag.p, nullptr, nullptr, nullptr, dist, off, raw_rhs,
                   idx->counters);
    }
    return GPL_OK;
}

static int check_query(int64_t n, double maxd) {
    GPL_REQUIRE(n <= 0x7fffffffLL, GPL_ERR_UNSUPPORTED, "nearest join: at most 2^31 - 1 points per call (got %lld)", (long long)n);
    GPL_REQUIRE(maxd >= 0.0, GPL_ERR_INVALID_ARG, "nearest join: max_distance must be >= 0 or +inf (got %g)", maxd);
    return GPL_OK;
}

}  // namespace gpl

using namespace gpl;

extern "C" void gpl_nearest_index_free(gpl_nearest_index *idx) {
    if (!idx) return;
    gpl_ctx *ctx = idx->ctx;
    ctx->release(idx->cell_start);
    ctx->release(idx->recs);
    ctx->release(idx->item_rep);
    ctx->release(idx->item_row);
    ctx->release(idx->every);
    ctx->release(idx->counters);
    delete idx;
}

extern "C" int gpl_nearest_index_build(gpl_ctx *ctx, const gpl_array *rhs, gpl_nearest_index **out) {
    GPL_REQUIRE(ctx && rhs && out, GPL_ERR_INVALID_ARG, "gpl_nearest_index_build: NULL argument");
    const int t = rhs->type;
    GPL_REQUIRE(t == GPL_POINT || t == GPL_LINESTRING || t == GPL_POLYGON || t == GPL_MULTIPOINT || t == GPL_MULTILINESTRING ||
                    t == GPL_MULTIPOLYGON,
                GPL_ERR_INVALID_TYPE, "nearest join: unsupported right geometry type %s", type_name_nn(t));
    GPL_REQUIRE(rhs->n_geoms < (1LL << 31), GPL_ERR_UNSUPPORTED, "nearest join: at most 2^31 - 1 right rows (got %lld)",
                (long long)rhs->n_geoms);
    GPL_CUDA(cudaSetDevice(ctx->device));
    gpl_nearest_index *idx = new gpl_nearest_index();
    idx->ctx = ctx, idx->type = t, idx->xy = reinterpret_cast<const double2 *>(rhs->xy);
    idx->go = rhs->geom_off, idx->po = rhs->part_off, idx->ro = rhs->ring_off;
    const int64_t n = rhs->n_geoms;
    idx->n_rows = n;
    auto fail = [&](int rc) {
        gpl_nearest_index_free(idx);
        return rc;
    };
#define TRYF(expr)                             \
    do {                                       \
        int rc__ = (expr);                     \
        if (rc__ != GPL_OK) return fail(rc__); \
    } while (0)
#define CUDAF(expr)                                                                     \
    do {                                                                                \
        cudaError_t e__ = (expr);                                                       \
        if (e__ != cudaSuccess) return fail(cuda_fail(e__, #expr, __FILE__, __LINE__)); \
    } while (0)
    {
        void *p = nullptr;
        TRYF(ctx->alloc(2 * sizeof(unsigned long long), &p));
        idx->counters = (unsigned long long *)p;
        CUDAF(cudaMemsetAsync(idx->counters, 0, 2 * sizeof(unsigned long long), ctx->stream));
    }
    if (n == 0) {
        CUDAF(cudaStreamSynchronize(ctx->stream));
        *out = idx;
        return GPL_OK;
    }
    Scratch<double> env4, box4;
    Scratch<uint8_t> has, cls, ghas;
    Scratch<double2> rep;
    Scratch<unsigned long long> cnt;
    TRYF(env4.get(ctx, (size_t)n * 4));
    TRYF(box4.get(ctx, (size_t)n * 4));
    TRYF(has.get(ctx, (size_t)n));
    TRYF(cls.get(ctx, (size_t)n));
    TRYF(ghas.get(ctx, (size_t)n));
    TRYF(rep.get(ctx, (size_t)n));
    TRYF(cnt.get(ctx, 8));
    CUDAF(cudaMemsetAsync(cnt.p, 0, 8 * sizeof(unsigned long long), ctx->stream));
    TRYF(envelope_raw(ctx, rhs, env4.p, has.p));
    GPL_LAUNCH(ctx, k_nearest_classify, (int)ceil_div(n, 256), 256, 0, t, n, idx->xy, idx->go, idx->po, idx->ro, rhs->validity, has.p, box4.p,
               rep.p, cls.p, ghas.p, cnt.p);
    unsigned long long h[2];
    CUDAF(cudaMemcpyAsync(h, cnt.p, sizeof(h), cudaMemcpyDeviceToHost, ctx->stream));
    CUDAF(cudaStreamSynchronize(ctx->stream));
    const int64_t n_grid = (int64_t)h[0];
    idx->n_every = (int64_t)h[1];
    idx->n_r = n_grid + idx->n_every;
    size_t bytes = 2 * sizeof(unsigned long long);
    if (idx->n_every > 0) {
        void *p = nullptr;
        TRYF(ctx->alloc(sizeof(int32_t) * (size_t)idx->n_every, &p));
        idx->every = (int32_t *)p;
        bytes += sizeof(int32_t) * (size_t)idx->n_every;
        GPL_LAUNCH(ctx, k_nearest_every, (int)ceil_div(n, 256), 256, 0, cls.p, n, cnt.p + 2, idx->every);
    }
    if (n_grid > 0) {
        // ---- the grid over the union box of the grid rows' boxes (same G rule as gpl_spatial_join) ----------------------------
        unsigned long long *acc = cnt.p + 4;
        GPL_LAUNCH(ctx, k_join_union, (int)std::min<int64_t>(ceil_div(n, 256), kSMs * 8), 256, 0, box4.p, ghas.p, n, acc);
        unsigned long long ha[4];
        CUDAF(cudaMemcpyAsync(ha, acc, sizeof(ha), cudaMemcpyDeviceToHost, ctx->stream));
        CUDAF(cudaStreamSynchronize(ctx->stream));
        auto dec = [](unsigned long long u) {
            const unsigned long long b = (u >> 63) ? (u & 0x7fffffffffffffffULL) : ~u;
            double d;
            memcpy(&d, &b, sizeof(d));
            return d;
        };
        idx->ux0 = dec(~ha[0]), idx->uy0 = dec(~ha[1]), idx->ux1 = dec(ha[2]), idx->uy1 = dec(ha[3]);
        JoinGrid &jg = idx->jg;
        jg.g = (int32_t)std::min<int64_t>(2048, std::max<int64_t>(1, (int64_t)ceil(sqrt((double)idx->n_r))));
        jg.x0 = idx->ux0, jg.y0 = idx->uy0;
        const double w = idx->ux1 - idx->ux0, hh = idx->uy1 - idx->uy0;
        jg.inv_w = (w > 0.0 && std::isfinite(w) && std::isfinite(jg.g / w)) ? jg.g / w : 0.0;
        jg.inv_h = (hh > 0.0 && std::isfinite(hh) && std::isfinite(jg.g / hh)) ? jg.g / hh : 0.0;
        // a box without width (height) maps every x (y) to cell 0: the search then has one column (row)
        idx->gx = jg.inv_w == 0.0 ? 1 : jg.g;
        idx->gy = jg.inv_h == 0.0 ? 1 : jg.g;
        idx->cw = w / jg.g, idx->ch = hh / jg.g;
        idx->M = std::max(std::max(std::fabs(idx->ux0), std::fabs(idx->uy0)), std::max(std::fabs(idx->ux1), std::fabs(idx->uy1)));
        const int64_t n_cells = (int64_t)jg.g * jg.g;
        Scratch<int32_t> cell_count, items;
        Scratch<int64_t> tot;
        TRYF(cell_count.get(ctx, (size_t)n_cells + 1));
        TRYF(tot.get(ctx, 1));
        void *p = nullptr;
        TRYF(ctx->alloc(sizeof(int32_t) * ((size_t)n_cells + 1), &p));
        idx->cell_start = (int32_t *)p;
        bytes += sizeof(int32_t) * ((size_t)n_cells + 1);
        CUDAF(cudaMemsetAsync(cell_count.p, 0, sizeof(int32_t) * (n_cells + 1), ctx->stream));
        GPL_LAUNCH(ctx, k_join_cells<0>, (int)ceil_div(n, 128), 128, 0, box4.p, ghas.p, n, jg, cell_count.p, nullptr);
        TRYF((exclusive_scan<int32_t, int32_t>(ctx, cell_count.p, n_cells, idx->cell_start, tot.p)));
        int64_t n_items = 0;
        CUDAF(cudaMemcpyAsync(&n_items, tot.p, sizeof(int64_t), cudaMemcpyDeviceToHost, ctx->stream));
        CUDAF(cudaStreamSynchronize(ctx->stream));
        GPL_REQUIRE(n_items < (1LL << 31), fail(GPL_ERR_UNSUPPORTED), "nearest join: grid too dense (%lld cell items)", (long long)n_items);
        idx->n_items = n_items;
        TRYF(ctx->alloc(sizeof(int32_t) * ((size_t)n_items + 1), &p));
        idx->item_row = (int32_t *)p;
        TRYF(ctx->alloc(sizeof(double2) * 2 * ((size_t)n_items + 1), &p));
        idx->recs = (double2 *)p;
        TRYF(ctx->alloc(sizeof(double2) * ((size_t)n_items + 1), &p));
        idx->item_rep = (double2 *)p;
        bytes += (size_t)n_items * (sizeof(int32_t) + 3 * sizeof(double2));
        CUDAF(cudaMemcpyAsync(cell_count.p, idx->cell_start, sizeof(int32_t) * n_cells, cudaMemcpyDeviceToDevice, ctx->stream));  // cursors
        GPL_LAUNCH(ctx, k_join_cells<1>, (int)ceil_div(n, 128), 128, 0, box4.p, ghas.p, n, jg, cell_count.p, idx->item_row);
        if (n_items > 0)
            GPL_LAUNCH(ctx, k_nearest_records, (int)ceil_div(n_items, 256), 256, 0, idx->item_row, n_items, box4.p, rep.p, idx->recs,
                       idx->item_rep);
    }
    idx->bytes = (int64_t)bytes;
    CUDAF(cudaStreamSynchronize(ctx->stream));  // the scratch above returns to the cache when this scope ends
    *out = idx;
    return GPL_OK;
#undef TRYF
#undef CUDAF
}

extern "C" int gpl_nearest_index_stats(gpl_ctx *ctx, const gpl_nearest_index *idx, int64_t *out8) {
    GPL_REQUIRE(ctx && idx && out8, GPL_ERR_INVALID_ARG, "gpl_nearest_index_stats: NULL argument");
    GPL_CUDA(cudaSetDevice(ctx->device));
    unsigned long long h[2] = {0, 0};
    GPL_CUDA(cudaMemcpyAsync(h, idx->counters, sizeof(h), cudaMemcpyDeviceToHost, ctx->stream));
    GPL_CUDA(cudaStreamSynchronize(ctx->stream));
    out8[0] = idx->n_r;
    out8[1] = idx->n_rows - idx->n_r;
    out8[2] = idx->n_every;
    out8[3] = idx->jg.g;
    out8[4] = idx->n_items;
    out8[5] = idx->bytes;
    out8[6] = (int64_t)h[0];
    out8[7] = (int64_t)h[1];
    return GPL_OK;
}

extern "C" int gpl_nearest_join(gpl_ctx *ctx, const gpl_nearest_index *idx, const double *points_xy, int64_t n_points, double max_distance,
                                int32_t *nearest_id, double *distance, int32_t *n_tied, int mem) {
    GPL_REQUIRE(ctx && idx && nearest_id && (points_xy || n_points <= 0), GPL_ERR_INVALID_ARG, "gpl_nearest_join: NULL argument");
    GPL_REQUIRE(n_points >= 0, GPL_ERR_INVALID_ARG, "gpl_nearest_join: negative point count");
    GPL_TRY(check_query(n_points, max_distance));
    GPL_CUDA(cudaSetDevice(ctx->device));
    const double2 *pts = reinterpret_cast<const double2 *>(points_xy);
    if (mem == GPL_DEVICE) {
        GPL_TRY(nearest_run(ctx, idx, pts, nullptr, n_points, max_distance, nearest_id, distance, n_tied, nullptr, nullptr));
        return GPL_OK;
    }
    const size_t n = (size_t)n_points;
    Scratch<double> dp, dd;
    Scratch<int32_t> di, dt;
    GPL_TRY(dp.get(ctx, n * 2));
    GPL_TRY(di.get(ctx, n));
    if (distance) GPL_TRY(dd.get(ctx, n));
    if (n_tied) GPL_TRY(dt.get(ctx, n));
    if (n) GPL_CUDA(cudaMemcpyAsync(dp.p, points_xy, sizeof(double) * 2 * n, cudaMemcpyHostToDevice, ctx->stream));
    GPL_TRY(nearest_run(ctx, idx, reinterpret_cast<const double2 *>(dp.p), nullptr, n_points, max_distance, di.p, distance ? dd.p : nullptr,
                        n_tied ? dt.p : nullptr, nullptr, nullptr));
    if (n) {
        GPL_CUDA(cudaMemcpyAsync(nearest_id, di.p, sizeof(int32_t) * n, cudaMemcpyDeviceToHost, ctx->stream));
        if (distance) GPL_CUDA(cudaMemcpyAsync(distance, dd.p, sizeof(double) * n, cudaMemcpyDeviceToHost, ctx->stream));
        if (n_tied) GPL_CUDA(cudaMemcpyAsync(n_tied, dt.p, sizeof(int32_t) * n, cudaMemcpyDeviceToHost, ctx->stream));
    }
    GPL_CUDA(cudaStreamSynchronize(ctx->stream));
    return GPL_OK;
}

extern "C" int gpl_nearest_join_array(gpl_ctx *ctx, const gpl_nearest_index *idx, const gpl_array *points, double max_distance,
                                      int32_t *nearest_id, double *distance, int32_t *n_tied, int mem) {
    GPL_REQUIRE(ctx && idx && points && nearest_id, GPL_ERR_INVALID_ARG, "gpl_nearest_join_array: NULL argument");
    GPL_REQUIRE(points->type == GPL_POINT, GPL_ERR_INVALID_TYPE, "nearest join: the left side must be Point (found %s)",
                type_name_nn(points->type));
    GPL_TRY(check_query(points->n_geoms, max_distance));
    GPL_CUDA(cudaSetDevice(ctx->device));
    const int64_t n = points->n_geoms;
    const double2 *pts = reinterpret_cast<const double2 *>(points->xy);
    if (mem == GPL_DEVICE) return nearest_run(ctx, idx, pts, points->validity, n, max_distance, nearest_id, distance, n_tied, nullptr, nullptr);
    Scratch<double> dd;
    Scratch<int32_t> di, dt;
    GPL_TRY(di.get(ctx, (size_t)n));
    if (distance) GPL_TRY(dd.get(ctx, (size_t)n));
    if (n_tied) GPL_TRY(dt.get(ctx, (size_t)n));
    GPL_TRY(nearest_run(ctx, idx, pts, points->validity, n, max_distance, di.p, distance ? dd.p : nullptr, n_tied ? dt.p : nullptr, nullptr,
                        nullptr));
    if (n) {
        GPL_CUDA(cudaMemcpyAsync(nearest_id, di.p, sizeof(int32_t) * n, cudaMemcpyDeviceToHost, ctx->stream));
        if (distance) GPL_CUDA(cudaMemcpyAsync(distance, dd.p, sizeof(double) * n, cudaMemcpyDeviceToHost, ctx->stream));
        if (n_tied) GPL_CUDA(cudaMemcpyAsync(n_tied, dt.p, sizeof(int32_t) * n, cudaMemcpyDeviceToHost, ctx->stream));
    }
    GPL_CUDA(cudaStreamSynchronize(ctx->stream));
    return GPL_OK;
}

extern "C" int gpl_nearest_join_pairs_array(gpl_ctx *ctx, const gpl_nearest_index *idx, const gpl_array *points, double max_distance,
                                            gpl_pairs **out, double *distance, int mem) {
    GPL_REQUIRE(ctx && idx && points && out, GPL_ERR_INVALID_ARG, "gpl_nearest_join_pairs_array: NULL argument");
    GPL_REQUIRE(points->type == GPL_POINT, GPL_ERR_INVALID_TYPE, "nearest join: the left side must be Point (found %s)",
                type_name_nn(points->type));
    GPL_TRY(check_query(points->n_geoms, max_distance));
    GPL_CUDA(cudaSetDevice(ctx->device));
    gpl_pairs *res = new gpl_pairs();
    res->ctx = ctx;
    *out = res;
    const int64_t n = points->n_geoms;
    if (n == 0) return GPL_OK;
    const double2 *pts = reinterpret_cast<const double2 *>(points->xy);
    Scratch<int32_t> ids, cnt, raw;
    Scratch<double> dist;
    Scratch<int64_t> off;
    GPL_TRY(ids.get(ctx, (size_t)n));
    GPL_TRY(cnt.get(ctx, (size_t)n));
    GPL_TRY(dist.get(ctx, (size_t)n));
    GPL_TRY(off.get(ctx, (size_t)n + 2));
    GPL_CUDA(cudaMemsetAsync(cnt.p, 0, sizeof(int32_t) * (size_t)n, ctx->stream));  // the offsets below never see stale counts
    GPL_TRY(nearest_run(ctx, idx, pts, points->validity, n, max_distance, ids.p, dist.p, cnt.p, nullptr, nullptr));
    if (distance) GPL_TRY(deliver(ctx, distance, dist.p, sizeof(double) * (size_t)n, mem));  // the dense distances, for free
    GPL_TRY((exclusive_scan<int32_t, int64_t>(ctx, cnt.p, n, off.p, off.p + n + 1)));
    int64_t total = 0;
    GPL_CUDA(cudaMemcpyAsync(&total, off.p + n + 1, sizeof(int64_t), cudaMemcpyDeviceToHost, ctx->stream));
    GPL_CUDA(cudaStreamSynchronize(ctx->stream));
    if (total == 0) return GPL_OK;
    GPL_TRY(raw.get(ctx, (size_t)total));
    GPL_TRY(nearest_run(ctx, idx, pts, points->validity, n, max_distance, nullptr, dist.p, nullptr, off.p, raw.p));
    void *pl = nullptr, *pr = nullptr;
    GPL_TRY(ctx->alloc(sizeof(uint64_t) * (size_t)total, &pl));
    res->lhs = (uint64_t *)pl;
    GPL_TRY(ctx->alloc(sizeof(uint64_t) * (size_t)total, &pr));
    res->rhs = (uint64_t *)pr;
    res->n = total;
    GPL_LAUNCH(ctx, k_nearest_sort_pairs, (int)std::max<int64_t>(1, std::min<int64_t>(ceil_div(n, 8), (int64_t)kSMs * 16)), 256, 0, n, off.p,
               raw.p, res->lhs, res->rhs);
    GPL_CUDA(cudaStreamSynchronize(ctx->stream));
    return GPL_OK;
}
