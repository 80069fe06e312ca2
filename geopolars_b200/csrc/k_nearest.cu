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
// Pairs (pair_list, join_host.cuh): the dense pass gives n_tied, a scan gives offsets, the same kernels in MODE 1 write the
// tied rows and k_sort_rows_* order each point's rows.
// The distance-within join (gpl_dwithin_*, DESIGN.md §4.14) queries the same index over a fixed window per left row.
#include <math.h>

#include <algorithm>
#include <cmath>
#include <memory>

#include "common.cuh"
#include "join_grid.cuh"
#include "join_host.cuh"
#include "output.cuh"
#include "pair_dist.cuh"
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
// tau of a left box (DESIGN.md §4.13 "Slack")
__device__ __forceinline__ double box_slack(const NearestView &v, double lx0, double ly0, double lx1, double ly1) {
    return 0x1p-40 * fmax(v.M, fmax(fmax(fabs(lx0), fabs(ly0)), fmax(fabs(lx1), fabs(ly1))));
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

static int nn_grid(int64_t n) { return (int)std::max<int64_t>(1, std::min<int64_t>(ceil_div(n, kNnWarps * 32), (int64_t)kSMs * 8)); }

// a column of one of the six types with at most 2^31 - 1 rows (row ids are int32); `per` follows "rows" in the message
static int check_column(const gpl_array *a, const char *join, const char *side, const char *per) {
    const int t = a->type;
    GPL_REQUIRE(t == GPL_POINT || t == GPL_LINESTRING || t == GPL_POLYGON || t == GPL_MULTIPOINT || t == GPL_MULTILINESTRING ||
                    t == GPL_MULTIPOLYGON,
                GPL_ERR_INVALID_TYPE, "%s: unsupported %s geometry type %s", join, side, type_name(t));
    GPL_REQUIRE(a->n_geoms <= 0x7fffffffLL, GPL_ERR_UNSUPPORTED, "%s: at most 2^31 - 1 %s rows%s (got %lld)", join, side, per,
                (long long)a->n_geoms);
    return GPL_OK;
}

// the classes, boxes and representative vertices of a column's rows (k_nearest_classify), and the number of grid and everywhere
// rows; the right side of the index and the left side of a query are classified alike
struct RowClasses {
    Scratch<double> box4;
    Scratch<double2> rep;
    Scratch<uint8_t> cls, grid_has;
    int64_t n_grid = 0, n_every = 0;
};
static int classify_rows(gpl_ctx *ctx, const gpl_array *a, RowClasses &rc) {
    const int64_t n = a->n_geoms;
    Scratch<double> env4;
    Scratch<uint8_t> has;
    Scratch<unsigned long long> cnt;
    GPL_TRY(env4.get(ctx, (size_t)n * 4));
    GPL_TRY(rc.box4.get(ctx, (size_t)n * 4));
    GPL_TRY(has.get(ctx, (size_t)n));
    GPL_TRY(rc.cls.get(ctx, (size_t)n));
    GPL_TRY(rc.grid_has.get(ctx, (size_t)n));
    GPL_TRY(rc.rep.get(ctx, (size_t)n));
    GPL_TRY(cnt.get(ctx, 2));
    GPL_CUDA(cudaMemsetAsync(cnt.p, 0, 2 * sizeof(unsigned long long), ctx->stream));
    GPL_TRY(envelope_raw(ctx, a, env4.p, has.p));
    GPL_LAUNCH(ctx, k_nearest_classify, (int)ceil_div(n, 256), 256, 0, a->type, n, reinterpret_cast<const double2 *>(a->xy), a->geom_off,
               a->part_off, a->ring_off, a->validity, has.p, rc.box4.p, rc.rep.p, rc.cls.p, rc.grid_has.p, cnt.p);
    unsigned long long h[2];
    GPL_CUDA(cudaMemcpyAsync(h, cnt.p, sizeof(h), cudaMemcpyDeviceToHost, ctx->stream));
    GPL_CUDA(cudaStreamSynchronize(ctx->stream));  // env4 / has / cnt return to the cache when this scope ends
    rc.n_grid = (int64_t)h[0], rc.n_every = (int64_t)h[1];
    return GPL_OK;
}

// one pass over the points (device buffers).  MODE 0 fills nid / dist / ntied; MODE 1 writes raw_rhs at off.
static int nearest_run(gpl_ctx *ctx, const gpl_nearest_index *idx, const double2 *pts, const uint8_t *pvalid, int64_t n, double maxd,
                       int32_t *nid, double *dist, int32_t *ntied, const int64_t *off, int32_t *raw_rhs) {
    GPL_CUDA(cudaMemsetAsync(idx->counters, 0, 2 * sizeof(unsigned long long), ctx->stream));
    if (n == 0) return GPL_OK;
    Scratch<uint8_t> flag;
    GPL_TRY(flag.get(ctx, (size_t)n));
    const NearestView v = view_of(idx);
    const int ogrid = warp_grid(ceil_div(n, 32), 8);  // one warp per 32-point block
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

// ---- geometry query (gpl_nearest_join_geom*): any left geometry type, DESIGN.md §4.13 ----------------------------------------
// One left row per warp (rows from an atomic cursor: a row has 2 to tens of thousands of coordinates).  The left rows are
// classified by k_nearest_classify like the right rows: excluded rows match nothing; irregular rows (an empty member, an
// empty ring, a 1-coordinate linestring / ring) are evaluated against every row of R; the others are pruned with the box
// of all their coordinates.
constexpr int kNgWarps = 4;     // warps per CTA
constexpr int kNgQueue = 128;   // queued right rows per warp (a full queue is drained and the walk continues)
static int ng_grid(int64_t n) { return (int)std::max<int64_t>(1, std::min<int64_t>(ceil_div(n, kNgWarps), (int64_t)kSMs * 8)); }

// member views of a Multi* column (k_pairs.cu gpl_distance): MultiPoint -> POINT over coordinates, MultiLineString ->
// LINESTRING over rings, MultiPolygon -> POLYGON over parts; a single type is its own view
__host__ __device__ __forceinline__ bool is_multi_type(int t) { return t == GPL_MULTIPOINT || t == GPL_MULTILINESTRING || t == GPL_MULTIPOLYGON; }
__device__ __forceinline__ Side member_view(const Side &s) {
    switch (s.type) {
    case GPL_MULTIPOINT: return Side{GPL_POINT, s.xy, nullptr, nullptr, nullptr};
    case GPL_MULTILINESTRING: return Side{GPL_LINESTRING, s.xy, s.ro, nullptr, nullptr};
    case GPL_MULTIPOLYGON: return Side{GPL_POLYGON, s.xy, s.po, nullptr, s.ro};
    default: return s;
    }
}

// per-warp shared scratch of the LineString x LineString fast path (k_ls_ls_fast's staging, s_box and s_queue)
struct LsLsScratch {
    double2 *xy;          // 68 coordinates
    float4 *box;          // 64
    unsigned short *queue;  // kPairQueue
};

// exactly gpl_distance(lhs row i, rhs row j): the routine gpl_distance dispatches the pair to (k_pairs.cu), with lhs as the
// first operand.  ok = false: gpl_distance returns null for the pair.  Warp cooperative, warp-uniform result.  The left
// side is never a Point column here (that goes to k_nearest).
__device__ __forceinline__ double geom_pair_distance(const Side &L, int64_t i, const NearestView &v, int64_t j, const LsLsScratch &sc,
                                                     int lane, bool &ok) {
    const Side R{v.type, v.xy, v.go, v.po, v.ro};
    if (is_multi_type(L.type) || is_multi_type(R.type)) {  // k_distance_multi
        const Side a = member_view(L), b = member_view(R);
        const int64_t a0 = is_multi_type(L.type) ? L.go[i] : i, a1 = is_multi_type(L.type) ? L.go[i + 1] : i + 1;
        const int64_t b0 = is_multi_type(R.type) ? R.go[j] : j, b1 = is_multi_type(R.type) ? R.go[j + 1] : j + 1;
        double d = 1.7976931348623157e308;
        for (int64_t p = a0; p < a1 && ok; ++p)
            for (int64_t q = b0; q < b1 && ok; ++q) d = fmin(d, member_distance(a, p, b, q, lane, ok));
        return d;
    }
    if (L.type == GPL_LINESTRING && R.type == GPL_LINESTRING) {  // k_ls_ls_fast, then k_ls_ls_exact for what it defers
        const int64_t a0 = L.go[i], la = L.go[i + 1] - a0, b0 = R.go[j], lb = R.go[j + 1] - b0;
        if (la <= 33 && lb <= 33) {
            const int32_t na = (int32_t)la, nb = (int32_t)lb;
            __syncwarp();
            for (int32_t c = lane; c < na + nb; c += 32) sc.xy[c] = c < na ? L.xy[a0 + c] : R.xy[b0 + (c - na)];
            __syncwarp();
            const int isect = ls_intersects_ls_short(sc.xy, na, sc.xy + na, nb, sc.box, sc.queue, lane);
            if (isect == 1) return 0.0;
            if (isect == 0) {
                if (na < 2 || nb < 2) {
                    ok = false;
                    return 0.0;
                }
                return ls_ls_distance_short(sc.xy, na, sc.xy + na, nb, lane);
            }
        }
        const Coords A{L.xy + a0}, B{R.xy + b0};
        if (ls_intersects_ls(A, la, B, lb, lane)) return 0.0;
        if (la < 2 || lb < 2) {
            ok = false;
            return 0.0;
        }
        return sqrt(ls_ls_min_dist2(A, la, B, lb, lane));
    }
    if (R.type == GPL_POINT) {
        if (L.type == GPL_LINESTRING) return point_ls_distance(L.xy, L.go[i], L.go[i + 1] - L.go[i], R.xy[j], lane);  // k_point_ls_dist
        return point_polygon_distance(L, i, R.xy[j], lane);  // k_poly_point<1>
    }
    return generic_distance(L, i, R, j, lane, ok);  // k_distance_generic
}

// Euclidean distance between two closed boxes (the §4.12 box_dist with a box for the point)
__device__ __forceinline__ double box_box_dist(double ax0, double ay0, double ax1, double ay1, double bx0, double by0, double bx1, double by1) {
    return hypot(fmax(fmax(bx0 - ax1, ax0 - bx1), 0.0), fmax(fmax(by0 - ay1, ay0 - by1), 0.0));
}
// the designated cell of a right row whose cells span [i0, i1] on one axis, for a left range [l0, l1]: the cell of the row
// nearest to the left range, the lowest one where they overlap.  (x, y) of the designated cell is the one cell of the row on
// the ring at the Chebyshev distance between the two cell ranges, so the row is enqueued once.
__device__ __forceinline__ int32_t designated(int32_t i0, int32_t i1, int32_t l0, int32_t l1) {
    return i1 < l0 ? i1 : (i0 > l1 ? i0 : max(i0, l0));
}

// MODE 0: nearest_id / distance / n_tied per left row.  MODE 1: the rows at dist_in[i] into raw_rhs[off[i] .. off[i+1]).
// ctr[0]: exact evaluations, cursor: the row cursor (zeroed by the host).
template <int MODE>
__global__ void __launch_bounds__(kNgWarps * 32) k_nearest_geom(NearestView v, Side L, const uint8_t *__restrict__ cls,
                                                               const double *__restrict__ box4, int64_t n, double maxd,
                                                               int32_t *__restrict__ nid, double *__restrict__ dist,
                                                               int32_t *__restrict__ ntied, const double *__restrict__ dist_in,
                                                               const int64_t *__restrict__ off, int32_t *__restrict__ raw_rhs,
                                                               unsigned long long *__restrict__ ctr, unsigned long long *__restrict__ cursor) {
    __shared__ int32_t s_row[kNgWarps][kNgQueue];
    __shared__ double2 s_xy[kNgWarps][68];
    __shared__ float4 s_box[kNgWarps][64];
    __shared__ unsigned short s_q[kNgWarps][kPairQueue];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const LsLsScratch sc{s_xy[wid], s_box[wid], s_q[wid]};
    const double inf = __longlong_as_double(0x7ff0000000000000LL);
    unsigned long long evals = 0;
    for (;;) {
        unsigned long long t = 0;
        if (lane == 0) t = atomicAdd(cursor, 1ULL);
        const int64_t i = (int64_t)__shfl_sync(0xffffffffu, t, 0);
        if (i >= n) break;
        const uint8_t c = cls[i];
        double best = inf;
        int32_t id = 0x7fffffff, cnt = 0;
        // U: a distance already evaluated exactly (or max_distance); MODE 1 starts from the dense pass's exact minimum
        double U = MODE == 0 ? maxd : dist_in[i];
        const int64_t b = MODE == 1 && c ? off[i] : 0, cap = MODE == 1 && c ? off[i + 1] - b : 0;
        int64_t w = 0;
        if (c != 0 && (MODE == 0 || cap > 0)) {
            auto consider = [&](int32_t j) {  // warp-uniform
                bool ok = true;
                const double d = geom_pair_distance(L, i, v, j, sc, lane, ok);
                ++evals;
                if (!ok || !(d <= maxd)) return;
                if (MODE == 0) {
                    if (d < best || cnt == 0) best = d, id = j, cnt = 1;
                    else if (d == best) ++cnt, id = min(id, j);
                    U = fmin(U, d);
                } else if (d == U && w < cap) {
                    if (lane == 0) raw_rhs[b + w] = j;
                    ++w;
                }
            };
            for (int32_t e = 0; e < v.n_every; ++e) consider(v.every[e]);
            if (v.jg.g > 0) {
                const double lx0 = box4[4 * i], ly0 = box4[4 * i + 1], lx1 = box4[4 * i + 2], ly1 = box4[4 * i + 3];
                const double tau = box_slack(v, lx0, ly0, lx1, ly1);
                const bool prune = c == 1;  // irregular rows: every row of R
                const int32_t lcx0 = cell_x(v, lx0), lcx1 = cell_x(v, lx1), lcy0 = cell_y(v, ly0), lcy1 = cell_y(v, ly1);
                int qn = 0;  // warp-uniform
                auto drain = [&]() {
                    __syncwarp();
                    for (int e = 0; e < qn; ++e) consider(s_row[wid][e]);
                    qn = 0;
                    __syncwarp();
                };
                auto visit = [&](int32_t cx, int32_t cy) {
                    const int64_t cc = (int64_t)cy * v.jg.g + cx;
                    const int32_t k0 = v.cell_start[cc], k1 = v.cell_start[cc + 1];
                    for (int32_t kb = k0; kb < k1; kb += 32) {
                        const int32_t k = kb + lane;
                        bool cand = false;
                        if (k < k1) {
                            const double2 lo = v.recs[2 * (int64_t)k], hi = v.recs[2 * (int64_t)k + 1];
                            cand = !prune || box_box_dist(lx0, ly0, lx1, ly1, lo.x, lo.y, hi.x, hi.y) <= U + tau;
                            cand = cand && designated(cell_x(v, lo.x), cell_x(v, hi.x), lcx0, lcx1) == cx &&
                                   designated(cell_y(v, lo.y), cell_y(v, hi.y), lcy0, lcy1) == cy;
                        }
                        const unsigned m = __ballot_sync(0xffffffffu, cand);
                        if (!m) continue;
                        if (qn + __popc(m) > kNgQueue) drain();
                        if (cand) s_row[wid][qn + __popc(m & ((1u << lane) - 1u))] = v.item_row[k];
                        qn += __popc(m);
                    }
                };
                for (int32_t r = 0;; ++r) {
                    const int32_t y0 = max(lcy0 - r, 0), y1 = min(lcy1 + r, v.gy - 1);
                    const int32_t x0 = max(lcx0 - r, 0), x1 = min(lcx1 + r, v.gx - 1);
                    for (int32_t cy = y0; cy <= y1; ++cy) {
                        if (r == 0 || cy == lcy0 - r || cy == lcy1 + r) {
                            for (int32_t cx = x0; cx <= x1; ++cx) visit(cx, cy);
                        } else {
                            if (lcx0 - r >= 0) visit(lcx0 - r, cy);
                            if (lcx1 + r < v.gx) visit(lcx1 + r, cy);
                        }
                    }
                    drain();
                    // distance from the left box to the cells outside the window (one box per side that still has cells)
                    double B = inf;
                    bool more = false;
                    if (lcx1 + r + 1 < v.gx) more = true, B = fmin(B, box_box_dist(lx0, ly0, lx1, ly1, v.ux0 + (lcx1 + r + 1) * v.cw, v.uy0, v.ux1, v.uy1));
                    if (lcx0 - r - 1 >= 0) more = true, B = fmin(B, box_box_dist(lx0, ly0, lx1, ly1, v.ux0, v.uy0, v.ux0 + (lcx0 - r) * v.cw, v.uy1));
                    if (lcy1 + r + 1 < v.gy) more = true, B = fmin(B, box_box_dist(lx0, ly0, lx1, ly1, v.ux0, v.uy0 + (lcy1 + r + 1) * v.ch, v.ux1, v.uy1));
                    if (lcy0 - r - 1 >= 0) more = true, B = fmin(B, box_box_dist(lx0, ly0, lx1, ly1, v.ux0, v.uy0, v.ux1, v.uy0 + (lcy0 - r) * v.ch));
                    if (!more || (prune && B - 2.0 * tau > U)) break;
                }
            }
        }
        if (MODE == 0 && lane == 0) {
            nid[i] = cnt ? id : -1;
            if (dist) dist[i] = cnt ? best : nan("");
            if (ntied) ntied[i] = cnt;
        }
    }
    if (lane == 0 && evals) atomicAdd(ctr, evals);
}

// one pass over the left rows (device buffers).  MODE 0 (raw_rhs == NULL) fills nid / dist / ntied; MODE 1 writes the rows at
// dist_in[i] into raw_rhs at off.
static int geom_run(gpl_ctx *ctx, const gpl_nearest_index *idx, const gpl_array *lhs, const uint8_t *cls, const double *box4, double maxd,
                    int32_t *nid, double *dist, int32_t *ntied, const double *dist_in, const int64_t *off, int32_t *raw_rhs) {
    GPL_CUDA(cudaMemsetAsync(idx->counters, 0, 2 * sizeof(unsigned long long), ctx->stream));
    const int64_t n = lhs->n_geoms;
    if (n == 0) return GPL_OK;
    Scratch<unsigned long long> cursor;
    GPL_TRY(cursor.get(ctx, 1));
    GPL_CUDA(cudaMemsetAsync(cursor.p, 0, sizeof(unsigned long long), ctx->stream));
    const NearestView v = view_of(idx);
    const Side L{lhs->type, reinterpret_cast<const double2 *>(lhs->xy), lhs->geom_off, lhs->part_off, lhs->ring_off};
    if (raw_rhs == nullptr)
        GPL_LAUNCH(ctx, k_nearest_geom<0>, ng_grid(n), kNgWarps * 32, 0, v, L, cls, box4, n, maxd, nid, dist, ntied, nullptr, nullptr, nullptr,
                   idx->counters, cursor.p);
    else
        GPL_LAUNCH(ctx, k_nearest_geom<1>, ng_grid(n), kNgWarps * 32, 0, v, L, cls, box4, n, maxd, nullptr, nullptr, nullptr, dist_in, off,
                   raw_rhs, idx->counters, cursor.p);
    GPL_CUDA(cudaStreamSynchronize(ctx->stream));  // the cursor returns to the cache when this scope ends
    return GPL_OK;
}

static int check_geom_left(const gpl_array *lhs, double maxd) {
    GPL_TRY(check_column(lhs, "nearest join", "left", " per call"));
    return check_query(lhs->n_geoms, maxd);
}

// ---- distance-within join (gpl_dwithin_*): every row of R within D of each left row, DESIGN.md §4.14 ------------------------
// Kept in this file: it queries the nearest index through NearestView and reuses is_candidate, designated, row_distance,
// geom_pair_distance, the left-row classification and the pair-list pipeline unchanged.  Instead of a ring search each left row walks a FIXED window:
// the cells that can hold its box expanded by dw_margin(D, tau) on every side.  There is no overflow path: the walk runs in
// warp-synchronous rounds, and a full queue is drained by the whole warp before the walk resumes.
// MODE 0 writes the match count of each left row.  MODE 1 writes (rhs, d) into the row's slots [off[i], off[i+1]) in the
// order they are found (k_sort_rows_* orders them) and adds to *bad each row whose write pass found a different number of
// matches than its count pass; both passes evaluate the same pairs with the same routines, so the host treats bad != 0 as
// an internal error.

// Half-width of the window.  A row with computed lb <= D + tau has its designated cell at a coordinate within
// lb * (1 + 4u) of the left box; the window edge fl(x - m) is within u * |x - m| of x - m.  (D + 2 tau)(1 + 2^-40) covers
// both with tau to spare for any D (DESIGN.md §4.14 "Window").
__device__ __forceinline__ double dw_margin(double D, double tau) { return (D + 2.0 * tau) * (1.0 + 0x1p-40); }

// Point left side: persistent warps, one lane per point (k_nearest's tile loop and queue)
template <int MODE>
__global__ void __launch_bounds__(kNnWarps * 32) k_dwithin_pts(NearestView v, const double2 *__restrict__ pts, const uint8_t *__restrict__ pvalid,
                                                              int64_t n, double D, int32_t *__restrict__ cnt, const int64_t *__restrict__ off,
                                                              int32_t *__restrict__ raw_rhs, double *__restrict__ raw_d,
                                                              unsigned long long *__restrict__ ctr, unsigned long long *__restrict__ bad) {
    __shared__ int32_t s_row[kNnWarps][kNnQueue];
    __shared__ uint8_t s_own[kNnWarps][kNnQueue];
    __shared__ double2 s_pt[kNnWarps][32];
    __shared__ int32_t s_cnt[kNnWarps][32];  // matches of each point so far (MODE 1: its next slot)
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
        s_cnt[wid][lane] = 0;
        __syncwarp();
        // one evaluated pair, by one thread: count a match; MODE 1 also stores it in the owner's next slot
        auto take = [&](int own, int32_t j, double d) {
            if (!(d <= D)) return;
            const int s = atomicAdd(&s_cnt[wid][own], 1);
            if (MODE == 1) {
                const int64_t b = off[t0 + own];
                if (b + s < off[t0 + own + 1]) {
                    raw_rhs[b + s] = j;
                    if (raw_d) raw_d[b + s] = d;
                }
            }
        };
        // the everywhere rows, with the whole warp for each live point (never queued)
        const unsigned live = __ballot_sync(0xffffffffu, valid);
        for (int32_t e = 0; e < v.n_every; ++e) {
            const int32_t j = v.every[e];
            for (unsigned m = live; m; m &= m - 1) {
                const int l = __ffs(m) - 1;
                const double d = row_distance(v, j, s_pt[wid][l], lane);
                if (lane == l) take(l, j, d), ++evals;
            }
        }
        // the window, walked in rounds: each lane pushes its candidates until its window is done or the queue is full, the
        // warp drains the queue, and the lanes resume where they stopped (the item that found the queue full is retried)
        bool walking = valid && grid;
        int32_t wx0 = 0, wx1 = 0, wy1 = 0, cx = 0, cy = 0, k = 0, k1 = 0;
        double lim = 0.0;
        if (walking) {
            const double tau = slack(v, p), m = dw_margin(D, tau);
            lim = D + tau;
            wx0 = min(cell_x(v, p.x - m), v.gx - 1), wx1 = min(cell_x(v, p.x + m), v.gx - 1);
            cy = min(cell_y(v, p.y - m), v.gy - 1), wy1 = min(cell_y(v, p.y + m), v.gy - 1);
            cx = wx0;
            const int64_t c = (int64_t)cy * v.jg.g + cx;
            k = v.cell_start[c], k1 = v.cell_start[c + 1];
        }
        while (__any_sync(0xffffffffu, walking)) {
            while (walking) {
                if (k >= k1) {
                    if (++cx > wx1) {
                        cx = wx0;
                        if (++cy > wy1) {
                            walking = false;
                            break;
                        }
                    }
                    const int64_t c = (int64_t)cy * v.jg.g + cx;
                    k = v.cell_start[c], k1 = v.cell_start[c + 1];
                    continue;
                }
                if (is_candidate(v, k, p, lim, cx, cy)) {
                    const int s = atomicAdd(&s_qn[wid], 1);
                    if (s >= kNnQueue) break;  // full
                    s_row[wid][s] = v.item_row[k], s_own[wid][s] = (uint8_t)lane;
                }
                ++k;
            }
            __syncwarp();
            const int nq = min(s_qn[wid], kNnQueue);
            if (lane_rows(v.type)) {
                for (int e = lane; e < nq; e += 32) {
                    const int own = s_own[wid][e];
                    const int32_t j = s_row[wid][e];
                    take(own, j, row_distance(v, j, s_pt[wid][own], lane));
                    ++evals;
                }
            } else {
                for (int e = 0; e < nq; ++e) {
                    const int own = s_own[wid][e];
                    const int32_t j = s_row[wid][e];
                    const double d = row_distance(v, j, s_pt[wid][own], lane);
                    if (lane == 0) take(own, j, d), ++evals;
                }
            }
            __syncwarp();
            if (lane == 0) s_qn[wid] = 0;
            __syncwarp();
        }
        __syncwarp();
        if (i < n) {
            const int32_t got = s_cnt[wid][lane];
            if (MODE == 0) cnt[i] = got;
            else if (got != off[i + 1] - off[i]) atomicAdd(bad, 1ULL);
        }
        __syncwarp();  // s_pt / s_cnt are reused by the next tile
    }
    evals = (unsigned long long)warp_sum((double)evals);
    if (lane == 0 && evals) atomicAdd(ctr, evals);
}

// any other left side: one warp per left row from an atomic cursor (k_nearest_geom's queue and dispatch)
template <int MODE>
__global__ void __launch_bounds__(kNgWarps * 32) k_dwithin_geom(NearestView v, Side L, const uint8_t *__restrict__ cls,
                                                               const double *__restrict__ box4, int64_t n, double D, int32_t *__restrict__ cnt,
                                                               const int64_t *__restrict__ off, int32_t *__restrict__ raw_rhs,
                                                               double *__restrict__ raw_d, unsigned long long *__restrict__ ctr,
                                                               unsigned long long *__restrict__ cursor, unsigned long long *__restrict__ bad) {
    __shared__ int32_t s_row[kNgWarps][kNgQueue];
    __shared__ double2 s_xy[kNgWarps][68];
    __shared__ float4 s_box[kNgWarps][64];
    __shared__ unsigned short s_q[kNgWarps][kPairQueue];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const LsLsScratch sc{s_xy[wid], s_box[wid], s_q[wid]};
    unsigned long long evals = 0;
    for (;;) {
        unsigned long long t = 0;
        if (lane == 0) t = atomicAdd(cursor, 1ULL);
        const int64_t i = (int64_t)__shfl_sync(0xffffffffu, t, 0);
        if (i >= n) break;
        const uint8_t c = cls[i];
        const int64_t b = MODE == 1 ? off[i] : 0, cap = MODE == 1 ? off[i + 1] - b : 0;
        int64_t w = 0;  // matches so far (warp-uniform)
        if (c != 0 && (MODE == 0 || cap > 0)) {
            auto consider = [&](int32_t j) {  // warp-uniform
                bool ok = true;
                const double d = geom_pair_distance(L, i, v, j, sc, lane, ok);
                ++evals;
                if (!ok || !(d <= D)) return;
                if (MODE == 1 && w < cap && lane == 0) {
                    raw_rhs[b + w] = j;
                    if (raw_d) raw_d[b + w] = d;
                }
                ++w;
            };
            for (int32_t e = 0; e < v.n_every; ++e) consider(v.every[e]);
            if (v.jg.g > 0) {
                const double lx0 = box4[4 * i], ly0 = box4[4 * i + 1], lx1 = box4[4 * i + 2], ly1 = box4[4 * i + 3];
                const double tau = box_slack(v, lx0, ly0, lx1, ly1);
                const double lim = D + tau, m = dw_margin(D, tau);
                const bool prune = c == 1;  // irregular rows: every row of R
                const int32_t lcx0 = cell_x(v, lx0), lcx1 = cell_x(v, lx1), lcy0 = cell_y(v, ly0), lcy1 = cell_y(v, ly1);
                const int32_t wx0 = prune ? min(cell_x(v, lx0 - m), v.gx - 1) : 0, wx1 = prune ? min(cell_x(v, lx1 + m), v.gx - 1) : v.gx - 1;
                const int32_t wy0 = prune ? min(cell_y(v, ly0 - m), v.gy - 1) : 0, wy1 = prune ? min(cell_y(v, ly1 + m), v.gy - 1) : v.gy - 1;
                int qn = 0;  // warp-uniform
                auto drain = [&]() {
                    __syncwarp();
                    for (int e = 0; e < qn; ++e) consider(s_row[wid][e]);
                    qn = 0;
                    __syncwarp();
                };
                for (int32_t cy = wy0; cy <= wy1; ++cy)
                    for (int32_t cx = wx0; cx <= wx1; ++cx) {
                        const int64_t cc = (int64_t)cy * v.jg.g + cx;
                        const int32_t k0 = v.cell_start[cc], k1 = v.cell_start[cc + 1];
                        for (int32_t kb = k0; kb < k1; kb += 32) {
                            const int32_t k = kb + lane;
                            bool cand = false;
                            if (k < k1) {
                                const double2 lo = v.recs[2 * (int64_t)k], hi = v.recs[2 * (int64_t)k + 1];
                                cand = !prune || box_box_dist(lx0, ly0, lx1, ly1, lo.x, lo.y, hi.x, hi.y) <= lim;
                                cand = cand && designated(cell_x(v, lo.x), cell_x(v, hi.x), lcx0, lcx1) == cx &&
                                       designated(cell_y(v, lo.y), cell_y(v, hi.y), lcy0, lcy1) == cy;
                            }
                            const unsigned bm = __ballot_sync(0xffffffffu, cand);
                            if (!bm) continue;
                            if (qn + __popc(bm) > kNgQueue) drain();
                            if (cand) s_row[wid][qn + __popc(bm & ((1u << lane) - 1u))] = v.item_row[k];
                            qn += __popc(bm);
                        }
                    }
                drain();
            }
        }
        if (lane == 0) {
            if (MODE == 0) cnt[i] = (int32_t)w;
            else if (w != cap) atomicAdd(bad, 1ULL);
        }
    }
    if (lane == 0 && evals) atomicAdd(ctr, evals);
}

static int check_dwithin(const gpl_array *lhs, double D) {
    GPL_TRY(check_column(lhs, "dwithin join", "left", " per call"));
    GPL_REQUIRE(std::isfinite(D) && D >= 0.0, GPL_ERR_INVALID_ARG, "dwithin join: distance must be finite and >= 0 (got %g)", D);
    return GPL_OK;
}

// one pass over the left rows (device buffers): a POINT column on k_dwithin_pts, any other on k_dwithin_geom (cls / box4 from
// classify_rows).  MODE 0 (raw_rhs == NULL) writes cnt; MODE 1 writes the matches at off and fails when a row's write pass
// disagrees with its count pass.
static int dwithin_run(gpl_ctx *ctx, const gpl_nearest_index *idx, const gpl_array *lhs, const uint8_t *cls, const double *box4, double D,
                       int32_t *cnt, const int64_t *off, int32_t *raw_rhs, double *raw_d) {
    GPL_CUDA(cudaMemsetAsync(idx->counters, 0, 2 * sizeof(unsigned long long), ctx->stream));
    const int64_t n = lhs->n_geoms;
    if (n == 0) return GPL_OK;
    Scratch<unsigned long long> aux;  // [0] row cursor, [1] rows whose write pass disagreed with the count pass
    GPL_TRY(aux.get(ctx, 2));
    GPL_CUDA(cudaMemsetAsync(aux.p, 0, 2 * sizeof(unsigned long long), ctx->stream));
    const NearestView v = view_of(idx);
    if (lhs->type == GPL_POINT) {
        const double2 *pts = reinterpret_cast<const double2 *>(lhs->xy);
        if (raw_rhs == nullptr)
            GPL_LAUNCH(ctx, k_dwithin_pts<0>, nn_grid(n), kNnWarps * 32, 0, v, pts, lhs->validity, n, D, cnt, nullptr, nullptr, nullptr,
                       idx->counters, aux.p + 1);
        else
            GPL_LAUNCH(ctx, k_dwithin_pts<1>, nn_grid(n), kNnWarps * 32, 0, v, pts, lhs->validity, n, D, nullptr, off, raw_rhs, raw_d,
                       idx->counters, aux.p + 1);
    } else {
        const Side L{lhs->type, reinterpret_cast<const double2 *>(lhs->xy), lhs->geom_off, lhs->part_off, lhs->ring_off};
        if (raw_rhs == nullptr)
            GPL_LAUNCH(ctx, k_dwithin_geom<0>, ng_grid(n), kNgWarps * 32, 0, v, L, cls, box4, n, D, cnt, nullptr, nullptr, nullptr, idx->counters,
                       aux.p, aux.p + 1);
        else
            GPL_LAUNCH(ctx, k_dwithin_geom<1>, ng_grid(n), kNgWarps * 32, 0, v, L, cls, box4, n, D, nullptr, off, raw_rhs, raw_d, idx->counters,
                       aux.p, aux.p + 1);
    }
    unsigned long long bad = 0;
    GPL_CUDA(cudaMemcpyAsync(&bad, aux.p + 1, sizeof(bad), cudaMemcpyDeviceToHost, ctx->stream));
    GPL_CUDA(cudaStreamSynchronize(ctx->stream));  // aux returns to the cache when this scope ends
    GPL_REQUIRE(bad == 0, GPL_ERR_CUDA, "dwithin join: the write pass found a different number of matches than the count pass on %llu rows",
                bad);
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
    GPL_TRY(check_column(rhs, "nearest join", "right", ""));
    GPL_CUDA(cudaSetDevice(ctx->device));
    // freed on every early return; released to the caller at the end
    std::unique_ptr<gpl_nearest_index, void (*)(gpl_nearest_index *)> idx(new gpl_nearest_index(), gpl_nearest_index_free);
    idx->ctx = ctx, idx->type = rhs->type, idx->xy = reinterpret_cast<const double2 *>(rhs->xy);
    idx->go = rhs->geom_off, idx->po = rhs->part_off, idx->ro = rhs->ring_off;
    const int64_t n = rhs->n_geoms;
    idx->n_rows = n;
    Scratch<unsigned long long> counters;
    GPL_TRY(counters.get(ctx, 2));
    idx->counters = counters.take();
    GPL_CUDA(cudaMemsetAsync(idx->counters, 0, 2 * sizeof(unsigned long long), ctx->stream));
    if (n == 0) {
        GPL_CUDA(cudaStreamSynchronize(ctx->stream));
        *out = idx.release();
        return GPL_OK;
    }
    RowClasses rc;
    GPL_TRY(classify_rows(ctx, rhs, rc));
    idx->n_every = rc.n_every;
    idx->n_r = rc.n_grid + rc.n_every;
    size_t bytes = 2 * sizeof(unsigned long long);
    if (idx->n_every > 0) {
        Scratch<int32_t> every;
        Scratch<unsigned long long> cursor;
        GPL_TRY(every.get(ctx, (size_t)idx->n_every));
        idx->every = every.take();
        bytes += sizeof(int32_t) * (size_t)idx->n_every;
        GPL_TRY(cursor.get(ctx, 1));
        GPL_CUDA(cudaMemsetAsync(cursor.p, 0, sizeof(unsigned long long), ctx->stream));
        GPL_LAUNCH(ctx, k_nearest_every, (int)ceil_div(n, 256), 256, 0, rc.cls.p, n, cursor.p, idx->every);
    }
    if (rc.n_grid > 0) {
        // the grid over the union box of the grid rows' boxes, G from all rows of R
        GridBuild grid;
        GPL_TRY(join_grid_build(ctx, rc.box4.p, rc.grid_has.p, n, idx->n_r, "nearest join", grid));
        const JoinGrid &jg = idx->jg = grid.jg;
        idx->ux0 = grid.ux0, idx->uy0 = grid.uy0, idx->ux1 = grid.ux1, idx->uy1 = grid.uy1;
        // a box without width (height) maps every x (y) to cell 0: the search then has one column (row)
        idx->gx = jg.inv_w == 0.0 ? 1 : jg.g;
        idx->gy = jg.inv_h == 0.0 ? 1 : jg.g;
        idx->cw = (idx->ux1 - idx->ux0) / jg.g, idx->ch = (idx->uy1 - idx->uy0) / jg.g;
        idx->M = std::max(std::max(std::fabs(idx->ux0), std::fabs(idx->uy0)), std::max(std::fabs(idx->ux1), std::fabs(idx->uy1)));
        const int64_t n_items = idx->n_items = grid.n_items;
        idx->cell_start = grid.cell_start.take();
        idx->item_row = grid.items.take();
        bytes += sizeof(int32_t) * ((size_t)jg.g * jg.g + 1);
        Scratch<double2> recs, item_rep;
        GPL_TRY(recs.get(ctx, 2 * ((size_t)n_items + 1)));
        idx->recs = recs.take();
        GPL_TRY(item_rep.get(ctx, (size_t)n_items + 1));
        idx->item_rep = item_rep.take();
        bytes += (size_t)n_items * (sizeof(int32_t) + 3 * sizeof(double2));
        if (n_items > 0)
            GPL_LAUNCH(ctx, k_nearest_records, (int)ceil_div(n_items, 256), 256, 0, idx->item_row, n_items, rc.box4.p, rc.rep.p, idx->recs,
                       idx->item_rep);
    }
    idx->bytes = (int64_t)bytes;
    GPL_CUDA(cudaStreamSynchronize(ctx->stream));  // the scratch above returns to the cache when this scope ends
    *out = idx.release();
    return GPL_OK;
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
    GPL_TRY(check_mem(mem, "gpl_nearest_join"));
    GPL_REQUIRE(n_points >= 0, GPL_ERR_INVALID_ARG, "gpl_nearest_join: negative point count");
    GPL_TRY(check_query(n_points, max_distance));
    GPL_CUDA(cudaSetDevice(ctx->device));
    const double2 *pts = reinterpret_cast<const double2 *>(points_xy);
    Scratch<double2> dp;
    if (mem != GPL_DEVICE) {  // the points are in the caller's memory too
        GPL_TRY(dp.get(ctx, (size_t)n_points));
        if (n_points) GPL_CUDA(cudaMemcpyAsync(dp.p, points_xy, sizeof(double2) * n_points, cudaMemcpyHostToDevice, ctx->stream));
        pts = dp.p;
    }
    return dense_outputs(ctx, n_points, mem, nearest_id, distance, n_tied, [&](int32_t *nid, double *dist, int32_t *ntied) {
        return nearest_run(ctx, idx, pts, nullptr, n_points, max_distance, nid, dist, ntied, nullptr, nullptr);
    });
}

extern "C" int gpl_nearest_join_array(gpl_ctx *ctx, const gpl_nearest_index *idx, const gpl_array *points, double max_distance,
                                      int32_t *nearest_id, double *distance, int32_t *n_tied, int mem) {
    GPL_REQUIRE(ctx && idx && points && nearest_id, GPL_ERR_INVALID_ARG, "gpl_nearest_join_array: NULL argument");
    GPL_TRY(check_mem(mem, "gpl_nearest_join_array"));
    GPL_REQUIRE(points->type == GPL_POINT, GPL_ERR_INVALID_TYPE, "nearest join: the left side must be Point (found %s)",
                type_name(points->type));
    GPL_TRY(check_query(points->n_geoms, max_distance));
    GPL_CUDA(cudaSetDevice(ctx->device));
    const double2 *pts = reinterpret_cast<const double2 *>(points->xy);
    return dense_outputs(ctx, points->n_geoms, mem, nearest_id, distance, n_tied, [&](int32_t *nid, double *dist, int32_t *ntied) {
        return nearest_run(ctx, idx, pts, points->validity, points->n_geoms, max_distance, nid, dist, ntied, nullptr, nullptr);
    });
}

extern "C" int gpl_nearest_join_pairs_array(gpl_ctx *ctx, const gpl_nearest_index *idx, const gpl_array *points, double max_distance,
                                            gpl_pairs **out, double *distance, int mem) {
    GPL_REQUIRE(ctx && idx && points && out, GPL_ERR_INVALID_ARG, "gpl_nearest_join_pairs_array: NULL argument");
    *out = nullptr;
    GPL_TRY(check_mem(mem, "gpl_nearest_join_pairs_array"));
    GPL_REQUIRE(points->type == GPL_POINT, GPL_ERR_INVALID_TYPE, "nearest join: the left side must be Point (found %s)",
                type_name(points->type));
    GPL_TRY(check_query(points->n_geoms, max_distance));
    GPL_CUDA(cudaSetDevice(ctx->device));
    const int64_t n = points->n_geoms;
    const double2 *pts = reinterpret_cast<const double2 *>(points->xy);
    Scratch<int32_t> ids;
    Scratch<double> dist;  // the dense distance: MODE 1 writes the rows at it
    auto count = [&](int32_t *cnt) -> int {
        GPL_TRY(ids.get(ctx, (size_t)n));
        GPL_TRY(dist.get(ctx, (size_t)n));
        GPL_CUDA(cudaMemsetAsync(cnt, 0, sizeof(int32_t) * (size_t)n, ctx->stream));  // the offsets never see stale counts
        GPL_TRY(nearest_run(ctx, idx, pts, points->validity, n, max_distance, ids.p, dist.p, cnt, nullptr, nullptr));
        if (distance) GPL_TRY(deliver(ctx, distance, dist.p, sizeof(double) * (size_t)n, mem));  // the dense distances, for free
        return GPL_OK;
    };
    auto write = [&](const int64_t *off, int32_t *raw, double *) {
        return nearest_run(ctx, idx, pts, points->validity, n, max_distance, nullptr, dist.p, nullptr, off, raw);
    };
    return pair_list(ctx, n, false, out, count, write);
}

extern "C" int gpl_nearest_join_geom(gpl_ctx *ctx, const gpl_nearest_index *idx, const gpl_array *lhs, double max_distance,
                                     int32_t *nearest_id, double *distance, int32_t *n_tied, int mem) {
    GPL_REQUIRE(ctx && idx && lhs && nearest_id, GPL_ERR_INVALID_ARG, "gpl_nearest_join_geom: NULL argument");
    GPL_TRY(check_mem(mem, "gpl_nearest_join_geom"));
    GPL_TRY(check_geom_left(lhs, max_distance));
    if (lhs->type == GPL_POINT) return gpl_nearest_join_array(ctx, idx, lhs, max_distance, nearest_id, distance, n_tied, mem);
    GPL_CUDA(cudaSetDevice(ctx->device));
    RowClasses lc;
    if (lhs->n_geoms) GPL_TRY(classify_rows(ctx, lhs, lc));
    return dense_outputs(ctx, lhs->n_geoms, mem, nearest_id, distance, n_tied, [&](int32_t *nid, double *dist, int32_t *ntied) {
        return geom_run(ctx, idx, lhs, lc.cls.p, lc.box4.p, max_distance, nid, dist, ntied, nullptr, nullptr, nullptr);
    });
}

extern "C" int gpl_nearest_join_geom_pairs(gpl_ctx *ctx, const gpl_nearest_index *idx, const gpl_array *lhs, double max_distance,
                                           gpl_pairs **out, double *distance, int mem) {
    GPL_REQUIRE(ctx && idx && lhs && out, GPL_ERR_INVALID_ARG, "gpl_nearest_join_geom_pairs: NULL argument");
    *out = nullptr;
    GPL_TRY(check_mem(mem, "gpl_nearest_join_geom_pairs"));
    GPL_TRY(check_geom_left(lhs, max_distance));
    if (lhs->type == GPL_POINT) return gpl_nearest_join_pairs_array(ctx, idx, lhs, max_distance, out, distance, mem);
    GPL_CUDA(cudaSetDevice(ctx->device));
    const int64_t n = lhs->n_geoms;
    RowClasses lc;
    Scratch<int32_t> ids;
    Scratch<double> dist;  // the dense distance: MODE 1 writes the rows at it
    auto count = [&](int32_t *cnt) -> int {
        GPL_TRY(classify_rows(ctx, lhs, lc));
        GPL_TRY(ids.get(ctx, (size_t)n));
        GPL_TRY(dist.get(ctx, (size_t)n));
        GPL_TRY(geom_run(ctx, idx, lhs, lc.cls.p, lc.box4.p, max_distance, ids.p, dist.p, cnt, nullptr, nullptr, nullptr));
        if (distance) GPL_TRY(deliver(ctx, distance, dist.p, sizeof(double) * (size_t)n, mem));
        return GPL_OK;
    };
    auto write = [&](const int64_t *off, int32_t *raw, double *) {
        return geom_run(ctx, idx, lhs, lc.cls.p, lc.box4.p, max_distance, nullptr, nullptr, nullptr, dist.p, off, raw);
    };
    return pair_list(ctx, n, false, out, count, write);
}

extern "C" int gpl_dwithin_count(gpl_ctx *ctx, const gpl_nearest_index *idx, const gpl_array *lhs, double distance, int32_t *count, int mem) {
    GPL_REQUIRE(ctx && idx && lhs && (count || lhs->n_geoms == 0), GPL_ERR_INVALID_ARG, "gpl_dwithin_count: NULL argument");
    GPL_TRY(check_mem(mem, "gpl_dwithin_count"));
    GPL_TRY(check_dwithin(lhs, distance));
    GPL_CUDA(cudaSetDevice(ctx->device));
    const int64_t n = lhs->n_geoms;
    RowClasses lc;
    if (n && lhs->type != GPL_POINT) GPL_TRY(classify_rows(ctx, lhs, lc));
    RowOut<int32_t> res;
    GPL_TRY(res.get(ctx, count, n, mem));
    GPL_TRY(dwithin_run(ctx, idx, lhs, lc.cls.p, lc.box4.p, distance, res.p, nullptr, nullptr, nullptr));
    return res.deliver(ctx);
}

extern "C" int gpl_dwithin_join_pairs(gpl_ctx *ctx, const gpl_nearest_index *idx, const gpl_array *lhs, double distance, int with_distance,
                                      gpl_pairs **out) {
    GPL_REQUIRE(ctx && idx && lhs && out, GPL_ERR_INVALID_ARG, "gpl_dwithin_join_pairs: NULL argument");
    *out = nullptr;
    GPL_TRY(check_dwithin(lhs, distance));
    GPL_CUDA(cudaSetDevice(ctx->device));
    RowClasses lc;
    auto count = [&](int32_t *cnt) -> int {
        if (lhs->type != GPL_POINT) GPL_TRY(classify_rows(ctx, lhs, lc));
        return dwithin_run(ctx, idx, lhs, lc.cls.p, lc.box4.p, distance, cnt, nullptr, nullptr, nullptr);
    };
    auto write = [&](const int64_t *off, int32_t *raw, double *raw_d) {
        return dwithin_run(ctx, idx, lhs, lc.cls.p, lc.box4.p, distance, nullptr, off, raw, raw_d);
    };
    return pair_list(ctx, lhs->n_geoms, with_distance != 0, out, count, write);
}
