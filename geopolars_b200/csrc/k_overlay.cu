// k_overlay.cu — intersection area of two (Multi)Polygon columns: row-wise (gpl_intersection_area) and as an area-weighted
// overlay join (gpl_overlay_area_join).  geo 0.27 has it as BooleanOps::intersection(..).unsigned_area() (recalled); only the
// area is computed here, never the intersection polygons.  DESIGN.md §4.16 has the derivation.
//
// Every ring is used with its interior on the left: σ = ±1 per ring (exteriors counter-clockwise, holes clockwise), from
// the exact turn at the ring's lexicographically lowest vertex.  B is translated by the symbolic δ = (ε, ε²), which removes
// every degeneracy (shared edges and vertices, vertices on edges) while area(A ∩ (B + δ)) -> area(A ∩ B).  Then
//     area = ½ Σ_{x ∈ ∂A ∪ ∂B} σ_x · cross(x0 − o, x1 − o) · λ(x),
// where λ(x) is the fraction of edge x inside the other region: [x1 inside] (the signed ray-crossing winding sum, which is
// the 0/1 indicator for valid input) plus, at every crossing with the other boundary, +t at an exit and −t at an entry
// (t = o_p / (o_p − o_q) from the f64 orient2d values of x's ends).  Every sign is an exact orient2d sign with the
// coordinate-difference tie-break of the perturbation, so the combinatorics are exact; only t and the sums round.
//
// Layout: one warp per row (or per candidate pair).  Two passes, edges of A against B + δ and edges of B + δ against A.
// The edges of one ring of the outer side go to groups of G lanes (G = 32 / groups, groups = the smallest power of two >= the
// ring's edge count, at most 32); the G lanes of a group stride over the other side's edges, skipping whole rings by their
// boxes, and the group reduces its integer winding and its crossing sum with shuffles.  Each lane then owns λ of its edge,
// so an edge whose end is outside and that crosses nothing contributes exactly 0, and disjoint inputs give exactly 0.0.
// The order of every sum is fixed by the ring sizes alone: the result is deterministic and the join reproduces the
// row-wise value bit for bit.  Per-ring σ and boxes come from a pre-pass (k_ring_prep) over each column.
#include <math.h>

#include "common.cuh"
#include "join_grid.cuh"
#include "output.cuh"
#include "overlay.cuh"
#include "pair_dist.cuh"

namespace gpl {

// k_overlap_area: 4 warps per CTA and 3 CTAs per SM cap it at 170 registers; it needs ~136, and at the default cap of 128
// it spills around the calls into orient2d's adaptive stages
constexpr int kOverlapThreads = 128;

// sign of orient(p, q, s + δ), δ = (ε, ε²): the exact orient2d sign, else the sign of −(q.y − p.y), else of (q.x − p.x).
// o: the f64 orient2d(p, q, s) (its sign is exact)
__device__ __forceinline__ int sgn_at_moved(double2 p, double2 q, double2 s, double &o) {
    o = orient2d(p.x, p.y, q.x, q.y, s.x, s.y);
    if (o != 0.0) return o > 0.0 ? 1 : -1;
    const int c = cmpd(p.y, q.y);
    return c ? c : cmpd(q.x, p.x);
}
// sign of orient(s + δ, g + δ, p): the exact sign, else the sign of (g.y − s.y), else of −(g.x − s.x)
__device__ __forceinline__ int sgn_of_moved(double2 s, double2 g, double2 p, double &o) {
    o = orient2d(s.x, s.y, g.x, g.y, p.x, p.y);
    if (o != 0.0) return o > 0.0 ? 1 : -1;
    const int c = cmpd(g.y, s.y);
    return c ? c : cmpd(s.x, g.x);
}

// per ring of a POLYGON view: σ (0 for a ring with fewer than 4 coordinates after closing, or without a turn at its lowest
// vertex) and the box of its coordinates.  One warp per polygon member; ring k > 0 of a member is a hole.
__global__ void __launch_bounds__(256) k_ring_prep(int64_t n_members, Side v, int8_t *__restrict__ sigma, double4 *__restrict__ box) {
    const int lane = threadIdx.x & 31;
    int64_t warp = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
    const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    const double inf = __longlong_as_double(0x7ff0000000000000LL);
    for (int64_t m = warp; m < n_members; m += nwarps) {
        for (int64_t r = v.go[m]; r < v.go[m + 1]; ++r) {
            const Chain c = part_ring(v, r);
            const int64_t nv = c.coords() - 1;  // distinct positions of the closed ring: vertices 0 .. nv-1
            double x0 = inf, y0 = inf, x1 = -inf, y1 = -inf;
            int64_t best = -1;
            double bx = inf, by = inf;
            for (int64_t i = lane; i < c.n; i += 32) {
                const double2 q = c.p[i];
                x0 = fmin(x0, q.x), y0 = fmin(y0, q.y), x1 = fmax(x1, q.x), y1 = fmax(y1, q.y);
                if (i < nv && (best < 0 || q.x < bx || (q.x == bx && q.y < by))) bx = q.x, by = q.y, best = i;
            }
            x0 = warp_min(x0), y0 = warp_min(y0), x1 = warp_max(x1), y1 = warp_max(y1);
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) {  // lexicographic minimum, lowest index on ties
                const double ox = __shfl_xor_sync(0xffffffffu, bx, o), oy = __shfl_xor_sync(0xffffffffu, by, o);
                const int64_t ob = __shfl_xor_sync(0xffffffffu, best, o);
                if (ob >= 0 && (best < 0 || ox < bx || (ox == bx && (oy < by || (oy == by && ob < best))))) bx = ox, by = oy, best = ob;
            }
            if (lane == 0) {
                int s = 0;
                if (c.coords() >= 4 && best >= 0) {
                    const double2 w = make_double2(bx, by);
                    int64_t j = best, k = best;
                    for (int64_t t = 0; t < nv; ++t) {
                        j = j == 0 ? nv - 1 : j - 1;
                        if (c[j].x != w.x || c[j].y != w.y) break;
                    }
                    for (int64_t t = 0; t < nv; ++t) {
                        k = k + 1 == nv ? 0 : k + 1;
                        if (c[k].x != w.x || c[k].y != w.y) break;
                    }
                    s = orient_sign(c[j], w, c[k]);
                    if (r > v.go[m]) s = -s;
                }
                sigma[r] = (int8_t)s;
                box[r] = make_double4(x0, y0, x1, y1);
            }
        }
    }
}

// One pass of overlap_area: Σ over the edges x of rings [xr0, xr1) of X of σ_x · cross(x0 − o, x1 − o) · λ_Y(x), this lane's
// share.  MOVED_X: X is B (translated by δ) and Y is A; otherwise X is A and Y is B.
template <bool MOVED_X>
__device__ __forceinline__ double overlap_pass(const Side &X, const int8_t *__restrict__ xs, int64_t xr0, int64_t xr1, const Side &Y,
                                               const int8_t *__restrict__ ys, const double4 *__restrict__ ybox, int64_t yr0, int64_t yr1,
                                               double2 o, int lane) {
    double acc = 0.0;
    for (int64_t rx = xr0; rx < xr1; ++rx) {
        const int sx = xs[rx];
        if (sx == 0) continue;
        const Chain cx = part_ring(X, rx);
        const int64_t nseg = cx.coords() - 1;
        int groups = 32;
        while (groups > 1 && groups / 2 >= nseg) groups >>= 1;
        const int G = 32 / groups, grp = lane / G, sub = lane - grp * G;
        for (int64_t base = 0; base < nseg; base += groups) {
            const int64_t i = base + grp;
            double2 a0 = make_double2(0.0, 0.0), a1 = a0;
            bool act = i < nseg;
            if (act) {
                a0 = cx[i], a1 = cx[i + 1];
                act = a0.x != a1.x || a0.y != a1.y;
            }
            int wind = 0;
            double cr = 0.0;
            if (act) {
                // the end of x tested for insideness: a1 (moved by δ when X is B)
                const double ex0 = fmin(a0.x, a1.x), ex1 = fmax(a0.x, a1.x), ey0 = fmin(a0.y, a1.y), ey1 = fmax(a0.y, a1.y);
                for (int64_t ry = yr0; ry < yr1; ++ry) {
                    const int sy = ys[ry];
                    if (sy == 0) continue;
                    const double4 rb = ybox[ry];
                    const bool rbox = !(ex1 < rb.x || rb.z < ex0 || ey1 < rb.y || rb.w < ey0);
                    const bool rray = rb.y <= a1.y && a1.y <= rb.w && rb.z >= a1.x;
                    if (!rbox && !rray) continue;
                    const Chain cy = part_ring(Y, ry);
                    const int64_t ny = cy.coords() - 1;
                    for (int64_t j = sub; j < ny; j += G) {
                        const double2 b0 = cy[j], b1 = cy[j + 1];
                        const bool box = !(ex1 < fmin(b0.x, b1.x) || fmax(b0.x, b1.x) < ex0 || ey1 < fmin(b0.y, b1.y) || fmax(b0.y, b1.y) < ey0);
                        if (!MOVED_X) {  // x = (p, q) of A, y = (s, g) of B + δ
                            const double2 p = a0, q = a1, s = b0, g = b1;
                            const bool straddle = ((s.y < q.y) != (g.y < q.y)) && fmax(s.x, g.x) >= q.x;
                            if (!(straddle || box)) continue;
                            double oq, op, d;
                            const int sq = sgn_of_moved(s, g, q, oq);
                            if (straddle) wind += s.y < q.y ? sy * (sq > 0) : -sy * (sq < 0);
                            if (box) {
                                const int sp = sgn_of_moved(s, g, p, op);
                                if (sp != sq && sgn_at_moved(p, q, s, d) != sgn_at_moved(p, q, g, d)) cr += (double)(sy * sp) * (op / (op - oq));
                            }
                        } else {  // x = (s, g) of B + δ, y = (p, q) of A
                            const double2 s = a0, g = a1, p = b0, q = b1;
                            const bool straddle = ((p.y <= g.y) != (q.y <= g.y)) && fmax(p.x, q.x) > g.x;
                            if (!(straddle || box)) continue;
                            double og, os, d;
                            const int sg = sgn_at_moved(p, q, g, og);
                            if (straddle) wind += p.y <= g.y ? sy * (sg > 0) : -sy * (sg < 0);
                            if (box) {
                                const int ss = sgn_at_moved(p, q, s, os);
                                if (ss != sg && sgn_of_moved(s, g, p, d) != sgn_of_moved(s, g, q, d)) cr += (double)(sy * ss) * (os / (os - og));
                            }
                        }
                    }
                }
            }
            for (int off = G >> 1; off > 0; off >>= 1) {
                wind += __shfl_xor_sync(0xffffffffu, wind, off);
                cr += __shfl_xor_sync(0xffffffffu, cr, off);
            }
            if (act && sub == 0) {
                const double c = (a0.x - o.x) * (a1.y - o.y) - (a1.x - o.x) * (a0.y - o.y);
                acc += (double)sx * c * ((double)wind + cr);
            }
        }
    }
    return acc;
}

// area of closed(A) ∩ closed(B); A = members [am0, am1) of the POLYGON view a, B = members [bm0, bm1) of b; *s: per-ring σ,
// *box: per-ring boxes (k_ring_prep).  Warp cooperative, warp-uniform result, >= 0.  o = the first coordinate of A.
__device__ double overlap_area(const Side &a, const int8_t *__restrict__ as, const double4 *__restrict__ abox, int64_t am0, int64_t am1,
                               const Side &b, const int8_t *__restrict__ bs, const double4 *__restrict__ bbox, int64_t bm0, int64_t bm1,
                               int lane) {
    const int64_t ar0 = a.go[am0], ar1 = a.go[am1], br0 = b.go[bm0], br1 = b.go[bm1];
    if (ar1 <= ar0 || br1 <= br0 || a.ro[ar1] <= a.ro[ar0]) return 0.0;
    const double2 o = a.xy[a.ro[ar0]];
    double acc = overlap_pass<false>(a, as, ar0, ar1, b, bs, bbox, br0, br1, o, lane);
    acc += overlap_pass<true>(b, bs, br0, br1, a, as, abox, ar0, ar1, o, lane);
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, off);
    const double v = 0.5 * acc;
    return v > 0.0 ? v : 0.0;
}

// One warp per row, or per pair of a join (ia / ib select the rows).  am / bm: member offsets of a MultiPolygon column
// (NULL: one member per row).  A null row or a non-finite coordinate gives NaN and validity 0.
__global__ void __launch_bounds__(kOverlapThreads, 3) k_overlap_area(int64_t n, Side a, const int64_t *__restrict__ am, const uint8_t *__restrict__ av,
                                                      const int8_t *__restrict__ as, const double4 *__restrict__ abox, Side b,
                                                      const int64_t *__restrict__ bm, const uint8_t *__restrict__ bv,
                                                      const int8_t *__restrict__ bs, const double4 *__restrict__ bbox,
                                                      const uint64_t *__restrict__ ia, const uint64_t *__restrict__ ib, double *__restrict__ out,
                                                      uint8_t *__restrict__ out_valid) {
    const int lane = threadIdx.x & 31;
    int64_t warp = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
    const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t r = warp; r < n; r += nwarps) {
        const int64_t ra = ia ? (int64_t)ia[r] : r, rb = ib ? (int64_t)ib[r] : r;
        bool ok = bit_get(av, ra) && bit_get(bv, rb);
        double v = nan("");
        if (ok) {
            const int64_t a0 = am ? am[ra] : ra, a1 = am ? am[ra + 1] : ra + 1, b0 = bm ? bm[rb] : rb, b1 = bm ? bm[rb + 1] : rb + 1;
            ok = members_finite(a, a0, a1, lane) && members_finite(b, b0, b1, lane);
            if (ok) v = overlap_area(a, as, abox, a0, a1, b, bs, bbox, b0, b1, lane);
        }
        if (lane == 0) {
            out[r] = ok ? v : nan("");
            if (out_valid) out_valid[r] = ok ? 1 : 0;
        }
    }
}

// per-ring σ and boxes of a (Multi)Polygon column (overlay.cuh)
int ring_prep(gpl_ctx *ctx, const gpl_array *g, RingPrep &out) {
    out.view = polygon_view(g);
    out.members = g->type == GPL_MULTIPOLYGON ? g->geom_off : nullptr;
    const int64_t n_members = g->type == GPL_MULTIPOLYGON ? g->n_parts : g->n_geoms;
    GPL_TRY(out.sigma.get(ctx, (size_t)g->n_rings));
    GPL_TRY(out.box.get(ctx, (size_t)g->n_rings));
    if (n_members > 0) GPL_LAUNCH(ctx, k_ring_prep, warp_grid(n_members, 8), 256, 0, n_members, out.view, out.sigma.p, out.box.p);
    return GPL_OK;
}

}  // namespace gpl

using namespace gpl;

extern "C" int gpl_intersection_area(gpl_ctx *ctx, const gpl_array *a, const gpl_array *b, double *out, uint8_t *out_validity, int mem) {
    GPL_REQUIRE(ctx && a && b && out, GPL_ERR_INVALID_ARG, "gpl_intersection_area: NULL argument");
    GPL_TRY(check_mem(mem, "gpl_intersection_area"));
    GPL_REQUIRE(is_area(a->type) && is_area(b->type), GPL_ERR_INVALID_TYPE, "Expected (Multi)Polygon x (Multi)Polygon (found %s x %s)",
                type_name(a->type), type_name(b->type));
    GPL_TRY(require_same_length(a, b, "intersection_area"));
    GPL_CUDA(cudaSetDevice(ctx->device));
    const int64_t n = a->n_geoms;
    if (n == 0) return GPL_OK;
    RingPrep pa, pb;
    GPL_TRY(ring_prep(ctx, a, pa));
    GPL_TRY(ring_prep(ctx, b, pb));
    RowOut<double> res;
    ValidOut valid;
    GPL_TRY(res.get(ctx, out, n, mem));
    GPL_TRY(valid.get(ctx, out_validity, n, mem, false));
    GPL_LAUNCH(ctx, k_overlap_area, warp_grid(n, kOverlapThreads / 32), kOverlapThreads, 0, n, pa.view, pa.members, a->validity, pa.sigma.p, pa.box.p, pb.view, pb.members,
               b->validity, pb.sigma.p, pb.box.p, nullptr, nullptr, res.p, valid.p);
    GPL_TRY(valid.deliver(ctx));
    return res.deliver(ctx);
}

extern "C" int gpl_overlay_area_join(gpl_ctx *ctx, const gpl_array *lhs, const gpl_array *rhs, gpl_pairs **out) {
    GPL_REQUIRE(ctx && lhs && rhs && out, GPL_ERR_INVALID_ARG, "gpl_overlay_area_join: NULL argument");
    *out = nullptr;
    GPL_REQUIRE(is_area(lhs->type) && is_area(rhs->type), GPL_ERR_INVALID_TYPE, "Expected (Multi)Polygon x (Multi)Polygon (found %s x %s)",
                type_name(lhs->type), type_name(rhs->type));
    GPL_CUDA(cudaSetDevice(ctx->device));
    const int64_t nl = lhs->n_geoms, nr = rhs->n_geoms;
    GPL_REQUIRE(nl < (1LL << 31) && nr < (1LL << 31), GPL_ERR_UNSUPPORTED, "gpl_overlay_area_join: at most 2^31 rows per side");
    Pairs res(nullptr, gpl_pairs_free);
    GPL_TRY(join_candidate_pairs(ctx, lhs, rhs, JOIN_INTERSECTS, "gpl_overlay_area_join", true, res));
    if (res->n > 0) {
        RingPrep pl, pr;
        GPL_TRY(ring_prep(ctx, lhs, pl));
        GPL_TRY(ring_prep(ctx, rhs, pr));
        GPL_LAUNCH(ctx, k_overlap_area, warp_grid(res->n, kOverlapThreads / 32), kOverlapThreads, 0, res->n, pl.view, pl.members, lhs->validity, pl.sigma.p, pl.box.p, pr.view,
                   pr.members, rhs->validity, pr.sigma.p, pr.box.p, res->lhs, res->rhs, res->dist, nullptr);
        GPL_CUDA(cudaStreamSynchronize(ctx->stream));  // the ring tables return to the cache when this scope ends
    }
    *out = res.release();
    return GPL_OK;
}
