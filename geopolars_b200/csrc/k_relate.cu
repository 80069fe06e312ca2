// k_relate.cu — the DE-9IM matrix of two geometry columns of any of the six types, row-wise (gpl_relate), the named OGC
// predicates derived from it (gpl_relate_predicate) and a predicate join (gpl_predicate_join).  DESIGN.md §4.20 has the
// construction and the argument that it is complete.
//
// Every decision is an exact sign of input coordinates; no intersection point is built.  The matrix is filled by samples,
// once with a as X and b as Y and once with the roles swapped (transposed):
//   0-dim  every vertex of X, located in Y (a line's vertex is in X's boundary when it ends an odd number of members, Mod-2),
//          and every proper crossing of an X edge with a Y edge when no vertex of either sits on it;
//   1-dim  every X edge is cut by the Y vertices on it; the symbolic point just after the edge's start and just after each
//          such vertex (SymQ, side 0) is located in Y.  A proper crossing with a polygon edge of Y (no Y vertex on it) puts
//          the pieces on both of its sides in Y's interior and exterior, one each;
//   2-dim  for a polygon X, the points just beside each of those pieces on X's interior and exterior side (side ±σ, σ from
//          ring_prep) are located in Y; the proper crossing of two polygon edges gives II, IE and EI; EE is always 2.
// The matrix is a warp-uniform 27-bit set: bit 3 * (3 * row + col) + d records a sample of dimension d in that entry, and
// an entry's value is its highest bit (F when none).  A predicate stops the row as soon as the set decides it.
// Layout: one warp per row (or per candidate pair of the join); the lanes stride over Y's edges and vertices, skipping
// polygon rings whose box misses the X edge or the sampled point.
#include <math.h>
#include <string.h>

#include "common.cuh"
#include "join_grid.cuh"
#include "join_host.cuh"
#include "output.cuh"
#include "overlay.cuh"
#include "pair_dist.cuh"
#include "scan.cuh"
#include "sym_point.cuh"

namespace gpl {

// k_relate: 4 warps per CTA and 3 CTAs per SM cap it at 170 registers; at the default cap of 128 it spills (as k_overlap_area)
constexpr int kRelateThreads = 128;

enum { LI = 0, LB = 1, LE = 2 };  // interior, boundary, exterior: the matrix's row / column index

// one operand column.  cls 0: coordinates [mo[r], mo[r+1]) (Point: [r, r+1)); cls 1: chains [mo[r], mo[r+1]) (LineString:
// [r, r+1)) with coordinates [ro[k], ro[k+1]); cls 2: polygon members [mo[r], mo[r+1]) (Polygon: [r, r+1)), rings
// [go[m], go[m+1]), coordinates [ro[k], ro[k+1]), σ and box per ring
struct ROp {
    int cls;
    const double2 *xy;
    const int64_t *mo, *go, *ro;
    const int8_t *sigma;
    const double4 *box;
    const uint8_t *valid;
};
struct RRow {
    int64_t m0, m1, k0, k1, c0, c1;  // members, chains / rings, coordinates of the row
};
__device__ __forceinline__ RRow rrow(const ROp &o, int64_t r) {
    RRow w;
    w.m0 = o.mo ? o.mo[r] : r;
    w.m1 = o.mo ? o.mo[r + 1] : r + 1;
    if (o.cls == 0) {
        w.k0 = w.k1 = 0, w.c0 = w.m0, w.c1 = w.m1;
    } else {
        w.k0 = o.cls == 1 ? w.m0 : o.go[w.m0];
        w.k1 = o.cls == 1 ? w.m1 : o.go[w.m1];
        w.c0 = o.ro[w.k0], w.c1 = o.ro[w.k1];
    }
    return w;
}
__device__ __forceinline__ Chain rchain(const ROp &o, int64_t k) {
    return o.cls == 2 ? make_ring(o.xy, o.ro[k], o.ro[k + 1]) : make_line(o.xy, o.ro[k], o.ro[k + 1]);
}

// ---- the matrix as a bit set -----------------------------------------------------------------------------------------
__device__ __forceinline__ int ent_shift(bool tr, int r, int c) { return 3 * (tr ? 3 * c + r : 3 * r + c); }
__device__ __forceinline__ void put(uint32_t &M, bool tr, int r, int c, int d) { M |= 1u << (ent_shift(tr, r, c) + d); }
__device__ __forceinline__ bool have(uint32_t M, bool tr, int r, int c, int d) { return ((M >> ent_shift(tr, r, c)) & 7u) >> d; }

// A predicate: any of n patterns; pattern p holds when every entry named in nz[p] is non-F, every bit of bits[p] is set and
// no bit of f[p] is set.  n = 0: the full matrix is wanted (no early exit).
struct RelSpec {
    int n;
    int empty_equal;  // geom_equals: two empty rows are equal
    int never;        // the operands' dimensions rule the predicate out (every row false, no work)
    uint32_t nz[4], bits[4], f[4];
};
__device__ __forceinline__ uint32_t nonzero_groups(uint32_t M) { return (M | (M >> 1) | (M >> 2)) & 0x09249249u; }
// 1 true, 0 false, -1 not decided yet (entries only grow: an F, '0' or '1' requirement can still break)
__device__ __forceinline__ int spec_decided(const RelSpec &s, uint32_t M) {
    const uint32_t nz = nonzero_groups(M);
    bool all_broken = true;
    for (int p = 0; p < s.n; ++p) {
        const bool broken = (M & s.f[p]) != 0;
        all_broken = all_broken && broken;
        if (!broken && s.f[p] == 0 && (nz & s.nz[p]) == s.nz[p] && (M & s.bits[p]) == s.bits[p]) return 1;
    }
    return all_broken ? 0 : -1;
}
__device__ __forceinline__ bool spec_holds(const RelSpec &s, uint32_t M) {
    const uint32_t nz = nonzero_groups(M);
    for (int p = 0; p < s.n; ++p)
        if ((M & s.f[p]) == 0 && (nz & s.nz[p]) == s.nz[p] && (M & s.bits[p]) == s.bits[p]) return true;
    return false;
}

// ---- exact location of a point or a symbolic point in Y -------------------------------------------------------------
// q is an ordinary point when its v equals its x (and side is 0): every sym_* comparison then reduces to the exact one
__device__ __forceinline__ bool sym_is_point(const SymQ &q) { return q.vx == q.xx && q.vy == q.xy; }
__device__ __forceinline__ bool sym_on_segment(double2 s, double2 e, const SymQ &q) {
    if (sym_orient(s, e, q) != 0) return false;
    const double x0 = fmin(s.x, e.x), x1 = fmax(s.x, e.x), y0 = fmin(s.y, e.y), y1 = fmax(s.y, e.y);
    return sym_cmp_x(q, x0) <= 0 && sym_cmp_x(q, x1) >= 0 && sym_cmp_y(q, y0) <= 0 && sym_cmp_y(q, y1) >= 0;
}
__device__ __forceinline__ bool box_may_hold(double4 b, const SymQ &q) { return q.xx >= b.x && q.xx <= b.z && q.xy >= b.y && q.xy <= b.w; }
// sym_region_pos with the ring boxes: 2 inside / 1 boundary / 0 outside the union of the polygon members [m0, m1)
__device__ __forceinline__ int region_pos(const ROp &y, int64_t m0, int64_t m1, const SymQ &q, int lane) {
    bool boundary = false;
    for (int64_t m = m0; m < m1; ++m) {
        const int64_t r0 = y.go[m], r1 = y.go[m + 1];
        if (r1 <= r0 || !box_may_hold(y.box[r0], q)) continue;
        const int pe = sym_ring_pos(q, rchain(y, r0), lane);
        if (pe == 0) continue;
        if (pe == 1) {
            boundary = true;
            continue;
        }
        bool in_hole = false;
        for (int64_t r = r0 + 1; r < r1 && !in_hole; ++r) {
            if (!box_may_hold(y.box[r], q)) continue;
            const int ph = sym_ring_pos(q, rchain(y, r), lane);
            if (ph == 2) in_hole = true;
            else if (ph == 1) in_hole = boundary = true;
        }
        if (!in_hole) return 2;
    }
    return boundary ? 1 : 0;
}
// the chains of a line row that end at p (both ends of a closed chain count): odd -> p is in the boundary (Mod-2)
__device__ __forceinline__ int ends_at(const ROp &y, const RRow &w, double2 p, int lane) {
    int cnt = 0;
    for (int64_t k = w.k0 + lane; k < w.k1; k += 32) {
        const int64_t c0 = y.ro[k], c1 = y.ro[k + 1];
        if (c1 - c0 < 2) continue;
        const double2 f = y.xy[c0], l = y.xy[c1 - 1];
        cnt += (f.x == p.x && f.y == p.y) + (l.x == p.x && l.y == p.y);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
    return cnt;
}
// LI / LB / LE of q in row w of Y (warp-uniform)
__device__ __noinline__ int locate(const ROp &y, const RRow &w, const SymQ &q, int lane) {
    const bool pt = sym_is_point(q);
    if (y.cls == 0) {
        if (!pt) return LE;
        bool hit = false;
        for (int64_t c = w.c0 + lane; c < w.c1; c += 32) {
            const double2 p = y.xy[c];
            hit = hit || (p.x == q.xx && p.y == q.xy);
        }
        return __any_sync(0xffffffffu, hit) ? LI : LE;
    }
    if (y.cls == 1) {
        if (q.side != 0) return LE;  // a point beside an edge is on no line
        bool on = false;
        for (int64_t k = w.k0; k < w.k1; ++k) {
            const int64_t c0 = y.ro[k], c1 = y.ro[k + 1];
            for (int64_t i = c0 + lane; i + 1 < c1; i += 32) on = on || sym_on_segment(y.xy[i], y.xy[i + 1], q);
        }
        if (!__any_sync(0xffffffffu, on)) return LE;
        if (!pt) return LI;
        return (ends_at(y, w, make_double2(q.xx, q.xy), lane) & 1) ? LB : LI;
    }
    const int pos = region_pos(y, w.m0, w.m1, q, lane);
    return pos == 2 ? LI : pos == 1 ? LB : LE;
}

// is some coordinate of row w of o on both lines u-v and s-e (exactly at their crossing)?
__device__ __noinline__ bool vertex_at(const ROp &o, const RRow &w, double2 u, double2 v, double2 s, double2 e, int lane) {
    bool hit = false;
    for (int64_t c = w.c0 + lane; c < w.c1; c += 32) {
        const double2 p = o.xy[c];
        hit = hit || (orient2d(u.x, u.y, v.x, v.y, p.x, p.y) == 0.0 && orient2d(s.x, s.y, e.x, e.y, p.x, p.y) == 0.0);
    }
    return __any_sync(0xffffffffu, hit);
}
__device__ __forceinline__ bool strictly_inside(double2 c, double2 u, double2 v) {
    if (u.x != v.x) return c.x > fmin(u.x, v.x) && c.x < fmax(u.x, v.x);
    return c.y > fmin(u.y, v.y) && c.y < fmax(u.y, v.y);
}

// the samples of the open piece of X edge (w, v) that starts at w.  xp: X's part the edge belongs to; sig: σ of its ring
// (polygons; 0 for a ring without a turn)
__device__ __forceinline__ void sample_piece(const ROp &X, int sig, double2 w, double2 v, const ROp &Y, const RRow &wy, bool tr, uint32_t &M,
                                             int lane) {
    if (X.cls == 1 || sig == 0) {
        const int xp = X.cls == 1 ? LI : LB;
        if (have(M, tr, xp, LI, 1) && have(M, tr, xp, LB, 1) && have(M, tr, xp, LE, 1)) return;
        put(M, tr, xp, locate(Y, wy, SymQ{w.x, w.y, v.x, v.y, 0}, lane), 1);
        return;
    }
    if (have(M, tr, LI, LI, 2) && have(M, tr, LI, LE, 2) && have(M, tr, LE, LI, 2) && have(M, tr, LB, LI, 1) && have(M, tr, LB, LB, 1) &&
        have(M, tr, LB, LE, 1))
        return;
    const int lin = locate(Y, wy, SymQ{w.x, w.y, v.x, v.y, sig}, lane);
    const int lout = locate(Y, wy, SymQ{w.x, w.y, v.x, v.y, -sig}, lane);
    put(M, tr, LI, lin, 2);
    put(M, tr, LE, lout, 2);
    // a polygon Y: the piece lies where both sides lie, or on Y's boundary when they differ (one side each, valid Y)
    const int lon = Y.cls == 2 ? (lin == lout ? lin : LB) : locate(Y, wy, SymQ{w.x, w.y, v.x, v.y, 0}, lane);
    put(M, tr, LB, lon, 1);
}

// One direction: X = row wx of X, Y = row wy of Y, entries transposed when tr.  Returns the predicate's answer as soon as it
// is decided (-1: not decided, or the full matrix is wanted).
__device__ int relate_pass(const ROp &X, const RRow &wx, const ROp &Y, const RRow &wy, bool tr, const RelSpec &spec, uint32_t &M, int lane) {
    // ---- 0-dim: X's vertices ----------------------------------------------------------------------------------------
    for (int64_t c = wx.c0; c < wx.c1; ++c) {
        const double2 p = X.xy[c];
        const SymQ q{p.x, p.y, p.x, p.y, 0};
        int role = X.cls == 0 ? LI : LB;
        if (X.cls == 1) {
            if (have(M, tr, LI, LI, 0) && have(M, tr, LI, LB, 0) && have(M, tr, LI, LE, 0) && have(M, tr, LB, LI, 0) && have(M, tr, LB, LB, 0) &&
                have(M, tr, LB, LE, 0))
                continue;
            role = (ends_at(X, wx, p, lane) & 1) ? LB : LI;
        }
        if (have(M, tr, role, LI, 0) && have(M, tr, role, LB, 0) && have(M, tr, role, LE, 0)) continue;
        put(M, tr, role, locate(Y, wy, q, lane), 0);
        if (spec.n) {
            const int d = spec_decided(spec, M);
            if (d >= 0) return d;
        }
    }
    if (X.cls == 0) return -1;
    // ---- 1-dim and 2-dim: X's edges ---------------------------------------------------------------------------------
    const int xp = X.cls == 1 ? LI : LB, yp = Y.cls == 2 ? LB : LI;
    for (int64_t k = wx.k0; k < wx.k1; ++k) {
        const Chain cx = rchain(X, k);
        const int sig = X.cls == 2 ? X.sigma[k] : 0;
        const int64_t nx = cx.coords();
        for (int64_t i = 0; i + 1 < nx; ++i) {
            const double2 u = cx[i], v = cx[i + 1];
            if (u.x == v.x && u.y == v.y) continue;
            sample_piece(X, sig, u, v, Y, wy, tr, M, lane);
            if (Y.cls > 0) {
                const double ex0 = fmin(u.x, v.x), ex1 = fmax(u.x, v.x), ey0 = fmin(u.y, v.y), ey1 = fmax(u.y, v.y);
                for (int64_t ky = wy.k0; ky < wy.k1; ++ky) {
                    if (Y.cls == 2) {
                        const double4 b = Y.box[ky];
                        if (b.x > ex1 || b.z < ex0 || b.y > ey1 || b.w < ey0) continue;
                    }
                    const Chain cy = rchain(Y, ky);
                    const int64_t ny = cy.coords();
                    for (int64_t j0 = 0; j0 < ny; j0 += 32) {
                        const int64_t j = j0 + lane;
                        bool touch = false, cross = false;
                        double2 s = make_double2(0.0, 0.0), e = s;
                        if (j < ny) {
                            s = cy[j];
                            const int o1 = orient_sign(u, v, s);
                            touch = j < cy.n && o1 == 0 && strictly_inside(s, u, v);
                            if (j + 1 < ny && o1 != 0) {
                                e = cy[j + 1];
                                const int o2 = orient_sign(u, v, e);
                                if (o1 * o2 < 0) cross = orient_sign(s, e, u) * orient_sign(s, e, v) < 0;
                            }
                        }
                        unsigned mt = __ballot_sync(0xffffffffu, touch);
                        while (mt) {  // a Y vertex inside the edge: the piece after it
                            const int src = __ffs(mt) - 1;
                            mt &= mt - 1;
                            sample_piece(X, sig, bcast2(s, src), v, Y, wy, tr, M, lane);
                        }
                        unsigned mc = __ballot_sync(0xffffffffu, cross);
                        while (mc) {  // a proper crossing: its point, and the pieces and faces around it
                            const int src = __ffs(mc) - 1;
                            mc &= mc - 1;
                            const bool side_done = (Y.cls != 2 || (have(M, tr, xp, LI, 1) && have(M, tr, xp, LE, 1))) &&
                                                   (X.cls != 2 || Y.cls != 2 ||
                                                    (have(M, tr, LI, LI, 2) && have(M, tr, LI, LE, 2) && have(M, tr, LE, LI, 2)));
                            const bool point_done = have(M, tr, xp, yp, 0);
                            if (side_done && point_done) continue;
                            const double2 ss = bcast2(s, src), ee = bcast2(e, src);
                            if (vertex_at(Y, wy, u, v, ss, ee, lane)) continue;  // the Y vertex there is sampled as an event
                            if (Y.cls == 2) {
                                put(M, tr, xp, LI, 1), put(M, tr, xp, LE, 1);
                                if (X.cls == 2) put(M, tr, LI, LI, 2), put(M, tr, LI, LE, 2), put(M, tr, LE, LI, 2);
                            }
                            if (!point_done && !vertex_at(X, wx, u, v, ss, ee, lane)) put(M, tr, xp, yp, 0);
                        }
                    }
                }
            }
            if (spec.n) {
                const int d = spec_decided(spec, M);
                if (d >= 0) return d;
            }
        }
    }
    return -1;
}

// a line row has a boundary point when some chain end is the end of an odd number of chains (Mod-2)
__device__ __forceinline__ bool lines_have_boundary(const ROp &o, const RRow &w, int lane) {
    for (int64_t k = w.k0; k < w.k1; ++k) {
        const int64_t c0 = o.ro[k], c1 = o.ro[k + 1];
        if (c1 - c0 < 2) continue;
        if ((ends_at(o, w, o.xy[c0], lane) & 1) || (ends_at(o, w, o.xy[c1 - 1], lane) & 1)) return true;
    }
    return false;
}

// box of the row's coordinates (x0 > x1 when it has none); ok = every coordinate is finite
__device__ __forceinline__ double4 row_box(const ROp &o, const RRow &w, bool &ok, int lane) {
    const double inf = __longlong_as_double(0x7ff0000000000000LL);
    double x0 = inf, y0 = inf, x1 = -inf, y1 = -inf;
    bool fin = true;
    for (int64_t c = w.c0 + lane; c < w.c1; c += 32) {
        const double2 q = o.xy[c];
        fin = fin && isfinite(q.x) && isfinite(q.y);
        x0 = fmin(x0, q.x), y0 = fmin(y0, q.y), x1 = fmax(x1, q.x), y1 = fmax(y1, q.y);
    }
    ok = __all_sync(0xffffffffu, fin);
    return make_double4(warp_min(x0), warp_min(y0), warp_max(x1), warp_max(y1));
}

// the row pair (ra, rb): false for a null matrix.  M: the matrix; res: the predicate (when spec.n > 0)
__device__ __forceinline__ bool relate_row(const ROp &a, int64_t ra, const ROp &b, int64_t rb, const RelSpec &spec, uint32_t &M, bool &res,
                                           int lane) {
    M = 0;
    res = false;
    if (!bit_get(a.valid, ra) || !bit_get(b.valid, rb)) return false;
    const RRow wa = rrow(a, ra), wb = rrow(b, rb);
    bool fa, fb;
    const double4 ba = row_box(a, wa, fa, lane), bb = row_box(b, wb, fb, lane);
    if (!fa || !fb) return false;
    const bool ea = wa.c1 == wa.c0, eb = wb.c1 == wb.c0;
    if (spec.n && ea && eb && spec.empty_equal) {
        res = true;
        return true;
    }
    put(M, false, LE, LE, 2);
    if (ba.x > bb.z || bb.x > ba.z || ba.y > bb.w || bb.y > ba.w) {  // disjoint envelopes (or an empty side): X meets Y's exterior only
        if (!ea) {
            put(M, false, LI, LE, a.cls);
            if (a.cls == 2 || (a.cls == 1 && lines_have_boundary(a, wa, lane))) put(M, false, LB, LE, a.cls - 1);
        }
        if (!eb) {
            put(M, true, LI, LE, b.cls);
            if (b.cls == 2 || (b.cls == 1 && lines_have_boundary(b, wb, lane))) put(M, true, LB, LE, b.cls - 1);
        }
    } else {
        int d = relate_pass(a, wa, b, wb, false, spec, M, lane);
        if (d < 0) d = relate_pass(b, wb, a, wa, true, spec, M, lane);
        if (d >= 0) {
            res = d == 1;
            return true;
        }
    }
    if (spec.n) res = spec_holds(spec, M);
    return true;
}

// One warp per row, or per candidate pair (ia / ib select the rows).  mat: 9 int8 per row (-1 = F), or NULL; ok: 1 for a
// non-null matrix (may be NULL); out: the predicate's byte (spec.n > 0)
__global__ void __launch_bounds__(kRelateThreads, 3) k_relate(int64_t n, ROp a, ROp b, const uint64_t *__restrict__ ia, const uint64_t *__restrict__ ib,
                                                RelSpec spec, int8_t *__restrict__ mat, uint8_t *__restrict__ ok, uint8_t *__restrict__ out) {
    const int lane = threadIdx.x & 31;
    int64_t warp = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
    const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t r = warp; r < n; r += nwarps) {
        const int64_t ra = ia ? (int64_t)ia[r] : r, rb = ib ? (int64_t)ib[r] : r;
        uint32_t M = 0;
        bool res = false;
        const bool good = !spec.never && relate_row(a, ra, b, rb, spec, M, res, lane);
        if (mat && lane < 9) {
            const uint32_t g = (M >> (3 * lane)) & 7u;
            mat[9 * r + lane] = good ? (int8_t)(g >= 4 ? 2 : g >= 2 ? 1 : g ? 0 : -1) : (int8_t)-1;
        }
        if (lane == 0) {
            if (ok) ok[r] = good ? 1 : 0;
            if (out) out[r] = res ? 1 : 0;
        }
    }
}

// ---- host side --------------------------------------------------------------------------------------------------------
static int cls_of(int t) {
    return (t == GPL_POINT || t == GPL_MULTIPOINT) ? 0 : (t == GPL_LINESTRING || t == GPL_MULTILINESTRING) ? 1 : 2;
}
// the column as an ROp; a (Multi)Polygon column gets its ring σ / boxes in prep
static int make_op(gpl_ctx *ctx, const gpl_array *g, RingPrep &prep, ROp &o) {
    const double2 *xy = reinterpret_cast<const double2 *>(g->xy);
    const bool multi = is_multi(g->type);
    o = ROp{cls_of(g->type), xy, multi ? g->geom_off : nullptr, nullptr, nullptr, nullptr, nullptr, g->validity};
    if (o.cls == 1) o.ro = g->type == GPL_LINESTRING ? g->geom_off : g->ring_off;
    if (o.cls == 2) {
        GPL_TRY(ring_prep(ctx, g, prep));
        o.go = prep.view.go, o.ro = prep.view.ro, o.sigma = prep.sigma.p, o.box = prep.box.p;
    }
    return GPL_OK;
}

// a 9-character pattern over TF*012 (either case) -> one RelSpec pattern
static bool add_pattern(RelSpec &s, const char *pat) {
    if (!pat || strlen(pat) != 9 || s.n >= 4) return false;
    uint32_t nz = 0, bits = 0, f = 0;
    for (int i = 0; i < 9; ++i) {
        const int sh = 3 * i;
        switch (pat[i]) {
        case '*': break;
        case 'T': case 't': nz |= 1u << sh; break;
        case 'F': case 'f': f |= 7u << sh; break;
        case '0': bits |= 1u << sh, f |= 6u << sh; break;
        case '1': bits |= 2u << sh, f |= 4u << sh; break;
        case '2': bits |= 4u << sh; break;
        default: return false;
        }
    }
    s.nz[s.n] = nz, s.bits[s.n] = bits, s.f[s.n] = f;
    ++s.n;
    return true;
}
// the RelSpec of a predicate for operands of dimensions da, db (JTS's definitions); false: unknown predicate or bad pattern
static bool make_spec(int predicate, const char *pattern, int da, int db, RelSpec &s) {
    memset(&s, 0, sizeof(s));
    auto any = [&](std::initializer_list<const char *> l) {
        for (const char *p : l) add_pattern(s, p);
        return true;
    };
    switch (predicate) {
    case GPL_PREDICATE_INTERSECTS: return any({"T********", "*T*******", "***T*****", "****T****"});
    case GPL_PREDICATE_CONTAINS: return any({"T*****FF*"});
    case GPL_PREDICATE_WITHIN: return any({"T*F**F***"});
    case GPL_PREDICATE_CONTAINS_PROPERLY: return any({"T**FF*FF*"});
    case GPL_PREDICATE_COVERS: return any({"T*****FF*", "*T****FF*", "***T**FF*", "****T*FF*"});
    case GPL_PREDICATE_COVERED_BY: return any({"T*F**F***", "*TF**F***", "**FT*F***", "**F*TF***"});
    case GPL_PREDICATE_TOUCHES:
        if (da == 0 && db == 0) s.never = 1;
        return any({"FT*******", "F**T*****", "F***T****"});
    case GPL_PREDICATE_CROSSES:
        if (da < db) return any({"T*T******"});
        if (da > db) return any({"T*****T**"});
        if (da == 1) return any({"0********"});
        s.never = 1;
        return true;
    case GPL_PREDICATE_OVERLAPS:
        if (da != db) s.never = 1;
        return any({da == 1 ? "1*T***T**" : "T*T***T**"});
    case GPL_PREDICATE_DISJOINT: return any({"FF*FF****"});
    case GPL_PREDICATE_EQUALS:
        if (da != db) s.never = 1;
        s.empty_equal = 1;
        return any({"T*F**FFF*"});
    case GPL_PREDICATE_PATTERN: return add_pattern(s, pattern);
    default: return false;
    }
}

static int check_pair(const gpl_array *a, const gpl_array *b, const char *who) {
    GPL_REQUIRE(known_type(a->type) && known_type(b->type), GPL_ERR_INVALID_TYPE, "%s: unsupported geometry pair %s x %s", who,
                type_name(a->type), type_name(b->type));
    return GPL_OK;
}

}  // namespace gpl

using namespace gpl;

extern "C" int gpl_relate(gpl_ctx *ctx, const gpl_array *a, const gpl_array *b, int8_t *matrix, uint8_t *out_validity, int mem) {
    GPL_REQUIRE(ctx && a && b && matrix, GPL_ERR_INVALID_ARG, "gpl_relate: NULL argument");
    GPL_TRY(check_mem(mem, "gpl_relate"));
    GPL_TRY(require_same_length(a, b, "relate"));
    GPL_TRY(check_pair(a, b, "relate"));
    GPL_CUDA(cudaSetDevice(ctx->device));
    const int64_t n = a->n_geoms;
    if (n == 0) return GPL_OK;
    RingPrep pa, pb;
    ROp oa, ob;
    GPL_TRY(make_op(ctx, a, pa, oa));
    GPL_TRY(make_op(ctx, b, pb, ob));
    RelSpec full;
    memset(&full, 0, sizeof(full));
    RowOut<int8_t> mat;
    ValidOut valid;
    GPL_TRY(mat.get(ctx, matrix, n * 9, mem));
    GPL_TRY(valid.get(ctx, out_validity, n, mem, true));
    GPL_LAUNCH(ctx, k_relate, warp_grid(n, kRelateThreads / 32), kRelateThreads, 0, n, oa, ob, nullptr, nullptr, full, mat.p, valid.p, nullptr);
    GPL_TRY(valid.deliver(ctx));
    return mat.deliver(ctx);
}

extern "C" int gpl_relate_predicate(gpl_ctx *ctx, const gpl_array *a, const gpl_array *b, int predicate, const char *pattern, uint8_t *out_bitmap,
                                    int mem) {
    GPL_REQUIRE(ctx && a && b && out_bitmap, GPL_ERR_INVALID_ARG, "gpl_relate_predicate: NULL argument");
    GPL_TRY(check_mem(mem, "gpl_relate_predicate"));
    GPL_TRY(require_same_length(a, b, "relate_predicate"));
    GPL_TRY(check_pair(a, b, "relate_predicate"));
    RelSpec spec;
    GPL_REQUIRE(make_spec(predicate, pattern, cls_of(a->type), cls_of(b->type), spec), GPL_ERR_INVALID_ARG,
                "relate_predicate: unknown predicate %d or a pattern that is not 9 characters of TF*012", predicate);
    GPL_CUDA(cudaSetDevice(ctx->device));
    const int64_t n = a->n_geoms;
    if (n == 0) return GPL_OK;
    RingPrep pa, pb;
    ROp oa, ob;
    GPL_TRY(make_op(ctx, a, pa, oa));
    GPL_TRY(make_op(ctx, b, pb, ob));
    Scratch<uint8_t> bytes;
    GPL_TRY(bytes.get(ctx, (size_t)n));
    GPL_LAUNCH(ctx, k_relate, warp_grid(n, kRelateThreads / 32), kRelateThreads, 0, n, oa, ob, nullptr, nullptr, spec, nullptr, nullptr, bytes.p);
    return finish_bitmap(ctx, bytes.p, n, out_bitmap, mem);
}

extern "C" int gpl_predicate_join(gpl_ctx *ctx, const gpl_array *lhs, const gpl_array *rhs, int predicate, const char *pattern, gpl_pairs **out) {
    GPL_REQUIRE(ctx && lhs && rhs && out, GPL_ERR_INVALID_ARG, "gpl_predicate_join: NULL argument");
    *out = nullptr;
    GPL_TRY(check_pair(lhs, rhs, "predicate_join"));
    RelSpec spec;
    GPL_REQUIRE(make_spec(predicate, pattern, cls_of(lhs->type), cls_of(rhs->type), spec), GPL_ERR_INVALID_ARG,
                "predicate_join: unknown predicate %d or a pattern that is not 9 characters of TF*012", predicate);
    // envelope candidates miss the pairs that are disjoint: a predicate that can hold for them has no candidate list
    bool needs_contact = true;
    for (int p = 0; p < spec.n; ++p) {
        const uint32_t contact = 0x3fu | (0x3fu << 9);  // the II, IB, BI and BB entries
        needs_contact = needs_contact && ((spec.nz[p] | spec.bits[p]) & contact) != 0;
    }
    GPL_REQUIRE(needs_contact || spec.never, GPL_ERR_INVALID_ARG,
                "predicate_join: the predicate can hold for disjoint pairs (disjoint, or a pattern with II, IB, BI and BB all F or *)");
    GPL_CUDA(cudaSetDevice(ctx->device));
    const int64_t nl = lhs->n_geoms, nr = rhs->n_geoms;
    GPL_REQUIRE(nl < (1LL << 31) && nr < (1LL << 31), GPL_ERR_UNSUPPORTED, "gpl_predicate_join: at most 2^31 rows per side");
    // every accepted predicate implies intersects: the candidates are the pairs gpl_intersects accepts, in (lhs, rhs) order
    Pairs cand(nullptr, gpl_pairs_free);
    GPL_TRY(spec.never ? pairs_new(ctx, 0, false, cand) : join_candidate_pairs(ctx, lhs, rhs, JOIN_INTERSECTS, "gpl_predicate_join", false, cand));
    const int64_t n = cand->n;
    if (predicate == GPL_PREDICATE_INTERSECTS || n == 0) {
        *out = cand.release();
        return GPL_OK;
    }
    RingPrep pl, pr;
    ROp ol, orr;
    GPL_TRY(make_op(ctx, lhs, pl, ol));
    GPL_TRY(make_op(ctx, rhs, pr, orr));
    Scratch<uint8_t> hit;
    GPL_TRY(hit.get(ctx, (size_t)n));
    GPL_LAUNCH(ctx, k_relate, warp_grid(n, kRelateThreads / 32), kRelateThreads, 0, n, ol, orr, cand->lhs, cand->rhs, spec, nullptr, nullptr, hit.p);
    Pairs res(nullptr, gpl_pairs_free);
    GPL_TRY(keep_pairs(ctx, cand.get(), hit.p, res));
    *out = res.release();
    return GPL_OK;
}
