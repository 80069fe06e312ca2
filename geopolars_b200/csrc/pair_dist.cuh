// pair_dist.cuh — the row-pair routines of GeoSeries::distance and GeoSeries::intersects for linestrings and polygons
// (geo 0.27, recalled; restated in oracle/geo_oracle.c), shared by the row-wise kernels of k_pairs.cu and the
// geometry-query nearest join of k_nearest_geom.cu.  Every routine is warp cooperative: all 32 lanes call it with the
// same rows, and the result is warp-uniform.
#pragma once

#include "common.cuh"
#include "point_dist.cuh"

namespace gpl {


struct Coords {  // accessor over either staging area
    const double2 *p;
    __device__ __forceinline__ double2 operator[](int64_t i) const { return p[i]; }
};

__device__ __forceinline__ bool seg_bbox_disjoint(double2 a0, double2 a1, double2 b0, double2 b1) {
    return fmax(a0.x, a1.x) < fmin(b0.x, b1.x) || fmax(b0.x, b1.x) < fmin(a0.x, a1.x) || fmax(a0.y, a1.y) < fmin(b0.y, b1.y) ||
           fmax(b0.y, b1.y) < fmin(a0.y, a1.y);
}
__device__ __forceinline__ bool line_intersects_coord(double2 s, double2 e, double2 c) {
    return orient_sign(s, e, c) == 0 && point_in_rect(c, s, e);
}
// impl Intersects<Line> for Line, self = (s0,e0), rhs = (s1,e1)
__device__ __forceinline__ bool line_intersects_line(double2 s0, double2 e0, double2 s1, double2 e1) {
    if (s0.x == e0.x && s0.y == e0.y) return line_intersects_coord(s1, e1, s0);
    int c11 = orient_sign(s0, e0, s1);
    int c12 = orient_sign(s0, e0, e1);
    if (c11 != c12) {
        int c21 = orient_sign(s1, e1, s0);
        int c22 = orient_sign(s1, e1, e0);
        return c21 != c22;
    } else if (c11 == 0) {
        return point_in_rect(s1, s0, e0) || point_in_rect(e1, s0, e0) || point_in_rect(e0, s1, e1);
    }
    return false;
}

// LineString x LineString intersects, warp cooperative.  Result is warp-uniform.  CA / CB: anything indexable
// that yields double2 (Coords, Chain).
template <class CA, class CB>
__device__ __forceinline__ bool ls_intersects_ls(CA A, int64_t na, CB B, int64_t nb, int lane) {
    if (na < 2 || nb < 2) return false;  // no lines() on either side
    // has_disjoint_bboxes
    const double inf = __longlong_as_double(0x7ff0000000000000LL);
    double ax0 = inf, ay0 = inf, ax1 = -inf, ay1 = -inf, bx0 = inf, by0 = inf, bx1 = -inf, by1 = -inf;
    for (int64_t i = lane; i < na; i += 32) {
        double2 q = A[i];
        ax0 = fmin(ax0, q.x), ay0 = fmin(ay0, q.y), ax1 = fmax(ax1, q.x), ay1 = fmax(ay1, q.y);
    }
    for (int64_t i = lane; i < nb; i += 32) {
        double2 q = B[i];
        bx0 = fmin(bx0, q.x), by0 = fmin(by0, q.y), bx1 = fmax(bx1, q.x), by1 = fmax(by1, q.y);
    }
    ax0 = warp_min(ax0), ay0 = warp_min(ay0), ax1 = warp_max(ax1), ay1 = warp_max(ay1);
    bx0 = warp_min(bx0), by0 = warp_min(by0), bx1 = warp_max(bx1), by1 = warp_max(by1);
    if (ax0 > bx1 || bx0 > ax1 || ay0 > by1 || by0 > ay1) return false;
    const int64_t sa = na - 1, sb = nb - 1, total = sa * sb;
    for (int64_t base = 0; base < total; base += 32) {
        int64_t t = base + lane;
        bool hit = false;
        if (t < total) {
            int64_t i = t / sb, j = t - i * sb;
            double2 a0 = A[i], a1 = A[i + 1], b0 = B[j], b1 = B[j + 1];
            if (!seg_bbox_disjoint(a0, a1, b0, b1)) hit = line_intersects_line(b0, b1, a0, a1);
        }
        if (__any_sync(0xffffffffu, hit)) return true;
    }
    return false;
}

// squared distance point -> segment with the reference's case split and cross-product expression
__device__ __forceinline__ double seg_dist2(double2 p, double2 s, double2 e) {
    double dx = e.x - s.x, dy = e.y - s.y;
    double wx = p.x - s.x, wy = p.y - s.y;
    if (dx == 0.0 && dy == 0.0) return wx * wx + wy * wy;  // start == end
    double dd = dx * dx + dy * dy;
    double num = wx * dx + wy * dy;
    if (num <= 0.0) return wx * wx + wy * wy;  // r <= 0
    if (num >= dd) {                             // r >= 1 (exact: the correctly rounded quotient is >= 1 iff num >= dd)
        double ux = p.x - e.x, uy = p.y - e.y;
        return ux * ux + uy * uy;
    }
    double cross = (s.y - p.y) * dx - (s.x - p.x) * dy;
    return (cross * cross) / dd;
}

template <class CA, class CB>
__device__ __forceinline__ double ls_ls_min_dist2(CA A, int64_t na, CB B, int64_t nb, int lane) {
    const double big = 1.7976931348623157e308;
    double best = big;
    const int64_t sa = na - 1, sb = nb - 1;
    const int64_t t1 = nb * sa, total = t1 + na * sb;
    for (int64_t t = lane; t < total; t += 32) {
        double d;
        if (t < t1) {  // vertex j of B against segment i of A
            int64_t j = t / sa, i = t - j * sa;
            d = seg_dist2(B[j], A[i], A[i + 1]);
        } else {
            int64_t u = t - t1;
            int64_t i = u / sb, j = u - i * sb;
            d = seg_dist2(A[i], B[j], B[j + 1]);
        }
        best = fmin(best, d);
    }
    return warp_min(best);
}

// ---- fast paths for short linestrings (<= 33 coords per side, staged in shared memory) ----------------
constexpr int kPairQueue = 64;

// sign of orient2d(a,b,c) when the stage-A filter certifies it (non-zero), else 0 and `unsure` is raised
__device__ __forceinline__ int certified_sign(double2 a, double2 b, double2 c, bool &unsure) {
    const double dl = (a.x - c.x) * (b.y - c.y);
    const double dr = (a.y - c.y) * (b.x - c.x);
    const double det = dl - dr;
    const bool certain = fabs(det) > kCcwA * (fabs(dl) + fabs(dr));
    unsure = unsure || !certain;
    return certain ? ((det > 0.0) ? 1 : -1) : 0;
}

// intersects for na, nb <= 33.  A, B: the row's coordinates in SHARED memory; box: per-warp scratch of 64
// float4 (conservative float bounding boxes of A's and B's segments: min rounded down, max rounded up — a
// looser box only adds candidates); queue: per-warp scratch of kPairQueue ushorts.  Warp-uniform result:
// 0 / 1 = geo's answer (has_disjoint_bboxes of the whole linestrings is implied: disjoint boxes give no
// candidate), 2 = undecided by the filter: the row goes to k_ls_ls_exact.
__device__ __forceinline__ int ls_intersects_ls_short(const double2 *A, int32_t na, const double2 *B, int32_t nb, float4 *box,
                                                      unsigned short *queue, int lane) {
    if (na < 2 || nb < 2) return 0;
    const int32_t sa = na - 1, sb = nb - 1;
    if (lane < sa) {
        const double2 p = A[lane], q = A[lane + 1];
        box[lane] = make_float4(__double2float_rd(fmin(p.x, q.x)), __double2float_rd(fmin(p.y, q.y)), __double2float_ru(fmax(p.x, q.x)),
                                __double2float_ru(fmax(p.y, q.y)));
    }
    if (lane < sb) {
        const double2 p = B[lane], q = B[lane + 1];
        box[32 + lane] = make_float4(__double2float_rd(fmin(p.x, q.x)), __double2float_rd(fmin(p.y, q.y)),
                                     __double2float_ru(fmax(p.x, q.x)), __double2float_ru(fmax(p.y, q.y)));
    }
    __syncwarp();
    const int32_t total = sa * sb;
    // (i, j) of this lane's segment pair, advanced by 32 pairs per step without dividing
    int32_t i = lane / sb, j = lane - i * sb;
    const int32_t di = 32 / sb, dj = 32 - di * sb;
    int32_t qn = 0;
    bool unsure_any = false;
    for (int32_t base = 0; base < total || qn > 0; base += 32) {
        // 1. bbox filter of 32 segment pairs, survivors appended to the queue
        bool cand = false;
        if (base + lane < total) {
            const float4 x = box[i], y = box[32 + j];
            cand = !(x.z < y.x || y.z < x.x || x.w < y.y || y.w < x.y);
        }
        const unsigned m = __ballot_sync(0xffffffffu, cand);
        if (cand) queue[qn + __popc(m & ((1u << lane) - 1u))] = (unsigned short)((i << 8) | j);
        qn += __popc(m);
        i += di, j += dj;
        if (j >= sb) j -= sb, ++i;
        __syncwarp();
        // 2. dense exact-sign test of up to 32 queued candidates (when a full batch is available, or at the end)
        if (qn >= 32 || (base + 32 >= total && qn > 0)) {
            const int32_t take = min(qn, 32);
            bool hit = false, unsure = false;
            if (lane < take) {
                const unsigned short c = queue[qn - take + lane];
                const int32_t ci = c >> 8, cj = c & 0xff;
                const double2 a0 = A[ci], a1 = A[ci + 1], b0 = B[cj], b1 = B[cj + 1];
                // geo: self = (b0,b1), rhs = (a0,a1)
                const int c11 = certified_sign(b0, b1, a0, unsure), c12 = certified_sign(b0, b1, a1, unsure);
                const int c21 = certified_sign(a0, a1, b0, unsure), c22 = certified_sign(a0, a1, b1, unsure);
                hit = !unsure && c11 != c12 && c21 != c22;
                // certified c11 == c12 (both non-zero) means "no intersection" whatever c21/c22 are
                if (c11 != 0 && c11 == c12) unsure = false;
            }
            if (__any_sync(0xffffffffu, hit)) return 1;
            unsure_any = unsure_any || __any_sync(0xffffffffu, unsure);
            qn -= take;
            __syncwarp();
        }
    }
    return unsure_any ? 2 : 0;  // 2: some candidate was collinear / degenerate / too close to call and nothing certified
}

// min distance for na, nb <= 33, not intersecting: fraction-tracked squared distance, branch-free
__device__ __forceinline__ double ls_ls_distance_short(const double2 *A, int32_t na, const double2 *B, int32_t nb, int lane) {
    const int32_t sa = na - 1, sb = nb - 1;
    double best_n = 1.7976931348623157e308, best_d = 1.0;
    // two sweeps with the same body: vertices of P against segments of S
    for (int sweep = 0; sweep < 2; ++sweep) {
        const double2 *P = sweep == 0 ? B : A, *S = sweep == 0 ? A : B;
        const int32_t np = sweep == 0 ? nb : na, ns = sweep == 0 ? sa : sb;
        const int32_t total = np * ns;
        int32_t pi = lane / ns, si = lane - pi * ns;
        const int32_t dp = 32 / ns, ds = 32 - dp * ns;
        for (int32_t t = lane; t < total; t += 32) {
            const double2 p = P[pi], s = S[si], e = S[si + 1];
            const double dx = e.x - s.x, dy = e.y - s.y;
            const double wx = p.x - s.x, wy = p.y - s.y;
            const double ux = p.x - e.x, uy = p.y - e.y;
            const double dd = dx * dx + dy * dy;
            const double num = wx * dx + wy * dy;
            const double ww = wx * wx + wy * wy, uu = ux * ux + uy * uy;
            const double cross = (s.y - p.y) * dx - (s.x - p.x) * dy;  // the reference's expression
            const bool interior = num > 0.0 && num < dd;               // 0 < r < 1 (exact: see seg_dist2)
            const double n = interior ? cross * cross : ((num <= 0.0 || dd == 0.0) ? ww : uu);
            const double d = interior ? dd : 1.0;
            if (n * best_d < best_n * d) {
                best_n = n;
                best_d = d;
            }
            pi += dp, si += ds;
            if (si >= ns) si -= ns, ++pi;
        }
    }
    double v = best_n / best_d;
    v = warp_min(v);
    return sqrt(v);
}

// ---- generic row-wise intersects: every pair of GeoArrow types --------------------------------------------
// geo 0.27 intersects/{coordinate,line,line_string,polygon,collections}.rs (recalled).  The boolean is decided
// by exact predicates only, so any exact decision procedure gives geo's answer on valid input; the parts of
// geo's procedure that are NOT neutral on invalid input (polygon-level rejects use the EXTERIOR ring's box,
// Polygon x Coord is `exterior != Outside && no hole strictly contains it`, Polygon x Polygon tests all rings
// of `other` against `self` but only self's exterior against `other`) are reproduced as they are.
// One shortcut is taken: where geo tests every vertex of a chain against a polygon after all segment pairs
// failed, the first vertex is tested — with no crossing of any ring the chain lies in one face of the ring
// arrangement, so all its vertices give the same answer (the oracle tests every vertex, the tests compare).
struct Chain {  // a linestring, or a ring with Polygon::new's closing coordinate emulated
    const double2 *p;
    int64_t n;
    bool closing;
    __device__ __forceinline__ int64_t coords() const { return n + (closing ? 1 : 0); }
    __device__ __forceinline__ double2 operator[](int64_t i) const { return p[i < n ? i : 0]; }
};
__device__ __forceinline__ Chain make_line(const double2 *xy, int64_t c0, int64_t c1) { return Chain{xy + c0, c1 - c0, false}; }
__device__ __forceinline__ Chain make_ring(const double2 *xy, int64_t c0, int64_t c1) {
    const int64_t n = c1 - c0;
    bool closing = false;
    if (n >= 2) {
        const double2 f = xy[c0], l = xy[c1 - 1];
        closing = !(f.x == l.x && f.y == l.y);
    }
    return Chain{xy + c0, n, closing};
}
struct Box {
    double x0, y0, x1, y1;
    bool has;
};
__device__ __forceinline__ Box chain_box(const Chain &c, int lane) {
    const double inf = __longlong_as_double(0x7ff0000000000000LL);
    Box b{inf, inf, -inf, -inf, c.n > 0};
    for (int64_t i = lane; i < c.n; i += 32) {
        const double2 q = c.p[i];
        b.x0 = fmin(b.x0, q.x), b.y0 = fmin(b.y0, q.y), b.x1 = fmax(b.x1, q.x), b.y1 = fmax(b.y1, q.y);
    }
    b.x0 = warp_min(b.x0), b.y0 = warp_min(b.y0), b.x1 = warp_max(b.x1), b.y1 = warp_max(b.y1);
    return b;
}
// has_disjoint_bboxes: only when both sides have a box
__device__ __forceinline__ bool boxes_disjoint(const Box &a, const Box &b) {
    return a.has && b.has && (a.x0 > b.x1 || b.x0 > a.x1 || a.y0 > b.y1 || b.y0 > a.y1);
}

__device__ __forceinline__ int side_class(int t) { return (t == GPL_POINT || t == GPL_MULTIPOINT) ? 0 : (t == GPL_LINESTRING || t == GPL_MULTILINESTRING) ? 1 : 2; }
// sub-geometries of row r: points [lo,hi) of class 0; chains of class 1; polygon parts of class 2
__device__ __forceinline__ void side_range(const Side &s, int64_t r, int64_t &lo, int64_t &hi) {
    if (s.type == GPL_POINT) lo = r, hi = r + 1;
    else if (s.type == GPL_LINESTRING || s.type == GPL_POLYGON) lo = 0, hi = 1;
    else lo = s.go[r], hi = s.go[r + 1];
}
__device__ __forceinline__ Chain side_chain(const Side &s, int64_t r, int64_t k) {
    if (s.type == GPL_LINESTRING) return make_line(s.xy, s.go[r], s.go[r + 1]);
    return make_line(s.xy, s.ro[k], s.ro[k + 1]);
}
__device__ __forceinline__ void side_part(const Side &s, int64_t r, int64_t q, int64_t &r0, int64_t &r1) {
    if (s.type == GPL_POLYGON) r0 = s.go[r], r1 = s.go[r + 1];
    else r0 = s.po[q], r1 = s.po[q + 1];
}
__device__ __forceinline__ Chain part_ring(const Side &s, int64_t ring) { return make_ring(s.xy, s.ro[ring], s.ro[ring + 1]); }

// impl Intersects<Coord> for Polygon: exterior != Outside && all holes != Inside
__device__ __forceinline__ bool polygon_intersects_coord(const Side &s, int64_t r0, int64_t r1, double2 p, int lane) {
    if (r1 <= r0) return false;
    if (ring_position(s.xy, s.ro[r0], s.ro[r0 + 1] - s.ro[r0], p, lane) == 0) return false;
    for (int64_t h = r0 + 1; h < r1; ++h)
        if (ring_position(s.xy, s.ro[h], s.ro[h + 1] - s.ro[h], p, lane) == 2) return false;
    return true;
}
// chain (>= 1 line) against one polygon part; `reject_box`: geo's has_disjoint_bboxes(chain, polygon)
__device__ __forceinline__ bool chain_intersects_polygon(const Chain &c, const Side &s, int64_t r0, int64_t r1, const Box &ext_box,
                                                         bool reject_box, int lane) {
    if (c.coords() < 2 || r1 <= r0) return false;  // no lines() / no exterior
    if (reject_box && boxes_disjoint(chain_box(c, lane), ext_box)) return false;
    for (int64_t rs = r0; rs < r1; ++rs) {
        const Chain ring = part_ring(s, rs);
        if (ls_intersects_ls(ring, ring.coords(), c, c.coords(), lane)) return true;
    }
    return polygon_intersects_coord(s, r0, r1, c[0], lane);
}
// impl Intersects<Polygon> for Polygon, self = S, polygon = O
__device__ __forceinline__ bool polygon_intersects_polygon(const Side &S, int64_t s0, int64_t s1, const Side &O, int64_t o0, int64_t o1,
                                                           int lane) {
    if (s1 <= s0 || o1 <= o0) return false;
    const Chain sext = part_ring(S, s0), oext = part_ring(O, o0);
    const Box sbox = chain_box(sext, lane), obox = chain_box(oext, lane);
    if (boxes_disjoint(sbox, obox)) return false;
    // self.intersects(polygon.exterior()) || polygon.interiors().any(|r| self.intersects(r))
    for (int64_t ro = o0; ro < o1; ++ro)
        if (chain_intersects_polygon(part_ring(O, ro), S, s0, s1, sbox, ro > o0, lane)) return true;
    // polygon.intersects(self.exterior()): its segment tests are a subset of the ones above
    return sext.coords() >= 2 && polygon_intersects_coord(O, o0, o1, sext[0], lane);
}

__device__ __forceinline__ bool row_intersects(Side a, int64_t ra, Side b, int64_t rb, int lane) {
    int ca = side_class(a.type), cb = side_class(b.type);
    if (ca == 2 && cb == 2) {
        int64_t pa0, pa1, pb0, pb1;
        side_range(a, ra, pa0, pa1);
        side_range(b, rb, pb0, pb1);
        const bool self_is_a = b.type == GPL_POLYGON;  // (Multi)Polygon x Polygon: parts of a are `self`; x MultiPolygon: parts of b
        for (int64_t p = pa0; p < pa1; ++p) {
            int64_t s0, s1;
            side_part(a, ra, p, s0, s1);
            for (int64_t q = pb0; q < pb1; ++q) {
                int64_t o0, o1;
                side_part(b, rb, q, o0, o1);
                if (self_is_a ? polygon_intersects_polygon(a, s0, s1, b, o0, o1, lane) : polygon_intersects_polygon(b, o0, o1, a, s0, s1, lane))
                    return true;
            }
        }
        return false;
    }
    if (ca > cb) {  // the remaining cases do not depend on which side is `self`
        Side t = a; a = b; b = t;
        int64_t tr = ra; ra = rb; rb = tr;
        int tc = ca; ca = cb; cb = tc;
    }
    int64_t a0, a1, b0, b1;
    side_range(a, ra, a0, a1);
    side_range(b, rb, b0, b1);
    if (ca == 0) {
        for (int64_t i = a0; i < a1; ++i) {
            const double2 p = a.xy[i];
            if (cb == 0) {  // Point x Point: equality
                bool hit = false;
                for (int64_t j = b0 + lane; j < b1; j += 32) {
                    const double2 q = b.xy[j];
                    hit = hit || (q.x == p.x && q.y == p.y);
                }
                if (__any_sync(0xffffffffu, hit)) return true;
            } else if (cb == 1) {  // lines().any(|l| l.intersects(coord))
                for (int64_t k = b0; k < b1; ++k) {
                    const Chain c = side_chain(b, rb, k);
                    bool hit = false;
                    for (int64_t j = lane; j + 1 < c.n; j += 32) hit = hit || line_intersects_coord(c.p[j], c.p[j + 1], p);
                    if (__any_sync(0xffffffffu, hit)) return true;
                }
            } else {
                for (int64_t q = b0; q < b1; ++q) {
                    int64_t r0, r1;
                    side_part(b, rb, q, r0, r1);
                    if (polygon_intersects_coord(b, r0, r1, p, lane)) return true;
                }
            }
        }
        return false;
    }
    // ca == 1
    for (int64_t k = a0; k < a1; ++k) {
        const Chain c = side_chain(a, ra, k);
        if (cb == 1) {
            for (int64_t m = b0; m < b1; ++m) {
                const Chain d = side_chain(b, rb, m);
                if (ls_intersects_ls(c, c.n, d, d.n, lane)) return true;
            }
        } else {
            for (int64_t q = b0; q < b1; ++q) {
                int64_t r0, r1;
                side_part(b, rb, q, r0, r1);
                if (r1 <= r0) continue;
                const Box ext = chain_box(part_ring(b, r0), lane);
                if (chain_intersects_polygon(c, b, r0, r1, ext, true, lane)) return true;
            }
        }
    }
    return false;
}

// distance for LineString x Polygon, Polygon x LineString, Polygon x Polygon rows (geo 0.27
// euclidean_distance.rs, recalled): 0 when the row intersects; a geometry lying strictly inside the other's
// exterior (hence in a hole) is measured against the interior rings, everything else exterior to exterior /
// linestring to exterior; each of those is the nearest-neighbour minimum over (vertex, segment) items.
// geo's rotating-calipers branch for two convex polygons computes the same minimum (different roundings).
__device__ __forceinline__ double chain_nn_dist2(const Chain &a, const Chain &b, int lane) {
    return ls_ls_min_dist2(a, a.coords(), b, b.coords(), lane);
}

// one row pair of k_distance_generic; ok = false: a first chain without a line (the reference panics -> null)
__device__ __forceinline__ double generic_distance(const Side &a, int64_t ra, const Side &b, int64_t rb, int lane, bool &ok) {
    const double big = 1.7976931348623157e308;
    // first chain of each side (the linestring, or the exterior ring) must have a line
    int64_t a0 = a.go[ra], a1 = a.go[ra + 1], b0 = b.go[rb], b1 = b.go[rb + 1];
    const bool pa = a.type == GPL_POLYGON, pb = b.type == GPL_POLYGON;
    const Chain ea = pa ? (a1 > a0 ? part_ring(a, a0) : Chain{a.xy, 0, false}) : make_line(a.xy, a0, a1);
    const Chain eb = pb ? (b1 > b0 ? part_ring(b, b0) : Chain{b.xy, 0, false}) : make_line(b.xy, b0, b1);
    if (ea.n < 2 || eb.n < 2) {
        ok = false;
        return nan("");
    }
    if (row_intersects(a, ra, b, rb, lane)) return 0.0;
    double m = big;
    bool done = false;
    if (pa && a1 - a0 > 1 && ring_position(a.xy, a.ro[a0], a.ro[a0 + 1] - a.ro[a0], eb.p[0], lane) == 2) {
        for (int64_t h = a0 + 1; h < a1; ++h) m = fmin(m, chain_nn_dist2(eb, part_ring(a, h), lane));
        done = true;
    } else if (pb && b1 - b0 > 1 && ring_position(b.xy, b.ro[b0], b.ro[b0 + 1] - b.ro[b0], ea.p[0], lane) == 2) {
        for (int64_t h = b0 + 1; h < b1; ++h) m = fmin(m, chain_nn_dist2(ea, part_ring(b, h), lane));
        done = true;
    }
    if (!done) m = chain_nn_dist2(ea, eb, lane);
    return sqrt(m);
}

// ---- Multi* operands of GeoSeries::distance ----------------------------------------------------------------------
// geo 0.27 euclidean_distance.rs (recalled), `impl_euclidean_distance_for_iter_geometry!`:
//     self.iter().map(|g| g.euclidean_distance(target)).fold(T::max_value(), |acc, v| acc.min(v))
// i.e. the minimum over the members (f64::MAX for an empty collection); min is exact, so the order is irrelevant.
// Members are addressed through VIEW sides of the single types: MultiPoint -> coordinate index, MultiLineString ->
// LINESTRING view whose go is the ring_off level, MultiPolygon -> POLYGON view whose go is the part_off level.
// A member pair on which geo would panic (nearest_neighbor on an empty tree) makes the row invalid.
// a, b: single-type views (POINT / LINESTRING / POLYGON), ia / ib: member indices
__device__ __forceinline__ double member_distance(const Side &a, int64_t ia, const Side &b, int64_t ib, int lane, bool &ok) {
    const int ca = side_class(a.type), cb = side_class(b.type);
    if (ca == 0 && cb == 0) return pt_dist(a.xy[ia], b.xy[ib]);
    if (ca == 0 && cb == 1) return point_ls_distance(b.xy, b.go[ib], b.go[ib + 1] - b.go[ib], a.xy[ia], lane);
    if (ca == 1 && cb == 0) return point_ls_distance(a.xy, a.go[ia], a.go[ia + 1] - a.go[ia], b.xy[ib], lane);
    if (ca == 0) return point_polygon_distance(b, ib, a.xy[ia], lane);
    if (cb == 0) return point_polygon_distance(a, ia, b.xy[ib], lane);
    const int64_t a0 = a.go[ia], a1 = a.go[ia + 1], b0 = b.go[ib], b1 = b.go[ib + 1];
    const bool pa = ca == 2, pb = cb == 2;
    const Chain ea = pa ? (a1 > a0 ? part_ring(a, a0) : Chain{a.xy, 0, false}) : make_line(a.xy, a0, a1);
    const Chain eb = pb ? (b1 > b0 ? part_ring(b, b0) : Chain{b.xy, 0, false}) : make_line(b.xy, b0, b1);
    if (!pa && !pb) {  // LineString x LineString: the intersection test comes first (geo), then the tree lookup that may panic
        if (ls_intersects_ls(ea, ea.n, eb, eb.n, lane)) return 0.0;
        if (ea.n < 2 || eb.n < 2) {
            ok = false;
            return 0.0;
        }
        return sqrt(chain_nn_dist2(ea, eb, lane));
    }
    if (ea.n < 2 || eb.n < 2) {  // the first chain of each side (the linestring, or the exterior ring) must have a line
        ok = false;
        return 0.0;
    }
    if (row_intersects(a, ia, b, ib, lane)) return 0.0;
    double m = 1.7976931348623157e308;
    if (pa && a1 - a0 > 1 && ring_position(a.xy, a.ro[a0], a.ro[a0 + 1] - a.ro[a0], eb.p[0], lane) == 2) {
        for (int64_t h = a0 + 1; h < a1; ++h) m = fmin(m, chain_nn_dist2(eb, part_ring(a, h), lane));
    } else if (pb && b1 - b0 > 1 && ring_position(b.xy, b.ro[b0], b.ro[b0 + 1] - b.ro[b0], ea.p[0], lane) == 2) {
        for (int64_t h = b0 + 1; h < b1; ++h) m = fmin(m, chain_nn_dist2(ea, part_ring(b, h), lane));
    } else {
        m = chain_nn_dist2(ea, eb, lane);
    }
    return sqrt(m);
}

// ---- host side ------------------------------------------------------------------------------------------------------
// POLYGON view of a Polygon or MultiPolygon array: `go` gives the rings of each polygon member (a MultiPolygon row's
// members are [geom_off[r], geom_off[r + 1]) of this view, a Polygon row is member r)
static Side polygon_view(const gpl_array *g) {
    const double2 *xy = reinterpret_cast<const double2 *>(g->xy);
    if (g->type == GPL_MULTIPOLYGON) return Side{GPL_POLYGON, xy, g->part_off, nullptr, g->ring_off};
    return Side{g->type, xy, g->geom_off, g->part_off, g->ring_off};
}

}  // namespace gpl
