// sym_point.cuh — symbolic points "just after / just beside" an edge start, and their exact position against a ring or a
// set of polygon members.  A SymQ is q = x + eps (v - x) + eps^2 side L(v - x) for infinitesimal eps (L: the left normal):
// every comparison of geo's coord_pos_relative_to_ring is made on x first and on the eps / eps^2 terms on a tie, so all
// results are exact signs.  Used by (Multi)Polygon contains Polygon (k_pairs.cu) and the validity checks (k_valid.cu).
#pragma once

#include "common.cuh"
#include "pair_dist.cuh"

namespace gpl {

struct SymQ {
    double xx, xy, vx, vy;
    int side;
};
// cmpd, sgnd: common.cuh
__device__ __forceinline__ int sym_cmp_y(const SymQ &q, double cy) {  // sign of cy - q.y
    int c = cmpd(cy, q.xy);
    if (c) return c;
    c = -cmpd(q.vy, q.xy);
    if (c) return c;
    return -q.side * cmpd(q.vx, q.xx);
}
__device__ __forceinline__ int sym_cmp_x(const SymQ &q, double cx) {  // sign of cx - q.x
    int c = cmpd(cx, q.xx);
    if (c) return c;
    c = -cmpd(q.vx, q.xx);
    if (c) return c;
    return q.side * cmpd(q.vy, q.xy);
}
__device__ __forceinline__ int sym_orient(double2 s, double2 e, const SymQ &q) {  // sign of orient2d(s, e, q)
    int o = sgnd(orient2d(s.x, s.y, e.x, e.y, q.xx, q.xy));
    if (o) return o;
    o = sgnd(orient2d(s.x, s.y, e.x, e.y, q.vx, q.vy));
    if (o || !q.side) return o;
    int d1, d2;  // s, e, x, v collinear: sign of side * dot(e - s, v - x)
    if (e.x != s.x) d1 = cmpd(e.x, s.x), d2 = cmpd(q.vx, q.xx);
    else d1 = cmpd(e.y, s.y), d2 = cmpd(q.vy, q.xy);
    return q.side * d1 * d2;
}
__device__ __forceinline__ bool sym_between_x(const SymQ &q, double b1, double b2) {
    if (b1 < b2) return sym_cmp_x(q, b1) <= 0 && sym_cmp_x(q, b2) >= 0;
    return sym_cmp_x(q, b2) <= 0 && sym_cmp_x(q, b1) >= 0;
}
// 0 outside / 1 boundary / 2 inside; lanes stride over the ring's segments
__device__ __forceinline__ int sym_ring_pos(const SymQ &q, const Chain &c, int lane) {
    if (c.n < 2) return 0;
    const int64_t m = c.coords();
    int wn = 0;
    bool boundary = false;
    for (int64_t i = lane; i + 1 < m; i += 32) {
        const double2 s = c[i], e = c[i + 1];
        const int cs = sym_cmp_y(q, s.y), ce = sym_cmp_y(q, e.y);
        if (cs <= 0) {
            if (ce >= 0) {
                const int o = sym_orient(s, e, q);
                if (o > 0 && ce != 0) wn += 1;
                else if (o == 0 && sym_between_x(q, s.x, e.x)) boundary = true;
            }
        } else if (ce <= 0) {
            const int o = sym_orient(s, e, q);
            if (o < 0) wn -= 1;
            else if (o == 0 && sym_between_x(q, s.x, e.x)) boundary = true;
        }
    }
    if (__any_sync(0xffffffffu, boundary)) return 1;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) wn += __shfl_xor_sync(0xffffffffu, wn, o);
    return wn ? 2 : 0;
}
// position of q in the union of the polygon members [m0, m1) of the POLYGON view `a`
__device__ __forceinline__ int sym_region_pos(const Side &a, int64_t m0, int64_t m1, const SymQ &q, int lane) {
    bool boundary = false;
    for (int64_t m = m0; m < m1; ++m) {
        const int64_t r0 = a.go[m], r1 = a.go[m + 1];
        if (r1 <= r0) continue;
        const int pe = sym_ring_pos(q, part_ring(a, r0), lane);
        if (pe == 0) continue;
        if (pe == 1) {
            boundary = true;
            continue;
        }
        bool in_hole = false;
        for (int64_t r = r0 + 1; r < r1 && !in_hole; ++r) {
            const int ph = sym_ring_pos(q, part_ring(a, r), lane);
            if (ph == 2) in_hole = true;
            else if (ph == 1) in_hole = boundary = true;
        }
        if (!in_hole) return 2;
    }
    return boundary ? 1 : 0;
}

}  // namespace gpl
