// k_pairs.cu — row-wise binary ops: distance, intersects, contains (1:1 aligned rows).
// Reference: GeoSeries::distance geoseries.rs:141-146 (impl :248-251 names the historical callee
// ops::distance::euclidean_distance); intersects / contains semantics from the dead join code
// geopolars/src/spatial_index.rs:89-137.  Arithmetic = geo 0.27 euclidean_distance.rs,
// intersects/{line,line_string}.rs, coordinate_position.rs and geo-types private_utils.rs (recalled;
// restated in oracle/geo_oracle.c).
//
// Design: one warp per row.  Both linestrings of the row are staged into shared memory with one
// coalesced LDG.128 per lane (BASELINE config 3: 16+16 coords = 512 B per row, one warp-wide load), then
//   intersects: per-segment bounding boxes once; lanes stride over the (na-1)*(nb-1) segment pairs doing only
//               the closed-bbox reject (exact), survivors are compacted with __ballot_sync into a small
//               shared-memory queue and tested 32 at a time by a BRANCH-FREE rule: four orientation
//               determinants with Shewchuk's stage-A filter; four certified non-zero signs decide the pair
//               exactly like geo's Line x Line rule, anything else (collinear, degenerate, within rounding)
//               marks the row and — only if no certified hit exists — the whole row is redone with the
//               exact adaptive predicate (warp-uniform call, rare).  Early exit with __any_sync.
//   distance  : only if not intersecting; lanes stride over the nb*(na-1) + na*(nb-1) (vertex, segment)
//               items, branch-free: the three candidate squared distances are formed and the minimum is
//               tracked as a FRACTION (numerator, denominator) compared by cross-multiplication, one
//               division + one sqrt per row.  The cancellation-prone term (the cross product) uses
//               exactly the reference's expression, so the result differs from geo's |s|*hypot(dx,dy) only
//               by the last roundings (<= 4 ulp; the stated tolerance for f64 outputs is 1e-9 relative).
// Rows longer than 33 coordinates per side use the straightforward generic path below.
// These kernels are FP64-ALU bound, not HBM bound (~225 segment tests + ~480 distance items per 512 B).
#include <math.h>

#include <cmath>
#include <string.h>

#include "common.cuh"
#include "join_grid.cuh"
#include "join_host.cuh"
#include "output.cuh"
#include "pair_dist.cuh"
#include "point_dist.cuh"
#include "scan.cuh"
#include "sym_point.cuh"

namespace gpl {

constexpr int kPairWarps = 8;     // warps per CTA
constexpr int kPairSmemCoords = 128;  // coords of (A,B) staged per warp; longer rows read global memory

// Coords, seg_dist2, ls_intersects_ls, ls_ls_min_dist2, ls_intersects_ls_short, ls_ls_distance_short: pair_dist.cuh

// stage a row's coordinates in shared memory when they fit, else hand back the global pointer
__device__ __forceinline__ Coords stage(const double2 *__restrict__ g, int64_t c0, int64_t n, double2 *smem, bool fits, int lane) {
    if (!fits) return Coords{g + c0};
    for (int64_t i = lane; i < n; i += 32) smem[i] = __ldcs(g + c0 + i);
    return Coords{smem};
}

// MODE 0: intersects -> byte per row   MODE 1: distance -> f64 (+ validity byte)
//
// Fast kernel: rows with <= 33 coordinates per side.  No calls, no adaptive-precision code (64-ish
// registers instead of 108); the next row's coordinates are prefetched into registers while the current
// row is processed.  Rows it cannot finish — longer linestrings, or a filter that could not certify a
// sign that mattered — get flag[r] = 1 and are redone by k_ls_ls_exact.
template <int MODE>
__global__ void __launch_bounds__(kPairWarps * 32, 3) k_ls_ls_fast(int64_t n, const double2 *__restrict__ axy,
                                                                   const int64_t *__restrict__ aoff, const uint8_t *__restrict__ avalid,
                                                                   const double2 *__restrict__ bxy, const int64_t *__restrict__ boff,
                                                                   const uint8_t *__restrict__ bvalid, uint8_t *__restrict__ out_bool,
                                                                   double *__restrict__ out_dist, uint8_t *__restrict__ out_valid,
                                                                   uint8_t *__restrict__ flag) {
    __shared__ double2 smem[kPairWarps][68];
    __shared__ float4 s_box[kPairWarps][64];
    __shared__ unsigned short s_queue[kPairWarps][kPairQueue];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    double2 *sm = smem[wid];
    const int64_t nwarps = (int64_t)gridDim.x * kPairWarps;
    int64_t r = (int64_t)blockIdx.x * kPairWarps + wid;
    // prefetch registers: lane holds coords lane, lane+32, lane+64 of the concatenation A ++ B of the next row
    double2 pf[3];
    int64_t a0 = 0, b0 = 0;
    int32_t na = 0, nb = 0;
    bool shortp = false;
    auto fetch = [&](int64_t row) {
        a0 = aoff[row], b0 = boff[row];
        const int64_t la = aoff[row + 1] - a0, lb = boff[row + 1] - b0;
        shortp = la <= 33 && lb <= 33;
        na = (int32_t)min(la, (int64_t)34), nb = (int32_t)min(lb, (int64_t)34);
        if (shortp) {
#pragma unroll
            for (int k = 0; k < 3; ++k) {
                const int32_t c = lane + 32 * k;
                if (c < na) pf[k] = __ldcs(axy + a0 + c);
                else if (c < na + nb) pf[k] = __ldcs(bxy + b0 + (c - na));
            }
        }
    };
    if (r < n) fetch(r);
    for (; r < n; r += nwarps) {
        const bool valid = bit_get(avalid, r) && bit_get(bvalid, r);
        const bool cur_short = shortp;
        const int32_t cna = na, cnb = nb;
        __syncwarp();
        if (cur_short) {
#pragma unroll
            for (int k = 0; k < 3; ++k) {
                const int32_t c = lane + 32 * k;
                if (c < cna + cnb) sm[c] = pf[k];
            }
        }
        if (r + nwarps < n) fetch(r + nwarps);  // overlaps the HBM latency of the next row with this row's math
        __syncwarp();
        int isect = 0;
        if (valid && cur_short) isect = ls_intersects_ls_short(sm, cna, sm + cna, cnb, s_box[wid], s_queue[wid], lane);
        const bool defer = valid && (!cur_short || isect == 2);
        if (lane == 0) flag[r] = defer ? 1 : 0;
        if (defer) continue;
        if (MODE == 0) {
            if (lane == 0) out_bool[r] = isect == 1 ? 1 : 0;
        } else {
            double d = 0.0;
            bool ok = valid;
            if (valid && isect == 0) {
                if (cna < 2 || cnb < 2) ok = false;  // reference: nearest_neighbor(..).unwrap() on an empty r-tree panics -> null
                else d = ls_ls_distance_short(sm, cna, sm + cna, cnb, lane);
            }
            if (lane == 0) {
                out_dist[r] = ok ? d : nan("");
                if (out_valid) out_valid[r] = ok ? 1 : 0;
            }
        }
    }
}

// Exact/generic kernel: redoes the rows k_ls_ls_fast flagged (any length, adaptive exact predicate).
// Each warp scans 32 flags at a time and processes the flagged rows one after the other.
template <int MODE>
__global__ void __launch_bounds__(kPairWarps * 32) k_ls_ls_exact(int64_t n, const double2 *__restrict__ axy,
                                                                 const int64_t *__restrict__ aoff, const double2 *__restrict__ bxy,
                                                                 const int64_t *__restrict__ boff, const uint8_t *__restrict__ flag,
                                                                 uint8_t *__restrict__ out_bool, double *__restrict__ out_dist,
                                                                 uint8_t *__restrict__ out_valid) {
    __shared__ double2 smem[kPairWarps][kPairSmemCoords];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const int64_t nwarps = (int64_t)gridDim.x * kPairWarps;
    const int64_t n_blocks = (n + 31) >> 5;
    for (int64_t blk = (int64_t)blockIdx.x * kPairWarps + wid; blk < n_blocks; blk += nwarps) {
        const int64_t row0 = blk << 5;
        unsigned todo = __ballot_sync(0xffffffffu, row0 + lane < n && flag[row0 + lane] != 0);
        while (todo) {
            const int bit = __ffs(todo) - 1;
            todo &= todo - 1;
            const int64_t r = row0 + bit;
            const int64_t a0 = aoff[r], na = aoff[r + 1] - a0, b0 = boff[r], nb = boff[r + 1] - b0;
            const bool fits = na + nb <= kPairSmemCoords;
            __syncwarp();
            Coords A = stage(axy, a0, na, smem[wid], fits, lane);
            Coords B = stage(bxy, b0, nb, smem[wid] + (fits ? na : 0), fits, lane);
            __syncwarp();
            const bool isect = ls_intersects_ls(A, na, B, nb, lane);
            if (MODE == 0) {
                if (lane == 0) out_bool[r] = isect ? 1 : 0;
            } else {
                double d = 0.0;
                bool ok = true;
                if (!isect) {
                    if (na < 2 || nb < 2) ok = false;
                    else d = sqrt(ls_ls_min_dist2(A, na, B, nb, lane));
                }
                if (lane == 0) {
                    out_dist[r] = ok ? d : nan("");
                    if (out_valid) out_valid[r] = ok ? 1 : 0;
                }
            }
        }
    }
}

// ---- point vs linestring / polygon -------------------------------------------------------------
// pt_dist / line_segment_distance: common.cuh; line_string_contains_point, point_ls_distance, ring_position,
// polygon_position, Side, point_polygon_distance: point_dist.cuh

// Chain, Box, the Side helpers, row_intersects: pair_dist.cuh

__global__ void __launch_bounds__(256) k_intersects_generic(int64_t n, Side a, const uint8_t *__restrict__ av, Side b,
                                                            const uint8_t *__restrict__ bv, uint8_t *__restrict__ out) {
    const int lane = threadIdx.x & 31;
    int64_t warp = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
    const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t r = warp; r < n; r += nwarps) {
        bool res = false;
        if (bit_get(av, r) && bit_get(bv, r)) res = row_intersects(a, r, b, r, lane);
        if (lane == 0) out[r] = res ? 1 : 0;
    }
}

// chain_nn_dist2, generic_distance: pair_dist.cuh
__global__ void __launch_bounds__(256) k_distance_generic(int64_t n, Side a, const uint8_t *__restrict__ av, Side b,
                                                          const uint8_t *__restrict__ bv, double *__restrict__ out,
                                                          uint8_t *__restrict__ out_valid) {
    const int lane = threadIdx.x & 31;
    int64_t warp = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
    const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t r = warp; r < n; r += nwarps) {
        bool ok = bit_get(av, r) && bit_get(bv, r);
        double d = nan("");
        if (ok) d = generic_distance(a, r, b, r, lane, ok);
        if (lane == 0) {
            out[r] = ok ? d : nan("");
            if (out_valid) out_valid[r] = ok ? 1 : 0;
        }
    }
}

// ---- Multi* operands of GeoSeries::distance: member_distance is in pair_dist.cuh ---------------------------------------
// one warp per row; am / bm: the geom_off level of a Multi* operand (members [am[r], am[r+1])), NULL for a single type
__global__ void __launch_bounds__(256) k_distance_multi(int64_t n, Side a, const int64_t *__restrict__ am, const uint8_t *__restrict__ av,
                                                        Side b, const int64_t *__restrict__ bm, const uint8_t *__restrict__ bv,
                                                        double *__restrict__ out, uint8_t *__restrict__ out_valid) {
    const int lane = threadIdx.x & 31;
    int64_t warp = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
    const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t r = warp; r < n; r += nwarps) {
        bool ok = bit_get(av, r) && bit_get(bv, r);
        double d = 1.7976931348623157e308;
        if (ok) {
            const int64_t a0 = am ? am[r] : r, a1 = am ? am[r + 1] : r + 1, b0 = bm ? bm[r] : r, b1 = bm ? bm[r + 1] : r + 1;
            for (int64_t p = a0; p < a1; ++p)
                for (int64_t q = b0; q < b1; ++q) d = fmin(d, member_distance(a, p, b, q, lane, ok));
        }
        if (lane == 0) {
            out[r] = ok ? d : nan("");
            if (out_valid) out_valid[r] = ok ? 1 : 0;
        }
    }
}

// ---- (Multi)Polygon contains Polygon (spatial_index.rs:99-110: `poly_lhs.contains(poly_rhs)`) -------------------------
// geo 0.27 contains/polygon.rs (recalled): `impl_contains_from_relate!`, i.e. self.relate(rhs).is_contains() = DE-9IM
// [T*****FF*].  For VALID operands: B inside closure(A) and the interiors meet, decided with exact orientation signs only
// (the derivation is in oracle/geo_oracle.c, "Polygon / MultiPolygon contains Polygon"):
//   C1 no edge of B leaves closure(A): just after its start and just after every A vertex lying on it the edge is not in
//      the exterior of A, and it crosses no A edge properly (unless an A vertex sits on the crossing);
//   C2 no edge of A enters the interior of B (same events, roles swapped);
//   C3 a point just beside B's first edge, on B's interior side, is inside A.
// "Just after / beside" are symbolic points q = x + eps (v - x) + eps^2 side L(v - x): every comparison of geo's
// coord_pos_relative_to_ring is made on x first and on the eps / eps^2 terms on a tie — all exact signs.
// SymQ, sym_ring_pos, sym_region_pos: sym_point.cuh
__device__ __forceinline__ bool strictly_between(double2 c, double2 u, double2 v) {
    if (u.x != v.x) return c.x > fmin(u.x, v.x) && c.x < fmax(u.x, v.x);
    return c.y > fmin(u.y, v.y) && c.y < fmax(u.y, v.y);
}
// is some vertex of the members [m0, m1) of `a` on both lines u-v and s-e (exactly at their crossing)?
__device__ __forceinline__ bool vertex_at_crossing(const Side &a, int64_t m0, int64_t m1, double2 u, double2 v, double2 s, double2 e, int lane) {
    bool hit = false;
    for (int64_t c = a.ro[a.go[m0]] + lane; c < a.ro[a.go[m1]]; c += 32) {
        const double2 w = a.xy[c];
        hit = hit || (orient2d(u.x, u.y, v.x, v.y, w.x, w.y) == 0.0 && orient2d(s.x, s.y, e.x, e.y, w.x, w.y) == 0.0);
    }
    return __any_sync(0xffffffffu, hit);
}
// the edges of X = members [x0,x1) of view x must not reach into `forbidden` (0 exterior / 2 interior) of Y = members
// [y0,y1) of view y; check_cross: a proper crossing fails (C1).  Warp-uniform control flow.
__device__ __forceinline__ bool edges_avoid(const Side &x, int64_t x0, int64_t x1, const Side &y, int64_t y0, int64_t y1, int forbidden,
                                            bool check_cross, int lane) {
    for (int64_t rx = x.go[x0]; rx < x.go[x1]; ++rx) {
        const Chain cx = part_ring(x, rx);
        const int64_t nx = cx.coords();
        for (int64_t i = 0; i + 1 < nx; ++i) {
            const double2 u = cx[i], v = cx[i + 1];
            if (u.x == v.x && u.y == v.y) continue;
            const SymQ q{u.x, u.y, v.x, v.y, 0};
            if (sym_region_pos(y, y0, y1, q, lane) == forbidden) return false;
            for (int64_t ry = y.go[y0]; ry < y.go[y1]; ++ry) {
                const Chain cy = part_ring(y, ry);
                const int64_t ny = cy.coords();
                for (int64_t j0 = 0; j0 + 1 < ny; j0 += 32) {
                    const int64_t j = j0 + lane;
                    bool cross = false, touch = false;
                    double2 s = make_double2(0.0, 0.0), e = s;
                    if (j + 1 < ny) {
                        s = cy[j], e = cy[j + 1];
                        const int o1 = sgnd(orient2d(u.x, u.y, v.x, v.y, s.x, s.y));
                        if (check_cross && !(s.x == e.x && s.y == e.y)) {
                            const int o2 = sgnd(orient2d(u.x, u.y, v.x, v.y, e.x, e.y));
                            if (o1 * o2 < 0) {
                                const int o3 = sgnd(orient2d(s.x, s.y, e.x, e.y, u.x, u.y)), o4 = sgnd(orient2d(s.x, s.y, e.x, e.y, v.x, v.y));
                                cross = o3 * o4 < 0;
                            }
                        }
                        touch = o1 == 0 && strictly_between(s, u, v);
                    }
                    unsigned mc = __ballot_sync(0xffffffffu, cross);
                    while (mc) {  // an A vertex exactly on the crossing (members touching there) leaves the verdict to `touch`
                        const int src = __ffs(mc) - 1;
                        mc &= mc - 1;
                        if (!vertex_at_crossing(y, y0, y1, u, v, bcast2(s, src), bcast2(e, src), lane)) return false;
                    }
                    unsigned mt = __ballot_sync(0xffffffffu, touch);
                    while (mt) {  // a vertex of Y inside this edge: the part of the edge after it
                        const int src = __ffs(mt) - 1;
                        mt &= mt - 1;
                        const double2 w = bcast2(s, src);
                        const SymQ q2{w.x, w.y, v.x, v.y, 0};
                        if (sym_region_pos(y, y0, y1, q2, lane) == forbidden) return false;
                    }
                }
            }
        }
    }
    return true;
}
// A = members [a0,a1) of the POLYGON view `a`; B = polygon b of the POLYGON view `bv`
__device__ __forceinline__ bool region_contains_polygon(const Side &a, int64_t a0, int64_t a1, const Side &bv, int64_t b, int lane) {
    const int64_t br0 = bv.go[b], br1 = bv.go[b + 1];
    if (a1 <= a0 || br1 <= br0 || bv.ro[br0 + 1] - bv.ro[br0] < 3) return false;
    if (!edges_avoid(bv, b, b + 1, a, a0, a1, 0, true, lane)) return false;   // C1
    if (!edges_avoid(a, a0, a1, bv, b, b + 1, 2, false, lane)) return false;  // C2
    const Chain ce = part_ring(bv, br0);
    const int64_t n = ce.coords();
    for (int64_t i = 0; i + 1 < n; ++i) {  // C3: the first non-degenerate edge of B's exterior ring
        const double2 u = ce[i], v = ce[i + 1];
        if (u.x == v.x && u.y == v.y) continue;
        SymQ q{u.x, u.y, v.x, v.y, 1};
        if (sym_region_pos(bv, b, b + 1, q, lane) != 2) {
            q.side = -1;
            if (sym_region_pos(bv, b, b + 1, q, lane) != 2) return false;  // no interior beside its own boundary: degenerate
        }
        return sym_region_pos(a, a0, a1, q, lane) == 2;
    }
    return false;
}
// One warp per row (or per candidate pair of a join: ia / ib select the rows).  a: POLYGON view of the (Multi)Polygon
// side, am its member offsets (NULL: one member per row); b: POLYGON.
__global__ void __launch_bounds__(256) k_contains_polygon(int64_t n, Side a, const int64_t *__restrict__ am, const uint8_t *__restrict__ av,
                                                          Side b, const uint8_t *__restrict__ bv, const uint64_t *__restrict__ ia,
                                                          const uint64_t *__restrict__ ib, uint8_t *__restrict__ out) {
    const int lane = threadIdx.x & 31;
    int64_t warp = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
    const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t r = warp; r < n; r += nwarps) {
        const int64_t ra = ia ? (int64_t)ia[r] : r, rb = ib ? (int64_t)ib[r] : r;
        bool res = false;
        if (bit_get(av, ra) && bit_get(bv, rb)) {
            const int64_t m0 = am ? am[ra] : ra, m1 = am ? am[ra + 1] : ra + 1;
            res = region_contains_polygon(a, m0, m1, b, rb, lane);
        }
        if (lane == 0) out[r] = res ? 1 : 0;
    }
}
// row_intersects over candidate pairs of a join
__global__ void __launch_bounds__(256) k_intersects_pairs(int64_t n, Side a, const uint8_t *__restrict__ av, Side b,
                                                          const uint8_t *__restrict__ bv, const uint64_t *__restrict__ ia,
                                                          const uint64_t *__restrict__ ib, uint8_t *__restrict__ out) {
    const int lane = threadIdx.x & 31;
    int64_t warp = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
    const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t r = warp; r < n; r += nwarps) {
        const int64_t ra = (int64_t)ia[r], rb = (int64_t)ib[r];
        bool res = false;
        if (bit_get(av, ra) && bit_get(bv, rb)) res = row_intersects(a, ra, b, rb, lane);
        if (lane == 0) out[r] = res ? 1 : 0;
    }
}

// impl Contains<Coord> for LineString (interior only: an end point counts only on a closed linestring);
// MultiLineString: any member.  geo 0.27 contains/line_string.rs, contains/line.rs (recalled).
__device__ __forceinline__ bool lines_contain_point(const Side &a, int64_t r, double2 p, int lane) {
    bool res = false;
    int64_t k0, k1;
    side_range(a, r, k0, k1);
    for (int64_t k = k0; k < k1 && !res; ++k) {
        const Chain c = side_chain(a, r, k);
        if (c.n == 0) continue;
        const double2 f = c.p[0], l = c.p[c.n - 1];
        if ((p.x == f.x && p.y == f.y) || (p.x == l.x && p.y == l.y)) {
            res = (f.x == l.x && f.y == l.y);  // is_closed()
            continue;
        }
        bool hit = false;
        for (int64_t i = lane; i + 1 < c.n; i += 32) {
            const double2 s = c.p[i], e = c.p[i + 1];
            const bool ps = (p.x == s.x && p.y == s.y), pe = (p.x == e.x && p.y == e.y);
            const bool in_line = (s.x == e.x && s.y == e.y) ? ps : (!ps && !pe && line_intersects_coord(s, e, p));
            hit = hit || in_line || (i > 0 && ps);
        }
        res = __any_sync(0xffffffffu, hit);
    }
    return res;
}
// (Multi)Polygon::contains(coord): strictly inside some part (geo coordinate_position == Inside)
__device__ __forceinline__ bool area_contains_point(const Side &a, int64_t r, double2 p, int lane) {
    int64_t q0, q1;
    side_range(a, r, q0, q1);
    for (int64_t q = q0; q < q1; ++q) {
        int64_t r0, r1;
        side_part(a, r, q, r0, r1);
        bool inside = false;
        int bc = 0;
        polygon_position(a.xy, a.ro, r0, r1, p, lane, inside, bc);
        if ((bc % 2 == 0) && inside) return true;
    }
    return false;
}
__global__ void __launch_bounds__(256) k_lines_contain_point(int64_t n, Side a, const uint8_t *__restrict__ av,
                                                             const double2 *__restrict__ pts, const uint8_t *__restrict__ pv,
                                                             uint8_t *__restrict__ out) {
    const int lane = threadIdx.x & 31;
    int64_t warp = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
    const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t r = warp; r < n; r += nwarps) {
        bool res = false;
        if (bit_get(av, r) && bit_get(pv, r)) res = lines_contain_point(a, r, pts[r], lane);
        if (lane == 0) out[r] = res ? 1 : 0;
    }
}
// candidate pairs of a join: row ia[k] of the (Multi)Polygon / (Multi)LineString side contains point row ib[k]
__global__ void __launch_bounds__(256) k_contains_point_pairs(int64_t n, Side a, const uint8_t *__restrict__ av,
                                                              const double2 *__restrict__ pts, const uint8_t *__restrict__ pv,
                                                              const uint64_t *__restrict__ ia, const uint64_t *__restrict__ ib,
                                                              uint8_t *__restrict__ out) {
    const int lane = threadIdx.x & 31;
    int64_t warp = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
    const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    const bool lines = side_class(a.type) == 1;
    for (int64_t k = warp; k < n; k += nwarps) {
        const int64_t ra = (int64_t)ia[k], rb = (int64_t)ib[k];
        bool res = false;
        if (bit_get(av, ra) && bit_get(pv, rb)) {
            const double2 p = pts[rb];
            res = lines ? lines_contain_point(a, ra, p, lane) : area_contains_point(a, ra, p, lane);
        }
        if (lane == 0) out[k] = res ? 1 : 0;
    }
}

// poly rows vs point rows.  MODE 0: contains byte   MODE 1: distance
template <int MODE>
__global__ void __launch_bounds__(256) k_poly_point(int ptype, int64_t n, const double2 *__restrict__ pxy,
                                                    const int64_t *__restrict__ geom_off, const int64_t *__restrict__ part_off,
                                                    const int64_t *__restrict__ ring_off, const uint8_t *__restrict__ pvalid,
                                                    const double2 *__restrict__ pts, const uint8_t *__restrict__ tvalid,
                                                    uint8_t *__restrict__ out_bool, double *__restrict__ out_dist,
                                                    uint8_t *__restrict__ out_valid) {
    const int lane = threadIdx.x & 31;
    int64_t warp = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
    const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t r = warp; r < n; r += nwarps) {
        bool valid = bit_get(pvalid, r) && bit_get(tvalid, r);
        double2 p = pts[r];
        if (MODE == 0) {
            bool res = false;
            if (valid) {
                if (ptype == GPL_POLYGON) {
                    bool inside = false;
                    int bc = 0;
                    polygon_position(pxy, ring_off, geom_off[r], geom_off[r + 1], p, lane, inside, bc);
                    res = (bc % 2 == 0) && inside;
                } else {
                    for (int64_t q = geom_off[r]; q < geom_off[r + 1] && !res; ++q) {
                        bool inside = false;
                        int bc = 0;
                        polygon_position(pxy, ring_off, part_off[q], part_off[q + 1], p, lane, inside, bc);
                        res = (bc % 2 == 0) && inside;
                    }
                }
            }
            if (lane == 0) out_bool[r] = res ? 1 : 0;
        } else {  // Point-Polygon distance (POLYGON rows only)
            double d = nan("");
            if (valid) {
                int64_t r0 = geom_off[r], r1 = geom_off[r + 1];
                if (r1 <= r0 || ring_off[r0 + 1] - ring_off[r0] == 0) {
                    d = 0.0;
                } else {
                    bool inside = false;
                    int bc = 0;
                    polygon_position(pxy, ring_off, r0, r1, p, lane, inside, bc);
                    if (bc % 2 == 1 || inside) {
                        d = 0.0;
                    } else {
                        double acc = 1.7976931348623157e308;
                        for (int64_t h = r0 + 1; h < r1; ++h)
                            acc = fmin(acc, point_ls_distance(pxy, ring_off[h], ring_off[h + 1] - ring_off[h], p, lane));
                        double ext = 1.7976931348623157e308;
                        int64_t c0 = ring_off[r0], nn = ring_off[r0 + 1] - c0;
                        for (int64_t i = lane; i < nn - 1; i += 32) ext = fmin(ext, line_segment_distance(p, pxy[c0 + i], pxy[c0 + i + 1]));
                        d = fmin(acc, warp_min(ext));
                    }
                }
            }
            if (lane == 0) {
                out_dist[r] = d;
                if (out_valid) out_valid[r] = valid ? 1 : 0;
            }
        }
    }
}

__global__ void __launch_bounds__(256) k_point_ls_dist(int64_t n, const double2 *__restrict__ pts, const uint8_t *__restrict__ tvalid,
                                                       const double2 *__restrict__ lxy, const int64_t *__restrict__ loff,
                                                       const uint8_t *__restrict__ lvalid, double *__restrict__ out,
                                                       uint8_t *__restrict__ out_valid) {
    const int lane = threadIdx.x & 31;
    int64_t warp = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
    const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t r = warp; r < n; r += nwarps) {
        bool valid = bit_get(tvalid, r) && bit_get(lvalid, r);
        double d = nan("");
        if (valid) d = point_ls_distance(lxy, loff[r], loff[r + 1] - loff[r], pts[r], lane);
        if (lane == 0) {
            out[r] = d;
            if (out_valid) out_valid[r] = valid ? 1 : 0;
        }
    }
}
__global__ void k_point_point_dist(int64_t n, const double2 *__restrict__ a, const uint8_t *__restrict__ av,
                                   const double2 *__restrict__ b, const uint8_t *__restrict__ bv, double *__restrict__ out,
                                   uint8_t *__restrict__ out_valid) {
    int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= n) return;
    bool valid = bit_get(av, i) && bit_get(bv, i);
    out[i] = valid ? pt_dist(a[i], b[i]) : nan("");
    if (out_valid) out_valid[i] = valid ? 1 : 0;
}

static int side_class_host(int t) { return (t == GPL_POINT || t == GPL_MULTIPOINT) ? 0 : (t == GPL_LINESTRING || t == GPL_MULTILINESTRING) ? 1 : 2; }

// polygon_view: pair_dist.cuh

}  // namespace gpl

using namespace gpl;

extern "C" int gpl_intersects(gpl_ctx *ctx, const gpl_array *a, const gpl_array *b, uint8_t *out_bitmap, int mem) {
    GPL_REQUIRE(ctx && a && b && out_bitmap, GPL_ERR_INVALID_ARG, "gpl_intersects: NULL argument");
    GPL_TRY(check_mem(mem, "gpl_intersects"));
    GPL_TRY(require_same_length(a, b, "intersects"));
    GPL_REQUIRE(known_type(a->type) && known_type(b->type), GPL_ERR_INVALID_TYPE, "intersects: unsupported geometry pair %s x %s", type_name(a->type), type_name(b->type));
    GPL_CUDA(cudaSetDevice(ctx->device));
    int64_t n = a->n_geoms;
    if (n == 0) return GPL_OK;
    Scratch<uint8_t> bytes, flag;
    GPL_TRY(bytes.get(ctx, (size_t)n));
    const double2 *axy = reinterpret_cast<const double2 *>(a->xy), *bxy = reinterpret_cast<const double2 *>(b->xy);
    if (!(a->type == GPL_LINESTRING && b->type == GPL_LINESTRING)) {  // every other pair: one warp per row, exact predicates
        Side sa{a->type, axy, a->geom_off, a->part_off, a->ring_off}, sb{b->type, bxy, b->geom_off, b->part_off, b->ring_off};
        GPL_LAUNCH(ctx, k_intersects_generic, warp_grid(n, 8), 256, 0, n, sa, a->validity, sb, b->validity, bytes.p);
        return finish_bitmap(ctx, bytes.p, n, out_bitmap, mem);
    }
    GPL_TRY(flag.get(ctx, (size_t)n));
    GPL_LAUNCH(ctx, k_ls_ls_fast<0>, warp_grid(n, kPairWarps), kPairWarps * 32, 0, n, axy, a->geom_off, a->validity, bxy, b->geom_off,
               b->validity, bytes.p, nullptr, nullptr, flag.p);
    GPL_LAUNCH(ctx, k_ls_ls_exact<0>, warp_grid(ceil_div(n, 32), kPairWarps), kPairWarps * 32, 0, n, axy, a->geom_off, bxy, b->geom_off,
               flag.p, bytes.p, nullptr, nullptr);
    return finish_bitmap(ctx, bytes.p, n, out_bitmap, mem);
}

extern "C" int gpl_contains(gpl_ctx *ctx, const gpl_array *polygons, const gpl_array *points, uint8_t *out_bitmap, int mem) {
    GPL_REQUIRE(ctx && polygons && points && out_bitmap, GPL_ERR_INVALID_ARG, "gpl_contains: NULL argument");
    GPL_TRY(check_mem(mem, "gpl_contains"));
    GPL_TRY(require_same_length(polygons, points, "contains"));
    const bool lines = is_line(polygons->type);
    GPL_REQUIRE((is_area(polygons->type) || lines) && points->type == GPL_POINT, GPL_ERR_INVALID_TYPE,
                "Expected (Multi)Polygon or (Multi)LineString x Point (found %s x %s)", type_name(polygons->type),
                type_name(points->type));
    GPL_CUDA(cudaSetDevice(ctx->device));
    int64_t n = polygons->n_geoms;
    if (n == 0) return GPL_OK;
    Scratch<uint8_t> bytes;
    GPL_TRY(bytes.get(ctx, (size_t)n));
    if (lines) {
        Side sl{polygons->type, reinterpret_cast<const double2 *>(polygons->xy), polygons->geom_off, polygons->part_off, polygons->ring_off};
        GPL_LAUNCH(ctx, k_lines_contain_point, warp_grid(n, 8), 256, 0, n, sl, polygons->validity,
                   reinterpret_cast<const double2 *>(points->xy), points->validity, bytes.p);
        return finish_bitmap(ctx, bytes.p, n, out_bitmap, mem);
    }
    GPL_LAUNCH(ctx, k_poly_point<0>, warp_grid(n, 8), 256, 0, polygons->type, n, reinterpret_cast<const double2 *>(polygons->xy),
               polygons->geom_off, polygons->part_off, polygons->ring_off, polygons->validity,
               reinterpret_cast<const double2 *>(points->xy), points->validity, bytes.p, nullptr, nullptr);
    return finish_bitmap(ctx, bytes.p, n, out_bitmap, mem);
}

extern "C" int gpl_distance(gpl_ctx *ctx, const gpl_array *a, const gpl_array *b, double *out, uint8_t *out_validity, int mem) {
    GPL_REQUIRE(ctx && a && b && out, GPL_ERR_INVALID_ARG, "gpl_distance: NULL argument");
    GPL_TRY(check_mem(mem, "gpl_distance"));
    GPL_TRY(require_same_length(a, b, "distance"));
    const int ta = a->type, tb = b->type;
    GPL_REQUIRE(known_type(ta) && known_type(tb), GPL_ERR_INVALID_TYPE, "distance: unsupported geometry pair %s x %s", type_name(ta), type_name(tb));
    GPL_CUDA(cudaSetDevice(ctx->device));
    int64_t n = a->n_geoms;
    if (n == 0) return GPL_OK;
    RowOut<double> res;
    ValidOut valid;
    GPL_TRY(res.get(ctx, out, n, mem));
    GPL_TRY(valid.get(ctx, out_validity, n, mem, false));
    const double2 *axy = reinterpret_cast<const double2 *>(a->xy), *bxy = reinterpret_cast<const double2 *>(b->xy);
    if (is_multi(ta) || is_multi(tb)) {  // minimum over the members (geo's impl for iterable geometries)
        auto view = [](const gpl_array *g, const double2 *xy) {
            switch (g->type) {
            case GPL_MULTIPOINT: return Side{GPL_POINT, xy, nullptr, nullptr, nullptr};
            case GPL_MULTILINESTRING: return Side{GPL_LINESTRING, xy, g->ring_off, nullptr, nullptr};
            case GPL_MULTIPOLYGON: return Side{GPL_POLYGON, xy, g->part_off, nullptr, g->ring_off};
            default: return Side{g->type, xy, g->geom_off, g->part_off, g->ring_off};
            }
        };
        GPL_LAUNCH(ctx, k_distance_multi, warp_grid(n, 8), 256, 0, n, view(a, axy), is_multi(ta) ? a->geom_off : nullptr, a->validity,
                   view(b, bxy), is_multi(tb) ? b->geom_off : nullptr, b->validity, res.p, valid.p);
    } else if (ta == GPL_LINESTRING && tb == GPL_LINESTRING) {
        Scratch<uint8_t> flag;
        GPL_TRY(flag.get(ctx, (size_t)n));
        GPL_LAUNCH(ctx, k_ls_ls_fast<1>, warp_grid(n, kPairWarps), kPairWarps * 32, 0, n, axy, a->geom_off, a->validity, bxy, b->geom_off,
                   b->validity, nullptr, res.p, valid.p, flag.p);
        GPL_LAUNCH(ctx, k_ls_ls_exact<1>, warp_grid(ceil_div(n, 32), kPairWarps), kPairWarps * 32, 0, n, axy, a->geom_off, bxy, b->geom_off,
                   flag.p, nullptr, res.p, valid.p);
    } else if (ta == GPL_POINT && tb == GPL_POINT) {
        GPL_LAUNCH(ctx, k_point_point_dist, (int)ceil_div(n, 256), 256, 0, n, axy, a->validity, bxy, b->validity, res.p, valid.p);
    } else if (ta == GPL_POINT && tb == GPL_LINESTRING) {
        GPL_LAUNCH(ctx, k_point_ls_dist, warp_grid(n, 8), 256, 0, n, axy, a->validity, bxy, b->geom_off, b->validity, res.p, valid.p);
    } else if (ta == GPL_LINESTRING && tb == GPL_POINT) {
        GPL_LAUNCH(ctx, k_point_ls_dist, warp_grid(n, 8), 256, 0, n, bxy, b->validity, axy, a->geom_off, a->validity, res.p, valid.p);
    } else if (ta == GPL_POINT && tb == GPL_POLYGON) {
        GPL_LAUNCH(ctx, k_poly_point<1>, warp_grid(n, 8), 256, 0, b->type, n, bxy, b->geom_off, b->part_off, b->ring_off, b->validity,
                   axy, a->validity, nullptr, res.p, valid.p);
    } else if (tb != GPL_POINT) {  // LineString x Polygon, Polygon x LineString, Polygon x Polygon
        Side sa{ta, axy, a->geom_off, a->part_off, a->ring_off}, sb{tb, bxy, b->geom_off, b->part_off, b->ring_off};
        GPL_LAUNCH(ctx, k_distance_generic, warp_grid(n, 8), 256, 0, n, sa, a->validity, sb, b->validity, res.p, valid.p);
    } else {
        GPL_LAUNCH(ctx, k_poly_point<1>, warp_grid(n, 8), 256, 0, a->type, n, axy, a->geom_off, a->part_off, a->ring_off, a->validity,
                   bxy, b->validity, nullptr, res.p, valid.p);
    }
    GPL_TRY(valid.deliver(ctx));
    return res.deliver(ctx);
}

// ================================================================================================================
// general spatial join: spatial_join(lhs, rhs, predicate) for any two geometry columns (spatial_index.rs:37-157)
// ================================================================================================================
// Reference: both sides get an R-tree of per-row envelopes (:314-350), `intersection_candidates_with_other_tree`
// yields every pair whose envelopes intersect (closed intervals, :74-76), and each pair is tested by type-pair dispatch
// (:89-137); pairs that pass are emitted as (lhs_index, rhs_index) in tree-traversal order (unspecified; compare as sets).
// Here: envelopes of both sides (k_envelope), a uniform grid over the union box of the RIGHT envelopes holding, per cell,
// the rows whose envelope overlaps it; one thread per LEFT row walks the cells its envelope overlaps and keeps the
// candidates whose envelope intersects (each pair is reported from the single cell that holds the lower-left corner of
// the intersection box); count -> scan -> write gives the candidate list, a warp per candidate evaluates the
// dispatched predicate, and a second scan compacts the hits.  The compaction keeps them grouped by left row, so a sort of
// each row's right rows (sorted_pairs, join_host.cuh) puts the list in (lhs, rhs) order.  Points x (Multi)Polygons with
// millions of points should use gpl_pip_index_build + gpl_contains_join (the north-star path); this entry point is the
// general one.
// JoinGrid, jg_cell and the grid build (join_grid_build): join_grid.cuh; struct gpl_pairs: common.cuh
namespace gpl {

template <int PASS>
__global__ void k_join_candidates(const double *__restrict__ l4, const uint8_t *__restrict__ lhas, int64_t nl, const double *__restrict__ r4,
                                  JoinGrid jg, double ux1, double uy1, const int32_t *__restrict__ cell_start,
                                  const int32_t *__restrict__ items, int32_t *__restrict__ counts, const int64_t *__restrict__ off,
                                  uint64_t *__restrict__ lhs, uint64_t *__restrict__ rhs) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= nl) return;
    int32_t cnt = 0;
    int64_t w = PASS == 1 ? off[i] : 0;
    if (lhas[i]) {
        const double lx0 = l4[4 * i], ly0 = l4[4 * i + 1], lx1 = l4[4 * i + 2], ly1 = l4[4 * i + 3];
        // outside the union box of the right side: no candidate (closed intervals)
        if (!(lx1 < jg.x0 || ly1 < jg.y0 || lx0 > ux1 || ly0 > uy1)) {
            const int32_t cx0 = jg_cell(lx0, jg.x0, jg.inv_w, jg.g), cx1 = jg_cell(lx1, jg.x0, jg.inv_w, jg.g);
            const int32_t cy0 = jg_cell(ly0, jg.y0, jg.inv_h, jg.g), cy1 = jg_cell(ly1, jg.y0, jg.inv_h, jg.g);
            for (int32_t cy = cy0; cy <= cy1; ++cy)
                for (int32_t cx = cx0; cx <= cx1; ++cx) {
                    const int64_t c = (int64_t)cy * jg.g + cx;
                    for (int32_t k = cell_start[c]; k < cell_start[c + 1]; ++k) {
                        const int32_t j = items[k];
                        const double rx0 = r4[4 * j], ry0 = r4[4 * j + 1], rx1 = r4[4 * j + 2], ry1 = r4[4 * j + 3];
                        if (lx0 > rx1 || rx0 > lx1 || ly0 > ry1 || ry0 > ly1) continue;  // AABB intersection, closed
                        // report the pair from the one cell that holds the lower-left corner of the intersection box
                        if (jg_cell(fmax(lx0, rx0), jg.x0, jg.inv_w, jg.g) != cx || jg_cell(fmax(ly0, ry0), jg.y0, jg.inv_h, jg.g) != cy) continue;
                        if (PASS == 1) lhs[w] = (uint64_t)i, rhs[w] = (uint64_t)j, ++w;
                        ++cnt;
                    }
                }
        }
    }
    if (PASS == 0) counts[i] = cnt;
}
// the right rows of the hits, in candidate order, and the first hit of each left row: row i's candidates are
// [cand_off[i], cand_off[i + 1]) and the compaction keeps their order, so its hits are [row_off[i], row_off[i + 1])
__global__ void __launch_bounds__(256) k_join_hits(int64_t n_cand, const uint8_t *__restrict__ hit, const int64_t *__restrict__ hit_off,
                                                   const uint64_t *__restrict__ cr, int32_t *__restrict__ raw, int64_t nl,
                                                   const int64_t *__restrict__ cand_off, int64_t *__restrict__ row_off) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t k = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; k < n_cand || k <= nl; k += stride) {
        if (k < n_cand && hit[k]) raw[hit_off[k]] = (int32_t)cr[k];
        if (k <= nl) row_off[k] = hit_off[cand_off[k]];
    }
}

// The candidate stage of the general join: envelopes of both sides, the grid over the right side's union box, the
// candidate list (count -> scan -> write), the exact test `test` per candidate, the compaction of the hits and their sort
// by (lhs, rhs) (sorted_pairs, join_host.cuh) into out.
int join_candidate_pairs(gpl_ctx *ctx, const gpl_array *lhs, const gpl_array *rhs, JoinTest test, const char *who, bool with_dist, Pairs &out) {
    const int64_t nl = lhs->n_geoms, nr = rhs->n_geoms;
    const int tl = lhs->type, tr = rhs->type;
    if (nl == 0 || nr == 0) return pairs_new(ctx, 0, with_dist, out);
    // ---- envelopes -----------------------------------------------------------------------------------------------------
    Scratch<double> l4, r4;
    Scratch<uint8_t> lh, rh;
    GPL_TRY(l4.get(ctx, (size_t)nl * 4));
    GPL_TRY(r4.get(ctx, (size_t)nr * 4));
    GPL_TRY(lh.get(ctx, (size_t)nl));
    GPL_TRY(rh.get(ctx, (size_t)nr));
    GPL_TRY(envelope_raw(ctx, lhs, l4.p, lh.p));
    GPL_TRY(envelope_raw(ctx, rhs, r4.p, rh.p));
    // ---- grid over the right side's union box ------------------------------------------------------------------------------
    GridBuild grid;
    GPL_TRY(join_grid_build(ctx, r4.p, rh.p, nr, nr, who, grid));
    if (grid.jg.g == 0) return pairs_new(ctx, 0, with_dist, out);  // no right row has an envelope
    // ---- candidates: count -> scan -> write ----------------------------------------------------------------------------------
    Scratch<int32_t> cand_count;
    Scratch<int64_t> tot, cand_off;
    GPL_TRY(tot.get(ctx, 1));
    GPL_TRY(cand_count.get(ctx, (size_t)nl + 1));
    GPL_TRY(cand_off.get(ctx, (size_t)nl + 2));
    GPL_LAUNCH(ctx, k_join_candidates<0>, (int)ceil_div(nl, 128), 128, 0, l4.p, lh.p, nl, r4.p, grid.jg, grid.ux1, grid.uy1, grid.cell_start.p,
               grid.items.p, cand_count.p, nullptr, nullptr, nullptr);
    GPL_TRY((exclusive_scan<int32_t, int64_t>(ctx, cand_count.p, nl, cand_off.p, tot.p)));
    int64_t n_cand = 0;
    GPL_CUDA(cudaMemcpyAsync(&n_cand, tot.p, sizeof(int64_t), cudaMemcpyDeviceToHost, ctx->stream));
    GPL_CUDA(cudaStreamSynchronize(ctx->stream));
    if (n_cand == 0) return pairs_new(ctx, 0, with_dist, out);
    Scratch<uint64_t> cl, cr;
    GPL_TRY(cl.get(ctx, (size_t)n_cand));
    GPL_TRY(cr.get(ctx, (size_t)n_cand));
    GPL_LAUNCH(ctx, k_join_candidates<1>, (int)ceil_div(nl, 128), 128, 0, l4.p, lh.p, nl, r4.p, grid.jg, grid.ux1, grid.uy1, grid.cell_start.p,
               grid.items.p, nullptr, cand_off.p, cl.p, cr.p);
    // ---- exact predicate per candidate ------------------------------------------------------------------------------------------
    Scratch<uint8_t> hit;
    GPL_TRY(hit.get(ctx, (size_t)n_cand));
    const double2 *lxy = reinterpret_cast<const double2 *>(lhs->xy), *rxy = reinterpret_cast<const double2 *>(rhs->xy);
    const Side sl{tl, lxy, lhs->geom_off, lhs->part_off, lhs->ring_off}, sr{tr, rxy, rhs->geom_off, rhs->part_off, rhs->ring_off};
    const int pgrid = warp_grid(n_cand, 8);
    switch (test) {
    case JOIN_POINT_IN_R: GPL_LAUNCH(ctx, k_contains_point_pairs, pgrid, 256, 0, n_cand, sr, rhs->validity, lxy, lhs->validity, cr.p, cl.p, hit.p); break;
    case JOIN_POINT_IN_L: GPL_LAUNCH(ctx, k_contains_point_pairs, pgrid, 256, 0, n_cand, sl, lhs->validity, rxy, rhs->validity, cl.p, cr.p, hit.p); break;
    case JOIN_POLY_CONTAINS:
        GPL_LAUNCH(ctx, k_contains_polygon, pgrid, 256, 0, n_cand, polygon_view(lhs), tl == GPL_MULTIPOLYGON ? lhs->geom_off : nullptr, lhs->validity,
                   polygon_view(rhs), rhs->validity, cl.p, cr.p, hit.p);
        break;
    default: GPL_LAUNCH(ctx, k_intersects_pairs, pgrid, 256, 0, n_cand, sl, lhs->validity, sr, rhs->validity, cl.p, cr.p, hit.p); break;
    }
    // ---- compaction and per-row sort ---------------------------------------------------------------------------------------------
    Scratch<int64_t> hit_off, row_off;
    GPL_TRY(hit_off.get(ctx, (size_t)n_cand + 2));
    GPL_TRY((exclusive_scan<uint8_t, int64_t>(ctx, hit.p, n_cand, hit_off.p, tot.p)));
    int64_t n_hit = 0;
    GPL_CUDA(cudaMemcpyAsync(&n_hit, tot.p, sizeof(int64_t), cudaMemcpyDeviceToHost, ctx->stream));
    GPL_CUDA(cudaStreamSynchronize(ctx->stream));
    if (n_hit == 0) return pairs_new(ctx, 0, with_dist, out);
    Scratch<int32_t> raw;
    GPL_TRY(raw.get(ctx, (size_t)n_hit));
    GPL_TRY(row_off.get(ctx, (size_t)nl + 1));
    GPL_LAUNCH(ctx, k_join_hits, flat_grid(std::max(n_cand, nl + 1)), 256, 0, n_cand, hit.p, hit_off.p, cr.p, raw.p, nl, cand_off.p, row_off.p);
    return sorted_pairs(ctx, nl, row_off.p, raw.p, nullptr, n_hit, with_dist, out);
}

// the order-preserving compaction of keep_pairs (join_host.cuh): pair i (with goff, also its row's offset) to pos[i]
__global__ void __launch_bounds__(256) k_keep_pairs(int64_t n, const uint8_t *__restrict__ keep, const int64_t *__restrict__ pos,
                                                    const uint64_t *__restrict__ l, const uint64_t *__restrict__ r, uint64_t *__restrict__ ol,
                                                    uint64_t *__restrict__ orr, const int64_t *__restrict__ goff, int64_t *__restrict__ ogoff) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i <= n; i += stride) {
        if (i == n) {
            if (goff) ogoff[pos[n]] = goff[n];
        } else if (keep[i]) {
            ol[pos[i]] = l[i], orr[pos[i]] = r[i];
            if (goff) ogoff[pos[i]] = goff[i];
        }
    }
}
int keep_pairs(gpl_ctx *ctx, const gpl_pairs *in, const uint8_t *keep, Pairs &out, const int64_t *goff, Scratch<int64_t> *ogoff) {
    const int64_t n = in->n;
    Scratch<int64_t> pos;
    GPL_TRY(pos.get(ctx, (size_t)n + 1));
    GPL_TRY((exclusive_scan<uint8_t, int64_t>(ctx, keep, n, pos.p, nullptr)));
    int64_t m = 0;
    GPL_CUDA(cudaMemcpyAsync(&m, pos.p + n, sizeof(int64_t), cudaMemcpyDeviceToHost, ctx->stream));
    GPL_CUDA(cudaStreamSynchronize(ctx->stream));
    GPL_TRY(pairs_new(ctx, m, false, out));
    if (goff) GPL_TRY(ogoff->get(ctx, (size_t)m + 1));
    GPL_LAUNCH(ctx, k_keep_pairs, flat_grid(n + 1), 256, 0, n, keep, pos.p, in->lhs, in->rhs, out->lhs, out->rhs, goff, goff ? ogoff->p : nullptr);
    GPL_CUDA(cudaStreamSynchronize(ctx->stream));  // pos returns to the cache when this scope ends
    return GPL_OK;
}

}  // namespace gpl

extern "C" void gpl_pairs_free(gpl_pairs *p) {
    if (!p) return;
    p->ctx->release(p->lhs);
    p->ctx->release(p->rhs);
    p->ctx->release(p->dist);
    delete p;
}
extern "C" int64_t gpl_pairs_count(const gpl_pairs *p) { return p ? p->n : 0; }
extern "C" int gpl_pairs_copy_distance(gpl_ctx *ctx, const gpl_pairs *p, double *distance, int mem) {
    GPL_REQUIRE(ctx && p && (p->n == 0 || distance), GPL_ERR_INVALID_ARG, "gpl_pairs_copy_distance: NULL argument");
    GPL_REQUIRE(p->with_dist, GPL_ERR_INVALID_ARG, "gpl_pairs_copy_distance: this pair list carries no distances");
    GPL_TRY(check_mem(mem, "gpl_pairs_copy_distance"));
    GPL_CUDA(cudaSetDevice(ctx->device));
    if (p->n == 0) return GPL_OK;
    const cudaMemcpyKind kind = mem == GPL_HOST ? cudaMemcpyDeviceToHost : cudaMemcpyDeviceToDevice;
    GPL_CUDA(cudaMemcpyAsync(distance, p->dist, sizeof(double) * p->n, kind, ctx->stream));
    if (mem == GPL_HOST) GPL_CUDA(cudaStreamSynchronize(ctx->stream));
    return GPL_OK;
}
extern "C" int gpl_pairs_copy(gpl_ctx *ctx, const gpl_pairs *p, uint64_t *lhs, uint64_t *rhs, int mem) {
    GPL_REQUIRE(ctx && p && (p->n == 0 || (lhs && rhs)), GPL_ERR_INVALID_ARG, "gpl_pairs_copy: NULL argument");
    GPL_TRY(check_mem(mem, "gpl_pairs_copy"));
    GPL_CUDA(cudaSetDevice(ctx->device));
    if (p->n == 0) return GPL_OK;
    const cudaMemcpyKind kind = mem == GPL_HOST ? cudaMemcpyDeviceToHost : cudaMemcpyDeviceToDevice;
    GPL_CUDA(cudaMemcpyAsync(lhs, p->lhs, sizeof(uint64_t) * p->n, kind, ctx->stream));
    GPL_CUDA(cudaMemcpyAsync(rhs, p->rhs, sizeof(uint64_t) * p->n, kind, ctx->stream));
    if (mem == GPL_HOST) GPL_CUDA(cudaStreamSynchronize(ctx->stream));
    return GPL_OK;
}

// row-wise (Multi)Polygon.contains(Polygon)
extern "C" int gpl_contains_polygon(gpl_ctx *ctx, const gpl_array *a, const gpl_array *b, uint8_t *out_bitmap, int mem) {
    GPL_REQUIRE(ctx && a && b && out_bitmap, GPL_ERR_INVALID_ARG, "gpl_contains_polygon: NULL argument");
    GPL_TRY(check_mem(mem, "gpl_contains_polygon"));
    GPL_TRY(require_same_length(a, b, "contains"));
    GPL_REQUIRE((a->type == GPL_POLYGON || a->type == GPL_MULTIPOLYGON) && b->type == GPL_POLYGON, GPL_ERR_INVALID_TYPE,
                "Expected (Multi)Polygon x Polygon (found %s x %s)", type_name(a->type), type_name(b->type));
    GPL_CUDA(cudaSetDevice(ctx->device));
    const int64_t n = a->n_geoms;
    if (n == 0) return GPL_OK;
    Scratch<uint8_t> bytes;
    GPL_TRY(bytes.get(ctx, (size_t)n));
    GPL_LAUNCH(ctx, k_contains_polygon, warp_grid(n, 8), 256, 0, n, polygon_view(a), a->type == GPL_MULTIPOLYGON ? a->geom_off : nullptr, a->validity,
               polygon_view(b), b->validity, nullptr, nullptr, bytes.p);
    return finish_bitmap(ctx, bytes.p, n, out_bitmap, mem);
}

extern "C" int gpl_spatial_join(gpl_ctx *ctx, const gpl_array *lhs, const gpl_array *rhs, int predicate, gpl_pairs **out) {
    GPL_REQUIRE(ctx && lhs && rhs && out, GPL_ERR_INVALID_ARG, "gpl_spatial_join: NULL argument");
    *out = nullptr;
    GPL_REQUIRE(predicate == GPL_PREDICATE_INTERSECTS || predicate == GPL_PREDICATE_CONTAINS, GPL_ERR_INVALID_ARG,
                "gpl_spatial_join: predicate must be GPL_PREDICATE_INTERSECTS or GPL_PREDICATE_CONTAINS");
    GPL_CUDA(cudaSetDevice(ctx->device));
    const int64_t nl = lhs->n_geoms, nr = rhs->n_geoms;
    GPL_REQUIRE(nl == 0 || nr == 0 || (nl < (1LL << 31) && nr < (1LL << 31)), GPL_ERR_UNSUPPORTED, "gpl_spatial_join: at most 2^31 rows per side");
    // ---- the type-pair dispatch table of spatial_index.rs:89-137 (anything else: no pair matches) ------------------------
    const int tl = lhs->type, tr = rhs->type;
    const int cl_ = side_class_host(tl), cr_ = side_class_host(tr);
    int test = -1;
    if (tl == GPL_POINT && (cr_ == 2 || tr == GPL_LINESTRING || tr == GPL_MULTILINESTRING)) test = JOIN_POINT_IN_R;       // :91, :95, :130-134
    else if (tr == GPL_POINT && (cl_ == 2 || tl == GPL_LINESTRING || tl == GPL_MULTILINESTRING)) test = JOIN_POINT_IN_L;  // :92, :96, :129-133
    else if ((tl == GPL_POLYGON || tl == GPL_MULTIPOLYGON) && tr == GPL_POLYGON) test = predicate == GPL_PREDICATE_CONTAINS ? JOIN_POLY_CONTAINS : JOIN_INTERSECTS;  // :99-115
    else if (tl == GPL_POLYGON && tr == GPL_MULTIPOLYGON && predicate == GPL_PREDICATE_INTERSECTS) test = JOIN_INTERSECTS;  // :118-122
    Pairs res(nullptr, gpl_pairs_free);
    GPL_TRY(test < 0 ? pairs_new(ctx, 0, false, res) : join_candidate_pairs(ctx, lhs, rhs, (JoinTest)test, "gpl_spatial_join", false, res));
    *out = res.release();
    return GPL_OK;
}
