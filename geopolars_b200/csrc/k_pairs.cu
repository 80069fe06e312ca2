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
#include "point_dist.cuh"
#include "scan.cuh"

namespace gpl {

constexpr int kPairWarps = 8;     // warps per CTA
constexpr int kPairSmemCoords = 128;  // coords of (A,B) staged per warp; longer rows read global memory

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

// distance for LineString x Polygon, Polygon x LineString, Polygon x Polygon rows (geo 0.27
// euclidean_distance.rs, recalled): 0 when the row intersects; a geometry lying strictly inside the other's
// exterior (hence in a hole) is measured against the interior rings, everything else exterior to exterior /
// linestring to exterior; each of those is the nearest-neighbour minimum over (vertex, segment) items.
// geo's rotating-calipers branch for two convex polygons computes the same minimum (different roundings).
__device__ __forceinline__ double chain_nn_dist2(const Chain &a, const Chain &b, int lane) {
    return ls_ls_min_dist2(a, a.coords(), b, b.coords(), lane);
}
__global__ void __launch_bounds__(256) k_distance_generic(int64_t n, Side a, const uint8_t *__restrict__ av, Side b,
                                                          const uint8_t *__restrict__ bv, double *__restrict__ out,
                                                          uint8_t *__restrict__ out_valid) {
    const int lane = threadIdx.x & 31;
    int64_t warp = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
    const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    const double big = 1.7976931348623157e308;
    for (int64_t r = warp; r < n; r += nwarps) {
        bool ok = bit_get(av, r) && bit_get(bv, r);
        double d = nan("");
        if (ok) {
            // first chain of each side (the linestring, or the exterior ring) must have a line
            int64_t a0 = a.go[r], a1 = a.go[r + 1], b0 = b.go[r], b1 = b.go[r + 1];
            const bool pa = a.type == GPL_POLYGON, pb = b.type == GPL_POLYGON;
            const Chain ea = pa ? (a1 > a0 ? part_ring(a, a0) : Chain{a.xy, 0, false}) : make_line(a.xy, a0, a1);
            const Chain eb = pb ? (b1 > b0 ? part_ring(b, b0) : Chain{b.xy, 0, false}) : make_line(b.xy, b0, b1);
            if (ea.n < 2 || eb.n < 2) {
                ok = false;
            } else if (row_intersects(a, r, b, r, lane)) {
                d = 0.0;
            } else {
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
                d = sqrt(m);
            }
        }
        if (lane == 0) {
            out[r] = ok ? d : nan("");
            if (out_valid) out_valid[r] = ok ? 1 : 0;
        }
    }
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
struct SymQ {
    double xx, xy, vx, vy;
    int side;
};
__device__ __forceinline__ int cmpd(double a, double b) { return (a > b) - (a < b); }
__device__ __forceinline__ int sgnd(double a) { return (a > 0.0) - (a < 0.0); }
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
__device__ __forceinline__ double2 bcast2(double2 v, int src) {
    return make_double2(__shfl_sync(0xffffffffu, v.x, src), __shfl_sync(0xffffffffu, v.y, src));
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

int pack_bits(gpl_ctx *ctx, const uint8_t *bytes_dev, uint8_t *bitmap_dev, int64_t n);
int deliver(gpl_ctx *ctx, void *dst, const void *src_dev, size_t bytes, int mem);

static int warp_grid(int64_t rows, int warps_per_cta) {
    int64_t want = ceil_div(rows, warps_per_cta);
    return (int)std::max<int64_t>(1, std::min<int64_t>(want, (int64_t)kSMs * 16));
}

static int side_class_host(int t) { return (t == GPL_POINT || t == GPL_MULTIPOINT) ? 0 : (t == GPL_LINESTRING || t == GPL_MULTILINESTRING) ? 1 : 2; }
static const char *type_name(int t) {
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

// bool result: bytes on device -> Arrow bitmap in the caller's memory
static int finish_bitmap(gpl_ctx *ctx, const uint8_t *bytes_dev, int64_t n, uint8_t *out_bitmap, int mem) {
    size_t nb = (size_t)(n + 7) / 8;
    if (mem == GPL_DEVICE) return pack_bits(ctx, bytes_dev, out_bitmap, n);
    Scratch<uint8_t> bm;
    GPL_TRY(bm.get(ctx, nb));
    GPL_TRY(pack_bits(ctx, bytes_dev, bm.p, n));
    return deliver(ctx, out_bitmap, bm.p, nb, GPL_HOST);
}

}  // namespace gpl

using namespace gpl;

extern "C" int gpl_intersects(gpl_ctx *ctx, const gpl_array *a, const gpl_array *b, uint8_t *out_bitmap, int mem) {
    GPL_REQUIRE(ctx && a && b && out_bitmap, GPL_ERR_INVALID_ARG, "gpl_intersects: NULL argument");
    GPL_REQUIRE(a->n_geoms == b->n_geoms, GPL_ERR_LENGTH_MISMATCH, "intersects: lengths differ (%lld vs %lld)",
                (long long)a->n_geoms, (long long)b->n_geoms);
    GPL_REQUIRE(a->type >= GPL_POINT && a->type <= GPL_MULTIPOLYGON && a->type != GPL_LINEARRING && b->type >= GPL_POINT &&
                    b->type <= GPL_MULTIPOLYGON && b->type != GPL_LINEARRING,
                GPL_ERR_INVALID_TYPE, "intersects: unsupported geometry pair %s x %s", type_name(a->type), type_name(b->type));
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
    GPL_REQUIRE(polygons->n_geoms == points->n_geoms, GPL_ERR_LENGTH_MISMATCH, "contains: lengths differ (%lld vs %lld)",
                (long long)polygons->n_geoms, (long long)points->n_geoms);
    const bool area = polygons->type == GPL_POLYGON || polygons->type == GPL_MULTIPOLYGON;
    const bool lines = polygons->type == GPL_LINESTRING || polygons->type == GPL_MULTILINESTRING;
    GPL_REQUIRE((area || lines) && points->type == GPL_POINT, GPL_ERR_INVALID_TYPE,
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
    GPL_REQUIRE(a->n_geoms == b->n_geoms, GPL_ERR_LENGTH_MISMATCH, "distance: lengths differ (%lld vs %lld)",
                (long long)a->n_geoms, (long long)b->n_geoms);
    const int ta = a->type, tb = b->type;
    auto known = [](int t) {
        return t == GPL_POINT || t == GPL_LINESTRING || t == GPL_POLYGON || t == GPL_MULTIPOINT || t == GPL_MULTILINESTRING || t == GPL_MULTIPOLYGON;
    };
    GPL_REQUIRE(known(ta) && known(tb), GPL_ERR_INVALID_TYPE, "distance: unsupported geometry pair %s x %s", type_name(ta), type_name(tb));
    auto is_multi = [](int t) { return t == GPL_MULTIPOINT || t == GPL_MULTILINESTRING || t == GPL_MULTIPOLYGON; };
    GPL_CUDA(cudaSetDevice(ctx->device));
    int64_t n = a->n_geoms;
    if (n == 0) return GPL_OK;
    Scratch<double> tmp;
    Scratch<uint8_t> vbytes;
    double *dst = out;
    if (mem == GPL_HOST) {
        GPL_TRY(tmp.get(ctx, (size_t)n));
        dst = tmp.p;
    }
    uint8_t *vb = nullptr;
    if (out_validity) {
        GPL_TRY(vbytes.get(ctx, (size_t)n));
        vb = vbytes.p;
    }
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
                   view(b, bxy), is_multi(tb) ? b->geom_off : nullptr, b->validity, dst, vb);
    } else if (ta == GPL_LINESTRING && tb == GPL_LINESTRING) {
        Scratch<uint8_t> flag;
        GPL_TRY(flag.get(ctx, (size_t)n));
        GPL_LAUNCH(ctx, k_ls_ls_fast<1>, warp_grid(n, kPairWarps), kPairWarps * 32, 0, n, axy, a->geom_off, a->validity, bxy, b->geom_off,
                   b->validity, nullptr, dst, vb, flag.p);
        GPL_LAUNCH(ctx, k_ls_ls_exact<1>, warp_grid(ceil_div(n, 32), kPairWarps), kPairWarps * 32, 0, n, axy, a->geom_off, bxy, b->geom_off,
                   flag.p, nullptr, dst, vb);
    } else if (ta == GPL_POINT && tb == GPL_POINT) {
        GPL_LAUNCH(ctx, k_point_point_dist, (int)ceil_div(n, 256), 256, 0, n, axy, a->validity, bxy, b->validity, dst, vb);
    } else if (ta == GPL_POINT && tb == GPL_LINESTRING) {
        GPL_LAUNCH(ctx, k_point_ls_dist, warp_grid(n, 8), 256, 0, n, axy, a->validity, bxy, b->geom_off, b->validity, dst, vb);
    } else if (ta == GPL_LINESTRING && tb == GPL_POINT) {
        GPL_LAUNCH(ctx, k_point_ls_dist, warp_grid(n, 8), 256, 0, n, bxy, b->validity, axy, a->geom_off, a->validity, dst, vb);
    } else if (ta == GPL_POINT && tb == GPL_POLYGON) {
        GPL_LAUNCH(ctx, k_poly_point<1>, warp_grid(n, 8), 256, 0, b->type, n, bxy, b->geom_off, b->part_off, b->ring_off, b->validity,
                   axy, a->validity, nullptr, dst, vb);
    } else if (tb != GPL_POINT) {  // LineString x Polygon, Polygon x LineString, Polygon x Polygon
        Side sa{ta, axy, a->geom_off, a->part_off, a->ring_off}, sb{tb, bxy, b->geom_off, b->part_off, b->ring_off};
        GPL_LAUNCH(ctx, k_distance_generic, warp_grid(n, 8), 256, 0, n, sa, a->validity, sb, b->validity, dst, vb);
    } else {
        GPL_LAUNCH(ctx, k_poly_point<1>, warp_grid(n, 8), 256, 0, a->type, n, axy, a->geom_off, a->part_off, a->ring_off, a->validity,
                   bxy, b->validity, nullptr, dst, vb);
    }
    if (out_validity) GPL_TRY(finish_bitmap(ctx, vb, n, out_validity, mem));
    return deliver(ctx, out, dst, sizeof(double) * n, mem);
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
// dispatched predicate, and a second scan compacts the hits.  Points x (Multi)Polygons with millions of points should
// use gpl_pip_index_build + gpl_contains_join (the north-star path); this entry point is the general one.
// JoinGrid, jg_cell, k_join_union, k_join_cells: join_grid.cuh; struct gpl_pairs: common.cuh
namespace gpl {

int envelope_raw(gpl_ctx *ctx, const gpl_array *in, double *out4_dev, uint8_t *valid_bytes_dev);

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
__global__ void k_join_compact(const uint8_t *__restrict__ hit, const int64_t *__restrict__ off, int64_t n, const uint64_t *__restrict__ cl,
                               const uint64_t *__restrict__ cr, uint64_t *__restrict__ ol, uint64_t *__restrict__ orr) {
    const int64_t k = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (k < n && hit[k]) ol[off[k]] = cl[k], orr[off[k]] = cr[k];
}

static Side polygon_view(const gpl_array *g) {
    const double2 *xy = reinterpret_cast<const double2 *>(g->xy);
    if (g->type == GPL_MULTIPOLYGON) return Side{GPL_POLYGON, xy, g->part_off, nullptr, g->ring_off};
    return Side{g->type, xy, g->geom_off, g->part_off, g->ring_off};
}

}  // namespace gpl

extern "C" void gpl_pairs_free(gpl_pairs *p) {
    if (!p) return;
    p->ctx->release(p->lhs);
    p->ctx->release(p->rhs);
    delete p;
}
extern "C" int64_t gpl_pairs_count(const gpl_pairs *p) { return p ? p->n : 0; }
extern "C" int gpl_pairs_copy(gpl_ctx *ctx, const gpl_pairs *p, uint64_t *lhs, uint64_t *rhs, int mem) {
    GPL_REQUIRE(ctx && p && (p->n == 0 || (lhs && rhs)), GPL_ERR_INVALID_ARG, "gpl_pairs_copy: NULL argument");
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
    GPL_REQUIRE(a->n_geoms == b->n_geoms, GPL_ERR_LENGTH_MISMATCH, "contains: lengths differ (%lld vs %lld)", (long long)a->n_geoms,
                (long long)b->n_geoms);
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
    GPL_REQUIRE(predicate == GPL_PREDICATE_INTERSECTS || predicate == GPL_PREDICATE_CONTAINS, GPL_ERR_INVALID_ARG,
                "gpl_spatial_join: predicate must be GPL_PREDICATE_INTERSECTS or GPL_PREDICATE_CONTAINS");
    GPL_CUDA(cudaSetDevice(ctx->device));
    gpl_pairs *res = new gpl_pairs();
    res->ctx = ctx;
    *out = res;
    const int64_t nl = lhs->n_geoms, nr = rhs->n_geoms;
    if (nl == 0 || nr == 0) return GPL_OK;
    GPL_REQUIRE(nl < (1LL << 31) && nr < (1LL << 31), GPL_ERR_UNSUPPORTED, "gpl_spatial_join: at most 2^31 rows per side");
    // ---- the type-pair dispatch table of spatial_index.rs:89-137 (anything else: no pair matches) ------------------------
    const int tl = lhs->type, tr = rhs->type;
    const int cl_ = side_class_host(tl), cr_ = side_class_host(tr);
    enum { NONE, POINT_IN_R, POINT_IN_L, POLY_CONTAINS, INTERSECTS } mode = NONE;
    if (tl == GPL_POINT && (cr_ == 2 || tr == GPL_LINESTRING || tr == GPL_MULTILINESTRING)) mode = POINT_IN_R;       // :91, :95, :130-134
    else if (tr == GPL_POINT && (cl_ == 2 || tl == GPL_LINESTRING || tl == GPL_MULTILINESTRING)) mode = POINT_IN_L;  // :92, :96, :129-133
    else if ((tl == GPL_POLYGON || tl == GPL_MULTIPOLYGON) && tr == GPL_POLYGON) mode = predicate == GPL_PREDICATE_CONTAINS ? POLY_CONTAINS : INTERSECTS;  // :99-115
    else if (tl == GPL_POLYGON && tr == GPL_MULTIPOLYGON && predicate == GPL_PREDICATE_INTERSECTS) mode = INTERSECTS;  // :118-122
    if (mode == NONE) return GPL_OK;
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
    Scratch<unsigned long long> acc;
    GPL_TRY(acc.get(ctx, 4));
    GPL_CUDA(cudaMemsetAsync(acc.p, 0, 4 * sizeof(unsigned long long), ctx->stream));
    GPL_LAUNCH(ctx, k_join_union, (int)std::min<int64_t>(ceil_div(nr, 256), kSMs * 8), 256, 0, r4.p, rh.p, nr, acc.p);
    unsigned long long h_acc[4];
    GPL_CUDA(cudaMemcpyAsync(h_acc, acc.p, sizeof(h_acc), cudaMemcpyDeviceToHost, ctx->stream));
    GPL_CUDA(cudaStreamSynchronize(ctx->stream));
    if (h_acc[2] == 0ULL) return GPL_OK;  // no right row has an envelope
    auto dec = [](unsigned long long u) {
        const unsigned long long b = (u >> 63) ? (u & 0x7fffffffffffffffULL) : ~u;
        double d;
        memcpy(&d, &b, sizeof(d));
        return d;
    };
    const double ux0 = dec(~h_acc[0]), uy0 = dec(~h_acc[1]), ux1 = dec(h_acc[2]), uy1 = dec(h_acc[3]);
    JoinGrid jg;
    jg.g = (int32_t)std::min<int64_t>(2048, std::max<int64_t>(1, (int64_t)ceil(sqrt((double)nr))));
    jg.x0 = ux0, jg.y0 = uy0;
    const double w = ux1 - ux0, h = uy1 - uy0;
    jg.inv_w = (w > 0.0 && std::isfinite(w) && std::isfinite(jg.g / w)) ? jg.g / w : 0.0;
    jg.inv_h = (h > 0.0 && std::isfinite(h) && std::isfinite(jg.g / h)) ? jg.g / h : 0.0;
    const int64_t n_cells = (int64_t)jg.g * jg.g;
    Scratch<int32_t> cell_count, cell_start, items, cand_count;
    Scratch<int64_t> tot, cand_off;
    GPL_TRY(cell_count.get(ctx, (size_t)n_cells + 1));
    GPL_TRY(cell_start.get(ctx, (size_t)n_cells + 1));
    GPL_TRY(tot.get(ctx, 2));
    GPL_CUDA(cudaMemsetAsync(cell_count.p, 0, sizeof(int32_t) * (n_cells + 1), ctx->stream));
    GPL_LAUNCH(ctx, k_join_cells<0>, (int)ceil_div(nr, 128), 128, 0, r4.p, rh.p, nr, jg, cell_count.p, nullptr);
    GPL_TRY((exclusive_scan<int32_t, int32_t>(ctx, cell_count.p, n_cells, cell_start.p, tot.p)));
    int64_t n_items = 0;
    GPL_CUDA(cudaMemcpyAsync(&n_items, tot.p, sizeof(int64_t), cudaMemcpyDeviceToHost, ctx->stream));
    GPL_CUDA(cudaStreamSynchronize(ctx->stream));
    GPL_REQUIRE(n_items < (1LL << 31), GPL_ERR_UNSUPPORTED, "gpl_spatial_join: grid too dense (%lld cell items)", (long long)n_items);
    GPL_TRY(items.get(ctx, (size_t)n_items + 1));
    GPL_CUDA(cudaMemcpyAsync(cell_count.p, cell_start.p, sizeof(int32_t) * n_cells, cudaMemcpyDeviceToDevice, ctx->stream));  // cursors
    GPL_LAUNCH(ctx, k_join_cells<1>, (int)ceil_div(nr, 128), 128, 0, r4.p, rh.p, nr, jg, cell_count.p, items.p);
    // ---- candidates: count -> scan -> write ----------------------------------------------------------------------------------
    GPL_TRY(cand_count.get(ctx, (size_t)nl + 1));
    GPL_TRY(cand_off.get(ctx, (size_t)nl + 2));
    GPL_LAUNCH(ctx, k_join_candidates<0>, (int)ceil_div(nl, 128), 128, 0, l4.p, lh.p, nl, r4.p, jg, ux1, uy1, cell_start.p, items.p, cand_count.p,
               nullptr, nullptr, nullptr);
    GPL_TRY((exclusive_scan<int32_t, int64_t>(ctx, cand_count.p, nl, cand_off.p, tot.p + 1)));
    int64_t n_cand = 0;
    GPL_CUDA(cudaMemcpyAsync(&n_cand, tot.p + 1, sizeof(int64_t), cudaMemcpyDeviceToHost, ctx->stream));
    GPL_CUDA(cudaStreamSynchronize(ctx->stream));
    if (n_cand == 0) return GPL_OK;
    Scratch<uint64_t> cl, cr;
    GPL_TRY(cl.get(ctx, (size_t)n_cand));
    GPL_TRY(cr.get(ctx, (size_t)n_cand));
    GPL_LAUNCH(ctx, k_join_candidates<1>, (int)ceil_div(nl, 128), 128, 0, l4.p, lh.p, nl, r4.p, jg, ux1, uy1, cell_start.p, items.p, nullptr,
               cand_off.p, cl.p, cr.p);
    // ---- exact predicate per candidate ------------------------------------------------------------------------------------------
    Scratch<uint8_t> hit;
    GPL_TRY(hit.get(ctx, (size_t)n_cand));
    const double2 *lxy = reinterpret_cast<const double2 *>(lhs->xy), *rxy = reinterpret_cast<const double2 *>(rhs->xy);
    const Side sl{tl, lxy, lhs->geom_off, lhs->part_off, lhs->ring_off}, sr{tr, rxy, rhs->geom_off, rhs->part_off, rhs->ring_off};
    const int pgrid = warp_grid(n_cand, 8);
    switch (mode) {
    case POINT_IN_R: GPL_LAUNCH(ctx, k_contains_point_pairs, pgrid, 256, 0, n_cand, sr, rhs->validity, lxy, lhs->validity, cr.p, cl.p, hit.p); break;
    case POINT_IN_L: GPL_LAUNCH(ctx, k_contains_point_pairs, pgrid, 256, 0, n_cand, sl, lhs->validity, rxy, rhs->validity, cl.p, cr.p, hit.p); break;
    case POLY_CONTAINS:
        GPL_LAUNCH(ctx, k_contains_polygon, pgrid, 256, 0, n_cand, polygon_view(lhs), tl == GPL_MULTIPOLYGON ? lhs->geom_off : nullptr, lhs->validity,
                   polygon_view(rhs), rhs->validity, cl.p, cr.p, hit.p);
        break;
    default: GPL_LAUNCH(ctx, k_intersects_pairs, pgrid, 256, 0, n_cand, sl, lhs->validity, sr, rhs->validity, cl.p, cr.p, hit.p); break;
    }
    // ---- compaction ----------------------------------------------------------------------------------------------------------------
    Scratch<int64_t> hit_off;
    GPL_TRY(hit_off.get(ctx, (size_t)n_cand + 2));
    GPL_TRY((exclusive_scan<uint8_t, int64_t>(ctx, hit.p, n_cand, hit_off.p, tot.p)));
    int64_t n_hit = 0;
    GPL_CUDA(cudaMemcpyAsync(&n_hit, tot.p, sizeof(int64_t), cudaMemcpyDeviceToHost, ctx->stream));
    GPL_CUDA(cudaStreamSynchronize(ctx->stream));
    if (n_hit == 0) return GPL_OK;
    void *pl = nullptr, *pr = nullptr;
    GPL_TRY(ctx->alloc(sizeof(uint64_t) * (size_t)n_hit, &pl));
    res->lhs = (uint64_t *)pl;
    GPL_TRY(ctx->alloc(sizeof(uint64_t) * (size_t)n_hit, &pr));
    res->rhs = (uint64_t *)pr;
    res->n = n_hit;
    GPL_LAUNCH(ctx, k_join_compact, (int)ceil_div(n_cand, 256), 256, 0, hit.p, hit_off.p, n_cand, cl.p, cr.p, res->lhs, res->rhs);
    GPL_CUDA(cudaStreamSynchronize(ctx->stream));  // the scratch lists above return to the cache when this scope ends
    return GPL_OK;
}
