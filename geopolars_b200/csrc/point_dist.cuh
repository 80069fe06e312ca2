// point_dist.cuh — the point-to-geometry distance routines of GeoSeries::distance (geo 0.27 euclidean_distance.rs,
// recalled; restated in oracle/geo_oracle.c), shared by the row-wise kernels of k_pairs.cu and the nearest join of
// k_nearest.cu.  Every routine is warp cooperative: all 32 lanes call it with the same point and the same row, and
// the result is warp-uniform.  `min` is exact, so the result does not depend on how lanes split the segments.
#pragma once

#include "common.cuh"

namespace gpl {

// geo-types line_string_contains_point (epsilon based, inexact by design), warp cooperative
__device__ __forceinline__ bool line_string_contains_point(const double2 *__restrict__ xy, int64_t c0, int64_t n, double2 p,
                                                           int lane) {
    if (n == 0) return false;
    if (n == 1) {
        float d = (float)pt_dist(xy[c0], p);
        return d <= 1.1920929e-07f;
    }
    bool hit = false;
    for (int64_t i = lane; i < n; i += 32) {
        double2 q = xy[c0 + i];
        if (q.x == p.x && q.y == p.y) hit = true;
    }
    for (int64_t i = lane; i < n - 1; i += 32) {
        double2 s = xy[c0 + i], e = xy[c0 + i + 1];
        double dx = e.x - s.x, dy = e.y - s.y;
        bool hx = dx != 0.0, hy = dy != 0.0;
        double tx = hx ? (p.x - s.x) / dx : 0.0;
        double ty = hy ? (p.y - s.y) / dy : 0.0;
        bool c;
        if (!hx && !hy) c = (p.x == s.x && p.y == s.y);
        else if (hx && !hy) c = (p.y == s.y && 0.0 <= tx && tx <= 1.0);
        else if (!hx && hy) c = (p.x == s.x && 0.0 <= ty && ty <= 1.0);
        else c = (fabs(tx - ty) <= 2.220446049250313e-16 && 0.0 <= tx && tx <= 1.0);
        hit = hit || c;
    }
    return __any_sync(0xffffffffu, hit);
}
__device__ __forceinline__ double point_ls_distance(const double2 *__restrict__ xy, int64_t c0, int64_t n, double2 p, int lane) {
    if (n == 0 || line_string_contains_point(xy, c0, n, p, lane)) return 0.0;
    double best = 1.7976931348623157e308;
    for (int64_t i = lane; i < n - 1; i += 32) best = fmin(best, line_segment_distance(p, xy[c0 + i], xy[c0 + i + 1]));
    return warp_min(best);
}

// coord_pos_relative_to_ring, warp cooperative: 0 outside, 1 boundary, 2 inside
__device__ __forceinline__ int ring_position(const double2 *__restrict__ xy, int64_t c0, int64_t n, double2 p, int lane) {
    if (n == 0) return 0;
    if (n == 1) {
        double2 q = xy[c0];
        return (q.x == p.x && q.y == p.y) ? 1 : 0;
    }
    double2 first = xy[c0], last = xy[c0 + n - 1];
    bool closing = !(first.x == last.x && first.y == last.y);  // Polygon::new would close the ring
    int64_t nseg = n - 1 + (closing ? 1 : 0);
    int wn = 0;
    bool boundary = false;
    for (int64_t i = lane; i < nseg; i += 32) {
        double2 s = xy[c0 + i];
        double2 e = (i + 1 < n) ? xy[c0 + i + 1] : first;
        if (s.y <= p.y) {
            if (e.y >= p.y) {
                double o = orient2d(s.x, s.y, e.x, e.y, p.x, p.y);
                if (o > 0.0 && e.y != p.y) wn += 1;
                else if (o == 0.0 && value_in_between(p.x, s.x, e.x)) boundary = true;
            }
        } else if (e.y <= p.y) {
            double o = orient2d(s.x, s.y, e.x, e.y, p.x, p.y);
            if (o < 0.0) wn -= 1;
            else if (o == 0.0 && value_in_between(p.x, s.x, e.x)) boundary = true;
        }
    }
    if (__any_sync(0xffffffffu, boundary)) return 1;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) wn += __shfl_xor_sync(0xffffffffu, wn, o);
    return wn == 0 ? 0 : 2;
}
// Polygon::calculate_coordinate_position over rings [r0,r1)
__device__ __forceinline__ void polygon_position(const double2 *__restrict__ xy, const int64_t *__restrict__ ring_off, int64_t r0,
                                                 int64_t r1, double2 p, int lane, bool &inside, int &boundary_count) {
    if (r1 <= r0) return;
    if (ring_off[r0 + 1] - ring_off[r0] == 0) return;
    int pos = ring_position(xy, ring_off[r0], ring_off[r0 + 1] - ring_off[r0], p, lane);
    if (pos == 0) return;
    if (pos == 1) {
        boundary_count += 1;
        return;
    }
    for (int64_t r = r0 + 1; r < r1; ++r) {
        int hp = ring_position(xy, ring_off[r], ring_off[r + 1] - ring_off[r], p, lane);
        if (hp == 1) {
            boundary_count += 1;
            return;
        }
        if (hp == 2) return;
    }
    inside = true;
}

struct Side {
    int type;
    const double2 *xy;
    const int64_t *go, *po, *ro;
};

// Point x Polygon distance of the polygon q of the POLYGON view `s` (go: ring offsets of each polygon, ro: coordinate
// offsets of each ring): 0 inside or on the boundary, else the minimum over the holes and the exterior's segments.
__device__ __forceinline__ double point_polygon_distance(const Side &s, int64_t q, double2 p, int lane) {
    const int64_t r0 = s.go[q], r1 = s.go[q + 1];
    if (r1 <= r0 || s.ro[r0 + 1] - s.ro[r0] == 0) return 0.0;
    bool inside = false;
    int bc = 0;
    polygon_position(s.xy, s.ro, r0, r1, p, lane, inside, bc);
    if (bc % 2 == 1 || inside) return 0.0;
    double acc = 1.7976931348623157e308;
    for (int64_t h = r0 + 1; h < r1; ++h) acc = fmin(acc, point_ls_distance(s.xy, s.ro[h], s.ro[h + 1] - s.ro[h], p, lane));
    double ext = 1.7976931348623157e308;
    const int64_t c0 = s.ro[r0], nn = s.ro[r0 + 1] - c0;
    for (int64_t i = lane; i < nn - 1; i += 32) ext = fmin(ext, line_segment_distance(p, s.xy[c0 + i], s.xy[c0 + i + 1]));
    return fmin(acc, warp_min(ext));
}

}  // namespace gpl
