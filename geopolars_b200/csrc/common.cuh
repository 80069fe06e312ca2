// common.cuh — context, device arrays, error plumbing and the exact orientation predicate shared by
// every kernel of libgeopolars_b200.so.  sm_90a only; compiled with -fmad=false so that a*b+c is two
// rounded operations exactly like the reference's Rust (which never contracts to FMA).
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include <algorithm>
#include <map>
#include <memory>
#include <mutex>
#include <string>
#include <vector>

#include "../../include/geopolars_b200.h"

namespace gpl {

// ------------------------------------------------------------------------------------------------
// errors
// ------------------------------------------------------------------------------------------------
void set_error(const char *fmt, ...);
int cuda_fail(cudaError_t e, const char *what, const char *file, int line);

#define GPL_CUDA(expr)                                                           \
    do {                                                                         \
        cudaError_t e__ = (expr);                                                \
        if (e__ != cudaSuccess) return gpl::cuda_fail(e__, #expr, __FILE__, __LINE__); \
    } while (0)

#define GPL_TRY(expr)             \
    do {                          \
        int rc__ = (expr);        \
        if (rc__ != GPL_OK) return rc__; \
    } while (0)

#define GPL_REQUIRE(cond, code, ...) \
    do {                             \
        if (!(cond)) {               \
            gpl::set_error(__VA_ARGS__); \
            return (code);           \
        }                            \
    } while (0)

constexpr int kSMs = 132;  // H100 SXM

static inline int64_t ceil_div(int64_t a, int64_t b) { return (a + b - 1) / b; }

// CTAs for one warp per row, at most ctas_per_sm per SM (the warps stride over the remaining rows)
static int warp_grid(int64_t rows, int warps_per_cta, int ctas_per_sm = 16) {
    int64_t want = ceil_div(rows, warps_per_cta);
    return (int)std::max<int64_t>(1, std::min<int64_t>(want, (int64_t)kSMs * ctas_per_sm));
}
// CTAs of 256 threads for one thread per item, at most 16 per SM (the threads stride over the remaining items)
static int flat_grid(int64_t n) { return (int)std::max<int64_t>(1, std::min<int64_t>(ceil_div(n, 256), (int64_t)kSMs * 16)); }

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

// geometry type tests of the host side
static inline bool is_point(int t) { return t == GPL_POINT || t == GPL_MULTIPOINT; }
static inline bool is_line(int t) { return t == GPL_LINESTRING || t == GPL_MULTILINESTRING; }
static inline bool is_area(int t) { return t == GPL_POLYGON || t == GPL_MULTIPOLYGON; }
static inline bool is_multi(int t) { return t == GPL_MULTIPOINT || t == GPL_MULTILINESTRING || t == GPL_MULTIPOLYGON; }
static inline bool known_type(int t) { return is_point(t) || is_line(t) || is_area(t); }  // the six OGC types

}  // namespace gpl

// ------------------------------------------------------------------------------------------------
// context: device, stream, caching allocator (grow-only free lists by size class so that steady
// state ops never call cudaMalloc), launch counter.
// ------------------------------------------------------------------------------------------------
struct gpl_ctx {
    int device = 0;
    cudaStream_t stream = nullptr;
    bool owns_stream = false;
    cudaStream_t copy_in = nullptr, copy_out = nullptr;  // e2e pipeline streams (lazily created)
    int64_t launches = 0;
    std::mutex mu;
    std::multimap<size_t, void *> free_blocks;  // size -> ptr
    std::map<void *, size_t> live;              // ptr -> size (blocks handed out)
    size_t bytes_reserved = 0;
    size_t l2_persist_max = 0, l2_window_max = 0;  // device limits, read once at creation
    const void *l2_pinned = nullptr;               // slab currently covered by the access-policy window
    size_t l2_prev_limit = 0, l2_cur_limit = 0;    // cudaLimitPersistingL2CacheSize before the first pin / now
    bool l2_limit_saved = false;
    // gpl_ctx_kernel_timing: event pairs around the launches of the streaming join kernel (a measurement aid)
    bool kt_on = false;
    std::vector<cudaEvent_t> kt_events;  // pairs
    size_t kt_used = 0;                  // events handed out since the last read
    bool kernel_timing_pair(cudaEvent_t *a, cudaEvent_t *b);

    int alloc(size_t bytes, void **out);
    void release(void *p);
    void trim();
};

namespace gpl {

// RAII scratch buffer from the context's cache.
template <typename T>
struct Scratch {
    gpl_ctx *ctx = nullptr;
    T *p = nullptr;
    Scratch() = default;
    Scratch(const Scratch &) = delete;
    Scratch &operator=(const Scratch &) = delete;
    ~Scratch() { reset(); }
    int get(gpl_ctx *c, size_t n) {
        reset();
        ctx = c;
        void *q = nullptr;
        int rc = c->alloc((n ? n : 1) * sizeof(T), &q);
        p = static_cast<T *>(q);
        return rc;
    }
    void reset() {
        if (p && ctx) ctx->release(p);
        p = nullptr;
    }
    T *take() {
        T *q = p;
        p = nullptr;
        return q;
    }
};

}  // namespace gpl

// ------------------------------------------------------------------------------------------------
// device-resident GeoArrow array: interleaved double2 coords, int64 offsets, LSB validity bitmap.
// ------------------------------------------------------------------------------------------------
struct gpl_array {
    gpl_ctx *ctx = nullptr;
    int32_t type = GPL_MISSING;
    int64_t n_geoms = 0, n_parts = 0, n_rings = 0, n_coords = 0;
    const double *xy = nullptr;
    const int64_t *geom_off = nullptr, *part_off = nullptr, *ring_off = nullptr;
    const uint8_t *validity = nullptr;
    // ownership flags: owned buffers go back to ctx's cache on free
    bool own_xy = false, own_geom = false, own_part = false, own_ring = false, own_valid = false;
    // shared buffers: an output that shares offsets/validity with its input keeps the input alive
    // by reference count rather than by copy (affine_transform only rewrites coords).
    gpl_array *parent = nullptr;
    int refcount = 1;
};

// result of a join (gpl_spatial_join, gpl_overlay_area_join, gpl_overlay_join, gpl_predicate_join,
// gpl_contains_join_pairs_array, the nearest, distance-within and great-circle pair joins):
// (lhs, rhs) row pairs, sorted by (lhs, rhs), no pair twice
struct gpl_pairs {
    gpl_ctx *ctx = nullptr;
    uint64_t *lhs = nullptr, *rhs = nullptr;  // device
    double *dist = nullptr;                   // device, the distance of each pair (with_distance joins) or its area (gpl_overlay_area_join)
    bool with_dist = false;                   // dist was asked for (it stays NULL when the list is empty)
    int64_t n = 0;
};

namespace gpl {

// An owned pair list: freed when it goes out of scope unless it is released to the caller.
using Pairs = std::unique_ptr<gpl_pairs, void (*)(gpl_pairs *)>;
// A list of n pairs of ctx with lhs / rhs (and, with_dist, dist) allocated but not written.
static int pairs_new(gpl_ctx *ctx, int64_t n, bool with_dist, Pairs &out) {
    out.reset(new gpl_pairs());
    out->ctx = ctx;
    out->with_dist = with_dist;
    if (n == 0) return GPL_OK;
    out->n = n;
    void *p = nullptr;
    GPL_TRY(ctx->alloc(sizeof(uint64_t) * (size_t)n, &p));
    out->lhs = (uint64_t *)p;
    GPL_TRY(ctx->alloc(sizeof(uint64_t) * (size_t)n, &p));
    out->rhs = (uint64_t *)p;
    if (with_dist) {
        GPL_TRY(ctx->alloc(sizeof(double) * (size_t)n, &p));
        out->dist = (double *)p;
    }
    return GPL_OK;
}

gpl_array *array_new(gpl_ctx *ctx, int32_t type);
void array_retain(gpl_array *a);

// the two columns of a row-wise binary op have one row each per output row
static int require_same_length(const gpl_array *a, const gpl_array *b, const char *who) {
    GPL_REQUIRE(a->n_geoms == b->n_geoms, GPL_ERR_LENGTH_MISMATCH, "%s: lengths differ (%lld vs %lld)", who, (long long)a->n_geoms,
                (long long)b->n_geoms);
    return GPL_OK;
}

// ------------------------------------------------------------------------------------------------
// launch helper: counts launches for bench.py's gpu_launches and checks the launch error.
// ------------------------------------------------------------------------------------------------
#define GPL_LAUNCH(ctx, kernel, grid, block, smem, ...)                           \
    do {                                                                          \
        kernel<<<(grid), (block), (smem), (ctx)->stream>>>(__VA_ARGS__);          \
        (ctx)->launches++;                                                        \
        GPL_CUDA(cudaGetLastError());                                             \
    } while (0)

}  // namespace gpl

// ------------------------------------------------------------------------------------------------
// device code
// ------------------------------------------------------------------------------------------------
#ifdef __CUDACC__
namespace gpl {

// hypot as glibc >= 2.35 computes it (sysdeps/ieee754/dbl-64/e_hypot.c, the kernel without FMA: one sqrt and
// one correction step) — Rust's f64::hypot is the platform libm's.  CUDA's own hypot differs from it in the
// last bit often enough to flip exact ties (simplify's `distance >= farthest`, `> epsilon` on lattice input);
// this one agreed with glibc 2.39 on 2e7 random and lattice inputs bit for bit.  The exponent rescaling glibc
// applies above 2^511 / below 2^-459 is omitted (coordinates do not live there).
__device__ __forceinline__ double gpl_hypot(double x, double y) {
    x = fabs(x), y = fabs(y);
    if (!(x <= 1.7976931348623157e308 && y <= 1.7976931348623157e308))  // inf or nan
        return (x > 1.7976931348623157e308 || y > 1.7976931348623157e308) ? __longlong_as_double(0x7ff0000000000000LL) : x + y;
    const double ax = x < y ? y : x, ay = x < y ? x : y;
    if (ax >= ay * 18014398509481984.0) return ax + ay;  // ay / 2^-54 <= ax
    double h = sqrt(ax * ax + ay * ay), t1, t2;
    if (h <= 2.0 * ay) {
        const double delta = h - ay;
        t1 = ax * (2.0 * delta - ax);
        t2 = (delta - 2.0 * (ax - ay)) * delta;
    } else {
        const double delta = h - ax;
        t1 = 2.0 * delta * (ax - 2.0 * ay);
        t2 = (4.0 * delta - ay) * ay + delta * delta;
    }
    h -= (t1 + t2) / (2.0 * h);
    return h;
}
__device__ __forceinline__ double pt_dist(double2 a, double2 b) { return gpl_hypot(b.x - a.x, b.y - a.y); }
// geo-types private_utils::line_segment_distance (recalled): distance from p to the SEGMENT s-e
__device__ __forceinline__ double line_segment_distance(double2 p, double2 s, double2 e) {
    if (s.x == e.x && s.y == e.y) return pt_dist(p, s);
    double dx = e.x - s.x, dy = e.y - s.y;
    double d2 = dx * dx + dy * dy;
    double r = ((p.x - s.x) * dx + (p.y - s.y) * dy) / d2;
    if (r <= 0.0) return pt_dist(p, s);
    if (r >= 1.0) return pt_dist(p, e);
    double sv = ((s.y - p.y) * dx - (s.x - p.x) * dy) / d2;
    return fabs(sv) * gpl_hypot(dx, dy);
}

__device__ __forceinline__ double2 ld2(const double *xy, int64_t i) {
    return reinterpret_cast<const double2 *>(xy)[i];
}
// streaming (read-once) load: bypass L1 allocation so the polygon-side tables keep the cache
__device__ __forceinline__ double2 ld2_stream(const double *xy, int64_t i) {
    return __ldcs(reinterpret_cast<const double2 *>(xy) + i);
}
__device__ __forceinline__ bool bit_get(const uint8_t *bm, int64_t i) {
    return bm == nullptr || ((bm[i >> 3] >> (i & 7)) & 1);
}

// ---- robust orient2d (Shewchuk adaptive, what robust 1.1.0 implements; geo's RobustKernel) ------
// Only the sign is consumed.  Stage A (the fast filter) is inline; the adaptive stages B-D live in
// a non-inlined function because they are reached by ~1e-9 of random inputs and would otherwise
// cost registers in every caller.  All arithmetic here relies on -fmad=false.
constexpr double kEps = 1.1102230246251565e-16;
constexpr double kCcwA = (3.0 + 16.0 * kEps) * kEps;

constexpr double kSplitter = 134217729.0;  // 2^27 + 1
constexpr double kResultErr = (3.0 + 8.0 * kEps) * kEps;
constexpr double kCcwB = (2.0 + 12.0 * kEps) * kEps;
constexpr double kCcwC = (9.0 + 64.0 * kEps) * kEps * kEps;

__device__ __forceinline__ void two_sum(double a, double b, double &x, double &y) {
    x = a + b;
    double bvirt = x - a;
    double avirt = x - bvirt;
    double bround = b - bvirt;
    double around = a - avirt;
    y = around + bround;
}
__device__ __forceinline__ void fast_two_sum(double a, double b, double &x, double &y) {
    x = a + b;
    double bvirt = x - a;
    y = b - bvirt;
}
__device__ __forceinline__ double two_diff_tail(double a, double b, double x) {
    double bvirt = a - x;
    double avirt = x + bvirt;
    double bround = bvirt - b;
    double around = a - avirt;
    return around + bround;
}
__device__ __forceinline__ void two_diff(double a, double b, double &x, double &y) {
    x = a - b;
    y = two_diff_tail(a, b, x);
}
__device__ __forceinline__ void split(double a, double &hi, double &lo) {
    double c = kSplitter * a;
    double abig = c - a;
    hi = c - abig;
    lo = a - hi;
}
__device__ __forceinline__ void two_product(double a, double b, double &x, double &y) {
    x = a * b;
    double ahi, alo, bhi, blo;
    split(a, ahi, alo);
    split(b, bhi, blo);
    double err1 = x - (ahi * bhi);
    double err2 = err1 - (alo * bhi);
    double err3 = err2 - (ahi * blo);
    y = (alo * blo) - err3;
}
__device__ __forceinline__ void two_two_diff(double a1, double a0, double b1, double b0, double *x) {
    double i, j, z;
    two_diff(a0, b0, i, x[0]);
    two_sum(a1, i, j, z);
    two_diff(z, b1, i, x[1]);
    two_sum(j, i, x[3], x[2]);
}
__device__ __forceinline__ int fast_expansion_sum_zeroelim(int elen, const double *e, int flen, const double *f,
                                                           double *h) {
    double Q, Qnew, hh;
    int ei = 0, fi = 0, hi = 0;
    double enow = e[0], fnow = f[0];
    if ((fnow > enow) == (fnow > -enow)) {
        Q = enow;
        ++ei;
        enow = ei < elen ? e[ei] : 0.0;
    } else {
        Q = fnow;
        ++fi;
        fnow = fi < flen ? f[fi] : 0.0;
    }
    if ((ei < elen) && (fi < flen)) {
        if ((fnow > enow) == (fnow > -enow)) {
            fast_two_sum(enow, Q, Qnew, hh);
            ++ei;
            enow = ei < elen ? e[ei] : 0.0;
        } else {
            fast_two_sum(fnow, Q, Qnew, hh);
            ++fi;
            fnow = fi < flen ? f[fi] : 0.0;
        }
        Q = Qnew;
        if (hh != 0.0) h[hi++] = hh;
        while ((ei < elen) && (fi < flen)) {
            if ((fnow > enow) == (fnow > -enow)) {
                two_sum(Q, enow, Qnew, hh);
                ++ei;
                enow = ei < elen ? e[ei] : 0.0;
            } else {
                two_sum(Q, fnow, Qnew, hh);
                ++fi;
                fnow = fi < flen ? f[fi] : 0.0;
            }
            Q = Qnew;
            if (hh != 0.0) h[hi++] = hh;
        }
    }
    while (ei < elen) {
        two_sum(Q, enow, Qnew, hh);
        ++ei;
        enow = ei < elen ? e[ei] : 0.0;
        Q = Qnew;
        if (hh != 0.0) h[hi++] = hh;
    }
    while (fi < flen) {
        two_sum(Q, fnow, Qnew, hh);
        ++fi;
        fnow = fi < flen ? f[fi] : 0.0;
        Q = Qnew;
        if (hh != 0.0) h[hi++] = hh;
    }
    if ((Q != 0.0) || (hi == 0)) h[hi++] = Q;
    return hi;
}
// h = b * e exactly (at most 2 elen terms, zeros eliminated, at least one term)
__device__ __forceinline__ int scale_expansion_zeroelim(int elen, const double *e, double b, double *h) {
    double Q, sum, hh, p1, p0;
    int hi = 0;
    two_product(e[0], b, Q, hh);
    if (hh != 0.0) h[hi++] = hh;
    for (int ei = 1; ei < elen; ++ei) {
        two_product(e[ei], b, p1, p0);
        two_sum(Q, p0, sum, hh);
        if (hh != 0.0) h[hi++] = hh;
        fast_two_sum(p1, sum, Q, hh);
        if (hh != 0.0) h[hi++] = hh;
    }
    if ((Q != 0.0) || (hi == 0)) h[hi++] = Q;
    return hi;
}

// stages B, C, D of the adaptive predicate: exact sign whenever the filter cannot decide
static __device__ __noinline__ double orient2d_adapt(double ax, double ay, double bx, double by, double cx, double cy,
                                                     double detsum) {
    double acx = ax - cx, bcx = bx - cx, acy = ay - cy, bcy = by - cy;
    double detleft, detlefttail, detright, detrighttail;
    double B[4], u[4], C1[8], C2[12], D[16];
    two_product(acx, bcy, detleft, detlefttail);
    two_product(acy, bcx, detright, detrighttail);
    two_two_diff(detleft, detlefttail, detright, detrighttail, B);
    double det = B[0] + B[1] + B[2] + B[3];
    double errbound = kCcwB * detsum;
    if ((det >= errbound) || (-det >= errbound)) return det;

    double acxtail = two_diff_tail(ax, cx, acx);
    double bcxtail = two_diff_tail(bx, cx, bcx);
    double acytail = two_diff_tail(ay, cy, acy);
    double bcytail = two_diff_tail(by, cy, bcy);
    if ((acxtail == 0.0) && (acytail == 0.0) && (bcxtail == 0.0) && (bcytail == 0.0)) return det;

    errbound = kCcwC * detsum + kResultErr * fabs(det);
    det += (acx * bcytail + bcy * acxtail) - (acy * bcxtail + bcx * acytail);
    if ((det >= errbound) || (-det >= errbound)) return det;

    double s1, s0, t1, t0;
    two_product(acxtail, bcy, s1, s0);
    two_product(acytail, bcx, t1, t0);
    two_two_diff(s1, s0, t1, t0, u);
    int c1len = fast_expansion_sum_zeroelim(4, B, 4, u, C1);

    two_product(acx, bcytail, s1, s0);
    two_product(acy, bcxtail, t1, t0);
    two_two_diff(s1, s0, t1, t0, u);
    int c2len = fast_expansion_sum_zeroelim(c1len, C1, 4, u, C2);

    two_product(acxtail, bcytail, s1, s0);
    two_product(acytail, bcxtail, t1, t0);
    two_two_diff(s1, s0, t1, t0, u);
    int dlen = fast_expansion_sum_zeroelim(c2len, C2, 4, u, D);
    return D[dlen - 1];
}

// returns a value whose SIGN is exact: >0 counter-clockwise, <0 clockwise, 0 collinear
__device__ __forceinline__ double orient2d(double ax, double ay, double bx, double by, double cx, double cy) {
    double detleft = (ax - cx) * (by - cy);
    double detright = (ay - cy) * (bx - cx);
    double det = detleft - detright;
    double detsum;
    if (detleft > 0.0) {
        if (detright <= 0.0) return det;
        detsum = detleft + detright;
    } else if (detleft < 0.0) {
        if (detright >= 0.0) return det;
        detsum = -detleft - detright;
    } else {
        return det;
    }
    double errbound = kCcwA * detsum;
    if ((det >= errbound) || (-det >= errbound)) return det;
    return orient2d_adapt(ax, ay, bx, by, cx, cy, detsum);
}
__device__ __forceinline__ int orient_sign(double2 a, double2 b, double2 c) {
    double d = orient2d(a.x, a.y, b.x, b.y, c.x, c.y);
    return (d > 0.0) - (d < 0.0);
}
__device__ __forceinline__ int cmpd(double a, double b) { return (a > b) - (a < b); }
__device__ __forceinline__ int sgnd(double a) { return (a > 0.0) - (a < 0.0); }
__device__ __forceinline__ bool value_in_between(double v, double b1, double b2) {
    return (b1 < b2) ? (v >= b1 && v <= b2) : (v >= b2 && v <= b1);
}
__device__ __forceinline__ bool point_in_rect(double2 v, double2 b1, double2 b2) {
    return value_in_between(v.x, b1.x, b2.x) && value_in_between(v.y, b1.y, b2.y);
}

// lane src's value, to every lane
__device__ __forceinline__ double2 bcast2(double2 v, int src) {
    return make_double2(__shfl_sync(0xffffffffu, v.x, src), __shfl_sync(0xffffffffu, v.y, src));
}
// warp reductions on doubles
__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ double warp_min(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmin(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}
__device__ __forceinline__ double warp_max(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmax(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}

}  // namespace gpl
#endif  // __CUDACC__
