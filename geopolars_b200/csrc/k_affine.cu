// k_affine.cu — GeoSeries::affine_transform / translate / scale / rotate / skew
// (reference: geopolars/geopolars-geo/src/geoseries.rs:11-12, 93, 107, 139, 174; arithmetic = geo 0.27
// AffineTransform::apply, recalled: x' = a*x + b*y + xoff ; y' = d*x + e*y + yoff, each product and sum
// separately rounded — this file is compiled with -fmad=false).
//
// Roofline: pure streaming, 16 B read + 16 B written per coordinate, bound by HBM.
//   * fixed matrix: grid-stride over double2 with 4 independent 128-bit loads in flight per thread
//     (MLP), streaming cache hints (.cs) because nothing is re-read; grid = 132 SMs x 8 CTAs.
//   * per-geometry origin (rotate/scale/skew about centroid / bbox centre): the 6 coefficients are
//     derived per geometry from a [n_geoms][2] origin table; one warp per geometry streams that
//     geometry's contiguous coordinate range (coalesced 512 B per warp iteration).
#include <math.h>

#include "common.cuh"
#include "output.cuh"

namespace gpl {

struct Affine {
    double a, b, xoff, d, e, yoff;
};

__device__ __forceinline__ double2 apply(const Affine &m, double2 p) {
    double2 r;
    r.x = m.a * p.x + m.b * p.y + m.xoff;
    r.y = m.d * p.x + m.e * p.y + m.yoff;
    return r;
}

__global__ void __launch_bounds__(256) k_affine(const double2 *__restrict__ in, double2 *__restrict__ out, int64_t n,
                                                Affine m) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    // 4-way unrolled: four independent LDG.128 in flight per thread before the first use
    for (; i + 3 * stride < n; i += 4 * stride) {
        double2 p0 = __ldcs(in + i);
        double2 p1 = __ldcs(in + i + stride);
        double2 p2 = __ldcs(in + i + 2 * stride);
        double2 p3 = __ldcs(in + i + 3 * stride);
        __stcs(out + i, apply(m, p0));
        __stcs(out + i + stride, apply(m, p1));
        __stcs(out + i + 2 * stride, apply(m, p2));
        __stcs(out + i + 3 * stride, apply(m, p3));
    }
    for (; i < n; i += stride) __stcs(out + i, apply(m, __ldcs(in + i)));
}

// kind: 0 scale(p0=xfact,p1=yfact) 1 rotate(p0=cos,p1=sin) 2 skew(p0=tan xs,p1=tan ys)
__device__ __forceinline__ Affine origin_matrix(int kind, double p0, double p1, double x0, double y0) {
    Affine m;
    if (kind == 0) {  // geo AffineTransform::scale: (fx, 0, x0 - x0*fx, 0, fy, y0 - y0*fy)
        m.a = p0, m.b = 0.0, m.xoff = x0 - x0 * p0;
        m.d = 0.0, m.e = p1, m.yoff = y0 - y0 * p1;
    } else if (kind == 1) {  // rotate: (cos, -sin, x0 - x0*cos + y0*sin, sin, cos, y0 - x0*sin - y0*cos)
        m.a = p0, m.b = -p1, m.xoff = x0 - x0 * p0 + y0 * p1;
        m.d = p1, m.e = p0, m.yoff = y0 - x0 * p1 - y0 * p0;
    } else {  // skew: (1, tan xs, -y0*tan xs, tan ys, 1, -x0*tan ys)   (geoseries.rs:129-138)
        m.a = 1.0, m.b = p0, m.xoff = -y0 * p0;
        m.d = p1, m.e = 1.0, m.yoff = -x0 * p1;
    }
    return m;
}

// coordinate range [c0,c1) of geometry g for any nesting
__device__ __forceinline__ void geom_coord_range(int type, int64_t g, const int64_t *geom_off, const int64_t *part_off,
                                                 const int64_t *ring_off, int64_t &c0, int64_t &c1) {
    switch (type) {
    case GPL_POINT:
        c0 = g, c1 = g + 1;
        break;
    case GPL_LINESTRING:
    case GPL_MULTIPOINT:
        c0 = geom_off[g], c1 = geom_off[g + 1];
        break;
    case GPL_POLYGON:
    case GPL_MULTILINESTRING:
        c0 = ring_off[geom_off[g]], c1 = ring_off[geom_off[g + 1]];
        break;
    default:  // MULTIPOLYGON
        c0 = ring_off[part_off[geom_off[g]]], c1 = ring_off[part_off[geom_off[g + 1]]];
        break;
    }
}

__global__ void __launch_bounds__(256) k_affine_per_geom(int type, int64_t n_geoms, const double2 *__restrict__ in,
                                                         const int64_t *__restrict__ geom_off,
                                                         const int64_t *__restrict__ part_off,
                                                         const int64_t *__restrict__ ring_off,
                                                         const double2 *__restrict__ origin,  // per geometry, NaN = none
                                                         int kind, double p0, double p1, double2 *__restrict__ out) {
    const int lane = threadIdx.x & 31;
    int64_t warp = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
    const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t g = warp; g < n_geoms; g += nwarps) {
        int64_t c0, c1;
        geom_coord_range(type, g, geom_off, part_off, ring_off, c0, c1);
        double2 o = origin[g];
        Affine m = origin_matrix(kind, p0, p1, o.x, o.y);
        if (isnan(o.x) || isnan(o.y)) m = Affine{1.0, 0.0, 0.0, 0.0, 1.0, 0.0};  // no centroid/bbox: unchanged
        for (int64_t c = c0 + lane; c < c1; c += 32) __stcs(out + c, apply(m, __ldcs(in + c)));
    }
}

static int make_output_like(gpl_ctx *ctx, const gpl_array *in, gpl_array **out, double **xy_out) {
    Scratch<double> xy;
    GPL_TRY(xy.get(ctx, (size_t)in->n_coords * 2));
    gpl_array *o = array_new(ctx, in->type);
    o->n_geoms = in->n_geoms, o->n_parts = in->n_parts, o->n_rings = in->n_rings, o->n_coords = in->n_coords;
    *xy_out = xy.p;
    o->xy = xy.take();
    o->own_xy = true;
    // offsets and validity are unchanged by an affine map: share them, keep the input alive
    o->geom_off = in->geom_off, o->part_off = in->part_off, o->ring_off = in->ring_off, o->validity = in->validity;
    o->parent = const_cast<gpl_array *>(in);
    array_retain(o->parent);
    *out = o;
    return GPL_OK;
}

int affine_fixed(gpl_ctx *ctx, const gpl_array *in, Affine m, gpl_array **out) {
    GPL_REQUIRE(ctx && in && out, GPL_ERR_INVALID_ARG, "affine_transform: NULL argument");
    GPL_CUDA(cudaSetDevice(ctx->device));
    double *oxy = nullptr;
    GPL_TRY(make_output_like(ctx, in, out, &oxy));
    if (in->n_coords > 0) {
        int64_t want = ceil_div(in->n_coords, 256 * 4);
        int grid = (int)std::max<int64_t>(1, std::min<int64_t>(want, kSMs * 8));
        GPL_LAUNCH(ctx, k_affine, grid, 256, 0, reinterpret_cast<const double2 *>(in->xy),
                   reinterpret_cast<double2 *>(oxy), in->n_coords, m);
    }
    return GPL_OK;
}

// defined in k_measure.cu: per-geometry origin table (centroid or bbox centre)

int affine_about_origin(gpl_ctx *ctx, const gpl_array *in, int kind, double p0, double p1, int origin, double ox,
                        double oy, gpl_array **out) {
    GPL_REQUIRE(ctx && in && out, GPL_ERR_INVALID_ARG, "NULL argument");
    GPL_REQUIRE(origin == GPL_ORIGIN_CENTROID || origin == GPL_ORIGIN_CENTER || origin == GPL_ORIGIN_POINT,
                GPL_ERR_INVALID_ARG, "Invalid argument: origin must be centroid, center or a point");
    GPL_CUDA(cudaSetDevice(ctx->device));
    if (origin == GPL_ORIGIN_POINT) {
        // host evaluation of the same formulas (no FMA on the host either: see Makefile -ffp-contract=off)
        Affine m;
        if (kind == 0) {
            m.a = p0, m.b = 0.0, m.xoff = ox - ox * p0, m.d = 0.0, m.e = p1, m.yoff = oy - oy * p1;
        } else if (kind == 1) {
            m.a = p0, m.b = -p1, m.xoff = ox - ox * p0 + oy * p1, m.d = p1, m.e = p0, m.yoff = oy - ox * p1 - oy * p0;
        } else {
            m.a = 1.0, m.b = p0, m.xoff = -oy * p0, m.d = p1, m.e = 1.0, m.yoff = -ox * p1;
        }
        return affine_fixed(ctx, in, m, out);
    }
    Scratch<double2> org;
    GPL_TRY(org.get(ctx, (size_t)in->n_geoms));
    GPL_TRY(origin_table(ctx, in, origin, org.p));
    double *oxy = nullptr;
    GPL_TRY(make_output_like(ctx, in, out, &oxy));
    if (in->n_geoms > 0 && in->n_coords > 0) {
        int64_t want = ceil_div(in->n_geoms, 8);
        int grid = (int)std::max<int64_t>(1, std::min<int64_t>(want, kSMs * 8));
        GPL_LAUNCH(ctx, k_affine_per_geom, grid, 256, 0, in->type, in->n_geoms, reinterpret_cast<const double2 *>(in->xy),
                   in->geom_off, in->part_off, in->ring_off, org.p, kind, p0, p1, reinterpret_cast<double2 *>(oxy));
    }
    return GPL_OK;
}

}  // namespace gpl

using namespace gpl;

extern "C" int gpl_affine_transform(gpl_ctx *ctx, const gpl_array *in, double a, double b, double xoff, double d,
                                    double e, double yoff, gpl_array **out) {
    Affine m{a, b, xoff, d, e, yoff};
    return affine_fixed(ctx, in, m, out);
}
extern "C" int gpl_translate(gpl_ctx *ctx, const gpl_array *in, double xoff, double yoff, gpl_array **out) {
    Affine m{1.0, 0.0, xoff, 0.0, 1.0, yoff};  // geo AffineTransform::translate
    return affine_fixed(ctx, in, m, out);
}
extern "C" int gpl_scale(gpl_ctx *ctx, const gpl_array *in, double xfact, double yfact, int origin, double ox,
                         double oy, gpl_array **out) {
    return affine_about_origin(ctx, in, 0, xfact, yfact, origin, ox, oy, out);
}
extern "C" int gpl_rotate(gpl_ctx *ctx, const gpl_array *in, double angle_deg, int origin, double ox, double oy,
                          gpl_array **out) {
    // geo: let (sin, cos) = degrees.to_radians().sin_cos(); to_radians = deg * (PI / 180)
    double rad = angle_deg * (3.14159265358979323846 / 180.0);
    return affine_about_origin(ctx, in, 1, cos(rad), sin(rad), origin, ox, oy, out);
}
extern "C" int gpl_skew(gpl_ctx *ctx, const gpl_array *in, double xs_deg, double ys_deg, int origin, double ox,
                        double oy, gpl_array **out) {
    double tx = tan(xs_deg * (3.14159265358979323846 / 180.0));
    double ty = tan(ys_deg * (3.14159265358979323846 / 180.0));
    // geo AffineTransform::skew zeroes tangents below 2.5e-16 (a check it took from shapely)
    if (fabs(tx) < 2.5e-16) tx = 0.0;
    if (fabs(ty) < 2.5e-16) ty = 0.0;
    return affine_about_origin(ctx, in, 2, tx, ty, origin, ox, oy, out);
}
