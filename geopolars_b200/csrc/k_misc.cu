// k_misc.cu — the secondary GeoSeries ops that are offset relabelling or trivial maps once the data is
// GeoArrow-resident: geom_type (geoseries.rs:60-73), is_empty (:75-76), is_ring (:78-83), x / y (:176-180),
// exterior (:43-47), explode (:49-50).  SURVEY.md §8 row a9.
#include <math.h>

#include "common.cuh"
#include "output.cuh"
#include "scan.cuh"

namespace gpl {

__global__ void k_geom_type(int type, int64_t n, const uint8_t *__restrict__ validity, int8_t *__restrict__ out) {
    int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i < n) out[i] = bit_get(validity, i) ? (int8_t)type : (int8_t)GPL_MISSING;
}

// geo HasDimensions::is_empty; a GeoArrow (NaN, NaN) point is the empty point
__global__ void k_is_empty(int type, int64_t n, const double2 *__restrict__ xy, const int64_t *__restrict__ geom_off,
                           const int64_t *__restrict__ part_off, const int64_t *__restrict__ ring_off, uint8_t *__restrict__ out) {
    int64_t g = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (g >= n) return;
    bool empty = true;
    switch (type) {
    case GPL_POINT: {
        double2 p = xy[g];
        empty = isnan(p.x) && isnan(p.y);
        break;
    }
    case GPL_LINESTRING:
    case GPL_MULTIPOINT:
        empty = geom_off[g + 1] == geom_off[g];
        break;
    case GPL_MULTILINESTRING:
        for (int64_t l = geom_off[g]; l < geom_off[g + 1] && empty; ++l) empty = ring_off[l + 1] == ring_off[l];
        break;
    case GPL_POLYGON:
        empty = geom_off[g + 1] == geom_off[g] || ring_off[geom_off[g] + 1] == ring_off[geom_off[g]];
        break;
    case GPL_MULTIPOLYGON:
        for (int64_t p = geom_off[g]; p < geom_off[g + 1] && empty; ++p)
            empty = part_off[p + 1] == part_off[p] || ring_off[part_off[p] + 1] == ring_off[part_off[p]];
        break;
    default:
        break;
    }
    out[g] = empty ? 1 : 0;
}

// LineString::is_closed (first == last; an empty linestring compares None == None => true); other types false
__global__ void k_is_ring(int type, int64_t n, const double2 *__restrict__ xy, const int64_t *__restrict__ geom_off,
                          uint8_t *__restrict__ out) {
    int64_t g = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (g >= n) return;
    bool r = false;
    if (type == GPL_LINESTRING) {
        int64_t c0 = geom_off[g], c1 = geom_off[g + 1];
        if (c1 == c0) {
            r = true;
        } else {
            double2 a = xy[c0], b = xy[c1 - 1];
            r = a.x == b.x && a.y == b.y;
        }
    }
    out[g] = r ? 1 : 0;
}

__global__ void k_component(const double2 *__restrict__ xy, int64_t n, int comp, double *__restrict__ out) {
    int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i < n) {
        double2 p = xy[i];
        out[i] = comp == 0 ? p.x : p.y;
    }
}

__global__ void k_exterior_len(int64_t n, const int64_t *__restrict__ geom_off, const int64_t *__restrict__ ring_off,
                               int64_t *__restrict__ len) {
    int64_t g = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (g >= n) return;
    int64_t r0 = geom_off[g], r1 = geom_off[g + 1];
    len[g] = r1 > r0 ? ring_off[r0 + 1] - ring_off[r0] : 0;
}
__global__ void __launch_bounds__(256) k_exterior_copy(int64_t n, const double2 *__restrict__ xy, const int64_t *__restrict__ geom_off,
                                                       const int64_t *__restrict__ ring_off, const int64_t *__restrict__ out_off,
                                                       double2 *__restrict__ out) {
    const int lane = threadIdx.x & 31;
    int64_t warp = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
    const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t g = warp; g < n; g += nwarps) {
        int64_t r0 = geom_off[g], r1 = geom_off[g + 1];
        if (r1 <= r0) continue;
        int64_t c0 = ring_off[r0], c1 = ring_off[r0 + 1], o = out_off[g];
        for (int64_t c = c0 + lane; c < c1; c += 32) out[o + (c - c0)] = xy[c];
    }
}

}  // namespace gpl

using namespace gpl;

extern "C" int gpl_geom_type(gpl_ctx *ctx, const gpl_array *in, int8_t *out, int mem) {
    GPL_REQUIRE(ctx && in && out, GPL_ERR_INVALID_ARG, "gpl_geom_type: NULL argument");
    GPL_TRY(check_mem(mem, "gpl_geom_type"));
    GPL_CUDA(cudaSetDevice(ctx->device));
    int64_t n = in->n_geoms;
    if (n == 0) return GPL_OK;
    RowOut<int8_t> res;
    GPL_TRY(res.get(ctx, out, n, mem));
    GPL_LAUNCH(ctx, k_geom_type, (int)ceil_div(n, 256), 256, 0, in->type, n, in->validity, res.p);
    return res.deliver(ctx);
}

extern "C" int gpl_is_empty(gpl_ctx *ctx, const gpl_array *in, uint8_t *out_bitmap, int mem) {
    GPL_REQUIRE(ctx && in && out_bitmap, GPL_ERR_INVALID_ARG, "gpl_is_empty: NULL argument");
    GPL_TRY(check_mem(mem, "gpl_is_empty"));
    GPL_CUDA(cudaSetDevice(ctx->device));
    int64_t n = in->n_geoms;
    if (n == 0) return GPL_OK;
    Scratch<uint8_t> bytes;
    GPL_TRY(bytes.get(ctx, (size_t)n));
    GPL_LAUNCH(ctx, k_is_empty, (int)ceil_div(n, 256), 256, 0, in->type, n, reinterpret_cast<const double2 *>(in->xy), in->geom_off,
               in->part_off, in->ring_off, bytes.p);
    return finish_bitmap(ctx, bytes.p, n, out_bitmap, mem);
}

extern "C" int gpl_is_ring(gpl_ctx *ctx, const gpl_array *in, uint8_t *out_bitmap, int mem) {
    GPL_REQUIRE(ctx && in && out_bitmap, GPL_ERR_INVALID_ARG, "gpl_is_ring: NULL argument");
    GPL_TRY(check_mem(mem, "gpl_is_ring"));
    GPL_CUDA(cudaSetDevice(ctx->device));
    int64_t n = in->n_geoms;
    if (n == 0) return GPL_OK;
    Scratch<uint8_t> bytes;
    GPL_TRY(bytes.get(ctx, (size_t)n));
    GPL_LAUNCH(ctx, k_is_ring, (int)ceil_div(n, 256), 256, 0, in->type, n, reinterpret_cast<const double2 *>(in->xy), in->geom_off,
               bytes.p);
    return finish_bitmap(ctx, bytes.p, n, out_bitmap, mem);
}

static int component(gpl_ctx *ctx, const gpl_array *in, int comp, double *out, int mem) {
    GPL_REQUIRE(ctx && in && out, GPL_ERR_INVALID_ARG, "gpl_x/gpl_y: NULL argument");
    GPL_REQUIRE(in->type == GPL_POINT, GPL_ERR_INVALID_TYPE, "Expected Point (found geometry type %d)", in->type);
    GPL_TRY(check_mem(mem, "gpl_x/gpl_y"));
    GPL_CUDA(cudaSetDevice(ctx->device));
    int64_t n = in->n_geoms;
    if (n == 0) return GPL_OK;
    RowOut<double> res;
    GPL_TRY(res.get(ctx, out, n, mem));
    GPL_LAUNCH(ctx, k_component, (int)ceil_div(n, 256), 256, 0, reinterpret_cast<const double2 *>(in->xy), n, comp, res.p);
    return res.deliver(ctx);
}
extern "C" int gpl_x(gpl_ctx *ctx, const gpl_array *in, double *out, int mem) { return component(ctx, in, 0, out, mem); }
extern "C" int gpl_y(gpl_ctx *ctx, const gpl_array *in, double *out, int mem) { return component(ctx, in, 1, out, mem); }

extern "C" int gpl_exterior(gpl_ctx *ctx, const gpl_array *in, gpl_array **out) {
    GPL_REQUIRE(ctx && in && out, GPL_ERR_INVALID_ARG, "gpl_exterior: NULL argument");
    GPL_REQUIRE(in->type == GPL_POLYGON, GPL_ERR_INVALID_TYPE, "Expected Polygon (found geometry type %d)", in->type);
    GPL_CUDA(cudaSetDevice(ctx->device));
    int64_t n = in->n_geoms;
    Scratch<int64_t> len, off, total;
    GPL_TRY(len.get(ctx, (size_t)n + 1));
    GPL_TRY(off.get(ctx, (size_t)n + 1));
    GPL_TRY(total.get(ctx, 1));
    if (n > 0) GPL_LAUNCH(ctx, k_exterior_len, (int)ceil_div(n, 256), 256, 0, n, in->geom_off, in->ring_off, len.p);
    GPL_TRY((exclusive_scan<int64_t, int64_t>(ctx, len.p, n, off.p, total.p)));
    int64_t h_total = 0;
    GPL_CUDA(cudaMemcpyAsync(&h_total, total.p, sizeof(int64_t), cudaMemcpyDeviceToHost, ctx->stream));
    GPL_CUDA(cudaStreamSynchronize(ctx->stream));
    Scratch<double> xy;
    GPL_TRY(xy.get(ctx, (size_t)h_total * 2));
    if (n > 0 && h_total > 0) {
        GPL_LAUNCH(ctx, k_exterior_copy, warp_grid(n, 8, 8), 256, 0, n, reinterpret_cast<const double2 *>(in->xy), in->geom_off, in->ring_off, off.p,
                   reinterpret_cast<double2 *>(xy.p));
    }
    gpl_array *o = array_new(ctx, GPL_LINESTRING);
    o->n_geoms = n, o->n_coords = h_total;
    o->xy = xy.take(), o->own_xy = true;
    o->geom_off = off.take(), o->own_geom = true;
    o->validity = in->validity;  // shared with the input
    o->parent = const_cast<gpl_array *>(in);
    array_retain(o->parent);
    *out = o;
    return GPL_OK;
}

// explode: multi-part -> single-part by relabelling offset levels; zero copies, the input is kept alive
extern "C" int gpl_explode(gpl_ctx *ctx, const gpl_array *in, gpl_array **out) {
    GPL_REQUIRE(ctx && in && out, GPL_ERR_INVALID_ARG, "gpl_explode: NULL argument");
    gpl_array *o = nullptr;
    switch (in->type) {
    case GPL_MULTIPOINT:
        o = array_new(ctx, GPL_POINT);
        o->n_geoms = o->n_coords = in->n_coords;
        o->xy = in->xy;
        break;
    case GPL_MULTILINESTRING:
        o = array_new(ctx, GPL_LINESTRING);
        o->n_geoms = in->n_rings, o->n_coords = in->n_coords;
        o->xy = in->xy, o->geom_off = in->ring_off;
        break;
    case GPL_MULTIPOLYGON:
        o = array_new(ctx, GPL_POLYGON);
        o->n_geoms = in->n_parts, o->n_rings = in->n_rings, o->n_coords = in->n_coords;
        o->xy = in->xy, o->geom_off = in->part_off, o->ring_off = in->ring_off;
        break;
    default:  // already single-part: same buffers, same validity
        o = array_new(ctx, in->type);
        o->n_geoms = in->n_geoms, o->n_rings = in->n_rings, o->n_parts = in->n_parts, o->n_coords = in->n_coords;
        o->xy = in->xy, o->geom_off = in->geom_off, o->part_off = in->part_off, o->ring_off = in->ring_off;
        o->validity = in->validity;
        break;
    }
    o->parent = const_cast<gpl_array *>(in);
    array_retain(o->parent);
    *out = o;
    return GPL_OK;
}
