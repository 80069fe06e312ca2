// k_measure.cu — segmented reductions over rings: area, centroid, envelope, euclidean_length.
// Reference: GeoSeries::area geoseries.rs:14-16, ::centroid :18-21, ::envelope :28-33,
// ::euclidean_length :35-41 (bodies `todo!()` at :188-206; arithmetic = geo 0.27 area.rs / centroid.rs /
// bounding_rect.rs / euclidean_length.rs, recalled — see oracle/geo_oracle.c for the restatement).
//
// Layout/roofline: one warp per geometry; lanes stride over the geometry's segments, so a warp
// iteration reads 512 contiguous bytes (coalesced LDG.128 per lane, the i+1 neighbour comes from L1).
// 16 B of coordinates per segment => HBM-bound; per-ring sums are combined with __shfl_xor butterflies
// so every lane holds the ring result and the (serial, reference-ordered) ring/part state machine is
// executed redundantly without divergence.  Summation order inside a ring is lane-strided then a
// butterfly, not the reference's left-to-right loop: results agree to ~1e-15 relative (tolerance for
// f64 outputs is 1e-9, north_star).
#include <math.h>

#include "common.cuh"
#include "output.cuh"

namespace gpl {

__device__ __forceinline__ double bfly_sum(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// twice the signed area of ring [c0,c1) with geo's shift-by-first-coordinate; 0 unless n>=3 and closed.
// Also returns the shifted first-moment sums used by the centroid.
template <bool MOMENTS>
__device__ __forceinline__ double ring_twice_area(const double2 *__restrict__ xy, int64_t c0, int64_t c1, int lane,
                                                  double &mx, double &my, double2 &shift) {
    mx = my = 0.0;
    int64_t n = c1 - c0;
    if (n < 3) return 0.0;
    double2 first = xy[c0], last = xy[c1 - 1];
    shift = first;
    if (first.x != last.x || first.y != last.y) return 0.0;
    double acc = 0.0, ax = 0.0, ay = 0.0;
    // unrolled x4: eight independent 128-bit loads in flight per lane (the loop is a pure HBM stream)
#pragma unroll 4
    for (int64_t i = c0 + lane; i < c1 - 1; i += 32) {
        double2 p = __ldcs(xy + i), q = __ldcs(xy + i + 1);
        double x0 = p.x - first.x, y0 = p.y - first.y;
        double x1 = q.x - first.x, y1 = q.y - first.y;
        double det = x0 * y1 - y0 * x1;
        acc += det;
        if (MOMENTS) {
            ax += (x1 + x0) * det;
            ay += (y1 + y0) * det;
        }
    }
    acc = bfly_sum(acc);
    if (MOMENTS) {
        mx = bfly_sum(ax);
        my = bfly_sum(ay);
    }
    return acc;
}

// Polygon::signed_area over rings [r0,r1): |exterior| - sum |holes|, exterior sign restored
__device__ __forceinline__ double polygon_signed_area(const double2 *xy, const int64_t *ring_off, int64_t r0, int64_t r1,
                                                      int lane) {
    if (r1 <= r0) return 0.0;
    double mx, my;
    double2 sh;
    double area = ring_twice_area<false>(xy, ring_off[r0], ring_off[r0 + 1], lane, mx, my, sh) / 2.0;
    bool neg = area < 0.0;
    double tot = fabs(area);
    for (int64_t r = r0 + 1; r < r1; ++r)
        tot = tot - fabs(ring_twice_area<false>(xy, ring_off[r], ring_off[r + 1], lane, mx, my, sh) / 2.0);
    return neg ? -tot : tot;
}

__global__ void __launch_bounds__(256) k_area(int type, int64_t n_geoms, const double2 *__restrict__ xy,
                                              const int64_t *__restrict__ geom_off, const int64_t *__restrict__ part_off,
                                              const int64_t *__restrict__ ring_off, double *__restrict__ out) {
    const int lane = threadIdx.x & 31;
    int64_t warp = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
    const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t g = warp; g < n_geoms; g += nwarps) {
        double v = 0.0;
        if (type == GPL_POLYGON) {
            v = fabs(polygon_signed_area(xy, ring_off, geom_off[g], geom_off[g + 1], lane));
        } else if (type == GPL_MULTIPOLYGON) {
            for (int64_t p = geom_off[g]; p < geom_off[g + 1]; ++p)
                v = v + fabs(polygon_signed_area(xy, ring_off, part_off[p], part_off[p + 1], lane));
        }
        if (lane == 0) out[g] = v;
    }
}

// ---- centroid: geo's CentroidOperation with dimension precedence ---------------------------------
struct WC {
    int dim;  // -1 empty, 0 points, 1 lines, 2 areas
    double w, ax, ay;
};
__device__ __forceinline__ void wc_add(WC &s, const WC &b) {
    if (b.dim < 0) return;
    if (s.dim < b.dim) {
        s = b;
    } else if (s.dim == b.dim) {
        s.ax = s.ax + b.ax;
        s.ay = s.ay + b.ay;
        s.w = s.w + b.w;
    }
}
// add_line_string over coords [c0,c1): 1-D sum of midpoint*len, 0-D sum of degenerate segment starts
// out of line: reached only by linestring rows and by degenerate (zero-area) rings; keeps the polygon hot
// path of k_centroid at 64 registers
static __device__ __noinline__ WC line_string_wc(const double2 *__restrict__ xy, int64_t c0, int64_t c1, int lane) {
    WC r{-1, 0.0, 0.0, 0.0};
    int64_t n = c1 - c0;
    if (n <= 0) return r;
    if (n == 1) {
        double2 p = xy[c0];
        return WC{0, 1.0, p.x, p.y};
    }
    double L = 0.0, lx = 0.0, ly = 0.0, n0 = 0.0, px = 0.0, py = 0.0;
    for (int64_t i = c0 + lane; i < c1 - 1; i += 32) {
        double2 p = xy[i], q = xy[i + 1];
        if (p.x == q.x && p.y == q.y) {
            n0 += 1.0;
            px += p.x;
            py += p.y;
        } else {
            double len = gpl_hypot(q.x - p.x, q.y - p.y);
            L += len;
            lx += ((q.x + p.x) / 2.0) * len;
            ly += ((q.y + p.y) / 2.0) * len;
        }
    }
    L = bfly_sum(L), lx = bfly_sum(lx), ly = bfly_sum(ly);
    n0 = bfly_sum(n0), px = bfly_sum(px), py = bfly_sum(py);
    // dimension precedence: any non-degenerate segment makes the result 1-D and drops the 0-D terms
    bool has1 = (double)(n - 1) != n0;
    if (has1) return WC{1, L, lx, ly};
    return WC{0, n0, px, py};
}
__device__ __forceinline__ WC ring_wc(const double2 *__restrict__ xy, int64_t c0, int64_t c1, int lane) {
    double mx, my;
    double2 shift;
    double area = ring_twice_area<true>(xy, c0, c1, lane, mx, my, shift) / 2.0;
    if (area == 0.0) return line_string_wc(xy, c0, c1, lane);  // n==0 -> none, n==1 -> point, else linestring
    double cx = mx / (6.0 * area) + shift.x;
    double cy = my / (6.0 * area) + shift.y;
    double w = fabs(area);
    return WC{2, w, cx * w, cy * w};
}
__device__ __forceinline__ void polygon_wc(WC &s, const double2 *xy, const int64_t *ring_off, int64_t r0, int64_t r1,
                                           int lane) {
    if (r1 <= r0) return;
    WC ext = ring_wc(xy, ring_off[r0], ring_off[r0 + 1], lane);
    WC itr{-1, 0.0, 0.0, 0.0};
    for (int64_t r = r0 + 1; r < r1; ++r) {
        WC h = ring_wc(xy, ring_off[r], ring_off[r + 1], lane);
        if (itr.dim < 0) itr = h;
        else wc_add(itr, h);
    }
    if (ext.dim >= 0) {
        WC poly = ext;
        if (itr.dim >= 0) {
            if (poly.dim == itr.dim) {
                poly.ax = poly.ax - itr.ax;
                poly.ay = poly.ay - itr.ay;
                poly.w = poly.w - itr.w;
            }
            if (poly.w == 0.0) {  // holes cover the exterior: degenerate to the exterior linestring
                if (s.dim <= 1) {
                    WC l = line_string_wc(xy, ring_off[r0], ring_off[r0 + 1], lane);
                    if (s.dim < 0) s = l;
                    else wc_add(s, l);
                }
                return;
            }
        }
        if (s.dim < 0) s = poly;
        else wc_add(s, poly);
    }
}

__global__ void __launch_bounds__(256, 3) k_centroid(int type, int64_t n_geoms, const double2 *__restrict__ xy,
                                                  const int64_t *__restrict__ geom_off,
                                                  const int64_t *__restrict__ part_off,
                                                  const int64_t *__restrict__ ring_off,
                                                  const uint8_t *__restrict__ validity, double2 *__restrict__ out,
                                                  uint8_t *__restrict__ out_valid_bytes) {
    const int lane = threadIdx.x & 31;
    int64_t warp = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
    const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t g = warp; g < n_geoms; g += nwarps) {
        WC s{-1, 0.0, 0.0, 0.0};
        if (bit_get(validity, g)) {
            switch (type) {
            case GPL_POINT: {
                double2 p = xy[g];
                if (!(isnan(p.x) && isnan(p.y))) s = WC{0, 1.0, p.x, p.y};
                break;
            }
            case GPL_MULTIPOINT: {
                double sx = 0.0, sy = 0.0;
                int64_t c0 = geom_off[g], c1 = geom_off[g + 1];
                for (int64_t c = c0 + lane; c < c1; c += 32) {
                    double2 p = xy[c];
                    sx += p.x;
                    sy += p.y;
                }
                if (c1 > c0) s = WC{0, (double)(c1 - c0), bfly_sum(sx), bfly_sum(sy)};
                break;
            }
            case GPL_LINESTRING:
                s = line_string_wc(xy, geom_off[g], geom_off[g + 1], lane);
                break;
            case GPL_MULTILINESTRING:
                for (int64_t l = geom_off[g]; l < geom_off[g + 1]; ++l) {
                    if (s.dim > 1) break;
                    WC w = line_string_wc(xy, ring_off[l], ring_off[l + 1], lane);
                    if (s.dim < 0) s = w;
                    else wc_add(s, w);
                }
                break;
            case GPL_POLYGON:
                polygon_wc(s, xy, ring_off, geom_off[g], geom_off[g + 1], lane);
                break;
            case GPL_MULTIPOLYGON:
                for (int64_t p = geom_off[g]; p < geom_off[g + 1]; ++p)
                    polygon_wc(s, xy, ring_off, part_off[p], part_off[p + 1], lane);
                break;
            default:
                break;
            }
        }
        if (lane == 0) {
            if (s.dim >= 0) {
                out[g] = make_double2(s.ax / s.w, s.ay / s.w);
                out_valid_bytes[g] = 1;
            } else {
                out[g] = make_double2(nan(""), nan(""));
                out_valid_bytes[g] = 0;
            }
        }
    }
}

// ---- envelope: bounding rect over exterior coordinates --------------------------------------------
__device__ __forceinline__ void bbox_range(const double2 *__restrict__ xy, int64_t c0, int64_t c1, int lane, double &x0,
                                           double &y0, double &x1, double &y1) {
    for (int64_t c = c0 + lane; c < c1; c += 32) {
        double2 p = xy[c];
        x0 = fmin(x0, p.x), y0 = fmin(y0, p.y), x1 = fmax(x1, p.x), y1 = fmax(y1, p.y);
    }
}
__global__ void __launch_bounds__(256) k_envelope(int type, int64_t n_geoms, const double2 *__restrict__ xy,
                                                  const int64_t *__restrict__ geom_off,
                                                  const int64_t *__restrict__ part_off,
                                                  const int64_t *__restrict__ ring_off,
                                                  const uint8_t *__restrict__ validity, double *__restrict__ out4,
                                                  uint8_t *__restrict__ out_valid_bytes) {
    const int lane = threadIdx.x & 31;
    int64_t warp = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
    const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    const double inf = __longlong_as_double(0x7ff0000000000000LL);
    for (int64_t g = warp; g < n_geoms; g += nwarps) {
        double x0 = inf, y0 = inf, x1 = -inf, y1 = -inf;
        int64_t total = 0;
        if (bit_get(validity, g)) {
            switch (type) {
            case GPL_POINT: {
                double2 p = xy[g];
                if (!(isnan(p.x) && isnan(p.y))) {
                    total = 1;
                    x0 = x1 = p.x, y0 = y1 = p.y;
                }
                break;
            }
            case GPL_LINESTRING:
            case GPL_MULTIPOINT:
                total = geom_off[g + 1] - geom_off[g];
                bbox_range(xy, geom_off[g], geom_off[g + 1], lane, x0, y0, x1, y1);
                break;
            case GPL_MULTILINESTRING:
                for (int64_t l = geom_off[g]; l < geom_off[g + 1]; ++l) {
                    total += ring_off[l + 1] - ring_off[l];
                    bbox_range(xy, ring_off[l], ring_off[l + 1], lane, x0, y0, x1, y1);
                }
                break;
            case GPL_POLYGON:
                if (geom_off[g + 1] > geom_off[g]) {
                    int64_t r = geom_off[g];
                    total = ring_off[r + 1] - ring_off[r];
                    bbox_range(xy, ring_off[r], ring_off[r + 1], lane, x0, y0, x1, y1);
                }
                break;
            case GPL_MULTIPOLYGON:
                for (int64_t p = geom_off[g]; p < geom_off[g + 1]; ++p)
                    if (part_off[p + 1] > part_off[p]) {
                        int64_t r = part_off[p];
                        total += ring_off[r + 1] - ring_off[r];
                        bbox_range(xy, ring_off[r], ring_off[r + 1], lane, x0, y0, x1, y1);
                    }
                break;
            default:
                break;
            }
        }
        x0 = warp_min(x0), y0 = warp_min(y0), x1 = warp_max(x1), y1 = warp_max(y1);
        if (lane == 0) {
            bool has = total > 0;
            double qn = nan("");
            out4[4 * g] = has ? x0 : qn;
            out4[4 * g + 1] = has ? y0 : qn;
            out4[4 * g + 2] = has ? x1 : qn;
            out4[4 * g + 3] = has ? y1 : qn;
            out_valid_bytes[g] = has ? 1 : 0;
        }
    }
}

// ---- euclidean length ------------------------------------------------------------------------------
__device__ __forceinline__ double range_length(const double2 *__restrict__ xy, int64_t c0, int64_t c1, int lane) {
    double s = 0.0;
    for (int64_t i = c0 + lane; i < c1 - 1; i += 32) {
        double2 p = xy[i], q = xy[i + 1];
        s += gpl_hypot(q.x - p.x, q.y - p.y);
    }
    return s;
}
__global__ void __launch_bounds__(256) k_length(int type, int64_t n_geoms, const double2 *__restrict__ xy,
                                                const int64_t *__restrict__ geom_off, const int64_t *__restrict__ part_off,
                                                const int64_t *__restrict__ ring_off, double *__restrict__ out) {
    const int lane = threadIdx.x & 31;
    int64_t warp = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
    const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t g = warp; g < n_geoms; g += nwarps) {
        double s = 0.0;
        switch (type) {
        case GPL_LINESTRING:
            s = range_length(xy, geom_off[g], geom_off[g + 1], lane);
            break;
        case GPL_MULTILINESTRING:
            for (int64_t l = geom_off[g]; l < geom_off[g + 1]; ++l) s += range_length(xy, ring_off[l], ring_off[l + 1], lane);
            break;
        case GPL_POLYGON:
            if (geom_off[g + 1] > geom_off[g]) s = range_length(xy, ring_off[geom_off[g]], ring_off[geom_off[g] + 1], lane);
            break;
        case GPL_MULTIPOLYGON:
            for (int64_t p = geom_off[g]; p < geom_off[g + 1]; ++p)
                if (part_off[p + 1] > part_off[p]) s += range_length(xy, ring_off[part_off[p]], ring_off[part_off[p] + 1], lane);
            break;
        default:
            break;
        }
        s = bfly_sum(s);
        if (lane == 0) out[g] = s;
    }
}

int centroid_raw(gpl_ctx *ctx, const gpl_array *in, double2 *out_dev, uint8_t *valid_bytes_dev) {
    if (in->n_geoms == 0) return GPL_OK;
    GPL_LAUNCH(ctx, k_centroid, warp_grid(in->n_geoms, 8, 8), 256, 0, in->type, in->n_geoms,
               reinterpret_cast<const double2 *>(in->xy), in->geom_off, in->part_off, in->ring_off, in->validity, out_dev,
               valid_bytes_dev);
    return GPL_OK;
}
int envelope_raw(gpl_ctx *ctx, const gpl_array *in, double *out4_dev, uint8_t *valid_bytes_dev) {
    if (in->n_geoms == 0) return GPL_OK;
    GPL_LAUNCH(ctx, k_envelope, warp_grid(in->n_geoms, 8, 8), 256, 0, in->type, in->n_geoms,
               reinterpret_cast<const double2 *>(in->xy), in->geom_off, in->part_off, in->ring_off, in->validity, out4_dev,
               valid_bytes_dev);
    return GPL_OK;
}

__global__ void k_bbox_center(const double *__restrict__ b4, double2 *__restrict__ out, int64_t n) {
    int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= n) return;
    // geo Rect::center: (max + min) / 2
    out[i] = make_double2((b4[4 * i + 2] + b4[4 * i]) / 2.0, (b4[4 * i + 3] + b4[4 * i + 1]) / 2.0);
}

// per-geometry transform origin: centroid (TransformOrigin::Centroid) or bbox centre (::Center),
// py-geopolars/src/utils.rs:17-23.  NaN where the geometry has neither.
int origin_table(gpl_ctx *ctx, const gpl_array *in, int origin, double2 *out_dev) {
    if (in->n_geoms == 0) return GPL_OK;
    Scratch<uint8_t> vb;
    GPL_TRY(vb.get(ctx, (size_t)in->n_geoms));
    if (origin == GPL_ORIGIN_CENTROID) return centroid_raw(ctx, in, out_dev, vb.p);
    Scratch<double> b4;
    GPL_TRY(b4.get(ctx, (size_t)in->n_geoms * 4));
    GPL_TRY(envelope_raw(ctx, in, b4.p, vb.p));
    GPL_LAUNCH(ctx, k_bbox_center, (int)ceil_div(in->n_geoms, 256), 256, 0, b4.p, out_dev, in->n_geoms);
    return GPL_OK;
}

// envelope as a POLYGON array: one 5-coord ring per geometry (geo Rect::to_polygon order:
// (min.x,min.y) (min.x,max.y) (max.x,max.y) (max.x,min.y) (min.x,min.y))
__global__ void k_envelope_polys(const double *__restrict__ b4, const uint8_t *__restrict__ vb, double2 *__restrict__ xy,
                                 int64_t *__restrict__ ring_off, int64_t *__restrict__ geom_off, int64_t n) {
    int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i > n) return;
    ring_off[i] = 5 * i;
    geom_off[i] = i;
    if (i == n) return;
    double x0 = b4[4 * i], y0 = b4[4 * i + 1], x1 = b4[4 * i + 2], y1 = b4[4 * i + 3];
    double2 *o = xy + 5 * i;
    o[0] = make_double2(x0, y0);
    o[1] = make_double2(x0, y1);
    o[2] = make_double2(x1, y1);
    o[3] = make_double2(x1, y0);
    o[4] = make_double2(x0, y0);
    (void)vb;
}

// rstar's AABB tests on the per-row envelopes: mode 0 = `contains_envelope` (row envelope inside the closed query
// box: RTree::locate_in_envelope, the reference's tests at spatial_index.rs:361-430), mode 1 = `intersects` (closed
// intervals: locate_in_envelope_intersecting / the candidate test of intersection_candidates_with_other_tree, :74-76)
__global__ void k_envelope_query(const double *__restrict__ b4, const uint8_t *__restrict__ has, int64_t n, double qx0, double qy0,
                                 double qx1, double qy1, int mode, uint8_t *__restrict__ out_bytes) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= n) return;
    const double x0 = b4[4 * i], y0 = b4[4 * i + 1], x1 = b4[4 * i + 2], y1 = b4[4 * i + 3];
    bool m;
    if (mode == 0) m = x0 >= qx0 && y0 >= qy0 && x1 <= qx1 && y1 <= qy1;
    else m = x0 <= qx1 && x1 >= qx0 && y0 <= qy1 && y1 >= qy0;
    out_bytes[i] = (m && has[i]) ? 1 : 0;  // NaN bounds (empty row) fail every comparison anyway
}

}  // namespace gpl

using namespace gpl;

extern "C" int gpl_envelope_query(gpl_ctx *ctx, const gpl_array *in, double minx, double miny, double maxx, double maxy, int mode,
                                  uint8_t *out_bitmap, int mem) {
    GPL_REQUIRE(ctx && in && out_bitmap, GPL_ERR_INVALID_ARG, "gpl_envelope_query: NULL argument");
    GPL_REQUIRE(mode == 0 || mode == 1, GPL_ERR_INVALID_ARG, "gpl_envelope_query: mode must be 0 (contained) or 1 (intersecting)");
    GPL_TRY(check_mem(mem, "gpl_envelope_query"));
    GPL_CUDA(cudaSetDevice(ctx->device));
    const int64_t n = in->n_geoms;
    if (n == 0) return GPL_OK;
    Scratch<double> b4;
    Scratch<uint8_t> vb, hit;
    GPL_TRY(b4.get(ctx, (size_t)n * 4));
    GPL_TRY(vb.get(ctx, (size_t)n));
    GPL_TRY(hit.get(ctx, (size_t)n));
    GPL_TRY(envelope_raw(ctx, in, b4.p, vb.p));
    GPL_LAUNCH(ctx, k_envelope_query, (int)ceil_div(n, 256), 256, 0, b4.p, vb.p, n, minx, miny, maxx, maxy, mode, hit.p);
    return finish_bitmap(ctx, hit.p, n, out_bitmap, mem);
}

extern "C" int gpl_area(gpl_ctx *ctx, const gpl_array *in, double *out, int mem) {
    GPL_REQUIRE(ctx && in && out, GPL_ERR_INVALID_ARG, "gpl_area: NULL argument");
    GPL_TRY(check_mem(mem, "gpl_area"));
    GPL_CUDA(cudaSetDevice(ctx->device));
    if (in->n_geoms == 0) return GPL_OK;
    RowOut<double> res;
    GPL_TRY(res.get(ctx, out, in->n_geoms, mem));
    GPL_LAUNCH(ctx, k_area, warp_grid(in->n_geoms, 8, 8), 256, 0, in->type, in->n_geoms, reinterpret_cast<const double2 *>(in->xy),
               in->geom_off, in->part_off, in->ring_off, res.p);
    return res.deliver(ctx);
}

extern "C" int gpl_euclidean_length(gpl_ctx *ctx, const gpl_array *in, double *out, int mem) {
    GPL_REQUIRE(ctx && in && out, GPL_ERR_INVALID_ARG, "gpl_euclidean_length: NULL argument");
    GPL_TRY(check_mem(mem, "gpl_euclidean_length"));
    GPL_CUDA(cudaSetDevice(ctx->device));
    if (in->n_geoms == 0) return GPL_OK;
    RowOut<double> res;
    GPL_TRY(res.get(ctx, out, in->n_geoms, mem));
    GPL_LAUNCH(ctx, k_length, warp_grid(in->n_geoms, 8, 8), 256, 0, in->type, in->n_geoms,
               reinterpret_cast<const double2 *>(in->xy), in->geom_off, in->part_off, in->ring_off, res.p);
    return res.deliver(ctx);
}

extern "C" int gpl_centroid(gpl_ctx *ctx, const gpl_array *in, gpl_array **out) {
    GPL_REQUIRE(ctx && in && out, GPL_ERR_INVALID_ARG, "gpl_centroid: NULL argument");
    GPL_CUDA(cudaSetDevice(ctx->device));
    Scratch<double> xy;
    Scratch<uint8_t> vb, bm;
    GPL_TRY(xy.get(ctx, (size_t)in->n_geoms * 2));
    GPL_TRY(vb.get(ctx, (size_t)in->n_geoms));
    GPL_TRY(bm.get(ctx, (size_t)(in->n_geoms + 7) / 8));
    GPL_TRY(centroid_raw(ctx, in, reinterpret_cast<double2 *>(xy.p), vb.p));
    GPL_TRY(pack_bits(ctx, vb.p, bm.p, in->n_geoms));
    gpl_array *o = array_new(ctx, GPL_POINT);
    o->n_geoms = o->n_coords = in->n_geoms;
    o->xy = xy.take(), o->own_xy = true;
    o->validity = bm.take(), o->own_valid = true;
    *out = o;
    return GPL_OK;
}

extern "C" int gpl_envelope(gpl_ctx *ctx, const gpl_array *in, gpl_array **out, double *out4, int mem) {
    GPL_REQUIRE(ctx && in && (out || out4), GPL_ERR_INVALID_ARG, "gpl_envelope: NULL argument");
    GPL_TRY(check_mem(mem, "gpl_envelope"));
    GPL_CUDA(cudaSetDevice(ctx->device));
    int64_t n = in->n_geoms;
    Scratch<double> b4;
    Scratch<uint8_t> vb;
    GPL_TRY(b4.get(ctx, (size_t)n * 4));
    GPL_TRY(vb.get(ctx, (size_t)n));
    GPL_TRY(envelope_raw(ctx, in, b4.p, vb.p));
    if (out) {
        Scratch<double> xy;
        Scratch<int64_t> ro, go;
        Scratch<uint8_t> bm;
        GPL_TRY(xy.get(ctx, (size_t)n * 10));
        GPL_TRY(ro.get(ctx, (size_t)n + 1));
        GPL_TRY(go.get(ctx, (size_t)n + 1));
        GPL_TRY(bm.get(ctx, (size_t)(n + 7) / 8));
        GPL_LAUNCH(ctx, k_envelope_polys, (int)ceil_div(n + 1, 256), 256, 0, b4.p, vb.p, reinterpret_cast<double2 *>(xy.p), ro.p,
                   go.p, n);
        GPL_TRY(pack_bits(ctx, vb.p, bm.p, n));
        gpl_array *o = array_new(ctx, GPL_POLYGON);
        o->n_geoms = n, o->n_rings = n, o->n_coords = 5 * n;
        o->xy = xy.take(), o->own_xy = true;
        o->ring_off = ro.take(), o->own_ring = true;
        o->geom_off = go.take(), o->own_geom = true;
        o->validity = bm.take(), o->own_valid = true;
        *out = o;
    }
    if (out4) GPL_TRY(deliver(ctx, out4, b4.p, sizeof(double) * 4 * n, mem));
    return GPL_OK;
}
