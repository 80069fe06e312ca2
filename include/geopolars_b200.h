/*
 * geopolars_b200.h — C ABI of the H100-native GeoSeries engine (libgeopolars_b200.so).
 *
 * This is the drop-in boundary for the reference's GeoSeries hot path: every entry point below is
 * what a reference-side FFI shim binds in place of the per-row `iter_geom(..).map(geo_algo)` loop
 * (reference: geopolars/geopolars-geo/src/util.rs:27-37) behind `impl GeoSeries for Series`
 * (geopolars/geopolars-geo/src/geoseries.rs:183-279).  Plain pointers and sizes only; no torch,
 * polars or C++ types cross this line.  INTEGRATION.md shows the Rust / PyO3 / ctypes binding.
 *
 * Conventions
 *   - every function returns gpl_status (0 = ok, <0 = error); the message for the calling thread is
 *     returned by gpl_last_error().  Error codes mirror GeopolarsError
 *     (geopolars/geopolars-geo/src/error.rs:9-28): INVALID_TYPE = MismatchedGeometry,
 *     LENGTH_MISMATCH = polars ShapeMisMatch.
 *   - geometry arrays use the GeoArrow nesting (coords + geom/part/ring offsets + validity bitmap),
 *     geometry type codes are the reference's GeometryType enum
 *     (py-geopolars/python/geopolars/enums.py:4-15).
 *   - inputs are borrowed for the duration of the call (Arrow C Data Interface ownership rules,
 *     py-geopolars/src/ffi.rs:10-31); outputs are either caller-provided buffers or library-owned
 *     gpl_array handles released with gpl_array_free().
 *   - `mem` arguments say where a caller buffer lives: GPL_HOST (copied with cudaMemcpyAsync on the
 *     context stream; pinned memory from gpl_host_alloc() makes that truly asynchronous) or
 *     GPL_DEVICE (used in place).  Any other value is rejected with GPL_ERR_INVALID_ARG.
 *   - null rows propagate to null outputs (the reference panics on them, util.rs:32): a strict
 *     superset of the reference behaviour.
 *   - all work is enqueued on the context stream; functions that return data to GPL_HOST buffers
 *     synchronise that stream before returning, GPL_DEVICE results are stream-ordered.
 */
#ifndef GEOPOLARS_B200_H
#define GEOPOLARS_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define GPL_ABI_VERSION 1

typedef enum gpl_status {
    GPL_OK = 0,
    GPL_ERR_INVALID_TYPE = -1,    /* GeopolarsError::MismatchedGeometry (error.rs:12-16) */
    GPL_ERR_LENGTH_MISMATCH = -2, /* polars ShapeMisMatch (py-geopolars/src/error.rs:27-60) */
    GPL_ERR_CUDA = -3,
    GPL_ERR_NCCL = -4,
    GPL_ERR_OOM = -5,
    GPL_ERR_UNSUPPORTED = -6,
    GPL_ERR_INVALID_ARG = -7
} gpl_status;

typedef enum gpl_mem { GPL_HOST = 0, GPL_DEVICE = 1 } gpl_mem;

/* reference: py-geopolars/python/geopolars/enums.py:4-15 ; geoseries.rs:60-73 */
typedef enum gpl_geometry_type {
    GPL_MISSING = -1,
    GPL_POINT = 0,
    GPL_LINESTRING = 1,
    GPL_LINEARRING = 2,
    GPL_POLYGON = 3,
    GPL_MULTIPOINT = 4,
    GPL_MULTILINESTRING = 5,
    GPL_MULTIPOLYGON = 6,
    GPL_GEOMETRYCOLLECTION = 7
} gpl_geometry_type;

/* TransformOrigin of rotate/scale/skew (py-geopolars/src/utils.rs:5-27) */
typedef enum gpl_origin { GPL_ORIGIN_CENTROID = 0, GPL_ORIGIN_CENTER = 1, GPL_ORIGIN_POINT = 2 } gpl_origin;

typedef struct gpl_ctx gpl_ctx;             /* one per (host thread, device) */
typedef struct gpl_array gpl_array;         /* GeoArrow geometry array resident in HBM */
typedef struct gpl_pip_index gpl_pip_index;
typedef struct gpl_nearest_index gpl_nearest_index; /* right side of a nearest join */
typedef struct gpl_geo_index gpl_geo_index; /* right side of a great-circle join */
/* (lhs_index, rhs_index) pair list of a join, resident on the device.  Every pair list the library returns is sorted by
 * (lhs, rhs) and holds no pair twice.  An entry point that returns one through gpl_pairs **out stores it only when it returns
 * GPL_OK; on any error *out is NULL and nothing is left to free. */
typedef struct gpl_pairs gpl_pairs;

/* Raw GeoArrow buffers (the zero-dependency form of an Arrow array; replaces the WKB BinaryArray the
 * reference re-parses on every op, util.rs:27-37).
 *   POINT            coords[n_geoms]
 *   LINESTRING       geom_offsets[n_geoms+1] -> coords
 *   POLYGON          geom_offsets[n_geoms+1] -> rings ; ring_offsets[n_rings+1] -> coords
 *   MULTIPOINT       geom_offsets[n_geoms+1] -> coords
 *   MULTILINESTRING  geom_offsets[n_geoms+1] -> lines ; ring_offsets[n_rings+1] -> coords
 *   MULTIPOLYGON     geom_offsets[n_geoms+1] -> polygons ; part_offsets[n_parts+1] -> rings ;
 *                    ring_offsets[n_rings+1] -> coords
 * coords: interleaved (x = xy pairs, y = NULL; GeoArrow FixedSizeList<f64>[2]) or separated
 * (x, y; GeoArrow Struct{x,y}, what py-geopolars builds, internals/geoseries.py:87-107).
 * offsets: int32 (List) or int64 (LargeList), all three the same width. */
typedef struct gpl_buffers {
    int32_t geom_type;    /* gpl_geometry_type */
    int32_t offset_width; /* 32 or 64 */
    int32_t mem;          /* gpl_mem: where every pointer below lives */
    int32_t reserved;
    int64_t n_geoms;
    int64_t n_parts; /* MULTIPOLYGON only */
    int64_t n_rings; /* POLYGON, MULTILINESTRING, MULTIPOLYGON */
    int64_t n_coords;
    const double *x; /* interleaved xy when y == NULL */
    const double *y;
    const void *geom_offsets;
    const void *part_offsets;
    const void *ring_offsets;
    const uint8_t *validity; /* Arrow LSB-first bitmap over geometries, or NULL (= all valid) */
} gpl_buffers;

/* device-side view of a gpl_array (always interleaved coords + int64 offsets); pointers stay valid
 * until the array is freed. */
typedef struct gpl_device_view {
    int32_t geom_type;
    int32_t reserved;
    int64_t n_geoms, n_parts, n_rings, n_coords;
    const double *xy;
    const int64_t *geom_offsets, *part_offsets, *ring_offsets;
    const uint8_t *validity;
} gpl_device_view;

/* ---------------------------------------------------------------- context ---------------- */
int gpl_abi_version(void);
const char *gpl_last_error(void);
/* device: CUDA ordinal.  stream: an existing cudaStream_t to enqueue on (e.g. the caller's current
 * stream) or NULL to let the context create its own non-blocking stream. */
int gpl_ctx_create(int device, void *stream, gpl_ctx **out);
int gpl_ctx_set_stream(gpl_ctx *ctx, void *stream);
int gpl_ctx_synchronize(gpl_ctx *ctx);
/* Measurement aid (bench.py's roofline line): while enabled, every launch of the streaming points-in-polygons kernel
 * (k_pip_stream, the kernel behind gpl_contains_join* — reference path spatial_index.rs:139-157 + geo `Contains`) on this
 * context is bracketed by two CUDA events on the context's stream.  _read waits for the recorded pairs and returns their
 * summed duration (ms) and count since the previous read. */
int gpl_ctx_kernel_timing(gpl_ctx *ctx, int enable);
int gpl_ctx_kernel_timing_read(gpl_ctx *ctx, double *ms_total, int64_t *launches);
void gpl_ctx_destroy(gpl_ctx *ctx);
/* give the cached (free) device blocks of the context's allocator back to the driver */
int gpl_ctx_trim(gpl_ctx *ctx);
/* number of kernels this context has launched (bench.py's gpu_launches) */
int64_t gpl_ctx_launch_count(const gpl_ctx *ctx);
/* pinned host memory for truly asynchronous H2D/D2H */
int gpl_host_alloc(size_t bytes, void **out);
void gpl_host_free(void *p);

/* ---------------------------------------------------------------- arrays ----------------- */
/* Host buffers are copied to HBM once (cudaMemcpyAsync); device buffers are borrowed when they are
 * already interleaved / int64, converted into owned copies otherwise. */
int gpl_array_from_buffers(gpl_ctx *ctx, const gpl_buffers *b, gpl_array **out);
int gpl_array_view(const gpl_array *a, gpl_device_view *out);
/* copy an array back into caller buffers (any pointer may be NULL to skip it); offsets are written
 * as int64. */
int gpl_array_copy_out(gpl_ctx *ctx, const gpl_array *a, double *xy, int64_t *geom_offsets, int64_t *part_offsets,
                       int64_t *ring_offsets, uint8_t *validity, int mem);
void gpl_array_free(gpl_array *a);

/* WKB (ISO, either endianness, XY) -> GeoArrow, decoded ONCE (replaces util.rs:27-37 per-op parse).
 * offsets: int32[n+1] Arrow binary offsets into bytes; all rows must share one geometry type
 * (Polygon rows are promoted when mixed with MultiPolygon, LineString with MultiLineString,
 * Point with MultiPoint).  Host input. */
int gpl_array_from_wkb(gpl_ctx *ctx, const uint8_t *bytes, const int32_t *offsets, const uint8_t *validity,
                       int64_t n, gpl_array **out);
/* GeoArrow -> WKB (from_geom_vec, util.rs:11-24). Two calls: first with bytes == NULL to get
 * *n_bytes and offsets, then with a buffer of that size. Host output. */
int gpl_array_to_wkb(gpl_ctx *ctx, const gpl_array *a, int32_t *offsets, uint8_t *bytes, int64_t *n_bytes);
/* The codec itself, on the GPU (util.rs:11-37 is the per-row, per-op host loop it replaces): bytes / offsets /
 * validity in host OR device memory (`mem`), offsets int32 (`binary`) or int64 (`large_binary`) per
 * `offset_width`; offsets need not start at 0 (sliced arrays).  gpl_wkb_encode follows the two-call protocol
 * of gpl_array_to_wkb (bytes == NULL: offsets and *n_bytes only) and writes little-endian ISO WKB; null rows
 * are zero-length.  gpl_array_from_wkb / gpl_array_to_wkb are the (host, int32) forms of these. */
int gpl_wkb_decode(gpl_ctx *ctx, const uint8_t *bytes, const void *offsets, int offset_width, const uint8_t *validity,
                   int64_t n, int mem, gpl_array **out);
int gpl_wkb_encode(gpl_ctx *ctx, const gpl_array *a, void *offsets, int offset_width, uint8_t *bytes, int64_t *n_bytes,
                   int mem);

/* Arrow C Data Interface (same structs the reference moves across its FFI, py-geopolars/src/ffi.rs:14-49).
 * Accepts geoarrow nested layouts (interleaved or struct coords, List or LargeList) and WKB
 * binary / large_binary columns.  `array`/`schema` are struct ArrowArray* / struct ArrowSchema*;
 * import borrows (never releases) them. export fills caller-allocated structs whose release
 * callbacks free library-owned host memory. */
int gpl_array_import_arrow(gpl_ctx *ctx, const void *array, const void *schema, gpl_array **out);
int gpl_array_export_arrow(gpl_ctx *ctx, const gpl_array *a, void *out_array, void *out_schema);
/* primitive result columns (float64 / bool bitmap / int8 / int32) as Arrow arrays */
int gpl_export_f64_arrow(const double *values_host, const uint8_t *validity, int64_t n, void *out_array, void *out_schema);
int gpl_export_bool_arrow(const uint8_t *bitmap_host, const uint8_t *validity, int64_t n, void *out_array, void *out_schema);

/* ---------------------------------------------------------------- GeoSeries ops ---------- */
/* GeoSeries::affine_transform (geoseries.rs:11-12): x' = a*x + b*y + xoff ; y' = d*x + e*y + yoff.
 * Named scalars, not a [f64;6], because the reference's array order is ambiguous (SURVEY.md §7). */
int gpl_affine_transform(gpl_ctx *ctx, const gpl_array *in, double a, double b, double xoff, double d, double e,
                         double yoff, gpl_array **out);
/* GeoSeries::translate (geoseries.rs:174), scale (:107), rotate (:93, degrees), skew (:139, degrees).
 * origin: per-geometry centroid / bbox centre, or the fixed point (ox, oy). */
int gpl_translate(gpl_ctx *ctx, const gpl_array *in, double xoff, double yoff, gpl_array **out);
int gpl_scale(gpl_ctx *ctx, const gpl_array *in, double xfact, double yfact, int origin, double ox, double oy,
              gpl_array **out);
int gpl_rotate(gpl_ctx *ctx, const gpl_array *in, double angle_deg, int origin, double ox, double oy, gpl_array **out);
int gpl_skew(gpl_ctx *ctx, const gpl_array *in, double xs_deg, double ys_deg, int origin, double ox, double oy,
             gpl_array **out);

/* GeoSeries::area (geoseries.rs:14-16): out[n_geoms] f64 */
int gpl_area(gpl_ctx *ctx, const gpl_array *in, double *out, int mem);
/* GeoSeries::centroid (geoseries.rs:18-21): POINT array; empty geometries -> null */
int gpl_centroid(gpl_ctx *ctx, const gpl_array *in, gpl_array **out);
/* GeoSeries::envelope (geoseries.rs:28-33): POLYGON array of 5-coord rectangles; out4 (optional,
 * may be NULL) additionally receives minx,miny,maxx,maxy per geometry */
int gpl_envelope(gpl_ctx *ctx, const gpl_array *in, gpl_array **out, double *out4, int mem);
/* GeoSeries::euclidean_length (geoseries.rs:35-41) */
int gpl_euclidean_length(gpl_ctx *ctx, const gpl_array *in, double *out, int mem);
/* GeoSeries::geodesic_length (geoseries.rs:52-58; method names py-geopolars/src/geo.rs:64-67): metres, input in
 * (lon, lat) degrees.  method 0 = geodesic (Karney 2013, WGS84), 1 = haversine, 2 = vincenty.  out_validity
 * (optional bitmap): a row is null when a Vincenty segment does not converge (the reference returns Err) */
int gpl_geodesic_length(gpl_ctx *ctx, const gpl_array *in, int method, double *out, uint8_t *out_validity, int mem);
/* geo 0.27 GeodesicArea on WGS84 (DESIGN.md 4.17), input in (lon, lat) degrees, any finite longitude.  One pass fills
 * area[n] (m^2) and perimeter[n] (m); either may be NULL, not both.  Each ring is geographiclib's PolygonArea over its
 * vertices, closing edge always included (a ring whose last coordinate equals its first is summed without that zero-length
 * edge, so a closed and an unclosed copy of a ring agree bit for bit), reduced modulo the
 * ellipsoid's area A0.  sign = 1: counter-clockwise positive, in (-A0/2, A0/2]; sign = 0: in [0, A0), so a clockwise exterior
 * gives A0 minus the enclosed area, as in geo.  Polygon: exterior minus the summed magnitudes of the holes (holes taken
 * clockwise positive; a negative exterior subtracts a negated sum), so with wrongly wound rings an unsigned value can leave
 * [0, A0) as geo's does; perimeter over every ring.  MultiPolygon: the sum over its
 * parts.  Point / LineString / MultiPoint / MultiLineString: 0.  Empty rows: 0.  A null row, a non-finite coordinate or
 * |lat| > 90 gives a null row (NaN, validity 0 in out_validity, which may be NULL).  Results are deterministic and a row's
 * value does not depend on the other rows of the call.  NULL ctx / in, both outputs NULL, sign not 0 or 1, or an unknown
 * mem: GPL_ERR_INVALID_ARG before any launch. */
int gpl_geodesic_area(gpl_ctx *ctx, const gpl_array *in, int sign, double *area, double *perimeter, uint8_t *out_validity, int mem);
/* GeoSeries::convex_hull (geoseries.rs:23-26): POLYGON array, one closed CCW ring per geometry, in
 * geo's quick_hull vertex order */
int gpl_convex_hull(gpl_ctx *ctx, const gpl_array *in, gpl_array **out);
/* GeoSeries::simplify (geoseries.rs:108-116, impl :240-242): Ramer-Douglas-Peucker with geo 0.27's minimum-size
 * guard (2 points per linestring, 4 per polygon ring); LineString / MultiLineString / Polygon / MultiPolygon;
 * tolerance <= 0 returns the input coordinates.  Outer offsets and validity are shared with the input. */
int gpl_simplify(gpl_ctx *ctx, const gpl_array *in, double tolerance, gpl_array **out);
/* GeoSeries::distance (geoseries.rs:141-146), row-wise 1:1; out[n] f64, out_validity bitmap
 * (may be NULL).  Pairs: any of Point / LineString / Polygon / MultiPoint / MultiLineString / MultiPolygon on
 * either side (geo EuclideanDistance; a Multi* operand is the minimum over its members, f64::MAX when it has none).
 * A row without a single segment where geo needs one (it would panic) is null. */
int gpl_distance(gpl_ctx *ctx, const gpl_array *a, const gpl_array *b, double *out, uint8_t *out_validity, int mem);
/* row-wise intersects (call sites spatial_index.rs:102-123 / geo Intersects); Arrow bitmap out.  Every pair of
 * Point, MultiPoint, LineString, MultiLineString, Polygon, MultiPolygon arrays; null row -> false */
int gpl_intersects(gpl_ctx *ctx, const gpl_array *a, const gpl_array *b, uint8_t *out_bitmap, int mem);
/* row-wise contains of a point: polygons[i] contains points[i] (spatial_index.rs:91-96); `polygons` may also be a
 * (Multi)LineString array (spatial_index.rs:125-135: interior of the line, end points only when closed).
 * Polygon-contains-Polygon (spatial_index.rs:99-101,107-111) is DE-9IM relate in geo and is not provided:
 * GPL_ERR_INVALID_TYPE.  Arrow bitmap out */
int gpl_contains(gpl_ctx *ctx, const gpl_array *polygons, const gpl_array *points, uint8_t *out_bitmap, int mem);
/* secondary trait ops (geoseries.rs:43-83,176-180) */
int gpl_geom_type(gpl_ctx *ctx, const gpl_array *in, int8_t *out, int mem);
int gpl_is_empty(gpl_ctx *ctx, const gpl_array *in, uint8_t *out_bitmap, int mem);
int gpl_is_ring(gpl_ctx *ctx, const gpl_array *in, uint8_t *out_bitmap, int mem);
int gpl_x(gpl_ctx *ctx, const gpl_array *in, double *out, int mem);
int gpl_y(gpl_ctx *ctx, const gpl_array *in, double *out, int mem);
int gpl_exterior(gpl_ctx *ctx, const gpl_array *in, gpl_array **out);
int gpl_explode(gpl_ctx *ctx, const gpl_array *in, gpl_array **out);

/* SpatialIndex envelope queries (spatial_index.rs:206-312 builds one AABB per row, the tests at :361-430 query them
 * with rstar's RTree::locate_in_envelope): out bit i = row i's envelope lies inside the closed box [min,max]
 * (mode 0, `AABB::contains_envelope`) or intersects it (mode 1, closed intervals — the candidate test of the join,
 * :74-76).  Rows without an envelope (null / empty) never match (the reference unwraps and panics on them). */
int gpl_envelope_query(gpl_ctx *ctx, const gpl_array *in, double minx, double miny, double maxx, double maxy, int mode,
                       uint8_t *out_bitmap, int mem);

/* ---------------------------------------------------------------- spatial join ----------- */
/* Replaces SpatialIndex (spatial_index.rs:314-350) for the polygon side of a points-in-polygons
 * join: per-polygon bounding boxes in a uniform grid (candidate generation, closed intervals like
 * rstar's AABB test) plus a per-polygon y-bucketed edge table for the exact test.  Built on the
 * GPU from a POLYGON or MULTIPOLYGON array; keeps a reference to `polygons` (must outlive it). */
int gpl_pip_index_build(gpl_ctx *ctx, const gpl_array *polygons, gpl_pip_index **out);
void gpl_pip_index_free(gpl_pip_index *idx);
int64_t gpl_pip_index_bytes(const gpl_pip_index *idx);
/* diagnostic counters (synchronises the context stream): out8[0] = points the exact kernel re-evaluated since the
 * index was built, [1] = fine raster cells per axis, [2] = log2(fine cells per coarse cell and axis),
 * [3] = raster cells coded "walk", [4] = raster cells coded "inside", [5] = parts without FP32 lists,
 * [6] = index bytes, [7] = coarse cells per axis. */
int gpl_pip_index_stats(gpl_ctx *ctx, const gpl_pip_index *idx, int64_t *out8);
/* diagnostics: microseconds from the start of the index fill kernel to each of its phase boundaries (out12[5..11]) */
int gpl_pip_index_phases(gpl_ctx *ctx, const gpl_pip_index *idx, double *out12);
/* diagnostics: microseconds from the start of the index COUNT kernel to each build phase boundary: out12[0..4] = the count
 * kernel (start, after its three grid barriers, FP32 plan done), out12[5..11] = the fill kernel as above */
int gpl_pip_index_timeline(gpl_ctx *ctx, const gpl_pip_index *idx, double *out12);
/* diagnostics: read-only copy of one index table into host memory (synchronises the context stream).  which: 0 = raster
 * words (8 bytes per 16 fine cells), 1 = cand01 (8 bytes per coarse cell), 2 = cell records (32 bytes per coarse cell),
 * 3 = part records (32 bytes per part).  *nbytes: in = capacity of dst, out = size of the table; dst == NULL asks for the size. */
int gpl_pip_index_dump(gpl_ctx *ctx, const gpl_pip_index *idx, int which, void *dst, int64_t *nbytes);
/* spatial_join(points, polygons, Inner) candidate+exact test (spatial_index.rs:74-143):
 * first_id[p] = lowest polygon row containing point p, or -1; count[p] (may be NULL) = number of
 * containing rows.  points: xy interleaved, n points, in `mem`; a device column must be 16-byte aligned
 * (GPL_ERR_INVALID_ARG otherwise). */
int gpl_contains_join(gpl_ctx *ctx, const gpl_pip_index *idx, const double *points_xy, int64_t n_points,
                      int32_t *first_id, int32_t *count, int mem);
/* the join and the per-polygon hit counts of config 4 in ONE pass over the points: counts[n polygon rows] (u64) +=
 * number of points whose first containing row is that polygon (what gpl_join_histogram computes from first_id). */
int gpl_contains_join_counts(gpl_ctx *ctx, const gpl_pip_index *idx, const double *points_xy, int64_t n_points,
                             int32_t *first_id, uint64_t *counts, int mem);
/* same with the points given as a POINT gpl_array (null points -> -1) */
int gpl_contains_join_array(gpl_ctx *ctx, const gpl_pip_index *idx, const gpl_array *points, int32_t *first_id,
                            int32_t *count, int mem);
/* the (lhs_index, rhs_index) pair list the reference emits (spatial_index.rs:139-157), sorted by
 * (point, polygon).  Call with lhs == NULL to get *n_pairs, then with buffers of that size. */
int gpl_contains_join_pairs(gpl_ctx *ctx, const gpl_pip_index *idx, const double *points_xy, int64_t n_points,
                            uint64_t *lhs, uint64_t *rhs, int64_t *n_pairs, int mem);
/* the same pair list for a POINT gpl_array already in HBM (null points match nothing), as a device-resident gpl_pairs
 * (gpl_pairs_count / gpl_pairs_copy / gpl_pairs_free): no host round trip of the point column */
int gpl_contains_join_pairs_array(gpl_ctx *ctx, const gpl_pip_index *idx, const gpl_array *points, gpl_pairs **out);
/* host-resident points streamed through HBM in chunks with H2D / kernel / D2H overlapped on three
 * streams (the end-to-end path: PCIe-bound).  chunk_points = 0 picks a default. */
int gpl_contains_join_host(gpl_ctx *ctx, const gpl_pip_index *idx, const double *points_xy_host, int64_t n_points,
                           int32_t *first_id_host, int64_t chunk_points);
/* per-polygon hit counts: counts[n_polygons] u64 += hits (config 4's all-reduce input) */
int gpl_join_histogram(gpl_ctx *ctx, const int32_t *first_id, int64_t n_points, uint64_t *counts, int64_t n_polygons,
                       int mem);

/* row-wise (Multi)Polygon.contains(Polygon) (the Predicate::Contains arms of spatial_index.rs:99-110; geo's
 * relate(..).is_contains(), DE-9IM [T*****FF*], for valid operands): Arrow bitmap, null rows -> false. */
int gpl_contains_polygon(gpl_ctx *ctx, const gpl_array *a, const gpl_array *b, uint8_t *out_bitmap, int mem);
/* spatial_join(lhs, rhs, predicate) for ANY two geometry columns (spatial_index.rs:37-157): candidates = pairs whose
 * envelopes intersect (closed intervals, :74-76), exact test by the reference's type-pair dispatch (:89-137: Point x
 * (Multi)Polygon / (Multi)LineString in either order -> contains(point) whatever the predicate; (Multi)Polygon x Polygon ->
 * contains or intersects; Polygon x MultiPolygon -> intersects only; every other pair of types -> no match).  The
 * result is the pair list the reference builds at :139-157 (whose order is the tree traversal's), sorted by (lhs, rhs). */
#define GPL_PREDICATE_INTERSECTS 0
#define GPL_PREDICATE_CONTAINS 1
int gpl_spatial_join(gpl_ctx *ctx, const gpl_array *lhs, const gpl_array *rhs, int predicate, gpl_pairs **out);

/* ---------------------------------------------------------------- DE-9IM relate ---------- */
/* The DE-9IM matrix of a[i] and b[i] for any pair of the six types (DESIGN.md §4.20): rows are a's Interior, Boundary and
 * Exterior, columns b's; boundaries follow the OGC defaults (a point has none, a line's is the Mod-2 set of its chain ends, a
 * polygon's is its rings; rings are closed implicitly).  Every decision is an exact sign of input coordinates.  Defined for
 * valid (OGC) operands; on invalid input every entry is still F, 0, 1 or 2 but its value is not specified.  An empty operand
 * has F in its Interior and Boundary rows / columns.  A null row, or a row with a non-finite coordinate, gives a null matrix.
 * matrix[9 n] int8 in `mem`, row-major, -1 = F; out_validity (Arrow bitmap in `mem`, may be NULL).  Unequal lengths:
 * GPL_ERR_LENGTH_MISMATCH; a type outside the six: GPL_ERR_INVALID_TYPE. */
int gpl_relate(gpl_ctx *ctx, const gpl_array *a, const gpl_array *b, int8_t *matrix, uint8_t *out_validity, int mem);
/* predicates of gpl_relate_predicate / gpl_predicate_join, JTS's definitions on the matrix (dims: the operands' type
 * dimensions).  GPL_PREDICATE_CONTAINS here is the DE-9IM [T*****FF*] for any pair of types. */
#define GPL_PREDICATE_WITHIN 2            /* T*F**F*** */
#define GPL_PREDICATE_CONTAINS_PROPERLY 3 /* T**FF*FF* */
#define GPL_PREDICATE_COVERS 4            /* T*****FF*, *T****FF*, ***T**FF* or ****T*FF* */
#define GPL_PREDICATE_COVERED_BY 5        /* T*F**F***, *TF**F***, **FT*F*** or **F*TF*** */
#define GPL_PREDICATE_TOUCHES 6           /* FT*******, F**T***** or F***T****; false when both dims are 0 */
#define GPL_PREDICATE_CROSSES 7           /* dims a < b: T*T******; a > b: T*****T**; both 1: 0********; else false */
#define GPL_PREDICATE_OVERLAPS 8          /* dims both 0 or both 2: T*T***T**; both 1: 1*T***T**; else false */
#define GPL_PREDICATE_DISJOINT 9          /* FF*FF**** */
#define GPL_PREDICATE_EQUALS 10           /* same dimension and T*F**FFF*; two empty rows are equal */
#define GPL_PREDICATE_PATTERN 11          /* `pattern`: 9 characters over TF*012, either case */
/* row-wise predicate as an Arrow bitmap in `mem`; a null or non-finite row gives false.  `pattern` is read only for
 * GPL_PREDICATE_PATTERN.  An unknown predicate or a bad pattern: GPL_ERR_INVALID_ARG.  A row stops as soon as its answer is
 * decided. */
int gpl_relate_predicate(gpl_ctx *ctx, const gpl_array *a, const gpl_array *b, int predicate, const char *pattern, uint8_t *out_bitmap,
                         int mem);
/* Predicate join (GeoPandas' sjoin(predicate=...)): every pair (i, j) for which gpl_relate_predicate(lhs[i], rhs[j]) holds,
 * sorted by (lhs, rhs), as a device-resident gpl_pairs.  Candidates are the pairs gpl_intersects accepts (every accepted
 * predicate implies it); GPL_PREDICATE_INTERSECTS returns them as they are.  A predicate that can hold for disjoint pairs
 * (GPL_PREDICATE_DISJOINT, or a pattern whose II, IB, BI and BB entries are all F or *) is GPL_ERR_INVALID_ARG.  Fewer than
 * 2^31 rows per side (else GPL_ERR_UNSUPPORTED). */
int gpl_predicate_join(gpl_ctx *ctx, const gpl_array *lhs, const gpl_array *rhs, int predicate, const char *pattern, gpl_pairs **out);

int64_t gpl_pairs_count(const gpl_pairs *pairs);
int gpl_pairs_copy(gpl_ctx *ctx, const gpl_pairs *pairs, uint64_t *lhs, uint64_t *rhs, int mem);
void gpl_pairs_free(gpl_pairs *pairs);

/* ---------------------------------------------------------------- nearest join ----------- */
/* Nearest-geometry join (GeoPandas sjoin_nearest; rstar's nearest_neighbor): for each point of a POINT column, the right
 * rows at the smallest distance.  Right side: Point / LineString / Polygon / MultiPoint / MultiLineString / MultiPolygon,
 * fewer than 2^31 rows.  Candidate rows R: non-null, with an envelope and only finite coordinates; no other row matches.
 * d(i, j) is exactly the f64 value gpl_distance returns for the row pair (lhs[i], rhs[j]).  The nearest rows of point i
 * are those of R at the minimum d <= max_distance (inclusive; +inf = unbounded; NaN or negative -> GPL_ERR_INVALID_ARG);
 * rows tie when their distances are equal f64 values.  Null points and points with a non-finite coordinate match nothing.
 * The index keeps a reference to `rhs` (must outlive it). */
int gpl_nearest_index_build(gpl_ctx *ctx, const gpl_array *rhs, gpl_nearest_index **out);
void gpl_nearest_index_free(gpl_nearest_index *idx);
/* synchronises the context stream: out8[0] = rows in R, [1] = excluded rows, [2] = rows every query evaluates (an empty
 * member, an empty ring or a 1-coordinate linestring / ring), [3] = grid cells per axis, [4] = cell items, [5] = index
 * bytes, [6] = exact distance evaluations of the last query pass, [7] = points the last query pass sent to the overflow
 * path.  The distance-within passes (gpl_dwithin_*) update [6] too and leave [7] at 0 (they have no overflow path).
 * [6] and [7] live in the index: gpl_nearest_join_pairs_array runs two passes and leaves the counts of its second,
 * and queries of one index issued concurrently on different streams overwrite each other's counts (never their results). */
int gpl_nearest_index_stats(gpl_ctx *ctx, const gpl_nearest_index *idx, int64_t *out8);
/* dense form: nearest_id[i] = lowest tied row or -1, distance[i] (may be NULL) = its distance or NaN, n_tied[i] (may be
 * NULL) = number of tied rows.  points_xy interleaved, n_points < 2^31 (else GPL_ERR_UNSUPPORTED), all buffers in `mem`. */
int gpl_nearest_join(gpl_ctx *ctx, const gpl_nearest_index *idx, const double *points_xy, int64_t n_points, double max_distance,
                     int32_t *nearest_id, double *distance, int32_t *n_tied, int mem);
/* the same for a POINT gpl_array (any other type: GPL_ERR_INVALID_TYPE); outputs in `mem` */
int gpl_nearest_join_array(gpl_ctx *ctx, const gpl_nearest_index *idx, const gpl_array *points, double max_distance,
                           int32_t *nearest_id, double *distance, int32_t *n_tied, int mem);
/* every tied (point, row) pair once, sorted by (lhs, rhs), as a device-resident gpl_pairs; distance (may be NULL, in
 * `mem`) receives the dense distance of every point (NaN: no match), which the pair list is built from. */
int gpl_nearest_join_pairs_array(gpl_ctx *ctx, const gpl_nearest_index *idx, const gpl_array *points, double max_distance,
                                 gpl_pairs **out, double *distance, int mem);
/* Nearest join for a left column of ANY of the six types (DESIGN.md §4.13), fewer than 2^31 rows (else GPL_ERR_UNSUPPORTED,
 * checked before any access).  A left row takes part only if it is non-null, has an envelope and only finite coordinates;
 * any other left row matches nothing.  d(i, j) is exactly the f64 that gpl_distance(lhs, rhs) returns for the row pair, with
 * lhs as the FIRST operand; a pair for which gpl_distance returns null never matches.  max_distance, ties and the outputs
 * are those of gpl_nearest_join_array / gpl_nearest_join_pairs_array; a POINT left column goes to those entry points and
 * gives the same bits.  One warp evaluates one left row; a left row with an empty member, an empty ring or a 1-coordinate
 * linestring / ring is evaluated against every row of R (correct at any count, slow when there are many of them). */
int gpl_nearest_join_geom(gpl_ctx *ctx, const gpl_nearest_index *idx, const gpl_array *lhs, double max_distance, int32_t *nearest_id,
                          double *distance, int32_t *n_tied, int mem);
int gpl_nearest_join_geom_pairs(gpl_ctx *ctx, const gpl_nearest_index *idx, const gpl_array *lhs, double max_distance, gpl_pairs **out,
                                double *distance, int mem);

/* ---------------------------------------------------------------- distance-within join --- */
/* Every row of R within `distance` of each left row (GeoPandas sjoin(predicate="dwithin", distance=D)), on a nearest index
 * (DESIGN.md §4.14).  The eligible right rows R are those of the nearest index; a left row of any of the six types takes part
 * only if it is non-null, has an envelope and only finite coordinates; no other row matches anything.  d(i, j) is exactly the
 * f64 that gpl_distance(lhs, rhs) returns for the row pair, with lhs as the FIRST operand; a pair for which gpl_distance
 * returns null never matches.  (i, j) matches when d(i, j) <= distance (inclusive).  distance must be finite and >= 0 (NaN,
 * negative or +-inf -> GPL_ERR_INVALID_ARG); 0 means touching or intersecting, as `distance` computes it.  Fewer than 2^31
 * left rows per call (else GPL_ERR_UNSUPPORTED); both checked before any launch or access.  A POINT left column runs one lane
 * per point, any other type one warp per row.  Outputs are deterministic (two calls give byte-identical results). */
/* count[i] (int32, in `mem`) = number of matching right rows of left row i */
int gpl_dwithin_count(gpl_ctx *ctx, const gpl_nearest_index *idx, const gpl_array *lhs, double distance, int32_t *count, int mem);
/* every matching pair once, sorted by (lhs, rhs), as a device-resident gpl_pairs (int64 total count); with_distance != 0
 * also keeps d(i, j) of each pair (gpl_pairs_copy_distance) */
int gpl_dwithin_join_pairs(gpl_ctx *ctx, const gpl_nearest_index *idx, const gpl_array *lhs, double distance, int with_distance,
                           gpl_pairs **out);
/* the distance of each pair of a list built with distances (any other list: GPL_ERR_INVALID_ARG); distance[n] in `mem`.
 * For a list from gpl_overlay_area_join the value of each pair is its intersection area, from gpl_overlay_length_join its
 * intersection length. */
int gpl_pairs_copy_distance(gpl_ctx *ctx, const gpl_pairs *pairs, double *distance, int mem);

/* ---------------------------------------------------------------- intersection area ------ */
/* Area of the intersection of the closed regions a[i] and b[i] (geo's BooleanOps::intersection(..).unsigned_area(); only the
 * area is computed, never the intersection polygons), DESIGN.md §4.16.  Both columns Polygon or MultiPolygon, in any
 * combination (else GPL_ERR_INVALID_TYPE); unequal lengths: GPL_ERR_LENGTH_MISMATCH.  Rings are used whatever their stored
 * orientation; unclosed rings are closed as Polygon::new does; a ring with fewer than 4 coordinates after closing contributes
 * nothing.  A null row, or a row with a non-finite coordinate, gives null (NaN, validity 0); an empty geometry gives 0.  The
 * value is never negative, and exactly 0.0 when no edges cross and no vertex of either side lies inside the other.  The
 * operands must be valid (OGC): on invalid input the value is finite but not specified.  out[n] f64, out_validity bitmap (may be
 * NULL), both in `mem`.  Deterministic. */
int gpl_intersection_area(gpl_ctx *ctx, const gpl_array *a, const gpl_array *b, double *out, uint8_t *out_validity, int mem);
/* Area-weighted overlay join of two (Multi)Polygon columns: every pair (i, j) whose closed geometries intersect — exactly the
 * pairs for which gpl_intersects(lhs[i], rhs[j]) is true, touching pairs included — with the area of lhs[i] ∩ rhs[j], bit for
 * bit what gpl_intersection_area returns for that row pair (lhs as the first operand).  Touching pairs carry 0 (or rounding
 * noise clamped at 0), so the areas of the pairs of a row over a partition sum to the row's area.  A device-resident gpl_pairs
 * sorted by (lhs, rhs); the area of each pair is read with gpl_pairs_copy_distance.  Fewer than 2^31 rows per side (else
 * GPL_ERR_UNSUPPORTED); any other type: GPL_ERR_INVALID_TYPE. */
int gpl_overlay_area_join(gpl_ctx *ctx, const gpl_array *lhs, const gpl_array *rhs, gpl_pairs **out);

/* ---------------------------------------------------------------- boolean geometry ------- */
enum { GPL_BOOLEAN_INTERSECTION = 0, GPL_BOOLEAN_UNION = 1, GPL_BOOLEAN_DIFFERENCE = 2, GPL_BOOLEAN_SYMMETRIC_DIFFERENCE = 3 };
/* Intersection, union, difference (a - b) or symmetric difference ((a - b) ∪ (b - a)) of the closed regions a[i] and b[i]
 * (geo's BooleanOps::{intersection, union, difference, xor}), DESIGN.md §4.19 and §4.23: the regularised result (lower-dimensional contact is dropped) as a MultiPolygon column, always.
 * Both columns Polygon or MultiPolygon, in any combination (else GPL_ERR_INVALID_TYPE); unequal lengths: GPL_ERR_LENGTH_MISMATCH;
 * any other op: GPL_ERR_INVALID_ARG; all before any launch.  Input rings are read as gpl_intersection_area reads them (any
 * orientation, closed implicitly, fewer than 4 coordinates after closing: no contribution).  A null row or a row with a
 * non-finite coordinate gives a null row; an empty result is an empty MultiPolygon.  Output: rings closed, shells
 * counter-clockwise and holes clockwise, each ring starting at its lexicographically smallest vertex, holes ordered by their first
 * vertex, members by their shell's first vertex; every cut point is a vertex; consecutive equal coordinates are merged and a
 * ring left with fewer than 3 distinct vertices is dropped (a shell with its holes).  Every combinatorial decision is an exact
 * sign except the assignment of holes to shells; only crossing points are rounded.  For valid (OGC) operands the output is valid;
 * on invalid operands it is a well-formed MultiPolygon column of bounded size whose geometry is not specified.  A row's output
 * depends on that row only, bit for bit. */
int gpl_boolean_op(gpl_ctx *ctx, const gpl_array *a, const gpl_array *b, int op, gpl_array **out);
/* Geometry overlay join of two (Multi)Polygon columns (GeoPandas' overlay(how="intersection"), keep_geom_type=True): every pair
 * (i, j) whose intersection has at least one member, sorted by (lhs, rhs), as a device-resident gpl_pairs; row k of *out (a
 * MultiPolygon column) is the intersection of pair k, bit for bit what gpl_boolean_op(lhs[i], rhs[j], GPL_BOOLEAN_INTERSECTION)
 * returns.  Candidates are the pairs gpl_intersects accepts; touching pairs are dropped.  Fewer than 2^31 rows per side (else
 * GPL_ERR_UNSUPPORTED); any other type: GPL_ERR_INVALID_TYPE. */
int gpl_overlay_join(gpl_ctx *ctx, const gpl_array *lhs, const gpl_array *rhs, gpl_pairs **pairs, gpl_array **out);
/* Dissolve (GeoPandas' dissolve(by=...), union_all(); geo's unary_union), DESIGN.md §4.21: row g of *out (a MultiPolygon
 * column of n_groups rows) is the regularised union of the closed rows whose group code is g.  group has in->n_geoms
 * entries in [-1, n_groups), in `mem` (gpl_mem); code -1 skips a row, as does a null row.  Rows are read as gpl_boolean_op
 * reads them; the output has its form (closed rings, counter-clockwise shells and clockwise holes starting at their smallest
 * vertex, holes and members in the same order, every cut point a vertex).  A row with a non-finite coordinate makes its group's
 * row null; a group with no present row is an empty MultiPolygon.  Every combinatorial decision is an exact sign for valid
 * (OGC) rows, only crossing points are rounded, and a group of exactly two present rows i < j is bit for bit
 * gpl_boolean_op(in[i], in[j], GPL_BOOLEAN_UNION) (one row: its union with an empty row).  Invalid rows give a well-formed
 * MultiPolygon column of bounded size whose geometry is not specified.  Deterministic.  Any other type: GPL_ERR_INVALID_TYPE;
 * a code outside [-1, n_groups) or n_groups < 0: GPL_ERR_INVALID_ARG; 2^31 or more rows or groups, or a group with 2^30 or more
 * boundary nodes: GPL_ERR_UNSUPPORTED. */
int gpl_dissolve(gpl_ctx *ctx, const gpl_array *in, const int64_t *group, int mem, int64_t n_groups, gpl_array **out);
enum {
    GPL_OVERLAY_INTERSECTION = 0,
    GPL_OVERLAY_UNION = 1,
    GPL_OVERLAY_IDENTITY = 2,
    GPL_OVERLAY_SYMMETRIC_DIFFERENCE = 3,
    GPL_OVERLAY_DIFFERENCE = 4,
};
/* Overlay of two (Multi)Polygon columns (GeoPandas' overlay(lhs, rhs, how), keep_geom_type=True), DESIGN.md §4.23.  The rows
 * are of three kinds:
 *   intersection rows (i, j): bit for bit the rows of gpl_overlay_join (how INTERSECTION, IDENTITY, UNION);
 *   left remainders (i, UINT64_MAX): lhs[i] minus the union of every rhs row it intersects (DIFFERENCE, IDENTITY,
 *   SYMMETRIC_DIFFERENCE, UNION);
 *   right remainders (UINT64_MAX, j): rhs[j] minus the union of every lhs row it intersects (SYMMETRIC_DIFFERENCE, UNION).
 * A remainder with no member is dropped; a null lhs / rhs row, or one with a non-finite coordinate, has no remainder and cuts
 * nothing.  A remainder with no cutter is bit for bit gpl_boolean_op(row, <empty row>, GPL_BOOLEAN_DIFFERENCE), and a left
 * remainder with one cutter gpl_boolean_op(lhs[i], rhs[j], GPL_BOOLEAN_DIFFERENCE) except where a crossing passes through a
 * vertex of another ring of the cutter.  *pairs is sorted by (lhs, rhs) as unsigned values (so a left row's intersections come
 * before its remainder, and the right remainders last); *out is one MultiPolygon column aligned with it, every row valid, in
 * gpl_boolean_op's output form.  Any other how: GPL_ERR_INVALID_ARG; any other type: GPL_ERR_INVALID_TYPE; 2^31 or more rows
 * in the two columns together: GPL_ERR_UNSUPPORTED; all before any launch.  A remainder with 2^30 or more boundary nodes:
 * GPL_ERR_UNSUPPORTED.  The operands must be valid (OGC); on invalid
 * operands the output is well formed but not specified.  Deterministic. */
int gpl_overlay(gpl_ctx *ctx, const gpl_array *lhs, const gpl_array *rhs, int how, gpl_pairs **pairs, gpl_array **out);

/* ---------------------------------------------------------------- clipping ---------------- */
/* Clip of a line or point column by a polygon column (GeoPandas' clip / overlay with lines, geo's BooleanOps::clip),
 * DESIGN.md §4.22.  a: LineString or MultiLineString (or, for gpl_clip and gpl_clip_join, Point or MultiPoint); b: Polygon or
 * MultiPolygon (any other pair: GPL_ERR_INVALID_TYPE); unequal lengths: GPL_ERR_LENGTH_MISMATCH; both before any launch.
 * invert = 0 keeps what lies in closed(b[i]) (its interior or boundary: pieces along a polygon edge are kept); invert != 0
 * keeps what lies strictly outside it.  Line output is a MultiLineString column: one member per maximal run of consecutive
 * kept pieces of one input chain, in input order (difference also splits a run at a point where the line touches the
 * boundary); runs are never joined across chains or across the start of a closed chain.  Every cut point is a vertex: a
 * crossing is a0 + t (a1 - a0) along the line's own segment, a polygon vertex on the line keeps its coordinates, input
 * vertices are copied bit for bit; consecutive equal coordinates are written once and a member left with fewer than 2
 * distinct points is dropped.  Point output is a MultiPoint column of the points of a[i] in closed(b[i]) (strictly outside
 * with invert), in input order, duplicates kept.  Polygon rings are read as gpl_boolean_op reads them; line chains in stored
 * order, never closed implicitly.  A null row or a row with a non-finite coordinate on either side gives a null row; an
 * empty result is an empty Multi* row.  Every in / on / out decision is an exact sign of input coordinates; only crossing
 * points are rounded.  The polygon operand must be valid (OGC): on invalid polygons the output is a well-formed column whose
 * geometry is not specified.  A row's output depends on that row only, bit for bit.  A row with 2^30 or more nodes:
 * GPL_ERR_UNSUPPORTED. */
int gpl_clip(gpl_ctx *ctx, const gpl_array *a, const gpl_array *b, int invert, gpl_array **out);
/* Length of the intersection of a (Multi)LineString row with closed(b[i]), computed without writing geometry: the f64 sum of
 * the kept pieces' lengths, >= 0, 0 when there is no 1-dimensional overlap; null (NaN, validity 0) under gpl_clip's rules.
 * Equal to the euclidean length of gpl_clip's row within a few ulps per piece.  out[n] f64, out_validity bitmap (may be
 * NULL), both in `mem`.  Types and errors as gpl_clip (point columns: GPL_ERR_INVALID_TYPE).  Deterministic. */
int gpl_clip_length(gpl_ctx *ctx, const gpl_array *a, const gpl_array *b, double *out, uint8_t *out_validity, int mem);
/* Geometry clip join of a line or point column with a (Multi)Polygon column: every pair (i, j) whose intersection has at
 * least one member (one point), sorted by (lhs, rhs), as a device-resident gpl_pairs; row k of *out (MultiLineString or
 * MultiPoint) is bit for bit gpl_clip(lhs[i], rhs[j], 0).  Candidates are the pairs gpl_intersects accepts; lines that only
 * touch are dropped.  A one-row rhs is GeoPandas' clip(lhs, mask).  Fewer than 2^31 rows per side (else GPL_ERR_UNSUPPORTED);
 * any other type: GPL_ERR_INVALID_TYPE.  *pairs and *out are set only on success. */
int gpl_clip_join(gpl_ctx *ctx, const gpl_array *lhs, const gpl_array *rhs, gpl_pairs **pairs, gpl_array **out);
/* Length-weighted overlay join of a (Multi)LineString column with a (Multi)Polygon column: every pair (i, j) for which
 * gpl_intersects(lhs[i], rhs[j]) is true, touching pairs included with length 0 (so the lengths of a line over a partition
 * sum to its length), with the length of lhs[i] in closed(rhs[j]), bit for bit what gpl_clip_length returns for that row
 * pair.  A device-resident gpl_pairs sorted by (lhs, rhs); the length of each pair is read with gpl_pairs_copy_distance.
 * Fewer than 2^31 rows per side (else GPL_ERR_UNSUPPORTED); any other type: GPL_ERR_INVALID_TYPE. */
int gpl_overlay_length_join(gpl_ctx *ctx, const gpl_array *lhs, const gpl_array *rhs, gpl_pairs **out);

/* ---------------------------------------------------------------- validity ---------------- */
/* OGC validity of every row, any geometry type, DESIGN.md §4.18: reason[n] (int8, in `mem`) is the first failing rule in the
 * order below, numbered as GEOS's TopologyValidationError except that 0 means valid:
 *   10 Invalid Coordinate: a NaN or infinite coordinate (a Point row that is exactly (NaN, NaN) is the empty point: valid);
 *    9 Too few distinct points in geometry component: a non-empty (Multi)LineString member with fewer than 2 distinct
 *      coordinates, or a non-empty ring with fewer than 3 distinct consecutive vertices;
 *    5 Self-intersection: two edges of the row's rings cross properly or overlap over a positive length (spikes, zero-area
 *      rings, shared edges of rings or members included);
 *    6 Ring Self-intersection: two non-adjacent edges of one ring touch at a point;
 *    2 Hole lies outside shell (also a non-empty hole of a polygon whose exterior ring is empty);
 *    3 Holes are nested;
 *    7 Nested shells: a MultiPolygon member lies in the interior of another (inside its hole is fine);
 *    4 Interior is disconnected: the rings of one polygon and their touch points form a cycle.
 * Points and MultiPoints fail only 10, (Multi)LineStrings only 10 and 9.  Rings are closed implicitly, consecutive repeated
 * coordinates are ignored ("adjacent" is among the non-degenerate edges, across the closing vertex too), orientation is
 * ignored; an empty geometry, a polygon without rings and a ring without coordinates are valid.  Every decision is an exact
 * sign of input coordinates, and a row's code depends on that row only.  A null row gets validity 0 in out_validity (Arrow
 * bitmap in `mem`, may be NULL) and reason 0.  NULL ctx, in or reason: GPL_ERR_INVALID_ARG before any launch. */
int gpl_is_valid(gpl_ctx *ctx, const gpl_array *in, int8_t *reason, uint8_t *out_validity, int mem);

/* ---------------------------------------------------------------- great-circle joins ----- */
/* Great-circle distance in metres of two POINT columns read as (lon, lat) degrees: geo 0.27 HaversineDistance on the mean
 * sphere (6 371 008.8 m), the expression gpl_geodesic_length(method 1) sums over segments, bit for bit.  Row-wise 1:1;
 * out[n] f64, out_validity bitmap (may be NULL).  A null or empty point gives a null row (NaN, validity 0); a non-finite
 * coordinate gives what the expression gives (NaN).  `a` is not clamped: within about 1e-8 rad of the antipode rounding can
 * push it above 1 and the result is NaN, as in geo.  Any other geometry type: GPL_ERR_INVALID_TYPE; unequal lengths:
 * GPL_ERR_LENGTH_MISMATCH. */
int gpl_haversine_distance(gpl_ctx *ctx, const gpl_array *lhs, const gpl_array *rhs, double *out, uint8_t *out_validity, int mem);
/* Joins of two POINT columns in (lon, lat) degrees by that distance (DESIGN.md 4.15).  d(i, j) is exactly the f64 that
 * gpl_haversine_distance returns for (lhs[i], rhs[j]).  A row of either side takes part only if it is non-null, non-empty,
 * finite and has |lat| <= 90 and |lon| <= 360 (so both the -180..180 and the 0..360 convention are accepted, and may be
 * mixed); no other row matches anything.  A NaN distance never matches.  Fewer than 2^31 rows on the right, and on the left
 * per call (else GPL_ERR_UNSUPPORTED); a non-POINT column: GPL_ERR_INVALID_TYPE; both checked before any launch.  Outputs
 * are deterministic (two calls give byte-identical results).  The index copies what it needs: `rhs` need not outlive it. */
int gpl_geo_index_build(gpl_ctx *ctx, const gpl_array *rhs, gpl_geo_index **out);
void gpl_geo_index_free(gpl_geo_index *idx);
/* synchronises the context stream: out8[0] = eligible right rows, [1] = ineligible rows, [2] = grid cells per axis,
 * [3] = columns and [4] = rows of cells in use (1 when the rows share one meridian / parallel), [5] = cell items, [6] = index
 * bytes, [7] = exact distance evaluations of the last query pass (a pair-list call runs two passes and leaves the count of
 * its second; concurrent queries of one index overwrite each other's count, never their results). */
int gpl_geo_index_stats(gpl_ctx *ctx, const gpl_geo_index *idx, int64_t *out8);
/* count[i] (int32, in `mem`) = number of right rows with d(i, j) <= distance (inclusive).  distance in metres, finite and
 * >= 0 (NaN, negative or +-inf -> GPL_ERR_INVALID_ARG before any launch) */
int gpl_geo_dwithin_count(gpl_ctx *ctx, const gpl_geo_index *idx, const gpl_array *lhs, double distance, int32_t *count, int mem);
/* every such pair once, sorted by (lhs, rhs), as a device-resident gpl_pairs; with_distance != 0 also keeps d(i, j) of each
 * pair (gpl_pairs_copy_distance) */
int gpl_geo_dwithin_join_pairs(gpl_ctx *ctx, const gpl_geo_index *idx, const gpl_array *lhs, double distance, int with_distance,
                               gpl_pairs **out);
/* the right rows at the minimum d(i, j) <= max_distance (metres, inclusive; +inf = unbounded; NaN or negative ->
 * GPL_ERR_INVALID_ARG); rows tie when their distances are equal f64 values.  nearest_id[i] = lowest tied row or -1,
 * distance[i] (may be NULL) = its distance or NaN, n_tied[i] (may be NULL) = number of tied rows; all in `mem`. */
int gpl_geo_nearest_join(gpl_ctx *ctx, const gpl_geo_index *idx, const gpl_array *lhs, double max_distance, int32_t *nearest_id,
                         double *distance, int32_t *n_tied, int mem);
/* every tied (left row, right row) pair once, sorted by (lhs, rhs); distance (may be NULL, in `mem`) receives the dense
 * distance of every left row (NaN: no match) */
int gpl_geo_nearest_join_pairs(gpl_ctx *ctx, const gpl_geo_index *idx, const gpl_array *lhs, double max_distance, gpl_pairs **out,
                               double *distance, int mem);

/* ---------------------------------------------------------------- synthetic data --------- */
/* device-side generators, bit-identical to geopolars_b200/synth.py (SURVEY.md §8d RNG) */
int gpl_gen_uniform_points(gpl_ctx *ctx, uint64_t stream_id, int64_t first, int64_t n, double scale, double *out_xy_dev);
int gpl_gen_walk_linestrings(gpl_ctx *ctx, uint64_t stream_id, int64_t other_of, int64_t first, int64_t n, int32_t k,
                             double *out_xy_dev, int64_t *out_geom_off_dev);
int gpl_gen_blob_polygons(gpl_ctx *ctx, uint64_t stream_id, int64_t first, int64_t n, int32_t nvert, double *out_xy_dev,
                          int64_t *out_ring_off_dev, int64_t *out_geom_off_dev);

#ifdef __cplusplus
}
#endif
#endif /* GEOPOLARS_B200_H */
