//! geoseries_b200.rs — `impl GeoSeries for Series` over libgeopolars_b200.so.
//!
//! Drop this file into `geopolars/geopolars-geo/src/` next to `geoseries.rs` and replace the placeholder bodies at
//! `geopolars/geopolars-geo/src/geoseries.rs:183-279` (`impl GeoSeries for Series`) by `mod geoseries_b200;`.  Every
//! method of the trait (`geoseries.rs:10-181`) is implemented here by the same three steps: export the Series' single
//! chunk through the Arrow C Data Interface (the calls the reference already uses between Python and Rust,
//! `py-geopolars/src/ffi.rs:36-41`), call one `extern "C"` entry point of `include/geopolars_b200.h`, import the result
//! (`ffi.rs:28-29`).  A WKB `BinaryArray` column (`util.rs:27-37`) is accepted as it is: the library decodes it on the GPU
//! once per call instead of once per row.
//!
//! NOT compiled in the authoring image (no rustc / cargo there); it is written against polars 0.3x's re-export of arrow2
//! (`polars::export::arrow::ffi`), the crate versions pinned by the reference's `Cargo.lock`.
//!
//! Additions to the trait surface (north_star: contains / intersects, absent from `geoseries.rs`): `GeoSeriesB200Ext`.
#![allow(clippy::missing_safety_doc)]

use crate::error::{GeopolarsError, Result};
use crate::geoseries::GeoSeries;
use crate::ops::affine::TransformOrigin; // referenced by py-geopolars/src/utils.rs:2,17-23
use crate::ops::length::GeodesicLengthMethod; // referenced by py-geopolars/src/geo.rs:5,64-67
use geo::algorithm::affine_ops::AffineTransform;
use polars::export::arrow::array::{ArrayRef, BooleanArray, PrimitiveArray};
use polars::export::arrow::bitmap::Bitmap;
use polars::export::arrow::datatypes::Field as ArrowField;
use polars::export::arrow::ffi::{self, ArrowArray, ArrowSchema};
use polars::prelude::*;
use std::cell::RefCell;
use std::ffi::CStr;
use std::os::raw::{c_char, c_int, c_void};

// ---------------------------------------------------------------------------------------------------------------
// the C ABI (include/geopolars_b200.h)
// ---------------------------------------------------------------------------------------------------------------
#[repr(C)]
pub struct GplCtx {
    _p: [u8; 0],
}
#[repr(C)]
pub struct GplArray {
    _p: [u8; 0],
}
#[repr(C)]
pub struct GplPairs {
    _p: [u8; 0],
}
#[repr(C)]
pub struct GplNearestIndex {
    _p: [u8; 0],
}

const GPL_HOST: c_int = 0;
const GPL_ORIGIN_CENTROID: c_int = 0;
const GPL_ORIGIN_CENTER: c_int = 1;
const GPL_ORIGIN_POINT: c_int = 2;
pub const GPL_PREDICATE_INTERSECTS: c_int = 0;
pub const GPL_PREDICATE_CONTAINS: c_int = 1;

#[link(name = "geopolars_b200")]
extern "C" {
    fn gpl_last_error() -> *const c_char;
    fn gpl_ctx_create(device: c_int, stream: *mut c_void, out: *mut *mut GplCtx) -> c_int;
    fn gpl_ctx_destroy(ctx: *mut GplCtx);
    fn gpl_array_import_arrow(ctx: *mut GplCtx, array: *const ArrowArray, schema: *const ArrowSchema, out: *mut *mut GplArray) -> c_int;
    fn gpl_array_export_arrow(ctx: *mut GplCtx, a: *const GplArray, out_array: *mut ArrowArray, out_schema: *mut ArrowSchema) -> c_int;
    fn gpl_array_free(a: *mut GplArray);
    fn gpl_affine_transform(ctx: *mut GplCtx, a: *const GplArray, a_: f64, b: f64, xoff: f64, d: f64, e: f64, yoff: f64, out: *mut *mut GplArray) -> c_int;
    fn gpl_translate(ctx: *mut GplCtx, a: *const GplArray, xoff: f64, yoff: f64, out: *mut *mut GplArray) -> c_int;
    fn gpl_scale(ctx: *mut GplCtx, a: *const GplArray, xfact: f64, yfact: f64, origin: c_int, ox: f64, oy: f64, out: *mut *mut GplArray) -> c_int;
    fn gpl_rotate(ctx: *mut GplCtx, a: *const GplArray, angle_deg: f64, origin: c_int, ox: f64, oy: f64, out: *mut *mut GplArray) -> c_int;
    fn gpl_skew(ctx: *mut GplCtx, a: *const GplArray, xs_deg: f64, ys_deg: f64, origin: c_int, ox: f64, oy: f64, out: *mut *mut GplArray) -> c_int;
    fn gpl_area(ctx: *mut GplCtx, a: *const GplArray, out: *mut f64, mem: c_int) -> c_int;
    fn gpl_centroid(ctx: *mut GplCtx, a: *const GplArray, out: *mut *mut GplArray) -> c_int;
    fn gpl_envelope(ctx: *mut GplCtx, a: *const GplArray, out: *mut *mut GplArray, out4: *mut f64, mem: c_int) -> c_int;
    fn gpl_euclidean_length(ctx: *mut GplCtx, a: *const GplArray, out: *mut f64, mem: c_int) -> c_int;
    fn gpl_geodesic_length(ctx: *mut GplCtx, a: *const GplArray, method: c_int, out: *mut f64, out_validity: *mut u8, mem: c_int) -> c_int;
    fn gpl_convex_hull(ctx: *mut GplCtx, a: *const GplArray, out: *mut *mut GplArray) -> c_int;
    fn gpl_simplify(ctx: *mut GplCtx, a: *const GplArray, tolerance: f64, out: *mut *mut GplArray) -> c_int;
    fn gpl_distance(ctx: *mut GplCtx, a: *const GplArray, b: *const GplArray, out: *mut f64, out_validity: *mut u8, mem: c_int) -> c_int;
    fn gpl_intersects(ctx: *mut GplCtx, a: *const GplArray, b: *const GplArray, out_bitmap: *mut u8, mem: c_int) -> c_int;
    fn gpl_contains(ctx: *mut GplCtx, a: *const GplArray, points: *const GplArray, out_bitmap: *mut u8, mem: c_int) -> c_int;
    fn gpl_contains_polygon(ctx: *mut GplCtx, a: *const GplArray, b: *const GplArray, out_bitmap: *mut u8, mem: c_int) -> c_int;
    fn gpl_geom_type(ctx: *mut GplCtx, a: *const GplArray, out: *mut i8, mem: c_int) -> c_int;
    fn gpl_is_empty(ctx: *mut GplCtx, a: *const GplArray, out_bitmap: *mut u8, mem: c_int) -> c_int;
    fn gpl_is_ring(ctx: *mut GplCtx, a: *const GplArray, out_bitmap: *mut u8, mem: c_int) -> c_int;
    fn gpl_x(ctx: *mut GplCtx, a: *const GplArray, out: *mut f64, mem: c_int) -> c_int;
    fn gpl_y(ctx: *mut GplCtx, a: *const GplArray, out: *mut f64, mem: c_int) -> c_int;
    fn gpl_exterior(ctx: *mut GplCtx, a: *const GplArray, out: *mut *mut GplArray) -> c_int;
    fn gpl_explode(ctx: *mut GplCtx, a: *const GplArray, out: *mut *mut GplArray) -> c_int;
    fn gpl_spatial_join(ctx: *mut GplCtx, lhs: *const GplArray, rhs: *const GplArray, predicate: c_int, out: *mut *mut GplPairs) -> c_int;
    fn gpl_pairs_count(pairs: *const GplPairs) -> i64;
    fn gpl_pairs_copy(ctx: *mut GplCtx, pairs: *const GplPairs, lhs: *mut u64, rhs: *mut u64, mem: c_int) -> c_int;
    fn gpl_pairs_free(pairs: *mut GplPairs);
    fn gpl_nearest_index_build(ctx: *mut GplCtx, rhs: *const GplArray, out: *mut *mut GplNearestIndex) -> c_int;
    fn gpl_nearest_index_free(idx: *mut GplNearestIndex);
    fn gpl_nearest_join_pairs_array(ctx: *mut GplCtx, idx: *const GplNearestIndex, points: *const GplArray, max_distance: f64, out: *mut *mut GplPairs, distance: *mut f64, mem: c_int) -> c_int;
}

// ---------------------------------------------------------------------------------------------------------------
// errors: status code + gpl_last_error() -> GeopolarsError (error.rs:9-30)
// ---------------------------------------------------------------------------------------------------------------
fn check(rc: c_int) -> Result<()> {
    if rc == 0 {
        return Ok(());
    }
    let msg = unsafe { CStr::from_ptr(gpl_last_error()) }.to_string_lossy().into_owned();
    Err(match rc {
        // GPL_ERR_INVALID_TYPE: the library's message is already "Expected X (found Y)" (error.rs:11-16)
        -1 => GeopolarsError::MismatchedGeometry { expected: leak(expected_of(&msg)), found: leak(found_of(&msg)) },
        // GPL_ERR_LENGTH_MISMATCH
        -2 => PolarsError::ShapeMismatch(msg.into()).into(),
        // GPL_ERR_CUDA / NCCL / OOM / UNSUPPORTED / INVALID_ARG
        _ => PolarsError::ComputeError(msg.into()).into(),
    })
}
fn expected_of(msg: &str) -> String {
    msg.strip_prefix("Expected ").and_then(|m| m.split(" (found ").next()).unwrap_or(msg).to_string()
}
fn found_of(msg: &str) -> String {
    msg.split(" (found ").nth(1).map(|m| m.trim_end_matches(')').to_string()).unwrap_or_default()
}
fn leak(s: String) -> &'static str {
    Box::leak(s.into_boxed_str()) // MismatchedGeometry carries &'static str; error paths only
}

// ---------------------------------------------------------------------------------------------------------------
// context: one per host thread (the trait methods are single-threaded and blocking, like the reference)
// ---------------------------------------------------------------------------------------------------------------
struct CtxHandle(*mut GplCtx);
impl Drop for CtxHandle {
    fn drop(&mut self) {
        unsafe { gpl_ctx_destroy(self.0) }
    }
}
thread_local! {
    static CTX: RefCell<Option<CtxHandle>> = RefCell::new(None);
}
/// The thread's device context (device from GEOPOLARS_B200_DEVICE, default 0; a private non-blocking stream).
fn ctx() -> Result<*mut GplCtx> {
    CTX.with(|c| {
        let mut c = c.borrow_mut();
        if c.is_none() {
            let device = std::env::var("GEOPOLARS_B200_DEVICE").ok().and_then(|v| v.parse().ok()).unwrap_or(0);
            let mut h = std::ptr::null_mut();
            check(unsafe { gpl_ctx_create(device, std::ptr::null_mut(), &mut h) })?; // fails loudly without a GPU: no CPU fallback
            *c = Some(CtxHandle(h));
        }
        Ok(c.as_ref().unwrap().0)
    })
}

// ---------------------------------------------------------------------------------------------------------------
// Series <-> device array through the Arrow C Data Interface
// ---------------------------------------------------------------------------------------------------------------
struct Dev(*mut GplArray);
impl Drop for Dev {
    fn drop(&mut self) {
        unsafe { gpl_array_free(self.0) }
    }
}
/// Series (rechunked to one chunk like ffi.rs:56) -> HBM.  The library borrows the buffers for the call only and never
/// calls `release` on them; dropping `c_arr` at the end of this function does (ffi.rs:10-11).
fn to_device(ctx: *mut GplCtx, s: &Series) -> Result<Dev> {
    let s = s.rechunk();
    let arr = s.to_arrow(0);
    let field = ArrowField::new(s.name(), arr.data_type().clone(), true);
    let c_arr = ffi::export_array_to_c(arr);
    let c_schema = ffi::export_field_to_c(&field);
    let mut h = std::ptr::null_mut();
    check(unsafe { gpl_array_import_arrow(ctx, &c_arr, &c_schema, &mut h) })?;
    Ok(Dev(h))
}
/// device geometry array -> Series named "geometry" (GeoArrow nested layout; buffers are library-owned pinned host
/// memory released through the ArrowArray's `release` callback)
fn from_device(ctx: *mut GplCtx, d: Dev) -> Result<Series> {
    let mut c_arr = ArrowArray::empty();
    let mut c_schema = ArrowSchema::empty();
    check(unsafe { gpl_array_export_arrow(ctx, d.0, &mut c_arr, &mut c_schema) })?;
    let field = unsafe { ffi::import_field_from_c(&c_schema) }.map_err(PolarsError::from)?; // ffi.rs:28
    let arr: ArrayRef = unsafe { ffi::import_array_from_c(c_arr, field.data_type) }.map_err(PolarsError::from)?; // ffi.rs:29
    Ok(Series::try_from(("geometry", arr))?)
}
type UnaryFn = unsafe extern "C" fn(*mut GplCtx, *const GplArray, *mut *mut GplArray) -> c_int;
/// geometry -> geometry ops without scalar arguments
fn unary(s: &Series, f: UnaryFn) -> Result<Series> {
    let ctx = ctx()?;
    let a = to_device(ctx, s)?;
    let mut out = std::ptr::null_mut();
    check(unsafe { f(ctx, a.0, &mut out) })?;
    from_device(ctx, Dev(out))
}
type F64Fn = unsafe extern "C" fn(*mut GplCtx, *const GplArray, *mut f64, c_int) -> c_int;
/// geometry -> Float64 column; null geometry rows stay null
fn unary_f64(s: &Series, name: &str, f: F64Fn) -> Result<Series> {
    let ctx = ctx()?;
    let a = to_device(ctx, s)?;
    let mut v = vec![0f64; s.len()];
    check(unsafe { f(ctx, a.0, v.as_mut_ptr(), GPL_HOST) })?;
    Ok(with_validity_of(s, Float64Chunked::from_vec(name, v).into_series()))
}
type BoolFn = unsafe extern "C" fn(*mut GplCtx, *const GplArray, *mut u8, c_int) -> c_int;
fn unary_bool(s: &Series, name: &str, f: BoolFn) -> Result<Series> {
    let ctx = ctx()?;
    let a = to_device(ctx, s)?;
    let mut bits = vec![0u8; (s.len() + 7) / 8];
    check(unsafe { f(ctx, a.0, bits.as_mut_ptr(), GPL_HOST) })?;
    Ok(bool_series(name, bits, s.len(), None))
}
fn bool_series(name: &str, bits: Vec<u8>, len: usize, validity: Option<Bitmap>) -> Series {
    let values = Bitmap::from_u8_vec(bits, len);
    let arr = BooleanArray::new(polars::export::arrow::datatypes::DataType::Boolean, values, validity);
    BooleanChunked::from_chunks(name, vec![Box::new(arr) as ArrayRef]).into_series()
}
fn f64_series(name: &str, v: Vec<f64>, validity_bits: Vec<u8>) -> Series {
    let len = v.len();
    let arr = PrimitiveArray::<f64>::new(polars::export::arrow::datatypes::DataType::Float64, v.into(), Some(Bitmap::from_u8_vec(validity_bits, len)));
    Float64Chunked::from_chunks(name, vec![Box::new(arr) as ArrayRef]).into_series()
}
/// copy the input's null mask onto a value column (area / length / x / y of a null geometry is null)
fn with_validity_of(input: &Series, out: Series) -> Series {
    match input.is_not_null() {
        mask if mask.all() => out,
        mask => out.zip_with(&mask, &Series::full_null(out.name(), out.len(), out.dtype())).unwrap_or(out),
    }
}
/// TransformOrigin (py-geopolars/src/utils.rs:5-27) -> (kind, x, y)
fn origin_args(origin: TransformOrigin) -> (c_int, f64, f64) {
    match origin {
        TransformOrigin::Centroid => (GPL_ORIGIN_CENTROID, 0.0, 0.0),
        TransformOrigin::Center => (GPL_ORIGIN_CENTER, 0.0, 0.0),
        TransformOrigin::Point(p) => (GPL_ORIGIN_POINT, p.x(), p.y()),
    }
}

// ---------------------------------------------------------------------------------------------------------------
// the trait (geoseries.rs:10-181), method for method
// ---------------------------------------------------------------------------------------------------------------
impl GeoSeries for Series {
    fn affine_transform(&self, matrix: impl Into<AffineTransform<f64>>) -> Result<Series> {
        let m: AffineTransform<f64> = matrix.into(); // named coefficients: no [f64; 6] order ambiguity
        let ctx = ctx()?;
        let a = to_device(ctx, self)?;
        let mut out = std::ptr::null_mut();
        check(unsafe { gpl_affine_transform(ctx, a.0, m.a(), m.b(), m.xoff(), m.d(), m.e(), m.yoff(), &mut out) })?;
        from_device(ctx, Dev(out))
    }

    fn area(&self) -> Result<Series> {
        unary_f64(self, "area", gpl_area)
    }

    fn centroid(&self) -> Result<Series> {
        unary(self, gpl_centroid)
    }

    fn convex_hull(&self) -> Result<Series> {
        unary(self, gpl_convex_hull)
    }

    fn envelope(&self) -> Result<Series> {
        let ctx = ctx()?;
        let a = to_device(ctx, self)?;
        let mut out = std::ptr::null_mut();
        check(unsafe { gpl_envelope(ctx, a.0, &mut out, std::ptr::null_mut(), GPL_HOST) })?;
        from_device(ctx, Dev(out))
    }

    fn euclidean_length(&self) -> Result<Series> {
        unary_f64(self, "euclidean_length", gpl_euclidean_length)
    }

    fn exterior(&self) -> Result<Series> {
        unary(self, gpl_exterior)
    }

    fn explode(&self) -> Result<Series> {
        unary(self, gpl_explode)
    }

    fn geodesic_length(&self, method: GeodesicLengthMethod) -> Result<Series> {
        let m = match method {
            GeodesicLengthMethod::Geodesic => 0,
            GeodesicLengthMethod::Haversine => 1,
            GeodesicLengthMethod::Vincenty => 2,
        };
        let ctx = ctx()?;
        let a = to_device(ctx, self)?;
        let mut v = vec![0f64; self.len()];
        let mut valid = vec![0u8; (self.len() + 7) / 8]; // a row Vincenty cannot converge on is null (geo returns Err)
        check(unsafe { gpl_geodesic_length(ctx, a.0, m, v.as_mut_ptr(), valid.as_mut_ptr(), GPL_HOST) })?;
        Ok(f64_series("geodesic_length", v, valid))
    }

    fn geom_type(&self) -> Result<Series> {
        let ctx = ctx()?;
        let a = to_device(ctx, self)?;
        let mut v = vec![0i8; self.len()]; // -1 missing, 0 Point .. 7 GeometryCollection (geoseries.rs:60-73)
        check(unsafe { gpl_geom_type(ctx, a.0, v.as_mut_ptr(), GPL_HOST) })?;
        Ok(Int8Chunked::from_vec("geom_type", v).into_series())
    }

    fn is_empty(&self) -> Result<Series> {
        unary_bool(self, "is_empty", gpl_is_empty)
    }

    fn is_ring(&self) -> Result<Series> {
        unary_bool(self, "is_ring", gpl_is_ring)
    }

    fn rotate(&self, angle: f64, origin: TransformOrigin) -> Result<Series> {
        let (k, ox, oy) = origin_args(origin);
        let ctx = ctx()?;
        let a = to_device(ctx, self)?;
        let mut out = std::ptr::null_mut();
        check(unsafe { gpl_rotate(ctx, a.0, angle, k, ox, oy, &mut out) })?;
        from_device(ctx, Dev(out))
    }

    fn scale(&self, xfact: f64, yfact: f64, origin: TransformOrigin) -> Result<Series> {
        let (k, ox, oy) = origin_args(origin);
        let ctx = ctx()?;
        let a = to_device(ctx, self)?;
        let mut out = std::ptr::null_mut();
        check(unsafe { gpl_scale(ctx, a.0, xfact, yfact, k, ox, oy, &mut out) })?;
        from_device(ctx, Dev(out))
    }

    fn simplify(&self, tolerance: f64) -> Result<Series> {
        let ctx = ctx()?;
        let a = to_device(ctx, self)?;
        let mut out = std::ptr::null_mut();
        check(unsafe { gpl_simplify(ctx, a.0, tolerance, &mut out) })?;
        from_device(ctx, Dev(out))
    }

    fn skew(&self, xs: f64, ys: f64, origin: TransformOrigin) -> Result<Series> {
        let (k, ox, oy) = origin_args(origin);
        let ctx = ctx()?;
        let a = to_device(ctx, self)?;
        let mut out = std::ptr::null_mut();
        check(unsafe { gpl_skew(ctx, a.0, xs, ys, k, ox, oy, &mut out) })?;
        from_device(ctx, Dev(out))
    }

    fn distance(&self, other: &Series) -> Result<Series> {
        let ctx = ctx()?;
        let (a, b) = (to_device(ctx, self)?, to_device(ctx, other)?);
        let mut v = vec![0f64; self.len()];
        let mut valid = vec![0u8; (self.len() + 7) / 8];
        check(unsafe { gpl_distance(ctx, a.0, b.0, v.as_mut_ptr(), valid.as_mut_ptr(), GPL_HOST) })?; // length mismatch -> ShapeMismatch
        Ok(f64_series("distance", v, valid))
    }

    #[cfg(feature = "proj")]
    fn to_crs(&self, from: &str, to: &str) -> Result<Series> {
        crate::ops::proj::to_crs(self, from, to) // PROJ stays on the host (ops/proj.rs): not on the GPU path
    }

    #[cfg(feature = "proj")]
    fn to_crs_with_options(&self, from: &str, to: &str, proj_options: crate::ops::proj::ProjOptions) -> Result<Series> {
        crate::ops::proj::to_crs_with_options(self, from, to, proj_options)
    }

    fn translate(&self, x: f64, y: f64) -> Result<Series> {
        let ctx = ctx()?;
        let a = to_device(ctx, self)?;
        let mut out = std::ptr::null_mut();
        check(unsafe { gpl_translate(ctx, a.0, x, y, &mut out) })?;
        from_device(ctx, Dev(out))
    }

    fn x(&self) -> Result<Series> {
        unary_f64(self, "x", gpl_x)
    }

    fn y(&self) -> Result<Series> {
        unary_f64(self, "y", gpl_y)
    }
}

// ---------------------------------------------------------------------------------------------------------------
// additions named by the north star (absent from the reference's trait): row-wise predicates and the join
// ---------------------------------------------------------------------------------------------------------------
pub trait GeoSeriesB200Ext {
    /// row-wise `geo::Intersects` for every pair of (Multi)Point / (Multi)LineString / (Multi)Polygon columns
    fn intersects(&self, other: &Series) -> Result<Series>;
    /// row-wise contains: (Multi)Polygon / (Multi)LineString x Point, or (Multi)Polygon x Polygon — the pairs
    /// `spatial_join` dispatches (geopolars/src/spatial_index.rs:89-135)
    fn contains(&self, other: &Series) -> Result<Series>;
    /// the (lhs_index, rhs_index) pair list of `spatial_join(lhs, rhs, SpatialJoinArgs { predicate, .. })`
    /// (spatial_index.rs:139-157) for any two geometry columns; feed it to the DataFrame joins at :159-203
    fn spatial_join_pairs(&self, rhs: &Series, predicate: c_int) -> Result<(Vec<u64>, Vec<u64>)>;
    /// nearest-geometry join of this Point column against any geometry column (GeoPandas' `sjoin_nearest`): every
    /// right row at the minimum distance <= `max_distance` (inclusive, `f64::INFINITY` = unbounded), as (lhs_index,
    /// rhs_index, distance) sorted by (lhs, rhs); the distance is exactly what `distance` computes for the pair
    fn nearest_join_pairs(&self, rhs: &Series, max_distance: f64) -> Result<(Vec<u64>, Vec<u64>, Vec<f64>)>;
}

impl GeoSeriesB200Ext for Series {
    fn intersects(&self, other: &Series) -> Result<Series> {
        let ctx = ctx()?;
        let (a, b) = (to_device(ctx, self)?, to_device(ctx, other)?);
        let mut bits = vec![0u8; (self.len() + 7) / 8];
        check(unsafe { gpl_intersects(ctx, a.0, b.0, bits.as_mut_ptr(), GPL_HOST) })?;
        Ok(bool_series("intersects", bits, self.len(), None))
    }

    fn contains(&self, other: &Series) -> Result<Series> {
        let ctx = ctx()?;
        let (a, b) = (to_device(ctx, self)?, to_device(ctx, other)?);
        let mut bits = vec![0u8; (self.len() + 7) / 8];
        // the library tells the two families apart by the type of `other`; try the point form first
        let rc = unsafe { gpl_contains(ctx, a.0, b.0, bits.as_mut_ptr(), GPL_HOST) };
        if rc == -1 {
            check(unsafe { gpl_contains_polygon(ctx, a.0, b.0, bits.as_mut_ptr(), GPL_HOST) })?;
        } else {
            check(rc)?;
        }
        Ok(bool_series("contains", bits, self.len(), None))
    }

    fn spatial_join_pairs(&self, rhs: &Series, predicate: c_int) -> Result<(Vec<u64>, Vec<u64>)> {
        let ctx = ctx()?;
        let (a, b) = (to_device(ctx, self)?, to_device(ctx, rhs)?);
        let mut pairs = std::ptr::null_mut();
        check(unsafe { gpl_spatial_join(ctx, a.0, b.0, predicate, &mut pairs) })?;
        let n = unsafe { gpl_pairs_count(pairs) } as usize;
        let (mut l, mut r) = (vec![0u64; n], vec![0u64; n]);
        let rc = if n > 0 { unsafe { gpl_pairs_copy(ctx, pairs, l.as_mut_ptr(), r.as_mut_ptr(), GPL_HOST) } } else { 0 };
        unsafe { gpl_pairs_free(pairs) };
        check(rc)?;
        Ok((l, r))
    }

    fn nearest_join_pairs(&self, rhs: &Series, max_distance: f64) -> Result<(Vec<u64>, Vec<u64>, Vec<f64>)> {
        let ctx = ctx()?;
        let (a, b) = (to_device(ctx, self)?, to_device(ctx, rhs)?);
        let mut idx = std::ptr::null_mut();
        check(unsafe { gpl_nearest_index_build(ctx, b.0, &mut idx) })?;
        let mut dist = vec![0f64; self.len()];
        let mut pairs = std::ptr::null_mut();
        let rc = unsafe { gpl_nearest_join_pairs_array(ctx, idx, a.0, max_distance, &mut pairs, dist.as_mut_ptr(), GPL_HOST) };
        unsafe { gpl_nearest_index_free(idx) };
        if rc != 0 && !pairs.is_null() {
            unsafe { gpl_pairs_free(pairs) };
        }
        check(rc)?;
        let n = unsafe { gpl_pairs_count(pairs) } as usize;
        let (mut l, mut r) = (vec![0u64; n], vec![0u64; n]);
        let rc = if n > 0 { unsafe { gpl_pairs_copy(ctx, pairs, l.as_mut_ptr(), r.as_mut_ptr(), GPL_HOST) } } else { 0 };
        unsafe { gpl_pairs_free(pairs) };
        check(rc)?;
        let d = l.iter().map(|&i| dist[i as usize]).collect();
        Ok((l, r, d))
    }
}
