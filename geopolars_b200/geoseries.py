"""GeoSeries + `.geo` accessor: the user-facing surface of the reference, on the CUDA engine.

Mirrors py-geopolars/python/geopolars/internals/geoseries.py:33-54 (`GeoSeries`, `.geo`) and
py-geopolars/python/geopolars/internals/georust/geoseries.py:16-320 (`GeoRustSeries`: 18 methods and
properties forwarding to `_geopolars.geo.*`).  Same names, same argument meaning, same error classes;
differences forced by this environment are stated where they occur:
  * polars is not installed here, so a GeoSeries wraps a pyarrow array and scalar results are pyarrow
    arrays (the reference returns polars Series via `polars.from_arrow`, ffi.rs:84-87);
  * the accessor passes the SERIES to the engine (the reference passes the accessor object itself,
    a latent bug: georust/geoseries.py:41, SURVEY.md §3A);
  * `contains` / `intersects` / `spatial_join` are additions to the surface (they exist in the
    reference only in the uncompiled geopolars/src/spatial_index.rs).
Every operation runs in libgeopolars_b200.so on the GPU; nothing here computes geometry on the CPU.
"""
from __future__ import annotations

import threading
from dataclasses import dataclass
from typing import Optional, Sequence, Union

import numpy as np

from . import engine as E
from .geoarrow import GeometryType

_ctx_lock = threading.Lock()
_default_ctx: Optional[E.Context] = None


def get_context(device: int = 0) -> E.Context:
    """process-wide default engine context on `device` (created on first use; fails loudly without a GPU)"""
    global _default_ctx
    with _ctx_lock:
        if _default_ctx is None:
            _default_ctx = E.Context(device)
        return _default_ctx


def set_context(ctx: E.Context) -> None:
    global _default_ctx
    with _ctx_lock:
        _default_ctx = ctx


AffineTransform = Sequence[float]
TransformOrigin = Union[str, tuple, dict]


def _pa():
    import pyarrow as pa

    return pa


class GeoSeries:
    """A geometry column.  Holds the Arrow data on the host and, once touched by an op, its GeoArrow
    buffers in HBM (copied once, reused by every subsequent op — the reference re-parses WKB per op)."""

    def __init__(self, data=None, *, _device: Optional[E.DeviceArray] = None, name: str = "geometry"):
        self.name = name
        self._arrow = None
        self._device = _device
        if data is not None:
            pa = _pa()
            if isinstance(data, GeoSeries):
                self._arrow, self._device = data._arrow, data._device
            elif isinstance(data, (pa.Array, pa.ChunkedArray)):
                self._arrow = data
            else:  # iterable of WKB bytes / None
                self._arrow = pa.array(list(data), type=pa.binary())

    # -- plumbing -----------------------------------------------------------------------------------
    @property
    def device(self) -> E.DeviceArray:
        if self._device is None:
            self._device = get_context().import_arrow(self._arrow)
        return self._device

    def to_arrow(self):
        """geoarrow-nested pyarrow array (interleaved coordinates)"""
        if self._arrow is not None:
            pa = _pa()
            t = self._arrow.type
            if not (pa.types.is_binary(t) or pa.types.is_large_binary(t)):
                return self._arrow
        return self.device.to_arrow()

    def to_wkb(self):
        return self.device.to_wkb()

    def __len__(self) -> int:
        return len(self._arrow) if self._arrow is not None else len(self._device)

    def __repr__(self) -> str:
        return f"GeoSeries(name={self.name!r}, len={len(self)})"

    # -- accessors (geoseries.py:48-54) ---------------------------------------------------------------
    @property
    def geo(self) -> "GeoRustSeries":
        return GeoRustSeries(series=self)

    @property
    def geos(self):
        """the reference's GEOS namespace is empty (internals/geos/geoseries.py:6-16)"""
        raise NotImplementedError("the GEOS backend has no operations in the reference either")


class GeoDataFrame:
    """The reference's GeoDataFrame (py-geopolars/python/geopolars/internals/geodataframe.py) is a polars DataFrame
    whose `geometry` column is a GeoSeries; polars is not installed here, so this one wraps a pyarrow Table: `geometry`
    (a GeoSeries whose buffers move to HBM on first use), `columns`, `shape`, `__getitem__`, `to_arrow`."""

    def __init__(self, table, geometry: str = "geometry"):
        pa = _pa()
        if isinstance(table, GeoDataFrame):
            table = table._table
        if not isinstance(table, pa.Table):
            raise TypeError("GeoDataFrame expects a pyarrow.Table")
        if geometry not in table.column_names:
            raise ValueError(f"no '{geometry}' column (columns: {', '.join(table.column_names)})")
        self._table = table
        self._geometry_name = geometry
        self._geometry: Optional[GeoSeries] = None

    @property
    def geometry(self) -> GeoSeries:
        if self._geometry is None:
            self._geometry = GeoSeries(self._table.column(self._geometry_name), name=self._geometry_name)
        return self._geometry

    @property
    def columns(self):
        return list(self._table.column_names)

    @property
    def shape(self):
        return (self._table.num_rows, self._table.num_columns)

    def __len__(self) -> int:
        return self._table.num_rows

    def __getitem__(self, name: str):
        return self.geometry if name == self._geometry_name else self._table.column(name)

    def to_arrow(self):
        return self._table

    def __repr__(self) -> str:
        return f"GeoDataFrame(shape={self.shape}, columns={self.columns})"


def from_arrow(data):
    """geopolars.from_arrow (py-geopolars/python/geopolars/convert.py:33-56): a Table becomes a GeoDataFrame, an Array or
    ChunkedArray a GeoSeries"""
    pa = _pa()
    if isinstance(data, pa.Table):
        return GeoDataFrame(data)
    return GeoSeries(data)


def _f64(values: np.ndarray, valid: Optional[np.ndarray] = None):
    pa = _pa()
    if valid is not None and not valid.all():
        return pa.array(values, mask=~valid)
    return pa.array(values)


def _valid_bits(d: E.DeviceArray) -> Optional[np.ndarray]:
    gt = E.geom_type(d)
    valid = gt >= 0
    return None if valid.all() else valid


@dataclass
class GeoRustSeries:
    """`GeoSeries.geo` — same 18 entry points as georust/geoseries.py:22-320."""

    series: GeoSeries

    def _d(self) -> E.DeviceArray:
        return self.series.device

    def _wrap(self, d: E.DeviceArray) -> GeoSeries:
        return GeoSeries(_device=d, name=self.series.name)

    def affine_transform(self, matrix: AffineTransform) -> GeoSeries:
        """The 6 numbers are handed to geo's `AffineTransform` unchanged, exactly as the reference binding does
        (py-geopolars/src/geo.rs:10-13 passes `[f64; 6]` into `impl Into<AffineTransform>`, whose
        `From<[T; 6]>` is `new(a, b, xoff, d, e, yoff)`): matrix = [a, b, xoff, d, e, yoff],
        x' = a*x + b*y + xoff, y' = d*x + e*y + yoff.  The reference's docstring
        (georust/geoseries.py:33) advertises shapely's order [a, b, d, e, xoff, yoff]; its executable path
        does not reorder, and parity follows the executable path (pinned by
        tests/test_gpu_formats.py::test_affine_matrix_order_is_geos)."""
        if len(matrix) != 6:
            raise ValueError("matrix must have 6 elements [a, b, xoff, d, e, yoff]")
        a, b, xoff, d, e, yoff = [float(v) for v in matrix]
        return self._wrap(E.affine_transform(self._d(), (a, b, xoff, d, e, yoff)))

    @property
    def area(self):
        d = self._d()
        return _f64(E.area(d), _valid_bits(d))

    @property
    def centroid(self) -> GeoSeries:
        return self._wrap(E.centroid(self._d()))

    def convex_hull(self) -> GeoSeries:
        return self._wrap(E.convex_hull(self._d()))

    def envelope(self) -> GeoSeries:
        return self._wrap(E.envelope(self._d()))

    def euclidean_length(self):
        d = self._d()
        return _f64(E.euclidean_length(d), _valid_bits(d))

    def exterior(self) -> GeoSeries:
        return self._wrap(E.exterior(self._d()))

    def explode(self) -> GeoSeries:
        return self._wrap(E.explode(self._d()))

    def geodesic_length(self, method: str = "geodesic"):
        if method.lower() not in ("geodesic", "haversine", "vincenty"):
            raise ValueError("Geodesic calculation method not valid. Use one of geodesic, haversine or vincenty")
        out, valid = E.geodesic_length(self._d(), method)
        return _f64(out, valid)

    @property
    def geom_type(self):
        return _pa().array(E.geom_type(self._d()))

    def is_empty(self):
        d = self._d()
        v = _valid_bits(d)
        pa = _pa()
        return pa.array(E.is_empty(d), mask=None if v is None else ~v)

    def is_ring(self):
        d = self._d()
        v = _valid_bits(d)
        pa = _pa()
        return pa.array(E.is_ring(d), mask=None if v is None else ~v)

    def rotate(self, angle: float, origin: TransformOrigin = "center") -> GeoSeries:
        return self._wrap(E.rotate(self._d(), angle, origin))

    def scale(self, xfact: float = 1.0, yfact: float = 1.0, origin: TransformOrigin = "center") -> GeoSeries:
        return self._wrap(E.scale(self._d(), xfact, yfact, origin))

    def skew(self, xs: float = 0.0, ys: float = 0.0, origin: TransformOrigin = "center") -> GeoSeries:
        return self._wrap(E.skew(self._d(), xs, ys, origin))

    def simplify(self, tolerance: float) -> GeoSeries:
        """Douglas-Peucker simplification (geoseries.rs:108-116); end points are always preserved"""
        return self._wrap(E.simplify(self._d(), tolerance))

    def distance(self, other: GeoSeries):
        out, valid = E.distance(self._d(), other.device)
        return _f64(out, valid)

    def translate(self, xoff: float = 0.0, yoff: float = 0.0) -> GeoSeries:
        return self._wrap(E.translate(self._d(), xoff, yoff))

    @property
    def x(self):
        d = self._d()
        return _f64(E.x(d), _valid_bits(d))

    @property
    def y(self):
        d = self._d()
        return _f64(E.y(d), _valid_bits(d))

    # -- additions: binary predicates (planned-only in the reference docs, geoseries.rst:47-64) ----------
    def contains(self, other: GeoSeries):
        """row-wise: self[i] ((Multi)Polygon or (Multi)LineString) contains other[i] (Point), or (Multi)Polygon contains Polygon"""
        return _pa().array(E.contains(self._d(), other.device))

    def intersects(self, other: GeoSeries):
        """row-wise geo `Intersects` for every pair of (Multi)Point / (Multi)LineString / (Multi)Polygon columns"""
        return _pa().array(E.intersects(self._d(), other.device))


def spatial_join(lhs: GeoSeries, rhs: GeoSeries, how: str = "inner", predicate: str = "intersects"):
    """spatial_join(lhs, rhs, SpatialJoinArgs{join_type, predicate}) (geopolars/src/spatial_index.rs:37-204): the
    (lhs_index, rhs_index) pairs the reference builds before its polars joins (:139-157), for any two geometry
    columns.  Candidates are the pairs whose envelopes intersect, the exact test is the reference's type-pair dispatch
    (:89-137; Point x (Multi)Polygon uses contains(point) whatever the predicate).  how='inner' -> matching pairs;
    how='left' -> every lhs row once per match, or once with rhs = -1 (null) when it has none — the row set of the
    reference's Left join (9 rows for the 9-point test, :483-484).  Points x (Multi)Polygons run on the points-in-polygons
    index (the north-star path) without moving the device-resident point column; everything else on gpl_spatial_join."""
    if how not in ("inner", "left"):
        raise ValueError("how must be 'inner' or 'left'")
    lt, rt = lhs.device.type, rhs.device.type
    if lt == E.GeometryType.POINT and rt in (E.GeometryType.POLYGON, E.GeometryType.MULTIPOLYGON):
        a, b = E.PipIndex(rhs.device).pairs_array(lhs.device)
    else:
        a, b = E.spatial_join(lhs.device, rhs.device, predicate)
    a = a.astype(np.int64)
    b = b.astype(np.int64)
    if how == "left":
        n = len(lhs)
        matched = np.zeros(n, dtype=bool)
        matched[a] = True
        miss = np.nonzero(~matched)[0]
        a = np.concatenate([a, miss])
        b = np.concatenate([b, np.full(len(miss), -1, dtype=np.int64)])
        order = np.lexsort((b, a))
        a, b = a[order], b[order]
    return a, b


def nearest_join(lhs: GeoSeries, rhs: GeoSeries, how: str = "inner", max_distance: Optional[float] = None):
    """Nearest-geometry join of a Point column against any geometry column (GeoPandas' sjoin_nearest with
    max_distance / distance_col): (lhs_index int64, rhs_index int64, distance float64), sorted by (lhs, rhs).  Every right
    row at the minimum distance is returned (ties are equal f64 distances, as GeoPandas returns all equidistant rows); the
    distance is exactly what `lhs.geo.distance` computes for the pair.  max_distance is inclusive (None: unbounded).
    how='inner' -> matched points only; how='left' -> unmatched points once, with rhs_index -1 and distance NaN."""
    if how not in ("inner", "left"):
        raise ValueError("how must be 'inner' or 'left'")
    idx = E.NearestIndex(rhs.device)
    try:
        a, b, dist = idx.pairs_array(lhs.device, max_distance, with_distance=True)
    finally:
        idx.free()
    a = a.astype(np.int64)
    b = b.astype(np.int64)
    d = dist[a]
    if how == "left":
        miss = np.nonzero(np.isnan(dist))[0]
        a = np.concatenate([a, miss])
        b = np.concatenate([b, np.full(len(miss), -1, dtype=np.int64)])
        d = np.concatenate([d, np.full(len(miss), np.nan)])
        order = np.lexsort((b, a))
        a, b, d = a[order], b[order], d[order]
    return a, b, d
