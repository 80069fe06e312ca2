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

    def dissolve(self, by: str) -> "GeoDataFrame":
        """GeoPandas' `dissolve(by=by)` with sort=True, dropna=True: one row per distinct non-null value of column `by`, in
        ascending order, with the union of the geometries of its rows (see `dissolve` below).  Only the `by` column and the
        geometry are returned: aggregating other columns (GeoPandas' `aggfunc`) is not done here; pyarrow's `Table.group_by`
        does it on the same keys."""
        pa = _pa()
        keys, geoms = dissolve(self.geometry, self._table.column(by))
        return GeoDataFrame(pa.table({by: keys, self._geometry_name: geoms.to_arrow()}), geometry=self._geometry_name)

    def overlay(self, other: "GeoDataFrame", how: str = "intersection") -> "GeoDataFrame":
        """GeoPandas' `overlay(self, other, how)` for two (Multi)Polygon frames, keep_geom_type=True (see `overlay` below): the
        left columns, then the right columns, then the geometry (named as this frame's).  A remainder row's other-side
        columns are null; a column name both frames have gets GeoPandas' suffixes, `_1` on the left and `_2` on the right, and
        a right column named as this frame's geometry gets `_2`.
        Attributes are not aggregated.  The rows are `overlay`'s, so their order differs from GeoPandas' (which concatenates
        its parts) but the set of rows is the same.  Both frames' geometries must be valid (OGC); `is_valid()` tells."""
        pa = _pa()
        a, b, geoms = overlay(self.geometry, other.geometry, how)
        lt = self._table.drop_columns([self._geometry_name])
        rt = other._table.drop_columns([other._geometry_name])
        lt = lt.take(pa.array(a, mask=a < 0))  # a null index takes a null row
        rt = rt.take(pa.array(b, mask=b < 0))
        common = set(lt.column_names) & set(rt.column_names)
        names = [n + "_1" if n in common else n for n in lt.column_names]
        names += [n + "_2" if n in common or n == self._geometry_name else n for n in rt.column_names]
        cols = list(lt.columns) + list(rt.columns) + [geoms.to_arrow()]
        return GeoDataFrame(pa.table(cols, names=names + [self._geometry_name]), geometry=self._geometry_name)


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

    def geodesic_area_signed(self):
        """geo's GeodesicArea::geodesic_area_signed on WGS84, square metres, for (lon, lat) degree columns (DESIGN.md §4.17):
        counter-clockwise exteriors positive, holes subtract.  Null for a null row, a non-finite coordinate or |lat| > 90"""
        area, _, valid = E.geodesic_area(self._d(), signed=True)
        return _f64(area, valid)

    def geodesic_area_unsigned(self):
        """geo's GeodesicArea::geodesic_area_unsigned on WGS84, square metres, in [0, area of the ellipsoid): a clockwise
        exterior gives the ellipsoid's area minus the enclosed area, as in geo.  Nulls as geodesic_area_signed"""
        area, _, valid = E.geodesic_area(self._d(), signed=False)
        return _f64(area, valid)

    def geodesic_perimeter(self):
        """geo's GeodesicArea::geodesic_perimeter on WGS84, metres: the closed geodesic length of every ring, holes included
        (geodesic_length uses the exterior only).  Nulls as geodesic_area_signed"""
        _, perimeter, valid = E.geodesic_area(self._d(), signed=True)
        return _f64(perimeter, valid)

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

    def is_valid(self):
        """OGC validity of every row (GeoPandas' `is_valid`, DESIGN.md §4.18), as exact decisions on the GPU; null rows give
        null.  Filter with it before `intersection_area`, `overlay_area_join` or Polygon `contains`, which need valid input"""
        reason, valid = E.is_valid(self._d())
        return _pa().array(reason == 0, mask=~valid)

    def is_valid_reason(self):
        """why each row is invalid (shapely's `explain_validity` without the location): "Valid Geometry" or GEOS's message
        of the first failing rule, e.g. "Self-intersection"; null rows give null"""
        reason, valid = E.is_valid(self._d())
        return _pa().array([E.VALIDITY_REASONS[int(c)] for c in reason], type=_pa().string(), mask=~valid)

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

    def dwithin(self, other: GeoSeries, distance: float):
        """row-wise `distance(self, other) <= distance` (GeoPandas' GeoSeries.dwithin); a null distance gives False"""
        out, valid = E.distance(self._d(), other.device)
        return _pa().array(valid.astype(bool) & (out <= float(distance)))

    def haversine_distance(self, other: GeoSeries):
        """row-wise great-circle distance in metres to `other`, both Point columns in (lon, lat) degrees (geo's
        HaversineDistance, mean earth radius 6 371 008.8 m); a null or empty point gives null"""
        out, valid = E.haversine_distance(self._d(), other.device)
        return _f64(out, valid)

    def intersection_area(self, other: GeoSeries):
        """row-wise area of the intersection of self[i] and other[i], both (Multi)Polygon columns (GeoPandas'
        `a.intersection(b).area`; only the area is computed, DESIGN.md §4.16).  Null when either row is null or has a
        non-finite coordinate; 0 for an empty geometry; never negative.  Rings may have any orientation and need not be
        closed.  The operands must be valid (OGC): on invalid input the value is finite but not specified; `is_valid()` tells."""
        out, valid = E.intersection_area(self._d(), other.device)
        return _f64(out, valid)

    def intersection(self, other: GeoSeries) -> GeoSeries:
        """row-wise intersection of self[i] and other[i], both (Multi)Polygon columns (GeoPandas' `a.intersection(b)`, geo's
        BooleanOps), as a MultiPolygon column (DESIGN.md §4.19).  Null when either row is null or has a non-finite coordinate;
        an empty result is an empty MultiPolygon.  Valid (OGC) operands give valid output; on invalid operands the output is
        well formed but not specified; `is_valid()` tells."""
        return self._wrap(E.boolean_op(self._d(), other.device, "intersection"))

    def union(self, other: GeoSeries) -> GeoSeries:
        """row-wise union of self[i] and other[i] (GeoPandas' `a.union(b)`), as `intersection`"""
        return self._wrap(E.boolean_op(self._d(), other.device, "union"))

    def difference(self, other: GeoSeries) -> GeoSeries:
        """row-wise difference self[i] - other[i] (GeoPandas' `a.difference(b)`), as `intersection`"""
        return self._wrap(E.boolean_op(self._d(), other.device, "difference"))

    def symmetric_difference(self, other: GeoSeries) -> GeoSeries:
        """row-wise symmetric difference of self[i] and other[i], the parts covered by exactly one of them (GeoPandas'
        `a.symmetric_difference(b)`, geo's `BooleanOps::xor`; DESIGN.md §4.23), as `intersection`.  Members of
        self[i] - other[i] and other[i] - self[i] that touch at a point stay separate members."""
        return self._wrap(E.boolean_op(self._d(), other.device, "symmetric_difference"))

    def clip(self, mask: GeoSeries, invert: bool = False) -> GeoSeries:
        """row-wise clip of self[i], a (Multi)LineString or (Multi)Point column, by mask[i], a (Multi)Polygon column
        (GeoPandas' `a.intersection(b)` for lines, geo's `BooleanOps::clip`; DESIGN.md §4.22): the parts of self[i] in the
        closed polygon (pieces along its boundary included), or with invert=True the parts strictly outside it, as a
        MultiLineString (MultiPoint) column.  Cut points are vertices and input vertices are kept bit for bit.  Null when
        either row is null or has a non-finite coordinate; an empty result is an empty row.  The polygons must be valid (OGC);
        `is_valid()` tells.  For GeoPandas' `clip(series, mask)` with one mask, use `clip_join` with a one-row mask column."""
        return self._wrap(E.clip(self._d(), mask.device, invert))

    def intersection_length(self, other: GeoSeries):
        """row-wise length of the part of self[i], a (Multi)LineString column, in the closed (Multi)Polygon other[i]
        (GeoPandas' `a.intersection(b).length`, without building the geometry; DESIGN.md §4.22).  Null when either row is null
        or has a non-finite coordinate; 0 when there is no overlap of positive length."""
        out, valid = E.clip_length(self._d(), other.device)
        return _f64(out, valid)

    def union_all(self) -> GeoSeries:
        """the union of every row, a (Multi)Polygon column, as a GeoSeries of one MultiPolygon row (GeoPandas'
        `union_all()`, formerly `unary_union`; DESIGN.md §4.21).  Null rows are skipped; a row with a non-finite coordinate
        makes the result null; no present row gives an empty MultiPolygon.  Valid (OGC) rows give valid output."""
        return self._wrap(E.union_all(self._d()))

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
        """row-wise: self[i] ((Multi)Polygon or (Multi)LineString) contains other[i] (Point), or (Multi)Polygon contains Polygon
        (defined for valid polygons: check with `is_valid()`)"""
        return _pa().array(E.contains(self._d(), other.device))

    def intersects(self, other: GeoSeries):
        """row-wise geo `Intersects` for every pair of (Multi)Point / (Multi)LineString / (Multi)Polygon columns"""
        return _pa().array(E.intersects(self._d(), other.device))

    # -- DE-9IM (DESIGN.md §4.20): any two of the six types; defined for valid (OGC) operands, a null row gives False --
    def relate(self, other: GeoSeries):
        """row-wise DE-9IM matrix of self[i] and other[i] as a string such as "FF2F11212" (rows: self's Interior, Boundary,
        Exterior; columns: other's); null when either row is null or has a non-finite coordinate"""
        m, valid = E.relate(self._d(), other.device)
        chars = np.array(list("F012"))[m.astype(np.int64) + 1]
        return _pa().array(["".join(r) if v else None for r, v in zip(chars, valid)], type=_pa().string())

    def relate_pattern(self, other: GeoSeries, pattern: str):
        """row-wise: the DE-9IM matrix matches `pattern`, 9 characters over T, F, *, 0, 1, 2 (either case; else ValueError)"""
        return _pa().array(E.relate_predicate(self._d(), other.device, "relate_pattern", pattern))

    def _pred(self, other: GeoSeries, name: str):
        return _pa().array(E.relate_predicate(self._d(), other.device, name))

    def within(self, other: GeoSeries):
        """row-wise DE-9IM within: T*F**F***"""
        return self._pred(other, "within")

    def covers(self, other: GeoSeries):
        """row-wise DE-9IM covers: T*****FF*, *T****FF*, ***T**FF* or ****T*FF*"""
        return self._pred(other, "covers")

    def covered_by(self, other: GeoSeries):
        """row-wise DE-9IM covered_by: T*F**F***, *TF**F***, **FT*F*** or **F*TF***"""
        return self._pred(other, "covered_by")

    def touches(self, other: GeoSeries):
        """row-wise DE-9IM touches: FT*******, F**T***** or F***T****; False for two (Multi)Point rows"""
        return self._pred(other, "touches")

    def crosses(self, other: GeoSeries):
        """row-wise DE-9IM crosses: T*T****** (lower dimension first), T*****T** (higher first), 0******** (two lines)"""
        return self._pred(other, "crosses")

    def overlaps(self, other: GeoSeries):
        """row-wise DE-9IM overlaps: T*T***T** (two point or two polygon columns), 1*T***T** (two line columns)"""
        return self._pred(other, "overlaps")

    def disjoint(self, other: GeoSeries):
        """row-wise DE-9IM disjoint: FF*FF****"""
        return self._pred(other, "disjoint")

    def geom_equals(self, other: GeoSeries):
        """row-wise topological equality: same dimension and T*F**FFF*; two empty rows are equal"""
        return self._pred(other, "geom_equals")

    def contains_properly(self, other: GeoSeries):
        """row-wise DE-9IM contains_properly: T**FF*FF*"""
        return self._pred(other, "contains_properly")


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
        matched = np.zeros(len(lhs), dtype=bool)
        matched[a] = True
        a, b = _left_rows(a, b, None, np.nonzero(~matched)[0])
    return a, b


def predicate_join(lhs: GeoSeries, rhs: GeoSeries, predicate: str = "intersects", how: str = "inner", pattern: Optional[str] = None):
    """Predicate join of any two geometry columns (GeoPandas' sjoin(predicate=...)): (lhs_index int64, rhs_index int64) for
    every pair for which `lhs.geo.<predicate>(rhs)` holds row-wise, sorted by (lhs, rhs).  predicate: intersects, contains,
    within, contains_properly, covers, covered_by, touches, crosses, overlaps, geom_equals, or relate_pattern with `pattern`;
    disjoint (and a pattern that matches disjoint pairs) raises ValueError.  how='inner' -> matching pairs; how='left' -> each
    unmatched lhs row once more, with rhs_index -1.  Points within (Multi)Polygons, and (Multi)Polygons containing points, run
    on the points-in-polygons index; everything else on the DE-9IM kernel over envelope candidates (DESIGN.md §4.20)."""
    if how not in ("inner", "left"):
        raise ValueError("how must be 'inner' or 'left'")
    lt, rt = lhs.device.type, rhs.device.type
    areas = (GeometryType.POLYGON, GeometryType.MULTIPOLYGON)
    if predicate == "within" and lt == GeometryType.POINT and rt in areas:
        a, b = E.PipIndex(rhs.device).pairs_array(lhs.device)
    elif predicate == "contains" and rt == GeometryType.POINT and lt in areas:
        p, q = E.PipIndex(lhs.device).pairs_array(rhs.device)
        order = np.lexsort((p, q))
        a, b = q[order], p[order]
    else:
        a, b = E.predicate_join(lhs.device, rhs.device, predicate, pattern)
    a = a.astype(np.int64)
    b = b.astype(np.int64)
    if how == "left":
        matched = np.zeros(len(lhs), dtype=bool)
        matched[a] = True
        a, b = _left_rows(a, b, None, np.nonzero(~matched)[0])
    return a, b


def nearest_join(lhs: GeoSeries, rhs: GeoSeries, how: str = "inner", max_distance: Optional[float] = None):
    """Nearest-geometry join of any geometry column against any geometry column (GeoPandas' sjoin_nearest with
    max_distance / distance_col): (lhs_index int64, rhs_index int64, distance float64), sorted by (lhs, rhs).  Every right
    row at the minimum distance is returned (ties are equal f64 distances, as GeoPandas returns all equidistant rows); the
    distance is exactly what `lhs.geo.distance` computes for the pair, with the left row as the first operand.
    max_distance is inclusive (None: unbounded).  Null left rows, and left rows that are empty or have a non-finite
    coordinate, match nothing.  how='inner' -> matched left rows only; how='left' -> unmatched left rows once, with
    rhs_index -1 and distance NaN.  A Point left side runs the point kernel (DESIGN.md §4.12), any other the geometry
    kernel (§4.13)."""
    if how not in ("inner", "left"):
        raise ValueError("how must be 'inner' or 'left'")
    idx = E.NearestIndex(rhs.device)
    try:
        if lhs.device.type == GeometryType.POINT:
            a, b, dist = idx.pairs_array(lhs.device, max_distance, with_distance=True)
        else:
            a, b, dist = idx.pairs_geom(lhs.device, max_distance, with_distance=True)
    finally:
        idx.free()
    a = a.astype(np.int64)
    b = b.astype(np.int64)
    d = dist[a]
    if how == "left":
        a, b, d = _left_rows(a, b, d, np.nonzero(np.isnan(dist))[0])
    return a, b, d


def dwithin_join(lhs: GeoSeries, rhs: GeoSeries, distance: float, how: str = "inner"):
    """Distance-within join of any geometry column against any geometry column (GeoPandas' sjoin(predicate="dwithin",
    distance=D)): (lhs_index int64, rhs_index int64, distance float64) for every right row whose distance to the left row is
    <= `distance` (inclusive; finite and >= 0), sorted by (lhs, rhs).  The distance is exactly what `lhs.geo.distance`
    computes for the pair, with the left row as the first operand; a null distance never matches.  Null left rows, and left
    rows that are empty or have a non-finite coordinate, match nothing.  how='inner' -> matched left rows only; how='left' ->
    unmatched left rows once, with rhs_index -1 and distance NaN (DESIGN.md §4.14)."""
    if how not in ("inner", "left"):
        raise ValueError("how must be 'inner' or 'left'")
    idx = E.NearestIndex(rhs.device)
    try:
        a, b, d = idx.pairs_within(lhs.device, distance, with_distance=True)
    finally:
        idx.free()
    a = a.astype(np.int64)
    b = b.astype(np.int64)
    if how == "left":
        matched = np.zeros(len(lhs), dtype=bool)
        matched[a] = True
        a, b, d = _left_rows(a, b, d, np.nonzero(~matched)[0])
    return a, b, d


def _left_rows(a, b, d, unmatched):
    """how='left': the unmatched left rows once, with rhs_index -1 (and distance NaN when there is a distance column d),
    merged in (lhs, rhs) order: (a, b, d), or (a, b) when d is None"""
    a = np.concatenate([a, unmatched])
    b = np.concatenate([b, np.full(len(unmatched), -1, dtype=np.int64)])
    order = np.lexsort((b, a))
    if d is None:
        return a[order], b[order]
    d = np.concatenate([d, np.full(len(unmatched), np.nan)])
    return a[order], b[order], d[order]


def overlay_area_join(lhs: GeoSeries, rhs: GeoSeries, how: str = "inner"):
    """Area-weighted overlay join of two (Multi)Polygon columns (GeoPandas' `overlay(a, b, how="intersection")` followed by
    `.area`, without building the intersection polygons): (lhs_index int64, rhs_index int64, area float64) for every pair
    whose closed geometries intersect — exactly the pairs `lhs.geo.intersects` accepts row-wise — sorted by (lhs, rhs).  The
    area is bit for bit what `lhs.geo.intersection_area` computes for the pair.  Pairs that only touch are kept with area 0,
    so the areas of a row over a partition sum to the row's area; keep `area > 0` to drop them.  how='inner' -> matched left
    rows only; how='left' -> unmatched left rows once, with rhs_index -1 and area NaN.  The operands must be valid (OGC); on
    invalid input the areas are finite but not specified (DESIGN.md §4.16); filter with `is_valid()` first."""
    if how not in ("inner", "left"):
        raise ValueError("how must be 'inner' or 'left'")
    a, b, d = E.overlay_area_join(lhs.device, rhs.device)
    a = a.astype(np.int64)
    b = b.astype(np.int64)
    if how == "left":
        matched = np.zeros(len(lhs), dtype=bool)
        matched[a] = True
        a, b, d = _left_rows(a, b, d, np.nonzero(~matched)[0])
    return a, b, d


def overlay_join(lhs: GeoSeries, rhs: GeoSeries):
    """Geometry overlay join of two (Multi)Polygon columns (GeoPandas' `overlay(a, b, how="intersection")` with
    keep_geom_type=True): (lhs_index int64, rhs_index int64, GeoSeries of MultiPolygons) for every pair whose intersection has
    at least one member, sorted by (lhs, rhs); pairs that only touch are dropped.  Geometry k is bit for bit
    `lhs.geo.intersection` of the pair (DESIGN.md §4.19).  Valid (OGC) operands only; filter with `is_valid()` first."""
    a, b, g = E.overlay_join(lhs.device, rhs.device)
    return a.astype(np.int64), b.astype(np.int64), GeoSeries(_device=g, name=lhs.name)


def overlay(lhs: GeoSeries, rhs: GeoSeries, how: str = "intersection"):
    """GeoPandas' `overlay(lhs, rhs, how)` for two (Multi)Polygon columns, keep_geom_type=True (DESIGN.md §4.23):
    (lhs_index int64, rhs_index int64, GeoSeries of MultiPolygons), -1 marking the absent side.  The rows are:

    - intersection rows (i, j), for how 'intersection', 'identity' and 'union': exactly `overlay_join`'s rows;
    - left remainders (i, -1), for every how but 'intersection': lhs[i] minus the union of every rhs row it intersects;
    - right remainders (-1, j), for 'symmetric_difference' and 'union': rhs[j] minus every lhs row it intersects.

    'difference' gives the left remainders alone.  A remainder with no member is dropped; null and non-finite rows have no
    remainder and cut nothing.  Rows are sorted by (lhs, rhs) with -1 after every index: each left row's intersections, then
    its remainder, then the right remainders.  GeoPandas concatenates its parts in another order, but the set of rows is the
    same.  The operands must be valid (OGC); filter with `is_valid()` first."""
    a, b, g = E.overlay(lhs.device, rhs.device, how)
    la, lb = a.astype(np.int64), b.astype(np.int64)
    la[a == E.ABSENT] = -1
    lb[b == E.ABSENT] = -1
    return la, lb, GeoSeries(_device=g, name=lhs.name)


def clip_join(lhs: GeoSeries, rhs: GeoSeries):
    """Geometry clip join of a (Multi)LineString or (Multi)Point column with a (Multi)Polygon column (GeoPandas'
    `overlay(lines, polys, how="intersection")` with keep_geom_type=True): (lhs_index int64, rhs_index int64, GeoSeries of
    MultiLineStrings or MultiPoints) for every pair whose clip has at least one member, sorted by (lhs, rhs); lines that only
    touch a polygon are dropped.  Geometry k is bit for bit `lhs.geo.clip` of the pair (DESIGN.md §4.22).  With a one-row
    `rhs` this is GeoPandas' `clip(lhs, mask)`: the clipped rows, with their left indices.  Valid (OGC) polygons only."""
    a, b, g = E.clip_join(lhs.device, rhs.device)
    return a.astype(np.int64), b.astype(np.int64), GeoSeries(_device=g, name=lhs.name)


def overlay_length_join(lhs: GeoSeries, rhs: GeoSeries, how: str = "inner"):
    """Length-weighted overlay join of a (Multi)LineString column with a (Multi)Polygon column ("the length of each road in
    each county"): (lhs_index int64, rhs_index int64, length float64) for every pair that intersects — exactly the pairs
    `lhs.geo.intersects` accepts row-wise — sorted by (lhs, rhs).  The length is bit for bit what
    `lhs.geo.intersection_length` computes for the pair.  Pairs that only touch are kept with length 0, so the lengths of a
    line over a partition sum to its length; keep `length > 0` to drop them.  how='inner' -> matched left rows only;
    how='left' -> unmatched left rows once, with rhs_index -1 and length NaN (DESIGN.md §4.22).  Valid (OGC) polygons only."""
    if how not in ("inner", "left"):
        raise ValueError("how must be 'inner' or 'left'")
    a, b, d = E.overlay_length_join(lhs.device, rhs.device)
    a = a.astype(np.int64)
    b = b.astype(np.int64)
    if how == "left":
        matched = np.zeros(len(lhs), dtype=bool)
        matched[a] = True
        a, b, d = _left_rows(a, b, d, np.nonzero(~matched)[0])
    return a, b, d


def geo_nearest_join(lhs: GeoSeries, rhs: GeoSeries, how: str = "inner", max_distance: Optional[float] = None):
    """`nearest_join` for two Point columns in (lon, lat) degrees, by great-circle distance in metres: (lhs_index int64,
    rhs_index int64, distance float64), sorted by (lhs, rhs).  The distance is exactly what `lhs.geo.haversine_distance`
    computes for the pair, so the join is right across the antimeridian and at the poles, where degrees are not distances.
    Every right row at the minimum distance is returned (ties are equal f64 values); max_distance is in metres and inclusive
    (None: unbounded).  Rows that are null, empty, non-finite or outside |lat| <= 90, |lon| <= 360 match nothing, on either
    side.  how='inner' -> matched left rows only; how='left' -> unmatched left rows once, with rhs_index -1 and distance NaN
    (DESIGN.md §4.15)."""
    if how not in ("inner", "left"):
        raise ValueError("how must be 'inner' or 'left'")
    idx = E.GeoIndex(rhs.device)
    try:
        a, b, dist = idx.pairs(lhs.device, max_distance, with_distance=True)
    finally:
        idx.free()
    a = a.astype(np.int64)
    b = b.astype(np.int64)
    d = dist[a]
    if how == "left":
        a, b, d = _left_rows(a, b, d, np.nonzero(np.isnan(dist))[0])
    return a, b, d


def geo_dwithin_join(lhs: GeoSeries, rhs: GeoSeries, distance: float, how: str = "inner"):
    """`dwithin_join` for two Point columns in (lon, lat) degrees, by great-circle distance: (lhs_index int64, rhs_index
    int64, distance float64) for every right row within `distance` metres (inclusive; finite and >= 0) of the left row,
    sorted by (lhs, rhs).  The distance is exactly what `lhs.geo.haversine_distance` computes for the pair; a NaN distance
    never matches.  Rows that are null, empty, non-finite or outside |lat| <= 90, |lon| <= 360 match nothing, on either side.
    how='inner' -> matched left rows only; how='left' -> unmatched left rows once, with rhs_index -1 and distance NaN
    (DESIGN.md §4.15)."""
    if how not in ("inner", "left"):
        raise ValueError("how must be 'inner' or 'left'")
    idx = E.GeoIndex(rhs.device)
    try:
        a, b, d = idx.pairs_within(lhs.device, distance, with_distance=True)
    finally:
        idx.free()
    a = a.astype(np.int64)
    b = b.astype(np.int64)
    if how == "left":
        matched = np.zeros(len(lhs), dtype=bool)
        matched[a] = True
        a, b, d = _left_rows(a, b, d, np.nonzero(~matched)[0])
    return a, b, d


def _factorize(by, n: int):
    """(sorted distinct non-null keys as a pyarrow Array, int64 code per row with -1 for a null key)"""
    pa = _pa()
    arr = by.combine_chunks() if isinstance(by, pa.ChunkedArray) else by if isinstance(by, pa.Array) else pa.array(list(by) if not isinstance(by, np.ndarray) else by, from_pandas=True)
    if len(arr) != n:
        raise ValueError("dissolve: `by` has %d values for %d rows" % (len(arr), n))
    valid = ~np.asarray(arr.is_null(nan_is_null=True).to_numpy(zero_copy_only=False), dtype=bool)
    keys = pa.compute.unique(arr.filter(pa.array(valid))) if valid.any() else arr.slice(0, 0)
    keys = keys.take(pa.compute.sort_indices(keys))
    codes = np.asarray(pa.compute.index_in(arr, value_set=keys).fill_null(-1).to_numpy(zero_copy_only=False), dtype=np.int64)
    codes[~valid] = -1
    return keys, codes


def dissolve(series: GeoSeries, by):
    """GeoPandas' `GeoSeries.groupby(by).union_all()` / `dissolve(by=...)` with sort=True, dropna=True: (keys, GeoSeries) with
    one MultiPolygon row per distinct non-null key of `by` (array-like of one key per row: integers, strings or anything
    pyarrow can sort), keys ascending, row k the union of the rows whose key is keys[k] (DESIGN.md §4.21).  Rows with a null
    key and null rows are skipped; a row with a non-finite coordinate makes its group's row null.  Aggregating other columns
    (GeoPandas' `aggfunc`) is not done here; pyarrow's `Table.group_by` does it on the same keys."""
    import pyarrow.compute  # noqa: F401 (pa.compute)

    d = series.device
    keys, codes = _factorize(by, len(d))
    return keys, GeoSeries(_device=E.dissolve(d, codes, len(keys)), name=series.name)
