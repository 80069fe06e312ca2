"""An executable model of the 2-bit interior raster of the points-in-polygons index (geopolars_b200/csrc/k_pip.cu:
grid_from_acc / fine_index / raster_mark_row / ph_raster) in Python double arithmetic — the same operations in the same
order, no FMA (the library is compiled with -fmad=false) — refereed by exact rational arithmetic (oracle/exact.py).

What it establishes, independently of any GPU: for every fine cell the build leaves UNMARKED, every double that the query
kernel maps to that cell (including the smallest and the largest such double on both axes) is strictly inside exactly the
parts the scanline fill claimed for the cell and strictly outside all others — i.e. answering such a point from the raster
is answering geo's `Polygon::contains`.  The GPU tests compare the CUDA implementation with the oracle; this file checks
the ARGUMENT (DESIGN.md 4.2 "Exactness of the raster") on shapes chosen to stress it: spiky stars, nearly horizontal and
exactly horizontal / vertical edges, vertices on cell lines, a hole, overlapping parts, rows with more crossings than the
per-row list holds.  It also packs the codes into raster words and decodes them as the streaming kernel does, for fine rasters
(one coarse cell per word) and coarse ones (rs < 4: a word spans several coarse cells; odd G: a partly used last word)."""
import math

import numpy as np
import pytest

from oracle import exact

K_ROW_CROSS = 24  # kRowCross


def d2i_rd(v):  # __double2int_rd: floor, saturating
    if v != v:
        return 0
    f = math.floor(v)
    return int(max(-(2 ** 31), min(2 ** 31 - 1, f)))


def fine_index(v, lo, inv, n):
    return min(max(d2i_rd((v - lo) * inv), 0), n - 1)


CAND_IN_CELLS = 0xFFFFFFFE  # ph_raster_cand: the word spans several coarse cells, stage 2 asks cand01


class RasterModel:
    """polys: list of parts, a part = list of closed rings (ring 0 = exterior), a ring = list of (x, y) doubles.

    Besides the mark / claim sets, the model keeps the packed raster the build writes: 16 cells of 2 bits per 32-bit word
    (raster_or_span's masks, every write an OR), the coarse cells' ascending candidate lists (ph_cells), cand01
    (ph_cell_finish) and the candidate row beside each word (ph_raster_cand); `decode` is stage 2 of k_pip_stream."""

    def __init__(self, polys, G, rs):
        self.polys = polys
        ext = [p[0] for p in polys]
        self.x0 = min(c[0] for r in ext for c in r)
        self.x1 = max(c[0] for r in ext for c in r)
        self.y0 = min(c[1] for r in ext for c in r)
        self.y1 = max(c[1] for r in ext for c in r)
        self.G, self.rs = G, rs
        self.fg = G << rs
        self.wpr = (self.fg + 15) >> 4
        self.inv_fw = self.fg / (self.x1 - self.x0)
        self.inv_fh = self.fg / (self.y1 - self.y0)
        self.marked = np.zeros((self.fg, self.fg), dtype=bool)
        self.claims = {}  # (fy, fx) -> set of parts whose fill covered the cell
        self.words = [[0] * self.wpr for _ in range(self.fg)]
        self.items = [[] for _ in range(G * G)]  # coarse cell -> ascending part ids whose exterior bbox overlaps it
        for p, rings in enumerate(polys):
            xs, ys = [c[0] for c in rings[0]], [c[1] for c in rings[0]]
            cx0, cx1 = fine_index(min(xs), self.x0, self.inv_fw, self.fg) >> rs, fine_index(max(xs), self.x0, self.inv_fw, self.fg) >> rs
            cy0, cy1 = fine_index(min(ys), self.y0, self.inv_fh, self.fg) >> rs, fine_index(max(ys), self.y0, self.inv_fh, self.fg) >> rs
            for cy in range(cy0, cy1 + 1):
                for cx in range(cx0, cx1 + 1):
                    self.items[cy * G + cx].append(p)
        self.cand01 = [(it[0] if it else -1, it[1] if len(it) > 1 else -1) for it in self.items]
        for p, rings in enumerate(polys):
            self._part(p, rings)
        # ph_raster_cand: the row of candidate #0 beside the codes when a word lies inside one coarse cell
        self.word_cand = [[self.cand01[(fy >> rs) * G + ((wx << 4) >> rs)][0] & 0xFFFFFFFF if rs >= 4 else CAND_IN_CELLS
                           for wx in range(self.wpr)] for fy in range(self.fg)]

    # -- query side -------------------------------------------------------------------------------------------------
    def cell_of(self, x, y):
        return fine_index(y, self.y0, self.inv_fh, self.fg), fine_index(x, self.x0, self.inv_fw, self.fg)

    def code(self, fy, fx):
        return (self.words[fy][fx >> 4] >> ((fx & 15) * 2)) & 3

    def decode(self, fy, fx):
        """stage 2 of k_pip_stream for a point in fine cell (fy, fx): the row it answers, -1, or None (code 3: walk)"""
        code = self.code(fy, fx)
        if code == 0:
            return -1
        if code == 3:
            return None
        cc = (fy >> self.rs) * self.G + (fx >> self.rs)
        y = self.word_cand[fy][fx >> 4]
        if code == 1 and y != CAND_IN_CELLS:
            return y - (1 << 32) if y >= 1 << 31 else y
        return self.cand01[cc][0] if code == 1 else self.cand01[cc][1]

    # -- build side -------------------------------------------------------------------------------------------------
    def _raster_or_span(self, fy, c0, c1, code):
        row, rep = self.words[fy], (code * 0x55555555) & 0xFFFFFFFF
        for w in range(c0 >> 4, (c1 >> 4) + 1):
            lo, hi = max(c0 - (w << 4), 0), min(c1 - (w << 4), 15)
            m = (0xFFFFFFFF >> (2 * (15 - hi))) & ((0xFFFFFFFF << (2 * lo)) & 0xFFFFFFFF)
            row[w] |= rep & m

    def _fill_span(self, fy, lo, hi, p):  # raster_fill_span + raster_rank_code
        for cc in range(lo >> self.rs, (hi >> self.rs) + 1):
            x0, x1 = max(lo, cc << self.rs), min(hi, ((cc + 1) << self.rs) - 1)
            it = self.items[(fy >> self.rs) * self.G + cc]
            code = 1 if it[:1] == [p] else 2 if it[1:2] == [p] else 3
            self._raster_or_span(fy, x0, x1, code)

    def _or_span(self, fy, c0, c1):
        if c0 <= c1:
            self.marked[fy, c0:c1 + 1] = True
            self._raster_or_span(fy, c0, c1, 3)

    def _mark_row(self, r, tsx, tsy, tex, tey, inv_dy):
        eps = 1e-6
        if inv_dy == 0.0:
            xa, xb = min(tsx, tex), max(tsx, tex)
        else:
            l0, l1 = (float(r) - eps - tsy) * inv_dy, (float(r) + 1.0 + eps - tsy) * inv_dy
            if l0 > l1:
                l0, l1 = l1, l0
            l0, l1 = max(l0, 0.0), min(l1, 1.0)
            if l0 > l1:
                return
            dx = tex - tsx
            xa, xb = tsx + l0 * dx, tsx + l1 * dx
            if xa > xb:
                xa, xb = xb, xa
        c0 = min(max(d2i_rd(xa - 2e-6), 0), self.fg - 1)
        c1 = min(max(d2i_rd(xb + 2e-6), 0), self.fg - 1)
        self._or_span(r, c0, c1)

    def _part(self, p, rings):
        g = self
        xs, ys = [c[0] for c in rings[0]], [c[1] for c in rings[0]]
        fx0, fx1 = fine_index(min(xs), g.x0, g.inv_fw, g.fg), fine_index(max(xs), g.x0, g.inv_fw, g.fg)
        fy0, fy1 = fine_index(min(ys), g.y0, g.inv_fh, g.fg), fine_index(max(ys), g.y0, g.inv_fh, g.fg)
        for ra in range(fy0, fy1 + 1, 32):
            rb = min(ra + 31, fy1)
            cnt = [0] * 32
            lists = [[] for _ in range(32)]
            row_y = [g.y0 + ((ra + lane) + 0.5) / g.inv_fh for lane in range(32)]
            for r, ring in enumerate(rings):
                ring_tag = min(r, 2047)
                for s, e in zip(ring[:-1], ring[1:]):  # closed input rings: edge_of_slot's closing rule is not exercised
                    tsx, tsy = (s[0] - g.x0) * g.inv_fw, (s[1] - g.y0) * g.inv_fh
                    tex, tey = (e[0] - g.x0) * g.inv_fw, (e[1] - g.y0) * g.inv_fh
                    ylo, yhi = min(tsy, tey), max(tsy, tey)
                    er0 = max(min(max(d2i_rd(ylo - 1e-6), 0), g.fg - 1), ra)
                    er1 = min(min(max(d2i_rd(yhi + 1e-6), 0), g.fg - 1), rb)
                    tdy, tdx = tey - tsy, tex - tsx
                    inv_dy = 0.0 if abs(tdy) < 1e-3 else 1.0 / tdy
                    for row in range(er0, er1 + 1):
                        self._mark_row(row, tsx, tsy, tex, tey, inv_dy)
                        ry = row_y[row - ra]
                        up, down = s[1] <= ry < e[1], e[1] <= ry < s[1]
                        if up or down:
                            lam = ((float(row) + 0.5 - tsy) * inv_dy) if inv_dy != 0.0 else 0.5
                            lam = min(max(lam, 0.0), 1.0)
                            cj = min(max(d2i_rd(tsx + lam * tdx), 0), g.fg - 1)
                            slot = cnt[row - ra]
                            cnt[row - ra] += 1
                            if slot < K_ROW_CROSS:
                                lists[row - ra].append((cj, down, ring_tag))
            for lane in range(32):
                fy = ra + lane
                if fy > rb:
                    break
                n, ry = cnt[lane], row_y[lane]
                if n > K_ROW_CROSS or fine_index(ry, g.y0, g.inv_fh, g.fg) != fy:
                    self._or_span(fy, fx0, fx1)
                    continue
                L = sorted(lists[lane], key=lambda t: t[0])  # the kernel's insertion sort is stable too; ties have empty intervals
                for k in range(1, n):
                    lo, hi = L[k - 1][0] + 1, L[k][0] - 1
                    if lo > hi:
                        continue
                    wn_ext, in_hole = 0, False
                    for j in range(k, n):
                        ring = L[j][2]
                        d = -1 if L[j][1] else 1
                        if ring == 0:
                            wn_ext += d
                        elif all(L[i][2] != ring for i in range(k, j)):  # this hole's first entry: sum it once
                            w = sum((-1 if L[i][1] else 1) for i in range(j, n) if L[i][2] == ring)
                            in_hole = in_hole or w != 0
                    if wn_ext != 0 and not in_hole:
                        for fx in range(lo, hi + 1):
                            self.claims.setdefault((fy, fx), set()).add(p)
                        self._fill_span(fy, lo, hi, p)

    # -- every double that maps to a cell, sampled: its extremes and a few interior values -----------------------------
    def _axis_samples(self, c, lo, inv):
        def idx(v):
            return fine_index(v, lo, inv, self.fg)

        def first_with(pred, a, b):  # smallest double in [a, b] with pred true (pred monotone false -> true)
            assert not pred(a) and pred(b)
            while np.nextafter(a, np.inf) < b:
                m = a + (b - a) / 2
                if pred(m):
                    b = m
                else:
                    a = m
            return b

        centre = lo + (c + 0.5) / inv
        assert idx(centre) == c
        out = {centre, lo + (c + 0.25) / inv, lo + (c + 0.999) / inv}
        below, above = lo + (c - 0.5) / inv, lo + (c + 1.5) / inv
        if c > 0:
            out.add(first_with(lambda v: idx(v) >= c, below, centre))  # the smallest double of the cell
        if c < self.fg - 1:
            nxt = first_with(lambda v: idx(v) >= c + 1, centre, above)
            out.add(float(np.nextafter(nxt, -np.inf)))  # the largest double of the cell
        return sorted(v for v in out if idx(v) == c)

    def check_unmarked_cells(self, every=1):
        """returns (cells checked, cells claimed inside something).  Raises on the first wrong classification."""
        boxes = [(min(c[0] for c in r[0]), max(c[0] for c in r[0]), min(c[1] for c in r[0]), max(c[1] for c in r[0])) for r in self.polys]
        checked = inside = 0
        k = 0
        for fy in range(self.fg):
            ys = None
            for fx in range(self.fg):
                if self.marked[fy, fx]:
                    continue
                k += 1
                if k % every:
                    continue
                ys = ys or self._axis_samples(fy, self.y0, self.inv_fh)
                xs = self._axis_samples(fx, self.x0, self.inv_fw)
                claim = self.claims.get((fy, fx), set())
                checked += 1
                inside += bool(claim)
                for y in ys:
                    for x in xs:
                        assert self.cell_of(x, y) == (fy, fx)
                        for p, rings in enumerate(self.polys):
                            bx0, bx1, by0, by1 = boxes[p]
                            if not (bx0 <= x <= bx1 and by0 <= y <= by1):
                                assert p not in claim, f"cell ({fy},{fx}) claims part {p} outside its bbox"
                                continue
                            want = exact.polygon_contains((x, y), rings)
                            assert want == (p in claim), f"cell ({fy},{fx}) point ({x!r},{y!r}) part {p}: exact {want}, raster {p in claim}"
                            if not want:  # an unmarked cell holds no boundary point either
                                assert all(exact.ring_position((x, y), r) != 1 for r in rings)
        return checked, inside

    def check_decode(self):
        """the packed words against the mark / claim sets: every marked cell reads code 3; every other cell decodes (stage 2)
        to the row its claim set gives (none -> -1, one part -> that part unless it ranks after #1 in its coarse cell, two or
        more -> walk); cells past fgx in a row's last word stay 0.  Returns {code: cells} over the unmarked cells."""
        census = {0: 0, 1: 0, 2: 0, 3: 0}
        for fy in range(self.fg):
            for fx in range(self.fg):
                code = self.code(fy, fx)
                if self.marked[fy, fx]:
                    assert code == 3, f"marked cell ({fy},{fx}) reads code {code}"
                    continue
                census[code] += 1
                claim = self.claims.get((fy, fx), set())
                got = self.decode(fy, fx)
                it = self.items[(fy >> self.rs) * self.G + (fx >> self.rs)]
                if not claim:
                    assert got == -1, (fy, fx, got)
                elif len(claim) == 1 and next(iter(claim)) in it[:2]:
                    assert got == next(iter(claim)), f"cell ({fy},{fx}) claimed by {claim} decodes to {got} (candidates {it[:2]})"
                else:
                    assert got is None, (fy, fx, claim, got)
            for fx in range(self.fg, self.wpr * 16):
                assert self.code(fy, fx) == 0
        return census


def star(rng, cx, cy, n, r0, r1):
    th = 2 * np.pi * (np.arange(n) + rng.uniform(0, 1)) / n
    r = rng.uniform(r0, r1, n)
    pts = [(float(cx + r[i] * np.cos(th[i])), float(cy + r[i] * np.sin(th[i]))) for i in range(n)]
    return pts + [pts[0]]


def test_ring_position_convention():
    sq = [(0.0, 0.0), (4.0, 0.0), (4.0, 4.0), (0.0, 4.0), (0.0, 0.0)]
    assert [exact.ring_position(p, sq) for p in [(5.0, 1.0), (0.0, 1.0), (1.0, 1.0)]] == [0, 1, 2]  # the checker relies on "1 = boundary"


@pytest.mark.parametrize("seed,nvert", [(1, 16), (2, 7), (3, 33)])
def test_unmarked_cells_of_a_star_grid_are_classified_exactly(seed, nvert):
    """config-2-like: a 3 x 3 grid of spiky stars, 2^4 fine cells per coarse cell"""
    rng = np.random.default_rng(seed)
    polys = [[star(rng, 10.0 * i + 5.0 + rng.uniform(-1, 1), 10.0 * j + 5.0 + rng.uniform(-1, 1), nvert, 1.0, 4.5)] for j in range(3) for i in range(3)]
    m = RasterModel(polys, G=3, rs=4)
    checked, inside = m.check_unmarked_cells()
    frac_marked = m.marked.mean()
    assert checked > 400 and inside > 30, (checked, inside)
    assert 0.05 < frac_marked < 0.8, frac_marked  # the test is not vacuous: most cells are answered by the raster


def test_axis_aligned_edges_vertices_on_cell_lines_hole_and_overlap():
    """coordinates chosen ON fine-cell lines (the grid is 32 x 32 over [0, 32]^2: cell width exactly 1), horizontal and vertical
    edges, a hole whose edges lie on cell lines, a second part overlapping the first, a sliver thinner than a cell"""
    outer = [(0.0, 0.0), (32.0, 0.0), (32.0, 32.0), (0.0, 32.0), (0.0, 0.0)]
    hole = [(8.0, 8.0), (8.0, 20.0), (20.0, 20.0), (20.0, 8.0), (8.0, 8.0)]
    tri = [(4.5, 4.25), (30.0, 6.0), (10.0, 29.5), (4.5, 4.25)]
    sliver = [(22.0, 22.3), (31.0, 22.4), (31.0, 22.45), (22.0, 22.3)]
    m = RasterModel([[outer, hole], [tri], [sliver]], G=2, rs=4)
    assert m.fg == 32 and m.inv_fw == 1.0 and m.inv_fh == 1.0
    checked, inside = m.check_unmarked_cells()
    assert checked > 300 and inside > 200
    # the kinds of answers that occur: inside the square only, inside square and triangle, inside the triangle only (in the hole)
    kinds = {frozenset(v) for v in m.claims.values()}
    assert {frozenset({0}), frozenset({0, 1}), frozenset({1})} <= kinds
    # cells on both sides of an edge that lies ON a cell line are marked (the hole's top edge y = 20 marks rows 19 and 20)
    assert m.marked[19, 9:19].all() and m.marked[20, 9:19].all()


def test_rows_with_more_crossings_than_the_list_holds_are_marked_whole():
    """a comb with 20 teeth: 40 crossings per row > kRowCross -> those rows take the walk over the part's whole column range"""
    teeth = []
    for i in range(20):
        teeth += [(1.0 + 1.5 * i, 1.0), (1.25 + 1.5 * i, 30.0), (1.5 + 1.5 * i, 30.0), (1.75 + 1.5 * i, 1.0)]
    comb = [(0.5, 0.5)] + teeth + [(31.5, 0.5), (0.5, 0.5)]
    frame = [(0.0, 0.0), (64.0, 0.0), (64.0, 64.0), (0.0, 64.0), (0.0, 0.0)]
    m = RasterModel([[frame], [comb]], G=2, rs=5)
    assert m.fg == 64 and m.inv_fw == 1.0
    rows_through_teeth = range(3, 29)
    fx0, fx1 = fine_index(0.5, m.x0, m.inv_fw, m.fg), fine_index(31.5, m.x0, m.inv_fw, m.fg)
    for fy in rows_through_teeth:
        assert m.marked[fy, fx0:fx1 + 1].all()
    checked, inside = m.check_unmarked_cells()
    assert checked > 2000 and inside == checked  # what is left (beside and above the comb) is inside the frame only, exactly


def test_offset_and_scale_do_not_matter():
    """nybb-like magnitudes: coordinates around 1e6 with extents of 1e3; and a tiny grid around 1e-9"""
    rng = np.random.default_rng(7)
    for cx, cy, sc in [(9.8e5, 1.9e5, 100.0), (1e-9, -2e-9, 1e-10)]:
        polys = [[[(cx + sc * x, cy + sc * y) for x, y in star(rng, 10.0 * i + 5.0, 10.0 * j + 5.0, 11, 1.0, 4.5)]] for j in range(2) for i in range(2)]
        m = RasterModel(polys, G=2, rs=4)
        checked, inside = m.check_unmarked_cells()
        assert checked > 200 and inside > 10


def test_the_referee_has_teeth():
    """negative control: a build that forgets to mark the cells along ONE edge must be caught by the exact check"""

    class Forgetful(RasterModel):
        def _mark_row(self, r, tsx, tsy, tex, tey, inv_dy):
            if abs(tsx - 4.5) < 1e-9 and abs(tex - 30.0) < 1e-9:  # the triangle's first edge
                return
            super()._mark_row(r, tsx, tsy, tex, tey, inv_dy)

    outer = [(0.0, 0.0), (32.0, 0.0), (32.0, 32.0), (0.0, 32.0), (0.0, 0.0)]
    tri = [(4.5, 4.25), (30.0, 6.0), (10.0, 29.5), (4.5, 4.25)]
    RasterModel([[outer], [tri]], G=2, rs=4).check_unmarked_cells()  # the faithful model passes
    with pytest.raises(AssertionError):
        Forgetful([[outer], [tri]], G=2, rs=4).check_unmarked_cells()


def _coarse_field(rng):
    """overlapping spiky stars on a 4 x 4 lattice (bboxes overlap, so cells have second and third candidates), one of them
    with a hole, and one large polygon over a corner of the lattice"""
    polys = []
    for j in range(4):
        for i in range(4):
            rings = [star(rng, 10.0 * i + 5.0 + rng.uniform(-1, 1), 10.0 * j + 5.0 + rng.uniform(-1, 1), 9, 2.5, 7.0)]
            if (i, j) == (1, 2):
                cx = sum(c[0] for c in rings[0][:-1]) / 9.0
                cy = sum(c[1] for c in rings[0][:-1]) / 9.0
                rings.append(star(rng, cx, cy, 5, 0.5, 1.0)[::-1])
            polys.append(rings)
    polys.append([star(rng, 28.0, 28.0, 7, 6.0, 11.0)])
    return polys


@pytest.mark.parametrize("rs,G", [(0, 15), (1, 13), (2, 9), (3, 5)])
def test_coarse_rasters_decode_to_the_claimed_row(rs, G):
    """rs < 4: a raster word spans several coarse cells, so the build stores 0xfffffffe beside the codes and stage 2 takes
    candidate #0 from cand01 of the point's OWN coarse cell; G odd: the last word of each row is only partly used"""
    m = RasterModel(_coarse_field(np.random.default_rng(40 + rs)), G=G, rs=rs)
    assert m.fg % 16 != 0 and m.wpr * 16 > m.fg  # the partial last word is modelled
    assert all(v == CAND_IN_CELLS for row in m.word_cand for v in row)
    checked, inside = m.check_unmarked_cells()
    assert checked > 20 and inside > 5, (checked, inside)
    census = m.check_decode()
    assert census[1] > 0 and census[0] > 0, census
    # code-1 cells whose coarse cell is not the coarse cell of their word's first fine cell: only cand01 answers them right
    foreign = sum(1 for fy in range(m.fg) for fx in range(m.fg)
                  if not m.marked[fy, fx] and m.code(fy, fx) == 1 and (fx >> rs) != (((fx >> 4) << 4) >> rs))
    assert foreign > 0
    assert max(len(it) for it in m.items) >= 3


def test_fine_raster_keeps_the_row_beside_the_codes():
    """rs >= 4: every word lies inside one coarse cell and carries its candidate #0"""
    m = RasterModel(_coarse_field(np.random.default_rng(44)), G=3, rs=4)
    assert all(v != CAND_IN_CELLS for row in m.word_cand for v in row)
    census = m.check_decode()
    assert census[1] > 0 and census[2] >= 0


def test_the_decode_referee_has_teeth():
    """negative controls: the candidate row of a word's first coarse cell used for every cell of the word (the rs >= 4 guard
    dropped), and a span mask one cell short at its upper end, must both be caught by check_decode"""

    class NoGuard(RasterModel):
        def __init__(self, polys, G, rs):
            super().__init__(polys, G, rs)
            self.word_cand = [[self.cand01[(fy >> rs) * G + ((wx << 4) >> rs)][0] & 0xFFFFFFFF for wx in range(self.wpr)]
                              for fy in range(self.fg)]

    class ShortMask(RasterModel):
        def _raster_or_span(self, fy, c0, c1, code):
            super()._raster_or_span(fy, c0, c1 - 1, code)

    polys = _coarse_field(np.random.default_rng(42))
    RasterModel(polys, G=9, rs=2).check_decode()
    for bad in (NoGuard, ShortMask):
        with pytest.raises(AssertionError):
            bad(polys, G=9, rs=2).check_decode()
