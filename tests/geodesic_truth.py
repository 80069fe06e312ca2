"""The true geodesic on WGS84 at 40 significant digits — TEST INFRASTRUCTURE ONLY (CPU, mpmath).

An independent reference for the ellipsoid kernels (DESIGN.md §4.9, §4.17): it shares nothing with Karney's series, with
Vincenty's iteration or with tests/geodesic_area_reference.py.  It integrates the exact auxiliary-sphere integrals by
quadrature.  With the reduced latitude beta (tan beta = (1 - f) tan phi), sin alp0 = sin alp1 cos beta1 and
k^2 = e'^2 cos^2 alp0, along a geodesic parametrised by the arc length sigma on the auxiliary sphere:

    s      = b Int sqrt(1 + k^2 sin^2 sigma) dsigma
    lambda = omega - f sin alp0 Int (2 - f) / (1 + (1 - f) sqrt(1 + k^2 sin^2 sigma)) dsigma
    omega  = atan2(sin alp0 sin sigma, cos sigma)            (the longitude on the auxiliary sphere)

Inverse problem: each pair is reduced to beta1 <= 0, |beta2| <= -beta1, 0 <= lambda12 <= pi, where lambda12(alp1) rises
monotonically from 0 (alp1 = 0) to pi (alp1 = pi), and the root is found by regula falsi (Illinois) inside that bracket,
so it never leaves the branch.  Meridional pairs (lambda12 = 0 or pi) and equatorial pairs with lambda12 <= (1 - f) pi are
closed forms.

Area: F(phi) = (b^2 / 2) (sin phi / (1 - e^2 sin^2 phi) + atanh(e sin phi) / e) is the area between the equator and
latitude phi per radian of longitude (F(90) = c^2).  An edge contributes E = Int F(phi) dlambda along its geodesic (a
longitude jump at a pole counts there with F(+-90) = +-c^2), and a ring's counter-clockwise-positive area is
-Sum E + c^2 Sum dlambda, where Sum dlambda is 0 or +-2 pi (a ring around a pole): the result is exact modulo area0.

Haversine: the central angle on the sphere of radius 6 371 008.8 m, evaluated at 40 digits from the same double inputs.

Every public function works at 40 digits inside its own mpmath precision context and leaves the process-wide precision
alone; a caller doing arithmetic on the mpf values it returns sets its own (`with mpmath.workdps(DPS)`).
"""
import functools

import mpmath as mp

DPS = 40


def _at_dps(fn):
    @functools.wraps(fn)
    def run(*args, **kwargs):
        with mp.workdps(DPS):
            return fn(*args, **kwargs)

    return run


with mp.workdps(DPS):  # the ellipsoid's constants, held at 40 digits
    A = mp.mpf(6378137)
    F_ = 1 / mp.mpf("298.257223563")
    B = A * (1 - F_)
    E2 = F_ * (2 - F_)
    EP2 = E2 / (1 - F_) ** 2
    E = mp.sqrt(E2)
    C2 = A**2 / 2 + B**2 * mp.atanh(E) / (2 * E)
    AREA0 = 4 * mp.pi * C2
    R_MEAN = mp.mpf(6371008.8)  # the double geo's MEAN_EARTH_RADIUS rounds to, taken exactly
    EQ_LIMIT = (1 - F_) * 180  # degrees: beyond it an equatorial pair's shortest geodesic leaves the equator


@_at_dps
def authalic_F(sphi):
    """F(phi) from sin(phi)"""
    return B**2 / 2 * (sphi / (1 - E2 * sphi**2) + mp.atanh(E * sphi) / E)


def _beta(lat):
    if abs(lat) == 90:
        return mp.sign(lat) * mp.pi / 2
    phi = mp.radians(lat)
    return mp.atan2((1 - F_) * mp.sin(phi), mp.cos(phi))


def _reduce180(d):
    """degrees -> (-180, 180]"""
    d = d - 360 * mp.floor(d / 360)
    return d - 360 if d > 180 else d


def _sphi(sbet):
    cbet2 = 1 - sbet**2
    return sbet / mp.sqrt(sbet**2 + (1 - F_) ** 2 * cbet2)


class _Line:
    """the geodesic leaving beta1 with azimuth alp1, followed to the point where it reaches beta2 heading north"""

    def __init__(self, b1, b2, alp1):
        sb1, cb1, sb2, cb2 = mp.sin(b1), mp.cos(b1), mp.sin(b2), mp.cos(b2)
        sa1, ca1 = mp.sin(alp1), mp.cos(alp1)
        self.sa0 = sa1 * cb1
        self.ca0 = mp.sqrt(1 - self.sa0**2)
        self.k2 = EP2 * self.ca0**2
        ca2cb2 = mp.sqrt(max((ca1 * cb1) ** 2 + (cb2 - cb1) * (cb2 + cb1), mp.mpf(0)))
        if b1 == 0:  # both on the equator (canonical form): the line dips south from sigma = -pi to sigma = 0
            self.s1 = self.w1 = -mp.pi
        else:
            self.s1 = mp.atan2(sb1, ca1 * cb1)
            self.w1 = mp.atan2(self.sa0 * mp.sin(self.s1), mp.cos(self.s1))
        self.s2 = mp.atan2(sb2, ca2cb2)
        self.w2 = mp.atan2(self.sa0 * mp.sin(self.s2), mp.cos(self.s2))
        self.alp2 = mp.atan2(self.sa0, ca2cb2)

    def _pts(self):
        """[s1, s2] split where lambda' peaks (sigma = +-pi/2, width sin alp0) so that quadrature sees smooth pieces"""
        pts = [self.s1]
        for v in (-mp.pi / 2, mp.pi / 2):
            for d in (-100 * self.sa0, -self.sa0, 0, self.sa0, 100 * self.sa0):
                x = v + d
                if self.s1 < x < self.s2 and (x - pts[-1]) > 0:
                    pts.append(x)
        pts.append(self.s2)
        return pts

    def lam(self):
        k2, sa0 = self.k2, self.sa0
        i3 = mp.quad(lambda s: (2 - F_) / (1 + (1 - F_) * mp.sqrt(1 + k2 * mp.sin(s) ** 2)), [self.s1, self.s2])
        return (self.w2 - self.w1) - F_ * sa0 * i3

    def dist(self):
        k2 = self.k2
        return B * mp.quad(lambda s: mp.sqrt(1 + k2 * mp.sin(s) ** 2), [self.s1, self.s2])

    def area(self):
        k2, sa0, ca0 = self.k2, self.sa0, self.ca0

        def g(s):
            ss, cs = mp.sin(s), mp.cos(s)
            dlam = sa0 / (cs**2 + sa0**2 * ss**2) - F_ * sa0 * (2 - F_) / (1 + (1 - F_) * mp.sqrt(1 + k2 * ss**2))
            return authalic_F(_sphi(ca0 * ss)) * dlam

        return mp.quad(g, self._pts())


def _solve(b1, b2, lam, lo, flo, hi, fhi):
    """regula falsi with the Illinois step on lambda12(alp1) - lam, bracket [lo, hi]; raises if neither the residual nor the
    bracket reaches its tolerance, so a failed solve can never become a truth"""
    side = 0
    for _ in range(400):
        x = hi - fhi * (hi - lo) / (fhi - flo)
        if not lo < x < hi:
            x = (lo + hi) / 2
        fx = _Line(b1, b2, x).lam() - lam
        if fx == 0 or hi - lo < mp.mpf(10) ** (-mp.mp.dps + 2):
            return x
        if abs(fx) < mp.mpf(10) ** (-mp.mp.dps + 1) * (1 + abs(lam)):
            return x
        if (fx < 0) == (flo < 0):
            lo, flo = x, fx
            if side == -1:
                fhi /= 2
            side = -1
        else:
            hi, fhi = x, fx
            if side == 1:
                flo /= 2
            side = 1
    raise ArithmeticError(f"lambda12(alp1) = {mp.nstr(lam, 20)} not solved in [{mp.nstr(lo, 20)}, {mp.nstr(hi, 20)}]")


def _canonical(lon1, lat1, lon2, lat2):
    """the pair as (beta1, beta2, lambda12 degrees) with beta1 <= 0, |beta2| <= -beta1, 0 <= lambda12 <= 180, and the signs that
    map an edge integral and a longitude change back (swap, lon mirror, lat mirror)"""
    lon1, lat1, lon2, lat2 = (mp.mpf(float(v)) for v in (lon1, lat1, lon2, lat2))
    sw = 1
    if abs(lat1) < abs(lat2):
        lon1, lat1, lon2, lat2 = lon2, lat2, lon1, lat1
        sw = -1
    lam = _reduce180(lon2 - lon1)
    sl = -1 if lam < 0 else 1
    lam = abs(lam)
    sb = -1 if lat1 > 0 else 1
    return _beta(sb * lat1), _beta(sb * lat2), lam, sw, sl, sb


@_at_dps
def inverse(lon1, lat1, lon2, lat2, with_area=False):
    """true s12 (m), alp1 and alp2 (degrees, in (-180, 180]), the unwrapped longitude change lambda12 (degrees) along the
    geodesic and, with_area, the edge integral E = Int F dlambda (m^2); mpf values.  Inputs are the doubles of the
    (lon, lat) degree coordinates, taken exactly."""
    b1, b2, lamd, sw, sl, sb = _canonical(lon1, lat1, lon2, lat2)
    lam = mp.radians(lamd)
    e = mp.mpf(0)
    if b1 == -mp.pi / 2 or lamd == 0 or lamd == 180:
        # meridional (or from a pole): sigma runs with beta, through the south pole when lambda12 = 180
        q = lambda s: mp.sqrt(1 + EP2 * mp.sin(s) ** 2)  # noqa: E731
        if lamd == 0 or b1 == -mp.pi / 2:
            s = B * mp.quad(q, [b1, b2])
            a1, a2 = (mp.mpf(0), mp.mpf(0))
        else:
            s = B * (mp.quad(q, [-mp.pi / 2, b1]) + mp.quad(q, [-mp.pi / 2, b2]))
            a1, a2 = mp.pi, mp.mpf(0)
        if b1 == -mp.pi / 2 or lamd == 180:
            e = -C2 * lam  # the longitude jumps by lambda12 at the south pole, where F = -c^2
        if b1 == -mp.pi / 2 and b2 == -mp.pi / 2:
            s = mp.mpf(0)
    elif b1 == 0 and b2 == 0 and lamd <= EQ_LIMIT:
        s, a1, a2 = A * lam, mp.pi / 2, mp.pi / 2
    else:
        lo = mp.pi / 2 if b1 == 0 else mp.mpf(0)  # on the equator the line must dip south: alp1 in (90, 180)
        flo = (mp.pi * (1 - F_) if b1 == 0 else mp.mpf(0)) - lam
        a1 = _solve(b1, b2, lam, lo, flo, mp.pi, mp.pi - lam)
        line = _Line(b1, b2, a1)
        lam = line.lam()
        s, a2 = line.dist(), line.alp2
        if with_area:
            e = line.area()
    # back to the pair as given
    if sb < 0:
        a1, a2 = mp.pi - a1, mp.pi - a2
    if sl < 0:
        a1, a2 = -a1, -a2
    if sw < 0:
        a1, a2 = a2 + mp.pi, a1 + mp.pi
    a1, a2 = (_reduce180(mp.degrees(a)) for a in (a1, a2))
    out = (s, a1, a2, sw * sl * mp.degrees(lam))
    return out + (sw * sl * sb * e,) if with_area else out


@_at_dps
def ring(coords, reverse=False, signed=True):
    """the true (area, perimeter) of one ring of (lon, lat) doubles, closing edge included (a repeated closing vertex is
    dropped), with geographiclib's PolygonArea ranges: signed in (-area0/2, area0/2], unsigned in [0, area0); reverse makes
    clockwise positive.  Also returns the per-edge (s, E, dlambda) it summed."""
    pts = [(float(x), float(y)) for x, y in coords]
    if len(pts) >= 2 and pts[-1] == pts[0]:
        pts = pts[:-1]
    if len(pts) < 2:
        return mp.mpf(0), mp.mpf(0), []
    edges = []
    for i, p in enumerate(pts):
        q = pts[(i + 1) % len(pts)]
        s, _, _, dlam, e = inverse(p[0], p[1], q[0], q[1], with_area=True)
        edges.append((s, e, dlam))
    return ring_from_edges(edges, reverse, signed) + (edges,)


@_at_dps
def ring_from_edges(edges, reverse=False, signed=True):
    per = mp.fsum(s for s, _, _ in edges)
    turn = mp.fsum(d for _, _, d in edges)
    area = -mp.fsum(e for _, e, _ in edges) + C2 * mp.radians(turn)
    if reverse:
        area = -area
    area -= AREA0 * mp.floor(area / AREA0)  # [0, area0)
    if signed and area > AREA0 / 2:
        area -= AREA0
    return area, per


@_at_dps
def polygon_from_rings(rings, signed=True):
    """geo's rule over rings given as (exterior (area, per), [hole (area, per) with reverse=True]): holes subtract by
    magnitude, negated when the exterior is negative"""
    (ea, per), holes = rings[0], rings[1:]
    h = mp.fsum(abs(a) for a, _ in holes)
    per += mp.fsum(p for _, p in holes)
    if ea < 0 and h > 0:
        h = -h
    return ea - h, per


@_at_dps
def haversine(lon1, lat1, lon2, lat2):
    """the great-circle distance (m) on the mean sphere between the two double (lon, lat) points"""
    p1, p2 = mp.radians(mp.mpf(float(lat1))), mp.radians(mp.mpf(float(lat2)))
    dl = mp.radians(mp.mpf(float(lon2)) - mp.mpf(float(lon1)))
    a = mp.sin((p2 - p1) / 2) ** 2 + mp.cos(p1) * mp.cos(p2) * mp.sin(dl / 2) ** 2
    return R_MEAN * 2 * mp.asin(mp.sqrt(min(a, mp.mpf(1)))), a


@_at_dps
def split(x):
    """mpf -> (hi, lo) doubles with hi + lo = x to about 1e-32 relative"""
    hi = float(x)
    return hi, float(x - hi)
