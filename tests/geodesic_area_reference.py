"""CPU reference for the geodesic area and perimeter of (lon, lat) polygon columns on WGS84 — TEST INFRASTRUCTURE ONLY.

A plain-Python restatement of geo 0.27's GeodesicArea (DESIGN.md §4.17): Karney's inverse problem (arXiv:1109.4448) with
the azimuths and the area term S12 (geographiclib's GenInverse with the AREA output), geographiclib's PolygonArea per ring
(double-double Accumulator, prime-meridian transits, reduceArea) and geo's rules for holes, multipolygons and other types.
The rings are summed sequentially, edge by edge, as PolygonArea does; the GPU combines per-lane sums in a tree, so the two
agree to the rounding of the summed terms, not bit for bit.  `scale` sums, over a row's edges, the magnitudes of the terms
that make up each S12 (|A4 B41|, |A4 B42| and |c^2 alp12|, each up to about 1e11 m^2): the error of a small polygon is set by
the rounding of those terms, which are large and cancel within an edge and across edges, so tests bound it with that.
"""
import math

import numpy as np

A = 6378137.0
F = 1 / 298.257223563
F1 = 1 - F
E2 = F * (2 - F)
EP2 = E2 / (F1 * F1)
N = F / (2 - F)
B = A * F1
C2 = (A * A + B * B * (math.atanh(math.sqrt(E2)) / math.sqrt(abs(E2)))) / 2
AREA0 = 4 * math.pi * C2
TINY = math.sqrt(2.2250738585072014e-308)
TOL0 = 2.220446049250313e-16
TOL1 = 200 * TOL0
TOL2 = math.sqrt(TOL0)
TOLB = TOL0 * TOL2
XTHRESH = 1000 * TOL2
MAXIT1 = 20
MAXIT2 = MAXIT1 + 53 + 10
ETOL2 = 0.1 * TOL2 / math.sqrt(max(0.001, abs(F)) * min(1.0, 1 - F / 2) / 2)
DEG = math.pi / 180


def _sq(x):
    return x * x


def _norm2(x, y):
    r = math.hypot(x, y)
    return x / r, y / r


def _sum(u, v):
    s = u + v
    up = s - v
    vpp = s - up
    up -= u
    vpp -= v
    t = 0.0 - (up + vpp) if s != 0 else s
    return s, t


def _ang_round(x):
    z = 1 / 16.0
    y = abs(x)
    w = z - y
    y = z - w if w > 0 else y
    return math.copysign(y, x)


def _remainder(x, y):
    return math.remainder(x, y) if math.isfinite(x) else math.nan


def ang_normalize(x):
    y = _remainder(x, 360.0)
    return math.copysign(180.0, x) if abs(y) == 180 else y


def ang_diff(x, y):
    d, t = _sum(_remainder(-x, 360.0), _remainder(y, 360.0))
    d, t = _sum(_remainder(d, 360.0), t)
    if d == 0 or abs(d) == 180:
        d = math.copysign(d, y - x if t == 0 else -t)
    return d, t


def _sincosd_q(r, q):
    s, c = math.sin(r), math.cos(r)
    q &= 3
    if q == 1:
        s, c = c, -s
    elif q == 2:
        s, c = -s, -c
    elif q == 3:
        s, c = -c, s
    return s, c + 0.0


def _quadrant(x):
    r = math.fmod(x, 360.0)
    q = int(round(r / 90))
    return r - 90 * q, q


def sincosd(x):
    r, q = _quadrant(x)
    s, c = _sincosd_q(r * DEG, q)
    if s == 0:
        s = math.copysign(s, x)
    return s, c


def sincosde(x, t):
    r, q = _quadrant(x)
    s, c = _sincosd_q(_ang_round(r + t) * DEG, q)
    if s == 0:
        s = math.copysign(s, x)
    return s, c


def _sin_series(sinx, cosx, c, n):
    """sum_{l=1..n} c[l] sin(2 l x)"""
    k = n + 1
    ar = 2 * (cosx - sinx) * (cosx + sinx)
    y0, y1 = 0.0, 0.0
    if n & 1:
        k -= 1
        y0 = c[k]
    for _ in range(n // 2):
        k -= 1
        y1 = ar * y0 - y1 + c[k]
        k -= 1
        y0 = ar * y1 - y0 + c[k]
    return 2 * sinx * cosx * y0


def _cos_series(sinx, cosx, c, n):
    """sum_{l=0..n-1} c[l] cos((2 l + 1) x)"""
    k = n
    ar = 2 * (cosx - sinx) * (cosx + sinx)
    y0, y1 = 0.0, 0.0
    if n & 1:
        k -= 1
        y0 = c[k]
    for _ in range(n // 2):
        k -= 1
        y1 = ar * y0 - y1 + c[k]
        k -= 1
        y0 = ar * y1 - y0 + c[k]
    return cosx * (y0 - y1)


def _A1m1f(eps):
    e2 = eps * eps
    t = e2 * (64 + e2 * (4 + e2)) / 256
    return (t + eps) / (1 - eps)


def _C1f(eps):
    e2, d, c = eps * eps, eps, [0.0] * 7
    c[1] = d * (-16 + e2 * (6 - e2)) / 32
    d *= eps
    c[2] = d * (-128 + e2 * (64 - 9 * e2)) / 2048
    d *= eps
    c[3] = d * (9 * e2 - 16) / 768
    d *= eps
    c[4] = d * (3 * e2 - 5) / 512
    d *= eps
    c[5] = -7 * d / 1280
    d *= eps
    c[6] = -7 * d / 2048
    return c


def _A2m1f(eps):
    e2 = eps * eps
    t = e2 * (-192 + e2 * (-28 - 11 * e2)) / 256
    return (t - eps) / (1 + eps)


def _C2f(eps):
    e2, d, c = eps * eps, eps, [0.0] * 7
    c[1] = d * (16 + e2 * (2 + e2)) / 32
    d *= eps
    c[2] = d * (384 + e2 * (64 + 35 * e2)) / 2048
    d *= eps
    c[3] = d * (80 + 15 * e2) / 768
    d *= eps
    c[4] = d * (35 + 7 * e2) / 512
    d *= eps
    c[5] = 63 * d / 1280
    d *= eps
    c[6] = 77 * d / 2048
    return c


def _A3f(eps):
    n = N
    c1, c2, c3, c4, c5 = (n - 1) / 2, (n * (3 * n - 1) - 2) / 8, ((-n - 3) * n - 1) / 16, (-2 * n - 3) / 64, -3.0 / 128
    return 1 + eps * (c1 + eps * (c2 + eps * (c3 + eps * (c4 + eps * c5))))


def _C3f(eps):
    n, n2, d, c = N, N * N, eps, [0.0] * 6
    c[1] = d * ((1 - n) / 4 + eps * ((1 - n2) / 8 + eps * ((3 + 3 * n - n2) / 64 + eps * ((5 + 2 * n) / 128 + eps * (3.0 / 128)))))
    d *= eps
    c[2] = d * ((2 - 3 * n + n2) / 32 + eps * ((3 - 2 * n - 3 * n2) / 64 + eps * ((3 + n) / 128 + eps * (5.0 / 256))))
    d *= eps
    c[3] = d * ((5 - 9 * n + 5 * n2) / 192 + eps * ((9 - 10 * n) / 384 + eps * (7.0 / 512)))
    d *= eps
    c[4] = d * ((7 - 14 * n) / 512 + eps * (7.0 / 512))
    d *= eps
    c[5] = d * (21.0 / 2560)
    return c


def _polyval(m, p, o, x):
    y = p[o]
    for k in range(1, m + 1):
        y = y * x + p[o + k]
    return y


# geographiclib C4coeff (order 6): for l = 0..5 and j = 5..l, the coefficient of eps^j in C4[l] as a polynomial in n of order
# 5 - j (highest power first) over an integer denominator
_C4_COEFF = [
    97, 15015, 1088, 156, 45045, -224, -4784, 1573, 45045, -10656, 14144, -4576, -858, 45045,
    64, 624, -4576, 6864, -3003, 15015, 100, 208, 572, 3432, -12012, 30030, 45045,
    1, 9009, -2944, 468, 135135, 5792, 1040, -1287, 135135, 5952, -11648, 9152, -2574, 135135,
    -64, -624, 4576, -6864, 3003, 135135,
    8, 10725, 1856, -936, 225225, -8448, 4992, -1144, 225225, -1440, 4160, -4576, 1716, 225225,
    -136, 63063, 1024, -208, 105105, 3584, -3328, 1144, 315315,
    -128, 135135, -2560, 832, 405405,
    128, 99099,
]


def _c4x():
    out, o = [], 0
    for l in range(6):
        for j in range(5, l - 1, -1):
            m = 5 - j
            out.append(_polyval(m, [float(v) for v in _C4_COEFF], o, N) / _C4_COEFF[o + m + 1])
            o += m + 2
    return out


C4X = _c4x()


def _C4f(eps):
    c, mult, o = [0.0] * 6, 1.0, 0
    for l in range(6):
        m = 5 - l
        c[l] = mult * _polyval(m, C4X, o, eps)
        o += m + 1
        mult *= eps
    return c


def _lengths(eps, sig12, ssig1, csig1, dn1, ssig2, csig2, dn2, want_s, want_m):
    Ca = _C1f(eps)
    A1 = _A1m1f(eps)
    s12b = m12b = None
    m0 = J12 = A2 = 0.0
    if want_m:
        A2 = _A2m1f(eps)
        Cb = _C2f(eps)
        m0 = A1 - A2
        A2 = 1 + A2
    A1 = 1 + A1
    if want_s:
        B1 = _sin_series(ssig2, csig2, Ca, 6) - _sin_series(ssig1, csig1, Ca, 6)
        s12b = A1 * (sig12 + B1)
        if want_m:
            B2 = _sin_series(ssig2, csig2, Cb, 6) - _sin_series(ssig1, csig1, Cb, 6)
            J12 = m0 * sig12 + (A1 * B1 - A2 * B2)
    elif want_m:
        Cb = [0.0] + [A1 * Ca[l] - A2 * Cb[l] for l in range(1, 7)]
        J12 = m0 * sig12 + (_sin_series(ssig2, csig2, Cb, 6) - _sin_series(ssig1, csig1, Cb, 6))
    if want_m:
        m12b = dn2 * (csig1 * ssig2) - dn1 * (ssig1 * csig2) - csig1 * csig2 * J12
    return s12b, m12b


def _astroid(x, y):
    p, q = _sq(x), _sq(y)
    r = (p + q - 1) / 6
    if not (q == 0 and r <= 0):
        S = p * q / 4
        r2 = _sq(r)
        r3 = r * r2
        disc = S * (S + 2 * r3)
        u = r
        if disc >= 0:
            T3 = S + r3
            T3 += -math.sqrt(disc) if T3 < 0 else math.sqrt(disc)
            T = math.copysign(abs(T3) ** (1 / 3), T3)
            u += T + (r2 / T if T != 0 else 0)
        else:
            ang = math.atan2(math.sqrt(-disc), -(S + r3))
            u += 2 * r * math.cos(ang / 3)
        v = math.sqrt(_sq(u) + q)
        uv = q / (v - u) if u < 0 else u + v
        w = (uv - q) / (2 * v)
        return uv / (math.sqrt(uv + _sq(w)) + w)
    return 0.0


def _inverse_start(sbet1, cbet1, dn1, sbet2, cbet2, dn2, lam12, slam12, clam12):
    sig12, salp2, calp2, dnm = -1.0, 0.0, 0.0, 0.0
    sbet12 = sbet2 * cbet1 - cbet2 * sbet1
    cbet12 = cbet2 * cbet1 + sbet2 * sbet1
    sbet12a = sbet2 * cbet1 + cbet2 * sbet1
    shortline = cbet12 >= 0 and sbet12 < 0.5 and cbet2 * lam12 < 0.5
    if shortline:
        sbetm2 = _sq(sbet1 + sbet2)
        sbetm2 /= sbetm2 + _sq(cbet1 + cbet2)
        dnm = math.sqrt(1 + EP2 * sbetm2)
        omg12 = lam12 / (F1 * dnm)
        somg12, comg12 = math.sin(omg12), math.cos(omg12)
    else:
        somg12, comg12 = slam12, clam12
    salp1 = cbet2 * somg12
    if comg12 >= 0:
        calp1 = sbet12 + cbet2 * sbet1 * _sq(somg12) / (1 + comg12)
    else:
        calp1 = sbet12a - cbet2 * sbet1 * _sq(somg12) / (1 - comg12)
    ssig12 = math.hypot(salp1, calp1)
    csig12 = sbet1 * sbet2 + cbet1 * cbet2 * comg12
    if shortline and ssig12 < ETOL2:
        salp2 = cbet1 * somg12
        calp2 = sbet12 - cbet1 * sbet2 * (_sq(somg12) / (1 + comg12) if comg12 >= 0 else 1 - comg12)
        salp2, calp2 = _norm2(salp2, calp2)
        sig12 = math.atan2(ssig12, csig12)
    elif abs(N) > 0.1 or csig12 >= 0 or ssig12 >= 6 * abs(N) * math.pi * _sq(cbet1):
        pass
    else:
        lam12x = math.atan2(-slam12, -clam12)
        k2 = _sq(sbet1) * EP2
        eps = k2 / (2 * (1 + math.sqrt(1 + k2)) + k2)
        lamscale = F * cbet1 * _A3f(eps) * math.pi
        betscale = lamscale * cbet1
        x = lam12x / lamscale
        y = sbet12a / betscale
        if y > -TOL1 and x > -1 - XTHRESH:
            salp1 = min(1.0, -x)
            calp1 = -math.sqrt(1 - _sq(salp1))
        else:
            k = _astroid(x, y)
            omg12a = lamscale * (-x * k / (1 + k))
            somg12, comg12 = math.sin(omg12a), -math.cos(omg12a)
            salp1 = cbet2 * somg12
            calp1 = sbet12a - cbet2 * sbet1 * _sq(somg12) / (1 - comg12)
    if not (salp1 <= 0):
        salp1, calp1 = _norm2(salp1, calp1)
    else:
        salp1, calp1 = 1.0, 0.0
    return sig12, salp1, calp1, salp2, calp2, dnm


def _lambda12(sbet1, cbet1, dn1, sbet2, cbet2, dn2, salp1, calp1, slam120, clam120, diffp):
    if sbet1 == 0 and calp1 == 0:
        calp1 = -TINY
    salp0 = salp1 * cbet1
    calp0 = math.hypot(calp1, salp1 * sbet1)
    ssig1 = sbet1
    somg1 = salp0 * sbet1
    csig1 = comg1 = calp1 * cbet1
    ssig1, csig1 = _norm2(ssig1, csig1)
    if cbet2 != cbet1 or abs(sbet2) != -sbet1:
        calp2 = math.sqrt(_sq(calp1 * cbet1) + ((cbet2 - cbet1) * (cbet1 + cbet2) if cbet1 < -sbet1 else (sbet1 - sbet2) * (sbet1 + sbet2))) / cbet2
    else:
        calp2 = abs(calp1)
    salp2 = salp0 / cbet2 if cbet2 != cbet1 else salp1
    ssig2 = sbet2
    somg2 = salp0 * sbet2
    csig2 = comg2 = calp2 * cbet2
    ssig2, csig2 = _norm2(ssig2, csig2)
    sig12 = math.atan2(max(0.0, csig1 * ssig2 - ssig1 * csig2) + 0.0, csig1 * csig2 + ssig1 * ssig2)
    somg12 = max(0.0, comg1 * somg2 - somg1 * comg2) + 0.0
    comg12 = comg1 * comg2 + somg1 * somg2
    eta = math.atan2(somg12 * clam120 - comg12 * slam120, comg12 * clam120 + somg12 * slam120)
    k2 = _sq(calp0) * EP2
    eps = k2 / (2 * (1 + math.sqrt(1 + k2)) + k2)
    Ca = _C3f(eps)
    B312 = _sin_series(ssig2, csig2, Ca, 5) - _sin_series(ssig1, csig1, Ca, 5)
    domg12 = -F * _A3f(eps) * salp0 * (sig12 + B312)
    lam12 = eta + domg12
    dlam12 = 0.0
    if diffp:
        if calp2 == 0:
            dlam12 = -2 * F1 * dn1 / sbet1
        else:
            _, dlam12 = _lengths(eps, sig12, ssig1, csig1, dn1, ssig2, csig2, dn2, False, True)
            dlam12 *= F1 / (calp2 * cbet2)
    return lam12, salp2, calp2, sig12, ssig1, csig1, ssig2, csig2, eps, domg12, dlam12


def inverse(lon1, lat1, lon2, lat2):
    """Geodesic::wgs84().inverse -> (s12 metres, S12 square metres, the summed magnitudes of the terms that make up S12)"""
    lon12, lon12s = ang_diff(lon1, lon2)
    lonsign = -1 if math.copysign(1, lon12) < 0 else 1
    lon12 *= lonsign
    lon12s *= lonsign
    lam12 = lon12 * DEG
    slam12, clam12 = sincosde(lon12, lon12s)
    lon12s = (180.0 - lon12) - lon12s
    lat1 = _ang_round(math.nan if abs(lat1) > 90 else lat1)
    lat2 = _ang_round(math.nan if abs(lat2) > 90 else lat2)
    swapp = 1
    if abs(lat1) < abs(lat2) or lat2 != lat2:
        swapp, lonsign = -1, -lonsign
        lat1, lat2 = lat2, lat1
    latsign = 1 if math.copysign(1, lat1) < 0 else -1
    lat1 *= latsign
    lat2 *= latsign
    sbet1, cbet1 = sincosd(lat1)
    sbet1 *= F1
    sbet1, cbet1 = _norm2(sbet1, cbet1)
    cbet1 = max(TINY, cbet1)
    sbet2, cbet2 = sincosd(lat2)
    sbet2 *= F1
    sbet2, cbet2 = _norm2(sbet2, cbet2)
    cbet2 = max(TINY, cbet2)
    if cbet1 < -sbet1:
        if cbet2 == cbet1:
            sbet2 = math.copysign(sbet1, sbet2)
    elif abs(sbet2) == -sbet1:
        cbet2 = cbet1
    dn1 = math.sqrt(1 + EP2 * _sq(sbet1))
    dn2 = math.sqrt(1 + EP2 * _sq(sbet2))
    s12x = m12x = 0.0
    salp1 = calp1 = salp2 = calp2 = 0.0
    omg12, somg12, comg12 = 0.0, 2.0, 0.0
    meridian = lat1 == -90 or slam12 == 0
    if meridian:
        calp1, salp1, calp2, salp2 = clam12, slam12, 1.0, 0.0
        ssig1, csig1, ssig2, csig2 = sbet1, calp1 * cbet1, sbet2, calp2 * cbet2
        sig12 = math.atan2(max(0.0, csig1 * ssig2 - ssig1 * csig2) + 0.0, csig1 * csig2 + ssig1 * ssig2)
        s12x, m12x = _lengths(N, sig12, ssig1, csig1, dn1, ssig2, csig2, dn2, True, True)
        if sig12 < 1 or m12x >= 0:
            if sig12 < 3 * TINY or (sig12 < TOL0 and (s12x < 0 or m12x < 0)):
                sig12 = m12x = s12x = 0.0
            s12x *= B
        else:
            meridian = False
    if not meridian and sbet1 == 0 and (F <= 0 or lon12s >= F * 180):
        calp1 = calp2 = 0.0
        salp1 = salp2 = 1.0
        s12x = A * lam12
        omg12 = lam12 / F1
    elif not meridian:
        sig12, salp1, calp1, salp2, calp2, dnm = _inverse_start(sbet1, cbet1, dn1, sbet2, cbet2, dn2, lam12, slam12, clam12)
        if sig12 >= 0:
            s12x = sig12 * B * dnm
            omg12 = lam12 / (F1 * dnm)
        else:
            numit = 0
            salp1a, calp1a, salp1b, calp1b = TINY, 1.0, TINY, -1.0
            tripn = tripb = False
            while True:
                (v, salp2, calp2, sig12, ssig1, csig1, ssig2, csig2, eps, domg12, dv) = _lambda12(
                    sbet1, cbet1, dn1, sbet2, cbet2, dn2, salp1, calp1, slam12, clam12, numit < MAXIT1)
                if tripb or not (abs(v) >= (8 if tripn else 1) * TOL0) or numit == MAXIT2:
                    break
                if v > 0 and (numit > MAXIT1 or calp1 / salp1 > calp1b / salp1b):
                    salp1b, calp1b = salp1, calp1
                elif v < 0 and (numit > MAXIT1 or calp1 / salp1 < calp1a / salp1a):
                    salp1a, calp1a = salp1, calp1
                numit += 1
                if numit - 1 < MAXIT1 and dv > 0:
                    dalp1 = -v / dv
                    if abs(dalp1) < math.pi:
                        sdalp1, cdalp1 = math.sin(dalp1), math.cos(dalp1)
                        nsalp1 = salp1 * cdalp1 + calp1 * sdalp1
                        if nsalp1 > 0:
                            calp1 = calp1 * cdalp1 - salp1 * sdalp1
                            salp1 = nsalp1
                            salp1, calp1 = _norm2(salp1, calp1)
                            tripn = abs(v) <= 16 * TOL0
                            continue
                salp1 = (salp1a + salp1b) / 2
                calp1 = (calp1a + calp1b) / 2
                salp1, calp1 = _norm2(salp1, calp1)
                tripn = False
                tripb = abs(salp1a - salp1) + (calp1a - calp1) < TOLB or abs(salp1 - salp1b) + (calp1 - calp1b) < TOLB
            s12x, _ = _lengths(eps, sig12, ssig1, csig1, dn1, ssig2, csig2, dn2, True, False)
            s12x *= B
            sdomg12, cdomg12 = math.sin(domg12), math.cos(domg12)
            somg12 = slam12 * cdomg12 - clam12 * sdomg12
            comg12 = clam12 * cdomg12 + slam12 * sdomg12
    # area term
    salp0 = salp1 * cbet1
    calp0 = math.hypot(calp1, salp1 * sbet1)
    if calp0 != 0 and salp0 != 0:
        ssig1, csig1 = _norm2(sbet1, calp1 * cbet1)
        ssig2, csig2 = _norm2(sbet2, calp2 * cbet2)
        k2 = _sq(calp0) * EP2
        eps = k2 / (2 * (1 + math.sqrt(1 + k2)) + k2)
        A4 = A * A * calp0 * salp0 * E2
        Ca = _C4f(eps)
        B41, B42 = _cos_series(ssig1, csig1, Ca, 6), _cos_series(ssig2, csig2, Ca, 6)
        S12 = A4 * (B42 - B41)
        mag = abs(A4 * B41) + abs(A4 * B42)
    else:
        S12 = mag = 0.0
    if not meridian and somg12 == 2:
        somg12, comg12 = math.sin(omg12), math.cos(omg12)
    if not meridian and comg12 > -0.7071 and sbet2 - sbet1 < 1.75:
        domg12, dbet1, dbet2 = 1 + comg12, 1 + cbet1, 1 + cbet2
        alp12 = 2 * math.atan2(somg12 * (sbet1 * dbet2 + sbet2 * dbet1), domg12 * (sbet1 * sbet2 + dbet1 * dbet2))
    else:
        salp12 = salp2 * calp1 - calp2 * salp1
        calp12 = calp2 * calp1 + salp2 * salp1
        if salp12 == 0 and calp12 < 0:
            salp12 = TINY * calp1
            calp12 = -1.0
        alp12 = math.atan2(salp12, calp12)
    S12 += C2 * alp12
    S12 *= swapp * lonsign * latsign
    return 0.0 + s12x, S12 + 0.0, mag + abs(C2 * alp12)


def transit(lon1, lon2):
    lon12, _ = ang_diff(lon1, lon2)
    lon1, lon2 = ang_normalize(lon1), ang_normalize(lon2)
    if lon12 > 0 and ((lon1 < 0 <= lon2) or (lon1 > 0 and lon2 == 0)):
        return 1
    return -1 if (lon12 < 0 and lon2 < 0 <= lon1) else 0


class _Acc:
    """geographiclib Accumulator"""

    def __init__(self):
        self.s, self.t = 0.0, 0.0

    def add(self, y):
        z, u = _sum(y, self.t)
        self.s, self.t = _sum(z, self.s)
        if self.s == 0:
            self.s = u
        else:
            self.t += u


def _reduce(acc, crossings, reverse, sign):
    acc.s = math.remainder(acc.s, AREA0)
    acc.add(0.0)
    if crossings & 1:
        acc.add((1 if acc.s < 0 else -1) * AREA0 / 2)
    if not reverse:
        acc.s, acc.t = -acc.s, -acc.t
    if sign:
        if acc.s > AREA0 / 2:
            acc.add(-AREA0)
        elif acc.s <= -AREA0 / 2:
            acc.add(AREA0)
    else:
        if acc.s >= AREA0:
            acc.add(-AREA0)
        elif acc.s < 0:
            acc.add(AREA0)
    return 0.0 + acc.s


def _ok(p):
    return math.isfinite(p[0]) and math.isfinite(p[1]) and abs(p[1]) <= 90


def ring(coords, reverse=False, sign=True):
    """PolygonArea over the vertices (lon, lat), closing edge included -> (area, perimeter, scale); None if a coordinate is
    non-finite or has |lat| > 90"""
    pts = [(float(x), float(y)) for x, y in coords]
    if not all(_ok(p) for p in pts):
        return None
    if len(pts) >= 2 and pts[-1] == pts[0]:
        pts = pts[:-1]  # a closed ring sums the edges of the same ring unclosed, as gpl_geodesic_area does
    if len(pts) < 2:
        return 0.0, 0.0, 0.0
    A_, P_, cross, scale = _Acc(), _Acc(), 0, 0.0
    for i, p in enumerate(pts):
        q = pts[(i + 1) % len(pts)]
        s12, S12, mag = inverse(p[0], p[1], q[0], q[1])
        P_.add(s12)
        A_.add(S12)
        scale += mag
        cross += transit(p[0], q[0])
    return _reduce(A_, cross, reverse, sign), 0.0 + P_.s, scale


def polygon(rings, sign=True):
    """geo's geodesic_area for one polygon (a list of rings) -> (area, perimeter, scale) or None"""
    if not rings:
        return 0.0, 0.0, 0.0
    ext = ring(rings[0], False, sign)
    if ext is None:
        return None
    area, per, scale = ext
    holes = 0.0
    for r in rings[1:]:
        h = ring(r, True, sign)
        if h is None:
            return None
        holes += abs(h[0])
        per += h[1]
        scale += h[2]
    if area < 0 and holes > 0:
        holes = -holes
    return area - holes, per, scale


def geodesic_area(shapes, type_, sign=True):
    """rows as nested lists (the shapes given to GeoArrowArray.from_shapes; None = null row) -> (area, perimeter, valid,
    scale) arrays"""
    n = len(shapes)
    area, per, scale = np.full(n, np.nan), np.full(n, np.nan), np.zeros(n)
    valid = np.zeros(n, dtype=bool)
    for i, s in enumerate(shapes):
        if s is None:
            continue
        if type_ == "polygon":
            r = polygon(s, sign)
        elif type_ == "multipolygon":
            r = (0.0, 0.0, 0.0)
            for part in s:
                q = polygon(part, sign)
                if q is None:
                    r = None
                    break
                r = (r[0] + q[0], r[1] + q[1], r[2] + q[2])
        else:
            coords = [s] if type_ == "point" else (s if type_ in ("linestring", "multipoint") else [c for l in s for c in l])
            r = (0.0, 0.0, 0.0) if all(_ok(c) for c in coords) else None
        if r is not None:
            area[i], per[i], scale[i] = r
            valid[i] = True
    return area, per, valid, scale


def column_shapes(arr):
    """GeoArrowArray (Polygon / MultiPolygon) -> nested lists of rings, None for null rows"""
    from geopolars_b200 import GeometryType

    xy, go, ro = arr.xy, arr.geom_off, arr.ring_off
    valid = arr.valid
    out = []
    for g in range(len(go) - 1):
        if valid is not None and not valid[g]:
            out.append(None)
            continue
        if arr.type == GeometryType.POLYGON:
            out.append([xy[ro[r]:ro[r + 1]].tolist() for r in range(go[g], go[g + 1])])
        else:
            po = arr.part_off
            out.append([[xy[ro[r]:ro[r + 1]].tolist() for r in range(po[p], po[p + 1])] for p in range(go[g], go[g + 1])])
    return out
