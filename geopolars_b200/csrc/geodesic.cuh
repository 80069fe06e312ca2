// geodesic.cuh — the WGS84 ellipsoid solvers: geo's Vincenty distance (geodesic_length(method="vincenty")) and
// Karney's inverse problem on WGS84 (arXiv:1109.4448) as geographiclib implements it and its Rust port
// geographiclib-rs that geo 0.27 calls (recalled): order-6 series, Newton on alp1 with bisection fallback, astroid starting
// guess near the antipode.  One solve behind geodesic_length(method="geodesic") (k_geodesic.cu) and the geodesic polygon
// area and perimeter (k_geodesic_area.cu).
//
// The outputs follow geographiclib's GenInverse output mask, chosen at compile time: karney_inverse<false> computes the
// distance s12 only and executes exactly the operations the distance-only solve always has; karney_inverse<true> also tracks
// the azimuths alp1 / alp2 and returns the area term S12 (the area between the geodesic and the equator, C4 series of
// order 6, plus c^2 * alp12).  Inputs are (lon, lat) degrees, outputs metres and square metres.
#pragma once

#include <math.h>

#include "common.cuh"
#include "haversine.cuh"

namespace gpl {

constexpr double kWgs84A = 6378137.0;
constexpr double kPi = 3.14159265358979323846;

constexpr double kWgs84B = 6356752.314245;  // geo POLAR_EARTH_RADIUS (Vincenty)
/* Ok(distance) -> 1, Err(FailedToConvergeError) -> 0 */
static __device__ __noinline__ int vincenty_distance(double2 p, double2 q, double *out) {
    const double a = kWgs84A, b = kWgs84B, f = (kWgs84A - kWgs84B) / kWgs84A;
    double L = (q.x - p.x) * DEG;
    double U1 = atan((1.0 - f) * tan(p.y * DEG)), U2 = atan((1.0 - f) * tan(q.y * DEG));
    double sinU1 = sin(U1), cosU1 = cos(U1), sinU2 = sin(U2), cosU2 = cos(U2);
    double cosSqAlpha, sinSigma, cos2SigmaM, cosSigma, sigma;
    double lambda = L, lambdaP;
    int iterLimit = 100;
    for (;;) {
        double sinLambda = sin(lambda), cosLambda = cos(lambda);
        double t1 = cosU2 * sinLambda, t2 = cosU1 * sinU2 - sinU1 * cosU2 * cosLambda;
        sinSigma = sqrt(t1 * t1 + t2 * t2);
        if (sinSigma == 0.0) {
            if (p.x == q.x && p.y == q.y) { /* coincident points */
                *out = 0.0;
                return 1;
            }
            return 0; /* antipodal */
        }
        cosSigma = sinU1 * sinU2 + cosU1 * cosU2 * cosLambda;
        sigma = atan2(sinSigma, cosSigma);
        double sinAlpha = cosU1 * cosU2 * sinLambda / sinSigma;
        cosSqAlpha = 1.0 - sinAlpha * sinAlpha;
        if (cosSqAlpha == 0.0) cos2SigmaM = 0.0; /* equatorial geodesics */
        else cos2SigmaM = cosSigma - 2.0 * sinU1 * sinU2 / cosSqAlpha;
        double C = f / 16.0 * cosSqAlpha * (4.0 + f * (4.0 - 3.0 * cosSqAlpha));
        lambdaP = lambda;
        lambda = L + (1.0 - C) * f * sinAlpha * (sigma + C * sinSigma * (cos2SigmaM + C * cosSigma * (-1.0 + 2.0 * cos2SigmaM * cos2SigmaM)));
        if (fabs(lambda - lambdaP) <= 1e-12) break;
        iterLimit -= 1;
        if (iterLimit == 0) break;
    }
    if (iterLimit == 0) return 0;
    double uSq = cosSqAlpha * (a * a - b * b) / (b * b);
    double A = 1.0 + uSq / 16384.0 * (4096.0 + uSq * (-768.0 + uSq * (320.0 - 175.0 * uSq)));
    double B = uSq / 1024.0 * (256.0 + uSq * (-128.0 + uSq * (74.0 - 47.0 * uSq)));
    double deltaSigma = B * sinSigma *
                        (cos2SigmaM + B / 4.0 * (cosSigma * (-1.0 + 2.0 * cos2SigmaM * cos2SigmaM) -
                                                 B / 6.0 * cos2SigmaM * (-3.0 + 4.0 * sinSigma * sinSigma) * (-3.0 + 4.0 * cos2SigmaM * cos2SigmaM)));
    *out = b * A * (sigma - deltaSigma);
    return 1;
}

/* ---- Karney inverse, WGS84 ---- */
struct kg_t {
    double a, f, f1, e2, ep2, n, b, etol2;
};
constexpr double K_TINY = 1.4916681462400413e-154;  // sqrt(DBL_MIN)
constexpr double K_TOL0 = 2.220446049250313e-16;
#define K_TOL1 (200 * K_TOL0)
#define K_TOL2 1.4901161193847656e-08 /* sqrt(tol0) */
#define K_TOLB (K_TOL0 * K_TOL2)
#define K_XTHRESH (1000 * K_TOL2)
#define K_MAXIT1 20
#define K_MAXIT2 (K_MAXIT1 + 53 + 10)
__device__ __forceinline__ double ksq(double x) { return x * x; }
__device__ __forceinline__ void knorm2(double *x, double *y) {
    double r = gpl_hypot(*x, *y);
    *x /= r;
    *y /= r;
}
__device__ __forceinline__ double ksum(double u, double v, double *t) {
    double s = u + v;
    double up = s - v;
    double vpp = s - up;
    up -= u;
    vpp -= v;
    *t = s != 0 ? 0.0 - (up + vpp) : s;
    return s;
}
__device__ __forceinline__ double kang_round(double x) {
    const double z = 1.0 / 16.0;
    double y = fabs(x);
    double w = z - y;
    y = w > 0 ? z - w : y;
    return copysign(y, x);
}
__device__ __forceinline__ double kang_diff(double x, double y, double *e) {
    double t, d = ksum(remainder(-x, 360.0), remainder(y, 360.0), &t);
    d = ksum(remainder(d, 360.0), t, &t);
    if (d == 0 || fabs(d) == 180.0) d = copysign(d, t == 0 ? y - x : -t);
    *e = t;
    return d;
}
__device__ __forceinline__ void ksincosd_q(double r, int q, double *sinx, double *cosx) {
    double s = sin(r), c = cos(r);
    switch ((unsigned)q & 3U) {
    case 0U: *sinx = s, *cosx = c; break;
    case 1U: *sinx = c, *cosx = -s; break;
    case 2U: *sinx = -s, *cosx = -c; break;
    default: *sinx = -c, *cosx = s; break;
    }
    *cosx += 0.0;
}
__device__ __forceinline__ void ksincosd(double x, double *sinx, double *cosx) {
    int q = 0;
    double r = remquo(x, 90.0, &q);
    ksincosd_q(r * DEG, q, sinx, cosx);
    if (*sinx == 0) *sinx = copysign(*sinx, x);
}
__device__ __forceinline__ void ksincosde(double x, double t, double *sinx, double *cosx) {
    int q = 0;
    double r = remquo(x, 90.0, &q);
    r = kang_round(r + t);
    ksincosd_q(r * DEG, q, sinx, cosx);
    if (*sinx == 0) *sinx = copysign(*sinx, x);
}
/* sum_{l=1..n} c[l] sin(2 l x), Clenshaw */
__device__ __forceinline__ double ksin_series(double sinx, double cosx, const double *c, int n) {
    const double *p = c + n + 1;
    double ar = 2 * (cosx - sinx) * (cosx + sinx), y0 = (n & 1) ? *--p : 0, y1 = 0;
    n /= 2;
    while (n--) {
        y1 = ar * y0 - y1 + *--p;
        y0 = ar * y1 - y0 + *--p;
    }
    return 2 * sinx * cosx * y0;
}
/* sum_{l=0..n-1} c[l] cos((2 l + 1) x), Clenshaw (SinCosSeries with sinp = false) */
__device__ __forceinline__ double kcos_series(double sinx, double cosx, const double *c, int n) {
    const double *p = c + n;
    double ar = 2 * (cosx - sinx) * (cosx + sinx), y0 = (n & 1) ? *--p : 0, y1 = 0;
    n /= 2;
    while (n--) {
        y1 = ar * y0 - y1 + *--p;
        y0 = ar * y1 - y0 + *--p;
    }
    return cosx * (y0 - y1);
}
__device__ __forceinline__ double kA1m1f(double eps) {
    double e2 = eps * eps, t = e2 * (64 + e2 * (4 + e2)) / 256;
    return (t + eps) / (1 - eps);
}
__device__ __forceinline__ void kC1f(double eps, double *c) {
    double e2 = eps * eps, d = eps;
    c[1] = d * (-16 + e2 * (6 - e2)) / 32;
    d *= eps;
    c[2] = d * (-128 + e2 * (64 - 9 * e2)) / 2048;
    d *= eps;
    c[3] = d * (9 * e2 - 16) / 768;
    d *= eps;
    c[4] = d * (3 * e2 - 5) / 512;
    d *= eps;
    c[5] = -7 * d / 1280;
    d *= eps;
    c[6] = -7 * d / 2048;
}
__device__ __forceinline__ double kA2m1f(double eps) {
    double e2 = eps * eps, t = e2 * (-192 + e2 * (-28 - 11 * e2)) / 256;
    return (t - eps) / (1 + eps);
}
__device__ __forceinline__ void kC2f(double eps, double *c) {
    double e2 = eps * eps, d = eps;
    c[1] = d * (16 + e2 * (2 + e2)) / 32;
    d *= eps;
    c[2] = d * (384 + e2 * (64 + 35 * e2)) / 2048;
    d *= eps;
    c[3] = d * (80 + 15 * e2) / 768;
    d *= eps;
    c[4] = d * (35 + 7 * e2) / 512;
    d *= eps;
    c[5] = 63 * d / 1280;
    d *= eps;
    c[6] = 77 * d / 2048;
}
__device__ __forceinline__ double kA3f(const kg_t *g, double eps) {
    double n = g->n;
    double c1 = (n - 1) / 2, c2 = (n * (3 * n - 1) - 2) / 8, c3 = ((-n - 3) * n - 1) / 16, c4 = (-2 * n - 3) / 64, c5 = -3.0 / 128;
    return 1 + eps * (c1 + eps * (c2 + eps * (c3 + eps * (c4 + eps * c5))));
}
__device__ __forceinline__ void kC3f(const kg_t *g, double eps, double *c) {
    double n = g->n, n2 = n * n, d = eps;
    c[1] = d * ((1 - n) / 4 + eps * ((1 - n2) / 8 + eps * ((3 + 3 * n - n2) / 64 + eps * ((5 + 2 * n) / 128 + eps * (3.0 / 128)))));
    d *= eps;
    c[2] = d * ((2 - 3 * n + n2) / 32 + eps * ((3 - 2 * n - 3 * n2) / 64 + eps * ((3 + n) / 128 + eps * (5.0 / 256))));
    d *= eps;
    c[3] = d * ((5 - 9 * n + 5 * n2) / 192 + eps * ((9 - 10 * n) / 384 + eps * (7.0 / 512)));
    d *= eps;
    c[4] = d * ((7 - 14 * n) / 512 + eps * (7.0 / 512));
    d *= eps;
    c[5] = d * (21.0 / 2560);
}
/* Horner: p[0] x^m + ... + p[m] (geographiclib polyval) */
__device__ __forceinline__ double kpolyval(int m, const double *p, double x) {
    double y = *p++;
    while (--m >= 0) y = y * x + *p++;
    return y;
}
/* C4 coefficients c[0..5] of the area integral I4 (geographiclib C4coeff + C4f, nC4 = 6): C4x[k] is a polynomial in n
 * over an integer denominator, c[l] = eps^l * sum_j C4x eps^(j-l).  n is a compile-time constant here, so the C4x fold. */
__device__ __forceinline__ void kC4f(const kg_t *g, double eps, double *c) {
    const double coeff[] = {
        97, 15015, 1088, 156, 45045, -224, -4784, 1573, 45045, -10656, 14144, -4576, -858, 45045,
        64, 624, -4576, 6864, -3003, 15015, 100, 208, 572, 3432, -12012, 30030, 45045,
        1, 9009, -2944, 468, 135135, 5792, 1040, -1287, 135135, 5952, -11648, 9152, -2574, 135135,
        -64, -624, 4576, -6864, 3003, 135135,
        8, 10725, 1856, -936, 225225, -8448, 4992, -1144, 225225, -1440, 4160, -4576, 1716, 225225,
        -136, 63063, 1024, -208, 105105, 3584, -3328, 1144, 315315,
        -128, 135135, -2560, 832, 405405,
        128, 99099,
    };
    double C4x[21];
    int o = 0, k = 0;
#pragma unroll
    for (int l = 0; l < 6; ++l)
#pragma unroll
        for (int j = 5; j >= l; --j) {
            const int m = 5 - j;
            C4x[k++] = kpolyval(m, coeff + o, g->n) / coeff[o + m + 1];
            o += m + 2;
        }
    double mult = 1;
    o = 0;
#pragma unroll
    for (int l = 0; l < 6; ++l) {
        const int m = 5 - l;
        c[l] = mult * kpolyval(m, C4x + o, eps);
        o += m + 1;
        mult *= eps;
    }
}
/* ps12b and/or pm12b may be nullptr */
static __device__ __noinline__ void klengths(double eps, double sig12, double ssig1, double csig1, double dn1, double ssig2, double csig2, double dn2,
                     double *ps12b, double *pm12b) {
    double Ca[7], Cb[7], m0 = 0, J12 = 0, A1, A2 = 0;
    A1 = kA1m1f(eps);
    kC1f(eps, Ca);
    if (pm12b) {
        A2 = kA2m1f(eps);
        kC2f(eps, Cb);
        m0 = A1 - A2;
        A2 = 1 + A2;
    }
    A1 = 1 + A1;
    if (ps12b) {
        double B1 = ksin_series(ssig2, csig2, Ca, 6) - ksin_series(ssig1, csig1, Ca, 6);
        *ps12b = A1 * (sig12 + B1);
        if (pm12b) {
            double B2 = ksin_series(ssig2, csig2, Cb, 6) - ksin_series(ssig1, csig1, Cb, 6);
            J12 = m0 * sig12 + (A1 * B1 - A2 * B2);
        }
    } else if (pm12b) {
        for (int l = 1; l <= 6; ++l) Cb[l] = A1 * Ca[l] - A2 * Cb[l];
        J12 = m0 * sig12 + (ksin_series(ssig2, csig2, Cb, 6) - ksin_series(ssig1, csig1, Cb, 6));
    }
    if (pm12b) *pm12b = dn2 * (csig1 * ssig2) - dn1 * (ssig1 * csig2) - csig1 * csig2 * J12;
}
__device__ __forceinline__ double kastroid(double x, double y) {
    double k, p = ksq(x), q = ksq(y), r = (p + q - 1) / 6;
    if (!(q == 0 && r <= 0)) {
        double S = p * q / 4, r2 = ksq(r), r3 = r * r2, disc = S * (S + 2 * r3), u = r;
        if (disc >= 0) {
            double T3 = S + r3;
            T3 += T3 < 0 ? -sqrt(disc) : sqrt(disc);
            double T = cbrt(T3);
            u += T + (T != 0 ? r2 / T : 0);
        } else {
            double ang = atan2(sqrt(-disc), -(S + r3));
            u += 2 * r * cos(ang / 3);
        }
        double v = sqrt(ksq(u) + q), uv = u < 0 ? q / (v - u) : u + v, w = (uv - q) / (2 * v);
        k = uv / (sqrt(uv + ksq(w)) + w);
    } else
        k = 0;
    return k;
}
static __device__ __noinline__ double kinverse_start(const kg_t *g, double sbet1, double cbet1, double dn1, double sbet2, double cbet2, double dn2, double lam12,
                             double slam12, double clam12, double *psalp1, double *pcalp1, double *psalp2, double *pcalp2, double *pdnm) {
    (void)dn1, (void)dn2;
    double sig12 = -1, salp1, calp1, salp2 = 0, calp2 = 0, dnm = 0;
    double sbet12 = sbet2 * cbet1 - cbet2 * sbet1, cbet12 = cbet2 * cbet1 + sbet2 * sbet1;
    double sbet12a = sbet2 * cbet1 + cbet2 * sbet1;
    int shortline = cbet12 >= 0 && sbet12 < 0.5 && cbet2 * lam12 < 0.5;
    double somg12, comg12, ssig12, csig12;
    if (shortline) {
        double sbetm2 = ksq(sbet1 + sbet2), omg12;
        sbetm2 /= sbetm2 + ksq(cbet1 + cbet2);
        dnm = sqrt(1 + g->ep2 * sbetm2);
        omg12 = lam12 / (g->f1 * dnm);
        somg12 = sin(omg12);
        comg12 = cos(omg12);
    } else {
        somg12 = slam12;
        comg12 = clam12;
    }
    salp1 = cbet2 * somg12;
    calp1 = comg12 >= 0 ? sbet12 + cbet2 * sbet1 * ksq(somg12) / (1 + comg12) : sbet12a - cbet2 * sbet1 * ksq(somg12) / (1 - comg12);
    ssig12 = gpl_hypot(salp1, calp1);
    csig12 = sbet1 * sbet2 + cbet1 * cbet2 * comg12;
    if (shortline && ssig12 < g->etol2) {
        salp2 = cbet1 * somg12;
        calp2 = sbet12 - cbet1 * sbet2 * (comg12 >= 0 ? ksq(somg12) / (1 + comg12) : 1 - comg12);
        knorm2(&salp2, &calp2);
        sig12 = atan2(ssig12, csig12);
    } else if (fabs(g->n) > 0.1 || csig12 >= 0 || ssig12 >= 6 * fabs(g->n) * kPi * ksq(cbet1)) {
        /* zeroth order spherical approximation is OK */
    } else {
        double x, y, lamscale, betscale;
        double lam12x = atan2(-slam12, -clam12); /* lam12 - pi */
        {
            double k2 = ksq(sbet1) * g->ep2, eps = k2 / (2 * (1 + sqrt(1 + k2)) + k2);
            lamscale = g->f * cbet1 * kA3f(g, eps) * kPi;
        }
        betscale = lamscale * cbet1;
        x = lam12x / lamscale;
        y = sbet12a / betscale;
        if (y > -K_TOL1 && x > -1 - K_XTHRESH) { /* strip near cut */
            salp1 = fmin(1.0, -x);
            calp1 = -sqrt(1 - ksq(salp1));
        } else {
            double k = kastroid(x, y);
            double omg12a = lamscale * (-x * k / (1 + k));
            somg12 = sin(omg12a);
            comg12 = -cos(omg12a);
            salp1 = cbet2 * somg12;
            calp1 = sbet12a - cbet2 * sbet1 * ksq(somg12) / (1 - comg12);
        }
    }
    if (!(salp1 <= 0)) knorm2(&salp1, &calp1);
    else {
        salp1 = 1;
        calp1 = 0;
    }
    *psalp1 = salp1;
    *pcalp1 = calp1;
    if (shortline) *pdnm = dnm;
    if (sig12 >= 0) {
        *psalp2 = salp2;
        *pcalp2 = calp2;
    }
    return sig12;
}
/* Lambda12.  AREA also returns salp2, calp2 and domg12 (the area term needs the azimuth at point 2 and omg12). */
template <bool AREA>
__device__ __forceinline__ double klambda12_impl(const kg_t *g, double sbet1, double cbet1, double dn1, double sbet2, double cbet2, double dn2,
                                                 double salp1, double calp1, double slam120, double clam120, double *psig12, double *pssig1,
                                                 double *pcsig1, double *pssig2, double *pcsig2, double *peps, int diffp, double *pdlam12,
                                                 double *psalp2, double *pcalp2, double *pdomg12) {
    double calp2, sig12, ssig1, csig1, ssig2, csig2, eps, domg12, dlam12 = 0;
    double salp0, calp0, somg1, comg1, somg2, comg2, somg12, comg12, lam12, B312, eta, k2, Ca[7];
    if (sbet1 == 0 && calp1 == 0) calp1 = -K_TINY;
    salp0 = salp1 * cbet1;
    calp0 = gpl_hypot(calp1, salp1 * sbet1);
    ssig1 = sbet1;
    somg1 = salp0 * sbet1;
    csig1 = comg1 = calp1 * cbet1;
    knorm2(&ssig1, &csig1);
    calp2 = cbet2 != cbet1 || fabs(sbet2) != -sbet1
                ? sqrt(ksq(calp1 * cbet1) + (cbet1 < -sbet1 ? (cbet2 - cbet1) * (cbet1 + cbet2) : (sbet1 - sbet2) * (sbet1 + sbet2))) / cbet2
                : fabs(calp1);
    if constexpr (AREA) {
        *psalp2 = cbet2 != cbet1 ? salp0 / cbet2 : salp1;
        *pcalp2 = calp2;
    }
    ssig2 = sbet2;
    somg2 = salp0 * sbet2;
    csig2 = comg2 = calp2 * cbet2;
    knorm2(&ssig2, &csig2);
    sig12 = atan2(fmax(0.0, csig1 * ssig2 - ssig1 * csig2) + 0.0, csig1 * csig2 + ssig1 * ssig2);
    somg12 = fmax(0.0, comg1 * somg2 - somg1 * comg2) + 0.0;
    comg12 = comg1 * comg2 + somg1 * somg2;
    eta = atan2(somg12 * clam120 - comg12 * slam120, comg12 * clam120 + somg12 * slam120);
    k2 = ksq(calp0) * g->ep2;
    eps = k2 / (2 * (1 + sqrt(1 + k2)) + k2);
    kC3f(g, eps, Ca);
    B312 = ksin_series(ssig2, csig2, Ca, 5) - ksin_series(ssig1, csig1, Ca, 5);
    domg12 = -g->f * kA3f(g, eps) * salp0 * (sig12 + B312);
    lam12 = eta + domg12;
    if (diffp) {
        if (calp2 == 0) dlam12 = -2 * g->f1 * dn1 / sbet1;
        else {
            klengths(eps, sig12, ssig1, csig1, dn1, ssig2, csig2, dn2, nullptr, &dlam12);
            dlam12 *= g->f1 / (calp2 * cbet2);
        }
    }
    *psig12 = sig12, *pssig1 = ssig1, *pcsig1 = csig1, *pssig2 = ssig2, *pcsig2 = csig2, *peps = eps;
    *pdlam12 = dlam12;
    if constexpr (AREA) *pdomg12 = domg12;
    return lam12;
}
static __device__ __noinline__ double klambda12(const kg_t *g, double sbet1, double cbet1, double dn1, double sbet2, double cbet2, double dn2, double salp1,
                        double calp1, double slam120, double clam120, double *psig12, double *pssig1, double *pcsig1, double *pssig2,
                        double *pcsig2, double *peps, int diffp, double *pdlam12) {
    return klambda12_impl<false>(g, sbet1, cbet1, dn1, sbet2, cbet2, dn2, salp1, calp1, slam120, clam120, psig12, pssig1, pcsig1, pssig2,
                                 pcsig2, peps, diffp, pdlam12, nullptr, nullptr, nullptr);
}
static __device__ __noinline__ double klambda12_area(const kg_t *g, double sbet1, double cbet1, double dn1, double sbet2, double cbet2, double dn2,
                                              double salp1, double calp1, double slam120, double clam120, double *psig12, double *pssig1,
                                              double *pcsig1, double *pssig2, double *pcsig2, double *peps, int diffp, double *pdlam12,
                                              double *psalp2, double *pcalp2, double *pdomg12) {
    return klambda12_impl<true>(g, sbet1, cbet1, dn1, sbet2, cbet2, dn2, salp1, calp1, slam120, clam120, psig12, pssig1, pcsig1, pssig2,
                                pcsig2, peps, diffp, pdlam12, psalp2, pcalp2, pdomg12);
}
__device__ __forceinline__ kg_t kwgs84(void) {
    kg_t g;
    g.a = kWgs84A;
    g.f = 1.0 / 298.257223563;
    g.f1 = 1 - g.f;
    g.e2 = g.f * (2 - g.f);
    g.ep2 = g.e2 / ksq(g.f1);
    g.n = g.f / (2 - g.f);
    g.b = g.a * g.f1;
    g.etol2 = 0.1 * K_TOL2 / sqrt(fmax(0.001, fabs(g.f)) * fmin(1.0, 1 - g.f / 2) / 2);
    return g;
}
/* authalic radius squared c^2 = (a^2 + b^2 atanh(e) / e) / 2; the ellipsoid's area is 4 pi c^2 */
__device__ __forceinline__ double kc2(const kg_t *g) {
    return (ksq(g->a) + ksq(g->b) * (atanh(sqrt(g->e2)) / sqrt(fabs(g->e2)))) / 2;
}
/* Geodesic::wgs84().inverse(lat1, lon1, lat2, lon2) -> s12 (metres).  karney_inverse(p, q) is the distance-only solve;
 * karney_inverse(p, q, &S12) also returns the area term S12 (square metres).  The optional output is a parameter pack so that
 * the distance-only instantiation keeps the two-argument signature and code it has always had. */
template <class... Out>
__device__ __noinline__ double karney_inverse(double2 p, double2 q, Out... pS12) {
    constexpr bool AREA = sizeof...(Out) == 1;
    static_assert(sizeof...(Out) <= 1, "karney_inverse(p, q) or karney_inverse(p, q, double *S12)");
    const kg_t G = kwgs84();
    const kg_t *g = &G;
    double lat1 = p.y, lon1 = p.x, lat2 = q.y, lon2 = q.x;
    double lon12s, lon12 = kang_diff(lon1, lon2, &lon12s);
    int lonsign = signbit(lon12) ? -1 : 1;
    lon12 *= lonsign;
    lon12s *= lonsign;
    double lam12 = lon12 * DEG, slam12, clam12;
    ksincosde(lon12, lon12s, &slam12, &clam12);
    lon12s = (180.0 - lon12) - lon12s;
    lat1 = kang_round(fabs(lat1) > 90 ? nan("") : lat1);
    lat2 = kang_round(fabs(lat2) > 90 ? nan("") : lat2);
    int swapp = 1;
    if (fabs(lat1) < fabs(lat2) || lat2 != lat2) {
        if constexpr (AREA) {
            swapp = -1;
            lonsign *= -1;
        }
        double t = lat1;
        lat1 = lat2;
        lat2 = t;
    }
    int latsign = signbit(lat1) ? 1 : -1;
    lat1 *= latsign;
    lat2 *= latsign;
    double sbet1, cbet1, sbet2, cbet2, s12x = 0, m12x = 0, sig12;
    /* the azimuths at both ends and omg12 (somg12 == 2: still to be computed from omg12), tracked for the area only */
    double asalp1 = 0, acalp1 = 0, asalp2 = 0, acalp2 = 0, omg12 = 0, somg12 = 2, comg12 = 0;
    ksincosd(lat1, &sbet1, &cbet1);
    sbet1 *= g->f1;
    knorm2(&sbet1, &cbet1);
    cbet1 = fmax(K_TINY, cbet1);
    ksincosd(lat2, &sbet2, &cbet2);
    sbet2 *= g->f1;
    knorm2(&sbet2, &cbet2);
    cbet2 = fmax(K_TINY, cbet2);
    if (cbet1 < -sbet1) {
        if (cbet2 == cbet1) sbet2 = copysign(sbet1, sbet2);
    } else {
        if (fabs(sbet2) == -sbet1) cbet2 = cbet1;
    }
    double dn1 = sqrt(1 + g->ep2 * ksq(sbet1)), dn2 = sqrt(1 + g->ep2 * ksq(sbet2));
    int meridian = lat1 == -90 || slam12 == 0;
    if (meridian) {
        double calp1 = clam12, calp2 = 1;
        double ssig1 = sbet1, csig1 = calp1 * cbet1, ssig2 = sbet2, csig2 = calp2 * cbet2;
        if constexpr (AREA) asalp1 = slam12, acalp1 = calp1, asalp2 = 0, acalp2 = calp2;
        sig12 = atan2(fmax(0.0, csig1 * ssig2 - ssig1 * csig2) + 0.0, csig1 * csig2 + ssig1 * ssig2);
        klengths(g->n, sig12, ssig1, csig1, dn1, ssig2, csig2, dn2, &s12x, &m12x);
        if (sig12 < 1 || m12x >= 0) {
            if (sig12 < 3 * K_TINY || (sig12 < K_TOL0 && (s12x < 0 || m12x < 0))) sig12 = m12x = s12x = 0;
            s12x *= g->b;
        } else
            meridian = 0;
    }
    if (!meridian && sbet1 == 0 && (g->f <= 0 || lon12s >= g->f * 180.0)) {
        s12x = g->a * lam12; /* geodesic runs along the equator */
        if constexpr (AREA) asalp1 = asalp2 = 1, acalp1 = acalp2 = 0, omg12 = lam12 / g->f1;
    } else if (!meridian) {
        double salp1, calp1, salp2 = 0, calp2 = 0, dnm = 0;
        sig12 = kinverse_start(g, sbet1, cbet1, dn1, sbet2, cbet2, dn2, lam12, slam12, clam12, &salp1, &calp1, &salp2, &calp2, &dnm);
        if (sig12 >= 0) {
            s12x = sig12 * g->b * dnm; /* short lines */
            if constexpr (AREA) omg12 = lam12 / (g->f1 * dnm);
        } else {
            double ssig1 = 0, csig1 = 0, ssig2 = 0, csig2 = 0, eps = 0, domg12 = 0;
            unsigned numit = 0;
            double salp1a = K_TINY, calp1a = 1, salp1b = K_TINY, calp1b = -1;
            int tripn = 0, tripb = 0;
            for (;; ++numit) {
                double dv = 0, v;
                if constexpr (AREA)
                    v = klambda12_area(g, sbet1, cbet1, dn1, sbet2, cbet2, dn2, salp1, calp1, slam12, clam12, &sig12, &ssig1, &csig1, &ssig2,
                                       &csig2, &eps, numit < K_MAXIT1, &dv, &salp2, &calp2, &domg12);
                else
                    v = klambda12(g, sbet1, cbet1, dn1, sbet2, cbet2, dn2, salp1, calp1, slam12, clam12, &sig12, &ssig1, &csig1, &ssig2,
                                  &csig2, &eps, numit < K_MAXIT1, &dv);
                if (tripb || !(fabs(v) >= (tripn ? 8 : 1) * K_TOL0) || numit == K_MAXIT2) break;
                if (v > 0 && (numit > K_MAXIT1 || calp1 / salp1 > calp1b / salp1b)) {
                    salp1b = salp1;
                    calp1b = calp1;
                } else if (v < 0 && (numit > K_MAXIT1 || calp1 / salp1 < calp1a / salp1a)) {
                    salp1a = salp1;
                    calp1a = calp1;
                }
                if (numit < K_MAXIT1 && dv > 0) {
                    double dalp1 = -v / dv;
                    if (fabs(dalp1) < kPi) {
                        double sdalp1 = sin(dalp1), cdalp1 = cos(dalp1), nsalp1 = salp1 * cdalp1 + calp1 * sdalp1;
                        if (nsalp1 > 0) {
                            calp1 = calp1 * cdalp1 - salp1 * sdalp1;
                            salp1 = nsalp1;
                            knorm2(&salp1, &calp1);
                            tripn = fabs(v) <= 16 * K_TOL0;
                            continue;
                        }
                    }
                }
                salp1 = (salp1a + salp1b) / 2;
                calp1 = (calp1a + calp1b) / 2;
                knorm2(&salp1, &calp1);
                tripn = 0;
                tripb = (fabs(salp1a - salp1) + (calp1a - calp1) < K_TOLB || fabs(salp1 - salp1b) + (calp1 - calp1b) < K_TOLB);
            }
            klengths(eps, sig12, ssig1, csig1, dn1, ssig2, csig2, dn2, &s12x, nullptr);
            s12x *= g->b;
            if constexpr (AREA) { /* omg12 = lam12 - domg12 */
                double sdomg12 = sin(domg12), cdomg12 = cos(domg12);
                somg12 = slam12 * cdomg12 - clam12 * sdomg12;
                comg12 = clam12 * cdomg12 + slam12 * sdomg12;
            }
        }
        if constexpr (AREA) asalp1 = salp1, acalp1 = calp1, asalp2 = salp2, acalp2 = calp2;
    }
    if constexpr (AREA) {
        double S12, alp12;
        const double salp0 = asalp1 * cbet1, calp0 = gpl_hypot(acalp1, asalp1 * sbet1); /* calp0 > 0 */
        if (calp0 != 0 && salp0 != 0) {
            double ssig1 = sbet1, csig1 = acalp1 * cbet1, ssig2 = sbet2, csig2 = acalp2 * cbet2;
            double k2 = ksq(calp0) * g->ep2, eps = k2 / (2 * (1 + sqrt(1 + k2)) + k2);
            double A4 = ksq(g->a) * calp0 * salp0 * g->e2, Ca[6]; /* a^2 e^2 cos(alp0) sin(alp0) */
            knorm2(&ssig1, &csig1);
            knorm2(&ssig2, &csig2);
            kC4f(g, eps, Ca);
            double B41 = kcos_series(ssig1, csig1, Ca, 6), B42 = kcos_series(ssig2, csig2, Ca, 6);
            S12 = A4 * (B42 - B41);
        } else
            S12 = 0; /* indeterminate sig1, sig2 on the equator */
        if (!meridian && somg12 == 2) {
            somg12 = sin(omg12);
            comg12 = cos(omg12);
        }
        if (!meridian && comg12 > -0.7071 && sbet2 - sbet1 < 1.75) {
            /* tan(alp12/2) = tan(omg12/2) (tan(bet1/2) + tan(bet2/2)) / (1 + tan(bet1/2) tan(bet2/2)) */
            double domg12 = 1 + comg12, dbet1 = 1 + cbet1, dbet2 = 1 + cbet2;
            alp12 = 2 * atan2(somg12 * (sbet1 * dbet2 + sbet2 * dbet1), domg12 * (sbet1 * sbet2 + dbet1 * dbet2));
        } else {
            double salp12 = asalp2 * acalp1 - acalp2 * asalp1, calp12 = acalp2 * acalp1 + asalp2 * asalp1;
            if (salp12 == 0 && calp12 < 0) {
                salp12 = K_TINY * acalp1;
                calp12 = -1;
            }
            alp12 = atan2(salp12, calp12);
        }
        S12 += kc2(g) * alp12;
        S12 *= swapp * lonsign * latsign;
        ((*pS12 = S12 + 0.0), ...);
    }
    return 0.0 + s12x;
}
__device__ __forceinline__ double karney_distance(double2 p, double2 q) { return karney_inverse(p, q); }

}  // namespace gpl
