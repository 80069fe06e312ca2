// haversine.cuh — geo 0.27 HaversineDistance (haversine_distance.rs, recalled) for Point x Point on the mean sphere: the one
// evaluation behind geodesic_length(method="haversine") (k_geodesic.cu) and the great-circle row-wise op and joins
// (k_geo_join.cu).  Inputs are (lon, lat) degrees, the result is metres.  `a` is not clamped: near the antipode rounding can
// push it above 1 and asin then gives NaN, as geo's expression does.
#pragma once

#include <math.h>

#include "common.cuh"

namespace gpl {

constexpr double kMeanEarthRadius = 6371008.8;  // geo MEAN_EARTH_RADIUS
constexpr double DEG = 0.017453292519943295769;

// The expression.  cos1(theta1) and cos2(theta2) give cos of the two latitudes in radians: haversine_distance computes them in
// place; a join passes the values those same operations gave earlier (cos(p.y * DEG) once per left point, cos(q.y * DEG) from
// its index), so the result has the same bits.
template <class Cos1, class Cos2>
__device__ __forceinline__ double haversine_eval(double2 p, double2 q, Cos1 &&cos1, Cos2 &&cos2) {
    double theta1 = p.y * DEG, theta2 = q.y * DEG;
    double delta_theta = (q.y - p.y) * DEG, delta_lambda = (q.x - p.x) * DEG;
    double s1 = sin(delta_theta / 2.0), s2 = sin(delta_lambda / 2.0);
    double a = s1 * s1 + cos1(theta1) * cos2(theta2) * (s2 * s2);
    double c = 2.0 * asin(sqrt(a));
    return kMeanEarthRadius * c;
}
__device__ __forceinline__ double haversine_distance(double2 p, double2 q) {
    return haversine_eval(p, q, [](double t) { return cos(t); }, [](double t) { return cos(t); });
}
__device__ __forceinline__ double haversine_with_cos(double2 p, double cos_theta1, double2 q, double cos_theta2) {
    return haversine_eval(p, q, [=](double) { return cos_theta1; }, [=](double) { return cos_theta2; });
}

}  // namespace gpl
