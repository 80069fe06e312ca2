// overlay.cuh — what the intersection-area kernels (k_overlay.cu) and the boolean geometry ops (k_boolean.cu) share: the
// per-ring σ / box tables of a (Multi)Polygon column (k_ring_prep, defined in k_overlay.cu) and the finiteness test of a row.
#pragma once

#include "common.cuh"
#include "pair_dist.cuh"

namespace gpl {

// per-ring σ (+1: the ring is used as stored, interior on the left; -1: reversed; 0: unused) and boxes of a (Multi)Polygon
// column, from k_ring_prep
struct RingPrep {
    Side view;
    const int64_t *members;  // the MultiPolygon's geom_off, NULL for a Polygon column
    Scratch<int8_t> sigma;
    Scratch<double4> box;
};
int ring_prep(gpl_ctx *ctx, const gpl_array *g, RingPrep &out);

// every coordinate of the rings of members [m0, m1) of the POLYGON view s is finite (warp-uniform)
__device__ __forceinline__ bool members_finite(const Side &s, int64_t m0, int64_t m1, int lane) {
    bool ok = true;
    for (int64_t c = s.ro[s.go[m0]] + lane; c < s.ro[s.go[m1]]; c += 32) {
        const double2 q = s.xy[c];
        ok = ok && isfinite(q.x) && isfinite(q.y);
    }
    return __all_sync(0xffffffffu, ok);
}

}  // namespace gpl
