// k_overlay_modes.cu — the overlay of two (Multi)Polygon columns in GeoPandas' five modes (gpl_overlay, DESIGN.md §4.23) and
// the row gather its output and the remainders' concatenated column are built with.
//
// A mode's rows are intersection rows (i, j) (gpl_overlay_join's own), left remainders (i, ABSENT) and right remainders
// (ABSENT, j) (remainder_rows, k_dissolve.cu), ABSENT = UINT64_MAX.  One thread per left row places its intersection rows and
// then its remainder, one thread per right row its remainder after every left row, so the list is sorted by (lhs, rhs) as
// unsigned values; one gather copies the selected rows of the three MultiPolygon columns into one.
#include <memory>

#include "boolean.cuh"
#include "common.cuh"
#include "join_host.cuh"
#include "output.cuh"
#include "overlay.cuh"
#include "pair_dist.cuh"
#include "scan.cuh"

namespace gpl {

struct PolySrc {
    Side v;                // POLYGON view
    const int64_t *mem;    // member offsets of a MultiPolygon column, NULL for Polygon
    const uint8_t *valid;
};
struct PolySrcs {
    PolySrc s[3];
};

// the members [m0, m1), rings [e0, e1) and coordinates [c0, c1) of row r
__device__ __forceinline__ void src_row(const PolySrc &s, int64_t r, int64_t &m0, int64_t &m1, int64_t &e0, int64_t &e1, int64_t &c0, int64_t &c1) {
    m0 = s.mem ? s.mem[r] : r, m1 = s.mem ? s.mem[r + 1] : r + 1;
    e0 = s.v.go[m0], e1 = s.v.go[m1];
    c0 = s.v.ro[e0], c1 = s.v.ro[e1];
}

__global__ void __launch_bounds__(256) k_gather_count(int64_t m, PolySrcs ps, const int8_t *__restrict__ src, const uint64_t *__restrict__ row,
                                                      int64_t *__restrict__ cm, int64_t *__restrict__ cr, int64_t *__restrict__ cc,
                                                      uint8_t *__restrict__ rv) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t k = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; k < m; k += stride) {
        const PolySrc &s = ps.s[src[k]];
        const int64_t r = (int64_t)row[k];
        int64_t m0, m1, e0, e1, c0, c1;
        src_row(s, r, m0, m1, e0, e1, c0, c1);
        cm[k] = m1 - m0, cr[k] = e1 - e0, cc[k] = c1 - c0;
        rv[k] = bit_get(s.valid, r) ? 1 : 0;
    }
}

// one warp per output row: its member, ring and coordinate offsets rebased to the output's, and its coordinates
__global__ void __launch_bounds__(256) k_gather_write(int64_t m, PolySrcs ps, const int8_t *__restrict__ src, const uint64_t *__restrict__ row,
                                                      const int64_t *__restrict__ mbase, const int64_t *__restrict__ rbase,
                                                      const int64_t *__restrict__ cbase, int64_t *__restrict__ part_off,
                                                      int64_t *__restrict__ ring_off, double2 *__restrict__ oxy) {
    const int lane = threadIdx.x & 31;
    const int64_t warp = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5, nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t k = warp; k < m; k += nwarps) {
        const PolySrc &s = ps.s[src[k]];
        int64_t m0, m1, e0, e1, c0, c1;
        src_row(s, (int64_t)row[k], m0, m1, e0, e1, c0, c1);
        const int64_t mb = mbase[k], rb = rbase[k], cb = cbase[k];
        for (int64_t t = lane; t < m1 - m0; t += 32) part_off[mb + t] = rb + s.v.go[m0 + t] - e0;
        for (int64_t t = lane; t < e1 - e0; t += 32) ring_off[rb + t] = cb + s.v.ro[e0 + t] - c0;
        for (int64_t t = lane; t < c1 - c0; t += 32) oxy[cb + t] = s.v.xy[c0 + t];
    }
}

int gather_polygons(gpl_ctx *ctx, const gpl_array *const srcs[3], const int8_t *src, const uint64_t *row, int64_t m, gpl_array **out) {
    PolySrcs ps{};
    for (int s = 0; s < 3; ++s)
        if (srcs[s]) ps.s[s] = PolySrc{polygon_view(srcs[s]), srcs[s]->type == GPL_MULTIPOLYGON ? srcs[s]->geom_off : nullptr, srcs[s]->validity};
    RaggedOut res;
    Scratch<uint8_t> rv;
    GPL_TRY(res.init(ctx, m, 3));
    GPL_TRY(rv.get(ctx, (size_t)m));
    if (m > 0) GPL_LAUNCH(ctx, k_gather_count, flat_grid(m), 256, 0, m, ps, src, row, res.count[0].p, res.count[1].p, res.count[2].p, rv.p);
    GPL_TRY(res.scan_and_allocate());
    if (m > 0)
        GPL_LAUNCH(ctx, k_gather_write, warp_grid(m, 8), 256, 0, m, ps, src, row, res.base[0].p, res.base[1].p, res.base[2].p, res.off[0].p,
                   res.off[1].p, reinterpret_cast<double2 *>(res.xy.p));
    return res.finish(rv.p, GPL_MULTIPOLYGON, out);
}

// a remainder is emitted when it has a member
__device__ __forceinline__ bool has_member(const int64_t *goff, int64_t r) { return goff && goff[r + 1] > goff[r]; }

// the output rows of left row i: its intersection rows ilb[i] .. ilb[i + 1] (ilb NULL: none), then its remainder
__global__ void __launch_bounds__(256) k_ovl_left_count(int64_t nl, const int64_t *__restrict__ ilb, const int64_t *__restrict__ lgoff,
                                                        int64_t *__restrict__ cnt) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < nl; i += stride)
        cnt[i] = (ilb ? ilb[i + 1] - ilb[i] : 0) + (has_member(lgoff, i) ? 1 : 0);
}
__global__ void __launch_bounds__(256) k_ovl_right_count(int64_t nr, const int64_t *__restrict__ rgoff, int64_t *__restrict__ cnt) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t j = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; j < nr; j += stride) cnt[j] = has_member(rgoff, j) ? 1 : 0;
}
// pairs and gather sources: source 0 the intersection rows, 1 the left remainders, 2 the right remainders
__global__ void __launch_bounds__(256) k_ovl_left_write(int64_t nl, const int64_t *__restrict__ ilb, const uint64_t *__restrict__ irhs,
                                                        const int64_t *__restrict__ lgoff, const int64_t *__restrict__ base,
                                                        uint64_t *__restrict__ plhs, uint64_t *__restrict__ prhs, int8_t *__restrict__ src,
                                                        uint64_t *__restrict__ row) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < nl; i += stride) {
        int64_t b = base[i];
        if (ilb)
            for (int64_t t = ilb[i]; t < ilb[i + 1]; ++t, ++b) plhs[b] = (uint64_t)i, prhs[b] = irhs[t], src[b] = 0, row[b] = (uint64_t)t;
        if (has_member(lgoff, i)) plhs[b] = (uint64_t)i, prhs[b] = UINT64_MAX, src[b] = 1, row[b] = (uint64_t)i;
    }
}
__global__ void __launch_bounds__(256) k_ovl_right_write(int64_t nr, const int64_t *__restrict__ rgoff, const int64_t *__restrict__ base,
                                                         const int64_t *__restrict__ n_left, uint64_t *__restrict__ plhs, uint64_t *__restrict__ prhs,
                                                         int8_t *__restrict__ src, uint64_t *__restrict__ row) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t j = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; j < nr; j += stride) {
        if (!has_member(rgoff, j)) continue;
        const int64_t b = *n_left + base[j];
        plhs[b] = UINT64_MAX, prhs[b] = (uint64_t)j, src[b] = 2, row[b] = (uint64_t)j;
    }
}
}  // namespace gpl

using namespace gpl;

extern "C" int gpl_overlay(gpl_ctx *ctx, const gpl_array *lhs, const gpl_array *rhs, int how, gpl_pairs **pairs, gpl_array **out) {
    GPL_REQUIRE(ctx && lhs && rhs && pairs && out, GPL_ERR_INVALID_ARG, "gpl_overlay: NULL argument");
    *pairs = nullptr, *out = nullptr;
    GPL_REQUIRE(how >= GPL_OVERLAY_INTERSECTION && how <= GPL_OVERLAY_DIFFERENCE, GPL_ERR_INVALID_ARG, "gpl_overlay: unknown how %d", how);
    GPL_REQUIRE(is_area(lhs->type) && is_area(rhs->type), GPL_ERR_INVALID_TYPE, "Expected (Multi)Polygon x (Multi)Polygon (found %s x %s)",
                type_name(lhs->type), type_name(rhs->type));
    const int64_t nl = lhs->n_geoms, nr = rhs->n_geoms;
    GPL_REQUIRE(nl + nr < (1LL << 31), GPL_ERR_UNSUPPORTED, "gpl_overlay: fewer than 2^31 rows in the two columns together");
    GPL_CUDA(cudaSetDevice(ctx->device));
    using ArrayPtr = std::unique_ptr<gpl_array, void (*)(gpl_array *)>;
    const bool inter = how == GPL_OVERLAY_INTERSECTION || how == GPL_OVERLAY_IDENTITY || how == GPL_OVERLAY_UNION;
    const bool right = how == GPL_OVERLAY_SYMMETRIC_DIFFERENCE || how == GPL_OVERLAY_UNION;
    gpl_pairs *ip_raw = nullptr;
    gpl_array *ia_raw = nullptr, *lr_raw = nullptr, *rr_raw = nullptr;
    if (inter) GPL_TRY(gpl_overlay_join(ctx, lhs, rhs, &ip_raw, &ia_raw));
    Pairs ip(ip_raw, gpl_pairs_free);
    ArrayPtr ia(ia_raw, gpl_array_free);
    if (how == GPL_OVERLAY_INTERSECTION) {
        *pairs = ip.release();
        *out = ia.release();
        return GPL_OK;
    }
    GPL_TRY(remainder_rows(ctx, lhs, rhs, &lr_raw));  // every mode but intersection has the left remainders
    ArrayPtr lr(lr_raw, gpl_array_free);
    if (right) GPL_TRY(remainder_rows(ctx, rhs, lhs, &rr_raw));
    ArrayPtr rr(rr_raw, gpl_array_free);
    // places: per left row its intersections and remainder, then the right remainders
    Scratch<int64_t> ilb, lcnt, lbase, rcnt, rbase, tot;
    GPL_TRY(lcnt.get(ctx, (size_t)nl));
    GPL_TRY(lbase.get(ctx, (size_t)nl + 1));
    GPL_TRY(rcnt.get(ctx, (size_t)nr));
    GPL_TRY(rbase.get(ctx, (size_t)nr + 1));
    GPL_TRY(tot.get(ctx, 2));
    if (inter) {
        GPL_TRY(ilb.get(ctx, (size_t)nl + 1));
        GPL_LAUNCH(ctx, k_lower_bounds, flat_grid(nl + 1), 256, 0, ip->lhs, ip->n, nl, ilb.p);
    }
    const int64_t *lgoff = lr->geom_off, *rgoff = rr ? rr->geom_off : nullptr;
    if (nl > 0) GPL_LAUNCH(ctx, k_ovl_left_count, flat_grid(nl), 256, 0, nl, ilb.p, lgoff, lcnt.p);
    if (nr > 0) GPL_LAUNCH(ctx, k_ovl_right_count, flat_grid(nr), 256, 0, nr, rgoff, rcnt.p);
    GPL_TRY((exclusive_scan<int64_t, int64_t>(ctx, lcnt.p, nl, lbase.p, tot.p)));
    GPL_TRY((exclusive_scan<int64_t, int64_t>(ctx, rcnt.p, nr, rbase.p, tot.p + 1)));
    int64_t h_tot[2] = {0, 0};
    GPL_CUDA(cudaMemcpyAsync(h_tot, tot.p, sizeof(h_tot), cudaMemcpyDeviceToHost, ctx->stream));
    GPL_CUDA(cudaStreamSynchronize(ctx->stream));
    const int64_t m = h_tot[0] + h_tot[1];
    Pairs res(nullptr, gpl_pairs_free);
    GPL_TRY(pairs_new(ctx, m, false, res));
    Scratch<int8_t> src;
    Scratch<uint64_t> row;
    GPL_TRY(src.get(ctx, (size_t)m));
    GPL_TRY(row.get(ctx, (size_t)m));
    if (nl > 0 && h_tot[0] > 0)
        GPL_LAUNCH(ctx, k_ovl_left_write, flat_grid(nl), 256, 0, nl, ilb.p, inter ? ip->rhs : nullptr, lgoff, lbase.p, res->lhs, res->rhs, src.p, row.p);
    if (nr > 0 && h_tot[1] > 0)
        GPL_LAUNCH(ctx, k_ovl_right_write, flat_grid(nr), 256, 0, nr, rgoff, rbase.p, tot.p, res->lhs, res->rhs, src.p, row.p);
    const gpl_array *srcs[3] = {ia.get(), lr.get(), rr.get()};
    gpl_array *g = nullptr;
    GPL_TRY(gather_polygons(ctx, srcs, src.p, row.p, m, &g));
    *pairs = res.release();
    *out = g;
    return GPL_OK;
}
