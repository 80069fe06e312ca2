// join_grid.cuh — the uniform envelope grid of the general spatial join (k_pairs.cu) and the nearest join
// (k_nearest.cu): a G x G grid over the union box of the listed envelopes, each row listed in every cell its
// envelope overlaps.
#pragma once

#include <string.h>

#include <cmath>

#include "common.cuh"
#include "scan.cuh"

namespace gpl {

struct JoinGrid {
    double x0, y0, inv_w, inv_h;
    int32_t g;
};
__device__ __forceinline__ int32_t jg_cell(double v, double lo, double inv, int32_t g) {
    return min(max(__double2int_rd((v - lo) * inv), 0), g - 1);  // monotone (see k_pip.cu fine_index)
}
// union box of the valid envelopes: block reduce + ordered atomics (acc[0..3] zeroed by the host)
static __global__ void __launch_bounds__(256) k_join_union(const double *__restrict__ b4, const uint8_t *__restrict__ has, int64_t n,
                                                           unsigned long long *__restrict__ acc) {
    const double inf = __longlong_as_double(0x7ff0000000000000LL);
    double x0 = inf, y0 = inf, x1 = -inf, y1 = -inf;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
        if (has[i]) x0 = fmin(x0, b4[4 * i]), y0 = fmin(y0, b4[4 * i + 1]), x1 = fmax(x1, b4[4 * i + 2]), y1 = fmax(y1, b4[4 * i + 3]);
    x0 = warp_min(x0), y0 = warp_min(y0), x1 = warp_max(x1), y1 = warp_max(y1);
    auto enc = [](double d) {
        const unsigned long long b = (unsigned long long)__double_as_longlong(d);
        return (b >> 63) ? ~b : (b | 0x8000000000000000ULL);
    };
    if ((threadIdx.x & 31) == 0 && x0 <= x1 && y0 <= y1) {
        atomicMax(acc + 0, ~enc(x0));
        atomicMax(acc + 1, ~enc(y0));
        atomicMax(acc + 2, enc(x1));
        atomicMax(acc + 3, enc(y1));
    }
}
// right rows into grid cells: pass 0 counts, pass 1 fills
template <int PASS>
__global__ void k_join_cells(const double *__restrict__ b4, const uint8_t *__restrict__ has, int64_t n, JoinGrid jg,
                             int32_t *__restrict__ count_or_cursor, int32_t *__restrict__ items) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= n || !has[i]) return;
    const int32_t cx0 = jg_cell(b4[4 * i], jg.x0, jg.inv_w, jg.g), cx1 = jg_cell(b4[4 * i + 2], jg.x0, jg.inv_w, jg.g);
    const int32_t cy0 = jg_cell(b4[4 * i + 1], jg.y0, jg.inv_h, jg.g), cy1 = jg_cell(b4[4 * i + 3], jg.y0, jg.inv_h, jg.g);
    for (int32_t cy = cy0; cy <= cy1; ++cy)
        for (int32_t cx = cx0; cx <= cx1; ++cx) {
            const int64_t c = (int64_t)cy * jg.g + cx;
            if (PASS == 0) atomicAdd(&count_or_cursor[c], 1);
            else items[atomicAdd(&count_or_cursor[c], 1)] = (int32_t)i;
        }
}

// A built grid: the union box, the grid (g == 0 when no envelope is listed), and the cell lists (cell c holds
// items[cell_start[c] .. cell_start[c + 1]), G * G + 1 offsets and n_items + 1 entries).
struct GridBuild {
    double ux0 = 0.0, uy0 = 0.0, ux1 = 0.0, uy1 = 0.0;
    JoinGrid jg{0.0, 0.0, 0.0, 0.0, 0};
    int64_t n_items = 0;
    Scratch<int32_t> cell_start, items;
};

// The grid over the envelopes b4[i] with has[i] of n rows.  G = ceil(sqrt(n_g)) capped at 2048; a box without width
// (height) gets inv_w = 0 (inv_h = 0), so every x (y) maps to cell 0.  More than 2^31 - 1 cell items: GPL_ERR_UNSUPPORTED
// with the message "<what>: grid too dense".
static int join_grid_build(gpl_ctx *ctx, const double *b4, const uint8_t *has, int64_t n, int64_t n_g, const char *what, GridBuild &out) {
    Scratch<unsigned long long> acc;
    GPL_TRY(acc.get(ctx, 4));
    GPL_CUDA(cudaMemsetAsync(acc.p, 0, 4 * sizeof(unsigned long long), ctx->stream));
    GPL_LAUNCH(ctx, k_join_union, (int)std::min<int64_t>(ceil_div(n, 256), kSMs * 8), 256, 0, b4, has, n, acc.p);
    unsigned long long h_acc[4];
    GPL_CUDA(cudaMemcpyAsync(h_acc, acc.p, sizeof(h_acc), cudaMemcpyDeviceToHost, ctx->stream));
    GPL_CUDA(cudaStreamSynchronize(ctx->stream));
    if (h_acc[2] == 0ULL) return GPL_OK;  // no envelope listed
    auto dec = [](unsigned long long u) {  // the inverse of k_join_union's order-preserving encoding
        const unsigned long long b = (u >> 63) ? (u & 0x7fffffffffffffffULL) : ~u;
        double d;
        memcpy(&d, &b, sizeof(d));
        return d;
    };
    out.ux0 = dec(~h_acc[0]), out.uy0 = dec(~h_acc[1]), out.ux1 = dec(h_acc[2]), out.uy1 = dec(h_acc[3]);
    JoinGrid &jg = out.jg;
    jg.g = (int32_t)std::min<int64_t>(2048, std::max<int64_t>(1, (int64_t)ceil(sqrt((double)n_g))));
    jg.x0 = out.ux0, jg.y0 = out.uy0;
    const double w = out.ux1 - out.ux0, h = out.uy1 - out.uy0;
    jg.inv_w = (w > 0.0 && std::isfinite(w) && std::isfinite(jg.g / w)) ? jg.g / w : 0.0;
    jg.inv_h = (h > 0.0 && std::isfinite(h) && std::isfinite(jg.g / h)) ? jg.g / h : 0.0;
    const int64_t n_cells = (int64_t)jg.g * jg.g;
    Scratch<int32_t> cell_count;
    Scratch<int64_t> tot;
    GPL_TRY(cell_count.get(ctx, (size_t)n_cells + 1));
    GPL_TRY(out.cell_start.get(ctx, (size_t)n_cells + 1));
    GPL_TRY(tot.get(ctx, 1));
    GPL_CUDA(cudaMemsetAsync(cell_count.p, 0, sizeof(int32_t) * (n_cells + 1), ctx->stream));
    GPL_LAUNCH(ctx, k_join_cells<0>, (int)ceil_div(n, 128), 128, 0, b4, has, n, jg, cell_count.p, nullptr);
    GPL_TRY((exclusive_scan<int32_t, int32_t>(ctx, cell_count.p, n_cells, out.cell_start.p, tot.p)));
    int64_t n_items = 0;
    GPL_CUDA(cudaMemcpyAsync(&n_items, tot.p, sizeof(int64_t), cudaMemcpyDeviceToHost, ctx->stream));
    GPL_CUDA(cudaStreamSynchronize(ctx->stream));
    GPL_REQUIRE(n_items < (1LL << 31), GPL_ERR_UNSUPPORTED, "%s: grid too dense (%lld cell items)", what, (long long)n_items);
    out.n_items = n_items;
    GPL_TRY(out.items.get(ctx, (size_t)n_items + 1));
    GPL_CUDA(cudaMemcpyAsync(cell_count.p, out.cell_start.p, sizeof(int32_t) * n_cells, cudaMemcpyDeviceToDevice, ctx->stream));  // cursors
    GPL_LAUNCH(ctx, k_join_cells<1>, (int)ceil_div(n, 128), 128, 0, b4, has, n, jg, cell_count.p, out.items.p);
    return GPL_OK;
}

// The candidate stage of gpl_spatial_join (k_pairs.cu), shared with gpl_overlay_area_join, gpl_overlay_join,
// gpl_predicate_join and gpl_dissolve: every pair whose envelopes intersect (closed intervals) that passes `test`, as a list
// sorted by (lhs, rhs) in out (with_dist: its dist allocated, not written).  Both sides: fewer than 2^31 rows.
enum JoinTest {
    JOIN_POINT_IN_R,     // the Point row of lhs lies in the (Multi)Polygon / (Multi)LineString row of rhs (contains(point))
    JOIN_POINT_IN_L,     // the same with the roles swapped
    JOIN_POLY_CONTAINS,  // (Multi)Polygon lhs row contains the Polygon rhs row
    JOIN_INTERSECTS      // geo Intersects of the two rows, as gpl_intersects decides it
};
int join_candidate_pairs(gpl_ctx *ctx, const gpl_array *lhs, const gpl_array *rhs, JoinTest test, const char *who, bool with_dist, Pairs &out);

}  // namespace gpl
