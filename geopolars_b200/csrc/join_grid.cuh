// join_grid.cuh — the uniform envelope grid of the general spatial join (k_pairs.cu) and the nearest join
// (k_nearest.cu): a G x G grid over the union box of the listed envelopes, each row listed in every cell its
// envelope overlaps.
#pragma once

#include "common.cuh"

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

}  // namespace gpl
