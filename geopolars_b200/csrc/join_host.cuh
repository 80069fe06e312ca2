// join_host.cuh — the host pipeline of the joins: the dense outputs of the nearest joins (k_nearest.cu, k_geo_join.cu)
// delivered to host or device memory, and the pair list every join returns, sorted by (lhs, rhs): sorted_pairs (allocation
// and per-row sort by rhs), pair_list (count, scan, write, sorted_pairs) and keep_pairs (order-preserving compaction).
#pragma once

#include <algorithm>

#include "common.cuh"
#include "output.cuh"
#include "scan.cuh"

namespace gpl {

// The dense outputs of a nearest pass: run(nid, dist, ntied) fills device buffers (dist / ntied may be NULL).  Outputs in host
// memory are filled through scratch.
template <class Run>
static int dense_outputs(gpl_ctx *ctx, int64_t n, int mem, int32_t *nid, double *dist, int32_t *ntied, Run &&run) {
    if (mem == GPL_DEVICE) return run(nid, dist, ntied);
    Scratch<double> dd;
    Scratch<int32_t> di, dt;
    GPL_TRY(di.get(ctx, (size_t)n));
    if (dist) GPL_TRY(dd.get(ctx, (size_t)n));
    if (ntied) GPL_TRY(dt.get(ctx, (size_t)n));
    GPL_TRY(run(di.p, dd.p, dt.p));
    if (n) {
        GPL_CUDA(cudaMemcpyAsync(nid, di.p, sizeof(int32_t) * n, cudaMemcpyDeviceToHost, ctx->stream));
        if (dist) GPL_CUDA(cudaMemcpyAsync(dist, dd.p, sizeof(double) * n, cudaMemcpyDeviceToHost, ctx->stream));
        if (ntied) GPL_CUDA(cudaMemcpyAsync(ntied, dt.p, sizeof(int32_t) * n, cudaMemcpyDeviceToHost, ctx->stream));
    }
    GPL_CUDA(cudaStreamSynchronize(ctx->stream));
    return GPL_OK;
}

// ---- per-row sort of a pair list by rhs, carrying d when raw_d != NULL (the rows of a segment are distinct) -----------------
constexpr int kSortSmall = 256;  // segments up to this size are sorted on chip by one warp
constexpr int kSortRadixThreads = 256;

// one warp per segment of <= kSortSmall pairs: the row ids are staged in shared memory and each pair is written at its rank.
// Larger segments are appended to big[] for k_sort_rows_large.
static __global__ void __launch_bounds__(256) k_sort_rows_small(int64_t n, const int64_t *__restrict__ off, const int32_t *__restrict__ raw,
                                                         const double *__restrict__ raw_d, uint64_t *__restrict__ lhs,
                                                         uint64_t *__restrict__ rhs, double *__restrict__ dist, int32_t *__restrict__ big,
                                                         unsigned long long *__restrict__ n_big) {
    __shared__ int32_t s_key[8][kSortSmall];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const int64_t warp = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5, nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t i = warp; i < n; i += nwarps) {
        const int64_t b = off[i], k = off[i + 1] - b;
        if (k > kSortSmall) {
            if (lane == 0) big[atomicAdd(n_big, 1ULL)] = (int32_t)i;
            continue;
        }
        for (int q = lane; q < k; q += 32) s_key[wid][q] = raw[b + q];
        __syncwarp();
        for (int q = lane; q < k; q += 32) {
            const int32_t j = s_key[wid][q];
            int r = 0;
            for (int t = 0; t < k; ++t) r += s_key[wid][t] < j;
            lhs[b + r] = (uint64_t)i;
            rhs[b + r] = (uint64_t)j;
            if (dist) dist[b + r] = raw_d[b + q];
        }
        __syncwarp();
    }
}

// one CTA per listed segment: a stable LSD radix sort of the row ids (< 2^31: four 8-bit digits), O(k) per segment, between
// (raw, raw_d) and (tmp, tmp_d); the last pass scatters into the outputs.  Within a 256-pair tile a pair's place among equal
// digits is its warp's offset plus its rank among the lanes of its warp with that digit (__match_any_sync), so the order of
// equal digits is kept.
static __global__ void __launch_bounds__(kSortRadixThreads) k_sort_rows_large(const int32_t *__restrict__ big, int64_t n_big, const int64_t *__restrict__ off,
                                                                       int32_t *__restrict__ raw, double *__restrict__ raw_d, int32_t *__restrict__ tmp,
                                                                       double *__restrict__ tmp_d, uint64_t *__restrict__ lhs,
                                                                       uint64_t *__restrict__ rhs, double *__restrict__ dist) {
    constexpr int NW = kSortRadixThreads / 32;
    __shared__ int32_t s_base[256];     // next place of each digit in this pass
    __shared__ int32_t s_wcnt[NW][256];  // the tile's per-warp digit counts, then each warp's first place per digit
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    for (int64_t s = blockIdx.x; s < n_big; s += gridDim.x) {
        const int64_t i = big[s], b = off[i], k = off[i + 1] - b;
        for (int pass = 0; pass < 4; ++pass) {
            const int shift = 8 * pass;
            const int32_t *src = (pass & 1) ? tmp + b : raw + b;
            const double *src_d = raw_d ? ((pass & 1) ? tmp_d + b : raw_d + b) : nullptr;
            int32_t *dst = (pass & 1) ? raw + b : tmp + b;
            double *dst_d = raw_d ? ((pass & 1) ? raw_d + b : tmp_d + b) : nullptr;
            s_base[threadIdx.x] = 0;
            __syncthreads();
            for (int64_t q = threadIdx.x; q < k; q += kSortRadixThreads) atomicAdd(&s_base[(src[q] >> shift) & 255], 1);
            __syncthreads();
            if (threadIdx.x == 0)
                for (int32_t d = 0, run = 0; d < 256; ++d) {
                    const int32_t c = s_base[d];
                    s_base[d] = run, run += c;
                }
            __syncthreads();
            for (int64_t t0 = 0; t0 < k; t0 += kSortRadixThreads) {
                const int64_t q = t0 + threadIdx.x;
                const bool has = q < k;
                const int32_t key = has ? src[q] : 0;
                const int dg = has ? (key >> shift) & 255 : 256 + lane;  // absent pairs match nobody
                for (int w = 0; w < NW; ++w) s_wcnt[w][threadIdx.x] = 0;
                __syncthreads();
                const unsigned peers = __match_any_sync(0xffffffffu, dg);
                const int rank = __popc(peers & ((1u << lane) - 1u));
                if (has && rank == 0) s_wcnt[wid][dg] = __popc(peers);
                __syncthreads();
                {
                    int32_t run = s_base[threadIdx.x];  // thread d owns digit d
                    for (int w = 0; w < NW; ++w) {
                        const int32_t c = s_wcnt[w][threadIdx.x];
                        s_wcnt[w][threadIdx.x] = run, run += c;
                    }
                    s_base[threadIdx.x] = run;
                }
                __syncthreads();
                if (has) {
                    const int32_t pos = s_wcnt[wid][dg] + rank;
                    if (pass < 3) {
                        dst[pos] = key;
                        if (dst_d) dst_d[pos] = src_d[q];
                    } else {
                        lhs[b + pos] = (uint64_t)i;
                        rhs[b + pos] = (uint64_t)key;
                        if (dist) dist[b + pos] = src_d[q];
                    }
                }
                __syncthreads();
            }
        }
    }
}

// The pair list of n left rows from each row's right rows raw[off[i] .. off[i + 1]) (distinct, in any order; with raw_d,
// their distances), total of them: lhs / rhs (/ dist) allocated and each row's pairs sorted by rhs (k_sort_rows_*), so the
// list is sorted by (lhs, rhs) whatever the order of raw.  raw and raw_d are overwritten.  with_dist and no raw_d: dist is
// allocated for the caller to fill.
static int sorted_pairs(gpl_ctx *ctx, int64_t n, const int64_t *off, int32_t *raw, double *raw_d, int64_t total, bool with_dist, Pairs &out) {
    GPL_TRY(pairs_new(ctx, total, with_dist, out));
    if (total == 0) return GPL_OK;
    double *dist = raw_d ? out->dist : nullptr;
    Scratch<double> tmp_d;
    Scratch<int32_t> tmp, big;
    Scratch<unsigned long long> n_big;
    // segments of more than kSortSmall pairs: at most total / (kSortSmall + 1) of them
    GPL_TRY(big.get(ctx, (size_t)(total / (kSortSmall + 1) + 1)));
    GPL_TRY(n_big.get(ctx, 1));
    GPL_CUDA(cudaMemsetAsync(n_big.p, 0, sizeof(unsigned long long), ctx->stream));
    GPL_LAUNCH(ctx, k_sort_rows_small, warp_grid(n, 8), 256, 0, n, off, raw, raw_d, out->lhs, out->rhs, dist, big.p, n_big.p);
    unsigned long long h_big = 0;
    GPL_CUDA(cudaMemcpyAsync(&h_big, n_big.p, sizeof(h_big), cudaMemcpyDeviceToHost, ctx->stream));
    GPL_CUDA(cudaStreamSynchronize(ctx->stream));
    if (h_big > 0) {
        GPL_TRY(tmp.get(ctx, (size_t)total));
        if (raw_d) GPL_TRY(tmp_d.get(ctx, (size_t)total));
        GPL_LAUNCH(ctx, k_sort_rows_large, (int)std::min<int64_t>((int64_t)h_big, (int64_t)kSMs * 8), kSortRadixThreads, 0, big.p,
                   (int64_t)h_big, off, raw, raw_d, tmp.p, tmp_d.p, out->lhs, out->rhs, dist);
    }
    GPL_CUDA(cudaStreamSynchronize(ctx->stream));  // the scratch above returns to the cache when this scope ends
    return GPL_OK;
}

// A pair list of n left rows: count(cnt) writes each left row's number of pairs, a scan turns the counts into int64 offsets,
// write(off, raw, raw_d) writes each row's right rows (and, when raw_d != NULL, their distances) at its offsets in any order,
// and sorted_pairs orders them.  *out is set only on success.
template <class Count, class Write>
static int pair_list(gpl_ctx *ctx, int64_t n, bool with_dist, gpl_pairs **out, Count &&count, Write &&write) {
    Scratch<double> raw_d;
    Scratch<int32_t> cnt, raw;
    Scratch<int64_t> off;
    int64_t total = 0;
    if (n > 0) {
        GPL_TRY(cnt.get(ctx, (size_t)n));
        GPL_TRY(off.get(ctx, (size_t)n + 2));
        GPL_TRY(count(cnt.p));
        GPL_TRY((exclusive_scan<int32_t, int64_t>(ctx, cnt.p, n, off.p, off.p + n + 1)));
        GPL_CUDA(cudaMemcpyAsync(&total, off.p + n + 1, sizeof(int64_t), cudaMemcpyDeviceToHost, ctx->stream));
        GPL_CUDA(cudaStreamSynchronize(ctx->stream));
    }
    if (total > 0) {
        GPL_TRY(raw.get(ctx, (size_t)total));
        if (with_dist) GPL_TRY(raw_d.get(ctx, (size_t)total));
        GPL_TRY(write(off.p, raw.p, raw_d.p));
    }
    Pairs res(nullptr, gpl_pairs_free);
    GPL_TRY(sorted_pairs(ctx, n, off.p, raw.p, raw_d.p, total, with_dist, res));
    *out = res.release();
    return GPL_OK;
}

// in's pairs with keep[k] set, in their order (so still sorted), into out.  With goff (n + 1 geometry offsets of in's rows),
// ogoff receives the kept rows' offsets and goff[n] after them.  k_pairs.cu.
int keep_pairs(gpl_ctx *ctx, const gpl_pairs *in, const uint8_t *keep, Pairs &out, const int64_t *goff = nullptr, Scratch<int64_t> *ogoff = nullptr);

}  // namespace gpl
