// k_valid.cu — OGC validity of every row of any geometry column, one reason code per row (gpl_is_valid).  geo 0.27 has no
// validation; the rules and their reason numbers follow the OGC Simple Features rules and GEOS's TopologyValidationError
// (0 = valid).  DESIGN.md §4.18 has the contract and the derivation.  Every decision is an exact sign of input coordinates.
//
// Passes (polygon columns; Points and lines stop after the row pass):
//   row pass      one warp per row: non-finite coordinates (10), too few distinct points (9).
//   chunks        one warp per ring of a row still at 0: the ring's edges in chunks of 32 consecutive edges, with the box
//                 of each chunk's non-degenerate edges, and a flag per non-degenerate edge (scanned: its rank in its ring,
//                 which decides adjacency across repeated coordinates and the closing vertex).
//   row grids     a G x G grid over each row's box, G = ceil(sqrt(chunks of the row)); each chunk is listed in every cell its
//                 box overlaps, and a pair of chunks is a candidate in the one cell holding the low corner of the
//                 intersection of their boxes.  The work of a row is therefore not all pairs of its chunks.
//   edge pairs    one warp per candidate chunk pair, one edge per lane, the other chunk's edges broadcast: proper crossing
//                 or collinear overlap (5), a touch of two non-adjacent edges of one ring (6), and touches between two
//                 rings of one polygon member, written as events (count -> scan -> write).
//   touch cycles  one warp per row with events: union-find over the rings, each distinct touch point joining its rings in a
//                 star (the smallest ring to each other), a redundant union is a cycle of the ring / point graph (4).
//   ring position one warp per ring: the point just after the ring's first non-degenerate vertex (sym_point.cuh) against the
//                 shell (2), the other holes (3) or the other members (7), pruned by boxes.  Once rules 5 and 6 passed the
//                 point is on no other ring's boundary, so the test is exact.
// The rules found are OR'ed into one flag word per row; the code is the first failing rule in the order 10, 9, 5, 6, 2, 3, 7,
// 4.  Nothing depends on the order of the cell lists or of the events, so a row's code depends only on that row.
#include <math.h>

#include "common.cuh"
#include "join_grid.cuh"
#include "output.cuh"
#include "pair_dist.cuh"
#include "scan.cuh"
#include "sym_point.cuh"

namespace gpl {

enum : uint32_t { VF_CROSS = 1u, VF_RING_TOUCH = 2u, VF_HOLE_OUT = 4u, VF_NESTED_HOLES = 8u, VF_NESTED_SHELLS = 16u, VF_DISCONNECTED = 32u };

struct ValidTouch {  // two rings of one polygon member touch at the input vertex (x, y); ring_a < ring_b
    int64_t ring_a, ring_b;
    double x, y;
};

__device__ __forceinline__ bool finite2(double2 q) { return isfinite(q.x) && isfinite(q.y); }
__device__ __forceinline__ bool same2(double2 a, double2 b) { return a.x == b.x && a.y == b.y; }

// number of non-degenerate edges of the chain (warp-uniform)
__device__ __forceinline__ int64_t nd_edges(const Chain &c, int lane) {
    int64_t k = 0;
    const int64_t m = c.coords();
    for (int64_t i = lane; i + 1 < m; i += 32) k += same2(c[i], c[i + 1]) ? 0 : 1;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) k += __shfl_xor_sync(0xffffffffu, k, o);
    return k;
}

// rules 10 and 9 for every geometry type.  code: 0, 9 or 10; live: the row is not null
__global__ void __launch_bounds__(256) k_valid_rows(int type, int64_t n, const double2 *__restrict__ xy, const int64_t *__restrict__ go,
                                                    const int64_t *__restrict__ po, const int64_t *__restrict__ ro,
                                                    const uint8_t *__restrict__ validity, int8_t *__restrict__ code, uint8_t *__restrict__ live) {
    const int lane = threadIdx.x & 31;
    int64_t warp = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
    const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t r = warp; r < n; r += nwarps) {
        const bool ok = bit_get(validity, r);
        int c = 0;
        if (ok) {
            int64_t c0 = r, c1 = r + 1;  // the row's coordinates
            if (type == GPL_MULTIPOINT || type == GPL_LINESTRING) c0 = go[r], c1 = go[r + 1];
            else if (type == GPL_MULTILINESTRING || type == GPL_POLYGON) c0 = ro[go[r]], c1 = ro[go[r + 1]];
            else if (type == GPL_MULTIPOLYGON) c0 = ro[po[go[r]]], c1 = ro[po[go[r + 1]]];
            bool fin = true;
            for (int64_t i = c0 + lane; i < c1; i += 32) {
                const double2 q = xy[i];
                fin = fin && (finite2(q) || (type == GPL_POINT && isnan(q.x) && isnan(q.y)));
            }
            if (!__all_sync(0xffffffffu, fin)) c = 10;
            else if (type == GPL_LINESTRING) {
                if (c1 > c0 && nd_edges(make_line(xy, c0, c1), lane) == 0) c = 9;
            } else if (type != GPL_POINT && type != GPL_MULTIPOINT) {  // lines of a MultiLineString, rings of a (Multi)Polygon
                const int64_t g0 = type == GPL_MULTIPOLYGON ? po[go[r]] : go[r], g1 = type == GPL_MULTIPOLYGON ? po[go[r + 1]] : go[r + 1];
                const bool rings = type != GPL_MULTILINESTRING;
                for (int64_t g = g0; g < g1 && c == 0; ++g) {
                    if (ro[g + 1] == ro[g]) continue;
                    const int64_t k = nd_edges(rings ? make_ring(xy, ro[g], ro[g + 1]) : make_line(xy, ro[g], ro[g + 1]), lane);
                    if (k < (rings ? 3 : 1)) c = 9;
                }
            }
        }
        if (lane == 0) code[r] = (int8_t)c, live[r] = ok ? 1 : 0;
    }
}

__device__ __forceinline__ int64_t ring_edges(const Chain &c) { return c.n >= 2 ? c.coords() - 1 : 0; }
__device__ __forceinline__ void member_range(const int64_t *mo, int64_t r, int64_t &m0, int64_t &m1) {
    m0 = mo ? mo[r] : r, m1 = mo ? mo[r + 1] : r + 1;
}

// thread per row: member -> row, ring -> member, and the chunk count of each ring of a row still at 0 (others get none)
__global__ void k_valid_ring_rows(int64_t n, Side v, const int64_t *__restrict__ mo, const int8_t *__restrict__ code,
                                  const uint8_t *__restrict__ live, int64_t *__restrict__ member_row, int64_t *__restrict__ ring_member,
                                  int64_t *__restrict__ chunks) {
    const int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (r >= n) return;
    const bool act = live[r] && code[r] == 0;
    int64_t m0, m1;
    member_range(mo, r, m0, m1);
    for (int64_t m = m0; m < m1; ++m) {
        member_row[m] = r;
        for (int64_t g = v.go[m]; g < v.go[m + 1]; ++g) {
            ring_member[g] = m;
            chunks[g] = act ? (ring_edges(part_ring(v, g)) + 31) / 32 : 0;
        }
    }
}

// warp per ring with chunks: chunk records (ring, box of the chunk's non-degenerate edges; an empty box has x0 > x1), the
// ring's box, and nd[start coordinate of each non-degenerate edge] = 1 (nd zeroed by the host)
__global__ void __launch_bounds__(256) k_valid_chunks(int64_t n_rings, Side v, const int64_t *__restrict__ chunk_off,
                                                      int64_t *__restrict__ chunk_ring, double4 *__restrict__ chunk_box,
                                                      double4 *__restrict__ ring_box, uint8_t *__restrict__ nd) {
    const int lane = threadIdx.x & 31;
    int64_t warp = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
    const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    const double inf = __longlong_as_double(0x7ff0000000000000LL);
    for (int64_t g = warp; g < n_rings; g += nwarps) {
        const int64_t k0 = chunk_off[g], k1 = chunk_off[g + 1];
        if (k1 == k0) continue;
        const Chain c = part_ring(v, g);
        const int64_t ne = ring_edges(c);
        double rx0 = inf, ry0 = inf, rx1 = -inf, ry1 = -inf;
        for (int64_t k = k0; k < k1; ++k) {
            const int64_t e = (k - k0) * 32 + lane;
            double x0 = inf, y0 = inf, x1 = -inf, y1 = -inf;
            if (e < ne) {
                const double2 p = c[e], q = c[e + 1];
                if (!same2(p, q)) {
                    nd[v.ro[g] + e] = 1;
                    x0 = fmin(p.x, q.x), y0 = fmin(p.y, q.y), x1 = fmax(p.x, q.x), y1 = fmax(p.y, q.y);
                }
            }
            x0 = warp_min(x0), y0 = warp_min(y0), x1 = warp_max(x1), y1 = warp_max(y1);
            if (lane == 0) chunk_ring[k] = g, chunk_box[k] = make_double4(x0, y0, x1, y1);
            rx0 = fmin(rx0, x0), ry0 = fmin(ry0, y0), rx1 = fmax(rx1, x1), ry1 = fmax(ry1, y1);
        }
        if (lane == 0) ring_box[g] = make_double4(rx0, ry0, rx1, ry1);
    }
}

// warp per row: the row's grid over the union of its chunk boxes (g = 0: no chunk with an edge) and its cell count
__global__ void __launch_bounds__(256) k_valid_row_grid(int64_t n, Side v, const int64_t *__restrict__ mo, const int64_t *__restrict__ chunk_off,
                                                        const double4 *__restrict__ chunk_box, JoinGrid *__restrict__ grid,
                                                        int64_t *__restrict__ cells) {
    const int lane = threadIdx.x & 31;
    int64_t warp = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
    const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    const double inf = __longlong_as_double(0x7ff0000000000000LL);
    for (int64_t r = warp; r < n; r += nwarps) {
        int64_t m0, m1;
        member_range(mo, r, m0, m1);
        const int64_t k0 = chunk_off[v.go[m0]], k1 = chunk_off[v.go[m1]];
        double x0 = inf, y0 = inf, x1 = -inf, y1 = -inf;
        for (int64_t k = k0 + lane; k < k1; k += 32) {
            const double4 b = chunk_box[k];
            if (b.x <= b.z) x0 = fmin(x0, b.x), y0 = fmin(y0, b.y), x1 = fmax(x1, b.z), y1 = fmax(y1, b.w);
        }
        x0 = warp_min(x0), y0 = warp_min(y0), x1 = warp_max(x1), y1 = warp_max(y1);
        if (lane == 0) {
            JoinGrid jg{x0, y0, 0.0, 0.0, 0};
            if (x0 <= x1) {
                jg.g = (int32_t)min(1024.0, ceil(sqrt((double)(k1 - k0))));
                const double w = x1 - x0, h = y1 - y0;
                jg.inv_w = (w > 0.0 && isfinite(jg.g / w)) ? jg.g / w : 0.0;
                jg.inv_h = (h > 0.0 && isfinite(jg.g / h)) ? jg.g / h : 0.0;
            }
            grid[r] = jg;
            cells[r] = (int64_t)jg.g * jg.g;
        }
    }
}

// thread per chunk: pass 0 counts the chunk into every cell of its row's grid that its box overlaps, pass 1 lists it there
template <int PASS>
__global__ void k_valid_cells(int64_t n_chunks, const int64_t *__restrict__ chunk_ring, const double4 *__restrict__ chunk_box,
                              const int64_t *__restrict__ ring_member, const int64_t *__restrict__ member_row, const JoinGrid *__restrict__ grid,
                              const int64_t *__restrict__ cell_base, unsigned long long *__restrict__ count_or_cursor, int64_t *__restrict__ items) {
    const int64_t k = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (k >= n_chunks) return;
    const double4 b = chunk_box[k];
    if (!(b.x <= b.z)) return;
    const int64_t r = member_row[ring_member[chunk_ring[k]]];
    const JoinGrid jg = grid[r];
    const int32_t cx0 = jg_cell(b.x, jg.x0, jg.inv_w, jg.g), cx1 = jg_cell(b.z, jg.x0, jg.inv_w, jg.g);
    const int32_t cy0 = jg_cell(b.y, jg.y0, jg.inv_h, jg.g), cy1 = jg_cell(b.w, jg.y0, jg.inv_h, jg.g);
    for (int32_t cy = cy0; cy <= cy1; ++cy)
        for (int32_t cx = cx0; cx <= cx1; ++cx) {
            const int64_t c = cell_base[r] + (int64_t)cy * jg.g + cx;
            if (PASS == 0) atomicAdd(&count_or_cursor[c], 1ULL);
            else items[atomicAdd(&count_or_cursor[c], 1ULL)] = k;
        }
}

// thread per cell item t (chunk a in cell c): the candidate pairs (a, b) for the items b after t in the cell whose boxes meet
// a's, taken in the cell of the low corner of the two boxes' intersection, and (a, a) in the cell of a's low corner.
// Pass 0 counts them into cnt[t], pass 1 writes them from off[t].
template <int PASS>
__global__ void k_valid_candidates(int64_t n_items, int64_t n_cells, const int64_t *__restrict__ cell_start, const int64_t *__restrict__ items,
                                   const int64_t *__restrict__ chunk_ring, const double4 *__restrict__ chunk_box,
                                   const int64_t *__restrict__ ring_member, const int64_t *__restrict__ member_row,
                                   const JoinGrid *__restrict__ grid, const int64_t *__restrict__ cell_base, int64_t *__restrict__ cnt,
                                   const int64_t *__restrict__ off, int64_t *__restrict__ pa, int64_t *__restrict__ pb) {
    const int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (t >= n_items) return;
    int64_t lo = 0, hi = n_cells - 1;  // the cell c with cell_start[c] <= t < cell_start[c + 1]
    while (lo < hi) {
        const int64_t mid = (lo + hi + 1) >> 1;
        if (cell_start[mid] <= t) lo = mid;
        else hi = mid - 1;
    }
    const int64_t c = lo, a = items[t];
    const int64_t r = member_row[ring_member[chunk_ring[a]]];
    const JoinGrid jg = grid[r];
    const int64_t local = c - cell_base[r];
    const double4 ba = chunk_box[a];
    auto cell_of = [&](double x, double y) { return (int64_t)jg_cell(y, jg.y0, jg.inv_h, jg.g) * jg.g + jg_cell(x, jg.x0, jg.inv_w, jg.g); };
    int64_t k = 0, w = PASS ? off[t] : 0;
    if (cell_of(ba.x, ba.y) == local) {
        if (PASS) pa[w] = a, pb[w] = a, ++w;
        ++k;
    }
    for (int64_t u = t + 1; u < cell_start[c + 1]; ++u) {
        const int64_t b = items[u];
        const double4 bb = chunk_box[b];
        if (bb.z < ba.x || ba.z < bb.x || bb.w < ba.y || ba.w < bb.y) continue;
        if (cell_of(fmax(ba.x, bb.x), fmax(ba.y, bb.y)) != local) continue;
        if (PASS) pa[w] = a, pb[w] = b, ++w;
        ++k;
    }
    if (!PASS) cnt[t] = k;
}

// Relation of two non-degenerate edges p-q and r-s: 0 disjoint, 1 a proper crossing or a collinear overlap of positive
// length, 2 a single common point, returned in w (always one of the four ends).
__device__ __forceinline__ int edge_relation(double2 p, double2 q, double2 r, double2 s, double2 &w) {
    if (fmax(p.x, q.x) < fmin(r.x, s.x) || fmax(r.x, s.x) < fmin(p.x, q.x) || fmax(p.y, q.y) < fmin(r.y, s.y) ||
        fmax(r.y, s.y) < fmin(p.y, q.y))
        return 0;
    const int o1 = orient_sign(p, q, r), o2 = orient_sign(p, q, s);
    if (o1 * o2 > 0) return 0;
    if (o1 == 0 && o2 == 0) {  // collinear: compare along x unless the line is vertical
        const bool ax = p.x != q.x;
        const double pp = ax ? p.x : p.y, qq = ax ? q.x : q.y, rr = ax ? r.x : r.y, ss = ax ? s.x : s.y;
        const double lo = fmax(fmin(pp, qq), fmin(rr, ss)), hi = fmin(fmax(pp, qq), fmax(rr, ss));
        if (lo < hi) return 1;
        if (lo > hi) return 0;
        w = (pp == lo) ? p : q;
        return 2;
    }
    const int o3 = orient_sign(r, s, p), o4 = orient_sign(r, s, q);
    if (o3 * o4 > 0) return 0;
    if (o1 * o2 < 0 && o3 * o4 < 0) return 1;
    w = o1 == 0 ? r : o2 == 0 ? s : o3 == 0 ? p : q;
    return 2;
}

struct ValidEdges {  // what the edge-pair kernel reads
    Side v;
    const int64_t *chunk_off, *chunk_ring, *ring_member, *member_row, *nd_off;
};

// the edge of chunk k that lane `e` owns: ends, ring, rank among the ring's non-degenerate edges and their count; false
// when the lane has no edge or a degenerate one
__device__ __forceinline__ bool chunk_edge(const ValidEdges &V, int64_t k, int e, double2 &p, double2 &q, int64_t &ring, int64_t &rank, int64_t &kring) {
    ring = V.chunk_ring[k];
    const Chain c = part_ring(V.v, ring);
    const int64_t i = (k - V.chunk_off[ring]) * 32 + e;
    if (i >= ring_edges(c)) return false;
    p = c[i], q = c[i + 1];
    if (same2(p, q)) return false;
    const int64_t base = V.nd_off[V.v.ro[ring]];
    rank = V.nd_off[V.v.ro[ring] + i] - base;
    kring = V.nd_off[V.v.ro[ring + 1]] - base;
    return true;
}

// warp per candidate chunk pair.  Pass 0: rules 5 and 6 into flags, the number of touch events into row_events and a
// has-events byte per pair.  Pass 1 (pairs with events only): the events, at cursor[row].
template <int PASS>
__global__ void __launch_bounds__(256) k_valid_edges(int64_t n_pairs, const int64_t *__restrict__ pa, const int64_t *__restrict__ pb, ValidEdges V,
                                                     uint32_t *__restrict__ flags, uint8_t *__restrict__ pair_events,
                                                     unsigned long long *__restrict__ row_events, ValidTouch *__restrict__ events) {
    const int lane = threadIdx.x & 31;
    int64_t warp = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
    const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t t = warp; t < n_pairs; t += nwarps) {
        if (PASS == 1 && !pair_events[t]) continue;
        const int64_t ka = pa[t], kb = pb[t];
        double2 p, q, s0, s1;
        int64_t ra, rka, ka_n, rb, rkb, kb_n;
        const bool ea = chunk_edge(V, ka, lane, p, q, ra, rka, ka_n);
        const bool eb = chunk_edge(V, kb, lane, s0, s1, rb, rkb, kb_n);
        const int64_t ma = V.ring_member[ra], mb = V.ring_member[rb];
        const int64_t row = V.member_row[ma];
        uint32_t f = 0;
        int nev = 0;
        unsigned mb_mask = __ballot_sync(0xffffffffu, eb);
        while (mb_mask) {
            const int j = __ffs(mb_mask) - 1;
            mb_mask &= mb_mask - 1;
            const double2 r = bcast2(s0, j), s = bcast2(s1, j);
            const int64_t rk = __shfl_sync(0xffffffffu, rkb, j);
            if (!ea || (ka == kb && j <= lane)) continue;
            double2 w;
            const int rel = edge_relation(p, q, r, s, w);
            if (rel == 1) f |= VF_CROSS;
            else if (rel == 2) {
                if (ra == rb) {
                    const int64_t d = (rk - rka + ka_n) % ka_n;
                    if (d != 1 && d != ka_n - 1) f |= VF_RING_TOUCH;
                } else if (ma == mb) {
                    if (PASS == 1) {
                        const unsigned long long slot = atomicAdd(&row_events[row], 1ULL);
                        events[slot] = ValidTouch{min(ra, rb), max(ra, rb), w.x, w.y};
                    }
                    ++nev;
                }
            }
        }
        if (PASS == 0) {
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) f |= __shfl_xor_sync(0xffffffffu, f, o), nev += __shfl_xor_sync(0xffffffffu, nev, o);
            if (lane == 0) {
                if (f) atomicOr(&flags[row], f);
                pair_events[t] = nev ? 1 : 0;
                if (nev) atomicAdd(&row_events[row], (unsigned long long)nev);
            }
        }
    }
}

__device__ __forceinline__ int64_t uf_find(int64_t *parent, int64_t x) {
    while (parent[x] != x) {
        parent[x] = parent[parent[x]];
        x = parent[x];
    }
    return x;
}

// warp per row with touch events and without rules 5 / 6: events [ev_off[r], ev_off[r + 1]).  At a touch point P every pair
// of the rings through P is an event (rule 6 excludes a ring passing P twice), so the edges (min ring at P, other ring),
// each taken once, form a spanning tree of those rings; the interior is disconnected iff some such union closes a cycle.
__global__ void __launch_bounds__(256) k_valid_touch(int64_t n, Side v, const int64_t *__restrict__ mo, const unsigned long long *__restrict__ ev_off,
                                                     const ValidTouch *__restrict__ ev, uint32_t *__restrict__ flags, int64_t *__restrict__ parent) {
    const int lane = threadIdx.x & 31;
    int64_t warp = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
    const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t r = warp; r < n; r += nwarps) {
        const int64_t e0 = (int64_t)ev_off[r], e1 = (int64_t)ev_off[r + 1];
        if (e1 == e0 || (flags[r] & (VF_CROSS | VF_RING_TOUCH))) continue;
        int64_t m0, m1;
        member_range(mo, r, m0, m1);
        for (int64_t g = v.go[m0] + lane; g < v.go[m1]; g += 32) parent[g] = g;
        __syncwarp();
        bool cycle = false;
        for (int64_t base = e0; base < e1; base += 32) {
            const int64_t i = base + lane;
            bool tree = i < e1;
            if (tree) {
                const ValidTouch a = ev[i];
                for (int64_t j = e0; j < e1 && tree; ++j) {
                    const ValidTouch b = ev[j];
                    if (b.x != a.x || b.y != a.y) continue;
                    if (b.ring_a < a.ring_a || (j < i && b.ring_a == a.ring_a && b.ring_b == a.ring_b)) tree = false;
                }
            }
            const unsigned mask = __ballot_sync(0xffffffffu, tree);
            if (lane == 0) {
                for (unsigned mm = mask; mm && !cycle; mm &= mm - 1) {
                    const ValidTouch a = ev[base + __ffs(mm) - 1];
                    const int64_t x = uf_find(parent, a.ring_a), y = uf_find(parent, a.ring_b);
                    if (x == y) cycle = true;
                    else parent[max(x, y)] = min(x, y);
                }
            }
            cycle = __shfl_sync(0xffffffffu, cycle, 0);
            if (cycle) break;
        }
        if (lane == 0 && cycle) atomicOr(&flags[r], VF_DISCONNECTED);
    }
}

__device__ __forceinline__ bool box_has(const double4 &b, double2 u) { return b.x <= u.x && u.x <= b.z && b.y <= u.y && u.y <= b.w; }

// warp per non-empty ring of a row with chunks and without rules 5 / 6: rules 2, 3 and 7 for the point just after the ring's
// first non-degenerate vertex
__global__ void __launch_bounds__(256) k_valid_rings(int64_t n_rings, Side v, const int64_t *__restrict__ mo, const int64_t *__restrict__ chunk_off,
                                                     const int64_t *__restrict__ ring_member, const int64_t *__restrict__ member_row,
                                                     const double4 *__restrict__ ring_box, uint32_t *__restrict__ flags) {
    const int lane = threadIdx.x & 31;
    int64_t warp = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
    const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t g = warp; g < n_rings; g += nwarps) {
        if (chunk_off[g + 1] == chunk_off[g]) continue;  // empty ring, or a row already decided
        const int64_t m = ring_member[g], r = member_row[m];
        if (flags[r] & (VF_CROSS | VF_RING_TOUCH)) continue;
        const Chain c = part_ring(v, g);
        int64_t i = 0;
        while (same2(c[i], c[i + 1])) ++i;  // the row pass guarantees >= 3 non-degenerate edges
        const double2 u = c[i], w = c[i + 1];
        const SymQ q{u.x, u.y, w.x, w.y, 0};
        const int64_t g0 = v.go[m], g1 = v.go[m + 1];
        uint32_t f = 0;
        if (g > g0) {
            if (v.ro[g0 + 1] == v.ro[g0] || sym_ring_pos(q, part_ring(v, g0), lane) != 2) f |= VF_HOLE_OUT;
            for (int64_t h0 = g0 + 1; h0 < g1 && !(f & VF_NESTED_HOLES); h0 += 32) {
                const int64_t h = h0 + lane;
                const bool cand = h < g1 && h != g && v.ro[h + 1] > v.ro[h] && box_has(ring_box[h], u);
                for (unsigned mm = __ballot_sync(0xffffffffu, cand); mm; mm &= mm - 1)
                    if (sym_ring_pos(q, part_ring(v, h0 + __ffs(mm) - 1), lane) == 2) {
                        f |= VF_NESTED_HOLES;
                        break;
                    }
            }
        } else if (mo) {
            const int64_t j0 = mo[r], j1 = mo[r + 1];
            for (int64_t jb = j0; jb < j1 && !(f & VF_NESTED_SHELLS); jb += 32) {
                const int64_t j = jb + lane;
                const bool cand = j < j1 && j != m && v.go[j + 1] > v.go[j] && v.ro[v.go[j] + 1] > v.ro[v.go[j]] && box_has(ring_box[v.go[j]], u);
                for (unsigned mm = __ballot_sync(0xffffffffu, cand); mm; mm &= mm - 1) {
                    const int64_t jj = jb + __ffs(mm) - 1;
                    if (sym_region_pos(v, jj, jj + 1, q, lane) == 2) {
                        f |= VF_NESTED_SHELLS;
                        break;
                    }
                }
            }
        }
        if (lane == 0 && f) atomicOr(&flags[r], f);
    }
}

// the first failing rule in the order 10, 9, 5, 6, 2, 3, 7, 4
__global__ void k_valid_finish(int64_t n, const int8_t *__restrict__ code, const uint32_t *__restrict__ flags, int8_t *__restrict__ reason) {
    const int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (r >= n) return;
    int c = code[r];
    if (c == 0 && flags) {
        const uint32_t f = flags[r];
        c = (f & VF_CROSS) ? 5 : (f & VF_RING_TOUCH) ? 6 : (f & VF_HOLE_OUT) ? 2 : (f & VF_NESTED_HOLES) ? 3 : (f & VF_NESTED_SHELLS) ? 7
            : (f & VF_DISCONNECTED) ? 4 : 0;
    }
    reason[r] = (int8_t)c;
}

template <typename T>
static int read_back(gpl_ctx *ctx, const T *dev, T &host) {
    GPL_CUDA(cudaMemcpyAsync(&host, dev, sizeof(T), cudaMemcpyDeviceToHost, ctx->stream));
    GPL_CUDA(cudaStreamSynchronize(ctx->stream));
    return GPL_OK;
}

// rules 5, 6, 2, 3, 7, 4 of the rows of a (Multi)Polygon column that the row pass left at 0, OR'ed into flags[n]
static int polygon_rules(gpl_ctx *ctx, const gpl_array *in, const int8_t *code, const uint8_t *live, uint32_t *flags) {
    const int64_t n = in->n_geoms, n_rings = in->n_rings, n_coords = in->n_coords;
    const Side v = polygon_view(in);
    const int64_t *mo = in->type == GPL_MULTIPOLYGON ? in->geom_off : nullptr;
    const int64_t n_members = mo ? in->n_parts : n;
    if (n_rings == 0) return GPL_OK;
    Scratch<int64_t> member_row, ring_member, chunks, chunk_off;
    GPL_TRY(member_row.get(ctx, (size_t)n_members));
    GPL_TRY(ring_member.get(ctx, (size_t)n_rings));
    GPL_TRY(chunks.get(ctx, (size_t)n_rings));
    GPL_TRY(chunk_off.get(ctx, (size_t)n_rings + 1));
    GPL_LAUNCH(ctx, k_valid_ring_rows, (int)ceil_div(n, 128), 128, 0, n, v, mo, code, live, member_row.p, ring_member.p, chunks.p);
    GPL_TRY((exclusive_scan<int64_t, int64_t>(ctx, chunks.p, n_rings, chunk_off.p, nullptr)));
    int64_t n_chunks = 0;
    GPL_TRY(read_back(ctx, chunk_off.p + n_rings, n_chunks));
    if (n_chunks == 0) return GPL_OK;

    Scratch<int64_t> chunk_ring, nd_off, cells, cell_base;
    Scratch<double4> chunk_box, ring_box;
    Scratch<uint8_t> nd;
    Scratch<JoinGrid> grid;
    GPL_TRY(chunk_ring.get(ctx, (size_t)n_chunks));
    GPL_TRY(chunk_box.get(ctx, (size_t)n_chunks));
    GPL_TRY(ring_box.get(ctx, (size_t)n_rings));
    GPL_TRY(nd.get(ctx, (size_t)n_coords));
    GPL_TRY(nd_off.get(ctx, (size_t)n_coords + 1));
    GPL_CUDA(cudaMemsetAsync(nd.p, 0, (size_t)n_coords, ctx->stream));
    GPL_LAUNCH(ctx, k_valid_chunks, warp_grid(n_rings, 8), 256, 0, n_rings, v, chunk_off.p, chunk_ring.p, chunk_box.p, ring_box.p, nd.p);
    GPL_TRY((exclusive_scan<uint8_t, int64_t>(ctx, nd.p, n_coords, nd_off.p, nullptr)));

    GPL_TRY(grid.get(ctx, (size_t)n));
    GPL_TRY(cells.get(ctx, (size_t)n));
    GPL_TRY(cell_base.get(ctx, (size_t)n + 1));
    GPL_LAUNCH(ctx, k_valid_row_grid, warp_grid(n, 8), 256, 0, n, v, mo, chunk_off.p, chunk_box.p, grid.p, cells.p);
    GPL_TRY((exclusive_scan<int64_t, int64_t>(ctx, cells.p, n, cell_base.p, nullptr)));
    int64_t n_cells = 0;
    GPL_TRY(read_back(ctx, cell_base.p + n, n_cells));
    GPL_REQUIRE(n_cells > 0 && n_cells < (1LL << 40), GPL_ERR_UNSUPPORTED, "gpl_is_valid: %lld grid cells", (long long)n_cells);

    Scratch<unsigned long long> cell_count;
    Scratch<int64_t> cell_start, items;
    GPL_TRY(cell_count.get(ctx, (size_t)n_cells));
    GPL_TRY(cell_start.get(ctx, (size_t)n_cells + 1));
    GPL_CUDA(cudaMemsetAsync(cell_count.p, 0, sizeof(unsigned long long) * (size_t)n_cells, ctx->stream));
    GPL_LAUNCH(ctx, k_valid_cells<0>, (int)ceil_div(n_chunks, 128), 128, 0, n_chunks, chunk_ring.p, chunk_box.p, ring_member.p, member_row.p, grid.p,
               cell_base.p, cell_count.p, nullptr);
    GPL_TRY((exclusive_scan<unsigned long long, int64_t>(ctx, cell_count.p, n_cells, cell_start.p, nullptr)));
    int64_t n_items = 0;
    GPL_TRY(read_back(ctx, cell_start.p + n_cells, n_items));
    GPL_REQUIRE(n_items < (1LL << 31), GPL_ERR_UNSUPPORTED, "gpl_is_valid: grid too dense (%lld cell items)", (long long)n_items);
    GPL_TRY(items.get(ctx, (size_t)n_items));
    GPL_CUDA(cudaMemcpyAsync(cell_count.p, cell_start.p, sizeof(int64_t) * (size_t)n_cells, cudaMemcpyDeviceToDevice, ctx->stream));  // cursors
    GPL_LAUNCH(ctx, k_valid_cells<1>, (int)ceil_div(n_chunks, 128), 128, 0, n_chunks, chunk_ring.p, chunk_box.p, ring_member.p, member_row.p, grid.p,
               cell_base.p, cell_count.p, items.p);

    // candidate chunk pairs
    Scratch<int64_t> pair_cnt, pair_off, pa, pb;
    GPL_TRY(pair_cnt.get(ctx, (size_t)n_items));
    GPL_TRY(pair_off.get(ctx, (size_t)n_items + 1));
    GPL_LAUNCH(ctx, k_valid_candidates<0>, (int)ceil_div(n_items, 128), 128, 0, n_items, n_cells, cell_start.p, items.p, chunk_ring.p, chunk_box.p,
               ring_member.p, member_row.p, grid.p, cell_base.p, pair_cnt.p, nullptr, nullptr, nullptr);
    GPL_TRY((exclusive_scan<int64_t, int64_t>(ctx, pair_cnt.p, n_items, pair_off.p, nullptr)));
    int64_t n_pairs = 0;
    GPL_TRY(read_back(ctx, pair_off.p + n_items, n_pairs));
    GPL_TRY(pa.get(ctx, (size_t)n_pairs));
    GPL_TRY(pb.get(ctx, (size_t)n_pairs));
    GPL_LAUNCH(ctx, k_valid_candidates<1>, (int)ceil_div(n_items, 128), 128, 0, n_items, n_cells, cell_start.p, items.p, chunk_ring.p, chunk_box.p,
               ring_member.p, member_row.p, grid.p, cell_base.p, nullptr, pair_off.p, pa.p, pb.p);

    // edge pairs: rules 5 and 6, then the touch events of the rows that have some
    const ValidEdges V{v, chunk_off.p, chunk_ring.p, ring_member.p, member_row.p, nd_off.p};
    Scratch<uint8_t> pair_events;
    Scratch<unsigned long long> row_events, ev_off;
    GPL_TRY(pair_events.get(ctx, (size_t)n_pairs));
    GPL_TRY(row_events.get(ctx, (size_t)n));
    GPL_TRY(ev_off.get(ctx, (size_t)n + 1));
    GPL_CUDA(cudaMemsetAsync(row_events.p, 0, sizeof(unsigned long long) * (size_t)n, ctx->stream));
    GPL_LAUNCH(ctx, k_valid_edges<0>, warp_grid(n_pairs, 8), 256, 0, n_pairs, pa.p, pb.p, V, flags, pair_events.p, row_events.p, nullptr);
    GPL_TRY((exclusive_scan<unsigned long long, unsigned long long>(ctx, row_events.p, n, ev_off.p, nullptr)));
    unsigned long long n_events = 0;
    GPL_TRY(read_back(ctx, ev_off.p + n, n_events));
    if (n_events > 0) {
        Scratch<ValidTouch> events;
        Scratch<int64_t> parent;
        GPL_TRY(events.get(ctx, (size_t)n_events));
        GPL_TRY(parent.get(ctx, (size_t)n_rings));
        GPL_CUDA(cudaMemcpyAsync(row_events.p, ev_off.p, sizeof(unsigned long long) * (size_t)n, cudaMemcpyDeviceToDevice, ctx->stream));  // cursors
        GPL_LAUNCH(ctx, k_valid_edges<1>, warp_grid(n_pairs, 8), 256, 0, n_pairs, pa.p, pb.p, V, flags, pair_events.p, row_events.p, events.p);
        GPL_LAUNCH(ctx, k_valid_touch, warp_grid(n, 8), 256, 0, n, v, mo, ev_off.p, events.p, flags, parent.p);
        GPL_CUDA(cudaStreamSynchronize(ctx->stream));  // the event tables return to the cache when this scope ends
    }
    GPL_LAUNCH(ctx, k_valid_rings, warp_grid(n_rings, 8), 256, 0, n_rings, v, mo, chunk_off.p, ring_member.p, member_row.p, ring_box.p, flags);
    GPL_CUDA(cudaStreamSynchronize(ctx->stream));
    return GPL_OK;
}

}  // namespace gpl

using namespace gpl;

extern "C" int gpl_is_valid(gpl_ctx *ctx, const gpl_array *in, int8_t *reason, uint8_t *out_validity, int mem) {
    GPL_REQUIRE(ctx && in && reason, GPL_ERR_INVALID_ARG, "gpl_is_valid: NULL argument");
    GPL_TRY(check_mem(mem, "gpl_is_valid"));
    GPL_CUDA(cudaSetDevice(ctx->device));
    const int64_t n = in->n_geoms;
    if (n == 0) return GPL_OK;
    Scratch<int8_t> code;
    Scratch<uint32_t> flags;
    ValidOut live;
    GPL_TRY(code.get(ctx, (size_t)n));
    GPL_TRY(live.get(ctx, out_validity, n, mem, true));
    GPL_LAUNCH(ctx, k_valid_rows, warp_grid(n, 8), 256, 0, in->type, n, reinterpret_cast<const double2 *>(in->xy), in->geom_off, in->part_off,
               in->ring_off, in->validity, code.p, live.p);
    if (is_area(in->type)) {
        GPL_TRY(flags.get(ctx, (size_t)n));
        GPL_CUDA(cudaMemsetAsync(flags.p, 0, sizeof(uint32_t) * (size_t)n, ctx->stream));
        GPL_TRY(polygon_rules(ctx, in, code.p, live.p, flags.p));
    }
    RowOut<int8_t> res;
    GPL_TRY(res.get(ctx, reason, n, mem));
    GPL_LAUNCH(ctx, k_valid_finish, (int)ceil_div(n, 256), 256, 0, n, code.p, flags.p, res.p);
    GPL_TRY(live.deliver(ctx));
    return res.deliver(ctx);
}
