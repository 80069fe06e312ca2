// k_dissolve.cu — dissolve: the union of the rows of each group of a (Multi)Polygon column (GeoPandas' dissolve(by=...) and
// union_all(), geo's unary_union), gpl_dissolve.  DESIGN.md §4.21 has the derivation; this is the N-row form of the union of
// k_boolean.cu (§4.19), whose node records, node order and ring assembly it shares (boolean.cuh).
//
// Every ring is used with its interior on the left.  A row is cut only against its partners: the rows of its group whose closed
// geometry it intersects (join_candidate_pairs, touching pairs included: linking at a shared point needs the edge cut there).
//   nodes     one warp per (row, partner) item, count pass, scan, write pass: node_pass of the row's edges against the
//             partner's rings, plus one item per row for its edge starts.  A crossing's point comes from the lower row's stored
//             edge first, so the two records of a crossing carry the same bits and a two-row group reproduces §4.19;
//   order     one warp per row sorts the row's records along each edge by §4.19's exact signs; two crossings whose partner edges
//             cross each other (partners overlapping near the edge) are ordered by the sign of A_k C_j - A_j C_k (A: orient2d
//             of the edge start against the partner edge, C: cross product of the two directions), a degree-4 polynomial
//             evaluated in f64 under an error bound, exactly (expansions) when the bound cannot decide.  Ties are single
//             nodes: crossings of three edges at one point take the crossing of the two lowest rows there, a crossing through a
//             third row's vertex takes that vertex;
//   classes   the number of partners that block a piece: inside, on the boundary running the opposite way, or on the boundary
//             running the same way with a lower row index.  It is recomputed at every edge start and vertex node by locating
//             the symbolic point just after it against every partner (sym_ring_pos), and changes by one at a crossing
//             (entering or leaving that partner: the exact side of the partner edge the edge's end lies on).  A piece is
//             kept when nothing blocks it;
//   rings     one thread per group links the kept pieces of all its rows into rings as §4.19 does (assemble_pieces), the
//             hole-to-shell search skipping shells by box.
#include <math.h>

#include <algorithm>
#include <memory>

#include "boolean.cuh"
#include "common.cuh"
#include "join_grid.cuh"
#include "join_host.cuh"
#include "output.cuh"
#include "overlay.cuh"
#include "pair_dist.cuh"
#include "scan.cuh"
#include "sym_point.cuh"

namespace gpl {

constexpr int kX4 = 1664;  // doubles of exact scratch per warp for the degree-4 order of two crossings

// e (len n) += a * b exactly; tmp holds n + 2 doubles
__device__ __forceinline__ int add_product(double *e, int n, double a, double b, double *tmp) {
    double p[2];
    two_product(a, b, p[1], p[0]);
    const int m = fast_expansion_sum_zeroelim(n, e, 2, p, tmp);
    for (int i = 0; i < m; ++i) e[i] = tmp[i];
    return m;
}
__device__ __forceinline__ int exp_sign(const double *e, int n) { return e[n - 1] > 0.0 ? 1 : e[n - 1] < 0.0 ? -1 : 0; }

// A = orient2d(s, g, p) (12 terms at most) and C = cross(g - s, q - p) (16 at most) exactly
__device__ int exact_a(double2 s, double2 g, double2 p, double *e, double *tmp) {
    int n = 1;
    e[0] = 0.0;
    n = add_product(e, n, g.x, p.y, tmp), n = add_product(e, n, -g.x, s.y, tmp), n = add_product(e, n, -s.x, p.y, tmp);
    n = add_product(e, n, -g.y, p.x, tmp), n = add_product(e, n, g.y, s.x, tmp), n = add_product(e, n, s.y, p.x, tmp);
    return n;
}
__device__ int exact_c(double2 s, double2 g, double2 p, double2 q, double *e, double *tmp) {
    int n = 1;
    e[0] = 0.0;
    n = add_product(e, n, g.x, q.y, tmp), n = add_product(e, n, -g.x, p.y, tmp), n = add_product(e, n, -s.x, q.y, tmp);
    n = add_product(e, n, s.x, p.y, tmp), n = add_product(e, n, -g.y, q.x, tmp), n = add_product(e, n, g.y, p.x, tmp);
    n = add_product(e, n, s.y, q.x, tmp), n = add_product(e, n, -s.y, p.x, tmp);
    return n;
}
// acc (len n) += sgn * x (len nx) * y (len ny), with buffers t (2 ny) and u (n + 2 ny)
__device__ int add_exp_product(double *acc, int n, const double *x, int nx, const double *y, int ny, double sgn, double *t, double *u) {
    for (int i = 0; i < nx; ++i) {
        const int m = scale_expansion_zeroelim(ny, y, sgn * x[i], t);
        const int k = fast_expansion_sum_zeroelim(n, acc, m, t, u);
        for (int j = 0; j < k; ++j) acc[j] = u[j];
        n = k;
    }
    return n;
}

// Order along the directed edge (p, q) of its crossings with the stored edges (s1, g1) and (s2, g2): -1 when the first comes
// first, 0 at one point.  t_k = -A_k / C_k, so sign(t_1 - t_2) = sign(A_2 C_1 - A_1 C_2) sign(C_1) sign(C_2).
__device__ int cross_order(double2 p, double2 q, double2 s1, double2 g1, double2 s2, double2 g2, double *w) {
    auto naive = [](double2 a, double2 b, double2 c, double2 d, double &err) {  // (b - a) x (d - c), bound on its error
        const double l = (b.x - a.x) * (d.y - c.y), r = (b.y - a.y) * (d.x - c.x);
        err = kCcwA * (fabs(l) + fabs(r));
        return l - r;
    };
    double e1, e2, f1, f2;
    const double A1 = naive(p, s1, p, g1, e1), A2 = naive(p, s2, p, g2, e2);  // orient2d(s, g, p) = (s - p) x (g - p)
    const double C1 = naive(s1, g1, p, q, f1), C2 = naive(s2, g2, p, q, f2);
    if (fabs(C1) > f1 && fabs(C2) > f2) {
        const double t1 = A2 * C1, t2 = A1 * C2, D = t1 - t2;
        const double err = (fabs(A2) * f1 + fabs(C1) * e2 + e2 * f1 + fabs(A1) * f2 + fabs(C2) * e1 + e1 * f2) * (1.0 + 16.0 * kEps) +
                           8.0 * kEps * (fabs(t1) + fabs(t2));
        if (fabs(D) > err) return (D > 0.0 ? 1 : -1) * (C1 > 0.0 ? 1 : -1) * (C2 > 0.0 ? 1 : -1) > 0 ? 1 : -1;
    }
    double *a1 = w, *a2 = w + 12, *c1 = w + 24, *c2 = w + 40, *tmp = w + 56, *t = w + 80, *acc = w + 112, *u = w + 112 + 768;
    const int na1 = exact_a(s1, g1, p, a1, tmp), na2 = exact_a(s2, g2, p, a2, tmp);
    const int nc1 = exact_c(s1, g1, p, q, c1, tmp), nc2 = exact_c(s2, g2, p, q, c2, tmp);
    int n = 1;
    acc[0] = 0.0;
    n = add_exp_product(acc, n, a2, na2, c1, nc1, 1.0, t, u);
    n = add_exp_product(acc, n, a1, na1, c2, nc2, -1.0, t, u);
    return exp_sign(acc, n) * exp_sign(c1, nc1) * exp_sign(c2, nc2);
}

// the records of one row: by edge, the start first, then along the edge by exact signs; at one point crossings come before
// vertices (a vertex node re-locates against every partner, so the crossings at its point must already be counted)
struct DisLess {
    const BOperands *o;
    double *x4;
    __device__ int along(const BNode &a, const BNode &b, double2 p, double2 q) const {
        if (a.kind == K_VERTEX && b.kind == K_VERTEX) {
            const int d = cmpd(q.x, p.x);
            return d ? cmpd(a.pt.x, b.pt.x) * d : cmpd(a.pt.y, b.pt.y) * cmpd(q.y, p.y);
        }
        if (a.kind == K_VERTEX || b.kind == K_VERTEX) {
            const BNode &v = a.kind == K_VERTEX ? a : b, &x = a.kind == K_VERTEX ? b : a;
            double2 s, g;
            stored_edge(*o, 0, x.oring, x.oseg, s, g);
            const int sv = orient_sign(s, g, v.pt);
            if (sv == 0) return 0;
            const int vb = sv == orient_sign(s, g, p) ? -1 : 1;
            return a.kind == K_VERTEX ? vb : -vb;
        }
        double2 s1, g1, s2, g2;
        stored_edge(*o, 0, a.oring, a.oseg, s1, g1);
        stored_edge(*o, 0, b.oring, b.oseg, s2, g2);
        int c1 = orient_sign(s1, g1, s2), c2 = orient_sign(s1, g1, g2);
        if (c1 * c2 >= 0 && (c1 | c2)) return (c1 ? c1 : c2) == orient_sign(s1, g1, p) ? 1 : -1;
        c1 = orient_sign(s2, g2, s1), c2 = orient_sign(s2, g2, g1);
        if (c1 * c2 >= 0 && (c1 | c2)) return (c1 ? c1 : c2) == orient_sign(s2, g2, p) ? -1 : 1;
        return cross_order(p, q, s1, g1, s2, g2, x4);
    }
    __device__ bool operator()(const BNode &a, const BNode &b) const {
        if (a.ring != b.ring) return a.ring < b.ring;
        if (a.seg != b.seg) return a.seg < b.seg;
        if ((a.kind == K_START) != (b.kind == K_START)) return a.kind == K_START;
        if (a.kind != K_START) {
            double2 p, q;
            dir_edge(*o, 0, a.ring, a.seg, p, q);
            const int c = along(a, b, p, q);
            if (c) return c < 0;
        }
        if (a.kind != b.kind) return a.kind > b.kind;
        if (a.oring != b.oring) return a.oring < b.oring;
        if (a.oseg != b.oseg) return a.oseg < b.oseg;
        if (a.pt.x != b.pt.x) return a.pt.x < b.pt.x;
        return a.pt.y < b.pt.y;
    }
};

// per row: 0 skipped (null, code -1), 1 present, 2 present with a non-finite coordinate (nulls its group); the row of
// every ring.  group NULL: every row in group 0, and gnull (then NULL too) is not written
__global__ void __launch_bounds__(128) k_dis_rows(int64_t n, Side v, const int64_t *__restrict__ mem, const uint8_t *__restrict__ valid,
                                                  const int64_t *__restrict__ group, uint8_t *__restrict__ status, uint8_t *__restrict__ gnull,
                                                  int64_t *__restrict__ ring_row) {
    const int lane = threadIdx.x & 31;
    const int64_t warp = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5, nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t r = warp; r < n; r += nwarps) {
        const int64_t m0 = mem ? mem[r] : r, m1 = mem ? mem[r + 1] : r + 1, g = group ? group[r] : 0;
        for (int64_t e = v.go[m0] + lane; e < v.go[m1]; e += 32) ring_row[e] = r;
        const bool present = g >= 0 && bit_get(valid, r);
        const bool finite = present ? members_finite(v, m0, m1, lane) : true;
        if (lane == 0) {
            status[r] = !present ? 0 : finite ? 1 : 2;
            if (present && !finite && gnull) gnull[g] = 1;
        }
    }
}

// the candidate pairs (i, j), i != j, of present rows of one group, in both directions, grouped by i for pair_list
__device__ __forceinline__ bool dis_pair(int64_t i, int64_t j, const uint8_t *status, const int64_t *group) {
    return i < j && status[i] == 1 && status[j] == 1 && group[i] == group[j];
}
__global__ void __launch_bounds__(256) k_dis_pair_count(int64_t n, const uint64_t *__restrict__ l, const uint64_t *__restrict__ r,
                                                        const uint8_t *__restrict__ status, const int64_t *__restrict__ group, int32_t *__restrict__ cnt) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t k = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; k < n; k += stride) {
        const int64_t i = (int64_t)l[k], j = (int64_t)r[k];
        if (!dis_pair(i, j, status, group)) continue;
        atomicAdd(&cnt[i], 1);
        atomicAdd(&cnt[j], 1);
    }
}
__global__ void __launch_bounds__(256) k_dis_pair_write(int64_t n, const uint64_t *__restrict__ l, const uint64_t *__restrict__ r,
                                                        const uint8_t *__restrict__ status, const int64_t *__restrict__ group,
                                                        const int64_t *__restrict__ off, int32_t *__restrict__ cursor, int32_t *__restrict__ raw) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t k = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; k < n; k += stride) {
        const int64_t i = (int64_t)l[k], j = (int64_t)r[k];
        if (!dis_pair(i, j, status, group)) continue;
        raw[off[i] + atomicAdd(&cursor[i], 1)] = (int32_t)j;
        raw[off[j] + atomicAdd(&cursor[j], 1)] = (int32_t)i;
    }
}
// the present rows grouped by group code for pair_list
__global__ void __launch_bounds__(256) k_dis_group_count(int64_t n, const uint8_t *__restrict__ status, const int64_t *__restrict__ group,
                                                         int32_t *__restrict__ cnt) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += stride)
        if (status[i] == 1) atomicAdd(&cnt[group[i]], 1);
}
__global__ void __launch_bounds__(256) k_dis_group_write(int64_t n, const uint8_t *__restrict__ status, const int64_t *__restrict__ group,
                                                         const int64_t *__restrict__ off, int32_t *__restrict__ cursor, int32_t *__restrict__ raw) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += stride)
        if (status[i] == 1) raw[off[group[i]] + atomicAdd(&cursor[group[i]], 1)] = (int32_t)i;
}
// out[k] = the first position of keys (sorted, length m) that is >= k, for k in [0, nq]
__global__ void __launch_bounds__(256) k_lower_bounds(const uint64_t *__restrict__ keys, int64_t m, int64_t nq, int64_t *__restrict__ out) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t k = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; k <= nq; k += stride) {
        int64_t lo = 0, hi = m;
        while (lo < hi) {
            const int64_t mid = (lo + hi) >> 1;
            if ((int64_t)keys[mid] < k) lo = mid + 1;
            else hi = mid;
        }
        out[k] = lo;
    }
}
// the partner list of position p: partners[poff[q] .. poff[q + 1]) with q = pkey[p] (dissolve: the row), or q = p when pkey
// is NULL (remainder: the partners depend on the group)
__device__ __forceinline__ int64_t pos_key(const uint64_t *pkey, int64_t p) { return pkey ? (int64_t)pkey[p] : p; }
// the items of the row at position p: its edge starts, then one per partner
__global__ void __launch_bounds__(256) k_dis_item_count(int64_t m, const uint64_t *__restrict__ pkey, const int64_t *__restrict__ poff,
                                                        int64_t *__restrict__ cnt) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t p = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; p < m; p += stride) {
        const int64_t q = pos_key(pkey, p);
        cnt[p] = 1 + poff[q + 1] - poff[q];
    }
}
__global__ void __launch_bounds__(256) k_dis_items(int64_t m, const uint64_t *__restrict__ prow, const uint64_t *__restrict__ pkey,
                                                   const int64_t *__restrict__ poff, const uint64_t *__restrict__ partners,
                                                   const int64_t *__restrict__ ib, int64_t *__restrict__ irow, int64_t *__restrict__ ipart) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t p = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; p < m; p += stride) {
        const int64_t r = (int64_t)prow[p], q = pos_key(pkey, p), b = ib[p];
        irow[b] = r, ipart[b] = -1;
        for (int64_t t = poff[q]; t < poff[q + 1]; ++t) irow[b + 1 + t - poff[q]] = r, ipart[b + 1 + t - poff[q]] = (int64_t)partners[t];
    }
}

// One warp per item: the edge starts of the row, or the nodes of its edges against one partner's rings (the lower row's
// stored edge first in every crossing point: side 0 when the row is the lower one)
template <bool WRITE>
__global__ void __launch_bounds__(kBoolThreads) k_dis_nodes(int64_t ni, BOperands o, const int64_t *__restrict__ irow, const int64_t *__restrict__ ipart,
                                                            int64_t *__restrict__ cnt, const int64_t *__restrict__ off, BNode *__restrict__ nodes,
                                                            int *__restrict__ too_big) {
    __shared__ int slots[kBoolThreads / 32];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const int64_t warp = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5, nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t it = warp; it < ni; it += nwarps) {
        const int64_t r = irow[it], j = ipart[it];
        int64_t a0, a1;
        row_members(o, 0, r, a0, a1);
        const int64_t xr0 = o.v[0].go[a0], xr1 = o.v[0].go[a1];
        if (lane == 0) slots[wid] = 0;
        __syncwarp();
        BNode *base = WRITE ? nodes + off[it] : nullptr;
        int64_t c;
        if (j < 0) {
            c = node_pass<WRITE, true>(o, 0, xr0, xr1, 0, 0, lane, base, &slots[wid]);
        } else {
            int64_t b0, b1;
            row_members(o, 0, j, b0, b1);
            c = node_pass<WRITE, false>(o, r < j ? 0 : 1, xr0, xr1, o.v[0].go[b0], o.v[0].go[b1], lane, base, &slots[wid]);
        }
        __syncwarp();
#pragma unroll
        for (int s = 16; s > 0; s >>= 1) c += __shfl_xor_sync(0xffffffffu, c, s);
        if (!WRITE && lane == 0) {
            cnt[it] = c;
            if (c >= (1LL << 30)) atomicExch(too_big, 1);
        }
    }
}

// position of the symbolic point just after pt towards q against row j, as k_bool_classify locates against one operand
__device__ int locate_row(const BOperands &o, int64_t j, double2 pt, double2 q, int lane) {
    int64_t m0, m1;
    row_members(o, 0, j, m0, m1);
    bool onb = false;
    for (int pass = 0; pass < 2; ++pass) {
        if (pass == 1 && !onb) break;
        const SymQ sq{pt.x, pt.y, q.x, q.y, pass};
        for (int64_t m = m0; m < m1; ++m) {
            const int64_t e = o.v[0].go[m];
            if (e >= o.v[0].go[m + 1] || o.sg[0][e] == 0) continue;
            const double4 b = o.box[0][e];
            if (!(b.x <= pt.x && pt.x <= b.z && b.y <= pt.y && pt.y <= b.w)) continue;
            int pos = sym_ring_pos(sq, part_ring(o.v[0], e), lane);
            for (int64_t h = e + 1; pos == 2 && h < o.v[0].go[m + 1]; ++h) {
                if (o.sg[0][h] == 0) continue;
                const int ph = sym_ring_pos(sq, part_ring(o.v[0], h), lane);
                if (ph != 0) pos = ph == 2 ? 0 : 1;
            }
            if (pos == 2) return pass == 0 ? S_IN : S_ON_SAME;
            onb = onb || pos == 1;
        }
    }
    return onb ? S_ON_OPP : S_OUT;
}

// One warp per position: sort the row's records, give every node met by several records one point, count the partners
// blocking the piece after each record and keep the unblocked pieces.  pinv (NULL for dissolve): the position's inverted
// partner, the subject of a remainder (§4.23), which blocks a cutter's piece unless the piece is strictly inside it; the
// subject's own pieces are blocked by a cutter they are inside or on running the same way
__global__ void __launch_bounds__(kBoolThreads) k_dis_classify(int64_t m, BOperands o, const uint64_t *__restrict__ prow, const uint64_t *__restrict__ pkey,
                                                               const uint64_t *__restrict__ pinv, const int64_t *__restrict__ ib,
                                                               const int64_t *__restrict__ off, const int64_t *__restrict__ poff,
                                                               const uint64_t *__restrict__ partners, const int64_t *__restrict__ ring_row,
                                                               BNode *__restrict__ nodes, double *__restrict__ x4) {
    const int lane = threadIdx.x & 31;
    const int64_t warp = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5, nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    const DisLess less{&o, x4 + warp * kX4};
    for (int64_t p = warp; p < m; p += nwarps) {
        const int64_t r = (int64_t)prow[p], q0 = pos_key(pkey, p), inv = pinv ? (int64_t)pinv[p] : -1, o0 = off[ib[p]], o1 = off[ib[p + 1]];
        if (o1 == o0) continue;
        BNode *nd = nodes + o0;
        const int64_t nn = o1 - o0;
        if (lane == 0) {
            heap_sort(nd, nn, less);
            // nodes met by several records: crossings tied with a vertex take its coordinates; three or more edges through one
            // point take the crossing of the two lowest rows there, lower row's stored edge first
            for (int64_t k = 0; k < nn;) {
                int64_t e = k + 1;
                if (nd[k].kind == K_CROSS) {
                    double2 p0, q0;
                    dir_edge(o, 0, nd[k].ring, nd[k].seg, p0, q0);
                    while (e < nn && nd[e].ring == nd[k].ring && nd[e].seg == nd[k].seg && less.along(nd[k], nd[e], p0, q0) == 0) ++e;
                }
                if (e - k > 1) {
                    double2 pt;
                    if (nd[e - 1].kind == K_VERTEX) {
                        pt = nd[e - 1].pt;
                    } else {
                        // the lowest row's edge, then the lowest row whose edge is not on that edge's line (rows with
                        // overlapping collinear edges meet the point along one line)
                        int64_t r1 = r, e1 = nd[k].ring, s1 = nd[k].seg, r2 = INT64_MAX, e2 = -1, s2 = -1;
                        for (int64_t i = k; i < e; ++i) {
                            const int64_t rr = ring_row[nd[i].oring];
                            if (rr < r1) r1 = rr, e1 = nd[i].oring, s1 = nd[i].oseg;
                        }
                        double2 a0, a1, b0, b1;
                        stored_edge(o, 0, e1, (int32_t)s1, a0, a1);
                        for (int64_t i = k - 1; i < e; ++i) {  // i = k - 1: the row's own edge
                            const int64_t rr = i < k ? r : ring_row[nd[i].oring], ee = i < k ? nd[k].ring : nd[i].oring;
                            const int32_t ss = i < k ? nd[k].seg : nd[i].oseg;
                            if (rr >= r2 || rr == r1) continue;
                            stored_edge(o, 0, ee, ss, b0, b1);
                            if (orient_sign(a0, a1, b0) != 0 || orient_sign(a0, a1, b1) != 0) r2 = rr, e2 = ee, s2 = ss;
                        }
                        stored_edge(o, 0, e2, (int32_t)s2, b0, b1);
                        pt = crossing_point(a0, a1, b0, b1);
                    }
                    for (int64_t i = k; i < e; ++i)
                        if (nd[i].kind == K_CROSS) nd[i].pt = pt;
                }
                k = e;
            }
        }
        __syncwarp();
        int blocked = 0;
        for (int64_t k = 0; k < nn; ++k) {
            const BNode n = nd[k];
            double2 pp, q;
            dir_edge(o, 0, n.ring, n.seg, pp, q);
            if (n.kind == K_CROSS) {
                double2 s, g;
                dir_edge(o, 0, n.oring, n.oseg, s, g);
                const int enter = orient_sign(s, g, q) > 0 ? 1 : -1;  // entering the partner (its interior left of its edge) or leaving it
                blocked += inv >= 0 && ring_row[n.oring] == inv ? -enter : enter;
            } else {
                blocked = 0;
                for (int64_t t = poff[q0]; t < poff[q0 + 1]; ++t) {
                    const int64_t j = (int64_t)partners[t];
                    const int st = locate_row(o, j, n.pt, q, lane);
                    if (j == inv) blocked += st != S_IN;
                    else if (r == inv) blocked += st == S_IN || st == S_ON_SAME;
                    else blocked += st == S_IN || st == S_ON_OPP || (st == S_ON_SAME && j < r);
                }
            }
            // a piece between two coincident vertices has no length
            const bool next_same_edge = k + 1 < nn && nd[k + 1].ring == n.ring && nd[k + 1].seg == n.seg;
            const double2 end = next_same_edge ? nd[k + 1].pt : q;
            const bool end_vertex = !next_same_edge || nd[k + 1].kind != K_CROSS;
            const bool empty = n.kind != K_CROSS && end_vertex && same_pt(n.pt, end);
            if (lane == 0) {
                nd[k].side = 0;
                nd[k].state = (int8_t)(inv >= 0 && r != inv ? S_IN : S_OUT);  // S_IN: written reversed (a cutter's piece)
                nd[k].keep = (!empty && blocked == 0) ? 1 : 0;
            }
        }
        __syncwarp();
    }
}

// per group: its first node, null flag -> too big
__global__ void __launch_bounds__(256) k_dis_groups(int64_t ng, const int64_t *__restrict__ gpos, const int64_t *__restrict__ ib,
                                                    const int64_t *__restrict__ off, int64_t *__restrict__ gnode, int *__restrict__ too_big) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t g = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; g <= ng; g += stride) {
        gnode[g] = off[ib[gpos[g]]];
        if (g < ng && off[ib[gpos[g + 1]]] - off[ib[gpos[g]]] >= (1LL << 30)) atomicExch(too_big, 1);
    }
}

// One thread per group (§4.19's assembly over the group's records); a null group has no output.  BY_STATE (the remainders):
// kept pieces in state S_IN, the cutters', are written reversed
template <bool WRITE, bool BY_STATE>
__global__ void __launch_bounds__(128) k_dis_assemble(int64_t ng, BOperands o, const int64_t *__restrict__ gnode, const uint8_t *__restrict__ gnull,
                                                      const BNode *__restrict__ nodes, int32_t *__restrict__ ws, int64_t ws_stride,
                                                      BLoop *__restrict__ loops, double4 *__restrict__ lbox, int64_t *__restrict__ cm,
                                                      int64_t *__restrict__ cr, int64_t *__restrict__ cc, const int64_t *__restrict__ mbase,
                                                      const int64_t *__restrict__ rbase, const int64_t *__restrict__ cbase,
                                                      int64_t *__restrict__ part_off, int64_t *__restrict__ ring_off, double2 *__restrict__ oxy) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t g = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; g < ng; g += stride) {
        const int64_t o0 = gnode[g], nn = gnull[g] ? 0 : gnode[g + 1] - o0;
        int64_t nm, nr, nc;
        assemble_pieces<WRITE, BY_STATE>(o, false, nodes + o0, nn, ws + o0, ws_stride, loops + o0, lbox + o0, nm, nr, nc, WRITE ? mbase[g] : 0,
                               WRITE ? rbase[g] : 0, WRITE ? cbase[g] : 0, part_off, ring_off, oxy);
        if (!WRITE) cm[g] = nm, cr[g] = nr, cc[g] = nc;
    }
}

__global__ void __launch_bounds__(256) k_dis_check_codes(int64_t n, const int64_t *__restrict__ group, int64_t ng, int *__restrict__ bad) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += stride)
        if (group[i] < -1 || group[i] >= ng) atomicExch(bad, 1);
}
__global__ void __launch_bounds__(256) k_dis_valid(int64_t ng, const uint8_t *__restrict__ gnull, uint8_t *__restrict__ rv) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t g = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; g < ng; g += stride) rv[g] = gnull[g] ? 0 : 1;
}

// The union pipeline over groups of positions (§4.21; the remainders of §4.23 run it too).  Positions [0, m) are rows
// prow[p] of the one column o reads on both sides, ordered by group (gpos[g]: the first position of group g, gpos[ng] = m)
// and by row within a group.  The partners of position p are partners[poff[q] .. poff[q + 1]), q = pkey[p] (p when pkey is
// NULL), and pinv[p] (none when pinv is NULL) is its inverted partner.  *out: the MultiPolygon column of the ng groups, row g
// null when gnull[g].
static int group_rings(gpl_ctx *ctx, const BOperands &o, int64_t ng, const int64_t *gpos, int64_t m, const uint64_t *prow,
                       const uint64_t *pkey, const uint64_t *pinv, const int64_t *poff, const uint64_t *partners,
                       const int64_t *ring_row, const uint8_t *gnull, const char *who, gpl_array **out) {
    Scratch<int> flag;
    GPL_TRY(flag.get(ctx, 2));
    GPL_CUDA(cudaMemsetAsync(flag.p, 0, 2 * sizeof(int), ctx->stream));
    Scratch<int64_t> icnt, ib, tot;
    GPL_TRY(icnt.get(ctx, (size_t)m));
    GPL_TRY(ib.get(ctx, (size_t)m + 1));
    GPL_TRY(tot.get(ctx, 3));
    if (m > 0) GPL_LAUNCH(ctx, k_dis_item_count, flat_grid(m), 256, 0, m, pkey, poff, icnt.p);
    GPL_TRY((exclusive_scan<int64_t, int64_t>(ctx, icnt.p, m, ib.p, tot.p)));
    int64_t ni = 0;
    GPL_CUDA(cudaMemcpyAsync(&ni, tot.p, sizeof(int64_t), cudaMemcpyDeviceToHost, ctx->stream));
    GPL_CUDA(cudaStreamSynchronize(ctx->stream));
    Scratch<int64_t> irow, ipart, ncnt, noff;
    GPL_TRY(irow.get(ctx, (size_t)ni));
    GPL_TRY(ipart.get(ctx, (size_t)ni));
    GPL_TRY(ncnt.get(ctx, (size_t)ni));
    GPL_TRY(noff.get(ctx, (size_t)ni + 1));
    if (m > 0) GPL_LAUNCH(ctx, k_dis_items, flat_grid(m), 256, 0, m, prow, pkey, poff, partners, ib.p, irow.p, ipart.p);
    // nodes: count, scan, write
    const int igrid = warp_grid(ni, kBoolThreads / 32);
    if (ni > 0) GPL_LAUNCH(ctx, k_dis_nodes<false>, igrid, kBoolThreads, 0, ni, o, irow.p, ipart.p, ncnt.p, nullptr, nullptr, flag.p);
    GPL_TRY((exclusive_scan<int64_t, int64_t>(ctx, ncnt.p, ni, noff.p, tot.p)));
    Scratch<int64_t> gnode;
    GPL_TRY(gnode.get(ctx, (size_t)ng + 1));
    GPL_LAUNCH(ctx, k_dis_groups, flat_grid(ng + 1), 256, 0, ng, gpos, ib.p, noff.p, gnode.p, flag.p + 1);
    int64_t h_nodes = 0;
    int h_big[2] = {0, 0};
    GPL_CUDA(cudaMemcpyAsync(&h_nodes, tot.p, sizeof(int64_t), cudaMemcpyDeviceToHost, ctx->stream));
    GPL_CUDA(cudaMemcpyAsync(h_big, flag.p, sizeof(h_big), cudaMemcpyDeviceToHost, ctx->stream));
    GPL_CUDA(cudaStreamSynchronize(ctx->stream));
    GPL_REQUIRE(!h_big[0] && !h_big[1], GPL_ERR_UNSUPPORTED, "%s: a group has 2^30 or more boundary nodes", who);
    Scratch<BNode> nodes;
    Scratch<int32_t> ws;
    Scratch<BLoop> loops;
    Scratch<double4> lbox;
    Scratch<double> x4;
    GPL_TRY(nodes.get(ctx, (size_t)h_nodes));
    GPL_TRY(ws.get(ctx, (size_t)h_nodes * 8));
    GPL_TRY(loops.get(ctx, (size_t)h_nodes));
    GPL_TRY(lbox.get(ctx, (size_t)h_nodes));
    const int cgrid = warp_grid(m, kBoolThreads / 32);
    GPL_TRY(x4.get(ctx, (size_t)cgrid * (kBoolThreads / 32) * kX4));
    if (ni > 0) GPL_LAUNCH(ctx, k_dis_nodes<true>, igrid, kBoolThreads, 0, ni, o, irow.p, ipart.p, ncnt.p, noff.p, nodes.p, flag.p);
    if (m > 0)
        GPL_LAUNCH(ctx, k_dis_classify, cgrid, kBoolThreads, 0, m, o, prow, pkey, pinv, ib.p, noff.p, poff, partners, ring_row, nodes.p, x4.p);
    // assembly: counts, scans, write
    RaggedOut res;
    Scratch<uint8_t> rv;
    GPL_TRY(res.init(ctx, ng, 3));
    GPL_TRY(rv.get(ctx, (size_t)ng));
    int64_t *cm = res.count[0].p, *cr = res.count[1].p, *cc = res.count[2].p;
    const int tgrid = (int)std::max<int64_t>(1, std::min<int64_t>(ceil_div(ng, 128), (int64_t)kSMs * 16));
    if (ng > 0)
        GPL_LAUNCH(ctx, (pinv ? k_dis_assemble<false, true> : k_dis_assemble<false, false>), tgrid, 128, 0, ng, o, gnode.p, gnull, nodes.p, ws.p, h_nodes, loops.p, lbox.p, cm, cr, cc,
                   nullptr, nullptr, nullptr, nullptr, nullptr, nullptr);
    GPL_TRY(res.scan_and_allocate());
    if (ng > 0) {
        GPL_LAUNCH(ctx, (pinv ? k_dis_assemble<true, true> : k_dis_assemble<true, false>), tgrid, 128, 0, ng, o, gnode.p, gnull, nodes.p, ws.p, h_nodes, loops.p, lbox.p, cm, cr, cc,
                   res.base[0].p, res.base[1].p, res.base[2].p, res.off[0].p, res.off[1].p, reinterpret_cast<double2 *>(res.xy.p));
        GPL_LAUNCH(ctx, k_dis_valid, flat_grid(ng), 256, 0, ng, gnull, rv.p);
    }
    return res.finish(rv.p, GPL_MULTIPOLYGON, out);
}

// ---- remainders (§4.23): subject i minus the union of the cutters C(i) it intersects, as a group of positions of the
// concatenated column (subjects [0, ns), then cutters ns + j), so the subject's row is below every cutter's and its stored
// edge comes first in every crossing point, as in gpl_boolean_op(s, c, difference)

// the positions: every present subject i and, for each candidate pair (i, j) of present rows, the cutter ns + j, grouped by
// subject for pair_list
__global__ void __launch_bounds__(256) k_rem_pos_count(int64_t ncand, const uint64_t *__restrict__ l, const uint64_t *__restrict__ r, int64_t ns,
                                                       const uint8_t *__restrict__ status, int32_t *__restrict__ cnt) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t k = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; k < ncand + ns; k += stride) {
        const int64_t i = k < ncand ? (int64_t)l[k] : k - ncand, j = k < ncand ? ns + (int64_t)r[k] : i;
        if (status[i] == 1 && status[j] == 1) atomicAdd(&cnt[i], 1);
    }
}
__global__ void __launch_bounds__(256) k_rem_pos_write(int64_t ncand, const uint64_t *__restrict__ l, const uint64_t *__restrict__ r, int64_t ns,
                                                       const uint8_t *__restrict__ status, const int64_t *__restrict__ off,
                                                       int32_t *__restrict__ cursor, int32_t *__restrict__ raw) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t k = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; k < ncand + ns; k += stride) {
        const int64_t i = k < ncand ? (int64_t)l[k] : k - ncand, j = k < ncand ? ns + (int64_t)r[k] : i;
        if (status[i] == 1 && status[j] == 1) raw[off[i] + atomicAdd(&cursor[i], 1)] = (int32_t)j;
    }
}

// The partners of position p = (subject i, row r), ascending: a subject's are its cutters (the other positions of its group);
// a cutter's are the subject and the cutters of the group it intersects (ccr[ccoff[j] .. ccoff[j + 1]): the cutter x cutter
// candidates of cutter j, membership by binary search in the group).  out NULL: count only.
__device__ int64_t rem_partners(int64_t p, int64_t ns, const uint64_t *pgrp, const uint64_t *prow, const int64_t *gpos, const uint64_t *ccr,
                                const int64_t *ccoff, uint64_t *out) {
    const int64_t i = (int64_t)pgrp[p], r = (int64_t)prow[p], g0 = gpos[i] + 1, g1 = gpos[i + 1];
    if (r == i) {
        if (out)
            for (int64_t t = g0; t < g1; ++t) out[t - g0] = prow[t];
        return g1 - g0;
    }
    int64_t c = 0;
    if (out) out[c] = (uint64_t)i;
    ++c;
    for (int64_t t = ccoff[r - ns]; t < ccoff[r - ns + 1]; ++t) {
        const int64_t k = ns + (int64_t)ccr[t];
        if (k == r) continue;
        int64_t lo = g0, hi = g1;
        while (lo < hi) {
            const int64_t mid = (lo + hi) >> 1;
            if ((int64_t)prow[mid] < k) lo = mid + 1;
            else hi = mid;
        }
        if (lo < g1 && (int64_t)prow[lo] == k) {
            if (out) out[c] = (uint64_t)k;
            ++c;
        }
    }
    return c;
}
__global__ void __launch_bounds__(256) k_rem_partner_count(int64_t m, int64_t ns, const uint64_t *__restrict__ pgrp, const uint64_t *__restrict__ prow,
                                                           const int64_t *__restrict__ gpos, const uint64_t *__restrict__ ccr,
                                                           const int64_t *__restrict__ ccoff, int64_t *__restrict__ cnt) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t p = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; p < m; p += stride) cnt[p] = rem_partners(p, ns, pgrp, prow, gpos, ccr, ccoff, nullptr);
}
__global__ void __launch_bounds__(256) k_rem_partner_write(int64_t m, int64_t ns, const uint64_t *__restrict__ pgrp, const uint64_t *__restrict__ prow,
                                                           const int64_t *__restrict__ gpos, const uint64_t *__restrict__ ccr,
                                                           const int64_t *__restrict__ ccoff, const int64_t *__restrict__ poff,
                                                           uint64_t *__restrict__ partners) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t p = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; p < m; p += stride) rem_partners(p, ns, pgrp, prow, gpos, ccr, ccoff, partners + poff[p]);
}
// output row k of the concatenation: row k of source 0, then row k - ns of source 1
__global__ void __launch_bounds__(256) k_concat_index(int64_t ns, int64_t n, int8_t *__restrict__ src, uint64_t *__restrict__ row) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t k = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; k < n; k += stride) src[k] = k < ns ? 0 : 1, row[k] = (uint64_t)(k < ns ? k : k - ns);
}

int remainder_rows(gpl_ctx *ctx, const gpl_array *subj, const gpl_array *cut, gpl_array **out) {
    const int64_t ns = subj->n_geoms, nc = cut->n_geoms, n = ns + nc;
    Pairs cand(nullptr, gpl_pairs_free), cc(nullptr, gpl_pairs_free);
    GPL_TRY(join_candidate_pairs(ctx, subj, cut, JOIN_INTERSECTS, "gpl_overlay", false, cand));
    GPL_TRY(join_candidate_pairs(ctx, cut, cut, JOIN_INTERSECTS, "gpl_overlay", false, cc));
    // the concatenated column, read on both sides
    Scratch<int8_t> csrc;
    Scratch<uint64_t> crow;
    GPL_TRY(csrc.get(ctx, (size_t)n));
    GPL_TRY(crow.get(ctx, (size_t)n));
    if (n > 0) GPL_LAUNCH(ctx, k_concat_index, flat_grid(n), 256, 0, ns, n, csrc.p, crow.p);
    const gpl_array *srcs[3] = {subj, cut, nullptr};
    gpl_array *both_raw = nullptr;
    GPL_TRY(gather_polygons(ctx, srcs, csrc.p, crow.p, n, &both_raw));
    std::unique_ptr<gpl_array, void (*)(gpl_array *)> both(both_raw, gpl_array_free);
    RingPrep pr;
    GPL_TRY(ring_prep(ctx, both.get(), pr));
    BOperands o;
    o.v[0] = o.v[1] = pr.view;
    o.mem[0] = o.mem[1] = pr.members;
    o.valid[0] = o.valid[1] = both->validity;
    o.sg[0] = o.sg[1] = pr.sigma.p;
    o.box[0] = o.box[1] = pr.box.p;
    Scratch<uint8_t> status;
    Scratch<int64_t> ring_row;
    GPL_TRY(status.get(ctx, (size_t)n));
    GPL_TRY(ring_row.get(ctx, (size_t)both->n_rings));
    if (n > 0) GPL_LAUNCH(ctx, k_dis_rows, warp_grid(n, 4), 128, 0, n, pr.view, pr.members, both->validity, nullptr, status.p, nullptr, ring_row.p);
    // positions, sorted by (subject, row): the subject first
    const int64_t ncand = cand->n;
    Scratch<int32_t> cursor;
    GPL_TRY(cursor.get(ctx, (size_t)ns));
    gpl_pairs *plist_raw = nullptr;
    GPL_TRY(pair_list(
        ctx, ns, false, &plist_raw,
        [&](int32_t *cnt) -> int {
            GPL_CUDA(cudaMemsetAsync(cnt, 0, sizeof(int32_t) * (size_t)ns, ctx->stream));
            GPL_LAUNCH(ctx, k_rem_pos_count, flat_grid(ncand + ns), 256, 0, ncand, cand->lhs, cand->rhs, ns, status.p, cnt);
            return GPL_OK;
        },
        [&](const int64_t *off, int32_t *raw, double *) -> int {
            GPL_CUDA(cudaMemsetAsync(cursor.p, 0, sizeof(int32_t) * (size_t)ns, ctx->stream));
            GPL_LAUNCH(ctx, k_rem_pos_write, flat_grid(ncand + ns), 256, 0, ncand, cand->lhs, cand->rhs, ns, status.p, off, cursor.p, raw);
            return GPL_OK;
        }));
    Pairs plist(plist_raw, gpl_pairs_free);
    cand.reset();
    const int64_t m = plist->n;
    Scratch<int64_t> gpos, ccoff, pcnt, poff, tot;
    GPL_TRY(gpos.get(ctx, (size_t)ns + 1));
    GPL_TRY(ccoff.get(ctx, (size_t)nc + 1));
    GPL_TRY(pcnt.get(ctx, (size_t)m));
    GPL_TRY(poff.get(ctx, (size_t)m + 1));
    GPL_TRY(tot.get(ctx, 1));
    GPL_LAUNCH(ctx, k_lower_bounds, flat_grid(ns + 1), 256, 0, plist->lhs, m, ns, gpos.p);
    GPL_LAUNCH(ctx, k_lower_bounds, flat_grid(nc + 1), 256, 0, cc->lhs, cc->n, nc, ccoff.p);
    if (m > 0) GPL_LAUNCH(ctx, k_rem_partner_count, flat_grid(m), 256, 0, m, ns, plist->lhs, plist->rhs, gpos.p, cc->rhs, ccoff.p, pcnt.p);
    GPL_TRY((exclusive_scan<int64_t, int64_t>(ctx, pcnt.p, m, poff.p, tot.p)));
    int64_t h_part = 0;
    GPL_CUDA(cudaMemcpyAsync(&h_part, tot.p, sizeof(int64_t), cudaMemcpyDeviceToHost, ctx->stream));
    GPL_CUDA(cudaStreamSynchronize(ctx->stream));
    Scratch<uint64_t> partners;
    GPL_TRY(partners.get(ctx, (size_t)h_part));
    if (m > 0)
        GPL_LAUNCH(ctx, k_rem_partner_write, flat_grid(m), 256, 0, m, ns, plist->lhs, plist->rhs, gpos.p, cc->rhs, ccoff.p, poff.p, partners.p);
    // the subject of each position (its group) is its inverted partner; no remainder is null (a null or non-finite subject has
    // no position)
    Scratch<uint8_t> gnull;
    GPL_TRY(gnull.get(ctx, (size_t)ns));
    GPL_CUDA(cudaMemsetAsync(gnull.p, 0, (size_t)ns, ctx->stream));
    return group_rings(ctx, o, ns, gpos.p, m, plist->rhs, nullptr, plist->lhs, poff.p, partners.p, ring_row.p, gnull.p, "overlay", out);
}

}  // namespace gpl

using namespace gpl;

extern "C" int gpl_dissolve(gpl_ctx *ctx, const gpl_array *in, const int64_t *group, int mem, int64_t n_groups, gpl_array **out) {
    GPL_REQUIRE(ctx && in && out && (group || in->n_geoms == 0), GPL_ERR_INVALID_ARG, "gpl_dissolve: NULL argument");
    GPL_TRY(check_mem(mem, "gpl_dissolve"));
    GPL_REQUIRE(n_groups >= 0, GPL_ERR_INVALID_ARG, "gpl_dissolve: n_groups must be >= 0 (found %lld)", (long long)n_groups);
    GPL_REQUIRE(is_area(in->type), GPL_ERR_INVALID_TYPE, "Expected (Multi)Polygon (found %s)", type_name(in->type));
    const int64_t n = in->n_geoms, ng = n_groups;
    GPL_REQUIRE(n < (1LL << 31) && ng < (1LL << 31), GPL_ERR_UNSUPPORTED, "gpl_dissolve: at most 2^31 rows and groups");
    if (mem == GPL_HOST)
        for (int64_t i = 0; i < n; ++i)
            GPL_REQUIRE(group[i] >= -1 && group[i] < ng, GPL_ERR_INVALID_ARG, "gpl_dissolve: group code %lld of row %lld is outside [-1, %lld)",
                        (long long)group[i], (long long)i, (long long)ng);
    GPL_CUDA(cudaSetDevice(ctx->device));
    Scratch<int64_t> dgroup;
    const int64_t *grp = group;
    Scratch<int> flag;
    GPL_TRY(flag.get(ctx, 1));
    GPL_CUDA(cudaMemsetAsync(flag.p, 0, sizeof(int), ctx->stream));
    if (mem == GPL_HOST) {
        GPL_TRY(dgroup.get(ctx, (size_t)n));
        if (n) GPL_CUDA(cudaMemcpyAsync(dgroup.p, group, sizeof(int64_t) * (size_t)n, cudaMemcpyHostToDevice, ctx->stream));
        grp = dgroup.p;
    } else if (n > 0) {
        GPL_LAUNCH(ctx, k_dis_check_codes, flat_grid(n), 256, 0, n, group, ng, flag.p);
        int h_bad = 0;
        GPL_CUDA(cudaMemcpyAsync(&h_bad, flag.p, sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
        GPL_CUDA(cudaStreamSynchronize(ctx->stream));
        GPL_REQUIRE(!h_bad, GPL_ERR_INVALID_ARG, "gpl_dissolve: a group code is outside [-1, %lld)", (long long)ng);
    }
    RingPrep pr;
    GPL_TRY(ring_prep(ctx, in, pr));
    BOperands o;
    o.v[0] = o.v[1] = pr.view;
    o.mem[0] = o.mem[1] = pr.members;
    o.valid[0] = o.valid[1] = in->validity;
    o.sg[0] = o.sg[1] = pr.sigma.p;
    o.box[0] = o.box[1] = pr.box.p;
    // rows: status, null groups, the row of every ring
    Scratch<uint8_t> status, gnull;
    Scratch<int64_t> ring_row;
    GPL_TRY(status.get(ctx, (size_t)n));
    GPL_TRY(gnull.get(ctx, (size_t)ng));
    GPL_TRY(ring_row.get(ctx, (size_t)in->n_rings));
    GPL_CUDA(cudaMemsetAsync(gnull.p, 0, (size_t)ng, ctx->stream));
    if (n > 0) GPL_LAUNCH(ctx, k_dis_rows, warp_grid(n, 4), 128, 0, n, pr.view, pr.members, in->validity, grp, status.p, gnull.p, ring_row.p);
    // partners: the intersecting pairs of present rows of one group, per row, sorted
    Pairs cand(nullptr, gpl_pairs_free);
    GPL_TRY(join_candidate_pairs(ctx, in, in, JOIN_INTERSECTS, "gpl_dissolve", false, cand));
    const int64_t nc = cand->n;
    Scratch<int32_t> cursor;
    GPL_TRY(cursor.get(ctx, (size_t)std::max(n, ng)));
    gpl_pairs *plist_raw = nullptr;
    GPL_TRY(pair_list(
        ctx, n, false, &plist_raw,
        [&](int32_t *cnt) -> int {
            GPL_CUDA(cudaMemsetAsync(cnt, 0, sizeof(int32_t) * (size_t)n, ctx->stream));
            if (nc > 0) GPL_LAUNCH(ctx, k_dis_pair_count, flat_grid(nc), 256, 0, nc, cand->lhs, cand->rhs, status.p, grp, cnt);
            return GPL_OK;
        },
        [&](const int64_t *off, int32_t *raw, double *) -> int {
            GPL_CUDA(cudaMemsetAsync(cursor.p, 0, sizeof(int32_t) * (size_t)n, ctx->stream));
            GPL_LAUNCH(ctx, k_dis_pair_write, flat_grid(nc), 256, 0, nc, cand->lhs, cand->rhs, status.p, grp, off, cursor.p, raw);
            return GPL_OK;
        }));
    Pairs plist(plist_raw, gpl_pairs_free);
    cand.reset();
    Scratch<int64_t> poff;
    GPL_TRY(poff.get(ctx, (size_t)n + 1));
    GPL_LAUNCH(ctx, k_lower_bounds, flat_grid(n + 1), 256, 0, plist->lhs, plist->n, n, poff.p);
    // positions: the present rows ordered by (group, row)
    gpl_pairs *glist_raw = nullptr;
    GPL_TRY(pair_list(
        ctx, ng, false, &glist_raw,
        [&](int32_t *cnt) -> int {
            GPL_CUDA(cudaMemsetAsync(cnt, 0, sizeof(int32_t) * (size_t)ng, ctx->stream));
            if (n > 0) GPL_LAUNCH(ctx, k_dis_group_count, flat_grid(n), 256, 0, n, status.p, grp, cnt);
            return GPL_OK;
        },
        [&](const int64_t *off, int32_t *raw, double *) -> int {
            GPL_CUDA(cudaMemsetAsync(cursor.p, 0, sizeof(int32_t) * (size_t)ng, ctx->stream));
            GPL_LAUNCH(ctx, k_dis_group_write, flat_grid(n), 256, 0, n, status.p, grp, off, cursor.p, raw);
            return GPL_OK;
        }));
    Pairs glist(glist_raw, gpl_pairs_free);
    const int64_t m = glist->n;
    Scratch<int64_t> gpos;
    GPL_TRY(gpos.get(ctx, (size_t)ng + 1));
    GPL_LAUNCH(ctx, k_lower_bounds, flat_grid(ng + 1), 256, 0, glist->lhs, m, ng, gpos.p);
    return group_rings(ctx, o, ng, gpos.p, m, glist->rhs, glist->rhs, nullptr, poff.p, plist->rhs, ring_row.p, gnull.p, "dissolve", out);
}
