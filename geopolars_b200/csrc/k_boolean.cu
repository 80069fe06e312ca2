// k_boolean.cu — intersection, union and difference geometry of two (Multi)Polygon columns, row-wise (gpl_boolean_op) and as
// a geometry overlay join (gpl_overlay_join).  geo 0.27 has them as BooleanOps::{intersection, union, difference} (recalled),
// each returning a MultiPolygon.  DESIGN.md §4.19 has the derivation.
//
// Every ring is used with its interior on the left (σ per ring from k_ring_prep, as in k_overlay.cu).  Each directed edge of
// ∂A is cut at the vertices of ∂B lying inside it and at its proper crossings with ∂B, and each edge of ∂B likewise at ∂A:
//   nodes     one record per edge start, per vertex of the other side inside the edge, per proper crossing; a vertex node is
//             keyed by its exact coordinates, a crossing by its (A edge, B edge) pair, and its point p + t (q - p) with
//             t = o_p / (o_p - o_q) is computed from the stored A and B edges, so both of its records carry the same bits;
//   order     the records of an edge are ordered along it by exact signs: two vertices by their coordinates, a vertex against a
//             crossing by the side of the crossing edge's line it lies on, two crossings by the side of one crossing edge's line
//             the other crossing edge lies on (one of the two lies wholly on one side when the edges do not cross each other);
//             the f64 t only breaks what invalid input leaves undecided;
//   classes   the piece after an edge start or a vertex is classified by sym_ring_pos of the symbolic point just after it
//             (on the other boundary: the symbolic point just left of it tells the direction), the piece after a crossing is
//             the other state of the piece before it; the keep rules of the op select the pieces;
//   linking   a kept piece ends at the output point where the next one starts (nodes are points: two crossings that round
//             to one point are one node); where several kept pieces leave a point, the one bounding the same interior sector
//             follows (the first clockwise from the reversed incoming direction, an exact angular order by quadrant and
//             orient2d of the point and input points); every ring that visits a point twice is then split into the loops
//             between its visits, loops of fewer than 3 points dropped;
//   rings     the sign of a loop's f64 shoelace makes it a shell (counter-clockwise) or a hole, a loop whose area is within
//             the sum's rounding bound is dropped; a hole goes to the smallest shell containing one of its vertices that is not
//             on that shell (orient2d on the output coordinates).
// Layout: the cut-point enumeration (O(|∂A| |∂B|) per row, the hot path) is one warp per row, groups of lanes per outer edge
// and ring-box skipping as in overlap_pass; it runs as a count pass, a scan and a write pass.  One warp per row orders and
// classifies the records; one thread per row links and assembles them, twice (counts, then the MultiPolygon's offsets and
// coordinates at the scanned positions).  Every step depends on the row alone, so a row's output is deterministic and the join
// reproduces the row-wise bytes.
#include <math.h>

#include <algorithm>
#include <memory>

#include "common.cuh"
#include "join_grid.cuh"
#include "join_host.cuh"
#include "overlay.cuh"
#include "pair_dist.cuh"
#include "scan.cuh"
#include "sym_point.cuh"

namespace gpl {

constexpr int kBoolThreads = 128;

// one node on a directed input edge: its start, a vertex of the other side inside it, or a proper crossing
struct BNode {
    double2 pt;
    double t;              // f64 parameter along the directed edge (a tie-break for invalid input only)
    int64_t ring, oring;   // the edge's ring; a crossing: the other edge's ring (else -1)
    int32_t seg, oseg;     // segment index in the ring (stored orientation)
    int8_t side, kind, state, keep;
};
enum { K_START = 0, K_VERTEX = 1, K_CROSS = 2 };
enum { S_OUT = 0, S_IN = 2, S_ON_SAME = 3, S_ON_OPP = 4 };

// one closed loop of kept pieces
struct BLoop {
    int32_t start, len, ncoord, rot, type, parent;  // type: 1 shell, -1 hole, 0 dropped
    double2 first;                                  // the lexicographically smallest vertex
};

struct BOperands {
    Side v[2];
    const int64_t *mem[2];   // member offsets of a MultiPolygon column, NULL for Polygon
    const uint8_t *valid[2];
    const int8_t *sg[2];
    const double4 *box[2];
};

__device__ __forceinline__ void row_members(const BOperands &o, int s, int64_t r, int64_t &m0, int64_t &m1) {
    m0 = o.mem[s] ? o.mem[s][r] : r, m1 = o.mem[s] ? o.mem[s][r + 1] : r + 1;
}

// the directed edge (interior on the left) of segment `seg` of ring `ring`
__device__ __forceinline__ void dir_edge(const BOperands &o, int side, int64_t ring, int32_t seg, double2 &p, double2 &q) {
    const Chain c = part_ring(o.v[side], ring);
    const double2 u = c[seg], w = c[seg + 1];
    if (o.sg[side][ring] > 0) p = u, q = w;
    else p = w, q = u;
}
__device__ __forceinline__ void stored_edge(const BOperands &o, int side, int64_t ring, int32_t seg, double2 &p, double2 &q) {
    const Chain c = part_ring(o.v[side], ring);
    p = c[seg], q = c[seg + 1];
}
__device__ __forceinline__ bool same_pt(double2 a, double2 b) { return a.x == b.x && a.y == b.y; }

// the crossing point of the stored A edge (a0, a1) and B edge (b0, b1): the same bits from either side's records
__device__ __forceinline__ double2 crossing_point(double2 a0, double2 a1, double2 b0, double2 b1) {
    const double o0 = orient2d(b0.x, b0.y, b1.x, b1.y, a0.x, a0.y), o1 = orient2d(b0.x, b0.y, b1.x, b1.y, a1.x, a1.y);
    const double t = o0 / (o0 - o1);
    return make_double2(a0.x + t * (a1.x - a0.x), a0.y + t * (a1.y - a0.y));
}

// One enumeration pass: the nodes of the directed edges of rings [xr0, xr1) of side X against the rings [yr0, yr1) of the
// other side.  Returns this lane's number of nodes; WRITE: also stores them at base + atomicAdd(slot).
template <bool WRITE>
__device__ int64_t node_pass(const BOperands &o, int X, int64_t xr0, int64_t xr1, int64_t yr0, int64_t yr1, int lane, BNode *base,
                             int *slot) {
    const int Y = 1 - X;
    const Side &xv = o.v[X], &yv = o.v[Y];
    int64_t cnt = 0;
    for (int64_t rx = xr0; rx < xr1; ++rx) {
        const int sx = o.sg[X][rx];
        if (sx == 0) continue;
        const Chain cx = part_ring(xv, rx);
        const int64_t nseg = cx.coords() - 1;
        int groups = 32;
        while (groups > 1 && groups / 2 >= nseg) groups >>= 1;
        const int G = 32 / groups, grp = lane / G, sub = lane - grp * G;
        for (int64_t b0 = 0; b0 < nseg; b0 += groups) {
            const int64_t i = b0 + grp;
            if (i >= nseg) continue;
            const double2 u = cx[i], w = cx[i + 1];
            if (same_pt(u, w)) continue;
            const double2 p = sx > 0 ? u : w, q = sx > 0 ? w : u;
            if (sub == 0) {
                ++cnt;
                if (WRITE) base[atomicAdd(slot, 1)] = BNode{p, 0.0, rx, -1, (int32_t)i, -1, (int8_t)X, K_START, 0, 0};
            }
            const double ex0 = fmin(p.x, q.x), ex1 = fmax(p.x, q.x), ey0 = fmin(p.y, q.y), ey1 = fmax(p.y, q.y);
            const double dx = q.x - p.x, dy = q.y - p.y, dd = dx * dx + dy * dy;
            for (int64_t ry = yr0; ry < yr1; ++ry) {
                if (o.sg[Y][ry] == 0) continue;
                const double4 rb = o.box[Y][ry];
                if (ex1 < rb.x || rb.z < ex0 || ey1 < rb.y || rb.w < ey0) continue;
                const Chain cy = part_ring(yv, ry);
                const int64_t ny = cy.coords() - 1;
                for (int64_t j = sub; j < ny; j += G) {
                    const double2 s = cy[j], g = cy[j + 1];
                    if (same_pt(s, g)) continue;
                    if (ex1 < fmin(s.x, g.x) || fmax(s.x, g.x) < ex0 || ey1 < fmin(s.y, g.y) || fmax(s.y, g.y) < ey0) continue;
                    const int os = orient_sign(p, q, s), og = orient_sign(p, q, g);
                    if (os == 0 && point_in_rect(s, p, q) && !same_pt(s, p) && !same_pt(s, q)) {  // s: a vertex inside (p, q)
                        ++cnt;
                        if (WRITE) {
                            const double t = ((s.x - p.x) * dx + (s.y - p.y) * dy) / dd;
                            base[atomicAdd(slot, 1)] = BNode{s, t, rx, -1, (int32_t)i, -1, (int8_t)X, K_VERTEX, 0, 0};
                        }
                    }
                    if (os * og < 0 && orient_sign(s, g, p) * orient_sign(s, g, q) < 0) {  // a proper crossing
                        ++cnt;
                        if (WRITE) {
                            const double2 pt = X == 0 ? crossing_point(u, w, s, g) : crossing_point(s, g, u, w);
                            const double op = orient2d(s.x, s.y, g.x, g.y, p.x, p.y), oq = orient2d(s.x, s.y, g.x, g.y, q.x, q.y);
                            base[atomicAdd(slot, 1)] = BNode{pt, op / (op - oq), rx, ry, (int32_t)i, (int32_t)j, (int8_t)X, K_CROSS, 0, 0};
                        }
                    }
                }
            }
        }
    }
    return cnt;
}

// the row's validity (both rows present and finite) and, when valid, its node count; the rows are ia[r] / ib[r] (or r)
__device__ __forceinline__ bool row_ok(const BOperands &o, int64_t ra, int64_t rb, int lane) {
    if (!(bit_get(o.valid[0], ra) && bit_get(o.valid[1], rb))) return false;
    int64_t a0, a1, b0, b1;
    row_members(o, 0, ra, a0, a1);
    row_members(o, 1, rb, b0, b1);
    return members_finite(o.v[0], a0, a1, lane) && members_finite(o.v[1], b0, b1, lane);
}

template <bool WRITE>
__global__ void __launch_bounds__(kBoolThreads) k_bool_nodes(int64_t n, BOperands o, const uint64_t *__restrict__ ia, const uint64_t *__restrict__ ib,
                                                             int64_t *__restrict__ cnt, uint8_t *__restrict__ row_valid,
                                                             const int64_t *__restrict__ off, BNode *__restrict__ nodes, int *__restrict__ too_big) {
    __shared__ int slots[kBoolThreads / 32];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    int64_t warp = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
    const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t r = warp; r < n; r += nwarps) {
        const int64_t ra = ia ? (int64_t)ia[r] : r, rb = ib ? (int64_t)ib[r] : r;
        const bool ok = WRITE ? row_valid[r] != 0 : row_ok(o, ra, rb, lane);
        int64_t c = 0;
        if (ok) {
            int64_t a0, a1, b0, b1;
            row_members(o, 0, ra, a0, a1);
            row_members(o, 1, rb, b0, b1);
            const int64_t ar0 = o.v[0].go[a0], ar1 = o.v[0].go[a1], br0 = o.v[1].go[b0], br1 = o.v[1].go[b1];
            if (lane == 0) slots[wid] = 0;
            __syncwarp();
            BNode *base = WRITE ? nodes + off[r] : nullptr;
            c = node_pass<WRITE>(o, 0, ar0, ar1, br0, br1, lane, base, &slots[wid]);
            c += node_pass<WRITE>(o, 1, br0, br1, ar0, ar1, lane, base, &slots[wid]);
            __syncwarp();
        }
#pragma unroll
        for (int s = 16; s > 0; s >>= 1) c += __shfl_xor_sync(0xffffffffu, c, s);
        if (!WRITE && lane == 0) {
            cnt[r] = c;
            row_valid[r] = ok ? 1 : 0;
            if (c >= (1LL << 30)) atomicExch(too_big, 1);
        }
    }
}

// ---- ordering of the nodes of one row: by edge, the start first, then along the edge by exact signs ---------------------
struct NodeLess {
    const BOperands *o;
    // -1: a before b along the directed edge (p, q); 0: undecided
    __device__ int along(const BNode &a, const BNode &b, double2 p, double2 q) const {
        if (a.kind == K_VERTEX && b.kind == K_VERTEX) {
            const int d = cmpd(q.x, p.x);
            return d ? cmpd(a.pt.x, b.pt.x) * d : cmpd(a.pt.y, b.pt.y) * cmpd(q.y, p.y);
        }
        if (a.kind == K_VERTEX || b.kind == K_VERTEX) {
            const BNode &v = a.kind == K_VERTEX ? a : b, &x = a.kind == K_VERTEX ? b : a;
            double2 s, g;
            stored_edge(*o, 1 - x.side, x.oring, x.oseg, s, g);
            const int sv = orient_sign(s, g, v.pt);
            if (sv == 0) return 0;
            const int vb = sv == orient_sign(s, g, p) ? -1 : 1;  // v before the crossing
            return a.kind == K_VERTEX ? vb : -vb;
        }
        double2 s1, g1, s2, g2;
        stored_edge(*o, 1 - a.side, a.oring, a.oseg, s1, g1);
        stored_edge(*o, 1 - b.side, b.oring, b.oseg, s2, g2);
        int c1 = orient_sign(s1, g1, s2), c2 = orient_sign(s1, g1, g2);
        if (c1 * c2 >= 0 && (c1 | c2)) return (c1 ? c1 : c2) == orient_sign(s1, g1, p) ? 1 : -1;  // b's edge on one side of a's line
        c1 = orient_sign(s2, g2, s1), c2 = orient_sign(s2, g2, g1);
        if (c1 * c2 >= 0 && (c1 | c2)) return (c1 ? c1 : c2) == orient_sign(s2, g2, p) ? -1 : 1;
        return cmpd(a.t, b.t);
    }
    __device__ bool operator()(const BNode &a, const BNode &b) const {
        if (a.side != b.side) return a.side < b.side;
        if (a.ring != b.ring) return a.ring < b.ring;
        if (a.seg != b.seg) return a.seg < b.seg;
        if ((a.kind == K_START) != (b.kind == K_START)) return a.kind == K_START;
        if (a.kind != K_START) {
            double2 p, q;
            dir_edge(*o, a.side, a.ring, a.seg, p, q);
            const int c = along(a, b, p, q);
            if (c) return c < 0;
        }
        if (a.kind != b.kind) return a.kind < b.kind;
        if (a.oring != b.oring) return a.oring < b.oring;
        if (a.oseg != b.oseg) return a.oseg < b.oseg;
        if (a.pt.x != b.pt.x) return a.pt.x < b.pt.x;
        return a.pt.y < b.pt.y;
    }
};

template <class T, class Less>
__device__ void heap_sort(T *a, int64_t n, const Less &less) {
    auto sift = [&](int64_t i, int64_t m) {
        for (;;) {
            int64_t c = 2 * i + 1;
            if (c >= m) return;
            if (c + 1 < m && less(a[c], a[c + 1])) ++c;
            if (!less(a[i], a[c])) return;
            const T t = a[i];
            a[i] = a[c], a[c] = t;
            i = c;
        }
    };
    for (int64_t i = n / 2 - 1; i >= 0; --i) sift(i, n);
    for (int64_t m = n - 1; m > 0; --m) {
        const T t = a[0];
        a[0] = a[m], a[m] = t;
        sift(0, m);
    }
}

__device__ __forceinline__ bool keep_piece(int op, int side, int st) {
    if (side == 0) {
        if (op == GPL_BOOLEAN_INTERSECTION) return st == S_IN || st == S_ON_SAME;
        if (op == GPL_BOOLEAN_UNION) return st == S_OUT || st == S_ON_SAME;
        return st == S_OUT || st == S_ON_OPP;
    }
    return op == GPL_BOOLEAN_UNION ? st == S_OUT : st == S_IN;
}

// One warp per row: sort the row's nodes, classify the piece after each one and mark the kept pieces.
__global__ void __launch_bounds__(kBoolThreads) k_bool_classify(int64_t n, BOperands o, const uint64_t *__restrict__ ia, const uint64_t *__restrict__ ib,
                                                                int op, const int64_t *__restrict__ off, BNode *__restrict__ nodes) {
    const int lane = threadIdx.x & 31;
    int64_t warp = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
    const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    const NodeLess less{&o};
    for (int64_t r = warp; r < n; r += nwarps) {
        const int64_t o0 = off[r], o1 = off[r + 1];
        if (o1 == o0) continue;
        if (lane == 0) heap_sort(nodes + o0, o1 - o0, less);
        __syncwarp();
        const int64_t ra = ia ? (int64_t)ia[r] : r, rb = ib ? (int64_t)ib[r] : r;
        int64_t m0[2], m1[2];
        row_members(o, 0, ra, m0[0], m1[0]);
        row_members(o, 1, rb, m0[1], m1[1]);
        int prev = S_OUT;
        for (int64_t k = o0; k < o1; ++k) {
            const BNode nd = nodes[k];
            const int Y = 1 - nd.side;
            double2 p, q;
            dir_edge(o, nd.side, nd.ring, nd.seg, p, q);
            int st;
            if (nd.kind == K_CROSS) {
                st = prev == S_IN ? S_OUT : S_IN;
            } else {
                // rings that contribute nothing (sigma 0) are skipped, as are members whose exterior box does not contain
                // the point
                st = S_OUT;
                bool onb = false;
                for (int pass = 0; pass < 2 && st == S_OUT; ++pass) {
                    if (pass == 1 && !onb) break;
                    const SymQ sq{nd.pt.x, nd.pt.y, q.x, q.y, pass};
                    for (int64_t m = m0[Y]; m < m1[Y]; ++m) {
                        const int64_t e = o.v[Y].go[m];
                        if (e >= o.v[Y].go[m + 1] || o.sg[Y][e] == 0) continue;
                        const double4 b = o.box[Y][e];
                        if (!(b.x <= nd.pt.x && nd.pt.x <= b.z && b.y <= nd.pt.y && nd.pt.y <= b.w)) continue;
                        // the member's region: its exterior less its holes, holes with sigma 0 contributing nothing
                        int pos = sym_ring_pos(sq, part_ring(o.v[Y], e), lane);
                        for (int64_t h = e + 1; pos == 2 && h < o.v[Y].go[m + 1]; ++h) {
                            if (o.sg[Y][h] == 0) continue;
                            const int ph = sym_ring_pos(sq, part_ring(o.v[Y], h), lane);
                            if (ph != 0) pos = ph == 2 ? 0 : 1;
                        }
                        if (pos == 2) {
                            st = pass == 0 ? S_IN : S_ON_SAME;
                            break;
                        }
                        onb = onb || pos == 1;
                    }
                    if (pass == 1 && st == S_OUT) st = S_ON_OPP;
                }
            }
            prev = st;
            // a piece between two coincident vertices (a vertex of the other side met twice) has no length
            const bool next_same_edge = k + 1 < o1 && nodes[k + 1].side == nd.side && nodes[k + 1].ring == nd.ring && nodes[k + 1].seg == nd.seg;
            const double2 end = next_same_edge ? nodes[k + 1].pt : q;
            const bool end_vertex = !next_same_edge || nodes[k + 1].kind != K_CROSS;
            const bool empty = nd.kind != K_CROSS && end_vertex && same_pt(nd.pt, end);
            if (lane == 0) {
                nodes[k].state = (int8_t)st;
                nodes[k].keep = (!empty && keep_piece(op, nd.side, st)) ? 1 : 0;
            }
        }
        __syncwarp();
    }
}

// ---- linking and ring assembly: one thread per row ----------------------------------------------------------------------
// the kept pieces of one row, in output direction (B pieces of a difference reversed)
struct Pieces {
    const BOperands *o;
    const BNode *nd;  // the row's nodes
    int64_t nn;
    const int32_t *kp;  // kept piece -> node index
    bool rev_b;
    __device__ bool rev(int j) const { return rev_b && nd[kp[j]].side == 1; }
    __device__ bool next_on_edge(int64_t k) const {
        return k + 1 < nn && nd[k + 1].side == nd[k].side && nd[k + 1].ring == nd[k].ring && nd[k + 1].seg == nd[k].seg;
    }
    // start (a = 0) or end (a = 1) of the piece along its directed input edge
    __device__ double2 raw_pt(int j, int a) const {
        const int64_t k = kp[j];
        if (a == 0) return nd[k].pt;
        if (next_on_edge(k)) return nd[k + 1].pt;
        double2 p, q;
        dir_edge(*o, nd[k].side, nd[k].ring, nd[k].seg, p, q);
        return q;
    }
    __device__ double2 from_pt(int j) const { return raw_pt(j, rev(j) ? 1 : 0); }
    __device__ double2 to_pt(int j) const { return raw_pt(j, rev(j) ? 0 : 1); }
    // the input edge of the piece, in output direction
    __device__ void edge(int j, double2 &P, double2 &Q) const {
        const BNode &n = nd[kp[j]];
        dir_edge(*o, n.side, n.ring, n.seg, P, Q);
        if (rev(j)) {
            const double2 t = P;
            P = Q, Q = t;
        }
    }
};

__device__ __forceinline__ int pt_cmp(double2 a, double2 b) { return a.x != b.x ? (a.x < b.x ? -1 : 1) : (a.y != b.y ? (a.y < b.y ? -1 : 1) : 0); }

struct FromPtLess {  // pieces by the output coordinates of their start
    const Pieces *pc;
    __device__ bool operator()(int32_t a, int32_t b) const {
        const int c = pt_cmp(pc->from_pt(a), pc->from_pt(b));
        return c ? c < 0 : a < b;
    }
};

// 0 outside / 1 on the boundary / 2 inside of the loop through the from-points of its pieces
__device__ int point_in_loop(const Pieces &pc, const int32_t *lp, const BLoop &L, double2 v) {
    int wn = 0;
    for (int i = 0; i < L.len; ++i) {
        const double2 s = pc.from_pt(lp[L.start + i]), e = pc.from_pt(lp[L.start + (i + 1 == L.len ? 0 : i + 1)]);
        if (same_pt(s, e)) continue;
        const int o = orient_sign(s, e, v);
        if (o == 0 && point_in_rect(v, s, e)) return 1;
        if (s.y <= v.y) {
            if (e.y > v.y && o > 0) ++wn;
        } else if (e.y <= v.y && o < 0) {
            --wn;
        }
    }
    return wn ? 2 : 0;
}

__device__ double loop_area2(const Pieces &pc, const int32_t *lp, const BLoop &L) {
    double a = 0.0;
    const double2 o = pc.from_pt(lp[L.start]);
    for (int i = 1; i + 1 < L.len; ++i) {
        const double2 s = pc.from_pt(lp[L.start + i]), e = pc.from_pt(lp[L.start + i + 1]);
        a += (s.x - o.x) * (e.y - o.y) - (e.x - o.x) * (s.y - o.y);
    }
    return a;
}

struct LoopLess {  // members by their shell's first vertex, holes after their shell by their first vertex
    const BLoop *L;
    __device__ bool operator()(int32_t a, int32_t b) const {
        const int pa = L[a].type > 0 ? a : L[a].parent, pb = L[b].type > 0 ? b : L[b].parent;
        int c = pt_cmp(L[pa].first, L[pb].first);
        if (c) return c < 0;
        if (pa != pb) return pa < pb;
        if ((L[a].type > 0) != (L[b].type > 0)) return L[a].type > 0;
        c = pt_cmp(L[a].first, L[b].first);
        return c ? c < 0 : a < b;
    }
};

// One thread per row.  Scratch (8 int32 per node, one BLoop per node) is indexed by the row's node offset.  Counting pass:
// members, rings and coordinates of the row; WRITE: the MultiPolygon's part / ring offsets and coordinates at the row's bases.
template <bool WRITE>
__global__ void __launch_bounds__(128) k_bool_assemble(int64_t n, BOperands o, int op, const int64_t *__restrict__ off, const BNode *__restrict__ nodes,
                                                       int32_t *__restrict__ ws, int64_t ws_stride, BLoop *__restrict__ loops,
                                                       int64_t *__restrict__ cm, int64_t *__restrict__ cr, int64_t *__restrict__ cc,
                                                       const int64_t *__restrict__ mbase, const int64_t *__restrict__ rbase,
                                                       const int64_t *__restrict__ cbase, int64_t *__restrict__ part_off,
                                                       int64_t *__restrict__ ring_off, double2 *__restrict__ oxy) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; r < n; r += stride) {
        const int64_t o0 = off[r], nn = off[r + 1] - o0;
        int32_t *kp = ws + o0, *ord = kp + ws_stride, *rank = ord + ws_stride, *gs = rank + ws_stride, *nxt = gs + ws_stride,
                *npos = nxt + ws_stride, *stk = npos + ws_stride, *lp = stk + ws_stride;
        BLoop *L = loops + o0;
        const BNode *nd = nodes + o0;
        int J = 0;
        for (int64_t k = 0; k < nn; ++k)
            if (nd[k].keep) kp[J++] = (int32_t)k;
        const Pieces pc{&o, nd, nn, kp, op == GPL_BOOLEAN_DIFFERENCE};
        // a piece whose two ends round to one point (between two crossings within half an ulp of each other) has no length
        int Jp = 0;
        for (int j = 0; j < J; ++j)
            if (!same_pt(pc.raw_pt(j, 0), pc.raw_pt(j, 1))) kp[Jp++] = kp[j];
        J = Jp;
        // nodes are output coordinates: the kept pieces sorted by the point they start at; gs: the first position of each
        // point.  Distinct input nodes are distinct points unless rounding puts two crossings (or a crossing and a vertex) on
        // one point; linking at that point by the angular rule below then joins the rings that meet there as the rounded
        // coordinates require, where linking by input node would leave a ring through the point twice or rings touching in
        // a cycle of such points
        for (int j = 0; j < J; ++j) ord[j] = j;
        heap_sort(ord, (int64_t)J, FromPtLess{&pc});
        for (int i = 0; i < J; ++i) {
            rank[ord[i]] = i;
            gs[i] = (i > 0 && same_pt(pc.from_pt(ord[i]), pc.from_pt(ord[i - 1]))) ? gs[i - 1] : i;
        }
        // successor of every kept piece
        for (int j = 0; j < J; ++j) {
            const double2 V = pc.to_pt(j);
            int lo = 0, hi = J;
            while (lo < hi) {
                const int mid = (lo + hi) >> 1;
                if (pt_cmp(pc.from_pt(ord[mid]), V) < 0) lo = mid + 1;
                else hi = mid;
            }
            int end = lo;
            while (end < J && same_pt(pc.from_pt(ord[end]), V)) ++end;
            if (end == lo) {
                nxt[j] = -1;  // a dangling piece (invalid input)
            } else if (end == lo + 1) {
                nxt[j] = ord[lo];
            } else {  // several pieces leave this point: the first clockwise from the reversed incoming direction; a piece
                      // straight back along it comes last (it bounds the sector on the far side of a notch that rounding
                      // folded to zero width; kept pieces of valid operands never run back along each other in exact terms)
                double2 Pu, Qu;
                pc.edge(j, Pu, Qu);
                int best = -1, bh = -1;
                double2 bq = V;
                for (int i = lo; i < end; ++i) {
                    double2 Pw, Qw;
                    pc.edge(ord[i], Pw, Qw);
                    const int c = orient_sign(V, Pu, Qw);
                    int h;
                    if (c > 0) h = 0;
                    else if (c < 0) h = 2;
                    else h = (cmpd(Qw.x, V.x) == cmpd(Pu.x, V.x) && cmpd(Qw.y, V.y) == cmpd(Pu.y, V.y)) ? -1 : 1;
                    if (best < 0 || h > bh || (h == bh && (h == 0 || h == 2) && orient_sign(V, bq, Qw) > 0)) best = ord[i], bh = h, bq = Qw;
                }
                nxt[j] = best;
            }
        }
        // trace the rings and split each at its repeated points: stk holds the open path, npos[point] its position there
        // (a visited piece has rank -1 - rank).  A spike ... X Y X ... closes the loop (X, Y), dropped below with fewer than
        // 3 coordinates
        for (int i = 0; i < J; ++i) npos[i] = -1;
        int nl = 0, nlp = 0;
        for (int j0 = 0; j0 < J; ++j0) {
            if (rank[j0] < 0) continue;  // visited
            int sp = 0, cur = j0;
            while (cur >= 0 && rank[cur] >= 0) {
                const int node = gs[rank[cur]];
                rank[cur] = -1 - rank[cur];
                if (npos[node] >= 0) {  // a loop closes here: stk[npos[node] .. sp)
                    const int i0 = npos[node];
                    L[nl].start = nlp, L[nl].len = sp - i0;
                    for (int i = i0; i < sp; ++i) {
                        lp[nlp++] = stk[i];
                        npos[gs[-1 - rank[stk[i]]]] = -1;
                    }
                    ++nl;
                    sp = i0;
                }
                npos[node] = sp;
                stk[sp++] = cur;
                cur = nxt[cur];
            }
            if (cur == j0 && sp > 0) {
                L[nl].start = nlp, L[nl].len = sp;
                for (int i = 0; i < sp; ++i) lp[nlp++] = stk[i];
                ++nl;
            }
            for (int i = 0; i < sp; ++i) npos[gs[-1 - rank[stk[i]]]] = -1;
        }
        // shells and holes: the sign of each loop's shoelace (f64, relative to its first coordinate), a loop of fewer than 3
        // points or whose area is within the rounding bound of that sum dropped; the first (smallest) vertex
        for (int l = 0; l < nl; ++l) {
            BLoop &lo = L[l];
            int rot = 0;
            const double2 o0 = pc.from_pt(lp[lo.start]);
            double2 first = o0;
            double a2 = 0.0, mag = 0.0;
            for (int i = 1; i < lo.len; ++i) {
                const double2 v = pc.from_pt(lp[lo.start + i]);
                if (pt_cmp(v, first) < 0) rot = i, first = v;
                if (i + 1 < lo.len) {
                    const double2 e = pc.from_pt(lp[lo.start + i + 1]);
                    const double t1 = (v.x - o0.x) * (e.y - o0.y), t2 = (e.x - o0.x) * (v.y - o0.y);
                    a2 += t1 - t2;
                    mag += fabs(t1) + fabs(t2);
                }
            }
            lo.ncoord = lo.len, lo.rot = rot, lo.first = first, lo.parent = -1;
            lo.type = lo.len < 3 || fabs(a2) <= (double)(lo.len + 4) * 0x1p-52 * mag ? 0 : a2 > 0.0 ? 1 : -1;
        }
        // every hole to the smallest shell containing it
        for (int h = 0; h < nl; ++h) {
            if (L[h].type >= 0) continue;
            int best = -1;
            double barea = 0.0;
            for (int s = 0; s < nl; ++s) {
                if (L[s].type <= 0) continue;
                // the hole's smallest vertex first: for intersection and difference it is an input vertex
                int pos = point_in_loop(pc, lp, L[s], L[h].first);
                for (int i = 0; i < L[h].len && pos == 1; ++i) pos = point_in_loop(pc, lp, L[s], pc.from_pt(lp[L[h].start + i]));
                if (pos != 2) continue;
                const double a = loop_area2(pc, lp, L[s]);
                if (best < 0 || a < barea) best = s, barea = a;
            }
            if (best < 0) L[h].type = 0;
            else L[h].parent = best;
        }
        // output order
        int nout = 0, nm = 0;
        int64_t ncoords = 0;
        for (int l = 0; l < nl; ++l)
            if (L[l].type != 0) {
                stk[nout++] = l;
                nm += L[l].type > 0;
                ncoords += L[l].ncoord + 1;
            }
        if (!WRITE) {
            cm[r] = nm, cr[r] = nout, cc[r] = ncoords;
            continue;
        }
        heap_sort(stk, (int64_t)nout, LoopLess{L});
        int64_t mb = mbase[r], rb = rbase[r], cb = cbase[r];
        for (int k = 0; k < nout; ++k) {
            const BLoop &lo = L[stk[k]];
            if (lo.type > 0) part_off[mb++] = rb;
            ring_off[rb++] = cb;
            for (int i = 0; i < lo.len; ++i) {
                const int idx = lo.rot + i < lo.len ? lo.rot + i : lo.rot + i - lo.len;
                const double2 v = pc.from_pt(lp[lo.start + idx]), pv = pc.from_pt(lp[lo.start + (idx == 0 ? lo.len - 1 : idx - 1)]);
                if (i == 0 || !same_pt(v, pv)) oxy[cb++] = v;
            }
            oxy[cb++] = lo.first;
        }
    }
}

// the MultiPolygon of `op` for n row pairs (a[ia[r]], b[ib[r]]), or (a[r], b[r]) when ia / ib are NULL; members[r] (optional,
// device) receives the member count of each row
static int boolean_rows(gpl_ctx *ctx, const BOperands &ops, int64_t n, const uint64_t *ia, const uint64_t *ib, int op, gpl_array **out,
                        Scratch<int64_t> *members) {
    Scratch<int64_t> cnt, off, cm_own, cr, cc, rbase, cbase, tot;
    Scratch<int64_t> &cm = members ? *members : cm_own;
    Scratch<uint8_t> rv, bm;
    Scratch<int> too_big;
    Scratch<int64_t> geom_off, part_off, ring_off;
    Scratch<double> oxy;
    GPL_TRY(cnt.get(ctx, (size_t)n));
    GPL_TRY(off.get(ctx, (size_t)n + 1));
    GPL_TRY(rv.get(ctx, (size_t)n));
    GPL_TRY(too_big.get(ctx, 1));
    GPL_TRY(tot.get(ctx, 3));
    GPL_TRY(geom_off.get(ctx, (size_t)n + 1));
    GPL_CUDA(cudaMemsetAsync(too_big.p, 0, sizeof(int), ctx->stream));
    const int grid = warp_grid(n, kBoolThreads / 32);
    if (n > 0)
        GPL_LAUNCH(ctx, k_bool_nodes<false>, grid, kBoolThreads, 0, n, ops, ia, ib, cnt.p, rv.p, nullptr, nullptr, too_big.p);
    GPL_TRY((exclusive_scan<int64_t, int64_t>(ctx, cnt.p, n, off.p, tot.p)));
    int64_t h_nodes = 0;
    int h_big = 0;
    GPL_CUDA(cudaMemcpyAsync(&h_nodes, tot.p, sizeof(int64_t), cudaMemcpyDeviceToHost, ctx->stream));
    GPL_CUDA(cudaMemcpyAsync(&h_big, too_big.p, sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
    GPL_CUDA(cudaStreamSynchronize(ctx->stream));
    GPL_REQUIRE(!h_big, GPL_ERR_UNSUPPORTED, "boolean_op: a row has 2^30 or more boundary nodes");
    Scratch<BNode> nodes;
    Scratch<int32_t> ws;
    Scratch<BLoop> loops;
    GPL_TRY(nodes.get(ctx, (size_t)h_nodes));
    GPL_TRY(ws.get(ctx, (size_t)h_nodes * 8));
    GPL_TRY(loops.get(ctx, (size_t)h_nodes));
    GPL_TRY(cm.get(ctx, (size_t)n));
    GPL_TRY(cr.get(ctx, (size_t)n));
    GPL_TRY(cc.get(ctx, (size_t)n));
    GPL_TRY(rbase.get(ctx, (size_t)n + 1));
    GPL_TRY(cbase.get(ctx, (size_t)n + 1));
    const int tgrid = (int)std::max<int64_t>(1, std::min<int64_t>(ceil_div(n, 128), (int64_t)kSMs * 16));
    if (n > 0) {
        GPL_LAUNCH(ctx, k_bool_nodes<true>, grid, kBoolThreads, 0, n, ops, ia, ib, cnt.p, rv.p, off.p, nodes.p, too_big.p);
        GPL_LAUNCH(ctx, k_bool_classify, grid, kBoolThreads, 0, n, ops, ia, ib, op, off.p, nodes.p);
        GPL_LAUNCH(ctx, k_bool_assemble<false>, tgrid, 128, 0, n, ops, op, off.p, nodes.p, ws.p, h_nodes, loops.p, cm.p, cr.p, cc.p,
                   nullptr, nullptr, nullptr, nullptr, nullptr, nullptr);
    }
    GPL_TRY((exclusive_scan<int64_t, int64_t>(ctx, cm.p, n, geom_off.p, tot.p)));
    GPL_TRY((exclusive_scan<int64_t, int64_t>(ctx, cr.p, n, rbase.p, tot.p + 1)));
    GPL_TRY((exclusive_scan<int64_t, int64_t>(ctx, cc.p, n, cbase.p, tot.p + 2)));
    int64_t h_tot[3] = {0, 0, 0};
    GPL_CUDA(cudaMemcpyAsync(h_tot, tot.p, sizeof(h_tot), cudaMemcpyDeviceToHost, ctx->stream));
    GPL_CUDA(cudaStreamSynchronize(ctx->stream));
    GPL_TRY(part_off.get(ctx, (size_t)h_tot[0] + 1));
    GPL_TRY(ring_off.get(ctx, (size_t)h_tot[1] + 1));
    GPL_TRY(oxy.get(ctx, (size_t)h_tot[2] * 2));
    if (n > 0)
        GPL_LAUNCH(ctx, k_bool_assemble<true>, tgrid, 128, 0, n, ops, op, off.p, nodes.p, ws.p, h_nodes, loops.p, cm.p, cr.p, cc.p,
                   geom_off.p, rbase.p, cbase.p, part_off.p, ring_off.p, reinterpret_cast<double2 *>(oxy.p));
    GPL_CUDA(cudaMemcpyAsync(part_off.p + h_tot[0], rbase.p + n, sizeof(int64_t), cudaMemcpyDeviceToDevice, ctx->stream));
    GPL_CUDA(cudaMemcpyAsync(ring_off.p + h_tot[1], cbase.p + n, sizeof(int64_t), cudaMemcpyDeviceToDevice, ctx->stream));
    GPL_TRY(bm.get(ctx, (size_t)(n + 7) / 8));
    if (n > 0) GPL_TRY(pack_bits(ctx, rv.p, bm.p, n));
    GPL_CUDA(cudaStreamSynchronize(ctx->stream));  // the scratch above returns to the cache when this scope ends
    gpl_array *res = array_new(ctx, GPL_MULTIPOLYGON);
    res->n_geoms = n, res->n_parts = h_tot[0], res->n_rings = h_tot[1], res->n_coords = h_tot[2];
    res->geom_off = geom_off.take(), res->own_geom = true;
    res->part_off = part_off.take(), res->own_part = true;
    res->ring_off = ring_off.take(), res->own_ring = true;
    res->xy = oxy.take(), res->own_xy = true;
    res->validity = bm.take(), res->own_valid = true;
    *out = res;
    return GPL_OK;
}

static BOperands operands(const gpl_array *a, const RingPrep &pa, const gpl_array *b, const RingPrep &pb) {
    BOperands o;
    o.v[0] = pa.view, o.v[1] = pb.view;
    o.mem[0] = pa.members, o.mem[1] = pb.members;
    o.valid[0] = a->validity, o.valid[1] = b->validity;
    o.sg[0] = pa.sigma.p, o.sg[1] = pb.sigma.p;
    o.box[0] = pa.box.p, o.box[1] = pb.box.p;
    return o;
}

// the candidate pairs grouped by left row for pair_list (join_host.cuh), which sorts each row's right rows
__global__ void __launch_bounds__(256) k_cand_count(int64_t n, const uint64_t *__restrict__ l, int32_t *__restrict__ cnt) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += stride) atomicAdd(&cnt[l[i]], 1);
}
__global__ void __launch_bounds__(256) k_cand_write(int64_t n, const uint64_t *__restrict__ l, const uint64_t *__restrict__ r,
                                                    const int64_t *__restrict__ off, int32_t *__restrict__ cursor, int32_t *__restrict__ raw) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += stride)
        raw[off[l[i]] + atomicAdd(&cursor[l[i]], 1)] = (int32_t)r[i];
}

// keep[k] = 1 when row k of the join's output has a member
__global__ void __launch_bounds__(256) k_nonempty(int64_t n, const int64_t *__restrict__ members, uint8_t *__restrict__ keep) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += stride) keep[i] = members[i] > 0;
}
// the kept pairs and the geometry offsets of their rows (the parts, rings and coordinates of the empty rows are empty)
__global__ void __launch_bounds__(256) k_compact_pairs(int64_t n, const uint8_t *__restrict__ keep, const int64_t *__restrict__ pos,
                                                       const uint64_t *__restrict__ l, const uint64_t *__restrict__ r,
                                                       const int64_t *__restrict__ goff, uint64_t *__restrict__ ol, uint64_t *__restrict__ orr,
                                                       int64_t *__restrict__ ogoff) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i <= n; i += stride) {
        if (i == n) {
            ogoff[pos[n]] = goff[n];
        } else if (keep[i]) {
            ol[pos[i]] = l[i], orr[pos[i]] = r[i], ogoff[pos[i]] = goff[i];
        }
    }
}

}  // namespace gpl

using namespace gpl;

extern "C" int gpl_boolean_op(gpl_ctx *ctx, const gpl_array *a, const gpl_array *b, int op, gpl_array **out) {
    GPL_REQUIRE(ctx && a && b && out, GPL_ERR_INVALID_ARG, "gpl_boolean_op: NULL argument");
    GPL_REQUIRE(op == GPL_BOOLEAN_INTERSECTION || op == GPL_BOOLEAN_UNION || op == GPL_BOOLEAN_DIFFERENCE, GPL_ERR_INVALID_ARG,
                "gpl_boolean_op: unknown op %d", op);
    GPL_REQUIRE(is_area(a->type) && is_area(b->type), GPL_ERR_INVALID_TYPE, "Expected (Multi)Polygon x (Multi)Polygon (found %s x %s)",
                type_name(a->type), type_name(b->type));
    GPL_REQUIRE(a->n_geoms == b->n_geoms, GPL_ERR_LENGTH_MISMATCH, "boolean_op: lengths differ (%lld vs %lld)", (long long)a->n_geoms,
                (long long)b->n_geoms);
    GPL_CUDA(cudaSetDevice(ctx->device));
    RingPrep pa, pb;
    GPL_TRY(ring_prep(ctx, a, pa));
    GPL_TRY(ring_prep(ctx, b, pb));
    return boolean_rows(ctx, operands(a, pa, b, pb), a->n_geoms, nullptr, nullptr, op, out, nullptr);
}

extern "C" int gpl_overlay_join(gpl_ctx *ctx, const gpl_array *lhs, const gpl_array *rhs, gpl_pairs **pairs, gpl_array **out) {
    GPL_REQUIRE(ctx && lhs && rhs && pairs && out, GPL_ERR_INVALID_ARG, "gpl_overlay_join: NULL argument");
    GPL_REQUIRE(is_area(lhs->type) && is_area(rhs->type), GPL_ERR_INVALID_TYPE, "Expected (Multi)Polygon x (Multi)Polygon (found %s x %s)",
                type_name(lhs->type), type_name(rhs->type));
    GPL_CUDA(cudaSetDevice(ctx->device));
    const int64_t nl = lhs->n_geoms, nr = rhs->n_geoms;
    GPL_REQUIRE(nl < (1LL << 31) && nr < (1LL << 31), GPL_ERR_UNSUPPORTED, "gpl_overlay_join: at most 2^31 rows per side");
    std::unique_ptr<gpl_pairs, void (*)(gpl_pairs *)> cand(new gpl_pairs(), gpl_pairs_free);
    cand->ctx = ctx;
    if (nl > 0 && nr > 0) GPL_TRY(join_candidate_pairs(ctx, lhs, rhs, JOIN_INTERSECTS, "gpl_overlay_join", cand.get()));
    // the candidates in (lhs, rhs) order (their order from the candidate stage is unspecified)
    gpl_pairs *sorted_raw = nullptr;
    const int64_t nc = cand->n;
    const int cg = (int)std::max<int64_t>(1, std::min<int64_t>(ceil_div(nc, 256), (int64_t)kSMs * 16));
    Scratch<int32_t> cursor;
    GPL_TRY(cursor.get(ctx, (size_t)nl));
    GPL_TRY(pair_list(
        ctx, nl, false, &sorted_raw,
        [&](int32_t *cnt) -> int {
            GPL_CUDA(cudaMemsetAsync(cnt, 0, sizeof(int32_t) * (size_t)nl, ctx->stream));
            if (nc > 0) GPL_LAUNCH(ctx, k_cand_count, cg, 256, 0, nc, cand->lhs, cnt);
            return GPL_OK;
        },
        [&](const int64_t *off, int32_t *raw, double *) -> int {
            GPL_CUDA(cudaMemsetAsync(cursor.p, 0, sizeof(int32_t) * (size_t)nl, ctx->stream));
            GPL_LAUNCH(ctx, k_cand_write, cg, 256, 0, nc, cand->lhs, cand->rhs, off, cursor.p, raw);
            return GPL_OK;
        }));
    std::unique_ptr<gpl_pairs, void (*)(gpl_pairs *)> sorted(sorted_raw, gpl_pairs_free);
    const int64_t n = sorted->n;
    const uint64_t *sl = sorted->lhs, *sr = sorted->rhs;
    cand.reset();
    RingPrep pl, pr;
    GPL_TRY(ring_prep(ctx, lhs, pl));
    GPL_TRY(ring_prep(ctx, rhs, pr));
    gpl_array *all = nullptr;
    Scratch<int64_t> members;
    GPL_TRY(boolean_rows(ctx, operands(lhs, pl, rhs, pr), n, sl, sr, GPL_BOOLEAN_INTERSECTION, &all, &members));
    std::unique_ptr<gpl_array, void (*)(gpl_array *)> geo(all, gpl_array_free);
    // drop the pairs whose intersection has no member (touching pairs)
    Scratch<uint8_t> keep;
    Scratch<int64_t> pos, goff;
    GPL_TRY(keep.get(ctx, (size_t)n));
    GPL_TRY(pos.get(ctx, (size_t)n + 1));
    const int g = (int)std::max<int64_t>(1, std::min<int64_t>(ceil_div(n + 1, 256), (int64_t)kSMs * 16));
    if (n > 0) GPL_LAUNCH(ctx, k_nonempty, g, 256, 0, n, members.p, keep.p);
    GPL_TRY((exclusive_scan<uint8_t, int64_t>(ctx, keep.p, n, pos.p, nullptr)));
    int64_t m = 0;
    GPL_CUDA(cudaMemcpyAsync(&m, pos.p + n, sizeof(int64_t), cudaMemcpyDeviceToHost, ctx->stream));
    GPL_CUDA(cudaStreamSynchronize(ctx->stream));
    std::unique_ptr<gpl_pairs, void (*)(gpl_pairs *)> res(new gpl_pairs(), gpl_pairs_free);
    res->ctx = ctx;
    res->n = m;
    GPL_TRY(goff.get(ctx, (size_t)m + 1));
    if (m > 0) {
        void *pl_ = nullptr, *pr_ = nullptr;
        GPL_TRY(ctx->alloc(sizeof(uint64_t) * (size_t)m, &pl_));
        res->lhs = (uint64_t *)pl_;
        GPL_TRY(ctx->alloc(sizeof(uint64_t) * (size_t)m, &pr_));
        res->rhs = (uint64_t *)pr_;
    }
    GPL_LAUNCH(ctx, k_compact_pairs, g, 256, 0, n, keep.p, pos.p, sl, sr, all->geom_off, res->lhs, res->rhs, goff.p);
    // every output row is valid: a null or non-finite pair has no member and is dropped
    Scratch<uint8_t> bm;
    GPL_TRY(bm.get(ctx, (size_t)(m + 7) / 8));
    GPL_CUDA(cudaMemsetAsync(bm.p, 0xff, (size_t)(m + 7) / 8, ctx->stream));
    GPL_CUDA(cudaStreamSynchronize(ctx->stream));
    gpl_array *o = array_new(ctx, GPL_MULTIPOLYGON);
    o->n_geoms = m, o->n_parts = all->n_parts, o->n_rings = all->n_rings, o->n_coords = all->n_coords;
    o->geom_off = goff.take(), o->own_geom = true;
    o->part_off = all->part_off, o->ring_off = all->ring_off, o->xy = all->xy;  // shared with the uncompacted result
    o->validity = bm.take(), o->own_valid = true;
    o->parent = all;
    geo.release();  // o holds the reference
    *pairs = res.release();
    *out = o;
    return GPL_OK;
}
