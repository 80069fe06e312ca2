// boolean.cuh — the device code the boolean geometry ops (k_boolean.cu, DESIGN.md §4.19), dissolve (k_dissolve.cu, §4.21)
// and the line clip (k_clip.cu, §4.22) share: the boundary node records and their enumeration, the exact order of the nodes
// along an edge, and the linking of kept pieces into output rings.
#pragma once

#include <math.h>

#include "common.cuh"
#include "overlay.cuh"
#include "pair_dist.cuh"

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
    double a2;                                      // twice the f64 shoelace area, relative to the first coordinate
};

// Side 0 may instead be a line or point column (clip, k_clip.cu): v[0].ro gives the coordinates of each chain, mem[0] the
// chains (points) of a row (NULL for LineString / Point), and sg[0] / box[0] are NULL.
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

// the node the edge (s, g) of the other side puts on the directed edge (p, q): K_VERTEX when s lies strictly inside (p, q),
// K_CROSS for a proper crossing, else -1 (s on the line of (p, q) rules a proper crossing out, so there is at most one)
__device__ __forceinline__ int edge_node(double2 p, double2 q, double2 s, double2 g) {
    const int os = orient_sign(p, q, s), og = orient_sign(p, q, g);
    if (os == 0 && point_in_rect(s, p, q) && !same_pt(s, p) && !same_pt(s, q)) return K_VERTEX;
    if (os * og < 0 && orient_sign(s, g, p) * orient_sign(s, g, q) < 0) return K_CROSS;
    return -1;
}

// One enumeration pass: the nodes of the directed edges of rings [xr0, xr1) of side X against the rings [yr0, yr1) of the
// other side (and, when STARTS, their starts).  Returns this lane's number of nodes; WRITE: also stores them at
// base + atomicAdd(slot).
template <bool WRITE, bool STARTS = true>
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
            if (STARTS && sub == 0) {
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
                    const int kind = edge_node(p, q, s, g);
                    if (kind == K_VERTEX) {  // s: a vertex inside (p, q)
                        ++cnt;
                        if (WRITE) {
                            const double t = ((s.x - p.x) * dx + (s.y - p.y) * dy) / dd;
                            base[atomicAdd(slot, 1)] = BNode{s, t, rx, -1, (int32_t)i, -1, (int8_t)X, K_VERTEX, 0, 0};
                        }
                    }
                    if (kind == K_CROSS) {  // a proper crossing
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

// The enumeration pass with a line chain as side X (side 0; clip, k_clip.cu): the chain is directed in stored order and has
// no closing edge and no σ.  Segment i with distinct ends gets a K_START record, then one record per vertex of the rings
// [yr0, yr1) of side 1 strictly inside it and per proper crossing, in enumeration order; a segment with equal ends gets
// none.  The START record's keep is 1 when the segment's start lies on one of those rings (a contact).  Lanes form groups
// per segment as in node_pass; the G lanes of a group place their records by group ballots, so the order is fixed and no
// atomics are needed.  Count pass: nrec[i] = the segment's record count; WRITE: the records of segment i go to
// nodes + roff[i].  Returns this lane's number of records.
template <bool WRITE>
__device__ int64_t line_node_pass(const BOperands &o, const Chain &cx, int64_t chain, int64_t yr0, int64_t yr1, int lane,
                                  int64_t *nrec, const int64_t *roff, BNode *nodes) {
    const Side &yv = o.v[1];
    const int64_t nseg = cx.coords() - 1;
    int64_t cnt = 0;
    int groups = 32;
    while (groups > 1 && groups / 2 >= nseg) groups >>= 1;
    const int G = 32 / groups, grp = lane / G, sub = lane - grp * G;
    const unsigned gmask = G == 32 ? 0xffffffffu : ((1u << G) - 1u) << (grp * G), below = (1u << lane) - 1u;
    for (int64_t b0 = 0; b0 < nseg; b0 += groups) {
        const int64_t i = b0 + grp;
        if (i >= nseg) continue;
        const double2 p = cx[i], q = cx[i + 1];
        if (same_pt(p, q)) continue;
        const double ex0 = fmin(p.x, q.x), ex1 = fmax(p.x, q.x), ey0 = fmin(p.y, q.y), ey1 = fmax(p.y, q.y);
        const double dx = q.x - p.x, dy = q.y - p.y, dd = dx * dx + dy * dy;
        BNode *base = WRITE ? nodes + roff[i] : nullptr;
        int64_t k = 1;  // records of the segment so far (the START is record 0)
        bool contact = false;
        for (int64_t ry = yr0; ry < yr1; ++ry) {
            if (o.sg[1][ry] == 0) continue;
            const double4 rb = o.box[1][ry];
            if (ex1 < rb.x || rb.z < ex0 || ey1 < rb.y || rb.w < ey0) continue;
            const Chain cy = part_ring(yv, ry);
            const int64_t ny = cy.coords() - 1;
            for (int64_t jb = 0; jb < ny; jb += G) {
                const int64_t j = jb + sub;
                int kind = -1;
                double2 s = p, g = p;
                if (j < ny) {
                    s = cy[j], g = cy[j + 1];
                    if (!same_pt(s, g) && !(ex1 < fmin(s.x, g.x) || fmax(s.x, g.x) < ex0 || ey1 < fmin(s.y, g.y) || fmax(s.y, g.y) < ey0)) {
                        kind = edge_node(p, q, s, g);
                        contact = contact || (point_in_rect(p, s, g) && orient_sign(s, g, p) == 0);
                    }
                }
                const unsigned hits = __ballot_sync(gmask, kind >= 0);
                if (WRITE && kind >= 0) {
                    const int64_t at = k + __popc(hits & below);
                    if (kind == K_VERTEX) {
                        const double t = ((s.x - p.x) * dx + (s.y - p.y) * dy) / dd;
                        base[at] = BNode{s, t, chain, -1, (int32_t)i, -1, 0, K_VERTEX, 0, 0};
                    } else {
                        const double op = orient2d(s.x, s.y, g.x, g.y, p.x, p.y), oq = orient2d(s.x, s.y, g.x, g.y, q.x, q.y);
                        base[at] = BNode{crossing_point(p, q, s, g), op / (op - oq), chain, ry, (int32_t)i, (int32_t)j, 0, K_CROSS, 0, 0};
                    }
                }
                k += __popc(hits);
            }
        }
        contact = __ballot_sync(gmask, contact) != 0;
        if (sub == 0) {
            cnt += k;
            if (WRITE) base[0] = BNode{p, 0.0, chain, -1, (int32_t)i, -1, 0, K_START, 0, (int8_t)(contact ? 1 : 0)};
            else nrec[i] = k;
        }
    }
    return cnt;
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

// ---- linking and ring assembly: one thread per row ----------------------------------------------------------------------
// the kept pieces of one row, in output direction.  BY_STATE: a kept piece in state S_IN is written reversed (either side's
// pieces in the other of a symmetric difference, a remainder's cutter pieces, §4.23); else, with rev_b, B's pieces (a
// difference)
template <bool BY_STATE>
struct Pieces {
    const BOperands *o;
    const BNode *nd;  // the row's nodes
    int64_t nn;
    const int32_t *kp;  // kept piece -> node index
    bool rev_b;
    __device__ bool rev(int j) const { return BY_STATE ? nd[kp[j]].state == S_IN : rev_b && nd[kp[j]].side == 1; }
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

template <bool BY_STATE>
struct FromPtLess {  // pieces by the output coordinates of their start
    const Pieces<BY_STATE> *pc;
    __device__ bool operator()(int32_t a, int32_t b) const {
        const int c = pt_cmp(pc->from_pt(a), pc->from_pt(b));
        return c ? c < 0 : a < b;
    }
};

// 0 outside / 1 on the boundary / 2 inside of the loop through the from-points of its pieces
template <bool BY_STATE>
static __device__ int point_in_loop(const Pieces<BY_STATE> &pc, const int32_t *lp, const BLoop &L, double2 v) {
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

// Link the kept pieces of the nodes nd[0, nn) (ordered by edge) into output rings: scratch ws (8 int32 per node, at stride
// ws_stride) and L (one BLoop per node); lbox (one double4 per node, or NULL) lets the hole-to-shell search skip the shells
// whose box does not contain the hole's first vertex, and give a hole to the only shell whose box does without walking it.  Counting pass: the members, rings and coordinates (nm, nr, nc);
// WRITE: the MultiPolygon's part / ring offsets and coordinates from the bases mb, rb, cb.  The pieces written reversed: with
// BY_STATE those in state S_IN, else with rev_b those of side 1 (Pieces).  BY_STATE is a template argument so that the ops
// that do not need it compile to what they did before it existed.
template <bool WRITE, bool BY_STATE>
__device__ void assemble_pieces(const BOperands &o, bool rev_b, const BNode *__restrict__ nd, int64_t nn, int32_t *__restrict__ ws,
                                int64_t ws_stride, BLoop *__restrict__ L, double4 *__restrict__ lbox, int64_t &nm_out, int64_t &nr_out,
                                int64_t &nc_out, int64_t mb, int64_t rb, int64_t cb, int64_t *__restrict__ part_off,
                                int64_t *__restrict__ ring_off, double2 *__restrict__ oxy) {
    int32_t *kp = ws, *ord = kp + ws_stride, *rank = ord + ws_stride, *gs = rank + ws_stride, *nxt = gs + ws_stride,
            *npos = nxt + ws_stride, *stk = npos + ws_stride, *lp = stk + ws_stride;
    int J = 0;
    for (int64_t k = 0; k < nn; ++k)
        if (nd[k].keep) kp[J++] = (int32_t)k;
    const Pieces<BY_STATE> pc{&o, nd, nn, kp, rev_b};
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
    heap_sort(ord, (int64_t)J, FromPtLess<BY_STATE>{&pc});
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
        double4 bx = make_double4(o0.x, o0.y, o0.x, o0.y);
        for (int i = 1; i < lo.len; ++i) {
            const double2 v = pc.from_pt(lp[lo.start + i]);
            if (lbox) bx = make_double4(fmin(bx.x, v.x), fmin(bx.y, v.y), fmax(bx.z, v.x), fmax(bx.w, v.y));
            if (pt_cmp(v, first) < 0) rot = i, first = v;
            if (i + 1 < lo.len) {
                const double2 e = pc.from_pt(lp[lo.start + i + 1]);
                const double t1 = (v.x - o0.x) * (e.y - o0.y), t2 = (e.x - o0.x) * (v.y - o0.y);
                a2 += t1 - t2;
                mag += fabs(t1) + fabs(t2);
            }
        }
        lo.ncoord = lo.len, lo.rot = rot, lo.first = first, lo.parent = -1, lo.a2 = a2;
        if (lbox) lbox[l] = bx;
        lo.type = lo.len < 3 || fabs(a2) <= (double)(lo.len + 4) * 0x1p-52 * mag ? 0 : a2 > 0.0 ? 1 : -1;
    }
    // every hole to the smallest shell containing it.  With boxes: a shell whose box misses the hole's first vertex cannot
    // contain it, and when only one shell's box holds it, that shell is the hole's (every hole of a union of valid rows lies
    // in a shell), so the hole is given to it without walking the shell
    for (int h = 0; h < nl; ++h) {
        if (L[h].type >= 0) continue;
        int best = -1, only = -1, nbox = 0;
        if (lbox) {
            const double2 f = L[h].first;
            for (int s = 0; s < nl && nbox < 2; ++s) {
                if (L[s].type <= 0) continue;
                const double4 sb = lbox[s];
                if (f.x < sb.x || sb.z < f.x || f.y < sb.y || sb.w < f.y) continue;
                only = s, ++nbox;
            }
            if (nbox == 1) best = only;
        }
        double barea = 0.0;
        for (int s = 0; s < nl && !(lbox && nbox < 2); ++s) {
            if (L[s].type <= 0) continue;
            if (lbox) {  // the hole's first vertex outside the shell's box: point_in_loop below would give 0
                const double4 sb = lbox[s];
                const double2 f = L[h].first;
                if (f.x < sb.x || sb.z < f.x || f.y < sb.y || sb.w < f.y) continue;
            }
            // the hole's smallest vertex first: for intersection and difference it is an input vertex
            int pos = point_in_loop(pc, lp, L[s], L[h].first);
            for (int i = 0; i < L[h].len && pos == 1; ++i) pos = point_in_loop(pc, lp, L[s], pc.from_pt(lp[L[h].start + i]));
            if (pos != 2) continue;
            const double a = L[s].a2;
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
    nm_out = nm, nr_out = nout, nc_out = ncoords;
    if (!WRITE) return;
    heap_sort(stk, (int64_t)nout, LoopLess{L});
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

// out[k] = the first position of keys (sorted, length m) that is >= k, for k in [0, nq] (k_dissolve.cu)
__global__ void __launch_bounds__(256) k_lower_bounds(const uint64_t *__restrict__ keys, int64_t m, int64_t nq, int64_t *__restrict__ out);
// Row k of the MultiPolygon column *out is row row[k] of srcs[src[k]] (each a Polygon or MultiPolygon column, or NULL when no
// row names it), validity included, with offsets rebased; src and row on the device (k_overlay_modes.cu)
int gather_polygons(gpl_ctx *ctx, const gpl_array *const srcs[3], const int8_t *src, const uint64_t *row, int64_t m, gpl_array **out);
// The remainder of every row of subj: the row minus the union of the rows of cut its closed geometry intersects, as a
// MultiPolygon column of subj's length (DESIGN.md §4.23; k_dissolve.cu).  Fewer than 2^31 rows in the two columns together.
int remainder_rows(gpl_ctx *ctx, const gpl_array *subj, const gpl_array *cut, gpl_array **out);

}  // namespace gpl
