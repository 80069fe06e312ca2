// k_clip.cu — clipping of (Multi)LineString and (Multi)Point columns by (Multi)Polygon columns: row-wise geometry
// (gpl_clip, intersection or difference), the length of the intersection (gpl_clip_length), a geometry clip join
// (gpl_clip_join) and a length-weighted overlay join (gpl_overlay_length_join).  geo 0.27 has the line case as
// BooleanOps::clip(&self, &MultiLineString, invert) (recalled).  DESIGN.md §4.22 has the derivation.
//
// Both ops work on the closed polygon: intersection keeps what lies in its interior or on its boundary, difference what lies
// strictly outside.  Each directed line segment is cut at the polygon vertices strictly inside it and at its proper crossings
// with polygon edges (line_node_pass, boolean.cuh):
//   records   one per segment start (with a flag: the start lies on the polygon boundary, a contact), one per polygon vertex
//             inside the segment, one per proper crossing, whose point is crossing_point(line segment, polygon edge); a count
//             pass writes one count per segment and a scan gives every segment fixed record slots;
//   order     the records of a segment are sorted along it by NodeLess::along (exact signs), by the lane owning the segment;
//             a crossing at the point of a polygon vertex just before it (a hole touching its shell there) is dropped: the
//             vertex is the node;
//   states    the piece after a record is in, on or out of the closed polygon.  It is located exactly (region_pos of the
//             symbolic point just after the record's point along the segment) only after the first start of a chain, after
//             a start that is a contact or follows a zero-length segment, and after a polygon vertex; every other piece
//             takes the state of the piece before it, flipped at a proper crossing (which lies on exactly one edge of a valid
//             polygon).  The states are carried across segments by a warp scan of (constant | flip) transfer functions;
//   emit      runs of consecutive kept pieces of one chain become members (difference also splits a run at a kept piece that
//             starts on the boundary); the first point of every piece of nonzero rounded length and the end of every run are
//             written, placed by warp scans of per-segment counts in a count pass and a write pass.
// Points are located one lane per point (exact, sequential over the polygon's edges) and compacted by ballots.
// Layout: one warp per row, or per candidate pair of a join; lanes own segments in row order, 32 at a time.  No stage runs
// one thread per row, and every step depends on the row alone, so a row's output is deterministic and the joins reproduce
// the row-wise bytes.
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

constexpr int kClipThreads = 128;
constexpr unsigned kFull = 0xffffffffu;

enum { P_OUT = 0, P_ON = 1, P_IN = 2 };            // a piece's position: region_pos's codes
enum { SF_FIRST = 1, SF_END = 2, SF_DEGEN = 4 };   // slot flags: a chain's first coordinate, its last, a zero-length segment
enum { N_CONTACT = 1, N_VOID = 2 };                // BNode::keep of a START record / of a dropped crossing

__device__ __forceinline__ int flip(int s) { return s == P_IN ? P_OUT : P_IN; }

// the chains (lines) or points [k0, k1) of row r of side 0 and its coordinates [c0, c1)
__device__ __forceinline__ void row_coords(const BOperands &o, bool lines, int64_t r, int64_t &k0, int64_t &k1, int64_t &c0, int64_t &c1) {
    row_members(o, 0, r, k0, k1);
    if (lines) c0 = o.v[0].ro[k0], c1 = o.v[0].ro[k1];
    else c0 = k0, c1 = k1;
}
__device__ __forceinline__ bool box_holds(double4 b, double x, double y) { return b.x <= x && x <= b.z && b.y <= y && y <= b.w; }

// 2 inside / 1 on the boundary / 0 outside of the polygon members [m0, m1) of side 1 for the symbolic point q, as
// k_bool_classify reads the members: rings with σ 0 contribute nothing.  Warp cooperative.
__device__ int clip_region_pos(const BOperands &o, int64_t m0, int64_t m1, const SymQ &q, int lane) {
    const Side &v = o.v[1];
    bool boundary = false;
    for (int64_t m = m0; m < m1; ++m) {
        const int64_t e = v.go[m], e1 = v.go[m + 1];
        if (e >= e1 || o.sg[1][e] == 0 || !box_holds(o.box[1][e], q.xx, q.xy)) continue;
        int pos = sym_ring_pos(q, part_ring(v, e), lane);
        for (int64_t h = e + 1; pos == 2 && h < e1; ++h) {
            if (o.sg[1][h] == 0 || !box_holds(o.box[1][h], q.xx, q.xy)) continue;
            const int ph = sym_ring_pos(q, part_ring(v, h), lane);
            if (ph != 0) pos = ph == 2 ? 0 : 1;
        }
        if (pos == 2) return 2;
        boundary = boundary || pos == 1;
    }
    return boundary ? 1 : 0;
}

// the same for a point, by one thread
__device__ int ring_pos_thread(const Chain &c, double2 p) {
    if (c.n < 2) return 0;
    const int64_t m = c.coords();
    int wn = 0;
    for (int64_t i = 0; i + 1 < m; ++i) {
        const double2 s = c[i], e = c[i + 1];
        if (s.y <= p.y) {
            if (e.y >= p.y) {
                const int o = orient_sign(s, e, p);
                if (o > 0 && e.y != p.y) ++wn;
                else if (o == 0 && value_in_between(p.x, s.x, e.x)) return 1;
            }
        } else if (e.y <= p.y) {
            const int o = orient_sign(s, e, p);
            if (o < 0) --wn;
            else if (o == 0 && value_in_between(p.x, s.x, e.x)) return 1;
        }
    }
    return wn ? 2 : 0;
}
__device__ int point_region_pos(const BOperands &o, int64_t m0, int64_t m1, double2 p) {
    const Side &v = o.v[1];
    bool boundary = false;
    for (int64_t m = m0; m < m1; ++m) {
        const int64_t e = v.go[m], e1 = v.go[m + 1];
        if (e >= e1 || o.sg[1][e] == 0 || !box_holds(o.box[1][e], p.x, p.y)) continue;
        int pos = ring_pos_thread(part_ring(v, e), p);
        for (int64_t h = e + 1; pos == 2 && h < e1; ++h) {
            if (o.sg[1][h] == 0 || !box_holds(o.box[1][h], p.x, p.y)) continue;
            const int ph = ring_pos_thread(part_ring(v, h), p);
            if (ph != 0) pos = ph == 2 ? 0 : 1;
        }
        if (pos == 2) return 2;
        boundary = boundary || pos == 1;
    }
    return boundary ? 1 : 0;
}

// One warp per row pair: rv[r] = both rows present with only finite coordinates; ncoord[r] = the left row's coordinates
// (0 for an invalid row)
__global__ void __launch_bounds__(kClipThreads) k_clip_prep(int64_t n, BOperands o, bool lines, const uint64_t *__restrict__ ia,
                                                            const uint64_t *__restrict__ ib, int64_t *__restrict__ ncoord, uint8_t *__restrict__ rv) {
    const int lane = threadIdx.x & 31;
    int64_t warp = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
    const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t r = warp; r < n; r += nwarps) {
        const int64_t ra = ia ? (int64_t)ia[r] : r, rb = ib ? (int64_t)ib[r] : r;
        bool ok = bit_get(o.valid[0], ra) && bit_get(o.valid[1], rb);
        int64_t k0, k1, c0 = 0, c1 = 0;
        if (ok) {
            row_coords(o, lines, ra, k0, k1, c0, c1);
            bool fin = true;
            for (int64_t c = c0 + lane; c < c1; c += 32) {
                const double2 q = o.v[0].xy[c];
                fin = fin && isfinite(q.x) && isfinite(q.y);
            }
            int64_t b0, b1;
            row_members(o, 1, rb, b0, b1);
            ok = __all_sync(kFull, fin) && members_finite(o.v[1], b0, b1, lane);
        }
        if (lane == 0) {
            rv[r] = ok ? 1 : 0;
            ncoord[r] = ok ? c1 - c0 : 0;
        }
    }
}

// One warp per row pair: the records of every segment (line_node_pass) at slots sbase[r] + (coordinate index in the row).
// Count pass: nrec and the slot flags (a chain's last coordinate and a zero-length segment get no record), and too_big
// when the row has 2^30 or more records; WRITE: the records at nodes + roff[slot].
template <bool WRITE>
__global__ void __launch_bounds__(kClipThreads, 3) k_clip_nodes(int64_t n, BOperands o, const uint64_t *__restrict__ ia, const uint64_t *__restrict__ ib,
                                                             const uint8_t *__restrict__ rv, const int64_t *__restrict__ sbase, int64_t *__restrict__ nrec,
                                                             uint8_t *__restrict__ sflag, const int64_t *__restrict__ roff, BNode *__restrict__ nodes,
                                                             int *__restrict__ too_big) {
    const int lane = threadIdx.x & 31;
    int64_t warp = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
    const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t r = warp; r < n; r += nwarps) {
        if (!rv[r]) continue;
        const int64_t ra = ia ? (int64_t)ia[r] : r, rb = ib ? (int64_t)ib[r] : r;
        int64_t k0, k1, c0, c1, b0, b1;
        row_coords(o, true, ra, k0, k1, c0, c1);
        row_members(o, 1, rb, b0, b1);
        const int64_t yr0 = o.v[1].go[b0], yr1 = o.v[1].go[b1];
        int64_t c = 0;
        for (int64_t k = k0; k < k1; ++k) {
            const Chain cx = make_line(o.v[0].xy, o.v[0].ro[k], o.v[0].ro[k + 1]);
            const int64_t sb = sbase[r] + (o.v[0].ro[k] - c0);
            if (!WRITE) {
                for (int64_t j = lane; j < cx.n; j += 32) {
                    const bool end = j + 1 == cx.n, degen = !end && same_pt(cx[j], cx[j + 1]);
                    sflag[sb + j] = (uint8_t)((j == 0 ? SF_FIRST : 0) | (end ? SF_END : 0) | (degen ? SF_DEGEN : 0));
                    if (end || degen) nrec[sb + j] = 0;
                }
            }
            c += line_node_pass<WRITE>(o, cx, k, yr0, yr1, lane, nrec + sb, roff + sb, nodes);
        }
        if (!WRITE) {
#pragma unroll
            for (int s = 16; s > 0; s >>= 1) c += __shfl_xor_sync(kFull, c, s);
            if (lane == 0 && c >= (1LL << 30)) atomicExch(too_big, 1);
        }
    }
}

// the records of one segment, [b, e), in the order along it
struct ClipLess {
    const NodeLess *nl;
    double2 p, q;
    __device__ bool operator()(const BNode &a, const BNode &b) const {
        const int c = nl->along(a, b, p, q);
        if (c) return c < 0;
        if (a.kind != b.kind) return a.kind < b.kind;
        if (a.oring != b.oring) return a.oring < b.oring;
        if (a.oseg != b.oseg) return a.oseg < b.oseg;
        if (a.pt.x != b.pt.x) return a.pt.x < b.pt.x;
        return a.pt.y < b.pt.y;
    }
};

// the piece after record k is located exactly (not inferred from the piece before it)
__device__ __forceinline__ bool needs_locate(const BNode &nd, bool first_piece) {
    return nd.kind == K_VERTEX || (nd.kind == K_START && (first_piece || nd.keep == N_CONTACT));
}
__device__ __forceinline__ int64_t next_record(const BNode *nodes, int64_t k, int64_t e) {
    while (k < e && nodes[k].kind == K_CROSS && nodes[k].keep == N_VOID) ++k;
    return k;
}

// the segment owned by this lane: its records [b, e) (none: not a segment with distinct ends), its end w and its flags
struct SegView {
    int64_t b, e;
    double2 w;
    uint8_t f;
    bool first_piece;  // the START is located: the chain's first segment, or one after a zero-length segment
};
__device__ __forceinline__ SegView seg_view(const BOperands &o, int64_t j, int64_t s0, int64_t s1, int64_t c0, const uint8_t *sflag, const int64_t *roff) {
    SegView v{0, 0, make_double2(0.0, 0.0), 0, false};
    if (j >= s1) return v;
    v.f = sflag[j];
    v.b = roff[j], v.e = roff[j + 1];
    if (v.e > v.b) {
        v.w = o.v[0].xy[c0 + (j - s0) + 1];
        v.first_piece = (v.f & SF_FIRST) || (sflag[j - 1] & SF_DEGEN);
    }
    return v;
}

// One warp per row pair: sort each segment's records, drop the crossings that coincide with the vertex before them, locate
// the pieces that need it and carry the states across segments.  LENGTH: len[r] = the length of the kept pieces (in or on),
// NaN for an invalid row.
template <bool LENGTH>
__global__ void __launch_bounds__(kClipThreads, 3) k_clip_classify(int64_t n, BOperands o, const uint64_t *__restrict__ ia, const uint64_t *__restrict__ ib,
                                                                const uint8_t *__restrict__ rv, const int64_t *__restrict__ sbase,
                                                                const uint8_t *__restrict__ sflag, const int64_t *__restrict__ roff,
                                                                BNode *__restrict__ nodes, double *__restrict__ len) {
    const int lane = threadIdx.x & 31;
    int64_t warp = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
    const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    const NodeLess nl{&o};
    for (int64_t r = warp; r < n; r += nwarps) {
        const bool ok = rv[r] != 0;
        double acc = 0.0;
        if (ok) {
            const int64_t ra = ia ? (int64_t)ia[r] : r, rb = ib ? (int64_t)ib[r] : r;
            int64_t k0, k1, c0, c1, m0, m1;
            row_coords(o, true, ra, k0, k1, c0, c1);
            row_members(o, 1, rb, m0, m1);
            const int64_t s0 = sbase[r], s1 = sbase[r + 1];
            int carry = P_OUT;
            for (int64_t jb = s0; jb < s1; jb += 32) {
                const SegView sv = seg_view(o, jb + lane, s0, s1, c0, sflag, roff);
                const int64_t b = sv.b, e = sv.e;
                if (e > b) {
                    const double2 p = nodes[b].pt;
                    heap_sort(nodes + b + 1, e - b - 1, ClipLess{&nl, p, sv.w});
                    for (int64_t k = b + 1; k < e; ++k) {
                        if (nodes[k].kind != K_CROSS || nodes[k - 1].kind != K_VERTEX) continue;
                        double2 s, g;
                        stored_edge(o, 1, nodes[k].oring, nodes[k].oseg, s, g);
                        if (orient_sign(s, g, nodes[k - 1].pt) == 0) nodes[k].keep = N_VOID;
                    }
                }
                // exact locations, one at a time for the whole warp
                int64_t cur = b;
                while (cur < e && !needs_locate(nodes[cur], cur == b && sv.first_piece)) ++cur;
                for (;;) {
                    const bool want = cur < e;
                    unsigned m = __ballot_sync(kFull, want);
                    if (!m) break;
                    const double2 mine = want ? nodes[cur].pt : sv.w;
                    while (m) {
                        const int src = __ffs(m) - 1;
                        m &= m - 1;
                        const double2 x = bcast2(mine, src), v = bcast2(sv.w, src);
                        const int pos = clip_region_pos(o, m0, m1, SymQ{x.x, x.y, v.x, v.y, 0}, lane);
                        if (lane == src) nodes[cur].state = (int8_t)pos;
                    }
                    if (want)
                        for (++cur; cur < e && !needs_locate(nodes[cur], false);) ++cur;
                }
                // the segment's transfer: a constant (it has a located piece) or a flip count; then an inclusive scan
                bool cst = false;
                int val = 0;
                for (int64_t k = next_record(nodes, b, e); k < e; k = next_record(nodes, k + 1, e)) {
                    if (needs_locate(nodes[k], k == b && sv.first_piece)) cst = true, val = nodes[k].state;
                    else if (nodes[k].kind == K_CROSS) val = cst ? flip(val) : val ^ 1;
                }
#pragma unroll
                for (int d = 1; d < 32; d <<= 1) {
                    const bool c2 = __shfl_up_sync(kFull, cst, d);
                    const int v2 = __shfl_up_sync(kFull, val, d);
                    if (lane >= d && !cst) {
                        if (c2) cst = true, val = val ? flip(v2) : v2;
                        else val ^= v2;
                    }
                }
                const bool pc = __shfl_up_sync(kFull, cst, 1);
                const int pv = __shfl_up_sync(kFull, val, 1);
                const int in = lane == 0 ? carry : pc ? pv : pv ? flip(carry) : carry;
                const bool lc = __shfl_sync(kFull, cst, 31);
                const int lv = __shfl_sync(kFull, val, 31);
                carry = lc ? lv : lv ? flip(carry) : carry;
                // every piece's state; LENGTH: the kept pieces' lengths
                int st = in;
                for (int64_t k = next_record(nodes, b, e); k < e;) {
                    if (needs_locate(nodes[k], k == b && sv.first_piece)) st = nodes[k].state;
                    else if (nodes[k].kind == K_CROSS) st = flip(st);
                    nodes[k].state = (int8_t)st;
                    const int64_t kn = next_record(nodes, k + 1, e);
                    if (LENGTH && st != P_OUT) {
                        const double2 a = nodes[k].pt, z = kn < e ? nodes[kn].pt : sv.w;
                        acc += gpl_hypot(z.x - a.x, z.y - a.y);
                    }
                    k = kn;
                }
            }
        }
        if (LENGTH) {
#pragma unroll
            for (int s = 16; s > 0; s >>= 1) acc += __shfl_xor_sync(kFull, acc, s);
            if (lane == 0) len[r] = ok ? acc : nan("");
        }
    }
}

// the value of the nearest lane below this one that defines one, else carry; carry becomes the highest definer's value
__device__ __forceinline__ int last_defined(bool def, int val, int &carry, int lane) {
    const unsigned all = __ballot_sync(kFull, def), below = all & ((1u << lane) - 1u);
    const int got = __shfl_sync(kFull, val, below ? 31 - __clz(below) : 0);
    const int in = below ? got : carry;
    const int top = __shfl_sync(kFull, val, all ? 31 - __clz(all) : 0);
    if (all) carry = top;
    return in;
}
// exclusive warp sum; total: the sum over the warp
__device__ __forceinline__ int64_t warp_excl(int64_t v, int64_t &total, int lane) {
    int64_t inc = v;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const int64_t t = __shfl_up_sync(kFull, inc, d);
        if (lane >= d) inc += t;
    }
    total = __shfl_sync(kFull, inc, 31);
    return inc - v;
}

// The pieces of one segment in order, skipping the dropped crossings and the pieces of zero exact length (between two
// vertex records at one point): fn(pt, end, state, on), on = the piece starts on the polygon boundary.
template <class Fn>
__device__ __forceinline__ void for_pieces(const BNode *nodes, const SegView &sv, Fn &&fn) {
    for (int64_t k = next_record(nodes, sv.b, sv.e); k < sv.e;) {
        const int64_t kn = next_record(nodes, k + 1, sv.e);
        const BNode &nd = nodes[k];
        const double2 end = kn < sv.e ? nodes[kn].pt : sv.w;
        const bool end_vertex = kn >= sv.e || nodes[kn].kind != K_CROSS;
        if (!(nd.kind != K_CROSS && end_vertex && same_pt(nd.pt, end))) fn(nd.pt, end, (int)nd.state, nd.kind != K_START || nd.keep == N_CONTACT);
        k = kn;
    }
}

// One warp per row pair: the MultiLineString of the kept pieces.  Count pass: cm[r] members and cc[r] coordinates; WRITE: the
// members' coordinate offsets at ring_off + mbase[r] and the coordinates at oxy + cbase[r].
template <bool WRITE>
__global__ void __launch_bounds__(kClipThreads) k_clip_emit(int64_t n, BOperands o, const uint64_t *__restrict__ ia, const uint8_t *__restrict__ rv,
                                                            const int64_t *__restrict__ sbase, const uint8_t *__restrict__ sflag,
                                                            const int64_t *__restrict__ roff, const BNode *__restrict__ nodes, bool invert,
                                                            int64_t *__restrict__ cm, int64_t *__restrict__ cc, const int64_t *__restrict__ mbase,
                                                            const int64_t *__restrict__ cbase, int64_t *__restrict__ ring_off, double2 *__restrict__ oxy) {
    const int lane = threadIdx.x & 31;
    int64_t warp = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
    const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t r = warp; r < n; r += nwarps) {
        int64_t tm = 0, tc = 0;  // members and coordinates of the row so far
        if (rv[r]) {
            const int64_t ra = ia ? (int64_t)ia[r] : r;
            int64_t k0, k1, c0, c1;
            row_coords(o, true, ra, k0, k1, c0, c1);
            const int64_t s0 = sbase[r], s1 = sbase[r + 1];
            int kept_carry = 0, run_carry = 0;
            for (int64_t jb = s0; jb < s1; jb += 32) {
                const int64_t j = jb + lane;
                const SegView sv = seg_view(o, j, s0, s1, c0, sflag, roff);
                const bool end = j < s1 && (sv.f & SF_END);
                auto kept = [&](int st) { return invert ? st == P_OUT : st != P_OUT; };
                // was the last piece before this segment kept (false at a chain's start)?
                bool def = end;
                int val = 0;
                for_pieces(nodes, sv, [&](double2, double2, int st, bool) { def = true, val = kept(st); });
                const bool prev_kept = last_defined(def, val, kept_carry, lane) != 0;
                // run events: a break (B, 0) before a piece that is not kept or starts a new run, a piece of nonzero length
                // in a run (N, 1); was the last event before this segment an N?
                def = end, val = 0;
                bool pk = prev_kept;
                for_pieces(nodes, sv, [&](double2 pt, double2 e2, int st, bool on) {
                    const bool kp = kept(st);
                    if (!kp || !pk || (invert && on)) def = true, val = 0;
                    if (kp && !same_pt(pt, e2)) def = true, val = 1;
                    pk = kp;
                });
                const int run_in = last_defined(def, val, run_carry, lane);
                // members and coordinates: a run's first N starts a member, every N writes its start, a B after an N (or the
                // chain's end) writes the run's end point
                auto walk = [&](bool write, int64_t mpos, int64_t cpos, int64_t &nm, int64_t &nc) {
                    nm = 0, nc = 0;
                    int lbn = run_in;
                    bool pk2 = prev_kept;
                    for_pieces(nodes, sv, [&](double2 pt, double2 e2, int st, bool on) {
                        const bool kp = kept(st);
                        if (!kp || !pk2 || (invert && on)) {
                            if (lbn) {
                                if (write) oxy[cpos + nc] = pt;
                                ++nc;
                            }
                            lbn = 0;
                        }
                        if (kp && !same_pt(pt, e2)) {
                            if (!lbn) {
                                if (write) ring_off[mpos + nm] = cpos + nc;
                                ++nm;
                            }
                            if (write) oxy[cpos + nc] = pt;
                            ++nc;
                            lbn = 1;
                        }
                        pk2 = kp;
                    });
                    if (end && lbn) {
                        if (write) oxy[cpos + nc] = o.v[0].xy[c0 + (j - s0)];
                        ++nc;
                    }
                };
                int64_t nm, nc, sm, sc;
                walk(false, 0, 0, nm, nc);
                const int64_t em = warp_excl(nm, sm, lane), ec = warp_excl(nc, sc, lane);
                if (WRITE) walk(true, mbase[r] + tm + em, cbase[r] + tc + ec, nm, nc);
                tm += sm, tc += sc;
            }
        }
        if (!WRITE && lane == 0) cm[r] = tm, cc[r] = tc;
    }
}

// One warp per row pair, one lane per point: the points of the left row in the closed polygon (outside it with invert).
// Count pass: cnt[r]; WRITE: the points at oxy + base[r], in input order.
template <bool WRITE>
__global__ void __launch_bounds__(kClipThreads, 3) k_clip_points(int64_t n, BOperands o, const uint64_t *__restrict__ ia, const uint64_t *__restrict__ ib,
                                                              const uint8_t *__restrict__ rv, bool invert, int64_t *__restrict__ cnt,
                                                              const int64_t *__restrict__ base, double2 *__restrict__ oxy) {
    const int lane = threadIdx.x & 31;
    int64_t warp = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
    const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t r = warp; r < n; r += nwarps) {
        int64_t run = 0;
        if (rv[r]) {
            const int64_t ra = ia ? (int64_t)ia[r] : r, rb = ib ? (int64_t)ib[r] : r;
            int64_t k0, k1, c0, c1, m0, m1;
            row_coords(o, false, ra, k0, k1, c0, c1);
            row_members(o, 1, rb, m0, m1);
            for (int64_t cb = c0; cb < c1; cb += 32) {
                const int64_t c = cb + lane;
                bool keep = false;
                double2 p = make_double2(0.0, 0.0);
                if (c < c1) {
                    p = o.v[0].xy[c];
                    const int pos = point_region_pos(o, m0, m1, p);
                    keep = invert ? pos == P_OUT : pos != P_OUT;
                }
                const unsigned m = __ballot_sync(kFull, keep);
                if (WRITE && keep) oxy[base[r] + run + __popc(m & ((1u << lane) - 1u))] = p;
                run += __popc(m);
            }
        }
        if (!WRITE && lane == 0) cnt[r] = run;
    }
}

// ---- host side --------------------------------------------------------------------------------------------------------
static BOperands clip_operands(const gpl_array *a, const gpl_array *b, const RingPrep &pb) {
    BOperands o;
    const bool multi = a->type == GPL_MULTILINESTRING || a->type == GPL_MULTIPOINT;
    const int64_t *ro = a->type == GPL_LINESTRING ? a->geom_off : a->type == GPL_MULTILINESTRING ? a->ring_off : nullptr;
    o.v[0] = Side{a->type, reinterpret_cast<const double2 *>(a->xy), nullptr, nullptr, ro};
    o.mem[0] = multi ? a->geom_off : nullptr;
    o.valid[0] = a->validity, o.sg[0] = nullptr, o.box[0] = nullptr;
    o.v[1] = pb.view, o.mem[1] = pb.members, o.valid[1] = b->validity, o.sg[1] = pb.sigma.p, o.box[1] = pb.box.p;
    return o;
}

// the stages every line clip shares, for n row pairs: row validity, the records and their states; LENGTH also writes len
struct LineStage {
    Scratch<uint8_t> rv, sflag;
    Scratch<int64_t> sbase, nrec, roff;
    Scratch<BNode> nodes;
};
static int line_stage(gpl_ctx *ctx, const BOperands &o, int64_t n, const uint64_t *ia, const uint64_t *ib, double *len, LineStage &st) {
    Scratch<int64_t> ncoord, tot;
    Scratch<int> too_big;
    GPL_TRY(st.rv.get(ctx, (size_t)n));
    GPL_TRY(ncoord.get(ctx, (size_t)n));
    GPL_TRY(st.sbase.get(ctx, (size_t)n + 1));
    GPL_TRY(tot.get(ctx, 2));
    GPL_TRY(too_big.get(ctx, 1));
    GPL_CUDA(cudaMemsetAsync(too_big.p, 0, sizeof(int), ctx->stream));
    const int grid = warp_grid(n, kClipThreads / 32);
    if (n > 0) GPL_LAUNCH(ctx, k_clip_prep, grid, kClipThreads, 0, n, o, true, ia, ib, ncoord.p, st.rv.p);
    GPL_TRY((exclusive_scan<int64_t, int64_t>(ctx, ncoord.p, n, st.sbase.p, tot.p)));
    int64_t h_slots = 0;
    GPL_CUDA(cudaMemcpyAsync(&h_slots, tot.p, sizeof(int64_t), cudaMemcpyDeviceToHost, ctx->stream));
    GPL_CUDA(cudaStreamSynchronize(ctx->stream));
    GPL_TRY(st.nrec.get(ctx, (size_t)h_slots));
    GPL_TRY(st.sflag.get(ctx, (size_t)h_slots));
    GPL_TRY(st.roff.get(ctx, (size_t)h_slots + 1));
    if (n > 0)
        GPL_LAUNCH(ctx, k_clip_nodes<false>, grid, kClipThreads, 0, n, o, ia, ib, st.rv.p, st.sbase.p, st.nrec.p, st.sflag.p, nullptr, nullptr, too_big.p);
    GPL_TRY((exclusive_scan<int64_t, int64_t>(ctx, st.nrec.p, h_slots, st.roff.p, tot.p + 1)));
    int64_t h_nodes = 0;
    int h_big = 0;
    GPL_CUDA(cudaMemcpyAsync(&h_nodes, tot.p + 1, sizeof(int64_t), cudaMemcpyDeviceToHost, ctx->stream));
    GPL_CUDA(cudaMemcpyAsync(&h_big, too_big.p, sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
    GPL_CUDA(cudaStreamSynchronize(ctx->stream));
    GPL_REQUIRE(!h_big, GPL_ERR_UNSUPPORTED, "clip: a row has 2^30 or more nodes");
    GPL_TRY(st.nodes.get(ctx, (size_t)h_nodes));
    if (n > 0) {
        GPL_LAUNCH(ctx, k_clip_nodes<true>, grid, kClipThreads, 0, n, o, ia, ib, st.rv.p, st.sbase.p, st.nrec.p, st.sflag.p, st.roff.p, st.nodes.p,
                   too_big.p);
        if (len)
            GPL_LAUNCH(ctx, k_clip_classify<true>, grid, kClipThreads, 0, n, o, ia, ib, st.rv.p, st.sbase.p, st.sflag.p, st.roff.p, st.nodes.p, len);
        else
            GPL_LAUNCH(ctx, k_clip_classify<false>, grid, kClipThreads, 0, n, o, ia, ib, st.rv.p, st.sbase.p, st.sflag.p, st.roff.p, st.nodes.p,
                       nullptr);
    }
    return GPL_OK;
}

// the clip of n row pairs (a[ia[r]], b[ib[r]]), or (a[r], b[r]) when ia / ib are NULL, as a MultiLineString or MultiPoint
// column; members[r] (optional, device) receives the member (point) count of each row
static int clip_rows(gpl_ctx *ctx, const BOperands &o, bool lines, int64_t n, const uint64_t *ia, const uint64_t *ib, bool invert, gpl_array **out,
                     Scratch<int64_t> *members) {
    RaggedOut res;
    LineStage st;
    const int grid = warp_grid(n, kClipThreads / 32);
    GPL_TRY(res.init(ctx, n, lines ? 2 : 1));
    int64_t *cm = res.count[0].p;
    if (lines) {
        int64_t *cc = res.count[1].p;
        GPL_TRY(line_stage(ctx, o, n, ia, ib, nullptr, st));
        if (n > 0)
            GPL_LAUNCH(ctx, k_clip_emit<false>, grid, kClipThreads, 0, n, o, ia, st.rv.p, st.sbase.p, st.sflag.p, st.roff.p, st.nodes.p, invert, cm,
                       cc, nullptr, nullptr, nullptr, nullptr);
        GPL_TRY(res.scan_and_allocate());
        if (n > 0)
            GPL_LAUNCH(ctx, k_clip_emit<true>, grid, kClipThreads, 0, n, o, ia, st.rv.p, st.sbase.p, st.sflag.p, st.roff.p, st.nodes.p, invert, cm,
                       cc, res.base[0].p, res.base[1].p, res.off[0].p, reinterpret_cast<double2 *>(res.xy.p));
    } else {
        Scratch<int64_t> ncoord;
        GPL_TRY(st.rv.get(ctx, (size_t)n));
        GPL_TRY(ncoord.get(ctx, (size_t)n));
        if (n > 0) {
            GPL_LAUNCH(ctx, k_clip_prep, grid, kClipThreads, 0, n, o, false, ia, ib, ncoord.p, st.rv.p);
            GPL_LAUNCH(ctx, k_clip_points<false>, grid, kClipThreads, 0, n, o, ia, ib, st.rv.p, invert, cm, nullptr, nullptr);
        }
        GPL_TRY(res.scan_and_allocate());
        if (n > 0)
            GPL_LAUNCH(ctx, k_clip_points<true>, grid, kClipThreads, 0, n, o, ia, ib, st.rv.p, invert, nullptr, res.base[0].p,
                       reinterpret_cast<double2 *>(res.xy.p));
    }
    GPL_TRY(res.finish(st.rv.p, lines ? GPL_MULTILINESTRING : GPL_MULTIPOINT, out));
    if (members) members->ctx = ctx, members->p = res.count[0].take();
    return GPL_OK;
}

}  // namespace gpl

using namespace gpl;

extern "C" int gpl_clip(gpl_ctx *ctx, const gpl_array *a, const gpl_array *b, int invert, gpl_array **out) {
    GPL_REQUIRE(ctx && a && b && out, GPL_ERR_INVALID_ARG, "gpl_clip: NULL argument");
    GPL_REQUIRE((is_line(a->type) || is_point(a->type)) && is_area(b->type), GPL_ERR_INVALID_TYPE,
                "Expected (Multi)LineString or (Multi)Point x (Multi)Polygon (found %s x %s)", type_name(a->type), type_name(b->type));
    GPL_TRY(require_same_length(a, b, "clip"));
    GPL_CUDA(cudaSetDevice(ctx->device));
    RingPrep pb;
    GPL_TRY(ring_prep(ctx, b, pb));
    return clip_rows(ctx, clip_operands(a, b, pb), is_line(a->type), a->n_geoms, nullptr, nullptr, invert != 0, out, nullptr);
}

extern "C" int gpl_clip_length(gpl_ctx *ctx, const gpl_array *a, const gpl_array *b, double *out, uint8_t *out_validity, int mem) {
    GPL_REQUIRE(ctx && a && b && out, GPL_ERR_INVALID_ARG, "gpl_clip_length: NULL argument");
    GPL_TRY(check_mem(mem, "gpl_clip_length"));
    GPL_REQUIRE(is_line(a->type) && is_area(b->type), GPL_ERR_INVALID_TYPE, "Expected (Multi)LineString x (Multi)Polygon (found %s x %s)",
                type_name(a->type), type_name(b->type));
    GPL_TRY(require_same_length(a, b, "clip_length"));
    GPL_CUDA(cudaSetDevice(ctx->device));
    const int64_t n = a->n_geoms;
    if (n == 0) return GPL_OK;
    RingPrep pb;
    GPL_TRY(ring_prep(ctx, b, pb));
    RowOut<double> res;
    GPL_TRY(res.get(ctx, out, n, mem));
    LineStage st;
    GPL_TRY(line_stage(ctx, clip_operands(a, b, pb), n, nullptr, nullptr, res.p, st));
    if (out_validity) GPL_TRY(finish_bitmap(ctx, st.rv.p, n, out_validity, mem));
    return res.deliver(ctx);
}

extern "C" int gpl_clip_join(gpl_ctx *ctx, const gpl_array *lhs, const gpl_array *rhs, gpl_pairs **pairs, gpl_array **out) {
    GPL_REQUIRE(ctx && lhs && rhs && pairs && out, GPL_ERR_INVALID_ARG, "gpl_clip_join: NULL argument");
    *pairs = nullptr, *out = nullptr;
    GPL_REQUIRE((is_line(lhs->type) || is_point(lhs->type)) && is_area(rhs->type), GPL_ERR_INVALID_TYPE,
                "Expected (Multi)LineString or (Multi)Point x (Multi)Polygon (found %s x %s)", type_name(lhs->type), type_name(rhs->type));
    GPL_CUDA(cudaSetDevice(ctx->device));
    const int64_t nl = lhs->n_geoms, nr = rhs->n_geoms;
    GPL_REQUIRE(nl < (1LL << 31) && nr < (1LL << 31), GPL_ERR_UNSUPPORTED, "gpl_clip_join: at most 2^31 rows per side");
    Pairs cand(nullptr, gpl_pairs_free);
    GPL_TRY(join_candidate_pairs(ctx, lhs, rhs, JOIN_INTERSECTS, "gpl_clip_join", false, cand));
    const int64_t n = cand->n;
    RingPrep pr;
    GPL_TRY(ring_prep(ctx, rhs, pr));
    const bool lines = is_line(lhs->type);
    gpl_array *all = nullptr;
    Scratch<int64_t> members;
    GPL_TRY(clip_rows(ctx, clip_operands(lhs, rhs, pr), lines, n, cand->lhs, cand->rhs, false, &all, &members));
    std::unique_ptr<gpl_array, void (*)(gpl_array *)> geo(all, gpl_array_free);
    // drop the pairs whose intersection has no member (lines that only touch)
    GPL_TRY(keep_nonempty_rows(ctx, cand.get(), all, members.p, pairs, out));
    geo.release();  // *out holds the reference
    return GPL_OK;
}

extern "C" int gpl_overlay_length_join(gpl_ctx *ctx, const gpl_array *lhs, const gpl_array *rhs, gpl_pairs **out) {
    GPL_REQUIRE(ctx && lhs && rhs && out, GPL_ERR_INVALID_ARG, "gpl_overlay_length_join: NULL argument");
    *out = nullptr;
    GPL_REQUIRE(is_line(lhs->type) && is_area(rhs->type), GPL_ERR_INVALID_TYPE, "Expected (Multi)LineString x (Multi)Polygon (found %s x %s)",
                type_name(lhs->type), type_name(rhs->type));
    GPL_CUDA(cudaSetDevice(ctx->device));
    const int64_t nl = lhs->n_geoms, nr = rhs->n_geoms;
    GPL_REQUIRE(nl < (1LL << 31) && nr < (1LL << 31), GPL_ERR_UNSUPPORTED, "gpl_overlay_length_join: at most 2^31 rows per side");
    Pairs res(nullptr, gpl_pairs_free);
    GPL_TRY(join_candidate_pairs(ctx, lhs, rhs, JOIN_INTERSECTS, "gpl_overlay_length_join", true, res));
    if (res->n > 0) {
        RingPrep pr;
        GPL_TRY(ring_prep(ctx, rhs, pr));
        LineStage st;
        GPL_TRY(line_stage(ctx, clip_operands(lhs, rhs, pr), res->n, res->lhs, res->rhs, res->dist, st));
        GPL_CUDA(cudaStreamSynchronize(ctx->stream));  // the stage's scratch returns to the cache when this scope ends
    }
    *out = res.release();
    return GPL_OK;
}
