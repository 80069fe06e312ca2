// k_boolean.cu — intersection, union, difference and symmetric difference geometry of two (Multi)Polygon columns, row-wise (gpl_boolean_op) and as
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

__device__ __forceinline__ bool keep_piece(int op, int side, int st) {
    // symmetric difference, either side: outside the other operand as it is, inside it reversed; on a shared edge both sides
    // of the edge are in the same number of operands (same direction) or both in the result (opposite): never kept
    if (op == GPL_BOOLEAN_SYMMETRIC_DIFFERENCE) return st == S_OUT || st == S_IN;
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

// One thread per row.  Scratch (8 int32 per node, one BLoop per node) is indexed by the row's node offset.  Counting pass:
// members, rings and coordinates of the row; WRITE: the MultiPolygon's part / ring offsets and coordinates at the row's bases.
template <bool WRITE, bool BY_STATE>
__global__ void __launch_bounds__(128) k_bool_assemble(int64_t n, BOperands o, int op, const int64_t *__restrict__ off, const BNode *__restrict__ nodes,
                                                       int32_t *__restrict__ ws, int64_t ws_stride, BLoop *__restrict__ loops,
                                                       int64_t *__restrict__ cm, int64_t *__restrict__ cr, int64_t *__restrict__ cc,
                                                       const int64_t *__restrict__ mbase, const int64_t *__restrict__ rbase,
                                                       const int64_t *__restrict__ cbase, int64_t *__restrict__ part_off,
                                                       int64_t *__restrict__ ring_off, double2 *__restrict__ oxy) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; r < n; r += stride) {
        const int64_t o0 = off[r], nn = off[r + 1] - o0;
        int64_t nm, nr, nc;
        assemble_pieces<WRITE, BY_STATE>(o, op == GPL_BOOLEAN_DIFFERENCE, nodes + o0, nn, ws + o0, ws_stride, loops + o0, nullptr, nm, nr, nc,
                               WRITE ? mbase[r] : 0, WRITE ? rbase[r] : 0, WRITE ? cbase[r] : 0, part_off, ring_off, oxy);
        if (!WRITE) cm[r] = nm, cr[r] = nr, cc[r] = nc;
    }
}

// the MultiPolygon of `op` for n row pairs (a[ia[r]], b[ib[r]]), or (a[r], b[r]) when ia / ib are NULL; members[r] (optional,
// device) receives the member count of each row
static int boolean_rows(gpl_ctx *ctx, const BOperands &ops, int64_t n, const uint64_t *ia, const uint64_t *ib, int op, gpl_array **out,
                        Scratch<int64_t> *members) {
    RaggedOut res;
    Scratch<int64_t> cnt, off;
    Scratch<uint8_t> rv;
    Scratch<int> too_big;
    GPL_TRY(res.init(ctx, n, 3));
    GPL_TRY(cnt.get(ctx, (size_t)n));
    GPL_TRY(off.get(ctx, (size_t)n + 1));
    GPL_TRY(rv.get(ctx, (size_t)n));
    GPL_TRY(too_big.get(ctx, 1));
    GPL_CUDA(cudaMemsetAsync(too_big.p, 0, sizeof(int), ctx->stream));
    const int grid = warp_grid(n, kBoolThreads / 32);
    if (n > 0)
        GPL_LAUNCH(ctx, k_bool_nodes<false>, grid, kBoolThreads, 0, n, ops, ia, ib, cnt.p, rv.p, nullptr, nullptr, too_big.p);
    GPL_TRY((exclusive_scan<int64_t, int64_t>(ctx, cnt.p, n, off.p, res.tot.p)));
    int64_t h_nodes = 0;
    int h_big = 0;
    GPL_CUDA(cudaMemcpyAsync(&h_nodes, res.tot.p, sizeof(int64_t), cudaMemcpyDeviceToHost, ctx->stream));
    GPL_CUDA(cudaMemcpyAsync(&h_big, too_big.p, sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
    GPL_CUDA(cudaStreamSynchronize(ctx->stream));
    GPL_REQUIRE(!h_big, GPL_ERR_UNSUPPORTED, "boolean_op: a row has 2^30 or more boundary nodes");
    Scratch<BNode> nodes;
    Scratch<int32_t> ws;
    Scratch<BLoop> loops;
    GPL_TRY(nodes.get(ctx, (size_t)h_nodes));
    GPL_TRY(ws.get(ctx, (size_t)h_nodes * 8));
    GPL_TRY(loops.get(ctx, (size_t)h_nodes));
    const int tgrid = (int)std::max<int64_t>(1, std::min<int64_t>(ceil_div(n, 128), (int64_t)kSMs * 16));
    const bool sym = op == GPL_BOOLEAN_SYMMETRIC_DIFFERENCE;  // pieces reversed by their state
    int64_t *cm = res.count[0].p, *cr = res.count[1].p, *cc = res.count[2].p;
    if (n > 0) {
        GPL_LAUNCH(ctx, k_bool_nodes<true>, grid, kBoolThreads, 0, n, ops, ia, ib, cnt.p, rv.p, off.p, nodes.p, too_big.p);
        GPL_LAUNCH(ctx, k_bool_classify, grid, kBoolThreads, 0, n, ops, ia, ib, op, off.p, nodes.p);
        GPL_LAUNCH(ctx, (sym ? k_bool_assemble<false, true> : k_bool_assemble<false, false>), tgrid, 128, 0, n, ops, op, off.p, nodes.p, ws.p,
                   h_nodes, loops.p, cm, cr, cc, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr);
    }
    GPL_TRY(res.scan_and_allocate());
    if (n > 0)
        GPL_LAUNCH(ctx, (sym ? k_bool_assemble<true, true> : k_bool_assemble<true, false>), tgrid, 128, 0, n, ops, op, off.p, nodes.p, ws.p,
                   h_nodes, loops.p, cm, cr, cc, res.base[0].p, res.base[1].p, res.base[2].p, res.off[0].p, res.off[1].p,
                   reinterpret_cast<double2 *>(res.xy.p));
    GPL_TRY(res.finish(rv.p, GPL_MULTIPOLYGON, out));
    if (members) members->ctx = ctx, members->p = res.count[0].take();
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

// keep[k] = 1 when row k of the join's output has a member
__global__ void __launch_bounds__(256) k_nonempty(int64_t n, const int64_t *__restrict__ members, uint8_t *__restrict__ keep) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += stride) keep[i] = members[i] > 0;
}

int keep_nonempty_rows(gpl_ctx *ctx, const gpl_pairs *cand, gpl_array *all, const int64_t *members, gpl_pairs **pairs, gpl_array **out) {
    const int64_t n = cand->n;
    Scratch<uint8_t> keep;
    Scratch<int64_t> goff;
    GPL_TRY(keep.get(ctx, (size_t)n));
    if (n > 0) GPL_LAUNCH(ctx, k_nonempty, flat_grid(n), 256, 0, n, members, keep.p);
    Pairs res(nullptr, gpl_pairs_free);
    GPL_TRY(keep_pairs(ctx, cand, keep.p, res, all->geom_off, &goff));
    const int64_t m = res->n;
    // every output row is valid: a null or non-finite pair has no member and is dropped
    Scratch<uint8_t> bm;
    GPL_TRY(bm.get(ctx, (size_t)(m + 7) / 8));
    GPL_CUDA(cudaMemsetAsync(bm.p, 0xff, (size_t)(m + 7) / 8, ctx->stream));
    GPL_CUDA(cudaStreamSynchronize(ctx->stream));
    gpl_array *o = array_new(ctx, all->type);
    o->n_geoms = m, o->n_parts = all->n_parts, o->n_rings = all->n_rings, o->n_coords = all->n_coords;
    o->geom_off = goff.take(), o->own_geom = true;
    o->part_off = all->part_off, o->ring_off = all->ring_off, o->xy = all->xy;  // shared with the uncompacted result
    o->validity = bm.take(), o->own_valid = true;
    o->parent = all;
    *pairs = res.release();
    *out = o;
    return GPL_OK;
}

int RaggedOut::init(gpl_ctx *c, int64_t rows, int nlevels) {
    ctx = c, n = rows, levels = nlevels;
    for (int k = 0; k < levels; ++k) {
        GPL_TRY(count[k].get(ctx, (size_t)n));
        GPL_TRY(base[k].get(ctx, (size_t)n + 1));
    }
    return tot.get(ctx, 3);
}

int RaggedOut::scan_and_allocate() {
    for (int k = 0; k < levels; ++k) GPL_TRY((exclusive_scan<int64_t, int64_t>(ctx, count[k].p, n, base[k].p, tot.p + k)));
    GPL_CUDA(cudaMemcpyAsync(total, tot.p, sizeof(int64_t) * levels, cudaMemcpyDeviceToHost, ctx->stream));
    GPL_CUDA(cudaStreamSynchronize(ctx->stream));
    for (int k = 0; k + 1 < levels; ++k) GPL_TRY(off[k].get(ctx, (size_t)total[k] + 1));
    return xy.get(ctx, (size_t)total[levels - 1] * 2);
}

int RaggedOut::finish(const uint8_t *row_valid_bytes, int type, gpl_array **out) {
    // the last offset of each lower level: the total of the level below, which the scan left at base[k + 1][n]
    for (int k = 0; k + 1 < levels; ++k)
        GPL_CUDA(cudaMemcpyAsync(off[k].p + total[k], base[k + 1].p + n, sizeof(int64_t), cudaMemcpyDeviceToDevice, ctx->stream));
    Scratch<uint8_t> bm;
    GPL_TRY(bm.get(ctx, (size_t)(n + 7) / 8));
    GPL_TRY(pack_bits(ctx, row_valid_bytes, bm.p, n));
    GPL_CUDA(cudaStreamSynchronize(ctx->stream));  // the caller's scratch returns to the cache after this
    gpl_array *res = array_new(ctx, type);
    res->n_geoms = n, res->n_coords = total[levels - 1];
    res->geom_off = base[0].take(), res->own_geom = true;
    if (levels == 3) res->n_parts = total[0], res->part_off = off[0].take(), res->own_part = true;
    if (levels >= 2) res->n_rings = total[levels - 2], res->ring_off = off[levels - 2].take(), res->own_ring = true;
    res->xy = xy.take(), res->own_xy = true;
    res->validity = bm.take(), res->own_valid = true;
    *out = res;
    return GPL_OK;
}
}  // namespace gpl

using namespace gpl;

extern "C" int gpl_boolean_op(gpl_ctx *ctx, const gpl_array *a, const gpl_array *b, int op, gpl_array **out) {
    GPL_REQUIRE(ctx && a && b && out, GPL_ERR_INVALID_ARG, "gpl_boolean_op: NULL argument");
    GPL_REQUIRE(op == GPL_BOOLEAN_INTERSECTION || op == GPL_BOOLEAN_UNION || op == GPL_BOOLEAN_DIFFERENCE ||
                    op == GPL_BOOLEAN_SYMMETRIC_DIFFERENCE,
                GPL_ERR_INVALID_ARG,
                "gpl_boolean_op: unknown op %d", op);
    GPL_REQUIRE(is_area(a->type) && is_area(b->type), GPL_ERR_INVALID_TYPE, "Expected (Multi)Polygon x (Multi)Polygon (found %s x %s)",
                type_name(a->type), type_name(b->type));
    GPL_TRY(require_same_length(a, b, "boolean_op"));
    GPL_CUDA(cudaSetDevice(ctx->device));
    RingPrep pa, pb;
    GPL_TRY(ring_prep(ctx, a, pa));
    GPL_TRY(ring_prep(ctx, b, pb));
    return boolean_rows(ctx, operands(a, pa, b, pb), a->n_geoms, nullptr, nullptr, op, out, nullptr);
}

extern "C" int gpl_overlay_join(gpl_ctx *ctx, const gpl_array *lhs, const gpl_array *rhs, gpl_pairs **pairs, gpl_array **out) {
    GPL_REQUIRE(ctx && lhs && rhs && pairs && out, GPL_ERR_INVALID_ARG, "gpl_overlay_join: NULL argument");
    *pairs = nullptr, *out = nullptr;
    GPL_REQUIRE(is_area(lhs->type) && is_area(rhs->type), GPL_ERR_INVALID_TYPE, "Expected (Multi)Polygon x (Multi)Polygon (found %s x %s)",
                type_name(lhs->type), type_name(rhs->type));
    GPL_CUDA(cudaSetDevice(ctx->device));
    const int64_t nl = lhs->n_geoms, nr = rhs->n_geoms;
    GPL_REQUIRE(nl < (1LL << 31) && nr < (1LL << 31), GPL_ERR_UNSUPPORTED, "gpl_overlay_join: at most 2^31 rows per side");
    Pairs cand(nullptr, gpl_pairs_free);
    GPL_TRY(join_candidate_pairs(ctx, lhs, rhs, JOIN_INTERSECTS, "gpl_overlay_join", false, cand));
    const int64_t n = cand->n;
    RingPrep pl, pr;
    GPL_TRY(ring_prep(ctx, lhs, pl));
    GPL_TRY(ring_prep(ctx, rhs, pr));
    gpl_array *all = nullptr;
    Scratch<int64_t> members;
    GPL_TRY(boolean_rows(ctx, operands(lhs, pl, rhs, pr), n, cand->lhs, cand->rhs, GPL_BOOLEAN_INTERSECTION, &all, &members));
    std::unique_ptr<gpl_array, void (*)(gpl_array *)> geo(all, gpl_array_free);
    // drop the pairs whose intersection has no member (touching pairs)
    GPL_TRY(keep_nonempty_rows(ctx, cand.get(), all, members.p, pairs, out));
    geo.release();  // *out holds the reference
    return GPL_OK;
}
