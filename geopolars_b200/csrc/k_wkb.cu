// k_wkb.cu — WKB <-> GeoArrow on the GPU (SURVEY.md §8f rank 1).
//
// The reference decodes WKB into heap-allocated geo structs on EVERY op and encodes the result back
// (geopolars/geopolars-geo/src/util.rs:27-37 `iter_geom`, :11-24 `from_geom_vec`; README.md:83 names it as
// the dominant cost).  Here a column is decoded ONCE, on the device:
//
//   decode  k_wkb_count  one thread per row walks the row's headers and ring counts (never the coordinates):
//                        per-row coordinate / ring / part counts, the set of WKB types seen, first bad row
//           3 x scan     row starts at every nesting level; one host sync for totals + type set
//           k_wkb_fill   second walk writes ring / part offsets and copies the coordinates.  WKB payloads sit
//                        at arbitrary byte alignment (1+4(+4) header bytes): every destination double is
//                        assembled from the two aligned 8-byte words that cover it (funnel shift), so loads
//                        and stores are aligned and coalesced.  One warp per row for long rows, one thread per
//                        row for short ones (Point columns: 21 B per row).
//   encode  k_wkb_sizes  row sizes from the offsets alone; scan -> Arrow binary offsets
//           k_wkb_write  headers byte-wise by one lane, coordinate runs as aligned 8-byte stores assembled
//                        from the (aligned) source doubles, head / tail bytes of a run byte-wise.
// Accepted input: ISO WKB XY Point..MultiPolygon, either byte order, EWKB SRID flag tolerated, Z/M rejected —
// the same contract as the host parser this file replaces.  A column may mix single and multi rows of one
// family (Polygon + MultiPolygon -> MULTIPOLYGON), like geopandas/pyogrio hand-offs do.
// HBM-bound by design: the payload is read once by the fill pass (+ the sparse header reads of the count pass).
#include <limits.h>

#include "common.cuh"
#include "output.cuh"
#include "scan.cuh"

namespace gpl {

struct Cur {
    const uint8_t *p, *end;
    bool le, ok;
};
__device__ __forceinline__ uint8_t rd_u8(Cur &c) {
    if (c.end - c.p < 1) {
        c.ok = false;
        return 0;
    }
    return *c.p++;
}
__device__ __forceinline__ uint32_t rd_u32(Cur &c) {
    if (c.end - c.p < 4) {
        c.ok = false;
        return 0;
    }
    const uint32_t b0 = c.p[0], b1 = c.p[1], b2 = c.p[2], b3 = c.p[3];
    c.p += 4;
    return c.le ? (b0 | (b1 << 8) | (b2 << 16) | (b3 << 24)) : (b3 | (b2 << 8) | (b1 << 16) | (b0 << 24));
}
__device__ __forceinline__ void rd_skip(Cur &c, uint64_t nbytes) {
    if ((uint64_t)(c.end - c.p) < nbytes) c.ok = false;
    else c.p += nbytes;
}
// geometry header: byte order + type (ISO codes 1..6; EWKB SRID flag tolerated; Z/M rejected) -> 1..6 or -1
__device__ __forceinline__ int rd_header(Cur &c) {
    c.le = rd_u8(c) != 0;
    uint32_t t = rd_u32(c);
    if (t & 0x20000000u) (void)rd_u32(c);
    if (t & 0xC0000000u) return -1;
    t &= 0x0fffffffu;
    if (t < 1 || t > 6) return -1;
    return c.ok ? (int)t : -1;
}
__device__ __forceinline__ int wkb_code(int t) {  // WKB type -> GeometryType code (enums.py:4-15)
    return t == 1 ? GPL_POINT : t == 2 ? GPL_LINESTRING : t == 3 ? GPL_POLYGON : t == 4 ? GPL_MULTIPOINT : t == 5 ? GPL_MULTILINESTRING : GPL_MULTIPOLYGON;
}

// unaligned little-endian 8-byte load assembled from aligned words.  The second word is touched only when
// it holds at least one byte of the value, so the read never leaves the 8-byte word of a valid byte.
__device__ __forceinline__ uint64_t ld_u64_unaligned(const uint8_t *p) {
    const uintptr_t a = reinterpret_cast<uintptr_t>(p);
    const uint64_t *base = reinterpret_cast<const uint64_t *>(a & ~(uintptr_t)7);
    const unsigned sh = (unsigned)(a & 7) * 8;
    const uint64_t lo = __ldg(base);
    if (sh == 0) return lo;
    const uint64_t hi = __ldg(base + 1);
    return (lo >> sh) | (hi << (64 - sh));
}
__device__ __forceinline__ uint64_t bswap64(uint64_t v) {
    const uint32_t lo = (uint32_t)v, hi = (uint32_t)(v >> 32);
    return ((uint64_t)__byte_perm(lo, 0, 0x0123) << 32) | __byte_perm(hi, 0, 0x0123);
}

struct RowCounts {
    int64_t c, r, q;
};
// polygon body (after its header): ring count, then per ring a point count and the points
__device__ __forceinline__ void count_polygon(Cur &c, RowCounts &k) {
    const uint32_t nr = rd_u32(c);
    for (uint32_t i = 0; i < nr && c.ok; ++i) {
        const uint32_t np = rd_u32(c);
        rd_skip(c, 16ull * np);
        k.c += np;
    }
    k.r += nr;
}

template <typename Off>
__global__ void __launch_bounds__(256) k_wkb_count(int64_t n, const uint8_t *__restrict__ bytes, const Off *__restrict__ off,
                                                   const uint8_t *__restrict__ valid, int64_t total_bytes, int32_t *__restrict__ cc,
                                                   int32_t *__restrict__ rr, int32_t *__restrict__ qq, uint8_t *__restrict__ row_valid,
                                                   unsigned *__restrict__ seen, unsigned long long *__restrict__ bad_row) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int64_t b0 = (int64_t)off[i] - (int64_t)off[0], b1 = (int64_t)off[i + 1] - (int64_t)off[0];
    RowCounts k{0, 0, 0};
    if (b0 < 0 || b1 < b0 || b1 > total_bytes) {  // offsets must be monotone and inside the payload: never read outside it
        atomicMin(bad_row, (unsigned long long)i);
        cc[i] = rr[i] = qq[i] = 0;
        row_valid[i] = 0;
        return;
    }
    bool isnull = !bit_get(valid, i) || b1 - b0 < 5;
    if (!isnull) {
        Cur c{bytes + b0, bytes + b1, true, true};
        const int t = rd_header(c);
        bool good = t > 0;
        if (good) {
            switch (t) {
            case 1:
                rd_skip(c, 16);
                k.c = 1;
                break;
            case 2: {
                const uint32_t np = rd_u32(c);
                rd_skip(c, 16ull * np);
                k.c = np, k.r = 1;
                break;
            }
            case 3:
                count_polygon(c, k);
                k.q = 1;
                break;
            case 4: {
                const uint32_t m = rd_u32(c);
                for (uint32_t j = 0; j < m && c.ok; ++j) {
                    if (rd_header(c) != 1) c.ok = false;
                    rd_skip(c, 16);
                }
                k.c = m;
                break;
            }
            case 5: {
                const uint32_t m = rd_u32(c);
                for (uint32_t j = 0; j < m && c.ok; ++j) {
                    if (rd_header(c) != 2) c.ok = false;
                    const uint32_t np = rd_u32(c);
                    rd_skip(c, 16ull * np);
                    k.c += np;
                }
                k.r = m;
                break;
            }
            default: {
                const uint32_t m = rd_u32(c);
                for (uint32_t j = 0; j < m && c.ok; ++j) {
                    if (rd_header(c) != 3) c.ok = false;
                    count_polygon(c, k);
                }
                k.q = m;
                break;
            }
            }
            good = c.ok && k.c < INT_MAX && k.r < INT_MAX;
        }
        if (!good) {
            atomicMin(bad_row, (unsigned long long)i);
            k = RowCounts{0, 0, 0};
            isnull = true;
        } else {
            atomicOr(seen, 1u << wkb_code(t));
        }
    }
    cc[i] = (int32_t)k.c, rr[i] = (int32_t)k.r, qq[i] = (int32_t)k.q;
    row_valid[i] = isnull ? 0 : 1;
}

// copy `cnt` points from the WKB payload at `src` to xy[dst..): destination words are aligned
__device__ __forceinline__ void copy_points(double *__restrict__ xy, int64_t dst, const uint8_t *src, uint32_t cnt, bool le, int lane,
                                            int step) {
    uint64_t *o = reinterpret_cast<uint64_t *>(xy) + 2 * dst;
    const int64_t words = 2 * (int64_t)cnt;
    for (int64_t j = lane; j < words; j += step) {
        uint64_t v = ld_u64_unaligned(src + 8 * j);
        o[j] = le ? v : bswap64(v);
    }
}

struct FillOut {
    double *xy;
    int64_t *ring_off, *part_off;  // may be NULL when the target type has no such level
};
__device__ __forceinline__ void fill_polygon(Cur &c, const FillOut &o, int64_t &ci, int64_t &ri, int lane, int step) {
    const uint32_t nr = rd_u32(c);
    for (uint32_t i = 0; i < nr; ++i) {
        const uint32_t np = rd_u32(c);
        if (lane == 0) o.ring_off[ri] = ci;
        copy_points(o.xy, ci, c.p, np, c.le, lane, step);
        c.p += 16ull * np;
        ci += np, ri += 1;
    }
}

// WARP: one warp per row (lanes share the walk, split the copies); else one thread per row
template <typename Off, bool WARP>
__global__ void __launch_bounds__(256) k_wkb_fill(int64_t n, int target, const uint8_t *__restrict__ bytes, const Off *__restrict__ off,
                                                  const uint8_t *__restrict__ row_valid, const int64_t *__restrict__ cs,
                                                  const int64_t *__restrict__ rs, const int64_t *__restrict__ qs, FillOut o) {
    const int lane = WARP ? (threadIdx.x & 31) : 0, step = WARP ? 32 : 1;
    const int64_t tid = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    const int64_t first = WARP ? (tid >> 5) : tid, stride = WARP ? (((int64_t)gridDim.x * blockDim.x) >> 5) : (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = first; i < n; i += stride) {
        if (!row_valid[i]) {
            if (target == GPL_POINT && lane == 0) o.xy[2 * i] = o.xy[2 * i + 1] = nan("");
            continue;
        }
        const int64_t b0 = (int64_t)off[i] - (int64_t)off[0], b1 = (int64_t)off[i + 1] - (int64_t)off[0];
        Cur c{bytes + b0, bytes + b1, true, true};  // validated by k_wkb_count: no bounds checks needed below
        const int t = rd_header(c);
        int64_t ci = target == GPL_POINT ? i : cs[i], ri = rs[i], qi = qs[i];
        switch (t) {
        case 1:
            copy_points(o.xy, ci, c.p, 1, c.le, lane, step);
            break;
        case 2: {
            const uint32_t np = rd_u32(c);
            if (target == GPL_MULTILINESTRING && lane == 0) o.ring_off[ri] = ci;
            copy_points(o.xy, ci, c.p, np, c.le, lane, step);
            break;
        }
        case 3:
            if (target == GPL_MULTIPOLYGON && lane == 0) o.part_off[qi] = ri;
            fill_polygon(c, o, ci, ri, lane, step);
            break;
        case 4: {
            const uint32_t m = rd_u32(c);
            for (uint32_t j = 0; j < m; ++j) {
                (void)rd_header(c);
                copy_points(o.xy, ci + j, c.p, 1, c.le, lane, step);
                c.p += 16;
            }
            break;
        }
        case 5: {
            const uint32_t m = rd_u32(c);
            for (uint32_t j = 0; j < m; ++j) {
                (void)rd_header(c);
                const uint32_t np = rd_u32(c);
                if (lane == 0) o.ring_off[ri] = ci;
                copy_points(o.xy, ci, c.p, np, c.le, lane, step);
                c.p += 16ull * np;
                ci += np, ri += 1;
            }
            break;
        }
        default: {
            const uint32_t m = rd_u32(c);
            for (uint32_t j = 0; j < m; ++j) {
                (void)rd_header(c);
                if (lane == 0) o.part_off[qi] = ri;
                fill_polygon(c, o, ci, ri, lane, step);
                qi += 1;
            }
            break;
        }
        }
    }
}

__global__ void k_wkb_close(int64_t *ring_off, int64_t n_rings, int64_t n_coords, int64_t *part_off, int64_t n_parts) {
    if (ring_off) ring_off[n_rings] = n_coords;
    if (part_off) part_off[n_parts] = n_rings;
}

// ---- encode ------------------------------------------------------------------------------------------
struct Src {
    int type;
    const double *xy;
    const int64_t *go, *po, *ro;
    const uint8_t *valid;
};
__device__ __forceinline__ int64_t polygon_bytes(const Src &s, int64_t r0, int64_t r1) {
    return 4 + 4 * (r1 - r0) + 16 * (s.ro[r1] - s.ro[r0]);
}
__global__ void __launch_bounds__(256) k_wkb_sizes(int64_t n, Src s, int64_t *__restrict__ size) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= n) return;
    int64_t b = 0;
    if (bit_get(s.valid, i)) {
        switch (s.type) {
        case GPL_POINT: b = 21; break;
        case GPL_LINESTRING: b = 9 + 16 * (s.go[i + 1] - s.go[i]); break;
        case GPL_POLYGON: b = 5 + polygon_bytes(s, s.go[i], s.go[i + 1]); break;
        case GPL_MULTIPOINT: b = 9 + 21 * (s.go[i + 1] - s.go[i]); break;
        case GPL_MULTILINESTRING: b = 9 + 9 * (s.go[i + 1] - s.go[i]) + 16 * (s.ro[s.go[i + 1]] - s.ro[s.go[i]]); break;
        default:
            b = 9;
            for (int64_t q = s.go[i]; q < s.go[i + 1]; ++q) b += 5 + polygon_bytes(s, s.po[q], s.po[q + 1]);
            break;
        }
    }
    size[i] = b;
}

__device__ __forceinline__ void put_u32(uint8_t *p, uint32_t v) { p[0] = (uint8_t)v, p[1] = (uint8_t)(v >> 8), p[2] = (uint8_t)(v >> 16), p[3] = (uint8_t)(v >> 24); }
__device__ __forceinline__ void put_head(uint8_t *&p, uint32_t type, int lane) {  // byte order 1 (little endian) + type
    if (lane == 0) {
        p[0] = 1;
        put_u32(p + 1, type);
    }
    p += 5;
}
__device__ __forceinline__ void put_count(uint8_t *&p, uint32_t v, int lane) {
    if (lane == 0) put_u32(p, v);
    p += 4;
}
// a run of `cnt` points from xy[c0..) to the (unaligned) byte address p
__device__ __forceinline__ void put_points(uint8_t *&p, const double *__restrict__ xy, int64_t c0, int64_t cnt, int lane, int step) {
    const uint64_t *S = reinterpret_cast<const uint64_t *>(xy) + 2 * c0;
    const int64_t words = 2 * cnt;
    const unsigned head = (unsigned)((8 - (reinterpret_cast<uintptr_t>(p) & 7)) & 7);
    if (words > 0) {
        if (head == 0) {
            uint64_t *D = reinterpret_cast<uint64_t *>(p);
            for (int64_t k = lane; k < words; k += step) D[k] = S[k];
        } else {
            const unsigned sh = head * 8;
            for (unsigned b = lane; b < head; b += step) p[b] = (uint8_t)(S[0] >> (8 * b));  // bytes up to the first aligned word
            uint64_t *D = reinterpret_cast<uint64_t *>(p + head);
            for (int64_t k = lane; k < words - 1; k += step) D[k] = (S[k] >> sh) | (S[k + 1] << (64 - sh));
            uint8_t *tail = p + head + 8 * (words - 1);
            const uint64_t last = S[words - 1] >> sh;
            for (unsigned b = lane; b < 8 - head; b += step) tail[b] = (uint8_t)(last >> (8 * b));
        }
    }
    p += 8 * words;
}
__device__ __forceinline__ void put_polygon(uint8_t *&p, const Src &s, int64_t r0, int64_t r1, int lane, int step) {
    put_count(p, (uint32_t)(r1 - r0), lane);
    for (int64_t r = r0; r < r1; ++r) {
        put_count(p, (uint32_t)(s.ro[r + 1] - s.ro[r]), lane);
        put_points(p, s.xy, s.ro[r], s.ro[r + 1] - s.ro[r], lane, step);
    }
}
template <bool WARP>
__global__ void __launch_bounds__(256) k_wkb_write(int64_t n, Src s, const int64_t *__restrict__ boff, uint8_t *__restrict__ out) {
    const int lane = WARP ? (threadIdx.x & 31) : 0, step = WARP ? 32 : 1;
    const int64_t tid = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    const int64_t first = WARP ? (tid >> 5) : tid, stride = WARP ? (((int64_t)gridDim.x * blockDim.x) >> 5) : (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = first; i < n; i += stride) {
        if (boff[i + 1] == boff[i]) continue;  // null row
        uint8_t *p = out + boff[i];
        switch (s.type) {
        case GPL_POINT:
            put_head(p, 1, lane);
            put_points(p, s.xy, i, 1, lane, step);
            break;
        case GPL_LINESTRING:
            put_head(p, 2, lane);
            put_count(p, (uint32_t)(s.go[i + 1] - s.go[i]), lane);
            put_points(p, s.xy, s.go[i], s.go[i + 1] - s.go[i], lane, step);
            break;
        case GPL_POLYGON:
            put_head(p, 3, lane);
            put_polygon(p, s, s.go[i], s.go[i + 1], lane, step);
            break;
        case GPL_MULTIPOINT:
            put_head(p, 4, lane);
            put_count(p, (uint32_t)(s.go[i + 1] - s.go[i]), lane);
            for (int64_t c = s.go[i]; c < s.go[i + 1]; ++c) {
                put_head(p, 1, lane);
                put_points(p, s.xy, c, 1, lane, step);
            }
            break;
        case GPL_MULTILINESTRING:
            put_head(p, 5, lane);
            put_count(p, (uint32_t)(s.go[i + 1] - s.go[i]), lane);
            for (int64_t l = s.go[i]; l < s.go[i + 1]; ++l) {
                put_head(p, 2, lane);
                put_count(p, (uint32_t)(s.ro[l + 1] - s.ro[l]), lane);
                put_points(p, s.xy, s.ro[l], s.ro[l + 1] - s.ro[l], lane, step);
            }
            break;
        default:
            put_head(p, 6, lane);
            put_count(p, (uint32_t)(s.go[i + 1] - s.go[i]), lane);
            for (int64_t q = s.go[i]; q < s.go[i + 1]; ++q) {
                put_head(p, 3, lane);
                put_polygon(p, s, s.po[q], s.po[q + 1], lane, step);
            }
            break;
        }
    }
}
__global__ void k_narrow_offsets(int64_t n, const int64_t *__restrict__ in, int32_t *__restrict__ out) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i < n) out[i] = (int32_t)in[i];
}
__global__ void k_valid_bytes_from_bitmap(int64_t n, const uint8_t *__restrict__ bm, uint8_t *__restrict__ bytes) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i < n) bytes[i] = bit_get(bm, i) ? 1 : 0;
}

static int stream_grid(int64_t rows, bool warp) {
    const int64_t want = warp ? ceil_div(rows, 8) : ceil_div(rows, 256);
    return (int)std::max<int64_t>(1, std::min<int64_t>(want, (int64_t)kSMs * 16));
}

template <typename Off>
static int decode(gpl_ctx *ctx, const uint8_t *bytes_d, const Off *off_d, const uint8_t *valid_d, int64_t n, int64_t total_bytes,
                  gpl_array **out) {
    Scratch<int32_t> cc, rr, qq;
    Scratch<uint8_t> rv;
    Scratch<int64_t> cs, rs, qs, meta;
    GPL_TRY(cc.get(ctx, (size_t)n));
    GPL_TRY(rr.get(ctx, (size_t)n));
    GPL_TRY(qq.get(ctx, (size_t)n));
    GPL_TRY(rv.get(ctx, (size_t)n));
    GPL_TRY(cs.get(ctx, (size_t)n + 1));
    GPL_TRY(rs.get(ctx, (size_t)n + 1));
    GPL_TRY(qs.get(ctx, (size_t)n + 1));
    GPL_TRY(meta.get(ctx, 8));  // [0] seen (unsigned) [1] first bad row [2..4] totals c, r, q
    int64_t h_meta[5] = {0, -1, 0, 0, 0};
    h_meta[1] = (int64_t)ULLONG_MAX;
    GPL_CUDA(cudaMemcpyAsync(meta.p, h_meta, sizeof(h_meta), cudaMemcpyHostToDevice, ctx->stream));
    if (n > 0)
        GPL_LAUNCH(ctx, (k_wkb_count<Off>), (int)ceil_div(n, 256), 256, 0, n, bytes_d, off_d, valid_d, total_bytes, cc.p, rr.p, qq.p, rv.p,
                   reinterpret_cast<unsigned *>(meta.p), reinterpret_cast<unsigned long long *>(meta.p + 1));
    GPL_TRY((exclusive_scan<int32_t, int64_t>(ctx, cc.p, n, cs.p, meta.p + 2)));
    GPL_TRY((exclusive_scan<int32_t, int64_t>(ctx, rr.p, n, rs.p, meta.p + 3)));
    GPL_TRY((exclusive_scan<int32_t, int64_t>(ctx, qq.p, n, qs.p, meta.p + 4)));
    GPL_CUDA(cudaMemcpyAsync(h_meta, meta.p, sizeof(h_meta), cudaMemcpyDeviceToHost, ctx->stream));
    GPL_CUDA(cudaStreamSynchronize(ctx->stream));
    GPL_REQUIRE((unsigned long long)h_meta[1] == ULLONG_MAX, GPL_ERR_INVALID_ARG,
                "row %lld: truncated, malformed or unsupported WKB (XY Point..MultiPolygon only), or offsets out of order",
                (long long)h_meta[1]);
    const unsigned seen = (unsigned)(h_meta[0] & 0xffffffffu);
    auto has = [&](int code) { return (seen >> code) & 1u; };
    const bool pt = has(GPL_POINT) || has(GPL_MULTIPOINT), ls = has(GPL_LINESTRING) || has(GPL_MULTILINESTRING),
               pg = has(GPL_POLYGON) || has(GPL_MULTIPOLYGON);
    GPL_REQUIRE((int)pt + (int)ls + (int)pg <= 1, GPL_ERR_INVALID_TYPE,
                "Expected a single geometry family per column (found a mix of point/line/polygon rows)");
    int target = GPL_POINT;
    if (pg) target = has(GPL_MULTIPOLYGON) ? GPL_MULTIPOLYGON : GPL_POLYGON;
    else if (ls) target = has(GPL_MULTILINESTRING) ? GPL_MULTILINESTRING : GPL_LINESTRING;
    else target = has(GPL_MULTIPOINT) ? GPL_MULTIPOINT : GPL_POINT;
    const int64_t C = target == GPL_POINT ? n : h_meta[2], R = h_meta[3], Q = h_meta[4];
    const bool has_ring = target == GPL_POLYGON || target == GPL_MULTILINESTRING || target == GPL_MULTIPOLYGON;
    const bool has_part = target == GPL_MULTIPOLYGON;

    Scratch<double> xy;
    Scratch<int64_t> ring, part;
    Scratch<uint8_t> bitmap;
    GPL_TRY(xy.get(ctx, (size_t)C * 2));
    if (has_ring) GPL_TRY(ring.get(ctx, (size_t)R + 1));
    if (has_part) GPL_TRY(part.get(ctx, (size_t)Q + 1));
    if (n > 0) {
        FillOut fo{xy.p, ring.p, part.p};
        const bool warp = total_bytes / n > 96;  // long rows: lanes split the coordinate copies
        if (warp)
            GPL_LAUNCH(ctx, (k_wkb_fill<Off, true>), stream_grid(n, true), 256, 0, n, target, bytes_d, off_d, rv.p, cs.p, rs.p, qs.p, fo);
        else
            GPL_LAUNCH(ctx, (k_wkb_fill<Off, false>), stream_grid(n, false), 256, 0, n, target, bytes_d, off_d, rv.p, cs.p, rs.p, qs.p, fo);
    }
    if (has_ring) GPL_LAUNCH(ctx, k_wkb_close, 1, 1, 0, ring.p, R, C, part.p, Q);
    // validity bitmap only when a null row exists
    Scratch<int64_t> nvalid;
    GPL_TRY(nvalid.get(ctx, (size_t)n + 2));
    int64_t h_valid = n;
    if (n > 0) {
        GPL_TRY((exclusive_scan<uint8_t, int64_t>(ctx, rv.p, n, nvalid.p, nullptr)));
        GPL_CUDA(cudaMemcpyAsync(&h_valid, nvalid.p + n, sizeof(int64_t), cudaMemcpyDeviceToHost, ctx->stream));
        GPL_CUDA(cudaStreamSynchronize(ctx->stream));
    }
    if (h_valid != n) {
        GPL_TRY(bitmap.get(ctx, (size_t)(n + 7) / 8));
        GPL_TRY(pack_bits(ctx, rv.p, bitmap.p, n));
    }
    gpl_array *o = array_new(ctx, target);
    o->n_geoms = n, o->n_coords = C;
    o->n_rings = has_ring ? R : 0, o->n_parts = has_part ? Q : 0;
    o->xy = xy.take(), o->own_xy = true;
    if (target == GPL_LINESTRING || target == GPL_MULTIPOINT) o->geom_off = cs.take(), o->own_geom = true;
    else if (target == GPL_POLYGON || target == GPL_MULTILINESTRING) o->geom_off = rs.take(), o->own_geom = true;
    else if (target == GPL_MULTIPOLYGON) o->geom_off = qs.take(), o->own_geom = true;
    if (has_ring) o->ring_off = ring.take(), o->own_ring = true;
    if (has_part) o->part_off = part.take(), o->own_part = true;
    if (bitmap.p) o->validity = bitmap.take(), o->own_valid = true;
    *out = o;
    return GPL_OK;
}

}  // namespace gpl

using namespace gpl;

extern "C" int gpl_wkb_decode(gpl_ctx *ctx, const uint8_t *bytes, const void *offsets, int offset_width, const uint8_t *validity,
                              int64_t n, int mem, gpl_array **out) {
    GPL_REQUIRE(ctx && out && n >= 0 && (n == 0 || (bytes && offsets)), GPL_ERR_INVALID_ARG, "gpl_wkb_decode: NULL argument");
    GPL_TRY(check_mem(mem, "gpl_wkb_decode"));
    GPL_REQUIRE(offset_width == 32 || offset_width == 64, GPL_ERR_INVALID_ARG, "gpl_wkb_decode: offset_width must be 32 or 64");
    GPL_CUDA(cudaSetDevice(ctx->device));
    const size_t ow = (size_t)offset_width / 8;
    // first / last offset: the payload range (a sliced Arrow array need not start at 0)
    int64_t o_first = 0, o_last = 0;
    if (n > 0) {
        uint8_t ends[16];
        if (mem == GPL_HOST) {
            memcpy(ends, offsets, ow);
            memcpy(ends + 8, static_cast<const uint8_t *>(offsets) + ow * (size_t)n, ow);
        } else {
            GPL_CUDA(cudaMemcpyAsync(ends, offsets, ow, cudaMemcpyDeviceToHost, ctx->stream));
            GPL_CUDA(cudaMemcpyAsync(ends + 8, static_cast<const uint8_t *>(offsets) + ow * (size_t)n, ow, cudaMemcpyDeviceToHost, ctx->stream));
            GPL_CUDA(cudaStreamSynchronize(ctx->stream));
        }
        if (offset_width == 32) {
            int32_t a, b;
            memcpy(&a, ends, 4), memcpy(&b, ends + 8, 4);
            o_first = a, o_last = b;
        } else {
            memcpy(&o_first, ends, 8), memcpy(&o_last, ends + 8, 8);
        }
    }
    GPL_REQUIRE(o_last >= o_first, GPL_ERR_INVALID_ARG, "gpl_wkb_decode: offsets are not monotone");
    const int64_t total = o_last - o_first;
    Scratch<uint8_t> bytes_d, valid_d, off_d;
    const uint8_t *bp = bytes ? bytes + o_first : nullptr;
    const void *op = offsets;
    const uint8_t *vp = validity;
    if (mem == GPL_HOST && n > 0) {
        GPL_TRY(bytes_d.get(ctx, (size_t)total + 16));  // + slack: the funnel-shift loads read whole aligned words
        GPL_TRY(off_d.get(ctx, ow * ((size_t)n + 1)));
        if (total > 0) GPL_CUDA(cudaMemcpyAsync(bytes_d.p, bp, (size_t)total, cudaMemcpyHostToDevice, ctx->stream));
        GPL_CUDA(cudaMemcpyAsync(off_d.p, offsets, ow * ((size_t)n + 1), cudaMemcpyHostToDevice, ctx->stream));
        bp = bytes_d.p, op = off_d.p;
        if (validity) {
            GPL_TRY(valid_d.get(ctx, (size_t)(n + 7) / 8));
            GPL_CUDA(cudaMemcpyAsync(valid_d.p, validity, (size_t)(n + 7) / 8, cudaMemcpyHostToDevice, ctx->stream));
            vp = valid_d.p;
        }
    }
    if (offset_width == 32) return decode<int32_t>(ctx, bp, static_cast<const int32_t *>(op), vp, n, total, out);
    return decode<int64_t>(ctx, bp, static_cast<const int64_t *>(op), vp, n, total, out);
}

extern "C" int gpl_wkb_encode(gpl_ctx *ctx, const gpl_array *a, void *offsets, int offset_width, uint8_t *bytes, int64_t *n_bytes,
                              int mem) {
    GPL_REQUIRE(ctx && a && offsets && n_bytes, GPL_ERR_INVALID_ARG, "gpl_wkb_encode: NULL argument");
    GPL_TRY(check_mem(mem, "gpl_wkb_encode"));
    GPL_REQUIRE(offset_width == 32 || offset_width == 64, GPL_ERR_INVALID_ARG, "gpl_wkb_encode: offset_width must be 32 or 64");
    GPL_REQUIRE(known_type(a->type), GPL_ERR_INVALID_TYPE,
                "cannot encode geometry type %d as WKB", a->type);
    GPL_CUDA(cudaSetDevice(ctx->device));
    const int64_t n = a->n_geoms;
    Src s{a->type, a->xy, a->geom_off, a->part_off, a->ring_off, a->validity};
    Scratch<int64_t> size, boff, total;
    GPL_TRY(size.get(ctx, (size_t)n + 1));
    GPL_TRY(boff.get(ctx, (size_t)n + 1));
    GPL_TRY(total.get(ctx, 1));
    if (n > 0) GPL_LAUNCH(ctx, k_wkb_sizes, (int)ceil_div(n, 256), 256, 0, n, s, size.p);
    GPL_TRY((exclusive_scan<int64_t, int64_t>(ctx, size.p, n, boff.p, total.p)));
    int64_t h_total = 0;
    GPL_CUDA(cudaMemcpyAsync(&h_total, total.p, sizeof(int64_t), cudaMemcpyDeviceToHost, ctx->stream));
    GPL_CUDA(cudaStreamSynchronize(ctx->stream));
    GPL_REQUIRE(offset_width == 64 || h_total < (1LL << 31), GPL_ERR_UNSUPPORTED,
                "WKB column needs %lld bytes: use 64-bit offsets (large_binary)", (long long)h_total);
    if (offset_width == 64) {
        GPL_TRY(deliver(ctx, offsets, boff.p, sizeof(int64_t) * ((size_t)n + 1), mem));
    } else {
        Scratch<int32_t> o32;
        GPL_TRY(o32.get(ctx, (size_t)n + 1));
        GPL_LAUNCH(ctx, k_narrow_offsets, (int)ceil_div(n + 1, 256), 256, 0, n + 1, boff.p, o32.p);
        GPL_TRY(deliver(ctx, offsets, o32.p, sizeof(int32_t) * ((size_t)n + 1), mem));
    }
    if (bytes) {
        GPL_REQUIRE(*n_bytes >= h_total, GPL_ERR_INVALID_ARG, "WKB buffer too small: need %lld bytes", (long long)h_total);
        if (n > 0 && h_total > 0) {
            Scratch<uint8_t> tmp;
            uint8_t *dst = bytes;
            if (mem == GPL_HOST) {
                GPL_TRY(tmp.get(ctx, (size_t)h_total + 8));
                dst = tmp.p;
            }
            // the aligned-word stores assume nothing about `dst`'s own alignment: head / tail bytes are byte stores
            const bool warp = h_total / n > 96;
            if (warp) GPL_LAUNCH(ctx, k_wkb_write<true>, stream_grid(n, true), 256, 0, n, s, boff.p, dst);
            else GPL_LAUNCH(ctx, k_wkb_write<false>, stream_grid(n, false), 256, 0, n, s, boff.p, dst);
            if (mem == GPL_HOST) GPL_TRY(deliver(ctx, bytes, tmp.p, (size_t)h_total, GPL_HOST));
        }
    }
    *n_bytes = h_total;
    return GPL_OK;
}

// host-buffer forms kept for the existing callers (Arrow `binary` columns: int32 offsets)
extern "C" int gpl_array_from_wkb(gpl_ctx *ctx, const uint8_t *bytes, const int32_t *offsets, const uint8_t *validity, int64_t n,
                                  gpl_array **out) {
    return gpl_wkb_decode(ctx, bytes, offsets, 32, validity, n, GPL_HOST, out);
}
extern "C" int gpl_array_to_wkb(gpl_ctx *ctx, const gpl_array *a, int32_t *offsets, uint8_t *bytes, int64_t *n_bytes) {
    return gpl_wkb_encode(ctx, a, offsets, 32, bytes, n_bytes, GPL_HOST);
}
