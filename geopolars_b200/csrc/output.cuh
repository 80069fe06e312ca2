// output.cuh — how the C entry points return their results: row values and validity bitmaps in the caller's memory
// (`mem`), and the geometry columns they build on the device.
#pragma once

#include "common.cuh"

namespace gpl {

// abi.cu
int pack_bits(gpl_ctx *ctx, const uint8_t *bytes_dev, uint8_t *bitmap_dev, int64_t n);  // one byte per row -> Arrow LSB bitmap
int deliver(gpl_ctx *ctx, void *dst, const void *src_dev, size_t bytes, int mem);       // host: stream-ordered D2H + sync

// k_measure.cu
int centroid_raw(gpl_ctx *ctx, const gpl_array *in, double2 *out_dev, uint8_t *valid_bytes_dev);
int envelope_raw(gpl_ctx *ctx, const gpl_array *in, double *out4_dev, uint8_t *valid_bytes_dev);
int origin_table(gpl_ctx *ctx, const gpl_array *in, int origin, double2 *out_dev);

// every entry point that takes `mem` rejects any other value before it copies or launches anything
static int check_mem(int mem, const char *who) {
    GPL_REQUIRE(mem == GPL_HOST || mem == GPL_DEVICE, GPL_ERR_INVALID_ARG, "%s: mem must be GPL_HOST or GPL_DEVICE (got %d)", who, mem);
    return GPL_OK;
}

// bool result: bytes on device -> Arrow bitmap in the caller's memory
static int finish_bitmap(gpl_ctx *ctx, const uint8_t *bytes_dev, int64_t n, uint8_t *out_bitmap, int mem) {
    size_t nb = (size_t)(n + 7) / 8;
    if (mem == GPL_DEVICE) return pack_bits(ctx, bytes_dev, out_bitmap, n);
    Scratch<uint8_t> bm;
    GPL_TRY(bm.get(ctx, nb));
    GPL_TRY(pack_bits(ctx, bytes_dev, bm.p, n));
    return deliver(ctx, out_bitmap, bm.p, nb, GPL_HOST);
}

// n values the caller wants in `mem` at out: the kernel writes p (out itself for GPL_DEVICE, scratch for GPL_HOST) and
// deliver() hands them over.  out NULL: p stays NULL and nothing is delivered.
template <typename T>
struct RowOut {
    T *out = nullptr, *p = nullptr;
    int64_t n = 0;
    int mem = GPL_DEVICE;
    Scratch<T> tmp;
    int get(gpl_ctx *ctx, T *dst, int64_t rows, int where) {
        out = p = dst, n = rows, mem = where;
        if (dst && mem == GPL_HOST) {
            GPL_TRY(tmp.get(ctx, (size_t)n));
            p = tmp.p;
        }
        return GPL_OK;
    }
    int deliver(gpl_ctx *ctx) const { return out ? gpl::deliver(ctx, out, p, sizeof(T) * (size_t)n, mem) : GPL_OK; }
};

// the validity bytes of n rows, delivered as an Arrow bitmap to `bitmap` in `mem` (nothing when bitmap is NULL).  The bytes are
// allocated when a bitmap is asked for, or always (for the kernels that always write them); otherwise p stays NULL.
struct ValidOut {
    uint8_t *bitmap = nullptr, *p = nullptr;
    int64_t n = 0;
    int mem = GPL_DEVICE;
    Scratch<uint8_t> bytes;
    int get(gpl_ctx *ctx, uint8_t *dst, int64_t rows, int where, bool always) {
        bitmap = dst, n = rows, mem = where;
        if (dst || always) {
            GPL_TRY(bytes.get(ctx, (size_t)n));
            p = bytes.p;
        }
        return GPL_OK;
    }
    int deliver(gpl_ctx *ctx) const { return bitmap ? finish_bitmap(ctx, p, n, bitmap, mem) : GPL_OK; }
};

// A geometry column of n rows built on the device with 1 (MultiPoint), 2 (MultiLineString) or 3 (MultiPolygon) offset levels.
// A count pass writes each row's items of every level into count[k] (level 0: its members; the last level: its coordinates);
// scan_and_allocate() scans them into base[k] (base[0] is the column's geometry offsets, the others the rows' first ring /
// coordinate), reads the totals back and allocates the lower offset levels off[k] (part_off, then ring_off) and xy; a write
// pass fills them at the rows' bases, and finish() closes the offsets and returns the column.  k_boolean.cu.
struct RaggedOut {
    gpl_ctx *ctx = nullptr;
    int64_t n = 0;
    int levels = 0;
    Scratch<int64_t> count[3], base[3], off[2], tot;
    Scratch<double> xy;
    int64_t total[3] = {0, 0, 0};
    int init(gpl_ctx *c, int64_t rows, int nlevels);  // count, base and tot (one total per level)
    int scan_and_allocate();
    // the closing offsets, the validity bitmap of row_valid_bytes, a synchronise (the caller's scratch returns to the cache
    // after it) and the column of `type` that owns every buffer
    int finish(const uint8_t *row_valid_bytes, int type, gpl_array **out);
};

// The output of a geometry join over the candidate pairs `cand`: `all` holds one row per candidate and members[k] its member
// count.  Keeps the pairs and rows with a member (in order), every kept row valid; out shares all's buffers and holds it as
// its parent (on success it takes over the caller's reference to all).  k_boolean.cu.
int keep_nonempty_rows(gpl_ctx *ctx, const gpl_pairs *cand, gpl_array *all, const int64_t *members, gpl_pairs **pairs, gpl_array **out);

}  // namespace gpl
