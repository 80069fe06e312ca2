// abi.cu — context, caching allocator and device-array plumbing behind include/geopolars_b200.h.
// Reference boundary replaced: the Arrow C Data Interface hop of py-geopolars/src/ffi.rs:12-109 (buffers
// arrive once, are copied to HBM once with cudaMemcpyAsync, and stay resident across ops).
#include <stdarg.h>
#include <string.h>

#include "common.cuh"
#include "output.cuh"

namespace gpl {

static thread_local char g_err[1024] = "";

void set_error(const char *fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}
int cuda_fail(cudaError_t e, const char *what, const char *file, int line) {
    set_error("CUDA error %d (%s) at %s:%d: %s", (int)e, cudaGetErrorString(e), file, line, what);
    return e == cudaErrorMemoryAllocation ? GPL_ERR_OOM : GPL_ERR_CUDA;
}

gpl_array *array_new(gpl_ctx *ctx, int32_t type) {
    gpl_array *a = new gpl_array();
    a->ctx = ctx;
    a->type = type;
    return a;
}
void array_retain(gpl_array *a) {
    if (a) a->refcount++;
}

// ---- conversion kernels ------------------------------------------------------------------------
__global__ void k_interleave(const double *__restrict__ x, const double *__restrict__ y, double2 *__restrict__ out,
                             int64_t n) {
    int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (; i < n; i += stride) out[i] = make_double2(x[i], y[i]);
}
__global__ void k_widen(const int32_t *__restrict__ in, int64_t *__restrict__ out, int64_t n) {
    int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (; i < n; i += stride) out[i] = in[i];
}

// bytes (one per row) -> Arrow LSB bitmap
__global__ void k_pack_bits(const uint8_t *__restrict__ bytes, uint8_t *__restrict__ bitmap, int64_t n) {
    int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;  // output byte
    int64_t nb = (n + 7) / 8;
    if (i >= nb) return;
    uint8_t v = 0;
#pragma unroll
    for (int k = 0; k < 8; ++k) {
        int64_t j = i * 8 + k;
        if (j < n && bytes[j]) v |= (uint8_t)(1u << k);
    }
    bitmap[i] = v;
}
int pack_bits(gpl_ctx *ctx, const uint8_t *bytes_dev, uint8_t *bitmap_dev, int64_t n) {
    if (n == 0) return GPL_OK;
    int64_t nb = (n + 7) / 8;
    GPL_LAUNCH(ctx, k_pack_bits, (int)ceil_div(nb, 256), 256, 0, bytes_dev, bitmap_dev, n);
    return GPL_OK;
}

// copy a device result to the caller's buffer (host: stream-ordered D2H + sync)
int deliver(gpl_ctx *ctx, void *dst, const void *src_dev, size_t bytes, int mem) {
    if (bytes == 0) return GPL_OK;
    if (mem == GPL_HOST) {
        GPL_CUDA(cudaMemcpyAsync(dst, src_dev, bytes, cudaMemcpyDeviceToHost, ctx->stream));
        GPL_CUDA(cudaStreamSynchronize(ctx->stream));
    } else if (dst != src_dev) {
        GPL_CUDA(cudaMemcpyAsync(dst, src_dev, bytes, cudaMemcpyDeviceToDevice, ctx->stream));
    }
    return GPL_OK;
}

}  // namespace gpl

using namespace gpl;

// ---- allocator -----------------------------------------------------------------------------------
static size_t round_size(size_t b) {
    if (b < 512) return 512;
    if (b < (1u << 20)) {  // next power of two below 1 MiB
        size_t p = 512;
        while (p < b) p <<= 1;
        return p;
    }
    const size_t q = 2u << 20;  // 2 MiB granules above
    return (b + q - 1) / q * q;
}
int gpl_ctx::alloc(size_t bytes, void **out) {
    size_t sz = round_size(bytes);
    {
        std::lock_guard<std::mutex> g(mu);
        auto it = free_blocks.lower_bound(sz);
        if (it != free_blocks.end() && it->first <= sz + sz / 4 + (1u << 20)) {
            *out = it->second;
            live[it->second] = it->first;
            free_blocks.erase(it);
            return GPL_OK;
        }
    }
    void *p = nullptr;
    cudaError_t e = cudaMalloc(&p, sz);
    if (e != cudaSuccess) {
        (void)cudaGetLastError();
        trim();
        e = cudaMalloc(&p, sz);
        if (e != cudaSuccess) {
            set_error("out of device memory allocating %zu bytes (%s)", sz, cudaGetErrorString(e));
            (void)cudaGetLastError();
            return GPL_ERR_OOM;
        }
    }
    std::lock_guard<std::mutex> g(mu);
    live[p] = sz;
    bytes_reserved += sz;
    *out = p;
    return GPL_OK;
}
void gpl_ctx::release(void *p) {
    if (!p) return;
    std::lock_guard<std::mutex> g(mu);
    auto it = live.find(p);
    if (it == live.end()) return;  // not ours (borrowed)
    free_blocks.emplace(it->second, p);
    live.erase(it);
}
void gpl_ctx::trim() {
    std::lock_guard<std::mutex> g(mu);
    for (auto &kv : free_blocks) {
        cudaFree(kv.second);
        bytes_reserved -= kv.first;
    }
    free_blocks.clear();
}

// ---- context -------------------------------------------------------------------------------------
extern "C" int gpl_abi_version(void) { return GPL_ABI_VERSION; }
extern "C" const char *gpl_last_error(void) { return g_err; }

extern "C" int gpl_ctx_create(int device, void *stream, gpl_ctx **out) {
    GPL_REQUIRE(out != nullptr, GPL_ERR_INVALID_ARG, "gpl_ctx_create: out is NULL");
    int n = 0;
    cudaError_t e = cudaGetDeviceCount(&n);
    if (e != cudaSuccess || n == 0) {
        set_error("no CUDA device available (%s); libgeopolars_b200 has no CPU fallback",
                  e != cudaSuccess ? cudaGetErrorString(e) : "device count is 0");
        (void)cudaGetLastError();
        return GPL_ERR_CUDA;
    }
    GPL_REQUIRE(device >= 0 && device < n, GPL_ERR_INVALID_ARG, "device %d out of range [0,%d)", device, n);
    GPL_CUDA(cudaSetDevice(device));
    gpl_ctx *c = new gpl_ctx();
    c->device = device;
    {
        int v = 0;
        if (cudaDeviceGetAttribute(&v, cudaDevAttrMaxPersistingL2CacheSize, device) == cudaSuccess) c->l2_persist_max = (size_t)v;
        if (cudaDeviceGetAttribute(&v, cudaDevAttrMaxAccessPolicyWindowSize, device) == cudaSuccess) c->l2_window_max = (size_t)v;
        (void)cudaGetLastError();
    }
    if (stream) {
        c->stream = (cudaStream_t)stream;
    } else {
        cudaError_t se = cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking);
        if (se != cudaSuccess) {
            delete c;
            return cuda_fail(se, "cudaStreamCreateWithFlags", __FILE__, __LINE__);
        }
        c->owns_stream = true;
    }
    *out = c;
    return GPL_OK;
}
extern "C" int gpl_ctx_set_stream(gpl_ctx *ctx, void *stream) {
    GPL_REQUIRE(ctx != nullptr, GPL_ERR_INVALID_ARG, "ctx is NULL");
    GPL_CUDA(cudaSetDevice(ctx->device));
    cudaStream_t old = ctx->stream, next = nullptr;
    const bool owned_old = ctx->owns_stream;
    if (stream) {
        next = (cudaStream_t)stream;
    } else {
        GPL_CUDA(cudaStreamCreateWithFlags(&next, cudaStreamNonBlocking));
    }
    if (old && old != next) {
        // The caching allocator hands blocks back for reuse in STREAM ORDER (a Scratch block returns to the cache
        // while kernels enqueued on the old stream may still read it) and the join index skips its final
        // synchronize for the same reason: everything enqueued on the new stream must therefore run after
        // everything already enqueued on the old one.
        cudaEvent_t ev = nullptr;
        GPL_CUDA(cudaEventCreateWithFlags(&ev, cudaEventDisableTiming));
        cudaError_t e1 = cudaEventRecord(ev, old);
        cudaError_t e2 = e1 == cudaSuccess ? cudaStreamWaitEvent(next, ev, 0) : e1;
        cudaEventDestroy(ev);
        if (e2 != cudaSuccess) {
            if (!stream) cudaStreamDestroy(next);
            return cuda_fail(e2, "ordering the new stream after the old one", __FILE__, __LINE__);
        }
        // a live join index keeps its L2 access-policy window on the context stream: move it along
        if (ctx->l2_pinned) {
            cudaStreamAttrValue attr;
            if (cudaStreamGetAttribute(old, cudaStreamAttributeAccessPolicyWindow, &attr) == cudaSuccess) {
                (void)cudaStreamSetAttribute(next, cudaStreamAttributeAccessPolicyWindow, &attr);
                attr.accessPolicyWindow.num_bytes = 0;
                attr.accessPolicyWindow.hitProp = cudaAccessPropertyNormal;
                attr.accessPolicyWindow.missProp = cudaAccessPropertyNormal;
                (void)cudaStreamSetAttribute(old, cudaStreamAttributeAccessPolicyWindow, &attr);
            }
            (void)cudaGetLastError();
        }
        if (owned_old) {
            cudaStreamSynchronize(old);
            cudaStreamDestroy(old);
        }
    }
    ctx->stream = next;
    ctx->owns_stream = (stream == nullptr);
    return GPL_OK;
}
extern "C" int gpl_ctx_synchronize(gpl_ctx *ctx) {
    GPL_REQUIRE(ctx != nullptr, GPL_ERR_INVALID_ARG, "ctx is NULL");
    GPL_CUDA(cudaSetDevice(ctx->device));
    GPL_CUDA(cudaStreamSynchronize(ctx->stream));
    return GPL_OK;
}
extern "C" void gpl_ctx_destroy(gpl_ctx *ctx) {
    if (!ctx) return;
    cudaSetDevice(ctx->device);
    cudaStreamSynchronize(ctx->stream);
    ctx->trim();
    for (auto &kv : ctx->live) cudaFree(kv.first);
    if (ctx->l2_limit_saved) {  // undo the L2 carve-out a join index asked for (k_pip.cu l2_pin)
        (void)cudaCtxResetPersistingL2Cache();
        (void)cudaDeviceSetLimit(cudaLimitPersistingL2CacheSize, ctx->l2_prev_limit);
        (void)cudaGetLastError();
    }
    for (cudaEvent_t ev : ctx->kt_events) cudaEventDestroy(ev);
    if (ctx->copy_in) cudaStreamDestroy(ctx->copy_in);
    if (ctx->copy_out) cudaStreamDestroy(ctx->copy_out);
    if (ctx->owns_stream) cudaStreamDestroy(ctx->stream);
    delete ctx;
}
extern "C" int gpl_ctx_trim(gpl_ctx *ctx) {
    GPL_REQUIRE(ctx != nullptr, GPL_ERR_INVALID_ARG, "ctx is NULL");
    GPL_CUDA(cudaSetDevice(ctx->device));
    GPL_CUDA(cudaStreamSynchronize(ctx->stream));  // cached blocks may still be in use by enqueued work
    ctx->trim();
    return GPL_OK;
}
extern "C" int64_t gpl_ctx_launch_count(const gpl_ctx *ctx) { return ctx ? ctx->launches : 0; }

// ---- kernel timing (measurement aid): event pairs around the streaming join kernel's launches ------------------
bool gpl_ctx::kernel_timing_pair(cudaEvent_t *a, cudaEvent_t *b) {
    constexpr size_t kMaxPairs = 4096;
    if (kt_used + 2 > kt_events.size()) {
        if (kt_events.size() >= 2 * kMaxPairs) return false;  // not read for a long time: stop recording
        cudaEvent_t e0 = nullptr, e1 = nullptr;
        if (cudaEventCreate(&e0) != cudaSuccess || cudaEventCreate(&e1) != cudaSuccess) {
            (void)cudaGetLastError();
            if (e0) cudaEventDestroy(e0);
            return false;
        }
        kt_events.push_back(e0);
        kt_events.push_back(e1);
    }
    *a = kt_events[kt_used], *b = kt_events[kt_used + 1];
    kt_used += 2;
    return true;
}
extern "C" int gpl_ctx_kernel_timing(gpl_ctx *ctx, int enable) {
    GPL_REQUIRE(ctx != nullptr, GPL_ERR_INVALID_ARG, "ctx is NULL");
    ctx->kt_on = enable != 0;
    if (!ctx->kt_on) ctx->kt_used = 0;
    return GPL_OK;
}
extern "C" int gpl_ctx_kernel_timing_read(gpl_ctx *ctx, double *ms_total, int64_t *launches) {
    GPL_REQUIRE(ctx && ms_total && launches, GPL_ERR_INVALID_ARG, "gpl_ctx_kernel_timing_read: NULL argument");
    GPL_CUDA(cudaSetDevice(ctx->device));
    double sum = 0.0;
    for (size_t i = 0; i + 1 < ctx->kt_used; i += 2) {
        GPL_CUDA(cudaEventSynchronize(ctx->kt_events[i + 1]));
        float ms = 0.0f;
        GPL_CUDA(cudaEventElapsedTime(&ms, ctx->kt_events[i], ctx->kt_events[i + 1]));
        sum += (double)ms;
    }
    *ms_total = sum;
    *launches = (int64_t)(ctx->kt_used / 2);
    ctx->kt_used = 0;
    return GPL_OK;
}

extern "C" int gpl_host_alloc(size_t bytes, void **out) {
    GPL_REQUIRE(out != nullptr, GPL_ERR_INVALID_ARG, "out is NULL");
    GPL_CUDA(cudaMallocHost(out, bytes ? bytes : 1));
    return GPL_OK;
}
extern "C" void gpl_host_free(void *p) {
    if (p) cudaFreeHost(p);
}

// ---- arrays --------------------------------------------------------------------------------------
static int expected_levels(int type, bool *geom, bool *part, bool *ring) {
    *geom = *part = *ring = false;
    switch (type) {
    case GPL_POINT:
        return GPL_OK;
    case GPL_LINESTRING:
    case GPL_MULTIPOINT:
        *geom = true;
        return GPL_OK;
    case GPL_POLYGON:
    case GPL_MULTILINESTRING:
        *geom = *ring = true;
        return GPL_OK;
    case GPL_MULTIPOLYGON:
        *geom = *part = *ring = true;
        return GPL_OK;
    default:
        set_error("unsupported geometry type code %d", type);
        return GPL_ERR_INVALID_TYPE;
    }
}

// copy (host) or adopt (device) one offsets buffer as int64 on the device
static int take_offsets(gpl_ctx *ctx, const void *src, int64_t n, int width, int mem, const int64_t **dst, bool *own) {
    if (mem == GPL_DEVICE && width == 64) {
        *dst = static_cast<const int64_t *>(src);
        *own = false;
        return GPL_OK;
    }
    Scratch<int64_t> out;
    GPL_TRY(out.get(ctx, (size_t)n));
    if (width == 64) {
        GPL_CUDA(cudaMemcpyAsync(out.p, src, sizeof(int64_t) * n, cudaMemcpyHostToDevice, ctx->stream));
    } else {
        const int32_t *src32 = static_cast<const int32_t *>(src);
        Scratch<int32_t> tmp;
        if (mem == GPL_HOST) {
            GPL_TRY(tmp.get(ctx, (size_t)n));
            GPL_CUDA(cudaMemcpyAsync(tmp.p, src, sizeof(int32_t) * n, cudaMemcpyHostToDevice, ctx->stream));
            src32 = tmp.p;
        }
        int grid = (int)std::min<int64_t>(ceil_div(n, 256), kSMs * 8);
        GPL_LAUNCH(ctx, k_widen, grid, 256, 0, src32, out.p, n);
        // tmp returns to the cache here; stream order keeps the kernel's read valid because the cache
        // only hands blocks to work enqueued later on the same stream.
    }
    *dst = out.take();
    *own = true;
    return GPL_OK;
}

extern "C" int gpl_array_from_buffers(gpl_ctx *ctx, const gpl_buffers *b, gpl_array **out) {
    GPL_REQUIRE(ctx && b && out, GPL_ERR_INVALID_ARG, "gpl_array_from_buffers: NULL argument");
    GPL_REQUIRE(b->offset_width == 32 || b->offset_width == 64 || b->geom_type == GPL_POINT, GPL_ERR_INVALID_ARG,
                "offset_width must be 32 or 64");
    GPL_REQUIRE(b->mem == GPL_HOST || b->mem == GPL_DEVICE, GPL_ERR_INVALID_ARG, "mem must be GPL_HOST or GPL_DEVICE");
    bool need_geom, need_part, need_ring;
    GPL_TRY(expected_levels(b->geom_type, &need_geom, &need_part, &need_ring));
    GPL_REQUIRE(b->n_geoms >= 0 && b->n_coords >= 0, GPL_ERR_INVALID_ARG, "negative length");
    GPL_REQUIRE(b->n_coords == 0 || b->x != nullptr, GPL_ERR_INVALID_ARG, "coords pointer is NULL");
    GPL_REQUIRE(!need_geom || b->geom_offsets, GPL_ERR_INVALID_ARG, "geom_offsets required for this type");
    GPL_REQUIRE(!need_part || b->part_offsets, GPL_ERR_INVALID_ARG, "part_offsets required for MULTIPOLYGON");
    GPL_REQUIRE(!need_ring || b->ring_offsets, GPL_ERR_INVALID_ARG, "ring_offsets required for this type");
    if (b->geom_type == GPL_POINT)
        GPL_REQUIRE(b->n_coords == b->n_geoms, GPL_ERR_LENGTH_MISMATCH, "POINT array: n_coords (%lld) != n_geoms (%lld)",
                    (long long)b->n_coords, (long long)b->n_geoms);
    GPL_CUDA(cudaSetDevice(ctx->device));

    gpl_array *a = array_new(ctx, b->geom_type);
    a->n_geoms = b->n_geoms;
    a->n_parts = need_part ? b->n_parts : 0;
    a->n_rings = need_ring ? b->n_rings : 0;
    a->n_coords = b->n_coords;
    int rc = GPL_OK;
    auto fail = [&](int code) {
        gpl_array_free(a);
        return code;
    };
    // coordinates
    if (b->mem == GPL_DEVICE && b->y == nullptr) {
        a->xy = b->x;
    } else {
        Scratch<double> xy;
        if ((rc = xy.get(ctx, (size_t)b->n_coords * 2)) != GPL_OK) return fail(rc);
        if (b->y == nullptr) {
            cudaError_t e = cudaMemcpyAsync(xy.p, b->x, sizeof(double) * 2 * b->n_coords, cudaMemcpyHostToDevice, ctx->stream);
            if (e != cudaSuccess) return fail(cuda_fail(e, "H2D coords", __FILE__, __LINE__));
        } else {
            const double *dx = b->x, *dy = b->y;
            Scratch<double> tx, ty;
            if (b->mem == GPL_HOST) {
                if ((rc = tx.get(ctx, (size_t)b->n_coords)) != GPL_OK) return fail(rc);
                if ((rc = ty.get(ctx, (size_t)b->n_coords)) != GPL_OK) return fail(rc);
                cudaMemcpyAsync(tx.p, b->x, sizeof(double) * b->n_coords, cudaMemcpyHostToDevice, ctx->stream);
                cudaError_t e = cudaMemcpyAsync(ty.p, b->y, sizeof(double) * b->n_coords, cudaMemcpyHostToDevice, ctx->stream);
                if (e != cudaSuccess) return fail(cuda_fail(e, "H2D coords", __FILE__, __LINE__));
                dx = tx.p;
                dy = ty.p;
            }
            int grid = (int)std::max<int64_t>(1, std::min<int64_t>(ceil_div(b->n_coords, 256), kSMs * 8));
            k_interleave<<<grid, 256, 0, ctx->stream>>>(dx, dy, reinterpret_cast<double2 *>(xy.p), b->n_coords);
            ctx->launches++;
        }
        a->xy = xy.take();
        a->own_xy = true;
    }
    // offsets
    if (need_geom) {
        if ((rc = take_offsets(ctx, b->geom_offsets, b->n_geoms + 1, b->offset_width, b->mem, &a->geom_off, &a->own_geom)) != GPL_OK)
            return fail(rc);
    }
    if (need_part) {
        if ((rc = take_offsets(ctx, b->part_offsets, b->n_parts + 1, b->offset_width, b->mem, &a->part_off, &a->own_part)) != GPL_OK)
            return fail(rc);
    }
    if (need_ring) {
        if ((rc = take_offsets(ctx, b->ring_offsets, b->n_rings + 1, b->offset_width, b->mem, &a->ring_off, &a->own_ring)) != GPL_OK)
            return fail(rc);
    }
    if (b->validity) {
        if (b->mem == GPL_DEVICE) {
            a->validity = b->validity;
        } else {
            Scratch<uint8_t> v;
            size_t nb = (size_t)(b->n_geoms + 7) / 8;
            if ((rc = v.get(ctx, nb)) != GPL_OK) return fail(rc);
            cudaError_t e = cudaMemcpyAsync(v.p, b->validity, nb, cudaMemcpyHostToDevice, ctx->stream);
            if (e != cudaSuccess) return fail(cuda_fail(e, "H2D validity", __FILE__, __LINE__));
            a->validity = v.take();
            a->own_valid = true;
        }
    }
    if (b->mem == GPL_HOST) {
        // the caller may reuse its (possibly pageable) buffers as soon as we return
        cudaError_t e = cudaStreamSynchronize(ctx->stream);
        if (e != cudaSuccess) return fail(cuda_fail(e, "sync after H2D", __FILE__, __LINE__));
    }
    *out = a;
    return GPL_OK;
}

extern "C" int gpl_array_view(const gpl_array *a, gpl_device_view *v) {
    GPL_REQUIRE(a && v, GPL_ERR_INVALID_ARG, "gpl_array_view: NULL argument");
    v->geom_type = a->type;
    v->reserved = 0;
    v->n_geoms = a->n_geoms;
    v->n_parts = a->n_parts;
    v->n_rings = a->n_rings;
    v->n_coords = a->n_coords;
    v->xy = a->xy;
    v->geom_offsets = a->geom_off;
    v->part_offsets = a->part_off;
    v->ring_offsets = a->ring_off;
    v->validity = a->validity;
    return GPL_OK;
}

extern "C" int gpl_array_copy_out(gpl_ctx *ctx, const gpl_array *a, double *xy, int64_t *geom_offsets,
                                  int64_t *part_offsets, int64_t *ring_offsets, uint8_t *validity, int mem) {
    GPL_REQUIRE(ctx && a, GPL_ERR_INVALID_ARG, "gpl_array_copy_out: NULL argument");
    GPL_TRY(check_mem(mem, "gpl_array_copy_out"));
    GPL_CUDA(cudaSetDevice(ctx->device));
    cudaMemcpyKind k = mem == GPL_HOST ? cudaMemcpyDeviceToHost : cudaMemcpyDeviceToDevice;
    if (xy && a->n_coords) GPL_CUDA(cudaMemcpyAsync(xy, a->xy, sizeof(double) * 2 * a->n_coords, k, ctx->stream));
    if (geom_offsets && a->geom_off)
        GPL_CUDA(cudaMemcpyAsync(geom_offsets, a->geom_off, sizeof(int64_t) * (a->n_geoms + 1), k, ctx->stream));
    if (part_offsets && a->part_off)
        GPL_CUDA(cudaMemcpyAsync(part_offsets, a->part_off, sizeof(int64_t) * (a->n_parts + 1), k, ctx->stream));
    if (ring_offsets && a->ring_off)
        GPL_CUDA(cudaMemcpyAsync(ring_offsets, a->ring_off, sizeof(int64_t) * (a->n_rings + 1), k, ctx->stream));
    if (validity) {
        size_t nb = (size_t)(a->n_geoms + 7) / 8;
        if (a->validity) {
            GPL_CUDA(cudaMemcpyAsync(validity, a->validity, nb, k, ctx->stream));
        } else if (mem == GPL_HOST) {
            memset(validity, 0xff, nb);
        } else {
            GPL_CUDA(cudaMemsetAsync(validity, 0xff, nb, ctx->stream));
        }
    }
    if (mem == GPL_HOST) GPL_CUDA(cudaStreamSynchronize(ctx->stream));
    return GPL_OK;
}

extern "C" void gpl_array_free(gpl_array *a) {
    if (!a) return;
    if (--a->refcount > 0) return;
    gpl_ctx *c = a->ctx;
    if (a->own_xy) c->release(const_cast<double *>(a->xy));
    if (a->own_geom) c->release(const_cast<int64_t *>(a->geom_off));
    if (a->own_part) c->release(const_cast<int64_t *>(a->part_off));
    if (a->own_ring) c->release(const_cast<int64_t *>(a->ring_off));
    if (a->own_valid) c->release(const_cast<uint8_t *>(a->validity));
    gpl_array *parent = a->parent;
    delete a;
    if (parent) gpl_array_free(parent);
}
