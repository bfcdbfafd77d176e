// runtime.cu — device context, stream-ordered memory pool, pinned-host cache, per-kernel launch
// accounting, and the bl_column <-> device-column transfer (pinned DMA, chunk concatenation,
// bitmap bit-offset normalisation).
#include <time.h>

#include <algorithm>
#include <cstdlib>
#include <map>
#include <unordered_map>

#include "common.cuh"
#include "dev_utils.cuh"

namespace plb {

static Context* g_ctx = nullptr;
static std::mutex g_init_mu;
static std::unordered_map<void*, size_t> g_pinned_sizes;           // live pinned allocations
static std::multimap<size_t, void*> g_pinned_free;                 // cache: size class -> buffer
static size_t g_pinned_cached = 0;
static const size_t kPinnedCacheMax = (size_t)24 << 30;

void ensure_init(int device) {
    std::lock_guard<std::mutex> lk(g_init_mu);
    if (g_ctx) return;
    int n = 0;
    cudaError_t e = cudaGetDeviceCount(&n);
    if (e != cudaSuccess || n == 0)
        fail(BL_ERR_CUDA, std::string("no CUDA device available: ") + (e == cudaSuccess ? "device count is 0" : cudaGetErrorString(e)) +
                              " — libpolars_b200 has no CPU fallback");
    if (device < 0) {
        const char* lr = getenv("LOCAL_RANK");
        if (lr) device = atoi(lr) % n;
        else PLB_CUDA(cudaGetDevice(&device));
    }
    PLB_REQUIRE(device < n, BL_ERR_INVALID, "device index out of range");
    PLB_CUDA(cudaSetDevice(device));
    auto* c = new Context();
    c->device = device;
    PLB_CUDA(cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking));
    PLB_CUDA(cudaStreamCreateWithFlags(&c->copy_stream, cudaStreamNonBlocking));
    cudaDeviceProp prop;
    PLB_CUDA(cudaGetDeviceProperties(&prop, device));
    c->sm_count = prop.multiProcessorCount;
    c->l2_bytes = prop.l2CacheSize;
    // keep freed blocks in the pool: allocation cost must not show up in steady state
    cudaMemPool_t pool;
    PLB_CUDA(cudaDeviceGetDefaultMemPool(&pool, device));
    uint64_t thr = UINT64_MAX;
    PLB_CUDA(cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &thr));
    // L2 fetch granularity (cudaLimitMaxL2FetchGranularity, default 64 B): the random-access kernels (hashed join probe, gather
    // from HBM) move ~100 B of DRAM per 8..32-byte access (ncu: 10.1 GB for 1e8 probes); BL_L2_FETCH=32 asks for sector-sized fetches
    { const char* g = getenv("BL_L2_FETCH"); if (g && atoi(g) >= 16 && atoi(g) <= 128) PLB_CUDA(cudaDeviceSetLimit(cudaLimitMaxL2FetchGranularity, (size_t)atoi(g))); }
    { const char* d = getenv("BL_DETERMINISTIC"); c->deterministic = d != nullptr && d[0] != '\0' && d[0] != '0'; }
    g_ctx = c;
}

Context& ctx() {
    if (!g_ctx) ensure_init(-1);
    // worker threads of the caller (Rayon) may not have the device current
    cudaSetDevice(g_ctx->device);
    return *g_ctx;
}

int Context::stat_index(const char* name) {
    for (size_t i = 0; i < stats.size(); i++) if (stats[i].name == name) return (int)i;
    stats.push_back(KernelStat{name, 0, 0.0});
    return (int)stats.size() - 1;
}
void Context::begin_launch(const char* name, int& stat, cudaEvent_t& a, cudaEvent_t& b) {
    launch_count++;
    stat = stat_index(name);
    stats[stat].launches++;
    if (!profiling) return;
    auto get = [&]() { cudaEvent_t e; if (!event_pool.empty()) { e = event_pool.back(); event_pool.pop_back(); } else cudaEventCreate(&e); return e; };
    a = get(); b = get();
    cudaEventRecord(a, stream);
}
void Context::end_launch(int stat, cudaEvent_t a, cudaEvent_t b) {
    if (!profiling || !a) return;
    cudaEventRecord(b, stream);
    pending.push_back(Pending{stat, a, b});
    if (pending.size() > 4096) drain_events();
}
void Context::drain_events() {
    if (pending.empty()) return;
    cudaStreamSynchronize(stream);
    for (auto& p : pending) {
        float ms = 0; cudaEventElapsedTime(&ms, p.a, p.b);
        stats[p.stat].ms += ms;
        event_pool.push_back(p.a); event_pool.push_back(p.b);
    }
    pending.clear();
}

void trace_point(const char* label) {
    static int on = -1;
    static double last = 0;
    if (on < 0) { const char* e = getenv("BL_TRACE"); on = (e && e[0] == '1') ? 1 : 0; }
    if (!on) return;
    cudaStreamSynchronize(ctx().stream);
    struct timespec ts; clock_gettime(CLOCK_MONOTONIC, &ts);
    double now = ts.tv_sec * 1e3 + ts.tv_nsec * 1e-6;
    fprintf(stderr, "[bl_trace] %-28s +%.3f ms\n", label, last ? now - last : 0.0);
    last = now;
}

// ---------------------------------------------------------------------------- memory
// Device blocks are cached by size class (16 classes per power of two) and reused in stream order:
// every kernel and copy of the library runs on ONE stream, so a freed block may be handed out again
// immediately.  Steady-state operator calls therefore never reach the driver allocator (measured:
// cudaMallocAsync/FreeAsync of the 300 MB join table cost ~15 ms per call without this cache).
static std::unordered_map<void*, size_t> g_dev_sizes;
static std::unordered_multimap<size_t, void*> g_dev_free;
static size_t g_dev_cached = 0;
static const size_t kDevCacheMax = (size_t)96 << 30;
static size_t dev_class(size_t bytes) {
    if (bytes <= 512) return 512;
    size_t p = 1; while (p < bytes) p <<= 1;
    size_t step = p >> 4;
    return (bytes + step - 1) / step * step;
}
static void dev_cache_release_all() {
    for (auto& kv : g_dev_free) cudaFreeAsync(kv.second, g_ctx->stream);
    g_dev_free.clear(); g_dev_cached = 0;
    cudaStreamSynchronize(g_ctx->stream);
}
void* dev_alloc_raw(size_t bytes) {
    Context& c = ctx();
    const size_t cls = dev_class(bytes);
    {
        std::lock_guard<std::mutex> lk(g_init_mu);
        auto it = g_dev_free.find(cls);
        if (it != g_dev_free.end()) { void* p = it->second; g_dev_free.erase(it); g_dev_cached -= cls; g_dev_sizes[p] = cls; return p; }
    }
    void* p = nullptr;
    cudaError_t e = cudaMallocAsync(&p, cls, c.stream);
    if (e != cudaSuccess) {      // give cached blocks back to the driver and retry once
        cudaGetLastError();
        { std::lock_guard<std::mutex> lk(g_init_mu); dev_cache_release_all(); }
        e = cudaMallocAsync(&p, cls, c.stream);
    }
    if (e != cudaSuccess) { cudaGetLastError(); fail(BL_ERR_OOM, "device allocation of " + std::to_string(cls) + " bytes failed: " + cudaGetErrorString(e)); }
    std::lock_guard<std::mutex> lk(g_init_mu);
    g_dev_sizes[p] = cls;
    return p;
}
void dev_free_raw(void* p) {
    if (!p || !g_ctx) return;
    std::lock_guard<std::mutex> lk(g_init_mu);
    auto it = g_dev_sizes.find(p);
    if (it == g_dev_sizes.end()) { cudaFreeAsync(p, g_ctx->stream); return; }
    const size_t cls = it->second; g_dev_sizes.erase(it);
    if (g_dev_cached + cls <= kDevCacheMax) { g_dev_free.emplace(cls, p); g_dev_cached += cls; }
    else cudaFreeAsync(p, g_ctx->stream);
}

static size_t pinned_class(size_t bytes) {
    size_t c = 4096; while (c < bytes) c <<= 1;
    // above 64 MiB round to 16 MiB instead of the next power of two
    if (c > ((size_t)64 << 20)) { size_t g = (size_t)16 << 20; c = (bytes + g - 1) / g * g; }
    return c;
}
void* pinned_alloc_raw(size_t bytes) {
    ctx();
    size_t cls = pinned_class(bytes ? bytes : 1);
    {
        std::lock_guard<std::mutex> lk(g_init_mu);
        auto it = g_pinned_free.find(cls);
        if (it != g_pinned_free.end()) { void* p = it->second; g_pinned_free.erase(it); g_pinned_cached -= cls; g_pinned_sizes[p] = cls; return p; }
    }
    void* p = nullptr;
    cudaError_t e = cudaHostAlloc(&p, cls, cudaHostAllocDefault);
    if (e != cudaSuccess) { cudaGetLastError(); fail(BL_ERR_OOM, "pinned host allocation of " + std::to_string(cls) + " bytes failed"); }
    std::lock_guard<std::mutex> lk(g_init_mu);
    g_pinned_sizes[p] = cls;
    return p;
}
void pinned_free_raw(void* p) {
    if (!p) return;
    std::lock_guard<std::mutex> lk(g_init_mu);
    auto it = g_pinned_sizes.find(p);
    if (it == g_pinned_sizes.end()) return;
    size_t cls = it->second; g_pinned_sizes.erase(it);
    if (g_pinned_cached + cls <= kPinnedCacheMax) { g_pinned_free.emplace(cls, p); g_pinned_cached += cls; }
    else cudaFreeHost(p);
}

DevCol make_col(int dtype, int64_t len, bool with_validity) {
    DevCol c; c.dtype = dtype; c.len = len;
    size_t vb = dtype == BL_BOOL ? bitmap_bytes(len) : (size_t)len * dtype_size(dtype);
    c.values = dev_alloc(vb + 16);
    if (with_validity) c.validity = dev_alloc(bitmap_bytes(len) + 16);
    c.null_count = with_validity ? -1 : 0;
    return c;
}

// ---------------------------------------------------------------------------- bitmap copy
// dst[dpos .. dpos+len) |= src[spos .. spos+len)   (dst zero-initialised, word array; src bytes)
__global__ void k_bitmap_copy(uint32_t* __restrict__ dst, int64_t dpos, const uint8_t* __restrict__ src, int64_t spos, int64_t len) {
    int64_t first_word = dpos >> 5, last_word = (dpos + len - 1) >> 5;
    int64_t nwords = last_word - first_word + 1;
    for (int64_t w = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; w < nwords; w += (int64_t)gridDim.x * blockDim.x) {
        int64_t word = first_word + w;
        int64_t lo = word * 32 > dpos ? word * 32 : dpos;                     // dst bit range in this word
        int64_t hi = word * 32 + 32 < dpos + len ? word * 32 + 32 : dpos + len;
        int64_t s = spos + (lo - dpos);                                            // first src bit
        int nb = (int)(hi - lo);
        // gather up to 40 source bits starting at byte s>>3
        uint64_t acc = 0; int64_t b0 = s >> 3; int nbytes = (int)(((s & 7) + nb + 7) >> 3);
        for (int i = 0; i < nbytes; i++) acc |= (uint64_t)src[b0 + i] << (8 * i);
        uint32_t bits = (uint32_t)(acc >> (s & 7));
        if (nb < 32) bits &= (1u << nb) - 1u;
        bits <<= (int)(lo - word * 32);
        if (nb == 32) dst[word] = bits; else atomicOr(&dst[word], bits);
    }
}

DevPtr bitmap_slice(const uint32_t* bm, int64_t pos, int64_t len) {
    DevPtr out = dev_alloc(bitmap_bytes(len) + 16);
    dev_memset(out->p, 0, bitmap_bytes(len) + 16);
    if (len > 0) PLB_LAUNCH("bitmap_copy", k_bitmap_copy, grid_for((len + 31) / 32 + 1, 256), 256, 0, as<uint32_t>(out), (int64_t)0, reinterpret_cast<const uint8_t*>(bm), pos, len);
    return out;
}

// ---------------------------------------------------------------------------- import / export
DevCol import_column(const bl_column* chunks, int n_chunks) {
    PLB_REQUIRE(chunks != nullptr && n_chunks >= 1, BL_ERR_INVALID, "column: no chunks");
    Context& c = ctx();
    int dtype = chunks[0].dtype;
    int64_t total = 0; bool any_validity = false; bool all_device = true;
    for (int i = 0; i < n_chunks; i++) {
        PLB_REQUIRE(chunks[i].dtype == dtype, BL_ERR_DTYPE, "column: chunks have different dtypes");
        PLB_REQUIRE(chunks[i].length >= 0 && chunks[i].offset >= 0, BL_ERR_INVALID, "column: negative length/offset");
        PLB_REQUIRE(chunks[i].length == 0 || chunks[i].values != nullptr, BL_ERR_INVALID, "column: null values pointer");
        total += chunks[i].length;
        any_validity |= (chunks[i].validity != nullptr && chunks[i].null_count != 0);
        all_device &= chunks[i].location == BL_DEVICE;
    }
    PLB_REQUIRE(dtype >= BL_INT8 && dtype <= BL_BOOL, BL_ERR_UNSUPPORTED, "column: unknown dtype");
    int es = dtype_size(dtype);
    DevCol out; out.dtype = dtype; out.len = total;
    // zero-copy: single device chunk, values 16-byte aligned, validity byte-aligned and 4-byte aligned
    if (n_chunks == 1 && all_device && dtype != BL_BOOL) {
        const char* vp = (const char*)chunks[0].values + chunks[0].offset * es;
        bool ok = ((uintptr_t)vp % 16) == 0;
        const uint8_t* mp = nullptr;
        if (any_validity) { ok &= (chunks[0].offset % 8) == 0; mp = chunks[0].validity + chunks[0].offset / 8; ok &= ((uintptr_t)mp % 4) == 0; }
        if (ok) {
            out.values = dev_borrow(vp, (size_t)total * es);
            if (any_validity) {
                // the kernels read validity as 32-bit words: an Arrow bitmap only guarantees ceil(n / 8) bytes, so the last
                // word may only be borrowed when it lies wholly inside them; otherwise the bitmap (1/64 of the column) is copied
                if (total % 32 == 0) out.validity = dev_borrow(mp, bitmap_bytes(total));
                else {
                    out.validity = dev_alloc(bitmap_bytes(total) + 16);
                    dev_memset(out.validity->p, 0, bitmap_bytes(total) + 16);
                    PLB_LAUNCH("bitmap_copy", k_bitmap_copy, grid_for((total + 31) / 32 + 1, 256), 256, 0, as<uint32_t>(out.validity), (int64_t)0, mp, (int64_t)0, total);
                }
            }
            out.null_count = any_validity ? chunks[0].null_count : 0;
            return out;
        }
    }
    if (dtype == BL_BOOL) {
        out.values = dev_alloc(bitmap_bytes(total) + 16);
        dev_memset(out.values->p, 0, bitmap_bytes(total) + 16);
    } else out.values = dev_alloc((size_t)total * es + 16);
    if (any_validity) { out.validity = dev_alloc(bitmap_bytes(total) + 16); dev_memset(out.validity->p, 0, bitmap_bytes(total) + 16); }
    std::vector<DevPtr> staging;   // device copies of host bitmaps
    auto stage_bits = [&](const uint8_t* src, int location, int64_t bit_off, int64_t nbits, const uint8_t*& dsrc, int64_t& dspos) {
        int64_t b0 = bit_off >> 3, b1 = (bit_off + nbits + 7) >> 3;
        if (location == BL_DEVICE) { dsrc = src + b0; dspos = bit_off & 7; return; }
        DevPtr t = dev_alloc((size_t)(b1 - b0) + 16);
        PLB_CUDA(cudaMemcpyAsync(t->p, src + b0, (size_t)(b1 - b0), cudaMemcpyHostToDevice, c.stream));
        staging.push_back(t); dsrc = (const uint8_t*)t->p; dspos = bit_off & 7;
    };
    int64_t pos = 0; int64_t nulls_known = 0; bool nulls_exact = true;
    for (int i = 0; i < n_chunks; i++) {
        const bl_column& ch = chunks[i];
        if (ch.length == 0) continue;
        cudaMemcpyKind kind = ch.location == BL_DEVICE ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice;
        if (dtype == BL_BOOL) {
            const uint8_t* dsrc; int64_t dspos;
            stage_bits((const uint8_t*)ch.values, ch.location, ch.offset, ch.length, dsrc, dspos);
            PLB_LAUNCH("bitmap_copy", k_bitmap_copy, grid_for((ch.length + 31) / 32 + 1, 256), 256, 0, as<uint32_t>(out.values), pos, dsrc, dspos, ch.length);
        } else {
            PLB_CUDA(cudaMemcpyAsync((char*)out.values->p + pos * es, (const char*)ch.values + ch.offset * es, (size_t)ch.length * es, kind, c.stream));
        }
        if (any_validity) {
            if (ch.validity != nullptr && ch.null_count != 0) {
                const uint8_t* dsrc; int64_t dspos;
                stage_bits(ch.validity, ch.location, ch.offset, ch.length, dsrc, dspos);
                PLB_LAUNCH("bitmap_copy", k_bitmap_copy, grid_for((ch.length + 31) / 32 + 1, 256), 256, 0, as<uint32_t>(out.validity), pos, dsrc, dspos, ch.length);
                if (ch.null_count > 0) nulls_known += ch.null_count; else nulls_exact = false;
            } else {
                // all-valid chunk inside a nullable column: set its bits
                DevPtr ones = dev_alloc((size_t)((ch.length + 7) / 8) + 16);
                dev_memset(ones->p, 0xFF, (size_t)((ch.length + 7) / 8) + 16);
                staging.push_back(ones);
                PLB_LAUNCH("bitmap_copy", k_bitmap_copy, grid_for((ch.length + 31) / 32 + 1, 256), 256, 0, as<uint32_t>(out.validity), pos, (const uint8_t*)ones->p, (int64_t)0, ch.length);
            }
        }
        pos += ch.length;
    }
    out.null_count = any_validity ? (nulls_exact ? nulls_known : -1) : 0;
    return out;
}

struct ColOwner { DevPtr values, validity; void* hv = nullptr; void* hm = nullptr; };

void export_column(const DevCol& col, int location, bl_column* out, bool sync) {
    PLB_REQUIRE(out != nullptr, BL_ERR_INVALID, "null output column");
    Context& c = ctx();
    auto* own = new ColOwner();
    size_t vb = col.dtype == BL_BOOL ? bitmap_bytes(col.len) : (size_t)col.len * dtype_size(col.dtype);
    size_t mb = col.validity ? bitmap_bytes(col.len) : 0;
    bl_column r; memset(&r, 0, sizeof(r));
    r.dtype = col.dtype; r.location = location; r.length = col.len; r.offset = 0; r.null_count = col.null_count;
    try {
        if (location == BL_DEVICE) {
            own->values = col.values; own->validity = col.validity;
            r.values = col.values ? col.values->p : nullptr;
            r.validity = col.validity ? (const uint8_t*)col.validity->p : nullptr;
            // borrowed inputs must not escape as outputs: copy them
            if (col.values && !col.values->owned) { DevPtr t = dev_alloc(vb + 16); PLB_CUDA(cudaMemcpyAsync(t->p, col.values->p, vb, cudaMemcpyDeviceToDevice, c.stream)); own->values = t; r.values = t->p; }
            if (col.validity && !col.validity->owned) { DevPtr t = dev_alloc(mb + 16); PLB_CUDA(cudaMemcpyAsync(t->p, col.validity->p, mb, cudaMemcpyDeviceToDevice, c.stream)); own->validity = t; r.validity = (const uint8_t*)t->p; }
            if (sync) PLB_CUDA(cudaStreamSynchronize(c.stream));
        } else {
            own->hv = pinned_alloc_raw(vb + 16);
            if (vb) PLB_CUDA(cudaMemcpyAsync(own->hv, col.values->p, vb, cudaMemcpyDeviceToHost, c.stream));
            if (col.validity) { own->hm = pinned_alloc_raw(mb + 16); PLB_CUDA(cudaMemcpyAsync(own->hm, col.validity->p, mb, cudaMemcpyDeviceToHost, c.stream)); }
            if (sync) PLB_CUDA(cudaStreamSynchronize(c.stream));
            r.values = own->hv; r.validity = (const uint8_t*)own->hm;
        }
    } catch (...) { pinned_free_raw(own->hv); pinned_free_raw(own->hm); delete own; throw; }
    r.owner = own;
    *out = r;
}

// Export several columns with ONE stream synchronisation (all copies are queued first).
void export_many(const std::vector<DevCol>& cols, int location, bl_column* outs) {
    std::vector<bl_column> tmp(cols.size());
    size_t done = 0;
    try {
        for (; done < cols.size(); done++) export_column(cols[done], location, &tmp[done], false);
        PLB_CUDA(cudaStreamSynchronize(ctx().stream));
    } catch (...) { cudaStreamSynchronize(ctx().stream); for (size_t i = 0; i < done; i++) bl_column_free(&tmp[i]); throw; }
    for (size_t i = 0; i < cols.size(); i++) outs[i] = tmp[i];
}

}  // namespace plb

// ================================================================================ C ABI
using namespace plb;
static thread_local std::string t_last_error;
namespace plb { void set_last_error(const std::string& m) { t_last_error = m; } }

extern "C" {

int32_t bl_abi_version(void) { return BL_ABI_VERSION; }
const char* bl_last_error(void) { return t_last_error.c_str(); }

bl_status bl_init(int32_t device) {
    try { ensure_init(device); return BL_OK; }
    catch (const plb::Error& e) { t_last_error = e.what(); return e.code; }
    catch (...) { t_last_error = "bl_init failed"; return BL_ERR_CUDA; }
}
void bl_set_deterministic(int32_t on) { try { ctx().deterministic = on != 0; } catch (...) {} }
void bl_shutdown(void) {
    if (!g_ctx) return;
    cudaStreamSynchronize(g_ctx->stream);
}
bl_status bl_device_info(int32_t* sm_count, int64_t* l2_bytes, int64_t* hbm_total, int64_t* hbm_free) {
    BL_TRY
    Context& c = ctx();
    size_t f = 0, t = 0; PLB_CUDA(cudaMemGetInfo(&f, &t));
    if (sm_count) *sm_count = c.sm_count;
    if (l2_bytes) *l2_bytes = c.l2_bytes;
    if (hbm_total) *hbm_total = (int64_t)t;
    if (hbm_free) *hbm_free = (int64_t)f;
    BL_CATCH
}
bl_status bl_release_cached(void) {
    BL_TRY
    Context& c = ctx();
    { std::lock_guard<std::mutex> lk(g_init_mu); dev_cache_release_all(); }
    cudaMemPool_t pool;
    PLB_CUDA(cudaDeviceGetDefaultMemPool(&pool, c.device));
    PLB_CUDA(cudaMemPoolTrimTo(pool, 0));
    BL_CATCH
}
bl_status bl_alloc_pinned(size_t bytes, void** out) {
    BL_TRY
    PLB_REQUIRE(out, BL_ERR_INVALID, "null out");
    *out = pinned_alloc_raw(bytes);
    BL_CATCH
}
void bl_free_pinned(void* p) { pinned_free_raw(p); }
bl_status bl_dev_alloc(size_t bytes, void** out) {
    BL_TRY
    PLB_REQUIRE(out, BL_ERR_INVALID, "null out");
    *out = dev_alloc_raw(bytes ? bytes : 16);
    PLB_CUDA(cudaStreamSynchronize(ctx().stream));
    BL_CATCH
}
void bl_dev_free(void* p) { dev_free_raw(p); }
bl_status bl_memcpy_h2d(void* dst, const void* src, size_t bytes) {
    BL_TRY
    PLB_CUDA(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, ctx().stream));
    PLB_CUDA(cudaStreamSynchronize(ctx().stream));
    BL_CATCH
}
bl_status bl_memcpy_d2h(void* dst, const void* src, size_t bytes) {
    BL_TRY
    PLB_CUDA(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToHost, ctx().stream));
    PLB_CUDA(cudaStreamSynchronize(ctx().stream));
    BL_CATCH
}
bl_status bl_column_to(const bl_column* chunks, int32_t n_chunks, int32_t location, bl_column* out) {
    BL_TRY
    DevCol c = import_column(chunks, n_chunks);
    export_column(c, location, out);
    BL_CATCH
}
void bl_column_free(bl_column* col) {
    if (!col || !col->owner) return;
    auto* own = reinterpret_cast<plb::ColOwner*>(col->owner);
    pinned_free_raw(own->hv); pinned_free_raw(own->hm);
    delete own;
    col->owner = nullptr; col->values = nullptr; col->validity = nullptr;
}
bl_status bl_sync(void) {
    BL_TRY
    PLB_CUDA(cudaStreamSynchronize(ctx().stream));
    BL_CATCH
}
void* bl_stream(void) { try { return (void*)ctx().stream; } catch (...) { return nullptr; } }

void bl_profile_enable(int32_t enable) { try { Context& c = ctx(); c.drain_events(); c.profiling = enable != 0; } catch (...) {} }
void bl_profile_reset(void) { try { Context& c = ctx(); c.drain_events(); c.stats.clear(); c.launch_count = 0; } catch (...) {} }
int64_t bl_launch_count(void) { try { return ctx().launch_count; } catch (...) { return 0; } }
int64_t bl_profile_json(char* buf, int64_t cap) {
    try {
        Context& c = ctx(); c.drain_events();
        std::string s = "{";
        for (size_t i = 0; i < c.stats.size(); i++) {
            char tmp[256];
            snprintf(tmp, sizeof tmp, "%s\"%s\": {\"launches\": %lld, \"ms\": %.6f}", i ? ", " : "", c.stats[i].name.c_str(), (long long)c.stats[i].launches, c.stats[i].ms);
            s += tmp;
        }
        s += "}";
        if (buf && cap > 0) { size_t n = std::min((size_t)cap - 1, s.size()); memcpy(buf, s.data(), n); buf[n] = 0; }
        return (int64_t)s.size() + 1;
    } catch (...) { return 0; }
}
}  // extern "C"
