// strings.cu — string / binary key columns (SURVEY.md §8(f1)): device-side dictionary encoding.
//
// Reference path being replaced (paths relative to /root/reference/crates):
//   BinaryChunked::group_tuples  polars-core/src/frame/group_by/into_groups.rs:215-251 — hashes every value's bytes
//   (to_bytes_hashes) and groups the (hash, bytes) pairs with group_by_threaded_slice: equal BYTES form a group, nulls form the
//   null group, the group's `first` is the row of its first occurrence.
// Here the same relation is materialised as a u32 code column: code[row] = index of the FIRST row that holds the same bytes
// (null rows keep a null code).  A code column is an ordinary UInt32 key for bl_groupby_agg / bl_hash_join / bl_group_tuples,
// and the distinct codes a group_by returns are exactly the gather indices that materialise the group keys
// (bl_string_gather) — the pair (first, groups) the reference builds, with the bytes touched twice (hash, verify).
//
//   k_str_hash      one thread per row: seeded 64-bit hash of the row's bytes (8 bytes per mixing step)
//   op_group_first_ids (groupby.cu)  row -> first row with the same HASH (the L2-resident table plan of K5)
//   k_str_verify    row's bytes == its representative's bytes?  Equal hash + equal bytes to ONE representative makes the
//                   classes exact; a mismatch means two different strings collided in 64 bits (probability ~ n^2 / 2^65):
//                   the encoding is redone with another seed (4 attempts, then BL_ERR_UNSUPPORTED — never a wrong answer).
//   k_str_lens / k_str_copy   gather: lengths -> exclusive scan -> one warp copies one string
//
// Layout: Arrow LargeBinary / LargeUtf8 (polars-arrow/src/array/binary/mod.rs): int64 offsets (len + 1), bytes, validity.
// Algorithmic bytes: encode reads the bytes twice + 8 B/row of offsets, writes 4 B/row; roofline: HBM.
#include <algorithm>
#include <cstring>
#include <vector>

#include "common.cuh"
#include "dev_utils.cuh"
#include "strings.cuh"

namespace plb {

__device__ __forceinline__ uint64_t str_mix(uint64_t h, uint64_t w) { h = (h ^ w) * 0xff51afd7ed558ccdULL; return h ^ (h >> 29); }
__device__ __forceinline__ uint64_t str_hash_bytes(const uint8_t* __restrict__ p, int64_t n, uint64_t seed) {
    uint64_t h = seed ^ ((uint64_t)n * 0x9E3779B97F4A7C15ULL);
    int64_t i = 0;
    for (; i + 8 <= n; i += 8) {
        uint64_t w = 0;
#pragma unroll
        for (int b = 0; b < 8; b++) w |= (uint64_t)p[i + b] << (8 * b);
        h = str_mix(h, w);
    }
    if (i < n) {
        uint64_t w = 0;
        for (int b = 0; i + b < n; b++) w |= (uint64_t)p[i + b] << (8 * b);
        h = str_mix(h, w ^ 0xc4ceb9fe1a85ec53ULL);
    }
    h ^= h >> 33; h *= 0xc4ceb9fe1a85ec53ULL; h ^= h >> 33;
    return h;
}
__global__ void __launch_bounds__(256) k_str_hash(const int64_t* __restrict__ off, const uint8_t* __restrict__ data, const uint32_t* __restrict__ valid, int64_t n, uint64_t seed,
                                                  uint64_t* __restrict__ out) {
    for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < n; r += (int64_t)gridDim.x * blockDim.x) {
        uint64_t h = 0;
        if (valid == nullptr || bit_get(valid, r)) { const int64_t a = off[r]; h = str_hash_bytes(data + a, off[r + 1] - a, seed); }
        out[r] = h;
    }
}
// stats[0] = rows whose bytes differ from their representative's, stats[1] = representatives (distinct non-null values)
__global__ void __launch_bounds__(256) k_str_verify(const int64_t* __restrict__ off, const uint8_t* __restrict__ data, const uint32_t* __restrict__ valid, const uint32_t* __restrict__ ids,
                                                    int64_t n, unsigned long long* stats) {
    unsigned bad = 0, reps = 0;
    for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < n; r += (int64_t)gridDim.x * blockDim.x) {
        if (valid != nullptr && !bit_get(valid, r)) continue;
        const int64_t q = ids[r];
        if (q == r) { reps++; continue; }
        const int64_t a = off[r], b = off[q], la = off[r + 1] - a;
        bool same = la == off[q + 1] - b && (valid == nullptr || bit_get(valid, q));
        for (int64_t i = 0; same && i < la; i++) same = data[a + i] == data[b + i];
        bad += !same;
    }
    bad = __reduce_add_sync(0xffffffffu, bad); reps = __reduce_add_sync(0xffffffffu, reps);
    if ((threadIdx.x & 31) == 0) { if (bad) atomicAdd(&stats[0], (unsigned long long)bad); if (reps) atomicAdd(&stats[1], (unsigned long long)reps); }
}

// code column (UInt32, validity = the input's) and the number of distinct non-null values
DevCol op_string_codes(const DevStr& s, int64_t* n_distinct) {
    const int64_t n = s.len;
    PLB_REQUIRE(n <= 0xFFFFFFFEll, BL_ERR_UNSUPPORTED, "string keys: more than 2^32-2 rows (IdxSize = u32)");
    DevCol codes; codes.dtype = BL_UINT32; codes.len = n; codes.validity = s.validity; codes.null_count = s.validity ? s.null_count : 0;
    if (n == 0) { codes.values = dev_alloc(16); if (n_distinct) *n_distinct = 0; return codes; }
    DevPtr stats = dev_alloc(16);
    for (int attempt = 0; attempt < 4; attempt++) {
        DevCol hk; hk.dtype = BL_UINT64; hk.len = n; hk.values = dev_alloc((size_t)n * 8 + 16); hk.validity = s.validity; hk.null_count = codes.null_count;
        const uint64_t seed = 0x2545F4914F6CDD1DULL * (uint64_t)(attempt + 1);
        PLB_LAUNCH("str_hash", k_str_hash, grid_for(n, 256, 16), 256, 0, s.off(), s.bytes(), s.vm(), n, seed, as<uint64_t>(hk.values));
        DevCol ids = op_group_first_ids(hk);
        dev_memset(stats->p, 0, 16);
        PLB_LAUNCH("str_verify", k_str_verify, grid_for(n, 256, 16), 256, 0, s.off(), s.bytes(), s.vm(), as<uint32_t>(ids.values), n, as<unsigned long long>(stats));
        unsigned long long h[2];
        PLB_CUDA(cudaMemcpyAsync(h, stats->p, 16, cudaMemcpyDeviceToHost, ctx().stream));
        PLB_CUDA(cudaStreamSynchronize(ctx().stream));
        if (h[0] == 0) { codes.values = ids.values; if (n_distinct) *n_distinct = (int64_t)h[1]; return codes; }
    }
    fail(BL_ERR_UNSUPPORTED, "string keys: 64-bit hash collisions under four seeds");
    return codes;
}

__global__ void __launch_bounds__(256) k_str_lens(const int64_t* __restrict__ off, const uint32_t* __restrict__ valid, int64_t n_src, const uint32_t* __restrict__ idx, const uint32_t* __restrict__ idx_valid,
                                                  int64_t n, uint64_t* __restrict__ lens, uint32_t* __restrict__ out_valid, int* oob) {
    for (int64_t i0 = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) & ~31ll; i0 < n; i0 += (int64_t)gridDim.x * blockDim.x) {
        const int64_t i = i0 + (threadIdx.x & 31);
        bool ok = false; uint64_t l = 0;
        if (i < n && (idx_valid == nullptr || bit_get(idx_valid, i))) {
            const uint32_t q = idx[i];
            if (q != 0xFFFFFFFFu) {
                if ((int64_t)q >= n_src) *oob = 1;
                else if (valid == nullptr || bit_get(valid, q)) { ok = true; l = (uint64_t)(off[q + 1] - off[q]); }
            }
        }
        if (i < n) lens[i] = l;
        const unsigned b = __ballot_sync(0xffffffffu, ok);
        if ((threadIdx.x & 31) == 0 && out_valid) out_valid[i0 >> 5] = b;
    }
}
__global__ void __launch_bounds__(256) k_str_copy(const int64_t* __restrict__ off, const uint8_t* __restrict__ data, const uint32_t* __restrict__ idx, const int64_t* __restrict__ out_off,
                                                  int64_t n, uint8_t* __restrict__ out) {
    const int lane = threadIdx.x & 31;
    for (int64_t i = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; i < n; i += ((int64_t)gridDim.x * blockDim.x) >> 5) {
        const int64_t o = out_off[i], l = out_off[i + 1] - o;
        if (l == 0) continue;
        const int64_t a = off[idx[i]];
        for (int64_t b = lane; b < l; b += 32) out[o + b] = data[a + b];
    }
}

DevStr op_string_gather(const DevStr& s, const DevCol& idx) {
    PLB_REQUIRE(idx.dtype == BL_UINT32, BL_ERR_DTYPE, "string gather: indices must be UInt32 (IdxSize)");
    const int64_t n = idx.len;
    DevStr out; out.len = n;
    out.offsets = dev_alloc((size_t)(n + 1) * 8 + 16);
    const int64_t n_round = (n + 31) / 32 * 32;
    out.validity = dev_alloc(bitmap_bytes(n_round) + 16);
    DevPtr tot = dev_alloc(16), oob = dev_alloc(16);
    dev_memset(oob->p, 0, 4); dev_memset(tot->p, 0, 8);
    if (n > 0) {
        DevPtr lens = dev_alloc((size_t)n * 8 + 16);
        PLB_LAUNCH("str_lens", k_str_lens, grid_for(n_round, 256, 16), 256, 0, s.off(), s.vm(), s.len, as<uint32_t>(idx.values), idx.vm(), n, as<uint64_t>(lens), as<uint32_t>(out.validity), as<int>(oob));
        exclusive_scan_u64(as<uint64_t>(lens), as<uint64_t>(out.offsets), n, as<uint64_t>(tot));
    }
    struct { unsigned long long total; } h{0}; int hoob = 0;
    PLB_CUDA(cudaMemcpyAsync(&h.total, tot->p, 8, cudaMemcpyDeviceToHost, ctx().stream));
    PLB_CUDA(cudaMemcpyAsync(&hoob, oob->p, 4, cudaMemcpyDeviceToHost, ctx().stream));
    PLB_CUDA(cudaStreamSynchronize(ctx().stream));
    PLB_REQUIRE(!hoob, BL_ERR_BOUNDS, "string gather: index out of bounds");
    out.data_bytes = (int64_t)h.total;
    PLB_CUDA(cudaMemcpyAsync((char*)out.offsets->p + (size_t)n * 8, &h.total, 8, cudaMemcpyHostToDevice, ctx().stream));
    PLB_CUDA(cudaStreamSynchronize(ctx().stream));       // h lives on this frame
    out.data = dev_alloc((size_t)out.data_bytes + 16);
    if (n > 0 && out.data_bytes > 0)
        PLB_LAUNCH("str_copy", k_str_copy, grid_for(n * 32, 256, 16), 256, 0, s.off(), s.bytes(), as<uint32_t>(idx.values), as<int64_t>(out.offsets), n, as<uint8_t>(out.data));
    out.null_count = n > 0 ? n - bitmap_popcount(as<uint32_t>(out.validity), n) : 0;
    if (out.null_count == 0) out.validity.reset();
    return out;
}

// ---------------------------------------------------------------------------- import / export
__global__ void k_str_rebase(const int64_t* __restrict__ in, int64_t n_plus_1, int64_t delta, int64_t* __restrict__ out) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_plus_1; i += (int64_t)gridDim.x * blockDim.x) out[i] = in[i] + delta;
}

DevStr import_string(const bl_string_column* chunks, int n_chunks) {
    PLB_REQUIRE(chunks != nullptr && n_chunks >= 1, BL_ERR_INVALID, "string column: no chunks");
    Context& c = ctx();
    int64_t total = 0; bool any_validity = false;
    for (int i = 0; i < n_chunks; i++) {
        PLB_REQUIRE(chunks[i].length >= 0 && chunks[i].offset >= 0, BL_ERR_INVALID, "string column: negative length/offset");
        PLB_REQUIRE(chunks[i].offsets != nullptr, BL_ERR_INVALID, "string column: null offsets pointer");
        total += chunks[i].length;
        any_validity |= chunks[i].validity != nullptr && chunks[i].null_count != 0;
    }
    // first / last offset of every chunk (device chunks: two small reads each)
    std::vector<int64_t> lo(n_chunks), hi(n_chunks);
    for (int i = 0; i < n_chunks; i++) {
        const int64_t* o = chunks[i].offsets + chunks[i].offset;
        if (chunks[i].location == BL_DEVICE) {
            PLB_CUDA(cudaMemcpyAsync(&lo[i], o, 8, cudaMemcpyDeviceToHost, c.stream));
            PLB_CUDA(cudaMemcpyAsync(&hi[i], o + chunks[i].length, 8, cudaMemcpyDeviceToHost, c.stream));
            PLB_CUDA(cudaStreamSynchronize(c.stream));
        } else { lo[i] = o[0]; hi[i] = o[chunks[i].length]; }
        PLB_REQUIRE(hi[i] >= lo[i] && lo[i] >= 0, BL_ERR_INVALID, "string column: offsets are not monotonic");
        PLB_REQUIRE(hi[i] == lo[i] || chunks[i].data != nullptr, BL_ERR_INVALID, "string column: null data pointer");
    }
    DevStr out; out.len = total;
    for (int i = 0; i < n_chunks; i++) out.data_bytes += hi[i] - lo[i];
    out.offsets = dev_alloc((size_t)(total + 1) * 8 + 16);
    out.data = dev_alloc((size_t)out.data_bytes + 16);
    dev_memset(out.offsets->p, 0, 8);
    std::vector<DevPtr> staging;
    int64_t pos = 0, cursor = 0;
    for (int i = 0; i < n_chunks; i++) {
        const bl_string_column& ch = chunks[i];
        const cudaMemcpyKind kind = ch.location == BL_DEVICE ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice;
        const int64_t* o = ch.offsets + ch.offset;
        const int64_t* dsrc = o;
        if (ch.location != BL_DEVICE) {
            DevPtr t = dev_alloc((size_t)(ch.length + 1) * 8 + 16);
            PLB_CUDA(cudaMemcpyAsync(t->p, o, (size_t)(ch.length + 1) * 8, cudaMemcpyHostToDevice, c.stream));
            staging.push_back(t); dsrc = as<int64_t>(t);
        }
        PLB_LAUNCH("str_rebase", k_str_rebase, grid_for(ch.length + 1, 256), 256, 0, dsrc, ch.length + 1, cursor - lo[i], as<int64_t>(out.offsets) + pos);
        if (hi[i] > lo[i]) PLB_CUDA(cudaMemcpyAsync((char*)out.data->p + cursor, ch.data + lo[i], (size_t)(hi[i] - lo[i]), kind, c.stream));
        pos += ch.length; cursor += hi[i] - lo[i];
    }
    if (any_validity) {
        // the validity bitmaps, concatenated at their bit offsets: import them as the VALUES of a boolean column
        std::vector<bl_column> fake(n_chunks);
        std::vector<std::vector<uint8_t>> ones;
        for (int i = 0; i < n_chunks; i++) {
            bl_column& f = fake[i]; memset(&f, 0, sizeof f);
            f.dtype = BL_BOOL; f.location = chunks[i].location; f.length = chunks[i].length; f.offset = chunks[i].offset; f.values = chunks[i].validity;
            if (chunks[i].validity == nullptr || chunks[i].null_count == 0) {      // an all-valid chunk of a nullable column
                ones.emplace_back((size_t)(chunks[i].length + 7) / 8 + 8, (uint8_t)0xFF);
                f.location = BL_HOST; f.offset = 0; f.values = ones.back().data();
            }
        }
        DevCol bits = import_column(fake.data(), n_chunks);
        PLB_CUDA(cudaStreamSynchronize(c.stream));      // `ones` lives on this frame
        out.validity = bits.values;
        out.null_count = total - bitmap_popcount(as<uint32_t>(out.validity), total);
        if (out.null_count == 0) out.validity.reset();
    }
    PLB_CUDA(cudaStreamSynchronize(c.stream));          // staging buffers / host offsets may go
    return out;
}

struct StrOwner { DevPtr offsets, data, validity; void* ho = nullptr; void* hd = nullptr; void* hm = nullptr; };

void export_string(const DevStr& s, int location, bl_string_column* out) {
    PLB_REQUIRE(out != nullptr, BL_ERR_INVALID, "null output string column");
    Context& c = ctx();
    auto* own = new StrOwner();
    bl_string_column r; memset(&r, 0, sizeof r);
    r.location = location; r.length = s.len; r.offset = 0; r.null_count = s.validity ? s.null_count : 0;
    const size_t ob = (size_t)(s.len + 1) * 8, db = (size_t)s.data_bytes, mb = s.validity ? bitmap_bytes(s.len) : 0;
    try {
        if (location == BL_DEVICE) {
            own->offsets = s.offsets; own->data = s.data; own->validity = s.validity;
            r.offsets = s.off(); r.data = s.bytes(); r.validity = s.validity ? (const uint8_t*)s.validity->p : nullptr;
        } else {
            own->ho = pinned_alloc_raw(ob + 16); own->hd = pinned_alloc_raw(db + 16);
            PLB_CUDA(cudaMemcpyAsync(own->ho, s.offsets->p, ob, cudaMemcpyDeviceToHost, c.stream));
            if (db) PLB_CUDA(cudaMemcpyAsync(own->hd, s.data->p, db, cudaMemcpyDeviceToHost, c.stream));
            if (s.validity) { own->hm = pinned_alloc_raw(mb + 16); PLB_CUDA(cudaMemcpyAsync(own->hm, s.validity->p, mb, cudaMemcpyDeviceToHost, c.stream)); }
            r.offsets = (const int64_t*)own->ho; r.data = (const uint8_t*)own->hd; r.validity = (const uint8_t*)own->hm;
        }
        PLB_CUDA(cudaStreamSynchronize(c.stream));
    } catch (...) { pinned_free_raw(own->ho); pinned_free_raw(own->hd); pinned_free_raw(own->hm); delete own; throw; }
    r.owner = own;
    *out = r;
}

}  // namespace plb

// ================================================================================ C ABI
using namespace plb;
extern "C" {

bl_status bl_string_encode(const bl_string_column* chunks, int32_t n_chunks, int32_t out_location, bl_column* out_codes, int64_t* n_distinct) {
    BL_TRY
    PLB_REQUIRE(out_codes != nullptr, BL_ERR_INVALID, "string_encode: null output");
    DevStr s = import_string(chunks, n_chunks);
    int64_t nd = 0;
    DevCol codes = op_string_codes(s, &nd);
    export_column(codes, out_location, out_codes);
    if (n_distinct) *n_distinct = nd;
    BL_CATCH
}

bl_status bl_string_gather(const bl_string_column* chunks, int32_t n_chunks, const bl_column* idx, int32_t out_location, bl_string_column* out) {
    BL_TRY
    PLB_REQUIRE(idx != nullptr && out != nullptr, BL_ERR_INVALID, "string_gather: null argument");
    DevStr s = import_string(chunks, n_chunks);
    DevCol ix = import_column(idx, 1);
    DevStr g = op_string_gather(s, ix);
    export_string(g, out_location, out);
    BL_CATCH
}

bl_status bl_string_column_to(const bl_string_column* chunks, int32_t n_chunks, int32_t location, bl_string_column* out) {
    BL_TRY
    DevStr s = import_string(chunks, n_chunks);
    export_string(s, location, out);
    BL_CATCH
}

// device view of a code column slice [pos, pos + len) as a caller-owned bl_column
static bl_column codes_view(const DevCol& codes, int64_t pos, int64_t len) {
    bl_column v; memset(&v, 0, sizeof v);
    v.dtype = BL_UINT32; v.location = BL_DEVICE; v.length = len; v.offset = pos; v.null_count = codes.validity ? -1 : 0;
    v.values = codes.v(); v.validity = codes.validity ? (const uint8_t*)codes.validity->p : nullptr;
    return v;
}

bl_status bl_groupby_agg_strings(const bl_string_column* key_chunks, int32_t n_key_chunks, const bl_agg* aggs, int32_t n_aggs, int32_t maintain_order, int32_t out_location,
                                 bl_string_column* out_key, bl_column* out_aggs) {
    BL_TRY
    PLB_REQUIRE(out_key != nullptr, BL_ERR_INVALID, "groupby_agg_strings: null output");
    DevStr s = import_string(key_chunks, n_key_chunks);
    DevCol codes = op_string_codes(s, nullptr);
    const bl_column cv = codes_view(codes, 0, codes.len);
    bl_column ok; memset(&ok, 0, sizeof ok);
    const bl_status st = bl_groupby_agg(&cv, 1, aggs, n_aggs, maintain_order, out_location, &ok, out_aggs);      // the context lock is recursive
    if (st != BL_OK) return st;
    try {
        DevCol ix = import_column(&ok, 1);
        DevStr g = op_string_gather(s, ix);
        export_string(g, out_location, out_key);
    } catch (...) { bl_column_free(&ok); for (int i = 0; i < n_aggs; i++) bl_column_free(&out_aggs[i]); throw; }
    bl_column_free(&ok);
    BL_CATCH
}

bl_status bl_hash_join_strings(const bl_string_column* left_chunks, int32_t n_left_chunks, const bl_string_column* right_chunks, int32_t n_right_chunks, int32_t how,
                               int32_t nulls_equal, int32_t maintain_order, int32_t out_location, bl_column* out_left_idx, bl_column* out_right_idx) {
    BL_TRY
    PLB_REQUIRE(left_chunks && right_chunks && n_left_chunks >= 1 && n_right_chunks >= 1, BL_ERR_INVALID, "hash_join_strings: null argument");
    // both relations are encoded TOGETHER so that equal bytes get the same code on either side
    std::vector<bl_string_column> all(left_chunks, left_chunks + n_left_chunks);
    all.insert(all.end(), right_chunks, right_chunks + n_right_chunks);
    int64_t nl = 0; for (int i = 0; i < n_left_chunks; i++) nl += left_chunks[i].length;
    DevStr s = import_string(all.data(), (int)all.size());
    DevCol codes = op_string_codes(s, nullptr);
    const bl_column lv = codes_view(codes, 0, nl), rv = codes_view(codes, nl, codes.len - nl);
    const bl_status st = bl_hash_join(&lv, 1, &rv, 1, how, nulls_equal, maintain_order, out_location, out_left_idx, out_right_idx);
    if (st != BL_OK) return st;
    BL_CATCH
}

void bl_string_column_free(bl_string_column* col) {
    if (!col || !col->owner) return;
    auto* own = reinterpret_cast<plb::StrOwner*>(col->owner);
    pinned_free_raw(own->ho); pinned_free_raw(own->hd); pinned_free_raw(own->hm);
    delete own;
    col->owner = nullptr; col->offsets = nullptr; col->data = nullptr; col->validity = nullptr;
}

}  // extern "C"
