// string_rank.cu — dense lexicographic rank of a string / binary column, and arg_sort over keys that may be strings.
//
// Reference (paths relative to /root/reference/crates): StringChunked sorts as BinaryChunked
// (polars-core/src/chunked_array/ops/sort/mod.rs:369-403), and binary values compare by tot_cmp on &[u8] (mod.rs:405-499):
// unsigned lexicographic byte order, a proper prefix first.  The rank is RankMethod::Dense (polars-ops/src/series/ops/rank.rs:
// 61-188): 1-based IdxSize, equal values equal ranks, consecutive, null rows null.
//
// Plan (DESIGN.md §9):
//   1. dedup       op_string_codes (exact) -> the m distinct non-null values ("representatives"), their largest length
//   2. refine      MSD over positions p in [0, m) in 7-byte chunks.  State: ord[p] = representative row at position p, the
//                  active list A (ascending positions of the members of buckets with more than one member) and bid[j], the
//                  bucket of A[j] (ids ascend with position).  Round r:
//                    k_str_rank_key     u64 key per active entry: bytes [7r, 7r + 7) big-endian in the high 56 bits, zero
//                                       padded, min(len - 7r, 8) in the low byte ("ended here" before "continues"); AND/OR
//                                       of the keys and of the bucket ids
//                    (keys all equal)   nothing splits: next round
//                    radix sort         stable by key (varying digits only), then stable by bucket id (skipped while one
//                                       bucket is active): the two-stage pattern of quantile_large_groups
//                    k_str_rank_heads   the j-th refined entry belongs at position A[j] (active buckets are whole,
//                                       contiguous and listed in order); a new bucket starts where the bucket or the key
//                                       changes: one head bit per entry, counted per tile
//                    k_str_rank_apply   writes ord, numbers the new buckets (scan of the head bits) and marks the entries
//                                       left in buckets with more than one member; op_filter compacts A and bid by that mask
//                  The values are distinct, so a bucket whose strings end inside the chunk is a singleton: the loop ends
//                  after at most (largest length) / 7 + 1 rounds.
//   3. rows        rk[ord[p]] = p + 1, then rank[row] = rk[code[row]] for valid rows (validity = the input's).
// Bytes per round: 4 (A) + 4 (ord) + 16 (offsets) + the chunk's bytes per active entry for the key, then per radix pass
// 2 * 12 per active entry (plus 2 * 8 per bucket pass), and about 40 per active entry for heads, apply and compaction.
#include <algorithm>
#include <vector>

#include "common.cuh"
#include "dev_utils.cuh"
#include "strings.cuh"

namespace plb {

bool radix_sort_pairs_u32(uint32_t* k0, uint32_t* v0, uint32_t* k1, uint32_t* v1, int64_t n, uint64_t vary, int* passes_run);
bool radix_sort_pairs_u64(uint64_t* k0, uint32_t* v0, uint64_t* k1, uint32_t* v1, int64_t n, uint64_t vary, int* passes_run);

constexpr int SR_THREADS = 256, SR_ITEMS = 16, SR_TILE = SR_THREADS * SR_ITEMS, SR_TILE_WORDS = SR_TILE / 32;

// the representatives (valid rows whose code is their own row) in any order; ctr[0] = count, ctr[1] = largest length
__global__ void __launch_bounds__(256) k_str_rank_reps(const uint32_t* __restrict__ code, const uint32_t* __restrict__ valid, const int64_t* __restrict__ off, int64_t n,
                                                       uint32_t* __restrict__ rep, unsigned long long* __restrict__ ctr) {
    unsigned long long mx = 0;
    const unsigned lane = lane_id();
    for (int64_t base = (int64_t)blockIdx.x * blockDim.x; base < n; base += (int64_t)gridDim.x * blockDim.x) {
        const int64_t i = base + threadIdx.x;
        const bool is = i < n && (valid == nullptr || bit_get(valid, i)) && code[i] == (uint32_t)i;
        if (is) mx = max(mx, (unsigned long long)(off[i + 1] - off[i]));
        const unsigned b = __ballot_sync(0xffffffffu, is);
        unsigned long long p0 = 0;
        if (lane == 0 && b) p0 = atomicAdd(&ctr[0], (unsigned long long)__popc(b));
        p0 = __shfl_sync(0xffffffffu, p0, 0);
        if (is) rep[p0 + __popc(b & lanemask_lt())] = (uint32_t)i;
    }
    for (int o = 16; o; o >>= 1) mx = max(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    if (lane == 0 && mx) atomicMax(&ctr[1], mx);
}

// bytes [o, o + 7) of the row's value big-endian in bits 63..8 (zero past its end), min(len - o, 8) in bits 7..0
__device__ __forceinline__ uint64_t str_chunk_key(const int64_t* __restrict__ off, const uint8_t* __restrict__ data, uint32_t row, int64_t o) {
    const int64_t a = off[row], rem = off[row + 1] - a - o;
    uint64_t k = rem <= 0 ? 0 : (uint64_t)min(rem, (int64_t)8);
#pragma unroll
    for (int b = 0; b < 7; b++)
        if (b < rem) k |= (uint64_t)data[a + o + b] << (56 - 8 * b);
    return k;
}

// keys[j] / vals[j] = j for the active entries; andor[0..1] = AND / OR of the keys, andor[2..3] = AND / OR of the bucket ids
__global__ void __launch_bounds__(256) k_str_rank_key(const uint32_t* __restrict__ A, const uint32_t* __restrict__ bid, const uint32_t* __restrict__ ord, int64_t nA,
                                                      const int64_t* __restrict__ off, const uint8_t* __restrict__ data, int64_t o, uint64_t* __restrict__ keys,
                                                      uint32_t* __restrict__ vals, unsigned long long* __restrict__ andor) {
    uint64_t a = ~0ull, r = 0;
    uint32_t ba = ~0u, bo = 0;
    for (int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; j < nA; j += (int64_t)gridDim.x * blockDim.x) {
        const uint64_t k = str_chunk_key(off, data, ord[A[j]], o);
        keys[j] = k; vals[j] = (uint32_t)j;
        a &= k; r |= k;
        ba &= bid[j]; bo |= bid[j];
    }
    const uint32_t al = __reduce_and_sync(0xffffffffu, (uint32_t)a), ah = __reduce_and_sync(0xffffffffu, (uint32_t)(a >> 32));
    const uint32_t rl = __reduce_or_sync(0xffffffffu, (uint32_t)r), rh = __reduce_or_sync(0xffffffffu, (uint32_t)(r >> 32));
    ba = __reduce_and_sync(0xffffffffu, ba); bo = __reduce_or_sync(0xffffffffu, bo);
    if (lane_id() == 0) {
        atomicAnd(&andor[0], ((unsigned long long)ah << 32) | al); atomicOr(&andor[1], ((unsigned long long)rh << 32) | rl);
        atomicAnd(&andor[2], (unsigned long long)ba); atomicOr(&andor[3], (unsigned long long)bo);
    }
}

// second stage: bucket id of the entry at each key-sorted position, payload = that position
__global__ void __launch_bounds__(256) k_str_rank_bucket_keys(const uint32_t* __restrict__ v1, const uint32_t* __restrict__ bid, int64_t nA, uint32_t* __restrict__ bk,
                                                              uint32_t* __restrict__ pos) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < nA; i += (int64_t)gridDim.x * blockDim.x) { bk[i] = bid[v1[i]]; pos[i] = (uint32_t)i; }
}

// entry i of the refined order (p2[i] = its key-sorted position; p2 == nullptr: the identity) goes to position A[i]:
// rows[i] = its row; head bit i = it starts a bucket (bucket or key differs from entry i - 1); tile_cnt[t] = heads in tile t
__global__ void __launch_bounds__(SR_THREADS) k_str_rank_heads(const uint32_t* __restrict__ p2, const uint64_t* __restrict__ k1, const uint32_t* __restrict__ v1,
                                                               const uint32_t* __restrict__ A, const uint32_t* __restrict__ bid, const uint32_t* __restrict__ ord, int64_t nA,
                                                               int64_t ntiles, uint32_t* __restrict__ rows, uint32_t* __restrict__ heads, uint32_t* __restrict__ tile_cnt) {
    __shared__ unsigned s_cnt[SR_THREADS / 32];
    const unsigned lane = lane_id(), warp = threadIdx.x >> 5;
    for (int64_t t = blockIdx.x; t < ntiles; t += gridDim.x) {
        unsigned c = 0;
#pragma unroll 4
        for (int r = 0; r < SR_ITEMS; r++) {
            const int64_t i = t * SR_TILE + (int64_t)r * SR_THREADS + threadIdx.x;
            bool h = false;
            if (i < nA) {
                const uint32_t i1 = p2 ? p2[i] : (uint32_t)i;
                rows[i] = ord[A[v1[i1]]];
                h = i == 0 || bid[i] != bid[i - 1] || k1[i1] != k1[p2 ? p2[i - 1] : (uint32_t)(i - 1)];
            }
            const unsigned b = __ballot_sync(0xffffffffu, h);
            if (lane == 0 && i < nA) heads[i >> 5] = b;
            c += lane == 0 ? __popc(b) : 0;
        }
        if (lane == 0) s_cnt[warp] = c;
        __syncthreads();
        if (threadIdx.x == 0) {
            unsigned tot = 0;
            for (int w = 0; w < SR_THREADS / 32; w++) tot += s_cnt[w];
            tile_cnt[t] = tot;
        }
        __syncthreads();
    }
}

// ord[A[i]] = rows[i]; nb[i] = the new bucket id of entry i (heads up to i, minus one); keep bit i = entry i is not alone
// in its bucket
__global__ void __launch_bounds__(SR_THREADS) k_str_rank_apply(const uint32_t* __restrict__ heads, const uint64_t* __restrict__ tile_off, const uint32_t* __restrict__ rows,
                                                               const uint32_t* __restrict__ A, int64_t nA, int64_t ntiles, uint32_t* __restrict__ ord, uint32_t* __restrict__ nb,
                                                               uint32_t* __restrict__ keep) {
    __shared__ uint32_t s_word[SR_TILE_WORDS], s_pre[SR_TILE_WORDS], s_grp[SR_TILE_WORDS / 32];
    const unsigned lane = lane_id(), warp = threadIdx.x >> 5;
    for (int64_t t = blockIdx.x; t < ntiles; t += gridDim.x) {
        if (threadIdx.x < SR_TILE_WORDS) {
            const int64_t w = t * SR_TILE_WORDS + threadIdx.x;
            const uint32_t m = w * 32 < nA ? heads[w] : 0u;
            const uint32_t c = __popc(m);
            uint32_t x = c;
            for (int o = 1; o < 32; o <<= 1) { const uint32_t y = __shfl_up_sync(0xffffffffu, x, o); if (lane >= (unsigned)o) x += y; }
            s_word[threadIdx.x] = m; s_pre[threadIdx.x] = x - c;
            if (lane == 31) s_grp[warp] = x;
        }
        __syncthreads();
        if (threadIdx.x == 0) {
            uint32_t acc = 0;
            for (int g = 0; g < SR_TILE_WORDS / 32; g++) { const uint32_t v = s_grp[g]; s_grp[g] = acc; acc += v; }
        }
        __syncthreads();
#pragma unroll 4
        for (int r = 0; r < SR_ITEMS; r++) {
            const int64_t i = t * SR_TILE + (int64_t)r * SR_THREADS + threadIdx.x;
            bool kp = false;
            if (i < nA) {
                const int wl = r * (SR_THREADS / 32) + (int)warp;
                const uint32_t m = s_word[wl];
                const bool h = (m >> lane) & 1u;
                nb[i] = (uint32_t)(tile_off[t] + s_grp[wl >> 5] + s_pre[wl] + __popc(m & lanemask_lt()) + (h ? 1u : 0u) - 1u);
                ord[A[i]] = rows[i];
                const bool next_h = i + 1 >= nA || ((heads[(i + 1) >> 5] >> ((i + 1) & 31)) & 1u);
                kp = !(h && next_h);
            }
            const unsigned b = __ballot_sync(0xffffffffu, kp);
            if (lane == 0 && i < nA) keep[i >> 5] = b;
        }
        __syncthreads();
    }
}

__global__ void __launch_bounds__(256) k_str_rank_scatter(const uint32_t* __restrict__ ord, int64_t m, uint32_t* __restrict__ rk) {
    for (int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; p < m; p += (int64_t)gridDim.x * blockDim.x) rk[ord[p]] = (uint32_t)(p + 1);
}

__global__ void __launch_bounds__(256) k_str_rank_rows(const uint32_t* __restrict__ code, const uint32_t* __restrict__ valid, const uint32_t* __restrict__ rk, int64_t n,
                                                       int descending, uint32_t m, uint32_t* __restrict__ out) {
    for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < n; r += (int64_t)gridDim.x * blockDim.x) {
        uint32_t v = 0;
        if (valid == nullptr || bit_get(valid, r)) { v = rk[code[r]]; if (descending) v = m + 1 - v; }
        out[r] = v;
    }
}

static DevCol u32_col(const DevPtr& p, int64_t len) { DevCol c; c.dtype = BL_UINT32; c.len = len; c.values = p; c.null_count = 0; return c; }

DevCol op_string_rank(const DevStr& s, bool descending, int64_t* n_distinct) {
    Context& c = ctx();
    const int64_t n = s.len;
    int64_t m = 0;
    DevCol codes = op_string_codes(s, &m);        // more than 2^32 - 2 rows: BL_ERR_UNSUPPORTED there
    if (n_distinct) *n_distinct = m;
    DevCol out = codes;
    out.values = dev_alloc((size_t)n * 4 + 16);
    if (n == 0) return out;
    const int64_t* off = s.off();
    const uint8_t* data = s.bytes();
    DevPtr ord = dev_alloc((size_t)m * 4 + 16), ctr = dev_alloc(16);
    dev_memset(ctr->p, 0, 16);
    PLB_LAUNCH("str_rank_reps", k_str_rank_reps, grid_for(n, 256), 256, 0, as<uint32_t>(codes.values), s.vm(), off, n, as<uint32_t>(ord), as<unsigned long long>(ctr));
    uint64_t hc[2];
    PLB_CUDA(cudaMemcpyAsync(hc, ctr->p, 16, cudaMemcpyDeviceToHost, c.stream));
    PLB_CUDA(cudaStreamSynchronize(c.stream));
    PLB_REQUIRE((int64_t)hc[0] == m, BL_ERR_INVALID, "string rank: internal error (representatives != distinct values)");
    const int64_t max_len = (int64_t)hc[1];
    // refinement state over the active entries
    int64_t nA = m > 1 ? m : 0;
    DevCol A = u32_col(dev_alloc((size_t)std::max<int64_t>(nA, 1) * 4 + 16), nA), bid = u32_col(dev_alloc((size_t)std::max<int64_t>(nA, 1) * 4 + 16), nA);
    if (nA) { iota_u32(as<uint32_t>(A.values), nA, 0); dev_memset(bid.values->p, 0, (size_t)nA * 4); }
    DevPtr andor = dev_alloc(32);
    for (int64_t round = 0; nA > 0; round++) {
        PLB_REQUIRE(round <= max_len / 7 + 1, BL_ERR_INVALID, "string rank: internal error (refinement did not converge)");
        const int64_t o = round * 7;
        DevPtr ka = dev_alloc((size_t)nA * 8), kb = dev_alloc((size_t)nA * 8), va = dev_alloc((size_t)nA * 4), vb = dev_alloc((size_t)nA * 4);
        dev_memset(andor->p, 0xFF, 8); dev_memset((char*)andor->p + 8, 0, 8);
        dev_memset((char*)andor->p + 16, 0xFF, 8); dev_memset((char*)andor->p + 24, 0, 8);
        PLB_LAUNCH("str_rank_key", k_str_rank_key, grid_for(nA, 256), 256, 0, as<uint32_t>(A.values), as<uint32_t>(bid.values), as<uint32_t>(ord), nA, off, data, o,
                   as<uint64_t>(ka), as<uint32_t>(va), as<unsigned long long>(andor));
        uint64_t ao[4];
        PLB_CUDA(cudaMemcpyAsync(ao, andor->p, 32, cudaMemcpyDeviceToHost, c.stream));
        PLB_CUDA(cudaStreamSynchronize(c.stream));
        const uint64_t vary = ao[0] ^ ao[1], bvary = ao[2] ^ ao[3];
        if (vary == 0) continue;            // one chunk for every active value (a shared prefix): nothing splits
        // stage 1: by key
        const bool sw1 = radix_sort_pairs_u64(as<uint64_t>(ka), as<uint32_t>(va), as<uint64_t>(kb), as<uint32_t>(vb), nA, vary, nullptr);
        const uint64_t* k1 = as<uint64_t>(sw1 ? kb : ka);
        const uint32_t* v1 = as<uint32_t>(sw1 ? vb : va);
        // stage 2: stable by bucket, so every bucket holds its entries in key order
        uint32_t* spare_v = as<uint32_t>(sw1 ? va : vb);
        uint32_t* spare_k = reinterpret_cast<uint32_t*>(sw1 ? ka->p : kb->p);      // 8 nA bytes: two u32 key buffers
        DevPtr p2a;
        const uint32_t* p2 = nullptr;
        if (bvary) {
            p2a = dev_alloc((size_t)nA * 4);
            PLB_LAUNCH("str_rank_bucket_keys", k_str_rank_bucket_keys, grid_for(nA, 256), 256, 0, v1, as<uint32_t>(bid.values), nA, spare_k, spare_v);
            const bool sw2 = radix_sort_pairs_u32(spare_k, spare_v, spare_k + nA, as<uint32_t>(p2a), nA, bvary, nullptr);
            p2 = sw2 ? as<uint32_t>(p2a) : spare_v;
        }
        const int64_t ntiles = (nA + SR_TILE - 1) / SR_TILE;
        DevPtr rows = dev_alloc((size_t)nA * 4), heads = dev_alloc((size_t)ntiles * SR_TILE_WORDS * 4), keep = dev_alloc((size_t)ntiles * SR_TILE_WORDS * 4);
        DevPtr cnt = dev_alloc((size_t)ntiles * 4), toff = dev_alloc((size_t)ntiles * 8 + 8), nb = dev_alloc((size_t)nA * 4);
        const int tgrid = (int)std::min<int64_t>(ntiles, (int64_t)c.sm_count * 8);
        PLB_LAUNCH("str_rank_heads", k_str_rank_heads, tgrid, SR_THREADS, 0, p2, k1, v1, as<uint32_t>(A.values), as<uint32_t>(bid.values), as<uint32_t>(ord), nA, ntiles,
                   as<uint32_t>(rows), as<uint32_t>(heads), as<uint32_t>(cnt));
        exclusive_scan_u32_to_u64(as<uint32_t>(cnt), as<uint64_t>(toff), ntiles, as<uint64_t>(toff) + ntiles);
        PLB_LAUNCH("str_rank_apply", k_str_rank_apply, tgrid, SR_THREADS, 0, as<uint32_t>(heads), as<uint64_t>(toff), as<uint32_t>(rows), as<uint32_t>(A.values), nA, ntiles,
                   as<uint32_t>(ord), as<uint32_t>(nb), as<uint32_t>(keep));
        DevCol mask; mask.dtype = BL_BOOL; mask.len = nA; mask.values = keep; mask.null_count = 0;
        std::vector<DevCol> next;
        op_filter({A, u32_col(nb, nA)}, mask, next);
        A = next[0]; bid = next[1];
        nA = A.len;
    }
    // back to rows
    DevPtr rk = dev_alloc((size_t)n * 4 + 16);
    if (m > 0) PLB_LAUNCH("str_rank_scatter", k_str_rank_scatter, grid_for(m, 256), 256, 0, as<uint32_t>(ord), m, as<uint32_t>(rk));
    PLB_LAUNCH("str_rank_rows", k_str_rank_rows, grid_for(n, 256), 256, 0, as<uint32_t>(codes.values), s.vm(), as<uint32_t>(rk), n, descending ? 1 : 0, (uint32_t)m,
               as<uint32_t>(out.values));
    return out;
}

}  // namespace plb

// ================================================================================ C ABI
using namespace plb;
extern "C" {

bl_status bl_string_rank(const bl_string_column* chunks, int32_t n_chunks, int32_t descending, int32_t out_location, bl_column* out_rank, int64_t* n_distinct) {
    BL_TRY
    PLB_REQUIRE(out_rank != nullptr, BL_ERR_INVALID, "string_rank: null output");
    DevStr s = import_string(chunks, n_chunks);
    int64_t nd = 0;
    DevCol rk = op_string_rank(s, descending != 0, &nd);
    export_column(rk, out_location, out_rank);
    if (n_distinct) *n_distinct = nd;
    BL_CATCH
}

bl_status bl_arg_sort_keys(const bl_sort_key* by, int32_t n_by, int64_t limit, int32_t out_location, bl_column* out_idx) {
    BL_TRY
    PLB_REQUIRE(out_idx != nullptr, BL_ERR_INVALID, "arg_sort_keys: null output");
    PLB_REQUIRE(by != nullptr && n_by >= 1, BL_ERR_INVALID, "arg_sort_keys: no key column");
    int64_t n0 = -1;
    for (int i = 0; i < n_by; i++) {
        const bl_sort_key& k = by[i];
        PLB_REQUIRE((k.column != nullptr) != (k.strings != nullptr), BL_ERR_INVALID,
                    "arg_sort_keys: key " + std::to_string(i) + " must set exactly one of `column` and `strings`");
        int64_t len = 0;
        if (k.column) len = k.column->length;
        else {
            PLB_REQUIRE(k.n_chunks >= 1, BL_ERR_INVALID, "arg_sort_keys: string key " + std::to_string(i) + " has no chunks");
            for (int j = 0; j < k.n_chunks; j++) len += k.strings[j].length;
        }
        if (n0 < 0) n0 = len;
        PLB_REQUIRE(len == n0, BL_ERR_INVALID, "arg_sort_keys: key columns differ in length (" + std::to_string(len) + " != " + std::to_string(n0) + ")");
    }
    std::vector<DevCol> keys; std::vector<int> fl;
    for (int i = 0; i < n_by; i++) {
        keys.push_back(by[i].column ? import_column(by[i].column, 1) : op_string_rank(import_string(by[i].strings, by[i].n_chunks), false, nullptr));
        fl.push_back(by[i].flags);
    }
    DevCol perm = op_arg_sort(keys, fl, limit);
    export_column(perm, out_location, out_idx);
    BL_CATCH
}

}  // extern "C"
