// sort.cu — multi-column arg_sort / sort on the device: order-preserving key encoding + the stable LSD radix sort.
//
// Reference: DataFrame::sort_impl polars-core/src/frame/mod.rs:1432-1561 (rechunk, IdxSize permutation, take),
// arg_sort / arg_sort_multiple polars-core/src/chunked_array/ops/sort/arg_sort.rs:118-185,
// arg_sort_multiple.rs:66-75, SortMultipleOptions options.rs:85-105, value order reorder_cmp
// polars-utils/src/sort.rs:113-128 (floats by tot_cmp: NaN == NaN and greatest, -0.0 == +0.0; nulls placed by
// nulls_last only, never by descending).
//
// Design: columns are processed as an LSD sequence, last column first, starting from iota.  Every column is one or
// two stable radix stages on the permutation built so far:
//   value stage  k_sort_encode reads col[perm[i]] (a fused gather) and writes an order-preserving unsigned key
//                (u32 for 8/16/32-bit types and Bool, u64 for 64-bit types; descending = inverted bits; null rows = 0),
//                reducing the AND and OR of the valid rows' keys on the way; digits where AND == OR are the same in every
//                valid row and are not sorted on (null rows may differ there: the null stage puts them in place anyway).
//   null stage   only for a column with a validity bitmap: a 1-bit key (null rank from nulls_last) sorted after the
//                value stage, so it is the more significant part.  Nulls share value key 0, so their relative order is
//                the order the earlier stages left (later columns, then row index) — as the reference's tie rule.
// Every stage is stable, so the result is THE stable order (what the reference returns whenever it pins the order).
// Algorithmic bytes per stage: encode 4 + elem + (key bytes) per row (+4 for the first stage's iota), then per radix
// pass 2 * (key bytes + 4) per row plus one key read for the histogram.
#include "common.cuh"
#include "dev_utils.cuh"
#include "sort_keys.cuh"

namespace plb {

// NULL_STAGE: key = null rank (nulls_last: valid 0 / null 1; else valid 1 / null 0).  Otherwise the value key.
// perm == nullptr: the identity (first stage), and iota_out receives it.  andor[0] &= keys, andor[1] |= keys (value stage:
// valid rows only).
template <typename K, bool NULL_STAGE>
__global__ void __launch_bounds__(256) k_sort_encode(const void* __restrict__ col, const uint32_t* __restrict__ valid, const uint32_t* __restrict__ perm, uint32_t* __restrict__ iota_out,
                                                     int64_t n, int dtype, int descending, int nulls_last, K* __restrict__ out, unsigned long long* __restrict__ andor) {
    K a = ~K(0), o = K(0);
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t r = perm ? (int64_t)perm[i] : i;
        if (!perm && iota_out) iota_out[i] = (uint32_t)i;
        const bool ok = valid == nullptr || bit_get(valid, r);
        K k;
        if (NULL_STAGE) k = (K)((ok ? 0u : 1u) ^ (nulls_last ? 0u : 1u));
        else k = ok ? (K)(descending ? ~sort_value_key(col, r, dtype) : sort_value_key(col, r, dtype)) : K(0);
        out[i] = k;
        if (NULL_STAGE || ok) { a &= k; o |= k; }      // null rows' key 0 must not make a digit look varying: the null stage orders them
    }
    __shared__ unsigned long long s_and[8], s_or[8];
    const unsigned lane = lane_id(), warp = threadIdx.x >> 5;
    uint64_t a64 = (uint64_t)a, o64 = (uint64_t)o;
    const uint32_t al = __reduce_and_sync(0xffffffffu, (uint32_t)a64), ah = __reduce_and_sync(0xffffffffu, (uint32_t)(a64 >> 32));
    const uint32_t ol = __reduce_or_sync(0xffffffffu, (uint32_t)o64), oh = __reduce_or_sync(0xffffffffu, (uint32_t)(o64 >> 32));
    if (lane == 0) { s_and[warp] = ((uint64_t)ah << 32) | al; s_or[warp] = ((uint64_t)oh << 32) | ol; }
    __syncthreads();
    if (threadIdx.x == 0) {
        unsigned long long ba = ~0ull, bo = 0;
        for (int w = 0; w < 8; w++) { ba &= s_and[w]; bo |= s_or[w]; }
        if (sizeof(K) == 4) { ba &= 0xFFFFFFFFull; }
        atomicAnd(&andor[0], ba); atomicOr(&andor[1], bo);
    }
}

bool radix_sort_pairs_u32(uint32_t* k0, uint32_t* v0, uint32_t* k1, uint32_t* v1, int64_t n, uint64_t vary, int* passes_run);
bool radix_sort_pairs_u64(uint64_t* k0, uint32_t* v0, uint64_t* k1, uint32_t* v1, int64_t n, uint64_t vary, int* passes_run);

bool sortable_dtype(int dt) { return (dt >= BL_INT8 && dt <= BL_FLOAT64) || dt == BL_BOOL; }

// limit <= n / SORT_SELECT_DIV takes the selection plan: op_top_k, a gather of the keys at the selected rows, the stable
// sort of those rows and a gather of the row ids (DESIGN.md §17 measures both sides).  Only for keys the K4 gather moves
// (4- and 8-byte dtypes); 1- / 2-byte and Bool keys keep the full sort.
constexpr int64_t SORT_SELECT_DIV = 8;
// a measurement knob (read per call, as BL_QUANTILE_GLOBAL is): BL_SORT_SELECT_DIV = d selects for limit <= n / d, 0 never
static bool select_for_limit(int64_t limit, int64_t n) {
    const char* e = getenv("BL_SORT_SELECT_DIV");
    const long d = e ? atol(e) : SORT_SELECT_DIV;
    return limit >= 0 && d >= 1 && limit <= n / d;
}
static bool selection_gathers(const std::vector<DevCol>& by) {
    for (auto& c : by)
        if (dtype_size(c.dtype) != 4 && dtype_size(c.dtype) != 8) return false;
    return true;
}

DevCol op_arg_sort(const std::vector<DevCol>& by, const std::vector<int>& flags, int64_t limit) {
    PLB_REQUIRE(!by.empty(), BL_ERR_INVALID, "arg_sort: no key column");
    PLB_REQUIRE(flags.size() == by.size(), BL_ERR_INVALID, "arg_sort: one flag word per key column");
    const int64_t n = by[0].len;
    for (auto& c : by) {
        PLB_REQUIRE(c.len == n, BL_ERR_INVALID, "arg_sort: key columns differ in length (" + std::to_string(c.len) + " != " + std::to_string(n) + ")");
        PLB_REQUIRE(sortable_dtype(c.dtype), BL_ERR_UNSUPPORTED, std::string("arg_sort: key dtype ") + dtype_name(c.dtype) + " is not supported");
    }
    PLB_REQUIRE(n <= (int64_t)0xFFFFFFFFll, BL_ERR_UNSUPPORTED, "arg_sort: more than 2^32 - 1 rows (IdxSize is u32)");
    if (select_for_limit(limit, n) && selection_gathers(by)) {
        // the selected rows ascend and keep their keys' encoding, so the stable sort of them is the stable order's first
        // `limit` rows: the same bytes as the full sort below
        const DevCol ids = op_top_k(by, flags, limit);
        std::vector<DevCol> sub, composed;
        if (ids.len) op_gather(by, ids, false, sub);
        if (sub.empty()) return ids;
        const DevCol perm = op_arg_sort(sub, flags, -1);
        op_gather({ids}, perm, false, composed);
        return composed[0];
    }
    DevCol out;
    out.dtype = BL_UINT32; out.null_count = 0;
    out.len = limit < 0 ? n : std::min<int64_t>(limit, n);
    DevPtr cur = dev_alloc((size_t)n * 4);
    out.values = cur;
    if (n == 0) return out;
    DevPtr alt = dev_alloc((size_t)n * 4), ka = dev_alloc((size_t)n * 8), kb = dev_alloc((size_t)n * 8), andor = dev_alloc(16);
    bool have_perm = false;
    const int grid = grid_for(n, 256);
    for (int c = (int)by.size() - 1; c >= 0; c--) {
        const DevCol& col = by[c];
        const int desc = (flags[c] & BL_SORT_DESCENDING) != 0, nl = (flags[c] & BL_SORT_NULLS_LAST) != 0;
        for (int stage = 0; stage < (col.validity ? 2 : 1); stage++) {
            const bool null_stage = stage == 1;
            const bool wide = !null_stage && dtype_size(col.dtype) == 8;
            dev_memset(andor->p, 0xFF, 8);
            dev_memset((char*)andor->p + 8, 0, 8);
            const uint32_t* perm = have_perm ? as<uint32_t>(cur) : nullptr;
            uint32_t* iota = have_perm ? nullptr : as<uint32_t>(cur);
            if (wide) PLB_LAUNCH("sort_encode", (k_sort_encode<uint64_t, false>), grid, 256, 0, col.v(), col.vm(), perm, iota, n, col.dtype, desc, nl, as<uint64_t>(ka), as<unsigned long long>(andor));
            else if (null_stage) PLB_LAUNCH("sort_encode_nulls", (k_sort_encode<uint32_t, true>), grid, 256, 0, col.v(), col.vm(), perm, iota, n, col.dtype, desc, nl, as<uint32_t>(ka), as<unsigned long long>(andor));
            else PLB_LAUNCH("sort_encode", (k_sort_encode<uint32_t, false>), grid, 256, 0, col.v(), col.vm(), perm, iota, n, col.dtype, desc, nl, as<uint32_t>(ka), as<unsigned long long>(andor));
            have_perm = true;
            uint64_t ao[2];
            PLB_CUDA(cudaMemcpyAsync(ao, andor->p, 16, cudaMemcpyDeviceToHost, ctx().stream));
            PLB_CUDA(cudaStreamSynchronize(ctx().stream));
            // bits that differ between at least two (valid) rows; AND not contained in OR = no row was reduced (all null)
            const uint64_t vary = (ao[0] & ~ao[1]) ? 0 : ao[0] ^ ao[1];
            if (vary == 0) continue;
            const bool swapped = wide ? radix_sort_pairs_u64(as<uint64_t>(ka), as<uint32_t>(cur), as<uint64_t>(kb), as<uint32_t>(alt), n, vary, nullptr)
                                      : radix_sort_pairs_u32(as<uint32_t>(ka), as<uint32_t>(cur), as<uint32_t>(kb), as<uint32_t>(alt), n, vary, nullptr);
            if (swapped) std::swap(cur, alt);
        }
    }
    out.values = cur;
    return out;      // alt and the key buffers go back to the pool here
}

void op_sort(const std::vector<DevCol>& by, const std::vector<int>& flags, const std::vector<DevCol>& cols, int64_t limit, std::vector<DevCol>& outs) {
    const int64_t n = by.empty() ? 0 : by[0].len;
    for (auto& c : cols) {
        PLB_REQUIRE(c.len == n, BL_ERR_INVALID, "sort: payload column length " + std::to_string(c.len) + " != key length " + std::to_string(n));
        PLB_REQUIRE(dtype_size(c.dtype) == 8 || dtype_size(c.dtype) == 4, BL_ERR_UNSUPPORTED, std::string("sort: payload dtype ") + dtype_name(c.dtype) + " is outside the gather hot path");
    }
    DevCol perm = op_arg_sort(by, flags, limit);
    outs.clear();
    if (!cols.empty()) op_gather(cols, perm, false, outs);      // only the first `limit` rows are gathered
}

}  // namespace plb
