// unique.cu — DataFrame.unique / drop_duplicates, Series.unique / arg_unique and the is_unique / is_duplicated /
// is_first_distinct / is_last_distinct masks.
//
// Reference: DataFrame::unique_impl polars-core/src/frame/mod.rs:2317-2392 (First / Any: the group firsts; Last with
// maintain_order: the groups' last rows sorted ascending; None: filter(is_unique); unstable variants: the same rows in an
// open order; `slice` applies to that result), is_unique / is_duplicated frame/mod.rs:2408-2442 and
// polars-ops/src/series/ops/is_unique.rs:11-41,113-119, is_first_distinct is_first_distinct.rs:107-161, is_last_distinct
// is_last_distinct.rs:12-….  One answer serves every keep strategy: the kept rows as ascending row ids, exact for
// maintain_order and a valid order without it.  Key equality is the group_by one: null is a value, floats by total
// equality (canonical bits), strings by bytes, several columns form one row key.
//
// Plan (DESIGN.md §18):
//   key        one column: 4- / 8-byte numeric as is, 8- / 16-bit integers zero-extended (op_cast_small_int), strings as
//              their codes (op_string_codes), Boolean as a UInt8 0 / 1 column; several columns: op_pack_keys.
//   table      the K5 build with LEN and first tracking (the same state op_group_first_ids builds): word 1 of a slot holds
//              the key's first row and its row count; `len > 1` <=> the key has duplicates.  Its sizing, heavy-hitter,
//              shared-memory and overflow-redo plans apply; first tracking keeps the partitioned plan (K5r) out.
//   uniq_last  (LAST only) one thread per row raises last[slot] with atomicMax, one atomic per distinct slot of a warp.
//   uniq_mark  one warp per 32 consecutive rows: re-probes each row's slot and writes one bitmap word from the ballot of
//              FIRST (row == first), LAST (row == last), UNIQUE (len == 1) or DUPLICATED (len > 1).
//   ids        op_mask_rows compacts the bitmap into ascending row ids.
// Device memory: the K5 table, 4 (cap + 2) B of `last` (LAST only), n / 8 B of mask, 4 B per kept row.
#include "common.cuh"
#include "dev_utils.cuh"
#include "groupby.h"
#include "groupby_dev.cuh"
#include "strings.cuh"

namespace plb {

constexpr int UQ_THREADS = 256;

__global__ void __launch_bounds__(UQ_THREADS) k_bool_to_u8(const uint32_t* __restrict__ bits, int64_t n, uint8_t* __restrict__ out) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) out[i] = bit_get(bits, i) ? 1 : 0;
}

// last[slot] = the highest row holding the slot's key.  n_round: n rounded up to 32, so whole warps take part in the match.
__global__ void __launch_bounds__(UQ_THREADS) k_uniq_last(const __grid_constant__ GbTableDev T, const void* keys, const uint32_t* key_validity, int key_dtype, int64_t n,
                                                          int64_t n_round, uint32_t* __restrict__ last) {
    for (int64_t row = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; row < n_round; row += (int64_t)gridDim.x * blockDim.x) {
        const bool in = row < n;
        const uint64_t slot = in ? gb_lookup_slot(T, keys, key_validity, key_dtype, row) : ~0ull;
        const unsigned peers = __match_any_sync(0xffffffffu, slot);
        // the warp's rows ascend with the lane: the highest lane of a slot holds its highest row
        if (in && lane_id() == 31u - __clz(peers) && __ldcg(last + slot) < (uint32_t)row) atomicMax(last + slot, (uint32_t)row);
    }
}

template <int KIND>
__global__ void __launch_bounds__(UQ_THREADS) k_uniq_mark(const __grid_constant__ GbTableDev T, const void* keys, const uint32_t* key_validity, int key_dtype, int64_t n,
                                                          int64_t n_round, const uint32_t* __restrict__ last, uint32_t* __restrict__ mask) {
    for (int64_t row = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; row < n_round; row += (int64_t)gridDim.x * blockDim.x) {
        bool hit = false;
        if (row < n) {
            const uint64_t slot = gb_lookup_slot(T, keys, key_validity, key_dtype, row);
            if (KIND == BL_DISTINCT_LAST) hit = __ldcg(last + slot) == (uint32_t)row;
            else {
                const uint64_t w1 = gb_slot_word1(T, slot);
                if (KIND == BL_DISTINCT_FIRST) hit = (uint32_t)(w1 >> 32) == (uint32_t)row;
                else if (KIND == BL_DISTINCT_UNIQUE) hit = (uint32_t)w1 == 1u;
                else hit = (uint32_t)w1 > 1u;
            }
        }
        const unsigned b = __ballot_sync(0xffffffffu, hit);
        if (lane_id() == 0) mask[row >> 5] = b;
    }
}

// the subset columns -> one key column K5 takes
static DevCol unique_key(const std::vector<DevCol>& cols) {
    std::vector<DevCol> ks;
    for (const DevCol& c : cols) {
        if (c.dtype != BL_BOOL) { ks.push_back(c); continue; }
        DevCol u = make_col(BL_UINT8, c.len, false);
        u.validity = c.validity; u.null_count = c.null_count;
        if (c.len) PLB_LAUNCH("uniq_bool_key", k_bool_to_u8, grid_for(c.len, UQ_THREADS), UQ_THREADS, 0, as<uint32_t>(c.values), c.len, as<uint8_t>(u.values));
        ks.push_back(u);
    }
    if (ks.size() > 1) return op_pack_keys(ks);
    return dtype_is_small_int(ks[0].dtype) ? op_cast_small_int(ks[0], BL_UINT32, true) : ks[0];
}

// the BL_DISTINCT_* mask of the rows (BL_BOOL, n rows, no nulls)
DevCol op_unique_mask(const std::vector<DevCol>& cols, int kind) {
    PLB_REQUIRE(!cols.empty(), BL_ERR_INVALID, "unique: no key column");
    const int64_t n = cols[0].len;
    for (const DevCol& c : cols) PLB_REQUIRE(c.len == n, BL_ERR_INVALID, "unique: key columns differ in length (" + std::to_string(c.len) + " != " + std::to_string(n) + ")");
    PLB_REQUIRE(n <= 0xFFFFFFFEll, BL_ERR_UNSUPPORTED, "unique: more than 2^32 - 2 rows (IdxSize is u32)");
    DevCol mask = make_col(BL_BOOL, n, false);
    if (n == 0) return mask;
    const DevCol key = unique_key(cols);
    GroupByState st(key.dtype, {BL_AGG_LEN}, {BL_INT64}, {0}, 0, /*track_first=*/true);
    st.consume_all(key, {nullptr});
    st.settle();
    const int64_t n_round = (n + 31) / 32 * 32;
    const int grid = grid_for(n_round, UQ_THREADS, 16);
    DevPtr last;
    if (kind == BL_DISTINCT_LAST) {
        last = dev_alloc((size_t)(st.T.cap + 2) * 4);
        dev_memset(last->p, 0, (size_t)(st.T.cap + 2) * 4);
        PLB_LAUNCH("uniq_last", k_uniq_last, grid, UQ_THREADS, 0, st.T, key.v(), key.vm(), key.dtype, n, n_round, as<uint32_t>(last));
    }
    auto mark = [&](auto k) {
        PLB_LAUNCH("uniq_mark", k_uniq_mark<decltype(k)::value>, grid, UQ_THREADS, 0, st.T, key.v(), key.vm(), key.dtype, n, n_round, as<uint32_t>(last),
                   as<uint32_t>(mask.values));
    };
    switch (kind) {
        case BL_DISTINCT_FIRST: mark(IntC<BL_DISTINCT_FIRST>{}); break;
        case BL_DISTINCT_LAST: mark(IntC<BL_DISTINCT_LAST>{}); break;
        case BL_DISTINCT_UNIQUE: mark(IntC<BL_DISTINCT_UNIQUE>{}); break;
        case BL_DISTINCT_DUPLICATED: mark(IntC<BL_DISTINCT_DUPLICATED>{}); break;
        default: fail(BL_ERR_INVALID, "unique: unknown mask kind " + std::to_string(kind));
    }
    return mask;
}

// descriptor checks (before any column is read), then the key columns (strings: their codes)
static std::vector<DevCol> import_unique_keys(const bl_sort_key* keys, int32_t n_keys, const char* who) {
    const std::string w(who);
    PLB_REQUIRE(keys != nullptr && n_keys >= 1, BL_ERR_INVALID, w + ": no key column");
    int64_t n = -1;
    for (int i = 0; i < n_keys; i++) {
        const bl_sort_key& k = keys[i];
        const std::string ki = w + ": key " + std::to_string(i);
        PLB_REQUIRE((k.column != nullptr) != (k.strings != nullptr), BL_ERR_INVALID, ki + " must set exactly one of `column` and `strings`");
        PLB_REQUIRE(k.flags == 0, BL_ERR_INVALID, ki + ": flags must be 0");
        int64_t len = 0;
        if (k.column) {
            PLB_REQUIRE(sortable_dtype(k.column->dtype), BL_ERR_UNSUPPORTED, ki + ": dtype " + dtype_name(k.column->dtype) + " is not supported");
            len = k.column->length;
        } else {
            PLB_REQUIRE(k.n_chunks >= 1, BL_ERR_INVALID, ki + ": a string column without chunks");
            for (int j = 0; j < k.n_chunks; j++) len += k.strings[j].length;
        }
        if (n < 0) n = len;
        PLB_REQUIRE(len == n, BL_ERR_INVALID, w + ": key columns differ in length (" + std::to_string(len) + " != " + std::to_string(n) + ")");
    }
    PLB_REQUIRE(n <= 0xFFFFFFFEll, BL_ERR_UNSUPPORTED, w + ": more than 2^32 - 2 rows (IdxSize is u32)");
    std::vector<DevCol> cols;
    for (int i = 0; i < n_keys; i++) cols.push_back(import_key(keys[i], true));
    return cols;
}

}  // namespace plb

// ================================================================================ C ABI
using namespace plb;
extern "C" {

bl_status bl_unique(const bl_sort_key* subset, int32_t n_subset, int32_t keep, int32_t out_location, bl_column* out_idx) {
    BL_TRY
    PLB_REQUIRE(out_idx != nullptr, BL_ERR_INVALID, "unique: null output");
    PLB_REQUIRE(keep >= BL_UNIQUE_FIRST && keep <= BL_UNIQUE_NONE, BL_ERR_INVALID, "unique: unknown keep strategy " + std::to_string(keep));
    const std::vector<DevCol> cols = import_unique_keys(subset, n_subset, "unique");
    const int kind = keep == BL_UNIQUE_LAST ? BL_DISTINCT_LAST : keep == BL_UNIQUE_NONE ? BL_DISTINCT_UNIQUE : BL_DISTINCT_FIRST;
    const DevCol mask = op_unique_mask(cols, kind);
    export_column(op_mask_rows(as<uint32_t>(mask.values), mask.len), out_location, out_idx);
    BL_CATCH
}

bl_status bl_unique_mask(const bl_sort_key* keys, int32_t n_keys, int32_t kind, int32_t out_location, bl_column* out_mask) {
    BL_TRY
    PLB_REQUIRE(out_mask != nullptr, BL_ERR_INVALID, "unique_mask: null output");
    PLB_REQUIRE(kind >= BL_DISTINCT_FIRST && kind <= BL_DISTINCT_DUPLICATED, BL_ERR_INVALID, "unique_mask: unknown kind " + std::to_string(kind));
    export_column(op_unique_mask(import_unique_keys(keys, n_keys, "unique_mask"), kind), out_location, out_mask);
    BL_CATCH
}

}  // extern "C"
