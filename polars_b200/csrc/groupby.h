// groupby.h — shared definitions + host-side state of the fused hash group_by (K5); see groupby.cu.
#pragma once
#include <cstdlib>
#include <type_traits>

#include "common.cuh"

namespace plb {

// tuning knobs (environment variables): read on every call, so that they can change between calls
inline int knob_int(const char* name, int dflt) { const char* e = getenv(name); return e ? atoi(e) : dflt; }
inline double knob_double(const char* name, double dflt) { const char* e = getenv(name); return e ? atof(e) : dflt; }

// ---- host dispatch onto kernel template arguments: f receives std::integral_constant arguments
template <int V> using IntC = std::integral_constant<int, V>;
// key form of a key dtype: f(element size 4 / 8, canonicalisation 0 raw bits / 1 f64 / 2 f32)
template <class F> void with_key_form(int key_dtype, F&& f) {
    if (dtype_size(key_dtype) == 8) { if (key_dtype == BL_FLOAT64) f(IntC<8>{}, IntC<1>{}); else f(IntC<8>{}, IntC<0>{}); }
    else { if (key_dtype == BL_FLOAT32) f(IntC<4>{}, IntC<2>{}); else f(IntC<4>{}, IntC<0>{}); }
}
// f(the first V of Vs with n <= V; the last one otherwise)
template <int V, int... Vs, class F> void with_at_least(int n, F&& f) {
    if constexpr (sizeof...(Vs) == 0) f(IntC<V>{});
    else if (n <= V) f(IntC<V>{});
    else with_at_least<Vs...>(n, f);
}
template <class F> void with_bool(bool b, F&& f) { if (b) f(std::true_type{}); else f(std::false_type{}); }

constexpr uint64_t GB_EMPTY = 0x8000000000000000ULL;   // i64::MIN / -0.0 bits (never a canonical float key)
constexpr uint64_t GB_W1_INIT = 0xFFFFFFFF00000000ULL;  // first = u32::MAX, len = 0
constexpr int GB_MAX_COLS = 8;
constexpr int GB_MAX_WORDS = 14;
constexpr int GB_MAX_PROBE = 1024;
constexpr int GB_WINDOW_HEADER_WORDS = 128;   // peer-window half: [src * 2] = rows sent by rank src, [src * 2 + 1] = epoch flag; regions follow

enum WordOp { W_ADD_INT = 0, W_ADD_F64 = 1, W_MIN_S64 = 2, W_MAX_S64 = 3, W_MIN_U64 = 4, W_MAX_U64 = 5, W_MIN_F64 = 6, W_MAX_F64 = 7, W_NULLCNT = 8 };

struct GbColDev { const void* values; const uint32_t* validity; int32_t dtype; int32_t elem; };
struct GbLayout {
    int32_t stride, n_words, n_cols, need_len, need_first;
    int32_t pair_k, pair_c;           // per batch: iteration index k (and its column) of the accumulator that shares a 16-byte cell with word 1 (-1: none)
    int32_t wslot[GB_MAX_WORDS];      // iteration order k -> accumulator word index (table word = 2 + slot)
    int32_t wop[GB_MAX_WORDS];        // iteration order k -> WordOp
    int32_t col_kbegin[GB_MAX_COLS + 1];
    int32_t slot_op[GB_MAX_WORDS];    // word index -> WordOp (merge / init)
    uint64_t init[GB_MAX_WORDS];      // word index -> identity
};
// word w of entry s: entries[s * es + w * ws]  (AoS: es = stride, ws = 1;  word-major planes: es = 1, ws = cap + 2).
// Pair layout (pw != 0, word-major only): word 1 (len | first) and accumulator word pw (a 64-bit integer sum) of slot s share the
// 16-byte cell entries[ws + 2 s .. ws + 2 s + 1] (planes 1 and 2 of the word-major form), so that ONE bulk reduce
// (cp.reduce.async.bulk .add.u64, 16 bytes) updates both; word 2, if it is not pw itself, moves to plane pw.  gb_woff() is the
// only place that knows this.
struct GbTableDev { uint64_t* entries; uint64_t cap; int64_t es, ws; int32_t shift; int32_t soa; int32_t* status; int32_t hint; int32_t pass_bits; int32_t pass_id; int32_t pw; int32_t bulk_lanes; int32_t pad; };
// offset of word w of slot s, in words from (entries + s * es)
__host__ __device__ __forceinline__ int64_t gb_woff(int64_t s, int w, int64_t ws, int pw) {
    if (pw) {
        if (w == 1 || w == pw) return ws + s + (w != 1);
        if (w == 2) w = pw;
    }
    return (int64_t)w * ws;
}
struct GbBatch {
    const void* keys; const uint32_t* key_validity; int64_t n; uint32_t row_base; int32_t key_dtype;
    GbColDev cols[GB_MAX_COLS];
};


// Heavy-hitter keys (skewed distributions): the rows of a hot key would serialise on one L2 address
// (a few ns per same-address RED: Zipf(1.1) keys take an order of magnitude longer than uniform keys).
// k_gb_consume_hot aggregates them in warp-private shared-memory rows instead; see groupby.cu.
constexpr int GB_HOT_MAX = 62;              // hot keys (+2 rows: the null-key and the GB_EMPTY-key group)
constexpr int GB_HOT_BITS = 8;
constexpr int GB_HOT_SLOTS = 1 << GB_HOT_BITS;   // lookup table slots (open addressing, <= 25 % full)
struct GbHotDev { const uint64_t* keys; const uint8_t* idx; int32_t n_hot, null_hot, empty_hot, rows; };

// dense per-group arrays (the layout k_gb_extract produces): filled directly by the partitioned plan (groupby_radix.cu)
struct GbDense { DevPtr keys, first, len, words, ctl; int64_t Gb = 0; bool ready = false; };

struct AggPlan { int kind, in_dtype, out_dtype; int main, nullcnt; bool nullable; };

// Host mirror of group_by_helper (crates/polars-mem-engine/src/executors/group_by.rs:60-98): owns
// the device hash table and the aggregation plan.
struct GroupByState {
    int key_dtype;
    std::vector<int> agg_kinds, agg_dtypes;
    int64_t expected_groups;
    std::vector<AggPlan> plans;
    GbLayout L;
    bool lean_shape = false;     // the first batch had the shape of k_gb_consume_lean (note_batch_shape)
    int pair_word = 0;           // table word (>= 2) of the first 64-bit integer sum when len is tracked too: candidates for the pair layout
    GbTableDev T{};
    DevPtr entries, status;
    uint64_t cap = 0;
    int64_t rows_seen = 0;
    int64_t merged_rows = 0;     // partial-aggregate rows merged in (bounds the group count together with rows_seen)
    int64_t est_groups = 0;      // sampled / hinted cardinality; selects the shared-memory plan
    double sample_adjacent = 0;  // sampled fraction of rows whose successor carries the same key (skew / sortedness)
    double est_f2 = 0;           // sampled sum over groups of (rows in the group)^2 in the batch (0: not sampled); sizes K5r's bucket streams
    // sampled ranges for K5r's packed records (choose_cap): the key fits the window of 2^32 - 1 offsets from pack_base,
    // and the 8-byte integer value columns in pack_cols fit 32 bits (Int64 within +-2^30, UInt64 below 2^31)
    bool pack_key = false;
    uint64_t pack_base = 0;
    std::vector<const void*> pack_cols;
    GbHotDev hot{};              // heavy hitters found in the sample (rows == 0: none)
    double hot_share = 0;        // sampled share of the hottest key
    DevPtr hot_buf;

    GroupByState(int key_dt, const std::vector<int>& kinds, const std::vector<int>& dtypes, const std::vector<int>& nullable, int64_t expected, bool track_first);
    void consume_all(const DevCol& key, const std::vector<const DevCol*>& values);
    bool consume_radix(const DevCol& key, const std::vector<const DevCol*>& values, uint64_t planned_cap);   // partitioned plan (tables beyond L2); false = not applicable
    GbDense dense;               // set by consume_radix: finish() takes the groups from here, there is no table
    void consume_pipelined(const DevCol& key, const std::vector<const DevCol*>& values, int64_t chunk_rows, const std::vector<cudaEvent_t>& ready);
    void consume(const DevCol& key, const std::vector<const DevCol*>& values, int64_t row_base);
    void merge_partials(const uint64_t* rows, int64_t n_rows);
    void merge_partial_regions(const uint64_t* const* ptrs, const int64_t* counts, int n_regions);
    DevPtr export_partials(int n_partitions, int* row_words_out, int64_t* offsets_host);
    void export_partials_p2p(int n_ranks, int my_rank, void* const* windows, int64_t rows_per_src, int* row_words_out, int64_t* sent_rows);
    void export_partials_p2p_async(int n_ranks, int my_rank, void* const* window_halves, int64_t rows_per_src, uint64_t epoch, int* row_words_out);
    void merge_window_async(const void* own_half, int n_ranks, int64_t rows_per_src, uint64_t epoch);
    void settle();               // resolves a deferred one-shot overflow check now (host sync); for users of the table that skip finish()
    int read_status();           // host sync: 0 ok, 1 table overflow, 2 peer window overflow, 3 peer timeout
    bool defer_status = false;   // consume() leaves the overflow check to read_status() / finish()
    // one-shot consume_all: the overflow check rides on finish()'s synchronisation; on overflow finish() redoes the batch
    const DevCol* redo_key = nullptr; std::vector<const DevCol*> redo_values; uint64_t redo_cap = 0;
    void finish(bool maintain_order, const DevCol* key_col_for_gather, DevCol& out_key, std::vector<DevCol>& out_aggs, DevCol* out_first = nullptr);
    void reset();
    int64_t count_groups();

   private:
    void alloc_table(uint64_t new_cap);
    int smem_table_cap() const;
    bool bind_columns(const DevCol& key, const std::vector<const DevCol*>& values, int64_t row_base, int pw, int max_cols, GbBatch& B, GbLayout& Lb,
                      const void* first_col = nullptr) const;
    void note_batch_shape(const DevCol& key, const std::vector<const DevCol*>& values);
    uint64_t choose_cap(const DevCol& key, int64_t n_total, const std::vector<const DevCol*>* values = nullptr);
    void build_hot_list(const void* candidates, int n_cand, bool null_hot, bool empty_hot, double sample_rows);
    void launch_batch(const DevCol& key, const std::vector<const DevCol*>& values, int64_t row_base);
    void grow(uint64_t new_cap);
};

}  // namespace plb
