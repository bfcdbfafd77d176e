// common.cuh — shared host/device utilities of libpolars_b200 (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <cstdio>
#include <cstring>
#include <memory>
#include <mutex>
#include <stdexcept>
#include <string>
#include <vector>

#include "../../include/polars_b200.h"

namespace plb {

// ------------------------------------------------------------------------------------------
// errors: C++ exceptions inside, bl_status + thread-local message at the C boundary
// ------------------------------------------------------------------------------------------
struct Error : std::runtime_error {
    bl_status code;
    Error(bl_status c, const std::string& m) : std::runtime_error(m), code(c) {}
};
[[noreturn]] inline void fail(bl_status c, const std::string& m) { throw Error(c, m); }

#define PLB_CUDA(expr)                                                                          \
    do {                                                                                        \
        cudaError_t _e = (expr);                                                                \
        if (_e != cudaSuccess) {                                                                \
            ::plb::fail(_e == cudaErrorMemoryAllocation ? BL_ERR_OOM : BL_ERR_CUDA,             \
                        std::string(#expr) + ": " + cudaGetErrorString(_e) + " (" + __FILE__ +  \
                            ":" + std::to_string(__LINE__) + ")");                              \
        }                                                                                       \
    } while (0)
#define PLB_REQUIRE(cond, code, msg)                 \
    do {                                             \
        if (!(cond)) ::plb::fail((code), (msg));     \
    } while (0)

inline int dtype_size(int dt) {
    switch (dt) {
        case BL_INT8: case BL_UINT8: return 1;
        case BL_INT16: case BL_UINT16: return 2;
        case BL_INT32: case BL_UINT32: case BL_FLOAT32: return 4;
        case BL_INT64: case BL_UINT64: case BL_FLOAT64: return 8;
        default: return 0;  // BL_BOOL: bit-packed
    }
}
inline bool dtype_is_float(int dt) { return dt == BL_FLOAT32 || dt == BL_FLOAT64; }
inline bool dtype_is_signed(int dt) { return dt <= BL_INT64; }
inline bool dtype_is_int(int dt) { return dt >= BL_INT8 && dt <= BL_UINT64; }
inline const char* dtype_name(int dt) {
    static const char* n[] = {"i8", "i16", "i32", "i64", "u8", "u16", "u32", "u64", "f32", "f64", "bool"};
    return (dt >= 0 && dt <= 10) ? n[dt] : "?";
}

// ------------------------------------------------------------------------------------------
// Context: one device, one compute stream, a stream-ordered memory pool, a pinned-host cache,
// per-kernel launch accounting (CUDA events on the compute stream).
// ------------------------------------------------------------------------------------------
struct KernelStat { std::string name; int64_t launches = 0; double ms = 0; };
struct Context {
    int device = -1;
    cudaStream_t stream = nullptr;
    cudaStream_t copy_stream = nullptr;
    int sm_count = 132;        // H100 SXM; ensure_init reads the device's own count
    int64_t l2_bytes = 0;
    bool profiling = false;
    bool deterministic = false;      // bl_set_deterministic / BL_DETERMINISTIC: group_by folds every group sequentially in row order
    int64_t launch_count = 0;
    std::vector<KernelStat> stats;
    struct Pending { int stat; cudaEvent_t a, b; };
    std::vector<Pending> pending;
    std::vector<cudaEvent_t> event_pool;
    std::recursive_mutex mu;

    int stat_index(const char* name);
    void begin_launch(const char* name, int& stat, cudaEvent_t& a, cudaEvent_t& b);
    void end_launch(int stat, cudaEvent_t a, cudaEvent_t b);
    void drain_events();
};
Context& ctx();          // throws BL_ERR_CUDA when no device / not initialisable
void ensure_init(int device);

// launch wrapper: counts every launch; times it when profiling is enabled
#define PLB_LAUNCH(NAME, KERNEL, GRID, BLOCK, SMEM, ...)                                   \
    do {                                                                                   \
        ::plb::Context& _c = ::plb::ctx();                                                 \
        int _st; cudaEvent_t _a = nullptr, _b = nullptr;                                   \
        _c.begin_launch(NAME, _st, _a, _b);                                                \
        KERNEL<<<(GRID), (BLOCK), (SMEM), _c.stream>>>(__VA_ARGS__);                       \
        _c.end_launch(_st, _a, _b);                                                        \
        PLB_CUDA(cudaGetLastError());                                                      \
    } while (0)

// ------------------------------------------------------------------------------------------
// Device memory (stream-ordered pool) and pinned host memory (cached)
// ------------------------------------------------------------------------------------------
void* dev_alloc_raw(size_t bytes);
void dev_free_raw(void* p);
void* pinned_alloc_raw(size_t bytes);
void pinned_free_raw(void* p);

struct DevMem {
    void* p = nullptr; size_t bytes = 0; bool owned = true;
    DevMem() = default;
    DevMem(void* q, size_t b, bool o) : p(q), bytes(b), owned(o) {}
    ~DevMem() { if (owned && p) dev_free_raw(p); }
    DevMem(const DevMem&) = delete; DevMem& operator=(const DevMem&) = delete;
};
using DevPtr = std::shared_ptr<DevMem>;
inline DevPtr dev_alloc(size_t bytes) { return std::make_shared<DevMem>(dev_alloc_raw(bytes ? bytes : 16), bytes, true); }
inline DevPtr dev_borrow(const void* p, size_t bytes) { return std::make_shared<DevMem>(const_cast<void*>(p), bytes, false); }
template <typename T> inline T* as(const DevPtr& d) { return d ? reinterpret_cast<T*>(d->p) : nullptr; }

// A device-resident column: offset 0, validity bitmap (32-bit-word padded) or none.
struct DevCol {
    int dtype = BL_INT64;
    int64_t len = 0;
    DevPtr values;     // len * dtype_size bytes (BL_BOOL: bitmap, padded to 4-byte words)
    DevPtr validity;   // bitmap padded to 4-byte words, or null
    int64_t null_count = -1;
    const void* v() const { return values ? values->p : nullptr; }
    const uint32_t* vm() const { return validity ? reinterpret_cast<const uint32_t*>(validity->p) : nullptr; }
};
inline size_t bitmap_bytes(int64_t bits) { return (size_t)((bits + 31) / 32) * 4; }

// bl_column (host/device, chunked, arbitrary offset)  <->  DevCol
DevCol import_column(const bl_column* chunks, int n_chunks);
void export_column(const DevCol& c, int location, bl_column* out, bool sync = true);
void export_many(const std::vector<DevCol>& cols, int location, bl_column* outs);   // one sync for all
DevCol make_col(int dtype, int64_t len, bool with_validity);

// small device scalar readback (sync on compute stream)
template <typename T> T read_scalar(const T* dev) {
    T h; PLB_CUDA(cudaMemcpyAsync(&h, dev, sizeof(T), cudaMemcpyDeviceToHost, ctx().stream));
    PLB_CUDA(cudaStreamSynchronize(ctx().stream)); return h;
}
inline void dev_memset(void* p, int v, size_t bytes) { if (bytes) PLB_CUDA(cudaMemsetAsync(p, v, bytes, ctx().stream)); }

inline int grid_for(int64_t work_items, int block, int per_sm_blocks = 8) {
    int64_t need = (work_items + block - 1) / block;
    int64_t cap = (int64_t)ctx().sm_count * per_sm_blocks;
    if (need < 1) need = 1;
    return (int)(need < cap ? need : cap);
}

// ---- operators (device-resident in/out) -----------------------------------------------------
DevCol op_elementwise(int op, const DevCol& lhs, const DevCol& rhs);
DevCol op_compare(int op, const DevCol& lhs, const DevCol& rhs, bool missing);
void op_filter(const std::vector<DevCol>& cols, const DevCol& mask, std::vector<DevCol>& outs);
DevCol op_cmp_scalar_mask(const DevCol& col, int cmp_op, const DevCol& scalar);
// find_sentinel: scan an index column without nulls for BL_IDX_NULL (implied by check_bounds)
void op_gather(const std::vector<DevCol>& cols, const DevCol& idx, bool check_bounds, std::vector<DevCol>& outs, bool find_sentinel = false);
bool dtype_is_small_int(int dt);
DevCol op_cast_small_int(const DevCol& in, int to_dtype, bool bits);
DevCol op_group_first_ids(const DevCol& key);
DevCol op_pack_keys(const std::vector<DevCol>& keys);
void op_group_tuples(const DevCol& key, DevCol& out_first, DevCol& out_offsets, DevCol& out_all);
// op_group_tuples from the row -> first-row group ids; ids is sorted in place (on return ids[p] is the group of out_all[p])
void op_group_tuples_ids(DevCol& ids, DevCol& out_first, DevCol& out_offsets, DevCol& out_all);
// groups of an order whose group ids ascend: out_offsets = the positions where sorted_ids changes (+ n), out_first = all there
void op_group_offsets(const DevCol& sorted_ids, const DevCol& all, DevCol& out_first, DevCol& out_offsets);
// the sequential per-group folds of op_group_by_exact over given groups: group g owns rows all[offsets[g] .. offsets[g+1])
void op_group_fold(const DevCol& offsets, const DevCol& all, const std::vector<int>& kinds, const std::vector<const DevCol*>& values, std::vector<DevCol>& outs,
                   const bl_agg_param* params = nullptr);
// deterministic mode: GroupsIdx + one sequential fold per group in the reference's order (groupby_exact.cu)
// params[i] (quantile, method) is read where kinds[i] == BL_AGG_QUANTILE; nullptr = none given
void op_group_by_exact(const DevCol& key, const std::vector<int>& kinds, const std::vector<const DevCol*>& values, DevCol& out_first, std::vector<DevCol>& outs,
                       const bl_agg_param* params = nullptr);
// per-group quantiles over GroupsIdx (offsets: G + 1 entries, all: row lists; quantile.cu): outs[k] = quantile qs[k] with methods[k]
void op_group_quantiles(const DevCol& offsets, const DevCol& all, const DevCol& values, const std::vector<double>& qs, const std::vector<int>& methods,
                        std::vector<DevCol>& outs);
DevPtr bitmap_and(const uint32_t* a, const uint32_t* b, const uint32_t* c, int64_t bits);
int64_t bitmap_popcount(const uint32_t* bm, int64_t bits);
DevPtr bitmap_slice(const uint32_t* bm, int64_t pos, int64_t len);      // bits [pos, pos + len) as a fresh word-aligned bitmap
void exclusive_scan_u32_to_u64(const uint32_t* in, uint64_t* out, int64_t n, uint64_t* total_dev);
void exclusive_scan_u64(const uint64_t* in, uint64_t* out, int64_t n, uint64_t* total_dev);
void sort_pairs_u32(uint32_t* keys, uint32_t* vals, int64_t n, int key_bits = 32);   // stable LSD radix sort on the low key_bits, ascending (device)
// multi-column arg_sort (sort.cu): flags[i] = BL_SORT_* of by[i]; the UInt32 permutation, truncated to limit (< 0: all rows)
DevCol op_arg_sort(const std::vector<DevCol>& by, const std::vector<int>& flags, int64_t limit);
void op_sort(const std::vector<DevCol>& by, const std::vector<int>& flags, const std::vector<DevCol>& cols, int64_t limit, std::vector<DevCol>& outs);
bool sortable_dtype(int dt);      // the key dtypes op_arg_sort and op_top_k take (sort.cu)
// the first k rows of op_arg_sort's stable order, as ascending UInt32 row ids (top_k.cu)
DevCol op_top_k(const std::vector<DevCol>& by, const std::vector<int>& flags, int64_t k);
DevCol op_mask_rows(const uint32_t* mask, int64_t n);      // the ascending row ids of the set bits (filter.cu)
// the BL_DISTINCT_* mask of the rows keyed by cols (numeric / Boolean columns or string codes; unique.cu): BL_BOOL, no nulls
DevCol op_unique_mask(const std::vector<DevCol>& cols, int kind);
void mask_first_into(const uint32_t* mask, int64_t n, int64_t count, uint32_t* out);      // out |= the first `count` set bits of mask (filter.cu)
// bl_sort_key descriptors -> key columns (string keys as their ascending dense rank) and flags; who: the message prefix
void import_sort_key_list(const bl_sort_key* by, int32_t n_by, const char* who, std::vector<DevCol>& keys, std::vector<int>& flags);
void iota_u32(uint32_t* p, int64_t n, uint32_t base);
inline int bits_for(uint64_t max_value) { int b = 1; while (b < 32 && (max_value >> b)) b++; return b; }   // digits the radix sort has to look at

// window functions (window.cu): one output row per input row for every op; values NULL only for BL_AGG_LEN
struct OverOp { int kind = 0; bool reverse = false; int64_t periods = 0; const DevCol* values = nullptr; bl_agg_param param{0.5, BL_QUANTILE_LINEAR, 0}; };
void check_over_op(int kind_word, int value_dtype);      // BL_ERR_INVALID / BL_ERR_UNSUPPORTED of one op (value_dtype < 0: none)
std::vector<DevCol> op_over(const std::vector<DevCol>& partition_by, const DevCol* order_key, int order_flags, const std::vector<OverOp>& ops, int64_t n);
int over_scan_dtype(int kind, int dtype);      // output dtype of BL_CUM_* / BL_SHIFT
// the partition order shared by bl_over and bl_rolling (window.cu)
struct OverOrder {
    DevCol gid;               // row -> first row of its partition (UInt32)
    DevCol perm, seg, offsets, inv;     // partition order, its group id per position, segment offsets (G + 1), inverse permutation
    int64_t G = 0;
};
DevCol partition_ids(const std::vector<DevCol>& partition_by, int64_t n);      // row -> first row of its partition
void build_order(OverOrder& o, const DevCol* order_key, int order_flags, bool need_inv);      // o.gid set by the caller
DevCol import_key(const bl_sort_key& k, bool partition);      // partition: string codes; else: string ranks
// argument checks of bl_over / bl_rolling (who: the message prefix); n: the common row count, -1 until a column sets it
void set_window_len(const char* who, int64_t len, const std::string& what, int64_t& n);
void check_window_keys(const char* who, const bl_sort_key* partition_by, int32_t n_partition_by, const bl_sort_key* order_by, int64_t& n);
// rolling windows (rolling.cu)
struct RollOp { int kind = 0; bool center = false; int64_t window_size = 1, min_samples = 1; int ddof = 1; const DevCol* values = nullptr; };
void check_rolling_op(int kind, int center, int64_t window_size, int64_t min_samples, int ddof, int reserved, int value_dtype);
int rolling_dtype(int kind, int dtype);
std::vector<DevCol> op_rolling(const std::vector<DevCol>& partition_by, const DevCol* order_key, int order_flags, const std::vector<RollOp>& ops, int64_t n);
// time-based rolling windows (rolling_by.cu)
struct RollByOp { int kind = 0; int closed = 0; int64_t window_size = 1, min_samples = 1; int ddof = 1; const DevCol* values = nullptr; };
void check_rolling_by_op(int kind, int closed, int64_t window_size, int64_t min_samples, int ddof, int reserved, int value_dtype);
std::vector<DevCol> op_rolling_by(const std::vector<DevCol>& partition_by, const DevCol& by, const std::vector<RollByOp>& ops, int64_t n);
// rolling quantile (rolling_quantile.cu): fixed windows (window_size, center) or time windows (window_size = P, closed)
struct RollQuantileOp { double quantile = 0.5; int method = BL_QUANTILE_LINEAR; bool center = false; int closed = 0; int64_t window_size = 1, min_samples = 1; const DevCol* values = nullptr; };
void check_rolling_quantile_op(double q, int method, int center, int64_t window_size, int64_t min_samples, int value_dtype);
void check_rolling_quantile_by_op(double q, int method, int closed, int64_t window_size, int64_t min_samples, int value_dtype);
int rolling_quantile_dtype(int dtype);
std::vector<DevCol> op_rolling_quantile(const std::vector<DevCol>& partition_by, const DevCol* order_key, int order_flags, const std::vector<RollQuantileOp>& ops, int64_t n);
std::vector<DevCol> op_rolling_quantile_by(const std::vector<DevCol>& partition_by, const DevCol& by, const std::vector<RollQuantileOp>& ops, int64_t n);
// rank (rank.cu): values are numeric / Bool columns (a string column arrives as its ascending dense rank)
struct RankOp { int method = 0; bool descending = false; uint64_t seed = 0; const DevCol* values = nullptr; };
void check_rank_op(int method);      // BL_ERR_INVALID for an unknown method
int rank_dtype(int method);
std::vector<DevCol> op_rank(const std::vector<DevCol>& partition_by, const DevCol* order_key, int order_flags, const std::vector<RankOp>& ops, int64_t n);

struct JoinResult { DevCol left, right; };
JoinResult op_hash_join(const DevCol& left, const DevCol& right, int how, bool nulls_equal, int maintain_order);

void op_hash_partition(const DevCol& key, const std::vector<DevCol>& payload, int n_partitions, DevCol& out_key,
                       std::vector<DevCol>& out_payload, int64_t* offsets_host);

void set_last_error(const std::string& m);

// host-side phase tracing (BL_TRACE=1): wall-clock since the previous trace point, after a stream sync
void trace_point(const char* label);

}  // namespace plb

// C-ABI boundary guards: serialise on the context, translate exceptions into bl_status
#define BL_TRY try { std::lock_guard<std::recursive_mutex> _lk(::plb::ctx().mu);
#define BL_CATCH                                                                                        \
    return BL_OK; }                                                                                     \
    catch (const ::plb::Error& e) { ::plb::set_last_error(e.what()); cudaGetLastError(); return e.code; } \
    catch (const std::bad_alloc&) { ::plb::set_last_error("host out of memory"); return BL_ERR_OOM; }   \
    catch (const std::exception& e) { ::plb::set_last_error(e.what()); return BL_ERR_INVALID; }         \
    catch (...) { ::plb::set_last_error("unknown error"); return BL_ERR_INVALID; }
