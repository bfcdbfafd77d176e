/*
 * polars_b200.h — C ABI of the H100-native (sm_90a) hot-path library (libpolars_b200.so).
 *
 * This is the drop-in boundary B3 of SURVEY.md §8(b): the operator-level entry points a thin
 * Rust `extern "C"` crate inside polars-mem-engine binds in place of the Rayon dispatch of
 *   FilterExec::execute        crates/polars-mem-engine/src/executors/filter.rs:60-144
 *   group_by_helper            crates/polars-mem-engine/src/executors/group_by.rs:60-98
 *   DataFrameJoinOps::_join_impl  crates/polars-ops/src/frame/join/mod.rs:125-459
 *   DataFrame::take_unchecked  crates/polars-core/src/frame/mod.rs:1238-1294
 *   DataFrame::sort_impl       crates/polars-core/src/frame/mod.rs:1432-1561
 *   apply_operator             crates/polars-expr/src/expressions/binary.rs:61-131
 * (binding stubs: INTEGRATION.md).  Plain C: pointers, sizes, PODs.  No torch / C++ types.
 *
 * Memory model.  A `bl_column` describes one contiguous Arrow-layout primitive array
 * (crates/polars-arrow/src/array/primitive/mod.rs:56-60): a values buffer, an optional
 * LSB-first bit-packed validity bitmap (crates/polars-arrow/src/bitmap/immutable.rs:56-68) and
 * a logical element `offset` that applies to both (so arbitrary bitmap bit offsets are legal).
 * `location` says where the buffers live: BL_HOST (pageable or pinned host memory; pinned
 * buffers — bl_alloc_pinned or cudaHostRegister'ed — are DMA'd directly, pageable ones are staged
 * through an internal pinned ring) or BL_DEVICE (device pointers on the library's device).
 * A ChunkedArray (crates/polars-core/src/chunked_array/mod.rs:139-148) is an array of
 * bl_column chunks; the library concatenates chunks while uploading (the "rechunk" the
 * reference does first: executors/group_by.rs:70, join/mod.rs:194-218).
 *
 * Ownership.  Inputs are caller-owned and only read.  Outputs are written into caller-provided
 * `bl_column` structs; their buffers are library-owned (`owner != NULL`) in the requested
 * `out_location` and released with bl_column_free().  Nothing is retained across calls.
 *
 * Errors.  Every entry point returns a bl_status; BL_OK == 0.  On failure outputs are untouched
 * and bl_last_error() returns a thread-local NUL-terminated message (the channel the plugin ABI
 * forwards through _polars_plugin_get_last_error_message).  No exceptions cross the boundary,
 * the process is never aborted.  If the CUDA runtime or a device is missing every call fails
 * with BL_ERR_CUDA — there is no CPU fallback.
 *
 * Threading.  Entry points are thread-safe (calls are serialised per library context).
 */
#ifndef POLARS_B200_H
#define POLARS_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define BL_ABI_VERSION 1

typedef int32_t bl_status;
enum {
    BL_OK = 0,
    BL_ERR_INVALID = 1,     /* bad argument (null pointer, length mismatch, ...) */
    BL_ERR_CUDA = 2,        /* CUDA runtime / driver error, or no device */
    BL_ERR_OOM = 3,         /* device or pinned-host allocation failed */
    BL_ERR_UNSUPPORTED = 4, /* dtype / mode outside the hot path (caller falls back to its CPU path) */
    BL_ERR_DTYPE = 5,       /* key dtypes differ etc. (reference: ComputeError, join/mod.rs:231-241) */
    BL_ERR_BOUNDS = 6       /* gather index out of bounds (reference: check_bounds_ca, gather.rs:14-39) */
};

/* physical dtypes (Arrow primitive types) */
enum {
    BL_INT8 = 0, BL_INT16 = 1, BL_INT32 = 2, BL_INT64 = 3,
    BL_UINT8 = 4, BL_UINT16 = 5, BL_UINT32 = 6, BL_UINT64 = 7,
    BL_FLOAT32 = 8, BL_FLOAT64 = 9,
    BL_BOOL = 10            /* bit-packed values buffer (BooleanArray) */
};

enum { BL_HOST = 0, BL_DEVICE = 1 };

typedef struct bl_column {
    int32_t dtype;            /* BL_INT64 ... */
    int32_t location;         /* BL_HOST | BL_DEVICE */
    int64_t length;           /* logical number of rows */
    int64_t offset;           /* logical element offset into values and validity */
    int64_t null_count;       /* -1 = unknown */
    const void* values;       /* length+offset elements (BL_BOOL: bits) */
    const uint8_t* validity;  /* NULL = no nulls */
    void* owner;              /* NULL = caller-owned; else release with bl_column_free */
} bl_column;

/* IdxSize = u32 (crates/polars-utils/src/index.rs:9); null index (left join, gather) */
#define BL_IDX_NULL 0xFFFFFFFFu

/* ---- lifecycle ------------------------------------------------------------------------- */
int32_t bl_abi_version(void);
/* Binds the library to a CUDA device (-1 = current device / LOCAL_RANK env).  Idempotent. */
bl_status bl_init(int32_t device);
void bl_shutdown(void);
const char* bl_last_error(void);
/* device facts for the host side: writes sm count, L2 bytes, total/free HBM bytes */
bl_status bl_device_info(int32_t* sm_count, int64_t* l2_bytes, int64_t* hbm_total, int64_t* hbm_free);
/* Returns the library's cached device blocks and its memory pool's unused memory to the driver, so that hbm_free counts
   them and another allocator (PyTorch) can use them.  The next calls allocate afresh. */
bl_status bl_release_cached(void);

/* Deterministic aggregation (SURVEY.md §7(b)): on != 0 makes bl_groupby_agg / bl_groupby_agg_keys build the reference's
 * GroupsIdx and fold every group sequentially in row order with the reference's reducers (sequential Kahan float sums,
 * aggregations/mod.rs:854-977): results are bit-identical from run to run and to the reference's in-memory engine, floats
 * included, at a fraction of the fused path's speed.  Also enabled by the environment variable BL_DETERMINISTIC=1. */
void bl_set_deterministic(int32_t on);

/* ---- memory ---------------------------------------------------------------------------- */
/* Pinned host buffers (the SharedStorage::ForeignOwner seam, crates/polars-buffer/src/storage.rs:37-53). */
bl_status bl_alloc_pinned(size_t bytes, void** out);
void bl_free_pinned(void* p);
bl_status bl_dev_alloc(size_t bytes, void** out);
void bl_dev_free(void* p);
bl_status bl_memcpy_h2d(void* dst_dev, const void* src_host, size_t bytes);
bl_status bl_memcpy_d2h(void* dst_host, const void* src_dev, size_t bytes);
/* Copies a (possibly chunked) column to the other location; result is library-owned. */
bl_status bl_column_to(const bl_column* chunks, int32_t n_chunks, int32_t location, bl_column* out);
void bl_column_free(bl_column* col);
/* Blocks until all work queued by this thread's calls has finished (outputs are already
 * complete when an entry point returns; this is for bl_dev_* / profiling users). */
bl_status bl_sync(void);
/* The CUDA stream (cudaStream_t) every kernel of this library is launched on. */
void* bl_stream(void);

/* ---- K1: elementwise arithmetic  (ArithmeticKernel, polars-compute/src/arithmetic/mod.rs:8-76) */
enum { BL_OP_ADD = 0, BL_OP_SUB = 1, BL_OP_MUL = 2, BL_OP_FLOOR_DIV = 3, BL_OP_MOD = 4, BL_OP_TRUE_DIV = 5 };
/* lhs (op) rhs.  A length-1 side broadcasts as a scalar (apply_operator, binary.rs:61-131) and
 * takes the reference's scalar code path (e.g. float x / c == x * (1/c), float.rs:113-115).
 * Integer FLOOR_DIV / MOD by zero yield null (signed.rs:35-70); integer TRUE_DIV yields FLOAT64.
 * Output validity = AND of input validities (arity.rs:90). */
bl_status bl_elementwise(int32_t op, const bl_column* lhs, const bl_column* rhs, int32_t out_location, bl_column* out);

/* ---- K2: comparisons -> BooleanArray  (TotalOrdKernel/TotalEqKernel, comparisons/mod.rs:4-76) */
enum { BL_CMP_EQ = 0, BL_CMP_NE = 1, BL_CMP_LT = 2, BL_CMP_LE = 3, BL_CMP_GT = 4, BL_CMP_GE = 5 };
/* Total order on floats: NaN == NaN, NaN greatest (polars-utils/src/total_ord.rs:317-364).
 * missing != 0 selects eq_missing / ne_missing (null == null, never-null result). */
bl_status bl_compare(int32_t op, const bl_column* lhs, const bl_column* rhs, int32_t missing, int32_t out_location, bl_column* out);

/* ---- K3: filter  (polars-compute/src/filter/mod.rs:18-110; DataFrame::filter frame/mod.rs:1148-1180) */
/* mask: BL_BOOL column; a null mask slot counts as false.  All n_cols columns are compacted with
 * one mask pass.  outs[i] keeps cols[i].dtype. */
bl_status bl_filter(const bl_column* cols, int32_t n_cols, const bl_column* mask, int32_t out_location, bl_column* outs);
/* Fused predicate + compaction: keep rows where cols[pred_col] (cmp_op) scalar
 * (FilterExec over BinaryExpr(col, op, lit), executors/filter.rs:117-144).  scalar: length-1 column. */
bl_status bl_filter_cmp(const bl_column* cols, int32_t n_cols, int32_t pred_col, int32_t cmp_op, const bl_column* scalar,
                        int32_t out_location, bl_column* outs);

/* ---- K4: gather  (take_primitive_unchecked, polars-compute/src/gather/primitive.rs:9-78) */
/* idx: BL_UINT32 column (IdxSize).  A null idx slot or idx == BL_IDX_NULL gives a null row with
 * value 0.  check_bounds != 0 validates idx < col.length first (BL_ERR_BOUNDS). */
bl_status bl_gather(const bl_column* cols, int32_t n_cols, const bl_column* idx, int32_t check_bounds, int32_t out_location, bl_column* outs);

/* ---- K5: hash group_by + aggregation --------------------------------------------------- */
/* (group_by_threaded_slice hashing.rs:116-167 + agg_sum/mean/min/max aggregations/mod.rs:486-1018,
 *  fused: index lists are never materialised) */
enum { BL_AGG_SUM = 0, BL_AGG_MEAN = 1, BL_AGG_MIN = 2, BL_AGG_MAX = 3, BL_AGG_COUNT = 4, BL_AGG_LEN = 5,
       /* evaluated per group over the reference's GroupsIdx (row lists in row order), not by the fused atomics path: */
       BL_AGG_FIRST = 6, BL_AGG_LAST = 7,   /* value at the group's first / last row, nulls included (dispatch.rs:57-120) */
       BL_AGG_VAR = 8, BL_AGG_STD = 9,      /* Welford in row order, f64; null when count <= ddof (aggregations/mod.rs:1020-1178, take_agg/var.rs:11-41) */
       BL_AGG_N_UNIQUE = 10,                /* distinct values per group, a null counts as one (aggregations/dispatch.rs:285-345); UInt32; bl_groupby_agg only */
       BL_AGG_MEDIAN = 11,                  /* quantile(0.5, LINEAR) (aggregations/mod.rs:385-408) */
       BL_AGG_QUANTILE = 12 };              /* probability and method from bl_agg_param: bl_groupby_agg_params only (aggregations/mod.rs:297-383) */
/* Interpolation of BL_AGG_QUANTILE (QuantileMethod, polars-compute/src/rolling/mod.rs:40-48; Polars' default is NEAREST).
 * Per group with m valid values and c nulls (quantile.rs:21-65): float_idx = (m - 1) * q + c into the values sorted nulls first
 * in the total order (NaN greatest, -0.0 == +0.0); NEAREST takes round(float_idx) (half away from zero), LOWER / MIDPOINT /
 * LINEAR trunc(float_idx), HIGHER ceil(float_idx), EQUIPROBABLE max(ceil(m * q) - 1, 0) + c; MIDPOINT and LINEAR interpolate
 * towards the next value in f64 when float_idx is not whole.  A group without a valid value gives null. */
enum { BL_QUANTILE_NEAREST = 0, BL_QUANTILE_LOWER = 1, BL_QUANTILE_HIGHER = 2, BL_QUANTILE_MIDPOINT = 3, BL_QUANTILE_LINEAR = 4,
       BL_QUANTILE_EQUIPROBABLE = 5 };
typedef struct bl_agg_param {
    double quantile;        /* in [0, 1]; NaN or outside: BL_ERR_UNSUPPORTED (the reference returns an all-null column of the input dtype) */
    int32_t method;         /* BL_QUANTILE_* */
    int32_t reserved;
} bl_agg_param;
/* delta degrees of freedom of VAR / STD travel in bits 16..23 of `kind` (Polars' default is 1) */
#define BL_AGG_WITH_DDOF(kind, ddof) ((kind) | ((ddof) << 16))
typedef struct bl_agg {
    int32_t kind;           /* BL_AGG_* */
    int32_t n_chunks;       /* chunks of the value column (ignored for BL_AGG_LEN) */
    const bl_column* values;
} bl_agg;
/* Single numeric key (ints are grouped on their bit pattern, floats canonicalised: -0 == +0,
 * all NaNs equal; a null key is its own group — into_groups.rs:25-58,142-191).
 * maintain_order != 0: groups ordered by first occurrence (hashing.rs:41-63); else unspecified.
 * out_key = key taken at each group's first row (group_by/mod.rs:258-266).
 * Output dtypes: SUM keeps the dtype (Int8/16,UInt8/16 -> Int64), ints wrap; MEAN -> FLOAT64
 * (FLOAT32 stays); MIN/MAX keep dtype; COUNT/LEN -> UINT32.  All-null group: SUM 0, MEAN/MIN/MAX null.
 * FIRST/LAST keep dtype; VAR/STD/MEDIAN/QUANTILE -> FLOAT64 (FLOAT32 stays).  A call that asks for any of
 * FIRST/LAST/VAR/STD/MEDIAN/QUANTILE is evaluated whole over GroupsIdx (groups then come in first-occurrence order), like
 * bl_set_deterministic.  MEDIAN / QUANTILE on a BL_BOOL column: BL_ERR_UNSUPPORTED; BL_AGG_QUANTILE needs
 * bl_groupby_agg_params (here: BL_ERR_INVALID).  All MEDIAN / QUANTILE aggregations of one value column share one sort. */
bl_status bl_groupby_agg(const bl_column* key_chunks, int32_t n_key_chunks, const bl_agg* aggs, int32_t n_aggs,
                         int32_t maintain_order, int32_t out_location, bl_column* out_key, bl_column* out_aggs);

/* Several key columns (DataFrame::group_by_with_series routes them through row encoding,
 * polars-core/src/frame/group_by/mod.rs:88-94; polars-row/src/fixed/numeric.rs:100-145): numeric columns of the
 * dtypes above plus Int8/16, UInt8/16, one chunk each.  Equality per column as for a single key (null == null,
 * -0 == +0, NaN == NaN).  out_keys[i] = keys[i] taken at each group's first row; the rest as bl_groupby_agg. */
bl_status bl_groupby_agg_keys(const bl_column* keys, int32_t n_keys, const bl_agg* aggs, int32_t n_aggs,
                              int32_t maintain_order, int32_t out_location, bl_column* out_keys, bl_column* out_aggs);
/* bl_groupby_agg_keys with per-aggregation parameters: params[i] is read only where aggs[i].kind == BL_AGG_QUANTILE
 * (params may be NULL when there is none).  bl_groupby_agg_keys is this call with params = NULL.  An unknown method, or a
 * BL_AGG_QUANTILE without params: BL_ERR_INVALID. */
bl_status bl_groupby_agg_params(const bl_column* keys, int32_t n_keys, const bl_agg* aggs, const bl_agg_param* params, int32_t n_aggs,
                                int32_t maintain_order, int32_t out_location, bl_column* out_keys, bl_column* out_aggs);

/* Group tuples: the reference's GroupsIdx{first, all} (polars-core/src/frame/group_by/position.rs:16-22)
 * as built by group_by_threaded_slice with sorted = true (hashing.rs:116-167, finish_group_order :41-63),
 * for aggregations outside the fused set above.  Groups come in first-occurrence order; group g owns
 * out_all[out_offsets[g] .. out_offsets[g+1]) (row indices ascending), out_first[g] = its first row.
 * All three outputs are BL_UINT32 (IdxSize); out_offsets has n_groups + 1 entries.  Null key = own group. */
bl_status bl_group_tuples(const bl_column* key_chunks, int32_t n_key_chunks, int32_t out_location,
                          bl_column* out_first, bl_column* out_offsets, bl_column* out_all);

/* ---- string / binary keys: device-side dictionary encoding (SURVEY.md 8(f1)) ------------------------ */
/* Arrow LargeUtf8 / LargeBinary layout (polars-arrow/src/array/binary/mod.rs): value i = data[offsets[offset+i] ..
 * offsets[offset+i+1]); validity bit (offset + i).  Polars hands strings out as view arrays (plugin.rs:165-166); the glue
 * casts them with polars_compute::cast::utf8view_to_utf8::<i64> (crates/polars-compute/src/cast/binview_to.rs:56) first (INTEGRATION.md). */
typedef struct bl_string_column {
    int32_t location;         /* BL_HOST | BL_DEVICE */
    int32_t reserved;
    int64_t length;           /* logical number of rows */
    int64_t offset;           /* logical element offset into offsets and validity */
    int64_t null_count;       /* -1 = unknown */
    const int64_t* offsets;   /* offset + length + 1 entries */
    const uint8_t* data;
    const uint8_t* validity;  /* NULL = no nulls */
    void* owner;              /* NULL = caller-owned; else release with bl_string_column_free */
} bl_string_column;

/* BinaryChunked::group_tuples (polars-core/src/frame/group_by/into_groups.rs:215-251) groups rows by their BYTES (hash of
 * the bytes + equality, nulls = own group).  bl_string_encode materialises that relation as a UInt32 code column:
 * out_codes[i] = index of the first row holding the same bytes as row i (null rows: null code).  The codes are an ordinary
 * key for bl_groupby_agg / bl_hash_join / bl_group_tuples (for a join, encode the concatenation of both sides' chunks and
 * split the codes), and the key values a group_by returns are the gather indices of the group keys (bl_string_gather).
 * *n_distinct (optional) = number of distinct non-null values.  Exact: equal codes <=> equal bytes (verified on the device). */
bl_status bl_string_encode(const bl_string_column* chunks, int32_t n_chunks, int32_t out_location, bl_column* out_codes, int64_t* n_distinct);
/* out[i] = the string at row idx[i] of the (concatenated) chunks; a null index, BL_IDX_NULL or a null source row gives a
 * null.  idx: BL_UINT32.  Out-of-range indices: BL_ERR_BOUNDS. */
bl_status bl_string_gather(const bl_string_column* chunks, int32_t n_chunks, const bl_column* idx, int32_t out_location, bl_string_column* out);
/* group_by / join on a string key in ONE call: encode -> bl_groupby_agg on the codes -> gather of the group keys
 * (out_key: LargeUtf8, one value per group, null = the null group), resp. encode both sides together -> bl_hash_join on the
 * codes (row-index tuples as bl_hash_join; with nulls_equal a null matches a null, single_keys_dispatch.rs:20-60). */
bl_status bl_groupby_agg_strings(const bl_string_column* key_chunks, int32_t n_key_chunks, const bl_agg* aggs, int32_t n_aggs, int32_t maintain_order,
                                 int32_t out_location, bl_string_column* out_key, bl_column* out_aggs);
bl_status bl_hash_join_strings(const bl_string_column* left_chunks, int32_t n_left_chunks, const bl_string_column* right_chunks, int32_t n_right_chunks, int32_t how,
                               int32_t nulls_equal, int32_t maintain_order, int32_t out_location, bl_column* out_left_idx, bl_column* out_right_idx);
/* copy / move a string column between host and device (concatenates chunks) */
bl_status bl_string_column_to(const bl_string_column* chunks, int32_t n_chunks, int32_t location, bl_string_column* out);
void bl_string_column_free(bl_string_column* col);

/* ---- string predicates and filter (DESIGN.md §19) ------------------------------------------------------------------ */
/* Every result is a BL_BOOL column of the column's length whose validity is the AND of the input validities.  A single
 * device chunk is read in place (its Arrow offset and a first offset other than 0 included; no byte past offsets[n] is
 * read); host and multi-chunk inputs are copied to the device first.  A column of length 1 is a scalar.
 * lhs (op) rhs; rhs has lhs's length or length 1.  Lexicographic unsigned-byte order, a proper prefix first, so
 * "a" < "a\0" < "b" (polars-compute/src/comparisons/binary.rs:8-70).  A null on either side gives null; a null scalar gives
 * an all-null column.  missing != 0 (EQ / NE only): eq_missing / ne_missing, null == null is true and the result has no
 * nulls; against a null scalar that is is_null (EQ) / is_not_null (NE).
 * Errors: an unknown op, missing with another op, rhs of another length: BL_ERR_INVALID; more than 2^32 - 2 rows:
 * BL_ERR_UNSUPPORTED (as bl_string_encode). */
bl_status bl_string_compare(int32_t op, const bl_string_column* lhs, int32_t n_lhs_chunks, const bl_string_column* rhs, int32_t n_rhs_chunks,
                            int32_t missing, int32_t out_location, bl_column* out);
enum { BL_STR_STARTS_WITH = 0, BL_STR_ENDS_WITH = 1, BL_STR_CONTAINS = 2, BL_STR_LIKE = 3 };
/* flags: BL_STR_NEGATE (NOT) flips each valid result, nulls stay null.  LIKE only: BL_LIKE_NO_NEWLINE: '%' and '_' do not
 * match '\n' (the regex '.' without (?s)); BL_LIKE_OPEN_START / BL_LIKE_OPEN_END: the match may begin / end anywhere, as if
 * the pattern had a leading / trailing run of any bytes that newlines do not stop (a regex search without '^' / '$'). */
enum { BL_STR_NEGATE = 1, BL_LIKE_NO_NEWLINE = 2, BL_LIKE_OPEN_START = 4, BL_LIKE_OPEN_END = 8 };
/* STARTS_WITH / ENDS_WITH / CONTAINS are byte predicates (polars-ops/src/chunked_array/binary/namespace.rs:58-125); on Utf8
 * columns CONTAINS is str.contains(literal=True) (strings/namespace.rs:174-200, 348-353).  The empty pattern matches every
 * non-null row; a null scalar pattern gives an all-null column; with a per-row pattern column a null pattern gives a null
 * row.  Needles of any length.
 * LIKE is what polars-sql builds for `col LIKE 'pattern'` (sql_expr.rs:435-479, visit_like): ^(?s)<pattern>$ where '%'
 * matches any run of characters, '_' exactly one character (one UTF-8 sequence, not one byte) and every other byte itself.
 * LIKE reads the bytes as UTF-8: the ABI cannot tell Utf8 from Binary, and '_' over bytes that are not UTF-8 is undefined.
 * escape (LIKE only; 0 = none) is an extension the reference rejects: that byte followed by '%', '_' or itself is that
 * literal byte; followed by anything else, or at the end, it is BL_ERR_INVALID.  The pattern must be a scalar.
 * Errors: an unknown kind or flag, a BL_LIKE_* flag or escape with another kind, a per-row LIKE pattern, a pattern whose
 * length is neither 1 nor the column's: BL_ERR_INVALID; a LIKE pattern with more than 63 literal bytes and '_' ('%' is
 * free): BL_ERR_UNSUPPORTED; more than 2^32 - 2 rows: BL_ERR_UNSUPPORTED. */
bl_status bl_string_match(int32_t kind, int32_t flags, int32_t escape, const bl_string_column* col, int32_t n_chunks,
                          const bl_string_column* pattern, int32_t n_pattern_chunks, int32_t out_location, bl_column* out);
/* The rows whose mask bit is set, in row order (polars-compute/src/filter/mod.rs:18-110); a null mask slot counts as false,
 * as bl_filter.  mask: BL_BOOL (BL_ERR_DTYPE otherwise) of the column's length (BL_ERR_INVALID otherwise).  More than
 * 2^32 - 2 rows: BL_ERR_UNSUPPORTED. */
bl_status bl_string_filter(const bl_string_column* chunks, int32_t n_chunks, const bl_column* mask, int32_t out_location, bl_string_column* out);

/* ---- K7/K8: hash join on one numeric key ----------------------------------------------- */
/* (build_tables single_keys.rs:16-167, probe_inner single_keys_inner.rs:11-149,
 *  hash_join_tuples_left single_keys_left.rs:106-195) */
enum { BL_JOIN_INNER = 0, BL_JOIN_LEFT = 1, BL_JOIN_SEMI = 2, BL_JOIN_ANTI = 3, BL_JOIN_FULL = 4 };
enum { BL_ORDER_NONE = 0, BL_ORDER_LEFT = 1, BL_ORDER_LEFT_RIGHT = 2, BL_ORDER_RIGHT = 3, BL_ORDER_RIGHT_LEFT = 4 };
/* Returns the join tuples as two UINT32 columns.  BL_ORDER_NONE reproduces the in-memory engine's
 * order (probe = longer relation, tie -> right probes; probe-row order; matches ascending build
 * idx — hash_join/mod.rs:41-50).  Null keys match only if nulls_equal.  Left join: unmatched
 * right idx = BL_IDX_NULL (and a null slot).  BL_JOIN_SEMI / BL_JOIN_ANTI (single_keys_semi_anti.rs:41-140):
 * out_left_idx = the left rows, in row order, with / without a match; out_right_idx is an empty column.
 * BL_JOIN_FULL (hash_join_tuples_outer, single_keys_outer.rs:100-260): the longer relation probes; first its left-join
 * tuples in probe order, then the build rows no probe key matched with a null on the probe side (ascending build row;
 * the reference drains its hash tables there, order unspecified).  Both outputs are nullable; BL_ORDER_NONE only. */
bl_status bl_hash_join(const bl_column* left_key, int32_t n_left_chunks, const bl_column* right_key, int32_t n_right_chunks,
                       int32_t how, int32_t nulls_equal, int32_t maintain_order, int32_t out_location,
                       bl_column* out_left_idx, bl_column* out_right_idx);

/* Several key columns per side (prepare_keys_multiple, polars-ops/src/frame/join/mod.rs:658-678: the reference row-encodes
 * the key columns of each side and runs the single-key machinery on the encoded rows).  left_keys[i] pairs with
 * right_keys[i] (same dtype; any numeric dtype incl. 8/16-bit; one chunk each).  nulls_equal == 0: a null in ANY key
 * column makes the row's key null (it matches nothing); != 0: nulls are part of the key and match each other per column.
 * Everything else as bl_hash_join. */
bl_status bl_hash_join_keys(const bl_column* left_keys, const bl_column* right_keys, int32_t n_keys, int32_t how, int32_t nulls_equal,
                            int32_t maintain_order, int32_t out_location, bl_column* out_left_idx, bl_column* out_right_idx);

/* Join + materialisation (_finish_join, polars-ops/src/frame/join/general.rs:17-49; JoinExec,
 * polars-mem-engine/src/executors/join.rs:39-120): bl_hash_join on the key columns followed by one K4
 * gather per side, the tuples never leaving the device.  out_left_cols[i] = left_cols[i] taken at the left
 * idx, out_right_cols[j] = right_cols[j] taken at the right idx (left join: unmatched rows are null).
 * Column naming (the `_right` suffix, dropping the right key) is the caller's metadata.  One chunk per column. */
bl_status bl_join(const bl_column* left_key, const bl_column* right_key,
                  const bl_column* left_cols, int32_t n_left_cols, const bl_column* right_cols, int32_t n_right_cols,
                  int32_t how, int32_t nulls_equal, int32_t maintain_order, int32_t out_location,
                  bl_column* out_left_cols, bl_column* out_right_cols);

/* ---- K9: sort  (DataFrame::sort_impl polars-core/src/frame/mod.rs:1432-1561; arg_sort_multiple arg_sort_multiple.rs:66-75) */
enum { BL_SORT_DESCENDING = 1, BL_SORT_NULLS_LAST = 2 };
/* The IdxSize permutation that sorts the rows by by[0], then by[1], ... (one chunk per column; any numeric dtype incl.
 * 8/16-bit, and BL_BOOL: false < true).  flags[i]: bits above for by[i]; NULL = all ascending, nulls first
 * (SortMultipleOptions, options.rs:85-105).  Values in the total order of reorder_cmp (polars-utils/src/sort.rs:113-128):
 * floats by tot_cmp (NaN == NaN and greatest, -0.0 == +0.0), descending reverses it; null placement follows
 * BL_SORT_NULLS_LAST only, and nulls compare equal.  The result is always the STABLE order (ties keep row order), which is
 * the reference's answer wherever it pins one (single column: arg_sort.rs:118-185; maintain_order).
 * limit >= 0 keeps the first `limit` rows of the sorted order (the (0, k) slice, frame/mod.rs:1482-1486).
 * out_idx: BL_UINT32.  More than 2^32 - 1 rows: BL_ERR_UNSUPPORTED.  String / binary keys: bl_arg_sort_keys. */
bl_status bl_arg_sort(const bl_column* by, int32_t n_by, const int32_t* flags, int64_t limit,
                      int32_t out_location, bl_column* out_idx);
/* bl_arg_sort + one K4 gather of the payload columns (4- and 8-byte dtypes) at the first `limit` rows of the
 * permutation: out_cols[i] = cols[i] in sorted order, validity included.  Key columns appear in cols if wanted. */
bl_status bl_sort(const bl_column* by, int32_t n_by, const int32_t* flags, const bl_column* cols, int32_t n_cols,
                  int64_t limit, int32_t out_location, bl_column* out_cols);

/* Dense lexicographic rank (RankMethod::Dense, rank.rs:61-188) of a LargeUtf8 / LargeBinary column: UInt32, 1-based, bytes
 * compared unsigned with a proper prefix first; descending != 0 ranks the largest value 1; null rows give null.
 * *n_distinct (optional) = number of distinct non-null values = the largest rank.  More than 2^32 - 2 rows: BL_ERR_UNSUPPORTED. */
bl_status bl_string_rank(const bl_string_column* chunks, int32_t n_chunks, int32_t descending, int32_t out_location,
                         bl_column* out_rank, int64_t* n_distinct);

typedef struct bl_sort_key {
    const bl_column* column;          /* numeric / Boolean key (one chunk), or NULL */
    const bl_string_column* strings;  /* LargeUtf8 / LargeBinary key, or NULL; exactly one of the two is set */
    int32_t n_chunks;                 /* chunks of `strings` */
    int32_t flags;                    /* BL_SORT_DESCENDING | BL_SORT_NULLS_LAST */
} bl_sort_key;
/* bl_arg_sort over keys that may be strings: each string key is ranked (bl_string_rank, ascending) and sorted as that
 * UInt32 column with its own flags; everything else exactly as bl_arg_sort.  A descriptor with both or neither pointer set,
 * or keys of different lengths: BL_ERR_INVALID.  String payload columns are materialised with bl_string_gather on the
 * permutation, numeric ones with bl_gather. */
bl_status bl_arg_sort_keys(const bl_sort_key* by, int32_t n_by, int64_t limit, int32_t out_location, bl_column* out_idx);
/* Top-k selection: the first k rows of the stable order of `by` (flags per key as in bl_arg_sort_keys), as UInt32 row
 * ids in ASCENDING ROW ORDER; min(k, n) of them.  The same key dtypes as bl_arg_sort_keys; a string / binary key costs
 * its rank (bl_string_rank), which is a sort of its own.  The reference: top_k / bottom_k of a column
 * (polars-ops/src/chunked_array/top_k.rs:151-229) put non-null values before nulls, pad with nulls when fewer than k are
 * valid and leave the output order open (select_nth_unstable); top_k_by / bottom_k_by (top_k.rs:231-297) and
 * DataFrame.top_k / bottom_k (_arg_bottom_k, polars-core/src/chunked_array/ops/sort/arg_bottom_k.rs:33-…) use
 * descending = !reverse and nulls_last for every column and return the rows sorted, ties in an open order; sort(...,
 * limit = k) is the (0, k) slice of the stable order (frame/mod.rs:1482-1486).  This call returns the one set that
 * answers all of them with ties broken by row index; the sorted form is bl_arg_sort / bl_arg_sort_keys with limit = k
 * (which selects through this plan when k <= n / 8).  Plan (DESIGN.md §17): an MSD radix select, one histogram pass per
 * varying 8-bit digit of the key.  Device memory: n / 8 B of selection bitmap, n / 8 B of tie bitmap, row-id lists of at most n / 4 B, the
 * output.  Errors: k < 0, keys of different lengths, a descriptor with both or neither pointer set: BL_ERR_INVALID; a
 * key dtype bl_arg_sort does not take: BL_ERR_UNSUPPORTED; more than 2^32 - 1 rows: BL_ERR_UNSUPPORTED. */
bl_status bl_top_k(const bl_sort_key* by, int32_t n_by, int64_t k, int32_t out_location, bl_column* out_idx);

/* ---- unique  (DataFrame::unique_impl polars-core/src/frame/mod.rs:2317-2392; is_unique / is_duplicated frame/mod.rs:2408-2442,
 * polars-ops/src/series/ops/is_unique.rs:11-41,113-119; is_first_distinct.rs:107-161; is_last_distinct.rs:12-…) -------- */
enum { BL_UNIQUE_FIRST = 0, BL_UNIQUE_LAST = 1, BL_UNIQUE_ANY = 2, BL_UNIQUE_NONE = 3 };
enum { BL_DISTINCT_FIRST = 0, BL_DISTINCT_LAST = 1, BL_DISTINCT_UNIQUE = 2, BL_DISTINCT_DUPLICATED = 3 };
/* The rows DataFrame.unique(subset, keep, maintain_order, slice) keeps, as UInt32 row ids in ASCENDING ROW ORDER.  The
 * reference: First / Any with maintain_order take each key's first row in first-occurrence order; Last with maintain_order
 * takes the keys' last rows sorted ascending; None is filter(is_unique); without maintain_order the same rows come in an
 * open order.  Row order is therefore exact for maintain_order and a valid order otherwise; a `slice` (offset, len) is that
 * sub-range of the ids.  BL_UNIQUE_ANY is BL_UNIQUE_FIRST.  Key equality as group_by: null is a value of its own, floats
 * compare by total equality (-0.0 == +0.0, every NaN equal), strings by bytes, several columns form one row key; a kept row
 * keeps its own bytes (on [+0.0, -0.0] FIRST keeps +0.0 and LAST -0.0).  Empty input: no rows.
 * subset: one bl_sort_key per key column with flags 0: numeric / Boolean (one chunk) or LargeUtf8 / LargeBinary.
 * Plan (DESIGN.md §18): the K5 table with each key's first row and row count, one more pass for the last rows (LAST only),
 * one pass that marks the kept rows in a bitmap, its compaction.  Device memory: the K5 table, 4 B per table slot for the
 * last rows (LAST only), n / 8 B of mask, the ids; string keys add their codes (4 B per row).
 * Errors: an unknown keep, flags != 0, a descriptor with both or neither pointer set, n_subset < 1, null pointers, key
 * columns of different lengths: BL_ERR_INVALID; another key dtype: BL_ERR_UNSUPPORTED; more than 2^32 - 2 rows:
 * BL_ERR_UNSUPPORTED (checked before any upload). */
bl_status bl_unique(const bl_sort_key* subset, int32_t n_subset, int32_t keep, int32_t out_location, bl_column* out_idx);
/* One Boolean per row (BL_BOOL, n rows, no nulls) over the same keys: BL_DISTINCT_FIRST = is_first_distinct (the row is its
 * key's first), BL_DISTINCT_LAST = is_last_distinct (its key's last), BL_DISTINCT_UNIQUE = is_unique (the key occurs once),
 * BL_DISTINCT_DUPLICATED = is_duplicated (more than once).  Arguments, errors and memory as bl_unique; an unknown kind:
 * BL_ERR_INVALID. */
bl_status bl_unique_mask(const bl_sort_key* keys, int32_t n_keys, int32_t kind, int32_t out_location, bl_column* out_mask);

/* ---- asof join  (_join_asof_dispatch polars-ops/src/frame/join/asof/mod.rs:325-394; by keys groups.rs:39-345) ------- */
enum { BL_ASOF_BACKWARD = 0, BL_ASOF_FORWARD = 1, BL_ASOF_NEAREST = 2 };
/* The reference's take_idx: out_right_idx (BL_UINT32, left_on->length rows, nullable; a null slot holds BL_IDX_NULL) names,
 * per left row, the right row its asof search picks.  The frame is then left ‖ right.take(idx) (_finish_join, mod.rs:300-321).
 * Precondition, checked on the device on every call with at least one left row (per group when n_by > 0; an empty left side
 * returns an empty index at once, which is the reference's answer whatever the right side holds): the non-null left `on` values are
 * non-decreasing (nulls anywhere), the right `on` column is nulls first and then non-decreasing (is_sorted with the default
 * SortOptions), both in the total order (NaN greatest, -0.0 == +0.0).  Outside it: BL_ERR_UNSUPPORTED, the message naming
 * the side; the caller's CPU path gives the reference's answer there.  Inside it, the reference's cursors (mod.rs:47-200)
 * give, per non-null left value l over V = [z, n), the right's non-null rows (a null l, or an empty V, gives null):
 *   BL_ASOF_BACKWARD  the last j in V with r_j <= l (r_j < l when allow_eq == 0), total order
 *   BL_ASOF_FORWARD   the first j in V with r_j >= l (r_j > l when allow_eq == 0), total order
 *   BL_ASOF_NEAREST   partial order (the reference compares with >, >= and ==, mod.rs:143-180): U = the first j in V with
 *                     r_j > l, else n; with allow_eq, U > z and r_{U-1} == l: U - 1.  Otherwise U moves to the last row of its
 *                     run of equal values (U < n), L = (the first j in [z, U) with r_j >= l) - 1, or U - 1 when there is none;
 *                     the one of L (>= z) and U (< n) that exists, and with both U when |l - r_U| <= |l - r_L|, else L.
 * tolerance (NULL, or a non-null length-1 column of the key dtype; for an 8/16-bit key also Int32, the type the reference
 * extracts it as, so e.g. 200 on an Int8 key is accepted): the pick stays only when |l - r| <= |tolerance|, else the row is
 * null (default.rs:127-135).  |a - b| is abs_diff in the key's own type: exact unsigned for integers, a > b ? a - b :
 * b - a in the float's precision (a NaN difference fails every comparison).  Key dtypes: Int/UInt 8-64 (8/16-bit searched as
 * Int32, mod.rs:333-338) and Float32/64, one chunk per side; Bool keys: BL_ERR_UNSUPPORTED.
 * by (n_by > 0): left_by[i] pairs with right_by[i], a numeric column (one chunk) or a string column (chunks) of the same type
 * on both sides, flags 0; only right rows with equal `by` values are searched, in row order, exactly as bl_hash_join_keys
 * with nulls_equal == 0 matches rows (floats -0 == +0, NaN == NaN; a null in any `by` column matches nothing).
 * Errors: BL_ERR_DTYPE for `on` or `by` dtypes that differ (string vs numeric included); BL_ERR_INVALID for an unknown
 * strategy, flags != 0, lengths that differ, a bad tolerance, n_by > 0 with a NULL array; BL_ERR_UNSUPPORTED for Bool `on`
 * or `by` columns, an unsorted side, more than 2^32 - 2 rows on a side (both sides together with `by`). */
bl_status bl_join_asof(const bl_column* left_on, const bl_column* right_on, const bl_sort_key* left_by, const bl_sort_key* right_by, int32_t n_by,
                       int32_t strategy, int32_t allow_eq, const bl_column* tolerance, int32_t out_location, bl_column* out_right_idx);

/* ---- inequality join  (IEJoin: _join_impl polars-ops/src/frame/join/mod.rs:243-270; iejoin/mod.rs:572-799) ---- */
enum { BL_IE_LT = 0, BL_IE_LE = 1, BL_IE_GT = 2, BL_IE_GE = 3 };
/* The reference's join_where with one or two inequality predicates (the planner's JoinType::IEJoin): left_on[k] ops[k]
 * right_on[k] for k < n_pred (1 or 2).  The pair (i, j) is in the result iff left_on[k][i] ops[k] right_on[k][j] holds for
 * every k, compared in the total order (NaN greatest and equal to NaN, -0.0 == +0.0: tot_lt / tot_le ...), and every
 * predicate column is valid in both rows.  This is the set both serial algorithms compute (piecewise_merge_join_tuples
 * mod.rs:667-799, iejoin_tuples :572-665) and the reference's own test rule, a cross join filtered by the predicates.
 *   how = BL_JOIN_INNER  those pairs.
 *   how = BL_JOIN_LEFT   those pairs plus one (i, null) for every left row without one, a row with a null predicate value
 *                        included (append_unmatched_left, mod.rs:232-265).
 * A right join is this call with the sides swapped, every operator flipped (< and >, <= and >=) and the outputs swapped
 * (emit_unmatched_right_via_flip, mod.rs:279-296).  Semi, anti, full and any other `how`: BL_ERR_INVALID, as the reference
 * rejects them for non-equi predicates.
 * Outputs: two BL_UINT32 columns of one row per pair.  out_left_idx has no nulls; out_right_idx has a validity bitmap only
 * for BL_JOIN_LEFT, with BL_IDX_NULL in its null slots.
 * Order (the reference pins none; join_where documents that the row order is not preserved): pairs are grouped by left row,
 * left rows ascending, an unmatched left row of a left join at its place.  The order inside one left row is deterministic
 * (the same inputs give the same bytes) but unspecified.
 * Quirk, not reproduced: the parallel path (iejoin_par_indices, mod.rs:331-458) skips a pair of blocks when their first /
 * last x-values fail `<` / `<=` compared as AnyValue (mod.rs:372-400), a partial order for floats; with NaN x-values it can
 * drop pairs that the serial algorithms and the cross-join rule keep.  This call follows the total-order rule.
 * Columns: one chunk each; both sides of one predicate have the same dtype, the two predicates may differ.  Dtypes: Int/UInt
 * 8-64, Float32/64.
 * Device memory: with two predicates, a merge-sort tree of L x m x 8 bytes for m right rows valid in both predicate columns,
 * L = 1 + ceil(log2 m) (about 2 GB at m = 1e7).  The pair count is known before the output is allocated.
 * Errors: BL_ERR_DTYPE for dtypes that differ within a predicate (the reference's ComputeError, mod.rs:231-241);
 * BL_ERR_UNSUPPORTED for a Bool column or more than 2^32 - 2 rows on a side; BL_ERR_INVALID for a NULL pointer, n_pred
 * outside {1, 2}, an unknown operator or `how`, predicate columns of different lengths on one side; BL_ERR_OOM when the
 * tree or the output (the message gives the pair count) does not fit in device memory. */
bl_status bl_ie_join(const bl_column* left_on, const bl_column* right_on, const int32_t* ops, int32_t n_pred,
                     int32_t how, int32_t out_location, bl_column* out_left_idx, bl_column* out_right_idx);

/* ---- window functions  (expr.over(partition_by, order_by), polars-expr/src/expressions/window.rs; cum_* cum_agg.rs) ---- */
enum { BL_CUM_SUM = 32, BL_CUM_PROD = 33, BL_CUM_MIN = 34, BL_CUM_MAX = 35, BL_CUM_COUNT = 36, BL_SHIFT = 37 };
typedef struct bl_over_op {
    int32_t kind;             /* BL_AGG_* (broadcast to the group's rows) or BL_CUM_* / BL_SHIFT */
    int32_t reverse;          /* BL_CUM_*: scan from the partition's last row */
    int64_t periods;          /* BL_SHIFT */
    const bl_column* values;  /* one chunk; NULL only for BL_AGG_LEN */
    bl_agg_param param;       /* BL_AGG_QUANTILE */
} bl_over_op;
/* mapping_strategy "group_to_rows": outs[i] has one row per input row, in input row order.
 * Partitions: the partition_by columns (numeric or string, one chunk for a numeric column, flags 0) group rows exactly as
 * bl_groupby_agg_keys / bl_groupby_agg_strings do (a null key is its own group, floats -0 == +0 and NaN == NaN, strings by
 * their bytes).  n_partition_by == 0: all rows form one partition (over() without keys, and the plain cum_sum() of a column).
 * Order inside a partition: row order (GroupsIdx), or with order_by (NULL or ONE key, numeric, Bool or string, its flags
 * BL_SORT_DESCENDING | BL_SORT_NULLS_LAST) each partition's rows stably sorted by that key in the total order (NaN greatest),
 * ties in row order (update_groups_sort_by, polars-expr/src/expressions/sortby.rs:57-100).
 * Aggregations (every BL_AGG_* kind, BL_AGG_WITH_DDOF, BL_AGG_N_UNIQUE, MEDIAN, QUANTILE through `param`): the group's value
 * on each of its rows, with the output dtypes, validity and errors of bl_groupby_agg_params.  order_by only changes what FIRST,
 * LAST, VAR / STD (Welford order) and float SUM / MEAN (sequential order) see: with order_by every aggregation is folded over
 * the sorted rows.  A Bool value column takes only BL_AGG_COUNT and BL_AGG_LEN.
 * Scans (polars-ops/src/series/ops/cum_agg.rs): a null input gives a null output and leaves the state unchanged (:14-53);
 * `reverse` scans from the partition's last row.
 *   BL_CUM_SUM    Int8/16, UInt8/16 -> Int64, Bool -> UInt32, 32/64-bit integers keep their dtype and wrap; Float64 in f64;
 *                 Float32 accumulates in f64 and rounds every output to f32 (det_sum_to_f64, :38-45; :302-333)
 *   BL_CUM_PROD   Bool, Int8..UInt32 -> Int64; Int64 / UInt64 keep their dtype and wrap; floats keep theirs (:261-285)
 *   BL_CUM_MIN / BL_CUM_MAX  keep the dtype; floats ignore NaN (the initial state is NaN, an all-NaN prefix gives NaN,
 *                 :78-112; the float impl of min_ignore_nan / max_ignore_nan is <$T>::min / <$T>::max,
 *                 polars-utils/src/min_max.rs:87-108, which returns the non-NaN argument).  Between two equal values
 *                 (only -0.0 and +0.0 differ in bits) MIN keeps the later in scan order and MAX the earlier: this tie rule
 *                 is this library's statement, not read from the reference (IEEE minNum / maxNum leave the sign of a zero
 *                 result open).  Bool: BL_ERR_UNSUPPORTED.
 *   BL_CUM_COUNT  UInt32, never null, any dtype: valid values in [partition start, row], reverse [row, partition end] (:428-466)
 *   BL_SHIFT      the value `periods` positions earlier in partition order (later for periods < 0), null when that position
 *                 is outside the partition or null; keeps the dtype.  Bool: BL_ERR_UNSUPPORTED.
 * Exactness: integer scans, CUM_MIN / MAX, CUM_COUNT and SHIFT are bit-identical to the reference.  Float CUM_SUM / CUM_PROD
 * run a parallel scan: at the k-th row of a partition's scan |dev - ref| <= 2 (k - 1) u sum_{i<=k} |a_i| (products:
 * 2 (k - 1) u |ref| while no partial product overflows or underflows), 0 for exactly summable values.  Under
 * bl_set_deterministic(1) each partition is folded sequentially in scan order and floats are bit-identical too.
 * Errors: BL_ERR_INVALID for value / key columns of different lengths, an unknown kind, partition flags != 0, unknown order_by
 * flags, a missing value column, no column at all to give the row count; BL_ERR_UNSUPPORTED for the dtypes above, Bool
 * partition columns, more than 2^31 - 1 rows when a sort is needed (partitioned scans, shifts, anything with order_by), and
 * the aggregation errors of bl_groupby_agg_params.  One order_by key per call: the caller sorts by several keys itself. */
bl_status bl_over(const bl_sort_key* partition_by, int32_t n_partition_by, const bl_sort_key* order_by, const bl_over_op* ops, int32_t n_ops,
                  int32_t out_location, bl_column* outs);

/* ---- rolling windows  (expr.rolling_*(window_size, min_samples, center), polars-compute/src/rolling; .over() as bl_over) ---- */
enum { BL_ROLLING_SUM = 40, BL_ROLLING_MEAN = 41, BL_ROLLING_MIN = 42, BL_ROLLING_MAX = 43, BL_ROLLING_VAR = 44, BL_ROLLING_STD = 45 };
typedef struct bl_rolling_op {
    int32_t kind;            /* BL_ROLLING_* */
    int32_t center;
    int64_t window_size;     /* >= 1 */
    int64_t min_samples;     /* 0 .. window_size */
    int32_t ddof;            /* VAR / STD, 0 .. 255 */
    int32_t reserved;        /* 0 */
    const bl_column* values; /* one chunk */
} bl_rolling_op;
/* outs[i] has one row per input row, in input row order.  partition_by / order_by: exactly bl_over's meaning and checks; each
 * partition is evaluated on its own, in partition order, and the results go back to the rows.
 * Window of the k-th position of a partition of m positions (w = window_size; polars-compute/src/rolling/mod.rs:72-87):
 *   trailing  [k - w + 1, k], center  [k - (w - r), k + r) with r = ceil(w / 2); both clipped to [0, m) (det_offsets /
 *   det_offsets_center, saturating_sub at the start, min(len, .) at the end).
 * Validity: null when the window holds fewer than min_samples non-null values (is_valid, rolling/sum.rs:219-221,
 * nulls/mod.rs:46-98; create_validity mod.rs:89-127 only nulls a subset of those rows).  The C ABI takes min_samples
 * explicitly (the Python default window_size is the binding's, polars-python/src/expr/rolling.rs:19).
 *   BL_ROLLING_SUM   Int8/16, UInt8/16 -> Int64, Bool -> UInt32, 32/64-bit integers keep their dtype and wrap
 *                    (polars-time/src/chunkedarray/rolling_window/dispatch.rs:284-312).  Floats keep theirs; only finite values
 *                    are summed, non-finite ones are counted: only +inf gives +inf, only -inf gives -inf, any other mix NaN
 *                    (rolling/sum.rs:68-108).  A window without non-null values sums to 0 (valid when min_samples == 0).
 *   BL_ROLLING_MEAN  Float32 for Float32, Float64 for everything else (to_float, dispatch.rs:238-249): the sum in f64 with the
 *                    same non-finite rule, cast to the output type, divided by the non-null count in that type
 *                    (rolling/mean.rs:98-108); a window without non-null values is null whatever min_samples.
 *   BL_ROLLING_MIN / BL_ROLLING_MAX  keep the dtype; NaN propagates (any NaN in the window gives NaN), and among equal values
 *                    (-0.0 / +0.0) the earliest in the window wins (ArgMinMaxWindow, rolling/arg_min_max.rs: a later value
 *                    replaces the deque's tail only when strictly better; MinPropagateNan / MaxPropagateNan,
 *                    polars-utils/src/min_max.rs:91-98,155-186).  A window without non-null values is null.  Bool: unsupported.
 *   BL_ROLLING_VAR / BL_ROLLING_STD  Float32 for Float32, Float64 otherwise, computed in f64 (VarState,
 *                    polars-compute/src/moment.rs:90-129): null when the non-null count <= ddof; a negative variance is 0;
 *                    any non-finite value in the window gives NaN (its validity still follows the count, rolling/moment.rs:
 *                    163-206).  Float32: (float)var; STD is sqrt of that value in the output type (dispatch.rs:565-576).
 * Temporal columns: pass their physical Int64 and convert the result back.
 * Exactness: integer SUM, every MIN / MAX, every validity bit and the non-finite class (NaN / +inf / -inf) of every window
 * holding a non-finite value are bit-identical to the reference.  Not reproduced: a window of finite values whose sum
 * overflows gives +-inf here, where the reference's Kahan state (f32 for Float32 SUM) overflows to inf and then to NaN
 * (err_add = inf, inf + -inf).  Finite float windows are reduced as two sequential runs joined by one combine (DESIGN.md §13); against
 * the EXACT value of a window of k non-null values a_i (u the unit roundoff of f64, u_o of the output type):
 *   SUM   |dev - exact| <= 1.01 (k - 1) u sum|a_i| + u_o |exact|
 *   MEAN  |dev - exact| <= (1.01 (k - 1) u sum|a_i| + u_o |sum|) / k + 2 u_o |exact|
 *   VAR   |dev - exact| <= 4.04 (k + 2) u sum (a_i - mean)^2 (1 + k mean^2 / sum (a_i - mean)^2)^(1/2) / (k - ddof) + u_o |exact|
 *   STD   |dev - exact| <= sqrt(the VAR bound) + u_o |exact|
 * These bound the distance to the exact window value, not to the reference's incremental Kahan / two-stack value, which
 * depends on the history of the column.  Under bl_set_deterministic(1), float SUM / MEAN / VAR / STD replay the reference's
 * state machines (SumWindow's Kahan add / sub and its reset when a window starts at or past the previous end; MomentWindow's
 * two stacks and flip) sequentially per partition and are bit-identical.
 * Plans (DESIGN.md §13), chosen from B = min(window_size, rows): B <= 128 runs one pass that stages each 1024-row tile and
 * its halo in shared memory; larger B writes per-block prefix and suffix states to device memory (2 x rows x 16..32 bytes of
 * scratch: 6.4 GB for VAR / STD over 1e8 rows) and its scans run ceil(rows / B) CTAs wide, so a window of a large share of
 * the column (say 1e7 of 1e8 rows) uses only a few SMs.
 * Errors: BL_ERR_INVALID for min_samples > window_size (dispatch.rs:42), a negative window_size or min_samples, ddof outside
 * 0..255, reserved != 0, an unknown kind, a missing value column, columns of different lengths and bl_over's key errors;
 * BL_ERR_UNSUPPORTED for window_size == 0, a Bool column for anything but SUM, Bool partition columns, more than 2^31 - 1
 * rows with partitions or order_by and more than 2^32 - 1 rows otherwise. */
bl_status bl_rolling(const bl_sort_key* partition_by, int32_t n_partition_by, const bl_sort_key* order_by, const bl_rolling_op* ops,
                     int32_t n_ops, int32_t out_location, bl_column* outs);

/* ---- time-based rolling windows  (expr.rolling_*_by(by, window_size, min_samples, closed), .over() as bl_rolling) ---- */
enum { BL_CLOSED_RIGHT = 0, BL_CLOSED_LEFT = 1, BL_CLOSED_BOTH = 2, BL_CLOSED_NONE = 3 };
typedef struct bl_rolling_by_op {
    int32_t kind;            /* BL_ROLLING_* */
    int32_t closed;          /* BL_CLOSED_* */
    int64_t window_size;     /* P >= 1, in the physical unit of `by` */
    int64_t min_samples;     /* >= 0 (no upper limit) */
    int32_t ddof;            /* VAR / STD, 0 .. 255 */
    int32_t reserved;        /* 0 */
    const bl_column* values; /* one chunk */
} bl_rolling_by_op;
/* outs[i] has one row per input row, in input row order.  partition_by: bl_rolling's meaning and checks (each partition is
 * evaluated on its own, as rolling_*_by(...).over(g) is).  Entry: rolling_agg_by, polars-time/src/chunkedarray/
 * rolling_window/dispatch.rs:71-218.
 * `by`: Int32, Int64, UInt32 or UInt64, one chunk, cast to Int64 as the reference does (:163-175).  A Date column is passed as
 * its days times 86 400 000 000 (the reference casts it to Datetime(us)), a Datetime as its physical Int64, and P in the
 * same unit: the Python binding parses durations ("5m", "1d", "3i") as Duration::add_ns / add_us / add_ms do
 * (duration.rs:929-1045, sub-unit parts truncated).  Calendar durations (mo, q, y) and d / w on time-zone-aware columns are
 * not expressible here.  Any other `by` dtype is BL_ERR_INVALID (:176-179); a UInt64 value >= 2^63 is BL_ERR_INVALID (the
 * reference's non-strict cast makes it null and then fails on cont_slice().unwrap()).
 * Order: each partition's rows sorted by `by`, ties in row order (a stable sort).  The reference arg-sorts an unsorted `by`
 * with an unstable sort (SortOptions::default()); the tie order decides only the float summation order and which of -0.0 /
 * +0.0 a MIN / MAX returns, which the reference leaves open.
 * Window of the row at time t (group_by_values_iter_lookbehind, polars-time/src/windows/group_by.rs:247-326): the rows of
 * its partition with lb < u <= t for BL_CLOSED_RIGHT, lb <= u <= t BOTH, lb <= u < t LEFT, lb < u < t NONE, lb = t - P
 * (Bounds::is_member, bounds.rs:33-60).  Rows with equal times share one window (the duplicate fast path, :286-291): with
 * RIGHT / BOTH it runs to the end of t's run of equal times; with LEFT / NONE it can be empty.  t - P is plain i64
 * arithmetic and wraps near i64::MIN, as the reference's does in a release build: a wrapped lower bound is above every
 * time, so such a row's window starts at its own run (empty for LEFT / NONE) and the reference's window start never moves
 * back before the last such run of its partition.
 * Output (rolling_apply_agg_window(_sorted), rolling_kernels/shared.rs:109-204): a window of fewer than min_samples rows,
 * nulls included, is null; otherwise the kind's bl_rolling rule below (dtypes, validity by non-null count, non-finite
 * classes, NaN-propagating MIN / MAX with the earliest of equal values, VarState) decides.  An empty window (min_samples
 * = 0): SUM 0 (valid), MEAN / MIN / MAX / VAR / STD null.  A row whose `by` is null is null and belongs to no window
 * (:101-129).  The Python defaults are min_samples 0 for rolling_sum_by and 1 for the others, closed "right", ddof 1.
 * Exactness: as bl_rolling.  Integer SUM, MIN / MAX, validity and non-finite classes are bit-identical; the SUM / MEAN
 * bounds of bl_rolling hold unchanged (they hold for any summation order of the window's k values).  A window is combined
 * from at most five runs (prefix, suffix, two sparse-table states, or the in-block equivalents), each itself a combination
 * of sequential runs, so the VAR bound takes the constant of DESIGN.md §14:
 *   VAR   |dev - exact| <= 8.08 (k + 4) u sum (a_i - mean)^2 (1 + k mean^2 / sum (a_i - mean)^2)^(1/2) / (k - ddof) + u_o |exact|
 *   STD   |dev - exact| <= sqrt(the VAR bound) + u_o |exact|
 * Under bl_set_deterministic(1) float SUM / MEAN / VAR / STD replay the reference's window machines over the same windows,
 * skipping update for the windows below min_samples; they are bit-identical when no two rows of a partition share a time
 * (with ties, the reference's unstable order decides).
 * Plans (DESIGN.md §14), chosen from the largest window W the bounds pass observes: W <= 128 runs one pass that stages each
 * 1024-row tile and 128 positions on each side in shared memory (device memory: 8 bytes per row of window bounds); wider
 * windows add blocks of 1024 positions with prefix / suffix states (2 x rows x 16..32 bytes: 6.4 GB for VAR over 1e8 rows)
 * and a disjoint sparse table over the block totals (2 x ceil(log2(rows / 1024)) x rows / 1024 states: 106 MB for VAR over
 * 1e8 rows).  The sort of the partitioned or unsorted form adds bl_over's.
 * Errors: BL_ERR_INVALID for window_size <= 0, a negative min_samples, ddof outside 0..255, reserved != 0, an unknown kind or
 * closed, a missing value or `by` column, the `by` dtypes and values above, columns of different lengths and bl_over's key
 * errors; BL_ERR_UNSUPPORTED for a Bool column for anything but SUM, Bool partition columns, more than 2^31 - 1 rows when a
 * sort is needed (partitions, a null or unsorted `by`) and more than 2^32 - 1 rows otherwise. */
bl_status bl_rolling_by(const bl_sort_key* partition_by, int32_t n_partition_by, const bl_column* by, const bl_rolling_by_op* ops,
                        int32_t n_ops, int32_t out_location, bl_column* outs);

/* ---- rolling quantile / median  (expr.rolling_quantile(...) / rolling_quantile_by(by, ...), plain or .over()) ---------- */
typedef struct bl_rolling_quantile_op {
    double quantile;          /* [0, 1] */
    int32_t method;           /* BL_QUANTILE_* */
    int32_t center;           /* 0 / 1 */
    int64_t window_size;      /* >= 1 */
    int64_t min_samples;      /* 0 .. window_size */
    const bl_column* values;  /* one chunk */
} bl_rolling_quantile_op;
typedef struct bl_rolling_quantile_by_op {
    double quantile;          /* [0, 1] */
    int32_t method;           /* BL_QUANTILE_* */
    int32_t closed;           /* BL_CLOSED_* */
    int64_t window_size;      /* P >= 1, in the physical unit of `by` */
    int64_t min_samples;      /* >= 0 */
    const bl_column* values;  /* one chunk */
} bl_rolling_quantile_by_op;
/* outs[i] has one row per input row, in input row order.  Partitions, order_by, the window of each row (center; by, closed,
 * P), the `by` dtypes and units, the order of a shuffled or null `by` and the row limits are exactly bl_rolling's and
 * bl_rolling_by's.  rolling_median(_by) is quantile 0.5 with BL_QUANTILE_LINEAR (polars-plan/src/dsl/mod.rs:1213-1215,
 * 1258-1260).  What differs:
 * Dtype: Float32 stays Float32, every other numeric dtype becomes Float64 (to_float, polars-core/src/series/mod.rs:629-634;
 * rolling_window/dispatch.rs:314-346), and all arithmetic happens in that type: a Float32 column interpolates in f32 (the
 * group_by quantile interpolates in f64).  Bool: BL_ERR_UNSUPPORTED.  Temporal value columns: pass their physical Int64.
 * Window order: the window's non-null values sorted by tot_cmp (NaN greatest, -0.0 == +0.0; SortedBuf, rolling/window.rs).
 * Index, with m the window's non-null count and all index arithmetic in f64 (no_nulls/quantile.rs:55-105,
 * nulls/quantile.rs:52-106, quantile_filter.rs:610-671):
 *   NEAREST       round((m - 1) q), half away from zero, clamped to m - 1
 *   LOWER         floor((m - 1) q)
 *   HIGHER        ceil((m - 1) q), clamped to m - 1
 *   EQUIPROBABLE  max(ceil(m q) - 1, 0)
 *   MIDPOINT      (lo + hi) / 2 in T when floor((m - 1) q) and ceil((m - 1) q) differ, else lo
 *   LINEAR        T((m - 1) q - floor((m - 1) q)) * (hi - lo) + lo in T when they differ (quantile_filter.rs:559-567), else lo
 * There is no lo == hi guard: LINEAR between +inf and +inf is NaN (inf - inf), unlike BL_AGG_QUANTILE.  The three reference
 * paths (no nulls centered, no nulls trailing through quantile_filter, with nulls) give the same index and arithmetic for q
 * in [0, 1]; only their clamps differ, and no clamp is reached there.
 * Validity: a window whose non-null count is below max(min_samples, 1) is null (is_valid, rolling/window.rs:179-181;
 * create_validity; an all-null window gives None, nulls/quantile.rs:58-61).  A time window also is null when it holds fewer
 * than min_samples rows, nulls included, or its row's `by` is null (rolling_kernels/shared.rs:109-204).  The Python defaults
 * are min_samples = window_size for fixed windows and 1 for time windows.
 * Exactness: bit-identical to the reference, except which of tot_eq values (-0.0 / +0.0, NaN payloads) a result takes: the
 * reference's sorted buffer leaves that open.  Every result is a value of its window or the interpolation of two of them.
 * bl_set_deterministic changes nothing.  weights are not in the ABI (the reference's weighted path differs and fails on nulls).
 * Plan (DESIGN.md §16): per value column, a wavelet matrix over the values' stable ranks (bl_arg_sort with nulls last) in
 * position order, L = max(1, ceil(log2 rows)) levels of 224-bit blocks with an interleaved rank directory (one 32-byte read
 * per rank query), then one thread per row: two rank queries per level for the k-th smallest of its window, two descents for
 * MIDPOINT / LINEAR.  The cost does not depend on the window width.  Ops whose `values` point to the same bl_column share one
 * matrix.  Device memory, beyond inputs and outputs: the sort's 24 bytes per row (freed before the build), 8 bytes per row of
 * ranks (two u32 orders), 4 or 8 bytes per row of sorted values, L x rows / 7 bytes of levels (rows / 7 more with nulls),
 * the 8 bytes per row of window bounds of a time window, and bl_over's order (with its inverse) when a sort is needed.
 * Errors: BL_ERR_INVALID for a quantile outside [0, 1] or NaN (the reference's rolling path has no range check and indexes
 * past the window: RollingQuantileParams { prob, method } reaches get_agg unchecked, rolling/mod.rs:140-143,
 * polars-plan/src/dsl/mod.rs:1181-1196), an unknown method, and otherwise
 * the window, `by` and key errors of bl_rolling / bl_rolling_by; BL_ERR_UNSUPPORTED for a Bool value column, window_size 0
 * (fixed windows) and the row limits of bl_rolling / bl_rolling_by. */
bl_status bl_rolling_quantile(const bl_sort_key* partition_by, int32_t n_partition_by, const bl_sort_key* order_by,
                              const bl_rolling_quantile_op* ops, int32_t n_ops, int32_t out_location, bl_column* outs);
bl_status bl_rolling_quantile_by(const bl_sort_key* partition_by, int32_t n_partition_by, const bl_column* by,
                                 const bl_rolling_quantile_by_op* ops, int32_t n_ops, int32_t out_location, bl_column* outs);

/* ---- rank  (expr.rank(method, descending, seed), plain or .over(partition_by, order_by); polars-ops/src/series/ops/rank.rs) ---- */
enum { BL_RANK_AVERAGE = 0, BL_RANK_MIN = 1, BL_RANK_MAX = 2, BL_RANK_DENSE = 3, BL_RANK_ORDINAL = 4, BL_RANK_RANDOM = 5 };
typedef struct bl_rank_op {
    int32_t method;             /* BL_RANK_* */
    int32_t descending;         /* rank the largest value 1 */
    uint64_t seed;              /* BL_RANK_RANDOM */
    const bl_sort_key* values;  /* a numeric / Boolean column (one chunk) or a LargeUtf8 / LargeBinary column; flags 0 */
} bl_rank_op;
/* outs[i] has one row per input row, in input row order.  partition_by / order_by: exactly bl_over's meaning and checks; each
 * partition is ranked on its own, as rank(...).over(g) is.  The C ABI takes the method explicitly (the Rust default is
 * Dense, rank.rs:32-39; the Python default is "average").
 * Per partition (rank.rs:61-188): the non-null values are stably arg-sorted with nulls last and `descending` as given
 * (:101-107), then split into tie runs where consecutive values are not equal (:117-123), equality being tot_eq: NaN ==
 * NaN, -0.0 == +0.0 (polars-utils/src/total_ord.rs:321-326).  NaN is the greatest value: last ascending, first descending.
 * Strings and binary compare their bytes unsigned, a proper prefix first.  A row at sorted position p (0-based among its
 * partition's non-null rows) in the run [s, e):
 *   BL_RANK_AVERAGE  Float64, 0.5 ((s + 1) + e) (:141-152), exact for every u32 rank
 *   BL_RANK_MIN      UInt32, s + 1 (:153-161)
 *   BL_RANK_MAX      UInt32, e (:162-170)
 *   BL_RANK_DENSE    UInt32, 1 + the number of runs before this one in the partition (:171-179)
 *   BL_RANK_ORDINAL  UInt32, p + 1 (:109-116): ties keep the stable order, row order, or with order_by the partition's
 *                    order_by order (its flags), then row order
 *   BL_RANK_RANDOM   UInt32, s + 1 + the row's place in a seeded random permutation of its run (:128-140)
 * A null value gives a null rank (the output validity is the input validity; the null slots hold 0, as the reference's
 * buffers do); an all-null partition is all null; an empty column gives an empty column of the method's dtype.
 * Temporal columns: pass their physical Int64.
 * Not reproduced: BL_RANK_RANDOM.  The reference shuffles each run with one sequential SmallRng, so how many values a run
 * consumes depends on every earlier run, and no parallel order gives its bytes (its seed-1 answer [2, 5, 7, 3, 4, 6, 1],
 * py-polars/tests/unit/operations/test_rank.py:27-32, is not this call's).  This call breaks ties by the 32-bit key
 * fmix32(fmix32(row ^ seed_lo) + seed_hi) (murmur3's finaliser, a bijection of the row index), then takes the ordinal rank:
 * the ranks of a run are a permutation of [s + 1, e], the same inputs and seed give the same bytes, and the permutation
 * passes a chi-square test of uniformity.  order_by changes only BL_RANK_ORDINAL.
 * Exactness: every other method is bit-identical to the reference.
 * Plan (DESIGN.md §15), per op: bl_arg_sort's stable radix sort of (partition id, value, tie key), then three passes over
 * the sorted positions: k_rank_heads (tie runs and partition starts as bitmaps, from one gather of the value per position),
 * k_rank_starts (each run's first position, MIN / MAX / AVERAGE and partitioned ranks only) and k_rank_out (the rank,
 * scattered to its row).  A string DENSE rank without partitions is bl_string_rank.  Several ops in one call share the
 * partition ids and the imported keys.
 * Device memory, beyond the inputs and outputs: the sort's 24 bytes per row (UInt32 permutation, its alternate and two u64
 * key buffers), up to three position bitmaps (3 / 8 bytes per row), 4 bytes per row of run starts, 4 bytes per row of
 * RANDOM's tie key and, with partitions, 4 bytes per row of partition ids and 4 to 8 bytes per row of partition starts.
 * Errors: BL_ERR_INVALID for an unknown method, values->flags != 0, a missing value column, a descriptor with both or neither
 * of `column` and `strings` set, columns of different lengths and bl_over's key errors; BL_ERR_UNSUPPORTED for Bool
 * partition columns, more than 2^31 - 1 rows with partitions or order_by and more than 2^32 - 1 rows otherwise. */
bl_status bl_rank(const bl_sort_key* partition_by, int32_t n_partition_by, const bl_sort_key* order_by, const bl_rank_op* ops, int32_t n_ops,
                  int32_t out_location, bl_column* outs);

/* ---- K6: radix hash partition (multi-GPU exchange step) --------------------------------- */
/* partition id = hash_to_partition(dirty_hash(key), n_partitions)
 *              = ((key * 0x55fbfd6bfc5458e9 mod 2^64) * n_partitions) >> 64   (hashing.rs:62-69,132-142),
 * null keys -> partition 0 (hashing.rs:113-115,183-187).  Rows are scattered so that partition p
 * occupies [offsets[p], offsets[p+1]) of every output column (the same permutation for every column; the row order
 * inside a partition is unspecified).
 * offsets: caller array of n_partitions+1 int64 (host). */
bl_status bl_hash_partition(const bl_column* key, const bl_column* payload, int32_t n_payload, int32_t n_partitions,
                            int32_t out_location, bl_column* out_key, bl_column* out_payload, int64_t* offsets);

/* ---- streaming group_by state (device-resident; used for chunked H2D overlap and multi-GPU) */
typedef struct bl_groupby bl_groupby;
/* key_dtype / value dtypes fix the plan; expected_groups <= 0 lets the library estimate.
 * track_first != 0 records each group's first row index (one extra 32-bit atomic per row); it is
 * required for bl_groupby_finish(maintain_order != 0). */
/* value_nullable[i] == 0 promises that aggregation i's column never carries nulls (saves its null
 * counter: smaller table entries); NULL = every column may be nullable.  MEDIAN / QUANTILE cannot be pre-aggregated:
 * BL_ERR_UNSUPPORTED here and in bl_groupby_agg_partitioned. */
bl_status bl_groupby_create(int32_t key_dtype, const int32_t* agg_kinds, const int32_t* value_dtypes, const int32_t* value_nullable,
                            int32_t n_aggs, int64_t expected_groups, int32_t track_first, bl_groupby** out);
/* Accumulate one batch: key + one value column per agg (values[i] ignored for LEN).  Columns may
 * be BL_HOST or BL_DEVICE.  row_base = global index of the batch's first row. */
bl_status bl_groupby_consume(bl_groupby* g, const bl_column* key, const bl_column* values, int64_t row_base);
/* Partial-aggregate exchange for the partitioned multi-GPU plan (SURVEY.md §8(e)):
 * export the table as dense rows of `*row_words` 64-bit words, scattered by key partition
 * (device memory, library-owned: free with bl_dev_free); offsets: n_partitions+1 int64 (host). */
bl_status bl_groupby_export_partials(bl_groupby* g, int32_t n_partitions, void** out_rows_dev, int32_t* row_words, int64_t* offsets);
/* Merge partial rows (from any rank) into this state. */
bl_status bl_groupby_merge_partials(bl_groupby* g, const void* rows_dev, int64_t n_rows);
/* Same for several regions (one per source rank) in one launch: rows_dev[i] holds n_rows[i] rows. */
bl_status bl_groupby_merge_partial_regions(bl_groupby* g, const void* const* rows_dev, const int64_t* n_rows, int32_t n_regions);
bl_status bl_groupby_finish(bl_groupby* g, int32_t maintain_order, int32_t out_location, bl_column* out_key, bl_column* out_aggs);
void bl_groupby_reset(bl_groupby* g);
void bl_groupby_destroy(bl_groupby* g);

/* ---- peer windows: fused partition + exchange over NVLink (one process per GPU) ----------- */
/* A window is plain device memory (cudaMalloc) exported with CUDA IPC so that the partition
 * kernels of the OTHER ranks can store into it directly (P2P stores over NVLink / NVSwitch):
 * partition and transfer are one kernel, no staging buffer, no NCCL on the data path.
 * Layout of a window used by bl_groupby_export_partials_p2p: n_ranks regions of
 * `rows_per_src` rows x row_words 64-bit words; region s is written only by rank s. */
typedef struct bl_window bl_window;
#define BL_IPC_HANDLE_BYTES 64
bl_status bl_window_create(size_t bytes, bl_window** out, void* ipc_handle_out /* BL_IPC_HANDLE_BYTES */);
void* bl_window_ptr(bl_window* w);
void bl_window_destroy(bl_window* w);
/* Maps a peer rank's window into this process (cudaIpcOpenMemHandle). */
bl_status bl_window_open(const void* ipc_handle, void** peer_ptr_out);
void bl_window_close(void* peer_ptr);
/* Fused K6 + exchange for the partitioned group_by: scatters this rank's partial-aggregate rows by
 * key partition straight into region `my_rank` of the destination rank's window.
 * windows[p] = device pointer of rank p's window as mapped in THIS process (own window for
 * p == my_rank).  sent_rows[p] (host) = rows written to rank p; the caller exchanges these counts and
 * merges region s of its own window with bl_groupby_merge_partials.  Returns after the kernel and
 * its peer stores have completed. */
bl_status bl_groupby_export_partials_p2p(bl_groupby* g, int32_t n_ranks, int32_t my_rank, void* const* windows, int64_t rows_per_src,
                                         int32_t* row_words, int64_t* sent_rows);

/* Exchange without host round trips.  window_halves[p] = base of the half of rank p's window used by this step (as
 * mapped in THIS process); a half is BL_WINDOW_HEADER_BYTES of header followed by n_ranks regions of rows_per_src
 * rows.  The export kernel stores the rows AND, from its last thread block, the per-destination row counts plus an
 * epoch flag into the destination headers (release, system scope); nothing is read back and the call returns as
 * soon as the kernel is queued.  `epoch` must grow from step to step (flags are never reset); windows must be
 * zero-initialised (bl_window_create does). */
#define BL_WINDOW_HEADER_BYTES 1024
bl_status bl_groupby_export_partials_p2p_async(bl_groupby* g, int32_t n_ranks, int32_t my_rank, void* const* window_halves, int64_t rows_per_src,
                                               uint64_t epoch, int32_t* row_words);
/* The owner's side: queues a kernel that waits (acquire, system scope, bounded) until every source rank has published
 * `epoch` in own_half's header, then merges the n_ranks regions into this state using the published counts.  Errors
 * (peer region overflow, peer timeout, table overflow) surface at bl_groupby_finish / bl_groupby_status. */
bl_status bl_groupby_merge_window_async(bl_groupby* g, const void* own_half, int32_t n_ranks, int64_t rows_per_src, uint64_t epoch);
/* on != 0: bl_groupby_consume no longer synchronises to check for table overflow; the check happens at
 * bl_groupby_finish (same state) or bl_groupby_status. */
void bl_groupby_defer_status(bl_groupby* g, int32_t on);
/* Synchronises and reports the state's device status word: 0 ok, 1 table overflow, 2 peer region overflow, 3 peer timeout. */
bl_status bl_groupby_status(bl_groupby* g, int32_t* status_out);
/* Sampled cardinality estimate of the consumed batches (0 before the first consume; no synchronisation). */
int64_t bl_groupby_estimated_groups(bl_groupby* g);

/* One rank's whole step of the partitioned group_by in ONE call (what polars_b200/dist.py composes from the pieces above):
 * local pre-aggregation of (key, aggs) -> bl_groupby_export_partials_p2p_async into the peers' window halves -> merge of this
 * rank's own half -> finish.  The outputs are the groups this rank owns (hash_to_partition(dirty_hash(key), n_ranks) ==
 * my_rank).  peer_halves[p] / own_half / rows_per_src / epoch as for the two calls it fuses; value columns one chunk each. */
bl_status bl_groupby_agg_partitioned(const bl_column* key, const bl_agg* aggs, int32_t n_aggs, int32_t n_ranks, int32_t my_rank,
                                     void* const* peer_halves, const void* own_half, int64_t rows_per_src, uint64_t epoch,
                                     int64_t expected_groups, int32_t out_location, bl_column* out_key, bl_column* out_aggs);

/* ---- profiling (CUDA events on the library stream) -------------------------------------- */
/* enable != 0: every kernel launch is bracketed by events; totals accumulate per kernel name. */
void bl_profile_enable(int32_t enable);
void bl_profile_reset(void);
/* Writes a JSON object {"kernel": {"launches": n, "ms": t}, ...} into buf; returns bytes needed. */
int64_t bl_profile_json(char* buf, int64_t cap);
/* Kernel launches issued by this library since bl_profile_reset (counted even when timing is off). */
int64_t bl_launch_count(void);

#ifdef __cplusplus
}
#endif
#endif /* POLARS_B200_H */
