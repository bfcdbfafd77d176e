// plugin.cu — boundary B1: the Polars expression-plugin ABI v0.1, served by the CUDA operators.
//
// A stock Polars build dlopen()s this library through `register_plugin_function`
// (py-polars/src/polars/plugins.py:24-37) and calls
//   _polars_plugin_get_version()                       crates/polars-plan/src/plans/aexpr/function_expr/plugin.rs:36-52
//   _polars_plugin_<name>(inputs, n, kwargs, kwargs_len, ret, ctx)          plugin.rs:70-137
//   _polars_plugin_field_<name>(fields, n, out, kwargs, kwargs_len)         plugin.rs:178-217
//   _polars_plugin_get_last_error_message()                                 plugin.rs:139-158
// with SeriesExport / CallerContext as in crates/polars-ffi/src/version_0.rs:7-16,134-140 and
// Arrow C Data Interface structs (crates/polars-arrow/src/ffi/generated.rs:6-34).
// Ownership (plugin.rs:118-125): the caller forgets the inputs, so this side releases every input
// array and every input SeriesExport; the return value carries its own release callbacks.
// Errors: `ret` is left untouched (private_data == NULL) and the message is kept thread-local.
#include <cmath>
#include <cstdlib>
#include <random>
#include <string>
#include <vector>

#include "common.cuh"
#include "groupby.h"

using namespace plb;

extern "C" {
struct ArrowSchema {
    const char* format; const char* name; const char* metadata; int64_t flags; int64_t n_children;
    struct ArrowSchema** children; struct ArrowSchema* dictionary; void (*release)(struct ArrowSchema*); void* private_data;
};
struct ArrowArray {
    int64_t length; int64_t null_count; int64_t offset; int64_t n_buffers; int64_t n_children;
    const void** buffers; struct ArrowArray** children; struct ArrowArray* dictionary; void (*release)(struct ArrowArray*); void* private_data;
};
struct SeriesExport {
    ArrowSchema* field; ArrowArray** arrays; size_t len; void (*release)(SeriesExport*); void* private_data;
};
struct CallerContext { uint64_t bitflags; };
}

static thread_local std::string t_plugin_error;

static int dtype_from_format(const char* f) {
    if (!f || !f[0] || f[1]) return -1;
    switch (f[0]) {
        case 'c': return BL_INT8; case 's': return BL_INT16; case 'i': return BL_INT32; case 'l': return BL_INT64;
        case 'C': return BL_UINT8; case 'S': return BL_UINT16; case 'I': return BL_UINT32; case 'L': return BL_UINT64;
        case 'f': return BL_FLOAT32; case 'g': return BL_FLOAT64; case 'b': return BL_BOOL;
        default: return -1;
    }
}
static const char* format_of(int dt) {
    static const char* f[] = {"c", "s", "i", "l", "C", "S", "I", "L", "f", "g", "b"};
    return f[dt];
}

// ---- schema / array construction with release callbacks -----------------------------------------
struct SchemaPriv { std::string name, format; std::vector<ArrowSchema*> kids; };
static void release_schema(ArrowSchema* s) {
    if (!s || !s->release) return;
    auto* p = reinterpret_cast<SchemaPriv*>(s->private_data);
    for (auto* k : p->kids) { if (k->release) k->release(k); free(k); }
    delete p;
    s->release = nullptr;
}
static void fill_schema(ArrowSchema* out, const std::string& name, const std::string& format, const std::vector<std::pair<std::string, int>>& children = {}) {
    auto* p = new SchemaPriv{name, format, {}};
    for (auto& c : children) {
        auto* k = reinterpret_cast<ArrowSchema*>(calloc(1, sizeof(ArrowSchema)));
        fill_schema(k, c.first, format_of(c.second));
        p->kids.push_back(k);
    }
    out->format = p->format.c_str(); out->name = p->name.c_str(); out->metadata = nullptr;
    out->flags = 2 /* ARROW_FLAG_NULLABLE */; out->n_children = (int64_t)p->kids.size();
    out->children = p->kids.empty() ? nullptr : p->kids.data(); out->dictionary = nullptr;
    out->release = release_schema; out->private_data = p;
}

struct ArrayPriv { bl_column col; const void* bufs[2]; std::vector<ArrowArray*> kids; };
static void release_array(ArrowArray* a) {
    if (!a || !a->release) return;
    auto* p = reinterpret_cast<ArrayPriv*>(a->private_data);
    for (auto* k : p->kids) { if (k->release) k->release(k); free(k); }
    bl_column_free(&p->col);
    delete p;
    a->release = nullptr;
}
static void fill_array(ArrowArray* out, const bl_column& col) {   // takes ownership of a host bl_column
    auto* p = new ArrayPriv();
    p->col = col; p->bufs[0] = col.validity; p->bufs[1] = col.values;
    out->length = col.length; out->null_count = col.validity ? -1 : 0; out->offset = 0; out->n_buffers = 2; out->n_children = 0;
    out->buffers = p->bufs; out->children = nullptr; out->dictionary = nullptr; out->release = release_array; out->private_data = p;
}
static void fill_struct_array(ArrowArray* out, const std::vector<bl_column>& kids) {
    auto* p = new ArrayPriv();
    memset(&p->col, 0, sizeof p->col);
    p->bufs[0] = nullptr;
    for (auto& k : kids) { auto* a = reinterpret_cast<ArrowArray*>(calloc(1, sizeof(ArrowArray))); fill_array(a, k); p->kids.push_back(a); }
    out->length = kids.empty() ? 0 : kids[0].length; out->null_count = 0; out->offset = 0; out->n_buffers = 1; out->n_children = (int64_t)p->kids.size();
    out->buffers = p->bufs; out->children = p->kids.data(); out->dictionary = nullptr; out->release = release_array; out->private_data = p;
}

struct SeriesPriv { ArrowSchema* schema; ArrowArray** arrays; size_t n; };
static void release_series(SeriesExport* e) {
    if (!e || !e->release) return;
    auto* p = reinterpret_cast<SeriesPriv*>(e->private_data);
    // the importer moved the ArrowArray structs out (ptr::read, version_0.rs:92-104): free the boxes only
    for (size_t i = 0; i < p->n; i++) free(p->arrays[i]);
    free(p->arrays);
    if (p->schema->release) p->schema->release(p->schema);
    free(p->schema);
    delete p;
    e->release = nullptr;
}
static void make_series(SeriesExport* ret, ArrowSchema* schema, ArrowArray* array) {
    auto* p = new SeriesPriv{schema, reinterpret_cast<ArrowArray**>(calloc(1, sizeof(ArrowArray*))), 1};
    p->arrays[0] = array;
    ret->field = schema; ret->arrays = p->arrays; ret->len = 1; ret->release = release_series; ret->private_data = p;
}

// ---- inputs --------------------------------------------------------------------------------------
static std::vector<bl_column> input_chunks(const SeriesExport& s, int* dtype_out) {
    int dt = dtype_from_format(s.field ? s.field->format : nullptr);
    PLB_REQUIRE(dt >= 0, BL_ERR_UNSUPPORTED, std::string("plugin: unsupported input dtype '") + (s.field && s.field->format ? s.field->format : "?") + "'");
    std::vector<bl_column> ch;
    for (size_t i = 0; i < s.len; i++) {
        const ArrowArray* a = s.arrays[i];
        bl_column c; memset(&c, 0, sizeof c);
        c.dtype = dt; c.location = BL_HOST; c.length = a->length; c.offset = a->offset; c.null_count = a->null_count;
        c.validity = a->n_buffers > 0 ? reinterpret_cast<const uint8_t*>(a->buffers[0]) : nullptr;
        c.values = a->n_buffers > 1 ? a->buffers[1] : nullptr;
        ch.push_back(c);
    }
    if (ch.empty()) { bl_column c; memset(&c, 0, sizeof c); c.dtype = dt; c.null_count = 0; static const uint64_t z = 0; c.values = &z; ch.push_back(c); }
    *dtype_out = dt;
    return ch;
}
static void release_inputs(SeriesExport* inputs, size_t n) {
    for (size_t i = 0; i < n; i++) {
        for (size_t j = 0; j < inputs[i].len; j++) { ArrowArray* a = inputs[i].arrays[j]; if (a && a->release) a->release(a); }
        if (inputs[i].release) inputs[i].release(&inputs[i]);
    }
}

enum PluginOp { P_ARITH, P_CMP, P_FILTER, P_GATHER, P_GROUP, P_JOIN, P_SORT, P_OVER, P_ROLL, P_ROLL_BY, P_RANK, P_ROLL_Q, P_ROLL_Q_BY, P_TOP_K, P_UNIQUE, P_DISTINCT };

// ---- kwargs ----------------------------------------------------------------------------------------
// register_plugin_function(kwargs={...}) pickles the dict (py-polars/src/polars/plugins.py:100-115) and the caller hands
// the bytes through (plugin.rs:70-137; Rust plugins read them with serde-pickle).  The subset a flat {str: bool | int |
// float | str | None} dict produces under protocols 2..5 is parsed here: PROTO FRAME EMPTY_DICT MARK (SHORT_)BINUNICODE
// BININT BININT1 BININT2 LONG1 BINFLOAT NEWTRUE NEWFALSE NONE MEMOIZE BINPUT SETITEM SETITEMS STOP.
struct Kwargs { std::vector<std::pair<std::string, double>> num; std::vector<std::pair<std::string, std::string>> str; std::vector<std::string> bools, nones;
    double get(const char* k, double dflt) const { for (auto& e : num) if (e.first == k) return e.second; return dflt; }
    bool is_bool(const char* k) const { for (auto& e : bools) if (e == k) return true; return false; }
    bool is_none(const char* k) const { for (auto& e : nones) if (e == k) return true; return false; }
    std::string gets(const char* k, const char* dflt) const { for (auto& e : str) if (e.first == k) return e.second; return dflt; } };
static Kwargs parse_kwargs(const uint8_t* p, size_t n) {
    Kwargs kw;
    if (!p || n == 0) return kw;
    struct Val { int kind; double num; std::string s; };      // kind: 0 none, 1 number, 2 string, 3 dict marker, 4 mark, 5 bool
    std::vector<Val> st;
    size_t i = 0;
    auto need = [&](size_t k) { PLB_REQUIRE(i + k <= n, BL_ERR_INVALID, "plugin kwargs: truncated pickle"); };
    auto flush_items = [&](size_t from) {      // st[from..] = key, value, key, value ... -> into kw
        for (size_t j = from; j + 1 < st.size(); j += 2) {
            PLB_REQUIRE(st[j].kind == 2, BL_ERR_UNSUPPORTED, "plugin kwargs: only string keys are supported");
            if (st[j + 1].kind == 2) kw.str.push_back({st[j].s, st[j + 1].s});
            else kw.num.push_back({st[j].s, (st[j + 1].kind == 1 || st[j + 1].kind == 5) ? st[j + 1].num : 0.0});
            if (st[j + 1].kind == 5) kw.bools.push_back(st[j].s);
            if (st[j + 1].kind == 0) kw.nones.push_back(st[j].s);
        }
        st.resize(from);
    };
    while (i < n) {
        const uint8_t op = p[i++];
        switch (op) {
            case 0x80: need(1); i += 1; break;                                   // PROTO
            case 0x95: need(8); i += 8; break;                                   // FRAME
            case '}': st.push_back({3, 0, ""}); break;                           // EMPTY_DICT
            case '(': st.push_back({4, 0, ""}); break;                           // MARK
            case 0x94: break;                                                    // MEMOIZE
            case 'q': need(1); i += 1; break;                                    // BINPUT
            case 'r': need(4); i += 4; break;                                    // LONG_BINPUT
            case 0x8c: { need(1); const size_t l = p[i++]; need(l); st.push_back({2, 0, std::string((const char*)p + i, l)}); i += l; break; }      // SHORT_BINUNICODE
            case 'X': { need(4); size_t l = p[i] | (p[i + 1] << 8) | (p[i + 2] << 16) | ((size_t)p[i + 3] << 24); i += 4; need(l); st.push_back({2, 0, std::string((const char*)p + i, l)}); i += l; break; }
            case 'K': need(1); st.push_back({1, (double)p[i], ""}); i += 1; break;                                                           // BININT1
            case 'M': need(2); st.push_back({1, (double)(p[i] | (p[i + 1] << 8)), ""}); i += 2; break;                                     // BININT2
            case 'J': { need(4); int32_t v; memcpy(&v, p + i, 4); st.push_back({1, (double)v, ""}); i += 4; break; }                        // BININT
            case 0x8a: { need(1); const size_t l = p[i++]; need(l); int64_t v = 0; for (size_t b = 0; b < l && b < 8; b++) v |= (int64_t)p[i + b] << (8 * b);
                         if (l > 0 && l < 8 && (p[i + l - 1] & 0x80)) v |= -((int64_t)1 << (8 * l)); st.push_back({1, (double)v, ""}); i += l; break; }  // LONG1
            case 'G': { need(8); uint64_t b = 0; for (int k = 0; k < 8; k++) b = (b << 8) | p[i + k]; double d; memcpy(&d, &b, 8); st.push_back({1, d, ""}); i += 8; break; }   // BINFLOAT (big endian)
            case 0x88: st.push_back({5, 1.0, ""}); break;                        // NEWTRUE
            case 0x89: st.push_back({5, 0.0, ""}); break;                        // NEWFALSE
            case 'N': st.push_back({0, 0, ""}); break;                           // NONE
            case 's': { PLB_REQUIRE(st.size() >= 3, BL_ERR_INVALID, "plugin kwargs: malformed pickle"); flush_items(st.size() - 2); break; }       // SETITEM
            case 'u': { size_t m = st.size(); while (m > 0 && st[m - 1].kind != 4) m--; PLB_REQUIRE(m > 0, BL_ERR_INVALID, "plugin kwargs: malformed pickle");
                        flush_items(m); st.pop_back(); break; }                  // SETITEMS (pops the MARK)
            case '.': return kw;                                                 // STOP
            default: fail(BL_ERR_UNSUPPORTED, "plugin kwargs: unsupported pickle opcode " + std::to_string((int)op) + " (flat dicts of bool / int / float / str only)");
        }
    }
    return kw;
}

static int join_how_of(int op) { return op; }

// closed: "right" / "left" / "both" / "none", or its BL_CLOSED_* code (default "right")
static int closed_kwarg(const Kwargs& kw) {
    const std::string cs = kw.gets("closed", "");
    if (!cs.empty()) {
        const char* names[] = {"right", "left", "both", "none"};      // BL_CLOSED_RIGHT .. BL_CLOSED_NONE
        int closed = -1;
        for (int c = 0; c < 4; c++) if (cs == names[c]) closed = c;
        PLB_REQUIRE(closed >= 0, BL_ERR_INVALID, "plugin rolling_*_by: unknown closed '" + cs + "'");
        return closed;
    }
    const double c = kw.get("closed", BL_CLOSED_RIGHT);
    PLB_REQUIRE(!kw.is_bool("closed") && c == std::floor(c) && c >= BL_CLOSED_RIGHT && c <= BL_CLOSED_NONE, BL_ERR_INVALID,
                "plugin rolling_*_by: closed must be 'right', 'left', 'both', 'none' or its code 0..3");
    return (int)c;
}

// quantile (float, required) and method (str, default "nearest"), as group_quantile takes them
static void quantile_kwargs(const Kwargs& kw, const char* who, double& q, int& method) {
    q = kw.get("quantile", std::nan(""));
    PLB_REQUIRE(!std::isnan(q), BL_ERR_INVALID, std::string("plugin ") + who + ": the `quantile` kwarg is required");
    const std::string m = kw.gets("method", "nearest");
    static const char* names[] = {"nearest", "lower", "higher", "midpoint", "linear", "equiprobable"};
    method = -1;
    for (int j = 0; j < 6; j++) if (m == names[j]) method = j;
    PLB_REQUIRE(method >= 0, BL_ERR_INVALID, std::string("plugin ") + who + ": unknown method '" + m + "'");
}

// the kwargs carry numbers as doubles: only integers up to 2^53 arrive exactly
static void require_int_kwargs(std::initializer_list<double> vs, const char* who) {
    for (double v : vs)
        PLB_REQUIRE(v == std::floor(v) && std::fabs(v) <= 9007199254740992.0, BL_ERR_INVALID, std::string("plugin ") + who + ": window_size and min_samples must be integers of at most 2^53");
}

static void run_plugin(PluginOp kind, int op, SeriesExport* inputs, size_t n, const Kwargs& kw, SeriesExport* ret) {
    std::lock_guard<std::recursive_mutex> lk(ctx().mu);
    PLB_REQUIRE(n >= 1, BL_ERR_INVALID, "plugin: no input series");
    if (kind != P_GROUP && kind != P_JOIN && kind != P_SORT && kind != P_OVER && kind != P_ROLL && kind != P_ROLL_BY && kind != P_RANK && kind != P_ROLL_Q && kind != P_ROLL_Q_BY && kind != P_TOP_K && kind != P_UNIQUE && kind != P_DISTINCT) PLB_REQUIRE(n == 2, BL_ERR_INVALID, "plugin: expected exactly 2 input series");
    std::vector<std::vector<bl_column>> chunks(n);
    std::vector<DevCol> in;
    for (size_t i = 0; i < n; i++) { int dt; chunks[i] = input_chunks(inputs[i], &dt); in.push_back(import_column(chunks[i].data(), (int)chunks[i].size())); }
    const std::string name = inputs[0].field && inputs[0].field->name ? inputs[0].field->name : "";
    auto* schema = reinterpret_cast<ArrowSchema*>(calloc(1, sizeof(ArrowSchema)));
    auto* array = reinterpret_cast<ArrowArray*>(calloc(1, sizeof(ArrowArray)));
    auto export_struct = [&](const std::vector<DevCol>& cols, const std::vector<std::string>& names) {
        std::vector<bl_column> h(cols.size());
        size_t done = 0;
        try { for (; done < cols.size(); done++) export_column(cols[done], BL_HOST, &h[done]); }
        catch (...) { for (size_t j = 0; j < done; j++) bl_column_free(&h[j]); throw; }
        fill_struct_array(array, h);
        std::vector<std::pair<std::string, int>> kids;
        for (size_t j = 0; j < cols.size(); j++) kids.push_back({names[j], cols[j].dtype});
        fill_schema(schema, name, "+s", kids);
    };
    try {
        if (kind == P_ARITH || kind == P_CMP || kind == P_FILTER || kind == P_GATHER) {
            const DevCol &a = in[0], &b = in[1];
            DevCol o;
            if (kind == P_ARITH) o = op_elementwise(op, a, b);
            else if (kind == P_CMP) o = op_compare(op, a, b, kw.get("missing", 0) != 0);
            else if (kind == P_FILTER) { std::vector<DevCol> outs; op_filter({a}, b, outs); o = outs[0]; }
            else { std::vector<DevCol> outs; op_gather({a}, b, true, outs); o = outs[0]; }
            bl_column h; export_column(o, BL_HOST, &h);
            fill_array(array, h);
            fill_schema(schema, name, format_of(o.dtype));
        } else if (kind == P_SORT) {
            // inputs: the `by` columns -> UInt32 permutation.  kwargs descending / nulls_last: a bool (every column) or an int
            // bitmask (bit i = column i)
            std::vector<int> flags(n, 0);
            for (size_t j = 0; j < n; j++) {
                for (auto f : {std::make_pair("descending", (int)BL_SORT_DESCENDING), std::make_pair("nulls_last", (int)BL_SORT_NULLS_LAST)}) {
                    const int64_t v = (int64_t)kw.get(f.first, 0);
                    if (kw.is_bool(f.first) ? v != 0 : j < 63 && ((v >> j) & 1)) flags[j] |= f.second;
                }
            }
            DevCol perm = op_arg_sort(in, flags, -1);
            bl_column h; export_column(perm, BL_HOST, &h);
            fill_array(array, h);
            fill_schema(schema, name, format_of(BL_UINT32));
        } else if (kind == P_UNIQUE || kind == P_DISTINCT) {
            // inputs: the key columns (numeric or Boolean).  bl_arg_unique -> the kept rows as ascending UInt32 row ids, kwarg
            // keep ("first" (default), "last", "any", "none"); bl_is_* -> one Boolean per row
            int mk = op;
            if (kind == P_UNIQUE) {
                const std::string keep = kw.gets("keep", "first");
                static const char* names[] = {"first", "last", "any", "none"};      // BL_UNIQUE_FIRST .. BL_UNIQUE_NONE
                int k = -1;
                for (int j = 0; j < 4; j++) if (keep == names[j]) k = j;
                PLB_REQUIRE(k >= 0, BL_ERR_INVALID, "`keep` must be one of {'first', 'last', 'any', 'none'}, got " + keep);
                mk = k == BL_UNIQUE_LAST ? BL_DISTINCT_LAST : k == BL_UNIQUE_NONE ? BL_DISTINCT_UNIQUE : BL_DISTINCT_FIRST;
            }
            for (auto& c : in) PLB_REQUIRE(sortable_dtype(c.dtype), BL_ERR_UNSUPPORTED, std::string("plugin unique: key dtype ") + dtype_name(c.dtype) + " is not supported");
            DevCol o = op_unique_mask(in, mk);
            if (kind == P_UNIQUE) o = op_mask_rows(as<uint32_t>(o.values), o.len);
            bl_column h; export_column(o, BL_HOST, &h);
            fill_array(array, h);
            fill_schema(schema, name, format_of(o.dtype));
        } else if (kind == P_TOP_K) {
            // inputs: the `by` columns -> the UInt32 ids of the first k rows, best first (DataFrame.top_k / bottom_k:
            // descending = !reverse for top (op 0), reverse for bottom (op 1), nulls last).  kwargs: k (int, required),
            // reverse (a bool or an int bitmask, bit i = column i)
            const double kd = kw.is_none("k") ? std::nan("") : kw.get("k", std::nan(""));
            PLB_REQUIRE(!std::isnan(kd) && !kw.is_bool("k"), BL_ERR_INVALID, "plugin top_k: the `k` kwarg is required");
            PLB_REQUIRE(kd == std::floor(kd) && kd >= 0 && kd <= 9007199254740992.0, BL_ERR_INVALID, "plugin top_k: k must be an integer >= 0");
            const int64_t rv = (int64_t)kw.get("reverse", 0);
            std::vector<int> flags(n, BL_SORT_NULLS_LAST);
            for (size_t j = 0; j < n; j++) {
                const bool reverse = kw.is_bool("reverse") ? rv != 0 : j < 63 && ((rv >> j) & 1);
                if (reverse == (op == 1)) flags[j] |= BL_SORT_DESCENDING;
            }
            DevCol perm = op_arg_sort(in, flags, (int64_t)kd);
            bl_column h; export_column(perm, BL_HOST, &h);
            fill_array(array, h);
            fill_schema(schema, name, format_of(BL_UINT32));
        } else if (kind == P_OVER) {
            // inputs: the values, then the partition keys (none: one partition) -> one row per input row (bl_over).
            // kwargs: reverse (bool), periods (int, default 1)
            check_over_op(op, in[0].dtype);
            OverOp o;
            o.kind = op; o.reverse = kw.get("reverse", 0) != 0; o.periods = (int64_t)kw.get("periods", 1); o.values = &in[0];
            const std::vector<DevCol> parts(in.begin() + 1, in.end());
            const DevCol r = op_over(parts, nullptr, 0, {o}, in[0].len)[0];
            bl_column h; export_column(r, BL_HOST, &h);
            fill_array(array, h);
            fill_schema(schema, name, format_of(r.dtype));
        } else if (kind == P_ROLL) {
            // inputs: the values, then the partition keys (none: one partition) -> one row per input row (bl_rolling).
            // kwargs: window_size (int, required), min_samples (int; absent or None: window_size, as rolling_*(min_samples=None)
            // means), center (bool), ddof (int, default 1)
            const double ws = kw.is_none("window_size") ? std::nan("") : kw.get("window_size", std::nan(""));
            PLB_REQUIRE(!std::isnan(ws), BL_ERR_INVALID, "plugin rolling_*: the `window_size` kwarg is required");
            RollOp o;
            o.kind = op; o.window_size = (int64_t)ws; o.min_samples = kw.is_none("min_samples") ? (int64_t)ws : (int64_t)kw.get("min_samples", ws); o.center = kw.get("center", 0) != 0;
            o.ddof = (int)kw.get("ddof", 1); o.values = &in[0];
            check_rolling_op(o.kind, o.center ? 1 : 0, o.window_size, o.min_samples, o.ddof, 0, in[0].dtype);
            const std::vector<DevCol> parts(in.begin() + 1, in.end());
            const DevCol r = op_rolling(parts, nullptr, 0, {o}, in[0].len)[0];
            bl_column h; export_column(r, BL_HOST, &h);
            fill_array(array, h);
            fill_schema(schema, name, format_of(r.dtype));
        } else if (kind == P_ROLL_BY) {
            // inputs: the values, the `by` column, then the partition keys -> one row per input row (bl_rolling_by).
            // kwargs: window_size (int, required, in the physical unit of `by`), min_samples (int; absent or None: 0 for
            // rolling_sum_by and 1 for the others, as the Python signatures default), closed ("right" / "left" / "both" /
            // "none" or its BL_CLOSED_* code, default "right"), ddof (int, default 1)
            PLB_REQUIRE(n >= 2, BL_ERR_INVALID, "plugin rolling_*_by: expected the values and the `by` column");
            const double ws = kw.is_none("window_size") ? std::nan("") : kw.get("window_size", std::nan(""));
            PLB_REQUIRE(!std::isnan(ws), BL_ERR_INVALID, "plugin rolling_*_by: the `window_size` kwarg is required");
            const double ms = kw.is_none("min_samples") ? (op == BL_ROLLING_SUM ? 0 : 1) : kw.get("min_samples", op == BL_ROLLING_SUM ? 0 : 1);
            require_int_kwargs({ws, ms}, "rolling_*_by");
            const int closed = closed_kwarg(kw);
            RollByOp o;
            o.kind = op; o.window_size = (int64_t)ws; o.min_samples = (int64_t)ms;
            o.closed = closed; o.ddof = (int)kw.get("ddof", 1); o.values = &in[0];
            check_rolling_by_op(o.kind, o.closed, o.window_size, o.min_samples, o.ddof, 0, in[0].dtype);
            const std::vector<DevCol> parts(in.begin() + 2, in.end());
            const DevCol r = op_rolling_by(parts, in[1], {o}, in[0].len)[0];
            bl_column h; export_column(r, BL_HOST, &h);
            fill_array(array, h);
            fill_schema(schema, name, format_of(r.dtype));
        } else if (kind == P_ROLL_Q || kind == P_ROLL_Q_BY) {
            // rolling_quantile / rolling_median (op 1: quantile 0.5, "linear") and their _by forms.  inputs: the values (then
            // the `by` column for _by), then the partition keys.  kwargs: quantile and method (rolling_quantile*, as
            // group_quantile takes them), window_size (int, required; _by: in the physical unit of `by`), min_samples (int;
            // absent or None: window_size, or 1 for _by), center (bool) or closed (as rolling_*_by)
            const bool by = kind == P_ROLL_Q_BY;
            const char* who = by ? "rolling_quantile_by" : "rolling_quantile";
            PLB_REQUIRE(!by || n >= 2, BL_ERR_INVALID, "plugin rolling_quantile_by: expected the values and the `by` column");
            RollQuantileOp o;
            if (op == 0) quantile_kwargs(kw, who, o.quantile, o.method);
            const double ws = kw.is_none("window_size") ? std::nan("") : kw.get("window_size", std::nan(""));
            PLB_REQUIRE(!std::isnan(ws), BL_ERR_INVALID, std::string("plugin ") + who + ": the `window_size` kwarg is required");
            const double ms = kw.is_none("min_samples") ? (by ? 1 : ws) : kw.get("min_samples", by ? 1 : ws);
            require_int_kwargs({ws, ms}, who);
            o.window_size = (int64_t)ws; o.min_samples = (int64_t)ms; o.values = &in[0];
            if (by) {
                o.closed = closed_kwarg(kw);
                check_rolling_quantile_by_op(o.quantile, o.method, o.closed, o.window_size, o.min_samples, in[0].dtype);
            } else {
                o.center = kw.get("center", 0) != 0;
                check_rolling_quantile_op(o.quantile, o.method, o.center ? 1 : 0, o.window_size, o.min_samples, in[0].dtype);
            }
            const std::vector<DevCol> parts(in.begin() + (by ? 2 : 1), in.end());
            const DevCol r = by ? op_rolling_quantile_by(parts, in[1], {o}, in[0].len)[0] : op_rolling_quantile(parts, nullptr, 0, {o}, in[0].len)[0];
            bl_column h; export_column(r, BL_HOST, &h);
            fill_array(array, h);
            fill_schema(schema, name, format_of(r.dtype));
        } else if (kind == P_RANK) {
            // inputs: the values, then the partition keys (none: one partition) -> one row per input row (bl_rank).
            // kwargs: descending (bool), seed (int for bl_rank_random; absent or None: drawn here)
            RankOp o;
            o.method = op; o.descending = kw.get("descending", 0) != 0; o.values = &in[0];
            const double sd = kw.is_none("seed") ? std::nan("") : kw.get("seed", std::nan(""));
            if (std::isnan(sd)) { std::random_device rd; o.seed = ((uint64_t)rd() << 32) | rd(); }
            else {
                // the kwargs carry numbers as doubles: only integers up to 2^53 arrive exactly
                PLB_REQUIRE(!kw.is_bool("seed") && sd == std::floor(sd) && sd >= 0 && sd <= 9007199254740992.0, BL_ERR_INVALID,
                            "plugin rank_*: seed must be an integer in 0..2^53");
                o.seed = (uint64_t)sd;
            }
            const std::vector<DevCol> parts(in.begin() + 1, in.end());
            const DevCol r = op_rank(parts, nullptr, 0, {o}, in[0].len)[0];
            bl_column h; export_column(r, BL_HOST, &h);
            fill_array(array, h);
            fill_schema(schema, name, format_of(r.dtype));
        } else if (kind == P_GROUP) {
            // inputs: key_0 .. key_{k-1}, value (LEN: keys only)  ->  struct {key, key_1, ..., agg}, groups in first-occurrence order
            const bool is_len = op == BL_AGG_LEN;
            PLB_REQUIRE(is_len ? n >= 1 : n >= 2, BL_ERR_INVALID, "plugin group_*: expected key column(s) followed by the value column");
            const size_t nk = is_len ? n : n - 1;
            int agg_kind = op;
            if (op == BL_AGG_VAR || op == BL_AGG_STD) agg_kind = BL_AGG_WITH_DDOF(op, (int)kw.get("ddof", 1));
            bl_agg_param qp{0.5, BL_QUANTILE_LINEAR, 0};
            if (op == BL_AGG_QUANTILE) {      // kwargs: quantile (float, required), method (str, default "nearest")
                qp.quantile = kw.get("quantile", std::nan(""));
                PLB_REQUIRE(!std::isnan(qp.quantile), BL_ERR_INVALID, "plugin group_quantile: the `quantile` kwarg is required");
                const std::string m = kw.gets("method", "nearest");
                static const char* names[] = {"nearest", "lower", "higher", "midpoint", "linear", "equiprobable"};
                qp.method = -1;
                for (int j = 0; j < 6; j++) if (m == names[j]) qp.method = j;
                PLB_REQUIRE(qp.method >= 0, BL_ERR_INVALID, "plugin group_quantile: unknown method '" + m + "'");
            }
            // median / quantile are Float64 for every integer width: 8/16-bit columns aggregate as Int64, as in bl_groupby_agg
            if ((op == BL_AGG_MEDIAN || op == BL_AGG_QUANTILE) && dtype_is_small_int(in[n - 1].dtype)) in[n - 1] = op_cast_small_int(in[n - 1], BL_INT64, false);
            std::vector<DevCol> key_outs; DevCol agg_out;
            if (nk == 1 && op <= BL_AGG_LEN && !ctx().deterministic) {
                const DevCol& a = in[0];
                std::vector<int> dts{is_len ? BL_INT64 : in[1].dtype}, nl{(!is_len && in[1].validity != nullptr) ? 1 : 0};
                GroupByState st(a.dtype, {op}, dts, nl, 0, true);
                st.consume_all(a, {is_len ? nullptr : &in[1]});
                DevCol ok; std::vector<DevCol> oa;
                st.finish(true, &a, ok, oa);
                key_outs.push_back(ok); agg_out = oa[0];
            } else {      // several key columns, first / last / var / std / median / quantile, deterministic mode: GroupsIdx
                std::vector<DevCol> keys(in.begin(), in.begin() + nk);
                DevCol packed = nk == 1 ? keys[0] : op_pack_keys(keys);
                DevCol first; std::vector<DevCol> oa;
                op_group_by_exact(packed, {agg_kind}, {is_len ? nullptr : &in[n - 1]}, first, oa, &qp);
                for (auto& k : keys) { std::vector<DevCol> o; op_gather({k}, first, false, o); key_outs.push_back(o[0]); }
                agg_out = oa[0];
            }
            std::vector<DevCol> cols = key_outs; cols.push_back(agg_out);
            std::vector<std::string> names;
            for (size_t j = 0; j < nk; j++) names.push_back(j == 0 ? "key" : "key_" + std::to_string(j));
            names.push_back("agg");
            export_struct(cols, names);
        } else {
            // inputs: left key column(s) followed by the same number of right key columns
            PLB_REQUIRE(n >= 2 && n % 2 == 0, BL_ERR_INVALID, "plugin join_*: expected k left key columns followed by k right key columns");
            const int how = join_how_of(op);
            const bool nulls_equal = kw.get("nulls_equal", 0) != 0;
            if (n == 2) {
                JoinResult jr = op_hash_join(in[0], in[1], how, nulls_equal, BL_ORDER_NONE);
                if (how == BL_JOIN_SEMI || how == BL_JOIN_ANTI) {
                    bl_column h; export_column(jr.left, BL_HOST, &h);
                    fill_array(array, h);
                    fill_schema(schema, name, format_of(BL_UINT32));
                } else export_struct({jr.left, jr.right}, {"left_idx", "right_idx"});
            } else {
                const size_t k = n / 2;
                for (size_t j = 0; j < n; j++) PLB_REQUIRE(chunks[j].size() == 1, BL_ERR_UNSUPPORTED, "plugin join_* on several key columns: rechunk the inputs first");
                std::vector<bl_column> l, r;
                for (size_t j = 0; j < k; j++) { l.push_back(chunks[j][0]); r.push_back(chunks[k + j][0]); }
                bl_column ol, orr;      // host columns owned by the library: the Arrow arrays below take them over
                const bl_status stt = bl_hash_join_keys(l.data(), r.data(), (int32_t)k, how, nulls_equal ? 1 : 0, BL_ORDER_NONE, BL_HOST, &ol, &orr);
                PLB_REQUIRE(stt == BL_OK, stt, bl_last_error());
                if (how == BL_JOIN_SEMI || how == BL_JOIN_ANTI) {
                    bl_column_free(&orr);
                    fill_array(array, ol);
                    fill_schema(schema, name, format_of(BL_UINT32));
                } else {
                    fill_struct_array(array, {ol, orr});
                    fill_schema(schema, name, "+s", {{"left_idx", BL_UINT32}, {"right_idx", BL_UINT32}});
                }
            }
        }
    } catch (...) { free(schema); free(array); throw; }
    make_series(ret, schema, array);
}

static void plugin_entry(PluginOp kind, int op, SeriesExport* inputs, size_t n, const uint8_t* kwargs, size_t kwargs_len, SeriesExport* ret) {
    try { run_plugin(kind, op, inputs, n, parse_kwargs(kwargs, kwargs_len), ret); }
    catch (const std::exception& e) { t_plugin_error = e.what(); cudaGetLastError(); }
    catch (...) { t_plugin_error = "PANIC"; }      // special-cased by the caller (plugin.rs:219-221)
    release_inputs(inputs, n);
}

static void field_entry(PluginOp kind, int op, const ArrowSchema* fields, size_t n, ArrowSchema* out) {
    const std::string name = n > 0 && fields[0].name ? fields[0].name : "";
    const int dt = n > 0 ? dtype_from_format(fields[0].format) : -1;
    const int vdt = n > 1 ? dtype_from_format(fields[1].format) : -1;
    switch (kind) {
        case P_ARITH: fill_schema(out, name, format_of((op == BL_OP_TRUE_DIV && dt >= 0 && dt <= BL_UINT64) ? BL_FLOAT64 : (dt < 0 ? BL_INT64 : dt))); break;
        case P_CMP: fill_schema(out, name, "b"); break;
        case P_SORT: case P_TOP_K: case P_UNIQUE: fill_schema(out, name, format_of(BL_UINT32)); break;
        case P_DISTINCT: fill_schema(out, name, "b"); break;
        case P_OVER: fill_schema(out, name, format_of(over_scan_dtype(op, dt < 0 ? BL_INT64 : dt))); break;
        case P_ROLL: fill_schema(out, name, format_of(rolling_dtype(op, dt < 0 ? BL_INT64 : dt))); break;
        case P_ROLL_BY: fill_schema(out, name, format_of(rolling_dtype(op, dt < 0 ? BL_INT64 : dt))); break;
        case P_RANK: fill_schema(out, name, format_of(rank_dtype(op))); break;
        case P_ROLL_Q: case P_ROLL_Q_BY: fill_schema(out, name, format_of(rolling_quantile_dtype(dt < 0 ? BL_INT64 : dt))); break;
        case P_FILTER: case P_GATHER: fill_schema(out, name, format_of(dt < 0 ? BL_INT64 : dt)); break;
        case P_GROUP: {
            const size_t nk = op == BL_AGG_LEN ? n : (n > 0 ? n - 1 : 0);
            const int v = (op == BL_AGG_LEN || n < 2) ? -1 : dtype_from_format(fields[n - 1].format);
            int adt = v < 0 ? BL_INT64 : v;
            if (v == BL_INT8 || v == BL_INT16 || v == BL_UINT8 || v == BL_UINT16) adt = (op == BL_AGG_SUM) ? BL_INT64 : v;
            if (op == BL_AGG_MEAN || op == BL_AGG_VAR || op == BL_AGG_STD || op == BL_AGG_MEDIAN || op == BL_AGG_QUANTILE) adt = v == BL_FLOAT32 ? BL_FLOAT32 : BL_FLOAT64;
            if (op == BL_AGG_COUNT || op == BL_AGG_LEN) adt = BL_UINT32;
            std::vector<std::pair<std::string, int>> kids;
            for (size_t j = 0; j < nk; j++) { const int kd = dtype_from_format(fields[j].format); kids.push_back({j == 0 ? "key" : "key_" + std::to_string(j), kd < 0 ? BL_INT64 : kd}); }
            kids.push_back({"agg", adt});
            fill_schema(out, name, "+s", kids);
            (void)vdt;
            break;
        }
        default:
            if (op == BL_JOIN_SEMI || op == BL_JOIN_ANTI) fill_schema(out, name, format_of(BL_UINT32));
            else fill_schema(out, name, "+s", {{"left_idx", BL_UINT32}, {"right_idx", BL_UINT32}});
            break;
    }
}

#define PLUGIN(NAME, KIND, OP)                                                                                            \
    void _polars_plugin_bl_##NAME(SeriesExport* inputs, size_t n, const uint8_t* kwargs, size_t kwargs_len, SeriesExport* ret, CallerContext*) { \
        plugin_entry(KIND, OP, inputs, n, kwargs, kwargs_len, ret);                                                       \
    }                                                                                                                     \
    void _polars_plugin_field_bl_##NAME(const ArrowSchema* fields, size_t n, ArrowSchema* out, const uint8_t*, size_t) {  \
        try { field_entry(KIND, OP, fields, n, out); } catch (...) { t_plugin_error = "PANIC"; }                          \
    }

extern "C" {
uint32_t _polars_plugin_get_version(void) { return (0u << 16) + 1u; }     // (major 0, minor 1): polars-ffi/src/lib.rs:12-17
const char* _polars_plugin_get_last_error_message(void) { return t_plugin_error.c_str(); }

PLUGIN(add, P_ARITH, BL_OP_ADD)
PLUGIN(sub, P_ARITH, BL_OP_SUB)
PLUGIN(mul, P_ARITH, BL_OP_MUL)
PLUGIN(floordiv, P_ARITH, BL_OP_FLOOR_DIV)
PLUGIN(mod, P_ARITH, BL_OP_MOD)
PLUGIN(truediv, P_ARITH, BL_OP_TRUE_DIV)
PLUGIN(eq, P_CMP, BL_CMP_EQ)
PLUGIN(ne, P_CMP, BL_CMP_NE)
PLUGIN(lt, P_CMP, BL_CMP_LT)
PLUGIN(le, P_CMP, BL_CMP_LE)
PLUGIN(gt, P_CMP, BL_CMP_GT)
PLUGIN(ge, P_CMP, BL_CMP_GE)
PLUGIN(filter, P_FILTER, 0)
PLUGIN(gather, P_GATHER, 0)
PLUGIN(group_sum, P_GROUP, BL_AGG_SUM)
PLUGIN(group_mean, P_GROUP, BL_AGG_MEAN)
PLUGIN(group_min, P_GROUP, BL_AGG_MIN)
PLUGIN(group_max, P_GROUP, BL_AGG_MAX)
PLUGIN(group_count, P_GROUP, BL_AGG_COUNT)
PLUGIN(group_len, P_GROUP, BL_AGG_LEN)
PLUGIN(group_first, P_GROUP, BL_AGG_FIRST)
PLUGIN(group_last, P_GROUP, BL_AGG_LAST)
PLUGIN(group_var, P_GROUP, BL_AGG_VAR)          /* kwargs: ddof (default 1) */
PLUGIN(group_std, P_GROUP, BL_AGG_STD)
PLUGIN(group_median, P_GROUP, BL_AGG_MEDIAN)
PLUGIN(group_quantile, P_GROUP, BL_AGG_QUANTILE)    /* kwargs: quantile (float, required), method (str, default "nearest") */
PLUGIN(join_inner_idx, P_JOIN, BL_JOIN_INNER)   /* kwargs: nulls_equal; 2k inputs = k key columns per side */
PLUGIN(join_left_idx, P_JOIN, BL_JOIN_LEFT)
PLUGIN(join_full_idx, P_JOIN, BL_JOIN_FULL)
PLUGIN(join_semi_idx, P_JOIN, BL_JOIN_SEMI)
PLUGIN(join_anti_idx, P_JOIN, BL_JOIN_ANTI)
PLUGIN(arg_sort, P_SORT, 0)                     /* kwargs: descending, nulls_last (bool or bitmask); inputs = by columns */
PLUGIN(top_k_idx, P_TOP_K, 0)                   /* kwargs: k, reverse (bool or bitmask); inputs = by columns */
PLUGIN(bottom_k_idx, P_TOP_K, 1)
PLUGIN(arg_unique, P_UNIQUE, 0)                 /* kwargs: keep (default "first"); inputs = key columns */
PLUGIN(is_unique, P_DISTINCT, BL_DISTINCT_UNIQUE)
PLUGIN(is_duplicated, P_DISTINCT, BL_DISTINCT_DUPLICATED)
PLUGIN(is_first_distinct, P_DISTINCT, BL_DISTINCT_FIRST)
PLUGIN(is_last_distinct, P_DISTINCT, BL_DISTINCT_LAST)
PLUGIN(cum_sum, P_OVER, BL_CUM_SUM)             /* kwargs: reverse; inputs = values, then partition keys */
PLUGIN(cum_prod, P_OVER, BL_CUM_PROD)
PLUGIN(cum_min, P_OVER, BL_CUM_MIN)
PLUGIN(cum_max, P_OVER, BL_CUM_MAX)
PLUGIN(cum_count, P_OVER, BL_CUM_COUNT)
PLUGIN(shift, P_OVER, BL_SHIFT)                 /* kwargs: periods (default 1) */
PLUGIN(rolling_sum, P_ROLL, BL_ROLLING_SUM)     /* kwargs: window_size, min_samples, center, ddof; inputs = values, then partition keys */
PLUGIN(rolling_mean, P_ROLL, BL_ROLLING_MEAN)
PLUGIN(rolling_min, P_ROLL, BL_ROLLING_MIN)
PLUGIN(rolling_max, P_ROLL, BL_ROLLING_MAX)
PLUGIN(rolling_var, P_ROLL, BL_ROLLING_VAR)
PLUGIN(rolling_std, P_ROLL, BL_ROLLING_STD)
PLUGIN(rolling_sum_by, P_ROLL_BY, BL_ROLLING_SUM)     /* kwargs: window_size, min_samples, closed (str or code), ddof; inputs = values, by, then partition keys */
PLUGIN(rolling_mean_by, P_ROLL_BY, BL_ROLLING_MEAN)
PLUGIN(rolling_min_by, P_ROLL_BY, BL_ROLLING_MIN)
PLUGIN(rolling_max_by, P_ROLL_BY, BL_ROLLING_MAX)
PLUGIN(rolling_var_by, P_ROLL_BY, BL_ROLLING_VAR)
PLUGIN(rolling_std_by, P_ROLL_BY, BL_ROLLING_STD)
PLUGIN(rolling_quantile, P_ROLL_Q, 0)             /* kwargs: quantile, method, window_size, min_samples, center; inputs = values, then partition keys */
PLUGIN(rolling_median, P_ROLL_Q, 1)               /* quantile 0.5, "linear" */
PLUGIN(rolling_quantile_by, P_ROLL_Q_BY, 0)       /* kwargs: quantile, method, window_size, min_samples, closed; inputs = values, by, then partition keys */
PLUGIN(rolling_median_by, P_ROLL_Q_BY, 1)
PLUGIN(rank_average, P_RANK, BL_RANK_AVERAGE)     /* kwargs: descending, seed (random; None: drawn); inputs = values, then partition keys */
PLUGIN(rank_min, P_RANK, BL_RANK_MIN)
PLUGIN(rank_max, P_RANK, BL_RANK_MAX)
PLUGIN(rank_dense, P_RANK, BL_RANK_DENSE)
PLUGIN(rank_ordinal, P_RANK, BL_RANK_ORDINAL)
PLUGIN(rank_random, P_RANK, BL_RANK_RANDOM)
}
