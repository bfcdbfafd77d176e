// cabi.cu — extern "C" operator entry points of include/polars_b200.h.
// Each entry point: import the bl_column arguments (pinned DMA / zero-copy device views), run the
// device operator, export the outputs into the requested location.  No CPU compute path exists.
#include "common.cuh"
#include "groupby.h"

using namespace plb;

static void require_out(const void* p, const char* what) { PLB_REQUIRE(p != nullptr, BL_ERR_INVALID, std::string("null output: ") + what); }

extern "C" {

bl_status bl_elementwise(int32_t op, const bl_column* lhs, const bl_column* rhs, int32_t out_location, bl_column* out) {
    BL_TRY
    require_out(out, "out");
    PLB_REQUIRE(lhs && rhs, BL_ERR_INVALID, "elementwise: null input");
    DevCol l = import_column(lhs, 1), r = import_column(rhs, 1);
    DevCol o = op_elementwise(op, l, r);
    export_column(o, out_location, out);
    BL_CATCH
}

bl_status bl_compare(int32_t op, const bl_column* lhs, const bl_column* rhs, int32_t missing, int32_t out_location, bl_column* out) {
    BL_TRY
    require_out(out, "out");
    PLB_REQUIRE(lhs && rhs, BL_ERR_INVALID, "compare: null input");
    DevCol l = import_column(lhs, 1), r = import_column(rhs, 1);
    DevCol o = op_compare(op, l, r, missing != 0);
    export_column(o, out_location, out);
    BL_CATCH
}

static void filter_impl(const bl_column* cols, int32_t n_cols, const DevCol& mask, int32_t out_location, bl_column* outs, const std::vector<DevCol>* pre = nullptr) {
    std::vector<DevCol> in, o;
    for (int i = 0; i < n_cols; i++) in.push_back(pre ? (*pre)[i] : import_column(&cols[i], 1));
    op_filter(in, mask, o);
    export_many(o, out_location, outs);
}

bl_status bl_filter(const bl_column* cols, int32_t n_cols, const bl_column* mask, int32_t out_location, bl_column* outs) {
    BL_TRY
    PLB_REQUIRE(cols && mask && outs && n_cols >= 1, BL_ERR_INVALID, "filter: null argument");
    DevCol m = import_column(mask, 1);
    filter_impl(cols, n_cols, m, out_location, outs);
    BL_CATCH
}

bl_status bl_filter_cmp(const bl_column* cols, int32_t n_cols, int32_t pred_col, int32_t cmp_op, const bl_column* scalar, int32_t out_location, bl_column* outs) {
    BL_TRY
    PLB_REQUIRE(cols && scalar && outs && n_cols >= 1, BL_ERR_INVALID, "filter_cmp: null argument");
    PLB_REQUIRE(pred_col >= 0 && pred_col < n_cols, BL_ERR_INVALID, "filter_cmp: pred_col out of range");
    PLB_REQUIRE(scalar->length == 1, BL_ERR_INVALID, "filter_cmp: scalar must be a length-1 column");
    std::vector<DevCol> in;
    for (int i = 0; i < n_cols; i++) in.push_back(import_column(&cols[i], 1));
    DevCol s = import_column(scalar, 1);
    DevCol m = op_cmp_scalar_mask(in[pred_col], cmp_op, s);
    filter_impl(cols, n_cols, m, out_location, outs, &in);
    BL_CATCH
}

bl_status bl_gather(const bl_column* cols, int32_t n_cols, const bl_column* idx, int32_t check_bounds, int32_t out_location, bl_column* outs) {
    BL_TRY
    PLB_REQUIRE(cols && idx && outs && n_cols >= 1, BL_ERR_INVALID, "gather: null argument");
    std::vector<DevCol> in, o;
    for (int i = 0; i < n_cols; i++) in.push_back(import_column(&cols[i], 1));
    DevCol ix = import_column(idx, 1);
    op_gather(in, ix, check_bounds != 0, o, true);      // a caller's index column may hold BL_IDX_NULL without a bitmap
    export_many(o, out_location, outs);
    BL_CATCH
}

bl_status bl_groupby_agg(const bl_column* key_chunks, int32_t n_key_chunks, const bl_agg* aggs, int32_t n_aggs, int32_t maintain_order, int32_t out_location,
                         bl_column* out_key, bl_column* out_aggs) {
    BL_TRY
    PLB_REQUIRE(key_chunks && n_key_chunks >= 1 && out_key, BL_ERR_INVALID, "groupby_agg: null key / output");
    PLB_REQUIRE(n_aggs == 0 || (aggs && out_aggs), BL_ERR_INVALID, "groupby_agg: null aggs / outputs");
    std::vector<int> kinds, dts;
    for (int i = 0; i < n_aggs; i++) {
        kinds.push_back(aggs[i].kind);
        if (aggs[i].kind != BL_AGG_LEN) PLB_REQUIRE(aggs[i].values && aggs[i].n_chunks >= 1, BL_ERR_INVALID, "groupby_agg: aggregation without a value column");
    }
    auto same_col = [](const bl_agg& a, const bl_agg& b) {
        return a.n_chunks == b.n_chunks && (a.values == b.values || (a.n_chunks == 1 && a.values[0].values == b.values[0].values && a.values[0].validity == b.values[0].validity &&
                                                                    a.values[0].offset == b.values[0].offset && a.values[0].length == b.values[0].length && a.values[0].dtype == b.values[0].dtype));
    };
    // Host inputs without nulls: chunked H2D on the copy stream overlapped with K5 on the compute stream.
    bool needs_groups_idx = ctx().deterministic;      // FIRST / LAST / VAR / STD fold per group over GroupsIdx (groupby_exact.cu)
    bool has_n_unique = false;
    for (int i = 0; i < n_aggs; i++) {
        if (aggs[i].kind == BL_AGG_N_UNIQUE) { has_n_unique = true; continue; }
        needs_groups_idx |= (aggs[i].kind & 0xFFFF) >= BL_AGG_FIRST;
    }
    bool pipelined = !needs_groups_idx && !has_n_unique && n_key_chunks == 1 && key_chunks[0].location == BL_HOST && (key_chunks[0].validity == nullptr || key_chunks[0].null_count == 0) &&
                     key_chunks[0].length >= (int64_t)1 << 22 && dtype_size(key_chunks[0].dtype) >= 4 && key_chunks[0].dtype != BL_BOOL;
    for (int i = 0; i < n_aggs && pipelined; i++)
        if (aggs[i].kind != BL_AGG_LEN)
            pipelined = aggs[i].n_chunks == 1 && aggs[i].values[0].location == BL_HOST && (aggs[i].values[0].validity == nullptr || aggs[i].values[0].null_count == 0) &&
                        aggs[i].values[0].length == key_chunks[0].length && dtype_size(aggs[i].values[0].dtype) >= 4 && aggs[i].values[0].dtype != BL_BOOL;
    DevCol key;
    std::vector<DevCol> vals(n_aggs);
    std::vector<const DevCol*> vptr(n_aggs, nullptr);
    std::vector<int> nullable(n_aggs, 0);
    if (pipelined) {
        Context& c = ctx();
        const int64_t n = key_chunks[0].length;
        key = make_col(key_chunks[0].dtype, n, false);
        for (int i = 0; i < n_aggs; i++) {
            if (aggs[i].kind == BL_AGG_LEN) { dts.push_back(BL_INT64); continue; }
            int dup = -1;
            for (int j = 0; j < i; j++) if (aggs[j].kind != BL_AGG_LEN && same_col(aggs[j], aggs[i])) { dup = j; break; }
            if (dup >= 0) vptr[i] = vptr[dup]; else { vals[i] = make_col(aggs[i].values[0].dtype, n, false); vptr[i] = &vals[i]; }
            dts.push_back(vptr[i]->dtype);
        }
        const int64_t chunk_rows = (int64_t)1 << 23;      // 8M rows: 64 MB per 8-byte column
        const size_t n_chunks = (size_t)((n + chunk_rows - 1) / chunk_rows);
        std::vector<cudaEvent_t> ready(n_chunks);
        // the copy stream must not run ahead of the allocation order of the compute stream
        cudaEvent_t alloc_done; PLB_CUDA(cudaEventCreateWithFlags(&alloc_done, cudaEventDisableTiming));
        PLB_CUDA(cudaEventRecord(alloc_done, c.stream));
        PLB_CUDA(cudaStreamWaitEvent(c.copy_stream, alloc_done, 0));
        for (size_t ci = 0; ci < n_chunks; ci++) {
            const int64_t lo = (int64_t)ci * chunk_rows, len = std::min<int64_t>(chunk_rows, n - lo);
            const int kes = dtype_size(key.dtype);
            PLB_CUDA(cudaMemcpyAsync((char*)key.values->p + lo * kes, (const char*)key_chunks[0].values + (key_chunks[0].offset + lo) * kes, (size_t)len * kes, cudaMemcpyHostToDevice, c.copy_stream));
            for (int i = 0; i < n_aggs; i++) {
                if (vptr[i] != &vals[i]) continue;      // LEN or duplicate column
                const int ves = dtype_size(vals[i].dtype);
                PLB_CUDA(cudaMemcpyAsync((char*)vals[i].values->p + lo * ves, (const char*)aggs[i].values[0].values + (aggs[i].values[0].offset + lo) * ves, (size_t)len * ves, cudaMemcpyHostToDevice, c.copy_stream));
            }
            PLB_CUDA(cudaEventCreateWithFlags(&ready[ci], cudaEventDisableTiming));
            PLB_CUDA(cudaEventRecord(ready[ci], c.copy_stream));
        }
        GroupByState st(key.dtype, kinds, dts, nullable, 0, maintain_order != 0 || dtype_is_float(key.dtype));
        try { st.consume_pipelined(key, vptr, chunk_rows, ready); }
        catch (...) { cudaStreamSynchronize(c.copy_stream); for (auto e : ready) cudaEventDestroy(e); cudaEventDestroy(alloc_done); throw; }
        for (auto e : ready) cudaEventDestroy(e);
        cudaEventDestroy(alloc_done);
        DevCol ok; std::vector<DevCol> oa;
        st.finish(maintain_order != 0, &key, ok, oa);
        { std::vector<DevCol> all{ok}; all.insert(all.end(), oa.begin(), oa.end());
          std::vector<bl_column> t(all.size()); export_many(all, out_location, t.data());
          *out_key = t[0]; for (int i = 0; i < n_aggs; i++) out_aggs[i] = t[i + 1]; }
        return BL_OK;
    }
    key = import_column(key_chunks, n_key_chunks);
    // 8/16-bit integers: keys are grouped on their zero-extended bit pattern, value columns aggregate as Int64
    // (series/implementations/mod.rs:145-154); key / min / max outputs are narrowed back below
    const int key_in_dtype = key.dtype;
    if (dtype_is_small_int(key_in_dtype)) key = op_cast_small_int(key, BL_UINT32, true);
    std::vector<int> val_in_dtype(n_aggs, -1);
    // aggregations over the same chunk list share one device copy
    for (int i = 0; i < n_aggs; i++) {
        if (aggs[i].kind == BL_AGG_LEN) { dts.push_back(BL_INT64); continue; }
        int dup = -1;
        for (int j = 0; j < i; j++) if (aggs[j].kind != BL_AGG_LEN && same_col(aggs[j], aggs[i])) { dup = j; break; }
        if (dup >= 0) { vals[i] = vals[dup]; val_in_dtype[i] = val_in_dtype[dup]; }
        else {
            vals[i] = import_column(aggs[i].values, aggs[i].n_chunks);
            val_in_dtype[i] = vals[i].dtype;
            if (dtype_is_small_int(vals[i].dtype)) vals[i] = op_cast_small_int(vals[i], BL_INT64, false);
        }
        vptr[i] = &vals[i];
        dts.push_back(vals[i].dtype);
    }
    // n_unique (agg_n_unique, aggregations/dispatch.rs:285-345: distinct values per group, a null counts as a value): a row is
    // the FIRST occurrence of its (key, value) pair <=> its pair-group id equals its own index; the number of such rows per group
    // is a COUNT over a flag column whose validity bitmap is that predicate.  Composed of K5 pieces: op_pack_keys (nulls and
    // canonical floats folded into the packed value), op_group_first_ids, K2 compare against iota.
    for (int i = 0; i < n_aggs; i++) {
        if (aggs[i].kind != BL_AGG_N_UNIQUE) continue;
        const int64_t n = key.len;
        std::vector<DevCol> kv{key, vals[i]};
        DevCol ids = op_group_first_ids(op_pack_keys(kv));
        DevCol iota = make_col(BL_UINT32, n, false);
        iota_u32(as<uint32_t>(iota.values), n, 0);
        DevCol is_first = op_compare(BL_CMP_EQ, ids, iota, false);
        DevCol flag; flag.dtype = BL_UINT32; flag.len = n; flag.values = ids.values; flag.validity = is_first.values; flag.null_count = -1;
        vals[i] = flag; kinds[i] = BL_AGG_COUNT; dts[i] = BL_UINT32;
    }
    for (int i = 0; i < n_aggs; i++) nullable[i] = vptr[i] != nullptr && vptr[i]->validity != nullptr;
    DevCol ok; std::vector<DevCol> oa;
    if (needs_groups_idx) {      // the reference's own order: GroupsIdx + sequential folds (groupby_exact.cu); groups in first-occurrence order
        DevCol first;
        op_group_by_exact(key, kinds, vptr, first, oa);
        std::vector<DevCol> in{key}, o;
        op_gather(in, first, false, o);
        ok = o[0];
    } else {
        GroupByState st(key.dtype, kinds, dts, nullable, 0, maintain_order != 0 || dtype_is_float(key.dtype));
        st.consume_all(key, vptr);
        st.finish(maintain_order != 0, &key, ok, oa);
    }
    if (dtype_is_small_int(key_in_dtype)) ok = op_cast_small_int(ok, key_in_dtype, true);
    for (int i = 0; i < n_aggs; i++)
        if ((aggs[i].kind == BL_AGG_MIN || aggs[i].kind == BL_AGG_MAX || aggs[i].kind == BL_AGG_FIRST || aggs[i].kind == BL_AGG_LAST) && dtype_is_small_int(val_in_dtype[i]))
            oa[i] = op_cast_small_int(oa[i], val_in_dtype[i], false);
    { std::vector<DevCol> all{ok}; all.insert(all.end(), oa.begin(), oa.end());
      std::vector<bl_column> t(all.size()); export_many(all, out_location, t.data());
      *out_key = t[0]; for (int i = 0; i < n_aggs; i++) out_aggs[i] = t[i + 1]; }
    BL_CATCH
}

bl_status bl_groupby_agg_keys(const bl_column* keys, int32_t n_keys, const bl_agg* aggs, int32_t n_aggs, int32_t maintain_order, int32_t out_location,
                              bl_column* out_keys, bl_column* out_aggs) {
    return bl_groupby_agg_params(keys, n_keys, aggs, nullptr, n_aggs, maintain_order, out_location, out_keys, out_aggs);
}

bl_status bl_groupby_agg_params(const bl_column* keys, int32_t n_keys, const bl_agg* aggs, const bl_agg_param* params, int32_t n_aggs, int32_t maintain_order,
                                int32_t out_location, bl_column* out_keys, bl_column* out_aggs) {
    BL_TRY
    PLB_REQUIRE(keys && n_keys >= 1 && out_keys, BL_ERR_INVALID, "groupby_agg_keys: null keys / output");
    PLB_REQUIRE(n_aggs == 0 || (aggs && out_aggs), BL_ERR_INVALID, "groupby_agg_keys: null aggs / outputs");
    std::vector<DevCol> kcols;
    for (int i = 0; i < n_keys; i++) kcols.push_back(import_column(&keys[i], 1));
    DevCol packed = op_pack_keys(kcols);
    auto same_col = [](const bl_agg& a, const bl_agg& b) {
        return a.n_chunks == b.n_chunks && (a.values == b.values || (a.n_chunks == 1 && a.values[0].values == b.values[0].values && a.values[0].validity == b.values[0].validity &&
                                                                    a.values[0].offset == b.values[0].offset && a.values[0].length == b.values[0].length && a.values[0].dtype == b.values[0].dtype));
    };
    std::vector<int> kinds, dts, nullable(n_aggs, 0), val_in_dtype(n_aggs, -1);
    std::vector<DevCol> vals(n_aggs);
    std::vector<const DevCol*> vptr(n_aggs, nullptr);
    for (int i = 0; i < n_aggs; i++) {
        kinds.push_back(aggs[i].kind);
        if (aggs[i].kind == BL_AGG_LEN) { dts.push_back(BL_INT64); continue; }
        PLB_REQUIRE(aggs[i].values && aggs[i].n_chunks >= 1, BL_ERR_INVALID, "groupby_agg_keys: aggregation without a value column");
        int dup = -1;
        for (int j = 0; j < i; j++) if (aggs[j].kind != BL_AGG_LEN && same_col(aggs[j], aggs[i])) { dup = j; break; }
        if (dup >= 0) { vals[i] = vals[dup]; val_in_dtype[i] = val_in_dtype[dup]; }
        else {
            vals[i] = import_column(aggs[i].values, aggs[i].n_chunks);
            val_in_dtype[i] = vals[i].dtype;
            if (dtype_is_small_int(vals[i].dtype)) vals[i] = op_cast_small_int(vals[i], BL_INT64, false);
        }
        vptr[i] = &vals[i];
        dts.push_back(vals[i].dtype);
        nullable[i] = vals[i].validity != nullptr;
    }
    DevCol ok, first; std::vector<DevCol> oa;
    bool needs_groups_idx = ctx().deterministic;
    for (int i = 0; i < n_aggs; i++) needs_groups_idx |= (aggs[i].kind & 0xFFFF) >= BL_AGG_FIRST;
    if (needs_groups_idx) op_group_by_exact(packed, kinds, vptr, first, oa, params);
    else {
        GroupByState st(BL_UINT64, kinds, dts, nullable, 0, true);
        st.consume_all(packed, vptr);
        st.finish(maintain_order != 0, nullptr, ok, oa, &first);
    }
    for (int i = 0; i < n_aggs; i++)
        if ((aggs[i].kind == BL_AGG_MIN || aggs[i].kind == BL_AGG_MAX || aggs[i].kind == BL_AGG_FIRST || aggs[i].kind == BL_AGG_LAST) && dtype_is_small_int(val_in_dtype[i]))
            oa[i] = op_cast_small_int(oa[i], val_in_dtype[i], false);
    // key output = every key column taken at the group's first row (group_by/mod.rs:258-266)
    std::vector<DevCol> all;
    for (int i = 0; i < n_keys; i++) {
        if (dtype_size(kcols[i].dtype) >= 4) { std::vector<DevCol> in{kcols[i]}, o; op_gather(in, first, false, o); all.push_back(o[0]); }
        else {      // K4 takes 4- and 8-byte elements: gather the widened bit pattern, narrow it back
            std::vector<DevCol> in{op_cast_small_int(kcols[i], BL_UINT32, true)}, o; op_gather(in, first, false, o);
            all.push_back(op_cast_small_int(o[0], kcols[i].dtype, true));
        }
    }
    all.insert(all.end(), oa.begin(), oa.end());
    std::vector<bl_column> t(all.size()); export_many(all, out_location, t.data());
    for (int i = 0; i < n_keys; i++) out_keys[i] = t[i];
    for (int i = 0; i < n_aggs; i++) out_aggs[i] = t[n_keys + i];
    BL_CATCH
}

bl_status bl_group_tuples(const bl_column* key_chunks, int32_t n_key_chunks, int32_t out_location, bl_column* out_first, bl_column* out_offsets, bl_column* out_all) {
    BL_TRY
    PLB_REQUIRE(key_chunks && n_key_chunks >= 1 && out_first && out_offsets && out_all, BL_ERR_INVALID, "group_tuples: null argument");
    DevCol key = import_column(key_chunks, n_key_chunks);
    if (dtype_is_small_int(key.dtype)) key = op_cast_small_int(key, BL_UINT32, true);
    DevCol first, offsets, all;
    op_group_tuples(key, first, offsets, all);
    { std::vector<DevCol> cols{first, offsets, all}; bl_column t[3]; export_many(cols, out_location, t); *out_first = t[0]; *out_offsets = t[1]; *out_all = t[2]; }
    BL_CATCH
}

bl_status bl_hash_join(const bl_column* left_key, int32_t n_left_chunks, const bl_column* right_key, int32_t n_right_chunks, int32_t how, int32_t nulls_equal,
                       int32_t maintain_order, int32_t out_location, bl_column* out_left_idx, bl_column* out_right_idx) {
    BL_TRY
    PLB_REQUIRE(left_key && right_key && out_left_idx && out_right_idx, BL_ERR_INVALID, "hash_join: null argument");
    PLB_REQUIRE(maintain_order >= BL_ORDER_NONE && maintain_order <= BL_ORDER_RIGHT_LEFT, BL_ERR_INVALID, "hash_join: unknown maintain_order");
    DevCol l = import_column(left_key, n_left_chunks), r = import_column(right_key, n_right_chunks);
    PLB_REQUIRE(l.dtype == r.dtype, BL_ERR_DTYPE, "hash_join: key dtypes differ");
    if (dtype_is_small_int(l.dtype)) { l = op_cast_small_int(l, BL_UINT32, true); r = op_cast_small_int(r, BL_UINT32, true); }
    trace_point("cabi:join imported");
    JoinResult jr = op_hash_join(l, r, how, nulls_equal != 0, maintain_order);
    { std::vector<DevCol> both{jr.left, jr.right}; bl_column t[2]; export_many(both, out_location, t); *out_left_idx = t[0]; *out_right_idx = t[1]; }
    trace_point("cabi:join exported");
    BL_CATCH
}

bl_status bl_hash_join_keys(const bl_column* left_keys, const bl_column* right_keys, int32_t n_keys, int32_t how, int32_t nulls_equal, int32_t maintain_order,
                            int32_t out_location, bl_column* out_left_idx, bl_column* out_right_idx) {
    BL_TRY
    PLB_REQUIRE(left_keys && right_keys && out_left_idx && out_right_idx && n_keys >= 1, BL_ERR_INVALID, "hash_join_keys: null argument");
    PLB_REQUIRE(maintain_order >= BL_ORDER_NONE && maintain_order <= BL_ORDER_RIGHT_LEFT, BL_ERR_INVALID, "hash_join_keys: unknown maintain_order");
    const int64_t nl = left_keys[0].length, nr = right_keys[0].length;
    // Both relations are packed TOGETHER (left rows followed by right rows) so that the id compression of wide columns
    // (op_pack_keys) assigns the same id to equal values on either side; nulls become part of the packed value.
    std::vector<DevCol> cats;
    DevPtr lvalid, rvalid;          // AND of the key columns' validities per side (nulls_equal == 0)
    bool l_nullable = false, r_nullable = false;
    for (int i = 0; i < n_keys; i++) {
        PLB_REQUIRE(left_keys[i].dtype == right_keys[i].dtype, BL_ERR_DTYPE, "hash_join_keys: key dtypes differ");      // join/mod.rs:231-241
        PLB_REQUIRE(left_keys[i].length == nl && right_keys[i].length == nr, BL_ERR_INVALID, "hash_join_keys: key columns of one side differ in length");
        const bl_column pair[2] = {left_keys[i], right_keys[i]};
        cats.push_back(import_column(pair, 2));
        if (!nulls_equal) {
            DevCol l = import_column(&left_keys[i], 1), r = import_column(&right_keys[i], 1);
            if (l.validity) { lvalid = l_nullable ? bitmap_and(as<uint32_t>(lvalid), l.vm(), nullptr, nl) : l.validity; l_nullable = true; }
            if (r.validity) { rvalid = r_nullable ? bitmap_and(as<uint32_t>(rvalid), r.vm(), nullptr, nr) : r.validity; r_nullable = true; }
        }
    }
    DevCol packed = n_keys == 1 && !dtype_is_small_int(cats[0].dtype) && cats[0].dtype != BL_BOOL ? cats[0] : op_pack_keys(cats);
    if (n_keys == 1 && packed.validity && nulls_equal) packed = op_pack_keys(cats);      // fold the nulls into the value
    const int es = dtype_size(packed.dtype);
    DevCol lk, rk;
    lk.dtype = rk.dtype = packed.dtype; lk.len = nl; rk.len = nr;
    lk.values = dev_alloc((size_t)std::max<int64_t>(nl, 1) * es + 16); rk.values = dev_alloc((size_t)std::max<int64_t>(nr, 1) * es + 16);
    if (nl) PLB_CUDA(cudaMemcpyAsync(lk.values->p, packed.v(), (size_t)nl * es, cudaMemcpyDeviceToDevice, ctx().stream));
    if (nr) PLB_CUDA(cudaMemcpyAsync(rk.values->p, (const char*)packed.v() + (size_t)nl * es, (size_t)nr * es, cudaMemcpyDeviceToDevice, ctx().stream));
    if (!nulls_equal) { lk.validity = lvalid; rk.validity = rvalid; lk.null_count = l_nullable ? -1 : 0; rk.null_count = r_nullable ? -1 : 0; }
    JoinResult jr = op_hash_join(lk, rk, how, nulls_equal != 0, maintain_order);
    { std::vector<DevCol> both{jr.left, jr.right}; bl_column t[2]; export_many(both, out_location, t); *out_left_idx = t[0]; *out_right_idx = t[1]; }
    BL_CATCH
}

bl_status bl_join(const bl_column* left_key, const bl_column* right_key, const bl_column* left_cols, int32_t n_left_cols, const bl_column* right_cols, int32_t n_right_cols,
                  int32_t how, int32_t nulls_equal, int32_t maintain_order, int32_t out_location, bl_column* out_left_cols, bl_column* out_right_cols) {
    BL_TRY
    PLB_REQUIRE(left_key && right_key, BL_ERR_INVALID, "join: null key");
    PLB_REQUIRE((n_left_cols == 0 || (left_cols && out_left_cols)) && (n_right_cols == 0 || (right_cols && out_right_cols)) && n_left_cols >= 0 && n_right_cols >= 0, BL_ERR_INVALID, "join: null payload / output");
    PLB_REQUIRE(maintain_order >= BL_ORDER_NONE && maintain_order <= BL_ORDER_RIGHT_LEFT, BL_ERR_INVALID, "join: unknown maintain_order");
    DevCol l = import_column(left_key, 1), r = import_column(right_key, 1);
    PLB_REQUIRE(l.dtype == r.dtype, BL_ERR_DTYPE, "join: key dtypes differ");
    if (dtype_is_small_int(l.dtype)) { l = op_cast_small_int(l, BL_UINT32, true); r = op_cast_small_int(r, BL_UINT32, true); }
    std::vector<DevCol> lin, rin, lout, rout;
    for (int i = 0; i < n_left_cols; i++) { lin.push_back(import_column(&left_cols[i], 1)); PLB_REQUIRE(lin.back().len == l.len, BL_ERR_INVALID, "join: left payload length differs from the key"); }
    for (int i = 0; i < n_right_cols; i++) { rin.push_back(import_column(&right_cols[i], 1)); PLB_REQUIRE(rin.back().len == r.len, BL_ERR_INVALID, "join: right payload length differs from the key"); }
    PLB_REQUIRE((how != BL_JOIN_SEMI && how != BL_JOIN_ANTI) || n_right_cols == 0, BL_ERR_INVALID, "join: semi / anti joins produce no right-hand columns");
    // tuples stay on the device: _finish_join (join/general.rs:17-49) = one gather per side
    JoinResult jr = op_hash_join(l, r, how, nulls_equal != 0, maintain_order);
    if (!lin.empty()) op_gather(lin, jr.left, false, lout);
    if (!rin.empty()) op_gather(rin, jr.right, false, rout);
    std::vector<DevCol> all(lout); all.insert(all.end(), rout.begin(), rout.end());
    std::vector<bl_column> t(all.size());
    if (!all.empty()) export_many(all, out_location, t.data());
    for (int i = 0; i < n_left_cols; i++) out_left_cols[i] = t[i];
    for (int i = 0; i < n_right_cols; i++) out_right_cols[i] = t[n_left_cols + i];
    BL_CATCH
}

static void import_sort_keys(const bl_column* by, int32_t n_by, const int32_t* flags, std::vector<DevCol>& keys, std::vector<int>& fl) {
    PLB_REQUIRE(by && n_by >= 1, BL_ERR_INVALID, "sort: no key column");
    for (int i = 0; i < n_by; i++) {
        PLB_REQUIRE(by[i].length == by[0].length, BL_ERR_INVALID, "sort: key columns differ in length");
        keys.push_back(import_column(&by[i], 1));
        fl.push_back(flags ? flags[i] : 0);
    }
}

bl_status bl_arg_sort(const bl_column* by, int32_t n_by, const int32_t* flags, int64_t limit, int32_t out_location, bl_column* out_idx) {
    BL_TRY
    require_out(out_idx, "out_idx");
    std::vector<DevCol> keys; std::vector<int> fl;
    import_sort_keys(by, n_by, flags, keys, fl);
    DevCol perm = op_arg_sort(keys, fl, limit);
    export_column(perm, out_location, out_idx);
    BL_CATCH
}

bl_status bl_sort(const bl_column* by, int32_t n_by, const int32_t* flags, const bl_column* cols, int32_t n_cols, int64_t limit, int32_t out_location, bl_column* out_cols) {
    BL_TRY
    PLB_REQUIRE(n_cols >= 0 && (n_cols == 0 || (cols && out_cols)), BL_ERR_INVALID, "sort: null payload / output");
    std::vector<DevCol> keys, in, outs; std::vector<int> fl;
    import_sort_keys(by, n_by, flags, keys, fl);
    for (int i = 0; i < n_cols; i++) {
        PLB_REQUIRE(cols[i].length == by[0].length, BL_ERR_INVALID, "sort: payload length differs from the keys");
        in.push_back(import_column(&cols[i], 1));
    }
    op_sort(keys, fl, in, limit, outs);
    if (!outs.empty()) export_many(outs, out_location, out_cols);
    BL_CATCH
}

bl_status bl_hash_partition(const bl_column* key, const bl_column* payload, int32_t n_payload, int32_t n_partitions, int32_t out_location, bl_column* out_key,
                            bl_column* out_payload, int64_t* offsets) {
    BL_TRY
    PLB_REQUIRE(key && out_key && offsets && (n_payload == 0 || (payload && out_payload)), BL_ERR_INVALID, "hash_partition: null argument");
    DevCol k = import_column(key, 1);
    std::vector<DevCol> pl, po;
    for (int i = 0; i < n_payload; i++) pl.push_back(import_column(&payload[i], 1));
    DevCol ok;
    op_hash_partition(k, pl, n_partitions, ok, po, offsets);
    bl_column tk; std::vector<bl_column> tp(n_payload);
    export_column(ok, out_location, &tk);
    int done = 0;
    try { for (; done < n_payload; done++) export_column(po[done], out_location, &tp[done]); }
    catch (...) { bl_column_free(&tk); for (int i = 0; i < done; i++) bl_column_free(&tp[i]); throw; }
    *out_key = tk;
    for (int i = 0; i < n_payload; i++) out_payload[i] = tp[i];
    BL_CATCH
}

// ---- streaming group_by state ---------------------------------------------------------------
struct bl_groupby { GroupByState* st; };

bl_status bl_groupby_create(int32_t key_dtype, const int32_t* agg_kinds, const int32_t* value_dtypes, const int32_t* value_nullable, int32_t n_aggs, int64_t expected_groups, int32_t track_first, bl_groupby** out) {
    BL_TRY
    PLB_REQUIRE(out && (n_aggs == 0 || (agg_kinds && value_dtypes)), BL_ERR_INVALID, "groupby_create: null argument");
    std::vector<int> k(agg_kinds, agg_kinds + n_aggs), d(value_dtypes, value_dtypes + n_aggs);
    std::vector<int> nl;
    if (value_nullable) nl.assign(value_nullable, value_nullable + n_aggs);
    auto* g = new bl_groupby{new GroupByState(key_dtype, k, d, nl, expected_groups, track_first != 0)};
    *out = g;
    BL_CATCH
}
bl_status bl_groupby_consume(bl_groupby* g, const bl_column* key, const bl_column* values, int64_t row_base) {
    BL_TRY
    PLB_REQUIRE(g && key, BL_ERR_INVALID, "groupby_consume: null argument");
    DevCol k = import_column(key, 1);
    const size_t na = g->st->plans.size();
    std::vector<DevCol> vals(na); std::vector<const DevCol*> vp(na, nullptr);
    for (size_t i = 0; i < na; i++) {
        if (g->st->plans[i].kind == BL_AGG_LEN) continue;
        PLB_REQUIRE(values != nullptr, BL_ERR_INVALID, "groupby_consume: null values");
        int dup = -1;
        for (size_t j = 0; j < i; j++)
            if (vp[j] && values[j].values == values[i].values && values[j].validity == values[i].validity && values[j].offset == values[i].offset && values[j].dtype == values[i].dtype) { dup = (int)j; break; }
        vals[i] = dup >= 0 ? vals[dup] : import_column(&values[i], 1);
        vp[i] = &vals[i];
    }
    g->st->consume(k, vp, row_base);   // reads the overflow flag back: the batch has completed when this returns
    BL_CATCH
}
bl_status bl_groupby_export_partials(bl_groupby* g, int32_t n_partitions, void** out_rows_dev, int32_t* row_words, int64_t* offsets) {
    BL_TRY
    PLB_REQUIRE(g && out_rows_dev && row_words && offsets, BL_ERR_INVALID, "groupby_export_partials: null argument");
    int rw = 0;
    DevPtr rows = g->st->export_partials(n_partitions, &rw, offsets);
    // hand the raw allocation to the caller (released with bl_dev_free)
    rows->owned = false;
    *out_rows_dev = rows->p; *row_words = rw;
    BL_CATCH
}
bl_status bl_groupby_merge_partials(bl_groupby* g, const void* rows_dev, int64_t n_rows) {
    BL_TRY
    PLB_REQUIRE(g && (rows_dev || n_rows == 0), BL_ERR_INVALID, "groupby_merge_partials: null argument");
    g->st->merge_partials(reinterpret_cast<const uint64_t*>(rows_dev), n_rows);
    BL_CATCH
}
bl_status bl_groupby_merge_partial_regions(bl_groupby* g, const void* const* rows_dev, const int64_t* n_rows, int32_t n_regions) {
    BL_TRY
    PLB_REQUIRE(g && rows_dev && n_rows, BL_ERR_INVALID, "groupby_merge_partial_regions: null argument");
    g->st->merge_partial_regions(reinterpret_cast<const uint64_t* const*>(rows_dev), n_rows, n_regions);
    BL_CATCH
}
bl_status bl_groupby_finish(bl_groupby* g, int32_t maintain_order, int32_t out_location, bl_column* out_key, bl_column* out_aggs) {
    BL_TRY
    PLB_REQUIRE(g && out_key, BL_ERR_INVALID, "groupby_finish: null argument");
    DevCol ok; std::vector<DevCol> oa;
    g->st->finish(maintain_order != 0, nullptr, ok, oa);
    const int n_aggs = (int)oa.size();
    { std::vector<DevCol> all{ok}; all.insert(all.end(), oa.begin(), oa.end());
      std::vector<bl_column> t(all.size()); export_many(all, out_location, t.data());
      *out_key = t[0]; for (int i = 0; i < n_aggs; i++) out_aggs[i] = t[i + 1]; }
    BL_CATCH
}
bl_status bl_groupby_export_partials_p2p(bl_groupby* g, int32_t n_ranks, int32_t my_rank, void* const* windows, int64_t rows_per_src, int32_t* row_words, int64_t* sent_rows) {
    BL_TRY
    PLB_REQUIRE(g && windows && row_words && sent_rows, BL_ERR_INVALID, "groupby_export_partials_p2p: null argument");
    int rw = 0;
    g->st->export_partials_p2p(n_ranks, my_rank, windows, rows_per_src, &rw, sent_rows);
    *row_words = rw;
    BL_CATCH
}

bl_status bl_groupby_export_partials_p2p_async(bl_groupby* g, int32_t n_ranks, int32_t my_rank, void* const* window_halves, int64_t rows_per_src, uint64_t epoch, int32_t* row_words) {
    BL_TRY
    PLB_REQUIRE(g && window_halves && row_words, BL_ERR_INVALID, "groupby_export_partials_p2p_async: null argument");
    static_assert(GB_WINDOW_HEADER_WORDS * 8 == BL_WINDOW_HEADER_BYTES, "window header size");
    int rw = 0;
    g->st->export_partials_p2p_async(n_ranks, my_rank, window_halves, rows_per_src, epoch, &rw);
    *row_words = rw;
    BL_CATCH
}
bl_status bl_groupby_merge_window_async(bl_groupby* g, const void* own_half, int32_t n_ranks, int64_t rows_per_src, uint64_t epoch) {
    BL_TRY
    PLB_REQUIRE(g && own_half, BL_ERR_INVALID, "groupby_merge_window_async: null argument");
    g->st->merge_window_async(own_half, n_ranks, rows_per_src, epoch);
    BL_CATCH
}
void bl_groupby_defer_status(bl_groupby* g, int32_t on) { if (g) g->st->defer_status = on != 0; }
bl_status bl_groupby_status(bl_groupby* g, int32_t* status_out) {
    BL_TRY
    PLB_REQUIRE(g && status_out, BL_ERR_INVALID, "groupby_status: null argument");
    *status_out = g->st->read_status();
    BL_CATCH
}
int64_t bl_groupby_estimated_groups(bl_groupby* g) { return g ? g->st->est_groups : 0; }

bl_status bl_groupby_agg_partitioned(const bl_column* key, const bl_agg* aggs, int32_t n_aggs, int32_t n_ranks, int32_t my_rank, void* const* peer_halves, const void* own_half,
                                     int64_t rows_per_src, uint64_t epoch, int64_t expected_groups, int32_t out_location, bl_column* out_key, bl_column* out_aggs) {
    BL_TRY
    PLB_REQUIRE(key && out_key && peer_halves && own_half && (n_aggs == 0 || (aggs && out_aggs)), BL_ERR_INVALID, "groupby_agg_partitioned: null argument");
    DevCol k = import_column(key, 1);
    std::vector<int> kinds, dts, nullable(n_aggs, 0);
    std::vector<DevCol> vals(n_aggs);
    std::vector<const DevCol*> vptr(n_aggs, nullptr);
    for (int i = 0; i < n_aggs; i++) {
        kinds.push_back(aggs[i].kind);
        if (aggs[i].kind == BL_AGG_LEN) { dts.push_back(BL_INT64); continue; }
        PLB_REQUIRE(aggs[i].values && aggs[i].n_chunks >= 1, BL_ERR_INVALID, "groupby_agg_partitioned: aggregation without a value column");
        int dup = -1;
        for (int j = 0; j < i; j++) if (aggs[j].kind != BL_AGG_LEN && aggs[j].values == aggs[i].values) { dup = j; break; }
        if (dup >= 0) vals[i] = vals[dup]; else vals[i] = import_column(aggs[i].values, aggs[i].n_chunks);
        vptr[i] = &vals[i];
        dts.push_back(vals[i].dtype);
        nullable[i] = vals[i].validity != nullptr;
    }
    // local pre-aggregation (overflow check deferred to the end of the step: no host round trip before the exchange)
    GroupByState local(k.dtype, kinds, dts, nullable, expected_groups, false);
    local.defer_status = true;
    local.consume(k, vptr, 0);
    int rw = 0;
    local.export_partials_p2p_async(n_ranks, my_rank, peer_halves, rows_per_src, epoch, &rw);
    // the owner's table: the groups of one rank's worth of rows when the ranks share a key domain, up to the local group count when they do not
    const int64_t est = std::max<int64_t>(std::max<int64_t>(local.est_groups, expected_groups), 1024);
    GroupByState owner(k.dtype, kinds, dts, nullable, est + est / 4 + 1024, false);
    owner.merge_window_async(own_half, n_ranks, rows_per_src, epoch);
    DevCol ok; std::vector<DevCol> oa;
    owner.finish(false, nullptr, ok, oa);
    PLB_REQUIRE(local.read_status() == 0, BL_ERR_OOM, "groupby_agg_partitioned: the local pre-aggregation table overflowed — pass expected_groups");
    { std::vector<DevCol> all{ok}; all.insert(all.end(), oa.begin(), oa.end());
      std::vector<bl_column> t(all.size()); export_many(all, out_location, t.data());
      *out_key = t[0]; for (int i = 0; i < n_aggs; i++) out_aggs[i] = t[i + 1]; }
    BL_CATCH
}

// ---- peer windows (CUDA IPC) -------------------------------------------------------------------
struct bl_window { void* p; size_t bytes; };
bl_status bl_window_create(size_t bytes, bl_window** out, void* ipc_handle_out) {
    BL_TRY
    PLB_REQUIRE(out && ipc_handle_out && bytes > 0, BL_ERR_INVALID, "window_create: null argument");
    static_assert(sizeof(cudaIpcMemHandle_t) == BL_IPC_HANDLE_BYTES, "IPC handle size");
    void* p = nullptr;
    PLB_CUDA(cudaMalloc(&p, bytes));                       // IPC needs a plain cudaMalloc allocation
    cudaIpcMemHandle_t h;
    cudaError_t e = cudaIpcGetMemHandle(&h, p);
    if (e != cudaSuccess) { cudaFree(p); PLB_CUDA(e); }
    e = cudaMemset(p, 0, bytes);                           // epoch flags of the async exchange start at 0
    if (e != cudaSuccess) { cudaFree(p); PLB_CUDA(e); }
    memcpy(ipc_handle_out, &h, sizeof h);
    *out = new bl_window{p, bytes};
    BL_CATCH
}
void* bl_window_ptr(bl_window* w) { return w ? w->p : nullptr; }
void bl_window_destroy(bl_window* w) { if (w) { cudaFree(w->p); delete w; } }
bl_status bl_window_open(const void* ipc_handle, void** peer_ptr_out) {
    BL_TRY
    PLB_REQUIRE(ipc_handle && peer_ptr_out, BL_ERR_INVALID, "window_open: null argument");
    cudaIpcMemHandle_t h; memcpy(&h, ipc_handle, sizeof h);
    PLB_CUDA(cudaIpcOpenMemHandle(peer_ptr_out, h, cudaIpcMemLazyEnablePeerAccess));
    BL_CATCH
}
void bl_window_close(void* peer_ptr) { if (peer_ptr) cudaIpcCloseMemHandle(peer_ptr); }

void bl_groupby_reset(bl_groupby* g) { try { if (g) { std::lock_guard<std::recursive_mutex> lk(ctx().mu); g->st->reset(); } } catch (...) {} }
void bl_groupby_destroy(bl_groupby* g) { try { if (g) { std::lock_guard<std::recursive_mutex> lk(ctx().mu); delete g->st; delete g; } } catch (...) {} }

}  // extern "C"
