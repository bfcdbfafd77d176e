// groupby_exact.cu — the reference's aggregation ORDER, literally (deterministic / bit-stable mode).
//
// The fused K5 plans add f64 values with order-free atomics, so a float sum can differ in its last bits from run to run
// and from the reference (which differs between its own engines too; DESIGN.md §2).  SURVEY.md §7(b) asks for a
// deterministic test mode; this is it: build the reference's GroupsIdx {first, all} (bl_group_tuples: groups in
// first-occurrence order, row lists ascending — group_by_threaded_slice + finish_group_order, hashing.rs:26-167) and
// fold every group sequentially in row order with exactly the reference's reducers:
//   sum   ints: wrapping add in the column's width (polars-compute/src/sum.rs:13-49); floats: sequential KahanSum
//         (polars-utils/src/kahan_sum.rs:36-47), a one-row group returns the value itself
//         (aggregations/mod.rs:854-879)
//   mean  Kahan f64 sum / valid count; one-row group = the value; all-null -> null (:939-977, :1227-1267)
//   min / max  NaN-ignoring reduce (polars-utils/src/min_max.rs:41-48, :96-108); all-null -> null
//   count / len  (aggregations/dispatch.rs:25-55, position.rs:555-569)
// One thread folds one group (the point is the ORDER, not speed: enable with bl_set_deterministic(1) or
// BL_DETERMINISTIC=1).  Results are bit-identical to the CPU oracle's restatement for every dtype, floats included.
#include <cmath>

#include "common.cuh"
#include "dev_utils.cuh"

namespace plb {

struct SegArgs {
    const void* values; const uint32_t* validity; const uint32_t* offsets; const uint32_t* all; int64_t G;
    void* out; uint32_t* out_valid; int kind, ddof;
};

struct KahanD { double sum, err; };
__device__ __forceinline__ void kahan_add(KahanD& k, double rhs) {      // kahan_sum.rs:36-47
    const double y = rhs - k.err; const double ns = k.sum + y; const double ne = (ns - k.sum) - y;
    k.sum = ns; if (isfinite(ne)) k.err = ne;
}
struct KahanF { float sum, err; };
__device__ __forceinline__ void kahan_add(KahanF& k, float rhs) {
    const float y = rhs - k.err; const float ns = k.sum + y; const float ne = (ns - k.sum) - y;
    k.sum = ns; if (isfinite(ne)) k.err = ne;
}
template <typename T> struct is_fp { static constexpr bool v = false; };
template <> struct is_fp<double> { static constexpr bool v = true; };
template <> struct is_fp<float> { static constexpr bool v = true; };
template <typename T> __device__ __forceinline__ T red_min(T a, T b) { return a < b ? a : b; }
template <typename T> __device__ __forceinline__ T red_max(T a, T b) { return a < b ? b : a; }
template <> __device__ __forceinline__ double red_min<double>(double a, double b) { return fmin(a, b); }      // f64::min == IEEE minNum
template <> __device__ __forceinline__ double red_max<double>(double a, double b) { return fmax(a, b); }
template <> __device__ __forceinline__ float red_min<float>(float a, float b) { return fminf(a, b); }
template <> __device__ __forceinline__ float red_max<float>(float a, float b) { return fmaxf(a, b); }

template <typename T>
__global__ void __launch_bounds__(128) k_seg_agg(const __grid_constant__ SegArgs a) {
    const T* v = reinterpret_cast<const T*>(a.values);
    const int64_t rounded = (a.G + 31) / 32 * 32;
    for (int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; g < rounded; g += (int64_t)gridDim.x * blockDim.x) {
        bool ok = false;
        if (g < a.G) {
            const uint32_t lo = a.offsets[g], hi = a.offsets[g + 1];
            ok = true;
            switch (a.kind) {
                case BL_AGG_LEN: reinterpret_cast<uint32_t*>(a.out)[g] = hi - lo; break;
                case BL_AGG_COUNT: {
                    uint32_t c = 0;
                    for (uint32_t j = lo; j < hi; j++) c += (a.validity == nullptr || bit_get(a.validity, a.all[j])) ? 1u : 0u;
                    reinterpret_cast<uint32_t*>(a.out)[g] = c; break;
                }
                case BL_AGG_SUM: {
                    T* out = reinterpret_cast<T*>(a.out);
                    if constexpr (is_fp<T>::v) {
                        if (hi == lo) { out[g] = (T)0; break; }
                        if (hi - lo == 1) { const uint32_t r = a.all[lo]; out[g] = (a.validity == nullptr || bit_get(a.validity, r)) ? v[r] : (T)0; break; }
                        if constexpr (sizeof(T) == 8) { KahanD k{0.0, 0.0}; for (uint32_t j = lo; j < hi; j++) { const uint32_t r = a.all[j]; if (a.validity == nullptr || bit_get(a.validity, r)) kahan_add(k, v[r]); } out[g] = k.sum; }
                        else { KahanF k{0.0f, 0.0f}; for (uint32_t j = lo; j < hi; j++) { const uint32_t r = a.all[j]; if (a.validity == nullptr || bit_get(a.validity, r)) kahan_add(k, v[r]); } out[g] = k.sum; }
                    } else {
                        typename make_unsigned_t<T>::type s = 0;
                        for (uint32_t j = lo; j < hi; j++) { const uint32_t r = a.all[j]; if (a.validity == nullptr || bit_get(a.validity, r)) s += (typename make_unsigned_t<T>::type)v[r]; }
                        out[g] = (T)s;
                    }
                    break;
                }
                case BL_AGG_MEAN: {
                    double m = 0.0;
                    if (hi == lo) ok = false;
                    else if (hi - lo == 1) { const uint32_t r = a.all[lo]; ok = a.validity == nullptr || bit_get(a.validity, r); m = ok ? (double)v[r] : 0.0; }
                    else {
                        KahanD k{0.0, 0.0}; uint32_t nulls = 0;
                        for (uint32_t j = lo; j < hi; j++) { const uint32_t r = a.all[j]; if (a.validity == nullptr || bit_get(a.validity, r)) kahan_add(k, (double)v[r]); else nulls++; }
                        if (nulls == hi - lo) ok = false; else m = k.sum / ((double)(hi - lo) - (double)nulls);
                    }
                    if constexpr (sizeof(T) == 4 && is_fp<T>::v) reinterpret_cast<float*>(a.out)[g] = (float)m; else reinterpret_cast<double*>(a.out)[g] = m;
                    break;
                }
                case BL_AGG_FIRST: case BL_AGG_LAST: {
                    if (hi == lo) { ok = false; reinterpret_cast<T*>(a.out)[g] = (T)0; break; }
                    const uint32_t r = a.all[a.kind == BL_AGG_FIRST ? lo : hi - 1];
                    ok = a.validity == nullptr || bit_get(a.validity, r);
                    reinterpret_cast<T*>(a.out)[g] = ok ? v[r] : (T)0;
                    break;
                }
                case BL_AGG_VAR: case BL_AGG_STD: {      // Welford, row order (take_agg/var.rs:11-41)
                    double m2 = 0.0, mean = 0.0; uint32_t count = 0;
                    for (uint32_t j = lo; j < hi; j++) {
                        const uint32_t r = a.all[j];
                        if (a.validity != nullptr && !bit_get(a.validity, r)) continue;
                        const double value = (double)v[r];
                        const uint32_t new_count = count + 1;
                        const double delta_1 = value - mean;
                        const double new_mean = delta_1 / (double)new_count + mean;
                        const double delta_2 = value - new_mean;
                        m2 = m2 + delta_1 * delta_2; count = new_count; mean = new_mean;
                    }
                    ok = count > (uint32_t)a.ddof;
                    double res = ok ? m2 / ((double)count - (double)a.ddof) : 0.0;
                    if (a.kind == BL_AGG_STD) res = sqrt(res);
                    if constexpr (sizeof(T) == 4 && is_fp<T>::v) reinterpret_cast<float*>(a.out)[g] = (float)res; else reinterpret_cast<double*>(a.out)[g] = res;
                    break;
                }
                default: {      // MIN / MAX
                    bool have = false; T acc = (T)0;
                    for (uint32_t j = lo; j < hi; j++) {
                        const uint32_t r = a.all[j];
                        if (a.validity != nullptr && !bit_get(a.validity, r)) continue;
                        const T x = v[r];
                        if (!have) { acc = x; have = true; } else acc = a.kind == BL_AGG_MIN ? red_min<T>(acc, x) : red_max<T>(acc, x);
                    }
                    reinterpret_cast<T*>(a.out)[g] = have ? acc : (T)0; ok = have;
                    break;
                }
            }
        }
        if (a.out_valid) { const unsigned b = __ballot_sync(0xffffffffu, ok); if (lane_id() == 0) a.out_valid[g >> 5] = b; }
    }
}

static int exact_out_dtype(int kind, int in_dtype) {
    switch (kind) {
        case BL_AGG_SUM: return in_dtype;                                   // 8/16-bit columns arrive widened to Int64 (cabi.cu)
        case BL_AGG_MEAN: return in_dtype == BL_FLOAT32 ? BL_FLOAT32 : BL_FLOAT64;
        case BL_AGG_MIN: case BL_AGG_MAX: case BL_AGG_FIRST: case BL_AGG_LAST: return in_dtype;
        case BL_AGG_VAR: case BL_AGG_STD: return in_dtype == BL_FLOAT32 ? BL_FLOAT32 : BL_FLOAT64;
        default: return BL_UINT32;
    }
}

// key: the (single, possibly packed) key column; values[i] == nullptr for LEN.  Groups come in first-occurrence order.
// MEDIAN / QUANTILE go to op_group_quantiles (quantile.cu), one call per distinct value column.
void op_group_by_exact(const DevCol& key, const std::vector<int>& kinds, const std::vector<const DevCol*>& values, DevCol& out_first, std::vector<DevCol>& outs,
                       const bl_agg_param* params) {
    std::vector<double> qs(kinds.size(), 0.5);
    std::vector<int> methods(kinds.size(), BL_QUANTILE_LINEAR);      // MEDIAN = quantile(0.5, Linear) (aggregations/mod.rs:385-408)
    for (size_t i = 0; i < kinds.size(); i++) {      // argument errors before any device work
        const int kind = kinds[i] & 0xFFFF;
        PLB_REQUIRE(kind >= BL_AGG_SUM && kind <= BL_AGG_QUANTILE && kind != BL_AGG_N_UNIQUE, BL_ERR_INVALID, "group_by: unknown aggregation kind");
        if (kind != BL_AGG_QUANTILE) continue;
        PLB_REQUIRE(params != nullptr, BL_ERR_INVALID, "group_by: BL_AGG_QUANTILE needs its parameters (bl_groupby_agg_params)");
        PLB_REQUIRE(params[i].method >= BL_QUANTILE_NEAREST && params[i].method <= BL_QUANTILE_EQUIPROBABLE, BL_ERR_INVALID,
                    "group_by: unknown quantile method " + std::to_string(params[i].method));
        // the reference answers an all-null column of the input dtype (aggregations/mod.rs:309-312): the caller's CPU path
        PLB_REQUIRE(params[i].quantile >= 0.0 && params[i].quantile <= 1.0, BL_ERR_UNSUPPORTED, "group_by: quantile " + std::to_string(params[i].quantile) + " is outside [0, 1]");
        qs[i] = params[i].quantile; methods[i] = params[i].method;
    }
    DevCol offsets, all;
    op_group_tuples(key, out_first, offsets, all);
    const int64_t G = out_first.len;
    outs.assign(kinds.size(), DevCol());
    std::vector<bool> done(kinds.size(), false);
    for (size_t i = 0; i < kinds.size(); i++) {
        const int kind = kinds[i] & 0xFFFF, ddof = (kinds[i] >> 16) & 0xFF;
        const DevCol* v = values[i];
        PLB_REQUIRE(kind == BL_AGG_LEN || v != nullptr, BL_ERR_INVALID, "group_by: aggregation without a value column");
        const int in_dt = v ? v->dtype : BL_INT64;
        PLB_REQUIRE(kind == BL_AGG_LEN || in_dt == BL_INT64 || in_dt == BL_UINT64 || in_dt == BL_INT32 || in_dt == BL_UINT32 || in_dt == BL_FLOAT64 || in_dt == BL_FLOAT32, BL_ERR_UNSUPPORTED,
                    std::string("group_by: value dtype ") + dtype_name(in_dt) + " is outside the hot path");
        if (done[i]) continue;
        if (kind == BL_AGG_MEDIAN || kind == BL_AGG_QUANTILE) {      // every median / quantile of this value column: one sort
            std::vector<size_t> at;
            std::vector<double> q; std::vector<int> m;
            for (size_t j = i; j < kinds.size(); j++) {
                const int kj = kinds[j] & 0xFFFF;
                if ((kj == BL_AGG_MEDIAN || kj == BL_AGG_QUANTILE) && values[j]->values == v->values && values[j]->validity == v->validity && values[j]->dtype == v->dtype) {
                    at.push_back(j); q.push_back(qs[j]); m.push_back(methods[j]); done[j] = true;
                }
            }
            std::vector<DevCol> qo;
            op_group_quantiles(offsets, all, *v, q, m, qo);
            for (size_t k = 0; k < at.size(); k++) outs[at[k]] = qo[k];
            continue;
        }
        const bool nullable = kind == BL_AGG_MEAN || kind == BL_AGG_MIN || kind == BL_AGG_MAX || kind >= BL_AGG_FIRST;
        DevCol o = make_col(exact_out_dtype(kind, in_dt), G, nullable);
        if (G > 0) {
            SegArgs a; memset(&a, 0, sizeof a);
            a.values = v ? v->v() : nullptr; a.validity = v ? v->vm() : nullptr; a.offsets = as<uint32_t>(offsets.values); a.all = as<uint32_t>(all.values);
            a.G = G; a.out = o.values->p; a.out_valid = as<uint32_t>(o.validity); a.kind = kind; a.ddof = ddof;
            const int grid = grid_for(G, 128, 16);
            switch (in_dt) {
                case BL_INT64: PLB_LAUNCH("k5x_fold_groups", k_seg_agg<int64_t>, grid, 128, 0, a); break;
                case BL_UINT64: PLB_LAUNCH("k5x_fold_groups", k_seg_agg<uint64_t>, grid, 128, 0, a); break;
                case BL_INT32: PLB_LAUNCH("k5x_fold_groups", k_seg_agg<int32_t>, grid, 128, 0, a); break;
                case BL_UINT32: PLB_LAUNCH("k5x_fold_groups", k_seg_agg<uint32_t>, grid, 128, 0, a); break;
                case BL_FLOAT64: PLB_LAUNCH("k5x_fold_groups", k_seg_agg<double>, grid, 128, 0, a); break;
                default: PLB_LAUNCH("k5x_fold_groups", k_seg_agg<float>, grid, 128, 0, a); break;
            }
        }
        outs[i] = o;
    }
}

}  // namespace plb
