// rolling.cuh — what the fixed-window (rolling.cu) and the time-based (rolling_by.cu) rolling aggregations share: the
// associative window states, their finishers, the segmented block scan k_roll_scan, the output writer and the
// deterministic replays of the reference's window machines.
#pragma once
#include <algorithm>
#include <cmath>

#include "common.cuh"
#include "dev_utils.cuh"

namespace plb {

// ---------------------------------------------------------------------------------------------------- states
// S: the state of a run of positions; empty(): no non-null value; combine(a, b): a earlier in position order
template <typename Acc> struct SumIntSt {      // integer SUM: wraps in Acc
    struct S { Acc s; uint32_t c; };
    __device__ static S empty() { return S{Acc(0), 0u}; }
    __device__ static S combine(S a, S b) { return S{Acc(a.s + b.s), a.c + b.c}; }
    template <typename In> __device__ static S lift(In x) {
        if constexpr (std::is_same<In, BoolBit>::value) return S{Acc(x.b ? 1 : 0), 1u};
        else return S{(Acc)x, 1u};
    }
};
struct SumFltSt {      // float SUM / MEAN: finite values summed in f64, non-finite ones counted (rolling/sum.rs:68-108)
    struct S { double s; uint32_t c, pinf, ninf, nan; };
    __device__ static S empty() { return S{0.0, 0u, 0u, 0u, 0u}; }
    __device__ static S combine(S a, S b) { return S{a.s + b.s, a.c + b.c, a.pinf + b.pinf, a.ninf + b.ninf, a.nan + b.nan}; }
    template <typename In> __device__ static S lift(In v) {
        const double x = (double)v;
        if (isfinite(x)) return S{x, 1u, 0u, 0u, 0u};
        return S{0.0, 1u, x > 0 ? 1u : 0u, x < 0 ? 1u : 0u, x != x ? 1u : 0u};
    }
};
// MIN / MAX with NaN propagating and the earliest of equal values winning (MinPropagateNan / MaxPropagateNan is_better)
template <typename T, bool MAX> struct MinMaxSt {
    struct S { T v; uint32_t c; };
    __device__ static S empty() { return S{T(0), 0u}; }
    __device__ static bool better(T b, T a) {      // b strictly better than a
        if constexpr (std::is_floating_point<T>::value) {
            if (a != a) return false;
            if (b != b) return true;
        }
        return MAX ? a < b : b < a;
    }
    __device__ static S combine(S a, S b) {
        if (a.c == 0) return b;
        if (b.c == 0) return a;
        return S{better(b.v, a.v) ? b.v : a.v, a.c + b.c};
    }
    template <typename In> __device__ static S lift(In x) { return S{x, 1u}; }
};
// VarState (polars-compute/src/moment.rs:90-129) plus the count of non-finite values (held as 0.0, rolling/moment.rs push)
struct VarSt {
    struct S { double w, mean, dp; uint32_t nf; };
    __device__ static S empty() { return S{0.0, 0.0, 0.0, 0u}; }
    __device__ static void insert_one(S& s, double x) {
        const double nw = s.w + 1.0, dm = x - s.mean, nm = s.mean + dm / nw;
        s.dp += (x - nm) * dm;
        s.w = nw; s.mean = nm;
        if (s.w == 0.0) { s.mean = 0.0; s.dp = 0.0; }
    }
    __device__ static void combine_into(S& s, const S& o) {
        if (o.w == 0.0) return;
        const double nw = s.w + o.w, frac = o.w / nw, dm = o.mean - s.mean, nm = s.mean + dm * frac;
        s.dp += o.dp + o.w * (o.mean - nm) * dm;
        s.w = nw; s.mean = nm;
        if (s.w == 0.0) { s.mean = 0.0; s.dp = 0.0; }
    }
    __device__ static S combine(S a, S b) { combine_into(a, b); a.nf += b.nf; return a; }
    template <typename In> __device__ static S lift(In v) {
        const double x = (double)v;
        return isfinite(x) ? S{1.0, x, 0.0, 0u} : S{1.0, 0.0, 0.0, 1u};
    }
    // finalize(ddof) with the non-finite rule: false = null
    __device__ static bool var(const S& s, int ddof, double& out) {
        if (s.w <= (double)ddof) return false;
        double v = s.dp / (s.w - (double)ddof);
        if (v < 0.0) v = 0.0;
        out = s.nf ? __longlong_as_double(0x7ff8000000000000ll) : v;
        return true;
    }
};

// The lifted state of the value at row r.  In = StateIn: the array holds states already (rolling_by scans its block totals).
struct StateIn {};
template <class St, typename In> __device__ __forceinline__ typename St::S lift_at(const void* v, int64_t r) {
    if constexpr (std::is_same<In, StateIn>::value) return reinterpret_cast<const typename St::S*>(v)[r];
    else return St::lift(load_in<In>(v, r));
}

// ---------------------------------------------------------------------------------------------------- finishers
struct RollArgs {
    const void* values; const uint32_t* validity;
    const uint32_t* perm; const uint32_t* seg; const uint32_t* offsets; int64_t G;      // partition order (NULL: the rows, one segment)
    int64_t n, L, R; uint32_t B;      // window [i - L, i + R) clipped to the segment; block size
    int64_t min_samples; int ddof;
    void* pre; void* suf; void* out; uint32_t* out_valid;
    const uint32_t* ws; const uint32_t* we;      // time-based windows: [ws[i], we[i]) per position (NULL: the fixed window above)
    int64_t W;      // time-based windows: the largest we[i] - ws[i]
};
constexpr uint32_t BY_NULL = 0xFFFFFFFFu;      // ws[i] of a position whose `by` is null: no window, a null output

// The fixed window [s, e) of position i: [i - L, i + R) clipped to its segment, found by binary search in offsets (none:
// [0, n)).  Returns the segment's first position.
__device__ __forceinline__ int64_t fixed_window(const RollArgs& a, int64_t i, int64_t& s, int64_t& e) {
    int64_t lo = 0, hi = a.n;
    if (a.offsets) {
        int64_t gl = 0, gh = a.G;      // offsets[gl] <= i < offsets[gh]
        while (gh - gl > 1) {
            const int64_t m = (gl + gh) >> 1;
            if ((int64_t)__ldg(a.offsets + m) <= i) gl = m; else gh = m;
        }
        lo = __ldg(a.offsets + gl); hi = __ldg(a.offsets + gl + 1);
    }
    s = max(i - a.L, lo); e = min(i + a.R, hi);
    return lo;
}

// The positions of a time-based rolling call (rolling_by.cu): the rows when no partition is given and `by` is non-null and
// ascending, else bl_over's partition order with `by` as the key, nulls last (need_inv: with its inverse).  Checks the `by`
// column and the row limits; messages start with `who`.
struct ByOrder { bool need_order = false; OverOrder o; };
ByOrder rolling_by_order(const char* who, const std::vector<DevCol>& partition_by, const DevCol& by, int64_t n, bool need_inv);
// Writes each position's window [ws, we) of width P and `closed` (ws = BY_NULL where `by` is null); returns the widest window
int64_t rolling_by_bounds(const DevCol& by, const ByOrder& bo, int64_t n, int64_t P, int closed, uint32_t* ws, uint32_t* we);
template <typename Out> __device__ __forceinline__ Out class_value(const SumFltSt::S& s) {      // get_sum (rolling/sum.rs:98-108)
    const uint32_t nf = s.pinf + s.ninf + s.nan;
    if (nf == 0) return (Out)s.s;
    if (nf == s.pinf) return (Out)INFINITY;
    if (nf == s.ninf) return (Out)-INFINITY;
    return (Out)NAN;
}
template <typename Out> struct FinSumInt {
    using out_t = Out;
    template <typename S> __device__ static bool fin(const S& s, const RollArgs& a, Out& o) { o = (Out)s.s; return s.c >= a.min_samples; }
};
template <typename Out> struct FinSumFlt {
    using out_t = Out;
    __device__ static bool fin(const SumFltSt::S& s, const RollArgs& a, Out& o) { o = class_value<Out>(s); return s.c >= a.min_samples; }
};
template <typename Out> struct FinMean {
    using out_t = Out;
    __device__ static bool fin(const SumFltSt::S& s, const RollArgs& a, Out& o) { o = class_value<Out>(s) / (Out)s.c; return s.c > 0 && s.c >= a.min_samples; }
};
struct FinMinMax {
    template <typename S> __device__ static bool fin(const S& s, const RollArgs& a, decltype(S::v)& o) { o = s.v; return s.c > 0 && s.c >= a.min_samples; }
};
template <typename T> struct FinMinMaxT : FinMinMax { using out_t = T; };
template <typename Out, bool STD> struct FinVar {
    using out_t = Out;
    __device__ static bool fin(const VarSt::S& s, const RollArgs& a, Out& o) {
        double v;
        if (!VarSt::var(s, a.ddof, v) || (int64_t)s.w < a.min_samples) { o = Out(0); return false; }
        o = (Out)v;
        if (STD) o = sqrt(o);
        return true;
    }
};

// ---------------------------------------------------------------------------------------------------- k_roll_scan
// One CTA owns the positions [lo, hi) = whole blocks (span = a multiple of B), so no carry crosses CTAs.  It walks them in
// tiles of RS_TILE logical elements (REV: from hi - 1 down), each thread 8 consecutive ones: a sequential segmented scan per
// thread, a Hillis-Steele segmented scan of the 256 thread totals in shared memory, then the carry of the previous tile.
// Forward: element p is a head at a block start or a segment head, and the output is prefix[p].  REV: a head at a block end or
// a segment end, the output suffix[p], and the scan runs towards earlier positions (the accumulated run is LATER than p).
constexpr int RS_THREADS = 256, RS_ITEMS = 8, RS_TILE = RS_THREADS * RS_ITEMS;

template <class St, bool REV> __device__ __forceinline__ typename St::S cmb(const typename St::S& prev, const typename St::S& cur) {
    return REV ? St::combine(cur, prev) : St::combine(prev, cur);      // prev: earlier in scan order
}

template <class St, typename In, bool REV>
__global__ void __launch_bounds__(RS_THREADS) k_roll_scan(const __grid_constant__ RollArgs a, int64_t span) {
    using S = typename St::S;
    __shared__ S s_v[RS_THREADS];
    __shared__ int s_f[RS_THREADS];
    const int64_t lo = (int64_t)blockIdx.x * span, hi = min(a.n, lo + span), len = hi - lo;
    S* outp = reinterpret_cast<S*>(REV ? a.suf : a.pre);
    S carry = St::empty();
    for (int64_t base = 0; base < len; base += RS_TILE) {
        S v[RS_ITEMS];
        bool f[RS_ITEMS];
        const int64_t j0 = base + (int64_t)threadIdx.x * RS_ITEMS;
        // r: distance to the block's first element in scan order, mod B (REV: (p + 1 - lo) mod B, p = hi - 1 - j)
        uint32_t r = (uint32_t)((uint64_t)(REV ? len - j0 : j0) % a.B);
        bool any = false;
#pragma unroll
        for (int k = 0; k < RS_ITEMS; k++) {
            const int64_t j = j0 + k;
            f[k] = false;
            v[k] = St::empty();
            if (j < len) {
                const int64_t p = REV ? hi - 1 - j : lo + j;
                f[k] = r == 0 || j == 0;
                if (a.seg && !f[k]) f[k] = __ldg(a.seg + p) != __ldg(a.seg + (REV ? p + 1 : p - 1));
                const int64_t row = a.perm ? (int64_t)__ldg(a.perm + p) : p;
                if (a.validity == nullptr || bit_get(a.validity, row)) v[k] = lift_at<St, In>(a.values, row);
            }
            if (REV) r = r == 0 ? a.B - 1 : r - 1;
            else r = r + 1 == a.B ? 0 : r + 1;
            if (k > 0 && !f[k]) v[k] = cmb<St, REV>(v[k - 1], v[k]);
            any = any || f[k];
        }
        S tv = v[RS_ITEMS - 1];
        bool tf = any;
        s_v[threadIdx.x] = tv; s_f[threadIdx.x] = tf;
        __syncthreads();
        for (int o = 1; o < RS_THREADS; o <<= 1) {
            S pv = St::empty();
            int pf = 1;
            if ((int)threadIdx.x >= o) { pv = s_v[threadIdx.x - o]; pf = s_f[threadIdx.x - o]; }
            __syncthreads();
            if ((int)threadIdx.x >= o) {
                if (!tf) tv = cmb<St, REV>(pv, tv);
                tf = tf || pf;
                s_v[threadIdx.x] = tv; s_f[threadIdx.x] = tf;
            }
            __syncthreads();
        }
        S ex = carry;
        if (threadIdx.x > 0) ex = s_f[threadIdx.x - 1] ? s_v[threadIdx.x - 1] : cmb<St, REV>(carry, s_v[threadIdx.x - 1]);
        const S next = s_f[RS_THREADS - 1] ? s_v[RS_THREADS - 1] : cmb<St, REV>(carry, s_v[RS_THREADS - 1]);
        bool seen = false;
#pragma unroll
        for (int k = 0; k < RS_ITEMS; k++) {
            const int64_t j = j0 + k;
            if (j >= len) break;
            seen = seen || f[k];
            if (!seen) v[k] = cmb<St, REV>(ex, v[k]);
            outp[REV ? hi - 1 - j : lo + j] = v[k];
        }
        carry = next;
        __syncthreads();      // s_v is rewritten by the next tile
    }
}

// Writes position i's result to row perm[i] (the row itself without an order).  Validity: whole words by ballot over the
// rows (every lane of the warp calls this, `live` = the lane has a position), or atomicOr into a zeroed bitmap through perm.
template <class Fin> __device__ __forceinline__ void write_out(const RollArgs& a, int64_t i, bool live, bool ok, typename Fin::out_t x) {
    using Out = typename Fin::out_t;
    if (live) {
        const int64_t row = a.perm ? (int64_t)__ldg(a.perm + i) : i;
        reinterpret_cast<Out*>(a.out)[row] = ok ? x : Out(0);
        if (a.perm && ok) atomicOr(a.out_valid + (row >> 5), 1u << (row & 31));
    }
    if (!a.perm) {
        const unsigned bits = __ballot_sync(0xffffffffu, live && ok);
        if (lane_id() == 0 && i - (int64_t)lane_id() < a.n) a.out_valid[i >> 5] = bits;
    }
}

// ---------------------------------------------------------------------------------------------------- deterministic mode
// One thread replays one segment in the reference's order: rolling_apply_agg_window (nulls/mod.rs:46-98) calls
// update(start, end) for every position; both window types reset when the new start is at or past the old end.
__device__ __forceinline__ void seg_bounds(const RollArgs& a, int64_t g, int64_t& lo, int64_t& hi) {
    if (a.offsets) { lo = a.offsets[g]; hi = a.offsets[g + 1]; } else { lo = 0; hi = a.n; }
}
__device__ __forceinline__ void set_valid(uint32_t* bm, int64_t row) { atomicOr(bm + (row >> 5), 1u << (row & 31)); }
// The window [s, e) of position i of segment [lo, hi).  false: the output is null and update is not called -- a time-based
// window of fewer than min_samples positions, nulls included (rolling_apply_agg_window, rolling_kernels/shared.rs:109-204),
// or a position whose `by` is null.
__device__ __forceinline__ bool fold_window(const RollArgs& a, int64_t i, int64_t lo, int64_t hi, int64_t& s, int64_t& e) {
    if (!a.ws) { s = max(i - a.L, lo); e = min(i + a.R, hi); return true; }
    s = a.ws[i]; e = a.we[i];
    return a.ws[i] != BY_NULL && e - s >= a.min_samples;
}

// SumWindow<T, K> (rolling/sum.rs): Kahan add / sub of finite values in K, non-finite counters, null count.  In: the loaded
// type (integers for MEAN are cast to T = f64 first, as to_float does).  MEAN: (T)sum / (T)count (rolling/mean.rs:98-108).
template <typename In, typename T, typename K, bool MEAN>
__global__ void __launch_bounds__(64, 1) k_roll_fold_sum(const __grid_constant__ RollArgs a) {
    T* out = reinterpret_cast<T*>(a.out);
    for (int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; g < a.G; g += (int64_t)gridDim.x * blockDim.x) {
        int64_t lo, hi;
        seg_bounds(a, g, lo, hi);
        K sum = 0, ea = 0, es = 0;
        int64_t nf = 0, pinf = 0, ninf = 0, nulls = 0, start = lo, end = lo;
        auto at = [&](int64_t p, T& x) {
            const int64_t row = a.perm ? (int64_t)a.perm[p] : p;
            if (a.validity && !bit_get(a.validity, row)) return false;
            x = (T)load_in<In>(a.values, row);
            return true;
        };
        for (int64_t i = lo; i < hi; i++) {
            int64_t s, e;
            if (!fold_window(a, i, lo, hi, s, e)) { out[a.perm ? (int64_t)a.perm[i] : i] = T(0); continue; }
            if (s >= end) { sum = 0; ea = 0; es = 0; nf = pinf = ninf = nulls = 0; start = end = s; }
            for (int64_t p = start; p < s; p++) {
                T x;
                if (!at(p, x)) { nulls--; continue; }
                if (isfinite(x)) { const K y = (K)(T(0) - x) - es, ns = sum + y; es = (ns - sum) - y; sum = ns; }
                else { nf--; pinf -= x > T(0); ninf -= x < T(0); }
            }
            for (int64_t p = end; p < e; p++) {
                T x;
                if (!at(p, x)) { nulls++; continue; }
                if (isfinite(x)) { const K y = (K)x - ea, ns = sum + y; ea = (ns - sum) - y; sum = ns; }
                else { nf++; pinf += x > T(0); ninf += x < T(0); }
            }
            start = s; end = e;
            const int64_t cnt = (end - start) - nulls;
            T v = nf == 0 ? (T)sum : nf == pinf ? (T)INFINITY : nf == ninf ? (T)-INFINITY : (T)NAN;
            bool ok = cnt >= a.min_samples;
            if (MEAN) { ok = ok && cnt > 0; v = v / (T)cnt; }
            const int64_t row = a.perm ? (int64_t)a.perm[i] : i;
            out[row] = ok ? v : T(0);
            if (ok) set_valid(a.out_valid, row);
        }
    }
}

// MomentWindow<T, VarianceMoment> (rolling/moment.rs): a queue of two stacks.  back / agg_back take pushes; a pop from an
// empty front flips back into front (each entry the VarState of itself and everything pushed after it).  The stacks of
// segment [lo, hi) live in front[lo ..] / back[lo ..]: each holds at most min(w, hi - lo) entries.
template <typename In, typename Out, bool STD>
__global__ void __launch_bounds__(64, 1) k_roll_fold_var(const __grid_constant__ RollArgs a, VarSt::S* front, double* back) {
    Out* out = reinterpret_cast<Out*>(a.out);
    for (int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; g < a.G; g += (int64_t)gridDim.x * blockDim.x) {
        int64_t lo, hi;
        seg_bounds(a, g, lo, hi);
        VarSt::S agg_back = VarSt::empty();
        VarSt::S* fr = front + lo;
        double* bk = back + lo;
        // stack depths and counters stay below 2^32 (n <= 2^32 - 1)
        uint32_t nfront = 0, nback = 0, nf = 0, nulls = 0;
        int64_t start = lo, end = lo;
        auto at = [&](int64_t p, double& x) {
            const int64_t row = a.perm ? (int64_t)a.perm[p] : p;
            if (a.validity && !bit_get(a.validity, row)) return false;
            x = (double)load_in<In>(a.values, row);
            return true;
        };
        for (int64_t i = lo; i < hi; i++) {
            int64_t s, e;
            if (!fold_window(a, i, lo, hi, s, e)) { out[a.perm ? (int64_t)a.perm[i] : i] = Out(0); continue; }
            if (s >= end) { nf = nulls = 0; nfront = nback = 0; agg_back = VarSt::empty(); start = end = s; }
            for (int64_t p = start; p < s; p++) {
                double x;
                if (!at(p, x)) { nulls--; continue; }
                if (nfront == 0) {      // flip
                    VarSt::S agg = VarSt::empty();
                    while (nback > 0) { VarSt::insert_one(agg, bk[--nback]); fr[nfront++] = agg; }
                    agg_back = VarSt::empty();
                }
                nfront--;
                nf -= isfinite(x) ? 0u : 1u;
            }
            for (int64_t p = end; p < e; p++) {
                double x;
                if (!at(p, x)) { nulls++; continue; }
                if (!isfinite(x)) { x = 0.0; nf++; }
                bk[nback++] = x;
                VarSt::insert_one(agg_back, x);
            }
            start = s; end = e;
            VarSt::S st = agg_back;
            if (nfront) VarSt::combine_into(st, fr[nfront - 1]);
            st.nf = nf;
            double v;
            bool ok = VarSt::var(st, a.ddof, v) && (end - start) - (int64_t)nulls >= a.min_samples;
            Out o = ok ? (Out)v : Out(0);
            if (STD) o = sqrt(o);
            const int64_t row = a.perm ? (int64_t)a.perm[i] : i;
            out[row] = ok ? o : Out(0);
            if (ok) set_valid(a.out_valid, row);
        }
    }
}

// ---------------------------------------------------------------------------------------------------- host dispatch
// One plan per (kind, loaded type).  Plan::run<St, In, Fin>(a) runs the parallel plan of a state St over values loaded as In
// with the finisher Fin; deterministic mode runs the reference's machines instead (float SUM / MEAN / VAR / STD).
template <typename In, typename T, typename K, bool MEAN> static void run_fold_sum(const RollArgs& a) {
    PLB_LAUNCH("rolling_fold", (k_roll_fold_sum<In, T, K, MEAN>), grid_for(a.G, 64, 32), 64, 0, a);
}
template <typename In, typename Out, bool STD> static void run_fold_var(const RollArgs& a) {
    DevPtr front = dev_alloc((size_t)a.n * sizeof(VarSt::S)), back = dev_alloc((size_t)a.n * 8);
    PLB_LAUNCH("rolling_fold", (k_roll_fold_var<In, Out, STD>), grid_for(a.G, 64, 32), 64, 0, a, as<VarSt::S>(front), as<double>(back));
}

// one parallel plan per (kind, loaded type); In: the value type after small integers were widened to Int64
template <class Plan, typename In, typename Out> static void dispatch_float_kinds(int kind, const RollArgs& a, bool det) {
    constexpr bool in_f32 = std::is_same<In, float>::value;
    using TM = typename std::conditional<in_f32, float, double>::type;      // the reference's value type after to_float
    switch (kind) {
        case BL_ROLLING_MEAN:
            if (det) run_fold_sum<In, TM, double, true>(a);
            else Plan::template run<SumFltSt, In, FinMean<Out>>(a);
            break;
        case BL_ROLLING_VAR:
            if (det) run_fold_var<In, Out, false>(a);
            else Plan::template run<VarSt, In, FinVar<Out, false>>(a);
            break;
        default:
            if (det) run_fold_var<In, Out, true>(a);
            else Plan::template run<VarSt, In, FinVar<Out, true>>(a);
            break;
    }
}
template <class Plan, typename T> static void dispatch_minmax(int kind, const RollArgs& a) {
    if (kind == BL_ROLLING_MIN) Plan::template run<MinMaxSt<T, false>, T, FinMinMaxT<T>>(a);
    else Plan::template run<MinMaxSt<T, true>, T, FinMinMaxT<T>>(a);
}


template <class Plan> static void roll_dispatch(int kind, int dt, const RollArgs& a, bool det) {
    switch (kind) {
        case BL_ROLLING_SUM:
            switch (dt) {
                case BL_BOOL: Plan::template run<SumIntSt<uint32_t>, BoolBit, FinSumInt<uint32_t>>(a); break;
                case BL_INT32: case BL_UINT32: Plan::template run<SumIntSt<uint32_t>, uint32_t, FinSumInt<uint32_t>>(a); break;
                case BL_INT64: case BL_UINT64: Plan::template run<SumIntSt<uint64_t>, uint64_t, FinSumInt<uint64_t>>(a); break;
                case BL_FLOAT32: if (det) run_fold_sum<float, float, float, false>(a); else Plan::template run<SumFltSt, float, FinSumFlt<float>>(a); break;
                default: if (det) run_fold_sum<double, double, double, false>(a); else Plan::template run<SumFltSt, double, FinSumFlt<double>>(a); break;
            }
            break;
        case BL_ROLLING_MIN: case BL_ROLLING_MAX:
            switch (dt) {
                case BL_INT32: dispatch_minmax<Plan, int32_t>(kind, a); break;
                case BL_UINT32: dispatch_minmax<Plan, uint32_t>(kind, a); break;
                case BL_INT64: dispatch_minmax<Plan, int64_t>(kind, a); break;
                case BL_UINT64: dispatch_minmax<Plan, uint64_t>(kind, a); break;
                case BL_FLOAT32: dispatch_minmax<Plan, float>(kind, a); break;
                default: dispatch_minmax<Plan, double>(kind, a); break;
            }
            break;
        default:      // MEAN / VAR / STD
            switch (dt) {
                case BL_INT32: dispatch_float_kinds<Plan, int32_t, double>(kind, a, det); break;
                case BL_UINT32: dispatch_float_kinds<Plan, uint32_t, double>(kind, a, det); break;
                case BL_INT64: dispatch_float_kinds<Plan, int64_t, double>(kind, a, det); break;
                case BL_UINT64: dispatch_float_kinds<Plan, uint64_t, double>(kind, a, det); break;
                case BL_FLOAT32: dispatch_float_kinds<Plan, float, float>(kind, a, det); break;
                default: dispatch_float_kinds<Plan, double, double>(kind, a, det); break;
            }
            break;
    }
}

}  // namespace plb
