// window.cu — window functions `expr.over(partition_by, order_by=...)` with one output row per input row
// (mapping_strategy "group_to_rows": polars-expr/src/expressions/window.rs), and the plain cumulative functions.
//
// Plans (DESIGN.md §12):
//   1. whole column, no order_by   cum_* : k_over_scan straight over the rows (a decoupled look-back scan, no sort, no
//                                   gather); shift: k_over_shift as a shifted copy
//   2. aggregations, no order_by   the group_by plan bl_groupby_agg_params takes (fused K5, or GroupsIdx for FIRST / VAR /
//                                   MEDIAN ... and in deterministic mode) on the row -> first-row group ids, then ONE K4 gather
//                                   of every aggregate column through the row -> group ordinal map (so the fused plan needs
//                                   no group order: no sort at all)
//   3. everything else             the partition order, built once per call: op_group_tuples' sort of the group ids, or with
//                                   order_by a stable arg_sort of (group id, order key) (sortby.rs:57-100).  On that order:
//                                   k_over_scan (segmented: carries stop at a segment head), k_over_shift through the inverse
//                                   permutation, and op_group_fold for aggregations.
// The cumulative rules restate polars-ops/src/series/ops/cum_agg.rs: a null input gives a null output and leaves the state
// unchanged (:14-53), so the output validity of cum_sum / prod / min / max IS the input validity, and the scans write values
// only.  Integer scans wrap and are exact in any bracketing; min / max follow min_ignore_nan / max_ignore_nan (for floats
// <$T>::min / <$T>::max, polars-utils/src/min_max.rs:87-108): NaN is ignored (it is the identity), and between equal values
// (-0.0 / +0.0) min keeps the LATER one and max the EARLIER one in scan order (the tie rule the header states) — associative,
// so the parallel scan is bit-exact.  Float sums and products are
// reassociated by the parallel scan; bl_set_deterministic folds each partition sequentially instead (k_over_fold).
#include <algorithm>

#include "common.cuh"
#include "dev_utils.cuh"
#include "groupby.h"
#include "strings.cuh"

namespace plb {

// ---------------------------------------------------------------------------------------------------- scan operators
// S: the scan state; lift(x): a valid input as a state; combine(a, b): a earlier in scan order; out(s): the output value.

// SUM: integers wrap in the output width (Int8/16, UInt8/16 arrive as Int64; Bool -> UInt32); Float32 accumulates in f64 and
// rounds each output to f32 (det_sum_to_f64, cum_agg.rs:38-45)
template <typename In, typename S, typename Out> struct OpSum {
    using state = S; using in = In; using out_t = Out;
    __device__ static S identity() { return S(0); }
    __device__ static S lift(In x) { if constexpr (std::is_same<In, BoolBit>::value) return S(x.b ? 1 : 0); else return (S)x; }
    __device__ static S combine(S a, S b) { return a + b; }
    __device__ static Out out(S s) { return (Out)s; }
};
// PROD: Bool, Int8..UInt32 -> Int64 (cum_agg.rs:268-271); Int64 / UInt64 wrap (release build); floats keep the dtype
template <typename In, typename S, typename Out> struct OpProd {
    using state = S; using in = In; using out_t = Out;
    __device__ static S identity() { return S(1); }
    __device__ static S lift(In x) { if constexpr (std::is_same<In, BoolBit>::value) return S(x.b ? 1 : 0); else return (S)x; }
    __device__ static S combine(S a, S b) { return a * b; }
    __device__ static Out out(S s) { return (Out)s; }
};
template <typename T> struct Lim;
template <> struct Lim<int32_t> { __device__ static int32_t lo() { return INT32_MIN; } __device__ static int32_t hi() { return INT32_MAX; } };
template <> struct Lim<uint32_t> { __device__ static uint32_t lo() { return 0; } __device__ static uint32_t hi() { return UINT32_MAX; } };
template <> struct Lim<int64_t> { __device__ static int64_t lo() { return INT64_MIN; } __device__ static int64_t hi() { return INT64_MAX; } };
template <> struct Lim<uint64_t> { __device__ static uint64_t lo() { return 0; } __device__ static uint64_t hi() { return UINT64_MAX; } };
template <> struct Lim<float> { __device__ static float lo() { return __int_as_float(0x7fc00000); } __device__ static float hi() { return lo(); } };
template <> struct Lim<double> { __device__ static double lo() { return __longlong_as_double(0x7ff8000000000000ll); } __device__ static double hi() { return lo(); } };
template <typename T> __device__ __forceinline__ bool is_nan_v(T x) { if constexpr (std::is_floating_point<T>::value) return x != x; else return false; }
// min_ignore_nan(state, v) = state < v ? state : v, max_ignore_nan(state, v) = state < v ? v : state with NaN ignored
// (min_max.rs:33-48, floats :87-108; the ±0 tie as the header states): NaN is the identity (the initial state for floats, cum_agg.rs:78-112; the type's bound for integers)
template <typename T> struct OpMin {
    using state = T; using in = T; using out_t = T;
    __device__ static T identity() { return Lim<T>::hi(); }
    __device__ static T lift(T x) { return x; }
    __device__ static T combine(T a, T b) { if (is_nan_v(b)) return a; if (is_nan_v(a)) return b; return a < b ? a : b; }
    __device__ static T out(T s) { return s; }
};
template <typename T> struct OpMax {
    using state = T; using in = T; using out_t = T;
    __device__ static T identity() { return Lim<T>::lo(); }
    __device__ static T lift(T x) { return x; }
    __device__ static T combine(T a, T b) { if (is_nan_v(b)) return a; if (is_nan_v(a)) return b; return a < b ? b : a; }
    __device__ static T out(T s) { return s; }
};
// CUM_COUNT: valid values in [start, row] (forward) / [row, end] (reverse), cum_agg.rs:428-466
struct OpCount {
    using state = uint32_t; using in = BoolBit; using out_t = uint32_t;
    __device__ static uint32_t identity() { return 0; }
    __device__ static uint32_t lift(BoolBit) { return 1; }
    __device__ static uint32_t combine(uint32_t a, uint32_t b) { return a + b; }
    __device__ static uint32_t out(uint32_t s) { return s; }
};

// every scan but CUM_COUNT gives a null (written as 0) at a null input
template <class Op> constexpr bool kNullOut = !std::is_same<Op, OpCount>::value;

template <typename S> __device__ __forceinline__ uint64_t to_bits(S s) {
    if constexpr (sizeof(S) == 8) { uint64_t u; memcpy(&u, &s, 8); return u; }
    else { uint32_t u; memcpy(&u, &s, 4); return u; }
}
template <typename S> __device__ __forceinline__ S from_bits(uint64_t u) {
    S s;
    if constexpr (sizeof(S) == 8) memcpy(&s, &u, 8);
    else { const uint32_t w = (uint32_t)u; memcpy(&s, &w, 4); }
    return s;
}

// ---------------------------------------------------------------------------------------------------- k_over_scan
// Logical element i in [0, n) is position p = reverse ? n - 1 - i : i of the partition order, row = perm[p] (perm == NULL:
// the rows themselves).  i starts a segment when i == 0 or seg[p] != seg[p of i - 1] (seg: the group id of each position;
// NULL: one segment).  A segmented value is (head, v): combine((fa, a), (fb, b)) = (fa | fb, fb ? b : a (+) b).
// Tiles of OS_TILE elements: each warp takes 256 consecutive elements as 8 coalesced rounds of 32; tiles are handed out by an
// atomic counter, so every predecessor of a tile is already running when it looks back (forward progress).
// Tile status: st_flag[t] = OS_AGG / OS_INC | OS_HEAD (the tile holds a segment head); the value bits are in st_agg[t] /
// st_inc[t], two slots that are each written once, before the flag that announces them (with a fence between), so that a
// reader that saw OS_AGG never reads the inclusive value in its place.
constexpr int OS_THREADS = 256, OS_ITEMS = 8, OS_TILE = OS_THREADS * OS_ITEMS;
constexpr uint32_t OS_AGG = 1, OS_INC = 2, OS_HEAD = 4;
struct ScanArgs {
    const void* values; const uint32_t* validity; const uint32_t* perm; const uint32_t* seg; int64_t n; int reverse;
    void* out; uint64_t* st_agg; uint64_t* st_inc; uint32_t* st_flag; unsigned* tile_counter; int* error;
};

template <class Op> __device__ __forceinline__ void seg_combine(bool& f, typename Op::state& v, bool fa, typename Op::state a) {
    // (fa, a) earlier, (f, v) later
    if (!f) v = Op::combine(a, v);
    f = f || fa;
}

template <class Op>
__global__ void __launch_bounds__(OS_THREADS, 2) k_over_scan(const __grid_constant__ ScanArgs a) {
    using S = typename Op::state;
    using Out = typename Op::out_t;
    __shared__ S s_wv[OS_THREADS / 32];
    __shared__ int s_wf[OS_THREADS / 32];
    __shared__ long long s_tile;
    const unsigned lane = lane_id(), warp = threadIdx.x >> 5;
    const int64_t n = a.n, ntiles = (n + OS_TILE - 1) / OS_TILE;
    while (true) {
        if (threadIdx.x == 0) s_tile = (long long)atomicAdd(a.tile_counter, 1u);
        __syncthreads();
        const int64_t t = s_tile;
        if (t >= ntiles) break;
        const int64_t wbase = t * OS_TILE + (int64_t)warp * (32 * OS_ITEMS);
        S v[OS_ITEMS]; bool f[OS_ITEMS]; int64_t rows[OS_ITEMS];
        // loads first (8 independent rounds in flight), then the warp scans
#pragma unroll
        for (int j = 0; j < OS_ITEMS; j++) {
            const int64_t i = wbase + j * 32 + lane;
            v[j] = Op::identity(); f[j] = false; rows[j] = -1;
            if (i < n) {
                const int64_t p = a.reverse ? n - 1 - i : i;
                const int64_t row = a.perm ? (int64_t)__ldg(a.perm + p) : p;
                rows[j] = row;
                f[j] = i == 0 || (a.seg && __ldg(a.seg + p) != __ldg(a.seg + (a.reverse ? p + 1 : p - 1)));
                const bool valid = a.validity == nullptr || bit_get(a.validity, row);
                if (valid) v[j] = Op::lift(load_in<typename Op::in>(a.values, row));
            }
        }
        S carry = Op::identity(); bool cf = false;
#pragma unroll
        for (int j = 0; j < OS_ITEMS; j++) {
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const S pv = from_bits<S>(__shfl_up_sync(0xffffffffu, to_bits(v[j]), o));
                const bool pf = __shfl_up_sync(0xffffffffu, (int)f[j], o) != 0;
                if (lane >= (unsigned)o) seg_combine<Op>(f[j], v[j], pf, pv);
            }
            seg_combine<Op>(f[j], v[j], cf, carry);
            carry = from_bits<S>(__shfl_sync(0xffffffffu, to_bits(v[j]), 31));
            cf = __shfl_sync(0xffffffffu, (int)f[j], 31) != 0;
        }
        if (lane == 31) { s_wv[warp] = carry; s_wf[warp] = cf; }
        __syncthreads();
        if (warp == 0) {
            // exclusive prefix of the 8 warp totals (lanes 0..7), the tile total in lane 7
            S wv = lane < OS_THREADS / 32 ? s_wv[lane] : Op::identity();
            bool wf = lane < OS_THREADS / 32 ? s_wf[lane] != 0 : false;
#pragma unroll
            for (int o = 1; o < OS_THREADS / 32; o <<= 1) {
                const S pv = from_bits<S>(__shfl_up_sync(0xffffffffu, to_bits(wv), o));
                const bool pf = __shfl_up_sync(0xffffffffu, (int)wf, o) != 0;
                if (lane >= (unsigned)o) seg_combine<Op>(wf, wv, pf, pv);
            }
            const S tot = from_bits<S>(__shfl_sync(0xffffffffu, to_bits(wv), OS_THREADS / 32 - 1));
            const bool totf = __shfl_sync(0xffffffffu, (int)wf, OS_THREADS / 32 - 1) != 0;
            S wex = from_bits<S>(__shfl_up_sync(0xffffffffu, to_bits(wv), 1));
            bool wexf = __shfl_up_sync(0xffffffffu, (int)wf, 1) != 0;
            if (lane == 0) { wex = Op::identity(); wexf = false; }
            // decoupled look-back: the tile's exclusive prefix
            if (lane == 0) {
                (t == 0 ? a.st_inc : a.st_agg)[t] = to_bits(tot);
                __threadfence();
                atomicExch(&a.st_flag[t], (t == 0 ? OS_INC : OS_AGG) | (totf ? OS_HEAD : 0u));
            }
            S ex = Op::identity(); bool exf = false;
            int64_t look = t - 1;
            while (look >= 0) {
                const int64_t idx = look - lane;      // lane 0 = the nearest predecessor
                uint32_t fl = OS_INC;                 // before tile 0: an inclusive identity
                int spins = 0;
                bool failed = false;
                if (idx >= 0) fl = *reinterpret_cast<volatile uint32_t*>(&a.st_flag[idx]);
                while (__any_sync(0xffffffffu, fl == 0)) {
                    if (idx >= 0 && fl == 0) fl = *reinterpret_cast<volatile uint32_t*>(&a.st_flag[idx]);
                    // never hang the device: lane 0 decides for the whole warp, so every lane leaves the loop together
                    int give_up = 0;
                    if (lane == 0) give_up = ++spins > (1 << 22) || ((spins & 1023) == 0 && *reinterpret_cast<volatile int*>(a.error));
                    if (__shfl_sync(0xffffffffu, give_up, 0)) { failed = true; break; }
                }
                if (failed) { if (lane == 0) *a.error = 1; break; }
                __threadfence();
                S pv = Op::identity(); bool pf = false;
                if (idx >= 0) { pv = from_bits<S>(*reinterpret_cast<volatile uint64_t*>((fl & OS_INC) ? &a.st_inc[idx] : &a.st_agg[idx])); pf = (fl & OS_HEAD) != 0; }
                // the nearest predecessor whose value needs nothing earlier: an inclusive prefix or a tile with a head
                const unsigned stop = __ballot_sync(0xffffffffu, (fl & OS_INC) != 0 || (fl & OS_HEAD) != 0);
                const int k = stop ? __ffs(stop) - 1 : 31;
                if ((int)lane > k) { pv = Op::identity(); pf = false; }
                // ordered reduction: lane l + o is earlier than lane l
#pragma unroll
                for (int o = 1; o < 32; o <<= 1) {
                    const S qv = from_bits<S>(__shfl_down_sync(0xffffffffu, to_bits(pv), o));
                    const bool qf = __shfl_down_sync(0xffffffffu, (int)pf, o) != 0;
                    if (lane + o < 32) seg_combine<Op>(pf, pv, qf, qv);
                }
                pv = from_bits<S>(__shfl_sync(0xffffffffu, to_bits(pv), 0));
                pf = __shfl_sync(0xffffffffu, (int)pf, 0) != 0;
                seg_combine<Op>(exf, ex, pf, pv);      // the window is earlier than what was gathered so far
                if (stop) break;
                look -= 32;
            }
            if (lane == 0 && t > 0) {
                bool incf = totf; S inc = tot;
                seg_combine<Op>(incf, inc, exf, ex);
                a.st_inc[t] = to_bits(inc);
                __threadfence();
                atomicExch(&a.st_flag[t], OS_INC | (incf ? OS_HEAD : 0u));
            }
            // prefix of warp w = tile exclusive (+) warp exclusive
            seg_combine<Op>(wexf, wex, exf, ex);
            if (lane < OS_THREADS / 32) { s_wv[lane] = wex; s_wf[lane] = wexf; }
        }
        __syncthreads();
        const S pre = s_wv[warp];
        Out* out = reinterpret_cast<Out*>(a.out);
#pragma unroll
        for (int j = 0; j < OS_ITEMS; j++) {
            if (rows[j] < 0) continue;
            S r = v[j];
            if (!f[j]) r = Op::combine(pre, r);
            const bool valid = !kNullOut<Op> || a.validity == nullptr || bit_get(a.validity, rows[j]);
            out[rows[j]] = valid ? Op::out(r) : Out(0);
        }
        __syncthreads();      // s_wv / s_tile are reused by the next tile
    }
}

// Deterministic mode: one thread folds one segment sequentially in scan order (float CUM_SUM / CUM_PROD bit-identical to the
// reference's det_sum / det_sum_to_f64 / det_prod).  offsets: G + 1 positions of the partition order; perm NULL = the rows.
template <class Op>
__global__ void __launch_bounds__(128) k_over_fold(const void* values, const uint32_t* validity, const uint32_t* perm, const uint32_t* offsets, int64_t G,
                                                  int reverse, void* out_) {
    using S = typename Op::state;
    using Out = typename Op::out_t;
    Out* out = reinterpret_cast<Out*>(out_);
    for (int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; g < G; g += (int64_t)gridDim.x * blockDim.x) {
        const int64_t lo = offsets[g], hi = offsets[g + 1];
        S s = Op::identity();
        for (int64_t k = 0; k < hi - lo; k++) {
            const int64_t p = reverse ? hi - 1 - k : lo + k;
            const int64_t row = perm ? (int64_t)perm[p] : p;
            if (validity && !bit_get(validity, row)) { if (kNullOut<Op>) out[row] = Out(0); else out[row] = Op::out(s); continue; }
            s = Op::combine(s, Op::lift(load_in<typename Op::in>(values, row)));
            out[row] = Op::out(s);
        }
    }
}

// ---------------------------------------------------------------------------------------------------- k_over_shift
// Over rows: row r sits at position p = inv[r] of the partition order (inv NULL: p = r); its output is the value at position
// q = p - periods when q is inside the array and in r's segment (seg[q] == seg[p]) and that row is valid, else null.
// Validity words are written whole, one ballot per 32 rows.
template <int ES>
__global__ void __launch_bounds__(256) k_over_shift(const void* __restrict__ values, const uint32_t* __restrict__ validity, const uint32_t* __restrict__ perm,
                                                   const uint32_t* __restrict__ inv, const uint32_t* __restrict__ seg, int64_t n, int64_t periods,
                                                   void* __restrict__ out, uint32_t* __restrict__ out_valid) {
    using E = typename std::conditional<ES == 8, uint64_t, typename std::conditional<ES == 4, uint32_t, typename std::conditional<ES == 2, uint16_t, uint8_t>::type>::type>::type;
    const int64_t n_round = (n + 31) / 32 * 32;
    for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < n_round; r += (int64_t)gridDim.x * blockDim.x) {
        bool ok = false; E x = 0;
        if (r < n) {
            const int64_t p = inv ? (int64_t)inv[r] : r;
            const int64_t q = p - periods;      // |periods| <= n + 1 (clamped on the host)
            if (q >= 0 && q < n && (seg == nullptr || __ldg(seg + q) == __ldg(seg + p))) {
                const int64_t src = perm ? (int64_t)__ldg(perm + q) : q;
                ok = validity == nullptr || bit_get(validity, src);
                if (ok) x = __ldg(reinterpret_cast<const E*>(values) + src);
            }
            reinterpret_cast<E*>(out)[r] = x;
        }
        const unsigned b = __ballot_sync(0xffffffffu, ok);
        if (lane_id() == 0) out_valid[r >> 5] = b;
    }
}

// ---------------------------------------------------------------------------------------------------- order helpers
__global__ void __launch_bounds__(256) k_over_inverse(const uint32_t* __restrict__ perm, int64_t n, uint32_t* __restrict__ inv) {
    for (int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; p < n; p += (int64_t)gridDim.x * blockDim.x) inv[perm[p]] = (uint32_t)p;
}
// seg[p] = gid[perm[p]]: the group id of every position of the partition order (one per order build)
__global__ void __launch_bounds__(256) k_over_seg_ids(const uint32_t* __restrict__ gid, const uint32_t* __restrict__ perm, int64_t n, uint32_t* __restrict__ seg) {
    for (int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; p < n; p += (int64_t)gridDim.x * blockDim.x) seg[p] = __ldg(gid + perm[p]);
}
// slot[first row of group g] = g; the first row is first[offsets[g]] (offsets != NULL: first = seg ids of the order) or first[g]
__global__ void __launch_bounds__(256) k_over_first_ordinal(const uint32_t* __restrict__ first, const uint32_t* __restrict__ offsets, int64_t G, uint32_t* __restrict__ slot) {
    for (int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; g < G; g += (int64_t)gridDim.x * blockDim.x)
        slot[first[offsets ? offsets[g] : g]] = (uint32_t)g;
}
__global__ void __launch_bounds__(256) k_over_row_ordinal(const uint32_t* __restrict__ gid, const uint32_t* __restrict__ slot, int64_t n, uint32_t* __restrict__ ord) {
    for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < n; r += (int64_t)gridDim.x * blockDim.x) ord[r] = __ldg(slot + gid[r]);
}

// ---------------------------------------------------------------------------------------------------- host side
static bool is_agg(int kind) { return kind >= BL_AGG_SUM && kind <= BL_AGG_QUANTILE; }
static bool is_cum(int kind) { return kind >= BL_CUM_SUM && kind <= BL_CUM_COUNT; }

// output dtype of a scan / shift (aggregations: the group_by's own)
int over_scan_dtype(int kind, int dt) {
    switch (kind) {
        case BL_CUM_SUM:
            if (dt == BL_BOOL) return BL_UINT32;
            return dtype_is_small_int(dt) ? BL_INT64 : dt;
        case BL_CUM_PROD:
            if (dt == BL_BOOL || dtype_is_small_int(dt) || dt == BL_INT32 || dt == BL_UINT32) return BL_INT64;
            return dt;
        case BL_CUM_COUNT: return BL_UINT32;
        default: return dt;      // MIN / MAX / SHIFT
    }
}

template <class Op> static void launch_scan(const DevCol& v, const OverOrder* o, bool reverse, DevCol& out) {
    const int64_t n = v.len;
    if (n == 0) return;
    const int64_t ntiles = (n + OS_TILE - 1) / OS_TILE;
    DevPtr sv = dev_alloc((size_t)ntiles * 16), sf = dev_alloc((size_t)ntiles * 4 + 16);
    dev_memset(sf->p, 0, (size_t)ntiles * 4 + 16);
    ScanArgs a;
    memset(&a, 0, sizeof a);
    a.values = v.v(); a.validity = v.vm(); a.n = n; a.reverse = reverse ? 1 : 0; a.out = out.values->p;
    a.perm = o ? as<uint32_t>(o->perm.values) : nullptr;
    a.seg = o ? as<uint32_t>(o->seg.values) : nullptr;
    a.st_agg = as<uint64_t>(sv); a.st_inc = as<uint64_t>(sv) + ntiles; a.st_flag = as<uint32_t>(sf);
    a.tile_counter = reinterpret_cast<unsigned*>(as<uint32_t>(sf) + ntiles);
    a.error = reinterpret_cast<int*>(as<uint32_t>(sf) + ntiles + 1);
    const int grid = (int)std::min<int64_t>(ntiles, (int64_t)ctx().sm_count * 8);
    PLB_LAUNCH(o ? "over_scan_seg" : "over_scan", k_over_scan<Op>, grid, OS_THREADS, 0, a);
    PLB_REQUIRE(read_scalar(a.error) == 0, BL_ERR_CUDA, "over: the scan's look-back did not complete");
}

template <class Op> static void launch_fold(const DevCol& v, const OverOrder* o, bool reverse, DevCol& out) {
    const int64_t n = v.len;
    if (n == 0) return;
    DevPtr whole;
    const uint32_t* offsets;
    int64_t G;
    if (o) { offsets = as<uint32_t>(o->offsets.values); G = o->G; }
    else {
        whole = dev_alloc(8);
        const uint32_t h[2] = {0u, (uint32_t)n};
        PLB_CUDA(cudaMemcpyAsync(whole->p, h, 8, cudaMemcpyHostToDevice, ctx().stream));
        PLB_CUDA(cudaStreamSynchronize(ctx().stream));      // h lives on this frame
        offsets = as<uint32_t>(whole); G = 1;
    }
    PLB_LAUNCH("over_fold", k_over_fold<Op>, grid_for(G, 128, 16), 128, 0, v.v(), v.vm(), o ? as<uint32_t>(o->perm.values) : nullptr, offsets, G, reverse ? 1 : 0, out.values->p);
}

template <class Op> static void run_scan(const DevCol& v, const OverOrder* o, bool reverse, DevCol& out, bool sequential) {
    if (sequential) launch_fold<Op>(v, o, reverse, out);
    else launch_scan<Op>(v, o, reverse, out);
}

// CUM_SUM / PROD / MIN / MAX / COUNT of one column; v: small integers already widened where the reference casts
static DevCol over_cum(int kind, const DevCol& v, int in_dt, const OverOrder* o, bool reverse) {
    const int odt = over_scan_dtype(kind, in_dt);
    DevCol out = make_col(odt, v.len, false);
    if (kind != BL_CUM_COUNT) { out.validity = v.validity; out.null_count = v.null_count; }
    else out.null_count = 0;
    const bool det = ctx().deterministic;      // float SUM / PROD: the reference's sequential fold
    switch (kind) {
        case BL_CUM_COUNT: run_scan<OpCount>(v, o, reverse, out, false); break;
        case BL_CUM_SUM:
            switch (v.dtype) {
                case BL_BOOL: run_scan<OpSum<BoolBit, uint32_t, uint32_t>>(v, o, reverse, out, false); break;
                case BL_INT32: case BL_UINT32: run_scan<OpSum<uint32_t, uint32_t, uint32_t>>(v, o, reverse, out, false); break;
                case BL_INT64: case BL_UINT64: run_scan<OpSum<uint64_t, uint64_t, uint64_t>>(v, o, reverse, out, false); break;
                case BL_FLOAT32: run_scan<OpSum<float, double, float>>(v, o, reverse, out, det); break;
                default: run_scan<OpSum<double, double, double>>(v, o, reverse, out, det); break;
            }
            break;
        case BL_CUM_PROD:
            switch (v.dtype) {
                case BL_BOOL: run_scan<OpProd<BoolBit, uint64_t, uint64_t>>(v, o, reverse, out, false); break;
                case BL_INT32: run_scan<OpProd<int32_t, uint64_t, uint64_t>>(v, o, reverse, out, false); break;
                case BL_UINT32: run_scan<OpProd<uint32_t, uint64_t, uint64_t>>(v, o, reverse, out, false); break;
                case BL_INT64: case BL_UINT64: run_scan<OpProd<uint64_t, uint64_t, uint64_t>>(v, o, reverse, out, false); break;
                case BL_FLOAT32: run_scan<OpProd<float, float, float>>(v, o, reverse, out, det); break;
                default: run_scan<OpProd<double, double, double>>(v, o, reverse, out, det); break;
            }
            break;
        case BL_CUM_MIN:
            switch (v.dtype) {
                case BL_INT32: run_scan<OpMin<int32_t>>(v, o, reverse, out, false); break;
                case BL_UINT32: run_scan<OpMin<uint32_t>>(v, o, reverse, out, false); break;
                case BL_INT64: run_scan<OpMin<int64_t>>(v, o, reverse, out, false); break;
                case BL_UINT64: run_scan<OpMin<uint64_t>>(v, o, reverse, out, false); break;
                case BL_FLOAT32: run_scan<OpMin<float>>(v, o, reverse, out, false); break;
                default: run_scan<OpMin<double>>(v, o, reverse, out, false); break;
            }
            break;
        default:
            switch (v.dtype) {
                case BL_INT32: run_scan<OpMax<int32_t>>(v, o, reverse, out, false); break;
                case BL_UINT32: run_scan<OpMax<uint32_t>>(v, o, reverse, out, false); break;
                case BL_INT64: run_scan<OpMax<int64_t>>(v, o, reverse, out, false); break;
                case BL_UINT64: run_scan<OpMax<uint64_t>>(v, o, reverse, out, false); break;
                case BL_FLOAT32: run_scan<OpMax<float>>(v, o, reverse, out, false); break;
                default: run_scan<OpMax<double>>(v, o, reverse, out, false); break;
            }
            break;
    }
    return out;
}

static DevCol over_shift(const DevCol& v, const OverOrder* o, int64_t periods) {
    const int64_t n = v.len;
    DevCol out = make_col(v.dtype, n, true);
    out.null_count = -1;
    if (n == 0) return out;
    periods = std::max<int64_t>(-(n + 1), std::min<int64_t>(n + 1, periods));
    const uint32_t* perm = o ? as<uint32_t>(o->perm.values) : nullptr;
    const uint32_t* inv = o ? as<uint32_t>(o->inv.values) : nullptr;
    const uint32_t* seg = o ? as<uint32_t>(o->seg.values) : nullptr;
    const int grid = grid_for((n + 31) / 32 * 32, 256);
    switch (dtype_size(v.dtype)) {
        case 1: PLB_LAUNCH("over_shift", k_over_shift<1>, grid, 256, 0, v.v(), v.vm(), perm, inv, seg, n, periods, out.values->p, as<uint32_t>(out.validity)); break;
        case 2: PLB_LAUNCH("over_shift", k_over_shift<2>, grid, 256, 0, v.v(), v.vm(), perm, inv, seg, n, periods, out.values->p, as<uint32_t>(out.validity)); break;
        case 4: PLB_LAUNCH("over_shift", k_over_shift<4>, grid, 256, 0, v.v(), v.vm(), perm, inv, seg, n, periods, out.values->p, as<uint32_t>(out.validity)); break;
        default: PLB_LAUNCH("over_shift", k_over_shift<8>, grid, 256, 0, v.v(), v.vm(), perm, inv, seg, n, periods, out.values->p, as<uint32_t>(out.validity)); break;
    }
    return out;
}

// The partition order, once per call.  Without order_by: op_group_tuples_ids (groups in first-occurrence order, rows
// ascending).  With it: the stable arg_sort of (group id, order key), exactly update_groups_sort_by's per-group stable sort
// (sortby.rs:57-100) with the groups in first-occurrence order; segments start where the group id changes.
void build_order(OverOrder& o, const DevCol* order_key, int order_flags, bool need_inv) {
    const int64_t n = o.gid.len;
    DevCol first;
    if (!order_key) {
        o.seg = make_col(BL_UINT32, n, false);
        if (n) PLB_CUDA(cudaMemcpyAsync(o.seg.values->p, o.gid.v(), (size_t)n * 4, cudaMemcpyDeviceToDevice, ctx().stream));
        op_group_tuples_ids(o.seg, first, o.offsets, o.perm);
    } else {
        o.perm = op_arg_sort({o.gid, *order_key}, {0, order_flags}, -1);
        o.seg = make_col(BL_UINT32, n, false);
        if (n) PLB_LAUNCH("over_seg_ids", k_over_seg_ids, grid_for(n, 256), 256, 0, as<uint32_t>(o.gid.values), as<uint32_t>(o.perm.values), n, as<uint32_t>(o.seg.values));
        op_group_offsets(o.seg, o.perm, first, o.offsets);
    }
    o.G = o.offsets.len - 1;
    if (need_inv) {
        o.inv = make_col(BL_UINT32, n, false);
        if (n) PLB_LAUNCH("over_inverse", k_over_inverse, grid_for(n, 256), 256, 0, as<uint32_t>(o.perm.values), n, as<uint32_t>(o.inv.values));
    }
}

// row -> ordinal of its group, given the groups' first rows (first[offsets[g]] when offsets is set)
static DevCol row_ordinals(const DevCol& gid, const uint32_t* first, const uint32_t* offsets, int64_t G) {
    const int64_t n = gid.len;
    DevCol slot = make_col(BL_UINT32, n, false), ord = make_col(BL_UINT32, n, false);
    ord.null_count = 0;
    if (G) PLB_LAUNCH("over_first_ordinal", k_over_first_ordinal, grid_for(G, 256), 256, 0, first, offsets, G, as<uint32_t>(slot.values));
    if (n) PLB_LAUNCH("over_row_ordinal", k_over_row_ordinal, grid_for(n, 256), 256, 0, as<uint32_t>(gid.values), as<uint32_t>(slot.values), n, as<uint32_t>(ord.values));
    return ord;
}

// every aggregation of the call: per-group results broadcast to the rows in ONE K4 gather
static void over_aggs(const OverOrder& o, bool with_order, const std::vector<OverOp>& ops, const std::vector<DevCol>& vals, std::vector<DevCol>& outs) {
    std::vector<int> at, kinds, dts, nullable, in_dt;
    std::vector<const DevCol*> vptr;
    std::vector<bl_agg_param> params;
    std::vector<DevCol> tmp(ops.size());
    for (size_t i = 0; i < ops.size(); i++) {
        const int kind = ops[i].kind & 0xFFFF;
        if (!is_agg(kind)) continue;
        at.push_back((int)i);
        params.push_back(ops[i].param);
        if (kind == BL_AGG_LEN) { kinds.push_back(ops[i].kind); dts.push_back(BL_INT64); nullable.push_back(0); in_dt.push_back(-1); continue; }
        DevCol v = vals[i];
        in_dt.push_back(v.dtype);
        if (kind == BL_AGG_N_UNIQUE) {
            // distinct values per group, a null counting as one (aggregations/dispatch.rs:285-345): COUNT of the rows that are the
            // first of their (group, value) pair, as bl_groupby_agg does it
            DevCol ids = op_group_first_ids(op_pack_keys({o.gid, v}));
            DevCol iota = make_col(BL_UINT32, v.len, false);
            iota_u32(as<uint32_t>(iota.values), v.len, 0);
            DevCol is_first = op_compare(BL_CMP_EQ, ids, iota, false);
            tmp[i].dtype = BL_UINT32; tmp[i].len = v.len; tmp[i].values = ids.values; tmp[i].validity = is_first.values; tmp[i].null_count = -1;
            kinds.push_back(BL_AGG_COUNT);
        } else {
            if (kind == BL_AGG_COUNT && v.dtype == BL_BOOL) { tmp[i] = v; tmp[i].dtype = BL_UINT32; tmp[i].values = v.validity ? v.validity : v.values; }      // only the validity is read
            else tmp[i] = dtype_is_small_int(v.dtype) ? op_cast_small_int(v, BL_INT64, false) : v;
            kinds.push_back(ops[i].kind);
        }
        dts.push_back(tmp[i].dtype);
        nullable.push_back(tmp[i].validity != nullptr);
    }
    if (at.empty()) return;
    vptr.assign(at.size(), nullptr);
    for (size_t k = 0; k < at.size(); k++) if ((ops[at[k]].kind & 0xFFFF) != BL_AGG_LEN) vptr[k] = &tmp[at[k]];
    std::vector<DevCol> oa;
    DevCol ord;
    if (with_order) {      // fold over the order_by order (the order-sensitive kinds see it)
        op_group_fold(o.offsets, o.perm, kinds, vptr, oa, params.data());
        ord = row_ordinals(o.gid, as<uint32_t>(o.seg.values), as<uint32_t>(o.offsets.values), o.G);
    } else {
        DevCol first;
        bool groups_idx = ctx().deterministic;
        for (int k : kinds) groups_idx |= (k & 0xFFFF) >= BL_AGG_FIRST;
        if (groups_idx) op_group_by_exact(o.gid, kinds, vptr, first, oa, params.data());
        else {
            GroupByState st(BL_UINT32, kinds, dts, nullable, 0, true);
            st.consume_all(o.gid, vptr);
            DevCol ok;
            st.finish(false, nullptr, ok, oa, &first);      // any group order: the ordinals map every row to its own group
        }
        ord = row_ordinals(o.gid, as<uint32_t>(first.values), nullptr, first.len);
    }
    std::vector<DevCol> rows;
    op_gather(oa, ord, false, rows);
    for (size_t k = 0; k < at.size(); k++) {
        const int kind = ops[at[k]].kind & 0xFFFF;
        DevCol r = rows[k];
        if ((kind == BL_AGG_MIN || kind == BL_AGG_MAX || kind == BL_AGG_FIRST || kind == BL_AGG_LAST) && dtype_is_small_int(in_dt[k])) r = op_cast_small_int(r, in_dt[k], false);
        outs[at[k]] = r;
    }
}

// argument errors of one operation, from its descriptor (before any upload); value_dtype < 0: no value column
void check_over_op(int kind_word, int value_dtype) {
    const int kind = kind_word & 0xFFFF;
    PLB_REQUIRE(is_agg(kind) || is_cum(kind) || kind == BL_SHIFT, BL_ERR_INVALID, "over: unknown kind " + std::to_string(kind_word));
    PLB_REQUIRE(kind == BL_AGG_LEN || value_dtype >= 0, BL_ERR_INVALID, "over: an operation without a value column");
    if (value_dtype < 0) return;
    PLB_REQUIRE(value_dtype <= BL_BOOL, BL_ERR_INVALID, "over: unknown value dtype");
    if (value_dtype != BL_BOOL) return;
    PLB_REQUIRE(kind != BL_CUM_MIN && kind != BL_CUM_MAX && kind != BL_SHIFT, BL_ERR_UNSUPPORTED, "over: cum_min / cum_max / shift of a Boolean column are outside the hot path");
    PLB_REQUIRE(!is_agg(kind) || kind == BL_AGG_LEN || kind == BL_AGG_COUNT, BL_ERR_UNSUPPORTED, "over: aggregations other than count / len of a Boolean column are outside the hot path");
}

// output dtype of an aggregation broadcast over an empty column (the group_by's rules)
static int over_agg_dtype(int kind, int dt) {
    switch (kind) {
        case BL_AGG_SUM: return dtype_is_small_int(dt) ? BL_INT64 : dt;
        case BL_AGG_MIN: case BL_AGG_MAX: case BL_AGG_FIRST: case BL_AGG_LAST: return dt;
        case BL_AGG_MEAN: case BL_AGG_VAR: case BL_AGG_STD: case BL_AGG_MEDIAN: case BL_AGG_QUANTILE: return dt == BL_FLOAT32 ? BL_FLOAT32 : BL_FLOAT64;
        default: return BL_UINT32;
    }
}

// row -> first row of its partition (UInt32); no partition columns: every row in partition 0
DevCol partition_ids(const std::vector<DevCol>& partition_by, int64_t n) {
    DevCol gid;
    if (!partition_by.empty()) gid = op_group_first_ids(op_pack_keys(partition_by));
    else { gid = make_col(BL_UINT32, n, false); dev_memset(gid.values->p, 0, (size_t)n * 4); }
    gid.null_count = 0;
    return gid;
}

// ops are checked by the caller (check_over_op) before any column is uploaded
std::vector<DevCol> op_over(const std::vector<DevCol>& partition_by, const DevCol* order_key, int order_flags, const std::vector<OverOp>& ops, int64_t n) {
    std::vector<DevCol> vals(ops.size());
    for (size_t i = 0; i < ops.size(); i++) {
        if (!ops[i].values) continue;
        PLB_REQUIRE(ops[i].values->len == n, BL_ERR_INVALID, "over: value column " + std::to_string(i) + " has " + std::to_string(ops[i].values->len) + " rows, not " + std::to_string(n));
        vals[i] = *ops[i].values;
    }
    for (auto& k : partition_by) PLB_REQUIRE(k.len == n, BL_ERR_INVALID, "over: partition columns differ in length");
    if (order_key) PLB_REQUIRE(order_key->len == n, BL_ERR_INVALID, "over: the order_by column differs in length");
    const bool partitioned = !partition_by.empty();
    bool need_order = false, need_inv = false, any_agg = false;
    for (auto& op : ops) {
        const int kind = op.kind & 0xFFFF;
        any_agg |= is_agg(kind);
        if (!is_agg(kind) && (partitioned || order_key)) need_order = true;
        if (kind == BL_SHIFT && (partitioned || order_key)) need_inv = true;
    }
    if (any_agg && order_key) need_order = true;
    PLB_REQUIRE(!need_order || n <= 0x7FFFFFFFll, BL_ERR_UNSUPPORTED, "over: more than 2^31 - 1 rows need a sort (group tuples)");
    PLB_REQUIRE(n <= 0xFFFFFFFFll, BL_ERR_UNSUPPORTED, "over: more than 2^32 - 1 rows (IdxSize is u32)");
    std::vector<DevCol> outs(ops.size());
    if (n == 0) {
        for (size_t i = 0; i < ops.size(); i++) {
            const int kind = ops[i].kind & 0xFFFF, dt = vals[i].dtype;
            outs[i] = make_col(is_agg(kind) ? over_agg_dtype(kind, ops[i].values ? dt : BL_UINT32) : over_scan_dtype(kind, dt), 0, false);
            outs[i].null_count = 0;
        }
        return outs;
    }

    OverOrder o;
    if (any_agg || need_order) o.gid = partition_ids(partition_by, n);
    if (need_order) build_order(o, order_key, order_flags, need_inv);
    over_aggs(o, order_key != nullptr, ops, vals, outs);
    const OverOrder* order = need_order ? &o : nullptr;
    for (size_t i = 0; i < ops.size(); i++) {
        const int kind = ops[i].kind & 0xFFFF;
        if (is_agg(kind)) continue;
        const DevCol& v = vals[i];
        if (kind == BL_SHIFT) { outs[i] = over_shift(v, order, ops[i].periods); continue; }
        if (kind == BL_CUM_COUNT) {      // reads the validity only
            DevCol w = v; w.values.reset(); w.dtype = BL_BOOL;
            outs[i] = over_cum(kind, w, BL_BOOL, order, ops[i].reverse);
            continue;
        }
        // the reference casts before it scans: SUM Int8/16 / UInt8/16 -> Int64, PROD Int8..UInt32 -> Int64 (cum_agg.rs:268-321;
        // Int32 / UInt32 products are widened as they are loaded).  MIN / MAX keep the dtype: small integers are scanned as
        // their Int64 value and narrowed back.
        const bool small = dtype_is_small_int(v.dtype);
        const DevCol w = small ? op_cast_small_int(v, BL_INT64, false) : v;
        DevCol r = over_cum(kind, w, (kind == BL_CUM_MIN || kind == BL_CUM_MAX) ? w.dtype : v.dtype, order, ops[i].reverse);
        if (small && (kind == BL_CUM_MIN || kind == BL_CUM_MAX)) r = op_cast_small_int(r, v.dtype, false);
        outs[i] = r;
    }
    return outs;
}

static int64_t key_length(const bl_sort_key& k) {
    if (k.column) return k.column->length;
    int64_t n = 0;
    for (int j = 0; j < k.n_chunks; j++) n += k.strings[j].length;
    return n;
}

DevCol import_key(const bl_sort_key& k, bool partition) {
    if (k.column) return import_column(k.column, 1);
    DevStr s = import_string(k.strings, k.n_chunks);
    return partition ? op_string_codes(s, nullptr) : op_string_rank(s, false, nullptr);
}

void set_window_len(const char* who, int64_t len, const std::string& what, int64_t& n) {
    if (n < 0) n = len;
    PLB_REQUIRE(len == n, BL_ERR_INVALID, std::string(who) + ": " + what + " has " + std::to_string(len) + " rows, not " + std::to_string(n));
}

void check_window_keys(const char* who, const bl_sort_key* partition_by, int32_t n_partition_by, const bl_sort_key* order_by, int64_t& n) {
    const std::string w0 = who;
    PLB_REQUIRE(n_partition_by >= 0 && (n_partition_by == 0 || partition_by), BL_ERR_INVALID, w0 + ": n_partition_by > 0 needs partition_by");
    auto check_key = [&](const bl_sort_key& k, const std::string& w) {
        PLB_REQUIRE((k.column != nullptr) != (k.strings != nullptr), BL_ERR_INVALID, w + " must set exactly one of `column` and `strings`");
        PLB_REQUIRE(k.strings == nullptr || k.n_chunks >= 1, BL_ERR_INVALID, w + ": a string column without chunks");
        set_window_len(who, key_length(k), w, n);
    };
    for (int i = 0; i < n_partition_by; i++) {
        const std::string w = "partition column " + std::to_string(i);
        check_key(partition_by[i], w);
        PLB_REQUIRE(partition_by[i].flags == 0, BL_ERR_INVALID, w0 + ": " + w + ": flags must be 0");
        if (partition_by[i].column) PLB_REQUIRE(partition_by[i].column->dtype != BL_BOOL, BL_ERR_UNSUPPORTED, w0 + ": Boolean partition columns are outside the hot path");
    }
    if (order_by) {
        check_key(*order_by, "the order_by column");
        PLB_REQUIRE((order_by->flags & ~(BL_SORT_DESCENDING | BL_SORT_NULLS_LAST)) == 0, BL_ERR_INVALID, w0 + ": unknown order_by flags");
    }
}

}  // namespace plb

// ================================================================================ C ABI
using namespace plb;
extern "C" {

bl_status bl_over(const bl_sort_key* partition_by, int32_t n_partition_by, const bl_sort_key* order_by, const bl_over_op* ops, int32_t n_ops,
                  int32_t out_location, bl_column* outs) {
    BL_TRY
    PLB_REQUIRE(n_ops >= 1 && ops && outs, BL_ERR_INVALID, "over: no operations or no outputs");
    int64_t n = -1;
    check_window_keys("over", partition_by, n_partition_by, order_by, n);
    for (int i = 0; i < n_ops; i++) {
        if (ops[i].values) set_window_len("over", ops[i].values->length, "value column " + std::to_string(i), n);
        else PLB_REQUIRE((ops[i].kind & 0xFFFF) == BL_AGG_LEN, BL_ERR_INVALID, "over: operation " + std::to_string(i) + " has no value column");
    }
    PLB_REQUIRE(n >= 0, BL_ERR_INVALID, "over: no column gives the number of rows");
    std::vector<DevCol> parts;
    for (int i = 0; i < n_partition_by; i++) parts.push_back(import_key(partition_by[i], true));
    DevCol okey;
    if (order_by) okey = import_key(*order_by, false);
    std::vector<DevCol> vals(n_ops);
    std::vector<OverOp> v(n_ops);
    for (int i = 0; i < n_ops; i++) {
        v[i].kind = ops[i].kind; v[i].reverse = ops[i].reverse != 0; v[i].periods = ops[i].periods; v[i].param = ops[i].param;
        check_over_op(ops[i].kind, ops[i].values ? ops[i].values->dtype : -1);
    }
    for (int i = 0; i < n_ops; i++) {
        if (ops[i].values) { vals[i] = import_column(ops[i].values, 1); v[i].values = &vals[i]; }
    }
    std::vector<DevCol> res = op_over(parts, order_by ? &okey : nullptr, order_by ? order_by->flags : 0, v, n);
    export_many(res, out_location, outs);
    BL_CATCH
}

}  // extern "C"
