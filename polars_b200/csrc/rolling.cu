// rolling.cu — fixed-window rolling aggregations `expr.rolling_*(window_size, min_samples, center)` and their
// `.over(partition_by, order_by=...)` form, one output row per input row (polars-compute/src/rolling).
//
// Plans (DESIGN.md §13), chosen from B = min(w, n): B <= RT_MAX_B runs k_roll_tile, one pass with the tile and its halo in
// shared memory; larger B runs the three-pass plan below through HBM.  Positions are the rows themselves (whole column) or
// bl_over's partition order (`perm`, segments = partitions).  The positions are cut into blocks of B (van Herk /
// Gil-Werman); in the three-pass plan k_roll_scan writes, for every
// position, the reduction of its block from the block start (prefix, restarted at a segment head) and to the block end
// (suffix, restarted at a segment end).  A window holds at most B positions, so it lies in one block or in two adjacent ones
// and k_roll_out reads it as suffix[start] (+) prefix[last], or one of the two alone (see k_roll_out).  Every operator is
// associative, so MIN / MAX, integer SUM, the counts and the non-finite counters are exact; float sums and the variance
// state are reassociated (the header's bound).  Deterministic mode replays the reference's state machines instead
// (k_roll_fold_sum / k_roll_fold_var, one thread per partition).
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

// ---------------------------------------------------------------------------------------------------- finishers
struct RollArgs {
    const void* values; const uint32_t* validity;
    const uint32_t* perm; const uint32_t* seg; const uint32_t* offsets; int64_t G;      // partition order (NULL: the rows, one segment)
    int64_t n, L, R; uint32_t B;      // window [i - L, i + R) clipped to the segment; block size
    int64_t min_samples; int ddof;
    void* pre; void* suf; void* out; uint32_t* out_valid;
};
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
                if (a.validity == nullptr || bit_get(a.validity, row)) v[k] = St::lift(load_in<In>(a.values, row));
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

// ---------------------------------------------------------------------------------------------------- k_roll_out
// Position i of segment [lo, hi) (found by binary search in offsets; none: [0, n)) has the window [s, l], s = max(i - L, lo),
// l = min(i + R, hi) - 1, at most B positions.  With b = the start of l's block:
//   s < b               the window spans two blocks: suffix[s] (+) prefix[l] (no segment boundary lies inside it)
//   s == max(b, lo)     prefix[l] (the prefix of l starts at its block start or at a later segment head, which is then s)
//   otherwise           the window was clipped at the segment end: l = hi - 1 and suffix[s] ends there
// The output goes to row perm[i] (the row itself without an order); validity: whole words by ballot over the rows, or
// atomicOr into a zeroed bitmap through perm.
// The window state of position i; pre / suf hold the positions from `base` on (global memory: 0; a staged tile: its start).
template <class St>
__device__ __forceinline__ typename St::S window_state(const RollArgs& a, int64_t i, const typename St::S* pre, const typename St::S* suf, int64_t base) {
    int64_t lo = 0, hi = a.n;
    if (a.offsets) {
        int64_t gl = 0, gh = a.G;      // offsets[gl] <= i < offsets[gh]
        while (gh - gl > 1) {
            const int64_t m = (gl + gh) >> 1;
            if ((int64_t)__ldg(a.offsets + m) <= i) gl = m; else gh = m;
        }
        lo = __ldg(a.offsets + gl); hi = __ldg(a.offsets + gl + 1);
    }
    const int64_t s = max(i - a.L, lo), l = min(i + a.R, hi) - 1;
    const int64_t b = l - (int64_t)((uint32_t)l % a.B);
    if (s < b) return St::combine(suf[s - base], pre[l - base]);
    return s == max(b, lo) ? pre[l - base] : suf[s - base];
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

template <class St, class Fin>
__global__ void __launch_bounds__(256) k_roll_out(const __grid_constant__ RollArgs a) {
    using S = typename St::S;
    using Out = typename Fin::out_t;
    const S* pre = reinterpret_cast<const S*>(a.pre);
    const S* suf = reinterpret_cast<const S*>(a.suf);
    const int64_t n_round = (a.n + 31) / 32 * 32;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_round; i += (int64_t)gridDim.x * blockDim.x) {
        bool ok = false;
        Out x = Out(0);
        if (i < a.n) ok = Fin::fin(window_state<St>(a, i, pre, suf, 0), a, x);
        write_out<Fin>(a, i, i < a.n, ok, x);
    }
}

// ---------------------------------------------------------------------------------------------------- k_roll_tile
// The small-window plan (B <= RT_MAX_B): one pass, no state in HBM.  A CTA owns the outputs [o0, o0 + RT_TILE) and stages
// the positions [first block start <= o0 - L, last block end >= o0 + RT_TILE - 2 + R) -- the tile plus its halo, at most
// RT_TILE + 3 B positions -- as lifted states in shared memory.  One thread per block then forms that block's suffixes
// (restarted at segment ends) and prefixes in place (restarted at segment heads), and every output reads its window as
// k_roll_out does.  The blocks are aligned at multiples of B from position 0, as in the three-pass plan.
constexpr int RT_THREADS = 256, RT_TILE = 1024, RT_MAX_B = 128, RT_CAP = RT_TILE + 3 * RT_MAX_B;

template <class St> constexpr size_t tile_smem() { return (size_t)RT_CAP * (2 * sizeof(typename St::S) + 4); }

template <class St, typename In, class Fin>
__global__ void __launch_bounds__(RT_THREADS) k_roll_tile(const __grid_constant__ RollArgs a) {
    using S = typename St::S;
    using Out = typename Fin::out_t;
    extern __shared__ __align__(16) unsigned char rt_smem[];
    S* P = reinterpret_cast<S*>(rt_smem);
    S* Q = P + RT_CAP;
    uint32_t* sg = reinterpret_cast<uint32_t*>(Q + RT_CAP);
    const int64_t B = a.B;
    const int64_t o0 = (int64_t)blockIdx.x * RT_TILE, o1 = min(a.n, o0 + RT_TILE);
    const int64_t A = max(o0 - a.L, (int64_t)0) / B * B;
    const int64_t last = min(a.n - 1, o1 - 2 + a.R);
    const int len = (int)(min(a.n, (last / B + 1) * B) - A);
    for (int j = threadIdx.x; j < len; j += RT_THREADS) {
        const int64_t p = A + j;
        const int64_t row = a.perm ? (int64_t)__ldg(a.perm + p) : p;
        P[j] = (a.validity == nullptr || bit_get(a.validity, row)) ? St::lift(load_in<In>(a.values, row)) : St::empty();
        if (a.seg) sg[j] = __ldg(a.seg + p);
    }
    __syncthreads();
    const int nb = (len + (int)B - 1) / (int)B;
    for (int k = threadIdx.x; k < nb; k += RT_THREADS) {
        const int b0 = k * (int)B, b1 = min(len, b0 + (int)B);
        Q[b1 - 1] = P[b1 - 1];
        for (int j = b1 - 2; j >= b0; j--) Q[j] = (a.seg && sg[j] != sg[j + 1]) ? P[j] : St::combine(P[j], Q[j + 1]);
        for (int j = b0 + 1; j < b1; j++)
            if (!(a.seg && sg[j] != sg[j - 1])) P[j] = St::combine(P[j - 1], P[j]);
    }
    __syncthreads();
    for (int64_t i = o0 + threadIdx.x; i < o0 + RT_TILE; i += RT_THREADS) {      // whole warps: the ballot needs every lane
        bool ok = false;
        Out x = Out(0);
        if (i < a.n) ok = Fin::fin(window_state<St>(a, i, P, Q, A), a, x);
        write_out<Fin>(a, i, i < a.n, ok, x);
    }
}

// ---------------------------------------------------------------------------------------------------- deterministic mode
// One thread replays one segment in the reference's order: rolling_apply_agg_window (nulls/mod.rs:46-98) calls
// update(start, end) for every position; both window types reset when the new start is at or past the old end.
__device__ __forceinline__ void seg_bounds(const RollArgs& a, int64_t g, int64_t& lo, int64_t& hi) {
    if (a.offsets) { lo = a.offsets[g]; hi = a.offsets[g + 1]; } else { lo = 0; hi = a.n; }
}
__device__ __forceinline__ void set_valid(uint32_t* bm, int64_t row) { atomicOr(bm + (row >> 5), 1u << (row & 31)); }

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
            const int64_t s = max(i - a.L, lo), e = min(i + a.R, hi);
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
            const int64_t s = max(i - a.L, lo), e = min(i + a.R, hi);
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

// ---------------------------------------------------------------------------------------------------- host side
static bool is_rolling(int kind) { return kind >= BL_ROLLING_SUM && kind <= BL_ROLLING_STD; }

int rolling_dtype(int kind, int dt) {
    switch (kind) {
        case BL_ROLLING_SUM:
            if (dt == BL_BOOL) return BL_UINT32;
            return dtype_is_small_int(dt) ? BL_INT64 : dt;
        case BL_ROLLING_MIN: case BL_ROLLING_MAX: return dt;
        default: return dt == BL_FLOAT32 ? BL_FLOAT32 : BL_FLOAT64;      // MEAN / VAR / STD
    }
}

void check_rolling_op(int kind, int center, int64_t window_size, int64_t min_samples, int ddof, int reserved, int value_dtype) {
    PLB_REQUIRE(is_rolling(kind), BL_ERR_INVALID, "rolling: unknown kind " + std::to_string(kind));
    PLB_REQUIRE(value_dtype >= 0, BL_ERR_INVALID, "rolling: an operation without a value column");
    PLB_REQUIRE(value_dtype <= BL_BOOL, BL_ERR_INVALID, "rolling: unknown value dtype");
    PLB_REQUIRE(reserved == 0, BL_ERR_INVALID, "rolling: reserved must be 0");
    PLB_REQUIRE(center == 0 || center == 1, BL_ERR_INVALID, "rolling: center must be 0 or 1");
    PLB_REQUIRE(window_size >= 0 && min_samples >= 0, BL_ERR_INVALID, "rolling: window_size and min_samples must not be negative");
    PLB_REQUIRE(min_samples <= window_size, BL_ERR_INVALID, "rolling: min_samples (" + std::to_string(min_samples) + ") must be <= window_size (" + std::to_string(window_size) + ")");
    PLB_REQUIRE(ddof >= 0 && ddof <= 255, BL_ERR_INVALID, "rolling: ddof must be in 0..255");
    PLB_REQUIRE(window_size > 0, BL_ERR_UNSUPPORTED, "rolling: window_size 0 is outside the hot path");
    PLB_REQUIRE(value_dtype != BL_BOOL || kind == BL_ROLLING_SUM, BL_ERR_UNSUPPORTED, "rolling: a Boolean column takes only rolling_sum on the device");
}

// B <= RT_MAX_B: k_roll_tile (one pass); larger blocks: the three-pass plan through HBM
template <class St, typename In, class Fin> static void run_parallel(RollArgs a) {
    using S = typename St::S;
    if (a.B <= (uint32_t)RT_MAX_B) {
        static bool attr = false;      // the opt-in above 48 KB of dynamic shared memory, once per instantiation
        if (!attr) { PLB_CUDA(cudaFuncSetAttribute(k_roll_tile<St, In, Fin>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)tile_smem<St>())); attr = true; }
        PLB_LAUNCH("rolling_tile", (k_roll_tile<St, In, Fin>), (int)((a.n + RT_TILE - 1) / RT_TILE), RT_THREADS, tile_smem<St>(), a);
        return;
    }
    DevPtr pre = dev_alloc((size_t)a.n * sizeof(S)), suf = dev_alloc((size_t)a.n * sizeof(S));
    a.pre = pre->p; a.suf = suf->p;
    const int64_t span = (int64_t)a.B * std::max<int64_t>(1, RS_TILE / a.B);
    const int64_t ctas = (a.n + span - 1) / span;
    PLB_LAUNCH("rolling_prefix", (k_roll_scan<St, In, false>), (int)ctas, RS_THREADS, 0, a, span);
    PLB_LAUNCH("rolling_suffix", (k_roll_scan<St, In, true>), (int)ctas, RS_THREADS, 0, a, span);
    PLB_LAUNCH("rolling_out", (k_roll_out<St, Fin>), grid_for((a.n + 31) / 32 * 32, 256), 256, 0, a);
}

template <typename In, typename T, typename K, bool MEAN> static void run_fold_sum(const RollArgs& a) {
    PLB_LAUNCH("rolling_fold", (k_roll_fold_sum<In, T, K, MEAN>), grid_for(a.G, 64, 32), 64, 0, a);
}
template <typename In, typename Out, bool STD> static void run_fold_var(const RollArgs& a) {
    DevPtr front = dev_alloc((size_t)a.n * sizeof(VarSt::S)), back = dev_alloc((size_t)a.n * 8);
    PLB_LAUNCH("rolling_fold", (k_roll_fold_var<In, Out, STD>), grid_for(a.G, 64, 32), 64, 0, a, as<VarSt::S>(front), as<double>(back));
}

// one parallel plan per (kind, loaded type); In: the value type after small integers were widened to Int64
template <typename In, typename Out> static void dispatch_float_kinds(int kind, const RollArgs& a, bool det) {
    constexpr bool in_f32 = std::is_same<In, float>::value;
    using TM = typename std::conditional<in_f32, float, double>::type;      // the reference's value type after to_float
    switch (kind) {
        case BL_ROLLING_MEAN:
            if (det) run_fold_sum<In, TM, double, true>(a);
            else run_parallel<SumFltSt, In, FinMean<Out>>(a);
            break;
        case BL_ROLLING_VAR:
            if (det) run_fold_var<In, Out, false>(a);
            else run_parallel<VarSt, In, FinVar<Out, false>>(a);
            break;
        default:
            if (det) run_fold_var<In, Out, true>(a);
            else run_parallel<VarSt, In, FinVar<Out, true>>(a);
            break;
    }
}
template <typename T> static void dispatch_minmax(int kind, const RollArgs& a) {
    if (kind == BL_ROLLING_MIN) run_parallel<MinMaxSt<T, false>, T, FinMinMaxT<T>>(a);
    else run_parallel<MinMaxSt<T, true>, T, FinMinMaxT<T>>(a);
}

static DevCol rolling_one(const RollOp& op, const DevCol& v, const OverOrder* o) {
    const int64_t n = v.len;
    const int kind = op.kind;
    DevCol out = make_col(rolling_dtype(kind, v.dtype), n, true);
    out.null_count = -1;
    if (n == 0) return out;
    const bool det = ctx().deterministic && (kind != BL_ROLLING_SUM || dtype_is_float(v.dtype)) && kind != BL_ROLLING_MIN && kind != BL_ROLLING_MAX;
    RollArgs a;
    memset(&a, 0, sizeof a);
    a.values = v.v(); a.validity = v.vm(); a.n = n;
    if (o) { a.perm = as<uint32_t>(o->perm.values); a.seg = as<uint32_t>(o->seg.values); a.offsets = as<uint32_t>(o->offsets.values); a.G = o->G; }
    else a.G = 1;
    const int64_t w = op.window_size;
    int64_t L = w - 1, R = 1;
    if (op.center) { R = w / 2 + (w & 1); L = w - R; }
    a.L = std::min(L, n); a.R = std::min(R, n);
    a.B = (uint32_t)std::min(w, n);
    a.min_samples = op.min_samples; a.ddof = op.ddof;
    a.out = out.values->p; a.out_valid = as<uint32_t>(out.validity);
    if (o || det) dev_memset(a.out_valid, 0, bitmap_bytes(n));
    const int dt = v.dtype;
    switch (kind) {
        case BL_ROLLING_SUM:
            switch (dt) {
                case BL_BOOL: run_parallel<SumIntSt<uint32_t>, BoolBit, FinSumInt<uint32_t>>(a); break;
                case BL_INT32: case BL_UINT32: run_parallel<SumIntSt<uint32_t>, uint32_t, FinSumInt<uint32_t>>(a); break;
                case BL_INT64: case BL_UINT64: run_parallel<SumIntSt<uint64_t>, uint64_t, FinSumInt<uint64_t>>(a); break;
                case BL_FLOAT32: if (det) run_fold_sum<float, float, float, false>(a); else run_parallel<SumFltSt, float, FinSumFlt<float>>(a); break;
                default: if (det) run_fold_sum<double, double, double, false>(a); else run_parallel<SumFltSt, double, FinSumFlt<double>>(a); break;
            }
            break;
        case BL_ROLLING_MIN: case BL_ROLLING_MAX:
            switch (dt) {
                case BL_INT32: dispatch_minmax<int32_t>(kind, a); break;
                case BL_UINT32: dispatch_minmax<uint32_t>(kind, a); break;
                case BL_INT64: dispatch_minmax<int64_t>(kind, a); break;
                case BL_UINT64: dispatch_minmax<uint64_t>(kind, a); break;
                case BL_FLOAT32: dispatch_minmax<float>(kind, a); break;
                default: dispatch_minmax<double>(kind, a); break;
            }
            break;
        default:      // MEAN / VAR / STD
            switch (dt) {
                case BL_INT32: dispatch_float_kinds<int32_t, double>(kind, a, det); break;
                case BL_UINT32: dispatch_float_kinds<uint32_t, double>(kind, a, det); break;
                case BL_INT64: dispatch_float_kinds<int64_t, double>(kind, a, det); break;
                case BL_UINT64: dispatch_float_kinds<uint64_t, double>(kind, a, det); break;
                case BL_FLOAT32: dispatch_float_kinds<float, float>(kind, a, det); break;
                default: dispatch_float_kinds<double, double>(kind, a, det); break;
            }
            break;
    }
    return out;
}

// ops are checked by the caller (check_rolling_op) before any column is uploaded
std::vector<DevCol> op_rolling(const std::vector<DevCol>& partition_by, const DevCol* order_key, int order_flags, const std::vector<RollOp>& ops, int64_t n) {
    for (auto& op : ops) PLB_REQUIRE(op.values && op.values->len == n, BL_ERR_INVALID, "rolling: value columns differ in length");
    for (auto& k : partition_by) PLB_REQUIRE(k.len == n, BL_ERR_INVALID, "rolling: partition columns differ in length");
    if (order_key) PLB_REQUIRE(order_key->len == n, BL_ERR_INVALID, "rolling: the order_by column differs in length");
    const bool need_order = !partition_by.empty() || order_key;
    PLB_REQUIRE(!need_order || n <= 0x7FFFFFFFll, BL_ERR_UNSUPPORTED, "rolling: more than 2^31 - 1 rows need a sort (group tuples)");
    PLB_REQUIRE(n <= 0xFFFFFFFFll, BL_ERR_UNSUPPORTED, "rolling: more than 2^32 - 1 rows (IdxSize is u32)");
    OverOrder o;
    if (need_order && n > 0) {
        o.gid = partition_ids(partition_by, n);
        build_order(o, order_key, order_flags, false);
    }
    std::vector<DevCol> outs;
    for (auto& op : ops) {
        // the reference casts before it rolls: SUM Int8/16 / UInt8/16 -> Int64, MEAN / VAR / STD -> Float64 (exact from Int64);
        // MIN / MAX keep the dtype: small integers roll as their Int64 value and are narrowed back
        const DevCol& v = *op.values;
        const bool small = dtype_is_small_int(v.dtype);
        const DevCol w = small ? op_cast_small_int(v, BL_INT64, false) : v;
        DevCol r = rolling_one(op, w, need_order && n > 0 ? &o : nullptr);
        if (small && (op.kind == BL_ROLLING_MIN || op.kind == BL_ROLLING_MAX)) r = op_cast_small_int(r, v.dtype, false);
        outs.push_back(r);
    }
    return outs;
}

}  // namespace plb

// ================================================================================ C ABI
using namespace plb;
extern "C" {

bl_status bl_rolling(const bl_sort_key* partition_by, int32_t n_partition_by, const bl_sort_key* order_by, const bl_rolling_op* ops, int32_t n_ops,
                     int32_t out_location, bl_column* outs) {
    BL_TRY
    PLB_REQUIRE(n_ops >= 1 && ops && outs, BL_ERR_INVALID, "rolling: no operations or no outputs");
    int64_t n = -1;
    check_window_keys("rolling", partition_by, n_partition_by, order_by, n);
    for (int i = 0; i < n_ops; i++) {
        PLB_REQUIRE(ops[i].values != nullptr, BL_ERR_INVALID, "rolling: operation " + std::to_string(i) + " has no value column");
        check_rolling_op(ops[i].kind, ops[i].center, ops[i].window_size, ops[i].min_samples, ops[i].ddof, ops[i].reserved, ops[i].values->dtype);
        set_window_len("rolling", ops[i].values->length, "value column " + std::to_string(i), n);
    }
    std::vector<DevCol> parts;
    for (int i = 0; i < n_partition_by; i++) parts.push_back(import_key(partition_by[i], true));
    DevCol okey;
    if (order_by) okey = import_key(*order_by, false);
    std::vector<DevCol> vals(n_ops);
    std::vector<RollOp> v(n_ops);
    for (int i = 0; i < n_ops; i++) {
        vals[i] = import_column(ops[i].values, 1);
        v[i].kind = ops[i].kind; v[i].center = ops[i].center != 0; v[i].window_size = ops[i].window_size; v[i].min_samples = ops[i].min_samples;
        v[i].ddof = ops[i].ddof; v[i].values = &vals[i];
    }
    std::vector<DevCol> res = op_rolling(parts, order_by ? &okey : nullptr, order_by ? order_by->flags : 0, v, n);
    export_many(res, out_location, outs);
    BL_CATCH
}

}  // extern "C"
