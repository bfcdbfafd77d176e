// rolling_by.cu — time-based rolling aggregations `expr.rolling_*_by(by, window_size, min_samples, closed)` and their
// `.over(partition_by)` form, one output row per input row (polars-time/src/chunkedarray/rolling_window/dispatch.rs:71-580).
//
// The window of a row is every row of its partition whose time lies in (t - P, t] (or the other `closed` forms), so its
// width varies from row to row, from empty to the whole partition (DESIGN.md §14).  Positions are the rows (no partition,
// `by` non-null and ascending) or bl_over's partition order with `by` as the order key, nulls last (segments = partitions,
// the null-`by` positions at each segment's tail belong to no window).  k_rollby_bounds writes each position's window
// [ws, we) by binary search.  The positions are cut into blocks of RB_B = 1024; k_roll_scan writes per-position prefix /
// suffix states inside each block (restarted at segment heads / ends) and a disjoint sparse table over the block totals
// (one prefix / suffix scan of the totals per level) answers any run of whole blocks with two states.  k_rollby_out then
// reduces a window that crosses blocks as suffix[s] (+) table(middle blocks) (+) prefix[e - 1]; a window inside the CTA's
// own block from the same structure one level down, staged in shared memory (32-position sub-blocks, a 5-level table over
// their totals).  Deterministic mode replays the reference's window machines over [ws, we) (k_roll_fold_sum / _var).
#include "rolling.cuh"

namespace plb {

constexpr int RB_B = 1024, RB_THREADS = 256, RB_SUB = 32, RB_NSUB = RB_B / RB_SUB, RB_LVL = 5;

// the Int64 time of row r (the reference casts Int32 / UInt32 / UInt64 `by` columns to Int64, dispatch.rs:163-175)
__device__ __forceinline__ int64_t load_time(const void* by, int dt, int64_t r) {
    if (dt == BL_INT32) return __ldg(reinterpret_cast<const int32_t*>(by) + r);
    if (dt == BL_UINT32) return __ldg(reinterpret_cast<const uint32_t*>(by) + r);
    return __ldg(reinterpret_cast<const int64_t*>(by) + r);
}

// ---------------------------------------------------------------------------------------------------- k_rollby_check
// stats[0] += null `by` rows, stats[1] += adjacent non-null pairs out of ascending order, stats[2] += UInt64 values >= 2^63
__global__ void k_rollby_check(const void* by, const uint32_t* valid, int dt, int64_t n, unsigned long long* stats) {
    unsigned long long nulls = 0, desc = 0, big = 0;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        if (valid && !bit_get(valid, i)) { nulls++; continue; }
        const int64_t t = load_time(by, dt, i);
        if (dt == BL_UINT64 && t < 0) big++;
        if (i > 0 && (!valid || bit_get(valid, i - 1))) {
            const int64_t u = load_time(by, dt, i - 1);
            desc += dt == BL_UINT64 ? ((uint64_t)t < (uint64_t)u) : (t < u);
        }
    }
    for (int o = 16; o; o >>= 1) {
        nulls += __shfl_xor_sync(0xffffffffu, nulls, o);
        desc += __shfl_xor_sync(0xffffffffu, desc, o);
        big += __shfl_xor_sync(0xffffffffu, big, o);
    }
    if (lane_id() == 0 && (nulls | desc | big)) {
        atomicAdd(stats, nulls); atomicAdd(stats + 1, desc); atomicAdd(stats + 2, big);
    }
}

// ---------------------------------------------------------------------------------------------------- k_rollby_bounds
struct BoundsArgs {
    const void* by; const uint32_t* by_valid; int dt;
    const uint32_t* perm; const uint32_t* offsets; int64_t G, n;
    int64_t P; int closed;
    uint32_t* ws; uint32_t* we; unsigned long long* wmax;      // wmax: the largest e - s
};

// group_by_values_iter_lookbehind (polars-time/src/windows/group_by.rs:247-326) in closed form, for position p of segment
// [lo, hi) at time t (times ascend in a segment; null times sit at its tail and count as +inf below):
//   s = the first q <= p that enters (t_q > t - P, or >= for left / both; Bounds::is_member_entry, bounds.rs:33-60)
//   e = the end of p's run of equal times (right / both) or its start (left / none: t itself is not a member)
// t - P wraps like the reference's i64 arithmetic (Duration::add_ns / add_us / add_ms).  A wrapped lower bound is above every
// time, so the iterator's scan restarts at p's run and its start never moves back past the last such run: s is at least
// the head of the last run of times below i64::MIN + P.
__global__ void __launch_bounds__(256) k_rollby_bounds(const __grid_constant__ BoundsArgs a) {
    unsigned long long w = 0;
    for (int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; p < a.n; p += (int64_t)gridDim.x * blockDim.x) {
        const int64_t row = a.perm ? (int64_t)__ldg(a.perm + p) : p;
        if (a.by_valid && !bit_get(a.by_valid, row)) { a.ws[p] = BY_NULL; a.we[p] = BY_NULL; continue; }
        int64_t lo = 0, hi = a.n;
        if (a.offsets) {
            int64_t gl = 0, gh = a.G;
            while (gh - gl > 1) {
                const int64_t m = (gl + gh) >> 1;
                if ((int64_t)__ldg(a.offsets + m) <= p) gl = m; else gh = m;
            }
            lo = __ldg(a.offsets + gl); hi = __ldg(a.offsets + gl + 1);
        }
        struct Time { int64_t t; bool null; };      // a null time counts as +inf
        auto time_at = [&](int64_t q) {
            const int64_t r = a.perm ? (int64_t)__ldg(a.perm + q) : q;
            if (a.by_valid && !bit_get(a.by_valid, r)) return Time{0, true};
            return Time{load_time(a.by, a.dt, r), false};
        };
        // the first q in [l, h) whose time is >= x (strict: > x), h if none
        auto first = [&](int64_t l, int64_t h, int64_t x, bool strict) {
            while (l < h) {
                const int64_t m = (l + h) >> 1;
                const Time u = time_at(m);
                if (u.null || (strict ? u.t > x : u.t >= x)) h = m; else l = m + 1;
            }
            return l;
        };
        const int64_t t = time_at(p).t;
        const int64_t lb = (int64_t)((uint64_t)t - (uint64_t)a.P);
        const bool incl = a.closed == BL_CLOSED_LEFT || a.closed == BL_CLOSED_BOTH;
        const int64_t thr = INT64_MIN + a.P;      // times below wrap
        int64_t s;
        if (t < thr) s = first(lo, p + 1, t, false);
        else {
            s = first(lo, p + 1, lb, !incl);
            if (time_at(lo).t < thr) {
                const int64_t x = first(lo, p, thr, false);
                s = max(s, first(lo, x, time_at(x - 1).t, false));
            }
        }
        const int64_t e = (a.closed == BL_CLOSED_RIGHT || a.closed == BL_CLOSED_BOTH) ? first(p + 1, hi, t, true) : first(lo, p + 1, t, false);
        a.ws[p] = (uint32_t)s; a.we[p] = (uint32_t)e;
        w = max(w, (unsigned long long)(e - s));
    }
    for (int o = 16; o; o >>= 1) w = max(w, __shfl_xor_sync(0xffffffffu, w, o));
    if (lane_id() == 0 && w) atomicMax(a.wmax, w);
}

// ---------------------------------------------------------------------------------------------------- the block totals
template <class S> __global__ void k_rollby_totals(const S* suf, int64_t nb, S* tot) {
    for (int64_t b = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; b < nb; b += (int64_t)gridDim.x * blockDim.x) tot[b] = suf[b * RB_B];
}

// ---------------------------------------------------------------------------------------------------- k_rollby_out
struct ByOut { const void* gpre; const void* gsuf; int64_t nb; };      // the sparse table: level k's prefix / suffix states at k * nb

// the reduction of the lifted values of positions [s, e) in order, from global memory
template <class St, typename In> __device__ typename St::S fold_global(const RollArgs& a, int64_t s, int64_t e) {
    typename St::S st = St::empty();
    for (int64_t q = s; q < e; q++) {
        const int64_t row = a.perm ? (int64_t)__ldg(a.perm + q) : q;
        if (a.validity == nullptr || bit_get(a.validity, row)) st = St::combine(st, St::lift(load_in<In>(a.values, row)));
    }
    return st;
}

// The window [s, e) (non-empty, inside one segment) from the states in global memory.  Blocks bs < be: suffix[s], the
// blocks between from the table, prefix[e - 1].  One block: prefix[e - 1] when s is its block start or segment head (the
// prefix starts there), suffix[s] when e is its block end or segment end, else a fold of at most RB_B - 2 values -- only a
// left / none window behind its row's own block gets here (a run of equal times longer than the rest of the block).
template <class St, typename In>
__device__ typename St::S window_global(const RollArgs& a, const ByOut& t, int64_t s, int64_t e) {
    using S = typename St::S;
    const S* pre = reinterpret_cast<const S*>(a.pre);
    const S* suf = reinterpret_cast<const S*>(a.suf);
    const int64_t bs = s / RB_B, be = (e - 1) / RB_B;
    if (bs < be) {
        S st = suf[s];
        if (be - bs > 1) {
            const int64_t l = bs + 1, r = be - 1;
            const S* gp = reinterpret_cast<const S*>(t.gpre);
            const S* gs = reinterpret_cast<const S*>(t.gsuf);
            if (l == r) st = St::combine(st, gs[l]);
            else {
                const int k = 63 - __clzll((unsigned long long)(l ^ r));
                st = St::combine(St::combine(st, gs[k * t.nb + l]), gp[k * t.nb + r]);
            }
        }
        return St::combine(st, pre[e - 1]);
    }
    if (s % RB_B == 0 || (a.seg && __ldg(a.seg + s - 1) != __ldg(a.seg + s))) return pre[e - 1];
    if (e % RB_B == 0 || e == a.n || (a.seg && __ldg(a.seg + e) != __ldg(a.seg + e - 1))) return suf[s];
    return fold_global<St, In>(a, s, e);
}

// The staged tile of k_rollby_out: the general plan stages its own block of RB_B positions; the small-window plan (every
// window at most RB_HALO wide) stages the outputs' positions plus RB_HALO on each side, which holds every window except a
// left / none one behind a run of equal times longer than RB_HALO.
constexpr int RB_HALO = 128;
template <bool TILE> struct Stage {
    static constexpr int CAP = TILE ? RB_B + 2 * RB_HALO : RB_B, NSUB = CAP / RB_SUB, LVL = TILE ? 6 : 5;      // 2^LVL >= NSUB
};
template <class St, bool TILE> constexpr size_t out_smem() {
    using G = Stage<TILE>;
    return (size_t)(3 * G::CAP + 2 * G::LVL * G::NSUB) * sizeof(typename St::S) + G::CAP * 4;
}

// One CTA per RB_B outputs.  It stages the lifted states L of its positions [A, A + len) and forms, per 32-position
// sub-block, prefixes P (restarted at segment heads) and suffixes Q (restarted at segment ends), then a disjoint sparse table
// over the sub-block totals (TP / TS: level k's prefix / suffix inside groups of 2^k sub-blocks).  A window inside the stage
// is Q[l] (+) table (+) P[r] across sub-blocks; inside one sub-block P[r] or Q[l] when it touches the sub-block's or the
// segment's edge, else a fold of at most 30 states of L.  Other windows read global memory: the general plan's states and
// table (window_global), or in the small-window plan a fold of at most RB_HALO values (fold_global).
template <class St, typename In, class Fin, bool TILE>
__global__ void __launch_bounds__(RB_THREADS) k_rollby_out(const __grid_constant__ RollArgs a, const __grid_constant__ ByOut t) {
    using S = typename St::S;
    using Out = typename Fin::out_t;
    using G = Stage<TILE>;
    extern __shared__ __align__(16) unsigned char rb_smem[];
    S* L = reinterpret_cast<S*>(rb_smem);
    S* P = L + G::CAP;
    S* Q = P + G::CAP;
    S* TP = Q + G::CAP;
    S* TS = TP + G::LVL * G::NSUB;
    uint32_t* sg = reinterpret_cast<uint32_t*>(TS + G::LVL * G::NSUB);
    const int64_t o0 = (int64_t)blockIdx.x * RB_B;
    const int64_t A = TILE ? max((int64_t)0, o0 - RB_HALO) : o0;
    const int len = (int)(min(a.n, TILE ? o0 + RB_B + RB_HALO : o0 + RB_B) - A);
    for (int j = threadIdx.x; j < G::CAP; j += RB_THREADS) {
        S v = St::empty();
        if (j < len) {
            const int64_t row = a.perm ? (int64_t)__ldg(a.perm + A + j) : A + j;
            if (a.validity == nullptr || bit_get(a.validity, row)) v = St::lift(load_in<In>(a.values, row));
            if (a.seg) sg[j] = __ldg(a.seg + A + j);
        }
        L[j] = v; P[j] = v;
    }
    __syncthreads();
    if (threadIdx.x < G::NSUB) {
        const int b0 = threadIdx.x * RB_SUB, b1 = min(len, b0 + RB_SUB);
        if (b0 < b1) {
            Q[b1 - 1] = P[b1 - 1];
            for (int j = b1 - 2; j >= b0; j--) Q[j] = (a.seg && sg[j] != sg[j + 1]) ? P[j] : St::combine(P[j], Q[j + 1]);
            for (int j = b0 + 1; j < b1; j++)
                if (!(a.seg && sg[j] != sg[j - 1])) P[j] = St::combine(P[j - 1], P[j]);
        }
    }
    __syncthreads();
    // the table: the total of sub-block k is Q[32 k] (exact whenever no segment boundary lies inside it -- the only case read)
    for (int x = threadIdx.x; x < G::LVL * G::NSUB; x += RB_THREADS) {
        const int k = x / G::NSUB, j = x % G::NSUB, g0 = j >> k << k, g1 = min(G::NSUB, g0 + (1 << k));
        auto tot = [&](int m) { return m * RB_SUB < len ? Q[m * RB_SUB] : St::empty(); };
        S pv = tot(g0), sv = tot(g1 - 1);
        for (int m = g0 + 1; m <= j; m++) pv = St::combine(pv, tot(m));
        for (int m = g1 - 2; m >= j; m--) sv = St::combine(tot(m), sv);
        TP[x] = pv; TS[x] = sv;
    }
    __syncthreads();
    for (int j = threadIdx.x; j < RB_B; j += RB_THREADS) {      // whole warps: the ballot needs every lane
        const int64_t i = o0 + j;
        bool ok = false;
        Out x = Out(0);
        if (i < a.n) {
            const uint32_t s32 = __ldg(a.ws + i);
            const int64_t s = s32, e = __ldg(a.we + i);
            if (s32 != BY_NULL && e - s >= a.min_samples) {
                S st = St::empty();
                if (e > s) {
                    if (s >= A && e <= A + len) {
                        const int l = (int)(s - A), r = (int)(e - 1 - A), sl = l / RB_SUB, sr = r / RB_SUB;
                        if (sl < sr) {
                            st = Q[l];
                            if (sr - sl > 1) {
                                const int bl = sl + 1, br = sr - 1;
                                if (bl == br) st = St::combine(st, TS[bl]);
                                else {
                                    const int k = 31 - __clz(bl ^ br);
                                    st = St::combine(St::combine(st, TS[k * G::NSUB + bl]), TP[k * G::NSUB + br]);
                                }
                            }
                            st = St::combine(st, P[r]);
                        } else if (l % RB_SUB == 0 || (a.seg && sg[l - 1] != sg[l])) st = P[r];
                        else if (r % RB_SUB == RB_SUB - 1 || r == len - 1 || (a.seg && sg[r + 1] != sg[r])) st = Q[l];
                        else for (int q = l; q <= r; q++) st = St::combine(st, L[q]);
                    } else if (TILE) st = fold_global<St, In>(a, s, e);
                    else st = window_global<St, In>(a, t, s, e);
                }
                ok = Fin::fin(st, a, x);
            }
        }
        write_out<Fin>(a, i, i < a.n, ok, x);
    }
}

template <class St, typename In, class Fin, bool TILE> static void launch_out(const RollArgs& a, const ByOut& t, const char* name) {
    static bool attr = false;      // the opt-in above 48 KB of dynamic shared memory, once per instantiation
    const int bytes = (int)out_smem<St, TILE>();
    if (!attr) {
        auto* k = k_rollby_out<St, In, Fin, TILE>;
        PLB_CUDA(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes));
        attr = true;
    }
    PLB_LAUNCH(name, (k_rollby_out<St, In, Fin, TILE>), (int)((a.n + RB_B - 1) / RB_B), RB_THREADS, (size_t)bytes, a, t);
}

struct ByPlan { template <class St, typename In, class Fin> static void run(RollArgs a); };
// The largest window W (reduced by k_rollby_bounds) chooses the plan: W <= RB_HALO runs the one-pass small-window plan (no
// state through HBM); wider windows run the prefix / suffix scans, the sparse table and the general output kernel.
template <class St, typename In, class Fin> void ByPlan::run(RollArgs a) {
    using S = typename St::S;
    if (a.W <= RB_HALO) { launch_out<St, In, Fin, true>(a, ByOut{nullptr, nullptr, 0}, "rolling_by_tile"); return; }
    const int64_t nb = (a.n + RB_B - 1) / RB_B;
    int K = 0;
    while ((int64_t(1) << K) < nb) K++;
    DevPtr pre = dev_alloc((size_t)a.n * sizeof(S)), suf = dev_alloc((size_t)a.n * sizeof(S));
    DevPtr tot = dev_alloc((size_t)nb * sizeof(S)), gpre = dev_alloc((size_t)std::max(K, 1) * nb * sizeof(S)), gsuf = dev_alloc((size_t)std::max(K, 1) * nb * sizeof(S));
    a.B = RB_B; a.pre = pre->p; a.suf = suf->p;
    const int64_t ctas = (a.n + RS_TILE - 1) / RS_TILE;
    PLB_LAUNCH("rolling_by_prefix", (k_roll_scan<St, In, false>), (int)ctas, RS_THREADS, 0, a, (int64_t)RS_TILE);
    PLB_LAUNCH("rolling_by_suffix", (k_roll_scan<St, In, true>), (int)ctas, RS_THREADS, 0, a, (int64_t)RS_TILE);
    ByOut t{gpre->p, gsuf->p, nb};
    if (K > 0) {
        PLB_LAUNCH("rolling_by_totals", (k_rollby_totals<S>), grid_for(nb, 256), 256, 0, as<S>(suf), nb, as<S>(tot));
        for (int k = 0; k < K; k++) {      // level k: prefix / suffix scans of the totals in groups of 2^k blocks
            RollArgs l;
            memset(&l, 0, sizeof l);
            l.values = tot->p; l.n = nb; l.B = 1u << k;
            l.pre = as<S>(gpre) + (size_t)k * nb; l.suf = as<S>(gsuf) + (size_t)k * nb;
            const int64_t span = (int64_t)l.B * std::max<int64_t>(1, RS_TILE / l.B);
            const int64_t c = (nb + span - 1) / span;
            PLB_LAUNCH("rolling_by_sparse", (k_roll_scan<St, StateIn, false>), (int)c, RS_THREADS, 0, l, span);
            PLB_LAUNCH("rolling_by_sparse", (k_roll_scan<St, StateIn, true>), (int)c, RS_THREADS, 0, l, span);
        }
    }
    launch_out<St, In, Fin, false>(a, t, "rolling_by_out");
}

// ---------------------------------------------------------------------------------------------------- host side
void check_rolling_by_op(int kind, int closed, int64_t window_size, int64_t min_samples, int ddof, int reserved, int value_dtype) {
    PLB_REQUIRE(kind >= BL_ROLLING_SUM && kind <= BL_ROLLING_STD, BL_ERR_INVALID, "rolling_by: unknown kind " + std::to_string(kind));
    PLB_REQUIRE(value_dtype >= 0, BL_ERR_INVALID, "rolling_by: an operation without a value column");
    PLB_REQUIRE(value_dtype <= BL_BOOL, BL_ERR_INVALID, "rolling_by: unknown value dtype");
    PLB_REQUIRE(reserved == 0, BL_ERR_INVALID, "rolling_by: reserved must be 0");
    PLB_REQUIRE(closed >= BL_CLOSED_RIGHT && closed <= BL_CLOSED_NONE, BL_ERR_INVALID, "rolling_by: unknown closed " + std::to_string(closed));
    PLB_REQUIRE(window_size > 0, BL_ERR_INVALID, "rolling_by: window_size must be strictly positive");
    PLB_REQUIRE(min_samples >= 0, BL_ERR_INVALID, "rolling_by: min_samples must not be negative");
    PLB_REQUIRE(ddof >= 0 && ddof <= 255, BL_ERR_INVALID, "rolling_by: ddof must be in 0..255");
    PLB_REQUIRE(value_dtype != BL_BOOL || kind == BL_ROLLING_SUM, BL_ERR_UNSUPPORTED, "rolling_by: a Boolean column takes only rolling_sum on the device");
}

// ops are checked by the caller (check_rolling_by_op) before any column is uploaded
std::vector<DevCol> op_rolling_by(const std::vector<DevCol>& partition_by, const DevCol& by, const std::vector<RollByOp>& ops, int64_t n) {
    for (auto& op : ops) PLB_REQUIRE(op.values && op.values->len == n, BL_ERR_INVALID, "rolling_by: value columns differ in length");
    for (auto& k : partition_by) PLB_REQUIRE(k.len == n, BL_ERR_INVALID, "rolling_by: partition columns differ in length");
    PLB_REQUIRE(by.len == n, BL_ERR_INVALID, "rolling_by: the `by` column differs in length");
    PLB_REQUIRE(by.dtype == BL_INT32 || by.dtype == BL_INT64 || by.dtype == BL_UINT32 || by.dtype == BL_UINT64, BL_ERR_INVALID,
                "rolling_by: a `by` column must be Int32, Int64, UInt32 or UInt64 (Date / Datetime: their physical Int64)");
    PLB_REQUIRE(n <= 0xFFFFFFFFll, BL_ERR_UNSUPPORTED, "rolling_by: more than 2^32 - 1 rows (IdxSize is u32)");
    std::vector<DevCol> outs;
    if (n == 0) {
        for (auto& op : ops) { outs.push_back(make_col(rolling_dtype(op.kind, op.values->dtype), 0, false)); outs.back().null_count = 0; }
        return outs;
    }
    DevPtr st = dev_alloc(3 * 8);
    dev_memset(st->p, 0, 3 * 8);
    PLB_LAUNCH("rolling_by_check", k_rollby_check, grid_for(n, 256), 256, 0, by.v(), by.vm(), by.dtype, n, as<unsigned long long>(st));
    unsigned long long stats[3];
    PLB_CUDA(cudaMemcpyAsync(stats, st->p, sizeof stats, cudaMemcpyDeviceToHost, ctx().stream));
    PLB_CUDA(cudaStreamSynchronize(ctx().stream));
    PLB_REQUIRE(stats[2] == 0, BL_ERR_INVALID, "rolling_by: a UInt64 `by` value >= 2^63 does not fit the Int64 time (the reference fails on it)");
    const bool need_order = !partition_by.empty() || stats[0] || stats[1];
    PLB_REQUIRE(!need_order || n <= 0x7FFFFFFFll, BL_ERR_UNSUPPORTED, "rolling_by: more than 2^31 - 1 rows need a sort (group tuples)");
    OverOrder o;
    if (need_order) {
        o.gid = partition_ids(partition_by, n);
        build_order(o, &by, BL_SORT_NULLS_LAST, false);
    }
    DevPtr ws = dev_alloc((size_t)n * 4), we = dev_alloc((size_t)n * 4);
    std::vector<DevCol> res;
    unsigned long long W = 0;
    for (size_t k = 0; k < ops.size(); k++) {
        const RollByOp& op = ops[k];
        BoundsArgs b{by.v(), by.vm(), by.dtype, need_order ? as<uint32_t>(o.perm.values) : nullptr, need_order ? as<uint32_t>(o.offsets.values) : nullptr,
                     need_order ? o.G : 1, n, op.window_size, op.closed, as<uint32_t>(ws), as<uint32_t>(we), as<unsigned long long>(st)};
        if (k == 0 || op.window_size != ops[k - 1].window_size || op.closed != ops[k - 1].closed) {
            dev_memset(st->p, 0, 8);
            PLB_LAUNCH("rolling_by_bounds", k_rollby_bounds, grid_for(n, 256), 256, 0, b);
            PLB_CUDA(cudaMemcpyAsync(&W, st->p, 8, cudaMemcpyDeviceToHost, ctx().stream));
            PLB_CUDA(cudaStreamSynchronize(ctx().stream));
        }
        // the casts of op_rolling: SUM Int8/16 / UInt8/16 -> Int64, MEAN / VAR / STD in f64, MIN / MAX narrowed back
        const DevCol& v = *op.values;
        const bool small = dtype_is_small_int(v.dtype);
        const DevCol w = small ? op_cast_small_int(v, BL_INT64, false) : v;
        DevCol out = make_col(rolling_dtype(op.kind, w.dtype), n, true);
        out.null_count = -1;
        RollArgs a;
        memset(&a, 0, sizeof a);
        a.values = w.v(); a.validity = w.vm(); a.n = n;
        if (need_order) { a.perm = as<uint32_t>(o.perm.values); a.seg = as<uint32_t>(o.seg.values); a.offsets = as<uint32_t>(o.offsets.values); a.G = o.G; }
        else a.G = 1;
        a.ws = as<uint32_t>(ws); a.we = as<uint32_t>(we); a.W = (int64_t)W;
        a.min_samples = op.min_samples; a.ddof = op.ddof;
        a.out = out.values->p; a.out_valid = as<uint32_t>(out.validity);
        const int kind = op.kind;
        const bool det = ctx().deterministic && (kind != BL_ROLLING_SUM || dtype_is_float(w.dtype)) && kind != BL_ROLLING_MIN && kind != BL_ROLLING_MAX;
        if (need_order || det) dev_memset(a.out_valid, 0, bitmap_bytes(n));
        roll_dispatch<ByPlan>(kind, w.dtype, a, det);
        if (small && (kind == BL_ROLLING_MIN || kind == BL_ROLLING_MAX)) out = op_cast_small_int(out, v.dtype, false);
        res.push_back(out);
    }
    return res;
}

}  // namespace plb

// ================================================================================ C ABI
using namespace plb;
extern "C" {

bl_status bl_rolling_by(const bl_sort_key* partition_by, int32_t n_partition_by, const bl_column* by, const bl_rolling_by_op* ops, int32_t n_ops,
                        int32_t out_location, bl_column* outs) {
    BL_TRY
    PLB_REQUIRE(n_ops >= 1 && ops && outs, BL_ERR_INVALID, "rolling_by: no operations or no outputs");
    PLB_REQUIRE(by != nullptr, BL_ERR_INVALID, "rolling_by: no `by` column");
    int64_t n = -1;
    check_window_keys("rolling_by", partition_by, n_partition_by, nullptr, n);
    set_window_len("rolling_by", by->length, "the `by` column", n);
    for (int i = 0; i < n_ops; i++) {
        PLB_REQUIRE(ops[i].values != nullptr, BL_ERR_INVALID, "rolling_by: operation " + std::to_string(i) + " has no value column");
        check_rolling_by_op(ops[i].kind, ops[i].closed, ops[i].window_size, ops[i].min_samples, ops[i].ddof, ops[i].reserved, ops[i].values->dtype);
        set_window_len("rolling_by", ops[i].values->length, "value column " + std::to_string(i), n);
    }
    std::vector<DevCol> parts;
    for (int i = 0; i < n_partition_by; i++) parts.push_back(import_key(partition_by[i], true));
    const DevCol byc = import_column(by, 1);
    std::vector<DevCol> vals(n_ops);
    std::vector<RollByOp> v(n_ops);
    for (int i = 0; i < n_ops; i++) {
        vals[i] = import_column(ops[i].values, 1);
        v[i].kind = ops[i].kind; v[i].closed = ops[i].closed; v[i].window_size = ops[i].window_size; v[i].min_samples = ops[i].min_samples;
        v[i].ddof = ops[i].ddof; v[i].values = &vals[i];
    }
    std::vector<DevCol> res = op_rolling_by(parts, byc, v, n);
    export_many(res, out_location, outs);
    BL_CATCH
}

}  // extern "C"
