// asof.cu — asof join on the device: for each left row, the right row a backward / forward / nearest search picks.
//
// Reference (paths relative to the reference checkout's crates/): _join_asof_dispatch polars-ops/src/frame/join/asof/mod.rs:325-394,
// the cursors AsofJoinForwardState / AsofJoinBackwardState / AsofJoinNearestState mod.rs:47-200, join_asof_impl and the
// tolerance filter default.rs:12-145, the `by` paths (one cursor per right group) groups.rs:39-345.
//
// The reference walks the right side with a cursor while the left rows go by.  Under the precondition checked here (the
// non-null left values non-decreasing, the right side nulls first and then non-decreasing, both in the total order; per
// group with `by`) the cursor's answer for a left value depends on that value alone, so every left row is answered by
// asof_pick below: a few binary searches over its sorted right segment.  Inputs outside the precondition give
// BL_ERR_UNSUPPORTED and the caller keeps the reference's own answer.
//
// Plans (DESIGN.md §10):
//   no `by`  k_asof_right_check   right precondition, z = first non-null right row
//            k_asof_search        one CTA per 2048 left rows: the left precondition inside the tile (prefix max), the tile's
//                                 right window (two binary searches), staged in shared memory when it fits, then asof_pick
//            k_asof_tiles_sorted  the left precondition across tiles
//   `by`     group ids over left ‖ right (op_pack_keys + op_group_first_ids; strings op_string_codes first); right rows
//            stable-sorted by group (sort_pairs_u32); k_asof_segments gathers the right keys into segment order, writes each
//            group's [z, e) and checks the right precondition per segment; k_asof_search as above with per-row segments and
//            the global left check; only when that fails, the left rows are stable-sorted by group and k_asof_left_groups
//            checks them per group.
#include <algorithm>
#include <vector>

#include "common.cuh"
#include "dev_utils.cuh"
#include "strings.cuh"

namespace plb {

constexpr uint32_t ASOF_NONE = 0xFFFFFFFFu;
constexpr int AS_THREADS = 256, AS_ITEMS = 8, AS_TILE = AS_THREADS * AS_ITEMS;
constexpr int AS_WIN_BYTES = 16384;      // right window staged in shared memory

// Per key type: the total-order key (tot_cmp, polars-utils/src/total_ord.rs: NaN greatest and equal to itself, -0.0 == +0.0),
// NaN, and abs_diff (polars-utils/src/abs_diff.rs: exact unsigned difference for integers, `a > b ? a - b : b - a` in the
// float's own precision, NaN when either side is NaN).
template <typename T> struct AsofNum;
template <> struct AsofNum<int32_t> {
    using D = uint32_t;
    __device__ static uint64_t key(int32_t v) { return (uint32_t)v ^ 0x80000000u; }
    __device__ static bool nan(int32_t) { return false; }
    __device__ static D diff(int32_t a, int32_t b) { return a > b ? (D)a - (D)b : (D)b - (D)a; }
};
template <> struct AsofNum<int64_t> {
    using D = uint64_t;
    __device__ static uint64_t key(int64_t v) { return (uint64_t)v ^ 0x8000000000000000ull; }
    __device__ static bool nan(int64_t) { return false; }
    __device__ static D diff(int64_t a, int64_t b) { return a > b ? (D)a - (D)b : (D)b - (D)a; }
};
template <> struct AsofNum<uint32_t> {
    using D = uint32_t;
    __device__ static uint64_t key(uint32_t v) { return v; }
    __device__ static bool nan(uint32_t) { return false; }
    __device__ static D diff(uint32_t a, uint32_t b) { return a > b ? a - b : b - a; }
};
template <> struct AsofNum<uint64_t> {
    using D = uint64_t;
    __device__ static uint64_t key(uint64_t v) { return v; }
    __device__ static bool nan(uint64_t) { return false; }
    __device__ static D diff(uint64_t a, uint64_t b) { return a > b ? a - b : b - a; }
};
template <> struct AsofNum<float> {
    using D = float;
    __device__ static uint64_t key(float v) { const uint32_t u = (uint32_t)canonical_f32_bits(v); return (u >> 31) ? (uint32_t)~u : (u | 0x80000000u); }
    __device__ static bool nan(float v) { return v != v; }
    __device__ static D diff(float a, float b) { return a > b ? a - b : b - a; }
};
template <> struct AsofNum<double> {
    using D = double;
    __device__ static uint64_t key(double v) { const uint64_t u = canonical_f64_bits(v); return (u >> 63) ? ~u : (u | 0x8000000000000000ull); }
    __device__ static bool nan(double v) { return v != v; }
    __device__ static D diff(double a, double b) { return a > b ? a - b : b - a; }
};

// right keys: rows [lo, hi) from shared memory, the rest from global memory
template <typename T> struct AsofRight {
    const T* g; const T* s; int64_t lo, hi;
    __device__ T operator()(int64_t j) const { return (j >= lo && j < hi) ? s[j - lo] : g[j]; }
};

// first j in [a, b) whose key is > k (upper) or >= k (lower); b when there is none
template <typename T> __device__ int64_t asof_bound(const AsofRight<T>& R, int64_t a, int64_t b, uint64_t k, bool upper) {
    while (a < b) {
        const int64_t m = a + ((b - a) >> 1);
        const uint64_t km = AsofNum<T>::key(R(m));
        if (upper ? km <= k : km < k) a = m + 1; else b = m;
    }
    return a;
}

// The position in [z, e) a sorted, null-free right segment gives the left value l, or -1.  Every lower / upper bound of l
// in [z, e) lies in [blo, bhi] (the whole segment when nothing narrower is known).
//   backward  the last j with r_j <= l (< l without allow_eq), total order
//   forward   the first j with r_j >= l (> l without allow_eq), total order
//   nearest   partial order, as AsofJoinNearestState (mod.rs:135-199): U = the first j with r_j > l (else e); with allow_eq
//             and r_{U-1} == l, U - 1; else U moves to the end of its run of equal values, L = (the first j in [z, U) with
//             r_j >= l) - 1 (U - 1 when there is none), and the closer of L and U wins, U on a tie
template <typename T>
__device__ int64_t asof_pick(const AsofRight<T>& R, int64_t z, int64_t e, int64_t blo, int64_t bhi, T l, int strategy, bool allow_eq) {
    using N = AsofNum<T>;
    const uint64_t k = N::key(l);
    if (strategy == BL_ASOF_BACKWARD) { const int64_t j = asof_bound(R, blo, bhi, k, allow_eq) - 1; return j >= z ? j : -1; }
    if (strategy == BL_ASOF_FORWARD) { const int64_t j = asof_bound(R, blo, bhi, k, !allow_eq); return j < e ? j : -1; }
    int64_t U = asof_bound(R, blo, bhi, k, true);
    if (U < e && N::nan(R(U))) U = e;                      // only NaNs lie above l: `r > l` never holds
    if (allow_eq && U > z && R(U - 1) == l) return U - 1;
    if (U < e) U = asof_bound(R, U, e, N::key(R(U)), true) - 1;
    const int64_t lb = min(asof_bound(R, blo, bhi, k, false), U);
    const int64_t L = (lb < U && !N::nan(R(lb))) ? lb - 1 : U - 1;
    const bool hasL = L >= z, hasU = U < e;
    if (hasL && hasU) return N::diff(l, R(U)) <= N::diff(l, R(L)) ? U : L;
    return hasU ? U : hasL ? L : -1;
}

template <typename T> struct AsofArgs {
    const T* L; const uint32_t* lvalid; int64_t nl;
    const T* R; int64_t nr;                  // right keys (`by`: in segment order)
    const uint64_t* rz;                      // no `by`: the first non-null right row
    const uint32_t* perm;                    // `by`: right row at each segment position
    const uint32_t* lgid;                    // `by`: group of each left row (ASOF_NONE: null `by` key)
    const uint32_t* seg_z; const uint32_t* seg_e;
    int strategy, allow_eq, has_tol;
    T tol;
    uint32_t* out; uint32_t* out_valid;
    uint64_t* tile_lo; uint64_t* tile_hi;    // smallest / largest non-null left key of each tile (none: ~0 / 0)
    int* bad;                                // bad[0]: the left side is not sorted
};

// Tile position -> shared-memory slot: one spare slot after every thread's AS_ITEMS rows, so that the threads of a warp,
// each walking its own consecutive rows, hit different banks (8-byte keys: two ways, the minimum; 4-byte keys: none).
__device__ __forceinline__ int as_pad(int i) { return i + i / AS_ITEMS; }

template <typename T, bool BY>
__global__ void __launch_bounds__(AS_THREADS) k_asof_search(const AsofArgs<T> a) {
    using N = AsofNum<T>;
    __shared__ T s_l[AS_TILE + AS_TILE / AS_ITEMS];
    __shared__ uint32_t s_ok[AS_TILE / 32];
    __shared__ uint32_t s_out[AS_TILE + AS_TILE / AS_ITEMS];
    __shared__ __align__(16) unsigned char s_rbuf[AS_WIN_BYTES];
    __shared__ uint64_t s_wmax[AS_THREADS / 32], s_wmin[AS_THREADS / 32];
    __shared__ int64_t s_win[5];
    T* s_r = reinterpret_cast<T*>(s_rbuf);
    const unsigned lane = lane_id(), warp = threadIdx.x >> 5;
    const int64_t base = (int64_t)blockIdx.x * AS_TILE;
    // coalesced load of the tile's keys and validity
#pragma unroll
    for (int k = 0; k < AS_ITEMS; k++) {
        const int i = k * AS_THREADS + threadIdx.x;
        const int64_t row = base + i;
        const bool ok = row < a.nl && (a.lvalid == nullptr || bit_get(a.lvalid, row));
        s_l[as_pad(i)] = row < a.nl ? a.L[row] : T(0);
        const unsigned b = __ballot_sync(0xffffffffu, ok);
        if (lane == 0) s_ok[i >> 5] = b;
    }
    __syncthreads();
    // left precondition inside the tile: every non-null key >= the largest non-null key before it
    const int t0 = threadIdx.x * AS_ITEMS;
    uint64_t mx = 0, mn = ~0ull, first = 0;
    bool bad = false, have = false;
#pragma unroll
    for (int k = 0; k < AS_ITEMS; k++) {
        const int i = t0 + k;
        if (!((s_ok[i >> 5] >> (i & 31)) & 1u)) continue;
        const uint64_t kk = N::key(s_l[as_pad(i)]);
        if (!have) { first = kk; have = true; }
        bad |= kk < mx;
        mx = max(mx, kk); mn = min(mn, kk);
    }
    uint64_t incl = mx;                      // prefix max over the threads of the warp
    for (int o = 1; o < 32; o <<= 1) { const uint64_t y = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= (unsigned)o) incl = max(incl, y); }
    uint64_t wmn = mn;
    for (int o = 16; o; o >>= 1) wmn = min(wmn, __shfl_xor_sync(0xffffffffu, wmn, o));
    if (lane == 31) s_wmax[warp] = incl;
    if (lane == 0) s_wmin[warp] = wmn;
    uint64_t excl = __shfl_up_sync(0xffffffffu, incl, 1);
    if (lane == 0) excl = 0;
    __syncthreads();
    for (unsigned w = 0; w < warp; w++) excl = max(excl, s_wmax[w]);
    bad |= have && first < excl;
    if (__syncthreads_or(bad) && threadIdx.x == 0) atomicOr(&a.bad[0], 1);
    const bool tile_any = __syncthreads_or(have);
    uint64_t tmx = 0, tmn = ~0ull;
    for (int w = 0; w < AS_THREADS / 32; w++) { tmx = max(tmx, s_wmax[w]); tmn = min(tmn, s_wmin[w]); }
    if (threadIdx.x == 0) { a.tile_lo[blockIdx.x] = tmn; a.tile_hi[blockIdx.x] = tmx; }
    // no `by`: every lower / upper bound of a key in [tmn, tmx] lies in [blo, bhi]; the window around it is staged when it fits
    AsofRight<T> R{a.R, s_r, 0, 0};
    int64_t z = 0, e = a.nr, blo = 0, bhi = 0;
    if (!BY) {
        if (threadIdx.x == 0) {
            z = (int64_t)*a.rz;
            int64_t wlo = 0, whi = 0;
            if (tile_any && z < e) {
                blo = asof_bound(R, z, e, tmn, false);
                bhi = asof_bound(R, blo, e, tmx, true);
                wlo = max(z, blo - 1); whi = min(e, bhi + 1);
                if ((whi - wlo) * (int64_t)sizeof(T) > AS_WIN_BYTES) wlo = whi = 0;
            }
            s_win[0] = z; s_win[1] = blo; s_win[2] = bhi; s_win[3] = wlo; s_win[4] = whi;
        }
        __syncthreads();
        z = s_win[0]; blo = s_win[1]; bhi = s_win[2];
        R.lo = s_win[3]; R.hi = s_win[4];
        for (int64_t j = R.lo + threadIdx.x; j < R.hi; j += AS_THREADS) s_r[j - R.lo] = a.R[j];
        __syncthreads();
    }
    const typename N::D abs_tol = N::diff(a.tol, T(0));
#pragma unroll 1
    for (int k = 0; k < AS_ITEMS; k++) {
        const int i = t0 + k;
        const int64_t row = base + i;
        uint32_t res = ASOF_NONE;
        if (row < a.nl && ((s_ok[i >> 5] >> (i & 31)) & 1u)) {
            const T l = s_l[as_pad(i)];
            int64_t sz = z, se = e, slo = blo, shi = bhi;
            bool go = true;
            if (BY) {
                const uint32_t g = a.lgid[row];
                go = g != ASOF_NONE;
                if (go) { sz = a.seg_z[g]; se = a.seg_e[g]; slo = sz; shi = se; }
            } else go = z < e;
            if (go) {
                const int64_t j = asof_pick(R, sz, se, slo, shi, l, a.strategy, a.allow_eq != 0);
                if (j >= 0 && (!a.has_tol || N::diff(l, R(j)) <= abs_tol)) res = BY ? a.perm[j] : (uint32_t)j;
            }
        }
        s_out[as_pad(i)] = res;
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < AS_ITEMS; k++) {
        const int i = k * AS_THREADS + threadIdx.x;
        const int64_t row = base + i;
        const uint32_t v = s_out[as_pad(i)];
        if (row < a.nl) a.out[row] = v;
        const unsigned b = __ballot_sync(0xffffffffu, row < a.nl && v != ASOF_NONE);
        if (lane == 0 && row < a.nl) a.out_valid[row >> 5] = b;
    }
}

// the left precondition across tiles: each tile's smallest key >= the largest key of every tile before it
__global__ void __launch_bounds__(1024) k_asof_tiles_sorted(const uint64_t* __restrict__ lo, const uint64_t* __restrict__ hi, int64_t ntiles, int* bad) {
    __shared__ uint64_t s_mx[1024];
    const int64_t per = (ntiles + 1023) / 1024, a = threadIdx.x * per, b = min(a + per, ntiles);
    uint64_t m = 0;
    for (int64_t t = a; t < b; t++) m = max(m, hi[t]);
    s_mx[threadIdx.x] = m;
    __syncthreads();
    if (threadIdx.x == 0) { uint64_t acc = 0; for (int t = 0; t < 1024; t++) { const uint64_t v = s_mx[t]; s_mx[t] = acc; acc = max(acc, v); } }
    __syncthreads();
    m = s_mx[threadIdx.x];
    bool bd = false;
    for (int64_t t = a; t < b; t++) { bd |= lo[t] < m; m = max(m, hi[t]); }
    if (bd) atomicOr(bad, 1);
}

// no `by`: nulls first, then non-decreasing; rz = the first non-null row (nr when there is none); bad[1] on a violation
template <typename T>
__global__ void __launch_bounds__(256) k_asof_right_check(const T* __restrict__ R, const uint32_t* __restrict__ valid, int64_t nr, unsigned long long* rz, int* bad) {
    bool bd = false;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < nr; i += (int64_t)gridDim.x * blockDim.x) {
        const bool v = valid == nullptr || bit_get(valid, i);
        const bool pv = i > 0 && (valid == nullptr || bit_get(valid, i - 1));
        if (v && !pv) atomicMin(rz, (unsigned long long)i);
        if (pv && !v) bd = true;
        if (pv && v && AsofNum<T>::key(R[i - 1]) > AsofNum<T>::key(R[i])) bd = true;
    }
    if (bd) atomicOr(&bad[1], 1);
}

// `by`: group id of every row of left ‖ right (ASOF_NONE for a null `by` key); sort keys: the group, or gnull when the row is
// outside every group (null `by` key, or for the left side a null `on` value too)
__global__ void __launch_bounds__(256) k_asof_group_keys(const uint32_t* __restrict__ gid, const uint32_t* __restrict__ byvalid, const uint32_t* __restrict__ lvalid, int64_t nl,
                                                         int64_t n, uint32_t gnull, uint32_t* __restrict__ g_out, uint32_t* __restrict__ sk, uint32_t* __restrict__ iota) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const bool bv = byvalid == nullptr || bit_get(byvalid, i);
        const uint32_t g = bv ? gid[i] : ASOF_NONE;
        g_out[i] = g;
        const bool on_ok = i >= nl || lvalid == nullptr || bit_get(lvalid, i);
        sk[i] = (g != ASOF_NONE && on_ok) ? g : gnull;
        iota[i] = (uint32_t)(i < nl ? i : i - nl);
    }
}

// `by`, right side sorted by group (sk, perm): rs = the right keys in that order; each group's non-null range [z, e) of
// positions; bad[1] when a segment is not nulls-first-then-sorted
template <typename T>
__global__ void __launch_bounds__(256) k_asof_segments(const uint32_t* __restrict__ sk, const uint32_t* __restrict__ perm, const T* __restrict__ R, const uint32_t* __restrict__ rvalid,
                                                       int64_t nr, uint32_t gnull, T* __restrict__ rs, uint32_t* __restrict__ seg_z, uint32_t* __restrict__ seg_e, int* bad) {
    bool bd = false;
    for (int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; p < nr; p += (int64_t)gridDim.x * blockDim.x) {
        const uint32_t g = sk[p], r = perm[p];
        const T x = R[r];
        rs[p] = x;
        if (g == gnull) continue;
        const bool start = p == 0 || sk[p - 1] != g, end = p == nr - 1 || sk[p + 1] != g;
        const bool v = rvalid == nullptr || bit_get(rvalid, r);
        const bool pv = !start && (rvalid == nullptr || bit_get(rvalid, perm[p - 1]));
        if (end) { seg_e[g] = (uint32_t)(p + 1); if (!v) seg_z[g] = (uint32_t)(p + 1); }
        if (v && !pv) seg_z[g] = (uint32_t)p;
        if (pv && !v) bd = true;
        if (pv && v && AsofNum<T>::key(R[perm[p - 1]]) > AsofNum<T>::key(x)) bd = true;
    }
    if (bd) atomicOr(&bad[1], 1);
}

// `by`, left rows stable-sorted by group: bad[0] when two neighbours of one group decrease
template <typename T>
__global__ void __launch_bounds__(256) k_asof_left_groups(const uint32_t* __restrict__ sk, const uint32_t* __restrict__ perm, const T* __restrict__ L, int64_t nl, uint32_t gnull, int* bad) {
    bool bd = false;
    for (int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x + 1; p < nl; p += (int64_t)gridDim.x * blockDim.x)
        if (sk[p] != gnull && sk[p] == sk[p - 1] && AsofNum<T>::key(L[perm[p - 1]]) > AsofNum<T>::key(L[perm[p]])) bd = true;
    if (bd) atomicOr(&bad[0], 1);
}

template <typename S>
__global__ void __launch_bounds__(256) k_asof_widen(const S* __restrict__ in, int32_t* __restrict__ out, int64_t n) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) out[i] = (int32_t)in[i];
}

// 8/16-bit keys are searched as Int32, as _join_asof_dispatch casts them (mod.rs:333-338)
static DevCol widen_to_i32(const DevCol& in) {
    if (!dtype_is_small_int(in.dtype)) return in;
    DevCol out = make_col(BL_INT32, in.len, false);
    out.validity = in.validity; out.null_count = in.null_count;
    const int grid = grid_for(in.len, 256, 16);
    if (in.len == 0) return out;
    switch (in.dtype) {
        case BL_INT8: PLB_LAUNCH("asof_widen", k_asof_widen<int8_t>, grid, 256, 0, reinterpret_cast<const int8_t*>(in.v()), as<int32_t>(out.values), in.len); break;
        case BL_INT16: PLB_LAUNCH("asof_widen", k_asof_widen<int16_t>, grid, 256, 0, reinterpret_cast<const int16_t*>(in.v()), as<int32_t>(out.values), in.len); break;
        case BL_UINT8: PLB_LAUNCH("asof_widen", k_asof_widen<uint8_t>, grid, 256, 0, reinterpret_cast<const uint8_t*>(in.v()), as<int32_t>(out.values), in.len); break;
        default: PLB_LAUNCH("asof_widen", k_asof_widen<uint16_t>, grid, 256, 0, reinterpret_cast<const uint16_t*>(in.v()), as<int32_t>(out.values), in.len); break;
    }
    return out;
}

// The `by` groups of left ‖ right: gid (nl + nr entries, the first row of each group in the concatenation) and the AND of
// the `by` validities (null = no nulls).  Equal values get equal ids on both sides because both are encoded together.
struct AsofGroups { DevCol gid; DevPtr valid; };

static AsofGroups asof_groups(const bl_sort_key* left_by, const bl_sort_key* right_by, int n_by, int64_t nl, int64_t nr) {
    const int64_t n = nl + nr;
    std::vector<DevCol> cats;
    DevPtr valid;
    for (int i = 0; i < n_by; i++) {
        DevCol c;
        if (left_by[i].strings) {
            std::vector<bl_string_column> all(left_by[i].strings, left_by[i].strings + left_by[i].n_chunks);
            all.insert(all.end(), right_by[i].strings, right_by[i].strings + right_by[i].n_chunks);
            c = op_string_codes(import_string(all.data(), (int)all.size()), nullptr);
        } else {
            const bl_column pair[2] = {*left_by[i].column, *right_by[i].column};
            c = import_column(pair, 2);
        }
        if (c.validity) valid = valid ? bitmap_and(as<uint32_t>(valid), c.vm(), nullptr, n) : c.validity;
        c.validity = nullptr; c.null_count = 0;      // a null `by` key matches nothing: the rows are masked by `valid` instead
        cats.push_back(c);
    }
    return {op_group_first_ids(op_pack_keys(cats)), valid};
}

template <typename T>
static DevCol asof_run(const DevCol& lc, const DevCol& rc, const AsofGroups* grp, int strategy, bool allow_eq, bool has_tol, T tol) {
    Context& c = ctx();
    const int64_t nl = lc.len, nr = rc.len;
    DevCol out = make_col(BL_UINT32, nl, true);
    out.null_count = -1;
    if (nl == 0) return out;
    const int64_t ntiles = (nl + AS_TILE - 1) / AS_TILE;
    DevPtr flags = dev_alloc(16), tiles = dev_alloc((size_t)ntiles * 16);
    dev_memset(flags->p, 0, 16);
    int* bad = as<int>(flags);
    unsigned long long* rz = reinterpret_cast<unsigned long long*>((char*)flags->p + 8);
    AsofArgs<T> a;
    memset(&a, 0, sizeof a);
    a.L = reinterpret_cast<const T*>(lc.v()); a.lvalid = lc.vm(); a.nl = nl; a.nr = nr;
    a.strategy = strategy; a.allow_eq = allow_eq; a.has_tol = has_tol; a.tol = tol;
    a.out = as<uint32_t>(out.values); a.out_valid = as<uint32_t>(out.validity);
    a.tile_lo = as<uint64_t>(tiles); a.tile_hi = as<uint64_t>(tiles) + ntiles;
    a.bad = bad;
    DevPtr rs, perm, seg, lg, lsk, lperm;
    const uint32_t gnull = (uint32_t)(nl + nr);
    if (!grp) {
        PLB_CUDA(cudaMemcpyAsync(rz, &nr, 8, cudaMemcpyHostToDevice, c.stream));
        if (nr) PLB_LAUNCH("asof_right_check", k_asof_right_check<T>, grid_for(nr, 256), 256, 0, reinterpret_cast<const T*>(rc.v()), rc.vm(), nr, rz, bad);
        a.R = reinterpret_cast<const T*>(rc.v()); a.rz = reinterpret_cast<const uint64_t*>(rz);
        PLB_LAUNCH("asof_search", (k_asof_search<T, false>), (int)ntiles, AS_THREADS, 0, a);
    } else {
        const int64_t n = nl + nr;
        DevPtr g = dev_alloc((size_t)n * 4), sk = dev_alloc((size_t)n * 4), io = dev_alloc((size_t)n * 4);
        PLB_LAUNCH("asof_group_keys", k_asof_group_keys, grid_for(n, 256), 256, 0, as<uint32_t>(grp->gid.values), as<uint32_t>(grp->valid), lc.vm(), nl, n, gnull,
                   as<uint32_t>(g), as<uint32_t>(sk), as<uint32_t>(io));
        const int kb = bits_for((uint64_t)gnull);
        // right rows by group, each group's rows in row order
        uint32_t* rsk = as<uint32_t>(sk) + nl;
        uint32_t* rperm = as<uint32_t>(io) + nl;
        sort_pairs_u32(rsk, rperm, nr, kb);
        rs = dev_alloc((size_t)std::max<int64_t>(nr, 1) * sizeof(T));
        seg = dev_alloc((size_t)n * 8);
        dev_memset(seg->p, 0, (size_t)n * 8);
        uint32_t* seg_z = as<uint32_t>(seg);
        uint32_t* seg_e = seg_z + n;
        if (nr) PLB_LAUNCH("asof_segments", k_asof_segments<T>, grid_for(nr, 256), 256, 0, rsk, rperm, reinterpret_cast<const T*>(rc.v()), rc.vm(), nr, gnull, as<T>(rs), seg_z, seg_e, bad);
        a.R = as<T>(rs); a.perm = rperm; a.lgid = as<uint32_t>(g); a.seg_z = seg_z; a.seg_e = seg_e;
        PLB_LAUNCH("asof_search_by", (k_asof_search<T, true>), (int)ntiles, AS_THREADS, 0, a);
        PLB_LAUNCH("asof_tiles_sorted", k_asof_tiles_sorted, 1, 1024, 0, a.tile_lo, a.tile_hi, ntiles, bad);
        int hb[2];
        PLB_CUDA(cudaMemcpyAsync(hb, bad, 8, cudaMemcpyDeviceToHost, c.stream));
        PLB_CUDA(cudaStreamSynchronize(c.stream));
        if (hb[0] && !hb[1]) {      // not sorted globally: sorted within every group?
            dev_memset(bad, 0, 4);
            uint32_t* lk = as<uint32_t>(sk);
            uint32_t* lp = as<uint32_t>(io);
            sort_pairs_u32(lk, lp, nl, kb);
            PLB_LAUNCH("asof_left_groups", k_asof_left_groups<T>, grid_for(nl, 256), 256, 0, lk, lp, reinterpret_cast<const T*>(lc.v()), nl, gnull, bad);
        }
    }
    if (!grp) PLB_LAUNCH("asof_tiles_sorted", k_asof_tiles_sorted, 1, 1024, 0, a.tile_lo, a.tile_hi, ntiles, bad);
    int hb[2];
    PLB_CUDA(cudaMemcpyAsync(hb, bad, 8, cudaMemcpyDeviceToHost, c.stream));
    PLB_CUDA(cudaStreamSynchronize(c.stream));
    PLB_REQUIRE(!hb[1], BL_ERR_UNSUPPORTED, grp ? "join_asof: the right `on` column is not sorted (nulls first) within every `by` group"
                                                : "join_asof: the right `on` column is not sorted (nulls first)");
    PLB_REQUIRE(!hb[0], BL_ERR_UNSUPPORTED, grp ? "join_asof: the left `on` column is not sorted within every `by` group"
                                                : "join_asof: the left `on` column is not sorted (non-null values)");
    return out;
}

// host copy of the length-1 tolerance column as the key type (8/16-bit: widened like the key)
template <typename T> static T tol_value(const DevCol& t) {
    DevCol w = widen_to_i32(t);
    T v;
    PLB_CUDA(cudaMemcpyAsync(&v, w.v(), sizeof(T), cudaMemcpyDeviceToHost, ctx().stream));
    PLB_CUDA(cudaStreamSynchronize(ctx().stream));
    return v;
}

template <typename T> static DevCol asof_typed(const DevCol& l, const DevCol& r, const AsofGroups* g, int strategy, bool allow_eq, const DevCol* tol) {
    return asof_run<T>(l, r, g, strategy, allow_eq, tol != nullptr, tol ? tol_value<T>(*tol) : T(0));
}

static int64_t by_length(const bl_sort_key& k) {
    if (k.column) return k.column->length;
    int64_t n = 0;
    for (int j = 0; j < k.n_chunks; j++) n += k.strings[j].length;
    return n;
}

}  // namespace plb

// ================================================================================ C ABI
using namespace plb;
extern "C" {

bl_status bl_join_asof(const bl_column* left_on, const bl_column* right_on, const bl_sort_key* left_by, const bl_sort_key* right_by, int32_t n_by, int32_t strategy,
                       int32_t allow_eq, const bl_column* tolerance, int32_t out_location, bl_column* out_right_idx) {
    BL_TRY
    PLB_REQUIRE(left_on && right_on && out_right_idx, BL_ERR_INVALID, "join_asof: null argument");
    PLB_REQUIRE(strategy == BL_ASOF_BACKWARD || strategy == BL_ASOF_FORWARD || strategy == BL_ASOF_NEAREST, BL_ERR_INVALID, "join_asof: unknown strategy");
    PLB_REQUIRE(n_by >= 0 && (n_by == 0 || (left_by && right_by)), BL_ERR_INVALID, "join_asof: n_by > 0 needs left_by and right_by");
    const int dt = left_on->dtype;
    PLB_REQUIRE(dt >= BL_INT8 && dt <= BL_BOOL, BL_ERR_INVALID, "join_asof: unknown key dtype");
    PLB_REQUIRE(dt == right_on->dtype, BL_ERR_DTYPE, std::string("join_asof: mismatching key dtypes ") + dtype_name(dt) + " and " + dtype_name(right_on->dtype));
    PLB_REQUIRE(dt != BL_BOOL, BL_ERR_UNSUPPORTED, "join_asof: Boolean keys are outside the hot path");
    const int64_t nl = left_on->length, nr = right_on->length;
    for (int i = 0; i < n_by; i++) {
        const bl_sort_key &lb = left_by[i], &rb = right_by[i];
        const std::string w = "join_asof: `by` column " + std::to_string(i);
        PLB_REQUIRE(lb.flags == 0 && rb.flags == 0, BL_ERR_INVALID, w + ": flags must be 0");
        PLB_REQUIRE((lb.column != nullptr) != (lb.strings != nullptr) && (rb.column != nullptr) != (rb.strings != nullptr), BL_ERR_INVALID,
                    w + " must set exactly one of `column` and `strings` on each side");
        PLB_REQUIRE((lb.strings == nullptr || lb.n_chunks >= 1) && (rb.strings == nullptr || rb.n_chunks >= 1), BL_ERR_INVALID, w + ": a string column without chunks");
        PLB_REQUIRE((lb.strings != nullptr) == (rb.strings != nullptr), BL_ERR_DTYPE, w + ": a string column on one side only");
        if (lb.column) {
            PLB_REQUIRE(lb.column->dtype == rb.column->dtype, BL_ERR_DTYPE, w + ": mismatching dtypes " + dtype_name(lb.column->dtype) + " and " + dtype_name(rb.column->dtype));
            PLB_REQUIRE(lb.column->dtype != BL_BOOL, BL_ERR_UNSUPPORTED, w + ": Boolean `by` columns are outside the hot path");
        }
        PLB_REQUIRE(by_length(lb) == nl && by_length(rb) == nr, BL_ERR_INVALID, w + ": length differs from its side's `on` column");
    }
    if (tolerance) {
        // 8/16-bit keys are searched as Int32 and the reference extracts their tolerance as Int32 (mod.rs:333-338, default.rs:128)
        PLB_REQUIRE(tolerance->length == 1 && (tolerance->dtype == dt || (dtype_is_small_int(dt) && tolerance->dtype == BL_INT32)), BL_ERR_INVALID,
                    "join_asof: the tolerance must be a length-1 column of the key dtype (or Int32 for an 8/16-bit key)");
    }
    PLB_REQUIRE(nl <= 0xFFFFFFFEll && nr <= 0xFFFFFFFEll, BL_ERR_UNSUPPORTED, "join_asof: more than 2^32 - 2 rows on one side (IdxSize is u32)");
    PLB_REQUIRE(n_by == 0 || nl + nr <= 0xFFFFFFFEll, BL_ERR_UNSUPPORTED, "join_asof: more than 2^32 - 2 rows on both sides together with `by`");
    DevCol tol;
    if (tolerance) {
        tol = import_column(tolerance, 1);
        if (tol.validity) {
            uint32_t w0 = 0;
            PLB_CUDA(cudaMemcpyAsync(&w0, tol.vm(), 4, cudaMemcpyDeviceToHost, ctx().stream));
            PLB_CUDA(cudaStreamSynchronize(ctx().stream));
            PLB_REQUIRE(w0 & 1u, BL_ERR_INVALID, "join_asof: the tolerance is null");
        }
    }
    DevCol l = widen_to_i32(import_column(left_on, 1)), r = widen_to_i32(import_column(right_on, 1));
    AsofGroups g;
    if (n_by) g = asof_groups(left_by, right_by, n_by, nl, nr);
    const AsofGroups* gp = n_by ? &g : nullptr;
    const DevCol* tp = tolerance ? &tol : nullptr;
    DevCol o;
    switch (l.dtype) {
        case BL_INT32: o = asof_typed<int32_t>(l, r, gp, strategy, allow_eq != 0, tp); break;
        case BL_INT64: o = asof_typed<int64_t>(l, r, gp, strategy, allow_eq != 0, tp); break;
        case BL_UINT32: o = asof_typed<uint32_t>(l, r, gp, strategy, allow_eq != 0, tp); break;
        case BL_UINT64: o = asof_typed<uint64_t>(l, r, gp, strategy, allow_eq != 0, tp); break;
        case BL_FLOAT32: o = asof_typed<float>(l, r, gp, strategy, allow_eq != 0, tp); break;
        default: o = asof_typed<double>(l, r, gp, strategy, allow_eq != 0, tp); break;
    }
    export_column(o, out_location, out_right_idx);
    BL_CATCH
}

}  // extern "C"
