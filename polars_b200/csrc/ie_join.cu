// ie_join.cu — inequality join on the device: every (left row, right row) pair that one or two `<` / `<=` / `>` / `>=`
// predicates accept, as an inner or a left join.
//
// Reference (paths relative to the reference checkout's crates/): the IEJoin arm of _join_impl polars-ops/src/frame/join/mod.rs:243-270,
// piecewise_merge_join_tuples (one predicate) iejoin/mod.rs:667-799, iejoin_tuples (two predicates, Khayyat et al.'s bit-array
// sweep) :572-665, append_unmatched_left (left join) :232-265.
//
// Rule: (i, j) is a pair iff left_on[k][i] op[k] right_on[k][j] for every predicate k, compared in the total order (NaN greatest
// and equal to itself, -0.0 == +0.0: the order of sort_value_key), and every predicate column is valid in both rows.
//
// Plan (DESIGN.md §11):
//   x-order          the live right rows (every predicate column valid), stable-sorted by the first predicate: op_arg_sort
//                    with the live bitmap as validity, the non-live rows sliced off the front.  XS = their keys.  A left key
//                    selects a prefix or a suffix of it (one binary search).
//   tree             two predicates only.  Q[p] = the position of x-position p's row in the stable y-order (keys YS).  Level l
//                    holds every aligned block of 2^l x-positions (the last one truncated) sorted by Q, as Q and right row in two
//                    level-major arrays: one stable sort_pairs_u32 of the y-order on the block id p >> l per level.  A left row's
//                    x-range splits into at most one block per level, and its y-range (a prefix or suffix of Q) is one run of
//                    each block, found by a binary search on Q.
//   k_ie_count       one warp per left row, one lane per level: the row's runs; per-CTA exclusive offsets of the counts
//                    (a left join counts an unmatched row as 1); exclusive_scan_u64 over the CTA sums.
//   k_ie_emit        one warp per IE_WSLOTS output slots: the owner row of a slot by binary search over the offsets, the row's
//                    runs again, coalesced stores of (i, right row); a left join's validity words from the same warp.
// Output order: grouped by left row, left rows ascending; inside a row, run by run (level 0 first), each run in Q order.
#include <algorithm>
#include <vector>

#include "common.cuh"
#include "dev_utils.cuh"
#include "sort_keys.cuh"

namespace plb {

constexpr int IE_THREADS = 256, IE_WARPS = IE_THREADS / 32;
constexpr int IE_CROWS = IE_THREADS;       // left rows per k_ie_count CTA
constexpr int IE_WSLOTS = 512;             // output slots per k_ie_emit warp (a multiple of 32: no validity word is shared)
constexpr unsigned IE_FULL = 0xffffffffu;

struct IeArgs {
    const void* lx; const void* ly; int dtx, dty;      // left predicate columns (ly: two predicates only)
    const uint32_t* lvalid; int64_t nl;                // AND of the left predicate validities (null: no nulls)
    const uint64_t* XS; const uint64_t* YS; int64_t m; // live right keys in x-order / y-order
    int op1, op2, n_pred, levels;                      // levels: 0 when m == 0; one predicate: 1
    const uint32_t* lvQ;                               // levels x m, level-major: Q of each tree entry (two predicates)
    const uint32_t* lvRow;                             // levels x m: right row of each entry (one predicate: the x-order)
};

// first p in [a, b) with K[p] > k (upper) or K[p] >= k (lower); b when there is none
template <typename K> __device__ __forceinline__ int64_t ie_bound(const K* __restrict__ keys, int64_t a, int64_t b, K k, bool upper) {
    while (a < b) {
        const int64_t mid = a + ((b - a) >> 1);
        const K km = keys[mid];
        if (upper ? km <= k : km < k) a = mid + 1; else b = mid;
    }
    return a;
}

// [a, b): the positions of an ascending key array of length m whose keys r satisfy `v op r`
__device__ __forceinline__ void ie_range(const uint64_t* __restrict__ keys, int64_t m, uint64_t v, int op, int64_t& a, int64_t& b) {
    switch (op) {
        case BL_IE_LT: a = ie_bound<uint64_t>(keys, 0, m, v, true); b = m; break;      // r > v
        case BL_IE_LE: a = ie_bound<uint64_t>(keys, 0, m, v, false); b = m; break;     // r >= v
        case BL_IE_GT: a = 0; b = ie_bound<uint64_t>(keys, 0, m, v, false); break;     // r < v
        default: a = 0; b = ie_bound<uint64_t>(keys, 0, m, v, true); break;            // r <= v
    }
}

// Called by a whole warp for left row i (warp-uniform): lane l's run [lo, hi) of row i's matches in the level-major arrays
// (lo == hi: none).  Lane 0 finds the x-range, lane 1 the y-range; lane l then takes the level-l block of the x-range, if any.
//   x-range [0, xb)  level l contributes when bit l of xb is set: the block [xb >> (l+1) << (l+1), + 2^l)
//   x-range [xa, m)  s = xa rounded up to a multiple of 2^l; level l contributes when s / 2^l is odd and s < m: [s, min(s + 2^l, m))
__device__ __forceinline__ void ie_run(const IeArgs& t, int64_t i, unsigned lane, int64_t& lo, int64_t& hi) {
    lo = hi = 0;
    const bool ok = i < t.nl && t.levels > 0 && (t.lvalid == nullptr || bit_get(t.lvalid, i));
    int64_t a = 0, b = 0;
    if (ok && (lane == 0 || (lane == 1 && t.n_pred == 2))) {
        if (lane == 0) ie_range(t.XS, t.m, sort_value_key(t.lx, i, t.dtx), t.op1, a, b);
        else ie_range(t.YS, t.m, sort_value_key(t.ly, i, t.dty), t.op2, a, b);
    }
    const int64_t xa = __shfl_sync(IE_FULL, a, 0), xb = __shfl_sync(IE_FULL, b, 0);
    const int64_t qa = __shfl_sync(IE_FULL, a, 1), qb = __shfl_sync(IE_FULL, b, 1);
    if (!ok || (int)lane >= t.levels) return;
    if (t.n_pred == 1) { lo = xa; hi = xb; return; }       // levels == 1: lane 0 only
    const int l = (int)lane;
    const int64_t w = (int64_t)1 << l;
    int64_t s, e;
    if (xa == 0) {
        if (!((xb >> l) & 1)) return;
        s = (xb >> (l + 1)) << (l + 1); e = s + w;
    } else {
        s = ((xa + w - 1) >> l) << l;
        if (!((s >> l) & 1) || s >= t.m) return;
        e = min(s + w, t.m);
    }
    const int64_t base = (int64_t)l * t.m;
    const uint32_t* Q = t.lvQ + base;
    const int64_t rlo = qa > 0 ? ie_bound<uint32_t>(Q, s, e, (uint32_t)qa, false) : s;
    const int64_t rhi = qb < t.m ? ie_bound<uint32_t>(Q, rlo, e, (uint32_t)qb, false) : e;
    lo = base + rlo; hi = base + rhi;
}

__device__ __forceinline__ uint64_t warp_sum_u64(uint64_t v) {
    for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(IE_FULL, v, o);
    return v;
}

// one warp per left row: off[i] = the row's first output slot relative to its CTA's IE_CROWS rows, bsum[cta] = their total
__global__ void __launch_bounds__(IE_THREADS) k_ie_count(const IeArgs t, int left_join, uint64_t* __restrict__ off, uint64_t* __restrict__ bsum) {
    __shared__ uint64_t s_c[IE_CROWS];
    __shared__ uint64_t s_w[IE_WARPS];
    const unsigned lane = lane_id(), warp = threadIdx.x >> 5;
    const int64_t base = (int64_t)blockIdx.x * IE_CROWS;
    for (int k = warp; k < IE_CROWS; k += IE_WARPS) {
        const int64_t i = base + k;
        int64_t lo, hi;
        ie_run(t, i, lane, lo, hi);
        const uint64_t c = warp_sum_u64((uint64_t)(hi - lo));
        if (lane == 0) s_c[k] = i < t.nl ? ((left_join && c == 0) ? 1 : c) : 0;
    }
    __syncthreads();
    const uint64_t v = s_c[threadIdx.x];
    uint64_t x = v;
    for (int o = 1; o < 32; o <<= 1) { const uint64_t y = __shfl_up_sync(IE_FULL, x, o); if (lane >= (unsigned)o) x += y; }
    if (lane == 31) s_w[warp] = x;
    __syncthreads();
    uint64_t before = 0, all = 0;
    for (int w = 0; w < IE_WARPS; w++) { if (w < (int)warp) before += s_w[w]; all += s_w[w]; }
    const int64_t i = base + threadIdx.x;
    if (i < t.nl) off[i] = before + x - v;
    if (threadIdx.x == 0) bsum[blockIdx.x] = all;
}

// the first output slot of left row r (r < nl)
__device__ __forceinline__ uint64_t ie_start(const uint64_t* __restrict__ off, const uint64_t* __restrict__ bbase, int64_t r) {
    return bbase[r / IE_CROWS] + off[r];
}

// one warp per IE_WSLOTS output slots [u0, u1): out_l / out_r, and out_valid (left join) for those slots
__global__ void __launch_bounds__(IE_THREADS) k_ie_emit(const IeArgs t, const uint64_t* __restrict__ off, const uint64_t* __restrict__ bbase, uint64_t total,
                                                       uint32_t* __restrict__ out_l, uint32_t* __restrict__ out_r, uint32_t* __restrict__ out_valid) {
    __shared__ uint32_t s_valid[IE_WARPS][IE_WSLOTS / 32];
    const unsigned lane = lane_id(), warp = threadIdx.x >> 5;
    const uint64_t u0 = ((uint64_t)blockIdx.x * IE_WARPS + warp) * IE_WSLOTS;
    if (u0 >= total) return;                               // warp-uniform; only __syncwarp below
    const uint64_t u1 = min(u0 + (uint64_t)IE_WSLOTS, total);
    if (out_valid && lane < IE_WSLOTS / 32) s_valid[warp][lane] = ~0u;
    __syncwarp();
    uint64_t tt = u0;
    while (tt < u1) {
        // owner of slot tt: the last row whose first slot is <= tt (rows before it with the same first slot own none)
        int64_t a = 0, b = t.nl;
        while (a < b) {
            const int64_t mid = a + ((b - a) >> 1);
            if (ie_start(off, bbase, mid) <= tt) a = mid + 1; else b = mid;
        }
        const int64_t r = a - 1;
        const uint64_t rb = ie_start(off, bbase, r);
        const uint64_t re = min(r + 1 < t.nl ? ie_start(off, bbase, r + 1) : total, u1);
        int64_t lo, hi;
        ie_run(t, r, lane, lo, hi);
        // inclusive scan of the run lengths over the lanes: pair j of the row lies in the first lane whose `end` exceeds j
        const uint64_t len = (uint64_t)(hi - lo);
        uint64_t end = len;
        for (int o = 1; o < 32; o <<= 1) { const uint64_t y = __shfl_up_sync(IE_FULL, end, o); if (lane >= (unsigned)o) end += y; }
        const int64_t shift = lo - (int64_t)(end - len);   // tree index of pair j in this lane's run: shift + j
        const bool unmatched = __shfl_sync(IE_FULL, end, 31) == 0;
        for (uint64_t k0 = tt; k0 < re; k0 += 32) {
            const uint64_t k = k0 + lane, j = k - rb;
            int s = 0;
#pragma unroll
            for (int step = 16; step; step >>= 1) { const uint64_t e = __shfl_sync(IE_FULL, end, s + step - 1); if (e <= j) s += step; }
            const int64_t sh = __shfl_sync(IE_FULL, shift, s);
            if (k < re) {
                out_l[k] = (uint32_t)r;
                if (unmatched) {
                    out_r[k] = BL_IDX_NULL;
                    atomicAnd(&s_valid[warp][(k - u0) >> 5], ~(1u << (k & 31)));
                } else {
                    out_r[k] = t.lvRow[sh + (int64_t)j];
                }
            }
        }
        tt = re;
    }
    __syncwarp();
    if (out_valid && lane < IE_WSLOTS / 32) {
        const uint64_t w = (u0 >> 5) + lane;
        if (w * 32 < total) {
            uint32_t v = s_valid[warp][lane];
            if ((w + 1) * 32 > total) v &= (1u << (total & 31)) - 1u;
            out_valid[w] = v;
        }
    }
}

// out[p] = the order key of col[perm[p]]
__global__ void __launch_bounds__(256) k_ie_keys(const void* __restrict__ col, int dtype, const uint32_t* __restrict__ perm, int64_t m, uint64_t* __restrict__ out) {
    for (int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; p < m; p += (int64_t)gridDim.x * blockDim.x) out[p] = sort_value_key(col, perm[p], dtype);
}

// xpos[xperm[p]] = p
__global__ void __launch_bounds__(256) k_ie_xpos(const uint32_t* __restrict__ xperm, int64_t m, uint32_t* __restrict__ xpos) {
    for (int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; p < m; p += (int64_t)gridDim.x * blockDim.x) xpos[xperm[p]] = (uint32_t)p;
}

// the y-order with each entry's block id at one level: keys[q] = xpos[yperm[q]] >> level, vals[q] = q
__global__ void __launch_bounds__(256) k_ie_level_keys(const uint32_t* __restrict__ px, int64_t m, int level, uint32_t* __restrict__ keys, uint32_t* __restrict__ vals) {
    for (int64_t q = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; q < m; q += (int64_t)gridDim.x * blockDim.x) { keys[q] = px[q] >> level; vals[q] = (uint32_t)q; }
}

// px[q] = xpos[yperm[q]]
__global__ void __launch_bounds__(256) k_ie_px(const uint32_t* __restrict__ yperm, const uint32_t* __restrict__ xpos, int64_t m, uint32_t* __restrict__ px) {
    for (int64_t q = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; q < m; q += (int64_t)gridDim.x * blockDim.x) px[q] = xpos[yperm[q]];
}

// rows[k] = yperm[lq[k]]
__global__ void __launch_bounds__(256) k_ie_level_rows(const uint32_t* __restrict__ lq, const uint32_t* __restrict__ yperm, int64_t m, uint32_t* __restrict__ rows) {
    for (int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; k < m; k += (int64_t)gridDim.x * blockDim.x) rows[k] = yperm[lq[k]];
}

// the stable order of the live rows of c by value: a permutation of the m live rows (the non-live ones, sorted first as nulls,
// are sliced off)
static DevPtr ie_live_order(const DevCol& c, const DevPtr& live, int64_t m, DevCol& keep) {
    DevCol k = c;
    k.validity = live; k.null_count = -1;
    keep = op_arg_sort({k}, {0}, -1);
    return keep.values;      // the first c.len - m entries are the non-live rows
}

static DevPtr ie_alloc(size_t bytes, const std::string& what) {
    try {
        return dev_alloc(bytes);
    } catch (const Error& e) {
        if (e.code != BL_ERR_OOM) throw;
        fail(BL_ERR_OOM, "ie_join: " + what + " (" + std::to_string(bytes) + " bytes) does not fit in device memory: " + e.what());
    }
}

static void ie_run_join(const std::vector<DevCol>& L, const std::vector<DevCol>& R, const int32_t* ops, int n_pred, bool left_join, DevCol& out_l, DevCol& out_r) {
    const int64_t nl = L[0].len, nr = R[0].len;
    IeArgs t;
    memset(&t, 0, sizeof t);
    t.lx = L[0].v(); t.dtx = L[0].dtype; t.nl = nl; t.n_pred = n_pred; t.op1 = ops[0];
    if (n_pred == 2) { t.ly = L[1].v(); t.dty = L[1].dtype; t.op2 = ops[1]; }
    DevPtr lvalid = bitmap_and(L[0].vm(), n_pred == 2 ? L[1].vm() : nullptr, nullptr, nl);
    t.lvalid = as<uint32_t>(lvalid);
    // the live right rows in x-order (and y-order)
    DevPtr live = bitmap_and(R[0].vm(), n_pred == 2 ? R[1].vm() : nullptr, nullptr, nr);
    const int64_t m = live ? bitmap_popcount(as<uint32_t>(live), nr) : nr;
    t.m = m;
    DevCol xkeep, ykeep;
    DevPtr XS, YS, xpos, px, lvQ, lvRow;
    const uint32_t *xperm = nullptr, *yperm = nullptr;
    if (m > 0) {
        xperm = as<uint32_t>(ie_live_order(R[0], live, m, xkeep)) + (nr - m);
        XS = dev_alloc((size_t)m * 8);
        PLB_LAUNCH("ie_keys", k_ie_keys, grid_for(m, 256), 256, 0, R[0].v(), R[0].dtype, xperm, m, as<uint64_t>(XS));
        t.XS = as<uint64_t>(XS);
        if (n_pred == 1) {
            t.levels = 1;
            t.lvRow = xperm;
        } else {
            int levels = 1;
            while (levels < 64 && ((int64_t)1 << (levels - 1)) < m) levels++;
            PLB_REQUIRE(levels <= 32, BL_ERR_OOM, "ie_join: " + std::to_string(m) + " live right rows need a merge-sort tree of " + std::to_string(levels) +
                                                  " levels (at most 32, i.e. 2^31 rows, with two predicates)");
            t.levels = levels;
            yperm = as<uint32_t>(ie_live_order(R[1], live, m, ykeep)) + (nr - m);
            YS = dev_alloc((size_t)m * 8);
            PLB_LAUNCH("ie_keys", k_ie_keys, grid_for(m, 256), 256, 0, R[1].v(), R[1].dtype, yperm, m, as<uint64_t>(YS));
            t.YS = as<uint64_t>(YS);
            xpos = dev_alloc((size_t)nr * 4);
            px = dev_alloc((size_t)m * 4);
            PLB_LAUNCH("ie_xpos", k_ie_xpos, grid_for(m, 256), 256, 0, xperm, m, as<uint32_t>(xpos));
            PLB_LAUNCH("ie_px", k_ie_px, grid_for(m, 256), 256, 0, yperm, as<uint32_t>(xpos), m, as<uint32_t>(px));
            xpos.reset();
            const std::string tree = "the merge-sort tree of " + std::to_string(levels) + " levels x " + std::to_string(m) + " live right rows";
            lvQ = ie_alloc((size_t)levels * m * 4, tree);
            lvRow = ie_alloc((size_t)levels * m * 4, tree);
            DevPtr keys = dev_alloc((size_t)m * 4);
            for (int l = 0; l < levels; l++) {
                uint32_t* q = as<uint32_t>(lvQ) + (int64_t)l * m;
                PLB_LAUNCH("ie_level_keys", k_ie_level_keys, grid_for(m, 256), 256, 0, as<uint32_t>(px), m, l, as<uint32_t>(keys), q);
                sort_pairs_u32(as<uint32_t>(keys), q, m, bits_for((uint64_t)(m - 1) >> l));
                PLB_LAUNCH("ie_level_rows", k_ie_level_rows, grid_for(m, 256), 256, 0, q, yperm, m, as<uint32_t>(lvRow) + (int64_t)l * m);
            }
            t.lvQ = as<uint32_t>(lvQ); t.lvRow = as<uint32_t>(lvRow);
        }
    }
    // counts -> offsets -> the pair count
    const int64_t nblk = std::max<int64_t>((nl + IE_CROWS - 1) / IE_CROWS, 1);
    DevPtr off = dev_alloc((size_t)std::max<int64_t>(nl, 1) * 8), bsum = dev_alloc((size_t)nblk * 8), bbase = dev_alloc((size_t)(nblk + 1) * 8);
    uint64_t total = 0;
    if (nl > 0) {
        PLB_LAUNCH("ie_count", k_ie_count, (int)nblk, IE_THREADS, 0, t, left_join ? 1 : 0, as<uint64_t>(off), as<uint64_t>(bsum));
        exclusive_scan_u64(as<uint64_t>(bsum), as<uint64_t>(bbase), nblk, as<uint64_t>(bbase) + nblk);
        total = read_scalar(as<uint64_t>(bbase) + nblk);
    }
    const std::string pairs = "the output of " + std::to_string(total) + " pairs";
    out_l = DevCol(); out_r = DevCol();
    out_l.dtype = out_r.dtype = BL_UINT32;
    out_l.len = out_r.len = (int64_t)total;
    out_l.null_count = 0; out_r.null_count = left_join ? -1 : 0;
    out_l.values = ie_alloc((size_t)total * 4 + 16, pairs);
    out_r.values = ie_alloc((size_t)total * 4 + 16, pairs);
    if (left_join) out_r.validity = ie_alloc(bitmap_bytes((int64_t)total) + 16, pairs);
    if (total == 0) return;
    const uint64_t slots_per_cta = (uint64_t)IE_WARPS * IE_WSLOTS;
    const uint64_t grid = (total + slots_per_cta - 1) / slots_per_cta;
    PLB_REQUIRE(grid <= 0x7FFFFFFFull, BL_ERR_OOM, "ie_join: " + pairs + " exceed one launch");
    PLB_LAUNCH("ie_emit", k_ie_emit, (int)grid, IE_THREADS, 0, t, as<uint64_t>(off), as<uint64_t>(bbase), total, as<uint32_t>(out_l.values), as<uint32_t>(out_r.values),
               left_join ? as<uint32_t>(out_r.validity) : nullptr);
}

}  // namespace plb

// ================================================================================ C ABI
using namespace plb;
extern "C" {

bl_status bl_ie_join(const bl_column* left_on, const bl_column* right_on, const int32_t* ops, int32_t n_pred, int32_t how, int32_t out_location,
                     bl_column* out_left_idx, bl_column* out_right_idx) {
    BL_TRY
    PLB_REQUIRE(left_on && right_on && ops && out_left_idx && out_right_idx, BL_ERR_INVALID, "ie_join: null argument");
    PLB_REQUIRE(n_pred == 1 || n_pred == 2, BL_ERR_INVALID, "ie_join: n_pred must be 1 or 2, got " + std::to_string(n_pred));
    PLB_REQUIRE(how == BL_JOIN_INNER || how == BL_JOIN_LEFT, BL_ERR_INVALID, "ie_join: how must be BL_JOIN_INNER or BL_JOIN_LEFT, got " + std::to_string(how));
    for (int k = 0; k < n_pred; k++) {
        const std::string w = "ie_join: predicate " + std::to_string(k);
        PLB_REQUIRE(ops[k] >= BL_IE_LT && ops[k] <= BL_IE_GE, BL_ERR_INVALID, w + ": unknown operator " + std::to_string(ops[k]));
        const int dl = left_on[k].dtype, dr = right_on[k].dtype;
        PLB_REQUIRE(dl >= BL_INT8 && dl <= BL_BOOL && dr >= BL_INT8 && dr <= BL_BOOL, BL_ERR_INVALID, w + ": unknown dtype");
        PLB_REQUIRE(dl == dr, BL_ERR_DTYPE, w + ": mismatching dtypes " + dtype_name(dl) + " and " + dtype_name(dr));
        PLB_REQUIRE(dl != BL_BOOL, BL_ERR_UNSUPPORTED, w + ": Boolean columns are outside the hot path");
        PLB_REQUIRE(left_on[k].length == left_on[0].length && right_on[k].length == right_on[0].length, BL_ERR_INVALID,
                    w + ": length differs from the first predicate's column on the same side");
    }
    PLB_REQUIRE(left_on[0].length <= 0xFFFFFFFEll && right_on[0].length <= 0xFFFFFFFEll, BL_ERR_UNSUPPORTED, "ie_join: more than 2^32 - 2 rows on one side (IdxSize is u32)");
    std::vector<DevCol> L, R;
    for (int k = 0; k < n_pred; k++) { L.push_back(import_column(&left_on[k], 1)); R.push_back(import_column(&right_on[k], 1)); }
    DevCol ol, orr;
    ie_run_join(L, R, ops, n_pred, how == BL_JOIN_LEFT, ol, orr);
    { std::vector<DevCol> both{ol, orr}; bl_column o[2]; export_many(both, out_location, o); *out_left_idx = o[0]; *out_right_idx = o[1]; }
    BL_CATCH
}

}  // extern "C"
