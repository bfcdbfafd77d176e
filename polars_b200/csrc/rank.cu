// rank.cu — Expr.rank(method, descending, seed), plain or .over(partition_by, order_by) (polars-ops/src/series/ops/rank.rs:61-188).
//
// Plan (DESIGN.md §15), per op:
//   1. order       op_arg_sort of (partition id, value with BL_SORT_NULLS_LAST [+ DESCENDING], tie key): the reference's stable
//                  arg_sort per partition (rank.rs:101-107).  The tie key is the order_by key for ORDINAL, the keyed bijection
//                  k_rank_random_key for RANDOM, and nothing otherwise (ties do not change the other methods).
//   2. k_rank_heads   one pass over the sorted positions: the value's canonical key (sort_value_key: exactly the tot_eq
//                  classes), its validity and partition id at perm[i]; the left neighbour comes through the warp's registers
//                  (one extra load per 256 positions).  Writes three bitmaps over the positions (run heads, partition heads,
//                  validity) and each tile's (runs, partitions) count.
//   3. exclusive_scan_u64 of the tile counts: the global run / partition number of every tile's first head.
//   4. k_rank_starts  (MIN / MAX / AVERAGE, and any partitioned rank) run r's first position start[r], partition q's first
//                  position seg_pos[q] and first run seg_run[q]; reads only the bitmaps.
//   5. k_rank_out     every position's run r and partition q from the bitmaps, its rank from start[r], start[r + 1],
//                  seg_pos[q] and seg_run[q], scattered to out[perm[i]] (4 or 8 bytes per row).  The output validity is the
//                  input validity.
// A string DENSE rank without partitions is op_string_rank itself.
#include <algorithm>

#include "common.cuh"
#include "dev_utils.cuh"
#include "sort_keys.cuh"
#include "strings.cuh"

namespace plb {

constexpr int RK_THREADS = 256, RK_WARP_WORDS = 8, RK_TILE_WORDS = (RK_THREADS / 32) * RK_WARP_WORDS, RK_TILE = RK_TILE_WORDS * 32;

// murmur3's finaliser, a bijection of u32
__device__ __forceinline__ uint32_t fmix32(uint32_t h) {
    h ^= h >> 16; h *= 0x85ebca6bu; h ^= h >> 13; h *= 0xc2b2ae35u; h ^= h >> 16;
    return h;
}
// RANDOM's tie key: a keyed bijection of the row index, so no two rows tie on it and ORDINAL over it permutes each run
__global__ void __launch_bounds__(256) k_rank_random_key(int64_t n, uint32_t seed_lo, uint32_t seed_hi, uint32_t* __restrict__ out) {
    for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < n; r += (int64_t)gridDim.x * blockDim.x)
        out[r] = fmix32(fmix32((uint32_t)r ^ seed_lo) + seed_hi);
}

struct RankArgs {
    const void* values; const uint32_t* validity; int dtype; const uint32_t* gid; const uint32_t* perm; int64_t n; int need_runs;
    uint32_t* run_bm; uint32_t* seg_bm; uint32_t* valid_bm; unsigned long long* tile_cnt;      // heads
    const unsigned long long* tile_off;                                                          // starts / out: exclusive tile offsets, [ntiles] = totals
    uint32_t* start; uint32_t* seg_pos; uint32_t* seg_run;
    int method; void* out;
};

// k_rank_heads: warp w of tile t owns the RK_WARP_WORDS words t * RK_TILE_WORDS + w * RK_WARP_WORDS + j, one position per lane
__global__ void __launch_bounds__(RK_THREADS) k_rank_heads(const __grid_constant__ RankArgs a) {
    __shared__ unsigned long long s_cnt[RK_THREADS / 32];
    const unsigned lane = lane_id(), warp = threadIdx.x >> 5;
    const int64_t n = a.n, ntiles = (n + RK_TILE - 1) / RK_TILE;
    for (int64_t t = blockIdx.x; t < ntiles; t += gridDim.x) {
        const int64_t w0 = t * RK_TILE_WORDS + (int64_t)warp * RK_WARP_WORDS;
        uint64_t pkey = 0; uint32_t pg = 0; bool pv = false;      // the previous position (lane 31 of the previous word)
        if (w0 > 0 && w0 * 32 < n && lane == 0) {
            const int64_t r = a.perm[w0 * 32 - 1];
            pv = a.validity == nullptr || bit_get(a.validity, r);
            if (a.need_runs && pv) pkey = sort_value_key(a.values, r, a.dtype);
            if (a.gid) pg = __ldg(a.gid + r);
        }
        uint32_t runs = 0, segs = 0;
#pragma unroll 2
        for (int j = 0; j < RK_WARP_WORDS; j++) {
            const int64_t word = w0 + j, i = word * 32 + lane;
            if (word * 32 >= n) break;
            uint64_t key = 0; uint32_t g = 0; bool v = false;
            const bool in = i < n;
            if (in) {
                const int64_t r = __ldg(a.perm + i);
                v = a.validity == nullptr || bit_get(a.validity, r);
                if (a.need_runs && v) key = sort_value_key(a.values, r, a.dtype);
                if (a.gid) g = __ldg(a.gid + r);
            }
            uint64_t lkey = __shfl_up_sync(0xffffffffu, key, 1);
            uint32_t lg = __shfl_up_sync(0xffffffffu, g, 1);
            bool lv = __shfl_up_sync(0xffffffffu, (int)v, 1) != 0;
            if (lane == 0) { lkey = pkey; lg = pg; lv = pv; }
            pkey = __shfl_sync(0xffffffffu, key, 31); pg = __shfl_sync(0xffffffffu, g, 31); pv = __shfl_sync(0xffffffffu, (int)v, 31) != 0;
            const bool seg_head = in && (i == 0 || g != lg);
            const bool run_head = in && (seg_head || (a.need_runs && (v != lv || (v && key != lkey))));
            const uint32_t rw = __ballot_sync(0xffffffffu, run_head), sw = __ballot_sync(0xffffffffu, seg_head), vw = __ballot_sync(0xffffffffu, v);
            if (lane == 0) {
                a.run_bm[word] = rw;
                if (a.seg_bm) a.seg_bm[word] = sw;
                if (a.valid_bm) a.valid_bm[word] = vw;
            }
            runs += __popc(rw); segs += __popc(sw);
        }
        if (lane == 0) s_cnt[warp] = (unsigned long long)runs | ((unsigned long long)segs << 32);
        __syncthreads();
        if (threadIdx.x == 0) {
            unsigned long long c = 0;
            for (int k = 0; k < RK_THREADS / 32; k++) c += s_cnt[k];
            a.tile_cnt[t] = c;
        }
        __syncthreads();
    }
}

// The exclusive (run, partition) head counts before each of this warp's words: lane j < RK_WARP_WORDS holds word j's bitmap
// words; returns them through the shuffles of the caller.  One __syncthreads pair per tile.
struct WordPrefix { uint32_t rw, sw; uint64_t r0, q0; };
__device__ __forceinline__ WordPrefix word_prefix(const RankArgs& a, int64_t t, unsigned warp, unsigned lane, unsigned long long* s_w) {
    const int64_t nwords = (a.n + 31) / 32;
    const int64_t word = t * RK_TILE_WORDS + (int64_t)warp * RK_WARP_WORDS + lane;
    uint32_t rw = 0, sw = 0;
    if (lane < RK_WARP_WORDS && word < nwords) {
        rw = a.run_bm[word];
        sw = a.seg_bm ? a.seg_bm[word] : (word == 0 ? 1u : 0u);
    }
    unsigned long long c = (unsigned long long)__popc(rw) | ((unsigned long long)__popc(sw) << 32), inc = c;
#pragma unroll
    for (int o = 1; o < RK_WARP_WORDS; o <<= 1) {
        const unsigned long long y = __shfl_up_sync(0xffffffffu, inc, o);
        if (lane >= (unsigned)o) inc += y;
    }
    if (lane == RK_WARP_WORDS - 1) s_w[warp] = inc;
    __syncthreads();
    unsigned long long base = a.tile_off[t];
    for (unsigned k = 0; k < warp; k++) base += s_w[k];
    __syncthreads();      // s_w is rewritten by the next tile
    const unsigned long long ex = base + inc - c;
    return WordPrefix{rw, sw, ex & 0xFFFFFFFFull, ex >> 32};
}

__global__ void __launch_bounds__(RK_THREADS) k_rank_starts(const __grid_constant__ RankArgs a) {
    __shared__ unsigned long long s_w[RK_THREADS / 32];
    const unsigned lane = lane_id(), warp = threadIdx.x >> 5;
    const int64_t n = a.n, ntiles = (n + RK_TILE - 1) / RK_TILE;
    for (int64_t t = blockIdx.x; t < ntiles; t += gridDim.x) {
        const WordPrefix wp = word_prefix(a, t, warp, lane, s_w);
        for (int j = 0; j < RK_WARP_WORDS; j++) {
            const int64_t word = t * RK_TILE_WORDS + (int64_t)warp * RK_WARP_WORDS + j, i = word * 32 + lane;
            if (word * 32 >= n) break;      // warp-uniform: every lane takes part in the shuffles below
            const uint32_t rw = __shfl_sync(0xffffffffu, wp.rw, j), sw = __shfl_sync(0xffffffffu, wp.sw, j);
            const uint64_t r0 = __shfl_sync(0xffffffffu, wp.r0, j), q0 = __shfl_sync(0xffffffffu, wp.q0, j);
            if (i >= n) continue;
            const uint64_t r = r0 + __popc(rw & lanemask_lt());
            if (a.start && ((rw >> lane) & 1)) a.start[r] = (uint32_t)i;
            if ((sw >> lane) & 1) {
                const uint64_t q = q0 + __popc(sw & lanemask_lt());
                if (a.seg_pos) a.seg_pos[q] = (uint32_t)i;
                if (a.seg_run) a.seg_run[q] = (uint32_t)r;
            }
        }
    }
}

__global__ void __launch_bounds__(RK_THREADS) k_rank_out(const __grid_constant__ RankArgs a) {
    __shared__ unsigned long long s_w[RK_THREADS / 32];
    const unsigned lane = lane_id(), warp = threadIdx.x >> 5;
    const int64_t n = a.n, ntiles = (n + RK_TILE - 1) / RK_TILE;
    const uint64_t n_runs = a.tile_off[ntiles] & 0xFFFFFFFFull;
    for (int64_t t = blockIdx.x; t < ntiles; t += gridDim.x) {
        const WordPrefix wp = word_prefix(a, t, warp, lane, s_w);
        for (int j = 0; j < RK_WARP_WORDS; j++) {
            const int64_t word = t * RK_TILE_WORDS + (int64_t)warp * RK_WARP_WORDS + j, i = word * 32 + lane;
            if (word * 32 >= n) break;
            const uint32_t rw = __shfl_sync(0xffffffffu, wp.rw, j), sw = __shfl_sync(0xffffffffu, wp.sw, j);
            const uint64_t r0 = __shfl_sync(0xffffffffu, wp.r0, j), q0 = __shfl_sync(0xffffffffu, wp.q0, j);
            if (i >= n) continue;
            const unsigned le = lanemask_lt() | (1u << lane);
            const uint64_t r = r0 + __popc(rw & le) - 1;      // the run holding position i
            const uint64_t q = q0 + __popc(sw & le) - 1;      // its partition
            const bool v = a.valid_bm == nullptr || ((a.valid_bm[word] >> lane) & 1);
            const uint32_t row = __ldg(a.perm + i);
            const uint64_t S = a.seg_pos ? a.seg_pos[q] : 0;
            uint64_t rank = 0;
            double avg = 0;
            if (v) {
                const int m = a.method;
                if (m == BL_RANK_ORDINAL || m == BL_RANK_RANDOM) rank = (uint64_t)i - S + 1;
                else if (m == BL_RANK_DENSE) rank = r - (a.seg_run ? a.seg_run[q] : 0) + 1;
                else {
                    const uint64_t s = (uint64_t)a.start[r] - S + 1, e = (r + 1 < n_runs ? (uint64_t)a.start[r + 1] : (uint64_t)n) - S;
                    rank = m == BL_RANK_MIN ? s : e;
                    avg = 0.5 * ((double)s + (double)e);      // rank.rs:145-149; exact: both are below 2^32
                }
            }
            if (a.method == BL_RANK_AVERAGE) reinterpret_cast<double*>(a.out)[row] = avg;
            else reinterpret_cast<uint32_t*>(a.out)[row] = (uint32_t)rank;
        }
    }
}

// ---------------------------------------------------------------------------------------------------- host side
int rank_dtype(int method) { return method == BL_RANK_AVERAGE ? BL_FLOAT64 : BL_UINT32; }

void check_rank_op(int method) {
    PLB_REQUIRE(method >= BL_RANK_AVERAGE && method <= BL_RANK_RANDOM, BL_ERR_INVALID, "rank: unknown method " + std::to_string(method));
}

// the rank of one value column (strings arrive as their ascending dense rank) over the partition ids gid (none: one partition)
static DevCol rank_one(const RankOp& op, const DevCol& v, const DevCol* gid, const DevCol* order_key, int order_flags) {
    const int64_t n = v.len;
    DevCol out = make_col(rank_dtype(op.method), n, false);
    out.validity = v.validity; out.null_count = v.null_count;
    if (n == 0) return out;
    std::vector<DevCol> keys;
    std::vector<int> flags;
    if (gid) { keys.push_back(*gid); flags.push_back(0); }
    keys.push_back(v); flags.push_back(BL_SORT_NULLS_LAST | (op.descending ? BL_SORT_DESCENDING : 0));
    if (op.method == BL_RANK_ORDINAL && order_key) { keys.push_back(*order_key); flags.push_back(order_flags); }
    if (op.method == BL_RANK_RANDOM) {
        DevCol rk = make_col(BL_UINT32, n, false);
        rk.null_count = 0;
        PLB_LAUNCH("rank_random_key", k_rank_random_key, grid_for(n, 256), 256, 0, n, (uint32_t)op.seed, (uint32_t)(op.seed >> 32), as<uint32_t>(rk.values));
        keys.push_back(rk); flags.push_back(0);
    }
    const DevCol perm = op_arg_sort(keys, flags, -1);

    const bool runs = op.method == BL_RANK_MIN || op.method == BL_RANK_MAX || op.method == BL_RANK_AVERAGE || op.method == BL_RANK_DENSE;
    const bool need_start = runs && op.method != BL_RANK_DENSE;
    const int64_t nwords = (n + 31) / 32, ntiles = (n + RK_TILE - 1) / RK_TILE;
    DevPtr run_bm = dev_alloc((size_t)nwords * 4), seg_bm, valid_bm, cnt = dev_alloc((size_t)ntiles * 8), off = dev_alloc((size_t)ntiles * 8 + 8);
    DevPtr start, seg_pos, seg_run;
    if (gid) { seg_bm = dev_alloc((size_t)nwords * 4); seg_pos = dev_alloc((size_t)n * 4); }
    if (gid && op.method == BL_RANK_DENSE) seg_run = dev_alloc((size_t)n * 4);
    if (v.validity) valid_bm = dev_alloc((size_t)nwords * 4);
    if (need_start) start = dev_alloc((size_t)n * 4);
    RankArgs a;
    memset(&a, 0, sizeof a);
    a.values = v.v(); a.validity = v.vm(); a.dtype = v.dtype; a.gid = gid ? as<uint32_t>(gid->values) : nullptr;
    a.perm = as<uint32_t>(perm.values); a.n = n; a.need_runs = runs ? 1 : 0;
    a.run_bm = as<uint32_t>(run_bm); a.seg_bm = as<uint32_t>(seg_bm); a.valid_bm = as<uint32_t>(valid_bm);
    a.tile_cnt = as<unsigned long long>(cnt); a.tile_off = as<unsigned long long>(off);
    a.start = as<uint32_t>(start); a.seg_pos = as<uint32_t>(seg_pos); a.seg_run = as<uint32_t>(seg_run);
    a.method = op.method; a.out = out.values->p;
    const int grid = (int)std::min<int64_t>(ntiles, (int64_t)ctx().sm_count * 8);
    PLB_LAUNCH("rank_heads", k_rank_heads, grid, RK_THREADS, 0, a);
    exclusive_scan_u64(as<uint64_t>(cnt), as<uint64_t>(off), ntiles, as<uint64_t>(off) + ntiles);
    if (start || seg_pos) PLB_LAUNCH("rank_starts", k_rank_starts, grid, RK_THREADS, 0, a);
    PLB_LAUNCH("rank_out", k_rank_out, grid, RK_THREADS, 0, a);
    return out;
}

static void check_rank_rows(int64_t n, bool grouped) {
    PLB_REQUIRE(!grouped || n <= 0x7FFFFFFFll, BL_ERR_UNSUPPORTED, "rank: more than 2^31 - 1 rows with partitions or order_by");
    PLB_REQUIRE(n <= 0xFFFFFFFFll, BL_ERR_UNSUPPORTED, "rank: more than 2^32 - 1 rows (IdxSize is u32)");
}

std::vector<DevCol> op_rank(const std::vector<DevCol>& partition_by, const DevCol* order_key, int order_flags, const std::vector<RankOp>& ops, int64_t n) {
    for (auto& op : ops) PLB_REQUIRE(op.values->len == n, BL_ERR_INVALID, "rank: value columns differ in length");
    for (auto& k : partition_by) PLB_REQUIRE(k.len == n, BL_ERR_INVALID, "rank: partition columns differ in length");
    if (order_key) PLB_REQUIRE(order_key->len == n, BL_ERR_INVALID, "rank: the order_by column differs in length");
    check_rank_rows(n, !partition_by.empty() || order_key);
    DevCol gid;
    if (!partition_by.empty() && n > 0) gid = partition_ids(partition_by, n);
    std::vector<DevCol> outs;
    for (auto& op : ops) outs.push_back(rank_one(op, *op.values, gid.values ? &gid : nullptr, order_key, order_flags));
    return outs;
}

}  // namespace plb

// ================================================================================ C ABI
using namespace plb;
extern "C" {

bl_status bl_rank(const bl_sort_key* partition_by, int32_t n_partition_by, const bl_sort_key* order_by, const bl_rank_op* ops, int32_t n_ops,
                  int32_t out_location, bl_column* outs) {
    BL_TRY
    PLB_REQUIRE(n_ops >= 1 && ops && outs, BL_ERR_INVALID, "rank: no operations or no outputs");
    int64_t n = -1;
    check_window_keys("rank", partition_by, n_partition_by, order_by, n);
    for (int i = 0; i < n_ops; i++) {
        const bl_sort_key* k = ops[i].values;
        const std::string w = "value column " + std::to_string(i);
        PLB_REQUIRE(k != nullptr, BL_ERR_INVALID, "rank: operation " + std::to_string(i) + " has no value column");
        check_rank_op(ops[i].method);
        PLB_REQUIRE((k->column != nullptr) != (k->strings != nullptr), BL_ERR_INVALID, "rank: " + w + " must set exactly one of `column` and `strings`");
        PLB_REQUIRE(k->strings == nullptr || k->n_chunks >= 1, BL_ERR_INVALID, "rank: " + w + ": a string column without chunks");
        PLB_REQUIRE(k->flags == 0, BL_ERR_INVALID, "rank: " + w + ": flags must be 0 (descending is the op's)");
        PLB_REQUIRE(k->strings || k->column->dtype <= BL_BOOL, BL_ERR_INVALID, "rank: " + w + ": unknown dtype");
        int64_t len = 0;
        if (k->column) len = k->column->length;
        else for (int j = 0; j < k->n_chunks; j++) len += k->strings[j].length;
        set_window_len("rank", len, w, n);
    }
    check_rank_rows(n, n_partition_by > 0 || order_by);      // before any column is read
    std::vector<DevCol> parts;
    for (int i = 0; i < n_partition_by; i++) parts.push_back(import_key(partition_by[i], true));
    DevCol okey;
    if (order_by) okey = import_key(*order_by, false);
    std::vector<DevCol> vals(n_ops), res(n_ops);
    std::vector<RankOp> v;
    std::vector<int> at;
    for (int i = 0; i < n_ops; i++) {
        const bl_sort_key& k = *ops[i].values;
        if (k.strings && ops[i].method == BL_RANK_DENSE && n_partition_by == 0) {      // bl_string_rank's own answer
            res[i] = op_string_rank(import_string(k.strings, k.n_chunks), ops[i].descending != 0, nullptr);
            continue;
        }
        vals[i] = k.column ? import_column(k.column, 1) : op_string_rank(import_string(k.strings, k.n_chunks), false, nullptr);
        RankOp o;
        o.method = ops[i].method; o.descending = ops[i].descending != 0; o.seed = ops[i].seed; o.values = &vals[i];
        v.push_back(o); at.push_back(i);
    }
    std::vector<DevCol> r = op_rank(parts, order_by ? &okey : nullptr, order_by ? order_by->flags : 0, v, n);
    for (size_t j = 0; j < at.size(); j++) res[at[j]] = r[j];
    export_many(res, out_location, outs);
    BL_CATCH
}

}  // extern "C"
