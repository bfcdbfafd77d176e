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
#include "rolling.cuh"

namespace plb {

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
    int64_t s, e;
    const int64_t lo = fixed_window(a, i, s, e);
    const int64_t l = e - 1, b = l - (int64_t)((uint32_t)l % a.B);
    if (s < b) return St::combine(suf[s - base], pre[l - base]);
    return s == max(b, lo) ? pre[l - base] : suf[s - base];
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
struct FixedPlan { template <class St, typename In, class Fin> static void run(RollArgs a); };
template <class St, typename In, class Fin> void FixedPlan::run(RollArgs a) {
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
    roll_dispatch<FixedPlan>(kind, v.dtype, a, det);
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
