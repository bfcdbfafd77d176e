// rolling_quantile.cu — rolling quantile / median over fixed windows `expr.rolling_quantile(q, method, window_size,
// min_samples, center)` and time windows `expr.rolling_quantile_by(by, ...)`, plain or `.over()`, one output row per input
// row (polars-compute/src/rolling/{no_nulls,nulls}/quantile.rs, quantile_filter.rs; polars-time rolling_window/dispatch.rs).
//
// A quantile has no associative combine, so the block plans of rolling.cu / rolling_by.cu do not apply.  Instead each value
// column builds one wavelet matrix over its value ranks (DESIGN.md §16), which answers "the k-th smallest value among
// positions [s, e)" for any window in L = ceil(log2 n) rank steps, whatever the window's width:
//   1. order     positions are the rows, or bl_over's partition order (perm, with its inverse inv)
//   2. ranks     op_arg_sort(values, nulls last): stable, so rank r is the r-th row of the total order (tot_cmp: NaN greatest,
//                -0.0 == +0.0; nulls rank >= n_valid).  k_rq_ranks writes A[position] = rank and V[rank] = the row's value
//                in the output type T (to_float), so every result is one of its window's values or their interpolation.
//   3. nulls     a bitvector over positions (bit = the position's rank >= n_valid) whose rank query counts a window's nulls
//   4. levels    level l holds bit L-1-l of every element of A in that level's order; the next order is the stable split
//                zeros-then-ones (k_wm_count: per-tile zero counts; a scan; k_wm_split: the bits, the directory, the scatter)
//   5. k_rq_out  one thread per position: its window, the valid count m, the method's index in f64 as the reference computes
//                it, one or two descents, the arithmetic in T, write_out to row perm[i]
// Bitvectors are 32-byte blocks of one u32 count of the ones before the block and 7 words of bits (224 positions), so a rank
// query reads one sector.
#include "rolling.cuh"

namespace plb {

constexpr int BV_THREADS = 256, BV_ITEMS = 7, BV_TILE = BV_THREADS * BV_ITEMS, BV_BITS = 224, BV_WORDS = BV_TILE / 32;
static_assert(BV_TILE % BV_BITS == 0, "a tile holds whole blocks");

// ---------------------------------------------------------------------------------------------------- bitvectors
// the ones before position i (0 <= i <= n) of the bitvector bv
__device__ __forceinline__ uint32_t bv_rank1(const uint32_t* __restrict__ bv, uint32_t i) {
    const uint32_t b = i / BV_BITS, off = i - b * BV_BITS;
    const uint4* p = reinterpret_cast<const uint4*>(bv + (size_t)b * 8);
    const uint4 h = __ldg(p), t = __ldg(p + 1);
    const uint32_t w[8] = {h.x, h.y, h.z, h.w, t.x, t.y, t.z, t.w};
    const uint32_t nw = off >> 5;
    uint32_t r = w[0];
#pragma unroll
    for (uint32_t k = 0; k < 7; k++) {
        if (k < nw) r += __popc(w[1 + k]);
        else if (k == nw) r += __popc(w[1 + k] & ((1u << (off & 31)) - 1u));
    }
    return r;
}
__device__ __forceinline__ uint32_t bv_rank0(const uint32_t* bv, uint32_t i) { return i - bv_rank1(bv, i); }

// the bit of rank x: bit `shift` of x, or (shift == BV_NULLS) whether x >= thr, i.e. the row is null
constexpr uint32_t BV_NULLS = 32;
__device__ __forceinline__ bool wm_bit(uint32_t x, uint32_t shift, uint32_t thr) { return shift == BV_NULLS ? x >= thr : ((x >> shift) & 1u); }

// zeros of tile t (positions [t * BV_TILE, +BV_TILE) below n); one CTA per tile
__global__ void __launch_bounds__(BV_THREADS) k_wm_count(const uint32_t* __restrict__ cur, int64_t n, uint32_t shift, uint32_t thr, uint32_t* __restrict__ tile_zeros) {
    __shared__ uint32_t s_c[BV_THREADS / 32];
    const int64_t base = (int64_t)blockIdx.x * BV_TILE;
    uint32_t z = 0;
#pragma unroll
    for (int it = 0; it < BV_ITEMS; it++) {
        const int64_t p = base + it * BV_THREADS + threadIdx.x;
        if (p < n) z += wm_bit(__ldg(cur + p), shift, thr) ? 0u : 1u;
    }
    z = __reduce_add_sync(0xffffffffu, z);
    if (lane_id() == 0) s_c[threadIdx.x >> 5] = z;
    __syncthreads();
    if (threadIdx.x == 0) {
        uint32_t t = 0;
        for (int k = 0; k < BV_THREADS / 32; k++) t += s_c[k];
        tile_zeros[blockIdx.x] = t;
    }
}

// Tile t's bits and directory counts into bv, and (next != NULL) the stable split: zeros to next[zeros before], ones to
// next[Z + ones before].  tile_zoff: the exclusive scan of tile_zeros, Z = *zeros_total.  Warp w of iteration it owns word
// it * 8 + w of the tile (32 consecutive positions), i.e. word 1 + j % 7 of the tile's block j / 7.
__global__ void __launch_bounds__(BV_THREADS) k_wm_split(const uint32_t* __restrict__ cur, int64_t n, uint32_t shift, uint32_t thr,
                                                         const unsigned long long* __restrict__ tile_zoff, const unsigned long long* __restrict__ zeros_total,
                                                         uint32_t* __restrict__ next, uint32_t* __restrict__ bv) {
    __shared__ uint32_t s_z[BV_WORDS];      // zeros per word, then their exclusive scan
    const unsigned lane = lane_id(), warp = threadIdx.x >> 5;
    const int64_t base = (int64_t)blockIdx.x * BV_TILE;
    uint32_t x[BV_ITEMS], zw[BV_ITEMS];
#pragma unroll
    for (int it = 0; it < BV_ITEMS; it++) {
        const int j = it * (BV_THREADS / 32) + (int)warp;
        const int64_t p = base + (int64_t)j * 32 + lane;
        const bool in = p < n;
        x[it] = in ? __ldg(cur + p) : 0u;
        const bool one = in && wm_bit(x[it], shift, thr);
        const uint32_t ow = __ballot_sync(0xffffffffu, one);
        zw[it] = __ballot_sync(0xffffffffu, in && !one);
        if (lane == 0) {
            s_z[j] = __popc(zw[it]);
            bv[((size_t)blockIdx.x * (BV_TILE / BV_BITS) + j / 7) * 8 + 1 + j % 7] = ow;
        }
    }
    __syncthreads();
    if (warp == 0) {      // exclusive scan of the BV_WORDS = 56 word counts, two per lane
        const uint32_t a = lane * 2 < BV_WORDS ? s_z[lane * 2] : 0u, b = lane * 2 + 1 < BV_WORDS ? s_z[lane * 2 + 1] : 0u;
        uint32_t inc = a + b;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const uint32_t y = __shfl_up_sync(0xffffffffu, inc, o);
            if ((int)lane >= o) inc += y;
        }
        const uint32_t ex = inc - a - b;
        __syncwarp();
        if (lane * 2 < BV_WORDS) s_z[lane * 2] = ex;
        if (lane * 2 + 1 < BV_WORDS) s_z[lane * 2 + 1] = ex + a;
    }
    __syncthreads();
    const unsigned long long z0 = tile_zoff[blockIdx.x];
    if (threadIdx.x < BV_TILE / BV_BITS) {      // block k starts at position base + 224 k: its ones-before count
        const int64_t start = base + (int64_t)threadIdx.x * BV_BITS;
        if (start <= n) bv[((size_t)blockIdx.x * (BV_TILE / BV_BITS) + threadIdx.x) * 8] = (uint32_t)(start - (int64_t)(z0 + s_z[threadIdx.x * 7]));
    }
    if (next == nullptr) return;
    const unsigned long long Z = *zeros_total;
#pragma unroll
    for (int it = 0; it < BV_ITEMS; it++) {
        const int j = it * (BV_THREADS / 32) + (int)warp;
        const int64_t p = base + (int64_t)j * 32 + lane;
        const unsigned long long zb = z0 + s_z[j] + __popc(zw[it] & lanemask_lt());      // zeros before p
        if (p < n) next[((zw[it] >> lane) & 1u) ? zb : Z + ((unsigned long long)p - zb)] = x[it];
    }
}

// ---------------------------------------------------------------------------------------------------- ranks
// A[position of the row at rank k] = k; V[k] = that row's value in T
template <typename In, typename T>
__global__ void __launch_bounds__(256) k_rq_ranks(const void* __restrict__ values, const uint32_t* __restrict__ sorted, const uint32_t* __restrict__ inv, int64_t n,
                                                  uint32_t* __restrict__ A, T* __restrict__ V) {
    for (int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; k < n; k += (int64_t)gridDim.x * blockDim.x) {
        const uint32_t row = __ldg(sorted + k);
        A[inv ? __ldg(inv + row) : row] = (uint32_t)k;
        V[k] = (T)load_in<In>(values, row);
    }
}

// ---------------------------------------------------------------------------------------------------- k_rq_out
struct WMArgs {
    const uint32_t* levels; int64_t level_words; int L;      // level l at levels + l * level_words
    const unsigned long long* Z;                              // zeros per level
    const uint32_t* nulls;                                    // the null bitvector over positions (NULL: no nulls)
    const void* V;
    double q; int method;
};

// the rank of the k-th smallest (0-based) element of A over positions [s, e)
__device__ __forceinline__ uint32_t wm_kth(const WMArgs& w, uint32_t s, uint32_t e, uint32_t k) {
    uint32_t v = 0;
    for (int l = 0; l < w.L; l++) {
        const uint32_t* bv = w.levels + (size_t)l * w.level_words;
        const uint32_t zs = bv_rank0(bv, s), ze = bv_rank0(bv, e), z = ze - zs;
        if (k < z) { s = zs; e = ze; }
        else {
            const uint32_t Z = (uint32_t)__ldg(w.Z + l);
            k -= z; s = Z + (s - zs); e = Z + (e - ze);
            v |= 1u << (w.L - 1 - l);
        }
    }
    return v;
}

template <typename T> struct FinQ { using out_t = T; };

// The window of position i, its valid count m (null when m < max(min_samples, 1); a time window also when it holds fewer than
// min_samples rows, nulls included, or i's `by` is null), the index of QuantileWindow::get_agg / QuantileUpdate::quantile
// in f64 (no_nulls/quantile.rs:55-105, nulls/quantile.rs:52-106, quantile_filter.rs:610-671) and the arithmetic in T
// (FinishLinear, quantile_filter.rs:559-567).
template <typename T>
__global__ void __launch_bounds__(256) k_rq_out(const __grid_constant__ RollArgs a, const __grid_constant__ WMArgs w) {
    const T* V = reinterpret_cast<const T*>(w.V);
    const int64_t n_round = (a.n + 31) / 32 * 32;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_round; i += (int64_t)gridDim.x * blockDim.x) {
        bool ok = false;
        T x = T(0);
        if (i < a.n) {
            int64_t s, e;
            bool has = true;
            if (a.ws) {
                const uint32_t s32 = __ldg(a.ws + i);
                s = s32; e = __ldg(a.we + i);
                has = s32 != BY_NULL && e - s >= a.min_samples;
            } else fixed_window(a, i, s, e);
            const uint64_t m = !has ? 0 : w.nulls ? bv_rank0(w.nulls, (uint32_t)e) - bv_rank0(w.nulls, (uint32_t)s) : (uint64_t)(e - s);
            if (m > 0 && (int64_t)m >= a.min_samples) {
                const double mf = (double)m, fi = (mf - 1.0) * w.q;
                uint64_t lo, hi;
                switch (w.method) {
                    case BL_QUANTILE_NEAREST: lo = (uint64_t)round(fi); break;      // f64::round: half away from zero
                    case BL_QUANTILE_HIGHER: lo = (uint64_t)ceil(fi); break;
                    case BL_QUANTILE_EQUIPROBABLE: lo = (uint64_t)fmax(ceil(mf * w.q) - 1.0, 0.0); break;
                    default: lo = (uint64_t)floor(fi); break;                      // LOWER / MIDPOINT / LINEAR
                }
                lo = min(lo, m - 1);
                hi = (uint64_t)ceil(fi);
                x = V[wm_kth(w, (uint32_t)s, (uint32_t)e, (uint32_t)lo)];
                if ((w.method == BL_QUANTILE_MIDPOINT || w.method == BL_QUANTILE_LINEAR) && hi != lo) {
                    const T y = V[wm_kth(w, (uint32_t)s, (uint32_t)e, (uint32_t)hi)];
                    if (w.method == BL_QUANTILE_MIDPOINT) x = (x + y) / T(2);
                    else x = (T)(fi - (double)lo) * (y - x) + x;      // no lo == hi guard: inf, inf -> NaN
                }
                ok = true;
            }
        }
        write_out<FinQ<T>>(a, i, i < a.n, ok, x);
    }
}

// ---------------------------------------------------------------------------------------------------- host side
int rolling_quantile_dtype(int dt) { return dt == BL_FLOAT32 ? BL_FLOAT32 : BL_FLOAT64; }

static void check_quantile(const char* who, double q, int method) {
    PLB_REQUIRE(q >= 0.0 && q <= 1.0, BL_ERR_INVALID, std::string(who) + ": quantile must be in [0, 1], not " + std::to_string(q));
    PLB_REQUIRE(method >= BL_QUANTILE_NEAREST && method <= BL_QUANTILE_EQUIPROBABLE, BL_ERR_INVALID, std::string(who) + ": unknown method " + std::to_string(method));
}
static void check_value_dtype(const char* who, int dt) {
    PLB_REQUIRE(dt >= 0 && dt <= BL_BOOL, BL_ERR_INVALID, std::string(who) + ": unknown value dtype");
    PLB_REQUIRE(dt != BL_BOOL, BL_ERR_UNSUPPORTED, std::string(who) + ": a Boolean column has no quantile on the device");
}

void check_rolling_quantile_op(double q, int method, int center, int64_t window_size, int64_t min_samples, int value_dtype) {
    check_quantile("rolling_quantile", q, method);
    check_value_dtype("rolling_quantile", value_dtype);
    PLB_REQUIRE(center == 0 || center == 1, BL_ERR_INVALID, "rolling_quantile: center must be 0 or 1");
    PLB_REQUIRE(window_size >= 0 && min_samples >= 0, BL_ERR_INVALID, "rolling_quantile: window_size and min_samples must not be negative");
    PLB_REQUIRE(min_samples <= window_size, BL_ERR_INVALID, "rolling_quantile: min_samples (" + std::to_string(min_samples) + ") must be <= window_size (" + std::to_string(window_size) + ")");
    PLB_REQUIRE(window_size > 0, BL_ERR_UNSUPPORTED, "rolling_quantile: window_size 0 is outside the hot path");
}

void check_rolling_quantile_by_op(double q, int method, int closed, int64_t window_size, int64_t min_samples, int value_dtype) {
    check_quantile("rolling_quantile_by", q, method);
    check_value_dtype("rolling_quantile_by", value_dtype);
    PLB_REQUIRE(closed >= BL_CLOSED_RIGHT && closed <= BL_CLOSED_NONE, BL_ERR_INVALID, "rolling_quantile_by: unknown closed " + std::to_string(closed));
    PLB_REQUIRE(window_size > 0, BL_ERR_INVALID, "rolling_quantile_by: window_size must be strictly positive");
    PLB_REQUIRE(min_samples >= 0, BL_ERR_INVALID, "rolling_quantile_by: min_samples must not be negative");
}

// The wavelet matrix of one value column over the positions (perm / inv: the partition order; NULL: the rows)
struct WMatrix {
    DevPtr levels, Z, nulls, V;
    int L = 1, dtype = BL_FLOAT64;
    int64_t level_words = 0;
};

template <typename In, typename T> static void launch_ranks(const DevCol& v, const uint32_t* sorted, const uint32_t* inv, uint32_t* A, void* V) {
    PLB_LAUNCH("rolling_quantile_ranks", (k_rq_ranks<In, T>), grid_for(v.len, 256), 256, 0, v.v(), sorted, inv, v.len, A, reinterpret_cast<T*>(V));
}

// one bitvector of cur (bit `shift` of each rank, or rank >= thr when shift == BV_NULLS) into bv; next != NULL: the split order too
static void build_bitvector(const uint32_t* cur, int64_t n, uint32_t shift, uint32_t thr, uint32_t* next, uint32_t* bv, unsigned long long* zeros_total) {
    const int64_t ntiles = n / BV_TILE + 1;      // the last tile holds position n: the directory entry a rank query at n reads
    DevPtr tz = dev_alloc((size_t)ntiles * 4), toff = dev_alloc((size_t)ntiles * 8);
    PLB_LAUNCH("rolling_quantile_wm_count", k_wm_count, (int)ntiles, BV_THREADS, 0, cur, n, shift, thr, as<uint32_t>(tz));
    exclusive_scan_u32_to_u64(as<uint32_t>(tz), as<uint64_t>(toff), ntiles, reinterpret_cast<uint64_t*>(zeros_total));
    PLB_LAUNCH("rolling_quantile_wm_split", k_wm_split, (int)ntiles, BV_THREADS, 0, cur, n, shift, thr, as<unsigned long long>(toff), zeros_total, next, bv);
}

static WMatrix wm_build(const DevCol& v, const uint32_t* inv) {
    const int64_t n = v.len;
    WMatrix w;
    w.dtype = rolling_quantile_dtype(v.dtype);
    while ((int64_t(1) << w.L) < n) w.L++;
    w.level_words = (n / BV_TILE + 1) * (BV_TILE / BV_BITS) * 8;
    DevPtr A;
    {
        // A and V are allocated after the sort, whose scratch is freed on return: the peak is the sort's plus the input,
        // which keeps a column past 2^31 rows within one 80 GB device
        const DevCol sorted = op_arg_sort({v}, {BL_SORT_NULLS_LAST}, -1);
        A = dev_alloc((size_t)n * 4);
        w.V = dev_alloc((size_t)n * dtype_size(w.dtype));
        const uint32_t* s = as<uint32_t>(sorted.values);
        switch (v.dtype) {
            case BL_INT8: launch_ranks<int8_t, double>(v, s, inv, as<uint32_t>(A), w.V->p); break;
            case BL_INT16: launch_ranks<int16_t, double>(v, s, inv, as<uint32_t>(A), w.V->p); break;
            case BL_INT32: launch_ranks<int32_t, double>(v, s, inv, as<uint32_t>(A), w.V->p); break;
            case BL_INT64: launch_ranks<int64_t, double>(v, s, inv, as<uint32_t>(A), w.V->p); break;
            case BL_UINT8: launch_ranks<uint8_t, double>(v, s, inv, as<uint32_t>(A), w.V->p); break;
            case BL_UINT16: launch_ranks<uint16_t, double>(v, s, inv, as<uint32_t>(A), w.V->p); break;
            case BL_UINT32: launch_ranks<uint32_t, double>(v, s, inv, as<uint32_t>(A), w.V->p); break;
            case BL_UINT64: launch_ranks<uint64_t, double>(v, s, inv, as<uint32_t>(A), w.V->p); break;
            case BL_FLOAT32: launch_ranks<float, float>(v, s, inv, as<uint32_t>(A), w.V->p); break;
            default: launch_ranks<double, double>(v, s, inv, as<uint32_t>(A), w.V->p); break;
        }
    }
    w.Z = dev_alloc((size_t)(w.L + 1) * 8);
    const int64_t n_valid = v.validity ? bitmap_popcount(v.vm(), n) : n;
    if (n_valid < n) {
        w.nulls = dev_alloc((size_t)w.level_words * 4);
        build_bitvector(as<uint32_t>(A), n, BV_NULLS, (uint32_t)n_valid, nullptr, as<uint32_t>(w.nulls), as<unsigned long long>(w.Z) + w.L);
    }
    w.levels = dev_alloc((size_t)w.L * w.level_words * 4);
    DevPtr B = dev_alloc((size_t)n * 4);
    for (int l = 0; l < w.L; l++) {
        const bool last = l + 1 == w.L;
        build_bitvector(as<uint32_t>(A), n, (uint32_t)(w.L - 1 - l), 0, last ? nullptr : as<uint32_t>(B), as<uint32_t>(w.levels) + (size_t)l * w.level_words,
                        as<unsigned long long>(w.Z) + l);
        std::swap(A, B);
    }
    return w;
}

template <typename T> static void run_query(const RollArgs& a, const WMArgs& w) {
    PLB_LAUNCH("rolling_quantile_out", k_rq_out<T>, grid_for((a.n + 31) / 32 * 32, 256), 256, 0, a, w);
}

// ops[k] of one column through the matrix; a: the positions and window of the op, everything but the output set
static DevCol wm_query(const WMatrix& m, RollArgs a, double q, int method) {
    DevCol out = make_col(m.dtype, a.n, true);
    out.null_count = -1;
    a.out = out.values->p; a.out_valid = as<uint32_t>(out.validity);
    if (a.perm) dev_memset(a.out_valid, 0, bitmap_bytes(a.n));
    WMArgs w{as<uint32_t>(m.levels), m.level_words, m.L, as<unsigned long long>(m.Z), as<uint32_t>(m.nulls), m.V->p, q, method};
    if (m.dtype == BL_FLOAT32) run_query<float>(a, w);
    else run_query<double>(a, w);
    return out;
}

// Every op over its column's matrix: ops that share a value column (the same DevCol) share one build.  set_window(k, a) fills
// the window fields of op k.
template <class Op, class SetWindow>
static std::vector<DevCol> quantile_ops(const std::vector<Op>& ops, int64_t n, const OverOrder* o, SetWindow set_window) {
    std::vector<DevCol> res(ops.size());
    std::vector<bool> done(ops.size(), false);
    for (size_t k = 0; k < ops.size(); k++) {
        if (done[k]) continue;
        if (n == 0) {
            res[k] = make_col(rolling_quantile_dtype(ops[k].values->dtype), 0, false);
            res[k].null_count = 0;
            done[k] = true;
            continue;
        }
        const WMatrix m = wm_build(*ops[k].values, o ? as<uint32_t>(o->inv.values) : nullptr);
        for (size_t j = k; j < ops.size(); j++) {
            if (done[j] || ops[j].values != ops[k].values) continue;
            RollArgs a;
            memset(&a, 0, sizeof a);
            a.n = n;
            if (o) { a.perm = as<uint32_t>(o->perm.values); a.offsets = as<uint32_t>(o->offsets.values); a.G = o->G; }
            else a.G = 1;
            a.min_samples = ops[j].min_samples;
            set_window(j, a);
            res[j] = wm_query(m, a, ops[j].quantile, ops[j].method);
            done[j] = true;
        }
    }
    return res;
}

// the row limits, checked before any column is read: IdxSize positions, and group tuples when a sort is needed (`grouped`:
// partitions or order_by; a null or unsorted `by` is found on the device, by rolling_by_order)
static void check_quantile_rows(const char* who, int64_t n, bool grouped) {
    PLB_REQUIRE(!grouped || n <= 0x7FFFFFFFll, BL_ERR_UNSUPPORTED, std::string(who) + ": more than 2^31 - 1 rows need a sort (group tuples)");
    PLB_REQUIRE(n <= 0xFFFFFFFFll, BL_ERR_UNSUPPORTED, std::string(who) + ": more than 2^32 - 1 rows (IdxSize is u32)");
}

// ops are checked by the caller (check_rolling_quantile_op) before any column is uploaded
std::vector<DevCol> op_rolling_quantile(const std::vector<DevCol>& partition_by, const DevCol* order_key, int order_flags, const std::vector<RollQuantileOp>& ops, int64_t n) {
    for (auto& op : ops) PLB_REQUIRE(op.values && op.values->len == n, BL_ERR_INVALID, "rolling_quantile: value columns differ in length");
    for (auto& k : partition_by) PLB_REQUIRE(k.len == n, BL_ERR_INVALID, "rolling_quantile: partition columns differ in length");
    if (order_key) PLB_REQUIRE(order_key->len == n, BL_ERR_INVALID, "rolling_quantile: the order_by column differs in length");
    const bool need_order = !partition_by.empty() || order_key;
    check_quantile_rows("rolling_quantile", n, need_order);
    OverOrder o;
    if (need_order && n > 0) {
        o.gid = partition_ids(partition_by, n);
        build_order(o, order_key, order_flags, true);
    }
    return quantile_ops(ops, n, need_order ? &o : nullptr, [&](size_t k, RollArgs& a) {
        const int64_t w = ops[k].window_size;      // det_offsets / det_offsets_center (rolling/mod.rs:72-87), as rolling_one
        int64_t L = w - 1, R = 1;
        if (ops[k].center) { R = w / 2 + (w & 1); L = w - R; }
        a.L = std::min(L, n); a.R = std::min(R, n);
    });
}

std::vector<DevCol> op_rolling_quantile_by(const std::vector<DevCol>& partition_by, const DevCol& by, const std::vector<RollQuantileOp>& ops, int64_t n) {
    for (auto& op : ops) PLB_REQUIRE(op.values && op.values->len == n, BL_ERR_INVALID, "rolling_quantile_by: value columns differ in length");
    for (auto& k : partition_by) PLB_REQUIRE(k.len == n, BL_ERR_INVALID, "rolling_quantile_by: partition columns differ in length");
    const ByOrder bo = rolling_by_order("rolling_quantile_by", partition_by, by, n, true);
    DevPtr ws = dev_alloc((size_t)n * 4), we = dev_alloc((size_t)n * 4);
    int64_t P = -1;
    int closed = -1;
    return quantile_ops(ops, n, bo.need_order ? &bo.o : nullptr, [&](size_t k, RollArgs& a) {
        if (ops[k].window_size != P || ops[k].closed != closed) {
            P = ops[k].window_size; closed = ops[k].closed;
            rolling_by_bounds(by, bo, n, P, closed, as<uint32_t>(ws), as<uint32_t>(we));
        }
        a.ws = as<uint32_t>(ws); a.we = as<uint32_t>(we);
    });
}

}  // namespace plb

// ================================================================================ C ABI
using namespace plb;
extern "C" {

bl_status bl_rolling_quantile(const bl_sort_key* partition_by, int32_t n_partition_by, const bl_sort_key* order_by, const bl_rolling_quantile_op* ops,
                              int32_t n_ops, int32_t out_location, bl_column* outs) {
    BL_TRY
    PLB_REQUIRE(n_ops >= 1 && ops && outs, BL_ERR_INVALID, "rolling_quantile: no operations or no outputs");
    int64_t n = -1;
    check_window_keys("rolling_quantile", partition_by, n_partition_by, order_by, n);
    for (int i = 0; i < n_ops; i++) {
        PLB_REQUIRE(ops[i].values != nullptr, BL_ERR_INVALID, "rolling_quantile: operation " + std::to_string(i) + " has no value column");
        check_rolling_quantile_op(ops[i].quantile, ops[i].method, ops[i].center, ops[i].window_size, ops[i].min_samples, ops[i].values->dtype);
        set_window_len("rolling_quantile", ops[i].values->length, "value column " + std::to_string(i), n);
    }
    check_quantile_rows("rolling_quantile", n, n_partition_by > 0 || order_by);
    std::vector<DevCol> parts;
    for (int i = 0; i < n_partition_by; i++) parts.push_back(import_key(partition_by[i], true));
    DevCol okey;
    if (order_by) okey = import_key(*order_by, false);
    std::vector<DevCol> vals(n_ops);
    std::vector<RollQuantileOp> v(n_ops);
    for (int i = 0; i < n_ops; i++) {
        int first = 0;      // ops that point to the same bl_column share its upload and its matrix
        while (ops[first].values != ops[i].values) first++;
        if (first == i) vals[i] = import_column(ops[i].values, 1);
        v[i].quantile = ops[i].quantile; v[i].method = ops[i].method; v[i].center = ops[i].center != 0;
        v[i].window_size = ops[i].window_size; v[i].min_samples = ops[i].min_samples; v[i].values = &vals[first];
    }
    std::vector<DevCol> res = op_rolling_quantile(parts, order_by ? &okey : nullptr, order_by ? order_by->flags : 0, v, n);
    export_many(res, out_location, outs);
    BL_CATCH
}

bl_status bl_rolling_quantile_by(const bl_sort_key* partition_by, int32_t n_partition_by, const bl_column* by, const bl_rolling_quantile_by_op* ops,
                                 int32_t n_ops, int32_t out_location, bl_column* outs) {
    BL_TRY
    PLB_REQUIRE(n_ops >= 1 && ops && outs, BL_ERR_INVALID, "rolling_quantile_by: no operations or no outputs");
    PLB_REQUIRE(by != nullptr, BL_ERR_INVALID, "rolling_quantile_by: no `by` column");
    int64_t n = -1;
    check_window_keys("rolling_quantile_by", partition_by, n_partition_by, nullptr, n);
    set_window_len("rolling_quantile_by", by->length, "the `by` column", n);
    for (int i = 0; i < n_ops; i++) {
        PLB_REQUIRE(ops[i].values != nullptr, BL_ERR_INVALID, "rolling_quantile_by: operation " + std::to_string(i) + " has no value column");
        check_rolling_quantile_by_op(ops[i].quantile, ops[i].method, ops[i].closed, ops[i].window_size, ops[i].min_samples, ops[i].values->dtype);
        set_window_len("rolling_quantile_by", ops[i].values->length, "value column " + std::to_string(i), n);
    }
    check_quantile_rows("rolling_quantile_by", n, n_partition_by > 0);
    std::vector<DevCol> parts;
    for (int i = 0; i < n_partition_by; i++) parts.push_back(import_key(partition_by[i], true));
    const DevCol byc = import_column(by, 1);
    std::vector<DevCol> vals(n_ops);
    std::vector<RollQuantileOp> v(n_ops);
    for (int i = 0; i < n_ops; i++) {
        int first = 0;
        while (ops[first].values != ops[i].values) first++;
        if (first == i) vals[i] = import_column(ops[i].values, 1);
        v[i].quantile = ops[i].quantile; v[i].method = ops[i].method; v[i].closed = ops[i].closed;
        v[i].window_size = ops[i].window_size; v[i].min_samples = ops[i].min_samples; v[i].values = &vals[first];
    }
    std::vector<DevCol> res = op_rolling_quantile_by(parts, byc, v, n);
    export_many(res, out_location, outs);
    BL_CATCH
}

}  // extern "C"
