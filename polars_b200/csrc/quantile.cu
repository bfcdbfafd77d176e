// quantile.cu — median / quantile per group over GroupsIdx (BL_AGG_MEDIAN, BL_AGG_QUANTILE).
//
// Reference: agg_quantile_generic / agg_median_generic polars-core/src/frame/group_by/aggregations/mod.rs:297-408 (take of the
// group's rows, then _quantile), quantile_idx / linear_interpol / midpoint_interpol chunked_array/ops/aggregate/quantile.rs:21-65,
// the sort path for groups with nulls :179-234 (nulls first, picks at idx / idx + 1), output Float64 (Float32 stays: :1194-1219).
//
// A group's quantile needs its values in total order and one or two picks.  Values are encoded with sort_value_key (null rows:
// key 0).  Nulls and valid values that encode to 0 tie, so positions >= c (the null count) of the sorted group hold exactly
// the sorted valid values, and every pick index is >= c: the picks never see a null.  Two plans, chosen per group by size:
//   small (size <= QS_H)  k_quantile_small: CTA b takes the groups whose start offset lies in [b*QS_H, (b+1)*QS_H); at most
//                         QS_T = 2*QS_H rows.  It gathers their keys through `all` (read once, a random gather like K4), sorts
//                         (local group, key) with a bitonic network in shared memory, and picks every requested quantile
//                         there.  Nothing is written per row.
//   large (size > QS_H)   the large groups' keys are compacted in group order and sorted by (segment, key) with the stable
//                         LSD radix sort (filter.cu): first on the key (only the digits that vary), then on the segment, as
//                         op_arg_sort's two-stage scheme; k_quantile_pick_large then reads one thread per (group, quantile).
// Both plans call quantile_pick, so the arithmetic exists once.  All quantiles of one value column share the sort.
// Algorithmic bytes per row: small 4 (all) + elem (random gather) + 1/8 (validity); large 4 + elem + 12 (encode) + per radix
// pass 2 * (8 + 4) + 8 (histogram), + 4 + 8 for the segment stage.  Host synchronisations per column: two (the large-group
// count, the varying key bits), none per group.
// BL_QUANTILE_GLOBAL=1 (read per call) sends every group through the large-group plan: it exists so that tests compare the two
// plans byte for byte and tools/bench_quantile.py times both on the same input.
#include <cmath>
#include <cstdlib>

#include "common.cuh"
#include "dev_utils.cuh"
#include "sort_keys.cuh"

namespace plb {

bool radix_sort_pairs_u32(uint32_t* k0, uint32_t* v0, uint32_t* k1, uint32_t* v1, int64_t n, uint64_t vary, int* passes_run);
bool radix_sort_pairs_u64(uint64_t* k0, uint32_t* v0, uint64_t* k1, uint32_t* v1, int64_t n, uint64_t vary, int* passes_run);

constexpr int QS_T = 4096, QS_H = QS_T / 2, QS_THREADS = 512, QS_MAX_PICKS = 16;
constexpr size_t QS_SMEM = (size_t)QS_T * 8 + (size_t)QS_H * 4 + (size_t)QS_T * 2 + (size_t)(QS_H + 1) * 2;

struct QPick { double q; void* out; uint32_t* out_valid; int32_t method; int32_t out_f32; };
struct QArgs {
    const void* values; const uint32_t* validity; const uint32_t* offsets; const uint32_t* all;
    int64_t G, N; int32_t dtype, n_picks; QPick pick[QS_MAX_PICKS];
};

// inverse of sort_value_key for the value dtypes of the group_by hot path, as f64 (to_f64); -0.0 and NaN come back canonical
__device__ __forceinline__ double sort_key_to_f64(uint64_t k, int dtype) {
    switch (dtype) {
        case BL_INT32: return (double)(int32_t)((uint32_t)k ^ 0x80000000u);
        case BL_INT64: return (double)(int64_t)(k ^ 0x8000000000000000ull);
        case BL_FLOAT32: { uint32_t u = (uint32_t)k; u = (u >> 31) ? (u & 0x7fffffffu) : ~u; return (double)__uint_as_float(u); }
        case BL_FLOAT64: return ordered_to_f64(k);
        default: return (double)k;      // UInt32 / UInt64
    }
}

// quantile_idx + the interpolation of generic_quantiles (quantile.rs:21-65, :205-231), in f64 and in this order (the library is
// built with -fmad=false, so nothing is fused).  at(i) = the value at position i of the group sorted nulls first.
template <typename At>
__device__ __forceinline__ bool quantile_pick(uint32_t len, uint32_t nulls, double q, int method, At at, double& res) {
    const uint32_t m = len - nulls;
    if (m == 0) return false;
    const double float_idx = ((double)m - 1.0) * q + (double)nulls;
    uint32_t idx;
    switch (method) {
        case BL_QUANTILE_NEAREST: res = at((uint32_t)round(float_idx)); return true;      // f64::round: half away from zero
        case BL_QUANTILE_EQUIPROBABLE: res = at((uint32_t)fmax(ceil((double)m * q) - 1.0, 0.0) + nulls); return true;
        case BL_QUANTILE_HIGHER: idx = (uint32_t)ceil(float_idx); break;
        default: idx = (uint32_t)float_idx; break;                                        // LOWER / MIDPOINT / LINEAR
    }
    idx = min(idx, len - 1);
    const uint32_t top = (uint32_t)ceil(float_idx);
    const double lower = at(idx);
    if (idx == top || (method != BL_QUANTILE_MIDPOINT && method != BL_QUANTILE_LINEAR)) { res = lower; return true; }
    const double upper = at(idx + 1);
    if (lower == upper) res = lower;                                                      // inf, inf -> inf (not NaN)
    else if (method == BL_QUANTILE_MIDPOINT) res = (lower + upper) / 2.0;
    else res = (float_idx - (double)idx) * (upper - lower) + lower;
    return true;
}

__device__ __forceinline__ void quantile_store(const QPick& p, int64_t g, bool ok, double r) {
    if (p.out_f32) reinterpret_cast<float*>(p.out)[g] = ok ? (float)r : 0.0f;             // `as f32`: round to nearest
    else reinterpret_cast<double*>(p.out)[g] = ok ? r : 0.0;
    if (ok) atomicOr(&p.out_valid[g >> 5], 1u << (g & 31));
}

// first index in [0, n) with a[index] > x (a ascending)
template <typename T>
__device__ __forceinline__ uint32_t upper_bound_dev(const T* a, uint32_t n, uint64_t x) {
    uint32_t lo = 0, hi = n;
    while (lo < hi) { const uint32_t mid = (lo + hi) >> 1; if ((uint64_t)a[mid] <= x) lo = mid + 1; else hi = mid; }
    return lo;
}
// first index in [0, n) with a[index] >= x
__device__ __forceinline__ uint32_t lower_bound_dev(const uint32_t* a, uint32_t n, uint64_t x) {
    uint32_t lo = 0, hi = n;
    while (lo < hi) { const uint32_t mid = (lo + hi) >> 1; if ((uint64_t)a[mid] < x) lo = mid + 1; else hi = mid; }
    return lo;
}

// ---------------------------------------------------------------------------------------------- small groups
__global__ void __launch_bounds__(QS_THREADS) k_quantile_small(const __grid_constant__ QArgs a) {
    extern __shared__ __align__(16) unsigned char qs_smem[];
    uint64_t* skey = reinterpret_cast<uint64_t*>(qs_smem);                  // QS_T keys
    uint32_t* snull = reinterpret_cast<uint32_t*>(skey + QS_T);             // QS_H null counts per local group
    uint16_t* sseg = reinterpret_cast<uint16_t*>(snull + QS_H);             // QS_T local group ids
    uint16_t* soff = sseg + QS_T;                                           // QS_H + 1 local group starts
    __shared__ uint32_t s_g0, s_ng, s_p0, s_cnt;
    if (threadIdx.x == 0) {
        const uint64_t lo = (uint64_t)blockIdx.x * QS_H, hi = min((uint64_t)a.N, lo + QS_H);
        // groups [g0, g1) start inside the window; only the last one can be larger than QS_H (it then reaches past the window)
        // (offsets has G + 1 entries and offsets[G] = N >= hi, so both searches stay inside it)
        const uint32_t g0 = lower_bound_dev(a.offsets, (uint32_t)a.G + 1, lo);
        uint32_t g1 = lower_bound_dev(a.offsets, (uint32_t)a.G + 1, hi);
        if (g1 > g0 && a.offsets[g1] - a.offsets[g1 - 1] > (uint32_t)QS_H) g1--;
        s_g0 = g0; s_ng = g1 > g0 ? g1 - g0 : 0;
        s_p0 = a.offsets[g0]; s_cnt = a.offsets[g1] - a.offsets[g0];
    }
    __syncthreads();
    const uint32_t g0 = s_g0, ng = s_ng, p0 = s_p0, cnt = s_cnt;
    if (ng == 0) return;
    for (uint32_t j = threadIdx.x; j <= ng; j += QS_THREADS) soff[j] = (uint16_t)(a.offsets[g0 + j] - p0);
    for (uint32_t j = threadIdx.x; j < ng; j += QS_THREADS) snull[j] = 0;
    __syncthreads();
    uint32_t n2 = 2;
    while (n2 < cnt) n2 <<= 1;
    for (uint32_t i = threadIdx.x; i < n2; i += QS_THREADS) {
        if (i < cnt) {
            const uint32_t r = a.all[p0 + i];
            const bool ok = a.validity == nullptr || bit_get(a.validity, r);
            const uint32_t seg = upper_bound_dev(soff, ng + 1, i) - 1;
            skey[i] = ok ? sort_value_key(a.values, r, a.dtype) : 0;
            sseg[i] = (uint16_t)seg;
            if (!ok) atomicAdd(&snull[seg], 1u);
        } else { skey[i] = ~0ull; sseg[i] = 0xFFFF; }      // padding sorts after every group
    }
    __syncthreads();
    // bitonic sort of (local group, key), n2 / 2 compare-exchanges per step
    for (uint32_t k = 2; k <= n2; k <<= 1) {
        for (uint32_t j = k >> 1; j > 0; j >>= 1) {
            for (uint32_t t = threadIdx.x; t < n2 / 2; t += QS_THREADS) {
                const uint32_t i = 2 * t - (t & (j - 1)), l = i + j;
                const uint16_t si = sseg[i], sl = sseg[l];
                const uint64_t ki = skey[i], kl = skey[l];
                const bool gt = si > sl || (si == sl && ki > kl);
                if (gt == ((i & k) == 0)) { sseg[i] = sl; sseg[l] = si; skey[i] = kl; skey[l] = ki; }
            }
            __syncthreads();
        }
    }
    for (uint32_t w = threadIdx.x; w < ng * (uint32_t)a.n_picks; w += QS_THREADS) {
        const uint32_t gl = w % ng;
        const QPick& p = a.pick[w / ng];
        const uint32_t base = soff[gl], len = soff[gl + 1] - base;
        double r = 0.0;
        const bool ok = quantile_pick(len, snull[gl], p.q, p.method, [&](uint32_t i) { return sort_key_to_f64(skey[base + i], a.dtype); }, r);
        quantile_store(p, (int64_t)g0 + gl, ok, r);
    }
}

// ---------------------------------------------------------------------------------------------- large groups
// large[] = the groups of more than `thr` rows (any order); ctr[0] = their number, ctr[1] = their rows
__global__ void __launch_bounds__(256) k_quantile_find_large(const uint32_t* __restrict__ offsets, int64_t G, uint32_t thr, uint32_t* __restrict__ large,
                                                             unsigned long long* __restrict__ ctr) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t base = (int64_t)blockIdx.x * blockDim.x; base < G; base += stride) {
        const int64_t g = base + threadIdx.x;
        const uint32_t size = g < G ? offsets[g + 1] - offsets[g] : 0;
        const bool big = size > thr;
        const unsigned m = __ballot_sync(0xffffffffu, big);
        if (m == 0) continue;
        unsigned long long rows = big ? size : 0;
        for (int o = 16; o; o >>= 1) rows += __shfl_xor_sync(0xffffffffu, rows, o);
        unsigned slot = 0;
        if (lane_id() == 0) { slot = (unsigned)atomicAdd(&ctr[0], (unsigned long long)__popc(m)); atomicAdd(&ctr[1], rows); }
        slot = __shfl_sync(0xffffffffu, slot, 0);
        if (big) large[slot + __popc(m & lanemask_lt())] = (uint32_t)g;
    }
}

__global__ void k_quantile_large_sizes(const uint32_t* __restrict__ offsets, const uint32_t* __restrict__ large, int64_t NL, uint32_t* __restrict__ sizes) {
    for (int64_t s = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; s < NL; s += (int64_t)gridDim.x * blockDim.x) sizes[s] = offsets[large[s] + 1] - offsets[large[s]];
}

// keys of the large groups' rows, segment after segment (starts[s] = first position of segment s, starts[NL] = L); vals = iota;
// null rows counted per segment; andor[0] &= keys, andor[1] |= keys over all rows (nulls included: their key 0 must sort first)
__global__ void __launch_bounds__(256) k_quantile_encode_large(const void* __restrict__ values, const uint32_t* __restrict__ validity, int dtype, const uint32_t* __restrict__ offsets,
                                                               const uint32_t* __restrict__ all, const uint32_t* __restrict__ large, const uint64_t* __restrict__ starts, int64_t NL, int64_t L,
                                                               uint64_t* __restrict__ keys, uint32_t* __restrict__ vals, uint32_t* __restrict__ nulls, unsigned long long* __restrict__ andor) {
    uint64_t an = ~0ull, orr = 0;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t base = (int64_t)blockIdx.x * blockDim.x; base < L; base += stride) {
        const int64_t i = base + threadIdx.x;
        const bool in = i < L;
        uint32_t s = 0xFFFFFFFFu;
        bool ok = true;
        if (in) {
            s = upper_bound_dev(starts, (uint32_t)NL + 1, (uint64_t)i) - 1;
            const uint32_t r = all[offsets[large[s]] + (uint32_t)(i - (int64_t)starts[s])];
            ok = validity == nullptr || bit_get(validity, r);
            const uint64_t k = ok ? sort_value_key(values, r, dtype) : 0;
            keys[i] = k; vals[i] = (uint32_t)i;
            an &= k; orr |= k;
        }
        const uint32_t ns = in && !ok ? s : 0xFFFFFFFFu;
        const unsigned peers = __match_any_sync(0xffffffffu, ns);
        if (ns != 0xFFFFFFFFu && lane_id() == (unsigned)(__ffs(peers) - 1)) atomicAdd(&nulls[ns], (uint32_t)__popc(peers));
    }
    const uint32_t al = __reduce_and_sync(0xffffffffu, (uint32_t)an), ah = __reduce_and_sync(0xffffffffu, (uint32_t)(an >> 32));
    const uint32_t ol = __reduce_or_sync(0xffffffffu, (uint32_t)orr), oh = __reduce_or_sync(0xffffffffu, (uint32_t)(orr >> 32));
    if (lane_id() == 0) { atomicAnd(&andor[0], ((unsigned long long)ah << 32) | al); atomicOr(&andor[1], ((unsigned long long)oh << 32) | ol); }
}

// second stage: the segment of the row at each key-sorted position, payload = that position
__global__ void k_quantile_segment_keys(const uint32_t* __restrict__ pos, const uint64_t* __restrict__ starts, int64_t NL, int64_t L, uint32_t* __restrict__ seg, uint32_t* __restrict__ idx) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < L; i += (int64_t)gridDim.x * blockDim.x) {
        seg[i] = upper_bound_dev(starts, (uint32_t)NL + 1, (uint64_t)pos[i]) - 1;
        idx[i] = (uint32_t)i;
    }
}

// one thread per (large group, quantile): sorted position j of segment s holds keys[perm ? perm[j] : j]
__global__ void k_quantile_pick_large(const __grid_constant__ QArgs a, const uint32_t* __restrict__ large, const uint64_t* __restrict__ starts, const uint32_t* __restrict__ nulls,
                                      int64_t NL, const uint64_t* __restrict__ keys, const uint32_t* __restrict__ perm) {
    for (int64_t w = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; w < NL * a.n_picks; w += (int64_t)gridDim.x * blockDim.x) {
        const int64_t s = w % NL;
        const QPick& p = a.pick[w / NL];
        const uint32_t g = large[s];
        const uint64_t base = starts[s];
        double r = 0.0;
        const bool ok = quantile_pick(a.offsets[g + 1] - a.offsets[g], nulls[s], p.q, p.method,
                                      [&](uint32_t i) { const uint64_t j = base + i; return sort_key_to_f64(keys[perm ? perm[j] : j], a.dtype); }, r);
        quantile_store(p, g, ok, r);
    }
}

static void quantile_large_groups(const QArgs& a, uint32_t thr) {
    Context& c = ctx();
    const int64_t G = a.G;
    DevPtr large = dev_alloc((size_t)G * 4), ctr = dev_alloc(16);
    dev_memset(ctr->p, 0, 16);
    PLB_LAUNCH("quantile_find_large", k_quantile_find_large, grid_for(G, 256), 256, 0, a.offsets, G, thr, as<uint32_t>(large), as<unsigned long long>(ctr));
    uint64_t cnt[2];
    PLB_CUDA(cudaMemcpyAsync(cnt, ctr->p, 16, cudaMemcpyDeviceToHost, c.stream));
    PLB_CUDA(cudaStreamSynchronize(c.stream));
    const int64_t NL = (int64_t)cnt[0], L = (int64_t)cnt[1];
    if (NL == 0) return;
    DevPtr sizes = dev_alloc((size_t)NL * 4), starts = dev_alloc((size_t)(NL + 1) * 8), nulls = dev_alloc((size_t)NL * 4), andor = dev_alloc(16);
    PLB_LAUNCH("quantile_large_sizes", k_quantile_large_sizes, grid_for(NL, 256), 256, 0, a.offsets, as<uint32_t>(large), NL, as<uint32_t>(sizes));
    exclusive_scan_u32_to_u64(as<uint32_t>(sizes), as<uint64_t>(starts), NL, as<uint64_t>(starts) + NL);
    dev_memset(nulls->p, 0, (size_t)NL * 4);
    dev_memset(andor->p, 0xFF, 8);
    dev_memset((char*)andor->p + 8, 0, 8);
    DevPtr ka = dev_alloc((size_t)L * 8), kb = dev_alloc((size_t)L * 8), va = dev_alloc((size_t)L * 4), vb = dev_alloc((size_t)L * 4);
    PLB_LAUNCH("quantile_encode_large", k_quantile_encode_large, grid_for(L, 256), 256, 0, a.values, a.validity, a.dtype, a.offsets, a.all, as<uint32_t>(large), as<uint64_t>(starts),
               NL, L, as<uint64_t>(ka), as<uint32_t>(va), as<uint32_t>(nulls), as<unsigned long long>(andor));
    uint64_t ao[2];
    PLB_CUDA(cudaMemcpyAsync(ao, andor->p, 16, cudaMemcpyDeviceToHost, c.stream));
    PLB_CUDA(cudaStreamSynchronize(c.stream));
    // stage 1: by key (only the digits that differ between rows)
    const bool sw1 = radix_sort_pairs_u64(as<uint64_t>(ka), as<uint32_t>(va), as<uint64_t>(kb), as<uint32_t>(vb), L, ao[0] ^ ao[1], nullptr);
    const uint64_t* keys = as<uint64_t>(sw1 ? kb : ka);
    uint32_t* pos = as<uint32_t>(sw1 ? vb : va);
    uint32_t* spare_v = as<uint32_t>(sw1 ? va : vb);
    uint32_t* spare_k = reinterpret_cast<uint32_t*>(sw1 ? ka->p : kb->p);      // 8 L bytes: two u32 key buffers
    // stage 2: stable by segment, so every segment holds its rows in key order
    const uint32_t* perm = nullptr;
    if (NL > 1) {
        PLB_LAUNCH("quantile_segment_keys", k_quantile_segment_keys, grid_for(L, 256), 256, 0, pos, as<uint64_t>(starts), NL, L, spare_k, spare_v);
        const uint64_t vary = (1ull << bits_for((uint64_t)(NL - 1))) - 1;
        const bool sw2 = radix_sort_pairs_u32(spare_k, spare_v, spare_k + L, pos, L, vary, nullptr);
        perm = sw2 ? pos : spare_v;
    }
    PLB_LAUNCH("quantile_pick_large", k_quantile_pick_large, grid_for(NL * a.n_picks, 256), 256, 0, a, as<uint32_t>(large), as<uint64_t>(starts), as<uint32_t>(nulls), NL, keys, perm);
}

static bool quantile_force_global() { const char* e = getenv("BL_QUANTILE_GLOBAL"); return e != nullptr && e[0] == '1'; }      // read per call

void op_group_quantiles(const DevCol& offsets, const DevCol& all, const DevCol& values, const std::vector<double>& qs, const std::vector<int>& methods,
                        std::vector<DevCol>& outs) {
    const int64_t G = offsets.len - 1, N = all.len;
    const int dt = values.dtype;
    PLB_REQUIRE(dt == BL_INT64 || dt == BL_UINT64 || dt == BL_INT32 || dt == BL_UINT32 || dt == BL_FLOAT64 || dt == BL_FLOAT32, BL_ERR_UNSUPPORTED,
                std::string("group_by quantile: value dtype ") + dtype_name(dt) + " is outside the hot path");
    PLB_REQUIRE(N <= (int64_t)0xFFFFFFFFll, BL_ERR_UNSUPPORTED, "group_by quantile: more than 2^32 - 1 rows (IdxSize is u32)");
    outs.clear();
    for (size_t k = 0; k < qs.size(); k++) {
        DevCol o = make_col(dt == BL_FLOAT32 ? BL_FLOAT32 : BL_FLOAT64, G, true);
        dev_memset(o.validity->p, 0, o.validity->bytes);
        outs.push_back(o);
    }
    if (G <= 0) return;
    const bool global = quantile_force_global();
    static bool attr_set = false;        // serialised by the context lock
    if (!attr_set) { PLB_CUDA(cudaFuncSetAttribute(k_quantile_small, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)QS_SMEM)); attr_set = true; }
    // more than QS_MAX_PICKS quantiles of one column: one sort per QS_MAX_PICKS of them
    for (size_t b = 0; b < qs.size(); b += QS_MAX_PICKS) {
        QArgs a; memset(&a, 0, sizeof a);
        a.values = values.v(); a.validity = values.vm(); a.offsets = as<uint32_t>(offsets.values); a.all = as<uint32_t>(all.values);
        a.G = G; a.N = N; a.dtype = dt;
        a.n_picks = (int)std::min<size_t>(QS_MAX_PICKS, qs.size() - b);
        for (int k = 0; k < a.n_picks; k++) {
            const DevCol& o = outs[b + k];
            a.pick[k].q = qs[b + k]; a.pick[k].method = methods[b + k]; a.pick[k].out = o.values->p; a.pick[k].out_valid = as<uint32_t>(o.validity);
            a.pick[k].out_f32 = o.dtype == BL_FLOAT32;
        }
        if (!global) PLB_LAUNCH("quantile_small", k_quantile_small, (unsigned)((N + QS_H - 1) / QS_H), QS_THREADS, QS_SMEM, a);
        quantile_large_groups(a, global ? 0u : (uint32_t)QS_H);
    }
}

}  // namespace plb
