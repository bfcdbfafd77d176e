// filter.cu — K3: stream compaction of c columns by one bit mask, plus the tile-scan helper.
//
// Reference: polars-compute/src/filter/mod.rs:18-110 (null mask slot = false; values and validity
// of the kept rows are compacted in row order), scalar.rs:9-138 / avx512.rs:45-115 (64-wide
// compaction), DataFrame::filter polars-core/src/frame/mod.rs:1148-1180 (all columns, one mask).
//
// Design: the mask is a bitmap (1/64 of a column), so the prefix offsets are computed from
// it once — per-tile popcounts (TILE rows) + one exclusive scan — and every column is compacted in
// a single pass with no inter-CTA dependency: row -> rank = tile_offset + popcount of mask bits
// before it.  Kept rows of a warp are contiguous in the output, so stores coalesce; unselected
// rows are never loaded (predicated loads skip whole sectors at low selectivity).
// Algorithmic bytes: 8*c + 8*c*s per row (+1/8 for the mask); bound: HBM.
#include "common.cuh"
#include "dev_utils.cuh"

namespace plb {

constexpr int F_TILE = 4096;            // rows per tile
constexpr int F_TILE_WORDS = F_TILE / 32;
constexpr int F_THREADS = 256;

// per-tile popcount of the mask
__global__ void __launch_bounds__(128) k_mask_tile_counts(const uint32_t* __restrict__ mask, int64_t n, uint32_t* __restrict__ counts, int64_t ntiles) {
    for (int64_t t = blockIdx.x; t < ntiles; t += gridDim.x) {
        int64_t w = t * F_TILE_WORDS + threadIdx.x;
        int64_t row0 = w * 32;
        uint32_t c = 0;
        if (row0 < n) {
            uint32_t m = mask[w];
            if (row0 + 32 > n) m &= (1u << (n - row0)) - 1u;
            c = __popc(m);
        }
        for (int o = 16; o; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
        __shared__ uint32_t s[4];
        if (lane_id() == 0) s[threadIdx.x >> 5] = c;
        __syncthreads();
        if (threadIdx.x == 0) counts[t] = s[0] + s[1] + s[2] + s[3];
        __syncthreads();
    }
}

// single-CTA exclusive scan u32 -> u64 (n up to a few hundred thousand tiles; negligible time)
template <typename TIN>
__global__ void __launch_bounds__(1024) k_scan_u64(const TIN* __restrict__ in, uint64_t* __restrict__ out, int64_t n, uint64_t* total) {
    __shared__ uint64_t warp_sums[32];
    __shared__ uint64_t carry_s;
    if (threadIdx.x == 0) carry_s = 0;
    __syncthreads();
    const unsigned lane = lane_id(), warp = threadIdx.x >> 5;
    for (int64_t base = 0; base < n; base += 1024) {
        int64_t i = base + threadIdx.x;
        uint64_t v = i < n ? in[i] : 0, x = v;
        for (int o = 1; o < 32; o <<= 1) { uint64_t y = __shfl_up_sync(0xffffffffu, x, o); if (lane >= (unsigned)o) x += y; }
        if (lane == 31) warp_sums[warp] = x;
        __syncthreads();
        if (warp == 0) {
            uint64_t s = warp_sums[lane], t = s;
            for (int o = 1; o < 32; o <<= 1) { uint64_t y = __shfl_up_sync(0xffffffffu, t, o); if (lane >= (unsigned)o) t += y; }
            warp_sums[lane] = t - s;    // exclusive warp offsets
        }
        __syncthreads();
        uint64_t carry = carry_s;
        uint64_t incl = carry + warp_sums[warp] + x;
        if (i < n) out[i] = incl - v;
        __syncthreads();
        if (threadIdx.x == 1023) carry_s = incl;
        __syncthreads();
    }
    if (threadIdx.x == 0 && total) *total = carry_s;
}
void exclusive_scan_u32_to_u64(const uint32_t* in, uint64_t* out, int64_t n, uint64_t* total_dev) {
    PLB_LAUNCH("scan_u32_u64", (k_scan_u64<uint32_t>), 1, 1024, 0, in, out, n, total_dev);
}
void exclusive_scan_u64(const uint64_t* in, uint64_t* out, int64_t n, uint64_t* total_dev) {
    PLB_LAUNCH("scan_u64", (k_scan_u64<uint64_t>), 1, 1024, 0, in, out, n, total_dev);
}

struct FilterCol { const void* in; void* out; const uint32_t* vin; uint32_t* vout; int elem; int pad; };
constexpr int F_MAX_COLS = 16;
struct FilterArgs { FilterCol c[F_MAX_COLS]; };

// grid.x = tiles (grid-stride), grid.y = column
__global__ void __launch_bounds__(F_THREADS) k_compact(FilterArgs args, const uint32_t* __restrict__ mask, const uint64_t* __restrict__ tile_off, int64_t n, int64_t ntiles) {
    const FilterCol col = args.c[blockIdx.y];
    __shared__ uint32_t wmask[F_TILE_WORDS];
    __shared__ uint32_t wpre[F_TILE_WORDS];
    const unsigned lane = lane_id(), warp = threadIdx.x >> 5;
    for (int64_t t = blockIdx.x; t < ntiles; t += gridDim.x) {
        const int64_t row_base = t * F_TILE;
        // load the tile's 128 mask words, exclusive-scan their popcounts (first 4 warps: 32 words each)
        if (threadIdx.x < F_TILE_WORDS) {
            int64_t w = t * F_TILE_WORDS + threadIdx.x;
            int64_t row0 = w * 32;
            uint32_t m = 0;
            if (row0 < n) { m = mask[w]; if (row0 + 32 > n) m &= (1u << (n - row0)) - 1u; }
            wmask[threadIdx.x] = m;
            uint32_t c = __popc(m), x = c;
            for (int o = 1; o < 32; o <<= 1) { uint32_t y = __shfl_up_sync(0xffffffffu, x, o); if (lane >= (unsigned)o) x += y; }
            wpre[threadIdx.x] = x - c;      // exclusive within this warp's 32 words
        }
        __syncthreads();
        // add the totals of the preceding 32-word groups (4 groups)
        __shared__ uint32_t gsum[5];
        if (threadIdx.x == 0) {
            uint32_t acc = 0;
            for (int g = 0; g < 4; g++) { gsum[g] = acc; acc += wpre[g * 32 + 31] + __popc(wmask[g * 32 + 31]); }
            gsum[4] = acc;
        }
        __syncthreads();
        const uint64_t out_base = tile_off[t];
        // values: lane l of a warp-step owns the row PAIR (2l, 2l+1) of a 64-row group — one 128-bit (8-byte elements) or 64-bit
        // load per kept pair, skipped when neither row is kept; unselected rows cost their sector anyway, so the wide load is free
        // (round 1 issued one 8-byte load and one store per thread-step and sat at 0.57-0.72 of the copy peak)
#pragma unroll 4
        for (int j = 0; j < F_TILE / (2 * F_THREADS); j++) {
            const int wa = (j * (F_THREADS / 32) + warp) * 2;
            if ((wmask[wa] | wmask[wa + 1]) == 0) continue;          // warp-uniform
            const int w = wa + (lane >> 4);
            const unsigned b0 = (lane & 15) * 2;
            const uint32_t m = wmask[w];
            const bool k0 = (m >> b0) & 1u, k1 = (m >> (b0 + 1)) & 1u;
            if (!(k0 | k1)) continue;
            const uint64_t dst = out_base + gsum[w >> 5] + wpre[w] + __popc(m & ((1u << b0) - 1u));
            const int64_t row = row_base + (int64_t)w * 32 + b0;
            if (col.elem == 8) {
                uint64_t v0, v1 = 0;
                if (row + 1 < n) { const ulonglong2 v = ld_stream_u64x2(reinterpret_cast<const uint64_t*>(col.in) + row); v0 = v.x; v1 = v.y; }
                else v0 = reinterpret_cast<const uint64_t*>(col.in)[row];
                uint64_t* o = reinterpret_cast<uint64_t*>(col.out);
                if (k0) o[dst] = v0;
                if (k1) o[dst + (k0 ? 1 : 0)] = v1;
            } else {
                uint32_t v0, v1 = 0;
                if (row + 1 < n) { const uint2 v = ld_stream_u32x2(reinterpret_cast<const uint32_t*>(col.in) + row); v0 = v.x; v1 = v.y; }
                else v0 = reinterpret_cast<const uint32_t*>(col.in)[row];
                uint32_t* o = reinterpret_cast<uint32_t*>(col.out);
                if (k0) o[dst] = v0;
                if (k1) o[dst + (k0 ? 1 : 0)] = v1;
            }
        }
        // validity: one 32-row mask word per warp-step (rows row_base + j*256 + tid; word index = j*8 + warp)
        if (col.vin != nullptr) {
#pragma unroll 4
            for (int j = 0; j < F_TILE / F_THREADS; j++) {
                const int widx = j * (F_THREADS / 32) + warp;
                const uint32_t m = wmask[widx];
                if (m == 0) continue;                                  // warp-uniform
                const bool keep = (m >> lane) & 1u;
                // compact the validity bits of this 32-row word: kept rows occupy output bits
                // [first, first + cnt) — build them with a warp OR-reduce, then <= 2 atomicOr
                const uint32_t vw = col.vin[row_base / 32 + widx];
                const uint32_t bit = (keep && ((vw >> lane) & 1u)) ? 1u : 0u;
                const uint32_t rw = __popc(m & lanemask_lt());       // rank inside the warp
                const uint64_t first = out_base + gsum[widx >> 5] + wpre[widx];
                const unsigned sh = (unsigned)(first & 31);
                uint64_t contrib = (uint64_t)bit << (rw + sh);       // rw + sh <= 62
                uint32_t lo = __reduce_or_sync(0xffffffffu, (uint32_t)contrib);
                uint32_t hi = __reduce_or_sync(0xffffffffu, (uint32_t)(contrib >> 32));
                if (lane == 0) {
                    if (lo) atomicOr(&col.vout[first >> 5], lo);
                    if (hi) atomicOr(&col.vout[(first >> 5) + 1], hi);
                }
            }
        }
        __syncthreads();
    }
}

void op_filter(const std::vector<DevCol>& cols, const DevCol& mask, std::vector<DevCol>& outs) {
    PLB_REQUIRE(mask.dtype == BL_BOOL, BL_ERR_DTYPE, "filter: mask must be BL_BOOL");
    const int64_t n = mask.len;
    for (auto& c : cols) {
        PLB_REQUIRE(c.len == n, BL_ERR_INVALID, "filter: column length " + std::to_string(c.len) + " != mask length " + std::to_string(n));
        PLB_REQUIRE(dtype_size(c.dtype) == 8 || dtype_size(c.dtype) == 4, BL_ERR_UNSUPPORTED, std::string("filter: dtype ") + dtype_name(c.dtype) + " is outside the hot path");
    }
    outs.clear();
    // null mask slots count as false (filter/mod.rs:21-27)
    DevPtr eff = mask.values;
    if (mask.validity) eff = bitmap_and(as<uint32_t>(mask.values), mask.vm(), nullptr, n);
    const uint32_t* m = as<uint32_t>(eff);
    const int64_t ntiles = (n + F_TILE - 1) / F_TILE;
    uint64_t total = 0;
    DevPtr counts, offs, tot;
    if (n > 0) {
        counts = dev_alloc((size_t)ntiles * 4); offs = dev_alloc((size_t)ntiles * 8); tot = dev_alloc(8);
        PLB_LAUNCH("k3_tile_counts", k_mask_tile_counts, grid_for(ntiles * 128, 128, 16), 128, 0, m, n, as<uint32_t>(counts), ntiles);
        exclusive_scan_u32_to_u64(as<uint32_t>(counts), as<uint64_t>(offs), ntiles, as<uint64_t>(tot));
        total = read_scalar(as<uint64_t>(tot));
    }
    for (auto& c : cols) {
        DevCol o = make_col(c.dtype, (int64_t)total, c.validity != nullptr);
        if (o.validity) dev_memset(o.validity->p, 0, o.validity->bytes);
        outs.push_back(o);
    }
    if (total == 0 || cols.empty()) return;
    for (size_t base = 0; base < cols.size(); base += F_MAX_COLS) {
        FilterArgs a; memset(&a, 0, sizeof a);
        int nc = (int)std::min<size_t>(F_MAX_COLS, cols.size() - base);
        for (int i = 0; i < nc; i++) {
            a.c[i].in = cols[base + i].v(); a.c[i].out = outs[base + i].values->p;
            a.c[i].vin = cols[base + i].vm(); a.c[i].vout = as<uint32_t>(outs[base + i].validity);
            a.c[i].elem = dtype_size(cols[base + i].dtype);
        }
        dim3 grid((unsigned)std::min<int64_t>(ntiles, (int64_t)ctx().sm_count * 8), (unsigned)nc);
        PLB_LAUNCH("k3_compact", k_compact, grid, F_THREADS, 0, a, m, as<uint64_t>(offs), n, ntiles);
    }
}

// ---------------------------------------------------------------------------- radix sort
// Stable ascending LSD radix sort of (key, u32 value) pairs, 8-bit digits, keys u32 or u64.  It serves the internal
// ordering modes (maintain_order, ascending row lists of duplicate build keys, GroupsIdx: sort_pairs_u32) and the
// public sort (sort.cu: one stage per encoded key column).  Per pass over digit `shift / 8`:
//   k_rs_hist     every CTA owns one contiguous chunk of the input; 256-bin shared-memory histogram -> hist[digit][cta],
//                 plus the digit's total over all CTAs (one atomic per CTA and digit)
//   k_rs_scan     one CTA per digit: start of every (digit, cta) run = totals of the smaller digits + the exclusive scan
//                 of the digit's row (the rows are independent, so the scan costs one launch instead of one long CTA)
//   k_rs_scatter  the CTA walks its chunk tile by tile, in order.  Inside a tile warp w owns a contiguous segment and
//                 ranks its items 32 at a time with __match_any_sync (lanes holding the same digit): rank = the warp's
//                 running count of the digit + the number of equal-digit lanes below — original order is kept at every
//                 level (tile, warp segment, round, lane), which is what makes the pass stable.  The tile is then
//                 staged in shared memory in digit order and every (tile, digit) run is written out contiguously, so
//                 consecutive lanes store consecutive addresses (the K5r / K6 scatter design) instead of one sector each.
// Only digits whose bits vary over the input are processed (`vary` = AND ^ OR of the keys, or the low key_bits).
constexpr int RS_THREADS = 256, RS_ITEMS = 16, RS_TILE = RS_THREADS * RS_ITEMS, RS_WARPS = RS_THREADS / 32;
constexpr int RS_MAX_CTAS = 1024;        // one k_rs_scan CTA covers a digit's row

template <typename K>
__global__ void __launch_bounds__(RS_THREADS) k_rs_hist(const K* __restrict__ keys, int64_t n, int64_t chunk, int shift, uint32_t* __restrict__ hist, int n_ctas,
                                                        uint32_t* __restrict__ digit_tot) {
    __shared__ unsigned h[256];
    h[threadIdx.x] = 0;
    __syncthreads();
    const int64_t lo = (int64_t)blockIdx.x * chunk, hi = min(n, lo + chunk);
    for (int64_t i = lo + threadIdx.x; i < hi; i += RS_THREADS) atomicAdd(&h[(unsigned)(keys[i] >> shift) & 255u], 1u);
    __syncthreads();
    const unsigned c = h[threadIdx.x];
    hist[(int64_t)threadIdx.x * n_ctas + blockIdx.x] = c;
    if (c) atomicAdd(&digit_tot[threadIdx.x], c);
}

// grid = 256 (one CTA per digit), block = RS_MAX_CTAS
__global__ void __launch_bounds__(RS_MAX_CTAS) k_rs_scan(const uint32_t* __restrict__ hist, const uint32_t* __restrict__ digit_tot, uint64_t* __restrict__ starts, int n_ctas) {
    __shared__ uint64_t warp_sums[32];
    const unsigned lane = lane_id(), warp = threadIdx.x >> 5, d = blockIdx.x;
    // base of the digit = sum of the totals of the smaller digits (warps 0..7 hold digits 0..255)
    uint64_t b = (threadIdx.x < d) ? digit_tot[threadIdx.x] : 0;
    for (int o = 16; o; o >>= 1) b += __shfl_xor_sync(0xffffffffu, b, o);
    if (lane == 0) warp_sums[warp] = b;
    __syncthreads();
    uint64_t base = 0;
    for (int w = 0; w < RS_MAX_CTAS / 32; w++) base += warp_sums[w];
    __syncthreads();
    const uint64_t v = (int)threadIdx.x < n_ctas ? hist[(int64_t)d * n_ctas + threadIdx.x] : 0;
    uint64_t x = v;
    for (int o = 1; o < 32; o <<= 1) { uint64_t y = __shfl_up_sync(0xffffffffu, x, o); if (lane >= (unsigned)o) x += y; }
    if (lane == 31) warp_sums[warp] = x;
    __syncthreads();
    if (warp == 0) {
        uint64_t s = warp_sums[lane], t = s;
        for (int o = 1; o < 32; o <<= 1) { uint64_t y = __shfl_up_sync(0xffffffffu, t, o); if (lane >= (unsigned)o) t += y; }
        warp_sums[lane] = t - s;
    }
    __syncthreads();
    if ((int)threadIdx.x < n_ctas) starts[(int64_t)d * n_ctas + threadIdx.x] = base + warp_sums[warp] + x - v;
}

// dynamic shared memory: RS_TILE keys followed by RS_TILE values
template <typename K>
__global__ void __launch_bounds__(RS_THREADS) k_rs_scatter(const K* __restrict__ keys_in, const uint32_t* __restrict__ vals_in, K* __restrict__ keys_out, uint32_t* __restrict__ vals_out,
                                                           int64_t n, int64_t chunk, int shift, const uint64_t* __restrict__ starts, int n_ctas) {
    extern __shared__ __align__(16) unsigned char rs_smem[];
    K* skey = reinterpret_cast<K*>(rs_smem);
    uint32_t* sval = reinterpret_cast<uint32_t*>(skey + RS_TILE);
    __shared__ unsigned warp_cnt[RS_WARPS][256];
    __shared__ unsigned dstart[256];            // tile-local start of each digit's run
    __shared__ unsigned scan_w[RS_WARPS];
    __shared__ unsigned long long gbase[256];
    const unsigned lane = lane_id(), warp = threadIdx.x >> 5;
    gbase[threadIdx.x] = starts[(int64_t)threadIdx.x * n_ctas + blockIdx.x];
    const int64_t lo = (int64_t)blockIdx.x * chunk, hi = min(n, lo + chunk);
    for (int64_t tile = lo; tile < hi; tile += RS_TILE) {
        for (int w = 0; w < RS_WARPS; w++) warp_cnt[w][threadIdx.x] = 0;
        __syncthreads();
        K k[RS_ITEMS]; uint32_t v[RS_ITEMS]; unsigned rank[RS_ITEMS];
#pragma unroll
        for (int r = 0; r < RS_ITEMS; r++) {
            const int64_t i = tile + ((int64_t)warp * RS_ITEMS + r) * 32 + lane;
            const bool in = i < hi;
            k[r] = in ? keys_in[i] : K(0); v[r] = in ? vals_in[i] : 0u;
            const unsigned d = in ? ((unsigned)(k[r] >> shift) & 255u) : 256u;     // 256 = "no item": its own match class
            const unsigned peers = __match_any_sync(0xffffffffu, d);
            const unsigned leader = __ffs(peers) - 1;
            unsigned old = 0;
            if (in && lane == leader) { old = warp_cnt[warp][d]; warp_cnt[warp][d] = old + __popc(peers); }
            old = __shfl_sync(0xffffffffu, old, leader);
            rank[r] = old + __popc(peers & lanemask_lt());
            __syncwarp();
        }
        __syncthreads();
        // digit = threadIdx.x: the warps' exclusive offsets inside the digit's run, then the tile-local start of every run
        unsigned tot = 0;
        for (int w = 0; w < RS_WARPS; w++) { const unsigned c = warp_cnt[w][threadIdx.x]; warp_cnt[w][threadIdx.x] = tot; tot += c; }
        unsigned x = tot;
        for (int o = 1; o < 32; o <<= 1) { const unsigned y = __shfl_up_sync(0xffffffffu, x, o); if (lane >= (unsigned)o) x += y; }
        if (lane == 31) scan_w[warp] = x;
        __syncthreads();
        unsigned wbase = 0;
        for (int w = 0; w < (int)warp; w++) wbase += scan_w[w];
        dstart[threadIdx.x] = wbase + x - tot;
        __syncthreads();
        // stage the tile in digit order
#pragma unroll
        for (int r = 0; r < RS_ITEMS; r++) {
            const int64_t i = tile + ((int64_t)warp * RS_ITEMS + r) * 32 + lane;
            if (i < hi) {
                const unsigned d = (unsigned)(k[r] >> shift) & 255u;
                const unsigned p = dstart[d] + warp_cnt[warp][d] + rank[r];
                skey[p] = k[r]; sval[p] = v[r];
            }
        }
        __syncthreads();
        // write every (tile, digit) run contiguously: staged position p of digit d goes to gbase[d] + (p - dstart[d])
        const int cnt = (int)min((int64_t)RS_TILE, hi - tile);
#pragma unroll 4
        for (int p = threadIdx.x; p < cnt; p += RS_THREADS) {
            const K kk = skey[p];
            const unsigned d = (unsigned)(kk >> shift) & 255u;
            const unsigned long long pos = gbase[d] + (unsigned)(p - dstart[d]);
            keys_out[pos] = kk; vals_out[pos] = sval[p];
        }
        __syncthreads();
        gbase[threadIdx.x] += tot;
    }
}

template <typename K>
static bool radix_sort_pairs(K* k0, uint32_t* v0, K* k1, uint32_t* v1, int64_t n, uint64_t vary, int* passes_run) {
    int digits[8], passes = 0;
    for (int d = 0; d < (int)sizeof(K); d++) if ((vary >> (8 * d)) & 255u) digits[passes++] = d;
    if (passes_run) *passes_run = n > 1 ? passes : 0;
    if (n <= 1 || passes == 0) return false;
    PLB_REQUIRE(n <= (int64_t)0xFFFFFFFFll, BL_ERR_UNSUPPORTED, "radix sort: more than 2^32 - 1 rows");
    Context& c = ctx();
    const size_t smem = (size_t)RS_TILE * (sizeof(K) + 4);
    static bool attr_set = false;        // serialised by the context lock
    if (!attr_set) {
        PLB_CUDA(cudaFuncSetAttribute(k_rs_scatter<uint32_t>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(RS_TILE * 8)));
        PLB_CUDA(cudaFuncSetAttribute(k_rs_scatter<uint64_t>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(RS_TILE * 12)));
        attr_set = true;
    }
    int per_sm = 0;
    PLB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_rs_scatter<K>, RS_THREADS, smem));
    const int64_t tiles = (n + RS_TILE - 1) / RS_TILE;
    const int n_ctas0 = (int)std::min<int64_t>(tiles, std::min<int64_t>((int64_t)c.sm_count * std::max(per_sm, 1), RS_MAX_CTAS));
    const int64_t chunk = (tiles + n_ctas0 - 1) / n_ctas0 * RS_TILE;
    const int n_ctas = (int)((n + chunk - 1) / chunk);       // no empty trailing CTA
    DevPtr hist = dev_alloc((size_t)256 * n_ctas * 4), starts = dev_alloc((size_t)256 * n_ctas * 8), tot = dev_alloc((size_t)passes * 256 * 4);
    dev_memset(tot->p, 0, (size_t)passes * 256 * 4);
    K *ki = k0, *ko = k1;
    uint32_t *vi = v0, *vo = v1;
    for (int p = 0; p < passes; p++) {
        const int shift = 8 * digits[p];
        uint32_t* dt = as<uint32_t>(tot) + 256 * p;
        PLB_LAUNCH("sort_hist", k_rs_hist<K>, n_ctas, RS_THREADS, 0, ki, n, chunk, shift, as<uint32_t>(hist), n_ctas, dt);
        PLB_LAUNCH("sort_scan", k_rs_scan, 256, RS_MAX_CTAS, 0, as<uint32_t>(hist), dt, as<uint64_t>(starts), n_ctas);
        PLB_LAUNCH("sort_scatter", k_rs_scatter<K>, n_ctas, RS_THREADS, smem, ki, vi, ko, vo, n, chunk, shift, as<uint64_t>(starts), n_ctas);
        std::swap(ki, ko); std::swap(vi, vo);
    }
    return ki != k0;
}

bool radix_sort_pairs_u32(uint32_t* k0, uint32_t* v0, uint32_t* k1, uint32_t* v1, int64_t n, uint64_t vary, int* passes_run) {
    return radix_sort_pairs<uint32_t>(k0, v0, k1, v1, n, vary, passes_run);
}
bool radix_sort_pairs_u64(uint64_t* k0, uint32_t* v0, uint64_t* k1, uint32_t* v1, int64_t n, uint64_t vary, int* passes_run) {
    return radix_sort_pairs<uint64_t>(k0, v0, k1, v1, n, vary, passes_run);
}

void sort_pairs_u32(uint32_t* keys, uint32_t* vals, int64_t n, int key_bits) {
    if (n <= 1) return;
    if (key_bits < 1 || key_bits > 32) key_bits = 32;
    const int passes = (key_bits + 7) / 8;
    const uint64_t digits = passes == 4 ? 0xFFFFFFFFull : ((1ull << (8 * passes)) - 1);
    DevPtr k2 = dev_alloc((size_t)n * 4), v2 = dev_alloc((size_t)n * 4);
    if (radix_sort_pairs<uint32_t>(keys, vals, as<uint32_t>(k2), as<uint32_t>(v2), n, digits, nullptr)) {
        PLB_CUDA(cudaMemcpyAsync(keys, k2->p, (size_t)n * 4, cudaMemcpyDeviceToDevice, ctx().stream));
        PLB_CUDA(cudaMemcpyAsync(vals, v2->p, (size_t)n * 4, cudaMemcpyDeviceToDevice, ctx().stream));
    }
}

}  // namespace plb
