// groupby_radix.cu — K5r: the partitioned group_by plan for tables that cannot stay resident in L2.
//
// Reference path being replaced: the same as groupby.cu (group_by_threaded_slice, polars-core/src/frame/group_by/
// hashing.rs:116-167, which ALSO partitions the keys by hash_to_partition before it builds one table per partition, and
// agg_sum/mean/min/max, aggregations/mod.rs:486-1018).  groupby.cu aggregates with L2 atomics into one open-addressing
// table; once that table outgrows L2 every RED becomes a DRAM read-modify-write.  This plan moves the rows instead of the atomics:
//   pass 0  k_gbr_hist      rows per bucket (bucket = top bits of table_hash(key): the slot function of the L2 plan), only
//                           when the sample cannot size the bucket streams (consume_radix: "exact" sizing)
//   pass 1  k_gbr_scatter   every CTA sorts a 2048-row tile by bucket in shared memory as ROW-MAJOR records
//                           [key, v0, v1, ...] (packed: [key offset | v0, v1, ...], see GbRadixDev) and writes each
//                           (tile, bucket) run with ONE cp.async.bulk (TMA)
//                           shared->global copy (runs padded to an even record count with a GB_EMPTY-key record so both
//                           ends stay 16-byte aligned).  Past 512 buckets the runs shrink to single records:
//           k_gbr_scatter_wc    instead collects every bucket's rows in a 4-record chunk buffer in shared memory
//                           (software write-combining) and writes each full chunk with one cp.async.bulk copy of
//                           whole 32-byte sectors; when a buffer per bucket does not fit one CTA's shared memory,
//                           k_gbr_scatter writes the sorted tile with coalesced 8-byte stores (no padding).
//   pass 2  k_gbr_agg       one CTA per bucket: the bucket's record stream is staged into shared memory by
//                           cp.async.bulk (TMA) global->shared copies on an mbarrier ring (a producer warp issues,
//                           31 consumer warps each release their slice of a stage on an `empty` mbarrier, behind a
//                           proxy fence, as soon as it sits in registers); rows aggregate into a shared-memory
//                           open-addressing table; a bucket's groups are final, so they leave compacted straight into
//                           the dense output arrays — the global table, its initialisation and its extraction disappear.
// While the L2 plan's table stays in L2 this plan loses to it (64-bit shared-memory atomics on random slots cost several
// SM cycles per row), so it is only taken when the L2 plan's table would exceed the L2 budget.
// Restrictions (anything else stays on the L2 plan): no validity bitmaps, no first-row tracking, <= 4 value columns,
// no heavy hitters in the sample.  Records are packed (one 8-byte word less) when the sample puts the key in a window of
// 2^32 - 1 offsets and one value column in 32 bits; the plan (buckets, table, store path, stream sizing) is the one of
// the plain width either way.  Exact for any input: a row outside the packed form raises status 4 and the caller redoes
// the batch with plain records; a bucket that outgrows the stream the sample sized for it raises status 2 and the
// caller redoes the batch with capacities from the exact histogram (both at once: one redo, plain and exactly sized);
// a bucket with more groups than its shared-memory table holds raises status 1 and the caller redoes the batch on the
// L2 plan.
#include <algorithm>
#include <cstdlib>

#include "common.cuh"
#include "dev_utils.cuh"
#include "groupby.h"
#include "groupby_dev.cuh"

namespace plb {

constexpr int GBR_THREADS = 512;      // pass 1: 2048-row tiles (bulk stores) / 4096-row tiles (many buckets: longer runs per bucket)
constexpr int GBR_MAX_LOGB = 13;
constexpr int GBR_NCW = 31, GBR_NCT = GBR_NCW * 32;                                    // pass 2: 31 consumer warps + 1 producer warp
// pass 1: a reservation that would end past its bucket's stream (R.cap records) stores nothing and sets status 2 (GBR_ST_STREAM); pass 2
// then returns at entry and the caller redoes the batch with exact sizing.  The bound is a kernel parameter rather than
// off[p + 1] - off[p]: two more loads per reservation made ptxas spill in k_gbr_scatter_wc<3, 8, *>.
constexpr unsigned GBR_NO_ROOM = 0xFFFFFFFFu;

// status bits (atomicOr: one attempt may raise several; pass 2 returns at entry on GBR_ST_STREAM | GBR_ST_UNFIT)
constexpr int GBR_ST_TABLE = 1;       // a bucket's pass-2 table overflowed (or the dense output bound): the L2 plan redoes the batch
constexpr int GBR_ST_STREAM = 2;      // a bucket's record stream overflowed (pass 1): redone with exact sizing
constexpr int GBR_ST_UNFIT = 4;       // a row does not fit the packed records (pass 1): redone with plain records

struct GbRadixDev {
    uint64_t* recs;                 // record streams, bucket b at recs + off[b] * (record words)
    const unsigned long long* off;  // first record of bucket b (even; a multiple of GBR_WC_F for the write-combining scatter)
    unsigned* cursor;               // records written to bucket b so far (pads included)
    unsigned* counts;               // pass 0 (exact sizing): rows of bucket b
    int logB, roww;
    uint64_t* special;              // accumulator row of the GB_EMPTY-key group: [len, words...] (RED target; rare rows only)
    unsigned cap;                   // records of every bucket stream (sample sizing); ~0u: exact sizing, whose streams hold their rows by construction
    int* status;                    // GBR_ST_* bits
    // Packed records (the PACK form of the kernels): word 0 = (key - pk_base) as a u32 in its low half and value column 0
    // as a u32 in its high half, columns 1.. in their own words: ROWW - 1 words instead of ROWW.  Offset GBR_PK_PAD is the
    // pad marker.  Column 0 widens back to the 64-bit raw pattern by sign extension (Int64) or zero extension (4-byte
    // columns, whose raw pattern is the zero-extended value, and UInt64).
    uint64_t pk_base;
    int pk_sext;
};
constexpr uint32_t GBR_PK_PAD = 0xFFFFFFFFu;
// word 0 of a packed record; fit = false when the key lies outside the window or the value does not widen back to itself
__device__ __forceinline__ uint64_t gbr_pack(const GbRadixDev& R, uint64_t key, uint64_t v, bool& fit) {
    const uint64_t off = key - R.pk_base, wide = R.pk_sext ? (uint64_t)(int64_t)(int32_t)(uint32_t)v : (uint64_t)(uint32_t)v;
    fit = off < GBR_PK_PAD && wide == v;
    return (uint64_t)(uint32_t)off | (v << 32);
}
__device__ __forceinline__ uint64_t gbr_unpack_value(const GbRadixDev& R, uint64_t w) {
    return R.pk_sext ? (uint64_t)(int64_t)(int32_t)(uint32_t)(w >> 32) : w >> 32;
}
// record words of the unpacked width ROWW
template <int ROWW, bool PACK> constexpr int gbr_rw() { return PACK ? ROWW - 1 : ROWW; }
// one record at rec: [key, v0, v1, ...] or, packed, [pack(key, v0), v1, ...].  A row that does not fit the packed form
// raises GBR_ST_UNFIT (the status is read first: rows of a batch that misses the window would otherwise queue atomics on
// one address).  Its record is written all the same: pass 2 does not run on such a batch.
template <int NC, bool PACK, class Val>
__device__ __forceinline__ void gbr_put(uint64_t* rec, const GbRadixDev& R, uint64_t key, Val val) {
    if constexpr (PACK) {
        bool fit;
        rec[0] = gbr_pack(R, key, val(0), fit);
        if (!fit && !(*reinterpret_cast<volatile int*>(R.status) & GBR_ST_UNFIT)) atomicOr(R.status, GBR_ST_UNFIT);
#pragma unroll
        for (int c = 1; c < NC; c++) rec[c] = val(c);
    } else {
        rec[0] = key;
#pragma unroll
        for (int c = 0; c < NC; c++) rec[1 + c] = val(c);
    }
}

// gb_load_pair of rows r0, r0 + 1 with a bounds check against n (rows past the end read as 0)
template <int KEY_ELEM> __device__ __forceinline__ void gbr_load_pair(const void* col, int64_t r0, int64_t n, uint64_t& a, uint64_t& b) {
    a = 0; b = 0;
    if (r0 + 1 < n) gb_load_pair<KEY_ELEM>(col, r0, a, b);
    else if (r0 < n) a = KEY_ELEM == 8 ? reinterpret_cast<const uint64_t*>(col)[r0] : reinterpret_cast<const uint32_t*>(col)[r0];
}
__device__ __forceinline__ void gbr_load_pair_rt(const void* col, int elem, int64_t r0, int64_t n, uint64_t& a, uint64_t& b) {
    if (elem == 8) gbr_load_pair<8>(col, r0, n, a, b); else gbr_load_pair<4>(col, r0, n, a, b);
}

// ---------------------------------------------------------------------------- pass 0: exact bucket sizes
template <int KEY_ELEM, int KEY_CANON>
__global__ void __launch_bounds__(512) k_gbr_hist(const void* __restrict__ keys, int64_t n, int logB, unsigned* __restrict__ counts) {
    extern __shared__ unsigned h_s[];
    const int B = 1 << logB;
    for (int i = threadIdx.x; i < B; i += blockDim.x) h_s[i] = 0;
    __syncthreads();
    const int64_t npairs = (n + 1) >> 1;
    for (int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; p < npairs; p += (int64_t)gridDim.x * blockDim.x) {
        uint64_t k0, k1;
        gbr_load_pair<KEY_ELEM>(keys, 2 * p, n, k0, k1);
        k0 = canon_key<KEY_CANON>(k0); k1 = canon_key<KEY_CANON>(k1);
        if (k0 != GB_EMPTY) atomicAdd(&h_s[(unsigned)(table_hash(k0) >> (64 - logB))], 1u);
        if (2 * p + 1 < n && k1 != GB_EMPTY) atomicAdd(&h_s[(unsigned)(table_hash(k1) >> (64 - logB))], 1u);
    }
    __syncthreads();
    for (int i = threadIdx.x; i < B; i += blockDim.x) if (h_s[i]) atomicAdd(&counts[i], h_s[i]);
}
// records of a bucket stream for `rows` rows: worst-case padding, `pad_each` records for each of up to `pad_units` writers
// that touch the bucket (tile runs: one per tile; write-combining: F - 1 per CTA), rounded up to `align` records so that
// every stream starts 16-byte (even) / 32-byte (F) aligned
__host__ __device__ __forceinline__ unsigned long long gbr_stream_records(unsigned long long rows, unsigned long long pad_units, unsigned pad_each, unsigned align) {
    rows += (rows < pad_units ? rows : pad_units) * pad_each;
    return (rows + align - 1) & ~(unsigned long long)(align - 1);
}
// set-up of pass 1, one CTA: exclusive stream offsets from the exact row counts of k_gbr_hist (counts != nullptr) or from
// `rows` rows for every bucket; zero cursors and status; the identities of the special row (a redone batch starts afresh)
__global__ void __launch_bounds__(1024) k_gbr_offsets(const __grid_constant__ GbLayout L, const unsigned* __restrict__ counts, unsigned long long rows, int B, unsigned long long pad_units,
                                                      unsigned pad_each, unsigned align, unsigned long long* __restrict__ off, unsigned* __restrict__ cursor, uint64_t* __restrict__ special, int* __restrict__ status) {
    __shared__ unsigned long long wsum[32];
    __shared__ unsigned long long carry_s;
    if (threadIdx.x == 0) { carry_s = 0; *status = 0; special[0] = 0; }
    if (threadIdx.x < (unsigned)L.n_words) special[1 + threadIdx.x] = L.init[threadIdx.x];
    __syncthreads();
    const unsigned lane = lane_id(), warp = threadIdx.x >> 5;
    for (int base = 0; base < B; base += 1024) {
        const int i = base + threadIdx.x;
        unsigned long long c = 0;
        if (i < B) { c = gbr_stream_records(counts ? counts[i] : rows, pad_units, pad_each, align); cursor[i] = 0; }
        unsigned long long x = c;
        for (int o = 1; o < 32; o <<= 1) { const unsigned long long y = __shfl_up_sync(0xffffffffu, x, o); if (lane >= (unsigned)o) x += y; }
        if (lane == 31) wsum[warp] = x;
        __syncthreads();
        if (warp == 0) {
            unsigned long long s = wsum[lane], t = s;
            for (int o = 1; o < 32; o <<= 1) { const unsigned long long y = __shfl_up_sync(0xffffffffu, t, o); if (lane >= (unsigned)o) t += y; }
            wsum[lane] = t - s;
        }
        __syncthreads();
        const unsigned long long incl = carry_s + wsum[warp] + x;
        if (i < B) off[i] = incl - c;
        __syncthreads();
        if (threadIdx.x == 1023) carry_s = incl;
        __syncthreads();
    }
    if (threadIdx.x == 0) off[B] = carry_s;
}

// ---------------------------------------------------------------------------- pass 1: tile sort + TMA bulk stores
// the GB_EMPTY key is the pad marker of the record streams: its (rare) rows aggregate straight into sp = [len, words...].
// Not gb_apply: inlined into the scatters, gb_apply changed ptxas's register allocation of every k_gbr_scatter /
// k_gbr_scatter_wc instantiation (k_gbr_scatter_wc<3, 8, 0>: a 16-byte frame without spills became 64 bytes with spills).
__device__ __forceinline__ void gbr_apply_special(const GbLayout& L, const GbBatch& Bt, uint64_t* sp, const uint64_t* raw) {
    atomicAdd(reinterpret_cast<unsigned long long*>(sp), 1ull);
    for (int c = 0; c < L.n_cols; c++)
        for (int k = L.col_kbegin[c]; k < L.col_kbegin[c + 1]; k++) {
            uint64_t* a = sp + 1 + L.wslot[k];
            const int dt = Bt.cols[c].dtype;
            switch (L.wop[k]) {
                case W_ADD_INT: atomicAdd(reinterpret_cast<unsigned long long*>(a), (unsigned long long)raw_to_int(dt, raw[c])); break;
                case W_ADD_F64: atomicAdd(reinterpret_cast<double*>(a), raw_to_f64(dt, raw[c])); break;
                case W_MIN_S64: atomicMin(reinterpret_cast<long long*>(a), (long long)raw_to_int(dt, raw[c])); break;
                case W_MAX_S64: atomicMax(reinterpret_cast<long long*>(a), (long long)raw_to_int(dt, raw[c])); break;
                case W_MIN_U64: atomicMin(reinterpret_cast<unsigned long long*>(a), (unsigned long long)raw[c]); break;
                case W_MAX_U64: atomicMax(reinterpret_cast<unsigned long long*>(a), (unsigned long long)raw[c]); break;
                case W_MIN_F64: { const double f = raw_to_f64(dt, raw[c]); if (f == f) atomicMin(reinterpret_cast<unsigned long long*>(a), (unsigned long long)f64_to_ordered(f)); break; }
                case W_MAX_F64: { const double f = raw_to_f64(dt, raw[c]); if (f == f) atomicMax(reinterpret_cast<unsigned long long*>(a), (unsigned long long)f64_to_ordered(f)); break; }
                default: break;
            }
        }
}

constexpr int GBR_RPT = 4;      // rows per thread: 2048-row tiles (8 rows per thread, 4096-row tiles at 1 CTA / SM, was slower)
template <int ROWW, int KEY_ELEM, int KEY_CANON, bool BULK, bool PACK>
__global__ void __launch_bounds__(GBR_THREADS) k_gbr_scatter(const __grid_constant__ GbLayout L, const __grid_constant__ GbBatch Bt, const __grid_constant__ GbRadixDev R) {
    constexpr int RPT = GBR_RPT, T = GBR_THREADS * RPT, THREADS = GBR_THREADS, NC = ROWW - 1, RW = gbr_rw<ROWW, PACK>();
    const int logB = R.logB, B = 1 << logB;
    extern __shared__ __align__(16) uint64_t gbr_smem[];
    uint64_t* stage = gbr_smem;                                        // (T + (BULK ? B : 0)) records
    unsigned* hist = reinterpret_cast<unsigned*>(stage + (size_t)(T + (BULK ? B : 0)) * RW);
    unsigned* start = hist + B;
    unsigned* gpos = start + B;
    uint16_t* sp = reinterpret_cast<uint16_t*>(gpos + B);             // !BULK: bucket of every sorted slot
    __shared__ unsigned warp_tot[THREADS / 32];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int64_t n = Bt.n;
    const int64_t ntiles = (n + T - 1) / T;
    for (int64_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
        const int64_t base = tile * T;
        for (int p = tid; p < B; p += THREADS) hist[p] = 0;
        __syncthreads();
        uint64_t k[RPT]; unsigned pk[RPT];      // pk: bucket << 16 | rank in the tile's run;  ~0 = no row;  ~0 - 1 = GB_EMPTY-key row
#pragma unroll
        for (int j = 0; j < RPT / 2; j++) gbr_load_pair<KEY_ELEM>(Bt.keys, base + 2 * (int64_t)(j * THREADS + tid), n, k[2 * j], k[2 * j + 1]);
#pragma unroll
        for (int j = 0; j < RPT; j++) {
            const int64_t r = base + 2 * (int64_t)((j >> 1) * THREADS + tid) + (j & 1);
            pk[j] = 0xFFFFFFFFu;
            if (r < n) {
                k[j] = canon_key<KEY_CANON>(k[j]);
                if (k[j] == GB_EMPTY) pk[j] = 0xFFFFFFFEu;
                else { const unsigned b = (unsigned)(table_hash(k[j]) >> (64 - logB)); pk[j] = (b << 16) | atomicAdd(&hist[b], 1u); }
            }
        }
        __syncthreads();
        // exclusive scan of the (padded) run lengths; one global reservation per non-empty (tile, bucket)
        const int bins = (B + THREADS - 1) / THREADS;
        unsigned mine = 0;
        for (int q = 0; q < bins; q++) { const int p = tid * bins + q; if (p < B) { unsigned c = hist[p]; if (BULK) c = (c + 1u) & ~1u; mine += c; } }
        unsigned x = mine;
        for (int o = 1; o < 32; o <<= 1) { const unsigned y = __shfl_up_sync(0xffffffffu, x, o); if (lane >= o) x += y; }
        if (lane == 31) warp_tot[warp] = x;
        __syncthreads();
        if (warp == 0) {
            unsigned w = lane < THREADS / 32 ? warp_tot[lane] : 0, s = w;
            for (int o = 1; o < 32; o <<= 1) { const unsigned y = __shfl_up_sync(0xffffffffu, s, o); if (lane >= o) s += y; }
            if (lane < THREADS / 32) warp_tot[lane] = s - w;
        }
        __syncthreads();
        unsigned run = warp_tot[warp] + x - mine;
        for (int q = 0; q < bins; q++) {
            const int p = tid * bins + q;
            if (p < B) {
                const unsigned c = hist[p], cp = BULK ? ((c + 1u) & ~1u) : c;
                start[p] = run;
                unsigned g = cp ? atomicAdd(&R.cursor[p], cp) : 0u;
                if (g + cp > R.cap) { atomicOr(R.status, GBR_ST_STREAM); g = GBR_NO_ROOM; }
                gpos[p] = g;
                run += cp;
            }
        }
        if (BULK) bulk_wait_read0();        // the previous tile's copies have finished reading the staging buffer
        __syncthreads();
        if (BULK) for (int p = tid; p < B; p += THREADS) { const unsigned c = hist[p]; if (c & 1u) { uint64_t* pad = stage + (size_t)(start[p] + c) * RW; pad[0] = PACK ? GBR_PK_PAD : GB_EMPTY;
#pragma unroll
                                                                                                      for (int w = 1; w < RW; w++) pad[w] = 0; } }
        // place the records (order inside a run is arbitrary)
#pragma unroll
        for (int j = 0; j < RPT / 2; j++) {
            const int64_t r0 = base + 2 * (int64_t)(j * THREADS + tid);
            uint64_t v[NC > 0 ? NC : 1][2];
#pragma unroll
            for (int c = 0; c < NC; c++) gbr_load_pair_rt(Bt.cols[c].values, Bt.cols[c].elem, r0, n, v[c][0], v[c][1]);
#pragma unroll
            for (int e = 0; e < 2; e++) {
                const unsigned q = pk[2 * j + e];
                if (q == 0xFFFFFFFFu) continue;
                if (q == 0xFFFFFFFEu) {      // the GB_EMPTY key is the pad marker of the record streams: its (rare) rows aggregate right here
                    uint64_t raw[NC > 0 ? NC : 1];
#pragma unroll
                    for (int c = 0; c < NC; c++) raw[c] = v[c][e];
                    gbr_apply_special(L, Bt, R.special, raw);
                    continue;
                }
                const unsigned bkt = q >> 16, pos = start[bkt] + (q & 0xFFFFu);
                gbr_put<NC, PACK>(stage + (size_t)pos * RW, R, k[2 * j + e], [&](int c) { return v[c][e]; });
                if (!BULK) sp[pos] = (uint16_t)bkt;
            }
        }
        if (BULK) fence_async_smem();
        __syncthreads();
        if (BULK) {
            for (int p = tid; p < B; p += THREADS) {
                const unsigned c = hist[p], cp = (c + 1u) & ~1u;
                if (cp && gpos[p] != GBR_NO_ROOM) bulk_s2g(R.recs + (R.off[p] + gpos[p]) * RW, stage + (size_t)start[p] * RW, cp * RW * 8);
            }
            bulk_commit();
        } else {
            const unsigned total = start[B - 1] + hist[B - 1];
            for (unsigned w = tid; w < total * RW; w += THREADS) {
                const unsigned row = w / RW, c = w - row * RW;
                const unsigned p = sp[row], g = gpos[p];
                if (g != GBR_NO_ROOM) R.recs[(R.off[p] + g + (row - start[p])) * RW + c] = stage[w];
            }
            __syncthreads();
        }
    }
    if (BULK) bulk_wait0();
}

// ---------------------------------------------------------------------------- pass 1, many buckets: write-combining buffers
// A persistent CTA keeps one chunk buffer of F records per bucket in shared memory.  Rows take a slot s in their bucket's
// chunk sequence with one shared-memory atomic; in round r the rows of chunk s / F == r land in the buffer, and every chunk
// that round completed leaves with one global reservation (atomicAdd(cursor, F)) and one cp.async.bulk shared->global
// copy.  Bucket streams start on whole chunks (k_gbr_offsets aligns them to F records), so every store is whole 32-byte
// sectors.  The next tile's keys and values load into registers while the current tile is bucketed.  At the end each
// CTA flushes its partial chunks padded with GB_EMPTY-key records (pass 2 skips them).
constexpr int GBR_WC_THREADS = 256, GBR_WC_F = 4;
template <int ROWW> constexpr int gbr_wc_rpt() { return ROWW <= 3 ? 8 : 4; }
template <int ROWW, int KEY_ELEM, int RPT>
__device__ __forceinline__ void gbr_wc_load(const GbBatch& Bt, int64_t base, uint64_t (&k)[RPT], uint64_t (&v)[ROWW > 1 ? ROWW - 1 : 1][RPT]) {
#pragma unroll
    for (int j = 0; j < RPT / 2; j++) {
        const int64_t r0 = base + 2 * (int64_t)(j * GBR_WC_THREADS + threadIdx.x);
        gbr_load_pair<KEY_ELEM>(Bt.keys, r0, Bt.n, k[2 * j], k[2 * j + 1]);
#pragma unroll
        for (int c = 0; c < ROWW - 1; c++) gbr_load_pair_rt(Bt.cols[c].values, Bt.cols[c].elem, r0, Bt.n, v[c][2 * j], v[c][2 * j + 1]);
    }
}

template <int ROWW, int KEY_ELEM, int KEY_CANON, bool PACK>
__global__ void __launch_bounds__(GBR_WC_THREADS, 2) k_gbr_scatter_wc(const __grid_constant__ GbLayout L, const __grid_constant__ GbBatch Bt, const __grid_constant__ GbRadixDev R) {
    constexpr int THREADS = GBR_WC_THREADS, F = GBR_WC_F, RPT = gbr_wc_rpt<ROWW>(), T = THREADS * RPT, NC = ROWW - 1, NCX = NC > 0 ? NC : 1, RW = gbr_rw<ROWW, PACK>(),
                  CH = F * RW;
    constexpr unsigned NONE = 0xFFFFFFFFu;
    const int logB = R.logB, B = 1 << logB, tid = threadIdx.x;
    extern __shared__ __align__(16) uint64_t gbr_smem[];
    uint64_t* buf = gbr_smem;                                                       // B chunks of CH words
    unsigned* fill = reinterpret_cast<unsigned*>(buf + (size_t)B * CH);             // records in the bucket's open chunk (< F between tiles)
    const int64_t n = Bt.n, ntiles = (n + T - 1) / T;
    for (int p = tid; p < B; p += THREADS) fill[p] = 0;
    uint64_t k[RPT], v[NCX][RPT], kn[RPT], vn[NCX][RPT];
    if ((int64_t)blockIdx.x < ntiles) gbr_wc_load<ROWW, KEY_ELEM, RPT>(Bt, (int64_t)blockIdx.x * T, kn, vn);
    for (int64_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
#pragma unroll
        for (int e = 0; e < RPT; e++) { k[e] = kn[e];
#pragma unroll
                                        for (int c = 0; c < NC; c++) v[c][e] = vn[c][e]; }
        if (tile + gridDim.x < ntiles) gbr_wc_load<ROWW, KEY_ELEM, RPT>(Bt, (tile + gridDim.x) * T, kn, vn);
        const int64_t base = tile * T;
        unsigned pk[RPT];        // bucket << 16 | slot in the bucket's chunk sequence of this tile;  NONE = no row
#pragma unroll
        for (int e = 0; e < RPT; e++) {
            const int64_t r = base + 2 * (int64_t)((e >> 1) * THREADS + tid) + (e & 1);
            pk[e] = NONE;
            if (r < n) {
                k[e] = canon_key<KEY_CANON>(k[e]);
                if (k[e] == GB_EMPTY) {      // the GB_EMPTY key is the pad marker of the record streams: its (rare) rows aggregate right here
                    uint64_t raw[NCX];
#pragma unroll
                    for (int c = 0; c < NC; c++) raw[c] = v[c][e];
                    gbr_apply_special(L, Bt, R.special, raw);
                } else pk[e] = (unsigned)(table_hash(k[e]) >> (64 - logB)) << 16;
            }
        }
        __syncthreads();                 // the previous tile's owners have reset fill[]
        unsigned last = 0;               // highest chunk index among this thread's rows
#pragma unroll
        for (int e = 0; e < RPT; e++)
            if (pk[e] != NONE) { const unsigned s = atomicAdd(&fill[pk[e] >> 16], 1u); pk[e] |= s; last = max(last, s / F); }
        bulk_wait_read0();               // this thread's copies of the previous tile have finished reading their buffers
        __syncthreads();
        for (unsigned r = 0;; r++) {
#pragma unroll
            for (int e = 0; e < RPT; e++) {
                const unsigned s = pk[e] & 0xFFFFu;
                if (pk[e] == NONE || s / F != r) continue;
                gbr_put<NC, PACK>(buf + (size_t)(pk[e] >> 16) * CH + (s % F) * RW, R, k[e], [&](int c) { return v[c][e]; });
            }
            fence_async_smem();
            const bool more = __syncthreads_or(last > r);
            // owners (bucket p belongs to thread p % THREADS) write out the chunks this round completed
            const unsigned full = (r + 1) * F;
            for (int p0 = 0; p0 < B; p0 += 4 * THREADS) {
                unsigned g[4];
#pragma unroll
                for (int q = 0; q < 4; q++) {            // reservations first, so their latencies overlap
                    const int p = p0 + q * THREADS + tid;
                    g[q] = NONE;
                    if (p < B) {
                        const unsigned f = fill[p];
                        if (f >= full) g[q] = atomicAdd(&R.cursor[p], (unsigned)F);
                        if (!more) fill[p] = f % F;
                    }
                }
#pragma unroll
                for (int q = 0; q < 4; q++) {
                    const int p = p0 + q * THREADS + tid;
                    if (g[q] == NONE) continue;
                    if (g[q] + F <= R.cap) bulk_s2g(R.recs + (R.off[p] + g[q]) * RW, buf + (size_t)p * CH, CH * 8);
                    else atomicOr(R.status, GBR_ST_STREAM);
                }
            }
            bulk_commit();
            if (!more) break;
            bulk_wait_read0();
            __syncthreads();
        }
    }
    // partial chunks, padded to F records with GB_EMPTY keys / GBR_PK_PAD offsets (their buffers are not in flight: a
    // chunk that left in the last round was full, which leaves its bucket's buffer empty)
    __syncthreads();
    for (int p = tid; p < B; p += THREADS) {
        const unsigned f = fill[p];
        if (f == 0) continue;
        for (unsigned i = f; i < F; i++) buf[(size_t)p * CH + i * RW] = PACK ? GBR_PK_PAD : GB_EMPTY;
        fence_async_smem();
        const unsigned g = atomicAdd(&R.cursor[p], (unsigned)F);
        if (g + F <= R.cap) bulk_s2g(R.recs + (R.off[p] + g) * RW, buf + (size_t)p * CH, CH * 8);
        else atomicOr(R.status, GBR_ST_STREAM);
    }
    bulk_commit();
    bulk_wait0();
}

// ---------------------------------------------------------------------------- pass 2: TMA ring -> shared-memory table -> dense output
struct GbDenseDev { uint64_t* keys; uint32_t* first; uint32_t* len; uint64_t* words; int64_t Gb; unsigned long long* cursor; };

constexpr int GBR_NST = 2;      // ring stages of plain records
// the ring keeps the bytes of GBR_NST stages of plain ROWW-word records (the plan's table size S depends on them); packed
// records fill that room with more stages (3 of 2 words where 2 of 3 were)
template <int ROWW, bool PACK> constexpr int gbr_nst() { return GBR_NST * ROWW / gbr_rw<ROWW, PACK>(); }
template <int ROWW, bool PACK>
__global__ void __launch_bounds__(1024) k_gbr_agg(const __grid_constant__ GbLayout L, const __grid_constant__ GbBatch Bt, const __grid_constant__ GbRadixDev R, const __grid_constant__ GbDenseDev D, unsigned S) {
    constexpr int NST = gbr_nst<ROWW, PACK>(), CR = GBR_NCT, NC = ROWW - 1, RW = gbr_rw<ROWW, PACK>();      // one record per consumer thread and stage
    extern __shared__ __align__(128) uint64_t gbr_smem2[];
    uint64_t* ring = gbr_smem2;                                       // NST x CR records
    uint64_t* tkey = ring + (size_t)GBR_NST * CR * ROWW;              // S keys
    uint64_t* tacc = tkey + S;                                        // n_words planes of S
    unsigned* tlen = reinterpret_cast<unsigned*>(tacc + (size_t)L.n_words * S);
    __shared__ uint64_t full[NST], empty[NST];
    __shared__ unsigned s_used, s_base;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, B = 1 << R.logB;
    if (*R.status & (GBR_ST_STREAM | GBR_ST_UNFIT)) return;      // pass 1 failed (every warp, the producer's included): the batch is redone
    if (tid == 0) { for (int s = 0; s < NST; s++) { mbar_init(&full[s], 1); mbar_init(&empty[s], GBR_NCW); } mbar_fence_init(); }
    __syncthreads();
    if (warp == GBR_NCW) {                      // producer warp: keeps the ring full across bucket boundaries
        if (lane == 0) {
            unsigned q = 0;
            for (int p = blockIdx.x; p < B; p += gridDim.x) {
                const int64_t rows = (int64_t)R.cursor[p];
                const uint64_t* src = R.recs + R.off[p] * RW;
                const int nch = (int)((rows + CR - 1) / CR);
                for (int c = 0; c < nch; c++, q++) {
                    const int st = q % NST; const unsigned use = q / NST;
                    if (use > 0) while (!mbar_try_wait(&empty[st], (use - 1) & 1u)) {}
                    const int64_t crow = min((int64_t)CR, rows - (int64_t)c * CR);
                    const unsigned bytes = (unsigned)(((crow + 1) & ~(int64_t)1) * RW * 8);      // whole 16-byte units (the buffer is padded)
                    mbar_expect_tx(&full[st], bytes);
                    bulk_g2s(ring + (size_t)st * CR * RW, src + (size_t)c * CR * RW, bytes, &full[st]);
                }
            }
        }
        return;
    }
    const unsigned max_used = S - (S >> 2);
    unsigned q = 0;
    for (int p = blockIdx.x; p < B; p += gridDim.x) {
        for (unsigned i = tid; i < S; i += GBR_NCT) { tkey[i] = GB_EMPTY; tlen[i] = 0; for (int w = 0; w < L.n_words; w++) tacc[(size_t)w * S + i] = L.init[w]; }
        if (tid == 0) s_used = 0;
        named_bar_sync(1, GBR_NCT);
        const int64_t rows = (int64_t)R.cursor[p];
        const int nch = (int)((rows + CR - 1) / CR);
        for (int c = 0; c < nch; c++, q++) {
            const int st = q % NST; const unsigned par = (q / NST) & 1u;
            while (!mbar_try_wait(&full[st], par)) {}
            const uint64_t* buf = ring + (size_t)st * CR * RW;
            const int crow = (int)min((int64_t)CR, rows - (int64_t)c * CR);
            uint64_t rec[RW];
            rec[0] = PACK ? GBR_PK_PAD : GB_EMPTY;
            if (tid < crow) {
#pragma unroll
                for (int w = 0; w < RW; w++) rec[w] = buf[tid * RW + w];
            }
            // the release below lets the producer's next TMA write overwrite this stage.  The warp signals before it uses
            // the record, so nothing else waits for these loads: without the proxy fence, a copy issued on lane 0's arrival
            // could land before another lane's load had read the stage (that lane then aggregated a record of the
            // bucket's next chunk but one in place of its own)
            fence_async_smem();
            __syncwarp();
            if (lane == 0) mbar_arrive(&empty[st]);
            if (PACK ? (uint32_t)rec[0] == GBR_PK_PAD : rec[0] == GB_EMPTY) continue;      // pad record
            const uint64_t key = PACK ? R.pk_base + (uint32_t)rec[0] : rec[0];
            unsigned slot = __umulhi((unsigned)((table_hash(key) << R.logB) >> 32), S);
            bool found = false;
            for (unsigned probes = 0; probes < 128u; probes++) {
                const uint64_t cur = *reinterpret_cast<volatile uint64_t*>(tkey + slot);
                if (cur == key) { found = true; break; }
                if (cur == GB_EMPTY) {
                    if (*reinterpret_cast<volatile unsigned*>(&s_used) >= max_used) break;
                    const unsigned long long old = atomicCAS(reinterpret_cast<unsigned long long*>(tkey + slot), (unsigned long long)GB_EMPTY, (unsigned long long)key);
                    if (old == GB_EMPTY) { atomicAdd(&s_used, 1u); found = true; break; }
                    if (old == key) { found = true; break; }
                }
                if (++slot == S) slot = 0;
            }
            if (!found) { atomicOr(R.status, GBR_ST_TABLE); continue; }      // more groups in this bucket than its table holds: the caller falls back
            if (L.need_len) atomicAdd(tlen + slot, 1u);
#pragma unroll
            for (int cix = 0; cix < NC; cix++) {
                const int dt = Bt.cols[cix].dtype;
                const uint64_t raw = PACK && cix == 0 ? gbr_unpack_value(R, rec[0]) : rec[PACK ? cix : 1 + cix];
                for (int kk = L.col_kbegin[cix]; kk < L.col_kbegin[cix + 1]; kk++) gb_apply_smem<false>(L.wop[kk], tacc + (size_t)L.wslot[kk] * S + slot, dt, raw, true);
            }
        }
        named_bar_sync(1, GBR_NCT);
        if (tid == 0) s_base = (unsigned)atomicAdd(D.cursor, (unsigned long long)s_used);
        named_bar_sync(1, GBR_NCT);
        // the bucket's groups are final: compact them straight into the dense output (order inside a bucket = slot order)
        const unsigned long long base = s_base;
        for (unsigned i0 = 0; i0 < S; i0 += GBR_NCT) {
            const unsigned i = i0 + tid;
            const bool used = i < S && tkey[i] != GB_EMPTY;
            unsigned at = 0;
            if (used) at = atomicSub(&s_used, 1u) - 1u;
            if (used) {
                const unsigned long long pos = base + at;
                if ((int64_t)pos >= D.Gb) atomicOr(R.status, GBR_ST_TABLE);
                else {
                    D.keys[pos] = tkey[i]; D.len[pos] = tlen[i]; D.first[pos] = 0xFFFFFFFFu;
                    for (int w = 0; w < L.n_words; w++) D.words[(int64_t)w * D.Gb + pos] = tacc[(size_t)w * S + i];
                }
            }
        }
        named_bar_sync(1, GBR_NCT);
    }
}

// the GB_EMPTY-key group (if any row carried that key) joins the dense output
__global__ void k_gbr_append_special(const uint64_t* __restrict__ special, int n_words, GbDenseDev D, int* status) {
    if (threadIdx.x != 0 || blockIdx.x != 0 || special[0] == 0) return;
    const unsigned long long pos = atomicAdd(D.cursor, 1ull);
    if ((int64_t)pos >= D.Gb) { *status = 1; return; }
    D.keys[pos] = GB_EMPTY; D.len[pos] = (uint32_t)special[0]; D.first[pos] = 0xFFFFFFFFu;
    for (int w = 0; w < n_words; w++) D.words[(int64_t)w * D.Gb + pos] = special[1 + w];
}

// =============================================================================================
// Host side
// =============================================================================================
static size_t gbr_wc_smem(int B, int roww) { return (size_t)B * (GBR_WC_F * roww * 8 + 4); }
// k_gbr_scatter: the staged tile (+ one pad record per bucket for the runs), hist / start / gpos, the bucket of every slot (coalesced)
static size_t gbr_scatter_smem(int B, int roww, bool bulk) {
    const size_t tile = (size_t)GBR_THREADS * GBR_RPT;
    return (tile + (bulk ? B : 0)) * roww * 8 + (size_t)3 * B * 4 + (bulk ? 0 : tile * 2);
}
// write-combining scatter: grid = the CTAs that fit at once (persistent; k_gbr_offsets pads for each of them)
template <int ROWW, int KEY_ELEM, int KEY_CANON, bool PACK>
static int scatter_wc_grid(int B) {
    auto kfn = k_gbr_scatter_wc<ROWW, KEY_ELEM, KEY_CANON, PACK>;
    const size_t smem = gbr_wc_smem(B, gbr_rw<ROWW, PACK>());
    PLB_CUDA(cudaFuncSetAttribute(kfn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    int occ = 0;
    PLB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kfn, GBR_WC_THREADS, smem));
    return ctx().sm_count * std::max(occ, 1);
}
template <int ROWW, int KEY_ELEM, int KEY_CANON, bool PACK>
static void launch_scatter(const GbLayout& L, const GbBatch& Bt, const GbRadixDev& R, bool bulk) {
    const size_t smem = gbr_scatter_smem(1 << R.logB, gbr_rw<ROWW, PACK>(), bulk);
    auto kfn = bulk ? k_gbr_scatter<ROWW, KEY_ELEM, KEY_CANON, true, PACK> : k_gbr_scatter<ROWW, KEY_ELEM, KEY_CANON, false, PACK>;
    PLB_CUDA(cudaFuncSetAttribute(kfn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    int occ = 0;
    PLB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kfn, GBR_THREADS, smem));
    PLB_LAUNCH("k5r_scatter", kfn, ctx().sm_count * std::max(occ, 1), GBR_THREADS, smem, L, Bt, R);
}
template <int ROWW, bool PACK>
static void launch_agg(const GbLayout& L, const GbBatch& Bt, const GbRadixDev& R, const GbDenseDev& D, unsigned S) {
    auto kfn = k_gbr_agg<ROWW, PACK>;
    const size_t smem = (size_t)GBR_NST * GBR_NCT * ROWW * 8 + (size_t)S * (8 + 4 + 8 * L.n_words) + 16;      // ring + table
    PLB_CUDA(cudaFuncSetAttribute(kfn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    int occ = 0;
    PLB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kfn, 1024, smem));
    PLB_LAUNCH("k5r_aggregate", kfn, std::min(1 << R.logB, ctx().sm_count * std::max(occ, 1)), 1024, smem, L, Bt, R, D, S);
}

// Returns false when the plan does not apply (or gave up): nothing is left behind and the caller runs the L2 plan.
bool GroupByState::consume_radix(const DevCol& key, const std::vector<const DevCol*>& values, uint64_t planned_cap) {
    const int mode = knob_int("BL_K5_RADIX", 1);      // 0 never, 1 when the table would leave L2, 2 whenever eligible
    if (mode == 0 || L.need_first || key.validity != nullptr || hot.rows > 0 || key.len < (1 << 20)) return false;
    // records carry 4- or 8-byte values without validity, at most 4 value columns
    for (size_t i = 0; i < plans.size(); i++) {
        if (plans[i].kind == BL_AGG_LEN) continue;
        const DevCol* v = values[i];
        if (v == nullptr || v->len != key.len || v->dtype != plans[i].in_dtype || v->validity != nullptr) return false;
        if (dtype_size(v->dtype) != 4 && dtype_size(v->dtype) != 8) return false;
    }
    // packed records (GbRadixDev): the key in the sampled window (pack_key: integer keys only) and one value column that
    // fits 32 bits, by dtype (4-byte columns, preferred: no row can miss) or by its sampled range (pack_cols); bound as
    // column 0.  The plan below (buckets, table, store path, stream sizing) stays the one of the plain width.
    const void* pk_col = nullptr;
    if (pack_key && knob_int("BL_K5R_PACK", 1) != 0 && (key.dtype == BL_INT64 || key.dtype == BL_UINT64 || key.dtype == BL_INT32 || key.dtype == BL_UINT32))
        for (size_t i = 0; i < plans.size(); i++) {
            if (plans[i].kind == BL_AGG_LEN) continue;
            const void* v = values[i]->v();
            if (dtype_size(values[i]->dtype) == 4) { pk_col = v; break; }
            if (!pk_col && std::find(pack_cols.begin(), pack_cols.end(), v) != pack_cols.end()) pk_col = v;
        }
    GbBatch Bt; GbLayout Lb;
    if (!bind_columns(key, values, 0, 0, 4, Bt, Lb, pk_col)) return false;
    const int roww = 1 + Lb.n_cols;
    bool pack = pk_col != nullptr;
    const int64_t n = key.len;
    // shared-memory table per bucket: what is left of ~110 KB (2 CTAs / SM) after a
    // 2-stage ring; when even 8192 buckets of that size cannot take the estimated groups, one CTA / SM with a ~200 KB table
    const size_t entry = 8 + 4 + 8 * (size_t)L.n_words;
    const size_t ring2 = (size_t)GBR_NST * GBR_NCT * roww * 8;
    unsigned S = 0; int logB = 6;
    for (const size_t total_kb : {(size_t)110, (size_t)222}) {
        if (total_kb * 1024 < ring2 + 1024 + 512 * entry) continue;
        S = (unsigned)((total_kb * 1024 - ring2 - 1024) / entry) & ~31u;
        const double per_bucket = 0.55 * (double)S;                   // groups per bucket the table takes comfortably
        logB = 6;
        while (logB < GBR_MAX_LOGB && (double)est_groups / (double)(1 << logB) > per_bucket) logB++;
        if ((double)est_groups / (double)(1 << logB) <= 0.7 * (double)S) break;
        S = 0;
    }
    if (S == 0) return false;                                         // too many groups even for 8192 buckets of the large table
    if (mode == 1) {
        // the L2 plan fills a table of up to 2x its L2 budget in two slot-range passes at full speed (launch_batch: pass_bits);
        // beyond that it needs four passes or misses L2, and this plan wins.
        const double l2_budget = 0.55 * (double)ctx().l2_bytes;
        if ((double)planned_cap * L.stride * 8 <= 2.0 * l2_budget) return false;
    }
    const int B = 1 << logB;
    // store path of the scatter: TMA runs up to 512 buckets; past that write-combining buffers when a chunk buffer per
    // bucket fits one CTA's shared memory, else the tile is written with coalesced stores.  BL_K5R_STORE (1 coalesced,
    // 2 write-combining, 3 runs) picks a path instead wherever its shared memory fits.
    int smem_optin = 0;
    PLB_CUDA(cudaDeviceGetAttribute(&smem_optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, ctx().device));
    const bool wc_fits = gbr_wc_smem(B, roww) <= (size_t)smem_optin;
    const int store = knob_int("BL_K5R_STORE", 0);
    bool bulk = logB <= 9, wc = !bulk && wc_fits;
    if (store == 1 && gbr_scatter_smem(B, roww, false) <= (size_t)smem_optin) bulk = wc = false;
    else if (store == 2 && wc_fits) { bulk = false; wc = true; }
    else if (store == 3 && gbr_scatter_smem(B, roww, true) <= (size_t)smem_optin) { bulk = true; wc = false; }
    const int64_t ntiles = (n + GBR_THREADS * GBR_RPT - 1) / (GBR_THREADS * GBR_RPT);
    // f(KEY_ELEM, KEY_CANON, ROWW, PACK) of the scatter kernels for this batch (packed forms: integer keys, value columns)
    auto with_scatter_form = [&](bool pk, auto f) {
        with_key_form(key.dtype, [&](auto e, auto c) { constexpr bool int_key = decltype(c)::value == 0; with_at_least<1, 2, 3, 4, 5>(roww, [&](auto w) {
            if constexpr (int_key && decltype(w)::value >= 2) { if (pk) { f(e, c, w, std::true_type{}); return; } }
            f(e, c, w, std::false_type{});
        }); });
    };
    // the grid (and so the padding) of the plain form, whichever form runs
    int wc_grid = 0;
    if (wc) with_scatter_form(false, [&](auto e, auto c, auto w, auto) { wc_grid = scatter_wc_grid<decltype(w)::value, decltype(e)::value, decltype(c)::value, false>(B); });
    // worst-case padding of a bucket stream (gbr_stream_records): one record per tile for the runs, F - 1 per CTA for the
    // write-combining buffers, none for the coalesced store
    const unsigned long long pad_units = wc ? (unsigned long long)wc_grid : (unsigned long long)ntiles;
    const unsigned pad_each = wc ? GBR_WC_F - 1 : bulk ? 1u : 0u, align = wc ? GBR_WC_F : 2u;
    // Bucket streams.  Sample sizing: every bucket gets room for n / B + 5 sqrt(F2 / B) rows (+ padding), F2 = est_f2 (the
    // sum over groups of their rows squared).  A group lands in bucket b with probability 1 / B, so the rows of b have mean
    // n / B and variance ~F2 / B; at z = 5 one bucket overflows with probability ~3e-7, one of 1024 with ~3e-4, and an
    // overflow costs one redone batch.  Taken when the margin is at most half the mean (streams <= 1.5 n records + padding).
    // Otherwise, and when nothing was sampled, exact sizing up front: k_gbr_hist counts every bucket's rows, one more read
    // of the keys.  C2 (1e8 rows, 1e6 uniform keys: F2 ~1.01e10, 1024 buckets): 97,656 + 15,700 rows per bucket.
    const double mean = (double)n / B, margin = 5.0 * std::sqrt(est_f2 / B);
    unsigned long long bucket_rows = est_f2 > 0 && margin <= 0.5 * mean ? (unsigned long long)std::ceil(mean + margin) : 0;      // 0: exact sizing
    const int64_t exact_rows = n + std::min<int64_t>(n, (int64_t)B * (int64_t)pad_units) * pad_each + (int64_t)align * B + 16;
    int64_t rec_rows = bucket_rows ? (int64_t)B * (int64_t)gbr_stream_records(bucket_rows, pad_units, pad_each, align) + 16 : exact_rows;
    DevPtr recs, ctl;
    try {
        recs = dev_alloc((size_t)rec_rows * roww * 8);
        ctl = dev_alloc((size_t)B * 4 * 2 + (size_t)(B + 1) * 8 + (size_t)(1 + GB_MAX_WORDS) * 8 + 64);
    } catch (const Error&) { cudaGetLastError(); return false; }       // not enough free HBM for the record streams
    GbRadixDev R; memset(&R, 0, sizeof R);
    R.recs = as<uint64_t>(recs); R.logB = logB; R.roww = roww; R.status = as<int>(status);
    R.pk_base = pack_base; R.pk_sext = Bt.cols[0].dtype == BL_INT64;
    char* cp = reinterpret_cast<char*>(ctl->p);
    R.off = reinterpret_cast<unsigned long long*>(cp); cp += (size_t)(B + 1) * 8;
    R.special = reinterpret_cast<uint64_t*>(cp); cp += (size_t)(1 + GB_MAX_WORDS) * 8;
    R.counts = reinterpret_cast<unsigned*>(cp); cp += (size_t)B * 4;
    R.cursor = reinterpret_cast<unsigned*>(cp);
    // dense output, sized by a generous bound on the group count (overflow -> status -> fall back)
    const int64_t Gb = std::max<int64_t>(1024, std::min<int64_t>(n + 1, 3 * est_groups + (1 << 16)));
    dense.keys = dev_alloc((size_t)Gb * 8); dense.first = dev_alloc((size_t)Gb * 4); dense.len = dev_alloc((size_t)Gb * 4);
    dense.words = dev_alloc((size_t)Gb * 8 * std::max(L.n_words, 1)); dense.ctl = dev_alloc(16); dense.Gb = Gb;
    GbDenseDev D{as<uint64_t>(dense.keys), as<uint32_t>(dense.first), as<uint32_t>(dense.len), as<uint64_t>(dense.words), Gb, as<unsigned long long>(dense.ctl)};
    for (;;) {
        const unsigned long long cap = bucket_rows ? gbr_stream_records(bucket_rows, pad_units, pad_each, align) : 0;      // records per bucket stream
        R.cap = cap ? (unsigned)cap : ~0u;
        if (!bucket_rows) {
            dev_memset(R.counts, 0, (size_t)B * 4);
            with_key_form(key.dtype, [&](auto e, auto c) {
                PLB_LAUNCH("k5r_histogram", (k_gbr_hist<decltype(e)::value, decltype(c)::value>), ctx().sm_count * 4, 512, (size_t)B * 4, key.v(), n, logB, R.counts);
            });
        }
        PLB_LAUNCH("k5r_setup", k_gbr_offsets, 1, 1024, 0, L, bucket_rows ? nullptr : R.counts, bucket_rows, B, pad_units, pad_each, align,
                   const_cast<unsigned long long*>(R.off), R.cursor, R.special, R.status);
        with_scatter_form(pack, [&](auto e, auto c, auto w, auto pk) {
            constexpr int E = decltype(e)::value, C = decltype(c)::value, ROWW = decltype(w)::value;
            constexpr bool P = decltype(pk)::value;
            if (wc) {
                if (P) (void)scatter_wc_grid<ROWW, E, C, P>(B);      // sets the packed form's shared-memory limit
                PLB_LAUNCH("k5r_scatter", (k_gbr_scatter_wc<ROWW, E, C, P>), wc_grid, GBR_WC_THREADS, gbr_wc_smem(B, gbr_rw<ROWW, P>()), Lb, Bt, R);
            }
            else launch_scatter<ROWW, E, C, P>(Lb, Bt, R, bulk);
        });
        dev_memset(dense.ctl->p, 0, 8); dev_memset(static_cast<char*>(dense.ctl->p) + 8, 0xFF, 8);      // {0, -1}
        with_at_least<1, 2, 3, 4, 5>(roww, [&](auto w) { with_bool(pack, [&](auto pk) {
            constexpr int ROWW = decltype(w)::value;
            if constexpr (ROWW >= 2 || !decltype(pk)::value) launch_agg<ROWW, decltype(pk)::value>(Lb, Bt, R, D, S);
        }); });
        PLB_LAUNCH("k5r_special", k_gbr_append_special, 1, 32, 0, R.special, L.n_words, D, as<int>(status));
        const int st = read_scalar(as<int>(status));      // also orders the recs lifetime
        if (getenv("BL_K5_DEBUG"))
            fprintf(stderr, "[k5r] rows=%lld est_groups=%lld buckets=%d slots=%u bulk=%d store=%s sizing=%s cap=%llu packed=%d status=%d\n", (long long)n, (long long)est_groups, B, S,
                    (int)bulk, bulk ? "runs" : wc ? "wc" : "coalesced", bucket_rows ? "sample" : "exact", cap, (int)pack, st);
        // pass 1 failed: once more with plain records (a row outside the packed form) and / or exact sizing (a bucket
        // outgrew its sampled stream), both in the same redo
        const bool unfit = st & GBR_ST_UNFIT, overflow = st & GBR_ST_STREAM;
        if ((unfit || overflow) && (!unfit || pack) && (!overflow || bucket_rows)) {
            if (unfit) pack = false;
            if (!overflow) continue;
            bucket_rows = 0;
            if (exact_rows > rec_rows) {
                recs.reset();
                try { recs = dev_alloc((size_t)exact_rows * roww * 8); } catch (const Error&) { cudaGetLastError(); dense = GbDense{}; dev_memset(status->p, 0, 4); return false; }
                R.recs = as<uint64_t>(recs); rec_rows = exact_rows;
            }
            continue;
        }
        if (st != 0) { dense = GbDense{}; dev_memset(status->p, 0, 4); return false; }
        dense.ready = true;
        rows_seen = n;
        return true;
    }
}

}  // namespace plb
