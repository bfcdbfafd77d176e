// groupby.cu — K5: fused hash group_by build + per-group aggregation, and K6 for partial
// aggregates (hash-partitioned export / merge for the multi-GPU plan).
//
// Reference path being replaced (paths relative to /root/reference/crates):
//   group_by_threaded_slice / finish_group_order   polars-core/src/frame/group_by/hashing.rs:26-167
//   key representation, null group                 polars-core/src/frame/group_by/into_groups.rs:25-58,142-191
//   agg_sum / agg_mean / agg_min / agg_max         polars-core/src/frame/group_by/aggregations/mod.rs:486-1018,1227-1296
//   take_agg null handling                         polars-arrow/src/legacy/kernels/take_agg/mod.rs:16-84
//   count / len                                    aggregations/dispatch.rs:25-55, position.rs:555-569
// The reference first materialises per-group row-index lists (GroupsIdx) and then gather-reduces
// every aggregate per group.  Here the index lists are never built: one pass over the rows
// finds/claims the key's entry in an open-addressing table in HBM (L2-resident for <= ~2M groups)
// and applies the row to the entry's accumulators with native 64-bit L2 atomics (RED.ADD.64,
// RED.ADD.F64, RED.MIN/MAX.S64/U64).  All of these are order-independent except the f64 sum
// (tolerance 1e-6 relative; the reference itself differs between its engines there).
//
// Entry layout (AoS, `stride` 64-bit words, 32-byte multiples so one entry = whole sectors):
//   word0 key bits (GB_EMPTY = free) | word1 lo32 = len, hi32 = first row idx | words 2.. accumulators
// Slots [0, cap) are hashed; slot cap = the null-key group, slot cap+1 = the group whose key bits
// equal GB_EMPTY (their word0 is only a "used" marker).
//
// Algorithmic bytes (SURVEY.md §8(d)): 8*(1 + value columns) per row in, G*(8 + 8*n_aggs) out.
// Roofline: HBM for the scan; the binding unit in practice is L2 atomic throughput
// (1 key load + 1 RED per accumulator per row).
#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstdlib>

#include "common.cuh"
#include "dev_utils.cuh"
#include "groupby.h"
#include "groupby_dev.cuh"

namespace plb {

// ---------------------------------------------------------------------------- device pieces
// ---- L2 cache-policy hints (sm_80+ createpolicy): the hash table is the only data with reuse, the
//      scanned columns are read once.  hint != 0: table loads / CAS / REDs carry an evict_last policy.
__device__ __forceinline__ uint64_t make_policy_evict_last() {
    uint64_t p; asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(p)); return p;
}
// Key-plane loads.  hint bit 1: L1-cached (ld.ca) — safe because a key word only ever changes EMPTY -> key: a
// stale EMPTY from L1 is caught by the CAS that follows (it returns the real key), a non-EMPTY value is final.
// The second linear probe usually falls into the sector the first one fetched (4 keys per sector).
__device__ __forceinline__ uint64_t tbl_load(const uint64_t* p, uint64_t pol, int hint) {
    uint64_t v;
    if (hint & 2) asm volatile("ld.global.ca.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    else if (hint & 1) asm volatile("ld.global.cg.L2::cache_hint.u64 %0, [%1], %2;" : "=l"(v) : "l"(p), "l"(pol));
    else v = __ldcg(reinterpret_cast<const unsigned long long*>(p));
    return v;
}
__device__ __forceinline__ void red_add_u64(uint64_t* p, uint64_t v, uint64_t pol, bool hint) {
    if (hint) asm volatile("red.global.add.L2::cache_hint.u64 [%0], %1, %2;" :: "l"(p), "l"(v), "l"(pol) : "memory");
    else atomicAdd(reinterpret_cast<unsigned long long*>(p), (unsigned long long)v);
}
__device__ __forceinline__ void red_add_f64(uint64_t* p, double v, uint64_t pol, bool hint) {
    if (hint) asm volatile("red.global.add.L2::cache_hint.f64 [%0], %1, %2;" :: "l"(p), "d"(v), "l"(pol) : "memory");
    else atomicAdd(reinterpret_cast<double*>(p), v);
}
__device__ __forceinline__ void red_add_u32(uint32_t* p, uint32_t v, uint64_t pol, bool hint) {
    if (hint) asm volatile("red.global.add.L2::cache_hint.u32 [%0], %1, %2;" :: "l"(p), "r"(v), "l"(pol) : "memory");
    else atomicAdd(p, v);
}

// claim / find the entry of `key`, continuing from slot `slot` whose key word `k` has already been
// loaded (the first probes of all rows of an iteration are issued together).
// nullptr => probe limit hit (table too small): status set.
__device__ __forceinline__ uint64_t* gb_resolve(const GbTableDev& T, uint64_t key, uint64_t slot, uint64_t k, uint64_t pol, int hint) {
    const uint64_t mask = T.cap - 1;
    for (int probes = 0; probes < GB_MAX_PROBE; ++probes) {
        uint64_t* e = T.entries + slot * T.es;
        if (k == key) return e;
        if (k == GB_EMPTY) {
            unsigned long long old = atomicCAS(reinterpret_cast<unsigned long long*>(e), (unsigned long long)GB_EMPTY, (unsigned long long)key);
            if (old == GB_EMPTY || old == key) return e;
        }
        slot = (slot + 1) & mask;
        k = tbl_load(T.entries + slot * T.es, pol, hint);
    }
    *T.status = 1;
    return nullptr;
}
__device__ __forceinline__ uint64_t* gb_find_or_insert(const GbTableDev& T, uint64_t key) {
    const uint64_t slot = table_hash(key) >> T.shift;
    return gb_resolve(T, key, slot, __ldcg(reinterpret_cast<const unsigned long long*>(T.entries + slot * T.es)), 0, 0);
}
__device__ __forceinline__ uint64_t* gb_special(const GbTableDev& T, int which) {
    uint64_t* e = T.entries + (T.cap + which) * T.es;
    if (__ldcg(reinterpret_cast<const unsigned long long*>(e)) == GB_EMPTY)
        atomicCAS(reinterpret_cast<unsigned long long*>(e), (unsigned long long)GB_EMPTY, (unsigned long long)which);
    return e;
}

// address of word w of the entry whose key word is at `e` (the layouts are described at GbTableDev)
__device__ __forceinline__ uint64_t* gb_wp(const GbTableDev& T, uint64_t* e, int w) {
    return e + gb_woff(T.pw ? (int64_t)(e - T.entries) : 0, w, T.ws, T.pw);
}
// ---- bulk reduce (TMA): one cp.reduce.async.bulk adds the 16-byte shared-memory cell {1, v} to the table cell {len | first, sum}.
//      Key load + this + 1 RED.F64 replaces key load + 3 REDs per row: the L2 / LSU RED rate is the ceiling of the table
//      update and the TMA unit is a second, otherwise idle, path into the same L2 atomic units (sm_90 and later).  SASS: UBLKRED.G.S.ADD.U64 (uniform datapath: ptxas serialises the lanes).
__device__ __forceinline__ void bulk_add_u64x2(uint64_t* dst, const uint64_t* src_smem, uint64_t pol, bool hint) {
    const uint32_t sa = (uint32_t)__cvta_generic_to_shared(src_smem);
    if (hint) asm volatile("cp.reduce.async.bulk.global.shared::cta.bulk_group.L2::cache_hint.add.u64 [%0], [%1], 16, %2;" :: "l"(dst), "r"(sa), "l"(pol) : "memory");
    else asm volatile("cp.reduce.async.bulk.global.shared::cta.bulk_group.add.u64 [%0], [%1], 16;" :: "l"(dst), "r"(sa) : "memory");
}

__device__ __forceinline__ void gb_apply(int op, uint64_t* addr, int dtype, uint64_t raw, bool valid, uint64_t pol = 0, bool hint = false) {
    switch (op) {
        case W_ADD_INT: { uint64_t v = raw_to_int(dtype, raw); if (valid && v) red_add_u64(addr, v, pol, hint); break; }
        case W_ADD_F64: { double f = raw_to_f64(dtype, raw); if (valid && f != 0.0) red_add_f64(addr, f, pol, hint); break; }
        case W_MIN_S64: if (valid) atomicMin(reinterpret_cast<long long*>(addr), (long long)raw_to_int(dtype, raw)); break;
        case W_MAX_S64: if (valid) atomicMax(reinterpret_cast<long long*>(addr), (long long)raw_to_int(dtype, raw)); break;
        case W_MIN_U64: if (valid) atomicMin(reinterpret_cast<unsigned long long*>(addr), (unsigned long long)raw); break;
        case W_MAX_U64: if (valid) atomicMax(reinterpret_cast<unsigned long long*>(addr), (unsigned long long)raw); break;
        case W_MIN_F64: { double f = raw_to_f64(dtype, raw); if (valid && f == f) atomicMin(reinterpret_cast<unsigned long long*>(addr), (unsigned long long)f64_to_ordered(f)); break; }
        case W_MAX_F64: { double f = raw_to_f64(dtype, raw); if (valid && f == f) atomicMax(reinterpret_cast<unsigned long long*>(addr), (unsigned long long)f64_to_ordered(f)); break; }
        default: if (!valid) atomicAdd(reinterpret_cast<unsigned long long*>(addr), 1ull); break;   // W_NULLCNT
    }
}

// ---------------------------------------------------------------------------- K5 main kernel
// Each thread owns PAIRS row pairs per iteration (pair p and p + k * grid stride: every load
// instruction is a fully coalesced 128-bit access): 128-bit loads of the key pair and of every
// value-column pair (64-bit loads for 4-byte types), then the first table probe of ALL its rows is
// issued before any of them is resolved (memory-level parallelism: the kernel is bound by L2
// latency, not by any throughput unit), then one RED per accumulator.
// BULK (pair layout only): len and the paired integer sum of a row travel as ONE 16-byte bulk reduce issued from a per-thread
// staging cell in shared memory (R x 256 cells); lanes >= T.bulk_lanes keep the plain REDs (knob: balance of the two paths).
template <int KEY_ELEM, int KEY_CANON, bool KEY_NULLS, int MAXC, int PAIRS, bool BULK>
__global__ void __launch_bounds__(256) k_gb_consume(const __grid_constant__ GbLayout L, const __grid_constant__ GbTableDev T, const __grid_constant__ GbBatch B) {
    constexpr int R = 2 * PAIRS;
    extern __shared__ __align__(16) uint64_t gb_stage[];
    const bool bulk_lane = BULK && (int)(threadIdx.x & 31) < T.bulk_lanes;
    const int64_t npairs = B.n >> 1;
    const int64_t gstride = (int64_t)gridDim.x * blockDim.x;
    const int khint = T.hint;                 // key-load flavour (bit 0: evict_last policy, bit 1: L1-cached)
    const bool hint = (T.hint & 1) != 0;      // evict_last policy on the REDs
    const uint64_t pol = hint ? make_policy_evict_last() : 0;
    int iter = 0;
    for (int64_t p0 = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; p0 < npairs; p0 += gstride * PAIRS) {
        if (((iter++) & 15) == 0 && *reinterpret_cast<volatile int*>(T.status)) break;
        uint64_t kraw[R];
        uint64_t raw[MAXC][R];
#pragma unroll
        for (int u = 0; u < PAIRS; u++) {
            const int64_t p = p0 + u * gstride;
            if (p < npairs) {
                if (KEY_ELEM == 8) { ulonglong2 t = ld_stream_u64x2(reinterpret_cast<const uint64_t*>(B.keys) + 2 * p); kraw[2 * u] = t.x; kraw[2 * u + 1] = t.y; }
                else { uint2 t = ld_stream_u32x2(reinterpret_cast<const uint32_t*>(B.keys) + 2 * p); kraw[2 * u] = t.x; kraw[2 * u + 1] = t.y; }
#pragma unroll
                for (int c = 0; c < MAXC; c++) {
                    if (c < L.n_cols) {
                        if (B.cols[c].elem == 8) { ulonglong2 t = ld_stream_u64x2(reinterpret_cast<const uint64_t*>(B.cols[c].values) + 2 * p); raw[c][2 * u] = t.x; raw[c][2 * u + 1] = t.y; }
                        else { uint2 t = ld_stream_u32x2(reinterpret_cast<const uint32_t*>(B.cols[c].values) + 2 * p); raw[c][2 * u] = t.x; raw[c][2 * u + 1] = t.y; }
                    }
                }
            }
        }
        // first probe of every row
        uint64_t key[R], slot[R], k0[R];
        int kind[R];   // 0 regular, 1 null-key group, 2 GB_EMPTY-key group, -1 no row
#pragma unroll
        for (int r = 0; r < R; r++) {
            const int64_t p = p0 + (r >> 1) * gstride;
            kind[r] = -1; key[r] = 0; slot[r] = 0; k0[r] = 0;
            if (p < npairs) {
                const int64_t row = 2 * p + (r & 1);
                bool kvalid = true;
                if (KEY_NULLS) kvalid = bit_get(B.key_validity, row);
                key[r] = canon_key<KEY_CANON>(kraw[r]);
                kind[r] = !kvalid ? 1 : (key[r] == GB_EMPTY ? 2 : 0);
                const uint64_t hsh = table_hash(key[r]);
                // multi-pass mode (tables larger than L2): this launch only owns the slot sub-range `pass_id`
                if (T.pass_bits && (kind[r] == 0 ? (int)(hsh >> (64 - T.pass_bits)) != T.pass_id : T.pass_id != 0)) kind[r] = -1;
                if (kind[r] == 0) { slot[r] = hsh >> T.shift; k0[r] = tbl_load(T.entries + slot[r] * T.es, pol, khint); }
            }
        }
        uint64_t* ent[R];
#pragma unroll
        for (int r = 0; r < R; r++) ent[r] = kind[r] < 0 ? nullptr : (kind[r] == 0 ? gb_resolve(T, key[r], slot[r], k0[r], pol, khint) : gb_special(T, kind[r] - 1));
        if (BULK) {
            // Bulk reduces FIRST: the proxy fence below is a MEMBAR.ALL.CTA + FENCE.VIEW.ASYNC in SASS and would wait for every RED this
            // thread has in flight (with the REDs ahead of it the bulk kernel was slower than the plain 3-RED kernel).
            // The staging cells are reused every iteration: the previous iteration's bulk reduces must have read them.
            asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
            if (bulk_lane) {
#pragma unroll
                for (int r = 0; r < R; r++) {
                    if (ent[r] == nullptr) continue;
                    const int64_t row = 2 * (p0 + (r >> 1) * gstride) + (r & 1);
                    // the paired sum's column is bound to column 0 of the batch (launch_batch): a runtime column index here made
                    // ptxas spill raw[][] to local memory (STL.128 per row: 1.6 GB of local stores, 1.1 GB of DRAM writes in ncu)
                    const uint64_t pv = (B.cols[0].validity == nullptr || bit_get(B.cols[0].validity, row)) ? raw_to_int(B.cols[0].dtype, raw[0][r]) : 0ull;
                    uint64_t* cell = gb_stage + 2 * (r * 256 + (int)threadIdx.x);
                    asm volatile("st.shared.v2.u64 [%0], {%1, %2};" :: "r"((uint32_t)__cvta_generic_to_shared(cell)), "l"((uint64_t)(L.need_len ? 1 : 0)), "l"(pv) : "memory");
                }
                asm volatile("fence.proxy.async.shared::cta;" ::: "memory");     // generic-proxy stores above -> visible to the TMA unit
#pragma unroll
                for (int r = 0; r < R; r++) if (ent[r]) bulk_add_u64x2(gb_wp(T, ent[r], 1), gb_stage + 2 * (r * 256 + (int)threadIdx.x), pol, hint);
                asm volatile("cp.async.bulk.commit_group;" ::: "memory");
            }
        }
#pragma unroll
        for (int r = 0; r < R; r++) {
            uint64_t* e = ent[r];
            if (e == nullptr) continue;
            const int64_t row = 2 * (p0 + (r >> 1) * gstride) + (r & 1);
            uint64_t* const w1 = gb_wp(T, e, 1);
            if (L.need_len && !bulk_lane) red_add_u32(reinterpret_cast<uint32_t*>(w1), 1u, pol, hint);
            if (L.need_first) atomicMin(reinterpret_cast<unsigned*>(w1) + 1, B.row_base + (uint32_t)row);
#pragma unroll
            for (int c = 0; c < MAXC; c++) {
                if (c < L.n_cols) {
                    const bool valid = B.cols[c].validity == nullptr || bit_get(B.cols[c].validity, row);
                    const int dt = B.cols[c].dtype;
                    for (int k = L.col_kbegin[c]; k < L.col_kbegin[c + 1]; k++) {
                        if (bulk_lane && k == L.pair_k) continue;      // already on its way as half of the bulk reduce
                        gb_apply(L.wop[k], gb_wp(T, e, 2 + L.wslot[k]), dt, raw[c][r], valid, pol, hint);
                    }
                }
            }
        }
    }
    // all bulk reduces of this thread have been performed (not just read) before the CTA may retire
    if (BULK) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
    // odd tail row
    if ((B.n & 1) && blockIdx.x == 0 && threadIdx.x == 0) {
        const int64_t row = B.n - 1;
        bool kvalid = B.key_validity == nullptr || bit_get(B.key_validity, row);
        uint64_t key = load_key_rt(B.keys, B.key_dtype, row);
        const bool regular = kvalid && key != GB_EMPTY;
        const bool mine = !T.pass_bits || (regular ? (int)(table_hash(key) >> (64 - T.pass_bits)) == T.pass_id : T.pass_id == 0);
        uint64_t* e = !mine ? nullptr : (!kvalid ? gb_special(T, 0) : (key == GB_EMPTY ? gb_special(T, 1) : gb_find_or_insert(T, key)));
        if (e) {
            if (L.need_len) atomicAdd(reinterpret_cast<unsigned*>(gb_wp(T, e, 1)), 1u);
            if (L.need_first) atomicMin(reinterpret_cast<unsigned*>(gb_wp(T, e, 1)) + 1, B.row_base + (uint32_t)row);
            for (int c = 0; c < L.n_cols; c++) {
                const bool valid = B.cols[c].validity == nullptr || bit_get(B.cols[c].validity, row);
                uint64_t raw = B.cols[c].elem == 8 ? reinterpret_cast<const uint64_t*>(B.cols[c].values)[row] : (uint64_t)reinterpret_cast<const uint32_t*>(B.cols[c].values)[row];
                for (int k = L.col_kbegin[c]; k < L.col_kbegin[c + 1]; k++) gb_apply(L.wop[k], gb_wp(T, e, 2 + L.wslot[k]), B.cols[c].dtype, raw, valid);
            }
        }
    }
}

// ---------------------------------------------------------------------------- K5, lean bulk-reduce kernel
// The general k_gb_consume<BULK> executes ~570 warp instructions per row pair (dtype / validity / layout dispatch + two 32-lane
// UBLKRED issue loops) and is issue-bound (ncu: 65 % issue slots busy, L2 at 54 %).  This kernel is the same algorithm for the
// common analytic shape — 8-byte integer key without nulls, every value column 8 bytes wide without a validity bitmap, at most
// two accumulators per column, single pass, pair layout — with everything that is uniform per launch hoisted out of the row
// loop.  Column 0 carries the paired integer sum (launch_batch binds it there).
// NULLS: the key and / or value columns may carry validity bitmaps (null keys -> the null group's slot, null values -> 0 for the
// paired sum, skipped by the REDs, counted by W_NULLCNT words).
template <int NC, bool NULLS>
__global__ void __launch_bounds__(256) k_gb_consume_lean(const __grid_constant__ GbLayout L, const __grid_constant__ GbTableDev T, const __grid_constant__ GbBatch B) {
    extern __shared__ __align__(16) uint64_t gb_stage[];
    const int64_t npairs = B.n >> 1;
    const int64_t gstride = (int64_t)gridDim.x * blockDim.x;
    uint64_t* const cells = T.entries + T.ws;              // {len | first, paired sum} per slot
    int op[NC][2]; uint64_t* plane[NC][2]; int dt[NC];
#pragma unroll
    for (int c = 0; c < NC; c++) {
        dt[c] = B.cols[c].dtype;
#pragma unroll
        for (int j = 0; j < 2; j++) {
            const int k = L.col_kbegin[c] + j;
            const bool on = k < L.col_kbegin[c + 1] && k != L.pair_k;
            op[c][j] = on ? L.wop[k] : -1;
            plane[c][j] = on ? T.entries + gb_woff(0, 2 + L.wslot[k], T.ws, T.pw) : nullptr;
        }
    }
    uint64_t* const cell0 = gb_stage + 2 * (int)threadIdx.x, * const cell1 = cell0 + 512;
    int iter = 0;
    for (int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; p < npairs; p += gstride) {
        if (((iter++) & 15) == 0 && *reinterpret_cast<volatile int*>(T.status)) break;
        const ulonglong2 k2 = ld_stream_u64x2(reinterpret_cast<const uint64_t*>(B.keys) + 2 * p);
        ulonglong2 raw[NC];
#pragma unroll
        for (int c = 0; c < NC; c++) raw[c] = ld_stream_u64x2(reinterpret_cast<const uint64_t*>(B.cols[c].values) + 2 * p);
        // validity of the row pair (rows 2p, 2p+1 sit in one bitmap word): bit 0 / 1 of vbits[c]; key validity in kbits
        unsigned vbits[NC], kbits = 3u;
#pragma unroll
        for (int c = 0; c < NC; c++) vbits[c] = 3u;
        if (NULLS) {
            const int sh = (int)((2 * p) & 31);
            if (B.key_validity) kbits = (B.key_validity[(2 * p) >> 5] >> sh) & 3u;
#pragma unroll
            for (int c = 0; c < NC; c++) if (B.cols[c].validity) vbits[c] = (B.cols[c].validity[(2 * p) >> 5] >> sh) & 3u;
        }
        const uint64_t key0 = k2.x, key1 = k2.y;
        const uint64_t h0 = table_hash(key0), h1 = table_hash(key1);
        const uint64_t s0 = h0 >> T.shift, s1 = h1 >> T.shift;
        const bool reg0 = (kbits & 1u) && key0 != GB_EMPTY, reg1 = (kbits & 2u) && key1 != GB_EMPTY;
        // multi-pass mode (tables larger than L2): this launch only owns the slot sub-range `pass_id` (special groups: pass 0)
        bool mine0 = true, mine1 = true;
        if (T.pass_bits) {
            mine0 = reg0 ? (int)(h0 >> (64 - T.pass_bits)) == T.pass_id : T.pass_id == 0;
            mine1 = reg1 ? (int)(h1 >> (64 - T.pass_bits)) == T.pass_id : T.pass_id == 0;
        }
        const uint64_t q0 = (reg0 && mine0) ? __ldcg(reinterpret_cast<const unsigned long long*>(T.entries + s0)) : 0ull;
        const uint64_t q1 = (reg1 && mine1) ? __ldcg(reinterpret_cast<const unsigned long long*>(T.entries + s1)) : 0ull;
        uint64_t* const e0 = !mine0 ? nullptr : (!(kbits & 1u) ? gb_special(T, 0) : (key0 == GB_EMPTY ? gb_special(T, 1) : gb_resolve(T, key0, s0, q0, 0, 0)));
        uint64_t* const e1 = !mine1 ? nullptr : (!(kbits & 2u) ? gb_special(T, 0) : (key1 == GB_EMPTY ? gb_special(T, 1) : gb_resolve(T, key1, s1, q1, 0, 0)));
        // bulk reduces first (see k_gb_consume); the staging cells of the previous iteration must have been read
        asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
        asm volatile("st.shared.v2.u64 [%0], {%1, %2};" :: "r"((uint32_t)__cvta_generic_to_shared(cell0)), "l"(1ull), "l"((vbits[0] & 1u) ? raw[0].x : 0ull) : "memory");
        asm volatile("st.shared.v2.u64 [%0], {%1, %2};" :: "r"((uint32_t)__cvta_generic_to_shared(cell1)), "l"(1ull), "l"((vbits[0] & 2u) ? raw[0].y : 0ull) : "memory");
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
        if (e0) bulk_add_u64x2(cells + 2 * (e0 - T.entries), cell0, 0, false);
        if (e1) bulk_add_u64x2(cells + 2 * (e1 - T.entries), cell1, 0, false);
        asm volatile("cp.async.bulk.commit_group;" ::: "memory");
#pragma unroll
        for (int c = 0; c < NC; c++) {
#pragma unroll
            for (int j = 0; j < 2; j++) {
                if (op[c][j] < 0) continue;
                if (e0) gb_apply(op[c][j], plane[c][j] + (e0 - T.entries), dt[c], raw[c].x, (vbits[c] & 1u) != 0);
                if (e1) gb_apply(op[c][j], plane[c][j] + (e1 - T.entries), dt[c], raw[c].y, (vbits[c] & 2u) != 0);
            }
        }
    }
    // odd tail row: plain atomics
    if ((B.n & 1) && blockIdx.x == 0 && threadIdx.x == 0) {
        const int64_t row = B.n - 1;
        const uint64_t key = reinterpret_cast<const uint64_t*>(B.keys)[row];
        const bool kvalid = B.key_validity == nullptr || bit_get(B.key_validity, row);
        const bool regular = kvalid && key != GB_EMPTY;
        const bool mine = !T.pass_bits || (regular ? (int)(table_hash(key) >> (64 - T.pass_bits)) == T.pass_id : T.pass_id == 0);
        uint64_t* e = !mine ? nullptr : (!kvalid ? gb_special(T, 0) : (key == GB_EMPTY ? gb_special(T, 1) : gb_find_or_insert(T, key)));
        if (e) {
            atomicAdd(reinterpret_cast<unsigned*>(gb_wp(T, e, 1)), 1u);
            for (int c = 0; c < L.n_cols; c++) {
                const uint64_t rv = reinterpret_cast<const uint64_t*>(B.cols[c].values)[row];
                const bool valid = B.cols[c].validity == nullptr || bit_get(B.cols[c].validity, row);
                for (int k = L.col_kbegin[c]; k < L.col_kbegin[c + 1]; k++) gb_apply(L.wop[k], gb_wp(T, e, 2 + L.wslot[k]), B.cols[c].dtype, rv, valid);
            }
        }
    }
    asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
}

__device__ __forceinline__ void gb_merge_row(const GbLayout& L, const GbTableDev& T, const uint64_t* src, int meta, int64_t sws = 1, int64_t sslot = 0, int spw = 0);

// ---------------------------------------------------------------------------- K5, heavy-hitter variant
// Skewed keys: all rows of a hot key hit ONE entry, and same-address L2 atomics retire serially
// (Zipf(1.1) keys cost k_gb_consume an order of magnitude more time than uniform keys).  Here the keys the sample flagged as heavy hitters (plus the null / GB_EMPTY key
// groups when those are frequent) never touch the global table row by row: a warp groups its lanes
// by hot key (__match_any_sync), reduces each group with shuffles and lets the group's first lane
// update a WARP-PRIVATE accumulator row in shared memory with plain loads/stores — no atomics at
// all.  The rows are merged into the global table once per warp at the end.  Cold keys take the
// same path as in k_gb_consume.
__device__ __forceinline__ uint64_t hot_contrib(int op, int dtype, uint64_t raw, bool valid) {
    switch (op) {
        case W_ADD_INT: return valid ? raw_to_int(dtype, raw) : 0ull;
        case W_ADD_F64: return valid ? (uint64_t)__double_as_longlong(raw_to_f64(dtype, raw)) : 0ull;
        case W_MIN_S64: case W_MAX_S64: return valid ? raw_to_int(dtype, raw) : word_identity(op);
        case W_MIN_U64: case W_MAX_U64: return valid ? raw : word_identity(op);
        case W_MIN_F64: case W_MAX_F64: { const double f = raw_to_f64(dtype, raw); return (valid && f == f) ? (uint64_t)f64_to_ordered(f) : word_identity(op); }
        default: return valid ? 0ull : 1ull;   // W_NULLCNT
    }
}
__device__ __forceinline__ uint64_t hot_combine(int op, uint64_t a, uint64_t b) {
    switch (op) {
        case W_ADD_F64: return (uint64_t)__double_as_longlong(__longlong_as_double((long long)a) + __longlong_as_double((long long)b));
        case W_MIN_S64: return (long long)a < (long long)b ? a : b;
        case W_MAX_S64: return (long long)a > (long long)b ? a : b;
        case W_MIN_U64: case W_MIN_F64: return a < b ? a : b;
        case W_MAX_U64: case W_MAX_F64: return a > b ? a : b;
        default: return a + b;                  // W_ADD_INT, W_NULLCNT
    }
}
// reduction over the lanes of `peers` (every lane of the group calls this with the same mask)
__device__ __forceinline__ uint64_t hot_group_reduce(int op, unsigned peers, uint64_t v) {
    unsigned m = peers;
    int src = __ffs(m) - 1;
    uint64_t acc = __shfl_sync(peers, (unsigned long long)v, src);
    for (m &= m - 1; m; m &= m - 1) {
        src = __ffs(m) - 1;
        acc = hot_combine(op, acc, __shfl_sync(peers, (unsigned long long)v, src));
    }
    return acc;
}

template <int KEY_ELEM, int KEY_CANON, bool KEY_NULLS, int MAXC>
__global__ void __launch_bounds__(256) k_gb_consume_hot(const __grid_constant__ GbLayout L, const __grid_constant__ GbTableDev T, const __grid_constant__ GbBatch B, const __grid_constant__ GbHotDev H) {
    // shared memory: [GB_HOT_SLOTS lookup keys][8 warps x H.rows x row_words accumulator rows][GB_HOT_SLOTS dense row indices]
    // accumulator row = [key, len | first << 32, words...]: the source-row format of gb_merge_row
    extern __shared__ uint64_t hot_smem[];
    const int row_words = 2 + L.n_words;
    uint64_t* const s_keys = hot_smem;
    uint64_t* const s_acc = hot_smem + GB_HOT_SLOTS;
    uint8_t* const s_idx = reinterpret_cast<uint8_t*>(s_acc + 8 * H.rows * row_words);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int i = threadIdx.x; i < GB_HOT_SLOTS; i += blockDim.x) { s_keys[i] = H.keys[i]; s_idx[i] = H.idx[i]; }
    for (int i = threadIdx.x; i < 8 * H.rows * row_words; i += blockDim.x) {
        const int w = i % row_words;
        s_acc[i] = w == 0 ? 0ull : (w == 1 ? GB_W1_INIT : L.init[w - 2]);
    }
    __syncthreads();
    uint64_t* const wacc = s_acc + warp * H.rows * row_words;
    const int64_t npairs = B.n >> 1;
    const int64_t gstride = (int64_t)gridDim.x * blockDim.x;
    const int khint = T.hint & 2;
    int iter = 0;
    // warp-uniform trip count: the hot path is warp-collective
    for (int64_t pb = (int64_t)blockIdx.x * blockDim.x + (threadIdx.x & ~31); pb < npairs; pb += gstride) {
        if (((iter++) & 15) == 0) {
            const int st = *reinterpret_cast<volatile int*>(T.status);
            if (__any_sync(0xffffffffu, st != 0)) break;
        }
        const int64_t p = pb + lane;
        const bool in = p < npairs;
        uint64_t kraw[2] = {0, 0};
        uint64_t raw[MAXC][2];
        if (in) {
            if (KEY_ELEM == 8) { ulonglong2 t = ld_stream_u64x2(reinterpret_cast<const uint64_t*>(B.keys) + 2 * p); kraw[0] = t.x; kraw[1] = t.y; }
            else { uint2 t = ld_stream_u32x2(reinterpret_cast<const uint32_t*>(B.keys) + 2 * p); kraw[0] = t.x; kraw[1] = t.y; }
#pragma unroll
            for (int c = 0; c < MAXC; c++) {
                if (c < L.n_cols) {
                    if (B.cols[c].elem == 8) { ulonglong2 t = ld_stream_u64x2(reinterpret_cast<const uint64_t*>(B.cols[c].values) + 2 * p); raw[c][0] = t.x; raw[c][1] = t.y; }
                    else { uint2 t = ld_stream_u32x2(reinterpret_cast<const uint32_t*>(B.cols[c].values) + 2 * p); raw[c][0] = t.x; raw[c][1] = t.y; }
                }
            }
        }
        uint64_t key[2], slot[2], k0[2];
        int kind[2], hidx[2];   // kind: 0 regular, 1 null-key group, 2 GB_EMPTY-key group, -1 no row;  hidx: accumulator row or -1 (cold)
#pragma unroll
        for (int r = 0; r < 2; r++) {
            kind[r] = -1; hidx[r] = -1; key[r] = 0; slot[r] = 0; k0[r] = 0;
            if (in) {
                const int64_t row = 2 * p + r;
                bool kvalid = true;
                if (KEY_NULLS) kvalid = bit_get(B.key_validity, row);
                key[r] = canon_key<KEY_CANON>(kraw[r]);
                kind[r] = !kvalid ? 1 : (key[r] == GB_EMPTY ? 2 : 0);
                const uint64_t hsh = table_hash(key[r]);
                if (T.pass_bits && (kind[r] == 0 ? (int)(hsh >> (64 - T.pass_bits)) != T.pass_id : T.pass_id != 0)) kind[r] = -1;
                if (kind[r] == 0) {
                    unsigned hs = (unsigned)(hsh >> (64 - GB_HOT_BITS));
                    for (;;) {
                        const uint64_t hk = s_keys[hs];
                        if (hk == key[r]) { hidx[r] = (int)s_idx[hs]; break; }
                        if (hk == GB_EMPTY) break;
                        hs = (hs + 1) & (GB_HOT_SLOTS - 1);
                    }
                    if (hidx[r] < 0) { slot[r] = hsh >> T.shift; k0[r] = tbl_load(T.entries + slot[r] * T.es, 0, khint); }
                } else if (kind[r] == 1) { if (H.null_hot) hidx[r] = H.n_hot; }
                else if (kind[r] == 2) { if (H.empty_hot) hidx[r] = H.n_hot + 1; }
            }
        }
        // hot rows: group lanes by accumulator row, reduce, first lane of the group updates the warp's row
#pragma unroll
        for (int r = 0; r < 2; r++) {
            if (__ballot_sync(0xffffffffu, hidx[r] >= 0) == 0) continue;      // warp-uniform
            const unsigned peers = __match_any_sync(0xffffffffu, hidx[r]);
            if (hidx[r] >= 0) {
                const bool lead = lane == __ffs(peers) - 1;
                uint64_t* const arow = wacc + hidx[r] * row_words;
                const int64_t row = 2 * p + r;
                if (lead) {
                    const uint64_t w1 = arow[1];
                    const uint32_t len = (uint32_t)w1 + (uint32_t)__popc(peers);
                    uint32_t first = (uint32_t)(w1 >> 32);
                    // lanes hold ascending rows: the group's first lane owns its smallest row
                    if (L.need_first) first = min(first, B.row_base + (uint32_t)row);
                    arow[0] = key[r];
                    arow[1] = ((uint64_t)first << 32) | len;
                }
#pragma unroll
                for (int c = 0; c < MAXC; c++) {
                    if (c < L.n_cols) {
                        const bool valid = B.cols[c].validity == nullptr || bit_get(B.cols[c].validity, row);
                        const int dt = B.cols[c].dtype;
                        for (int k = L.col_kbegin[c]; k < L.col_kbegin[c + 1]; k++) {
                            const int op = L.wop[k];
                            const uint64_t tot = hot_group_reduce(op, peers, hot_contrib(op, dt, raw[c][r], valid));
                            if (lead) { uint64_t* a = arow + 2 + L.wslot[k]; *a = hot_combine(op, *a, tot); }
                        }
                    }
                }
            }
            __syncwarp();
        }
        // cold rows: the global table, as in k_gb_consume
#pragma unroll
        for (int r = 0; r < 2; r++) {
            if (kind[r] < 0 || hidx[r] >= 0) continue;
            uint64_t* e = kind[r] == 0 ? gb_resolve(T, key[r], slot[r], k0[r], 0, khint) : gb_special(T, kind[r] - 1);
            if (e == nullptr) continue;
            const int64_t row = 2 * p + r;
            if (L.need_len) atomicAdd(reinterpret_cast<unsigned*>(gb_wp(T, e, 1)), 1u);
            if (L.need_first) atomicMin(reinterpret_cast<unsigned*>(gb_wp(T, e, 1)) + 1, B.row_base + (uint32_t)row);
#pragma unroll
            for (int c = 0; c < MAXC; c++) {
                if (c < L.n_cols) {
                    const bool valid = B.cols[c].validity == nullptr || bit_get(B.cols[c].validity, row);
                    const int dt = B.cols[c].dtype;
                    for (int k = L.col_kbegin[c]; k < L.col_kbegin[c + 1]; k++) gb_apply(L.wop[k], gb_wp(T, e, 2 + L.wslot[k]), dt, raw[c][r], valid);
                }
            }
        }
    }
    // odd tail row: straight to the global table
    if ((B.n & 1) && blockIdx.x == 0 && threadIdx.x == 0) {
        const int64_t row = B.n - 1;
        bool kvalid = B.key_validity == nullptr || bit_get(B.key_validity, row);
        uint64_t key = load_key_rt(B.keys, B.key_dtype, row);
        const bool regular = kvalid && key != GB_EMPTY;
        const bool mine = !T.pass_bits || (regular ? (int)(table_hash(key) >> (64 - T.pass_bits)) == T.pass_id : T.pass_id == 0);
        uint64_t* e = !mine ? nullptr : (!kvalid ? gb_special(T, 0) : (key == GB_EMPTY ? gb_special(T, 1) : gb_find_or_insert(T, key)));
        if (e) {
            if (L.need_len) atomicAdd(reinterpret_cast<unsigned*>(gb_wp(T, e, 1)), 1u);
            if (L.need_first) atomicMin(reinterpret_cast<unsigned*>(gb_wp(T, e, 1)) + 1, B.row_base + (uint32_t)row);
            for (int c = 0; c < L.n_cols; c++) {
                const bool valid = B.cols[c].validity == nullptr || bit_get(B.cols[c].validity, row);
                uint64_t raw = B.cols[c].elem == 8 ? reinterpret_cast<const uint64_t*>(B.cols[c].values)[row] : (uint64_t)reinterpret_cast<const uint32_t*>(B.cols[c].values)[row];
                for (int k = L.col_kbegin[c]; k < L.col_kbegin[c + 1]; k++) gb_apply(L.wop[k], gb_wp(T, e, 2 + L.wslot[k]), B.cols[c].dtype, raw, valid);
            }
        }
    }
    // merge the warp's accumulator rows into the global table (rows no lane touched keep len == 0)
    __syncwarp();
    for (int h = lane; h < H.rows; h += 32) {
        const uint64_t* arow = wacc + h * row_words;
        if ((uint32_t)arow[1] == 0) continue;
        gb_merge_row(L, T, arow, h == H.n_hot ? 1 : (h == H.n_hot + 1 ? 2 : 0));
    }
}

// word w of entry s lives at entries[s * es + w * ws]: AoS (es = stride, ws = 1) or word-major planes (es = 1, ws = n_entries)
__global__ void k_gb_init(uint64_t* entries, int64_t n_entries, int stride, int soa, int pw, const __grid_constant__ GbLayout L) {
    const int64_t total = n_entries * stride;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        int w = soa ? (int)(i / n_entries) : (int)(i % stride);
        if (pw) {   // pair layout: planes 1 and 2 hold the cells {word 1, word pw}; plane pw holds word 2
            if (w == 1 || w == 2) w = ((i - n_entries) & 1) ? pw : 1;
            else if (w == pw) w = 2;
        }
        uint64_t v = 0;
        if (w == 0) v = GB_EMPTY; else if (w == 1) v = GB_W1_INIT; else if (w - 2 < L.n_words) v = L.init[w - 2];
        entries[i] = v;
    }
}

// cardinality sample: insert m strided keys into a scratch key table with per-slot multiplicities.
// stats[0] = distinct keys, stats[3] = sampled rows whose successor row carries the same key
// (collision rate of neighbouring rows: skew / sortedness); stats[1], stats[2] are filled by
// k_gb_estimate_stats (keys seen exactly once / exactly twice in the sample).
constexpr int GB_CAND_MAX = 1024;
struct GbSampleStats { unsigned distinct, f1, f2, adjacent, nulls, empties, n_cand, pad; };
struct GbCandidate { uint64_t key; uint64_t mult; };
__global__ void k_gb_estimate(const void* keys, const uint32_t* key_validity, int key_dtype, int64_t n, int64_t m, uint64_t* scratch, unsigned* mult, uint64_t cap, int shift, GbSampleStats* stats) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < m; i += (int64_t)gridDim.x * blockDim.x) {
        int64_t row = (int64_t)(((unsigned __int128)i * (unsigned __int128)n) / (unsigned __int128)m);
        bool ins = false, adj = false, isnull = false, isempty = false;
        if (key_validity == nullptr || bit_get(key_validity, row)) {
            uint64_t key = load_key_rt(keys, key_dtype, row);
            adj = row + 1 < n && load_key_rt(keys, key_dtype, row + 1) == key && (key_validity == nullptr || bit_get(key_validity, row + 1));
            if (key != GB_EMPTY) {
                uint64_t slot = table_hash(key) >> shift;
                for (int pr = 0; pr < (int)cap; pr++) {
                    uint64_t k = __ldcg(reinterpret_cast<const unsigned long long*>(scratch + slot));
                    if (k == GB_EMPTY) {
                        unsigned long long old = atomicCAS(reinterpret_cast<unsigned long long*>(scratch + slot), (unsigned long long)GB_EMPTY, (unsigned long long)key);
                        if (old == GB_EMPTY) { ins = true; k = key; } else k = old;
                    }
                    if (k == key) { atomicAdd(mult + slot, 1u); break; }
                    slot = (slot + 1) & (cap - 1);
                }
            } else isempty = true;
        } else {
            isnull = true;
            adj = row + 1 < n && !bit_get(key_validity, row + 1);
        }
        unsigned act = __activemask();
        unsigned b = __ballot_sync(act, ins), a = __ballot_sync(act, adj), bn = __ballot_sync(act, isnull), be = __ballot_sync(act, isempty);
        if (lane_id() == (unsigned)(__ffs(act) - 1)) {
            if (b) atomicAdd(&stats->distinct, (unsigned)__popc(b));
            if (a) atomicAdd(&stats->adjacent, (unsigned)__popc(a));
            if (bn) atomicAdd(&stats->nulls, (unsigned)__popc(bn));
            if (be) atomicAdd(&stats->empties, (unsigned)__popc(be));
        }
    }
}
// f1 / f2 (keys sampled exactly once / twice) and the heavy-hitter candidates (multiplicity >= hot_thr)
__global__ void k_gb_estimate_stats(const uint64_t* scratch, const unsigned* mult, int64_t cap, unsigned hot_thr, GbSampleStats* stats, GbCandidate* cand) {
    unsigned f1 = 0, f2 = 0;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < cap; i += (int64_t)gridDim.x * blockDim.x) {
        const unsigned c = mult[i];
        f1 += c == 1; f2 += c == 2;
        if (c >= hot_thr) {
            const unsigned at = atomicAdd(&stats->n_cand, 1u);
            if (at < GB_CAND_MAX) { cand[at].key = scratch[i]; cand[at].mult = c; }
        }
    }
    f1 = __reduce_add_sync(0xffffffffu, f1); f2 = __reduce_add_sync(0xffffffffu, f2);
    if (lane_id() == 0) { if (f1) atomicAdd(&stats->f1, f1); if (f2) atomicAdd(&stats->f2, f2); }
}
__global__ void k_fill_u64(uint64_t* p, uint64_t v, int64_t n) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) p[i] = v;
}

// ---------------------------------------------------------------------------- merge (partials / rehash)
// rows: n_rows x row_words.  table_mode: rows are the slots of another table (stride = row_words,
// special slots at src_cap, src_cap+1); else exported partial rows whose last word is meta
// (0 normal, 1 null-key group, 2 GB_EMPTY-key group).
// (sslot, spw): the source is slot sslot of a table in the pair layout (rehash); spw == 0 for rows and word-major / AoS tables.
__device__ __forceinline__ void gb_merge_row(const GbLayout& L, const GbTableDev& T, const uint64_t* src, int meta, int64_t sws, int64_t sslot, int spw) {
    uint64_t* e = meta == 1 ? gb_special(T, 0) : (meta == 2 ? gb_special(T, 1) : gb_find_or_insert(T, src[0]));
    if (!e) return;
    const uint64_t lf = src[gb_woff(sslot, 1, sws, spw)];
    if ((uint32_t)lf) atomicAdd(reinterpret_cast<unsigned*>(gb_wp(T, e, 1)), (uint32_t)lf);
    if ((uint32_t)(lf >> 32) != 0xFFFFFFFFu) atomicMin(reinterpret_cast<unsigned*>(gb_wp(T, e, 1)) + 1, (uint32_t)(lf >> 32));
    for (int w = 0; w < L.n_words; w++) {
        const uint64_t v = src[gb_woff(sslot, 2 + w, sws, spw)];
        if (v == L.init[w]) continue;
        uint64_t* a = gb_wp(T, e, 2 + w);
        switch (L.slot_op[w]) {
            case W_ADD_F64: atomicAdd(reinterpret_cast<double*>(a), __longlong_as_double((long long)v)); break;
            case W_MIN_S64: atomicMin(reinterpret_cast<long long*>(a), (long long)v); break;
            case W_MAX_S64: atomicMax(reinterpret_cast<long long*>(a), (long long)v); break;
            case W_MIN_U64: case W_MIN_F64: atomicMin(reinterpret_cast<unsigned long long*>(a), (unsigned long long)v); break;
            case W_MAX_U64: case W_MAX_F64: atomicMax(reinterpret_cast<unsigned long long*>(a), (unsigned long long)v); break;
            default: atomicAdd(reinterpret_cast<unsigned long long*>(a), (unsigned long long)v); break;   // ADD_INT, NULLCNT
        }
    }
}
__global__ void __launch_bounds__(256) k_gb_merge(const __grid_constant__ GbLayout L, const __grid_constant__ GbTableDev T, const uint64_t* __restrict__ rows, int64_t n_rows, int64_t src_es, int64_t src_ws, int table_mode, int64_t src_cap, int src_pw) {
    for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < n_rows; r += (int64_t)gridDim.x * blockDim.x) {
        const uint64_t* src = rows + r * src_es;
        int meta;
        if (table_mode) { if (src[0] == GB_EMPTY) continue; meta = r == src_cap ? 1 : (r == src_cap + 1 ? 2 : 0); }
        else meta = (int)src[(L.n_words + 2) * src_ws];
        gb_merge_row(L, T, src, meta, src_ws, r, table_mode ? src_pw : 0);
    }
}

// ---------------------------------------------------------------------------- K5, low-cardinality variant
// When the sampled estimate says the groups fit a shared-memory table (<= a few thousand), every
// CTA aggregates into a PRIVATE open-addressing table in shared memory and merges it into the
// global table once at the end: an SM retires shared-memory atomics several times faster than the
// L2 atomic units do, so this path is bound by the HBM scan instead of the L2 atomic units.  Shared-memory accumulators: 32-bit native ATOMS; 64-bit integer adds as two
// 32-bit adds with carry (exact, order-free); f64 add and 64-bit min/max as CAS loops.
// Rows whose key cannot be placed (table 3/4 full) fall through to the global table, so the
// result is exact for any input; a wrong estimate only costs speed.
template <int KEY_ELEM, int KEY_CANON, bool KEY_NULLS, int MAXC, bool FAST>
__global__ void __launch_bounds__(512) k_gb_consume_smem(const __grid_constant__ GbLayout L, const __grid_constant__ GbTableDev T, const __grid_constant__ GbBatch B, int scap, int sshift, int copies) {
    // `copies` replicas of the table (tiny cardinalities): lane l works on replica l % copies, so the
    // lanes of a warp that hit the SAME group do not serialise on one shared-memory address.
    extern __shared__ uint64_t stab_all[];
    __shared__ int s_used_all[32];
    const int stride = L.stride;
    const int n_ent = scap + 2;
    const int tab_words = n_ent * stride + 2;          // +2 words: replicas start in different banks
    for (int i = threadIdx.x; i < copies * tab_words; i += blockDim.x) {
        const int j = i % tab_words;
        const int w = j % stride;
        stab_all[i] = j >= n_ent * stride ? 0ull : (w == 0 ? GB_EMPTY : (w == 1 ? GB_W1_INIT : (w - 2 < L.n_words ? L.init[w - 2] : 0ull)));
    }
    if (threadIdx.x < 32) s_used_all[threadIdx.x] = 0;
    __syncthreads();
    const int my_copy = (int)(lane_id() % (unsigned)copies);
    uint64_t* const stab = stab_all + (size_t)my_copy * tab_words;
    int& s_used = s_used_all[my_copy];
    const int max_used = scap - (scap >> 2);
    const int64_t npairs = B.n >> 1;
    const int64_t gstride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; p < npairs; p += gstride) {
        uint64_t kraw[2];
        if (KEY_ELEM == 8) { ulonglong2 t = ld_stream_u64x2(reinterpret_cast<const uint64_t*>(B.keys) + 2 * p); kraw[0] = t.x; kraw[1] = t.y; }
        else { uint2 t = ld_stream_u32x2(reinterpret_cast<const uint32_t*>(B.keys) + 2 * p); kraw[0] = t.x; kraw[1] = t.y; }
        uint64_t raw[MAXC][2];
#pragma unroll
        for (int c = 0; c < MAXC; c++) {
            if (c < L.n_cols) {
                if (FAST || B.cols[c].elem == 8) { ulonglong2 t = ld_stream_u64x2(reinterpret_cast<const uint64_t*>(B.cols[c].values) + 2 * p); raw[c][0] = t.x; raw[c][1] = t.y; }
                else { uint2 t = ld_stream_u32x2(reinterpret_cast<const uint32_t*>(B.cols[c].values) + 2 * p); raw[c][0] = t.x; raw[c][1] = t.y; }
            }
        }
#pragma unroll
        for (int j = 0; j < 2; j++) {
            const int64_t row = 2 * p + j;
            bool kvalid = true;
            if (KEY_NULLS) kvalid = bit_get(B.key_validity, row);
            const uint64_t key = canon_key<KEY_CANON>(kraw[j]);
            uint64_t* se = nullptr;     // entry in the CTA's shared table, or nullptr -> global path
            if (!kvalid || key == GB_EMPTY) {
                se = stab + (scap + (kvalid ? 1 : 0)) * stride;
                if (*reinterpret_cast<volatile uint64_t*>(se) == GB_EMPTY) atomicCAS(reinterpret_cast<unsigned long long*>(se), (unsigned long long)GB_EMPTY, kvalid ? 1ull : 0ull);
            } else {
                uint32_t slot = (uint32_t)(table_hash(key) >> sshift);
                for (int probes = 0; probes < 32; probes++) {
                    uint64_t* e = stab + slot * stride;
                    const uint64_t k = *reinterpret_cast<volatile uint64_t*>(e);
                    if (k == key) { se = e; break; }
                    if (k == GB_EMPTY) {
                        if (*reinterpret_cast<volatile int*>(&s_used) >= max_used) break;
                        const unsigned long long old = atomicCAS(reinterpret_cast<unsigned long long*>(e), (unsigned long long)GB_EMPTY, (unsigned long long)key);
                        if (old == GB_EMPTY) { atomicAdd(&s_used, 1); se = e; break; }
                        if (old == key) { se = e; break; }
                    }
                    slot = (slot + 1) & (uint32_t)(scap - 1);
                }
            }
            if (se != nullptr) {
                if (L.need_len) atomicAdd(reinterpret_cast<unsigned*>(se + 1), 1u);
                if (L.need_first) atomicMin(reinterpret_cast<unsigned*>(se + 1) + 1, B.row_base + (uint32_t)row);
#pragma unroll
                for (int c = 0; c < MAXC; c++) {
                    if (c < L.n_cols) {
                        const bool valid = FAST || B.cols[c].validity == nullptr || bit_get(B.cols[c].validity, row);
                        const int dt = B.cols[c].dtype;
                        for (int k = L.col_kbegin[c]; k < L.col_kbegin[c + 1]; k++) gb_apply_smem<FAST>(L.wop[k], se + 2 + L.wslot[k], dt, raw[c][j], valid);
                    }
                }
            } else {
                uint64_t* e = gb_find_or_insert(T, key);
                if (e != nullptr) {
                    if (L.need_len) atomicAdd(reinterpret_cast<unsigned*>(gb_wp(T, e, 1)), 1u);
                    if (L.need_first) atomicMin(reinterpret_cast<unsigned*>(gb_wp(T, e, 1)) + 1, B.row_base + (uint32_t)row);
#pragma unroll
                    for (int c = 0; c < MAXC; c++) {
                        if (c < L.n_cols) {
                            const bool valid = B.cols[c].validity == nullptr || bit_get(B.cols[c].validity, row);
                            const int dt = B.cols[c].dtype;
                            for (int k = L.col_kbegin[c]; k < L.col_kbegin[c + 1]; k++) gb_apply(L.wop[k], gb_wp(T, e, 2 + L.wslot[k]), dt, raw[c][j], valid);
                        }
                    }
                }
            }
        }
    }
    // odd tail row: straight to the global table
    if ((B.n & 1) && blockIdx.x == 0 && threadIdx.x == 0) {
        const int64_t row = B.n - 1;
        bool kvalid = B.key_validity == nullptr || bit_get(B.key_validity, row);
        uint64_t key = load_key_rt(B.keys, B.key_dtype, row);
        uint64_t* e = !kvalid ? gb_special(T, 0) : (key == GB_EMPTY ? gb_special(T, 1) : gb_find_or_insert(T, key));
        if (e) {
            if (L.need_len) atomicAdd(reinterpret_cast<unsigned*>(gb_wp(T, e, 1)), 1u);
            if (L.need_first) atomicMin(reinterpret_cast<unsigned*>(gb_wp(T, e, 1)) + 1, B.row_base + (uint32_t)row);
            for (int c = 0; c < L.n_cols; c++) {
                const bool valid = B.cols[c].validity == nullptr || bit_get(B.cols[c].validity, row);
                uint64_t raw = B.cols[c].elem == 8 ? reinterpret_cast<const uint64_t*>(B.cols[c].values)[row] : (uint64_t)reinterpret_cast<const uint32_t*>(B.cols[c].values)[row];
                for (int k = L.col_kbegin[c]; k < L.col_kbegin[c + 1]; k++) gb_apply(L.wop[k], gb_wp(T, e, 2 + L.wslot[k]), B.cols[c].dtype, raw, valid);
            }
        }
    }
    __syncthreads();
    // merge the CTA's partial aggregates into the global table
    for (int i = threadIdx.x; i < copies * n_ent; i += blockDim.x) {
        const int sidx = i % n_ent;
        const uint64_t* src = stab_all + (size_t)(i / n_ent) * tab_words + sidx * stride;
        if (src[0] == GB_EMPTY) continue;
        gb_merge_row(L, T, src, sidx == scap ? 1 : (sidx == scap + 1 ? 2 : 0));
    }
}

// ---------------------------------------------------------------------------- extraction
__global__ void k_gb_count_used(const uint64_t* entries, int64_t n_entries, int64_t es, unsigned long long* count) {
    unsigned long long c = 0;
    for (int64_t s = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; s < n_entries; s += (int64_t)gridDim.x * blockDim.x)
        c += entries[s * es] != GB_EMPTY;
    for (int o = 16; o; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
    if (lane_id() == 0 && c) atomicAdd(count, c);
}

// Dense SoA extraction.  Group order = slot order within 256-slot tiles, tiles in atomic-arrival
// order (unspecified, like the reference's hashbrown iteration order).
// out_words: n_words arrays of G u64.  null_pos: position of the null-key group or -1.
__global__ void __launch_bounds__(256) k_gb_extract(const uint64_t* __restrict__ entries, int64_t cap, int64_t es, int64_t ws, int pw, int n_words, unsigned long long* cursor,
                                                    uint64_t* __restrict__ out_keys, uint32_t* __restrict__ out_first, uint32_t* __restrict__ out_len,
                                                    uint64_t* __restrict__ out_words, int64_t G, long long* null_pos) {
    const int64_t n_entries = cap + 2;
    __shared__ unsigned warp_cnt[8];
    __shared__ unsigned long long tile_base;
    const int64_t ntiles = (n_entries + 255) / 256;
    for (int64_t t = blockIdx.x; t < ntiles; t += gridDim.x) {
        const int64_t s = t * 256 + threadIdx.x;
        uint64_t key = GB_EMPTY;
        if (s < n_entries) key = entries[s * es];
        const bool used = key != GB_EMPTY;
        const unsigned b = __ballot_sync(0xffffffffu, used);
        if (lane_id() == 0) warp_cnt[threadIdx.x >> 5] = __popc(b);
        __syncthreads();
        if (threadIdx.x == 0) {
            unsigned tot = 0;
            for (int w = 0; w < 8; w++) { unsigned c = warp_cnt[w]; warp_cnt[w] = tot; tot += c; }
            tile_base = tot ? atomicAdd(cursor, (unsigned long long)tot) : 0ull;
        }
        __syncthreads();
        if (used) {
            const int64_t pos = (int64_t)tile_base + warp_cnt[threadIdx.x >> 5] + __popc(b & lanemask_lt());
            const uint64_t* e = entries + s * es;
            uint64_t kout = key;
            if (s == cap) { kout = 0; *null_pos = pos; }
            else if (s == cap + 1) kout = GB_EMPTY;
            out_keys[pos] = kout;
            const uint64_t lf = e[gb_woff(s, 1, ws, pw)];
            out_len[pos] = (uint32_t)lf;
            out_first[pos] = (uint32_t)(lf >> 32);
            for (int w = 0; w < n_words; w++) out_words[(int64_t)w * G + pos] = e[gb_woff(s, 2 + w, ws, pw)];
        }
        __syncthreads();
    }
}

// per-aggregate finalisation over the dense arrays
struct FinalizeArgs {
    int kind, in_dtype, out_dtype;
    const uint64_t* main_word;     // sum / min / max accumulator (G)
    const uint64_t* nullcnt_word;  // per-group null count or nullptr
    const uint32_t* len;           // per-group len
    void* out; uint32_t* out_valid; int64_t G;
};
__device__ __forceinline__ void gb_finalize_one(const FinalizeArgs& a, int64_t g) {
    {
        bool valid = false;
        if (g < a.G) {
            const uint64_t len = a.len ? a.len[g] : 0;
            const uint64_t cnt = len - (a.nullcnt_word ? a.nullcnt_word[g] : 0);
            const uint64_t w = a.main_word ? a.main_word[g] : 0;
            valid = true;
            switch (a.kind) {
                case BL_AGG_SUM:
                    if (a.out_dtype == BL_FLOAT64) reinterpret_cast<double*>(a.out)[g] = __longlong_as_double((long long)w);
                    else if (a.out_dtype == BL_FLOAT32) reinterpret_cast<float*>(a.out)[g] = (float)__longlong_as_double((long long)w);
                    else if (dtype_size_dev(a.out_dtype) == 8) reinterpret_cast<uint64_t*>(a.out)[g] = w;
                    else reinterpret_cast<uint32_t*>(a.out)[g] = (uint32_t)w;
                    break;
                case BL_AGG_MEAN: {
                    valid = cnt > 0;
                    double m = valid ? __longlong_as_double((long long)w) / (double)cnt : 0.0;
                    if (a.out_dtype == BL_FLOAT32) reinterpret_cast<float*>(a.out)[g] = (float)m; else reinterpret_cast<double*>(a.out)[g] = m;
                    break;
                }
                case BL_AGG_MIN: case BL_AGG_MAX: {
                    valid = cnt > 0;
                    if (a.out_dtype == BL_FLOAT64 || a.out_dtype == BL_FLOAT32) {
                        const uint64_t sentinel = a.kind == BL_AGG_MIN ? 0xFFFFFFFFFFFFFFFFULL : 0ULL;
                        double v = !valid ? 0.0 : (w == sentinel ? __longlong_as_double(0x7ff8000000000000LL) : ordered_to_f64(w));   // all-NaN group -> NaN
                        if (a.out_dtype == BL_FLOAT32) reinterpret_cast<float*>(a.out)[g] = (float)v; else reinterpret_cast<double*>(a.out)[g] = v;
                    } else {
                        const uint64_t v = valid ? w : 0;
                        if (dtype_size_dev(a.out_dtype) == 8) reinterpret_cast<uint64_t*>(a.out)[g] = v; else reinterpret_cast<uint32_t*>(a.out)[g] = (uint32_t)v;
                    }
                    break;
                }
                case BL_AGG_COUNT: reinterpret_cast<uint32_t*>(a.out)[g] = (uint32_t)cnt; break;
                default: reinterpret_cast<uint32_t*>(a.out)[g] = (uint32_t)len; break;
            }
        }
        if (a.out_valid) { unsigned b = __ballot_sync(0xffffffffu, valid); if (lane_id() == 0) a.out_valid[g >> 5] = b; }
    }
}

// all outputs of finish() in ONE launch: the typed key column and every aggregate (round 1: one launch each)
constexpr int GB_FIN_MAX = 16;
struct FinalizeAll { FinalizeArgs agg[GB_FIN_MAX]; int n_aggs; const uint64_t* key_bits; int key_elem; void* key_out; uint32_t* key_valid; long long null_pos; int64_t G; };
__global__ void __launch_bounds__(256) k_gb_finalize_all(const __grid_constant__ FinalizeAll f) {
    const int64_t rounded = (f.G + 31) / 32 * 32;
    for (int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; g < rounded; g += (int64_t)gridDim.x * blockDim.x) {
        if (f.key_out != nullptr && g < f.G) { if (f.key_elem == 8) reinterpret_cast<uint64_t*>(f.key_out)[g] = f.key_bits[g]; else reinterpret_cast<uint32_t*>(f.key_out)[g] = (uint32_t)f.key_bits[g]; }
        if (f.key_valid) { const unsigned b = __ballot_sync(0xffffffffu, g < f.G && g != f.null_pos); if (lane_id() == 0) f.key_valid[g >> 5] = b; }
        for (int i = 0; i < f.n_aggs; i++) gb_finalize_one(f.agg[i], g);
    }
}

// typed key column from u64 key bits (+ validity with the null group cleared)
__global__ void k_gb_keys_out(const uint64_t* bits, int64_t G, int elem, void* out, uint32_t* out_valid, long long null_pos) {
    const int64_t rounded = (G + 31) / 32 * 32;
    for (int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; g < rounded; g += (int64_t)gridDim.x * blockDim.x) {
        if (g < G) { if (elem == 8) reinterpret_cast<uint64_t*>(out)[g] = bits[g]; else reinterpret_cast<uint32_t*>(out)[g] = (uint32_t)bits[g]; }
        if (out_valid) { unsigned b = __ballot_sync(0xffffffffu, g < G && g != null_pos); if (lane_id() == 0) out_valid[g >> 5] = b; }
    }
}

// ---------------------------------------------------------------------------- K6: partitioned export of partial rows
// row = [key, len|first, words..., meta]; partition = hash_to_partition(dirty_hash(key), P), null-key group -> 0.
// Block-local reservation: smem histogram -> one global atomicAdd per (block, partition) -> smem cursors.
constexpr int EXP_MAX_PARTS = 64;
__device__ __forceinline__ int gb_row_partition(uint64_t key, int64_t s, int64_t cap, int P) {
    if (s == cap) return 0;                                            // null key -> partition 0 (hashing.rs:113-115)
    return (int)hash_to_partition(dirty_hash(s == cap + 1 ? GB_EMPTY : key), (uint32_t)P);
}
__global__ void __launch_bounds__(256) k_gb_export_count(const uint64_t* __restrict__ entries, int64_t cap, int64_t es, int P, unsigned long long* part_counts) {
    __shared__ unsigned hist[EXP_MAX_PARTS];
    if (threadIdx.x < EXP_MAX_PARTS) hist[threadIdx.x] = 0;
    __syncthreads();
    for (int64_t s = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; s < cap + 2; s += (int64_t)gridDim.x * blockDim.x) {
        uint64_t key = entries[s * es];
        if (key != GB_EMPTY) atomicAdd(&hist[gb_row_partition(key, s, cap, P)], 1u);
    }
    __syncthreads();
    if (threadIdx.x < P && hist[threadIdx.x]) atomicAdd(&part_counts[threadIdx.x], (unsigned long long)hist[threadIdx.x]);
}
__global__ void __launch_bounds__(256) k_gb_export_scatter(const uint64_t* __restrict__ entries, int64_t cap, int64_t es, int64_t ws, int pw, int n_words, int P,
                                                           const unsigned long long* __restrict__ part_off, unsigned long long* part_cursor, uint64_t* __restrict__ rows) {
    __shared__ unsigned hist[EXP_MAX_PARTS];
    __shared__ unsigned long long base[EXP_MAX_PARTS];
    const int row_words = n_words + 3;
    const int64_t n_entries = cap + 2;
    const int64_t ntiles = (n_entries + 255) / 256;
    for (int64_t t = blockIdx.x; t < ntiles; t += gridDim.x) {
        if (threadIdx.x < EXP_MAX_PARTS) hist[threadIdx.x] = 0;
        __syncthreads();
        const int64_t s = t * 256 + threadIdx.x;
        uint64_t key = GB_EMPTY; int p = 0; unsigned local = 0;
        if (s < n_entries) key = entries[s * es];
        if (key != GB_EMPTY) { p = gb_row_partition(key, s, cap, P); local = atomicAdd(&hist[p], 1u); }
        __syncthreads();
        if (threadIdx.x < P && hist[threadIdx.x]) base[threadIdx.x] = part_off[threadIdx.x] + atomicAdd(&part_cursor[threadIdx.x], (unsigned long long)hist[threadIdx.x]);
        __syncthreads();
        if (key != GB_EMPTY) {
            const uint64_t* e = entries + s * es;
            uint64_t* dst = rows + (base[p] + local) * row_words;
            dst[0] = s == cap ? 0 : (s == cap + 1 ? GB_EMPTY : key);
            dst[1] = e[gb_woff(s, 1, ws, pw)];
            for (int w = 0; w < n_words; w++) dst[2 + w] = e[gb_woff(s, 2 + w, ws, pw)];
            dst[2 + n_words] = s == cap ? 1 : (s == cap + 1 ? 2 : 0);
        }
        __syncthreads();
    }
}

// Fused partition + exchange: same block-local reservation as k_gb_export_scatter, but the row is
// stored straight into the destination rank's window (peer memory over NVLink): partition p's rows
// land in region `my_rank` of windows[p] at [cursor .. cursor + n).  No staging copy, no collective.
struct PeerWindows { uint64_t* base[EXP_MAX_PARTS]; };
__global__ void __launch_bounds__(256) k_gb_export_p2p(const uint64_t* __restrict__ entries, int64_t cap, int64_t es, int64_t ws, int pw, int n_words, int P, const __grid_constant__ PeerWindows W,
                                                       int64_t region_words, int my_rank, int64_t rows_per_src, unsigned long long* part_cursor, int* overflow) {
    __shared__ unsigned hist[EXP_MAX_PARTS];
    __shared__ unsigned long long base[EXP_MAX_PARTS];
    const int row_words = n_words + 3;
    const int64_t n_entries = cap + 2;
    const int64_t ntiles = (n_entries + 255) / 256;
    for (int64_t t = blockIdx.x; t < ntiles; t += gridDim.x) {
        if (threadIdx.x < EXP_MAX_PARTS) hist[threadIdx.x] = 0;
        __syncthreads();
        const int64_t s = t * 256 + threadIdx.x;
        uint64_t key = GB_EMPTY; int p = 0; unsigned local = 0;
        if (s < n_entries) key = entries[s * es];
        if (key != GB_EMPTY) { p = gb_row_partition(key, s, cap, P); local = atomicAdd(&hist[p], 1u); }
        __syncthreads();
        if (threadIdx.x < P && hist[threadIdx.x]) base[threadIdx.x] = atomicAdd(&part_cursor[threadIdx.x], (unsigned long long)hist[threadIdx.x]);
        __syncthreads();
        if (key != GB_EMPTY) {
            const uint64_t pos = base[p] + local;
            if ((int64_t)pos >= rows_per_src) *overflow = 1;
            else {
                const uint64_t* e = entries + s * es;
                uint64_t* dst = W.base[p] + (int64_t)my_rank * region_words + pos * row_words;     // peer store
                dst[0] = s == cap ? 0 : (s == cap + 1 ? GB_EMPTY : key);
                dst[1] = e[gb_woff(s, 1, ws, pw)];
                for (int w = 0; w < n_words; w++) dst[2 + w] = e[gb_woff(s, 2 + w, ws, pw)];
                dst[2 + n_words] = s == cap ? 1 : (s == cap + 1 ? 2 : 0);
            }
        }
        __syncthreads();
    }
}


// ---------------------------------------------------------------------------- exchange without the host (zero syncs)
// Round 1 exchanged the per-destination row counts with an NCCL all-to-all and read them back on the host before the
// merge could be sized and launched (3 host round trips per step).  Here the counts travel through the peer windows
// themselves: the LAST CTA of the export kernel (every CTA fences its peer stores system-wide, then bumps a done
// counter) stores count and an epoch flag into the header of every destination's window (st.release.sys), and the
// owner's merge kernel — already queued on its stream — spins on the P flags with ld.acquire.sys and reads the counts
// on the device.  Window half: GB_WINDOW_HEADER_WORDS header words, then one region of rows_per_src rows per source.
__device__ __forceinline__ void st_release_sys_u64(uint64_t* p, uint64_t v) { asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory"); }
__device__ __forceinline__ uint64_t ld_acquire_sys_u64(const uint64_t* p) { uint64_t v; asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory"); return v; }
constexpr unsigned long long GB_WINDOW_OVERFLOW = ~0ull;

__global__ void __launch_bounds__(256) k_gb_export_p2p_async(const uint64_t* __restrict__ entries, int64_t cap, int64_t es, int64_t ws, int pw, int n_words, int P, const __grid_constant__ PeerWindows W,
                                                             int64_t region_words, int my_rank, int64_t rows_per_src, unsigned long long* part_cursor, unsigned* done, uint64_t epoch) {
    __shared__ unsigned hist[EXP_MAX_PARTS];
    __shared__ unsigned long long base[EXP_MAX_PARTS];
    __shared__ unsigned s_last;
    constexpr int SPT = 4, TILE = 256 * SPT;          // 1024 slots per reservation round (one global atomic per (round, partition))
    const int row_words = n_words + 3;
    const int64_t n_entries = cap + 2;
    const int64_t ntiles = (n_entries + TILE - 1) / TILE;
    for (int64_t t = blockIdx.x; t < ntiles; t += gridDim.x) {
        if (threadIdx.x < EXP_MAX_PARTS) hist[threadIdx.x] = 0;
        __syncthreads();
        uint64_t key[SPT]; int p[SPT]; unsigned local[SPT];
#pragma unroll
        for (int u = 0; u < SPT; u++) {
            const int64_t s = t * TILE + u * 256 + threadIdx.x;
            key[u] = s < n_entries ? entries[s * es] : GB_EMPTY;
        }
#pragma unroll
        for (int u = 0; u < SPT; u++) {
            const int64_t s = t * TILE + u * 256 + threadIdx.x;
            p[u] = 0; local[u] = 0;
            if (key[u] != GB_EMPTY) { p[u] = gb_row_partition(key[u], s, cap, P); local[u] = atomicAdd(&hist[p[u]], 1u); }
        }
        __syncthreads();
        if (threadIdx.x < P && hist[threadIdx.x]) base[threadIdx.x] = atomicAdd(&part_cursor[threadIdx.x], (unsigned long long)hist[threadIdx.x]);
        __syncthreads();
#pragma unroll
        for (int u = 0; u < SPT; u++) {
            if (key[u] == GB_EMPTY) continue;
            const int64_t s = t * TILE + u * 256 + threadIdx.x;
            const uint64_t pos = base[p[u]] + local[u];
            if ((int64_t)pos < rows_per_src) {
                const uint64_t* e = entries + s * es;
                uint64_t* dst = W.base[p[u]] + GB_WINDOW_HEADER_WORDS + (int64_t)my_rank * region_words + pos * row_words;     // peer store
                dst[0] = s == cap ? 0 : (s == cap + 1 ? GB_EMPTY : key[u]);
                dst[1] = e[gb_woff(s, 1, ws, pw)];
                for (int w = 0; w < n_words; w++) dst[2 + w] = e[gb_woff(s, 2 + w, ws, pw)];
                dst[2 + n_words] = s == cap ? 1 : (s == cap + 1 ? 2 : 0);
            }
        }
        __syncthreads();
    }
    // publish: all peer stores of this CTA are ordered before its done-ticket; the last CTA's flags are ordered after every ticket
    __threadfence_system();
    __syncthreads();
    if (threadIdx.x == 0) s_last = atomicAdd(done, 1u) == gridDim.x - 1 ? 1u : 0u;
    __syncthreads();
    if (s_last && threadIdx.x < P) {
        __threadfence_system();
        unsigned long long cnt = atomicAdd(&part_cursor[threadIdx.x], 0ull);
        if ((int64_t)cnt > rows_per_src) cnt = GB_WINDOW_OVERFLOW;
        uint64_t* hdr = W.base[threadIdx.x] + 2 * my_rank;
        *reinterpret_cast<volatile uint64_t*>(hdr) = cnt;
        __threadfence_system();
        st_release_sys_u64(hdr + 1, epoch);
    }
}

__global__ void __launch_bounds__(256) k_gb_merge_window(const __grid_constant__ GbLayout L, const __grid_constant__ GbTableDev T, const uint64_t* __restrict__ half, int P, int64_t rows_per_src,
                                                         int row_words, uint64_t epoch) {
    __shared__ long long s_end[EXP_MAX_PARTS];
    __shared__ int s_fail;
    if (threadIdx.x == 0) s_fail = 0;
    __syncthreads();
    if (threadIdx.x < P) {
        const long long t0 = clock64();
        uint64_t f = ld_acquire_sys_u64(half + 2 * threadIdx.x + 1);
        while (f < epoch) {
            if (clock64() - t0 > 6000000000ll) break;          // ~3 s: a peer never published (never hang the device)
            __nanosleep(200);
            f = ld_acquire_sys_u64(half + 2 * threadIdx.x + 1);
        }
        long long c = 0;
        if (f < epoch) { s_fail = 3; }
        else {
            const unsigned long long cnt = *reinterpret_cast<const volatile unsigned long long*>(half + 2 * threadIdx.x);
            if (cnt == GB_WINDOW_OVERFLOW) s_fail = 2; else c = (long long)cnt;
        }
        s_end[threadIdx.x] = c;
    }
    __syncthreads();
    if (s_fail) { if (threadIdx.x == 0) *T.status = s_fail; return; }
    if (threadIdx.x == 0) { long long acc = 0; for (int r = 0; r < P; r++) { acc += s_end[r]; s_end[r] = acc; } }
    __syncthreads();
    const int64_t total = s_end[P - 1];
    const int64_t region_words = rows_per_src * row_words;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        int r = 0; while (i >= s_end[r]) r++;
        const int64_t local = i - (r ? s_end[r - 1] : 0);
        const uint64_t* src = half + GB_WINDOW_HEADER_WORDS + (int64_t)r * region_words + local * row_words;
        gb_merge_row(L, T, src, (int)src[row_words - 1]);
    }
}

}  // namespace plb

// =============================================================================================
// Host side: plan, table sizing (sampled cardinality estimate, overflow -> grow), finish.
// Mirrors group_by_helper + evaluate_aggs (crates/polars-mem-engine/src/executors/group_by.rs:5-98).
// =============================================================================================
namespace plb {

static int knob_int(const char* name, int dflt) { const char* e = getenv(name); return e ? atoi(e) : dflt; }   // read per call (tests flip them)

static int sum_out_dtype(int dt) {
    // series/implementations/mod.rs:145-154: Int8/16, UInt8/16 sums are computed as Int64
    if (dt == BL_INT8 || dt == BL_INT16 || dt == BL_UINT8 || dt == BL_UINT16) return BL_INT64;
    return dt;
}

GroupByState::GroupByState(int key_dt, const std::vector<int>& kinds, const std::vector<int>& dtypes, const std::vector<int>& nullable, int64_t expected, bool track_first)
    : key_dtype(key_dt), agg_kinds(kinds), agg_dtypes(dtypes), expected_groups(expected) {
    PLB_REQUIRE(key_dt == BL_INT64 || key_dt == BL_UINT64 || key_dt == BL_INT32 || key_dt == BL_UINT32 || key_dt == BL_FLOAT64 || key_dt == BL_FLOAT32,
                BL_ERR_UNSUPPORTED, std::string("group_by: key dtype ") + dtype_name(key_dt) + " is outside the hot path");
    memset(&L, 0, sizeof L);
    int nw = 0;
    auto add_word = [&](int op) { PLB_REQUIRE(nw < GB_MAX_WORDS, BL_ERR_UNSUPPORTED, "group_by: too many aggregations for one pass"); L.slot_op[nw] = op; L.init[nw] = word_identity(op); return nw++; };
    for (size_t i = 0; i < kinds.size(); i++) {
        AggPlan ap; ap.kind = kinds[i]; ap.in_dtype = dtypes[i]; ap.main = -1; ap.nullcnt = -1; ap.nullable = nullable.empty() || nullable[i] != 0;
        if (ap.kind != BL_AGG_LEN)
            PLB_REQUIRE(ap.in_dtype == BL_INT64 || ap.in_dtype == BL_UINT64 || ap.in_dtype == BL_INT32 || ap.in_dtype == BL_UINT32 || ap.in_dtype == BL_FLOAT64 || ap.in_dtype == BL_FLOAT32,
                        BL_ERR_UNSUPPORTED, std::string("group_by: value dtype ") + dtype_name(ap.in_dtype) + " is outside the hot path");
        const bool flt = dtype_is_float(ap.in_dtype), sgn = dtype_is_signed(ap.in_dtype);
        // a null counter is only needed when the column can hold nulls (valid count = len - nulls); without it
        // the C2 entry is key + len|first + 2 accumulators = 32 bytes = one sector
        const bool nl = nullable.empty() || nullable[i] != 0;
        auto null_word = [&]() { return nl ? add_word(W_NULLCNT) : -1; };
        switch (ap.kind) {
            case BL_AGG_SUM: ap.main = add_word(flt ? W_ADD_F64 : W_ADD_INT); ap.out_dtype = sum_out_dtype(ap.in_dtype); break;
            case BL_AGG_MEAN: ap.main = add_word(W_ADD_F64); ap.nullcnt = null_word(); ap.out_dtype = ap.in_dtype == BL_FLOAT32 ? BL_FLOAT32 : BL_FLOAT64; L.need_len = 1; break;
            case BL_AGG_MIN: ap.main = add_word(flt ? W_MIN_F64 : (sgn ? W_MIN_S64 : W_MIN_U64)); ap.nullcnt = null_word(); ap.out_dtype = ap.in_dtype; L.need_len = 1; break;
            case BL_AGG_MAX: ap.main = add_word(flt ? W_MAX_F64 : (sgn ? W_MAX_S64 : W_MAX_U64)); ap.nullcnt = null_word(); ap.out_dtype = ap.in_dtype; L.need_len = 1; break;
            case BL_AGG_COUNT: ap.nullcnt = null_word(); ap.out_dtype = BL_UINT32; L.need_len = 1; break;
            case BL_AGG_LEN: ap.out_dtype = BL_UINT32; L.need_len = 1; break;
            case BL_AGG_MEDIAN: case BL_AGG_QUANTILE: fail(BL_ERR_UNSUPPORTED, "group_by: median / quantile cannot be pre-aggregated (use bl_groupby_agg)");
            default: fail(BL_ERR_INVALID, "group_by: unknown aggregation kind");
        }
        plans.push_back(ap);
    }
    L.n_words = nw;
    L.pair_k = -1; L.pair_c = -1;
    if (L.need_len) for (int w = 0; w < nw && !pair_word; w++) if (L.slot_op[w] == W_ADD_INT) pair_word = 2 + w;
    L.stride = ((2 + nw + 3) / 4) * 4;      // whole 32-byte sectors per entry
    L.need_first = track_first ? 1 : 0;      // maintain_order / first-occurrence key output; costs one 32-bit RED per row
    status = dev_alloc(4);
}

void GroupByState::alloc_table(uint64_t new_cap) {
    cap = new_cap;
    entries = dev_alloc((size_t)(cap + 2) * L.stride * 8);
    int shift = 64; for (uint64_t c = cap; c > 1; c >>= 1) shift--;
    const int hint = [] { const char* e = getenv("BL_K5_HINT"); return e ? atoi(e) : 0; }();
    // word-major planes by default: the REDs of one row then hit different sectors / L2 slices (ubench: 54 vs 38 G rows/s)
    const int soa = [] { const char* e = getenv("BL_K5_SOA"); return e ? atoi(e) : 1; }();
    T.entries = as<uint64_t>(entries); T.cap = cap; T.shift = shift; T.status = as<int>(status); T.hint = hint;
    T.es = soa ? 1 : L.stride; T.ws = soa ? (int64_t)(cap + 2) : 1; T.soa = soa; T.pass_bits = 0; T.pass_id = 0;
    // pair layout + bulk reduce (k_gb_consume<BULK>): only where the plain-RED kernels do not run on this table — the shared-memory plan
    // (few groups) and the heavy-hitter kernel keep word-major planes (their cold-path REDs on len and the paired sum would share a sector)
    // BL_K5_BULK: 0 never; 1 (default) where the lean kernel applies (faster than the 3-RED kernel on C2;
    // the GENERAL bulk kernel is issue-bound and loses, most with nulls); 2 always (parity tests of the general kernel)
    const int bulk_knob = knob_int("BL_K5_BULK", 1);
    const int bulk = bulk_knob >= 2 ? 1 : (bulk_knob == 1 && lean_shape ? 1 : 0);
    bool smem_plan = false;     // same rule as launch_batch
    if (est_groups > 0 && knob_int("BL_K5_SMEM", 1)) { int64_t want = 16; while (2 * want < 3 * est_groups && want < (1 << 20)) want <<= 1; smem_plan = (size_t)(want + 2) * L.stride * 8 <= (size_t)72 * 1024; }
    T.pw = (soa && bulk > 0 && pair_word >= 2 && hot.rows == 0 && !smem_plan) ? pair_word : 0;
    T.bulk_lanes = T.pw ? std::min(32, std::max(0, knob_int("BL_K5_BULK_LANES", 32))) : 0;
    PLB_LAUNCH("k5_table_init", k_gb_init, grid_for((int64_t)(cap + 2) * L.stride, 256), 256, 0, T.entries, (int64_t)(cap + 2), L.stride, soa, T.pw, L);
    dev_memset(status->p, 0, 4);
}

static uint64_t pow2_at_least(double x) { uint64_t c = 1024; while ((double)c < x && c < (1ull << 40)) c <<= 1; return c; }

// Birthday-style inversion: d distinct keys in a sample of m rows out of n  ->  estimate of the
// number of groups.  (The reference samples too: executors/group_by_streaming.rs:117-139.)
static double estimate_groups(double d, double m, double n) {
    if (d >= m * 0.995) return n;               // (almost) all distinct: could be anything up to n
    double lo = d, hi = n > d ? n : d;
    for (int it = 0; it < 60; it++) { double G = 0.5 * (lo + hi); double ex = G * (1.0 - exp(-m / G)); if (ex < d) lo = G; else hi = G; }
    return hi;
}

// Heavy hitters -> device lookup table for k_gb_consume_hot (keys at their hashed slot, dense row index per slot).
void GroupByState::build_hot_list(const void* cand_v, int n_cand, bool null_hot, bool empty_hot, double m) {
    const GbCandidate* cand = static_cast<const GbCandidate*>(cand_v);
    hot = GbHotDev{}; hot_share = 0; hot_buf.reset();
    const int on = [] { const char* e = getenv("BL_K5_HOTKEYS"); return e ? atoi(e) : 1; }();
    if (!on || (n_cand <= 0 && !null_hot && !empty_hot)) return;
    std::vector<GbCandidate> c(cand, cand + std::max(n_cand, 0));
    std::sort(c.begin(), c.end(), [](const GbCandidate& a, const GbCandidate& b) { return a.mult > b.mult || (a.mult == b.mult && a.key < b.key); });
    const int row_words = 2 + L.n_words;
    int n_hot = std::min<int>((int)c.size(), std::min(GB_HOT_MAX, 512 / row_words - 2));     // <= 4 KB of accumulator rows per warp
    if (n_hot < 0) n_hot = 0;
    if (!c.empty()) hot_share = (double)c[0].mult / m;
    std::vector<unsigned char> h(GB_HOT_SLOTS * 8 + GB_HOT_SLOTS, 0);
    uint64_t* hk = reinterpret_cast<uint64_t*>(h.data());
    unsigned char* hi = h.data() + GB_HOT_SLOTS * 8;
    for (int i = 0; i < GB_HOT_SLOTS; i++) hk[i] = GB_EMPTY;
    for (int i = 0; i < n_hot; i++) {
        unsigned sl = (unsigned)(table_hash(c[i].key) >> (64 - GB_HOT_BITS));
        while (hk[sl] != GB_EMPTY) sl = (sl + 1) & (GB_HOT_SLOTS - 1);
        hk[sl] = c[i].key; hi[sl] = (unsigned char)i;
    }
    hot_buf = dev_alloc(h.size());
    PLB_CUDA(cudaMemcpyAsync(hot_buf->p, h.data(), h.size(), cudaMemcpyHostToDevice, ctx().stream));
    PLB_CUDA(cudaStreamSynchronize(ctx().stream));      // `h` lives on this frame
    hot.keys = as<uint64_t>(hot_buf); hot.idx = reinterpret_cast<const uint8_t*>(hot_buf->p) + GB_HOT_SLOTS * 8;
    hot.n_hot = n_hot; hot.null_hot = null_hot ? 1 : 0; hot.empty_hot = empty_hot ? 1 : 0; hot.rows = n_hot + 2;
}

uint64_t GroupByState::choose_cap(const DevCol& key, int64_t n_total) {
    double G, G_raw, G_upper = 0;
    if (expected_groups > 0) G = G_raw = (double)expected_groups;
    else {
        const int64_t n = key.len, m = std::min<int64_t>(n, 65536);
        const uint64_t scap = 1 << 18;
        // one allocation: multiplicities | stats | heavy-hitter candidates (read back with one copy)
        const size_t tail_bytes = sizeof(GbSampleStats) + sizeof(GbCandidate) * GB_CAND_MAX;
        DevPtr scratch = dev_alloc(scap * 8), mult = dev_alloc(scap * 4 + tail_bytes);
        GbSampleStats* dstats = reinterpret_cast<GbSampleStats*>(as<unsigned>(mult) + scap);
        GbCandidate* dcand = reinterpret_cast<GbCandidate*>(dstats + 1);
        const double nt = (double)std::max<int64_t>(n_total, n);
        // a key is "hot" when its rows would serialise on one L2 address for >~0.15 ms (a few ns per same-address RED)
        const double hot_rows = [] { const char* e = getenv("BL_K5_HOT_ROWS"); double v = e ? atof(e) : 30000.0; return v >= 0 ? v : 30000.0; }();
        const unsigned hot_thr = (unsigned)std::max(12.0, std::ceil(hot_rows * (double)m / nt));
        PLB_LAUNCH("k5_fill", k_fill_u64, grid_for(scap, 256), 256, 0, as<uint64_t>(scratch), GB_EMPTY, (int64_t)scap);
        dev_memset(mult->p, 0, scap * 4 + sizeof(GbSampleStats));
        PLB_LAUNCH("k5_estimate", k_gb_estimate, grid_for(m, 256), 256, 0, key.v(), key.vm(), key.dtype, n, m, as<uint64_t>(scratch), as<unsigned>(mult), scap, 64 - 18, dstats);
        PLB_LAUNCH("k5_estimate", k_gb_estimate_stats, grid_for(scap, 256), 256, 0, as<uint64_t>(scratch), as<unsigned>(mult), (int64_t)scap, hot_thr, dstats, dcand);
        std::vector<unsigned char> hbuf(tail_bytes);
        PLB_CUDA(cudaMemcpyAsync(hbuf.data(), dstats, tail_bytes, cudaMemcpyDeviceToHost, ctx().stream));
        PLB_CUDA(cudaStreamSynchronize(ctx().stream));
        GbSampleStats st; memcpy(&st, hbuf.data(), sizeof st);
        const GbCandidate* cand = reinterpret_cast<const GbCandidate*>(hbuf.data() + sizeof(GbSampleStats));
        G_raw = estimate_groups((double)st.distinct, (double)m, nt);
        // skewed keys: the uniform inversion collapses onto the hot head of the distribution.  Chao's
        // estimator (distinct + f1^2 / 2 f2, from the keys sampled exactly once / twice) recovers the
        // long tail; take the larger of the two (an under-estimate costs a restart, an over-estimate L2 misses)
        if (m < n && st.f1 > 0) {
            const double chao = (double)st.distinct + (double)st.f1 * ((double)st.f1 - 1.0) / (2.0 * ((double)st.f2 + 1.0));
            if (chao > G_raw) G_raw = chao;
            // (almost) every sampled key distinct: the inversion above gives up and answers "up to one group per row" (1e7 keys
            // in 1e8 rows were sized for 1e8 groups: an 8 GB table).  With a handful of keys seen twice Chao's estimator
            // is already tight (f2 = 215 for that case -> 9.9e6); keep a 2x margin, an under-estimate only costs a restart.
            if ((double)st.distinct >= (double)m * 0.995 && st.f2 >= 16) G_raw = std::min(G_raw, 2.0 * chao);
        }
        // sorted / clustered keys: every group is at least one run of equal neighbours, so groups <= runs
        // = rows * (1 - P[next row has the same key]) — a strided sample of such data looks all-distinct
        sample_adjacent = m > 0 ? (double)st.adjacent / (double)m : 0.0;
        if (m < n && sample_adjacent > 0.5) {
            const double q = 1.0 - sample_adjacent;
            const double runs = nt * std::min(1.0, q + 3.0 * std::sqrt(q * sample_adjacent / (double)m) + 2.0 / (double)m) + 1.0;
            if (runs < G_raw) G_raw = runs;
        }
        G = G_raw * 1.25 + 64;
        if (G > nt) G = nt;
        if (G_raw > nt) G_raw = nt;
        // Good-Turing: a fraction f1/m of the rows carries keys the sample has not seen; if every such row were a
        // new key the table would need distinct + (f1/m) * rows entries.  Heavy-tailed keys sit between the two
        // (Zipf(1.1): Chao 2.6e5, truth 1e6), so the table takes whatever the L2 budget allows up to that bound.
        G_upper = std::min(nt, (double)st.distinct + (double)st.f1 / (double)m * nt);
        build_hot_list(cand, (int)std::min<unsigned>(st.n_cand, GB_CAND_MAX), st.nulls >= hot_thr, st.empties >= hot_thr, (double)m);
    }
    est_groups = (int64_t)(G_raw * 1.25) + 2;      // for the shared-memory plan (overflow falls through to the global table)
    const double lf = [] { const char* e = getenv("BL_K5_LF"); double v = e ? atof(e) / 100.0 : 0.6; return (v > 0.05 && v < 0.95) ? v : 0.6; }();
    uint64_t c = pow2_at_least(G / lf);       // load factor <= 0.6 by default
    // keep the table inside L2 when a load factor <= 0.85 allows it: past ~55 % of L2 the REDs miss and the
    // kernel slows down ~3x, while linear probing over
    // word-major key planes (4 keys per sector) stays cheap at higher load factors
    const double l2_budget = 0.55 * (double)ctx().l2_bytes;
    if ((double)c * L.stride * 8 > l2_budget && G_raw / ((double)c / 2) <= 0.8 && c > 1024) c >>= 1;   // an under-estimate costs one restart
    // spare L2 is free insurance against an under-estimate (load factors 0.15-0.6 run at the same speed; a table at
    // 95 % load ran 7x slower): grow towards the Good-Turing bound while the table stays inside the L2 budget
    while (G_upper / lf > (double)c && (double)(2 * c) * L.stride * 8 <= l2_budget) c <<= 1;
    if (getenv("BL_K5_DEBUG"))
        fprintf(stderr, "[k5] rows=%lld est_groups=%.0f upper=%.0f cap=%llu (%.1f MB) hot_keys=%d null_hot=%d empty_hot=%d hot_share=%.4f adjacent=%.3f\n", (long long)n_total, G_raw, G_upper,
                (unsigned long long)c, (double)c * L.stride * 8 / 1e6, hot.n_hot, hot.null_hot, hot.empty_hot, hot_share, sample_adjacent);
    return c;
}

template <int KEY_ELEM, int KEY_CANON, bool KEY_NULLS, int PAIRS, bool BULK>
static void launch_consume_p(const GbLayout& L, const GbTableDev& T, const GbBatch& B, int grid) {
    const size_t smem = BULK ? (size_t)2 * PAIRS * 256 * 16 : 0;     // staging cells of the bulk reduces
    if (L.n_cols <= 1) PLB_LAUNCH("k5_groupby_agg", (k_gb_consume<KEY_ELEM, KEY_CANON, KEY_NULLS, 1, PAIRS, BULK>), grid, 256, smem, L, T, B);
    else if (L.n_cols <= 2) PLB_LAUNCH("k5_groupby_agg", (k_gb_consume<KEY_ELEM, KEY_CANON, KEY_NULLS, 2, PAIRS, BULK>), grid, 256, smem, L, T, B);
    else if (L.n_cols <= 4) PLB_LAUNCH("k5_groupby_agg", (k_gb_consume<KEY_ELEM, KEY_CANON, KEY_NULLS, 4, PAIRS, BULK>), grid, 256, smem, L, T, B);
    else PLB_LAUNCH("k5_groupby_agg", (k_gb_consume<KEY_ELEM, KEY_CANON, KEY_NULLS, 8, 1, BULK>), grid, 256, BULK ? (size_t)2 * 256 * 16 : 0, L, T, B);
}
template <int KEY_ELEM, int KEY_CANON, bool KEY_NULLS>
static void launch_consume(const GbLayout& L, const GbTableDev& T, const GbBatch& B, int grid) {
    const int pairs = knob_int("BL_K5_PAIRS", 1) == 2 ? 2 : 1;
    if (T.pw && T.bulk_lanes > 0 && L.pair_k >= 0) {
        // lean kernel for the common analytic shape (see k_gb_consume_lean)
        bool lean = KEY_ELEM == 8 && KEY_CANON == 0 && T.bulk_lanes == 32 && !T.hint && !L.need_first && L.need_len && L.n_cols >= 1 && L.n_cols <= 3 &&
                    knob_int("BL_K5_LEAN", 1) != 0;
        bool nulls = KEY_NULLS;
        for (int c = 0; lean && c < L.n_cols; c++) { lean = B.cols[c].elem == 8 && L.col_kbegin[c + 1] - L.col_kbegin[c] <= 2; nulls = nulls || B.cols[c].validity != nullptr; }
        if (lean) {
            const size_t smem = (size_t)2 * 256 * 16;
#define GB_LEAN(NC) do { if (nulls) PLB_LAUNCH("k5_groupby_agg", (k_gb_consume_lean<NC, true>), grid, 256, smem, L, T, B); \
                         else PLB_LAUNCH("k5_groupby_agg", (k_gb_consume_lean<NC, false>), grid, 256, smem, L, T, B); } while (0)
            if (L.n_cols == 1) GB_LEAN(1); else if (L.n_cols == 2) GB_LEAN(2); else GB_LEAN(3);
#undef GB_LEAN
        } else launch_consume_p<KEY_ELEM, KEY_CANON, KEY_NULLS, 1, true>(L, T, B, grid);
    }
    else if (pairs == 2) launch_consume_p<KEY_ELEM, KEY_CANON, KEY_NULLS, 2, false>(L, T, B, grid);
    else launch_consume_p<KEY_ELEM, KEY_CANON, KEY_NULLS, 1, false>(L, T, B, grid);
}

template <int KEY_ELEM, int KEY_CANON, bool KEY_NULLS, int MAXC>
static void launch_hot_c(const GbLayout& L, const GbTableDev& T, const GbBatch& B, const GbHotDev& H, int grid) {
    auto kfn = k_gb_consume_hot<KEY_ELEM, KEY_CANON, KEY_NULLS, MAXC>;
    const size_t smem = (size_t)GB_HOT_SLOTS * 8 + (size_t)8 * H.rows * (2 + L.n_words) * 8 + GB_HOT_SLOTS;
    PLB_CUDA(cudaFuncSetAttribute(kfn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    PLB_LAUNCH("k5_groupby_agg_hot", kfn, grid, 256, smem, L, T, B, H);
}
template <int KEY_ELEM, int KEY_CANON, bool KEY_NULLS>
static void launch_hot(const GbLayout& L, const GbTableDev& T, const GbBatch& B, const GbHotDev& H, int grid) {
    if (L.n_cols <= 1) launch_hot_c<KEY_ELEM, KEY_CANON, KEY_NULLS, 1>(L, T, B, H, grid);
    else if (L.n_cols <= 2) launch_hot_c<KEY_ELEM, KEY_CANON, KEY_NULLS, 2>(L, T, B, H, grid);
    else if (L.n_cols <= 4) launch_hot_c<KEY_ELEM, KEY_CANON, KEY_NULLS, 4>(L, T, B, H, grid);
    else launch_hot_c<KEY_ELEM, KEY_CANON, KEY_NULLS, 8>(L, T, B, H, grid);
}

template <int KEY_ELEM, int KEY_CANON, bool KEY_NULLS, int MAXC, bool FAST>
static void launch_smem_cf(const GbLayout& L, const GbTableDev& T, const GbBatch& B, int scap) {
    auto kfn = k_gb_consume_smem<KEY_ELEM, KEY_CANON, KEY_NULLS, MAXC, FAST>;
    const size_t tab_bytes = ((size_t)(scap + 2) * L.stride + 2) * 8;
    const int copies = (int)std::min<size_t>(32, std::max<size_t>(1, (size_t)(96 * 1024) / tab_bytes));
    const size_t smem = tab_bytes * copies;
    PLB_CUDA(cudaFuncSetAttribute(kfn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    int per_sm = (int)std::min<size_t>(4, std::max<size_t>(1, (size_t)(220 * 1024) / (smem + 1024)));
    int sshift = 64; for (int c = scap; c > 1; c >>= 1) sshift--;
    const int grid = (int)std::min<int64_t>((int64_t)ctx().sm_count * per_sm, std::max<int64_t>(1, (B.n / 2 + 511) / 512));
    PLB_LAUNCH("k5_groupby_agg_smem", kfn, grid, 512, smem, L, T, B, scap, sshift, copies);
}
template <int KEY_ELEM, int KEY_CANON, bool KEY_NULLS, int MAXC>
static void launch_smem_c(const GbLayout& L, const GbTableDev& T, const GbBatch& B, int scap) {
    bool fast = true;
    for (int c = 0; c < L.n_cols; c++) fast = fast && B.cols[c].elem == 8 && B.cols[c].validity == nullptr;
    if (fast) launch_smem_cf<KEY_ELEM, KEY_CANON, KEY_NULLS, MAXC, true>(L, T, B, scap);
    else launch_smem_cf<KEY_ELEM, KEY_CANON, KEY_NULLS, MAXC, false>(L, T, B, scap);
}
template <int KEY_ELEM, int KEY_CANON, bool KEY_NULLS>
static void launch_smem(const GbLayout& L, const GbTableDev& T, const GbBatch& B, int scap) {
    if (L.n_cols <= 1) launch_smem_c<KEY_ELEM, KEY_CANON, KEY_NULLS, 1>(L, T, B, scap);
    else if (L.n_cols <= 2) launch_smem_c<KEY_ELEM, KEY_CANON, KEY_NULLS, 2>(L, T, B, scap);
    else if (L.n_cols <= 4) launch_smem_c<KEY_ELEM, KEY_CANON, KEY_NULLS, 4>(L, T, B, scap);
    else launch_smem_c<KEY_ELEM, KEY_CANON, KEY_NULLS, 8>(L, T, B, scap);
}

void GroupByState::launch_batch(const DevCol& key, const std::vector<const DevCol*>& values, int64_t row_base) {
    // per-batch column binding: aggregations over the same buffer share one column slot
    GbBatch B; memset(&B, 0, sizeof B);
    B.keys = key.v(); B.key_validity = key.vm(); B.n = key.len; B.row_base = (uint32_t)row_base; B.key_dtype = key.dtype;
    std::vector<const void*> col_ptr; std::vector<int> col_of_agg(plans.size(), -1);
    // pair layout: the column of the paired integer sum is bound first (column 0: the bulk-reduce kernel reads it with a static index)
    std::vector<size_t> plan_order;
    for (size_t i = 0; i < plans.size(); i++) if (T.pw && plans[i].main == T.pw - 2) plan_order.push_back(i);
    for (size_t i = 0; i < plans.size(); i++) if (!(T.pw && plans[i].main == T.pw - 2)) plan_order.push_back(i);
    for (size_t i : plan_order) {
        if (plans[i].kind == BL_AGG_LEN) continue;
        const DevCol* v = values[i];
        PLB_REQUIRE(v != nullptr && v->len == key.len, BL_ERR_INVALID, "group_by: value column length differs from key length");
        PLB_REQUIRE(v->dtype == plans[i].in_dtype, BL_ERR_DTYPE, "group_by: value dtype differs from the plan");
        PLB_REQUIRE(plans[i].nullable || v->validity == nullptr, BL_ERR_INVALID, "group_by: a column declared non-nullable carries a validity bitmap");
        int c = -1;
        for (size_t j = 0; j < col_ptr.size(); j++) if (col_ptr[j] == v->v() && B.cols[j].validity == v->vm()) c = (int)j;
        if (c < 0) {
            PLB_REQUIRE(col_ptr.size() < GB_MAX_COLS, BL_ERR_UNSUPPORTED, "group_by: more than 8 distinct value columns in one pass");
            c = (int)col_ptr.size(); col_ptr.push_back(v->v());
            B.cols[c].values = v->v(); B.cols[c].validity = v->vm(); B.cols[c].dtype = v->dtype; B.cols[c].elem = dtype_size(v->dtype);
        }
        col_of_agg[i] = c;
    }
    GbLayout Lb = L;
    Lb.n_cols = (int)col_ptr.size();
    int k = 0;
    for (int c = 0; c < Lb.n_cols; c++) {
        Lb.col_kbegin[c] = k;
        for (size_t i = 0; i < plans.size(); i++) {
            if (col_of_agg[i] != c) continue;
            if (plans[i].main >= 0) { Lb.wslot[k] = plans[i].main; Lb.wop[k] = L.slot_op[plans[i].main]; k++; }
            // null counters only matter when the column can hold nulls
            if (plans[i].nullcnt >= 0 && B.cols[c].validity != nullptr) { Lb.wslot[k] = plans[i].nullcnt; Lb.wop[k] = W_NULLCNT; k++; }
        }
    }
    for (int c = Lb.n_cols; c <= GB_MAX_COLS; c++) Lb.col_kbegin[c] = k;
    Lb.pair_k = -1; Lb.pair_c = -1;
    if (T.pw) for (int c = 0; c < Lb.n_cols; c++) for (int j = Lb.col_kbegin[c]; j < Lb.col_kbegin[c + 1]; j++) if (c == 0 && 2 + Lb.wslot[j] == T.pw && Lb.wop[j] == W_ADD_INT) { Lb.pair_k = j; Lb.pair_c = c; }
    const int64_t n = key.len;
    if (n == 0) return;
    // CTAs per SM of the grid-stride launch (more than are resident: 5-6; shorter CTAs even out the tail).  BL_K5_BPS overrides.
    const bool lean_table = T.pw != 0 && lean_shape;
    const int bps = std::max(1, knob_int("BL_K5_BPS", lean_table ? 48 : 24));
    const int grid = grid_for((n / 2 + 1), 256, bps);
    const int grid_hot = grid_for((n / 2 + 1), 256, std::max(1, knob_int("BL_K5_BPS", 8)));     // every warp merges its private rows at the end: keep the CTA count low
    const bool kn = key.validity != nullptr;
    const int elem = dtype_size(key.dtype);
    const int canon = key.dtype == BL_FLOAT64 ? 1 : (key.dtype == BL_FLOAT32 ? 2 : 0);
    // keys must be 16-byte aligned for the 128-bit path (device columns always are)
    // low-cardinality plan: CTA-private shared-memory tables (largest table that leaves >= 1 CTA per SM)
    const int smem_on = [] { const char* e = getenv("BL_K5_SMEM"); return e ? atoi(e) : 1; }();
    int scap = 0;
    if (smem_on && est_groups > 0) {
        // load factor <= 2/3 (probing a shared-memory table is cheap; occupancy is not)
        int want = 16; while (2 * want < 3 * est_groups && want < (1 << 20)) want <<= 1;   // tiny tables leave room for up to 32 replicas
        // beyond ~72 KB of table per CTA the occupancy loss outweighs the cheaper atomics
        if ((size_t)(want + 2) * Lb.stride * 8 <= (size_t)72 * 1024) scap = want;
    }
    // skewed keys: the CTA-private tables serialise on the hot key's shared-memory address as soon as more than a
    // few of the CTA's 512 threads work on it; with too few replicas to spread
    // that load, take the global table + warp-private heavy-hitter rows instead
    if (scap && hot.rows > 0) {
        const size_t tab_bytes = ((size_t)(scap + 2) * Lb.stride + 2) * 8;
        const double copies = (double)std::min<size_t>(32, std::max<size_t>(1, (size_t)(96 * 1024) / tab_bytes));
        if (hot_share * 512.0 / copies > 4.0) scap = 0;
    }
    // hot-table mode (experimental knob): run the shared-memory kernel with BL_K5_HOT slots even though the
    // groups do not fit; the first keys a CTA sees (the hot head of a skewed distribution) aggregate in shared
    // memory, everything else falls through to the global table
    const int hot_slots = [] { const char* e = getenv("BL_K5_HOT"); int v = e ? atoi(e) : 0; int c = 0; if (v > 0) { c = 16; while (c < v && c < 2048) c <<= 1; } return c; }();
    if (!scap && hot_slots) scap = hot_slots;
    // tables that cannot stay L2-resident are filled in several passes over the batch: pass h only touches the
    // slot sub-range h of every plane (slot = top hash bits), so each pass works on an L2-sized slice
    int pass_bits = 0;
    if (!scap) {
        const int mp = [] { const char* e = getenv("BL_K5_MULTIPASS"); return e ? atoi(e) : 1; }();
        const double tbl = (double)(cap + 2) * L.stride * 8, budget = 0.55 * (double)ctx().l2_bytes;
        while (mp && pass_bits < 3 && tbl / (double)(1 << pass_bits) > budget) pass_bits++;
        // every pass re-reads the batch: beyond 4 passes (or when even a quarter does not fit) the extra scans cost
        // more than the L2 misses they avoid
        if (pass_bits > 2) pass_bits = 0;
    }
    GbTableDev Tp = T;
    const bool use_hot = hot.rows > 0;
#define GB_LAUNCH_ALL(E, C, KN)                                                      \
    do { for (int h = 0; h < (1 << pass_bits); h++) { Tp.pass_bits = pass_bits; Tp.pass_id = h;                                              \
             if (use_hot) launch_hot<E, C, KN>(Lb, Tp, B, hot, grid_hot); else launch_consume<E, C, KN>(Lb, Tp, B, grid); } } while (0)
#define GB_DISPATCH(E, C)                                                            \
    do { if (scap) { if (kn) launch_smem<E, C, true>(Lb, T, B, scap); else launch_smem<E, C, false>(Lb, T, B, scap); }                       \
         else if (kn) GB_LAUNCH_ALL(E, C, true); else GB_LAUNCH_ALL(E, C, false); } while (0)
    if (elem == 8) { if (canon == 1) GB_DISPATCH(8, 1); else GB_DISPATCH(8, 0); }
    else { if (canon == 2) GB_DISPATCH(4, 2); else GB_DISPATCH(4, 0); }
#undef GB_DISPATCH
#undef GB_LAUNCH_ALL
}

// does the batch have the shape k_gb_consume_lean takes?  (decides the table layout, so it is asked before alloc_table)
void GroupByState::note_batch_shape(const DevCol& key, const std::vector<const DevCol*>& values) {
    bool ok = pair_word >= 2 && !L.need_first && L.need_len && (key.dtype == BL_INT64 || key.dtype == BL_UINT64);
    std::vector<const void*> cols; std::vector<int> words;
    for (size_t i = 0; ok && i < plans.size(); i++) {
        if (plans[i].kind == BL_AGG_LEN) continue;
        const DevCol* v = i < values.size() ? values[i] : nullptr;
        if (!v || dtype_size(v->dtype) != 8) { ok = false; break; }
        size_t c = 0; while (c < cols.size() && cols[c] != v->v()) c++;
        if (c == cols.size()) { cols.push_back(v->v()); words.push_back(0); }
        words[c] += (plans[i].main >= 0 ? 1 : 0) + (plans[i].nullcnt >= 0 && v->validity != nullptr ? 1 : 0);
    }
    for (int w : words) ok = ok && w <= 2;
    lean_shape = ok && !cols.empty() && cols.size() <= 3;
}

void GroupByState::grow(uint64_t new_cap) {
    // rehash: merge the old table's entries into a bigger one
    DevPtr old = entries; const uint64_t old_cap = cap; const int64_t old_es = T.es, old_ws = T.ws; const int old_pw = T.pw;
    alloc_table(new_cap);
    if (old) PLB_LAUNCH("k5_rehash", k_gb_merge, grid_for((int64_t)old_cap + 2, 256), 256, 0, L, T, as<uint64_t>(old), (int64_t)old_cap + 2, old_es, old_ws, 1, (int64_t)old_cap, old_pw);
}

int64_t GroupByState::count_groups() {
    DevPtr c = dev_alloc(8); dev_memset(c->p, 0, 8);
    PLB_LAUNCH("k5_count_used", k_gb_count_used, grid_for((int64_t)cap + 2, 256), 256, 0, T.entries, (int64_t)cap + 2, T.es, as<unsigned long long>(c));
    return (int64_t)read_scalar(as<unsigned long long>(c));
}

// One-shot consume with restart: if the optimistic table overflows the whole pass is redone into a
// table 8x larger (the batch stays resident on the device, so this costs compute only).
// Pipelined one-shot consume for host inputs: `ready[c]` is recorded on the copy stream when chunk c
// (rows [c*chunk_rows, ...)) of every column has landed in the resident device copies; the compute
// stream consumes chunk c while chunk c+1 is still in flight.  Falls back to a full restart on the
// resident copy if the optimistic table overflows.
void GroupByState::consume_pipelined(const DevCol& key, const std::vector<const DevCol*>& values, int64_t chunk_rows, const std::vector<cudaEvent_t>& ready) {
    PLB_REQUIRE(key.dtype == key_dtype, BL_ERR_DTYPE, "group_by: key dtype differs from the plan");
    PLB_REQUIRE(key.len <= 0xFFFFFFFEll, BL_ERR_UNSUPPORTED, "group_by: more than 2^32-2 rows (IdxSize = u32)");
    Context& c = ctx();
    const int64_t n = key.len;
    const int es = dtype_size(key.dtype);
    auto slice = [&](const DevCol& col, int64_t lo, int64_t len) {
        DevCol s; s.dtype = col.dtype; s.len = len; s.null_count = 0;
        s.values = dev_borrow((const char*)col.v() + lo * dtype_size(col.dtype), (size_t)len * dtype_size(col.dtype));
        return s;
    };
    (void)es;
    for (size_t ci = 0; ci < ready.size(); ci++) {
        const int64_t lo = (int64_t)ci * chunk_rows, len = std::min<int64_t>(chunk_rows, n - lo);
        PLB_CUDA(cudaStreamWaitEvent(c.stream, ready[ci], 0));
        DevCol ks = slice(key, lo, len);
        if (ci == 0) { note_batch_shape(key, values); alloc_table(choose_cap(ks, n)); }
        std::vector<DevCol> vs(values.size()); std::vector<const DevCol*> vp(values.size(), nullptr);
        for (size_t i = 0; i < values.size(); i++) {
            if (!values[i]) continue;
            size_t dup = i;
            for (size_t j = 0; j < i; j++) if (values[j] == values[i]) { dup = j; break; }
            if (dup != i) { vp[i] = vp[dup]; continue; }
            vs[i] = slice(*values[i], lo, len); vp[i] = &vs[i];
        }
        launch_batch(ks, vp, lo);
    }
    if (read_scalar(as<int>(status)) == 0) { rows_seen = n; return; }
    // rare: the sampled estimate was too small — redo on the (now fully resident) device copy
    uint64_t cap2 = cap * 8;
    for (int attempt = 0; attempt < 8; attempt++) {
        alloc_table(cap2);
        launch_batch(key, values, 0);
        if (read_scalar(as<int>(status)) == 0) { rows_seen = n; return; }
        cap2 *= 8;
    }
    fail(BL_ERR_OOM, "group_by: hash table kept overflowing");
}

void GroupByState::consume_all(const DevCol& key, const std::vector<const DevCol*>& values) {
    PLB_REQUIRE(key.dtype == key_dtype, BL_ERR_DTYPE, "group_by: key dtype differs from the plan");
    PLB_REQUIRE(key.len <= 0xFFFFFFFEll, BL_ERR_UNSUPPORTED, "group_by: more than 2^32-2 rows (IdxSize = u32)");
    uint64_t c = choose_cap(key, key.len);
    note_batch_shape(key, values);
    if (consume_radix(key, values, c)) return;      // tables beyond L2: partition the rows instead (groupby_radix.cu)
    // optimistic: no host round trip here — finish() reads the status word together with the group count and, if the sampled
    // estimate was too small, redoes the batch into a table 8x larger (the inputs outlive the state in every caller)
    alloc_table(c);
    launch_batch(key, values, 0);
    rows_seen = key.len;
    redo_key = &key; redo_values = values; redo_cap = c;
}

// Streaming consume (chunked H2D overlap, multi-GPU): the table is grown between batches so that it
// can absorb a batch of entirely new keys up to 4x the groups seen so far; an overflow inside a
// batch is reported (pass expected_groups to bl_groupby_create).
void GroupByState::consume(const DevCol& key, const std::vector<const DevCol*>& values, int64_t row_base) {
    PLB_REQUIRE(key.dtype == key_dtype, BL_ERR_DTYPE, "group_by: key dtype differs from the plan");
    PLB_REQUIRE(row_base + key.len <= 0xFFFFFFFEll, BL_ERR_UNSUPPORTED, "group_by: more than 2^32-2 rows (IdxSize = u32)");
    if (!entries) { note_batch_shape(key, values); alloc_table(choose_cap(key, key.len)); }
    else if (expected_groups <= 0) {
        // a later batch can bring more NEW keys than the spare capacity (sorted / time-clustered streams): sample every
        // batch and grow (a rehash keeps the accumulators) until groups so far + the batch's estimate fit at load <= 0.6
        const int64_t g = count_groups();
        (void)choose_cap(key, key.len);                         // refreshes est_groups / the heavy-hitter list for this batch
        const double need = ((double)g + (double)est_groups) / 0.6;
        if ((double)g > 0.25 * (double)cap || need > (double)cap) grow(std::max<uint64_t>(cap * 4, pow2_at_least(need)));
    }
    launch_batch(key, values, row_base);
    if (!defer_status && read_scalar(as<int>(status)) != 0)
        fail(BL_ERR_UNSUPPORTED, "group_by: table overflow inside a streamed batch — create the state with expected_groups set");
    rows_seen += key.len;
}

void GroupByState::reset() {
    if (entries) {
        PLB_LAUNCH("k5_table_init", k_gb_init, grid_for((int64_t)(cap + 2) * L.stride, 256), 256, 0, T.entries, (int64_t)(cap + 2), L.stride, T.soa, T.pw, L);
        dev_memset(status->p, 0, 4);
    }
    rows_seen = 0; merged_rows = 0;
}

void GroupByState::merge_partials(const uint64_t* rows, int64_t n_rows) {
    const uint64_t* ptrs[1] = {rows}; int64_t counts[1] = {n_rows};
    merge_partial_regions(ptrs, counts, 1);
}

// Merge several regions of partial rows (one per source rank) with ONE kernel launch and one sync.
struct MergeRegions { const uint64_t* ptr[EXP_MAX_PARTS]; int64_t end[EXP_MAX_PARTS]; int n; };
__global__ void __launch_bounds__(256) k_gb_merge_regions(const __grid_constant__ GbLayout L, const __grid_constant__ GbTableDev T, const __grid_constant__ MergeRegions R, int row_words) {
    const int64_t total = R.end[R.n - 1];
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        int r = 0; while (i >= R.end[r]) r++;
        const int64_t local = i - (r ? R.end[r - 1] : 0);
        const uint64_t* src = R.ptr[r] + local * row_words;
        gb_merge_row(L, T, src, (int)src[row_words - 1]);
    }
}
void GroupByState::merge_partial_regions(const uint64_t* const* ptrs, const int64_t* counts, int n_regions) {
    PLB_REQUIRE(n_regions >= 1 && n_regions <= EXP_MAX_PARTS, BL_ERR_INVALID, "merge_partials: 1..64 regions");
    const int row_words = L.n_words + 3;
    int64_t n_rows = 0;
    for (int r = 0; r < n_regions; r++) n_rows += counts[r];
    if (!entries) alloc_table(pow2_at_least((double)std::max<int64_t>(std::max<int64_t>(n_rows, expected_groups), 1) / 0.6));
    else if (expected_groups <= 0) {
        int64_t g = count_groups();
        if ((double)(g + n_rows) > 0.6 * (double)cap) grow(pow2_at_least((double)(g + n_rows) / 0.5));
    }
    if (n_rows == 0) return;
    MergeRegions R; memset(&R, 0, sizeof R);
    int64_t acc = 0;
    for (int r = 0; r < n_regions; r++) { R.ptr[r] = ptrs[r]; acc += counts[r]; R.end[r] = acc; }
    R.n = n_regions;
    merged_rows += n_rows;
    PLB_LAUNCH("k5_merge_partials", k_gb_merge_regions, grid_for(n_rows, 256), 256, 0, L, T, R, row_words);
    if (read_scalar(as<int>(status)) != 0) fail(BL_ERR_OOM, "group_by: table overflow while merging partial aggregates (expected_groups too small)");
}

DevPtr GroupByState::export_partials(int n_partitions, int* row_words_out, int64_t* offsets_host) {
    PLB_REQUIRE(n_partitions >= 1 && n_partitions <= EXP_MAX_PARTS, BL_ERR_INVALID, "export_partials: 1..64 partitions");
    const int row_words = L.n_words + 3;
    *row_words_out = row_words;
    if (!entries) { for (int p = 0; p <= n_partitions; p++) offsets_host[p] = 0; return dev_alloc(16); }
    DevPtr counts = dev_alloc(8 * EXP_MAX_PARTS), cursor = dev_alloc(8 * EXP_MAX_PARTS), off = dev_alloc(8 * EXP_MAX_PARTS);
    dev_memset(counts->p, 0, 8 * EXP_MAX_PARTS); dev_memset(cursor->p, 0, 8 * EXP_MAX_PARTS);
    PLB_LAUNCH("k6_export_count", k_gb_export_count, grid_for((int64_t)cap + 2, 256), 256, 0, T.entries, (int64_t)cap, T.es, n_partitions, as<unsigned long long>(counts));
    unsigned long long h[EXP_MAX_PARTS];
    PLB_CUDA(cudaMemcpyAsync(h, counts->p, 8 * n_partitions, cudaMemcpyDeviceToHost, ctx().stream));
    PLB_CUDA(cudaStreamSynchronize(ctx().stream));
    unsigned long long ho[EXP_MAX_PARTS + 1]; ho[0] = 0;
    for (int p = 0; p < n_partitions; p++) ho[p + 1] = ho[p] + h[p];
    for (int p = 0; p <= n_partitions; p++) offsets_host[p] = (int64_t)ho[p];
    PLB_CUDA(cudaMemcpyAsync(off->p, ho, 8 * n_partitions, cudaMemcpyHostToDevice, ctx().stream));
    const int64_t G = (int64_t)ho[n_partitions];
    DevPtr rows = dev_alloc((size_t)std::max<int64_t>(G, 1) * row_words * 8);
    if (G > 0)
        PLB_LAUNCH("k6_export_scatter", k_gb_export_scatter, grid_for((int64_t)cap + 2, 256), 256, 0, T.entries, (int64_t)cap, T.es, T.ws, T.pw, L.n_words, n_partitions,
                   as<unsigned long long>(off), as<unsigned long long>(cursor), as<uint64_t>(rows));
    PLB_CUDA(cudaStreamSynchronize(ctx().stream));   // ho[] is on this stack frame
    return rows;
}

void GroupByState::export_partials_p2p(int n_ranks, int my_rank, void* const* windows, int64_t rows_per_src, int* row_words_out, int64_t* sent_rows) {
    PLB_REQUIRE(n_ranks >= 1 && n_ranks <= EXP_MAX_PARTS && my_rank >= 0 && my_rank < n_ranks, BL_ERR_INVALID, "export_partials_p2p: bad rank / world size");
    const int row_words = L.n_words + 3;
    *row_words_out = row_words;
    for (int p = 0; p < n_ranks; p++) sent_rows[p] = 0;
    if (!entries) return;
    PeerWindows W; memset(&W, 0, sizeof W);
    for (int p = 0; p < n_ranks; p++) { PLB_REQUIRE(windows[p] != nullptr, BL_ERR_INVALID, "export_partials_p2p: null window"); W.base[p] = reinterpret_cast<uint64_t*>(windows[p]); }
    DevPtr cursor = dev_alloc(8 * EXP_MAX_PARTS), ovf = dev_alloc(4);
    dev_memset(cursor->p, 0, 8 * EXP_MAX_PARTS); dev_memset(ovf->p, 0, 4);
    PLB_LAUNCH("k6_export_p2p", k_gb_export_p2p, grid_for((int64_t)cap + 2, 256), 256, 0, T.entries, (int64_t)cap, T.es, T.ws, T.pw, L.n_words, n_ranks, W,
               rows_per_src * row_words, my_rank, rows_per_src, as<unsigned long long>(cursor), as<int>(ovf));
    unsigned long long h[EXP_MAX_PARTS];
    PLB_CUDA(cudaMemcpyAsync(h, cursor->p, 8 * n_ranks, cudaMemcpyDeviceToHost, ctx().stream));
    const int o = read_scalar(as<int>(ovf));      // also completes the kernel and its peer stores
    PLB_REQUIRE(o == 0, BL_ERR_INVALID, "export_partials_p2p: window region too small for the partial aggregates");
    for (int p = 0; p < n_ranks; p++) sent_rows[p] = (int64_t)h[p];
}

void GroupByState::export_partials_p2p_async(int n_ranks, int my_rank, void* const* window_halves, int64_t rows_per_src, uint64_t epoch, int* row_words_out) {
    PLB_REQUIRE(n_ranks >= 1 && n_ranks <= EXP_MAX_PARTS && my_rank >= 0 && my_rank < n_ranks, BL_ERR_INVALID, "export_partials_p2p_async: bad rank / world size");
    PLB_REQUIRE(epoch > 0, BL_ERR_INVALID, "export_partials_p2p_async: epoch must be positive");
    const int row_words = L.n_words + 3;
    *row_words_out = row_words;
    PeerWindows W; memset(&W, 0, sizeof W);
    for (int p = 0; p < n_ranks; p++) { PLB_REQUIRE(window_halves[p] != nullptr, BL_ERR_INVALID, "export_partials_p2p_async: null window"); W.base[p] = reinterpret_cast<uint64_t*>(window_halves[p]); }
    if (!entries) alloc_table(1024);          // nothing consumed: still publish zero counts so that no peer waits
    DevPtr ctl = dev_alloc(8 * EXP_MAX_PARTS + 8);
    dev_memset(ctl->p, 0, 8 * EXP_MAX_PARTS + 8);
    PLB_LAUNCH("k6_export_p2p", k_gb_export_p2p_async, grid_for(((int64_t)cap + 2 + 3) / 4, 256), 256, 0, T.entries, (int64_t)cap, T.es, T.ws, T.pw, L.n_words, n_ranks, W,
               rows_per_src * row_words, my_rank, rows_per_src, as<unsigned long long>(ctl), reinterpret_cast<unsigned*>(as<unsigned long long>(ctl) + EXP_MAX_PARTS), epoch);
}

void GroupByState::merge_window_async(const void* own_half, int n_ranks, int64_t rows_per_src, uint64_t epoch) {
    PLB_REQUIRE(own_half != nullptr && n_ranks >= 1 && n_ranks <= EXP_MAX_PARTS, BL_ERR_INVALID, "merge_window_async: bad arguments");
    const int row_words = L.n_words + 3;
    if (!entries) alloc_table(pow2_at_least((double)std::max<int64_t>(expected_groups, 1024) / 0.6));
    merged_rows += (int64_t)n_ranks * rows_per_src;          // upper bound (sizes the extraction buffers)
    PLB_LAUNCH("k5_merge_partials", k_gb_merge_window, ctx().sm_count * 4, 256, 0, L, T, reinterpret_cast<const uint64_t*>(own_half), n_ranks, rows_per_src, row_words, epoch);
}

void GroupByState::settle() {
    if (redo_key == nullptr || dense.ready) return;
    for (int attempt = 0; attempt < 8; attempt++) {
        if (read_scalar(as<int>(status)) == 0) { redo_key = nullptr; return; }
        redo_cap *= 8;
        alloc_table(redo_cap);
        launch_batch(*redo_key, redo_values, 0);
    }
    fail(BL_ERR_OOM, "group_by: hash table kept overflowing");
}

int GroupByState::read_status() { return status ? read_scalar(as<int>(status)) : 0; }

void GroupByState::finish(bool maintain_order, const DevCol* key_col_for_gather, DevCol& out_key, std::vector<DevCol>& out_aggs, DevCol* out_first) {
    out_aggs.clear();
    PLB_REQUIRE(!maintain_order || L.need_first, BL_ERR_INVALID, "group_by: maintain_order needs a state created with track_first");
    // Extract into buffers sized by an upper bound of the group count, then read the real count and
    // the null-group position back with ONE 16-byte copy (one host sync for the whole finish).
    const int kelem = dtype_size(key_dtype);
    int64_t Gb = 1;
    DevPtr keys, first, len, words, ctl;
    long long ctl_host[2] = {0, -1};
    int status_host = 0;
  for (int attempt = 0;; attempt++) {
    Gb = dense.ready ? dense.Gb : (entries ? std::max<int64_t>(1, std::min<int64_t>((int64_t)cap + 2, rows_seen + merged_rows + 2)) : 1);
    ctl_host[0] = 0; ctl_host[1] = -1; status_host = 0;
    if (dense.ready) {      // the partitioned plan wrote the dense arrays itself
        keys = dense.keys; first = dense.first; len = dense.len; words = dense.words; ctl = dense.ctl;
        PLB_CUDA(cudaMemcpyAsync(ctl_host, ctl->p, 16, cudaMemcpyDeviceToHost, ctx().stream));
    } else {
        keys = dev_alloc((size_t)Gb * 8); first = dev_alloc((size_t)Gb * 4); len = dev_alloc((size_t)Gb * 4);
        words = dev_alloc((size_t)Gb * 8 * std::max(L.n_words, 1));
        ctl = dev_alloc(16);                       // [0] cursor (#groups), [1] null-group position
        const long long ctl_init[2] = {0, -1};
        PLB_CUDA(cudaMemcpyAsync(ctl->p, ctl_init, 16, cudaMemcpyHostToDevice, ctx().stream));
    }
    if (entries && !dense.ready) {
        PLB_CUDA(cudaMemcpyAsync(&status_host, status->p, 4, cudaMemcpyDeviceToHost, ctx().stream));
        PLB_LAUNCH("k5_extract", k_gb_extract, grid_for((int64_t)cap + 2, 256), 256, 0, T.entries, (int64_t)cap, T.es, T.ws, T.pw, L.n_words, as<unsigned long long>(ctl),
                   as<uint64_t>(keys), as<uint32_t>(first), as<uint32_t>(len), as<uint64_t>(words), Gb, as<long long>(ctl) + 1);
        PLB_CUDA(cudaMemcpyAsync(ctl_host, ctl->p, 16, cudaMemcpyDeviceToHost, ctx().stream));
    }
    PLB_CUDA(cudaStreamSynchronize(ctx().stream));
    if (status_host == 1 && redo_key != nullptr && attempt < 8) {      // one-shot batch, table too small: redo into a larger one
        redo_cap *= 8;
        alloc_table(redo_cap);
        launch_batch(*redo_key, redo_values, 0);
        continue;
    }
    break;
  }
    if (status_host == 2) fail(BL_ERR_INVALID, "group_by: a peer window region was too small for the partial aggregates sent to this rank");
    if (status_host == 3) fail(BL_ERR_CUDA, "group_by: timed out waiting for a peer rank's partial aggregates");
    if (status_host != 0) fail(BL_ERR_OOM, "group_by: hash table overflow (deferred check) — create the state with expected_groups set");
    const int64_t G = ctl_host[0];
    const long long null_pos = ctl_host[1];
    // key column + aggregates: one launch (k_gb_finalize_all); more than 16 aggregates take further launches
    out_key = make_col(key_dtype, G, null_pos >= 0);
    out_key.null_count = null_pos >= 0 ? 1 : 0;
    FinalizeAll fall; memset(&fall, 0, sizeof fall);
    fall.key_bits = as<uint64_t>(keys); fall.key_elem = kelem; fall.key_out = out_key.values->p; fall.key_valid = as<uint32_t>(out_key.validity); fall.null_pos = null_pos; fall.G = G;
    bool keys_pending = true;
    auto flush = [&]() {
        if (G > 0 && (fall.n_aggs > 0 || keys_pending)) {
            if (!keys_pending) { fall.key_out = nullptr; fall.key_valid = nullptr; fall.key_elem = 0; }
            PLB_LAUNCH("k5_finalize", k_gb_finalize_all, grid_for(G, 256), 256, 0, fall);
        }
        keys_pending = false; fall.n_aggs = 0;
    };
    for (auto& ap : plans) {
        const bool nullable = ap.kind == BL_AGG_MEAN || ap.kind == BL_AGG_MIN || ap.kind == BL_AGG_MAX;
        DevCol o = make_col(ap.out_dtype, G, nullable);
        FinalizeArgs& fa = fall.agg[fall.n_aggs++];
        memset(&fa, 0, sizeof fa);
        fa.kind = ap.kind; fa.in_dtype = ap.in_dtype; fa.out_dtype = ap.out_dtype; fa.G = G;
        fa.main_word = ap.main >= 0 ? as<uint64_t>(words) + (int64_t)ap.main * Gb : nullptr;
        fa.nullcnt_word = ap.nullcnt >= 0 ? as<uint64_t>(words) + (int64_t)ap.nullcnt * Gb : nullptr;
        fa.len = as<uint32_t>(len); fa.out = o.values->p; fa.out_valid = as<uint32_t>(o.validity);
        out_aggs.push_back(o);
        if (fall.n_aggs == GB_FIN_MAX) flush();
    }
    flush();
    // float keys (and any key when the column is at hand): output = key at the group's first row
    // (group_by/mod.rs:258-266) so that -0.0 / NaN payloads of the first occurrence survive
    const bool gather_keys = key_col_for_gather != nullptr && dtype_is_float(key_dtype) && G > 0 && L.need_first;
    DevCol first_col; first_col.dtype = BL_UINT32; first_col.len = G; first_col.values = first; first_col.null_count = 0;
    if (gather_keys) {
        std::vector<DevCol> in{*key_col_for_gather}, outv;
        op_gather(in, first_col, false, outv);
        out_key = outv[0];
        if (!out_key.validity && null_pos >= 0) { /* unreachable: nullable key col gathers validity */ }
    }
    if (maintain_order && G > 1) {
        // sort groups by first row idx (hashing.rs:41-63) and permute every output column
        DevPtr perm = dev_alloc((size_t)G * 4), fkeys = dev_alloc((size_t)G * 4);
        PLB_CUDA(cudaMemcpyAsync(fkeys->p, first->p, (size_t)G * 4, cudaMemcpyDeviceToDevice, ctx().stream));
        iota_u32(as<uint32_t>(perm), G, 0);
        sort_pairs_u32(as<uint32_t>(fkeys), as<uint32_t>(perm), G);      // first-row ids carry the caller's row_base: all 32 bits
        DevCol pidx; pidx.dtype = BL_UINT32; pidx.len = G; pidx.values = perm; pidx.null_count = 0;
        std::vector<DevCol> in{out_key}, outv;
        for (auto& a : out_aggs) in.push_back(a);
        if (out_first) in.push_back(first_col);
        op_gather(in, pidx, false, outv);
        out_key = outv[0];
        for (size_t i = 0; i < out_aggs.size(); i++) out_aggs[i] = outv[i + 1];
        if (out_first) first_col = outv.back();
    }
    if (out_first) *out_first = first_col;
}

// ---------------------------------------------------------------------------- group tuples (GroupsIdx)
// The reference's group_by materialises GroupsIdx{first, all} (position.rs:16-22) in
// group_by_threaded_slice (hashing.rs:116-167); finish_group_order (hashing.rs:41-63) orders the groups
// by first row.  The fused aggregation path above never needs the index lists; this entry point builds
// them for callers that do (aggregations outside the fused set evaluate per group over `all`):
//   1. K5 with no accumulators: table of (key, len, first row)
//   2. row -> first row of its group (a lookup; the first row is the group's identity)
//   3. stable radix sort of (first-of-group, row): groups in first-occurrence order, rows ascending
//   4. run starts of the sorted keys -> offsets, first = all[offsets]
__global__ void __launch_bounds__(256) k_gb_lookup_first(const __grid_constant__ GbTableDev T, const void* keys, const uint32_t* key_validity, int key_dtype, int64_t n, uint32_t* __restrict__ out) {
    const uint64_t mask = T.cap - 1;
    for (int64_t row = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; row < n; row += (int64_t)gridDim.x * blockDim.x) {
        const bool kvalid = key_validity == nullptr || bit_get(key_validity, row);
        const uint64_t key = load_key_rt(keys, key_dtype, row);
        uint64_t slot;
        if (!kvalid) slot = T.cap;
        else if (key == GB_EMPTY) slot = T.cap + 1;
        else {
            slot = table_hash(key) >> T.shift;
            for (int probes = 0; probes < GB_MAX_PROBE; ++probes) {
                if (__ldcg(reinterpret_cast<const unsigned long long*>(T.entries + slot * T.es)) == key) break;
                slot = (slot + 1) & mask;
            }
        }
        const uint64_t w1 = __ldcg(reinterpret_cast<const unsigned long long*>(T.entries + slot * T.es + gb_woff((int64_t)slot, 1, T.ws, T.pw)));
        out[row] = (uint32_t)(w1 >> 32);
    }
}
// bit i of the mask = sorted[i] starts a run (i == 0 or sorted[i] != sorted[i-1]); n_round = n rounded up to 32
__global__ void __launch_bounds__(256) k_run_starts(const uint32_t* __restrict__ sorted, int64_t n, int64_t n_round, uint32_t* __restrict__ mask_words) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_round; i += (int64_t)gridDim.x * blockDim.x) {
        const bool start = i < n && (i == 0 || sorted[i] != sorted[i - 1]);
        const unsigned b = __ballot_sync(0xffffffffu, start);
        if ((threadIdx.x & 31) == 0) mask_words[i >> 5] = b;
    }
}

// row -> first row index of the row's group (u32): a group id that needs no renumbering
DevCol op_group_first_ids(const DevCol& key) {
    const int64_t n = key.len;
    DevCol ids = make_col(BL_UINT32, n, false);
    if (n == 0) return ids;
    GroupByState st(key.dtype, {}, {}, {}, 0, true);
    st.consume_all(key, {});
    st.settle();
    PLB_LAUNCH("k5_lookup_first", k_gb_lookup_first, grid_for(n, 256, 16), 256, 0, st.T, key.v(), key.vm(), key.dtype, n, as<uint32_t>(ids.values));
    return ids;
}

// ---------------------------------------------------------------------------- multi-column keys
// The reference row-encodes several key columns into one binary key (group_by/mod.rs:88-94,
// polars-row/src/fixed/numeric.rs:100-145: floats canonicalised, one validity sentinel per column) and groups
// on that.  Fixed-width columns pack into ONE 64-bit key instead: each column contributes its (canonical) bit
// pattern plus a validity bit when it can hold nulls; when the next column does not fit, the key so far is
// replaced by its 32-bit group id (first row of its group: one K5 build + lookup), so any number of columns
// of any hot-path dtype works and narrow keys (Q1's two flag bytes, two Int32s) need no extra pass at all.
__global__ void __launch_bounds__(256) k_pack_append(const uint64_t* __restrict__ acc, int shift, const void* __restrict__ values, const uint32_t* __restrict__ validity, int dtype, int vbits,
                                                     int64_t n, uint64_t* __restrict__ out) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        uint64_t rep = 0;
        const bool valid = validity == nullptr || bit_get(validity, i);
        if (valid) {
            switch (dtype) {
                case BL_INT8: case BL_UINT8: rep = reinterpret_cast<const uint8_t*>(values)[i]; break;
                case BL_INT16: case BL_UINT16: rep = reinterpret_cast<const uint16_t*>(values)[i]; break;
                default: rep = load_key_rt(values, dtype, i); break;      // canonical float bits / zero-extended 32-bit pattern / 64-bit pattern
            }
            if (validity != nullptr) rep |= 1ull << vbits;                 // validity bit above the value bits (never reached for 64-bit values: those are id-compressed first)
        }
        out[i] = (acc ? acc[i] : 0ull) | (rep << shift);
    }
}

// Packs the key columns into one BL_UINT64 key column (no validity: nulls are part of the packed value).
DevCol op_pack_keys(const std::vector<DevCol>& keys) {
    PLB_REQUIRE(!keys.empty(), BL_ERR_INVALID, "group_by: no key columns");
    const int64_t n = keys[0].len;
    DevCol acc; bool have = false; int used = 0;
    for (const DevCol& k0 : keys) {
        PLB_REQUIRE(k0.len == n, BL_ERR_INVALID, "group_by: key columns differ in length");
        PLB_REQUIRE(k0.dtype != BL_BOOL, BL_ERR_UNSUPPORTED, "group_by: Boolean keys are outside the hot path");
        DevCol k = k0;
        int vbits = dtype_size(k.dtype) * 8;
        int w = vbits + (k.validity ? 1 : 0);
        if (w > 64 || (w > 32 && have && used + w > 64)) {      // wide column that cannot sit beside the rest: use its group id
            k = op_group_first_ids(k); vbits = 32; w = 32;
        }
        if (have && used + w > 64) {                              // key so far -> its 32-bit group id
            DevCol ids = op_group_first_ids(acc);
            DevCol wide = make_col(BL_UINT64, n, false);
            if (n) PLB_LAUNCH("k5_pack_keys", k_pack_append, grid_for(n, 256, 16), 256, 0, (const uint64_t*)nullptr, 0, ids.v(), ids.vm(), BL_UINT32, 32, n, as<uint64_t>(wide.values));
            acc = wide; used = 32;
        }
        DevCol out = make_col(BL_UINT64, n, false);
        if (n) PLB_LAUNCH("k5_pack_keys", k_pack_append, grid_for(n, 256, 16), 256, 0, have ? as<uint64_t>(acc.values) : (const uint64_t*)nullptr, used, k.v(), k.vm(), k.dtype, vbits, n, as<uint64_t>(out.values));
        acc = out; have = true; used += w;
    }
    return acc;
}

void op_group_tuples(const DevCol& key, DevCol& out_first, DevCol& out_offsets, DevCol& out_all) {
    const int64_t n = key.len;
    PLB_REQUIRE(n <= 0x7FFFFFFFll, BL_ERR_UNSUPPORTED, "group_tuples: more than 2^31-1 rows");
    out_all = make_col(BL_UINT32, n, false);
    if (n == 0) {
        out_first = make_col(BL_UINT32, 0, false);
        out_offsets = make_col(BL_UINT32, 1, false);
        dev_memset(out_offsets.values->p, 0, 4);
        return;
    }
    DevCol ids = op_group_first_ids(key);
    DevPtr gid = ids.values;
    iota_u32(as<uint32_t>(out_all.values), n, 0);
    sort_pairs_u32(as<uint32_t>(gid), as<uint32_t>(out_all.values), n, bits_for((uint64_t)n));
    DevCol starts = make_col(BL_BOOL, n, false);
    const int64_t n_round = (n + 31) / 32 * 32;
    PLB_LAUNCH("k5_run_starts", k_run_starts, grid_for(n_round, 256, 16), 256, 0, as<uint32_t>(gid), n, n_round, as<uint32_t>(starts.values));
    DevCol pos = make_col(BL_UINT32, n, false);
    iota_u32(as<uint32_t>(pos.values), n, 0);
    std::vector<DevCol> in{pos, out_all}, outv;
    op_filter(in, starts, outv);
    const int64_t G = outv[0].len;
    out_first = outv[1];
    out_offsets = make_col(BL_UINT32, G + 1, false);
    PLB_CUDA(cudaMemcpyAsync(out_offsets.values->p, outv[0].values->p, (size_t)G * 4, cudaMemcpyDeviceToDevice, ctx().stream));
    const uint32_t n32 = (uint32_t)n;
    PLB_CUDA(cudaMemcpyAsync((char*)out_offsets.values->p + (size_t)G * 4, &n32, 4, cudaMemcpyHostToDevice, ctx().stream));
    PLB_CUDA(cudaStreamSynchronize(ctx().stream));      // n32 lives on this frame
}

}  // namespace plb
