// join.cu — K7 (hash-join build) and K8 (probe + deterministic tuple emission).
//
// Reference path being replaced (paths relative to /root/reference/crates):
//   build_tables            polars-ops/src/frame/join/hash_join/single_keys.rs:16-167
//   probe_inner / hash_join_tuples_inner   .../single_keys_inner.rs:11-149
//   hash_join_tuples_left   .../single_keys_left.rs:106-195
//   semi / anti             .../single_keys_semi_anti.rs:8-140
//   which side builds       .../hash_join/mod.rs:41-50 (probe = longer relation, tie -> right probes)
//   maintain_order sort     polars-ops/src/frame/join/mod.rs:577-642
// The reference radix-partitions the build side over threads and keeps a hashbrown map
// key -> ascending row-index vector per partition; probing walks the probe side in row order and
// emits (probe idx, build idx) for every build idx in ascending order.
//
// H100 design.  Three table forms, chosen per build relation:
//   DENSE    build keys are integers whose value range is a few times the row count (surrogate / primary keys):
//            u32 table[key - min] = build row.  4 B per key value, L2-resident for 1e7 keys.
//   WIDE     (default hashed form) 32-byte buckets of two {key, val, cnt} entries (half full), bucket = mulhi(key *
//            RANDOM_ODD, buckets) — the reference's own hash_to_partition.  One sector (two 128-bit loads) per probe step
//            carries everything (both keys, build row or CSR offset, match count).
//   COMPACT  (BL_JOIN_TABLE=compact) u32 table[slot] = fingerprint:8 | build row:24 (plain row ids past 2^24 rows),
//            slot = top bits of key * RANDOM_ODD, capacity = the power of two >= 1.5x the build rows.  The table never
//            stores the key: a fingerprint match is verified against the build key column itself.  4 B per slot
//            (1e7 keys: 64 MB, L2-resident) instead of 16 B, so a probe is one L2 hit plus one 8-byte read of the build
//            column; a miss usually costs the L2 hit only (slower than WIDE when most probes hit: two dependent accesses).
//   build:   claim the key's slot with one CAS; duplicates are detected by the claim that loses.  Unique build keys
//            (the primary-key case) need nothing else.  With duplicates: per-slot counts -> exclusive scan -> CSR
//            offsets; the rows of a slot are listed ascending (stable sort of the rows by slot) — the reference's IdxVec.
//   probe:   unique build keys: ONE fused pass — lookup + decoupled look-back scan over 2048-row tiles + coalesced
//            tuple stores.  Duplicates: pass 1 stores (list offset, match count) per probe row and per-tile match counts; a scan
//            gives every tile its output offset; pass 2 expands the handles warp-cooperatively (every 32 consecutive
//            output tuples are written by the 32 lanes of one warp, whatever the run lengths).
//   semi / anti: probe-only — one hit bit per left row, then K3 over iota(left): O(left + right), never the
//            duplicate expansion.
// Algorithmic bytes (SURVEY.md §8(d)): build 8 B read + 4..16 B table write per build row; probe 8 B key read + 8 B
// tuple write per match.  Bound: random L2 / HBM sector reads of the table (and of the build column for COMPACT).
#include <cstdlib>
#include <cstring>

#include "common.cuh"
#include "dev_utils.cuh"

namespace plb {

constexpr uint64_t J_EMPTY = 0x8000000000000000ULL;
constexpr uint32_t J_NONE = 0xFFFFFFFFu;
constexpr int J_TILE = 2048;
enum { JM_WIDE = 0, JM_DENSE = 1, JM_COMPACT = 2 };

// WIDE: 32-byte buckets of two entries — one sector per probe step.  Logical slot id = 2 * bucket + j.
// buckets[nb] is the special bucket: entry 0 = null-key group, entry 1 = J_EMPTY-key group (their key word is only a "used" marker).
struct JoinBucket { unsigned long long key[2]; uint32_t val[2]; uint32_t cnt[2]; };
static_assert(sizeof(JoinBucket) == 32, "bucket = one 32-byte sector");
struct JoinTableDev { JoinBucket* buckets; uint64_t nb; };
__device__ __forceinline__ void j_load_bucket(const JoinBucket* b, unsigned long long& k0, unsigned long long& k1, unsigned long long& v, unsigned long long& c) {
    // sm_90 has no 256-bit load: two independent 128-bit loads (LDG.E.128) of the same 32-byte sector, issued back to back
    asm volatile("ld.global.nc.v2.u64 {%0,%1}, [%4];\n\t"
                 "ld.global.nc.v2.u64 {%2,%3}, [%4+16];" : "=l"(k0), "=l"(k1), "=l"(v), "=l"(c) : "l"(b));
}

// Everything a probe needs, for any table form (unused members stay zero).
struct JoinDev {
    JoinTableDev W;                                         // WIDE
    const uint32_t* dense; uint64_t kmin, range; int sign_bits;   // DENSE
    const uint32_t* tab; uint32_t cmask; int cshift; int fp_mode; uint32_t ccap;   // COMPACT: tab[ccap] = a null-key build row or J_NONE
    const void* bkeys; const uint32_t* ccnt; const uint32_t* coff;
    int nulls_equal, csr;
};

__device__ __forceinline__ uint64_t j_load_key(const void* keys, int dtype, int64_t row) {
    switch (dtype) {
        case BL_INT64: case BL_UINT64: return reinterpret_cast<const uint64_t*>(keys)[row];
        case BL_FLOAT64: return canonical_f64_bits(reinterpret_cast<const double*>(keys)[row]);   // NaN joins NaN (single_keys_dispatch.rs:316-322)
        case BL_FLOAT32: return canonical_f32_bits(reinterpret_cast<const float*>(keys)[row]);
        default: return (uint64_t)reinterpret_cast<const uint32_t*>(keys)[row];
    }
}
template <int KEY_CANON> __device__ __forceinline__ uint64_t j_canon(uint64_t raw) {
    if (KEY_CANON == 1) return canonical_f64_bits(__longlong_as_double((long long)raw));
    if (KEY_CANON == 2) return canonical_f32_bits(__uint_as_float((uint32_t)raw));
    return raw;
}
template <int KEY_ELEM, int KEY_CANON> __device__ __forceinline__ uint64_t j_bkey(const void* bkeys, uint32_t row) {
    const uint64_t raw = KEY_ELEM == 8 ? __ldg(reinterpret_cast<const unsigned long long*>(bkeys) + row) : (uint64_t)__ldg(reinterpret_cast<const unsigned int*>(bkeys) + row);
    return j_canon<KEY_CANON>(raw);
}
__device__ __forceinline__ uint64_t j_ordered(uint64_t raw, int sign_bits) {
    // order-preserving map to u64: signed types flip the sign bit (32-bit patterns are sign-extended first)
    if (sign_bits == 64) return raw ^ 0x8000000000000000ULL;
    if (sign_bits == 32) return (uint64_t)(int64_t)(int32_t)(uint32_t)raw ^ 0x8000000000000000ULL;
    return raw;
}

__global__ void k_join_init(JoinBucket* buckets, int64_t n) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        uint4* q = reinterpret_cast<uint4*>(buckets + i);
        q[0] = make_uint4((uint32_t)J_EMPTY, (uint32_t)(J_EMPTY >> 32), (uint32_t)J_EMPTY, (uint32_t)(J_EMPTY >> 32));
        q[1] = make_uint4(J_NONE, J_NONE, 0u, 0u);
    }
}
__global__ void k_fill_u32j(uint32_t* p, uint32_t v, int64_t n) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) p[i] = v;
}

// ---------------------------------------------------------------------------- K7 build: WIDE
// A key lives in the first bucket of its probe sequence that had a free entry when it arrived (entries are never
// removed), so a lookup may stop at the first bucket that still has a free entry.
__global__ void __launch_bounds__(256) k_join_build(JoinTableDev T, const void* __restrict__ keys, const uint32_t* __restrict__ valid, int key_dtype, int64_t n,
                                                    int nulls_equal, uint32_t* __restrict__ slot_of_row, int* __restrict__ has_dups) {
    for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < n; r += (int64_t)gridDim.x * blockDim.x) {
        const bool v = valid == nullptr || bit_get(valid, r);
        uint64_t b; int j;
        if (!v) {
            if (!nulls_equal) { slot_of_row[r] = J_NONE; continue; }     // null keys are not inserted (single_keys.rs:41,148)
            b = T.nb; j = 0;
            atomicCAS(&T.buckets[b].key[0], (unsigned long long)J_EMPTY, 0ull);
        } else {
            const uint64_t key = j_load_key(keys, key_dtype, r);
            if (key == J_EMPTY) { b = T.nb; j = 1; atomicCAS(&T.buckets[b].key[1], (unsigned long long)J_EMPTY, 1ull); }
            else {
                b = __umul64hi(table_hash(key), T.nb);
                j = 0;
                while (true) {
                    bool found = false;
#pragma unroll
                    for (int jj = 0; jj < 2; jj++) {
                        if (found) continue;
                        unsigned long long* kp = &T.buckets[b].key[jj];
                        unsigned long long k = __ldcg(kp);
                        if (k == J_EMPTY) k = atomicCAS(kp, (unsigned long long)J_EMPTY, (unsigned long long)key);
                        if (k == key || k == J_EMPTY) { found = true; j = jj; }
                    }
                    if (found) break;
                    if (++b == T.nb) b = 0;
                }
            }
        }
        const uint32_t old = atomicAdd(&T.buckets[b].cnt[j], 1u);
        atomicMin(&T.buckets[b].val[j], (uint32_t)r);
        if (old != 0) *has_dups = 1;
        slot_of_row[r] = (uint32_t)(2 * b + j);
    }
}
// WIDE duplicates: val <- CSR offset (exclusive scan of cnt over the logical slots, in slot order).  The table is walked as
// an array of u32 words: slot s -> cnt at word (s >> 1) * 8 + 6 + (s & 1), val at word (s >> 1) * 8 + 4 + (s & 1).
__device__ __forceinline__ int64_t j_cnt_word(int64_t s) { return (s >> 1) * 8 + 6 + (s & 1); }
__global__ void __launch_bounds__(256) k_join_tile_sums(const uint32_t* __restrict__ words, int64_t n, uint32_t* __restrict__ sums) {
    __shared__ uint32_t ws[8];
    const int64_t ntiles = (n + J_TILE - 1) / J_TILE;
    for (int64_t t = blockIdx.x; t < ntiles; t += gridDim.x) {
        uint32_t c = 0;
        for (int k = 0; k < J_TILE / 256; k++) { int64_t i = t * J_TILE + k * 256 + threadIdx.x; if (i < n) c += words[j_cnt_word(i)]; }
        for (int o = 16; o; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
        if (lane_id() == 0) ws[threadIdx.x >> 5] = c;
        __syncthreads();
        if (threadIdx.x == 0) { uint32_t s = 0; for (int w = 0; w < 8; w++) s += ws[w]; sums[t] = s; }
        __syncthreads();
    }
}
__global__ void __launch_bounds__(256) k_join_csr_offsets(uint32_t* __restrict__ words, int64_t n, const uint64_t* __restrict__ tile_off) {
    __shared__ uint32_t ws[8];
    __shared__ uint32_t carry;
    const int64_t ntiles = (n + J_TILE - 1) / J_TILE;
    for (int64_t t = blockIdx.x; t < ntiles; t += gridDim.x) {
        if (threadIdx.x == 0) carry = (uint32_t)tile_off[t];
        __syncthreads();
        for (int k = 0; k < J_TILE / 256; k++) {
            const int64_t i = t * J_TILE + k * 256 + threadIdx.x;
            const uint32_t c = i < n ? words[j_cnt_word(i)] : 0;
            uint32_t x = c;
            for (int o = 1; o < 32; o <<= 1) { uint32_t y = __shfl_up_sync(0xffffffffu, x, o); if (lane_id() >= (unsigned)o) x += y; }
            if (lane_id() == 31) ws[threadIdx.x >> 5] = x;
            __syncthreads();
            uint32_t wbase = 0;
            for (unsigned w = 0; w < (threadIdx.x >> 5); w++) wbase += ws[w];
            if (i < n) words[j_cnt_word(i) - 2] = carry + wbase + x - c;      // the slot's val word
            __syncthreads();
            if (threadIdx.x == 255) carry += wbase + x;
            __syncthreads();
        }
    }
}

// ---------------------------------------------------------------------------- K7 build: COMPACT
// One CAS per build row claims the first free slot of the key's probe sequence with (fingerprint | row).  Two rows
// with the same key walk the same sequence, so the second one always meets the first one's entry: that is the
// duplicate test (and the row -> slot map the CSR lists are built from).
template <int KEY_ELEM, int KEY_CANON>
__global__ void __launch_bounds__(256) k_jc_build(uint32_t* __restrict__ tab, uint32_t mask, int shift, int fp_mode, uint32_t cap, const void* __restrict__ keys,
                                                  const uint32_t* __restrict__ valid, int64_t n, int nulls_equal, uint32_t* __restrict__ slot_of_row, int* __restrict__ has_dups) {
    for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < n; r += (int64_t)gridDim.x * blockDim.x) {
        const bool v = valid == nullptr || bit_get(valid, r);
        if (!v) {
            if (!nulls_equal) { slot_of_row[r] = J_NONE; continue; }     // null keys are not inserted (single_keys.rs:41,148)
            if (atomicCAS(&tab[cap], J_NONE, (uint32_t)r) != J_NONE) *has_dups = 1;
            slot_of_row[r] = cap;
            continue;
        }
        const uint64_t key = j_bkey<KEY_ELEM, KEY_CANON>(keys, (uint32_t)r);
        const uint64_t h = table_hash(key);
        uint32_t slot = (uint32_t)(h >> shift);
        const uint32_t fp = (uint32_t)(h >> (shift - 8)) & 0xFFu;
        const uint32_t mine = fp_mode ? ((fp << 24) | (uint32_t)r) : (uint32_t)r;
        while (true) {
            uint32_t e = __ldcg(tab + slot);
            if (e == J_NONE) { e = atomicCAS(&tab[slot], J_NONE, mine); if (e == J_NONE) break; }
            const uint32_t row = fp_mode ? (e & 0xFFFFFFu) : e;
            if ((!fp_mode || (e >> 24) == fp) && j_bkey<KEY_ELEM, KEY_CANON>(keys, row) == key) { *has_dups = 1; break; }
            slot = (slot + 1) & mask;
        }
        slot_of_row[r] = slot;
    }
}
__global__ void __launch_bounds__(256) k_jc_count(const uint32_t* __restrict__ slot_of_row, int64_t n, uint32_t* __restrict__ cnt) {
    for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < n; r += (int64_t)gridDim.x * blockDim.x) {
        const uint32_t s = slot_of_row[r];
        if (s != J_NONE) atomicAdd(&cnt[s], 1u);
    }
}
__global__ void __launch_bounds__(256) k_jc_tile_sums(const uint32_t* __restrict__ cnt, int64_t n, uint32_t* __restrict__ sums) {
    __shared__ uint32_t ws[8];
    const int64_t ntiles = (n + J_TILE - 1) / J_TILE;
    for (int64_t t = blockIdx.x; t < ntiles; t += gridDim.x) {
        uint32_t c = 0;
        for (int k = 0; k < J_TILE / 256; k++) { int64_t i = t * J_TILE + k * 256 + threadIdx.x; if (i < n) c += cnt[i]; }
        for (int o = 16; o; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
        if (lane_id() == 0) ws[threadIdx.x >> 5] = c;
        __syncthreads();
        if (threadIdx.x == 0) { uint32_t s = 0; for (int w = 0; w < 8; w++) s += ws[w]; sums[t] = s; }
        __syncthreads();
    }
}
__global__ void __launch_bounds__(256) k_jc_offsets(const uint32_t* __restrict__ cnt, int64_t n, const uint64_t* __restrict__ tile_off, uint32_t* __restrict__ off) {
    __shared__ uint32_t ws[8];
    __shared__ uint32_t carry;
    const int64_t ntiles = (n + J_TILE - 1) / J_TILE;
    for (int64_t t = blockIdx.x; t < ntiles; t += gridDim.x) {
        if (threadIdx.x == 0) carry = (uint32_t)tile_off[t];
        __syncthreads();
        for (int k = 0; k < J_TILE / 256; k++) {
            const int64_t i = t * J_TILE + k * 256 + threadIdx.x;
            const uint32_t c = i < n ? cnt[i] : 0;
            uint32_t x = c;
            for (int o = 1; o < 32; o <<= 1) { uint32_t y = __shfl_up_sync(0xffffffffu, x, o); if (lane_id() >= (unsigned)o) x += y; }
            if (lane_id() == 31) ws[threadIdx.x >> 5] = x;
            __syncthreads();
            uint32_t wbase = 0;
            for (unsigned w = 0; w < (threadIdx.x >> 5); w++) wbase += ws[w];
            if (i < n) off[i] = carry + wbase + x - c;
            __syncthreads();
            if (threadIdx.x == 255) carry += wbase + x;
            __syncthreads();
        }
    }
}

// ---------------------------------------------------------------------------- K7 build: DENSE
__global__ void k_join_minmax(const void* __restrict__ keys, const uint32_t* __restrict__ valid, int elem, int sign_bits, int64_t n, unsigned long long* mm) {
    unsigned long long lo = ~0ull, hi = 0ull;
    for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < n; r += (int64_t)gridDim.x * blockDim.x) {
        if (valid != nullptr && !bit_get(valid, r)) continue;
        uint64_t raw = elem == 8 ? reinterpret_cast<const uint64_t*>(keys)[r] : (uint64_t)reinterpret_cast<const uint32_t*>(keys)[r];
        unsigned long long k = j_ordered(raw, sign_bits);
        lo = k < lo ? k : lo; hi = k > hi ? k : hi;
    }
    for (int o = 16; o; o >>= 1) {
        unsigned long long a = __shfl_xor_sync(0xffffffffu, lo, o), b = __shfl_xor_sync(0xffffffffu, hi, o);
        lo = a < lo ? a : lo; hi = b > hi ? b : hi;
    }
    if (lane_id() == 0) { atomicMin(&mm[0], lo); atomicMax(&mm[1], hi); }
}
__global__ void __launch_bounds__(256) k_join_dense_build(uint32_t* __restrict__ table, const void* __restrict__ keys, const uint32_t* __restrict__ valid, int elem, int sign_bits,
                                                          int64_t n, uint64_t kmin, int* __restrict__ has_dups) {
    for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < n; r += (int64_t)gridDim.x * blockDim.x) {
        if (valid != nullptr && !bit_get(valid, r)) continue;
        uint64_t raw = elem == 8 ? reinterpret_cast<const uint64_t*>(keys)[r] : (uint64_t)reinterpret_cast<const uint32_t*>(keys)[r];
        const uint32_t old = atomicMin(&table[j_ordered(raw, sign_bits) - kmin], (uint32_t)r);
        if (old != J_NONE) *has_dups = 1;
    }
}

// ---------------------------------------------------------------------------- lookup (any table form)
// Returns the match handle of one probe key — unique mode: the build row; CSR mode: the offset of the key's ascending
// row list in sorted_rows — or J_NONE; cnt = number of matches.  `kraw` is the raw (not yet canonical) key pattern.
template <int MODE, int KEY_ELEM, int KEY_CANON>
__device__ __forceinline__ uint32_t j_lookup(const JoinDev& J, uint64_t kraw, bool valid, uint32_t& cnt) {
    cnt = 0;
    if (MODE == JM_DENSE) {
        const uint64_t d = j_ordered(kraw, J.sign_bits) - J.kmin;
        uint32_t h = J_NONE;
        if (valid && d < J.range) h = __ldg(&J.dense[d]);
        cnt = h != J_NONE ? 1u : 0u;
        return h;
    }
    const uint64_t key = j_canon<KEY_CANON>(kraw);
    if (MODE == JM_WIDE) {
        unsigned long long k0, k1, vv, cc;
        int j;
        if (!valid || key == J_EMPTY) {
            if (!valid && !J.nulls_equal) return J_NONE;
            j_load_bucket(J.W.buckets + J.W.nb, k0, k1, vv, cc);
            j = valid ? 1 : 0;
            if (((uint32_t)(cc >> (32 * j))) == 0) return J_NONE;
        } else {
            uint64_t b = __umul64hi(table_hash(key), J.W.nb);
            while (true) {
                j_load_bucket(J.W.buckets + b, k0, k1, vv, cc);
                if (k0 == key) { j = 0; break; }
                if (k1 == key) { j = 1; break; }
                if (k0 == J_EMPTY || k1 == J_EMPTY) return J_NONE;
                if (++b == J.W.nb) b = 0;
            }
        }
        cnt = J.csr ? (uint32_t)(cc >> (32 * j)) : 1u;
        return (uint32_t)(vv >> (32 * j));            // unique: the build row; CSR: the list offset (k_join_csr_offsets)
    }
    // COMPACT
    uint32_t slot, row;
    if (!valid) {
        if (!J.nulls_equal) return J_NONE;
        slot = J.ccap; row = __ldg(J.tab + slot);
        if (row == J_NONE) return J_NONE;
    } else {
        const uint64_t h = table_hash(key);
        slot = (uint32_t)(h >> J.cshift);
        const uint32_t fp = (uint32_t)(h >> (J.cshift - 8)) & 0xFFu;
        while (true) {
            const uint32_t e = __ldg(J.tab + slot);
            if (e == J_NONE) return J_NONE;
            row = J.fp_mode ? (e & 0xFFFFFFu) : e;
            if ((!J.fp_mode || (e >> 24) == fp) && j_bkey<KEY_ELEM, KEY_CANON>(J.bkeys, row) == key) break;
            slot = (slot + 1) & J.cmask;
        }
    }
    cnt = J.csr ? __ldg(J.ccnt + slot) : 1u;
    return J.csr ? __ldg(J.coff + slot) : row;
}

// ---------------------------------------------------------------------------- K8 probe, pass 1 (two-pass form)
// handle[i] = unique mode: build row; CSR mode: offset of the row list, hcnt[i] = its length (J_NONE on miss) — pass 2
// never goes back to the table (round 1 re-read the entry of every probe row there: a random HBM sector per row).
template <int MODE, int KEY_ELEM, int KEY_CANON>
__global__ void __launch_bounds__(256) k_join_probe(const __grid_constant__ JoinDev J, const void* __restrict__ keys, const uint32_t* __restrict__ valid, int64_t n, int left_join,
                                                    uint32_t* __restrict__ handle, uint32_t* __restrict__ hcnt, unsigned long long* __restrict__ tile_counts) {
    const int64_t npairs = (n + 1) >> 1;
    const int64_t rounded = (npairs + 31) / 32 * 32;
    for (int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; p < rounded; p += (int64_t)gridDim.x * blockDim.x) {
        const int64_t r0 = 2 * p;
        uint64_t kraw[2] = {0, 0};
        if (r0 + 1 < n) {
            if (KEY_ELEM == 8) { ulonglong2 t = ld_stream_u64x2(reinterpret_cast<const uint64_t*>(keys) + r0); kraw[0] = t.x; kraw[1] = t.y; }
            else { uint2 t = ld_stream_u32x2(reinterpret_cast<const uint32_t*>(keys) + r0); kraw[0] = t.x; kraw[1] = t.y; }
        } else if (r0 < n) kraw[0] = KEY_ELEM == 8 ? reinterpret_cast<const uint64_t*>(keys)[r0] : (uint64_t)reinterpret_cast<const uint32_t*>(keys)[r0];
        uint32_t h[2] = {J_NONE, J_NONE}, hc[2] = {0, 0};
        uint32_t cnt = 0;
#pragma unroll
        for (int j = 0; j < 2; j++) {
            const int64_t row = r0 + j;
            if (row >= n) continue;
            const bool v = valid == nullptr || bit_get(valid, row);
            h[j] = j_lookup<MODE, KEY_ELEM, KEY_CANON>(J, kraw[j], v, hc[j]);
            cnt += h[j] != J_NONE ? hc[j] : (left_join ? 1u : 0u);
        }
        if (r0 + 1 < n) { *reinterpret_cast<uint2*>(handle + r0) = make_uint2(h[0], h[1]); if (J.csr) *reinterpret_cast<uint2*>(hcnt + r0) = make_uint2(hc[0], hc[1]); }
        else if (r0 < n) { handle[r0] = h[0]; if (J.csr) hcnt[r0] = hc[0]; }
        // 32 lanes x 2 rows = 64 consecutive rows: always inside one J_TILE
        unsigned long long c = cnt;
        for (int o = 16; o; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
        if (lane_id() == 0 && c) atomicAdd(&tile_counts[r0 / J_TILE], c);   // one address per 2048-row tile; the grand total comes from the scan
    }
}

// ---------------------------------------------------------------------------- K8 probe, pass 2 (emit)
// Rows are mapped lane-strided (row = tile + j*256 + tid): the handles load coalesced, and the tuples of every
// (iteration, warp) segment are written WARP-COOPERATIVELY: output element q of the segment belongs to the lane
// whose exclusive prefix is the last one <= q (5-step search over the lanes' prefixes by shuffles), so 32
// consecutive tuples are always stored by the 32 lanes of the warp — coalesced for any mix of run lengths
// (round 1 wrote every run with its own thread: 1 TB/s for 4 matches per probe row).
struct JoinEmitDev { const uint32_t* hcnt; const uint32_t* sorted_rows; int csr; };
__global__ void __launch_bounds__(256) k_join_emit(const __grid_constant__ JoinEmitDev E, const uint32_t* __restrict__ handle, int64_t n, int left_join,
                                                   const uint64_t* __restrict__ tile_off, uint32_t* __restrict__ out_probe, uint32_t* __restrict__ out_build) {
    constexpr int ITERS = J_TILE / 256;           // 8
    __shared__ uint32_t seg[ITERS * 8];           // segment = j * 8 + warp, in row order
    const unsigned lane = lane_id(), warp = threadIdx.x >> 5;
    const int64_t ntiles = (n + J_TILE - 1) / J_TILE;
    for (int64_t t = blockIdx.x; t < ntiles; t += gridDim.x) {
        uint32_t h[ITERS], c[ITERS], off[ITERS], lane_excl[ITERS];
#pragma unroll
        for (int j = 0; j < ITERS; j++) {
            const int64_t row = t * J_TILE + j * 256 + threadIdx.x;
            h[j] = row < n ? handle[row] : J_NONE;
            uint32_t ck = 0; off[j] = h[j];
            if (row < n) {
                if (h[j] != J_NONE) ck = E.csr ? __ldcs(E.hcnt + row) : 1u;
                else if (left_join) ck = 1;
            }
            c[j] = ck;
            uint32_t x = ck;
            for (int o = 1; o < 32; o <<= 1) { uint32_t y = __shfl_up_sync(0xffffffffu, x, o); if (lane >= (unsigned)o) x += y; }
            lane_excl[j] = x - ck;
            if (lane == 31) seg[j * 8 + warp] = x;
        }
        __syncthreads();
        uint32_t seg_tot[ITERS];
#pragma unroll
        for (int j = 0; j < ITERS; j++) seg_tot[j] = seg[j * 8 + warp];
        __syncthreads();
        if (warp == 0) {      // exclusive scan of the 64 segment totals (2 per lane)
            uint32_t a = seg[2 * lane], b = seg[2 * lane + 1], s2 = a + b, x = s2;
            for (int o = 1; o < 32; o <<= 1) { uint32_t y = __shfl_up_sync(0xffffffffu, x, o); if (lane >= (unsigned)o) x += y; }
            seg[2 * lane] = x - s2; seg[2 * lane + 1] = x - s2 + a;
        }
        __syncthreads();
        const uint64_t base = tile_off[t];
#pragma unroll
        for (int j = 0; j < ITERS; j++) {
            const uint32_t total = seg_tot[j];                   // warp-uniform
            if (total == 0) continue;
            const uint64_t sbase = base + seg[j * 8 + warp];
            const uint32_t pi = (uint32_t)(t * J_TILE + j * 256 + threadIdx.x);
            // 4 independent 32-tuple groups per round: the owner search (shuffles) of all four runs first, then their four
            // sorted_rows loads together, then the stores — one dependent L2 access per round instead of per group
            for (uint32_t q0 = 0; q0 < total; q0 += 128) {
                uint32_t s_h[4], s_pi[4], s_at[4]; bool live[4];
#pragma unroll
                for (int u = 0; u < 4; u++) {
                    const uint32_t q = q0 + 32 * u + lane;
                    int lo = 0;
#pragma unroll
                    for (int step = 16; step; step >>= 1) {
                        const int cand = lo + step;
                        const uint32_t pe = __shfl_sync(0xffffffffu, lane_excl[j], cand & 31);
                        if (cand < 32 && pe <= q) lo = cand;      // owner = last lane whose exclusive prefix is <= q (empty lanes lose the tie)
                    }
                    const uint32_t s_excl = __shfl_sync(0xffffffffu, lane_excl[j], lo);
                    s_h[u] = __shfl_sync(0xffffffffu, h[j], lo);
                    s_pi[u] = __shfl_sync(0xffffffffu, pi, lo);
                    s_at[u] = __shfl_sync(0xffffffffu, off[j], lo) + (q - s_excl);
                    live[u] = q < total;
                }
                uint32_t b[4];
#pragma unroll
                for (int u = 0; u < 4; u++) {
                    b[u] = s_h[u];
                    if (live[u] && E.csr && s_h[u] != J_NONE) b[u] = __ldg(E.sorted_rows + s_at[u]);
                }
#pragma unroll
                for (int u = 0; u < 4; u++)
                    if (live[u]) { const uint64_t at = sbase + q0 + 32 * u + lane; __stcs(out_probe + at, s_pi[u]); __stcs(out_build + at, b[u]); }
            }
        }
        __syncthreads();
    }
}

// ---------------------------------------------------------------------------- K8 fused probe + emit
// Unique build keys (any table form): every probe row yields at most one tuple, so probe and emission fuse into ONE
// pass with a decoupled look-back scan over 2048-row tiles (tiles are handed out by an atomic counter, so every
// predecessor of a tile is already running: the look-back cannot wait on an unscheduled CTA).  HBM traffic: 8 B key
// in + 8 B tuple out per match — exactly the algorithmic 16 B/row, instead of 24 B/row for the two-pass form.
// COMPACT: the first table load of 4 rows is issued before any of them is resolved, then the 4 verifying loads of
// the build column (two dependent L2 / HBM accesses per probe: the memory-level parallelism has to come from here).
// status[t]: bits 63..62 = 0 empty / 1 tile aggregate / 2 inclusive prefix, bits 61..0 = value.
constexpr unsigned long long LB_AGG = 1ull << 62, LB_INC = 2ull << 62, LB_VAL = (1ull << 62) - 1;
template <int MODE, int KEY_ELEM, int KEY_CANON>
__global__ void __launch_bounds__(256) k_join_probe_emit(const __grid_constant__ JoinDev J, const void* __restrict__ keys, const uint32_t* __restrict__ valid, int64_t n, int left_join,
                                                         unsigned long long* __restrict__ status, unsigned int* __restrict__ tile_counter, int* __restrict__ error,
                                                         uint32_t* __restrict__ out_probe, uint32_t* __restrict__ out_build) {
    constexpr int ITERS = J_TILE / 256;
    __shared__ uint32_t seg[ITERS * 8];
    __shared__ long long s_tile;
    __shared__ unsigned long long s_prefix;
    const unsigned lane = lane_id(), warp = threadIdx.x >> 5;
    const int64_t ntiles = (n + J_TILE - 1) / J_TILE;
    while (true) {
        if (threadIdx.x == 0) s_tile = (long long)atomicAdd(tile_counter, 1u);
        __syncthreads();
        const int64_t t = s_tile;
        if (t >= ntiles) break;
        uint32_t h[ITERS], lane_excl[ITERS]; bool emit[ITERS];
        uint64_t kraw[ITERS];
#pragma unroll
        for (int j = 0; j < ITERS; j++) {        // all key loads of the tile first (coalesced, 8 in flight per thread)
            const int64_t row = t * J_TILE + j * 256 + threadIdx.x;
            kraw[j] = 0;
            if (row < n) kraw[j] = KEY_ELEM == 8 ? __ldcs(reinterpret_cast<const unsigned long long*>(keys) + row) : (uint64_t)__ldcs(reinterpret_cast<const unsigned int*>(keys) + row);
        }
        if (MODE == JM_COMPACT) {
#pragma unroll
            for (int g = 0; g < ITERS; g += 4) {
                uint32_t slot[4], e[4], fp[4]; uint64_t key[4], bk[4]; int st[4];      // st: 0 miss, 1 verify pending, 2 continue probing, 3 hit
#pragma unroll
                for (int u = 0; u < 4; u++) {
                    const int j = g + u;
                    const int64_t row = t * J_TILE + j * 256 + threadIdx.x;
                    h[j] = J_NONE; st[u] = 0; slot[u] = 0; e[u] = J_NONE; fp[u] = 0; key[u] = 0; bk[u] = 0;
                    if (row >= n) continue;
                    const bool v = valid == nullptr || bit_get(valid, row);
                    if (!v) { if (J.nulls_equal) h[j] = __ldg(J.tab + J.ccap); continue; }
                    key[u] = j_canon<KEY_CANON>(kraw[j]);
                    const uint64_t hs = table_hash(key[u]);
                    slot[u] = (uint32_t)(hs >> J.cshift); fp[u] = (uint32_t)(hs >> (J.cshift - 8)) & 0xFFu;
                    e[u] = __ldg(J.tab + slot[u]);
                    st[u] = 2;
                }
#pragma unroll
                for (int u = 0; u < 4; u++) {
                    if (st[u] != 2) continue;
                    if (e[u] == J_NONE) { st[u] = 0; continue; }
                    if (!J.fp_mode || (e[u] >> 24) == fp[u]) { bk[u] = j_bkey<KEY_ELEM, KEY_CANON>(J.bkeys, J.fp_mode ? (e[u] & 0xFFFFFFu) : e[u]); st[u] = 1; }
                }
#pragma unroll
                for (int u = 0; u < 4; u++) {
                    const int j = g + u;
                    if (st[u] == 1 && bk[u] == key[u]) { h[j] = J.fp_mode ? (e[u] & 0xFFFFFFu) : e[u]; continue; }
                    if (st[u] == 0) continue;
                    // slow path: keep walking the probe sequence
                    uint32_t s = (slot[u] + 1) & J.cmask;
                    while (true) {
                        const uint32_t ee = __ldg(J.tab + s);
                        if (ee == J_NONE) break;
                        const uint32_t rr = J.fp_mode ? (ee & 0xFFFFFFu) : ee;
                        if ((!J.fp_mode || (ee >> 24) == fp[u]) && j_bkey<KEY_ELEM, KEY_CANON>(J.bkeys, rr) == key[u]) { h[j] = rr; break; }
                        s = (s + 1) & J.cmask;
                    }
                }
            }
        } else {
#pragma unroll
            for (int j = 0; j < ITERS; j++) {
                const int64_t row = t * J_TILE + j * 256 + threadIdx.x;
                h[j] = J_NONE;
                if (row < n) { const bool v = valid == nullptr || bit_get(valid, row); uint32_t c; h[j] = j_lookup<MODE, KEY_ELEM, KEY_CANON>(J, kraw[j], v, c); }
            }
        }
#pragma unroll
        for (int j = 0; j < ITERS; j++) {
            const int64_t row = t * J_TILE + j * 256 + threadIdx.x;
            emit[j] = row < n && (h[j] != J_NONE || left_join);
            const uint32_t b = __ballot_sync(0xffffffffu, emit[j]);
            lane_excl[j] = __popc(b & lanemask_lt());
            if (lane == 0) seg[j * 8 + warp] = __popc(b);
        }
        __syncthreads();
        if (warp == 0) {
            // exclusive scan of the 64 segment counts; tile total
            uint32_t a = seg[2 * lane], b2 = seg[2 * lane + 1], s2 = a + b2, x = s2;
            for (int o = 1; o < 32; o <<= 1) { uint32_t y = __shfl_up_sync(0xffffffffu, x, o); if (lane >= (unsigned)o) x += y; }
            seg[2 * lane] = x - s2; seg[2 * lane + 1] = x - s2 + a;
            const unsigned long long tile_total = __shfl_sync(0xffffffffu, x, 31);
            // decoupled look-back
            if (lane == 0) atomicExch(&status[t], (t == 0 ? LB_INC : LB_AGG) | tile_total);
            unsigned long long exclusive = 0;
            if (t > 0) {
                int64_t look = t - 1;
                while (true) {
                    const int64_t idx = look - lane;
                    unsigned long long stv = LB_INC;          // virtual predecessor before tile 0: inclusive 0
                    int spins = 0;
                    if (idx >= 0) stv = *reinterpret_cast<volatile unsigned long long*>(&status[idx]);
                    while (__any_sync(0xffffffffu, (stv >> 62) == 0)) {
                        if (idx >= 0 && (stv >> 62) == 0) stv = *reinterpret_cast<volatile unsigned long long*>(&status[idx]);
                        if (++spins > (1 << 22) || ((spins & 1023) == 0 && *reinterpret_cast<volatile int*>(error))) { *error = 1; break; }   // never hang the device
                    }
                    const unsigned inc = __ballot_sync(0xffffffffu, (stv >> 62) == 2);
                    const unsigned upto = inc ? (unsigned)(__ffs(inc) - 1) : 31u;     // nearest inclusive predecessor
                    unsigned long long v = lane <= upto ? (stv & LB_VAL) : 0ull;
                    for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
                    exclusive += v;
                    if (inc || *reinterpret_cast<volatile int*>(error)) break;
                    look -= 32;
                }
                if (lane == 0) atomicExch(&status[t], LB_INC | ((exclusive + tile_total) & LB_VAL));
            }
            if (lane == 0) s_prefix = exclusive;
        }
        __syncthreads();
        const uint64_t base = s_prefix;
#pragma unroll
        for (int j = 0; j < ITERS; j++) {
            if (!emit[j]) continue;
            const uint64_t pos = base + seg[j * 8 + warp] + lane_excl[j];
            out_probe[pos] = (uint32_t)(t * J_TILE + j * 256 + threadIdx.x);
            out_build[pos] = h[j];
        }
        __syncthreads();
    }
}

// ---------------------------------------------------------------------------- semi / anti: one hit bit per left row
// hash_join_tuples_left_semi / _anti (single_keys_semi_anti.rs:41-140): the left rows, in row order, that have (semi) /
// do not have (anti) a key match on the right; a null left key never matches unless nulls_equal.
template <int MODE, int KEY_ELEM, int KEY_CANON>
__global__ void __launch_bounds__(256) k_join_probe_bits(const __grid_constant__ JoinDev J, const void* __restrict__ keys, const uint32_t* __restrict__ valid, int64_t n, int64_t n_round,
                                                         int anti, uint32_t* __restrict__ mask_words) {
    for (int64_t row = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; row < n_round; row += (int64_t)gridDim.x * blockDim.x) {
        bool keep = false;
        if (row < n) {
            const uint64_t kraw = KEY_ELEM == 8 ? __ldcs(reinterpret_cast<const unsigned long long*>(keys) + row) : (uint64_t)__ldcs(reinterpret_cast<const unsigned int*>(keys) + row);
            const bool v = valid == nullptr || bit_get(valid, row);
            uint32_t c;
            const bool hit = j_lookup<MODE, KEY_ELEM, KEY_CANON>(J, kraw, v, c) != J_NONE;
            keep = anti ? !hit : hit;
        }
        const unsigned b = __ballot_sync(0xffffffffu, keep);
        if ((threadIdx.x & 31) == 0) mask_words[row >> 5] = b;
    }
}

// =============================================================================================
// Host side
// =============================================================================================
static DevCol idx_col(DevPtr p, int64_t n, int64_t null_count) { DevCol c; c.dtype = BL_UINT32; c.len = n; c.values = p; c.null_count = null_count; return c; }

struct JoinBuilt {
    int mode = JM_COMPACT;
    bool csr = false;
    JoinDev J;
    DevPtr entries, dense_table, tab, cnt, off, slot_of_row, sorted_rows;
};

static int join_table_pref() {
    const char* e = getenv("BL_JOIN_TABLE");
    return (e && (e[0] == 'c' || e[0] == 'C')) ? JM_COMPACT : JM_WIDE;      // WIDE: one sector per lookup, COMPACT: two dependent ones
}

// K7.  need_lists = false (semi / anti): duplicates need no row lists, only membership.
static JoinBuilt join_build(const DevCol& build, bool nulls_equal, bool need_lists) {
    Context& c = ctx();
    JoinBuilt B; memset(&B.J, 0, sizeof B.J);
    const int dt = build.dtype;
    const int64_t nb = build.len;
    const int elem = dtype_size(dt);
    const int sign_bits = dtype_is_signed(dt) ? elem * 8 : 0;
    B.J.nulls_equal = nulls_equal ? 1 : 0; B.J.sign_bits = sign_bits;
    // ---- dense direct-address table when the build keys are dense integers (unique, or membership only)
    const char* env_dense = getenv("BL_JOIN_DENSE");
    if (dtype_is_int(dt) && !nulls_equal && nb >= 1024 && !(env_dense && env_dense[0] == '0')) {
        DevPtr mm = dev_alloc(16);
        unsigned long long init_mm[2] = {~0ull, 0ull};
        PLB_CUDA(cudaMemcpyAsync(mm->p, init_mm, 16, cudaMemcpyHostToDevice, c.stream));
        PLB_LAUNCH("k7_join_minmax", k_join_minmax, grid_for(nb, 256), 256, 0, build.v(), build.vm(), elem, sign_bits, nb, as<unsigned long long>(mm));
        unsigned long long hmm[2];
        PLB_CUDA(cudaMemcpyAsync(hmm, mm->p, 16, cudaMemcpyDeviceToHost, c.stream));
        PLB_CUDA(cudaStreamSynchronize(c.stream));
        if (hmm[0] <= hmm[1] && hmm[1] - hmm[0] < (unsigned long long)8 * (unsigned long long)nb) {
            const uint64_t kmin = hmm[0], range = hmm[1] - hmm[0] + 1;
            DevPtr table = dev_alloc((size_t)range * 4 + 16);
            DevPtr dups = dev_alloc(4); dev_memset(dups->p, 0, 4);
            PLB_LAUNCH("k7_dense_init", k_fill_u32j, grid_for((int64_t)range, 256), 256, 0, as<uint32_t>(table), J_NONE, (int64_t)range);
            PLB_LAUNCH("k7_dense_build", k_join_dense_build, grid_for(nb, 256), 256, 0, as<uint32_t>(table), build.v(), build.vm(), elem, sign_bits, nb, (uint64_t)kmin, as<int>(dups));
            if (!need_lists || read_scalar(as<int>(dups)) == 0) {       // duplicates + row lists wanted -> hashed table + CSR lists
                B.mode = JM_DENSE; B.dense_table = table;
                B.J.dense = as<uint32_t>(table); B.J.kmin = kmin; B.J.range = range;
                return B;
            }
        }
    }
    B.mode = join_table_pref();
    B.slot_of_row = dev_alloc((size_t)std::max<int64_t>(nb, 1) * 4);
    DevPtr has_dups = dev_alloc(4);
    dev_memset(has_dups->p, 0, 4);
    if (B.mode == JM_WIDE) {
        // two-entry buckets, half full by default: C3 (1e7 keys) = 1e7 buckets = 320 MB
        const double per_bucket = [] { const char* e = getenv("BL_JOIN_BUCKET_FILL"); double v = e ? atof(e) : 1.0; return (v >= 0.5 && v <= 1.9) ? v : 1.0; }();      // build rows per 2-entry bucket
        JoinTableDev T; T.nb = (uint64_t)std::max<int64_t>((int64_t)((double)nb / per_bucket) + 1, 8);
        PLB_REQUIRE(2 * (T.nb + 1) < 0xFFFFFFFFull, BL_ERR_UNSUPPORTED, "join: build side too large for 32-bit slots");
        B.entries = dev_alloc((size_t)(T.nb + 1) * sizeof(JoinBucket));
        T.buckets = as<JoinBucket>(B.entries);
        PLB_LAUNCH("k7_join_init", k_join_init, grid_for((int64_t)T.nb + 1, 256), 256, 0, T.buckets, (int64_t)T.nb + 1);
        if (nb > 0)
            PLB_LAUNCH("k7_join_build", k_join_build, grid_for(nb, 256), 256, 0, T, build.v(), build.vm(), dt, nb, nulls_equal ? 1 : 0, as<uint32_t>(B.slot_of_row), as<int>(has_dups));
        B.J.W = T;
        B.csr = need_lists && nb > 0 && read_scalar(as<int>(has_dups)) != 0;
        if (B.csr) {
            const int64_t ne = 2 * ((int64_t)T.nb + 1), ntiles_e = (ne + J_TILE - 1) / J_TILE;
            DevPtr sums = dev_alloc((size_t)ntiles_e * 4), offs = dev_alloc((size_t)ntiles_e * 8);
            PLB_LAUNCH("k7_tile_sums", k_join_tile_sums, grid_for(ntiles_e * 256, 256), 256, 0, as<uint32_t>(B.entries), ne, as<uint32_t>(sums));
            exclusive_scan_u32_to_u64(as<uint32_t>(sums), as<uint64_t>(offs), ntiles_e, nullptr);
            PLB_LAUNCH("k7_csr_offsets", k_join_csr_offsets, grid_for(ntiles_e * 256, 256), 256, 0, as<uint32_t>(B.entries), ne, as<uint64_t>(offs));
        }
    } else {
        uint64_t cap = 1024; while (cap < (uint64_t)nb + (uint64_t)nb / 2) cap <<= 1;
        PLB_REQUIRE(cap <= (1ull << 32), BL_ERR_UNSUPPORTED, "join: build side too large for 32-bit slots");
        int shift = 64; for (uint64_t x = cap; x > 1; x >>= 1) shift--;
        B.tab = dev_alloc((size_t)(cap + 1) * 4);
        PLB_LAUNCH("k7_jc_init", k_fill_u32j, grid_for((int64_t)cap + 1, 256), 256, 0, as<uint32_t>(B.tab), J_NONE, (int64_t)cap + 1);
        const int fp_mode = nb < (1 << 24) - 1 ? 1 : 0;
        if (nb > 0) {
            const int grid = grid_for(nb, 256);
            const int ne = nulls_equal ? 1 : 0;
#define JC_BUILD(E, CN) PLB_LAUNCH("k7_jc_build", (k_jc_build<E, CN>), grid, 256, 0, as<uint32_t>(B.tab), (uint32_t)(cap - 1), shift, fp_mode, (uint32_t)cap, build.v(), build.vm(), nb, ne, as<uint32_t>(B.slot_of_row), as<int>(has_dups))
            if (dt == BL_FLOAT64) JC_BUILD(8, 1); else if (dt == BL_FLOAT32) JC_BUILD(4, 2); else if (elem == 8) JC_BUILD(8, 0); else JC_BUILD(4, 0);
#undef JC_BUILD
        }
        B.J.tab = as<uint32_t>(B.tab); B.J.cmask = (uint32_t)(cap - 1); B.J.cshift = shift; B.J.fp_mode = fp_mode; B.J.ccap = (uint32_t)cap; B.J.bkeys = build.v();
        B.csr = need_lists && nb > 0 && read_scalar(as<int>(has_dups)) != 0;
        if (B.csr) {
            const int64_t ne = (int64_t)cap + 1, ntiles_e = (ne + J_TILE - 1) / J_TILE;
            B.cnt = dev_alloc((size_t)ne * 4); B.off = dev_alloc((size_t)ne * 4);
            dev_memset(B.cnt->p, 0, (size_t)ne * 4);
            PLB_LAUNCH("k7_slot_counts", k_jc_count, grid_for(nb, 256), 256, 0, as<uint32_t>(B.slot_of_row), nb, as<uint32_t>(B.cnt));
            DevPtr sums = dev_alloc((size_t)ntiles_e * 4), offs = dev_alloc((size_t)ntiles_e * 8);
            PLB_LAUNCH("k7_tile_sums", k_jc_tile_sums, grid_for(ntiles_e * 256, 256), 256, 0, as<uint32_t>(B.cnt), ne, as<uint32_t>(sums));
            exclusive_scan_u32_to_u64(as<uint32_t>(sums), as<uint64_t>(offs), ntiles_e, nullptr);
            PLB_LAUNCH("k7_csr_offsets", k_jc_offsets, grid_for(ntiles_e * 256, 256), 256, 0, as<uint32_t>(B.cnt), ne, as<uint64_t>(offs), as<uint32_t>(B.off));
            B.J.ccnt = as<uint32_t>(B.cnt); B.J.coff = as<uint32_t>(B.off);
        }
    }
    if (B.csr) {
        // ascending row lists: stable sort of the build rows by slot (skipped null rows sort last)
        B.sorted_rows = dev_alloc((size_t)nb * 4);
        iota_u32(as<uint32_t>(B.sorted_rows), nb, 0);
        // J_NONE (skipped null rows) has every bit set and sorts last with any digit count that covers the real slots + 1 bit
        const uint64_t max_slot = B.mode == JM_WIDE ? 2 * (B.J.W.nb + 1) : (uint64_t)B.J.ccap + 1;
        sort_pairs_u32(as<uint32_t>(B.slot_of_row), as<uint32_t>(B.sorted_rows), nb, std::min(32, bits_for(max_slot) + 1));
    }
    B.J.csr = B.csr ? 1 : 0;
    return B;
}

// dispatch a kernel template over (table form, key width, float canonicalisation)
#define J_DISPATCH(KERNEL_CALL)                                                                  \
    do {                                                                                         \
        if (B.mode == JM_DENSE) { if (elem == 8) { KERNEL_CALL(JM_DENSE, 8, 0); } else { KERNEL_CALL(JM_DENSE, 4, 0); } }                       \
        else if (B.mode == JM_WIDE) {                                                            \
            if (dt == BL_FLOAT64) { KERNEL_CALL(JM_WIDE, 8, 1); } else if (dt == BL_FLOAT32) { KERNEL_CALL(JM_WIDE, 4, 2); }                    \
            else if (elem == 8) { KERNEL_CALL(JM_WIDE, 8, 0); } else { KERNEL_CALL(JM_WIDE, 4, 0); } }                                          \
        else {                                                                                   \
            if (dt == BL_FLOAT64) { KERNEL_CALL(JM_COMPACT, 8, 1); } else if (dt == BL_FLOAT32) { KERNEL_CALL(JM_COMPACT, 4, 2); }              \
            else if (elem == 8) { KERNEL_CALL(JM_COMPACT, 8, 0); } else { KERNEL_CALL(JM_COMPACT, 4, 0); } }                                    \
    } while (0)

static void check_join_keys(const DevCol& left, const DevCol& right) {
    PLB_REQUIRE(left.dtype == right.dtype, BL_ERR_DTYPE, std::string("join: key dtypes differ (") + dtype_name(left.dtype) + " vs " + dtype_name(right.dtype) + ")");   // join/mod.rs:231-241
    const int dt = left.dtype;
    PLB_REQUIRE(dt == BL_INT64 || dt == BL_UINT64 || dt == BL_INT32 || dt == BL_UINT32 || dt == BL_FLOAT64 || dt == BL_FLOAT32, BL_ERR_UNSUPPORTED,
                std::string("join: key dtype ") + dtype_name(dt) + " is outside the hot path");
    PLB_REQUIRE(left.len < 0xFFFFFFFFll && right.len < 0xFFFFFFFFll, BL_ERR_UNSUPPORTED, "join: more than 2^32-2 rows (IdxSize = u32)");
}

static JoinResult hash_join_semi_anti(const DevCol& left, const DevCol& right, int how, bool nulls_equal) {
    check_join_keys(left, right);
    const int dt = left.dtype, elem = dtype_size(dt);
    const int64_t n = left.len;
    JoinResult r;
    r.right = idx_col(dev_alloc(16), 0, 0);
    if (n == 0) { r.left = idx_col(dev_alloc(16), 0, 0); return r; }
    JoinBuilt B = join_build(right, nulls_equal, false);
    DevCol mask = make_col(BL_BOOL, n, false);
    const int64_t n_round = (n + 31) / 32 * 32;
    const int grid = grid_for(n_round, 256, 16);
    const int anti = how == BL_JOIN_ANTI ? 1 : 0;
#define SA_CALL(M, E, CN) PLB_LAUNCH("k8_join_probe_bits", (k_join_probe_bits<M, E, CN>), grid, 256, 0, B.J, left.v(), left.vm(), n, n_round, anti, as<uint32_t>(mask.values))
    J_DISPATCH(SA_CALL);
#undef SA_CALL
    DevCol rows = make_col(BL_UINT32, n, false);
    iota_u32(as<uint32_t>(rows.values), n, 0);
    std::vector<DevCol> in{rows}, out;
    op_filter(in, mask, out);
    r.left = out[0];
    return r;
}

// Probe `probe` against a table built over `build`: tuples (probe row, build row) in probe-row order, matches ascending
// by build row; left_join != 0 also emits (probe row, J_NONE) for probe rows without a match.
struct ProbeTuples { DevPtr out_probe, out_build; uint64_t M = 0; };
static ProbeTuples probe_tuples(const DevCol& probe, const DevCol& build, bool nulls_equal, int left_join) {
    const int dt = probe.dtype;
    const int64_t np = probe.len;
    const int elem = dtype_size(dt);
    Context& c = ctx();

    trace_point("join:start");
    JoinBuilt B = join_build(build, nulls_equal, true);
    trace_point("join:build");
    // ---- unique build keys: fused single-pass probe + emit
    const int fused_on = [] { const char* e = getenv("BL_JOIN_FUSED"); return e ? atoi(e) : 1; }();
    const int64_t ntiles = (np + J_TILE - 1) / J_TILE;
    uint64_t M = 0;
    DevPtr out_probe, out_build;
    bool done = false;
    if (fused_on && !B.csr && np > 0) {
        out_probe = dev_alloc((size_t)np * 4 + 16); out_build = dev_alloc((size_t)np * 4 + 16);
        DevPtr st = dev_alloc((size_t)ntiles * 8 + 16), ctl = dev_alloc(8);
        dev_memset(st->p, 0, (size_t)ntiles * 8 + 16); dev_memset(ctl->p, 0, 8);
        const int grid = (int)std::min<int64_t>(ntiles, (int64_t)c.sm_count * 6);
        unsigned long long* stp = as<unsigned long long>(st); unsigned* cnt = as<unsigned>(ctl); int* err = as<int>(ctl) + 1;
#define PE_CALL(M_, E, CN) PLB_LAUNCH("k8_join_probe_emit", (k_join_probe_emit<M_, E, CN>), grid, 256, 0, B.J, probe.v(), probe.vm(), np, left_join, stp, cnt, err, as<uint32_t>(out_probe), as<uint32_t>(out_build))
        J_DISPATCH(PE_CALL);
#undef PE_CALL
        unsigned long long last = 0; int herr[2] = {0, 0};
        PLB_CUDA(cudaMemcpyAsync(&last, stp + (ntiles - 1), 8, cudaMemcpyDeviceToHost, c.stream));
        PLB_CUDA(cudaMemcpyAsync(herr, ctl->p, 8, cudaMemcpyDeviceToHost, c.stream));
        PLB_CUDA(cudaStreamSynchronize(c.stream));
        if (herr[1] == 0) { M = last & LB_VAL; done = true; }     // else: look-back gave up -> two-pass path below
    }
    trace_point("join:probe");
    if (!done) {
        // ---- probe pass 1
        DevPtr handle = dev_alloc((size_t)std::max<int64_t>(np, 1) * 4 + 16), hcnt = dev_alloc(B.csr ? (size_t)std::max<int64_t>(np, 1) * 4 + 16 : 16), tc = dev_alloc((size_t)std::max<int64_t>(ntiles, 1) * 8), toff = dev_alloc((size_t)std::max<int64_t>(ntiles, 1) * 8), total = dev_alloc(8);
        dev_memset(tc->p, 0, (size_t)std::max<int64_t>(ntiles, 1) * 8); dev_memset(total->p, 0, 8);
        if (np > 0) {
            const int grid = grid_for((np + 1) / 2, 256);
            uint32_t* hp = as<uint32_t>(handle); unsigned long long* tcp = as<unsigned long long>(tc);
#define PR_CALL(M_, E, CN) PLB_LAUNCH("k8_join_probe", (k_join_probe<M_, E, CN>), grid, 256, 0, B.J, probe.v(), probe.vm(), np, left_join, hp, as<uint32_t>(hcnt), tcp)
            J_DISPATCH(PR_CALL);
#undef PR_CALL
            exclusive_scan_u64(as<uint64_t>(tc), as<uint64_t>(toff), ntiles, as<uint64_t>(total));
            M = read_scalar(as<unsigned long long>(total));
        }
        PLB_REQUIRE(M < 0xFFFFFFFFull, BL_ERR_UNSUPPORTED, "join: result has more than 2^32-2 rows (IdxSize = u32)");
        // ---- probe pass 2
        out_probe = dev_alloc((size_t)std::max<uint64_t>(M, 1) * 4 + 16); out_build = dev_alloc((size_t)std::max<uint64_t>(M, 1) * 4 + 16);
        if (M > 0) {
            JoinEmitDev E; memset(&E, 0, sizeof E);
            E.hcnt = as<uint32_t>(hcnt); E.sorted_rows = as<uint32_t>(B.sorted_rows); E.csr = B.csr ? 1 : 0;
            PLB_LAUNCH("k8_join_emit", k_join_emit, (int)std::min<int64_t>(ntiles, (int64_t)c.sm_count * 8), 256, 0, E, as<uint32_t>(handle), np, left_join,
                       as<uint64_t>(toff), as<uint32_t>(out_probe), as<uint32_t>(out_build));
        }
    }
    if (!out_probe) { out_probe = dev_alloc(16); out_build = dev_alloc(16); }
    trace_point("join:emit");
    ProbeTuples t; t.out_probe = out_probe; t.out_build = out_build; t.M = M;
    return t;
}

// nullable index column: validity bit = (idx != BL_IDX_NULL)
static void set_idx_validity(DevCol& col) {
    if (col.len == 0) return;
    DevCol none = make_col(BL_UINT32, 1, false);
    const uint32_t nv = J_NONE;
    PLB_CUDA(cudaMemcpyAsync(none.values->p, &nv, 4, cudaMemcpyHostToDevice, ctx().stream));
    PLB_CUDA(cudaStreamSynchronize(ctx().stream));
    DevCol m = op_compare(BL_CMP_NE, col, none, false);
    col.validity = m.values;
    col.null_count = -1;
}

__global__ void __launch_bounds__(256) k_join_mark_rows(const uint32_t* __restrict__ rows, int64_t m, uint32_t* __restrict__ bits) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < m; i += (int64_t)gridDim.x * blockDim.x) {
        const uint32_t r = __ldcs(rows + i);
        if (r != J_NONE) atomicOr(&bits[r >> 5], 1u << (r & 31));
    }
}
__global__ void __launch_bounds__(256) k_join_invert_bits(uint32_t* __restrict__ bits, int64_t words) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < words; i += (int64_t)gridDim.x * blockDim.x) bits[i] = ~bits[i];
}

// hash_join_tuples_outer (single_keys_outer.rs:100-260): left-join tuples of the probing (longer) side, then the build rows
// nobody matched — found from the emitted build indices themselves (one bit per build row), compacted in ascending order.
static JoinResult hash_join_full(const DevCol& left, const DevCol& right, bool nulls_equal, int maintain_order) {
    PLB_REQUIRE(maintain_order == BL_ORDER_NONE, BL_ERR_UNSUPPORTED, "join: maintain_order on a full join is outside the hot path");
    check_join_keys(left, right);
    const bool swapped = !(left.len > right.len);
    const DevCol& probe = swapped ? right : left;
    const DevCol& build = swapped ? left : right;
    ProbeTuples t = probe_tuples(probe, build, nulls_equal, 1);
    PLB_REQUIRE(t.M + (uint64_t)build.len < 0xFFFFFFFFull, BL_ERR_UNSUPPORTED, "join: result has more than 2^32-2 rows (IdxSize = u32)");
    const int64_t nb = build.len;
    DevCol unmatched; unmatched.dtype = BL_UINT32; unmatched.len = 0;
    if (nb > 0) {
        DevCol mask = make_col(BL_BOOL, nb, false);
        const int64_t words = (nb + 31) / 32;
        dev_memset(mask.values->p, 0, (size_t)words * 4);
        if (t.M > 0) PLB_LAUNCH("k8_join_mark_rows", k_join_mark_rows, grid_for((int64_t)t.M, 256, 16), 256, 0, as<uint32_t>(t.out_build), (int64_t)t.M, as<uint32_t>(mask.values));
        PLB_LAUNCH("k8_join_invert", k_join_invert_bits, grid_for(words, 256), 256, 0, as<uint32_t>(mask.values), words);
        DevCol rows = make_col(BL_UINT32, nb, false);
        iota_u32(as<uint32_t>(rows.values), nb, 0);
        std::vector<DevCol> in{rows}, out;
        op_filter(in, mask, out);
        unmatched = out[0];
    }
    const int64_t D = unmatched.len, M = (int64_t)t.M;
    DevPtr fp = dev_alloc((size_t)std::max<int64_t>(M + D, 1) * 4 + 16), fb = dev_alloc((size_t)std::max<int64_t>(M + D, 1) * 4 + 16);
    if (M > 0) {
        PLB_CUDA(cudaMemcpyAsync(fp->p, t.out_probe->p, (size_t)M * 4, cudaMemcpyDeviceToDevice, ctx().stream));
        PLB_CUDA(cudaMemcpyAsync(fb->p, t.out_build->p, (size_t)M * 4, cudaMemcpyDeviceToDevice, ctx().stream));
    }
    if (D > 0) {
        PLB_LAUNCH("k7_dense_init", k_fill_u32j, grid_for(D, 256), 256, 0, as<uint32_t>(fp) + M, J_NONE, D);
        PLB_CUDA(cudaMemcpyAsync(as<uint32_t>(fb) + M, unmatched.values->p, (size_t)D * 4, cudaMemcpyDeviceToDevice, ctx().stream));
    }
    JoinResult r;
    r.left = idx_col(swapped ? fb : fp, M + D, -1);
    r.right = idx_col(swapped ? fp : fb, M + D, -1);
    set_idx_validity(r.left);
    set_idx_validity(r.right);
    return r;
}

static JoinResult hash_join_inner_left(const DevCol& left, const DevCol& right, int how, bool nulls_equal, int maintain_order) {
    PLB_REQUIRE(how == BL_JOIN_INNER || how == BL_JOIN_LEFT, BL_ERR_UNSUPPORTED, "join: only inner, left, full, semi and anti joins are on the hot path");
    check_join_keys(left, right);
    // hash_join/mod.rs:41-50: probe the longer relation; on a tie the right side probes (swapped)
    const bool swapped = how == BL_JOIN_INNER && !(left.len > right.len);
    const DevCol& probe = swapped ? right : left;
    const DevCol& build = swapped ? left : right;
    Context& c = ctx();
    ProbeTuples t = probe_tuples(probe, build, nulls_equal, how == BL_JOIN_LEFT ? 1 : 0);
    DevPtr out_probe = t.out_probe, out_build = t.out_build;
    const uint64_t M = t.M;

    JoinResult r;
    r.left = idx_col(swapped ? out_build : out_probe, (int64_t)M, 0);
    r.right = idx_col(swapped ? out_probe : out_build, (int64_t)M, how == BL_JOIN_LEFT ? -1 : 0);
    // maintain_order (join/mod.rs:577-642): stable sort on the requested side unless already in that order
    if (how == BL_JOIN_INNER && maintain_order != BL_ORDER_NONE && M > 1) {
        const bool by_left = maintain_order == BL_ORDER_LEFT || maintain_order == BL_ORDER_LEFT_RIGHT;
        const bool left_sorted = !swapped;
        if (by_left && !left_sorted) sort_pairs_u32(as<uint32_t>(r.left.values), as<uint32_t>(r.right.values), (int64_t)M, bits_for((uint64_t)left.len));
        else if (!by_left && !swapped) sort_pairs_u32(as<uint32_t>(r.right.values), as<uint32_t>(r.left.values), (int64_t)M, bits_for((uint64_t)right.len));
    }
    // left join: only Right / RightLeft reorder (stable sort on the right idx, unmatched rows = u32::MAX last;
    // dispatch_left_right.rs:142-170); the probe order already is the left order
    if (how == BL_JOIN_LEFT && (maintain_order == BL_ORDER_RIGHT || maintain_order == BL_ORDER_RIGHT_LEFT) && M > 1)
        sort_pairs_u32(as<uint32_t>(r.right.values), as<uint32_t>(r.left.values), (int64_t)M);
    if (how == BL_JOIN_LEFT && M > 0) set_idx_validity(r.right);      // Arrow-proper validity for the nullable right index
    (void)c;
    trace_point("join:done");
    return r;
}

JoinResult op_hash_join(const DevCol& left, const DevCol& right, int how, bool nulls_equal, int maintain_order) {
    if (how == BL_JOIN_SEMI || how == BL_JOIN_ANTI) return hash_join_semi_anti(left, right, how, nulls_equal);
    if (how == BL_JOIN_FULL) return hash_join_full(left, right, nulls_equal, maintain_order);
    return hash_join_inner_left(left, right, how, nulls_equal, maintain_order);
}

}  // namespace plb
