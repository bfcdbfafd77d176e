// groupby_dev.cuh — device helpers shared by the group_by kernels (groupby.cu: L2-resident table plans; groupby_radix.cu:
// partitioned plan).  Semantics cited in groupby.cu's header.
#pragma once
#include "common.cuh"
#include "dev_utils.cuh"
#include "groupby.h"

namespace plb {

__host__ __device__ inline uint64_t word_identity(int op) {
    switch (op) {
        case W_MIN_S64: return 0x7FFFFFFFFFFFFFFFULL;
        case W_MAX_S64: return 0x8000000000000000ULL;
        case W_MIN_U64: case W_MIN_F64: return 0xFFFFFFFFFFFFFFFFULL;
        default: return 0;   // adds, MAX_U64, MAX_F64
    }
}


template <int KEY_CANON> __device__ __forceinline__ uint64_t canon_key(uint64_t raw) {
    if (KEY_CANON == 1) return canonical_f64_bits(__longlong_as_double((long long)raw));
    if (KEY_CANON == 2) return canonical_f32_bits(__uint_as_float((uint32_t)raw));
    return raw;
}
__device__ __forceinline__ uint64_t load_key_rt(const void* keys, int dtype, int64_t row) {
    switch (dtype) {
        case BL_INT64: case BL_UINT64: return reinterpret_cast<const uint64_t*>(keys)[row];
        case BL_FLOAT64: return canonical_f64_bits(reinterpret_cast<const double*>(keys)[row]);
        case BL_FLOAT32: return canonical_f32_bits(reinterpret_cast<const float*>(keys)[row]);
        default: return (uint64_t)reinterpret_cast<const uint32_t*>(keys)[row];   // i32/u32 bit pattern, zero-extended
    }
}

// the slot of a row's key in a built table, by the build's rules: a null key -> cap, the GB_EMPTY key -> cap + 1, any other
// key -> linear probing from its hash (k_gb_lookup_first, unique.cu)
__device__ __forceinline__ uint64_t gb_lookup_slot(const GbTableDev& T, const void* keys, const uint32_t* key_validity, int key_dtype, int64_t row) {
    if (key_validity != nullptr && !bit_get(key_validity, row)) return T.cap;
    const uint64_t key = load_key_rt(keys, key_dtype, row);
    if (key == GB_EMPTY) return T.cap + 1;
    const uint64_t mask = T.cap - 1;
    uint64_t slot = table_hash(key) >> T.shift;
    for (int probes = 0; probes < GB_MAX_PROBE; ++probes) {
        if (__ldcg(reinterpret_cast<const unsigned long long*>(T.entries + slot * T.es)) == key) break;
        slot = (slot + 1) & mask;
    }
    return slot;
}
// word 1 of a slot: lo32 = len, hi32 = first row
__device__ __forceinline__ uint64_t gb_slot_word1(const GbTableDev& T, uint64_t slot) {
    return __ldcg(reinterpret_cast<const unsigned long long*>(T.entries + slot * T.es + gb_woff((int64_t)slot, 1, T.ws, T.pw)));
}


__device__ __forceinline__ double raw_to_f64(int dtype, uint64_t raw) {
    switch (dtype) {
        case BL_INT64: return (double)(long long)raw;
        case BL_UINT64: return (double)(unsigned long long)raw;
        case BL_INT32: return (double)(int)(uint32_t)raw;
        case BL_UINT32: return (double)(uint32_t)raw;
        case BL_FLOAT64: return __longlong_as_double((long long)raw);
        default: return (double)__uint_as_float((uint32_t)raw);
    }
}
__device__ __forceinline__ uint64_t raw_to_int(int dtype, uint64_t raw) {
    return dtype == BL_INT32 ? (uint64_t)(long long)(int)(uint32_t)raw : raw;   // sign-extend i32; u32 already zero-extended
}

// rows r0 and r0 + 1 of a column of ELEM-byte values: one 128-bit (8-byte types) or 64-bit (4-byte types) streaming load
template <int ELEM> __device__ __forceinline__ void gb_load_pair(const void* col, int64_t r0, uint64_t& a, uint64_t& b) {
    if (ELEM == 8) { const ulonglong2 t = ld_stream_u64x2(reinterpret_cast<const uint64_t*>(col) + r0); a = t.x; b = t.y; }
    else { const uint2 t = ld_stream_u32x2(reinterpret_cast<const uint32_t*>(col) + r0); a = t.x; b = t.y; }
}
__device__ __forceinline__ void gb_load_pair_rt(const void* col, int elem, int64_t r0, uint64_t& a, uint64_t& b) {
    if (elem == 8) gb_load_pair<8>(col, r0, a, b); else gb_load_pair<4>(col, r0, a, b);
}

// ---- global-memory accumulators: REDs, optionally with an L2 cache-policy hint (groupby.cu: make_policy_evict_last)
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
// an integer 0 or a float +-0.0 is not added: the accumulator starts at 0 / +0.0 and never becomes -0.0, so the bits agree
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
// every accumulator word of one row: val(c) = the row's raw value in column c, word(w) = address of accumulator word w.
// skip_pair: word L.pair_k travels in a bulk reduce instead.  MAXC >= L.n_cols: the row loops, column loop unrolled
// (values in registers).  MAXC = 0: a plain loop for the odd tail row, value loaded once per column.  The two loops
// are written so that the row-loop kernels get the same ptxas allocation as the hand-inlined code they replace: an
// `#pragma unroll (expr)` form, or the value hoisted in the unrolled loop, moved registers and spills in some of them.
template <int MAXC, class Val, class Word>
__device__ __forceinline__ void gb_apply_words(const GbLayout& L, const GbBatch& B, int64_t row, Val val, Word word, uint64_t pol = 0, bool hint = false, bool skip_pair = false) {
    if constexpr (MAXC > 0) {
#pragma unroll
        for (int c = 0; c < MAXC; c++) {
            if (c < L.n_cols) {
                const bool valid = B.cols[c].validity == nullptr || bit_get(B.cols[c].validity, row);
                const int dt = B.cols[c].dtype;
                for (int k = L.col_kbegin[c]; k < L.col_kbegin[c + 1]; k++) {
                    if (skip_pair && k == L.pair_k) continue;
                    gb_apply(L.wop[k], word(L.wslot[k]), dt, val(c), valid, pol, hint);
                }
            }
        }
    } else {
        for (int c = 0; c < L.n_cols; c++) {
            const bool valid = B.cols[c].validity == nullptr || bit_get(B.cols[c].validity, row);
            const uint64_t raw = val(c);
            for (int k = L.col_kbegin[c]; k < L.col_kbegin[c + 1]; k++) {
                if (skip_pair && k == L.pair_k) continue;
                gb_apply(L.wop[k], word(L.wslot[k]), B.cols[c].dtype, raw, valid, pol, hint);
            }
        }
    }
}


// ---- shared-memory accumulators: 32-bit native ATOMS; 64-bit integer adds as two 32-bit adds with carry (exact,
//      order-free); f64 add and 64-bit min/max are CAS loops (ATOMS.CAST.SPIN.64).
__device__ __forceinline__ void s_add_u64(uint64_t* a, uint64_t v) {
    uint32_t* w = reinterpret_cast<uint32_t*>(a);
    const uint32_t lo = (uint32_t)v, hi = (uint32_t)(v >> 32);
    const uint32_t old = atomicAdd(w, lo);
    const uint32_t up = hi + (((uint32_t)(old + lo) < old) ? 1u : 0u);
    if (up) atomicAdd(w + 1, up);
}
// FAST: every value column is 8 bytes wide and has no validity bitmap (the common analytic case): the
// dtype dispatch collapses to one select and the null checks disappear (this kernel is issue-bound).
template <bool FAST>
__device__ __forceinline__ void gb_apply_smem(int op, uint64_t* addr, int dtype, uint64_t raw, bool valid) {
    switch (op) {
        case W_ADD_INT: { uint64_t v = FAST ? raw : raw_to_int(dtype, raw); if (valid && v) s_add_u64(addr, v); break; }
        case W_ADD_F64: { double f = FAST ? (dtype == BL_FLOAT64 ? __longlong_as_double((long long)raw) : (dtype == BL_INT64 ? (double)(long long)raw : (double)(unsigned long long)raw)) : raw_to_f64(dtype, raw);
                          if (valid && f != 0.0) atomicAdd(reinterpret_cast<double*>(addr), f); break; }
        case W_MIN_S64: if (valid) atomicMin(reinterpret_cast<long long*>(addr), (long long)raw_to_int(dtype, raw)); break;
        case W_MAX_S64: if (valid) atomicMax(reinterpret_cast<long long*>(addr), (long long)raw_to_int(dtype, raw)); break;
        case W_MIN_U64: if (valid) atomicMin(reinterpret_cast<unsigned long long*>(addr), (unsigned long long)raw); break;
        case W_MAX_U64: if (valid) atomicMax(reinterpret_cast<unsigned long long*>(addr), (unsigned long long)raw); break;
        case W_MIN_F64: { double f = raw_to_f64(dtype, raw); if (valid && f == f) atomicMin(reinterpret_cast<unsigned long long*>(addr), (unsigned long long)f64_to_ordered(f)); break; }
        case W_MAX_F64: { double f = raw_to_f64(dtype, raw); if (valid && f == f) atomicMax(reinterpret_cast<unsigned long long*>(addr), (unsigned long long)f64_to_ordered(f)); break; }
        default: if (!valid) atomicAdd(reinterpret_cast<unsigned*>(addr), 1u); break;   // W_NULLCNT (< 2^32 per CTA)
    }
}


}  // namespace plb
