// sort_keys.cuh — the order-preserving key encoding shared by the sort (sort.cu) and the per-group quantiles (quantile.cu).
#pragma once
#include "common.cuh"
#include "dev_utils.cuh"

namespace plb {

// Unsigned key whose ascending order is the value order of reorder_cmp (polars-utils/src/sort.rs:113-128): ints by value,
// floats by tot_cmp (NaN == NaN and greatest, -0.0 == +0.0), Bool false < true.  8/16/32-bit types use the low 32 bits.
__device__ __forceinline__ uint64_t sort_value_key(const void* col, int64_t r, int dtype) {
    switch (dtype) {
        case BL_INT8: return (uint8_t)reinterpret_cast<const int8_t*>(col)[r] ^ 0x80u;           // flip the type's own sign bit:
        case BL_INT16: return (uint16_t)reinterpret_cast<const int16_t*>(col)[r] ^ 0x8000u;      // narrow ranges stay in few digits
        case BL_INT32: return (uint32_t)reinterpret_cast<const int32_t*>(col)[r] ^ 0x80000000u;
        case BL_INT64: return (uint64_t)reinterpret_cast<const int64_t*>(col)[r] ^ 0x8000000000000000ull;
        case BL_UINT8: return reinterpret_cast<const uint8_t*>(col)[r];
        case BL_UINT16: return reinterpret_cast<const uint16_t*>(col)[r];
        case BL_UINT32: return reinterpret_cast<const uint32_t*>(col)[r];
        case BL_UINT64: return reinterpret_cast<const uint64_t*>(col)[r];
        case BL_FLOAT32: {      // canonical (-0 -> +0, one NaN) then the order-preserving map; NaN lands above +inf
            const uint32_t u = (uint32_t)canonical_f32_bits(reinterpret_cast<const float*>(col)[r]);
            return (u >> 31) ? (uint32_t)~u : (u | 0x80000000u);
        }
        case BL_FLOAT64: {
            const uint64_t u = canonical_f64_bits(reinterpret_cast<const double*>(col)[r]);
            return (u >> 63) ? ~u : (u | 0x8000000000000000ull);
        }
        default: return bit_get(reinterpret_cast<const uint32_t*>(col), r) ? 1u : 0u;     // BL_BOOL: false < true
    }
}

}  // namespace plb
