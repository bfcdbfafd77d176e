// dev_utils.cuh — device-side scalar semantics shared by all kernels.
// Each helper cites the reference rule it restates (paths relative to /root/reference/crates).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace plb {

// ---- hashing / partitioning: polars-utils/src/hashing.rs:62-69 (hash_to_partition),
//      :123-147 (DirtyHash: k * RANDOM_ODD), null -> hash 0 (:183-187)
#define PLB_RANDOM_ODD 0x55fbfd6bfc5458e9ULL
__host__ __device__ __forceinline__ uint64_t dirty_hash(uint64_t k) { return k * PLB_RANDOM_ODD; }
__device__ __forceinline__ uint32_t hash_to_partition(uint64_t h, uint32_t n) { return (uint32_t)__umul64hi(h, (uint64_t)n); }
// Slot hash of every hash TABLE (group_by tables and buckets, join tables).  It must not be the partition hash: rows that
// reach a GPU through hash_to_partition(dirty_hash(key), P) all carry the same top bits of key * RANDOM_ODD, so a table
// slotted on those bits would use 1/P of its slots (measured: the 2-GPU partitioned join on sparse keys ran 1000x slower
// on exactly full buckets).  The reference has the same separation: hash_to_partition(dirty_hash) picks the thread,
// hashbrown + foldhash place the key inside the thread's table.
__host__ __device__ __forceinline__ uint64_t table_hash(uint64_t k) { return (k ^ (k >> 31)) * 0x9E3779B97F4A7C15ULL; }

// ---- float canonicalisation for keys: polars-utils/src/total_ord.rs:37-47 (-0 -> +0, one NaN)
__device__ __forceinline__ uint64_t canonical_f64_bits(double x) {
    double z = x + 0.0;
    return (z != z) ? 0x7ff8000000000000ULL : (uint64_t)__double_as_longlong(z);
}
__device__ __forceinline__ uint64_t canonical_f32_bits(float x) {
    float z = x + 0.0f;
    return (z != z) ? 0x7fc00000ULL : (uint64_t)__float_as_uint(z);
}

// ---- order-preserving map f64 -> u64 (for atomicMin/Max on floats): all non-NaN values map
//      inside [T(-inf), T(+inf)]; NaN is never inserted (min/max ignore NaN,
//      polars-utils/src/min_max.rs:96-108)
__device__ __forceinline__ uint64_t f64_to_ordered(double x) {
    uint64_t u = (uint64_t)__double_as_longlong(x);
    return (u >> 63) ? ~u : (u | 0x8000000000000000ULL);
}
__device__ __forceinline__ double ordered_to_f64(uint64_t u) {
    u = (u >> 63) ? (u & 0x7fffffffffffffffULL) : ~u;
    return __longlong_as_double((long long)u);
}

__host__ __device__ __forceinline__ int dtype_size_dev(int dt) {
    // BL_INT8=0 INT16=1 INT32=2 INT64=3 UINT8=4 UINT16=5 UINT32=6 UINT64=7 FLOAT32=8 FLOAT64=9
    return dt == 9 ? 8 : dt == 8 ? 4 : (1 << (dt & 3));
}

// ---- bitmaps (LSB-first; polars-arrow/src/bitmap/utils/mod.rs:42-46); device bitmaps are
//      32-bit-word arrays with bit offset 0
__device__ __forceinline__ bool bit_get(const uint32_t* bm, int64_t i) { return (bm[i >> 5] >> (i & 31)) & 1u; }
// a value of column v at row r; BL_BOOL values are bit-packed (v NULL: every row counts as set, for CUM_COUNT)
struct BoolBit { bool b; };
template <typename In> __device__ __forceinline__ In load_in(const void* v, int64_t r) { return __ldg(reinterpret_cast<const In*>(v) + r); }
template <> __device__ __forceinline__ BoolBit load_in<BoolBit>(const void* v, int64_t r) { return BoolBit{v == nullptr || bit_get(reinterpret_cast<const uint32_t*>(v), r)}; }

// spread the 32 bits of x to the even bit positions of a 64-bit word
__device__ __forceinline__ uint64_t spread_bits(uint32_t v) {
    uint64_t x = v;
    x = (x | (x << 16)) & 0x0000FFFF0000FFFFULL;
    x = (x | (x << 8)) & 0x00FF00FF00FF00FFULL;
    x = (x | (x << 4)) & 0x0F0F0F0F0F0F0F0FULL;
    x = (x | (x << 2)) & 0x3333333333333333ULL;
    x = (x | (x << 1)) & 0x5555555555555555ULL;
    return x;
}

// ---- streaming 128-bit loads/stores (read-once inputs: evict-first so the L2-resident hash
//      table is not displaced by the scan)
__device__ __forceinline__ ulonglong2 ld_stream_u64x2(const void* p) { return __ldcs(reinterpret_cast<const ulonglong2*>(p)); }
__device__ __forceinline__ uint4 ld_stream_u32x4(const void* p) { return __ldcs(reinterpret_cast<const uint4*>(p)); }
__device__ __forceinline__ uint2 ld_stream_u32x2(const void* p) { return __ldcs(reinterpret_cast<const uint2*>(p)); }
__device__ __forceinline__ void st_stream_u64x2(void* p, ulonglong2 v) { __stcs(reinterpret_cast<ulonglong2*>(p), v); }
__device__ __forceinline__ void st_stream_u32x4(void* p, uint4 v) { __stcs(reinterpret_cast<uint4*>(p), v); }

__device__ __forceinline__ unsigned lane_id() { return threadIdx.x & 31u; }
__device__ __forceinline__ unsigned lanemask_lt() { unsigned m; asm("mov.u32 %0, %%lanemask_lt;" : "=r"(m)); return m; }

// ---- TMA bulk copies (cp.async.bulk, SASS UBLKCP) and mbarriers: contiguous tiles between global and shared memory
//      without going through registers.  Sizes and both addresses must be multiples of 16 bytes.
__device__ __forceinline__ unsigned smem_u32(const void* p) { return (unsigned)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, unsigned count) { asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory"); }
__device__ __forceinline__ void mbar_fence_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, unsigned bytes) { asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory"); }
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) { asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory"); }
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, unsigned parity) {
    unsigned ok;
    asm volatile("{\n .reg .pred p;\n mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n selp.u32 %0, 1, 0, p;\n}" : "=r"(ok) : "r"(smem_u32(bar)), "r"(parity) : "memory");
    return ok != 0;
}
// global -> shared, completion signalled on the mbarrier (complete_tx::bytes)
__device__ __forceinline__ void bulk_g2s(void* sdst, const void* gsrc, unsigned bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(sdst)), "l"(gsrc), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}
// shared -> global, tracked by the issuing thread's bulk async-group
__device__ __forceinline__ void bulk_s2g(void* gdst, const void* ssrc, unsigned bytes) {
    asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(gdst), "r"(smem_u32(ssrc)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
__device__ __forceinline__ void bulk_wait_read0() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }     // sources may be overwritten
__device__ __forceinline__ void bulk_wait0() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }               // writes are complete
__device__ __forceinline__ void fence_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }      // generic-proxy smem writes -> visible to TMA
__device__ __forceinline__ void named_bar_sync(int id, int nthreads) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory"); }

// ---- integer floor div / mod: polars-utils/src/floor_divmod.rs:38-66 (Python semantics;
//      (0,0) when the divisor is 0; wrapping for MIN / -1)
template <typename T> struct make_unsigned_t;
template <> struct make_unsigned_t<int64_t> { using type = uint64_t; };
template <> struct make_unsigned_t<int32_t> { using type = uint32_t; };
template <> struct make_unsigned_t<uint64_t> { using type = uint64_t; };
template <> struct make_unsigned_t<uint32_t> { using type = uint32_t; };

template <typename T> __device__ __forceinline__ void floor_divmod(T a, T b, T& d, T& m) {
    using U = typename make_unsigned_t<T>::type;
    if (b == 0) { d = 0; m = 0; return; }
    if (T(-1) < T(0)) {  // signed
        T q, r;
        if (b == T(-1)) { q = (T)((U)0 - (U)a); r = 0; }
        else { q = a / b; r = a % b; }
        if (r != 0 && ((a < 0) != (b < 0))) { q -= 1; r += b; }
        d = q; m = r;
    } else { d = a / b; m = a % b; }
}

}  // namespace plb
