// gather.cu — K4: out[i] = values[idx[i]] for c columns sharing one index vector.
//
// Reference: take_primitive_unchecked polars-compute/src/gather/primitive.rs:9-78 (null index ->
// T::default() and a null slot; source validity is gathered bitwise), bounds check
// polars-core/src/chunked_array/ops/gather.rs:14-39, column-parallel DataFrame::take_unchecked_impl
// polars-core/src/frame/mod.rs:1256-1294.
//
// Design: each thread owns 4 consecutive output rows: one 128-bit index load, 4 independent
// random 8-byte (or 4-byte) reads in flight, one or two 128-bit streaming stores.  Output validity
// nibbles are merged to 32-bit words with 3 xor-shuffles.  Algorithmic bytes: 4 + 8 + 8 per output
// row and column; bound: random-sector HBM/L2 reads.
#include "common.cuh"
#include "dev_utils.cuh"

namespace plb {

constexpr int G_MAX_COLS = 8;
struct GatherCol { const void* in; void* out; const uint32_t* vin; uint32_t* vout; int elem; int pad; };
struct GatherArgs { GatherCol c[G_MAX_COLS]; int ncols; };

template <bool NULLABLE>
__global__ void __launch_bounds__(256) k_gather(GatherArgs args, const uint32_t* __restrict__ idx, const uint32_t* __restrict__ idx_valid, int64_t m) {
    const int64_t nquads = (m + 3) / 4;
    for (int64_t q = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; q < ((nquads + 31) / 32) * 32; q += (int64_t)gridDim.x * blockDim.x) {
        const int64_t r0 = q * 4;
        uint32_t ix[4] = {0, 0, 0, 0};
        bool ok[4] = {false, false, false, false};
        if (r0 + 3 < m) {
            uint4 t = ld_stream_u32x4(idx + r0);
            ix[0] = t.x; ix[1] = t.y; ix[2] = t.z; ix[3] = t.w;
            ok[0] = ok[1] = ok[2] = ok[3] = true;
        } else {
#pragma unroll
            for (int k = 0; k < 4; k++) if (r0 + k < m) { ix[k] = idx[r0 + k]; ok[k] = true; }
        }
        // the sentinel is never dereferenced, even on the path for index columns known to hold no nulls
#pragma unroll
        for (int k = 0; k < 4; k++) {
            if (ok[k] && ix[k] == BL_IDX_NULL) ok[k] = false;
            if (NULLABLE && ok[k] && idx_valid != nullptr && !bit_get(idx_valid, r0 + k)) ok[k] = false;
        }
        for (int c = 0; c < args.ncols; c++) {
            const GatherCol col = args.c[c];
            if (col.elem == 8) {
                uint64_t v[4];
#pragma unroll
                for (int k = 0; k < 4; k++) v[k] = ok[k] ? __ldg(reinterpret_cast<const uint64_t*>(col.in) + ix[k]) : 0ull;
                if (r0 + 3 < m) {
                    st_stream_u64x2(reinterpret_cast<uint64_t*>(col.out) + r0, make_ulonglong2(v[0], v[1]));
                    st_stream_u64x2(reinterpret_cast<uint64_t*>(col.out) + r0 + 2, make_ulonglong2(v[2], v[3]));
                } else {
#pragma unroll
                    for (int k = 0; k < 4; k++) if (r0 + k < m) reinterpret_cast<uint64_t*>(col.out)[r0 + k] = v[k];
                }
            } else {
                uint32_t v[4];
#pragma unroll
                for (int k = 0; k < 4; k++) v[k] = ok[k] ? __ldg(reinterpret_cast<const uint32_t*>(col.in) + ix[k]) : 0u;
                if (r0 + 3 < m) st_stream_u32x4(reinterpret_cast<uint32_t*>(col.out) + r0, make_uint4(v[0], v[1], v[2], v[3]));
                else {
#pragma unroll
                    for (int k = 0; k < 4; k++) if (r0 + k < m) reinterpret_cast<uint32_t*>(col.out)[r0 + k] = v[k];
                }
            }
            if (col.vout != nullptr) {
                uint32_t nib = 0;
#pragma unroll
                for (int k = 0; k < 4; k++) {
                    bool valid = ok[k] && (col.vin == nullptr || bit_get(col.vin, ix[k]));
                    nib |= (valid ? 1u : 0u) << k;
                }
                uint32_t w = nib << (4 * (lane_id() & 7));
                w |= __shfl_xor_sync(0xffffffffu, w, 1);
                w |= __shfl_xor_sync(0xffffffffu, w, 2);
                w |= __shfl_xor_sync(0xffffffffu, w, 4);
                if ((lane_id() & 7) == 0 && r0 < m) col.vout[q >> 3] = w;
            }
        }
    }
}

// flags[0]: a non-null index >= len; flags[1]: a non-null slot holds the BL_IDX_NULL sentinel
__global__ void k_check_idx(const uint32_t* __restrict__ idx, const uint32_t* __restrict__ idx_valid, int64_t m, uint32_t len, int* flags) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < m; i += (int64_t)gridDim.x * blockDim.x) {
        if (idx_valid != nullptr && !bit_get(idx_valid, i)) continue;
        uint32_t x = idx[i];
        if (x == BL_IDX_NULL) flags[1] = 1;
        else if (x >= len) flags[0] = 1;
    }
}

void op_gather(const std::vector<DevCol>& cols, const DevCol& idx, bool check_bounds, std::vector<DevCol>& outs, bool find_sentinel) {
    PLB_REQUIRE(idx.dtype == BL_UINT32, BL_ERR_DTYPE, "gather: idx must be BL_UINT32 (IdxSize)");
    const int64_t m = idx.len;
    outs.clear();
    for (auto& c : cols)
        PLB_REQUIRE(dtype_size(c.dtype) == 8 || dtype_size(c.dtype) == 4, BL_ERR_UNSUPPORTED, std::string("gather: dtype ") + dtype_name(c.dtype) + " is outside the hot path");
    // nullable path when the idx column may carry nulls: a bitmap, a non-zero null count, or the BL_IDX_NULL sentinel.
    // An index column without a bitmap that claims no nulls may still hold the sentinel: the bounds check finds it in
    // the same pass, and callers that cannot rule it out ask for the scan (find_sentinel).
    bool nullable = idx.validity != nullptr || idx.null_count != 0;
    if (m > 0 && (check_bounds || (find_sentinel && !nullable))) {
        int64_t len = 0xFFFFFFFFll;                  // no index is out of range for the sentinel scan alone
        if (check_bounds)
            for (auto& c : cols) len = std::min<int64_t>(len, c.len);
        DevPtr flags = dev_alloc(8); dev_memset(flags->p, 0, 8);
        PLB_LAUNCH("k4_check_idx", k_check_idx, grid_for(m, 256), 256, 0, (const uint32_t*)idx.v(), idx.vm(), m, (uint32_t)len, as<int>(flags));
        int f[2];
        PLB_CUDA(cudaMemcpyAsync(f, flags->p, 8, cudaMemcpyDeviceToHost, ctx().stream));
        PLB_CUDA(cudaStreamSynchronize(ctx().stream));
        if (f[0]) fail(BL_ERR_BOUNDS, "gather: index out of bounds");
        nullable |= f[1] != 0;
    }
    for (auto& c : cols) {
        DevCol o = make_col(c.dtype, m, nullable || c.validity != nullptr);
        outs.push_back(o);
    }
    if (m == 0) return;
    for (size_t base = 0; base < cols.size(); base += G_MAX_COLS) {
        GatherArgs a; memset(&a, 0, sizeof a);
        a.ncols = (int)std::min<size_t>(G_MAX_COLS, cols.size() - base);
        for (int i = 0; i < a.ncols; i++) {
            a.c[i].in = cols[base + i].v(); a.c[i].out = outs[base + i].values->p;
            a.c[i].vin = cols[base + i].vm(); a.c[i].vout = as<uint32_t>(outs[base + i].validity);
            a.c[i].elem = dtype_size(cols[base + i].dtype);
        }
        int grid = grid_for((m + 3) / 4, 256);
        if (nullable) PLB_LAUNCH("k4_gather", (k_gather<true>), grid, 256, 0, a, (const uint32_t*)idx.v(), idx.vm(), m);
        else PLB_LAUNCH("k4_gather", (k_gather<false>), grid, 256, 0, a, (const uint32_t*)idx.v(), idx.vm(), m);
    }
}

}  // namespace plb
