// top_k.cu — the first k rows of the stable sort order, selected without sorting: an MSD radix select.
//
// Reference: top_k / bottom_k of one column polars-ops/src/chunked_array/top_k.rs:151-229 (select_nth_unstable: the
// order of the output and of ties is open; non-null values first, padded with nulls), top_k_by / bottom_k_by
// top_k.rs:231-297 and DataFrame.top_k / bottom_k through _arg_bottom_k
// polars-core/src/chunked_array/ops/sort/arg_bottom_k.rs:33-… (sorted output, tied rows in an open order), sort(...,
// limit = k) = the (0, k) slice of the stable order (polars-core/src/frame/mod.rs:1482-1486).  The device answer is the
// same everywhere: the first k rows of the stable order of op_arg_sort (sort.cu), returned as ascending row ids.
//
// Key.  The lexicographic key op_arg_sort sorts by, split into parts, most significant first: per `by` column its null
// rank (only with a validity bitmap; nulls_last: valid 0 / null 1) and its value key (sort_value_key, inverted if
// descending; null rows 0), then the row index.  The row index makes every key distinct, so "the first k keys" is one
// set and the stable tie rule is part of the key: the candidates left after the last column's digits are a tie run, and
// the row-index digits pick the first `need` of them in row order.
//
// State: a selection bitmap (n bits), `need` (rows still to choose) and the candidate set (rows whose decided digits
// equal the chosen prefix).
//   k_topk_andor  first, one read of every key part: its AND / OR over the rows (value parts: valid rows only).  Digits
//                 where AND == OR are the same in every row and never get a pass; keys with no varying digit at all
//                 select rows 0 .. k without any.
//   k_topk_pass   one per varying digit, most significant first, over the candidates: marks those whose previous digit
//                 is below the previous step's bucket, keeps the ones in that bucket, and builds the 256-bin histogram of
//                 the next digit over them (shared memory per CTA, then global bins).  The host reads the histogram back
//                 (1 KB) and picks the bucket b where the running count crosses `need`.  When the bucket holds exactly
//                 `need` rows, a last pass marks every candidate at or below b.
//   Large sets    a streaming pass over all n rows with a prefix test (every decided digit of every part is compared),
//                 so nothing but the bitmap words holding selected rows is written.
//   Small sets    once a bucket holds at most n / TK_LIST_DIV rows, the pass that keeps it also appends the kept row ids
//                 to a list (one atomic per warp), and every later pass runs over the list (and appends a shorter one).
//                 The list holds exactly the candidates, so list passes skip the prefix test; its order is open, and the
//                 result does not depend on it, since the row index is part of the key.
//   Tie step      after the last key digit, a candidate set too large for a list ties on the whole key: one streaming
//                 pass (topk_tie) writes it as a bitmap and mask_first_into selects its first `need` rows from per-tile
//                 counts, instead of a pass per row-index digit.
//   Output        op_mask_rows compacts the bitmap into ascending row ids.
// TK_LIST_DIV = 32 and the limit rule of op_arg_sort are measured (DESIGN.md §17, tools/bench_top_k.py T8-T10).
// Memory: n / 8 B of bitmap (twice with a tie step) plus the lists (at most 2 x 4n / TK_LIST_DIV B), no n-sized key buffers.
// Algorithmic bytes per streaming pass: the key bytes of every part with a decided digit plus the current part, per row.
#include "common.cuh"
#include "dev_utils.cuh"
#include "sort_keys.cuh"

namespace plb {

enum { TK_NULLS = 0, TK_VALUE = 1, TK_ROW = 2 };
struct TkPart {
    const void* col; const uint32_t* valid;
    int kind, dtype, descending, nulls_last;
    uint64_t width;          // all-ones over the part's key bits
    uint64_t mask, val;      // decided digits: a candidate has (key & mask) == val
};
constexpr int64_t TK_LIST_DIV = 32;      // candidate sets of at most n / TK_LIST_DIV rows run over a row-id list (DESIGN.md §17)
constexpr int TK_THREADS = 256;

__device__ __forceinline__ uint64_t tk_key(const TkPart& p, int64_t r) {
    if (p.kind == TK_ROW) return (uint64_t)r;
    const bool ok = p.valid == nullptr || bit_get(p.valid, r);
    if (p.kind == TK_NULLS) return (ok ? 0u : 1u) ^ (p.nulls_last ? 0u : 1u);
    if (!ok) return 0;
    const uint64_t k = sort_value_key(p.col, r, p.dtype);
    return (p.descending ? ~k : k) & p.width;
}

// AND / OR of one part's keys over every row (a value part: valid rows only, as k_sort_encode reduces them; null rows
// share key 0 and the null part orders them)
__global__ void __launch_bounds__(TK_THREADS) k_topk_andor(const TkPart* __restrict__ part, int64_t n, unsigned long long* __restrict__ andor) {
    const TkPart p = *part;
    uint64_t a = ~0ull, o = 0;
    for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < n; r += (int64_t)gridDim.x * blockDim.x) {
        if (p.kind == TK_VALUE && p.valid && !bit_get(p.valid, r)) continue;
        const uint64_t k = tk_key(p, r);
        a &= k; o |= k;
    }
    __shared__ unsigned long long s_and[TK_THREADS / 32], s_or[TK_THREADS / 32];
    const unsigned lane = lane_id(), warp = threadIdx.x >> 5;
    const uint32_t al = __reduce_and_sync(0xffffffffu, (uint32_t)a), ah = __reduce_and_sync(0xffffffffu, (uint32_t)(a >> 32));
    const uint32_t ol = __reduce_or_sync(0xffffffffu, (uint32_t)o), oh = __reduce_or_sync(0xffffffffu, (uint32_t)(o >> 32));
    if (lane == 0) { s_and[warp] = ((uint64_t)ah << 32) | al; s_or[warp] = ((uint64_t)oh << 32) | ol; }
    __syncthreads();
    if (threadIdx.x == 0) {
        unsigned long long ba = ~0ull, bo = 0;
        for (int w = 0; w < TK_THREADS / 32; w++) { ba &= s_and[w]; bo |= s_or[w]; }
        atomicAnd(&andor[0], ba); atomicOr(&andor[1], bo);
    }
}

// One step.  Rows: ids[0 .. m) (list mode) or 0 .. m (streaming).  A row is a candidate when every part in [0, n_test)
// matches its decided digits.  prev >= 0: the previous step's digit (part prev, shift prev_shift) splits the candidates:
// below prev_b (or at it, when mark_le) -> selected, equal -> kept.  cand_out (streaming only): the kept rows as a
// bitmap.  cur >= 0: the kept rows' histogram of the digit at cur_shift of part cur; with list_out, their row ids are
// appended.
__global__ void __launch_bounds__(TK_THREADS) k_topk_pass(const TkPart* __restrict__ parts, int n_test, int prev, int prev_shift, int prev_b, int mark_le,
                                                          int cur, int cur_shift, const uint32_t* __restrict__ ids, int64_t m, uint32_t* __restrict__ sel,
                                                          uint32_t* __restrict__ cand_out, uint32_t* __restrict__ hist, uint32_t* __restrict__ list_out,
                                                          unsigned long long* __restrict__ list_n) {
    __shared__ uint32_t s_hist[256];
    for (int i = threadIdx.x; i < 256; i += blockDim.x) s_hist[i] = 0;
    __syncthreads();
    const unsigned lane = lane_id(), warp = threadIdx.x >> 5;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    // every lane of a warp runs the same iterations (ballots); in streaming mode a warp's 32 rows are one bitmap word
    for (int64_t base = (int64_t)blockIdx.x * blockDim.x + warp * 32; base < m; base += stride) {
        const int64_t i = base + lane;
        bool cand = i < m;
        const int64_t r = !cand ? 0 : ids ? (int64_t)ids[i] : i;
        for (int j = 0; j < n_test && cand; j++) {
            const TkPart& p = parts[j];
            if (p.mask) cand = (tk_key(p, r) & p.mask) == p.val;
        }
        uint64_t ck = 0;
        bool mark = false;
        if (prev >= 0 && cand) {
            ck = tk_key(parts[prev], r);
            const int d = (int)((ck >> prev_shift) & 0xFF);
            mark = mark_le ? d <= prev_b : d < prev_b;
            cand = !mark_le && d == prev_b;
        }
        const unsigned marks = __ballot_sync(0xffffffffu, mark);
        if (marks) {
            if (ids) { if (mark) atomicOr(&sel[r >> 5], 1u << (r & 31)); }
            else if (lane == 0) sel[base >> 5] |= marks;      // this warp owns the word in this pass
        }
        if (cand_out) {
            const unsigned keep = __ballot_sync(0xffffffffu, cand);
            if (lane == 0) cand_out[base >> 5] = keep;
        }
        if (cur < 0) continue;
        if (cand && cur != prev) ck = tk_key(parts[cur], r);
        const uint32_t d = cand ? (uint32_t)((ck >> cur_shift) & 0xFF) : 256u;
        const unsigned peers = __match_any_sync(0xffffffffu, d);      // one shared atomic per distinct digit of the warp
        if (cand && (peers & lanemask_lt()) == 0) atomicAdd(&s_hist[d], (uint32_t)__popc(peers));
        if (list_out) {
            const unsigned keep = __ballot_sync(0xffffffffu, cand);
            unsigned long long at = 0;
            if (lane == 0 && keep) at = atomicAdd(list_n, (unsigned long long)__popc(keep));
            at = __shfl_sync(0xffffffffu, at, 0);
            if (cand) list_out[at + __popc(keep & lanemask_lt())] = (uint32_t)r;
        }
    }
    if (cur < 0) return;
    __syncthreads();
    for (int i = threadIdx.x; i < 256; i += blockDim.x)
        if (s_hist[i]) atomicAdd(&hist[i], s_hist[i]);
}

// a measurement knob (read per call, as BL_QUANTILE_GLOBAL is): BL_TOPK_LIST_DIV overrides TK_LIST_DIV
static int64_t topk_list_div() { const char* e = getenv("BL_TOPK_LIST_DIV"); const long v = e ? atol(e) : 0; return v >= 1 ? v : TK_LIST_DIV; }

DevCol op_top_k(const std::vector<DevCol>& by, const std::vector<int>& flags, int64_t k) {
    PLB_REQUIRE(!by.empty(), BL_ERR_INVALID, "top_k: no key column");
    PLB_REQUIRE(flags.size() == by.size(), BL_ERR_INVALID, "top_k: one flag word per key column");
    PLB_REQUIRE(k >= 0, BL_ERR_INVALID, "top_k: k must be >= 0 (got " + std::to_string(k) + ")");
    const int64_t n = by[0].len;
    for (auto& c : by) {
        PLB_REQUIRE(c.len == n, BL_ERR_INVALID, "top_k: key columns differ in length (" + std::to_string(c.len) + " != " + std::to_string(n) + ")");
        PLB_REQUIRE(sortable_dtype(c.dtype), BL_ERR_UNSUPPORTED, std::string("top_k: key dtype ") + dtype_name(c.dtype) + " is not supported");
    }
    PLB_REQUIRE(n <= (int64_t)0xFFFFFFFFll, BL_ERR_UNSUPPORTED, "top_k: more than 2^32 - 1 rows (IdxSize is u32)");
    auto iota = [](int64_t len) { DevCol out = make_col(BL_UINT32, len, false); iota_u32(as<uint32_t>(out.values), len, 0); return out; };
    if (k >= n) return iota(n);
    if (k == 0) return make_col(BL_UINT32, 0, false);
    const int64_t list_max = n / topk_list_div();

    std::vector<TkPart> parts;
    std::vector<int> top_shift;      // the shift of each part's most significant digit
    for (size_t c = 0; c < by.size(); c++) {
        const DevCol& col = by[c];
        const int desc = (flags[c] & BL_SORT_DESCENDING) != 0, nl = (flags[c] & BL_SORT_NULLS_LAST) != 0;
        if (col.validity) { parts.push_back({col.v(), col.vm(), TK_NULLS, col.dtype, desc, nl, 1, 0, 0}); top_shift.push_back(0); }
        const bool wide = dtype_size(col.dtype) == 8;
        parts.push_back({col.v(), col.vm(), TK_VALUE, col.dtype, desc, nl, wide ? ~0ull : 0xFFFFFFFFull, 0, 0});
        top_shift.push_back(wide ? 56 : 24);
    }
    const int n_key_parts = (int)parts.size();
    const int row_bits = bits_for((uint64_t)(n - 1));
    parts.push_back({nullptr, nullptr, TK_ROW, 0, 0, 0, row_bits == 64 ? ~0ull : (1ull << row_bits) - 1, 0, 0});
    top_shift.push_back((row_bits - 1) / 8 * 8);

    DevPtr sel = dev_alloc(bitmap_bytes(n)), dparts = dev_alloc(parts.size() * sizeof(TkPart));
    DevPtr scratch = dev_alloc(256 * 4 + 16 * parts.size() + 8);      // hist, AND / OR per part, list length
    uint32_t* hist = as<uint32_t>(scratch);
    unsigned long long* andor = reinterpret_cast<unsigned long long*>((char*)scratch->p + 1024);
    unsigned long long* list_n = andor + 2 * parts.size();
    PLB_CUDA(cudaMemcpyAsync(dparts->p, parts.data(), parts.size() * sizeof(TkPart), cudaMemcpyHostToDevice, ctx().stream));
    // every part's AND / OR in one read of the key columns: the digits no pass has to look at
    dev_memset(andor, 0xFF, 16 * n_key_parts);
    for (int p = 0; p < n_key_parts; p++) {
        dev_memset(andor + 2 * p + 1, 0, 8);
        PLB_LAUNCH("topk_andor", k_topk_andor, grid_for(n, TK_THREADS), TK_THREADS, 0, as<TkPart>(dparts) + p, n, andor + 2 * p);
    }
    std::vector<uint64_t> ao(2 * n_key_parts);
    PLB_CUDA(cudaMemcpyAsync(ao.data(), andor, 16 * n_key_parts, cudaMemcpyDeviceToHost, ctx().stream));
    PLB_CUDA(cudaStreamSynchronize(ctx().stream));
    std::vector<std::pair<int, int>> digits;      // (part, shift), most significant first: the varying key digits, then the row index's
    for (int p = 0; p < n_key_parts; p++) {
        const uint64_t vary = (ao[2 * p] & ~ao[2 * p + 1]) ? 0 : ao[2 * p] ^ ao[2 * p + 1];      // AND not in OR: no row reduced
        for (int sh = top_shift[p]; sh >= 0; sh -= 8)
            if ((vary >> sh) & 0xFF) digits.push_back({p, sh});
    }
    const size_t n_key_digits = digits.size();
    for (int sh = top_shift.back(); sh >= 0; sh -= 8) digits.push_back({n_key_parts, sh});

    dev_memset(sel->p, 0, bitmap_bytes(n));
    DevPtr ids;             // the candidate list (nullptr: streaming over all rows)
    int64_t m = n;          // rows a pass runs over
    int64_t need = k, count = n;      // rows still to choose; candidates
    int prev = -1, prev_shift = 0, prev_b = 0;
    uint32_t h[256];
    for (size_t di = 0;; di++) {
        if (di >= n_key_digits && !ids && count > list_max) {
            // the tie step: the candidates tie on the whole key and are too many for a list; take the first `need` of them
            // in row order.  Nothing narrowed the rows at all: those are rows 0 .. need.
            if (count == n) return iota(need);
            DevPtr cand = dev_alloc(bitmap_bytes(n));
            PLB_CUDA(cudaMemcpyAsync(dparts->p, parts.data(), parts.size() * sizeof(TkPart), cudaMemcpyHostToDevice, ctx().stream));
            PLB_LAUNCH("topk_tie", k_topk_pass, grid_for(n, TK_THREADS), TK_THREADS, 0, as<TkPart>(dparts), prev + 1, prev, prev_shift, prev_b, 0, -1, 0,
                       nullptr, n, as<uint32_t>(sel), as<uint32_t>(cand), hist, nullptr, list_n);
            mask_first_into(as<uint32_t>(cand), n, need, as<uint32_t>(sel));
            return op_mask_rows(as<uint32_t>(sel), n);
        }
        PLB_REQUIRE(di < digits.size(), BL_ERR_CUDA, "top_k: the selection did not converge");      // the row index is unique
        const int cur = digits[di].first, cur_shift = digits[di].second;
        PLB_CUDA(cudaMemcpyAsync(dparts->p, parts.data(), parts.size() * sizeof(TkPart), cudaMemcpyHostToDevice, ctx().stream));
        dev_memset(hist, 0, 1024);
        dev_memset(list_n, 0, 8);
        DevPtr list_out;
        if (count <= list_max && count < m) list_out = dev_alloc((size_t)count * 4);
        PLB_LAUNCH(ids ? "topk_pass_list" : "topk_pass", k_topk_pass, grid_for(m, TK_THREADS), TK_THREADS, 0, as<TkPart>(dparts), ids ? 0 : cur + 1, prev, prev_shift,
                   prev_b, 0, cur, cur_shift, as<uint32_t>(ids), m, as<uint32_t>(sel), nullptr, hist, as<uint32_t>(list_out), list_n);
        PLB_CUDA(cudaMemcpyAsync(h, hist, sizeof h, cudaMemcpyDeviceToHost, ctx().stream));
        PLB_CUDA(cudaStreamSynchronize(ctx().stream));
        if (list_out) { ids = list_out; m = count; }
        if (prev >= 0) { parts[prev].mask |= 0xFFull << prev_shift; parts[prev].val |= (uint64_t)prev_b << prev_shift; }
        int64_t below = 0;
        int b = 0;
        while (below + h[b] < need) below += h[b++];
        need -= below;
        count = h[b];
        prev = cur; prev_shift = cur_shift; prev_b = b;
        if (count == need) break;
    }
    // the last bucket is taken whole: mark every candidate at or below it
    PLB_CUDA(cudaMemcpyAsync(dparts->p, parts.data(), parts.size() * sizeof(TkPart), cudaMemcpyHostToDevice, ctx().stream));
    PLB_LAUNCH(ids ? "topk_mark_list" : "topk_mark", k_topk_pass, grid_for(m, TK_THREADS), TK_THREADS, 0, as<TkPart>(dparts), ids ? 0 : prev + 1, prev, prev_shift, prev_b, 1, -1, 0,
               as<uint32_t>(ids), m, as<uint32_t>(sel), nullptr, hist, nullptr, list_n);
    return op_mask_rows(as<uint32_t>(sel), n);
}

}  // namespace plb

// ================================================================================ C ABI
using namespace plb;
extern "C" {

bl_status bl_top_k(const bl_sort_key* by, int32_t n_by, int64_t k, int32_t out_location, bl_column* out_idx) {
    BL_TRY
    PLB_REQUIRE(out_idx != nullptr, BL_ERR_INVALID, "top_k: null output");
    PLB_REQUIRE(by != nullptr && n_by >= 1, BL_ERR_INVALID, "top_k: no key column");
    PLB_REQUIRE(k >= 0, BL_ERR_INVALID, "top_k: k must be >= 0 (got " + std::to_string(k) + ")");
    std::vector<DevCol> keys; std::vector<int> fl;
    import_sort_key_list(by, n_by, "top_k", keys, fl);
    DevCol ids = op_top_k(keys, fl, k);
    export_column(ids, out_location, out_idx);
    BL_CATCH
}

}  // extern "C"
