// string_match.cu — predicates over string / binary columns (DESIGN.md §19): comparisons, starts_with / ends_with /
// contains, SQL LIKE, and the filter that materialises a string column under a mask.
//
// Reference semantics (paths relative to /root/reference/crates):
//   comparisons   polars-compute/src/comparisons/binary.rs:8-70 — unsigned byte order, a proper prefix first; the view
//                 kernels (comparisons/view.rs) decide most rows on a 4-byte inline prefix.  Null on either side: null;
//                 eq_missing / ne_missing: null == null.
//   starts_with / ends_with / contains   polars-ops/src/chunked_array/binary/namespace.rs:58-125 (memchr::memmem::find),
//                 strings/namespace.rs:174-200, 348-353 (contains_literal: the same bytes for a valid UTF-8 needle).
//   LIKE          polars-sql/src/sql_expr.rs:435-479 (visit_like): the regex ^(?s)<escaped pattern, % -> .*, _ -> .>$.
//
// Kernels (every output is a BL_BOOL bitmap written one ballot per 32 rows, validity = AND of the input validities):
//   k_str_rows<KIND>   one thread per row; a scalar pattern is staged in shared memory.  Compare / starts_with decide on
//                      an 8-byte big-endian prefix and read further only on a tie; LIKE runs a bit-parallel NFA (extended
//                      Shift-And) in one 64-bit word; contains with a per-row (or over-long) needle searches naively.
//   k_str_tile_rows    the byte-parallel contains plan: the first row of every data tile (one binary search per tile)
//   k_str_scan         one CTA per data tile + (m - 1) halo bytes staged with 16-byte loads; every position is tested on
//                      its first four bytes, then compared; a hit at byte p sets its row's bit when p + m <= row end
//   k_str_scan_finish  validity and NOT over the hit bitmap
// bl_string_filter is op_mask_rows (filter.cu) + op_string_gather (strings.cu): no kernel of its own.
//
// A single device chunk is read in place (offsets, bytes and validity at its bit offset): the kernels read only bytes in
// [offsets[0], offsets[n]) and never past the caller's buffer.  Host and multi-chunk inputs go through import_string.
#include <algorithm>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

#include "common.cuh"
#include "strings.cuh"

namespace plb {

enum { SM_CMP = 0, SM_STARTS = 1, SM_ENDS = 2, SM_CONTAINS = 3, SM_LIKE = 4 };
constexpr int SM_THREADS = 256;
constexpr int SM_PAT_SMEM = 16384;       // scalar patterns up to this many bytes are staged in shared memory
constexpr int SCAN_TILE = 8192;          // data bytes per tile of the byte-parallel plan
constexpr int SCAN_HALO = 512;           // the longest needle the byte-parallel plan takes (m - 1 halo bytes)
constexpr int LIKE_MAX_STATES = 63;      // literal bytes + '_' of a LIKE pattern (one 64-bit NFA word)
// the average row length (bytes) from which contains with a scalar needle takes the byte-parallel plan (DESIGN.md §19)
constexpr double SCAN_MIN_ROW_BYTES = 64.0;

// a string column as the kernels read it: absolute offsets into `data`, validity bits from bit `vbit` (or none)
struct StrArg {
    const int64_t* off = nullptr;
    const uint8_t* data = nullptr;
    const uint8_t* valid = nullptr;
    int64_t vbit = 0;
};
__device__ __forceinline__ bool str_valid(const StrArg& s, int64_t r) {
    if (s.valid == nullptr) return true;
    const int64_t b = s.vbit + r;
    return (s.valid[b >> 3] >> (b & 7)) & 1;
}
// up to 8 leading bytes as a big-endian word, zero-padded
__device__ __forceinline__ uint64_t prefix_be8(const uint8_t* p, int64_t l) {
    uint64_t w = 0;
    const int k = l < 8 ? (int)l : 8;
    for (int i = 0; i < k; i++) w |= (uint64_t)p[i] << (56 - 8 * i);
    return w;
}
// lexicographic unsigned-byte order, a proper prefix first; pa / pb: prefix_be8 of a / b
__device__ __forceinline__ int str_order(const uint8_t* a, int64_t la, uint64_t pa, const uint8_t* b, int64_t lb, uint64_t pb) {
    if (pa != pb) return pa < pb ? -1 : 1;
    const int64_t l = la < lb ? la : lb;
    for (int64_t i = 8; i < l; i++)
        if (a[i] != b[i]) return a[i] < b[i] ? -1 : 1;
    return (la > lb) - (la < lb);
}
__device__ __forceinline__ bool cmp_holds(int op, int c) {
    switch (op) {
        case BL_CMP_EQ: return c == 0;
        case BL_CMP_NE: return c != 0;
        case BL_CMP_LT: return c < 0;
        case BL_CMP_LE: return c <= 0;
        case BL_CMP_GT: return c > 0;
        default: return c >= 0;
    }
}
__device__ __forceinline__ bool bytes_eq(const uint8_t* a, const uint8_t* b, int64_t m) {
    for (int64_t i = 0; i < m; i++)
        if (a[i] != b[i]) return false;
    return true;
}
__device__ __forceinline__ bool find_naive(const uint8_t* s, int64_t l, const uint8_t* p, int64_t m) {
    if (m == 0) return true;
    const uint8_t p0 = p[0];
    for (int64_t i = 0; i + m <= l; i++)
        if (s[i] == p0 && bytes_eq(s + i + 1, p + 1, m - 1)) return true;
    return false;
}

struct RowsArgs {
    StrArg col, pat;            // pat: the per-row pattern column (pat_rows)
    const uint8_t* scalar = nullptr;      // else the scalar pattern's bytes
    int64_t n = 0;
    int op = 0, missing = 0, negate = 0, pat_rows = 0, pat_null = 0;
    int64_t m = 0;              // scalar pattern length
    uint64_t pprefix = 0;       // prefix_be8 of the scalar pattern
    const uint64_t* like_tab = nullptr;   // LIKE: B[256] then L[256]
    int like_k = 0, like_tail_any = 0;
    uint32_t* out = nullptr;
    uint32_t* out_valid = nullptr;        // nullptr: the result has no nulls
};

template <int KIND>
__global__ void __launch_bounds__(SM_THREADS) k_str_rows(RowsArgs a) {
    extern __shared__ uint64_t s_dyn[];
    const uint8_t* pat = nullptr;       // the scalar pattern (shared memory when it fits)
    uint64_t* s_tab = s_dyn;
    if (KIND == SM_LIKE) {
        for (int i = threadIdx.x; i < 512; i += blockDim.x) s_tab[i] = a.like_tab[i];
        __syncthreads();
    } else if (!a.pat_rows && !a.pat_null) {
        const uint8_t* g = a.scalar;
        if (a.m <= SM_PAT_SMEM) {
            uint8_t* s = reinterpret_cast<uint8_t*>(s_dyn);
            for (int64_t i = threadIdx.x; i < a.m; i += blockDim.x) s[i] = g[i];
            __syncthreads();
            pat = s;
        } else pat = g;
    }
    const int lane = threadIdx.x & 31;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i0 = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) & ~31ll; i0 < a.n; i0 += stride) {
        const int64_t r = i0 + lane;
        bool v = false, res = false;
        if (r < a.n) {
            const bool vc = str_valid(a.col, r);
            const bool vp = a.pat_rows ? str_valid(a.pat, r) : !a.pat_null;
            if (KIND == SM_CMP && a.missing) {
                v = true;
                if (!vc || !vp) res = (vc == vp) == (a.op == BL_CMP_EQ);
            } else v = vc && vp;
            if (v && (KIND != SM_CMP || !a.missing || (vc && vp))) {
                const int64_t o = a.col.off[r], l = a.col.off[r + 1] - o;
                const uint8_t* s = a.col.data + o;
                const uint8_t* p = pat;
                int64_t m = a.m;
                if (a.pat_rows) { const int64_t po = a.pat.off[r]; m = a.pat.off[r + 1] - po; p = a.pat.data + po; }
                if (KIND == SM_CMP) {
                    if ((a.op == BL_CMP_EQ || a.op == BL_CMP_NE) && l != m) res = a.op == BL_CMP_NE;
                    else {
                        const uint64_t pp = a.pat_rows ? prefix_be8(p, m) : a.pprefix;
                        res = cmp_holds(a.op, str_order(s, l, prefix_be8(s, l), p, m, pp));
                    }
                } else if (KIND == SM_STARTS) {
                    if (l >= m) {
                        if (a.pat_rows || m == 0) res = bytes_eq(s, p, m);
                        else {
                            const uint64_t mask = m >= 8 ? ~0ull : ~0ull << (64 - 8 * m);
                            res = ((prefix_be8(s, m) ^ a.pprefix) & mask) == 0 && bytes_eq(s + 8, p + 8, m - 8);
                        }
                    }
                } else if (KIND == SM_ENDS) {
                    res = l >= m && bytes_eq(s + l - m, p, m);
                } else if (KIND == SM_CONTAINS) {
                    res = find_naive(s, l, p, m);
                } else {      // SM_LIKE
                    if (l >= a.like_k) {
                        const uint64_t acc = 1ull << a.like_k;
                        uint64_t D = 1;
                        for (int64_t j = 0; j < l; j++) {
                            const uint8_t c = s[j];
                            D = ((D << 1) & s_tab[c]) | (D & s_tab[256 + c]);
                            if (D == 0) break;
                            if (a.like_tail_any && (D & acc)) break;      // a trailing '%' accepts whatever follows
                        }
                        res = (D & acc) != 0;
                    }
                }
                res = res != (bool)a.negate;
            }
        }
        const uint32_t bv = __ballot_sync(0xffffffffu, v), br = __ballot_sync(0xffffffffu, res && v);
        if (lane == 0) {
            a.out[i0 >> 5] = br;
            if (a.out_valid) a.out_valid[i0 >> 5] = bv;
        }
    }
}

// ---------------------------------------------------------------------------- byte-parallel contains
// tile t covers the bytes [base + t * SCAN_TILE, base + (t + 1) * SCAN_TILE) of `data` (base: offsets[0] rounded down to
// 16 bytes); rows[t] = the last row whose start is <= the tile's first byte (clamped to offsets[0]), rows[ntiles] = n
__global__ void __launch_bounds__(256) k_str_tile_rows(const int64_t* __restrict__ off, int64_t n, int64_t base, int64_t ntiles, uint32_t* __restrict__ rows) {
    for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t <= ntiles; t += (int64_t)gridDim.x * blockDim.x) {
        if (t == ntiles) { rows[t] = (uint32_t)n; continue; }
        const int64_t p = base + t * SCAN_TILE;
        int64_t lo = 0, hi = n - 1;      // the last r in [0, n) with off[r] <= p (0 when none)
        while (lo < hi) {
            const int64_t mid = (lo + hi + 1) >> 1;
            if (off[mid] <= p) lo = mid; else hi = mid - 1;
        }
        rows[t] = (uint32_t)lo;
    }
}

struct ScanArgs {
    const int64_t* off = nullptr;
    const uint8_t* data = nullptr;
    int64_t n = 0, lo = 0, hi = 0, base = 0, ntiles = 0;      // lo / hi: offsets[0] / offsets[n]; base: lo rounded down to 16
    const uint8_t* needle = nullptr;
    int m = 0;
    uint32_t first4 = 0, mask4 = 0;      // the needle's first min(m, 4) bytes (little-endian) and their mask
    const uint32_t* rows = nullptr;
    uint32_t* hits = nullptr;            // zeroed; bit r set when row r contains the needle
};

__global__ void __launch_bounds__(256) k_str_scan(ScanArgs a) {
    __shared__ __align__(16) uint8_t s_buf[SCAN_TILE + SCAN_HALO + 16];
    __shared__ uint8_t s_needle[SCAN_HALO];
    for (int i = threadIdx.x; i < a.m; i += blockDim.x) s_needle[i] = a.needle[i];
    const int load = (SCAN_TILE + ((a.m - 1 + 4 + 15) & ~15)) / 16;     // 16-byte chunks: the tile, the halo, the filter's next word
    for (int64_t t = blockIdx.x; t < a.ntiles; t += gridDim.x) {
        const int64_t t0 = a.base + t * SCAN_TILE;
        __syncthreads();      // the previous tile is no longer read
        for (int c = threadIdx.x; c < load; c += blockDim.x) {
            const int64_t p = t0 + 16 * (int64_t)c;
            uint4 v;
            if (p >= a.lo && p + 16 <= a.hi) v = *reinterpret_cast<const uint4*>(a.data + p);
            else {
                uint8_t b[16];
#pragma unroll
                for (int k = 0; k < 16; k++) b[k] = (p + k >= a.lo && p + k < a.hi) ? a.data[p + k] : 0;
                memcpy(&v, b, 16);
            }
            *reinterpret_cast<uint4*>(s_buf + 16 * c) = v;
        }
        __syncthreads();
        const int64_t r_lo = a.rows[t], r_hi = a.rows[t + 1];
        const uint32_t* s32 = reinterpret_cast<const uint32_t*>(s_buf);
        for (int q = threadIdx.x; q < SCAN_TILE / 4; q += blockDim.x) {
            const uint32_t w0 = s32[q], w1 = s32[q + 1];
#pragma unroll
            for (int k = 0; k < 4; k++) {
                const uint32_t w = __funnelshift_r(w0, w1, 8 * k);
                if ((w & a.mask4) != a.first4) continue;
                const int pos = 4 * q + k;
                const int64_t p = t0 + pos;
                if (p < a.lo || p + a.m > a.hi) continue;
                bool eq = true;
                for (int j = 4; j < a.m && eq; j++) eq = s_buf[pos + j] == s_needle[j];
                if (!eq) continue;
                int64_t lo = r_lo, hi = r_hi < a.n ? r_hi : a.n - 1;      // the last row whose start is <= p
                while (lo < hi) {
                    const int64_t mid = (lo + hi + 1) >> 1;
                    if (a.off[mid] <= p) lo = mid; else hi = mid - 1;
                }
                if (p + a.m <= a.off[lo + 1]) atomicOr(&a.hits[lo >> 5], 1u << (lo & 31));
            }
        }
    }
}

// out = (hits XOR negate) AND validity, one ballot of validity per 32 rows
__global__ void __launch_bounds__(256) k_str_scan_finish(StrArg col, int64_t n, int negate, uint32_t* __restrict__ out, uint32_t* __restrict__ out_valid) {
    const int lane = threadIdx.x & 31;
    for (int64_t i0 = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) & ~31ll; i0 < n; i0 += (int64_t)gridDim.x * blockDim.x) {
        const int64_t r = i0 + lane;
        const uint32_t bv = __ballot_sync(0xffffffffu, r < n && str_valid(col, r));
        if (lane == 0) {
            out[i0 >> 5] = (out[i0 >> 5] ^ (negate ? 0xffffffffu : 0u)) & bv;
            if (out_valid) out_valid[i0 >> 5] = bv;
        }
    }
}

// ---------------------------------------------------------------------------- host side
// the rows of a chunk list (checked before anything is read)
static int64_t rows_of(const bl_string_column* chunks, int32_t n_chunks, const std::string& who) {
    PLB_REQUIRE(chunks != nullptr && n_chunks >= 1, BL_ERR_INVALID, who + ": no chunks");
    int64_t n = 0;
    for (int i = 0; i < n_chunks; i++) {
        PLB_REQUIRE(chunks[i].length >= 0 && chunks[i].offset >= 0, BL_ERR_INVALID, who + ": negative length/offset");
        PLB_REQUIRE(chunks[i].offsets != nullptr, BL_ERR_INVALID, who + ": null offsets pointer");
        n += chunks[i].length;
    }
    return n;
}
// a string argument: a single device chunk read in place, anything else through import_string
struct StrIn {
    StrArg a;
    int64_t n = 0, lo = 0, hi = 0;      // rows; offsets[0] and offsets[n] (absolute, in bytes of a.data)
    bool nullable = false;
    DevStr owned;
};
static StrIn str_input(const bl_string_column* chunks, int32_t n_chunks, const std::string& who) {
    StrIn in;
    in.n = rows_of(chunks, n_chunks, who);
    PLB_REQUIRE(in.n <= 0xFFFFFFFEll, BL_ERR_UNSUPPORTED, who + ": more than 2^32 - 2 rows (IdxSize is u32)");
    const bl_string_column& c = chunks[0];
    if (n_chunks == 1 && c.location == BL_DEVICE) {
        const int64_t* o = c.offsets + c.offset;
        int64_t ends[2];
        PLB_CUDA(cudaMemcpyAsync(&ends[0], o, 8, cudaMemcpyDeviceToHost, ctx().stream));
        PLB_CUDA(cudaMemcpyAsync(&ends[1], o + c.length, 8, cudaMemcpyDeviceToHost, ctx().stream));
        PLB_CUDA(cudaStreamSynchronize(ctx().stream));
        PLB_REQUIRE(ends[1] >= ends[0] && ends[0] >= 0, BL_ERR_INVALID, who + ": offsets are not monotonic");
        PLB_REQUIRE(ends[1] == ends[0] || c.data != nullptr, BL_ERR_INVALID, who + ": null data pointer");
        in.a.off = o; in.a.data = c.data; in.lo = ends[0]; in.hi = ends[1];
        if (c.validity != nullptr && c.null_count != 0) { in.a.valid = c.validity; in.a.vbit = c.offset; in.nullable = true; }
        return in;
    }
    in.owned = import_string(chunks, n_chunks);
    in.a.off = in.owned.off(); in.a.data = in.owned.bytes(); in.lo = 0; in.hi = in.owned.data_bytes;
    if (in.owned.validity) { in.a.valid = as<uint8_t>(in.owned.validity); in.nullable = true; }
    return in;
}

// a scalar pattern (the one row of chunks whose lengths add up to 1): its bytes on the host and in a device buffer
struct Scalar { std::string bytes; bool null = false; DevPtr dev; };
static Scalar scalar_pattern(const bl_string_column* chunks, int32_t n_chunks) {
    Scalar s;
    int i = 0;
    while (chunks[i].length == 0) i++;
    const bl_string_column& c = chunks[i];
    const bool dev = c.location == BL_DEVICE;
    auto get = [&](void* dst, const void* src, size_t bytes) {
        if (dev) PLB_CUDA(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToHost, ctx().stream));
        else memcpy(dst, src, bytes);
    };
    int64_t o[2];
    get(o, c.offsets + c.offset, 16);
    uint8_t vb = 0xFF;
    if (c.validity != nullptr && c.null_count != 0) get(&vb, c.validity + (c.offset >> 3), 1);
    if (dev) PLB_CUDA(cudaStreamSynchronize(ctx().stream));
    PLB_REQUIRE(o[1] >= o[0] && o[0] >= 0, BL_ERR_INVALID, "string pattern: offsets are not monotonic");
    PLB_REQUIRE(o[1] == o[0] || c.data != nullptr, BL_ERR_INVALID, "string pattern: null data pointer");
    s.null = !((vb >> (c.offset & 7)) & 1);
    if (!s.null && o[1] > o[0]) {
        s.bytes.resize((size_t)(o[1] - o[0]));
        get(&s.bytes[0], c.data + o[0], s.bytes.size());
    }
    s.dev = dev_alloc(s.bytes.size() + 16);
    if (!s.bytes.empty()) PLB_CUDA(cudaMemcpyAsync(s.dev->p, s.bytes.data(), s.bytes.size(), cudaMemcpyHostToDevice, ctx().stream));
    PLB_CUDA(cudaStreamSynchronize(ctx().stream));
    return s;
}
static uint64_t prefix_of(const std::string& b) {
    uint64_t pp = 0;
    for (size_t i = 0; i < b.size() && i < 8; i++) pp |= (uint64_t)(uint8_t)b[i] << (56 - 8 * i);
    return pp;
}

// The NFA of a LIKE pattern (extended Shift-And over bytes, one 64-bit word).  State j is "the first j byte-consuming
// tokens matched"; a literal byte or a '_' moves j -> j + 1, '%' adds a self-loop to the current state, '_' consumes one
// UTF-8 lead byte and adds a self-loop on continuation bytes (10xxxxxx) to its target; an open start / end is a self-loop
// on every byte at state 0 / k.  Per byte c:
//   D = ((D << 1) & B[c]) | (D & L[c]);   match when bit k is set after the last byte.
struct LikeNfa { std::vector<uint64_t> tab = std::vector<uint64_t>(512, 0); int k = 0; bool tail_any = false; };
static LikeNfa compile_like(const std::string& pat, int escape, int flags) {
    const bool no_newline = (flags & BL_LIKE_NO_NEWLINE) != 0;
    LikeNfa f;
    uint64_t* B = f.tab.data();
    uint64_t* L = f.tab.data() + 256;
    auto any_byte = [&](int c) { return !(no_newline && c == '\n'); };
    bool last_star = false;
    for (size_t i = 0; i < pat.size(); i++) {
        int c = (uint8_t)pat[i];
        bool literal = false;
        if (escape != 0 && c == escape) {
            PLB_REQUIRE(i + 1 < pat.size(), BL_ERR_INVALID, "string_match: LIKE pattern ends with its escape character");
            const int d = (uint8_t)pat[++i];
            PLB_REQUIRE(d == '%' || d == '_' || d == escape, BL_ERR_INVALID,
                        "string_match: the LIKE escape character must precede '%', '_' or itself");
            c = d; literal = true;
        }
        if (!literal && c == '%') {
            for (int b = 0; b < 256; b++) if (any_byte(b)) L[b] |= 1ull << f.k;
            last_star = true;
            continue;
        }
        last_star = false;
        PLB_REQUIRE(f.k < LIKE_MAX_STATES, BL_ERR_UNSUPPORTED,
                    "string_match: LIKE patterns take at most " + std::to_string(LIKE_MAX_STATES) + " literal bytes and '_' wildcards");
        const uint64_t next = 1ull << (f.k + 1);
        if (!literal && c == '_') {
            for (int b = 0; b < 256; b++) {
                if ((b & 0xC0) == 0x80) L[b] |= next;      // the rest of the character
                else if (any_byte(b)) B[b] |= next;        // its lead byte
            }
        } else B[c] |= next;
        f.k++;
    }
    f.tail_any = last_star && !no_newline;
    if (flags & BL_LIKE_OPEN_START)
        for (int b = 0; b < 256; b++) L[b] |= 1ull;
    if (flags & BL_LIKE_OPEN_END) {
        for (int b = 0; b < 256; b++) L[b] |= 1ull << f.k;
        f.tail_any = true;
    }
    return f;
}

static double scan_min_row_bytes() {      // read per call; a measurement override of the plan rule (DESIGN.md §19)
    const char* e = getenv("BL_STR_SCAN_MIN_ROW");
    return e ? atof(e) : SCAN_MIN_ROW_BYTES;
}

// the result column: values + validity (when it can hold nulls), null_count exact
static DevCol bool_result(int64_t n, bool nullable) {
    DevCol out; out.dtype = BL_BOOL; out.len = n;
    out.values = dev_alloc(bitmap_bytes(n) + 16);
    if (nullable) out.validity = dev_alloc(bitmap_bytes(n) + 16);
    out.null_count = 0;
    return out;
}
static void finish_nulls(DevCol& out) {
    if (!out.validity) return;
    out.null_count = out.len - bitmap_popcount(out.vm(), out.len);
    if (out.null_count == 0) out.validity.reset();
}

static void launch_rows(int kind, RowsArgs& a, size_t smem) {
    if (a.n == 0) return;
    const int grid = grid_for((a.n + 31) / 32 * 32, SM_THREADS, 16);
    switch (kind) {
        case SM_CMP: PLB_LAUNCH("str_cmp", k_str_rows<SM_CMP>, grid, SM_THREADS, smem, a); break;
        case SM_STARTS: PLB_LAUNCH("str_starts", k_str_rows<SM_STARTS>, grid, SM_THREADS, smem, a); break;
        case SM_ENDS: PLB_LAUNCH("str_ends", k_str_rows<SM_ENDS>, grid, SM_THREADS, smem, a); break;
        case SM_CONTAINS: PLB_LAUNCH("str_contains_rows", k_str_rows<SM_CONTAINS>, grid, SM_THREADS, smem, a); break;
        default: PLB_LAUNCH("str_like", k_str_rows<SM_LIKE>, grid, SM_THREADS, smem, a); break;
    }
}

// rhs: a column of lhs's length (rhs_rows) or the scalar `sc`
DevCol op_string_compare(int op, const StrIn& lhs, const StrIn* rhs_rows, const Scalar* sc, bool missing) {
    RowsArgs a;
    a.col = lhs.a; a.n = lhs.n; a.op = op; a.missing = missing;
    size_t smem = 0;
    bool nullable = lhs.nullable;
    if (sc) {
        a.scalar = as<uint8_t>(sc->dev); a.pat_null = sc->null; a.m = (int64_t)sc->bytes.size(); a.pprefix = prefix_of(sc->bytes);
        smem = sc->null ? 0 : std::min<size_t>(sc->bytes.size(), SM_PAT_SMEM);
        nullable |= sc->null;
    } else { a.pat = rhs_rows->a; a.pat_rows = 1; nullable |= rhs_rows->nullable; }
    DevCol out = bool_result(lhs.n, !missing && nullable);
    a.out = as<uint32_t>(out.values); a.out_valid = as<uint32_t>(out.validity);
    launch_rows(SM_CMP, a, smem);
    finish_nulls(out);
    return out;
}

// pattern: a column of col's length (pat_rows) or the scalar `sc` (LIKE: always the scalar)
DevCol op_string_match(int kind, int flags, int escape, const StrIn& col, const StrIn* pat_rows, const Scalar* sc) {
    const int k = kind == BL_STR_STARTS_WITH ? SM_STARTS : kind == BL_STR_ENDS_WITH ? SM_ENDS : kind == BL_STR_CONTAINS ? SM_CONTAINS : SM_LIKE;
    RowsArgs a;
    a.col = col.a; a.n = col.n; a.negate = (flags & BL_STR_NEGATE) != 0;
    if (!sc) {
        a.pat = pat_rows->a; a.pat_rows = 1;
        DevCol out = bool_result(col.n, col.nullable || pat_rows->nullable);
        a.out = as<uint32_t>(out.values); a.out_valid = as<uint32_t>(out.validity);
        launch_rows(k, a, 0);
        finish_nulls(out);
        return out;
    }
    a.scalar = as<uint8_t>(sc->dev); a.pat_null = sc->null; a.m = (int64_t)sc->bytes.size(); a.pprefix = prefix_of(sc->bytes);
    DevCol out = bool_result(col.n, col.nullable || sc->null);
    a.out = as<uint32_t>(out.values); a.out_valid = as<uint32_t>(out.validity);
    if (sc->null) {      // a null scalar: all null
        dev_memset(out.values->p, 0, bitmap_bytes(col.n));
        dev_memset(out.validity->p, 0, bitmap_bytes(col.n));
        out.null_count = col.n;
        if (col.n == 0) out.validity.reset();
        return out;
    }
    if (k == SM_LIKE) {
        const LikeNfa f = compile_like(sc->bytes, escape, flags);
        DevPtr tab = dev_alloc(512 * 8);
        PLB_CUDA(cudaMemcpyAsync(tab->p, f.tab.data(), 512 * 8, cudaMemcpyHostToDevice, ctx().stream));
        a.like_tab = as<uint64_t>(tab); a.like_k = f.k; a.like_tail_any = f.tail_any;
        launch_rows(SM_LIKE, a, 512 * 8);
        PLB_CUDA(cudaStreamSynchronize(ctx().stream));      // `f` lives on this frame
        finish_nulls(out);
        return out;
    }
    const double row_bytes = col.n ? (double)(col.hi - col.lo) / (double)col.n : 0.0;
    if (k == SM_CONTAINS && a.m >= 1 && a.m <= SCAN_HALO && col.n > 0 && row_bytes >= scan_min_row_bytes()) {      // byte-parallel plan
        ScanArgs sa;
        sa.off = col.a.off; sa.data = col.a.data; sa.n = col.n; sa.lo = col.lo; sa.hi = col.hi;
        const int64_t abs_lo = (int64_t)(reinterpret_cast<uintptr_t>(col.a.data) + (uintptr_t)col.lo);
        sa.base = col.lo - (abs_lo & 15);
        sa.ntiles = (col.hi - sa.base + SCAN_TILE - 1) / SCAN_TILE;
        sa.needle = a.scalar; sa.m = (int)a.m;
        for (int i = 0; i < 4 && i < sa.m; i++) { sa.first4 |= (uint32_t)(uint8_t)sc->bytes[i] << (8 * i); sa.mask4 |= 0xFFu << (8 * i); }
        DevPtr rows = dev_alloc((size_t)(sa.ntiles + 1) * 4);
        sa.rows = as<uint32_t>(rows); sa.hits = a.out;
        dev_memset(a.out, 0, bitmap_bytes(col.n));
        PLB_LAUNCH("str_tile_rows", k_str_tile_rows, grid_for(sa.ntiles + 1, 256), 256, 0, col.a.off, col.n, sa.base, sa.ntiles, as<uint32_t>(rows));
        PLB_LAUNCH("str_scan", k_str_scan, grid_for(sa.ntiles * 256, 256, 8), 256, 0, sa);
        PLB_LAUNCH("str_scan_finish", k_str_scan_finish, grid_for((col.n + 31) / 32 * 32, 256, 16), 256, 0, col.a, col.n, a.negate, a.out, a.out_valid);
        finish_nulls(out);
        return out;
    }
    launch_rows(k, a, std::min<size_t>(sc->bytes.size(), SM_PAT_SMEM));
    finish_nulls(out);
    return out;
}

}  // namespace plb

// ================================================================================ C ABI
using namespace plb;
extern "C" {

bl_status bl_string_compare(int32_t op, const bl_string_column* lhs, int32_t n_lhs_chunks, const bl_string_column* rhs, int32_t n_rhs_chunks, int32_t missing,
                            int32_t out_location, bl_column* out) {
    BL_TRY
    PLB_REQUIRE(out != nullptr, BL_ERR_INVALID, "string_compare: null output");
    PLB_REQUIRE(op >= BL_CMP_EQ && op <= BL_CMP_GE, BL_ERR_INVALID, "string_compare: unknown operator " + std::to_string(op));
    PLB_REQUIRE(!missing || op == BL_CMP_EQ || op == BL_CMP_NE, BL_ERR_INVALID, "string_compare: `missing` takes EQ or NE only");
    const StrIn l = str_input(lhs, n_lhs_chunks, "string_compare: lhs");
    const int64_t rn = rows_of(rhs, n_rhs_chunks, "string_compare: rhs");
    PLB_REQUIRE(rn == l.n || rn == 1, BL_ERR_INVALID,
                "string_compare: rhs has " + std::to_string(rn) + " rows, lhs " + std::to_string(l.n) + " (rhs must match or be a scalar)");
    if (rn == 1) {
        const Scalar sc = scalar_pattern(rhs, n_rhs_chunks);
        export_column(op_string_compare(op, l, nullptr, &sc, missing != 0), out_location, out);
    } else {
        const StrIn r = str_input(rhs, n_rhs_chunks, "string_compare: rhs");
        export_column(op_string_compare(op, l, &r, nullptr, missing != 0), out_location, out);
    }
    BL_CATCH
}

bl_status bl_string_match(int32_t kind, int32_t flags, int32_t escape, const bl_string_column* col, int32_t n_chunks, const bl_string_column* pattern,
                          int32_t n_pattern_chunks, int32_t out_location, bl_column* out) {
    BL_TRY
    PLB_REQUIRE(out != nullptr, BL_ERR_INVALID, "string_match: null output");
    PLB_REQUIRE(kind >= BL_STR_STARTS_WITH && kind <= BL_STR_LIKE, BL_ERR_INVALID, "string_match: unknown kind " + std::to_string(kind));
    const int like_flags = BL_LIKE_NO_NEWLINE | BL_LIKE_OPEN_START | BL_LIKE_OPEN_END;
    PLB_REQUIRE((flags & ~(BL_STR_NEGATE | like_flags)) == 0, BL_ERR_INVALID, "string_match: unknown flags " + std::to_string(flags));
    PLB_REQUIRE(kind == BL_STR_LIKE || ((flags & like_flags) == 0 && escape == 0), BL_ERR_INVALID,
                "string_match: the BL_LIKE_* flags and `escape` apply to BL_STR_LIKE only");
    PLB_REQUIRE(escape >= 0 && escape <= 255, BL_ERR_INVALID, "string_match: `escape` must be a byte");
    const StrIn c = str_input(col, n_chunks, "string_match: column");
    const int64_t pn = rows_of(pattern, n_pattern_chunks, "string_match: pattern");
    PLB_REQUIRE(pn == c.n || pn == 1, BL_ERR_INVALID,
                "string_match: the pattern has " + std::to_string(pn) + " rows, the column " + std::to_string(c.n) + " (it must match or be a scalar)");
    PLB_REQUIRE(kind != BL_STR_LIKE || pn == 1, BL_ERR_INVALID, "string_match: a LIKE pattern must be a scalar");
    if (pn == 1) {
        const Scalar sc = scalar_pattern(pattern, n_pattern_chunks);
        export_column(op_string_match(kind, flags, escape, c, nullptr, &sc), out_location, out);
    } else {
        const StrIn p = str_input(pattern, n_pattern_chunks, "string_match: pattern");
        export_column(op_string_match(kind, flags, escape, c, &p, nullptr), out_location, out);
    }
    BL_CATCH
}

bl_status bl_string_filter(const bl_string_column* chunks, int32_t n_chunks, const bl_column* mask, int32_t out_location, bl_string_column* out) {
    BL_TRY
    PLB_REQUIRE(out != nullptr && mask != nullptr, BL_ERR_INVALID, "string_filter: null argument");
    PLB_REQUIRE(chunks != nullptr && n_chunks >= 1, BL_ERR_INVALID, "string_filter: no chunks");
    PLB_REQUIRE(mask->dtype == BL_BOOL, BL_ERR_DTYPE, "string_filter: mask must be BL_BOOL");
    int64_t n = 0;
    for (int i = 0; i < n_chunks; i++) n += chunks[i].length;
    PLB_REQUIRE(mask->length == n, BL_ERR_INVALID, "string_filter: mask has " + std::to_string(mask->length) + " rows, the column " + std::to_string(n));
    PLB_REQUIRE(n <= 0xFFFFFFFEll, BL_ERR_UNSUPPORTED, "string_filter: more than 2^32 - 2 rows (IdxSize is u32)");
    DevCol m = import_column(mask, 1);
    const uint32_t* bits = as<uint32_t>(m.values);
    DevPtr both;
    if (m.validity) { both = bitmap_and(bits, m.vm(), nullptr, n); bits = as<uint32_t>(both); }      // a null slot counts as false
    const DevCol idx = op_mask_rows(bits, n);
    const bl_string_column& c = chunks[0];
    const bool aligned_validity = c.validity == nullptr || c.null_count == 0 || (c.offset % 32 == 0 && reinterpret_cast<uintptr_t>(c.validity) % 4 == 0);
    DevStr s;
    if (n_chunks == 1 && c.location == BL_DEVICE && aligned_validity) {      // read in place: only the kept rows' bytes move
        PLB_REQUIRE(c.offsets != nullptr && c.offset >= 0, BL_ERR_INVALID, "string_filter: bad offsets");
        s.len = n;
        s.offsets = dev_borrow(c.offsets + c.offset, (size_t)(n + 1) * 8);
        s.data = dev_borrow(c.data, 0);
        if (c.validity != nullptr && c.null_count != 0) { s.validity = dev_borrow(c.validity + c.offset / 8, bitmap_bytes(n)); s.null_count = -1; }
    } else s = import_string(chunks, n_chunks);
    export_string(op_string_gather(s, idx), out_location, out);
    BL_CATCH
}

}  // extern "C"
