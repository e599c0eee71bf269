// k_list.cu -- list values: split (spark_strings.rs:93-115), array (spark_make_array.rs), broadcast list literals, and the
// row mapping of explode / posexplode (generate/explode.rs, generate_exec.rs:191-310).  Every kernel's work is proportional to
// the bytes or elements it produces: a long row is spread over many threads, never looped over by one.
#include "device_utils.cuh"
#include "kernels.h"

namespace auron {

#define LAUNCH_CHECK(ctx)            \
    do {                             \
        CUDA_OK(cudaGetLastError()); \
        launch_count(ctx);           \
    } while (0)

static unsigned grid_of(int64_t n) { return (unsigned)((n + 255) / 256); }

// last i in [0, n) with off[i] <= j, for off[0] <= j < off[n] (rows without elements are skipped over)
template <typename T>
__device__ __forceinline__ int64_t last_le(const T* __restrict__ off, int64_t n, int64_t j) {
    int64_t lo = 0, hi = n;
    while (hi - lo > 1) {
        int64_t mid = (lo + hi) >> 1;
        if ((int64_t)off[mid] <= j) lo = mid;
        else hi = mid;
    }
    return lo;
}
// first i in [0, n) with a[i] >= v (n when none)
__device__ __forceinline__ int64_t lower_bound_i32(const int32_t* __restrict__ a, int64_t n, int64_t v) {
    int64_t lo = 0, hi = n;
    while (lo < hi) {
        int64_t mid = (lo + hi) >> 1;
        if ((int64_t)a[mid] < v) lo = mid + 1;
        else hi = mid;
    }
    return lo;
}

__global__ void narrow_i64_kernel(const int64_t* __restrict__ in, int32_t* __restrict__ out, int64_t n) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = (int32_t)in[i];
}
// int64 lengths [n] (+1 slot) -> int32 offsets [n + 1]; returns the total, which must fit int32 (`what` names the column)
static int64_t offsets_from_lens(Ctx& ctx, const Buf& lens, int64_t n, int32_t* out_off, const char* what) {
    exclusive_scan_i64(ctx, P<int64_t>(lens), P<int64_t>(lens), n, P<int64_t>(lens) + n);
    narrow_i64_kernel<<<grid_of(n + 1), 256, 0, ctx.stream>>>(P<int64_t>(lens), out_off, n + 1);
    LAUNCH_CHECK(ctx);
    int64_t total = 0;
    to_host(ctx, &total, P<int64_t>(lens) + n, 8);
    AURON_CHECK(total <= (int64_t)INT32_MAX, std::string(what) + " of " + std::to_string(total) + " exceeds 2^31 - 1 in one batch");
    return total;
}

// ------------------------------------------------------------------------------------------ split
// bit p of `cand`: a match of the pattern starts at byte p and ends inside p's row (NULL rows have none)
__global__ void __launch_bounds__(256) split_candidates_kernel(const int32_t* __restrict__ off, const uint8_t* __restrict__ valid,
                                                               const uint8_t* __restrict__ data, int64_t n, int64_t total,
                                                               const uint8_t* __restrict__ pat, int32_t m, uint32_t* __restrict__ cand) {
    int64_t p = (int64_t)blockIdx.x * 256 + threadIdx.x;
    bool hit = false;
    if (p < total) {
        const int64_t r = last_le(off, n, p);
        if (valid_at(valid, r) && p + m <= (int64_t)off[r + 1]) {
            hit = true;
            for (int32_t k = 0; k < m && hit; k++) hit = data[p + k] == pat[k];
        }
    }
    const uint32_t w = __ballot_sync(FULL_MASK, hit);
    if (lane_id() == 0 && p < total) cand[p >> 5] = w;
}
__device__ __forceinline__ bool mask_bit(const uint32_t* __restrict__ m, int64_t i) { return (m[i >> 5] >> (i & 31)) & 1u; }
// a pattern that overlaps itself ("--" over "---"): candidates that overlap form chains, and the leftmost non-overlapping matches
// of a chain follow from its head, the candidate with no candidate in the m - 1 bytes before it (candidates of two rows never
// overlap: a candidate ends inside its row)
__global__ void __launch_bounds__(256) split_resolve_kernel(const uint32_t* __restrict__ cand, int64_t total, int32_t m, uint32_t* __restrict__ sel) {
    int64_t p = (int64_t)blockIdx.x * 256 + threadIdx.x;
    if (p >= total || !mask_bit(cand, p)) return;
    for (int64_t q = p - 1; q > p - m && q >= 0; q--)
        if (mask_bit(cand, q)) return;
    int64_t last = p, prev = p;
    atomicOr(&sel[p >> 5], 1u << (p & 31));
    for (int64_t q = p + 1; q < total && q < prev + m; q++) {
        if (!mask_bit(cand, q)) continue;
        if (q >= last + m) {
            atomicOr(&sel[q >> 5], 1u << (q & 31));
            last = q;
        }
        prev = q;
    }
}
// per row: pieces = matches + 1 (0 for NULL), and the index of its first match among all matches
__global__ void __launch_bounds__(256) split_count_kernel(const int32_t* __restrict__ off, const uint8_t* __restrict__ valid, int64_t n,
                                                          const int32_t* __restrict__ matches, int64_t n_matches, int64_t* __restrict__ lens,
                                                          int32_t* __restrict__ first_match) {
    int64_t r = (int64_t)blockIdx.x * 256 + threadIdx.x;
    if (r >= n) return;
    const int64_t a = lower_bound_i32(matches, n_matches, off[r]), b = lower_bound_i32(matches, n_matches, off[r + 1]);
    first_match[r] = (int32_t)a;
    lens[r] = valid_at(valid, r) ? b - a + 1 : 0;
}
// per piece: where its bytes start in the input and how many there are
__global__ void __launch_bounds__(256) split_piece_kernel(const int32_t* __restrict__ off, const int32_t* __restrict__ list_off, int64_t n,
                                                          const int32_t* __restrict__ matches, const int32_t* __restrict__ first_match, int32_t m,
                                                          int64_t pieces, int32_t* __restrict__ start, int64_t* __restrict__ lens) {
    int64_t j = (int64_t)blockIdx.x * 256 + threadIdx.x;
    if (j >= pieces) return;
    const int64_t r = last_le(list_off, n, j);
    const int64_t t = j - list_off[r], last = (int64_t)list_off[r + 1] - list_off[r] - 1;
    const int64_t s = t == 0 ? off[r] : (int64_t)matches[first_match[r] + t - 1] + m;
    const int64_t e = t == last ? off[r + 1] : (int64_t)matches[first_match[r] + t];
    start[j] = (int32_t)s;
    lens[j] = e - s;
}
// out bytes of segment j = src[start[j] ..): each thread copies 16 consecutive output bytes, finding its segment once
__global__ void __launch_bounds__(256) copy_segments_kernel(const uint8_t* __restrict__ src, const int32_t* __restrict__ start,
                                                            const int32_t* __restrict__ out_off, int64_t segs, int64_t total,
                                                            uint8_t* __restrict__ out) {
    const int64_t b0 = ((int64_t)blockIdx.x * 256 + threadIdx.x) * 16;
    if (b0 >= total) return;
    int64_t j = last_le(out_off, segs, b0);
    const int64_t b1 = min(b0 + 16, total);
    for (int64_t b = b0; b < b1; b++) {
        while (b >= out_off[j + 1]) j++;
        out[b] = src[start[j] + (b - out_off[j])];
    }
}

ColumnPtr string_split(Ctx& ctx, const Column& s, const std::string& pattern, const DType& out_type) {
    AURON_CHECK(s.type.id == T_UTF8, "Spark_StringSplit needs a utf8 argument, got " + s.type.str());
    AURON_CHECK(!pattern.empty(), "Spark_StringSplit needs a non-empty pattern");
    ProfScope ps(ctx, "string_split");
    const int64_t n = s.len, total = s.data_bytes;
    const int32_t m = (int32_t)pattern.size();
    auto out = std::make_shared<Column>();
    out->type = out_type;
    out->len = n;
    out->offsets = dalloc(ctx, (size_t)(n + 1) * 4);
    if (s.validity) {   // the list is NULL where the string is
        out->validity = dalloc(ctx, bitmap_alloc_bytes(n));
        if (n) CUDA_OK(cudaMemcpyAsync(out->validity->ptr, s.validity->ptr, bitmap_alloc_bytes(n), cudaMemcpyDeviceToDevice, ctx.stream));
        out->null_count = s.null_count;
    }
    // 1. match positions, leftmost and non-overlapping within each row
    const int64_t words = (total + 31) / 32;
    Buf cand = dalloc_zero(ctx, (size_t)std::max<int64_t>(words, 1) * 4);
    Buf pat = to_device(ctx, pattern.data(), pattern.size());
    if (total > 0) {
        split_candidates_kernel<<<grid_of(total), 256, 0, ctx.stream>>>(P<int32_t>(s.offsets), s.vbits(), P<uint8_t>(s.data), n, total,
                                                                        P<uint8_t>(pat), m, P<uint32_t>(cand));
        LAUNCH_CHECK(ctx);
    }
    bool self_overlapping = false;   // a proper prefix of the pattern that is also its suffix
    for (int32_t k = 1; k < m && !self_overlapping; k++) self_overlapping = pattern.compare(0, (size_t)k, pattern, (size_t)(m - k), (size_t)k) == 0;
    Buf sel = cand;
    if (self_overlapping && total > 0) {
        sel = dalloc_zero(ctx, (size_t)words * 4);
        split_resolve_kernel<<<grid_of(total), 256, 0, ctx.stream>>>(P<uint32_t>(cand), total, m, P<uint32_t>(sel));
        LAUNCH_CHECK(ctx);
    }
    int64_t n_matches = 0;
    Buf matches = total > 0 ? mask_to_indices(ctx, P<uint32_t>(sel), total, &n_matches) : dalloc(ctx, 4);
    // 2. list offsets: pieces per row
    Buf lens = dalloc(ctx, (size_t)(n + 1) * 8);
    Buf first = dalloc(ctx, (size_t)std::max<int64_t>(n, 1) * 4);
    if (n) {
        split_count_kernel<<<grid_of(n), 256, 0, ctx.stream>>>(P<int32_t>(s.offsets), s.vbits(), n, P<int32_t>(matches), n_matches, P<int64_t>(lens),
                                                               P<int32_t>(first));
        LAUNCH_CHECK(ctx);
    }
    const int64_t pieces = offsets_from_lens(ctx, lens, n, P<int32_t>(out->offsets), "Spark_StringSplit: pieces");
    // 3. the pieces as one utf8 child column
    auto child = std::make_shared<Column>();
    child->type = *out_type.elem;
    child->len = pieces;
    child->offsets = dalloc(ctx, (size_t)(pieces + 1) * 4);
    Buf start = dalloc(ctx, (size_t)std::max<int64_t>(pieces, 1) * 4);
    Buf plens = dalloc(ctx, (size_t)(pieces + 1) * 8);
    if (pieces) {
        split_piece_kernel<<<grid_of(pieces), 256, 0, ctx.stream>>>(P<int32_t>(s.offsets), P<int32_t>(out->offsets), n, P<int32_t>(matches), P<int32_t>(first), m,
                                                                    pieces, P<int32_t>(start), P<int64_t>(plens));
        LAUNCH_CHECK(ctx);
    }
    child->data_bytes = offsets_from_lens(ctx, plens, pieces, P<int32_t>(child->offsets), "Spark_StringSplit: bytes");
    child->data = dalloc(ctx, (size_t)child->data_bytes);
    if (child->data_bytes) {
        copy_segments_kernel<<<grid_of((child->data_bytes + 15) / 16), 256, 0, ctx.stream>>>(P<uint8_t>(s.data), P<int32_t>(start), P<int32_t>(child->offsets),
                                                                                            pieces, child->data_bytes, P<uint8_t>(child->data));
        LAUNCH_CHECK(ctx);
    }
    out->child = child;
    return out;
}

// ------------------------------------------------------------------------------------------ array() and list literals
__global__ void strided_offsets_kernel(int32_t* __restrict__ off, int64_t n_plus_1, int32_t stride) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n_plus_1) off[i] = (int32_t)(i * stride);
}
// element t of list i (j = i * k + t) copies element t * col_stride + i * row_stride: array() reads row i of argument t from the
// arguments concatenated (col_stride n, row_stride 1), a literal repeats its k elements (col_stride 1, row_stride 0)
__global__ void interleave_index_kernel(int32_t* __restrict__ idx, int64_t total, int32_t k, int64_t col_stride, int64_t row_stride) {
    int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (j < total) idx[j] = (int32_t)((j % k) * col_stride + (j / k) * row_stride);
}
static ColumnPtr fixed_lists(Ctx& ctx, const DType& out_type, int64_t n, int64_t k, const Column& elems, int64_t col_stride, int64_t row_stride) {
    const int64_t total = n * k;
    AURON_CHECK(total <= (int64_t)INT32_MAX, "list column of " + std::to_string(total) + " elements exceeds 2^31 - 1 elements in one batch");
    auto out = std::make_shared<Column>();
    out->type = out_type;
    out->len = n;
    out->offsets = dalloc(ctx, (size_t)(n + 1) * 4);
    strided_offsets_kernel<<<grid_of(n + 1), 256, 0, ctx.stream>>>(P<int32_t>(out->offsets), n + 1, (int32_t)k);
    LAUNCH_CHECK(ctx);
    Buf idx = dalloc(ctx, (size_t)std::max<int64_t>(total, 1) * 4);
    if (total) {
        interleave_index_kernel<<<grid_of(total), 256, 0, ctx.stream>>>(P<int32_t>(idx), total, (int32_t)k, col_stride, row_stride);
        LAUNCH_CHECK(ctx);
    }
    out->child = take(ctx, elems, P<int32_t>(idx), total, false);
    return out;
}
ColumnPtr make_array(Ctx& ctx, const std::vector<ColumnPtr>& args, int64_t n, const DType& out_type) {
    AURON_CHECK(!args.empty(), "Spark_MakeArray needs at least one argument");
    ProfScope ps(ctx, "make_array");
    ColumnPtr all = concat_columns(ctx, args);
    return fixed_lists(ctx, out_type, n, (int64_t)args.size(), *all, n, 1);
}
ColumnPtr broadcast_list(Ctx& ctx, const ColumnPtr& elems, bool is_null, int64_t n, const DType& out_type) {
    if (!is_null) return fixed_lists(ctx, out_type, n, elems->len, *elems, 1, 0);
    auto out = std::make_shared<Column>();
    out->type = out_type;
    out->len = n;
    out->offsets = dalloc_zero(ctx, (size_t)(n + 1) * 4);
    out->validity = dalloc_zero(ctx, bitmap_alloc_bytes(n));
    out->null_count = n;
    out->child = take(ctx, *elems, nullptr, 0, false);
    return out;
}

// ------------------------------------------------------------------------------------------ explode
// per selected row s: output rows (elements; 1 for a NULL or empty list under outer) and the bytes they copy of the required
// variable-length columns
struct VarCols {
    const int32_t* off[kMaxExplodeVarCols];
    int32_t n;
};
__global__ void __launch_bounds__(256) explode_count_kernel(const int32_t* __restrict__ loff, const uint8_t* __restrict__ lvalid,
                                                            const int32_t* __restrict__ sel, int64_t n, bool outer, VarCols vc,
                                                            int64_t* __restrict__ rows, int64_t* __restrict__ bytes) {
    int64_t s = (int64_t)blockIdx.x * 256 + threadIdx.x;
    if (s >= n) return;
    const int64_t len = valid_at(lvalid, s) ? (int64_t)(loff[s + 1] - loff[s]) : 0;
    const int64_t c = len > 0 ? len : (outer ? 1 : 0);
    const int64_t r = sel ? sel[s] : s;
    int64_t w = 0;
    for (int k = 0; k < vc.n; k++) w += (int64_t)(vc.off[k][r + 1] - vc.off[k][r]);
    rows[s] = c;
    bytes[s] = c * w;
}
void explode_scan(Ctx& ctx, const Column& list, bool outer, const std::vector<ColumnPtr>& var_cols, const int32_t* sel, int64_t n, Buf* rows_cum,
                  Buf* bytes_cum) {
    AURON_CHECK(var_cols.size() <= (size_t)kMaxExplodeVarCols, "GenerateExec: too many required string columns");
    VarCols vc{};
    vc.n = (int32_t)var_cols.size();
    for (size_t k = 0; k < var_cols.size(); k++) vc.off[k] = P<int32_t>(var_cols[k]->offsets);
    *rows_cum = dalloc(ctx, (size_t)(n + 1) * 8);
    *bytes_cum = dalloc(ctx, (size_t)(n + 1) * 8);
    if (n) {
        explode_count_kernel<<<grid_of(n), 256, 0, ctx.stream>>>(P<int32_t>(list.offsets), list.vbits(), sel, n, outer, vc, P<int64_t>(*rows_cum),
                                                                 P<int64_t>(*bytes_cum));
        LAUNCH_CHECK(ctx);
    }
    exclusive_scan_i64(ctx, P<int64_t>(*rows_cum), P<int64_t>(*rows_cum), n, P<int64_t>(*rows_cum) + n);
    exclusive_scan_i64(ctx, P<int64_t>(*bytes_cum), P<int64_t>(*bytes_cum), n, P<int64_t>(*bytes_cum) + n);
}
// the largest r1 <= n with rows(r0, r1) <= max_rows and bytes(r0, r1) <= max_bytes (both sums are non-decreasing in r1); out[1..2]:
// the rows and bytes of [r0, r1)
__global__ void explode_cut_kernel(const int64_t* __restrict__ rows, const int64_t* __restrict__ bytes, int64_t n, int64_t r0, int64_t max_rows,
                                   int64_t max_bytes, int64_t* __restrict__ out) {
    int64_t lo = r0, hi = n;
    while (lo < hi) {
        int64_t mid = (lo + hi + 1) >> 1;
        if (rows[mid] - rows[r0] <= max_rows && bytes[mid] - bytes[r0] <= max_bytes) lo = mid;
        else hi = mid - 1;
    }
    if (lo == r0 && r0 < n) lo = r0 + 1;   // one input row beyond the limits is a piece of its own
    out[0] = lo;
    out[1] = rows[lo] - rows[r0];
    out[2] = bytes[lo] - bytes[r0];
}
int64_t explode_cut(Ctx& ctx, const Buf& rows_cum, const Buf& bytes_cum, int64_t n, int64_t r0, int64_t max_rows, int64_t max_bytes, int64_t* out_rows,
                    int64_t* out_bytes) {
    Buf o = dalloc(ctx, 24);
    explode_cut_kernel<<<1, 1, 0, ctx.stream>>>(P<int64_t>(rows_cum), P<int64_t>(bytes_cum), n, r0, max_rows, max_bytes, P<int64_t>(o));
    LAUNCH_CHECK(ctx);
    int64_t h[3];
    to_host(ctx, h, o->ptr, 24);
    *out_rows = h[1];
    *out_bytes = h[2];
    return h[0];
}
// output row o of the piece that starts at selected row r0: its input row, its element (-1: the NULL row of outer) and position
__global__ void __launch_bounds__(256) explode_map_kernel(const int32_t* __restrict__ loff, const uint8_t* __restrict__ lvalid,
                                                          const int32_t* __restrict__ sel, const int64_t* __restrict__ rows, int64_t r0, int64_t r1,
                                                          int64_t n_out, int32_t* __restrict__ row_idx, int32_t* __restrict__ elem_idx,
                                                          int32_t* __restrict__ pos, uint32_t* __restrict__ pos_valid) {
    int64_t o = (int64_t)blockIdx.x * 256 + threadIdx.x;
    bool ok = false;
    if (o < n_out) {
        const int64_t g = rows[r0] + o;
        const int64_t s = r0 + last_le(rows + r0, r1 - r0, g);
        const int64_t k = g - rows[s];
        const bool has = valid_at(lvalid, s) && loff[s + 1] > loff[s];
        ok = has;
        row_idx[o] = (int32_t)(sel ? sel[s] : s);
        elem_idx[o] = has ? loff[s] + (int32_t)k : -1;
        if (pos) pos[o] = has ? (int32_t)k : 0;
    }
    if (pos_valid) {
        const uint32_t w = __ballot_sync(FULL_MASK, ok);
        if (lane_id() == 0 && o < n_out) pos_valid[o >> 5] = w;
    }
}
void explode_map(Ctx& ctx, const Column& list, const int32_t* sel, const Buf& rows_cum, int64_t r0, int64_t r1, int64_t n_out, int32_t* row_idx,
                 int32_t* elem_idx, int32_t* pos, uint32_t* pos_valid) {
    if (!n_out) return;
    ProfScope ps(ctx, "explode_map");
    explode_map_kernel<<<grid_of(n_out), 256, 0, ctx.stream>>>(P<int32_t>(list.offsets), list.vbits(), sel, P<int64_t>(rows_cum), r0, r1, n_out, row_idx,
                                                               elem_idx, pos, pos_valid);
    LAUNCH_CHECK(ctx);
}

}  // namespace auron
