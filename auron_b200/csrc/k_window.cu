// k_window.cu -- window functions over rows that arrive sorted by (partition keys, order keys), the contract of WindowExec
// (datafusion-ext-plans/src/window_exec.rs:162-345, window/processors/*.rs).  The reference walks the rows one by one and
// carries (current partition, current order key, rank, accumulator) from row to row; on the GPU the same recurrences are
// segmented scans:
//   partition / peer-group boundaries   flags[i] = row i differs from row i - 1 in the partition (order) keys
//   ROW_NUMBER                          segmented inclusive sum of 1, reset at partition boundaries      (row_number_processor.rs)
//   DENSE_RANK                          segmented inclusive sum of the peer-group flags                  (rank_processor.rs, is_dense)
//   RANK                                segmented running max of (peer-group start ? row_number : 0)     (rank_processor.rs)
//   SUM / COUNT / MIN / MAX / AVG       segmented inclusive scan of the argument: the accumulator after every row,
//                                       partial_update + final_merge per row                             (agg_processor.rs:49-93)
// One scan = three launches: a block-local segmented scan of 2048 elements that also reports the block's aggregate and its first
// boundary, one block that scans the block aggregates, and a fix-up of the elements in front of each block's first boundary.
// WindowExec feeds the input batch by batch: a scan may start from a carry (its value at the last row of the previous batch), and
// row 0's boundary flags compare it with that row's keys.  The carry enters the block-aggregate scan as what reaches block 0 from
// the left and the fix-up applies it: no new kernel, but a carried scan always runs those two launches, also when its batch fits in
// one block of 2048 elements.
#include "device_utils.cuh"
#include "kernels.h"
#include "rowkeys.cuh"

namespace auron {

#define LAUNCH_CHECK(ctx)            \
    do {                             \
        CUDA_OK(cudaGetLastError()); \
        launch_count(ctx);           \
    } while (0)

// prev (has_prev): one-row key set holding the last row of the previous batch
__global__ void __launch_bounds__(256) win_flags_kernel(RowKeys keys, RowKeys prev, int has_prev, int64_t n, const uint8_t* __restrict__ also, uint8_t* __restrict__ flags) {
    const int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x;
    if (i >= n) return;
    bool f = (also && also[i]) || (i == 0 && !has_prev);
    if (!f && keys.ncols > 0) f = i == 0 ? !rowkey_equal(prev, 0, keys, 0) : !rowkey_equal(keys, i - 1, keys, i);
    flags[i] = f ? 1 : 0;
}
Buf window_boundaries(Ctx& ctx, const std::vector<ColumnPtr>& keys, int64_t n, const uint8_t* also, const std::vector<ColumnPtr>* prev) {
    Buf flags = dalloc(ctx, (size_t)std::max<int64_t>(n, 1));
    if (n == 0) return flags;
    RowKeys rk{}, pk{};
    if (!keys.empty()) rk = make_row_keys(keys);
    if (prev && !prev->empty()) {
        AURON_CHECK(prev->size() == keys.size(), "window boundaries: the previous row has other keys");
        pk = make_row_keys(*prev);
    }
    win_flags_kernel<<<(unsigned)((n + 255) / 256), 256, 0, ctx.stream>>>(rk, pk, prev ? 1 : 0, n, also, P<uint8_t>(flags));
    LAUNCH_CHECK(ctx);
    return flags;
}
// last row that starts a new group, stored + 1 (0: none); row 0 counts when it differs from the one-row key set prev
__global__ void __launch_bounds__(256) win_last_boundary_kernel(RowKeys keys, RowKeys prev, int has_prev, int64_t n, unsigned* __restrict__ last) {
    const int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x;
    bool f = false;
    if (i < n) f = i > 0 ? !rowkey_equal(keys, i - 1, keys, i) : (has_prev && !rowkey_equal(prev, 0, keys, 0));
    const unsigned m = __reduce_max_sync(FULL_MASK, f ? (unsigned)i + 1 : 0u);
    if (lane_id() == 0 && m) atomicMax(last, m);
}
int64_t window_last_boundary(Ctx& ctx, const std::vector<ColumnPtr>& keys, int64_t n, const std::vector<ColumnPtr>* prev) {
    if (n == 0 || keys.empty()) return -1;
    AURON_CHECK(n < (int64_t)UINT32_MAX, "window batch of 2^32 rows or more");
    RowKeys pk{};
    if (prev) {
        AURON_CHECK(prev->size() == keys.size(), "window boundaries: the previous row has other keys");
        pk = make_row_keys(*prev);
    }
    Buf last = dalloc_zero(ctx, 4);
    win_last_boundary_kernel<<<(unsigned)((n + 255) / 256), 256, 0, ctx.stream>>>(make_row_keys(keys), pk, prev ? 1 : 0, n, P<unsigned>(last));
    LAUNCH_CHECK(ctx);
    unsigned h = 0;
    to_host(ctx, &h, last->ptr, 4);
    return (int64_t)h - 1;
}

enum { WOP_ADD = 0, WOP_MIN = 1, WOP_MAX = 2 };
template <typename T, int OP>
__device__ __forceinline__ T wop(T a, T b) {
    if (OP == WOP_ADD) return a + b;
    if (OP == WOP_MIN) return a < b ? a : b;
    return a > b ? a : b;
}
template <>
__device__ __forceinline__ long long wop<long long, WOP_ADD>(long long a, long long b) {
    return (long long)((unsigned long long)a + (unsigned long long)b);   // wrapping, as the reference's i64 sum
}
// decimal128: wrapping i128 sum (sum.rs:115), signed compare (maxmin.rs)
template <>
__device__ __forceinline__ i128 wop<i128, WOP_ADD>(i128 a, i128 b) { return i128_add(a, b); }
template <>
__device__ __forceinline__ i128 wop<i128, WOP_MIN>(i128 a, i128 b) { return i128_cmp(a, b) <= 0 ? a : b; }
template <>
__device__ __forceinline__ i128 wop<i128, WOP_MAX>(i128 a, i128 b) { return i128_cmp(a, b) >= 0 ? a : b; }

// the combine step of a scan: V is the scanned type
template <typename T, int OP>
struct WinOp {
    using V = T;
    __device__ __forceinline__ T operator()(T a, T b) const { return wop<T, OP>(a, b); }
};
// MIN / MAX of utf8 / binary rows named by their index (-1: no value yet), byte-wise so a shorter prefix sorts first (maxmin.rs:149-165)
struct WinStrOp {
    using V = int32_t;
    const uint8_t* data;
    const int32_t* offs;
    int is_max;
    __device__ __forceinline__ int32_t operator()(int32_t a, int32_t b) const {
        if (a < 0) return b;
        if (b < 0) return a;
        const int c = str_row_cmp(data, offs, a, b);
        return (is_max ? c < 0 : c > 0) ? b : a;
    }
};
template <typename T>
__device__ __forceinline__ T win_shfl(T v, int k) { return __shfl_sync(FULL_MASK, v, k); }
__device__ __forceinline__ i128 win_shfl(i128 v, int k) {   // __shfl_sync moves at most 8 bytes
    return {(uint64_t)__shfl_sync(FULL_MASK, (unsigned long long)v.lo, k), (int64_t)__shfl_sync(FULL_MASK, (long long)v.hi, k)};
}
constexpr int WIN_ITEMS = 8, WIN_TILE = 256 * WIN_ITEMS;

// block-local inclusive segmented scan; blk_val / blk_flag: the block's aggregate; blk_first: index inside the block of its first boundary (WIN_TILE = none)
template <typename Op>
__global__ void __launch_bounds__(256) win_scan_local(Op op, const typename Op::V* __restrict__ in, const uint8_t* __restrict__ flags, int64_t n, typename Op::V* __restrict__ out,
                                                      typename Op::V* __restrict__ blk_val, uint8_t* __restrict__ blk_flag, int32_t* __restrict__ blk_first) {
    using T = typename Op::V;
    __shared__ T s_val[256];
    __shared__ uint8_t s_flag[256];
    __shared__ int s_first;
    const int64_t base = (int64_t)blockIdx.x * WIN_TILE + (int64_t)threadIdx.x * WIN_ITEMS;
    if (threadIdx.x == 0) s_first = WIN_TILE;
    __syncthreads();
    T v[WIN_ITEMS];
    bool f[WIN_ITEMS];
    T acc = T();
    bool any = false, have = false;
    int first = WIN_TILE;
#pragma unroll
    for (int k = 0; k < WIN_ITEMS; k++) {
        const int64_t i = base + k;
        f[k] = i < n && flags[i];
        if (i < n) {
            const T x = in[i];
            acc = (f[k] || !have) ? x : op(acc, x);
            have = true;
            v[k] = acc;
            if (f[k]) {
                any = true;
                if (first == WIN_TILE) first = threadIdx.x * WIN_ITEMS + k;
            }
        } else v[k] = T();
    }
    if (first != WIN_TILE) atomicMin(&s_first, first);
    s_val[threadIdx.x] = acc;
    s_flag[threadIdx.x] = any ? 1 : (have ? 0 : 2);   // 2: the thread holds no element (identity)
    __syncthreads();
    // inclusive scan of the thread aggregates (Hillis-Steele, 8 rounds)
    for (int d = 1; d < 256; d <<= 1) {
        T pv = T();
        uint8_t pf = 2;
        if ((int)threadIdx.x >= d) {
            pv = s_val[threadIdx.x - d];
            pf = s_flag[threadIdx.x - d];
        }
        __syncthreads();
        const uint8_t mf = s_flag[threadIdx.x];
        if ((int)threadIdx.x >= d && pf != 2) {
            if (mf == 2) {
                s_val[threadIdx.x] = pv;
                s_flag[threadIdx.x] = pf;
            } else if (mf == 0) {
                s_val[threadIdx.x] = op(pv, s_val[threadIdx.x]);
                s_flag[threadIdx.x] = pf;
            }   // mf == 1: a boundary inside this span: nothing from the left reaches its end
        }
        __syncthreads();
    }
    // exclusive prefix of this thread = inclusive result of the thread before it; applies to the items in front of the thread's first boundary
    T pre = T();
    bool pre_have = false;
    if (threadIdx.x > 0 && s_flag[threadIdx.x - 1] != 2) {
        pre = s_val[threadIdx.x - 1];
        pre_have = true;
    }
    bool open = true;
#pragma unroll
    for (int k = 0; k < WIN_ITEMS; k++) {
        const int64_t i = base + k;
        if (i >= n) break;
        if (f[k]) open = false;
        out[i] = (open && pre_have) ? op(pre, v[k]) : v[k];
    }
    if (threadIdx.x == 255) {
        blk_val[blockIdx.x] = s_val[255];
        blk_flag[blockIdx.x] = s_flag[255] == 1 ? 1 : 0;
    }
    __syncthreads();
    if (threadIdx.x == 0) blk_first[blockIdx.x] = s_first;
}
// exclusive segmented scan of the block aggregates by ONE warp: carry[b] = what reaches block b from the left (has[b] = 0: nothing).
// 32 aggregates are loaded at a time (coalesced) and folded through shuffles, so the serial chain never waits on memory
// (a few hundred thousand blocks at most).  init (optional): what reaches block 0 -- the scan's value at the previous batch's last row.
template <typename Op>
__global__ void __launch_bounds__(32) win_scan_blocks(Op op, const typename Op::V* __restrict__ blk_val, const uint8_t* __restrict__ blk_flag, int nb,
                                                      const typename Op::V* __restrict__ init, typename Op::V* __restrict__ carry, uint8_t* __restrict__ has) {
    using T = typename Op::V;
    const int lane = threadIdx.x;
    T acc = init ? *init : T();
    bool have = init != nullptr;
    for (int b0 = 0; b0 < nb; b0 += 32) {
        const int b = b0 + lane;
        const T v = b < nb ? blk_val[b] : T();
        const int f = b < nb ? (int)blk_flag[b] : 0;
        T my_carry = T();
        bool my_has = false;
        for (int k = 0; k < 32 && b0 + k < nb; k++) {
            const T vk = win_shfl(v, k);
            const int fk = __shfl_sync(FULL_MASK, f, k);
            if (lane == k) {
                my_carry = acc;
                my_has = have;
            }
            acc = (fk || !have) ? vk : op(acc, vk);
            have = true;
        }
        if (b < nb) {
            carry[b] = my_carry;
            has[b] = my_has ? 1 : 0;
        }
    }
}
template <typename Op>
__global__ void __launch_bounds__(256) win_scan_fix(Op op, typename Op::V* __restrict__ out, int64_t n, const typename Op::V* __restrict__ carry, const uint8_t* __restrict__ has,
                                                    const int32_t* __restrict__ blk_first) {
    const int b = blockIdx.x;
    if (!has[b]) return;
    const int first = blk_first[b];
    const typename Op::V c = carry[b];
    for (int k = threadIdx.x; k < first; k += 256) {
        const int64_t i = (int64_t)b * WIN_TILE + k;
        if (i < n) out[i] = op(c, out[i]);
    }
}
// init (device, optional): the scan's value at the last row of the previous batch; it reaches the rows in front of the first boundary
template <typename Op>
static Buf seg_scan(Ctx& ctx, Op op, const typename Op::V* in, const uint8_t* flags, int64_t n, const typename Op::V* init) {
    using T = typename Op::V;
    Buf out = dalloc(ctx, (size_t)std::max<int64_t>(n, 1) * sizeof(T));
    if (n == 0) return out;
    const int nb = (int)((n + WIN_TILE - 1) / WIN_TILE);
    Buf bv = dalloc(ctx, (size_t)nb * sizeof(T)), bf = dalloc(ctx, (size_t)nb), bfirst = dalloc(ctx, (size_t)nb * 4);
    Buf carry = dalloc(ctx, (size_t)nb * sizeof(T)), has = dalloc(ctx, (size_t)nb);
    win_scan_local<Op><<<nb, 256, 0, ctx.stream>>>(op, in, flags, n, P<T>(out), P<T>(bv), P<uint8_t>(bf), P<int32_t>(bfirst));
    LAUNCH_CHECK(ctx);
    if (nb > 1 || init) {
        win_scan_blocks<Op><<<1, 32, 0, ctx.stream>>>(op, P<T>(bv), P<uint8_t>(bf), nb, init, P<T>(carry), P<uint8_t>(has));
        LAUNCH_CHECK(ctx);
        win_scan_fix<Op><<<nb, 256, 0, ctx.stream>>>(op, P<T>(out), n, P<T>(carry), P<uint8_t>(has), P<int32_t>(bfirst));
        LAUNCH_CHECK(ctx);
    }
    return out;
}
template <typename T>
static Buf window_scan(Ctx& ctx, const T* in, const uint8_t* flags, int64_t n, int op, const T* init = nullptr) {
    ProfScope ps(ctx, "window_scan");
    if (op == WOP_ADD) return seg_scan(ctx, WinOp<T, WOP_ADD>{}, in, flags, n, init);
    if (op == WOP_MIN) return seg_scan(ctx, WinOp<T, WOP_MIN>{}, in, flags, n, init);
    return seg_scan(ctx, WinOp<T, WOP_MAX>{}, in, flags, n, init);
}
// the element at row n - 1 of a scan output, as the carry of the next batch
static Buf win_last(Ctx& ctx, const Buf& b, int64_t n, size_t w) {
    Buf c = dalloc(ctx, w);
    CUDA_OK(cudaMemcpyAsync(c->ptr, (const uint8_t*)b->ptr + (size_t)(n - 1) * w, w, cudaMemcpyDeviceToDevice, ctx.stream));
    return c;
}
template <typename T>
static const T* win_init(const Buf& b) { return b ? P<T>(b) : nullptr; }

static unsigned wgrid(int64_t n) { return (unsigned)((n + 255) / 256); }

// ---- element-wise helpers around the scans
__global__ void __launch_bounds__(256) win_fill_i64(long long* out, int64_t n, long long v) {
    const int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x;
    if (i < n) out[i] = v;
}
__global__ void __launch_bounds__(256) win_flags_to_i64(const uint8_t* __restrict__ f, int64_t n, long long* __restrict__ out) {
    const int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x;
    if (i < n) out[i] = f[i] ? 1 : 0;
}
__global__ void __launch_bounds__(256) win_rank_seed(const long long* __restrict__ rn, const uint8_t* __restrict__ oflags, int64_t n, long long* __restrict__ out) {
    const int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x;
    if (i < n) out[i] = oflags[i] ? rn[i] : 0;
}
__global__ void __launch_bounds__(256) win_i64_to_i32(const long long* __restrict__ in, int64_t n, int32_t* __restrict__ out) {
    const int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x;
    if (i < n) out[i] = (int32_t)in[i];
}
// argument column -> (value or identity, 1 if valid) as int64 / double
template <typename S, typename T>
__global__ void __launch_bounds__(256) win_arg_kernel(const S* __restrict__ data, const uint8_t* __restrict__ valid, int64_t n, T identity, T* __restrict__ val, long long* __restrict__ cnt) {
    const int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x;
    if (i >= n) return;
    const bool ok = !valid || bit_get(valid, i);
    if (val) val[i] = ok ? (T)data[i] : identity;
    if (cnt) cnt[i] = ok ? 1 : 0;
}
// boolean argument (a bitmap) -> 0 / 1 as int64: false < true
__global__ void __launch_bounds__(256) win_arg_bool(const uint8_t* __restrict__ data, const uint8_t* __restrict__ valid, int64_t n, long long identity, long long* __restrict__ val,
                                                    long long* __restrict__ cnt) {
    const int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x;
    if (i >= n) return;
    const bool ok = !valid || bit_get(valid, i);
    val[i] = ok ? (long long)bit_get(data, i) : identity;
    cnt[i] = ok ? 1 : 0;
}
__global__ void __launch_bounds__(256) win_arg_dec(const ulonglong2* __restrict__ data, const uint8_t* __restrict__ valid, int64_t n, i128 identity, i128* __restrict__ val,
                                                   long long* __restrict__ cnt) {
    const int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x;
    if (i >= n) return;
    const bool ok = !valid || bit_get(valid, i);
    if (ok) {
        const ulonglong2 x = data[i];
        val[i] = {x.x, (int64_t)x.y};
    } else val[i] = identity;
    cnt[i] = ok ? 1 : 0;
}
// utf8 / binary argument -> its row index, -1 where NULL (m rows: the argument's n and possibly the carried value at row n)
__global__ void __launch_bounds__(256) win_arg_row(const uint8_t* __restrict__ valid, int64_t m, int32_t* __restrict__ idx) {
    const int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x;
    if (i < m) idx[i] = (!valid || bit_get(valid, i)) ? (int32_t)i : -1;
}
__global__ void __launch_bounds__(256) win_valid_from_count(const long long* __restrict__ cnt, int64_t n, uint32_t* __restrict__ valid) {
    const int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x;
    const uint32_t w = __ballot_sync(FULL_MASK, i < n && cnt[i] > 0);
    if (lane_id() == 0 && i < n) valid[i >> 5] = w;
}
__global__ void __launch_bounds__(256) win_avg_kernel(const double* __restrict__ sum_f, const long long* __restrict__ sum_i, const long long* __restrict__ cnt, int64_t n, double* __restrict__ out) {
    const int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x;
    if (i < n) out[i] = cnt[i] > 0 ? (sum_f ? sum_f[i] : (double)sum_i[i]) / (double)cnt[i] : 0.0;
}
template <typename T>
__global__ void __launch_bounds__(256) win_narrow_kernel(const long long* __restrict__ in, int64_t n, T* __restrict__ out) {
    const int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x;
    if (i < n) out[i] = (T)in[i];
}
__global__ void __launch_bounds__(256) win_i64_to_bool(const long long* __restrict__ in, int64_t n, uint32_t* __restrict__ out) {
    const int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x;
    const uint32_t w = __ballot_sync(FULL_MASK, i < n && in[i] != 0);
    if (lane_id() == 0 && i < n) out[i >> 5] = w;
}
__global__ void __launch_bounds__(256) win_f64_to_f32(const double* __restrict__ in, int64_t n, float* __restrict__ out) {
    const int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x;
    if (i < n) out[i] = (float)in[i];
}
__global__ void __launch_bounds__(256) win_le_mask(const int32_t* __restrict__ v, int64_t n, int32_t k, uint32_t* __restrict__ mask) {
    const int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x;
    const uint32_t w = __ballot_sync(FULL_MASK, i < n && v[i] <= k);
    if (lane_id() == 0 && i < n) mask[i >> 5] = w;
}

// carry: a = the row number (ROW_NUMBER, RANK) or the dense rank, b = the rank (RANK)
ColumnPtr window_rank_column(Ctx& ctx, int func, const uint8_t* pflags, const uint8_t* oflags, int64_t n, WinCarry* carry) {
    // func: 0 ROW_NUMBER, 1 RANK, 2 DENSE_RANK ; Int32 output like the reference's builders
    auto col = make_column(ctx, DType(T_INT32), n, false);
    if (n == 0) return col;
    Buf tmp = dalloc(ctx, (size_t)n * 8);
    Buf res;
    const long long* init_a = carry ? win_init<long long>(carry->a) : nullptr;
    if (func == 2) {
        win_flags_to_i64<<<wgrid(n), 256, 0, ctx.stream>>>(oflags, n, P<long long>(tmp));
        LAUNCH_CHECK(ctx);
        res = window_scan<long long>(ctx, P<long long>(tmp), pflags, n, WOP_ADD, init_a);
        if (carry) carry->a = win_last(ctx, res, n, 8);
    } else {
        win_fill_i64<<<wgrid(n), 256, 0, ctx.stream>>>(P<long long>(tmp), n, 1);
        LAUNCH_CHECK(ctx);
        Buf rn = window_scan<long long>(ctx, P<long long>(tmp), pflags, n, WOP_ADD, init_a);   // row numbers
        res = rn;
        if (func == 1) {
            win_rank_seed<<<wgrid(n), 256, 0, ctx.stream>>>(P<long long>(rn), oflags, n, P<long long>(tmp));
            LAUNCH_CHECK(ctx);
            res = window_scan<long long>(ctx, P<long long>(tmp), pflags, n, WOP_MAX, carry ? win_init<long long>(carry->b) : nullptr);
            if (carry) carry->b = win_last(ctx, res, n, 8);
        }
        if (carry) carry->a = win_last(ctx, rn, n, 8);
    }
    win_i64_to_i32<<<wgrid(n), 256, 0, ctx.stream>>>(P<long long>(res), n, P<int32_t>(col->data));
    LAUNCH_CHECK(ctx);
    return col;
}

// running MIN / MAX of a utf8 / binary argument: a scan over row indices whose combine step compares the rows' bytes, then one
// gather.  The carried value is row n of (argument, carried value), so every batch after the first copies its argument once
// (profiled as window_string_carry); the carry becomes the result's last row.
static ColumnPtr window_str_extreme(Ctx& ctx, bool is_max, const ColumnPtr& arg, const uint8_t* pflags, int64_t n, WinCarry* carry) {
    const bool carried = carry && carry->value;
    ColumnPtr src = arg;
    if (carried) {   // a copy of the argument's bytes and offsets, one row longer
        ProfScope ps(ctx, "window_string_carry");
        src = concat_columns(ctx, {arg, carry->value});
    }
    const int64_t m = carried ? n + 1 : n;
    AURON_CHECK(m < (int64_t)INT32_MAX, "string MIN / MAX window over 2^31 rows in one batch");
    Buf idx = dalloc(ctx, (size_t)m * 4);
    win_arg_row<<<wgrid(m), 256, 0, ctx.stream>>>(src->vbits(), m, P<int32_t>(idx));
    LAUNCH_CHECK(ctx);
    Buf res;
    {
        ProfScope ps(ctx, "window_scan");
        res = seg_scan(ctx, WinStrOp{P<uint8_t>(src->data), P<int32_t>(src->offsets), is_max ? 1 : 0}, P<int32_t>(idx), pflags, n, carried ? P<int32_t>(idx) + n : nullptr);
    }
    ColumnPtr out = take(ctx, *src, P<int32_t>(res), n, true);
    if (carry) carry->value = slice_column(ctx, *out, n - 1, 1);
    return out;
}

// running aggregate of `arg` inside the partitions given by pflags; fn: AggFunction of the plan (0 MIN, 1 MAX, 2 SUM, 3 AVG, 4 COUNT).
// carry: a = the running count, b = the running value; value = the running string MIN / MAX
ColumnPtr window_agg_column(Ctx& ctx, int fn, const ColumnPtr& arg, const DType& out_type, const uint8_t* pflags, int64_t n, WinCarry* carry) {
    const DType& at = arg->type;
    const bool is_float = at.is_float();
    const bool is_int = at.is_intlike() || at.id == T_BOOL;   // the int64 plane; MIN / MAX only for bool, date64 and timestamps
    const bool is_dec = at.id == T_DECIMAL128;
    const bool minmax = fn == 0 || fn == 1;
    AURON_CHECK(fn == 4 || is_float || is_int || is_dec || (minmax && at.is_varlen()), "window aggregate #" + std::to_string(fn) + " over " + at.str() + " is not supported on device");
    if (fn != 4 && at.is_varlen()) {
        AURON_CHECK(out_type == at, "string MIN / MAX window returns its argument's type");
        return window_str_extreme(ctx, fn == 1, arg, pflags, n, carry);
    }
    auto out = make_column(ctx, out_type, n, fn != 4);
    if (n == 0) return out;
    const uint8_t* valid = arg->vbits();
    Buf cnt_in = dalloc(ctx, (size_t)n * 8);
    Buf vi, vf, vd;   // value plane as int64, double or i128
    const int op = fn == 0 ? WOP_MIN : fn == 1 ? WOP_MAX : WOP_ADD;
    auto launch_arg = [&](auto tag_src) {
        using S = decltype(tag_src);
        if (is_float) {
            vf = dalloc(ctx, (size_t)n * 8);
            const double id = op == WOP_MIN ? __builtin_inf() : op == WOP_MAX ? -__builtin_inf() : 0.0;
            win_arg_kernel<S, double><<<wgrid(n), 256, 0, ctx.stream>>>((const S*)arg->data->ptr, valid, n, id, fn == 4 ? nullptr : P<double>(vf), P<long long>(cnt_in));
        } else {
            vi = dalloc(ctx, (size_t)n * 8);
            const long long id = op == WOP_MIN ? 0x7fffffffffffffffll : op == WOP_MAX ? (-0x7fffffffffffffffll - 1) : 0ll;
            win_arg_kernel<S, long long><<<wgrid(n), 256, 0, ctx.stream>>>((const S*)arg->data->ptr, valid, n, id, fn == 4 ? nullptr : P<long long>(vi), P<long long>(cnt_in));
        }
        LAUNCH_CHECK(ctx);
    };
    switch (fn == 4 ? T_NULL : at.id) {   // COUNT: only the validity matters
        case T_INT8: launch_arg((int8_t)0); break;
        case T_INT16: launch_arg((int16_t)0); break;
        case T_INT32: case T_DATE32: launch_arg((int32_t)0); break;
        case T_INT64: case T_DATE64: case T_TIMESTAMP: launch_arg((long long)0); break;
        case T_FLOAT32: launch_arg((float)0); break;
        case T_FLOAT64: launch_arg((double)0); break;
        case T_BOOL:
            vi = dalloc(ctx, (size_t)n * 8);
            win_arg_bool<<<wgrid(n), 256, 0, ctx.stream>>>(P<uint8_t>(arg->data), valid, n, op == WOP_MIN ? 1ll : 0ll, P<long long>(vi), P<long long>(cnt_in));
            LAUNCH_CHECK(ctx);
            break;
        case T_DECIMAL128: {
            vd = dalloc(ctx, (size_t)n * 16);
            const i128 id = op == WOP_MIN ? i128{~0ull, 0x7fffffffffffffffll} : op == WOP_MAX ? i128{0ull, (-0x7fffffffffffffffll - 1)} : i128{0ull, 0ll};
            win_arg_dec<<<wgrid(n), 256, 0, ctx.stream>>>(P<ulonglong2>(arg->data), valid, n, id, P<i128>(vd), P<long long>(cnt_in));
            LAUNCH_CHECK(ctx);
            break;
        }
        default:
            win_arg_kernel<uint8_t, long long><<<wgrid(n), 256, 0, ctx.stream>>>(nullptr, valid, n, 0ll, nullptr, P<long long>(cnt_in));
            LAUNCH_CHECK(ctx);
    }
    Buf cnt = window_scan<long long>(ctx, P<long long>(cnt_in), pflags, n, WOP_ADD, carry ? win_init<long long>(carry->a) : nullptr);
    if (carry) carry->a = win_last(ctx, cnt, n, 8);
    if (fn == 4) {   // COUNT: int64, never NULL
        AURON_CHECK(out_type.id == T_INT64, "COUNT window must return int64");
        CUDA_OK(cudaMemcpyAsync(out->data->ptr, cnt->ptr, (size_t)n * 8, cudaMemcpyDeviceToDevice, ctx.stream));
        return out;
    }
    Buf ri, rf, rd;
    if (is_dec) rd = window_scan<i128>(ctx, P<i128>(vd), pflags, n, op, carry ? win_init<i128>(carry->b) : nullptr);
    else if (is_float) rf = window_scan<double>(ctx, P<double>(vf), pflags, n, op, carry ? win_init<double>(carry->b) : nullptr);
    else ri = window_scan<long long>(ctx, P<long long>(vi), pflags, n, op, carry ? win_init<long long>(carry->b) : nullptr);
    if (carry) carry->b = is_dec ? win_last(ctx, rd, n, 16) : win_last(ctx, is_float ? rf : ri, n, 8);
    if (fn == 3 && is_dec) {   // AVG over decimals: the running sum's checked_div_euclid(count) at the declared scale (avg.rs:161-168)
        AURON_CHECK(out_type.id == T_DECIMAL128, "AVG window over decimals returns a decimal");
        Column sum, count;
        sum.type = out_type;
        sum.len = n;
        sum.data = rd;
        count.type = DType(T_INT64);
        count.len = n;
        count.data = cnt;
        return avg_finalize(ctx, sum, count, out_type);
    }
    win_valid_from_count<<<wgrid(n), 256, 0, ctx.stream>>>(P<long long>(cnt), n, P<uint32_t>(out->validity));
    LAUNCH_CHECK(ctx);
    out->null_count = -1;
    if (fn == 3) {   // AVG -> double
        AURON_CHECK(out_type.id == T_FLOAT64, "AVG window over integers / floats returns float64");
        win_avg_kernel<<<wgrid(n), 256, 0, ctx.stream>>>(is_float ? P<double>(rf) : nullptr, is_float ? nullptr : P<long long>(ri), P<long long>(cnt), n, P<double>(out->data));
        LAUNCH_CHECK(ctx);
        return out;
    }
    // SUM / MIN / MAX: narrow to the declared type
    if (is_dec) {
        AURON_CHECK(out_type.id == T_DECIMAL128, "window aggregate: decimal argument with result type " + out_type.str());
        CUDA_OK(cudaMemcpyAsync(out->data->ptr, rd->ptr, (size_t)n * 16, cudaMemcpyDeviceToDevice, ctx.stream));
    } else if (is_float) {
        if (out_type.id == T_FLOAT64) CUDA_OK(cudaMemcpyAsync(out->data->ptr, rf->ptr, (size_t)n * 8, cudaMemcpyDeviceToDevice, ctx.stream));
        else if (out_type.id == T_FLOAT32) {
            win_f64_to_f32<<<wgrid(n), 256, 0, ctx.stream>>>(P<double>(rf), n, P<float>(out->data));
            LAUNCH_CHECK(ctx);
        } else fail("window aggregate: float argument with result type " + out_type.str());
    } else {
        switch (out_type.id) {
            case T_INT64: case T_DATE64: case T_TIMESTAMP: CUDA_OK(cudaMemcpyAsync(out->data->ptr, ri->ptr, (size_t)n * 8, cudaMemcpyDeviceToDevice, ctx.stream)); break;
            case T_INT32: case T_DATE32: win_narrow_kernel<int32_t><<<wgrid(n), 256, 0, ctx.stream>>>(P<long long>(ri), n, P<int32_t>(out->data)); LAUNCH_CHECK(ctx); break;
            case T_INT16: win_narrow_kernel<int16_t><<<wgrid(n), 256, 0, ctx.stream>>>(P<long long>(ri), n, P<int16_t>(out->data)); LAUNCH_CHECK(ctx); break;
            case T_INT8: win_narrow_kernel<int8_t><<<wgrid(n), 256, 0, ctx.stream>>>(P<long long>(ri), n, P<int8_t>(out->data)); LAUNCH_CHECK(ctx); break;
            case T_BOOL: win_i64_to_bool<<<wgrid(n), 256, 0, ctx.stream>>>(P<long long>(ri), n, P<uint32_t>(out->data)); LAUNCH_CHECK(ctx); break;
            default: fail("window aggregate: integer argument with result type " + out_type.str());
        }
    }
    return out;
}

// ---- functions that look at the whole partition: PERCENT_RANK, CUME_DIST, LEAD, NTH_VALUE (window/processors/{percent_rank,cume_dist,
// lead,nth_value}_processor.rs).  Everything is derived from per-row scans plus one scatter to the first row of a group:
//   start[i]   first row of row i's partition            running max of (boundary ? i : 0)
//   size       rows of the partition                     row number of the partition's last row, scattered to start, gathered back
//   peer end   rows of the partition up to the end of the current peer group: the same with the order boundaries
__global__ void __launch_bounds__(256) win_start_seed(const uint8_t* __restrict__ flags, int64_t n, long long* __restrict__ out) {
    const int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x;
    if (i < n) out[i] = flags[i] ? i : 0;
}
// rn of the last row of every group (flags mark group starts) -> at_start[start of the group]
__global__ void __launch_bounds__(256) win_scatter_last(const long long* __restrict__ rn, const uint8_t* __restrict__ flags, const long long* __restrict__ start, int64_t n,
                                                        long long* __restrict__ at_start) {
    const int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x;
    if (i < n && (i == n - 1 || flags[i + 1])) at_start[start[i]] = rn[i];
}
__global__ void __launch_bounds__(256) win_percent_rank_kernel(const long long* __restrict__ rank, const long long* __restrict__ size_at, const long long* __restrict__ pstart, int64_t n,
                                                               double* __restrict__ out) {
    const int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x;
    if (i >= n) return;
    const long long size = size_at[pstart[i]];
    out[i] = size <= 1 ? 0.0 : (double)(rank[i] - 1) / (double)(size - 1);
}
__global__ void __launch_bounds__(256) win_cume_dist_kernel(const long long* __restrict__ peer_at, const long long* __restrict__ ostart, const long long* __restrict__ size_at,
                                                            const long long* __restrict__ pstart, int64_t n, double* __restrict__ out) {
    const int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x;
    if (i < n) out[i] = (double)peer_at[ostart[i]] / (double)size_at[pstart[i]];
}
// LEAD: row i + offset if it lies in the same partition, else the row's default, which sits at n + i of the concatenated (values, defaults) column
__global__ void __launch_bounds__(256) win_lead_idx(const long long* __restrict__ pstart, int64_t n, int64_t offset, int32_t* __restrict__ idx) {
    const int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x;
    if (i >= n) return;
    const int64_t t = i + offset;
    idx[i] = (t >= 0 && t < n && pstart[t] == pstart[i]) ? (int32_t)t : (int32_t)(n + i);
}
// NTH_VALUE: the row at which the running count reaches `nth` for the first time -> at_start; then -1 (NULL) until the count is there
__global__ void __launch_bounds__(256) win_nth_scatter(const long long* __restrict__ cnt, const uint8_t* __restrict__ counts_here, const long long* __restrict__ pstart, int64_t n,
                                                       long long nth, long long* __restrict__ at_start) {
    const int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x;
    if (i < n && cnt[i] == nth && counts_here[i]) at_start[pstart[i]] = i;
}
__global__ void __launch_bounds__(256) win_nth_idx(const long long* __restrict__ cnt, const long long* __restrict__ pstart, const long long* __restrict__ at_start, int64_t n, long long nth,
                                                   int32_t* __restrict__ idx) {
    const int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x;
    if (i < n) idx[i] = cnt[i] >= nth ? (int32_t)at_start[pstart[i]] : -1;
}
__global__ void __launch_bounds__(256) win_valid_bytes(const uint8_t* __restrict__ valid, int64_t n, uint8_t* __restrict__ out, long long* __restrict__ as_i64) {
    const int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x;
    if (i >= n) return;
    const bool ok = !valid || bit_get(valid, i);
    out[i] = ok ? 1 : 0;
    as_i64[i] = ok ? 1 : 0;
}

struct WinFrame {   // per-row scans shared by the functions below
    Buf first_only, pstart, rn, size_at;
};
static WinFrame win_frame(Ctx& ctx, const uint8_t* pflags, int64_t n) {
    WinFrame f;
    f.first_only = window_boundaries(ctx, {}, n, nullptr, nullptr);   // a flag on row 0 only: turns the segmented scan into a plain one
    Buf seed = dalloc(ctx, (size_t)n * 8);
    win_start_seed<<<wgrid(n), 256, 0, ctx.stream>>>(pflags, n, P<long long>(seed));
    LAUNCH_CHECK(ctx);
    f.pstart = window_scan<long long>(ctx, P<long long>(seed), P<uint8_t>(f.first_only), n, WOP_MAX);
    win_fill_i64<<<wgrid(n), 256, 0, ctx.stream>>>(P<long long>(seed), n, 1);
    LAUNCH_CHECK(ctx);
    f.rn = window_scan<long long>(ctx, P<long long>(seed), pflags, n, WOP_ADD);
    f.size_at = dalloc(ctx, (size_t)n * 8);
    win_scatter_last<<<wgrid(n), 256, 0, ctx.stream>>>(P<long long>(f.rn), pflags, P<long long>(f.pstart), n, P<long long>(f.size_at));
    LAUNCH_CHECK(ctx);
    return f;
}
ColumnPtr window_dist_column(Ctx& ctx, int func /* 6 PERCENT_RANK, 7 CUME_DIST */, const uint8_t* pflags, const uint8_t* oflags, int64_t n) {
    auto col = make_column(ctx, DType(T_FLOAT64), n, false);
    if (n == 0) return col;
    WinFrame f = win_frame(ctx, pflags, n);
    Buf tmp = dalloc(ctx, (size_t)n * 8);
    if (func == 6) {
        win_rank_seed<<<wgrid(n), 256, 0, ctx.stream>>>(P<long long>(f.rn), oflags, n, P<long long>(tmp));
        LAUNCH_CHECK(ctx);
        Buf rank = window_scan<long long>(ctx, P<long long>(tmp), pflags, n, WOP_MAX);
        win_percent_rank_kernel<<<wgrid(n), 256, 0, ctx.stream>>>(P<long long>(rank), P<long long>(f.size_at), P<long long>(f.pstart), n, P<double>(col->data));
        LAUNCH_CHECK(ctx);
    } else {
        win_start_seed<<<wgrid(n), 256, 0, ctx.stream>>>(oflags, n, P<long long>(tmp));
        LAUNCH_CHECK(ctx);
        Buf ostart = window_scan<long long>(ctx, P<long long>(tmp), P<uint8_t>(f.first_only), n, WOP_MAX);
        Buf peer_at = dalloc(ctx, (size_t)n * 8);
        win_scatter_last<<<wgrid(n), 256, 0, ctx.stream>>>(P<long long>(f.rn), oflags, P<long long>(ostart), n, P<long long>(peer_at));
        LAUNCH_CHECK(ctx);
        win_cume_dist_kernel<<<wgrid(n), 256, 0, ctx.stream>>>(P<long long>(peer_at), P<long long>(ostart), P<long long>(f.size_at), P<long long>(f.pstart), n, P<double>(col->data));
        LAUNCH_CHECK(ctx);
    }
    return col;
}
// values and defaults have the same type and n rows each
ColumnPtr window_lead_column(Ctx& ctx, const ColumnPtr& values, const ColumnPtr& defaults, int64_t offset, const uint8_t* pflags, int64_t n) {
    if (n == 0) return values;
    AURON_CHECK(2 * n < (int64_t)INT32_MAX, "LEAD over more than 2^30 rows in one task");
    WinFrame f = win_frame(ctx, pflags, n);
    Buf idx = dalloc(ctx, (size_t)n * 4);
    win_lead_idx<<<wgrid(n), 256, 0, ctx.stream>>>(P<long long>(f.pstart), n, offset, P<int32_t>(idx));
    LAUNCH_CHECK(ctx);
    Batch both;
    both.num_rows = 2 * n;
    both.cols.push_back(concat_columns(ctx, {values, defaults}));
    return take_batch(ctx, both, P<int32_t>(idx), n, false)->cols[0];
}
// carry: a = the running count, value = the result at the last row (the found value once the count has reached nth).  A partition
// that continues from the previous batch starts at row 0 here; its found value, when it was found there, is row n of
// (values, carried value), which at[0] points to unless this batch reaches nth itself.
ColumnPtr window_nth_column(Ctx& ctx, const ColumnPtr& values, int64_t nth, bool ignore_nulls, const uint8_t* pflags, int64_t n, WinCarry* carry) {
    if (n == 0) return values;
    WinFrame f = win_frame(ctx, pflags, n);
    Buf counts_here = dalloc(ctx, (size_t)n), seed = dalloc(ctx, (size_t)n * 8);
    win_valid_bytes<<<wgrid(n), 256, 0, ctx.stream>>>(ignore_nulls ? values->vbits() : nullptr, n, P<uint8_t>(counts_here), P<long long>(seed));
    LAUNCH_CHECK(ctx);
    Buf cnt = window_scan<long long>(ctx, P<long long>(seed), pflags, n, WOP_ADD, carry ? win_init<long long>(carry->a) : nullptr);
    Buf at = dalloc(ctx, (size_t)n * 8), idx = dalloc(ctx, (size_t)n * 4);
    const bool carried = carry && carry->value;
    if (carried) {
        win_fill_i64<<<1, 256, 0, ctx.stream>>>(P<long long>(at), 1, n);
        LAUNCH_CHECK(ctx);
    }
    win_nth_scatter<<<wgrid(n), 256, 0, ctx.stream>>>(P<long long>(cnt), P<uint8_t>(counts_here), P<long long>(f.pstart), n, nth, P<long long>(at));
    LAUNCH_CHECK(ctx);
    win_nth_idx<<<wgrid(n), 256, 0, ctx.stream>>>(P<long long>(cnt), P<long long>(f.pstart), P<long long>(at), n, nth, P<int32_t>(idx));
    LAUNCH_CHECK(ctx);
    Batch one;
    one.num_rows = carried ? n + 1 : n;
    one.cols.push_back(carried ? concat_columns(ctx, {values, carry->value}) : values);
    ColumnPtr out = take_batch(ctx, one, P<int32_t>(idx), n, true)->cols[0];
    if (carry) {
        carry->a = win_last(ctx, cnt, n, 8);
        carry->value = slice_column(ctx, *out, n - 1, 1);
    }
    return out;
}

Buf window_le_mask(Ctx& ctx, const ColumnPtr& rank_col, int32_t k) {
    const int64_t n = rank_col->len;
    Buf mask = dalloc_zero(ctx, bitmap_alloc_bytes(n));
    if (n) {
        win_le_mask<<<wgrid(n), 256, 0, ctx.stream>>>(P<int32_t>(rank_col->data), n, k, P<uint32_t>(mask));
        LAUNCH_CHECK(ctx);
    }
    return mask;
}

}  // namespace auron
