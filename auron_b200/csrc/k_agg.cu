// k_agg.cu -- hash aggregation on device (rows A1-A4 of SURVEY.md section 8a).
//
// Replaces AggHashMap::upsert_records (datafusion-ext-plans/src/agg/agg_hash_map.rs:77-136) and the
// Agg::partial_update / partial_merge accumulators (agg/sum.rs:98-157, count.rs:89-157, maxmin.rs:100-296,
// first.rs, acc.rs:233-395) with ONE fused kernel per chunk: each thread finds-or-inserts its row's key
// in an open-addressed table in HBM (linear probing, power-of-two capacity, atomicCAS claim) and then
// scatter-updates every accumulator with native atomics.  A row selection vector (the output of a
// preceding filter) can be consumed directly so Filter -> HashAggregate never materialises filtered rows.
//
// Two key paths:
//   FAST    one key column of <= 8 bytes (ints, dates, floats by bits, decimal precision <= 18): the slot
//           stores the 64-bit key itself.  NULL and the EMPTY sentinel value get two dedicated slots.
//   GENERAL any other key set (multi-column, utf8, wide decimal): the slot stores a representative row
//           index of the chunk; candidate rows are verified with rowkey_equal (NULL == NULL as the
//           reference's row-format grouping keys, agg_ctx.rs:233-245).
// Group output order is unspecified, as in the reference (agg_table.rs:177-205).
//
// Roofline: HBM-bound stream over (key + argument) bytes; the table and accumulators are scratch.
// Algorithmic bytes per row for GROUP BY int64 / SUM(int64) / COUNT = 8 + 8 (+1/8 per validity) = 16 B.
#include "kernels.h"
#include "rowkeys.cuh"

namespace auron {

#define LAUNCH_CHECK(ctx)            \
    do {                             \
        CUDA_OK(cudaGetLastError()); \
        launch_count(ctx);           \
    } while (0)

constexpr int kMaxAccs = 16;
constexpr uint64_t EMPTY_KEY = 0x8A5C3F1E9D7B2461ull;   // sentinel; a real key with this value uses slot `cap`

struct AccDesc {
    int32_t kind;
    int32_t in_type;   // TypeId of the input column
    const void* in;
    const uint8_t* in_valid;
    const uint8_t* extra_valid[3];
    int32_t n_extra;
    int32_t in_is_dec64;   // decimal input with precision <= 18 (MIN/MAX use the low word)
    unsigned long long* acc_lo;
    unsigned long long* acc_hi;
    uint8_t* acc_valid;
    int32_t lo_stride;      // u64 words between consecutive slots (1 = SoA arrays, W = slot records interleaved with the key)
    int32_t valid_stride;   // bytes between consecutive slots' valid flags
    // SUM/MIN/MAX(x) next to COUNT(x) over the same column: the group's accumulator is valid iff that count is non-zero,
    // so the per-row valid-flag store (one more random L2 access per row) is dropped and validity is read from the count.
    const unsigned long long* valid_cnt;
    const int32_t* in_offsets;   // utf8 / binary input (MIN_STR / MAX_STR compare rows through it)
};
struct AccArgs {
    AccDesc a[kMaxAccs];
    int32_t n;
};

struct AccVal {
    uint64_t lo;
    int64_t hi;
};

// order-preserving map of a double onto int64 (IEEE total order)
__device__ __forceinline__ int64_t f64_to_ordered(double d) {
    int64_t b = __double_as_longlong(d);
    return b < 0 ? (b ^ 0x7fffffffffffffffll) : b;
}
__device__ __forceinline__ double ordered_to_f64(int64_t o) {
    int64_t b = o < 0 ? (o ^ 0x7fffffffffffffffll) : o;
    return __longlong_as_double(b);
}

__device__ __forceinline__ int64_t load_int(const void* p, int32_t type, int64_t row) {
    switch (type) {
        case T_INT8: return ((const int8_t*)p)[row];
        case T_INT16: return ((const int16_t*)p)[row];
        case T_INT32: case T_DATE32: return ((const int32_t*)p)[row];
        case T_DECIMAL128: return (int64_t)((const uint64_t*)p)[row * 2];
        default: return ((const int64_t*)p)[row];
    }
}
__device__ __forceinline__ double load_f64(const void* p, int32_t type, int64_t row) {
    if (type == T_FLOAT32) return (double)((const float*)p)[row];
    if (type == T_FLOAT64) return ((const double*)p)[row];
    return (double)load_int(p, type, row);
}

// contribution of one row; returns false when the row contributes nothing (NULL argument)
__device__ __forceinline__ bool acc_load(const AccDesc& d, int64_t row, int64_t pos, AccVal& v) {
    bool ok = valid_at(d.in_valid, row);
    switch (d.kind) {
        case ACC_SUM_I64: case ACC_ADD_I64:
            if (!ok) return false;
            v.lo = (uint64_t)load_int(d.in, d.in_type, row);
            return true;
        case ACC_SUM_F64:
            if (!ok) return false;
            v.lo = (uint64_t)__double_as_longlong(load_f64(d.in, d.in_type, row));
            return true;
        case ACC_SUM_DEC: {
            if (!ok) return false;
            ulonglong2 t = ((const ulonglong2*)d.in)[row];
            v.lo = t.x;
            v.hi = (int64_t)t.y;
            return true;
        }
        case ACC_COUNT:
            for (int e = 0; e < d.n_extra; e++) ok = ok && valid_at(d.extra_valid[e], row);
            if (!ok) return false;
            v.lo = 1;
            return true;
        case ACC_MIN: case ACC_MAX:
            if (!ok) return false;
            if (d.in_type == T_FLOAT32 || d.in_type == T_FLOAT64) v.lo = (uint64_t)f64_to_ordered(load_f64(d.in, d.in_type, row));
            else if (d.in_type == T_BOOL) v.lo = bit_get((const uint8_t*)d.in, row);
            else v.lo = (uint64_t)load_int(d.in, d.in_type, row);
            return true;
        case ACC_FIRST:
            // merge mode: extra_valid[0] holds the partial's is_set bits (first.rs:50 acc = [value, is_set])
            if (d.n_extra > 0 && !bit_get(d.extra_valid[0], row)) return false;
            v.lo = (uint64_t)pos;
            return true;
        case ACC_FIRST_IGNORES_NULL:
            if (!ok) return false;
            v.lo = (uint64_t)pos;
            return true;
        case ACC_MIN_STR: case ACC_MAX_STR:
            if (!ok) return false;
            v.lo = (uint64_t)row;
            return true;
    }
    return false;
}
// STR: the kernel instance handles string extremes (MIN_STR / MAX_STR).  Compiled into every instance, the CAS loop below
// slows the SUM / COUNT path of agg_direct_kernel, so plans without string extremes
// run instances that do not contain it.
template <bool STR = false>
__device__ __forceinline__ void acc_apply(const AccDesc& d, int64_t slot, const AccVal& v) {
    switch (d.kind) {
        case ACC_SUM_I64: case ACC_ADD_I64: case ACC_COUNT:
            atomicAdd(&d.acc_lo[slot * d.lo_stride], (unsigned long long)v.lo);   // wrapping, as sum.rs:115
            break;
        case ACC_SUM_F64:
            atomicAdd((double*)&d.acc_lo[slot * d.lo_stride], __longlong_as_double((int64_t)v.lo));
            break;
        case ACC_SUM_DEC: {
            unsigned long long old = atomicAdd(&d.acc_lo[slot * d.lo_stride], (unsigned long long)v.lo);
            unsigned long long carry = (old + v.lo) < old ? 1ull : 0ull;
            atomicAdd(&d.acc_hi[slot * d.lo_stride], (unsigned long long)v.hi + carry);
            break;
        }
        case ACC_MIN: case ACC_FIRST: case ACC_FIRST_IGNORES_NULL:
            atomicMin((long long*)&d.acc_lo[slot * d.lo_stride], (long long)v.lo);
            break;
        case ACC_MAX:
            atomicMax((long long*)&d.acc_lo[slot * d.lo_stride], (long long)v.lo);
            break;
        case ACC_MIN_STR: case ACC_MAX_STR:
            if constexpr (STR) {   // install this row unless the installed one is already at least as extreme
                unsigned long long* p = &d.acc_lo[slot * d.lo_stride];
                unsigned long long cur = *(volatile unsigned long long*)p;
                for (;;) {
                    if (cur != ~0ull) {
                        const int c = str_row_cmp((const uint8_t*)d.in, d.in_offsets, (int64_t)v.lo, (int64_t)cur);
                        if (d.kind == ACC_MIN_STR ? c >= 0 : c <= 0) break;
                    }
                    const unsigned long long old = atomicCAS(p, cur, (unsigned long long)v.lo);
                    if (old == cur) break;
                    cur = old;
                }
            }
            break;
    }
    if (d.acc_valid) d.acc_valid[slot * d.valid_stride] = 1;   // idempotent byte store, no atomic needed
}

// -------------------------------------------------------------------------------- FAST path
struct FastKey {
    const void* data;
    const uint8_t* validity;
    int32_t type;
};
__device__ __forceinline__ uint64_t load_key64(const FastKey& k, int64_t row) {
    switch (k.type) {
        case T_INT8: return (uint64_t)(int64_t)((const int8_t*)k.data)[row];
        case T_INT16: return (uint64_t)(int64_t)((const int16_t*)k.data)[row];
        case T_INT32: case T_DATE32: return (uint64_t)(int64_t)((const int32_t*)k.data)[row];
        case T_FLOAT32: return (uint64_t)((const uint32_t*)k.data)[row];
        case T_DECIMAL128: return ((const uint64_t*)k.data)[row * 2];
        default: return ((const uint64_t*)k.data)[row];
    }
}

constexpr int kMaxProbe = 128;

// one input row: key -> table slot (find or insert) -> accumulators
template <bool STR>
__device__ __forceinline__ void agg_fast_row(const FastKey& key, unsigned long long* __restrict__ table, int tw, int64_t cap, uint64_t mask,
                                             const AccArgs& accs, int64_t row, int64_t dense, int32_t* __restrict__ flags) {
    // flags[0] overflow, flags[1] sentinel-key slot used, flags[2] null slot used
    int64_t slot = -1;
    if (key.validity && !bit_get(key.validity, row)) {
        slot = cap + 1;
        flags[2] = 1;
    } else {
        const uint64_t k = load_key64(key, row);
        if (k == EMPTY_KEY) {
            slot = cap;
            flags[1] = 1;
        } else {
            uint64_t hh = mix64(k) & mask;
            unsigned long long c = table[hh * tw];
            for (int p = 0; p < kMaxProbe; p++) {
                if (c == k) { slot = (int64_t)hh; break; }
                if (c == EMPTY_KEY) {
                    unsigned long long old = atomicCAS(&table[hh * tw], (unsigned long long)EMPTY_KEY, (unsigned long long)k);
                    if (old == EMPTY_KEY || old == k) { slot = (int64_t)hh; break; }
                }
                hh = (hh + 1) & mask;
                c = table[hh * tw];
            }
            if (slot < 0) {
                flags[0] = 1;
                return;
            }
        }
    }
    for (int a = 0; a < accs.n; a++) {
        const AccDesc& d = accs.a[a];
        AccVal v = {0, 0};
        if (acc_load(d, row, dense, v)) acc_apply<STR>(d, slot, v);
    }
}
// The per-row chain selection -> key -> table slot -> accumulators is a sequence of dependent, mostly random accesses; the
// kernel is bound by the L2 atomic units and by the number of requests the resident warps keep in flight.  One row per
// thread: more rows in flight per thread cost registers, and so occupancy.
// With a pending filter mask (selmask) every warp first compacts the selected rows of a 128-row window into shared memory
// and then processes them 32 at a time: under the raw mask only the selected lanes would be active, and requests in flight
// scale with the active lanes.
template <bool STR>
__global__ void __launch_bounds__(256) agg_fast_kernel(FastKey key, unsigned long long* __restrict__ table, int tw, int64_t cap, AccArgs accs,
                                                       const int32_t* __restrict__ sel, int64_t n, int32_t* __restrict__ flags,
                                                       const uint32_t* __restrict__ selmask) {
    const uint64_t mask = (uint64_t)cap - 1;
    if (!selmask) {
        const int64_t stride = (int64_t)gridDim.x * 256;
        for (int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x; i < n; i += stride)
            agg_fast_row<STR>(key, table, tw, cap, mask, accs, sel ? (int64_t)sel[i] : i, i, flags);
        return;
    }
    __shared__ int32_t s_rows[8][128];
    const unsigned lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const unsigned lt = (1u << lane) - 1u;
    const int64_t n_words = (n + 31) >> 5;
    const int64_t warp = (int64_t)blockIdx.x * 8 + wid, nwarps = (int64_t)gridDim.x * 8;
    for (int64_t w0 = warp * 4; w0 < n_words; w0 += nwarps * 4) {
        // lanes 0..3 fetch the window's mask words; bits past the last row are cleared here, whatever the producer left there
        uint32_t mw = (lane < 4 && w0 + lane < n_words) ? selmask[w0 + lane] : 0u;
        if (w0 + lane == n_words - 1 && (n & 31)) mw &= (1u << (n & 31)) - 1u;
        int pos = 0;
#pragma unroll
        for (int q = 0; q < 4; q++) {
            const uint32_t wq = __shfl_sync(FULL_MASK, mw, q);
            if ((wq >> lane) & 1u) s_rows[wid][pos + __popc(wq & lt)] = (int32_t)((w0 + q) * 32 + lane);
            pos += __popc(wq);
        }
        __syncwarp();
        for (int j = lane; j < pos; j += 32) {
            const int64_t row = s_rows[wid][j];
            agg_fast_row<STR>(key, table, tw, cap, mask, accs, row, row, flags);
        }
        __syncwarp();
    }
}

// -------------------------------------------------------------------------------- DIRECT path
// One integer key whose value range in the chunk is small (TPC-DS surrogate keys: item_sk in [1, 204000]): the slot is
// key - min, so the per-row table probe (a random 8-byte load, plus CAS on insert) disappears and a row costs only its
// accumulator atomics.  The range comes from a min/max pass over the key column; slot `range` is the NULL group.  A group
// exists if some accumulator shows it (COUNT != 0 or a valid flag) or, for rows that contribute to no such accumulator, the
// `seen` byte written for exactly those rows.
struct DirectTable {
    long long kmin;
    int64_t range;
    uint8_t* seen;
    int32_t* oor;   // set when a key falls outside [kmin, kmin + range): the bounds came from file statistics and were wrong
};
__global__ void __launch_bounds__(256) key_minmax_kernel(FastKey key, int64_t n, long long* __restrict__ out) {
    long long mn = 0x7fffffffffffffffll, mx = (long long)0x8000000000000000ull;
    const int64_t stride = (int64_t)gridDim.x * 256;
    for (int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x; i < n; i += stride) {
        if (key.validity && !bit_get(key.validity, i)) continue;
        long long k = (long long)load_key64(key, i);
        mn = min(mn, k);
        mx = max(mx, k);
    }
    for (int d = 16; d; d >>= 1) {
        mn = min(mn, __shfl_down_sync(FULL_MASK, mn, d));
        mx = max(mx, __shfl_down_sync(FULL_MASK, mx, d));
    }
    if (lane_id() == 0 && mn <= mx) {
        atomicMin(&out[0], mn);
        atomicMax(&out[1], mx);
    }
}
// same reduction for int32 / int64 keys: 4 consecutive rows per lane from 128-bit loads, one validity nibble per lane
template <typename T>
__global__ void __launch_bounds__(256) key_minmax_vec_kernel(const T* __restrict__ data, const uint32_t* __restrict__ valid, int64_t n,
                                                             long long* __restrict__ out) {
    const unsigned lane = threadIdx.x & 31;
    const unsigned sub = (lane & 7) * 4;
    const int64_t warp = ((int64_t)blockIdx.x * 256 + threadIdx.x) >> 5, nwarps = ((int64_t)gridDim.x * 256) >> 5;
    long long mn = 0x7fffffffffffffffll, mx = (long long)0x8000000000000000ull;
    for (int64_t base = warp * 128; base < n; base += nwarps * 128) {
        if (base + 128 <= n) {
            T x[4];
            if (sizeof(T) == 4) {
                const int4 v = ((const int4*)(data + base))[lane];
                x[0] = (T)v.x, x[1] = (T)v.y, x[2] = (T)v.z, x[3] = (T)v.w;
            } else {
                const longlong2* q = (const longlong2*)(data + base) + 2 * lane;
                const longlong2 v0 = q[0], v1 = q[1];
                x[0] = (T)v0.x, x[1] = (T)v0.y, x[2] = (T)v1.x, x[3] = (T)v1.y;
            }
            const uint32_t m = valid ? (valid[(base >> 5) + (lane >> 3)] >> sub) & 0xFu : 0xFu;
#pragma unroll
            for (int k = 0; k < 4; k++)
                if ((m >> k) & 1u) {
                    mn = min(mn, (long long)x[k]);
                    mx = max(mx, (long long)x[k]);
                }
        } else {
            for (int k = 0; k < 4; k++) {
                const int64_t row = base + 4 * lane + k;
                if (row < n && (!valid || ((valid[row >> 5] >> (row & 31)) & 1u))) {
                    mn = min(mn, (long long)data[row]);
                    mx = max(mx, (long long)data[row]);
                }
            }
        }
    }
    for (int d = 16; d; d >>= 1) {
        mn = min(mn, __shfl_down_sync(FULL_MASK, mn, d));
        mx = max(mx, __shfl_down_sync(FULL_MASK, mx, d));
    }
    if (lane == 0 && mn <= mx) {
        atomicMin(&out[0], mn);
        atomicMax(&out[1], mx);
    }
}
template <bool STR>
__device__ __forceinline__ void agg_direct_row(const FastKey& key, const DirectTable& t, const AccArgs& accs, int64_t row, int64_t dense) {
    int64_t slot = t.range;
    if (!key.validity || bit_get(key.validity, row)) {
        slot = (int64_t)((long long)load_key64(key, row) - t.kmin);
        if ((uint64_t)slot >= (uint64_t)t.range) {   // never with bounds computed from the data; the flagged result is discarded
            *t.oor = 1;
            slot = t.range;
        }
    }
    bool marked = false;
    for (int a = 0; a < accs.n; a++) {
        const AccDesc& d = accs.a[a];
        AccVal v = {0, 0};
        if (acc_load(d, row, dense, v)) {
            acc_apply<STR>(d, slot, v);
            marked = marked || (((d.kind == ACC_COUNT || d.kind == ACC_ADD_I64) && v.lo != 0) || d.acc_valid != nullptr);
        }
    }
    if (!marked) t.seen[slot] = 1;
}
template <bool STR>
__global__ void __launch_bounds__(256) agg_direct_kernel(FastKey key, DirectTable t, AccArgs accs, const int32_t* __restrict__ sel, int64_t n,
                                                         const uint32_t* __restrict__ selmask) {
    if (!selmask) {
        const int64_t stride = (int64_t)gridDim.x * 256;
        for (int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x; i < n; i += stride) agg_direct_row<STR>(key, t, accs, sel ? (int64_t)sel[i] : i, i);
        return;
    }
    // pending filter mask: warp-local compaction of each 128-row window (see agg_fast_kernel)
    __shared__ int32_t s_rows[8][128];
    const unsigned lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const unsigned lt = (1u << lane) - 1u;
    const int64_t n_words = (n + 31) >> 5;
    const int64_t warp = (int64_t)blockIdx.x * 8 + wid, nwarps = (int64_t)gridDim.x * 8;
    for (int64_t w0 = warp * 4; w0 < n_words; w0 += nwarps * 4) {
        uint32_t mw = (lane < 4 && w0 + lane < n_words) ? selmask[w0 + lane] : 0u;
        if (w0 + lane == n_words - 1 && (n & 31)) mw &= (1u << (n & 31)) - 1u;
        int pos = 0;
#pragma unroll
        for (int q = 0; q < 4; q++) {
            const uint32_t wq = __shfl_sync(FULL_MASK, mw, q);
            if ((wq >> lane) & 1u) s_rows[wid][pos + __popc(wq & lt)] = (int32_t)((w0 + q) * 32 + lane);
            pos += __popc(wq);
        }
        __syncwarp();
        for (int j = lane; j < pos; j += 32) {
            const int64_t row = s_rows[wid][j];
            agg_direct_row<STR>(key, t, accs, row, row);
        }
        __syncwarp();
    }
}
__global__ void __launch_bounds__(256) occupied_mask_direct_kernel(DirectTable t, AccArgs accs, uint32_t* __restrict__ mask) {
    const int64_t s = (int64_t)blockIdx.x * 256 + threadIdx.x;
    bool occ = false;
    if (s <= t.range) {
        occ = t.seen[s] != 0;
        for (int a = 0; a < accs.n && !occ; a++) {
            const AccDesc& d = accs.a[a];
            if (d.kind == ACC_COUNT || d.kind == ACC_ADD_I64) occ = d.acc_lo[s] != 0;
            else if (d.acc_valid) occ = d.acc_valid[s] != 0;
        }
    }
    uint32_t w = __ballot_sync(FULL_MASK, occ);
    if (lane_id() == 0 && s <= t.range) mask[s >> 5] = w;
}
__global__ void __launch_bounds__(256) emit_direct_keys_kernel(DirectTable t, const int32_t* __restrict__ slot_ids, int64_t g, int32_t type,
                                                               void* __restrict__ out, uint32_t* __restrict__ out_valid) {
    int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x;
    bool valid = false;
    if (i < g) {
        const int64_t s = slot_ids[i];
        valid = s < t.range;
        const long long k = valid ? t.kmin + s : 0;
        switch (type) {
            case T_INT8: ((int8_t*)out)[i] = (int8_t)k; break;
            case T_INT16: ((int16_t*)out)[i] = (int16_t)k; break;
            case T_INT32: case T_DATE32: ((int32_t*)out)[i] = (int32_t)k; break;
            default: ((long long*)out)[i] = k; break;
        }
    }
    if (out_valid) {
        uint32_t w = __ballot_sync(FULL_MASK, valid);
        if (lane_id() == 0 && i < g) out_valid[i >> 5] = w;
    }
}

// -------------------------------------------------------------------------------- FAST path, low cardinality
// With a few hundred groups every row of the plain kernel hits the same handful of L2 atomics.  This variant keeps a
// per-CTA hash table + accumulators in shared memory (2048 slots), aggregates the CTA's rows there with shared-memory
// atomics and merges each occupied slot into the global table once at the end.  Rows that do not fit (table full after
// a few probes), NULL keys and the sentinel key take the global path directly, so the result is exact for any input;
// the host picks this variant when a sample of the chunk shows <= 1024 distinct keys.
constexpr int SM_SLOTS = 2048, SM_PROBE = 16, SM_MAX_ACCS = 4;
__device__ __forceinline__ int64_t global_slot_fast(unsigned long long* table, int tw, uint64_t mask, uint64_t k, int32_t* flags) {
    uint64_t h = mix64(k) & mask;
    for (int p = 0; p < kMaxProbe; p++) {
        unsigned long long cur = table[h * tw];
        if (cur == k) return (int64_t)h;
        if (cur == EMPTY_KEY) {
            unsigned long long old = atomicCAS(&table[h * tw], (unsigned long long)EMPTY_KEY, (unsigned long long)k);
            if (old == EMPTY_KEY || old == k) return (int64_t)h;
        }
        h = (h + 1) & mask;
    }
    flags[0] = 1;
    return -1;
}
__global__ void __launch_bounds__(256) agg_fast_smem_kernel(FastKey key, unsigned long long* __restrict__ table, int tw, int64_t cap, AccArgs accs,
                                                            const int32_t* __restrict__ sel, int64_t n, int32_t* __restrict__ flags, const uint32_t* __restrict__ selmask) {
    extern __shared__ __align__(16) unsigned long long sm[];
    unsigned long long* s_keys = sm;                                   // [SM_SLOTS]
    unsigned long long* s_acc = sm + SM_SLOTS;                         // [n_accs][SM_SLOTS]
    uint8_t* s_valid = (uint8_t*)(s_acc + (size_t)accs.n * SM_SLOTS);  // [n_accs][SM_SLOTS]
    for (int i = threadIdx.x; i < SM_SLOTS; i += 256) s_keys[i] = EMPTY_KEY;
    for (int a = 0; a < accs.n; a++) {
        unsigned long long init = 0;
        int kd = accs.a[a].kind;
        if (kd == ACC_MIN) init = 0x7fffffffffffffffull;
        else if (kd == ACC_MAX) init = 0x8000000000000000ull;
        for (int i = threadIdx.x; i < SM_SLOTS; i += 256) {
            s_acc[(size_t)a * SM_SLOTS + i] = init;
            s_valid[(size_t)a * SM_SLOTS + i] = 0;
        }
    }
    __syncthreads();
    const uint64_t gmask = (uint64_t)cap - 1;
    // contiguous slab of rows per CTA
    const int64_t per = (n + gridDim.x - 1) / gridDim.x;
    const int64_t lo = (int64_t)blockIdx.x * per, hi = min(n, lo + per);
    for (int64_t i = lo + threadIdx.x; i < hi; i += 256) {
        if (selmask && !((selmask[i >> 5] >> (i & 31)) & 1u)) continue;   // pending filter mask: row not selected
        int64_t row = sel ? (int64_t)sel[i] : i;
        bool knull = key.validity && !bit_get(key.validity, row);
        uint64_t k = knull ? 0 : load_key64(key, row);
        int sslot = -1;
        if (!knull && k != EMPTY_KEY) {
            uint32_t h = (uint32_t)mix64(k) & (SM_SLOTS - 1);
            for (int p = 0; p < SM_PROBE; p++) {
                unsigned long long cur = s_keys[h];
                if (cur == k) { sslot = (int)h; break; }
                if (cur == EMPTY_KEY) {
                    unsigned long long old = atomicCAS(&s_keys[h], (unsigned long long)EMPTY_KEY, (unsigned long long)k);
                    if (old == EMPTY_KEY || old == k) { sslot = (int)h; break; }
                }
                h = (h + 1) & (SM_SLOTS - 1);
            }
        }
        if (sslot >= 0) {
            for (int a = 0; a < accs.n; a++) {
                AccDesc d = accs.a[a];
                AccVal v;
                if (!acc_load(d, row, i, v)) continue;
                d.acc_lo = s_acc + (size_t)a * SM_SLOTS;
                d.acc_valid = d.acc_valid ? s_valid + (size_t)a * SM_SLOTS : nullptr;
                d.lo_stride = 1;
                d.valid_stride = 1;
                acc_apply(d, sslot, v);
            }
        } else {   // global path: NULL / sentinel key, or the shared table is full
            int64_t slot;
            if (knull) { slot = cap + 1; flags[2] = 1; }
            else if (k == EMPTY_KEY) { slot = cap; flags[1] = 1; }
            else slot = global_slot_fast(table, tw, gmask, k, flags);
            if (slot < 0) continue;
            for (int a = 0; a < accs.n; a++) {
                AccVal v;
                if (acc_load(accs.a[a], row, i, v)) acc_apply(accs.a[a], slot, v);
            }
        }
    }
    __syncthreads();
    // merge the CTA's groups into the global table
    for (int s = threadIdx.x; s < SM_SLOTS; s += 256) {
        unsigned long long k = s_keys[s];
        if (k == EMPTY_KEY) continue;
        int64_t slot = global_slot_fast(table, tw, gmask, k, flags);
        if (slot < 0) continue;
        for (int a = 0; a < accs.n; a++) {
            const AccDesc& d = accs.a[a];
            if (d.acc_valid && !s_valid[(size_t)a * SM_SLOTS + s]) continue;
            AccVal v{s_acc[(size_t)a * SM_SLOTS + s], 0};
            AccDesc m = d;
            if (m.kind == ACC_COUNT) m.kind = ACC_ADD_I64;   // partial counts add up
            acc_apply(m, slot, v);
        }
    }
}

// -------------------------------------------------------------------------------- GENERAL path
template <bool STR>
__global__ void __launch_bounds__(256) agg_general_kernel(RowKeys keys, int32_t* __restrict__ slots, int64_t cap, AccArgs accs,
                                                          const int32_t* __restrict__ sel, int64_t n, int32_t* __restrict__ flags, const uint32_t* __restrict__ selmask) {
    int64_t stride = (int64_t)gridDim.x * 256;
    uint64_t mask = (uint64_t)cap - 1;
    for (int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x; i < n; i += stride) {
        if (selmask && !((selmask[i >> 5] >> (i & 31)) & 1u)) continue;   // pending filter mask: row not selected
        int64_t row = sel ? (int64_t)sel[i] : i;
        uint64_t h = rowkey_hash(keys, row) & mask;
        int64_t slot = -1;
        for (int p = 0; p < kMaxProbe; p++) {
            int32_t cur = slots[h];
            if (cur < 0) {
                int32_t old = atomicCAS(&slots[h], -1, (int32_t)row);
                if (old < 0) { slot = (int64_t)h; break; }
                cur = old;
            }
            if (cur == (int32_t)row || rowkey_equal(keys, cur, keys, row)) { slot = (int64_t)h; break; }
            h = (h + 1) & mask;
        }
        if (slot < 0) {
            flags[0] = 1;
            continue;
        }
        for (int a = 0; a < accs.n; a++) {
            AccVal v;
            if (acc_load(accs.a[a], row, i, v)) acc_apply<STR>(accs.a[a], slot, v);
        }
    }
}

// -------------------------------------------------------------------------------- no-key path
__device__ __forceinline__ void acc_combine(int kind, AccVal& a, bool& av, const AccVal& b, bool bv) {
    if (!bv) return;
    if (!av) { a = b; av = true; return; }
    switch (kind) {
        case ACC_SUM_I64: case ACC_ADD_I64: case ACC_COUNT: a.lo += b.lo; break;
        case ACC_SUM_F64: a.lo = (uint64_t)__double_as_longlong(__longlong_as_double((int64_t)a.lo) + __longlong_as_double((int64_t)b.lo)); break;
        case ACC_SUM_DEC: {
            i128 r = i128_add({a.lo, a.hi}, {b.lo, b.hi});
            a.lo = r.lo; a.hi = r.hi;
            break;
        }
        case ACC_MIN: case ACC_FIRST: case ACC_FIRST_IGNORES_NULL: if ((int64_t)b.lo < (int64_t)a.lo) a.lo = b.lo; break;
        case ACC_MAX: if ((int64_t)b.lo > (int64_t)a.lo) a.lo = b.lo; break;
    }
}
template <bool STR>
__global__ void __launch_bounds__(256) agg_global_kernel(AccArgs accs, const int32_t* __restrict__ sel, int64_t n, const uint32_t* __restrict__ selmask) {
    int64_t stride = (int64_t)gridDim.x * 256;
    for (int a = 0; a < accs.n; a++) {
        const AccDesc& d = accs.a[a];
        AccVal acc = {0, 0};
        bool av = false;
        for (int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x; i < n; i += stride) {
            if (selmask && !((selmask[i >> 5] >> (i & 31)) & 1u)) continue;   // pending filter mask: row not selected
            int64_t row = sel ? (int64_t)sel[i] : i;
            AccVal v = {0, 0};
            bool ok = acc_load(d, row, i, v);
            if (d.kind == ACC_MIN_STR || d.kind == ACC_MAX_STR) {   // rows are compared through the column: straight to the slot
                if (ok) acc_apply<STR>(d, 0, v);
                continue;
            }
            acc_combine(d.kind, acc, av, v, ok);
        }
        for (int off = 16; off; off >>= 1) {
            AccVal o;
            o.lo = __shfl_down_sync(FULL_MASK, acc.lo, off);
            o.hi = __shfl_down_sync(FULL_MASK, acc.hi, off);
            bool ov = __shfl_down_sync(FULL_MASK, (int)av, off);
            acc_combine(d.kind, acc, av, o, ov);
        }
        if (lane_id() == 0 && av) acc_apply<STR>(d, 0, acc);
    }
}

// -------------------------------------------------------------------------------- emit
__global__ void occupied_mask_fast_kernel(const unsigned long long* __restrict__ table, int tw, int64_t cap, const int32_t* __restrict__ flags,
                                          uint32_t* __restrict__ mask) {
    int64_t s = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    bool occ = false;
    if (s < cap) occ = table[s * tw] != EMPTY_KEY;
    else if (s == cap) occ = flags[1] != 0;
    else if (s == cap + 1) occ = flags[2] != 0;
    uint32_t w = __ballot_sync(FULL_MASK, occ);
    if (lane_id() == 0 && s < cap + 2) mask[s >> 5] = w;
}
__global__ void occupied_mask_general_kernel(const int32_t* __restrict__ slots, int64_t cap, uint32_t* __restrict__ mask) {
    int64_t s = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    bool occ = s < cap && slots[s] >= 0;
    uint32_t w = __ballot_sync(FULL_MASK, occ);
    if (lane_id() == 0 && s < cap) mask[s >> 5] = w;
}
__global__ void gather_i32_kernel(const int32_t* __restrict__ in, const int32_t* __restrict__ idx, int64_t n, int32_t* __restrict__ out) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = in[idx[i]];
}
__global__ void __launch_bounds__(256) emit_fast_keys_kernel(const unsigned long long* __restrict__ table, int tw, int64_t cap,
                                                             const int32_t* __restrict__ slot_ids, int64_t g, int32_t type, void* __restrict__ out,
                                                             uint32_t* __restrict__ out_valid) {
    int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x;
    bool ok = false;
    if (i < g) {
        int64_t s = slot_ids[i];
        uint64_t k = s < cap ? table[s * tw] : (s == cap ? EMPTY_KEY : 0ull);
        ok = s != cap + 1;
        switch (type) {
            case T_INT8: ((int8_t*)out)[i] = (int8_t)k; break;
            case T_INT16: ((int16_t*)out)[i] = (int16_t)k; break;
            case T_INT32: case T_DATE32: case T_FLOAT32: ((uint32_t*)out)[i] = (uint32_t)k; break;
            case T_DECIMAL128: ((uint64_t*)out)[2 * i] = k; ((int64_t*)out)[2 * i + 1] = ((int64_t)k) < 0 ? -1ll : 0ll; break;
            default: ((uint64_t*)out)[i] = k; break;
        }
    }
    if (out_valid) {
        uint32_t w = __ballot_sync(FULL_MASK, ok);
        if (lane_id() == 0 && i < g) out_valid[i >> 5] = w;
    }
}
// accumulator array -> typed output column.  slot_ids == nullptr: identity (no-key path, one row)
__global__ void __launch_bounds__(256) emit_acc_kernel(AccDesc d, const int32_t* __restrict__ slot_ids, int64_t g, int32_t out_type,
                                                       void* __restrict__ out, uint32_t* __restrict__ out_valid) {
    int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x;
    bool ok = false;
    if (i < g) {
        int64_t s = slot_ids ? (int64_t)slot_ids[i] : i;
        ok = d.valid_cnt ? d.valid_cnt[s] != 0 : (d.acc_valid ? d.acc_valid[s * d.valid_stride] != 0 : true);
        uint64_t lo = d.acc_lo[s * d.lo_stride];
        switch (d.kind) {
            case ACC_SUM_DEC:
                ((uint64_t*)out)[2 * i] = ok ? lo : 0;
                ((uint64_t*)out)[2 * i + 1] = ok ? d.acc_hi[s * d.lo_stride] : 0;
                break;
            case ACC_SUM_F64:
                if (out_type == T_FLOAT32) ((float*)out)[i] = ok ? (float)__longlong_as_double((int64_t)lo) : 0.f;
                else ((uint64_t*)out)[i] = ok ? lo : 0;
                break;
            case ACC_MIN: case ACC_MAX: {
                if (!ok) lo = 0;
                switch (out_type) {
                    case T_BOOL: break;  // handled by the bool variant below (never reached)
                    case T_INT8: ((int8_t*)out)[i] = (int8_t)lo; break;
                    case T_INT16: ((int16_t*)out)[i] = (int16_t)lo; break;
                    case T_INT32: case T_DATE32: ((int32_t*)out)[i] = (int32_t)lo; break;
                    case T_FLOAT32: ((float*)out)[i] = ok ? (float)ordered_to_f64((int64_t)lo) : 0.f; break;
                    case T_FLOAT64: ((double*)out)[i] = ok ? ordered_to_f64((int64_t)lo) : 0.0; break;
                    case T_DECIMAL128: ((uint64_t*)out)[2 * i] = lo; ((int64_t*)out)[2 * i + 1] = ((int64_t)lo) < 0 ? -1ll : 0ll; break;
                    default: ((uint64_t*)out)[i] = lo; break;
                }
                break;
            }
            case ACC_FIRST: case ACC_FIRST_IGNORES_NULL:
                ((int32_t*)out)[i] = ok ? (int32_t)lo : -1;   // position; gathered by the host wrapper
                break;
            case ACC_MIN_STR: case ACC_MAX_STR:
                ((int32_t*)out)[i] = (int32_t)(int64_t)lo;    // row of the extreme (-1 = none); gathered by the host wrapper
                break;
            default:
                ((uint64_t*)out)[i] = lo;
        }
    }
    if (out_valid) {
        uint32_t w = __ballot_sync(FULL_MASK, ok);
        if (lane_id() == 0 && i < g) out_valid[i >> 5] = w;
    }
}
__global__ void sel_compose_kernel(const int32_t* __restrict__ pos, const int32_t* __restrict__ sel, int64_t n, int32_t* __restrict__ out) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = pos[i] < 0 ? -1 : (sel ? sel[pos[i]] : pos[i]);
}
__global__ void nonneg_mask_kernel(const int32_t* __restrict__ pos, int64_t n, uint32_t* __restrict__ bits) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    bool ok = i < n && pos[i] >= 0;
    uint32_t w = __ballot_sync(FULL_MASK, ok);
    if (lane_id() == 0 && i < n) bits[i >> 5] = w;
}

// -------------------------------------------------------------------------------- host side
static int64_t next_pow2(int64_t v) {
    int64_t p = 1;
    while (p < v) p <<= 1;
    return p;
}
static bool fast_key_ok(const std::vector<ColumnPtr>& keys) {
    if (keys.size() != 1) return false;
    const DType& t = keys[0]->type;
    if (t.id == T_DECIMAL128) return t.precision <= 18;
    return t.width() >= 1 && t.width() <= 8;
}

struct AccBuffers {
    std::vector<Buf> lo, hi, valid;
};
// slot-record layout of the FAST path: [key | acc words ... | flags word] padded to a power of two u64 words, so the key, every
// accumulator and the valid flags of a group share one or two 32-byte sectors (one L2 access pattern per row instead of 1 + n_accs)
struct RecLayout {
    int tw = 1;                 // u64 words per slot record (1 = no interleaving: separate SoA arrays)
    int lo_word[kMaxAccs];
    int hi_word[kMaxAccs];
    unsigned long long init[16];
};
static RecLayout make_layout(const std::vector<AccSpec>& specs) {
    RecLayout L;
    if (specs.size() > 8) return L;
    int w = 1;
    for (size_t i = 0; i < specs.size(); i++) {
        L.lo_word[i] = w++;
        L.hi_word[i] = specs[i].kind == ACC_SUM_DEC ? w++ : 0;
    }
    w++;   // flags word (one valid byte per accumulator)
    int tw = 1;
    while (tw < w) tw <<= 1;
    if (tw > 16) return L;
    L.tw = tw;
    for (int i = 0; i < 16; i++) L.init[i] = 0;
    L.init[0] = 0x8A5C3F1E9D7B2461ull;   // EMPTY_KEY
    for (size_t i = 0; i < specs.size(); i++) {
        AccKind k = specs[i].kind;
        if (k == ACC_MIN || k == ACC_FIRST || k == ACC_FIRST_IGNORES_NULL) L.init[L.lo_word[i]] = 0x7fffffffffffffffull;
        else if (k == ACC_MAX) L.init[L.lo_word[i]] = 0x8000000000000000ull;
    }
    return L;
}
struct RecInit {
    unsigned long long w[16];
};
__global__ void init_records_kernel(unsigned long long* __restrict__ rec, int64_t n_words, int tw, RecInit init) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n_words) rec[i] = init.w[i & (tw - 1)];
}
static AccArgs prepare_accs(Ctx& ctx, const std::vector<AccSpec>& specs, int64_t slots, AccBuffers& bufs, unsigned long long* rec_base = nullptr,
                            const RecLayout* layout = nullptr) {
    AURON_CHECK((int)specs.size() <= kMaxAccs, "too many aggregate accumulators in one AggExec");
    AccArgs args;
    args.n = (int)specs.size();
    for (int i = 0; i < args.n; i++) {
        const AccSpec& s = specs[i];
        AccDesc& d = args.a[i];
        memset(&d, 0, sizeof(d));
        d.kind = s.kind;
        if (s.input) {
            d.in = s.input->data ? s.input->data->ptr : nullptr;
            d.in_valid = s.input->vbits();
            d.in_type = s.input->type.id;
            d.in_is_dec64 = s.input->type.id == T_DECIMAL128 && s.input->type.precision <= 18;
            d.in_offsets = P<int32_t>(s.input->offsets);
        } else {
            d.in_type = T_NULL;
        }
        AURON_CHECK(s.extra.size() <= 3, "COUNT with more than 4 arguments");
        d.n_extra = 0;
        if (s.kind == ACC_COUNT)
            for (auto& e : s.extra) d.extra_valid[d.n_extra++] = e->vbits();
        if (s.kind == ACC_FIRST && !s.extra.empty()) {
            AURON_CHECK(s.extra[0]->type.id == T_BOOL, "FIRST merge needs the is_set boolean column");
            d.extra_valid[d.n_extra++] = P<uint8_t>(s.extra[0]->data);
        }
        if ((s.kind == ACC_MIN || s.kind == ACC_MAX) && s.input) {
            const DType& t = s.input->type;
            bool ok = t.is_intlike() || t.is_float() || t.id == T_BOOL || (t.id == T_DECIMAL128 && t.precision <= 18);
            AURON_CHECK(ok, "MIN/MAX over " + t.str() + " is not supported on device yet");
        }
        d.lo_stride = 1;
        d.valid_stride = 1;
        if (rec_base) {   // interleaved slot records
            d.lo_stride = layout->tw;
            d.valid_stride = layout->tw * 8;
            d.acc_lo = rec_base + layout->lo_word[i];
            d.acc_hi = s.kind == ACC_SUM_DEC ? rec_base + layout->hi_word[i] : nullptr;
            d.acc_valid = (s.kind == ACC_COUNT || s.kind == ACC_ADD_I64) ? nullptr : (uint8_t*)(rec_base + layout->tw - 1) + i;
            bufs.lo.push_back(nullptr);
            bufs.hi.push_back(nullptr);
            bufs.valid.push_back(nullptr);
            continue;
        }
        Buf lo;
        lo = dalloc(ctx, (size_t)slots * 8);
        bufs.lo.push_back(lo);
        d.acc_lo = P<unsigned long long>(lo);
        if (s.kind == ACC_SUM_DEC) {
            Buf hi = dalloc_zero(ctx, (size_t)slots * 8);
            bufs.hi.push_back(hi);
            d.acc_hi = P<unsigned long long>(hi);
        } else bufs.hi.push_back(nullptr);
        if (s.kind == ACC_COUNT || s.kind == ACC_ADD_I64 || s.kind == ACC_MIN_STR || s.kind == ACC_MAX_STR) {
            bufs.valid.push_back(nullptr);   // (string extremes: "no row yet" is the accumulator value -1)
        } else {
            Buf v = dalloc_zero(ctx, (size_t)slots);
            bufs.valid.push_back(v);
            d.acc_valid = P<uint8_t>(v);
        }
    }
    // pair SUM / MIN / MAX (x) with a COUNT(x) over the very same column (AVG lowers to exactly this pair)
    if (!rec_base && !getenv("AURON_DISABLE_AGG_VALID_FROM_COUNT") && !getenv("AURON_ENABLE_SMEM_AGG"))
        for (int i = 0; i < args.n; i++) {
            const AccSpec& s = specs[i];
            bool value_acc = s.kind == ACC_SUM_I64 || s.kind == ACC_SUM_F64 || s.kind == ACC_SUM_DEC || s.kind == ACC_MIN || s.kind == ACC_MAX;
            if (!value_acc || (!s.input && s.input_id < 0)) continue;
            for (int j = 0; j < args.n; j++)
                if (specs[j].kind == ACC_COUNT && specs[j].extra.empty() &&
                    (s.input ? (specs[j].input && specs[j].input.get() == s.input.get()) : (!specs[j].input && specs[j].input_id == s.input_id))) {
                    args.a[i].valid_cnt = args.a[j].acc_lo;
                    args.a[i].acc_valid = nullptr;   // the buffer stays allocated (zeroed) but is neither written nor read
                    break;
                }
        }
    return args;
}
__global__ void fill_u64_kernel(unsigned long long* p, int64_t n, unsigned long long v) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) p[i] = v;
}
static void fill_u64(Ctx& ctx, void* p, int64_t n, unsigned long long v) {
    if (n <= 0) return;
    fill_u64_kernel<<<(unsigned)((n + 255) / 256), 256, 0, ctx.stream>>>((unsigned long long*)p, n, v);
    LAUNCH_CHECK(ctx);
}
static void init_accs(Ctx& ctx, const std::vector<AccSpec>& specs, AccArgs& args, int64_t slots) {
    for (int i = 0; i < args.n; i++) {
        unsigned long long init = 0;
        switch (specs[i].kind) {
            case ACC_MIN: case ACC_FIRST: case ACC_FIRST_IGNORES_NULL: init = 0x7fffffffffffffffull; break;
            case ACC_MAX: init = 0x8000000000000000ull; break;
            case ACC_MIN_STR: case ACC_MAX_STR: init = ~0ull; break;
            default: init = 0;
        }
        if (init == 0) CUDA_OK(cudaMemsetAsync(args.a[i].acc_lo, 0, (size_t)slots * 8, ctx.stream));
        else fill_u64(ctx, args.a[i].acc_lo, slots, init);
    }
}

static unsigned agg_grid(Ctx& ctx, int64_t n) {
    int64_t blocks = (n + 255) / 256;
    return (unsigned)std::max<int64_t>(1, std::min<int64_t>(blocks, (int64_t)ctx.sm_count * 8));
}

// accumulator arrays -> output columns (FIRST yields value column + is_set bool column)
static void emit_accs(Ctx& ctx, const std::vector<AccSpec>& specs, const AccArgs& args, const int32_t* slot_ids, int64_t g,
                      const int32_t* sel, std::vector<ColumnPtr>& out) {
    unsigned blocks = (unsigned)((g + 255) / 256);
    for (int i = 0; i < args.n; i++) {
        const AccSpec& s = specs[i];
        const AccDesc& d = args.a[i];
        if (s.kind == ACC_FIRST || s.kind == ACC_FIRST_IGNORES_NULL) {
            Buf pos = dalloc(ctx, (size_t)std::max<int64_t>(g, 1) * 4);
            Buf rows = dalloc(ctx, (size_t)std::max<int64_t>(g, 1) * 4);
            auto isset = make_column(ctx, DType(T_BOOL), g, false);
            if (g) {
                emit_acc_kernel<<<blocks, 256, 0, ctx.stream>>>(d, slot_ids, g, T_INT32, pos->ptr, nullptr);
                LAUNCH_CHECK(ctx);
                sel_compose_kernel<<<blocks, 256, 0, ctx.stream>>>(P<int32_t>(pos), sel, g, P<int32_t>(rows));
                LAUNCH_CHECK(ctx);
                nonneg_mask_kernel<<<blocks, 256, 0, ctx.stream>>>(P<int32_t>(pos), g, P<uint32_t>(isset->data));
                LAUNCH_CHECK(ctx);
            }
            out.push_back(take(ctx, s.gather_from ? *s.gather_from : *s.input, P<int32_t>(rows), g, true));
            if (s.kind == ACC_FIRST) out.push_back(isset);
            continue;
        }
        if (s.kind == ACC_MIN_STR || s.kind == ACC_MAX_STR) {
            Buf rows = dalloc(ctx, (size_t)std::max<int64_t>(g, 1) * 4);
            if (g) {
                emit_acc_kernel<<<blocks, 256, 0, ctx.stream>>>(d, slot_ids, g, T_INT32, rows->ptr, nullptr);
                LAUNCH_CHECK(ctx);
            }
            out.push_back(take(ctx, *s.input, P<int32_t>(rows), g, true));
            continue;
        }
        bool nullable = d.acc_valid != nullptr || d.valid_cnt != nullptr;
        if (s.out_type.id == T_BOOL) {   // MIN/MAX over bool: emit as int8 then it is tiny; convert through take of a 2-entry table
            fail("MIN/MAX(bool) output not supported yet");
        }
        auto col = make_column(ctx, s.out_type, g, nullable);
        if (g) {
            emit_acc_kernel<<<blocks, 256, 0, ctx.stream>>>(d, slot_ids, g, s.out_type.id, col->data->ptr, P<uint32_t>(col->validity));
            LAUNCH_CHECK(ctx);
        }
        out.push_back(col);
    }
}


// -------------------------------------------------------------------------------- persistent DIRECT table
// The direct-address table as an object: created for a key range, updated by any number of kernel launches (the chunk
// aggregate below, or the fused Parquet scan -> filter -> aggregate kernels of k_fused.cu, batch after batch), widened when a
// later batch brings keys outside the range, and turned into [keys | accumulators] columns at the end.
struct DirectAgg {
    std::vector<AccSpec> specs;
    AccBuffers bufs;
    AccArgs args;
    DirectTable dt;
    Buf seen, oor;
    int64_t slots = 0;
};
static void direct_agg_alloc(Ctx& ctx, DirectAgg& da, long long kmin, long long kmax) {
    const bool any = kmin <= kmax;
    da.dt.kmin = any ? kmin : 0;
    da.dt.range = any ? (int64_t)((unsigned long long)kmax - (unsigned long long)kmin) + 1 : 0;
    da.slots = da.dt.range + 1;   // + the NULL group
    da.bufs = AccBuffers();
    da.args = prepare_accs(ctx, da.specs, da.slots, da.bufs);
    init_accs(ctx, da.specs, da.args, da.slots);
    da.seen = dalloc_zero(ctx, (size_t)da.slots + 8);
    da.dt.seen = P<uint8_t>(da.seen);
    if (!da.oor) da.oor = dalloc_zero(ctx, 4);
    da.dt.oor = P<int32_t>(da.oor);
}
std::shared_ptr<DirectAgg> direct_agg_create(Ctx& ctx, const std::vector<AccSpec>& specs, long long kmin, long long kmax) {
    auto da = std::make_shared<DirectAgg>();
    da->specs = specs;
    direct_agg_alloc(ctx, *da, kmin, kmax);
    return da;
}
bool direct_agg_out_of_range(Ctx& ctx, const DirectAgg& da) {
    int32_t bad = 0;
    to_host(ctx, &bad, da.oor->ptr, 4);
    return bad != 0;
}
DirectAggView direct_agg_view(const DirectAgg& da) {
    DirectAggView v;
    memset(&v, 0, sizeof(v));
    v.n = da.args.n;
    for (int i = 0; i < da.args.n; i++) {
        v.kind[i] = da.args.a[i].kind;
        v.acc[i] = da.args.a[i].acc_lo;
        v.valid[i] = da.args.a[i].acc_valid;
    }
    v.seen = da.dt.seen;
    v.oor = da.dt.oor;
    v.kmin = da.dt.kmin;
    v.range = da.dt.range;
    return v;
}
__global__ void __launch_bounds__(256) direct_rebase_kernel(const unsigned long long* __restrict__ src, unsigned long long* __restrict__ dst,
                                                            const uint8_t* __restrict__ srcb, uint8_t* __restrict__ dstb, int64_t old_range, int64_t shift,
                                                            int64_t new_range) {
    const int64_t s = (int64_t)blockIdx.x * 256 + threadIdx.x;
    if (s > old_range) return;
    const int64_t d = s == old_range ? new_range : s + shift;
    if (src) dst[d] = src[s];
    if (srcb) dstb[d] = srcb[s];
}
void direct_agg_grow(Ctx& ctx, DirectAgg& da, long long kmin, long long kmax) {
    if (da.dt.range > 0) {
        kmin = std::min(kmin, da.dt.kmin);
        kmax = std::max(kmax, (long long)(da.dt.kmin + da.dt.range - 1));
    }
    if (da.dt.range > 0 && kmin == da.dt.kmin && kmax == da.dt.kmin + da.dt.range - 1) return;
    DirectAgg old = da;   // keeps the old buffers alive until the copies below are queued (stream-ordered frees)
    direct_agg_alloc(ctx, da, kmin, kmax);
    const int64_t shift = old.dt.range > 0 ? (int64_t)(old.dt.kmin - da.dt.kmin) : 0;
    const unsigned grid = (unsigned)((old.slots + 255) / 256);
    for (int i = 0; i < da.args.n; i++) {
        direct_rebase_kernel<<<grid, 256, 0, ctx.stream>>>(old.args.a[i].acc_lo, da.args.a[i].acc_lo, old.args.a[i].acc_valid, da.args.a[i].acc_valid, old.dt.range, shift,
                                                           da.dt.range);
        LAUNCH_CHECK(ctx);
        AURON_CHECK(!old.args.a[i].acc_hi, "direct_agg_grow: wide accumulators are not rebased");
    }
    direct_rebase_kernel<<<grid, 256, 0, ctx.stream>>>(nullptr, nullptr, old.dt.seen, da.dt.seen, old.dt.range, shift, da.dt.range);
    LAUNCH_CHECK(ctx);
}
int64_t direct_agg_span_limit() { return (int64_t)1 << 22; }
GroupedResult direct_agg_finish(Ctx& ctx, DirectAgg& da, const DType& key_type, bool key_nullable, const int32_t* sel) {
    GroupedResult res;
    const int64_t slots = da.slots;
    Buf occ = dalloc(ctx, bitmap_alloc_bytes(slots));
    occupied_mask_direct_kernel<<<(unsigned)((slots + 255) / 256), 256, 0, ctx.stream>>>(da.dt, da.args, P<uint32_t>(occ));
    LAUNCH_CHECK(ctx);
    int64_t g = 0;
    Buf slot_ids = mask_to_indices(ctx, P<uint32_t>(occ), slots, &g);
    res.num_groups = g;
    res.keys = std::make_shared<Batch>();
    res.keys->num_rows = g;
    auto kc = make_column(ctx, key_type, g, key_nullable);
    if (g) {
        emit_direct_keys_kernel<<<(unsigned)((g + 255) / 256), 256, 0, ctx.stream>>>(da.dt, P<int32_t>(slot_ids), g, key_type.id, kc->data->ptr, P<uint32_t>(kc->validity));
        LAUNCH_CHECK(ctx);
    }
    res.keys->cols.push_back(kc);
    emit_accs(ctx, da.specs, da.args, P<int32_t>(slot_ids), g, sel, res.accs);
    return res;
}

GroupedResult hash_aggregate(Ctx& ctx, const std::vector<ColumnPtr>& keys, const std::vector<AccSpec>& accs, const int32_t* sel,
                             int64_t n_rows, const DType* fast_key_out, const uint32_t* selmask, int64_t n_selected) {
    // selmask != nullptr: a filter's pending bit mask over the batch rows (n_rows = batch rows, n_selected = set bits); the
    // kernels then skip unselected rows themselves and no index vector is ever materialised.  Mutually exclusive with sel.
    AURON_CHECK(!(sel && selmask), "hash_aggregate: both an index selection and a mask selection");
    const int64_t n_in = selmask && n_selected >= 0 ? n_selected : n_rows;   // rows that reach the table
    bool has_str = false;   // string extremes need the kernel instances that carry their CAS loop
    for (auto& sp : accs) has_str = has_str || sp.kind == ACC_MIN_STR || sp.kind == ACC_MAX_STR;
    AURON_CHECK(!keys.empty(), "hash_aggregate needs at least one key (use global_aggregate)");
    AURON_CHECK(n_rows < (int64_t)INT32_MAX, "chunk too large");
    GroupedResult res;
    bool fast = fast_key_ok(keys);
    // ---- DIRECT path: one integer key with a small value range in this chunk
    const TypeId kt0 = keys[0]->type.id;
    const bool int_key = fast && (kt0 == T_INT8 || kt0 == T_INT16 || kt0 == T_INT32 || kt0 == T_INT64 || kt0 == T_DATE32);
    if (int_key && (n_in >= (1 << 15) || getenv("AURON_FORCE_DIRECT_AGG")) && !getenv("AURON_DISABLE_DIRECT_AGG") && !getenv("AURON_AGG_INTERLEAVE") && !getenv("AURON_ENABLE_SMEM_AGG")) {
        FastKey k{keys[0]->data->ptr, keys[0]->vbits(), (int32_t)kt0};
        long long h[2];
        if (keys[0]->has_range) {   // bounds from the scan's column statistics: no pass over the keys
            h[0] = keys[0]->range_min;
            h[1] = keys[0]->range_max;
        } else {
            const long long init[2] = {0x7fffffffffffffffll, (long long)0x8000000000000000ull};
            Buf mm = to_device(ctx, init, 16);
            {
                ProfScope ps(ctx, "agg_key_range");
                const unsigned grid = (unsigned)std::max<int64_t>(1, std::min<int64_t>((n_rows + 1023) / 1024, (int64_t)ctx.sm_count * 8));
                const uint32_t* kv = (const uint32_t*)keys[0]->vbits();
                if (kt0 == T_INT32 || kt0 == T_DATE32) key_minmax_vec_kernel<int32_t><<<grid, 256, 0, ctx.stream>>>((const int32_t*)k.data, kv, n_rows, P<long long>(mm));
                else if (kt0 == T_INT64) key_minmax_vec_kernel<long long><<<grid, 256, 0, ctx.stream>>>((const long long*)k.data, kv, n_rows, P<long long>(mm));
                else key_minmax_kernel<<<agg_grid(ctx, n_rows), 256, 0, ctx.stream>>>(k, n_rows, P<long long>(mm));
                LAUNCH_CHECK(ctx);
            }
            to_host(ctx, h, mm->ptr, 16);
        }
        if (getenv("AURON_AGG_DEBUG")) fprintf(stderr, "[agg] direct candidate: has_range=%d min=%lld max=%lld rows=%lld\n", (int)keys[0]->has_range, h[0], h[1], (long long)n_in);
        const bool any = h[0] <= h[1];
        const unsigned long long span = any ? (unsigned long long)h[1] - (unsigned long long)h[0] : 0ull;
        if (span < (1ull << 22)) {
            auto da = direct_agg_create(ctx, accs, any ? h[0] : 0, any ? h[1] : -1);
            {
                ProfScope ps(ctx, "agg_update");
                if (has_str) agg_direct_kernel<true><<<agg_grid(ctx, n_rows), 256, 0, ctx.stream>>>(k, da->dt, da->args, sel, n_rows, selmask);
                else agg_direct_kernel<false><<<agg_grid(ctx, n_rows), 256, 0, ctx.stream>>>(k, da->dt, da->args, sel, n_rows, selmask);
                LAUNCH_CHECK(ctx);
            }
            bool trusted = !keys[0]->has_range;
            if (!trusted) trusted = !direct_agg_out_of_range(ctx, *da);
            if (trusted) {
                DType kt = keys[0]->type;
                if (fast_key_out) {
                    AURON_CHECK(kt.is_integer() && fast_key_out->is_integer() && kt.width() <= fast_key_out->width(), "bad widened key type");
                    kt = *fast_key_out;
                }
                return direct_agg_finish(ctx, *da, kt, keys[0]->may_have_nulls(), sel);
            }   // else: the file's statistics did not cover the data -> the hash table below starts from scratch
        }
    }
    // capacity: start at 1 Mi slots (covers <= ~500k groups), fall back to 2 x rows on overflow
    int64_t cap = std::min<int64_t>(next_pow2(std::max<int64_t>(2 * n_in, 1024)), 1 << 20);
    for (int attempt = 0;; attempt++) {
        int64_t slots = cap + 2;
        AccBuffers bufs;
        AccArgs args;
        Buf flags = dalloc_zero(ctx, 16);
        Buf table;
        // Separate accumulator arrays, not interleaved records.  The L2 atomic units serialise per cache line, so packing a group's key / sum / count into one sector makes every
        // row of that group contend on a single line, while separate arrays spread the same traffic over 1 + n_accs lines and
        // slices.  Interleaving therefore stays off (AURON_AGG_INTERLEAVE=1 re-enables it for experiments).
        RecLayout layout = (fast && getenv("AURON_AGG_INTERLEAVE")) ? make_layout(accs) : RecLayout();
        const int tw = layout.tw;
        if (fast && tw > 1) {
            table = dalloc(ctx, (size_t)slots * tw * 8);
            RecInit ri;
            memcpy(ri.w, layout.init, sizeof(ri.w));
            int64_t nw = slots * tw;
            init_records_kernel<<<(unsigned)((nw + 255) / 256), 256, 0, ctx.stream>>>(P<unsigned long long>(table), nw, tw, ri);
            LAUNCH_CHECK(ctx);
            args = prepare_accs(ctx, accs, slots, bufs, P<unsigned long long>(table), &layout);
        } else {
            args = prepare_accs(ctx, accs, slots, bufs);
            init_accs(ctx, accs, args, slots);
            if (fast) {
                table = dalloc(ctx, (size_t)cap * 8);
                fill_u64(ctx, table->ptr, cap, EMPTY_KEY);
            }
        }
        if (fast) {
            FastKey k{keys[0]->data->ptr, keys[0]->vbits(), (int32_t)keys[0]->type.id};
            // low-cardinality variant?  decided from a sample of the chunk (exact either way, see agg_fast_smem_kernel)
            bool use_smem = false;
            // 64-bit shared atomics at 2 CTAs/SM are not expected to beat the L2 atomic units (not measured on the H100), so the variant is opt-in (AURON_ENABLE_SMEM_AGG=1) until it is
            // reworked (32-bit partial sums, more CTAs per SM).
            if (attempt == 0 && n_rows >= (1 << 20) && !accs.empty() && (int)accs.size() <= SM_MAX_ACCS && getenv("AURON_ENABLE_SMEM_AGG")) {
                bool kinds_ok = true;
                for (auto& s : accs)
                    kinds_ok = kinds_ok && (s.kind == ACC_SUM_I64 || s.kind == ACC_SUM_F64 || s.kind == ACC_ADD_I64 || s.kind == ACC_COUNT || s.kind == ACC_MIN ||
                                            s.kind == ACC_MAX);
                if (kinds_ok) {
                    GroupedResult sample = hash_aggregate(ctx, keys, {}, sel, std::min<int64_t>(n_rows, 1 << 18), nullptr, selmask, -1);
                    use_smem = sample.num_groups <= 1024;
                }
            }
            if (n_rows && use_smem) {
                static bool attr = false;
                size_t smem = (size_t)SM_SLOTS * 8 * (1 + accs.size()) + (size_t)SM_SLOTS * accs.size();
                if (!attr) {
                    CUDA_OK(cudaFuncSetAttribute(agg_fast_smem_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, SM_SLOTS * 8 * (1 + SM_MAX_ACCS) + SM_SLOTS * SM_MAX_ACCS));
                    attr = true;
                }
                ProfScope ps(ctx, "agg_update");
                agg_fast_smem_kernel<<<ctx.sm_count * 2, 256, smem, ctx.stream>>>(k, P<unsigned long long>(table), tw, cap, args, sel, n_rows, P<int32_t>(flags), selmask);
                LAUNCH_CHECK(ctx);
            } else if (n_rows) {
                ProfScope ps(ctx, "agg_update");
                if (has_str) agg_fast_kernel<true><<<agg_grid(ctx, n_rows), 256, 0, ctx.stream>>>(k, P<unsigned long long>(table), tw, cap, args, sel, n_rows, P<int32_t>(flags), selmask);
                else agg_fast_kernel<false><<<agg_grid(ctx, n_rows), 256, 0, ctx.stream>>>(k, P<unsigned long long>(table), tw, cap, args, sel, n_rows, P<int32_t>(flags), selmask);
                LAUNCH_CHECK(ctx);
            }
        } else {
            table = dalloc_fill(ctx, (size_t)cap * 4, 0xff);
            RowKeys rk = make_row_keys(keys);
            if (n_rows) {
                ProfScope ps(ctx, "agg_update");
                if (has_str) agg_general_kernel<true><<<agg_grid(ctx, n_rows), 256, 0, ctx.stream>>>(rk, P<int32_t>(table), cap, args, sel, n_rows, P<int32_t>(flags), selmask);
                else agg_general_kernel<false><<<agg_grid(ctx, n_rows), 256, 0, ctx.stream>>>(rk, P<int32_t>(table), cap, args, sel, n_rows, P<int32_t>(flags), selmask);
                LAUNCH_CHECK(ctx);
            }
        }
        int32_t hflags[4];
        to_host(ctx, hflags, flags->ptr, 16);
        if (hflags[0]) {   // table too small: retry with the worst-case capacity
            AURON_CHECK(attempt == 0, "hash table overflow after resize");
            cap = next_pow2(std::max<int64_t>(2 * n_in, 1024));
            continue;
        }
        // dense group ids = occupied slots in slot order
        int64_t mask_slots = fast ? slots : cap;
        Buf occ = dalloc(ctx, bitmap_alloc_bytes(mask_slots));
        unsigned mblocks = (unsigned)((mask_slots + 255) / 256);
        if (fast) occupied_mask_fast_kernel<<<mblocks, 256, 0, ctx.stream>>>(P<unsigned long long>(table), tw, cap, P<int32_t>(flags), P<uint32_t>(occ));
        else occupied_mask_general_kernel<<<mblocks, 256, 0, ctx.stream>>>(P<int32_t>(table), cap, P<uint32_t>(occ));
        LAUNCH_CHECK(ctx);
        int64_t g = 0;
        Buf slot_ids = mask_to_indices(ctx, P<uint32_t>(occ), mask_slots, &g);
        res.num_groups = g;
        res.keys = std::make_shared<Batch>();
        res.keys->num_rows = g;
        unsigned gblocks = (unsigned)((g + 255) / 256);
        if (fast) {
            DType kt = keys[0]->type;
            if (fast_key_out) {
                AURON_CHECK(kt.is_integer() && fast_key_out->is_integer() && kt.width() <= fast_key_out->width(), "bad widened key type");
                kt = *fast_key_out;
            }
            auto kc = make_column(ctx, kt, g, keys[0]->may_have_nulls());
            if (g) {
                emit_fast_keys_kernel<<<gblocks, 256, 0, ctx.stream>>>(P<unsigned long long>(table), tw, cap, P<int32_t>(slot_ids), g, kt.id,
                                                                       kc->data->ptr, P<uint32_t>(kc->validity));
                LAUNCH_CHECK(ctx);
            }
            res.keys->cols.push_back(kc);
        } else {
            Buf rep = dalloc(ctx, (size_t)std::max<int64_t>(g, 1) * 4);
            if (g) {
                gather_i32_kernel<<<gblocks, 256, 0, ctx.stream>>>(P<int32_t>(table), P<int32_t>(slot_ids), g, P<int32_t>(rep));
                LAUNCH_CHECK(ctx);
            }
            for (auto& k : keys) res.keys->cols.push_back(take(ctx, *k, P<int32_t>(rep), g, false));
        }
        emit_accs(ctx, accs, args, P<int32_t>(slot_ids), g, sel, res.accs);
        return res;
    }
}

std::vector<ColumnPtr> global_aggregate(Ctx& ctx, const std::vector<AccSpec>& accs, const int32_t* sel, int64_t n_rows, const uint32_t* selmask) {
    AccBuffers bufs;
    AccArgs args = prepare_accs(ctx, accs, 1, bufs);
    init_accs(ctx, accs, args, 1);
    if (n_rows) {
        bool has_str = false;
        for (auto& sp : accs) has_str = has_str || sp.kind == ACC_MIN_STR || sp.kind == ACC_MAX_STR;
        if (has_str) agg_global_kernel<true><<<agg_grid(ctx, n_rows), 256, 0, ctx.stream>>>(args, sel, n_rows, selmask);
        else agg_global_kernel<false><<<agg_grid(ctx, n_rows), 256, 0, ctx.stream>>>(args, sel, n_rows, selmask);
        LAUNCH_CHECK(ctx);
    }
    std::vector<ColumnPtr> out;
    emit_accs(ctx, accs, args, nullptr, 1, sel, out);
    return out;
}

RowKeys make_row_keys(const std::vector<ColumnPtr>& cols) {
    AURON_CHECK((int)cols.size() <= kMaxKeyCols, "too many key columns");
    RowKeys rk;
    memset(&rk, 0, sizeof(rk));
    rk.ncols = (int)cols.size();
    for (int i = 0; i < rk.ncols; i++) {
        rk.c[i].data = cols[i]->data ? cols[i]->data->ptr : nullptr;
        rk.c[i].validity = cols[i]->vbits();
        rk.c[i].offsets = P<int32_t>(cols[i]->offsets);
        rk.c[i].type = cols[i]->type.id;
        rk.c[i].width = cols[i]->type.width();
    }
    return rk;
}

}  // namespace auron

namespace auron {
// AVG final merge (datafusion-ext-plans/src/agg/avg.rs:151-179): non-decimal = f64(sum) / f64(count);
// decimal = sum.checked_div_euclid(count) on the unscaled i128 at the same scale; count 0 or NULL sum => NULL.
__global__ void __launch_bounds__(256) avg_finalize_kernel(const void* __restrict__ sum, const uint8_t* __restrict__ sum_valid, int32_t sum_type,
                                                           const int64_t* __restrict__ cnt, const uint8_t* __restrict__ cnt_valid, int64_t n,
                                                           int32_t out_type, void* __restrict__ out, uint32_t* __restrict__ out_valid) {
    int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x;
    bool ok = false;
    if (i < n) {
        int64_t c = valid_at(cnt_valid, i) ? cnt[i] : 0;
        ok = valid_at(sum_valid, i) && c != 0;
        if (sum_type == T_DECIMAL128) {
            i128 q = {0, 0};
            if (ok) {
                ulonglong2 s = ((const ulonglong2*)sum)[i];
                i128 v = {s.x, (int64_t)s.y};
                bool neg = i128_is_neg(v);
                i128 a = neg ? i128_neg(v) : v;
                uint64_t rem;
                q = u128_divmod_u64(a, (uint64_t)c, &rem);   // c > 0 (a count)
                if (neg) {
                    q = i128_neg(q);
                    if (rem != 0) q = i128_sub(q, {1, 0});   // euclid: remainder stays non-negative
                }
            }
            ((uint64_t*)out)[2 * i] = q.lo;
            ((int64_t*)out)[2 * i + 1] = q.hi;
        } else {
            double s = ok ? (sum_type == T_FLOAT64 ? ((const double*)sum)[i] : (double)((const int64_t*)sum)[i]) : 0.0;
            double r = ok ? s / (double)c : 0.0;
            if (out_type == T_FLOAT32) ((float*)out)[i] = (float)r;
            else ((double*)out)[i] = r;
        }
    }
    uint32_t w = __ballot_sync(FULL_MASK, ok);
    if (lane_id() == 0 && i < n) out_valid[i >> 5] = w;
}
ColumnPtr avg_finalize(Ctx& ctx, const Column& sum, const Column& cnt, const DType& out_type) {
    AURON_CHECK(cnt.type.id == T_INT64, "AVG count accumulator must be int64");
    AURON_CHECK(sum.type.id == T_DECIMAL128 || sum.type.id == T_FLOAT64 || sum.type.id == T_INT64, "AVG sum accumulator type " + sum.type.str());
    AURON_CHECK(out_type.id == T_DECIMAL128 ? sum.type.id == T_DECIMAL128 : out_type.is_float(), "AVG result type " + out_type.str());
    int64_t n = sum.len;
    auto out = make_column(ctx, out_type, n, true);
    if (n) {
        avg_finalize_kernel<<<(unsigned)((n + 255) / 256), 256, 0, ctx.stream>>>(sum.data->ptr, sum.vbits(), sum.type.id, P<int64_t>(cnt.data), cnt.vbits(), n,
                                                                                 out_type.id, out->data->ptr, P<uint32_t>(out->validity));
        LAUNCH_CHECK(ctx);
    }
    return out;
}
}  // namespace auron
