// k_join.cu -- hash join build + probe on device (rows J2-J4 of SURVEY.md section 8a).
//
// Replaces JoinHashMap::create_from_data_batch / Table::create (datafusion-ext-plans/src/joins/
// join_hash_map.rs:99-193), Table::lookup_many (:231-274) and the pair generation of FullJoiner::join
// (joins/bhj/full_join.rs:216-325).  The reference sorts (hash, idx) pairs to group duplicate keys into
// `mapped_indices` runs; here the build is sort-free:
//   1. every build row with non-NULL keys claims / finds its key slot in an open-addressed table (HBM)
//      and bumps a per-slot counter                                  (join_hash_map.rs:118,127: NULL keys are skipped)
//   2. an exclusive scan of the counters gives each key its run in `rows`
//   3. a second pass drops each build row index into its key's run
// Probe: slot lookup + key verification (EqComparator semantics: hash hits are re-verified on the key
// values, eq_comparator.rs:42-98), a count pass, a scan, and a write pass that emits (probe_idx, build_idx)
// pairs; output columns are then gathered with take() (full_join.rs:148-211 flush_hash_joined).
//
// Roofline: the probe is an HBM stream over the probe key column (4-8 B/row) while the build table
// (date_dim: 73,049 rows -> 1 MiB) stays L2-resident; pairs cost 8 B/match out.
#include "kernels.h"
#include "rowkeys.cuh"

namespace auron {

#define LAUNCH_CHECK(ctx)            \
    do {                             \
        CUDA_OK(cudaGetLastError()); \
        launch_count(ctx);           \
    } while (0)

constexpr uint64_t J_EMPTY = 0x8A5C3F1E9D7B2461ull;
constexpr int J_MAX_PROBE = 1 << 20;   // table load <= 0.5, so probes are short; bound only guards against bugs

struct JoinTable {
    bool fast = false;
    int64_t cap = 0, n_build = 0, n_rows_in_table = 0;
    int32_t key_type = 0;
    Buf table;     // fast: u64 keys[cap] ; general: int32 representative build row[cap]
    Buf counts;    // int32[cap + 1]   (slot `cap` = sentinel-valued key on the fast path)
    Buf offsets;   // int32[cap + 2]   exclusive scan of counts
    Buf rows;      // int32[n_rows_in_table] build row indices grouped by key
    std::vector<ColumnPtr> keys;   // build key columns (kept alive for verification)
    bool has_null_key = false;
    bool unique = false;           // no key occurs twice on the build side (a dimension table joined on its primary key)
    // unique integer keys spanning a small range (surrogate keys): build row by key - dmin, -1 = absent.  One 4-byte load per probe
    // row from a table that mostly stays in L1 (date_dim: 292 KB), where the hashed table costs four dependent 32-byte L2 sectors
    // (slot, count, offset, row) -- the hashed probe would be bound by L2 bandwidth.
    Buf direct;
    long long dmin = 0;
    int64_t drange = -1;
};
bool join_table_has_null_key(const JoinTable& t) { return t.has_null_key; }
bool join_table_unique_fast(const JoinTable& t) { return t.unique && t.fast; }

struct JKey {
    const void* data;
    const uint8_t* validity;
    int32_t type;
};
__device__ __forceinline__ uint64_t jload_key64(const JKey& k, int64_t row) {
    switch (k.type) {
        case T_INT8: return (uint64_t)(int64_t)((const int8_t*)k.data)[row];
        case T_INT16: return (uint64_t)(int64_t)((const int16_t*)k.data)[row];
        case T_INT32: case T_DATE32: return (uint64_t)(int64_t)((const int32_t*)k.data)[row];
        case T_FLOAT32: return (uint64_t)((const uint32_t*)k.data)[row];
        case T_DECIMAL128: return ((const uint64_t*)k.data)[row * 2];
        default: return ((const uint64_t*)k.data)[row];
    }
}

// ---- build pass 1: claim slots + count
__global__ void __launch_bounds__(256) jbuild_count_fast(JKey key, unsigned long long* __restrict__ table, int64_t cap, int32_t* __restrict__ counts,
                                                         int64_t n, int32_t* __restrict__ flags) {
    int64_t row = (int64_t)blockIdx.x * 256 + threadIdx.x;
    if (row >= n) return;
    if (key.validity && !bit_get(key.validity, row)) {
        flags[0] = 1;   // build side has a NULL key
        return;
    }
    uint64_t k = jload_key64(key, row), mask = (uint64_t)cap - 1;
    if (k == J_EMPTY) {
        atomicAdd(&counts[cap], 1);
        return;
    }
    uint64_t h = mix64(k) & mask;
    for (int p = 0; p < J_MAX_PROBE; p++) {
        unsigned long long cur = table[h];
        if (cur == J_EMPTY) {
            unsigned long long old = atomicCAS(&table[h], (unsigned long long)J_EMPTY, (unsigned long long)k);
            if (old == J_EMPTY) cur = k;
            else cur = old;
        }
        if (cur == k) {
            atomicAdd(&counts[h], 1);
            return;
        }
        h = (h + 1) & mask;
    }
    flags[1] = 1;
}
__global__ void __launch_bounds__(256) jbuild_count_general(RowKeys keys, int32_t* __restrict__ slots, int64_t cap, int32_t* __restrict__ counts,
                                                            int64_t n, int32_t* __restrict__ flags) {
    int64_t row = (int64_t)blockIdx.x * 256 + threadIdx.x;
    if (row >= n) return;
    if (rowkey_has_null(keys, row)) {
        flags[0] = 1;
        return;
    }
    uint64_t mask = (uint64_t)cap - 1, h = rowkey_hash(keys, row) & mask;
    for (int p = 0; p < J_MAX_PROBE; p++) {
        int32_t cur = slots[h];
        if (cur < 0) {
            int32_t old = atomicCAS(&slots[h], -1, (int32_t)row);
            cur = old < 0 ? (int32_t)row : old;
        }
        if (cur == (int32_t)row || rowkey_equal(keys, cur, keys, row)) {
            atomicAdd(&counts[h], 1);
            return;
        }
        h = (h + 1) & mask;
    }
    flags[1] = 1;
}

// ---- lookup helpers (table is read-only from here on)
__device__ __forceinline__ int64_t jfind_fast(const unsigned long long* __restrict__ table, int64_t cap, uint64_t k) {
    if (k == J_EMPTY) return cap;
    uint64_t mask = (uint64_t)cap - 1, h = mix64(k) & mask;
    for (int p = 0; p < J_MAX_PROBE; p++) {
        unsigned long long cur = table[h];
        if (cur == k) return (int64_t)h;
        if (cur == J_EMPTY) return -1;
        h = (h + 1) & mask;
    }
    return -1;
}
__device__ __forceinline__ int64_t jfind_general(const int32_t* __restrict__ slots, int64_t cap, const RowKeys& bkeys, const RowKeys& pkeys,
                                                 int64_t prow) {
    uint64_t mask = (uint64_t)cap - 1, h = rowkey_hash(pkeys, prow) & mask;
    for (int p = 0; p < J_MAX_PROBE; p++) {
        int32_t cur = slots[h];
        if (cur < 0) return -1;
        if (rowkey_equal(bkeys, cur, pkeys, prow)) return (int64_t)h;
        h = (h + 1) & mask;
    }
    return -1;
}

// ---- build pass 2: fill runs
__global__ void __launch_bounds__(256) jbuild_fill_fast(JKey key, const unsigned long long* __restrict__ table, int64_t cap,
                                                        const int32_t* __restrict__ offsets, int32_t* __restrict__ cursors,
                                                        int32_t* __restrict__ rows, int64_t n) {
    int64_t row = (int64_t)blockIdx.x * 256 + threadIdx.x;
    if (row >= n) return;
    if (key.validity && !bit_get(key.validity, row)) return;
    int64_t s = jfind_fast(table, cap, jload_key64(key, row));
    if (s < 0) return;
    int32_t pos = atomicAdd(&cursors[s], 1);
    rows[offsets[s] + pos] = (int32_t)row;
}
__global__ void __launch_bounds__(256) jbuild_fill_general(RowKeys keys, const int32_t* __restrict__ slots, int64_t cap,
                                                           const int32_t* __restrict__ offsets, int32_t* __restrict__ cursors,
                                                           int32_t* __restrict__ rows, int64_t n) {
    int64_t row = (int64_t)blockIdx.x * 256 + threadIdx.x;
    if (row >= n) return;
    if (rowkey_has_null(keys, row)) return;
    int64_t s = jfind_general(slots, cap, keys, keys, row);
    if (s < 0) return;
    int32_t pos = atomicAdd(&cursors[s], 1);
    rows[offsets[s] + pos] = (int32_t)row;
}
// runs are filled in nondeterministic order; sort each run ascending so results are reproducible
// (runs are short: one thread insertion-sorts its slot's run)
__global__ void jbuild_sort_runs(const int32_t* __restrict__ offsets, int32_t* __restrict__ rows, int64_t nslots) {
    int64_t s = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= nslots) return;
    int32_t b = offsets[s], e = offsets[s + 1];
    if (e - b > 64) return;   // long duplicate runs keep their fill order (pair order is unspecified anyway)
    for (int32_t i = b + 1; i < e; i++) {
        int32_t v = rows[i], j = i - 1;
        while (j >= b && rows[j] > v) {
            rows[j + 1] = rows[j];
            j--;
        }
        rows[j + 1] = v;
    }
}

// ---- probe pass 1: slot + match count per probe row
__global__ void __launch_bounds__(256) jprobe_count_fast(JKey key, const unsigned long long* __restrict__ table, int64_t cap,
                                                         const int32_t* __restrict__ counts, int64_t n, bool probe_outer,
                                                         int32_t* __restrict__ slot_out, int32_t* __restrict__ cnt_out,
                                                         uint32_t* __restrict__ probe_matched) {
    int64_t row = (int64_t)blockIdx.x * 256 + threadIdx.x;
    int32_t c = 0;
    if (row < n) {
        int64_t s = -1;
        if (!(key.validity && !bit_get(key.validity, row))) s = jfind_fast(table, cap, jload_key64(key, row));
        if (s >= 0) c = counts[s];
        if (c == 0) s = -1;
        slot_out[row] = (int32_t)s;
        cnt_out[row] = (c == 0 && probe_outer) ? 1 : c;
    }
    if (probe_matched) {
        uint32_t w = __ballot_sync(FULL_MASK, c > 0);
        if (lane_id() == 0 && row < n) probe_matched[row >> 5] = w;
    }
}
__global__ void __launch_bounds__(256) jprobe_count_general(RowKeys bkeys, RowKeys pkeys, const int32_t* __restrict__ slots, int64_t cap,
                                                            const int32_t* __restrict__ counts, int64_t n, bool probe_outer,
                                                            int32_t* __restrict__ slot_out, int32_t* __restrict__ cnt_out,
                                                            uint32_t* __restrict__ probe_matched) {
    int64_t row = (int64_t)blockIdx.x * 256 + threadIdx.x;
    int32_t c = 0;
    if (row < n) {
        int64_t s = -1;
        if (!rowkey_has_null(pkeys, row)) s = jfind_general(slots, cap, bkeys, pkeys, row);
        if (s >= 0) c = counts[s];
        if (c == 0) s = -1;
        slot_out[row] = (int32_t)s;
        cnt_out[row] = (c == 0 && probe_outer) ? 1 : c;
    }
    if (probe_matched) {
        uint32_t w = __ballot_sync(FULL_MASK, c > 0);
        if (lane_id() == 0 && row < n) probe_matched[row >> 5] = w;
    }
}
// ---- probe pass 2: write pairs
__global__ void __launch_bounds__(256) jprobe_write(const int32_t* __restrict__ slot_of, const int32_t* __restrict__ out_pos,
                                                    const int32_t* __restrict__ offsets, const int32_t* __restrict__ rows, int64_t n,
                                                    bool probe_outer, int32_t* __restrict__ probe_idx, int32_t* __restrict__ build_idx,
                                                    uint32_t* __restrict__ matched_build) {
    int64_t row = (int64_t)blockIdx.x * 256 + threadIdx.x;
    if (row >= n) return;
    int32_t s = slot_of[row], pos = out_pos[row];
    if (s < 0) {
        if (probe_outer) {
            probe_idx[pos] = (int32_t)row;
            build_idx[pos] = -1;
        }
        return;
    }
    int32_t b = offsets[s], e = offsets[s + 1];
    for (int32_t j = b; j < e; j++) {
        int32_t br = rows[j];
        probe_idx[pos] = (int32_t)row;
        build_idx[pos] = br;
        pos++;
        if (matched_build) {
            uint32_t bit = 1u << (br & 31);
            if (!(matched_build[br >> 5] & bit)) atomicOr(&matched_build[br >> 5], bit);
        }
    }
}

__global__ void __launch_bounds__(256) jcount_max(const int32_t* __restrict__ counts, int64_t n, int32_t* __restrict__ out) {
    int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x;
    int c = i < n ? counts[i] : 0;
#pragma unroll
    for (int d = 16; d; d >>= 1) c = max(c, __shfl_xor_sync(FULL_MASK, c, d));
    if (lane_id() == 0 && c > 1) atomicMax(out, c);
}
// Probe of a build side without duplicate keys: every probe row has at most one partner, so the result is a partner index per probe row
// (-1 = none) plus a match mask -- one pass, no pair list; the probe-side columns are used in place under the mask.
__global__ void __launch_bounds__(256) jprobe_unique_fast(JKey key, const unsigned long long* __restrict__ table, int64_t cap, const int32_t* __restrict__ counts,
                                                          const int32_t* __restrict__ offsets, const int32_t* __restrict__ rows, int64_t n,
                                                          int32_t* __restrict__ build_idx, uint32_t* __restrict__ mask, unsigned long long* __restrict__ matched) {
    int cnt = 0;
    const int64_t n32 = (n + 31) & ~(int64_t)31;
    for (int64_t row = (int64_t)blockIdx.x * 256 + threadIdx.x; row < n32; row += (int64_t)gridDim.x * 256) {
        int32_t b = -1;
        if (row < n && !(key.validity && !bit_get(key.validity, row))) {
            const int64_t s = jfind_fast(table, cap, jload_key64(key, row));
            if (s >= 0 && counts[s] > 0) b = rows[offsets[s]];
        }
        if (row < n) build_idx[row] = b;
        const uint32_t w = __ballot_sync(FULL_MASK, b >= 0);
        if (lane_id() == 0) mask[row >> 5] = w;
        cnt += b >= 0;
    }
    __shared__ int s_cnt;
    if (threadIdx.x == 0) s_cnt = 0;
    __syncthreads();
    if (cnt) atomicAdd(&s_cnt, cnt);
    __syncthreads();
    if (threadIdx.x == 0 && s_cnt) atomicAdd(matched, (unsigned long long)s_cnt);
}
__global__ void __launch_bounds__(256) jkey_minmax(JKey key, int64_t n, long long* __restrict__ out) {
    const int64_t row = (int64_t)blockIdx.x * 256 + threadIdx.x;
    long long mn = 0x7fffffffffffffffll, mx = -0x7fffffffffffffffll - 1;
    if (row < n && !(key.validity && !bit_get(key.validity, row))) mn = mx = (long long)jload_key64(key, row);
#pragma unroll
    for (int d = 16; d; d >>= 1) {
        mn = min(mn, __shfl_xor_sync(FULL_MASK, mn, d));
        mx = max(mx, __shfl_xor_sync(FULL_MASK, mx, d));
    }
    if (lane_id() == 0 && mn <= mx) {
        atomicMin(&out[0], mn);
        atomicMax(&out[1], mx);
    }
}
__global__ void __launch_bounds__(256) jdirect_fill(JKey key, int64_t n, long long dmin, int32_t* __restrict__ direct) {
    const int64_t row = (int64_t)blockIdx.x * 256 + threadIdx.x;
    if (row < n && !(key.validity && !bit_get(key.validity, row))) direct[jload_key64(key, row) - (unsigned long long)dmin] = (int32_t)row;
}
// (grid-stride: a block counts its matches in registers and adds them once -- one atomic per warp on a single address
// serialised in L2 and cost 10x the lookups)
__global__ void __launch_bounds__(256) jprobe_unique_direct(JKey key, const int32_t* __restrict__ direct, long long dmin, int64_t drange, int64_t n,
                                                            int32_t* __restrict__ build_idx, uint32_t* __restrict__ mask, unsigned long long* __restrict__ matched) {
    int cnt = 0;
    const int64_t n32 = (n + 31) & ~(int64_t)31;   // whole warps take part in the ballot
    for (int64_t row = (int64_t)blockIdx.x * 256 + threadIdx.x; row < n32; row += (int64_t)gridDim.x * 256) {
        int32_t b = -1;
        if (row < n && !(key.validity && !bit_get(key.validity, row))) {
            const unsigned long long d = jload_key64(key, row) - (unsigned long long)dmin;   // wraps for keys below dmin
            if (d <= (unsigned long long)drange) b = __ldg(direct + d);
        }
        if (row < n) build_idx[row] = b;
        const uint32_t w = __ballot_sync(FULL_MASK, b >= 0);
        if (lane_id() == 0) mask[row >> 5] = w;
        cnt += b >= 0;
    }
    __shared__ int s_cnt;
    if (threadIdx.x == 0) s_cnt = 0;
    __syncthreads();
    if (cnt) atomicAdd(&s_cnt, cnt);
    __syncthreads();
    if (threadIdx.x == 0 && s_cnt) atomicAdd(matched, (unsigned long long)s_cnt);
}
static int64_t jnext_pow2(int64_t v) {
    int64_t p = 1;
    while (p < v) p <<= 1;
    return p;
}
static bool jfast_ok(const std::vector<ColumnPtr>& keys) {
    if (keys.size() != 1) return false;
    const DType& t = keys[0]->type;
    if (t.id == T_DECIMAL128) return t.precision <= 18;
    return t.width() >= 1 && t.width() <= 8;
}
__global__ void jfill_u64(unsigned long long* p, int64_t n, unsigned long long v) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) p[i] = v;
}

std::shared_ptr<JoinTable> join_build(Ctx& ctx, const std::vector<ColumnPtr>& build_keys, int64_t n_build) {
    ProfScope ps_fn(ctx, "join_build");
    AURON_CHECK(n_build < (1ll << 30), "join build side must be < 2^30 rows (join_hash_map.rs:100-103)");
    auto t = std::make_shared<JoinTable>();
    t->fast = jfast_ok(build_keys);
    t->n_build = n_build;
    t->keys = build_keys;
    t->key_type = build_keys[0]->type.id;
    t->cap = jnext_pow2(std::max<int64_t>(2 * n_build, 1024));
    int64_t cap = t->cap;
    t->counts = dalloc_zero(ctx, (size_t)(cap + 2) * 4);
    t->offsets = dalloc_zero(ctx, (size_t)(cap + 3) * 4);
    Buf flags = dalloc_zero(ctx, 16);
    unsigned blocks = (unsigned)((n_build + 255) / 256);
    RowKeys rk;
    JKey jk{};
    if (t->fast) {
        t->table = dalloc(ctx, (size_t)cap * 8);
        jfill_u64<<<(unsigned)((cap + 255) / 256), 256, 0, ctx.stream>>>(P<unsigned long long>(t->table), cap, J_EMPTY);
        LAUNCH_CHECK(ctx);
        jk = JKey{build_keys[0]->data->ptr, build_keys[0]->vbits(), (int32_t)build_keys[0]->type.id};
        if (n_build) {
            jbuild_count_fast<<<blocks, 256, 0, ctx.stream>>>(jk, P<unsigned long long>(t->table), cap, P<int32_t>(t->counts), n_build, P<int32_t>(flags));
            LAUNCH_CHECK(ctx);
        }
    } else {
        t->table = dalloc_fill(ctx, (size_t)cap * 4, 0xff);
        rk = make_row_keys(build_keys);
        if (n_build) {
            jbuild_count_general<<<blocks, 256, 0, ctx.stream>>>(rk, P<int32_t>(t->table), cap, P<int32_t>(t->counts), n_build, P<int32_t>(flags));
            LAUNCH_CHECK(ctx);
        }
    }
    Buf total = dalloc(ctx, 4);
    exclusive_scan_i32(ctx, P<int32_t>(t->counts), P<int32_t>(t->offsets), cap + 1, P<int32_t>(total));
    jcount_max<<<(unsigned)((cap + 1 + 255) / 256), 256, 0, ctx.stream>>>(P<int32_t>(t->counts), cap + 1, P<int32_t>(flags) + 2);
    LAUNCH_CHECK(ctx);
    int32_t hflags[4], htotal = 0;
    to_host(ctx, hflags, flags->ptr, 16);
    to_host(ctx, &htotal, total->ptr, 4);
    AURON_CHECK(!hflags[1], "join hash table probe overflow");
    t->has_null_key = hflags[0] != 0;
    t->unique = hflags[2] <= 1;
    t->n_rows_in_table = htotal;
    CUDA_OK(cudaMemcpyAsync(P<int32_t>(t->offsets) + cap + 1, total->ptr, 4, cudaMemcpyDeviceToDevice, ctx.stream));
    t->rows = dalloc(ctx, (size_t)std::max<int32_t>(htotal, 1) * 4);
    if (n_build && htotal) {
        Buf cursors = dalloc_zero(ctx, (size_t)(cap + 1) * 4);
        if (t->fast) jbuild_fill_fast<<<blocks, 256, 0, ctx.stream>>>(jk, P<unsigned long long>(t->table), cap, P<int32_t>(t->offsets), P<int32_t>(cursors), P<int32_t>(t->rows), n_build);
        else jbuild_fill_general<<<blocks, 256, 0, ctx.stream>>>(rk, P<int32_t>(t->table), cap, P<int32_t>(t->offsets), P<int32_t>(cursors), P<int32_t>(t->rows), n_build);
        LAUNCH_CHECK(ctx);
        jbuild_sort_runs<<<(unsigned)((cap + 1 + 255) / 256), 256, 0, ctx.stream>>>(P<int32_t>(t->offsets), P<int32_t>(t->rows), cap + 1);
        LAUNCH_CHECK(ctx);
    }
    const int kt = t->key_type;
    if (t->fast && t->unique && htotal > 0 && (kt == T_INT8 || kt == T_INT16 || kt == T_INT32 || kt == T_INT64 || kt == T_DATE32)) {
        const long long init[2] = {0x7fffffffffffffffll, -0x7fffffffffffffffll - 1};
        Buf mm = to_device(ctx, init, 16);
        jkey_minmax<<<blocks, 256, 0, ctx.stream>>>(jk, n_build, P<long long>(mm));
        LAUNCH_CHECK(ctx);
        long long h[2];
        to_host(ctx, h, mm->ptr, 16);
        // the span in unsigned arithmetic: h[1] - h[0] overflows int64 when the keys reach both ends of the range, and a compiler
        // may then fold the signed difference into a small one
        const unsigned long long span = (unsigned long long)h[1] - (unsigned long long)h[0];
        if (h[0] <= h[1] && span < (16ull << 20)) {
            t->dmin = h[0];
            t->drange = (int64_t)span;
            t->direct = dalloc_fill(ctx, (size_t)(t->drange + 1) * 4, 0xff);
            jdirect_fill<<<blocks, 256, 0, ctx.stream>>>(jk, n_build, t->dmin, P<int32_t>(t->direct));
            LAUNCH_CHECK(ctx);
        }
    }
    return t;
}

JoinPairs join_probe(Ctx& ctx, const JoinTable& t, const std::vector<ColumnPtr>& probe_keys, int64_t n_probe, bool probe_outer,
                     uint32_t* matched_build, Buf* probe_matched_out) {
    ProfScope ps_fn(ctx, "join_probe");
    JoinPairs out;
    AURON_CHECK(n_probe < (int64_t)INT32_MAX, "probe chunk too large");
    AURON_CHECK(probe_keys.size() == t.keys.size(), "join key arity mismatch");
    Buf slot_of = dalloc(ctx, (size_t)std::max<int64_t>(n_probe, 1) * 4);
    Buf cnt = dalloc(ctx, (size_t)(n_probe + 1) * 4);
    Buf pm;
    if (probe_matched_out) {
        pm = dalloc_zero(ctx, bitmap_alloc_bytes(n_probe));
        *probe_matched_out = pm;
    }
    unsigned blocks = (unsigned)((n_probe + 255) / 256);
    if (n_probe == 0) {
        out.probe_idx = dalloc(ctx, 4);
        out.build_idx = dalloc(ctx, 4);
        return out;
    }
    if (t.fast) {
        const DType& pt = probe_keys[0]->type;
        AURON_CHECK(pt.width() >= 1 && (pt.width() <= 8 || pt.id == T_DECIMAL128), "probe key type incompatible with build key");
        JKey jk{probe_keys[0]->data->ptr, probe_keys[0]->vbits(), (int32_t)pt.id};
        jprobe_count_fast<<<blocks, 256, 0, ctx.stream>>>(jk, P<unsigned long long>(t.table), t.cap, P<int32_t>(t.counts), n_probe, probe_outer,
                                                          P<int32_t>(slot_of), P<int32_t>(cnt), P<uint32_t>(pm));
    } else {
        RowKeys bk = make_row_keys(t.keys), pk = make_row_keys(probe_keys);
        for (int i = 0; i < bk.ncols; i++) AURON_CHECK(bk.c[i].width == pk.c[i].width && (bk.c[i].width > 0 || bk.c[i].type == pk.c[i].type || (t.keys[i]->type.is_varlen() && probe_keys[i]->type.is_varlen())), "join key type mismatch");
        jprobe_count_general<<<blocks, 256, 0, ctx.stream>>>(bk, pk, P<int32_t>(t.table), t.cap, P<int32_t>(t.counts), n_probe, probe_outer,
                                                             P<int32_t>(slot_of), P<int32_t>(cnt), P<uint32_t>(pm));
    }
    LAUNCH_CHECK(ctx);
    // positions: 64-bit total guards against > 2^31 pairs in one chunk
    Buf total = dalloc(ctx, 4);
    exclusive_scan_i32(ctx, P<int32_t>(cnt), P<int32_t>(cnt), n_probe, P<int32_t>(total));
    int32_t htotal = 0;
    to_host(ctx, &htotal, total->ptr, 4);
    AURON_CHECK(htotal >= 0, "join produced more than 2^31 pairs in one chunk");
    out.count = htotal;
    out.probe_idx = dalloc(ctx, (size_t)std::max<int32_t>(htotal, 1) * 4);
    out.build_idx = dalloc(ctx, (size_t)std::max<int32_t>(htotal, 1) * 4);
    if (htotal > 0 || matched_build) {
        jprobe_write<<<blocks, 256, 0, ctx.stream>>>(P<int32_t>(slot_of), P<int32_t>(cnt), P<int32_t>(t.offsets), P<int32_t>(t.rows), n_probe, probe_outer,
                                                     P<int32_t>(out.probe_idx), P<int32_t>(out.build_idx), matched_build);
        LAUNCH_CHECK(ctx);
    }
    return out;
}

int64_t join_probe_unique(Ctx& ctx, const JoinTable& t, const ColumnPtr& probe_key, int64_t n_probe, Buf* build_idx, Buf* mask) {
    ProfScope ps_fn(ctx, "join_probe");
    AURON_CHECK(t.unique && t.fast, "join_probe_unique needs a build side without duplicate keys and a single fixed-width key");
    AURON_CHECK(n_probe < (int64_t)INT32_MAX, "probe chunk too large");
    const DType& pt = probe_key->type;
    AURON_CHECK(pt.width() >= 1 && (pt.width() <= 8 || pt.id == T_DECIMAL128), "probe key type incompatible with build key");
    *build_idx = dalloc(ctx, (size_t)std::max<int64_t>(n_probe, 1) * 4);
    *mask = dalloc_zero(ctx, bitmap_alloc_bytes(n_probe));
    if (n_probe == 0) return 0;
    Buf matched = dalloc_zero(ctx, 8);
    JKey jk{probe_key->data->ptr, probe_key->vbits(), (int32_t)pt.id};
    const unsigned pgrid = (unsigned)std::min<int64_t>((n_probe + 255) / 256, (int64_t)ctx.sm_count * 16);   // 8 resident blocks per SM, two rounds
    const bool int_key = pt.id == T_INT8 || pt.id == T_INT16 || pt.id == T_INT32 || pt.id == T_INT64 || pt.id == T_DATE32;
    if (t.direct && int_key)
        jprobe_unique_direct<<<pgrid, 256, 0, ctx.stream>>>(jk, P<int32_t>(t.direct), t.dmin, t.drange, n_probe, P<int32_t>(*build_idx),
                                                                                     P<uint32_t>(*mask), P<unsigned long long>(matched));
    else
        jprobe_unique_fast<<<pgrid, 256, 0, ctx.stream>>>(jk, P<unsigned long long>(t.table), t.cap, P<int32_t>(t.counts), P<int32_t>(t.offsets),
                                                                                   P<int32_t>(t.rows), n_probe, P<int32_t>(*build_idx), P<uint32_t>(*mask),
                                                                                   P<unsigned long long>(matched));
    LAUNCH_CHECK(ctx);
    unsigned long long h = 0;
    to_host(ctx, &h, matched->ptr, 8);
    return (int64_t)h;
}

}  // namespace auron
