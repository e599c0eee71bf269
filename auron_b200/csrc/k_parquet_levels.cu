// k_parquet_levels.cu -- the level pass of one-level Parquet LIST columns (LogicalTypes.md, "Lists"; the reference reads them through
// arrow-rs and casts the elements to the table's element type, scan/mod.rs:143-156).
//
// A list page holds one level slot per element, empty list or NULL list: a repetition level (0 = the slot starts a row) and a
// definition level.  The element values are the page's value section, contiguous and without gaps, and are decoded by the flat
// page decoders (k_parquet.cu) as a required column.  This pass turns the levels of every page of a batch into
//   - the int32 list offsets   (row r starts at the number of elements in the slots before r's first slot),
//   - the list validity        (def >= list_def at a row's first slot),
//   - elem_idx                 (element e -> index of its value among the non-null values, -1 for a NULL element),
// in four steps: expand the hybrid streams into one byte per slot (one warp per page and stream), flag every slot, two exclusive
// scans, one scatter.  A batch holds whole row groups, so every row's slots are in the batch; a row may straddle pages.
#include "device_utils.cuh"
#include "kernels.h"
#include "parquet_dev.h"

namespace auron {

#define LAUNCH_CHECK(ctx)            \
    do {                             \
        CUDA_OK(cudaGetLastError()); \
        launch_count(ctx);           \
    } while (0)

// One RLE / bit-packed hybrid stream of bit width bw (<= 8) -> n bytes at out.  Every lane walks the run headers (the same bytes: one
// broadcast load each); the lanes write the values of a run in parallel.  True when the stream is well formed and no value exceeds
// max_value (a value that does is clamped, so the later steps stay in bounds whatever the bytes say).
__device__ bool expand_hybrid(const uint8_t* p, int32_t len, int bw, int32_t n, uint8_t* __restrict__ out, uint32_t max_value) {
    const unsigned lane = lane_id();
    const uint8_t* end = p + (len > 0 ? len : 0);
    const uint32_t mask = (1u << bw) - 1u;
    bool ok = true, lane_ok = true;
    int32_t f = 0;
    while (f < n) {
        uint32_t h = 0;
        bool got = false;
        for (int shift = 0; p < end && shift < 35; shift += 7) {
            const uint8_t b = *p++;
            h |= (uint32_t)(b & 0x7f) << shift;
            if (!(b & 0x80)) {
                got = true;
                break;
            }
        }
        if (!got) {
            ok = false;
            break;
        }
        if (h & 1) {   // bit-packed: (h >> 1) groups of 8 values
            const int64_t bytes = (int64_t)(h >> 1) * bw;
            if (bytes > end - p) {
                ok = false;
                break;
            }
            const int32_t t = (int32_t)min((int64_t)(n - f), (int64_t)(h >> 1) * 8);
            for (int32_t i = (int32_t)lane; i < t; i += 32) {
                const int64_t bit = (int64_t)i * bw;
                const uint8_t* q = p + (bit >> 3);
                uint32_t w = q[0];
                if ((int)(bit & 7) + bw > 8) w |= (uint32_t)q[1] << 8;   // (still inside the run's bytes)
                uint32_t v = (w >> (bit & 7)) & mask;
                if (v > max_value) lane_ok = false, v = max_value;
                out[f + i] = (uint8_t)v;
            }
            p += bytes;
            f += t;
        } else {   // RLE: (h >> 1) copies of one value of ceil(bw / 8) bytes
            const int nb = (bw + 7) / 8;
            if (nb > end - p) {
                ok = false;
                break;
            }
            uint32_t v = nb ? p[0] : 0;
            p += nb;
            if (v > max_value) ok = false, v = max_value;
            const int32_t t = (int32_t)min((int64_t)(n - f), (int64_t)(h >> 1));
            for (int32_t i = (int32_t)lane; i < t; i += 32) out[f + i] = (uint8_t)v;
            f += t;
        }
    }
    if (!ok)   // a stream that ends early: the rest of the page reads as level 0 (the batch fails on the status word)
        for (int32_t i = f + (int32_t)lane; i < n; i += 32) out[i] = 0;
    return !__any_sync(FULL_MASK, !(ok && lane_ok));
}

constexpr int LV_WARPS = 4;
// one warp per (page, stream): warp 2k expands page k's repetition levels, warp 2k + 1 its definition levels
__global__ void __launch_bounds__(LV_WARPS * 32) pq_levels_expand_kernel(const PqLevelPage* __restrict__ pages, int n_pages, PqListShape s,
                                                                         uint8_t* __restrict__ rep, uint8_t* __restrict__ def, int64_t* __restrict__ counts) {
    const int64_t w = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (w >= 2 * (int64_t)n_pages) return;
    const PqLevelPage pg = pages[w >> 1];
    const bool is_def = w & 1;
    const bool ok = is_def ? expand_hybrid(pg.def, pg.def_len, s.def_bw, pg.n_slots, def + pg.slot_start, (uint32_t)s.max_def)
                           : expand_hybrid(pg.rep, pg.rep_len, s.rep_bw, pg.n_slots, rep + pg.slot_start, 1u);
    if (!ok && lane_id() == 0) atomicCAS((unsigned long long*)&counts[3], 0ull, (unsigned long long)((w >> 1) + 1));
}

// re[s] = (starts a row) << 32 | (holds an element); vv[s] = holds a non-null value
__global__ void pq_levels_flags_kernel(const uint8_t* __restrict__ rep, const uint8_t* __restrict__ def, int64_t n, PqListShape s, int64_t* __restrict__ re,
                                       int32_t* __restrict__ vv) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int d = def[i];
    re[i] = ((int64_t)(rep[i] == 0) << 32) | (int64_t)(d >= s.elem_def);
    vv[i] = d == s.max_def;
}

__global__ void pq_levels_scatter_kernel(const uint8_t* __restrict__ rep, const uint8_t* __restrict__ def, const int64_t* __restrict__ re,
                                         const int32_t* __restrict__ vv, int64_t n, int64_t n_rows, PqListShape s, int32_t* __restrict__ offsets,
                                         uint32_t* __restrict__ validity, int32_t* __restrict__ elem_idx, const int64_t* __restrict__ counts) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i == 0) offsets[n_rows] = (int32_t)counts[1];
    if (i >= n) return;
    const int64_t x = re[i];
    const int64_t row = x >> 32;
    const int32_t e = (int32_t)(x & 0xffffffffll);
    const int d = def[i];
    if (rep[i] == 0 && row < n_rows) {
        offsets[row] = e;
        if (validity && d >= s.list_def) atomicOr(&validity[row >> 5], 1u << (row & 31));
    }
    if (d >= s.elem_def) elem_idx[e] = d == s.max_def ? vv[i] : -1;
}

__global__ void pq_levels_totals_kernel(int64_t* counts) {   // the scans' totals: re = rows << 32 | elements, vv = values
    const int64_t re = counts[0];
    counts[0] = re >> 32;
    counts[1] = re & 0xffffffffll;
    counts[2] = (int64_t)((const int32_t*)(counts + 2))[0];
}

void pq_list_levels(Ctx& ctx, const PqLevelPage* pages, int n_pages, int64_t n_slots, int64_t n_rows, const PqListShape& s, int32_t* offsets,
                    uint32_t* validity, int32_t* elem_idx, int64_t* counts) {
    ProfScope ps(ctx, "pq_list_levels");
    AURON_CHECK(n_slots >= 0 && n_slots <= (int64_t)INT32_MAX, "parquet list levels: too many slots in one batch");
    CUDA_OK(cudaMemsetAsync(counts, 0, 4 * sizeof(int64_t), ctx.stream));
    if (n_slots == 0) {
        CUDA_OK(cudaMemsetAsync(offsets, 0, (size_t)(n_rows + 1) * 4, ctx.stream));
        return;
    }
    Buf rep = dalloc(ctx, (size_t)n_slots), def = dalloc(ctx, (size_t)n_slots);
    Buf re = dalloc(ctx, (size_t)n_slots * 8), vv = dalloc(ctx, (size_t)n_slots * 4);
    if (n_pages > 0) {
        const int64_t threads = 2 * (int64_t)n_pages * 32;
        pq_levels_expand_kernel<<<(unsigned)((threads + LV_WARPS * 32 - 1) / (LV_WARPS * 32)), LV_WARPS * 32, 0, ctx.stream>>>(pages, n_pages, s, P<uint8_t>(rep),
                                                                                                                                P<uint8_t>(def), counts);
        LAUNCH_CHECK(ctx);
    }
    const unsigned grid = (unsigned)((n_slots + 255) / 256);
    pq_levels_flags_kernel<<<grid, 256, 0, ctx.stream>>>(P<uint8_t>(rep), P<uint8_t>(def), n_slots, s, P<int64_t>(re), P<int32_t>(vv));
    LAUNCH_CHECK(ctx);
    exclusive_scan_i64(ctx, P<int64_t>(re), P<int64_t>(re), n_slots, counts);
    exclusive_scan_i32(ctx, P<int32_t>(vv), P<int32_t>(vv), n_slots, (int32_t*)(counts + 2));
    pq_levels_totals_kernel<<<1, 1, 0, ctx.stream>>>(counts);
    LAUNCH_CHECK(ctx);
    pq_levels_scatter_kernel<<<grid, 256, 0, ctx.stream>>>(P<uint8_t>(rep), P<uint8_t>(def), P<int64_t>(re), P<int32_t>(vv), n_slots, n_rows, s, offsets,
                                                           validity, elem_idx, counts);
    LAUNCH_CHECK(ctx);
}

__global__ void pq_compose_index_kernel(int32_t* __restrict__ idx, const int32_t* __restrict__ value_idx, int64_t n) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int32_t v = idx[i];
    idx[i] = v < 0 ? -1 : value_idx[v];
}

void pq_compose_index(Ctx& ctx, int32_t* idx, const int32_t* value_idx, int64_t n) {
    if (n <= 0) return;
    ProfScope ps(ctx, "pq_compose_index");
    pq_compose_index_kernel<<<(unsigned)((n + 255) / 256), 256, 0, ctx.stream>>>(idx, value_idx, n);
    LAUNCH_CHECK(ctx);
}

}  // namespace auron
