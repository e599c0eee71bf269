// k_parquet.cu -- Parquet page decode on device (row P1 of SURVEY.md section 8a): RLE / bit-packed hybrid
// definition levels and dictionary indices, dictionary gather, PLAIN fixed-width values, PLAIN byte arrays,
// NULL scatter from definition levels and the INT32/INT64 -> Decimal128 widening of AuronSchemaAdapter
// (datafusion-ext-plans/src/scan/mod.rs:103-160).  The reference does this on the CPU inside the third-party
// `parquet` crate (call site parquet_exec.rs:175-197).
//
// One warp decodes one data page in a single pass: the hybrid streams are parsed run by run (the run header
// is read redundantly by all lanes = one broadcast load), each 32-row chunk turns its definition levels into
// a validity word with a ballot, the ranks of the valid lanes (popc of the lower-lane mask) index the value
// stream, values are fetched from the dictionary (L2-resident) or the PLAIN section and written once,
// converted to the Arrow type.  Pages of all row groups of a batch are decoded by one launch per column.
// HBM-bound: algorithmic bytes = encoded page bytes in + Arrow bytes out (+1/8 B validity).
#include "device_utils.cuh"
#include "kernels.h"
#include "parquet_dev.h"
#include "parquet_hybrid.cuh"

namespace auron {

#define LAUNCH_CHECK(ctx)            \
    do {                             \
        CUDA_OK(cudaGetLastError()); \
        launch_count(ctx);           \
    } while (0)

// FIXED_LEN_BYTE_ARRAY decimal: n big-endian two's complement bytes -> decimal128 (hi:lo)
__device__ __forceinline__ void load_flba(const uint8_t* src, int n, uint64_t& lo, uint64_t& hi) {
    hi = (src[0] & 0x80) ? ~0ull : 0ull;
    lo = hi;
    for (int i = 0; i < n; i++) {
        hi = (hi << 8) | (lo >> 56);
        lo = (lo << 8) | src[i];
    }
}
__device__ __forceinline__ void store_i128(const PqColumnArgs& a, int64_t row, uint64_t lo, uint64_t hi) {
    ((uint64_t*)a.out)[2 * row] = lo;
    ((uint64_t*)a.out)[2 * row + 1] = hi;
}
// The conversions that scale (PQ_CV_TS_MUL, PQ_CV_TS_DIV, PQ_CV_DEC).
// False when the product leaves int64 (a zero is stored and the row must be NULL).
__device__ __forceinline__ bool store_scaled(const PqColumnArgs& a, const uint8_t* src, int64_t row) {
    if (a.conv != PQ_CV_DEC) {   // INT64 timestamps
        const int64_t x = (int64_t)ld_u64_unaligned(src), m = (int64_t)a.conv_mul;
        if (a.conv == PQ_CV_TS_DIV) {
            ((int64_t*)a.out)[row] = x / m;   // truncating, as arrow divides
            return true;
        }
        const bool ok = x <= INT64_MAX / m && x >= INT64_MIN / m;   // arrow's safe cast: NULL where the product leaves int64
        ((int64_t*)a.out)[row] = ok ? x * m : 0;
        return ok;
    }
    // decimal on INT32 / INT64 / FLBA x 10^k; the host admits only targets wide enough for the product
    uint64_t lo, hi;
    if (a.phys_type == 7) load_flba(src, a.type_length, lo, hi);
    else {
        const int64_t x = a.phys_type == 1 ? (int64_t)(int32_t)ld_u32_unaligned(src) : (int64_t)ld_u64_unaligned(src);
        lo = (uint64_t)x;
        hi = x < 0 ? ~0ull : 0ull;
    }
    const unsigned __int128 r = (((unsigned __int128)hi << 64) | lo) * (((unsigned __int128)a.conv_mul_hi << 64) | a.conv_mul);   // two's complement: the low 128 bits
    store_i128(a, row, (uint64_t)r, (uint64_t)(r >> 64));
    return true;
}
// Converts the physical value at src (little-endian INT32/INT64/FLOAT/DOUBLE, big-endian FLBA) as a.conv says and stores it at `row`.
// False when the value has no representation in the table's type (PQ_CV_TS_MUL overflow): a zero is stored and the row must be NULL.
__device__ __forceinline__ bool store_converted(const PqColumnArgs& a, const uint8_t* src, int64_t row) {
    if (a.conv >= PQ_CV_TS_MUL) return store_scaled(a, src, row);
    switch (a.phys_type) {
        case 1: case 4: {   // INT32 / FLOAT
            const uint32_t v = ld_u32_unaligned(src);
            const int64_t x = a.conv == PQ_CV_ZEXT ? (int64_t)v : (int64_t)(int32_t)v;
            if (a.conv == PQ_CV_I32_F64) ((double*)a.out)[row] = (double)(int32_t)v;
            else if (a.conv == PQ_CV_F32_F64) ((double*)a.out)[row] = (double)__int_as_float((int)v);
            else switch (a.out_width) {   // PQ_CV_COPY (narrowing stores only where the annotation says the value fits), SEXT, ZEXT
                case 1: ((int8_t*)a.out)[row] = (int8_t)x; break;
                case 2: ((int16_t*)a.out)[row] = (int16_t)x; break;
                case 4: ((uint32_t*)a.out)[row] = v; break;
                case 8: ((int64_t*)a.out)[row] = x; break;
                case 16: store_i128(a, row, (uint64_t)x, x < 0 ? ~0ull : 0ull); break;   // scan/mod.rs:131-136: value copy, no rescale
            }
            return true;
        }
        case 2: case 5: {   // INT64 / DOUBLE
            const uint64_t v = ld_u64_unaligned(src);
            if (a.out_width == 16) store_i128(a, row, v, (int64_t)v < 0 ? ~0ull : 0ull);
            else ((uint64_t*)a.out)[row] = v;
            return true;
        }
        case 3: {   // INT96 timestamp: 8 bytes nanoseconds of the day (LE) + 4 bytes Julian day (LE) -> the output column's unit
            const int64_t nanos = (int64_t)ld_u64_unaligned(src);
            const int64_t days = (int64_t)(int32_t)ld_u32_unaligned(src + 8) - 2440588;   // Julian day of 1970-01-01
            int64_t v;
            switch (a.out_unit) {
                case 0: v = days * 86400ll + nanos / 1000000000ll; break;
                case 1: v = days * 86400000ll + nanos / 1000000ll; break;
                case 3: v = days * 86400000000000ll + nanos; break;
                default: v = days * 86400000000ll + nanos / 1000ll; break;
            }
            ((int64_t*)a.out)[row] = v;
            return true;
        }
        case 7: {   // FIXED_LEN_BYTE_ARRAY decimal at its own scale (the host admits decimal128 targets only)
            uint64_t lo, hi;
            load_flba(src, a.type_length, lo, hi);
            store_i128(a, row, lo, hi);
            return true;
        }
    }
    return true;
}
__device__ __forceinline__ void store_zero(const PqColumnArgs& a, int64_t row) {
    switch (a.out_width) {
        case 1: ((uint8_t*)a.out)[row] = 0; break;
        case 2: ((uint16_t*)a.out)[row] = 0; break;
        case 4: ((uint32_t*)a.out)[row] = 0; break;
        case 8: ((uint64_t*)a.out)[row] = 0; break;
        case 16: ((uint64_t*)a.out)[2 * row] = 0; ((uint64_t*)a.out)[2 * row + 1] = 0; break;
    }
}

struct PqLaunch {
    PqColumnArgs a;
    const int32_t* tile_base;   // [n_pages + 1]
    PqTile* tiles;
    uint32_t* tile_valid;       // [n_tiles][32] tile-local validity words written by the scout (nullable columns)
};

// Definition levels of one tile -> 32 validity words (lane L returns word L, bit i of the tile = row 32L+i).
// Writers emit very short level runs (a NULL every ~30 rows splits the stream into ~60 runs per 1024 rows), so a
// warp-wide step per run wastes 31 lanes.  Instead lane 0 walks up to 32 run headers (the only serial part) and drops
// a descriptor per run into shared memory; then every lane materialises one run into the tile bitmap in parallel.
// `def` is only meaningful in lane 0 afterwards.
__device__ __forceinline__ uint32_t extract_bits(const uint8_t* base, int64_t bitpos, int bw);
struct DefRun {
    int32_t dst, t;       // first tile-local row, row count
    int32_t srcbit;       // bit offset from the stream base (bit-packed runs)
    int32_t kind;         // 0 bit-packed, 1 RLE ones, 2 RLE zeros
};
__device__ __forceinline__ uint32_t def_tile_words(Hybrid& def, const uint8_t* def_base, int m, unsigned lane, uint32_t* bm /*[32] smem*/,
                                                   DefRun* runs /*[32] smem*/) {
    bm[lane] = 0;
    int filled = 0;
    __syncwarp();
    while (filled < m) {
        int nr = 0;
        if (lane == 0) {
            int f = filled;
            while (nr < 32 && f < m) {
                if (def.run_remaining == 0) def.next_run();
                int t = min(m - f, def.run_remaining);
                DefRun r;
                r.dst = f;
                r.t = t;
                r.kind = def.is_rle ? ((def.rle_value & 1) ? 1 : 2) : 0;
                r.srcbit = def.is_rle ? 0 : (int32_t)((def.bp_base - def_base) * 8 + def.bp_consumed);
                runs[nr++] = r;
                def.run_remaining -= t;
                if (!def.is_rle) def.bp_consumed += t;
                f += t;
            }
            filled = f;
        }
        nr = __shfl_sync(FULL_MASK, nr, 0);
        filled = __shfl_sync(FULL_MASK, filled, 0);
        __syncwarp();
        if ((int)lane < nr) {
            DefRun r = runs[lane];
            if (r.kind != 2) {
                int done = 0;
                while (done < r.t) {   // at most 32 bits per step, aligned to the destination word
                    int d = r.dst + done;
                    int take = min(r.t - done, 32 - (d & 31));
                    uint32_t bits = r.kind == 1 ? 0xffffffffu : extract_bits(def_base, (int64_t)r.srcbit + done, 32);
                    if (take < 32) bits &= (1u << take) - 1u;
                    if (bits) atomicOr(&bm[d >> 5], bits << (d & 31));
                    done += take;
                }
            }
        }
        __syncwarp();
    }
    return bm[lane];
}

// pass 1: one warp per page walks the run headers and checkpoints both streams every PQ_TILE rows
__device__ __forceinline__ void scout_page(const PqLaunch& L, int page_id, int (*s_exit_w)[33], int* s_entry_w) {
    const PqColumnArgs& a = L.a;
    const unsigned lane = lane_id();
    const PqPage pg = a.pages[page_id];
    Hybrid def, idx;
    const bool has_def = a.max_def > 0 && pg.def_len > 0;
    if (has_def) def.init(pg.def_ptr, pg.def_ptr + pg.def_len, 1);
    const bool dict = pg.encoding == 2 || pg.encoding == 8;
    const bool bool_rle = a.phys_type == 0 && pg.encoding == 3;
    const uint8_t* vals = pg.val_ptr;
    const uint8_t* idx_base = vals;
    if (dict) {
        idx_base = vals + 1;
        idx.init(idx_base, vals + pg.val_len, pg.val_len > 0 ? vals[0] : 0);
    } else if (bool_rle) {
        idx_base = vals + 4;
        idx.init(idx_base, vals + pg.val_len, 1);
    } else idx.init(vals, vals, 0);
    const int rows = pg.num_values;
    int64_t v0 = 0;
    const uint8_t* pf_idx = idx_base;
    int tile = L.tile_base[page_id];
    if (has_def) {
        lvl_page_bits(pg.def_ptr, pg.def_len, rows, lane, L.tile_valid + (int64_t)tile * 32, s_exit_w, s_entry_w);
        __threadfence();   // the bits were ORed into global memory by other lanes; they are read back below
        __syncwarp();
    }
    for (int r = 0; r < rows; r += PQ_TILE, tile++) {
        int m = min(PQ_TILE, rows - r);
        if (lane == 0) {
            PqTile t;
            t.page = page_id;
            t.row0 = r;
            t.n = m;
            t.pad = 0;
            t.v0 = v0;
            t.def = has_def ? hybrid_save(def, pg.def_ptr) : HybridCk{0, 0, 0, 0, 0, 1};
            t.idx = (dict || bool_rle) ? hybrid_save(idx, idx_base) : HybridCk{0, 0, 0, 0, 0, 1};
            L.tiles[tile] = t;
        }
        // the header walk is a pointer chase: pull the next 8 KB of both streams into L1 ahead of it (32 lines per shot)
        if (dict || bool_rle) {
            const uint8_t* send = vals + pg.val_len;
            while (pf_idx < idx.p + 8192 && pf_idx < send) {
                const uint8_t* q = pf_idx + 128 * lane;
                if (q < send) asm volatile("prefetch.global.L1 [%0];" ::"l"(q));
                pf_idx += 4096;
            }
        }
        int nvalid = m;
        if (has_def) {
            uint32_t w = L.tile_valid[(int64_t)tile * 32 + lane];   // written by lvl_page_bits above
            int c = __popc(w);
#pragma unroll
            for (int d = 16; d; d >>= 1) c += __shfl_xor_sync(FULL_MASK, c, d);
            nvalid = c;
        } else if (a.max_def > 0 && pg.all_null) nvalid = 0;
        if (dict || bool_rle) hybrid_skip(idx, nvalid);
        v0 += nvalid;
    }
}
__global__ void __launch_bounds__(PQ_WARPS * 32) pq_scout_kernel(PqLaunch L) {
    __shared__ int s_exit[PQ_WARPS][32][33];
    __shared__ int s_entry[PQ_WARPS][33];
    const int wid = threadIdx.x >> 5;
    const int page_id = blockIdx.x * PQ_WARPS + wid;
    if (page_id >= L.a.n_pages) return;
    scout_page(L, page_id, s_exit[wid], s_entry[wid]);
}
// The scout of one column is a few thousand warps (one per page): too few to fill 132 SMs.  All columns of a batch are
// scouted by ONE launch: warp g serves page g - page_base[c] of column c.
__global__ void __launch_bounds__(PQ_WARPS * 32) pq_scout_multi_kernel(const PqLaunch* __restrict__ Ls, const int32_t* __restrict__ page_base, int ncols) {
    __shared__ int s_exit[PQ_WARPS][32][33];
    __shared__ int s_entry[PQ_WARPS][33];
    const int wid = threadIdx.x >> 5;
    const int g = blockIdx.x * PQ_WARPS + wid;
    if (g >= page_base[ncols]) return;
    int c = 0;
    while (c + 1 < ncols && g >= page_base[c + 1]) c++;
    scout_page(Ls[c], g - page_base[c], s_exit[wid], s_entry[wid]);
}

// pass 2: one warp per tile
__global__ void __launch_bounds__(PQ_WARPS * 32) pq_decode_tiles_kernel(PqLaunch L, int n_tiles) {
    const PqColumnArgs& a = L.a;
    int tile_id = blockIdx.x * PQ_WARPS + (threadIdx.x >> 5);
    if (tile_id >= n_tiles) return;
    const unsigned lane = lane_id();
    const PqTile tl = L.tiles[tile_id];
    const PqPage pg = a.pages[tl.page];
    Hybrid def, idx;
    const bool has_def = a.max_def > 0 && pg.def_len > 0;
    if (has_def) hybrid_restore(def, tl.def, pg.def_ptr, pg.def_ptr + pg.def_len, 1);
    const bool dict = pg.encoding == 2 || pg.encoding == 8;
    const uint8_t* vals = pg.val_ptr;
    const bool bool_rle = a.phys_type == 0 && pg.encoding == 3;   // RLE booleans (data page v2 writers): u32 length + hybrid, bit width 1
    if (dict) hybrid_restore(idx, tl.idx, vals + 1, vals + pg.val_len, pg.val_len > 0 ? vals[0] : 0);
    else if (bool_rle) hybrid_restore(idx, tl.idx, vals + 4, vals + pg.val_len, 1);
    const PqDict dd = dict ? a.dicts[pg.dict_id] : PqDict{nullptr, 0, 0};
    const int w = a.phys_width;
    int done = tl.row0;
    int64_t value_base = tl.v0;
    const int rows = tl.row0 + tl.n;
    while (done < rows) {
        int64_t out_row = (int64_t)pg.row_start + done;
        int m = min(rows - done, 32 - (int)(out_row & 31));
        bool active = (int)lane < m;
        bool valid = active;
        if (has_def) {   // the scout already turned the definition levels into tile-local validity words
            int il = done - tl.row0 + (int)lane;
            valid = active && ((L.tile_valid[(int64_t)tile_id * 32 + (il >> 5)] >> (il & 31)) & 1u);
        } else if (a.max_def > 0 && pg.all_null) valid = false;
        uint32_t mask = __ballot_sync(FULL_MASK, valid);
        int rank = __popc(mask & lanemask_lt());
        int nvalid = __popc(mask);
        int64_t ordinal = value_base + rank;
        uint32_t myidx = 0;
        if (dict) {
            uint32_t got = nvalid ? idx.read_batch(nvalid, lane) : 0;
            myidx = __shfl_sync(FULL_MASK, got, rank & 31);
            if (myidx >= (uint32_t)dd.num_values) myidx = 0;   // corrupt index guard
        }
        int64_t row = out_row + lane;
        if (active) {
            if (a.mode == PQ_MODE_INDEX) {
                // strings: position in the chunk's value table (dictionary entries first, then PLAIN values)
                a.out_idx[row] = valid ? (dict ? dd.value_base + (int32_t)myidx : pg.plain_value_base + (int32_t)ordinal) : -1;
            } else if (a.phys_type == 0) {
                // BOOLEAN PLAIN = LSB-first bit-packed without run headers; handled below through a ballot
            } else if (valid) {
                const uint8_t* src = dict ? dd.data + (int64_t)myidx * w : vals + ordinal * w;
                store_converted(a, src, row);
            } else {
                store_zero(a, row);
            }
        }
        if (a.phys_type == 0 && a.mode != PQ_MODE_INDEX) {
            bool bit = false;
            if (bool_rle) {
                uint32_t got = nvalid ? idx.read_batch(nvalid, lane) : 0;
                uint32_t mine = __shfl_sync(FULL_MASK, got, rank & 31);   // every lane takes part (no short-circuit around the shuffle)
                bit = valid && (mine & 1);
            } else if (valid) bit = (vals[ordinal >> 3] >> (ordinal & 7)) & 1;
            uint32_t bits = __ballot_sync(FULL_MASK, bit) << (out_row & 31);
            if (lane == 0 && bits) atomicOr(&((uint32_t*)a.out)[out_row >> 5], bits);
        }
        if (a.out_valid && lane == 0) {
            uint32_t bits = mask << (out_row & 31);
            if (m == 32) a.out_valid[out_row >> 5] = bits;
            else if (bits) atomicOr(&a.out_valid[out_row >> 5], bits);
        }
        done += m;
        value_base += nvalid;
    }
}

// pass 2 (fast path): one warp per tile, three phases --
//   1. the tile's definition levels become 32 validity words (one per lane) straight from the hybrid runs,
//      a warp scan of their popcounts gives every word its rank base;
//   2. the tile's dictionary indices are unpacked into shared memory, lanes striding over each run;
//   3. 32 rows per iteration: rank = base + popc(lower lanes), dictionary / PLAIN load, typed store.
// Booleans keep the generic kernel above.
__global__ void __launch_bounds__(PQ_WARPS * 32) pq_decode_tiles_fast_kernel(PqLaunch L, int n_tiles) {
    __shared__ uint32_t s_vals[PQ_WARPS][PQ_TILE];
    __shared__ uint32_t s_w[PQ_WARPS][33];
    __shared__ int32_t s_pref[PQ_WARPS][32];
    const PqColumnArgs& a = L.a;
    const int wid = threadIdx.x >> 5;
    int tile_id = blockIdx.x * PQ_WARPS + wid;
    if (tile_id >= n_tiles) return;
    const unsigned lane = lane_id();
    const PqTile tl = L.tiles[tile_id];
    const PqPage pg = a.pages[tl.page];
    const int n = tl.n;
    const bool has_def = a.max_def > 0 && pg.def_len > 0;
    const bool dict = pg.encoding == 2 || pg.encoding == 8;
    const uint8_t* vals = pg.val_ptr;
    // ---- 1. validity words
    uint32_t w = 0;
    if (has_def) {
        w = L.tile_valid[(int64_t)tile_id * 32 + lane];   // decoded once, by the scout
    } else if (!(a.max_def > 0 && pg.all_null)) {
        int cnt = n - 32 * (int)lane;
        w = cnt >= 32 ? 0xffffffffu : (cnt > 0 ? (1u << cnt) - 1u : 0u);
    }
    int pc = __popc(w), inc = pc;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        int t = __shfl_up_sync(FULL_MASK, inc, d);
        if ((int)lane >= d) inc += t;
    }
    const int prefix = inc - pc;
    const int nv = __shfl_sync(FULL_MASK, inc, 31);
    // ---- 2. dictionary indices of the tile's non-null values
    if (dict) {
        Hybrid idx;
        const int bw = pg.val_len > 0 ? vals[0] : 0;
        hybrid_restore(idx, tl.idx, vals + 1, vals + pg.val_len, bw);
        int pos = 0;
        while (pos < nv) {
            if (idx.run_remaining == 0) idx.next_run();
            int t = min(nv - pos, idx.run_remaining);
            if (idx.is_rle) {
                for (int k = lane; k < t; k += 32) s_vals[wid][pos + k] = idx.rle_value;
            } else {
                // lane L unpacks values L, L+32, ...: 32 values are exactly `bw` 32-bit words, so the word pointer
                // advances by bw per step and the sub-word shift is a per-lane constant of the run
                const int64_t bit0 = (int64_t)(idx.bp_consumed + (int)lane) * bw;
                const uintptr_t qa = (uintptr_t)(idx.bp_base + (bit0 >> 3));
                const uint32_t* wp = (const uint32_t*)(qa & ~(uintptr_t)3);
                const unsigned sh = (unsigned)(qa & 3) * 8 + (unsigned)(bit0 & 7);
                const uint32_t vmask = bw >= 32 ? 0xffffffffu : ((1u << bw) - 1u);
                uint32_t* dst = &s_vals[wid][pos + (int)lane];
                int k = lane;
                for (; k + 96 < t; k += 128) {   // 4 independent unpacks in flight per lane
                    uint32_t v[4];
#pragma unroll
                    for (int u = 0; u < 4; u++) v[u] = __funnelshift_r(wp[u * bw], wp[u * bw + 1], sh) & vmask;
#pragma unroll
                    for (int u = 0; u < 4; u++) dst[32 * u] = v[u];
                    wp += 4 * bw;
                    dst += 128;
                }
                for (; k < t; k += 32) {
                    *dst = __funnelshift_r(wp[0], wp[1], sh) & vmask;
                    wp += bw;
                    dst += 32;
                }
            }
            pos += t;
            idx.run_remaining -= t;
            if (!idx.is_rle) idx.bp_consumed += t;
        }
    }
    s_w[wid][lane] = w;
    if (lane == 0) s_w[wid][32] = 0;
    __syncwarp();
    // ---- 3. rows
    const PqDict dd = dict ? a.dicts[pg.dict_id] : PqDict{nullptr, 0, 0};
    const int width = a.phys_width;
    const int64_t out0 = (int64_t)pg.row_start + tl.row0;
    s_pref[wid][lane] = prefix;
    __syncwarp();
    // specialised inner loops for the common fixed-width cases: no per-row type switches, rank base from shared memory
    // (copies and sign extensions only: every other conversion goes through store_converted)
    const bool same4 = a.mode == PQ_MODE_VALUES && a.conv == PQ_CV_COPY && width == 4 && a.out_width == 4 && (a.phys_type == 1 || a.phys_type == 4);
    const bool same8 = a.mode == PQ_MODE_VALUES && a.conv == PQ_CV_COPY && width == 8 && a.out_width == 8 && (a.phys_type == 2 || a.phys_type == 5);
    const bool widen = a.mode == PQ_MODE_VALUES && a.conv == PQ_CV_SEXT && a.phys_type == 1 && a.out_width == 8;
    if (same4 || widen) {
        // value r (dictionary index, or PLAIN ordinal within the tile) is the 32-bit word at base + 4r; the base is
        // not 4-byte aligned in general (page payloads sit at arbitrary file offsets): one uniform funnel shift
        const uint32_t ndict = (uint32_t)dd.num_values;
        const unsigned lt = lanemask_lt();
        const uintptr_t ba = (uintptr_t)(dict ? dd.data : vals + tl.v0 * 4);
        const uint32_t* bw32 = (const uint32_t*)(ba & ~(uintptr_t)3);
        const unsigned bsh = (unsigned)(ba & 3) * 8;
        uint32_t* out32 = (uint32_t*)a.out + out0 + lane;
        int64_t* out64 = (int64_t*)a.out + out0 + lane;
        const int nfull = n - (int)lane;   // row 32j + lane exists iff 32j < nfull
        // 4 row-groups (128 rows) per iteration: the four gathers are issued back to back before any store
        for (int j0 = 0; j0 * 32 < n; j0 += 4) {
            uint32_t e[4], v[4];
            bool valid[4];
#pragma unroll
            for (int u = 0; u < 4; u++) {
                const int j = j0 + u;   // < 32 (n <= 1024)
                const uint32_t wj = s_w[wid][j];
                const int rank = s_pref[wid][j] + __popc(wj & lt);
                valid[u] = (wj >> lane) & 1u;   // validity words carry no bits past the tile's rows
                e[u] = 0;
                if (valid[u]) {
                    e[u] = (uint32_t)rank;
                    if (dict) {
                        const uint32_t di = s_vals[wid][rank];
                        e[u] = di < ndict ? di : 0;   // corrupt index guard
                    }
                }
            }
            if (bsh == 0) {
#pragma unroll
                for (int u = 0; u < 4; u++) v[u] = valid[u] ? bw32[e[u]] : 0u;
            } else {
#pragma unroll
                for (int u = 0; u < 4; u++) v[u] = valid[u] ? __funnelshift_r(bw32[e[u]], bw32[e[u] + 1], bsh) : 0u;
            }
#pragma unroll
            for (int u = 0; u < 4; u++)
                if (32 * (j0 + u) < nfull) {
                    if (same4) out32[32 * (j0 + u)] = v[u];
                    else out64[32 * (j0 + u)] = (int64_t)(int32_t)v[u];
                }
        }
    } else if (same8) {
        const uint32_t ndict = (uint32_t)dd.num_values;
        const unsigned lt = lanemask_lt();
        for (int j0 = 0; j0 * 32 < n; j0 += 4) {
            const uint8_t* src[4];
            bool valid[4];
#pragma unroll
            for (int u = 0; u < 4; u++) {
                const int j = j0 + u;
                const uint32_t wj = s_w[wid][j];
                const int rank = s_pref[wid][j] + __popc(wj & lt);
                valid[u] = (wj >> lane) & 1u;
                src[u] = vals;
                if (valid[u]) {
                    if (dict) {
                        uint32_t di = s_vals[wid][rank];
                        di = di < ndict ? di : 0;
                        src[u] = dd.data + (int64_t)di * 8;
                    } else src[u] = vals + (tl.v0 + rank) * 8;
                }
            }
            uint64_t v[4];
#pragma unroll
            for (int u = 0; u < 4; u++) v[u] = valid[u] ? ld_u64_unaligned(src[u]) : 0ull;
#pragma unroll
            for (int u = 0; u < 4; u++)
                if (32 * (j0 + u) + (int)lane < n) ((uint64_t*)a.out)[out0 + 32 * (j0 + u) + lane] = v[u];
        }
    } else
    {
        for (int j = 0; j * 32 < n; j++) {
            int i = 32 * j + (int)lane;
            bool active = i < n;
            uint32_t wj = s_w[wid][j];
            int pj = __shfl_sync(FULL_MASK, prefix, j);
            bool valid = active && ((wj >> lane) & 1u);
            int rank = pj + __popc(wj & lanemask_lt());
            int64_t row = out0 + i;
            bool ok = true;
            if (active && a.mode == PQ_MODE_INDEX) {
                uint32_t di = dict ? s_vals[wid][rank] : 0;
                if (di >= (uint32_t)dd.num_values) di = 0;
                a.out_idx[row] = valid ? (dict ? dd.value_base + (int32_t)di : pg.plain_value_base + (int32_t)(tl.v0 + rank)) : -1;
            } else if (valid) {
                const uint8_t* src;
                if (dict) {
                    uint32_t di = s_vals[wid][rank];
                    if (di >= (uint32_t)dd.num_values) di = 0;   // corrupt index guard
                    src = dd.data + (int64_t)di * width;
                } else src = vals + (tl.v0 + rank) * width;
                ok = store_converted(a, src, row);
            } else if (active) {
                store_zero(a, row);
            }
            if (a.conv == PQ_CV_TS_MUL) {   // values the conversion cannot represent become NULL (the column has a validity buffer)
                const uint32_t bad = __ballot_sync(FULL_MASK, !ok);
                if (lane == 0 && bad) s_w[wid][j] = wj & ~bad;
            }
        }
        __syncwarp();
    }
    // ---- 4. validity words of the output (tile rows are not 32-aligned in general)
    if (a.out_valid) {
        const int sh = (int)(out0 & 31);
        const int64_t q0 = out0 >> 5;
        const int nwords = (sh + n + 31) / 32;
        for (int q = lane; q < nwords; q += 32) {
            uint32_t cur = q < 32 ? s_w[wid][q] : 0u, prev = q > 0 ? s_w[wid][q - 1] : 0u;
            uint32_t bits = sh ? ((cur << sh) | (prev >> (32 - sh))) : cur;
            bool full = (q > 0 || sh == 0) && ((q + 1) * 32 <= sh + n);
            if (full) a.out_valid[q0 + q] = bits;
            else if (bits) atomicOr(&a.out_valid[q0 + q], bits);
        }
    }
}

// ---------------------------------------------------------------------------------------------- DELTA_BINARY_PACKED -> PLAIN
// Parquet's delta encoding (Encodings.md, "Delta Encoding"): header = block size, miniblocks per block, total count (ULEB128), first
// value (zigzag ULEB128); every block = min delta (zigzag ULEB128), one bit-width byte per miniblock, then the miniblocks, each
// (block size / miniblocks) deltas bit-packed LSB first.  value[i] = value[i - 1] + min_delta + packed[i] in wrapping arithmetic.
// One warp per page walks the blocks in order (a block's position depends on the widths of the one before); inside a miniblock
// the lanes unpack 32 deltas at a time and a warp scan turns them into values.
__device__ __forceinline__ bool dl_varint(const uint8_t* p, int64_t n, int64_t& pos, uint64_t& v) {
    v = 0;
    for (int shift = 0; shift < 70; shift += 7) {
        if (pos >= n) return false;
        const uint8_t b = p[pos++];
        v |= (uint64_t)(b & 0x7f) << shift;
        if (!(b & 0x80)) return true;
    }
    return false;
}
__device__ __forceinline__ int64_t dl_zigzag(uint64_t v) { return (int64_t)(v >> 1) ^ -(int64_t)(v & 1); }
__global__ void __launch_bounds__(128) pq_delta_to_plain_kernel(PqPage* __restrict__ pages, int n_pages, uint8_t* __restrict__ scratch, int width, int32_t* __restrict__ status) {
    const int pi = blockIdx.x * 4 + (threadIdx.x >> 5);
    if (pi >= n_pages) return;
    const unsigned lane = threadIdx.x & 31;
    PqPage pg = pages[pi];
    if (pg.delta_dst16 == 0) return;
    uint8_t* dst = scratch + 16 * (int64_t)(pg.delta_dst16 - 1);
    const uint8_t* p = pg.val_ptr;
    const int64_t n = pg.val_len;
    int64_t pos = 0;
    uint64_t block_size = 0, n_mini = 0, total = 0, fv = 0;
    bool ok = dl_varint(p, n, pos, block_size) && dl_varint(p, n, pos, n_mini) && dl_varint(p, n, pos, total) && dl_varint(p, n, pos, fv);
    ok = ok && n_mini > 0 && n_mini <= 512 && block_size > 0 && block_size <= (1u << 20) && block_size % n_mini == 0 && (block_size / n_mini) % 32 == 0 &&
         total <= (uint64_t)pg.num_values;
    const int per_mini = ok ? (int)(block_size / n_mini) : 32;
    int64_t last = dl_zigzag(fv);   // value before the next delta
    int64_t done = 0;
    if (ok && total > 0) {
        if (lane == 0) {
            if (width == 4) ((int32_t*)dst)[0] = (int32_t)last;
            else ((int64_t*)dst)[0] = last;
        }
        done = 1;
    }
    while (ok && done < (int64_t)total) {
        uint64_t md = 0;
        if (!dl_varint(p, n, pos, md) || pos + (int64_t)n_mini > n) {
            ok = false;
            break;
        }
        const int64_t min_delta = dl_zigzag(md);
        const uint8_t* widths = p + pos;
        pos += (int64_t)n_mini;
        for (int m = 0; m < (int)n_mini && done < (int64_t)total; m++) {
            const int bw = widths[m];
            const int64_t bytes = (int64_t)per_mini * bw / 8;
            if (bw > 64 || pos + bytes > n) {
                ok = false;
                break;
            }
            for (int g = 0; g < per_mini && done < (int64_t)total; g += 32) {
                uint64_t d = 0;
                if (bw) {   // packed value g + lane: bits [(g + lane) * bw, +bw) of the miniblock
                    const int64_t bit = (int64_t)(g + (int)lane) * bw;
                    const uint8_t* q = p + pos + (bit >> 3);
                    const int sh = (int)(bit & 7), nb = (sh + bw + 7) >> 3;   // <= 9 bytes
                    uint64_t lo = 0;
                    for (int k = 0; k < nb && k < 8; k++) lo |= (uint64_t)q[k] << (8 * k);
                    d = lo >> sh;
                    if (nb > 8) d |= (uint64_t)q[8] << (64 - sh);
                    if (bw < 64) d &= (1ull << bw) - 1ull;
                }
                int64_t x = (int64_t)((uint64_t)min_delta + d);   // this lane's delta; inclusive scan -> offset from `last`
#pragma unroll
                for (int o = 1; o < 32; o <<= 1) {
                    const int64_t y = __shfl_up_sync(FULL_MASK, x, o);
                    if ((int)lane >= o) x = (int64_t)((uint64_t)x + (uint64_t)y);
                }
                const int64_t v = (int64_t)((uint64_t)last + (uint64_t)x);
                if (done + (int64_t)lane < (int64_t)total) {
                    if (width == 4) ((int32_t*)dst)[done + lane] = (int32_t)v;
                    else ((int64_t*)dst)[done + lane] = v;
                }
                last = __shfl_sync(FULL_MASK, v, 31);
                done += 32;
            }
            pos += bytes;
        }
    }
    if (lane == 0) {
        if (!ok) atomicCAS(status, 0, 0x40000000 + pi);
        pg.val_ptr = dst;
        pg.val_len = ok ? (int32_t)min((uint64_t)INT32_MAX, total * (uint64_t)width) : 0;
        pg.delta_dst16 = 0;
        pages[pi] = pg;
    }
}
void pq_delta_to_plain(Ctx& ctx, PqPage* pages, int n, uint8_t* scratch, int width, int32_t* status) {
    if (n <= 0) return;
    ProfScope ps(ctx, "pq_delta_to_plain");
    pq_delta_to_plain_kernel<<<(n + 3) / 4, 128, 0, ctx.stream>>>(pages, n, scratch, width, status);
    LAUNCH_CHECK(ctx);
}

PqPrepared pq_prepare(Ctx& ctx, const PqColumnArgs& a, const std::vector<PqPage>& host_pages) {
    PqPrepared pr;
    pr.a = a;
    if (a.n_pages == 0) return pr;
    std::vector<int32_t> tb(host_pages.size() + 1, 0);
    for (size_t i = 0; i < host_pages.size(); i++) tb[i + 1] = tb[i] + (host_pages[i].num_values + PQ_TILE - 1) / PQ_TILE;
    pr.n_tiles = tb.back();
    if (pr.n_tiles == 0) return pr;
    pr.tile_base = to_device(ctx, tb.data(), tb.size() * 4);   // staged before returning (pinned arena copy, or the driver's pageable-copy staging)
    pr.tiles = dalloc(ctx, (size_t)pr.n_tiles * sizeof(PqTile));
    pr.tile_valid = dalloc_zero(ctx, a.max_def > 0 ? (size_t)pr.n_tiles * 128 : 4);   // zeroed: the scout ORs level bits into it
    return pr;
}
static PqLaunch launch_of(const PqPrepared& pr) { return PqLaunch{pr.a, P<int32_t>(pr.tile_base), P<PqTile>(pr.tiles), P<uint32_t>(pr.tile_valid)}; }

void pq_scout_many(Ctx& ctx, const std::vector<PqPrepared*>& cols) {
    std::vector<PqLaunch> Ls;
    std::vector<int32_t> base{0};
    for (auto* pr : cols) {
        if (pr->n_tiles == 0) continue;
        Ls.push_back(launch_of(*pr));
        base.push_back(base.back() + pr->a.n_pages);
    }
    if (Ls.empty()) return;
    ProfScope ps(ctx, "pq_scout");
    if (Ls.size() == 1) {
        pq_scout_kernel<<<(Ls[0].a.n_pages + PQ_WARPS - 1) / PQ_WARPS, PQ_WARPS * 32, 0, ctx.stream>>>(Ls[0]);
    } else {
        Buf dL = to_device(ctx, Ls.data(), Ls.size() * sizeof(PqLaunch));
        Buf dbase = to_device(ctx, base.data(), base.size() * 4);
        pq_scout_multi_kernel<<<(base.back() + PQ_WARPS - 1) / PQ_WARPS, PQ_WARPS * 32, 0, ctx.stream>>>(P<PqLaunch>(dL), P<int32_t>(dbase), (int)Ls.size());
    }
    LAUNCH_CHECK(ctx);
}

void pq_decode_prepared(Ctx& ctx, const PqPrepared& pr) {
    if (pr.n_tiles == 0) return;
    PqLaunch L = launch_of(pr);
    ProfScope ps(ctx, "pq_decode_pages");
    if (pr.a.phys_type == 0) pq_decode_tiles_kernel<<<(pr.n_tiles + PQ_WARPS - 1) / PQ_WARPS, PQ_WARPS * 32, 0, ctx.stream>>>(L, pr.n_tiles);
    else pq_decode_tiles_fast_kernel<<<(pr.n_tiles + PQ_WARPS - 1) / PQ_WARPS, PQ_WARPS * 32, 0, ctx.stream>>>(L, pr.n_tiles);
    LAUNCH_CHECK(ctx);
}

void pq_decode_pages(Ctx& ctx, const PqColumnArgs& a, const std::vector<PqPage>& host_pages) {
    PqPrepared pr = pq_prepare(ctx, a, host_pages);
    pq_scout_many(ctx, {&pr});
    pq_decode_prepared(ctx, pr);
}

// ---- PLAIN BYTE_ARRAY sections (dictionary pages and non-dictionary data pages): one thread walks one section
__global__ void pq_walk_byte_arrays_kernel(const PqByteSection* __restrict__ secs, int n_secs, int64_t* __restrict__ lens,
                                           const uint8_t** __restrict__ srcs) {
    int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= n_secs) return;
    PqByteSection sec = secs[s];
    const uint8_t* p = sec.ptr;
    const uint8_t* end = sec.ptr + sec.len;
    for (int i = 0; i < sec.num_values; i++) {
        uint32_t l = 0;
        if (p + 4 <= end) {
            l = (uint32_t)p[0] | ((uint32_t)p[1] << 8) | ((uint32_t)p[2] << 16) | ((uint32_t)p[3] << 24);
            p += 4;
            if (p + l > end) l = (uint32_t)(end - p);
        }
        lens[sec.value_base + i] = l;
        srcs[sec.value_base + i] = p;
        p += l;
    }
}
__global__ void pq_copy_byte_arrays_kernel(const uint8_t* const* __restrict__ srcs, const int64_t* __restrict__ offs, int64_t n,
                                           int32_t* __restrict__ out_off, uint8_t* __restrict__ out_data) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i > n) return;
    out_off[i] = (int32_t)offs[i];
    if (i == n) return;
    const uint8_t* s = srcs[i];
    uint8_t* d = out_data + offs[i];
    int64_t l = offs[i + 1] - offs[i];
    for (int64_t k = 0; k < l; k++) d[k] = s[k];
}

ColumnPtr pq_build_value_table(Ctx& ctx, const std::vector<PqByteSection>& secs, int64_t total_values, const DType& type) {
    auto col = std::make_shared<Column>();
    col->type = type;
    col->len = total_values;
    col->offsets = dalloc_zero(ctx, (size_t)(total_values + 1) * 4);
    if (total_values == 0 || secs.empty()) {
        col->data = dalloc(ctx, 0);
        return col;
    }
    Buf dsecs = to_device(ctx, secs.data(), secs.size() * sizeof(PqByteSection));
    Buf lens = dalloc_zero(ctx, (size_t)(total_values + 1) * 8);
    Buf srcs = dalloc_zero(ctx, (size_t)(total_values + 1) * 8);
    int n = (int)secs.size();
    pq_walk_byte_arrays_kernel<<<(n + 63) / 64, 64, 0, ctx.stream>>>(P<PqByteSection>(dsecs), n, P<int64_t>(lens), (const uint8_t**)srcs->ptr);
    LAUNCH_CHECK(ctx);
    exclusive_scan_i64(ctx, P<int64_t>(lens), P<int64_t>(lens), total_values, P<int64_t>(lens) + total_values);
    int64_t total = 0;
    to_host(ctx, &total, P<int64_t>(lens) + total_values, 8);
    AURON_CHECK(total <= (int64_t)INT32_MAX, "parquet string chunk exceeds 2 GiB");
    col->data = dalloc(ctx, (size_t)total);
    col->data_bytes = total;
    pq_copy_byte_arrays_kernel<<<(unsigned)((total_values + 1 + 255) / 256), 256, 0, ctx.stream>>>((const uint8_t* const*)srcs->ptr, P<int64_t>(lens), total_values,
                                                                                                 P<int32_t>(col->offsets), P<uint8_t>(col->data));
    LAUNCH_CHECK(ctx);
    ctx.sync();   // secs (host vector) was read by an async copy
    return col;
}

}  // namespace auron
