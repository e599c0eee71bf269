// k_sort.cu -- device sort (row S1) and the shuffle partitioner's counting sort (row S4).
//
// Replaces ExternalSorter::insert_batch / Merger (datafusion-ext-plans/src/sort_exec.rs:637-768,913-1044):
// the reference encodes sort keys with arrow-row (memcmp-able bytes), comparison-sorts each 10k-row
// batch and k-way merges with a loser tree.  On device the whole chunk is sorted at once:
//   * each key column is normalised into order-preserving 64-bit words (Appendix B.13 of SURVEY.md:
//     sign-flipped ints, IEEE total order for floats, NULL sentinel per nulls_first, descending =
//     bitwise NOT, utf8 = big-endian 8-byte chunks + length tiebreak) -- same ORDER as arrow-row,
//   * a stable LSD radix sort (8-bit digits) orders (word, row-id) pairs, least significant word
//     first; digit passes whose histogram is a single bin are skipped,
//   * payload columns are gathered once by the final permutation (take()).
// radix pass = histogram kernel + scan + scatter kernel with an in-shared-memory reorder so global
// writes leave in digit-contiguous runs (coalesced).  HBM-bound: 2 reads + 1 write of 12 B per row per pass.
//
// partition_rows = the counting sort of sort_batches_by_partition_id (shuffle/buffered_data.rs:285-353,
// datafusion-ext-commons/src/algorithm/rdx_sort.rs:24-74) on the same radix machinery (stable here;
// the reference's in-place version is unstable, within-partition order is unspecified).
#include "device_utils.cuh"
#include "kernels.h"

namespace auron {

#define LAUNCH_CHECK(ctx)            \
    do {                             \
        CUDA_OK(cudaGetLastError()); \
        launch_count(ctx);           \
    } while (0)

constexpr int RS_THREADS = 256, RS_ITEMS = 16, RS_TILE = RS_THREADS * RS_ITEMS, RS_WARPS = RS_THREADS / 32;

// all eight digit histograms in one read of the keys
__global__ void __launch_bounds__(256) rs_digit_hist_kernel(const uint64_t* __restrict__ keys, int64_t n, unsigned long long* __restrict__ hist /*[8][256]*/) {
    __shared__ unsigned int sh[8 * 256];
    for (int i = threadIdx.x; i < 8 * 256; i += 256) sh[i] = 0;
    __syncthreads();
    int64_t stride = (int64_t)gridDim.x * 256;
    for (int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x; i < n; i += stride) {
        uint64_t k = keys[i];
#pragma unroll
        for (int d = 0; d < 8; d++) atomicAdd(&sh[d * 256 + ((k >> (8 * d)) & 0xff)], 1u);
    }
    __syncthreads();
    for (int i = threadIdx.x; i < 8 * 256; i += 256)
        if (sh[i]) atomicAdd(&hist[i], (unsigned long long)sh[i]);
}

__global__ void __launch_bounds__(RS_THREADS) rs_tile_hist_kernel(const uint64_t* __restrict__ keys, int64_t n, int shift,
                                                                  int32_t* __restrict__ hist /*[256][nblocks]*/, int nblocks) {
    __shared__ unsigned int sh[256];
    sh[threadIdx.x] = 0;
    __syncthreads();
    int64_t base = (int64_t)blockIdx.x * RS_TILE;
#pragma unroll
    for (int j = 0; j < RS_ITEMS; j++) {
        int64_t i = base + (int64_t)j * RS_THREADS + threadIdx.x;
        if (i < n) atomicAdd(&sh[(keys[i] >> shift) & 0xff], 1u);
    }
    __syncthreads();
    hist[(int64_t)threadIdx.x * nblocks + blockIdx.x] = (int32_t)sh[threadIdx.x];
}

// dynamic smem: keys[RS_TILE] u64 | vals[RS_TILE] i32 | warp_cnt[RS_WARPS][256] u32 | tile_base[256] u32 | gbase[256] i32
__global__ void __launch_bounds__(RS_THREADS) rs_scatter_kernel(const uint64_t* __restrict__ keys_in, const int32_t* __restrict__ vals_in,
                                                                uint64_t* __restrict__ keys_out, int32_t* __restrict__ vals_out, int64_t n,
                                                                int shift, const int32_t* __restrict__ hist_scanned, int nblocks) {
    extern __shared__ __align__(16) uint8_t smem[];
    uint64_t* s_keys = (uint64_t*)smem;
    int32_t* s_vals = (int32_t*)(smem + RS_TILE * 8);
    unsigned int* warp_cnt = (unsigned int*)(smem + RS_TILE * 12);
    unsigned int* tile_base = warp_cnt + RS_WARPS * 256;
    int32_t* gbase = (int32_t*)(tile_base + 256);

    const unsigned lane = lane_id(), warp = threadIdx.x >> 5;
    for (int i = threadIdx.x; i < RS_WARPS * 256; i += RS_THREADS) warp_cnt[i] = 0;
    gbase[threadIdx.x] = hist_scanned[(int64_t)threadIdx.x * nblocks + blockIdx.x];
    __syncthreads();

    int64_t tile0 = (int64_t)blockIdx.x * RS_TILE;
    int64_t warp0 = tile0 + (int64_t)warp * (32 * RS_ITEMS);
    uint64_t k[RS_ITEMS];
    int32_t v[RS_ITEMS];
    unsigned int off[RS_ITEMS];
    // phase A: stable rank of every item among equal digits inside its warp (rounds in index order)
#pragma unroll
    for (int r = 0; r < RS_ITEMS; r++) {
        int64_t i = warp0 + r * 32 + lane;
        bool in = i < n;
        k[r] = in ? keys_in[i] : ~0ull;
        v[r] = in ? vals_in[i] : 0;
        unsigned d = in ? (unsigned)((k[r] >> shift) & 0xff) : 256u;   // out-of-range items match only each other
        unsigned peers = __match_any_sync(FULL_MASK, d);
        unsigned rank = __popc(peers & lanemask_lt());
        int leader = __ffs(peers) - 1;
        unsigned old = 0;
        if (in && (int)lane == leader) {
            old = warp_cnt[warp * 256 + d];
            warp_cnt[warp * 256 + d] = old + __popc(peers);
        }
        old = __shfl_sync(FULL_MASK, old, leader);
        off[r] = old + rank;
        __syncwarp();
    }
    __syncthreads();
    // phase B: per digit, exclusive prefix over warps; then exclusive prefix over digits for the tile
    {
        unsigned d = threadIdx.x, run = 0;
#pragma unroll
        for (int w = 0; w < RS_WARPS; w++) {
            unsigned c = warp_cnt[w * 256 + d];
            warp_cnt[w * 256 + d] = run;
            run += c;
        }
        // block exclusive scan of `run` over 256 digits
        __shared__ unsigned int wsum[8];
        unsigned inc = run;
#pragma unroll
        for (int s = 1; s < 32; s <<= 1) {
            unsigned t = __shfl_up_sync(FULL_MASK, inc, s);
            if (lane >= (unsigned)s) inc += t;
        }
        if (lane == 31) wsum[warp] = inc;
        __syncthreads();
        unsigned wbase = 0;
        for (unsigned w = 0; w < warp; w++) wbase += wsum[w];
        tile_base[d] = wbase + inc - run;
    }
    __syncthreads();
    // phase C: reorder in shared memory
#pragma unroll
    for (int r = 0; r < RS_ITEMS; r++) {
        int64_t i = warp0 + r * 32 + lane;
        if (i < n) {
            unsigned d = (unsigned)((k[r] >> shift) & 0xff);
            unsigned p = tile_base[d] + warp_cnt[warp * 256 + d] + off[r];
            s_keys[p] = k[r];
            s_vals[p] = v[r];
        }
    }
    __syncthreads();
    // phase D: digit-contiguous runs go out coalesced
    int64_t tile_n = min((int64_t)RS_TILE, n - tile0);
#pragma unroll
    for (int j = 0; j < RS_ITEMS; j++) {
        int idx = j * RS_THREADS + threadIdx.x;
        if (idx < tile_n) {
            uint64_t kk = s_keys[idx];
            unsigned d = (unsigned)((kk >> shift) & 0xff);
            int64_t g = (int64_t)gbase[d] + (idx - (int)tile_base[d]);
            keys_out[g] = kk;
            vals_out[g] = s_vals[idx];
        }
    }
}

constexpr size_t RS_SMEM = RS_TILE * 12 + RS_WARPS * 256 * 4 + 256 * 4 + 256 * 4;

void radix_sort_pairs_u64(Ctx& ctx, Buf& keys, Buf& vals, int64_t n, int begin_bit, int end_bit) {
    ProfScope ps_fn(ctx, "radix_sort");
    if (n <= 1) return;
    AURON_CHECK(n < (int64_t)INT32_MAX, "sort chunk too large");
    static bool attr_set = false;
    if (!attr_set) {
        CUDA_OK(cudaFuncSetAttribute(rs_scatter_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)RS_SMEM));
        attr_set = true;
    }
    // which digit passes actually permute anything?
    Buf dh = dalloc_zero(ctx, 8 * 256 * 8);
    int hb = (int)std::min<int64_t>((n + 255) / 256, (int64_t)ctx.sm_count * 8);
    rs_digit_hist_kernel<<<hb, 256, 0, ctx.stream>>>(P<uint64_t>(keys), n, P<unsigned long long>(dh));
    LAUNCH_CHECK(ctx);
    std::vector<unsigned long long> h(8 * 256);
    to_host(ctx, h.data(), dh->ptr, 8 * 256 * 8);
    int nblocks = (int)((n + RS_TILE - 1) / RS_TILE);
    Buf keys2 = dalloc(ctx, (size_t)n * 8), vals2 = dalloc(ctx, (size_t)n * 4);
    Buf hist = dalloc(ctx, (size_t)256 * nblocks * 4);
    for (int d = 0; d < 8; d++) {
        int lo = d * 8, hi = lo + 8;
        if (hi <= begin_bit || lo >= end_bit) continue;
        bool trivial = false;
        for (int b = 0; b < 256; b++)
            if (h[d * 256 + b] == (unsigned long long)n) trivial = true;
        if (trivial) continue;
        rs_tile_hist_kernel<<<nblocks, RS_THREADS, 0, ctx.stream>>>(P<uint64_t>(keys), n, lo, P<int32_t>(hist), nblocks);
        LAUNCH_CHECK(ctx);
        exclusive_scan_i32(ctx, P<int32_t>(hist), P<int32_t>(hist), (int64_t)256 * nblocks, nullptr);
        rs_scatter_kernel<<<nblocks, RS_THREADS, RS_SMEM, ctx.stream>>>(P<uint64_t>(keys), P<int32_t>(vals), P<uint64_t>(keys2), P<int32_t>(vals2), n, lo,
                                                                        P<int32_t>(hist), nblocks);
        LAUNCH_CHECK(ctx);
        std::swap(keys, keys2);
        std::swap(vals, vals2);
    }
}

// ---------------------------------------------------------------------------------------------
// key normalisation
// ---------------------------------------------------------------------------------------------
struct SortCol {
    const void* data;
    const uint8_t* validity;
    const int32_t* offsets;
    int32_t type;
    int32_t asc, nulls_first;
};
// word kinds: 0 = value word (fixed width types; for decimal128 word_idx 0 = hi, 1 = lo)
//             1 = null-rank word ; 2 = utf8 chunk word (word_idx = chunk) ; 3 = utf8 length word
__global__ void __launch_bounds__(256) make_sort_word_kernel(SortCol c, int kind, int word_idx, bool fold_null, const int32_t* __restrict__ perm,
                                                             int64_t n, uint64_t* __restrict__ out) {
    int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x;
    if (i >= n) return;
    int64_t row = perm ? (int64_t)perm[i] : i;
    bool valid = valid_at(c.validity, row);
    uint64_t nullrank = valid ? (c.nulls_first ? 1ull : 0ull) : (c.nulls_first ? 0ull : 1ull);
    if (kind == 1) {
        out[i] = nullrank;
        return;
    }
    uint64_t w = 0;
    int bits = 64;
    if (kind == 0) {
        if (c.type == T_BOOL || c.type == T_INT8) bits = 8;
        else if (c.type == T_INT16) bits = 16;
        else if (c.type == T_INT32 || c.type == T_DATE32 || c.type == T_FLOAT32) bits = 32;
    } else if (kind == 3) {
        bits = 32;
    }
    if (valid) {
        if (kind == 0) {
            switch (c.type) {
                case T_BOOL: w = bit_get((const uint8_t*)c.data, row); break;
                case T_INT8: w = (uint64_t)(uint8_t)(((const int8_t*)c.data)[row] ^ 0x80); break;
                case T_INT16: w = (uint64_t)(uint16_t)(((const int16_t*)c.data)[row] ^ 0x8000); break;
                case T_INT32: case T_DATE32: w = (uint64_t)(((const uint32_t*)c.data)[row] ^ 0x80000000u); break;
                case T_FLOAT32: {
                    uint32_t b = ((const uint32_t*)c.data)[row];
                    w = (b & 0x80000000u) ? (uint32_t)~b : (b | 0x80000000u);
                    break;
                }
                case T_FLOAT64: {
                    uint64_t b = ((const uint64_t*)c.data)[row];
                    w = (b >> 63) ? ~b : (b | 0x8000000000000000ull);
                    break;
                }
                case T_DECIMAL128: {
                    uint64_t lo = ((const uint64_t*)c.data)[2 * row], hi = ((const uint64_t*)c.data)[2 * row + 1];
                    w = word_idx == 0 ? (hi ^ 0x8000000000000000ull) : lo;
                    break;
                }
                default: w = ((const uint64_t*)c.data)[row] ^ 0x8000000000000000ull; break;
            }
        } else if (kind == 2) {
            int32_t b = c.offsets[row], e = c.offsets[row + 1];
            const uint8_t* p = (const uint8_t*)c.data + b;
            int32_t len = e - b, start = word_idx * 8;
#pragma unroll
            for (int j = 0; j < 8; j++) {
                uint64_t byte = (start + j < len) ? p[start + j] : 0;
                w = (w << 8) | byte;
            }
        } else {
            w = (uint64_t)(uint32_t)(c.offsets[row + 1] - c.offsets[row]);
        }
        if (!c.asc) w = (bits == 64) ? ~w : (~w & ((1ull << bits) - 1ull));
    }
    if (fold_null) w |= nullrank << bits;   // only for words narrower than 64 bits
    out[i] = w;
}
__global__ void max_len_kernel(const int32_t* __restrict__ offsets, int64_t n, int32_t* out) {
    int32_t m = 0;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
        m = max(m, offsets[i + 1] - offsets[i]);
    for (int d = 16; d; d >>= 1) m = max(m, __shfl_down_sync(FULL_MASK, m, d));
    if (lane_id() == 0) atomicMax(out, m);
}

struct WordPlan {
    int col, kind, word_idx;
    bool fold_null;
};

Buf sort_indices(Ctx& ctx, const std::vector<SortKeySpec>& keys, int64_t n) {
    Buf perm = dalloc(ctx, (size_t)std::max<int64_t>(n, 1) * 4);
    fill_iota_i32(ctx, P<int32_t>(perm), n, 0);
    if (n <= 1 || keys.empty()) return perm;
    // most-significant-first list of words
    std::vector<WordPlan> words;
    std::vector<SortCol> cols;
    for (size_t ci = 0; ci < keys.size(); ci++) {
        const Column& c = *keys[ci].col;
        SortCol sc{c.data ? c.data->ptr : nullptr, c.vbits(), P<int32_t>(c.offsets), (int32_t)c.type.id, keys[ci].asc ? 1 : 0, keys[ci].nulls_first ? 1 : 0};
        cols.push_back(sc);
        bool nullable = c.may_have_nulls();
        int w = c.type.width();
        if (c.type.id == T_NULL) continue;
        if (c.type.is_varlen()) {
            Buf ml = dalloc_zero(ctx, 4);
            int blocks = (int)std::min<int64_t>((n + 255) / 256, (int64_t)ctx.sm_count * 4);
            max_len_kernel<<<blocks, 256, 0, ctx.stream>>>(P<int32_t>(c.offsets), n, P<int32_t>(ml));
            LAUNCH_CHECK(ctx);
            int32_t maxlen = 0;
            to_host(ctx, &maxlen, ml->ptr, 4);
            if (nullable) words.push_back({(int)ci, 1, 0, false});
            for (int k = 0; k < (maxlen + 7) / 8; k++) words.push_back({(int)ci, 2, k, false});
            words.push_back({(int)ci, 3, 0, false});
        } else if (c.type.id == T_DECIMAL128) {
            if (nullable) words.push_back({(int)ci, 1, 0, false});
            words.push_back({(int)ci, 0, 0, false});
            words.push_back({(int)ci, 0, 1, false});
        } else if (w == 8) {
            if (nullable) words.push_back({(int)ci, 1, 0, false});
            words.push_back({(int)ci, 0, 0, false});
        } else {
            words.push_back({(int)ci, 0, 0, nullable});
        }
    }
    Buf kbuf = dalloc(ctx, (size_t)n * 8);
    unsigned blocks = (unsigned)((n + 255) / 256);
    bool first = true;
    for (int wi = (int)words.size() - 1; wi >= 0; wi--) {
        const WordPlan& wp = words[wi];
        make_sort_word_kernel<<<blocks, 256, 0, ctx.stream>>>(cols[wp.col], wp.kind, wp.word_idx, wp.fold_null, first ? nullptr : P<int32_t>(perm), n,
                                                              P<uint64_t>(kbuf));
        LAUNCH_CHECK(ctx);
        radix_sort_pairs_u64(ctx, kbuf, perm, n, 0, 64);
        first = false;
    }
    return perm;
}

// ---------------------------------------------------------------------------------------------
// external sort support (sort_exec.rs:390-447 spill, :913-1061 Merger): sorted runs are merged by key RANGES -- splitters are
// sampled from the runs, every run is cut at the splitters by binary search over its normalised key words, and the slices
// of one range (from all runs) are sorted together.  The words of a run are comparable with those of any other run: the
// NULL rank is always part of the plan here, whether or not the run's column carries a validity bitmap.
// ---------------------------------------------------------------------------------------------
bool sort_key_words(Ctx& ctx, const std::vector<SortKeySpec>& keys, int64_t n, std::vector<Buf>* words) {
    std::vector<WordPlan> plan;
    std::vector<SortCol> cols;
    for (size_t ci = 0; ci < keys.size(); ci++) {
        const Column& c = *keys[ci].col;
        if (c.type.is_varlen()) return false;   // word count depends on the longest value of the run
        cols.push_back(SortCol{c.data ? c.data->ptr : nullptr, c.vbits(), P<int32_t>(c.offsets), (int32_t)c.type.id, keys[ci].asc ? 1 : 0, keys[ci].nulls_first ? 1 : 0});
        if (c.type.id == T_NULL) continue;
        if (c.type.id == T_DECIMAL128) {
            plan.push_back({(int)ci, 1, 0, false});
            plan.push_back({(int)ci, 0, 0, false});
            plan.push_back({(int)ci, 0, 1, false});
        } else if (c.type.width() == 8) {
            plan.push_back({(int)ci, 1, 0, false});
            plan.push_back({(int)ci, 0, 0, false});
        } else {
            plan.push_back({(int)ci, 0, 0, true});
        }
    }
    words->clear();
    const unsigned blocks = (unsigned)((std::max<int64_t>(n, 1) + 255) / 256);
    for (auto& wp : plan) {
        Buf w = dalloc(ctx, (size_t)std::max<int64_t>(n, 1) * 8);
        if (n > 0) {
            make_sort_word_kernel<<<blocks, 256, 0, ctx.stream>>>(cols[(size_t)wp.col], wp.kind, wp.word_idx, wp.fold_null, nullptr, n, P<uint64_t>(w));
            LAUNCH_CHECK(ctx);
        }
        words->push_back(w);
    }
    return true;
}
// the word arrays of a run as a device array of pointers: a key of k columns has up to 3 k words (NULL rank + two decimal128
// words), so there is no fixed bound to put in a kernel argument
struct WordPtrs {
    const uint64_t* const* w;
    int nw;
};
// out[s * W + w] = word w of row floor((2 s + 1) n / (2 S)): S evenly spaced samples of a sorted run
__global__ void sample_words_kernel(WordPtrs wp, int64_t n, int S, uint64_t* __restrict__ out) {
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= S) return;
    const int64_t row = min(n - 1, (int64_t)(((2 * (long long)s + 1) * n) / (2 * (long long)S)));
    for (int w = 0; w < wp.nw; w++) out[(int64_t)s * wp.nw + w] = wp.w[w][row];
}
// out[s] = number of rows of the run whose word tuple is lexicographically < splitter s
__global__ void lower_bound_words_kernel(WordPtrs wp, int64_t n, const uint64_t* __restrict__ splitters, int S, int64_t* __restrict__ out) {
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= S) return;
    int64_t lo = 0, hi = n;
    while (lo < hi) {
        const int64_t mid = lo + ((hi - lo) >> 1);
        bool less = false;
        for (int w = 0; w < wp.nw; w++) {
            const uint64_t a = wp.w[w][mid], b = splitters[(int64_t)s * wp.nw + w];
            if (a != b) {
                less = a < b;
                break;
            }
        }
        if (less) lo = mid + 1;
        else hi = mid;
    }
    out[s] = lo;
}
// *ptrs keeps the pointer array alive until the caller's kernel has been enqueued (frees are stream-ordered)
static WordPtrs word_ptrs(Ctx& ctx, const std::vector<Buf>& words, Buf* ptrs) {
    std::vector<const uint64_t*> host(words.size());
    for (size_t i = 0; i < words.size(); i++) host[i] = P<uint64_t>(words[i]);
    *ptrs = to_device(ctx, host.data(), host.size() * sizeof(host[0]));
    return WordPtrs{P<const uint64_t*>(*ptrs), (int)words.size()};
}
std::vector<uint64_t> sample_sorted_words(Ctx& ctx, const std::vector<Buf>& words, int64_t n, int S) {
    std::vector<uint64_t> host((size_t)S * words.size());
    if (S <= 0 || n <= 0 || words.empty()) return host;
    Buf out = dalloc(ctx, host.size() * 8), ptrs;
    sample_words_kernel<<<(S + 127) / 128, 128, 0, ctx.stream>>>(word_ptrs(ctx, words, &ptrs), n, S, P<uint64_t>(out));
    LAUNCH_CHECK(ctx);
    to_host(ctx, host.data(), out->ptr, host.size() * 8);
    return host;
}
std::vector<int64_t> lower_bound_sorted_words(Ctx& ctx, const std::vector<Buf>& words, int64_t n, const std::vector<uint64_t>& splitters, int S) {
    std::vector<int64_t> host((size_t)S, 0);
    if (S <= 0) return host;
    if (n <= 0 || words.empty()) return host;
    Buf ds = to_device(ctx, splitters.data(), splitters.size() * 8);
    Buf out = dalloc(ctx, (size_t)S * 8), ptrs;
    lower_bound_words_kernel<<<(S + 127) / 128, 128, 0, ctx.stream>>>(word_ptrs(ctx, words, &ptrs), n, P<uint64_t>(ds), S, P<int64_t>(out));
    LAUNCH_CHECK(ctx);
    to_host(ctx, host.data(), out->ptr, (size_t)S * 8);
    return host;
}

// ---------------------------------------------------------------------------------------------
// partitioner
// ---------------------------------------------------------------------------------------------
__global__ void widen_pid_kernel(const int32_t* __restrict__ pid, int64_t n, uint64_t* __restrict__ out) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = (uint64_t)(uint32_t)pid[i];
}
__global__ void __launch_bounds__(256) pid_hist_kernel(const int32_t* __restrict__ pid, int64_t n, int32_t num_parts, unsigned long long* __restrict__ counts) {
    extern __shared__ unsigned int shh[];
    bool use_sh = num_parts <= 8192;
    if (use_sh) {
        for (int i = threadIdx.x; i < num_parts; i += 256) shh[i] = 0;
        __syncthreads();
    }
    int64_t stride = (int64_t)gridDim.x * 256;
    for (int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x; i < n; i += stride) {
        int32_t p = pid[i];
        if (use_sh) atomicAdd(&shh[p], 1u);
        else atomicAdd(&counts[p], 1ull);
    }
    if (use_sh) {
        __syncthreads();
        for (int i = threadIdx.x; i < num_parts; i += 256)
            if (shh[i]) atomicAdd(&counts[i], (unsigned long long)shh[i]);
    }
}

// range partitioning: perm = stable sort order of [n key rows ++ nb bound rows]; out[key row] = bound rows in front of it
__global__ void bound_flag_kernel(const int32_t* __restrict__ perm, int64_t total, int32_t n, int32_t* __restrict__ flags) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < total) flags[i] = perm[i] >= n ? 1 : 0;
}
__global__ void bound_rank_scatter_kernel(const int32_t* __restrict__ perm, const int32_t* __restrict__ rank, int64_t total, int32_t n,
                                          int32_t* __restrict__ out) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < total && perm[i] < n) out[perm[i]] = rank[i];
}
Buf bound_ranks(Ctx& ctx, const int32_t* perm, int64_t n, int64_t nb) {
    const int64_t total = n + nb;
    Buf out = dalloc(ctx, (size_t)std::max<int64_t>(n, 1) * 4);
    if (total == 0) return out;
    Buf flags = dalloc(ctx, (size_t)total * 4), tot = dalloc(ctx, 4);
    unsigned blocks = (unsigned)((total + 255) / 256);
    bound_flag_kernel<<<blocks, 256, 0, ctx.stream>>>(perm, total, (int32_t)n, P<int32_t>(flags));
    LAUNCH_CHECK(ctx);
    exclusive_scan_i32(ctx, P<int32_t>(flags), P<int32_t>(flags), total, P<int32_t>(tot));
    bound_rank_scatter_kernel<<<blocks, 256, 0, ctx.stream>>>(perm, P<int32_t>(flags), total, (int32_t)n, P<int32_t>(out));
    LAUNCH_CHECK(ctx);
    return out;
}

void partition_rows(Ctx& ctx, const int32_t* part_ids, int64_t n, int32_t num_parts, Buf* rows_out, Buf* offsets_out) {
    ProfScope ps_fn(ctx, "partition_rows");
    Buf counts = dalloc_zero(ctx, (size_t)(num_parts + 1) * 8);
    Buf rows = dalloc(ctx, (size_t)std::max<int64_t>(n, 1) * 4);
    fill_iota_i32(ctx, P<int32_t>(rows), n, 0);
    if (n > 0) {
        int blocks = (int)std::min<int64_t>((n + 255) / 256, (int64_t)ctx.sm_count * 8);
        size_t sh = num_parts <= 8192 ? (size_t)num_parts * 4 : 0;
        pid_hist_kernel<<<blocks, 256, sh, ctx.stream>>>(part_ids, n, num_parts, P<unsigned long long>(counts));
        LAUNCH_CHECK(ctx);
        if (num_parts > 1) {
            Buf keys = dalloc(ctx, (size_t)n * 8);
            widen_pid_kernel<<<(unsigned)((n + 255) / 256), 256, 0, ctx.stream>>>(part_ids, n, P<uint64_t>(keys));
            LAUNCH_CHECK(ctx);
            int bits = 1;
            while ((1ll << bits) < num_parts) bits++;
            radix_sort_pairs_u64(ctx, keys, rows, n, 0, bits);
        }
    }
    exclusive_scan_i64(ctx, P<int64_t>(counts), P<int64_t>(counts), num_parts + 1, nullptr);
    *rows_out = rows;
    *offsets_out = counts;
}

}  // namespace auron
