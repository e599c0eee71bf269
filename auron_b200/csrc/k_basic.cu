// k_basic.cu -- context, stream-ordered device memory, prefix scans, bitmap compaction, gather
// (take), concat.  These are the HBM-bound building blocks every operator composes; the gather is
// the device counterpart of datafusion-ext-commons/src/arrow/selection.rs:32-304 (take/interleave)
// and arrow-select filter (cached_exprs_evaluator.rs:131).
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <mutex>

#include "device_utils.cuh"
#include "kernels.h"

namespace auron {

// ---------------------------------------------------------------------------------------------
std::string DType::str() const {
    switch (id) {
        case T_NULL: return "null";
        case T_BOOL: return "bool";
        case T_INT8: return "int8";
        case T_INT16: return "int16";
        case T_INT32: return "int32";
        case T_INT64: return "int64";
        case T_FLOAT32: return "float32";
        case T_FLOAT64: return "float64";
        case T_UTF8: return "utf8";
        case T_BINARY: return "binary";
        case T_DATE32: return "date32";
        case T_DATE64: return "date64";
        case T_TIMESTAMP: return "timestamp";
        case T_DECIMAL128: return "decimal128(" + std::to_string(precision) + "," + std::to_string(scale) + ")";
        case T_LIST: return "list<" + (elem ? elem->str() : std::string("?")) + ">";
    }
    return "?";
}

Ctx::Ctx(int dev, int stream_priority) : device(dev) {
    if (dev < 0) return;   // plan-only context (auron_b200_explain): no stream, nothing may be launched on it
    CUDA_OK(cudaSetDevice(dev));
    if (stream_priority != 0) {
        int least = 0, greatest = 0;
        CUDA_OK(cudaDeviceGetStreamPriorityRange(&least, &greatest));   // numerically lower = higher priority
        CUDA_OK(cudaStreamCreateWithPriority(&stream, cudaStreamNonBlocking, std::max(greatest, std::min(least, stream_priority))));
    } else {
        CUDA_OK(cudaStreamCreateWithFlags(&stream, cudaStreamNonBlocking));
    }
    CUDA_OK(cudaDeviceGetAttribute(&sm_count, cudaDevAttrMultiProcessorCount, dev));
    if (const char* e = getenv("AURON_PROFILE")) profile = atoi(e) != 0;
    if (const char* e = getenv("AURON_GPU_CHUNK_ROWS")) {   // device-side accumulation target (tests shrink it to force merges)
        long long v = atoll(e);
        if (v > 0) gpu_chunk_rows = v;
    }
    // keep freed blocks in the pool: operators allocate/free per chunk (HBM arena policy, exec.rs:79-82 analogue)
    static std::once_flag once[16];
    std::call_once(once[dev & 15], [&] {
        cudaMemPool_t pool;
        if (cudaDeviceGetDefaultMemPool(&pool, dev) == cudaSuccess) {
            uint64_t thr = UINT64_MAX;
            cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &thr);
        }
    });
}
std::vector<Ctx::ProfTotal> Ctx::prof_summary() {
    std::vector<ProfTotal> out;
    if (prof.empty()) return out;
    if (getenv("AURON_PROF_TIMELINE")) {   // start / end of every timed launch site relative to the first one (streams overlap: a timeline, not a sum)
        for (auto& e : prof) cudaEventSynchronize(e.e1);
        cudaEvent_t base = prof[0].e0;
        float best = 0;
        for (auto& e : prof) {
            float d = 0;
            if (cudaEventElapsedTime(&d, e.e0, base) == cudaSuccess && d > best) {   // e.e0 earlier than base
                best = d;
                base = e.e0;
            }
        }
        for (auto& e : prof) {
            float a = 0, b = 0;
            cudaEventElapsedTime(&a, base, e.e0);
            cudaEventElapsedTime(&b, base, e.e1);
            fprintf(stderr, "[timeline] %-22s %8.3f .. %8.3f ms\n", e.name, a, b);
        }
    }
    cudaStreamSynchronize(stream);
    for (auto& e : prof) {
        float ms = 0;
        cudaEventElapsedTime(&ms, e.e0, e.e1);
        cudaEventDestroy(e.e0);
        cudaEventDestroy(e.e1);
        bool found = false;
        for (auto& t : out)
            if (t.name == e.name) {
                t.ms += ms;
                t.launches++;
                found = true;
            }
        if (!found) out.push_back({e.name, ms, 1});
    }
    prof.clear();
    return out;
}
static void stage_arena_put(uint8_t* p);
static const bool g_stall_log = getenv("AURON_STALL_LOG") != nullptr;   // report host-side stalls of allocator / sync calls
void Ctx::sync() {
    if (g_stall_log) {
        auto t0 = std::chrono::steady_clock::now();
        CUDA_OK(cudaStreamSynchronize(stream));
        double ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
        if (ms > 40.0) fprintf(stderr, "[stall] stream sync took %.1f ms\n", ms);
    } else {
        CUDA_OK(cudaStreamSynchronize(stream));
    }
    stage_off = 0;   // every staged upload kernel has run
}
Ctx::~Ctx() {
    for (auto& e : prof) {
        cudaEventDestroy(e.e0);
        cudaEventDestroy(e.e1);
    }
    if (stream) {
        cudaStreamSynchronize(stream);
        cudaStreamDestroy(stream);
    }
    if (stage_host) stage_arena_put(stage_host);
}

DevMem::~DevMem() {
    if (!ptr) return;
    if (g_stall_log) {
        auto t0 = std::chrono::steady_clock::now();
        cudaFreeAsync(ptr, stream);
        double ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
        if (ms > 2.0) fprintf(stderr, "[stall] cudaFreeAsync(%zu) took %.1f ms\n", bytes, ms);
        return;
    }
    cudaFreeAsync(ptr, stream);
}

// AURON_STALL_LOG=1: report allocator calls that take longer than 2 ms on the host (pool growth shows up here)
Buf dalloc(Ctx& ctx, size_t bytes) {
    auto m = std::make_shared<DevMem>();
    m->bytes = bytes;
    m->stream = ctx.stream;
    if (g_stall_log) {
        auto t0 = std::chrono::steady_clock::now();
        CUDA_OK(cudaMallocAsync(&m->ptr, bytes + 64, ctx.stream));
        double ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
        if (ms > 2.0) fprintf(stderr, "[stall] cudaMallocAsync(%zu) took %.1f ms\n", bytes, ms);
        return m;
    }
    CUDA_OK(cudaMallocAsync(&m->ptr, bytes + 64, ctx.stream));
    return m;
}
Buf dalloc_fill(Ctx& ctx, size_t bytes, int byte) {
    Buf b = dalloc(ctx, bytes);
    CUDA_OK(cudaMemsetAsync(b->ptr, byte, bytes + 64, ctx.stream));
    return b;
}
Buf dalloc_zero(Ctx& ctx, size_t bytes) { return dalloc_fill(ctx, bytes, 0); }
// ---- staged small uploads (see Ctx::stage_host)
static const size_t kStageArena = 16u << 20, kStageMax = 4u << 20;
static std::mutex g_stage_mu;
static std::vector<uint8_t*> g_stage_free;
static uint8_t* stage_arena_get() {
    {
        std::lock_guard<std::mutex> l(g_stage_mu);
        if (!g_stage_free.empty()) {
            uint8_t* p = g_stage_free.back();
            g_stage_free.pop_back();
            return p;
        }
    }
    void* p = nullptr;
    CUDA_OK(cudaHostAlloc(&p, kStageArena, cudaHostAllocMapped | cudaHostAllocPortable));
    return (uint8_t*)p;
}
static void stage_arena_put(uint8_t* p) {
    std::lock_guard<std::mutex> l(g_stage_mu);
    g_stage_free.push_back(p);
}
__global__ void staged_upload_kernel(uint4* __restrict__ dst, const uint4* __restrict__ src, size_t n16) {
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n16; i += (size_t)gridDim.x * blockDim.x) dst[i] = src[i];
}
void upload_small(Ctx& ctx, void* dev, const void* host, size_t bytes) {
    if (bytes == 0) return;
    size_t padded = (bytes + 15) & ~(size_t)15;
    if (padded > kStageMax || ((uintptr_t)dev & 15)) {   // bulk or oddly placed: plain copy-engine transfer
        CUDA_OK(cudaMemcpyAsync(dev, host, bytes, cudaMemcpyHostToDevice, ctx.stream));
        return;
    }
    if (!ctx.stage_host) {
        ctx.stage_host = stage_arena_get();
        ctx.stage_cap = kStageArena;
        ctx.stage_off = 0;
    }
    if (ctx.stage_off + padded > ctx.stage_cap) ctx.sync();
    uint8_t* st = ctx.stage_host + ctx.stage_off;
    memcpy(st, host, bytes);
    ctx.stage_off += padded;
    size_t n16 = padded / 16;
    int blocks = (int)std::min<size_t>((n16 + 255) / 256, (size_t)ctx.sm_count * 4);
    staged_upload_kernel<<<blocks, 256, 0, ctx.stream>>>((uint4*)dev, (const uint4*)st, n16);
    CUDA_OK(cudaGetLastError());
}
Buf to_device(Ctx& ctx, const void* host, size_t bytes) {
    Buf b = dalloc(ctx, bytes);   // allocations are padded by 64 B, so the 16-byte rounding of the staged copy stays inside
    upload_small(ctx, b->ptr, host, bytes);
    return b;
}
void to_host(Ctx& ctx, void* host, const void* dev, size_t bytes) {
    if (bytes) CUDA_OK(cudaMemcpyAsync(host, dev, bytes, cudaMemcpyDeviceToHost, ctx.stream));
    ctx.sync();
}
void launch_count(Ctx& ctx, int n) { ctx.kernel_launches += n; }

#define LAUNCH_CHECK(ctx)            \
    do {                             \
        CUDA_OK(cudaGetLastError()); \
        launch_count(ctx);           \
    } while (0)

ColumnPtr make_column(Ctx& ctx, const DType& t, int64_t len, bool with_validity) {
    auto c = std::make_shared<Column>();
    c->type = t;
    c->len = len;
    if (t.id == T_BOOL) c->data = dalloc_zero(ctx, bitmap_alloc_bytes(len));
    else if (t.width() > 0) c->data = dalloc(ctx, (size_t)len * t.width());
    else if (t.is_varlen()) {
        c->offsets = dalloc_zero(ctx, (size_t)(len + 1) * 4);
        c->data = dalloc(ctx, 0);
    }
    if (with_validity) {
        c->validity = dalloc_zero(ctx, bitmap_alloc_bytes(len));
        c->null_count = -1;
    }
    return c;
}
ColumnPtr make_null_column(Ctx& ctx, const DType& t, int64_t len) {
    auto c = make_column(ctx, t, len, true);
    if (t.width() > 0) CUDA_OK(cudaMemsetAsync(c->data->ptr, 0, (size_t)len * t.width(), ctx.stream));
    c->null_count = len;
    return c;
}

// ---------------------------------------------------------------------------------------------
// exclusive scan: reduce-then-scan, 256 threads x 8 items per block
// ---------------------------------------------------------------------------------------------
constexpr int SCAN_T = 256, SCAN_I = 8, SCAN_TILE = SCAN_T * SCAN_I;

template <typename T>
__device__ __forceinline__ T block_exclusive_scan(T v, T* total) {
    __shared__ T warp_sums[SCAN_T / 32];
    __shared__ T block_total;
    unsigned lane = lane_id(), warp = threadIdx.x >> 5;
    T inc = v;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        T t = __shfl_up_sync(FULL_MASK, inc, d);
        if (lane >= (unsigned)d) inc += t;
    }
    if (lane == 31) warp_sums[warp] = inc;
    __syncthreads();
    if (warp == 0) {
        T w = lane < SCAN_T / 32 ? warp_sums[lane] : T(0);
        T winc = w;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            T t = __shfl_up_sync(FULL_MASK, winc, d);
            if (lane >= (unsigned)d) winc += t;
        }
        if (lane < SCAN_T / 32) warp_sums[lane] = winc - w;
        if (lane == SCAN_T / 32 - 1) block_total = winc;
    }
    __syncthreads();
    T res = inc - v + warp_sums[warp];
    *total = block_total;
    __syncthreads();
    return res;
}

template <typename T>
__global__ void __launch_bounds__(SCAN_T) scan_reduce_kernel(const T* __restrict__ in, T* __restrict__ block_sums, int64_t n) {
    int64_t base = (int64_t)blockIdx.x * SCAN_TILE;
    T s = 0;
#pragma unroll
    for (int k = 0; k < SCAN_I; k++) {
        int64_t i = base + (int64_t)k * SCAN_T + threadIdx.x;
        if (i < n) s += in[i];
    }
    T total;
    block_exclusive_scan<T>(s, &total);
    if (threadIdx.x == 0) block_sums[blockIdx.x] = total;
}

template <typename T>
__global__ void __launch_bounds__(SCAN_T) scan_apply_kernel(const T* __restrict__ in, T* __restrict__ out, const T* __restrict__ block_bases,
                                                            int64_t n, T* __restrict__ total_out) {
    int64_t base = (int64_t)blockIdx.x * SCAN_TILE + (int64_t)threadIdx.x * SCAN_I;
    T v[SCAN_I];
    T s = 0;
#pragma unroll
    for (int k = 0; k < SCAN_I; k++) {
        int64_t i = base + k;
        v[k] = i < n ? in[i] : T(0);
        s += v[k];
    }
    T total;
    T ex = block_exclusive_scan<T>(s, &total);
    T bb = block_bases ? block_bases[blockIdx.x] : T(0);
    T run = ex + bb;
#pragma unroll
    for (int k = 0; k < SCAN_I; k++) {
        int64_t i = base + k;
        if (i < n) out[i] = run;
        run += v[k];
    }
    if (total_out && blockIdx.x == gridDim.x - 1 && threadIdx.x == 0) *total_out = bb + total;
}

template <typename T>
static void exclusive_scan_t(Ctx& ctx, const T* in, T* out, int64_t n, T* total_dev) {
    if (n <= 0) {
        if (total_dev) CUDA_OK(cudaMemsetAsync(total_dev, 0, sizeof(T), ctx.stream));
        return;
    }
    int64_t nblocks = (n + SCAN_TILE - 1) / SCAN_TILE;
    if (nblocks == 1) {
        scan_apply_kernel<T><<<1, SCAN_T, 0, ctx.stream>>>(in, out, nullptr, n, total_dev);
        LAUNCH_CHECK(ctx);
        return;
    }
    Buf sums = dalloc(ctx, nblocks * sizeof(T));
    scan_reduce_kernel<T><<<(unsigned)nblocks, SCAN_T, 0, ctx.stream>>>(in, P<T>(sums), n);
    LAUNCH_CHECK(ctx);
    exclusive_scan_t<T>(ctx, P<T>(sums), P<T>(sums), nblocks, nullptr);
    scan_apply_kernel<T><<<(unsigned)nblocks, SCAN_T, 0, ctx.stream>>>(in, out, P<T>(sums), n, total_dev);
    LAUNCH_CHECK(ctx);
}
void exclusive_scan_i32(Ctx& ctx, const int32_t* in, int32_t* out, int64_t n, int32_t* total_dev) {
    exclusive_scan_t<int32_t>(ctx, in, out, n, total_dev);
}
void exclusive_scan_i64(Ctx& ctx, const int64_t* in, int64_t* out, int64_t n, int64_t* total_dev) {
    exclusive_scan_t<int64_t>(ctx, in, out, n, total_dev);
}

// ---------------------------------------------------------------------------------------------
// bitmap -> indices (stream compaction).  One thread per 32-bit mask word.
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) mask_popc_kernel(const uint32_t* __restrict__ mask, int64_t n_words, int64_t n_rows,
                                                        int32_t* __restrict__ block_counts) {
    int64_t w = (int64_t)blockIdx.x * 256 + threadIdx.x;
    uint32_t m = 0;
    if (w < n_words) {
        m = mask[w];
        int64_t rem = n_rows - w * 32;
        if (rem < 32) m &= (1u << rem) - 1u;
    }
    int c = __popc(m);
    int total;
    block_exclusive_scan<int>(c, &total);
    if (threadIdx.x == 0) block_counts[blockIdx.x] = total;
}
__global__ void __launch_bounds__(256) mask_write_kernel(const uint32_t* __restrict__ mask, int64_t n_words, int64_t n_rows,
                                                         const int32_t* __restrict__ block_bases, int32_t* __restrict__ out) {
    int64_t w = (int64_t)blockIdx.x * 256 + threadIdx.x;
    uint32_t m = 0;
    if (w < n_words) {
        m = mask[w];
        int64_t rem = n_rows - w * 32;
        if (rem < 32) m &= (1u << rem) - 1u;
    }
    int c = __popc(m);
    int total;
    int ex = block_exclusive_scan<int>(c, &total);
    int32_t pos = block_bases[blockIdx.x] + ex;
    int32_t row0 = (int32_t)(w * 32);
    while (m) {
        int b = __ffs(m) - 1;
        out[pos++] = row0 + b;
        m &= m - 1;
    }
}
__global__ void popc_reduce_kernel(const uint32_t* __restrict__ words, int64_t n_words, int64_t n_bits, unsigned long long* out) {
    unsigned long long s = 0;
    for (int64_t w = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; w < n_words; w += (int64_t)gridDim.x * blockDim.x) {
        uint32_t m = words[w];
        int64_t rem = n_bits - w * 32;
        if (rem < 32) m &= (1u << rem) - 1u;
        s += __popc(m);
    }
    for (int d = 16; d; d >>= 1) s += __shfl_down_sync(FULL_MASK, s, d);
    if (lane_id() == 0 && s) atomicAdd(out, s);
}
int64_t count_set_bits(Ctx& ctx, const uint8_t* bitmap, int64_t n) {
    if (n <= 0 || !bitmap) return 0;
    Buf out = dalloc_zero(ctx, 8);
    int64_t n_words = (n + 31) / 32;
    int blocks = (int)std::min<int64_t>((n_words + 255) / 256, ctx.sm_count * 8);
    popc_reduce_kernel<<<blocks, 256, 0, ctx.stream>>>((const uint32_t*)bitmap, n_words, n, P<unsigned long long>(out));
    LAUNCH_CHECK(ctx);
    int64_t h = 0;
    to_host(ctx, &h, out->ptr, 8);
    return h;
}
Buf mask_to_indices(Ctx& ctx, const uint32_t* mask_words, int64_t n_rows, int64_t* count_out) {
    AURON_CHECK(n_rows < (int64_t)INT32_MAX, "batch too large for int32 row indices");
    if (n_rows <= 0) {
        *count_out = 0;
        return dalloc(ctx, 4);
    }
    int64_t n_words = (n_rows + 31) / 32;
    int64_t nblocks = (n_words + 255) / 256;
    ProfScope ps(ctx, "mask_to_indices");
    Buf counts = dalloc(ctx, (nblocks + 1) * 4);
    mask_popc_kernel<<<(unsigned)nblocks, 256, 0, ctx.stream>>>(mask_words, n_words, n_rows, P<int32_t>(counts));
    LAUNCH_CHECK(ctx);
    Buf total = dalloc(ctx, 4);
    exclusive_scan_i32(ctx, P<int32_t>(counts), P<int32_t>(counts), nblocks, P<int32_t>(total));
    int32_t cnt = 0;
    to_host(ctx, &cnt, total->ptr, 4);
    *count_out = cnt;
    Buf out = dalloc(ctx, (size_t)std::max<int64_t>(cnt, 1) * 4);
    if (cnt > 0) {
        mask_write_kernel<<<(unsigned)nblocks, 256, 0, ctx.stream>>>(mask_words, n_words, n_rows, P<int32_t>(counts), P<int32_t>(out));
        LAUNCH_CHECK(ctx);
    }
    return out;
}

// dst is pre-zeroed; one thread per destination word touched
__global__ void copy_bits_kernel(uint32_t* __restrict__ dst, int64_t dst_off, const uint8_t* __restrict__ src, int64_t src_off, int64_t n) {
    int64_t first_word = dst_off >> 5;
    int64_t last_word = (dst_off + n - 1) >> 5;
    int64_t w = first_word + (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (w > last_word) return;
    int64_t lo = max(w * 32, dst_off), hi = min(w * 32 + 32, dst_off + n);  // dst bit range in this word
    uint32_t v = 0;
    for (int64_t b = lo; b < hi; b++) {
        int64_t s = src_off + (b - dst_off);
        if ((src[s >> 3] >> (s & 7)) & 1) v |= 1u << (b & 31);
    }
    if (v) atomicOr(&dst[w], v);
}
void copy_bits(Ctx& ctx, uint8_t* dst, int64_t dst_off, const uint8_t* src, int64_t src_off, int64_t n) {
    if (n <= 0) return;
    int64_t words = ((dst_off + n - 1) >> 5) - (dst_off >> 5) + 1;
    copy_bits_kernel<<<(unsigned)((words + 255) / 256), 256, 0, ctx.stream>>>((uint32_t*)dst, dst_off, src, src_off, n);
    LAUNCH_CHECK(ctx);
}
__global__ void set_bits_kernel(uint32_t* __restrict__ dst, int64_t off, int64_t n) {
    int64_t first_word = off >> 5, last_word = (off + n - 1) >> 5;
    int64_t w = first_word + (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (w > last_word) return;
    int64_t lo = max(w * 32, off), hi = min(w * 32 + 32, off + n);
    uint32_t v = (hi - lo == 32) ? 0xffffffffu : (((1u << (hi - lo)) - 1u) << (lo & 31));
    atomicOr(&dst[w], v);
}
static void set_bits(Ctx& ctx, uint8_t* dst, int64_t off, int64_t n) {
    if (n <= 0) return;
    int64_t words = ((off + n - 1) >> 5) - (off >> 5) + 1;
    set_bits_kernel<<<(unsigned)((words + 255) / 256), 256, 0, ctx.stream>>>((uint32_t*)dst, off, n);
    LAUNCH_CHECK(ctx);
}

__global__ void iota_kernel(int32_t* out, int64_t n, int32_t start) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = start + (int32_t)i;
}
void fill_iota_i32(Ctx& ctx, int32_t* out, int64_t n, int32_t start) {
    if (n <= 0) return;
    iota_kernel<<<(unsigned)((n + 255) / 256), 256, 0, ctx.stream>>>(out, n, start);
    LAUNCH_CHECK(ctx);
}
__global__ void and_words_kernel(const uint32_t* a, const uint32_t* b, uint32_t* out, int64_t nw) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < nw) out[i] = (a ? a[i] : 0xffffffffu) & (b ? b[i] : 0xffffffffu);
}
Buf and_bitmaps(Ctx& ctx, const uint8_t* a, const uint8_t* b, int64_t n_bits) {
    if (!a && !b) return nullptr;
    int64_t nw = (n_bits + 31) / 32;
    Buf out = dalloc(ctx, nw * 4);
    if (nw) {
        and_words_kernel<<<(unsigned)((nw + 255) / 256), 256, 0, ctx.stream>>>((const uint32_t*)a, (const uint32_t*)b, P<uint32_t>(out), nw);
        LAUNCH_CHECK(ctx);
    }
    return out;
}

// ---------------------------------------------------------------------------------------------
// gather (take).  Each thread owns one output row; validity words come from a warp ballot, so a
// CTA's rows must start on a multiple of 32 (they do: 256 rows per CTA).
// ---------------------------------------------------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(256) take_fixed_kernel(const T* __restrict__ in, const uint8_t* __restrict__ in_valid,
                                                         const int32_t* __restrict__ idx, int64_t n_out, T* __restrict__ out,
                                                         uint32_t* __restrict__ out_valid) {
    int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x;
    bool ok = false;
    if (i < n_out) {
        int64_t src = idx ? (int64_t)idx[i] : i;
        ok = src >= 0 && valid_at(in_valid, src);
        T v;
        if (src >= 0) v = in[src];
        else memset(&v, 0, sizeof(T));
        out[i] = v;
    }
    if (out_valid) {
        uint32_t word = __ballot_sync(FULL_MASK, ok);
        if (lane_id() == 0 && i < n_out) out_valid[i >> 5] = word;
    }
}
__global__ void __launch_bounds__(256) take_bool_kernel(const uint8_t* __restrict__ in_bits, const uint8_t* __restrict__ in_valid,
                                                        const int32_t* __restrict__ idx, int64_t n_out, uint32_t* __restrict__ out_bits,
                                                        uint32_t* __restrict__ out_valid) {
    int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x;
    bool ok = false, v = false;
    if (i < n_out) {
        int64_t src = idx ? (int64_t)idx[i] : i;
        ok = src >= 0 && valid_at(in_valid, src);
        v = src >= 0 && bit_get(in_bits, src);
    }
    uint32_t wv = __ballot_sync(FULL_MASK, v), wk = __ballot_sync(FULL_MASK, ok);
    if (lane_id() == 0 && i < n_out) {
        out_bits[i >> 5] = wv;
        if (out_valid) out_valid[i >> 5] = wk;
    }
}
__global__ void __launch_bounds__(256) take_lens_kernel(const int32_t* __restrict__ in_off, const uint8_t* __restrict__ in_valid,
                                                        const int32_t* __restrict__ idx, int64_t n_out, int64_t* __restrict__ lens,
                                                        uint32_t* __restrict__ out_valid) {
    int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x;
    bool ok = false;
    if (i < n_out) {
        int64_t src = idx ? (int64_t)idx[i] : i;
        ok = src >= 0 && valid_at(in_valid, src);
        lens[i] = src >= 0 ? (int64_t)(in_off[src + 1] - in_off[src]) : 0;
    }
    if (out_valid) {
        uint32_t word = __ballot_sync(FULL_MASK, ok);
        if (lane_id() == 0 && i < n_out) out_valid[i >> 5] = word;
    }
}
__global__ void narrow_offsets_kernel(const int64_t* __restrict__ off64, int32_t* __restrict__ off32, int64_t n_plus_1) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n_plus_1) off32[i] = (int32_t)off64[i];
}
// one thread per output row copies its bytes; rows are short (tens of bytes) on this path
__global__ void __launch_bounds__(256) take_bytes_kernel(const int32_t* __restrict__ in_off, const uint8_t* __restrict__ in_data,
                                                         const int32_t* __restrict__ idx, int64_t n_out,
                                                         const int32_t* __restrict__ out_off, uint8_t* __restrict__ out_data) {
    int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x;
    if (i >= n_out) return;
    int64_t src = idx ? (int64_t)idx[i] : i;
    if (src < 0) return;
    const uint8_t* s = in_data + in_off[src];
    uint8_t* d = out_data + out_off[i];
    int32_t len = out_off[i + 1] - out_off[i];
    for (int32_t k = 0; k < len; k++) d[k] = s[k];
}

// list rows: the element count of row idx[i]; a NULL row counts as empty (Arrow lets it cover a range of the child)
__global__ void __launch_bounds__(256) list_lens_kernel(const int32_t* __restrict__ in_off, const uint8_t* __restrict__ in_valid,
                                                        const int32_t* __restrict__ idx, int64_t n_out, int64_t* __restrict__ lens,
                                                        uint32_t* __restrict__ out_valid) {
    int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x;
    bool ok = false;
    if (i < n_out) {
        int64_t src = idx ? (int64_t)idx[i] : i;
        ok = src >= 0 && valid_at(in_valid, src);
        lens[i] = ok ? (int64_t)(in_off[src + 1] - in_off[src]) : 0;
    }
    if (out_valid) {
        uint32_t word = __ballot_sync(FULL_MASK, ok);
        if (lane_id() == 0 && i < n_out) out_valid[i >> 5] = word;
    }
}
// row of output element j: the last i with out_off[i] <= j among rows that own elements
__device__ __forceinline__ int64_t row_of_offset(const int32_t* __restrict__ off, int64_t n, int64_t j) {
    int64_t lo = 0, hi = n;   // off[lo] <= j < off[hi]
    while (hi - lo > 1) {
        int64_t mid = (lo + hi) >> 1;
        if ((int64_t)off[mid] <= j) lo = mid;
        else hi = mid;
    }
    return lo;
}
__global__ void __launch_bounds__(256) list_elem_index_kernel(const int32_t* __restrict__ in_off, const int32_t* __restrict__ idx,
                                                              const int32_t* __restrict__ out_off, int64_t n_out, int64_t total,
                                                              int32_t* __restrict__ eidx) {
    int64_t j = (int64_t)blockIdx.x * 256 + threadIdx.x;
    if (j >= total) return;
    int64_t i = row_of_offset(out_off, n_out, j);
    int64_t src = idx ? (int64_t)idx[i] : i;
    eidx[j] = in_off[src] + (int32_t)(j - out_off[i]);
}

struct alignas(16) u128_t {
    uint64_t a, b;
};

ColumnPtr take(Ctx& ctx, const Column& in, const int32_t* idx, int64_t n_out, bool idx_may_be_negative) {
    ProfScope ps(ctx, "take");
    auto out = std::make_shared<Column>();
    out->type = in.type;
    out->len = n_out;
    bool need_valid = in.may_have_nulls() || idx_may_be_negative;
    if (in.type.id == T_NULL) {
        out->null_count = n_out;
        return out;
    }
    if (need_valid) {
        out->validity = dalloc(ctx, bitmap_alloc_bytes(n_out));
        out->null_count = -1;
    }
    uint32_t* ov = P<uint32_t>(out->validity);
    unsigned blocks = (unsigned)((n_out + 255) / 256);
    if (n_out == 0) blocks = 0;
    int w = in.type.width();
    if (in.type.id == T_BOOL) {
        out->data = dalloc(ctx, bitmap_alloc_bytes(n_out));
        if (blocks) {
            take_bool_kernel<<<blocks, 256, 0, ctx.stream>>>(P<uint8_t>(in.data), in.vbits(), idx, n_out, P<uint32_t>(out->data), ov);
            LAUNCH_CHECK(ctx);
        }
    } else if (w > 0) {
        out->data = dalloc(ctx, (size_t)n_out * w);
        if (blocks) {
            switch (w) {
                case 1: take_fixed_kernel<uint8_t><<<blocks, 256, 0, ctx.stream>>>(P<uint8_t>(in.data), in.vbits(), idx, n_out, P<uint8_t>(out->data), ov); break;
                case 2: take_fixed_kernel<uint16_t><<<blocks, 256, 0, ctx.stream>>>(P<uint16_t>(in.data), in.vbits(), idx, n_out, P<uint16_t>(out->data), ov); break;
                case 4: take_fixed_kernel<uint32_t><<<blocks, 256, 0, ctx.stream>>>(P<uint32_t>(in.data), in.vbits(), idx, n_out, P<uint32_t>(out->data), ov); break;
                case 8: take_fixed_kernel<uint64_t><<<blocks, 256, 0, ctx.stream>>>(P<uint64_t>(in.data), in.vbits(), idx, n_out, P<uint64_t>(out->data), ov); break;
                case 16: take_fixed_kernel<u128_t><<<blocks, 256, 0, ctx.stream>>>(P<u128_t>(in.data), in.vbits(), idx, n_out, P<u128_t>(out->data), ov); break;
                default: fail("take: unsupported width");
            }
            LAUNCH_CHECK(ctx);
        }
    } else if (in.type.is_varlen()) {
        Buf lens = dalloc(ctx, (size_t)(n_out + 1) * 8);
        out->offsets = dalloc(ctx, (size_t)(n_out + 1) * 4);
        int64_t total = 0;
        if (blocks) {
            take_lens_kernel<<<blocks, 256, 0, ctx.stream>>>(P<int32_t>(in.offsets), in.vbits(), idx, n_out, P<int64_t>(lens), ov);
            LAUNCH_CHECK(ctx);
            exclusive_scan_i64(ctx, P<int64_t>(lens), P<int64_t>(lens), n_out, P<int64_t>(lens) + n_out);
            narrow_offsets_kernel<<<(unsigned)((n_out + 1 + 255) / 256), 256, 0, ctx.stream>>>(P<int64_t>(lens), P<int32_t>(out->offsets), n_out + 1);
            LAUNCH_CHECK(ctx);
            to_host(ctx, &total, P<int64_t>(lens) + n_out, 8);
            AURON_CHECK(total <= (int64_t)INT32_MAX, "utf8 column exceeds 2 GiB in one batch");
        } else {
            CUDA_OK(cudaMemsetAsync(out->offsets->ptr, 0, 4, ctx.stream));
        }
        out->data = dalloc(ctx, (size_t)total);
        out->data_bytes = total;
        if (blocks && total > 0) {
            take_bytes_kernel<<<blocks, 256, 0, ctx.stream>>>(P<int32_t>(in.offsets), P<uint8_t>(in.data), idx, n_out, P<int32_t>(out->offsets), P<uint8_t>(out->data));
            LAUNCH_CHECK(ctx);
        }
    } else if (in.type.id == T_LIST) {
        out->offsets = dalloc(ctx, (size_t)(n_out + 1) * 4);
        int64_t total = 0;
        Buf lens = dalloc(ctx, (size_t)(n_out + 1) * 8);
        if (blocks) {
            list_lens_kernel<<<blocks, 256, 0, ctx.stream>>>(P<int32_t>(in.offsets), in.vbits(), idx, n_out, P<int64_t>(lens), ov);
            LAUNCH_CHECK(ctx);
            exclusive_scan_i64(ctx, P<int64_t>(lens), P<int64_t>(lens), n_out, P<int64_t>(lens) + n_out);
            narrow_offsets_kernel<<<(unsigned)((n_out + 1 + 255) / 256), 256, 0, ctx.stream>>>(P<int64_t>(lens), P<int32_t>(out->offsets), n_out + 1);
            LAUNCH_CHECK(ctx);
            to_host(ctx, &total, P<int64_t>(lens) + n_out, 8);
            AURON_CHECK(total <= (int64_t)INT32_MAX, "list column of " + std::to_string(total) + " elements exceeds 2^31 - 1 elements in one batch");
        } else {
            CUDA_OK(cudaMemsetAsync(out->offsets->ptr, 0, 4, ctx.stream));
        }
        // the element each output element copies: one thread per output element finds its row by a search over the new offsets
        Buf eidx = dalloc(ctx, (size_t)std::max<int64_t>(total, 1) * 4);
        if (total > 0) {
            list_elem_index_kernel<<<(unsigned)((total + 255) / 256), 256, 0, ctx.stream>>>(P<int32_t>(in.offsets), idx, P<int32_t>(out->offsets), n_out,
                                                                                            total, P<int32_t>(eidx));
            LAUNCH_CHECK(ctx);
        }
        out->child = take(ctx, *in.child, P<int32_t>(eidx), total, false);
    } else {
        fail("take: unsupported type " + in.type.str());
    }
    return out;
}

BatchPtr take_batch(Ctx& ctx, const Batch& in, const int32_t* idx, int64_t n_out, bool neg) {
    auto out = std::make_shared<Batch>();
    out->num_rows = n_out;
    for (auto& c : in.cols) out->cols.push_back(take(ctx, *c, idx, n_out, neg));
    return out;
}

__global__ void rebase_offsets_kernel(const int32_t* __restrict__ in, int64_t n_plus_1, int32_t delta, int32_t* __restrict__ out) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n_plus_1) out[i] = in[i] + delta;
}

ColumnPtr concat_columns(Ctx& ctx, const std::vector<ColumnPtr>& cols) {
    AURON_CHECK(!cols.empty(), "concat of nothing");
    if (cols.size() == 1) return cols[0];
    int64_t total = 0, total_bytes = 0;
    bool any_valid = false;
    for (auto& c : cols) {
        total += c->len;
        total_bytes += c->data_bytes;
        any_valid |= c->may_have_nulls();
    }
    auto out = std::make_shared<Column>();
    out->type = cols[0]->type;
    out->len = total;
    int w = out->type.width();
    if (any_valid) {
        out->validity = dalloc_zero(ctx, bitmap_alloc_bytes(total));
        out->null_count = -1;
    }
    if (out->type.id == T_BOOL) out->data = dalloc_zero(ctx, bitmap_alloc_bytes(total));
    else if (w > 0) out->data = dalloc(ctx, (size_t)total * w);
    else if (out->type.is_varlen()) {
        AURON_CHECK(total_bytes <= (int64_t)INT32_MAX, "utf8 column exceeds 2 GiB in one batch");
        out->offsets = dalloc(ctx, (size_t)(total + 1) * 4);
        out->data = dalloc(ctx, (size_t)total_bytes);
        out->data_bytes = total_bytes;
    } else if (out->type.id == T_LIST) {
        int64_t elems = 0;
        std::vector<ColumnPtr> kids;
        for (auto& c : cols) {
            elems += c->child->len;
            kids.push_back(c->child);
        }
        AURON_CHECK(elems <= (int64_t)INT32_MAX, "list column of " + std::to_string(elems) + " elements exceeds 2^31 - 1 elements in one batch");
        out->offsets = dalloc(ctx, (size_t)(total + 1) * 4);
        out->child = concat_columns(ctx, kids);
    }
    int64_t row = 0, byte = 0;
    for (auto& c : cols) {
        if (c->len == 0) continue;
        if (any_valid) {
            if (c->may_have_nulls()) copy_bits(ctx, P<uint8_t>(out->validity), row, c->vbits(), 0, c->len);
            else set_bits(ctx, P<uint8_t>(out->validity), row, c->len);
        }
        if (out->type.id == T_BOOL) copy_bits(ctx, P<uint8_t>(out->data), row, P<uint8_t>(c->data), 0, c->len);
        else if (w > 0)
            CUDA_OK(cudaMemcpyAsync(P<uint8_t>(out->data) + row * w, c->data->ptr, (size_t)c->len * w, cudaMemcpyDeviceToDevice, ctx.stream));
        else if (out->type.is_varlen()) {
            rebase_offsets_kernel<<<(unsigned)((c->len + 1 + 255) / 256), 256, 0, ctx.stream>>>(P<int32_t>(c->offsets), c->len + 1, (int32_t)byte,
                                                                                              P<int32_t>(out->offsets) + row);
            LAUNCH_CHECK(ctx);
            if (c->data_bytes)
                CUDA_OK(cudaMemcpyAsync(P<uint8_t>(out->data) + byte, c->data->ptr, (size_t)c->data_bytes, cudaMemcpyDeviceToDevice, ctx.stream));
            byte += c->data_bytes;
        } else if (out->type.id == T_LIST) {
            rebase_offsets_kernel<<<(unsigned)((c->len + 1 + 255) / 256), 256, 0, ctx.stream>>>(P<int32_t>(c->offsets), c->len + 1, (int32_t)byte,
                                                                                              P<int32_t>(out->offsets) + row);
            LAUNCH_CHECK(ctx);
            byte += c->child->len;
        }
        row += c->len;
    }
    if ((out->type.is_varlen() || out->type.id == T_LIST) && total == 0) CUDA_OK(cudaMemsetAsync(out->offsets->ptr, 0, 4, ctx.stream));
    return out;
}

BatchPtr concat_batches(Ctx& ctx, const std::vector<BatchPtr>& batches) {
    AURON_CHECK(!batches.empty(), "concat of nothing");
    if (batches.size() == 1) return batches[0];
    auto out = std::make_shared<Batch>();
    size_t nc = batches[0]->cols.size();
    for (auto& b : batches) out->num_rows += b->num_rows;
    for (size_t c = 0; c < nc; c++) {
        std::vector<ColumnPtr> cs;
        for (auto& b : batches) cs.push_back(b->cols[c]);
        out->cols.push_back(concat_columns(ctx, cs));
    }
    return out;
}

ColumnPtr slice_column(Ctx& ctx, const Column& in, int64_t off, int64_t len) {
    AURON_CHECK(off >= 0 && len >= 0 && off + len <= in.len, "slice out of range");
    Buf idx = dalloc(ctx, (size_t)std::max<int64_t>(len, 1) * 4);
    fill_iota_i32(ctx, P<int32_t>(idx), len, (int32_t)off);
    return take(ctx, in, P<int32_t>(idx), len, false);
}
BatchPtr slice_batch(Ctx& ctx, const Batch& in, int64_t off, int64_t len) {
    Buf idx = dalloc(ctx, (size_t)std::max<int64_t>(len, 1) * 4);
    fill_iota_i32(ctx, P<int32_t>(idx), len, (int32_t)off);
    return take_batch(ctx, in, P<int32_t>(idx), len, false);
}

}  // namespace auron

namespace auron {
__global__ void not_words_kernel(const uint32_t* a, uint32_t* out, int64_t nw) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < nw) out[i] = ~a[i];
}
Buf not_bitmap(Ctx& ctx, const uint8_t* a, int64_t n_bits) {
    int64_t nw = (n_bits + 31) / 32;
    Buf out = dalloc(ctx, std::max<int64_t>(nw, 1) * 4);
    if (nw) {
        not_words_kernel<<<(unsigned)((nw + 255) / 256), 256, 0, ctx.stream>>>((const uint32_t*)a, P<uint32_t>(out), nw);
        LAUNCH_CHECK(ctx);
    }
    return out;
}
}  // namespace auron
