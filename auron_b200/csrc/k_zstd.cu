// k_zstd.cu -- ZSTD and LZ4_RAW Parquet pages decompressed on the device (row P1 of SURVEY.md section 8a; the reference
// decompresses every page with the `zstd` / `lz4_flex` crates on a CPU core, parquet_exec.rs:175-197).
//
// A ZSTD page body is a sequence of frames; a frame is a sequence of blocks of at most 128 KB; a compressed block holds Huffman-coded
// literals and FSE-coded sequences (literal length, match length, offset).  Entropy decoding is serial within a block and blocks
// depend on the tables and repeat offsets of the blocks before them, so the unit of parallelism is the page: ONE WARP PER PAGE, the
// decoder of zstd_dec.cuh with its tables in shared memory (14.8 KB per warp, two warps per CTA: 29.7 KB per CTA; ptxas for sm_90a:
// 102 registers, a 200-byte stack frame, no spills, so shared memory bounds residency at seven CTAs = 14 warps per SM).  Within the warp the four Huffman streams of a block decode on four lanes and every literal and
// match copy is cooperative (warp_copy, the overlapping-run pattern of k_lz4.cu).
//
// An LZ4_RAW page is one raw LZ4 block: lz4_decompress_blocks (k_lz4.cu, written for the shuffle reader) decodes it, and a check
// pass turns a wrong decoded length into the status word.
//
// Roofline: HBM-bound in the limit, algorithmic bytes = compressed bytes in + uncompressed bytes out; in practice the serial
// entropy decoding of one warp per page bounds it (profiles/h100_parquet_zstd.txt).
#include "device_utils.cuh"
#include "kernels.h"
#include "parquet_dev.h"
#include "zstd_dec.cuh"

namespace auron {

#define LAUNCH_CHECK(ctx)            \
    do {                             \
        CUDA_OK(cudaGetLastError()); \
        launch_count(ctx);           \
    } while (0)

constexpr int ZS_WARPS = 2;

// jobs[0, n) of kinds PQ_JOB_STORED / PQ_JOB_ZSTD / PQ_JOB_LZ4 (the last decoded by lz4_decompress_blocks); job0 = index of jobs[0] in
// the batch's job list, for the status word (1 + index of a failing job) and the results (no value section is ever left in place)
__global__ void __launch_bounds__(32 * ZS_WARPS) pq_zstd_kernel(const PqDecompJob* __restrict__ jobs, int n, int job0, int32_t* __restrict__ status,
                                                                PqDecompResult* __restrict__ results) {
    __shared__ zd::Tables s_tables[ZS_WARPS];
    const int j = blockIdx.x * ZS_WARPS + (int)(threadIdx.x >> 5);
    if (j >= n) return;
    const unsigned lane = threadIdx.x & 31;
    const PqDecompJob jb = jobs[j];
    if (lane == 0) results[job0 + j] = PqDecompResult{nullptr, -1, 0};
    if (jb.kind == PQ_JOB_STORED) {
        warp_copy(jb.dst, jb.src, jb.dst_len, lane);
        return;
    }
    if (jb.kind != PQ_JOB_ZSTD) return;
    const int64_t r = zd::decompress(jb.src, jb.src_len, jb.dst, jb.dst_len, &s_tables[threadIdx.x >> 5], lane, 32);
    if (r != jb.dst_len && lane == 0) atomicCAS(status, 0, job0 + j + 1);
}

// LZ4_RAW pages: the decoded length must be the page's
__global__ void pq_lz4_check_kernel(const PqDecompJob* __restrict__ jobs, const int32_t* __restrict__ job_idx, const int32_t* __restrict__ sizes, int n,
                                    int32_t* __restrict__ status) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int j = job_idx[i];
    if (sizes[i] != jobs[j].dst_len) atomicCAS(status, 0, j + 1);
}

void pq_decompress_zstd_lz4(Ctx& ctx, const std::vector<PqDecompJob>& jobs, size_t first, const PqDecompJob* dev_jobs, int32_t* status,
                            PqDecompResult* results) {
    const size_t n = jobs.size() - first;
    if (n == 0) return;
    {
        ProfScope ps(ctx, "pq_zstd");
        pq_zstd_kernel<<<(unsigned)((n + ZS_WARPS - 1) / ZS_WARPS), 32 * ZS_WARPS, 0, ctx.stream>>>(dev_jobs + first, (int)n, (int)first, status, results);
        LAUNCH_CHECK(ctx);
    }
    std::vector<Lz4DBlock> blocks;
    std::vector<int32_t> idx;
    for (size_t j = first; j < jobs.size(); j++)
        if (jobs[j].kind == PQ_JOB_LZ4) {
            blocks.push_back(Lz4DBlock{jobs[j].src, jobs[j].dst, jobs[j].src_len, jobs[j].dst_len, 0, 0});
            idx.push_back((int32_t)j);
        }
    if (blocks.empty()) return;
    Buf db = to_device(ctx, blocks.data(), blocks.size() * sizeof(Lz4DBlock));
    Buf di = to_device(ctx, idx.data(), idx.size() * sizeof(int32_t));
    Buf sizes = dalloc(ctx, blocks.size() * sizeof(int32_t));
    lz4_decompress_blocks(ctx, P<Lz4DBlock>(db), (int)blocks.size(), P<int32_t>(sizes));
    pq_lz4_check_kernel<<<(unsigned)((blocks.size() + 255) / 256), 256, 0, ctx.stream>>>(dev_jobs, P<int32_t>(di), P<int32_t>(sizes), (int)blocks.size(), status);
    LAUNCH_CHECK(ctx);
}

int64_t zstd_decompress_host(const uint8_t* in, int64_t in_len, uint8_t* out, int64_t out_len) {
    std::unique_ptr<zd::Tables> t(new zd::Tables);
    return zd::decompress(in, in_len, out, out_len, t.get(), 0, 1);
}

}  // namespace auron
