// k_snappy.cu -- Parquet page decompression on device (row P1 of SURVEY.md section 8a: the `parquet` crate decompresses
// every page with the `snap` crate on a CPU core before decoding it; call site parquet_exec.rs:175-197).
//
// Spark writes SNAPPY pages by default.  A page is an independent Snappy raw block (no framing): a varint with the
// uncompressed length, then a sequence of elements -- literals (copy the next L bytes of the input) and back references
// (copy L bytes that start `offset` bytes before the current output position).  Elements are inherently serial, so the
// unit of parallelism is the page: ONE WARP PER PAGE.  All 32 lanes read the same tag bytes (uniform, broadcast loads, no
// divergence) and then move the element's bytes cooperatively:
//   * literals: 16-byte vectors at the destination's alignment, the source re-aligned with funnel shifts (512 B per
//     warp instruction); short references byte-wise;
//   * overlapping references (offset < length, i.e. a repeated pattern): byte i of the run is out[pos - offset + i % offset],
//     every source byte is already written, so all lanes proceed in parallel as well.
// Dictionary-encoded, bit-packed index pages are close to incompressible: their Snappy form is a handful of 64 KB literals
// and the kernel runs at copy speed; highly repetitive pages are bound by the per-element tag latency instead.
//
// Roofline: HBM-bound copy, algorithmic bytes = compressed bytes in + uncompressed bytes out.
#include "device_utils.cuh"
#include "kernels.h"
#include "parquet_dev.h"

namespace auron {

#define LAUNCH_CHECK(ctx)            \
    do {                             \
        CUDA_OK(cudaGetLastError()); \
        launch_count(ctx);           \
    } while (0)

// status: 0 ok, else 1 + index of the first failing job
//
// Back references read bytes this warp wrote a few elements earlier.  Through global memory that is a store followed by a
// dependent load of the same line (an L2 round trip per element; the level prefixes of the SF100 bench are ~400 short
// elements each).  So every short element is ALSO written into a per-warp shared-memory ring holding the
// last SN_RING output bytes, and references that fall inside the ring are served from it; long literals bypass the ring
// (ring_from marks the first output position the ring is valid from).
constexpr int SN_RING = 4096;
// Where the prefix pass (below) left a job: ip < 0 = finished there, ip == 0 = not started (the warp parses the preamble),
// else resume at input offset ip / output offset op.
struct PqDecompState {
    int32_t ip, op;
};

// ---- prefix pass: FOUR LANES per nullable-v1-page job (eight jobs per warp).  The body of such a page is [u32 length][definition
// levels][values]; with dictionary-encoded values the Snappy stream is a few hundred tiny elements for the level bytes (4..8 bytes
// each: the level runs repeat) followed by one literal that holds the value section.  A warp per job executed every one of those
// elements 32-fold redundantly, so the kernel was bound by instruction issue.  An element offers
// a few bytes of parallelism, a launch offers one job per page, so a warp now advances eight streams at once, each by one
// element per iteration, with a 1 KB shared-memory ring per stream for the back references.  (One THREAD per stream would put
// 32 unrelated byte streams behind each load instruction and thrash L1.)  A job that does not have the
// expected shape within the budget (long literal in the middle, far back reference, large output) is handed to the warp kernel
// below, which resumes it from the recorded offsets.
constexpr int SN_TEAM = 4, SN_TEAMS = 32 / SN_TEAM, SN_TRING = 512, SN_WIN = 256;
constexpr int SN_PREFIX_MAX_OUT = 48 * 1024, SN_PREFIX_MAX_ELEMS = 12000;
__global__ void __launch_bounds__(128) pq_decompress_prefix_kernel(const PqDecompJob* __restrict__ jobs, int n_jobs, int32_t* __restrict__ status,
                                                                   PqDecompResult* __restrict__ results, PqDecompState* __restrict__ states) {
    __shared__ uint8_t s_ring[4][SN_TEAMS][SN_TRING];
    // The compressed bytes are read through a 256-byte window per stream, refilled with 16-byte loads: with 40 KB of shared memory
    // per CTA the SM has next to no L1 left, and byte loads straight from global memory paid an L2 round trip each (every
    // element three dependent L2 accesses).
    __shared__ uint4 s_win[4][SN_TEAMS][SN_WIN / 16];
    const unsigned lane = threadIdx.x & 31, team = lane / SN_TEAM, sub = lane % SN_TEAM;
    const int job = (blockIdx.x * 4 + (threadIdx.x >> 5)) * SN_TEAMS + (int)team;
    uint8_t* ring = s_ring[threadIdx.x >> 5][team];
    uint4* win4 = s_win[threadIdx.x >> 5][team];
    const uint8_t* win = (const uint8_t*)win4;
    bool active = false;
    const uint8_t* __restrict__ src = nullptr;
    uint8_t* dst = nullptr;
    int n_in = 0, n_out = 0, ip = 0, op = 0, elems = 0;
    int wbase = 0;   // input offset of win[0]
    bool have_win = false, head_only = false;   // head_only: the job is the front part of a block (its preamble counts the whole block)
    if (job < n_jobs) {
        const PqDecompJob jb = jobs[job];
        if (sub == 0) {
            results[job] = PqDecompResult{nullptr, -1, 0};
            states[job] = PqDecompState{0, 0};
        }
        if (jb.kind >= 1 && jb.v1_levels) {
            active = true;
            head_only = jb.kind == 2;
            src = jb.src;
            dst = jb.dst;
            n_in = jb.src_len;
            n_out = jb.dst_len;
        }
    }
    __syncwarp();   // the state records above are written before any lane of the team overwrites them below
    uint32_t head = 0;        // the body's first four bytes (the length of the level section), read from the ring before it wraps
    bool have_head = false, preamble = true;
    while (__any_sync(FULL_MASK, active)) {
        // ---- refill the input window when fewer than 136 bytes of it lie ahead (an element: <= 5 header bytes + <= 128 literal bytes)
        const bool refill = active && (!have_win || ip - wbase > SN_WIN - 136);
        if (refill) {
            const uintptr_t g = (uintptr_t)(src + ip), ga = g & ~(uintptr_t)15;
            wbase = ip - (int)(g - ga);
            const uint8_t* lim = src + n_in + 16;
#pragma unroll
            for (int j = 0; j < SN_WIN / 16 / SN_TEAM; j++) {
                const int q = j * SN_TEAM + (int)sub;
                const uint8_t* a = (const uint8_t*)ga + 16 * q;
                win4[q] = a < lim ? *(const uint4*)a : make_uint4(0, 0, 0, 0);
            }
            have_win = true;
        }
        __syncwarp();
        if (active) {
#define SN_RD(pos) ((uint32_t)win[(pos) - wbase])
            if (preamble) {   // uncompressed length (a malformed one is left to the warp kernel, which reports it)
                preamble = false;
                uint32_t v = 0;
                int shift = 0;
                for (;;) {
                    if (ip >= n_in || shift > 28) {
                        active = false;
                        break;
                    }
                    const uint32_t b = SN_RD(ip);
                    ip++;
                    v |= (b & 0x7f) << shift;
                    if (!(b & 0x80)) break;
                    shift += 7;
                }
                if (active && (head_only ? (int)v < n_out : (int)v != n_out)) active = false;
            }
        }
        if (active) {
            if (!have_head && op >= 4 && op <= SN_TRING) {
                head = (uint32_t)ring[0] | ((uint32_t)ring[1] << 8) | ((uint32_t)ring[2] << 16) | ((uint32_t)ring[3] << 24);
                have_head = true;
            }
            const int ip0 = ip;
            bool bad = false, handoff = false;
            if (ip >= n_in) {
                active = false;
                if (op == n_out) {
                    if (sub == 0) states[job] = PqDecompState{-1, 0};
                } else bad = true;
            } else if (op >= SN_PREFIX_MAX_OUT || elems++ >= SN_PREFIX_MAX_ELEMS) {
                handoff = true;
            } else if ([&]() {
                           // ---- fast path, the same instruction stream for every element type (the eight streams of the warp are at
                           // different kinds of elements: separate literal / copy branches serialise): short literal, or a 1- / 2-byte-
                           // offset copy whose source is still in the ring
                           const uint32_t tag = SN_RD(ip), kind = tag & 3, b1 = SN_RD(ip + 1), b2 = SN_RD(ip + 2);
                           const bool is_lit = kind == 0;
                           const int len = kind == 1 ? 4 + (int)((tag >> 2) & 7) : (int)(tag >> 2) + 1;
                           const int hdr = is_lit ? 1 : (kind == 1 ? 2 : 3);
                           const int off = kind == 1 ? (int)(((tag >> 5) << 8) | b1) : (int)(b1 | (b2 << 8));
                           const bool ok = kind != 3 && len <= n_out - op &&
                                           (is_lit ? (len <= 60 && ip + 1 + len <= n_in) : (ip + hdr <= n_in && off > 0 && off <= op && off <= SN_TRING - 64));
                           if (!ok) return false;
                           const uint8_t* sbase = is_lit ? win + (ip + 1 - wbase) : ring;
                           const int from = op - off;
                           for (int i = (int)sub; i < len; i += SN_TEAM) {
                               const int si = is_lit ? i : ((from + (off >= len ? i : (int)((unsigned)i % (unsigned)off))) & (SN_TRING - 1));
                               const uint8_t c = sbase[si];
                               dst[op + i] = c;
                               ring[(op + i) & (SN_TRING - 1)] = c;
                           }
                           ip += is_lit ? 1 + len : hdr;
                           op += len;
                           return true;
                       }()) {
            } else {
                const uint32_t tag = SN_RD(ip);
                ip++;
                const uint32_t kind = tag & 3;
                if (kind == 0) {
                    int len = (int)(tag >> 2) + 1;
                    if (len > 60) {
                        const int nb = len - 60;
                        if (ip + nb > n_in) bad = true;
                        else {
                            uint32_t v = 0;
                            for (int k = 0; k < nb; k++) v |= SN_RD(ip + k) << (8 * k);
                            ip += nb;
                            if (v >= 0x7fffffffu) bad = true;
                            len = (int)v + 1;
                        }
                    }
                    if (!bad && (len > n_in - ip || len > n_out - op)) bad = true;
                    if (!bad) {
                        if (len > 128) {
                            // the literal that holds the value section: only the level bytes that spill into it are copied (see the
                            // warp kernel); anything else of that size is the warp kernel's business
                            handoff = true;
                            if (ip + len == n_in && op + len == n_out && have_head) {
                                const int64_t val_off = 4 + (int64_t)head;
                                const int64_t keep = val_off - op;
                                if (keep >= 0 && keep <= 512 && len - keep >= 256) {
                                    for (int i = (int)sub; i < (int)keep; i += SN_TEAM) dst[op + i] = src[ip + i];
                                    if (sub == 0) {
                                        results[job] = PqDecompResult{src + ip + keep, (int32_t)val_off, 0};
                                        states[job] = PqDecompState{-1, 0};
                                    }
                                    handoff = false;
                                    active = false;
                                }
                            }
                            if (handoff) ip = ip0;
                        } else {
                            for (int i = (int)sub; i < len; i += SN_TEAM) {
                                const uint8_t c = (uint8_t)SN_RD(ip + i);
                                dst[op + i] = c;
                                ring[(op + i) & (SN_TRING - 1)] = c;
                            }
                            ip += len;
                            op += len;
                        }
                    }
                } else {
                    int len = 0, off = 0;
                    if (kind == 1) {
                        if (ip + 1 > n_in) bad = true;
                        else {
                            len = 4 + (int)((tag >> 2) & 7);
                            off = (int)(((tag >> 5) << 8) | SN_RD(ip));
                            ip += 1;
                        }
                    } else if (kind == 2) {
                        if (ip + 2 > n_in) bad = true;
                        else {
                            len = (int)(tag >> 2) + 1;
                            off = (int)(SN_RD(ip) | (SN_RD(ip + 1) << 8));
                            ip += 2;
                        }
                    } else {
                        if (ip + 4 > n_in) bad = true;
                        else {
                            len = (int)(tag >> 2) + 1;
                            const uint32_t o4 = SN_RD(ip) | (SN_RD(ip + 1) << 8) | (SN_RD(ip + 2) << 16) | (SN_RD(ip + 3) << 24);
                            if (o4 > 0x7fffffffu) bad = true;
                            off = (int)o4;
                            ip += 4;
                        }
                    }
                    if (!bad && (off <= 0 || off > op || len > n_out - op)) bad = true;
                    if (!bad) {
                        if (off > SN_TRING - 64) {
                            // the source left the ring (a dozen elements per page reach back further than 1 KB): read it back from
                            // global memory.  Those bytes were stored by this team before earlier __syncwarp barriers, which order
                            // them for the warp; ld.cg goes to L2, past any stale L1 line.
                            const uint8_t* from = dst + op - off;
                            for (int i = (int)sub; i < len; i += SN_TEAM) {
                                const int k = off >= len ? i : (int)((unsigned)i % (unsigned)off);
                                const uint8_t c = __ldcg(from + k);
                                dst[op + i] = c;
                                ring[(op + i) & (SN_TRING - 1)] = c;
                            }
                            op += len;
                        } else {
                            const int from = op - off;
                            // byte i of the run is out[from + i % off]: every source byte is older than this element, so the four
                            // lanes copy in parallel; a ring slot written here (op + i) is never one read here (off + len <= ring size)
                            for (int i = (int)sub; i < len; i += SN_TEAM) {
                                const int k = off >= len ? i : (int)((unsigned)i % (unsigned)off);
                                const uint8_t c = ring[(from + k) & (SN_TRING - 1)];
                                dst[op + i] = c;
                                ring[(op + i) & (SN_TRING - 1)] = c;
                            }
                            op += len;
                        }
                    }
                }
            }
#undef SN_RD
            if (bad) {
                if (sub == 0) atomicCAS(status, 0, job + 1);
                active = false;
            } else if (handoff) {
                if (sub == 0) states[job] = PqDecompState{ip, op};
                active = false;
            }
        }
        __syncwarp();   // ring bytes of this element are visible to the team before the next one reads them
    }
}

// ---- prefix pass, one THREAD per job (alternative to the teams above, off by default: see pq_decompress).  The four-lane teams spend
// ~2,600 cycles per element round (eight streams in lockstep, each at a different kind of element) and leave 89 % of the warp slots empty; the level prefix of a page is only ~1.5 KB of output behind
// ~400 elements, so a thread can walk it alone in ~30 k instructions -- if its byte traffic stays out of global memory: the last 512
// output bytes and a 64-byte input window live in shared memory, word-interleaved across the warp (byte j of lane L sits in bank L), so
// 32 unrelated streams never conflict and never touch L1.  Far back references (beyond the ring) read the thread's own earlier stores
// back from global memory.  Same protocol as the team kernel: a finished job leaves state {-1, 0}, anything unusual (a large literal
// that is not the page's value section, budget exceeded, malformed input) is left to the warp kernel, which resumes at {ip, op}.
constexpr int ST_RING = 512, ST_WIN = 64, ST_MAX_OUT = 16 * 1024, ST_MAX_ELEMS = 6000;
__global__ void __launch_bounds__(64) pq_decompress_thread_kernel(const PqDecompJob* __restrict__ jobs, int n_jobs, int32_t* __restrict__ status,
                                                                   PqDecompResult* __restrict__ results, PqDecompState* __restrict__ states) {
    __shared__ uint32_t s_ring[2][ST_RING / 4][32];   // [warp][word of the ring][lane]: 36 KB per block of two warps, six blocks per SM
    __shared__ uint32_t s_win[2][ST_WIN / 4][32];
    const unsigned lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const int job = blockIdx.x * 64 + threadIdx.x;
    if (job >= n_jobs) return;
    const PqDecompJob jb = jobs[job];
    results[job] = PqDecompResult{nullptr, -1, 0};
    states[job] = PqDecompState{0, 0};
    if (!(jb.kind >= 1 && jb.v1_levels)) return;   // not a level prefix: the warp kernel's business from the start
    uint8_t* ring = (uint8_t*)&s_ring[wid][0][lane];   // byte j: ring[(j >> 2) * 128 + (j & 3)]
    uint8_t* win = (uint8_t*)&s_win[wid][0][lane];
    const uint8_t* __restrict__ src = jb.src;
    uint8_t* dst = jb.dst;
    const int n_in = jb.src_len, n_out = jb.dst_len;
    int ip = 0, op = 0, wbase = -(1 << 30);
    auto rd = [&](int pos) -> uint32_t {   // input byte `pos` through the window (16-byte aligned refills; bytes behind the stream read as 0)
        if (pos < wbase || pos >= wbase + ST_WIN) {
            const uintptr_t g = (uintptr_t)(src + pos), ga = g & ~(uintptr_t)15;
            wbase = pos - (int)(g - ga);
            const uint8_t* lim = src + n_in + 16;
#pragma unroll
            for (int q = 0; q < ST_WIN / 16; q++) {
                const uint8_t* a = (const uint8_t*)ga + 16 * q;
                const uint4 v = a < lim ? *(const uint4*)a : make_uint4(0, 0, 0, 0);
                s_win[wid][4 * q + 0][lane] = v.x;
                s_win[wid][4 * q + 1][lane] = v.y;
                s_win[wid][4 * q + 2][lane] = v.z;
                s_win[wid][4 * q + 3][lane] = v.w;
            }
        }
        const int j = pos - wbase;
        return win[(j >> 2) * 128 + (j & 3)];
    };
    auto put = [&](int o, uint8_t c) {
        dst[o] = c;
        const int j = o & (ST_RING - 1);
        ring[(j >> 2) * 128 + (j & 3)] = c;
    };
    auto ring_at = [&](int o) -> uint8_t {
        const int j = o & (ST_RING - 1);
        return ring[(j >> 2) * 128 + (j & 3)];
    };
    // preamble: uncompressed length (a malformed one is left to the warp kernel, which reports it)
    {
        uint32_t v = 0;
        int shift = 0;
        for (;;) {
            if (ip >= n_in || shift > 28) return;
            const uint32_t b = rd(ip);
            ip++;
            v |= (b & 0x7f) << shift;
            if (!(b & 0x80)) break;
            shift += 7;
        }
        if (jb.kind == 2 ? (int)v < n_out : (int)v != n_out) return;
    }
    const int ip_first = ip;
    for (int elems = 0;; elems++) {
        if (ip >= n_in) {
            if (op == n_out) states[job] = PqDecompState{-1, 0};
            else states[job] = PqDecompState{ip_first == ip ? 0 : ip, op};   // short output: the warp kernel reports it
            return;
        }
        const int ip0 = ip;
        bool handoff = op >= ST_MAX_OUT || elems >= ST_MAX_ELEMS;
        if (!handoff) {
            const uint32_t tag = rd(ip);
            ip++;
            const uint32_t kind = tag & 3;
            if (kind == 0) {
                int len = (int)(tag >> 2) + 1;
                if (len > 60) {
                    const int nb = len - 60;
                    uint32_t v = 0;
                    if (ip + nb > n_in) handoff = true;
                    else {
                        for (int k = 0; k < nb; k++) v |= rd(ip + k) << (8 * k);
                        ip += nb;
                        if (v >= 0x7fffffffu) handoff = true;
                        len = (int)v + 1;
                    }
                }
                if (!handoff && (len > n_in - ip || len > n_out - op)) handoff = true;   // malformed: reported by the warp kernel
                if (!handoff) {
                    if (len > 256) {
                        // the literal that holds the value section: only the level bytes that spill into it are copied, the page reads its
                        // values in place from the compressed buffer (see the warp kernel); any other large literal is not for this kernel
                        handoff = true;
                        if (jb.kind == 1 && ip + len == n_in && op + len == n_out && op >= 4) {
                            const uint32_t head = (uint32_t)dst[0] | ((uint32_t)dst[1] << 8) | ((uint32_t)dst[2] << 16) | ((uint32_t)dst[3] << 24);
                            const int64_t val_off = 4 + (int64_t)head, keep = val_off - op;
                            if (keep >= 0 && keep <= 64 && len - keep >= 256) {   // (a longer spill is a job for 32 lanes: the warp kernel resumes here)
                                for (int i = 0; i < (int)keep; i++) dst[op + i] = src[ip + i];
                                results[job] = PqDecompResult{src + ip + keep, (int32_t)val_off, 0};
                                states[job] = PqDecompState{-1, 0};
                                return;
                            }
                        }
                    } else {
                        for (int i = 0; i < len; i++) put(op + i, (uint8_t)rd(ip + i));
                        ip += len;
                        op += len;
                    }
                }
            } else {
                int len, off;
                if (kind == 1) {
                    len = 4 + (int)((tag >> 2) & 7);
                    off = (int)(((tag >> 5) << 8) | rd(ip));
                    ip += 1;
                } else if (kind == 2) {
                    len = (int)(tag >> 2) + 1;
                    off = (int)(rd(ip) | (rd(ip + 1) << 8));
                    ip += 2;
                } else {
                    len = (int)(tag >> 2) + 1;
                    const uint32_t o4 = rd(ip) | (rd(ip + 1) << 8) | (rd(ip + 2) << 16) | (rd(ip + 3) << 24);
                    off = o4 > 0x7fffffffu ? 0 : (int)o4;
                    ip += 4;
                }
                if (ip > n_in || off <= 0 || off > op || len > n_out - op) handoff = true;   // malformed: reported by the warp kernel
                else if (off + len <= ST_RING) {   // every source byte is still in the ring, none of them is overwritten by this element
                    const int from = op - off;
                    for (int i = 0; i < len; i++) put(op + i, ring_at(from + (off >= len ? i : (int)((unsigned)i % (unsigned)off))));
                    op += len;
                } else {                           // far back reference: the thread's own earlier stores, read back from global memory
                    const uint8_t* from = dst + op - off;
                    for (int i = 0; i < len; i++) put(op + i, from[off >= len ? i : (int)((unsigned)i % (unsigned)off)]);
                    op += len;
                }
            }
        }
        if (handoff) {
            states[job] = PqDecompState{ip0 == ip_first ? 0 : ip0, op};
            return;
        }
    }
}

__global__ void __launch_bounds__(128) pq_decompress_kernel(const PqDecompJob* __restrict__ jobs, int n_jobs, int32_t* __restrict__ status,
                                                            PqDecompResult* __restrict__ results, const PqDecompState* __restrict__ states) {
    __shared__ uint8_t s_ring[4][SN_RING];
    const int job = blockIdx.x * 4 + (threadIdx.x >> 5);
    if (job >= n_jobs) return;
    const unsigned lane = threadIdx.x & 31;
    uint8_t* ring = s_ring[threadIdx.x >> 5];
    const PqDecompJob jb = jobs[job];
    const PqDecompState st0 = states[job];
    if (st0.ip < 0) return;   // finished by the prefix pass
    const uint8_t* __restrict__ src = jb.src;
    uint8_t* dst = jb.dst;
    if (jb.kind == 0) {   // stored bytes (v2 level sections)
        warp_copy(dst, src, jb.dst_len, lane);
        return;
    }
    const int n_in = jb.src_len, n_out = jb.dst_len;
    int ip = st0.ip, op = st0.op, ring_from = st0.op;   // resumed jobs: the ring holds nothing of the output so far
    bool bad = false;
    // preamble: uncompressed length
    if (st0.ip == 0) {
        uint32_t v = 0;
        int shift = 0;
        for (;;) {
            if (ip >= n_in || shift > 28) { bad = true; break; }
            uint8_t b = src[ip++];
            v |= (uint32_t)(b & 0x7f) << shift;
            if (!(b & 0x80)) break;
            shift += 7;
        }
        if (jb.kind == 2 ? (int)v < n_out : (int)v != n_out) bad = true;
    }
    while (!bad && ip < n_in) {
        const uint32_t tag = src[ip++];
        const uint32_t kind = tag & 3;
        if (kind == 0) {
            int len = (int)(tag >> 2) + 1;
            if (len > 60) {
                const int nb = len - 60;
                if (ip + nb > n_in) { bad = true; break; }
                uint32_t v = 0;
                for (int k = 0; k < nb; k++) v |= (uint32_t)src[ip + k] << (8 * k);
                ip += nb;
                if (v >= 0x7fffffffu) { bad = true; break; }
                len = (int)v + 1;
            }
            if (len > n_in - ip || len > n_out - op) { bad = true; break; }
            if (len <= 256) {   // short literal: global + ring
                for (int i = lane; i < len; i += 32) {
                    const uint8_t c = src[ip + i];
                    dst[op + i] = c;
                    ring[(op + i) & (SN_RING - 1)] = c;
                }
                ip += len;
                op += len;
                __syncwarp();
                continue;
            }
            // Nullable v1 data page whose stream ends with one literal that contains the whole value section (bit-packed
            // dictionary indices do not compress; the level bytes in front of them do): copy only the level bytes that
            // spill into this literal and let the page read its values in place from the compressed buffer.
            if (jb.v1_levels && jb.kind == 1 && ip + len == n_in && op + len == n_out && op >= 4) {
                __syncwarp();
                const int64_t val_off = 4 + (int64_t)((uint32_t)dst[0] | ((uint32_t)dst[1] << 8) | ((uint32_t)dst[2] << 16) | ((uint32_t)dst[3] << 24));
                const int64_t keep = val_off - op;
                if (keep >= 0 && len - keep >= 256) {
                    warp_copy(dst + op, src + ip, keep, lane);
                    if (lane == 0) results[job] = PqDecompResult{src + ip + keep, (int32_t)val_off, 0};
                    ip += len;
                    op += len;
                    break;
                }
            }
            warp_copy(dst + op, src + ip, len, lane);
            ip += len;
            op += len;
            ring_from = op;   // the ring does not hold this literal
            __syncwarp();
        } else {
            int len, off;
            if (kind == 1) {
                if (ip + 1 > n_in) { bad = true; break; }
                len = 4 + (int)((tag >> 2) & 7);
                off = (int)(((tag >> 5) << 8) | src[ip]);
                ip += 1;
            } else if (kind == 2) {
                if (ip + 2 > n_in) { bad = true; break; }
                len = (int)(tag >> 2) + 1;
                off = (int)((uint32_t)src[ip] | ((uint32_t)src[ip + 1] << 8));
                ip += 2;
            } else {
                if (ip + 4 > n_in) { bad = true; break; }
                len = (int)(tag >> 2) + 1;
                const uint32_t o4 = (uint32_t)src[ip] | ((uint32_t)src[ip + 1] << 8) | ((uint32_t)src[ip + 2] << 16) | ((uint32_t)src[ip + 3] << 24);
                if (o4 > 0x7fffffffu) { bad = true; break; }
                off = (int)o4;
                ip += 4;
            }
            if (off <= 0 || off > op || len > n_out - op) { bad = true; break; }
            const int from = op - off;
            // len <= 64: at most two bytes per lane; byte i of the run is out[from + i % off] (i % off == i when off >= len)
            if (from >= ring_from && off <= SN_RING - 64) {
                for (int i = lane; i < len; i += 32) {
                    const int k = off >= len ? i : (int)((unsigned)i % (unsigned)off);
                    const uint8_t c = ring[(from + k) & (SN_RING - 1)];
                    dst[op + i] = c;
                    ring[(op + i) & (SN_RING - 1)] = c;   // distinct from every source slot: off + len <= SN_RING
                }
            } else {
                for (int i = lane; i < len; i += 32) {
                    const int k = off >= len ? i : (int)((unsigned)i % (unsigned)off);
                    const uint8_t c = dst[from + k];
                    dst[op + i] = c;
                    ring[(op + i) & (SN_RING - 1)] = c;
                }
            }
            op += len;
            __syncwarp();
        }
    }
    if (!bad && op != n_out) bad = true;
    if (bad && lane == 0) atomicCAS(status, 0, job + 1);
}

// v1 data pages keep [u32 length][definition levels][values] inside the compressed body: once the body is in HBM the
// page descriptor's level / value sections are derived from that length word.
__global__ void pq_fix_v1_pages_kernel(PqPage* __restrict__ pages, int n, const PqDecompResult* __restrict__ results) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    PqPage pg = pages[i];
    if (pg.def_len != -1) return;
    const uint8_t* body = pg.def_ptr - 4;   // def_ptr was set to body + 4
    uint32_t dl = (uint32_t)body[0] | ((uint32_t)body[1] << 8) | ((uint32_t)body[2] << 16) | ((uint32_t)body[3] << 24);
    const int32_t total = pg.val_len;   // whole uncompressed body
    if ((int64_t)dl + 4 > total) dl = (uint32_t)(total - 4);   // corrupt length: clamp, the decode kernels stay in bounds
    pg.def_len = (int32_t)dl;
    pg.val_ptr = body + 4 + dl;
    pg.val_len = total - 4 - (int32_t)dl;
    if (results && pg.job >= 0 && results[pg.job].tail_start == (int32_t)(4 + dl)) pg.val_ptr = results[pg.job].tail_src;   // values were left in place
    if (dl == 0) pg.def_ptr = nullptr;
    pages[i] = pg;
}

PqDecompOut pq_decompress(Ctx& ctx, const std::vector<PqDecompJob>& jobs, size_t n_snappy) {
    PqDecompOut out;
    out.status = dalloc_zero(ctx, 4);
    if (jobs.empty()) return out;
    out.results = dalloc(ctx, jobs.size() * sizeof(PqDecompResult));
    Buf dj = to_device(ctx, jobs.data(), jobs.size() * sizeof(PqDecompJob));
    pq_decompress_zstd_lz4(ctx, jobs, n_snappy, P<PqDecompJob>(dj), P<int32_t>(out.status), P<PqDecompResult>(out.results));
    if (n_snappy == 0) return out;
    Buf states = dalloc(ctx, n_snappy * sizeof(PqDecompState));
    ProfScope ps(ctx, "pq_decompress");
    // AURON_SNAPPY_THREADS=1: the one-thread-per-job prefix pass.  A thread alone pays the full shared-memory latency per byte
    // (load, store, next byte); the four-lane teams overlap four bytes and eight streams per warp.  Kept selectable as the alternative.
    static const bool teams = getenv("AURON_SNAPPY_THREADS") == nullptr;
    if (teams)
        pq_decompress_prefix_kernel<<<(unsigned)((n_snappy + 4 * SN_TEAMS - 1) / (4 * SN_TEAMS)), 128, 0, ctx.stream>>>(P<PqDecompJob>(dj), (int)n_snappy, P<int32_t>(out.status),
                                                                                                     P<PqDecompResult>(out.results), P<PqDecompState>(states));
    else
        pq_decompress_thread_kernel<<<(unsigned)((n_snappy + 63) / 64), 64, 0, ctx.stream>>>(P<PqDecompJob>(dj), (int)n_snappy, P<int32_t>(out.status),
                                                                                                   P<PqDecompResult>(out.results), P<PqDecompState>(states));
    LAUNCH_CHECK(ctx);
    pq_decompress_kernel<<<(unsigned)((n_snappy + 3) / 4), 128, 0, ctx.stream>>>(P<PqDecompJob>(dj), (int)n_snappy, P<int32_t>(out.status),
                                                                                       P<PqDecompResult>(out.results), P<PqDecompState>(states));
    LAUNCH_CHECK(ctx);
    return out;
}
void pq_fix_v1_pages(Ctx& ctx, PqPage* pages, int n, const PqDecompResult* results) {
    if (n <= 0) return;
    pq_fix_v1_pages_kernel<<<(n + 255) / 256, 256, 0, ctx.stream>>>(pages, n, results);
    LAUNCH_CHECK(ctx);
}

}  // namespace auron
