// zstd_dec.cuh -- a Zstandard frame decoder written from RFC 8878, __host__ __device__ so that the Parquet scan's device kernel
// (k_zstd.cu) and auron_b200_zstd_decompress (the same code on the CPU) share one source.  Included by k_zstd.cu only.
//
// One decoder runs per page body (a sequence of Zstandard and skippable frames).  On the device a whole warp runs it: the serial
// parts (headers, entropy decoding of the sequences) run identically on every lane with warp-uniform control flow and broadcast
// loads, the table builds run on lane 0 (they write shared memory), the 4-stream Huffman literals on lanes 0..3 (one stream each),
// and the literal and match copies on all lanes.  On the CPU the same code runs with one lane.
//
// Literals of a compressed block are decoded into the tail of the output that is still to be written, [cap - size, cap): no scratch
// memory.  That is safe because the output still to come is at least the literals still to come, so the write position never
// passes the literal read position; a block that would need more output than `cap` is rejected before it could.
//
// Acceptance follows libzstd's ZSTD_decompress wherever the specification leaves a choice: a non-zero dictionary ID, trailing
// bytes after the last frame, the reserved bits of the frame header and of the sequences section and Huffman codes of 12 bits
// are handled as it handles them.  A Huffman stream must be consumed exactly (libzstd's double-symbol decoder lets the last code
// of a stream run past its start).  Every read of `in` and every write of `out` is bounds-checked.
#pragma once
#include <stdint.h>
#include <string.h>

#ifdef __CUDACC__
#define ZD_HD __host__ __device__
#else
#define ZD_HD
#endif

namespace auron {
namespace zd {

constexpr int HUF_MAX_LOG = 12;   // RFC 8878 caps codes at 11 bits; libzstd decodes 12
constexpr int LL_MAX_LOG = 9, ML_MAX_LOG = 9, OF_MAX_LOG = 8;
constexpr int LL_MAX_SYM = 35, ML_MAX_SYM = 52, OF_MAX_SYM = 31;
constexpr int64_t BLOCK_MAX = 128 << 10;

struct Fse {   // one decoding state: symbol, bits to read, baseline of the next state
    uint8_t sym, nb;
    uint16_t base;
};
// Decoding tables of one decoder (shared memory on the device: 14.8 KB per warp).  LL / OF / ML and the Huffman table persist
// across the blocks of a frame (Repeat modes, treeless literals).
struct Tables {
    uint16_t huf[1 << HUF_MAX_LOG];   // (symbol << 4) | code length, indexed by the next HUF log bits
    Fse ll[1 << LL_MAX_LOG], ml[1 << ML_MAX_LOG], of[1 << OF_MAX_LOG];
    Fse wt[64];                       // FSE table of compressed Huffman weights (accuracy log <= 6)
    int16_t norm[256];                // scratch of the table builds
    uint16_t next[256];
    uint8_t w[256];
};

ZD_HD inline void zsync() {
#ifdef __CUDA_ARCH__
    __syncwarp();
#endif
}
ZD_HD inline int bcast(int v) {
#ifdef __CUDA_ARCH__
    return __shfl_sync(0xffffffffu, v, 0);
#else
    return v;
#endif
}
ZD_HD inline bool any(bool b) {
#ifdef __CUDA_ARCH__
    return __any_sync(0xffffffffu, b) != 0;
#else
    return b;
#endif
}
ZD_HD inline int hbit(uint32_t v) {   // index of the highest set bit, v > 0
#ifdef __CUDA_ARCH__
    return 31 - __clz(v);
#else
    return 31 - __builtin_clz(v);
#endif
}
ZD_HD inline uint32_t le16(const uint8_t* p) { return (uint32_t)p[0] | ((uint32_t)p[1] << 8); }
ZD_HD inline uint32_t le24(const uint8_t* p) { return le16(p) | ((uint32_t)p[2] << 16); }
ZD_HD inline uint32_t le32(const uint8_t* p) { return le24(p) | ((uint32_t)p[3] << 24); }

// ---- predefined distributions and code tables (RFC 8878 3.1.1.3.2.2)
#define ZD_LL_NORM {4, 3, 2, 2, 2, 2, 2, 2, 2, 2, 2, 2, 2, 1, 1, 1, 2, 2, 2, 2, 2, 2, 2, 2, 2, 3, 2, 1, 1, 1, 1, 1, -1, -1, -1, -1}
#define ZD_ML_NORM {1, 4, 3, 2, 2, 2, 2, 2, 2, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, -1, -1, -1, -1, -1, -1, -1}
#define ZD_OF_NORM {1, 1, 1, 1, 1, 1, 2, 2, 2, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, -1, -1, -1, -1, -1}
// literal length codes 16..35 and match length codes 32..52: baseline | extra bits << 24
#define ZD_LL_CODE {16 | 1 << 24, 18 | 1 << 24, 20 | 1 << 24, 22 | 1 << 24, 24 | 2 << 24, 28 | 2 << 24, 32 | 3 << 24, 40 | 3 << 24, 48 | 4 << 24, 64 | 6 << 24,      \
                    128 | 7 << 24, 256 | 8 << 24, 512 | 9 << 24, 1024 | 10 << 24, 2048 | 11 << 24, 4096 | 12 << 24, 8192 | 13 << 24, 16384 | 14 << 24, \
                    32768 | 15 << 24, 65536 | 16 << 24}
#define ZD_ML_CODE {35 | 1 << 24, 37 | 1 << 24, 39 | 1 << 24, 41 | 1 << 24, 43 | 2 << 24, 47 | 2 << 24, 51 | 3 << 24, 59 | 3 << 24, 67 | 4 << 24, 83 | 4 << 24, \
                    99 | 5 << 24, 131 | 7 << 24, 259 | 8 << 24, 515 | 9 << 24, 1027 | 10 << 24, 2051 | 11 << 24, 4099 | 12 << 24, 8195 | 13 << 24,        \
                    16387 | 14 << 24, 32771 | 15 << 24, 65539 | 16 << 24}
#ifdef __CUDACC__
static __device__ __constant__ int8_t c_ll_norm[36] = ZD_LL_NORM;
static __device__ __constant__ int8_t c_ml_norm[53] = ZD_ML_NORM;
static __device__ __constant__ int8_t c_of_norm[29] = ZD_OF_NORM;
static __device__ __constant__ uint32_t c_ll_code[20] = ZD_LL_CODE;
static __device__ __constant__ uint32_t c_ml_code[21] = ZD_ML_CODE;
#endif
static const int8_t h_ll_norm[36] = ZD_LL_NORM;
static const int8_t h_ml_norm[53] = ZD_ML_NORM;
static const int8_t h_of_norm[29] = ZD_OF_NORM;
static const uint32_t h_ll_code[20] = ZD_LL_CODE;
static const uint32_t h_ml_code[21] = ZD_ML_CODE;
#ifdef __CUDA_ARCH__
#define ZD_TAB(name) c_##name
#else
#define ZD_TAB(name) h_##name
#endif

// ---- backward bit stream (FSE and Huffman): read from the highest set bit of the last byte towards bit 0 of the first.  `pos`
// counts the bits not yet read and goes negative when a read runs past the start.  `win` caches the 64 stream bits
// [win_lo, win_lo + 64), out-of-range bytes read as zero.  A Huffman peek past the start sees zero bits (the stream must then be
// consumed exactly anyway); an FSE read past the start returns what libzstd's bit container returns there, the bits of the first
// eight bytes `head` taken modulo 64, because libzstd accepts a sequence stream that ends overdrawn and decodes those bits.
struct BitIn {
    const uint8_t* p;
    int64_t n, pos, win_lo;
    uint64_t win, head;
};
ZD_HD inline bool bits_init(BitIn& b, const uint8_t* p, int64_t n) {
    if (n < 1 || p[n - 1] == 0) return false;
    b.p = p;
    b.n = n;
    b.pos = (n - 1) * 8 + hbit(p[n - 1]);
    b.win_lo = INT64_MAX;   // empty
    b.win = 0;
    b.head = 0;
    for (int k = (n < 8 ? (int)n : 8) - 1; k >= 0; k--) b.head = (b.head << 8) | p[k];
    return true;
}
ZD_HD inline void bits_refill(BitIn& b) {
    const int64_t byte = (b.pos - 57) >> 3;   // floor: the window then holds [pos - 57 - 7, pos + 7)
    uint64_t w = 0;
    if (byte >= 0 && byte + 8 <= b.n) {
        for (int k = 7; k >= 0; k--) w = (w << 8) | b.p[byte + k];
    } else {
        for (int k = 7; k >= 0; k--) {
            const int64_t i = byte + k;
            w = (w << 8) | ((i >= 0 && i < b.n) ? b.p[i] : 0u);
        }
    }
    b.win = w;
    b.win_lo = byte * 8;
}
ZD_HD inline uint32_t bits_peek(BitIn& b, int nb) {   // nb <= 32
    if (b.pos - nb < b.win_lo) bits_refill(b);
    const int sh = (int)(b.pos - nb - b.win_lo);
    return nb ? (uint32_t)((b.win >> sh) & ((1ull << nb) - 1)) : 0u;
}
ZD_HD inline uint32_t bits_read(BitIn& b, int nb) {
    const uint32_t v = b.pos >= nb ? bits_peek(b, nb) : nb ? (uint32_t)((b.head >> ((b.pos - nb) & 63)) & ((1ull << nb) - 1)) : 0u;
    b.pos -= nb;
    return v;
}

// ---- FSE tables (RFC 8878 4.1)
// Normalised counts from an NCount header at p[0, n): norm[0, max_sym] (symbols past the described ones are 0), *log.  Returns the
// header's bytes, or -1.  Bits past the end read as zero; a header that needs them is rejected by its length.
ZD_HD inline int64_t read_ncount(const uint8_t* p, int64_t n, int max_sym, int max_log, int16_t* norm, int* log_out) {
    for (int s = 0; s <= max_sym; s++) norm[s] = 0;
    int64_t bit = 0;
    auto get = [&](int nb) -> uint32_t {   // nb <= 25: the next nb bits, little-endian, zero past the end
        uint32_t v = 0;
        const int64_t byte = bit >> 3;
        for (int k = 0; k < 4; k++) v |= (uint32_t)(byte + k < n ? p[byte + k] : 0u) << (8 * k);
        return (v >> (bit & 7)) & ((1u << nb) - 1);
    };
    const int log = (int)get(4) + 5;
    bit = 4;
    if (log > max_log) return -1;
    int remaining = (1 << log) + 1, threshold = 1 << log, nbits = log + 1, s = 0;
    bool prev0 = false;
    for (;;) {
        if (prev0) {   // zero-probability repeats: 2-bit flags, 3 = three more zeros and another flag
            for (;;) {
                const uint32_t r = get(2);
                bit += 2;
                s += (int)r;
                if (r != 3) break;
                if (s > max_sym + 1) break;
            }
            if (s >= max_sym + 1) break;
        }
        const int max = 2 * threshold - 1 - remaining;
        int count;
        const uint32_t v = get(nbits);
        if ((int)(v & (uint32_t)(threshold - 1)) < max) {
            count = (int)(v & (uint32_t)(threshold - 1));
            bit += nbits - 1;
        } else {
            count = (int)(v & (uint32_t)(2 * threshold - 1));
            if (count >= threshold) count -= max;
            bit += nbits;
        }
        count--;   // -1: a "less than 1" probability
        remaining -= count < 0 ? -count : count;
        norm[s++] = (int16_t)count;
        prev0 = count == 0;
        if (remaining < threshold) {
            if (remaining <= 1) break;
            nbits = hbit((uint32_t)remaining) + 1;
            threshold = 1 << (nbits - 1);
        }
        if (s >= max_sym + 1) break;
    }
    if (remaining != 1 || s > max_sym + 1) return -1;
    const int64_t bytes = (bit + 7) >> 3;
    if (bytes > n) return -1;
    *log_out = log;
    return bytes;
}
// decoding table of 1 << log states from counts that sum to 1 << log (-1 counts one slot)
ZD_HD inline void build_fse(Fse* t, const int16_t* norm, int nsym, int log, uint16_t* next) {
    const int size = 1 << log, mask = size - 1, step = (size >> 1) + (size >> 3) + 3;
    int high = size - 1;
    for (int s = 0; s < nsym; s++) {
        if (norm[s] == -1) {
            t[high--].sym = (uint8_t)s;
            next[s] = 1;
        } else {
            next[s] = (uint16_t)norm[s];
        }
    }
    int pos = 0;
    for (int s = 0; s < nsym; s++)
        for (int i = 0; i < norm[s]; i++) {
            t[pos].sym = (uint8_t)s;
            do pos = (pos + step) & mask;
            while (pos > high);
        }
    for (int u = 0; u < size; u++) {
        const uint32_t x = next[t[u].sym]++;
        const int nb = log - hbit(x);
        t[u].nb = (uint8_t)nb;
        t[u].base = (uint16_t)((x << nb) - (uint32_t)size);
    }
}
ZD_HD inline int sum_ok(const int16_t* norm, int nsym, int log) {
    int tot = 0;
    for (int s = 0; s < nsym; s++) tot += norm[s] == -1 ? 1 : norm[s];
    return tot == (1 << log);
}

// ---- XXH64 (seed 0) of the frame's output: the content checksum
ZD_HD inline uint64_t rotl64(uint64_t x, int r) { return (x << r) | (x >> (64 - r)); }
ZD_HD inline uint64_t rd64(const uint8_t* p) {
    uint64_t v = 0;
    for (int k = 7; k >= 0; k--) v = (v << 8) | p[k];
    return v;
}
ZD_HD inline uint64_t xxh64(const uint8_t* p, int64_t len) {
    const uint64_t P1 = 0x9E3779B185EBCA87ull, P2 = 0xC2B2AE3D27D4EB4Full, P3 = 0x165667B19E3779F9ull, P4 = 0x85EBCA77C2B2AE63ull,
                   P5 = 0x27D4EB2F165667C5ull;
    auto round = [&](uint64_t acc, uint64_t in) { return rotl64(acc + in * P2, 31) * P1; };
    int64_t i = 0;
    uint64_t h;
    if (len >= 32) {
        uint64_t v1 = P1 + P2, v2 = P2, v3 = 0, v4 = 0 - P1;
        for (; i + 32 <= len; i += 32) {
            v1 = round(v1, rd64(p + i));
            v2 = round(v2, rd64(p + i + 8));
            v3 = round(v3, rd64(p + i + 16));
            v4 = round(v4, rd64(p + i + 24));
        }
        h = rotl64(v1, 1) + rotl64(v2, 7) + rotl64(v3, 12) + rotl64(v4, 18);
        h = (h ^ round(0, v1)) * P1 + P4;
        h = (h ^ round(0, v2)) * P1 + P4;
        h = (h ^ round(0, v3)) * P1 + P4;
        h = (h ^ round(0, v4)) * P1 + P4;
    } else {
        h = P5;
    }
    h += (uint64_t)len;
    for (; i + 8 <= len; i += 8) h = rotl64(h ^ round(0, rd64(p + i)), 27) * P1 + P4;
    if (i + 4 <= len) {
        h = rotl64(h ^ ((uint64_t)le32(p + i) * P1), 23) * P2 + P3;
        i += 4;
    }
    for (; i < len; i++) h = rotl64(h ^ (p[i] * P5), 11) * P1;
    h ^= h >> 33;
    h *= P2;
    h ^= h >> 29;
    h *= P3;
    h ^= h >> 32;
    return h;
}

// ---- copies: dst and src disjoint
ZD_HD inline void copy_bytes(uint8_t* dst, const uint8_t* src, int64_t len, unsigned lane, unsigned nl) {
#ifdef __CUDA_ARCH__
    (void)nl;
    warp_copy(dst, src, len, lane);
#else
    (void)lane, (void)nl;
    if (len > 0) memcpy(dst, src, (size_t)len);
#endif
}

struct Decoder {
    const uint8_t* in;
    int64_t n;
    uint8_t* out;
    int64_t cap;
    Tables* T;
    unsigned lane, nl;
    // frame state
    int64_t frame_start;
    int huf_log, ll_log, of_log, ml_log;
    bool have_huf, have_seq;
    uint32_t rep[3];

    // ---- Huffman tree description at p[0, n) -> T->huf; returns its bytes or -1 (lane 0)
    ZD_HD int64_t read_huffman(const uint8_t* p, int64_t n) {
        if (n < 1) return -1;
        const int hb = p[0];
        uint8_t* w = T->w;
        int nw = 0;
        int64_t used;
        if (hb >= 128) {   // direct 4-bit weights, two per byte
            nw = hb - 127;
            used = 1 + (nw + 1) / 2;
            if (used > n) return -1;
            for (int i = 0; i < nw; i++) w[i] = (uint8_t)((i & 1) ? p[1 + i / 2] & 15 : p[1 + i / 2] >> 4);
        } else {   // FSE-compressed weights: two interleaved states over one backward stream
            used = 1 + hb;
            if (used > n) return -1;
            int log = 0;
            const int64_t hs = read_ncount(p + 1, hb, 255, 6, T->norm, &log);
            if (hs < 0) return -1;
            int nsym = 256;
            while (nsym > 0 && T->norm[nsym - 1] == 0) nsym--;
            build_fse(T->wt, T->norm, nsym, log, T->next);
            BitIn b;
            if (!bits_init(b, p + 1 + hs, hb - hs)) return -1;
            uint32_t s1 = bits_read(b, log), s2 = bits_read(b, log);
            for (;;) {
                if (nw > 253) return -1;
                w[nw++] = T->wt[s1].sym;
                s1 = T->wt[s1].base + bits_read(b, T->wt[s1].nb);
                if (b.pos < 0) {
                    w[nw++] = T->wt[s2].sym;
                    break;
                }
                if (nw > 253) return -1;
                w[nw++] = T->wt[s2].sym;
                s2 = T->wt[s2].base + bits_read(b, T->wt[s2].nb);
                if (b.pos < 0) {
                    w[nw++] = T->wt[s1].sym;
                    break;
                }
            }
        }
        // the last weight is implied: the weights sum to a power of two
        uint32_t total = 0, rank[HUF_MAX_LOG + 2] = {0};
        for (int i = 0; i < nw; i++) {
            if (w[i] > HUF_MAX_LOG) return -1;
            rank[w[i]]++;
            total += (1u << w[i]) >> 1;
        }
        if (total == 0) return -1;
        const int log = hbit(total) + 1;
        if (log > HUF_MAX_LOG) return -1;
        const uint32_t rest = (1u << log) - total;
        if (rest & (rest - 1)) return -1;
        const int last = hbit(rest) + 1;
        w[nw++] = (uint8_t)last;
        rank[last]++;
        if (rank[1] < 2 || (rank[1] & 1)) return -1;
        // codes: weight 1 first (the longest), symbols in order within a weight
        uint32_t start[HUF_MAX_LOG + 2], acc = 0;
        for (int k = 1; k <= log; k++) {
            start[k] = acc;
            acc += rank[k] << (k - 1);
        }
        for (int s = 0; s < nw; s++) {
            const int k = w[s];
            if (!k) continue;
            const uint16_t e = (uint16_t)((s << 4) | (log + 1 - k));
            for (uint32_t u = start[k]; u < start[k] + (1u << (k - 1)); u++) T->huf[u] = e;
            start[k] += 1u << (k - 1);
        }
        huf_log = log;
        return used;
    }
    // one Huffman stream p[0, n) -> dst[0, count); the stream must be consumed exactly
    ZD_HD bool huf_stream(const uint8_t* p, int64_t n, uint8_t* dst, int64_t count) const {
        BitIn b;
        if (!bits_init(b, p, n)) return false;
        const int log = huf_log;
        const uint16_t* t = T->huf;
        for (int64_t k = 0; k < count; k++) {
            const uint16_t e = t[bits_peek(b, log)];
            dst[k] = (uint8_t)(e >> 4);
            b.pos -= e & 15;
            if (b.pos < 0) return false;
        }
        return b.pos == 0;
    }

    // ---- one sequence table (mode: 0 predefined, 1 RLE, 2 FSE, 3 repeat); returns bytes used or -1 (lane 0)
    ZD_HD int64_t read_seq_table(int mode, const uint8_t* p, int64_t n, Fse* t, int* log, int max_sym, int max_log, const int8_t* dnorm, int dnsym, int dlog) {
        if (mode == 0) {
            for (int s = 0; s < dnsym; s++) T->norm[s] = dnorm[s];
            build_fse(t, T->norm, dnsym, dlog, T->next);
            *log = dlog;
            return 0;
        }
        if (mode == 1) {
            if (n < 1 || p[0] > max_sym) return -1;
            t[0] = Fse{p[0], 0, 0};
            *log = 0;
            return 1;
        }
        if (mode == 2) {
            int lg = 0;
            const int64_t hs = read_ncount(p, n, max_sym, max_log, T->norm, &lg);
            if (hs < 0 || !sum_ok(T->norm, max_sym + 1, lg)) return -1;
            build_fse(t, T->norm, max_sym + 1, lg, T->next);
            *log = lg;
            return hs;
        }
        return have_seq ? 0 : -1;
    }

    // literal length and match length values of a code
    ZD_HD static void ll_code(int c, uint32_t* base, int* nb) {
        if (c < 16) {
            *base = (uint32_t)c, *nb = 0;
        } else {
            const uint32_t v = ZD_TAB(ll_code)[c - 16];
            *base = v & 0xffffff, *nb = (int)(v >> 24);
        }
    }
    ZD_HD static void ml_code(int c, uint32_t* base, int* nb) {
        if (c < 32) {
            *base = (uint32_t)c + 3, *nb = 0;
        } else {
            const uint32_t v = ZD_TAB(ml_code)[c - 32];
            *base = v & 0xffffff, *nb = (int)(v >> 24);
        }
    }

    // ---- a compressed block at p[0, n), output from *op
    ZD_HD bool compressed_block(const uint8_t* p, int64_t n, int64_t* op_io) {
        int64_t op = *op_io;
        if (n < 2) return false;
        // literals section header
        const int lt = p[0] & 3, sf = (p[0] >> 2) & 3;
        int64_t lh, lsize, csize = 0;
        int nstreams = 1;
        if (lt < 2) {   // raw, RLE
            if (sf == 1) lh = 2;
            else if (sf == 3) lh = 3;
            else lh = 1;
            if (lh > n) return false;
            lsize = lh == 1 ? p[0] >> 3 : lh == 2 ? le16(p) >> 4 : le24(p) >> 4;
        } else {   // compressed, treeless
            if (n < 5) return false;
            lh = sf < 2 ? 3 : sf == 2 ? 4 : 5;
            nstreams = sf == 0 ? 1 : 4;
            if (lh == 3) {
                const uint32_t h = le24(p);
                lsize = (h >> 4) & 0x3ff, csize = (h >> 14) & 0x3ff;
            } else if (lh == 4) {
                const uint32_t h = le32(p);
                lsize = (h >> 4) & 0x3fff, csize = h >> 18;
            } else {
                const uint64_t h = le32(p) | ((uint64_t)p[4] << 32);
                lsize = (int64_t)((h >> 4) & 0x3ffff), csize = (int64_t)((h >> 22) & 0x3ffff);
            }
            if (nstreams == 4 && lsize < 6) return false;
            if (lt == 3 && !have_huf) return false;
        }
        if (lsize > BLOCK_MAX || lsize > cap - op) return false;
        const uint8_t* lit;   // the block's literals: in the input (raw) or in the output's tail
        int64_t ip;
        uint8_t* tail = out + cap - lsize;
        if (lt == 0) {
            if (lh + lsize > n) return false;
            lit = p + lh;
            ip = lh + lsize;
        } else if (lt == 1) {
            if (lh + 1 > n) return false;
            const uint8_t c = p[lh];
            for (int64_t i = lane; i < lsize; i += nl) tail[i] = c;
            lit = tail;
            ip = lh + 1;
        } else {
            if (lh + csize > n) return false;
            const uint8_t* q = p + lh;
            int64_t qn = csize;
            if (lt == 2) {
                int64_t hs = 0;
                if (lane == 0) hs = read_huffman(q, qn);
                hs = bcast((int)hs);
                huf_log = bcast(huf_log);
                zsync();
                if (hs < 0 || hs >= qn) return false;
                have_huf = true;
                q += hs, qn -= hs;
            }
            bool bad = false;
            if (nstreams == 1) {
                if (lane == 0) bad = !huf_stream(q, qn, tail, lsize);
            } else {
                if (qn < 10) return false;
                const int64_t s1 = le16(q), s2 = le16(q + 2), s3 = le16(q + 4), s4 = qn - 6 - s1 - s2 - s3;
                if (s4 < 0) return false;
                const int64_t seg = (lsize + 3) / 4, last = lsize - 3 * seg;
                if (last < 0) return false;
                for (unsigned s = lane; s < 4; s += nl) {
                    const int64_t off = 6 + (s > 0 ? s1 : 0) + (s > 1 ? s2 : 0) + (s > 2 ? s3 : 0);
                    const int64_t len = s == 0 ? s1 : s == 1 ? s2 : s == 2 ? s3 : s4;
                    bad = bad || !huf_stream(q + off, len, tail + s * seg, s == 3 ? last : seg);
                }
            }
            if (any(bad)) return false;
            lit = tail;
            ip = lh + csize;
        }
        zsync();   // literals decoded by some lanes are read by all
        // sequences section header
        if (ip >= n) return false;
        int64_t nseq = p[ip++];
        if (nseq >= 128) {
            if (nseq == 255) {
                if (ip + 2 > n) return false;
                nseq = le16(p + ip) + 0x7f00;
                ip += 2;
            } else {
                if (ip >= n) return false;
                nseq = ((nseq - 128) << 8) + p[ip++];
            }
        }
        int64_t lrem = lsize;   // literals not yet copied
        if (nseq > 0) {
            if (ip >= n) return false;
            const int modes = p[ip++];   // (its two reserved bits are ignored, as libzstd 1.5 ignores them)
            int64_t r = 0;
            if (lane == 0) {
                const int64_t a = read_seq_table(modes >> 6, p + ip, n - ip, T->ll, &ll_log, LL_MAX_SYM, LL_MAX_LOG, ZD_TAB(ll_norm), 36, 6);
                const int64_t b = a < 0 ? -1 : read_seq_table((modes >> 4) & 3, p + ip + a, n - ip - a, T->of, &of_log, OF_MAX_SYM, OF_MAX_LOG, ZD_TAB(of_norm), 29, 5);
                const int64_t c = b < 0 ? -1 : read_seq_table((modes >> 2) & 3, p + ip + a + b, n - ip - a - b, T->ml, &ml_log, ML_MAX_SYM, ML_MAX_LOG, ZD_TAB(ml_norm), 53, 6);
                r = c < 0 ? -1 : a + b + c;
            }
            r = bcast((int)r);
            ll_log = bcast(ll_log), of_log = bcast(of_log), ml_log = bcast(ml_log);
            zsync();
            if (r < 0) return false;
            have_seq = true;
            ip += r;
            BitIn b;
            if (!bits_init(b, p + ip, n - ip)) return false;
            const Fse* tll = T->ll;
            const Fse* tof = T->of;
            const Fse* tml = T->ml;
            uint32_t sll = bits_read(b, ll_log), sof = bits_read(b, of_log), sml = bits_read(b, ml_log);
            for (int64_t i = 0; i < nseq; i++) {
                const Fse ell = tll[sll], eof = tof[sof], eml = tml[sml];
                const int ofc = eof.sym;
                const uint32_t ofv = (1u << ofc) + bits_read(b, ofc);
                uint32_t mlb, llb;
                int mln, lln;
                ml_code(eml.sym, &mlb, &mln);
                ll_code(ell.sym, &llb, &lln);
                const int64_t ml = mlb + bits_read(b, mln);
                const int64_t ll = llb + bits_read(b, lln);
                if (i + 1 < nseq) {
                    sll = ell.base + bits_read(b, ell.nb);
                    sml = eml.base + bits_read(b, eml.nb);
                    sof = eof.base + bits_read(b, eof.nb);
                }
                // offset: a new one, or one of the three repeat offsets (shifted by one when the literal length is 0)
                uint32_t off;
                if (ofv > 3) {
                    off = ofv - 3;
                    rep[2] = rep[1], rep[1] = rep[0], rep[0] = off;
                } else {
                    const int idx = (int)ofv - 1 + (ll == 0 ? 1 : 0);
                    if (idx == 0) {
                        off = rep[0];
                    } else {
                        off = idx == 3 ? rep[0] - 1 : rep[idx];
                        if (idx != 1) rep[2] = rep[1];
                        rep[1] = rep[0];
                        rep[0] = off;
                    }
                }
                // execute: ll literals, then ml bytes from `off` back
                if (ll > lrem || ml > cap - op - lrem) return false;
                if (off == 0 || off > op + ll - frame_start) return false;
                copy_literals(op, lit, ll);
                lit += ll, op += ll, lrem -= ll;
                copy_match(op, off, ml);
                op += ml;
            }
            if (b.pos > 0) return false;   // every bit read; an overdrawn stream is accepted, as libzstd accepts it
        } else if (ip != n) {
            return false;
        }
        copy_literals(op, lit, lrem);
        op += lrem;
        *op_io = op;
        return true;
    }
    // out[op, op + len) = lit[0, len); lit is in the input or at or after out + op in the output's tail
    ZD_HD void copy_literals(int64_t op, const uint8_t* lit, int64_t len) {
        uint8_t* dst = out + op;
        if (len <= 0 || lit == dst) return;
        const bool in_out = lit >= out && lit < out + cap;
        const int64_t gap = in_out ? lit - dst : len;
#ifndef __CUDA_ARCH__
        if (in_out) {
            memmove(dst, lit, (size_t)len);
            return;
        }
#endif
        if (gap >= len) {
            copy_bytes(dst, lit, len, lane, nl);
        } else {   // the tail region overlaps: pieces of `gap` bytes, each read before the next is written
            for (int64_t c = 0; c < len; c += gap) {
                const int64_t m = len - c < gap ? len - c : gap;
                for (int64_t i = lane; i < m; i += nl) dst[c + i] = lit[c + i];
                zsync();
            }
        }
        zsync();
    }
    ZD_HD void copy_match(int64_t op, uint32_t off, int64_t len) {
        uint8_t* dst = out + op;
        const uint8_t* src = dst - off;
        if (off >= len) {
            copy_bytes(dst, src, len, lane, nl);
        } else {   // overlapping run: byte i repeats byte i % off of the period
            for (int64_t i = lane; i < len; i += nl) dst[i] = src[i % off];
        }
        zsync();
    }

    // ---- a page body: frames and skippable frames back to back.  Returns the output bytes, or -1.
    ZD_HD int64_t run() {
        int64_t ip = 0, op = 0;
        while (n - ip >= 5) {
            const uint32_t magic = le32(in + ip);
            if ((magic & 0xfffffff0u) == 0x184D2A50u) {   // skippable frame
                if (n - ip < 8) return -1;
                const int64_t sz = le32(in + ip + 4);
                if (sz > n - ip - 8) return -1;
                ip += 8 + sz;
                continue;
            }
            if (magic != 0xFD2FB528u) return -1;
            // frame header
            if (n - ip < 9) return -1;
            const int fhd = in[ip + 4];
            const int fcs_flag = fhd >> 6, single = (fhd >> 5) & 1, checksum = (fhd >> 2) & 1, did_flag = fhd & 3;
            if (fhd & 8) return -1;
            const int did_size = did_flag == 3 ? 4 : did_flag;
            const int fcs_size = fcs_flag == 0 ? single : fcs_flag == 1 ? 2 : fcs_flag == 2 ? 4 : 8;
            const int64_t fh = 5 + !single + did_size + fcs_size;
            if (n - ip < fh + 3) return -1;
            int64_t q = ip + 5;
            if (!single) {
                if ((in[q] >> 3) + 10 > 31) return -1;   // window log
                q++;
            }
            uint32_t did = 0;
            for (int k = 0; k < did_size; k++) did |= (uint32_t)in[q + k] << (8 * k);
            q += did_size;
            if (did != 0) return -1;   // Parquet pages use no dictionary
            uint64_t fcs = 0;
            for (int k = 0; k < fcs_size; k++) fcs |= (uint64_t)in[q + k] << (8 * k);
            if (fcs_size == 2) fcs += 256;
            ip = fh + ip;
            frame_start = op;
            have_huf = have_seq = false;
            rep[0] = 1, rep[1] = 4, rep[2] = 8;
            // blocks
            for (;;) {
                if (n - ip < 3) return -1;
                const uint32_t bh = le24(in + ip);
                ip += 3;
                const int last = bh & 1, type = (bh >> 1) & 3;
                const int64_t bsize = bh >> 3;
                if (type == 3) return -1;
                const int64_t csz = type == 1 ? 1 : bsize;
                if (csz > n - ip) return -1;
                if (type == 0) {
                    if (bsize > cap - op) return -1;
                    copy_bytes(out + op, in + ip, bsize, lane, nl);
                    zsync();
                    op += bsize;
                } else if (type == 1) {
                    if (bsize > cap - op) return -1;
                    const uint8_t c = in[ip];
                    for (int64_t i = lane; i < bsize; i += nl) out[op + i] = c;
                    zsync();
                    op += bsize;
                } else {
                    if (bsize >= BLOCK_MAX) return -1;
                    if (!compressed_block(in + ip, bsize, &op)) return -1;
                }
                ip += csz;
                if (last) break;
            }
            if (fcs_size && (uint64_t)(op - frame_start) != fcs) return -1;
            if (checksum) {
                if (n - ip < 4) return -1;
                uint32_t h = 0;
                if (lane == 0) h = (uint32_t)xxh64(out + frame_start, op - frame_start);
                h = (uint32_t)bcast((int)h);
                if (h != le32(in + ip)) return -1;
                ip += 4;
            }
        }
        return ip == n ? op : -1;
    }
};

// decode the page body in[0, n) into out[0, cap); returns the bytes written or -1 (malformed, or more than cap bytes)
ZD_HD inline int64_t decompress(const uint8_t* in, int64_t n, uint8_t* out, int64_t cap, Tables* T, unsigned lane, unsigned nl) {
    Decoder d;
    d.in = in, d.n = n, d.out = out, d.cap = cap, d.T = T, d.lane = lane, d.nl = nl;
    d.frame_start = 0;
    d.huf_log = d.ll_log = d.of_log = d.ml_log = 0;
    d.have_huf = d.have_seq = false;
    d.rep[0] = 1, d.rep[1] = 4, d.rep[2] = 8;
    return d.run();
}

}  // namespace zd
}  // namespace auron
