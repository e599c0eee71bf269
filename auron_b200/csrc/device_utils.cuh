// device_utils.cuh -- device-side helpers shared by the sm_90a kernels: bitmap access, warp
// primitives, Spark-compatible murmur3 / xxhash64 (bit-exact with
// datafusion-ext-commons/src/hash/{mur,xxhash}.rs), 128-bit integer helpers.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace auron {

#define FULL_MASK 0xffffffffu

__device__ __forceinline__ bool bit_get(const uint8_t* bm, int64_t i) { return (bm[i >> 3] >> (i & 7)) & 1; }
__device__ __forceinline__ bool valid_at(const uint8_t* bm, int64_t i) { return bm == nullptr || bit_get(bm, i); }
__device__ __forceinline__ unsigned lane_id() { return threadIdx.x & 31; }
// byte-wise (unsigned, shorter-prefix-first) order of two rows of a utf8 / binary column: < 0, 0, > 0
__device__ __forceinline__ int str_row_cmp(const uint8_t* __restrict__ data, const int32_t* __restrict__ offs, int64_t a, int64_t b) {
    const int32_t a0 = offs[a], la = offs[a + 1] - a0, b0 = offs[b], lb = offs[b + 1] - b0;
    const int32_t m = la < lb ? la : lb;
    for (int32_t i = 0; i < m; i++) {
        const int d = (int)data[a0 + i] - (int)data[b0 + i];
        if (d) return d;
    }
    return la - lb;
}
__device__ __forceinline__ unsigned lanemask_lt() {
    unsigned m;
    asm("mov.u32 %0, %%lanemask_lt;" : "=r"(m));
    return m;
}

// ---------------------------------------------------------------- murmur3_x86_32 (Spark flavour)
// mur.rs:38-62
__device__ __forceinline__ uint32_t mm_mix_k1(uint32_t k1) {
    k1 *= 0xcc9e2d51u;
    k1 = __funnelshift_l(k1, k1, 15);
    k1 *= 0x1b873593u;
    return k1;
}
__device__ __forceinline__ uint32_t mm_mix_h1(uint32_t h1, uint32_t k1) {
    h1 ^= k1;
    h1 = __funnelshift_l(h1, h1, 13);
    return h1 * 5u + 0xe6546b64u;
}
__device__ __forceinline__ uint32_t mm_fmix(uint32_t h1, uint32_t len) {
    h1 ^= len;
    h1 ^= h1 >> 16;
    h1 *= 0x85ebca6bu;
    h1 ^= h1 >> 13;
    h1 *= 0xc2b2ae35u;
    h1 ^= h1 >> 16;
    return h1;
}
__device__ __forceinline__ uint32_t murmur3_u32(uint32_t v, uint32_t seed) { return mm_fmix(mm_mix_h1(seed, mm_mix_k1(v)), 4); }
// mur.rs:76-87 hash_long == bytes path over 8 LE bytes
__device__ __forceinline__ uint32_t murmur3_u64(uint64_t v, uint32_t seed) {
    uint32_t h1 = mm_mix_h1(seed, mm_mix_k1((uint32_t)v));
    h1 = mm_mix_h1(h1, mm_mix_k1((uint32_t)(v >> 32)));
    return mm_fmix(h1, 8);
}
__device__ __forceinline__ uint32_t murmur3_u128(uint64_t lo, uint64_t hi, uint32_t seed) {
    uint32_t h1 = mm_mix_h1(seed, mm_mix_k1((uint32_t)lo));
    h1 = mm_mix_h1(h1, mm_mix_k1((uint32_t)(lo >> 32)));
    h1 = mm_mix_h1(h1, mm_mix_k1((uint32_t)hi));
    h1 = mm_mix_h1(h1, mm_mix_k1((uint32_t)(hi >> 32)));
    return mm_fmix(h1, 16);
}
// mur.rs:19-30: aligned words, then each trailing byte sign-extended as its own block
__device__ __forceinline__ uint32_t murmur3_bytes(const uint8_t* p, int32_t len, uint32_t seed) {
    uint32_t h1 = seed;
    int32_t aligned = len & ~3;
    for (int32_t i = 0; i < aligned; i += 4) {
        uint32_t w = (uint32_t)p[i] | ((uint32_t)p[i + 1] << 8) | ((uint32_t)p[i + 2] << 16) | ((uint32_t)p[i + 3] << 24);
        h1 = mm_mix_h1(h1, mm_mix_k1(w));
    }
    for (int32_t i = aligned; i < len; i++) h1 = mm_mix_h1(h1, mm_mix_k1((uint32_t)(int32_t)(int8_t)p[i]));
    return mm_fmix(h1, (uint32_t)len);
}

// ---------------------------------------------------------------- xxhash64 (xxhash.rs:30-120)
#define XXP1 0x9E3779B185EBCA87ull
#define XXP2 0xC2B2AE3D27D4EB4Full
#define XXP3 0x165667B19E3779F9ull
#define XXP4 0x85EBCA77C2B2AE63ull
#define XXP5 0x27D4EB2F165667C5ull
__device__ __forceinline__ uint64_t rotl64(uint64_t x, int r) { return (x << r) | (x >> (64 - r)); }
__device__ __forceinline__ uint64_t xx_round(uint64_t acc, uint64_t in) {
    acc += in * XXP2;
    acc = rotl64(acc, 31);
    return acc * XXP1;
}
__device__ __forceinline__ uint64_t xx_merge(uint64_t h, uint64_t acc) {
    h ^= xx_round(0, acc);
    return h * XXP1 + XXP4;
}
__device__ __forceinline__ uint64_t xx_avalanche(uint64_t h) {
    h ^= h >> 33;
    h *= XXP2;
    h ^= h >> 29;
    h *= XXP3;
    h ^= h >> 32;
    return h;
}
__device__ __forceinline__ uint64_t rd64(const uint8_t* p) {
    uint64_t v = 0;
#pragma unroll
    for (int i = 0; i < 8; i++) v |= (uint64_t)p[i] << (8 * i);
    return v;
}
__device__ __forceinline__ uint32_t rd32(const uint8_t* p) {
    return (uint32_t)p[0] | ((uint32_t)p[1] << 8) | ((uint32_t)p[2] << 16) | ((uint32_t)p[3] << 24);
}
__device__ __forceinline__ uint64_t xxhash64_bytes(const uint8_t* in, int32_t len, uint64_t seed) {
    uint64_t h;
    int32_t rem = len, off = 0;
    if (rem >= 32) {
        uint64_t a1 = seed + XXP1 + XXP2, a2 = seed + XXP2, a3 = seed, a4 = seed - XXP1;
        while (rem >= 32) {
            a1 = xx_round(a1, rd64(in + off));
            a2 = xx_round(a2, rd64(in + off + 8));
            a3 = xx_round(a3, rd64(in + off + 16));
            a4 = xx_round(a4, rd64(in + off + 24));
            off += 32;
            rem -= 32;
        }
        h = rotl64(a1, 1) + rotl64(a2, 7) + rotl64(a3, 12) + rotl64(a4, 18);
        h = xx_merge(h, a1);
        h = xx_merge(h, a2);
        h = xx_merge(h, a3);
        h = xx_merge(h, a4);
    } else {
        h = seed + XXP5;
    }
    h += (uint64_t)len;
    while (rem >= 8) {
        h ^= xx_round(0, rd64(in + off));
        h = rotl64(h, 27) * XXP1 + XXP4;
        off += 8;
        rem -= 8;
    }
    if (rem >= 4) {
        h ^= (uint64_t)rd32(in + off) * XXP1;
        h = rotl64(h, 23) * XXP2 + XXP3;
        off += 4;
        rem -= 4;
    }
    while (rem) {
        h ^= (uint64_t)in[off] * XXP5;
        h = rotl64(h, 11) * XXP1;
        off++;
        rem--;
    }
    return xx_avalanche(h);
}
__device__ __forceinline__ uint64_t xxhash64_u32(uint32_t v, uint64_t seed) {
    uint64_t h = seed + XXP5 + 4;
    h ^= (uint64_t)v * XXP1;
    h = rotl64(h, 23) * XXP2 + XXP3;
    return xx_avalanche(h);
}
__device__ __forceinline__ uint64_t xxhash64_u64(uint64_t v, uint64_t seed) {
    uint64_t h = seed + XXP5 + 8;
    h ^= xx_round(0, v);
    h = rotl64(h, 27) * XXP1 + XXP4;
    return xx_avalanche(h);
}
__device__ __forceinline__ uint64_t xxhash64_u128(uint64_t lo, uint64_t hi, uint64_t seed) {
    uint64_t h = seed + XXP5 + 16;
    h ^= xx_round(0, lo);
    h = rotl64(h, 27) * XXP1 + XXP4;
    h ^= xx_round(0, hi);
    h = rotl64(h, 27) * XXP1 + XXP4;
    return xx_avalanche(h);
}

// internal (non-Spark) 64-bit mixer for hash tables; results never leave an operator
// (the reference uses foldhash there: agg_hash_map.rs:228-234, join_hash_map.rs:441-457)
__device__ __forceinline__ uint64_t mix64(uint64_t x) {
    x ^= x >> 33;
    x *= 0xff51afd7ed558ccdull;
    x ^= x >> 33;
    x *= 0xc4ceb9fe1a85ec53ull;
    x ^= x >> 33;
    return x;
}

// ---------------------------------------------------------------- int128 helpers (lo: u64, hi: i64)
struct i128 {
    uint64_t lo;
    int64_t hi;
};
__device__ __forceinline__ i128 i128_from_i64(int64_t v) { return {(uint64_t)v, v < 0 ? -1ll : 0ll}; }
__device__ __forceinline__ i128 i128_add(i128 a, i128 b) {
    i128 r;
    r.lo = a.lo + b.lo;
    r.hi = a.hi + b.hi + (r.lo < a.lo ? 1 : 0);
    return r;
}
__device__ __forceinline__ i128 i128_neg(i128 a) {
    i128 r;
    r.lo = ~a.lo + 1;
    r.hi = ~a.hi + (r.lo == 0 ? 1 : 0);
    return r;
}
__device__ __forceinline__ i128 i128_sub(i128 a, i128 b) { return i128_add(a, i128_neg(b)); }
__device__ __forceinline__ int i128_cmp(i128 a, i128 b) {
    if (a.hi != b.hi) return a.hi < b.hi ? -1 : 1;
    if (a.lo != b.lo) return a.lo < b.lo ? -1 : 1;
    return 0;
}
__device__ __forceinline__ bool i128_is_neg(i128 a) { return a.hi < 0; }
// unsigned 128 x 64 -> low 128 (wrapping)
__device__ __forceinline__ i128 u128_mul_u64(i128 a, uint64_t m) {
    i128 r;
    r.lo = a.lo * m;
    r.hi = (int64_t)(__umul64hi(a.lo, m) + (uint64_t)a.hi * m);
    return r;
}
// signed 128 x signed 128 -> low 128 (wrapping)
__device__ __forceinline__ i128 i128_mul(i128 a, i128 b) {
    i128 r;
    r.lo = a.lo * b.lo;
    r.hi = (int64_t)(__umul64hi(a.lo, b.lo) + a.lo * (uint64_t)b.hi + (uint64_t)a.hi * b.lo);
    return r;
}
// unsigned 128 / 64 -> quotient (128) and remainder (64); simple bitwise long division
__device__ inline i128 u128_divmod_u64(i128 a, uint64_t d, uint64_t* rem) {
    uint64_t hi = (uint64_t)a.hi, lo = a.lo;
    uint64_t qhi = hi / d, r = hi % d, qlo = 0;
    for (int i = 63; i >= 0; i--) {
        uint64_t top = r >> 63;
        r = (r << 1) | ((lo >> i) & 1);
        if (top || r >= d) {
            r -= d;
            qlo |= 1ull << i;
        }
    }
    *rem = r;
    return {qlo, (int64_t)qhi};
}

// ---- warp-cooperative byte copy (page decompression, shuffle block assembly)
// 16 bytes of the byte stream that starts `sb` (0..15) bytes into the aligned vector pair (a, b)
__device__ __forceinline__ uint4 shift16(const uint4& a, const uint4& b, unsigned sb) {
    const unsigned bs = (sb & 3) * 8;
    uint4 r;
    switch (sb >> 2) {   // uniform across the warp
        case 0: r.x = __funnelshift_r(a.x, a.y, bs), r.y = __funnelshift_r(a.y, a.z, bs), r.z = __funnelshift_r(a.z, a.w, bs), r.w = __funnelshift_r(a.w, b.x, bs); break;
        case 1: r.x = __funnelshift_r(a.y, a.z, bs), r.y = __funnelshift_r(a.z, a.w, bs), r.z = __funnelshift_r(a.w, b.x, bs), r.w = __funnelshift_r(b.x, b.y, bs); break;
        case 2: r.x = __funnelshift_r(a.z, a.w, bs), r.y = __funnelshift_r(a.w, b.x, bs), r.z = __funnelshift_r(b.x, b.y, bs), r.w = __funnelshift_r(b.y, b.z, bs); break;
        default: r.x = __funnelshift_r(a.w, b.x, bs), r.y = __funnelshift_r(b.x, b.y, bs), r.z = __funnelshift_r(b.y, b.z, bs), r.w = __funnelshift_r(b.z, b.w, bs); break;
    }
    return r;
}
// dst[0, len) = src[0, len); no overlap; any alignment.  Bulk: 16-byte stores at the destination's alignment, the source
// re-aligned from two 16-byte loads (512 B per warp instruction, two vectors in flight per lane).
__device__ __forceinline__ void warp_copy(uint8_t* __restrict__ dst, const uint8_t* __restrict__ src, int64_t len, unsigned lane) {
    if (len < 256) {
        for (int64_t i = lane; i < len; i += 32) dst[i] = src[i];
        return;
    }
    const int head = (int)((16 - ((uintptr_t)dst & 15)) & 15);
    if ((int)lane < head) dst[lane] = src[lane];
    dst += head;
    src += head;
    len -= head;
    int64_t nv = len >> 4;                       // whole 16-byte vectors
    const uintptr_t sa = (uintptr_t)src;
    const uint4* sv = (const uint4*)(sa & ~(uintptr_t)15);
    const unsigned sb = (unsigned)(sa & 15);
    uint4* dv = (uint4*)dst;
    if (sb == 0) {
        int64_t j = lane;
        for (; j + 32 < nv; j += 64) {
            const uint4 a = sv[j], b = sv[j + 32];
            dv[j] = a;
            dv[j + 32] = b;
        }
        for (; j < nv; j += 32) dv[j] = sv[j];
    } else {
        // the last vector would read 16 bytes past the source's aligned end: leave it to the byte tail
        nv -= 1;
        int64_t j = lane;
        for (; j + 32 < nv; j += 64) {
            const uint4 a0 = sv[j], a1 = sv[j + 1], b0 = sv[j + 32], b1 = sv[j + 33];
            dv[j] = shift16(a0, a1, sb);
            dv[j + 32] = shift16(b0, b1, sb);
        }
        for (; j < nv; j += 32) dv[j] = shift16(sv[j], sv[j + 1], sb);
    }
    for (int64_t i = (nv << 4) + lane; i < len; i += 32) dst[i] = src[i];
}


}  // namespace auron
