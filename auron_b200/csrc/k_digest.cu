// k_digest.cu -- Spark md5 / sha2 of a utf8 or binary column as lowercase hex (spark_crypto.rs:33-105).
//
// One thread hashes one row: a digest is serial over the blocks of its message, and the rows of a batch are independent.
// The message is read with aligned 4-byte loads joined by funnel shifts; a load only touches a word that holds at least
// one byte of the message, so no producer of string buffers has to keep tail padding for it.  State and message schedule
// live in registers (the rounds are unrolled, every index is a constant); the round constants come from constant memory.
// NULL rows have an empty output, every other row 32 / 56 / 64 / 96 / 128 characters, so every output offset is a multiple
// of 8 and the hex goes out as aligned 8-byte stores.
//
// The compression functions and the padding walk are __host__ __device__: auron_b200_digest_hex runs the same code on the
// CPU, which pins the padding edge cases without a GPU.
#include "device_utils.cuh"
#include "kernels.h"

namespace auron {

#define MD5_K_LIST 0xd76aa478u, 0xe8c7b756u, 0x242070dbu, 0xc1bdceeeu, 0xf57c0fafu, 0x4787c62au, 0xa8304613u, 0xfd469501u, \
    0x698098d8u, 0x8b44f7afu, 0xffff5bb1u, 0x895cd7beu, 0x6b901122u, 0xfd987193u, 0xa679438eu, 0x49b40821u, \
    0xf61e2562u, 0xc040b340u, 0x265e5a51u, 0xe9b6c7aau, 0xd62f105du, 0x02441453u, 0xd8a1e681u, 0xe7d3fbc8u, \
    0x21e1cde6u, 0xc33707d6u, 0xf4d50d87u, 0x455a14edu, 0xa9e3e905u, 0xfcefa3f8u, 0x676f02d9u, 0x8d2a4c8au, \
    0xfffa3942u, 0x8771f681u, 0x6d9d6122u, 0xfde5380cu, 0xa4beea44u, 0x4bdecfa9u, 0xf6bb4b60u, 0xbebfbc70u, \
    0x289b7ec6u, 0xeaa127fau, 0xd4ef3085u, 0x04881d05u, 0xd9d4d039u, 0xe6db99e5u, 0x1fa27cf8u, 0xc4ac5665u, \
    0xf4292244u, 0x432aff97u, 0xab9423a7u, 0xfc93a039u, 0x655b59c3u, 0x8f0ccc92u, 0xffeff47du, 0x85845dd1u, \
    0x6fa87e4fu, 0xfe2ce6e0u, 0xa3014314u, 0x4e0811a1u, 0xf7537e82u, 0xbd3af235u, 0x2ad7d2bbu, 0xeb86d391u
#define SHA256_K_LIST 0x428a2f98u, 0x71374491u, 0xb5c0fbcfu, 0xe9b5dba5u, 0x3956c25bu, 0x59f111f1u, 0x923f82a4u, 0xab1c5ed5u, \
    0xd807aa98u, 0x12835b01u, 0x243185beu, 0x550c7dc3u, 0x72be5d74u, 0x80deb1feu, 0x9bdc06a7u, 0xc19bf174u, \
    0xe49b69c1u, 0xefbe4786u, 0x0fc19dc6u, 0x240ca1ccu, 0x2de92c6fu, 0x4a7484aau, 0x5cb0a9dcu, 0x76f988dau, \
    0x983e5152u, 0xa831c66du, 0xb00327c8u, 0xbf597fc7u, 0xc6e00bf3u, 0xd5a79147u, 0x06ca6351u, 0x14292967u, \
    0x27b70a85u, 0x2e1b2138u, 0x4d2c6dfcu, 0x53380d13u, 0x650a7354u, 0x766a0abbu, 0x81c2c92eu, 0x92722c85u, \
    0xa2bfe8a1u, 0xa81a664bu, 0xc24b8b70u, 0xc76c51a3u, 0xd192e819u, 0xd6990624u, 0xf40e3585u, 0x106aa070u, \
    0x19a4c116u, 0x1e376c08u, 0x2748774cu, 0x34b0bcb5u, 0x391c0cb3u, 0x4ed8aa4au, 0x5b9cca4fu, 0x682e6ff3u, \
    0x748f82eeu, 0x78a5636fu, 0x84c87814u, 0x8cc70208u, 0x90befffau, 0xa4506cebu, 0xbef9a3f7u, 0xc67178f2u
#define SHA512_K_LIST 0x428a2f98d728ae22ull, 0x7137449123ef65cdull, 0xb5c0fbcfec4d3b2full, 0xe9b5dba58189dbbcull, \
    0x3956c25bf348b538ull, 0x59f111f1b605d019ull, 0x923f82a4af194f9bull, 0xab1c5ed5da6d8118ull, \
    0xd807aa98a3030242ull, 0x12835b0145706fbeull, 0x243185be4ee4b28cull, 0x550c7dc3d5ffb4e2ull, \
    0x72be5d74f27b896full, 0x80deb1fe3b1696b1ull, 0x9bdc06a725c71235ull, 0xc19bf174cf692694ull, \
    0xe49b69c19ef14ad2ull, 0xefbe4786384f25e3ull, 0x0fc19dc68b8cd5b5ull, 0x240ca1cc77ac9c65ull, \
    0x2de92c6f592b0275ull, 0x4a7484aa6ea6e483ull, 0x5cb0a9dcbd41fbd4ull, 0x76f988da831153b5ull, \
    0x983e5152ee66dfabull, 0xa831c66d2db43210ull, 0xb00327c898fb213full, 0xbf597fc7beef0ee4ull, \
    0xc6e00bf33da88fc2ull, 0xd5a79147930aa725ull, 0x06ca6351e003826full, 0x142929670a0e6e70ull, \
    0x27b70a8546d22ffcull, 0x2e1b21385c26c926ull, 0x4d2c6dfc5ac42aedull, 0x53380d139d95b3dfull, \
    0x650a73548baf63deull, 0x766a0abb3c77b2a8ull, 0x81c2c92e47edaee6ull, 0x92722c851482353bull, \
    0xa2bfe8a14cf10364ull, 0xa81a664bbc423001ull, 0xc24b8b70d0f89791ull, 0xc76c51a30654be30ull, \
    0xd192e819d6ef5218ull, 0xd69906245565a910ull, 0xf40e35855771202aull, 0x106aa07032bbd1b8ull, \
    0x19a4c116b8d2d0c8ull, 0x1e376c085141ab53ull, 0x2748774cdf8eeb99ull, 0x34b0bcb5e19b48a8ull, \
    0x391c0cb3c5c95a63ull, 0x4ed8aa4ae3418acbull, 0x5b9cca4f7763e373ull, 0x682e6ff3d6b2b8a3ull, \
    0x748f82ee5defb2fcull, 0x78a5636f43172f60ull, 0x84c87814a1f0ab72ull, 0x8cc702081a6439ecull, \
    0x90befffa23631e28ull, 0xa4506cebde82bde9ull, 0xbef9a3f7b2c67915ull, 0xc67178f2e372532bull, \
    0xca273eceea26619cull, 0xd186b8c721c0c207ull, 0xeada7dd6cde0eb1eull, 0xf57d4f7fee6ed178ull, \
    0x06f067aa72176fbaull, 0x0a637dc5a2c898a6ull, 0x113f9804bef90daeull, 0x1b710b35131c471bull, \
    0x28db77f523047d84ull, 0x32caab7b40c72493ull, 0x3c9ebe0a15c9bebcull, 0x431d67c49c100d4cull, \
    0x4cc5d4becb3e42b6ull, 0x597f299cfc657e2aull, 0x5fcb6fab3ad6faecull, 0x6c44198c4a475817ull
__constant__ uint32_t d_md5_k[64] = {MD5_K_LIST};
__constant__ uint32_t d_sha256_k[64] = {SHA256_K_LIST};
__constant__ uint64_t d_sha512_k[80] = {SHA512_K_LIST};
#ifndef __CUDA_ARCH__
static const uint32_t h_md5_k[64] = {MD5_K_LIST};
static const uint32_t h_sha256_k[64] = {SHA256_K_LIST};
static const uint64_t h_sha512_k[80] = {SHA512_K_LIST};
#endif

// the host compiler of the __host__ __device__ functions below does not know `#pragma unroll`
#ifdef __CUDA_ARCH__
#define DIGEST_K(name, i) d_##name##_k[i]
#define DIGEST_UNROLL _Pragma("unroll")
#else
#define DIGEST_K(name, i) h_##name##_k[i]
#define DIGEST_UNROLL
#endif

__host__ __device__ __forceinline__ uint32_t rotr32(uint32_t x, int n) {
#ifdef __CUDA_ARCH__
    return __funnelshift_r(x, x, n);
#else
    return (x >> n) | (x << ((32 - n) & 31));
#endif
}
__host__ __device__ __forceinline__ uint64_t rotr64(uint64_t x, int n) { return (x >> n) | (x << (64 - n)); }
__host__ __device__ __forceinline__ uint32_t bswap32(uint32_t x) {
#ifdef __CUDA_ARCH__
    return __byte_perm(x, 0, 0x0123);
#else
    return __builtin_bswap32(x);
#endif
}

// ---- compression functions (RFC 1321, FIPS 180-4).  x = the block as little-endian 32-bit words, as it lies in memory.
__host__ __device__ __forceinline__ void md5_compress(uint32_t st[4], const uint32_t x[16]) {
    uint32_t a = st[0], b = st[1], c = st[2], d = st[3];
DIGEST_UNROLL
    for (int i = 0; i < 64; i++) {
        uint32_t f;
        int g, s;
        if (i < 16) {
            f = (b & c) | (~b & d);
            g = i;
            s = (i & 3) == 0 ? 7 : (i & 3) == 1 ? 12 : (i & 3) == 2 ? 17 : 22;
        } else if (i < 32) {
            f = (d & b) | (~d & c);
            g = (5 * i + 1) & 15;
            s = (i & 3) == 0 ? 5 : (i & 3) == 1 ? 9 : (i & 3) == 2 ? 14 : 20;
        } else if (i < 48) {
            f = b ^ c ^ d;
            g = (3 * i + 5) & 15;
            s = (i & 3) == 0 ? 4 : (i & 3) == 1 ? 11 : (i & 3) == 2 ? 16 : 23;
        } else {
            f = c ^ (b | ~d);
            g = (7 * i) & 15;
            s = (i & 3) == 0 ? 6 : (i & 3) == 1 ? 10 : (i & 3) == 2 ? 15 : 21;
        }
        const uint32_t t = d;
        d = c;
        c = b;
        b = b + rotr32(a + f + DIGEST_K(md5, i) + x[g], 32 - s);
        a = t;
    }
    st[0] += a, st[1] += b, st[2] += c, st[3] += d;
}

__host__ __device__ __forceinline__ void sha256_compress(uint32_t st[8], const uint32_t x[16]) {
    uint32_t w[16];
DIGEST_UNROLL
    for (int i = 0; i < 16; i++) w[i] = bswap32(x[i]);
    uint32_t a = st[0], b = st[1], c = st[2], d = st[3], e = st[4], f = st[5], g = st[6], h = st[7];
DIGEST_UNROLL
    for (int i = 0; i < 64; i++) {
        if (i >= 16) {
            const uint32_t w15 = w[(i + 1) & 15], w2 = w[(i + 14) & 15];
            w[i & 15] += (rotr32(w15, 7) ^ rotr32(w15, 18) ^ (w15 >> 3)) + w[(i + 9) & 15] + (rotr32(w2, 17) ^ rotr32(w2, 19) ^ (w2 >> 10));
        }
        const uint32_t t1 = h + (rotr32(e, 6) ^ rotr32(e, 11) ^ rotr32(e, 25)) + ((e & f) ^ (~e & g)) + DIGEST_K(sha256, i) + w[i & 15];
        const uint32_t t2 = (rotr32(a, 2) ^ rotr32(a, 13) ^ rotr32(a, 22)) + ((a & b) ^ (a & c) ^ (b & c));
        h = g, g = f, f = e, e = d + t1, d = c, c = b, b = a, a = t1 + t2;
    }
    st[0] += a, st[1] += b, st[2] += c, st[3] += d, st[4] += e, st[5] += f, st[6] += g, st[7] += h;
}

// x = the 128-byte block as 32 little-endian 32-bit words
__host__ __device__ __forceinline__ void sha512_compress(uint64_t st[8], const uint32_t x[32]) {
    uint64_t w[16];
DIGEST_UNROLL
    for (int i = 0; i < 16; i++) w[i] = ((uint64_t)bswap32(x[2 * i]) << 32) | bswap32(x[2 * i + 1]);
    uint64_t a = st[0], b = st[1], c = st[2], d = st[3], e = st[4], f = st[5], g = st[6], h = st[7];
DIGEST_UNROLL
    for (int i = 0; i < 80; i++) {
        if (i >= 16) {
            const uint64_t w15 = w[(i + 1) & 15], w2 = w[(i + 14) & 15];
            w[i & 15] += (rotr64(w15, 1) ^ rotr64(w15, 8) ^ (w15 >> 7)) + w[(i + 9) & 15] + (rotr64(w2, 19) ^ rotr64(w2, 61) ^ (w2 >> 6));
        }
        const uint64_t t1 = h + (rotr64(e, 14) ^ rotr64(e, 18) ^ rotr64(e, 41)) + ((e & f) ^ (~e & g)) + DIGEST_K(sha512, i) + w[i & 15];
        const uint64_t t2 = (rotr64(a, 28) ^ rotr64(a, 34) ^ rotr64(a, 39)) + ((a & b) ^ (a & c) ^ (b & c));
        h = g, g = f, f = e, e = d + t1, d = c, c = b, b = a, a = t1 + t2;
    }
    st[0] += a, st[1] += b, st[2] += c, st[3] += d, st[4] += e, st[5] += f, st[6] += g, st[7] += h;
}

// ---- message readers: word(q) = the 4 message bytes at offset q (q < len, q % 4 == 0) as a little-endian word; bytes at
// len and beyond are unspecified.  block(o, x) fills x with the NW words at offset o when o + 4 * NW <= len.
struct DeviceMessage {
    const uint32_t* w;   // the message's first byte rounded down to 4-byte alignment
    int sh;              // 8 * misalignment
    __device__ DeviceMessage(const uint8_t* p) : w((const uint32_t*)((uintptr_t)p & ~(uintptr_t)3)), sh((int)((uintptr_t)p & 3) * 8) {}
    // word q/4 and, when the message is misaligned, the next one: it holds message byte q + 3 - sh/8 only if q + 4 < len + sh/8
    __device__ __forceinline__ uint32_t word(int64_t q, int64_t len) const {
        const uint32_t lo = __ldg(w + (q >> 2));
        const uint32_t hi = (sh != 0 && q + 4 < len + (sh >> 3)) ? __ldg(w + (q >> 2) + 1) : 0u;
        return __funnelshift_r(lo, hi, sh);
    }
    template <int NW>
    __device__ __forceinline__ void block(int64_t o, uint32_t (&x)[NW]) const {
        uint32_t a[NW + 1];
DIGEST_UNROLL
        for (int k = 0; k < NW; k++) a[k] = __ldg(w + (o >> 2) + k);
        a[NW] = sh ? __ldg(w + (o >> 2) + NW) : 0u;   // holds message byte o + 4 NW - sh/8 < len
DIGEST_UNROLL
        for (int k = 0; k < NW; k++) x[k] = __funnelshift_r(a[k], a[k + 1], sh);
    }
};
struct HostMessage {
    const uint8_t* p;
    __host__ __device__ uint32_t word(int64_t q, int64_t len) const {
        uint32_t r = 0;
        for (int j = 0; j < 4 && q + j < len; j++) r |= (uint32_t)p[q + j] << (8 * j);
        return r;
    }
    template <int NW>
    __host__ __device__ void block(int64_t o, uint32_t (&x)[NW]) const {
        for (int k = 0; k < NW; k++) x[k] = word(o + 4 * k, o + 4 * NW);
    }
};

// The padded block at offset o: message bytes, 0x80 at offset len, zeros after.
template <int NW, class Msg>
__host__ __device__ __forceinline__ void padded_block(const Msg& m, int64_t o, int64_t len, uint32_t (&x)[NW]) {
    if (o + 4 * NW <= len) {
        m.block(o, x);
        return;
    }
DIGEST_UNROLL
    for (int k = 0; k < NW; k++) {
        const int64_t q = o + 4 * k, r = len - q;   // message bytes in this word
        uint32_t v = r > 0 ? m.word(q, len) : 0u;
        if (r < 4) v = r > 0 ? (v & ((1u << (8 * r)) - 1u)) | (0x80u << (8 * r)) : (r == 0 ? 0x80u : 0u);
        x[k] = v;
    }
}

// FAM 0: MD5, 1: SHA-256 / SHA-224 (trunc), 2: SHA-512 / SHA-384 (trunc).  Writes the digest as big-endian-ordered 32-bit
// words (out[0] holds the first four digest bytes, most significant first); returns their number.
template <int FAM, class Msg>
__host__ __device__ __forceinline__ int digest_words(const Msg& m, int64_t len, bool trunc, uint32_t out[16]) {
    if (FAM == 0) {
        uint32_t st[4] = {0x67452301u, 0xefcdab89u, 0x98badcfeu, 0x10325476u};
        const int64_t nb = (len + 8) / 64 + 1;
        for (int64_t b = 0; b < nb; b++) {
            uint32_t x[16];
            padded_block<16>(m, b * 64, len, x);
            if (b == nb - 1) {
                x[14] = (uint32_t)((uint64_t)len << 3);
                x[15] = (uint32_t)((uint64_t)len >> 29);
            }
            md5_compress(st, x);
        }
DIGEST_UNROLL
        for (int k = 0; k < 4; k++) out[k] = bswap32(st[k]);
        return 4;
    } else if (FAM == 1) {
        uint32_t st[8];
        if (trunc) st[0] = 0xc1059ed8u, st[1] = 0x367cd507u, st[2] = 0x3070dd17u, st[3] = 0xf70e5939u, st[4] = 0xffc00b31u, st[5] = 0x68581511u, st[6] = 0x64f98fa7u, st[7] = 0xbefa4fa4u;
        else st[0] = 0x6a09e667u, st[1] = 0xbb67ae85u, st[2] = 0x3c6ef372u, st[3] = 0xa54ff53au, st[4] = 0x510e527fu, st[5] = 0x9b05688cu, st[6] = 0x1f83d9abu, st[7] = 0x5be0cd19u;
        const int64_t nb = (len + 8) / 64 + 1;
        for (int64_t b = 0; b < nb; b++) {
            uint32_t x[16];
            padded_block<16>(m, b * 64, len, x);
            if (b == nb - 1) {   // big-endian bit length in the last 8 bytes
                x[14] = bswap32((uint32_t)((uint64_t)len >> 29));
                x[15] = bswap32((uint32_t)((uint64_t)len << 3));
            }
            sha256_compress(st, x);
        }
DIGEST_UNROLL
        for (int k = 0; k < 8; k++) out[k] = st[k];
        return trunc ? 7 : 8;
    } else {
        uint64_t st[8];
        if (trunc) st[0] = 0xcbbb9d5dc1059ed8ull, st[1] = 0x629a292a367cd507ull, st[2] = 0x9159015a3070dd17ull, st[3] = 0x152fecd8f70e5939ull, st[4] = 0x67332667ffc00b31ull, st[5] = 0x8eb44a8768581511ull, st[6] = 0xdb0c2e0d64f98fa7ull, st[7] = 0x47b5481dbefa4fa4ull;
        else st[0] = 0x6a09e667f3bcc908ull, st[1] = 0xbb67ae8584caa73bull, st[2] = 0x3c6ef372fe94f82bull, st[3] = 0xa54ff53a5f1d36f1ull, st[4] = 0x510e527fade682d1ull, st[5] = 0x9b05688c2b3e6c1full, st[6] = 0x1f83d9abfb41bd6bull, st[7] = 0x5be0cd19137e2179ull;
        const int64_t nb = (len + 16) / 128 + 1;
        for (int64_t b = 0; b < nb; b++) {
            uint32_t x[32];
            padded_block<32>(m, b * 128, len, x);
            if (b == nb - 1) {   // 128-bit big-endian bit length: high 64 bits are zero for any int64 length
                x[28] = 0;
                x[29] = 0;
                x[30] = bswap32((uint32_t)((uint64_t)len >> 29));
                x[31] = bswap32((uint32_t)((uint64_t)len << 3));
            }
            sha512_compress(st, x);
        }
DIGEST_UNROLL
        for (int k = 0; k < 8; k++) {
            out[2 * k] = (uint32_t)(st[k] >> 32);
            out[2 * k + 1] = (uint32_t)st[k];
        }
        return trunc ? 12 : 16;
    }
}

// 8 lowercase hex characters of w, most significant nibble first, packed little-endian (first character in the low byte)
__host__ __device__ __forceinline__ uint64_t hex8(uint32_t w) {
    uint64_t r = 0;
DIGEST_UNROLL
    for (int k = 0; k < 8; k++) {
        const uint32_t c = (w >> (28 - 4 * k)) & 15u;
        r |= (uint64_t)(c < 10 ? '0' + c : 'a' - 10 + c) << (8 * k);
    }
    return r;
}

struct DigestArgs {
    const int32_t* in_off;
    const uint8_t* in_data;
    const int32_t* sel;       // row ids (nullptr: row i)
    const int32_t* out_off;   // out_off[i + 1] == out_off[i] <=> row i is NULL
    uint64_t* out;
    int64_t n;
    int32_t trunc;
};

template <int FAM>
__global__ void __launch_bounds__(256) digest_kernel(DigestArgs a) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < a.n; i += (int64_t)gridDim.x * blockDim.x) {
        const int32_t o0 = a.out_off[i];
        if (a.out_off[i + 1] == o0) continue;
        const int64_t row = a.sel ? (int64_t)a.sel[i] : i;
        const int32_t b = a.in_off[row];
        const DeviceMessage m(a.in_data + b);
        uint32_t d[16];
        const int nw = digest_words<FAM>(m, (int64_t)(a.in_off[row + 1] - b), a.trunc != 0, d);
        uint64_t* out = a.out + (o0 >> 3);
DIGEST_UNROLL
        for (int k = 0; k < 16; k++)
            if (k < nw) out[k] = hex8(d[k]);
    }
}

// lens[i] = valid(row) ? width : 0 and the validity word of every 32 outputs
__global__ void digest_lengths_kernel(const uint8_t* __restrict__ in_valid, const int32_t* __restrict__ sel, int64_t n, int32_t width,
                                      uint32_t* __restrict__ out_valid, int64_t* __restrict__ lens) {
    for (int64_t base = (int64_t)blockIdx.x * blockDim.x; base < n; base += (int64_t)gridDim.x * blockDim.x) {
        const int64_t i = base + threadIdx.x;
        const bool active = i < n;
        const bool v = active && valid_at(in_valid, sel ? (int64_t)sel[i] : i);
        if (active) lens[i] = v ? width : 0;
        const uint32_t w = __ballot_sync(FULL_MASK, v);
        if ((threadIdx.x & 31) == 0 && active) out_valid[i >> 5] = w;
    }
}

int digest_hex_width(int alg) {
    switch (alg) {
        case DIGEST_MD5: return 32;
        case DIGEST_SHA224: return 56;
        case DIGEST_SHA256: return 64;
        case DIGEST_SHA384: return 96;
        case DIGEST_SHA512: return 128;
    }
    return -1;
}

void digest_lengths(Ctx& ctx, const uint8_t* in_valid, const int32_t* sel, int64_t n, int alg, uint32_t* out_valid, int64_t* lens) {
    if (n == 0) return;
    const unsigned grid = (unsigned)std::max<int64_t>(1, std::min<int64_t>((n + 255) / 256, (int64_t)ctx.sm_count * 8));
    digest_lengths_kernel<<<grid, 256, 0, ctx.stream>>>(in_valid, sel, n, digest_hex_width(alg), out_valid, lens);
    CUDA_OK(cudaGetLastError());
    launch_count(ctx);
}

void digest_hex(Ctx& ctx, int alg, const int32_t* in_off, const uint8_t* in_data, const int32_t* sel, int64_t n, const int32_t* out_off,
                uint8_t* out) {
    if (n == 0) return;
    DigestArgs a{in_off, in_data, sel, out_off, (uint64_t*)out, n, alg == DIGEST_SHA224 || alg == DIGEST_SHA384};
    const unsigned grid = (unsigned)std::max<int64_t>(1, std::min<int64_t>((n + 255) / 256, (int64_t)ctx.sm_count * 16));
    if (alg == DIGEST_MD5) {
        ProfScope ps(ctx, "digest_md5");
        digest_kernel<0><<<grid, 256, 0, ctx.stream>>>(a);
    } else if (alg == DIGEST_SHA224 || alg == DIGEST_SHA256) {
        ProfScope ps(ctx, "digest_sha256");
        digest_kernel<1><<<grid, 256, 0, ctx.stream>>>(a);
    } else {
        ProfScope ps(ctx, "digest_sha512");
        digest_kernel<2><<<grid, 256, 0, ctx.stream>>>(a);
    }
    CUDA_OK(cudaGetLastError());
    launch_count(ctx);
}

int digest_hex_host(int alg, const uint8_t* bytes, int64_t len, char* out) {
    const int width = digest_hex_width(alg);
    if (width < 0 || len < 0 || (len > 0 && !bytes)) return -1;
    const HostMessage m{bytes};
    uint32_t d[16];
    int nw;
    if (alg == DIGEST_MD5) nw = digest_words<0>(m, len, false, d);
    else if (alg == DIGEST_SHA224 || alg == DIGEST_SHA256) nw = digest_words<1>(m, len, alg == DIGEST_SHA224, d);
    else nw = digest_words<2>(m, len, alg == DIGEST_SHA384, d);
    for (int k = 0; k < nw; k++) {
        const uint64_t h = hex8(d[k]);
        memcpy(out + 8 * k, &h, 8);
    }
    return width;
}

}  // namespace auron
