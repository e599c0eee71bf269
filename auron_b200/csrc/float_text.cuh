// float_text.cuh -- Spark's CAST between utf8 and float32 / float64 (Cast.castToDouble / castToFloat, Double.toString /
// Float.toString), __host__ __device__ so that auron_b200_text_to_float / auron_b200_float_to_text run the device code on the
// CPU.  Included by k_expr.cu only.
//
// text -> float: Java's Double.parseDouble / Float.parseFloat grammar, then Spark's lower-cased special literals; the result
// is correctly rounded (nearest, ties to even) straight to the target width.  Up to 19 significant digits go through the
// Eisel-Lemire multiplication by a 128-bit truncated power of five (Lemire, "Number parsing at a gigabyte per second", 2021);
// a product too close to a rounding boundary, and longer inputs whose two 19-digit bounds round apart, go to an exact
// comparison of the decimal with the halfway point between two neighbouring floats on a fixed-size bignum.  Only the first
// 769 (binary64) / 114 (binary32) significant digits can decide that comparison; the rest contribute a sticky bit.
//
// float -> text: Giulietti's Schubfach ("The Schubfach way to render doubles", 2020), whose output is the JDK 19+
// specification: the decimal closest to x among the shortest that round to x (among those of length 1 or 2 when the
// shortest has one digit), ties to an even digit, laid out as plain digits for 10^-3 <= |d| < 10^7 and as d.dddE[-]n
// otherwise.  Both widths use the same 126-bit table of g = floor(10^-k 2^r) + 1.
#pragma once
#include <stdint.h>

#include "float_tables.h"

namespace auron {

static __device__ const uint64_t ft_pow5_d[] = {FT_POW5_LIST};
static __device__ const uint64_t ft_g_d[] = {FT_G_LIST};
#ifdef __CUDA_ARCH__
// rows of one warp index different entries: the read-only path, not __constant__ (which serialises distinct addresses)
#define FT_POW5(i) __ldg(&ft_pow5_d[i])
#define FT_G(i) __ldg(&ft_g_d[i])
#define FT_NOINLINE __noinline__
#else
static const uint64_t ft_pow5_h[] = {FT_POW5_LIST};
static const uint64_t ft_g_h[] = {FT_G_LIST};
#define FT_POW5(i) ft_pow5_h[i]
#define FT_G(i) ft_g_h[i]
#define FT_NOINLINE
#endif

__host__ __device__ __forceinline__ void ft_mul64(uint64_t a, uint64_t b, uint64_t* hi, uint64_t* lo) {
#ifdef __CUDA_ARCH__
    *lo = a * b;
    *hi = __umul64hi(a, b);
#else
    const unsigned __int128 p = (unsigned __int128)a * b;
    *lo = (uint64_t)p;
    *hi = (uint64_t)(p >> 64);
#endif
}
__host__ __device__ __forceinline__ int ft_clz64(uint64_t x) {
#ifdef __CUDA_ARCH__
    return __clzll((long long)x);
#else
    return __builtin_clzll(x);
#endif
}

// The binary formats: bits 64 or 32.
struct FtFormat {
    int mbits, bias;
    uint64_t inf;   // bit pattern of +infinity
    __host__ __device__ explicit FtFormat(int bits) : mbits(bits == 64 ? 52 : 23), bias(bits == 64 ? 1023 : 127), inf(bits == 64 ? 0x7ffull << 52 : 0xffull << 23) {}
};

// ------------------------------------------------------------------------------------------------ text -> float
// Eisel-Lemire: the non-negative bit pattern nearest w * 10^q (w != 0, FT_POW5_MIN <= q <= FT_POW5_MAX).  *ok is false when
// the 128-bit product leaves the rounding undecided; the pattern is then within one unit of the answer.
__host__ __device__ __forceinline__ uint64_t ft_eisel_lemire(uint64_t w, int64_t q, const FtFormat& f, bool* ok) {
    *ok = true;
    const int lz = ft_clz64(w);
    w <<= lz;
    const int ti = 2 * (int)(q - FT_POW5_MIN);
    uint64_t fh, fl, sh, sl;
    ft_mul64(w, FT_POW5(ti), &fh, &fl);
    ft_mul64(w, FT_POW5(ti + 1), &sh, &sl);
    // P = floor(w * T / 2^64) = (fh:fl) + sh; the exact w * 5^q * 2^s lies in [P, P + 2) (in units of the low word)
    const uint64_t lo = fl + sh;
    const uint64_t hi = fh + (lo < fl);
    const int ub = (int)(hi >> 63);
    int drop = ub + 63 - (f.mbits + 2);   // bits of hi below the round bit
    int64_t be = ((q * 217706) >> 16) + 63 + ub - lz + f.bias;   // biased exponent if normal
    if (be <= 0) {   // subnormal: the round bit moves up, the exponent field is 0 (be = 1 with no implicit bit)
        drop += (int)(1 - be);
        be = 1;
    }
    if (drop >= 64) return 0;   // below half the least subnormal
    uint64_t m = hi >> drop;    // significand and round bit
    const uint64_t mask = (1ull << drop) - 1, below = hi & mask;
    if (!(m & 1)) {
        if (below == mask && lo >= ~1ull) *ok = false;   // the exact value may reach the halfway point
        m >>= 1;
    } else if (below == 0 && lo == 0) {   // the product is exactly halfway
        // exact only for 0 <= q <= 55 (5^q fits the table entry); then a nonzero dropped word means above halfway
        if (q >= 0 && q <= 55) m = (m >> 1) + (sl != 0 ? 1 : ((m >> 1) & 1));
        else {
            *ok = false;
            m = (m >> 1) + 1;
        }
    } else m = (m >> 1) + 1;
    // (be - 1) << mbits + m: the implicit bit of m carries into the exponent field, as does a significand rounded up to 2^(mbits+1)
    const uint64_t bits = ((uint64_t)(be - 1) << f.mbits) + m;
    return bits >= f.inf ? f.inf : bits;
}

// fixed-size unsigned bignum, 32-bit limbs, least significant first
constexpr int FT_LIMBS = 84;   // 2688 bits: 10^769 (2555 bits) and (2^54) * 5^1093 (2593 bits)
struct FtBig {
    uint32_t v[FT_LIMBS];
    int n;
};
__host__ __device__ inline void ft_big_muladd(FtBig& x, uint32_t m, uint32_t add) {
    uint64_t carry = add;
    for (int i = 0; i < x.n; i++) {
        const uint64_t t = (uint64_t)x.v[i] * m + carry;
        x.v[i] = (uint32_t)t;
        carry = t >> 32;
    }
    if (carry && x.n < FT_LIMBS) x.v[x.n++] = (uint32_t)carry;
}
__host__ __device__ inline void ft_big_mulpow5(FtBig& x, int64_t e) {
    for (; e >= 13; e -= 13) ft_big_muladd(x, 1220703125u, 0);   // 5^13
    uint32_t m = 1;
    for (; e > 0; e--) m *= 5;
    if (m > 1) ft_big_muladd(x, m, 0);
}
__host__ __device__ inline int64_t ft_big_bits(const FtBig& x) {
    int n = x.n;
    while (n > 0 && x.v[n - 1] == 0) n--;
    return n == 0 ? 0 : 32 * (int64_t)n - (ft_clz64(x.v[n - 1]) - 32);
}
// limb `idx` of x * 2^s
__host__ __device__ __forceinline__ uint32_t ft_big_limb_shl(const FtBig& x, int64_t s, int64_t idx) {
    const int64_t j = idx - (s >> 5);
    const int bs = (int)(s & 31);
    const uint32_t hi = (j >= 0 && j < x.n) ? x.v[j] : 0u;
    const uint32_t lo = (j >= 1 && j - 1 < x.n) ? x.v[j - 1] : 0u;
    return bs ? (hi << bs) | (lo >> (32 - bs)) : hi;
}
// sign of a * 2^ea - b * 2^eb
__host__ __device__ inline int ft_big_cmp(const FtBig& a, int64_t ea, const FtBig& b, int64_t eb) {
    const int64_t m = ea < eb ? ea : eb;
    ea -= m;
    eb -= m;
    const int64_t la = ft_big_bits(a) + ea, lb = ft_big_bits(b) + eb;
    if (la != lb) return la < lb ? -1 : 1;
    for (int64_t idx = (la + 31) / 32 - 1; idx >= 0; idx--) {
        const uint32_t x = ft_big_limb_shl(a, ea, idx), y = ft_big_limb_shl(b, eb, idx);
        if (x != y) return x < y ? -1 : 1;
    }
    return 0;
}

// Exact rounding of the decimal whose significand digits are s[first, end) (a '.' skipped) times 10^q, nd significant
// digits, starting from a pattern `b` within a few units of the answer: walks b to the float whose rounding interval holds
// the decimal, comparing with the halfway points exactly.
FT_NOINLINE __host__ __device__ inline uint64_t ft_parse_exact(const uint8_t* s, int32_t first, int32_t end, int64_t nd, int64_t q, const FtFormat& f,
                                                              uint64_t b) {
    const int64_t cap = f.mbits == 52 ? 769 : 114;
    const int64_t nk = nd < cap ? nd : cap;
    const int64_t qk = q + (nd - nk);
    FtBig a;
    a.n = 1;
    a.v[0] = 0;
    bool sticky = false;
    int64_t taken = 0;
    uint32_t chunk = 0, scale = 1;
    for (int32_t i = first; i < end; i++) {
        const uint32_t c = (uint32_t)s[i] - '0';
        if (c > 9) continue;   // the point
        if (taken == nk) {
            sticky |= c != 0;
            continue;
        }
        chunk = chunk * 10 + c;
        scale *= 10;
        taken++;
        if (scale == 1000000000u || taken == nk) {
            ft_big_muladd(a, scale, chunk);
            chunk = 0;
            scale = 1;
        }
    }
    int64_t ea = 0;
    if (qk > 0) {
        ft_big_mulpow5(a, qk);
        ea = qk;
    }
    // sign of (decimal - the point halfway between pattern p and p + 1)
    auto cmp_half = [&](uint64_t p) {
        const uint64_t ef = p >> f.mbits, fr = p & ((1ull << f.mbits) - 1);
        const uint64_t m = ef ? fr | (1ull << f.mbits) : fr;
        const int64_t e = (ef ? (int64_t)ef : 1) - f.bias - f.mbits;
        FtBig r;
        const uint64_t mm = 2 * m + 1;   // halfway = (2m + 1) * 2^(e - 1)
        r.v[0] = (uint32_t)mm;
        r.v[1] = (uint32_t)(mm >> 32);
        r.n = 2;
        int64_t er = e - 1;
        if (qk < 0) {   // decimal * 10^-qk vs halfway * 5^-qk * 2^-qk
            ft_big_mulpow5(r, -qk);
            er -= qk;
        }
        const int c = ft_big_cmp(a, ea, r, er);
        return c == 0 && sticky ? 1 : c;
    };
    if (b > f.inf) b = f.inf;
    for (;;) {
        if (b < f.inf) {
            const int c = cmp_half(b);
            if (c > 0 || (c == 0 && (b & 1))) {
                b++;
                continue;
            }
        }
        if (b > 0) {
            const int c = cmp_half(b - 1);
            if (c < 0 || (c == 0 && (b & 1))) {
                b--;
                continue;
            }
        }
        return b;
    }
}

__host__ __device__ __forceinline__ bool ft_is_digit(uint8_t c) { return c >= '0' && c <= '9'; }
__host__ __device__ __forceinline__ uint8_t ft_lower(uint8_t c) { return c >= 'A' && c <= 'Z' ? c + 32 : c; }
// s[0, n) equals the ASCII word w (case-insensitively when `fold`)
__host__ __device__ inline bool ft_word(const uint8_t* s, int32_t n, const char* w, bool fold) {
    int32_t k = 0;
    for (; w[k]; k++)
        if (k >= n || (fold ? ft_lower(s[k]) : s[k]) != (uint8_t)w[k]) return false;
    return k == n;
}

// CAST(text AS FLOAT / DOUBLE) of bits 32 / 64 into *out (the bit pattern); false: NULL.  `marked`: the text is read through an
// upper / lower-case mark, so it cannot hold the mixed-case NaN / Infinity of Java's grammar.
FT_NOINLINE __host__ __device__ inline bool ft_text_to_float(int bits, const uint8_t* s, int32_t len, bool marked, uint64_t* out) {
    const FtFormat f(bits);
    int32_t a = 0, e = len;
    while (a < e && s[a] <= ' ') a++;   // Java's String.trim
    while (e > a && s[e - 1] <= ' ') e--;
    if (a == e) return false;
    int32_t i = a;
    const bool neg = s[i] == '-';
    const uint64_t sign = neg ? 1ull << (bits - 1) : 0;
    if (s[i] == '+' || s[i] == '-') i++;
    if (!marked && ft_word(s + i, e - i, "NaN", false)) {
        *out = f.inf | (1ull << (f.mbits - 1));
        return true;
    }
    if (!marked && ft_word(s + i, e - i, "Infinity", false)) {
        *out = sign | f.inf;
        return true;
    }
    // digits [. digits] or . digits, at least one digit
    int64_t nd = 0, frac = 0;
    uint64_t w = 0;
    int32_t first = -1;
    bool any = false, dot = false;
    for (; i < e; i++) {
        const uint8_t c = s[i];
        if (ft_is_digit(c)) {
            any = true;
            if (dot) frac++;
            if (nd == 0 && c == '0') continue;
            if (nd == 0) first = i;
            if (nd < 19) w = w * 10 + (c - '0');
            nd++;
        } else if (c == '.' && !dot) dot = true;
        else break;
    }
    const int32_t mant_end = i;
    bool ok = any;
    int64_t ex = 0;
    if (ok && i < e && (s[i] == 'e' || s[i] == 'E')) {
        i++;
        bool eneg = false;
        if (i < e && (s[i] == '+' || s[i] == '-')) eneg = s[i++] == '-';
        ok = i < e && ft_is_digit(s[i]);
        for (; i < e && ft_is_digit(s[i]); i++)
            if (ex < 1000000000) ex = ex * 10 + (s[i] - '0');   // saturates: far beyond every finite and nonzero result
        if (eneg) ex = -ex;
    }
    if (ok && i < e && (ft_lower(s[i]) == 'f' || ft_lower(s[i]) == 'd')) i++;
    if (!ok || i != e) {   // Spark's special literals, lower-cased
        const uint8_t* t = s + a;
        const int32_t n = e - a;
        if (ft_word(t, n, "inf", true) || ft_word(t, n, "+inf", true) || ft_word(t, n, "infinity", true) || ft_word(t, n, "+infinity", true)) {
            *out = f.inf;
            return true;
        }
        if (ft_word(t, n, "-inf", true) || ft_word(t, n, "-infinity", true)) {
            *out = (1ull << (bits - 1)) | f.inf;
            return true;
        }
        if (ft_word(t, n, "nan", true)) {
            *out = f.inf | (1ull << (f.mbits - 1));
            return true;
        }
        return false;
    }
    const int64_t q = ex - frac;   // value = (the nd significant digits) * 10^q
    const int64_t dexp = nd + q;   // 10^(dexp - 1) <= value < 10^dexp
    uint64_t r;
    if (nd == 0 || dexp <= (bits == 64 ? -324 : -46)) r = 0;
    else if (dexp - 1 >= (bits == 64 ? 309 : 39)) r = f.inf;
    else if (nd <= 19) {
        r = ft_eisel_lemire(w, q, f, &ok);
        if (!ok) r = ft_parse_exact(s, first, mant_end, nd, q, f, r);
    } else {   // the value lies in [w, w + 1) * 10^(q + nd - 19)
        bool ok2;
        r = ft_eisel_lemire(w, q + nd - 19, f, &ok);
        const uint64_t r2 = ft_eisel_lemire(w + 1, q + nd - 19, f, &ok2);
        if (!ok || !ok2 || r != r2) r = ft_parse_exact(s, first, mant_end, nd, q, f, r);
    }
    *out = sign | r;
    return true;
}

// ------------------------------------------------------------------------------------------------ float -> text
// floor(g * cp / 2^128) with its lowest bit set when the fraction is nonzero (Schubfach's round to odd).  The +1 of g moves
// the product by less than cp / 2^128, which stays inside the dropped lowest word.
__host__ __device__ __forceinline__ uint64_t ft_rop(uint64_t gh, uint64_t gl, uint64_t cp) {
    uint64_t x1, x0, y1, y0;
    ft_mul64(gl, cp, &x1, &x0);
    ft_mul64(gh, cp, &y1, &y0);
    const uint64_t mid = y0 + x1;
    return (y1 + (mid < y0)) | (mid != 0 ? 1 : 0);
}

// digits of v > 0 at the end of buf (backwards); returns the count
__host__ __device__ __forceinline__ int ft_digits(uint64_t v, char* end) {
    int n = 0;
    do {
        *--end = (char)('0' + (int)(v % 10));
        v /= 10;
        n++;
    } while (v);
    return n;
}

// Java's layout of the decimal dec * 10^e (dec > 0)
__host__ __device__ inline int ft_layout(uint64_t dec, int e, char* p) {
    while (dec % 10 == 0) {
        dec /= 10;
        e++;
    }
    char tmp[20];
    const int n = ft_digits(dec, tmp + 20);
    const char* d = tmp + 20 - n;
    const int x = e + n - 1;   // exponent of the first digit
    int k = 0;
    if (x >= -3 && x < 7) {
        if (x >= 0) {
            for (int i = 0; i <= x; i++) p[k++] = i < n ? d[i] : '0';
            p[k++] = '.';
            if (n > x + 1)
                for (int i = x + 1; i < n; i++) p[k++] = d[i];
            else p[k++] = '0';
        } else {
            p[k++] = '0';
            p[k++] = '.';
            for (int i = 0; i < -x - 1; i++) p[k++] = '0';
            for (int i = 0; i < n; i++) p[k++] = d[i];
        }
        return k;
    }
    p[k++] = d[0];
    p[k++] = '.';
    if (n > 1)
        for (int i = 1; i < n; i++) p[k++] = d[i];
    else p[k++] = '0';
    p[k++] = 'E';
    int ax = x;
    if (x < 0) {
        p[k++] = '-';
        ax = -x;
    }
    char et[4];
    const int ne = ft_digits((uint64_t)ax, et + 4);
    for (int i = 0; i < ne; i++) p[k++] = et[4 - ne + i];
    return k;
}

// CAST(float AS STRING) of the bit pattern x of width bits (32 / 64) into out (>= 24 bytes); returns the length
FT_NOINLINE __host__ __device__ inline int ft_float_to_text(int bits, uint64_t x, char* out) {
    const FtFormat f(bits);
    const uint64_t emask = f.inf >> f.mbits;
    const uint64_t ef = (x >> f.mbits) & emask, fr = x & ((1ull << f.mbits) - 1);
    const bool neg = (x >> (bits - 1)) & 1;
    int k = 0;
    auto put = [&](const char* w) {
        for (int i = 0; w[i]; i++) out[k++] = w[i];
        return k;
    };
    if (ef == emask) return fr ? put("NaN") : put(neg ? "-Infinity" : "Infinity");
    if (neg) out[k++] = '-';
    if (ef == 0 && fr == 0) return put("0.0");
    uint64_t c;
    int q, dk = 0;
    if (ef) {
        c = fr | (1ull << f.mbits);
        q = (int)ef - f.bias - f.mbits;
    } else {
        c = fr;
        q = 1 - f.bias - f.mbits;
        if (c < (bits == 64 ? 3u : 8u)) {   // so few significant bits that two digits need a finer grid: 10c * 10^-1
            c *= 10;
            dk = -1;
        }
    }
    const bool irregular = fr == 0 && ef > 1;   // the predecessor is in the binade below: the gap below is half the gap above
    const uint64_t out_ = c & 1;                // an odd significand does not round to itself from its interval's ends
    const uint64_t cb = c << 2, cbr = cb + 2, cbl = irregular ? cb - 1 : cb - 2;
    const int kk = irregular ? (q * 315653 - 131237) >> 20 : (q * 315653) >> 20;   // floor(log10(3/4 2^q)) / floor(log10(2^q))
    const int h = q + ((-kk * 217706) >> 16) + 3;
    const uint64_t gh = FT_G(2 * (kk - FT_G_MIN)), gl = FT_G(2 * (kk - FT_G_MIN) + 1);
    // 4 * (v, its interval's ends) * 10^-kk, rounded to odd
    const uint64_t vb = ft_rop(gh, gl, cb << h), vbl = ft_rop(gh, gl, cbl << h), vbr = ft_rop(gh, gl, cbr << h);
    const uint64_t s = vb >> 2;
    uint64_t dec;
    if (s >= 100) {   // one digit fewer: the multiple of 10 at most one of which is inside the interval
        const uint64_t sp = s / 10 * 10;
        const bool upin = vbl + out_ <= sp << 2, wpin = ((sp + 10) << 2) + out_ <= vbr;
        if (upin != wpin) return k + ft_layout(upin ? sp : sp + 10, kk + dk, out + k);
    }
    const uint64_t t = s + 1;
    const bool uin = vbl + out_ <= s << 2, win = (t << 2) + out_ <= vbr;
    if (uin != win) dec = uin ? s : t;
    else {   // both inside: the closer, ties to even
        const int64_t cmp = (int64_t)(vb - ((s + t) << 1));
        dec = cmp < 0 || (cmp == 0 && !(s & 1)) ? s : t;
    }
    return k + ft_layout(dec, kk + dk, out + k);
}

}  // namespace auron
