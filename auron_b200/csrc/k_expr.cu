// k_expr.cu -- fused expression VM (rows F1-F3, E1-E5 of SURVEY.md section 8a).
//
// The reference evaluates a PhysicalExpr tree node by node, materialising one Arrow array per node
// (DataFusion BinaryExpr / CaseExpr / LikeExpr ..., datafusion-ext-exprs, datafusion-ext-functions) and
// ANDs predicate masks one conjunct at a time (datafusion-ext-plans/src/common/cached_exprs_evaluator.rs:
// 90-163,493-522).  On a GPU that is one full HBM round trip per node.  Here the whole expression list
// of a Filter / Project is compiled once per plan into a register-machine program and ONE kernel
// evaluates it per row: operands are loaded from the Arrow columns with coalesced accesses (thread i
// <-> row i), intermediates live in a shared-memory register file laid out [reg][thread] (conflict
// free), validity is a per-thread bit mask, and only final outputs are written (value + validity word
// via warp ballot).  Algorithmic bytes = referenced input columns once + outputs once.
//
// Semantics restated from the reference / its third-party kernels (SURVEY.md Appendix B):
//   * predicate NULL => row dropped (cached_exprs_evaluator.rs:514-519)
//   * integer + - * wrap (arrow *_wrapping); x / 0 and x % 0 => NULL (Spark_NullIfZero wraps divisors,
//     datafusion-ext-functions/src/spark_null_if.rs:69-110); Kleene AND/OR
//   * decimal + - * => NULL when the result leaves i128 or the declared precision of the node (Spark's non-ANSI arithmetic)
//   * comparisons of floats use IEEE totalOrder like arrow-ord cmp (NaN == NaN, -0 < +0)
//   * CAST per datafusion-ext-commons/src/arrow/cast.rs: float->int saturating with NaN->0 (:54-95),
//     utf8->int / utf8->date Spark parsers (:394-529), other numeric casts as arrow safe casts
//     (out of range => NULL), decimal rescale rounds half away from zero
//   * starts_with / ends_with / contains (datafusion-ext-exprs/src/string_*.rs:68-110), LIKE with % _ and
//     backslash escape, substr with 1-based character positions, date_part family on Date32
//     (datafusion-ext-functions/src/spark_dates.rs:255ff; dayofweek Sunday = 1 :280-294)
#include <cmath>

#include "device_utils.cuh"
#include "expr.h"
#include "float_text.cuh"
#include "kernels.h"
#include "tzdb.h"

namespace auron {

#define LAUNCH_CHECK(ctx)            \
    do {                             \
        CUDA_OK(cudaGetLastError()); \
        launch_count(ctx);           \
    } while (0)

constexpr int VM_NREG = 16;
constexpr int VM_THREADS = 256;
constexpr int VM_MAX_COLS = 32;
constexpr int VM_POOL_BUF = 255;

enum Vt : uint8_t { VT_BOOL = 0, VT_I8, VT_I16, VT_I32, VT_I64, VT_F32, VT_F64, VT_DEC, VT_STR };

enum Op : uint16_t {
    OP_LOAD = 0, OP_CONST,
    OP_ADD, OP_SUB, OP_MUL, OP_DIV, OP_MOD, OP_NEG, OP_ABS,
    OP_EQ, OP_NE, OP_LT, OP_LE, OP_GT, OP_GE, OP_NSEQ,
    OP_AND, OP_OR, OP_NOT, OP_ISNULL, OP_ISNOTNULL, OP_SELECT, OP_COALESCE, OP_CAST,
    OP_STARTS, OP_ENDS, OP_CONTAINS, OP_LIKE, OP_SUBSTR, OP_CHARLEN, OP_OCTLEN, OP_TRIM, OP_CASEXF,
    OP_DATEPART, OP_TS_LOCAL_MS, OP_TIMEPART, OP_MS_TO_DAYS, OP_ROUND, OP_NULLIFZERO, OP_ISNAN, OP_NORMNAN, OP_CHECK_OVERFLOW, OP_MAKE_DECIMAL, OP_UNSCALED,
    OP_MATH1, OP_POW, OP_HASH,
    OP_BITAND, OP_BITOR, OP_BITXOR, OP_SHL, OP_SHR,
    OP_GREATEST, OP_DATE_TRUNC, OP_MAKE_DATE, OP_FACTORIAL, OP_ROWNUM, OP_MONTHS_BETWEEN,
    OP_OUT, OP_OUT_PRED, OP_FMT_OUT,
    OP_SB_BEGIN, OP_SB_APPEND, OP_SB_END,
};
// OP_SB_APPEND: flags = piece kind | SB_WS (concat_ws) | SB_REPEAT | SbFn << 4 (a string function of the view in a, with its
// arguments in b and c); aux = output | constant << 8 (the separator with SB_WS, the count with SB_REPEAT); aux2 = FmtKind << 8 |
// scale of an SB_FMT piece
enum SbPiece : int { SB_VIEW = 0, SB_FMT = 1, SB_SPACE = 2, SB_WS = 4, SB_REPEAT = 8 };
enum CharlenFlags : int { CL_CHARS = 0, CL_ASCII = 1, CL_FIND_IN_SET = 2 };
constexpr int TRIM_SET = 4;   // OP_TRIM flag: trim the characters of the view in b instead of ASCII spaces
enum DatePart : int { DP_YEAR = 0, DP_MONTH, DP_DAY, DP_DOW, DP_QUARTER, DP_WEEK, DP_DOY };
enum Math1 : int { M_SQRT = 0, M_EXP, M_LN, M_LOG10, M_LOG2, M_SIN, M_COS, M_TAN, M_ASIN, M_ACOS, M_ATAN, M_CEIL, M_FLOOR, M_SIGNUM, M_TRUNC, M_EXPM1, M_ACOSH };
// date_trunc levels, finest first (Spark's TruncTimestamp format names)
enum TruncLevel : int { TL_MICROSECOND = 0, TL_MILLISECOND, TL_SECOND, TL_MINUTE, TL_HOUR, TL_DAY, TL_WEEK, TL_MONTH, TL_QUARTER, TL_YEAR };

struct Instr {
    uint16_t op;
    uint8_t dst, a, b, c, t, flags;
    int32_t aux, aux2;
};
struct ConstEntry {
    uint64_t lo;
    int64_t hi;
    int32_t valid;
    int32_t pad;
};
struct VmParams {
    const void* in_data[VM_MAX_COLS];
    const uint8_t* in_valid[VM_MAX_COLS];
    const int32_t* in_off[VM_MAX_COLS];
    void* out_data[VM_MAX_COLS];
    uint32_t* out_valid[VM_MAX_COLS];
    int64_t* out_lens[VM_MAX_COLS];
    const int32_t* out_off[VM_MAX_COLS];
    const Instr* prog;
    const ConstEntry* consts;
    const uint8_t* pool;
    const int32_t* sel;
    uint32_t* pred_out;
    int64_t n;
    int64_t row_base;   // OP_ROWNUM: rows the projection emitted before this launch
    int32_t n_instr;
    int32_t mode;   // 0 eval (fixed outputs + string lengths), 1 copy string bytes
};

// 10^k as 128-bit, k = 0..38
static __constant__ uint64_t c_pow10_lo[39];
static __constant__ int64_t c_pow10_hi[39];
static void init_pow10_tables() {
    static bool done = false;
    if (done) return;
    unsigned __int128 v = 1;
    uint64_t lo[39];
    int64_t hi[39];
    for (int k = 0; k < 39; k++) {
        lo[k] = (uint64_t)v;
        hi[k] = (int64_t)(uint64_t)(v >> 64);
        v *= 10;
    }
    CUDA_OK(cudaMemcpyToSymbol(c_pow10_lo, lo, sizeof(lo)));
    CUDA_OK(cudaMemcpyToSymbol(c_pow10_hi, hi, sizeof(hi)));
    done = true;
}

// ------------------------------------------------------------------------------------------ device helpers
__device__ __forceinline__ i128 pow10_128(int k) { return {c_pow10_lo[k], c_pow10_hi[k]}; }
// exact double powers of ten (10^0..10^22 are exactly representable)
__device__ __forceinline__ double pow10_f64(int k) {
    const double tbl[23] = {1e0, 1e1, 1e2, 1e3, 1e4, 1e5, 1e6, 1e7, 1e8, 1e9, 1e10, 1e11, 1e12, 1e13, 1e14, 1e15, 1e16, 1e17, 1e18, 1e19, 1e20, 1e21, 1e22};
    if (k >= 0 && k <= 22) return tbl[k];
    return pow(10.0, (double)k);
}
__device__ __forceinline__ i128 i128_abs(i128 a) { return i128_is_neg(a) ? i128_neg(a) : a; }
__device__ __forceinline__ bool u128_lt(i128 a, i128 b) {   // unsigned compare
    if ((uint64_t)a.hi != (uint64_t)b.hi) return (uint64_t)a.hi < (uint64_t)b.hi;
    return a.lo < b.lo;
}
// unsigned 128 / 128 (bitwise long division)
__device__ inline i128 u128_divmod(i128 n, i128 d, i128* rem) {
    if (d.hi == 0) {
        uint64_t r;
        i128 q = u128_divmod_u64(n, d.lo, &r);
        *rem = {r, 0};
        return q;
    }
    i128 q = {0, 0}, r = {0, 0};
    for (int i = 127; i >= 0; i--) {
        r.hi = (int64_t)(((uint64_t)r.hi << 1) | (r.lo >> 63));
        r.lo = (r.lo << 1) | (i >= 64 ? (((uint64_t)n.hi >> (i - 64)) & 1) : ((n.lo >> i) & 1));
        if (!u128_lt(r, d)) {
            r = i128_sub(r, d);
            if (i >= 64) q.hi |= (int64_t)(1ull << (i - 64));
            else q.lo |= 1ull << i;
        }
    }
    *rem = r;
    return q;
}
// a * m of two magnitudes (< 2^127) with overflow detection (result must stay < 2^127)
__device__ inline bool u128_mul_checked(i128 a, i128 m, i128* out) {
    // a = a1:a0, m = m1:m0 ; overflow unless a1*m1 == 0 and cross terms fit
    uint64_t a0 = a.lo, a1 = (uint64_t)a.hi, m0 = m.lo, m1 = (uint64_t)m.hi;
    if (a1 != 0 && m1 != 0) return false;
    uint64_t lo = a0 * m0, hi = __umul64hi(a0, m0);
    uint64_t c1 = a0 * m1, c1h = __umul64hi(a0, m1);
    uint64_t c2 = a1 * m0, c2h = __umul64hi(a1, m0);
    if (c1h || c2h) return false;
    uint64_t h2 = hi + c1;
    if (h2 < hi) return false;
    uint64_t h3 = h2 + c2;
    if (h3 < h2) return false;
    if (h3 >> 63) return false;
    *out = {lo, (int64_t)h3};
    return true;
}
// |a| * 10^k with overflow detection (result must stay < 2^127)
__device__ __forceinline__ bool u128_mul_pow10(i128 a, int k, i128* out) { return u128_mul_checked(a, pow10_128(k), out); }
__device__ __forceinline__ bool dec_fits_precision(i128 v, int prec) {
    if (prec >= 39) return true;
    return u128_lt(i128_abs(v), pow10_128(prec));
}
// decimal + - * of unscaled values: false when the exact result leaves i128 or `prec` digits (Spark's non-ANSI arithmetic
// gives NULL there; a wrapped i128 would be a plausible wrong number)
__device__ inline bool dec_arith(int op, i128 x, i128 y, int prec, i128* z) {
    if (op == OP_MUL) {
        const bool neg = i128_is_neg(x) != i128_is_neg(y);
        i128 m;
        if (!u128_mul_checked(i128_abs(x), i128_abs(y), &m)) return false;   // |x|, |y| < 10^38 < 2^127
        *z = neg ? i128_neg(m) : m;
    } else {
        if (op == OP_SUB) y = i128_neg(y);
        *z = i128_add(x, y);
        if (((x.hi ^ z->hi) & (y.hi ^ z->hi)) < 0) return false;   // both operands' sign differs from the sum's: wrapped
    }
    return dec_fits_precision(*z, prec);
}
// correctly rounded (one rounding): the top 64 significant bits with a sticky bit for everything below, then an exact scaling
__device__ __forceinline__ double i128_to_f64(i128 v) {
    bool neg = i128_is_neg(v);
    i128 a = neg ? i128_neg(v) : v;
    const uint64_t hi = (uint64_t)a.hi;
    double d;
    if (hi == 0) d = (double)a.lo;
    else {
        const int sh = 64 - __clzll((long long)hi);   // 1..64 bits of `hi` are significant
        const uint64_t top = sh == 64 ? hi : (hi << (64 - sh)) | (a.lo >> sh);
        const uint64_t below = sh == 64 ? a.lo : a.lo << (64 - sh);
        d = ldexp((double)(top | (below != 0)), sh);
    }
    return neg ? -d : d;
}
__device__ inline bool f64_to_i128(double x, i128* out) {
    if (!isfinite(x)) return false;
    bool neg = x < 0;
    double a = fabs(x);
    if (a >= 1.7014118346046923e38) return false;   // 2^127
    double hi_d = floor(a / 18446744073709551616.0);
    double lo_d = a - hi_d * 18446744073709551616.0;
    i128 r = {(uint64_t)lo_d, (int64_t)(uint64_t)hi_d};
    *out = neg ? i128_neg(r) : r;
    return true;
}
__device__ __forceinline__ int64_t sext(int64_t v, int t) {
    switch (t) {
        case VT_I8: return (int8_t)v;
        case VT_I16: return (int16_t)v;
        case VT_I32: return (int32_t)v;
        default: return v;
    }
}
__device__ __forceinline__ int64_t f64_total(double d) {
    int64_t b = __double_as_longlong(d);
    return b < 0 ? (b ^ 0x7fffffffffffffffll) : b;
}
__device__ __forceinline__ int32_t f32_total(float f) {
    int32_t b = __float_as_int(f);
    return b < 0 ? (b ^ 0x7fffffff) : b;
}
// Hinnant civil_from_days
__device__ inline void civil_from_days(int64_t z, int64_t* y, unsigned* m, unsigned* d) {
    z += 719468;
    int64_t era = (z >= 0 ? z : z - 146096) / 146097;
    unsigned doe = (unsigned)(z - era * 146097);
    unsigned yoe = (doe - doe / 1460 + doe / 36524 - doe / 146096) / 365;
    int64_t yy = (int64_t)yoe + era * 400;
    unsigned doy = doe - (365 * yoe + yoe / 4 - yoe / 100);
    unsigned mp = (5 * doy + 2) / 153;
    *d = doy - (153 * mp + 2) / 5 + 1;
    *m = mp < 10 ? mp + 3 : mp - 9;
    *y = yy + (*m <= 2);
}
__device__ inline int64_t days_from_civil_d(int64_t y, unsigned m, unsigned d) {
    y -= m <= 2;
    int64_t era = (y >= 0 ? y : y - 399) / 400;
    unsigned yoe = (unsigned)(y - era * 400);
    unsigned doy = (153 * (m + (m > 2 ? -3 : 9)) + 2) / 5 + d - 1;
    unsigned doe = yoe * 365 + yoe / 4 - yoe / 100 + doy;
    return era * 146097 + (int64_t)doe - 719468;
}
__device__ inline int32_t date_part(int64_t days, int part) {
    int64_t y;
    unsigned m, d;
    civil_from_days(days, &y, &m, &d);
    switch (part) {
        case DP_YEAR: return (int32_t)y;
        case DP_MONTH: return (int32_t)m;
        case DP_DAY: return (int32_t)d;
        case DP_QUARTER: return (int32_t)((m - 1) / 3 + 1);
        case DP_DOW: {   // spark_dates.rs:280-294: ((days + 4) mod 7) + 1, Sunday = 1
            int64_t r = (days + 4) % 7;
            if (r < 0) r += 7;
            return (int32_t)r + 1;
        }
        case DP_DOY: return (int32_t)(days - days_from_civil_d(y, 1, 1) + 1);
        case DP_WEEK: {   // ISO-8601 week of year
            int64_t wd = (days + 3) % 7;   // Monday = 0
            if (wd < 0) wd += 7;
            int64_t thursday = days - wd + 3;
            int64_t ty;
            unsigned tm, td;
            civil_from_days(thursday, &ty, &tm, &td);
            int64_t jan1 = days_from_civil_d(ty, 1, 1);
            return (int32_t)((thursday - jan1) / 7 + 1);
        }
    }
    return 0;
}

// spark_round.rs:193-212: HALF_UP at 10^digits (digits > 0 digits dropped; <= 0: unchanged)
__device__ inline __int128 round_half_up_i128(__int128 value, int digits) {
    if (digits <= 0) return value;
    if (digits > 38) return 0;
    __int128 factor = 1;
    for (int k = 0; k < digits; k++) factor *= 10;
    const __int128 rem = value % factor, base = value - rem;
    if (value >= 0) return rem * 2 >= factor ? base + factor : base;
    return (-rem) * 2 >= factor ? base - factor : base;
}
// spark_bround.rs:219-247: HALF_EVEN at 10^digits
__device__ inline __int128 round_half_even_i128(__int128 value, int digits) {
    if (digits <= 0) return value;
    if (digits > 38) return 0;
    __int128 factor = 1;
    for (int k = 0; k < digits; k++) factor *= 10;
    const __int128 rem = value % factor, base = value - rem, twice = (rem < 0 ? -rem : rem) * 2;
    if (twice > factor) return value >= 0 ? base + factor : base - factor;
    if (twice < factor) return base;
    if ((base / factor) % 2 == 0) return base;   // tie: the even multiple of `factor`
    return value >= 0 ? base + factor : base - factor;
}
// spark_bround.rs:177-217 (x finite)
__device__ inline double round_half_even_f64(double x) {
    const double ax = fabs(x), f = floor(ax), diff = ax - f;
    const double r = diff > 0.5 ? f + 1.0 : diff < 0.5 ? f : ((((long long)f) & 1) == 0 ? f : f + 1.0);
    return copysign(r, x);
}
__device__ inline float round_half_even_f32(float x) {
    const float ax = fabsf(x), f = floorf(ax), diff = ax - f;
    const float r = diff > 0.5f ? f + 1.0f : diff < 0.5f ? f : ((((long long)f) & 1) == 0 ? f : f + 1.0f);
    return copysignf(r, x);
}
// 10^n as llvm.powi computes it for the exponents that occur (exact for |n| <= 22; 1 / 10^|n| for negative n)
__device__ inline double powi10(int n) {
    double f = 1.0;
    for (int k = 0; k < (n < 0 ? -n : n); k++) f *= 10.0;
    return n < 0 ? 1.0 / f : f;
}
// E4 with a session time zone (spark_dates.rs:200-227,313-345): `v` in `unit` (0 s, 1 ms, 2 us, 3 ns, 4 = Date32 days) becomes
// Timestamp(Millisecond) the way arrow's cast does it (division truncates toward zero), then the zone's UTC offset at that
// instant is added.  The zone is a table in the constant pool: int64 n | int64 transition_second[n] | int32 offset[n + 1].
// the number of transitions of zone table `tz` at or before UTC second `sec`: the index of its offset
__device__ __forceinline__ int64_t tz_interval(const uint8_t* tz, int64_t sec) {
    const int64_t n = *(const int64_t*)tz;
    const int64_t* trans = (const int64_t*)tz + 1;
    int64_t lo = 0, hi = n;
    while (lo < hi) {
        const int64_t mid = (lo + hi) >> 1;
        if (trans[mid] <= sec) lo = mid + 1;
        else hi = mid;
    }
    return lo;
}
__device__ __forceinline__ int32_t tz_offset(const uint8_t* tz, int64_t k) { return ((const int32_t*)((const int64_t*)tz + 1 + *(const int64_t*)tz))[k]; }
__device__ __forceinline__ int64_t ts_to_utc_ms(int64_t v, int unit) {
    return unit == 0 ? v * 1000 : unit == 1 ? v : unit == 2 ? v / 1000 : unit == 3 ? v / 1000000 : v * 86400000ll;
}
__device__ __forceinline__ int64_t floor_div(int64_t a, int64_t b) { return a / b - (a % b != 0 && (a < 0) != (b < 0)); }
__device__ inline int64_t ts_to_local_ms(int64_t v, int unit, const uint8_t* tz) {
    int64_t ms = ts_to_utc_ms(v, unit);
    // chrono: Utc.timestamp_millis_opt(ms) -> the instant's second is floor(ms / 1000)
    if (tz) ms += (int64_t)tz_offset(tz, tz_interval(tz, floor_div(ms, 1000))) * 1000;
    return ms;
}
// Local to UTC on zone table `tz` (start_of_local_day_ms, spark_dates.rs:112-139): the earliest UTC second whose local time is
// `local_s`; when that local time falls into a gap, the earliest one of the first whole minute after it that exists (at most a day
// later).  false when there is none.  Interval k (offset o, UTC [trans[k - 1], trans[k])) holds the local times
// [trans[k - 1] + o, trans[k] + o), so its first minute is found without walking; offsets lie within +-26 h, so only the intervals
// that cover [local_s - 26 h, local_s + 50 h] can hold the answer.  Out of line: inlined, it makes vm_kernel<true> spill.
static __device__ __noinline__ bool local_to_utc_s(const uint8_t* tz, int64_t local_s, int64_t* out) {
    const int64_t n = *(const int64_t*)tz;
    const int64_t* trans = (const int64_t*)tz + 1;
    const int64_t k0 = tz_interval(tz, local_s - 93600), k1 = tz_interval(tz, local_s + 180000);
    int64_t best = 24 * 60 + 1;
    for (int64_t k = k0; k <= k1; k++) {   // ascending intervals: at an equal minute the first fit is the earliest instant
        const int64_t o = tz_offset(tz, k);
        const int64_t m = k > 0 && trans[k - 1] + o > local_s ? (trans[k - 1] + o - local_s + 59) / 60 : 0;
        if (m < best && (k == n || local_s + 60 * m < trans[k] + o)) {
            best = m;
            *out = local_s + 60 * m - o;
        }
    }
    return best <= 24 * 60;
}
__device__ __forceinline__ int days_in_month(int64_t y, unsigned m) {
    const bool leap = (y % 4 == 0 && y % 100 != 0) || y % 400 == 0;
    return m == 2 ? 28 + leap : (m == 4 || m == 6 || m == 9 || m == 11) ? 30 : 31;
}
// months_between_value (spark_dates.rs:158-198) of two UTC millisecond instants with the zone table `tz` (nullptr: UTC)
__device__ inline bool months_between(int64_t ms1, int64_t ms2, bool round_off, const uint8_t* tz, double* out) {
    const int64_t l1 = tz ? ts_to_local_ms(ms1, 1, tz) : ms1, l2 = tz ? ts_to_local_ms(ms2, 1, tz) : ms2;
    const int64_t day1 = floor_div(l1, 86400000), day2 = floor_div(l2, 86400000);
    int64_t y1, y2;
    unsigned m1, d1, m2, d2;
    civil_from_days(day1, &y1, &m1, &d1);
    civil_from_days(day2, &y2, &m2, &d2);
    const double month_diff = (double)((y1 * 12 + m1) - (y2 * 12 + m2));
    if (d1 == d2 || (d1 == (unsigned)days_in_month(y1, m1) && d2 == (unsigned)days_in_month(y2, m2))) {
        *out = month_diff;
        return true;
    }
    int64_t s1 = day1 * 86400, s2 = day2 * 86400;   // local midnights, then their UTC instants
    if (tz && !(local_to_utc_s(tz, s1, &s1) && local_to_utc_s(tz, s2, &s2))) return false;
    const int64_t secs = ((int64_t)d1 - (int64_t)d2) * 86400 + (ms1 - s1 * 1000) / 1000 - (ms2 - s2 * 1000) / 1000;
    const double r = month_diff + (double)secs / 2678400.0;
    *out = round_off ? floor(__dadd_rn(__dmul_rn(r, 1e8), 0.5)) / 1e8 : r;   // two roundings, as Rust does it: no fused multiply-add
    return true;
}
// date_trunc(level, v) of a timestamp in `unit` (0 s .. 3 ns) toward -inf, converted to `out_unit` as arrow's cast does (a coarser
// unit divides toward zero); false when the result leaves int64
__device__ inline bool date_trunc(int64_t v, int unit, int level, int out_unit, int64_t* out) {
    const int64_t unit_ns = unit == 0 ? 1000000000 : unit == 1 ? 1000000 : unit == 2 ? 1000 : 1;
    const int64_t day = 86400000000000ll / unit_ns;   // units per day
    int64_t r;
    if (level <= TL_DAY) {
        const int64_t step_ns[6] = {1000, 1000000, 1000000000, 60000000000ll, 3600000000000ll, 86400000000000ll};
        const int64_t step = step_ns[level] > unit_ns ? step_ns[level] / unit_ns : 1;
        int64_t m = v % step;
        if (m < 0) m += step;
        if ((uint64_t)v - (uint64_t)INT64_MIN < (uint64_t)m) return false;
        r = v - m;
    } else {
        int64_t d = floor_div(v, day), y;
        unsigned mo, dd;
        civil_from_days(d, &y, &mo, &dd);
        if (level == TL_WEEK) {   // Monday: day 0 (1970-01-01) is a Thursday
            int64_t wd = (d + 3) % 7;
            d -= wd < 0 ? wd + 7 : wd;
        } else d = days_from_civil_d(y, level == TL_YEAR ? 1 : level == TL_QUARTER ? (mo - 1) / 3 * 3 + 1 : mo, 1);
        const __int128 w = (__int128)d * day;
        if (w < INT64_MIN) return false;
        r = (int64_t)w;
    }
    if (out_unit > unit) {
        int64_t f = 1;
        for (int k = unit; k < out_unit; k++) f *= 1000;
        const __int128 w = (__int128)r * f;
        if (w < INT64_MIN || w > INT64_MAX) return false;
        r = (int64_t)w;
    } else
        for (int k = out_unit; k < unit; k++) r /= 1000;
    *out = r;
    return true;
}
// make_date(y, m, d): the day number of a valid proleptic Gregorian date that fits int32 (Spark's non-ANSI MakeDate gives NULL otherwise)
__device__ inline bool make_date(int64_t y, int64_t m, int64_t d, int64_t* out) {
    if (m < 1 || m > 12 || d < 1 || d > days_in_month(y, (unsigned)m)) return false;
    const int64_t z = days_from_civil_d(y, (unsigned)m, (unsigned)d);
    if (z < INT32_MIN || z > INT32_MAX) return false;
    *out = z;
    return true;
}

__device__ __forceinline__ const uint8_t* str_ptr(const VmParams& p, int64_t bufid, uint64_t view) {
    const uint8_t* base = (bufid & 0xff) == VM_POOL_BUF ? p.pool : (const uint8_t*)p.in_data[bufid & 0xff];
    return base + (uint32_t)(view >> 32);
}
__device__ __forceinline__ int32_t str_len(uint64_t view) { return (int32_t)(uint32_t)view; }
__device__ __forceinline__ int utf8_char_len(uint8_t b) { return b < 0x80 ? 1 : (b >> 5) == 6 ? 2 : (b >> 4) == 14 ? 3 : (b >> 3) == 30 ? 4 : 1; }
__device__ __forceinline__ uint8_t ascii_lower(uint8_t c) { return (c >= 'A' && c <= 'Z') ? c + 32 : c; }

__device__ inline int str_cmp(const uint8_t* a, int32_t la, const uint8_t* b, int32_t lb) {
    int32_t n = la < lb ? la : lb;
    for (int32_t i = 0; i < n; i++)
        if (a[i] != b[i]) return a[i] < b[i] ? -1 : 1;
    return la == lb ? 0 : (la < lb ? -1 : 1);
}
__device__ inline bool str_contains(const uint8_t* s, int32_t ls, const uint8_t* pat, int32_t lp) {
    if (lp == 0) return true;
    for (int32_t i = 0; i + lp <= ls; i++) {
        int32_t j = 0;
        while (j < lp && s[i + j] == pat[j]) j++;
        if (j == lp) return true;
    }
    return false;
}
// SQL LIKE: % any run, _ one character, backslash escapes the next pattern char
__device__ inline bool str_like(const uint8_t* s, int32_t ls, const uint8_t* p, int32_t lp, bool ci) {
    int32_t si = 0, pi = 0, star_p = -1, star_s = 0;
    while (si < ls) {
        bool advanced = false;
        if (pi < lp) {
            uint8_t pc = p[pi];
            if (pc == '%') {
                star_p = pi++;
                star_s = si;
                continue;
            }
            if (pc == '_') {
                si += utf8_char_len(s[si]);
                pi++;
                advanced = true;
            } else {
                int32_t pj = pi;
                if (pc == '\\' && pi + 1 < lp) {
                    pj = pi + 1;
                    pc = p[pj];
                }
                uint8_t sc = s[si];
                if (ci ? ascii_lower(sc) == ascii_lower(pc) : sc == pc) {
                    si++;
                    pi = pj + 1;
                    advanced = true;
                }
            }
        }
        if (!advanced) {
            if (star_p < 0) return false;
            star_s += utf8_char_len(s[star_s]);
            si = star_s;
            pi = star_p + 1;
        }
    }
    if (si > ls) return false;
    while (pi < lp && p[pi] == '%') pi++;
    return pi == lp;
}
// Spark to_integer (cast.rs:394-468)
// utf8 -> decimal128(prec, scale): cast.rs:223-225 (scientific notation is rewritten to a plain decimal string first,
// cast.rs:328-351) followed by arrow's string -> decimal parser: [+-] digits [. digits] [e[+-]digits]; fraction digits beyond the
// scale are dropped (no rounding), no surrounding whitespace, anything else or more than `prec` digits -> NULL.
// Golden vectors: cast.rs:629-658.
__device__ inline bool str_to_decimal(const uint8_t* s, int32_t len, int prec, int scale, i128* out) {
    int32_t i = 0;
    bool neg = false;
    if (len > 0 && (s[0] == '-' || s[0] == '+')) {
        neg = s[0] == '-';
        i = 1;
    }
    if (i >= len) return false;
    // pass 1: structure
    int32_t dig0 = i, ni = 0, nf = 0, dot = -1, epos = -1;
    for (; i < len; i++) {
        const uint8_t c = s[i];
        if (c >= '0' && c <= '9') {
            if (dot < 0) ni++;
            else nf++;
        } else if (c == '.' && dot < 0) dot = i;
        else if (c == 'e' || c == 'E') {
            epos = i;
            break;
        } else return false;
    }
    if (ni + nf == 0) return false;
    int64_t E = 0;
    if (epos >= 0) {
        int32_t j = epos + 1;
        bool eneg = false;
        if (j < len && (s[j] == '-' || s[j] == '+')) {
            eneg = s[j] == '-';
            j++;
        }
        if (j >= len) return false;
        for (; j < len; j++) {
            if (s[j] < '0' || s[j] > '9') return false;
            E = E * 10 + (s[j] - '0');
            if (E > 100000) return false;
        }
        if (eneg) E = -E;
    }
    // value = D x 10^(E - nf), D = all mantissa digits; unscaled result = trunc(D x 10^shift)
    const int64_t shift = E - nf + scale;
    int64_t keep = (int64_t)ni + nf + (shift < 0 ? shift : 0);   // mantissa digits that survive the truncation
    const int32_t dend = epos >= 0 ? epos : len;
    i128 acc = {0, 0};
    int sig = 0;   // digits accumulated after the first non-zero one
    for (int32_t j = dig0; j < dend && keep > 0; j++) {
        const uint8_t c = s[j];
        if (c == '.') continue;
        keep--;
        if (sig == 0 && c == '0') continue;
        if (++sig > 38) return false;
        if (!u128_mul_pow10(acc, 1, &acc)) return false;
        acc = i128_add(acc, {(uint64_t)(c - '0'), 0});
    }
    if (shift > 0 && sig > 0) {
        if (shift + sig > 38) return false;
        if (!u128_mul_pow10(acc, (int)shift, &acc)) return false;
    }
    if (!dec_fits_precision(acc, prec)) return false;
    *out = neg ? i128_neg(acc) : acc;
    return true;
}
__device__ inline bool str_to_int(const uint8_t* s, int32_t len, int t, int64_t* out) {
    if (len == 0) return false;
    int bits = t == VT_I8 ? 8 : t == VT_I16 ? 16 : t == VT_I32 ? 32 : 64;
    int64_t minv = bits == 64 ? INT64_MIN : -((int64_t)1 << (bits - 1));
    bool negative = s[0] == '-';
    int32_t off = 0;
    if (negative || s[0] == '+') {
        off = 1;
        if (len == 1) return false;
    }
    int64_t stop = minv / 10, result = 0;
    while (off < len) {
        uint8_t b = s[off++];
        if (b == '.') break;
        if (b < '0' || b > '9') return false;
        if (result < stop) return false;
        result = sext((int64_t)((uint64_t)result * 10ull - (uint64_t)(b - '0')), t);
        if (result > 0) return false;
    }
    while (off < len) {
        if (s[off] < '0' || s[off] > '9') return false;
        off++;
    }
    if (!negative) {
        if (result == minv) return false;
        result = -result;
        if (result < 0) return false;
    }
    *out = result;
    return true;
}
// Spark to_date (cast.rs:471-529)
__device__ inline bool str_to_date(const uint8_t* s0, int32_t len0, int32_t* out) {
    int32_t a = 0, e = len0;
    while (a < e && (s0[a] == ' ' || (s0[a] >= 9 && s0[a] <= 13))) a++;
    while (e > a && (s0[e - 1] == ' ' || (s0[e - 1] >= 9 && s0[e - 1] <= 13))) e--;
    const uint8_t* s = s0 + a;
    int32_t len = e - a;
    if (len == 0) return false;
    int seg[3] = {1, 1, 1};
    int sign = 1, i = 0, cur = 0, digits = 0;
    int32_t j = 0;
    if (s[j] == '-' || s[j] == '+') {
        sign = s[j] == '-' ? -1 : 1;
        j++;
    }
    auto valid_digits = [](int sg, int dg) { return (sg == 0 && dg >= 4 && dg <= 7) || (sg != 0 && dg > 0 && dg <= 2); };
    while (j < len && (i < 3 && !(s[j] == ' ' || s[j] == 'T'))) {
        uint8_t b = s[j];
        if (i < 2 && b == '-') {
            if (!valid_digits(i, digits)) return false;
            seg[i] = cur;
            cur = 0;
            digits = 0;
            i++;
        } else {
            int pv = (int)b - '0';
            if (pv < 0 || pv > 9) return false;
            cur = cur * 10 + pv;
            digits++;
        }
        j++;
    }
    if (!valid_digits(i, digits)) return false;
    if (i < 2 && j < len) return false;
    seg[i] = cur;
    if (seg[0] > 9999 || seg[1] > 12 || seg[2] > 31) return false;
    int64_t y = (int64_t)sign * seg[0];
    int m = seg[1], d = seg[2];
    if (m < 1 || d < 1) return false;
    const int mdays[12] = {31, 28, 31, 30, 31, 30, 31, 31, 30, 31, 30, 31};
    bool leap = (y % 4 == 0 && y % 100 != 0) || y % 400 == 0;
    if (d > mdays[m - 1] + ((m == 2 && leap) ? 1 : 0)) return false;
    *out = (int32_t)days_from_civil_d(y, (unsigned)m, (unsigned)d);
    return true;
}

// cast; returns validity of the result (input known valid)
__device__ inline bool vm_cast(const VmParams& p, int st, int dt, int sscale, int dprec, int dscale, uint64_t& lo, int64_t& hi) {
    if (st <= VT_I64) {   // bool / ints
        int64_t v = (int64_t)lo;
        switch (dt) {
            case VT_BOOL: lo = v != 0; return true;
            case VT_I8: if (v < -128 || v > 127) return false; return true;
            case VT_I16: if (v < -32768 || v > 32767) return false; return true;
            case VT_I32: if (v < INT32_MIN || v > INT32_MAX) return false; return true;
            case VT_I64: return true;
            case VT_F32: lo = (uint32_t)__float_as_int((float)v); return true;
            case VT_F64: lo = (uint64_t)__double_as_longlong((double)v); return true;
            case VT_DEC: {
                i128 a = i128_from_i64(v);
                bool neg = v < 0;
                i128 r;
                if (!u128_mul_pow10(i128_abs(a), dscale, &r)) return false;
                if (neg) r = i128_neg(r);
                if (!dec_fits_precision(r, dprec)) return false;
                lo = r.lo; hi = r.hi;
                return true;
            }
        }
        return false;
    }
    if (st == VT_F32 || st == VT_F64) {
        double x = st == VT_F32 ? (double)__int_as_float((int)(uint32_t)lo) : __longlong_as_double((int64_t)lo);
        switch (dt) {
            case VT_F32: lo = (uint32_t)__float_as_int((float)x); return true;
            case VT_F64: lo = (uint64_t)__double_as_longlong(x); return true;
            case VT_BOOL: lo = x != 0.0; return true;
            case VT_I8: case VT_I16: case VT_I32: case VT_I64: {   // Rust `as`: saturating, NaN -> 0 (cast.rs:54-95)
                int bits = dt == VT_I8 ? 8 : dt == VT_I16 ? 16 : dt == VT_I32 ? 32 : 64;
                int64_t r;
                if (isnan(x)) r = 0;
                else if (bits == 64) r = x <= -9223372036854775808.0 ? INT64_MIN : (x >= 9223372036854775808.0 ? INT64_MAX : (int64_t)x);
                else {
                    double lim = (double)((int64_t)1 << (bits - 1));
                    r = x <= -lim ? -((int64_t)1 << (bits - 1)) : (x >= lim ? ((int64_t)1 << (bits - 1)) - 1 : (int64_t)x);
                }
                lo = (uint64_t)r;
                return true;
            }
            case VT_DEC: {
                double scaled = round(x * pow10_f64(dscale));
                i128 r;
                if (!f64_to_i128(scaled, &r)) return false;
                if (!dec_fits_precision(r, dprec)) return false;
                lo = r.lo; hi = r.hi;
                return true;
            }
        }
        return false;
    }
    if (st == VT_DEC) {
        i128 v = {lo, hi};
        switch (dt) {
            case VT_DEC: {
                i128 r;
                if (dscale >= sscale) {
                    bool neg = i128_is_neg(v);
                    if (!u128_mul_pow10(i128_abs(v), dscale - sscale, &r)) return false;
                    if (neg) r = i128_neg(r);
                } else {
                    bool neg = i128_is_neg(v);
                    i128 d = pow10_128(sscale - dscale), rem;
                    i128 q = u128_divmod(i128_abs(v), d, &rem);
                    // round half away from zero: rem * 2 >= d
                    i128 twice = i128_add(rem, rem);
                    if (!u128_lt(twice, d)) q = i128_add(q, {1, 0});
                    r = neg ? i128_neg(q) : q;
                }
                if (!dec_fits_precision(r, dprec)) return false;
                lo = r.lo; hi = r.hi;
                return true;
            }
            case VT_I8: case VT_I16: case VT_I32: case VT_I64: {
                bool neg = i128_is_neg(v);
                i128 rem, q = u128_divmod(i128_abs(v), pow10_128(sscale), &rem);
                if (q.hi != 0 || (q.lo >> 63)) {
                    if (!(neg && q.hi == 0 && q.lo == (1ull << 63))) return false;
                }
                int64_t r = neg ? (int64_t)(~q.lo + 1) : (int64_t)q.lo;
                if (dt == VT_I8 && (r < -128 || r > 127)) return false;
                if (dt == VT_I16 && (r < -32768 || r > 32767)) return false;
                if (dt == VT_I32 && (r < INT32_MIN || r > INT32_MAX)) return false;
                lo = (uint64_t)r;
                return true;
            }
            case VT_F32: case VT_F64: {
                double x = i128_to_f64(v) / pow10_f64(sscale);
                if (dt == VT_F32) lo = (uint32_t)__float_as_int((float)x);
                else lo = (uint64_t)__double_as_longlong(x);
                return true;
            }
        }
        return false;
    }
    if (st == VT_STR) {
        const uint8_t* s = str_ptr(p, hi, lo);
        int32_t len = str_len(lo);
        if (dt >= VT_I8 && dt <= VT_I64) {
            int64_t r;
            bool is_date = dprec == -1;
            if (is_date) {
                int32_t d;
                if (!str_to_date(s, len, &d)) return false;
                lo = (uint64_t)(int64_t)d;
                return true;
            }
            if (!str_to_int(s, len, dt, &r)) return false;
            lo = (uint64_t)r;
            return true;
        }
        if (dt == VT_DEC) {
            i128 r;
            if (!str_to_decimal(s, len, dprec, dscale, &r)) return false;
            lo = r.lo;
            hi = r.hi;
            return true;
        }
        return false;
    }
    return false;
}

// ------------------------------------------------------------------------------------------ the VM kernel
// ---- CAST(x AS STRING) of a projection output (TryCastExpr -> arrow cast; bool: cast.rs:104-112, decimal: cast.rs:660-690):
// format `kind` value into buf (>= 42 bytes), returns the length.  kind: 0 bool, 1 integer, 2 date32, 3 decimal (scale), 4 float32,
// 5 float64 (Java's Float / Double.toString, float_text.cuh).  Floats and decimal(p > 18) run in vm_kernel<true, true> only (the
// compiler sets need_text for them).
enum FmtKind : int { FMT_BOOL = 0, FMT_INT = 1, FMT_DATE = 2, FMT_DEC = 3, FMT_F32 = 4, FMT_F64 = 5 };
__device__ inline int fmt_u64(uint64_t v, char* end) {   // writes digits backwards, returns count
    int n = 0;
    do {
        *--end = (char)('0' + (int)(v % 10));
        v /= 10;
        n++;
    } while (v);
    return n;
}
// the unscaled i128 {lo, hi} at `scale`: a '-', the integer part (at least "0"), '.', `scale` fractional digits (cast.rs:660-690)
__device__ __forceinline__ int fmt_decimal(uint64_t lo, int64_t hi, int scale, char* buf) {
    char tmp[40];
    char* end = tmp + 40;
    const bool neg = hi < 0;
    const i128 mag = i128_abs({lo, hi});
    uint64_t low;
    const i128 top = u128_divmod_u64(mag, 10000000000000000000ull, &low);   // |v| <= 2^127: top < 2^64
    int n = fmt_u64(low, end);
    if (top.lo) {
        while (n < 19) *(end - ++n) = '0';
        n += fmt_u64(top.lo, end - n);
    }
    const char* digits = end - n;
    int k = 0;
    if (neg) buf[k++] = '-';
    if (scale <= 0) {
        for (int i = 0; i < n; i++) buf[k++] = digits[i];
    } else if (n > scale) {
        for (int i = 0; i < n - scale; i++) buf[k++] = digits[i];
        buf[k++] = '.';
        for (int i = n - scale; i < n; i++) buf[k++] = digits[i];
    } else {
        buf[k++] = '0';
        buf[k++] = '.';
        for (int i = n; i < scale; i++) buf[k++] = '0';
        for (int i = 0; i < n; i++) buf[k++] = digits[i];
    }
    return k;
}
template <bool TEXT>
__device__ inline int fmt_value(int kind, int scale, uint64_t lo, int64_t hi, char* buf) {
    if (TEXT && kind == FMT_DEC) return fmt_decimal(lo, hi, scale, buf);
    if (TEXT && kind >= FMT_F32) return ft_float_to_text(kind == FMT_F32 ? 32 : 64, lo, buf);
    // bool, integers, dates and decimal(p <= 18): the unscaled value fits lo
    char tmp[24];
    char* end = tmp + 24;
    int n = 0;
    if (kind == FMT_BOOL) {
        const char* t = lo ? "true" : "false";
        n = lo ? 4 : 5;
        for (int i = 0; i < n; i++) buf[i] = t[i];
        return n;
    }
    if (kind == FMT_DATE) {
        int64_t y;
        unsigned m, d;
        civil_from_days((int64_t)(int32_t)lo, &y, &m, &d);
        int k = 0;
        if (y < 0) {
            buf[k++] = '-';
            y = -y;
        } else if (y > 9999) buf[k++] = '+';   // chrono: years outside 0..9999 as {:+05}
        int yd = fmt_u64((uint64_t)y, end);
        for (int i = yd; i < 4; i++) buf[k++] = '0';
        for (int i = 0; i < yd; i++) buf[k++] = (end - yd)[i];
        buf[k++] = '-';
        buf[k++] = (char)('0' + m / 10);
        buf[k++] = (char)('0' + m % 10);
        buf[k++] = '-';
        buf[k++] = (char)('0' + d / 10);
        buf[k++] = (char)('0' + d % 10);
        return k;
    }
    const int64_t sv = (int64_t)lo;
    const bool neg = sv < 0;
    const uint64_t mag = neg ? (uint64_t)0 - (uint64_t)sv : (uint64_t)sv;
    n = fmt_u64(mag, end);
    const char* digits = end - n;
    int k = 0;
    if (neg) buf[k++] = '-';
    if (kind == FMT_INT || scale <= 0) {
        for (int i = 0; i < n; i++) buf[k++] = digits[i];
        return k;
    }
    // decimal: integer part (at least "0"), '.', `scale` fractional digits
    if (n > scale) {
        for (int i = 0; i < n - scale; i++) buf[k++] = digits[i];
        buf[k++] = '.';
        for (int i = n - scale; i < n; i++) buf[k++] = digits[i];
    } else {
        buf[k++] = '0';
        buf[k++] = '.';
        for (int i = n; i < scale; i++) buf[k++] = '0';
        for (int i = 0; i < n; i++) buf[k++] = digits[i];
    }
    return k;
}

// copy a string view into an output, applying the ASCII upper (xf 1) / lower (xf 2) mark of OP_CASEXF
__device__ __forceinline__ void copy_view(uint8_t* d, const uint8_t* s, int32_t len, int xf) {
    for (int32_t k = 0; k < len; k++) {
        uint8_t c = s[k];
        if (xf == 1 && c >= 'a' && c <= 'z') c -= 32;
        else if (xf == 2 && c >= 'A' && c <= 'Z') c += 32;
        d[k] = c;
    }
}

// ------------------------------------------------------------------------------------------ string functions
// A character is a lead byte and the continuation bytes it announces, cut at the end of the view (as OP_SUBSTR counts them).
// Every byte is read through the view's ASCII upper / lower mark, so that matching sees the bytes copying writes.
struct SView {
    const uint8_t* p;
    int32_t n;
    int xf;
    __device__ __forceinline__ uint8_t at(int32_t k) const {
        uint8_t c = p[k];
        if (xf == 1 && c >= 'a' && c <= 'z') c -= 32;
        else if (xf == 2 && c >= 'A' && c <= 'Z') c += 32;
        return c;
    }
    __device__ __forceinline__ int32_t clen(int32_t k) const {   // bytes of the character that starts at k
        const int32_t l = utf8_char_len(p[k]);
        return l < n - k ? l : n - k;
    }
};
__device__ __forceinline__ SView sview(const VmParams& p, int64_t h, uint64_t x) { return {str_ptr(p, h, x), str_len(x), (int)((h >> 8) & 0xff)}; }
// CAST(utf8 AS BOOLEAN), Spark's StringUtils.isTrueString / isFalseString: ASCII whitespace and control characters trimmed at
// both ends, ASCII case ignored; t true y yes 1 -> true, f false n no 0 -> false, anything else NULL
__device__ inline bool str_to_bool(const SView& s, uint64_t* out) {
    int32_t a = 0, e = s.n;
    while (a < e && (s.p[a] <= ' ' || s.p[a] == 0x7f)) a++;
    while (e > a && (s.p[e - 1] <= ' ' || s.p[e - 1] == 0x7f)) e--;
    const uint8_t* t = s.p + a;
    const int32_t n = e - a;
    if (ft_word(t, n, "t", true) || ft_word(t, n, "true", true) || ft_word(t, n, "y", true) || ft_word(t, n, "yes", true) || ft_word(t, n, "1", true))
        *out = 1;
    else if (ft_word(t, n, "f", true) || ft_word(t, n, "false", true) || ft_word(t, n, "n", true) || ft_word(t, n, "no", true) || ft_word(t, n, "0", true))
        *out = 0;
    else return false;
    return true;
}
// CAST(utf8 AS FLOAT / DOUBLE / BOOLEAN) of the view {lo, hi}; returns the validity, the value in lo
static __device__ __noinline__ bool str_to_float_or_bool(const VmParams& p, int dt, uint64_t& lo, int64_t& hi) {
    const SView s = sview(p, hi, lo);
    hi = 0;
    if (dt == VT_BOOL) return str_to_bool(s, &lo);
    return ft_text_to_float(dt == VT_F32 ? 32 : 64, s.p, s.n, s.xf != 0, &lo);
}
// unsigned byte order, the shorter prefix first
__device__ inline int sv_cmp(const SView& a, const SView& b) {
    if (a.xf == 0 && b.xf == 0) return str_cmp(a.p, a.n, b.p, b.n);
    const int32_t n = a.n < b.n ? a.n : b.n;
    for (int32_t k = 0; k < n; k++) {
        const uint8_t x = a.at(k), y = b.at(k);
        if (x != y) return x < y ? -1 : 1;
    }
    return a.n == b.n ? 0 : (a.n < b.n ? -1 : 1);
}
__device__ __forceinline__ bool sv_eq(const SView& a, int32_t i, const SView& b, int32_t j, int32_t len) {
    for (int32_t k = 0; k < len; k++)
        if (a.at(i + k) != b.at(j + k)) return false;
    return true;
}
// the index (in characters) of the first character of `set` equal to a[i, i + len), -1 when there is none
__device__ inline int32_t sv_char_index(const SView& set, const SView& a, int32_t i, int32_t len) {
    int32_t k = 0;
    for (int32_t j = 0; j < set.n; k++) {
        const int32_t cl = set.clen(j);
        if (cl == len && sv_eq(set, j, a, i, len)) return k;
        j += cl;
    }
    return -1;
}
// trim with a character set (DataFusion btrim / ltrim / rtrim with a second argument): sides 1 = leading, 2 = trailing
__device__ inline void trim_set(const SView& s, const SView& set, int sides, int32_t* b, int32_t* e) {
    if (sides & 1)
        while (*b < *e) {
            const int32_t cl = s.clen(*b);
            if (sv_char_index(set, s, *b, cl) < 0) break;
            *b += cl;
        }
    if (sides & 2)
        while (*e > *b) {
            int32_t j = *e - 1;
            while (j > *b && (s.p[j] & 0xc0) == 0x80) j--;
            if (sv_char_index(set, s, j, *e - j) < 0) break;
            *e = j;
        }
}
// ascii(s): the code point of the first character, 0 for ""
__device__ inline int32_t str_ascii(const SView& s) {
    if (s.n == 0) return 0;
    const int32_t cl = s.clen(0);
    int32_t r = s.at(0);
    if (cl > 1) {
        r &= 0x7f >> cl;
        for (int32_t k = 1; k < cl; k++) r = (r << 6) | (s.p[k] & 0x3f);
    }
    return r;
}
// find_in_set(a, list) (Spark UTF8String.findInSet): the 1-based index of `a` among the comma-separated pieces of `list`; 0 when
// `a` holds a comma or is not there
__device__ inline int32_t str_find_in_set(const SView& a, const SView& list) {
    for (int32_t k = 0; k < a.n; k++)
        if (a.at(k) == ',') return 0;
    int32_t idx = 1, start = 0;
    for (int32_t j = 0; j <= list.n; j++) {
        if (j < list.n && list.at(j) != ',') continue;
        if (j - start == a.n && sv_eq(list, start, a, 0, a.n)) return idx;
        idx++;
        start = j + 1;
    }
    return 0;
}

// A builder row's length saturates here, so that no row wraps the int64 scan of the lengths; such a row fails its batch's 2 GiB check.
constexpr int64_t SB_SAT = (int64_t)INT32_MAX + 1;
// the string functions the builder runs as pieces (OP_SB_APPEND flags >> 4); the first four take three arguments; SBF_HEX_INT and
// SBF_CHR take an int64 instead of a view
enum SbFn : int { SBF_NONE = 0, SBF_LPAD, SBF_RPAD, SBF_REPLACE, SBF_TRANSLATE, SBF_REVERSE, SBF_INITCAP, SBF_HEX, SBF_HEX_INT, SBF_CHR };

// One string-function piece of s: lpad / rpad to n characters with pad x, replace search x by y, translate characters of x into
// those of y, reverse, initcap, hex of s or of n, chr of n.  Returns its byte length (above SB_SAT only when the row is too long
// anyway); with d (pass 1) it also writes the piece there.
__device__ inline int64_t sb_fn_piece(int fn, const SView& s, const SView& x, const SView& y, int64_t n, uint8_t* d) {
    const char* hex_digits = "0123456789ABCDEF";
    switch (fn) {
        case SBF_HEX:   // Spark Hex of utf8 / binary: two upper-case digits per byte
            if (d)
                for (int32_t k = 0; k < s.n; k++) {
                    const uint8_t c = s.at(k);
                    d[2 * k] = hex_digits[c >> 4];
                    d[2 * k + 1] = hex_digits[c & 15];
                }
            return 2 * (int64_t)s.n;
        case SBF_HEX_INT: {   // Spark Hex of a long: the two's complement value in upper-case digits without leading zeros
            const uint64_t u = (uint64_t)n;
            const int len = u == 0 ? 1 : (67 - __clzll((long long)u)) / 4;
            if (d)
                for (int k = 0; k < len; k++) d[len - 1 - k] = hex_digits[(u >> (4 * k)) & 15];
            return len;
        }
        case SBF_CHR: {   // Spark Chr: "" below 0, else code point n & 0xFF in UTF-8
            if (n < 0) return 0;
            const uint8_t c = (uint8_t)(n & 0xff);
            if (c < 0x80) {
                if (d) d[0] = c;
                return 1;
            }
            if (d) {
                d[0] = (uint8_t)(0xc0 | (c >> 6));
                d[1] = (uint8_t)(0x80 | (c & 0x3f));
            }
            return 2;
        }
        case SBF_LPAD: case SBF_RPAD: {   // Spark UTF8String.lpad / rpad
            if (n <= 0) return 0;
            int32_t sb = 0;   // bytes of s's first n characters
            int64_t ch = 0;
            while (sb < s.n && ch < n) {
                sb += s.clen(sb);
                ch++;
            }
            if (ch == n || x.n == 0) {   // truncated to n characters, or nothing to pad with
                if (d) copy_view(d, s.p, sb, s.xf);
                return sb;
            }
            int64_t pc = 0;
            for (int32_t j = 0; j < x.n; j += x.clen(j)) pc++;
            const int64_t q = (n - ch) / pc, r = (n - ch) % pc;   // n - ch pad characters: q whole pads and r more
            int32_t rb = 0;
            for (int64_t c = 0; c < r; c++) rb += x.clen(rb);
            if (q > (SB_SAT - sb - rb) / x.n) return SB_SAT;
            if (d) {
                uint8_t* pd = fn == SBF_LPAD ? d : d + sb;
                for (int64_t c = 0; c < q; c++) copy_view(pd + c * x.n, x.p, x.n, x.xf);
                copy_view(pd + q * x.n, x.p, rb, x.xf);
                copy_view(fn == SBF_LPAD ? d + q * x.n + rb : d, s.p, sb, s.xf);
            }
            return sb + q * x.n + rb;
        }
        case SBF_REPLACE: {   // Spark UTF8String.replace: matches left to right, not overlapping; an empty search changes nothing
            if (x.n == 0) {
                if (d) copy_view(d, s.p, s.n, s.xf);
                return s.n;
            }
            int64_t o = 0;
            for (int32_t i = 0; i < s.n;) {
                if (i <= s.n - x.n && sv_eq(s, i, x, 0, x.n)) {
                    if (d) copy_view(d + o, y.p, y.n, y.xf);
                    o += y.n;
                    i += x.n;
                } else {
                    if (d) d[o] = s.at(i);
                    o++;
                    i++;
                }
            }
            return o;
        }
        case SBF_TRANSLATE: {   // Spark StringTranslate: the k-th character of x becomes the k-th of y, or is deleted when y is shorter;
                                // a character repeated in x keeps its first position
            int64_t o = 0;
            for (int32_t i = 0; i < s.n;) {
                const int32_t cl = s.clen(i);
                const int32_t k = sv_char_index(x, s, i, cl);
                if (k < 0) {
                    if (d) copy_view(d + o, s.p + i, cl, s.xf);
                    o += cl;
                } else {
                    int32_t j = 0;
                    for (int32_t c = 0; j < y.n && c < k; c++) j += y.clen(j);
                    if (j < y.n) {
                        const int32_t tl = y.clen(j);
                        if (d) copy_view(d + o, y.p + j, tl, y.xf);
                        o += tl;
                    }
                }
                i += cl;
            }
            return o;
        }
        case SBF_REVERSE:
            if (d)
                for (int32_t i = 0; i < s.n;) {
                    const int32_t cl = s.clen(i);
                    copy_view(d + s.n - i - cl, s.p + i, cl, s.xf);
                    i += cl;
                }
            return s.n;
        default:   // SBF_INITCAP, spark_initcap.rs:40-66 for ASCII: a letter or digit first or after ' ' upper-cased, every other
                   // letter lower-cased; other bytes copied
            if (d) {
                bool after_space = true;
                for (int32_t i = 0; i < s.n; i++) {
                    uint8_t c = s.at(i);
                    if (after_space && c >= 'a' && c <= 'z') c -= 32;
                    else if (!after_space && c >= 'A' && c <= 'Z') c += 32;
                    d[i] = c;
                    after_space = c == ' ';
                }
            }
            return s.n;
    }
}

// TEXT (implies HI): the program formats decimals or floats as text or parses floats or booleans from it.  That code runs in
// its own instantiation: calls into it cost the other programs of vm_kernel<true> registers and stack.
template <bool HI, bool TEXT = false>
__global__ void __launch_bounds__(VM_THREADS) vm_kernel(VmParams p) {
    extern __shared__ __align__(16) uint64_t vm_smem[];
    uint64_t* LO = vm_smem;
    int64_t* HIp = (int64_t*)(vm_smem + (HI ? VM_NREG * VM_THREADS : 0));
    Instr* prog = (Instr*)(vm_smem + (HI ? 2 : 1) * VM_NREG * VM_THREADS);
    const int tid = threadIdx.x;
    char buf[44];   // CAST(x AS STRING) text of OP_FMT_OUT / OP_SB_APPEND
    for (int i = tid; i < p.n_instr * (int)(sizeof(Instr) / 4); i += VM_THREADS) ((uint32_t*)prog)[i] = ((const uint32_t*)p.prog)[i];
    __syncthreads();

#define RLO(r) LO[(r) * VM_THREADS + tid]
#define RHI(r) HIp[(r) * VM_THREADS + tid]
#define VALID(r) ((vmask >> (r)) & 1u)
#define SETV(r, v) vmask = (vmask & ~(1u << (r))) | ((v) ? (1u << (r)) : 0u)

    for (int64_t base = (int64_t)blockIdx.x * VM_THREADS; base < p.n; base += (int64_t)gridDim.x * VM_THREADS) {
        const int64_t i = base + tid;
        const bool active = i < p.n;
        const int64_t row = active ? (p.sel ? (int64_t)p.sel[i] : i) : (p.sel ? (int64_t)p.sel[0] : 0);
        uint32_t vmask = 0;
        for (int pc = 0; pc < p.n_instr; pc++) {
            const Instr ins = prog[pc];
            const int t = ins.t;
            switch (ins.op) {
                case OP_LOAD: {
                    const int c = ins.aux;
                    bool v = valid_at(p.in_valid[c], row);
                    uint64_t x = 0;
                    const void* d = p.in_data[c];
                    switch (t) {
                        case VT_BOOL: x = bit_get((const uint8_t*)d, row); break;
                        case VT_I8: x = (uint64_t)(int64_t)((const int8_t*)d)[row]; break;
                        case VT_I16: x = (uint64_t)(int64_t)((const int16_t*)d)[row]; break;
                        case VT_I32: x = (uint64_t)(int64_t)((const int32_t*)d)[row]; break;
                        case VT_F32: x = ((const uint32_t*)d)[row]; break;
                        case VT_I64: case VT_F64: x = ((const uint64_t*)d)[row]; break;
                        case VT_DEC: {
                            ulonglong2 q = ((const ulonglong2*)d)[row];
                            x = q.x;
                            if (HI) RHI(ins.dst) = (int64_t)q.y;
                            break;
                        }
                        case VT_STR: {
                            int32_t b = p.in_off[c][row], e = p.in_off[c][row + 1];
                            x = ((uint64_t)(uint32_t)b << 32) | (uint32_t)(e - b);
                            if (HI) RHI(ins.dst) = c;
                            break;
                        }
                    }
                    RLO(ins.dst) = x;
                    SETV(ins.dst, v);
                    break;
                }
                case OP_CONST: {
                    ConstEntry ce = p.consts[ins.aux];
                    RLO(ins.dst) = ce.lo;
                    if (HI) RHI(ins.dst) = ce.hi;
                    SETV(ins.dst, ce.valid != 0);
                    break;
                }
                case OP_ADD: case OP_SUB: case OP_MUL: case OP_DIV: case OP_MOD:
                case OP_BITAND: case OP_BITOR: case OP_BITXOR: case OP_SHL: case OP_SHR: {
                    bool v = VALID(ins.a) && VALID(ins.b);
                    uint64_t a = RLO(ins.a), b = RLO(ins.b), r = 0;
                    if (t <= VT_I64) {
                        int64_t x = (int64_t)a, y = (int64_t)b, z = 0;
                        switch (ins.op) {
                            case OP_ADD: z = (int64_t)((uint64_t)x + (uint64_t)y); break;
                            case OP_SUB: z = (int64_t)((uint64_t)x - (uint64_t)y); break;
                            case OP_MUL: z = (int64_t)((uint64_t)x * (uint64_t)y); break;
                            case OP_DIV:
                                if (y == 0) v = false;
                                else z = (y == -1) ? (int64_t)(0ull - (uint64_t)x) : x / y;
                                break;
                            case OP_MOD:
                                if (y == 0) v = false;
                                else z = (y == -1) ? 0 : x % y;
                                break;
                            case OP_BITAND: z = x & y; break;
                            case OP_BITOR: z = x | y; break;
                            case OP_BITXOR: z = x ^ y; break;
                            case OP_SHL: z = (int64_t)((uint64_t)x << (y & (t == VT_I64 ? 63 : 31))); break;
                            case OP_SHR: z = x >> (y & (t == VT_I64 ? 63 : 31)); break;
                        }
                        r = (uint64_t)sext(z, t);
                    } else if (t == VT_F32) {
                        float x = __int_as_float((int)(uint32_t)a), y = __int_as_float((int)(uint32_t)b), z = 0;
                        switch (ins.op) {
                            case OP_ADD: z = x + y; break;
                            case OP_SUB: z = x - y; break;
                            case OP_MUL: z = x * y; break;
                            case OP_DIV: z = x / y; break;
                            case OP_MOD: z = fmodf(x, y); break;
                        }
                        r = (uint32_t)__float_as_int(z);
                    } else if (t == VT_F64) {
                        double x = __longlong_as_double((int64_t)a), y = __longlong_as_double((int64_t)b), z = 0;
                        switch (ins.op) {
                            case OP_ADD: z = x + y; break;
                            case OP_SUB: z = x - y; break;
                            case OP_MUL: z = x * y; break;
                            case OP_DIV: z = x / y; break;
                            case OP_MOD: z = fmod(x, y); break;
                        }
                        r = (uint64_t)__double_as_longlong(z);
                    } else if (t == VT_DEC && HI) {   // aux: the declared precision of the result
                        i128 x = {a, RHI(ins.a)}, y = {b, RHI(ins.b)}, z = {0, 0};
                        if (v && !dec_arith(ins.op, x, y, ins.aux, &z)) v = false;
                        if (!v) z = {0, 0};
                        r = z.lo;
                        RHI(ins.dst) = z.hi;
                    }
                    RLO(ins.dst) = r;
                    SETV(ins.dst, v);
                    break;
                }
                case OP_NEG: case OP_ABS: {
                    uint64_t a = RLO(ins.a), r = a;
                    bool neg_it = ins.op == OP_NEG;
                    if (t <= VT_I64) {
                        int64_t x = (int64_t)a;
                        if (neg_it || x < 0) r = (uint64_t)sext((int64_t)(0ull - (uint64_t)x), t);
                    } else if (t == VT_F32) {
                        r = neg_it ? (a ^ 0x80000000ull) : (a & 0x7fffffffull);
                    } else if (t == VT_F64) {
                        r = neg_it ? (a ^ 0x8000000000000000ull) : (a & 0x7fffffffffffffffull);
                    } else if (t == VT_DEC && HI) {
                        i128 x = {a, RHI(ins.a)};
                        if (neg_it || i128_is_neg(x)) x = i128_neg(x);
                        r = x.lo;
                        RHI(ins.dst) = x.hi;
                    }
                    RLO(ins.dst) = r;
                    SETV(ins.dst, VALID(ins.a));
                    break;
                }
                case OP_EQ: case OP_NE: case OP_LT: case OP_LE: case OP_GT: case OP_GE: case OP_NSEQ: case OP_GREATEST: {
                    bool va = VALID(ins.a), vb = VALID(ins.b);
                    uint64_t a = RLO(ins.a), b = RLO(ins.b);
                    int c = 0;
                    if (va && vb) {
                        if (t <= VT_I64) c = (int64_t)a < (int64_t)b ? -1 : ((int64_t)a > (int64_t)b ? 1 : 0);
                        else if (t == VT_F32) {
                            int32_t x = f32_total(__int_as_float((int)(uint32_t)a)), y = f32_total(__int_as_float((int)(uint32_t)b));
                            c = x < y ? -1 : (x > y ? 1 : 0);
                        } else if (t == VT_F64) {
                            int64_t x = f64_total(__longlong_as_double((int64_t)a)), y = f64_total(__longlong_as_double((int64_t)b));
                            c = x < y ? -1 : (x > y ? 1 : 0);
                        } else if (t == VT_DEC && HI) c = i128_cmp({a, RHI(ins.a)}, {b, RHI(ins.b)});
                        else if (t == VT_STR && HI) c = sv_cmp(sview(p, RHI(ins.a), a), sview(p, RHI(ins.b), b));   // through the case marks
                    }
                    if (ins.op == OP_GREATEST) {   // a = the running greatest (flags 0) / least (1): b replaces it when it is strictly
                                                   // beyond it or a is NULL; a NULL b is skipped
                        if (vb && (!va || (ins.flags ? c > 0 : c < 0))) {
                            RLO(ins.dst) = b;
                            if (HI) RHI(ins.dst) = RHI(ins.b);
                            SETV(ins.dst, true);
                        }
                        break;
                    }
                    bool r = false, v = va && vb;
                    switch (ins.op) {
                        case OP_EQ: r = c == 0; break;
                        case OP_NE: r = c != 0; break;
                        case OP_LT: r = c < 0; break;
                        case OP_LE: r = c <= 0; break;
                        case OP_GT: r = c > 0; break;
                        case OP_GE: r = c >= 0; break;
                        case OP_NSEQ: r = (va == vb) && (!va || c == 0); v = true; break;
                    }
                    RLO(ins.dst) = r;
                    SETV(ins.dst, v);
                    break;
                }
                case OP_AND: case OP_OR: {
                    bool va = VALID(ins.a), vb = VALID(ins.b);
                    bool a = va && RLO(ins.a) != 0, b = vb && RLO(ins.b) != 0;   // "definitely true"
                    bool fa = va && RLO(ins.a) == 0, fb = vb && RLO(ins.b) == 0; // "definitely false"
                    bool r, v;
                    if (ins.op == OP_AND) { r = a && b; v = (va && vb) || fa || fb; }
                    else { r = a || b; v = (va && vb) || a || b; }
                    RLO(ins.dst) = r;
                    SETV(ins.dst, v);
                    break;
                }
                case OP_NOT: RLO(ins.dst) = RLO(ins.a) == 0; SETV(ins.dst, VALID(ins.a)); break;
                case OP_ISNULL: RLO(ins.dst) = !VALID(ins.a); SETV(ins.dst, true); break;
                case OP_ISNOTNULL: RLO(ins.dst) = VALID(ins.a); SETV(ins.dst, true); break;
                case OP_SELECT: case OP_COALESCE: {
                    int src;
                    if (ins.op == OP_SELECT) src = (VALID(ins.a) && RLO(ins.a) != 0) ? ins.b : ins.c;
                    else src = VALID(ins.a) ? ins.a : ins.b;
                    uint64_t x = RLO(src);
                    bool v = VALID(src);
                    if (HI) {
                        int64_t h = RHI(src);
                        RHI(ins.dst) = h;
                    }
                    RLO(ins.dst) = x;
                    SETV(ins.dst, v);
                    break;
                }
                case OP_CAST: {
                    bool v = VALID(ins.a);
                    uint64_t lo = RLO(ins.a);
                    int64_t hi = HI ? RHI(ins.a) : 0;
                    int dt = ins.aux & 0xff, sscale = (ins.aux >> 8) & 0xff;
                    int dprec = (int8_t)((ins.aux2 >> 8) & 0xff), dscale = (int8_t)(ins.aux2 & 0xff);
                    if (v) {   // utf8 -> float / bool only in vm_kernel<true, true> (the compiler sets need_text for them)
                        if (TEXT && t == VT_STR && (dt == VT_F32 || dt == VT_F64 || dt == VT_BOOL)) v = str_to_float_or_bool(p, dt, lo, hi);
                        else v = vm_cast(p, t, dt, sscale, dprec, dscale, lo, hi);
                    }
                    RLO(ins.dst) = v ? lo : 0;
                    if (HI) RHI(ins.dst) = v ? hi : 0;
                    SETV(ins.dst, v);
                    break;
                }
                case OP_STARTS: case OP_ENDS: case OP_CONTAINS: case OP_LIKE: {
                    bool v = VALID(ins.a), r = false;
                    if (HI && v) {
                        uint64_t sv = RLO(ins.a);
                        const uint8_t* s = str_ptr(p, RHI(ins.a), sv);
                        int32_t ls = str_len(sv);
                        ConstEntry ce = p.consts[ins.aux];
                        const uint8_t* pat = p.pool + (uint32_t)(ce.lo >> 32);
                        int32_t lp = (int32_t)(uint32_t)ce.lo;
                        if (ins.op == OP_STARTS) {
                            r = ls >= lp;
                            for (int32_t k = 0; r && k < lp; k++) r = s[k] == pat[k];
                        } else if (ins.op == OP_ENDS) {
                            r = ls >= lp;
                            for (int32_t k = 0; r && k < lp; k++) r = s[ls - lp + k] == pat[k];
                        } else if (ins.op == OP_CONTAINS) r = str_contains(s, ls, pat, lp);
                        else {
                            r = str_like(s, ls, pat, lp, (ins.flags & 2) != 0);
                            if (ins.flags & 1) r = !r;
                        }
                    }
                    RLO(ins.dst) = r;
                    SETV(ins.dst, v);
                    break;
                }
                case OP_SUBSTR: {   // datafusion unicode::substr: 1-based character position, optional count
                    bool v = VALID(ins.a) && VALID(ins.b) && (ins.c == 0xff || VALID(ins.c));
                    uint64_t outv = 0;
                    int64_t h = 0;
                    if (HI && v) {
                        uint64_t sv = RLO(ins.a);
                        h = RHI(ins.a);
                        const uint8_t* s = str_ptr(p, h, sv);
                        int32_t ls = str_len(sv);
                        int64_t start = (int64_t)RLO(ins.b);
                        int64_t cb = 0, ce = ls;   // byte range
                        // characters wanted: [start, start+count) 1-based; clamp as datafusion does
                        int64_t first_char = start - 1, last_char = INT64_MAX;
                        bool empty = false;
                        if (ins.c != 0xff) {
                            int64_t cnt = (int64_t)RLO(ins.c);
                            if (cnt < 0) { v = false; }
                            last_char = start - 1 + cnt;
                            if (last_char <= 0 || cnt == 0) empty = true;
                        }
                        if (first_char < 0) first_char = 0;
                        if (v) {
                            if (empty) { cb = ce = 0; }
                            else {
                                int64_t ch = 0;
                                int32_t bi = 0;
                                while (bi < ls && ch < first_char) { bi += utf8_char_len(s[bi]); ch++; }
                                cb = bi > ls ? ls : bi;
                                while (bi < ls && ch < last_char) { bi += utf8_char_len(s[bi]); ch++; }
                                ce = bi > ls ? ls : bi;
                            }
                            outv = ((uint64_t)((uint32_t)(sv >> 32) + (uint32_t)cb) << 32) | (uint32_t)(ce - cb);
                        }
                    }
                    RLO(ins.dst) = outv;
                    if (HI) RHI(ins.dst) = h;
                    SETV(ins.dst, v);
                    break;
                }
                case OP_CHARLEN: case OP_OCTLEN: {   // OP_CHARLEN flags: CL_CHARS, CL_ASCII, CL_FIND_IN_SET (the list in b)
                    bool v = VALID(ins.a);
                    if (HI && ins.flags == CL_FIND_IN_SET) v = v && VALID(ins.b);
                    int64_t r = 0;
                    if (HI && v) {
                        uint64_t sv = RLO(ins.a);
                        int32_t ls = str_len(sv);
                        if (ins.op == OP_OCTLEN) r = ls;
                        else if (ins.flags == CL_ASCII) r = str_ascii(sview(p, RHI(ins.a), sv));
                        else if (ins.flags == CL_FIND_IN_SET) r = str_find_in_set(sview(p, RHI(ins.a), sv), sview(p, RHI(ins.b), RLO(ins.b)));
                        else {
                            const uint8_t* s = str_ptr(p, RHI(ins.a), sv);
                            for (int32_t k = 0; k < ls; k++) r += (s[k] & 0xc0) != 0x80;
                        }
                    }
                    RLO(ins.dst) = (uint64_t)r;
                    SETV(ins.dst, v);
                    break;
                }
                case OP_TRIM: {   // flags: 1 = left, 2 = right ; trims ASCII space, or with TRIM_SET the characters of the view in b
                    bool v = VALID(ins.a);
                    if (HI && (ins.flags & TRIM_SET)) v = v && VALID(ins.b);
                    uint64_t sv = RLO(ins.a);
                    int64_t h = HI ? RHI(ins.a) : 0;
                    if (HI && v) {
                        const uint8_t* s = str_ptr(p, h, sv);
                        int32_t b = 0, e = str_len(sv);
                        if (ins.flags & TRIM_SET) trim_set(sview(p, h, sv), sview(p, RHI(ins.b), RLO(ins.b)), ins.flags, &b, &e);
                        else {
                            if (ins.flags & 1) while (b < e && s[b] == ' ') b++;
                            if (ins.flags & 2) while (e > b && s[e - 1] == ' ') e--;
                        }
                        sv = ((uint64_t)((uint32_t)(sv >> 32) + (uint32_t)b) << 32) | (uint32_t)(e - b);
                    }
                    RLO(ins.dst) = sv;
                    if (HI) RHI(ins.dst) = h;
                    SETV(ins.dst, v);
                    break;
                }
                case OP_CASEXF: {   // mark view for ASCII upper (1) / lower (2) at materialisation
                    RLO(ins.dst) = RLO(ins.a);
                    if (HI) RHI(ins.dst) = (RHI(ins.a) & 0xff) | ((int64_t)ins.flags << 8);
                    SETV(ins.dst, VALID(ins.a));
                    break;
                }
                case OP_DATEPART: {
                    bool v = VALID(ins.a);
                    RLO(ins.dst) = v ? (uint64_t)(int64_t)date_part((int64_t)RLO(ins.a), ins.aux) : 0;
                    SETV(ins.dst, v);
                    break;
                }
                case OP_ROUND: {   // Spark round / bround(x, aux): HALF_UP (spark_round.rs:38-134), flags = 1: HALF_EVEN (spark_bround.rs:38-134);
                                   // aux2 = scale of a decimal input
                    bool v = VALID(ins.a);
                    const int sc = ins.aux;
                    const bool even = ins.flags != 0;
                    uint64_t lo = RLO(ins.a);
                    int64_t hi = HI ? RHI(ins.a) : 0;
                    if (t == VT_DEC) {
                        __int128 x = ((__int128)hi << 64) | (__int128)lo;
                        const int diff = ins.aux2 - sc;   // digits of the stored scale that are rounded away
                        if (diff >= 0) x = even ? round_half_even_i128(x, diff) : round_half_up_i128(x, diff);
                        else
                            for (int k = 0; k < -diff && k < 39; k++) x *= 10;   // the reference keeps the declared scale here (:69-75)
                        lo = (uint64_t)x;
                        hi = (int64_t)(x >> 64);
                    } else if (t <= VT_I64) {
                        const __int128 r = even ? round_half_even_i128((__int128)(int64_t)lo, -sc) : round_half_up_i128((__int128)(int64_t)lo, -sc);
                        const int64_t w = t == VT_I64 ? (int64_t)r : t == VT_I32 ? (int64_t)(int32_t)r : t == VT_I16 ? (int64_t)(int16_t)r : (int64_t)(int8_t)r;
                        lo = (uint64_t)w;
                    } else if (t == VT_F64) {
                        const double x = __longlong_as_double((int64_t)lo);
                        if (!(isnan(x) || isinf(x))) {
                            const double f = powi10(sc), y = x * f;
                            lo = (uint64_t)__double_as_longlong((even ? round_half_even_f64(y) : (y >= 0.0 ? floor(y + 0.5) : ceil(y - 0.5))) / f);
                        }
                    } else if (t == VT_F32) {
                        const float x = __int_as_float((int)(uint32_t)lo);
                        if (!(isnan(x) || isinf(x))) {
                            float f = 1.0f;
                            for (int k = 0; k < (sc < 0 ? -sc : sc); k++) f *= 10.0f;
                            if (sc < 0) f = 1.0f / f;
                            const float y = x * f;
                            lo = (uint64_t)(uint32_t)__float_as_int((even ? round_half_even_f32(y) : (y >= 0.0f ? floorf(y + 0.5f) : ceilf(y - 0.5f))) / f);
                        }
                    }
                    RLO(ins.dst) = v ? lo : 0;
                    if (HI) RHI(ins.dst) = v ? hi : 0;
                    SETV(ins.dst, v);
                    break;
                }
                case OP_TS_LOCAL_MS: {   // aux = pool offset of the zone table (-1: none), aux2 = unit of the input
                    bool v = VALID(ins.a);
                    RLO(ins.dst) = v ? (uint64_t)ts_to_local_ms((int64_t)RLO(ins.a), ins.aux2, ins.aux >= 0 ? p.pool + ins.aux : nullptr) : 0;
                    SETV(ins.dst, v);
                    break;
                }
                case OP_TIMEPART: {      // extract_hms_with_tz (spark_dates.rs:313-345): aux = 0 hour, 1 minute, 2 second of local ms
                    bool v = VALID(ins.a);
                    int64_t day_ms = (int64_t)RLO(ins.a) % 86400000ll;
                    if (day_ms < 0) day_ms += 86400000ll;
                    const int64_t r = ins.aux == 0 ? day_ms / 3600000 : ins.aux == 1 ? (day_ms % 3600000) / 60000 : (day_ms % 60000) / 1000;
                    RLO(ins.dst) = v ? (uint64_t)r : 0;
                    SETV(ins.dst, v);
                    break;
                }
                case OP_MS_TO_DAYS: {    // aux = 0: floor (ts_ms_to_local_date32, spark_dates.rs:213-227); 1: toward zero (arrow cast to Date32)
                    bool v = VALID(ins.a);
                    const int64_t ms = (int64_t)RLO(ins.a);
                    int64_t d = ms / 86400000ll;
                    if (ins.aux == 0 && ms < 0 && ms % 86400000ll != 0) d -= 1;
                    RLO(ins.dst) = v ? (uint64_t)(int64_t)(int32_t)d : 0;
                    SETV(ins.dst, v);
                    break;
                }
                case OP_NULLIFZERO: {
                    bool v = VALID(ins.a);
                    uint64_t a = RLO(ins.a);
                    bool zero = false;
                    if (t <= VT_I64) zero = a == 0;
                    else if (t == VT_F32) zero = __int_as_float((int)(uint32_t)a) == 0.0f;
                    else if (t == VT_F64) zero = __longlong_as_double((int64_t)a) == 0.0;
                    else if (t == VT_DEC && HI) zero = a == 0 && RHI(ins.a) == 0;
                    RLO(ins.dst) = a;
                    if (HI) RHI(ins.dst) = RHI(ins.a);
                    SETV(ins.dst, v && !zero);
                    break;
                }
                case OP_ISNAN: {
                    uint64_t a = RLO(ins.a);
                    bool r = VALID(ins.a) && (t == VT_F32 ? isnan(__int_as_float((int)(uint32_t)a)) : isnan(__longlong_as_double((int64_t)a)));
                    RLO(ins.dst) = r;
                    SETV(ins.dst, true);
                    break;
                }
                case OP_NORMNAN: {   // NaN -> canonical NaN, -0.0 -> 0.0
                    uint64_t a = RLO(ins.a);
                    if (t == VT_F32) {
                        float x = __int_as_float((int)(uint32_t)a);
                        if (isnan(x)) a = 0x7fc00000u;
                        else if (x == 0.0f) a = 0;
                    } else {
                        double x = __longlong_as_double((int64_t)a);
                        if (isnan(x)) a = 0x7ff8000000000000ull;
                        else if (x == 0.0) a = 0;
                    }
                    RLO(ins.dst) = a;
                    SETV(ins.dst, VALID(ins.a));
                    break;
                }
                case OP_CHECK_OVERFLOW: {   // decimal precision overflow -> NULL (spark_check_overflow.rs:25)
                    bool v = VALID(ins.a);
                    uint64_t lo = RLO(ins.a);
                    int64_t hi = HI ? RHI(ins.a) : 0;
                    if (v) v = vm_cast(p, VT_DEC, VT_DEC, (ins.aux >> 8) & 0xff, (int8_t)((ins.aux2 >> 8) & 0xff), (int8_t)(ins.aux2 & 0xff), lo, hi);
                    RLO(ins.dst) = v ? lo : 0;
                    if (HI) RHI(ins.dst) = v ? hi : 0;
                    SETV(ins.dst, v);
                    break;
                }
                case OP_MAKE_DECIMAL: {   // i64 unscaled -> decimal(p, s), overflow -> NULL (spark_make_decimal.rs:25)
                    bool v = VALID(ins.a);
                    i128 x = i128_from_i64((int64_t)RLO(ins.a));
                    if (v && !dec_fits_precision(x, ins.aux)) v = false;
                    RLO(ins.dst) = x.lo;
                    if (HI) RHI(ins.dst) = x.hi;
                    SETV(ins.dst, v);
                    break;
                }
                case OP_UNSCALED: RLO(ins.dst) = RLO(ins.a); SETV(ins.dst, VALID(ins.a)); break;   // low 64 bits (spark_unscaled_value.rs:25)
                case OP_MATH1: {
                    double x = __longlong_as_double((int64_t)RLO(ins.a)), r = 0;
                    switch (ins.aux) {
                        case M_SQRT: r = sqrt(x); break;
                        case M_EXP: r = exp(x); break;
                        case M_LN: r = log(x); break;
                        case M_LOG10: r = log10(x); break;
                        case M_LOG2: r = log2(x); break;
                        case M_SIN: r = sin(x); break;
                        case M_COS: r = cos(x); break;
                        case M_TAN: r = tan(x); break;
                        case M_ASIN: r = asin(x); break;
                        case M_ACOS: r = acos(x); break;
                        case M_ATAN: r = atan(x); break;
                        case M_CEIL: r = ceil(x); break;
                        case M_FLOOR: r = floor(x); break;
                        case M_SIGNUM: r = x > 0 ? 1.0 : (x < 0 ? -1.0 : x); break;
                        case M_TRUNC: r = trunc(x); break;
                        case M_EXPM1: r = expm1(x); break;
                        case M_ACOSH: r = acosh(x); break;
                    }
                    RLO(ins.dst) = (uint64_t)__double_as_longlong(r);
                    SETV(ins.dst, VALID(ins.a));
                    break;
                }
                case OP_POW: {
                    double x = __longlong_as_double((int64_t)RLO(ins.a)), y = __longlong_as_double((int64_t)RLO(ins.b));
                    RLO(ins.dst) = (uint64_t)__double_as_longlong(pow(x, y));
                    SETV(ins.dst, VALID(ins.a) && VALID(ins.b));
                    break;
                }
                case OP_HASH: {   // dst = running hash (i32 murmur3 flags=0 / i64 xxhash64 flags=1), a = value of type t
                    uint64_t h = RLO(ins.dst);
                    if (VALID(ins.a)) {
                        uint64_t a = RLO(ins.a);
                        bool mm = ins.flags == 0;
                        switch (t) {
                            case VT_BOOL: case VT_I8: case VT_I16: case VT_I32: case VT_F32:
                                h = mm ? (uint64_t)(int64_t)(int32_t)murmur3_u32((uint32_t)a, (uint32_t)h) : xxhash64_u32((uint32_t)a, h);
                                break;
                            case VT_I64: case VT_F64: h = mm ? (uint64_t)(int64_t)(int32_t)murmur3_u64(a, (uint32_t)h) : xxhash64_u64(a, h); break;
                            case VT_DEC:
                                if (HI) h = mm ? (uint64_t)(int64_t)(int32_t)murmur3_u128(a, (uint64_t)RHI(ins.a), (uint32_t)h) : xxhash64_u128(a, (uint64_t)RHI(ins.a), h);
                                break;
                            case VT_STR:
                                if (HI) {
                                    const uint8_t* s = str_ptr(p, RHI(ins.a), a);
                                    h = mm ? (uint64_t)(int64_t)(int32_t)murmur3_bytes(s, str_len(a), (uint32_t)h) : xxhash64_bytes(s, str_len(a), h);
                                }
                                break;
                        }
                    }
                    RLO(ins.dst) = h;
                    SETV(ins.dst, true);
                    break;
                }
                // The calendar operations run in vm_kernel<true> only (the compiler sets need_hi for them): in vm_kernel<false> they
                // would cost every plain numeric program 16 registers.
                case OP_DATE_TRUNC: {   // aux = TruncLevel, aux2 = unit of the input | unit of the result << 4
                    int64_t r = 0;
                    const bool v = HI && VALID(ins.a) && date_trunc((int64_t)RLO(ins.a), ins.aux2 & 15, ins.aux, ins.aux2 >> 4, &r);
                    RLO(ins.dst) = (uint64_t)r;
                    SETV(ins.dst, v);
                    break;
                }
                case OP_MAKE_DATE: {   // int32 year a, month b, day c -> date32
                    int64_t r = 0;
                    const bool v = HI && VALID(ins.a) && VALID(ins.b) && VALID(ins.c) &&
                                   make_date((int64_t)RLO(ins.a), (int64_t)RLO(ins.b), (int64_t)RLO(ins.c), &r);
                    RLO(ins.dst) = (uint64_t)r;
                    SETV(ins.dst, v);
                    break;
                }
                case OP_FACTORIAL: {   // int32 -> int64, NULL outside 0..20
                    const int64_t x = (int64_t)RLO(ins.a);
                    int64_t r = 1;
                    for (int64_t k = 2; k <= x && k <= 20; k++) r *= k;
                    RLO(ins.dst) = (uint64_t)r;
                    SETV(ins.dst, VALID(ins.a) && x >= 0 && x <= 20);
                    break;
                }
                case OP_ROWNUM: RLO(ins.dst) = (uint64_t)(p.row_base + i); SETV(ins.dst, true); break;
                case OP_MONTHS_BETWEEN: {   // UTC ms a, b, bool roundOff c; aux = pool offset of the zone table (-1: UTC)
                    double r = 0;
                    const bool v = HI && VALID(ins.a) && VALID(ins.b) && VALID(ins.c) &&
                                   months_between((int64_t)RLO(ins.a), (int64_t)RLO(ins.b), RLO(ins.c) != 0, ins.aux >= 0 ? p.pool + ins.aux : nullptr, &r);
                    RLO(ins.dst) = (uint64_t)__double_as_longlong(r);
                    SETV(ins.dst, v);
                    break;
                }
                case OP_OUT: {
                    const int o = ins.aux;
                    bool v = active && VALID(ins.a);
                    uint64_t x = RLO(ins.a);
                    if (t == VT_STR) {
                        if (HI) {
                            if (p.mode == 0) {
                                if (active) p.out_lens[o][i] = v ? (int64_t)str_len(x) : 0;
                            } else if (v) {
                                int64_t h = RHI(ins.a);
                                copy_view((uint8_t*)p.out_data[o] + p.out_off[o][i], str_ptr(p, h, x), str_len(x), (int)((h >> 8) & 0xff));
                            }
                        }
                        if (p.mode == 0) {
                            uint32_t w = __ballot_sync(FULL_MASK, v);
                            if ((tid & 31) == 0 && active) p.out_valid[o][i >> 5] = w;
                        }
                    } else if (p.mode == 0) {
                        if (t == VT_BOOL) {
                            uint32_t wb = __ballot_sync(FULL_MASK, v && x != 0);
                            if ((tid & 31) == 0 && active) ((uint32_t*)p.out_data[o])[i >> 5] = wb;
                        } else if (active) {
                            if (!v) x = 0;
                            switch (t) {
                                case VT_I8: ((int8_t*)p.out_data[o])[i] = (int8_t)x; break;
                                case VT_I16: ((int16_t*)p.out_data[o])[i] = (int16_t)x; break;
                                case VT_I32: case VT_F32: ((uint32_t*)p.out_data[o])[i] = (uint32_t)x; break;
                                case VT_I64: case VT_F64: ((uint64_t*)p.out_data[o])[i] = x; break;
                                case VT_DEC: {
                                    ulonglong2 q;
                                    q.x = x;
                                    q.y = (HI && v) ? (uint64_t)RHI(ins.a) : 0;
                                    ((ulonglong2*)p.out_data[o])[i] = q;
                                    break;
                                }
                            }
                        }
                        uint32_t w = __ballot_sync(FULL_MASK, v);
                        if ((tid & 31) == 0 && active) p.out_valid[o][i >> 5] = w;
                    }
                    break;
                }
                case OP_FMT_OUT: {   // CAST(value AS STRING) straight into a utf8 output column (both passes format the value)
                    const int o = ins.aux;
                    bool v = active && VALID(ins.a);
                    int len = v ? fmt_value<TEXT>((ins.aux2 >> 8) & 0xff, ins.aux2 & 0xff, RLO(ins.a), TEXT ? RHI(ins.a) : 0, buf) : 0;
                    if (p.mode == 0) {
                        if (active) p.out_lens[o][i] = len;
                        uint32_t w = __ballot_sync(FULL_MASK, v);
                        if ((tid & 31) == 0 && active) p.out_valid[o][i >> 5] = w;
                    } else if (v) {
                        uint8_t* d = (uint8_t*)p.out_data[o] + p.out_off[o][i];
                        for (int k = 0; k < len; k++) d[k] = (uint8_t)buf[k];
                    }
                    break;
                }
                // String builder (concat / concat_ws / repeat / space) into utf8 output `o`: dst holds the cursor (LO), whether a
                // piece was emitted (HI) and the row's validity.  Pass 0 adds up the piece lengths, pass 1 copies each piece at
                // out_off[i] + cursor; it takes the validity pass 0 found, so a row that ends NULL writes nothing.
                case OP_SB_BEGIN: {
                    const int o = ins.aux;
                    RLO(ins.dst) = 0;
                    if (HI) RHI(ins.dst) = 0;
                    SETV(ins.dst, active && (p.mode == 0 || ((p.out_valid[o][i >> 5] >> (i & 31)) & 1u)));
                    break;
                }
                case OP_SB_APPEND: {
                    if (!HI || !VALID(ins.dst)) break;
                    const int kind = ins.flags & 3, fn = ins.flags >> 4;
                    if (!VALID(ins.a) || (fn >= SBF_LPAD && fn <= SBF_TRANSLATE && !(VALID(ins.b) && VALID(ins.c)))) {
                        // concat: a NULL piece (a string function with a NULL argument) makes the row NULL; concat_ws skips it
                        if (!(ins.flags & SB_WS)) SETV(ins.dst, false);
                        break;
                    }
                    const int o = ins.aux & 0xff;
                    int64_t cur = (int64_t)RLO(ins.dst);
                    uint8_t* d = p.mode == 1 ? (uint8_t*)p.out_data[o] + p.out_off[o][i] : nullptr;
                    if ((ins.flags & SB_WS) && RHI(ins.dst)) {
                        const uint64_t sep = p.consts[ins.aux >> 8].lo;
                        if (d) copy_view(d + cur, p.pool + (uint32_t)(sep >> 32), str_len(sep), 0);
                        cur += str_len(sep);
                    }
                    RHI(ins.dst) = 1;
                    const uint64_t x = RLO(ins.a);
                    if (kind == SB_SPACE) {
                        const int64_t n = (int32_t)x > 0 ? (int32_t)x : 0;
                        if (d)
                            for (int64_t k = 0; k < n; k++) d[cur + k] = ' ';
                        cur += n;
                    } else if (fn != SBF_NONE) {   // lpad / rpad: b = length, c = pad; replace / translate: b, c; hex / chr of an
                                                   // integer: a; others: s only
                        SView s{nullptr, 0, 0}, u{nullptr, 0, 0}, w{nullptr, 0, 0};
                        int64_t n = 0;
                        if (fn == SBF_HEX_INT || fn == SBF_CHR) n = (int64_t)x;
                        else s = sview(p, RHI(ins.a), x);
                        if (fn <= SBF_RPAD) {
                            n = (int64_t)RLO(ins.b);
                            u = sview(p, RHI(ins.c), RLO(ins.c));
                        } else if (fn <= SBF_TRANSLATE) {
                            u = sview(p, RHI(ins.b), RLO(ins.b));
                            w = sview(p, RHI(ins.c), RLO(ins.c));
                        }
                        cur += sb_fn_piece(fn, s, u, w, n, d ? d + cur : nullptr);
                    } else {   // a view or a formatted value, once or `times` times
                        const int64_t times = (ins.flags & SB_REPEAT) ? (int64_t)p.consts[ins.aux >> 8].lo : 1;
                        const uint8_t* s;
                        int32_t len;
                        int xf = 0;
                        if (kind == SB_FMT) {
                            len = fmt_value<TEXT>((ins.aux2 >> 8) & 0xff, ins.aux2 & 0xff, x, TEXT ? RHI(ins.a) : 0, buf);
                            s = (const uint8_t*)buf;
                        } else {
                            const int64_t h = RHI(ins.a);
                            s = str_ptr(p, h, x);
                            len = str_len(x);
                            xf = (int)((h >> 8) & 0xff);
                        }
                        for (int64_t r = 0; d && r < times; r++) copy_view(d + cur + r * len, s, len, xf);
                        cur += times * len;
                    }
                    RLO(ins.dst) = (uint64_t)(cur < SB_SAT ? cur : SB_SAT);
                    break;
                }
                case OP_SB_END: {
                    const int o = ins.aux;
                    const bool v = VALID(ins.a);
                    if (p.mode == 0) {
                        if (active) p.out_lens[o][i] = v ? (int64_t)RLO(ins.a) : 0;
                        uint32_t w = __ballot_sync(FULL_MASK, v);
                        if ((tid & 31) == 0 && active) p.out_valid[o][i >> 5] = w;
                    }
                    break;
                }
                case OP_OUT_PRED: {
                    bool keep = active && VALID(ins.a) && RLO(ins.a) != 0;
                    uint32_t w = __ballot_sync(FULL_MASK, keep);
                    if ((tid & 31) == 0 && active) p.pred_out[i >> 5] = w;
                    break;
                }
            }
        }
    }
#undef RLO
#undef RHI
#undef VALID
#undef SETV
}

// vm_kernel<true, true> is compiled in a translation unit of its own (k_expr_text.cu, which includes this file): its out-of-line
// calls into the text casts, in one module with the other instantiations, cost vm_kernel<true> spills.
void launch_vm_text(unsigned grid, size_t smem, cudaStream_t stream, const VmParams& p);
#ifdef AURON_VM_TEXT_TU
void launch_vm_text(unsigned grid, size_t smem, cudaStream_t stream, const VmParams& p) {
    static bool attr = false;
    init_pow10_tables();   // this module's copy
    if (!attr) {
        CUDA_OK(cudaFuncSetAttribute(vm_kernel<true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 2 * VM_NREG * VM_THREADS * 8 + 1024 * 16));
        attr = true;
    }
    vm_kernel<true, true><<<grid, VM_THREADS, smem, stream>>>(p);
}
#else
// ------------------------------------------------------------------------------------------ conjunctive compare fast path
// The overwhelmingly common filter shape (TPC-DS: BETWEEN, =, <, IS NOT NULL on fixed-width columns) is a conjunction of
// `column <op> literal` terms.  Those skip the interpreter: every thread loads each referenced column once into
// registers, evaluates the terms and the warp ballots the keep-bits into the selection bitmap -- one coalesced pass
// over the referenced columns, nothing else.  Semantics are those of the VM ops (NULL => row dropped).
constexpr int SP_MAX_TERMS = 8, SP_MAX_COLS = 4;
struct SimpleTerm {
    int32_t col;     // slot into SimplePredArgs::data
    int32_t op;      // OP_EQ..OP_GE, OP_ISNULL, OP_ISNOTNULL
    int64_t c_lo, c_hi;
};
struct SimplePredArgs {
    const void* data[SP_MAX_COLS];
    const uint8_t* valid[SP_MAX_COLS];
    int32_t vt[SP_MAX_COLS];
    SimpleTerm t[SP_MAX_TERMS];
    int32_t n_terms, n_cols;
};
__global__ void __launch_bounds__(256) simple_predicate_kernel(SimplePredArgs a, int64_t n, uint32_t* __restrict__ out) {
    int64_t stride = (int64_t)gridDim.x * 256;
    for (int64_t base = (int64_t)blockIdx.x * 256; base < n; base += stride) {
        int64_t i = base + threadIdx.x;
        bool active = i < n;
        uint64_t lo[SP_MAX_COLS];
        int64_t hi[SP_MAX_COLS];
        bool ok[SP_MAX_COLS];
#pragma unroll
        for (int c = 0; c < SP_MAX_COLS; c++) {
            lo[c] = 0;
            hi[c] = 0;
            ok[c] = false;
            if (c < a.n_cols && active) {
                ok[c] = valid_at(a.valid[c], i);
                const void* d = a.data[c];
                switch (a.vt[c]) {
                    case VT_BOOL: lo[c] = bit_get((const uint8_t*)d, i); break;
                    case VT_I8: lo[c] = (uint64_t)(int64_t)((const int8_t*)d)[i]; break;
                    case VT_I16: lo[c] = (uint64_t)(int64_t)((const int16_t*)d)[i]; break;
                    case VT_I32: lo[c] = (uint64_t)(int64_t)((const int32_t*)d)[i]; break;
                    case VT_F32: lo[c] = (uint64_t)(int64_t)f32_total(((const float*)d)[i]); break;
                    case VT_F64: lo[c] = (uint64_t)f64_total(((const double*)d)[i]); break;
                    case VT_DEC: {
                        ulonglong2 q = ((const ulonglong2*)d)[i];
                        lo[c] = q.x;
                        hi[c] = (int64_t)q.y;
                        break;
                    }
                    default: lo[c] = ((const uint64_t*)d)[i]; break;
                }
            }
        }
        bool keep = active;
        for (int k = 0; k < a.n_terms; k++) {
            const SimpleTerm t = a.t[k];
            uint64_t x = 0;
            int64_t xh = 0;
            bool v = false;
            int vt = 0;
#pragma unroll
            for (int c = 0; c < SP_MAX_COLS; c++)
                if (c == t.col) {
                    x = lo[c];
                    xh = hi[c];
                    v = ok[c];
                    vt = a.vt[c];
                }
            if (t.op == OP_ISNULL) { keep = keep && !v; continue; }
            if (t.op == OP_ISNOTNULL) { keep = keep && v; continue; }
            int cmp;
            if (vt == VT_DEC) cmp = i128_cmp({x, xh}, {(uint64_t)t.c_lo, t.c_hi});
            else cmp = (int64_t)x < t.c_lo ? -1 : ((int64_t)x > t.c_lo ? 1 : 0);
            bool r = false;
            switch (t.op) {
                case OP_EQ: r = cmp == 0; break;
                case OP_NE: r = cmp != 0; break;
                case OP_LT: r = cmp < 0; break;
                case OP_LE: r = cmp <= 0; break;
                case OP_GT: r = cmp > 0; break;
                case OP_GE: r = cmp >= 0; break;
            }
            keep = keep && v && r;
        }
        uint32_t wbits = __ballot_sync(FULL_MASK, keep);
        if ((threadIdx.x & 31) == 0 && active) out[i >> 5] = wbits;
    }
}

// When every term is an ordering comparison the conjunction folds (on the host) into one closed interval per column in the
// order-preserving int64 domain, and the kernel is a handful of instructions per row: 4 independent coalesced loads per
// thread (128 rows per warp iteration), one validity word per 32 rows, two compares, a ballot.
struct IntervalArgs {
    const void* data[SP_MAX_COLS];
    const uint32_t* valid[SP_MAX_COLS];
    int32_t vt[SP_MAX_COLS];
    int64_t lo[SP_MAX_COLS], hi[SP_MAX_COLS];
    int32_t n_cols;
};
__device__ __forceinline__ int64_t ordered_load(const void* d, int vt, int64_t i) {
    switch (vt) {
        case VT_BOOL: return bit_get((const uint8_t*)d, i);
        case VT_I8: return ((const int8_t*)d)[i];
        case VT_I16: return ((const int16_t*)d)[i];
        case VT_I32: return ((const int32_t*)d)[i];
        case VT_F32: return f32_total(((const float*)d)[i]);
        case VT_F64: return f64_total(((const double*)d)[i]);
        default: return ((const int64_t*)d)[i];
    }
}
template <int NCOLS>
__global__ void __launch_bounds__(256) interval_predicate_kernel(IntervalArgs a, int64_t n, uint32_t* __restrict__ out) {
    const unsigned lane = threadIdx.x & 31;
    const int64_t warp = ((int64_t)blockIdx.x * 256 + threadIdx.x) >> 5, nwarps = ((int64_t)gridDim.x * 256) >> 5;
    for (int64_t base = warp * 128; base < n; base += nwarps * 128) {
        bool keep[4];
#pragma unroll
        for (int k = 0; k < 4; k++) keep[k] = base + 32 * k + lane < n;
#pragma unroll
        for (int c = 0; c < NCOLS; c++) {
            int64_t x[4];
#pragma unroll
            for (int k = 0; k < 4; k++) {
                int64_t row = base + 32 * k + lane;
                x[k] = row < n ? ordered_load(a.data[c], a.vt[c], row) : 0;
            }
            const int64_t lo = a.lo[c], hi = a.hi[c];
#pragma unroll
            for (int k = 0; k < 4; k++) {
                bool v = true;
                if (a.valid[c] && base + 32 * k < n) v = (a.valid[c][(base >> 5) + k] >> lane) & 1u;
                keep[k] = keep[k] && v && x[k] >= lo && x[k] <= hi;
            }
        }
#pragma unroll
        for (int k = 0; k < 4; k++) {
            uint32_t w = __ballot_sync(FULL_MASK, keep[k]);
            if (lane == 0 && base + 32 * k < n) out[(base >> 5) + k] = w;
        }
    }
}

// Same predicate, all columns int32 (T = int32_t) or all int64: every lane takes 4 consecutive rows with one (or two)
// 128-bit loads, the 4-bit results of 8 lanes are OR-assembled into a mask word with three shuffles.  ~6 instructions
// per row instead of ~44: the kernel streams at HBM rate instead of being issue-bound.
template <typename T, int NCOLS>
__global__ void __launch_bounds__(256) interval_predicate_vec_kernel(IntervalArgs a, int64_t n, uint32_t* __restrict__ out) {
    const unsigned lane = threadIdx.x & 31;
    const unsigned sub = (lane & 7) * 4;
    const int64_t warp = ((int64_t)blockIdx.x * 256 + threadIdx.x) >> 5, nwarps = ((int64_t)gridDim.x * 256) >> 5;
    constexpr int64_t TMIN = sizeof(T) == 4 ? (int64_t)INT32_MIN : INT64_MIN, TMAX = sizeof(T) == 4 ? (int64_t)INT32_MAX : INT64_MAX;
    T lo[NCOLS], hi[NCOLS];
    bool empty = false;
#pragma unroll
    for (int c = 0; c < NCOLS; c++) {
        empty = empty || a.lo[c] > TMAX || a.hi[c] < TMIN;
        lo[c] = (T)(a.lo[c] < TMIN ? TMIN : a.lo[c]);
        hi[c] = (T)(a.hi[c] > TMAX ? TMAX : a.hi[c]);
    }
    for (int64_t base = warp * 128; base < n; base += nwarps * 128) {
        uint32_t nib = empty ? 0u : 0xFu;   // keep bits of rows base + 4 * lane + {0..3}
        if (base + 128 <= n) {
#pragma unroll
            for (int c = 0; c < NCOLS; c++) {
                T x[4];
                if (sizeof(T) == 4) {
                    const int4 v = ((const int4*)((const int32_t*)a.data[c] + base))[lane];
                    x[0] = (T)v.x, x[1] = (T)v.y, x[2] = (T)v.z, x[3] = (T)v.w;
                } else {
                    const longlong2* q = (const longlong2*)((const int64_t*)a.data[c] + base) + 2 * lane;
                    const longlong2 v0 = q[0], v1 = q[1];
                    x[0] = (T)v0.x, x[1] = (T)v0.y, x[2] = (T)v1.x, x[3] = (T)v1.y;
                }
                uint32_t m = 0;
#pragma unroll
                for (int k = 0; k < 4; k++) m |= (uint32_t)(x[k] >= lo[c] && x[k] <= hi[c]) << k;
                if (a.valid[c]) m &= a.valid[c][(base >> 5) + (lane >> 3)] >> sub;
                nib &= m;
            }
        } else {   // last, partial group of the column
            uint32_t m = 0;
            for (int k = 0; k < 4; k++) {
                const int64_t row = base + 4 * lane + k;
                bool keep = row < n;
                for (int c = 0; c < NCOLS && keep; c++) {
                    const T x = ((const T*)a.data[c])[row];
                    keep = x >= lo[c] && x <= hi[c] && (!a.valid[c] || ((a.valid[c][row >> 5] >> (row & 31)) & 1u));
                }
                m |= (uint32_t)keep << k;
            }
            nib &= m;
        }
        uint32_t w = (nib & 0xFu) << sub;
        w |= __shfl_xor_sync(FULL_MASK, w, 1);
        w |= __shfl_xor_sync(FULL_MASK, w, 2);
        w |= __shfl_xor_sync(FULL_MASK, w, 4);
        if ((lane & 7) == 0 && base + 32 * (lane >> 3) < n) out[(base >> 5) + (lane >> 3)] = w;
    }
}
template <typename T>
static void launch_interval_vec(Ctx& ctx, const IntervalArgs& a, int64_t n_rows, uint32_t* mask, unsigned grid) {
    switch (a.n_cols) {
        case 1: interval_predicate_vec_kernel<T, 1><<<grid, 256, 0, ctx.stream>>>(a, n_rows, mask); break;
        case 2: interval_predicate_vec_kernel<T, 2><<<grid, 256, 0, ctx.stream>>>(a, n_rows, mask); break;
        case 3: interval_predicate_vec_kernel<T, 3><<<grid, 256, 0, ctx.stream>>>(a, n_rows, mask); break;
        default: interval_predicate_vec_kernel<T, 4><<<grid, 256, 0, ctx.stream>>>(a, n_rows, mask); break;
    }
}

// ------------------------------------------------------------------------------------------ compiler (host)
struct VmProgramImpl {
    // interval form of the fast path (one closed interval per column); empty => not foldable
    std::vector<int64_t> iv_lo, iv_hi;
    // conjunctive-compare fast path (empty => use the interpreter)
    std::vector<SimpleTerm> simple_terms;
    std::vector<int> simple_cols;   // schema column per slot
    std::vector<int> simple_vt;
    std::vector<Instr> code;
    std::vector<ConstEntry> consts;
    std::string pool;
    std::vector<int> in_cols;     // VM input slot -> input schema column index
    std::vector<uint8_t> out_vt;  // VM type per output
    // md5 / sha2 outputs: hashed after the VM from an input column or from a hidden utf8 output of the program (numbered
    // after the visible outputs)
    struct Digest {
        int out, alg, col, hidden;   // col >= 0: input column, else output `hidden`
    };
    std::vector<Digest> digests;
    int n_hidden = 0;
    bool need_hi = false;
    bool need_text = false;   // float / decimal text casts: vm_kernel<true, true>
    // device copies (uploaded lazily per ctx stream; programs are immutable after compile)
    Buf d_code, d_consts, d_pool;
};

static Vt vt_of(const DType& t) {
    switch (t.id) {
        case T_BOOL: return VT_BOOL;
        case T_INT8: return VT_I8;
        case T_INT16: return VT_I16;
        case T_INT32: case T_DATE32: return VT_I32;
        case T_INT64: case T_DATE64: case T_TIMESTAMP: return VT_I64;
        case T_FLOAT32: return VT_F32;
        case T_FLOAT64: return VT_F64;
        case T_DECIMAL128: return VT_DEC;
        case T_UTF8: case T_BINARY: return VT_STR;
        default: fail("expression VM: unsupported type " + t.str());
    }
}

ExprPtr col(const std::string& name) {
    auto e = std::make_shared<Expr>();
    e->kind = E_COLUMN;
    e->name = name;
    return e;
}
ExprPtr col_idx(int index) {
    auto e = std::make_shared<Expr>();
    e->kind = E_COLUMN;
    e->index = index;
    return e;
}
ExprPtr lit_i64(int64_t v) {
    auto e = std::make_shared<Expr>();
    e->kind = E_LITERAL;
    e->lit.type = DType(T_INT64);
    e->lit.is_null = false;
    e->lit.i = v;
    return e;
}
ExprPtr lit_null(const DType& t) {
    auto e = std::make_shared<Expr>();
    e->kind = E_LITERAL;
    e->lit.type = t;
    e->lit.is_null = true;
    return e;
}

static int resolve_col(const Expr& e, const Schema& in) {
    if (e.index >= 0) {
        AURON_CHECK(e.index < (int)in.fields.size(), "bound reference out of range");
        return e.index;
    }
    int idx = in.index_of(e.name);
    if (idx < 0) {   // case-insensitive fallback (scan/mod.rs:56-100)
        for (size_t i = 0; i < in.fields.size(); i++) {
            if (in.fields[i].name.size() != e.name.size()) continue;
            bool eq = true;
            for (size_t k = 0; k < e.name.size(); k++) eq = eq && tolower(in.fields[i].name[k]) == tolower(e.name[k]);
            if (eq) return (int)i;
        }
        fail("column not found: " + e.name);
    }
    return idx;
}
bool is_plain_column(const Expr& e, const Schema& input, int* idx) {
    if (e.kind != E_COLUMN) return false;
    *idx = resolve_col(e, input);
    return true;
}

// Spark string constructors and digests (NativeConverters.scala:927-942,1033-1047): their result is a new utf8 value, which the
// VM builds only as a whole projection output (OP_SB_*) and digests only after the VM (k_digest.cu)
static bool is_string_builder(const std::string& f) {
    return f == "Spark_StringConcat" || f == "Spark_StringConcatWs" || f == "Spark_StringRepeat" || f == "Spark_StringSpace";
}
static int digest_alg_of(const std::string& f) {
    return f == "Spark_MD5" ? DIGEST_MD5 : f == "Spark_Sha224" ? DIGEST_SHA224 : f == "Spark_Sha256" ? DIGEST_SHA256 :
           f == "Spark_Sha384" ? DIGEST_SHA384 : f == "Spark_Sha512" ? DIGEST_SHA512 : 0;
}
// the string functions the builder runs as one piece (NativeConverters.scala:902-905,929-932,1053-1062): a whole projection
// expression, a piece of concat / concat_ws or a digest's argument
static int string_fn_of(const std::string& f) {
    return f == "Lpad" ? SBF_LPAD : f == "Rpad" ? SBF_RPAD : f == "Replace" ? SBF_REPLACE : f == "Translate" ? SBF_TRANSLATE :
           f == "Reverse" ? SBF_REVERSE : f == "Spark_InitCap" ? SBF_INITCAP : f == "Hex" ? SBF_HEX : f == "Chr" ? SBF_CHR : SBF_NONE;
}
bool makes_string_fn(const std::string& f) { return is_string_builder(f) || digest_alg_of(f) != 0 || string_fn_of(f) != SBF_NONE; }
static bool makes_string(const Expr& e) { return e.kind == E_SCALAR_FN && makes_string_fn(e.name); }
// the planner's declared-type TRY_CAST around one of them (operators.cc ProjectExec) is the identity: their type is utf8
static const Expr& strip_utf8_cast(const Expr& e) {
    if ((e.kind == E_CAST || e.kind == E_TRY_CAST) && e.type.id == T_UTF8 && makes_string(*e.children[0])) return *e.children[0];
    return e;
}
// CAST(x AS STRING) of the kinds fmt_value formats (-1: not one of them)
static int fmt_kind_of(const DType& st, int* scale) {
    *scale = 0;
    if (st.id == T_BOOL) return FMT_BOOL;
    if (st.is_integer()) return FMT_INT;
    if (st.id == T_DATE32) return FMT_DATE;
    if (st.id == T_DECIMAL128 && st.scale >= 0 && st.scale <= 38) {
        *scale = st.scale;
        return FMT_DEC;
    }
    if (st.id == T_FLOAT32) return FMT_F32;
    if (st.id == T_FLOAT64) return FMT_F64;
    return -1;
}

// the kinds fmt_value formats in vm_kernel<true, true> only
static bool needs_text(int kind, const DType& st) { return kind == FMT_F32 || kind == FMT_F64 || (kind == FMT_DEC && st.precision > 18); }

static bool is_cmp_op(const std::string& op) {
    return op == "Eq" || op == "NotEq" || op == "Lt" || op == "LtEq" || op == "Gt" || op == "GtEq" || op == "IsDistinctFrom" || op == "IsNotDistinctFrom";
}
// the common type both operands of a decimal comparison, sum or difference are rescaled to (the kernels work on unscaled values)
static DType dec_common_type(const DType& a, const DType& b) {
    const int sc = std::max(a.scale, b.scale);
    const int ip = std::max(a.precision - a.scale, b.precision - b.scale);
    return DType::decimal(std::min(38, ip + sc), sc);
}
// decimal result types as arrow declares them, capped at 38 digits: p1 + p2 + 1 digits at scale s1 + s2 for a product,
// max(p) + 1 digits at the common scale for a sum or difference; the kernel gives NULL for a result that does not fit
static DType dec_arith_type(const std::string& op, DType a, DType b) {
    if (op == "Multiply") return DType::decimal(std::min(38, a.precision + b.precision + 1), a.scale + b.scale);
    if (a.scale != b.scale) {
        const DType common = dec_common_type(a, b);
        if (a.scale != common.scale) a = common;
        if (b.scale != common.scale) b = common;
    }
    return DType::decimal(std::min(38, std::max(a.precision, b.precision) + 1), a.scale);
}

bool is_list_fn(const std::string& f) { return f == "Spark_StringSplit" || f == "Spark_MakeArray"; }

// a list value at this node: a list column, a list literal, split / array, or a cast to a list type (never resolves a column that
// does not exist: that error belongs to the compiler)
static bool is_list_value(const Expr& e, const Schema& in) {
    if (e.kind == E_COLUMN) {
        if (e.index >= 0) return e.index < (int)in.fields.size() && in.fields[(size_t)e.index].type.id == T_LIST;
        const int i = in.index_of(e.name);
        return i >= 0 && in.fields[(size_t)i].type.id == T_LIST;
    }
    if (e.kind == E_LITERAL || e.kind == E_CAST || e.kind == E_TRY_CAST) return (e.kind == E_LITERAL ? e.lit.type : e.type).id == T_LIST;
    return e.kind == E_SCALAR_FN && (is_list_fn(e.name) || e.type.id == T_LIST);
}
static std::string list_value_name(const Expr& e) {
    if (e.kind == E_COLUMN) return e.index >= 0 ? "list column #" + std::to_string(e.index) : "list column " + e.name;
    if (e.kind == E_LITERAL) return "list literal";
    if (e.kind == E_SCALAR_FN) return e.name;
    return e.kind == E_CAST ? "CAST to a list" : "TRY_CAST to a list";
}
static std::string node_name(const Expr& e) {
    switch (e.kind) {
        case E_SCALAR_FN: return e.name;
        case E_CASE: return "CASE";
        case E_CAST: return "CAST";
        case E_TRY_CAST: return "TRY_CAST";
        case E_BINARY: return e.op;
        case E_IN_LIST: return "IN";
        case E_LIKE: return "LIKE";
        case E_IS_NULL: return "IS NULL";
        case E_IS_NOT_NULL: return "IS NOT NULL";
        default: return "an expression";
    }
}
// the VM has no list registers: a list value anywhere in a program is a plan error that names it and where it was used
static void reject_list_values(const Expr& e, const Schema& in, const Expr* parent, const char* where) {
    if (is_list_value(e, in))
        fail(list_value_name(e) + (parent ? " inside " + node_name(*parent) : std::string(" as ") + where) +
             " is not supported: a list value may only be a whole projection expression or a generator's child");
    for (auto& c : e.children)
        if (c) reject_list_values(*c, in, &e, where);
}

void reject_list_exprs(const std::vector<ExprPtr>& exprs, const Schema& input, const char* where) {
    for (auto& e : exprs)
        if (e) reject_list_values(*e, input, nullptr, where);
}

DType infer_type(const Expr& e, const Schema& in) {
    switch (e.kind) {
        case E_COLUMN: return in.fields[resolve_col(e, in)].type;
        case E_LITERAL: return e.lit.type;
        case E_BINARY: {
            if (is_cmp_op(e.op) || e.op == "And" || e.op == "Or") return DType(T_BOOL);
            const DType a = infer_type(*e.children[0], in);
            if (a.id == T_DECIMAL128 && (e.op == "Plus" || e.op == "Minus" || e.op == "Multiply")) {
                const DType b = infer_type(*e.children[1], in);
                if (b.id == T_DECIMAL128) return dec_arith_type(e.op, a, b);
            }
            return a;
        }
        case E_NOT: case E_IS_NULL: case E_IS_NOT_NULL: case E_IN_LIST: case E_LIKE: case E_STARTS_WITH: case E_ENDS_WITH: case E_CONTAINS:
        case E_SC_AND: case E_SC_OR:
            return DType(T_BOOL);
        case E_ROW_NUM: return DType(T_INT64);
        case E_NEGATIVE: return infer_type(*e.children[0], in);
        case E_CASE: return infer_type(*e.children[e.has_case_expr ? 2 : 1], in);
        case E_CAST: case E_TRY_CAST: return e.type;
        case E_SCALAR_FN:
            if (makes_string(e)) return DType(T_UTF8);
            if (e.name == "Spark_StringSplit") return DType::list(DType(T_UTF8), true, e.type.id == T_LIST ? e.type.elem_name : "item");
            if (e.name == "Spark_MakeArray" && !e.children.empty())
                return DType::list(infer_type(*e.children[0], in), true, e.type.id == T_LIST ? e.type.elem_name : "item");
            if (e.type.id != T_NULL) return e.type;
            return infer_type(*e.children[0], in);
    }
    return DType();
}

struct Compiler {
    const Schema& in;
    VmProgramImpl& prog;
    bool used[VM_NREG] = {false};
    std::map<int, int> col_slot;
    // RowNum counts the rows a projection emits, so it is valid only where every emitted row evaluates it: in a projection,
    // outside the branches the reference evaluates on a subset of the rows (CASE results and later conditions, coalesce's later
    // arguments, the right operand of a short-circuit AND / OR)
    bool row_num_ok = false;
    int cond_depth = 0;

    Compiler(const Schema& s, VmProgramImpl& p) : in(s), prog(p) {}
    struct Val {
        int reg;
        DType type;
    };
    int alloc() {
        for (int r = 0; r < VM_NREG; r++)
            if (!used[r]) {
                used[r] = true;
                return r;
            }
        fail("expression too deep for the VM register file (16 live values)");
    }
    void release(int r) { used[r] = false; }
    void emit(Op op, int dst, int a = 0, int b = 0, int c = 0, int t = 0, int flags = 0, int aux = 0, int aux2 = 0) {
        Instr i;
        i.op = op;
        i.dst = (uint8_t)dst;
        i.a = (uint8_t)a;
        i.b = (uint8_t)b;
        i.c = (uint8_t)c;
        i.t = (uint8_t)t;
        i.flags = (uint8_t)flags;
        i.aux = aux;
        i.aux2 = aux2;
        prog.code.push_back(i);
        AURON_CHECK(prog.code.size() <= 1024, "expression program too long");
    }
    void note_type(const DType& t) {
        if (t.id == T_DECIMAL128 || t.is_varlen()) prog.need_hi = true;
    }
    int add_const(uint64_t lo, int64_t hi, bool valid) {
        ConstEntry c{lo, hi, valid ? 1 : 0, 0};
        prog.consts.push_back(c);
        return (int)prog.consts.size() - 1;
    }
    int add_pool_string(const std::string& s) {
        uint32_t start = (uint32_t)prog.pool.size();
        prog.pool += s;
        prog.need_hi = true;
        return add_const(((uint64_t)start << 32) | (uint32_t)s.size(), VM_POOL_BUF, true);
    }
    int slot_of(int col) {
        auto it = col_slot.find(col);
        if (it != col_slot.end()) return it->second;
        AURON_CHECK((int)prog.in_cols.size() < VM_MAX_COLS, "too many input columns in one expression program");
        int s = (int)prog.in_cols.size();
        prog.in_cols.push_back(col);
        col_slot[col] = s;
        return s;
    }
    Val literal(const Literal& l) {
        int r = alloc();
        note_type(l.type);
        int ci;
        if (l.is_null) ci = add_const(0, l.type.is_varlen() ? VM_POOL_BUF : 0, false);
        else if (l.type.is_varlen()) ci = add_pool_string(l.s);
        else if (l.type.id == T_DECIMAL128) ci = add_const(l.lo, l.hi, true);
        else if (l.type.id == T_FLOAT32) {
            float f = (float)l.d;
            uint32_t b;
            memcpy(&b, &f, 4);
            ci = add_const(b, 0, true);
        } else if (l.type.id == T_FLOAT64) {
            uint64_t b;
            memcpy(&b, &l.d, 8);
            ci = add_const(b, 0, true);
        } else if (l.type.id == T_NULL) {
            ci = add_const(0, 0, false);
        } else ci = add_const((uint64_t)l.i, 0, true);
        emit(OP_CONST, r, 0, 0, 0, 0, 0, ci);
        return {r, l.type};
    }
    // explicit: a CAST / TRY_CAST of the plan, not a coercion the compiler inserts (only those parse text into floats / bools)
    Val cast_to(Val v, const DType& to, bool explicit_cast = false) {
        if (v.type == to) return v;
        if (v.type.id == T_NULL) {   // typed NULL
            emit(OP_CONST, v.reg, 0, 0, 0, 0, 0, add_const(0, to.is_varlen() ? VM_POOL_BUF : 0, false));
            note_type(to);
            return {v.reg, to};
        }
        Vt st = vt_of(v.type), dt = vt_of(to);
        note_type(to);
        bool date_target = to.id == T_DATE32;
        bool ok = false;
        if (st <= VT_I64 && dt != VT_STR) ok = true;
        if ((st == VT_F32 || st == VT_F64) && dt != VT_STR) ok = true;
        if (st == VT_DEC && dt != VT_STR && dt != VT_BOOL) ok = true;
        if (st == VT_STR && ((dt >= VT_I8 && dt <= VT_I64 && to.is_integer()) || date_target || dt == VT_DEC)) ok = true;
        if (explicit_cast && v.type.id == T_UTF8 && (dt == VT_F32 || dt == VT_F64 || dt == VT_BOOL)) {   // Spark's parsers (float_text.cuh, str_to_bool)
            ok = true;
            prog.need_hi = prog.need_text = true;   // they run in vm_kernel<true, true> only
        }
        if (st == VT_STR && dt == VT_STR) return {v.reg, to};
        // same physical representation (date32 <-> int32 etc.) are not native casts in the reference
        if ((v.type.id == T_DATE32 || to.id == T_DATE32 || v.type.id == T_TIMESTAMP || to.id == T_TIMESTAMP || v.type.id == T_DATE64 || to.id == T_DATE64) &&
            !(st == VT_STR && date_target))
            ok = false;
        if (!ok) fail("unsupported CAST " + v.type.str() + " -> " + to.str() + " on device");
        int dprec = to.id == T_DECIMAL128 ? to.precision : (date_target && st == VT_STR ? -1 : 0);
        int dscale = to.id == T_DECIMAL128 ? to.scale : 0;
        int sscale = v.type.id == T_DECIMAL128 ? v.type.scale : 0;
        emit(OP_CAST, v.reg, v.reg, 0, 0, st, 0, (int)dt | (sscale << 8), ((dprec & 0xff) << 8) | (dscale & 0xff));
        return {v.reg, to};
    }
    Val binary_cmp_or_arith(const Expr& e) {
        Val a = gen(*e.children[0]);
        Val b = gen(*e.children[1]);
        const std::string& op = e.op;
        // harmonise integer widths / NULL literals (Spark inserts casts, this is belt and braces)
        if (a.type != b.type) {
            if (a.type.id == T_NULL) a = cast_to(a, b.type);
            else if (b.type.id == T_NULL) b = cast_to(b, a.type);
            else if (a.type.is_integer() && b.type.is_integer()) {
                if (a.type.width() < b.type.width()) a = cast_to(a, b.type);
                else b = cast_to(b, a.type);
            } else if (a.type.id == T_DECIMAL128 && b.type.id == T_DECIMAL128) {
                // the kernels compare / add the unscaled i128 values: both operands must carry the same scale (arrow-rs rescales,
                // Spark inserts the casts itself; 1.00@2 vs 1.0000@4 must not compare 100 with 10000)
                // (a product needs no common scale: its unscaled value is the product of the operands' at scale s1 + s2)
                if (a.type.scale != b.type.scale && op != "Multiply") {
                    const DType common = dec_common_type(a.type, b.type);
                    if (a.type.scale != common.scale) a = cast_to(a, common);
                    if (b.type.scale != common.scale) b = cast_to(b, common);
                }
            } else if (a.type.id == T_TIMESTAMP && b.type.id == T_TIMESTAMP) {
                AURON_CHECK(a.type.unit == b.type.unit, "binary operator " + op + " on timestamps of different units");
            } else if (vt_of(a.type) == vt_of(b.type) && a.type.id != T_DECIMAL128 && a.type.id != T_TIMESTAMP) {
            } else fail("binary operator " + op + " on mismatched types " + a.type.str() + " / " + b.type.str());
        }
        Vt t = vt_of(a.type);
        note_type(a.type);
        if (op == "And" || op == "Or") {
            emit(op == "And" ? OP_AND : OP_OR, a.reg, a.reg, b.reg);
            release(b.reg);
            return {a.reg, DType(T_BOOL)};
        }
        if (is_cmp_op(op)) {
            Op o = op == "Eq" ? OP_EQ : op == "NotEq" ? OP_NE : op == "Lt" ? OP_LT : op == "LtEq" ? OP_LE : op == "Gt" ? OP_GT : op == "GtEq" ? OP_GE : OP_NSEQ;
            emit(o, a.reg, a.reg, b.reg, 0, t);
            if (op == "IsDistinctFrom") emit(OP_NOT, a.reg, a.reg);
            release(b.reg);
            return {a.reg, DType(T_BOOL)};
        }
        Op o;
        if (op == "Plus") o = OP_ADD;
        else if (op == "Minus") o = OP_SUB;
        else if (op == "Multiply") o = OP_MUL;
        else if (op == "Divide") o = OP_DIV;
        else if (op == "Modulo") o = OP_MOD;
        else if (op == "BitwiseAnd") o = OP_BITAND;
        else if (op == "BitwiseOr") o = OP_BITOR;
        else if (op == "BitwiseXor") o = OP_BITXOR;
        else if (op == "BitwiseShiftLeft") o = OP_SHL;
        else if (op == "BitwiseShiftRight") o = OP_SHR;
        else fail("unsupported binary operator " + op);
        if (t == VT_STR || t == VT_BOOL) fail("arithmetic on " + a.type.str());
        if (t == VT_DEC && (o == OP_DIV || o == OP_MOD || o > OP_MOD))
            fail("decimal " + op + " is not native (auron.decimal.arithOp.enabled=false in the reference)");
        const DType rt = t == VT_DEC ? dec_arith_type(op, a.type, b.type) : a.type;
        emit(o, a.reg, a.reg, b.reg, 0, t, 0, t == VT_DEC ? rt.precision : 0);
        release(b.reg);
        return {a.reg, rt};
    }
    Val scalar_fn(const Expr& e) {
        const std::string& f = e.name;
        auto unary_f64 = [&](int m) {
            Val a = cast_to(gen(*e.children[0]), DType(T_FLOAT64));
            emit(OP_MATH1, a.reg, a.reg, 0, 0, VT_F64, 0, m);
            return Val{a.reg, DType(T_FLOAT64)};
        };
        // the session time zone as a utf8 literal (spark_dates.rs:93-102) into the pool; a NULL literal, a non-literal or a name
        // chrono-tz would not parse means "no zone" (-1)
        auto zone_table_of = [&](const Expr& z) -> int {
            if (z.kind != E_LITERAL || z.lit.is_null || !z.lit.type.is_varlen()) return -1;
            TzTable tab;
            if (!load_tz_table(z.lit.s, &tab)) return -1;
            while (prog.pool.size() % 8) prog.pool.push_back('\0');
            const int at = (int)prog.pool.size();
            const int64_t n = (int64_t)tab.trans.size();
            prog.pool.append((const char*)&n, 8);
            prog.pool.append((const char*)tab.trans.data(), (size_t)n * 8);
            prog.pool.append((const char*)tab.offs.data(), (size_t)(n + 1) * 4);
            while (prog.pool.size() % 8) prog.pool.push_back('\0');
            return at;
        };
        auto zone_table = [&](bool* named, std::string* name) -> int {   // the optional second argument
            *named = false;
            if (e.children.size() < 2) return -1;
            const Expr& z = *e.children[1];
            if (z.kind != E_LITERAL || z.lit.is_null || !z.lit.type.is_varlen()) return -1;
            *named = true;
            *name = z.lit.s;
            return zone_table_of(z);
        };
        auto unit_of = [&](const DType& t) -> int {
            if (t.id == T_DATE32) return 4;
            if (t.id == T_TIMESTAMP) return t.unit;
            if (t.id == T_DATE64) return 1;
            fail(f + " needs a date or timestamp argument, got " + t.str());
            return 0;
        };
        // resolve_local_date32 (spark_dates.rs:231-254): with a zone the argument is cast to Timestamp(ms) and localized; without
        // one it is cast to Date32
        auto local_days = [&](Val a, int tz_at) {
            const int unit = unit_of(a.type);
            if (tz_at >= 0) {
                emit(OP_TS_LOCAL_MS, a.reg, a.reg, 0, 0, VT_I64, 0, tz_at, unit);
                emit(OP_MS_TO_DAYS, a.reg, a.reg, 0, 0, VT_I32, 0, 0);
            } else if (unit != 4) {
                emit(OP_TS_LOCAL_MS, a.reg, a.reg, 0, 0, VT_I64, 0, -1, unit);
                emit(OP_MS_TO_DAYS, a.reg, a.reg, 0, 0, VT_I32, 0, 1);
            }
            return a;
        };
        auto date_fn = [&](int part) {
            Val a = gen(*e.children[0]);
            bool named;
            std::string zname;
            int tz_at = zone_table(&named, &zname);
            if (part == DP_WEEK) {
                // spark_weekofyear (spark_dates.rs:36-91): an unknown zone is an error; only Timestamp(Millisecond) input is
                // localized (default zone UTC), every other type goes through the plain cast to Date32
                if (named && tz_at < 0) fail("spark_weekofyear invalid timezone: " + zname);
                if (!(a.type.id == T_TIMESTAMP && a.type.unit == 1)) tz_at = -1;
                else if (tz_at < 0) {
                    emit(OP_TS_LOCAL_MS, a.reg, a.reg, 0, 0, VT_I64, 0, -1, 1);
                    emit(OP_MS_TO_DAYS, a.reg, a.reg, 0, 0, VT_I32, 0, 0);   // UTC calendar date of the instant (floor)
                    emit(OP_DATEPART, a.reg, a.reg, 0, 0, VT_I32, 0, part);
                    return Val{a.reg, DType(T_INT32)};
                }
            }
            a = local_days(a, tz_at);
            emit(OP_DATEPART, a.reg, a.reg, 0, 0, VT_I32, 0, part);
            return Val{a.reg, DType(T_INT32)};
        };
        // spark_hour / spark_minute / spark_second (spark_dates.rs:347-399)
        auto time_fn = [&](int which) {
            Val a = gen(*e.children[0]);
            bool named;
            std::string zname;
            const int tz_at = zone_table(&named, &zname);
            emit(OP_TS_LOCAL_MS, a.reg, a.reg, 0, 0, VT_I64, 0, tz_at, unit_of(a.type));
            emit(OP_TIMEPART, a.reg, a.reg, 0, 0, VT_I32, 0, which);
            return Val{a.reg, DType(T_INT32)};
        };
        if (string_fn_of(f) != SBF_NONE)
            fail(f + " is only native as a whole projection expression, a piece of concat / concat_ws or the argument of md5 / sha2");
        if (makes_string(e)) fail(f + " is only native as a whole projection expression or as the argument of md5 / sha2");
        // a utf8 argument of a string function (a NULL literal gives NULL)
        auto text_arg = [&](const Expr& x) {
            Val v = gen(x);
            if (v.type.id != T_UTF8 && v.type.id != T_NULL) fail(f + " argument of type " + v.type.str() + " is not native (utf8 only)");
            return v;
        };
        Val r{-1, DType()};
        if (f == "Spark_Year") r = date_fn(DP_YEAR);
        else if (f == "Spark_Month") r = date_fn(DP_MONTH);
        else if (f == "Spark_Day") r = date_fn(DP_DAY);
        else if (f == "Spark_DayOfWeek") r = date_fn(DP_DOW);
        else if (f == "Spark_WeekOfYear") r = date_fn(DP_WEEK);
        else if (f == "Spark_Quarter") r = date_fn(DP_QUARTER);
        else if (f == "Spark_Hour") r = time_fn(0);
        else if (f == "Spark_Minute") r = time_fn(1);
        else if (f == "Spark_Second") r = time_fn(2);
        else if (f == "DatePart") {   // date_part('part', date)
            AURON_CHECK(e.children.size() == 2 && e.children[0]->kind == E_LITERAL, "date_part needs a literal part");
            std::string part = e.children[0]->lit.s;
            for (auto& ch : part) ch = (char)tolower(ch);
            int dp = part == "year" ? DP_YEAR : part == "month" ? DP_MONTH : part == "day" ? DP_DAY : part == "quarter" ? DP_QUARTER :
                     part == "week" ? DP_WEEK : part == "doy" ? DP_DOY : (part == "dow" ? 100 : -1);
            if (dp < 0) fail("date_part('" + part + "') is not native");
            Val a = gen(*e.children[1]);
            if (a.type.id != T_DATE32) fail("date_part is only native for Date32 input");
            if (dp == 100) {   // datafusion dow: Sunday = 0
                emit(OP_DATEPART, a.reg, a.reg, 0, 0, VT_I32, 0, DP_DOW);
                Val one = literal(Literal{DType(T_INT32), false, 1});
                emit(OP_SUB, a.reg, a.reg, one.reg, 0, VT_I32);
                release(one.reg);
            } else emit(OP_DATEPART, a.reg, a.reg, 0, 0, VT_I32, 0, dp);
            r = Val{a.reg, DType(T_INT32)};
        } else if (f == "Spark_NullIfZero") {
            Val a = gen(*e.children[0]);
            note_type(a.type);
            emit(OP_NULLIFZERO, a.reg, a.reg, 0, 0, vt_of(a.type));
            r = a;
        } else if (f == "Spark_NullIf" || f == "NullIf") {
            Val a = gen(*e.children[0]);
            Val b = cast_to(gen(*e.children[1]), a.type);
            int c = alloc();
            emit(OP_EQ, c, a.reg, b.reg, 0, vt_of(a.type));
            emit(OP_CONST, b.reg, 0, 0, 0, 0, 0, add_const(0, a.type.is_varlen() ? VM_POOL_BUF : 0, false));
            emit(OP_SELECT, a.reg, c, b.reg, a.reg);
            release(b.reg);
            release(c);
            r = a;
        } else if (f == "Spark_IsNaN" || f == "IsNaN") {
            Val a = gen(*e.children[0]);
            if (!a.type.is_float()) fail("isnan on non-float");
            emit(OP_ISNAN, a.reg, a.reg, 0, 0, vt_of(a.type));
            r = Val{a.reg, DType(T_BOOL)};
        } else if (f == "Spark_NormalizeNanAndZero") {
            Val a = gen(*e.children[0]);
            if (a.type.is_float()) emit(OP_NORMNAN, a.reg, a.reg, 0, 0, vt_of(a.type));
            r = a;
        } else if (f == "Spark_UnscaledValue") {
            Val a = gen(*e.children[0]);
            emit(OP_UNSCALED, a.reg, a.reg);
            r = Val{a.reg, DType(T_INT64)};
        } else if (f == "Spark_MakeDecimal") {
            Val a = cast_to(gen(*e.children[0]), DType(T_INT64));
            AURON_CHECK(e.type.id == T_DECIMAL128, "MakeDecimal needs a decimal return type");
            note_type(e.type);
            emit(OP_MAKE_DECIMAL, a.reg, a.reg, 0, 0, VT_I64, 0, e.type.precision);
            r = Val{a.reg, e.type};
        } else if (f == "Spark_Round" || f == "Spark_BRound") {
            // spark_round.rs:38-134: the scale is a literal integer; decimals keep their type, integers and floats theirs
            AURON_CHECK(e.children.size() == 2 && e.children[1]->kind == E_LITERAL && !e.children[1]->lit.is_null &&
                            (e.children[1]->lit.type.id == T_INT32 || e.children[1]->lit.type.id == T_INT64),
                        "spark_round() / spark_bround() scale must be a literal integer");
            const int sc = (int)e.children[1]->lit.i;
            Val a = gen(*e.children[0]);
            const Vt vt = vt_of(a.type);
            if (!(vt == VT_DEC || vt == VT_F32 || vt == VT_F64 || vt == VT_I16 || vt == VT_I32 || vt == VT_I64) || a.type.id == T_DATE32 ||
                a.type.id == T_DATE64 || a.type.id == T_TIMESTAMP)
                fail("spark_round() on " + a.type.str() + " is not native");
            emit(OP_ROUND, a.reg, a.reg, 0, 0, vt, f == "Spark_BRound" ? 1 : 0, sc, a.type.id == T_DECIMAL128 ? a.type.scale : 0);
            r = Val{a.reg, a.type};
        } else if (f == "Spark_CheckOverflow") {
            Val a = gen(*e.children[0]);
            AURON_CHECK(a.type.id == T_DECIMAL128 && e.type.id == T_DECIMAL128, "CheckOverflow needs decimals");
            emit(OP_CHECK_OVERFLOW, a.reg, a.reg, 0, 0, VT_DEC, 0, (a.type.scale << 8), ((e.type.precision & 0xff) << 8) | (e.type.scale & 0xff));
            r = Val{a.reg, e.type};
        } else if (f == "Spark_Murmur3Hash" || f == "Spark_XxHash64") {
            bool mm = f == "Spark_Murmur3Hash";
            Val acc = literal(Literal{DType(mm ? T_INT32 : T_INT64), false, 42});
            for (auto& ch : e.children) {
                Val a = gen(*ch);
                note_type(a.type);
                emit(OP_HASH, acc.reg, a.reg, 0, 0, vt_of(a.type), mm ? 0 : 1);
                release(a.reg);
            }
            r = Val{acc.reg, DType(mm ? T_INT32 : T_INT64)};
        } else if (f == "Substr") {
            Val s = gen(*e.children[0]);
            Val pos = cast_to(gen(*e.children[1]), DType(T_INT64));
            int creg = 0xff;
            Val cnt{-1, DType()};
            if (e.children.size() > 2) {
                cnt = cast_to(gen(*e.children[2]), DType(T_INT64));
                creg = cnt.reg;
            }
            note_type(s.type);
            emit(OP_SUBSTR, s.reg, s.reg, pos.reg, creg);
            release(pos.reg);
            if (cnt.reg >= 0) release(cnt.reg);
            r = s;
        } else if (f == "CharacterLength" || f == "OctetLength") {
            Val s = gen(*e.children[0]);
            emit(f == "CharacterLength" ? OP_CHARLEN : OP_OCTLEN, s.reg, s.reg);
            r = Val{s.reg, DType(T_INT32)};
        } else if (f == "Ascii" || f == "FindInSet") {   // int32: the first code point / the index of a in the list b
            Val s = text_arg(*e.children[0]);
            if (f == "Ascii") emit(OP_CHARLEN, s.reg, s.reg, 0, 0, VT_STR, CL_ASCII);
            else {
                AURON_CHECK(e.children.size() == 2, f + " takes two arguments");
                Val l = text_arg(*e.children[1]);
                emit(OP_CHARLEN, s.reg, s.reg, l.reg, 0, VT_STR, CL_FIND_IN_SET);
                release(l.reg);
            }
            r = Val{s.reg, DType(T_INT32)};
        } else if (f == "BitLength") {   // int32: 8 x the byte length of a utf8 or binary value
            Val s = gen(*e.children[0]);
            if (!s.type.is_varlen() && s.type.id != T_NULL) fail(f + " argument of type " + s.type.str() + " is not native (utf8 or binary only)");
            emit(OP_OCTLEN, s.reg, s.reg);
            Val eight = literal(Literal{DType(T_INT32), false, 8});
            emit(OP_MUL, s.reg, s.reg, eight.reg, 0, VT_I32);
            release(eight.reg);
            r = Val{s.reg, DType(T_INT32)};
        } else if (f == "Trim" || f == "Btrim" || f == "Ltrim" || f == "Rtrim") {
            AURON_CHECK(e.children.size() == 1 || e.children.size() == 2, f + " takes one or two arguments");
            const int sides = f == "Ltrim" ? 1 : f == "Rtrim" ? 2 : 3;
            Val s = gen(*e.children[0]);
            if (e.children.size() == 1) emit(OP_TRIM, s.reg, s.reg, 0, 0, VT_STR, sides);
            else {   // the characters of the second argument
                Val set = text_arg(*e.children[1]);
                emit(OP_TRIM, s.reg, s.reg, set.reg, 0, VT_STR, sides | TRIM_SET);
                release(set.reg);
            }
            r = s;
        } else if (f == "Upper" || f == "Lower" || f == "Spark_StringUpper" || f == "Spark_StringLower") {
            Val s = gen(*e.children[0]);
            emit(OP_CASEXF, s.reg, s.reg, 0, 0, VT_STR, (f == "Upper" || f == "Spark_StringUpper") ? 1 : 2);
            r = s;
        } else if (f == "StartsWith") {
            AURON_CHECK(e.children[1]->kind == E_LITERAL, "starts_with needs a literal prefix");
            Val s = gen(*e.children[0]);
            emit(OP_STARTS, s.reg, s.reg, 0, 0, VT_STR, 0, add_pool_string(e.children[1]->lit.s));
            r = Val{s.reg, DType(T_BOOL)};
        } else if (f == "Abs") {
            Val a = gen(*e.children[0]);
            note_type(a.type);
            emit(OP_ABS, a.reg, a.reg, 0, 0, vt_of(a.type));
            r = a;
        } else if (f == "Coalesce" || f == "Nvl") {
            Val a = gen(*e.children[0]);
            cond_depth++;
            for (size_t k = 1; k < e.children.size(); k++) {
                Val b = cast_to(gen(*e.children[k]), a.type);
                emit(OP_COALESCE, a.reg, a.reg, b.reg);
                release(b.reg);
            }
            cond_depth--;
            r = a;
        } else if (f == "Greatest" || f == "Least") {
            // 2..N arguments of one type, NULLs skipped, the VM's comparison order, the earlier argument on ties; one running value
            // and one argument live at a time
            if (e.children.size() < 2) fail(f + " takes at least two arguments");
            DType rt(T_NULL);
            for (auto& ch : e.children)
                if (rt.id == T_NULL) rt = infer_type(*ch, in);
            if (rt.id == T_NULL) rt = e.type;
            Val acc{-1, DType()};
            for (auto& ch : e.children) {
                Val b = gen(*ch);
                if (b.type.id == T_NULL) b = cast_to(b, rt);
                if (b.type != rt) fail(f + " needs arguments of one type, got " + rt.str() + " and " + b.type.str());
                if (acc.reg < 0) {
                    acc = b;
                    continue;
                }
                note_type(rt);
                emit(OP_GREATEST, acc.reg, acc.reg, b.reg, 0, vt_of(rt), f == "Least" ? 1 : 0);
                release(b.reg);
            }
            r = acc;
        } else if (f == "Nvl2") {   // b when a is not NULL, else c
            if (e.children.size() != 3) fail(f + " takes three arguments");
            DType rt = infer_type(*e.children[1], in);
            if (rt.id == T_NULL) rt = infer_type(*e.children[2], in);
            if (rt.id == T_NULL) rt = e.type;
            Val a = gen(*e.children[0]);
            emit(OP_ISNOTNULL, a.reg, a.reg);
            Val b = cast_to(gen(*e.children[1]), rt);
            Val c = cast_to(gen(*e.children[2]), rt);
            note_type(rt);
            emit(OP_SELECT, a.reg, a.reg, b.reg, c.reg);
            release(b.reg);
            release(c.reg);
            r = Val{a.reg, rt};
        } else if (f == "DateTrunc") {   // date_trunc('level', ts): the wall clock of the value as UTC, toward -inf
            if (e.children.size() != 2) fail("date_trunc takes two arguments");
            const Expr& fe = *e.children[0];
            if (fe.kind != E_LITERAL) fail("date_trunc needs a literal format");
            Val a = gen(*e.children[1]);
            if (a.type.id != T_TIMESTAMP) fail("date_trunc needs a timestamp argument, got " + a.type.str());
            const DType rt = e.type.id == T_TIMESTAMP ? e.type : a.type;
            std::string lv = fe.lit.is_null || !fe.lit.type.is_varlen() ? "" : fe.lit.s;
            for (auto& ch : lv) ch = (char)toupper(ch);
            const int level = lv == "YEAR" || lv == "YYYY" || lv == "YY" ? TL_YEAR : lv == "QUARTER" ? TL_QUARTER :
                              lv == "MONTH" || lv == "MON" || lv == "MM" ? TL_MONTH : lv == "WEEK" ? TL_WEEK : lv == "DAY" || lv == "DD" ? TL_DAY :
                              lv == "HOUR" ? TL_HOUR : lv == "MINUTE" ? TL_MINUTE : lv == "SECOND" ? TL_SECOND : lv == "MILLISECOND" ? TL_MILLISECOND :
                              lv == "MICROSECOND" ? TL_MICROSECOND : -1;
            if (level < 0) emit(OP_CONST, a.reg, 0, 0, 0, 0, 0, add_const(0, 0, false));   // an unknown or NULL format gives NULL
            else {
                prog.need_hi = true;
                emit(OP_DATE_TRUNC, a.reg, a.reg, 0, 0, VT_I64, 0, level, a.type.unit | (rt.unit << 4));
            }
            r = Val{a.reg, rt};
        } else if (f == "MakeDate") {
            if (e.children.size() != 3) fail("make_date takes three arguments");
            Val y = cast_to(gen(*e.children[0]), DType(T_INT32));
            Val m = cast_to(gen(*e.children[1]), DType(T_INT32));
            Val d = cast_to(gen(*e.children[2]), DType(T_INT32));
            prog.need_hi = true;
            emit(OP_MAKE_DATE, y.reg, y.reg, m.reg, d.reg, VT_I32);
            release(m.reg);
            release(d.reg);
            r = Val{y.reg, DType(T_DATE32)};
        } else if (f == "Factorial") {
            Val a = gen(*e.children[0]);
            if (a.type.id != T_INT32 && a.type.id != T_NULL) fail("factorial needs an int32 argument, got " + a.type.str());
            a = cast_to(a, DType(T_INT32));
            emit(OP_FACTORIAL, a.reg, a.reg, 0, 0, VT_I64);
            r = Val{a.reg, DType(T_INT64)};
        } else if (f == "Spark_MonthsBetween") {
            // spark_months_between (spark_dates.rs:403-458): both timestamps cast to Timestamp(ms), roundOff to bool, the zone a
            // utf8 literal (NULL or unknown: UTC)
            if (e.children.size() != 4) fail("spark_months_between() requires four arguments");
            const int tz_at = zone_table_of(*e.children[3]);
            Val a = gen(*e.children[0]);
            emit(OP_TS_LOCAL_MS, a.reg, a.reg, 0, 0, VT_I64, 0, -1, unit_of(a.type));
            Val b = gen(*e.children[1]);
            emit(OP_TS_LOCAL_MS, b.reg, b.reg, 0, 0, VT_I64, 0, -1, unit_of(b.type));
            Val c = cast_to(gen(*e.children[2]), DType(T_BOOL));
            prog.need_hi = true;
            emit(OP_MONTHS_BETWEEN, a.reg, a.reg, b.reg, c.reg, VT_F64, 0, tz_at);
            release(b.reg);
            release(c.reg);
            r = Val{a.reg, DType(T_FLOAT64)};
        } else if (f == "Power") {
            Val a = cast_to(gen(*e.children[0]), DType(T_FLOAT64));
            Val b = cast_to(gen(*e.children[1]), DType(T_FLOAT64));
            emit(OP_POW, a.reg, a.reg, b.reg);
            release(b.reg);
            r = Val{a.reg, DType(T_FLOAT64)};
        } else if (f == "Sqrt") r = unary_f64(M_SQRT);
        else if (f == "Exp") r = unary_f64(M_EXP);
        else if (f == "Ln") r = unary_f64(M_LN);
        else if (f == "Log10") r = unary_f64(M_LOG10);
        else if (f == "Log2") r = unary_f64(M_LOG2);
        else if (f == "Sin") r = unary_f64(M_SIN);
        else if (f == "Cos") r = unary_f64(M_COS);
        else if (f == "Tan") r = unary_f64(M_TAN);
        else if (f == "Asin") r = unary_f64(M_ASIN);
        else if (f == "Acos") r = unary_f64(M_ACOS);
        else if (f == "Atan") r = unary_f64(M_ATAN);
        else if (f == "Ceil") r = unary_f64(M_CEIL);
        else if (f == "Floor") r = unary_f64(M_FLOOR);
        else if (f == "Signum") r = unary_f64(M_SIGNUM);
        else if (f == "Trunc") r = unary_f64(M_TRUNC);
        else if (f == "Expm1") r = unary_f64(M_EXPM1);
        else if (f == "Acosh") r = unary_f64(M_ACOSH);
        else fail("scalar function " + f + " is not native on device");
        if (e.type.id != T_NULL && r.type != e.type) r = cast_to(r, e.type);
        return r;
    }
    Val gen(const Expr& e) {
        switch (e.kind) {
            case E_COLUMN: {
                int c = resolve_col(e, in);
                const DType& t = in.fields[c].type;
                int r = alloc();
                if (t.id == T_NULL) {
                    emit(OP_CONST, r, 0, 0, 0, 0, 0, add_const(0, 0, false));
                    return {r, t};
                }
                note_type(t);
                emit(OP_LOAD, r, 0, 0, 0, vt_of(t), 0, slot_of(c));
                return {r, t};
            }
            case E_LITERAL: return literal(e.lit);
            case E_BINARY: return binary_cmp_or_arith(e);
            case E_SC_AND: case E_SC_OR: {
                Val a = gen(*e.children[0]);
                cond_depth++;
                Val b = gen(*e.children[1]);
                cond_depth--;
                emit(e.kind == E_SC_AND ? OP_AND : OP_OR, a.reg, a.reg, b.reg);
                release(b.reg);
                return {a.reg, DType(T_BOOL)};
            }
            case E_NOT: {
                Val a = gen(*e.children[0]);
                emit(OP_NOT, a.reg, a.reg);
                return {a.reg, DType(T_BOOL)};
            }
            case E_IS_NULL: case E_IS_NOT_NULL: {
                Val a = gen(*e.children[0]);
                emit(e.kind == E_IS_NULL ? OP_ISNULL : OP_ISNOTNULL, a.reg, a.reg);
                return {a.reg, DType(T_BOOL)};
            }
            case E_NEGATIVE: {
                Val a = gen(*e.children[0]);
                note_type(a.type);
                emit(OP_NEG, a.reg, a.reg, 0, 0, vt_of(a.type));
                return a;
            }
            case E_CAST: case E_TRY_CAST: return cast_to(gen(*e.children[0]), e.type, true);
            case E_IN_LIST: {
                Val x = gen(*e.children[0]);
                note_type(x.type);
                int acc = alloc();
                emit(OP_CONST, acc, 0, 0, 0, 0, 0, add_const(0, 0, true));   // false
                for (size_t k = 1; k < e.children.size(); k++) {
                    Val v = cast_to(gen(*e.children[k]), x.type);
                    emit(OP_EQ, v.reg, x.reg, v.reg, 0, vt_of(x.type));
                    emit(OP_OR, acc, acc, v.reg);
                    release(v.reg);
                }
                if (e.negated) emit(OP_NOT, acc, acc);
                release(x.reg);
                return {acc, DType(T_BOOL)};
            }
            case E_CASE: {
                size_t k = 0;
                Val base{-1, DType()};
                if (e.has_case_expr) base = gen(*e.children[k++]);
                size_t n_pairs = (e.children.size() - k - (e.has_else ? 1 : 0)) / 2;
                DType rt = infer_type(*e.children[k + 1], in);
                if (rt.id == T_NULL && e.has_else) rt = infer_type(*e.children.back(), in);
                // evaluate from the last branch backwards: acc = else ; acc = cond_i ? then_i : acc
                cond_depth++;
                Val acc = e.has_else ? cast_to(gen(*e.children.back()), rt) : literal(Literal{rt, true});
                if (acc.type.id == T_NULL) acc.type = rt;
                note_type(rt);
                for (size_t pi = n_pairs; pi-- > 0;) {
                    const Expr& w = *e.children[k + 2 * pi];
                    const Expr& th = *e.children[k + 2 * pi + 1];
                    if (pi == 0) cond_depth--;   // the first condition sees every row
                    Val cond = gen(w);
                    if (pi == 0) cond_depth++;
                    if (e.has_case_expr) {
                        cond = cast_to(cond, base.type);
                        emit(OP_EQ, cond.reg, base.reg, cond.reg, 0, vt_of(base.type));
                    }
                    Val tv = cast_to(gen(th), rt);
                    emit(OP_SELECT, acc.reg, cond.reg, tv.reg, acc.reg);
                    release(cond.reg);
                    release(tv.reg);
                }
                cond_depth--;
                if (base.reg >= 0) release(base.reg);
                return {acc.reg, rt};
            }
            case E_LIKE: {
                AURON_CHECK(e.children[1]->kind == E_LITERAL && !e.children[1]->lit.is_null, "LIKE needs a literal pattern");
                Val s = gen(*e.children[0]);
                emit(OP_LIKE, s.reg, s.reg, 0, 0, VT_STR, (e.negated ? 1 : 0) | (e.case_insensitive ? 2 : 0), add_pool_string(e.children[1]->lit.s));
                return {s.reg, DType(T_BOOL)};
            }
            case E_STARTS_WITH: case E_ENDS_WITH: case E_CONTAINS: {
                Val s = gen(*e.children[0]);
                if (!s.type.is_varlen()) fail("string predicate on non-string");
                Op o = e.kind == E_STARTS_WITH ? OP_STARTS : e.kind == E_ENDS_WITH ? OP_ENDS : OP_CONTAINS;
                emit(o, s.reg, s.reg, 0, 0, VT_STR, 0, add_pool_string(e.lit.s));
                return {s.reg, DType(T_BOOL)};
            }
            case E_SCALAR_FN: return scalar_fn(e);
            case E_ROW_NUM: {
                if (!row_num_ok) fail("RowNum is only native in a projection");
                if (cond_depth > 0) fail("RowNum is not native inside a conditional branch (CASE, coalesce, short-circuit AND / OR)");
                const int r = alloc();
                emit(OP_ROWNUM, r, 0, 0, 0, VT_I64);
                return {r, DType(T_INT64)};
            }
        }
        fail("unsupported expression kind");
    }

    // one piece of a string constructor: a utf8 value (view), a formatted CAST to utf8, `times` copies of a view, or spaces
    void append_piece(const std::string& f, int b, int o, const Expr& x0, int flags, int const_idx = 0) {
        const Expr& x = strip_utf8_cast(x0);
        if (x.kind == E_SCALAR_FN && string_fn_of(x.name) != SBF_NONE && !(flags & (SB_REPEAT | SB_SPACE))) {
            append_fn_piece(x, b, o, flags, const_idx);
            return;
        }
        if ((flags & 3) == SB_SPACE) {   // space(n): n is an int32 value, never text
            const DType nt = infer_type(x, in);
            if (nt.id != T_INT32 && nt.id != T_NULL) fail(f + " needs an int32 argument, got " + nt.str());
            Val v = gen(x);
            if (v.type.id != T_INT32 && v.type.id != T_NULL) fail(f + " needs an int32 argument, got " + v.type.str());
            emit(OP_SB_APPEND, b, v.reg, 0, 0, VT_I32, flags, o);
            release(v.reg);
            return;
        }
        int scale = 0, kind = -1;
        if ((x.kind == E_CAST || x.kind == E_TRY_CAST) && x.type.id == T_UTF8) {
            const DType st = infer_type(*x.children[0], in);
            kind = fmt_kind_of(st, &scale);
            if (kind == FMT_F32 || kind == FMT_F64) kind = -1;   // float pieces are not built yet
            if (kind < 0 && st.id != T_UTF8 && st.id != T_NULL) fail(f + ": CAST " + st.str() + " -> utf8 is not native on device");
        }
        Val v = kind >= 0 ? gen(*x.children[0]) : gen(x);
        if (kind >= 0) {
            note_type(v.type);
            if (needs_text(kind, v.type)) prog.need_text = true;
            emit(OP_SB_APPEND, b, v.reg, 0, 0, vt_of(v.type), SB_FMT | flags, o | (const_idx << 8), (kind << 8) | scale);
        } else {
            if (v.type.id != T_UTF8 && v.type.id != T_NULL) fail(f + " argument of type " + v.type.str() + " is not native (utf8 pieces only)");
            emit(OP_SB_APPEND, b, v.reg, 0, 0, VT_STR, flags, o | (const_idx << 8));
        }
        release(v.reg);
    }
    // lpad / rpad (s, n, pad), replace (s, search, rep), translate (s, from, to), reverse (s), initcap (s) as one piece: every string
    // argument is any utf8 view, n any integer widened to int64; a NULL argument makes the piece NULL
    void append_fn_piece(const Expr& x, int b, int o, int flags, int const_idx) {
        const std::string& g = x.name;
        const int fn = string_fn_of(g);
        const size_t nargs = fn <= SBF_TRANSLATE ? 3 : 1;
        if (x.children.size() != nargs) fail(g + " takes " + std::to_string(nargs) + (nargs == 1 ? " argument" : " arguments"));
        if (fn == SBF_HEX || fn == SBF_CHR) {   // hex of an integer or of a utf8 / binary value's bytes, chr of an integer
            Val v = gen(*x.children[0]);
            int k = fn;
            if (v.type.is_integer() || v.type.id == T_NULL) {
                v = cast_to(v, DType(T_INT64));
                if (fn == SBF_HEX) k = SBF_HEX_INT;
            } else if (!(fn == SBF_HEX && v.type.is_varlen()))
                fail(g + " argument of type " + v.type.str() + " is not native" + (fn == SBF_HEX ? " (integers, utf8 and binary only)" : " (integers only)"));
            note_type(DType(T_UTF8));
            emit(OP_SB_APPEND, b, v.reg, 0, 0, vt_of(v.type), SB_VIEW | (flags & SB_WS) | (k << 4), o | (const_idx << 8));
            release(v.reg);
            return;
        }
        auto text = [&](const Expr& a) {
            Val v = gen(a);
            if (v.type.id != T_UTF8 && v.type.id != T_NULL) fail(g + " argument of type " + v.type.str() + " is not native (utf8 only)");
            return v;
        };
        Val s = text(*x.children[0]);
        int rb = 0, rc = 0;
        if (nargs == 3) {
            Val v1{-1, DType()};
            if (fn <= SBF_RPAD) {
                v1 = gen(*x.children[1]);
                if (!v1.type.is_integer() && v1.type.id != T_NULL) fail(g + " length of type " + v1.type.str() + " is not native (integers only)");
                v1 = cast_to(v1, DType(T_INT64));
            } else v1 = text(*x.children[1]);
            Val v2 = text(*x.children[2]);
            rb = v1.reg;
            rc = v2.reg;
        }
        emit(OP_SB_APPEND, b, s.reg, rb, rc, VT_STR, SB_VIEW | (flags & SB_WS) | (fn << 4), o | (const_idx << 8));
        release(s.reg);
        if (nargs == 3) {
            release(rb);
            release(rc);
        }
    }
    // concat (spark_strings.rs:117-192), concat_ws (:194-319), repeat (:75-91), space (:65-73) into utf8 output `o`.  Each piece is
    // generated, appended and released before the next, so the registers in use do not grow with the number of arguments.
    void build_string(const Expr& e, int o) {
        const std::string& f = e.name;
        const int b = alloc();
        note_type(DType(T_UTF8));
        emit(OP_SB_BEGIN, b, 0, 0, 0, VT_STR, 0, o);
        auto null_row = [&]() {   // a NULL literal argument that makes every row NULL
            Val v = literal(Literal{DType(T_UTF8), true});
            emit(OP_SB_APPEND, b, v.reg, 0, 0, VT_STR, SB_VIEW, o);
            release(v.reg);
        };
        auto is_lit = [](const Expr& x) { return x.kind == E_LITERAL; };
        if (f == "Spark_StringConcat") {
            for (auto& ch : e.children) append_piece(f, b, o, *ch, SB_VIEW);
        } else if (f == "Spark_StringConcatWs") {
            if (e.children.empty() || !is_lit(*e.children[0]) || e.children[0]->lit.type.id != T_UTF8)
                fail(f + " separator must be a utf8 literal");
            const Literal& sep = e.children[0]->lit;
            if (sep.is_null) null_row();
            else {
                const int sep_ci = add_pool_string(sep.s);
                for (size_t k = 1; k < e.children.size(); k++) {
                    const Expr& x = *e.children[k];
                    if (is_lit(x) && x.lit.is_null) continue;   // a NULL argument is skipped, separator included
                    append_piece(f, b, o, x, SB_VIEW | SB_WS, sep_ci);
                }
            }
        } else if (f == "Spark_StringRepeat") {
            if (e.children.size() != 2 || !is_lit(*e.children[1]) || e.children[1]->lit.type.id != T_INT32)
                fail(f + " count must be an int32 literal");
            const Literal& n = e.children[1]->lit;
            if (n.is_null) null_row();
            else append_piece(f, b, o, *e.children[0], SB_VIEW | SB_REPEAT, add_const((uint64_t)std::max<int64_t>(0, n.i), 0, true));
        } else if (f == "Spark_StringSpace") {
            if (e.children.size() != 1) fail(f + " takes one argument");
            append_piece(f, b, o, *e.children[0], SB_SPACE);
        } else append_fn_piece(e, b, o, SB_VIEW, 0);   // a string function as the whole value

        emit(OP_SB_END, 0, b, 0, 0, VT_STR, 0, o);
        release(b);
    }
    // the whole projection expression `ex` into output `o`; returns its type
    DType output(const Expr& ex, int o) {
        if (ex.kind == E_SCALAR_FN && (is_string_builder(ex.name) || string_fn_of(ex.name) != SBF_NONE)) {
            build_string(ex, o);
            return DType(T_UTF8);
        }
        if ((ex.kind == E_CAST || ex.kind == E_TRY_CAST) && ex.type.id == T_UTF8) {
            int scale = 0;
            const int kind = fmt_kind_of(infer_type(*ex.children[0], in), &scale);
            if (kind >= 0) {   // formatted directly into the output column
                Val v = gen(*ex.children[0]);
                note_type(v.type);
                note_type(ex.type);
                if (needs_text(kind, v.type)) prog.need_hi = prog.need_text = true;   // fmt_value formats them in vm_kernel<true, true> only
                emit(OP_FMT_OUT, 0, v.reg, 0, 0, vt_of(v.type), 0, o, (kind << 8) | scale);
                release(v.reg);
                return ex.type;
            }
        }
        Val v = gen(ex);
        DType t = v.type;
        if (t.id == T_NULL) fail("projection of an untyped NULL");
        note_type(t);
        emit(OP_OUT, 0, v.reg, 0, 0, vt_of(t), 0, o);
        release(v.reg);
        return t;
    }
};

VmProgram compile_projection(const std::vector<ExprPtr>& exprs, const Schema& input, bool row_num) {
    VmProgram p;
    p.impl = std::make_shared<VmProgramImpl>();
    Compiler c(input, *p.impl);
    c.row_num_ok = row_num;
    AURON_CHECK(exprs.size() <= VM_MAX_COLS, "too many projection expressions for one program");
    for (auto& e : exprs) reject_list_values(*e, input, nullptr, "a computed value (a key or argument of an aggregate, sort, join, window or shuffle)");
    for (size_t i = 0; i < exprs.size(); i++) {
        const Expr& ex = strip_utf8_cast(*exprs[i]);
        const int alg = ex.kind == E_SCALAR_FN ? digest_alg_of(ex.name) : 0;
        if (alg) {   // spark_crypto.rs:33-105: the digest of a utf8 or binary value's bytes
            if (ex.children.size() != 1) fail(ex.name + " takes one argument");
            const Expr& arg = strip_utf8_cast(*ex.children[0]);
            const DType at = infer_type(arg, input);
            if (!at.is_varlen()) fail(ex.name + " needs a utf8 or binary argument, got " + at.str());
            VmProgramImpl::Digest d{(int)i, alg, -1, -1};
            if (!is_plain_column(arg, input, &d.col)) {
                d.col = -1;
                d.hidden = (int)exprs.size() + p.impl->n_hidden++;
                AURON_CHECK(d.hidden < VM_MAX_COLS, "too many projection expressions for one program");
                c.output(arg, d.hidden);
            }
            p.impl->digests.push_back(d);
            p.out_types.push_back(DType(T_UTF8));
            p.impl->out_vt.push_back(VT_STR);
            continue;
        }
        const DType t = c.output(ex, (int)i);
        p.out_types.push_back(t);
        p.impl->out_vt.push_back(vt_of(t));
    }
    return p;
}
static int64_t host_f64_total(double d) {
    int64_t b;
    memcpy(&b, &d, 8);
    return b < 0 ? (b ^ 0x7fffffffffffffffll) : b;
}
static int64_t host_f32_total(float f) {
    int32_t b;
    memcpy(&b, &f, 4);
    return (int64_t)(b < 0 ? (b ^ 0x7fffffff) : b);
}
// conjunction of `column <cmp> literal` / IS [NOT] NULL terms over fixed-width columns?
static bool try_compile_simple(const std::vector<ExprPtr>& conjuncts, const Schema& input, VmProgramImpl& im) {
    std::vector<SimpleTerm> terms;
    std::vector<int> cols, vts;
    auto slot_of = [&](int col, int vt) {
        for (size_t i = 0; i < cols.size(); i++)
            if (cols[i] == col) return (int)i;
        cols.push_back(col);
        vts.push_back(vt);
        return (int)cols.size() - 1;
    };
    for (auto& e : conjuncts) {
        SimpleTerm t{};
        int idx;
        if ((e->kind == E_IS_NULL || e->kind == E_IS_NOT_NULL) && is_plain_column(*e->children[0], input, &idx)) {
            const DType& ct = input.fields[idx].type;
            if (ct.is_varlen() || ct.id == T_NULL) return false;
            t.col = slot_of(idx, vt_of(ct));
            t.op = e->kind == E_IS_NULL ? OP_ISNULL : OP_ISNOTNULL;
            terms.push_back(t);
            continue;
        }
        if (e->kind != E_BINARY) return false;
        int op = e->op == "Eq" ? OP_EQ : e->op == "NotEq" ? OP_NE : e->op == "Lt" ? OP_LT : e->op == "LtEq" ? OP_LE : e->op == "Gt" ? OP_GT : e->op == "GtEq" ? OP_GE : -1;
        if (op < 0) return false;
        const Expr* ce = e->children[0].get();
        const Expr* le = e->children[1].get();
        if (ce->kind == E_LITERAL && le->kind == E_COLUMN) {   // literal <op> column: mirror the operator
            std::swap(ce, le);
            op = op == OP_LT ? OP_GT : op == OP_LE ? OP_GE : op == OP_GT ? OP_LT : op == OP_GE ? OP_LE : op;
        }
        if (ce->kind != E_COLUMN || le->kind != E_LITERAL || le->lit.is_null) return false;
        idx = resolve_col(*ce, input);
        const DType& ct = input.fields[idx].type;
        const DType& lt = le->lit.type;
        if (ct.is_varlen() || ct.id == T_NULL) return false;
        // the VM compares a timestamp only with a timestamp of the same unit (raw numbers of two units mean different instants)
        if ((ct.id == T_TIMESTAMP || lt.id == T_TIMESTAMP) && !(lt == ct)) return false;
        int vt = vt_of(ct);
        if (ct.id == T_DECIMAL128) {
            if (!(lt == ct)) return false;
            t.c_lo = (int64_t)le->lit.lo;
            t.c_hi = le->lit.hi;
        } else if (ct.is_float()) {
            if (!(lt == ct)) return false;
            t.c_lo = ct.id == T_FLOAT32 ? host_f32_total((float)le->lit.d) : host_f64_total(le->lit.d);
        } else {
            if (vt_of(lt) > VT_I64 || lt.is_float() || lt.id == T_DECIMAL128 || (lt.id == T_BOOL) != (ct.id == T_BOOL)) return false;
            t.c_lo = le->lit.i;
        }
        t.col = slot_of(idx, vt);
        t.op = op;
        terms.push_back(t);
    }
    if (terms.empty() || terms.size() > (size_t)SP_MAX_TERMS || cols.size() > (size_t)SP_MAX_COLS) return false;
    im.simple_terms = terms;
    im.simple_cols = cols;
    im.simple_vt = vts;
    // fold into one closed interval per column when every term is an ordering comparison on a non-decimal column
    std::vector<int64_t> lo(cols.size(), INT64_MIN), hi(cols.size(), INT64_MAX);
    bool foldable = true;
    for (auto& t : terms) {
        if (vts[t.col] == VT_DEC || t.op == OP_NE || t.op == OP_ISNULL) {
            foldable = false;
            break;
        }
        int64_t c = t.c_lo;
        switch (t.op) {
            case OP_EQ: lo[t.col] = std::max(lo[t.col], c); hi[t.col] = std::min(hi[t.col], c); break;
            case OP_LT: if (c == INT64_MIN) { lo[t.col] = 1; hi[t.col] = 0; } else hi[t.col] = std::min(hi[t.col], c - 1); break;
            case OP_LE: hi[t.col] = std::min(hi[t.col], c); break;
            case OP_GT: if (c == INT64_MAX) { lo[t.col] = 1; hi[t.col] = 0; } else lo[t.col] = std::max(lo[t.col], c + 1); break;
            case OP_GE: lo[t.col] = std::max(lo[t.col], c); break;
            default: break;   // IS NOT NULL: validity is required by every interval anyway
        }
    }
    if (foldable) {
        im.iv_lo = lo;
        im.iv_hi = hi;
    }
    return true;
}

bool predicate_intervals(const VmProgram& p, std::vector<int>* cols, std::vector<int64_t>* lo, std::vector<int64_t>* hi) {
    if (!p.impl || p.impl->iv_lo.empty()) return false;
    for (int vt : p.impl->simple_vt)
        if (vt != VT_I8 && vt != VT_I16 && vt != VT_I32 && vt != VT_I64) return false;
    *cols = p.impl->simple_cols;
    *lo = p.impl->iv_lo;
    *hi = p.impl->iv_hi;
    return true;
}

VmProgram compile_predicate(const std::vector<ExprPtr>& conjuncts, const Schema& input) {
    VmProgram p;
    p.impl = std::make_shared<VmProgramImpl>();
    p.is_predicate = true;
    for (auto& e : conjuncts) reject_list_values(*e, input, nullptr, "a predicate");
    if (!getenv("AURON_DISABLE_SIMPLE_PREDICATE") && try_compile_simple(conjuncts, input, *p.impl)) return p;
    Compiler c(input, *p.impl);
    AURON_CHECK(!conjuncts.empty(), "empty predicate");
    Compiler::Val acc = c.gen(*conjuncts[0]);
    for (size_t i = 1; i < conjuncts.size(); i++) {
        Compiler::Val v = c.gen(*conjuncts[i]);
        c.emit(OP_AND, acc.reg, acc.reg, v.reg);
        c.release(v.reg);
    }
    c.emit(OP_OUT_PRED, 0, acc.reg);
    return p;
}

static void upload(Ctx& ctx, VmProgramImpl& im) {
    // programs are tiny; upload per evaluation keeps them stream-ordered with the launch
    im.d_code = to_device(ctx, im.code.data(), im.code.size() * sizeof(Instr));
    im.d_consts = to_device(ctx, im.consts.empty() ? (const void*)"" : (const void*)im.consts.data(), im.consts.size() * sizeof(ConstEntry));
    im.d_pool = to_device(ctx, im.pool.data(), im.pool.size());
}
static void bind_inputs(const VmProgramImpl& im, const Batch& in, VmParams& p) {
    memset(&p, 0, sizeof(p));
    for (size_t s = 0; s < im.in_cols.size(); s++) {
        const Column& c = *in.cols[im.in_cols[s]];
        p.in_data[s] = c.data ? c.data->ptr : nullptr;
        p.in_valid[s] = c.vbits();
        p.in_off[s] = P<int32_t>(c.offsets);
    }
    p.prog = P<Instr>(im.d_code);
    p.consts = P<ConstEntry>(im.d_consts);
    p.pool = P<uint8_t>(im.d_pool);
    p.n_instr = (int)im.code.size();
}
static void launch_vm(Ctx& ctx, const VmProgramImpl& im, const VmParams& p) {
    static bool attr = false;
    size_t prog_bytes = ((im.code.size() * sizeof(Instr) + 15) / 16) * 16;
    size_t smem = (im.need_hi ? 2 : 1) * VM_NREG * VM_THREADS * 8 + prog_bytes;
    if (!attr) {
        CUDA_OK(cudaFuncSetAttribute(vm_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 2 * VM_NREG * VM_THREADS * 8 + 1024 * 16));
        CUDA_OK(cudaFuncSetAttribute(vm_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, VM_NREG * VM_THREADS * 8 + 1024 * 16));
        attr = true;
    }
    int64_t blocks = (p.n + VM_THREADS - 1) / VM_THREADS;
    int per_sm = im.need_hi ? 3 : 6;
    unsigned grid = (unsigned)std::max<int64_t>(1, std::min<int64_t>(blocks, (int64_t)ctx.sm_count * per_sm));
    ProfScope ps(ctx, "expr_vm");
    if (im.need_text) launch_vm_text(grid, smem, ctx.stream, p);
    else if (im.need_hi) vm_kernel<true><<<grid, VM_THREADS, smem, ctx.stream>>>(p);
    else vm_kernel<false><<<grid, VM_THREADS, smem, ctx.stream>>>(p);
    LAUNCH_CHECK(ctx);
}

__global__ void narrow_offsets_kernel2(const int64_t* __restrict__ off64, int32_t* __restrict__ off32, int64_t n_plus_1) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n_plus_1) off32[i] = (int32_t)off64[i];
}

// utf8 output `c` from its int64 row lengths: offsets by an exclusive scan, then the data buffer
static void finish_offsets(Ctx& ctx, Column& c, int64_t* lens, int64_t n) {
    exclusive_scan_i64(ctx, lens, lens, n, lens + n);
    narrow_offsets_kernel2<<<(unsigned)((n + 1 + 255) / 256), 256, 0, ctx.stream>>>(lens, P<int32_t>(c.offsets), n + 1);
    LAUNCH_CHECK(ctx);
    int64_t total = 0;
    to_host(ctx, &total, lens + n, 8);
    AURON_CHECK(total <= (int64_t)INT32_MAX, "utf8 column exceeds 2 GiB in one batch");
    c.data = dalloc(ctx, (size_t)total);
    c.data_bytes = total;
}

std::vector<ColumnPtr> eval_projection(Ctx& ctx, const VmProgram& prog, const Batch& in, const int32_t* sel, int64_t n_out, int64_t row_base) {
    init_pow10_tables();
    VmProgramImpl& im = *prog.impl;
    const size_t n_vis = prog.out_types.size(), n_all = n_vis + (size_t)im.n_hidden;   // hidden outputs: digest arguments
    std::vector<bool> digested(n_all, false);
    for (auto& d : im.digests) digested[(size_t)d.out] = true;
    std::vector<ColumnPtr> outs;
    std::vector<Buf> lens(n_all);
    bool vm_str = false;
    for (size_t i = 0; i < n_all; i++) {
        const DType t = i < n_vis ? prog.out_types[i] : DType(T_UTF8);
        auto c = std::make_shared<Column>();
        c->type = t;
        c->len = n_out;
        c->validity = dalloc(ctx, bitmap_alloc_bytes(n_out));
        c->null_count = -1;
        if (t.id == T_BOOL) c->data = dalloc(ctx, bitmap_alloc_bytes(n_out));
        else if (t.is_varlen()) {
            lens[i] = dalloc(ctx, (size_t)(n_out + 1) * 8);
            c->offsets = dalloc(ctx, (size_t)(n_out + 1) * 4);
            vm_str = vm_str || !digested[i];
        } else c->data = dalloc(ctx, (size_t)n_out * t.width());
        outs.push_back(c);
    }
    if (n_out == 0) {
        for (auto& c : outs)
            if (c->type.is_varlen()) {
                CUDA_OK(cudaMemsetAsync(c->offsets->ptr, 0, 4, ctx.stream));
                c->data = dalloc(ctx, 0);
            }
        outs.resize(n_vis);
        return outs;
    }
    if (!im.code.empty()) {
        upload(ctx, im);
        VmParams p;
        bind_inputs(im, in, p);
        p.sel = sel;
        p.n = n_out;
        p.row_base = row_base;
        p.mode = 0;
        for (size_t i = 0; i < outs.size(); i++) {
            p.out_data[i] = outs[i]->data ? outs[i]->data->ptr : nullptr;
            p.out_valid[i] = P<uint32_t>(outs[i]->validity);
            p.out_lens[i] = P<int64_t>(lens[i]);
        }
        launch_vm(ctx, im, p);
        if (vm_str) {
            for (size_t i = 0; i < outs.size(); i++) {
                if (!outs[i]->type.is_varlen() || digested[i]) continue;
                finish_offsets(ctx, *outs[i], P<int64_t>(lens[i]), n_out);
                p.out_data[i] = outs[i]->data->ptr;
                p.out_off[i] = P<int32_t>(outs[i]->offsets);
            }
            p.mode = 1;
            launch_vm(ctx, im, p);
        }
    }
    for (auto& d : im.digests) {   // k_digest.cu: one launch per digest output, after the VM built any argument it needed
        const Column& src = d.col >= 0 ? *in.cols[(size_t)d.col] : *outs[(size_t)d.hidden];
        const int32_t* s = d.col >= 0 ? sel : nullptr;
        Column& out = *outs[(size_t)d.out];
        digest_lengths(ctx, src.vbits(), s, n_out, d.alg, P<uint32_t>(out.validity), P<int64_t>(lens[(size_t)d.out]));
        finish_offsets(ctx, out, P<int64_t>(lens[(size_t)d.out]), n_out);
        digest_hex(ctx, d.alg, P<int32_t>(src.offsets), P<uint8_t>(src.data), s, n_out, P<int32_t>(out.offsets), P<uint8_t>(out.data));
    }
    outs.resize(n_vis);
    return outs;
}

Buf eval_predicate(Ctx& ctx, const VmProgram& prog, const Batch& in, int64_t n_rows) {
    init_pow10_tables();
    VmProgramImpl& im = *prog.impl;
    Buf mask = dalloc(ctx, bitmap_alloc_bytes(n_rows));
    if (n_rows == 0) return mask;
    if (!im.iv_lo.empty()) {
        IntervalArgs a;
        memset(&a, 0, sizeof(a));
        a.n_cols = (int)im.simple_cols.size();
        for (int c = 0; c < a.n_cols; c++) {
            const Column& col = *in.cols[im.simple_cols[c]];
            a.data[c] = col.data ? col.data->ptr : nullptr;
            a.valid[c] = (const uint32_t*)col.vbits();
            a.vt[c] = im.simple_vt[c];
            a.lo[c] = im.iv_lo[c];
            a.hi[c] = im.iv_hi[c];
        }
        int64_t warps = (n_rows + 127) / 128;
        unsigned grid = (unsigned)std::max<int64_t>(1, std::min<int64_t>((warps + 7) / 8, (int64_t)ctx.sm_count * 8));
        ProfScope ps(ctx, "simple_predicate");
        bool all32 = a.n_cols <= 4, all64 = a.n_cols <= 4;
        for (int c = 0; c < a.n_cols; c++) {
            all32 = all32 && a.vt[c] == VT_I32;
            all64 = all64 && a.vt[c] == VT_I64;
        }
        if ((all32 || all64) && !getenv("AURON_DISABLE_VEC_PREDICATE")) {
            if (all32) launch_interval_vec<int32_t>(ctx, a, n_rows, P<uint32_t>(mask), grid);
            else launch_interval_vec<int64_t>(ctx, a, n_rows, P<uint32_t>(mask), grid);
            LAUNCH_CHECK(ctx);
            return mask;
        }
        switch (a.n_cols) {
            case 1: interval_predicate_kernel<1><<<grid, 256, 0, ctx.stream>>>(a, n_rows, P<uint32_t>(mask)); break;
            case 2: interval_predicate_kernel<2><<<grid, 256, 0, ctx.stream>>>(a, n_rows, P<uint32_t>(mask)); break;
            case 3: interval_predicate_kernel<3><<<grid, 256, 0, ctx.stream>>>(a, n_rows, P<uint32_t>(mask)); break;
            default: interval_predicate_kernel<4><<<grid, 256, 0, ctx.stream>>>(a, n_rows, P<uint32_t>(mask)); break;
        }
        LAUNCH_CHECK(ctx);
        return mask;
    }
    if (!im.simple_terms.empty()) {
        SimplePredArgs a;
        memset(&a, 0, sizeof(a));
        a.n_cols = (int)im.simple_cols.size();
        a.n_terms = (int)im.simple_terms.size();
        for (int c = 0; c < a.n_cols; c++) {
            const Column& col = *in.cols[im.simple_cols[c]];
            a.data[c] = col.data ? col.data->ptr : nullptr;
            a.valid[c] = col.vbits();
            a.vt[c] = im.simple_vt[c];
        }
        for (int k = 0; k < a.n_terms; k++) a.t[k] = im.simple_terms[k];
        int64_t blocks = (n_rows + 255) / 256;
        unsigned grid = (unsigned)std::max<int64_t>(1, std::min<int64_t>(blocks, (int64_t)ctx.sm_count * 16));
        ProfScope ps(ctx, "simple_predicate");
        simple_predicate_kernel<<<grid, 256, 0, ctx.stream>>>(a, n_rows, P<uint32_t>(mask));
        LAUNCH_CHECK(ctx);
        return mask;
    }
    upload(ctx, im);
    VmParams p;
    bind_inputs(im, in, p);
    p.n = n_rows;
    p.pred_out = P<uint32_t>(mask);
    launch_vm(ctx, im, p);
    return mask;
}

int float_to_text_host(int bits, uint64_t value, char* out) { return ft_float_to_text(bits, value, out); }
bool text_to_float_host(int bits, const uint8_t* text, int32_t len, uint64_t* value) { return ft_text_to_float(bits, text, len, false, value); }
#endif

}  // namespace auron
