// format_number.cuh — binary64 -> text exactly as CPython's str(): the arithmetic of the "string" cast of the
// /fieldTypes service,
//     values[field] = "" if document[field] is None else str(document[field])
// (data_type_handler_image/data_type_update.py:22-28), which the reference runs one document at a time.  It is the
// inverse of parse_number.cuh: parse_number(format_cell(v, s)) gives back v and s.
//
// Everything here is `__host__ __device__` and pure integer arithmetic, so the very same code is unit-tested on the CPU
// against Python's own repr() / str(int) (tests/test_format_cpu.py compiles it with g++) before it runs in the
// k_format_number_len / k_format_number_write kernels.
//
// Per cell, by the parser's status codes (parse_number.cuh):
//   kFloat   -> repr(float(v)): the shortest digits that read back as v (ties: the closer one, then even), placed
//               positionally when the decimal point position decpt (v = 0.d1d2... * 10^decpt) has -4 < decpt <= 16,
//               with ".0" after an integral value, else as d[.ddd]e+XX / e-XX with at least two exponent digits;
//               "0.0" / "-0.0", "inf" / "-inf", and "nan" for every NaN (CPython Python/pystrtod.c format_float_short,
//               repr style 'r' with Py_DTSF_ADD_DOT_0).  At most kMaxFloatLen bytes.
//   kInteger -> str(int(v)) of a finite integral v: every digit of the exact value (-0.0 -> "0").  |v| < 2^64 takes a
//               u64 digit loop; beyond that a 1024-bit integer divided by 10^9 (up to 309 digits for DBL_MAX).
//   kEmpty   -> "" (None -> "").
//
// Shortest digits: Ryu (U. Adams, "Ryu: fast float-to-string conversion", PLDI 2018).  The 64-bit significand,
// scaled by 4 so the interval bounds are integers, is multiplied by a 125-bit power of five (ryu_pow5.inc, rounded
// down, for negative binary exponents) or by a 125/126-bit reciprocal power of five (ryu_pow5_inv.inc, rounded up,
// for non-negative ones) and shifted, which gives the decimal scaled value vr and the bounds vp / vm of its rounding
// interval, all truncated at the same decimal position.  Digits are then removed while vp / 10 > vm / 10; the last
// removed digit of vr decides the rounding.  Where truncation could have hidden trailing zeros of vr or vm (small
// decimal exponents only) exact divisibility by 5^q or 2^q decides whether the bounds are reached and whether a
// removed "5" is an exact tie.  Both tables come from scripts/gen_ryu_table.py.
#pragma once
#include <stdint.h>
#include "parse_number.cuh"

namespace lo {
namespace fmt {

constexpr int kMaxFloatLen = 24;    // "-1.7976931348623157e+308"
constexpr int kMaxCell     = 310;   // "-" and the 309 digits of int(DBL_MAX)

constexpr int kPow5Bits = 125;      // significant bits of both tables
constexpr int kPow5N    = 326;      // 5^0 .. 5^325 (negative binary exponents down to the smallest subnormal)
constexpr int kPow5InvN = 291;      // 5^-0 .. 5^-290 (non-negative binary exponents up to DBL_MAX)

static
#ifdef __CUDACC__
__device__
#endif
const uint64_t kRyuPow5[kPow5N * 2] = {
#include "ryu_pow5.inc"
};
static
#ifdef __CUDACC__
__device__
#endif
const uint64_t kRyuPow5Inv[kPow5InvN * 2] = {
#include "ryu_pow5_inv.inc"
};
#ifdef __CUDACC__
static const uint64_t kRyuPow5Host[kPow5N * 2] = {
#include "ryu_pow5.inc"
};
static const uint64_t kRyuPow5InvHost[kPow5InvN * 2] = {
#include "ryu_pow5_inv.inc"
};
#endif

LO_HD const uint64_t *ryu_pow5(int i) {
#if defined(__CUDACC__) && !defined(__CUDA_ARCH__)
    return kRyuPow5Host + 2 * i;
#else
    return kRyuPow5 + 2 * i;
#endif
}

LO_HD const uint64_t *ryu_pow5_inv(int q) {
#if defined(__CUDACC__) && !defined(__CUDA_ARCH__)
    return kRyuPow5InvHost + 2 * q;
#else
    return kRyuPow5Inv + 2 * q;
#endif
}

// closed forms, exact over the exponents binary64 reaches (asserted by scripts/gen_ryu_table.py)
LO_HD int32_t log10_pow2(int32_t e) { return (int32_t)(((uint32_t)e * 78913u) >> 18); }          // floor(e log10 2)
LO_HD int32_t log10_pow5(int32_t e) { return (int32_t)(((uint32_t)e * 732923u) >> 20); }         // floor(e log10 5)
LO_HD int32_t pow5_bits(int32_t e) { return (int32_t)(((uint32_t)e * 1217359u) >> 19) + 1; }     // bit length of 5^e

// (m * mul) >> j for a 128-bit mul = {lo, hi}; 64 <= j < 128 for every binary64
LO_HD uint64_t mul_shift(uint64_t m, const uint64_t *mul, int32_t j) {
    uint64_t h0, l0, h1, l1;
    num::mul64(m, mul[0], h0, l0);
    num::mul64(m, mul[1], h1, l1);
    const uint64_t lo = l1 + h0;
    const uint64_t hi = h1 + (lo < h0);
    const int s = j - 64;
    return s == 0 ? lo : (lo >> s) | (hi << (64 - s));
}

LO_HD bool multiple_of_pow5(uint64_t v, int32_t p) {
    int32_t count = 0;
    while (v % 5 == 0) { v /= 5; ++count; }           // v != 0 here
    return count >= p;
}

struct Decimal {
    uint64_t digits;     // shortest digit string, as an integer (no trailing zeros unless they are needed)
    int32_t  exponent;   // |value| = digits * 10^exponent
};

// Ryu: the shortest decimal in the rounding interval of a finite nonzero binary64 (sign ignored)
LO_HD Decimal shortest(uint64_t bits) {
    const uint64_t ieee_m = bits & ((1ull << 52) - 1);
    const uint32_t ieee_e = (uint32_t)((bits >> 52) & 0x7FF);
    int32_t e2;
    uint64_t m2;
    if (ieee_e == 0) { e2 = 1 - 1023 - 52 - 2; m2 = ieee_m; }
    else             { e2 = (int32_t)ieee_e - 1023 - 52 - 2; m2 = (1ull << 52) | ieee_m; }
    const bool accept_bounds = (m2 & 1) == 0;           // round-to-even reads an exact bound back as v
    const uint64_t mv = 4 * m2;
    const uint32_t mm_shift = ieee_m != 0 || ieee_e <= 1;   // the lower neighbour is closer at a power of two
    uint64_t vr, vp, vm;
    int32_t e10;
    bool vm_tz = false, vr_tz = false;                  // the truncated parts of vm / vr are exactly zero
    if (e2 >= 0) {
        const int32_t q = log10_pow2(e2) - (e2 > 3);
        e10 = q;
        const int32_t j = -e2 + q + kPow5Bits + pow5_bits(q) - 1;
        const uint64_t *mul = ryu_pow5_inv(q);
        vr = mul_shift(mv, mul, j);
        vp = mul_shift(mv + 2, mul, j);
        vm = mul_shift(mv - 1 - mm_shift, mul, j);
        if (q <= 21) {                                  // only one of mv, mp, mm can be a multiple of 5
            if (mv % 5 == 0)        vr_tz = multiple_of_pow5(mv, q);
            else if (accept_bounds) vm_tz = multiple_of_pow5(mv - 1 - mm_shift, q);
            else                    vp -= multiple_of_pow5(mv + 2, q);
        }
    } else {
        const int32_t q = log10_pow5(-e2) - (-e2 > 1);
        e10 = q + e2;
        const int32_t i = -e2 - q;
        const int32_t j = q - (pow5_bits(i) - kPow5Bits);
        const uint64_t *mul = ryu_pow5(i);
        vr = mul_shift(mv, mul, j);
        vp = mul_shift(mv + 2, mul, j);
        vm = mul_shift(mv - 1 - mm_shift, mul, j);
        if (q <= 1) {                                   // mv has two trailing zero bits, mp one, mm one iff mm_shift
            vr_tz = true;
            if (accept_bounds) vm_tz = mm_shift == 1;
            else --vp;
        } else if (q < 63) {                            // vr = mv * 5^i / 2^q: exact iff 2^q divides mv
            vr_tz = (mv & ((1ull << q) - 1)) == 0;
        }
    }
    int32_t removed = 0;
    uint64_t out;
    if (vm_tz || vr_tz) {                               // rare: a bound or an exact tie may decide
        uint32_t last = 0;
        while (vp / 10 > vm / 10) {
            vm_tz &= vm % 10 == 0;
            vr_tz &= last == 0;
            last = (uint32_t)(vr % 10);
            vr /= 10; vp /= 10; vm /= 10;
            ++removed;
        }
        if (vm_tz) {
            while (vm % 10 == 0) {
                vr_tz &= last == 0;
                last = (uint32_t)(vr % 10);
                vr /= 10; vp /= 10; vm /= 10;
                ++removed;
            }
        }
        if (vr_tz && last == 5 && vr % 2 == 0) last = 4;     // exactly ...50..0: round half to even
        out = vr + ((vr == vm && (!accept_bounds || !vm_tz)) || last >= 5);
    } else {
        bool round_up = false;
        if (vp / 100 > vm / 100) {
            round_up = vr % 100 >= 50;
            vr /= 100; vp /= 100; vm /= 100;
            removed += 2;
        }
        while (vp / 10 > vm / 10) {
            round_up = vr % 10 >= 5;
            vr /= 10; vp /= 10; vm /= 10;
            ++removed;
        }
        out = vr + (vr == vm || round_up);
    }
    Decimal d;
    d.digits = out;
    d.exponent = e10 + removed;
    return d;
}

LO_HD int dec_len(uint64_t v) {                         // decimal digits of v (1 for 0)
    int n = 1;
    uint64_t p = 10;
    while (n < 20 && v >= p) { p *= 10; ++n; }
    return n;
}

// writes the low n decimal digits of v (leading zeros included) to dst, with a '.' after the first `split` of them
// when 0 < split < n; returns the bytes written
LO_HD int put_digits(uint64_t v, int n, int split, uint8_t *dst) {
    const int dot = (split > 0 && split < n) ? 1 : 0;
    for (int i = n - 1; i >= 0; --i) {
        dst[i + (dot && i >= split)] = (uint8_t)('0' + v % 10);
        v /= 10;
    }
    if (dot) dst[split] = '.';
    return n + dot;
}

LO_HD int put_text(const char *s, uint8_t *dst) {
    int n = 0;
    for (; s[n]; ++n) dst[n] = (uint8_t)s[n];
    return n;
}

// repr(float(v)); dst == nullptr returns the length only
LO_HD int format_float(uint64_t bits, uint8_t *dst) {
    const bool neg = bits >> 63;
    const uint32_t ieee_e = (uint32_t)((bits >> 52) & 0x7FF);
    const uint64_t ieee_m = bits & ((1ull << 52) - 1);
    if (ieee_e == 0x7FF) {
        const char *s = ieee_m ? "nan" : (neg ? "-inf" : "inf");
        return dst ? put_text(s, dst) : (ieee_m ? 3 : 3 + neg);
    }
    if (ieee_e == 0 && ieee_m == 0) return dst ? put_text(neg ? "-0.0" : "0.0", dst) : 3 + neg;
    const Decimal d = shortest(bits);
    const int olen = dec_len(d.digits);
    const int decpt = d.exponent + olen;                // |v| = 0.d1d2... * 10^decpt
    const bool positional = -4 < decpt && decpt <= 16;
    const int x = decpt - 1, ax = x < 0 ? -x : x;       // exponent of the d.ddd form
    const int xlen = ax >= 100 ? 3 : 2;
    int len = neg;
    if (!positional)       len += olen + (olen > 1) + 2 + xlen;
    else if (decpt <= 0)   len += 2 - decpt + olen;
    else if (decpt < olen) len += olen + 1;
    else                   len += decpt + 2;
    if (!dst) return len;
    int p = 0;
    if (neg) dst[p++] = '-';
    if (!positional) {
        p += put_digits(d.digits, olen, 1, dst + p);
        dst[p++] = 'e';
        dst[p++] = x < 0 ? '-' : '+';
        p += put_digits((uint64_t)ax, xlen, 0, dst + p);
    } else if (decpt <= 0) {
        dst[p++] = '0';
        dst[p++] = '.';
        for (int i = 0; i < -decpt; ++i) dst[p++] = '0';
        p += put_digits(d.digits, olen, 0, dst + p);
    } else if (decpt < olen) {
        p += put_digits(d.digits, olen, decpt, dst + p);
    } else {
        p += put_digits(d.digits, olen, 0, dst + p);
        for (int i = olen; i < decpt; ++i) dst[p++] = '0';
        dst[p++] = '.';
        dst[p++] = '0';
    }
    return p;
}

// finite and integer valued (float.is_integer()), so int(v) exists and is exact
LO_HD bool is_integral(uint64_t bits) {
    const uint32_t e = (uint32_t)((bits >> 52) & 0x7FF);
    const uint64_t m = bits & ((1ull << 52) - 1);
    if (e == 0x7FF) return false;
    if (e == 0) return m == 0;
    if (e < 1023) return false;
    if (e >= 1075) return true;
    return (m & ((1ull << (1075 - e)) - 1)) == 0;
}

// the digits of m2 * 2^e2 >= 2^64 (m2 < 2^53, e2 <= 971: at most 1024 bits, 309 digits); dst == nullptr counts only.
// Rare, so kept out of line: its 1024-bit scratch lives in its own frame, not in the registers of the common path.
LO_HD_NOINLINE int format_big_integer(uint64_t m2, int e2, uint8_t *dst) {
    uint32_t limb[33];                                   // little endian; the 33rd only ever receives zero bits
    for (int i = 0; i < 33; ++i) limb[i] = 0;
    const int w = e2 >> 5, r = e2 & 31;
    const uint64_t t0 = (uint64_t)(uint32_t)m2 << r, t1 = (m2 >> 32) << r;
    limb[w] = (uint32_t)t0;
    limb[w + 1] = (uint32_t)(t0 >> 32) | (uint32_t)t1;
    limb[w + 2] = (uint32_t)(t1 >> 32);
    uint32_t chunk[35];                                  // base-10^9 digits, least significant first
    int nc = 0, n = w + 3;
    while (n > 0 && limb[n - 1] == 0) --n;
    while (n > 0) {
        uint64_t rem = 0;
        for (int i = n - 1; i >= 0; --i) {
            const uint64_t cur = (rem << 32) | limb[i];
            limb[i] = (uint32_t)(cur / 1000000000u);
            rem = cur % 1000000000u;
        }
        chunk[nc++] = (uint32_t)rem;
        while (n > 0 && limb[n - 1] == 0) --n;
    }
    const int top = dec_len(chunk[nc - 1]);
    if (!dst) return 9 * (nc - 1) + top;
    int p = put_digits(chunk[nc - 1], top, 0, dst);
    for (int c = nc - 2; c >= 0; --c) p += put_digits(chunk[c], 9, 0, dst + p);
    return p;
}

// str(int(v)) of an integral v; dst == nullptr returns the length only
LO_HD int format_integer(uint64_t bits, uint8_t *dst) {
    const uint32_t e = (uint32_t)((bits >> 52) & 0x7FF);
    const uint64_t m2 = (bits & ((1ull << 52) - 1)) | (1ull << 52);
    const int neg = (e != 0 && (bits >> 63)) ? 1 : 0;  // int(-0.0) is 0
    if (neg && dst) dst[0] = '-';
    if (e >= 1023 + 64) return neg + format_big_integer(m2, (int)e - 1075, dst ? dst + neg : nullptr);
    const uint64_t u = e == 0 ? 0 : (e >= 1075 ? m2 << (e - 1075) : m2 >> (1075 - e));
    const int len = dec_len(u);
    return neg + (dst ? put_digits(u, len, 0, dst + neg) : len);
}

// one cell of the "string" cast; -1 for a status other than FLOAT / INTEGER / EMPTY or an INTEGER cell that is not
// finite and integral (nothing is written then).  dst == nullptr returns the length only.
LO_HD int format_cell(uint64_t bits, uint8_t status, uint8_t *dst) {
    if (status == num::kFloat) return format_float(bits, dst);
    if (status == num::kInteger) return is_integral(bits) ? format_integer(bits, dst) : -1;
    if (status == num::kEmpty) return 0;
    return -1;
}

}  // namespace fmt
}  // namespace lo
