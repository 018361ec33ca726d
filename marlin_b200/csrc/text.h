// The text tokens of the matrix files: java.lang.Double.toString as utils/mt_utils.py::_jdouble states it, and
// Long.toString, for one value at a time.  Host and device share this code (the host build is what
// tests/test_text_host.py compiles with g++), and it uses integer arithmetic only, so both give the same bytes.
//
// Digits: the shortest decimal d * 10^e that rounds back to the double, and of several such the closest to its exact
// value (ties to an even last digit), found Ryu's way: the value and the two midpoints to its neighbours, scaled by 4,
// are multiplied by a 125-bit approximation of 5^i or 2^k / 5^q (text_tables.h) and shifted, which gives their exact
// decimal floors at a precision a few digits beyond the value's; digits are then removed while the interval between the
// midpoints still holds a shorter number.  Trailing-zero bookkeeping makes the removal exact where a floor was exact.
//
// Layout: plain notation for 1e-3 <= |v| < 1e7, decided on the double itself (integer compares of its bits), else
// d.dddE[-]n; at least one digit after the point; NaN (every payload and sign), Infinity, -Infinity, -0.0.  That is at
// most TEXT_TOKEN_MAX bytes.  _jdouble prints the plain shortest digits where JDK 19's Double.toString may prefer a closer
// two-digit form (Double.MIN_VALUE: 5.0E-324 here, 4.9E-324 on the JVM), and so does this code.
#pragma once
#include "text_tables.h"

#include <cstdint>

#if defined(__CUDACC__)
#define MB_TEXT_FN __host__ __device__ __forceinline__
#else
#define MB_TEXT_FN inline
#endif

namespace mb {
namespace text {

constexpr int TEXT_TOKEN_MAX = 24;        // -1.2345678901234567E-308
constexpr int TEXT_LONG_MAX = 20;         // -9223372036854775808

// The double bounds of plain notation: 0.001 (the double nearest it, which is what 1e-3 means) and 1.0E7.
constexpr uint64_t PLAIN_LO_BITS = 0x3F50624DD2F1A9FCull;
constexpr uint64_t PLAIN_HI_BITS = 0x416312D000000000ull;

MB_TEXT_FN uint64_t umulh(uint64_t a, uint64_t b) {
#if defined(__CUDA_ARCH__)
    return __umul64hi(a, b);
#else
    return (uint64_t)(((unsigned __int128)a * b) >> 64);
#endif
}

MB_TEXT_FN int pow5bits(int e) { return (int)(((uint32_t)e * 1217359u) >> 19) + 1; }
MB_TEXT_FN int log10_pow2(int e) { return (int)(((uint32_t)e * 78913u) >> 18); }
MB_TEXT_FN int log10_pow5(int e) { return (int)(((uint32_t)e * 732923u) >> 20); }

// floor(m * mul / 2^j) for a 128-bit mul (low word first) and 64 <= j < 128; the quotient fits 64 bits here.
MB_TEXT_FN uint64_t mul_shift(uint64_t m, const uint64_t* mul, int j) {
    const uint64_t lo_hi = umulh(m, mul[0]);
    const uint64_t mid_lo = m * mul[1], mid_hi = umulh(m, mul[1]);
    const uint64_t sum = mid_lo + lo_hi;
    const uint64_t hi = mid_hi + (sum < mid_lo ? 1 : 0);
    const int s = j - 64;
    return s == 0 ? sum : (sum >> s) | (hi << (64 - s));
}

MB_TEXT_FN bool multiple_of_pow5(uint64_t v, int p) {
    int n = 0;
    while (v % 5 == 0 && n < p) {
        v /= 5;
        ++n;
    }
    return n >= p;
}

MB_TEXT_FN bool multiple_of_pow2(uint64_t v, int p) { return (v & ((1ull << p) - 1)) == 0; }

// value = digits * 10^exp, digits without trailing zeros.
struct Decimal {
    uint64_t digits;
    int exp;
};

// The shortest, closest decimal of a finite nonzero double's magnitude (bits without the sign).  pow5 and pow5_inv are
// MB_TEXT_POW5_TABLE and MB_TEXT_POW5_INV_TABLE, wherever the caller keeps them.
MB_TEXT_FN Decimal shortest(uint64_t bits, const uint64_t* pow5, const uint64_t* pow5_inv) {
    const uint64_t mant = bits & ((1ull << 52) - 1);
    const int bexp = (int)((bits >> 52) & 0x7ff);
    int e2;
    uint64_t m2;
    if (bexp == 0) {
        e2 = 1 - 1023 - 52 - 2;
        m2 = mant;
    } else {
        e2 = bexp - 1023 - 52 - 2;
        m2 = (1ull << 52) | mant;
    }
    const bool even = (m2 & 1) == 0;                 // round-half-even parsing: an even significand owns its midpoints
    const uint64_t mv = 4 * m2;
    const uint32_t mm_shift = (mant != 0 || bexp <= 1) ? 1 : 0;   // the lower neighbour is closer at a power of two
    uint64_t vr, vp, vm;
    int e10;
    bool vm_zeros = false, vr_zeros = false;
    if (e2 >= 0) {
        const int q = log10_pow2(e2) - (e2 > 3 ? 1 : 0);
        e10 = q;
        const int k = MB_TEXT_POW5_INV_BITS + pow5bits(q) - 1;
        const int i = -e2 + q + k;
        const uint64_t* mul = pow5_inv + 2 * q;
        vr = mul_shift(mv, mul, i);
        vp = mul_shift(mv + 2, mul, i);
        vm = mul_shift(mv - 1 - mm_shift, mul, i);
        if (q <= 23) {                               // mv < 2^55 < 5^24: no larger power of five divides it
            if (mv % 5 == 0) vr_zeros = multiple_of_pow5(mv, q);
            else if (even) vm_zeros = multiple_of_pow5(mv - 1 - mm_shift, q);
            else vp -= multiple_of_pow5(mv + 2, q) ? 1 : 0;
        }
    } else {
        const int q = log10_pow5(-e2) - (-e2 > 1 ? 1 : 0);
        e10 = q + e2;
        const int i = -e2 - q;
        const int k = pow5bits(i) - MB_TEXT_POW5_BITS;
        const int j = q - k;
        const uint64_t* mul = pow5 + 2 * i;
        vr = mul_shift(mv, mul, j);
        vp = mul_shift(mv + 2, mul, j);
        vm = mul_shift(mv - 1 - mm_shift, mul, j);
        if (q <= 1) {                                // the floors divide by at most 2^1: mv and mv + 2 are exact
            vr_zeros = true;
            if (even) vm_zeros = mm_shift == 1;
            else --vp;
        } else if (q < 63) {
            vr_zeros = multiple_of_pow2(mv, q);
        }
    }
    int removed = 0;
    uint32_t last = 0;
    uint64_t out;
    if (vm_zeros || vr_zeros) {
        while (vp / 10 > vm / 10) {
            vm_zeros &= vm % 10 == 0;
            vr_zeros &= last == 0;
            last = (uint32_t)(vr % 10);
            vr /= 10;
            vp /= 10;
            vm /= 10;
            ++removed;
        }
        if (vm_zeros) {
            while (vm % 10 == 0) {
                vr_zeros &= last == 0;
                last = (uint32_t)(vr % 10);
                vr /= 10;
                vp /= 10;
                vm /= 10;
                ++removed;
            }
        }
        if (vr_zeros && last == 5 && vr % 2 == 0) last = 4;                   // an exact tie: keep the even digit
        out = vr + (((vr == vm && (!even || !vm_zeros)) || last >= 5) ? 1 : 0);
    } else {
        bool round_up = false;
        while (vp / 10 > vm / 10) {
            round_up = vr % 10 >= 5;
            vr /= 10;
            vp /= 10;
            vm /= 10;
            ++removed;
        }
        out = vr + ((vr == vm || round_up) ? 1 : 0);
    }
    int exp = e10 + removed;
    while (out % 10 == 0) {
        out /= 10;
        ++exp;
    }
    return Decimal{out, exp};
}

MB_TEXT_FN int decimal_length(uint64_t v) {
    int n = 1;
    while (v >= 10) {
        v /= 10;
        ++n;
    }
    return n;
}

enum Kind { FINITE, ZERO, INF, NAN_ };

struct Token {
    Kind kind;
    bool neg;
    bool plain;
    int olen;            // digits of d.digits
    Decimal d;
};

MB_TEXT_FN Token classify(uint64_t bits, const uint64_t* pow5, const uint64_t* pow5_inv) {
    Token t{};
    t.neg = (bits >> 63) != 0;
    const uint64_t mag = bits & 0x7fffffffffffffffull;
    if (mag >= 0x7ff0000000000000ull) {
        t.kind = mag == 0x7ff0000000000000ull ? INF : NAN_;
        return t;
    }
    if (mag == 0) {
        t.kind = ZERO;
        return t;
    }
    t.kind = FINITE;
    t.plain = mag >= PLAIN_LO_BITS && mag < PLAIN_HI_BITS;
    t.d = shortest(mag, pow5, pow5_inv);
    t.olen = decimal_length(t.d.digits);
    return t;
}

// The length of the token of t.
MB_TEXT_FN int token_length(const Token& t) {
    switch (t.kind) {
    case NAN_: return 3;
    case INF: return t.neg ? 9 : 8;
    case ZERO: return t.neg ? 4 : 3;
    default: break;
    }
    const int sci = t.d.exp + t.olen - 1;                               // exponent of the leading digit
    int n = t.neg ? 1 : 0;
    if (t.plain) {
        if (sci >= 0) {
            const int frac = t.olen - (sci + 1);
            n += (sci + 1) + 1 + (frac > 0 ? frac : 1);
        } else {
            n += 2 + (-sci - 1) + t.olen;
        }
    } else {
        const int a = sci < 0 ? -sci : sci;
        n += 2 + (t.olen > 1 ? t.olen - 1 : 1) + 1 + (sci < 0 ? 1 : 0) + (a >= 100 ? 3 : a >= 10 ? 2 : 1);
    }
    return n;
}

// Writes the token of t at out (token_length(t) bytes) and returns its length.
MB_TEXT_FN int write_token(const Token& t, char* out) {
    int n = 0;
    if (t.kind == NAN_) {
        out[0] = 'N'; out[1] = 'a'; out[2] = 'N';
        return 3;
    }
    if (t.neg) out[n++] = '-';
    if (t.kind == INF) {
        const char* s = "Infinity";
        for (int i = 0; i < 8; ++i) out[n++] = s[i];
        return n;
    }
    if (t.kind == ZERO) {
        out[n++] = '0'; out[n++] = '.'; out[n++] = '0';
        return n;
    }
    // the fixed characters first, then the digits from the last one back, each straight to its place
    char* d = out + n;                                                  // where the first digit goes
    const int sci = t.d.exp + t.olen - 1;
    int point;                                                          // digits before the point, sci notation: 1
    if (t.plain && sci < 0) {
        d[0] = '0';
        d[1] = '.';
        for (int i = 0; i < -sci - 1; ++i) d[2 + i] = '0';
        d += 1 - sci;
        point = t.olen;                                                 // no point among the digits
        n += 1 - sci + t.olen;
    } else {
        point = t.plain ? sci + 1 : 1;
        if (t.olen <= point) {                                          // x.0 / x000.0: zeros up to the point, one after
            for (int i = t.olen; i < point; ++i) d[i] = '0';
            d[point] = '.';
            d[point + 1] = '0';
            n += point + 2;
        } else {
            d[point] = '.';
            n += t.olen + 1;
        }
    }
    uint64_t v = t.d.digits;
    for (int i = t.olen - 1; i >= 0; --i) {
        d[i < point ? i : i + 1] = (char)('0' + v % 10);
        v /= 10;
    }
    if (t.plain) return n;
    out[n++] = 'E';
    int a = sci;
    if (a < 0) {
        out[n++] = '-';
        a = -a;
    }
    if (a >= 100) out[n++] = (char)('0' + a / 100);
    if (a >= 10) out[n++] = (char)('0' + a / 10 % 10);
    out[n++] = (char)('0' + a % 10);
    return n;
}

// Long.toString: the length of v's decimal, and its bytes at out.
MB_TEXT_FN int long_length(int64_t v) {
    const uint64_t a = v < 0 ? 0 - (uint64_t)v : (uint64_t)v;
    return (v < 0 ? 1 : 0) + decimal_length(a);
}

MB_TEXT_FN int write_long(int64_t v, char* out) {
    const uint64_t a = v < 0 ? 0 - (uint64_t)v : (uint64_t)v;
    const int n = long_length(v);
    if (v < 0) out[0] = '-';
    uint64_t x = a;
    for (int i = n - 1; i >= (v < 0 ? 1 : 0); --i) {
        out[i] = (char)('0' + x % 10);
        x /= 10;
    }
    return n;
}

}  // namespace text
}  // namespace mb

#if defined(__CUDACC__)
// The device writer (text.cu), for the C ABI.
#include <cstdio>
#include <cuda_runtime.h>

namespace mb {

// One view in file order.  ids != null: a row shard, row by row, line `id:DenseVector(v, v)` per row with ids[r] (device
// int64); else a block, column by column, one line `block_row-block_col-rows-cols:v,v`.
struct TextSegment {
    const void* data;        // element (0, 0)
    long long rs, cs;        // element (r, c) is data[r * rs + c * cs]
    int rows, cols, dtype;   // dtype: MB_F64 / MB_F32 / MB_BF16
    const long long* ids;
    int block_row, block_col;
};

// Where the text goes: kernels run on `stream`, device-to-host copies on `copy_stream`; four events of the caller's.
struct TextIo {
    cudaStream_t stream, copy_stream;
    cudaEvent_t events[4];
    FILE* file;
};

// Writes the segments' lines, in order, to io.file.  host_ids[i]: segment i's row ids on the host (rows only).  Two
// launches per chunk of at most MB_TEXT_CHUNK_VALUES values; segments without values are formatted on the host.  A
// failed file write stops the work and sets *io_errno.  Blocking; every temporary is released before it returns.
cudaError_t save_text(const TextSegment* segs, const long long* const* host_ids, int count, const TextIo& io, int* io_errno);

}  // namespace mb
#endif
