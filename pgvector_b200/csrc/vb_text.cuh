// vb_text.cuh -- device text primitives of the type I/O (vb_text.cu): glibc strtof / strtol in the C locale, and
// PostgreSQL's float_to_shortest_decimal_bufn (shortest round-trip digits, %g-style layout at FLT_DIG = 6).
#pragma once

#include <stdint.h>

namespace vb {
namespace text {

// vector_isspace (src/vector.c:145-157), also glibc isspace in the C locale
__device__ __forceinline__ bool is_space(uint32_t c) { return c == ' ' || (c >= '\t' && c <= '\r'); }
__device__ __forceinline__ bool is_digit(uint32_t c) { return c - '0' < 10u; }
__device__ __forceinline__ uint32_t lower(uint32_t c) { return c | 0x20u; }
__device__ __forceinline__ int hex_value(uint32_t c) {
    if (c - '0' < 10u) return (int)(c - '0');
    const uint32_t l = lower(c);
    return l - 'a' < 6u ? (int)(l - 'a' + 10) : -1;
}

// A literal: bytes s[0 .. len), read as a cstring (a NUL in it ends it; past len reads as NUL)
struct Lit {
    const uint8_t* s;
    int64_t len;
    __device__ __forceinline__ uint32_t at(int64_t i) const { return i < len ? (uint32_t)__ldg(s + i) : 0u; }
};

// 10^q = kPow10Mant[q + 64] * 2^kPow10Exp2[q + 64] rounded down, mantissa in [2^63, 2^64), for q in [-64, 38]: every
// power that can meet a float32 result from at most 19 significant digits (generated with exact rationals)
static __device__ const unsigned long long kPow10Mant[103] = {
    0xa87fea27a539e9a5ull,
    0xd29fe4b18e88640eull,
    0x83a3eeeef9153e89ull,
    0xa48ceaaab75a8e2bull,
    0xcdb02555653131b6ull,
    0x808e17555f3ebf11ull,
    0xa0b19d2ab70e6ed6ull,
    0xc8de047564d20a8bull,
    0xfb158592be068d2eull,
    0x9ced737bb6c4183dull,
    0xc428d05aa4751e4cull,
    0xf53304714d9265dfull,
    0x993fe2c6d07b7fabull,
    0xbf8fdb78849a5f96ull,
    0xef73d256a5c0f77cull,
    0x95a8637627989aadull,
    0xbb127c53b17ec159ull,
    0xe9d71b689dde71afull,
    0x9226712162ab070dull,
    0xb6b00d69bb55c8d1ull,
    0xe45c10c42a2b3b05ull,
    0x8eb98a7a9a5b04e3ull,
    0xb267ed1940f1c61cull,
    0xdf01e85f912e37a3ull,
    0x8b61313bbabce2c6ull,
    0xae397d8aa96c1b77ull,
    0xd9c7dced53c72255ull,
    0x881cea14545c7575ull,
    0xaa242499697392d2ull,
    0xd4ad2dbfc3d07787ull,
    0x84ec3c97da624ab4ull,
    0xa6274bbdd0fadd61ull,
    0xcfb11ead453994baull,
    0x81ceb32c4b43fcf4ull,
    0xa2425ff75e14fc31ull,
    0xcad2f7f5359a3b3eull,
    0xfd87b5f28300ca0dull,
    0x9e74d1b791e07e48ull,
    0xc612062576589ddaull,
    0xf79687aed3eec551ull,
    0x9abe14cd44753b52ull,
    0xc16d9a0095928a27ull,
    0xf1c90080baf72cb1ull,
    0x971da05074da7beeull,
    0xbce5086492111aeaull,
    0xec1e4a7db69561a5ull,
    0x9392ee8e921d5d07ull,
    0xb877aa3236a4b449ull,
    0xe69594bec44de15bull,
    0x901d7cf73ab0acd9ull,
    0xb424dc35095cd80full,
    0xe12e13424bb40e13ull,
    0x8cbccc096f5088cbull,
    0xafebff0bcb24aafeull,
    0xdbe6fecebdedd5beull,
    0x89705f4136b4a597ull,
    0xabcc77118461cefcull,
    0xd6bf94d5e57a42bcull,
    0x8637bd05af6c69b5ull,
    0xa7c5ac471b478423ull,
    0xd1b71758e219652bull,
    0x83126e978d4fdf3bull,
    0xa3d70a3d70a3d70aull,
    0xccccccccccccccccull,
    0x8000000000000000ull,
    0xa000000000000000ull,
    0xc800000000000000ull,
    0xfa00000000000000ull,
    0x9c40000000000000ull,
    0xc350000000000000ull,
    0xf424000000000000ull,
    0x9896800000000000ull,
    0xbebc200000000000ull,
    0xee6b280000000000ull,
    0x9502f90000000000ull,
    0xba43b74000000000ull,
    0xe8d4a51000000000ull,
    0x9184e72a00000000ull,
    0xb5e620f480000000ull,
    0xe35fa931a0000000ull,
    0x8e1bc9bf04000000ull,
    0xb1a2bc2ec5000000ull,
    0xde0b6b3a76400000ull,
    0x8ac7230489e80000ull,
    0xad78ebc5ac620000ull,
    0xd8d726b7177a8000ull,
    0x878678326eac9000ull,
    0xa968163f0a57b400ull,
    0xd3c21bcecceda100ull,
    0x84595161401484a0ull,
    0xa56fa5b99019a5c8ull,
    0xcecb8f27f4200f3aull,
    0x813f3978f8940984ull,
    0xa18f07d736b90be5ull,
    0xc9f2c9cd04674edeull,
    0xfc6f7c4045812296ull,
    0x9dc5ada82b70b59dull,
    0xc5371912364ce305ull,
    0xf684df56c3e01bc6ull,
    0x9a130b963a6c115cull,
    0xc097ce7bc90715b3ull,
    0xf0bdc21abb48db20ull,
    0x96769950b50d88f4ull};
static __device__ const short kPow10Exp2[103] = {-276, -273, -269, -266, -263, -259, -256, -253, -250, -246, -243, -240, -236, -233, -230, -226, -223, -220, -216, -213, -210, -206, -203, -200, -196, -193, -190, -186, -183, -180, -176, -173, -170, -166, -163, -160, -157, -153, -150, -147, -143, -140, -137, -133, -130, -127, -123, -120, -117, -113, -110, -107, -103, -100, -97, -93, -90, -87, -83, -80, -77, -73, -70, -67, -63, -60, -57, -54, -50, -47, -44, -40, -37, -34, -30, -27, -24, -20, -17, -14, -10, -7, -4, 0, 3, 6, 10, 13, 16, 20, 23, 26, 30, 33, 36, 39, 43, 46, 49, 53, 56, 59, 63};


// exponent digits saturate here: with a token's dropped digits it still sums exactly in int64
constexpr int64_t kExpSat = 1000000000000000000ll / 10;
// the exact float powers of ten of the fast path
static __constant__ float kTens[11] = {1e0f, 1e1f, 1e2f, 1e3f, 1e4f, 1e5f, 1e6f, 1e7f, 1e8f, 1e9f, 1e10f};

// ------------------------------------------------------------------ small fixed-width unsigned integers (exact paths)
template <int N>
struct Big {
    uint32_t w[N];   // little-endian limbs
    __device__ __forceinline__ void set(uint64_t v) {
#pragma unroll
        for (int i = 0; i < N; ++i) w[i] = 0;
        w[0] = (uint32_t)v;
        w[1] = (uint32_t)(v >> 32);
    }
    __device__ __forceinline__ void mul_add(uint32_t m, uint32_t a) {
        uint64_t carry = a;
#pragma unroll
        for (int i = 0; i < N; ++i) {
            const uint64_t t = (uint64_t)w[i] * m + carry;
            w[i] = (uint32_t)t;
            carry = t >> 32;
        }
    }
    __device__ void mul_pow5(int k) {
        while (k >= 13) { mul_add(1220703125u, 0); k -= 13; }   // 5^13
        uint32_t p = 1;
        while (k-- > 0) p *= 5;
        if (p != 1) mul_add(p, 0);
    }
    __device__ void shl(int k) {
        const int limbs = k >> 5, bits = k & 31;
        for (int i = N - 1; i >= 0; --i) {
            const int j = i - limbs;
            uint32_t v = j >= 0 ? w[j] << bits : 0u;
            if (bits && j - 1 >= 0) v |= w[j - 1] >> (32 - bits);
            w[i] = v;
        }
    }
};
template <int N>
__device__ int big_cmp(const Big<N>& a, const Big<N>& b) {
    for (int i = N - 1; i >= 0; --i)
        if (a.w[i] != b.w[i]) return a.w[i] < b.w[i] ? -1 : 1;
    return 0;
}
// sign of a * 5^a5 * 2^a2 - b * 5^b5 * 2^b2 (a5, b5 >= 0)
template <int N>
__device__ int scaled_cmp(Big<N>& A, int a5, int a2, Big<N>& B, int b5, int b2) {
    A.mul_pow5(a5);
    B.mul_pow5(b5);
    if (a2 > b2) A.shl(a2 - b2);
    else if (b2 > a2) B.shl(b2 - a2);
    return big_cmp(A, B);
}

// ------------------------------------------------------------------ strtof
struct FloatParse {
    float v;
    int64_t end;     // one past the last byte read; == the start position when nothing was converted
    bool erange;     // glibc's errno == ERANGE: an infinite result from a finite token, or 0 from non-zero digits
};

// value = m * 2^e2 (+ something below when sticky), rounded to nearest even into float32; m != 0
__device__ __forceinline__ FloatParse round_binary(uint64_t m, int e2, bool sticky, bool neg) {
    const int lz = __clzll((long long)m);
    m <<= lz;
    e2 -= lz;                              // m in [2^63, 2^64): value in [2^(e2+63), 2^(e2+64))
    const int E = e2 + 63;                 // binary exponent of the leading bit
    const int keep = E >= -126 ? 24 : E + 150;
    FloatParse r{0.f, 0, false};
    uint32_t bits;
    if (keep < 0) {
        bits = 0;                          // below half of the least subnormal
    } else {
        const int shift = 64 - keep;       // 40 .. 64
        uint64_t q = shift == 64 ? 0 : m >> shift;
        const uint64_t rem = shift == 64 ? m : m << keep;      // the dropped bits, left-aligned
        const uint64_t half = 1ull << 63;
        if (rem > half || (rem == half && (sticky || (q & 1)))) ++q;
        if (E >= -126) {
            int ee = E;
            if (q >> 24) { q >>= 1; ++ee; }
            if (ee > 127) {
                r.v = neg ? -__int_as_float(0x7f800000) : __int_as_float(0x7f800000);
                r.erange = true;
                return r;
            }
            bits = ((uint32_t)(ee + 127) << 23) | ((uint32_t)q & 0x7fffffu);
        } else {
            bits = (uint32_t)q;            // subnormal; 2^23 is the least normal's encoding
        }
    }
    if (bits == 0) r.erange = true;
    r.v = __int_as_float((int)(bits | (neg ? 0x80000000u : 0u)));
    return r;
}

// The significant digits of a decimal literal from its first one (at p), skipping the decimal point
struct TextDigits {
    Lit L;
    int64_t p;
    __device__ __forceinline__ uint32_t next() {
        while (!is_digit(L.at(p))) ++p;
        return L.at(p++) - '0';
    }
};

// The exact decision of a decimal between two adjacent floats: its nd significant digits from D (D.next() yields them
// in order), value = digits * 10^q10 where q10 is the exponent of the last digit.  Returns the sign of
// value - (2c + 1) * 2^(h2).  Only the first 120 significant digits are exact; any non-zero digit after them is a
// sticky excess (a float32 halfway point has at most 113).
template <class Digits>
__device__ __noinline__ int decimal_vs_halfway(Digits D, int64_t nd, int64_t q10, uint64_t c, int h2) {
    Big<16> A, H;
    A.set(0);
    int64_t taken = 0;
    bool sticky = false;
    for (int64_t i = 0; i < nd; ++i) {
        const uint32_t v = D.next();
        if (taken < 120) { A.mul_add(10, v); ++taken; }
        else if (v != 0) sticky = true;
    }
    const int q = (int)(q10 + (nd - taken));   // within [-190, 40] for a value near a float32
    H.set(2 * c + 1);
    int s = scaled_cmp(A, q > 0 ? q : 0, q, H, q < 0 ? -q : 0, h2);
    if (s == 0 && sticky) s = 1;
    return s;
}

// The float32 nearest a decimal (ties to even), with glibc strtof's ERANGE: w = its first `kept` (<= 19) significant
// digits, value ~ w * 10^scale, trunc = a non-zero digit after them; nd = its significant digits in all, which D yields
// in order for the exact decision near a halfway point.  w == 0 is a zero.  end is not set.  The one copy of the
// decimal -> float32 decision: strtof of a literal (parse_float4) and numeric_float4 (vb_numeric.cuh).
template <class Digits>
__device__ __forceinline__ FloatParse decimal_to_float(uint64_t w, int kept, int64_t nd, int64_t scale, bool trunc, bool neg,
                                                       Digits D) {
    FloatParse r{0.f, 0, false};
    if (w == 0) { r.v = neg ? -0.f : 0.f; return r; }
    if (scale > 38) {
        r.v = neg ? -__int_as_float(0x7f800000) : __int_as_float(0x7f800000);
        r.erange = true;
        return r;
    }
    if (scale < -64) { r.v = neg ? -0.f : 0.f; r.erange = true; return r; }
    // exact fast path: w and 10^|scale| both exact in float, one rounding
    if (!trunc && w <= (1u << 24) && scale >= -10 && scale <= 10) {
        const float fw = (float)w;
        r.v = scale >= 0 ? __fmul_rn(fw, kTens[scale]) : __fdiv_rn(fw, kTens[-scale]);
        if (neg) r.v = -r.v;
        return r;
    }
    // one 64 x 64-bit product against the truncated power: the high word is at most 19 units below the exact value
    // (a truncated power, a truncated mantissa), so only a product within that distance of a halfway point is undecided
    const int lz = __clzll((long long)w);
    const uint64_t W = w << lz;
    const uint64_t T = kPow10Mant[scale + 64];
    uint64_t hi = __umul64hi(W, T);
    const int e2 = kPow10Exp2[scale + 64] + 64 - lz;        // value ~ hi * 2^e2
    const int msb = 63 - __clzll((long long)hi);
    const int E = msb + e2;
    const int keep = E >= -126 ? 24 : E + 150;
    if (keep == -1) {
        // within a factor of two below 2^-150, half the least subnormal (or at it, when hi fell short of a power
        // of two): decided exactly between 0 and 2^-149
        const int s = decimal_vs_halfway(D, nd, scale - (nd - kept), 0, -150);
        if (s <= 0) { r.v = neg ? -0.f : 0.f; r.erange = true; return r; }
        r.v = __int_as_float((int)(1u | (neg ? 0x80000000u : 0u)));
        return r;
    }
    if (keep >= 0) {
        const int shift = msb + 1 - keep;                   // >= 39
        const uint64_t rem = shift >= 64 ? hi : hi & ((1ull << shift) - 1);
        const uint64_t half = 1ull << (shift - 1);
        if (rem + 64 >= half && rem <= half + 1) {
            const uint64_t c = shift >= 64 ? 0 : hi >> shift;
            const int s = decimal_vs_halfway(D, nd, scale - (nd - kept), c, e2 + shift - 1);
            // decide exactly: c below, c + 1 above, the even one on a tie
            const bool up = s > 0 || (s == 0 && (c & 1));
            if (c == 0 && !up) { r.v = neg ? -0.f : 0.f; r.erange = true; return r; }
            return round_binary((c + (up ? 1 : 0)) << 1, e2 + shift - 1, false, neg);   // exact: kept as is
        }
    }
    return round_binary(hi, e2, true, neg);
}

// glibc strtof from position p of L in the C locale
static __device__ FloatParse parse_float4(Lit L, int64_t p0) {
    FloatParse r{0.f, p0, false};
    int64_t p = p0;
    while (is_space(L.at(p))) ++p;
    bool neg = false;
    if (L.at(p) == '+' || L.at(p) == '-') { neg = L.at(p) == '-'; ++p; }
    const uint32_t c0 = lower(L.at(p));
    if (c0 == 'i') {
        if (lower(L.at(p + 1)) == 'n' && lower(L.at(p + 2)) == 'f') {
            int64_t e = p + 3;
            const char* rest = "inity";
            int k = 0;
            while (k < 5 && lower(L.at(e + k)) == (uint32_t)rest[k]) ++k;
            if (k == 5) e += 5;
            r.v = neg ? -__int_as_float(0x7f800000) : __int_as_float(0x7f800000);
            r.end = e;
        }
        return r;
    }
    if (c0 == 'n') {
        if (lower(L.at(p + 1)) == 'a' && lower(L.at(p + 2)) == 'n') {
            int64_t e = p + 3;
            if (L.at(e) == '(') {
                int64_t q = e + 1;
                for (;;) {
                    const uint32_t ch = L.at(q);
                    if (is_digit(ch) || lower(ch) - 'a' < 26u || ch == '_') ++q;
                    else break;
                }
                if (L.at(q) == ')') e = q + 1;
            }
            r.v = __int_as_float(neg ? (int)0xffc00000 : 0x7fc00000);
            r.end = e;
        }
        return r;
    }
    // hexadecimal: "0x" followed by a hex digit, or by '.' and a hex digit; otherwise "0" is the token
    if (L.at(p) == '0' && lower(L.at(p + 1)) == 'x' &&
        (hex_value(L.at(p + 2)) >= 0 || (L.at(p + 2) == '.' && hex_value(L.at(p + 3)) >= 0))) {
        int64_t q = p + 2;
        uint64_t m = 0;
        int64_t e2 = 0;           // dropped digits and the exponent, summed without bound
        bool sticky = false, seen_point = false;
        for (;; ++q) {
            const uint32_t ch = L.at(q);
            if (ch == '.' && !seen_point) { seen_point = true; continue; }
            const int h = hex_value(ch);
            if (h < 0) break;
            if (m >> 60) {                 // 16 hex digits kept; the rest only counts as non-zero or as scale
                if (h) sticky = true;
                if (!seen_point) e2 += 4;
            } else {
                m = (m << 4) | (uint64_t)h;
                if (seen_point) e2 -= 4;
            }
        }
        if (lower(L.at(q)) == 'p') {
            int64_t t = q + 1;
            bool eneg = false;
            if (L.at(t) == '+' || L.at(t) == '-') { eneg = L.at(t) == '-'; ++t; }
            if (is_digit(L.at(t))) {
                int64_t x = 0;
                while (is_digit(L.at(t))) { if (x < kExpSat) x = x * 10 + (int64_t)(L.at(t) - '0'); ++t; }
                e2 += eneg ? -x : x;
                q = t;
            }
        }
        r.end = q;
        if (m == 0) { r.v = neg ? -0.f : 0.f; return r; }
        // past +-2^20 the result is 0 or infinite whatever the digits; the clamp keeps the int arithmetic exact
        FloatParse f = round_binary(m, (int)(e2 < -(1 << 20) ? -(1 << 20) : e2 > (1 << 20) ? (1 << 20) : e2), sticky, neg);
        f.end = q;
        return f;
    }
    // decimal
    int64_t q = p, d0 = -1, nd = 0;
    uint64_t w = 0;
    int kept = 0;
    int64_t scale = 0;                     // value = w * 10^scale (+ truncated digits), summed without bound
    bool any = false, seen_point = false, trunc = false;
    for (;; ++q) {
        const uint32_t ch = L.at(q);
        if (ch == '.' && !seen_point) { seen_point = true; continue; }
        if (!is_digit(ch)) break;
        any = true;
        if (ch == '0' && d0 < 0) { if (seen_point) --scale; continue; }
        if (d0 < 0) d0 = q;
        ++nd;
        if (kept < 19) {
            w = w * 10 + (ch - '0');
            ++kept;
            if (seen_point) --scale;
        } else {
            if (ch != '0') trunc = true;
            if (!seen_point) ++scale;
        }
    }
    if (!any) return r;                    // "", ".", "-", "e5": no conversion
    if (lower(L.at(q)) == 'e') {
        int64_t t = q + 1;
        bool eneg = false;
        if (L.at(t) == '+' || L.at(t) == '-') { eneg = L.at(t) == '-'; ++t; }
        if (is_digit(L.at(t))) {
            int64_t x = 0;
            while (is_digit(L.at(t))) { if (x < kExpSat) x = x * 10 + (int64_t)(L.at(t) - '0'); ++t; }
            scale += eneg ? -x : x;
            q = t;
        }
    }
    FloatParse f = decimal_to_float(w, kept, nd, scale, trunc, neg, TextDigits{L, d0});
    f.end = q;
    return f;
}

// glibc strtol(base 10) from position p, then clamped to [lo, hi]; end == p0 when nothing was converted
struct IntParse {
    int64_t v;
    int64_t end;
};
__device__ __forceinline__ IntParse parse_long(Lit L, int64_t p0, int64_t lo, int64_t hi) {
    int64_t p = p0;
    while (is_space(L.at(p))) ++p;
    bool neg = false;
    if (L.at(p) == '+' || L.at(p) == '-') { neg = L.at(p) == '-'; ++p; }
    if (!is_digit(L.at(p))) return IntParse{0, p0};
    int64_t v = 0;
    while (is_digit(L.at(p))) {
        if (v < (int64_t)1 << 40) v = v * 10 + (int64_t)(L.at(p) - '0');
        ++p;
    }
    v = neg ? -v : v;
    return IntParse{v < lo ? lo : v > hi ? hi : v, p};
}

// ------------------------------------------------------------------ float_to_shortest_decimal_bufn
// sign of c * 10^t - n * 2^s (c, n < 2^40)
static __device__ __noinline__ int dec_vs_bin(uint64_t c, int t, uint64_t n, int s) {
    Big<8> A, B;
    A.set(c);
    B.set(n);
    return scaled_cmp(A, t > 0 ? t : 0, t, B, t < 0 ? -t : 0, s);
}

__device__ __forceinline__ int put_uint(char* o, uint64_t v) {
    char tmp[20];
    int k = 0;
    do { tmp[k++] = (char)('0' + v % 10); v /= 10; } while (v);
    for (int i = 0; i < k; ++i) o[i] = tmp[k - 1 - i];
    return k;
}

// The shortest decimal that strtof reads back as f, the nearest to f among those (the even digit on a tie); fixed notation when the first
// digit's exponent X is in [-4, 6), else d[.ddd]e+-XX.  Writes at most 15 bytes to o, returns the count.
static __device__ int format_float4(float f, char* o) {
    const uint32_t u = (uint32_t)__float_as_int(f);
    int n = 0;
    const uint32_t ex = (u >> 23) & 0xff, fr = u & 0x7fffff;
    if (ex == 0xff) {
        if (fr) { o[0] = 'N'; o[1] = 'a'; o[2] = 'N'; return 3; }
        if (u >> 31) o[n++] = '-';
        const char* s = "Infinity";
        for (int i = 0; i < 8; ++i) o[n++] = s[i];
        return n;
    }
    if (u >> 31) o[n++] = '-';
    if (ex == 0 && fr == 0) { o[n++] = '0'; return n; }
    const uint64_t m = ex ? (fr | 0x800000u) : fr;
    const int e = ex ? (int)ex - 150 : -149;
    // the round-trip interval: reads back as f when strictly inside, and on its ends when m is even
    const bool incl = (m & 1) == 0;
    const bool tight_below = fr == 0 && ex > 1;
    const uint64_t lo_n = tight_below ? 4 * m - 1 : 2 * m - 1;
    const int lo_s = tight_below ? e - 2 : e - 1;
    const double v = (double)fabsf(f);
    int X = (int)floor(log10(v));
    while (dec_vs_bin(1, X + 1, m, e) <= 0) ++X;
    while (dec_vs_bin(1, X, m, e) > 0) --X;
    // binary search for the least digit count p whose floor or ceiling neighbour lies in the interval; a p-digit
    // decimal in it stays one at p + 1 digits, so the property is monotone in p
    int plo = 1, phi = 9;
    uint64_t best = 0;
    int best_t = 0;
    while (plo <= phi) {
        const int p = (plo + phi) >> 1;
        const int t = X - p + 1;
        uint64_t d = (uint64_t)floor(v / exp10((double)t));
        while (dec_vs_bin(d + 1, t, m, e) <= 0) ++d;
        while (d > 0 && dec_vs_bin(d, t, m, e) > 0) --d;
        const bool exact = dec_vs_bin(d, t, m, e) == 0;
        int s_lo = dec_vs_bin(d, t, lo_n, lo_s);
        const bool lo_in = exact || s_lo > 0 || (incl && s_lo == 0);
        int s_hi = dec_vs_bin(d + 1, t, 2 * m + 1, e - 1);
        const bool hi_in = !exact && (s_hi < 0 || (incl && s_hi == 0));
        if (lo_in || hi_in) {
            uint64_t pick = d;
            if (hi_in) {   // the nearer of the two, the even digit on a tie
                const int mid = lo_in ? dec_vs_bin(2 * d + 1, t, m, e + 1) : -1;
                if (mid < 0 || (mid == 0 && (d & 1))) pick = d + 1;
            }
            best = pick;
            best_t = t;
            phi = p - 1;
        } else {
            plo = p + 1;
        }
    }
    // digits of best, then the exponent of the first digit
    while (best % 10 == 0) { best /= 10; ++best_t; }
    char dg[10];
    const int nd = put_uint(dg, best);
    const int XO = best_t + nd - 1;
    if (XO >= -4 && XO < 6) {
        if (XO < 0) {
            o[n++] = '0';
            o[n++] = '.';
            for (int i = 0; i < -XO - 1; ++i) o[n++] = '0';
            for (int i = 0; i < nd; ++i) o[n++] = dg[i];
        } else {
            for (int i = 0; i <= XO; ++i) o[n++] = i < nd ? dg[i] : '0';
            if (nd > XO + 1) {
                o[n++] = '.';
                for (int i = XO + 1; i < nd; ++i) o[n++] = dg[i];
            }
        }
    } else {
        o[n++] = dg[0];
        if (nd > 1) {
            o[n++] = '.';
            for (int i = 1; i < nd; ++i) o[n++] = dg[i];
        }
        o[n++] = 'e';
        int x = XO;
        o[n++] = x < 0 ? '-' : '+';
        if (x < 0) x = -x;
        if (x >= 10) { o[n++] = (char)('0' + x / 10); o[n++] = (char)('0' + x % 10); }
        else { o[n++] = '0'; o[n++] = (char)('0' + x); }
    }
    return n;
}

}  // namespace text
}  // namespace vb
