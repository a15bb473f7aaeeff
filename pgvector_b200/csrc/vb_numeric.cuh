// vb_numeric.cuh -- numeric[] elements of the array casts (vb_ops.cu, vb_sparse.cu): PostgreSQL's numeric_recv checks
// of a numeric_send field and numeric_float4 of its value.  These rules are PostgreSQL core's (src/backend/utils/adt/
// numeric.c: numeric_recv, numeric_out, numeric_float4; float.c: float4in), not pgvector's.
//
// A field is big-endian int16 ndigits, int16 weight, uint16 sign, uint16 dscale, then ndigits base-10000 int16 digits;
// the value is sum(digit[i] * 10000^(weight - i)).  numeric_recv truncates digits past dscale fraction digits and
// numeric_out prints exactly dscale of them, so the value is the decimal those digits spell.  numeric_float4 is
// float4in(numeric_out(x)): glibc strtof of that decimal, an error when strtof sets ERANGE and the result is 0 or
// infinite (a subnormal result is kept); NaN and the infinities map to themselves; zero prints as "0", so it becomes +0
// whatever its sign.
#pragma once

#include <cstdio>
#include <cstdlib>
#include <string>
#include <vector>

#include "vb_common.cuh"
#include "vb_text.cuh"

namespace vb {

// numeric_recv's outcome for one field, in its read order: the first failing read or check
enum { NUM_OK = 0, NUM_SHORT, NUM_SIGN, NUM_SCALE, NUM_DIGIT, NUM_TRAILING, NUM_BAD_OFFSETS };
constexpr uint32_t NUMERIC_POS = 0x0000, NUMERIC_NEG = 0x4000, NUMERIC_NAN = 0xC000, NUMERIC_PINF = 0xD000, NUMERIC_NINF = 0xF000;
constexpr uint32_t NUMERIC_DSCALE_MASK = 0x3FFF;

__host__ __device__ __forceinline__ uint32_t be16(const uint8_t* p) { return ((uint32_t)p[0] << 8) | p[1]; }

// numeric_recv's checks of the field f[0 .. len): reads past the end ("insufficient data left in message"), the sign,
// dscale and each digit as read, then bytes left over (COPY's "incorrect binary data format")
__host__ __device__ inline int numeric_field_check(const uint8_t* f, int64_t len) {
    if (len < 0) return NUM_BAD_OFFSETS;
    if (len < 6) return NUM_SHORT;
    const uint32_t nd = be16(f), sign = be16(f + 4);
    if (!(sign == NUMERIC_POS || sign == NUMERIC_NEG || sign == NUMERIC_NAN || sign == NUMERIC_PINF || sign == NUMERIC_NINF))
        return NUM_SIGN;
    if (len < 8) return NUM_SHORT;
    if ((be16(f + 6) & ~NUMERIC_DSCALE_MASK) != 0) return NUM_SCALE;
    for (uint32_t i = 0; i < nd; ++i) {
        if (len < 8 + 2 * (int64_t)(i + 1)) return NUM_SHORT;
        if (be16(f + 8 + 2 * i) >= 10000) return NUM_DIGIT;   // an int16 below 0 is >= 0x8000 here
    }
    return len > 8 + 2 * (int64_t)nd ? NUM_TRAILING : NUM_OK;
}

// The decimal digits of a numeric from its first significant one: digit k of base-10000 group gi, in order
struct NumericDigits {
    const uint8_t* g;
    uint32_t gi, k;
    __device__ __forceinline__ uint32_t next() {
        const uint32_t d = be16(g + 2 * gi);
        const uint32_t v = (k == 0 ? d / 1000 : k == 1 ? d / 100 : k == 2 ? d / 10 : d) % 10;
        if (++k == 4) { k = 0; ++gi; }
        return v;
    }
};

// numeric_float4 of a field that passed numeric_field_check; erange: float4in's range error
__device__ inline text::FloatParse numeric_float4(const uint8_t* f) {
    const uint32_t nd = be16(f), sign = be16(f + 4), dscale = be16(f + 6);
    const int weight = (int16_t)be16(f + 2);
    text::FloatParse r{0.f, 0, false};
    if (sign == NUMERIC_NAN) { r.v = __int_as_float(0x7fc00000); return r; }
    if (sign == NUMERIC_PINF || sign == NUMERIC_NINF) { r.v = __int_as_float(sign == NUMERIC_PINF ? 0x7f800000 : (int)0xff800000); return r; }
    // digit k of group i has the decimal exponent 4 * (weight - i) + 3 - k; those below -dscale are truncated
    uint64_t w = 0;
    int kept = 0;
    int64_t nsig = 0, e_first = 0;
    bool trunc = false;
    uint32_t gi0 = 0, k0 = 0;
    for (uint32_t i = 0; i < nd; ++i) {
        const int ge = 4 * (weight - (int)i);
        if (ge + 3 < -(int)dscale) break;
        const uint32_t d = be16(f + 8 + 2 * i);
        if (nsig == 0 && d == 0) continue;
        for (uint32_t k = 0; k < 4; ++k) {
            const int e = ge + 3 - (int)k;
            if (e < -(int)dscale) break;
            const uint32_t v = (k == 0 ? d / 1000 : k == 1 ? d / 100 : k == 2 ? d / 10 : d) % 10;
            if (nsig == 0) {
                if (v == 0) continue;
                gi0 = i, k0 = k, e_first = e;
            }
            ++nsig;
            if (kept < 19) { w = w * 10 + v; ++kept; }
            else if (v != 0) trunc = true;
        }
    }
    // zero prints as "0": +0 whatever the sign
    return text::decimal_to_float(w, kept, nsig, e_first - kept + 1, trunc, nsig > 0 && sign == NUMERIC_NEG,
                                  NumericDigits{f + 8, gi0, k0});
}

// One thread per field: field e is bytes[off[e] - base .. off[e + 1] - base).  A malformed field lowers *malformed to
// its number; a good one goes to sink.put(e, value, float4in's range error).
template <class Sink>
__global__ void __launch_bounds__(256) numeric_cast_kernel(const uint8_t* __restrict__ bytes, const int64_t* __restrict__ off, int64_t base,
                                                           int64_t total, Sink sink, unsigned long long* __restrict__ malformed) {
    const int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (e >= total) return;
    const int64_t b = off[e], len = off[e + 1] - b;
    const uint8_t* f = bytes + (b - base);
    if (numeric_field_check(f, len) != NUM_OK) {
        atomicMin(malformed, (unsigned long long)e);
        return;
    }
    const text::FloatParse x = numeric_float4(f);
    sink.put(e, x.v, x.erange);
}

// ---------------------------------------------------------------- host side: the error texts
// numeric_recv's text for a malformed field, as VB_EINVAL naming the field
inline int numeric_field_error(const char* fn, int64_t field, const uint8_t* f, int64_t len) {
    static const char* const text[] = {"", "insufficient data left in message", "invalid sign in external \"numeric\" value",
                                       "invalid scale in external \"numeric\" value", "invalid digit in external \"numeric\" value",
                                       "incorrect binary data format", "offsets must not decrease"};
    set_error("%s: numeric field %lld: %s", fn, (long long)field, text[numeric_field_check(f, len)]);
    return VB_EINVAL;
}

// numeric_out of a finite field that passed numeric_field_check (get_str_from_var after numeric_recv's truncation)
inline std::string numeric_out(const uint8_t* f) {
    const int nd = (int)be16(f), dscale = (int)be16(f + 6);
    int weight = (int16_t)be16(f + 2);
    auto dig = [&](int i) { return i >= 0 && i < nd ? (int)be16(f + 8 + 2 * i) : 0; };
    // the digits numeric_recv keeps (trunc_var to dscale), then make_result's strip of leading zero groups
    int ndk = nd < weight + 1 + (dscale + 3) / 4 ? nd : weight + 1 + (dscale + 3) / 4;
    if (ndk < 0) ndk = 0;
    std::vector<int> d((size_t)ndk);
    for (int i = 0; i < ndk; ++i) d[i] = dig(i);
    if (ndk > 0 && dscale % 4 != 0 && weight + 1 + (dscale + 3) / 4 == ndk) {   // a partly kept last group
        static const int cut[4] = {1, 1000, 100, 10};
        d[ndk - 1] -= d[ndk - 1] % cut[dscale % 4];
    }
    size_t lead = 0;
    while (lead < d.size() && d[lead] == 0) ++lead;
    const bool zero = lead == d.size();
    d.erase(d.begin(), d.begin() + (long)lead);
    weight = zero ? 0 : weight - (int)lead;
    auto g = [&](int i) { return i >= 0 && i < (int)d.size() ? d[i] : 0; };
    std::string s;
    if (!zero && be16(f + 4) == NUMERIC_NEG) s += '-';
    int i = 0;
    if (weight < 0) {
        i = weight + 1;
        s += '0';
    } else {
        for (; i <= weight; ++i) {
            char b[8];
            snprintf(b, sizeof(b), i == 0 ? "%d" : "%04d", g(i));
            s += b;
        }
    }
    if (dscale > 0) {
        s += '.';
        std::string frac;
        for (; (int)frac.size() < dscale; ++i) {
            char b[8];
            snprintf(b, sizeof(b), "%04d", g(i));
            frac += b;
        }
        s += frac.substr(0, (size_t)dscale);
    }
    return s;
}

// float4in's range error for a field numeric_float4 could not convert
inline int numeric_range_error(const uint8_t* f) {
    set_error("\"%s\" is out of range for type real", numeric_out(f).c_str());
    return VB_EINVAL;
}

// numeric_float4 of a finite field on the host, for the halfvec range error's text: float4in's strtof of numeric_out
inline float numeric_float4_host(const uint8_t* f) { return strtof(numeric_out(f).c_str(), nullptr); }

// The offsets of n rows of dim fields (off[0 .. n * dim]) checked on the host: non-decreasing from 0 or more.  Returns
// VB_EINVAL naming the first bad field.
inline int numeric_offsets_check(const char* fn, const int64_t* off, int64_t total, int64_t* out_bad, int dim) {
    VB_REQUIRE(off[0] >= 0, "%s: numeric field offsets must not be negative", fn);
    for (int64_t e = 0; e < total; ++e)
        if (off[e + 1] < off[e]) {
            if (out_bad) *out_bad = e / dim;
            set_error("%s: numeric field %lld: offsets must not decrease", fn, (long long)e);
            return VB_EINVAL;
        }
    return VB_OK;
}

// Whole rows per chunk of the host variants: at most `budget` bytes of fields and offsets, a longer row alone.
// starts[c] is chunk c's first row; starts.back() == n.
inline void numeric_chunks(const int64_t* off, int64_t n, int dim, size_t budget, std::vector<int64_t>& starts) {
    starts.assign(1, 0);
    int64_t r0 = 0;
    for (int64_t r = 0; r < n; ++r) {
        const size_t b = (size_t)(off[(r + 1) * dim] - off[r0 * dim]) + sizeof(int64_t) * (size_t)((r + 1 - r0) * dim + 1);
        if (b > budget && r > r0) {
            starts.push_back(r);
            r0 = r;
        }
    }
    starts.push_back(n);
}

}  // namespace vb
