// vb_ops.cu -- batched row transforms that sit beside the distance path:
//   vb_norm_batch          vector_norm / halfvec l2_norm       (src/vector.c:767-780, src/halfvec.c:703-720)
//   vb_l2_normalize_batch  l2_normalize / halfvec_l2_normalize (src/vector.c:785-819, src/halfvec.c:725-759)
//   vb_binary_quantize_batch  binary_quantize                  (src/vector.c:952-978, src/halfvec.c twin)
//   vb_subvector_batch     subvector                           (src/vector.c:983-1025, src/halfvec.c:939-981)
//   vb_vector_to_halfvec_batch / vb_halfvec_to_vector_batch     the casts between the two
//   vb_arith_batch         + - * (src/vector.c:824-921, src/halfvec.c:766-879)
//   vb_concat_batch        ||    (src/vector.c:928-947, src/halfvec.c:886-903), two column copies
//   vb_array_to_rows_batch integer[] / real[] / double precision[] -> vector / halfvec (src/vector.c:443-512,
//                          src/halfvec.c:442-509)
//   vb_numeric_array_to_rows_batch  numeric[] -> vector / halfvec, the same functions' numeric_float4 branch
// The cosine opclasses normalise every indexed row and the query (src/ivfbuild.c:174-180,
// src/ivfscan.c:222-229, src/hnswutils.c:417-423); norms accumulate in fp64 like the reference.
// One warp per row; HBM bound (row read once, written once).
// Every transform is one launcher over device rows (the *_rows functions); the _dev entry points call it on the
// caller's buffers, the host variants stage the rows in device scratch, call it and copy the result back, so both give
// the same bits.
#include "vb_common.cuh"
#include "vb_numeric.cuh"
#include "vb_typio.cuh"

#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <type_traits>

namespace vb {

template <int ELEM>
__device__ __forceinline__ float load_elem(const uint8_t* row, int i) {
    return ELEM == VB_VECTOR ? reinterpret_cast<const float*>(row)[i] : __half2float(reinterpret_cast<const __half*>(row)[i]);
}

// mode 0: norms only; mode 1: normalise.  in and out may be the same rows (vb_l2_normalize_batch_dev in place): every
// element is read by the lane that writes it, before it writes it, so neither pointer is __restrict__.
template <int ELEM>
__global__ void norm_kernel(const uint8_t* in, size_t in_stride, int64_t n, int dim, int mode, double* __restrict__ norms,
                            uint8_t* out, size_t out_stride, int* __restrict__ overflow) {
    const int64_t r = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) / 32;
    const int lane = threadIdx.x % 32;
    if (r >= n) return;
    const uint8_t* row = in + (size_t)r * in_stride;
    double s = 0.0;
    for (int i = lane; i < dim; i += 32) {
        double x = (double)load_elem<ELEM>(row, i);
        s += x * x;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    const double norm = sqrt(s);
    if (mode == 0) {
        if (lane == 0) norms[r] = norm;
        return;
    }
    uint8_t* orow = out + (size_t)r * out_stride;
    bool inf = false;
    for (int i = lane; i < dim; i += 32) {
        // zero vector stays zero (src/vector.c:804, src/halfvec.c:745)
        if (ELEM == VB_VECTOR) {
            float v = norm > 0 ? (float)((double)load_elem<ELEM>(row, i) / norm) : 0.f;
            inf |= isinf(v);
            reinterpret_cast<float*>(orow)[i] = v;
        } else {
            // quotient in double, narrowed to float, then RNE to half (src/halfvec.c:748)
            __half h = norm > 0 ? __float2half_rn((float)((double)load_elem<ELEM>(row, i) / norm)) : __float2half_rn(0.f);
            inf |= __hisinf(h) != 0;
            reinterpret_cast<__half*>(orow)[i] = h;
        }
    }
    if (inf) atomicExch(overflow, 1);
}

// bit i = x[i] > 0, MSB first (src/vector.c:966-975); one thread per output byte
template <int ELEM>
__global__ void binary_quantize_kernel(const uint8_t* __restrict__ in, size_t in_stride, int64_t n, int dim, uint8_t* __restrict__ out,
                                       size_t out_stride) {
    const int nb = (dim + 7) / 8;
    const int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    const int64_t r = t / nb;
    const int b = (int)(t % nb);
    if (r >= n) return;
    const uint8_t* row = in + (size_t)r * in_stride;
    uint8_t v = 0;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        int i = b * 8 + j;
        if (i < dim && load_elem<ELEM>(row, i) > 0.f) v |= (uint8_t)(1u << (7 - j));
    }
    out[(size_t)r * out_stride + b] = v;
}

// vector -> halfvec (vector_to_halfvec, src/halfvec.c:540-555): Float4ToHalf = round to nearest even, and a finite value
// that becomes infinite is an error (src/halfutils.h:244-261); the first offender in row-major order is reported
__global__ void to_half_kernel(const float* __restrict__ in, int64_t total, __half* __restrict__ out, unsigned long long* __restrict__ first_bad) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= total) return;
    bool over;
    out[i] = float_to_half_checked(in[i], &over);
    if (over) atomicMin(first_bad, (unsigned long long)i);
}
__global__ void to_float_kernel(const __half* __restrict__ in, int64_t total, float* __restrict__ out) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i < total) out[i] = __half2float(in[i]);
}

// subvector and ||: `words` words of T from word `first` of every input row (`pitch` words apart; 0 repeats one row)
// to word `out_first` of every output row (`out_pitch` words apart).
// 2^lg lanes per row (lg <= 5), so short rows share a warp; consecutive lanes move consecutive words of a row, so a
// warp's loads and stores are contiguous runs.  T is the widest word (2 to 16 bytes) that the row pitches, the offsets,
// the run and both base addresses allow.
template <typename T>
__global__ void subvector_kernel(const T* __restrict__ in, int64_t pitch, int64_t first, int64_t n, int words, int lg,
                                 T* __restrict__ out, int64_t out_pitch, int64_t out_first) {
    const int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    const int64_t r = t >> lg;
    if (r >= n) return;
    const T* src = in + r * pitch + first;
    T* dst = out + r * out_pitch + out_first;
    for (int j = (int)(t & ((1 << lg) - 1)); j < words; j += 1 << lg) dst[j] = src[j];
}

// ---------------------------------------------------------------- + - * and the array casts
// The first data error of a batch is the one the reference's row-by-row execution raises: the lowest row, then within
// the row the first check its loops reach.  Every offender lowers one 64-bit key with atomicMin:
//   key = ((row * 2 + pass) * dim + element) * 4 + kind
// pass 0 / 1 are the two checking loops of array_to_halfvec (conversion, then CheckElement); the other functions have
// one.  A batch with no offender leaves the key at ~0.
enum { ERR_OVERFLOW = 0, ERR_UNDERFLOW = 1 };             // + - *: float_overflow_error / float_underflow_error
enum { ERR_RANGE = 0, ERR_NAN = 1, ERR_INF = 2, ERR_REAL = 3 };   // casts: Float4ToHalf, CheckElement, float4in
constexpr unsigned long long NO_ERROR = ~0ull;

__device__ __forceinline__ unsigned long long error_key(int64_t row, int pass, int64_t dim, int64_t elem, int kind) {
    return (unsigned long long)(((row * 2 + pass) * dim + elem) * 4 + kind);
}

// element bits of a word: fp32 as uint32_t, binary16 as uint16_t
template <typename W, int ES>
union Elems {
    W w;
    typename std::conditional<ES == 4, uint32_t, uint16_t>::type e[sizeof(W) / ES];
};

// a op b of one element as the reference computes it; *kind = the error its checking loop raises there, or -1.
// vector: fp32 (src/vector.c:824-921); halfvec: Float4ToHalfUnchecked(HalfToFloat4(a) op HalfToFloat4(b))
// (src/halfvec.c:766-879).  _rn intrinsics: one correctly rounded operation, never contracted.
template <int ELEM, int OP>
__device__ __forceinline__ uint32_t arith_elem(uint32_t a, uint32_t b, int* kind) {
    const float x = ELEM == VB_VECTOR ? __uint_as_float(a) : __half2float(__ushort_as_half((unsigned short)a));
    const float y = ELEM == VB_VECTOR ? __uint_as_float(b) : __half2float(__ushort_as_half((unsigned short)b));
    const float r = OP == VB_ADD ? __fadd_rn(x, y) : OP == VB_SUB ? __fsub_rn(x, y) : __fmul_rn(x, y);
    *kind = -1;
    // A NaN result takes the bits the reference gets on x86 (SSE, and F16C for the half conversions), where the GPU would
    // give its one canonical NaN: the first NaN operand, quieted, or the default NaN 0xFFC00000 for an invalid operation
    // such as inf - inf.  The half <-> float conversions keep the payload, so for halfvec that is the half operand | 0x200.
    if (ELEM == VB_VECTOR) {
        if (isnan(r)) return isnan(x) ? a | 0x400000u : isnan(y) ? b | 0x400000u : 0xFFC00000u;
        if (isinf(r)) *kind = ERR_OVERFLOW;
        else if (OP == VB_MUL && r == 0.f && !(x == 0.f || y == 0.f)) *kind = ERR_UNDERFLOW;
        return __float_as_uint(r);
    }
    if (isnan(r)) return isnan(x) ? a | 0x200u : isnan(y) ? b | 0x200u : 0xFE00u;
    const uint32_t h = __half_as_ushort(__float2half_rn(r));
    // HalfIsInf / HalfIsZero (src/halfutils.h:37-57) on the bits, so -0 is zero
    if ((h & 0x7FFF) == 0x7C00) *kind = ERR_OVERFLOW;
    else if (OP == VB_MUL && (h & 0x7FFF) == 0 && !((a & 0x7FFF) == 0 || (b & 0x7FFF) == 0)) *kind = ERR_UNDERFLOW;
    return h;
}

// out row r = a row r op b row r, in words of W; a broadcast operand has a row pitch of 0.  Lanes per row as in
// subvector_kernel.  out may be a or b (in place): every word is read by the thread that writes it, before it writes it,
// so no pointer is __restrict__.
template <typename W, int ELEM, int OP>
__global__ void arith_kernel(const W* a, int64_t pitch_a, const W* b, int64_t pitch_b, int64_t n, int dim, int words, int lg,
                             W* out, unsigned long long* __restrict__ first_bad) {
    constexpr int ES = ELEM == VB_VECTOR ? 4 : 2;
    constexpr int V = sizeof(W) / ES;
    const int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    const int64_t r = t >> lg;
    if (r >= n) return;
    const W* ra = a + r * pitch_a;
    const W* rb = b + r * pitch_b;
    W* ro = out + r * (int64_t)words;
    int bad = -1, bad_kind = 0;   // the first offending element this thread sees (its words ascend)
    for (int j = (int)(t & ((1 << lg) - 1)); j < words; j += 1 << lg) {
        Elems<W, ES> x, y, z;
        x.w = ra[j];
        y.w = rb[j];
#pragma unroll
        for (int v = 0; v < V; ++v) {
            int kind;
            z.e[v] = arith_elem<ELEM, OP>(x.e[v], y.e[v], &kind);
            if (kind >= 0 && bad < 0) {
                bad = j * V + v;
                bad_kind = kind;
            }
        }
        ro[j] = z.w;
    }
    if (bad >= 0) atomicMin(first_bad, error_key(r, 0, dim, bad, bad_kind));
}

// four consecutive source elements, 16-byte aligned
__device__ __forceinline__ void load4(const int32_t* p, int32_t s[4]) {
    const int4 u = *reinterpret_cast<const int4*>(p);
    s[0] = u.x, s[1] = u.y, s[2] = u.z, s[3] = u.w;
}
__device__ __forceinline__ void load4(const float* p, float s[4]) {
    const float4 u = *reinterpret_cast<const float4*>(p);
    s[0] = u.x, s[1] = u.y, s[2] = u.z, s[3] = u.w;
}
__device__ __forceinline__ void load4(const double* p, double s[4]) {
    const double2 u = reinterpret_cast<const double2*>(p)[0], w = reinterpret_cast<const double2*>(p)[1];
    s[0] = u.x, s[1] = u.y, s[2] = w.x, s[3] = w.y;
}
__device__ __forceinline__ float to_float4(int32_t x) { return __int2float_rn(x); }
__device__ __forceinline__ float to_float4(float x) { return x; }
__device__ __forceinline__ float to_float4(double x) { return __double2float_rn(x); }

// array_to_vector / array_to_halfvec of packed source rows (src/vector.c:443-512, src/halfvec.c:442-509): (float) of the
// int32 or double (round to nearest even), as is for float4; halfvec then Float4ToHalf.  V consecutive elements of the
// flattened rows per thread (V = 4 where both base addresses allow whole words, else 1); the last thread takes the
// tail.  A thread's elements may belong to two rows, so each offender makes its own key.
template <typename S, int ELEM, int V>
__global__ void array_cast_kernel(const S* __restrict__ in, int64_t total, int dim, void* __restrict__ out,
                                  unsigned long long* __restrict__ first_bad) {
    const int64_t i0 = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) * V;
    if (i0 >= total) return;
    const bool whole = total - i0 >= V;
    S s[V];
    if (V == 4 && whole) {
        load4(in + i0, s);
    } else {
#pragma unroll
        for (int v = 0; v < V; ++v) s[v] = i0 + v < total ? in[i0 + v] : S(0);
    }
    unsigned long long key = NO_ERROR;
    uint32_t o[V];   // result bits
#pragma unroll
    for (int v = 0; v < V; ++v) {
        const float f = to_float4(s[v]);
        const int64_t i = i0 + v;
        int pass = 0, kind = -1;
        if (ELEM == VB_VECTOR) {
            o[v] = __float_as_uint(f);
            // CheckElement (src/vector.c:112-123), after the whole row is converted
            if (isnan(f)) kind = ERR_NAN;
            else if (isinf(f)) kind = ERR_INF;
        } else {
            bool over;
            o[v] = __half_as_ushort(float_to_half_checked(f, &over));
            // pass 0: Float4ToHalf; pass 1: CheckElement (src/halfvec.c:113-126), HalfIsNan, then HalfIsInf
            if (over) kind = ERR_RANGE;
            else if ((o[v] & 0x7C00) == 0x7C00) pass = 1, kind = (o[v] & 0x7FFF) != 0x7C00 ? ERR_NAN : ERR_INF;
        }
        if (kind >= 0 && i < total) key = min(key, error_key(i / dim, pass, dim, i % dim, kind));
    }
    if (ELEM == VB_VECTOR) {
        float* dst = (float*)out + i0;
        if (V == 4 && whole) *reinterpret_cast<uint4*>(dst) = make_uint4(o[0], o[1], o[2], o[3]);
        else
#pragma unroll
            for (int v = 0; v < V; ++v)
                if (i0 + v < total) dst[v] = __uint_as_float(o[v]);
    } else {
        __half* dst = (__half*)out + i0;
        if (V == 4 && whole) *reinterpret_cast<uint2*>(dst) = make_uint2(o[0] | o[1] << 16, o[2] | o[3] << 16);
        else
#pragma unroll
            for (int v = 0; v < V; ++v)
                if (i0 + v < total) dst[v] = __ushort_as_half((unsigned short)o[v]);
    }
    if (key != NO_ERROR) atomicMin(first_bad, key);
}

// numeric[] -> vector / halfvec (numeric_cast_kernel's sink): vector stores numeric_float4's value, and its checking
// loop (CheckElement) runs after the whole row is converted, so float4in's range error is pass 0 and NaN / infinity
// pass 1.  halfvec runs numeric_float4 and then Float4ToHalf on each element in turn (pass 0: float4in's range error,
// or the half overflow), then CheckElement (pass 1).
template <int ELEM>
struct NumericRowSink {
    void* out;
    int dim;
    unsigned long long* first_bad;
    __device__ __forceinline__ void put(int64_t e, float f, bool real_range) const {
        const int64_t r = e / dim, i = e - r * dim;
        int pass = 0, kind = -1;
        if (real_range) {
            kind = ERR_REAL;
        } else if (ELEM == VB_VECTOR) {
            reinterpret_cast<float*>(out)[e] = f;
            if (isnan(f)) pass = 1, kind = ERR_NAN;
            else if (isinf(f)) pass = 1, kind = ERR_INF;
        } else {
            bool over;
            const uint32_t h = __half_as_ushort(float_to_half_checked(f, &over));
            reinterpret_cast<__half*>(out)[e] = __ushort_as_half((unsigned short)h);
            if (over) kind = ERR_RANGE;
            else if ((h & 0x7C00) == 0x7C00) pass = 1, kind = (h & 0x7FFF) != 0x7C00 ? ERR_NAN : ERR_INF;
        }
        if (kind >= 0) atomicMin(first_bad, error_key(r, pass, dim, i, kind));
    }
};

// total fields (total > 0) to rows; status[0] = the first-offender key, status[1] = the first malformed field (both set
// to ~0 here)
static int numeric_cast_rows(int elem, int dim, const uint8_t* bytes, const int64_t* off, int64_t base, int64_t total, void* out,
                             unsigned long long* status) {
    cudaStream_t s = ctx().stream;
    VB_CUDA(cudaMemsetAsync(status, 0xFF, 2 * sizeof(unsigned long long), s));
    const unsigned grid = (unsigned)((total + 255) / 256);
    if (elem == VB_VECTOR)
        numeric_cast_kernel<<<grid, 256, 0, s>>>(bytes, off, base, total, NumericRowSink<VB_VECTOR>{out, dim, status}, status + 1);
    else
        numeric_cast_kernel<<<grid, 256, 0, s>>>(bytes, off, base, total, NumericRowSink<VB_HALFVEC>{out, dim, status}, status + 1);
    VB_CUDA(cudaGetLastError());
    count_launch();
    return VB_OK;
}

// the shortest decimal that reads back as the same float, in PostgreSQL's float4 output style
// (float_to_shortest_decimal_buf: fixed notation for exponents -4 .. 14, scientific otherwise)
static void shortest_float(float v, char* buf, size_t cap) {
    char tmp[64];
    int digits = 9;
    for (int p = 1; p <= 9; ++p) {
        snprintf(tmp, sizeof(tmp), "%.*e", p - 1, (double)v);
        if (strtof(tmp, nullptr) == v) {
            digits = p;
            break;
        }
    }
    snprintf(tmp, sizeof(tmp), "%.*e", digits - 1, (double)v);
    const int exp10 = atoi(strchr(tmp, 'e') + 1);
    if (exp10 >= -4 && exp10 < 15) {
        const int frac = digits - 1 - exp10;
        snprintf(buf, cap, "%.*f", frac > 0 ? frac : 0, (double)v);
    } else {
        // mantissa without trailing zeros, exponent as e+NN
        char mant[32];
        size_t m = (size_t)(strchr(tmp, 'e') - tmp);
        memcpy(mant, tmp, m);
        mant[m] = 0;
        snprintf(buf, cap, "%se%c%02d", mant, exp10 < 0 ? '-' : '+', exp10 < 0 ? -exp10 : exp10);
    }
}

int half_range_error(float v) {
    char num[64];
    shortest_float(v, num, sizeof(num));
    set_error("\"%s\" is out of range for type halfvec", num);
    return VB_EINVAL;
}

static int stage_in(Scratch& sc, int elem, int dim, const void* rows, int64_t n, void** d_in) {
    const size_t raw = raw_row_bytes(elem, dim);
    VB_TRY(sc.take(raw * (size_t)n, d_in));
    VB_CUDA(cudaMemcpyAsync(*d_in, rows, raw * (size_t)n, cudaMemcpyHostToDevice, ctx().stream));
    return VB_OK;
}

// ---------------------------------------------------------------- the transforms over device rows
// n > 0 packed rows at `in` (device), results to device memory; enqueued on the library stream, nothing read back.

static int norm_rows(int elem, int dim, const void* in, int64_t n, double* norms) {
    cudaStream_t s = ctx().stream;
    const unsigned grid = (unsigned)((n * 32 + 255) / 256);
    const size_t raw = raw_row_bytes(elem, dim);
    if (elem == VB_VECTOR) norm_kernel<VB_VECTOR><<<grid, 256, 0, s>>>((const uint8_t*)in, raw, n, dim, 0, norms, nullptr, 0, nullptr);
    else norm_kernel<VB_HALFVEC><<<grid, 256, 0, s>>>((const uint8_t*)in, raw, n, dim, 0, norms, nullptr, 0, nullptr);
    VB_CUDA(cudaGetLastError());
    count_launch();
    return VB_OK;
}

// *flag (device int) is zeroed here and set to 1 where a quotient became infinite
static int normalize_rows(int elem, int dim, const void* in, int64_t n, void* out, int* flag) {
    cudaStream_t s = ctx().stream;
    VB_CUDA(cudaMemsetAsync(flag, 0, sizeof(int), s));
    const unsigned grid = (unsigned)((n * 32 + 255) / 256);
    const size_t raw = raw_row_bytes(elem, dim);
    if (elem == VB_VECTOR)
        norm_kernel<VB_VECTOR><<<grid, 256, 0, s>>>((const uint8_t*)in, raw, n, dim, 1, nullptr, (uint8_t*)out, raw, flag);
    else
        norm_kernel<VB_HALFVEC><<<grid, 256, 0, s>>>((const uint8_t*)in, raw, n, dim, 1, nullptr, (uint8_t*)out, raw, flag);
    VB_CUDA(cudaGetLastError());
    count_launch();
    return VB_OK;
}

static int quantize_rows(int elem, int dim, const void* in, int64_t n, uint8_t* out) {
    cudaStream_t s = ctx().stream;
    const size_t raw = raw_row_bytes(elem, dim);
    const size_t nb = ((size_t)dim + 7) / 8;
    const unsigned grid = (unsigned)(((size_t)n * nb + 255) / 256);
    if (elem == VB_VECTOR) binary_quantize_kernel<VB_VECTOR><<<grid, 256, 0, s>>>((const uint8_t*)in, raw, n, dim, out, nb);
    else binary_quantize_kernel<VB_HALFVEC><<<grid, 256, 0, s>>>((const uint8_t*)in, raw, n, dim, out, nb);
    VB_CUDA(cudaGetLastError());
    count_launch();
    return VB_OK;
}

// *first_bad (device) is set to ~0 here and lowered to the row-major index of every value that overflows
static int to_half_rows(int dim, const void* in, int64_t n, void* out, unsigned long long* first_bad) {
    cudaStream_t s = ctx().stream;
    const int64_t total = n * dim;
    VB_CUDA(cudaMemsetAsync(first_bad, 0xFF, sizeof(unsigned long long), s));
    to_half_kernel<<<(unsigned)((total + 255) / 256), 256, 0, s>>>((const float*)in, total, (__half*)out, first_bad);
    VB_CUDA(cudaGetLastError());
    count_launch();
    return VB_OK;
}

static int to_float_rows(int dim, const void* in, int64_t n, void* out) {
    cudaStream_t s = ctx().stream;
    const int64_t total = n * dim;
    to_float_kernel<<<(unsigned)((total + 255) / 256), 256, 0, s>>>((const __half*)in, total, (float*)out);
    VB_CUDA(cudaGetLastError());
    count_launch();
    return VB_OK;
}

// 2^lg lanes per row of `words` words: up to a warp
static int lanes_lg(int words) {
    int lg = 0;
    while (lg < 5 && (1 << lg) < words) ++lg;
    return lg;
}

template <typename T>
static void launch_subvector(const void* in, int64_t pitch_b, int64_t first_b, int64_t n, int64_t row_b, void* out, int64_t out_pitch_b,
                             int64_t out_first_b, cudaStream_t s) {
    const int64_t w = (int64_t)sizeof(T);
    const int words = (int)(row_b / w);
    const int lg = lanes_lg(words);
    const unsigned grid = (unsigned)(((n << lg) + 255) / 256);
    subvector_kernel<T><<<grid, 256, 0, s>>>((const T*)in, pitch_b / w, first_b / w, n, words, lg, (T*)out, out_pitch_b / w, out_first_b / w);
}

// row_b bytes from byte first_b of every input row (pitch_b apart, 0: one row repeated) to byte out_first_b of every
// output row (out_pitch_b apart), n rows, in the widest word that every pitch, offset, the run and both base addresses
// are aligned to
static int copy_columns(const void* in, int64_t pitch_b, int64_t first_b, int64_t n, int64_t row_b, void* out, int64_t out_pitch_b,
                        int64_t out_first_b) {
    cudaStream_t s = ctx().stream;
    const uint64_t a = (uint64_t)pitch_b | (uint64_t)first_b | (uint64_t)row_b | (uint64_t)out_pitch_b | (uint64_t)out_first_b |
                       (uint64_t)(uintptr_t)in | (uint64_t)(uintptr_t)out;
    if (a % 16 == 0) launch_subvector<uint4>(in, pitch_b, first_b, n, row_b, out, out_pitch_b, out_first_b, s);
    else if (a % 8 == 0) launch_subvector<uint2>(in, pitch_b, first_b, n, row_b, out, out_pitch_b, out_first_b, s);
    else if (a % 4 == 0) launch_subvector<uint32_t>(in, pitch_b, first_b, n, row_b, out, out_pitch_b, out_first_b, s);
    else launch_subvector<uint16_t>(in, pitch_b, first_b, n, row_b, out, out_pitch_b, out_first_b, s);
    VB_CUDA(cudaGetLastError());
    count_launch();
    return VB_OK;
}

// elements [first, first + out_dim) of every row
static int subvector_rows(int elem, int dim, const void* in, int64_t n, int first, int out_dim, void* out) {
    const int64_t es = elem == VB_VECTOR ? 4 : 2;
    return copy_columns(in, es * dim, es * first, n, es * out_dim, out, es * out_dim, 0);
}

// a || b: the m result rows (m = max(na, nb) where one count is 1); an operand of one row is repeated (pitch 0)
static int concat_rows(int elem, int dim_a, const void* a, int64_t na, int dim_b, const void* b, int64_t nb, int64_t m, void* out) {
    const int64_t es = elem == VB_VECTOR ? 4 : 2, pitch_o = es * (dim_a + dim_b);
    VB_TRY(copy_columns(a, na == 1 ? 0 : es * dim_a, 0, m, es * dim_a, out, pitch_o, 0));
    return copy_columns(b, nb == 1 ? 0 : es * dim_b, 0, m, es * dim_b, out, pitch_o, es * dim_a);
}

template <typename W, int ELEM, int OP>
static void launch_arith(const void* a, int64_t pitch_a_b, const void* b, int64_t pitch_b_b, int64_t m, int dim, void* out,
                         unsigned long long* first_bad, cudaStream_t s) {
    const int64_t w = (int64_t)sizeof(W);
    const int words = (int)(raw_row_bytes(ELEM, dim) / w);
    const int lg = lanes_lg(words);
    const unsigned grid = (unsigned)(((m << lg) + 255) / 256);
    arith_kernel<W, ELEM, OP><<<grid, 256, 0, s>>>((const W*)a, pitch_a_b / w, (const W*)b, pitch_b_b / w, m, dim, words, lg, (W*)out,
                                                   first_bad);
}

template <int ELEM, int OP>
static void launch_arith_words(const void* a, int64_t pitch_a_b, const void* b, int64_t pitch_b_b, int64_t m, int dim, void* out,
                               unsigned long long* first_bad, cudaStream_t s) {
    // the widest word every row start and the three base addresses are aligned to
    const uint64_t al = (uint64_t)raw_row_bytes(ELEM, dim) | (uint64_t)(uintptr_t)a | (uint64_t)(uintptr_t)b | (uint64_t)(uintptr_t)out;
    if (al % 16 == 0) launch_arith<uint4, ELEM, OP>(a, pitch_a_b, b, pitch_b_b, m, dim, out, first_bad, s);
    else if (al % 8 == 0) launch_arith<uint2, ELEM, OP>(a, pitch_a_b, b, pitch_b_b, m, dim, out, first_bad, s);
    else if constexpr (ELEM == VB_VECTOR) launch_arith<uint32_t, ELEM, OP>(a, pitch_a_b, b, pitch_b_b, m, dim, out, first_bad, s);
    else if (al % 4 == 0) launch_arith<uint32_t, ELEM, OP>(a, pitch_a_b, b, pitch_b_b, m, dim, out, first_bad, s);
    else launch_arith<uint16_t, ELEM, OP>(a, pitch_a_b, b, pitch_b_b, m, dim, out, first_bad, s);
}

// out = a op b over m result rows; *first_bad (device) is set to ~0 here and lowered to the key of every offender
static int arith_rows(int elem, int op, int dim, const void* a, int64_t na, const void* b, int64_t nb, int64_t m, void* out,
                      unsigned long long* first_bad) {
    cudaStream_t s = ctx().stream;
    VB_CUDA(cudaMemsetAsync(first_bad, 0xFF, sizeof(unsigned long long), s));
    const int64_t row_b = (int64_t)raw_row_bytes(elem, dim);
    const int64_t pa = na == 1 ? 0 : row_b, pb = nb == 1 ? 0 : row_b;
#define VB_ARITH_CASE(E, O) \
    if (elem == E && op == O) launch_arith_words<E, O>(a, pa, b, pb, m, dim, out, first_bad, s);
    VB_ARITH_CASE(VB_VECTOR, VB_ADD)
    VB_ARITH_CASE(VB_VECTOR, VB_SUB)
    VB_ARITH_CASE(VB_VECTOR, VB_MUL)
    VB_ARITH_CASE(VB_HALFVEC, VB_ADD)
    VB_ARITH_CASE(VB_HALFVEC, VB_SUB)
    VB_ARITH_CASE(VB_HALFVEC, VB_MUL)
#undef VB_ARITH_CASE
    VB_CUDA(cudaGetLastError());
    count_launch();
    return VB_OK;
}

template <typename S, int ELEM>
static void launch_array_cast(const void* in, int64_t total, int dim, void* out, unsigned long long* first_bad, cudaStream_t s) {
    // four elements per thread where the source and the result base addresses allow whole words
    if ((uintptr_t)in % (4 * sizeof(S)) == 0 && (uintptr_t)out % (ELEM == VB_VECTOR ? 16 : 8) == 0)
        array_cast_kernel<S, ELEM, 4><<<(unsigned)(((total + 3) / 4 + 255) / 256), 256, 0, s>>>((const S*)in, total, dim, out, first_bad);
    else
        array_cast_kernel<S, ELEM, 1><<<(unsigned)((total + 255) / 256), 256, 0, s>>>((const S*)in, total, dim, out, first_bad);
}

static size_t array_elem_bytes(int src) { return src == VB_ARRAY_FLOAT8 ? 8 : 4; }

// n source rows of dim elements to vector / halfvec rows; *first_bad as in arith_rows
static int array_cast_rows(int elem, int src, int dim, const void* in, int64_t n, void* out, unsigned long long* first_bad) {
    cudaStream_t s = ctx().stream;
    VB_CUDA(cudaMemsetAsync(first_bad, 0xFF, sizeof(unsigned long long), s));
    const int64_t total = n * dim;
#define VB_CAST_CASE(SRC, S, E) \
    if (src == SRC && elem == E) launch_array_cast<S, E>(in, total, dim, out, first_bad, s);
    VB_CAST_CASE(VB_ARRAY_INT4, int32_t, VB_VECTOR)
    VB_CAST_CASE(VB_ARRAY_FLOAT4, float, VB_VECTOR)
    VB_CAST_CASE(VB_ARRAY_FLOAT8, double, VB_VECTOR)
    VB_CAST_CASE(VB_ARRAY_INT4, int32_t, VB_HALFVEC)
    VB_CAST_CASE(VB_ARRAY_FLOAT4, float, VB_HALFVEC)
    VB_CAST_CASE(VB_ARRAY_FLOAT8, double, VB_HALFVEC)
#undef VB_CAST_CASE
    VB_CUDA(cudaGetLastError());
    count_launch();
    return VB_OK;
}

// subvector's dimension rule (src/vector.c:995-1018, src/halfvec.c:951-974): the first element (0-based) and the count
// of the result, decided from the scalars alone.  end is 64-bit so that dim + 1 cannot overflow for any int dim; for the
// reference's dimensions (<= 16000) it is the reference's int32 arithmetic.
static int subvector_range(int elem, int dim, int32_t start, int32_t count, int* first, int* out_dim) {
    const char* name = elem == VB_VECTOR ? "vector" : "halfvec";
    VB_REQUIRE(count >= 1, "%s must have at least 1 dimension", name);
    const int64_t end = start > dim - count ? (int64_t)dim + 1 : (int64_t)start + count;
    if (start < 1) start = 1;
    else VB_REQUIRE(start <= dim, "%s must have at least 1 dimension", name);
    const int64_t d = end - start;
    // CheckDim (src/vector.c:95-106, src/halfvec.c twin)
    VB_REQUIRE(d >= 1, "%s must have at least 1 dimension", name);
    VB_REQUIRE(d <= 16000, "%s cannot have more than %d dimensions", name, 16000);
    *first = start - 1;
    *out_dim = (int)d;
    return VB_OK;
}

// the checks of every transform, before any launch
static int check_rows(const char* fn, int elem, int dim, int64_t n, const void* in, const void* out) {
    VB_REQUIRE(elem == VB_VECTOR || elem == VB_HALFVEC, "%s: elem must be VB_VECTOR or VB_HALFVEC, got %d", fn, elem);
    VB_REQUIRE(dim > 0, "%s: dim must be positive, got %d", fn, dim);
    VB_REQUIRE(n >= 0, "%s: bad row count %lld", fn, (long long)n);
    VB_REQUIRE(n == 0 || (in && out), "%s: null rows or output", fn);
    return VB_OK;
}

// device rows and output must not overlap (vb_l2_normalize_batch_dev lets them be the same rows before calling this)
static int check_disjoint(const char* fn, const void* in, size_t in_bytes, const void* out, size_t out_bytes) {
    const uintptr_t i0 = (uintptr_t)in, o0 = (uintptr_t)out;
    VB_REQUIRE(i0 + in_bytes <= o0 || o0 + out_bytes <= i0, "%s: the output overlaps the rows", fn);
    return VB_OK;
}

static size_t dense_bytes(int elem, int dim, int64_t n) { return raw_row_bytes(elem, dim) * (size_t)n; }

static const char* type_name(int elem) { return elem == VB_VECTOR ? "vector" : "halfvec"; }

// the argument checks of + - * and ||: *m = the result rows (nb, or na when nb == 1)
static int check_pair(const char* fn, int elem, int dim_a, const void* a, int64_t na, int dim_b, const void* b, int64_t nb, const void* out,
                      int64_t* m) {
    VB_REQUIRE(elem == VB_VECTOR || elem == VB_HALFVEC, "%s: elem must be VB_VECTOR or VB_HALFVEC, got %d", fn, elem);
    VB_REQUIRE(dim_a > 0 && dim_b > 0, "%s: dimensions must be positive, got %d and %d", fn, dim_a, dim_b);
    VB_REQUIRE(na >= 0 && nb >= 0, "%s: bad row counts %lld and %lld", fn, (long long)na, (long long)nb);
    VB_REQUIRE(na == nb || na == 1 || nb == 1, "%s: row counts %lld and %lld neither match nor broadcast", fn, (long long)na,
               (long long)nb);
    *m = nb == 1 ? na : nb;
    VB_REQUIRE(*m == 0 || (a && b && out), "%s: null rows or output", fn);
    const uintptr_t es = elem == VB_VECTOR ? 4 : 2;
    VB_REQUIRE(((uintptr_t)a | (uintptr_t)b | (uintptr_t)out) % es == 0, "%s: rows and output must be %d-byte aligned", fn, (int)es);
    return VB_OK;
}

// the result of a batch from its first-offender key (host): VB_OK, or the reference's error for that offender.  For a
// halfvec range error, range_value(row-major element index) gives the float the text shows.
template <typename RangeValue>
static int batch_error(unsigned long long key, bool arith, int elem, int dim, RangeValue range_value) {
    if (key == NO_ERROR) return VB_OK;
    const int kind = (int)(key & 3);
    const unsigned long long rest = key >> 2, rp = rest / (unsigned)dim;
    if (arith) {
        // float_overflow_error / float_underflow_error
        set_error("value out of range: %s", kind == ERR_UNDERFLOW ? "underflow" : "overflow");
    } else if (kind == ERR_RANGE && elem == VB_HALFVEC) {
        float v;
        VB_TRY(range_value((int64_t)((rp >> 1) * (unsigned)dim + rest % (unsigned)dim), &v));
        return half_range_error(v);
    } else {
        set_error(kind == ERR_NAN ? "NaN not allowed in %s" : "infinite value not allowed in %s", type_name(elem));
    }
    return VB_EINVAL;
}

// (float) of source element i of an array cast, as the kernel forms it (host C casts round to nearest even too)
static float source_float(int src, const void* p, int64_t i) {
    if (src == VB_ARRAY_INT4) return (float)((const int32_t*)p)[i];
    if (src == VB_ARRAY_FLOAT8) return (float)((const double*)p)[i];
    return ((const float*)p)[i];
}

// the scalar checks of array_to_vector / array_to_halfvec, before any work
static int check_array_cast(const char* fn, int elem, int src, int dim, int32_t typmod, const void* in, int64_t n, const void* out) {
    VB_REQUIRE(elem == VB_VECTOR || elem == VB_HALFVEC, "%s: elem must be VB_VECTOR or VB_HALFVEC, got %d", fn, elem);
    VB_REQUIRE(src == VB_ARRAY_INT4 || src == VB_ARRAY_FLOAT4 || src == VB_ARRAY_FLOAT8, "%s: bad source type %d", fn, src);
    VB_REQUIRE(n >= 0, "%s: bad row count %lld", fn, (long long)n);
    // CheckDim, then CheckExpectedDim (src/vector.c:80-106, src/halfvec.c twins)
    VB_REQUIRE(dim >= 1, "%s must have at least 1 dimension", type_name(elem));
    VB_REQUIRE(dim <= 16000, "%s cannot have more than %d dimensions", type_name(elem), 16000);
    VB_REQUIRE(typmod == -1 || typmod == dim, "expected %d dimensions, not %d", typmod, dim);
    VB_REQUIRE(n == 0 || (in && out), "%s: null rows or output", fn);
    VB_REQUIRE((uintptr_t)in % array_elem_bytes(src) == 0 && (uintptr_t)out % (elem == VB_VECTOR ? 4 : 2) == 0,
               "%s: rows and output must be aligned to their elements", fn);
    return VB_OK;
}

// the scalar checks of numeric[] -> vector / halfvec, before any work
static int check_numeric_cast(const char* fn, int elem, int dim, int32_t typmod, const void* bytes, const int64_t* off, int64_t n,
                              const void* out) {
    VB_REQUIRE(elem == VB_VECTOR || elem == VB_HALFVEC, "%s: elem must be VB_VECTOR or VB_HALFVEC, got %d", fn, elem);
    VB_REQUIRE(n >= 0, "%s: bad row count %lld", fn, (long long)n);
    VB_REQUIRE(dim >= 1, "%s must have at least 1 dimension", type_name(elem));
    VB_REQUIRE(dim <= 16000, "%s cannot have more than %d dimensions", type_name(elem), 16000);
    VB_REQUIRE(typmod == -1 || typmod == dim, "expected %d dimensions, not %d", typmod, dim);
    VB_REQUIRE(n == 0 || (bytes && off && out), "%s: null fields, offsets or output", fn);
    VB_REQUIRE((uintptr_t)off % 8 == 0 && (uintptr_t)out % (elem == VB_VECTOR ? 4 : 2) == 0,
               "%s: offsets and output must be aligned to their elements", fn);
    return VB_OK;
}

// the numeric cast's error from its first-offender key; field(e) gives a host copy of field e's bytes
template <typename Field>
static int numeric_batch_error(unsigned long long key, int elem, int dim, int64_t* out_bad, Field field) {
    const int kind = (int)(key & 3);
    const unsigned long long rest = key >> 2, rp = rest / (unsigned)dim;
    const int64_t row = (int64_t)(rp >> 1), e = row * dim + (int64_t)(rest % (unsigned)dim);
    if (out_bad) *out_bad = row;
    if (kind == ERR_NAN || kind == ERR_INF) {
        set_error(kind == ERR_NAN ? "NaN not allowed in %s" : "infinite value not allowed in %s", type_name(elem));
        return VB_EINVAL;
    }
    std::vector<uint8_t> f;
    VB_TRY(field(e, f));
    return kind == ERR_REAL ? numeric_range_error(f.data()) : half_range_error(numeric_float4_host(f.data()));
}

}  // namespace vb

using namespace vb;

extern "C" {

// ---------------------------------------------------------------- host buffers

int vb_norm_batch(int elem, int dim, const void* rows, int64_t n, double* out) {
    Scratch sc;
    VB_TRY(require_init());
    VB_REQUIRE((elem == VB_VECTOR || elem == VB_HALFVEC) && dim > 0 && (rows || n == 0) && out, "bad norm arguments");
    if (n <= 0) return VB_OK;
    cudaStream_t s = ctx().stream;
    void *d_in, *d_out;
    VB_TRY(stage_in(sc, elem, dim, rows, n, &d_in));
    VB_TRY(sc.take(sizeof(double) * (size_t)n, &d_out));
    VB_TRY(norm_rows(elem, dim, d_in, n, (double*)d_out));
    VB_CUDA(cudaMemcpyAsync(out, d_out, sizeof(double) * (size_t)n, cudaMemcpyDeviceToHost, s));
    VB_CUDA(cudaStreamSynchronize(s));
    return VB_OK;
}

int vb_l2_normalize_batch(int elem, int dim, const void* rows, int64_t n, void* out) {
    Scratch sc;
    VB_TRY(require_init());
    VB_REQUIRE((elem == VB_VECTOR || elem == VB_HALFVEC) && dim > 0 && (rows || n == 0) && out, "bad normalize arguments");
    if (n <= 0) return VB_OK;
    cudaStream_t s = ctx().stream;
    void *d_in, *d_out, *d_flag;
    const size_t raw = raw_row_bytes(elem, dim);
    VB_TRY(stage_in(sc, elem, dim, rows, n, &d_in));
    VB_TRY(sc.take(raw * (size_t)n, &d_out));
    VB_TRY(sc.take(64, &d_flag));
    VB_TRY(normalize_rows(elem, dim, d_in, n, d_out, (int*)d_flag));
    int flag = 0;
    VB_CUDA(cudaMemcpyAsync(out, d_out, raw * (size_t)n, cudaMemcpyDeviceToHost, s));
    VB_CUDA(cudaMemcpyAsync(&flag, d_flag, sizeof(int), cudaMemcpyDeviceToHost, s));
    VB_CUDA(cudaStreamSynchronize(s));
    // float_overflow_error() of the reference (src/vector.c:809-813): "value out of range: overflow"
    VB_REQUIRE(!flag, "value out of range: overflow");
    return VB_OK;
}

int vb_binary_quantize_batch(int elem, int dim, const void* rows, int64_t n, uint8_t* out) {
    Scratch sc;
    VB_TRY(require_init());
    VB_REQUIRE((elem == VB_VECTOR || elem == VB_HALFVEC) && dim > 0 && (rows || n == 0) && out, "bad binary_quantize arguments");
    if (n <= 0) return VB_OK;
    cudaStream_t s = ctx().stream;
    void *d_in, *d_out;
    const size_t nb = ((size_t)dim + 7) / 8;
    VB_TRY(stage_in(sc, elem, dim, rows, n, &d_in));
    VB_TRY(sc.take(nb * (size_t)n, &d_out));
    VB_TRY(quantize_rows(elem, dim, d_in, n, (uint8_t*)d_out));
    VB_CUDA(cudaMemcpyAsync(out, d_out, nb * (size_t)n, cudaMemcpyDeviceToHost, s));
    VB_CUDA(cudaStreamSynchronize(s));
    return VB_OK;
}

int vb_vector_to_halfvec_batch(int dim, const void* rows, int64_t n, void* out) {
    Scratch sc;
    VB_TRY(require_init());
    VB_REQUIRE(dim > 0 && (rows || n == 0) && out, "bad cast arguments");
    if (n <= 0) return VB_OK;
    cudaStream_t s = ctx().stream;
    const int64_t total = n * dim;
    void *d_in, *d_out, *d_flag;
    VB_TRY(stage_in(sc, VB_VECTOR, dim, rows, n, &d_in));
    VB_TRY(sc.take(sizeof(__half) * (size_t)total, &d_out));
    VB_TRY(sc.take(64, &d_flag));
    VB_TRY(to_half_rows(dim, d_in, n, d_out, (unsigned long long*)d_flag));
    unsigned long long bad = ~0ull;
    VB_CUDA(cudaMemcpyAsync(out, d_out, sizeof(__half) * (size_t)total, cudaMemcpyDeviceToHost, s));
    VB_CUDA(cudaMemcpyAsync(&bad, d_flag, sizeof(bad), cudaMemcpyDeviceToHost, s));
    VB_CUDA(cudaStreamSynchronize(s));
    if (bad != ~0ull) return half_range_error(reinterpret_cast<const float*>(rows)[bad]);
    return VB_OK;
}

int vb_halfvec_to_vector_batch(int dim, const void* rows, int64_t n, void* out) {
    Scratch sc;
    VB_TRY(require_init());
    VB_REQUIRE(dim > 0 && (rows || n == 0) && out, "bad cast arguments");
    if (n <= 0) return VB_OK;
    cudaStream_t s = ctx().stream;
    const int64_t total = n * dim;
    void *d_in, *d_out;
    VB_TRY(stage_in(sc, VB_HALFVEC, dim, rows, n, &d_in));
    VB_TRY(sc.take(sizeof(float) * (size_t)total, &d_out));
    VB_TRY(to_float_rows(dim, d_in, n, d_out));
    VB_CUDA(cudaMemcpyAsync(out, d_out, sizeof(float) * (size_t)total, cudaMemcpyDeviceToHost, s));
    VB_CUDA(cudaStreamSynchronize(s));
    return VB_OK;
}

int vb_subvector_batch(int elem, int dim, const void* rows, int64_t n, int32_t start, int32_t count, void* out, int* out_dim) {
    Scratch sc;
    const char* fn = "vb_subvector_batch";
    VB_TRY(require_init());
    VB_TRY(check_rows(fn, elem, dim, n, rows, out));
    VB_REQUIRE(out_dim, "%s: null out_dim", fn);
    int first, d;
    VB_TRY(subvector_range(elem, dim, start, count, &first, &d));
    *out_dim = d;
    if (n == 0) return VB_OK;
    cudaStream_t s = ctx().stream;
    void *d_in, *d_out;
    VB_TRY(stage_in(sc, elem, dim, rows, n, &d_in));
    VB_TRY(sc.take(dense_bytes(elem, d, n), &d_out));
    VB_TRY(subvector_rows(elem, dim, d_in, n, first, d, d_out));
    VB_CUDA(cudaMemcpyAsync(out, d_out, dense_bytes(elem, d, n), cudaMemcpyDeviceToHost, s));
    VB_CUDA(cudaStreamSynchronize(s));
    return VB_OK;
}

// ---------------------------------------------------------------- device buffers

int vb_norm_batch_dev(int elem, int dim, const void* rows_dev, int64_t n, double* out_dev) {
    VB_TRY(require_init());
    const char* fn = "vb_norm_batch_dev";
    VB_TRY(check_rows(fn, elem, dim, n, rows_dev, out_dev));
    if (n == 0) return VB_OK;
    VB_TRY(check_disjoint(fn, rows_dev, dense_bytes(elem, dim, n), out_dev, sizeof(double) * (size_t)n));
    return norm_rows(elem, dim, rows_dev, n, out_dev);
}

int vb_l2_normalize_batch_dev(int elem, int dim, const void* rows_dev, int64_t n, void* out_dev) {
    Scratch sc;
    VB_TRY(require_init());
    const char* fn = "vb_l2_normalize_batch_dev";
    VB_TRY(check_rows(fn, elem, dim, n, rows_dev, out_dev));
    if (n == 0) return VB_OK;
    const size_t bytes = dense_bytes(elem, dim, n);
    if (rows_dev != out_dev) VB_TRY(check_disjoint(fn, rows_dev, bytes, out_dev, bytes));   // in place is allowed
    cudaStream_t s = ctx().stream;
    void* d_flag;
    VB_TRY(sc.take(64, &d_flag));
    VB_TRY(normalize_rows(elem, dim, rows_dev, n, out_dev, (int*)d_flag));
    int flag = 0;
    VB_CUDA(cudaMemcpyAsync(&flag, d_flag, sizeof(int), cudaMemcpyDeviceToHost, s));
    VB_CUDA(cudaStreamSynchronize(s));
    VB_REQUIRE(!flag, "value out of range: overflow");
    return VB_OK;
}

int vb_binary_quantize_batch_dev(int elem, int dim, const void* rows_dev, int64_t n, uint8_t* out_dev) {
    VB_TRY(require_init());
    const char* fn = "vb_binary_quantize_batch_dev";
    VB_TRY(check_rows(fn, elem, dim, n, rows_dev, out_dev));
    if (n == 0) return VB_OK;
    VB_TRY(check_disjoint(fn, rows_dev, dense_bytes(elem, dim, n), out_dev, ((size_t)dim + 7) / 8 * (size_t)n));
    return quantize_rows(elem, dim, rows_dev, n, out_dev);
}

int vb_vector_to_halfvec_batch_dev(int dim, const void* rows_dev, int64_t n, void* out_dev) {
    Scratch sc;
    VB_TRY(require_init());
    const char* fn = "vb_vector_to_halfvec_batch_dev";
    VB_TRY(check_rows(fn, VB_VECTOR, dim, n, rows_dev, out_dev));
    if (n == 0) return VB_OK;
    VB_TRY(check_disjoint(fn, rows_dev, dense_bytes(VB_VECTOR, dim, n), out_dev, dense_bytes(VB_HALFVEC, dim, n)));
    cudaStream_t s = ctx().stream;
    void* d_flag;
    VB_TRY(sc.take(64, &d_flag));
    VB_TRY(to_half_rows(dim, rows_dev, n, out_dev, (unsigned long long*)d_flag));
    unsigned long long bad = ~0ull;
    VB_CUDA(cudaMemcpyAsync(&bad, d_flag, sizeof(bad), cudaMemcpyDeviceToHost, s));
    VB_CUDA(cudaStreamSynchronize(s));
    if (bad == ~0ull) return VB_OK;
    float v;   // only the error reads the offending value, for the reference's text
    VB_CUDA(cudaMemcpyAsync(&v, (const float*)rows_dev + bad, sizeof(float), cudaMemcpyDeviceToHost, s));
    VB_CUDA(cudaStreamSynchronize(s));
    return half_range_error(v);
}

int vb_halfvec_to_vector_batch_dev(int dim, const void* rows_dev, int64_t n, void* out_dev) {
    VB_TRY(require_init());
    const char* fn = "vb_halfvec_to_vector_batch_dev";
    VB_TRY(check_rows(fn, VB_HALFVEC, dim, n, rows_dev, out_dev));
    if (n == 0) return VB_OK;
    VB_TRY(check_disjoint(fn, rows_dev, dense_bytes(VB_HALFVEC, dim, n), out_dev, dense_bytes(VB_VECTOR, dim, n)));
    return to_float_rows(dim, rows_dev, n, out_dev);
}

int vb_subvector_batch_dev(int elem, int dim, const void* rows_dev, int64_t n, int32_t start, int32_t count, void* out_dev, int* out_dim) {
    const char* fn = "vb_subvector_batch_dev";
    VB_TRY(require_init());
    VB_TRY(check_rows(fn, elem, dim, n, rows_dev, out_dev));
    VB_REQUIRE(out_dim, "%s: null out_dim", fn);
    int first, d;
    VB_TRY(subvector_range(elem, dim, start, count, &first, &d));
    if (n > 0) VB_TRY(check_disjoint(fn, rows_dev, dense_bytes(elem, dim, n), out_dev, dense_bytes(elem, d, n)));
    *out_dim = d;
    if (n == 0) return VB_OK;
    return subvector_rows(elem, dim, rows_dev, n, first, d, out_dev);
}

// ---------------------------------------------------------------- + - * ||, array casts

int vb_arith_batch(int elem, int op, int dim_a, const void* a, int64_t na, int dim_b, const void* b, int64_t nb, void* out) {
    Scratch sc;
    const char* fn = "vb_arith_batch";
    VB_TRY(require_init());
    int64_t m;
    VB_TRY(check_pair(fn, elem, dim_a, a, na, dim_b, b, nb, out, &m));
    VB_REQUIRE(op == VB_ADD || op == VB_SUB || op == VB_MUL, "%s: bad op %d", fn, op);
    // CheckDims (src/vector.c:71-77, src/halfvec.c:74-81)
    VB_REQUIRE(dim_a == dim_b, "different %s dimensions %d and %d", type_name(elem), dim_a, dim_b);
    if (m == 0) return VB_OK;
    cudaStream_t s = ctx().stream;
    void *d_a, *d_b, *d_out, *d_flag;
    const size_t raw = raw_row_bytes(elem, dim_a);
    VB_TRY(stage_in(sc, elem, dim_a, a, na, &d_a));
    VB_TRY(sc.take(raw * (size_t)nb, &d_b));
    VB_CUDA(cudaMemcpyAsync(d_b, b, raw * (size_t)nb, cudaMemcpyHostToDevice, s));
    VB_TRY(sc.take(raw * (size_t)m, &d_out));
    VB_TRY(sc.take(64, &d_flag));
    VB_TRY(arith_rows(elem, op, dim_a, d_a, na, d_b, nb, m, d_out, (unsigned long long*)d_flag));
    unsigned long long key = NO_ERROR;
    VB_CUDA(cudaMemcpyAsync(out, d_out, raw * (size_t)m, cudaMemcpyDeviceToHost, s));
    VB_CUDA(cudaMemcpyAsync(&key, d_flag, sizeof(key), cudaMemcpyDeviceToHost, s));
    VB_CUDA(cudaStreamSynchronize(s));
    return batch_error(key, true, elem, dim_a, [](int64_t, float*) { return VB_OK; });
}

int vb_arith_batch_dev(int elem, int op, int dim_a, const void* a_dev, int64_t na, int dim_b, const void* b_dev, int64_t nb, void* out_dev) {
    Scratch sc;
    const char* fn = "vb_arith_batch_dev";
    VB_TRY(require_init());
    int64_t m;
    VB_TRY(check_pair(fn, elem, dim_a, a_dev, na, dim_b, b_dev, nb, out_dev, &m));
    VB_REQUIRE(op == VB_ADD || op == VB_SUB || op == VB_MUL, "%s: bad op %d", fn, op);
    VB_REQUIRE(dim_a == dim_b, "different %s dimensions %d and %d", type_name(elem), dim_a, dim_b);
    if (m == 0) return VB_OK;
    // in place is allowed on an operand that is not broadcast; any other overlap is refused
    const size_t raw = raw_row_bytes(elem, dim_a);
    if (!(out_dev == a_dev && na == m)) VB_TRY(check_disjoint(fn, a_dev, raw * (size_t)na, out_dev, raw * (size_t)m));
    if (!(out_dev == b_dev && nb == m)) VB_TRY(check_disjoint(fn, b_dev, raw * (size_t)nb, out_dev, raw * (size_t)m));
    cudaStream_t s = ctx().stream;
    void* d_flag;
    VB_TRY(sc.take(64, &d_flag));
    VB_TRY(arith_rows(elem, op, dim_a, a_dev, na, b_dev, nb, m, out_dev, (unsigned long long*)d_flag));
    unsigned long long key = NO_ERROR;
    VB_CUDA(cudaMemcpyAsync(&key, d_flag, sizeof(key), cudaMemcpyDeviceToHost, s));
    VB_CUDA(cudaStreamSynchronize(s));
    return batch_error(key, true, elem, dim_a, [](int64_t, float*) { return VB_OK; });
}

// CheckDim of the concatenated dimension (src/vector.c:935, src/halfvec.c:893): both dimensions are positive, so only
// the upper bound can fail
static int concat_dim(int elem, int dim_a, int dim_b, int* d) {
    const int64_t sum = (int64_t)dim_a + dim_b;
    VB_REQUIRE(sum <= 16000, "%s cannot have more than %d dimensions", type_name(elem), 16000);
    *d = (int)sum;
    return VB_OK;
}

int vb_concat_batch(int elem, int dim_a, const void* a, int64_t na, int dim_b, const void* b, int64_t nb, void* out, int* out_dim) {
    Scratch sc;
    const char* fn = "vb_concat_batch";
    VB_TRY(require_init());
    int64_t m;
    VB_TRY(check_pair(fn, elem, dim_a, a, na, dim_b, b, nb, out, &m));
    VB_REQUIRE(out_dim, "%s: null out_dim", fn);
    int d;
    VB_TRY(concat_dim(elem, dim_a, dim_b, &d));
    *out_dim = d;
    if (m == 0) return VB_OK;
    cudaStream_t s = ctx().stream;
    void *d_a, *d_b, *d_out;
    VB_TRY(stage_in(sc, elem, dim_a, a, na, &d_a));
    VB_TRY(sc.take(dense_bytes(elem, dim_b, nb), &d_b));
    VB_CUDA(cudaMemcpyAsync(d_b, b, dense_bytes(elem, dim_b, nb), cudaMemcpyHostToDevice, s));
    VB_TRY(sc.take(dense_bytes(elem, d, m), &d_out));
    VB_TRY(concat_rows(elem, dim_a, d_a, na, dim_b, d_b, nb, m, d_out));
    VB_CUDA(cudaMemcpyAsync(out, d_out, dense_bytes(elem, d, m), cudaMemcpyDeviceToHost, s));
    VB_CUDA(cudaStreamSynchronize(s));
    return VB_OK;
}

int vb_concat_batch_dev(int elem, int dim_a, const void* a_dev, int64_t na, int dim_b, const void* b_dev, int64_t nb, void* out_dev,
                        int* out_dim) {
    const char* fn = "vb_concat_batch_dev";
    VB_TRY(require_init());
    int64_t m;
    VB_TRY(check_pair(fn, elem, dim_a, a_dev, na, dim_b, b_dev, nb, out_dev, &m));
    VB_REQUIRE(out_dim, "%s: null out_dim", fn);
    int d;
    VB_TRY(concat_dim(elem, dim_a, dim_b, &d));
    if (m > 0) {
        VB_TRY(check_disjoint(fn, a_dev, dense_bytes(elem, dim_a, na), out_dev, dense_bytes(elem, d, m)));
        VB_TRY(check_disjoint(fn, b_dev, dense_bytes(elem, dim_b, nb), out_dev, dense_bytes(elem, d, m)));
    }
    *out_dim = d;
    if (m == 0) return VB_OK;
    return concat_rows(elem, dim_a, a_dev, na, dim_b, b_dev, nb, m, out_dev);
}

int vb_array_to_rows_batch(int elem, int src, int dim, int32_t typmod, const void* in, int64_t n, void* out) {
    Scratch sc;
    const char* fn = "vb_array_to_rows_batch";
    VB_TRY(require_init());
    VB_TRY(check_array_cast(fn, elem, src, dim, typmod, in, n, out));
    if (n == 0) return VB_OK;
    cudaStream_t s = ctx().stream;
    const size_t in_bytes = array_elem_bytes(src) * (size_t)dim * (size_t)n;
    void *d_in, *d_out, *d_flag;
    VB_TRY(sc.take(in_bytes, &d_in));
    VB_CUDA(cudaMemcpyAsync(d_in, in, in_bytes, cudaMemcpyHostToDevice, s));
    VB_TRY(sc.take(dense_bytes(elem, dim, n), &d_out));
    VB_TRY(sc.take(64, &d_flag));
    VB_TRY(array_cast_rows(elem, src, dim, d_in, n, d_out, (unsigned long long*)d_flag));
    unsigned long long key = NO_ERROR;
    VB_CUDA(cudaMemcpyAsync(out, d_out, dense_bytes(elem, dim, n), cudaMemcpyDeviceToHost, s));
    VB_CUDA(cudaMemcpyAsync(&key, d_flag, sizeof(key), cudaMemcpyDeviceToHost, s));
    VB_CUDA(cudaStreamSynchronize(s));
    return batch_error(key, false, elem, dim, [&](int64_t i, float* v) {
        *v = source_float(src, in, i);
        return VB_OK;
    });
}

int vb_array_to_rows_batch_dev(int elem, int src, int dim, int32_t typmod, const void* in_dev, int64_t n, void* out_dev) {
    Scratch sc;
    const char* fn = "vb_array_to_rows_batch_dev";
    VB_TRY(require_init());
    VB_TRY(check_array_cast(fn, elem, src, dim, typmod, in_dev, n, out_dev));
    if (n == 0) return VB_OK;
    VB_TRY(check_disjoint(fn, in_dev, array_elem_bytes(src) * (size_t)dim * (size_t)n, out_dev, dense_bytes(elem, dim, n)));
    cudaStream_t s = ctx().stream;
    void* d_flag;
    VB_TRY(sc.take(64, &d_flag));
    VB_TRY(array_cast_rows(elem, src, dim, in_dev, n, out_dev, (unsigned long long*)d_flag));
    unsigned long long key = NO_ERROR;
    VB_CUDA(cudaMemcpyAsync(&key, d_flag, sizeof(key), cudaMemcpyDeviceToHost, s));
    VB_CUDA(cudaStreamSynchronize(s));
    return batch_error(key, false, elem, dim, [&](int64_t i, float* v) {
        // only the error reads the offending source element, for the reference's text
        double raw = 0;
        VB_CUDA(cudaMemcpyAsync(&raw, (const uint8_t*)in_dev + array_elem_bytes(src) * (size_t)i, array_elem_bytes(src),
                                cudaMemcpyDeviceToHost, s));
        VB_CUDA(cudaStreamSynchronize(s));
        *v = source_float(src, &raw, 0);
        return VB_OK;
    });
}

// numeric[] -> vector / halfvec.  Host: chunks of whole rows through the two staging slots; every chunk is converted
// and checked, so a malformed field anywhere wins over a data error, and the first chunk with a data error has the
// lowest failing row.
int vb_numeric_array_to_rows_batch(int elem, int dim, int32_t typmod, const void* bytes, const int64_t* off, int64_t n, void* out,
                                   int64_t* out_bad) {
    Scratch sc;
    const char* fn = "vb_numeric_array_to_rows_batch";
    if (out_bad) *out_bad = -1;
    VB_TRY(require_init());
    VB_TRY(check_numeric_cast(fn, elem, dim, typmod, bytes, off, n, out));
    if (n == 0) return VB_OK;
    const int64_t total = n * dim;
    VB_TRY(numeric_offsets_check(fn, off, total, out_bad, dim));
    std::vector<int64_t> starts;
    numeric_chunks(off, n, dim, (size_t)32 << 20, starts);
    const int64_t nch = (int64_t)starts.size() - 1;
    int64_t max_rows = 0, max_bytes = 0;
    for (int64_t c = 0; c < nch; ++c) {
        max_rows = std::max(max_rows, starts[c + 1] - starts[c]);
        max_bytes = std::max(max_bytes, off[starts[c + 1] * dim] - off[starts[c] * dim]);
    }
    const size_t esz = elem == VB_VECTOR ? 4 : 2;
    const size_t b_off = sizeof(int64_t) * (size_t)(max_rows * dim + 1), b_out = esz * (size_t)(max_rows * dim);
    Staging& st = staging();
    struct Slot {
        int64_t* off;
        uint8_t* bytes;
        void* out;
        unsigned long long* status;
    } slot[2];
    for (int k = 0; k < 2 && k < nch; ++k) {
        void *a, *b, *c, *d;
        VB_TRY(sc.take(b_off, &a));
        VB_TRY(sc.take((size_t)max_bytes + 16, &b));
        VB_TRY(sc.take(b_out, &c));
        VB_TRY(sc.take(16, &d));
        slot[k] = Slot{(int64_t*)a, (uint8_t*)b, c, (unsigned long long*)d};
        VB_TRY(pinned_grow(&st.in[k], &st.in_bytes[k], b_off + (size_t)max_bytes));
        VB_TRY(pinned_grow(&st.out[k], &st.out_bytes[k], b_out + 16));
    }
    cudaStream_t s = ctx().stream;
    const uint8_t* src = (const uint8_t*)bytes;
    int64_t malformed = -1, bad_chunk = -1;
    unsigned long long bad_key = NO_ERROR;
    auto enqueue = [&](int64_t c, int k) -> int {
        const int64_t e0 = starts[c] * dim, ne = (starts[c + 1] - starts[c]) * dim, b0 = off[e0], nb = off[e0 + ne] - b0;
        uint8_t* in = (uint8_t*)st.in[k];
        memcpy(in, off + e0, sizeof(int64_t) * (size_t)(ne + 1));
        memcpy(in + b_off, src + b0, (size_t)nb);
        VB_CUDA(cudaMemcpyAsync(slot[k].off, in, sizeof(int64_t) * (size_t)(ne + 1), cudaMemcpyHostToDevice, s));
        VB_CUDA(cudaMemcpyAsync(slot[k].bytes, in + b_off, (size_t)nb, cudaMemcpyHostToDevice, s));
        VB_TRY(numeric_cast_rows(elem, dim, slot[k].bytes, slot[k].off, b0, ne, slot[k].out, slot[k].status));
        uint8_t* o = (uint8_t*)st.out[k];
        VB_CUDA(cudaMemcpyAsync(o, slot[k].out, esz * (size_t)ne, cudaMemcpyDeviceToHost, s));
        VB_CUDA(cudaMemcpyAsync(o + b_out, slot[k].status, 16, cudaMemcpyDeviceToHost, s));
        return VB_OK;
    };
    auto finish = [&](int64_t c, int k) -> int {
        const int64_t e0 = starts[c] * dim, ne = (starts[c + 1] - starts[c]) * dim;
        const uint8_t* o = (const uint8_t*)st.out[k];
        unsigned long long status[2];
        memcpy(status, o + b_out, 16);
        if (malformed < 0 && status[1] != NO_ERROR) malformed = e0 + (int64_t)status[1];
        if (bad_chunk < 0 && status[0] != NO_ERROR) bad_chunk = c, bad_key = status[0];
        memcpy((uint8_t*)out + esz * (size_t)e0, o, esz * (size_t)ne);
        return VB_OK;
    };
    VB_TRY(pipeline_chunks(nch, enqueue, finish));
    if (malformed >= 0) {
        if (out_bad) *out_bad = malformed / dim;
        return numeric_field_error(fn, malformed, src + off[malformed], off[malformed + 1] - off[malformed]);
    }
    if (bad_chunk < 0) return VB_OK;
    const int64_t r0 = starts[bad_chunk];
    const int rc = numeric_batch_error(bad_key, elem, dim, out_bad, [&](int64_t e, std::vector<uint8_t>& f) {
        const int64_t g = r0 * dim + e;
        f.assign(src + off[g], src + off[g + 1]);
        return VB_OK;
    });
    if (out_bad) *out_bad += r0;
    return rc;
}

int vb_numeric_array_to_rows_batch_dev(int elem, int dim, int32_t typmod, const void* bytes_dev, const int64_t* off_dev, int64_t n,
                                       void* out_dev, int64_t* out_bad) {
    Scratch sc;
    const char* fn = "vb_numeric_array_to_rows_batch_dev";
    if (out_bad) *out_bad = -1;
    VB_TRY(require_init());
    VB_TRY(check_numeric_cast(fn, elem, dim, typmod, bytes_dev, off_dev, n, out_dev));
    if (n == 0) return VB_OK;
    cudaStream_t s = ctx().stream;
    void* d_status;
    VB_TRY(sc.take(16, &d_status));
    VB_TRY(numeric_cast_rows(elem, dim, (const uint8_t*)bytes_dev, off_dev, 0, n * dim, out_dev, (unsigned long long*)d_status));
    unsigned long long status[2];
    VB_CUDA(cudaMemcpyAsync(status, d_status, 16, cudaMemcpyDeviceToHost, s));
    VB_CUDA(cudaStreamSynchronize(s));
    if (status[0] == NO_ERROR && status[1] == NO_ERROR) return VB_OK;
    // only an error reads a field back, for its text
    auto field = [&](int64_t e, std::vector<uint8_t>& f) {
        int64_t o[2];
        VB_CUDA(cudaMemcpy(o, off_dev + e, sizeof(o), cudaMemcpyDeviceToHost));
        const int64_t len = std::max<int64_t>(0, std::min<int64_t>(o[1] - o[0], 8 + 2 * 65535 + 1));
        f.resize((size_t)len + 8);
        if (len > 0) VB_CUDA(cudaMemcpy(f.data(), (const uint8_t*)bytes_dev + o[0], (size_t)len, cudaMemcpyDeviceToHost));
        f.resize((size_t)len);   // past the longest valid field only the count of bytes left over matters
        return VB_OK;
    };
    if (status[1] != NO_ERROR) {
        const int64_t e = (int64_t)status[1];
        if (out_bad) *out_bad = e / dim;
        int64_t o[2];
        VB_CUDA(cudaMemcpy(o, off_dev + e, sizeof(o), cudaMemcpyDeviceToHost));
        std::vector<uint8_t> f;
        VB_TRY(field(e, f));
        return numeric_field_error(fn, e, f.data(), o[1] < o[0] ? o[1] - o[0] : (int64_t)f.size());
    }
    return numeric_batch_error(status[0], elem, dim, out_bad, field);
}

}  // extern "C"
