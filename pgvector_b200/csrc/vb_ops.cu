// vb_ops.cu -- batched row transforms that sit beside the distance path:
//   vb_norm_batch          vector_norm / halfvec l2_norm       (src/vector.c:767-780, src/halfvec.c:703-720)
//   vb_l2_normalize_batch  l2_normalize / halfvec_l2_normalize (src/vector.c:785-819, src/halfvec.c:725-759)
//   vb_binary_quantize_batch  binary_quantize                  (src/vector.c:952-978, src/halfvec.c twin)
//   vb_subvector_batch     subvector                           (src/vector.c:983-1025, src/halfvec.c:939-981)
//   vb_vector_to_halfvec_batch / vb_halfvec_to_vector_batch     the casts between the two
// The cosine opclasses normalise every indexed row and the query (src/ivfbuild.c:174-180,
// src/ivfscan.c:222-229, src/hnswutils.c:417-423); norms accumulate in fp64 like the reference.
// One warp per row; HBM bound (row read once, written once).
// Every transform is one launcher over device rows (the *_rows functions); the _dev entry points call it on the
// caller's buffers, the host variants stage the rows in a workspace, call it and copy the result back, so both give
// the same bits.
#include "vb_common.cuh"

#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <cstring>

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

// subvector: `words` words of T from word `first` of every input row (`pitch` words apart) into packed output rows.
// 2^lg lanes per row (lg <= 5), so short rows share a warp; consecutive lanes move consecutive words of a row, so a
// warp's loads and stores are contiguous runs.  T is the widest word (2 to 16 bytes) that the row pitch, the offset,
// the output row and both base addresses allow.
template <typename T>
__global__ void subvector_kernel(const T* __restrict__ in, int64_t pitch, int64_t first, int64_t n, int words, int lg,
                                 T* __restrict__ out) {
    const int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    const int64_t r = t >> lg;
    if (r >= n) return;
    const T* src = in + r * pitch + first;
    T* dst = out + r * (int64_t)words;
    for (int j = (int)(t & ((1 << lg) - 1)); j < words; j += 1 << lg) dst[j] = src[j];
}

enum { WSO_IN = 17, WSO_OUT = 18, WSO_FLAG = 19 };

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

static int stage_in(int elem, int dim, const void* rows, int64_t n, void** d_in) {
    const size_t raw = raw_row_bytes(elem, dim);
    VB_TRY(workspace(WSO_IN, raw * (size_t)n, d_in));
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

template <typename T>
static void launch_subvector(const void* in, int64_t pitch_b, int64_t first_b, int64_t n, int64_t row_b, void* out, cudaStream_t s) {
    const int words = (int)(row_b / (int64_t)sizeof(T));
    int lg = 0;
    while (lg < 5 && (1 << lg) < words) ++lg;
    const unsigned grid = (unsigned)(((n << lg) + 255) / 256);
    subvector_kernel<T><<<grid, 256, 0, s>>>((const T*)in, pitch_b / (int64_t)sizeof(T), first_b / (int64_t)sizeof(T), n, words, lg, (T*)out);
}

// elements [first, first + out_dim) of every row
static int subvector_rows(int elem, int dim, const void* in, int64_t n, int first, int out_dim, void* out) {
    cudaStream_t s = ctx().stream;
    const int64_t es = elem == VB_VECTOR ? 4 : 2;
    const int64_t pitch_b = es * dim, first_b = es * first, row_b = es * out_dim;
    // the widest word every row start, the offset, every output row and both base addresses are aligned to
    const uint64_t a = (uint64_t)pitch_b | (uint64_t)first_b | (uint64_t)row_b | (uint64_t)(uintptr_t)in | (uint64_t)(uintptr_t)out;
    if (a % 16 == 0) launch_subvector<uint4>(in, pitch_b, first_b, n, row_b, out, s);
    else if (a % 8 == 0) launch_subvector<uint2>(in, pitch_b, first_b, n, row_b, out, s);
    else if (a % 4 == 0) launch_subvector<uint32_t>(in, pitch_b, first_b, n, row_b, out, s);
    else launch_subvector<uint16_t>(in, pitch_b, first_b, n, row_b, out, s);
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

}  // namespace vb

using namespace vb;

extern "C" {

// ---------------------------------------------------------------- host buffers

int vb_norm_batch(int elem, int dim, const void* rows, int64_t n, double* out) {
    VB_TRY(require_init());
    VB_REQUIRE((elem == VB_VECTOR || elem == VB_HALFVEC) && dim > 0 && (rows || n == 0) && out, "bad norm arguments");
    if (n <= 0) return VB_OK;
    cudaStream_t s = ctx().stream;
    void *d_in, *d_out;
    VB_TRY(stage_in(elem, dim, rows, n, &d_in));
    VB_TRY(workspace(WSO_OUT, sizeof(double) * (size_t)n, &d_out));
    VB_TRY(norm_rows(elem, dim, d_in, n, (double*)d_out));
    VB_CUDA(cudaMemcpyAsync(out, d_out, sizeof(double) * (size_t)n, cudaMemcpyDeviceToHost, s));
    VB_CUDA(cudaStreamSynchronize(s));
    return VB_OK;
}

int vb_l2_normalize_batch(int elem, int dim, const void* rows, int64_t n, void* out) {
    VB_TRY(require_init());
    VB_REQUIRE((elem == VB_VECTOR || elem == VB_HALFVEC) && dim > 0 && (rows || n == 0) && out, "bad normalize arguments");
    if (n <= 0) return VB_OK;
    cudaStream_t s = ctx().stream;
    void *d_in, *d_out, *d_flag;
    const size_t raw = raw_row_bytes(elem, dim);
    VB_TRY(stage_in(elem, dim, rows, n, &d_in));
    VB_TRY(workspace(WSO_OUT, raw * (size_t)n, &d_out));
    VB_TRY(workspace(WSO_FLAG, 64, &d_flag));
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
    VB_TRY(require_init());
    VB_REQUIRE((elem == VB_VECTOR || elem == VB_HALFVEC) && dim > 0 && (rows || n == 0) && out, "bad binary_quantize arguments");
    if (n <= 0) return VB_OK;
    cudaStream_t s = ctx().stream;
    void *d_in, *d_out;
    const size_t nb = ((size_t)dim + 7) / 8;
    VB_TRY(stage_in(elem, dim, rows, n, &d_in));
    VB_TRY(workspace(WSO_OUT, nb * (size_t)n, &d_out));
    VB_TRY(quantize_rows(elem, dim, d_in, n, (uint8_t*)d_out));
    VB_CUDA(cudaMemcpyAsync(out, d_out, nb * (size_t)n, cudaMemcpyDeviceToHost, s));
    VB_CUDA(cudaStreamSynchronize(s));
    return VB_OK;
}

int vb_vector_to_halfvec_batch(int dim, const void* rows, int64_t n, void* out) {
    VB_TRY(require_init());
    VB_REQUIRE(dim > 0 && (rows || n == 0) && out, "bad cast arguments");
    if (n <= 0) return VB_OK;
    cudaStream_t s = ctx().stream;
    const int64_t total = n * dim;
    void *d_in, *d_out, *d_flag;
    VB_TRY(stage_in(VB_VECTOR, dim, rows, n, &d_in));
    VB_TRY(workspace(WSO_OUT, sizeof(__half) * (size_t)total, &d_out));
    VB_TRY(workspace(WSO_FLAG, 64, &d_flag));
    VB_TRY(to_half_rows(dim, d_in, n, d_out, (unsigned long long*)d_flag));
    unsigned long long bad = ~0ull;
    VB_CUDA(cudaMemcpyAsync(out, d_out, sizeof(__half) * (size_t)total, cudaMemcpyDeviceToHost, s));
    VB_CUDA(cudaMemcpyAsync(&bad, d_flag, sizeof(bad), cudaMemcpyDeviceToHost, s));
    VB_CUDA(cudaStreamSynchronize(s));
    if (bad != ~0ull) return half_range_error(reinterpret_cast<const float*>(rows)[bad]);
    return VB_OK;
}

int vb_halfvec_to_vector_batch(int dim, const void* rows, int64_t n, void* out) {
    VB_TRY(require_init());
    VB_REQUIRE(dim > 0 && (rows || n == 0) && out, "bad cast arguments");
    if (n <= 0) return VB_OK;
    cudaStream_t s = ctx().stream;
    const int64_t total = n * dim;
    void *d_in, *d_out;
    VB_TRY(stage_in(VB_HALFVEC, dim, rows, n, &d_in));
    VB_TRY(workspace(WSO_OUT, sizeof(float) * (size_t)total, &d_out));
    VB_TRY(to_float_rows(dim, d_in, n, d_out));
    VB_CUDA(cudaMemcpyAsync(out, d_out, sizeof(float) * (size_t)total, cudaMemcpyDeviceToHost, s));
    VB_CUDA(cudaStreamSynchronize(s));
    return VB_OK;
}

int vb_subvector_batch(int elem, int dim, const void* rows, int64_t n, int32_t start, int32_t count, void* out, int* out_dim) {
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
    VB_TRY(stage_in(elem, dim, rows, n, &d_in));
    VB_TRY(workspace(WSO_OUT, dense_bytes(elem, d, n), &d_out));
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
    VB_TRY(require_init());
    const char* fn = "vb_l2_normalize_batch_dev";
    VB_TRY(check_rows(fn, elem, dim, n, rows_dev, out_dev));
    if (n == 0) return VB_OK;
    const size_t bytes = dense_bytes(elem, dim, n);
    if (rows_dev != out_dev) VB_TRY(check_disjoint(fn, rows_dev, bytes, out_dev, bytes));   // in place is allowed
    cudaStream_t s = ctx().stream;
    void* d_flag;
    VB_TRY(workspace(WSO_FLAG, 64, &d_flag));
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
    VB_TRY(require_init());
    const char* fn = "vb_vector_to_halfvec_batch_dev";
    VB_TRY(check_rows(fn, VB_VECTOR, dim, n, rows_dev, out_dev));
    if (n == 0) return VB_OK;
    VB_TRY(check_disjoint(fn, rows_dev, dense_bytes(VB_VECTOR, dim, n), out_dev, dense_bytes(VB_HALFVEC, dim, n)));
    cudaStream_t s = ctx().stream;
    void* d_flag;
    VB_TRY(workspace(WSO_FLAG, 64, &d_flag));
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

}  // extern "C"
