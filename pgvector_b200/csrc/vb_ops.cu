// vb_ops.cu -- batched row transforms that sit beside the distance path:
//   vb_norm_batch          vector_norm / halfvec l2_norm       (src/vector.c:767-780, src/halfvec.c:703-720)
//   vb_l2_normalize_batch  l2_normalize / halfvec_l2_normalize (src/vector.c:785-819, src/halfvec.c:725-759)
//   vb_binary_quantize_batch  binary_quantize                  (src/vector.c:952-978, src/halfvec.c twin)
// The cosine opclasses normalise every indexed row and the query (src/ivfbuild.c:174-180,
// src/ivfscan.c:222-229, src/hnswutils.c:417-423); norms accumulate in fp64 like the reference.
// One warp per row; HBM bound (row read once, written once).
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

// mode 0: norms only; mode 1: normalise
template <int ELEM>
__global__ void norm_kernel(const uint8_t* __restrict__ in, size_t in_stride, int64_t n, int dim, int mode, double* __restrict__ norms,
                            uint8_t* __restrict__ out, size_t out_stride, int* __restrict__ overflow) {
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

}  // namespace vb

using namespace vb;

extern "C" {

int vb_norm_batch(int elem, int dim, const void* rows, int64_t n, double* out) {
    VB_TRY(require_init());
    VB_REQUIRE((elem == VB_VECTOR || elem == VB_HALFVEC) && dim > 0 && (rows || n == 0) && out, "bad norm arguments");
    if (n <= 0) return VB_OK;
    cudaStream_t s = ctx().stream;
    void *d_in, *d_out;
    VB_TRY(stage_in(elem, dim, rows, n, &d_in));
    VB_TRY(workspace(WSO_OUT, sizeof(double) * (size_t)n, &d_out));
    const unsigned grid = (unsigned)((n * 32 + 255) / 256);
    const size_t raw = raw_row_bytes(elem, dim);
    if (elem == VB_VECTOR) norm_kernel<VB_VECTOR><<<grid, 256, 0, s>>>((const uint8_t*)d_in, raw, n, dim, 0, (double*)d_out, nullptr, 0, nullptr);
    else norm_kernel<VB_HALFVEC><<<grid, 256, 0, s>>>((const uint8_t*)d_in, raw, n, dim, 0, (double*)d_out, nullptr, 0, nullptr);
    VB_CUDA(cudaGetLastError());
    count_launch();
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
    VB_CUDA(cudaMemsetAsync(d_flag, 0, sizeof(int), s));
    const unsigned grid = (unsigned)((n * 32 + 255) / 256);
    if (elem == VB_VECTOR)
        norm_kernel<VB_VECTOR><<<grid, 256, 0, s>>>((const uint8_t*)d_in, raw, n, dim, 1, nullptr, (uint8_t*)d_out, raw, (int*)d_flag);
    else
        norm_kernel<VB_HALFVEC><<<grid, 256, 0, s>>>((const uint8_t*)d_in, raw, n, dim, 1, nullptr, (uint8_t*)d_out, raw, (int*)d_flag);
    VB_CUDA(cudaGetLastError());
    count_launch();
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
    const size_t raw = raw_row_bytes(elem, dim);
    const size_t nb = ((size_t)dim + 7) / 8;
    VB_TRY(stage_in(elem, dim, rows, n, &d_in));
    VB_TRY(workspace(WSO_OUT, nb * (size_t)n, &d_out));
    const unsigned grid = (unsigned)(((size_t)n * nb + 255) / 256);
    if (elem == VB_VECTOR) binary_quantize_kernel<VB_VECTOR><<<grid, 256, 0, s>>>((const uint8_t*)d_in, raw, n, dim, (uint8_t*)d_out, nb);
    else binary_quantize_kernel<VB_HALFVEC><<<grid, 256, 0, s>>>((const uint8_t*)d_in, raw, n, dim, (uint8_t*)d_out, nb);
    VB_CUDA(cudaGetLastError());
    count_launch();
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
    VB_CUDA(cudaMemsetAsync(d_flag, 0xFF, sizeof(unsigned long long), s));
    to_half_kernel<<<(unsigned)((total + 255) / 256), 256, 0, s>>>((const float*)d_in, total, (__half*)d_out, (unsigned long long*)d_flag);
    VB_CUDA(cudaGetLastError());
    count_launch();
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
    to_float_kernel<<<(unsigned)((total + 255) / 256), 256, 0, s>>>((const __half*)d_in, total, (float*)d_out);
    VB_CUDA(cudaGetLastError());
    count_launch();
    VB_CUDA(cudaMemcpyAsync(out, d_out, sizeof(float) * (size_t)total, cudaMemcpyDeviceToHost, s));
    VB_CUDA(cudaStreamSynchronize(s));
    return VB_OK;
}

}  // extern "C"
