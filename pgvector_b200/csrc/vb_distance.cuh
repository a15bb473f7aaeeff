// vb_distance.cuh -- per-pair distance arithmetic shared by the scan, HNSW and k-means kernels.
// Restates the reference's kernels for the device: fp32 accumulation for L2 / inner product /
// cosine / L1 (src/vector.c:560-574, 607-617, 649-666, 725-735; halves widened exactly first,
// src/halfutils.c:29-240), integer popcounts for Hamming / Jaccard (src/bitutils.c:49-159), and
// the fmgr wrappers' fp64 epilogues (src/vector.c:576-750, src/bitvec.c:45-70).
#pragma once

#include "vb_common.cuh"

namespace vb {


__device__ __forceinline__ uint4 ldg_stream(const uint4* p) {
    // streaming read: rows are touched once per query, keep them out of L1
    uint4 r;
    asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
                 : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
                 : "l"(p));
    return r;
}

__device__ __forceinline__ uint32_t orderable_key(float f) {
    // monotone map float -> uint32; -0 == +0; NaN sorts last (float8 btree order)
    if (f != f) return 0xFFFFFFFFu;
    uint32_t u = __float_as_uint(f);
    if (u == 0x80000000u) u = 0;
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float key_to_float(uint32_t k) {
    if (k == 0xFFFFFFFFu) return __int_as_float(0x7FC00000);
    uint32_t u = (k & 0x80000000u) ? (k & 0x7FFFFFFFu) : ~k;
    return __uint_as_float(u);
}

// halfvec element arithmetic: float(a) * float(b) is exact in fp32 (22-bit product) and the addition rounds once, as in
// the reference's widen-then-accumulate loop (src/halfutils.c)
__device__ __forceinline__ float fh_fma(uint16_t a, uint16_t b, float c) {
    return __fmaf_rn(__half2float(__ushort_as_half(a)), __half2float(__ushort_as_half(b)), c);
}
__device__ __forceinline__ float fh_sub(uint16_t a, float c) { return __fsub_rn(__half2float(__ushort_as_half(a)), c); }

// the same read marked evict-first in L2 (random row gathers of a graph walk: each row is used once, and the lines it would
// displace -- the per-query visited tables, the neighbour lists -- are re-used)
__device__ __forceinline__ uint4 ldg_gather(const uint4* p) {
    uint64_t pol;
    asm("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol));
    uint4 r;
    asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.v4.u32 {%0,%1,%2,%3}, [%4], %5;"
                 : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
                 : "l"(p), "l"(pol));
    return r;
}

template <int ELEM, int METRIC>
struct Acc {
    // fp metrics: a = main sum, b = |row|^2, c = |query|^2 (cosine only)
    // bit metrics: a = popc(xor) or popc(and), b = popc(row), c = popc(query)
    float fa = 0.f, fb = 0.f, fc = 0.f;
    uint32_t ua = 0, ub = 0, uc = 0;

    __device__ __forceinline__ void add_f(float x, float q) {
        if (METRIC == VB_L2_SQUARED) {
            float d = x - q;
            fa = fmaf(d, d, fa);
        } else if (METRIC == VB_NEG_IP) {
            fa = fmaf(x, q, fa);
        } else if (METRIC == VB_L1) {
            fa += fabsf(x - q);
        } else {  // cosine
            fa = fmaf(x, q, fa);
            fb = fmaf(x, x, fb);
            fc = fmaf(q, q, fc);
        }
    }
    // halfvec element (raw bits) against an fp32 query element
    __device__ __forceinline__ void add_hf(uint16_t x, float q) {
        if (METRIC == VB_L2_SQUARED) {
            float d = fh_sub(x, q);
            fa = fmaf(d, d, fa);
        } else if (METRIC == VB_L1) {
            fa += fabsf(fh_sub(x, q));
        } else {
            add_f(__half2float(__ushort_as_half(x)), q);
        }
    }
    // halfvec element against a halfvec query element (both raw bits)
    __device__ __forceinline__ void add_hh(uint16_t x, uint16_t q) {
        if (METRIC == VB_NEG_IP) {
            fa = fh_fma(x, q, fa);
        } else if (METRIC == VB_COSINE) {
            fa = fh_fma(x, q, fa);
            fb = fh_fma(x, x, fb);
            fc = fh_fma(q, q, fc);
        } else {
            add_hf(x, __half2float(__ushort_as_half(q)));
        }
    }
    // one 16-byte row vector against the query image in shared memory
    __device__ __forceinline__ void add(uint4 r, const uint4* sq, int v) {
        if (ELEM == VB_VECTOR) {
            uint4 q = sq[v];
            add_f(__uint_as_float(r.x), __uint_as_float(q.x));
            add_f(__uint_as_float(r.y), __uint_as_float(q.y));
            add_f(__uint_as_float(r.z), __uint_as_float(q.z));
            add_f(__uint_as_float(r.w), __uint_as_float(q.w));
        } else if (ELEM == VB_HALFVEC) {
            uint4 q0 = sq[2 * v], q1 = sq[2 * v + 1];
            add_hf((uint16_t)(r.x & 0xffffu), __uint_as_float(q0.x));
            add_hf((uint16_t)(r.x >> 16), __uint_as_float(q0.y));
            add_hf((uint16_t)(r.y & 0xffffu), __uint_as_float(q0.z));
            add_hf((uint16_t)(r.y >> 16), __uint_as_float(q0.w));
            add_hf((uint16_t)(r.z & 0xffffu), __uint_as_float(q1.x));
            add_hf((uint16_t)(r.z >> 16), __uint_as_float(q1.y));
            add_hf((uint16_t)(r.w & 0xffffu), __uint_as_float(q1.z));
            add_hf((uint16_t)(r.w >> 16), __uint_as_float(q1.w));
        } else {
            uint4 q = sq[v];
            if (METRIC == VB_HAMMING) {
                ua += __popc(r.x ^ q.x) + __popc(r.y ^ q.y) + __popc(r.z ^ q.z) + __popc(r.w ^ q.w);
            } else {
                ua += __popc(r.x & q.x) + __popc(r.y & q.y) + __popc(r.z & q.z) + __popc(r.w & q.w);
                ub += __popc(r.x) + __popc(r.y) + __popc(r.z) + __popc(r.w);
                uc += __popc(q.x) + __popc(q.y) + __popc(q.z) + __popc(q.w);
            }
        }
    }
    // halfvec row vector against 8 query elements kept as packed halves (the fp32 image of a halfvec query
    // holds exact conversions of halves, so converting back and forth changes nothing)
    __device__ __forceinline__ void add_h(uint4 r, uint4 qh) {
        add_hh((uint16_t)(r.x & 0xffffu), (uint16_t)(qh.x & 0xffffu));
        add_hh((uint16_t)(r.x >> 16), (uint16_t)(qh.x >> 16));
        add_hh((uint16_t)(r.y & 0xffffu), (uint16_t)(qh.y & 0xffffu));
        add_hh((uint16_t)(r.y >> 16), (uint16_t)(qh.y >> 16));
        add_hh((uint16_t)(r.z & 0xffffu), (uint16_t)(qh.z & 0xffffu));
        add_hh((uint16_t)(r.z >> 16), (uint16_t)(qh.z >> 16));
        add_hh((uint16_t)(r.w & 0xffffu), (uint16_t)(qh.w & 0xffffu));
        add_hh((uint16_t)(r.w >> 16), (uint16_t)(qh.w >> 16));
    }
    template <int LPR>
    __device__ __forceinline__ void reduce() {
#pragma unroll
        for (int o = LPR / 2; o > 0; o >>= 1) {
            if (ELEM == VB_BIT) {
                ua += __shfl_xor_sync(0xffffffffu, ua, o);
                if (METRIC == VB_JACCARD) {
                    ub += __shfl_xor_sync(0xffffffffu, ub, o);
                    uc += __shfl_xor_sync(0xffffffffu, uc, o);
                }
            } else {
                fa += __shfl_xor_sync(0xffffffffu, fa, o);
                if (METRIC == VB_COSINE) {
                    fb += __shfl_xor_sync(0xffffffffu, fb, o);
                    fc += __shfl_xor_sync(0xffffffffu, fc, o);
                }
            }
        }
    }
    // the value handed to the AM: (double) of the fp32 kernel result, with the wrapper's epilogue
    __device__ __forceinline__ double value() const {
        if (ELEM == VB_BIT) {
            if (METRIC == VB_HAMMING) return (double)ua;
            // src/bitutils.c:127-130
            if (ua == 0) return 1.0;
            return 1.0 - ((double)ua / (double)((uint64_t)ub + (uint64_t)uc - (uint64_t)ua));
        }
        if (METRIC == VB_NEG_IP) return (double)(-fa);
        if (METRIC == VB_COSINE) {
            // src/vector.c:665, 690-695
            double s = (double)fa / sqrt((double)fb * (double)fc);
            if (s > 1.0) s = 1.0;
            else if (s < -1.0) s = -1.0;
            return 1.0 - s;
        }
        return (double)fa;
    }
};


// float key -> the operator's float8 (sqrt for <->, negate for inner_product)
__device__ __forceinline__ double finish_value(int metric, float key) {
    if (metric == VB_L2) return sqrt((double)key);
    if (metric == VB_IP) return -(double)key;
    return (double)key;
}

// arguments of the scan kernels (vb_scan.cu: LDG variant, vb_scan_bulk.cu: bulk-copy/TMA variant)
struct ScanArgs {
    const uint8_t* rows;
    size_t stride;        // padded row bytes
    int vec_per_row;      // stride / 16
    const uint8_t* queries;
    size_t qstride;       // bytes of one query image
    int qvec;             // qstride / 16
    // chunk-list mode
    const Chunk* chunks;
    const int* n_chunks_dev;
    // regular mode: every query x rows [0, n_rows) in chunks of rows_per_chunk
    int64_t n_rows;
    int64_t nq;
    int rows_per_chunk;
    int64_t chunks_per_q;
    int64_t out_stride;
    void* out;
};

// bulk-copy (TMA) variant; returns VB_EINVAL when the shape is not supported (caller falls back to the LDG variant)
int launch_scan_bulk(int elem, int metric, const ScanArgs& a, bool out_f64, int max_chunks_hint);
bool scan_bulk_supported(int elem, size_t stride, size_t qstride);

// monotone map double -> uint64 (same conventions as orderable_key)
__device__ __forceinline__ uint64_t orderable_key64(double d) {
    if (d != d) return ~0ull;
    uint64_t u = (uint64_t)__double_as_longlong(d);
    if (u == 0x8000000000000000ull) u = 0;
    return (u & 0x8000000000000000ull) ? ~u : (u | 0x8000000000000000ull);
}
__device__ __forceinline__ double key64_to_double(uint64_t k) {
    if (k == ~0ull) return __longlong_as_double(0x7FF8000000000000ll);
    uint64_t u = (k & 0x8000000000000000ull) ? (k & 0x7FFFFFFFFFFFFFFFull) : ~k;
    return __longlong_as_double((long long)u);
}

}  // namespace vb
