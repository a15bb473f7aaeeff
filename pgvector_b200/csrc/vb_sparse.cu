// vb_sparse.cu -- sparsevec on the device (SURVEY 8 f4): the distance functions of src/sparsevec.c:826-1057
// (l2_distance / l2_squared_distance / inner_product / negative_inner_product / cosine_distance / l1_distance),
// l2_norm / l2_normalize (src/sparsevec.c:1062-1150), a resident CSR row table and the exact (no index) top-k
// over it, filtered (row filters of vb_filter.cu) or over per-query candidate rows (re-rank), and the casts to and from
// sparsevec: vector / halfvec rows and integer[] / real[] / double precision[] / numeric[] arrays (array_to_sparsevec).
//
// A sparsevec is (dim, nnz, indices[nnz] ascending 0-based, values[nnz]) -- src/sparsevec.h:21-32; a batch of rows is
// CSR: row r = entries row_off[r] .. row_off[r+1] of idx[] / val[].
//
// Formulation.  The reference merges the two index lists with a moving cursor (one pair at a time, O(nnz_a + nnz_b)
// dependent steps).  Here ONE query faces many rows, so the query is staged once per CTA in shared memory
// (indices, values and a 1024-bucket directory over the index range) and every row entry LOOKS ITS INDEX UP in the
// query: bucket = index >> shift, then a binary search inside the bucket (1-2 probes for nnz <= 16000).  One warp per
// row, lanes stride the row's entries (coalesced 4-byte loads of idx / val: the row is read once, HBM bound at 8 bytes
// per stored entry).  The query entries NOT matched by the row contribute q^2 (L2) or |q| (L1): each warp keeps a bitmap
// of matched query positions in shared memory and sums the unmatched ones afterwards -- no subtraction of large sums,
// so no cancellation.  Inner product and cosine need no bitmap.  Sums are fp32 like the reference's (warp tree instead
// of index order: within 1e-5 relative of the fp64 truth, tested against the oracle).
#include "vb_common.cuh"
#include "vb_distance.cuh"
#include "vb_numeric.cuh"
#include "vb_typio.cuh"

#include <cub/device/device_scan.cuh>

#include <algorithm>
#include <cmath>
#include <cstring>
#include <type_traits>
#include <vector>

namespace vb {

constexpr int SP_WARPS = 8;
constexpr int SP_BUCKETS = 1024;
constexpr int SP_MAX_NNZ = 16000;           // SPARSEVEC_MAX_NNZ (src/sparsevec.h:12)
constexpr int SP_MAX_DIM = 1000000000;      // SPARSEVEC_MAX_DIM (src/sparsevec.h:11)

struct SparseTable {
    int dim = 0;
    int64_t n = 0, nnz = 0;
    int64_t cap_rows = 0, cap_nnz = 0;
    int64_t* row_off = nullptr;   // [n + 1]
    int32_t* idx = nullptr;
    float* val = nullptr;
};

// queries of a batch, CSR like the rows
struct SparseQueries {
    const int64_t* off;
    const int32_t* idx;
    const float* val;
};

__device__ __forceinline__ int sp_find(const int32_t* s_idx, const int32_t* s_bucket, int shift, int32_t key) {
    const int b = key >> shift;
    int lo = s_bucket[b], hi = s_bucket[b + 1];
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        const int32_t v = s_idx[mid];
        if (v == key) return mid;
        if (v < key) lo = mid + 1;
        else hi = mid;
    }
    return -1;
}

// A query staged in shared memory (sp_stage): its indices and values, the bucket directory and the matched-position
// bitmaps of the warps (L2 squared and L1 only).
struct SpStaged {
    const int32_t* idx;
    const float* val;
    const int32_t* bucket;
    uint32_t* flags;   // warp w's bitmap: flags + w * nwords
    int qn, nwords;
};

// where a query of qn entries is staged in the dynamic shared memory
__device__ __forceinline__ SpStaged sp_layout(uint8_t* smem, int qn) {
    int32_t* s_idx = reinterpret_cast<int32_t*>(smem);
    float* s_val = reinterpret_cast<float*>(s_idx + qn);
    int32_t* s_bucket = reinterpret_cast<int32_t*>(s_val + qn);
    uint32_t* s_flags = reinterpret_cast<uint32_t*>(s_bucket + SP_BUCKETS + 1);
    return SpStaged{s_idx, s_val, s_bucket, s_flags, qn, (qn + 31) >> 5};
}

// Every thread of the CTA stages query q; the staging ends with a barrier.  *s_qnorm (cosine): the query's fp32 sum of
// squares.  The caller must make sure no warp still reads a previous query's staging.
template <int KEY>
__device__ __forceinline__ SpStaged sp_stage(const SparseQueries& Q, int q, int shift, uint8_t* smem, float* s_qnorm) {
    const int64_t qb = Q.off[q];
    const int qn = (int)(Q.off[q + 1] - qb);
    const SpStaged sq = sp_layout(smem, qn);
    int32_t* s_idx = const_cast<int32_t*>(sq.idx);
    float* s_val = const_cast<float*>(sq.val);
    int32_t* s_bucket = const_cast<int32_t*>(sq.bucket);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

    for (int i = threadIdx.x; i < qn; i += blockDim.x) {
        s_idx[i] = Q.idx[qb + i];
        s_val[i] = Q.val[qb + i];
    }
    __syncthreads();
    // bucket b starts at the first query entry with index >= b << shift
    for (int b = threadIdx.x; b <= SP_BUCKETS; b += blockDim.x) {
        const int64_t first = (int64_t)b << shift;
        int lo = 0, hi = qn;
        while (lo < hi) {
            const int mid = (lo + hi) >> 1;
            if ((int64_t)s_idx[mid] < first) lo = mid + 1;
            else hi = mid;
        }
        s_bucket[b] = lo;
    }
    if (KEY == VB_COSINE && warp == 0) {   // fp32 sum of squares of the query (normb, src/sparsevec.c:992-993)
        float s = 0.f;
        for (int i = lane; i < qn; i += 32) s += s_val[i] * s_val[i];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
        if (lane == 0) *s_qnorm = s;
    }
    __syncthreads();
    return sq;
}

// The per-row arithmetic of every sparse scan: one warp scores the row of entries beg .. end against the staged query.
// Lanes stride the row's entries; the query entries the row does not match are summed from the warp's bitmap `flags`
// (L2 squared, L1); then an xor-shuffle reduce.  Returns, on every lane, the float8 of KEY's function -- `metric` tells
// VB_IP from VB_NEG_IP, sqrt_l2 takes the square root for VB_L2 -- whose float is the ordering key.  Every scan calls
// this one body, so their distances agree bit for bit.
template <int KEY>
__device__ __forceinline__ double sp_score_row(int64_t beg, int64_t end, const int32_t* __restrict__ idx, const float* __restrict__ val,
                                               const SpStaged& sq, int shift, uint32_t* flags, float qnorm, int metric, bool sqrt_l2,
                                               int lane) {
    constexpr bool FLAGS = KEY == VB_L2_SQUARED || KEY == VB_L1;
    const int32_t* s_idx = sq.idx;
    const float* s_val = sq.val;
    const int32_t* s_bucket = sq.bucket;
    const int qn = sq.qn, nwords = sq.nwords;
    if (FLAGS) {
        for (int w = lane; w < nwords; w += 32) flags[w] = 0u;
        __syncwarp();
    }
    float acc = 0.f, rn = 0.f;
    for (int64_t p = beg + lane; p < end; p += 32) {
        const int32_t ri = __ldg(idx + p);
        const float rv = __ldg(val + p);
        const int pos = sp_find(s_idx, s_bucket, shift, ri);
        const float qv = pos >= 0 ? s_val[pos] : 0.f;
        if (KEY == VB_L2_SQUARED) {
            const float t = rv - qv;
            acc += t * t;
        } else if (KEY == VB_L1) {
            acc += fabsf(rv - qv);
        } else {
            acc += rv * qv;
            if (KEY == VB_COSINE) rn += rv * rv;
        }
        if (FLAGS && pos >= 0) atomicOr(&flags[pos >> 5], 1u << (pos & 31));
    }
    if (FLAGS) {
        __syncwarp();
        for (int w = lane; w < nwords; w += 32) {
            uint32_t m = ~flags[w];
            if (w == nwords - 1 && (qn & 31)) m &= (1u << (qn & 31)) - 1u;
            while (m) {
                const int b = __ffs(m) - 1;
                m &= m - 1;
                const float qv = s_val[w * 32 + b];
                acc += KEY == VB_L2_SQUARED ? qv * qv : fabsf(qv);
            }
        }
        __syncwarp();
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        acc += __shfl_xor_sync(0xffffffffu, acc, o);
        if (KEY == VB_COSINE) rn += __shfl_xor_sync(0xffffffffu, rn, o);
    }
    double v;
    if (KEY == VB_COSINE) {
        // src/sparsevec.c:985-1009: similarity / sqrt((double) norma * (double) normb), clamped, 1 - similarity
        double sim = (double)acc / sqrt((double)rn * (double)qnorm);
        if (sim > 1.0) sim = 1.0;
        else if (sim < -1.0) sim = -1.0;
        v = 1.0 - sim;
    } else if (KEY == VB_NEG_IP) {
        v = metric == VB_IP ? (double)acc : (double)-acc;
    } else if (KEY == VB_L2_SQUARED) {
        v = sqrt_l2 ? sqrt((double)acc) : (double)acc;
    } else {
        v = (double)acc;
    }
    return v;
}

// KEY: VB_L2_SQUARED, VB_NEG_IP, VB_COSINE or VB_L1.  out_d (float8 of SQL function `metric`) or out_f (ordering key).
// grid: x = row slices, y = queries.  out[(q * n + r)].
template <int KEY>
__global__ void __launch_bounds__(SP_WARPS * 32)
sparse_scan_kernel(SparseQueries Q, int shift, const int64_t* __restrict__ row_off, const int32_t* __restrict__ idx,
                   const float* __restrict__ val, int64_t n, int metric, double* __restrict__ out_d, float* __restrict__ out_f) {
    extern __shared__ __align__(16) uint8_t smem[];
    __shared__ float s_qnorm;
    const int q = blockIdx.y;
    const SpStaged sq = sp_stage<KEY>(Q, q, shift, smem, &s_qnorm);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    uint32_t* flags = sq.flags + (size_t)warp * sq.nwords;
    const bool sqrt_l2 = metric == VB_L2 && out_d;
    const int64_t wstride = (int64_t)gridDim.x * SP_WARPS;
    for (int64_t r = (int64_t)blockIdx.x * SP_WARPS + warp; r < n; r += wstride) {
        const double v = sp_score_row<KEY>(row_off[r], row_off[r + 1], idx, val, sq, shift, flags, s_qnorm, metric, sqrt_l2, lane);
        if (lane == 0) {
            const size_t at = (size_t)q * (size_t)n + (size_t)r;
            if (out_d) out_d[at] = v;
            else out_f[at] = (float)v;
        }
    }
}

// The listed rows of a chunk list: row j of chunk c is table row rows[c.row_begin + j], its ordering key goes to
// out[c.out_off + j].  *n_chunks chunks; each CTA takes a contiguous slice of them and stages a query only when the
// slice moves on to the next one (the chunks of a query are consecutive), so a query is staged once per CTA that
// scores its rows.  One warp per listed row, through sp_score_row: keys bit-identical to sparse_scan_kernel's out_f.
// (The bound of 4 CTAs per SM lets ptxas use up to 64 registers; left to itself it stops at 32 and spills.)
template <int KEY>
__global__ void __launch_bounds__(SP_WARPS * 32, 4)
sparse_gather_kernel(SparseQueries Q, int shift, const int64_t* __restrict__ row_off, const int32_t* __restrict__ idx,
                     const float* __restrict__ val, const int64_t* __restrict__ rows, const Chunk* __restrict__ chunks,
                     const int* __restrict__ n_chunks, int metric, float* __restrict__ out) {
    extern __shared__ __align__(16) uint8_t smem[];
    __shared__ float s_qnorm;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int64_t total = *n_chunks;
    const int64_t per = (total + gridDim.x - 1) / gridDim.x;
    const int64_t c_begin = per * blockIdx.x;
    const int64_t c_end = min(total, c_begin + per);
    int cur_q = -1, qn = 0;
    for (int64_t c = c_begin; c < c_end; ++c) {
        const Chunk ch = chunks[c];
        if (ch.q != cur_q) {   // uniform over the CTA
            __syncthreads();   // every warp is done with the previous query
            qn = sp_stage<KEY>(Q, ch.q, shift, smem, &s_qnorm).qn;
            cur_q = ch.q;
        }
        const SpStaged sq = sp_layout(smem, qn);
        uint32_t* flags = sq.flags + (size_t)warp * sq.nwords;
        for (int j = warp; j < ch.n_rows; j += SP_WARPS) {
            const int64_t r = rows[ch.row_begin + j];
            const double v = sp_score_row<KEY>(row_off[r], row_off[r + 1], idx, val, sq, shift, flags, s_qnorm, metric, false, lane);
            if (lane == 0) out[ch.out_off + j] = (float)v;
        }
    }
}

static size_t sparse_smem_bytes(int max_qnnz) {
    const size_t words = ((size_t)max_qnnz + 31) / 32;
    return (size_t)max_qnnz * 8 + (SP_BUCKETS + 1) * 4 + words * 4 * SP_WARPS + 16;
}

static int sparse_shift(int dim) {
    int shift = 0;
    while ((((int64_t)dim - 1) >> shift) >= SP_BUCKETS) ++shift;
    return shift;
}

// distances of nq queries against the n CSR rows; metric = the SQL function (out_d) or its ordering key (out_f)
static int launch_sparse_scan(int metric, int dim, SparseQueries Q, int64_t nq, int max_qnnz, const int64_t* row_off, const int32_t* idx,
                              const float* val, int64_t n, double* out_d, float* out_f) {
    if (n <= 0 || nq <= 0) return VB_OK;
    Context& c = ctx();
    const size_t smem = sparse_smem_bytes(max_qnnz);
    const int shift = sparse_shift(dim);
    int64_t gx = std::max<int64_t>(1, (2 * (int64_t)c.sm_count + nq - 1) / nq);
    gx = std::min<int64_t>(gx, (n + SP_WARPS - 1) / SP_WARPS);
    VB_REQUIRE(nq <= 65535, "at most 65535 sparse queries per launch");
    dim3 grid((unsigned)gx, (unsigned)nq);
    const int km = key_metric(metric);
#define SP_LAUNCH(KEY)                                                                                                     \
    do {                                                                                                                   \
        VB_CUDA(cudaFuncSetAttribute(sparse_scan_kernel<KEY>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));      \
        sparse_scan_kernel<KEY><<<grid, SP_WARPS * 32, smem, c.stream>>>(Q, shift, row_off, idx, val, n, metric, out_d, out_f); \
    } while (0)
    switch (km) {
        case VB_L2_SQUARED: SP_LAUNCH(VB_L2_SQUARED); break;
        case VB_NEG_IP: SP_LAUNCH(VB_NEG_IP); break;
        case VB_COSINE: SP_LAUNCH(VB_COSINE); break;
        case VB_L1: SP_LAUNCH(VB_L1); break;
        default: set_error("metric %d is not defined for sparsevec", metric); return VB_EINVAL;
    }
#undef SP_LAUNCH
    VB_CUDA(cudaGetLastError());
    count_launch();
    return VB_OK;
}

constexpr int SP_CHUNK_ROWS = 256;   // listed rows per chunk of gather work: 32 per warp

// ordering keys of the chunk list's rows (sparse_gather_kernel); *n_chunks_dev <= max_chunks chunks
static int launch_sparse_gather(int key_metric, int dim, SparseQueries Q, int max_qnnz, const SparseTable& t, const int64_t* rows,
                                const Chunk* chunks, const int* n_chunks_dev, int max_chunks, float* out) {
    if (max_chunks <= 0) return VB_OK;
    Context& c = ctx();
    const size_t smem = sparse_smem_bytes(max_qnnz);
    const int shift = sparse_shift(dim);
    const unsigned grid = (unsigned)std::min(max_chunks, 8 * c.sm_count);
#define SP_LAUNCH(KEY)                                                                                                     \
    do {                                                                                                                   \
        VB_CUDA(cudaFuncSetAttribute(sparse_gather_kernel<KEY>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));    \
        sparse_gather_kernel<KEY><<<grid, SP_WARPS * 32, smem, c.stream>>>(Q, shift, t.row_off, t.idx, t.val, rows, chunks, n_chunks_dev, \
                                                                           key_metric, out);                               \
    } while (0)
    switch (key_metric) {
        case VB_L2_SQUARED: SP_LAUNCH(VB_L2_SQUARED); break;
        case VB_NEG_IP: SP_LAUNCH(VB_NEG_IP); break;
        case VB_COSINE: SP_LAUNCH(VB_COSINE); break;
        case VB_L1: SP_LAUNCH(VB_L1); break;
        default: set_error("metric %d is not defined for sparsevec", key_metric); return VB_EINVAL;
    }
#undef SP_LAUNCH
    VB_CUDA(cudaGetLastError());
    count_launch();
    return VB_OK;
}

// ----------------------------------------------------------------------------- norm / normalize

// mode 0: norms (fp64 sum of squares, src/sparsevec.c:1062-1077).  mode 1: quotients (float)(x / norm) into q_out,
// entries kept (quotient != 0) per row into kept, overflow flag (src/sparsevec.c:1100-1113)
__global__ void sparse_norm_kernel(const int64_t* __restrict__ row_off, const float* __restrict__ val, int64_t n, int mode,
                                   double* __restrict__ norms, float* __restrict__ q_out, int64_t* __restrict__ kept, int* __restrict__ overflow) {
    const int64_t r = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) / 32;
    const int lane = threadIdx.x % 32;
    if (r >= n) return;
    const int64_t beg = row_off[r], end = row_off[r + 1];
    double s = 0.0;
    for (int64_t p = beg + lane; p < end; p += 32) {
        const double x = (double)val[p];
        s += x * x;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    const double norm = sqrt(s);
    if (mode == 0) {
        if (lane == 0) norms[r] = norm;
        return;
    }
    int k = 0;
    bool inf = false;
    for (int64_t p = beg + lane; p < end; p += 32) {
        const float v = norm > 0 ? (float)((double)val[p] / norm) : 0.f;
        inf |= isinf(v);
        q_out[p] = v;
        k += v != 0.f;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) k += __shfl_xor_sync(0xffffffffu, k, o);
    if (lane == 0) kept[r] = k;
    if (inf) atomicExch(overflow, 1);
}

// rows without their zero quotients, in index order (src/sparsevec.c:1115-1140)
__global__ void sparse_compact_kernel(const int64_t* __restrict__ row_off, const int32_t* __restrict__ idx, const float* __restrict__ q_in,
                                      int64_t n, const int64_t* __restrict__ out_off, int32_t* __restrict__ out_idx,
                                      float* __restrict__ out_val) {
    const int64_t r = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) / 32;
    const int lane = threadIdx.x % 32;
    if (r >= n) return;
    const int64_t beg = row_off[r], end = row_off[r + 1];
    int64_t w = out_off[r];
    for (int64_t p0 = beg; p0 < end; p0 += 32) {
        const int64_t p = p0 + lane;
        const float v = p < end ? q_in[p] : 0.f;
        const bool keep = v != 0.f;
        const unsigned m = __ballot_sync(0xffffffffu, keep);
        if (keep) {
            const int64_t at = w + __popc(m & ((1u << lane) - 1u));
            out_idx[at] = idx[p];
            out_val[at] = v;
        }
        w += __popc(m);
    }
}

__global__ void sparse_segments_kernel(int64_t nseg, int64_t n, int64_t* begin, int32_t* lens) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i < nseg) {
        begin[i] = i * n;
        lens[i] = (int32_t)n;
    }
}

// Selected position -> row number, ordering key -> float8 (out_d), or the float of that float8 (out_f, the _dev
// variants).  rows == nullptr: the position is the row number (the scan of every row); else entry p of segment s is row
// rows[seg_rows[s * seg_rows_stride] + p] (a position list per segment).
__global__ void sparse_finish_kernel(int metric, int64_t total, int k, const int32_t* __restrict__ pos, const float* __restrict__ key,
                                     const int64_t* __restrict__ rows, const int64_t* __restrict__ seg_rows, int seg_rows_stride,
                                     int64_t* __restrict__ out_ids, double* __restrict__ out_d, float* __restrict__ out_f) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= total) return;
    const int32_t p = pos[i];
    out_ids[i] = !rows || p < 0 ? (int64_t)p : rows[seg_rows[(i / k) * seg_rows_stride] + p];
    // the ordering key is the float8 of the function except for <-> (sqrt of the fp32 L2 squared, src/sparsevec.c:872-883)
    const double v = metric == VB_L2 ? sqrt((double)key[i]) : (double)key[i];
    if (out_f) out_f[i] = (float)v;
    else out_d[i] = v;
}

// -1 / +inf: the result of every query over an empty table (_dev variants)
__global__ void sparse_pad_kernel(int64_t total, int64_t* __restrict__ out_ids, float* __restrict__ out_f) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= total) return;
    out_ids[i] = -1;
    out_f[i] = INFINITY;
}

// ----------------------------------------------------------------------------- CSR validation on the device

// What sparse_check_kernel finds in n device CSR rows, read back in one copy by check_csr_dev.  bad: the first defect as
// (row << 8) | SPC_* (~0 = none), the one check_csr would report first; max_nnz: the largest row nnz (sizes the query
// staging, sparse_smem_bytes); total: off[n].  over: the casts to halfvec, the first entry whose value overflows
// binary16 (INT64_MAX = none).
struct SparseCheck {
    unsigned long long bad;
    long long max_nnz;
    long long total;
    long long over;
};
enum { SPC_START = 1, SPC_DECREASE = 2, SPC_NNZ = 3, SPC_NULL_IDX = 4, SPC_BOUNDS = 5, SPC_ORDER = 6 };
constexpr size_t SPC_READ = offsetof(SparseCheck, over);   // the bytes a validation reads back (24)

__global__ void sparse_check_init_kernel(SparseCheck* c) {
    c->bad = ~0ull;
    c->max_nnz = 0;
    c->total = 0;
    c->over = INT64_MAX;
}

// One warp per row, check_csr's rules in check_csr's order: the offsets (off[0] = 0, non-decreasing, at most
// SP_MAX_NNZ per row), then the entries (each index inside [0, dim), then strictly above the one before; the first bad
// entry decides).  A row whose entries lie outside [0, off[n]) is not read: that happens only when some row's offsets
// are bad, and that row is reported.  The smallest (row << 8) | code wins (atomicMin), so the defect reported is the
// first one check_csr meets.
__global__ void __launch_bounds__(256) sparse_check_kernel(int64_t n, const int64_t* __restrict__ off, const int32_t* __restrict__ idx,
                                                           int dim, SparseCheck* __restrict__ out) {
    const int64_t r = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (r >= n) return;   // whole warps
    const int64_t beg = off[r], end = off[r + 1], total = off[n];
    const int64_t len = end - beg;
    int code = 0;
    if (r == 0 && beg != 0) code = SPC_START;
    else if (len < 0) code = SPC_DECREASE;
    else if (len > SP_MAX_NNZ) code = SPC_NNZ;
    else if (len > 0 && !idx) code = SPC_NULL_IDX;
    else if (beg >= 0 && end <= total) {
        for (int64_t p0 = beg; p0 < end && !code; p0 += 32) {
            const int64_t p = p0 + lane;
            int c = 0;
            if (p < end) {
                const int32_t v = idx[p];
                if (v < 0 || v >= dim) c = SPC_BOUNDS;
                else if (p > beg && v <= idx[p - 1]) c = SPC_ORDER;
            }
            const unsigned m = __ballot_sync(0xffffffffu, c != 0);
            if (m) code = __shfl_sync(0xffffffffu, c, __ffs(m) - 1);
        }
    }
    if (lane == 0) {
        if (code) atomicMin(&out->bad, ((unsigned long long)r << 8) | (unsigned)code);
        else atomicMax(&out->max_nnz, (long long)len);
        if (r == n - 1) out->total = total;
    }
}

// check_csr's text for a defect sparse_check_kernel found, with the row number
static int sparse_check_error(const char* what, unsigned long long bad) {
    const long long row = (long long)(bad >> 8);
    switch ((int)(bad & 0xFF)) {
        case SPC_START: set_error("%s: offsets must start at 0", what); break;
        case SPC_DECREASE: set_error("%s: offsets must not decrease (row %lld)", what, row); break;
        case SPC_NNZ: set_error("sparsevec cannot have more than %d non-zero elements (row %lld)", SP_MAX_NNZ, row); break;
        case SPC_NULL_IDX: set_error("%s: null indices (row %lld)", what, row); break;
        case SPC_BOUNDS: set_error("sparsevec index out of bounds (row %lld)", row); break;
        default: set_error("sparsevec indices must be in ascending order (row %lld)", row); break;
    }
    return VB_EINVAL;
}

// Launch the initialisation and the check of n >= 1 device CSR rows into *chk (a range of sc); no read.
static int launch_sparse_check(Scratch& sc, int dim, int64_t n, const int64_t* off, const int32_t* idx, SparseCheck** chk) {
    cudaStream_t s = ctx().stream;
    void* d;
    VB_TRY(sc.take(sizeof(SparseCheck), &d));
    *chk = (SparseCheck*)d;
    sparse_check_init_kernel<<<1, 1, 0, s>>>(*chk);
    sparse_check_kernel<<<(unsigned)((n * 32 + 255) / 256), 256, 0, s>>>(n, off, idx, dim, *chk);
    VB_CUDA(cudaGetLastError());
    count_launch(2);
    return VB_OK;
}

// check_csr for n >= 1 device CSR rows: one sparse_check_kernel pass and one read of its 24-byte result (which
// synchronises).  *max_nnz / *total (optional): the largest row nnz and off[n].
static int check_csr_dev(const char* what, int dim, int64_t n, const int64_t* off, const int32_t* idx, int* max_nnz, int64_t* total) {
    Scratch sc;
    VB_REQUIRE(dim >= 1 && dim <= SP_MAX_DIM, "sparsevec must have between 1 and %d dimensions", SP_MAX_DIM);
    VB_REQUIRE(off, "%s: offsets must start at 0", what);
    SparseCheck h{~0ull, 0, 0, 0};
    SparseCheck* d;
    VB_TRY(launch_sparse_check(sc, dim, n, off, idx, &d));
    cudaStream_t s = ctx().stream;
    VB_CUDA(cudaMemcpyAsync(&h, d, SPC_READ, cudaMemcpyDeviceToHost, s));
    VB_CUDA(cudaStreamSynchronize(s));
    if (h.bad != ~0ull) return sparse_check_error(what, h.bad);
    if (max_nnz) *max_nnz = (int)h.max_nnz;
    if (total) *total = h.total;
    return VB_OK;
}

int sparse_csr_check_dev(const char* what, int dim, int64_t n, const int64_t* off, const int32_t* idx, int64_t* total) {
    return check_csr_dev(what, dim, n, off, idx, nullptr, total);
}

static bool sparse_metric_ok(int metric) {
    return metric == VB_L2_SQUARED || metric == VB_L2 || metric == VB_IP || metric == VB_NEG_IP || metric == VB_COSINE || metric == VB_L1;
}

// Validate host CSR: offsets non-decreasing from 0, row nnz <= SPARSEVEC_MAX_NNZ, indices ascending inside [0, dim)
// (what sparsevec_in / sparsevec_recv guarantee for stored values, src/sparsevec.c:88-104, 511-521)
static int check_csr(const char* what, int dim, int64_t n, const int64_t* off, const int32_t* idx, int* max_nnz) {
    VB_REQUIRE(dim >= 1 && dim <= SP_MAX_DIM, "sparsevec must have between 1 and %d dimensions", SP_MAX_DIM);
    VB_REQUIRE(off && off[0] == 0, "%s: offsets must start at 0", what);
    int mx = 0;
    for (int64_t r = 0; r < n; ++r) {
        const int64_t len = off[r + 1] - off[r];
        VB_REQUIRE(len >= 0, "%s: offsets must not decrease (row %lld)", what, (long long)r);
        VB_REQUIRE(len <= SP_MAX_NNZ, "sparsevec cannot have more than %d non-zero elements", SP_MAX_NNZ);
        VB_REQUIRE(len == 0 || idx, "%s: null indices", what);
        for (int64_t p = off[r]; p < off[r + 1]; ++p) {
            VB_REQUIRE(idx[p] >= 0 && idx[p] < dim, "sparsevec index out of bounds");
            VB_REQUIRE(p == off[r] || idx[p] > idx[p - 1], "sparsevec indices must be in ascending order");
        }
        mx = std::max(mx, (int)len);
    }
    if (max_nnz) *max_nnz = mx;
    return VB_OK;
}

// queries to the device: [off (nq + 1) | idx | val] in one range of sc
static int upload_sparse_queries(Scratch& sc, int64_t nq, const int64_t* off, const int32_t* idx, const float* val, SparseQueries* Q) {
    const int64_t tot = off[nq];
    const size_t b_off = sizeof(int64_t) * (size_t)(nq + 1);
    const size_t b_idx = (sizeof(int32_t) * (size_t)tot + 15) & ~(size_t)15;
    void* d;
    VB_TRY(sc.take(b_off + b_idx + sizeof(float) * (size_t)tot + 64, &d));
    cudaStream_t s = ctx().stream;
    uint8_t* p = (uint8_t*)d;
    VB_CUDA(cudaMemcpyAsync(p, off, b_off, cudaMemcpyHostToDevice, s));
    if (tot > 0) {
        VB_CUDA(cudaMemcpyAsync(p + b_off, idx, sizeof(int32_t) * (size_t)tot, cudaMemcpyHostToDevice, s));
        VB_CUDA(cudaMemcpyAsync(p + b_off + b_idx, val, sizeof(float) * (size_t)tot, cudaMemcpyHostToDevice, s));
    }
    Q->off = (const int64_t*)p;
    Q->idx = (const int32_t*)(p + b_off);
    Q->val = (const float*)(p + b_off + b_idx);
    return VB_OK;
}

static int sparse_reserve(SparseTable& t, int64_t rows, int64_t nnz) {
    cudaStream_t s = ctx().stream;
    if (rows + 1 > t.cap_rows) {
        const int64_t cap = std::max<int64_t>(rows + 1, t.cap_rows * 2);
        int64_t* d;
        if (cudaMalloc(&d, sizeof(int64_t) * (size_t)cap) != cudaSuccess) {
            set_error("out of device memory (sparse row offsets)");
            return VB_ENOMEM;
        }
        if (t.row_off) {
            VB_CUDA(cudaMemcpyAsync(d, t.row_off, sizeof(int64_t) * (size_t)(t.n + 1), cudaMemcpyDeviceToDevice, s));
            VB_CUDA(cudaStreamSynchronize(s));
            cudaFree(t.row_off);
        } else {
            VB_CUDA(cudaMemsetAsync(d, 0, sizeof(int64_t), s));
        }
        t.row_off = d;
        t.cap_rows = cap;
    }
    if (nnz > t.cap_nnz) {
        const int64_t cap = std::max<int64_t>(nnz, t.cap_nnz * 2);
        int32_t* di;
        float* dv;
        if (cudaMalloc(&di, sizeof(int32_t) * (size_t)cap) != cudaSuccess) {
            set_error("out of device memory (sparse indices)");
            return VB_ENOMEM;
        }
        if (cudaMalloc(&dv, sizeof(float) * (size_t)cap) != cudaSuccess) {
            cudaFree(di);
            set_error("out of device memory (sparse values)");
            return VB_ENOMEM;
        }
        if (t.nnz > 0) {
            VB_CUDA(cudaMemcpyAsync(di, t.idx, sizeof(int32_t) * (size_t)t.nnz, cudaMemcpyDeviceToDevice, s));
            VB_CUDA(cudaMemcpyAsync(dv, t.val, sizeof(float) * (size_t)t.nnz, cudaMemcpyDeviceToDevice, s));
            VB_CUDA(cudaStreamSynchronize(s));
        }
        if (t.idx) cudaFree(t.idx);
        if (t.val) cudaFree(t.val);
        t.idx = di;
        t.val = dv;
        t.cap_nnz = cap;
    }
    return VB_OK;
}

__global__ void sparse_shift_offsets_kernel(int64_t* off, int64_t n, int64_t add) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i < n) off[i] += add;
}

// queries q0 .. q0 + m of a call's CSR batch to the device, offsets rebased to 0
static int upload_query_range(Scratch& sc, int64_t q0, int64_t m, const int64_t* q_off, const int32_t* q_idx, const float* q_val, SparseQueries* Q) {
    std::vector<int64_t> off((size_t)m + 1);
    for (int64_t i = 0; i <= m; ++i) off[(size_t)i] = q_off[q0 + i] - q_off[q0];
    VB_TRY(upload_sparse_queries(sc, m, off.data(), q_idx + q_off[q0], q_val + q_off[q0], Q));
    VB_CUDA(cudaStreamSynchronize(ctx().stream));   // `off` is a local vector
    return VB_OK;
}

// The queries q0 .. q0 + m of a call: host CSR is uploaded (upload_query_range); device CSR is read in place, its
// offsets absolute into the call's q_idx / q_val (sp_stage reads Q.off[q] .. Q.off[q + 1]), so nothing is copied.
static int sub_batch_queries(Scratch& sc, bool host, int64_t q0, int64_t m, const int64_t* q_off, const int32_t* q_idx, const float* q_val,
                             SparseQueries* Q) {
    if (host) return upload_query_range(sc, q0, m, q_off, q_idx, q_val, Q);
    *Q = SparseQueries{q_off + q0, q_idx, q_val};
    return VB_OK;
}

// The arguments every sparse top-k checks, in vb_sparse_exact_topk's order and with its texts (the dimension check
// after nq <= 0, which returns early; *max_q = the largest query nnz).  host == false: the query CSR is on the device
// and is validated there (check_csr_dev).
static int sparse_topk_args(vb_sparse_table* h, int metric, int q_dim, int64_t nq, const int64_t* q_off, const int32_t* q_idx,
                            const float* q_val, int k, bool host, int* max_q);

// The selection and the epilogue of a sub-batch of m queries whose ordering keys are in `key_runs`: the k nearest of
// each segment, position -> row number (rows / seg_rows / seg_rows_stride: see sparse_finish_kernel).  out_f == nullptr:
// the float8s are copied to out_ids / out_dist (host); else the ids and the floats go to out_ids / out_f (device), and
// nothing is waited for.
static int sparse_select_finish(int metric, int64_t m, int k, const float* key_runs, const int64_t* seg_begin, const int32_t* seg_len,
                                const int64_t* rows, const int64_t* seg_rows, int seg_rows_stride, int64_t* out_ids, double* out_dist,
                                float* out_f = nullptr) {
    Scratch sc;
    cudaStream_t s = ctx().stream;
    void *d_pos, *d_out;
    VB_TRY(sc.take((sizeof(int32_t) + sizeof(float)) * (size_t)m * k, &d_pos));
    int32_t* pos = (int32_t*)d_pos;
    float* key = (float*)(pos + (size_t)m * k);
    VB_TRY(launch_segment_topk_v(key_runs, seg_begin, seg_len, nullptr, nullptr, m, k, pos, key));
    if (out_f) {
        sparse_finish_kernel<<<(unsigned)((m * k + 255) / 256), 256, 0, s>>>(metric, m * k, k, pos, key, rows, seg_rows, seg_rows_stride,
                                                                             out_ids, nullptr, out_f);
        VB_CUDA(cudaGetLastError());
        count_launch();
        return VB_OK;
    }
    VB_TRY(sc.take((sizeof(int64_t) + sizeof(double)) * (size_t)m * k, &d_out));
    int64_t* o_ids = (int64_t*)d_out;
    double* o_d = (double*)(o_ids + (size_t)m * k);
    sparse_finish_kernel<<<(unsigned)((m * k + 255) / 256), 256, 0, s>>>(metric, m * k, k, pos, key, rows, seg_rows, seg_rows_stride, o_ids,
                                                                         o_d, nullptr);
    VB_CUDA(cudaGetLastError());
    count_launch();
    VB_CUDA(cudaMemcpyAsync(out_ids, o_ids, sizeof(int64_t) * (size_t)m * k, cudaMemcpyDeviceToHost, s));
    VB_CUDA(cudaMemcpyAsync(out_dist, o_d, sizeof(double) * (size_t)m * k, cudaMemcpyDeviceToHost, s));
    VB_CUDA(cudaStreamSynchronize(s));
    return VB_OK;
}

constexpr int64_t SP_MAX_BATCH = 65535;   // queries per sub-batch (the grid.y limit of sparse_scan_kernel)

}  // namespace vb

using namespace vb;

struct vb_sparse_table {
    SparseTable t;
    uint64_t uid = vb::next_owner_uid();
};

namespace vb {

static int sparse_topk_args(vb_sparse_table* h, int metric, int q_dim, int64_t nq, const int64_t* q_off, const int32_t* q_idx,
                            const float* q_val, int k, bool host, int* max_q) {
    VB_REQUIRE(h && sparse_metric_ok(metric) && metric != VB_IP, "bad sparse table / ordering metric");
    VB_REQUIRE(k > 0 && k <= 2048, "k must be in 1..2048");
    if (nq <= 0) return VB_OK;
    VB_REQUIRE(h->t.dim == q_dim, "different sparsevec dimensions %d and %d", h->t.dim, q_dim);
    VB_REQUIRE(q_off, "null query / output buffers");
    if (host) return check_csr("queries", h->t.dim, nq, q_off, q_idx, max_q);
    int64_t total = 0;
    VB_TRY(check_csr_dev("queries", h->t.dim, nq, q_off, q_idx, max_q, &total));
    VB_REQUIRE(total == 0 || q_val, "null query / output buffers");
    return VB_OK;
}

SparseCsr sparse_table_csr(const vb_sparse_table* h) { return SparseCsr{h->t.dim, h->t.n, h->t.row_off, h->t.idx, h->t.val}; }

uint64_t sparse_table_uid(const vb_sparse_table* h) { return h->uid; }

int sparse_queries_on_device(Scratch& sc, int dim, int q_dim, int64_t nq, const int64_t* q_off, const int32_t* q_idx, const float* q_val, bool host,
                             SparseCsr* out) {
    VB_REQUIRE(dim == q_dim, "different sparsevec dimensions %d and %d", dim, q_dim);
    VB_REQUIRE(q_off, "null query / output buffers");
    if (host) {
        VB_TRY(check_csr("queries", dim, nq, q_off, q_idx, nullptr));
        VB_REQUIRE(q_off[nq] == 0 || q_val, "null query / output buffers");
        SparseQueries Q;
        VB_TRY(upload_query_range(sc, 0, nq, q_off, q_idx, q_val, &Q));
        *out = SparseCsr{dim, nq, Q.off, Q.idx, Q.val};
        return VB_OK;
    }
    int64_t total = 0;
    VB_TRY(check_csr_dev("queries", dim, nq, q_off, q_idx, nullptr, &total));
    VB_REQUIRE(total == 0 || q_val, "null query / output buffers");
    *out = SparseCsr{dim, nq, q_off, q_idx, q_val};
    return VB_OK;
}

// Filtered top-k, one sub-batch after the other: filter_chunks_kernel lays out the chunks of each query's allowed rows
// (a filter's queries in one block), sparse_gather_kernel scores them (one launch per block that fills the grid, so the
// grid reads one filter's rows at a time), then the selection and the epilogue of vb_sparse_exact_topk.  host == false:
// queries and outputs on the device (out_f: floats), asynchronous after the query check.
static int sparse_topk_filtered(vb_sparse_table* h, int metric, int q_dim, int64_t nq, const int64_t* q_off, const int32_t* q_idx,
                                const float* q_val, int k, const vb_filter* const* filters, int nfilters, const int32_t* filter_of_query,
                                bool host, int64_t* out_ids, double* out_dist, float* out_f) {
    const char* fn = "vb_sparse_exact_topk_filtered";
    VB_TRY(require_init());
    int max_q = 0;
    VB_TRY(sparse_topk_args(h, metric, q_dim, 0, nullptr, nullptr, nullptr, k, host, nullptr));
    VB_REQUIRE(filters && nfilters >= 1, "%s: no row filter given", fn);
    VB_REQUIRE(filter_of_query || nfilters == 1, "%s: filter_of_query may only be NULL with one filter (got %d)", fn, nfilters);
    for (int i = 0; i < nfilters; ++i) {
        VB_REQUIRE(filters[i], "%s: filter %d is NULL", fn, i);
        const Filter& f = filters[i]->f;
        VB_REQUIRE(f.kind == FILTER_SPARSE && f.owner == h && f.owner_uid == h->uid, "%s: filter %d was made for another table or index", fn, i);
        VB_REQUIRE(f.n < (int64_t)INT32_MAX, "%s: filter %d allows %lld rows, at most %d", fn, i, (long long)f.n, INT32_MAX - 1);
    }
    if (nq <= 0) return VB_OK;
    VB_TRY(sparse_topk_args(h, metric, q_dim, nq, q_off, q_idx, q_val, k, host, &max_q));
    VB_REQUIRE(out_ids && (host ? out_dist != nullptr : out_f != nullptr), "null query / output buffers");
    for (int64_t q = 0; q < nq && filter_of_query; ++q)
        VB_REQUIRE(filter_of_query[q] >= 0 && filter_of_query[q] < nfilters, "%s: filter_of_query[%lld] = %d, not in 0..%d", fn, (long long)q,
                   filter_of_query[q], nfilters - 1);
    Context& c = ctx();
    const SparseTable& t = h->t;
    Scratch pos;
    std::vector<int64_t> fbase;
    const int64_t* rows;
    VB_TRY(filter_concat_positions(pos, filters, nfilters, &fbase, &rows));
    const int km = key_metric(metric);
    // host results are staged on the host so that a failing sub-batch leaves the caller's buffers untouched
    std::vector<int64_t> ids(host ? (size_t)(nq * k) : 0);
    std::vector<double> dist(host ? (size_t)(nq * k) : 0);
    FilterBatch b;
    for (int64_t q0 = 0; q0 < nq;) {
        Scratch sc;
        VB_TRY(filter_batch_plan(filters, nfilters, filter_of_query, fbase.data(), q0, nq, SP_MAX_BATCH, SP_CHUNK_ROWS, 8 * (int64_t)c.sm_count,
                                 &b));
        const int64_t m = (int64_t)b.qa.size();
        const size_t nl = b.launch_count.size();
        SparseQueries Q;
        VB_TRY(sub_batch_queries(sc, host, q0, m, q_off, q_idx, q_val, &Q));
        // per-query arguments | segments | chunks of each gather launch
        void *d_qa, *d_chunks, *d_keys;
        const size_t qa_bytes = (sizeof(FilterQuery) * (size_t)m + 255) & ~(size_t)255;
        VB_TRY(sc.take(qa_bytes + (sizeof(int64_t) + sizeof(int32_t)) * (size_t)m + sizeof(int32_t) * nl + 64, &d_qa));
        int64_t* seg_begin = (int64_t*)((uint8_t*)d_qa + qa_bytes);
        int32_t* seg_len = (int32_t*)(seg_begin + m);
        int32_t* d_count = seg_len + m;
        VB_CUDA(cudaMemcpyAsync(d_qa, b.qa.data(), sizeof(FilterQuery) * (size_t)m, cudaMemcpyHostToDevice, c.stream));
        if (nl) VB_CUDA(cudaMemcpyAsync(d_count, b.launch_count.data(), sizeof(int32_t) * nl, cudaMemcpyHostToDevice, c.stream));
        VB_TRY(sc.take(sizeof(Chunk) * (size_t)b.max_chunks + 64, &d_chunks));
        VB_TRY(launch_filter_chunks((const FilterQuery*)d_qa, m, SP_CHUNK_ROWS, seg_begin, seg_len, (Chunk*)d_chunks));
        VB_TRY(sc.take(sizeof(float) * (size_t)std::max<int64_t>(b.run, 1), &d_keys));
        for (size_t l = 0; l < nl; ++l)
            VB_TRY(launch_sparse_gather(km, t.dim, Q, max_q, t, rows, (const Chunk*)d_chunks + b.launch_begin[l], d_count + l, b.launch_count[l],
                                        (float*)d_keys));
        // entry p of query j's segment is rows[qa[j].base + p]
        static_assert(sizeof(FilterQuery) % sizeof(int64_t) == 0 && offsetof(FilterQuery, base) % sizeof(int64_t) == 0, "FilterQuery layout");
        VB_TRY(sparse_select_finish(metric, m, k, (const float*)d_keys, seg_begin, seg_len, rows,
                                    (const int64_t*)d_qa + offsetof(FilterQuery, base) / sizeof(int64_t),
                                    (int)(sizeof(FilterQuery) / sizeof(int64_t)), host ? ids.data() + q0 * k : out_ids + q0 * k,
                                    host ? dist.data() + q0 * k : nullptr, host ? nullptr : out_f + q0 * k));
        q0 += m;   // (qa is pageable: its copy has been staged by the time cudaMemcpyAsync returned, so it may be refilled)
    }
    if (host) {
        std::copy(ids.begin(), ids.end(), out_ids);
        std::copy(dist.begin(), dist.end(), out_dist);
    }
    return VB_OK;
}

// Re-rank, one sub-batch after the other: rerank_prepare_kernel compacts each query's candidates in candidate order and
// lays out their chunks, sparse_gather_kernel scores them, then the selection and the epilogue of vb_sparse_exact_topk.
// host == false: queries, candidates and outputs on the device (out_f: floats), candidates outside [0, n) absent,
// asynchronous after the query check.
static int sparse_rerank(vb_sparse_table* h, int metric, int q_dim, int64_t nq, const int64_t* q_off, const int32_t* q_idx,
                         const float* q_val, const int64_t* cand, int c, int k, bool host, int64_t* out_ids, double* out_dist, float* out_f) {
    const char* fn = "vb_sparse_table_rerank";
    VB_TRY(require_init());
    int max_q = 0;
    VB_TRY(sparse_topk_args(h, metric, q_dim, 0, nullptr, nullptr, nullptr, k, host, nullptr));
    VB_REQUIRE(c >= 0, "%s: negative candidate count %d", fn, c);
    if (nq <= 0) return VB_OK;
    VB_TRY(sparse_topk_args(h, metric, q_dim, nq, q_off, q_idx, q_val, k, host, &max_q));
    VB_REQUIRE((cand || c == 0) && out_ids && (host ? out_dist != nullptr : out_f != nullptr), "null query / output buffers");
    const SparseTable& t = h->t;
    const int64_t n = t.n;
    for (int64_t i = 0; host && i < nq * c; ++i) {
        const int64_t v = cand[i];
        VB_REQUIRE(v >= -1 && v < n, "%s: candidate %lld of query %lld is %lld, not a row of the table (-1 or 0..%lld)", fn,
                   (long long)(i % c), (long long)(i / c), (long long)v, (long long)n - 1);
    }
    Context& cx = ctx();
    const int km = key_metric(metric);
    std::vector<int64_t> ids(host ? (size_t)(nq * k) : 0);
    std::vector<double> dist(host ? (size_t)(nq * k) : 0);
    // sub-batches keep the keys under ~1 GiB
    const int64_t bq = std::max<int64_t>(1, std::min<int64_t>(std::min(nq, SP_MAX_BATCH), (int64_t)(1ull << 28) / std::max(c, 1)));
    for (int64_t q0 = 0; q0 < nq; q0 += bq) {
        Scratch sc;
        const int64_t m = std::min(bq, nq - q0);
        const size_t mc = (size_t)m * c;
        SparseQueries Q;
        VB_TRY(sub_batch_queries(sc, host, q0, m, q_off, q_idx, q_val, &Q));
        // candidates (host variant: their copy) | their compaction
        void *d_cand, *d_chunks, *d_seg, *d_keys;
        VB_TRY(sc.take(2 * sizeof(int64_t) * mc, &d_cand));
        int64_t* d_ids = (int64_t*)d_cand + mc;
        if (!host) d_cand = const_cast<int64_t*>(cand) + (size_t)q0 * c;
        else if (mc) VB_CUDA(cudaMemcpyAsync(d_cand, cand + (size_t)q0 * c, sizeof(int64_t) * mc, cudaMemcpyHostToDevice, cx.stream));
        const int64_t max_chunks = m * ((c + SP_CHUNK_ROWS - 1) / SP_CHUNK_ROWS);
        VB_TRY(sc.take(sizeof(Chunk) * (size_t)max_chunks + 64, &d_chunks));
        int* n_chunks = (int*)((Chunk*)d_chunks + max_chunks);
        VB_TRY(sc.take((sizeof(int64_t) + sizeof(int32_t)) * (size_t)m + 64, &d_seg));
        int64_t* seg_begin = (int64_t*)d_seg;
        int32_t* seg_len = (int32_t*)(seg_begin + m);
        VB_CUDA(cudaMemsetAsync(n_chunks, 0, sizeof(int), cx.stream));
        VB_TRY(launch_rerank_prepare((const int64_t*)d_cand, m, c, n, SP_CHUNK_ROWS, d_ids, seg_begin, seg_len, (Chunk*)d_chunks, n_chunks));
        VB_TRY(sc.take(sizeof(float) * mc, &d_keys));
        VB_TRY(launch_sparse_gather(km, t.dim, Q, max_q, t, d_ids, (const Chunk*)d_chunks, n_chunks, (int)max_chunks, (float*)d_keys));
        // entry p of query j's segment is d_ids[seg_begin[j] + p] (seg_begin[j] = j c)
        VB_TRY(sparse_select_finish(metric, m, k, (const float*)d_keys, seg_begin, seg_len, d_ids, seg_begin, 1,
                                    host ? ids.data() + q0 * k : out_ids + q0 * k, host ? dist.data() + q0 * k : nullptr,
                                    host ? nullptr : out_f + q0 * k));
    }
    if (host) {
        std::copy(ids.begin(), ids.end(), out_ids);
        std::copy(dist.begin(), dist.end(), out_dist);
    }
    return VB_OK;
}

// vb_sparse_exact_topk[_dev]: the scan of every row per sub-batch of queries, then the selection and the epilogue.
static int sparse_exact_topk(vb_sparse_table* h, int metric, int q_dim, int64_t nq, const int64_t* q_off, const int32_t* q_idx,
                             const float* q_val, int k, bool host, int64_t* out_ids, double* out_dist, float* out_f) {
    VB_TRY(require_init());
    VB_REQUIRE(h && sparse_metric_ok(metric) && metric != VB_IP, "bad sparse table / ordering metric");
    VB_REQUIRE(k > 0 && k <= 2048, "k must be in 1..2048");
    if (nq <= 0) return VB_OK;
    SparseTable& t = h->t;
    VB_REQUIRE(t.dim == q_dim, "different sparsevec dimensions %d and %d", t.dim, q_dim);
    VB_REQUIRE(q_off && out_ids && (host ? out_dist != nullptr : out_f != nullptr), "null query / output buffers");
    int max_q = 0;
    VB_TRY(sparse_topk_args(h, metric, q_dim, nq, q_off, q_idx, q_val, k, host, &max_q));
    Context& c = ctx();
    cudaStream_t s = c.stream;
    const int64_t n = t.n;
    if (n == 0) {
        if (!host) {
            sparse_pad_kernel<<<(unsigned)((nq * k + 255) / 256), 256, 0, s>>>(nq * k, out_ids, out_f);
            VB_CUDA(cudaGetLastError());
            count_launch();
            return VB_OK;
        }
        for (int64_t i = 0; i < nq * k; ++i) {
            out_ids[i] = -1;
            out_dist[i] = INFINITY;
        }
        return VB_OK;
    }
    // sub-batches keep the key matrix under ~1 GiB
    const int64_t bq = std::max<int64_t>(1, std::min<int64_t>(std::min<int64_t>(nq, 65535), (int64_t)(1ull << 30) / (4 * n)));
    for (int64_t q0 = 0; q0 < nq; q0 += bq) {
        Scratch sc;
        const int64_t m = std::min(bq, nq - q0);
        SparseQueries Q;
        VB_TRY(sub_batch_queries(sc, host, q0, m, q_off, q_idx, q_val, &Q));
        void *d_key, *d_seg;
        VB_TRY(sc.take(sizeof(float) * (size_t)m * (size_t)n, &d_key));
        VB_TRY(launch_sparse_scan(key_metric(metric), t.dim, Q, m, max_q, t.row_off, t.idx, t.val, n, nullptr, (float*)d_key));
        VB_TRY(sc.take((sizeof(int64_t) + sizeof(int32_t)) * (size_t)m + 64, &d_seg));
        int64_t* seg_begin = (int64_t*)d_seg;
        int32_t* seg_len = (int32_t*)(seg_begin + m);
        sparse_segments_kernel<<<(unsigned)((m + 255) / 256), 256, 0, s>>>(m, n, seg_begin, seg_len);
        VB_CUDA(cudaGetLastError());
        count_launch();
        VB_TRY(sparse_select_finish(metric, m, k, (const float*)d_key, seg_begin, seg_len, nullptr, nullptr, 0, out_ids + q0 * k,
                                    host ? out_dist + q0 * k : nullptr, host ? nullptr : out_f + q0 * k));
    }
    return VB_OK;
}

// vb_sparse_table_append[_dev]: rows validated first (nothing is appended on any error), then the table grows
// (sparse_reserve) and the new rows are copied behind the old ones, their offsets rebased by the table's nnz.
static int sparse_append(vb_sparse_table* h, int64_t n, const int64_t* row_off, const int32_t* idx, const float* val, bool host) {
    VB_TRY(require_init());
    VB_REQUIRE(h && n >= 0 && (n == 0 || row_off), "bad sparse table arguments");
    if (n == 0) return VB_OK;
    SparseTable& t = h->t;
    int64_t tot;
    if (host) {
        VB_TRY(check_csr("rows", t.dim, n, row_off, idx, nullptr));
        tot = row_off[n];
    } else {
        VB_TRY(check_csr_dev("rows", t.dim, n, row_off, idx, nullptr, &tot));
    }
    VB_REQUIRE(tot == 0 || val, "null sparsevec values");
    VB_TRY(sparse_reserve(t, t.n + n, t.nnz + tot));
    cudaStream_t s = ctx().stream;
    const cudaMemcpyKind kind = host ? cudaMemcpyHostToDevice : cudaMemcpyDeviceToDevice;
    // offsets of the new rows: row_off[1..n] + nnz so far
    VB_CUDA(cudaMemcpyAsync(t.row_off + t.n + 1, row_off + 1, sizeof(int64_t) * (size_t)n, kind, s));
    if (t.nnz > 0) {
        sparse_shift_offsets_kernel<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(t.row_off + t.n + 1, n, t.nnz);
        VB_CUDA(cudaGetLastError());
        count_launch();
    }
    if (tot > 0) {
        VB_CUDA(cudaMemcpyAsync(t.idx + t.nnz, idx, sizeof(int32_t) * (size_t)tot, kind, s));
        VB_CUDA(cudaMemcpyAsync(t.val + t.nnz, val, sizeof(float) * (size_t)tot, kind, s));
    }
    if (host) VB_CUDA(cudaStreamSynchronize(s));
    t.n += n;
    t.nnz += tot;
    return VB_OK;
}

// ----------------------------------------------------------------------------- casts between the dense types and sparsevec

// The element sources of the casts to sparsevec.  keep(i, &v): element i of the packed rows is kept, v its float value.
// nnz_key(r): the SparseCheck::bad key of CheckNnz's error in row r; elem_key(r, i, v): the key of CheckElement's error
// at kept element i (kCheck sources only).
//
// vector / halfvec rows (vector_to_sparsevec / halfvec_to_sparsevec): kept when x != 0 (halfvec: !HalfIsZero, so -0 is
// dropped in both), halfvec widened exactly; CheckNnz as check_csr reports it, (row << 8) | SPC_NNZ.
template <int ELEM>
struct DenseSource {
    const void* rows;
    static constexpr bool kCheck = false;
    __device__ __forceinline__ bool keep(size_t i, float* v) const {
        if (ELEM == VB_VECTOR) {
            *v = __ldg(reinterpret_cast<const float*>(rows) + i);
            return *v != 0.f;
        }
        const unsigned short b = __ldg(reinterpret_cast<const unsigned short*>(rows) + i);
        *v = __half2float(__ushort_as_half(b));
        return (b & 0x7FFFu) != 0;
    }
    __device__ __forceinline__ unsigned long long nnz_key(int64_t r) const { return ((unsigned long long)r << 8) | SPC_NNZ; }
    __device__ __forceinline__ unsigned long long elem_key(int64_t, int, float) const { return ~0ull; }
};

// array_to_sparsevec's first-offender key (src/sparsevec.c:694-821): (row, pass, element, kind) in 31 + 2 + 30 + 1 bits,
// so the lowest row wins, then the first pass its loops reach, then the element.  Pass 0 is numeric_float4's range
// error in the count loop (numeric[] only), pass 1 CheckNnz after it, pass 2 CheckElement over the kept values (kind 0:
// NaN, 1: infinite).  n < 2^31 rows and dim <= 10^9 < 2^30 fit.
enum { ASP_PASS_REAL = 0, ASP_PASS_NNZ = 1, ASP_PASS_ELEMENT = 2 };
__host__ __device__ __forceinline__ unsigned long long array_sparse_key(int64_t r, int pass, int64_t i, int kind) {
    return ((unsigned long long)r << 33) | ((unsigned long long)pass << 31) | ((unsigned long long)i << 1) | (unsigned)kind;
}

// numeric[] -> sparsevec, first step (numeric_cast_kernel's sink): numeric_float4 of every element into a float
// buffer that the count and write passes then read as real[]; float4in's range error lowers *first_bad
struct NumericFloatSink {
    float* out;
    int dim;
    unsigned long long* first_bad;
    __device__ __forceinline__ void put(int64_t e, float f, bool real_range) const {
        out[e] = real_range ? 0.f : f;
        if (real_range) atomicMin(first_bad, array_sparse_key(e / dim, ASP_PASS_REAL, e % dim, 0));
    }
};

__device__ __forceinline__ float array_float(int32_t x) { return __int2float_rn(x); }
__device__ __forceinline__ float array_float(float x) { return x; }
__device__ __forceinline__ float array_float(double x) { return __double2float_rn(x); }

// integer[] / real[] / double precision[] rows: (float) of the int32 or double (round to nearest even), real as is;
// kept when v != 0, so -0 and a double that rounds to 0 are dropped and NaN and the infinities are kept
template <typename S>
struct ArraySource {
    const S* rows;
    static constexpr bool kCheck = !std::is_same<S, int32_t>::value;   // an int32 is always finite
    __device__ __forceinline__ bool keep(size_t i, float* v) const {
        *v = array_float(__ldg(rows + i));
        return *v != 0.f;
    }
    __device__ __forceinline__ unsigned long long nnz_key(int64_t r) const { return array_sparse_key(r, ASP_PASS_NNZ, 0, 0); }
    __device__ __forceinline__ unsigned long long elem_key(int64_t r, int i, float v) const {
        return isnan(v) ? array_sparse_key(r, ASP_PASS_ELEMENT, i, 0) : isinf(v) ? array_sparse_key(r, ASP_PASS_ELEMENT, i, 1) : ~0ull;
    }
};

constexpr int SP_CAST_UNROLL = 4;   // elements per lane in flight: each lane loads 4 before the warp's ballots

// The work of the casts to sparsevec: one warp per segment of seg_len elements, nseg segments per row (row r's
// segment j is warp r * nseg + j), so a batch of a few long rows still fills the device.  With nseg == 1 a warp takes
// a whole row and the segment offsets are the row offsets.
struct SparseSegs {
    int nseg;
    int seg_len;   // a multiple of 32 * SP_CAST_UNROLL
};

// Count pass of the casts to sparsevec (vector_to_sparsevec / halfvec_to_sparsevec, src/sparsevec.c:606-689, and
// array_to_sparsevec, src/sparsevec.c:694-821): the kept elements of each segment ballot-counted into cnt[w].  With one
// segment per row a row above SP_MAX_NNZ is CheckNnz's error here (else segment_rows_kernel checks the row sums).  A
// kCheck source also lowers the key of each lane's first kept NaN or infinity.
template <typename Src>
__global__ void __launch_bounds__(256) dense_count_kernel(Src src, int dim, int64_t n, SparseSegs sg, int64_t* __restrict__ cnt,
                                                          SparseCheck* __restrict__ chk) {
    const int64_t w = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (w >= n * sg.nseg) return;   // whole warps
    const int64_t r = w / sg.nseg;
    const int lo = (int)(w - r * sg.nseg) * sg.seg_len;
    const int hi = min(dim, lo + sg.seg_len);
    const size_t base = (size_t)r * (size_t)dim;
    int64_t c = 0;
    unsigned long long key = ~0ull;
    for (int i0 = lo; i0 < hi; i0 += 32 * SP_CAST_UNROLL) {
        bool keep[SP_CAST_UNROLL];
#pragma unroll
        for (int u = 0; u < SP_CAST_UNROLL; ++u) {
            const int i = i0 + u * 32 + lane;
            float v;
            keep[u] = i < hi && src.keep(base + i, &v);
            if (Src::kCheck && keep[u] && key == ~0ull) key = src.elem_key(r, i, v);
        }
#pragma unroll
        for (int u = 0; u < SP_CAST_UNROLL; ++u) c += __popc(__ballot_sync(0xffffffffu, keep[u]));
    }
    if (Src::kCheck && key != ~0ull) atomicMin(&chk->bad, key);
    if (lane == 0) {
        cnt[w] = c;
        if (sg.nseg == 1 && c > SP_MAX_NNZ) atomicMin(&chk->bad, src.nnz_key(r));
    }
}

// Rows split into segments: row_off[r] = seg_off[r * nseg] for r in [0, n], and CheckNnz over each row's sum
template <typename Src>
__global__ void segment_rows_kernel(Src src, int64_t n, int nseg, const int64_t* __restrict__ seg_off, int64_t* __restrict__ row_off,
                                    SparseCheck* __restrict__ chk) {
    const int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (r > n) return;
    const int64_t b = seg_off[r * nseg];
    row_off[r] = b;
    if (r < n && seg_off[(r + 1) * nseg] - b > SP_MAX_NNZ) atomicMin(&chk->bad, src.nnz_key(r));
}

// Write pass: the kept elements of segment w at off[w] .. in ascending index order (ballot + the warp prefix of each
// step).  Entries at lim and above are not written: a buffer of lim entries is too small only for rows CheckNnz refuses.
template <typename Src>
__global__ void __launch_bounds__(256) dense_write_kernel(Src src, int dim, int64_t n, SparseSegs sg, const int64_t* __restrict__ off,
                                                          int64_t lim, int32_t* __restrict__ out_idx, float* __restrict__ out_val) {
    const int64_t ws = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (ws >= n * sg.nseg) return;   // whole warps
    const int64_t r = ws / sg.nseg;
    const int lo = (int)(ws - r * sg.nseg) * sg.seg_len;
    const int hi = min(dim, lo + sg.seg_len);
    const size_t base = (size_t)r * (size_t)dim;
    const unsigned below = (1u << lane) - 1u;
    int64_t w = off[ws];
    for (int i0 = lo; i0 < hi; i0 += 32 * SP_CAST_UNROLL) {
        bool keep[SP_CAST_UNROLL];
        float v[SP_CAST_UNROLL];
#pragma unroll
        for (int u = 0; u < SP_CAST_UNROLL; ++u) {
            const int i = i0 + u * 32 + lane;
            keep[u] = i < hi && src.keep(base + i, &v[u]);
        }
#pragma unroll
        for (int u = 0; u < SP_CAST_UNROLL; ++u) {
            const unsigned m = __ballot_sync(0xffffffffu, keep[u]);
            const int64_t at = w + __popc(m & below);
            if (keep[u] && at < lim) {
                out_idx[at] = i0 + u * 32 + lane;
                out_val[at] = v[u];
            }
            w += __popc(m);
        }
    }
}

// sparsevec_to_vector / sparsevec_to_halfvec (src/vector.c:1323-1349, src/halfvec.c:1199-1225): one warp per row, the
// row zero-filled, then its entries scattered (halfvec: Float4ToHalf, an overflow recorded as the first entry in
// chk->over).  Nothing is written when chk->bad records a CSR defect (the check ran before, on the same stream).
template <int ELEM>
__global__ void __launch_bounds__(256) sparse_to_dense_kernel(int64_t n, const int64_t* __restrict__ off, const int32_t* __restrict__ idx,
                                                              const float* __restrict__ val, int dim, void* __restrict__ out,
                                                              SparseCheck* __restrict__ chk) {
    const int64_t r = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (r >= n || chk->bad != ~0ull) return;   // whole warps
    const size_t base = (size_t)r * (size_t)dim;
    for (int i = lane; i < dim; i += 32) {
        if (ELEM == VB_VECTOR) reinterpret_cast<float*>(out)[base + i] = 0.f;
        else reinterpret_cast<__half*>(out)[base + i] = __ushort_as_half((unsigned short)0);
    }
    __syncwarp();
    const int64_t end = val ? off[r + 1] : off[r];   // null values: the call fails unless there are no entries
    for (int64_t p = off[r] + lane; p < end; p += 32) {
        const float x = val[p];
        if (ELEM == VB_VECTOR) {
            reinterpret_cast<float*>(out)[base + idx[p]] = x;
        } else {
            bool over;
            reinterpret_cast<__half*>(out)[base + idx[p]] = float_to_half_checked(x, &over);
            if (over) atomicMin(&chk->over, (long long)p);
        }
    }
}

static const char* dense_name(int elem) { return elem == VB_VECTOR ? "vector" : "halfvec"; }

// The segments of n rows of dim elements: one per row when the rows alone give every SM 64 warps or are short, else
// enough to do so, none shorter than 2048 elements
static SparseSegs sparse_segs(int dim, int64_t n) {
    const int64_t unit = 32 * SP_CAST_UNROLL, want = (int64_t)ctx().sm_count * 64;
    int64_t nseg = 1;
    if (n < want && dim > 2048) nseg = std::min<int64_t>((dim + 2047) / 2048, (want + n - 1) / n);
    const int64_t len = ((dim + nseg - 1) / nseg + unit - 1) / unit * unit;
    return SparseSegs{(int)((dim + len - 1) / len), (int)len};
}

// device buffers of a count pass over up to m segments
struct SparseCountBufs {
    int64_t* cnt;   // [m + 1]
    int64_t* seg;   // [m + 1], the segment offsets when a row has several
    void* scan;
    size_t scan_bytes;
};
static int sparse_count_bufs(Scratch& sc, int64_t m, SparseCountBufs* b) {
    void *c, *g;
    VB_TRY(sc.take(sizeof(int64_t) * (size_t)(m + 1), &c));
    VB_TRY(sc.take(sizeof(int64_t) * (size_t)(m + 1), &g));
    b->cnt = (int64_t*)c;
    b->seg = (int64_t*)g;
    b->scan_bytes = 0;
    VB_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, b->scan_bytes, b->cnt, b->seg, (int)(m + 1), ctx().stream));
    return sc.take(b->scan_bytes + 64, &b->scan);
}

// Enqueues the count pass of a cast to sparsevec over n >= 1 device rows: chk initialised, then lowered to the first
// error; row_off[0 .. n] (device) the row offsets and chk->total = row_off[n]; *seg_off the offsets the write pass
// takes (row_off itself when each row is one segment).  Reads nothing back.
template <typename Src>
static int sparse_cast_count(Src src, int dim, int64_t n, const SparseSegs& sg, const SparseCountBufs& b, int64_t* row_off,
                             SparseCheck* chk, const int64_t** seg_off) {
    cudaStream_t s = ctx().stream;
    const int64_t m = n * sg.nseg;
    int64_t* so = sg.nseg == 1 ? row_off : b.seg;
    sparse_check_init_kernel<<<1, 1, 0, s>>>(chk);
    dense_count_kernel<Src><<<(unsigned)((m * 32 + 255) / 256), 256, 0, s>>>(src, dim, n, sg, b.cnt, chk);
    VB_CUDA(cudaGetLastError());
    VB_CUDA(cudaMemsetAsync(b.cnt + m, 0, sizeof(int64_t), s));
    size_t scan_bytes = b.scan_bytes;
    VB_CUDA(cub::DeviceScan::ExclusiveSum(b.scan, scan_bytes, b.cnt, so, (int)(m + 1), s));
    count_launch(3);
    if (sg.nseg > 1) {
        segment_rows_kernel<Src><<<(unsigned)((n + 1 + 255) / 256), 256, 0, s>>>(src, n, sg.nseg, so, row_off, chk);
        VB_CUDA(cudaGetLastError());
        count_launch();
    }
    VB_CUDA(cudaMemcpyAsync(&chk->total, row_off + n, sizeof(int64_t), cudaMemcpyDeviceToDevice, s));
    *seg_off = so;
    return VB_OK;
}

// Enqueues the write pass after sparse_cast_count: at most lim entries into idx / val (device)
template <typename Src>
static int sparse_cast_write(Src src, int dim, int64_t n, const SparseSegs& sg, const int64_t* seg_off, int64_t lim, int32_t* idx,
                             float* val) {
    const int64_t m = n * sg.nseg;
    dense_write_kernel<Src><<<(unsigned)((m * 32 + 255) / 256), 256, 0, ctx().stream>>>(src, dim, n, sg, seg_off, lim, idx, val);
    VB_CUDA(cudaGetLastError());
    count_launch();
    return VB_OK;
}

// vb_dense_to_sparsevec_batch[_dev]
static int dense_to_sparse(int elem, int dim, const void* rows, int64_t n, int64_t cap, bool host, int64_t* out_row_off, int32_t* out_idx,
                           float* out_val) {
    Scratch sc;
    const char* fn = host ? "vb_dense_to_sparsevec_batch" : "vb_dense_to_sparsevec_batch_dev";
    VB_TRY(require_init());
    VB_REQUIRE(elem == VB_VECTOR || elem == VB_HALFVEC, "%s: elem must be VB_VECTOR or VB_HALFVEC, got %d", fn, elem);
    // CheckDim (src/sparsevec.c:68-80)
    VB_REQUIRE(dim >= 1, "sparsevec must have at least 1 dimension");
    VB_REQUIRE(dim <= SP_MAX_DIM, "sparsevec cannot have more than %d dimensions", SP_MAX_DIM);
    VB_REQUIRE(n >= 0 && n < (int64_t)INT32_MAX && cap >= 0, "%s: bad row count %lld or cap %lld", fn, (long long)n, (long long)cap);
    VB_REQUIRE(out_row_off && (rows || n == 0), "%s: null rows or offsets", fn);
    Context& cx = ctx();
    cudaStream_t s = cx.stream;
    if (n == 0) {
        if (host) out_row_off[0] = 0;
        else VB_CUDA(cudaMemsetAsync(out_row_off, 0, sizeof(int64_t), s));
        return VB_OK;
    }
    const size_t raw = raw_row_bytes(elem, dim);
    const size_t b_off = sizeof(int64_t) * (size_t)(n + 1);
    void *d_in = const_cast<void*>(rows), *d_off = out_row_off, *d_chk;
    if (host) {
        VB_TRY(sc.take(raw * (size_t)n, &d_in));
        VB_CUDA(cudaMemcpyAsync(d_in, rows, raw * (size_t)n, cudaMemcpyHostToDevice, s));
        VB_TRY(sc.take(b_off, &d_off));
    }
    VB_TRY(sc.take(sizeof(SparseCheck), &d_chk));
    SparseCheck* chk = (SparseCheck*)d_chk;
    int64_t* off = (int64_t*)d_off;
    const SparseSegs sg = sparse_segs(dim, n);
    SparseCountBufs cb;
    VB_TRY(sparse_count_bufs(sc, n * sg.nseg, &cb));
    const int64_t* seg_off;
    if (elem == VB_VECTOR) VB_TRY(sparse_cast_count(DenseSource<VB_VECTOR>{d_in}, dim, n, sg, cb, off, chk, &seg_off));
    else VB_TRY(sparse_cast_count(DenseSource<VB_HALFVEC>{d_in}, dim, n, sg, cb, off, chk, &seg_off));
    SparseCheck hc;
    if (host) VB_CUDA(cudaMemcpyAsync(out_row_off, off, b_off, cudaMemcpyDeviceToHost, s));
    VB_CUDA(cudaMemcpyAsync(&hc, chk, SPC_READ, cudaMemcpyDeviceToHost, s));
    VB_CUDA(cudaStreamSynchronize(s));
    if (hc.bad != ~0ull) return sparse_check_error(fn, hc.bad);
    const int64_t total = hc.total;
    VB_REQUIRE(total <= cap, "%s: the rows have %lld non-zero elements, more than cap = %lld", fn, (long long)total, (long long)cap);
    if (total == 0) return VB_OK;
    VB_REQUIRE(out_idx && out_val, "%s: null output indices or values", fn);
    int32_t* o_idx = out_idx;
    float* o_val = out_val;
    const size_t b_idx = (sizeof(int32_t) * (size_t)total + 15) & ~(size_t)15;
    if (host) {
        void* d_out;
        VB_TRY(sc.take(b_idx + sizeof(float) * (size_t)total, &d_out));
        o_idx = (int32_t*)d_out;
        o_val = (float*)((uint8_t*)d_out + b_idx);
    }
    if (elem == VB_VECTOR) VB_TRY(sparse_cast_write(DenseSource<VB_VECTOR>{d_in}, dim, n, sg, seg_off, total, o_idx, o_val));
    else VB_TRY(sparse_cast_write(DenseSource<VB_HALFVEC>{d_in}, dim, n, sg, seg_off, total, o_idx, o_val));
    if (host) {
        VB_CUDA(cudaMemcpyAsync(out_idx, o_idx, sizeof(int32_t) * (size_t)total, cudaMemcpyDeviceToHost, s));
        VB_CUDA(cudaMemcpyAsync(out_val, o_val, sizeof(float) * (size_t)total, cudaMemcpyDeviceToHost, s));
        VB_CUDA(cudaStreamSynchronize(s));
    }
    return VB_OK;
}

// array_to_sparsevec's error from a first-offender key; *out_bad = the failing row (plus first_row).  field(e) gives a
// host copy of numeric field e of the rows the key counts in, for float4in's range error.
template <typename Field>
static int array_sparse_error(unsigned long long key, int dim, int64_t first_row, int64_t* out_bad, Field field) {
    const int64_t row = (int64_t)(key >> 33);
    if (out_bad) *out_bad = first_row + row;
    const int pass = (int)((key >> 31) & 3);
    if (pass == ASP_PASS_REAL) {
        std::vector<uint8_t> f;
        VB_TRY(field(row * dim + (int64_t)((key >> 1) & 0x3FFFFFFF), f));
        return numeric_range_error(f.data());
    }
    if (pass == ASP_PASS_NNZ) set_error("sparsevec cannot have more than %d non-zero elements", SP_MAX_NNZ);
    else set_error((key & 1) ? "infinite value not allowed in sparsevec" : "NaN not allowed in sparsevec");
    return VB_EINVAL;
}

constexpr size_t ASP_CHUNK_BYTES = (size_t)32 << 20;   // source bytes (numeric: fields and offsets) per host chunk

// numeric_float4 of fields [0, total) into vals (device); status[0] / [1]: float4in's first range error (key) and the
// first malformed field, both set to ~0 here
static int numeric_to_floats(const uint8_t* bytes, const int64_t* off, int64_t base, int64_t total, int dim, float* vals,
                             unsigned long long* status) {
    cudaStream_t s = ctx().stream;
    VB_CUDA(cudaMemsetAsync(status, 0xFF, 2 * sizeof(unsigned long long), s));
    numeric_cast_kernel<<<(unsigned)((total + 255) / 256), 256, 0, s>>>(bytes, off, base, total, NumericFloatSink{vals, dim, status},
                                                                        status + 1);
    VB_CUDA(cudaGetLastError());
    count_launch();
    return VB_OK;
}

// vb_array_to_sparsevec_batch_dev (the arguments checked); NUM: numeric[] fields in[off[e] .. off[e + 1]), S = float
template <typename S, bool NUM>
static int array_to_sparse_dev(int dim, const void* in, const int64_t* in_off, int64_t n, int64_t cap, int64_t* out_row_off, int32_t* out_idx,
                               float* out_val, int64_t* out_bad) {
    Scratch sc;
    const char* fn = "vb_array_to_sparsevec_batch_dev";
    cudaStream_t s = ctx().stream;
    void *d_chk, *d_status = nullptr, *d_vals = nullptr;
    VB_TRY(sc.take(sizeof(SparseCheck), &d_chk));
    SparseCheck* chk = (SparseCheck*)d_chk;
    const S* rows = (const S*)in;
    unsigned long long status[2] = {~0ull, ~0ull};
    if (NUM) {
        VB_TRY(sc.take(16, &d_status));
        VB_TRY(sc.take(sizeof(float) * (size_t)(n * dim), &d_vals));
        VB_TRY(numeric_to_floats((const uint8_t*)in, in_off, 0, n * dim, dim, (float*)d_vals, (unsigned long long*)d_status));
        rows = (const S*)d_vals;
    }
    const SparseSegs sg = sparse_segs(dim, n);
    SparseCountBufs cb;
    VB_TRY(sparse_count_bufs(sc, n * sg.nseg, &cb));
    const int64_t* seg_off;
    VB_TRY(sparse_cast_count(ArraySource<S>{rows}, dim, n, sg, cb, out_row_off, chk, &seg_off));
    SparseCheck hc;
    VB_CUDA(cudaMemcpyAsync(&hc, chk, SPC_READ, cudaMemcpyDeviceToHost, s));
    if (NUM) VB_CUDA(cudaMemcpyAsync(status, d_status, 16, cudaMemcpyDeviceToHost, s));
    VB_CUDA(cudaStreamSynchronize(s));
    // only an error reads a field back, for its text
    auto field = [&](int64_t e, std::vector<uint8_t>& f) {
        int64_t o[2];
        VB_CUDA(cudaMemcpy(o, in_off + e, sizeof(o), cudaMemcpyDeviceToHost));
        const int64_t len = std::max<int64_t>(0, std::min<int64_t>(o[1] - o[0], 8 + 2 * 65535 + 1));
        f.resize((size_t)len + 8);
        if (len > 0) VB_CUDA(cudaMemcpy(f.data(), (const uint8_t*)in + o[0], (size_t)len, cudaMemcpyDeviceToHost));
        f.resize((size_t)len);   // past the longest valid field only the count of bytes left over matters
        return o[1] < o[0] ? VB_EINVAL : VB_OK;
    };
    if (status[1] != ~0ull) {
        const int64_t e = (int64_t)status[1];
        if (out_bad) *out_bad = e / dim;
        std::vector<uint8_t> f;
        if (field(e, f) != VB_OK) return numeric_field_error(fn, e, f.data(), -1);
        return numeric_field_error(fn, e, f.data(), (int64_t)f.size());
    }
    const unsigned long long key = std::min(hc.bad, status[0]);
    if (key != ~0ull) return array_sparse_error(key, dim, 0, out_bad, field);
    const int64_t total = hc.total;
    VB_REQUIRE(total <= cap, "%s: the rows have %lld non-zero elements, more than cap = %lld", fn, (long long)total, (long long)cap);
    if (total == 0) return VB_OK;
    VB_REQUIRE(out_idx && out_val, "%s: null output indices or values", fn);
    return sparse_cast_write(ArraySource<S>{rows}, dim, n, sg, seg_off, total, out_idx, out_val);
}

// vb_array_to_sparsevec_batch (the arguments checked): chunks of whole rows through the two staging slots.  Each slot
// has its device input (numeric: offsets, fields and their floats), offsets, entries (at most min(dim, SP_MAX_NNZ) per
// row: more is CheckNnz's error) and check.  A chunk's entries are copied out once its check is read, while the next
// chunk is on the device.  The chunks run in row order, so the first failing chunk has the lowest failing row; past cap
// the chunks are still counted and checked, so a data error still wins over the cap error.  numeric[]: every chunk is
// converted and checked, so a malformed field anywhere wins over a data error.
template <typename S, bool NUM>
static int array_to_sparse_host(int dim, const void* in, const int64_t* in_off, int64_t n, int64_t cap, int64_t* out_row_off,
                                int32_t* out_idx, float* out_val, int64_t* out_bad) {
    Scratch sc;
    const char* fn = "vb_array_to_sparsevec_batch";
    cudaStream_t s = ctx().stream;
    const uint8_t* src = (const uint8_t*)in;
    std::vector<int64_t> starts;
    if (NUM) {
        VB_TRY(numeric_offsets_check(fn, in_off, n * dim, out_bad, dim));
        numeric_chunks(in_off, n, dim, ASP_CHUNK_BYTES, starts);
    } else {
        const int64_t rc = std::min<int64_t>(n, std::max<int64_t>(1, (int64_t)(ASP_CHUNK_BYTES / (sizeof(S) * (size_t)dim))));
        for (int64_t r = 0; r < n; r += rc) starts.push_back(r);
        starts.push_back(n);
    }
    const int64_t nch = (int64_t)starts.size() - 1;
    // chunk c: rows [starts[c], starts[c + 1]), its source bytes at src_at(c) .. + src_bytes(c)
    auto src_at = [&](int64_t c) { return NUM ? in_off[starts[c] * dim] : (int64_t)sizeof(S) * starts[c] * dim; };
    auto src_bytes = [&](int64_t c) { return NUM ? in_off[starts[c + 1] * dim] - src_at(c) : (int64_t)sizeof(S) * (starts[c + 1] - starts[c]) * dim; };
    int64_t rc = 0, segs = 0, max_src = 0;
    for (int64_t c = 0; c < nch; ++c) {
        const int64_t m = starts[c + 1] - starts[c];
        rc = std::max(rc, m);
        segs = std::max(segs, m * sparse_segs(dim, m).nseg);
        max_src = std::max(max_src, src_bytes(c));
    }
    const int64_t ent = rc * std::min(dim, SP_MAX_NNZ);
    const size_t b_off = sizeof(int64_t) * (size_t)(rc + 1), b_in_off = NUM ? sizeof(int64_t) * (size_t)(rc * dim + 1) : 0;
    Staging& st = staging();
    struct Slot {
        uint8_t* in;
        int64_t* in_off;
        float* vals;
        unsigned long long* status;
        int64_t* off;
        int32_t* idx;
        float* val;
        SparseCheck* chk;
        SparseCountBufs cb;
        const int64_t* seg_off;
    } slot[2];
    for (int k = 0; k < 2 && k < nch; ++k) {
        void *a, *b = nullptr, *v = nullptr, *w = nullptr, *c, *d, *e, *f;
        VB_TRY(sc.take((size_t)max_src + 16, &a));
        if (NUM) {
            VB_TRY(sc.take(b_in_off, &b));
            VB_TRY(sc.take(sizeof(float) * (size_t)(rc * dim), &v));
            VB_TRY(sc.take(16, &w));
        }
        VB_TRY(sc.take(b_off, &c));
        VB_TRY(sc.take(sizeof(int32_t) * (size_t)ent, &d));
        VB_TRY(sc.take(sizeof(float) * (size_t)ent, &e));
        VB_TRY(sc.take(sizeof(SparseCheck), &f));
        slot[k] = Slot{(uint8_t*)a, (int64_t*)b, (float*)v, (unsigned long long*)w, (int64_t*)c, (int32_t*)d, (float*)e, (SparseCheck*)f, {}, nullptr};
        VB_TRY(sparse_count_bufs(sc, segs, &slot[k].cb));
        VB_TRY(pinned_grow(&st.in[k], &st.in_bytes[k], b_in_off + (size_t)max_src));
        VB_TRY(pinned_grow(&st.out[k], &st.out_bytes[k], b_off + sizeof(SparseCheck) + 16));
    }
    int64_t base = 0;   // entries of the rows finished so far
    int64_t malformed = -1, bad_chunk = -1;
    unsigned long long bad_key = ~0ull;
    out_row_off[0] = 0;
    auto enqueue = [&](int64_t c, int k) -> int {
        const int64_t r0 = starts[c], m = starts[c + 1] - r0, nb = src_bytes(c);
        Slot& sl = slot[k];
        uint8_t* pin = (uint8_t*)st.in[k];
        const S* rows = (const S*)sl.in;
        if (NUM) {
            memcpy(pin, in_off + r0 * dim, sizeof(int64_t) * (size_t)(m * dim + 1));
            VB_CUDA(cudaMemcpyAsync(sl.in_off, pin, sizeof(int64_t) * (size_t)(m * dim + 1), cudaMemcpyHostToDevice, s));
        }
        memcpy(pin + b_in_off, src + src_at(c), (size_t)nb);
        VB_CUDA(cudaMemcpyAsync(sl.in, pin + b_in_off, (size_t)nb, cudaMemcpyHostToDevice, s));
        if (NUM) {
            VB_TRY(numeric_to_floats(sl.in, sl.in_off, src_at(c), m * dim, dim, sl.vals, sl.status));
            rows = (const S*)sl.vals;
        }
        const SparseSegs sg = sparse_segs(dim, m);
        VB_TRY(sparse_cast_count(ArraySource<S>{rows}, dim, m, sg, sl.cb, sl.off, sl.chk, &sl.seg_off));
        VB_TRY(sparse_cast_write(ArraySource<S>{rows}, dim, m, sg, sl.seg_off, ent, sl.idx, sl.val));
        uint8_t* o = (uint8_t*)st.out[k];
        VB_CUDA(cudaMemcpyAsync(o, sl.off, sizeof(int64_t) * (size_t)(m + 1), cudaMemcpyDeviceToHost, s));
        VB_CUDA(cudaMemcpyAsync(o + b_off, sl.chk, SPC_READ, cudaMemcpyDeviceToHost, s));
        if (NUM) VB_CUDA(cudaMemcpyAsync(o + b_off + sizeof(SparseCheck), sl.status, 16, cudaMemcpyDeviceToHost, s));
        return VB_OK;
    };
    auto finish = [&](int64_t c, int k) -> int {
        const int64_t r0 = starts[c], m = starts[c + 1] - r0;
        const uint8_t* o = (const uint8_t*)st.out[k];
        SparseCheck hc;
        memcpy(&hc, o + b_off, SPC_READ);
        unsigned long long status[2] = {~0ull, ~0ull};
        if (NUM) memcpy(status, o + b_off + sizeof(SparseCheck), 16);
        if (malformed < 0 && status[1] != ~0ull) malformed = r0 * dim + (int64_t)status[1];
        const unsigned long long key = std::min(hc.bad, status[0]);
        if (bad_chunk < 0 && key != ~0ull) {
            bad_chunk = c, bad_key = key;
            if (!NUM) return VB_EINVAL;   // reported below
        }
        if (bad_chunk >= 0 || malformed >= 0) return VB_OK;   // numeric[]: the later chunks are only checked
        const int64_t* off = (const int64_t*)o;
        for (int64_t j = 1; j <= m; ++j) out_row_off[r0 + j] = base + off[j];
        const int64_t t = off[m];
        if (t > 0 && base + t <= cap) {
            VB_CUDA(cudaMemcpyAsync(out_idx + base, slot[k].idx, sizeof(int32_t) * (size_t)t, cudaMemcpyDeviceToHost, s));
            VB_CUDA(cudaMemcpyAsync(out_val + base, slot[k].val, sizeof(float) * (size_t)t, cudaMemcpyDeviceToHost, s));
            VB_CUDA(cudaStreamSynchronize(s));
        }
        base += t;
        return VB_OK;
    };
    const int rc_pipe = pipeline_chunks(nch, enqueue, finish);
    if (rc_pipe != VB_OK && bad_chunk < 0) return rc_pipe;
    if (malformed >= 0) {
        if (out_bad) *out_bad = malformed / dim;
        return numeric_field_error(fn, malformed, src + in_off[malformed], in_off[malformed + 1] - in_off[malformed]);
    }
    if (bad_chunk >= 0) {
        const int64_t r0 = starts[bad_chunk];
        return array_sparse_error(bad_key, dim, r0, out_bad, [&](int64_t e, std::vector<uint8_t>& f) {
            const int64_t g = r0 * dim + e;
            f.assign(src + in_off[g], src + in_off[g + 1]);
            return VB_OK;
        });
    }
    VB_REQUIRE(base <= cap, "%s: the rows have %lld non-zero elements, more than cap = %lld", fn, (long long)base, (long long)cap);
    return VB_OK;
}

// vb_array_to_sparsevec_batch[_dev]
static int array_to_sparse(int src, int dim, int32_t typmod, const void* in, const int64_t* in_off, int64_t n, int64_t cap, bool host,
                           int64_t* out_row_off, int32_t* out_idx, float* out_val, int64_t* out_bad) {
    const char* fn = host ? "vb_array_to_sparsevec_batch" : "vb_array_to_sparsevec_batch_dev";
    if (out_bad) *out_bad = -1;
    VB_TRY(require_init());
    VB_REQUIRE(src == VB_ARRAY_INT4 || src == VB_ARRAY_FLOAT4 || src == VB_ARRAY_FLOAT8 || src == VB_ARRAY_NUMERIC,
               "%s: bad source type %d", fn, src);
    VB_REQUIRE(n >= 0 && n < (int64_t)INT32_MAX && cap >= 0, "%s: bad row count %lld or cap %lld", fn, (long long)n, (long long)cap);
    // CheckDim, then CheckExpectedDim (src/sparsevec.c:68-94)
    VB_REQUIRE(dim >= 1, "sparsevec must have at least 1 dimension");
    VB_REQUIRE(dim <= SP_MAX_DIM, "sparsevec cannot have more than %d dimensions", SP_MAX_DIM);
    VB_REQUIRE(typmod == -1 || typmod == dim, "expected %d dimensions, not %d", typmod, dim);
    VB_REQUIRE(out_row_off && (in || n == 0), "%s: null rows or offsets", fn);
    const bool num = src == VB_ARRAY_NUMERIC;
    VB_REQUIRE(num == (in_off != nullptr || (num && n == 0)), "%s: in_off is required for numeric[] and only there", fn);
    const size_t es = src == VB_ARRAY_FLOAT8 ? 8 : num ? 1 : 4;
    VB_REQUIRE((uintptr_t)in % es == 0 && (uintptr_t)in_off % 8 == 0, "%s: rows must be aligned to their elements", fn);
    if (host) VB_REQUIRE(cap == 0 || (out_idx && out_val), "%s: null output indices or values", fn);
    if (n == 0) {
        if (host) out_row_off[0] = 0;
        else VB_CUDA(cudaMemsetAsync(out_row_off, 0, sizeof(int64_t), ctx().stream));
        return VB_OK;
    }
#define VB_ASP_CASE(SRC, S, NUM)                                                                                        \
    if (src == SRC)                                                                                                     \
        return host ? array_to_sparse_host<S, NUM>(dim, in, in_off, n, cap, out_row_off, out_idx, out_val, out_bad) \
                    : array_to_sparse_dev<S, NUM>(dim, in, in_off, n, cap, out_row_off, out_idx, out_val, out_bad);
    VB_ASP_CASE(VB_ARRAY_INT4, int32_t, false)
    VB_ASP_CASE(VB_ARRAY_FLOAT4, float, false)
    VB_ASP_CASE(VB_ARRAY_FLOAT8, double, false)
    VB_ASP_CASE(VB_ARRAY_NUMERIC, float, true)
#undef VB_ASP_CASE
    return VB_EINVAL;
}

// vb_sparsevec_to_dense_batch[_dev]
static int sparse_to_dense(int elem, int dim, int64_t n, const int64_t* row_off, const int32_t* idx, const float* val, void* out, bool host) {
    Scratch sc;
    const char* fn = host ? "vb_sparsevec_to_dense_batch" : "vb_sparsevec_to_dense_batch_dev";
    VB_TRY(require_init());
    VB_REQUIRE(elem == VB_VECTOR || elem == VB_HALFVEC, "%s: elem must be VB_VECTOR or VB_HALFVEC, got %d", fn, elem);
    // CheckDim of the target type (src/vector.c, src/halfvec.c: VECTOR_MAX_DIM = HALFVEC_MAX_DIM = 16000)
    VB_REQUIRE(dim >= 1, "%s must have at least 1 dimension", dense_name(elem));
    VB_REQUIRE(dim <= 16000, "%s cannot have more than %d dimensions", dense_name(elem), 16000);
    VB_REQUIRE(n >= 0 && (n == 0 || (row_off && out)), "%s: null rows or output", fn);
    if (n == 0) return VB_OK;
    Context& cx = ctx();
    cudaStream_t s = cx.stream;
    const int64_t* d_off = row_off;
    const int32_t* d_idx = idx;
    const float* d_val = val;
    int64_t total = 0;
    if (host) {
        VB_TRY(check_csr("rows", dim, n, row_off, idx, nullptr));
        total = row_off[n];
        VB_REQUIRE(total == 0 || val, "null sparsevec values");
        const size_t b_off = sizeof(int64_t) * (size_t)(n + 1);
        const size_t b_idx = (sizeof(int32_t) * (size_t)total + 15) & ~(size_t)15;
        void* d_rows;
        VB_TRY(sc.take(b_off + b_idx + sizeof(float) * (size_t)total + 64, &d_rows));
        uint8_t* p = (uint8_t*)d_rows;
        VB_CUDA(cudaMemcpyAsync(p, row_off, b_off, cudaMemcpyHostToDevice, s));
        if (total > 0) {
            VB_CUDA(cudaMemcpyAsync(p + b_off, idx, sizeof(int32_t) * (size_t)total, cudaMemcpyHostToDevice, s));
            VB_CUDA(cudaMemcpyAsync(p + b_off + b_idx, val, sizeof(float) * (size_t)total, cudaMemcpyHostToDevice, s));
        }
        d_off = (const int64_t*)p;
        d_idx = (const int32_t*)(p + b_off);
        d_val = (const float*)(p + b_off + b_idx);
    }
    const size_t out_bytes = (elem == VB_VECTOR ? sizeof(float) : sizeof(__half)) * (size_t)n * (size_t)dim;
    void* d_out = out;
    if (host) VB_TRY(sc.take(out_bytes, &d_out));
    SparseCheck* chk;
    if (host) {   // validated above: only the overflow word is needed
        void* d;
        VB_TRY(sc.take(sizeof(SparseCheck), &d));
        chk = (SparseCheck*)d;
        sparse_check_init_kernel<<<1, 1, 0, s>>>(chk);
        count_launch();
    } else {
        VB_TRY(launch_sparse_check(sc, dim, n, d_off, d_idx, &chk));
    }
    const unsigned grid = (unsigned)((n * 32 + 255) / 256);
    if (elem == VB_VECTOR) sparse_to_dense_kernel<VB_VECTOR><<<grid, 256, 0, s>>>(n, d_off, d_idx, d_val, dim, d_out, chk);
    else sparse_to_dense_kernel<VB_HALFVEC><<<grid, 256, 0, s>>>(n, d_off, d_idx, d_val, dim, d_out, chk);
    VB_CUDA(cudaGetLastError());
    count_launch();
    SparseCheck hc;
    VB_CUDA(cudaMemcpyAsync(&hc, chk, sizeof(SparseCheck), cudaMemcpyDeviceToHost, s));
    VB_CUDA(cudaStreamSynchronize(s));
    if (hc.bad != ~0ull) return sparse_check_error("rows", hc.bad);
    if (!host) VB_REQUIRE(hc.total == 0 || val, "null sparsevec values");
    if (hc.over != INT64_MAX) {
        float v;
        if (host) {
            v = val[hc.over];
        } else {   // the error path reads the offending value too
            VB_CUDA(cudaMemcpyAsync(&v, val + hc.over, sizeof(float), cudaMemcpyDeviceToHost, s));
            VB_CUDA(cudaStreamSynchronize(s));
        }
        return half_range_error(v);
    }
    if (host) {
        VB_CUDA(cudaMemcpyAsync(out, d_out, out_bytes, cudaMemcpyDeviceToHost, s));
        VB_CUDA(cudaStreamSynchronize(s));
    }
    return VB_OK;
}

}  // namespace vb

extern "C" {

int vb_sparsevec_distance_batch(int metric, int dim, int q_dim, int32_t q_nnz, const int32_t* q_idx, const float* q_val, int64_t n,
                                const int64_t* row_off, const int32_t* idx, const float* val, double* out) {
    Scratch sc;
    VB_TRY(require_init());
    VB_REQUIRE(sparse_metric_ok(metric), "metric %d is not defined for sparsevec", metric);
    VB_REQUIRE(n >= 0 && (n == 0 || (row_off && out)), "bad sparsevec batch arguments");
    if (n == 0) return VB_OK;
    if (q_nnz < 0) {   // NULL query: ZeroDistance (src/hnswutils.c:555-556)
        for (int64_t i = 0; i < n; ++i) out[i] = 0.0;
        return VB_OK;
    }
    // CheckDims (src/sparsevec.c:44-51)
    VB_REQUIRE(dim == q_dim, "different sparsevec dimensions %d and %d", dim, q_dim);
    VB_TRY(check_csr("rows", dim, n, row_off, idx, nullptr));
    const int64_t qoff[2] = {0, q_nnz};
    int max_q = 0;
    VB_TRY(check_csr("query", dim, 1, qoff, q_idx, &max_q));
    Context& c = ctx();
    SparseQueries Q;
    VB_TRY(upload_sparse_queries(sc, 1, qoff, q_idx, q_val, &Q));
    const int64_t tot = row_off[n];
    const size_t b_off = sizeof(int64_t) * (size_t)(n + 1);
    const size_t b_idx = (sizeof(int32_t) * (size_t)tot + 15) & ~(size_t)15;
    void *d_rows, *d_out;
    VB_TRY(sc.take(b_off + b_idx + sizeof(float) * (size_t)tot + 64, &d_rows));
    VB_TRY(sc.take(sizeof(double) * (size_t)n, &d_out));
    uint8_t* p = (uint8_t*)d_rows;
    VB_CUDA(cudaMemcpyAsync(p, row_off, b_off, cudaMemcpyHostToDevice, c.stream));
    if (tot > 0) {
        VB_CUDA(cudaMemcpyAsync(p + b_off, idx, sizeof(int32_t) * (size_t)tot, cudaMemcpyHostToDevice, c.stream));
        VB_CUDA(cudaMemcpyAsync(p + b_off + b_idx, val, sizeof(float) * (size_t)tot, cudaMemcpyHostToDevice, c.stream));
    }
    VB_TRY(launch_sparse_scan(metric, dim, Q, 1, max_q, (const int64_t*)p, (const int32_t*)(p + b_off), (const float*)(p + b_off + b_idx), n,
                              (double*)d_out, nullptr));
    VB_CUDA(cudaMemcpyAsync(out, d_out, sizeof(double) * (size_t)n, cudaMemcpyDeviceToHost, c.stream));
    VB_CUDA(cudaStreamSynchronize(c.stream));
    return VB_OK;
}

int vb_sparsevec_norm_batch(int64_t n, const int64_t* row_off, const float* val, double* out) {
    Scratch sc;
    VB_TRY(require_init());
    VB_REQUIRE(n >= 0 && (n == 0 || (row_off && out && row_off[0] == 0)), "bad sparsevec norm arguments");
    if (n == 0) return VB_OK;
    for (int64_t r = 0; r < n; ++r) VB_REQUIRE(row_off[r + 1] >= row_off[r], "offsets must not decrease (row %lld)", (long long)r);
    Context& c = ctx();
    const int64_t tot = row_off[n];
    const size_t b_off = sizeof(int64_t) * (size_t)(n + 1);
    void *d_rows, *d_out;
    VB_TRY(sc.take(b_off + sizeof(float) * (size_t)tot + 64, &d_rows));
    VB_TRY(sc.take(sizeof(double) * (size_t)n, &d_out));
    uint8_t* p = (uint8_t*)d_rows;
    VB_CUDA(cudaMemcpyAsync(p, row_off, b_off, cudaMemcpyHostToDevice, c.stream));
    if (tot > 0) VB_CUDA(cudaMemcpyAsync(p + b_off, val, sizeof(float) * (size_t)tot, cudaMemcpyHostToDevice, c.stream));
    sparse_norm_kernel<<<(unsigned)((n * 32 + 255) / 256), 256, 0, c.stream>>>((const int64_t*)p, (const float*)(p + b_off), n, 0, (double*)d_out,
                                                                                nullptr, nullptr, nullptr);
    VB_CUDA(cudaGetLastError());
    count_launch();
    VB_CUDA(cudaMemcpyAsync(out, d_out, sizeof(double) * (size_t)n, cudaMemcpyDeviceToHost, c.stream));
    VB_CUDA(cudaStreamSynchronize(c.stream));
    return VB_OK;
}

int vb_sparsevec_l2_normalize_batch(int64_t n, const int64_t* row_off, const int32_t* idx, const float* val, int64_t* out_row_off,
                                    int32_t* out_idx, float* out_val) {
    Scratch sc;
    VB_TRY(require_init());
    VB_REQUIRE(n >= 0 && (n == 0 || (row_off && out_row_off && row_off[0] == 0)), "bad sparsevec normalize arguments");
    if (n == 0) {
        if (out_row_off) out_row_off[0] = 0;
        return VB_OK;
    }
    for (int64_t r = 0; r < n; ++r) VB_REQUIRE(row_off[r + 1] >= row_off[r], "offsets must not decrease (row %lld)", (long long)r);
    Context& c = ctx();
    cudaStream_t s = c.stream;
    const int64_t tot = row_off[n];
    VB_REQUIRE(tot == 0 || (idx && val && out_idx && out_val), "null sparsevec buffers");
    const size_t b_off = sizeof(int64_t) * (size_t)(n + 1);
    const size_t b_idx = (sizeof(int32_t) * (size_t)tot + 15) & ~(size_t)15;
    const size_t b_val = (sizeof(float) * (size_t)tot + 15) & ~(size_t)15;
    void *d_rows, *d_tmp, *d_outb, *d_scan;
    VB_TRY(sc.take(b_off + b_idx + b_val + 64, &d_rows));
    // tmp: quotients | kept[n + 1] | out_off[n + 1] | overflow flag
    VB_TRY(sc.take(b_val + 2 * b_off + 64, &d_tmp));
    VB_TRY(sc.take(b_idx + b_val + 64, &d_outb));
    uint8_t* p = (uint8_t*)d_rows;
    uint8_t* t = (uint8_t*)d_tmp;
    float* d_q = (float*)t;
    int64_t* d_kept = (int64_t*)(t + b_val);
    int64_t* d_ooff = (int64_t*)(t + b_val + b_off);
    int* d_flag = (int*)(t + b_val + 2 * b_off);
    VB_CUDA(cudaMemcpyAsync(p, row_off, b_off, cudaMemcpyHostToDevice, s));
    if (tot > 0) {
        VB_CUDA(cudaMemcpyAsync(p + b_off, idx, sizeof(int32_t) * (size_t)tot, cudaMemcpyHostToDevice, s));
        VB_CUDA(cudaMemcpyAsync(p + b_off + b_idx, val, sizeof(float) * (size_t)tot, cudaMemcpyHostToDevice, s));
    }
    VB_CUDA(cudaMemsetAsync(d_flag, 0, sizeof(int), s));
    VB_CUDA(cudaMemsetAsync(d_kept + n, 0, sizeof(int64_t), s));
    const unsigned grid = (unsigned)((n * 32 + 255) / 256);
    sparse_norm_kernel<<<grid, 256, 0, s>>>((const int64_t*)p, (const float*)(p + b_off + b_idx), n, 1, nullptr, d_q, d_kept, d_flag);
    VB_CUDA(cudaGetLastError());
    count_launch();
    size_t scan_bytes = 0;
    VB_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, scan_bytes, d_kept, d_ooff, (int)(n + 1), s));
    VB_TRY(sc.take(scan_bytes + 64, &d_scan));
    VB_CUDA(cub::DeviceScan::ExclusiveSum(d_scan, scan_bytes, d_kept, d_ooff, (int)(n + 1), s));
    count_launch();
    uint8_t* o = (uint8_t*)d_outb;
    sparse_compact_kernel<<<grid, 256, 0, s>>>((const int64_t*)p, (const int32_t*)(p + b_off), d_q, n, d_ooff, (int32_t*)o, (float*)(o + b_idx));
    VB_CUDA(cudaGetLastError());
    count_launch();
    int flag = 0;
    VB_CUDA(cudaMemcpyAsync(out_row_off, d_ooff, b_off, cudaMemcpyDeviceToHost, s));
    VB_CUDA(cudaMemcpyAsync(&flag, d_flag, sizeof(int), cudaMemcpyDeviceToHost, s));
    VB_CUDA(cudaStreamSynchronize(s));
    // float_overflow_error() (src/sparsevec.c:1107-1108)
    VB_REQUIRE(!flag, "value out of range: overflow");
    const int64_t kept = out_row_off[n];
    if (kept > 0) {
        VB_CUDA(cudaMemcpyAsync(out_idx, o, sizeof(int32_t) * (size_t)kept, cudaMemcpyDeviceToHost, s));
        VB_CUDA(cudaMemcpyAsync(out_val, o + b_idx, sizeof(float) * (size_t)kept, cudaMemcpyDeviceToHost, s));
        VB_CUDA(cudaStreamSynchronize(s));
    }
    return VB_OK;
}

// ----------------------------------------------------------------------------- resident CSR table + exact scan

int vb_sparse_table_create(int dim, vb_sparse_table** out) {
    VB_TRY(require_init());
    VB_REQUIRE(out && dim >= 1 && dim <= SP_MAX_DIM, "sparsevec must have between 1 and %d dimensions", SP_MAX_DIM);
    vb_sparse_table* t = new vb_sparse_table();
    t->t.dim = dim;
    *out = t;
    return VB_OK;
}

int vb_sparse_table_append(vb_sparse_table* h, int64_t n, const int64_t* row_off, const int32_t* idx, const float* val) {
    return sparse_append(h, n, row_off, idx, val, true);
}

int vb_sparse_table_append_dev(vb_sparse_table* h, int64_t n, const int64_t* row_off_dev, const int32_t* idx_dev, const float* val_dev) {
    return sparse_append(h, n, row_off_dev, idx_dev, val_dev, false);
}

int64_t vb_sparse_table_rows(const vb_sparse_table* h) { return h ? h->t.n : 0; }
int64_t vb_sparse_table_nnz(const vb_sparse_table* h) { return h ? h->t.nnz : 0; }

int vb_sparse_table_free(vb_sparse_table* h) {
    if (h) {
        if (h->t.row_off) cudaFree(h->t.row_off);
        if (h->t.idx) cudaFree(h->t.idx);
        if (h->t.val) cudaFree(h->t.val);
        owner_released(h->uid);
        delete h;
    }
    return VB_OK;
}

int vb_sparse_exact_topk(vb_sparse_table* h, int metric, int q_dim, int64_t nq, const int64_t* q_off, const int32_t* q_idx, const float* q_val,
                         int k, int64_t* out_ids, double* out_dist) {
    return sparse_exact_topk(h, metric, q_dim, nq, q_off, q_idx, q_val, k, true, out_ids, out_dist, nullptr);
}

int vb_sparse_exact_topk_dev(vb_sparse_table* h, int metric, int q_dim, int64_t nq, const int64_t* q_off_dev, const int32_t* q_idx_dev,
                             const float* q_val_dev, int k, int64_t* out_ids_dev, float* out_dist_dev) {
    return sparse_exact_topk(h, metric, q_dim, nq, q_off_dev, q_idx_dev, q_val_dev, k, false, out_ids_dev, nullptr, out_dist_dev);
}

int vb_sparse_table_filter_create(vb_sparse_table* h, const int64_t* rows, int64_t n, vb_filter** out) {
    return table_filter_create("vb_sparse_table_filter_create", h, h ? h->uid : 0, h ? h->t.n : 0, FILTER_SPARSE, rows, n, true, out);
}

int vb_sparse_table_filter_create_dev(vb_sparse_table* h, const int64_t* rows_dev, int64_t n, vb_filter** out) {
    return table_filter_create("vb_sparse_table_filter_create", h, h ? h->uid : 0, h ? h->t.n : 0, FILTER_SPARSE, rows_dev, n, false, out);
}

int vb_sparse_exact_topk_filtered(vb_sparse_table* h, int metric, int q_dim, int64_t nq, const int64_t* q_off, const int32_t* q_idx,
                                  const float* q_val, int k, const vb_filter* const* filters, int nfilters, const int32_t* filter_of_query,
                                  int64_t* out_ids, double* out_dist) {
    return sparse_topk_filtered(h, metric, q_dim, nq, q_off, q_idx, q_val, k, filters, nfilters, filter_of_query, true, out_ids, out_dist,
                                nullptr);
}

int vb_sparse_exact_topk_filtered_dev(vb_sparse_table* h, int metric, int q_dim, int64_t nq, const int64_t* q_off_dev,
                                      const int32_t* q_idx_dev, const float* q_val_dev, int k, const vb_filter* const* filters, int nfilters,
                                      const int32_t* filter_of_query, int64_t* out_ids_dev, float* out_dist_dev) {
    return sparse_topk_filtered(h, metric, q_dim, nq, q_off_dev, q_idx_dev, q_val_dev, k, filters, nfilters, filter_of_query, false,
                                out_ids_dev, nullptr, out_dist_dev);
}

int vb_sparse_table_rerank(vb_sparse_table* h, int metric, int q_dim, int64_t nq, const int64_t* q_off, const int32_t* q_idx,
                           const float* q_val, const int64_t* cand, int c, int k, int64_t* out_ids, double* out_dist) {
    return sparse_rerank(h, metric, q_dim, nq, q_off, q_idx, q_val, cand, c, k, true, out_ids, out_dist, nullptr);
}

int vb_sparse_table_rerank_dev(vb_sparse_table* h, int metric, int q_dim, int64_t nq, const int64_t* q_off_dev, const int32_t* q_idx_dev,
                               const float* q_val_dev, const int64_t* cand_dev, int c, int k, int64_t* out_ids_dev, float* out_dist_dev) {
    return sparse_rerank(h, metric, q_dim, nq, q_off_dev, q_idx_dev, q_val_dev, cand_dev, c, k, false, out_ids_dev, nullptr, out_dist_dev);
}

// ----------------------------------------------------------------------------- casts

int vb_dense_to_sparsevec_batch(int elem, int dim, const void* rows, int64_t n, int64_t cap, int64_t* out_row_off, int32_t* out_idx,
                                float* out_val) {
    return dense_to_sparse(elem, dim, rows, n, cap, true, out_row_off, out_idx, out_val);
}

int vb_dense_to_sparsevec_batch_dev(int elem, int dim, const void* rows_dev, int64_t n, int64_t cap, int64_t* out_row_off_dev,
                                    int32_t* out_idx_dev, float* out_val_dev) {
    return dense_to_sparse(elem, dim, rows_dev, n, cap, false, out_row_off_dev, out_idx_dev, out_val_dev);
}

int vb_array_to_sparsevec_batch(int src, int dim, int32_t typmod, const void* in, const int64_t* in_off, int64_t n, int64_t cap,
                                int64_t* out_row_off, int32_t* out_idx, float* out_val, int64_t* out_bad) {
    return array_to_sparse(src, dim, typmod, in, in_off, n, cap, true, out_row_off, out_idx, out_val, out_bad);
}

int vb_array_to_sparsevec_batch_dev(int src, int dim, int32_t typmod, const void* in_dev, const int64_t* in_off_dev, int64_t n, int64_t cap,
                                    int64_t* out_row_off_dev, int32_t* out_idx_dev, float* out_val_dev, int64_t* out_bad) {
    return array_to_sparse(src, dim, typmod, in_dev, in_off_dev, n, cap, false, out_row_off_dev, out_idx_dev, out_val_dev, out_bad);
}

int vb_sparsevec_to_dense_batch(int elem, int dim, int64_t n, const int64_t* row_off, const int32_t* idx, const float* val, void* out) {
    return sparse_to_dense(elem, dim, n, row_off, idx, val, out, true);
}

int vb_sparsevec_to_dense_batch_dev(int elem, int dim, int64_t n, const int64_t* row_off_dev, const int32_t* idx_dev, const float* val_dev,
                                    void* out_dev) {
    return sparse_to_dense(elem, dim, n, row_off_dev, idx_dev, val_dev, out_dev, false);
}

}  // extern "C"
