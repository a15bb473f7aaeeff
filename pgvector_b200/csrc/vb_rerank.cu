// vb_rerank.cu -- re-rank of per-query candidate rows against a resident table: the outer
// "ORDER BY v <op> q LIMIT k" over an inner index scan's result (pgvector's quantize-then-rerank pattern:
// an index on binary_quantize(v), a subvector or a halfvec cast fetches the candidates, the full rows order them).
//
// Per sub-batch of queries:
//   1. rerank_prepare_kernel, one warp per query: keeps the candidates that name a row of the table, in candidate
//      order (ballot prefix), and writes the query's segment and its chunks of scan work;
//   2. scan_gather_kernel (vb_scan.cu): the exact scan's per-row arithmetic over the gathered rows, so distances are
//      bit-identical to vb_exact_topk's LDG scan;
//   3. segment_topk_kernel over [q c, q c + valid_q): its position tie-break is "earlier candidate first", and
//      padding never enters the selection (a NaN distance, e.g. cosine against a zero row, still ranks before -1);
//   4. rerank_finish_kernel: position -> row id, the operator's epilogue.
//
// Roofline: HBM gathers, bytes = sum over queries of valid candidates x row stride (each row is contiguous: 4 KB for
// 1024-d fp32, 128 B for bit(1024)); the ids, query images and keys are a few percent of that.
#include "vb_common.cuh"
#include "vb_distance.cuh"

#include <algorithm>

namespace vb {

constexpr int RERANK_MAX_K = 2048;   // the largest k segment_topk_kernel selects without host-side segment sizes

// One warp per query: ids[q c + j], j < valid_q = the candidates in [0, n), in candidate order.
__global__ void __launch_bounds__(256) rerank_prepare_kernel(const int64_t* __restrict__ cand, int64_t nq, int c, int64_t n,
                                                             int rows_per_chunk, int64_t* __restrict__ ids,
                                                             int64_t* __restrict__ seg_begin, int32_t* __restrict__ seg_len,
                                                             Chunk* __restrict__ chunks, int* __restrict__ n_chunks) {
    const int64_t q = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (q >= nq) return;   // whole warps
    const int64_t off = q * c;
    int valid = 0;
    for (int j0 = 0; j0 < c; j0 += 32) {
        const int j = j0 + lane;
        const int64_t id = j < c ? cand[off + j] : -1;
        const bool ok = id >= 0 && id < n;
        const unsigned b = __ballot_sync(0xffffffffu, ok);
        if (ok) ids[off + valid + __popc(b & ((1u << lane) - 1u))] = id;
        valid += __popc(b);
    }
    const int nch = (valid + rows_per_chunk - 1) / rows_per_chunk;
    int base = 0;
    if (lane == 0) {
        seg_begin[q] = off;
        seg_len[q] = valid;
        base = atomicAdd(n_chunks, nch);
    }
    base = __shfl_sync(0xffffffffu, base, 0);
    for (int i = lane; i < nch; i += 32) {
        Chunk ch;
        ch.row_begin = off + (int64_t)i * rows_per_chunk;   // into ids[]
        ch.out_off = ch.row_begin;                          // distances share the candidates' layout
        ch.n_rows = min(rows_per_chunk, valid - i * rows_per_chunk);
        ch.q = (int32_t)q;
        chunks[base + i] = ch;
    }
}

int launch_rerank_prepare(const int64_t* cand, int64_t nq, int c, int64_t n, int rows_per_chunk, int64_t* ids, int64_t* seg_begin,
                          int32_t* seg_len, Chunk* chunks, int* n_chunks) {
    Context& cx = ctx();
    rerank_prepare_kernel<<<(unsigned)((nq * 32 + 255) / 256), 256, 0, cx.stream>>>(cand, nq, c, n, rows_per_chunk, ids, seg_begin, seg_len,
                                                                                   chunks, n_chunks);
    VB_CUDA(cudaGetLastError());
    count_launch();
    return VB_OK;
}

__global__ void rerank_finish_kernel(int metric, int64_t total, int k, int c, const int32_t* __restrict__ pos,
                                     const float* __restrict__ key, const int64_t* __restrict__ ids, int64_t* __restrict__ out_ids,
                                     float* __restrict__ out_f, double* __restrict__ out_d) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= total) return;
    const int32_t p = pos[i];
    out_ids[i] = p >= 0 ? ids[(i / k) * c + p] : -1;
    const double v = finish_value(metric, key[i]);
    if (out_f) out_f[i] = (float)v;
    if (out_d) out_d[i] = v;
}

static int rerank_impl(vb_table* t, int metric, const void* queries, int64_t nq, const int64_t* cand, int c, int k, bool host,
                       int64_t* out_ids, float* out_f, double* out_d) {
    VB_TRY(require_init());
    VB_REQUIRE(t && metric_valid_for(t->t.elem, metric) && metric != VB_SPHERICAL, "bad table/metric");
    VB_REQUIRE(k >= 1 && k <= RERANK_MAX_K, "rerank: k must be in 1..%d, got %d", RERANK_MAX_K, k);
    VB_REQUIRE(c >= 0, "rerank: negative candidate count %d", c);
    if (nq <= 0) return VB_OK;
    VB_REQUIRE(queries && (cand || c == 0) && out_ids && (out_f || out_d), "rerank: null argument");
    Context& cx = ctx();
    Table& T = t->t;
    const int64_t n = T.n;
    if (host) {
        for (int64_t i = 0; i < nq * c; ++i) {
            const int64_t v = cand[i];
            VB_REQUIRE(v >= -1 && v < n, "rerank: candidate %lld of query %lld is %lld, not a row of the table (-1 or 0..%lld)",
                       (long long)(i % c), (long long)(i / c), (long long)v, (long long)n - 1);
        }
    }
    const size_t rawq = raw_row_bytes(T.elem, T.dim);
    const int rpc = scan_chunk_rows(T);
    const int km = key_metric(metric);
    // sub-batch so the distance array stays under ~1 GiB
    const int64_t bq = std::max<int64_t>(1, std::min<int64_t>(nq, (int64_t)(1ull << 30) / (4 * std::max(c, 1))));
    for (int64_t q0 = 0; q0 < nq; q0 += bq) {
        Scratch sc;
        const int64_t m = std::min(bq, nq - q0);
        const size_t mc = (size_t)m * c;
        void *qimg, *d_cand, *d_ids, *d_chunks, *d_seg, *d_dist, *d_pos;
        size_t qstride;
        VB_TRY(upload_queries(sc, T.elem, T.dim, (const uint8_t*)queries + (size_t)q0 * rawq, m, host, &qimg, &qstride));
        if (host) {
            VB_TRY(sc.take(sizeof(int64_t) * mc, &d_cand));
            if (mc) VB_CUDA(cudaMemcpyAsync(d_cand, cand + (size_t)q0 * c, sizeof(int64_t) * mc, cudaMemcpyHostToDevice, cx.stream));
        } else {
            d_cand = const_cast<int64_t*>(cand) + (size_t)q0 * c;
        }
        VB_TRY(sc.take(sizeof(int64_t) * mc, &d_ids));
        const int64_t max_chunks = m * ((c + rpc - 1) / rpc);
        VB_TRY(sc.take(sizeof(Chunk) * (size_t)max_chunks + 64, &d_chunks));
        int* n_chunks = (int*)((Chunk*)d_chunks + max_chunks);
        VB_TRY(sc.take((sizeof(int64_t) + sizeof(int32_t)) * (size_t)m + 64, &d_seg));
        int64_t* seg_begin = (int64_t*)d_seg;
        int32_t* seg_len = (int32_t*)(seg_begin + m);
        VB_CUDA(cudaMemsetAsync(n_chunks, 0, sizeof(int), cx.stream));
        VB_TRY(launch_rerank_prepare((const int64_t*)d_cand, m, c, n, rpc, (int64_t*)d_ids, seg_begin, seg_len, (Chunk*)d_chunks, n_chunks));
        VB_TRY(sc.take(sizeof(float) * mc, &d_dist));
        VB_TRY(launch_scan_gather(T, km, qimg, qstride, (const int64_t*)d_ids, (const Chunk*)d_chunks, n_chunks, (int)max_chunks,
                                  (float*)d_dist));
        VB_TRY(sc.take((sizeof(int32_t) + sizeof(float)) * (size_t)m * k, &d_pos));
        int32_t* pos = (int32_t*)d_pos;
        float* key = (float*)(pos + (size_t)m * k);
        VB_TRY(launch_segment_topk_v((const float*)d_dist, seg_begin, seg_len, nullptr, nullptr, m, k, pos, key));
        int64_t* o_ids;
        float* o_f = nullptr;
        double* o_d = nullptr;
        if (host) {
            void* d_out;
            VB_TRY(sc.take((sizeof(int64_t) + sizeof(double)) * (size_t)m * k, &d_out));
            o_ids = (int64_t*)d_out;
            o_d = (double*)(o_ids + (size_t)m * k);
        } else {
            o_ids = out_ids + q0 * k;
            o_f = out_f + q0 * k;
        }
        rerank_finish_kernel<<<(unsigned)((m * k + 255) / 256), 256, 0, cx.stream>>>(metric, m * k, k, c, pos, key, (const int64_t*)d_ids,
                                                                                    o_ids, o_f, o_d);
        VB_CUDA(cudaGetLastError());
        count_launch();
        if (host) {
            VB_CUDA(cudaMemcpyAsync(out_ids + q0 * k, o_ids, sizeof(int64_t) * (size_t)m * k, cudaMemcpyDeviceToHost, cx.stream));
            VB_CUDA(cudaMemcpyAsync(out_d + q0 * k, o_d, sizeof(double) * (size_t)m * k, cudaMemcpyDeviceToHost, cx.stream));
            VB_CUDA(cudaStreamSynchronize(cx.stream));
        }
    }
    return VB_OK;
}

}  // namespace vb

using namespace vb;

extern "C" {

int vb_table_rerank(vb_table* t, int metric, const void* queries, int64_t nq, const int64_t* cand, int c, int k, int64_t* out_ids,
                    double* out_dist) {
    return rerank_impl(t, metric, queries, nq, cand, c, k, true, out_ids, nullptr, out_dist);
}

int vb_table_rerank_dev(vb_table* t, int metric, const void* queries_dev, int64_t nq, const int64_t* cand_dev, int c, int k,
                        int64_t* out_ids_dev, float* out_dist_dev) {
    return rerank_impl(t, metric, queries_dev, nq, cand_dev, c, k, false, out_ids_dev, out_dist_dev, nullptr);
}

}  // extern "C"
