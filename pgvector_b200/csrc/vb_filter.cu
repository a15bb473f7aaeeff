// vb_filter.cu -- row filters: the allowed rows of a table or an IVFFlat image, on the device, and the filtered exact
// top-k.  This is the plan pgvector's README recommends for selective filters ("Filtering": a B-tree or bitmap scan on
// the filter column, then an exact sort by distance), and the row set the filtered IVFFlat iterative scan
// (vb_ivf_scan_begin_filtered, vb_ivf.cu) restricts its groups to.
//
// Construction, all on the device (the host never sees image positions):
//   IVFFlat: CUB radix sort of the given heap ids; filter_ivf_bits_kernel, one thread per image row, binary-searches
//            its id and a warp ballot writes each 32-row word of a bitset (no atomics);
//   table:   filter_table_bits_kernel sets the bits of the given row numbers (a sparse table's filters too, of their
//            own kind: vb_sparse_table_filter_create);
//   then filter_count_kernel / filter_scan_kernel / filter_write_kernel compact the bitset into ascending positions
//   (per-block popcounts, one scan of the block sums, per-thread offsets), and filter_list_off_kernel, one thread per
//   list, binary-searches the image's list offsets in the positions to give each list's run.
//
// Filtered exact top-k, per sub-batch of queries: the re-rank of vb_rerank.cu with implicit candidates --
//   1. filter_chunks_kernel, one warp per query: the scan chunks of its filter's positions (row_begin into the call's
//      concatenated position arrays, one copy per filter, not per query; out_off into the query's distance run), the
//      queries that share a filter in one block of chunks;
//   2. scan_gather_kernel (vb_scan.cu): the exact scan's per-row arithmetic over the gathered rows, one launch per
//      filter block that fills the grid, so that the whole grid reads one filter's rows at a time (L2 reuse);
//   3. segment_topk_kernel over each query's run: ties by position = by row number (positions are ascending);
//   4. filter_finish_kernel: position -> row number, the operator's epilogue.
// Roofline: HBM gathers of the allowed rows, bytes = sum over queries of allowed rows x row stride.
// The sparse filtered top-k (vb_sparse.cu) takes the same sub-batch plan, chunks and selection, with
// sparse_gather_kernel as step 2.
#include "vb_common.cuh"
#include "vb_distance.cuh"

#include <cub/cub.cuh>

#include <algorithm>
#include <atomic>
#include <vector>

namespace vb {

uint64_t next_owner_uid() {
    static std::atomic<uint64_t> next{1};
    return next.fetch_add(1);
}

constexpr int FILTER_MAX_K = 2048;   // as the re-rank: segment_topk_kernel selects without host-side segment sizes
constexpr int FB_THREADS = 256;      // compaction: one bitset word per thread, 8192 rows per block

// ---------------------------------------------------------------------------------------------- construction

// sorted[0 .. m) ascending: bit r of the bitset = the id of image row r is one of them
__global__ void __launch_bounds__(256) filter_ivf_bits_kernel(int64_t n_rows, const int64_t* __restrict__ image_ids,
                                                              const int64_t* __restrict__ sorted, int64_t m, uint32_t* __restrict__ bits) {
    const int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    bool hit = false;
    if (r < n_rows && m > 0) {
        const int64_t id = image_ids ? image_ids[r] : r;
        int64_t lo = 0, hi = m;   // first sorted[i] >= id
        while (lo < hi) {
            const int64_t mid = (lo + hi) >> 1;
            if (sorted[mid] < id) lo = mid + 1;
            else hi = mid;
        }
        hit = lo < m && sorted[lo] == id;
    }
    const unsigned b = __ballot_sync(0xffffffffu, hit);   // a warp covers one 32-row word (blockDim is a multiple of 32)
    if ((threadIdx.x & 31) == 0 && r < n_rows) bits[r >> 5] = b;
}

__global__ void filter_table_bits_kernel(const int64_t* __restrict__ rows, int64_t m, int64_t n_rows, uint32_t* __restrict__ bits) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= m) return;
    const int64_t r = rows[i];
    if (r >= 0 && r < n_rows) atomicOr(&bits[r >> 5], 1u << (r & 31));
}

// exclusive prefix of v over one block of FB_THREADS threads; *total = the block's sum
__device__ __forceinline__ int64_t block_exclusive(int64_t v, int64_t* total) {
    __shared__ int64_t s_warp[FB_THREADS / 32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    int64_t inc = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int64_t y = __shfl_up_sync(0xffffffffu, inc, o);
        if (lane >= o) inc += y;
    }
    if (lane == 31) s_warp[warp] = inc;
    __syncthreads();
    int64_t before = 0, sum = 0;
#pragma unroll
    for (int w = 0; w < FB_THREADS / 32; ++w) {
        if (w < warp) before += s_warp[w];
        sum += s_warp[w];
    }
    __syncthreads();   // s_warp may be reused by the caller's next call
    *total = sum;
    return before + inc - v;
}

__global__ void __launch_bounds__(FB_THREADS) filter_count_kernel(const uint32_t* __restrict__ bits, int64_t nwords,
                                                                  int64_t* __restrict__ block_sum) {
    const int64_t w = blockIdx.x * (int64_t)FB_THREADS + threadIdx.x;
    int64_t total;
    block_exclusive(w < nwords ? __popc(bits[w]) : 0, &total);
    if (threadIdx.x == 0) block_sum[blockIdx.x] = total;
}

// one block: v[0 .. nb) -> exclusive prefix, v[nb] = the sum
__global__ void __launch_bounds__(FB_THREADS) filter_scan_kernel(int64_t* __restrict__ v, int64_t nb) {
    int64_t carry = 0;
    for (int64_t b0 = 0; b0 < nb; b0 += FB_THREADS) {
        const int64_t i = b0 + threadIdx.x;
        const int64_t x = i < nb ? v[i] : 0;
        int64_t total;
        const int64_t ex = block_exclusive(x, &total);
        if (i < nb) v[i] = carry + ex;
        carry += total;
    }
    if (threadIdx.x == 0) v[nb] = carry;
}

// the set bits of word w go to pos[block_off[block] + the block's prefix before w ..], ascending
__global__ void __launch_bounds__(FB_THREADS) filter_write_kernel(const uint32_t* __restrict__ bits, int64_t nwords,
                                                                  const int64_t* __restrict__ block_off, const int64_t* __restrict__ image_ids,
                                                                  int64_t* __restrict__ pos, int64_t* __restrict__ ids) {
    const int64_t w = blockIdx.x * (int64_t)FB_THREADS + threadIdx.x;
    uint32_t b = w < nwords ? bits[w] : 0u;
    int64_t total;
    int64_t o = block_off[blockIdx.x] + block_exclusive(__popc(b), &total);
    while (b) {
        const int64_t r = w * 32 + (__ffs(b) - 1);
        b &= b - 1;
        pos[o] = r;
        if (ids) ids[o] = image_ids ? image_ids[r] : r;
        ++o;
    }
}

// off[l] = allowed positions below list_off[l] (l = lists: all of them)
__global__ void filter_list_off_kernel(const int64_t* __restrict__ list_off, int lists, const int64_t* __restrict__ pos,
                                       const int64_t* __restrict__ n_allowed, int64_t* __restrict__ off) {
    const int l = blockIdx.x * blockDim.x + threadIdx.x;
    if (l > lists) return;
    const int64_t x = list_off[l];
    int64_t lo = 0, hi = *n_allowed;
    while (lo < hi) {
        const int64_t mid = (lo + hi) >> 1;
        if (pos[mid] < x) lo = mid + 1;
        else hi = mid;
    }
    off[l] = lo;
}

void filter_release(Filter* f) {
    if (f->mem) cudaFree(f->mem);
    f->mem = nullptr;
    f->pos = f->ids = f->off = nullptr;
    f->bits = nullptr;
}

// bits (nwords words, set) -> f->pos / f->ids / f->off, f->n.  The buffers are sized by the count of set bits, read back
// after the scan of the block sums: an IVFFlat image may hold one heap id on several rows, so the allowed rows are not
// bounded by the number of ids given (only by the image's rows).
static int filter_compact(int64_t n_rows, uint32_t* bits, int64_t* block_sum, const int64_t* image_ids, const int64_t* list_off,
                          Filter* f) {
    Context& c = ctx();
    const int64_t nwords = (n_rows + 31) / 32;
    const int64_t nb = std::max<int64_t>(1, (nwords + FB_THREADS - 1) / FB_THREADS);
    filter_count_kernel<<<(unsigned)nb, FB_THREADS, 0, c.stream>>>(bits, nwords, block_sum);
    VB_CUDA(cudaGetLastError());
    filter_scan_kernel<<<1, FB_THREADS, 0, c.stream>>>(block_sum, nb);
    VB_CUDA(cudaGetLastError());
    count_launch(2);
    VB_CUDA(cudaMemcpyAsync(&f->n, block_sum + nb, sizeof(int64_t), cudaMemcpyDeviceToHost, c.stream));
    VB_CUDA(cudaStreamSynchronize(c.stream));
    const size_t n_pos = (size_t)std::max<int64_t>(f->n, 1);
    const bool ivf = f->kind == FILTER_IVF;
    const size_t bytes = 8 * n_pos * (ivf ? 2 : 1) + (ivf ? 8 * ((size_t)f->lists + 1) : 0);
    if (cudaMalloc(&f->mem, bytes) != cudaSuccess) {
        cudaGetLastError();
        f->mem = nullptr;
        set_error("row filter: allocation of %zu bytes failed", bytes);
        return VB_ENOMEM;
    }
    f->pos = (int64_t*)f->mem;
    f->ids = ivf ? f->pos + n_pos : nullptr;
    f->off = ivf ? f->ids + n_pos : nullptr;
    filter_write_kernel<<<(unsigned)nb, FB_THREADS, 0, c.stream>>>(bits, nwords, block_sum, image_ids, f->pos, f->ids);
    VB_CUDA(cudaGetLastError());
    count_launch();
    if (ivf) {
        filter_list_off_kernel<<<(unsigned)((f->lists + 1 + 255) / 256), 256, 0, c.stream>>>(list_off, f->lists, f->pos, block_sum + nb,
                                                                                            f->off);
        VB_CUDA(cudaGetLastError());
        count_launch();
        f->h_off.assign((size_t)f->lists + 1, 0);
        VB_CUDA(cudaMemcpyAsync(f->h_off.data(), f->off, 8 * ((size_t)f->lists + 1), cudaMemcpyDeviceToHost, c.stream));
    }
    VB_CUDA(cudaStreamSynchronize(c.stream));
    return VB_OK;
}

int filter_build_table(int64_t n_rows, const int64_t* rows, int64_t n, bool host, Filter* f) {
    Context& c = ctx();
    const int64_t nwords = (n_rows + 31) / 32;
    const int64_t nb = std::max<int64_t>(1, (nwords + FB_THREADS - 1) / FB_THREADS);
    Scratch sc("row filter");
    void* tmp;
    const size_t bits_bytes = (4 * (size_t)std::max<int64_t>(nwords, 1) + 15) & ~(size_t)15;
    const size_t bytes = bits_bytes + 8 * ((size_t)nb + 1) + (host ? 8 * (size_t)n : 0);
    VB_TRY(sc.own(bytes, &tmp));
    uint32_t* bits = (uint32_t*)tmp;
    int64_t* block_sum = (int64_t*)((uint8_t*)tmp + bits_bytes);
    const int64_t* d_rows = rows;
    if (host && n) {
        int64_t* up = block_sum + nb + 1;
        VB_CUDA(cudaMemcpyAsync(up, rows, 8 * (size_t)n, cudaMemcpyHostToDevice, c.stream));
        d_rows = up;
    }
    VB_CUDA(cudaMemsetAsync(bits, 0, bits_bytes, c.stream));
    if (n) {
        filter_table_bits_kernel<<<(unsigned)((n + 255) / 256), 256, 0, c.stream>>>(d_rows, n, n_rows, bits);
        VB_CUDA(cudaGetLastError());
        count_launch();
    }
    f->kind = FILTER_TABLE;
    return filter_compact(n_rows, bits, block_sum, nullptr, nullptr, f);
}

int filter_build_ivf(int64_t n_rows, const int64_t* image_ids, const int64_t* list_off, int lists, const int64_t* ids, int64_t n,
                     bool host, Filter* f) {
    Context& c = ctx();
    VB_REQUIRE(n < (int64_t)INT32_MAX, "row filter: %lld ids, at most %d per filter", (long long)n, INT32_MAX - 1);
    const int64_t nwords = (n_rows + 31) / 32;
    const int64_t nb = std::max<int64_t>(1, (nwords + FB_THREADS - 1) / FB_THREADS);
    size_t sort_bytes = 0;
    if (n) VB_CUDA(cub::DeviceRadixSort::SortKeys(nullptr, sort_bytes, (const int64_t*)nullptr, (int64_t*)nullptr, (int)n, 0, 64, c.stream));
    Scratch sc("row filter");
    void* tmp;
    const size_t bits_bytes = (4 * (size_t)std::max<int64_t>(nwords, 1) + 15) & ~(size_t)15;
    const size_t bytes = bits_bytes + 8 * ((size_t)nb + 1) + 8 * (size_t)n * (host ? 2 : 1) + sort_bytes + 256;
    VB_TRY(sc.own(bytes, &tmp));
    uint32_t* bits = (uint32_t*)tmp;
    int64_t* block_sum = (int64_t*)((uint8_t*)tmp + bits_bytes);
    int64_t* sorted = block_sum + nb + 1;
    int64_t* up = sorted + n;
    void* sort_tmp = (void*)(((uintptr_t)(up + (host ? n : 0)) + 255) & ~(uintptr_t)255);
    if (n) {
        const int64_t* d_ids = ids;
        if (host) {
            VB_CUDA(cudaMemcpyAsync(up, ids, 8 * (size_t)n, cudaMemcpyHostToDevice, c.stream));
            d_ids = up;
        }
        VB_CUDA(cub::DeviceRadixSort::SortKeys(sort_tmp, sort_bytes, d_ids, sorted, (int)n, 0, 64, c.stream));
    }
    if (nwords) {
        filter_ivf_bits_kernel<<<(unsigned)((nwords * 32 + 255) / 256), 256, 0, c.stream>>>(n_rows, image_ids, sorted, n, bits);
        VB_CUDA(cudaGetLastError());
        count_launch();
    }
    f->kind = FILTER_IVF;
    f->lists = lists;
    return filter_compact(n_rows, bits, block_sum, image_ids, list_off, f);
}

// The bitset is the filter itself (the HNSW iterative scan tests one bit per returned element); only its count is
// computed, by the first two steps of the compaction.
int filter_build_hnsw(int64_t n_elems, const int64_t* elems, int64_t n, bool host, Filter* f) {
    Context& c = ctx();
    const int64_t nwords = std::max<int64_t>(1, (n_elems + 31) / 32);
    const int64_t nb = (nwords + FB_THREADS - 1) / FB_THREADS;
    f->kind = FILTER_HNSW;
    f->words = nwords;
    if (cudaMalloc(&f->mem, 4 * (size_t)nwords) != cudaSuccess) {
        cudaGetLastError();
        f->mem = nullptr;
        set_error("row filter: allocation of %zu bytes failed", 4 * (size_t)nwords);
        return VB_ENOMEM;
    }
    f->bits = (uint32_t*)f->mem;
    Scratch sc("row filter");
    void* tmp;
    VB_TRY(sc.own(8 * ((size_t)nb + 1) + (host ? 8 * (size_t)n : 0), &tmp));
    int64_t* block_sum = (int64_t*)tmp;
    const int64_t* d_elems = elems;
    if (host && n) {
        int64_t* up = block_sum + nb + 1;
        VB_CUDA(cudaMemcpyAsync(up, elems, 8 * (size_t)n, cudaMemcpyHostToDevice, c.stream));
        d_elems = up;
    }
    VB_CUDA(cudaMemsetAsync(f->bits, 0, 4 * (size_t)nwords, c.stream));
    if (n) {
        filter_table_bits_kernel<<<(unsigned)((n + 255) / 256), 256, 0, c.stream>>>(d_elems, n, n_elems, f->bits);
        VB_CUDA(cudaGetLastError());
        count_launch();
    }
    filter_count_kernel<<<(unsigned)nb, FB_THREADS, 0, c.stream>>>(f->bits, nwords, block_sum);
    VB_CUDA(cudaGetLastError());
    filter_scan_kernel<<<1, FB_THREADS, 0, c.stream>>>(block_sum, nb);
    VB_CUDA(cudaGetLastError());
    count_launch(2);
    VB_CUDA(cudaMemcpyAsync(&f->n, block_sum + nb, sizeof(int64_t), cudaMemcpyDeviceToHost, c.stream));
    VB_CUDA(cudaStreamSynchronize(c.stream));
    return VB_OK;
}

// ---------------------------------------------------------------------------------------------- filtered exact top-k

// One warp per query: the chunks of its allowed rows and its segment.
__global__ void __launch_bounds__(256) filter_chunks_kernel(const FilterQuery* __restrict__ qa, int64_t nq, int rows_per_chunk,
                                                            int64_t* __restrict__ seg_begin, int32_t* __restrict__ seg_len,
                                                            Chunk* __restrict__ chunks) {
    const int64_t q = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (q >= nq) return;   // whole warps
    const FilterQuery a = qa[q];
    const int nch = (a.len + rows_per_chunk - 1) / rows_per_chunk;
    if (lane == 0) {
        seg_begin[q] = a.run;
        seg_len[q] = a.len;
    }
    for (int i = lane; i < nch; i += 32) {
        Chunk ch;
        ch.row_begin = a.base + (int64_t)i * rows_per_chunk;   // into the concatenated positions
        ch.out_off = a.run + (int64_t)i * rows_per_chunk;
        ch.n_rows = min(rows_per_chunk, a.len - i * rows_per_chunk);
        ch.q = (int32_t)q;
        chunks[a.cbase + i] = ch;
    }
}

int launch_filter_chunks(const FilterQuery* qa_dev, int64_t nq, int rows_per_chunk, int64_t* seg_begin, int32_t* seg_len, Chunk* chunks) {
    Context& cx = ctx();
    filter_chunks_kernel<<<(unsigned)((nq * 32 + 255) / 256), 256, 0, cx.stream>>>(qa_dev, nq, rows_per_chunk, seg_begin, seg_len, chunks);
    VB_CUDA(cudaGetLastError());
    count_launch();
    return VB_OK;
}

int filter_concat_positions(Scratch& sc, const vb_filter* const* filters, int nfilters, std::vector<int64_t>* fbase, const int64_t** rows) {
    Context& cx = ctx();
    fbase->assign((size_t)nfilters + 1, 0);
    for (int i = 0; i < nfilters; ++i) (*fbase)[(size_t)i + 1] = (*fbase)[(size_t)i] + filters[i]->f.n;
    *rows = filters[0]->f.pos;
    if (nfilters > 1) {
        void* d_cat;
        VB_TRY(sc.take(8 * (size_t)std::max<int64_t>(fbase->back(), 1), &d_cat));
        for (int i = 0; i < nfilters; ++i)
            if (filters[i]->f.n)
                VB_CUDA(cudaMemcpyAsync((int64_t*)d_cat + (*fbase)[(size_t)i], filters[i]->f.pos, 8 * (size_t)filters[i]->f.n,
                                        cudaMemcpyDeviceToDevice, cx.stream));
        *rows = (const int64_t*)d_cat;
    }
    return VB_OK;
}

int filter_batch_plan(const vb_filter* const* filters, int nfilters, const int32_t* filter_of_query, const int64_t* fbase, int64_t q0,
                      int64_t nq, int64_t max_q, int rpc, int64_t grid_chunks, FilterBatch* b) {
    const int64_t dist_cap = (int64_t)(1ull << 28);   // distances per sub-batch: ~1 GiB
    std::vector<int32_t> group((size_t)nfilters, 0);
    std::vector<int64_t> cbase((size_t)nfilters);
    b->qa.clear();
    b->run = 0;
    b->max_chunks = 0;
    for (int64_t q = q0; q < nq && q - q0 < max_q; ++q) {
        const int fi = filter_of_query ? filter_of_query[q] : 0;
        const int64_t len = filters[fi]->f.n;
        if (!b->qa.empty() && b->run + len > dist_cap) break;
        b->qa.push_back(FilterQuery{b->run, fbase[fi], (int64_t)group[(size_t)fi]++, (int32_t)len, 0});
        b->run += len;
        b->max_chunks += (len + rpc - 1) / rpc;
    }
    // each filter's queries get one block of chunks, in filter order, query after query (cbase held the rank)
    int64_t cb = 0;
    b->launch_begin.assign(1, 0);
    b->launch_count.clear();
    for (int i = 0; i < nfilters; ++i) {
        cbase[(size_t)i] = cb;
        cb += (int64_t)group[(size_t)i] * ((filters[i]->f.n + rpc - 1) / rpc);
        if (cb - b->launch_begin.back() >= grid_chunks || (i == nfilters - 1 && cb > b->launch_begin.back())) {
            b->launch_count.push_back((int32_t)(cb - b->launch_begin.back()));
            b->launch_begin.push_back(cb);
        }
    }
    for (size_t j = 0; j < b->qa.size(); ++j) {
        const int fi = filter_of_query ? filter_of_query[q0 + (int64_t)j] : 0;
        b->qa[j].cbase = cbase[(size_t)fi] + b->qa[j].cbase * ((b->qa[j].len + rpc - 1) / rpc);
    }
    VB_REQUIRE(b->max_chunks < (int64_t)INT32_MAX, "filtered top-k: too many scan chunks (%lld)", (long long)b->max_chunks);
    return VB_OK;
}

__global__ void filter_finish_kernel(int metric, int64_t total, int k, const FilterQuery* __restrict__ qa, const int32_t* __restrict__ pos,
                                     const float* __restrict__ key, const int64_t* __restrict__ rows, int64_t* __restrict__ out_ids,
                                     float* __restrict__ out_f, double* __restrict__ out_d) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= total) return;
    const int32_t p = pos[i];
    out_ids[i] = p >= 0 ? rows[qa[i / k].base + p] : -1;
    const double v = finish_value(metric, key[i]);
    if (out_f) out_f[i] = (float)v;
    if (out_d) out_d[i] = v;
}

static int exact_topk_filtered_impl(vb_table* t, int metric, const void* queries, int64_t nq, int k, const vb_filter* const* filters,
                                    int nfilters, const int32_t* filter_of_query, bool host, int64_t* out_ids, float* out_f,
                                    double* out_d) {
    VB_TRY(require_init());
    VB_REQUIRE(t && metric_valid_for(t->t.elem, metric) && metric != VB_SPHERICAL, "bad table/metric");
    VB_REQUIRE(k >= 1 && k <= FILTER_MAX_K, "filtered top-k: k must be in 1..%d, got %d", FILTER_MAX_K, k);
    VB_REQUIRE(filters && nfilters >= 1, "filtered top-k: no row filter given");
    VB_REQUIRE(filter_of_query || nfilters == 1, "filtered top-k: filter_of_query may only be NULL with one filter (got %d)", nfilters);
    for (int i = 0; i < nfilters; ++i) {
        VB_REQUIRE(filters[i], "filtered top-k: filter %d is NULL", i);
        const Filter& f = filters[i]->f;
        VB_REQUIRE(f.kind == FILTER_TABLE && f.owner == t && f.owner_uid == t->uid, "filtered top-k: filter %d was made for another table or index", i);
        VB_REQUIRE(f.n < (int64_t)INT32_MAX, "filtered top-k: filter %d allows %lld rows, at most %d", i, (long long)f.n, INT32_MAX - 1);
    }
    if (nq <= 0) return VB_OK;
    VB_REQUIRE(queries && out_ids && (out_f || out_d), "filtered top-k: null argument");
    for (int64_t q = 0; q < nq && filter_of_query; ++q)
        VB_REQUIRE(filter_of_query[q] >= 0 && filter_of_query[q] < nfilters, "filtered top-k: filter_of_query[%lld] = %d, not in 0..%d",
                   (long long)q, filter_of_query[q], nfilters - 1);
    Context& cx = ctx();
    Table& T = t->t;
    // the filters' positions side by side (one device copy per filter; a single filter is read in place)
    Scratch sc;
    std::vector<int64_t> fbase;
    const int64_t* rows;
    VB_TRY(filter_concat_positions(sc, filters, nfilters, &fbase, &rows));
    const size_t rawq = raw_row_bytes(T.elem, T.dim);
    const int rpc = scan_chunk_rows(T);
    const int km = key_metric(metric);
    // A scan launch spreads its chunk list over the whole grid in contiguous slices.  Queries that share a filter read
    // the same rows, so each filter's block of chunks gets a launch of its own once it fills the grid: every CTA then
    // reads that filter's rows, which stay in L2 for the other queries.  Smaller blocks share a launch.
    const int64_t grid_chunks = 8 * (int64_t)cx.sm_count;
    FilterBatch b;
    for (int64_t q0 = 0; q0 < nq;) {
        Scratch batch;
        VB_TRY(filter_batch_plan(filters, nfilters, filter_of_query, fbase.data(), q0, nq, INT64_MAX, rpc, grid_chunks, &b));
        const std::vector<FilterQuery>& qa = b.qa;
        const std::vector<int64_t>& launch_begin = b.launch_begin;
        const std::vector<int32_t>& launch_count = b.launch_count;
        const int64_t m = (int64_t)qa.size(), run = b.run, max_chunks = b.max_chunks;
        void *qimg, *d_qa, *d_chunks, *d_dist, *d_pos;
        size_t qstride;
        VB_TRY(upload_queries(batch, T.elem, T.dim, (const uint8_t*)queries + (size_t)q0 * rawq, m, host, &qimg, &qstride));
        const size_t qa_bytes = (sizeof(FilterQuery) * (size_t)m + 255) & ~(size_t)255;
        const size_t nl = launch_count.size();
        VB_TRY(batch.take(qa_bytes + (sizeof(int64_t) + sizeof(int32_t)) * (size_t)m + sizeof(int32_t) * nl + 64, &d_qa));
        int64_t* seg_begin = (int64_t*)((uint8_t*)d_qa + qa_bytes);
        int32_t* seg_len = (int32_t*)(seg_begin + m);
        int32_t* d_count = seg_len + m;   // chunks of each scan launch
        VB_CUDA(cudaMemcpyAsync(d_qa, qa.data(), sizeof(FilterQuery) * (size_t)m, cudaMemcpyHostToDevice, cx.stream));
        if (nl) VB_CUDA(cudaMemcpyAsync(d_count, launch_count.data(), sizeof(int32_t) * nl, cudaMemcpyHostToDevice, cx.stream));
        VB_TRY(batch.take(sizeof(Chunk) * (size_t)max_chunks + 64, &d_chunks));
        VB_TRY(launch_filter_chunks((const FilterQuery*)d_qa, m, rpc, seg_begin, seg_len, (Chunk*)d_chunks));
        VB_TRY(batch.take(sizeof(float) * (size_t)std::max<int64_t>(run, 1), &d_dist));
        for (size_t l = 0; l < nl; ++l)
            VB_TRY(launch_scan_gather(T, km, qimg, qstride, rows, (const Chunk*)d_chunks + launch_begin[l], d_count + l, launch_count[l],
                                      (float*)d_dist));
        VB_TRY(batch.take((sizeof(int32_t) + sizeof(float)) * (size_t)m * k, &d_pos));
        int32_t* pos = (int32_t*)d_pos;
        float* key = (float*)(pos + (size_t)m * k);
        VB_TRY(launch_segment_topk_v((const float*)d_dist, seg_begin, seg_len, nullptr, nullptr, m, k, pos, key));
        int64_t* o_ids;
        float* o_f = nullptr;
        double* o_d = nullptr;
        if (host) {
            void* d_out;
            VB_TRY(batch.take((sizeof(int64_t) + sizeof(double)) * (size_t)m * k, &d_out));
            o_ids = (int64_t*)d_out;
            o_d = (double*)(o_ids + (size_t)m * k);
        } else {
            o_ids = out_ids + q0 * k;
            o_f = out_f + q0 * k;
        }
        filter_finish_kernel<<<(unsigned)((m * k + 255) / 256), 256, 0, cx.stream>>>(metric, m * k, k, (const FilterQuery*)d_qa, pos, key,
                                                                                    rows, o_ids, o_f, o_d);
        VB_CUDA(cudaGetLastError());
        count_launch();
        if (host) {
            VB_CUDA(cudaMemcpyAsync(out_ids + q0 * k, o_ids, sizeof(int64_t) * (size_t)m * k, cudaMemcpyDeviceToHost, cx.stream));
            VB_CUDA(cudaMemcpyAsync(out_d + q0 * k, o_d, sizeof(double) * (size_t)m * k, cudaMemcpyDeviceToHost, cx.stream));
            VB_CUDA(cudaStreamSynchronize(cx.stream));
        }
        q0 += m;   // (qa is pageable: its copy has been staged by the time cudaMemcpyAsync returned, so it may be refilled)
    }
    return VB_OK;
}

int table_filter_create(const char* fn, const void* owner, uint64_t owner_uid, int64_t n_rows, FilterKind kind, const int64_t* rows,
                        int64_t n, bool host, vb_filter** out) {
    VB_TRY(require_init());
    VB_REQUIRE(out, "%s: null filter pointer", fn);
    *out = nullptr;
    VB_REQUIRE(owner, "%s: null table", fn);
    VB_REQUIRE(n >= 0 && (rows || n == 0), "%s: null rows or negative count %lld", fn, (long long)n);
    if (host)
        for (int64_t i = 0; i < n; ++i)
            VB_REQUIRE(rows[i] >= 0 && rows[i] < n_rows, "%s: rows[%lld] = %lld is not a row of the table (0..%lld)", fn, (long long)i,
                       (long long)rows[i], (long long)n_rows - 1);
    vb_filter* h = new vb_filter;
    h->f.owner = owner;
    h->f.owner_uid = owner_uid;
    const int rc = filter_build_table(n_rows, rows, n, host, &h->f);
    if (rc != VB_OK) {
        filter_release(&h->f);
        delete h;
        return rc;
    }
    h->f.kind = kind;
    *out = h;
    return VB_OK;
}

}  // namespace vb

using namespace vb;

extern "C" {

int vb_table_filter_create(vb_table* t, const int64_t* rows, int64_t n, vb_filter** out) {
    return table_filter_create("vb_table_filter_create", t, t ? t->uid : 0, t ? t->t.n : 0, FILTER_TABLE, rows, n, true, out);
}

int vb_table_filter_create_dev(vb_table* t, const int64_t* rows_dev, int64_t n, vb_filter** out) {
    return table_filter_create("vb_table_filter_create", t, t ? t->uid : 0, t ? t->t.n : 0, FILTER_TABLE, rows_dev, n, false, out);
}

int64_t vb_filter_rows(const vb_filter* f) { return f ? f->f.n : 0; }

int vb_filter_free(vb_filter* f) {
    if (!f) return VB_OK;
    if (f->f.mem) cudaStreamSynchronize(ctx().stream);
    filter_release(&f->f);
    delete f;
    return VB_OK;
}

int vb_exact_topk_filtered(vb_table* t, int metric, const void* queries, int64_t nq, int k, const vb_filter* const* filters, int nfilters,
                           const int32_t* filter_of_query, int64_t* out_ids, double* out_dist) {
    return exact_topk_filtered_impl(t, metric, queries, nq, k, filters, nfilters, filter_of_query, true, out_ids, nullptr, out_dist);
}

int vb_exact_topk_filtered_dev(vb_table* t, int metric, const void* queries_dev, int64_t nq, int k, const vb_filter* const* filters,
                               int nfilters, const int32_t* filter_of_query, int64_t* out_ids_dev, float* out_dist_dev) {
    return exact_topk_filtered_impl(t, metric, queries_dev, nq, k, filters, nfilters, filter_of_query, false, out_ids_dev, out_dist_dev,
                                    nullptr);
}

}  // extern "C"
