// vb_scan.cu -- the fused one-query-vs-many-rows distance kernels and the per-query
// top-k select.  sm_90a only.
//
// Replaces the inner loops of GetScanLists / GetScanItems (src/ivfscan.c:68-107,
// 150-174), the sequential-scan operator evaluation (src/vector.c:576-750,
// src/halfvec.c:557-686, src/bitvec.c:33-70) and feeds HNSW / k-means helpers.
//
// Roofline: HBM bandwidth.  Algorithmic bytes per distance = dim * element size
// (the row is read once; the query lives in shared memory; one 4-byte key is
// written per row = 0.07 % of a 1536-d fp32 row).
//
// Memory access: every row starts 16-byte aligned (padded stride), a group of
// LPR lanes walks one row with 128-bit loads (LPR * 16 contiguous bytes per
// step, 512 B per warp step for LPR = 32), RPI rows are in flight per group so
// each thread keeps RPI * UNROLL independent LDG.128 outstanding.
#include "vb_common.cuh"
#include "vb_distance.cuh"
#include "vb_slab_select.cuh"

#include <cub/cub.cuh>

#include <algorithm>
#include <vector>

namespace vb {

constexpr int SCAN_THREADS = 128;

// GATHER: row r of a chunk is table row ids[row_begin + r] (the candidate lists of vb_rerank.cu) instead of row
// row_begin + r; the per-row arithmetic is the same, so gathered distances are bit-identical to the contiguous scan's.
template <int ELEM, int METRIC, int LPR, int RPI, typename OUT, bool GATHER>
__device__ __forceinline__ void scan_body(const ScanArgs& a, const int64_t* __restrict__ ids) {
    extern __shared__ uint4 sq[];
    constexpr int G = SCAN_THREADS / LPR;  // row groups per CTA
    const int g = threadIdx.x / LPR;
    const int l = threadIdx.x % LPR;
    const int V = a.vec_per_row;

    int64_t total;
    if (a.chunks) total = *a.n_chunks_dev;
    else total = a.nq * a.chunks_per_q;
    // contiguous slice of the work list per CTA: consecutive chunks usually share a query
    const int64_t per = (total + gridDim.x - 1) / gridDim.x;
    const int64_t c_begin = per * blockIdx.x;
    const int64_t c_end = min(total, c_begin + per);

    int cur_q = -1;
    for (int64_t c = c_begin; c < c_end; ++c) {
        int64_t row_begin, out_off;
        int n_rows, q;
        if (a.chunks) {
            Chunk ch = a.chunks[c];
            row_begin = ch.row_begin;
            out_off = ch.out_off;
            n_rows = ch.n_rows;
            q = ch.q;
        } else {
            q = (int)(c / a.chunks_per_q);
            int64_t r0 = (c % a.chunks_per_q) * a.rows_per_chunk;
            row_begin = r0;
            n_rows = (int)min((int64_t)a.rows_per_chunk, a.n_rows - r0);
            out_off = (int64_t)q * a.out_stride + r0;
        }
        if (q != cur_q) {
            __syncthreads();
            const uint4* gq = reinterpret_cast<const uint4*>(a.queries + (size_t)q * a.qstride);
            for (int i = threadIdx.x; i < a.qvec; i += SCAN_THREADS) sq[i] = gq[i];
            __syncthreads();
            cur_q = q;
        }
        const uint8_t* base = a.rows + (size_t)row_begin * a.stride;
        OUT* out = reinterpret_cast<OUT*>(a.out) + out_off;

        // trip count is uniform over the CTA (groups of one warp must stay converged for the shuffles)
        for (int rb = 0; rb < n_rows; rb += G * RPI) {
            const int r0 = rb + g;
            Acc<ELEM, METRIC> acc[RPI];
            const uint4* rp[RPI];
#pragma unroll
            for (int i = 0; i < RPI; ++i) {
                int r = r0 + i * G;
                // clamp so out-of-range lanes re-read a valid row (result discarded)
                if constexpr (GATHER)
                    rp[i] = reinterpret_cast<const uint4*>(a.rows + (size_t)ids[row_begin + min(r, n_rows - 1)] * a.stride);
                else
                    rp[i] = reinterpret_cast<const uint4*>(base + (size_t)min(r, n_rows - 1) * a.stride);
            }
            // register double buffering: the loads of step v + LPR are issued before the FMAs of step v,
            // so 2 * RPI independent 128-bit loads per thread stay in flight through the whole row set
            uint4 cur[RPI];
            if (l < V) {
#pragma unroll
                for (int i = 0; i < RPI; ++i) cur[i] = ldg_stream(rp[i] + l);
            }
#pragma unroll 2
            for (int v = l; v < V; v += LPR) {
                uint4 nxt[RPI];
                const int vn = v + LPR;
                if (vn < V) {
#pragma unroll
                    for (int i = 0; i < RPI; ++i) nxt[i] = ldg_stream(rp[i] + vn);
                }
#pragma unroll
                for (int i = 0; i < RPI; ++i) acc[i].add(cur[i], sq, v);
                if (vn < V) {
#pragma unroll
                    for (int i = 0; i < RPI; ++i) cur[i] = nxt[i];
                }
            }
#pragma unroll
            for (int i = 0; i < RPI; ++i) {
                acc[i].template reduce<LPR>();
                int r = r0 + i * G;
                if (l == 0 && r < n_rows) out[r] = (OUT)acc[i].value();
            }
        }
    }
}

template <int ELEM, int METRIC, int LPR, int RPI, typename OUT>
__global__ void __launch_bounds__(SCAN_THREADS) scan_kernel(ScanArgs a) {
    scan_body<ELEM, METRIC, LPR, RPI, OUT, false>(a, nullptr);
}

template <int ELEM, int METRIC, int LPR, int RPI>
__global__ void __launch_bounds__(SCAN_THREADS) scan_gather_kernel(ScanArgs a, const int64_t* __restrict__ ids) {
    scan_body<ELEM, METRIC, LPR, RPI, float, true>(a, ids);
}

// ----------------------------------------------------------------------------- dispatch

template <int ELEM, int METRIC, typename OUT, bool GATHER>
static int launch_scan_t(const ScanArgs& a, const int64_t* ids, int grid, cudaStream_t s) {
    size_t smem = a.qstride;
    int V = a.vec_per_row;
#define VB_LAUNCH(LPR, RPI)                                                                          \
    do {                                                                                             \
        if constexpr (GATHER) {                                                                      \
            auto kern = scan_gather_kernel<ELEM, METRIC, LPR, RPI>;                                  \
            if (smem > 48 * 1024) VB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); \
            kern<<<grid, SCAN_THREADS, smem, s>>>(a, ids);                                           \
        } else {                                                                                     \
            auto kern = scan_kernel<ELEM, METRIC, LPR, RPI, OUT>;                                    \
            if (smem > 48 * 1024) VB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); \
            kern<<<grid, SCAN_THREADS, smem, s>>>(a);                                                \
        }                                                                                            \
    } while (0)
    if (V >= 32) VB_LAUNCH(32, 4);
    else if (V >= 16) VB_LAUNCH(16, 4);
    else if (V >= 8) VB_LAUNCH(8, 4);
    else if (V >= 4) VB_LAUNCH(4, 8);
    else if (V >= 2) VB_LAUNCH(2, 8);
    else VB_LAUNCH(1, 8);
#undef VB_LAUNCH
    VB_CUDA(cudaGetLastError());
    count_launch();
    return VB_OK;
}

template <typename OUT, bool GATHER = false>
static int launch_scan_any(int elem, int metric, const ScanArgs& a, int grid, cudaStream_t s, const int64_t* ids = nullptr) {
    if (elem == VB_VECTOR) {
        switch (metric) {
            case VB_L2_SQUARED: return launch_scan_t<VB_VECTOR, VB_L2_SQUARED, OUT, GATHER>(a, ids, grid, s);
            case VB_NEG_IP: return launch_scan_t<VB_VECTOR, VB_NEG_IP, OUT, GATHER>(a, ids, grid, s);
            case VB_COSINE: return launch_scan_t<VB_VECTOR, VB_COSINE, OUT, GATHER>(a, ids, grid, s);
            case VB_L1: return launch_scan_t<VB_VECTOR, VB_L1, OUT, GATHER>(a, ids, grid, s);
        }
    } else if (elem == VB_HALFVEC) {
        switch (metric) {
            case VB_L2_SQUARED: return launch_scan_t<VB_HALFVEC, VB_L2_SQUARED, OUT, GATHER>(a, ids, grid, s);
            case VB_NEG_IP: return launch_scan_t<VB_HALFVEC, VB_NEG_IP, OUT, GATHER>(a, ids, grid, s);
            case VB_COSINE: return launch_scan_t<VB_HALFVEC, VB_COSINE, OUT, GATHER>(a, ids, grid, s);
            case VB_L1: return launch_scan_t<VB_HALFVEC, VB_L1, OUT, GATHER>(a, ids, grid, s);
        }
    } else {
        switch (metric) {
            case VB_HAMMING: return launch_scan_t<VB_BIT, VB_HAMMING, OUT, GATHER>(a, ids, grid, s);
            case VB_JACCARD: return launch_scan_t<VB_BIT, VB_JACCARD, OUT, GATHER>(a, ids, grid, s);
        }
    }
    set_error("unsupported metric %d for element type %d", metric, elem);
    return VB_EINVAL;
}

static int scan_rows_per_chunk(size_t stride) {
    // ~128 KB of rows per chunk, a multiple of 32 rows so every group slot is used
    int64_t r = (int64_t)(128 * 1024 / stride);
    r = (r / 32) * 32;
    if (r < 32) r = 32;
    if (r > 4096) r = 4096;
    return (int)r;
}

int scan_chunk_rows(const Table& t) { return scan_rows_per_chunk(t.stride); }

// Which scan kernel?  The bulk-copy (TMA) kernel streams HBM at low warp occupancy but, with one CTA per SM, is
// slower than the LDG kernel when the rows are L2-resident (a centre table read by many queries).
// scan_impl: 0 = always LDG, 1 = bulk whenever the shape allows, 2 (default) = bulk for tables larger than the
// H100's 50 MB L2.
static bool use_bulk_scan(const Table& t, int64_t n_rows, size_t qstride) {
    const int impl = ctx().scan_impl;
    if (impl == 0 || !scan_bulk_supported(t.elem, t.stride, qstride)) return false;
    if (impl == 1) return true;
    return (size_t)n_rows * t.stride > ((size_t)50 << 20);
}

static int scan_grid() {
    // persistent-style grid: a few CTAs per SM (multiple of the SM count)
    return ctx().sm_count * 8;
}

template <typename OUT>
static int scan_regular_impl(const Table& t, int metric, const void* q_dev, size_t qstride, int64_t nq,
                             int64_t n_rows, OUT* out, int64_t out_stride) {
    if (nq == 0 || n_rows == 0) return VB_OK;
    ScanArgs a{};
    a.rows = t.d;
    a.stride = t.stride;
    a.vec_per_row = (int)(t.stride / 16);
    a.queries = (const uint8_t*)q_dev;
    a.qstride = qstride;
    a.qvec = (int)(qstride / 16);
    a.chunks = nullptr;
    a.n_chunks_dev = nullptr;
    a.n_rows = n_rows;
    a.nq = nq;
    a.rows_per_chunk = scan_rows_per_chunk(t.stride);
    a.chunks_per_q = (n_rows + a.rows_per_chunk - 1) / a.rows_per_chunk;
    a.out_stride = out_stride;
    a.out = out;
    int64_t total = nq * a.chunks_per_q;
    if (use_bulk_scan(t, n_rows, qstride))
        return launch_scan_bulk(t.elem, metric, a, sizeof(OUT) == 8, (int)std::min<int64_t>(total, 1 << 30));
    int grid = (int)std::min<int64_t>(total, scan_grid());
    return launch_scan_any<OUT>(t.elem, metric, a, grid, ctx().stream);
}

int launch_scan_regular(const Table& t, int metric, const void* q_dev, size_t qstride, int64_t nq, int64_t n_rows,
                        float* out, int64_t out_stride) {
    return scan_regular_impl<float>(t, metric, q_dev, qstride, nq, n_rows, out, out_stride);
}
int launch_scan_regular_f64(const Table& t, int metric, const void* q_dev, size_t qstride, int64_t nq,
                            int64_t n_rows, double* out, int64_t out_stride) {
    return scan_regular_impl<double>(t, metric, q_dev, qstride, nq, n_rows, out, out_stride);
}

int launch_scan_chunks(const Table& t, int metric, const void* q_dev, size_t qstride, const Chunk* chunks_dev,
                       const int* n_chunks_dev, int max_chunks, float* out, bool ldg_only) {
    if (max_chunks <= 0) return VB_OK;
    ScanArgs a{};
    a.rows = t.d;
    a.stride = t.stride;
    a.vec_per_row = (int)(t.stride / 16);
    a.queries = (const uint8_t*)q_dev;
    a.qstride = qstride;
    a.qvec = (int)(qstride / 16);
    a.chunks = chunks_dev;
    a.n_chunks_dev = n_chunks_dev;
    a.out = out;
    if (!ldg_only && use_bulk_scan(t, t.n, qstride))
        return launch_scan_bulk(t.elem, metric, a, false, max_chunks);
    int grid = std::min(max_chunks, scan_grid());
    return launch_scan_any<float>(t.elem, metric, a, grid, ctx().stream);
}

int launch_scan_gather(const Table& t, int metric, const void* q_dev, size_t qstride, const int64_t* ids_dev,
                       const Chunk* chunks_dev, const int* n_chunks_dev, int max_chunks, float* out) {
    if (max_chunks <= 0) return VB_OK;
    ScanArgs a{};
    a.rows = t.d;
    a.stride = t.stride;
    a.vec_per_row = (int)(t.stride / 16);
    a.queries = (const uint8_t*)q_dev;
    a.qstride = qstride;
    a.qvec = (int)(qstride / 16);
    a.chunks = chunks_dev;
    a.n_chunks_dev = n_chunks_dev;
    a.out = out;
    int grid = std::min(max_chunks, scan_grid());
    return launch_scan_any<float, true>(t.elem, metric, a, grid, ctx().stream, ids_dev);
}

// ----------------------------------------------------------------------------- per-segment top-k

constexpr int TOPK_THREADS = 256;
constexpr int TOPK_MAX_K = 2048;

__device__ __forceinline__ uint64_t composite_key(float f, uint32_t pos) {
    return ((uint64_t)orderable_key(f) << 32) | pos;
}

// One CTA per segment.  Radix-select the k smallest composite keys (distance, position)
// -- all keys are distinct, so there is no tie handling -- then bitonic-sort them in smem.
// FLOOR (the paged selection of vb_ivf_iter.cu): only keys strictly above floor_key[seg] compete when returned[seg] > 0;
// keys are unique, so those are exactly the ones not returned yet, and successive pages concatenate to the full sort.
// Thread 0 then moves the floor to the last key selected, adds the page to returned[seg] and writes its size to count[seg].
template <bool FLOOR>
__device__ __forceinline__ void segment_topk_body(const float* __restrict__ keys, const int64_t* __restrict__ seg_begin,
                                                  const int32_t* __restrict__ seg_len, int k, int kpow2, int32_t* __restrict__ out_pos,
                                                  float* __restrict__ out_key, const int32_t* __restrict__ only_flagged,
                                                  uint64_t* __restrict__ floor_key, int32_t* __restrict__ returned,
                                                  int32_t* __restrict__ count) {
    extern __shared__ uint64_t sel[];  // kpow2 entries
    if (only_flagged != nullptr && only_flagged[blockIdx.x] == 0) return;   // (the slab selection's overflow path)
    __shared__ uint32_t hist[256];
    __shared__ uint64_t s_prefix, s_mask;
    __shared__ uint32_t s_kk, s_done, s_count;

    const int seg = blockIdx.x;
    const float* kp = keys + seg_begin[seg];
    const uint32_t n = (uint32_t)seg_len[seg];
    const int tid = threadIdx.x;
    uint32_t done = 0;   // keys returned by earlier pages (FLOOR)
    uint64_t fl = 0;
    if constexpr (FLOOR) {
        done = (uint32_t)returned[seg];
        fl = floor_key[seg];
    }
    const uint32_t rem = n - done;
    auto above = [&](uint64_t key) { return !FLOOR || done == 0 || key > fl; };

    uint64_t thresh = ~0ull;  // select keys <= thresh
    if (rem > (uint32_t)k) {
        if (tid == 0) {
            s_prefix = 0;
            s_mask = 0;
            s_kk = (uint32_t)k;
            s_done = 0;
        }
        __syncthreads();
        for (int pass = 7; pass >= 0; --pass) {
            hist[tid] = 0;
            __syncthreads();
            const int shift = pass * 8;
            const uint64_t prefix = s_prefix, mask = s_mask;
            // warp-aggregated histogram: candidate distances of one query share their leading bytes, so without
            // aggregation every thread of the CTA hammers the same shared-memory counter (measured: ~110 us per launch
            // for 2048 x 10 k keys, most of it serialised atomics)
            for (uint32_t base = 0; base < n; base += TOPK_THREADS) {
                const uint32_t i = base + tid;
                uint64_t key = 0;
                bool in = false;
                if (i < n) {
                    key = composite_key(kp[i], i);
                    in = (key & mask) == prefix && above(key);
                }
                const unsigned act = __ballot_sync(0xffffffffu, in);
                if (in) {
                    const uint32_t bin = (uint32_t)(key >> shift) & 255u;
                    const unsigned peers = __match_any_sync(act, bin);
                    if ((tid & 31) == (uint32_t)(__ffs(peers) - 1)) atomicAdd(&hist[bin], (uint32_t)__popc(peers));
                }
            }
            __syncthreads();
            if (tid == 0) {
                uint32_t kk = s_kk, cum = 0;
                int b = 0;
                for (; b < 256; ++b) {
                    if (cum + hist[b] >= kk) break;
                    cum += hist[b];
                }
                s_prefix = prefix | ((uint64_t)b << shift);
                s_mask = mask | (0xFFull << shift);
                s_kk = kk - cum;
                // the whole bin is taken: everything with this prefix is selected
                if (hist[b] == kk - cum) s_done = 1;
            }
            __syncthreads();
            if (s_done) {
                thresh = s_prefix | ((shift == 0) ? 0ull : ((1ull << shift) - 1ull));
                break;
            }
        }
        if (!s_done) thresh = s_prefix;
    }
    if (tid == 0) s_count = 0;
    for (int i = tid; i < kpow2; i += TOPK_THREADS) sel[i] = ~0ull;
    __syncthreads();
    for (uint32_t i = tid; i < n; i += TOPK_THREADS) {
        uint64_t key = composite_key(kp[i], i);
        if (key <= thresh && above(key)) {
            uint32_t slot = atomicAdd(&s_count, 1u);
            if (slot < (uint32_t)kpow2) sel[slot] = key;
        }
    }
    __syncthreads();
    // bitonic sort ascending
    for (int size = 2; size <= kpow2; size <<= 1) {
        for (int st = size >> 1; st > 0; st >>= 1) {
            for (int i = tid; i < kpow2; i += TOPK_THREADS) {
                int j = i ^ st;
                if (j > i) {
                    uint64_t x = sel[i], y = sel[j];
                    bool up = (i & size) == 0;
                    if ((x > y) == up) {
                        sel[i] = y;
                        sel[j] = x;
                    }
                }
            }
            __syncthreads();
        }
    }
    const uint32_t m = min(rem, (uint32_t)k);
    for (int i = tid; i < k; i += TOPK_THREADS) {
        if ((uint32_t)i < m) {
            uint64_t key = sel[i];
            out_pos[(int64_t)seg * k + i] = (int32_t)(uint32_t)key;
            out_key[(int64_t)seg * k + i] = key_to_float((uint32_t)(key >> 32));
        } else {
            out_pos[(int64_t)seg * k + i] = -1;
            out_key[(int64_t)seg * k + i] = __int_as_float(0x7F800000);
        }
    }
    if constexpr (FLOOR) {
        if (tid == 0) {
            if (m > 0) {
                floor_key[seg] = sel[m - 1];
                returned[seg] = (int32_t)(done + m);
            }
            count[seg] = (int32_t)m;
        }
    }
}

__global__ void __launch_bounds__(TOPK_THREADS) segment_topk_kernel(const float* __restrict__ keys,
                                                                    const int64_t* __restrict__ seg_begin,
                                                                    const int32_t* __restrict__ seg_len, int k,
                                                                    int kpow2, int32_t* __restrict__ out_pos,
                                                                    float* __restrict__ out_key,
                                                                    const int32_t* __restrict__ only_flagged) {
    segment_topk_body<false>(keys, seg_begin, seg_len, k, kpow2, out_pos, out_key, only_flagged, nullptr, nullptr, nullptr);
}

__global__ void __launch_bounds__(TOPK_THREADS) segment_topk_floor_kernel(const float* __restrict__ keys,
                                                                          const int64_t* __restrict__ seg_begin,
                                                                          const int32_t* __restrict__ seg_len, int k, int kpow2,
                                                                          int32_t* __restrict__ out_pos, float* __restrict__ out_key,
                                                                          uint64_t* __restrict__ floor_key,
                                                                          int32_t* __restrict__ returned, int32_t* __restrict__ count) {
    segment_topk_body<true>(keys, seg_begin, seg_len, k, kpow2, out_pos, out_key, nullptr, floor_key, returned, count);
}

int launch_segment_topk_floor(const float* keys, const int64_t* seg_begin_dev, const int32_t* seg_len_dev, int64_t nseg, int k,
                              uint64_t* floor_key, int32_t* returned, int32_t* count, int32_t* out_pos, float* out_key) {
    if (nseg == 0) return VB_OK;
    VB_REQUIRE(k >= 1 && k <= TOPK_MAX_K, "paged selection: page %d outside 1..%d", k, TOPK_MAX_K);
    int kpow2 = 2;
    while (kpow2 < k) kpow2 <<= 1;
    segment_topk_floor_kernel<<<(unsigned)nseg, TOPK_THREADS, (size_t)kpow2 * 8, ctx().stream>>>(keys, seg_begin_dev, seg_len_dev, k, kpow2,
                                                                                                 out_pos, out_key, floor_key, returned, count);
    VB_CUDA(cudaGetLastError());
    count_launch();
    return VB_OK;
}

// ---- the k' nearest of a candidate run from the slab minima of the tensor-core filter -------------------------------------
//
// The filter's epilogue stores, beside the dense d~ array, min d~ of every slab (32 table-aligned rows of one probed list,
// slab_base() in vb_common.cuh).  tau = the k'-th smallest slab minimum is an upper bound of the k'-th smallest d~ (k'
// distinct candidates are <= tau), so the k' nearest all lie in slabs whose minimum is <= tau: exactly k' slabs when the
// minima are distinct -- 32 k' candidates are read per query instead of the whole run (100 k at the headline shape, where
// the eight radix passes of segment_topk_kernel over 2048 such runs took 190 us).
// One CTA per query: (1) the run's slab minima into shared memory, (2) radix-select tau, (3) gather the candidates <= tau
// of the qualifying slabs, (4) sort by (d~, position), emit k'.  More candidates than the buffer holds (massive ties)
// flags the query for segment_topk_kernel.  Output: identical to segment_topk_kernel's.
__global__ void __launch_bounds__(SS_THREADS) slab_select_kernel(const float* __restrict__ dist, const float* __restrict__ smin, int probes,
                                                                 const int32_t* __restrict__ probe_lists,
                                                                 const int32_t* __restrict__ cand_off, const int64_t* __restrict__ list_off,
                                                                 int64_t cap, int64_t cap_s, int n_slab_max, int k,
                                                                 int32_t* __restrict__ out_pos, float* __restrict__ out_key,
                                                                 int32_t* __restrict__ flagged) {
    extern __shared__ uint64_t ss_smem[];
    uint64_t* cand = ss_smem;                                             // [SS_CAND], then the selection's work area
    const int q = blockIdx.x;
    const int tid = threadIdx.x;
    const int n = slab_select_cta(dist, smin, probes, probe_lists, cand_off, list_off, cap, cap_s, q, k, cand, cand + SS_CAND);
    if (tid == 0) flagged[q] = n < 0 ? 1 : 0;
    if (n < 0) return;
    for (int i = tid; i < k; i += SS_THREADS) {
        if (i < n) {
            const uint64_t key = cand[i];
            out_pos[(int64_t)q * k + i] = (int32_t)(uint32_t)key;
            out_key[(int64_t)q * k + i] = key_to_float((uint32_t)(key >> 32));
        } else {
            out_pos[(int64_t)q * k + i] = -1;
            out_key[(int64_t)q * k + i] = __int_as_float(0x7F800000);
        }
    }
}

int launch_slab_select(const float* dist, const float* smin, int64_t nq, int probes, const int32_t* probe_lists, const int32_t* cand_off,
                       const int64_t* list_off, int64_t cap, int64_t cap_s, const int64_t* seg_begin, const int32_t* seg_len, int kp,
                       int32_t* out_pos, float* out_key) {
    Scratch sc;
    if (nq == 0) return VB_OK;
    cudaStream_t s = ctx().stream;
    VB_REQUIRE(kp <= TOPK_MAX_K, "slab selection: k' too large");
    void* d_flag;
    VB_TRY(sc.take(sizeof(int32_t) * (size_t)nq, &d_flag));
    const size_t smem = slab_select_launch_smem(cap_s, probes);
    VB_REQUIRE(smem <= SS_SMEM_MAX, "slab selection: %zu bytes of shared memory", smem);
    static size_t attr = 0;
    if (smem > 48 * 1024 && smem > attr) {
        VB_CUDA(cudaFuncSetAttribute(slab_select_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        attr = smem;
    }
    slab_select_kernel<<<(unsigned)nq, SS_THREADS, smem, s>>>(dist, smin, probes, probe_lists, cand_off, list_off, cap, cap_s, (int)cap_s, kp,
                                                            out_pos, out_key, (int32_t*)d_flag);
    // queries whose candidates did not fit (ties by the thousand) take the full selection
    int kpow2 = 2;
    while (kpow2 < kp) kpow2 <<= 1;
    segment_topk_kernel<<<(unsigned)nq, TOPK_THREADS, (size_t)kpow2 * 8, s>>>(dist, seg_begin, seg_len, kp, kpow2, out_pos, out_key,
                                                                            (const int32_t*)d_flag);
    VB_CUDA(cudaGetLastError());
    count_launch(2);
    return VB_OK;
}

// --- large k / "sort everything": composite keys + CUB segmented radix sort (not the hot path:
//     the keys are 0.07 % of the bytes the scan kernel streams)
__global__ void build_composite_kernel(const float* __restrict__ keys, const int64_t* __restrict__ seg_begin,
                                       const int32_t* __restrict__ seg_len, const int64_t* __restrict__ dst_off,
                                       uint64_t* __restrict__ out) {
    const int seg = blockIdx.y;
    const int32_t n = seg_len[seg];
    const float* kp = keys + seg_begin[seg];
    uint64_t* op = out + dst_off[seg];
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x)
        op[i] = composite_key(kp[i], (uint32_t)i);
}

__global__ void emit_sorted_kernel(const uint64_t* __restrict__ sorted, const int64_t* __restrict__ dst_off,
                                   const int32_t* __restrict__ seg_len, int k, int32_t* __restrict__ out_pos,
                                   float* __restrict__ out_key) {
    const int seg = blockIdx.y;
    const int32_t n = seg_len[seg];
    const uint64_t* sp = sorted + dst_off[seg];
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < k; i += gridDim.x * blockDim.x) {
        if (i < n) {
            uint64_t key = sp[i];
            out_pos[(int64_t)seg * k + i] = (int32_t)(uint32_t)key;
            out_key[(int64_t)seg * k + i] = key_to_float((uint32_t)(key >> 32));
        } else {
            out_pos[(int64_t)seg * k + i] = -1;
            out_key[(int64_t)seg * k + i] = __int_as_float(0x7F800000);
        }
    }
}

int launch_segment_topk_v(const float* keys, const int64_t* seg_begin_dev, const int32_t* seg_len_dev,
                          const int64_t* seg_begin_host, const int32_t* seg_len_host, int64_t nseg, int k,
                          int32_t* out_pos, float* out_key) {
    Scratch sc;
    if (nseg == 0 || k <= 0) return VB_OK;
    cudaStream_t s = ctx().stream;
    if (k <= TOPK_MAX_K) {
        int kpow2 = 2;
        while (kpow2 < k) kpow2 <<= 1;
        segment_topk_kernel<<<(unsigned)nseg, TOPK_THREADS, (size_t)kpow2 * 8, s>>>(keys, seg_begin_dev, seg_len_dev, k,
                                                                                 kpow2, out_pos, out_key, nullptr);
        VB_CUDA(cudaGetLastError());
        count_launch();
        return VB_OK;
    }
    // full segmented sort; needs host-side segment sizes to lay out a compact buffer
    if (!seg_len_host || !seg_begin_host) {
        set_error("k > %d needs host-visible segment sizes", TOPK_MAX_K);
        return VB_EINVAL;
    }
    std::string tmp;
    int64_t total = 0;
    std::vector<int64_t> off((size_t)nseg + 1);
    for (int64_t i = 0; i < nseg; ++i) {
        off[(size_t)i] = total;
        total += seg_len_host[i];
    }
    off[(size_t)nseg] = total;
    void *d_off, *d_in, *d_out, *d_tmp;
    VB_TRY(sc.take(sizeof(int64_t) * ((size_t)nseg + 1), &d_off));
    VB_TRY(sc.take(sizeof(uint64_t) * (size_t)std::max<int64_t>(total, 1), &d_in));
    VB_TRY(sc.take(sizeof(uint64_t) * (size_t)std::max<int64_t>(total, 1), &d_out));
    VB_CUDA(cudaMemcpyAsync(d_off, off.data(), sizeof(int64_t) * ((size_t)nseg + 1), cudaMemcpyHostToDevice, s));
    VB_CUDA(cudaStreamSynchronize(s));  // off is a stack-owned vector
    int32_t maxlen = 0;
    for (int64_t i = 0; i < nseg; ++i) maxlen = std::max(maxlen, seg_len_host[i]);
    if (total > 0) {
        dim3 grid((unsigned)std::min<int64_t>((maxlen + 255) / 256, 1024), (unsigned)nseg);
        build_composite_kernel<<<grid, 256, 0, s>>>(keys, seg_begin_dev, seg_len_dev, (const int64_t*)d_off, (uint64_t*)d_in);
        VB_CUDA(cudaGetLastError());
        count_launch();
        size_t tmp_bytes = 0;
        VB_CUDA(cub::DeviceSegmentedRadixSort::SortKeys(nullptr, tmp_bytes, (const uint64_t*)d_in, (uint64_t*)d_out,
                                                        (int)total, (int)nseg, (const int64_t*)d_off,
                                                        (const int64_t*)d_off + 1, 0, 64, s));
        VB_TRY(sc.take(tmp_bytes, &d_tmp));
        VB_CUDA(cub::DeviceSegmentedRadixSort::SortKeys(d_tmp, tmp_bytes, (const uint64_t*)d_in, (uint64_t*)d_out,
                                                        (int)total, (int)nseg, (const int64_t*)d_off,
                                                        (const int64_t*)d_off + 1, 0, 64, s));
        count_launch(2);
    }
    dim3 grid2((unsigned)std::min<int64_t>(((int64_t)k + 255) / 256, 1024), (unsigned)nseg);
    emit_sorted_kernel<<<grid2, 256, 0, s>>>((const uint64_t*)d_out, (const int64_t*)d_off, seg_len_dev, k, out_pos, out_key);
    VB_CUDA(cudaGetLastError());
    count_launch();
    return VB_OK;
}

}  // namespace vb
