// vb_ivf.cu -- C ABI for the batched distance operator, resident tables, exact
// top-k and the IVFFlat scan path (GetScanLists + GetScanItems, src/ivfscan.c:47-187).
#include "vb_common.cuh"
#include "vb_distance.cuh"
#include "vb_slab_select.cuh"

#include <algorithm>
#include <cmath>
#include <cstring>
#include <functional>
#include <numeric>
#include <vector>

namespace vb {

__global__ void regular_segments_kernel(int64_t nseg, int64_t stride, int32_t len, int64_t* begin, int32_t* lens) {
    int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i < nseg) {
        begin[i] = i * stride;
        lens[i] = len;
    }
}

__global__ void finish_exact_kernel(int metric, int64_t n, const int32_t* __restrict__ pos, const float* __restrict__ key,
                                    int64_t* __restrict__ out_ids, float* __restrict__ out_f, double* __restrict__ out_d) {
    int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= n) return;
    out_ids[i] = pos[i];
    double v = finish_value(metric, key[i]);
    if (out_f) out_f[i] = (float)v;
    if (out_d) out_d[i] = v;
}

// ----------------------------------------------------------------------------- IVFFlat device image

struct Ivf {
    int elem, metric, dim, lists;
    Table centers;
    Table rows;
    int64_t* d_ids = nullptr;
    int64_t* d_list_off = nullptr;
    std::vector<int64_t> h_list_off;
    std::vector<int64_t> sorted_len;  // list lengths, descending (bounds candidates per query)
    int64_t last_bytes = 0, last_cand = 0;
    int64_t* d_cand_sum = nullptr;    // device accumulator of candidates scanned (allocated and zeroed with the image)
    ListTile* d_tiles = nullptr;      // static row tiles of the lists (list-major batched scan)
    int n_tiles = 0;
    ListTcImage tc;                   // packed bf16 planes + norms + (list, tile) units, built on first tensor-core scan
    ListTcImage ctc;                  // the same for the centre table (one pseudo list probed by every query)
    int64_t* d_centre_off = nullptr;  // {0, lists}
    cudaStream_t q_stream = nullptr;  // copy stream of the pipelined host path (vb_ivf_prefetch_queries)
    cudaEvent_t q_ready[2] = {nullptr, nullptr};
    void* q_buf[2] = {nullptr, nullptr};
    size_t q_bytes[2] = {0, 0};
    int64_t q_nq[2] = {0, 0};
    unsigned* d_ticket = nullptr;     // 2 x ONE_MAX_Q arrival counters of the fused one-query kernels (zero between launches)
    int* d_tc_fail = nullptr;         // device counters of uncertified queries: [0] probe selection, [1] list scan (ivf_tc_fail_zero)
    int l1_cooldown = 0;              // batches left before level 1 is tried again after it failed
    int l0_cooldown = 0;              // the same for level 0 (after a batch where it failed often)
    int lp_cooldown = 0;              // the same for level P
    ListProj lp;                      // level P's basis and projected rows, built with level 0's image (vb_list_proj.cu)
    int32_t* d_l0_fail = nullptr;     // the queries level 0 could not certify ([d_tc_fail[1]] of them)
    int64_t l0_fail_cap = 0;
    void* d_repair[2] = {nullptr, nullptr};   // gathered queries and results of their re-run (device queries / results), by the
    size_t repair_bytes[2] = {0, 0};          // level it starts at (0: after level P; 1: after level 0, which a re-run from 0 may need)
    int64_t total_tc_failed = 0, total_l1_failed = 0, total_l0_failed = 0, total_lp_failed = 0;
    bool loaded = false;
    uint64_t generation = 0;          // bumped whenever rows or lists change: an iterative scan handle refuses a changed image
    bool has_ids = false;             // loaded with heap ids (vb_ivf_insert / vb_ivf_delete need them)
    int64_t ids_cap = -1;             // rows d_ids holds (-1: exactly rows.n, as a load allocates it)
    int64_t tc_cap_tiles = 0;         // tiles the plane buffers of tc hold (bf16 planes + xn; int8 plane + xs + r8)
    int64_t tc_cap_tiles8 = 0;
    // streaming load (vb_ivf_begin_load / vb_ivf_load_list / vb_ivf_end_load)
    bool loading = false;
    int next_list = 0;
    std::vector<int64_t> h_ids;
    std::vector<int64_t> pending_off;
};

// One CTA per query: candidate offsets of its probed lists and the chunk descriptors of the scan.
__global__ void __launch_bounds__(128) ivf_build_chunks_kernel(const int32_t* __restrict__ probe_lists, int probes,
                                                               const int64_t* __restrict__ list_off, int rows_per_chunk,
                                                               int64_t cap, int32_t* __restrict__ cand_off /*[nq][probes+1]*/,
                                                               int64_t* __restrict__ seg_begin, int32_t* __restrict__ seg_len,
                                                               Chunk* __restrict__ chunks, int* __restrict__ n_chunks,
                                                               int64_t* __restrict__ cand_sum, const int32_t* __restrict__ active) {
    const int q = blockIdx.x;
    // (an iterative scan rebuilds only the queries that moved to a new group; the others keep their runs)
    if (active != nullptr && active[q] == 0) return;
    const int32_t* pl = probe_lists + (int64_t)q * probes;
    int32_t* co = cand_off + (int64_t)q * (probes + 1);
    __shared__ int s_base;
    if (threadIdx.x == 0) {
        int32_t off = 0;
        int nch = 0;
        for (int p = 0; p < probes; ++p) {
            co[p] = off;
            int l = pl[p];
            int32_t len = l >= 0 ? (int32_t)(list_off[l + 1] - list_off[l]) : 0;
            off += len;
            nch += (len + rows_per_chunk - 1) / rows_per_chunk;
        }
        co[probes] = off;
        seg_begin[q] = (int64_t)q * cap;
        seg_len[q] = off;
        s_base = chunks ? atomicAdd(n_chunks, nch) : 0;
        atomicAdd((unsigned long long*)cand_sum, (unsigned long long)off);
    }
    __syncthreads();
    if (chunks == nullptr) return;   // the list-major kernels take the probe lists directly: no descriptors needed
    // emit descriptors; per-probe chunk base via a serial prefix held by each thread (probes is small)
    int base = s_base;
    for (int p = 0; p < probes; ++p) {
        int l = pl[p];
        if (l < 0) continue;
        int64_t lo = list_off[l];
        int32_t len = (int32_t)(list_off[l + 1] - lo);
        int nch = (len + rows_per_chunk - 1) / rows_per_chunk;
        for (int c = threadIdx.x; c < nch; c += blockDim.x) {
            Chunk ch;
            ch.row_begin = lo + (int64_t)c * rows_per_chunk;
            ch.n_rows = min(rows_per_chunk, len - c * rows_per_chunk);
            ch.q = q;
            ch.out_off = (int64_t)q * cap + co[p] + (int64_t)c * rows_per_chunk;
            chunks[base + c] = ch;
        }
        base += nch;
    }
}

// winners (position within the query's candidate run) -> heap ids and float8 distances
__global__ void ivf_finish_kernel(int metric, int64_t nq, int k, int probes, const int32_t* __restrict__ pos,
                                  const float* __restrict__ key, const int32_t* __restrict__ probe_lists,
                                  const int32_t* __restrict__ cand_off, const int64_t* __restrict__ list_off,
                                  const int64_t* __restrict__ ids, int64_t* __restrict__ out_ids,
                                  float* __restrict__ out_f, double* __restrict__ out_d) {
    int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= nq * k) return;
    int64_t q = i / k;
    int32_t ps = pos[i];
    int64_t id = -1;
    const int32_t* co = cand_off + q * (probes + 1);
    // (a query the tensor-core filter could not select or certify leaves its slots unwritten -- the batch is repeated --
    // so a position is only trusted inside the query's candidate run)
    if (ps >= 0 && ps < co[probes]) {
        int lo = 0, hi = probes;  // largest p with co[p] <= ps
        while (hi - lo > 1) {
            int mid = (lo + hi) >> 1;
            if (co[mid] <= ps) lo = mid;
            else hi = mid;
        }
        // skip empty lists that share the same offset
        while (lo + 1 < probes && co[lo + 1] <= ps) ++lo;
        int l = probe_lists[q * probes + lo];
        int64_t row = list_off[l] + (ps - co[lo]);
        id = ids ? ids[row] : row;
    }
    out_ids[i] = id;
    double v = finish_value(metric, key[i]);
    if (out_f) out_f[i] = (float)v;
    if (out_d) out_d[i] = v;
}

// ----------------------------------------------------------------------------- row filters of the batched search
//
// vb_ivf_search_filtered scans the probed lists whole, as vb_ivf_search does, and masks each query's run of candidate
// distances before anything selects from it: ivf_mask_kernel rewrites every entry whose row the query's filter rejects
// to FILTER_REJECTED and recomputes the slab minima over the allowed entries.  Every selection then sees the allowed
// entries first, in their unfiltered order; ivf_unmask_kernel turns a rejected entry that reached the top k into -1 / +inf.

struct MaskFilter {        // one row filter as the mask reads it (vb_filter.cu): sorted image rows, per-list runs
    const int64_t* pos;
    const int64_t* off;
};
struct IvfMask {           // the device arguments of one sub-batch
    const MaskFilter* filters;   // [nfilters]
    const int32_t* fq;           // [nq] filter of each query (nullptr: filters[0] for all)
    int32_t* has_nan;            // [nq] set when an allowed entry of the query's run is NaN
};

// One CTA per (query, probe) pair, one warp per 32-row slab of the list at a time: the slab's allowed rows are the
// filter's positions from a binary search for the slab's first row on (at most 32 of them, one per lane).
__global__ void __launch_bounds__(256) ivf_mask_kernel(IvfMask mk, int probes, const int32_t* __restrict__ probe_lists,
                                                       const int32_t* __restrict__ cand_off, const int64_t* __restrict__ list_off,
                                                       int64_t cap, float* __restrict__ dist, float* __restrict__ smin, int64_t cap_s) {
    const int64_t q = blockIdx.x / probes;
    const int p = (int)(blockIdx.x % probes);
    const int l = probe_lists[q * probes + p];
    if (l < 0) return;
    const int64_t lo = list_off[l], hi = list_off[l + 1];
    if (hi <= lo) return;
    const MaskFilter f = mk.filters[mk.fq ? mk.fq[q] : 0];
    const int64_t a0 = f.off[l], a1 = f.off[l + 1];
    const int32_t co = cand_off[q * (probes + 1) + p];
    float* dq = dist + q * cap + co - lo;   // dq[r]: row r of the list-ordered table
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int64_t s0 = lo >> 5, ns = ((hi - 1) >> 5) - s0 + 1;
    bool nan_seen = false;
    for (int64_t s = warp; s < ns; s += 8) {
        const int64_t r0 = (s0 + s) << 5;
        int64_t j = a0;
        if (lane == 0) {
            int64_t b = a1;   // first allowed position >= r0
            while (j < b) {
                const int64_t mid = (j + b) >> 1;
                if (f.pos[mid] < r0) j = mid + 1;
                else b = mid;
            }
        }
        j = __shfl_sync(0xffffffffu, j, 0);
        const int64_t pr = j + lane < a1 ? f.pos[j + lane] : INT64_MAX;
        const unsigned allowed = __reduce_or_sync(0xffffffffu, pr < r0 + 32 ? 1u << (unsigned)(pr - r0) : 0u);
        const int64_t r = r0 + lane;
        uint32_t key = 0xFFFFFFFFu;
        if (r >= lo && r < hi) {
            float d = __uint_as_float(FILTER_REJECTED);
            if ((allowed >> lane) & 1u) {
                d = dq[r];
                if (d != d) {
                    nan_seen = true;
                    d = __uint_as_float(0x7FFFFFFFu);
                }
            }
            dq[r] = d;
            key = orderable_key(d);
        }
        key = __reduce_min_sync(0xffffffffu, key);
        if (smin != nullptr && lane == 0) smin[slab_base(q, cap_s, co, p) + s] = key == 0xFFFFFFFFu ? __uint_as_float(FILTER_REJECTED) : key_to_float(key);
    }
    if (nan_seen) mk.has_nan[q] = 1;
}

// After ivf_finish_kernel on a masked run.  One warp per query.  Without an allowed NaN, rejected entries sort after every
// allowed one: a selected rejected entry becomes -1 / +inf.  With one, rejected and allowed NaN entries share the key of
// NaN and are ordered by position, so the NaN tail of the result (slot f on) is rebuilt: the allowed NaN entries of the
// run in scan order, then -1 / +inf.
__global__ void ivf_unmask_kernel(int metric, int64_t nq, int k, int probes, const int32_t* __restrict__ pos, const float* __restrict__ key,
                                  const float* __restrict__ dist, int64_t cap, const int32_t* __restrict__ has_nan,
                                  const int32_t* __restrict__ probe_lists, const int32_t* __restrict__ cand_off,
                                  const int64_t* __restrict__ list_off, const int64_t* __restrict__ ids, int64_t* __restrict__ out_ids,
                                  float* __restrict__ out_f, double* __restrict__ out_d) {
    const int64_t q = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (q >= nq) return;   // whole warps
    const float* dq = dist + q * cap;
    const double pad = finish_value(metric, __int_as_float(0x7F800000));
    auto clear = [&](int64_t i) {
        out_ids[i] = -1;
        if (out_f) out_f[i] = (float)pad;
        if (out_d) out_d[i] = pad;
    };
    if (has_nan[q] == 0) {
        for (int i = lane; i < k; i += 32) {
            const int32_t ps = pos[q * k + i];
            if (ps >= 0 && __float_as_uint(dq[ps]) == FILTER_REJECTED) clear(q * k + i);
        }
        return;
    }
    int f = k;   // the first slot holding padding or a NaN key
    for (int i0 = 0; i0 < k && f == k; i0 += 32) {
        const int i = i0 + lane;
        const unsigned b = __ballot_sync(0xffffffffu, i < k && (pos[q * k + i] < 0 || key[q * k + i] != key[q * k + i]));
        if (b) f = i0 + __ffs(b) - 1;
    }
    const int32_t* co = cand_off + q * (probes + 1);
    const double vnan = finish_value(metric, __int_as_float(0x7FC00000));
    for (int p = 0; p < probes && f < k; ++p) {
        const int l = probe_lists[q * probes + p];
        if (l < 0) continue;
        const int64_t lo = list_off[l];
        for (int32_t c = co[p]; c < co[p + 1] && f < k; c += 32) {
            const int32_t ps = c + lane;
            const float d = ps < co[p + 1] ? dq[ps] : 0.f;
            const bool take = d != d && __float_as_uint(d) != FILTER_REJECTED;
            const unsigned b = __ballot_sync(0xffffffffu, take);
            const int slot = f + __popc(b & ((1u << lane) - 1u));
            if (take && slot < k) {
                const int64_t row = lo + (ps - co[p]);
                out_ids[q * k + slot] = ids ? ids[row] : row;
                if (out_f) out_f[q * k + slot] = (float)vnan;
                if (out_d) out_d[q * k + slot] = vnan;
            }
            f += __popc(b);
        }
    }
    for (int i = f + lane; i < k; i += 32) clear(q * k + i);
}

static int ivf_mask_runs(const IvfMask& mk, int64_t nq, const int32_t* d_lists, int probes, const int32_t* cand_off, const int64_t* list_off,
                         int64_t cap, float* dist, float* smin, int64_t cap_s) {
    Context& c = ctx();
    prof_begin(VB_PROF_FILTER_MASK);
    VB_CUDA(cudaMemsetAsync(mk.has_nan, 0, sizeof(int32_t) * (size_t)nq, c.stream));
    ivf_mask_kernel<<<(unsigned)(nq * probes), 256, 0, c.stream>>>(mk, probes, d_lists, cand_off, list_off, cap, dist, smin, cap_s);
    VB_CUDA(cudaGetLastError());
    count_launch();
    prof_end(VB_PROF_FILTER_MASK);
    return VB_OK;
}

static int ivf_unmask(const Ivf& ix, const IvfMask& mk, int64_t nq, int k, int probes, const int32_t* pos, const float* key, const float* dist,
                      int64_t cap, const int32_t* d_lists, const int32_t* cand_off, int64_t* out_ids, float* out_f, double* out_d) {
    Context& c = ctx();
    ivf_unmask_kernel<<<(unsigned)((nq * 32 + 255) / 256), 256, 0, c.stream>>>(ix.metric, nq, k, probes, pos, key, dist, cap, mk.has_nan, d_lists,
                                                                             cand_off, ix.d_list_off, ix.d_ids, out_ids, out_f, out_d);
    VB_CUDA(cudaGetLastError());
    count_launch();
    return VB_OK;
}

static int64_t ivf_cap(const Ivf& ix, int probes) {
    int64_t cap = 0;
    for (int i = 0; i < probes && i < (int)ix.sorted_len.size(); ++i) cap += ix.sorted_len[(size_t)i];
    return std::max<int64_t>(cap, 1);
}

// every query "probes" pseudo list 0 = the whole centre table: probe_lists[q] = 0, cand_off[q] = {0, lists}
__global__ void centre_pairs_kernel(int64_t nq, int32_t lists, int32_t* __restrict__ probe_lists, int32_t* __restrict__ cand_off) {
    const int64_t q = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (q >= nq) return;
    probe_lists[q] = 0;
    cand_off[2 * q] = 0;
    cand_off[2 * q + 1] = lists;
}

static int ivf_ensure_centre_tc(Ivf& ix) {
    if (ix.ctc.planes || !ix.ctc.finite) return VB_OK;
    VB_TRY(list_tc_prepare(ix.centers, &ix.ctc));
    std::vector<ListUnit> units;
    for (int64_t t = 0; t * 128 < ix.lists; ++t) units.push_back(ListUnit{0, (int32_t)t});
    ix.ctc.n_units = (int)units.size();
    VB_CUDA(cudaMalloc(&ix.ctc.units, sizeof(ListUnit) * units.size()));
    VB_CUDA(cudaMemcpy(ix.ctc.units, units.data(), sizeof(ListUnit) * units.size(), cudaMemcpyHostToDevice));
    if (!ix.d_centre_off) VB_CUDA(cudaMalloc(&ix.d_centre_off, 2 * sizeof(int64_t)));
    const int64_t off[2] = {0, ix.lists};
    VB_CUDA(cudaMemcpy(ix.d_centre_off, off, sizeof(off), cudaMemcpyHostToDevice));
    return VB_OK;
}

// What one pass of probe selection and list scan may do.  A default-constructed pass is a plain one: the filter level is
// chosen automatically (never level 0), and each tensor-core certificate is read back by the pass itself.
struct IvfPass {
    enum Mode { AUTO, LEVEL2, EXACT };
    Mode mode = AUTO;           // LEVEL2: the repeat of a batch whose level-1 certificate failed; EXACT: no tensor-core filter
    bool defer_check = false;   // the caller reads the certificate counters (d_tc_fail) at its own synchronisation
    bool level0 = false;        // the list scan may start at level 0: the caller runs the queries it cannot certify again
    bool levelp = false;        // ... and at level P in front of it (the caller runs those queries again from level 0)
    bool repair = false;        // that re-run: it takes the batched filter chain whatever its size
};
constexpr int IVF_LEVEL_EXACT = -1;   // list level of a scan that ran on the exact kernels

// zero the certificate counters, allocating them first.  They are allocated by the first pass that needs them: until then
// the batched search neither clears nor reads them back.
static int ivf_tc_fail_zero(Ivf& ix) {
    if (!ix.d_tc_fail) VB_CUDA(cudaMalloc(&ix.d_tc_fail, 2 * sizeof(int)));
    VB_CUDA(cudaMemsetAsync(ix.d_tc_fail, 0, 2 * sizeof(int), ctx().stream));
    return VB_OK;
}

// probe selection for a batch of query images: d_probe_lists [nq x probes] ascending by (distance, list), in sc.  *qn: the
// batch's |q|^2 (list_tc_query_norms), computed here where the tensor-core filter first needs it
static int ivf_select_probes(Scratch& sc, Ivf& ix, const IvfPass& pass, const void* qimg, size_t qstride, int64_t nq, float** qn, int probes,
                             int32_t** d_lists, float** d_ldist) {
    Context& c = ctx();
    void *d_cdist, *d_seg, *d_probe;
    VB_TRY(sc.take(sizeof(float) * (size_t)nq * ix.lists, &d_cdist));
    // Query batches: the same tensor-core filter as the list scan, with the centre table as ONE list probed by every
    // query -- approximate distances to all centres, the k' nearest re-scored exactly, order (distance, list number)
    // certified; any uncertified query sends the batch through the exact tiles below.
    const int km = key_metric(ix.metric);
    bool tc = (c.scan_impl == 2 || c.scan_impl == 4) && pass.mode != IvfPass::EXACT && nq >= 256 && ix.lists >= 128 &&
              list_tc_supported(ix.elem, km, probes);
    if (tc) {
        VB_TRY(ivf_ensure_centre_tc(ix));
        tc = ix.ctc.finite && ix.ctc.planes != nullptr;
    }
    if (tc && !ix.d_tc_fail) VB_TRY(ivf_tc_fail_zero(ix));
    if (tc) {
        const int kp = list_tc_kp(probes);
        void *d_pairs, *d_seg2, *d_probe2;
        VB_TRY(sc.take(sizeof(int32_t) * (size_t)nq * 3 + 64, &d_pairs));
        int32_t* zero_lists = (int32_t*)d_pairs;
        int32_t* pair_off = zero_lists + nq;
        VB_TRY(sc.take((sizeof(int64_t) + sizeof(int32_t)) * (size_t)nq * 2 + 64, &d_seg2));
        int64_t* sb = (int64_t*)d_seg2;
        int32_t* sl = (int32_t*)(sb + nq);
        VB_TRY(sc.take((sizeof(int32_t) + sizeof(float)) * (size_t)nq * (probes + kp), &d_probe2));
        int32_t* lists = (int32_t*)d_probe2;
        float* ldist = (float*)(lists + (size_t)nq * probes);
        int32_t* pos_kp = (int32_t*)(ldist + (size_t)nq * probes);
        float* key_kp = (float*)(pos_kp + (size_t)nq * kp);
        prof_begin(VB_PROF_SCAN_LISTS);
        centre_pairs_kernel<<<(unsigned)((nq + 255) / 256), 256, 0, c.stream>>>(nq, ix.lists, zero_lists, pair_off);
        regular_segments_kernel<<<(unsigned)((nq + 255) / 256), 256, 0, c.stream>>>(nq, ix.lists, ix.lists, sb, sl);
        VB_CUDA(cudaGetLastError());
        count_launch(2);
        if (!*qn) VB_TRY(list_tc_query_norms(sc, qimg, qstride, nq, qn));
        VB_TRY(launch_list_tc(ix.centers, ix.ctc, km, qimg, qstride, nq, zero_lists, 1, pair_off, ix.lists, ix.d_centre_off, 1,
                              (float*)d_cdist, *qn, true));
        int n_failed = 0;
        if (!pass.defer_check) VB_CUDA(cudaMemsetAsync(ix.d_tc_fail, 0, sizeof(int), c.stream));
        // a run of at most CR_RUN_MAX centre distances is selected inside the refine kernel, a longer one by a launch of its own
        const bool pre = ix.lists > CR_RUN_MAX;
        if (pre) VB_TRY(launch_segment_topk_v((const float*)d_cdist, sb, sl, nullptr, nullptr, nq, kp, pos_kp, key_kp));
        VB_TRY(launch_list_tc_cta_refine(ix.centers, ix.ctc, km, qimg, qstride, nq, probes, kp, 1, zero_lists, pair_off, ix.d_centre_off,
                                         (const float*)d_cdist, nullptr, pre ? pos_kp : nullptr, pre ? key_kp : nullptr, ix.lists, 0, sl,
                                         *qn, lists, ldist, ix.d_tc_fail, 2));
        if (!pass.defer_check) {
            VB_CUDA(cudaMemcpyAsync(&n_failed, ix.d_tc_fail, sizeof(int), cudaMemcpyDeviceToHost, c.stream));
            VB_CUDA(cudaStreamSynchronize(c.stream));
        }
        prof_end(VB_PROF_SCAN_LISTS);
        ix.total_tc_failed += n_failed;
        if (n_failed == 0) {   // (deferred: optimistic, the caller checks the counter with its own synchronisation)
            *d_lists = lists;
            *d_ldist = ldist;
            return VB_OK;
        }
    }
    prof_begin(VB_PROF_SCAN_LISTS);
    // many queries at once: the query image is itself a row table with the centres' stride (vector, bit), so the
    // centre scan is computed tile-wise (both operands staged once per 128 x 128 tile) instead of one-query-at-a-time
    // scans that re-read the L2-resident centre table per query.
    const bool tiled = nq >= 64 && ix.elem != VB_HALFVEC && qstride == ix.centers.stride && ctx().scan_impl != 0 &&
                       (key_metric(ix.metric) == VB_L2_SQUARED || key_metric(ix.metric) == VB_NEG_IP || key_metric(ix.metric) == VB_HAMMING);
    if (tiled) {
        Table Q;
        Q.elem = ix.elem;
        Q.dim = ix.dim;
        Q.stride = qstride;
        Q.n = nq;
        Q.d = (uint8_t*)const_cast<void*>(qimg);
        VB_TRY(launch_distance_matrix(Q, ix.metric, ix.centers, ix.lists, (float*)d_cdist, ix.lists));
    } else {
        VB_TRY(launch_scan_regular(ix.centers, key_metric(ix.metric), qimg, qstride, nq, ix.lists, (float*)d_cdist, ix.lists));
    }
    prof_end(VB_PROF_SCAN_LISTS);
    VB_TRY(sc.take((sizeof(int64_t) + sizeof(int32_t)) * (size_t)nq * 2 + 64, &d_seg));
    int64_t* seg_begin = (int64_t*)d_seg;
    int32_t* seg_len = (int32_t*)(seg_begin + nq);
    regular_segments_kernel<<<(unsigned)((nq + 255) / 256), 256, 0, c.stream>>>(nq, ix.lists, ix.lists, seg_begin, seg_len);
    VB_CUDA(cudaGetLastError());
    count_launch();
    VB_TRY(sc.take((sizeof(int32_t) + sizeof(float)) * (size_t)nq * probes, &d_probe));
    int32_t* lists = (int32_t*)d_probe;
    float* ldist = (float*)(lists + (size_t)nq * probes);
    std::vector<int64_t> hb;
    std::vector<int32_t> hl;
    if (probes > 2048) {
        hb.resize((size_t)nq);
        hl.assign((size_t)nq, ix.lists);
        for (int64_t i = 0; i < nq; ++i) hb[(size_t)i] = i * ix.lists;
    }
    VB_TRY(launch_segment_topk_v((const float*)d_cdist, seg_begin, seg_len, hb.empty() ? nullptr : hb.data(),
                                 hl.empty() ? nullptr : hl.data(), nq, probes, lists, ldist));
    *d_lists = lists;
    *d_ldist = ldist;
    return VB_OK;
}

// the (list, table tile) work units of the tensor-core scan, from the list offsets
static int ivf_build_units(Ivf& ix) {
    std::vector<ListUnit> units;
    for (int l = 0; l < ix.lists; ++l) {
        const int64_t lo = ix.h_list_off[(size_t)l], hi = ix.h_list_off[(size_t)l + 1];
        if (hi <= lo) continue;
        for (int64_t t = lo / 128; t <= (hi - 1) / 128; ++t) units.push_back(ListUnit{l, (int32_t)t});
    }
    if (ix.tc.units) VB_CUDA(cudaFree(ix.tc.units));
    ix.tc.units = nullptr;
    ix.tc.n_units = (int)units.size();
    if (!units.empty()) {
        VB_CUDA(cudaMalloc(&ix.tc.units, sizeof(ListUnit) * units.size()));
        VB_CUDA(cudaMemcpy(ix.tc.units, units.data(), sizeof(ListUnit) * units.size(), cudaMemcpyHostToDevice));
    }
    return VB_OK;
}

// packed planes, row norms and the (list, table tile) work units of the tensor-core scan; built lazily because the
// planes double the index footprint and only batched searches use them
static int ivf_ensure_tc_image(Ivf& ix) {
    if (ix.tc.planes || !ix.tc.finite) return VB_OK;
    {
        // the planes are as large as an fp32 table: keep the exact kernels when they do not fit beside the index
        const size_t need = (size_t)((ix.rows.n + 127) / 128) * 128 * ((size_t)(ix.rows.dim + 63) / 64) * 64 * 4;
        size_t free_b = 0, total_b = 0;
        VB_CUDA(cudaMemGetInfo(&free_b, &total_b));
        if (free_b < need + ((size_t)4 << 30)) {
            ix.tc.finite = false;
            return VB_OK;
        }
    }
    VB_TRY(list_tc_prepare(ix.rows, &ix.tc));
    ix.tc_cap_tiles = ix.tc.n_tiles;
    return ivf_build_units(ix);
}

// the int8 plane of level 0 (a quarter of the bf16 planes), built on first use where it fits with 4 GiB to spare
static int ivf_ensure_l0_image(Ivf& ix) {
    if (ix.tc.l0_tried) return VB_OK;
    const size_t rows = (size_t)ix.tc.n_tiles * 128;
    const size_t need = rows * ((size_t)(ix.rows.dim + 127) / 128) * 128 + rows * 8;   // (plane, s_x, R_x)
    size_t free_b = 0, total_b = 0;
    VB_CUDA(cudaMemGetInfo(&free_b, &total_b));
    if (free_b < need + ((size_t)4 << 30)) {
        ix.tc.l0_tried = true;
        return VB_OK;
    }
    ix.tc_cap_tiles8 = ix.tc.n_tiles;
    return list_tc_prepare_l0(ix.rows, &ix.tc);
}

// level P's basis and projected plane (4 r bytes a row, r <= dim / 8), built on first use where it fits with 4 GiB to spare
static int ivf_ensure_lp_image(Ivf& ix) {
    if (ix.lp.tried) return VB_OK;
    const size_t need = (size_t)std::max(ix.rows.cap, ix.rows.n) * (size_t)(ix.rows.dim / 8) * 4 + (size_t)ix.rows.dim * ix.rows.dim * 10;
    size_t free_b = 0, total_b = 0;
    VB_CUDA(cudaMemGetInfo(&free_b, &total_b));
    if (free_b < need + ((size_t)4 << 30)) {
        ix.lp.tried = true;
        return VB_OK;
    }
    return list_proj_prepare(ix.rows, ix.lists, &ix.lp);
}

// Whether level P pays for a batch: it reads 4 r bytes of every probed row instead of level 0's dim, and its looser bound
// re-scores about LP_EXTRA_ROWS more rows per query than level 0's (44.7 against 13.7 on bench.py's rank16 law, DESIGN
// section 4), 4 dim bytes each.  The batch probes about n (1 - (1 - probes / lists)^nq) distinct rows.  Before the basis
// is built r is taken at its cap, dim / 8.  Those figures hold for batches of thousands of queries over an index of a
// thousand lists; as for the tensor-core probe selection, a batch of fewer than 256 queries or an index of fewer than 128
// lists keeps level 0.
constexpr double LP_EXTRA_ROWS = 32.0;
static bool ivf_levelp_pays(const Ivf& ix, int64_t nq, int probes) {
    if (nq < 256 || ix.lists < 128) return false;
    const int r = ix.lp.tried ? ix.lp.r : ix.rows.dim / 8 / 16 * 16;
    const double rows = (double)ix.rows.n * (1.0 - std::pow(1.0 - (double)probes / ix.lists, (double)nq));
    return rows * (ix.rows.dim - 4.0 * r) > (double)nq * LP_EXTRA_ROWS * 4.0 * ix.rows.dim;
}

// scan the given probe lists for a batch of queries and keep the k nearest per query (mask: of the rows each query's
// row filter allows).  cap bounds the candidates of one query; *qn as in ivf_select_probes; *level: the filter level
// the scan ran at, or IVF_LEVEL_EXACT
static int ivf_scan_topk(Scratch& sc, Ivf& ix, const IvfPass& pass, const void* qimg, size_t qstride, int64_t nq, float** qn,
                         const int32_t* d_lists, int probes, int64_t cap, int k, int64_t* out_ids_dev, float* out_f_dev, double* out_d_dev,
                         int* level_out = nullptr, const IvfMask* mask = nullptr) {
    Context& c = ctx();
    const int rpc = scan_chunk_rows(ix.rows);
    const int64_t max_chunks = nq * (cap / rpc + probes + 1);
    VB_REQUIRE(max_chunks < (int64_t)INT32_MAX, "too many scan chunks (%lld)", (long long)max_chunks);
    void *d_chunks, *d_seg, *d_dist, *d_pos;
    VB_TRY(sc.take(sizeof(Chunk) * (size_t)max_chunks + sizeof(int32_t) * (size_t)nq * (probes + 1) + 64, &d_chunks));
    Chunk* chunks = (Chunk*)d_chunks;
    int32_t* cand_off = (int32_t*)(chunks + max_chunks);
    VB_TRY(sc.take((sizeof(int64_t) + sizeof(int32_t)) * (size_t)nq * 2 + 64, &d_seg));
    int64_t* seg_begin = (int64_t*)d_seg;
    int32_t* seg_len = (int32_t*)(seg_begin + nq);
    int* n_chunks = (int*)(seg_len + nq);
    VB_CUDA(cudaMemsetAsync(n_chunks, 0, sizeof(int), c.stream));
    // chunk descriptors are for the per-query scan kernels only; batched scans (tensor-core filter, list-major) skip them
    const bool per_query_scan = !(list_major_supported(ix.elem, key_metric(ix.metric)) && ix.n_tiles > 0 &&
                                  (c.scan_impl >= 3 || (c.scan_impl == 2 && nq * probes >= 256)));
    ivf_build_chunks_kernel<<<(unsigned)nq, per_query_scan ? 128 : 32, 0, c.stream>>>(d_lists, probes, ix.d_list_off, rpc, cap, cand_off, seg_begin,
                                                                                      seg_len, per_query_scan ? chunks : nullptr, n_chunks,
                                                                                      ix.d_cand_sum, nullptr);
    VB_CUDA(cudaGetLastError());
    count_launch();
    VB_TRY(sc.take(sizeof(float) * (size_t)nq * cap, &d_dist));
    prof_begin(VB_PROF_SCAN_ITEMS);
    // scan_impl: 0 = per-query LDG scan, 1 = per-query bulk-copy scan, 2 = automatic, 3 = list-major fp32 wherever it
    // applies, 4 = tensor-core filter + exact re-score wherever it applies.
    // Automatic: once a batch carries enough (query, probe) pairs to fill the GPU with row tiles, group them by list
    // so each probed list is read once per batch instead of once per query; small k goes through the tensor-core
    // filter (HBM-bound), larger k through the fp32 list-major kernel (FMA-pipe bound).
    const int km = key_metric(ix.metric);
    const bool batched = nq * probes >= 256 || pass.repair;
    bool tc = (c.scan_impl == 4 || c.scan_impl == 2) && pass.mode != IvfPass::EXACT && batched && list_tc_supported(ix.elem, km, k) &&
              ix.rows.n > 0;
    if (tc) {
        VB_TRY(ivf_ensure_tc_image(ix));
        tc = ix.tc.finite;   // rows with Inf / NaN norms have no error bound: exact path
    }
    if (level_out) *level_out = IVF_LEVEL_EXACT;
    if (tc) {
        // level 1 reads only the hi plane of the rows (half the HBM traffic, error bound 2^-7 |x||q|): it certifies
        // whenever the neighbours are separated by more than that, otherwise the batch is repeated at level 2 (both
        // planes, 2^-12) and level 1 rests for a while
        const bool level2 = pass.mode == IvfPass::LEVEL2;
        int level = (c.tc_level1 && !level2 && ix.l1_cooldown == 0 && list_tc_kp(k, 1) <= 128) ? 1 : 2;
        if (ix.l1_cooldown > 0 && !level2) --ix.l1_cooldown;
        // slab minima for the selection (vb_common.cuh slab_base): with them the k' nearest are found from 32 k' candidates
        // per query instead of the whole run.  They hold a run's slab keys in shared memory, so they are taken only where
        // the launch that reads them fits: the refine at the level's k', or in a repeat at level 2 slab_select_kernel.
        // Elsewhere the k' are selected from the whole run (launch_segment_topk_v).
        const int64_t cap_s = slab_cap(cap, probes);
        auto slabs_fit = [&](int lvl) {
            const int kp = list_tc_kp(k, lvl);
            const size_t smem = level2 ? slab_select_launch_smem(cap_s, probes) : cta_refine_smem_bytes(kp, qstride, true, false, cap, cap_s, probes);
            return c.slab_select && nq * cap_s < (int64_t)INT32_MAX && kp <= 128 && smem <= SS_SMEM_MAX;
        };
        // level 0 in front of level 1: int8 rows (1 byte per element, bound ~R_max |q|, k' = 128).  Its uncertified queries
        // are listed by the one-CTA-per-query refine, and a pass allows it only where its caller searches them again on
        // their own.
        if (level == 1 && c.tc_level0 && pass.level0 && slabs_fit(0)) {
            if (ix.l0_cooldown > 0) {
                --ix.l0_cooldown;
            } else {
                VB_TRY(ivf_ensure_l0_image(ix));
                if (ix.tc.planes8) level = 0;
            }
        }
        // level P in front of level 0: lower bounds from the rows' projection on their principal directions (fp32 rows,
        // L2, where the rows' spectrum allows a basis: vb_list_proj.cu), where the scan is chosen automatically (scan_impl
        // 4 asks for the tensor-core filter) and the batch is large enough for it to pay.  Its uncertified queries are
        // listed by the same refine and searched again from level 0.
        if (level == 0 && c.tc_levelp && c.scan_impl == 2 && pass.levelp && km == VB_L2_SQUARED && ix.elem == VB_VECTOR && ix.n_tiles > 0 &&
            ivf_levelp_pays(ix, nq, probes)) {
            if (ix.lp_cooldown > 0) {
                --ix.lp_cooldown;
            } else {
                VB_TRY(ivf_ensure_lp_image(ix));
                if (ix.lp.r > 0) level = LIST_LEVEL_P;
            }
        }
        const bool listed = level == 0 || level == LIST_LEVEL_P;
        if (listed && ix.l0_fail_cap < nq) {
            if (ix.d_l0_fail) VB_CUDA(cudaFree(ix.d_l0_fail));
            VB_CUDA(cudaMalloc(&ix.d_l0_fail, sizeof(int32_t) * (size_t)nq));
            ix.l0_fail_cap = nq;
        }
        if (level_out) *level_out = level;
        const int kp = list_tc_kp(k, level);
        const bool slabs = slabs_fit(level);
        void* d_smin = nullptr;
        if (slabs) VB_TRY(sc.take(sizeof(float) * (size_t)nq * cap_s, &d_smin));
        if (!*qn) VB_TRY(list_tc_query_norms(sc, qimg, qstride, nq, qn));
        if (level == LIST_LEVEL_P)
            VB_TRY(launch_list_proj(sc, ix.rows, ix.lp, ix.tc, qimg, qstride, nq, d_lists, probes, cand_off, cap, ix.d_list_off, ix.lists,
                                    (float*)d_dist, *qn, (float*)d_smin, cap_s));
        else
            VB_TRY(launch_list_tc(ix.rows, ix.tc, km, qimg, qstride, nq, d_lists, probes, cand_off, cap, ix.d_list_off, ix.lists,
                                  (float*)d_dist, *qn, false, level, (float*)d_smin, cap_s));
        prof_end(VB_PROF_SCAN_ITEMS);
        if (mask)
            VB_TRY(ivf_mask_runs(*mask, nq, d_lists, probes, cand_off, ix.d_list_off, cap, (float*)d_dist, (float*)d_smin, cap_s));
        const int32_t* has_nan = mask ? mask->has_nan : nullptr;
        VB_TRY(sc.take((sizeof(int32_t) + sizeof(float)) * (size_t)nq * (k + kp), &d_pos));
        int32_t* pos = (int32_t*)d_pos;
        float* key = (float*)(pos + (size_t)nq * k);
        int32_t* pos_kp = (int32_t*)(key + (size_t)nq * k);
        float* key_kp = (float*)(pos_kp + (size_t)nq * kp);
        prof_begin(VB_PROF_TOPK);
        int n_failed = 0;
        if (!ix.d_tc_fail) VB_TRY(ivf_tc_fail_zero(ix));
        if (!pass.defer_check) VB_CUDA(cudaMemsetAsync(ix.d_tc_fail + 1, 0, sizeof(int), c.stream));
        if (slabs && !level2) {
            // one CTA per query: slab selection, re-score on eight warps, ranking, certificate (a selection that overflows
            // counts as uncertified: the repeat of the batch selects below)
            VB_TRY(launch_list_tc_cta_refine(ix.rows, ix.tc, km, qimg, qstride, nq, k, kp, probes, d_lists, cand_off, ix.d_list_off,
                                             (const float*)d_dist, (const float*)d_smin, nullptr, nullptr, cap, cap_s, seg_len, *qn, pos, key,
                                             ix.d_tc_fail + 1, level, listed ? ix.d_l0_fail : nullptr, has_nan));
        } else {
            // the k' selected by a launch of their own (slab_select_kernel hands what overflows it to the full selection)
            if (slabs)
                VB_TRY(launch_slab_select((const float*)d_dist, (const float*)d_smin, nq, probes, d_lists, cand_off, ix.d_list_off, cap,
                                          cap_s, seg_begin, seg_len, kp, pos_kp, key_kp));
            else
                VB_TRY(launch_segment_topk_v((const float*)d_dist, seg_begin, seg_len, nullptr, nullptr, nq, kp, pos_kp, key_kp));
            VB_TRY(launch_list_tc_cta_refine(ix.rows, ix.tc, km, qimg, qstride, nq, k, kp, probes, d_lists, cand_off, ix.d_list_off,
                                             (const float*)d_dist, nullptr, pos_kp, key_kp, cap, cap_s, seg_len, *qn, pos, key,
                                             ix.d_tc_fail + 1, level, nullptr, has_nan));
        }
        if (!pass.defer_check) {
            VB_CUDA(cudaMemcpyAsync(&n_failed, ix.d_tc_fail + 1, sizeof(int), cudaMemcpyDeviceToHost, c.stream));
            VB_CUDA(cudaStreamSynchronize(c.stream));
        }
        prof_end(VB_PROF_TOPK);
        ix.total_tc_failed += n_failed;
        if (n_failed == 0) {
            ivf_finish_kernel<<<(unsigned)((nq * k + 255) / 256), 256, 0, c.stream>>>(ix.metric, nq, k, probes, pos, key, d_lists, cand_off,
                                                                                      ix.d_list_off, ix.d_ids, out_ids_dev, out_f_dev,
                                                                                      out_d_dev);
            VB_CUDA(cudaGetLastError());
            count_launch();
            if (mask)
                VB_TRY(ivf_unmask(ix, *mask, nq, k, probes, pos, key, (const float*)d_dist, cap, d_lists, cand_off, out_ids_dev, out_f_dev,
                                  out_d_dev));
            return VB_OK;
        }
        // some certificate failed: the whole batch goes through the exact kernel below (rare by construction)
        prof_begin(VB_PROF_SCAN_ITEMS);
    }
    const bool list_major = list_major_supported(ix.elem, km) && ix.n_tiles > 0 && (c.scan_impl >= 3 || (c.scan_impl == 2 && batched));
    if (list_major) {
        VB_TRY(launch_list_major(ix.rows, km, qimg, qstride, nq, d_lists, probes, cand_off, cap, ix.d_list_off, ix.lists, ix.d_tiles,
                                 ix.n_tiles, (float*)d_dist));
    } else {
        VB_TRY(launch_scan_chunks(ix.rows, km, qimg, qstride, chunks, n_chunks, (int)max_chunks, (float*)d_dist));
    }
    prof_end(VB_PROF_SCAN_ITEMS);
    if (mask) VB_TRY(ivf_mask_runs(*mask, nq, d_lists, probes, cand_off, ix.d_list_off, cap, (float*)d_dist, nullptr, 0));
    VB_TRY(sc.take((sizeof(int32_t) + sizeof(float)) * (size_t)nq * k, &d_pos));
    int32_t* pos = (int32_t*)d_pos;
    float* key = (float*)(pos + (size_t)nq * k);
    std::vector<int64_t> hb;
    std::vector<int32_t> hl;
    if (k > 2048) {
        // "sort everything" path (reference semantics of GetScanItems): needs sizes on the host
        hb.resize((size_t)nq);
        hl.resize((size_t)nq);
        VB_CUDA(cudaMemcpyAsync(hl.data(), seg_len, sizeof(int32_t) * (size_t)nq, cudaMemcpyDeviceToHost, c.stream));
        VB_CUDA(cudaStreamSynchronize(c.stream));
        for (int64_t i = 0; i < nq; ++i) hb[(size_t)i] = i * cap;
    }
    prof_begin(VB_PROF_TOPK);
    VB_TRY(launch_segment_topk_v((const float*)d_dist, seg_begin, seg_len, hb.empty() ? nullptr : hb.data(),
                                 hl.empty() ? nullptr : hl.data(), nq, k, pos, key));
    prof_end(VB_PROF_TOPK);
    ivf_finish_kernel<<<(unsigned)((nq * k + 255) / 256), 256, 0, c.stream>>>(ix.metric, nq, k, probes, pos, key, d_lists, cand_off,
                                                                              ix.d_list_off, ix.d_ids, out_ids_dev, out_f_dev,
                                                                              out_d_dev);
    VB_CUDA(cudaGetLastError());
    count_launch();
    if (mask)
        VB_TRY(ivf_unmask(ix, *mask, nq, k, probes, pos, key, (const float*)d_dist, cap, d_lists, cand_off, out_ids_dev, out_f_dev, out_d_dev));
    return VB_OK;
}

// k-way merge of the per-rank results of the list-sharded scan: gathered [world][nq][k] (ids, distances) -> the k
// nearest per query by (distance, id).  One CTA per query, bitonic sort of the world * k entries in shared memory.
__global__ void __launch_bounds__(128) merge_ranks_kernel(const int64_t* __restrict__ g_ids, const float* __restrict__ g_dist, int world,
                                                          int64_t nq, int k, int P, int64_t* __restrict__ out_ids,
                                                          float* __restrict__ out_dist) {
    extern __shared__ uint64_t mk[];            // P keys: orderable(distance) << 32 | slot
    const int64_t q = blockIdx.x;
    const int total = world * k;
    for (int i = threadIdx.x; i < P; i += blockDim.x) {
        uint64_t key = ~0ull;
        if (i < total) {
            const int r = i / k, j = i % k;
            const size_t at = ((size_t)r * nq + q) * k + j;
            if (g_ids[at] >= 0) key = ((uint64_t)orderable_key(g_dist[at]) << 32) | (uint32_t)i;
        }
        mk[i] = key;
    }
    __syncthreads();
    // equal distances: the smaller id first (slots are rank-major, so compare ids explicitly on ties)
    for (int size = 2; size <= P; size <<= 1)
        for (int st = size >> 1; st > 0; st >>= 1) {
            for (int a = threadIdx.x; a < P; a += blockDim.x) {
                const int c = a ^ st;
                if (c > a) {
                    const uint64_t x = mk[a], y = mk[c];
                    bool gt = x > y;
                    if ((x >> 32) == (y >> 32) && x != ~0ull && y != ~0ull) {
                        const int sx = (int)(uint32_t)x, sy = (int)(uint32_t)y;
                        const int64_t ix = g_ids[((size_t)(sx / k) * nq + q) * k + sx % k];
                        const int64_t iy = g_ids[((size_t)(sy / k) * nq + q) * k + sy % k];
                        gt = ix > iy;
                    }
                    const bool up = (a & size) == 0;
                    if (gt == up) {
                        mk[a] = y;
                        mk[c] = x;
                    }
                }
            }
            __syncthreads();
        }
    for (int i = threadIdx.x; i < k; i += blockDim.x) {
        const uint64_t key = mk[i];
        int64_t id = -1;
        float d = __int_as_float(0x7F800000);
        if (key != ~0ull) {
            const int sl = (int)(uint32_t)key;
            const size_t at = ((size_t)(sl / k) * nq + q) * k + sl % k;
            id = g_ids[at];
            d = g_dist[at];
        }
        out_ids[q * k + i] = id;
        out_dist[q * k + i] = d;
    }
}

static int64_t ivf_batch_limit(const Ivf& ix, int probes) {
    // keep the candidate-distance buffer under ~1 GiB
    int64_t cap = ivf_cap(ix, probes);
    int64_t lim = (int64_t)(1ull << 30) / (4 * cap);
    return std::max<int64_t>(1, std::min<int64_t>(lim, 65535));
}

// ----------------------------------------------------------------------------- scans of one query (vb_ivf_one.cu)

static size_t ivf_qstride(const Ivf& ix) {   // stride of the query image upload_queries() builds
    const size_t pad = padded_row_bytes(ix.elem, ix.dim);
    return ix.elem == VB_HALFVEC ? pad * 2 : pad;
}

static int ivf_tickets(Ivf& ix, unsigned** probe_t, unsigned** scan_t) {
    if (!ix.d_ticket) {
        VB_CUDA(cudaMalloc(&ix.d_ticket, 2 * ONE_MAX_Q * sizeof(unsigned)));
        VB_CUDA(cudaMemsetAsync(ix.d_ticket, 0, 2 * ONE_MAX_Q * sizeof(unsigned), ctx().stream));
    }
    *probe_t = ix.d_ticket;
    *scan_t = ix.d_ticket + ONE_MAX_Q;
    return VB_OK;
}

// does a scan of nq queries (probes lists each, k results, at most cap candidates per query) take the fused kernels?
static int64_t one_cap(int64_t cap) { return (cap + 3) & ~(int64_t)3; }   // stride of a query's distance run: 16-byte aligned runs

static bool ivf_one_applies(const Ivf& ix, int64_t nq, int probes, int64_t k, int64_t cap) {
    if (!ctx().one_query || nq < 1 || nq > ONE_MAX_Q || ix.rows.n <= 0) return false;
    const size_t qs = ivf_qstride(ix);
    return one_probe_fits(ix.lists, qs, probes) && one_scan_fits(one_cap(cap), qs, probes, k);
}

// GetScanLists for nq <= ONE_MAX_Q query images: one launch (the lists in sc)
static int ivf_one_probes(Scratch& sc, Ivf& ix, const void* qimg, size_t qstride, int64_t nq, int probes, int32_t** d_lists, float** d_ldist) {
    void *d_cdist, *d_probe;
    VB_TRY(sc.take(sizeof(float) * (size_t)nq * ix.lists, &d_cdist));
    VB_TRY(sc.take((sizeof(int32_t) + sizeof(float)) * (size_t)nq * probes, &d_probe));
    int32_t* lists = (int32_t*)d_probe;
    float* ldist = (float*)(lists + (size_t)nq * probes);
    unsigned *tp, *ts;
    VB_TRY(ivf_tickets(ix, &tp, &ts));
    prof_begin(VB_PROF_SCAN_LISTS);
    VB_TRY(launch_one_probe(ix.centers, key_metric(ix.metric), qimg, qstride, nq, probes, (float*)d_cdist, tp, lists, ldist, ix.d_cand_sum));
    prof_end(VB_PROF_SCAN_LISTS);
    *d_lists = lists;
    *d_ldist = ldist;
    return VB_OK;
}

// GetScanItems + sort for nq <= ONE_MAX_Q query images over device-resident probe lists: one launch
static int ivf_one_items(Ivf& ix, const void* qimg, size_t qstride, int64_t nq, const int32_t* d_lists, int probes, int k, int64_t cap,
                         int64_t* out_ids_dev, float* out_f_dev, double* out_d_dev, bool cand_store) {
    cap = one_cap(cap);
    Scratch sc;
    void* d_dist;
    VB_TRY(sc.take(sizeof(float) * (size_t)nq * cap, &d_dist));
    unsigned *tp, *ts;
    VB_TRY(ivf_tickets(ix, &tp, &ts));
    prof_begin(VB_PROF_SCAN_ITEMS);
    VB_TRY(launch_one_scan(ix.rows, key_metric(ix.metric), ix.metric, ix.d_list_off, ix.d_ids, d_lists, probes, qimg, qstride, nq, k, cap,
                           (float*)d_dist, ts, out_ids_dev, out_f_dev, out_d_dev, nullptr, ix.d_cand_sum, cand_store));
    prof_end(VB_PROF_SCAN_ITEMS);
    return VB_OK;
}

// results of a fused scan to host memory: ONE copy (ids and float8 distances are adjacent in the scratch) into the pinned
// staging buffer, one synchronisation
static int ivf_one_fetch(const void* d_out, int64_t n, int64_t* out_ids, double* out_d) {
    void* pin;
    VB_TRY(pinned_buffer2(16 * (size_t)n, &pin));
    VB_CUDA(cudaMemcpyAsync(pin, d_out, 16 * (size_t)n, cudaMemcpyDeviceToHost, ctx().stream));
    VB_CUDA(cudaStreamSynchronize(ctx().stream));
    memcpy(out_ids, pin, 8 * (size_t)n);
    memcpy(out_d, (const uint8_t*)pin + 8 * (size_t)n, 8 * (size_t)n);
    return VB_OK;
}

}  // namespace vb

using namespace vb;

struct vb_ivf {
    Ivf ix;
    uint64_t uid = next_owner_uid();   // matched by the row filters made for this image
};

// ivfflat.iterative_scan for a batch of queries (vb_ivf_iter.cu).  Everything kept between calls lives in `mem`, one
// allocation the handle owns: scratch only carries data within a call.
struct vb_ivf_scan {
    Ivf* ix = nullptr;
    uint64_t generation = 0;   // ix->generation at begin
    int64_t nq = 0;
    int probes = 0, max_probes = 0, page = 0, rpc = 0;
    int64_t cap = 0, max_chunks = 0;
    size_t qstride = 0;
    void* mem = nullptr;
    uint8_t* qimg = nullptr;       // [nq][qstride] query image
    int32_t* probe = nullptr;      // [nq][max_probes] lists in probe order
    int32_t* glists = nullptr;     // [nq][probes] lists of the current group (-1 padded)
    int32_t* cand_off = nullptr;   // [nq][probes + 1]
    int64_t* seg_begin = nullptr;  // [nq]
    int32_t* seg_len = nullptr;    // [nq] candidates of the current group
    int32_t* list_index = nullptr; // [nq] the reference's listIndex
    uint64_t* floor_key = nullptr; // [nq] composite key of the last element returned
    int32_t* returned = nullptr;   // [nq] elements of the current group returned so far
    int32_t* active = nullptr;     // [nq] moved to a new group in this call
    float* dist = nullptr;         // [nq][cap] candidate distances of the current group
    Chunk* chunks = nullptr;       // [max_chunks]
    int* n_chunks = nullptr;
    int64_t* cand_sum = nullptr;
    int32_t* pos = nullptr;        // [nq][page] selected positions
    float* key = nullptr;          // [nq][page] their distances
    int64_t* out_ids = nullptr;    // staging, copied back at once: ids [nq][page] | float8 [nq][page] | counts [nq]
    double* out_d = nullptr;
    int32_t* counts = nullptr;
    // row filters (vb_ivf_scan_begin_filtered), copied at begin: probe[] holds virtual lists f * lists + l, whose runs
    // foff gives in fpos / fids; an unfiltered handle has nfilters = 0 and none of these
    int nfilters = 0;
    int64_t fallowed = 0;          // positions of all filters
    int64_t* fpos = nullptr;       // [fallowed] rows of the list-ordered image, filter after filter
    int64_t* fids = nullptr;       // [fallowed] their heap ids
    int64_t* foff = nullptr;       // [nfilters * lists + 1]
};

namespace vb {

// device bytes of a handle: per query (the rest is a few hundred bytes of alignment)
static size_t ivf_scan_bytes_per_query(const vb_ivf_scan& s) {
    return s.qstride + 4 * (size_t)s.max_probes + 4 * (size_t)s.probes + 4 * ((size_t)s.probes + 1) + 8 + 4 + 4 + 8 + 4 + 4 +
           4 * (size_t)s.cap + sizeof(Chunk) * (size_t)(s.max_chunks / s.nq) + (4 + 4 + 8 + 8) * (size_t)s.page + 4;
}

// carve the handle's allocation (bytes == 0: only count them)
static size_t ivf_scan_carve(vb_ivf_scan& s, uint8_t* base) {
    size_t off = 0;
    auto take = [&](size_t bytes) {
        uint8_t* p = base ? base + off : nullptr;
        off += (bytes + 255) & ~(size_t)255;
        return p;
    };
    const size_t nq = (size_t)s.nq;
    s.qimg = take(nq * s.qstride);
    s.probe = (int32_t*)take(4 * nq * s.max_probes);
    s.glists = (int32_t*)take(4 * nq * s.probes);
    s.cand_off = (int32_t*)take(4 * nq * (s.probes + 1));
    // cursor state, seg_begin .. cand_sum, zeroed at begin: every query starts with an empty group and listIndex 0
    s.seg_begin = (int64_t*)take(8 * nq);
    s.floor_key = (uint64_t*)take(8 * nq);
    s.seg_len = (int32_t*)take(4 * nq);
    s.list_index = (int32_t*)take(4 * nq);
    s.returned = (int32_t*)take(4 * nq);
    s.active = (int32_t*)take(4 * nq);
    s.n_chunks = (int*)take(8);
    s.cand_sum = (int64_t*)take(8);
    s.dist = (float*)take(4 * nq * (size_t)s.cap);
    s.chunks = (Chunk*)take(sizeof(Chunk) * (size_t)s.max_chunks);
    s.pos = (int32_t*)take(4 * nq * s.page);
    s.key = (float*)take(4 * nq * s.page);
    uint8_t* stage = take((8 + 8) * nq * s.page + 4 * nq);
    s.out_ids = (int64_t*)stage;
    s.out_d = stage ? (double*)(stage + 8 * nq * s.page) : nullptr;
    s.counts = stage ? (int32_t*)(stage + 16 * nq * s.page) : nullptr;
    if (s.nfilters) {
        s.fpos = (int64_t*)take(8 * (size_t)std::max<int64_t>(s.fallowed, 1));
        s.fids = (int64_t*)take(8 * (size_t)std::max<int64_t>(s.fallowed, 1));
        s.foff = (int64_t*)take(8 * ((size_t)s.nfilters * s.ix->lists + 1));
    }
    return off;
}

// device bytes the row filters' copies take in a handle
static size_t ivf_scan_filter_bytes(const vb_ivf_scan& s) {
    return s.nfilters ? 16 * (size_t)std::max<int64_t>(s.fallowed, 1) + 8 * ((size_t)s.nfilters * s.ix->lists + 1) : 0;
}

// query image and probe order of every query: the GetScanLists of vb_ivf_scan_lists, in sub-batches
static int ivf_scan_setup(vb_ivf_scan& s, const void* queries) {
    Ivf& ix = *s.ix;
    Context& c = ctx();
    const size_t state_bytes = (size_t)((uint8_t*)s.dist - (uint8_t*)s.seg_begin);
    VB_CUDA(cudaMemsetAsync(s.seg_begin, 0, state_bytes, c.stream));
    const size_t rawq = raw_row_bytes(ix.elem, ix.dim);
    const int64_t bq = std::min<int64_t>(s.nq, 65535);
    for (int64_t q0 = 0; q0 < s.nq; q0 += bq) {
        const int64_t m = std::min(bq, s.nq - q0);
        Scratch sc;
        void* qimg;
        size_t qstride;
        VB_TRY(upload_queries(sc, ix.elem, ix.dim, (const uint8_t*)queries + (size_t)q0 * rawq, m, true, &qimg, &qstride));
        VB_REQUIRE(qstride == s.qstride, "query image stride %zu, expected %zu", qstride, s.qstride);
        uint8_t* mine = s.qimg + (size_t)q0 * s.qstride;
        VB_CUDA(cudaMemcpyAsync(mine, qimg, (size_t)m * s.qstride, cudaMemcpyDeviceToDevice, c.stream));
        int32_t* d_lists;
        float* d_ldist;
        float* qn = nullptr;
        if (c.one_query && m <= ONE_MAX_Q && one_probe_fits(ix.lists, s.qstride, s.max_probes))
            VB_TRY(ivf_one_probes(sc, ix, mine, s.qstride, m, s.max_probes, &d_lists, &d_ldist));
        else
            VB_TRY(ivf_select_probes(sc, ix, IvfPass{}, mine, s.qstride, m, &qn, s.max_probes, &d_lists, &d_ldist));
        VB_CUDA(cudaMemcpyAsync(s.probe + (size_t)q0 * s.max_probes, d_lists, sizeof(int32_t) * (size_t)m * s.max_probes,
                                cudaMemcpyDeviceToDevice, c.stream));
    }
    VB_CUDA(cudaStreamSynchronize(c.stream));
    return VB_OK;
}

}  // namespace vb

extern "C" {

// ----------------------------------------------------------------------------- operator

int vb_distance_batch(int elem, int metric, int dim, const void* q, const void* rows, int64_t n, double* out) {
    VB_TRY(require_init());
    VB_REQUIRE(elem >= 0 && elem <= 2 && (dim > 0 || (elem == VB_BIT && dim == 0)) && metric_valid_for(elem, metric),
               "bad element type/metric/dim (%d, %d, %d)", elem, metric, dim);
    VB_TRY(require_scannable_rows(elem, dim));
    if (n <= 0) return VB_OK;
    // a zero-length bit string ('' :: bit) has no set bits: Hamming 0 and Jaccard 1 (ab == 0, src/bitvec.c:60-70), the
    // counts of eight zero bits -- scored as such by the same kernel
    std::vector<uint8_t> zero_rows, zero_q;
    if (dim == 0 && q != nullptr) {
        zero_rows.assign((size_t)n, 0);
        zero_q.assign(1, 0);
        rows = zero_rows.data();
        q = zero_q.data();
        dim = 8;
    }
    if (q == nullptr) {  // ZeroDistance (src/ivfscan.c:192-196)
        for (int64_t i = 0; i < n; ++i) out[i] = 0.0;
        return VB_OK;
    }
    Context& c = ctx();
    Table t;
    t.elem = elem;
    t.dim = dim;
    t.stride = padded_row_bytes(elem, dim);
    int rc = table_append_host(t, rows, n);
    if (rc != VB_OK) {
        table_free(t);
        return rc;
    }
    Scratch sc;
    void* qimg;
    size_t qstride;
    void* d_out;
    rc = upload_queries(sc, elem, dim, q, 1, true, &qimg, &qstride);
    if (rc == VB_OK) rc = sc.take(sizeof(double) * (size_t)n, &d_out);
    if (rc == VB_OK) rc = launch_scan_regular_f64(t, key_metric(metric), qimg, qstride, 1, n, (double*)d_out, n);
    if (rc == VB_OK) {
        cudaError_t e = cudaMemcpyAsync(out, d_out, sizeof(double) * (size_t)n, cudaMemcpyDeviceToHost, c.stream);
        if (e == cudaSuccess) e = cudaStreamSynchronize(c.stream);
        if (e != cudaSuccess) {
            set_error("copy back failed: %s", cudaGetErrorString(e));
            rc = VB_ECUDA;
        }
    }
    table_free(t);
    if (rc != VB_OK) return rc;
    // operator epilogues that are not the key metric (fp64, like the fmgr wrappers)
    if (metric == VB_L2)
        for (int64_t i = 0; i < n; ++i) out[i] = sqrt(out[i]);
    else if (metric == VB_IP)
        for (int64_t i = 0; i < n; ++i) out[i] = -out[i];
    else if (metric == VB_SPHERICAL)
        for (int64_t i = 0; i < n; ++i) {
            double d = -out[i];  // src/vector.c:714-722
            if (d > 1) d = 1;
            else if (d < -1) d = -1;
            out[i] = acos(d) / M_PI;
        }
    return VB_OK;
}

// ----------------------------------------------------------------------------- tables

int vb_table_create(int elem, int dim, vb_table** out) {
    VB_TRY(require_init());
    VB_REQUIRE(elem >= 0 && elem <= 2 && dim > 0 && out, "bad table arguments");
    VB_TRY(require_scannable_rows(elem, dim));
    vb_table* t = new vb_table();
    t->t.elem = elem;
    t->t.dim = dim;
    t->t.stride = padded_row_bytes(elem, dim);
    *out = t;
    return VB_OK;
}
int vb_table_append(vb_table* t, const void* rows, int64_t n) {
    VB_TRY(require_init());
    VB_REQUIRE(t && (rows || n == 0), "null table/rows");
    return table_append_host(t->t, rows, n);
}
int vb_table_append_dev(vb_table* t, const void* rows_dev, int64_t n) {
    VB_TRY(require_init());
    VB_REQUIRE(t && (rows_dev || n == 0), "null table/rows");
    return table_append_dev(t->t, rows_dev, n);
}
int64_t vb_table_rows(const vb_table* t) { return t ? t->t.n : 0; }
const void* vb_table_device_rows(const vb_table* t, size_t* stride_bytes) {
    if (!t) return nullptr;
    if (stride_bytes) *stride_bytes = t->t.stride;
    return t->t.d;
}
int vb_table_free(vb_table* t) {
    if (t) {
        table_free(t->t);
        owner_released(t->uid);
        delete t;
    }
    return VB_OK;
}

static int exact_topk_impl(vb_table* t, int metric, const void* queries, int64_t nq, int k, bool host, int64_t* out_ids,
                           float* out_f, double* out_d) {
    VB_TRY(require_init());
    VB_REQUIRE(t && metric_valid_for(t->t.elem, metric) && metric != VB_SPHERICAL, "bad table/metric");
    VB_REQUIRE(metric != VB_JACCARD || true, "");
    VB_REQUIRE(k > 0, "k must be positive");
    if (nq <= 0) return VB_OK;
    Context& c = ctx();
    Table& T = t->t;
    const int64_t n = T.n;
    const size_t rawq = raw_row_bytes(T.elem, T.dim);
    // sub-batch so the distance matrix stays under ~1 GiB
    int64_t bq = std::max<int64_t>(1, std::min<int64_t>(nq, (int64_t)(1ull << 30) / (4 * std::max<int64_t>(n, 1))));
    for (int64_t q0 = 0; q0 < nq; q0 += bq) {
        Scratch sc;
        int64_t m = std::min(bq, nq - q0);
        void *qimg, *d_dist, *d_seg, *d_pos, *d_ids, *d_of;
        size_t qstride;
        VB_TRY(upload_queries(sc, T.elem, T.dim, (const uint8_t*)queries + (size_t)q0 * rawq, m, host, &qimg, &qstride));
        VB_TRY(sc.take(sizeof(float) * (size_t)m * std::max<int64_t>(n, 1), &d_dist));
        // A batch of queries against the whole table is a distance matrix: tile it (table rows read once per 128
        // queries instead of once per query) when the query image has the table's row layout.  One query at a
        // time, or a metric with a per-row epilogue, streams the table through the scan kernel instead.
        const int km = key_metric(metric);
        const bool tiled = m >= 64 && n >= 128 && n <= 65535LL * 128 && T.elem != VB_HALFVEC && qstride == T.stride && c.scan_impl != 0 &&
                           (km == VB_L2_SQUARED || km == VB_NEG_IP || km == VB_HAMMING);
        if (tiled) {
            Table Q;
            Q.elem = T.elem;
            Q.dim = T.dim;
            Q.stride = qstride;
            Q.n = m;
            Q.d = (uint8_t*)qimg;
            VB_TRY(launch_distance_matrix(Q, km, T, (int)n, (float*)d_dist, n));
        } else {
            VB_TRY(launch_scan_regular(T, km, qimg, qstride, m, n, (float*)d_dist, n));
        }
        VB_TRY(sc.take((sizeof(int64_t) + sizeof(int32_t)) * (size_t)m + 64, &d_seg));
        int64_t* seg_begin = (int64_t*)d_seg;
        int32_t* seg_len = (int32_t*)(seg_begin + m);
        regular_segments_kernel<<<(unsigned)((m + 255) / 256), 256, 0, c.stream>>>(m, n, (int32_t)n, seg_begin, seg_len);
        VB_CUDA(cudaGetLastError());
        count_launch();
        VB_TRY(sc.take((sizeof(int32_t) + sizeof(float)) * (size_t)m * k, &d_pos));
        int32_t* pos = (int32_t*)d_pos;
        float* key = (float*)(pos + (size_t)m * k);
        std::vector<int64_t> hb;
        std::vector<int32_t> hl;
        if (k > 2048) {
            hb.resize((size_t)m);
            hl.assign((size_t)m, (int32_t)n);
            for (int64_t i = 0; i < m; ++i) hb[(size_t)i] = i * n;
        }
        VB_TRY(launch_segment_topk_v((const float*)d_dist, seg_begin, seg_len, hb.empty() ? nullptr : hb.data(),
                                     hl.empty() ? nullptr : hl.data(), m, k, pos, key));
        int64_t* o_ids;
        float* o_f = nullptr;
        double* o_d = nullptr;
        if (host) {
            VB_TRY(sc.take((sizeof(int64_t) + sizeof(double)) * (size_t)m * k, &d_ids));
            o_ids = (int64_t*)d_ids;
            o_d = (double*)(o_ids + (size_t)m * k);
        } else {
            o_ids = out_ids + q0 * k;
            o_f = out_f + q0 * k;
        }
        (void)d_of;
        finish_exact_kernel<<<(unsigned)((m * k + 255) / 256), 256, 0, c.stream>>>(metric, m * k, pos, key, o_ids, o_f, o_d);
        VB_CUDA(cudaGetLastError());
        count_launch();
        if (host) {
            VB_CUDA(cudaMemcpyAsync(out_ids + q0 * k, o_ids, sizeof(int64_t) * (size_t)m * k, cudaMemcpyDeviceToHost, c.stream));
            VB_CUDA(cudaMemcpyAsync(out_d + q0 * k, o_d, sizeof(double) * (size_t)m * k, cudaMemcpyDeviceToHost, c.stream));
            VB_CUDA(cudaStreamSynchronize(c.stream));
        }
    }
    return VB_OK;
}

int vb_exact_topk(vb_table* t, int metric, const void* queries, int64_t nq, int k, int64_t* out_ids, double* out_dist) {
    return exact_topk_impl(t, metric, queries, nq, k, true, out_ids, nullptr, out_dist);
}
int vb_exact_topk_dev(vb_table* t, int metric, const void* queries_dev, int64_t nq, int k, int64_t* out_ids_dev,
                      float* out_dist_dev) {
    return exact_topk_impl(t, metric, queries_dev, nq, k, false, out_ids_dev, out_dist_dev, nullptr);
}

// ----------------------------------------------------------------------------- IVFFlat

int vb_ivf_create(int elem, int metric, int dim, int lists, vb_ivf** out) {
    VB_TRY(require_init());
    VB_REQUIRE(out && elem >= 0 && elem <= 2 && dim > 0 && lists >= 1 && lists <= 32768, "bad ivfflat arguments (lists 1..32768, src/ivfflat.h:56-57)");
    bool ok = elem == VB_BIT ? metric == VB_HAMMING : (metric == VB_L2_SQUARED || metric == VB_NEG_IP);
    VB_REQUIRE(ok, "ivfflat opclass proc 1 must be L2 squared / negative inner product (vector, halfvec) or Hamming (bit)");
    int64_t* d_cand_sum;
    VB_CUDA(cudaMalloc(&d_cand_sum, sizeof(int64_t)));
    VB_CUDA(cudaMemsetAsync(d_cand_sum, 0, sizeof(int64_t), ctx().stream));
    vb_ivf* h = new vb_ivf();
    Ivf& ix = h->ix;
    ix.d_cand_sum = d_cand_sum;
    ix.elem = elem;
    ix.metric = metric;
    ix.dim = dim;
    ix.lists = lists;
    ix.centers.elem = ix.rows.elem = elem;
    ix.centers.dim = ix.rows.dim = dim;
    ix.centers.stride = ix.rows.stride = padded_row_bytes(elem, dim);
    *out = h;
    return VB_OK;
}

// list offsets, lengths, device offsets and list-major row tiles; release: a load or list replacement, whose rows are
// about to change (the packed planes are rebuilt on the next tensor-core scan), rather than an in-place insert or delete
// (which re-packs them itself)
static int ivf_set_layout(Ivf& ix, const int64_t* list_offsets, bool release) {
    ix.h_list_off.assign(list_offsets, list_offsets + ix.lists + 1);
    VB_REQUIRE(ix.h_list_off[0] == 0, "list_offsets[0] must be 0");
    ix.sorted_len.resize((size_t)ix.lists);
    for (int l = 0; l < ix.lists; ++l) {
        int64_t len = ix.h_list_off[(size_t)l + 1] - ix.h_list_off[(size_t)l];
        VB_REQUIRE(len >= 0 && len < (int64_t)INT32_MAX, "bad list length");
        ix.sorted_len[(size_t)l] = len;
    }
    std::sort(ix.sorted_len.begin(), ix.sorted_len.end(), std::greater<int64_t>());
    if (!ix.d_list_off) VB_CUDA(cudaMalloc(&ix.d_list_off, sizeof(int64_t) * ((size_t)ix.lists + 1)));
    VB_CUDA(cudaMemcpy(ix.d_list_off, ix.h_list_off.data(), sizeof(int64_t) * ((size_t)ix.lists + 1), cudaMemcpyHostToDevice));
    // row tiles of the list-major scan: fixed by the list boundaries, so built once per load
    std::vector<ListTile> tiles;
    const int tr = list_tile_rows();
    for (int l = 0; l < ix.lists; ++l) {
        const int64_t lo = ix.h_list_off[(size_t)l], hi = ix.h_list_off[(size_t)l + 1];
        for (int64_t r = lo; r < hi; r += tr) tiles.push_back(ListTile{r, l, (int32_t)std::min<int64_t>(tr, hi - r)});
    }
    if (ix.d_tiles) cudaFree(ix.d_tiles);
    ix.d_tiles = nullptr;
    if (release) {
        list_tc_release(&ix.tc);   // rows are about to change: planes are rebuilt on the next tensor-core scan
        list_tc_release(&ix.ctc);
        list_proj_release(&ix.lp);
        ix.ids_cap = -1;
    }
    ix.n_tiles = (int)tiles.size();
    if (ix.n_tiles) {
        VB_CUDA(cudaMalloc(&ix.d_tiles, sizeof(ListTile) * tiles.size()));
        VB_CUDA(cudaMemcpy(ix.d_tiles, tiles.data(), sizeof(ListTile) * tiles.size(), cudaMemcpyHostToDevice));
    }
    return VB_OK;
}

static int ivf_set_offsets(Ivf& ix, const int64_t* list_offsets) { return ivf_set_layout(ix, list_offsets, true); }

int vb_ivf_load(vb_ivf* h, const void* centers, const int64_t* list_offsets, const void* rows, const int64_t* ids) {
    VB_TRY(require_init());
    VB_REQUIRE(h && centers && list_offsets, "null argument");
    Ivf& ix = h->ix;
    ++ix.generation;
    table_free(ix.centers);
    table_free(ix.rows);
    VB_TRY(ivf_set_offsets(ix, list_offsets));
    const int64_t n = ix.h_list_off[(size_t)ix.lists];
    VB_TRY(table_append_host(ix.centers, centers, ix.lists));
    VB_TRY(table_append_host(ix.rows, rows, n));
    if (ix.d_ids) cudaFree(ix.d_ids);
    ix.d_ids = nullptr;
    ix.has_ids = ids != nullptr;
    if (ids && n > 0) {
        VB_CUDA(cudaMalloc(&ix.d_ids, sizeof(int64_t) * (size_t)n));
        VB_CUDA(cudaMemcpy(ix.d_ids, ids, sizeof(int64_t) * (size_t)n, cudaMemcpyHostToDevice));
    }
    ix.loaded = true;
    return VB_OK;
}

int vb_ivf_load_dev(vb_ivf* h, const void* centers_dev, const int64_t* list_offsets_host, const void* rows_dev,
                    const int64_t* ids_dev) {
    VB_TRY(require_init());
    VB_REQUIRE(h && centers_dev && list_offsets_host, "null argument");
    Ivf& ix = h->ix;
    ++ix.generation;
    table_free(ix.centers);
    table_free(ix.rows);
    VB_TRY(ivf_set_offsets(ix, list_offsets_host));
    const int64_t n = ix.h_list_off[(size_t)ix.lists];
    VB_TRY(table_append_dev(ix.centers, centers_dev, ix.lists));
    VB_TRY(table_append_dev(ix.rows, rows_dev, n));
    if (ix.d_ids) cudaFree(ix.d_ids);
    ix.d_ids = nullptr;
    ix.has_ids = ids_dev != nullptr;
    if (ids_dev && n > 0) {
        VB_CUDA(cudaMalloc(&ix.d_ids, sizeof(int64_t) * (size_t)n));
        VB_CUDA(cudaMemcpyAsync(ix.d_ids, ids_dev, sizeof(int64_t) * (size_t)n, cudaMemcpyDeviceToDevice, ctx().stream));
    }
    VB_CUDA(cudaStreamSynchronize(ctx().stream));
    ix.loaded = true;
    return VB_OK;
}

int64_t vb_ivf_rows(const vb_ivf* h) { return h ? h->ix.rows.n : 0; }

// ---- list-at-a-time loading: the packer walks one entry-page chain at a time (src/ivfscan.c:139-179) and never holds
// more than one list on the host

int vb_ivf_begin_load(vb_ivf* h, const void* centers) {
    VB_TRY(require_init());
    VB_REQUIRE(h && centers, "null argument");
    Ivf& ix = h->ix;
    ++ix.generation;
    table_free(ix.centers);
    table_free(ix.rows);
    VB_TRY(table_append_host(ix.centers, centers, ix.lists));
    ix.loaded = false;
    ix.loading = true;
    ix.next_list = 0;
    ix.h_ids.clear();
    ix.pending_off.assign((size_t)ix.lists + 1, 0);
    return VB_OK;
}

int vb_ivf_load_list(vb_ivf* h, int list, const void* rows, const int64_t* ids, int64_t n) {
    VB_TRY(require_init());
    VB_REQUIRE(h && h->ix.loading, "vb_ivf_load_list outside vb_ivf_begin_load / vb_ivf_end_load");
    Ivf& ix = h->ix;
    VB_REQUIRE(list >= ix.next_list && list < ix.lists, "lists must arrive in ascending order (got %d, expected >= %d)", list, ix.next_list);
    VB_REQUIRE(n >= 0 && (n == 0 || (rows && ids)), "null rows / ids");
    for (int l = ix.next_list; l <= list; ++l) ix.pending_off[(size_t)l] = ix.rows.n;
    if (n > 0) {
        VB_TRY(table_append_host(ix.rows, rows, n));
        ix.h_ids.insert(ix.h_ids.end(), ids, ids + n);
    }
    ix.next_list = list + 1;
    ix.pending_off[(size_t)list + 1] = ix.rows.n;
    return VB_OK;
}

int vb_ivf_end_load(vb_ivf* h) {
    VB_TRY(require_init());
    VB_REQUIRE(h && h->ix.loading, "vb_ivf_end_load without vb_ivf_begin_load");
    Ivf& ix = h->ix;
    for (int l = ix.next_list; l <= ix.lists; ++l) ix.pending_off[(size_t)l] = ix.rows.n;
    ix.loading = false;
    ++ix.generation;
    VB_TRY(ivf_set_offsets(ix, ix.pending_off.data()));
    if (ix.d_ids) cudaFree(ix.d_ids);
    ix.d_ids = nullptr;
    ix.has_ids = true;
    const int64_t n = ix.rows.n;
    if (n > 0) {
        VB_CUDA(cudaMalloc(&ix.d_ids, sizeof(int64_t) * (size_t)n));
        VB_CUDA(cudaMemcpy(ix.d_ids, ix.h_ids.data(), sizeof(int64_t) * (size_t)n, cudaMemcpyHostToDevice));
    }
    ix.h_ids.clear();
    ix.h_ids.shrink_to_fit();
    ix.loaded = true;
    return VB_OK;
}

// One list of a loaded image changed (insert into it, vacuum of it): only that list crosses PCIe; the rows behind it
// move on the device, and the packed planes of the tensor-core filter are rebuilt on the device at the next batched scan.
int vb_ivf_replace_list(vb_ivf* h, int list, const void* rows, const int64_t* ids, int64_t n) {
    VB_TRY(require_init());
    VB_REQUIRE(h && h->ix.loaded, "index not loaded");
    Ivf& ix = h->ix;
    VB_REQUIRE(list >= 0 && list < ix.lists && n >= 0 && (n == 0 || (rows && ids)), "bad list / rows");
    Context& c = ctx();
    ++ix.generation;
    const int64_t lo = ix.h_list_off[(size_t)list], hi = ix.h_list_off[(size_t)list + 1];
    const int64_t total = ix.rows.n, tail = total - hi, new_total = lo + n + tail;
    Table T;
    T.elem = ix.rows.elem;
    T.dim = ix.rows.dim;
    T.stride = ix.rows.stride;
    VB_TRY(table_reserve(T, std::max<int64_t>(new_total, 1)));
    int64_t* new_ids = nullptr;
    if (new_total > 0) VB_CUDA(cudaMalloc(&new_ids, sizeof(int64_t) * (size_t)new_total));
    if (lo > 0) {
        VB_CUDA(cudaMemcpyAsync(T.d, ix.rows.d, (size_t)lo * T.stride, cudaMemcpyDeviceToDevice, c.stream));
        VB_CUDA(cudaMemcpyAsync(new_ids, ix.d_ids, sizeof(int64_t) * (size_t)lo, cudaMemcpyDeviceToDevice, c.stream));
    }
    T.n = lo;
    int rc = n > 0 ? table_append_host(T, rows, n) : VB_OK;   // (synchronises the stream)
    if (rc == VB_OK && n > 0 &&
        cudaMemcpyAsync(new_ids + lo, ids, sizeof(int64_t) * (size_t)n, cudaMemcpyHostToDevice, c.stream) != cudaSuccess)
        rc = VB_ECUDA;
    if (rc == VB_OK && tail > 0) {
        if (cudaMemcpyAsync(T.d + (size_t)(lo + n) * T.stride, ix.rows.d + (size_t)hi * T.stride, (size_t)tail * T.stride,
                            cudaMemcpyDeviceToDevice, c.stream) != cudaSuccess ||
            cudaMemcpyAsync(new_ids + lo + n, ix.d_ids + hi, sizeof(int64_t) * (size_t)tail, cudaMemcpyDeviceToDevice, c.stream) != cudaSuccess)
            rc = VB_ECUDA;
    }
    if (rc == VB_OK && cudaStreamSynchronize(c.stream) != cudaSuccess) rc = VB_ECUDA;
    if (rc != VB_OK) {
        table_free(T);
        if (new_ids) cudaFree(new_ids);
        if (rc == VB_ECUDA) set_error("vb_ivf_replace_list: device copy failed");
        return rc;
    }
    T.n = new_total;
    table_free(ix.rows);
    ix.rows = T;
    if (ix.d_ids) cudaFree(ix.d_ids);
    ix.d_ids = new_ids;
    std::vector<int64_t> off = ix.h_list_off;
    const int64_t delta = n - (hi - lo);
    for (int l = list + 1; l <= ix.lists; ++l) off[(size_t)l] += delta;
    return ivf_set_offsets(ix, off.data());
}

// ---- in-place inserts and deletes (ivfflatinsert, ivfflatbulkdelete)
//
// Both move the rows of the list-ordered table to new places in a monotone pattern: an insert moves every row up by the
// rows inserted into lists before its own, a delete moves every kept row down by the rows removed before it.  Only the
// suffix from the first changed row moves, window by window through a bounded staging buffer -- back to front when rows
// move up, front to back when they move down -- so that no window's destinations reach the sources of a window not yet
// staged, and the table is never copied whole.  The derived state follows in place: list offsets and tiles, and the
// packed planes of the tensor-core filter (where built) from the 128-row tile that holds the first changed row on, with
// the norm statistics its certificates use recomputed over the whole table (list_tc_repack).

constexpr size_t IVF_MOVE_WINDOW_BYTES = (size_t)256 << 20;

// one warp per row: row i of src and its id to table row dst[i] (dst[i] < 0: dropped)
__global__ void ivf_move_rows_kernel(const uint8_t* __restrict__ src, const int64_t* __restrict__ src_ids, int64_t m,
                                     const int64_t* __restrict__ dst, size_t stride, uint8_t* __restrict__ rows, int64_t* __restrict__ ids) {
    const int64_t i = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (i >= m) return;
    const int64_t d = dst[i];
    if (d < 0) return;
    const uint4* s = reinterpret_cast<const uint4*>(src + (size_t)i * stride);
    uint4* o = reinterpret_cast<uint4*>(rows + (size_t)d * stride);
    for (size_t w = lane; w < stride / 16; w += 32) o[w] = s[w];
    if (lane == 0) ids[d] = src_ids[i];
}

// insert: row first + i of list l goes to first + i + shift[l] (list_off: the offsets before the insert)
__global__ void ivf_insert_dst_kernel(const int64_t* __restrict__ list_off, int lists, const int64_t* __restrict__ shift, int64_t first,
                                      int64_t n, int64_t* __restrict__ dst) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    const int64_t r = first + i;
    if (r >= n) return;
    int lo = 0, hi = lists;   // the list of row r: the largest l with list_off[l] <= r (list_off[lists] = n > r)
    while (hi - lo > 1) {
        const int mid = (lo + hi) >> 1;
        if (list_off[mid] <= r) lo = mid;
        else hi = mid;
    }
    dst[i] = r + shift[lo];
}

// delete: row first + i goes down by the removed rows before it, or is dropped (gone[0 .. m): the removed rows, ascending)
__global__ void ivf_delete_dst_kernel(const int64_t* __restrict__ gone, int64_t m, int64_t first, int64_t n, int64_t* __restrict__ dst) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    const int64_t r = first + i;
    if (r >= n) return;
    int64_t lo = 0, hi = m;   // first gone[j] >= r
    while (lo < hi) {
        const int64_t mid = (lo + hi) >> 1;
        if (gone[mid] < r) lo = mid + 1;
        else hi = mid;
    }
    dst[i] = lo < m && gone[lo] == r ? -1 : r - lo;
}

// table rows [first, n) to dst[0 .. n - first), in windows of `window` rows staged in stage / stage_ids
static int ivf_move_suffix(Ivf& ix, int64_t first, int64_t n, const int64_t* dst, bool up, uint8_t* stage, int64_t* stage_ids,
                           int64_t window) {
    Context& c = ctx();
    const size_t stride = ix.rows.stride;
    const int64_t nwin = (n - first + window - 1) / window;
    for (int64_t w = 0; w < nwin; ++w) {
        const int64_t a = up ? std::max(first, n - (w + 1) * window) : first + w * window;
        const int64_t m = up ? n - w * window - a : std::min(window, n - a);
        VB_CUDA(cudaMemcpyAsync(stage, ix.rows.d + (size_t)a * stride, (size_t)m * stride, cudaMemcpyDeviceToDevice, c.stream));
        VB_CUDA(cudaMemcpyAsync(stage_ids, ix.d_ids + a, sizeof(int64_t) * (size_t)m, cudaMemcpyDeviceToDevice, c.stream));
        ivf_move_rows_kernel<<<(unsigned)((m * 32 + 255) / 256), 256, 0, c.stream>>>(stage, stage_ids, m, dst + (a - first), stride, ix.rows.d,
                                                                                   ix.d_ids);
        VB_CUDA(cudaGetLastError());
        count_launch();
    }
    return VB_OK;
}

// FindInsertPage (src/ivfinsert.c:19-67) for n rows: the list vb_ivf_scan_lists(rows, 1) selects (the fused one-query
// kernel for a few rows, the certified tensor-core pass for batches), except that a row whose distance to centre 0 is NaN
// stays in list 0: the reference's running minimum starts there, and no distance compares smaller than a NaN
static int ivf_insert_lists(Ivf& ix, const void* rows, int64_t n, bool host, int32_t* out) {
    Context& c = ctx();
    const size_t raw = raw_row_bytes(ix.elem, ix.dim);
    const int64_t bq = 65535;
    std::vector<float> d0;
    for (int64_t q0 = 0; q0 < n; q0 += bq) {
        Scratch sc;
        const int64_t m = std::min(bq, n - q0);
        void* qimg;
        size_t qstride;
        VB_TRY(upload_queries(sc, ix.elem, ix.dim, (const uint8_t*)rows + (size_t)q0 * raw, m, host, &qimg, &qstride));
        int32_t* d_lists;
        float* d_ldist;
        float* qn = nullptr;
        if (c.one_query && m <= ONE_MAX_Q && one_probe_fits(ix.lists, qstride, 1))
            VB_TRY(ivf_one_probes(sc, ix, qimg, qstride, m, 1, &d_lists, &d_ldist));
        else
            VB_TRY(ivf_select_probes(sc, ix, IvfPass{}, qimg, qstride, m, &qn, 1, &d_lists, &d_ldist));
        VB_CUDA(cudaMemcpyAsync(out + q0, d_lists, sizeof(int32_t) * (size_t)m, cudaMemcpyDeviceToHost, c.stream));
        if (ix.elem != VB_BIT) {   // (Hamming distances are never NaN)
            void* d_d0;
            VB_TRY(sc.take(sizeof(float) * (size_t)m, &d_d0));
            VB_TRY(launch_scan_regular(ix.centers, key_metric(ix.metric), qimg, qstride, m, 1, (float*)d_d0, 1));
            d0.resize((size_t)m);
            VB_CUDA(cudaMemcpyAsync(d0.data(), d_d0, sizeof(float) * (size_t)m, cudaMemcpyDeviceToHost, c.stream));
        }
        VB_CUDA(cudaStreamSynchronize(c.stream));
        if (ix.elem != VB_BIT)
            for (int64_t i = 0; i < m; ++i)
                if (std::isnan(d0[(size_t)i])) out[q0 + i] = 0;
    }
    return VB_OK;
}

// list offsets and tiles of the changed image, and its planes re-packed from the tile of row `first` on
static int ivf_finish_update(Ivf& ix, const std::vector<int64_t>& new_off, int64_t first, bool whole, bool whole8, unsigned* d_stats) {
    // the move kernels still read the old offsets from d_list_off, which ivf_set_layout overwrites with a copy that is
    // not ordered after the library stream's work
    VB_CUDA(cudaStreamSynchronize(ctx().stream));
    VB_TRY(ivf_set_layout(ix, new_off.data(), false));
    if (ix.tc.planes) {
        VB_TRY(list_tc_repack(ix.rows, &ix.tc, whole ? 0 : first / 128, whole8 ? 0 : first / 128, d_stats));
        VB_TRY(ivf_build_units(ix));
        // level P's projections from the first changed row on; the basis stays (any basis is valid, a stale one looser)
        VB_TRY(list_proj_update(ix.rows, &ix.lp, first));
    } else {
        list_proj_release(&ix.lp);   // built again with the planes
    }
    VB_CUDA(cudaStreamSynchronize(ctx().stream));
    return VB_OK;
}

static size_t align256(size_t b) { return (b + 255) & ~(size_t)255; }

static int ivf_insert_impl(const char* fn, vb_ivf* h, const void* rows, const int64_t* ids, int64_t n, int32_t* out_lists, bool host) {
    VB_TRY(require_init());
    VB_REQUIRE(h, "%s: null index", fn);
    if (!h->ix.loaded) {
        set_error("%s: index not loaded", fn);
        return VB_ESTATE;
    }
    if (!h->ix.has_ids) {
        set_error("%s: the index was loaded without heap ids", fn);
        return VB_ESTATE;
    }
    VB_REQUIRE(n >= 0, "%s: negative row count %lld", fn, (long long)n);
    if (n == 0) return VB_OK;
    VB_REQUIRE(rows && ids, "%s: rows and ids must not be NULL", fn);
    Ivf& ix = h->ix;
    Context& c = ctx();
    const int64_t n_old = ix.rows.n, n_new = n_old + n;
    const size_t stride = ix.rows.stride, raw = raw_row_bytes(ix.elem, ix.dim);
    std::vector<int32_t> lists((size_t)n);
    VB_TRY(ivf_insert_lists(ix, rows, n, host, lists.data()));
    if (out_lists) memcpy(out_lists, lists.data(), sizeof(int32_t) * (size_t)n);
    // placement: appended to its list, rows of the call in call order
    const int L = ix.lists;
    std::vector<int64_t> cnt((size_t)L, 0), shift((size_t)L), new_off((size_t)L + 1), fill((size_t)L);
    for (int32_t l : lists) ++cnt[(size_t)l];
    int64_t before = 0;
    int lmin = L;
    for (int l = 0; l < L; ++l) {
        shift[(size_t)l] = before;
        new_off[(size_t)l] = ix.h_list_off[(size_t)l] + before;
        fill[(size_t)l] = ix.h_list_off[(size_t)l + 1] + before;   // the new rows of list l start at its old end, moved
        before += cnt[(size_t)l];
        if (cnt[(size_t)l] && lmin == L) lmin = l;
    }
    new_off[(size_t)L] = n_new;
    const int64_t first = ix.h_list_off[(size_t)lmin + 1];         // rows before the end of the first list that grows stay
    std::vector<int64_t> dst_new((size_t)n);
    for (int64_t i = 0; i < n; ++i) dst_new[(size_t)i] = fill[(size_t)lists[(size_t)i]]++;
    // reserve and allocate everything before a row moves
    const int64_t suffix = n_old - first;
    const int64_t window = std::max<int64_t>(1, std::min<int64_t>(suffix, (int64_t)(IVF_MOVE_WINDOW_BYTES / stride)));
    const size_t tmp_bytes = align256(8 * (size_t)(suffix + n)) + align256(8 * (size_t)L) + align256(16) +
                             (suffix > 0 ? align256((size_t)window * stride) + align256(8 * (size_t)window) : 0) + align256((size_t)n * stride) +
                             (host ? align256(8 * (size_t)n) : 0);
    const int64_t ids_cap = ix.ids_cap < 0 ? n_old : ix.ids_cap;
    if (n_new > ix.rows.cap || n_new > ids_cap) {
        // growth by half again: release the packed planes first when the larger table does not fit beside them (the
        // next batched scan rebuilds them, if they fit then)
        const int64_t ncap = std::max(n_new, ix.rows.cap + ix.rows.cap / 2);
        const size_t grow = (size_t)ncap * (stride + 8) + tmp_bytes;
        size_t free_b = 0, total_b = 0;
        VB_CUDA(cudaMemGetInfo(&free_b, &total_b));
        if (free_b < grow + ((size_t)1 << 30) && ix.tc.planes) {
            list_tc_release(&ix.tc);
            ix.tc_cap_tiles = ix.tc_cap_tiles8 = 0;
        }
        const int rc = table_reserve(ix.rows, n_new);
        if (rc != VB_OK) {
            set_error("%s: growing the row table to %lld rows (%zu bytes) failed", fn, (long long)n_new, (size_t)n_new * stride);
            return rc;
        }
        int64_t* nid = nullptr;
        if (cudaMalloc(&nid, sizeof(int64_t) * (size_t)ix.rows.cap) != cudaSuccess) {
            cudaGetLastError();
            set_error("%s: allocation of %zu bytes for the heap ids failed", fn, sizeof(int64_t) * (size_t)ix.rows.cap);
            return VB_ENOMEM;
        }
        if (n_old) VB_CUDA(cudaMemcpyAsync(nid, ix.d_ids, sizeof(int64_t) * (size_t)n_old, cudaMemcpyDeviceToDevice, c.stream));
        VB_CUDA(cudaStreamSynchronize(c.stream));
        if (ix.d_ids) cudaFree(ix.d_ids);
        ix.d_ids = nid;
        ix.ids_cap = ix.rows.cap;
    }
    Scratch sc(fn);
    void* tmp;
    VB_TRY(sc.own(tmp_bytes, &tmp));
    uint8_t* p = (uint8_t*)tmp;
    auto take = [&](size_t b) {
        uint8_t* q = p;
        p += align256(b);
        return q;
    };
    int64_t* d_dst = (int64_t*)take(8 * (size_t)(suffix + n));   // the suffix's destinations, then the new rows'
    int64_t* d_shift = (int64_t*)take(8 * (size_t)L);
    unsigned* d_stats = (unsigned*)take(16);
    uint8_t* stage = suffix > 0 ? take((size_t)window * stride) : nullptr;
    int64_t* stage_ids = suffix > 0 ? (int64_t*)take(8 * (size_t)window) : nullptr;
    uint8_t* d_rows = take((size_t)n * stride);
    const int64_t* d_new_ids = host ? (const int64_t*)take(8 * (size_t)n) : ids;
    bool whole = false, whole8 = false;
    if (ix.tc.planes && !list_tc_reserve(&ix.tc, (n_new + 127) / 128, &ix.tc_cap_tiles, &ix.tc_cap_tiles8, &whole, &whole8))
        ix.tc_cap_tiles = ix.tc_cap_tiles8 = 0;
    // the new rows at the table's stride, their ids and destinations
    if (raw != stride) VB_CUDA(cudaMemsetAsync(d_rows, 0, (size_t)n * stride, c.stream));
    VB_CUDA(cudaMemcpy2DAsync(d_rows, stride, rows, raw, raw, (size_t)n, host ? cudaMemcpyHostToDevice : cudaMemcpyDeviceToDevice, c.stream));
    if (host) VB_CUDA(cudaMemcpyAsync((void*)d_new_ids, ids, 8 * (size_t)n, cudaMemcpyHostToDevice, c.stream));
    VB_CUDA(cudaMemcpyAsync(d_dst + suffix, dst_new.data(), 8 * (size_t)n, cudaMemcpyHostToDevice, c.stream));
    VB_CUDA(cudaMemcpyAsync(d_shift, shift.data(), 8 * (size_t)L, cudaMemcpyHostToDevice, c.stream));
    VB_CUDA(cudaStreamSynchronize(c.stream));   // (host vectors)
    ++ix.generation;
    auto move = [&]() -> int {
        if (suffix > 0) {
            ivf_insert_dst_kernel<<<(unsigned)((suffix + 255) / 256), 256, 0, c.stream>>>(ix.d_list_off, L, d_shift, first, n_old, d_dst);
            VB_CUDA(cudaGetLastError());
            count_launch();
            VB_TRY(ivf_move_suffix(ix, first, n_old, d_dst, true, stage, stage_ids, window));
        }
        ivf_move_rows_kernel<<<(unsigned)((n * 32 + 255) / 256), 256, 0, c.stream>>>(d_rows, d_new_ids, n, d_dst + suffix, stride, ix.rows.d,
                                                                                    ix.d_ids);
        VB_CUDA(cudaGetLastError());
        count_launch();
        ix.rows.n = n_new;
        return ivf_finish_update(ix, new_off, first, whole, whole8, d_stats);
    };
    const int rc = move();
    if (rc != VB_OK) ix.loaded = false;   // rows may have moved: the image must be loaded again
    return rc;
}

int vb_ivf_insert(vb_ivf* h, const void* rows, const int64_t* ids, int64_t n, int32_t* out_lists) {
    VB_REQUIRE(out_lists || n <= 0, "vb_ivf_insert: out_lists must not be NULL");
    return ivf_insert_impl("vb_ivf_insert", h, rows, ids, n, out_lists, true);
}

int vb_ivf_insert_dev(vb_ivf* h, const void* rows_dev, const int64_t* ids_dev, int64_t n, int32_t* out_lists) {
    return ivf_insert_impl("vb_ivf_insert_dev", h, rows_dev, ids_dev, n, out_lists, false);
}

int vb_ivf_delete(vb_ivf* h, const int64_t* ids, int64_t n, int64_t* out_removed) {
    VB_TRY(require_init());
    const char* fn = "vb_ivf_delete";
    VB_REQUIRE(h, "%s: null index", fn);
    if (!h->ix.loaded) {
        set_error("%s: index not loaded", fn);
        return VB_ESTATE;
    }
    if (!h->ix.has_ids) {
        set_error("%s: the index was loaded without heap ids", fn);
        return VB_ESTATE;
    }
    VB_REQUIRE(n >= 0 && (ids || n == 0), "%s: null ids or negative count %lld", fn, (long long)n);
    if (out_removed) *out_removed = 0;
    Ivf& ix = h->ix;
    Context& c = ctx();
    const int64_t n_old = ix.rows.n;
    if (n == 0 || n_old == 0) return VB_OK;
    // the rows to remove: a row filter of the ids (sorted on the device, one binary search per row, a ballot per bitset
    // word, compacted by a prefix scan), and its per-list counts
    struct FilterHold {
        Filter f;
        ~FilterHold() {
            if (f.mem) cudaStreamSynchronize(ctx().stream);
            filter_release(&f);
        }
    } gone;
    VB_TRY(filter_build_ivf(n_old, ix.d_ids, ix.d_list_off, ix.lists, ids, n, true, &gone.f));
    const int64_t m = gone.f.n;
    if (m == 0) return VB_OK;
    int64_t first = 0;
    VB_CUDA(cudaMemcpy(&first, gone.f.pos, sizeof(int64_t), cudaMemcpyDeviceToHost));
    const int L = ix.lists;
    std::vector<int64_t> new_off((size_t)L + 1);
    for (int l = 0; l <= L; ++l) new_off[(size_t)l] = ix.h_list_off[(size_t)l] - gone.f.h_off[(size_t)l];
    const int64_t suffix = n_old - first;
    const size_t stride = ix.rows.stride;
    const int64_t window = std::max<int64_t>(1, std::min<int64_t>(suffix, (int64_t)(IVF_MOVE_WINDOW_BYTES / stride)));
    Scratch sc(fn);
    void* tmp;
    VB_TRY(sc.own(align256(8 * (size_t)suffix) + align256(16) + align256((size_t)window * stride) + align256(8 * (size_t)window), &tmp));
    int64_t* d_dst = (int64_t*)tmp;
    unsigned* d_stats = (unsigned*)((uint8_t*)tmp + align256(8 * (size_t)suffix));
    uint8_t* stage = (uint8_t*)d_stats + align256(16);
    int64_t* stage_ids = (int64_t*)(stage + align256((size_t)window * stride));
    ++ix.generation;
    auto move = [&]() -> int {
        ivf_delete_dst_kernel<<<(unsigned)((suffix + 255) / 256), 256, 0, c.stream>>>(gone.f.pos, m, first, n_old, d_dst);
        VB_CUDA(cudaGetLastError());
        count_launch();
        VB_TRY(ivf_move_suffix(ix, first, n_old, d_dst, false, stage, stage_ids, window));
        ix.rows.n = n_old - m;
        return ivf_finish_update(ix, new_off, first, false, false, d_stats);
    };
    const int rc = move();
    if (rc != VB_OK) {
        ix.loaded = false;
        return rc;
    }
    if (out_removed) *out_removed = m;
    return VB_OK;
}

int vb_ivf_list_offsets(const vb_ivf* h, int64_t* out) {
    VB_TRY(require_init());
    VB_REQUIRE(h && out, "vb_ivf_list_offsets: null argument");
    if (!h->ix.loaded) {
        set_error("vb_ivf_list_offsets: index not loaded");
        return VB_ESTATE;
    }
    memcpy(out, h->ix.h_list_off.data(), sizeof(int64_t) * ((size_t)h->ix.lists + 1));
    return VB_OK;
}

}  // extern "C"

// ---- CREATE INDEX in one call (ivfflatbuild): samples, k-means, assign, destinations, placement (vb_ivf_build.cu)

constexpr size_t IVF_BUILD_CHUNK_BYTES = (size_t)128 << 20;

// The caller's rows as device memory at the packed row pitch, `chunk` rows at a time.  Device rows are handed out in
// place.  Host rows go through two pinned and two device buffers: the copy of chunk c + 1 is issued on the copy stream
// before the work on chunk c is enqueued on the library stream, and events hand the buffers back and forth.  `pick`
// (host row numbers) streams those rows instead of all of them, gathered row by row into the pinned buffer.
// The pinned buffers are the library's shared, grow-only ones: another host upload (the centres of the k-means, say)
// may free and re-allocate them between two passes, so every pass asks for them again and no pass keeps the pointers.
struct IvfBuildSource {
    const uint8_t* rows;
    const int64_t* ids;
    int64_t n;
    size_t raw;
    bool host;
    int64_t chunk;
    void* pin[2] = {nullptr, nullptr};
    void* dev[2] = {nullptr, nullptr};   // owned by the caller's Scratch, released after the destructor drained the copy stream
    cudaEvent_t copied[2] = {nullptr, nullptr}, done[2] = {nullptr, nullptr};
    bool rows_pinned = false;
    ~IvfBuildSource() {
        for (int b = 0; b < 2; ++b) {
            if (copied[b]) cudaEventDestroy(copied[b]);
            if (done[b]) cudaEventDestroy(done[b]);
        }
        cudaStreamSynchronize(ctx().copy_stream);
    }
    size_t ids_at() const { return align256((size_t)chunk * raw + 16); }   // offset of a chunk's ids in its buffers
    size_t buffer_bytes() const { return ids_at() + 8 * (size_t)chunk; }
    int prepare(Scratch& sc) {
        if (!host) return VB_OK;
        for (int b = 0; b < 2; ++b) {
            VB_TRY(sc.own(buffer_bytes(), &dev[b]));
            VB_CUDA(cudaEventCreateWithFlags(&copied[b], cudaEventDisableTiming));
            VB_CUDA(cudaEventCreateWithFlags(&done[b], cudaEventDisableTiming));
        }
        VB_CUDA(cudaStreamSynchronize(ctx().stream));   // the buffers' stream-ordered allocations precede their copy-stream use
        cudaPointerAttributes attr;
        rows_pinned = cudaPointerGetAttributes(&attr, rows) == cudaSuccess && attr.type == cudaMemoryTypeHost;
        cudaGetLastError();   // (older drivers report an unregistered pointer as an error)
        return VB_OK;
    }
    int issue(int64_t c, const int64_t* pick, int64_t total, bool with_ids) {
        Context& cx = ctx();
        const int b = (int)(c & 1);
        const int64_t r0 = c * chunk, m = std::min(chunk, total - r0);
        VB_CUDA(cudaEventSynchronize(copied[b]));   // the pinned buffer's last copy has left it
        const uint8_t* src = rows + (size_t)r0 * raw;
        if (pick) {
            for (int64_t i = 0; i < m; ++i) memcpy((uint8_t*)pin[b] + (size_t)i * raw, rows + (size_t)pick[r0 + i] * raw, raw);
            src = (const uint8_t*)pin[b];
        } else if (!rows_pinned) {
            memcpy(pin[b], src, (size_t)m * raw);
            src = (const uint8_t*)pin[b];
        }
        VB_CUDA(cudaStreamWaitEvent(cx.copy_stream, done[b], 0));   // the device buffer's last chunk has been worked on
        VB_CUDA(cudaMemcpyAsync(dev[b], src, (size_t)m * raw, cudaMemcpyHostToDevice, cx.copy_stream));
        if (with_ids) {
            memcpy((uint8_t*)pin[b] + ids_at(), ids + r0, 8 * (size_t)m);
            VB_CUDA(cudaMemcpyAsync((uint8_t*)dev[b] + ids_at(), (uint8_t*)pin[b] + ids_at(), 8 * (size_t)m, cudaMemcpyHostToDevice,
                                    cx.copy_stream));
        }
        VB_CUDA(cudaEventRecord(copied[b], cx.copy_stream));
        return VB_OK;
    }
    // work(first row, rows, device rows, device ids) for every chunk, in order
    template <typename F>
    int stream(const int64_t* pick, int64_t total, bool with_ids, F&& work) {
        Context& cx = ctx();
        const int64_t nc = (total + chunk - 1) / chunk;
        if (!host) {
            for (int64_t c = 0; c < nc; ++c)
                VB_TRY(work(c * chunk, std::min(chunk, total - c * chunk), rows + (size_t)(c * chunk) * raw, ids + c * chunk));
            return VB_OK;
        }
        VB_CUDA(cudaStreamSynchronize(cx.copy_stream));   // (the last pass's copies: the buffers may move below)
        VB_TRY(pinned_buffer(buffer_bytes(), &pin[0]));
        VB_TRY(pinned_buffer2(buffer_bytes(), &pin[1]));
        VB_TRY(issue(0, pick, total, with_ids));
        for (int64_t c = 0; c < nc; ++c) {
            const int b = (int)(c & 1);
            if (c + 1 < nc) VB_TRY(issue(c + 1, pick, total, with_ids));
            VB_CUDA(cudaStreamWaitEvent(cx.stream, copied[b], 0));
            VB_TRY(work(c * chunk, std::min(chunk, total - c * chunk), (const uint8_t*)dev[b],
                        (const int64_t*)((const uint8_t*)dev[b] + ids_at())));
            VB_CUDA(cudaEventRecord(done[b], cx.stream));
        }
        return VB_OK;
    }
};

struct TableHold {   // a table freed on every exit unless it was handed on
    Table t;
    ~TableHold() { table_free(t); }
};

static int ivf_build_impl(const char* fn, vb_ivf* h, const void* rows, const int64_t* ids, int64_t n, int normalize,
                          const vb_ivf_build_opts* opts, int32_t* out_lists, int64_t* out_order, int* iters_out, bool host) {
    VB_TRY(require_init());
    VB_REQUIRE(h, "%s: null index", fn);
    VB_REQUIRE(rows && ids, "%s: rows and ids must not be NULL (an image without heap ids cannot take inserts)", fn);
    VB_REQUIRE(n >= 1 && n < (int64_t)INT32_MAX, "%s: row count %lld out of range (1 .. 2^31 - 2)", fn, (long long)n);
    Ivf& ix = h->ix;
    if (comm_world() > 1 || ix.loading) {
        set_error(ix.loading ? "%s: inside vb_ivf_begin_load / vb_ivf_end_load"
                             : "%s: a communicator is active and this image is a shard; the sharded build is not supported", fn);
        return VB_ESTATE;
    }
    VB_REQUIRE(!normalize || (ix.elem != VB_BIT && ix.metric == VB_NEG_IP),
               "%s: normalize is the rule of the cosine opclasses (vector / halfvec, negative inner product)", fn);
    static const vb_ivf_build_opts defaults = {42, 0, nullptr, 0, 0, nullptr, 0};
    const vb_ivf_build_opts& o = opts ? *opts : defaults;
    Context& c = ctx();
    const int L = ix.lists;
    const size_t stride = ix.rows.stride, raw = raw_row_bytes(ix.elem, ix.dim);
    const int km = ix.elem == VB_BIT ? VB_HAMMING : ix.metric == VB_L2_SQUARED ? VB_L2 : VB_SPHERICAL;
    const bool norm_rows = normalize != 0;

    // the sample rows
    std::vector<int64_t> pick;
    int64_t ns;
    if (o.sample_rows) {
        ns = o.n_samples;
        VB_REQUIRE(ns >= 1 && ns <= n, "%s: %lld sample rows for %lld rows", fn, (long long)ns, (long long)n);
        pick.assign(o.sample_rows, o.sample_rows + ns);
        std::vector<int64_t> sorted(pick);
        std::sort(sorted.begin(), sorted.end());
        VB_REQUIRE(sorted.front() >= 0 && sorted.back() < n, "%s: sample row %lld out of range (%lld rows)", fn,
                   (long long)(sorted.front() < 0 ? sorted.front() : sorted.back()), (long long)n);
        const auto dup = std::adjacent_find(sorted.begin(), sorted.end());
        VB_REQUIRE(dup == sorted.end(), "%s: sample row %lld is repeated", fn, dup == sorted.end() ? 0LL : (long long)*dup);
    } else {
        VB_REQUIRE(o.n_samples >= 0, "%s: negative sample count", fn);
        ns = std::min<int64_t>(n, o.n_samples > 0 ? o.n_samples : std::max<int64_t>(50 * (int64_t)L, 10000));   // src/ivfbuild.c:448-455
    }
    VB_REQUIRE(ns >= L, "%s: %lld samples are fewer than %d lists", fn, (long long)ns, L);
    VB_REQUIRE(!o.u || o.first_row >= 0, "%s: first_row must not be negative", fn);

    Scratch sc(fn);
    IvfBuildSource src{(const uint8_t*)rows, ids, n, raw, host, 0};
    const int64_t auto_chunk = std::min<int64_t>((int64_t)1 << 20, std::max<int64_t>(1024, (int64_t)(IVF_BUILD_CHUNK_BYTES / raw)));
    src.chunk = std::min<int64_t>(n, o.chunk_rows > 0 ? o.chunk_rows : auto_chunk);
    VB_TRY(src.prepare(sc));

    // centres: samples (spherical: the usable ones, normalised), seeding, Lloyd -- through the host, as vb_kmeans hands
    // them over (lists x dim elements)
    std::vector<uint8_t> cent(raw * (size_t)L);
    int iters = 0;
    {
        Scratch sample(fn);
        void *t_pick, *t_raw, *t_unit;
        VB_TRY(sample.own(8 * (size_t)ns, &t_pick));
        int64_t* d_pick = (int64_t*)t_pick;
        Table S = ix.rows;   // (element type, dimensions, stride)
        {
            ProfScope span(VB_PROF_BUILD_SAMPLE);
            if (o.sample_rows) {
                VB_CUDA(cudaMemcpyAsync(d_pick, pick.data(), 8 * (size_t)ns, cudaMemcpyHostToDevice, c.stream));
            } else {
                VB_TRY(build_draw_samples(n, ns, o.seed, d_pick));
                if (host) {
                    pick.resize((size_t)ns);
                    VB_CUDA(cudaMemcpyAsync(pick.data(), d_pick, 8 * (size_t)ns, cudaMemcpyDeviceToHost, c.stream));
                    VB_CUDA(cudaStreamSynchronize(c.stream));
                }
            }
            VB_TRY(sample.own((size_t)ns * stride + 16, &t_raw));
            S.d = (uint8_t*)t_raw;
            S.n = S.cap = ns;
            if (host)
                VB_TRY(src.stream(pick.data(), ns, false, [&](int64_t r0, int64_t m, const uint8_t* d_rows, const int64_t*) {
                    return launch_place_rows(ix.elem, ix.dim, false, d_rows, raw, nullptr, nullptr, nullptr, m, S.d + (size_t)r0 * stride, stride,
                                             nullptr, nullptr);
                }));
            else
                VB_TRY(launch_place_rows(ix.elem, ix.dim, false, rows, raw, nullptr, d_pick, nullptr, ns, S.d, stride, nullptr, nullptr));
            if (km == VB_SPHERICAL) {
                // AddSample: a sample that cannot be normalised is dropped, the others are stored as unit vectors
                const size_t b_rows = align256((size_t)ns * stride + 16), b_zero = align256(4 * (size_t)ns);
                VB_TRY(sample.own(b_rows + b_zero + 8 * (size_t)ns, &t_unit));
                int32_t* d_zero = (int32_t*)((uint8_t*)t_unit + b_rows);
                int64_t* d_to = (int64_t*)((uint8_t*)t_unit + b_rows + b_zero);
                int64_t kept = 0;
                VB_TRY(launch_place_rows(ix.elem, ix.dim, true, S.d, stride, nullptr, nullptr, nullptr, ns, nullptr, stride, nullptr, d_zero));
                VB_TRY(build_compact_map(d_zero, ns, d_to, &kept));
                VB_TRY(launch_place_rows(ix.elem, ix.dim, true, S.d, stride, nullptr, nullptr, d_to, ns, (uint8_t*)t_unit, stride, nullptr,
                                         nullptr));
                S.d = (uint8_t*)t_unit;
                S.n = kept;
            }
        }
        VB_REQUIRE(S.n >= L, "%s: %lld usable samples (norm > 0) are fewer than %d lists", fn, (long long)S.n, L);
        VB_REQUIRE(!o.u || o.first_row < S.n, "%s: first_row %lld is not one of the %lld usable samples", fn, (long long)o.first_row,
                   (long long)S.n);
        {
            ProfScope span(VB_PROF_BUILD_SEED);
            VB_TRY(o.u ? kmeans_pp(S, km, cent.data(), L, 0, o.first_row, o.u) : kmeans_pp(S, km, cent.data(), L, o.seed));
        }
        {
            ProfScope span(VB_PROF_BUILD_LLOYD);
            VB_TRY(kmeans_run(S, km, cent.data(), L, o.max_iter, o.seed, nullptr, nullptr, &iters));
        }
    }
    TableHold Cn;
    Cn.t = ix.rows;
    Cn.t.d = nullptr;
    Cn.t.n = Cn.t.cap = 0;
    VB_TRY(table_append_host(Cn.t, cent.data(), L));

    // pass one: the list of every row (4 bytes per row stay); cosine: of the normalised row, -1 for a row of norm 0
    void *t_lists, *t_prep, *t_dst;
    VB_TRY(sc.own(4 * (size_t)n, &t_lists));
    int32_t* d_lists = (int32_t*)t_lists;
    // A chunk is a table as it lies when its rows need no padding or normalisation and start 16-byte aligned.  Tables the
    // library allocates carry 16 spare bytes behind the last row; the caller's device rows carry none, so of those the
    // last row goes through the padded buffer like a chunk that needs preparing, and the row behind every row read in
    // place is the caller's own.
    const bool prep = norm_rows || raw != stride || (!host && ((uintptr_t)rows & 15) != 0);
    if (!host) src.chunk = prep ? std::min(n, auto_chunk) : std::max<int64_t>(n - 1, 1);
    const int64_t prep_rows = prep ? src.chunk : 1;
    const size_t b_prep = align256((size_t)prep_rows * stride + 16);
    VB_TRY(sc.own(b_prep + 4 * (size_t)prep_rows, &t_prep));
    uint8_t* d_prep = (uint8_t*)t_prep;
    int32_t* d_zero = norm_rows ? (int32_t*)(d_prep + b_prep) : nullptr;
    VB_TRY(src.stream(nullptr, n, false, [&](int64_t r0, int64_t m, const uint8_t* d_rows, const int64_t*) {
        ProfScope span(VB_PROF_BUILD_ASSIGN);
        Table X = ix.rows;
        X.d = const_cast<uint8_t*>(d_rows);
        X.n = X.cap = m;
        if (prep || (!host && r0 + m == n)) {
            VB_TRY(launch_place_rows(ix.elem, ix.dim, norm_rows, d_rows, raw, nullptr, nullptr, nullptr, m, d_prep, stride, nullptr, d_zero));
            X.d = d_prep;
        }
        VB_TRY(launch_assign(X, ix.metric, Cn.t, L, d_lists + r0));
        return norm_rows ? build_mark_skipped(d_zero, m, d_lists + r0) : VB_OK;
    }));

    // destinations: list offsets, the image order, and the image row of every row
    VB_TRY(sc.own(2 * align256(8 * (size_t)n), &t_dst));
    int64_t* d_order = (int64_t*)t_dst;
    int64_t* d_dst = (int64_t*)((uint8_t*)t_dst + align256(8 * (size_t)n));
    std::vector<int64_t> off((size_t)L + 1);
    VB_TRY(build_destinations(d_lists, n, L, d_order, d_dst, off.data()));
    const int64_t n_idx = off[(size_t)L];
    for (int l = 0; l < L; ++l)
        VB_REQUIRE(off[(size_t)l + 1] - off[(size_t)l] < (int64_t)INT32_MAX, "%s: list %d would hold too many rows", fn, l);

    // from here on the image changes: the old rows go before the new table is allocated
    ++ix.generation;
    ix.loaded = false;
    table_free(ix.rows);
    if (ix.d_ids) cudaFree(ix.d_ids);
    ix.d_ids = nullptr;
    ix.has_ids = false;
    list_tc_release(&ix.tc);
    list_tc_release(&ix.ctc);
    list_proj_release(&ix.lp);
    table_free(ix.centers);
    ix.centers = Cn.t;
    Cn.t.d = nullptr;
    if (table_reserve(ix.rows, std::max<int64_t>(n_idx, 1)) != VB_OK) {
        set_error("%s: allocation of %zu bytes of device memory for the row table failed", fn, (size_t)std::max<int64_t>(n_idx, 1) * stride + 16);
        return VB_ENOMEM;
    }
    if (n_idx > 0 && cudaMalloc(&ix.d_ids, 8 * (size_t)n_idx) != cudaSuccess) {
        cudaGetLastError();
        ix.d_ids = nullptr;
        set_error("%s: allocation of %zu bytes of device memory for the heap ids failed", fn, 8 * (size_t)n_idx);
        return VB_ENOMEM;
    }
    // pass two: every row moves once -- host rows scattered chunk by chunk to their image rows, device rows gathered in
    // image order
    if (!host) src.chunk = n;
    VB_TRY(src.stream(nullptr, n, true, [&](int64_t r0, int64_t m, const uint8_t* d_rows, const int64_t* d_ids) {
        ProfScope span(VB_PROF_BUILD_PLACE);
        return host ? launch_place_rows(ix.elem, ix.dim, norm_rows, d_rows, raw, d_ids, nullptr, d_dst + r0, m, ix.rows.d, stride,
                                                ix.d_ids, nullptr)
                            : launch_place_rows(ix.elem, ix.dim, norm_rows, d_rows, raw, d_ids, d_order, nullptr, n_idx, ix.rows.d, stride,
                                                ix.d_ids, nullptr);
    }));
    if (out_lists) VB_CUDA(cudaMemcpyAsync(out_lists, d_lists, 4 * (size_t)n, cudaMemcpyDeviceToHost, c.stream));
    if (out_order) VB_CUDA(cudaMemcpyAsync(out_order, d_order, 8 * (size_t)n, cudaMemcpyDeviceToHost, c.stream));
    VB_CUDA(cudaStreamSynchronize(c.stream));
    if (out_order) std::fill(out_order + n_idx, out_order + n, (int64_t)-1);
    ix.rows.n = n_idx;
    VB_TRY(ivf_set_offsets(ix, off.data()));
    ix.has_ids = true;
    ix.loaded = true;
    if (iters_out) *iters_out = iters;
    return VB_OK;
}

extern "C" {

int vb_ivf_build(vb_ivf* h, const void* rows, const int64_t* ids, int64_t n, int normalize, const vb_ivf_build_opts* opts,
                 int32_t* out_lists, int64_t* out_order, int* iters_out) {
    return ivf_build_impl("vb_ivf_build", h, rows, ids, n, normalize, opts, out_lists, out_order, iters_out, true);
}

int vb_ivf_build_dev(vb_ivf* h, const void* rows_dev, const int64_t* ids_dev, int64_t n, int normalize, const vb_ivf_build_opts* opts,
                     int32_t* out_lists, int64_t* out_order, int* iters_out) {
    return ivf_build_impl("vb_ivf_build_dev", h, rows_dev, ids_dev, n, normalize, opts, out_lists, out_order, iters_out, false);
}

int vb_ivf_centers(const vb_ivf* h, void* out) {
    VB_TRY(require_init());
    VB_REQUIRE(h && out, "vb_ivf_centers: null argument");
    if (!h->ix.loaded) {
        set_error("vb_ivf_centers: index not loaded");
        return VB_ESTATE;
    }
    const Ivf& ix = h->ix;
    const size_t raw = raw_row_bytes(ix.elem, ix.dim);
    VB_CUDA(cudaMemcpy2DAsync(out, raw, ix.centers.d, ix.centers.stride, raw, (size_t)ix.lists, cudaMemcpyDeviceToHost, ctx().stream));
    VB_CUDA(cudaStreamSynchronize(ctx().stream));
    return VB_OK;
}

int vb_ivf_free(vb_ivf* h) {
    if (!h) return VB_OK;
    table_free(h->ix.centers);
    table_free(h->ix.rows);
    if (h->ix.d_ids) cudaFree(h->ix.d_ids);
    if (h->ix.d_list_off) cudaFree(h->ix.d_list_off);
    if (h->ix.d_cand_sum) cudaFree(h->ix.d_cand_sum);
    if (h->ix.d_tiles) cudaFree(h->ix.d_tiles);
    list_tc_release(&h->ix.tc);
    list_tc_release(&h->ix.ctc);
    if (h->ix.d_centre_off) cudaFree(h->ix.d_centre_off);
    if (h->ix.d_tc_fail) cudaFree(h->ix.d_tc_fail);
    if (h->ix.d_l0_fail) cudaFree(h->ix.d_l0_fail);
    for (void* b : h->ix.d_repair)
        if (b) cudaFree(b);
    list_proj_release(&h->ix.lp);
    if (h->ix.d_ticket) cudaFree(h->ix.d_ticket);
    for (int i = 0; i < 2; ++i) {
        if (h->ix.q_buf[i]) cudaFree(h->ix.q_buf[i]);
        if (h->ix.q_ready[i]) cudaEventDestroy(h->ix.q_ready[i]);
    }
    if (h->ix.q_stream) cudaStreamDestroy(h->ix.q_stream);
    delete h;
    return VB_OK;
}

int vb_ivf_scan_lists(vb_ivf* h, const void* queries, int64_t nq, int max_probes, int32_t* out_lists, double* out_dist) {
    VB_TRY(require_init());
    VB_REQUIRE(h && h->ix.loaded, "index not loaded");
    VB_REQUIRE(max_probes >= 1, "max_probes must be >= 1");
    Ivf& ix = h->ix;
    Context& c = ctx();
    int probes = std::min(max_probes, ix.lists);  // src/ivfscan.c:279-283
    if (nq <= 0) return VB_OK;
    if (queries == nullptr) {
        // NULL query: every centre at distance 0; with this library's tie rule the first lists win
        for (int64_t q = 0; q < nq; ++q)
            for (int p = 0; p < probes; ++p) {
                out_lists[q * max_probes + p] = p;
                if (out_dist) out_dist[q * max_probes + p] = 0.0;
            }
        return VB_OK;
    }
    Scratch sc;
    void* qimg;
    size_t qstride;
    VB_TRY(upload_queries(sc, ix.elem, ix.dim, queries, nq, true, &qimg, &qstride));
    int32_t* d_lists;
    float* d_ldist;
    if (c.one_query && nq <= ONE_MAX_Q && one_probe_fits(ix.lists, qstride, probes)) {
        // one backend, one scan: distances to the centres and the selection in a single launch; list numbers and
        // distances (adjacent in the scratch) come back with one copy
        VB_TRY(ivf_one_probes(sc, ix, qimg, qstride, nq, probes, &d_lists, &d_ldist));
        void* pin;
        const size_t np = (size_t)nq * probes;
        VB_TRY(pinned_buffer2(8 * np, &pin));
        VB_CUDA(cudaMemcpyAsync(pin, d_lists, 8 * np, cudaMemcpyDeviceToHost, c.stream));
        VB_CUDA(cudaStreamSynchronize(c.stream));
        const int32_t* pl = (const int32_t*)pin;
        const float* pd = (const float*)(pl + np);
        for (int64_t q = 0; q < nq; ++q)
            for (int p = 0; p < max_probes; ++p) {
                const bool have = p < probes;
                out_lists[q * max_probes + p] = have ? pl[(size_t)(q * probes + p)] : -1;
                if (out_dist) out_dist[q * max_probes + p] = have ? (double)pd[(size_t)(q * probes + p)] : INFINITY;
            }
        return VB_OK;
    }
    float* qn = nullptr;
    VB_TRY(ivf_select_probes(sc, ix, IvfPass{}, qimg, qstride, nq, &qn, probes, &d_lists, &d_ldist));
    std::vector<int32_t> hl((size_t)nq * probes);
    std::vector<float> hd((size_t)nq * probes);
    VB_CUDA(cudaMemcpyAsync(hl.data(), d_lists, sizeof(int32_t) * hl.size(), cudaMemcpyDeviceToHost, c.stream));
    VB_CUDA(cudaMemcpyAsync(hd.data(), d_ldist, sizeof(float) * hd.size(), cudaMemcpyDeviceToHost, c.stream));
    VB_CUDA(cudaStreamSynchronize(c.stream));
    for (int64_t q = 0; q < nq; ++q)
        for (int p = 0; p < max_probes; ++p) {
            bool have = p < probes;
            out_lists[q * max_probes + p] = have ? hl[(size_t)(q * probes + p)] : -1;
            if (out_dist) out_dist[q * max_probes + p] = have ? (double)hd[(size_t)(q * probes + p)] : INFINITY;
        }
    return VB_OK;
}

int vb_ivf_scan_items(vb_ivf* h, const void* q, const int32_t* lists, int nlists, int64_t cap, int64_t* out_ids, double* out_dist,
                      int64_t* n_out) {
    VB_TRY(require_init());
    VB_REQUIRE(h && h->ix.loaded, "index not loaded");
    VB_REQUIRE(nlists >= 0 && lists && n_out, "bad arguments");
    Ivf& ix = h->ix;
    Context& c = ctx();
    int64_t total = 0;
    for (int i = 0; i < nlists; ++i) {
        VB_REQUIRE(lists[i] >= 0 && lists[i] < ix.lists, "list %d out of range", lists[i]);
        total += ix.h_list_off[(size_t)lists[i] + 1] - ix.h_list_off[(size_t)lists[i]];
    }
    *n_out = total;
    int64_t k = std::min(cap, total);
    if (k <= 0) return VB_OK;
    if (q == nullptr) {
        // NULL query: all distances 0, every probed row returned in scan order (src/ivfscan.c:207-211)
        std::vector<int64_t> hid;
        int64_t w = 0;
        for (int i = 0; i < nlists && w < k; ++i) {
            int64_t lo = ix.h_list_off[(size_t)lists[i]], hi = ix.h_list_off[(size_t)lists[i] + 1];
            int64_t m = std::min(hi - lo, k - w);
            if (ix.d_ids) VB_CUDA(cudaMemcpy(out_ids + w, ix.d_ids + lo, sizeof(int64_t) * (size_t)m, cudaMemcpyDeviceToHost));
            else
                for (int64_t j = 0; j < m; ++j) out_ids[w + j] = lo + j;
            for (int64_t j = 0; j < m; ++j) out_dist[w + j] = 0.0;
            w += m;
        }
        return VB_OK;
    }
    VB_REQUIRE(k < (int64_t)INT32_MAX, "too many candidates");
    Scratch sc;
    void* qimg;
    size_t qstride;
    VB_TRY(upload_queries(sc, ix.elem, ix.dim, q, 1, true, &qimg, &qstride));
    void* d_misc;
    VB_TRY(sc.take(sizeof(int32_t) * (size_t)nlists, &d_misc));
    void* d_out;
    VB_TRY(sc.take((sizeof(int64_t) + sizeof(double)) * (size_t)k, &d_out));
    int64_t* o_ids = (int64_t*)d_out;
    double* o_d = (double*)(o_ids + k);
    if (ivf_one_applies(ix, 1, nlists, k, total)) {
        // distances, selection, heap ids and the operator's epilogue in one launch.  The list numbers go out through the
        // second pinned buffer (no synchronisation), the results come back through it with one copy.
        void* pin;
        VB_TRY(pinned_buffer2(std::max(sizeof(int32_t) * (size_t)nlists, 16 * (size_t)k), &pin));
        memcpy(pin, lists, sizeof(int32_t) * (size_t)nlists);
        VB_CUDA(cudaMemcpyAsync(d_misc, pin, sizeof(int32_t) * (size_t)nlists, cudaMemcpyHostToDevice, c.stream));
        VB_TRY(ivf_one_items(ix, qimg, qstride, 1, (const int32_t*)d_misc, nlists, (int)k, total, o_ids, nullptr, o_d, true));
        ix.last_cand = -1;
        ix.last_bytes = 1;
        return ivf_one_fetch(d_out, k, out_ids, out_dist);
    }
    VB_CUDA(cudaMemcpyAsync(d_misc, lists, sizeof(int32_t) * (size_t)nlists, cudaMemcpyHostToDevice, c.stream));
    VB_CUDA(cudaStreamSynchronize(c.stream));
    float* qn = nullptr;
    // capacity bound: these particular lists
    VB_TRY(ivf_scan_topk(sc, ix, IvfPass{}, qimg, qstride, 1, &qn, (const int32_t*)d_misc, nlists, std::max<int64_t>(total, 1), (int)k, o_ids,
                         nullptr, o_d));
    VB_CUDA(cudaMemcpyAsync(out_ids, o_ids, sizeof(int64_t) * (size_t)k, cudaMemcpyDeviceToHost, c.stream));
    VB_CUDA(cudaMemcpyAsync(out_dist, o_d, sizeof(double) * (size_t)k, cudaMemcpyDeviceToHost, c.stream));
    VB_CUDA(cudaStreamSynchronize(c.stream));
    return VB_OK;
}

__global__ void gather_queries_kernel(const uint8_t* __restrict__ src, size_t row_bytes, const int32_t* __restrict__ idx,
                                      uint8_t* __restrict__ dst) {
    const uint8_t* s = src + (size_t)idx[blockIdx.x] * row_bytes;
    uint8_t* d = dst + (size_t)blockIdx.x * row_bytes;
    for (size_t i = threadIdx.x; i < row_bytes; i += blockDim.x) d[i] = s[i];
}
__global__ void scatter_results_kernel(const int64_t* __restrict__ ids, const float* __restrict__ dist, const int32_t* __restrict__ idx,
                                       int64_t n, int k, int64_t* __restrict__ out_ids, float* __restrict__ out_f) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= n * k) return;
    const int64_t o = (int64_t)idx[i / k] * k + i % k;
    out_ids[o] = ids[i];
    out_f[o] = dist[i];
}

// the row filters of a vb_ivf_search_filtered call (validated): query q of the call uses filters[fq ? fq[q] : 0]
struct IvfFilterSpec {
    const vb_filter* const* filters;
    int nfilters;
    const int32_t* fq;   // host
};

static int ivf_search_impl(vb_ivf* h, const void* queries, int64_t nq, int probes, int k, bool host, bool q_host, int64_t* out_ids,
                           float* out_f, double* out_d, bool repair = false, const IvfFilterSpec* filt = nullptr, int repair_from = 1);

// the mask arguments of queries [q0, q0 + m) of a filtered call (in sc): the filters' positions and runs, in place
static int ivf_upload_mask(Scratch& sc, const IvfFilterSpec& filt, int64_t q0, int64_t m, IvfMask* mk) {
    Context& c = ctx();
    const size_t tab = ((sizeof(MaskFilter) * (size_t)filt.nfilters) + 15) & ~(size_t)15;
    void* d;
    VB_TRY(sc.take(tab + 2 * sizeof(int32_t) * (size_t)m, &d));
    std::vector<MaskFilter> h((size_t)filt.nfilters);
    for (int i = 0; i < filt.nfilters; ++i) h[(size_t)i] = MaskFilter{filt.filters[i]->f.pos, filt.filters[i]->f.off};
    VB_CUDA(cudaMemcpyAsync(d, h.data(), sizeof(MaskFilter) * h.size(), cudaMemcpyHostToDevice, c.stream));
    int32_t* fq = (int32_t*)((uint8_t*)d + tab);
    if (filt.fq) VB_CUDA(cudaMemcpyAsync(fq, filt.fq + q0, sizeof(int32_t) * (size_t)m, cudaMemcpyHostToDevice, c.stream));
    mk->filters = (const MaskFilter*)d;
    mk->fq = filt.fq ? fq : nullptr;
    mk->has_nan = fq + m;
    return VB_OK;
}

// The queries `fail` (numbers within `queries`, nf of them) that level 0 (level P) could not certify are searched again on
// their own, from level 1 (level 0) on -- `from` -- and their rows of the outputs overwritten.  The re-run takes the batched filter chain whatever its size
// (not the fused one-query kernels): a query certified at level 1 or 2 carries the filter's exact re-score, as it would in
// a batch-wide repeat.  When the re-run needs the exact kernels, the caller computes the whole sub-batch there instead,
// as it does without level 0 (the list-major kernel's sums may differ from the re-score's in the last bit).
// (filt: the row filters of `queries`, whose failed queries' entries of filter_of_query go along)
static int ivf_repair_level0(vb_ivf* h, const void* queries, std::vector<int32_t>& fail, int probes, int k, bool host, bool q_host,
                             int64_t* out_ids, float* out_f, double* out_d, const IvfFilterSpec* filt, int from) {
    Ivf& ix = h->ix;
    Context& c = ctx();
    std::sort(fail.begin(), fail.end());
    const int64_t nf = (int64_t)fail.size();
    std::vector<int32_t> sub_fq;
    IvfFilterSpec sub_filt;
    if (filt) {
        sub_filt = *filt;
        if (filt->fq) {
            sub_fq.resize((size_t)nf);
            for (int64_t i = 0; i < nf; ++i) sub_fq[(size_t)i] = filt->fq[fail[(size_t)i]];
            sub_filt.fq = sub_fq.data();
        }
        filt = &sub_filt;
    }
    const size_t rawq = raw_row_bytes(ix.elem, ix.dim);
    const size_t q_bytes = (rawq * (size_t)nf + 15) & ~(size_t)15;
    const size_t need = q_bytes + (sizeof(int64_t) + sizeof(float)) * (size_t)nf * k + sizeof(int64_t) + sizeof(int32_t) * (size_t)nf;
    // (a re-run from level 0 may repair its own level-0 failures from level 1 while its buffer is in use: one buffer per level)
    const int slot = from == 0 ? 0 : 1;
    if (ix.repair_bytes[slot] < need) {
        if (ix.d_repair[slot]) VB_CUDA(cudaFree(ix.d_repair[slot]));
        VB_CUDA(cudaMalloc(&ix.d_repair[slot], need));
        ix.repair_bytes[slot] = need;
    }
    uint8_t* d_q = (uint8_t*)ix.d_repair[slot];
    int64_t* d_ids = (int64_t*)(d_q + q_bytes);
    int64_t* d_cand_saved = d_ids + (size_t)nf * k;   // the caller's candidate count: the re-run's scans do not add to it
    float* d_f = (float*)(d_cand_saved + 1);
    int32_t* d_idx = (int32_t*)(d_f + (size_t)nf * k);
    VB_CUDA(cudaMemcpyAsync(d_idx, fail.data(), sizeof(int32_t) * (size_t)nf, cudaMemcpyHostToDevice, c.stream));
    std::vector<uint8_t> hq;
    const void* sub = d_q;
    if (q_host) {
        hq.resize(rawq * (size_t)nf);
        for (int64_t i = 0; i < nf; ++i) memcpy(hq.data() + (size_t)i * rawq, (const uint8_t*)queries + (size_t)fail[(size_t)i] * rawq, rawq);
        sub = hq.data();
    } else {
        gather_queries_kernel<<<(unsigned)nf, 128, 0, c.stream>>>((const uint8_t*)queries, rawq, d_idx, d_q);
        VB_CUDA(cudaGetLastError());
        count_launch();
    }
    VB_CUDA(cudaMemcpyAsync(d_cand_saved, ix.d_cand_sum, sizeof(int64_t), cudaMemcpyDeviceToDevice, c.stream));
    if (host) {
        std::vector<int64_t> ti((size_t)nf * k);
        std::vector<double> td((size_t)nf * k);
        VB_TRY(ivf_search_impl(h, sub, nf, probes, k, true, q_host, ti.data(), nullptr, td.data(), true, filt, from));
        VB_CUDA(cudaMemcpyAsync(ix.d_cand_sum, d_cand_saved, sizeof(int64_t), cudaMemcpyDeviceToDevice, c.stream));
        for (int64_t i = 0; i < nf; ++i) {
            memcpy(out_ids + (size_t)fail[(size_t)i] * k, ti.data() + (size_t)i * k, sizeof(int64_t) * k);
            memcpy(out_d + (size_t)fail[(size_t)i] * k, td.data() + (size_t)i * k, sizeof(double) * k);
        }
        return VB_OK;
    }
    VB_TRY(ivf_search_impl(h, sub, nf, probes, k, false, false, d_ids, d_f, nullptr, true, filt, from));
    VB_CUDA(cudaMemcpyAsync(ix.d_cand_sum, d_cand_saved, sizeof(int64_t), cudaMemcpyDeviceToDevice, c.stream));
    scatter_results_kernel<<<(unsigned)((nf * k + 255) / 256), 256, 0, c.stream>>>(d_ids, d_f, d_idx, nf, k, out_ids, out_f);
    VB_CUDA(cudaGetLastError());
    count_launch();
    return VB_OK;
}

// The certificate repeat policy of one sub-batch of the batched search.  run(pass, fails, &level) computes the sub-batch
// once: the queries its probe selection (fails[0]) and list scan (fails[1]) could not certify, and the list level it ran
// at.  The tensor-core filter runs optimistically: the counters are read back together with the results (one
// synchronisation per pass).  pass is the first, automatic pass: where its level0 (levelp) lets the list scan start at
// level 0 (P), repair(n, from) searches the n queries that level could not certify again on their own, from level `from`.  Otherwise a sub-batch with an
// uncertified query is run again at level 2 when level 1 failed, then on the exact kernels.
static int ivf_certified_batch(Ivf& ix, int probes, IvfPass pass, const std::function<int(const IvfPass&, int*, int*)>& run,
                               const std::function<int(int, int)>& repair) {
    int fails[2], level;
    pass.defer_check = true;
    VB_TRY(run(pass, fails, &level));
    pass.level0 = pass.levelp = false;   // (a repeat never starts at level 0 or P)
    auto exact = [&] {
        pass.mode = IvfPass::EXACT;
        pass.defer_check = false;
        return run(pass, fails, &level);
    };
    if (fails[0] == 0 && fails[1] > 0 && level == LIST_LEVEL_P) {
        // level P could not certify some queries: only those go on, from level 0.  The rule is level 0's: their re-run
        // streams about 1 - (1 - probes / lists)^n of a level-0 pass, and level P saved most of one (it reads 4 r bytes a
        // row instead of dim); past half of it level P no longer pays and rests for the next 64 batches.
        ix.total_lp_failed += fails[1];
        if (1.0 - std::pow(1.0 - (double)probes / ix.lists, (double)fails[1]) > 0.5) ix.lp_cooldown = 64;
        const int64_t exact0 = ix.total_tc_failed;
        VB_TRY(repair(fails[1], 0));
        return ix.total_tc_failed > exact0 ? exact() : VB_OK;   // the re-run needed the exact kernels
    }
    if (fails[0] == 0 && fails[1] > 0 && level == 0) {
        // level 0 could not separate the neighbours of some queries: only those go on, from level 1.  Their re-run
        // streams the lists they probe at level 1: with n failed queries, about 1 - (1 - probes / lists)^n of what a
        // level-1 pass over the batch streams, while level 0 saved half of that pass.  Past a quarter (the re-run also
        // selects probes and synchronises again) level 0 no longer pays, and it rests for the next 64 batches (the data
        // decides this, not the batch).  At 1000 lists and probes 10 that is 29 failed queries.
        ix.total_l0_failed += fails[1];
        if (1.0 - std::pow(1.0 - (double)probes / ix.lists, (double)fails[1]) > 0.25) ix.l0_cooldown = 64;
        const int64_t exact0 = ix.total_tc_failed;
        VB_TRY(repair(fails[1], 1));
        return ix.total_tc_failed > exact0 ? exact() : VB_OK;   // neither level 1 nor 2 certified them
    }
    if (fails[0] == 0 && fails[1] > 0 && level == 1) {
        // the hi-plane filter could not separate the neighbours of some query: both planes, and leave level 1 alone
        // for the next batches (the data decides this, not the batch)
        ix.total_l1_failed += fails[1];
        ix.l1_cooldown = 64;
        pass.mode = IvfPass::LEVEL2;
        VB_TRY(run(pass, fails, &level));
    }
    if (fails[0] + fails[1] > 0) {
        ix.total_tc_failed += fails[0] + fails[1];
        return exact();
    }
    return VB_OK;
}

// host: results go to host memory (int64 ids + float8 distances); q_host: the queries are host memory.  repair: the re-run
// of the queries level 0 or P could not certify (ivf_repair_level0), which starts at level repair_from (0 or 1), never at
// level P, and adds to its caller's candidate count
static int ivf_search_impl(vb_ivf* h, const void* queries, int64_t nq, int probes, int k, bool host, bool q_host, int64_t* out_ids,
                           float* out_f, double* out_d, bool repair, const IvfFilterSpec* filt, int repair_from) {
    VB_TRY(require_init());
    VB_REQUIRE(h && h->ix.loaded, "index not loaded");
    VB_REQUIRE(queries && probes >= 1 && k >= 1, "bad search arguments");
    Ivf& ix = h->ix;
    Context& c = ctx();
    probes = std::min(probes, ix.lists);
    if (nq <= 0) return VB_OK;
    const size_t rawq = raw_row_bytes(ix.elem, ix.dim);
    const int64_t cap = ivf_cap(ix, probes);
    // (the fused one-query kernels select inside the scan: a filtered call takes the general path and its mask)
    if (!repair && !filt && ivf_one_applies(ix, nq, probes, k, cap)) {
        // a handful of queries (one backend's scan): two fused launches, no memsets, one copy back
        Scratch sc;
        void* qimg;
        size_t qstride;
        VB_TRY(upload_queries(sc, ix.elem, ix.dim, queries, nq, q_host, &qimg, &qstride));
        int32_t* d_lists;
        float* d_ldist;
        VB_TRY(ivf_one_probes(sc, ix, qimg, qstride, nq, probes, &d_lists, &d_ldist));
        if (host) {
            void* d_out;
            VB_TRY(sc.take((sizeof(int64_t) + sizeof(double)) * (size_t)nq * k, &d_out));
            int64_t* o_ids = (int64_t*)d_out;
            double* o_d = (double*)(o_ids + (size_t)nq * k);
            VB_TRY(ivf_one_items(ix, qimg, qstride, nq, d_lists, probes, k, cap, o_ids, nullptr, o_d, false));
            VB_TRY(ivf_one_fetch(d_out, nq * k, out_ids, out_d));
        } else {
            VB_TRY(ivf_one_items(ix, qimg, qstride, nq, d_lists, probes, k, cap, out_ids, out_f, nullptr, false));
        }
        ix.last_cand = -1;
        ix.last_bytes = nq;
        return VB_OK;
    }
    const int64_t bq = ivf_batch_limit(ix, probes);
    if (!repair) VB_CUDA(cudaMemsetAsync(ix.d_cand_sum, 0, sizeof(int64_t), c.stream));
    constexpr int L0_LIST_READ = 64;   // failed queries read back with the counters (more take a second copy)
    int32_t l0_list[L0_LIST_READ];
    IvfPass first;
    first.level0 = !repair || repair_from == 0;
    first.levelp = !repair;
    first.repair = repair;
    for (int64_t q0 = 0; q0 < nq; q0 += bq) {
        const int64_t m = std::min(bq, nq - q0);
        auto run = [&](const IvfPass& pass, int* fails, int* level) -> int {
            if (ix.d_tc_fail) VB_CUDA(cudaMemsetAsync(ix.d_tc_fail, 0, 2 * sizeof(int), c.stream));
            Scratch sc;
            void* qimg;
            size_t qstride;
            VB_TRY(upload_queries(sc, ix.elem, ix.dim, (const uint8_t*)queries + (size_t)q0 * rawq, m, q_host, &qimg, &qstride));
            IvfMask mk{};
            if (filt) VB_TRY(ivf_upload_mask(sc, *filt, q0, m, &mk));
            const IvfMask* mask = filt ? &mk : nullptr;
            int32_t* d_lists;
            float* d_ldist;
            float* qn = nullptr;   // |q|^2 of the sub-batch, shared by its probe selection and its list scan
            VB_TRY(ivf_select_probes(sc, ix, pass, qimg, qstride, m, &qn, probes, &d_lists, &d_ldist));
            if (host) {
                void* d_out;
                VB_TRY(sc.take((sizeof(int64_t) + sizeof(double)) * (size_t)m * k, &d_out));
                int64_t* o_ids = (int64_t*)d_out;
                double* o_d = (double*)(o_ids + (size_t)m * k);
                VB_TRY(ivf_scan_topk(sc, ix, pass, qimg, qstride, m, &qn, d_lists, probes, cap, k, o_ids, nullptr, o_d, level, mask));
                VB_CUDA(cudaMemcpyAsync(out_ids + q0 * k, o_ids, sizeof(int64_t) * (size_t)m * k, cudaMemcpyDeviceToHost, c.stream));
                VB_CUDA(cudaMemcpyAsync(out_d + q0 * k, o_d, sizeof(double) * (size_t)m * k, cudaMemcpyDeviceToHost, c.stream));
            } else {
                VB_TRY(ivf_scan_topk(sc, ix, pass, qimg, qstride, m, &qn, d_lists, probes, cap, k, out_ids + q0 * k, out_f + q0 * k, nullptr,
                                     level, mask));
            }
            fails[0] = fails[1] = 0;
            const bool check = pass.defer_check && ix.d_tc_fail != nullptr;
            if (check) VB_CUDA(cudaMemcpyAsync(fails, ix.d_tc_fail, 2 * sizeof(int), cudaMemcpyDeviceToHost, c.stream));
            if (check && (*level == 0 || *level == LIST_LEVEL_P))
                VB_CUDA(cudaMemcpyAsync(l0_list, ix.d_l0_fail, sizeof(int32_t) * (size_t)std::min<int64_t>(m, L0_LIST_READ),
                                        cudaMemcpyDeviceToHost, c.stream));
            if (host || check) VB_CUDA(cudaStreamSynchronize(c.stream));
            return VB_OK;
        };
        auto repair_level0 = [&](int n_failed, int from) -> int {
            std::vector<int32_t> fail(l0_list, l0_list + std::min(n_failed, L0_LIST_READ));
            if (n_failed > L0_LIST_READ) {
                fail.resize((size_t)n_failed);
                VB_CUDA(cudaMemcpy(fail.data(), ix.d_l0_fail, sizeof(int32_t) * (size_t)n_failed, cudaMemcpyDeviceToHost));
            }
            IvfFilterSpec sub_filt;
            if (filt) {
                sub_filt = *filt;
                if (filt->fq) sub_filt.fq = filt->fq + q0;
            }
            return ivf_repair_level0(h, (const uint8_t*)queries + (size_t)q0 * rawq, fail, probes, k, host, q_host, out_ids + q0 * k,
                                     out_f ? out_f + q0 * k : nullptr, out_d ? out_d + q0 * k : nullptr, filt ? &sub_filt : nullptr, from);
        };
        VB_TRY(ivf_certified_batch(ix, probes, first, run, repair_level0));
    }
    ix.last_cand = -1;  // fetched lazily
    ix.last_bytes = nq;
    return VB_OK;
}

int vb_ivf_search(vb_ivf* h, const void* queries, int64_t nq, int probes, int k, int64_t* out_ids, double* out_dist) {
    return ivf_search_impl(h, queries, nq, probes, k, true, true, out_ids, nullptr, out_dist);
}
int vb_ivf_search_dev(vb_ivf* h, const void* queries_dev, int64_t nq, int probes, int k, int64_t* out_ids_dev, float* out_dist_dev) {
    return ivf_search_impl(h, queries_dev, nq, probes, k, false, false, out_ids_dev, out_dist_dev, nullptr);
}

}  // extern "C"

// vb_ivf_search with a row filter per query: the arguments are checked as the filtered handle checks them, then the
// batched search runs with its runs masked.  The host variant searches into staging buffers and copies them out only
// when the whole call succeeded.
static int ivf_search_filtered_impl(const char* fn, vb_ivf* h, const void* queries, int64_t nq, int probes, int k,
                                    const vb_filter* const* filters, int nfilters, const int32_t* filter_of_query, bool host,
                                    int64_t* out_ids, float* out_f, double* out_d) {
    VB_TRY(require_init());
    if (!h || !h->ix.loaded) {
        set_error("%s: index not loaded", fn);
        return VB_ESTATE;
    }
    Ivf& ix = h->ix;
    VB_REQUIRE(queries, "%s: queries must not be NULL", fn);
    VB_REQUIRE(probes >= 1 && k >= 1, "%s: probes and k must be >= 1 (got %d, %d)", fn, probes, k);
    VB_REQUIRE(filters && nfilters >= 1, "%s: no row filter given", fn);
    VB_REQUIRE(filter_of_query || nfilters == 1, "%s: filter_of_query may only be NULL with one filter (got %d)", fn, nfilters);
    for (int i = 0; i < nfilters; ++i) {
        VB_REQUIRE(filters[i], "%s: filter %d is NULL", fn, i);
        const Filter& f = filters[i]->f;
        VB_REQUIRE(f.kind == FILTER_IVF && f.owner == h && f.owner_uid == h->uid, "%s: filter %d was made for another table or index", fn, i);
        if (f.generation != ix.generation) {
            set_error("%s: filter %d: index changed since the filter was created", fn, i);
            return VB_ESTATE;
        }
    }
    for (int64_t q = 0; q < nq && filter_of_query; ++q)
        VB_REQUIRE(filter_of_query[q] >= 0 && filter_of_query[q] < nfilters, "%s: filter_of_query[%lld] = %d, not in 0..%d", fn,
                   (long long)q, filter_of_query[q], nfilters - 1);
    if (nq <= 0) return VB_OK;
    VB_REQUIRE(out_ids && (out_f || out_d), "%s: null output", fn);
    const IvfFilterSpec filt{filters, nfilters, nfilters > 1 ? filter_of_query : nullptr};
    if (!host) return ivf_search_impl(h, queries, nq, probes, k, false, false, out_ids, out_f, nullptr, false, &filt);
    std::vector<int64_t> ids((size_t)nq * k);
    std::vector<double> dist((size_t)nq * k);
    VB_TRY(ivf_search_impl(h, queries, nq, probes, k, true, true, ids.data(), nullptr, dist.data(), false, &filt));
    memcpy(out_ids, ids.data(), sizeof(int64_t) * ids.size());
    memcpy(out_d, dist.data(), sizeof(double) * dist.size());
    return VB_OK;
}

extern "C" {

int vb_ivf_search_filtered(vb_ivf* h, const void* queries, int64_t nq, int probes, int k, const vb_filter* const* filters, int nfilters,
                           const int32_t* filter_of_query, int64_t* out_ids, double* out_dist) {
    return ivf_search_filtered_impl("vb_ivf_search_filtered", h, queries, nq, probes, k, filters, nfilters, filter_of_query, true, out_ids,
                                    nullptr, out_dist);
}
int vb_ivf_search_filtered_dev(vb_ivf* h, const void* queries_dev, int64_t nq, int probes, int k, const vb_filter* const* filters,
                               int nfilters, const int32_t* filter_of_query, int64_t* out_ids_dev, float* out_dist_dev) {
    return ivf_search_filtered_impl("vb_ivf_search_filtered_dev", h, queries_dev, nq, probes, k, filters, nfilters, filter_of_query, false,
                                    out_ids_dev, out_dist_dev, nullptr);
}

// Pipelined host path: the queries of the NEXT call are copied to the device on a second stream while the current
// call computes.  Two slots; a slot is reusable once the search that read it has been synchronised (it has, when
// vb_ivf_search_prefetched returns).
int vb_ivf_prefetch_queries(vb_ivf* h, const void* queries, int64_t nq, int slot) {
    VB_TRY(require_init());
    VB_REQUIRE(h && h->ix.loaded && queries && nq > 0 && (slot == 0 || slot == 1), "bad prefetch arguments");
    Ivf& ix = h->ix;
    const size_t raw = raw_row_bytes(ix.elem, ix.dim);
    VB_REQUIRE(ix.elem == VB_VECTOR && raw == padded_row_bytes(ix.elem, ix.dim),
               "query prefetch needs vector queries whose dimension is a multiple of 4 (use vb_ivf_search otherwise)");
    if (!ix.q_stream) {
        VB_CUDA(cudaStreamCreateWithFlags(&ix.q_stream, cudaStreamNonBlocking));
        for (int i = 0; i < 2; ++i) VB_CUDA(cudaEventCreateWithFlags(&ix.q_ready[i], cudaEventDisableTiming));
    }
    const size_t bytes = raw * (size_t)nq;
    if (ix.q_bytes[slot] < bytes) {
        if (ix.q_buf[slot]) {
            VB_CUDA(cudaStreamSynchronize(ctx().stream));
            VB_CUDA(cudaFree(ix.q_buf[slot]));
            ix.q_buf[slot] = nullptr;
            ix.q_bytes[slot] = 0;
        }
        VB_CUDA(cudaMalloc(&ix.q_buf[slot], bytes));
        ix.q_bytes[slot] = bytes;
    }
    VB_CUDA(cudaMemcpyAsync(ix.q_buf[slot], queries, bytes, cudaMemcpyHostToDevice, ix.q_stream));
    VB_CUDA(cudaEventRecord(ix.q_ready[slot], ix.q_stream));
    ix.q_nq[slot] = nq;
    return VB_OK;
}

int vb_ivf_search_prefetched(vb_ivf* h, int slot, int probes, int k, int64_t* out_ids, double* out_dist) {
    VB_TRY(require_init());
    VB_REQUIRE(h && h->ix.loaded && (slot == 0 || slot == 1) && h->ix.q_nq[slot] > 0, "no prefetched queries in this slot");
    Ivf& ix = h->ix;
    VB_CUDA(cudaStreamWaitEvent(ctx().stream, ix.q_ready[slot], 0));
    const int64_t nq = ix.q_nq[slot];
    ix.q_nq[slot] = 0;   // consumed: the slot may be refilled as soon as this call returns (it synchronises)
    return ivf_search_impl(h, ix.q_buf[slot], nq, probes, k, true, false, out_ids, nullptr, out_dist);
}

// List-sharded search (SURVEY 8e): this rank's image holds its own lists under the GLOBAL list numbering (the other
// lists are empty) and all centres.  Per batch: probe selection for this rank's slice of the queries -> all-gather of
// the probe lists -> local list scan + top-k for ALL queries -> all-gather of k (distance, id) pairs per rank ->
// k-way merge.  Every rank returns the full result.  Collectives are NCCL calls on the library stream; the
// certificate counters of the tensor-core filter are summed over the ranks before they are read, so all ranks
// repeat a batch together.
int vb_ivf_search_sharded_dev(vb_ivf* h, const void* queries_dev, int64_t nq, int probes, int k, int64_t* out_ids_dev,
                              float* out_dist_dev) {
    VB_TRY(require_init());
    VB_REQUIRE(h && h->ix.loaded, "index not loaded");
    VB_REQUIRE(queries_dev && probes >= 1 && k >= 1 && out_ids_dev && out_dist_dev, "bad search arguments");
    Ivf& ix = h->ix;
    Context& c = ctx();
    const int world = comm_world(), rank = comm_rank();
    probes = std::min(probes, ix.lists);
    if (nq <= 0) return VB_OK;
    VB_REQUIRE(nq <= ivf_batch_limit(ix, probes), "sharded search: at most %lld queries per call for this index", (long long)ivf_batch_limit(ix, probes));
    int P = 2;
    while (P < world * k) P <<= 1;
    VB_REQUIRE(P <= 4096, "sharded search: world * k must not exceed 4096");
    const int64_t chunk = (nq + world - 1) / world;
    const int64_t q0 = std::min<int64_t>(nq, (int64_t)rank * chunk), m = std::min<int64_t>(chunk, nq - q0);
    Scratch sc;
    void *d_sh, *d_res;
    VB_TRY(sc.take(sizeof(int32_t) * (size_t)chunk * probes * (world + 1) + 64, &d_sh));
    int32_t* my_lists = (int32_t*)d_sh;                          // [chunk x probes]
    int32_t* all_lists = my_lists + (size_t)chunk * probes;      // [world x chunk x probes] = [nq' x probes]
    const size_t res_ids = sizeof(int64_t) * (size_t)nq * k, res_dist = sizeof(float) * (size_t)nq * k;
    VB_TRY(sc.take((res_ids + res_dist) * (size_t)(world + 1) + 256, &d_res));
    int64_t* my_ids = (int64_t*)d_res;
    float* my_dist = (float*)((uint8_t*)d_res + res_ids);
    int64_t* all_ids = (int64_t*)((uint8_t*)d_res + res_ids + res_dist);
    float* all_dist = (float*)((uint8_t*)all_ids + res_ids * (size_t)world);
    VB_CUDA(cudaMemsetAsync(ix.d_cand_sum, 0, sizeof(int64_t), c.stream));
    const int64_t cap = ivf_cap(ix, probes);

    auto run = [&](const IvfPass& pass, int* fails, int* level) -> int {
        VB_TRY(ivf_tc_fail_zero(ix));
        Scratch batch;
        void* qimg;
        size_t qstride;
        VB_TRY(upload_queries(batch, ix.elem, ix.dim, queries_dev, nq, false, &qimg, &qstride));
        VB_CUDA(cudaMemsetAsync(my_lists, 0xFF, sizeof(int32_t) * (size_t)chunk * probes, c.stream));
        if (m > 0) {
            int32_t* d_lists;
            float* d_ldist;
            float* qn_mine = nullptr;
            VB_TRY(ivf_select_probes(batch, ix, pass, (const uint8_t*)qimg + (size_t)q0 * qstride, qstride, m, &qn_mine, probes,
                                     &d_lists, &d_ldist));
            VB_CUDA(cudaMemcpyAsync(my_lists, d_lists, sizeof(int32_t) * (size_t)m * probes, cudaMemcpyDeviceToDevice, c.stream));
        }
        VB_TRY(comm_allgather(my_lists, all_lists, (int64_t)sizeof(int32_t) * chunk * probes));
        // (ranks hold `chunk` queries each, the last one possibly fewer: the gathered array is query-major for q < nq)
        float* qn = nullptr;
        VB_TRY(ivf_scan_topk(batch, ix, pass, qimg, qstride, nq, &qn, all_lists, probes, cap, k, my_ids, my_dist, nullptr, level));
        // one buffer per rank: [ids | distances]; gathered rank-major, so view it as two strided arrays
        VB_TRY(comm_allgather(my_ids, all_ids, (int64_t)res_ids));
        VB_TRY(comm_allgather(my_dist, all_dist, (int64_t)res_dist));
        merge_ranks_kernel<<<(unsigned)nq, 128, (size_t)P * 8, c.stream>>>(all_ids, all_dist, world, nq, k, P, out_ids_dev, out_dist_dev);
        VB_CUDA(cudaGetLastError());
        count_launch();
        fails[0] = fails[1] = 0;
        if (pass.defer_check) {
            VB_TRY(comm_allreduce(ix.d_tc_fail, 2, 1));
            VB_CUDA(cudaMemcpyAsync(fails, ix.d_tc_fail, 2 * sizeof(int), cudaMemcpyDeviceToHost, c.stream));
            VB_CUDA(cudaStreamSynchronize(c.stream));
        }
        return VB_OK;
    };
    // no level 0: the sharded search keeps the batch-wide repeats, which every rank makes together
    VB_TRY(ivf_certified_batch(ix, probes, IvfPass{}, run, nullptr));
    ix.last_cand = -1;
    ix.last_bytes = nq;
    return VB_OK;
}

__global__ void add_id_offset_kernel(int64_t* ids, int64_t n, int64_t offset) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i < n && ids[i] >= 0) ids[i] += offset;
}

// Exact (no index) top-k over a row-sharded table (SURVEY 8e): every rank scans its own rows, the per-rank k nearest
// are all-gathered and merged by (distance, id).  id_offset = the global number of this rank's row 0.
int vb_exact_topk_sharded_dev(vb_table* t, int metric, const void* queries_dev, int64_t nq, int k, int64_t id_offset, int64_t* out_ids_dev,
                              float* out_dist_dev) {
    VB_TRY(require_init());
    VB_REQUIRE(t && queries_dev && out_ids_dev && out_dist_dev && k >= 1, "bad arguments");
    if (nq <= 0) return VB_OK;
    Context& c = ctx();
    const int world = comm_world();
    int P = 2;
    while (P < world * k) P <<= 1;
    VB_REQUIRE(P <= 4096, "sharded exact scan: world * k must not exceed 4096");
    Scratch sc;
    void* d_res;
    const size_t res_ids = sizeof(int64_t) * (size_t)nq * k, res_dist = sizeof(float) * (size_t)nq * k;
    VB_TRY(sc.take((res_ids + res_dist) * (size_t)(world + 1) + 256, &d_res));
    int64_t* my_ids = (int64_t*)d_res;
    float* my_dist = (float*)((uint8_t*)d_res + res_ids);
    int64_t* all_ids = (int64_t*)((uint8_t*)d_res + res_ids + res_dist);
    float* all_dist = (float*)((uint8_t*)all_ids + res_ids * (size_t)world);
    VB_TRY(vb_exact_topk_dev(t, metric, queries_dev, nq, k, my_ids, my_dist));
    add_id_offset_kernel<<<(unsigned)((nq * k + 255) / 256), 256, 0, c.stream>>>(my_ids, nq * k, id_offset);
    VB_TRY(comm_allgather(my_ids, all_ids, (int64_t)res_ids));
    VB_TRY(comm_allgather(my_dist, all_dist, (int64_t)res_dist));
    merge_ranks_kernel<<<(unsigned)nq, 128, (size_t)P * 8, c.stream>>>(all_ids, all_dist, world, nq, k, P, out_ids_dev, out_dist_dev);
    VB_CUDA(cudaGetLastError());
    count_launch(2);
    return VB_OK;
}

int vb_ivf_search_sharded(vb_ivf* h, const void* queries, int64_t nq, int probes, int k, int64_t* out_ids, double* out_dist) {
    VB_TRY(require_init());
    VB_REQUIRE(h && h->ix.loaded && queries && out_ids && out_dist && k >= 1, "bad search arguments");
    if (nq <= 0) return VB_OK;
    Ivf& ix = h->ix;
    Context& c = ctx();
    const size_t raw = raw_row_bytes(ix.elem, ix.dim);
    Scratch sc;
    void* d_q;
    VB_TRY(sc.take(raw * (size_t)nq + (sizeof(int64_t) + sizeof(float)) * (size_t)nq * k + 64, &d_q));
    int64_t* d_ids = (int64_t*)((uint8_t*)d_q + ((raw * (size_t)nq + 15) & ~(size_t)15));
    float* d_dist = (float*)(d_ids + (size_t)nq * k);
    VB_CUDA(cudaMemcpyAsync(d_q, queries, raw * (size_t)nq, cudaMemcpyHostToDevice, c.stream));
    VB_TRY(vb_ivf_search_sharded_dev(h, d_q, nq, probes, k, d_ids, d_dist));
    std::vector<float> hd((size_t)nq * k);
    VB_CUDA(cudaMemcpyAsync(out_ids, d_ids, sizeof(int64_t) * (size_t)nq * k, cudaMemcpyDeviceToHost, c.stream));
    VB_CUDA(cudaMemcpyAsync(hd.data(), d_dist, sizeof(float) * (size_t)nq * k, cudaMemcpyDeviceToHost, c.stream));
    VB_CUDA(cudaStreamSynchronize(c.stream));
    for (size_t i = 0; i < hd.size(); ++i) out_dist[i] = (double)hd[i];
    return VB_OK;
}

// ---- ivfflat.iterative_scan for a batch of queries (vb_ivf_iter.cu)

}  // extern "C"

namespace vb {

// filtered handle: the filters' positions, heap ids and offset tables into the handle's allocation, and the probe
// order renamed to the filters' virtual lists (launch_ivf_filter_lists)
static int ivf_scan_copy_filters(vb_ivf_scan& s, const vb_filter* const* filters, const int32_t* filter_of_query) {
    Ivf& ix = *s.ix;
    Context& c = ctx();
    const int lists = ix.lists;
    std::vector<int64_t> foff((size_t)s.nfilters * lists + 1);
    int64_t base = 0;
    for (int i = 0; i < s.nfilters; ++i) {
        const Filter& f = filters[i]->f;
        for (int l = 0; l < lists; ++l) foff[(size_t)i * lists + l] = base + f.h_off[(size_t)l];
        if (f.n) {
            VB_CUDA(cudaMemcpyAsync(s.fpos + base, f.pos, 8 * (size_t)f.n, cudaMemcpyDeviceToDevice, c.stream));
            VB_CUDA(cudaMemcpyAsync(s.fids + base, f.ids, 8 * (size_t)f.n, cudaMemcpyDeviceToDevice, c.stream));
        }
        base += f.n;
    }
    foff.back() = base;
    VB_CUDA(cudaMemcpyAsync(s.foff, foff.data(), 8 * foff.size(), cudaMemcpyHostToDevice, c.stream));
    if (filter_of_query && s.nfilters > 1) {
        Scratch sc;
        void* d_fq;
        VB_TRY(sc.take(sizeof(int32_t) * (size_t)s.nq, &d_fq));
        VB_CUDA(cudaMemcpyAsync(d_fq, filter_of_query, sizeof(int32_t) * (size_t)s.nq, cudaMemcpyHostToDevice, c.stream));
        VB_TRY(launch_ivf_filter_lists(s.nq, s.max_probes, lists, (const int32_t*)d_fq, s.probe));
    }
    VB_CUDA(cudaStreamSynchronize(c.stream));   // foff is a stack-owned vector
    return VB_OK;
}

static int ivf_scan_begin_impl(const char* fn, vb_ivf* h, const void* queries, int64_t nq, int probes, int max_probes, int page,
                               const vb_filter* const* filters, int nfilters, const int32_t* filter_of_query, vb_ivf_scan** out) {
    VB_TRY(require_init());
    VB_REQUIRE(out, "%s: null handle pointer", fn);
    *out = nullptr;
    if (!h || !h->ix.loaded) {
        set_error("%s: index not loaded", fn);
        return VB_ESTATE;
    }
    VB_REQUIRE(queries, "%s: queries must not be NULL (a NULL-query scan takes vb_ivf_scan_items)", fn);
    VB_REQUIRE(nq >= 1, "%s: nq must be >= 1 (got %lld)", fn, (long long)nq);
    VB_REQUIRE(probes >= 1 && max_probes >= 1, "%s: probes and max_probes must be >= 1 (got %d, %d)", fn, probes, max_probes);
    VB_REQUIRE(page >= 1 && page <= 2048, "%s: page must be in 1..2048 (got %d)", fn, page);
    Ivf& ix = h->ix;
    vb_ivf_scan s;
    s.ix = &ix;
    s.generation = ix.generation;
    s.nq = nq;
    s.probes = std::min(probes, ix.lists);                                   // src/ivfscan.c:268-277
    s.max_probes = std::min(std::max(max_probes, probes), ix.lists);
    s.page = page;
    if (filters) {
        VB_REQUIRE(nfilters >= 1 && (int64_t)nfilters * ix.lists < (int64_t)INT32_MAX, "%s: %d row filters", fn, nfilters);
        VB_REQUIRE(filter_of_query || nfilters == 1, "%s: filter_of_query may only be NULL with one filter (got %d)", fn, nfilters);
        for (int i = 0; i < nfilters; ++i) {
            VB_REQUIRE(filters[i], "%s: filter %d is NULL", fn, i);
            const Filter& f = filters[i]->f;
            VB_REQUIRE(f.kind == FILTER_IVF && f.owner == h && f.owner_uid == h->uid, "%s: filter %d was made for another table or index", fn, i);
            if (f.generation != ix.generation) {
                set_error("%s: filter %d: index changed since the filter was created", fn, i);
                return VB_ESTATE;
            }
        }
        for (int64_t q = 0; q < nq && filter_of_query; ++q)
            VB_REQUIRE(filter_of_query[q] >= 0 && filter_of_query[q] < nfilters, "%s: filter_of_query[%lld] = %d, not in 0..%d", fn,
                       (long long)q, filter_of_query[q], nfilters - 1);
        // a group holds at most the p largest allowed counts of one filter's lists
        s.nfilters = nfilters;
        s.cap = 1;
        std::vector<int64_t> cnt((size_t)ix.lists);
        for (int i = 0; i < nfilters; ++i) {
            const Filter& f = filters[i]->f;
            for (int l = 0; l < ix.lists; ++l) cnt[(size_t)l] = f.h_off[(size_t)l + 1] - f.h_off[(size_t)l];
            std::partial_sort(cnt.begin(), cnt.begin() + s.probes, cnt.end(), std::greater<int64_t>());
            s.cap = std::max(s.cap, std::accumulate(cnt.begin(), cnt.begin() + s.probes, (int64_t)0));
            s.fallowed += f.n;
        }
    } else {
        s.cap = ivf_cap(ix, s.probes);
    }
    VB_REQUIRE(s.cap < (int64_t)INT32_MAX, "%s: %lld candidates per group", fn, (long long)s.cap);
    s.rpc = scan_chunk_rows(ix.rows);
    s.max_chunks = nq * (s.cap / s.rpc + s.probes + 1);
    VB_REQUIRE(s.max_chunks < (int64_t)INT32_MAX, "%s: too many scan chunks (%lld): open fewer queries per handle", fn,
               (long long)s.max_chunks);
    s.qstride = ivf_qstride(ix);
    const size_t bytes = ivf_scan_carve(s, nullptr);
    size_t free_b = 0, total_b = 0;
    VB_CUDA(cudaMemGetInfo(&free_b, &total_b));
    if (bytes > free_b) {
        if (s.nfilters)
            set_error("%s: %lld queries need %zu bytes of device memory (%zu per query, %zu for the row filters), %zu are free", fn,
                      (long long)nq, bytes, ivf_scan_bytes_per_query(s), ivf_scan_filter_bytes(s), free_b);
        else
            set_error("%s: %lld queries need %zu bytes of device memory (%zu per query), %zu are free", fn, (long long)nq, bytes,
                      ivf_scan_bytes_per_query(s), free_b);
        return VB_ENOMEM;
    }
    if (cudaMalloc(&s.mem, bytes) != cudaSuccess) {
        cudaGetLastError();
        set_error("%s: allocation of %zu bytes failed (%zu per query)", fn, bytes, ivf_scan_bytes_per_query(s));
        return VB_ENOMEM;
    }
    ivf_scan_carve(s, (uint8_t*)s.mem);
    int rc = ivf_scan_setup(s, queries);
    if (rc == VB_OK && s.nfilters) rc = ivf_scan_copy_filters(s, filters, filter_of_query);
    if (rc != VB_OK) {
        cudaFree(s.mem);
        return rc;
    }
    *out = new vb_ivf_scan(s);
    return VB_OK;
}

}  // namespace vb

extern "C" {

int vb_ivf_scan_begin(vb_ivf* h, const void* queries, int64_t nq, int probes, int max_probes, int page, vb_ivf_scan** out) {
    return ivf_scan_begin_impl("vb_ivf_scan_begin", h, queries, nq, probes, max_probes, page, nullptr, 0, nullptr, out);
}

int vb_ivf_scan_begin_filtered(vb_ivf* h, const void* queries, int64_t nq, int probes, int max_probes, int page,
                               const vb_filter* const* filters, int nfilters, const int32_t* filter_of_query, vb_ivf_scan** out) {
    if (!filters) {
        set_error("vb_ivf_scan_begin_filtered: no row filter given");
        if (out) *out = nullptr;
        return VB_EINVAL;
    }
    return ivf_scan_begin_impl("vb_ivf_scan_begin_filtered", h, queries, nq, probes, max_probes, page, filters, nfilters, filter_of_query,
                               out);
}

static int ivf_filter_create(vb_ivf* h, const int64_t* ids, int64_t n, bool host, vb_filter** out) {
    VB_TRY(require_init());
    VB_REQUIRE(out, "vb_ivf_filter_create: null filter pointer");
    *out = nullptr;
    if (!h || !h->ix.loaded) {
        set_error("vb_ivf_filter_create: index not loaded");
        return VB_ESTATE;
    }
    VB_REQUIRE(n >= 0 && (ids || n == 0), "vb_ivf_filter_create: null ids or negative count %lld", (long long)n);
    Ivf& ix = h->ix;
    vb_filter* f = new vb_filter;
    f->f.owner = h;
    f->f.owner_uid = h->uid;
    f->f.generation = ix.generation;
    const int rc = filter_build_ivf(ix.rows.n, ix.d_ids, ix.d_list_off, ix.lists, ids, n, host, &f->f);
    if (rc != VB_OK) {
        filter_release(&f->f);
        delete f;
        return rc;
    }
    *out = f;
    return VB_OK;
}

int vb_ivf_filter_create(vb_ivf* h, const int64_t* ids, int64_t n, vb_filter** out) { return ivf_filter_create(h, ids, n, true, out); }

int vb_ivf_filter_create_dev(vb_ivf* h, const int64_t* ids_dev, int64_t n, vb_filter** out) {
    return ivf_filter_create(h, ids_dev, n, false, out);
}

int vb_ivf_scan_next(vb_ivf_scan* s, int64_t* out_ids, double* out_dist, int32_t* out_counts) {
    VB_TRY(require_init());
    VB_REQUIRE(s && out_ids && out_dist && out_counts, "vb_ivf_scan_next: null argument");
    Ivf& ix = *s->ix;
    if (!ix.loaded || ix.generation != s->generation) {
        set_error("vb_ivf_scan_next: index changed since the scan began");
        return VB_ESTATE;
    }
    Context& c = ctx();
    const int64_t nq = s->nq;
    // a filtered handle: the same kernels over the filters' runs (virtual lists), the allowed rows gathered by position
    const int64_t* list_off = s->nfilters ? s->foff : ix.d_list_off;
    const int64_t* ids = s->nfilters ? s->fids : ix.d_ids;
    VB_TRY(launch_ivf_iter_advance(nq, s->probes, s->max_probes, s->probe, list_off, s->glists, s->list_index, s->returned,
                                   s->seg_len, s->active));
    VB_CUDA(cudaMemsetAsync(s->n_chunks, 0, sizeof(int), c.stream));
    ivf_build_chunks_kernel<<<(unsigned)nq, 128, 0, c.stream>>>(s->glists, s->probes, list_off, s->rpc, s->cap, s->cand_off, s->seg_begin,
                                                                s->seg_len, s->chunks, s->n_chunks, s->cand_sum, s->active);
    VB_CUDA(cudaGetLastError());
    count_launch();
    if (s->nfilters)
        VB_TRY(launch_scan_gather(ix.rows, key_metric(ix.metric), s->qimg, s->qstride, s->fpos, s->chunks, s->n_chunks, (int)s->max_chunks,
                                  s->dist));
    else
        VB_TRY(launch_scan_chunks(ix.rows, key_metric(ix.metric), s->qimg, s->qstride, s->chunks, s->n_chunks, (int)s->max_chunks, s->dist,
                                  true));
    VB_TRY(launch_segment_topk_floor(s->dist, s->seg_begin, s->seg_len, nq, s->page, s->floor_key, s->returned, s->counts, s->pos, s->key));
    const int64_t n = nq * s->page;
    ivf_finish_kernel<<<(unsigned)((n + 255) / 256), 256, 0, c.stream>>>(ix.metric, nq, s->page, s->probes, s->pos, s->key, s->glists,
                                                                        s->cand_off, list_off, ids, s->out_ids, nullptr, s->out_d);
    VB_CUDA(cudaGetLastError());
    count_launch();
    void* pin;
    const size_t bytes = 16 * (size_t)n + 4 * (size_t)nq;
    VB_TRY(pinned_buffer2(bytes, &pin));
    VB_CUDA(cudaMemcpyAsync(pin, s->out_ids, bytes, cudaMemcpyDeviceToHost, c.stream));
    VB_CUDA(cudaStreamSynchronize(c.stream));
    memcpy(out_ids, pin, 8 * (size_t)n);
    memcpy(out_dist, (const uint8_t*)pin + 8 * (size_t)n, 8 * (size_t)n);
    memcpy(out_counts, (const uint8_t*)pin + 16 * (size_t)n, 4 * (size_t)nq);
    return VB_OK;
}

int vb_ivf_scan_lists_done(vb_ivf_scan* s, int32_t* out) {
    VB_TRY(require_init());
    VB_REQUIRE(s && out, "vb_ivf_scan_lists_done: null argument");
    VB_CUDA(cudaMemcpyAsync(out, s->list_index, sizeof(int32_t) * (size_t)s->nq, cudaMemcpyDeviceToHost, ctx().stream));
    VB_CUDA(cudaStreamSynchronize(ctx().stream));
    return VB_OK;
}

int vb_ivf_scan_end(vb_ivf_scan* s) {
    if (!s) return VB_OK;
    if (s->mem) {
        cudaStreamSynchronize(ctx().stream);
        cudaFree(s->mem);
    }
    delete s;
    return VB_OK;
}

int vb_ivf_tc_traffic(int on, int64_t* out8) {
    VB_TRY(require_init());
    return list_tc_traffic(on, out8);
}

int vb_ivf_tc_level0_rescored(int64_t* out3) {
    VB_TRY(require_init());
    VB_REQUIRE(out3 != nullptr, "vb_ivf_tc_level0_rescored: out3 is NULL");
    return list_tc_level0_rescored(out3);
}

int64_t vb_ivf_tc_fallbacks(const vb_ivf* h) { return h ? h->ix.total_tc_failed : 0; }
int64_t vb_ivf_tc_level1_fallbacks(const vb_ivf* h) { return h ? h->ix.total_l1_failed : 0; }
int64_t vb_ivf_tc_level0_fallbacks(const vb_ivf* h) { return h ? h->ix.total_l0_failed : 0; }
int64_t vb_ivf_tc_levelp_fallbacks(const vb_ivf* h) { return h ? h->ix.total_lp_failed : 0; }

int64_t vb_ivf_last_candidates(const vb_ivf* h) {
    if (!h || !h->ix.d_cand_sum) return 0;
    int64_t v = 0;
    cudaStreamSynchronize(ctx().stream);
    cudaMemcpy(&v, h->ix.d_cand_sum, sizeof(int64_t), cudaMemcpyDeviceToHost);
    return v;
}
int64_t vb_ivf_last_scan_bytes(const vb_ivf* h) {
    if (!h) return 0;
    const Ivf& ix = h->ix;
    int64_t cand = vb_ivf_last_candidates(h);
    int64_t nq = ix.last_bytes;  // number of queries of the last search
    return (nq * ix.lists + cand) * (int64_t)raw_row_bytes(ix.elem, ix.dim);
}

}  // extern "C"
