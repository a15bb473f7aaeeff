// vb_hnsw.cu -- HNSW search on the device: GetScanItems (src/hnswscan.c:25-56) =
// greedy descent with ef = 1 through the upper layers, then HnswSearchLayer
// (src/hnswutils.c:824-987) with ef at layer 0.  Many queries per launch, one warp per query.
//
// Formulation.  Every distance comparison of the reference is taken on the total order
// (distance, element number).  Under a total order the two pairing heaps collapse into ONE
// sorted array R of the best <= ef elements seen so far, each with an "expanded" flag:
//   W (results)    = R;   f = R[len-1]
//   C (candidates) = unexpanded elements of R  (anything evicted from W is > f for ever,
//                    so the reference would break on it before expanding it)
//   pop nearest(C) = first unexpanded element of R;  "c > f -> break" = no unexpanded left
//   admit e        = e lands inside the first ef entries of merge(R, {e})
// which is order independent, so the <= lm neighbours of one expansion are scored
// together: one 128-byte neighbour-list read, lm independent row gathers in flight,
// a warp bitonic sort of the batch and a parallel merge into R.
//
// Roofline: HBM (latency-bound random row gathers).  Algorithmic bytes per query =
// n_dist * dim * element size + n_expand * lm * 4 (SURVEY section 8d); n_dist is returned per query.
#include "vb_hnsw.cuh"

#include <algorithm>
#include <vector>

namespace vb {

// One warp = one query at a time.
template <int ELEM, int METRIC, int LPR>
__global__ void VB_HNSW_BOUNDS hnsw_search_kernel(HnswDev g, const uint8_t* __restrict__ queries, size_t qstride,
                                                                    int64_t nq, int ef, int k, uint32_t* __restrict__ vis_all,
                                                                    uint32_t vis_cap, uint32_t vis_upper, int64_t* __restrict__ out_ids,
                                                                    float* __restrict__ out_f, double* __restrict__ out_d,
                                                                    int64_t* __restrict__ out_ndist, int* __restrict__ overflow) {
    extern __shared__ uint4 smem[];
    const int warp = threadIdx.x / 32, lane = threadIdx.x % 32;
    const int qvec = (int)(qstride / 16);
    // per-warp carve-up: query image | keys A | keys B | batch keys | ids A | ids B | batch ids
    const size_t per_warp = (size_t)qvec * 16 + (size_t)ef * 2 * 8 + (size_t)ef * 2 * 4 + 32 * 8 + 32 * 4;
    const size_t per_warp_al = (per_warp + 15) & ~(size_t)15;
    uint8_t* base = reinterpret_cast<uint8_t*>(smem) + (size_t)warp * per_warp_al;
    uint4* sq = reinterpret_cast<uint4*>(base);
    uint64_t* keyA = reinterpret_cast<uint64_t*>(base + (size_t)qvec * 16);
    uint64_t* keyB = keyA + ef;
    uint64_t* bkey = keyB + ef;
    uint32_t* idA = reinterpret_cast<uint32_t*>(bkey + 32);
    uint32_t* idB = idA + ef;
    uint32_t* bid = idB + ef;

    const int gwarp = blockIdx.x * HN_WARPS + warp;
    const int nwarps = gridDim.x * HN_WARPS;
    uint32_t* vis = vis_all + (size_t)gwarp * vis_cap;

    // the first query of a warp is its own number; the following ones come from a counter (overflow[1], zeroed with the
    // flag before the launch): a search takes 0.5x - 2x the mean, and a static split left a third of the warps idle
    // through the tail of the launch
#ifndef VB_AB_DYNQ
#define VB_AB_DYNQ 1
#endif
    for (int64_t q = gwarp; q < nq;) {
        const uint4* gq = reinterpret_cast<const uint4*>(queries + (size_t)q * qstride);
        load_query_image<ELEM, METRIC>(gq, qvec, g.V, sq, lane);
        __syncwarp();

        HnswWarpState S;
        S.rk = keyA;
        S.ri = idA;
        S.nk = keyB;
        S.ni = idB;
        S.vcn = 2 * ef;
        S.bkey = bkey;
        S.bid = bid;
        S.len = 0;
        int64_t ndist = 0;
        bool failed = false;

        // entry point distance (HnswEntryCandidate, src/hnswutils.c:609-621)
        {
            Acc<ELEM, METRIC> acc;
            const uint4* rp = reinterpret_cast<const uint4*>(g.rows + (size_t)g.entry * g.stride);
            for (int v = lane; v < g.V; v += 32) hnsw_acc_add<ELEM, METRIC>(acc, ldg_stream(rp + v), sq, v);
            acc.template reduce<32>();
            if (lane == 0) {
                S.rk[0] = orderable_key64(acc.value());
                S.ri[0] = (uint32_t)g.entry;
            }
            S.len = 1;
            __syncwarp();
        }

        for (int lc = g.entry_level; lc >= 0 && !failed; --lc) {
            // (the ef = 1 layers use a small visited region of their own so only it is cleared per layer)
            uint32_t* tab = lc == 0 ? vis + vis_upper : vis;
            const uint32_t cap = lc == 0 ? vis_cap - vis_upper : vis_upper;
            failed = !hnsw_search_layer<ELEM, METRIC, LPR>(g, sq, lc, lc == 0 ? ef : 1, lane, S, tab, cap, lc == 0 ? &ndist : nullptr);
        }

        if (failed && lane == 0) atomicExch(overflow, 1);
        // results nearest first (src/hnswscan.c:293-326)
        for (int i = lane; i < k; i += 32) {
            bool have = i < S.len && !failed;
            int64_t id = have ? (int64_t)(S.ri[i] & 0x7fffffffu) : -1;
            double d = have ? key64_to_double(S.rk[i]) : (double)INFINITY;
            out_ids[q * k + i] = id;
            if (out_f) out_f[q * k + i] = (float)d;
            if (out_d) out_d[q * k + i] = d;
        }
        if (out_ndist && lane == 0) out_ndist[q] = ndist;
        __syncwarp();
#if VB_AB_DYNQ
        int nxt = 0;
        if (lane == 0) nxt = atomicAdd(overflow + 1, 1);
        q = (int64_t)nwarps + __shfl_sync(0xffffffffu, nxt, 0);
#else
        q += nwarps;
#endif
    }
}

template <int ELEM, int METRIC>
static int hnsw_launch_t(const HnswDev& g, const void* qimg, size_t qstride, int64_t nq, int ef, int k, uint32_t* vis, uint32_t vis_cap,
                         uint32_t vis_upper, int grid, int64_t* out_ids, float* out_f, double* out_d, int64_t* out_nd, int* overflow,
                         int* occ_out) {
    const int qvec = (int)(qstride / 16);
    size_t per_warp = (size_t)qvec * 16 + (size_t)ef * 2 * 8 + (size_t)ef * 2 * 4 + 32 * 8 + 32 * 4;
    per_warp = (per_warp + 15) & ~(size_t)15;
    const size_t smem = per_warp * HN_WARPS;
    VB_REQUIRE(smem <= 200 * 1024, "ef_search %d with this dimension needs %zu bytes of shared memory per CTA", ef, smem);
    cudaStream_t s = ctx().stream;
#ifndef VB_AB_LPR_V8
#define VB_AB_LPR_V8 8   /* lanes per row for 128-byte rows (bit(1024)); 8 = one 16-byte word per lane, 32 rows in one round trip */
#endif
#define VB_HL(LPR)                                                                                                        \
    do {                                                                                                                  \
        auto kern = hnsw_search_kernel<ELEM, METRIC, LPR>;                                                                \
        if (smem > 48 * 1024) VB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); \
        if (occ_out) {                                                                                                    \
            /* sizing pass: how many CTAs of this instantiation are resident per SM (the grid is exactly one wave) */     \
            VB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(occ_out, kern, HN_WARPS * 32, smem));                   \
            return VB_OK;                                                                                                 \
        }                                                                                                                 \
        kern<<<grid, HN_WARPS * 32, smem, s>>>(g, (const uint8_t*)qimg, qstride, nq, ef, k, vis, vis_cap, vis_upper, out_ids, out_f, out_d, \
                                               out_nd, overflow);                                                        \
    } while (0)
    // lanes per row: a whole warp for rows of >= 512 bytes; short rows take few lanes each so that the <= 32 neighbours of
    // one expansion are gathered in ONE pass (GROUPS * RPI >= 16 rows) instead of four dependent ones
    if (g.V >= 32) VB_HL(32);
    else if (g.V >= 16) VB_HL(4);
    else if (g.V == 8 && VB_AB_LPR_V8 == 8) VB_HL(8);
    else if (g.V >= 8) VB_HL(2);
    else VB_HL(1);
#undef VB_HL
    VB_CUDA(cudaGetLastError());
    count_launch();
    return VB_OK;
}

static int hnsw_launch(const Hnsw& h, const HnswDev& g, const void* qimg, size_t qstride, int64_t nq, int ef, int k, uint32_t* vis,
                       uint32_t vis_cap, uint32_t vis_upper, int grid, int64_t* out_ids, float* out_f, double* out_d, int64_t* out_nd, int* overflow,
                       int* occ_out = nullptr) {
#define VB_HC(E, M) return hnsw_launch_t<E, M>(g, qimg, qstride, nq, ef, k, vis, vis_cap, vis_upper, grid, out_ids, out_f, out_d, out_nd, overflow, occ_out)
    if (h.elem == VB_VECTOR) {
        switch (h.metric) {
            case VB_L2_SQUARED: VB_HC(VB_VECTOR, VB_L2_SQUARED);
            case VB_NEG_IP: VB_HC(VB_VECTOR, VB_NEG_IP);
            case VB_L1: VB_HC(VB_VECTOR, VB_L1);
        }
    } else if (h.elem == VB_HALFVEC) {
        switch (h.metric) {
            case VB_L2_SQUARED: VB_HC(VB_HALFVEC, VB_L2_SQUARED);
            case VB_NEG_IP: VB_HC(VB_HALFVEC, VB_NEG_IP);
            case VB_L1: VB_HC(VB_HALFVEC, VB_L1);
        }
    } else {
        switch (h.metric) {
            case VB_HAMMING: VB_HC(VB_BIT, VB_HAMMING);
            case VB_JACCARD: VB_HC(VB_BIT, VB_JACCARD);
        }
    }
#undef VB_HC
    set_error("hnsw: unsupported metric %d for element type %d", h.metric, h.elem);
    return VB_EINVAL;
}

// The visited tables are the only data of a graph walk that is re-used (32 probes per expansion, every one a random
// 32-byte sector); rows and neighbour lists stream past once.  Marking the tables' range persisting in L2 keeps the
// probes out of DRAM.
static void hnsw_l2_window(cudaStream_t s, void* base, size_t bytes, bool on) {
    static int max_window = -1, max_persist = -1;
    if (max_window < 0) {
        int dev = 0;
        cudaGetDevice(&dev);
        cudaDeviceGetAttribute(&max_window, cudaDevAttrMaxAccessPolicyWindowSize, dev);
        cudaDeviceGetAttribute(&max_persist, cudaDevAttrMaxPersistingL2CacheSize, dev);
        if (max_persist > 0) cudaDeviceSetLimit(cudaLimitPersistingL2CacheSize, (size_t)max_persist);
        cudaGetLastError();
    }
    if (max_window <= 0 || max_persist <= 0) return;
    cudaStreamAttrValue v{};
    if (on) {
        const size_t win = std::min(bytes, (size_t)max_window);
        v.accessPolicyWindow.base_ptr = base;
        v.accessPolicyWindow.num_bytes = win;
        v.accessPolicyWindow.hitRatio = (float)std::min(1.0, (double)max_persist / (double)win);
        v.accessPolicyWindow.hitProp = cudaAccessPropertyPersisting;
        v.accessPolicyWindow.missProp = cudaAccessPropertyStreaming;
    } else {
        v.accessPolicyWindow.num_bytes = 0;
        v.accessPolicyWindow.hitProp = cudaAccessPropertyNormal;
        v.accessPolicyWindow.missProp = cudaAccessPropertyNormal;
    }
    cudaStreamSetAttribute(s, cudaStreamAttributeAccessPolicyWindow, &v);
    cudaGetLastError();
}

static int hnsw_search_impl(Hnsw& h, const void* queries, int64_t nq, int ef, int k, bool host, int64_t* out_ids, float* out_f,
                            double* out_d, int64_t* out_nd) {
    Scratch sc;
    VB_REQUIRE(h.loaded, "hnsw index not loaded");
    VB_REQUIRE(ef >= 1 && ef <= 1000, "ef_search must be 1..1000 (src/hnsw.h:60-62)");
    VB_REQUIRE(k >= 1 && k <= ef, "k must be 1..ef_search");
    if (nq <= 0) return VB_OK;
    Context& c = ctx();
    cudaStream_t s = c.stream;
    if (h.entry < 0) {
        // empty index: no results
        std::vector<int64_t> ids((size_t)nq * k, -1);
        if (host) {
            memcpy(out_ids, ids.data(), sizeof(int64_t) * ids.size());
            for (int64_t i = 0; i < nq * k; ++i) out_d[i] = INFINITY;
            if (out_nd) memset(out_nd, 0, sizeof(int64_t) * (size_t)nq);
        }
        return VB_OK;
    }
    HnswDev g{};
    g.rows = h.rows.d;
    g.stride = h.rows.stride;
    g.V = (int)(h.rows.stride / 16);
    g.levels = h.levels;
    g.nbr0 = h.nbr0;
    g.upper_off = h.upper_off;
    g.upper = h.upper;
    g.m = h.m;
    g.n = h.n;
    g.entry = (int)h.entry;
    g.entry_level = h.entry_level;

    void* qimg;
    size_t qstride;
    VB_TRY(upload_queries(sc, h.elem, h.dim, queries, nq, host, &qimg, &qstride));

    int64_t* d_ids = out_ids;
    float* d_f = out_f;
    double* d_d = nullptr;
    int64_t* d_nd = out_nd;
    if (host) {
        void* d_out;
        VB_TRY(sc.take((sizeof(int64_t) + sizeof(double)) * (size_t)nq * k + sizeof(int64_t) * (size_t)nq, &d_out));
        d_ids = (int64_t*)d_out;
        d_d = (double*)(d_ids + (size_t)nq * k);
        d_nd = (int64_t*)(d_d + (size_t)nq * k);
        d_f = nullptr;
    }
    void* d_flag;
    VB_TRY(sc.take(64, &d_flag));

    // resident warps: a few CTAs per SM; every warp owns one visited table
    const int64_t want_ctas = (nq + HN_WARPS - 1) / HN_WARPS;
    int resident = 0;
    VB_TRY(hnsw_launch(h, g, qimg, qstride, nq, ef, k, nullptr, 0, 0, 0, nullptr, nullptr, nullptr, nullptr, nullptr, &resident));
    const int grid = (int)std::min<int64_t>(want_ctas, (int64_t)c.sm_count * std::max(1, resident));
    // layer-0 table: a search visits a few multiples of ef elements (about 20 ef at m = 16), and the table may fill to
    // three quarters.  It is sized tightly: the tables of all resident warps together should stay in L2 (64 KB per
    // warp did not: every visited probe of a 10 M-row bit graph went to DRAM), and the per-query clear
    // is proportional to it.  It grows on overflow -- the grown size is remembered per ef_search.
    uint32_t cap = 1u << 12;
    while (cap < (uint32_t)(ef * h.m * (VB_AB_VIS ? 2 : 4)) && cap < (1u << 22)) cap <<= 1;
    if (h.vis_hint_ef == ef && h.vis_hint_cap > cap) cap = h.vis_hint_cap;
    // the ef = 1 upper layers visit a few neighbour lists each
    uint32_t vis_upper = 1024;
    while (vis_upper < (uint32_t)(h.m * 16)) vis_upper <<= 1;
    for (int attempt = 0; attempt < 6; ++attempt) {
        if (attempt > 0) vis_upper = std::max<uint32_t>(vis_upper, cap / 8);
        const uint32_t vis_cap = cap + vis_upper;
        const size_t need = (size_t)grid * HN_WARPS * vis_cap * sizeof(uint32_t);
        if (h.vis_bytes < need) {
            if (h.vis) {
                VB_CUDA(cudaStreamSynchronize(s));
                cudaFree(h.vis);
                h.vis = nullptr;
                h.vis_bytes = 0;
            }
            if (cudaMalloc(&h.vis, need) != cudaSuccess) {
                set_error("hnsw: visited tables (%zu bytes) do not fit", need);
                return VB_ENOMEM;
            }
            h.vis_bytes = need;
        }
        VB_CUDA(cudaMemsetAsync(d_flag, 0, 2 * sizeof(int), s));   // overflow flag, query counter
        if (c.hnsw_l2_persist) hnsw_l2_window(s, h.vis, need, true);
        prof_begin(VB_PROF_HNSW);
        const int lrc = hnsw_launch(h, g, qimg, qstride, nq, ef, k, h.vis, vis_cap, vis_upper, grid, d_ids, d_f, d_d, d_nd, (int*)d_flag);
        prof_end(VB_PROF_HNSW);
        if (c.hnsw_l2_persist) hnsw_l2_window(s, nullptr, 0, false);
        VB_TRY(lrc);
        if (!host && attempt == 0) {
            // device variant stays asynchronous unless the table was too small; check lazily
        }
        int flag = 0;
        VB_CUDA(cudaMemcpyAsync(&flag, d_flag, sizeof(int), cudaMemcpyDeviceToHost, s));
        VB_CUDA(cudaStreamSynchronize(s));
        if (c.hnsw_l2_persist) {
            cudaCtxResetPersistingL2Cache();   // the walk is over: hand the set-aside lines back to everybody
            cudaGetLastError();
        }
        if (!flag) break;
        cap <<= 2;   // visited table overflowed for some query: retry everything with a larger one
        h.vis_hint_ef = ef;
        h.vis_hint_cap = cap;
        VB_REQUIRE(attempt < 5, "hnsw: visited set overflow");
    }
    if (host) {
        VB_CUDA(cudaMemcpyAsync(out_ids, d_ids, sizeof(int64_t) * (size_t)nq * k, cudaMemcpyDeviceToHost, s));
        VB_CUDA(cudaMemcpyAsync(out_d, d_d, sizeof(double) * (size_t)nq * k, cudaMemcpyDeviceToHost, s));
        if (out_nd) VB_CUDA(cudaMemcpyAsync(out_nd, d_nd, sizeof(int64_t) * (size_t)nq, cudaMemcpyDeviceToHost, s));
        VB_CUDA(cudaStreamSynchronize(s));
    }
    return VB_OK;
}

void hnsw_release(Hnsw& h) {
    table_free(h.rows);
    cudaFree(h.levels);
    cudaFree(h.nbr0);
    cudaFree(h.upper_off);
    cudaFree(h.upper);
    cudaFree(h.vis);
    cudaFree(h.nd0);
    cudaFree(h.upper_d);
    cudaFree(h.dup_of);
    cudaFree(h.n_heaptids);
    cudaFree(h.rec_key);
    cudaFree(h.rec_val);
    h.levels = h.nbr0 = h.upper_off = h.upper = nullptr;
    h.nd0 = h.upper_d = nullptr;
    h.dup_of = h.n_heaptids = nullptr;
    h.rec_key = nullptr;
    h.rec_val = nullptr;
    h.vis = nullptr;
    h.vis_bytes = 0;
    h.upper_slots = 0;
    h.elem_cap = h.slot_cap = h.rec_cap = h.n_changes = 0;
    h.loaded = false;
}

}  // namespace vb

using namespace vb;

extern "C" {

int vb_hnsw_create(int elem, int metric, int dim, int m, vb_hnsw** out) {
    VB_TRY(require_init());
    VB_REQUIRE(out && elem >= 0 && elem <= 2 && dim > 0, "bad hnsw arguments");
    VB_REQUIRE(m >= 2 && m <= 100, "m must be 2..100 (src/hnsw.h:54-56)");
    bool ok = elem == VB_BIT ? (metric == VB_HAMMING || metric == VB_JACCARD)
                             : (metric == VB_L2_SQUARED || metric == VB_NEG_IP || metric == VB_L1);
    VB_REQUIRE(ok, "hnsw opclass proc 1 must be L2 squared / negative inner product / L1 (vector, halfvec) or Hamming / Jaccard (bit)");
    vb_hnsw* p = new vb_hnsw();
    p->h.elem = elem;
    p->h.metric = metric;
    p->h.dim = dim;
    p->h.m = m;
    p->h.rows.elem = elem;
    p->h.rows.dim = dim;
    p->h.rows.stride = padded_row_bytes(elem, dim);
    *out = p;
    return VB_OK;
}

int vb_hnsw_load(vb_hnsw* p, const void* rows, int64_t n, const int32_t* levels, const int32_t* nbr0, const int64_t* upper_off,
                 const int32_t* upper, int64_t upper_slots, int64_t entry) {
    VB_TRY(require_init());
    VB_REQUIRE(p && n >= 0 && n < (int64_t)0x7fffffff, "bad hnsw load arguments");
    Hnsw& h = p->h;
    hnsw_release(h);
    ++h.generation;
    h.n = n;
    h.entry = n > 0 ? entry : -1;
    if (n == 0) {
        h.loaded = true;
        return VB_OK;
    }
    VB_REQUIRE(rows && levels && nbr0 && upper_off && entry >= 0 && entry < n, "null graph arrays / bad entry point");
    VB_TRY(table_append_host(h.rows, rows, n));
    const int lm0 = 2 * h.m;
    std::vector<int32_t> uo((size_t)n);
    for (int64_t i = 0; i < n; ++i) {
        VB_REQUIRE(upper_off[i] < (int64_t)0x7fffffff, "upper slot overflow");
        uo[(size_t)i] = (int32_t)upper_off[i];
        VB_REQUIRE(levels[i] == 0 || upper_off[i] >= 0, "element %lld has level %d but no upper slot", (long long)i, levels[i]);
    }
    h.entry_level = levels[entry];
    VB_CUDA(cudaMalloc(&h.levels, sizeof(int32_t) * (size_t)n));
    VB_CUDA(cudaMalloc(&h.nbr0, sizeof(int32_t) * (size_t)n * lm0));
    VB_CUDA(cudaMalloc(&h.upper_off, sizeof(int32_t) * (size_t)n));
    VB_CUDA(cudaMalloc(&h.upper, sizeof(int32_t) * (size_t)std::max<int64_t>(upper_slots, 1) * h.m));
    VB_CUDA(cudaMemcpy(h.levels, levels, sizeof(int32_t) * (size_t)n, cudaMemcpyHostToDevice));
    VB_CUDA(cudaMemcpy(h.nbr0, nbr0, sizeof(int32_t) * (size_t)n * lm0, cudaMemcpyHostToDevice));
    VB_CUDA(cudaMemcpy(h.upper_off, uo.data(), sizeof(int32_t) * (size_t)n, cudaMemcpyHostToDevice));
    if (upper_slots > 0) VB_CUDA(cudaMemcpy(h.upper, upper, sizeof(int32_t) * (size_t)upper_slots * h.m, cudaMemcpyHostToDevice));
    h.upper_slots = upper_slots;
    h.elem_cap = n;
    h.slot_cap = std::max<int64_t>(upper_slots, 1);
    h.loaded = true;
    return VB_OK;
}

int vb_hnsw_free(vb_hnsw* p) {
    if (p) {
        hnsw_release(p->h);
        delete p;
    }
    return VB_OK;
}

int vb_hnsw_search(vb_hnsw* p, const void* queries, int64_t nq, int ef, int k, int64_t* out_ids, double* out_dist, int64_t* out_ndist) {
    VB_TRY(require_init());
    VB_REQUIRE(p && queries && out_ids && out_dist, "null argument");
    return hnsw_search_impl(p->h, queries, nq, ef, k, true, out_ids, nullptr, out_dist, out_ndist);
}

int vb_hnsw_search_dev(vb_hnsw* p, const void* queries_dev, int64_t nq, int ef, int k, int64_t* out_ids_dev, float* out_dist_dev,
                       int64_t* out_ndist_dev) {
    VB_TRY(require_init());
    VB_REQUIRE(p && queries_dev && out_ids_dev && out_dist_dev, "null argument");
    return hnsw_search_impl(p->h, queries_dev, nq, ef, k, false, out_ids_dev, out_dist_dev, nullptr, out_ndist_dev);
}

}  // extern "C"
