// vb_hnsw_iter.cu -- hnsw.iterative_scan on the device (src/hnswscan.c:62-87 ResumeScanItems, :228-340 hnswgettuple).
//
// The reference keeps, per scan, the visited hash `v` and a pairing heap `discarded` of every candidate that was
// seen but is not in W: neighbours rejected at :929-937 and elements W evicted at :968-973.  When the executor has
// consumed W it pulls the ef_search nearest discarded candidates, makes them the entry points of another layer-0
// HnswSearchLayer on the SAME visited set, and so on; once the `tuples` counter has reached hnsw.max_scan_tuples the
// remaining discarded candidates are returned nearest first without searching.
//
// Here a scan handle owns that state for a batch of queries (one warp per query, like vb_hnsw.cu):
//   vis   [nq][vis_cap]   the visited table, persistent across batches (open addressing, never cleared after batch 0)
//   dkey / did [nq][cap]  `discarded` as an append-only array (hnsw_search_layer<ITER> appends)
//   dlen, tuples, inserted, status per query
// vb_hnsw_scan_next() = one kernel: batch 0 is GetScanItems (:25-56); every later batch first selects the ef nearest
// discarded entries into R (the search's own sort / merge), compacts them out of the array, and either searches
// (ResumeScanItems) or, past max_scan_tuples, returns them as they are.  Under the total order (distance, element
// number) the sequence of elements is the oracle's (oracle/pgv_hnsw.c pgv_hnsw_iter_scan) element for element.
//
// A filtered handle (vb_hnsw_scan_begin_filtered) runs the same batches (VB_ITER_FIRST / VB_ITER_RESUME) inside
// hnsw_iter_filtered_kernel and returns pages of the elements each query's filter allows.
//
// Every counted tuple is visited once and ends in W or in `discarded`, so both arrays are bounded by
// min(n, max_scan_tuples + one batch); a batch is bounded generously (32 ef lists) and an overflow is an error.
// The reference's second bound, work_mem * hnsw.scan_mem_multiplier (:247), is the caller's to map onto
// max_scan_tuples (INTEGRATION.md).
#include "vb_hnsw.cuh"

#include <algorithm>
#include <vector>

namespace vb {

struct IterDev {
    uint32_t* vis;        // [nq][vis_cap]
    uint32_t vis_cap;
    uint32_t* vis_up;     // [resident warps][vis_upper]: the ef = 1 layers of batch 0
    uint32_t vis_upper;
    uint64_t* dkey;       // [nq][dcap]
    uint32_t* did;
    int dcap;
    int32_t* dlen;        // [nq]
    int64_t* tuples;      // [nq]
    uint32_t* inserted;   // [nq]
    int32_t* status;      // [nq] 0 = not started, 1 = running, 2 = exhausted
    int64_t max_tuples;
    int* overflow;
};

// The two kinds of underlying batch of one query into the warp's R (S, S.len == 0 on entry), shared by the unfiltered
// and the filtered kernel (template parameters ELEM, METRIC, LPR of the kernel that expands them); ok = false when a
// search overflowed its tables.  They are statement macros rather than inline functions: expanded in hnsw_iter_kernel
// they give it exactly the code it had with the bodies written out (identical SASS), which inlined functions, whose
// blocks the compiler lays out differently, do not.
//
// VB_ITER_FIRST: GetScanItems (src/hnswscan.c:25-56): entry point, ef = 1 descents, layer 0 with the discarded heap.
#define VB_ITER_FIRST(g, it, sq, ef, lane, S, sink, tuples, tab, vis_up, ok)                                                \
    {                                                                                                                       \
        Acc<ELEM, METRIC> acc;                                                                                              \
        const uint4* rp = reinterpret_cast<const uint4*>(g.rows + (size_t)g.entry * g.stride);                              \
        for (int v = lane; v < g.V; v += 32) hnsw_acc_add<ELEM, METRIC>(acc, ldg_stream(rp + v), sq, v);                    \
        acc.template reduce<32>();                                                                                          \
        if (lane == 0) {                                                                                                    \
            S.rk[0] = orderable_key64(acc.value());                                                                         \
            S.ri[0] = (uint32_t)g.entry;                                                                                    \
        }                                                                                                                   \
        S.len = 1;                                                                                                          \
        __syncwarp();                                                                                                       \
    }                                                                                                                       \
    for (int lc = g.entry_level; lc >= 1 && ok; --lc)                                                                       \
        ok = hnsw_search_layer<ELEM, METRIC, LPR>(g, sq, lc, 1, lane, S, vis_up, it.vis_upper, nullptr);                    \
    if (ok) ok = hnsw_search_layer<ELEM, METRIC, LPR, true>(g, sq, 0, ef, lane, S, tab, it.vis_cap, &tuples, &sink, true);

// VB_ITER_RESUME: a later batch (sink.len > 0): the ef nearest discarded candidates (src/hnswscan.c:73-84), nearest
// first, all unexpanded, taken out of the array; then ResumeScanItems from them, unless the tuple budget is spent
// (src/hnswscan.c:247-254: the rest is returned as it is).
#define VB_ITER_RESUME(g, it, sq, ef, lane, S, sink, tuples, tab, ok)                                                    \
    for (int b0 = 0; b0 < sink.len; b0 += 32) {                                                                          \
        const int i = b0 + lane;                                                                                         \
        const int cnt = min(32, sink.len - b0);                                                                          \
        if (i < sink.len) {                                                                                              \
            S.bkey[lane] = sink.key[i];                                                                                  \
            S.bid[lane] = sink.id[i];                                                                                    \
        }                                                                                                                \
        __syncwarp();                                                                                                    \
        hnsw_merge_batch<false>(S, cnt, ef, lane, nullptr);                                                              \
        __syncwarp();                                                                                                    \
    }                                                                                                                    \
    /* take them out of the array: everything not after R's last element in the total order */                           \
    {                                                                                                                    \
        const uint64_t wk = S.rk[S.len - 1];                                                                             \
        const uint32_t wi = S.ri[S.len - 1];                                                                             \
        int out = 0;                                                                                                     \
        for (int b0 = 0; b0 < sink.len; b0 += 32) {                                                                      \
            const int i = b0 + lane;                                                                                     \
            uint64_t k0 = 0;                                                                                             \
            uint32_t i0 = 0;                                                                                             \
            bool stay = false;                                                                                           \
            if (i < sink.len) {                                                                                          \
                k0 = sink.key[i];                                                                                        \
                i0 = sink.id[i];                                                                                         \
                stay = ent_less(wk, wi, k0, i0);                                                                         \
            }                                                                                                            \
            const unsigned sm = __ballot_sync(0xffffffffu, stay);                                                        \
            __syncwarp();                                                                                                \
            if (stay) {                                                                                                  \
                const int p = out + __popc(sm & ((1u << lane) - 1u));                                                    \
                sink.key[p] = k0;                                                                                        \
                sink.id[p] = i0;                                                                                         \
            }                                                                                                            \
            out += __popc(sm);                                                                                           \
            __syncwarp();                                                                                                \
        }                                                                                                                \
        sink.len = out;                                                                                                  \
    }                                                                                                                    \
    if (tuples < it.max_tuples)                                                                                          \
        ok = hnsw_search_layer<ELEM, METRIC, LPR, true>(g, sq, 0, ef, lane, S, tab, it.vis_cap, &tuples, &sink, false);

template <int ELEM, int METRIC, int LPR>
__global__ void VB_HNSW_BOUNDS hnsw_iter_kernel(HnswDev g, IterDev it, const uint8_t* __restrict__ queries, size_t qstride,
                                                                  int64_t nq, int ef, int64_t* __restrict__ out_ids,
                                                                  double* __restrict__ out_d, int32_t* __restrict__ out_cnt) {
    extern __shared__ uint4 smem[];
    const int warp = threadIdx.x / 32, lane = threadIdx.x % 32;
    const int qvec = (int)(qstride / 16);
    // per-warp carve-up as in hnsw_search_kernel: query image | keys A | keys B | batch keys | ids A | ids B | batch ids
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
    uint32_t* vis_up = it.vis_up + (size_t)gwarp * it.vis_upper;

    for (int64_t q = gwarp; q < nq; q += nwarps) {
        const int st = it.status[q];
        if (st == 2) {
            for (int i = lane; i < ef; i += 32) {
                out_ids[q * ef + i] = -1;
                out_d[q * ef + i] = (double)INFINITY;
            }
            if (lane == 0) out_cnt[q] = 0;
            continue;
        }
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
        HnswSink sink;
        sink.key = it.dkey + (size_t)q * it.dcap;
        sink.id = it.did + (size_t)q * it.dcap;
        sink.len = it.dlen[q];
        sink.cap = it.dcap;
        sink.inserted = it.inserted[q];
        int64_t tuples = it.tuples[q];
        uint32_t* tab = it.vis + (size_t)q * it.vis_cap;
        bool ok = true;

        if (st == 0) {
            VB_ITER_FIRST(g, it, sq, ef, lane, S, sink, tuples, tab, vis_up, ok);
        } else if (sink.len == 0) {
            // nothing left to resume from (src/hnswscan.c:69-70, 249-250)
            for (int i = lane; i < ef; i += 32) {
                out_ids[q * ef + i] = -1;
                out_d[q * ef + i] = (double)INFINITY;
            }
            if (lane == 0) {
                out_cnt[q] = 0;
                it.status[q] = 2;
            }
            continue;
        } else {
            VB_ITER_RESUME(g, it, sq, ef, lane, S, sink, tuples, tab, ok);
        }

        if (!ok || sink.len > sink.cap) {
            if (lane == 0) atomicExch(it.overflow, 1);
            ok = false;
        }
        // this batch nearest first (hnswgettuple pops llast(w), src/hnswscan.c:293-326)
        for (int i = lane; i < ef; i += 32) {
            const bool have = ok && i < S.len;
            out_ids[q * ef + i] = have ? (int64_t)(S.ri[i] & 0x7fffffffu) : -1;
            out_d[q * ef + i] = have ? key64_to_double(S.rk[i]) : (double)INFINITY;
        }
        if (lane == 0) {
            out_cnt[q] = ok ? S.len : 0;
            it.dlen[q] = min(sink.len, sink.cap);
            it.tuples[q] = tuples;
            it.inserted[q] = sink.inserted;
            it.status[q] = 1;
        }
        __syncwarp();
    }
}


// ------------------------------------------------------------------------------------------------ filtered handle
// A filtered handle returns, per query, the unfiltered sequence restricted to the elements its filter allows, `page` at
// a time.  The traversal is the unfiltered one (rejected elements are visited, expanded, counted and discarded as in the
// reference, where the predicate is applied above the index); only the output is filtered, in the kernel.
struct IterFilt {
    const uint32_t* bits;   // [nfilters][words] the filters' bitsets
    int64_t words;
    const int32_t* fq;      // [nq] the filter of each query
    uint64_t* ckey;         // [nq][ef] carry: the part of the last batch a full page left unconsumed
    uint32_t* cid;
    int32_t* cpos;          // [nq] its first unconsumed entry
    int32_t* clen;          // [nq] its length
    int* next_q;            // queries handed out so far in this call
    int page;
};

__device__ __forceinline__ bool elem_allowed(const uint32_t* __restrict__ bits, uint32_t e) {
    return (__ldg(bits + (e >> 5)) >> (e & 31)) & 1u;
}

// Append the entries of key / id [from, len) that bits allows to out[emitted ..], in order, until page are out (one bitset
// word per lane and a ballot per 32 entries).  Returns the index after the last entry consumed: len unless the page filled.
__device__ __forceinline__ int emit_allowed(const uint64_t* key, const uint32_t* id, int from, int len, const uint32_t* __restrict__ bits,
                                            int page, int& emitted, int64_t* __restrict__ out_ids, double* __restrict__ out_d, int lane) {
    for (int b0 = from; b0 < len; b0 += 32) {
        const int i = b0 + lane;
        uint32_t e = 0;
        uint64_t k = 0;
        bool allow = false;
        if (i < len) {
            e = id[i] & 0x7fffffffu;
            k = key[i];
            allow = elem_allowed(bits, e);
        }
        unsigned m = __ballot_sync(0xffffffffu, allow);
        while (__popc(m) > page - emitted) m &= ~(0x80000000u >> __clz(m));   // the first page - emitted of them
        if ((m >> lane) & 1u) {
            const int p = emitted + __popc(m & ((1u << lane) - 1u));
            out_ids[p] = (int64_t)e;
            out_d[p] = key64_to_double(k);
        }
        emitted += __popc(m);
        if (emitted == page) return b0 + 32 - __clz(m);
    }
    return len;
}

// One warp per query, queries handed out from a counter (the batches a query needs per call range from none to the
// whole scan).  Per query: emit from the carry, then run underlying batches while the page is not full, emitting each
// batch's allowed elements; a batch the page cannot take whole is carried to the next call.  So a batch runs only when
// the previous one is consumed and the page still has room: `tuples` after a call that fills its page is the unfiltered
// handle's after the batch of the call's last element.
// status: 0 = not started, 1 = running, 3 = draining with the rejected entries compacted out, 2 = exhausted.
template <int ELEM, int METRIC, int LPR>
__global__ void VB_HNSW_BOUNDS hnsw_iter_filtered_kernel(HnswDev g, IterDev it, IterFilt f, const uint8_t* __restrict__ queries,
                                                         size_t qstride, int64_t nq, int ef, int64_t* __restrict__ out_ids,
                                                         double* __restrict__ out_d, int32_t* __restrict__ out_cnt) {
    extern __shared__ uint4 smem[];
    const int warp = threadIdx.x / 32, lane = threadIdx.x % 32;
    const int qvec = (int)(qstride / 16);
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
    uint32_t* vis_up = it.vis_up + (size_t)gwarp * it.vis_upper;
    const int page = f.page;

    for (;;) {
        int64_t q = 0;
        if (lane == 0) q = atomicAdd(f.next_q, 1);
        q = __shfl_sync(0xffffffffu, q, 0);
        if (q >= nq) break;
        int64_t* oi = out_ids + q * page;
        double* od = out_d + q * page;
        int st = it.status[q];
        int emitted = 0;
        bool ok = true;
        if (st != 2) {
            const uint32_t* bits = f.bits + (size_t)f.fq[q] * f.words;
            uint64_t* ck = f.ckey + (size_t)q * ef;
            uint32_t* ci = f.cid + (size_t)q * ef;
            int cpos = f.cpos[q], clen = f.clen[q];
            if (cpos < clen) cpos = emit_allowed(ck, ci, cpos, clen, bits, page, emitted, oi, od, lane);
            if (emitted < page) {
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
                HnswSink sink;
                sink.key = it.dkey + (size_t)q * it.dcap;
                sink.id = it.did + (size_t)q * it.dcap;
                sink.len = it.dlen[q];
                sink.cap = it.dcap;
                sink.inserted = it.inserted[q];
                int64_t tuples = it.tuples[q];
                uint32_t* tab = it.vis + (size_t)q * it.vis_cap;
                while (emitted < page) {
                    if (st == 1 && tuples >= it.max_tuples) {
                        // past max_scan_tuples the rest of the sequence is the discarded candidates nearest first, with no
                        // search: drop the rejected ones once, so that every later step selects allowed entries only
                        int out = 0;
                        for (int b0 = 0; b0 < sink.len; b0 += 32) {
                            const int i = b0 + lane;
                            uint64_t k0 = 0;
                            uint32_t i0 = 0;
                            bool keep = false;
                            if (i < sink.len) {
                                k0 = sink.key[i];
                                i0 = sink.id[i];
                                keep = elem_allowed(bits, i0);
                            }
                            const unsigned km = __ballot_sync(0xffffffffu, keep);
                            __syncwarp();
                            if (keep) {
                                const int p = out + __popc(km & ((1u << lane) - 1u));
                                sink.key[p] = k0;
                                sink.id[p] = i0;
                            }
                            out += __popc(km);
                            __syncwarp();
                        }
                        sink.len = out;
                        st = 3;
                    }
                    S.len = 0;
                    if (st == 0) {
                        VB_ITER_FIRST(g, it, sq, ef, lane, S, sink, tuples, tab, vis_up, ok);
                    } else if (sink.len == 0) {
                        st = 2;   // nothing left to resume from (src/hnswscan.c:69-70, 249-250)
                        break;
                    } else {
                        VB_ITER_RESUME(g, it, sq, ef, lane, S, sink, tuples, tab, ok);
                    }
                    if (!ok || sink.len > sink.cap) {
                        if (lane == 0) atomicExch(it.overflow, 1);
                        ok = false;
                        break;
                    }
                    if (st == 0) st = 1;
                    const int used = emit_allowed(S.rk, S.ri, 0, S.len, bits, page, emitted, oi, od, lane);
                    for (int i = used + lane; i < S.len; i += 32) {
                        ck[i - used] = S.rk[i];
                        ci[i - used] = S.ri[i];
                    }
                    cpos = 0;
                    clen = S.len - used;
                    __syncwarp();
                }
                if (lane == 0) {
                    it.dlen[q] = min(sink.len, sink.cap);
                    it.tuples[q] = tuples;
                    it.inserted[q] = sink.inserted;
                }
            }
            if (lane == 0) {
                f.cpos[q] = cpos;
                f.clen[q] = clen;
                it.status[q] = st;
            }
        }
        if (!ok) emitted = 0;
        for (int i = emitted + lane; i < page; i += 32) {
            oi[i] = -1;
            od[i] = (double)INFINITY;
        }
        if (lane == 0) out_cnt[q] = emitted;
        __syncwarp();
    }
}

#undef VB_ITER_FIRST
#undef VB_ITER_RESUME

}  // namespace vb

using namespace vb;

struct vb_hnsw_scan {
    vb_hnsw* ix = nullptr;
    int64_t nq = 0;
    int ef = 0;
    void* qimg = nullptr;
    size_t qstride = 0;
    IterDev it{};
    int grid = 0;
    size_t smem = 0;
    void* out = nullptr;   // device results of one call: ids | distances | counts, [nq][width()]
    // filtered handles (page > 0): the filters' bitsets, the carries and the work counter in one allocation
    int page = 0;
    uint64_t generation = 0;   // the image's generation at begin
    IterFilt f{};
    void* fmem = nullptr;
    int width() const { return page ? page : ef; }
};

namespace vb {

template <int ELEM, int METRIC>
static int iter_launch_t(const HnswDev& g, vb_hnsw_scan& sc, int* occ_out) {
    cudaStream_t s = ctx().stream;
    int64_t* d_ids = (int64_t*)sc.out;
    double* d_d = (double*)(d_ids + (size_t)sc.nq * sc.width());
    int32_t* d_cnt = (int32_t*)(d_d + (size_t)sc.nq * sc.width());
#define VB_HK(KERN, ...)                                                                                                     \
    do {                                                                                                                     \
        auto kern = KERN;                                                                                                    \
        if (sc.smem > 48 * 1024) VB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sc.smem)); \
        if (occ_out) {                                                                                                       \
            VB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(occ_out, kern, HN_WARPS * 32, sc.smem));                   \
            return VB_OK;                                                                                                    \
        }                                                                                                                    \
        kern<<<sc.grid, HN_WARPS * 32, sc.smem, s>>>(__VA_ARGS__);                                                           \
    } while (0)
#define VB_HL(LPR)                                                                                                           \
    do {                                                                                                                     \
        if (sc.page) {                                                                                                       \
            if (!occ_out) VB_CUDA(cudaMemsetAsync(sc.f.next_q, 0, sizeof(int), s));                                          \
            VB_HK((hnsw_iter_filtered_kernel<ELEM, METRIC, LPR>), g, sc.it, sc.f, (const uint8_t*)sc.qimg, sc.qstride, sc.nq, \
                  sc.ef, d_ids, d_d, d_cnt);                                                                                 \
        } else {                                                                                                             \
            VB_HK((hnsw_iter_kernel<ELEM, METRIC, LPR>), g, sc.it, (const uint8_t*)sc.qimg, sc.qstride, sc.nq, sc.ef, d_ids, d_d, \
                  d_cnt);                                                                                                    \
        }                                                                                                                    \
    } while (0)
    if (g.V >= 32) VB_HL(32);
    else if (g.V >= 8) VB_HL(4);
    else VB_HL(1);
#undef VB_HL
#undef VB_HK
    VB_CUDA(cudaGetLastError());
    count_launch();
    return VB_OK;
}

static int iter_launch(const Hnsw& h, const HnswDev& g, vb_hnsw_scan& sc, int* occ_out = nullptr) {
#define VB_HC(E, M) return iter_launch_t<E, M>(g, sc, occ_out)
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

static HnswDev iter_view(const Hnsw& h) {
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
    return g;
}

static void iter_free(vb_hnsw_scan* sc) {
    if (!sc) return;
    cudaFree(sc->qimg);
    cudaFree(sc->it.vis);
    cudaFree(sc->it.vis_up);
    cudaFree(sc->it.dkey);
    cudaFree(sc->it.did);
    cudaFree(sc->it.dlen);
    cudaFree(sc->it.tuples);
    cudaFree(sc->it.inserted);
    cudaFree(sc->it.status);
    cudaFree(sc->it.overflow);
    cudaFree(sc->out);
    cudaFree(sc->fmem);
    delete sc;
}

// The filtered handle's own allocation: ckey [nq][ef] | bits [nfilters][words] | cid [nq][ef] | fq, cpos, clen [nq] |
// next_q.  Returns its size; with base != nullptr also points f's arrays into it.
static size_t iter_filter_carve(IterFilt& f, int64_t nq, int ef, int nfilters, uint8_t* base) {
    size_t o = 0;
    auto take = [&](size_t bytes) {
        uint8_t* p = base ? base + o : nullptr;
        o += (bytes + 15) & ~(size_t)15;
        return p;
    };
    f.ckey = (uint64_t*)take(8 * (size_t)nq * ef);
    f.bits = (const uint32_t*)take(4 * (size_t)nfilters * f.words);
    f.cid = (uint32_t*)take(4 * (size_t)nq * ef);
    f.fq = (const int32_t*)take(4 * (size_t)nq);
    f.cpos = (int32_t*)take(4 * (size_t)nq);
    f.clen = (int32_t*)take(4 * (size_t)nq);
    f.next_q = (int*)take(sizeof(int));
    return o;
}

static int hnsw_scan_begin_impl(const char* fn, vb_hnsw* ix, const void* queries, int64_t nq, int ef_search, int64_t max_scan_tuples,
                                int page, const vb_filter* const* filters, int nfilters, const int32_t* filter_of_query,
                                vb_hnsw_scan** out) {
    VB_TRY(require_init());
    VB_REQUIRE(ix && out && queries, "null argument");
    Hnsw& h = ix->h;
    VB_REQUIRE(h.loaded, "hnsw index not loaded");
    VB_REQUIRE(ef_search >= 1 && ef_search <= 1000, "ef_search must be 1..1000 (src/hnsw.h:60-62)");
    VB_REQUIRE(max_scan_tuples >= 1, "hnsw.max_scan_tuples must be >= 1 (src/hnsw.c:101-105)");
    VB_REQUIRE(nq >= 1, "no queries");
    const int64_t words = std::max<int64_t>(1, (h.n + 31) / 32);
    if (filters) {
        VB_REQUIRE(page >= 1 && page <= 2048, "%s: page must be in 1..2048 (got %d)", fn, page);
        VB_REQUIRE(nfilters >= 1, "%s: %d element filters", fn, nfilters);
        VB_REQUIRE(filter_of_query || nfilters == 1, "%s: filter_of_query may only be NULL with one filter (got %d)", fn, nfilters);
        for (int i = 0; i < nfilters; ++i) {
            VB_REQUIRE(filters[i], "%s: filter %d is NULL", fn, i);
            const Filter& f = filters[i]->f;
            VB_REQUIRE(f.kind == FILTER_HNSW && f.owner == ix && f.owner_uid == ix->uid, "%s: filter %d was made for another table or index",
                       fn, i);
            if (f.generation != h.generation) {
                set_error("%s: filter %d: index changed since the filter was created", fn, i);
                return VB_ESTATE;
            }
        }
        for (int64_t q = 0; q < nq && filter_of_query; ++q)
            VB_REQUIRE(filter_of_query[q] >= 0 && filter_of_query[q] < nfilters, "%s: filter_of_query[%lld] = %d, not in 0..%d", fn,
                       (long long)q, filter_of_query[q], nfilters - 1);
    }
    Context& c = ctx();
    cudaStream_t s = c.stream;
    vb_hnsw_scan* sc = new vb_hnsw_scan();
    sc->ix = ix;
    sc->nq = nq;
    sc->ef = ef_search;
    sc->page = filters ? page : 0;
    sc->generation = h.generation;
    sc->f.page = sc->page;
    sc->f.words = words;
    const int64_t n = std::max<int64_t>(h.n, 1);
    // every element is counted at most once; one batch may run past the budget by what it visits (bounded generously)
    const int64_t batch_bound = (int64_t)32 * ef_search * 2 * h.m;
    const int64_t dcap = std::min<int64_t>(n, max_scan_tuples + batch_bound) + 32;
    uint32_t vis_cap = 1u << 12;
    while ((int64_t)vis_cap < 2 * dcap + 64 && vis_cap < (1u << 30)) vis_cap <<= 1;
    uint32_t vis_upper = 1024;
    while (vis_upper < (uint32_t)(h.m * 16)) vis_upper <<= 1;
    const size_t per_query = (size_t)vis_cap * 4 + (size_t)dcap * 12;
    const size_t fbytes = filters ? iter_filter_carve(sc->f, nq, ef_search, nfilters, nullptr) : 0;
    if ((double)per_query * (double)nq + (double)fbytes > 64e9) {
        delete sc;
        set_error("iterative scan state of %lld queries x %zu bytes%s does not fit; scan fewer queries at once or lower max_scan_tuples",
                  (long long)nq, per_query, filters ? " plus the filters and carries" : "");
        return VB_ENOMEM;
    }
    Scratch scratch;
    void* qimg;
    int rc = upload_queries(scratch, h.elem, h.dim, queries, nq, true, &qimg, &sc->qstride);
    if (rc != VB_OK) {
        delete sc;
        return rc;
    }
    const int qvec = (int)(sc->qstride / 16);
    size_t per_warp = (size_t)qvec * 16 + (size_t)ef_search * 2 * 8 + (size_t)ef_search * 2 * 4 + 32 * 8 + 32 * 4;
    per_warp = (per_warp + 15) & ~(size_t)15;
    sc->smem = per_warp * HN_WARPS;
    if (sc->smem > 200 * 1024) {
        delete sc;
        set_error("ef_search %d with this dimension needs %zu bytes of shared memory per CTA", ef_search, sc->smem);
        return VB_EINVAL;
    }
    IterDev& it = sc->it;
    it.vis_cap = vis_cap;
    it.vis_upper = vis_upper;
    it.dcap = (int)dcap;
    it.max_tuples = max_scan_tuples;
    HnswDev g = iter_view(h);
    int resident = 0;
    rc = iter_launch(h, g, *sc, &resident);
    if (rc != VB_OK) {
        delete sc;
        return rc;
    }
    sc->grid = (int)std::min<int64_t>((nq + HN_WARPS - 1) / HN_WARPS, (int64_t)c.sm_count * std::max(1, resident));
    const size_t out_bytes = (sizeof(int64_t) + sizeof(double)) * (size_t)nq * sc->width() + sizeof(int32_t) * (size_t)nq;
    bool ok = cudaMalloc(&sc->qimg, sc->qstride * (size_t)nq) == cudaSuccess &&
              cudaMalloc(&it.vis, (size_t)nq * vis_cap * 4) == cudaSuccess &&
              cudaMalloc(&it.vis_up, (size_t)sc->grid * HN_WARPS * vis_upper * 4) == cudaSuccess &&
              cudaMalloc(&it.dkey, (size_t)nq * dcap * 8) == cudaSuccess && cudaMalloc(&it.did, (size_t)nq * dcap * 4) == cudaSuccess &&
              cudaMalloc(&it.dlen, (size_t)nq * 4) == cudaSuccess && cudaMalloc(&it.tuples, (size_t)nq * 8) == cudaSuccess &&
              cudaMalloc(&it.inserted, (size_t)nq * 4) == cudaSuccess && cudaMalloc(&it.status, (size_t)nq * 4) == cudaSuccess &&
              cudaMalloc(&it.overflow, 64) == cudaSuccess && cudaMalloc(&sc->out, out_bytes) == cudaSuccess &&
              (!filters || cudaMalloc(&sc->fmem, fbytes) == cudaSuccess);
    if (!ok) {
        cudaGetLastError();
        iter_free(sc);
        set_error("iterative scan state does not fit in device memory");
        return VB_ENOMEM;
    }
    cudaMemcpyAsync(sc->qimg, qimg, sc->qstride * (size_t)nq, cudaMemcpyDeviceToDevice, s);
    cudaMemsetAsync(it.dlen, 0, (size_t)nq * 4, s);
    cudaMemsetAsync(it.tuples, 0, (size_t)nq * 8, s);
    cudaMemsetAsync(it.inserted, 0, (size_t)nq * 4, s);
    cudaMemsetAsync(it.status, 0, (size_t)nq * 4, s);
    cudaMemsetAsync(it.overflow, 0, 64, s);
    if (filters) {
        // the bitsets are copied: the filters may be freed as soon as begin returns
        IterFilt& f = sc->f;
        iter_filter_carve(f, nq, ef_search, nfilters, (uint8_t*)sc->fmem);
        for (int i = 0; i < nfilters; ++i)
            cudaMemcpyAsync((uint32_t*)f.bits + (size_t)i * words, filters[i]->f.bits, 4 * (size_t)words, cudaMemcpyDeviceToDevice, s);
        if (filter_of_query) cudaMemcpyAsync((int32_t*)f.fq, filter_of_query, 4 * (size_t)nq, cudaMemcpyHostToDevice, s);
        else cudaMemsetAsync((int32_t*)f.fq, 0, 4 * (size_t)nq, s);
        cudaMemsetAsync(f.cpos, 0, 4 * (size_t)nq, s);
        cudaMemsetAsync(f.clen, 0, 4 * (size_t)nq, s);
    }
    if (cudaStreamSynchronize(s) != cudaSuccess) {
        iter_free(sc);
        set_error("iterative scan: %s", cudaGetErrorString(cudaGetLastError()));
        return VB_ECUDA;
    }
    *out = sc;
    return VB_OK;
}

// Element filters: a bitset over the image's element numbers.  The image holds no heap TIDs, so the caller maps its
// allowed heap TIDs onto elements: an element is allowed when any of its heap TIDs passes (a GPU-built graph folds a
// duplicate row into another element, dup_of, whose TIDs it joins), and the caller withholds the rejected TIDs of an
// element the scan returns (INTEGRATION.md section 7c).
static int hnsw_filter_create(vb_hnsw* ix, const int64_t* elems, int64_t n, bool host, vb_filter** out) {
    VB_TRY(require_init());
    VB_REQUIRE(out, "vb_hnsw_filter_create: null filter pointer");
    *out = nullptr;
    if (!ix || !ix->h.loaded) {
        set_error("vb_hnsw_filter_create: index not loaded");
        return VB_ESTATE;
    }
    VB_REQUIRE(n >= 0 && (elems || n == 0), "vb_hnsw_filter_create: null elements or negative count %lld", (long long)n);
    const Hnsw& h = ix->h;
    if (host)
        for (int64_t i = 0; i < n; ++i)
            VB_REQUIRE(elems[i] >= 0 && elems[i] < h.n, "vb_hnsw_filter_create: elements[%lld] = %lld is not an element of the index (0..%lld)",
                       (long long)i, (long long)elems[i], (long long)h.n - 1);
    vb_filter* f = new vb_filter;
    f->f.owner = ix;
    f->f.owner_uid = ix->uid;
    f->f.generation = h.generation;
    const int rc = filter_build_hnsw(h.n, elems, n, host, &f->f);
    if (rc != VB_OK) {
        filter_release(&f->f);
        delete f;
        return rc;
    }
    *out = f;
    return VB_OK;
}

}  // namespace vb

extern "C" {

int vb_hnsw_scan_begin(vb_hnsw* ix, const void* queries, int64_t nq, int ef_search, int64_t max_scan_tuples, vb_hnsw_scan** out) {
    return hnsw_scan_begin_impl("vb_hnsw_scan_begin", ix, queries, nq, ef_search, max_scan_tuples, 0, nullptr, 0, nullptr, out);
}

int vb_hnsw_scan_begin_filtered(vb_hnsw* ix, const void* queries, int64_t nq, int ef_search, int64_t max_scan_tuples, int page,
                                const vb_filter* const* filters, int nfilters, const int32_t* filter_of_query, vb_hnsw_scan** out) {
    if (!filters) {
        set_error("vb_hnsw_scan_begin_filtered: no element filter given");
        if (out) *out = nullptr;
        return VB_EINVAL;
    }
    return hnsw_scan_begin_impl("vb_hnsw_scan_begin_filtered", ix, queries, nq, ef_search, max_scan_tuples, page, filters, nfilters,
                                filter_of_query, out);
}

int vb_hnsw_filter_create(vb_hnsw* ix, const int64_t* elements, int64_t n, vb_filter** out) {
    return hnsw_filter_create(ix, elements, n, true, out);
}

int vb_hnsw_filter_create_dev(vb_hnsw* ix, const int64_t* elements_dev, int64_t n, vb_filter** out) {
    return hnsw_filter_create(ix, elements_dev, n, false, out);
}

int vb_hnsw_scan_next(vb_hnsw_scan* sc, int64_t* out_ids, double* out_distances, int32_t* out_counts) {
    VB_TRY(require_init());
    VB_REQUIRE(sc && out_ids && out_distances && out_counts, "null argument");
    Hnsw& h = sc->ix->h;
    if (sc->page && (!h.loaded || h.generation != sc->generation)) {
        set_error("vb_hnsw_scan_next: index changed since the scan began");
        return VB_ESTATE;
    }
    VB_REQUIRE(h.loaded, "hnsw index not loaded");
    cudaStream_t s = ctx().stream;
    const size_t ne = (size_t)sc->nq * sc->width();
    if (h.entry < 0) {
        // empty index (src/hnswscan.c:44-45, 243-244)
        for (size_t i = 0; i < ne; ++i) {
            out_ids[i] = -1;
            out_distances[i] = INFINITY;
        }
        memset(out_counts, 0, sizeof(int32_t) * (size_t)sc->nq);
        return VB_OK;
    }
    HnswDev g = iter_view(h);
    prof_begin(VB_PROF_HNSW);
    VB_TRY(iter_launch(h, g, *sc));
    prof_end(VB_PROF_HNSW);
    int64_t* d_ids = (int64_t*)sc->out;
    double* d_d = (double*)(d_ids + ne);
    int32_t* d_cnt = (int32_t*)(d_d + ne);
    int flag = 0;
    VB_CUDA(cudaMemcpyAsync(out_ids, d_ids, sizeof(int64_t) * ne, cudaMemcpyDeviceToHost, s));
    VB_CUDA(cudaMemcpyAsync(out_distances, d_d, sizeof(double) * ne, cudaMemcpyDeviceToHost, s));
    VB_CUDA(cudaMemcpyAsync(out_counts, d_cnt, sizeof(int32_t) * (size_t)sc->nq, cudaMemcpyDeviceToHost, s));
    VB_CUDA(cudaMemcpyAsync(&flag, sc->it.overflow, sizeof(int), cudaMemcpyDeviceToHost, s));
    VB_CUDA(cudaStreamSynchronize(s));
    if (flag) {
        set_error("iterative scan: one batch visited more than 32 * ef_search neighbour lists beyond max_scan_tuples; the scan state is full");
        return VB_ENOMEM;
    }
    return VB_OK;
}

int vb_hnsw_scan_tuples(vb_hnsw_scan* sc, int64_t* out_tuples) {
    VB_TRY(require_init());
    VB_REQUIRE(sc && out_tuples, "null argument");
    cudaStream_t s = ctx().stream;
    VB_CUDA(cudaMemcpyAsync(out_tuples, sc->it.tuples, sizeof(int64_t) * (size_t)sc->nq, cudaMemcpyDeviceToHost, s));
    VB_CUDA(cudaStreamSynchronize(s));
    return VB_OK;
}

int vb_hnsw_scan_end(vb_hnsw_scan* sc) {
    if (!sc) return VB_OK;
    cudaStreamSynchronize(ctx().stream);
    iter_free(sc);
    return VB_OK;
}

}  // extern "C"
