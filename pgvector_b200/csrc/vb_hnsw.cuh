// vb_hnsw.cuh -- device pieces shared by the HNSW scan (vb_hnsw.cu) and the HNSW build (vb_hnsw_build.cu):
// the graph image, the per-warp visited hash, batched row scoring and HnswSearchLayer
// (src/hnswutils.c:824-987) in its sorted-array formulation.
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
// together: one neighbour-list read, lm independent row gathers in flight,
// a warp bitonic sort of the batch and a parallel merge into R.
#pragma once

#include "vb_common.cuh"
#include "vb_distance.cuh"

namespace vb {

struct HnswDev {
    const uint8_t* rows;
    size_t stride;
    int V;                    // 16-byte vectors per row
    const int32_t* levels;    // [n]
    const int32_t* nbr0;      // [n][2m]
    const int32_t* upper_off; // [n] slot index or -1
    const int32_t* upper;     // [slots][m]
    int m;
    int64_t n;
    int entry;
    int entry_level;
};

struct Hnsw {
    int elem, metric, dim, m;
    Table rows;
    int32_t *levels = nullptr, *nbr0 = nullptr, *upper_off = nullptr, *upper = nullptr;
    int64_t n = 0, entry = -1;
    int entry_level = -1;
    bool loaded = false;
    uint32_t* vis = nullptr;  // visited hash tables, one per resident warp
    size_t vis_bytes = 0;
    int vis_hint_ef = 0;        // the last ef_search whose layer-0 table had to grow, and the size it grew to
    uint32_t vis_hint_cap = 0;
    // build-side state (vb_hnsw_build.cu); nd0 / upper_d hold the distance stored with every neighbour
    // (HnswCandidate.distance, src/hnsw.h:143-148), dup_of the element a duplicate row was folded into
    float *nd0 = nullptr, *upper_d = nullptr;
    int32_t *dup_of = nullptr, *n_heaptids = nullptr;
    int64_t upper_slots = 0;
    uint64_t generation = 0;  // bumped by every load, build, insert and vacuum: filters and filtered scan handles refuse a changed image
    // capacities of the per-element arrays (levels, upper_off, nbr0, nd0, dup_of, n_heaptids) and of the upper slots
    // (upper, upper_d): vb_hnsw_insert grows them geometrically
    int64_t elem_cap = 0, slot_cap = 0;
    // the last insert's or vacuum's change records, sorted by (element, layer, slot): key = element << 14 | layer << 8 | slot
    uint64_t* rec_key = nullptr;
    int32_t* rec_val = nullptr;
    int64_t rec_cap = 0, n_changes = 0;
};

void hnsw_release(Hnsw& h);

constexpr int HN_WARPS = 4;             // queries (or inserted elements) per CTA

// Resident CTAs per SM the register allocation aims for.  Without the second __launch_bounds__ argument ptxas picks a
// target of its own per instantiation (56 .. 128 registers, the narrow-row ones with spills); the kernel waits on
// dependent gathers, so resident warps matter more than a spill-free loop.
#ifndef VB_HNSW_MINB
#define VB_HNSW_MINB 6
#endif
#if VB_HNSW_MINB > 0
#define VB_HNSW_BOUNDS __launch_bounds__(HN_WARPS * 32, VB_HNSW_MINB)
#else
#define VB_HNSW_BOUNDS __launch_bounds__(HN_WARPS * 32)
#endif
constexpr uint32_t VIS_EMPTY = 0xFFFFFFFFu;

__device__ __forceinline__ uint32_t hash_u32(uint32_t x) {
    x ^= x >> 16;
    x *= 0x7feb352du;
    x ^= x >> 15;
    x *= 0x846ca68bu;
    x ^= x >> 16;
    return x;
}

// returns true when id was NOT in the set (and inserts it)
__device__ __forceinline__ bool vis_insert(uint32_t* tab, uint32_t mask, uint32_t id) {
    uint32_t h = hash_u32(id) & mask;
    for (;;) {
        uint32_t old = atomicCAS(&tab[h], VIS_EMPTY, id);
        if (old == VIS_EMPTY) return true;
        if (old == id) return false;
        h = (h + 1) & mask;
    }
}

// Bucketed variant (VB_AB_VISB): the table is an array of 8-slot buckets, one 32-byte sector each.  A probe is ONE load
// round trip (two 16-byte loads of the same sector) instead of a chain of dependent atomicCAS round trips -- with linear
// probing the warp waited for the longest probe sequence of its 32 lanes, 3 - 4 atomics at the load factors of a search.
// The table belongs to one warp, so the only writers that can collide are lanes of the same call: they are arbitrated in
// registers (__match_any_sync on the slot they want, lowest lane wins, the others take the bucket's next empty slot) and
// the winners store plainly.  An id lives in the first bucket of its sequence that had an empty slot when it arrived;
// buckets never lose entries, so a lookup stops at the first bucket that holds the id or still has an empty slot.
// Warp-collective: every lane calls, lanes with want = true carry an id (< 2^31).  Returns true when the id was NOT in the
// set (and inserts it); a second lane carrying the same id in the same call reports "visited", like a second CAS would.
#ifndef VB_AB_VISB
#define VB_AB_VISB 1
#endif
__device__ __forceinline__ bool vis_insert_warp(uint32_t* tab, uint32_t mask, bool want, uint32_t id, int lane) {
    const uint32_t bmask = mask >> 3;
    const unsigned same = __match_any_sync(0xffffffffu, want ? id : (0x80000000u | (uint32_t)lane));
    bool pending = want && (__ffs(same) - 1 == lane);
    bool fresh = false;
    uint32_t b = hash_u32(id) & bmask;
    while (__any_sync(0xffffffffu, pending)) {
        unsigned empt = 0;
        if (pending) {
            const uint4* p = reinterpret_cast<const uint4*>(tab + ((size_t)b << 3));
            const uint4 s0 = __ldcg(p), s1 = __ldcg(p + 1);
            const bool found = s0.x == id || s0.y == id || s0.z == id || s0.w == id || s1.x == id || s1.y == id || s1.z == id || s1.w == id;
            if (found) {
                pending = false;
            } else {
                empt = (s0.x == VIS_EMPTY ? 1u : 0u) | (s0.y == VIS_EMPTY ? 2u : 0u) | (s0.z == VIS_EMPTY ? 4u : 0u) | (s0.w == VIS_EMPTY ? 8u : 0u) |
                       (s1.x == VIS_EMPTY ? 16u : 0u) | (s1.y == VIS_EMPTY ? 32u : 0u) | (s1.z == VIS_EMPTY ? 64u : 0u) | (s1.w == VIS_EMPTY ? 128u : 0u);
            }
        }
        bool claim = pending && empt != 0;
        while (__any_sync(0xffffffffu, claim)) {
            const uint32_t slot = (b << 3) + (uint32_t)(__ffs(empt) - 1);
            const unsigned peers = __match_any_sync(0xffffffffu, claim ? slot : (0x80000000u | (uint32_t)lane));
            if (claim) {
                if (__ffs(peers) - 1 == lane) {
                    __stcg(tab + slot, id);
                    fresh = true;
                    claim = false;
                    pending = false;
                } else {
                    empt &= empt - 1;            // taken by a lane of this call
                    if (empt == 0) claim = false; // the bucket filled up: on to the next one
                }
            }
        }
        if (pending) b = (b + 1) & bmask;
        __syncwarp();   // the stores above are visible to the loads of the next pass (and of the next call)
    }
    return fresh;
}

__device__ __forceinline__ bool ent_less(uint64_t ka, uint32_t ia, uint64_t kb, uint32_t ib) {
    return ka < kb || (ka == kb && (ia & 0x7fffffffu) < (ib & 0x7fffffffu));
}

// The "query image" the Acc<> arithmetic reads from shared memory.  vector and bit: the value as it is.  halfvec: widened
// to fp32 (exact, HalfToFloat4) for L2 / L1, whose subtraction takes an fp32 operand -- but kept as packed halves for the
// inner product, where one FHFMA per element multiplies two halves into the fp32 sum (half the shared-memory reads, no
// conversions; bit-identical to the widened arithmetic, see fh_fma).
template <int ELEM, int METRIC>
struct HnswImage {
#ifndef VB_AB_PACKED
#define VB_AB_PACKED 1
#endif
    static constexpr bool packed = VB_AB_PACKED && ELEM == VB_HALFVEC && METRIC == VB_NEG_IP;
};

template <int ELEM, int METRIC>
__device__ __forceinline__ void hnsw_acc_add(Acc<ELEM, METRIC>& acc, uint4 r, const uint4* sq, int v) {
    if (HnswImage<ELEM, METRIC>::packed) acc.add_h(r, sq[v]);
    else acc.add(r, sq, v);
}

// a table row as the image
template <int ELEM, int METRIC>
__device__ __forceinline__ void load_row_image(const uint8_t* row, int V, uint4* img, int lane) {
    const uint4* rp = reinterpret_cast<const uint4*>(row);
    for (int v = lane; v < V; v += 32) {
        const uint4 r = __ldg(rp + v);
        if (ELEM == VB_HALFVEC && !HnswImage<ELEM, METRIC>::packed) {
            const float2 x0 = __half22float2(*reinterpret_cast<const __half2*>(&r.x));
            const float2 x1 = __half22float2(*reinterpret_cast<const __half2*>(&r.y));
            const float2 x2 = __half22float2(*reinterpret_cast<const __half2*>(&r.z));
            const float2 x3 = __half22float2(*reinterpret_cast<const __half2*>(&r.w));
            img[2 * v] = make_uint4(__float_as_uint(x0.x), __float_as_uint(x0.y), __float_as_uint(x1.x), __float_as_uint(x1.y));
            img[2 * v + 1] = make_uint4(__float_as_uint(x2.x), __float_as_uint(x2.y), __float_as_uint(x3.x), __float_as_uint(x3.y));
        } else {
            img[v] = r;
        }
    }
}

// a query of the batch as the image: gq = what upload_queries() wrote (halfvec queries widened to fp32, qvec 16-byte
// words); V = 16-byte words of a table row
template <int ELEM, int METRIC>
__device__ __forceinline__ void load_query_image(const uint4* gq, int qvec, int V, uint4* img, int lane) {
    if (HnswImage<ELEM, METRIC>::packed) {
        for (int v = lane; v < V; v += 32) {
            const uint4 a = gq[2 * v], b = gq[2 * v + 1];
            const __half2 h0 = __floats2half2_rn(__uint_as_float(a.x), __uint_as_float(a.y));
            const __half2 h1 = __floats2half2_rn(__uint_as_float(a.z), __uint_as_float(a.w));
            const __half2 h2 = __floats2half2_rn(__uint_as_float(b.x), __uint_as_float(b.y));
            const __half2 h3 = __floats2half2_rn(__uint_as_float(b.z), __uint_as_float(b.w));
            img[v] = make_uint4(*reinterpret_cast<const uint32_t*>(&h0), *reinterpret_cast<const uint32_t*>(&h1),
                                *reinterpret_cast<const uint32_t*>(&h2), *reinterpret_cast<const uint32_t*>(&h3));
        }
    } else {
        for (int i = lane; i < qvec; i += 32) img[i] = gq[i];
    }
}

#ifndef VB_HNSW_EVICT_FIRST
#define VB_HNSW_EVICT_FIRST 1
#endif
// A/B switches of alternative search strategies (compile-time, off by default)
#ifndef VB_AB_PINGPONG
#define VB_AB_PINGPONG 1
#endif
#ifndef VB_AB_RANKSORT
#define VB_AB_RANKSORT 1
#endif
#ifndef VB_AB_INPLACE
#define VB_AB_INPLACE 1
#endif
#ifndef VB_AB_VCACHE
#define VB_AB_VCACHE 0
#endif
// rows in flight per lane group for rows narrower than a warp pass (bit(1024): 8 lanes per row, one 16-byte word per lane):
// 2 = 8 rows per pass, 4 = 16, 8 = 32 (a whole expansion in one round trip of the gather)
#ifndef VB_AB_RPI_NARROW
#define VB_AB_RPI_NARROW 2
#endif
// prefetch (into L2) the layer-0 neighbour list of every element that is about to be admitted to R: it is read when the
// element is expanded, many expansions later, and would otherwise be a dependent DRAM round trip at the top of the loop
#ifndef VB_AB_NBRPF
#define VB_AB_NBRPF 0
#endif
// rows of <= 96 words on a whole warp (LPR 32): W rows per pass with all three words per lane in flight (0 = the generic
// two-steps-in-flight walk)
#ifndef VB_AB_WIDE1
#define VB_AB_WIDE1 0
#endif
// rows in flight per pass for whole-warp rows (LPR 32): 4 (fewer leave registers for more resident CTAs, see VB_HNSW_MINB)
#ifndef VB_AB_RPI_WIDE
#define VB_AB_RPI_WIDE 4
#endif
// narrow rows: score all listed neighbours while their visited probes are in flight (see hnsw_search_layer).  Measured on
// config E (10M x bit(1024), ef_search 200) it ran slower with it than without -- the wasted scorings cost more than the
// overlapped round trip saves; kept as a switch
#ifndef VB_AB_SPEC
#define VB_AB_SPEC 0
#endif
// layer 0: while the neighbours of the nearest unexpanded element are processed, the neighbour list of the SECOND nearest
// unexpanded element is requested -- it is the next one to be expanded unless this expansion admits something nearer --
// and, for rows of at most 256 bytes, the rows it names are prefetched into L2.  Data movement only: the walk, the
// visited set and the `tuples` counter are untouched.  (Two of the three dependent round trips of an expansion -- list,
// visited bucket, rows -- leave the critical path when the guess holds.)
#ifndef VB_AB_NEXTPF
#define VB_AB_NEXTPF 0
#endif
__device__ __forceinline__ uint4 hnsw_row_ld(const uint4* p) {
#if VB_HNSW_EVICT_FIRST
    return ldg_gather(p);
#else
    return ldg_stream(p);
#endif
}

// distances of the image `sq` to the rows bid[0..cnt): GROUPS rows per pass (LPR lanes per row), RPI passes in flight.
// bkey[i] = orderable key of the float8 the opclass's proc 1 returns.
template <int ELEM, int METRIC, int LPR>
__device__ __forceinline__ void hnsw_score_batch(const HnswDev& g, const uint4* sq, const uint32_t* bid, int cnt, uint64_t* bkey,
                                                 int lane) {
    constexpr int GROUPS = 32 / LPR;
    constexpr int RPI = (LPR == 32) ? VB_AB_RPI_WIDE : VB_AB_RPI_NARROW;   // (LPR 32: 8 in flight measured the same: 821 k vs 816 k queries/s, at 128 registers)
    const int grp = lane / LPR, gl = lane % LPR;
    if constexpr (LPR == 8) {
        // rows of at most 8 words (bit(1024) = 128 bytes): one word per lane and 8 rows per lane group, so the <= 32 rows of
        // an expansion are ONE round trip with every load in flight (the generic path below walks a row in steps of LPR words
        // with two steps in flight)
        if (g.V <= 8) {
            constexpr int R1 = 8;
            for (int b0 = 0; b0 < cnt; b0 += GROUPS * R1) {
                Acc<ELEM, METRIC> acc[R1];
                uint4 w[R1];
#pragma unroll
                for (int i = 0; i < R1; ++i) {
                    const int bi = b0 + i * GROUPS + grp;
                    const uint32_t e = bid[min(bi, cnt - 1)] & 0x7fffffffu;
                    w[i] = gl < g.V ? hnsw_row_ld(reinterpret_cast<const uint4*>(g.rows + (size_t)e * g.stride) + gl) : make_uint4(0, 0, 0, 0);
                }
#pragma unroll
                for (int i = 0; i < R1; ++i) {
                    if (gl < g.V) hnsw_acc_add<ELEM, METRIC>(acc[i], w[i], sq, gl);
                    acc[i].template reduce<LPR>();
                    const int bi = b0 + i * GROUPS + grp;
                    if (gl == 0 && bi < cnt) bkey[bi] = orderable_key64(acc[i].value());
                }
            }
            return;
        }
    }
#if VB_AB_WIDE1
    if constexpr (LPR == 32) {
        // rows of at most 96 words (768-d halfvec = 1536 bytes): the three words a lane owns of each of W1 rows are all
        // requested before the first is used -- one round trip per pass instead of two (the generic path keeps two of the
        // three steps in flight)
        if (g.V <= 96) {
            constexpr int W1 = VB_AB_WIDE1;
            for (int b0 = 0; b0 < cnt; b0 += W1) {
                Acc<ELEM, METRIC> acc[W1];
                uint4 w[W1][3];
#pragma unroll
                for (int i = 0; i < W1; ++i) {
                    const uint32_t e = bid[min(b0 + i, cnt - 1)] & 0x7fffffffu;
                    const uint4* rp = reinterpret_cast<const uint4*>(g.rows + (size_t)e * g.stride);
#pragma unroll
                    for (int t = 0; t < 3; ++t) w[i][t] = lane + 32 * t < g.V ? hnsw_row_ld(rp + lane + 32 * t) : make_uint4(0, 0, 0, 0);
                }
#pragma unroll
                for (int i = 0; i < W1; ++i) {
#pragma unroll
                    for (int t = 0; t < 3; ++t)
                        if (lane + 32 * t < g.V) hnsw_acc_add<ELEM, METRIC>(acc[i], w[i][t], sq, lane + 32 * t);
                    acc[i].template reduce<32>();
                    if (lane == 0 && b0 + i < cnt) bkey[b0 + i] = orderable_key64(acc[i].value());
                }
            }
            return;
        }
    }
#endif
    for (int b0 = 0; b0 < cnt; b0 += GROUPS * RPI) {
        Acc<ELEM, METRIC> acc[RPI];
        const uint4* rp[RPI];
#pragma unroll
        for (int i = 0; i < RPI; ++i) {
            int bi = b0 + i * GROUPS + grp;
            uint32_t e = bid[min(bi, cnt - 1)] & 0x7fffffffu;
            rp[i] = reinterpret_cast<const uint4*>(g.rows + (size_t)e * g.stride);
        }
#if VB_AB_PINGPONG
        // register double buffering: the loads of step v + LPR are issued before the arithmetic of step v, so 2 * RPI
        // independent 128-bit gathers per lane are in flight instead of one dependent round trip per step.  Two named
        // buffers alternate (no register copies between steps).
        uint4 bufa[RPI], bufb[RPI];
        if (gl < g.V) {
#pragma unroll
            for (int i = 0; i < RPI; ++i) bufa[i] = hnsw_row_ld(rp[i] + gl);
        }
        for (int v = gl; v < g.V; v += 2 * LPR) {
            const int v1 = v + LPR, v2 = v + 2 * LPR;
            if (v1 < g.V) {
#pragma unroll
                for (int i = 0; i < RPI; ++i) bufb[i] = hnsw_row_ld(rp[i] + v1);
            }
#pragma unroll
            for (int i = 0; i < RPI; ++i) hnsw_acc_add<ELEM, METRIC>(acc[i], bufa[i], sq, v);
            if (v1 < g.V) {
                if (v2 < g.V) {
#pragma unroll
                    for (int i = 0; i < RPI; ++i) bufa[i] = hnsw_row_ld(rp[i] + v2);
                }
#pragma unroll
                for (int i = 0; i < RPI; ++i) hnsw_acc_add<ELEM, METRIC>(acc[i], bufb[i], sq, v1);
            }
        }
#else
        uint4 cur[RPI];
        if (gl < g.V) {
#pragma unroll
            for (int i = 0; i < RPI; ++i) cur[i] = hnsw_row_ld(rp[i] + gl);
        }
        for (int v = gl; v < g.V; v += LPR) {
            uint4 nxt[RPI];
            const int vn = v + LPR;
            if (vn < g.V) {
#pragma unroll
                for (int i = 0; i < RPI; ++i) nxt[i] = hnsw_row_ld(rp[i] + vn);
            }
#pragma unroll
            for (int i = 0; i < RPI; ++i) hnsw_acc_add<ELEM, METRIC>(acc[i], cur[i], sq, v);
            if (vn < g.V) {
#pragma unroll
                for (int i = 0; i < RPI; ++i) cur[i] = nxt[i];
            }
        }
#endif
#pragma unroll
        for (int i = 0; i < RPI; ++i) {
            acc[i].template reduce<LPR>();
            int bi = b0 + i * GROUPS + grp;
            if (gl == 0 && bi < cnt) bkey[bi] = orderable_key64(acc[i].value());
        }
    }
}

// the two buffers of the sorted result array R and the expansion batch of one warp (shared memory)
struct HnswWarpState {
    uint64_t *rk, *nk;    // keys of R (current / next)
    uint32_t *ri, *ni;    // ids of R, bit 31 = expanded
    uint64_t* bkey;       // [32]
    uint32_t* bid;        // [32]
    int len;
    int vcn;              // entries of the visited cache (the unused second key buffer: 2 ef words), 0 = none
};

// The iterative scan's `discarded` heap (src/hnswscan.c:62-87, src/hnswutils.c:929-937, 968-973) as an append-only
// array of one query: candidates that were seen but are not in R -- rejected neighbours and elements R evicted.
struct HnswSink {
    uint64_t* key;
    uint32_t* id;
    int len;            // may run past cap: the caller reports the overflow
    int cap;
    uint32_t inserted;  // entries in the (persistent) visited table
};

__device__ __forceinline__ void hnsw_sink_append(HnswSink& d, bool have, uint64_t k, uint32_t id, int lane) {
    const unsigned m = __ballot_sync(0xffffffffu, have);
    if (m == 0) return;
    const int p = d.len + __popc(m & ((1u << lane) - 1u));
    if (have && p < d.cap) {
        d.key[p] = k;
        d.id[p] = id & 0x7fffffffu;
    }
    d.len += __popc(m);
}

// R <- the efl nearest of R and the batch bkey / bid [0..cnt) (unsorted, unexpanded); everything that does not stay
// goes to the sink when ITER.  Once R holds efl elements, an entry that is not nearer than R's last one cannot be
// admitted ("eDistance < f->distance || alwaysAdd", src/hnswutils.c:927-938): those are dropped before the sort, and
// the sort and the merge are skipped altogether when nothing is left -- the common case once a search has converged.
template <bool ITER>
__device__ __forceinline__ void hnsw_merge_batch(HnswWarpState& S, int cnt, int efl, int lane, HnswSink* sink) {
    int cnt_in = cnt;
    if (S.len == efl) {
        const uint64_t wk = S.rk[efl - 1];
        const uint32_t wi = S.ri[efl - 1];
        const uint64_t k0 = lane < cnt ? S.bkey[lane] : 0;
        const uint32_t i0 = lane < cnt ? S.bid[lane] : 0;
        const bool keep = lane < cnt && ent_less(k0, i0, wk, wi);
        const unsigned km = __ballot_sync(0xffffffffu, keep);
        cnt_in = __popc(km);
        if (ITER) hnsw_sink_append(*sink, lane < cnt && !keep, k0, i0, lane);
        if (cnt_in == 0) return;
        if (cnt_in < cnt) {
            __syncwarp();
            if (keep) {
                const int p = __popc(km & ((1u << lane) - 1u));
                S.bkey[p] = k0;
                S.bid[p] = i0;
            }
            __syncwarp();
        }
    }
    // sort the batch by (key, id).  A converged search admits one or two neighbours per expansion: up to 8 survivors are
    // ranked by counting (each lane counts the entries before its own: cnt_in broadcasts), more go through a bitonic
    // network over the 32 lanes (empty lanes = +inf).
    uint64_t mk = lane < cnt_in ? S.bkey[lane] : ~0ull;
    uint32_t mi = lane < cnt_in ? S.bid[lane] : 0x7fffffffu;
    if (VB_AB_RANKSORT && cnt_in <= 8) {
        int rank = 0;
        for (int j = 0; j < cnt_in; ++j) {
            const uint64_t kj = __shfl_sync(0xffffffffu, mk, j);
            const uint32_t ij = __shfl_sync(0xffffffffu, mi, j);
            rank += ent_less(kj, ij, mk, mi) ? 1 : 0;
        }
        __syncwarp();
        if (lane < cnt_in) {
            S.bkey[rank] = mk;
            S.bid[rank] = mi;
        }
        __syncwarp();
        mk = lane < cnt_in ? S.bkey[lane] : ~0ull;
        mi = lane < cnt_in ? S.bid[lane] : 0x7fffffffu;
    } else {
#pragma unroll
        for (int size = 2; size <= 32; size <<= 1) {
#pragma unroll
            for (int st = size >> 1; st > 0; st >>= 1) {
                uint64_t ok = __shfl_xor_sync(0xffffffffu, mk, st);
                uint32_t oi = __shfl_xor_sync(0xffffffffu, mi, st);
                bool up = (lane & size) == 0;
                bool lower = (lane & st) == 0;
                bool other_less = ent_less(ok, oi, mk, mi);
                // keep min in the lower lane of an ascending pair, max otherwise
                bool take = (lower == up) ? other_less : !other_less;
                if (take) {
                    mk = ok;
                    mi = oi;
                }
            }
        }
        __syncwarp();
        if (lane < cnt_in) {
            S.bkey[lane] = mk;
            S.bid[lane] = mi;
        }
        __syncwarp();
    }

#if VB_AB_INPLACE
    // merge the batch (cnt_in, sorted) into R (len, sorted) IN PLACE, keeping efl.  Every element's final position is
    // its index plus the number of elements of the other sequence before it.  The batch's positions are computed first
    // (R still untouched); R is then shifted right chunk by chunk from the END -- a chunk's elements are read by all
    // lanes before any of them is written, and they only move to higher indices, where everything has been relocated
    // already -- and the walk stops at the first chunk that lies entirely before the smallest batch element: on average
    // half of R is never touched (the two-buffer merge rewrote all of it: 34 % of the kernel's instructions at ef = 200).
    const int len = S.len;
    int npb = 0;
    if (lane < cnt_in) {
        int lo = 0, hi = len;   // number of R elements < batch[lane]
        while (lo < hi) {
            int mid = (lo + hi) >> 1;
            if (ent_less(S.rk[mid], S.ri[mid], mk, mi)) lo = mid + 1;
            else hi = mid;
        }
        npb = lane + lo;
    }
    __syncwarp();
    for (int j0 = ((len - 1) / 32) * 32; j0 >= 0; j0 -= 32) {
        const int j = j0 + lane;
        const bool act = j < len;
        uint64_t kj = 0;
        uint32_t ij = 0;
        int np = 0;
        if (act) {
            kj = S.rk[j];
            ij = S.ri[j];
            int lo = 0;   // number of batch elements < R[j]
            if (cnt_in <= 8) {
                for (int b = 0; b < cnt_in; ++b) lo += ent_less(S.bkey[b], S.bid[b], kj, ij) ? 1 : 0;
            } else {
                int hi = cnt_in;
                while (lo < hi) {
                    int mid = (lo + hi) >> 1;
                    if (ent_less(S.bkey[mid], S.bid[mid], kj, ij)) lo = mid + 1;
                    else hi = mid;
                }
            }
            np = j + lo;
        }
        // nothing of this chunk (nor of the ones before it) moves when even its last element precedes the batch
        const bool moves = act && np != j;
        if (__ballot_sync(0xffffffffu, moves) == 0) {
            // (the chunk may still hold elements that are past efl only if len > efl, which never happens)
            break;
        }
        __syncwarp();
        if (act && np < efl) {
            S.rk[np] = kj;
            S.ri[np] = ij;
        }
        if (ITER) hnsw_sink_append(*sink, act && np >= efl, kj, ij, lane);
        __syncwarp();
    }
    if (lane < cnt_in && npb < efl) {
        S.rk[npb] = mk;
        S.ri[npb] = mi;     // unexpanded
    }
    if (ITER) hnsw_sink_append(*sink, lane < cnt_in && npb >= efl, mk, mi, lane);
    __syncwarp();
    S.len = min(efl, len + cnt_in);
}
#else
    const int len = S.len;
    for (int j0 = 0; j0 < len; j0 += 32) {
        const int j = j0 + lane;
        const bool act = j < len;
        uint64_t kj = 0;
        uint32_t ij = 0;
        int np = 0;
        if (act) {
            kj = S.rk[j];
            ij = S.ri[j];
            int lo = 0, hi = cnt_in;   // number of batch elements < R[j]
            while (lo < hi) {
                int mid = (lo + hi) >> 1;
                if (ent_less(S.bkey[mid], S.bid[mid], kj, ij)) lo = mid + 1;
                else hi = mid;
            }
            np = j + lo;
            if (np < efl) {
                S.nk[np] = kj;
                S.ni[np] = ij;
            }
        }
        if (ITER) hnsw_sink_append(*sink, act && np >= efl, kj, ij, lane);
    }
    {
        int np = 0;
        if (lane < cnt_in) {
            int lo = 0, hi = len;   // number of R elements < batch[lane]
            while (lo < hi) {
                int mid = (lo + hi) >> 1;
                if (ent_less(S.rk[mid], S.ri[mid], mk, mi)) lo = mid + 1;
                else hi = mid;
            }
            np = lane + lo;
            if (np < efl) {
                S.nk[np] = mk;
                S.ni[np] = mi;     // unexpanded
            }
        }
        if (ITER) hnsw_sink_append(*sink, lane < cnt_in && np >= efl, mk, mi, lane);
    }
    __syncwarp();
    S.len = min(efl, len + cnt_in);
    uint64_t* tk = S.rk;
    S.rk = S.nk;
    S.nk = tk;
    uint32_t* ti = S.ri;
    S.ri = S.ni;
    S.ni = ti;
}
#endif

// The vacuum's admission of one expansion's fresh neighbours (bkey / bid [0..cnt), list order) into R, one at a time as
// the reference does, because under CountElement (src/hnswutils.c:713-728, 957-974) the result depends on the order:
// elements with no heap TIDs do not count towards ef.  wlen counts the counted additions and is never decremented;
// while wlen < ef everything is added, afterwards an element is added when it is nearer than R's last one, and each
// counted addition past ef removes R's last one, counted or not.  R can therefore hold more than ef entries.  Returns
// false when an addition needs more than wcap entries (R is then incomplete: the caller reruns with a larger one).
__device__ __forceinline__ bool hnsw_admit_counted(HnswWarpState& S, int cnt, int ef, int& wlen, const int32_t* __restrict__ counts,
                                                   int wcap, int lane) {
    const uint64_t mk = lane < cnt ? S.bkey[lane] : 0ull;
    const uint32_t mi = lane < cnt ? S.bid[lane] : 0u;
    const unsigned cm = __ballot_sync(0xffffffffu, lane < cnt && counts[mi & 0x7fffffffu] != 0);
    for (int i = 0; i < cnt; ++i) {
        const uint64_t k = __shfl_sync(0xffffffffu, mk, i);
        const uint32_t id = __shfl_sync(0xffffffffu, mi, i) & 0x7fffffffu;
        const int len = S.len;
        if (!(wlen < ef || ent_less(k, id, S.rk[len - 1], S.ri[len - 1]))) continue;
        const bool counted = (cm >> i) & 1u;
        const bool pop = counted && wlen >= ef;   // (then k is nearer than R's last one: it lands before it)
        const int nlen = pop ? len : len + 1;
        if (nlen > wcap) return false;
        int p = 0;   // entries of R before (k, id)
        for (int j = lane; j < len; j += 32) p += ent_less(S.rk[j], S.ri[j], k, id) ? 1 : 0;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) p += __shfl_xor_sync(0xffffffffu, p, o);
        for (int j0 = nlen - 1; j0 > p; j0 -= 32) {
            const int j = j0 - lane;
            uint64_t kj = 0;
            uint32_t ij = 0;
            if (j > p) {
                kj = S.rk[j - 1];
                ij = S.ri[j - 1];
            }
            __syncwarp();
            if (j > p) {
                S.rk[j] = kj;
                S.ri[j] = ij;
            }
            __syncwarp();
        }
        if (lane == 0) {
            S.rk[p] = k;
            S.ri[p] = id;   // unexpanded
        }
        __syncwarp();
        S.len = nlen;
        if (counted) ++wlen;
    }
    return true;
}

// HnswSearchLayer (src/hnswutils.c:824-987) at layer lc with ef = efl from the entry points already in R
// (S.len of them, sorted).  tab / cap: this layer's visited table (cleared here, InitVisited :671-680).
// ndist (may be null) accumulates the reference's `tuples` counter (:866-873, 905-906).  Returns false when the
// visited table filled beyond three quarters (the caller retries with a larger one).
// ITER: the iterative scan's variant -- everything seen and not kept goes to `sink`; init_visited = false resumes on
// the visited table of the previous call (entry points are neither re-added nor counted, :864-873).
// VAC: the vacuum's variant -- elements with counts[] == 0 do not count towards ef (hnsw_admit_counted); R holds up to
// wcap entries, and *wfull is set (and false returned) when that is not enough.
template <int ELEM, int METRIC, int LPR, bool ITER = false, bool VAC = false>
__device__ __forceinline__ bool hnsw_search_layer(const HnswDev& g, const uint4* sq, int lc, int efl, int lane, HnswWarpState& S,
                                                  uint32_t* tab, uint32_t cap, int64_t* ndist, HnswSink* sink = nullptr,
                                                  bool init_visited = true, const int32_t* counts = nullptr, int wcap = 0,
                                                  bool* wfull = nullptr) {
    const int lm = lc == 0 ? 2 * g.m : g.m;
    const uint32_t mask = cap - 1;
    uint32_t inserted = 0;
    uint32_t* vc = reinterpret_cast<uint32_t*>(S.nk);
    const int vcn = (VB_AB_VCACHE && VB_AB_INPLACE) ? S.vcn : 0;
    for (int i = lane; i < vcn; i += 32) vc[i] = VIS_EMPTY;
    if (!ITER || init_visited) {
        {
            uint4* t4 = reinterpret_cast<uint4*>(tab);   // (cap is a power of two >= 1024, tab 4 KB aligned)
            const uint4 e4 = make_uint4(VIS_EMPTY, VIS_EMPTY, VIS_EMPTY, VIS_EMPTY);
            for (uint32_t i = lane; i < cap / 4; i += 32) __stcg(t4 + i, e4);
        }
        __syncwarp();
        // entry points: visited, unexpanded; they count towards `tuples` (src/hnswutils.c:866-873)
        if (!VAC && S.len > efl) S.len = efl;   // ef shrinks only between an ef_construction layer and ... never; kept for safety
#if VB_AB_VISB
        for (int i0 = 0; i0 < S.len; i0 += 32) {
            const int i = i0 + lane;
            uint32_t id = 0;
            if (i < S.len) {
                id = S.ri[i] & 0x7fffffffu;
                S.ri[i] = id;
            }
            vis_insert_warp(tab, mask, i < S.len, id, lane);
        }
#else
        for (int i = lane; i < S.len; i += 32) {
            S.ri[i] &= 0x7fffffffu;
            vis_insert(tab, mask, S.ri[i]);
        }
#endif
        inserted += (uint32_t)S.len;
        if (ndist) *ndist += S.len;
        __syncwarp();
    } else {
        inserted = sink->inserted;
    }

    bool ok = true;
    int wlen = 0;   // VAC: counted entries added (the entry points are the previous layer's W)
    if constexpr (VAC) {
        for (int i = lane; i < S.len; i += 32) wlen += counts[S.ri[i] & 0x7fffffffu] != 0 ? 1 : 0;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) wlen += __shfl_xor_sync(0xffffffffu, wlen, o);
    }
    uint32_t pre_c = VIS_EMPTY;   // VB_AB_NEXTPF: the element whose list sits in pre_nid
    int pre_nid = -1;
    for (;;) {
        // nearest unexpanded element of R
#if VB_AB_NEXTPF
        int first = -1, second = -1;
        for (int j0 = 0; j0 < S.len && second < 0; j0 += 32) {
            const int j = j0 + lane;
            unsigned um = __ballot_sync(0xffffffffu, j < S.len && !(S.ri[j] & 0x80000000u));
            if (um && first < 0) {
                first = j0 + __ffs(um) - 1;
                um &= um - 1;
            }
            if (um) second = j0 + __ffs(um) - 1;
            if (lc != 0 && first >= 0) break;
        }
        if (first < 0) break;
        const uint32_t next_c = (lc == 0 && second >= 0) ? (S.ri[second] & 0x7fffffffu) : VIS_EMPTY;
#else
        int first = 0x7fffffff;
        for (int i = lane; i < S.len; i += 32)
            if (!(S.ri[i] & 0x80000000u)) {
                first = i;
                break;
            }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) first = min(first, __shfl_xor_sync(0xffffffffu, first, o));
        if (first == 0x7fffffff) break;
#endif
        const uint32_t c = S.ri[first] & 0x7fffffffu;
        __syncwarp();
        if (lane == 0) S.ri[first] = c | 0x80000000u;
        __syncwarp();

        // neighbour list of c at layer lc, in on-disk order (HnswLoadNeighborTids, src/hnswutils.c:761-791)
        const int32_t* nb = nullptr;
        if (lc == 0) nb = g.nbr0 + (size_t)c * lm;
        else if (g.levels[c] >= lc) nb = g.upper + ((size_t)g.upper_off[c] + (lc - 1)) * (size_t)lm;
        if (nb == nullptr) continue;

        for (int off = 0; off < lm; off += 32) {
#if VB_AB_NEXTPF
            int nid;
            if (off == 0 && pre_c == c) nid = pre_nid;           // requested one expansion ago
            else nid = (off + lane < lm) ? nb[off + lane] : -1;
            if (off == 0) {
                pre_c = next_c;
                if (next_c != VIS_EMPTY) pre_nid = lane < lm ? __ldg(g.nbr0 + (size_t)next_c * lm + lane) : -1;
            }
#else
            int nid = (off + lane < lm) ? nb[off + lane] : -1;
#endif
            bool valid = nid >= 0;
            // an invalid TID terminates the list (src/hnswutils.c:809-810)
            unsigned vmask = __ballot_sync(0xffffffffu, valid);
            unsigned inval = ~vmask;
            int first_inval = inval ? __ffs(inval) - 1 : 32;
            valid = valid && lane < first_inval;
            // a small exact cache of recently visited ids in shared memory: a hit is a visited element for certain and
            // saves the probe of the global table (60 % of the neighbours of an expansion are visited already)
            bool known = false;
            uint32_t vslot = 0;
            if (VB_AB_VCACHE && VB_AB_INPLACE && vcn > 0 && valid) {
                vslot = (uint32_t)(((uint64_t)hash_u32((uint32_t)nid ^ 0x9e3779b9u) * (uint32_t)vcn) >> 32);
                known = vc[vslot] == (uint32_t)nid;
            }
            int cnt;
            static_assert(!(VB_AB_SPEC && VB_AB_VISB), "the speculative path probes the linear table");
            if constexpr (VB_AB_SPEC && LPR <= 8) {
                // Narrow rows (< 512 bytes; bit(1024) = 128): every listed neighbour is scored SPECULATIVELY while its visited
                // probe is in flight -- the probe (a random atomic on a table that lives in L2 / DRAM) and the row gather
                // are two dependent round trips otherwise, and the rows of the ~60 % already-visited neighbours cost less
                // than the wait.  The distances of the non-fresh ones are dropped; results, `tuples` and the visited set
                // are exactly those of the ordered version.
                const unsigned vm = __ballot_sync(0xffffffffu, valid);
                const int cnt_all = __popc(vm);
                if (cnt_all == 0) {
                    if (first_inval < 32) break;
                    continue;
                }
                const int pos_all = __popc(vm & ((1u << lane) - 1u));
                uint32_t hs = 0, old = 0;
                if (valid) {
                    S.bid[pos_all] = (uint32_t)nid;
                    hs = hash_u32((uint32_t)nid) & mask;
                    old = atomicCAS(&tab[hs], VIS_EMPTY, (uint32_t)nid);     // issued here, consumed after the scoring
                }
                __syncwarp();
                hnsw_score_batch<ELEM, METRIC, LPR>(g, sq, S.bid, cnt_all, S.bkey, lane);
                __syncwarp();
                bool fresh = false;
                if (valid) {
                    for (;;) {   // the rest of the probe sequence (collisions are rare below 3/4 load)
                        if (old == VIS_EMPTY) {
                            fresh = true;
                            break;
                        }
                        if (old == (uint32_t)nid) break;
                        hs = (hs + 1) & mask;
                        old = atomicCAS(&tab[hs], VIS_EMPTY, (uint32_t)nid);
                    }
                }
                inserted += (uint32_t)__popc(__ballot_sync(0xffffffffu, fresh));
                if (fresh && lc > 0 && g.levels[nid] < lc) fresh = false;   // src/hnswutils.c:949-950
                const unsigned fm = __ballot_sync(0xffffffffu, fresh);
                cnt = __popc(fm);
                if (cnt == 0) {
                    if (first_inval < 32) break;
                    continue;
                }
                if (ndist) *ndist += cnt;
                // keep the fresh entries of (bkey, bid), in list order
                const uint64_t mykey = valid ? S.bkey[pos_all] : 0ull;
                __syncwarp();
                const int pos = __popc(fm & ((1u << lane) - 1u));
                if (fresh) {
                    S.bkey[pos] = mykey;
                    S.bid[pos] = (uint32_t)nid;
                }
                __syncwarp();
            } else {
#if VB_AB_VISB
            bool fresh = vis_insert_warp(tab, mask, valid && !known, (uint32_t)nid, lane);
#if VB_AB_NEXTPF
            // (the list requested above has arrived behind the bucket loads) the visited buckets its elements hash to, and
            // -- narrow rows only: the rows of already visited elements are wasted traffic -- their rows, go to L2 now
            if (off == 0 && pre_c != VIS_EMPTY && pre_nid >= 0) {
                asm volatile("prefetch.global.L2 [%0];" ::"l"(tab + ((size_t)(hash_u32((uint32_t)pre_nid) & (mask >> 3)) << 3)));
                if (g.stride <= 256) {
                    const uint8_t* pr = g.rows + (size_t)pre_nid * g.stride;
                    asm volatile("prefetch.global.L2 [%0];" ::"l"(pr));
                    if (g.stride > 128) asm volatile("prefetch.global.L2 [%0];" ::"l"(pr + 128));
                }
            }
#endif
#else
            bool fresh = valid && !known && vis_insert(tab, mask, (uint32_t)nid);
#endif
            if (VB_AB_VCACHE && VB_AB_INPLACE && vcn > 0 && valid) vc[vslot] = (uint32_t)nid;
            inserted += (uint32_t)__popc(__ballot_sync(0xffffffffu, fresh));
            // elements below this layer are skipped (src/hnswutils.c:949-950)
            if (fresh && lc > 0 && g.levels[nid] < lc) fresh = false;
            unsigned fm = __ballot_sync(0xffffffffu, fresh);
            cnt = __popc(fm);
            if (cnt == 0) {
                if (first_inval < 32) break;
                continue;
            }
            if (ndist) *ndist += cnt;
            const int pos = __popc(fm & ((1u << lane) - 1u));
            if (fresh) S.bid[pos] = (uint32_t)nid;
            __syncwarp();

            hnsw_score_batch<ELEM, METRIC, LPR>(g, sq, S.bid, cnt, S.bkey, lane);
            __syncwarp();
            }
#if VB_AB_NBRPF
            if (lc == 0 && lane < cnt) {
                const bool admit = S.len < efl || ent_less(S.bkey[lane], S.bid[lane], S.rk[efl - 1], S.ri[efl - 1]);
                if (admit) asm volatile("prefetch.global.L2 [%0];" ::"l"(g.nbr0 + (size_t)(S.bid[lane] & 0x7fffffffu) * lm));
            }
#endif

            if constexpr (VAC) {
                if (!hnsw_admit_counted(S, cnt, efl, wlen, counts, wcap, lane)) {
                    *wfull = true;
                    ok = false;
                    break;
                }
            } else {
                hnsw_merge_batch<ITER>(S, cnt, efl, lane, sink);
            }
            if (first_inval < 32) break;
        }
        if constexpr (VAC) {
            if (!ok) break;
        }
        // keep the table at most three quarters full; otherwise report and let the host retry with a larger one
#ifndef VB_AB_VIS
#define VB_AB_VIS 1
#endif
        if (inserted > (VB_AB_VIS ? cap - cap / 4 : cap / 2)) {
            ok = false;
            break;
        }
    }
    if (ITER) sink->inserted = inserted;
    return ok;
}

}  // namespace vb

struct vb_hnsw {
    vb::Hnsw h;
    uint64_t uid = vb::next_owner_uid();   // matched by the element filters made for this image
};
