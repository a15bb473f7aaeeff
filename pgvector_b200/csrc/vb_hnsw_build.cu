// vb_hnsw_build.cu -- HNSW graph construction on the device (CREATE INDEX ... USING hnsw): the in-memory build of
// src/hnswbuild.c:437-480 = per element HnswFindElementNeighbors (src/hnswutils.c:1280-1357: greedy descent,
// HnswSearchLayer with ef_construction on every insertion layer, SelectNeighbors :1065-1165), duplicate folding
// (FindDuplicateInMemory, src/hnswbuild.c:343-364) and HnswUpdateConnection (:1184-1231) on every chosen neighbour.
//
// Formulation.  Elements are inserted in BATCHES, like the reference's parallel build inserts with several workers at
// once (src/hnswbuild.c:412-480: a worker sees the graph as other workers left it, not the elements in flight):
//   K1  hnsw_insert_kernel   one warp per new element: the scan's layer search (vb_hnsw.cuh, `inserting` semantics:
//                            every element counts towards ef) against the graph as of the batch start, then the
//                            neighbour-selection heuristic per layer, written to the element's own neighbour arrays;
//   K1b hnsw_finalize_kernel duplicate check against the chosen layer-0 neighbours, then one (target, layer, source,
//                            distance) record per chosen neighbour;
//       CUB radix sort of the records by (target, layer, source)  -> all updates of one neighbour array are contiguous
//                            and in insertion order;
//   K2  hnsw_update_kernel   one warp per (target, layer): HnswUpdateConnection for each incoming element in turn
//                            (append while there is room, otherwise the heuristic decides which connection goes).
// Batches grow with the graph (at most 1/64 of the elements already inserted, capped) and end at an element that
// becomes the new entry point, so the entry point every search starts from is the reference's.
//
// SelectNeighbors is evaluated EAGERLY: candidates are visited nearest first; an accepted candidate r marks every
// later candidate e with d(e, r) <= d(e, q) as pruned at once (one row image in shared memory, the surviving
// candidates scored against it in one pass).  That is the same predicate as CheckElementCloser (:1040-1060) applied
// in the same order, so the selected set, the order of the pruned candidates kept to fill up, and the connection
// HnswUpdateConnection drops (the farthest pruned candidate, or the farthest one when none is pruned) are the
// reference's.  The reference's `closer` cache (:1090-1122) only skips work; it is not reproduced.
//
// Roofline: HBM / L2 latency-bound row gathers, like the scan (n_dist * row bytes per element, ~3x the scan's because
// of the heuristic and the neighbour updates).  Parity: the graph depends on PRNG level draws and on insertion
// concurrency, which no reference test pins; parity is by the reference's recall floors (test/t/012, 020) on
// GPU-built graphs and by exact search equality of GPU and oracle on the SAME exported graph.
#include "vb_hnsw.cuh"

#include <cub/cub.cuh>

#include <algorithm>
#include <cmath>
#include <vector>

namespace vb {

struct BuildDev {
    HnswDev g;
    int32_t* nbr0_w;      // same arrays as g.nbr0 / g.upper, writable
    int32_t* upper_w;
    float* nd0;           // [n][2m] distance stored with each neighbour
    float* upper_d;       // [slots][m]
    int32_t* dup_of;      // [n] element this row was folded into, or -1
    int32_t* n_heaptids;  // [n] heap tids carried by the element (HNSW_HEAPTIDS = 10 at most, src/hnsw.h:69)
    int efc;
    int b0, B;            // this batch inserts elements [b0, b0 + B)
    int qvec;             // 16-byte vectors of a row image
    uint64_t* edge_key;   // target << 26 | layer << 20 | (source - b0)
    float* edge_val;
    int* n_edges;
    int* overflow;
};

// vb_hnsw_insert's change records: one (key, neighbour) per neighbour-array slot written, key = element << 14 | layer << 8
// | slot.  (A parameter of its own, so the build kernels' parameter layout stays as it was.)
struct InsertRec {
    uint64_t* key;
    int32_t* val;
    int* n;
};

// vb_hnsw_vacuum's side of K1 / K2 (a parameter of its own, so the build and insert kernels keep their parameter layout):
// the batch repairs the elements list[0..B); K1 writes their new lists to the staging area, which is published only after
// every search of the batch has finished.
struct VacDev {
    const int32_t* list;     // [B] elements repaired by this batch, ascending
    int32_t* stage0;         // [B][2m] new layer-0 lists, by list position
    int32_t* stage_up;       // [slots][m] new upper lists, at the element's own upper slots
    const int32_t* counts;   // [n] heap TID counts (0 = being deleted or deleted)
    uint64_t* wk;            // per-warp W in global memory ([warps][2][wcap] keys, ids, pruned indices and flags), or null:
    uint32_t* wi;            // W in shared memory, wcap entries
    uint16_t* wd;
    uint8_t* dead;
    int wcap;
    int* wfull;              // set when a repair's W needs more than wcap entries
};

constexpr int HB_CAND = 256;     // candidates of one HnswUpdateConnection: lm + 1 <= 201, padded to a power of two

__device__ __forceinline__ float key64_to_float(uint64_t k) { return (float)key64_to_double(k); }

// shared memory of one warp of hnsw_insert_kernel (bytes, 16-aligned)
__host__ __device__ inline size_t hb_insert_smem(int qvec, int efc, int lm0) {
    size_t b = (size_t)qvec * 16 * 2;          // image of the new element, image of an accepted candidate
    b += (size_t)efc * 2 * 8 + 32 * 8;         // keys A, keys B, batch keys
    b += (size_t)efc * 2 * 4 + 32 * 4 + 32 * 4; // ids A, ids B, batch ids, batch -> candidate index
    b += (size_t)lm0 * 4;                      // selected candidate indices
    b += (size_t)efc * 2;                      // pruned candidate indices (uint16)
    b += (size_t)efc;                          // pruned flags
    return (b + 15) & ~(size_t)15;
}
__host__ __device__ inline size_t hb_update_smem(int qvec) {
    size_t b = (size_t)qvec * 16;              // image of an accepted candidate
    b += (size_t)HB_CAND * 8 + 32 * 8;         // candidate keys, batch keys
    b += 32 * 4 + 32 * 4;                      // batch ids, batch -> candidate index
    b += HB_CAND;                              // pruned flags
    return (b + 15) & ~(size_t)15;
}

// dynamic shared memory one CTA of the build kernels may take: the one limit both the launches and the choice of where
// hnsw_insert_kernel keeps R are checked against
constexpr size_t HB_SMEM_MAX = 200 * 1024;

// the largest capacity of R in [lo, hi] whose hnsw_insert_kernel CTA fits in shared memory, or 0 when none does: R then lives
// in global memory (VacDev::wk, capacity hi) and only the row images stay in shared memory
static int hb_insert_shared_cap(int qvec, int lm0, int lo, int hi) {
    for (int cap = hi; cap >= lo; --cap)
        if (hb_insert_smem(qvec, cap, lm0) * HN_WARPS <= HB_SMEM_MAX) return cap;
    return 0;
}

// candidates cand[from..n) that are still unpruned are scored against the image `img` (the row of the candidate
// just accepted); those with d(e, r) <= d(e, q) are pruned (CheckElementCloser, src/hnswutils.c:1040-1060)
template <int ELEM, int METRIC, int LPR, typename IdOf, typename DistOf>
__device__ __forceinline__ void prune_against(const HnswDev& g, const uint4* img, int from, int n, uint8_t* dead, uint32_t* bid,
                                              int32_t* bj, uint64_t* bkey, int lane, IdOf id_of, DistOf dist_of) {
    for (int base = from; base < n; base += 32) {
        const int j = base + lane;
        const bool alive = j < n && !dead[j];
        const unsigned am = __ballot_sync(0xffffffffu, alive);
        const int cnt = __popc(am);
        if (cnt == 0) continue;
        const int pos = __popc(am & ((1u << lane) - 1u));
        if (alive) {
            bid[pos] = id_of(j);
            bj[pos] = j;
        }
        __syncwarp();
        hnsw_score_batch<ELEM, METRIC, LPR>(g, img, bid, cnt, bkey, lane);
        __syncwarp();
        if (lane < cnt) {
            const int jj = bj[lane];
            if (key64_to_float(bkey[lane]) <= dist_of(jj)) dead[jj] = 1;
        }
        __syncwarp();
    }
}

// K1: one warp = one new element.  INS (vb_hnsw_insert): candidates whose element is being deleted (heap TID count 0)
// help the search but are removed before SelectNeighbors (RemoveElements, src/hnswutils.c:1237-1259, 1343-1344).
// VAC (vb_hnsw_vacuum): one warp = one repaired element, list[w] = RepairGraphElement (src/hnswvacuum.c:225-274) =
// HnswFindElementNeighbors with existing = true: elements being deleted do not count towards ef (R holds v.wcap
// entries), ef_construction + 1 (b.efc already is), the element itself is removed too, and the whole new tuple goes to
// the staging area (the layers above the entry point's level are left empty, as the reference's are).
// R and the candidate arrays live in shared memory, or in global memory when v.wk is set (rows too wide for R of this
// capacity to fit beside the two row images, or a repair that outgrew the shared R).
template <int ELEM, int METRIC, int LPR, bool INS = false, bool VAC = false>
__global__ void __launch_bounds__(HN_WARPS * 32) hnsw_insert_kernel(BuildDev b, uint32_t* __restrict__ vis_all, uint32_t vis_cap,
                                                                    uint32_t vis_upper, VacDev v) {
    extern __shared__ uint4 smem[];
    const HnswDev& g = b.g;
    const int warp = threadIdx.x / 32, lane = threadIdx.x % 32;
    const int efc = b.efc, lm0 = 2 * g.m;
    const int wc = VAC ? v.wcap : efc;   // capacity of R and of the candidate arrays
    uint8_t* base = reinterpret_cast<uint8_t*>(smem) + (size_t)warp * hb_insert_smem(b.qvec, v.wk ? 0 : wc, lm0);
    uint4* sq = reinterpret_cast<uint4*>(base);
    uint4* img = sq + b.qvec;
    uint64_t* keyA = reinterpret_cast<uint64_t*>(img + b.qvec);
    uint64_t* keyB = keyA + (v.wk ? 0 : wc);
    uint64_t* bkey = keyB + (v.wk ? 0 : wc);
    uint32_t* idA = reinterpret_cast<uint32_t*>(bkey + 32);
    uint32_t* idB = idA + (v.wk ? 0 : wc);
    uint32_t* bid = idB + (v.wk ? 0 : wc);
    int32_t* bj = reinterpret_cast<int32_t*>(bid + 32);
    int32_t* sel = bj + 32;
    uint16_t* wd = reinterpret_cast<uint16_t*>(sel + lm0);
    uint8_t* dead = reinterpret_cast<uint8_t*>(wd + (v.wk ? 0 : wc));

    const int gwarp = blockIdx.x * HN_WARPS + warp;
    const int nwarps = gridDim.x * HN_WARPS;
    uint32_t* vis = vis_all + (size_t)gwarp * vis_cap;
    if (v.wk) {
        keyA = v.wk + (size_t)gwarp * 2 * wc;
        keyB = keyA + wc;
        idA = v.wi + (size_t)gwarp * 2 * wc;
        idB = idA + wc;
        wd = v.wd + (size_t)gwarp * wc;
        dead = v.dead + (size_t)gwarp * wc;
    }

    for (int w = gwarp; w < b.B; w += nwarps) {
        const int e = VAC ? v.list[w] : b.b0 + w;
        load_row_image<ELEM, METRIC>(g.rows + (size_t)e * g.stride, g.V, sq, lane);
        __syncwarp();
        const int level = g.levels[e];
        if constexpr (VAC) {
            // the whole tuple is rewritten: every layer starts empty
            for (int i = lane; i < lm0; i += 32) v.stage0[(size_t)w * lm0 + i] = -1;
            for (int lc = 1; lc <= level; ++lc)
                for (int i = lane; i < g.m; i += 32) v.stage_up[((size_t)g.upper_off[e] + (lc - 1)) * g.m + i] = -1;
            __syncwarp();
            if (g.entry < 0) continue;   // no entry point: no neighbours (src/hnswutils.c:1297-1299)
        }

        HnswWarpState S;
        S.rk = keyA;
        S.ri = idA;
        S.nk = keyB;
        S.ni = idB;
        S.vcn = 0;
        S.bkey = bkey;
        S.bid = bid;
        // entry point (HnswEntryCandidate, src/hnswutils.c:609-621)
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
        bool failed = false, wfull = false;
        // 1st phase: greedy search to the insert level (src/hnswutils.c:1308-1313)
        int lc = g.entry_level;
        for (; lc > level && !failed; --lc)
            failed = !hnsw_search_layer<ELEM, METRIC, LPR, false, VAC>(g, sq, lc, 1, lane, S, vis, vis_upper, nullptr, nullptr, true,
                                                                       v.counts, wc, &wfull);
        // 2nd phase (:1322-1354): level = min(level, entryLevel)
        for (; lc >= 0 && !failed; --lc) {
            failed = !hnsw_search_layer<ELEM, METRIC, LPR, false, VAC>(g, sq, lc, efc, lane, S, vis + vis_upper, vis_cap - vis_upper, nullptr,
                                                                       nullptr, true, v.counts, wc, &wfull);
            if (failed) break;
            const int lm = lc == 0 ? lm0 : g.m;
            int32_t* out_ids = VAC ? (lc == 0 ? v.stage0 + (size_t)w * lm : v.stage_up + ((size_t)g.upper_off[e] + (lc - 1)) * (size_t)lm)
                                   : lc == 0 ? b.nbr0_w + (size_t)e * lm : b.upper_w + ((size_t)g.upper_off[e] + (lc - 1)) * (size_t)lm;
            float* out_d = lc == 0 ? b.nd0 + (size_t)e * lm : b.upper_d + ((size_t)g.upper_off[e] + (lc - 1)) * (size_t)lm;
            int len = S.len;
            const uint64_t* wk = S.rk;     // W, nearest first; stays intact: it is the next layer's entry list (ep = w)
            const uint32_t* wi = S.ri;
            if constexpr (INS) {
                // the kept candidates go to the second key / id buffers, which the in-place merge leaves unused
                int kept = 0;
                for (int i0 = 0; i0 < len; i0 += 32) {
                    const int i = i0 + lane;
                    const uint32_t id = i < len ? S.ri[i] & 0x7fffffffu : 0u;
                    const bool keep = i < len && b.n_heaptids[id] != 0 && (!VAC || id != (uint32_t)e);
                    const unsigned km = __ballot_sync(0xffffffffu, keep);
                    if (keep) {
                        const int p = kept + __popc(km & ((1u << lane) - 1u));
                        S.nk[p] = S.rk[i];
                        S.ni[p] = S.ri[i];
                    }
                    kept += __popc(km);
                }
                __syncwarp();
                wk = S.nk;
                wi = S.ni;
                len = kept;
            }
            if (len <= lm) {
                // SelectNeighbors returns the list as it is (:1077-1078): W drained from the max-heap = farthest first
                for (int i = lane; i < lm; i += 32) {
                    const int j = len - 1 - i;
                    out_ids[i] = i < len ? (int32_t)(wi[j] & 0x7fffffffu) : -1;
                    out_d[i] = i < len ? key64_to_float(wk[j]) : 0.f;
                }
            } else {
                for (int i = lane; i < len; i += 32) dead[i] = 0;
                __syncwarp();
                int nR = 0, nWd = 0;
                for (int i = 0; i < len; ++i) {
                    if (dead[i]) {   // shared memory flag: the same value for every lane
                        if (lane == 0) wd[nWd] = (uint16_t)i;
                        ++nWd;
                        continue;
                    }
                    if (lane == 0) sel[nR] = i;
                    ++nR;
                    if (nR == lm || i + 1 >= len) break;
                    load_row_image<ELEM, METRIC>(g.rows + (size_t)(wi[i] & 0x7fffffffu) * g.stride, g.V, img, lane);
                    __syncwarp();
                    prune_against<ELEM, METRIC, LPR>(
                        g, img, i + 1, len, dead, bid, bj, bkey, lane, [&](int j) { return wi[j] & 0x7fffffffu; },
                        [&](int j) { return key64_to_float(wk[j]); });
                }
                __syncwarp();
                // keep pruned connections (:1151-1153)
                for (int t = 0; t < nWd && nR < lm; ++t, ++nR)
                    if (lane == 0) sel[nR] = wd[t];
                __syncwarp();
                for (int i = lane; i < lm; i += 32) {
                    const int j = i < nR ? sel[i] : 0;
                    out_ids[i] = i < nR ? (int32_t)(wi[j] & 0x7fffffffu) : -1;
                    out_d[i] = i < nR ? key64_to_float(wk[j]) : 0.f;
                }
            }
            __syncwarp();
        }
        if (failed && lane == 0) atomicExch(VAC && wfull ? v.wfull : b.overflow, 1);
        __syncwarp();
    }
}

// K1b: duplicates (FindDuplicateInMemory, src/hnswbuild.c:343-364) and the update records of every chosen neighbour.
// DISK (vb_hnsw_insert): FindDuplicateOnDisk / AddDuplicateOnDisk (src/hnswinsert.c:586-663): the row joins the first
// equal neighbour with 1..9 heap TIDs; one being deleted (0) or full (10) is skipped.
template <bool DISK = false>
__global__ void __launch_bounds__(128) hnsw_finalize_kernel(BuildDev b) {
    if (*b.overflow) return;   // K1 is repeated with larger visited tables: no side effect may have happened yet
    const HnswDev& g = b.g;
    const int lane = threadIdx.x % 32;
    const int gwarp = (int)((blockIdx.x * (int64_t)blockDim.x + threadIdx.x) / 32);
    const int nwarps = (int)((gridDim.x * (int64_t)blockDim.x) / 32);
    const int lm0 = 2 * g.m;
    for (int w = gwarp; w < b.B; w += nwarps) {
        const int e = b.b0 + w;
        const int level = g.levels[e];
        const int top = min(level, g.entry_level);
        int32_t* ids0 = b.nbr0_w + (size_t)e * lm0;
        const uint4* re = reinterpret_cast<const uint4*>(g.rows + (size_t)e * g.stride);
        bool dup = false;
        for (int i = 0; i < lm0; ++i) {
            const int t = ids0[i];
            if (t < 0) break;
            const uint4* rt = reinterpret_cast<const uint4*>(g.rows + (size_t)t * g.stride);
            bool eq = true;
            for (int v = lane; v < g.V; v += 32) {
                const uint4 x = __ldg(re + v), y = __ldg(rt + v);
                eq = eq && x.x == y.x && x.y == y.y && x.z == y.z && x.w == y.w;
            }
            if (!__all_sync(0xffffffffu, eq)) break;   // "exit early since ordered by distance"
            if constexpr (DISK) {
                int c = 0;
                if (lane == 0) {
                    c = b.n_heaptids[t];
                    while (c >= 1 && c < 10) {
                        const int o = atomicCAS(&b.n_heaptids[t], c, c + 1);
                        if (o == c) break;
                        c = o;
                    }
                }
                c = __shfl_sync(0xffffffffu, c, 0);
                if (c >= 1 && c < 10) {
                    dup = true;
                    if (lane == 0) b.dup_of[e] = t;
                    break;
                }
                continue;
            }
            int old = 0;
            if (lane == 0) old = atomicAdd(&b.n_heaptids[t], 1);
            old = __shfl_sync(0xffffffffu, old, 0);
            if (old < 10) {
                dup = true;
                if (lane == 0) b.dup_of[e] = t;
                break;
            }
            if (lane == 0) atomicSub(&b.n_heaptids[t], 1);
        }
        if (dup) {
            // the row rides on element t: it never becomes an element (no connections in either direction)
            for (int i = lane; i < lm0; i += 32) ids0[i] = -1;
            for (int lc = 1; lc <= top; ++lc) {
                int32_t* ids = b.upper_w + ((size_t)g.upper_off[e] + (lc - 1)) * (size_t)g.m;
                for (int i = lane; i < g.m; i += 32) ids[i] = -1;
            }
            if (lane == 0) b.n_heaptids[e] = 0;
            continue;
        }
        // UpdateNeighborsInMemory (src/hnswbuild.c:381-410): one record per (neighbour, layer)
        for (int lc = top; lc >= 0; --lc) {
            const int lm = lc == 0 ? lm0 : g.m;
            const int32_t* ids = lc == 0 ? ids0 : b.upper_w + ((size_t)g.upper_off[e] + (lc - 1)) * (size_t)lm;
            const float* ds = lc == 0 ? b.nd0 + (size_t)e * lm : b.upper_d + ((size_t)g.upper_off[e] + (lc - 1)) * (size_t)lm;
            for (int off = 0; off < lm; off += 32) {
                const int t = off + lane < lm ? ids[off + lane] : -1;
                const unsigned vm = __ballot_sync(0xffffffffu, t >= 0);
                const int cnt = __popc(vm);
                if (cnt == 0) break;
                int slot = 0;
                if (lane == 0) slot = atomicAdd(b.n_edges, cnt);
                slot = __shfl_sync(0xffffffffu, slot, 0);
                if (t >= 0) {
                    const int p = slot + __popc(vm & ((1u << lane) - 1u));
                    b.edge_key[p] = ((uint64_t)(uint32_t)t << 26) | ((uint64_t)lc << 20) | (uint64_t)w;
                    b.edge_val[p] = ds[off + lane];
                }
            }
        }
    }
}

// K2: one warp per (target, layer) run of the sorted records = HnswUpdateConnection (src/hnswutils.c:1184-1231) for each
// incoming element in insertion order
template <int ELEM, int METRIC, int LPR>
__global__ void __launch_bounds__(HN_WARPS * 32) hnsw_update_kernel(BuildDev b, const uint64_t* __restrict__ keys,
                                                                    const float* __restrict__ vals, int n_edges) {
    extern __shared__ uint4 smem[];
    const HnswDev& g = b.g;
    const int warp = threadIdx.x / 32, lane = threadIdx.x % 32;
    uint8_t* base = reinterpret_cast<uint8_t*>(smem) + (size_t)warp * hb_update_smem(b.qvec);
    uint4* img = reinterpret_cast<uint4*>(base);
    uint64_t* ck = reinterpret_cast<uint64_t*>(img + b.qvec);
    uint64_t* bkey = ck + HB_CAND;
    uint32_t* bid = reinterpret_cast<uint32_t*>(bkey + 32);
    int32_t* bj = reinterpret_cast<int32_t*>(bid + 32);
    uint8_t* dead = reinterpret_cast<uint8_t*>(bj + 32);

    const int64_t gwarp = blockIdx.x * (int64_t)HN_WARPS + warp;
    const int64_t nwarps = gridDim.x * (int64_t)HN_WARPS;
    for (int64_t i = gwarp; i < n_edges; i += nwarps) {
        const uint64_t head = keys[i] >> 20;
        if (i > 0 && (keys[i - 1] >> 20) == head) continue;   // not the first record of its (target, layer) run
        const int t = (int)(head >> 6), lc = (int)(head & 63);
        const int lm = lc == 0 ? 2 * g.m : g.m;
        int32_t* ids = lc == 0 ? b.nbr0_w + (size_t)t * lm : b.upper_w + ((size_t)g.upper_off[t] + (lc - 1)) * (size_t)lm;
        float* ds = lc == 0 ? b.nd0 + (size_t)t * lm : b.upper_d + ((size_t)g.upper_off[t] + (lc - 1)) * (size_t)lm;
        for (int64_t p = i; p < n_edges && (keys[p] >> 20) == head; ++p) {
            const int src = b.b0 + (int)(keys[p] & 0xFFFFFu);
            const float d = vals[p];
            // current length = first invalid entry
            int count = lm;
            for (int off = 0; off < lm; off += 32) {
                const int nid = off + lane < lm ? ids[off + lane] : -1;
                const unsigned inval = ~__ballot_sync(0xffffffffu, nid >= 0);
                if (inval) {
                    count = min(lm, off + __ffs(inval) - 1);
                    break;
                }
            }
            if (count < lm) {   // room left: append (:1192-1199)
                if (lane == 0) {
                    ids[count] = src;
                    ds[count] = d;
                }
                __syncwarp();
                continue;
            }
            // shrink connections (:1201-1230): candidates = the lm connections + the new element, nearest first
            const int n = lm + 1;
            int P = 2;
            while (P < n) P <<= 1;
            for (int j = lane; j < P; j += 32) {
                uint64_t key = ~0ull;
                if (j < lm) key = ((uint64_t)orderable_key(ds[j]) << 32) | (uint32_t)ids[j];
                else if (j == lm) key = ((uint64_t)orderable_key(d) << 32) | (uint32_t)src;
                ck[j] = key;
                dead[j] = 0;
            }
            __syncwarp();
            for (int size = 2; size <= P; size <<= 1)
                for (int st = size >> 1; st > 0; st >>= 1) {
                    for (int a = lane; a < P; a += 32) {
                        const int c = a ^ st;
                        if (c > a) {
                            const uint64_t x = ck[a], y = ck[c];
                            const bool up = (a & size) == 0;
                            if ((x > y) == up) {
                                ck[a] = y;
                                ck[c] = x;
                            }
                        }
                    }
                    __syncwarp();
                }
            int nAcc = 0;
            for (int c = 0; c < n; ++c) {
                if (dead[c]) continue;
                ++nAcc;
                if (nAcc == lm || c == n - 1) break;
                load_row_image<ELEM, METRIC>(g.rows + (size_t)(uint32_t)ck[c] * g.stride, g.V, img, lane);
                __syncwarp();
                prune_against<ELEM, METRIC, LPR>(
                    g, img, c + 1, n, dead, bid, bj, bkey, lane, [&](int j) { return (uint32_t)ck[j]; },
                    [&](int j) { return key_to_float((uint32_t)(ck[j] >> 32)); });
                if (dead[n - 1]) break;   // the farthest candidate is pruned: it is the one that goes
            }
            __syncwarp();
            // the connection that goes: the farthest pruned candidate, or the farthest candidate when none is pruned
            int drop = -1;
            for (int j0 = ((n - 1) / 32) * 32; j0 >= 0 && drop < 0; j0 -= 32) {
                const int j = j0 + lane;
                const unsigned dm = __ballot_sync(0xffffffffu, j < n && dead[j]);
                if (dm) drop = j0 + 31 - __clz(dm);
            }
            if (drop < 0) drop = n - 1;
            const uint32_t drop_id = (uint32_t)ck[drop];
            if (drop_id != (uint32_t)src) {
                for (int j = lane; j < lm; j += 32)
                    if ((uint32_t)ids[j] == drop_id) {
                        ids[j] = src;
                        ds[j] = d;
                    }
            }
            __syncwarp();
        }
    }
}

// shared memory of one warp of hnsw_update_disk_kernel (bytes, 16-aligned)
__host__ __device__ inline size_t hb_update_disk_smem(int qvec) {
    size_t b = hb_update_smem(qvec);
    b += (size_t)HB_CAND * 4 * 2;              // ids of the list as scored, their distances to the target
    return (b + 15) & ~(size_t)15;
}

__device__ __forceinline__ void hb_record(const InsertRec& r, int t, int lc, int slot, int32_t v) {
    const int p = atomicAdd(r.n, 1);
    r.key[p] = ((uint64_t)(uint32_t)t << 14) | ((uint64_t)lc << 8) | (uint64_t)slot;
    r.val[p] = v;
}

// K2 of vb_hnsw_insert: one warp per (target, layer) run = UpdateNeighborOnDisk (src/hnswinsert.c:409-448, 506-518)
// for each incoming element in insertion order.  The stored distances are not used: a full list has its distances
// recomputed from the target's own row (LoadElementsForInsert, :383-403), with the scan arithmetic, once per run and
// kept in shared memory for the run's later updates.  Then:
//   room left                     -> the first free slot;
//   a neighbour being deleted     -> the first such neighbour is replaced;
//   otherwise                     -> HnswUpdateConnection (src/hnswutils.c:1184-1231): SelectNeighbors over the lm
//                                    connections and the new element, nearest first; the pruned connection is replaced
//                                    in its slot, nothing changes when the new element is the one pruned.
// Every slot written is recorded (rec_key / rec_val); later records of a slot supersede earlier ones.
// VAC (vb_hnsw_vacuum): the source is the repaired element v.list[...], and a target that already links to it is left as
// it is (ConnectionExists, src/hnswinsert.c:453-468, 503-505); the records come from the diff of the whole call instead.
template <int ELEM, int METRIC, int LPR, bool VAC = false>
__global__ void __launch_bounds__(HN_WARPS * 32) hnsw_update_disk_kernel(BuildDev b, const uint64_t* __restrict__ keys,
                                                                         const float* __restrict__ vals, int n_edges, InsertRec r,
                                                                         VacDev v) {
    extern __shared__ uint4 smem[];
    const HnswDev& g = b.g;
    const int warp = threadIdx.x / 32, lane = threadIdx.x % 32;
    uint8_t* base = reinterpret_cast<uint8_t*>(smem) + (size_t)warp * hb_update_disk_smem(b.qvec);
    uint4* img = reinterpret_cast<uint4*>(base);
    uint64_t* ck = reinterpret_cast<uint64_t*>(img + b.qvec);
    uint64_t* bkey = ck + HB_CAND;
    uint32_t* bid = reinterpret_cast<uint32_t*>(bkey + 32);
    int32_t* bj = reinterpret_cast<int32_t*>(bid + 32);
    uint32_t* cid = reinterpret_cast<uint32_t*>(bj + 32);
    float* cd = reinterpret_cast<float*>(cid + HB_CAND);
    uint8_t* dead = reinterpret_cast<uint8_t*>(cd + HB_CAND);

    const int64_t gwarp = blockIdx.x * (int64_t)HN_WARPS + warp;
    const int64_t nwarps = gridDim.x * (int64_t)HN_WARPS;
    for (int64_t i = gwarp; i < n_edges; i += nwarps) {
        const uint64_t head = keys[i] >> 20;
        if (i > 0 && (keys[i - 1] >> 20) == head) continue;   // not the first record of its (target, layer) run
        const int t = (int)(head >> 6), lc = (int)(head & 63);
        const int lm = lc == 0 ? 2 * g.m : g.m;
        int32_t* ids = lc == 0 ? b.nbr0_w + (size_t)t * lm : b.upper_w + ((size_t)g.upper_off[t] + (lc - 1)) * (size_t)lm;
        bool have_d = false;
        for (int64_t p = i; p < n_edges && (keys[p] >> 20) == head; ++p) {
            const int src = VAC ? v.list[keys[p] & 0xFFFFFu] : b.b0 + (int)(keys[p] & 0xFFFFFu);
            const float d = vals[p];
            // current length = first invalid entry
            int count = lm;
            bool exists = false;
            for (int off = 0; off < lm; off += 32) {
                const int nid = off + lane < lm ? ids[off + lane] : -1;
                const unsigned inval = ~__ballot_sync(0xffffffffu, nid >= 0);
                if constexpr (VAC) {
                    const int valid = inval ? __ffs(inval) - 1 : 32;
                    exists = exists || __any_sync(0xffffffffu, lane < valid && nid == src);
                }
                if (inval) {
                    count = min(lm, off + __ffs(inval) - 1);
                    break;
                }
            }
            int slot = -1;
            if (VAC && exists) {
                // ConnectionExists: the target keeps its list
            } else if (count < lm) {
                slot = count;
            } else {
                if (!have_d) {
                    load_row_image<ELEM, METRIC>(g.rows + (size_t)t * g.stride, g.V, img, lane);
                    for (int j = lane; j < lm; j += 32) cid[j] = (uint32_t)ids[j];
                    __syncwarp();
                    hnsw_score_batch<ELEM, METRIC, LPR>(g, img, cid, lm, ck, lane);
                    __syncwarp();
                    for (int j = lane; j < lm; j += 32) cd[j] = key64_to_float(ck[j]);
                    __syncwarp();
                    have_d = true;
                }
                for (int off = 0; off < lm && slot < 0; off += 32) {
                    const int j = off + lane;
                    const unsigned zm = __ballot_sync(0xffffffffu, j < lm && b.n_heaptids[ids[j]] == 0);
                    if (zm) slot = off + __ffs(zm) - 1;
                }
                if (slot < 0) {
                    // candidates = the lm connections + the new element, nearest first
                    const int n = lm + 1;
                    int P = 2;
                    while (P < n) P <<= 1;
                    for (int j = lane; j < P; j += 32) {
                        uint64_t key = ~0ull;
                        if (j < lm) key = ((uint64_t)orderable_key(cd[j]) << 32) | (uint32_t)ids[j];
                        else if (j == lm) key = ((uint64_t)orderable_key(d) << 32) | (uint32_t)src;
                        ck[j] = key;
                        dead[j] = 0;
                    }
                    __syncwarp();
                    for (int size = 2; size <= P; size <<= 1)
                        for (int st = size >> 1; st > 0; st >>= 1) {
                            for (int a = lane; a < P; a += 32) {
                                const int c = a ^ st;
                                if (c > a) {
                                    const uint64_t x = ck[a], y = ck[c];
                                    const bool up = (a & size) == 0;
                                    if ((x > y) == up) {
                                        ck[a] = y;
                                        ck[c] = x;
                                    }
                                }
                            }
                            __syncwarp();
                        }
                    int nAcc = 0;
                    for (int c = 0; c < n; ++c) {
                        if (dead[c]) continue;
                        ++nAcc;
                        if (nAcc == lm || c == n - 1) break;
                        load_row_image<ELEM, METRIC>(g.rows + (size_t)(uint32_t)ck[c] * g.stride, g.V, img, lane);
                        __syncwarp();
                        prune_against<ELEM, METRIC, LPR>(
                            g, img, c + 1, n, dead, bid, bj, bkey, lane, [&](int j) { return (uint32_t)ck[j]; },
                            [&](int j) { return key_to_float((uint32_t)(ck[j] >> 32)); });
                        if (dead[n - 1]) break;   // the farthest candidate is pruned: it is the one that goes
                    }
                    __syncwarp();
                    int drop = -1;
                    for (int j0 = ((n - 1) / 32) * 32; j0 >= 0 && drop < 0; j0 -= 32) {
                        const int j = j0 + lane;
                        const unsigned dm = __ballot_sync(0xffffffffu, j < n && dead[j]);
                        if (dm) drop = j0 + 31 - __clz(dm);
                    }
                    if (drop < 0) drop = n - 1;
                    const uint32_t drop_id = (uint32_t)ck[drop];
                    if (drop_id != (uint32_t)src) {
                        for (int off = 0; off < lm && slot < 0; off += 32) {
                            const int j = off + lane;
                            const unsigned hm = __ballot_sync(0xffffffffu, j < lm && (uint32_t)ids[j] == drop_id);
                            if (hm) slot = off + __ffs(hm) - 1;
                        }
                    }
                    __syncwarp();
                }
            }
            if (slot >= 0 && lane == 0) {
                ids[slot] = src;
                if (have_d) cd[slot] = d;
                if (!VAC) hb_record(r, t, lc, slot, src);
            }
            __syncwarp();
        }
    }
}

// the change records of the new elements: every filled slot of their own lists, as they stand after the last batch
__global__ void __launch_bounds__(128) hnsw_new_records_kernel(BuildDev b, InsertRec r, int64_t e0, int64_t ne) {
    const HnswDev& g = b.g;
    const int lane = threadIdx.x % 32;
    const int64_t gwarp = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) / 32;
    const int64_t nwarps = (gridDim.x * (int64_t)blockDim.x) / 32;
    for (int64_t w = gwarp; w < ne; w += nwarps) {
        const int e = (int)(e0 + w);
        if (b.dup_of[e] >= 0) continue;
        for (int lc = 0; lc <= g.levels[e]; ++lc) {
            const int lm = lc == 0 ? 2 * g.m : g.m;
            const int32_t* ids = lc == 0 ? b.nbr0_w + (size_t)e * lm : b.upper_w + ((size_t)g.upper_off[e] + (lc - 1)) * (size_t)lm;
            for (int off = 0; off < lm; off += 32) {
                const int v = off + lane < lm ? ids[off + lane] : -1;
                const unsigned vm = __ballot_sync(0xffffffffu, v >= 0);
                if (vm == 0) break;
                int p = 0;
                if (lane == 0) p = atomicAdd(r.n, __popc(vm));
                p = __shfl_sync(0xffffffffu, p, 0) + __popc(vm & ((1u << lane) - 1u));
                if (v >= 0) {
                    r.key[p] = ((uint64_t)(uint32_t)e << 14) | ((uint64_t)lc << 8) | (uint64_t)(off + lane);
                    r.val[p] = v;
                }
            }
        }
    }
}

// after the stable sort by key: a record is kept when it is the last of its slot (the slot's final value)
__global__ void hnsw_last_of_key_kernel(const uint64_t* __restrict__ keys, int64_t n, uint8_t* __restrict__ keep) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i < n) keep[i] = (i + 1 == n || keys[i + 1] != keys[i]) ? 1 : 0;
}

__global__ void fill_i32_kernel(int32_t* p, int64_t n, int32_t v) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i < n) p[i] = v;
}

// ----------------------------------------------------------------------------- host side

struct BuildLaunch {
    int (*insert)(const BuildDev&, const VacDev&, uint32_t*, uint32_t, uint32_t, int, size_t, int*);
    int (*update)(const BuildDev&, const VacDev&, const uint64_t*, const float*, int, const InsertRec&, int, size_t, int*);
};

// the three modes of the batch loop: the build, vb_hnsw_insert (RemoveElements in K1, UpdateNeighborOnDisk in K2) and
// vb_hnsw_vacuum (RepairGraphElement in K1, UpdateNeighborOnDisk with ConnectionExists in K2)
enum { HB_BUILD = 0, HB_INSERT = 1, HB_VACUUM = 2 };

template <int ELEM, int METRIC, int LPR, int MODE>
static int launch_insert(const BuildDev& b, const VacDev& v, uint32_t* vis, uint32_t vis_cap, uint32_t vis_upper, int grid, size_t smem,
                         int* occ) {
    auto kern = hnsw_insert_kernel<ELEM, METRIC, LPR, MODE != HB_BUILD, MODE == HB_VACUUM>;
    VB_REQUIRE(smem <= HB_SMEM_MAX, "hnsw: %zu bytes of shared memory per CTA do not fit", smem);
    if (smem > 48 * 1024) VB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    if (occ) {
        VB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(occ, kern, HN_WARPS * 32, smem));
        return VB_OK;
    }
    kern<<<grid, HN_WARPS * 32, smem, ctx().stream>>>(b, vis, vis_cap, vis_upper, v);
    VB_CUDA(cudaGetLastError());
    count_launch();
    return VB_OK;
}
template <int ELEM, int METRIC, int LPR, int MODE>
static int launch_update(const BuildDev& b, const VacDev& v, const uint64_t* keys, const float* vals, int n_edges, const InsertRec& r,
                         int grid, size_t smem, int* occ) {
    auto kern = hnsw_update_kernel<ELEM, METRIC, LPR>;
    auto kern_disk = hnsw_update_disk_kernel<ELEM, METRIC, LPR, MODE == HB_VACUUM>;
    const void* k = MODE != HB_BUILD ? (const void*)kern_disk : (const void*)kern;
    VB_REQUIRE(smem <= HB_SMEM_MAX, "hnsw: %zu bytes of shared memory per CTA do not fit", smem);
    if (smem > 48 * 1024) VB_CUDA(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    if (occ) {
        VB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(occ, k, HN_WARPS * 32, smem));
        return VB_OK;
    }
    if (MODE != HB_BUILD) kern_disk<<<grid, HN_WARPS * 32, smem, ctx().stream>>>(b, keys, vals, n_edges, r, v);
    else kern<<<grid, HN_WARPS * 32, smem, ctx().stream>>>(b, keys, vals, n_edges);
    VB_CUDA(cudaGetLastError());
    count_launch();
    return VB_OK;
}

template <int ELEM, int METRIC, int MODE>
static BuildLaunch pick_lpr(int V) {
    // lanes per row: a whole warp for rows of >= 512 bytes, 8 lanes for >= 128 bytes, one lane for tiny rows
    if (V >= 32) return BuildLaunch{launch_insert<ELEM, METRIC, 32, MODE>, launch_update<ELEM, METRIC, 32, MODE>};
    if (V >= 8) return BuildLaunch{launch_insert<ELEM, METRIC, 8, MODE>, launch_update<ELEM, METRIC, 8, MODE>};
    return BuildLaunch{launch_insert<ELEM, METRIC, 1, MODE>, launch_update<ELEM, METRIC, 1, MODE>};
}

template <int MODE>
static bool pick_kernels(const Hnsw& h, int V, BuildLaunch* out) {
    if (h.elem == VB_VECTOR) {
        if (h.metric == VB_L2_SQUARED) *out = pick_lpr<VB_VECTOR, VB_L2_SQUARED, MODE>(V);
        else if (h.metric == VB_NEG_IP) *out = pick_lpr<VB_VECTOR, VB_NEG_IP, MODE>(V);
        else if (h.metric == VB_L1) *out = pick_lpr<VB_VECTOR, VB_L1, MODE>(V);
        else return false;
    } else if (h.elem == VB_HALFVEC) {
        if (h.metric == VB_L2_SQUARED) *out = pick_lpr<VB_HALFVEC, VB_L2_SQUARED, MODE>(V);
        else if (h.metric == VB_NEG_IP) *out = pick_lpr<VB_HALFVEC, VB_NEG_IP, MODE>(V);
        else if (h.metric == VB_L1) *out = pick_lpr<VB_HALFVEC, VB_L1, MODE>(V);
        else return false;
    } else {
        if (h.metric == VB_HAMMING) *out = pick_lpr<VB_BIT, VB_HAMMING, MODE>(V);
        else if (h.metric == VB_JACCARD) *out = pick_lpr<VB_BIT, VB_JACCARD, MODE>(V);
        else return false;
    }
    return true;
}

// R and the candidate arrays of hnsw_insert_kernel in global memory: `wcap` entries for each of `warps` warps
static void hb_point_global_r(void* buf, size_t warps, int wcap, VacDev* v) {
    const size_t nw = warps * (size_t)wcap;
    v->wcap = wcap;
    v->wk = (uint64_t*)buf;
    v->wi = (uint32_t*)(v->wk + 2 * nw);
    v->wd = (uint16_t*)(v->wi + 2 * nw);
    v->dead = (uint8_t*)(v->wd + nw);
}
static size_t hb_global_r_bytes(size_t warps, int wcap) { return warps * (size_t)wcap * (2 * 8 + 2 * 4 + 2 + 1); }
static int hb_take_global_r(Scratch& sc, size_t warps, int wcap, VacDev* v) {
    void* p;
    VB_TRY(sc.take(hb_global_r_bytes(warps, wcap), &p));
    hb_point_global_r(p, warps, wcap, v);
    return VB_OK;
}

static double build_uniform(uint64_t* st) {   // (0, 1]: -log() stays finite
    uint64_t z = (*st += 0x9e3779b97f4a7c15ULL);
    z = (z ^ (z >> 30)) * 0xbf58476d1ce4e5b9ULL;
    z = (z ^ (z >> 27)) * 0x94d049bb133111ebULL;
    z ^= z >> 31;
    return (double)((z >> 11) + 1) * (1.0 / 9007199254740992.0);
}

static int hnsw_build_impl(Hnsw& h, const void* rows, bool rows_on_host, int64_t n, int efc, uint64_t seed, const int32_t* levels_in) {
    Scratch sc;
    VB_REQUIRE(efc >= 4 && efc <= 1000, "ef_construction must be 4..1000 (src/hnsw.h:57-59)");
    VB_REQUIRE(efc >= 2 * h.m, "ef_construction must be greater than or equal to 2 * m (src/hnswbuild.c:713-716)");
    VB_REQUIRE(n >= 0 && n < (int64_t)0x7fffffff, "bad row count");
    Context& c = ctx();
    cudaStream_t s = c.stream;
    hnsw_release(h);
    ++h.generation;
    h.n = n;
    h.entry = -1;
    h.entry_level = -1;
    if (n == 0) {
        h.loaded = true;
        return VB_OK;
    }
    VB_REQUIRE(rows, "null rows");
    if (rows_on_host) VB_TRY(table_append_host(h.rows, rows, n));
    else VB_TRY(table_append_dev(h.rows, rows, n));

    // levels (HnswInitElement, src/hnswutils.c:248-254): (int) (-log(RandomDouble()) * ml), capped at HnswGetMaxLevel(m)
    const int m = h.m, lm0 = 2 * m;
    const double ml = 1.0 / std::log((double)m);
    const int max_level = std::min((int)((8192 - 24 - 8 - 4 - 4) / 6 / m) - 2, 63);   // src/hnsw.h:133 with BLCKSZ = 8192
    std::vector<int32_t> levels((size_t)n), uoff((size_t)n);
    uint64_t rs = seed ^ 0x2545f4914f6cdd1dULL;
    int64_t slots = 0;
    for (int64_t i = 0; i < n; ++i) {
        int lv = levels_in ? levels_in[i] : (int)(-std::log(build_uniform(&rs)) * ml);
        VB_REQUIRE(lv >= 0, "negative level");
        lv = std::min(lv, max_level);
        levels[(size_t)i] = lv;
        uoff[(size_t)i] = lv > 0 ? (int32_t)slots : -1;
        slots += lv;
        VB_REQUIRE(slots < (int64_t)0x7fffffff, "upper slot overflow");
    }
    h.upper_slots = slots;
    h.elem_cap = n;
    h.slot_cap = std::max<int64_t>(slots, 1);
    const size_t up_elems = (size_t)std::max<int64_t>(slots, 1) * m;
    VB_CUDA(cudaMalloc(&h.levels, sizeof(int32_t) * (size_t)n));
    VB_CUDA(cudaMalloc(&h.upper_off, sizeof(int32_t) * (size_t)n));
    VB_CUDA(cudaMalloc(&h.nbr0, sizeof(int32_t) * (size_t)n * lm0));
    VB_CUDA(cudaMalloc(&h.nd0, sizeof(float) * (size_t)n * lm0));
    VB_CUDA(cudaMalloc(&h.upper, sizeof(int32_t) * up_elems));
    VB_CUDA(cudaMalloc(&h.upper_d, sizeof(float) * up_elems));
    VB_CUDA(cudaMalloc(&h.dup_of, sizeof(int32_t) * (size_t)n));
    VB_CUDA(cudaMalloc(&h.n_heaptids, sizeof(int32_t) * (size_t)n));
    VB_CUDA(cudaMemcpyAsync(h.levels, levels.data(), sizeof(int32_t) * (size_t)n, cudaMemcpyHostToDevice, s));
    VB_CUDA(cudaMemcpyAsync(h.upper_off, uoff.data(), sizeof(int32_t) * (size_t)n, cudaMemcpyHostToDevice, s));
    VB_CUDA(cudaMemsetAsync(h.nbr0, 0xFF, sizeof(int32_t) * (size_t)n * lm0, s));
    VB_CUDA(cudaMemsetAsync(h.upper, 0xFF, sizeof(int32_t) * up_elems, s));
    VB_CUDA(cudaMemsetAsync(h.dup_of, 0xFF, sizeof(int32_t) * (size_t)n, s));
    fill_i32_kernel<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(h.n_heaptids, n, 1);
    VB_CUDA(cudaGetLastError());
    count_launch();

    BuildLaunch K;
    const int V = (int)(h.rows.stride / 16);
    if (!pick_kernels<HB_BUILD>(h, V, &K)) {
        set_error("hnsw build: unsupported metric %d for element type %d", h.metric, h.elem);
        return VB_EINVAL;
    }
    const int qvec = h.elem == VB_HALFVEC ? 2 * V : V;
    // R of ef_construction entries: in shared memory where it fits beside the row images, in global memory otherwise
    const bool r_shared = hb_insert_shared_cap(qvec, lm0, efc, efc) > 0;
    const size_t smem_ins = hb_insert_smem(qvec, r_shared ? efc : 0, lm0) * HN_WARPS;
    const size_t smem_upd = hb_update_smem(qvec) * HN_WARPS;

    BuildDev b{};
    b.g.rows = h.rows.d;
    b.g.stride = h.rows.stride;
    b.g.V = V;
    b.g.levels = h.levels;
    b.g.nbr0 = h.nbr0;
    b.g.upper_off = h.upper_off;
    b.g.upper = h.upper;
    b.g.m = m;
    b.g.n = n;
    b.nbr0_w = h.nbr0;
    b.upper_w = h.upper;
    b.nd0 = h.nd0;
    b.upper_d = h.upper_d;
    b.dup_of = h.dup_of;
    b.n_heaptids = h.n_heaptids;
    b.efc = efc;
    b.qvec = qvec;

    int occ_ins = 1, occ_upd = 1;
    VB_TRY(K.insert(b, VacDev{}, nullptr, 0, 0, 0, smem_ins, &occ_ins));
    VB_TRY(K.update(b, VacDev{}, nullptr, nullptr, 0, InsertRec{}, 0, smem_upd, &occ_upd));
    const int max_grid_ins = c.sm_count * std::max(1, occ_ins);
    const int max_grid_upd = c.sm_count * std::max(1, occ_upd) * 4;
    VacDev vr{};
    if (!r_shared) VB_TRY(hb_take_global_r(sc, (size_t)max_grid_ins * HN_WARPS, efc, &vr));

    void* d_flags;
    VB_TRY(sc.take(64, &d_flags));
    b.n_edges = (int*)d_flags;
    b.overflow = b.n_edges + 1;

    // visited tables: one per resident warp; the insertion layers share the large region, the greedy layers the small one
    uint32_t cap = 1u << 14;
    while (cap < (uint32_t)(efc * m * 16) && cap < (1u << 22)) cap <<= 1;

    // Elements of one batch do not see each other (like concurrent workers), so a batch stays a small fraction of the
    // graph it is inserted into: 1/64 by default (larger fractions lower the recall against the serial build).  Options "hnsw_build_fraction" / "hnsw_build_batch".
    const int64_t frac = std::max<int64_t>(1, c.hnsw_build_fraction);
    const int64_t b_max = std::min<int64_t>(1 << 20, std::max<int64_t>(1, c.hnsw_build_batch));
    int64_t done = 1;   // element 0 is the first entry point: no neighbours (src/hnswutils.c:1300-1302)
    h.entry = 0;
    h.entry_level = levels[0];
    while (done < n) {
        Scratch batch;
        int64_t B = std::min<int64_t>(std::min<int64_t>(b_max, std::max<int64_t>(1, done / frac)), n - done);
        // a batch ends at the first element that rises above the entry point: it becomes the entry point of the next batch
        int64_t promote = -1;
        int64_t max_edges = 0;
        for (int64_t i = 0; i < B; ++i) {
            const int lv = levels[(size_t)(done + i)];
            max_edges += lm0 + (int64_t)std::min(lv, h.entry_level) * m;
            if (lv > h.entry_level) {
                promote = done + i;
                B = i + 1;
                break;
            }
        }
        VB_REQUIRE(max_edges < (int64_t)0x7fffffff, "too many connection updates in one batch");
        b.g.entry = (int)h.entry;
        b.g.entry_level = h.entry_level;
        b.b0 = (int)done;
        b.B = (int)B;
        void *d_k1, *d_k2, *d_v1, *d_v2;
        VB_TRY(batch.take(sizeof(uint64_t) * (size_t)max_edges, &d_k1));
        VB_TRY(batch.take(sizeof(uint64_t) * (size_t)max_edges, &d_k2));
        VB_TRY(batch.take(sizeof(float) * (size_t)max_edges, &d_v1));
        VB_TRY(batch.take(sizeof(float) * (size_t)max_edges, &d_v2));
        b.edge_key = (uint64_t*)d_k1;
        b.edge_val = (float*)d_v1;
        const int grid_ins = (int)std::min<int64_t>((B + HN_WARPS - 1) / HN_WARPS, max_grid_ins);
        int flags[2] = {0, 0};
        for (int attempt = 0;; ++attempt) {
            const uint32_t vis_upper = std::max<uint32_t>(2048u, cap / 8);
            const uint32_t vis_cap = cap + vis_upper;
            const size_t need = (size_t)max_grid_ins * HN_WARPS * vis_cap * sizeof(uint32_t);
            if (h.vis_bytes < need) {
                if (h.vis) {
                    VB_CUDA(cudaStreamSynchronize(s));
                    cudaFree(h.vis);
                    h.vis = nullptr;
                    h.vis_bytes = 0;
                }
                if (cudaMalloc(&h.vis, need) != cudaSuccess) {
                    set_error("hnsw build: visited tables (%zu bytes) do not fit", need);
                    return VB_ENOMEM;
                }
                h.vis_bytes = need;
            }
            VB_CUDA(cudaMemsetAsync(d_flags, 0, 2 * sizeof(int), s));
            VB_TRY(K.insert(b, vr, h.vis, vis_cap, vis_upper, grid_ins, smem_ins, nullptr));
            hnsw_finalize_kernel<false><<<(unsigned)std::min<int64_t>((B * 32 + 127) / 128, (int64_t)c.sm_count * 16), 128, 0, s>>>(b);
            VB_CUDA(cudaGetLastError());
            count_launch();
            VB_CUDA(cudaMemcpyAsync(flags, d_flags, 2 * sizeof(int), cudaMemcpyDeviceToHost, s));
            VB_CUDA(cudaStreamSynchronize(s));
            if (!flags[1]) break;
            cap <<= 2;   // a visited table overflowed: repeat the batch's searches with larger ones (nothing was published)
            VB_REQUIRE(attempt < 5 && cap <= (1u << 26), "hnsw build: visited set overflow");
        }
        const int n_edges = flags[0];
        VB_REQUIRE(n_edges <= max_edges, "hnsw build: record overflow (%d > %lld)", n_edges, (long long)max_edges);
        if (n_edges > 0) {
            size_t tmp_bytes = 0;
            VB_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, tmp_bytes, (const uint64_t*)d_k1, (uint64_t*)d_k2, (const float*)d_v1,
                                                    (float*)d_v2, n_edges, 0, 57, s));
            Scratch sort;
            void* d_tmp;
            VB_TRY(sort.take(tmp_bytes, &d_tmp));
            VB_CUDA(cub::DeviceRadixSort::SortPairs(d_tmp, tmp_bytes, (const uint64_t*)d_k1, (uint64_t*)d_k2, (const float*)d_v1,
                                                    (float*)d_v2, n_edges, 0, 57, s));
            count_launch();
            const int grid_upd = (int)std::min<int64_t>(((int64_t)n_edges + HN_WARPS - 1) / HN_WARPS, max_grid_upd);
            VB_TRY(K.update(b, VacDev{}, (const uint64_t*)d_k2, (const float*)d_v2, n_edges, InsertRec{}, grid_upd, smem_upd, nullptr));
        }
        if (promote >= 0) {
            // UpdateGraphInMemory (src/hnswbuild.c:428-430): a duplicate never becomes the entry point
            int32_t dup = -1;
            VB_CUDA(cudaMemcpyAsync(&dup, h.dup_of + promote, sizeof(int32_t), cudaMemcpyDeviceToHost, s));
            VB_CUDA(cudaStreamSynchronize(s));
            if (dup < 0) {
                h.entry = promote;
                h.entry_level = levels[(size_t)promote];
            }
        }
        done += B;
    }
    VB_CUDA(cudaStreamSynchronize(s));
    h.loaded = true;
    return VB_OK;
}

// ----------------------------------------------------------------------------- insert into a resident image

// *p grows to new_bytes keeping its first used_bytes; fill >= -1: the array is new and its first fill_n entries are set
static int hnsw_grow(void** p, size_t used_bytes, size_t new_bytes, const char* what, int64_t fill_n = 0, int32_t fill = 0) {
    cudaStream_t s = ctx().stream;
    void* q = nullptr;
    if (cudaMalloc(&q, std::max<size_t>(new_bytes, 16)) != cudaSuccess) {
        cudaGetLastError();
        set_error("hnsw insert: %s (%zu bytes) does not fit in device memory", what, new_bytes);
        return VB_ENOMEM;
    }
    if (*p && used_bytes) VB_CUDA(cudaMemcpyAsync(q, *p, used_bytes, cudaMemcpyDeviceToDevice, s));
    if (fill_n > 0) {
        fill_i32_kernel<<<(unsigned)((fill_n + 255) / 256), 256, 0, s>>>((int32_t*)q, fill_n, fill);
        VB_CUDA(cudaGetLastError());
        count_launch();
    }
    VB_CUDA(cudaStreamSynchronize(s));
    cudaFree(*p);
    *p = q;
    return VB_OK;
}

// heap TID counts and the duplicate map of a loaded image: every element counts 1 and none is folded
static int hnsw_ensure_counts(Hnsw& h) {
    const size_t bytes = sizeof(int32_t) * (size_t)std::max<int64_t>(h.elem_cap, 1);
    if (!h.dup_of) VB_TRY(hnsw_grow((void**)&h.dup_of, 0, bytes, "duplicate map", h.n, -1));
    if (!h.n_heaptids) VB_TRY(hnsw_grow((void**)&h.n_heaptids, 0, bytes, "heap TID counts", h.n, 1));
    return VB_OK;
}

// Batched HnswInsertTupleOnDisk (src/hnswinsert.c:696-743) into the resident graph: the build's batch loop with the
// on-disk rules (RemoveElements in K1, FindDuplicateOnDisk in K1b, UpdateNeighborOnDisk in K2), then the change
// records: every slot K2 wrote plus the new elements' own lists, stably sorted by (element, layer, slot) and reduced to
// the last record of each slot.  Everything the call needs is reserved before the first kernel.
static int hnsw_insert_impl(Hnsw& h, const void* rows, bool rows_on_host, int64_t n, int efc, uint64_t seed, const int32_t* levels_in,
                            int32_t* out_dup_of, int64_t* out_nchanges) {
    Scratch sc;
    VB_REQUIRE(h.loaded, "hnsw index not loaded");
    VB_REQUIRE(efc >= 4 && efc <= 1000, "ef_construction must be 4..1000 (src/hnsw.h:57-59)");
    VB_REQUIRE(efc >= 2 * h.m, "ef_construction must be greater than or equal to 2 * m (src/hnswbuild.c:713-716)");
    const int64_t n0 = h.n;
    VB_REQUIRE(n >= 0 && n0 + n < (int64_t)0x7fffffff, "bad row count");
    VB_REQUIRE(rows || n == 0, "null rows");
    BuildLaunch K;
    const int V = (int)(h.rows.stride / 16);
    if (!pick_kernels<HB_INSERT>(h, V, &K)) {
        set_error("hnsw insert: unsupported metric %d for element type %d", h.metric, h.elem);
        return VB_EINVAL;
    }
    const int m = h.m, lm0 = 2 * m;
    const int qvec = h.elem == VB_HALFVEC ? 2 * V : V;
    const bool r_shared = hb_insert_shared_cap(qvec, lm0, efc, efc) > 0;   // (as the build's)
    const size_t smem_ins = hb_insert_smem(qvec, r_shared ? efc : 0, lm0) * HN_WARPS;
    const size_t smem_upd = hb_update_disk_smem(qvec) * HN_WARPS;

    // levels (HnswInitElement, src/hnswutils.c:248-254), capped at HnswGetMaxLevel(m), and the new upper slots
    const double ml = 1.0 / std::log((double)m);
    const int max_level = std::min((int)((8192 - 24 - 8 - 4 - 4) / 6 / m) - 2, 63);   // src/hnsw.h:133 with BLCKSZ = 8192
    std::vector<int32_t> levels((size_t)n), uoff((size_t)n);
    uint64_t rs = seed ^ 0x2545f4914f6cdd1dULL;
    const int64_t slots0 = h.upper_slots;
    int64_t slots = slots0, total_edges = 0;
    for (int64_t i = 0; i < n; ++i) {
        int lv = levels_in ? levels_in[i] : (int)(-std::log(build_uniform(&rs)) * ml);
        VB_REQUIRE(lv >= 0, "negative level");
        lv = std::min(lv, max_level);
        levels[(size_t)i] = lv;
        uoff[(size_t)i] = lv > 0 ? (int32_t)slots : -1;
        slots += lv;
        VB_REQUIRE(slots < (int64_t)0x7fffffff, "upper slot overflow");
        total_edges += lm0 + (int64_t)lv * m;
    }
    VB_REQUIRE(total_edges < (int64_t)0x7fffffff / 2, "too many connection updates in one call");
    if (out_nchanges) *out_nchanges = 0;
    if (n == 0) {
        h.n_changes = 0;
        return VB_OK;
    }
    // one record per slot K2 writes (at most one per connection update) plus the new elements' lists
    const int64_t recs = 2 * total_edges;
    const int64_t n1 = n0 + n;
    Context& c = ctx();
    cudaStream_t s = c.stream;

    // ---- reservations: nothing below changes the image until they have all succeeded
    VB_TRY(table_reserve(h.rows, n1));
    VB_TRY(hnsw_ensure_counts(h));
    {
        const int64_t ecap = n1 > h.elem_cap ? std::max<int64_t>(n1, h.elem_cap + h.elem_cap / 2) : h.elem_cap;
        const int64_t scap = slots > h.slot_cap ? std::max<int64_t>(slots, h.slot_cap + h.slot_cap / 2) : h.slot_cap;
        struct Arr {
            void** p;
            size_t bytes;   // per element or per upper slot
            bool upper, keep;
            const char* what;
        } arrs[] = {{(void**)&h.levels, 4, false, true, "levels"},
                    {(void**)&h.upper_off, 4, false, true, "upper slot offsets"},
                    {(void**)&h.nbr0, 4 * (size_t)lm0, false, true, "layer-0 neighbours"},
                    {(void**)&h.nd0, 4 * (size_t)lm0, false, false, "layer-0 distances"},
                    {(void**)&h.dup_of, 4, false, true, "duplicate map"},
                    {(void**)&h.n_heaptids, 4, false, true, "heap TID counts"},
                    {(void**)&h.upper, 4 * (size_t)m, true, true, "upper neighbours"},
                    {(void**)&h.upper_d, 4 * (size_t)m, true, false, "upper distances"}};
        // (the distances are scratch for the new elements' own lists: the on-disk update never reads a stored one)
        for (const Arr& a : arrs) {
            const int64_t cap = a.upper ? scap : ecap, have = a.upper ? h.slot_cap : h.elem_cap, used = a.upper ? slots0 : n0;
            if (*a.p && cap == have) continue;
            VB_TRY(hnsw_grow(a.p, a.keep ? (size_t)used * a.bytes : 0, (size_t)cap * a.bytes, a.what));
        }
        h.elem_cap = ecap;
        h.slot_cap = scap;
    }
    if (recs > h.rec_cap) {
        h.n_changes = 0;
        h.rec_cap = 0;
        VB_TRY(hnsw_grow((void**)&h.rec_key, 0, sizeof(uint64_t) * (size_t)recs, "change records"));
        VB_TRY(hnsw_grow((void**)&h.rec_val, 0, sizeof(int32_t) * (size_t)recs, "change records"));
        h.rec_cap = recs;
    }
    void *d_k1, *d_k2, *d_v1, *d_v2, *d_keep, *d_flags, *d_tmp;
    VB_TRY(sc.take(sizeof(uint64_t) * (size_t)total_edges, &d_k1));
    VB_TRY(sc.take(sizeof(uint64_t) * (size_t)recs, &d_k2));
    VB_TRY(sc.take(sizeof(float) * (size_t)total_edges, &d_v1));
    VB_TRY(sc.take(sizeof(float) * (size_t)recs, &d_v2));
    VB_TRY(sc.take((size_t)recs, &d_keep));
    VB_TRY(sc.take(64, &d_flags));
    // one CUB temporary for every sort and select below, sized for their largest counts
    size_t tmp_bytes = 0;
    {
        size_t t1 = 0, t2 = 0, t3 = 0, t4 = 0;
        VB_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, t1, (const uint64_t*)d_k1, (uint64_t*)d_k2, (const float*)d_v1, (float*)d_v2,
                                                (int)total_edges, 0, 57, s));
        VB_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, t2, (const uint64_t*)h.rec_key, (uint64_t*)d_k2, (const int32_t*)h.rec_val,
                                                (int32_t*)d_v2, (int)recs, 0, 45, s));
        VB_CUDA(cub::DeviceSelect::Flagged(nullptr, t3, (const uint64_t*)d_k2, (const uint8_t*)d_keep, h.rec_key, (int*)d_flags, (int)recs, s));
        VB_CUDA(cub::DeviceSelect::Flagged(nullptr, t4, (const int32_t*)d_v2, (const uint8_t*)d_keep, h.rec_val, (int*)d_flags, (int)recs, s));
        tmp_bytes = std::max(std::max(t1, t2), std::max(t3, t4));
        VB_TRY(sc.take(tmp_bytes, &d_tmp));
    }
    int occ_ins = 1, occ_upd = 1;
    VB_TRY(K.insert(BuildDev{}, VacDev{}, nullptr, 0, 0, 0, smem_ins, &occ_ins));
    VB_TRY(K.update(BuildDev{}, VacDev{}, nullptr, nullptr, 0, InsertRec{}, 0, smem_upd, &occ_upd));
    const int max_grid_ins = c.sm_count * std::max(1, occ_ins);
    const int max_grid_upd = c.sm_count * std::max(1, occ_upd) * 4;
    VacDev vr{};
    if (!r_shared) VB_TRY(hb_take_global_r(sc, (size_t)max_grid_ins * HN_WARPS, efc, &vr));
    uint32_t cap = 1u << 14;
    while (cap < (uint32_t)(efc * m * 16) && cap < (1u << 22)) cap <<= 1;
    auto reserve_vis = [&](uint32_t vis_cap) -> int {
        const size_t need = (size_t)max_grid_ins * HN_WARPS * vis_cap * sizeof(uint32_t);
        if (h.vis_bytes >= need) return VB_OK;
        if (h.vis) {
            VB_CUDA(cudaStreamSynchronize(s));
            cudaFree(h.vis);
            h.vis = nullptr;
            h.vis_bytes = 0;
        }
        if (cudaMalloc(&h.vis, need) != cudaSuccess) {
            cudaGetLastError();
            set_error("hnsw insert: visited tables (%zu bytes) do not fit", need);
            return VB_ENOMEM;
        }
        h.vis_bytes = need;
        return VB_OK;
    };
    VB_TRY(reserve_vis(cap + std::max<uint32_t>(2048u, cap / 8)));

    // ---- the image changes from here on
    ++h.generation;
    h.n_changes = 0;
    if (rows_on_host) VB_TRY(table_append_host(h.rows, rows, n));
    else VB_TRY(table_append_dev(h.rows, rows, n));
    VB_CUDA(cudaMemcpyAsync(h.levels + n0, levels.data(), sizeof(int32_t) * (size_t)n, cudaMemcpyHostToDevice, s));
    VB_CUDA(cudaMemcpyAsync(h.upper_off + n0, uoff.data(), sizeof(int32_t) * (size_t)n, cudaMemcpyHostToDevice, s));
    VB_CUDA(cudaMemsetAsync(h.nbr0 + (size_t)n0 * lm0, 0xFF, sizeof(int32_t) * (size_t)n * lm0, s));
    if (slots > slots0) VB_CUDA(cudaMemsetAsync(h.upper + (size_t)slots0 * m, 0xFF, sizeof(int32_t) * (size_t)(slots - slots0) * m, s));
    VB_CUDA(cudaMemsetAsync(h.dup_of + n0, 0xFF, sizeof(int32_t) * (size_t)n, s));
    fill_i32_kernel<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(h.n_heaptids + n0, n, 1);
    VB_CUDA(cudaGetLastError());
    count_launch();
    h.n = n1;
    h.upper_slots = slots;

    BuildDev b{};
    b.g.rows = h.rows.d;
    b.g.stride = h.rows.stride;
    b.g.V = V;
    b.g.levels = h.levels;
    b.g.nbr0 = h.nbr0;
    b.g.upper_off = h.upper_off;
    b.g.upper = h.upper;
    b.g.m = m;
    b.g.n = n1;
    b.nbr0_w = h.nbr0;
    b.upper_w = h.upper;
    b.nd0 = h.nd0;
    b.upper_d = h.upper_d;
    b.dup_of = h.dup_of;
    b.n_heaptids = h.n_heaptids;
    b.efc = efc;
    b.qvec = qvec;
    b.n_edges = (int*)d_flags;
    b.overflow = b.n_edges + 1;
    b.edge_key = (uint64_t*)d_k1;
    b.edge_val = (float*)d_v1;
    const InsertRec rec{h.rec_key, h.rec_val, b.n_edges + 2};
    VB_CUDA(cudaMemsetAsync(rec.n, 0, sizeof(int), s));

    // batches as in the build (hnsw_build_fraction / hnsw_build_batch of the graph inserted into so far)
    const int64_t frac = std::max<int64_t>(1, c.hnsw_build_fraction);
    const int64_t b_max = std::min<int64_t>(1 << 20, std::max<int64_t>(1, c.hnsw_build_batch));
    int64_t done = n0;
    if (h.entry < 0) {   // empty image: the first row is the entry point, with no neighbours (src/hnswutils.c:1300-1302)
        h.entry = n0;
        h.entry_level = levels[0];
        done = n0 + 1;
    }
    while (done < n1) {
        int64_t B = std::min<int64_t>(std::min<int64_t>(b_max, std::max<int64_t>(1, done / frac)), n1 - done);
        int64_t promote = -1;
        for (int64_t i = 0; i < B; ++i)
            if (levels[(size_t)(done - n0 + i)] > h.entry_level) {   // the entry point moves to a strictly higher level only
                promote = done + i;
                B = i + 1;
                break;
            }
        b.g.entry = (int)h.entry;
        b.g.entry_level = h.entry_level;
        b.b0 = (int)done;
        b.B = (int)B;
        const int grid_ins = (int)std::min<int64_t>((B + HN_WARPS - 1) / HN_WARPS, max_grid_ins);
        int flags[2] = {0, 0};
        for (int attempt = 0;; ++attempt) {
            const uint32_t vis_upper = std::max<uint32_t>(2048u, cap / 8);
            const uint32_t vis_cap = cap + vis_upper;
            VB_TRY(reserve_vis(vis_cap));
            VB_CUDA(cudaMemsetAsync(d_flags, 0, 2 * sizeof(int), s));
            VB_TRY(K.insert(b, vr, h.vis, vis_cap, vis_upper, grid_ins, smem_ins, nullptr));
            hnsw_finalize_kernel<true><<<(unsigned)std::min<int64_t>((B * 32 + 127) / 128, (int64_t)c.sm_count * 16), 128, 0, s>>>(b);
            VB_CUDA(cudaGetLastError());
            count_launch();
            VB_CUDA(cudaMemcpyAsync(flags, d_flags, 2 * sizeof(int), cudaMemcpyDeviceToHost, s));
            VB_CUDA(cudaStreamSynchronize(s));
            if (!flags[1]) break;
            cap <<= 2;   // a visited table overflowed: repeat the batch's searches with larger ones (nothing was published)
            VB_REQUIRE(attempt < 5 && cap <= (1u << 26), "hnsw insert: visited set overflow");
        }
        const int n_edges = flags[0];
        VB_REQUIRE(n_edges <= total_edges, "hnsw insert: record overflow (%d > %lld)", n_edges, (long long)total_edges);
        if (n_edges > 0) {
            size_t tb = tmp_bytes;
            VB_CUDA(cub::DeviceRadixSort::SortPairs(d_tmp, tb, (const uint64_t*)d_k1, (uint64_t*)d_k2, (const float*)d_v1, (float*)d_v2,
                                                    n_edges, 0, 57, s));
            count_launch();
            const int grid_upd = (int)std::min<int64_t>(((int64_t)n_edges + HN_WARPS - 1) / HN_WARPS, max_grid_upd);
            VB_TRY(K.update(b, VacDev{}, (const uint64_t*)d_k2, (const float*)d_v2, n_edges, rec, grid_upd, smem_upd, nullptr));
        }
        if (promote >= 0) {
            // a folded row never becomes the entry point
            int32_t dup = -1;
            VB_CUDA(cudaMemcpyAsync(&dup, h.dup_of + promote, sizeof(int32_t), cudaMemcpyDeviceToHost, s));
            VB_CUDA(cudaStreamSynchronize(s));
            if (dup < 0) {
                h.entry = promote;
                h.entry_level = levels[(size_t)(promote - n0)];
            }
        }
        done += B;
    }

    // ---- change records
    hnsw_new_records_kernel<<<(unsigned)std::min<int64_t>((n * 32 + 127) / 128, (int64_t)c.sm_count * 16), 128, 0, s>>>(b, rec, n0, n);
    VB_CUDA(cudaGetLastError());
    count_launch();
    int n_rec = 0, n_sel = 0;
    VB_CUDA(cudaMemcpyAsync(&n_rec, rec.n, sizeof(int), cudaMemcpyDeviceToHost, s));
    VB_CUDA(cudaStreamSynchronize(s));
    VB_REQUIRE(n_rec <= recs, "hnsw insert: change record overflow (%d > %lld)", n_rec, (long long)recs);
    if (n_rec > 0) {
        int* d_nsel = b.n_edges + 3;
        size_t tb = tmp_bytes;
        VB_CUDA(cub::DeviceRadixSort::SortPairs(d_tmp, tb, (const uint64_t*)h.rec_key, (uint64_t*)d_k2, (const int32_t*)h.rec_val,
                                                (int32_t*)d_v2, n_rec, 0, 45, s));
        hnsw_last_of_key_kernel<<<(unsigned)((n_rec + 255) / 256), 256, 0, s>>>((const uint64_t*)d_k2, n_rec, (uint8_t*)d_keep);
        VB_CUDA(cudaGetLastError());
        VB_CUDA(cub::DeviceSelect::Flagged(d_tmp, tb, (const uint64_t*)d_k2, (const uint8_t*)d_keep, h.rec_key, d_nsel, n_rec, s));
        VB_CUDA(cub::DeviceSelect::Flagged(d_tmp, tb, (const int32_t*)d_v2, (const uint8_t*)d_keep, h.rec_val, d_nsel, n_rec, s));
        count_launch(4);
        VB_CUDA(cudaMemcpyAsync(&n_sel, d_nsel, sizeof(int), cudaMemcpyDeviceToHost, s));
    }
    if (out_dup_of) VB_CUDA(cudaMemcpyAsync(out_dup_of, h.dup_of + n0, sizeof(int32_t) * (size_t)n, cudaMemcpyDeviceToHost, s));
    VB_CUDA(cudaStreamSynchronize(s));
    h.n_changes = n_sel;
    if (out_nchanges) *out_nchanges = n_sel;
    return VB_OK;
}

// ----------------------------------------------------------------------------- vacuum a resident image

// NeedsUpdated (src/hnswvacuum.c:178-220) of the elements [from, n): live, not `skip`, and a slot on any layer names an
// element with no heap TIDs, or the last layer-0 slot is empty
__global__ void hnsw_needs_update_kernel(HnswDev g, const int32_t* __restrict__ counts, int64_t from, int skip, uint8_t* __restrict__ flag) {
    const int64_t e = from + blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (e >= g.n) return;
    const int lm0 = 2 * g.m;
    bool need = false;
    if (counts[e] != 0 && e != skip) {
        const int32_t* l0 = g.nbr0 + (size_t)e * lm0;
        need = l0[lm0 - 1] < 0;
        for (int i = 0; i < lm0 && !need; ++i) need = l0[i] >= 0 && counts[l0[i]] == 0;
        for (int lc = 1; lc <= g.levels[e] && !need; ++lc) {
            const int32_t* u = g.upper + ((size_t)g.upper_off[e] + (lc - 1)) * g.m;
            for (int i = 0; i < g.m && !need; ++i) need = u[i] >= 0 && counts[u[i]] == 0;
        }
    }
    flag[e - from] = need ? 1 : 0;
}

// the update records of a repair batch (UpdateNeighborsOnDisk's loop, src/hnswinsert.c:545-580): one per staged neighbour,
// source = the position in the batch's list
__global__ void __launch_bounds__(128) hnsw_vacuum_edges_kernel(BuildDev b, VacDev v) {
    const HnswDev& g = b.g;
    const int lane = threadIdx.x % 32;
    const int gwarp = (int)((blockIdx.x * (int64_t)blockDim.x + threadIdx.x) / 32);
    const int nwarps = (int)((gridDim.x * (int64_t)blockDim.x) / 32);
    const int lm0 = 2 * g.m;
    if (g.entry < 0) return;
    for (int w = gwarp; w < b.B; w += nwarps) {
        const int e = v.list[w];
        const int top = min(g.levels[e], g.entry_level);
        for (int lc = top; lc >= 0; --lc) {
            const int lm = lc == 0 ? lm0 : g.m;
            const int32_t* ids = lc == 0 ? v.stage0 + (size_t)w * lm : v.stage_up + ((size_t)g.upper_off[e] + (lc - 1)) * (size_t)lm;
            const float* ds = lc == 0 ? b.nd0 + (size_t)e * lm : b.upper_d + ((size_t)g.upper_off[e] + (lc - 1)) * (size_t)lm;
            for (int off = 0; off < lm; off += 32) {
                const int t = off + lane < lm ? ids[off + lane] : -1;
                const unsigned vm = __ballot_sync(0xffffffffu, t >= 0);
                const int cnt = __popc(vm);
                if (cnt == 0) break;
                int slot = 0;
                if (lane == 0) slot = atomicAdd(b.n_edges, cnt);
                slot = __shfl_sync(0xffffffffu, slot, 0);
                if (t >= 0) {
                    const int p = slot + __popc(vm & ((1u << lane) - 1u));
                    b.edge_key[p] = ((uint64_t)(uint32_t)t << 26) | ((uint64_t)lc << 20) | (uint64_t)w;
                    b.edge_val[p] = ds[off + lane];
                }
            }
        }
    }
}

// the staged tuples of the batch replace the repaired elements' own (PageIndexTupleOverwrite, src/hnswvacuum.c:264-266)
__global__ void hnsw_vacuum_publish_kernel(BuildDev b, VacDev v) {
    const HnswDev& g = b.g;
    const int w = blockIdx.x;
    const int e = v.list[w];
    const int lm0 = 2 * g.m;
    for (int i = threadIdx.x; i < lm0; i += blockDim.x) b.nbr0_w[(size_t)e * lm0 + i] = v.stage0[(size_t)w * lm0 + i];
    for (int lc = 1; lc <= g.levels[e]; ++lc) {
        const size_t o = ((size_t)g.upper_off[e] + (lc - 1)) * g.m;
        for (int i = threadIdx.x; i < g.m; i += blockDim.x) b.upper_w[o + i] = v.stage_up[o + i];
    }
}

// MarkDeleted (src/hnswvacuum.c:594-729): every neighbour slot of an element with no heap TIDs is cleared
__global__ void hnsw_mark_deleted_kernel(BuildDev b, const int32_t* __restrict__ counts) {
    const HnswDev& g = b.g;
    const int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (e >= g.n || counts[e] != 0) return;
    const int lm0 = 2 * g.m;
    for (int i = 0; i < lm0; ++i) b.nbr0_w[(size_t)e * lm0 + i] = -1;
    for (int lc = 1; lc <= g.levels[e]; ++lc)
        for (int i = 0; i < g.m; ++i) b.upper_w[((size_t)g.upper_off[e] + (lc - 1)) * g.m + i] = -1;
}

// the change records of a vacuum: every slot whose value differs from the snapshot taken before the call
__global__ void hnsw_slot_diff_kernel(HnswDev g, const int32_t* __restrict__ old0, const int32_t* __restrict__ old_up, InsertRec r) {
    const int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (e >= g.n) return;
    const int lm0 = 2 * g.m;
    for (int lc = 0; lc <= g.levels[e]; ++lc) {
        const int lm = lc == 0 ? lm0 : g.m;
        const size_t o = lc == 0 ? (size_t)e * lm0 : ((size_t)g.upper_off[e] + (lc - 1)) * g.m;
        const int32_t* now = lc == 0 ? g.nbr0 : g.upper;
        const int32_t* was = lc == 0 ? old0 : old_up;
        for (int i = 0; i < lm; ++i)
            if (now[o + i] != was[o + i]) hb_record(r, (int)e, lc, i, now[o + i]);
    }
}

// hnswbulkdelete's graph work (src/hnswvacuum.c:776-797 without RemoveHeapTids, which the caller runs on the pages) on the
// resident image: RepairGraphEntryPoint, RepairGraph in batches (NeedsUpdated evaluated at each batch's start, the batch
// taken from the candidates in element order), MarkDeleted, then the change records as the diff against a snapshot of the
// neighbour arrays.  Everything the call needs is reserved before the first kernel.
static int hnsw_vacuum_impl(Hnsw& h, const int32_t* counts, int efc, int64_t* out_nrepaired, int64_t* out_nchanges) {
    Scratch sc;
    VB_REQUIRE(h.loaded, "hnsw index not loaded");
    VB_REQUIRE(efc >= 4 && efc <= 1000, "ef_construction must be 4..1000 (src/hnsw.h:57-59)");
    VB_REQUIRE(efc >= 2 * h.m, "ef_construction must be greater than or equal to 2 * m (src/hnswbuild.c:713-716)");
    const int64_t n = h.n;
    VB_REQUIRE(counts || n == 0, "null counts");
    for (int64_t i = 0; i < n; ++i)
        VB_REQUIRE(counts[i] >= 0 && counts[i] <= 10, "vb_hnsw_vacuum: counts[%lld] = %d is not in 0..10 (HNSW_HEAPTIDS, src/hnsw.h:69)",
                   (long long)i, counts[i]);
    BuildLaunch K;
    const int V = (int)(h.rows.stride / 16);
    if (!pick_kernels<HB_VACUUM>(h, V, &K)) {
        set_error("hnsw vacuum: unsupported metric %d for element type %d", h.metric, h.elem);
        return VB_EINVAL;
    }
    if (out_nrepaired) *out_nrepaired = 0;
    if (out_nchanges) *out_nchanges = 0;
    const int m = h.m, lm0 = 2 * m;
    const int qvec = h.elem == VB_HALFVEC ? 2 * V : V;
    const int efv = efc + 1;   // "Add one for existing element" (src/hnswutils.c:1315-1317)
    // R holds up to four times ef (elements being deleted do not count towards ef): the largest such capacity that fits in
    // shared memory, or four times ef in global memory when not even ef fits
    const int wcap_s = hb_insert_shared_cap(qvec, lm0, efv, 4 * efv);
    const size_t smem_glob = hb_insert_smem(qvec, 0, lm0) * HN_WARPS;
    const size_t smem_ins = wcap_s > 0 ? hb_insert_smem(qvec, wcap_s, lm0) * HN_WARPS : smem_glob;
    const size_t smem_upd = hb_update_disk_smem(qvec) * HN_WARPS;
    if (n == 0) {
        ++h.generation;
        h.n_changes = 0;
        return VB_OK;
    }
    Context& c = ctx();
    cudaStream_t s = c.stream;

    std::vector<int32_t> levels((size_t)n), dup((size_t)n, -1);
    VB_CUDA(cudaMemcpyAsync(levels.data(), h.levels, sizeof(int32_t) * (size_t)n, cudaMemcpyDeviceToHost, s));
    if (h.dup_of) VB_CUDA(cudaMemcpyAsync(dup.data(), h.dup_of, sizeof(int32_t) * (size_t)n, cudaMemcpyDeviceToHost, s));
    VB_CUDA(cudaStreamSynchronize(s));
    int64_t live = 0;
    for (int64_t i = 0; i < n; ++i) {
        VB_REQUIRE(dup[(size_t)i] < 0 || counts[i] == 0, "vb_hnsw_vacuum: row %lld was folded into element %d and is no element: its count must be 0",
                   (long long)i, dup[(size_t)i]);
        live += counts[i] != 0;
    }
    const int64_t frac = std::max<int64_t>(1, c.hnsw_build_fraction);
    const int64_t b_max = std::min<int64_t>(std::min<int64_t>(1 << 20, std::max<int64_t>(1, c.hnsw_build_batch)), std::max<int64_t>(1, live / frac));
    const int top_level = std::max(h.entry_level, 0);
    const int64_t max_edges = b_max * (lm0 + (int64_t)top_level * m);
    VB_REQUIRE(max_edges < (int64_t)0x7fffffff, "too many connection updates in one batch");
    const int64_t slots = h.upper_slots;
    const int64_t recs = n * lm0 + slots * m;   // every slot can change at most once
    VB_REQUIRE(recs < (int64_t)0x7fffffff, "hnsw vacuum: too many neighbour slots");

    // ---- reservations: nothing below changes the image until they have all succeeded
    VB_TRY(hnsw_ensure_counts(h));
    // distance scratch of the repaired elements' lists (an image made by vb_hnsw_load has none)
    if (!h.nd0) VB_TRY(hnsw_grow((void**)&h.nd0, 0, sizeof(float) * (size_t)h.elem_cap * lm0, "layer-0 distances"));
    if (!h.upper_d) VB_TRY(hnsw_grow((void**)&h.upper_d, 0, sizeof(float) * (size_t)h.slot_cap * m, "upper distances"));
    if (recs > h.rec_cap) {
        h.n_changes = 0;
        h.rec_cap = 0;
        VB_TRY(hnsw_grow((void**)&h.rec_key, 0, sizeof(uint64_t) * (size_t)recs, "change records"));
        VB_TRY(hnsw_grow((void**)&h.rec_val, 0, sizeof(int32_t) * (size_t)recs, "change records"));
        h.rec_cap = recs;
    }
    void *d_k1, *d_k2, *d_v1, *d_v2, *d_flags, *d_tmp, *d_need, *d_sel, *d_old0, *d_oldup, *d_stage0, *d_stageup;
    VB_TRY(sc.take(sizeof(uint64_t) * (size_t)std::max<int64_t>(max_edges, 1), &d_k1));
    VB_TRY(sc.take(sizeof(uint64_t) * (size_t)std::max(max_edges, recs), &d_k2));
    VB_TRY(sc.take(sizeof(float) * (size_t)std::max<int64_t>(max_edges, 1), &d_v1));
    VB_TRY(sc.take(sizeof(float) * (size_t)std::max(max_edges, recs), &d_v2));
    VB_TRY(sc.take((size_t)n, &d_need));
    VB_TRY(sc.take(64, &d_flags));
    VB_TRY(sc.take(sizeof(int32_t) * (size_t)(n + 1), &d_sel));
    VB_TRY(sc.take(sizeof(int32_t) * (size_t)n * lm0, &d_old0));
    VB_TRY(sc.take(sizeof(int32_t) * (size_t)std::max<int64_t>(slots, 1) * m, &d_oldup));
    VB_TRY(sc.take(sizeof(int32_t) * (size_t)b_max * lm0, &d_stage0));
    VB_TRY(sc.take(sizeof(int32_t) * (size_t)std::max<int64_t>(slots, 1) * m, &d_stageup));
    // one CUB temporary for every sort and select below, sized for their largest counts
    size_t tmp_bytes = 0;
    {
        size_t t1 = 0, t2 = 0, t3 = 0;
        VB_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, t1, (const uint64_t*)d_k1, (uint64_t*)d_k2, (const float*)d_v1, (float*)d_v2,
                                                (int)std::max<int64_t>(max_edges, 1), 0, 57, s));
        VB_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, t2, (const uint64_t*)d_k2, h.rec_key, (const int32_t*)d_v2, h.rec_val, (int)recs, 0,
                                                45, s));
        VB_CUDA(cub::DeviceSelect::Flagged(nullptr, t3, cub::CountingInputIterator<int32_t>(0), (const uint8_t*)d_need, (int32_t*)d_sel,
                                           (int*)d_flags, (int)n, s));
        tmp_bytes = std::max(t1, std::max(t2, t3));
        VB_TRY(sc.take(tmp_bytes, &d_tmp));
    }
    int occ_ins = 1, occ_glob = 1, occ_upd = 1;
    VB_TRY(K.insert(BuildDev{}, VacDev{}, nullptr, 0, 0, 0, smem_ins, &occ_ins));
    VB_TRY(K.insert(BuildDev{}, VacDev{}, nullptr, 0, 0, 0, smem_glob, &occ_glob));
    VB_TRY(K.update(BuildDev{}, VacDev{}, nullptr, nullptr, 0, InsertRec{}, 0, smem_upd, &occ_upd));
    const int max_grid_ins = c.sm_count * std::max(1, std::max(occ_ins, occ_glob));
    const int max_grid_upd = c.sm_count * std::max(1, occ_upd) * 4;
    uint32_t cap = 1u << 14;
    while (cap < (uint32_t)(efv * m * 16) && cap < (1u << 22)) cap <<= 1;
    auto reserve_vis = [&](uint32_t vis_cap) -> int {
        const size_t need = (size_t)max_grid_ins * HN_WARPS * vis_cap * sizeof(uint32_t);
        if (h.vis_bytes >= need) return VB_OK;
        if (h.vis) {
            VB_CUDA(cudaStreamSynchronize(s));
            cudaFree(h.vis);
            h.vis = nullptr;
            h.vis_bytes = 0;
        }
        if (cudaMalloc(&h.vis, need) != cudaSuccess) {
            cudaGetLastError();
            set_error("hnsw vacuum: visited tables (%zu bytes) do not fit", need);
            return VB_ENOMEM;
        }
        h.vis_bytes = need;
        return VB_OK;
    };
    VB_TRY(reserve_vis(cap + std::max<uint32_t>(2048u, cap / 8)));
    VacDev v{};
    v.wcap = wcap_s;
    if (wcap_s == 0) VB_TRY(hb_take_global_r(sc, (size_t)max_grid_ins * HN_WARPS, 4 * efv, &v));

    // ---- the image changes from here on
    ++h.generation;
    h.n_changes = 0;
    VB_CUDA(cudaMemcpyAsync(h.n_heaptids, counts, sizeof(int32_t) * (size_t)n, cudaMemcpyHostToDevice, s));
    VB_CUDA(cudaMemcpyAsync(d_old0, h.nbr0, sizeof(int32_t) * (size_t)n * lm0, cudaMemcpyDeviceToDevice, s));
    if (slots > 0) VB_CUDA(cudaMemcpyAsync(d_oldup, h.upper, sizeof(int32_t) * (size_t)slots * m, cudaMemcpyDeviceToDevice, s));

    BuildDev b{};
    b.g.rows = h.rows.d;
    b.g.stride = h.rows.stride;
    b.g.V = V;
    b.g.levels = h.levels;
    b.g.nbr0 = h.nbr0;
    b.g.upper_off = h.upper_off;
    b.g.upper = h.upper;
    b.g.m = m;
    b.g.n = n;
    b.nbr0_w = h.nbr0;
    b.upper_w = h.upper;
    b.nd0 = h.nd0;
    b.upper_d = h.upper_d;
    b.dup_of = h.dup_of;
    b.n_heaptids = h.n_heaptids;
    b.efc = efv;
    b.qvec = qvec;
    b.n_edges = (int*)d_flags;
    b.overflow = b.n_edges + 1;
    b.edge_key = (uint64_t*)d_k1;
    b.edge_val = (float*)d_v1;
    v.stage0 = (int32_t*)d_stage0;
    v.stage_up = (int32_t*)d_stageup;
    v.counts = h.n_heaptids;
    v.wfull = b.n_edges + 2;
    int* d_nsel = b.n_edges + 3;
    void* wbuf = nullptr;   // R in global memory after a repair overflowed the one it started on
    size_t wbuf_bytes = 0;
    int64_t nrep = 0;
    // R of wcap entries per warp in global memory
    auto global_r = [&](int wcap) -> int {
        const size_t need = hb_global_r_bytes((size_t)max_grid_ins * HN_WARPS, wcap);
        if (wbuf_bytes < need) {
            if (wbuf) {
                VB_CUDA(cudaStreamSynchronize(s));
                cudaFree(wbuf);
                wbuf = nullptr;
                wbuf_bytes = 0;
            }
            if (cudaMalloc(&wbuf, need) != cudaSuccess) {
                cudaGetLastError();
                set_error("hnsw vacuum: candidate buffers (%zu bytes) do not fit", need);
                return VB_ENOMEM;
            }
            wbuf_bytes = need;
        }
        hb_point_global_r(wbuf, (size_t)max_grid_ins * HN_WARPS, wcap, &v);
        return VB_OK;
    };

    // NeedsUpdated of the elements [from, n) (skip: the entry point) into d_need
    auto needs = [&](int64_t from, int skip) -> int {
        hnsw_needs_update_kernel<<<(unsigned)((n - from + 255) / 256), 256, 0, s>>>(b.g, h.n_heaptids, from, skip, (uint8_t*)d_need);
        VB_CUDA(cudaGetLastError());
        count_launch();
        return VB_OK;
    };
    // RepairGraphElement of the B elements d_list[0..B) against the graph as it stands, from entry point `ep`
    auto repair = [&](const int32_t* d_list, int B, int64_t ep) -> int {
        b.g.entry = (int)ep;
        b.g.entry_level = ep >= 0 ? levels[(size_t)ep] : -1;
        b.B = B;
        v.list = d_list;
        const int grid_ins = (int)std::min<int64_t>((B + HN_WARPS - 1) / HN_WARPS, max_grid_ins);
        int flags[3] = {0, 0, 0};
        for (int attempt = 0;; ++attempt) {
            const uint32_t vis_upper = std::max<uint32_t>(2048u, cap / 8);
            const uint32_t vis_cap = cap + vis_upper;
            VB_TRY(reserve_vis(vis_cap));
            VB_CUDA(cudaMemsetAsync(d_flags, 0, 3 * sizeof(int), s));
            VB_TRY(K.insert(b, v, h.vis, vis_cap, vis_upper, grid_ins, v.wk ? smem_glob : smem_ins, nullptr));
            VB_CUDA(cudaMemcpyAsync(flags, d_flags, 3 * sizeof(int), cudaMemcpyDeviceToHost, s));
            VB_CUDA(cudaStreamSynchronize(s));
            if (flags[2]) {
                // a repair's R overflowed: repeat the batch's searches with R in global memory, four times as large (nothing
                // was published)
                VB_REQUIRE(v.wcap < 65535, "hnsw vacuum: a repair keeps more than 65535 candidates");
                VB_TRY(global_r((int)std::min<int64_t>(65535, (int64_t)v.wcap * 4)));
                continue;
            }
            if (!flags[1]) break;
            cap <<= 2;   // a visited table overflowed: repeat the batch's searches with larger ones (nothing was published)
            VB_REQUIRE(attempt < 8 && cap <= (1u << 26), "hnsw vacuum: visited set overflow");
        }
        hnsw_vacuum_edges_kernel<<<(unsigned)std::min<int64_t>(((int64_t)B * 32 + 127) / 128, (int64_t)c.sm_count * 16), 128, 0, s>>>(b, v);
        VB_CUDA(cudaGetLastError());
        hnsw_vacuum_publish_kernel<<<(unsigned)B, 64, 0, s>>>(b, v);
        VB_CUDA(cudaGetLastError());
        count_launch(2);
        int n_edges = 0;
        VB_CUDA(cudaMemcpyAsync(&n_edges, b.n_edges, sizeof(int), cudaMemcpyDeviceToHost, s));
        VB_CUDA(cudaStreamSynchronize(s));
        VB_REQUIRE(n_edges <= max_edges, "hnsw vacuum: record overflow (%d > %lld)", n_edges, (long long)max_edges);
        if (n_edges > 0) {
            size_t tb = tmp_bytes;
            VB_CUDA(cub::DeviceRadixSort::SortPairs(d_tmp, tb, (const uint64_t*)d_k1, (uint64_t*)d_k2, (const float*)d_v1, (float*)d_v2,
                                                    n_edges, 0, 57, s));
            count_launch();
            const int grid_upd = (int)std::min<int64_t>(((int64_t)n_edges + HN_WARPS - 1) / HN_WARPS, max_grid_upd);
            VB_TRY(K.update(b, v, (const uint64_t*)d_k2, (const float*)d_v2, n_edges, InsertRec{}, grid_upd, smem_upd, nullptr));
        }
        nrep += B;
        return VB_OK;
    };
    auto repair_one = [&](int64_t e, int64_t ep) -> int {
        const int32_t e32 = (int32_t)e;
        VB_CUDA(cudaMemcpyAsync(d_sel, &e32, sizeof(int32_t), cudaMemcpyHostToDevice, s));
        return repair((const int32_t*)d_sel, 1, ep);
    };
    auto needs_one = [&](int64_t e, bool* out) -> int {
        VB_TRY(needs(e, -1));
        uint8_t f = 0;
        VB_CUDA(cudaMemcpyAsync(&f, d_need, 1, cudaMemcpyDeviceToHost, s));
        VB_CUDA(cudaStreamSynchronize(s));
        *out = f != 0;
        return VB_OK;
    };
    int rc = VB_OK;
    auto run = [&]() -> int {
        // RemoveHeapTids' highest and fallback points (src/hnswvacuum.c:133-157): live, the first of a strictly higher level
        int64_t highest = -1, fallback = -1;
        int hl = -1, fl = -1;
        for (int64_t i = 0; i < n; ++i) {
            if (counts[i] == 0) continue;
            const int lv = levels[(size_t)i];
            if (lv > hl) {
                fallback = highest;
                fl = hl;
                highest = i;
                hl = lv;
            } else if (lv > fl) {
                fallback = i;
                fl = lv;
            }
        }
        // RepairGraphEntryPoint (:279-373)
        if (highest >= 0) {
            if (highest == h.entry) highest = fallback;
            bool need = false;
            if (highest >= 0) VB_TRY(needs_one(highest, &need));
            if (need) VB_TRY(repair_one(highest, h.entry));
        }
        if (h.entry >= 0) {
            if (counts[h.entry] == 0) {
                h.entry = highest;
                h.entry_level = highest >= 0 ? levels[(size_t)highest] : -1;
            } else {
                bool need = false;
                VB_TRY(needs_one(h.entry, &need));
                if (need) VB_TRY(repair_one(h.entry, highest));
            }
        }
        // the entry point is the highest live element, so RepairGraph never moves it (:461-482)
        VB_REQUIRE(h.entry < 0 ? live == 0 : (counts[h.entry] != 0 && h.entry_level == hl),
                   "hnsw vacuum: the entry point (%lld, level %d) is not the highest live element (level %d)", (long long)h.entry,
                   h.entry_level, hl);
        // RepairGraph (:378-502): batches of the candidates in element order, NeedsUpdated at each batch's start
        int64_t from = 0;
        while (h.entry >= 0 && from < n) {
            VB_TRY(needs(from, (int)h.entry));
            size_t tb = tmp_bytes;
            VB_CUDA(cub::DeviceSelect::Flagged(d_tmp, tb, cub::CountingInputIterator<int32_t>((int32_t)from), (const uint8_t*)d_need,
                                               (int32_t*)d_sel, d_nsel, (int)(n - from), s));
            count_launch();
            int nsel = 0;
            VB_CUDA(cudaMemcpyAsync(&nsel, d_nsel, sizeof(int), cudaMemcpyDeviceToHost, s));
            VB_CUDA(cudaStreamSynchronize(s));
            if (nsel == 0) break;
            const int B = (int)std::min<int64_t>(nsel, b_max);
            int32_t last = 0;
            VB_CUDA(cudaMemcpyAsync(&last, (const int32_t*)d_sel + (B - 1), sizeof(int32_t), cudaMemcpyDeviceToHost, s));
            VB_TRY(repair((const int32_t*)d_sel, B, h.entry));
            from = B < nsel ? (int64_t)last + 1 : n;
        }
        // MarkDeleted (:594-729)
        hnsw_mark_deleted_kernel<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(b, h.n_heaptids);
        VB_CUDA(cudaGetLastError());
        count_launch();
        // change records: the slots that differ from the snapshot, sorted by (element, layer, slot)
        const InsertRec rec{(uint64_t*)d_k2, (int32_t*)d_v2, d_nsel};
        VB_CUDA(cudaMemsetAsync(d_nsel, 0, sizeof(int), s));
        hnsw_slot_diff_kernel<<<(unsigned)((n + 127) / 128), 128, 0, s>>>(b.g, (const int32_t*)d_old0, (const int32_t*)d_oldup, rec);
        VB_CUDA(cudaGetLastError());
        count_launch();
        int n_rec = 0;
        VB_CUDA(cudaMemcpyAsync(&n_rec, d_nsel, sizeof(int), cudaMemcpyDeviceToHost, s));
        VB_CUDA(cudaStreamSynchronize(s));
        if (n_rec > 0) {
            size_t tb = tmp_bytes;
            VB_CUDA(cub::DeviceRadixSort::SortPairs(d_tmp, tb, (const uint64_t*)d_k2, h.rec_key, (const int32_t*)d_v2, h.rec_val, n_rec, 0, 45,
                                                    s));
            count_launch();
        }
        VB_CUDA(cudaStreamSynchronize(s));
        h.n_changes = n_rec;
        if (out_nchanges) *out_nchanges = n_rec;
        if (out_nrepaired) *out_nrepaired = nrep;
        return VB_OK;
    };
    rc = run();
    if (wbuf) {
        cudaStreamSynchronize(s);
        cudaFree(wbuf);
    }
    return rc;
}

}  // namespace vb

using namespace vb;

extern "C" {

int vb_hnsw_build(vb_hnsw* p, const void* rows, int64_t n, int ef_construction, uint64_t seed, const int32_t* levels) {
    VB_TRY(require_init());
    VB_REQUIRE(p, "null index");
    return hnsw_build_impl(p->h, rows, true, n, ef_construction, seed, levels);
}

int vb_hnsw_build_dev(vb_hnsw* p, const void* rows_dev, int64_t n, int ef_construction, uint64_t seed, const int32_t* levels) {
    VB_TRY(require_init());
    VB_REQUIRE(p, "null index");
    return hnsw_build_impl(p->h, rows_dev, false, n, ef_construction, seed, levels);
}

int vb_hnsw_insert(vb_hnsw* p, const void* rows, int64_t n, int ef_construction, uint64_t seed, const int32_t* levels, int32_t* out_dup_of,
                   int64_t* out_nchanges) {
    VB_TRY(require_init());
    VB_REQUIRE(p, "null index");
    return hnsw_insert_impl(p->h, rows, true, n, ef_construction, seed, levels, out_dup_of, out_nchanges);
}

int vb_hnsw_insert_dev(vb_hnsw* p, const void* rows_dev, int64_t n, int ef_construction, uint64_t seed, const int32_t* levels,
                       int32_t* out_dup_of, int64_t* out_nchanges) {
    VB_TRY(require_init());
    VB_REQUIRE(p, "null index");
    return hnsw_insert_impl(p->h, rows_dev, false, n, ef_construction, seed, levels, out_dup_of, out_nchanges);
}

int vb_hnsw_insert_changes(vb_hnsw* p, vb_hnsw_slot* out, int64_t cap) {
    VB_TRY(require_init());
    VB_REQUIRE(p && p->h.loaded, "hnsw index not loaded");
    const Hnsw& h = p->h;
    const int64_t nc = h.n_changes;
    VB_REQUIRE(cap >= nc, "vb_hnsw_insert_changes: cap %lld is smaller than the %lld change records", (long long)cap, (long long)nc);
    VB_REQUIRE(out || nc == 0, "vb_hnsw_insert_changes: null output");
    if (nc == 0) return VB_OK;
    std::vector<uint64_t> k((size_t)nc);
    std::vector<int32_t> v((size_t)nc);
    cudaStream_t s = ctx().stream;
    VB_CUDA(cudaMemcpyAsync(k.data(), h.rec_key, sizeof(uint64_t) * (size_t)nc, cudaMemcpyDeviceToHost, s));
    VB_CUDA(cudaMemcpyAsync(v.data(), h.rec_val, sizeof(int32_t) * (size_t)nc, cudaMemcpyDeviceToHost, s));
    VB_CUDA(cudaStreamSynchronize(s));
    for (int64_t i = 0; i < nc; ++i) {
        out[i].element = (int32_t)(k[(size_t)i] >> 14);
        out[i].layer = (int32_t)((k[(size_t)i] >> 8) & 63);
        out[i].slot = (int32_t)(k[(size_t)i] & 255);
        out[i].neighbor = v[(size_t)i];
    }
    return VB_OK;
}

int vb_hnsw_vacuum(vb_hnsw* p, const int32_t* counts, int ef_construction, int64_t* out_nrepaired, int64_t* out_nchanges) {
    VB_TRY(require_init());
    VB_REQUIRE(p, "null index");
    return hnsw_vacuum_impl(p->h, counts, ef_construction, out_nrepaired, out_nchanges);
}

int vb_hnsw_set_heaptid_counts(vb_hnsw* p, const int32_t* counts) {
    VB_TRY(require_init());
    VB_REQUIRE(p && p->h.loaded, "hnsw index not loaded");
    Hnsw& h = p->h;
    VB_REQUIRE(counts || h.n == 0, "null counts");
    for (int64_t i = 0; i < h.n; ++i)
        VB_REQUIRE(counts[i] >= 0 && counts[i] <= 10, "vb_hnsw_set_heaptid_counts: counts[%lld] = %d is not in 0..10 (HNSW_HEAPTIDS, src/hnsw.h:69)",
                   (long long)i, counts[i]);
    if (h.n == 0) return VB_OK;
    VB_TRY(hnsw_ensure_counts(h));
    VB_CUDA(cudaMemcpy(h.n_heaptids, counts, sizeof(int32_t) * (size_t)h.n, cudaMemcpyHostToDevice));
    return VB_OK;
}

int64_t vb_hnsw_rows(const vb_hnsw* p) { return p ? p->h.n : 0; }
int64_t vb_hnsw_upper_slots(const vb_hnsw* p) { return p ? p->h.upper_slots : 0; }

int vb_hnsw_export(vb_hnsw* p, int32_t* levels, int32_t* nbr0, int64_t* upper_off, int32_t* upper, int64_t* entry, int32_t* dup_of) {
    VB_TRY(require_init());
    VB_REQUIRE(p && p->h.loaded, "hnsw index not loaded");
    Hnsw& h = p->h;
    const int64_t n = h.n;
    cudaStream_t s = ctx().stream;
    if (entry) *entry = h.entry;
    if (n == 0) return VB_OK;
    if (levels) VB_CUDA(cudaMemcpyAsync(levels, h.levels, sizeof(int32_t) * (size_t)n, cudaMemcpyDeviceToHost, s));
    if (nbr0) VB_CUDA(cudaMemcpyAsync(nbr0, h.nbr0, sizeof(int32_t) * (size_t)n * 2 * h.m, cudaMemcpyDeviceToHost, s));
    if (upper && h.upper_slots > 0)
        VB_CUDA(cudaMemcpyAsync(upper, h.upper, sizeof(int32_t) * (size_t)h.upper_slots * h.m, cudaMemcpyDeviceToHost, s));
    std::vector<int32_t> uo;
    if (upper_off) {
        uo.resize((size_t)n);
        VB_CUDA(cudaMemcpyAsync(uo.data(), h.upper_off, sizeof(int32_t) * (size_t)n, cudaMemcpyDeviceToHost, s));
    }
    if (dup_of) {
        if (h.dup_of) VB_CUDA(cudaMemcpyAsync(dup_of, h.dup_of, sizeof(int32_t) * (size_t)n, cudaMemcpyDeviceToHost, s));
        else
            for (int64_t i = 0; i < n; ++i) dup_of[i] = -1;
    }
    VB_CUDA(cudaStreamSynchronize(s));
    if (upper_off)
        for (int64_t i = 0; i < n; ++i) upper_off[i] = uo[(size_t)i];
    return VB_OK;
}

}  // extern "C"
