// vb_list_tc.cu -- the batched IVFFlat list scan on the tensor cores, as a FILTER in front of the exact
// fp32 arithmetic.
//
// GetScanItems (src/ivfscan.c:124-180) needs, per query, the k nearest of ~probes * rows/lists candidates.
// The list-major formulation (vb_list_tile.cu) already reads every probed list once per batch; what is left
// is 2 fp32 instructions per (row, query, dimension).  Here that arithmetic moves to the tensor cores (wgmma):
//
//   1. approximate pass:  d~ = |x|^2 + |q|^2 - 2 x.q   (or -x.q), x.q from three bf16 MMAs on the hi/lo split of
//      both operands (hi.hi + hi.lo + lo.hi, fp32 accumulation in registers) -- |d~ - d| <= eps(q), a rigorous bound;
//   2. the k' = k + slack smallest d~ of every query are selected (segment_topk_kernel);
//   3. of those, the candidates with d~ <= (k-th d~) + 2 eps are re-scored with the exact scan arithmetic (Acc<>,
//      same as scan_kernel) -- nothing above that threshold can be among the k nearest;
//   4. the k nearest by (exact distance, position) are emitted, and the query is CERTIFIED when the k'-th d~ is
//      itself above the threshold (then so is every candidate that was not selected), i.e. the result equals the
//      full exact scan.  A batch with an uncertified query is re-run on the exact kernel.
//
// Layout.  The index rows are packed once per load into bf16 hi/lo planes in the 128-byte-swizzled shared-memory
// image, one 32 KB block per (128-row table tile, 64-dimension block); a unit of work is a (list, table tile)
// pair (tiles straddling a list boundary are visited by both lists, rows outside the list masked).  The queries
// of each list's group are gathered and packed per batch into 64-query B tiles (16 KB per dimension block).
// CTA = persistent, one per SM: warps 0-7 = two consumer warpgroups (64 table rows each: MMAs, then the epilogue
// on the register accumulators), warp 8 = bulk-copy producer.  The query operand of a tile is ONE shared-memory tile
// [q_hi ; q_lo] of 2n rows (n = 32 or 64): x_hi . [q_hi ; q_lo] is a single wgmma 64 x 2n x 16 per K step whose two
// column groups the epilogue adds; level 2 adds x_lo . q_hi (64 x n x 16).
//
// Two filter levels.  Level 1 streams only the hi plane of the rows (16 KB + B per stage, 7 stages in flight): half
// the HBM traffic, error bound 2^-7 |x||q|.  A batch with an uncertified query is repeated at level 2 (both planes,
// 4 x 48 KB stages, bound 2^-12 |x||q|), and only then on the exact kernel; after a level-1 failure the level rests
// for 64 batches (whether it certifies is a property of the data, not of the batch).
//
// Roofline: HBM -- one pass over the packed hi planes (level 1: 2 bytes per row element) or both planes (level 2:
// 4 bytes) of the probed lists per batch.
#include "vb_tc.cuh"
#include "vb_slab_select.cuh"
#include "vb_distance.cuh"

#include <algorithm>
#include <cmath>
#include <cstring>
#include <vector>

namespace vb {

constexpr int LC_M = 128;
constexpr int LC_N = 64;
constexpr int LC_STAGES = 4;                             // level 2: 4 x 48 KB in flight per SM
constexpr int LC_STAGES_L1 = 7;                          // level 1: 7 x 32 KB (A hi plane + B)
constexpr int LC_MAX_STAGES = 8;
constexpr int LC_CONSUMERS = 256;                       // two warpgroups: rows 0-63 and 64-127 of the table tile
constexpr int LC_THREADS = LC_CONSUMERS + 32;            // + the producer warp
constexpr uint32_t LC_A_PLANE = LC_M * TC_K * 2;        // 16 KB
constexpr uint32_t LC_B_PLANE = LC_N * TC_K * 2;        // 8 KB
constexpr uint32_t LC_A_STAGE = 2 * LC_A_PLANE;
constexpr uint32_t LC_B_STAGE = 2 * LC_B_PLANE;
constexpr uint32_t LC_STAGE = LC_A_STAGE + LC_B_STAGE;  // 48 KB
constexpr uint32_t LC_STAGE_L1 = LC_A_PLANE + LC_B_STAGE;  // 32 KB
constexpr size_t LC_SMEM = std::max((size_t)LC_STAGES * LC_STAGE, (size_t)LC_STAGES_L1 * LC_STAGE_L1) + 1024 /*align*/ + 256 /*barriers*/ +
                           4 * LC_N * sizeof(float) /*slab minima*/;
constexpr int LC_MAX_KP = 128;                           // candidates selected per query, at most

struct LcArgs {
    const uint8_t* A;          // table planes [tile][kb][2][128 x 64]
    const uint8_t* B;          // query-group planes [gtile][kb][2][64 x 64]
    const ListUnit* units;
    int n_units;
    const int64_t* list_off;
    const int32_t* grp_begin;
    const int32_t* grp_cnt;
    const int32_t* gt_begin;
    const int32_t* pair_q;
    const int64_t* pair_out;
    const float* xn;           // |x|^2 per table row
    const float* qn;           // |q|^2 per query of the batch
    float* out;
    float* smin;               // slab minima (slab_base(), vb_common.cuh) or nullptr
    const int32_t* pair_sbase;
    int n_kblocks;
    int is_l2;
    int hi_only;               // level 1: only the hi plane of the rows is read and multiplied (x_hi . (q_hi + q_lo))
    int uniform_nqt;           // > 0: every unit has this many query tiles and a job is one (unit, query tile) pair --
                               // the centre scan, where ONE "list" (the centre table) is probed by every query
    int n_jobs;
};

struct LcJob {
    ListUnit un;
    int cnt, q_lo, q_hi;
};
// job j of the static round-robin: a (list, table tile) unit with all its query tiles, or one query tile of it
__device__ __forceinline__ bool lc_job(const LcArgs& a, int j, LcJob& jb) {
    jb.un = a.units[a.uniform_nqt ? j / a.uniform_nqt : j];
    jb.cnt = a.grp_cnt[jb.un.list];
    if (jb.cnt == 0) return false;
    const int nqt = (jb.cnt + LC_N - 1) / LC_N;
    jb.q_lo = a.uniform_nqt ? j % a.uniform_nqt : 0;
    jb.q_hi = a.uniform_nqt ? min(jb.q_lo + 1, nqt) : nqt;
    return jb.q_lo < jb.q_hi;
}

// One (unit, query tile) for one consumer warpgroup: the MMAs of all K blocks, then the epilogue.  NQ = queries per
// column group; the accumulator holds the 64 x 2 NQ product x . [q_hi ; q_lo] (NQ registers), whose column groups
// [0, NQ) and [NQ, 2 NQ) are added -- register i + NQ / 2 holds column c + NQ of register i's column c.
template <int NQ>
__device__ __forceinline__ void lc_tile(const LcArgs& a, uint8_t* smem, int n_stages, uint32_t stage_bytes, uint32_t a_bytes,
                                        uint64_t* full_bar, uint64_t* empty_bar, float* slab_buf, uint32_t& it, const LcJob& jb,
                                        int qt) {
    const int warp = threadIdx.x / 32, lane = threadIdx.x % 32;
    const int wg = warp / 4, t = threadIdx.x % 128;
    float acc[NQ];
    for (int kb = 0; kb < a.n_kblocks; ++kb, ++it) {
        const int s = it % n_stages;
        const uint32_t ph = (it / n_stages) & 1;
        mbar_wait(&full_bar[s], ph);
        const uint32_t sa = smem_u32(smem + (size_t)s * stage_bytes) + (uint32_t)wg * (64 * 128);
        const uint32_t sb = smem_u32(smem + (size_t)s * stage_bytes) + a_bytes;
        const uint64_t da_hi = make_sw128_desc(sa), da_lo = make_sw128_desc(sa + LC_A_PLANE);
        const uint64_t db = make_sw128_desc(sb);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < TC_K / 16; ++k) {
            const uint64_t adv = (uint64_t)((k * 16 * 2) >> 4);
            // wgmma of different shapes accumulating into the same registers are ordered by a fence between them
            if constexpr (NQ == 64) {
                wgmma_bf16_n128(acc, da_hi + adv, db + adv, (kb | k) != 0);
                if (!a.hi_only) {
                    wgmma_fence();
                    wgmma_bf16_n64(acc, da_lo + adv, db + adv, 1);
                }
            } else {
                wgmma_bf16_n64(acc, da_hi + adv, db + adv, (kb | k) != 0);
                if (!a.hi_only) {
                    wgmma_fence();
                    wgmma_bf16_n32(acc, da_lo + adv, db + adv, 1);
                }
            }
            if (!a.hi_only && k + 1 < TC_K / 16) wgmma_fence();   // the next K step returns to the wider shape
        }
        wgmma_commit();
        wgmma_wait<0>();
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty_bar[s]);
    }

    // ===== epilogue: rows of the table tile x queries of the group =====
    const ListUnit un = jb.un;
    const int cnt = jb.cnt;
    const int64_t lo = a.list_off[un.list], hi = a.list_off[un.list + 1];
    const int frag_row = wg * 64 + 16 * (t / 32) + (t % 32) / 4;   // and frag_row + 8
    const int frag_col = 2 * (t % 4);
    int64_t r_table[2];
    bool valid_row[2];
    float xnr[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        r_table[h] = (int64_t)un.tile * LC_M + frag_row + 8 * h;
        valid_row[h] = r_table[h] >= lo && r_table[h] < hi;
        xnr[h] = valid_row[h] && a.is_l2 ? a.xn[r_table[h]] : 0.f;
    }
    const int gb = a.grp_begin[un.list];
    // warps 2p and 2p + 1 hold the 32 rows of table-aligned slab p of the tile (if any of them belongs to the list)
    const int pair = warp / 2;
    const int64_t slab_row0 = (int64_t)un.tile * LC_M + pair * 32;
    const bool slabs = a.smin != nullptr && slab_row0 < hi && slab_row0 + 32 > lo;
    const int slab_local = (int)((slab_row0 >> 5) - (lo >> 5));
    float col_min[NQ / 4];
#pragma unroll
    for (int cb = 0; cb < NQ / 8; ++cb)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
            const int col = qt * LC_N + 8 * cb + frag_col + e;
            int64_t po = 0;
            float qn = 0.f;
            if (col < cnt) {
                po = a.pair_out[gb + col];
                if (a.is_l2) qn = a.qn[a.pair_q[gb + col]];
            }
            float m = __int_as_float(0x7F800000);
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int i = 4 * cb + 2 * h + e;
                if (col < cnt && valid_row[h]) {
                    const float dot = acc[i] + acc[i + NQ / 2];
                    const float val = a.is_l2 ? fmaf(-2.f, dot, xnr[h] + qn) : -dot;
                    a.out[po + (r_table[h] - lo)] = val;
                    m = fminf(m, val);
                }
            }
            col_min[2 * cb + e] = m;
        }
    if (slabs) {
        // minimum of each column over the slab's 32 rows: over the 16 rows of this warp (lanes of equal t % 4), then
        // the odd warp of the pair hands its minima to the even one
#pragma unroll
        for (int j = 0; j < NQ / 4; ++j)
#pragma unroll
            for (int o = 4; o < 32; o <<= 1) col_min[j] = fminf(col_min[j], __shfl_xor_sync(0xffffffffu, col_min[j], o));
        float* buf = slab_buf + pair * LC_N;
        if ((warp & 1) && lane < 4) {
#pragma unroll
            for (int j = 0; j < NQ / 4; ++j) buf[8 * (j / 2) + frag_col + (j % 2)] = col_min[j];
        }
        named_bar_sync(1 + pair, 64);
        if (!(warp & 1) && lane < 4) {
#pragma unroll
            for (int j = 0; j < NQ / 4; ++j) {
                const int c = 8 * (j / 2) + frag_col + (j % 2);
                const int col = qt * LC_N + c;
                if (col < cnt) a.smin[a.pair_sbase[gb + col] + slab_local] = fminf(col_min[j], buf[c]);
            }
        }
        named_bar_sync(1 + pair, 64);   // buf is rewritten by the next tile
    }
}

__device__ __forceinline__ void list_tc_body(const LcArgs& a) {
    extern __shared__ uint8_t lc_smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(lc_smem_raw) + 1023) & ~(uintptr_t)1023);
    // stage ring: level 2 = 4 stages of (A hi+lo 32 KB | B 16 KB), level 1 = 7 stages of (A hi 16 KB | B 16 KB) --
    // the bytes in flight per SM are what keeps HBM busy
    const int n_stages = a.hi_only ? LC_STAGES_L1 : LC_STAGES;
    const uint32_t stage_bytes = a.hi_only ? LC_STAGE_L1 : LC_STAGE;
    const uint32_t a_bytes = a.hi_only ? LC_A_PLANE : LC_A_STAGE;   // the hi plane leads each 32 KB block of the image
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem + (size_t)n_stages * stage_bytes);
    uint64_t* full_bar = bars;
    uint64_t* empty_bar = bars + LC_MAX_STAGES;
    float* slab_buf = reinterpret_cast<float*>(bars + 32);   // [4 warp pairs][LC_N]

    const int warp = threadIdx.x / 32;
    if (threadIdx.x == 0) {
        for (int s = 0; s < n_stages; ++s) {
            mbar_init(&full_bar[s], 1);
            mbar_init(&empty_bar[s], LC_CONSUMERS / 32);
        }
        fence_barrier_init();
    }
    __syncthreads();

    if (warp == LC_CONSUMERS / 32) {
        // ===== producer (whole warp converged, one elected lane issues the copies) =====
        const bool leader = elect_one();
        uint32_t it = 0;
        for (int j = blockIdx.x; j < a.n_jobs; j += gridDim.x) {
            LcJob jb;
            if (!lc_job(a, j, jb)) continue;
            const ListUnit un = jb.un;
            const int gt0 = a.gt_begin[un.list];
            for (int qt = jb.q_lo; qt < jb.q_hi; ++qt)
            {
                // a query tile with at most 32 queries is multiplied as N = 64: only the first half of each B plane moves
                const bool n32 = jb.cnt - qt * LC_N <= 32;
                for (int kb = 0; kb < a.n_kblocks; ++kb, ++it) {
                    const int s = it % n_stages;
                    const uint32_t ph = (it / n_stages) & 1;
                    mbar_wait(&empty_bar[s], ph ^ 1);
                    uint8_t* sa = smem + (size_t)s * stage_bytes;
                    uint8_t* sb = sa + a_bytes;
                    const uint8_t* gb = a.B + ((size_t)(gt0 + qt) * a.n_kblocks + kb) * LC_B_STAGE;
                    if (leader) {
                        mbar_arrive_expect_tx(&full_bar[s], a_bytes + (n32 ? LC_B_STAGE / 2 : LC_B_STAGE));
                        bulk_g2s(sa, a.A + ((size_t)un.tile * a.n_kblocks + kb) * LC_A_STAGE, a_bytes, &full_bar[s]);
                        if (n32) {   // [q_hi rows 0..31 | q_lo rows 0..31] back to back = one 64-row operand
                            bulk_g2s(sb, gb, LC_B_PLANE / 2, &full_bar[s]);
                            bulk_g2s(sb + LC_B_PLANE / 2, gb + LC_B_PLANE, LC_B_PLANE / 2, &full_bar[s]);
                        } else {
                            bulk_g2s(sb, gb, LC_B_STAGE, &full_bar[s]);
                        }
                    }
                    __syncwarp();
                }
            }
        }
    } else {
        // ===== consumers: warpgroup wg multiplies rows 64 wg .. 64 wg + 63 of the table tile.  The query operand of a
        // tile is ONE shared-memory tile [q_hi ; q_lo] of 2n rows (n = 32 or 64): x_hi . [q_hi ; q_lo] is a single
        // wgmma 64 x 2n x 16 per K step whose two column groups the epilogue adds; level 2 adds x_lo . q_hi (64 x n x 16)
        // into the first group. =====
        uint32_t it = 0;
        for (int j = blockIdx.x; j < a.n_jobs; j += gridDim.x) {
            LcJob jb;
            if (!lc_job(a, j, jb)) continue;
            for (int qt = jb.q_lo; qt < jb.q_hi; ++qt) {
                if (jb.cnt - qt * LC_N <= 32) lc_tile<32>(a, smem, n_stages, stage_bytes, a_bytes, full_bar, empty_bar, slab_buf, it, jb, qt);
                else lc_tile<64>(a, smem, n_stages, stage_bytes, a_bytes, full_bar, empty_bar, slab_buf, it, jb, qt);
            }
        }
    }
}

__global__ void __launch_bounds__(LC_THREADS, 1) list_tc_kernel(LcArgs a) { list_tc_body(a); }

// ----------------------------------------------------------------------------- level 0 (int8)
// a.A = the int8 plane ([tile][128-dimension block][128 rows x 128 B]), a.n_kblocks = its 128-dimension blocks, a.B =
// the [q_hi ; q_lo] int8 query tiles of pack_groups_i8_kernel.  Level 1's ring: 7 stages of 16 KB of rows + the 16 KB
// query tile.  What differs from list_tc_kernel:
//   - the producer tells the consumers which (unit, query tile) a stage starts through a tag beside the stage, so the
//     consumers read no job list;
//   - the consumers release a stage one K block late, behind wgmma_wait<1>: the next block's MMAs are issued before
//     the previous block's finish (the int32 sums are exact, so the order cannot change them);
//   - the epilogue's operands (list bounds, row scales and norms, each column's output offset, slab base, t_q and
//     |q|^2) are loaded while the MMAs of the tile run, one dependent level per K block, each column by one lane of
//     its quad group and shuffled to the others: the epilogue itself waits on no global load.  (It ran after the last
//     K block behind a chain of three dependent loads, with the ring's stages held and no MMA issued.)
struct L0Tag {
    int32_t list, tile, cnt, qt;   // list < 0: no more work
};

template <int NQ>
__device__ __forceinline__ void l0_tile(const LcArgs& a, uint8_t* smem, uint64_t* full_bar, uint64_t* empty_bar, float* slab_buf,
                                        uint32_t& it, const L0Tag tg, const float* __restrict__ xs, const float* __restrict__ tq) {
    const int warp = threadIdx.x / 32, lane = threadIdx.x % 32;
    const int wg = warp / 4, t = threadIdx.x % 128;
    const int qt = tg.qt, cnt = tg.cnt;
    const int frag_row = wg * 64 + 16 * (t / 32) + (t % 32) / 4;   // and frag_row + 8
    const int frag_col = 2 * (t % 4);
    // dependent level 1: the list and its rows
    const int64_t lo = a.list_off[tg.list], hi = a.list_off[tg.list + 1];
    const int gb = a.grp_begin[tg.list];
    int64_t r_table[2];
    float xn_r[2], xs_r[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        r_table[h] = (int64_t)tg.tile * LC_M + frag_row + 8 * h;   // < n_tiles * 128: xn and xs cover the padding
        xn_r[h] = a.is_l2 ? a.xn[r_table[h]] : 0.f;
        xs_r[h] = xs[r_table[h]];
    }
    // lane 4 c + (t % 4) loads columns 8 c + frag_col + {0, 1} of the tile (c < NQ / 8): levels 2 and 3 during the MMAs
    const int my_col = qt * LC_N + 8 * (lane / 4) + frag_col;
    const bool col_ok[2] = {lane / 4 < NQ / 8 && my_col < cnt, lane / 4 < NQ / 8 && my_col + 1 < cnt};
    int64_t po_l[2] = {0, 0};
    int32_t pq_l[2] = {0, 0}, sb_l[2] = {0, 0};
    float qn_l[2] = {0.f, 0.f}, tq_l[2] = {0.f, 0.f};
    int iacc[NQ];
    for (int kb = 0; kb < a.n_kblocks; ++kb, ++it) {
        const int s = it % LC_STAGES_L1;
        if (kb > 0) mbar_wait(&full_bar[s], (it / LC_STAGES_L1) & 1);   // (the first block's was waited for with the tag)
        const uint32_t st = smem_u32(smem + (size_t)s * LC_STAGE_L1);
        const uint64_t da = make_sw128_desc(st + (uint32_t)wg * (64 * 128)), db = make_sw128_desc(st + LC_A_PLANE);
        wgmma_fence();
        // x8 . [q_hi ; q_lo]: four k32 steps over the 128 int8 of the block
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const uint64_t adv = (uint64_t)((k * 32) >> 4);
            if constexpr (NQ == 64) wgmma_s8_n128(iacc, da + adv, db + adv, (kb | k) != 0);
            else wgmma_s8_n64(iacc, da + adv, db + adv, (kb | k) != 0);
        }
        wgmma_commit();
        // at most this block's group is pending: the previous block's stage is free
        wgmma_wait<1>();
        __syncwarp();
        if (kb > 0 && lane == 0) mbar_arrive(&empty_bar[(it + LC_STAGES_L1 - 1) % LC_STAGES_L1]);
        if (kb == 0) {
#pragma unroll
            for (int e = 0; e < 2; ++e)
                if (col_ok[e]) {
                    po_l[e] = a.pair_out[gb + my_col + e];
                    pq_l[e] = a.pair_q[gb + my_col + e];
                    if (a.smin) sb_l[e] = a.pair_sbase[gb + my_col + e];
                }
        }
        if (kb == a.n_kblocks / 2) {
#pragma unroll
            for (int e = 0; e < 2; ++e)
                if (col_ok[e]) {
                    if (a.is_l2) qn_l[e] = a.qn[pq_l[e]];
                    tq_l[e] = tq[pq_l[e]];
                }
        }
    }
    wgmma_wait<0>();
    __syncwarp();
    if (lane == 0) mbar_arrive(&empty_bar[(it + LC_STAGES_L1 - 1) % LC_STAGES_L1]);

    // ===== epilogue: rows of the table tile x queries of the group =====
    bool valid_row[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) valid_row[h] = r_table[h] >= lo && r_table[h] < hi;
    // warps 2p and 2p + 1 hold the 32 rows of table-aligned slab p of the tile (if any of them belongs to the list)
    const int pair = warp / 2;
    const int64_t slab_row0 = (int64_t)tg.tile * LC_M + pair * 32;
    const bool slabs = a.smin != nullptr && slab_row0 < hi && slab_row0 + 32 > lo;
    const int slab_local = (int)((slab_row0 >> 5) - (lo >> 5));
    float col_min[NQ / 4];
#pragma unroll
    for (int cb = 0; cb < NQ / 8; ++cb)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
            const int col = qt * LC_N + 8 * cb + frag_col + e;
            const int src = 4 * cb + (lane & 3);
            const int64_t po = __shfl_sync(0xffffffffu, po_l[e], src);
            const float qn = __shfl_sync(0xffffffffu, qn_l[e], src);
            const float tqc = __shfl_sync(0xffffffffu, tq_l[e], src);
            float m = __int_as_float(0x7F800000);
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int i = 4 * cb + 2 * h + e;
                if (col < cnt && valid_row[h]) {
                    // x^.q^ = s_x t_q (x8.q_hi + x8.q_lo / 254), the roundings bounded in lc_make_bound
                    const float dot = xs_r[h] * (tqc * fmaf((float)iacc[i + NQ / 2], 1.0f / 254.0f, (float)iacc[i]));
                    const float val = a.is_l2 ? fmaf(-2.f, dot, xn_r[h] + qn) : -dot;
                    a.out[po + (r_table[h] - lo)] = val;
                    m = fminf(m, val);
                }
            }
            col_min[2 * cb + e] = m;
        }
    if (slabs) {
        // minimum of each column over the slab's 32 rows: over the 16 rows of this warp (lanes of equal t % 4), then
        // the odd warp of the pair hands its minima to the even one
#pragma unroll
        for (int j = 0; j < NQ / 4; ++j)
#pragma unroll
            for (int o = 4; o < 32; o <<= 1) col_min[j] = fminf(col_min[j], __shfl_xor_sync(0xffffffffu, col_min[j], o));
        float* buf = slab_buf + pair * LC_N;
        if ((warp & 1) && lane < 4) {
#pragma unroll
            for (int j = 0; j < NQ / 4; ++j) buf[8 * (j / 2) + frag_col + (j % 2)] = col_min[j];
        }
        int32_t sb[NQ / 4];
#pragma unroll
        for (int j = 0; j < NQ / 4; ++j) sb[j] = __shfl_sync(0xffffffffu, sb_l[j % 2], 4 * (j / 2) + (lane & 3));
        named_bar_sync(1 + pair, 64);
        if (!(warp & 1) && lane < 4) {
#pragma unroll
            for (int j = 0; j < NQ / 4; ++j) {
                const int c = 8 * (j / 2) + frag_col + (j % 2);
                const int col = qt * LC_N + c;
                if (col < cnt) a.smin[sb[j] + slab_local] = fminf(col_min[j], buf[c]);
            }
        }
        named_bar_sync(1 + pair, 64);   // buf is rewritten by the next tile
    }
}

__global__ void __launch_bounds__(LC_THREADS, 1) list_tc_l0_kernel(LcArgs a, const float* __restrict__ xs, const float* __restrict__ tq) {
    extern __shared__ uint8_t lc_smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(lc_smem_raw) + 1023) & ~(uintptr_t)1023);
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem + (size_t)LC_STAGES_L1 * LC_STAGE_L1);
    uint64_t* full_bar = bars;
    uint64_t* empty_bar = bars + LC_MAX_STAGES;
    L0Tag* tags = reinterpret_cast<L0Tag*>(bars + 2 * LC_MAX_STAGES);   // [LC_MAX_STAGES], the tile of a stage's first K block
    float* slab_buf = reinterpret_cast<float*>(bars + 32);              // [4 warp pairs][LC_N]

    const int warp = threadIdx.x / 32;
    if (threadIdx.x == 0) {
        for (int s = 0; s < LC_STAGES_L1; ++s) {
            mbar_init(&full_bar[s], 1);
            mbar_init(&empty_bar[s], LC_CONSUMERS / 32);
        }
        fence_barrier_init();
    }
    __syncthreads();

    if (warp == LC_CONSUMERS / 32) {
        // ===== producer (whole warp converged, one elected lane issues the copies), jobs in static round-robin =====
        const bool leader = elect_one();
        uint32_t it = 0;
        for (int j = blockIdx.x; j < a.n_jobs; j += gridDim.x) {
            const ListUnit un = a.units[j];
            const int cnt = a.grp_cnt[un.list];
            const int gt0 = a.gt_begin[un.list];
            const int nqt = (cnt + LC_N - 1) / LC_N;
            for (int qt = 0; qt < nqt; ++qt) {
                // a query tile with at most 32 queries is multiplied as N = 64: only the first half of each B plane moves
                const bool n32 = cnt - qt * LC_N <= 32;
                for (int kb = 0; kb < a.n_kblocks; ++kb, ++it) {
                    const int s = it % LC_STAGES_L1;
                    mbar_wait(&empty_bar[s], ((it / LC_STAGES_L1) & 1) ^ 1);
                    uint8_t* sa = smem + (size_t)s * LC_STAGE_L1;
                    uint8_t* sb = sa + LC_A_PLANE;
                    const uint8_t* gb = a.B + ((size_t)(gt0 + qt) * a.n_kblocks + kb) * LC_B_STAGE;
                    const uint8_t* ga = a.A + ((size_t)un.tile * a.n_kblocks + kb) * LC_A_PLANE;
                    if (leader) {
                        if (kb == 0) tags[s] = L0Tag{un.list, un.tile, cnt, qt};   // published by the arrive below
                        mbar_arrive_expect_tx(&full_bar[s], LC_A_PLANE + (n32 ? LC_B_STAGE / 2 : LC_B_STAGE));
                        bulk_g2s(sa, ga, LC_A_PLANE, &full_bar[s]);
                        if (n32) {   // [q_hi rows 0..31 | q_lo rows 0..31] back to back = one 64-row operand
                            bulk_g2s(sb, gb, LC_B_PLANE / 2, &full_bar[s]);
                            bulk_g2s(sb + LC_B_PLANE / 2, gb + LC_B_PLANE, LC_B_PLANE / 2, &full_bar[s]);
                        } else {
                            bulk_g2s(sb, gb, LC_B_STAGE, &full_bar[s]);
                        }
                    }
                    __syncwarp();
                }
            }
        }
        // the end of the work: a tag with no copies behind it
        const int s = it % LC_STAGES_L1;
        mbar_wait(&empty_bar[s], ((it / LC_STAGES_L1) & 1) ^ 1);
        if (leader) {
            tags[s] = L0Tag{-1, 0, 0, 0};
            mbar_arrive(&full_bar[s]);
        }
        __syncwarp();
    } else {
        // ===== consumers: warpgroup wg multiplies rows 64 wg .. 64 wg + 63 of the table tile =====
        uint32_t it = 0;
        for (;;) {
            const int s = it % LC_STAGES_L1;
            mbar_wait(&full_bar[s], (it / LC_STAGES_L1) & 1);
            const L0Tag tg = tags[s];
            if (tg.list < 0) break;
            if (tg.cnt - tg.qt * LC_N <= 32) l0_tile<32>(a, smem, full_bar, empty_bar, slab_buf, it, tg, xs, tq);
            else l0_tile<64>(a, smem, full_bar, empty_bar, slab_buf, it, tg, xs, tq);
        }
    }
}

// gather + split the queries of every (query, list) pair into the B tiles of its list's group:
// thread = one 16-byte chunk (8 dimensions) of one pair
__global__ void pack_groups_kernel(const float* __restrict__ qimg, size_t qstride, int dim, int n_kblocks, int64_t n_pairs,
                                   const int32_t* __restrict__ pair_q, const int32_t* __restrict__ pair_list,
                                   const int32_t* __restrict__ grp_begin, const int32_t* __restrict__ gt_begin,
                                   uint8_t* __restrict__ out) {
    const int64_t chunk = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    const int chunks_per_row = n_kblocks * 8;
    const int64_t slot = chunk / chunks_per_row;
    if (slot >= n_pairs) return;
    const int cr = (int)(chunk % chunks_per_row);
    const int kb = cr / 8, c = cr % 8;
    const int l = pair_list[slot];
    const int j = (int)(slot - grp_begin[l]);
    const int64_t gtile = gt_begin[l] + j / LC_N;
    const int r = j % LC_N;
    const float* src = reinterpret_cast<const float*>(reinterpret_cast<const uint8_t*>(qimg) + (size_t)pair_q[slot] * qstride);
    const int e0 = kb * TC_K + c * 8;
    float v[8];
#pragma unroll
    for (int t = 0; t < 8; ++t) v[t] = e0 + t < dim ? src[e0 + t] : 0.f;
    uint32_t hi[4], lo[4];
#pragma unroll
    for (int t = 0; t < 4; ++t) {
        __nv_bfloat16 h0 = __float2bfloat16_rn(v[2 * t]), h1 = __float2bfloat16_rn(v[2 * t + 1]);
        __nv_bfloat16 l0 = __float2bfloat16_rn(v[2 * t] - __bfloat162float(h0));
        __nv_bfloat16 l1 = __float2bfloat16_rn(v[2 * t + 1] - __bfloat162float(h1));
        hi[t] = (uint32_t)__bfloat16_as_ushort(h0) | ((uint32_t)__bfloat16_as_ushort(h1) << 16);
        lo[t] = (uint32_t)__bfloat16_as_ushort(l0) | ((uint32_t)__bfloat16_as_ushort(l1) << 16);
    }
    uint8_t* base = out + ((size_t)(gtile * n_kblocks + kb) * 2) * LC_B_PLANE;
    const size_t off = (size_t)r * 128 + (size_t)((c ^ (r & 7)) * 16);
    *reinterpret_cast<uint4*>(base + off) = make_uint4(hi[0], hi[1], hi[2], hi[3]);
    *reinterpret_cast<uint4*>(base + LC_B_PLANE + off) = make_uint4(lo[0], lo[1], lo[2], lo[3]);
}


// ---- level 0: int8 rows and queries ----------------------------------------------------------------------------------
//
// Rows: x ~ s_x x8 with s_x = max |x_i| / 127 and x8 = rint(x / s_x) (per-row absmax).  Queries: q ~ t_q (q_hi + q_lo / 254)
// with t_q = max |q_i| / 127, q_hi = rint(q / t_q) and q_lo = rint((q - t_q q_hi) 254 / t_q), both in [-127, 127].  x8 . q_hi
// and x8 . q_lo are ONE wgmma m64 n(2n) k32 s8 per K step, exact in int32 (|x8 . q| <= 127^2 dim < 2^31 for dim < 133000).

// one query coordinate; the packing and the bound kernel call the same function, so the bound is computed from exactly
// the values the tensor cores multiply
__device__ __forceinline__ void l0_quant_q(float v, float tq, int& hi, int& lo) {
    if (!(tq > 0.f && tq < 3.0e38f)) {
        hi = lo = 0;
        return;
    }
    const float h = fminf(fmaxf(rintf(__fdiv_rn(v, tq)), -127.f), 127.f);
    const float r = fmaf(-tq, h, v);
    const float l = fminf(fmaxf(rintf(__fdiv_rn(r * 254.f, tq)), -127.f), 127.f);
    hi = (int)h;
    lo = (int)l;
}

// rows -> int8 plane [tile][128-dim block][128 rows x 128 B] (128-byte swizzle: byte (r, kk) at r * 128 +
// ((kk / 16) ^ (r & 7)) * 16 + kk % 16), s_x per row, |x - s_x x8| per row (rounded up; 0 on padding rows) and its max
// over the rows (as float bits): one warp per row of the tile-padded table
template <int ELEM>
__global__ void pack_rows_i8_kernel(const uint8_t* __restrict__ rows, size_t stride, int64_t n, int dim, int n_kblocks8, int64_t n_padded,
                                    uint8_t* __restrict__ out, float* __restrict__ xs, float* __restrict__ r8,
                                    unsigned* __restrict__ rmax_bits) {
    const int64_t r = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) / 32;
    const int lane = threadIdx.x % 32;
    if (r >= n_padded) return;
    const uint8_t* src = rows + (size_t)std::min<int64_t>(r, n - 1) * stride;
    auto ld = [&](int e) -> float {
        if (r >= n || e >= dim) return 0.f;
        return ELEM == VB_VECTOR ? reinterpret_cast<const float*>(src)[e] : __half2float(reinterpret_cast<const __half*>(src)[e]);
    };
    float amax = 0.f;
    for (int e = lane; e < dim; e += 32) amax = fmaxf(amax, fabsf(ld(e)));
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, o));
    const float sx = amax / 127.f;
    const int64_t tile = r / LC_M;
    const int rr = (int)(r % LC_M);
    double res = 0.0;
    for (int ch = lane; ch < n_kblocks8 * 8; ch += 32) {
        const int kb = ch / 8, c = ch % 8, e0 = kb * 128 + c * 16;
        uint32_t w[4] = {0u, 0u, 0u, 0u};
#pragma unroll
        for (int j = 0; j < 16; ++j) {
            const float v = ld(e0 + j);
            const float x8 = sx > 0.f ? fminf(fmaxf(rintf(__fdiv_rn(v, sx)), -127.f), 127.f) : 0.f;
            const double d = (double)v - (double)sx * (double)x8;
            res += d * d;
            w[j / 4] |= (uint32_t)(uint8_t)(int8_t)(int)x8 << (8 * (j % 4));
        }
        uint8_t* base = out + ((size_t)tile * n_kblocks8 + kb) * LC_A_PLANE;
        *reinterpret_cast<uint4*>(base + (size_t)rr * 128 + (size_t)((c ^ (rr & 7)) * 16)) = make_uint4(w[0], w[1], w[2], w[3]);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) res += __shfl_xor_sync(0xffffffffu, res, o);
    if (lane == 0) {
        xs[r] = sx;
        const float rx = r < n ? __double2float_ru(sqrt(res) * (1.0 + 1.0 / 1048576.0)) : 0.f;
        r8[r] = rx;
        if (r < n) atomicMax(rmax_bits, __float_as_uint(rx));
    }
}

// per query of the batch (one warp each): t_q, the packed query q8 = [q_hi | q_lo] (qpad int8 each, zero past qdim: quantised
// once here, copied into the tiles of every probed list by pack_groups_i8_kernel), and the level-0 bound eps(q) >= |d~ - d_fp32|
// over every row (lc_make_bound derives it), handed to the refine kernels squared, in the place of |q|^2 (qe2), and the
// coefficients (a, b, c, d) of the per-row bound E(x, q) = a R_x + b X_x + c X_x^2 + d (lc_make_bound), rounded up
__global__ void l0_query_kernel(const float* __restrict__ qimg, size_t qstride, int qdim, int qpad, int64_t nq, float xmax, float rmax,
                                int is_l2, float c_sum, float* __restrict__ tq_out, float* __restrict__ qe2_out, float4* __restrict__ coef,
                                int8_t* __restrict__ q8) {
    const int64_t q = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) / 32;
    const int lane = threadIdx.x % 32;
    if (q >= nq) return;
    const float* src = reinterpret_cast<const float*>(reinterpret_cast<const uint8_t*>(qimg) + (size_t)q * qstride);
    float amax = 0.f;
    for (int e = lane; e < qdim; e += 32) amax = fmaxf(amax, fabsf(src[e]));
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, o));
    const float tq = amax / 127.f;
    double n2 = 0.0, r2 = 0.0, h2 = 0.0, l2 = 0.0;
    int8_t* qh = q8 + (size_t)q * 2 * qpad;
    for (int e = qdim + lane; e < qpad; e += 32) qh[e] = qh[qpad + e] = 0;
    for (int e = lane; e < qdim; e += 32) {
        const float v = src[e];
        int hi, lo;
        l0_quant_q(v, tq, hi, lo);
        qh[e] = (int8_t)hi;
        qh[qpad + e] = (int8_t)lo;
        const double d = (double)v - (double)tq * ((double)hi + (double)lo / 254.0);
        n2 += (double)v * v;
        r2 += d * d;
        h2 += (double)hi * hi;
        l2 += (double)lo * lo;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        n2 += __shfl_xor_sync(0xffffffffu, n2, o);
        r2 += __shfl_xor_sync(0xffffffffu, r2, o);
        h2 += __shfl_xor_sync(0xffffffffu, h2, o);
        l2 += __shfl_xor_sync(0xffffffffu, l2, o);
    }
    if (lane == 0) {
        const double X = (double)xmax * (1.0 + 1.0 / 1024.0) + (double)rmax;   // >= |x^| = |s_x x8| of every row
        const double qnorm = sqrt(n2), rq = sqrt(r2), qabs = (double)tq * (sqrt(h2) + sqrt(l2) / 254.0);
        const double dot = (double)rmax * qnorm + X * rq + X * qabs / 1048576.0 + 1e-30;
        double eps = is_l2 ? 2.0 * dot + (double)c_sum * (X * X + n2) : dot + X * qnorm / 131072.0;
        eps *= 1.0 + 1.0 / 1024.0;
        tq_out[q] = tq;
        qe2_out[q] = __double2float_ru(eps * eps);   // NaN / Inf (a query without finite norm): the certificate fails
        // the same sum with R_x and X_x of one row in the place of rmax and X, split by its dependence on the row
        const double w = 1.0 + 1.0 / 1024.0, dq = rq + qabs / 1048576.0;
        const double ca = is_l2 ? 2.0 * qnorm : qnorm;
        const double cb = is_l2 ? 2.0 * dq : dq + qnorm / 131072.0;
        const double cc = is_l2 ? (double)c_sum : 0.0;
        const double cd = is_l2 ? 2e-30 + (double)c_sum * n2 : 1e-30;
        coef[q] = make_float4(__double2float_ru(ca * w), __double2float_ru(cb * w), __double2float_ru(cc * w), __double2float_ru(cd * w));
    }
}

// pack_groups_kernel for level 0: thread = one 16-byte chunk (16 dimensions) of one pair, copied from l0_query_kernel's q8
__global__ void pack_groups_i8_kernel(const int8_t* __restrict__ q8, int qpad, int n_kblocks8, int64_t n_pairs,
                                      const int32_t* __restrict__ pair_q, const int32_t* __restrict__ pair_list,
                                      const int32_t* __restrict__ grp_begin, const int32_t* __restrict__ gt_begin,
                                      uint8_t* __restrict__ out) {
    const int64_t chunk = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    const int chunks_per_row = n_kblocks8 * 8;
    const int64_t slot = chunk / chunks_per_row;
    if (slot >= n_pairs) return;
    const int cr = (int)(chunk % chunks_per_row);
    const int kb = cr / 8, c = cr % 8;
    const int l = pair_list[slot];
    const int j = (int)(slot - grp_begin[l]);
    const int64_t gtile = gt_begin[l] + j / LC_N;
    const int r = j % LC_N;
    const int8_t* src = q8 + (size_t)pair_q[slot] * 2 * qpad + kb * 128 + c * 16;
    uint8_t* base = out + ((size_t)(gtile * n_kblocks8 + kb) * 2) * LC_B_PLANE;
    const size_t off = (size_t)r * 128 + (size_t)((c ^ (r & 7)) * 16);
    *reinterpret_cast<uint4*>(base + off) = *reinterpret_cast<const uint4*>(src);
    *reinterpret_cast<uint4*>(base + LC_B_PLANE + off) = *reinterpret_cast<const uint4*>(src + qpad);
}

// |d~ - d_fp32| <= eps(q) for every candidate of query q
struct LcBound {
    int is_l2;
    float c_dot, c_sum, xmax;
};
__device__ __forceinline__ float lc_eps(const LcBound& b, float qn) {
    return b.c_dot * sqrtf(qn) * b.xmax + (b.is_l2 ? b.c_sum * (b.xmax * b.xmax + qn) : 0.f);
}
// shared memory of cta_refine_body's selection beside its fixed buffers: the slab tables, or a short run's keys
__host__ __device__ inline size_t cr_work_bytes(bool slabs, bool pre, int64_t cap, int64_t cap_s, int probes) {
    return slabs ? ss_select_smem_bytes(cap_s, probes) : pre ? 0 : (size_t)cap * 4;
}
// dynamic shared memory of one cta_refine_body CTA: cand, fin, rowp, the query image, the selection's work area, exact
size_t cta_refine_smem_bytes(int kp, size_t qstride, bool slabs, bool pre, int64_t cap, int64_t cap_s, int probes) {
    return (size_t)SS_CAND * 8 + (size_t)kp * 16 + qstride + cr_work_bytes(slabs, pre, cap, cap_s, probes) + (size_t)kp * 4 + 16;
}

// Steps 2 + 3 + 4 with ONE CTA per query (cta_refine_kernel): the k' nearest by (d~, position) come from one of three
// sources -- a CTA-wide selection from the slab minima (smin), the k' preselected by launch_slab_select /
// launch_segment_topk_v (pre_pos / pre_key [nq][kp], sorted, -1 padded), or an exact selection of the whole run when it
// is short (at most CR_RUN_MAX entries: the distances of a query to every centre).  The candidates under the certificate
// threshold are then re-scored by the CTA's eight warps in parallel (one row per warp at a time), ranked and certified.
// A query whose slab selection overflows its buffer (ties by the thousand) counts as uncertified and the batch is
// repeated with the k' preselected.
//
// LIST (level 0 only): the uncertified queries are also listed, and the re-score uses per-row bounds E_i (lc_make_bound)
// instead of (k-th d~) + 2 eps.  Phase 1 re-scores the k candidates of smallest d~ and sets T to their k-th exact
// distance; phase 2 re-scores every other listed candidate with d~_i - E_i <= T (NaN included).  A candidate left out has
// d >= d~_i - E_i > T, so it is behind k re-scored ones.  The certificate then needs d~_{k'} > T + E_max(q), T the k-th
// exact distance of the re-scored set: every unselected row has d >= d~ - E_max >= d~_{k'} - E_max > T.
//
// MASK (vb_ivf_search_filtered): the run is masked, rejected entries hold FILTER_REJECTED, the slab minima are those of the
// allowed entries, and has_nan[q] says an allowed entry of query q has a NaN d~.  Candidates with a NaN key are then
// rejected ones (such a query counts as uncertified otherwise) and are dropped: `have` counts the allowed candidates.
// Fewer than k' of them means every allowed row of the run is a candidate (a selection of at least k' entries holds a
// rejected one only after every allowed one: the slab selection then took every entry of the run, tau being the key of
// NaN), so the result is complete and needs no certificate.  A run with fewer than k' slabs that hold an allowed row and
// more than SS_CAND entries overflows the slab selection; the query then counts as uncertified, as a tie overflow does.
template <int ELEM, int METRIC, bool LIST, bool MASK = false>
__device__ __forceinline__ void cta_refine_body(const uint8_t* __restrict__ rows, size_t stride, int V,
                                                                const uint8_t* __restrict__ qimg, size_t qstride, int k, int kp, int probes,
                                                                LcBound bound, const float* __restrict__ qn, const float* __restrict__ dist,
                                                                const float* __restrict__ smin, const int32_t* __restrict__ pre_pos,
                                                                const float* __restrict__ pre_key, int64_t cap, int64_t cap_s,
                                                                const int32_t* __restrict__ seg_len, const int32_t* __restrict__ probe_lists,
                                                                const int32_t* __restrict__ cand_off, const int64_t* __restrict__ list_off,
                                                                int32_t* __restrict__ out_pos, float* __restrict__ out_key,
                                                                int* __restrict__ n_failed, int32_t* __restrict__ fail_list,
                                                                const float* __restrict__ xn, const float* __restrict__ r8,
                                                                const float4* __restrict__ coef, unsigned long long* __restrict__ counters,
                                                                const int32_t* __restrict__ has_nan = nullptr) {
    const bool slabs = LIST || smin != nullptr;                                 // (level 0 always has slab minima)
    const bool pre = !LIST && pre_pos != nullptr;
    extern __shared__ uint64_t cr_smem[];
    uint64_t* cand = cr_smem;                                                   // [SS_CAND]
    uint64_t* fin = cand + SS_CAND;                                             // [kp] final keys
    const uint8_t** rowp = reinterpret_cast<const uint8_t**>(fin + kp);         // [kp] row addresses
    uint4* sq = reinterpret_cast<uint4*>(rowp + kp);                            // [qvec] query image (cand, fin and rowp are 16 kp + 16384 bytes: aligned)
    const int qvec = (int)(qstride / 16);
    void* work = sq + qvec;                                                     // the selection's work area (16-byte aligned)
    float* exact = reinterpret_cast<float*>(reinterpret_cast<uint8_t*>(work) + cr_work_bytes(slabs, pre, cap, cap_s, probes));   // [kp]
    const int q = blockIdx.x;
    const int tid = threadIdx.x, warp = tid / 32, lane = tid % 32;
    const uint4* gq = reinterpret_cast<const uint4*>(qimg + (size_t)q * qstride);
    for (int i = tid; i < qvec; i += SS_THREADS) sq[i] = gq[i];
    const int n_run = seg_len[q];
    int n;
    if (pre) {
        // kp <= SS_THREADS: one entry per thread; the -1 padding follows the valid entries
        const int32_t p = tid < kp ? pre_pos[(int64_t)q * kp + tid] : -1;
        if (p >= 0) cand[tid] = ((uint64_t)orderable_key(pre_key[(int64_t)q * kp + tid]) << 32) | (uint32_t)p;
        n = __syncthreads_count(p >= 0);
    } else if (slabs) {
        n = slab_select_cta(dist, smin, probes, probe_lists, cand_off, list_off, cap, cap_s, q, kp, cand, work);
    } else {
        uint32_t* keys = reinterpret_cast<uint32_t*>(work);
        const float* dq = dist + (int64_t)q * cap;
        for (int i = tid; i < n_run; i += SS_THREADS) keys[i] = orderable_key(dq[i]);
        __syncthreads();
        n = select_exact_cta(keys, n_run, kp, cand);
    }
    if (n < 0) {
        // not selected here: the query reports as uncertified (outputs are rewritten by the repeat of the batch)
        if (tid == 0) {
            const int i = atomicAdd(n_failed, 1);
            if (LIST) fail_list[i] = q;
        }
        for (int i = tid; i < k; i += SS_THREADS) {
            out_pos[(int64_t)q * k + i] = -1;
            out_key[(int64_t)q * k + i] = __int_as_float(0x7F800000);
        }
        return;
    }
    int have = min(n, kp);
    if constexpr (MASK) have = __syncthreads_count(tid < have && (cand[tid] >> 32) != 0xFFFFFFFFull);   // (kp <= SS_THREADS; sorted)
    // ---- threshold: (k-th smallest approximate distance) + 2 eps.  Only candidates with d~ under it can belong to the k
    // nearest: the k candidates with the smallest d~ all have d <= (k-th d~) + eps, anything above it has d > (k-th d~) + eps.
    const int kth = min(k, kp) - 1;
    const uint64_t kth_key = kth < have ? cand[kth] : ~0ull;
    const float kth_approx = kth_key == ~0ull ? __int_as_float(0x7F800000) : key_to_float((uint32_t)(kth_key >> 32));
    const float T = kth_approx + 2.f * lc_eps(bound, qn[q]);
    const uint64_t thr = kp - 1 < have ? cand[kp - 1] : ~0ull;                    // the k'-th key
    // ---- row address of every listed candidate (one per thread): position -> probe -> row.  After a slab selection the
    // per-probe candidate offsets and list bounds are in shared memory already.
    const int32_t* co = cand_off + (int64_t)q * (probes + 1);
    const SsWork W = ss_work_layout(work, cap_s, probes);
    // LIST: d~_i - E_i of every listed candidate, in fin's storage until the ranking below
    float* lb = reinterpret_cast<float*>(fin);
    for (int i = tid; i < kp; i += SS_THREADS) {
        exact[i] = __int_as_float(0x7F800000);
        rowp[i] = rows;
        if (i < have) {
            const int32_t ps = (int32_t)(uint32_t)cand[i];
            int64_t g;                                        // row of the (list-ordered) table
            if (slabs) {
                int lo = 0, hi = probes;
                while (hi - lo > 1) {
                    const int mid = (lo + hi) >> 1;
                    if (W.co[mid] <= ps) lo = mid;
                    else hi = mid;
                }
                // (empty lists share an offset with their successor: the search ends on the last of them, the non-empty one)
                g = W.lo[lo] + (ps - W.co[lo]);
            } else {
                int lo = 0, hi = probes;
                while (hi - lo > 1) {
                    const int mid = (lo + hi) >> 1;
                    if (co[mid] <= ps) lo = mid;
                    else hi = mid;
                }
                while (lo + 1 < probes && co[lo + 1] <= ps) ++lo;   // empty lists share an offset
                const int l = probe_lists[(int64_t)q * probes + lo];
                g = list_off[l] + (ps - co[lo]);
            }
            rowp[i] = rows + (size_t)g * stride;
            if (LIST) {
                // E_i = a R_x + b X_x + c X_x^2 + d with X_x = |x| (1 + 2^-10) + R_x, every step rounded up (lc_make_bound)
                const float4 cf = coef[q];
                const float R = r8[g];
                const float X = __fadd_ru(__fmul_ru(__fsqrt_ru(xn[g]), 1.0f + 1.0f / 1024.0f), R);
                const float E = __fmaf_ru(cf.z, __fmul_ru(X, X), __fmaf_ru(cf.y, X, __fmaf_ru(cf.x, R, cf.w)));
                lb[i] = key_to_float((uint32_t)(cand[i] >> 32)) - E;
            }
        }
    }
    __syncthreads();
    auto rescore = [&](int i) {
        const uint4* rp = reinterpret_cast<const uint4*>(rowp[i]);
        Acc<ELEM, METRIC> acc;
#pragma unroll 4
        for (int v = lane; v < V; v += 32) acc.add(__ldg(rp + v), sq, v);
        acc.template reduce<32>();
        if (lane == 0) exact[i] = (float)acc.value();
    };
    __shared__ float s_tk;                                   // LIST: the k-th exact distance of the re-scored set
    if (!LIST) {
        // ---- exact re-score of the candidates with approx <= T (NaN compares false: re-scored too), one row per warp
        for (int i = warp; i < have; i += SS_THREADS / 32) {
            const float a = key_to_float((uint32_t)(cand[i] >> 32));
            if (a > T) continue;                             // warp-uniform
            rescore(i);
        }
    } else {
        // ---- phase 1: the k smallest d~; T1 = the k-th exact distance (+inf when fewer than k, or one is NaN)
        const float inf = __int_as_float(0x7F800000);
        const int kk = min(k, have);
        int n_rs = 0;                                        // rows this warp re-scored
        for (int i = warp; i < kk; i += SS_THREADS / 32, ++n_rs) rescore(i);
        __syncthreads();
        float T1 = kk < k ? inf : -inf;
        for (int i = 0; i < kk && T1 < inf; ++i) T1 = exact[i] == exact[i] ? fmaxf(T1, exact[i]) : inf;
        // ---- phase 2: the others with d~_i - E_i <= T1 (fl(d~_i - E_i) > T1 implies d~_i - E_i > T1: rounding is monotone)
        for (int i = kk + warp; i < have; i += SS_THREADS / 32) {
            if (lb[i] > T1) continue;                        // warp-uniform; NaN is re-scored
            rescore(i);
            ++n_rs;
        }
        if (counters) {
            // profiling: rows re-scored, and the rows the global bound would re-score (d~ <= d~_k + 2 eps(q))
            if (lane == 0) atomicAdd(&counters[0], (unsigned long long)n_rs);
            int n_glob = 0;
            for (int i = tid; i < have; i += SS_THREADS) n_glob += !(key_to_float((uint32_t)(cand[i] >> 32)) > T);
            n_glob = __reduce_add_sync(0xffffffffu, n_glob);
            if (lane == 0) atomicAdd(&counters[1], (unsigned long long)n_glob);
            if (tid == 0) atomicAdd(&counters[2], 1ull);
        }
    }
    __syncthreads();
    // ---- order by (exact distance, position), emit the first k
    for (int i = tid; i < kp; i += SS_THREADS)
        fin[i] = i < have ? (((uint64_t)orderable_key(exact[i]) << 32) | (uint32_t)cand[i]) : (0xFFFFFFFF00000000ull | (uint32_t)i);
    __syncthreads();
    for (int i = tid; i < kp; i += SS_THREADS) {
        const uint64_t mine = fin[i];
        int rank = 0;
        for (int j = 0; j < kp; ++j) rank += fin[j] < mine;
        if (rank < k) {
            const bool present = i < have;
            out_pos[(int64_t)q * k + rank] = present ? (int32_t)(uint32_t)mine : -1;
            out_key[(int64_t)q * k + rank] = present ? key_to_float((uint32_t)(mine >> 32)) : __int_as_float(0x7F800000);
        }
        if (LIST && rank == k - 1) s_tk = key_to_float((uint32_t)(mine >> 32));
    }
    if (LIST) __syncthreads();
    if constexpr (MASK) {
        // ---- certificate of a masked run: only when k' allowed candidates were kept and the run holds more entries
        if (tid == 0) {
            bool ok = has_nan[q] == 0;
            if (ok && have >= kp && n_run > kp) {
                const float Tc = LIST ? __fadd_ru(s_tk, __fsqrt_ru(qn[q])) : T;
                ok = key_to_float((uint32_t)(thr >> 32)) > Tc;
            }
            if (!ok) {
                const int i = atomicAdd(n_failed, 1);
                if (LIST) fail_list[i] = q;
            }
        }
        return;
    }
    // ---- certificate: candidates beyond the k' exist -> the last of the k' must already be above the threshold
    if (tid == 0 && n_run > kp) {
        // (LIST: the threshold T + E_max(q) is rounded up, E_max = eps(q) >= E_i of every row, from its square rounded up)
        const float Tc = LIST ? __fadd_ru(s_tk, __fsqrt_ru(qn[q])) : T;
        const bool ok = key_to_float((uint32_t)(thr >> 32)) > Tc;     // false for NaN
        if (!ok) {
            const int i = atomicAdd(n_failed, 1);
            if (LIST) fail_list[i] = q;
        }
    }
}

template <int ELEM, int METRIC>
__global__ void __launch_bounds__(SS_THREADS) cta_refine_kernel(const uint8_t* __restrict__ rows, size_t stride, int V,
                                                                const uint8_t* __restrict__ qimg, size_t qstride, int k, int kp, int probes,
                                                                LcBound bound, const float* __restrict__ qn, const float* __restrict__ dist,
                                                                const float* __restrict__ smin, const int32_t* __restrict__ pre_pos,
                                                                const float* __restrict__ pre_key, int64_t cap, int64_t cap_s,
                                                                const int32_t* __restrict__ seg_len, const int32_t* __restrict__ probe_lists,
                                                                const int32_t* __restrict__ cand_off, const int64_t* __restrict__ list_off,
                                                                int32_t* __restrict__ out_pos, float* __restrict__ out_key,
                                                                int* __restrict__ n_failed) {
    cta_refine_body<ELEM, METRIC, false>(rows, stride, V, qimg, qstride, k, kp, probes, bound, qn, dist, smin, pre_pos, pre_key, cap, cap_s, seg_len, probe_lists, cand_off, list_off, out_pos, out_key, n_failed, nullptr,
                                         nullptr, nullptr, nullptr, nullptr);
}
// level 0: the per-row re-score rule (xn, r8: the image's |x|^2 and residuals; coef: l0_query_kernel's coefficients;
// counters: profiling, or null), and the uncertified queries listed (fail_list[0 .. *n_failed)), then run again on their own
template <int ELEM, int METRIC>
__global__ void __launch_bounds__(SS_THREADS) cta_refine_list_kernel(const uint8_t* __restrict__ rows, size_t stride, int V,
                                                                const uint8_t* __restrict__ qimg, size_t qstride, int k, int kp, int probes,
                                                                LcBound bound, const float* __restrict__ qn, const float* __restrict__ dist,
                                                                const float* __restrict__ smin, int64_t cap, int64_t cap_s,
                                                                const int32_t* __restrict__ seg_len, const int32_t* __restrict__ probe_lists,
                                                                const int32_t* __restrict__ cand_off, const int64_t* __restrict__ list_off,
                                                                int32_t* __restrict__ out_pos, float* __restrict__ out_key,
                                                                int* __restrict__ n_failed, int32_t* __restrict__ fail_list,
                                                                const float* __restrict__ xn, const float* __restrict__ r8,
                                                                const float4* __restrict__ coef, unsigned long long* __restrict__ counters) {
    cta_refine_body<ELEM, METRIC, true>(rows, stride, V, qimg, qstride, k, kp, probes, bound, qn, dist, smin, nullptr, nullptr, cap, cap_s, seg_len, probe_lists, cand_off, list_off, out_pos, out_key, n_failed, fail_list,
                                        xn, r8, coef, counters);
}
// the two above over masked runs (vb_ivf_search_filtered)
template <int ELEM, int METRIC>
__global__ void __launch_bounds__(SS_THREADS) cta_refine_masked_kernel(const uint8_t* __restrict__ rows, size_t stride, int V,
                                                                const uint8_t* __restrict__ qimg, size_t qstride, int k, int kp, int probes,
                                                                LcBound bound, const float* __restrict__ qn, const float* __restrict__ dist,
                                                                const float* __restrict__ smin, const int32_t* __restrict__ pre_pos,
                                                                const float* __restrict__ pre_key, int64_t cap, int64_t cap_s,
                                                                const int32_t* __restrict__ seg_len, const int32_t* __restrict__ probe_lists,
                                                                const int32_t* __restrict__ cand_off, const int64_t* __restrict__ list_off,
                                                                int32_t* __restrict__ out_pos, float* __restrict__ out_key,
                                                                int* __restrict__ n_failed, const int32_t* __restrict__ has_nan) {
    cta_refine_body<ELEM, METRIC, false, true>(rows, stride, V, qimg, qstride, k, kp, probes, bound, qn, dist, smin, pre_pos, pre_key, cap, cap_s,
                                               seg_len, probe_lists, cand_off, list_off, out_pos, out_key, n_failed, nullptr, nullptr, nullptr,
                                               nullptr, nullptr, has_nan);
}
template <int ELEM, int METRIC>
__global__ void __launch_bounds__(SS_THREADS) cta_refine_list_masked_kernel(const uint8_t* __restrict__ rows, size_t stride, int V,
                                                                const uint8_t* __restrict__ qimg, size_t qstride, int k, int kp, int probes,
                                                                LcBound bound, const float* __restrict__ qn, const float* __restrict__ dist,
                                                                const float* __restrict__ smin, int64_t cap, int64_t cap_s,
                                                                const int32_t* __restrict__ seg_len, const int32_t* __restrict__ probe_lists,
                                                                const int32_t* __restrict__ cand_off, const int64_t* __restrict__ list_off,
                                                                int32_t* __restrict__ out_pos, float* __restrict__ out_key,
                                                                int* __restrict__ n_failed, int32_t* __restrict__ fail_list,
                                                                const float* __restrict__ xn, const float* __restrict__ r8,
                                                                const float4* __restrict__ coef, unsigned long long* __restrict__ counters,
                                                                const int32_t* __restrict__ has_nan) {
    cta_refine_body<ELEM, METRIC, true, true>(rows, stride, V, qimg, qstride, k, kp, probes, bound, qn, dist, smin, nullptr, nullptr, cap, cap_s,
                                              seg_len, probe_lists, cand_off, list_off, out_pos, out_key, n_failed, fail_list, xn, r8, coef,
                                              counters, has_nan);
}

// Bytes one launch of list_tc_kernel moves, from the same job list the kernel walks (profiling only):
//   [0] bytes requested by the bulk copies (every (unit, query tile, K block) stage: A tile + B tile),
//   [1] distinct A bytes (each active (list, table tile) unit's planes once: re-reads by further query tiles of the
//       same unit come from L2),   [2] distinct B bytes (each list's query tiles once: shared by the list's units),
//   [3] launches accounted.
__global__ void lc_traffic_kernel(LcArgs a, uint32_t a_bytes, unsigned long long* __restrict__ acc) {
    unsigned long long issued = 0, a_once = 0, b_once = 0;
    for (int u = blockIdx.x * blockDim.x + threadIdx.x; u < a.n_units; u += gridDim.x * blockDim.x) {
        const ListUnit un = a.units[u];
        const int cnt = a.grp_cnt[un.list];
        if (cnt == 0) continue;
        const int nqt = (cnt + LC_N - 1) / LC_N;
        unsigned long long b_list = 0;
        for (int qt = 0; qt < nqt; ++qt) b_list += (unsigned long long)a.n_kblocks * (cnt - qt * LC_N <= 32 ? LC_B_STAGE / 2 : LC_B_STAGE);
        issued += (unsigned long long)nqt * a.n_kblocks * a_bytes + b_list;
        // a table tile that straddles two lists is visited by both units back to back: its second read comes from L2
        if (!(u > 0 && a.units[u - 1].tile == un.tile && a.grp_cnt[a.units[u - 1].list] > 0)) a_once += (unsigned long long)a.n_kblocks * a_bytes;
        if (u == 0 || a.units[u - 1].list != un.list) b_once += b_list;
    }
    atomicAdd(&acc[0], issued);
    atomicAdd(&acc[1], a_once);
    atomicAdd(&acc[2], b_once);
    if (blockIdx.x == 0 && threadIdx.x == 0) atomicAdd(&acc[3], 1ull);
}

// ----------------------------------------------------------------------------- host side

// c_sum of lc_make_bound: the fp32 norms, the final sum and the exact distance, relative to |x|^2 + |q|^2
static float lc_c_sum(int dim) { return std::max(1.0f / 65536.0f, 3.0f * ((float)dim / 32.0f + 8.0f) / 16777216.0f); }

// the batch's bound inputs (list_tc_query_norms): [|q|^2 | level 0: t_q | level 0: eps(q)^2 | level 0: per-row bound
// coefficients]; the refine kernels read |q|^2, or at level 0 eps(q)^2 and the coefficients
static const float* l0_qe2(const float* qn, int64_t nq) { return qn + 2 * nq; }
static float4* l0_row_coef(const float* qe2, int64_t nq) {
    return reinterpret_cast<float4*>(((uintptr_t)(qe2 + nq) + 15) & ~(uintptr_t)15);
}

int list_tc_query_norms(Scratch& sc, const void* qimg, size_t qstride, int64_t nq, float** qn) {
    void* p;
    VB_TRY(sc.take(sizeof(float) * (size_t)nq * 3 + 16 + sizeof(float4) * (size_t)nq + 64, &p));
    *qn = (float*)p;
    // the query image is fp32 with the rows' padded dimension count for both element types
    row_sqnorm_kernel<VB_VECTOR><<<(unsigned)((nq * 32 + 255) / 256), 256, 0, ctx().stream>>>((const uint8_t*)qimg, qstride, nq,
                                                                                            (int)(qstride / 4), *qn, nq, 0.f);
    VB_CUDA(cudaGetLastError());
    count_launch();
    return VB_OK;
}

// device accumulators: [0..3] / [4..7] lc_traffic_kernel per filter use (lists / centres), [8..10] the level-0 refine's
// counters (list_tc_level0_rescored)
static unsigned long long* g_traffic = nullptr;
static bool g_traffic_on = false;

bool list_tc_supported(int elem, int key_metric, int k) {
    return (elem == VB_VECTOR || elem == VB_HALFVEC) && (key_metric == VB_L2_SQUARED || key_metric == VB_NEG_IP) && k >= 1 &&
           list_tc_kp(k, 2) <= LC_MAX_KP;
}

int list_tc_kp(int k, int level) {
    // candidates kept per query.  Only those under the threshold are re-scored, so a generous k' costs a slightly
    // larger selection, not more exact distances; the certificate fails only when ALL k' are under the threshold.
    if (level == 0 || level == LIST_LEVEL_P) return k <= 10 ? 128 : 1 << 20;   // level 0's bound is ~4x level 1's: twice the candidates
    if (level == 1) return k <= 10 ? 64 : k <= 40 ? 128 : 1 << 20;
    return k <= 10 ? 32 : k <= 24 ? 48 : k <= 40 ? 64 : 1 << 20;
}

// packed planes + norms of the whole table (once per index load)
int list_tc_prepare(const Table& rows, ListTcImage* im) {
    Context& c = ctx();
    cudaStream_t s = c.stream;
    const int64_t n = rows.n;
    const int n_kblocks = (rows.dim + TC_K - 1) / TC_K;
    const int64_t n_tiles = (n + LC_M - 1) / LC_M;
    const size_t bytes = (size_t)n_tiles * n_kblocks * LC_A_STAGE;
    VB_CUDA(cudaMalloc(&im->planes, std::max<size_t>(bytes, 16)));
    VB_CUDA(cudaMalloc(&im->xn, sizeof(float) * (size_t)std::max<int64_t>(n_tiles * LC_M, 1)));
    im->n_kblocks = n_kblocks;
    im->n_tiles = n_tiles;
    if (n == 0) {
        im->xmax = 0.f;
        return VB_OK;
    }
    const int64_t chunks = n_tiles * LC_M * n_kblocks * 8;
    const unsigned grid = (unsigned)((chunks + 255) / 256);
    const unsigned g2 = (unsigned)((n_tiles * LC_M * 32 + 255) / 256);
    if (rows.elem == VB_VECTOR) {
        pack_planes_kernel<VB_VECTOR><<<grid, 256, 0, s>>>(rows.d, rows.stride, 0, n, rows.dim, LC_M, n_kblocks, im->planes, nullptr);
        row_sqnorm_kernel<VB_VECTOR><<<g2, 256, 0, s>>>(rows.d, rows.stride, n, rows.dim, im->xn, n_tiles * LC_M, 0.f);
    } else {
        pack_planes_kernel<VB_HALFVEC><<<grid, 256, 0, s>>>(rows.d, rows.stride, 0, n, rows.dim, LC_M, n_kblocks, im->planes, nullptr);
        row_sqnorm_kernel<VB_HALFVEC><<<g2, 256, 0, s>>>(rows.d, rows.stride, n, rows.dim, im->xn, n_tiles * LC_M, 0.f);
    }
    VB_CUDA(cudaGetLastError());
    count_launch(2);
    std::vector<float> h((size_t)n);
    VB_CUDA(cudaMemcpyAsync(h.data(), im->xn, sizeof(float) * (size_t)n, cudaMemcpyDeviceToHost, s));
    VB_CUDA(cudaStreamSynchronize(s));
    float m2 = 0.f;
    bool finite = true;
    for (float v : h) {
        if (!(v == v) || v > 3.0e38f) finite = false;
        else m2 = std::max(m2, v);
    }
    im->xmax = std::sqrt(m2);
    im->finite = finite;
    return VB_OK;
}

int list_tc_prepare_l0(const Table& rows, ListTcImage* im) {
    cudaStream_t s = ctx().stream;
    im->l0_tried = true;
    const int n_kblocks8 = (rows.dim + 127) / 128;
    const int64_t n_padded = im->n_tiles * LC_M;
    VB_CUDA(cudaMalloc(&im->planes8, std::max<size_t>((size_t)im->n_tiles * n_kblocks8 * LC_A_PLANE, 16)));
    VB_CUDA(cudaMalloc(&im->xs, sizeof(float) * (size_t)std::max<int64_t>(n_padded, 1)));
    VB_CUDA(cudaMalloc(&im->r8, sizeof(float) * (size_t)std::max<int64_t>(n_padded, 1)));
    im->n_kblocks8 = n_kblocks8;
    im->rmax = 0.f;
    if (rows.n == 0) return VB_OK;
    unsigned* d_rmax;
    VB_CUDA(cudaMalloc(&d_rmax, sizeof(unsigned)));
    VB_CUDA(cudaMemsetAsync(d_rmax, 0, sizeof(unsigned), s));
    const unsigned grid = (unsigned)((n_padded * 32 + 255) / 256);
    if (rows.elem == VB_VECTOR)
        pack_rows_i8_kernel<VB_VECTOR><<<grid, 256, 0, s>>>(rows.d, rows.stride, rows.n, rows.dim, n_kblocks8, n_padded, im->planes8, im->xs,
                                                            im->r8, d_rmax);
    else
        pack_rows_i8_kernel<VB_HALFVEC><<<grid, 256, 0, s>>>(rows.d, rows.stride, rows.n, rows.dim, n_kblocks8, n_padded, im->planes8, im->xs,
                                                             im->r8, d_rmax);
    VB_CUDA(cudaGetLastError());
    count_launch();
    unsigned bits = 0;
    VB_CUDA(cudaMemcpyAsync(&bits, d_rmax, sizeof(unsigned), cudaMemcpyDeviceToHost, s));
    VB_CUDA(cudaStreamSynchronize(s));
    VB_CUDA(cudaFree(d_rmax));
    memcpy(&im->rmax, &bits, sizeof(float));
    return VB_OK;
}

void list_tc_release(ListTcImage* im) {
    if (im->planes8) cudaFree(im->planes8);
    if (im->xs) cudaFree(im->xs);
    if (im->r8) cudaFree(im->r8);
    if (im->planes) cudaFree(im->planes);
    if (im->xn) cudaFree(im->xn);
    if (im->units) cudaFree(im->units);
    *im = ListTcImage{};
}

// the whole table's norm statistics after an in-place change, as list_tc_prepare (host loop over |x|^2) and
// list_tc_prepare_l0 (atomicMax of R_x) compute them: out[0] = max finite |x|^2 (float bits), out[1] = 1 when some
// |x|^2 is NaN or above 3e38, out[2] = max R_x (float bits; r8 may be NULL)
__global__ void norm_stats_kernel(const float* __restrict__ xn, const float* __restrict__ r8, int64_t n, unsigned* __restrict__ out) {
    unsigned m2 = 0u, bad = 0u, rm = 0u;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const float v = xn[i];
        if (!(v == v) || v > 3.0e38f) bad = 1u;
        else m2 = max(m2, __float_as_uint(v));
        if (r8) rm = max(rm, __float_as_uint(r8[i]));
    }
    if (m2) atomicMax(&out[0], m2);
    if (bad) atomicMax(&out[1], bad);
    if (rm) atomicMax(&out[2], rm);
}

bool list_tc_reserve(ListTcImage* im, int64_t nt, int64_t* cap_tiles, int64_t* cap_tiles8, bool* whole, bool* whole8) {
    *whole = *whole8 = false;
    bool ok = true;
    if (im->planes && nt > *cap_tiles) {
        // planes and norms are derived from the rows: the old buffers go before the larger ones are allocated
        cudaFree(im->planes);
        cudaFree(im->xn);
        im->planes = nullptr;
        im->xn = nullptr;
        const int64_t cap = std::max(nt, *cap_tiles + *cap_tiles / 2);
        ok = cudaMalloc(&im->planes, std::max<size_t>((size_t)cap * im->n_kblocks * LC_A_STAGE, 16)) == cudaSuccess &&
             cudaMalloc(&im->xn, sizeof(float) * (size_t)cap * LC_M) == cudaSuccess;
        *cap_tiles = cap;
        *whole = true;
    }
    if (ok && im->planes8 && nt > *cap_tiles8) {
        cudaFree(im->planes8);
        cudaFree(im->xs);
        cudaFree(im->r8);
        im->planes8 = nullptr;
        im->xs = im->r8 = nullptr;
        const int64_t cap = std::max(nt, *cap_tiles8 + *cap_tiles8 / 2);
        ok = cudaMalloc(&im->planes8, std::max<size_t>((size_t)cap * im->n_kblocks8 * LC_A_PLANE, 16)) == cudaSuccess &&
             cudaMalloc(&im->xs, sizeof(float) * (size_t)cap * LC_M) == cudaSuccess &&
             cudaMalloc(&im->r8, sizeof(float) * (size_t)cap * LC_M) == cudaSuccess;
        *cap_tiles8 = cap;
        *whole8 = true;
    }
    if (!ok) {
        cudaGetLastError();
        list_tc_release(im);
        *cap_tiles = *cap_tiles8 = 0;
    }
    return ok;
}

int list_tc_repack(const Table& rows, ListTcImage* im, int64_t first_tile, int64_t first_tile8, unsigned* d_stats) {
    Context& c = ctx();
    cudaStream_t s = c.stream;
    const int64_t n = rows.n;
    const int64_t nt = (n + LC_M - 1) / LC_M;
    const bool l0 = im->planes8 != nullptr;
    const int64_t t0 = std::min(first_tile, nt), t08 = std::min(first_tile8, nt);
    im->n_tiles = nt;
    VB_CUDA(cudaMemsetAsync(d_stats, 0, 4 * sizeof(unsigned), s));
    if (nt > t0) {
        const int64_t r0 = t0 * LC_M, pr = (nt - t0) * LC_M;
        const unsigned grid = (unsigned)((pr * im->n_kblocks * 8 + 255) / 256);
        const unsigned g2 = (unsigned)((pr * 32 + 255) / 256);
        uint8_t* planes = im->planes + (size_t)t0 * im->n_kblocks * LC_A_STAGE;
        if (rows.elem == VB_VECTOR) {
            pack_planes_kernel<VB_VECTOR><<<grid, 256, 0, s>>>(rows.d, rows.stride, r0, n - r0, rows.dim, LC_M, im->n_kblocks, planes, nullptr);
            row_sqnorm_kernel<VB_VECTOR><<<g2, 256, 0, s>>>(rows.d + (size_t)r0 * rows.stride, rows.stride, n - r0, rows.dim, im->xn + r0, pr, 0.f);
        } else {
            pack_planes_kernel<VB_HALFVEC><<<grid, 256, 0, s>>>(rows.d, rows.stride, r0, n - r0, rows.dim, LC_M, im->n_kblocks, planes, nullptr);
            row_sqnorm_kernel<VB_HALFVEC><<<g2, 256, 0, s>>>(rows.d + (size_t)r0 * rows.stride, rows.stride, n - r0, rows.dim, im->xn + r0, pr, 0.f);
        }
        VB_CUDA(cudaGetLastError());
        count_launch(2);
    }
    if (l0 && nt > t08) {
        const int64_t r0 = t08 * LC_M, pr = (nt - t08) * LC_M;
        const unsigned grid = (unsigned)((pr * 32 + 255) / 256);
        uint8_t* planes8 = im->planes8 + (size_t)t08 * im->n_kblocks8 * LC_A_PLANE;
        const uint8_t* src = rows.d + (size_t)r0 * rows.stride;
        if (rows.elem == VB_VECTOR)
            pack_rows_i8_kernel<VB_VECTOR><<<grid, 256, 0, s>>>(src, rows.stride, n - r0, rows.dim, im->n_kblocks8, pr, planes8, im->xs + r0,
                                                                im->r8 + r0, d_stats + 3);
        else
            pack_rows_i8_kernel<VB_HALFVEC><<<grid, 256, 0, s>>>(src, rows.stride, n - r0, rows.dim, im->n_kblocks8, pr, planes8, im->xs + r0,
                                                                 im->r8 + r0, d_stats + 3);
        VB_CUDA(cudaGetLastError());
        count_launch();
    }
    if (n > 0) {
        norm_stats_kernel<<<(unsigned)std::min<int64_t>((n + 255) / 256, 4 * (int64_t)c.sm_count), 256, 0, s>>>(im->xn, l0 ? im->r8 : nullptr,
                                                                                                             n, d_stats);
        VB_CUDA(cudaGetLastError());
        count_launch();
    }
    unsigned st[4] = {0u, 0u, 0u, 0u};
    VB_CUDA(cudaMemcpyAsync(st, d_stats, sizeof(st), cudaMemcpyDeviceToHost, s));
    VB_CUDA(cudaStreamSynchronize(s));
    float m2, rmax;
    memcpy(&m2, &st[0], sizeof(float));
    memcpy(&rmax, &st[2], sizeof(float));
    im->xmax = std::sqrt(m2);
    im->finite = st[1] == 0u;
    if (l0) im->rmax = rmax;
    return VB_OK;
}

// approximate pass: fills `out` (the per-query candidate runs) with d~
int launch_list_tc(const Table& rows, const ListTcImage& im, int key_metric, const void* qimg, size_t qstride, int64_t nq,
                   const int32_t* d_lists, int probes, const int32_t* cand_off, int64_t cap, const int64_t* d_list_off, int n_lists,
                   float* out, float* qn, bool one_list_all_queries, int level, float* smin, int64_t cap_s) {
    Context& c = ctx();
    cudaStream_t s = c.stream;
    Scratch sc;
    QueryGroups g{};
    VB_TRY(build_query_groups(sc, d_lists, nq, probes, cand_off, cap, n_lists, LC_N, &g, smin ? cap_s : 0));
    const int64_t max_gtiles = g.n_pairs / LC_N + n_lists + 1;
    void* d_B;
    // (level 0: the B tiles take half of this, the packed queries q8 follow them)
    const size_t q8_bytes = level == 0 ? (size_t)nq * 2 * im.n_kblocks8 * 128 : 0;
    VB_TRY(sc.take((size_t)max_gtiles * im.n_kblocks * LC_B_STAGE + q8_bytes, &d_B));
    float* d_tq = qn + nq;
    float* d_qe2 = d_tq + nq;
    // the query image is fp32 with the rows' padded dimension count for both element types
    const int qdim = (int)(qstride / 4);
    const bool l0 = level == 0;
    const int n_kblocks = l0 ? im.n_kblocks8 : im.n_kblocks;
    const int64_t chunks = g.n_pairs * n_kblocks * 8;
    if (l0) {
        VB_REQUIRE(im.planes8 != nullptr && !one_list_all_queries, "list scan level 0 without its int8 image");
        const int qpad = n_kblocks * 128;
        int8_t* q8 = (int8_t*)d_B + (size_t)max_gtiles * n_kblocks * LC_B_STAGE;
        l0_query_kernel<<<(unsigned)((nq * 32 + 255) / 256), 256, 0, s>>>((const float*)qimg, qstride, std::min(qdim, qpad), qpad, nq, im.xmax,
                                                                          im.rmax, key_metric == VB_L2_SQUARED, lc_c_sum(rows.dim), d_tq,
                                                                          d_qe2, l0_row_coef(d_qe2, nq), q8);
        pack_groups_i8_kernel<<<(unsigned)((chunks + 255) / 256), 256, 0, s>>>(q8, qpad, n_kblocks, g.n_pairs, g.pair_q, g.pair_list,
                                                                               g.begin, g.gt_begin, (uint8_t*)d_B);
        count_launch();
    } else {
        pack_groups_kernel<<<(unsigned)((chunks + 255) / 256), 256, 0, s>>>((const float*)qimg, qstride, qdim, n_kblocks, g.n_pairs,
                                                                            g.pair_q, g.pair_list, g.begin, g.gt_begin, (uint8_t*)d_B);
    }
    VB_CUDA(cudaGetLastError());
    count_launch();
    static bool attr_set = false;
    if (!attr_set) {
        VB_CUDA(cudaFuncSetAttribute(list_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)LC_SMEM));
        VB_CUDA(cudaFuncSetAttribute(list_tc_l0_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)LC_SMEM));
        attr_set = true;
    }
    LcArgs a{};
    a.A = l0 ? im.planes8 : im.planes;
    a.B = (const uint8_t*)d_B;
    a.units = im.units;
    a.n_units = im.n_units;
    a.list_off = d_list_off;
    a.grp_begin = g.begin;
    a.grp_cnt = g.cnt;
    a.gt_begin = g.gt_begin;
    a.pair_q = g.pair_q;
    a.pair_out = g.pair_out;
    a.xn = im.xn;
    a.qn = qn;
    a.out = out;
    a.smin = smin;
    a.pair_sbase = g.pair_sbase;
    a.n_kblocks = n_kblocks;
    a.is_l2 = key_metric == VB_L2_SQUARED;
    a.hi_only = level == 1;
    a.uniform_nqt = one_list_all_queries ? (int)((nq * probes + LC_N - 1) / LC_N) : 0;
    a.n_jobs = a.uniform_nqt ? im.n_units * a.uniform_nqt : im.n_units;
    const int grid = std::max(1, std::min(a.n_jobs, c.sm_count));
    prof_begin(one_list_all_queries ? VB_PROF_CENTRE_TC : VB_PROF_LIST_TC);
    if (l0) list_tc_l0_kernel<<<grid, LC_THREADS, LC_SMEM, s>>>(a, im.xs, d_tq);
    else list_tc_kernel<<<grid, LC_THREADS, LC_SMEM, s>>>(a);
    prof_end(one_list_all_queries ? VB_PROF_CENTRE_TC : VB_PROF_LIST_TC);
    VB_CUDA(cudaGetLastError());
    count_launch();
    if (g_traffic_on && g_traffic) {
        // (level 0: a.n_kblocks counts 128-dimension blocks of 16 KB per tile)
        lc_traffic_kernel<<<32, 256, 0, s>>>(a, level <= 1 ? LC_A_PLANE : LC_A_STAGE, g_traffic + (one_list_all_queries ? 4 : 0));
        VB_CUDA(cudaGetLastError());
    }
    return VB_OK;
}

int list_tc_traffic(int on, int64_t* out8) {
    cudaStream_t s = ctx().stream;
    if (!g_traffic) {
        VB_CUDA(cudaMalloc(&g_traffic, 11 * sizeof(unsigned long long)));
        VB_CUDA(cudaMemsetAsync(g_traffic, 0, 11 * sizeof(unsigned long long), s));
    }
    if (out8) {
        VB_CUDA(cudaMemcpyAsync(out8, g_traffic, 8 * sizeof(int64_t), cudaMemcpyDeviceToHost, s));
        VB_CUDA(cudaStreamSynchronize(s));
        VB_CUDA(cudaMemsetAsync(g_traffic, 0, 8 * sizeof(unsigned long long), s));
    }
    g_traffic_on = on != 0;
    return VB_OK;
}

int list_tc_level0_rescored(int64_t* out3) {
    cudaStream_t s = ctx().stream;
    for (int i = 0; i < 3; ++i) out3[i] = 0;
    if (!g_traffic) return VB_OK;
    VB_CUDA(cudaMemcpyAsync(out3, g_traffic + 8, 3 * sizeof(int64_t), cudaMemcpyDeviceToHost, s));
    VB_CUDA(cudaStreamSynchronize(s));
    VB_CUDA(cudaMemsetAsync(g_traffic + 8, 0, 3 * sizeof(unsigned long long), s));
    return VB_OK;
}

// |d~ - d_fp32| <= eps, in units of |x||q| for the product (x2 in the L2 form):
//   representation: bf16 keeps 8 significant bits (unit roundoff 2^-8), so |x - x_hi| <= 2^-8 |x| and
//     |x - x_hi - x_lo| <= 2^-16 |x|.  Level 2 drops x_lo.q_lo and the two residuals: 3 * 2^-16.  Level 1 also
//     drops x_lo.q: 2^-8 + 2^-16.
//   accumulation: one fp32 rounding of the accumulator per MMA, (products per K step) * dim / 16 of them,
//     <= 2^-23 each if the unit truncates; doubled to cover the alignment of the 16 products inside an MMA.
// The constants below are the values the GPU tests and benches of round 1 ran with (dim <= 1536); the formula takes
// over for longer rows, where the accumulation term grows past them.
// The fp32 norms, the final sum and the rounding of the exact fp32 distance it is compared with: 2^-16 (|x|^2 +
// |q|^2) for L2, 2^-17 |x||q| for the inner product.
//
// Level 0 (int8, l0_query_kernel computes it per query).  x^ = s_x x8, q^ = t_q (q_hi + q_lo / 254), r_x = |x - x^| <= R
// (rmax, every row), r_q = |q - q^| (computed from the packed integers), so |x^| <= xmax + R =: X and
//   |x.q - x^.q^| = |(x - x^).q + x^.(q - q^)| <= R |q| + X r_q.
// The tensor cores compute I_hi = x8.q_hi and I_lo = x8.q_lo exactly (int32); the epilogue's
// s_x (t_q fma(float(I_lo), 1/254, float(I_hi))) rounds six times (two conversions, the constant, the fma, two products):
// <= 8 u s_x t_q (|I_hi| + |I_lo| / 254) <= 2^-21 X t_q (|q_hi| + |q_lo| / 254) by Cauchy-Schwarz (u = 2^-24); 2^-20 is used.
// L2: twice the dot term plus c_sum (X^2 + |q|^2) (the norms, the final sum, the exact distance, as at levels 1 / 2); the
// inner product: the dot term plus 2^-17 X |q|.  The sums are taken in double, the result widened by 2^-10 and rounded up.
// It reaches the refine kernels as eps(q)^2 in the place of |q|^2, with the unit bound below: lc_eps() = sqrt(eps(q)^2).
//
// Per row (the level-0 refine's re-score rule).  Every step above holds for one row with its own r_x in the place of R
// and |x| in the place of xmax: |x^| <= |x| + r_x, the epilogue's roundings are <= 2^-21 |x^| t_q (|q_hi| + |q_lo| / 254),
// and the norm term is c_sum (|x|^2 + |q|^2).  So with R_x = r8[x] >= r_x (pack_rows_i8_kernel: sqrt of the double sum,
// widened by 2^-20, rounded up) and X_x = |x| (1 + 2^-10) + R_x:
//   E(x, q) = [2 (R_x |q| + X_x r_q + X_x qabs 2^-20) + c_sum (X_x^2 + |q|^2)] (1 + 2^-10)          (L2; +2e-30)
//   E(x, q) = [R_x |q| + X_x r_q + X_x qabs 2^-20 + X_x |q| 2^-17] (1 + 2^-10)                       (inner product)
// E_max = eps(q) is E at R_max and xmax.  |x| comes from the fp32 |x|^2 of the image (xn), whose relative error
// (dim / 32 + 5) 2^-24 is far below the 2^-10 on |x|.  l0_query_kernel splits E = a R_x + b X_x + c X_x^2 + d, computing
// a, b, c, d in double with the factor 2^-10 folded in and rounding each up to fp32; the refine evaluates X_x and E
// with every fp32 operation rounded up (__fsqrt_ru, __fmul_ru, __fadd_ru, __fmaf_ru on non-negative terms), so its E_i
// >= E(x, q).  It then forms fl(d~_i - E_i) in round-to-nearest and skips the row when that is > T: rounding is monotone
// and T is an fp32 value, so fl(d~_i - E_i) > T implies d~_i - E_i > T exactly, and d_fp32 >= d~_i - E_i > T.  The
// certificate compares d~_{k'} with fl_ru(T + sqrt_ru(eps(q)^2)) >= T + eps(q).  NaN anywhere re-scores the row or
// fails the certificate.  (tests/test_level0_rowbound.py checks |d~ - d| <= E against float64 on rows with mixed
// residuals.)

static LcBound lc_make_bound(const Table& rows, const ListTcImage& im, int key_metric, int level) {
    LcBound bound;
    bound.is_l2 = key_metric == VB_L2_SQUARED;
    if (level == 0) {
        bound.c_dot = 1.0f;
        bound.c_sum = 0.0f;
        bound.xmax = 1.0f;
        return bound;
    }
    const float steps = (float)(im.n_kblocks * (TC_K / 16));
    const float rep = level == 1 ? 1.0f / 256.0f + 1.0f / 65536.0f : 3.0f / 65536.0f;
    const float acc = 2.0f * (level == 1 ? 2.0f : 3.0f) * steps / 8388608.0f;
    const float ip_unit = rep + acc;
    float c_ip = level == 1 ? 1.0f / 256.0f + 1.0f / 8192.0f : 1.0f / 8192.0f;   // validated constants
    c_ip = std::max(c_ip, ip_unit);
    bound.c_dot = bound.is_l2 ? 2.0f * c_ip : c_ip + 1.0f / 131072.0f;
    // norms and the exact fp32 distance each sum dim / 32 terms per lane plus a shuffle tree: 3 * (dim / 32 + 8) * 2^-24 of
    // (|x|^2 + |q|^2) covers the two norms and the distance (<= 2 (|x|^2 + |q|^2)); 2^-16 up to ~2700 dimensions
    bound.c_sum = lc_c_sum(rows.dim);
    bound.xmax = im.xmax;
    return bound;
}

// steps 2 + 3 + 4 with one CTA per query
int launch_list_tc_cta_refine(const Table& rows, const ListTcImage& im, int key_metric, const void* qimg, size_t qstride, int64_t nq,
                              int k, int kp, int probes, const int32_t* d_lists, const int32_t* cand_off, const int64_t* d_list_off,
                              const float* dist, const float* smin, const int32_t* pre_pos, const float* pre_key, int64_t cap,
                              int64_t cap_s, const int32_t* seg_len, const float* qn, int32_t* out_pos, float* out_key, int* fail_dev,
                              int level, int32_t* fail_list, const int32_t* has_nan) {
    if (nq == 0) return VB_OK;
    Context& c = ctx();
    cudaStream_t s = c.stream;
    // level P: the runs hold lower bounds of the fp32 distance (vb_list_proj.cu), refined as level 0's with zero per-row
    // terms and eps(q) = 0: the coefficients and eps(q)^2 are zeroed, and |x|^2 stands in for R_x (0 R_x = 0 on finite rows)
    const bool lp = level == LIST_LEVEL_P;
    if (lp) {
        VB_CUDA(cudaMemsetAsync(const_cast<float*>(l0_qe2(qn, nq)), 0, sizeof(float) * (size_t)nq, s));
        VB_CUDA(cudaMemsetAsync(l0_row_coef(l0_qe2(qn, nq), nq), 0, sizeof(float4) * (size_t)nq, s));
    }
    const LcBound bound = lc_make_bound(rows, im, key_metric, lp ? 0 : level);
    const float* r8 = lp ? im.xn : im.r8;
    // the bound's per-query input: |q|^2, or at level 0 eps(q)^2 (lc_make_bound)
    if (level == 0 || lp) qn = l0_qe2(qn, nq);
    const int V = (int)(rows.stride / 16);
    const size_t smem = cta_refine_smem_bytes(kp, qstride, smin, pre_pos, cap, cap_s, probes);
    VB_REQUIRE(kp <= SS_THREADS && smem <= SS_SMEM_MAX && (smin || pre_pos || cap <= CR_RUN_MAX),
               "cta_refine: k' = %d / %zu bytes of shared memory not supported", kp, smem);
    VB_REQUIRE(!fail_list || (((level == 0 && im.r8) || lp) && smin),
               "cta_refine: the listing kernel is level 0's and P's and needs level 0's int8 image and slab minima");
#define VB_CR(E, M)                                                                                                              \
    do {                                                                                                                         \
        if (fail_list && has_nan) {                                                                                              \
            auto kern = cta_refine_list_masked_kernel<E, M>;                                                                     \
            if (smem > 48 * 1024) VB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));   \
            kern<<<(unsigned)nq, SS_THREADS, smem, s>>>(rows.d, rows.stride, V, (const uint8_t*)qimg, qstride, k, kp, probes, bound, qn, dist, \
                                                       smin, cap, cap_s, seg_len, d_lists, cand_off, d_list_off, out_pos, out_key, fail_dev, \
                                                       fail_list, im.xn, r8, l0_row_coef(qn, nq),                                     \
                                                       g_traffic_on ? g_traffic + 8 : nullptr, has_nan);                        \
            break;                                                                                                               \
        }                                                                                                                        \
        if (has_nan) {                                                                                                           \
            auto kern = cta_refine_masked_kernel<E, M>;                                                                          \
            if (smem > 48 * 1024) VB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));   \
            kern<<<(unsigned)nq, SS_THREADS, smem, s>>>(rows.d, rows.stride, V, (const uint8_t*)qimg, qstride, k, kp, probes, bound, qn, dist, \
                                                       smin, pre_pos, pre_key, cap, cap_s, seg_len, d_lists, cand_off, d_list_off, out_pos, \
                                                       out_key, fail_dev, has_nan);                                              \
            break;                                                                                                               \
        }                                                                                                                        \
        if (fail_list) {                                                                                                         \
            auto kern = cta_refine_list_kernel<E, M>;                                                                            \
            if (smem > 48 * 1024) VB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));   \
            kern<<<(unsigned)nq, SS_THREADS, smem, s>>>(rows.d, rows.stride, V, (const uint8_t*)qimg, qstride, k, kp, probes, bound, qn, dist, \
                                                       smin, cap, cap_s, seg_len, d_lists, cand_off, d_list_off, out_pos, out_key, fail_dev, \
                                                       fail_list, im.xn, r8, l0_row_coef(qn, nq),                                     \
                                                       g_traffic_on ? g_traffic + 8 : nullptr);                                 \
            break;                                                                                                               \
        }                                                                                                                        \
        auto kern = cta_refine_kernel<E, M>;                                                                                     \
        if (smem > 48 * 1024) VB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));       \
        kern<<<(unsigned)nq, SS_THREADS, smem, s>>>(rows.d, rows.stride, V, (const uint8_t*)qimg, qstride, k, kp, probes, bound, qn, dist, smin, \
                                                   pre_pos, pre_key, cap, cap_s, seg_len, d_lists, cand_off, d_list_off, out_pos, out_key,   \
                                                   fail_dev);                                                                               \
    } while (0)
    if (rows.elem == VB_VECTOR) {
        if (key_metric == VB_L2_SQUARED) VB_CR(VB_VECTOR, VB_L2_SQUARED);
        else VB_CR(VB_VECTOR, VB_NEG_IP);
    } else {
        if (key_metric == VB_L2_SQUARED) VB_CR(VB_HALFVEC, VB_L2_SQUARED);
        else VB_CR(VB_HALFVEC, VB_NEG_IP);
    }
#undef VB_CR
    VB_CUDA(cudaGetLastError());
    count_launch();
    return VB_OK;
}

}  // namespace vb
