// vb_order.cu -- the btree operator classes of vector, halfvec and sparsevec (vector_ops, halfvec_ops, sparsevec_ops,
// sql/vector.sql:397, 810, 1180) over a resident table: the rows in the order of vector_cmp_internal /
// halfvec_cmp_internal / sparsevec_cmp_internal (src/vector.c:1030-1052, src/halfvec.c:987, src/sparsevec.c:1153-1188),
// their groups of equal rows, and batched lower / upper bounds of query rows in that order.  This is what ORDER BY v,
// SELECT DISTINCT v, GROUP BY v, a btree build on v and WHERE v = / < / <= / >= / > $1 need.
//
// Keys.  A row is a sequence of key words whose lexicographic order is the comparator's:
//   vector   one 32-bit word per element: -0 made +0, then bits ^ (sign ? 0xFFFFFFFF : 0x80000000);
//   halfvec  the same map on 16 bits, two elements per 32-bit word (element 2w in the high half; the missing half of an
//            odd dimension is 0 in every row);
//   sparse   one 64-bit key per stored entry (i, v): v < 0: (i << 32) | f(v), else (2 << 62) | ((2^30 - 1 - i) << 32) |
//            f(v), then the terminator 1 << 62 (f: the fp32 map above).  Exact for rows of one dimension, stored zeros
//            and +-inf included (the reference treats 0 as non-negative where the indices differ).
// Ties go to the smaller row number.  NaN has a place in the bit order, so a row holding one lands somewhere without
// harm; the reference's types never hold NaN.
//
// Sort: segmented refinement, host-driven, one 16-byte read-back per pass (live segments and their rows).
//   pass 1   order_keys_kernel builds a 64-bit key of every row (dense: key words 0 and 1; sparse: key 0), a stable CUB
//            radix sort orders (key, row number), and runs of equal keys are the segments;
//   pass k   for every unresolved segment of >= 2 rows: order_lcp_kernel (one warp per row, 32 key words per step,
//            ballot + atomicMin) finds p, the first key position at or past the segment's depth where some row differs
//            from the segment's first row.  No such p: the segment is a group.  Otherwise order_keys_kernel gathers the
//            64-bit key at p (dense: words p and p + 1), cub::DeviceSegmentedSort::StableSortPairs sorts every segment
//            by it, order_split_kernel cuts the segments at key changes and order_next_kernel lists the pieces of >= 2
//            rows that are not yet decided, at depth p + 2 (dense) or p + 1 (sparse).
// Stable sorts keep ascending row numbers inside a segment, so ties need no key.  Every pass raises each live segment's
// depth, so there are at most (key words + 1) passes, and a table of identical rows takes 2: one read of its rows in the
// LCP kernel resolves it.  The final segments are the groups (inclusive scan of the segment heads).
//
// Bounds: order_bounds_kernel, one warp per query, binary search over the order; each step compares the query with row
// perm[mid] 32 keys at a time (ballot, first difference), sparse keys generated from the CSR on the fly.  The search
// for lo (rows < q) narrows the range of the search for hi (rows <= q).
#include "vb_common.cuh"

#include <cub/cub.cuh>
#include <thrust/iterator/counting_iterator.h>

#include <algorithm>
#include <climits>
#include <mutex>
#include <unordered_set>
#include <vector>

namespace vb {

// ---------------------------------------------------------------------------------------------- owners
// An order reads its table's rows at every bounds call, long after creation, so it must know whether the table still
// exists: the stamps of tables that have an order, until the table is freed.
static std::mutex g_watch_mu;
static std::unordered_set<uint64_t> g_watched;

void owner_watch(uint64_t uid) {
    std::lock_guard<std::mutex> g(g_watch_mu);
    g_watched.insert(uid);
}

void owner_released(uint64_t uid) {
    std::lock_guard<std::mutex> g(g_watch_mu);
    g_watched.erase(uid);
}

static bool owner_alive(uint64_t uid) {
    std::lock_guard<std::mutex> g(g_watch_mu);
    return g_watched.count(uid) != 0;
}

// ---------------------------------------------------------------------------------------------- keys

constexpr uint64_t SP_TERM = 1ull << 62;   // ends every sparse row's key sequence
constexpr int LCP_NONE = INT_MAX;          // no differing position: the segment is a group

struct DenseSrc {
    const uint8_t* base;   // row r at base + r * stride
    size_t stride;
    int elem, dim, words;  // words: key words per row
};
struct SparseSrc {
    const int64_t* off;
    const int32_t* idx;
    const float* val;
};

__host__ __device__ inline int dense_words(int elem, int dim) { return elem == VB_VECTOR ? dim : (dim + 1) / 2; }

__device__ __forceinline__ uint32_t f32_key(uint32_t b) {
    if (b == 0x80000000u) b = 0u;
    return b ^ ((b >> 31) ? 0xFFFFFFFFu : 0x80000000u);
}
__device__ __forceinline__ uint32_t f16_key(uint32_t h) {
    if (h == 0x8000u) h = 0u;
    return h ^ ((h >> 15) ? 0xFFFFu : 0x8000u);
}

// key word w < words of a dense row
__device__ __forceinline__ uint32_t dense_word(const uint8_t* row, int elem, int dim, int w) {
    if (elem == VB_VECTOR) return f32_key(reinterpret_cast<const uint32_t*>(row)[w]);
    const uint16_t* h = reinterpret_cast<const uint16_t*>(row);
    const uint32_t lo = 2 * w + 1 < dim ? f16_key(h[2 * w + 1]) : 0u;
    return (f16_key(h[2 * w]) << 16) | lo;
}

__device__ __forceinline__ uint64_t sparse_entry_key(int32_t i, float v) {
    const uint32_t f = f32_key(__float_as_uint(v));
    if (v < 0.f) return ((uint64_t)(uint32_t)i << 32) | f;
    return (2ull << 62) | ((uint64_t)((1u << 30) - 1u - (uint32_t)i) << 32) | f;
}

// key p of the sparse row whose entries are beg .. beg + nnz (the terminator at p >= nnz)
__device__ __forceinline__ uint64_t sparse_key(const SparseSrc& S, int64_t beg, int64_t nnz, int64_t p) {
    return p < nnz ? sparse_entry_key(S.idx[beg + p], S.val[beg + p]) : SP_TERM;
}

// the 64-bit sort key of row r at key position p
template <bool SPARSE>
__device__ __forceinline__ uint64_t sort_key(const DenseSrc& D, const SparseSrc& S, int64_t r, int p) {
    if (SPARSE) {
        const int64_t beg = S.off[r];
        return sparse_key(S, beg, S.off[r + 1] - beg, p);
    }
    const uint8_t* row = D.base + (size_t)r * D.stride;
    const uint64_t hi = dense_word(row, D.elem, D.dim, p);
    const uint64_t lo = p + 1 < D.words ? dense_word(row, D.elem, D.dim, p + 1) : 0u;
    return (hi << 32) | lo;
}

// ---------------------------------------------------------------------------------------------- sort kernels

// The live segments of a pass: segment s holds the rows perm[start[s] .. start[s] + len[s]), equal in keys [0, depth[s]).
// In the pass they are laid out one after the other (compact positions aoff[s] .. aoff[s + 1]).
struct SegList {
    int32_t* start;
    int32_t* len;
    int32_t* depth;
};

__global__ void order_first_init_kernel(int32_t n, int32_t* aoff, int32_t* start, int32_t* p) {
    aoff[0] = 0;
    aoff[1] = n;
    start[0] = 0;
    p[0] = 0;
}

// compact position j -> its segment s (segof), its row (rows); p[s] = LCP_NONE, to be lowered by order_lcp_kernel
__global__ void __launch_bounds__(256) order_map_kernel(int32_t R, int32_t m, const int32_t* __restrict__ aoff,
                                                        const int32_t* __restrict__ start, const int32_t* __restrict__ perm,
                                                        int32_t* __restrict__ segof, int32_t* __restrict__ rows, int32_t* __restrict__ p) {
    const int32_t j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= R) return;
    int32_t a = 0, b = m;   // last s with aoff[s] <= j
    while (b - a > 1) {
        const int32_t mid = (a + b) >> 1;
        if (aoff[mid] <= j) a = mid;
        else b = mid;
    }
    segof[j] = a;
    rows[j] = perm[start[a] + (j - aoff[a])];
    if (j == aoff[a]) p[a] = LCP_NONE;
}

// One warp per compact position j that is not its segment's first: the first key position >= depth where row j
// differs from the first row, min-reduced into p[s].  A warp stops at a chunk that starts at or past the current p[s].
template <bool SPARSE>
__global__ void __launch_bounds__(256) order_lcp_kernel(int32_t R, const int32_t* __restrict__ segof, const int32_t* __restrict__ aoff,
                                                        const int32_t* __restrict__ depth, const int32_t* __restrict__ rows, DenseSrc D,
                                                        SparseSrc S, int32_t* p) {
    const int32_t j = (int32_t)((blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5);
    const int lane = threadIdx.x & 31;
    if (j >= R) return;   // whole warps
    const int32_t s = segof[j];
    const int32_t a = aoff[s];
    if (j == a) return;
    const int64_t r0 = rows[a], r1 = rows[j];
    const int d = depth[s];
    int64_t b0 = 0, b1 = 0, n0 = 0, n1 = 0;
    int L = D.words;
    if (SPARSE) {
        b0 = S.off[r0];
        n0 = S.off[r0 + 1] - b0;
        b1 = S.off[r1];
        n1 = S.off[r1 + 1] - b1;
        L = (int)n0 + 1;   // past the first row's terminator a differing row has differed already
    }
    const uint8_t* x0 = SPARSE ? nullptr : D.base + (size_t)r0 * D.stride;
    const uint8_t* x1 = SPARSE ? nullptr : D.base + (size_t)r1 * D.stride;
    for (int c = d; c < L; c += 32) {
        int cur = 0;
        if (lane == 0) cur = *(volatile int32_t*)&p[s];
        if (c >= __shfl_sync(0xffffffffu, cur, 0)) break;
        const int w = c + lane;
        bool ne = false;
        if (w < L) {
            if (SPARSE) ne = sparse_key(S, b0, n0, w) != sparse_key(S, b1, n1, w);
            else ne = dense_word(x0, D.elem, D.dim, w) != dense_word(x1, D.elem, D.dim, w);
        }
        const unsigned bal = __ballot_sync(0xffffffffu, ne);
        if (bal) {
            if (lane == 0) atomicMin(&p[s], c + __ffs(bal) - 1);
            break;
        }
    }
}

// kin[j] = the sort key of compact position j at its segment's p (0 for a resolved segment: the stable sort then keeps
// it as it is).  first: the first pass, rows[j] = j, one segment, p = 0.
template <bool SPARSE>
__global__ void __launch_bounds__(256) order_keys_kernel(int32_t R, bool first, int32_t* __restrict__ rows, int32_t* __restrict__ segof,
                                                         const int32_t* __restrict__ p, DenseSrc D, SparseSrc S, uint64_t* __restrict__ kin) {
    const int32_t j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= R) return;
    int32_t r, ps;
    if (first) {
        r = j;
        rows[j] = j;
        segof[j] = 0;
        ps = 0;
    } else {
        r = rows[j];
        ps = p[segof[j]];
    }
    kin[j] = ps == LCP_NONE ? 0ull : sort_key<SPARSE>(D, S, r, ps);
}

// The sorted segments back into the order; a head marks the first row of every new segment (flag: and of every piece
// of a segment that was split, the candidates for the next pass).
__global__ void __launch_bounds__(256) order_split_kernel(int32_t R, const int32_t* __restrict__ segof, const int32_t* __restrict__ aoff,
                                                          const int32_t* __restrict__ start, const int32_t* __restrict__ p,
                                                          const uint64_t* __restrict__ kout, const int32_t* __restrict__ vout,
                                                          int32_t* __restrict__ perm, int32_t* __restrict__ head, uint8_t* __restrict__ flag) {
    const int32_t j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= R) return;
    const int32_t s = segof[j];
    const int32_t a = aoff[s];
    const bool live = p[s] != LCP_NONE;
    const bool st = j == a || (live && kout[j] != kout[j - 1]);
    const int32_t pos = start[s] + (j - a);
    perm[pos] = vout[j];
    if (st) head[pos] = 1;
    flag[j] = st && live;
}

// Piece i of the split (compact positions starts[i] .. the next piece or its segment's end): a piece of >= 2 rows
// whose rows are not yet known equal joins the next pass at depth p + width.  cnt[0] / cnt[1] += segments / rows.
template <bool SPARSE>
__global__ void __launch_bounds__(256) order_next_kernel(int32_t R, const int32_t* __restrict__ nsel, const int32_t* __restrict__ starts,
                                                         const int32_t* __restrict__ segof, const int32_t* __restrict__ aoff,
                                                         const int32_t* __restrict__ start, const int32_t* __restrict__ p,
                                                         const uint64_t* __restrict__ kout, int words, SegList next,
                                                         unsigned long long* __restrict__ cnt) {
    const int32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    const int32_t ns = *nsel;
    if (i >= ns) return;
    const int32_t j = starts[i];
    const int32_t s = segof[j];
    const int32_t e = min(i + 1 < ns ? starts[i + 1] : R, aoff[s + 1]);
    const int32_t len = e - j;
    if (len < 2) return;
    const int32_t dnew = p[s] + (SPARSE ? 1 : 2);
    if (SPARSE ? kout[j] == SP_TERM : dnew >= words) return;   // keys equal to the end: a group
    const int32_t k = (int32_t)atomicAdd(&cnt[0], 1ull);
    atomicAdd(&cnt[1], (unsigned long long)len);
    next.start[k] = start[s] + (j - aoff[s]);
    next.len[k] = len;
    next.depth[k] = dnew;
}

// perm (int64), group_of_row, group_start from the final order and the inclusive scan of its heads
__global__ void __launch_bounds__(256) order_finish_kernel(int32_t n, const int32_t* __restrict__ perm, const int32_t* __restrict__ head,
                                                           const int32_t* __restrict__ gscan, int64_t* __restrict__ perm64,
                                                           int32_t* __restrict__ gor, int64_t* __restrict__ gstart) {
    const int32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int32_t g = gscan[i] - 1;
    const int32_t r = perm[i];
    perm64[i] = r;
    gor[r] = g;
    if (head[i]) gstart[g] = i;
    if (i == n - 1) gstart[g + 1] = n;
}

// ---------------------------------------------------------------------------------------------- bounds kernel

// -1 / 0 / 1 (on every lane) for query vs row: the first differing key decides, 32 keys per step
template <bool SPARSE>
__device__ __forceinline__ int warp_compare(const DenseSrc& D, const uint8_t* q, const SparseSrc& S, int64_t qb, int64_t qn,
                                            const SparseSrc& QS, int64_t r, int lane) {
    int64_t rb = 0, rn = 0;
    int64_t L = D.words;
    const uint8_t* x = nullptr;
    if (SPARSE) {
        rb = S.off[r];
        rn = S.off[r + 1] - rb;
        L = min(qn, rn) + 1;
    } else {
        x = D.base + (size_t)r * D.stride;
    }
    for (int64_t c = 0; c < L; c += 32) {
        const int64_t w = c + lane;
        uint64_t kq = 0, kr = 0;
        if (w < L) {
            if (SPARSE) {
                kq = sparse_key(QS, qb, qn, w);
                kr = sparse_key(S, rb, rn, w);
            } else {
                kq = dense_word(q, D.elem, D.dim, (int)w);
                kr = dense_word(x, D.elem, D.dim, (int)w);
            }
        }
        const unsigned bal = __ballot_sync(0xffffffffu, kq != kr);
        if (bal) return __shfl_sync(0xffffffffu, kq < kr ? -1 : 1, __ffs(bal) - 1);
    }
    return 0;
}

// One warp per query: lo = rows < q, hi = rows <= q in the order perm[0 .. n).  Dense queries are packed rows of
// qbytes bytes; sparse ones CSR (QS, offsets absolute into its idx / val).
template <bool SPARSE>
__global__ void __launch_bounds__(256) order_bounds_kernel(int64_t nq, const int64_t* __restrict__ perm, int64_t n, DenseSrc D, SparseSrc S,
                                                           const uint8_t* __restrict__ queries, size_t qbytes, SparseSrc QS,
                                                           int64_t* __restrict__ out_lo, int64_t* __restrict__ out_hi) {
    const int64_t q = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (q >= nq) return;   // whole warps
    const uint8_t* qrow = SPARSE ? nullptr : queries + (size_t)q * qbytes;
    int64_t qb = 0, qn = 0;
    if (SPARSE) {
        qb = QS.off[q];
        qn = QS.off[q + 1] - qb;
    }
    int64_t a = 0, b = n, hb = n;
    while (a < b) {   // first position whose row is >= q; rows found > q cap the second search
        const int64_t mid = (a + b) >> 1;
        const int c = warp_compare<SPARSE>(D, qrow, S, qb, qn, QS, perm[mid], lane);
        if (c > 0) a = mid + 1;
        else {
            b = mid;
            if (c < 0) hb = mid;
        }
    }
    const int64_t lo = a;
    b = hb;
    while (a < b) {   // first position whose row is > q
        const int64_t mid = (a + b) >> 1;
        if (warp_compare<SPARSE>(D, qrow, S, qb, qn, QS, perm[mid], lane) >= 0) a = mid + 1;
        else b = mid;
    }
    if (lane == 0) {
        out_lo[q] = lo;
        out_hi[q] = a;
    }
}

}  // namespace vb

using namespace vb;

struct vb_order {
    const void* owner = nullptr;   // the vb_table or vb_sparse_table it was made for
    uint64_t owner_uid = 0;
    bool sparse = false;
    int dim = 0;
    int64_t n = 0, groups = 0, passes = 0;
    void* mem = nullptr;           // perm [n] | group_start [n + 1] | group_of_row [n]
    int64_t* perm = nullptr;
    int64_t* gstart = nullptr;
    int32_t* gor = nullptr;
};

namespace vb {

static inline unsigned grid_of(int64_t threads) { return (unsigned)((threads + 255) / 256); }

// The sort of n rows (DenseSrc or SparseSrc, by SPARSE) into o: perm, group_of_row, group_start, groups, passes.
template <bool SPARSE>
static int order_build(const char* fn, const DenseSrc& D, const SparseSrc& S, int64_t n_rows, vb_order* o) {
    Context& c = ctx();
    cudaStream_t st = c.stream;
    const int32_t n = (int32_t)n_rows;
    const int64_t cap = n_rows / 2 + 2;   // live segments of a pass hold >= 2 rows each
    // CUB temporaries at their largest: the sizes grow with the item and segment counts
    size_t b_radix = 0, b_seg = 0, b_sel = 0, b_xscan = 0, b_iscan = 0;
    if (n > 0) {
        VB_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, b_radix, (const uint64_t*)nullptr, (uint64_t*)nullptr, (const int32_t*)nullptr,
                                                (int32_t*)nullptr, n, 0, 64, st));
        VB_CUDA(cub::DeviceSegmentedSort::StableSortPairs(nullptr, b_seg, (const uint64_t*)nullptr, (uint64_t*)nullptr,
                                                          (const int32_t*)nullptr, (int32_t*)nullptr, n, (int)(cap - 1),
                                                          (const int32_t*)nullptr, (const int32_t*)nullptr, st));
        VB_CUDA(cub::DeviceSelect::Flagged(nullptr, b_sel, thrust::counting_iterator<int32_t>(0), (const uint8_t*)nullptr, (int32_t*)nullptr,
                                           (int32_t*)nullptr, n, st));
        VB_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, b_xscan, (const int32_t*)nullptr, (int32_t*)nullptr, (int)cap, st));
        VB_CUDA(cub::DeviceScan::InclusiveSum(nullptr, b_iscan, (const int32_t*)nullptr, (int32_t*)nullptr, n, st));
    }
    const size_t b_cub = std::max({b_radix, b_seg, b_sel, b_xscan, b_iscan, (size_t)16});
    auto al = [](size_t b) { return (b + 255) & ~(size_t)255; };
    const size_t N = (size_t)std::max<int64_t>(n_rows, 1);
    // kin, kout | rows, vout, perm, head, segof, starts | flag | 8 lists of cap (cur: start, len, depth, p, aoff; next:
    // start, len, depth) | counters | CUB
    const size_t tmp_bytes = 2 * al(8 * N) + 6 * al(4 * N) + al(N) + 8 * al(4 * (size_t)cap) + al(16 + 4) + al(b_cub);
    const size_t out_bytes = al(8 * N) + al(8 * (N + 1)) + al(4 * N);
    if (cudaMalloc(&o->mem, out_bytes) != cudaSuccess) {
        cudaGetLastError();
        o->mem = nullptr;
        set_error("%s: allocation of %zu bytes for the order (and %zu bytes of temporaries) failed", fn, out_bytes, tmp_bytes);
        return VB_ENOMEM;
    }
    Scratch sc;
    void* tmp;
    if (sc.own(tmp_bytes, &tmp) != VB_OK) {
        cudaFree(o->mem);
        o->mem = nullptr;
        set_error("%s: allocation of %zu bytes of temporaries (beside %zu bytes for the order) failed", fn, tmp_bytes, out_bytes);
        return VB_ENOMEM;
    }
    uint8_t* q = (uint8_t*)o->mem;
    o->perm = (int64_t*)q;
    q += al(8 * N);
    o->gstart = (int64_t*)q;
    q += al(8 * (N + 1));
    o->gor = (int32_t*)q;
    o->n = n_rows;
    o->passes = 0;
    if (n == 0) {
        o->groups = 0;
        VB_CUDA(cudaMemsetAsync(o->gstart, 0, sizeof(int64_t), st));
        VB_CUDA(cudaStreamSynchronize(st));
        return VB_OK;
    }
    uint8_t* t = (uint8_t*)tmp;
    auto take = [&](size_t b) {
        uint8_t* r = t;
        t += al(b);
        return r;
    };
    uint64_t* kin = (uint64_t*)take(8 * N);
    uint64_t* kout = (uint64_t*)take(8 * N);
    int32_t* rows = (int32_t*)take(4 * N);
    int32_t* vout = (int32_t*)take(4 * N);
    int32_t* perm = (int32_t*)take(4 * N);
    int32_t* head = (int32_t*)take(4 * N);
    int32_t* segof = (int32_t*)take(4 * N);
    int32_t* starts = (int32_t*)take(4 * N);
    uint8_t* flag = take(N);
    SegList cur{(int32_t*)take(4 * cap), (int32_t*)take(4 * cap), (int32_t*)take(4 * cap)};
    int32_t* p = (int32_t*)take(4 * cap);
    int32_t* aoff = (int32_t*)take(4 * cap);
    SegList next{(int32_t*)take(4 * cap), (int32_t*)take(4 * cap), (int32_t*)take(4 * cap)};
    unsigned long long* cnt = (unsigned long long*)take(16 + 4);
    int32_t* nsel = (int32_t*)(cnt + 2);
    void* cub_tmp = take(b_cub);
    size_t cb;
    const int words = SPARSE ? 0 : D.words;
    // A pass can only lose segments or deepen them, so the loop ends within key length + 1 passes; the bound turns a
    // defect into an error instead of a hang.
    const int64_t max_passes = SPARSE ? 16000 + 3 : (int64_t)D.words + 2;

    VB_CUDA(cudaMemsetAsync(head, 0, 4 * N, st));
    order_first_init_kernel<<<1, 1, 0, st>>>(n, aoff, cur.start, p);
    order_keys_kernel<SPARSE><<<grid_of(n), 256, 0, st>>>(n, true, rows, segof, p, D, S, kin);
    VB_CUDA(cudaGetLastError());
    count_launch(2);
    cb = b_cub;
    VB_CUDA(cub::DeviceRadixSort::SortPairs(cub_tmp, cb, kin, kout, rows, vout, n, 0, 64, st));
    int32_t R = n;
    int64_t m = 1;
    for (;;) {
        ++o->passes;
        order_split_kernel<<<grid_of(R), 256, 0, st>>>(R, segof, aoff, cur.start, p, kout, vout, perm, head, flag);
        VB_CUDA(cudaGetLastError());
        cb = b_cub;
        VB_CUDA(cub::DeviceSelect::Flagged(cub_tmp, cb, thrust::counting_iterator<int32_t>(0), flag, starts, nsel, R, st));
        VB_CUDA(cudaMemsetAsync(cnt, 0, 16, st));
        order_next_kernel<SPARSE><<<grid_of(R), 256, 0, st>>>(R, nsel, starts, segof, aoff, cur.start, p, kout, words, next, cnt);
        VB_CUDA(cudaGetLastError());
        count_launch(2);
        unsigned long long h[2];
        VB_CUDA(cudaMemcpyAsync(h, cnt, 16, cudaMemcpyDeviceToHost, st));
        VB_CUDA(cudaStreamSynchronize(st));
        m = (int64_t)h[0];
        R = (int32_t)h[1];
        if (m == 0) break;
        if (o->passes >= max_passes) {
            set_error("%s: the sort did not converge in %lld passes (internal error)", fn, (long long)o->passes);
            return VB_ESTATE;
        }
        std::swap(cur, next);
        // compact offsets of the live segments (len[m] = 0 makes aoff[m] = R)
        VB_CUDA(cudaMemsetAsync(cur.len + m, 0, 4, st));
        cb = b_cub;
        VB_CUDA(cub::DeviceScan::ExclusiveSum(cub_tmp, cb, cur.len, aoff, (int)(m + 1), st));
        order_map_kernel<<<grid_of(R), 256, 0, st>>>(R, (int32_t)m, aoff, cur.start, perm, segof, rows, p);
        order_lcp_kernel<SPARSE><<<grid_of((int64_t)R * 32), 256, 0, st>>>(R, segof, aoff, cur.depth, rows, D, S, p);
        order_keys_kernel<SPARSE><<<grid_of(R), 256, 0, st>>>(R, false, rows, segof, p, D, S, kin);
        VB_CUDA(cudaGetLastError());
        count_launch(3);
        cb = b_cub;
        VB_CUDA(cub::DeviceSegmentedSort::StableSortPairs(cub_tmp, cb, kin, kout, rows, vout, R, (int)m, aoff, aoff + 1, st));
    }
    // groups: inclusive scan of the heads
    cb = b_cub;
    VB_CUDA(cub::DeviceScan::InclusiveSum(cub_tmp, cb, head, segof, n, st));
    order_finish_kernel<<<grid_of(n), 256, 0, st>>>(n, perm, head, segof, o->perm, o->gor, o->gstart);
    VB_CUDA(cudaGetLastError());
    count_launch();
    int32_t g = 0;
    VB_CUDA(cudaMemcpyAsync(&g, segof + n - 1, 4, cudaMemcpyDeviceToHost, st));
    VB_CUDA(cudaStreamSynchronize(st));
    o->groups = g;
    return VB_OK;
}

static int order_create(const char* fn, const void* owner, uint64_t uid, bool sparse, int dim, const DenseSrc& D, const SparseSrc& S,
                        int64_t n, vb_order** out) {
    VB_REQUIRE(n < (int64_t)INT32_MAX, "%s: %lld rows, an order takes at most %d (group_of_row is int32)", fn, (long long)n, INT32_MAX - 1);
    vb_order* o = new vb_order;
    o->owner = owner;
    o->owner_uid = uid;
    o->sparse = sparse;
    o->dim = dim;
    const int rc = sparse ? order_build<true>(fn, D, S, n, o) : order_build<false>(fn, D, S, n, o);
    if (rc != VB_OK) {
        if (o->mem) {
            cudaStreamSynchronize(ctx().stream);
            cudaFree(o->mem);
        }
        delete o;
        return rc;
    }
    owner_watch(uid);
    *out = o;
    return VB_OK;
}

// the order's table, as it is now (its rows may have moved since creation); refuses a freed owner and the wrong kind
static int order_owner(const char* fn, const vb_order* o, bool sparse) {
    VB_REQUIRE(o, "%s: null order", fn);
    VB_REQUIRE(o->sparse == sparse, "%s: the order is of a %s table (use %s)", fn, o->sparse ? "sparse" : "dense",
               o->sparse ? "vb_sparse_order_bounds" : "vb_order_bounds");
    VB_REQUIRE(owner_alive(o->owner_uid), "%s: the order's table was freed", fn);
    return VB_OK;
}

static int launch_bounds(const vb_order* o, bool sparse, const DenseSrc& D, const SparseSrc& S, const uint8_t* queries, size_t qbytes,
                         const SparseSrc& QS, int64_t nq, int64_t* lo, int64_t* hi) {
    cudaStream_t st = ctx().stream;
    if (sparse)
        order_bounds_kernel<true><<<grid_of(nq * 32), 256, 0, st>>>(nq, o->perm, o->n, D, S, queries, qbytes, QS, lo, hi);
    else
        order_bounds_kernel<false><<<grid_of(nq * 32), 256, 0, st>>>(nq, o->perm, o->n, D, S, queries, qbytes, QS, lo, hi);
    VB_CUDA(cudaGetLastError());
    count_launch();
    return VB_OK;
}

static DenseSrc dense_src(const Table& T) { return DenseSrc{T.d, T.stride, T.elem, T.dim, dense_words(T.elem, T.dim)}; }

static int dense_bounds(vb_order* o, const void* queries, int64_t nq, bool host, int64_t* out_lo, int64_t* out_hi) {
    const char* fn = host ? "vb_order_bounds" : "vb_order_bounds_dev";
    VB_TRY(require_init());
    VB_TRY(order_owner(fn, o, false));
    VB_REQUIRE(nq >= 0, "%s: negative query count %lld", fn, (long long)nq);
    if (nq == 0) return VB_OK;
    VB_REQUIRE(queries && out_lo && out_hi, "%s: null query / output buffers", fn);
    const Table& T = static_cast<const vb_table*>(o->owner)->t;
    const DenseSrc D = dense_src(T);
    const size_t qbytes = raw_row_bytes(T.elem, T.dim);
    if (!host) return launch_bounds(o, false, D, SparseSrc{}, (const uint8_t*)queries, qbytes, SparseSrc{}, nq, out_lo, out_hi);
    Context& c = ctx();
    Scratch sc;
    void *d_q, *d_out;
    VB_TRY(sc.take(qbytes * (size_t)nq, &d_q));
    VB_TRY(sc.take(16 * (size_t)nq, &d_out));
    int64_t* lo = (int64_t*)d_out;
    int64_t* hi = lo + nq;
    VB_CUDA(cudaMemcpyAsync(d_q, queries, qbytes * (size_t)nq, cudaMemcpyHostToDevice, c.stream));
    VB_TRY(launch_bounds(o, false, D, SparseSrc{}, (const uint8_t*)d_q, qbytes, SparseSrc{}, nq, lo, hi));
    VB_CUDA(cudaMemcpyAsync(out_lo, lo, 8 * (size_t)nq, cudaMemcpyDeviceToHost, c.stream));
    VB_CUDA(cudaMemcpyAsync(out_hi, hi, 8 * (size_t)nq, cudaMemcpyDeviceToHost, c.stream));
    VB_CUDA(cudaStreamSynchronize(c.stream));
    return VB_OK;
}

static int sparse_bounds(vb_order* o, int q_dim, int64_t nq, const int64_t* q_off, const int32_t* q_idx, const float* q_val, bool host,
                         int64_t* out_lo, int64_t* out_hi) {
    const char* fn = host ? "vb_sparse_order_bounds" : "vb_sparse_order_bounds_dev";
    VB_TRY(require_init());
    VB_TRY(order_owner(fn, o, true));
    VB_REQUIRE(nq >= 0, "%s: negative query count %lld", fn, (long long)nq);
    if (nq == 0) return VB_OK;
    VB_REQUIRE(out_lo && out_hi, "%s: null query / output buffers", fn);
    const SparseCsr T = sparse_table_csr(static_cast<const vb_sparse_table*>(o->owner));
    Scratch sc;
    SparseCsr Q;
    VB_TRY(sparse_queries_on_device(sc, T.dim, q_dim, nq, q_off, q_idx, q_val, host, &Q));
    const SparseSrc S{T.off, T.idx, T.val}, QS{Q.off, Q.idx, Q.val};
    if (!host) return launch_bounds(o, true, DenseSrc{}, S, nullptr, 0, QS, nq, out_lo, out_hi);
    Context& c = ctx();
    void* d_out;
    VB_TRY(sc.take(16 * (size_t)nq, &d_out));
    int64_t* lo = (int64_t*)d_out;
    int64_t* hi = lo + nq;
    VB_TRY(launch_bounds(o, true, DenseSrc{}, S, nullptr, 0, QS, nq, lo, hi));
    VB_CUDA(cudaMemcpyAsync(out_lo, lo, 8 * (size_t)nq, cudaMemcpyDeviceToHost, c.stream));
    VB_CUDA(cudaMemcpyAsync(out_hi, hi, 8 * (size_t)nq, cudaMemcpyDeviceToHost, c.stream));
    VB_CUDA(cudaStreamSynchronize(c.stream));
    return VB_OK;
}

static int order_read(const vb_order* o, bool host, int64_t* perm, int32_t* gor, int64_t* gstart) {
    const char* fn = host ? "vb_order_read" : "vb_order_read_dev";
    VB_TRY(require_init());
    VB_REQUIRE(o, "%s: null order", fn);
    const cudaMemcpyKind k = host ? cudaMemcpyDeviceToHost : cudaMemcpyDeviceToDevice;
    cudaStream_t st = ctx().stream;
    if (perm && o->n) VB_CUDA(cudaMemcpyAsync(perm, o->perm, 8 * (size_t)o->n, k, st));
    if (gor && o->n) VB_CUDA(cudaMemcpyAsync(gor, o->gor, 4 * (size_t)o->n, k, st));
    if (gstart) VB_CUDA(cudaMemcpyAsync(gstart, o->gstart, 8 * (size_t)(o->groups + 1), k, st));
    if (host) VB_CUDA(cudaStreamSynchronize(st));
    return VB_OK;
}

}  // namespace vb

extern "C" {

int vb_table_order_create(vb_table* t, vb_order** out) {
    const char* fn = "vb_table_order_create";
    VB_TRY(require_init());
    VB_REQUIRE(out, "%s: null order pointer", fn);
    VB_REQUIRE(t, "%s: null table", fn);
    VB_REQUIRE(t->t.elem == VB_VECTOR || t->t.elem == VB_HALFVEC,
               "%s: bit has no btree operator class in pgvector (bit columns use PostgreSQL's bit_ops)", fn);
    return order_create(fn, t, t->uid, false, t->t.dim, dense_src(t->t), SparseSrc{}, t->t.n, out);
}

int vb_sparse_table_order_create(vb_sparse_table* t, vb_order** out) {
    const char* fn = "vb_sparse_table_order_create";
    VB_TRY(require_init());
    VB_REQUIRE(out, "%s: null order pointer", fn);
    VB_REQUIRE(t, "%s: null table", fn);
    const SparseCsr T = sparse_table_csr(t);
    return order_create(fn, t, sparse_table_uid(t), true, T.dim, DenseSrc{}, SparseSrc{T.off, T.idx, T.val}, T.n, out);
}

int64_t vb_order_rows(const vb_order* o) { return o ? o->n : 0; }
int64_t vb_order_groups(const vb_order* o) { return o ? o->groups : 0; }
int64_t vb_order_passes(const vb_order* o) { return o ? o->passes : 0; }

int vb_order_read(const vb_order* o, int64_t* perm, int32_t* group_of_row, int64_t* group_start) {
    return order_read(o, true, perm, group_of_row, group_start);
}

int vb_order_read_dev(const vb_order* o, int64_t* perm_dev, int32_t* group_of_row_dev, int64_t* group_start_dev) {
    return order_read(o, false, perm_dev, group_of_row_dev, group_start_dev);
}

int vb_order_bounds(vb_order* o, const void* queries, int64_t nq, int64_t* out_lo, int64_t* out_hi) {
    return dense_bounds(o, queries, nq, true, out_lo, out_hi);
}

int vb_order_bounds_dev(vb_order* o, const void* queries_dev, int64_t nq, int64_t* out_lo_dev, int64_t* out_hi_dev) {
    return dense_bounds(o, queries_dev, nq, false, out_lo_dev, out_hi_dev);
}

int vb_sparse_order_bounds(vb_order* o, int q_dim, int64_t nq, const int64_t* q_off, const int32_t* q_idx, const float* q_val,
                           int64_t* out_lo, int64_t* out_hi) {
    return sparse_bounds(o, q_dim, nq, q_off, q_idx, q_val, true, out_lo, out_hi);
}

int vb_sparse_order_bounds_dev(vb_order* o, int q_dim, int64_t nq, const int64_t* q_off_dev, const int32_t* q_idx_dev,
                               const float* q_val_dev, int64_t* out_lo_dev, int64_t* out_hi_dev) {
    return sparse_bounds(o, q_dim, nq, q_off_dev, q_idx_dev, q_val_dev, false, out_lo_dev, out_hi_dev);
}

int vb_order_free(vb_order* o) {
    if (!o) return VB_OK;
    if (o->mem) {
        cudaStreamSynchronize(ctx().stream);
        cudaFree(o->mem);
    }
    delete o;
    return VB_OK;
}

}  // extern "C"
