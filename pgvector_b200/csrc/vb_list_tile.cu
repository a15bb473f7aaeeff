// vb_list_tile.cu -- the IVFFlat list scan for a BATCH of queries, list-major.
//
// The reference scans the probed lists once per query (GetScanItems, src/ivfscan.c:124-180: every
// tuple of every probed list goes through the distance function).  With B queries in flight each
// list is probed by B * probes / lists of them, so the per-query formulation (vb_scan*.cu) streams
// the same rows from HBM that many times -- 131 GB per 2048-query step for config B where the table
// is 6.1 GB.  Here the (query, list) pairs of a batch are grouped by list and one CTA computes the
// distances of a 256-row tile of a list against ALL queries that probe it: rows are read from HBM
// once per batch, the arithmetic (fp32, the same (x - q)^2 / x * q FMA chain per (row, query),
// accumulated sequentially over the dimensions) moves to the FMA pipe.  Distances land in the same
// per-query candidate run as the streaming scan writes them, so everything downstream (top-k by
// (distance, position), heap-id lookup) is unchanged.
//
// Tile: 256 rows x 32 queries per CTA, 8 warps.  Warp w owns rows 32w..32w+31 (one row per lane) against
// all queries of the sub-tile; the query loop is compiled for every count of query quads 1..8, so a group
// of 20 queries costs 20/32 of a full tile and every warp with rows stays busy.  Operands are staged
// through shared memory in steps of 16 dimensions, k-major, double buffered with register prefetch; the
// inner loop works on pairs of queries: (x, x) + (-q0, -q1), squared and accumulated, each lane rounded as
// the scalar instruction, so each (row, query) distance is the plain sequential fmaf chain over the dimensions.
//
// Bound: fp32 issue (2 instructions per pair for L2, 1 for inner product); HBM traffic is
// one pass over the probed lists per batch.
#include "vb_common.cuh"

#include <algorithm>

namespace vb {

constexpr int LT_ROWS = 256;
constexpr int LT_Q = 32;
constexpr int LT_KS = 16;                 // dimensions per staging step
constexpr int LT_THREADS = 256;
constexpr int LT_XP = LT_ROWS + 2;        // line of one dimension across the row tile; +2 words makes the transposing stores conflict-free

struct LtArgs {
    const uint8_t* rows;
    size_t stride;
    const uint8_t* qimg;
    size_t qstride;
    const ListTile* tiles;
    const int64_t* list_off;
    const int32_t* grp_begin;
    const int32_t* grp_cnt;
    const int32_t* pair_q;
    const int64_t* pair_out;
    float* out;
    int words;   // padded dimension count (elements per row including the zero padding)
};

__device__ __forceinline__ unsigned long long lt_pack(float lo, float hi) {
    unsigned long long r;
    asm("mov.b64 %0, {%1, %2};" : "=l"(r) : "f"(lo), "f"(hi));
    return r;
}
__device__ __forceinline__ void lt_unpack(unsigned long long v, float& lo, float& hi) {
    asm("mov.b64 {%0, %1}, %2;" : "=f"(lo), "=f"(hi) : "l"(v));
}
// two fp32 lanes of a packed pair, each rounded as the scalar instruction (never contracted: the distance of every
// (row, query) pair is the plain sequential fmaf chain)
__device__ __forceinline__ unsigned long long lt_add2(unsigned long long a, unsigned long long b) {
    float a0, a1, b0, b1;
    lt_unpack(a, a0, a1);
    lt_unpack(b, b0, b1);
    return lt_pack(__fadd_rn(a0, b0), __fadd_rn(a1, b1));
}
__device__ __forceinline__ unsigned long long lt_fma2(unsigned long long a, unsigned long long b, unsigned long long c) {
    float a0, a1, b0, b1, c0, c1;
    lt_unpack(a, a0, a1);
    lt_unpack(b, b0, b1);
    lt_unpack(c, c0, c1);
    return lt_pack(__fmaf_rn(a0, b0, c0), __fmaf_rn(a1, b1, c1));
}

// 4 consecutive elements of a row starting at element e (zero past the padded dimension count)
template <int ELEM>
__device__ __forceinline__ float4 lt_load4(const uint8_t* row, int e, int words) {
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (e < words) {
        if (ELEM == VB_VECTOR) {
            v = __ldg(reinterpret_cast<const float4*>(row) + (e >> 2));
        } else {
            const uint2 h = __ldg(reinterpret_cast<const uint2*>(row) + (e >> 2));
            const float2 a = __half22float2(*reinterpret_cast<const __half2*>(&h.x));
            const float2 b = __half22float2(*reinterpret_cast<const __half2*>(&h.y));
            v = make_float4(a.x, a.y, b.x, b.y);
        }
    }
    return v;
}

// one staging step (16 dimensions) of one row against the first 4 * NQ4 queries of the sub-tile
template <int KIND, int NQ4>
__device__ __forceinline__ void lt_step(const float (*__restrict__ xs)[LT_XP], const float (*__restrict__ qs)[LT_Q], int row,
                                        unsigned long long (&acc)[LT_Q / 2]) {
#pragma unroll
    for (int kk = 0; kk < LT_KS; ++kk) {
        const float x = xs[kk][row];
        const unsigned long long xx = lt_pack(x, x);
#pragma unroll
        for (int jq = 0; jq < NQ4; ++jq) {
            const ulonglong2 qv = *reinterpret_cast<const ulonglong2*>(&qs[kk][4 * jq]);
            if (KIND == 0) {
                const unsigned long long d0 = lt_add2(xx, qv.x);   // x + (-q)
                const unsigned long long d1 = lt_add2(xx, qv.y);
                acc[2 * jq] = lt_fma2(d0, d0, acc[2 * jq]);
                acc[2 * jq + 1] = lt_fma2(d1, d1, acc[2 * jq + 1]);
            } else {
                acc[2 * jq] = lt_fma2(xx, qv.x, acc[2 * jq]);
                acc[2 * jq + 1] = lt_fma2(xx, qv.y, acc[2 * jq + 1]);
            }
        }
    }
}

// KIND 0: sum (x - q)^2      KIND 1: -sum x * q
template <int ELEM, int KIND>
__global__ void __launch_bounds__(LT_THREADS, 2) list_tile_kernel(LtArgs a) {
    const ListTile t = a.tiles[blockIdx.x];
    const int cnt = a.grp_cnt[t.list];
    if (cnt == 0) return;   // list not probed by this batch

    __shared__ __align__(16) float Xs[2][LT_KS][LT_XP];
    __shared__ __align__(16) float Qs[2][LT_KS][LT_Q];   // negated for L2
    __shared__ int32_t s_q[LT_Q];
    __shared__ int64_t s_out[LT_Q];

    const int tid = threadIdx.x, warp = tid / 32, lane = tid % 32;
    const int gb = a.grp_begin[t.list];
    const int64_t row_in_list0 = t.row_begin - a.list_off[t.list];
    const int words = a.words;
    const int nsteps = (words + LT_KS - 1) / LT_KS;
    const int my_row = warp * 32 + lane;
    const bool has_rows = warp * 32 < t.n_rows;   // warp-uniform

    // staging roles: 4 threads per row (one 4-element piece each), 64 rows per pass, 4 passes
    const int sp = tid % 4;
    const uint8_t* xrow[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        const int r = min(tid / 4 + 64 * j, t.n_rows - 1);
        xrow[j] = a.rows + (size_t)(t.row_begin + r) * a.stride;
    }

    for (int q0 = 0; q0 < cnt; q0 += LT_Q) {
        const int nqt = min(LT_Q, cnt - q0);
        const int nq4 = (nqt + 3) / 4;
        __syncthreads();   // the previous query sub-tile is done with s_q / s_out and both buffers
        if (tid < LT_Q) {
            const int s = gb + q0 + min(tid, nqt - 1);
            s_q[tid] = a.pair_q[s];
            s_out[tid] = a.pair_out[s];
        }
        __syncthreads();
        const float* qrow = reinterpret_cast<const float*>(a.qimg + (size_t)s_q[(tid / 4) % LT_Q] * a.qstride);

        unsigned long long acc[LT_Q / 2];
#pragma unroll
        for (int j = 0; j < LT_Q / 2; ++j) acc[j] = 0ull;

        float4 xr[4], qr;
        auto fetch = [&](int ks) {
            const int e = ks * LT_KS + 4 * sp;
#pragma unroll
            for (int j = 0; j < 4; ++j) xr[j] = lt_load4<ELEM>(xrow[j], e, words);
            qr = make_float4(0.f, 0.f, 0.f, 0.f);
            if (tid < 4 * LT_Q && e < words) qr = __ldg(reinterpret_cast<const float4*>(qrow) + (e >> 2));
        };
        auto stage = [&](int buf) {
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const int r = tid / 4 + 64 * j;
                Xs[buf][4 * sp + 0][r] = xr[j].x;
                Xs[buf][4 * sp + 1][r] = xr[j].y;
                Xs[buf][4 * sp + 2][r] = xr[j].z;
                Xs[buf][4 * sp + 3][r] = xr[j].w;
            }
            if (tid < 4 * LT_Q) {
                const int qi = tid / 4;
                const float s = KIND == 0 ? -1.f : 1.f;
                Qs[buf][4 * sp + 0][qi] = s * qr.x;
                Qs[buf][4 * sp + 1][qi] = s * qr.y;
                Qs[buf][4 * sp + 2][qi] = s * qr.z;
                Qs[buf][4 * sp + 3][qi] = s * qr.w;
            }
        };

        fetch(0);
        stage(0);
        __syncthreads();
        for (int ks = 0; ks < nsteps; ++ks) {
            const int buf = ks & 1;
            if (ks + 1 < nsteps) fetch(ks + 1);
            if (has_rows) {
                switch (nq4) {   // block-uniform
                    case 1: lt_step<KIND, 1>(Xs[buf], Qs[buf], my_row, acc); break;
                    case 2: lt_step<KIND, 2>(Xs[buf], Qs[buf], my_row, acc); break;
                    case 3: lt_step<KIND, 3>(Xs[buf], Qs[buf], my_row, acc); break;
                    case 4: lt_step<KIND, 4>(Xs[buf], Qs[buf], my_row, acc); break;
                    case 5: lt_step<KIND, 5>(Xs[buf], Qs[buf], my_row, acc); break;
                    case 6: lt_step<KIND, 6>(Xs[buf], Qs[buf], my_row, acc); break;
                    case 7: lt_step<KIND, 7>(Xs[buf], Qs[buf], my_row, acc); break;
                    default: lt_step<KIND, 8>(Xs[buf], Qs[buf], my_row, acc); break;
                }
            }
            if (ks + 1 < nsteps) stage(buf ^ 1);
            __syncthreads();
        }

        if (my_row < t.n_rows) {
            // lanes = consecutive rows: one coalesced 128-byte store per (warp, query)
#pragma unroll
            for (int j = 0; j < LT_Q / 2; ++j) {
                if (2 * j >= nqt) break;
                float lo, hi;
                lt_unpack(acc[j], lo, hi);
                if (KIND == 1) {
                    lo = -lo;
                    hi = -hi;
                }
                a.out[s_out[2 * j] + row_in_list0 + my_row] = lo;
                if (2 * j + 1 < nqt) a.out[s_out[2 * j + 1] + row_in_list0 + my_row] = hi;
            }
        }
    }
}

// ----------------------------------------------------------------------------- grouping the (query, probe) pairs by list

__global__ void lt_count_kernel(const int32_t* __restrict__ probe_lists, int64_t n_pairs, int32_t* __restrict__ cnt) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= n_pairs) return;
    const int l = probe_lists[i];
    if (l >= 0) atomicAdd(&cnt[l], 1);
}

// exclusive prefix sum over the lists (one CTA; the list count is at most a few tens of thousands)
__global__ void __launch_bounds__(1024) lt_scan_kernel(const int32_t* __restrict__ cnt, int n, int32_t* __restrict__ begin) {
    __shared__ int32_t warp_sum[32];
    __shared__ int32_t carry;
    if (threadIdx.x == 0) carry = 0;
    __syncthreads();
    const int lane = threadIdx.x % 32, warp = threadIdx.x / 32;
    for (int base = 0; base < n; base += 1024) {
        const int i = base + threadIdx.x;
        const int32_t v = i < n ? cnt[i] : 0;
        int32_t s = v;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int32_t u = __shfl_up_sync(0xffffffffu, s, o);
            if (lane >= o) s += u;
        }
        if (lane == 31) warp_sum[warp] = s;
        __syncthreads();
        if (warp == 0) {
            int32_t w = warp_sum[lane];
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const int32_t u = __shfl_up_sync(0xffffffffu, w, o);
                if (lane >= o) w += u;
            }
            warp_sum[lane] = w;
        }
        __syncthreads();
        const int32_t before = carry + (warp ? warp_sum[warp - 1] : 0);
        if (i < n) begin[i] = before + s - v;
        __syncthreads();
        if (threadIdx.x == 1023) carry = before + s;
        __syncthreads();
    }
}

// exclusive prefix sum by one CTA of 1024 threads (shared scratch supplied by the caller)
__device__ __forceinline__ void lt_block_scan(const int32_t* __restrict__ cnt, int n, int32_t* __restrict__ begin, int32_t* warp_sum,
                                              int32_t* carry) {
    if (threadIdx.x == 0) *carry = 0;
    __syncthreads();
    const int lane = threadIdx.x % 32, warp = threadIdx.x / 32;
    for (int base = 0; base < n; base += 1024) {
        const int i = base + threadIdx.x;
        const int32_t v = i < n ? cnt[i] : 0;
        int32_t s = v;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int32_t u = __shfl_up_sync(0xffffffffu, s, o);
            if (lane >= o) s += u;
        }
        if (lane == 31) warp_sum[warp] = s;
        __syncthreads();
        if (warp == 0) {
            int32_t w = warp_sum[lane];
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const int32_t u = __shfl_up_sync(0xffffffffu, w, o);
                if (lane >= o) w += u;
            }
            warp_sum[lane] = w;
        }
        __syncthreads();
        const int32_t before = *carry + (warp ? warp_sum[warp - 1] : 0);
        if (i < n) begin[i] = before + s - v;
        __syncthreads();
        if (threadIdx.x == 1023) *carry = before + s;
        __syncthreads();
    }
}

// Counting, both prefix sums and the query-tile numbering of a moderate batch in ONE launch of one CTA -- counters in
// shared memory (instead of a memset and four kernels with global atomics; a 2048-query batch has 20 480 pairs = 20 per
// thread); lt_scatter_kernel then places the pairs
__global__ void __launch_bounds__(1024) lt_group_kernel(const int32_t* __restrict__ probe_lists, int n_pairs, int probes,
                                                        const int32_t* __restrict__ cand_off, int64_t cap, int n_lists, int gt_rows,
                                                        int32_t* __restrict__ cnt, int32_t* __restrict__ begin,
                                                        int32_t* __restrict__ gt_begin, int32_t* __restrict__ cursor) {
    extern __shared__ int32_t lg_smem[];
    int32_t* scnt = lg_smem;             // [n_lists]
    int32_t* scur = lg_smem + n_lists;   // [n_lists] begin, then the running cursor, then the tile counts
    __shared__ int32_t warp_sum[32];
    __shared__ int32_t carry;
    for (int i = threadIdx.x; i < n_lists; i += 1024) scnt[i] = 0;
    __syncthreads();
    // (8 independent loads per thread in flight: one CTA walking 20 k pairs one dependent load at a time took 42 us)
    constexpr int U = 8;
    for (int i0 = threadIdx.x; i0 < n_pairs; i0 += 1024 * U) {
        int l[U];
#pragma unroll
        for (int u = 0; u < U; ++u) l[u] = i0 + u * 1024 < n_pairs ? probe_lists[i0 + u * 1024] : -1;
#pragma unroll
        for (int u = 0; u < U; ++u)
            if (l[u] >= 0) atomicAdd(&scnt[l[u]], 1);
    }
    __syncthreads();
    lt_block_scan(scnt, n_lists, scur, warp_sum, &carry);
    for (int i = threadIdx.x; i < n_lists; i += 1024) {
        cnt[i] = scnt[i];
        begin[i] = scur[i];
    }
    __syncthreads();
    // (the scatter is lt_scatter_kernel's: 80 k scattered 4-byte stores through ONE SM's store path took ~40 us of this
    // kernel's 48; spread over the GPU they take a few)
    for (int i = threadIdx.x; i < n_lists; i += 1024) cursor[i] = 0;
    if (gt_rows > 0) {
        __syncthreads();
        for (int i = threadIdx.x; i < n_lists; i += 1024) scur[i] = (scnt[i] + gt_rows - 1) / gt_rows;
        __syncthreads();
        lt_block_scan(scur, n_lists, gt_begin, warp_sum, &carry);
    }
}

__global__ void lt_scatter_kernel(const int32_t* __restrict__ probe_lists, int64_t n_pairs, int probes,
                                  const int32_t* __restrict__ cand_off, int64_t cap, const int32_t* __restrict__ begin,
                                  int32_t* __restrict__ cursor, int32_t* __restrict__ pair_q, int64_t* __restrict__ pair_out,
                                  int32_t* __restrict__ pair_list, int32_t* __restrict__ pair_sbase, int64_t cap_s) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= n_pairs) return;
    const int l = probe_lists[i];
    if (l < 0) return;
    const int64_t q = i / probes;
    const int p = (int)(i % probes);
    const int slot = begin[l] + atomicAdd(&cursor[l], 1);
    pair_q[slot] = (int32_t)q;
    pair_out[slot] = q * cap + cand_off[q * (probes + 1) + p];
    pair_list[slot] = l;
    if (cap_s) pair_sbase[slot] = (int32_t)slab_base(q, cap_s, cand_off[q * (probes + 1) + p], p);
}

// tiles[l] = ceil(cnt[l] / rows_per_tile): the number of query tiles of each list (input of a second prefix sum)
__global__ void lt_tiles_kernel(const int32_t* __restrict__ cnt, int n, int rows_per_tile, int32_t* __restrict__ tiles) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) tiles[i] = (cnt[i] + rows_per_tile - 1) / rows_per_tile;
}

bool list_major_supported(int elem, int key_metric) {
    return (elem == VB_VECTOR || elem == VB_HALFVEC) && (key_metric == VB_L2_SQUARED || key_metric == VB_NEG_IP);
}

// Group the (query, probe) pairs of a batch by list.  gt_rows > 0 additionally numbers the query tiles of
// gt_rows queries over all lists (tensor-core path: one packed B tile per query tile).
int build_query_groups(Scratch& sc, const int32_t* d_lists, int64_t nq, int probes, const int32_t* cand_off, int64_t cap, int n_lists, int gt_rows,
                       QueryGroups* g, int64_t cap_s) {
    Context& c = ctx();
    cudaStream_t s = c.stream;
    const int64_t n_pairs = nq * probes;
    VB_REQUIRE(n_pairs < (int64_t)INT32_MAX, "too many (query, probe) pairs");
    void* d_ws;
    VB_REQUIRE(nq * cap_s < (int64_t)INT32_MAX, "slab-minimum array too large (%lld queries)", (long long)nq);
    const size_t ints = (size_t)n_lists * 5 + (size_t)n_pairs * 3;
    VB_TRY(sc.take(sizeof(int64_t) * (size_t)n_pairs + sizeof(int32_t) * ints + 64, &d_ws));
    g->pair_out = (int64_t*)d_ws;
    g->pair_q = (int32_t*)(g->pair_out + n_pairs);
    g->pair_list = g->pair_q + n_pairs;
    g->cnt = g->pair_list + n_pairs;
    int32_t* cursor = g->cnt + n_lists;
    g->begin = cursor + n_lists;
    int32_t* tiles = g->begin + n_lists;
    g->gt_begin = tiles + n_lists;
    g->pair_sbase = g->gt_begin + n_lists;
    g->n_pairs = n_pairs;
    if (n_pairs <= 131072 && n_lists <= 8192) {
        static bool attr_set = false;
        if (!attr_set) {
            VB_CUDA(cudaFuncSetAttribute(lt_group_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 8192 * 8));
            attr_set = true;
        }
        lt_group_kernel<<<1, 1024, sizeof(int32_t) * 2 * (size_t)n_lists, s>>>(d_lists, (int)n_pairs, probes, cand_off, cap, n_lists, gt_rows, g->cnt,
                                                                            g->begin, g->gt_begin, cursor);
        lt_scatter_kernel<<<(unsigned)((n_pairs + 255) / 256), 256, 0, s>>>(d_lists, n_pairs, probes, cand_off, cap, g->begin, cursor, g->pair_q,
                                                                          g->pair_out, g->pair_list, g->pair_sbase, cap_s);
        VB_CUDA(cudaGetLastError());
        count_launch(2);
        return VB_OK;
    }
    VB_CUDA(cudaMemsetAsync(g->cnt, 0, sizeof(int32_t) * (size_t)n_lists * 2, s));
    const unsigned gp = (unsigned)((n_pairs + 255) / 256);
    lt_count_kernel<<<gp, 256, 0, s>>>(d_lists, n_pairs, g->cnt);
    lt_scan_kernel<<<1, 1024, 0, s>>>(g->cnt, n_lists, g->begin);
    lt_scatter_kernel<<<gp, 256, 0, s>>>(d_lists, n_pairs, probes, cand_off, cap, g->begin, cursor, g->pair_q, g->pair_out, g->pair_list,
                                         g->pair_sbase, cap_s);
    count_launch(3);
    if (gt_rows > 0) {
        lt_tiles_kernel<<<(unsigned)((n_lists + 255) / 256), 256, 0, s>>>(g->cnt, n_lists, gt_rows, tiles);
        lt_scan_kernel<<<1, 1024, 0, s>>>(tiles, n_lists, g->gt_begin);
        count_launch(2);
    }
    VB_CUDA(cudaGetLastError());
    return VB_OK;
}

int launch_list_major(const Table& rows, int key_metric, const void* qimg, size_t qstride, int64_t nq, const int32_t* d_lists,
                      int probes, const int32_t* cand_off, int64_t cap, const int64_t* d_list_off, int n_lists,
                      const ListTile* d_tiles, int n_tiles, float* out) {
    VB_REQUIRE(list_major_supported(rows.elem, key_metric), "list-major scan: unsupported element type / metric");
    if (nq <= 0 || n_tiles <= 0) return VB_OK;
    cudaStream_t s = ctx().stream;
    Scratch sc;
    QueryGroups g{};
    VB_TRY(build_query_groups(sc, d_lists, nq, probes, cand_off, cap, n_lists, 0, &g));
    int32_t* begin = g.begin;
    int32_t* cnt = g.cnt;
    int32_t* pair_q = g.pair_q;
    int64_t* pair_out = g.pair_out;

    LtArgs a{};
    a.rows = rows.d;
    a.stride = rows.stride;
    a.qimg = (const uint8_t*)qimg;
    a.qstride = qstride;
    a.tiles = d_tiles;
    a.list_off = d_list_off;
    a.grp_begin = begin;
    a.grp_cnt = cnt;
    a.pair_q = pair_q;
    a.pair_out = pair_out;
    a.out = out;
    a.words = (int)(rows.elem == VB_HALFVEC ? rows.stride / 2 : rows.stride / 4);
    const int kind = key_metric == VB_L2_SQUARED ? 0 : 1;
    if (rows.elem == VB_VECTOR) {
        if (kind == 0) list_tile_kernel<VB_VECTOR, 0><<<n_tiles, LT_THREADS, 0, s>>>(a);
        else list_tile_kernel<VB_VECTOR, 1><<<n_tiles, LT_THREADS, 0, s>>>(a);
    } else {
        if (kind == 0) list_tile_kernel<VB_HALFVEC, 0><<<n_tiles, LT_THREADS, 0, s>>>(a);
        else list_tile_kernel<VB_HALFVEC, 1><<<n_tiles, LT_THREADS, 0, s>>>(a);
    }
    VB_CUDA(cudaGetLastError());
    count_launch();
    return VB_OK;
}

int list_tile_rows() { return LT_ROWS; }

}  // namespace vb
