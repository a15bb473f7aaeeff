// vb_agg.cu -- avg(vector), sum(vector), avg(halfvec), sum(halfvec) over a resident table, with GROUP BY
// (sql/vector.sql:163-198, 607-642), bit-identical to the reference's serial plan and to its partial-aggregate plans.
//
// The plan (include/vecb200.h, vb_table_aggregate): each group's rows in ascending row number are cut into runs of R
// consecutive rows; a run's state is the transition function over its rows in order, the group's state the run states
// combined left to right, and the result the final function of that.  The device follows it exactly:
//   - grouped calls sort the (group, row) pairs stably (CUB radix sort on the group, rows as values), mark each group's
//     range of the sorted list and lay out its runs (agg_keys_kernel, agg_bounds_kernel, agg_nruns_kernel + a scan);
//     without groups run r is simply rows [rR, (r+1)R);
//   - agg_run_kernel: one thread per (run, column slot) walks its run's rows in order.  A slot is one fp32 column or
//     two fp16 columns (half2), so each warp step reads a 128-byte span of one row; the loads of the next AGG_UNROLL
//     rows are issued before the dependent adds of the current ones;
//   - agg_final_kernel: one thread per (group, column) combines the group's run states left to right and applies the
//     final function, writing the result, the count and (avg) the float8 transition state.
// Every add is the reference's operation with explicit rounding (__dadd_rn / __fadd_rn, the fp16 add as an fp32 add
// rounded to half, which is the correctly rounded half sum since 24 >= 2 * 11 + 2), so nothing is contracted and the
// result does not depend on the launch configuration.
#include "vb_common.cuh"

#include <cub/cub.cuh>

#include <algorithm>

namespace vb {

constexpr int AGG_THREADS = 256;
constexpr int AGG_UNROLL = 8;     // rows per step of a thread; the next step's loads are in flight during a step's adds

// the fixed-shape description of the runs both kernels walk
struct RunPlan {
    int64_t n;                    // table rows
    int64_t R;                    // run length (grouped: as given, 0 = whole group; ungrouped: the effective length >= 1)
    int64_t nruns;                // ungrouped: the number of runs; grouped: an upper bound (the exact count is run_begin[ngroups])
    int ngroups;
    const int32_t* row_list;      // grouped: table rows sorted by (group, row)
    const int32_t* gstart;        // grouped: [ngroups] first position of the group in row_list
    const int32_t* gend;          // grouped: [ngroups] one past its last position (0 / 0 for an empty group)
    const int32_t* run_begin;     // grouped: [ngroups + 1] first run of each group; run_begin[ngroups] = runs
};

// (group, first position, length) of run `run`; false when the run does not exist (grouped bound)
template <bool GROUPED>
__device__ __forceinline__ bool locate_run(const RunPlan& p, int64_t run, int* g, int64_t* first, int64_t* len) {
    if (!GROUPED) {
        *g = 0;
        *first = run * p.R;
        *len = min(p.R, p.n - *first);
        return true;
    }
    if (run >= p.run_begin[p.ngroups]) return false;
    int lo = 0, hi = p.ngroups;          // largest g with run_begin[g] <= run (empty groups share their successor's start)
    while (hi - lo > 1) {
        const int mid = (lo + hi) >> 1;
        if (p.run_begin[mid] <= run) lo = mid; else hi = mid;
    }
    const int64_t k = run - p.run_begin[lo];
    const int64_t cnt = (int64_t)p.gend[lo] - p.gstart[lo];
    *g = lo;
    *first = p.gstart[lo] + k * p.R;
    *len = p.R == 0 ? cnt : min(p.R, cnt - k * p.R);
    return true;
}

__global__ void agg_keys_kernel(const int32_t* __restrict__ group_of_row, int64_t n, int ngroups, uint32_t* __restrict__ keys,
                                int32_t* __restrict__ rows) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int32_t g = group_of_row[i];
    keys[i] = (g >= 0 && g < ngroups) ? (uint32_t)g : (uint32_t)ngroups;   // ids outside [0, ngroups) sort last and are dropped
    rows[i] = (int32_t)i;
}

__global__ void agg_bounds_kernel(const uint32_t* __restrict__ keys, int64_t n, int ngroups, int32_t* __restrict__ gstart,
                                  int32_t* __restrict__ gend) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint32_t k = keys[i];
    if (k >= (uint32_t)ngroups) return;
    if (i == 0 || keys[i - 1] != k) gstart[k] = (int32_t)i;
    if (i == n - 1 || keys[i + 1] != k) gend[k] = (int32_t)(i + 1);
}

__global__ void agg_nruns_kernel(const int32_t* __restrict__ gstart, const int32_t* __restrict__ gend, int ngroups, int64_t R,
                                 int32_t* __restrict__ nruns) {
    const int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (g > ngroups) return;
    if (g == ngroups) {
        nruns[g] = 0;
        return;
    }
    const int64_t cnt = (int64_t)gend[g] - gstart[g];
    nruns[g] = (int32_t)(cnt == 0 ? 0 : R == 0 ? 1 : (cnt + R - 1) / R);
}

// element loads: one fp32 column, or two fp16 columns as their fp32 values (exact widening, HalfToFloat4)
template <int ELEM>
struct Slot;
template <>
struct Slot<VB_VECTOR> {
    static constexpr int COLS = 1;
    float v[1];
    __device__ __forceinline__ void load(const uint8_t* p) { v[0] = __ldg((const float*)p); }
};
template <>
struct Slot<VB_HALFVEC> {
    static constexpr int COLS = 2;
    float v[2];
    __device__ __forceinline__ void load(const uint8_t* p) {
        const __half2 h = __ldg((const __half2*)p);
        v[0] = __low2float(h);
        v[1] = __high2float(h);
    }
};

// sum(halfvec)'s add: halfvec_add rounds every element to fp16 (src/halfvec.c:780-788)
template <int ELEM>
__device__ __forceinline__ float sum_add(float a, float b) {
    const float s = __fadd_rn(a, b);
    return ELEM == VB_HALFVEC ? __half2float(__float2half_rn(s)) : s;
}

// One thread per (run, column slot): the run state of its columns.  avg: vector_accum / halfvec_accum from INITCOND
// '{0}' (the first row sets s = (double) x, later rows add (double) x in float8; src/vector.c:1148-1204,
// src/halfvec.c:1104-1160); states[run][col] is s (the count is the run length).  sum: the first row is the state,
// later rows are added by vector_add / halfvec_add (src/vector.c:824-852, src/halfvec.c:764-798); a run state that
// overflowed sets *flag (rows are finite, so an infinite partial sum stays infinite to the run's end).
template <int ELEM, int AGG, bool GROUPED>
__global__ void __launch_bounds__(AGG_THREADS) agg_run_kernel(const uint8_t* __restrict__ rows, size_t stride, int dim, int nslots,
                                                             RunPlan p, void* __restrict__ states, int* __restrict__ flag) {
    using S = Slot<ELEM>;
    constexpr int esize = ELEM == VB_VECTOR ? 4 : 2;
    const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t run = t / nslots;
    const int slot = (int)(t - run * nslots);
    if (run >= p.nruns) return;
    int g;
    int64_t first, len;
    if (!locate_run<GROUPED>(p, run, &g, &first, &len)) return;
    const uint8_t* base = rows + (size_t)slot * S::COLS * esize;
    auto row_ptr = [&](int64_t j) -> const uint8_t* {
        const int64_t r = GROUPED ? (int64_t)__ldg(p.row_list + first + j) : first + j;
        return base + (size_t)r * stride;
    };
    using Acc = typename std::conditional<AGG == VB_AGG_AVG, double, float>::type;
    Acc s[S::COLS];
    {
        S x;
        x.load(row_ptr(0));
#pragma unroll
        for (int c = 0; c < S::COLS; ++c) s[c] = (Acc)x.v[c];   // avg: (double) x, not 0.0 + x, so a -0 survives
    }
    // software-pipelined: the loads of the next AGG_UNROLL rows are issued before the adds of the current ones
    S x[AGG_UNROLL];
#pragma unroll
    for (int u = 0; u < AGG_UNROLL; ++u)
        if (1 + u < len) x[u].load(row_ptr(1 + u));
    for (int64_t j0 = 1; j0 < len; j0 += AGG_UNROLL) {
        S y[AGG_UNROLL];
#pragma unroll
        for (int u = 0; u < AGG_UNROLL; ++u)
            if (j0 + AGG_UNROLL + u < len) y[u].load(row_ptr(j0 + AGG_UNROLL + u));
#pragma unroll
        for (int u = 0; u < AGG_UNROLL; ++u)
            if (j0 + u < len) {
#pragma unroll
                for (int c = 0; c < S::COLS; ++c) {
                    if (AGG == VB_AGG_AVG)
                        s[c] = __dadd_rn(s[c], (double)x[u].v[c]);
                    else
                        s[c] = sum_add<ELEM>(s[c], x[u].v[c]);
                }
            }
#pragma unroll
        for (int u = 0; u < AGG_UNROLL; ++u) x[u] = y[u];
    }
    bool inf = false;
#pragma unroll
    for (int c = 0; c < S::COLS; ++c) {
        const int col = slot * S::COLS + c;
        if (col < dim) {
            ((Acc*)states)[run * dim + col] = s[c];
            if (AGG == VB_AGG_SUM) inf |= isinf(s[c]);
        }
    }
    if (inf) *flag = 1;
}

// One thread per (group, column): the run states of the group combined left to right (avg: vector_combine,
// src/vector.c:1209-1284, sums and counts added; sum: the transition's add), then the final function (avg:
// (float) (s / n), Float4ToHalf of it for halfvec, src/vector.c:1289-1318, src/halfvec.c:1165-1194; sum: the state).
// An empty group gives count 0 and a zero-filled result and state.
template <int ELEM, int AGG, bool GROUPED>
__global__ void __launch_bounds__(AGG_THREADS) agg_final_kernel(int dim, RunPlan p, const void* __restrict__ states,
                                                               void* __restrict__ out, int64_t* __restrict__ out_counts,
                                                               double* __restrict__ out_state, int* __restrict__ flag) {
    using Acc = typename std::conditional<AGG == VB_AGG_AVG, double, float>::type;
    const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t g = t / dim;
    const int col = (int)(t - g * dim);
    if (g >= p.ngroups) return;
    int64_t rb, re, cnt;
    if (GROUPED) {
        rb = p.run_begin[g];
        re = p.run_begin[g + 1];
        cnt = (int64_t)p.gend[g] - p.gstart[g];
    } else {
        rb = 0;
        re = p.nruns;
        cnt = p.n;
    }
    const Acc* st = (const Acc*)states + col;
    Acc s = 0;
    if (cnt > 0) {
        s = st[rb * dim];
        for (int64_t r0 = rb + 1; r0 < re; r0 += AGG_UNROLL) {
            Acc x[AGG_UNROLL];
#pragma unroll
            for (int u = 0; u < AGG_UNROLL; ++u)
                if (r0 + u < re) x[u] = st[(r0 + u) * dim];
#pragma unroll
            for (int u = 0; u < AGG_UNROLL; ++u)
                if (r0 + u < re) {
                    if (AGG == VB_AGG_AVG)
                        s = __dadd_rn(s, (double)x[u]);
                    else
                        s = sum_add<ELEM>(s, (float)x[u]);
                }
        }
    }
    const int64_t o = g * dim + col;
    if (AGG == VB_AGG_AVG) {
        const float m = cnt > 0 ? __double2float_rn(__ddiv_rn((double)s, (double)cnt)) : 0.f;
        if (ELEM == VB_VECTOR)
            ((float*)out)[o] = m;
        else
            ((__half*)out)[o] = __float2half_rn(m);
        if (out_state) {
            out_state[g * (dim + 1) + 1 + col] = (double)s;
            if (col == 0) out_state[g * (dim + 1)] = (double)cnt;
        }
    } else {
        if (ELEM == VB_VECTOR)
            ((float*)out)[o] = (float)s;
        else
            ((__half*)out)[o] = __float2half_rn((float)s);
        if (cnt > 0 && isinf((float)s)) *flag = 1;
    }
    if (col == 0) out_counts[g] = cnt;
}

template <int ELEM, int AGG, bool GROUPED>
int launch_agg(const Table& tb, const RunPlan& p, void* states, void* out, int64_t* counts, double* state, int* flag) {
    Context& c = ctx();
    constexpr int cols = ELEM == VB_VECTOR ? 1 : 2;
    const int nslots = (tb.dim + cols - 1) / cols;
    const int64_t threads = p.nruns * nslots;
    if (threads > 0) {
        agg_run_kernel<ELEM, AGG, GROUPED><<<(unsigned)((threads + AGG_THREADS - 1) / AGG_THREADS), AGG_THREADS, 0, c.stream>>>(
            tb.d, tb.stride, tb.dim, nslots, p, states, flag);
        VB_CUDA(cudaGetLastError());
        count_launch();
    }
    const int64_t fthreads = (int64_t)p.ngroups * tb.dim;
    agg_final_kernel<ELEM, AGG, GROUPED><<<(unsigned)((fthreads + AGG_THREADS - 1) / AGG_THREADS), AGG_THREADS, 0, c.stream>>>(
        tb.dim, p, states, out, counts, state, flag);
    VB_CUDA(cudaGetLastError());
    count_launch();
    return VB_OK;
}

template <bool GROUPED>
int dispatch_agg(int elem, int agg, const Table& tb, const RunPlan& p, void* states, void* out, int64_t* counts, double* state,
                 int* flag) {
    if (elem == VB_VECTOR)
        return agg == VB_AGG_AVG ? launch_agg<VB_VECTOR, VB_AGG_AVG, GROUPED>(tb, p, states, out, counts, state, flag)
                                 : launch_agg<VB_VECTOR, VB_AGG_SUM, GROUPED>(tb, p, states, out, counts, state, flag);
    return agg == VB_AGG_AVG ? launch_agg<VB_HALFVEC, VB_AGG_AVG, GROUPED>(tb, p, states, out, counts, state, flag)
                             : launch_agg<VB_HALFVEC, VB_AGG_SUM, GROUPED>(tb, p, states, out, counts, state, flag);
}

static inline size_t al256(size_t b) { return (b + 255) & ~(size_t)255; }

static int aggregate_impl(vb_table* t, int agg, const int32_t* group_of_row, int ngroups, int64_t run_rows, void* out,
                   int64_t* out_counts, double* out_state, bool host) {
    const char* fn = host ? "vb_table_aggregate" : "vb_table_aggregate_dev";
    VB_TRY(require_init());
    VB_REQUIRE(t, "%s: null table", fn);
    VB_REQUIRE(agg == VB_AGG_AVG || agg == VB_AGG_SUM, "%s: unknown aggregate %d (VB_AGG_AVG or VB_AGG_SUM)", fn, agg);
    const Table& tb = t->t;
    VB_REQUIRE(tb.elem == VB_VECTOR || tb.elem == VB_HALFVEC, "%s: %s has no aggregates (vector and halfvec only)", fn,
               tb.elem == VB_BIT ? "bit" : "this element type");
    VB_REQUIRE(ngroups >= 1, "%s: ngroups = %d, must be at least 1", fn, ngroups);
    VB_REQUIRE(run_rows >= 0, "%s: run_rows = %lld, must be >= 0 (0 = one run per group)", fn, (long long)run_rows);
    VB_REQUIRE(group_of_row || ngroups == 1, "%s: group_of_row is NULL (every row in group 0) but ngroups = %d", fn, ngroups);
    VB_REQUIRE(out && out_counts, "%s: null output", fn);
    VB_REQUIRE(agg == VB_AGG_AVG || !out_state, "%s: sum has no separate transition state (its state is the result); pass out_state = NULL",
               fn);
    const int64_t n = tb.n;
    const int dim = tb.dim;
    VB_REQUIRE((int64_t)ngroups * dim / AGG_THREADS < (int64_t)INT32_MAX, "%s: %d groups x %d columns is too many for one call", fn,
               ngroups, dim);
    const bool grouped = group_of_row != nullptr;
    VB_REQUIRE(!grouped || n <= (int64_t)INT32_MAX, "%s: a grouped aggregate takes tables of at most %d rows, this one has %lld", fn,
               INT32_MAX, (long long)n);
    if (host && grouped)
        for (int64_t i = 0; i < n; ++i)
            VB_REQUIRE(group_of_row[i] >= -1 && group_of_row[i] < ngroups, "%s: group_of_row[%lld] = %d is not a group (-1..%d)", fn,
                       (long long)i, group_of_row[i], ngroups - 1);
    Context& c = ctx();
    const size_t esize = tb.elem == VB_VECTOR ? 4 : 2;
    const size_t out_bytes = (size_t)ngroups * dim * esize;
    const size_t state_bytes = out_state ? (size_t)ngroups * ((size_t)dim + 1) * 8 : 0;

    // the runs: ungrouped, ceil(n / R) of them; grouped, at most one per row and at most n / R + one per group
    RunPlan p{};
    p.n = n;
    p.ngroups = ngroups;
    if (!grouped) {
        p.R = (run_rows == 0 || run_rows >= n) ? std::max<int64_t>(n, 1) : run_rows;
        p.nruns = n == 0 ? 0 : (n + p.R - 1) / p.R;
    } else {
        p.R = run_rows;
        p.nruns = run_rows == 0 ? std::min<int64_t>(n, ngroups) : std::min<int64_t>(n, n / run_rows + ngroups);
    }
    const size_t run_state_bytes = (size_t)p.nruns * dim * (agg == VB_AGG_AVG ? 8 : 4);
    size_t sort_tmp = 0, scan_tmp = 0;
    int end_bit = 1;
    while (end_bit < 32 && ((uint64_t)ngroups >> end_bit) != 0) ++end_bit;
    if (grouped && n > 0) {
        VB_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, sort_tmp, (const uint32_t*)nullptr, (uint32_t*)nullptr, (const int32_t*)nullptr,
                                                (int32_t*)nullptr, (int)n, 0, end_bit, c.stream));
        VB_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, scan_tmp, (const int32_t*)nullptr, (int32_t*)nullptr, ngroups + 1, c.stream));
    }
    const size_t list_bytes = grouped && n > 0 ? 4 * al256(4 * (size_t)n) : 0;               // keys, rows, sorted keys, sorted rows
    const size_t group_bytes = grouped && n > 0 ? 3 * al256(4 * ((size_t)ngroups + 1)) : 0;  // gstart, gend, run_begin
    const size_t tmp_bytes = al256(std::max(sort_tmp, scan_tmp));
    const size_t stage_bytes = host ? al256(out_bytes) + al256(8 * (size_t)ngroups) + al256(state_bytes) : 0;
    const size_t total = list_bytes + group_bytes + tmp_bytes + al256(run_state_bytes) + stage_bytes + 256;
    size_t free_b = 0, total_b = 0;
    VB_CUDA(cudaMemGetInfo(&free_b, &total_b));
    if (total > free_b) {
        set_error("%s: needs %zu bytes of device memory (row list and sort space %zu, run states %zu, staged results %zu), %zu are free",
                  fn, total, list_bytes + group_bytes + tmp_bytes, run_state_bytes, stage_bytes, free_b);
        return VB_ENOMEM;
    }
    Scratch scratch;
    void* mem;
    if (scratch.own(total, &mem) != VB_OK) {
        set_error("%s: allocation of %zu bytes (row list and sort space %zu, run states %zu, staged results %zu) failed", fn, total,
                  list_bytes + group_bytes + tmp_bytes, run_state_bytes, stage_bytes);
        return VB_ENOMEM;
    }
    uint8_t* cur = (uint8_t*)mem;
    auto take = [&](size_t b) {
        uint8_t* r = cur;
        cur += al256(b);
        return (void*)r;
    };
    int* flag = (int*)take(4);
    void* states = take(run_state_bytes);
    void* tmp = take(std::max(sort_tmp, scan_tmp));
    void* d_out = host ? take(out_bytes) : out;
    int64_t* d_counts = host ? (int64_t*)take(8 * (size_t)ngroups) : out_counts;
    double* d_state = host ? (out_state ? (double*)take(state_bytes) : nullptr) : out_state;
    VB_CUDA(cudaMemsetAsync(flag, 0, 4, c.stream));

    if (grouped && n > 0) {
        uint32_t* keys = (uint32_t*)take(4 * (size_t)n);
        int32_t* rows = (int32_t*)take(4 * (size_t)n);
        uint32_t* keys_sorted = (uint32_t*)take(4 * (size_t)n);
        int32_t* rows_sorted = (int32_t*)take(4 * (size_t)n);
        int32_t* gstart = (int32_t*)take(4 * ((size_t)ngroups + 1));
        int32_t* gend = (int32_t*)take(4 * ((size_t)ngroups + 1));
        int32_t* run_begin = (int32_t*)take(4 * ((size_t)ngroups + 1));
        const int32_t* d_groups = group_of_row;
        if (host) {   // staged through the sorted-keys buffer, which the sort fills later
            VB_CUDA(cudaMemcpyAsync(keys_sorted, group_of_row, 4 * (size_t)n, cudaMemcpyHostToDevice, c.stream));
            d_groups = (const int32_t*)keys_sorted;
        }
        const unsigned nb = (unsigned)((n + AGG_THREADS - 1) / AGG_THREADS);
        agg_keys_kernel<<<nb, AGG_THREADS, 0, c.stream>>>(d_groups, n, ngroups, keys, rows);
        VB_CUDA(cudaGetLastError());
        VB_CUDA(cub::DeviceRadixSort::SortPairs(tmp, sort_tmp, keys, keys_sorted, rows, rows_sorted, (int)n, 0, end_bit, c.stream));
        VB_CUDA(cudaMemsetAsync(gstart, 0, 4 * ((size_t)ngroups + 1), c.stream));
        VB_CUDA(cudaMemsetAsync(gend, 0, 4 * ((size_t)ngroups + 1), c.stream));
        agg_bounds_kernel<<<nb, AGG_THREADS, 0, c.stream>>>(keys_sorted, n, ngroups, gstart, gend);
        VB_CUDA(cudaGetLastError());
        agg_nruns_kernel<<<(unsigned)((ngroups + AGG_THREADS) / AGG_THREADS), AGG_THREADS, 0, c.stream>>>(gstart, gend, ngroups, run_rows,
                                                                                                       run_begin);
        VB_CUDA(cudaGetLastError());
        VB_CUDA(cub::DeviceScan::ExclusiveSum(tmp, scan_tmp, run_begin, run_begin, ngroups + 1, c.stream));
        count_launch(3);
        p.row_list = rows_sorted;
        p.gstart = gstart;
        p.gend = gend;
        p.run_begin = run_begin;
        VB_TRY(dispatch_agg<true>(tb.elem, agg, tb, p, states, d_out, d_counts, d_state, flag));
    } else if (grouped) {   // an empty table: every group is empty (the zero-run plan of a table without groups)
        RunPlan e = p;
        e.nruns = 0;
        e.n = 0;
        VB_TRY(dispatch_agg<false>(tb.elem, agg, tb, e, states, d_out, d_counts, d_state, flag));
    } else {
        VB_TRY(dispatch_agg<false>(tb.elem, agg, tb, p, states, d_out, d_counts, d_state, flag));
    }

    if (agg == VB_AGG_SUM) {   // float_overflow_error(): the one host read of the _dev variant
        int h_flag = 0;
        VB_CUDA(cudaMemcpyAsync(&h_flag, flag, 4, cudaMemcpyDeviceToHost, c.stream));
        VB_CUDA(cudaStreamSynchronize(c.stream));
        if (h_flag) {
            set_error("value out of range: overflow");
            return VB_EINVAL;
        }
    }
    if (host) {
        VB_CUDA(cudaMemcpyAsync(out, d_out, out_bytes, cudaMemcpyDeviceToHost, c.stream));
        VB_CUDA(cudaMemcpyAsync(out_counts, d_counts, 8 * (size_t)ngroups, cudaMemcpyDeviceToHost, c.stream));
        if (out_state) VB_CUDA(cudaMemcpyAsync(out_state, d_state, state_bytes, cudaMemcpyDeviceToHost, c.stream));
        VB_CUDA(cudaStreamSynchronize(c.stream));
    }
    return VB_OK;
}

}  // namespace vb

using namespace vb;

extern "C" {

int vb_table_aggregate(vb_table* t, int agg, const int32_t* group_of_row, int ngroups, int64_t run_rows, void* out, int64_t* out_counts,
                       double* out_state) {
    return aggregate_impl(t, agg, group_of_row, ngroups, run_rows, out, out_counts, out_state, true);
}

int vb_table_aggregate_dev(vb_table* t, int agg, const int32_t* group_of_row_dev, int ngroups, int64_t run_rows, void* out_dev,
                           int64_t* out_counts_dev, double* out_state_dev) {
    return aggregate_impl(t, agg, group_of_row_dev, ngroups, run_rows, out_dev, out_counts_dev, out_state_dev, false);
}

}  // extern "C"
