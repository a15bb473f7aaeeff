// vb_slab_select.cuh -- CTA-wide selection of the k' nearest of one query's candidate run, shared by
// slab_select_kernel (vb_scan.cu), cta_refine_kernel (vb_list_tc.cu) and the one-query kernels (vb_ivf_one.cu).
//
// The tensor-core filter's epilogue stores, beside the dense d~ array, min d~ of every slab (32 table-aligned rows of one
// probed list, slab_base() in vb_common.cuh).  tau = the k'-th smallest slab minimum is an upper bound of the k'-th
// smallest d~ (k' distinct candidates are <= tau), so the k' nearest all lie in slabs whose minimum is <= tau: exactly k'
// slabs when the minima are distinct -- 32 k' candidates are read per query instead of the whole run.
#pragma once

#include "vb_common.cuh"
#include "vb_distance.cuh"

namespace vb {

constexpr int SS_THREADS = 256;
constexpr int SS_CAND = 2048;

// cand[0 .. npow2) sorted ascending by (d~, position); entries past n are ~0ull.  All SS_THREADS threads call it.
__device__ __forceinline__ void ss_sort_cand(uint64_t* cand, uint32_t n) {
    const int tid = threadIdx.x;
    int npow2 = 2;
    while ((uint32_t)npow2 < n) npow2 <<= 1;
    for (int i = (int)n + tid; i < npow2; i += SS_THREADS) cand[i] = ~0ull;
    __syncthreads();
    for (int size = 2; size <= npow2; size <<= 1) {
        for (int st = size >> 1; st > 0; st >>= 1) {
            for (int i = tid; i < npow2; i += SS_THREADS) {
                const int j = i ^ st;
                if (j > i) {
                    const uint64_t x = cand[i], y = cand[j];
                    const bool up = (i & size) == 0;
                    if ((x > y) == up) {
                        cand[i] = y;
                        cand[j] = x;
                    }
                }
            }
            __syncthreads();
        }
    }
}

// the k-th smallest of the S orderable keys in shared memory (k <= S): four 8-bit radix passes over a 256-bin histogram
__device__ __forceinline__ uint32_t ss_radix_kth(const uint32_t* keys, int S, int k) {
    __shared__ uint32_t hist[256];
    __shared__ uint32_t s_prefix, s_mask, s_kk;
    const int tid = threadIdx.x;
    if (tid == 0) {
        s_prefix = 0;
        s_mask = 0;
        s_kk = (uint32_t)k;
    }
    __syncthreads();
    for (int pass = 3; pass >= 0; --pass) {
        hist[tid] = 0;
        __syncthreads();
        const int shift = pass * 8;
        const uint32_t prefix = s_prefix, mask = s_mask;
        // (plain shared-memory atomics: a warp-aggregated histogram -- __match_any_sync per key -- measured slower at the run
        // lengths this sees: +12 us per launch on 330 slab minima / 1000 centres, +10 us on the 10 k keys of a one-query scan)
        for (int i = tid; i < S; i += SS_THREADS) {
            const uint32_t key = keys[i];
            if ((key & mask) == prefix) atomicAdd(&hist[(key >> shift) & 255u], 1u);
        }
        __syncthreads();
        if (tid < 32) {
            // the bin holding the kk-th key: every lane sums 8 bins, a warp scan finds the lane, the lane its bin
            const uint32_t kk = s_kk;
            uint32_t h[8], mine = 0;
#pragma unroll
            for (int t = 0; t < 8; ++t) {
                h[t] = hist[tid * 8 + t];
                mine += h[t];
            }
            uint32_t incl = mine;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const uint32_t u = __shfl_up_sync(0xffffffffu, incl, o);
                if (tid >= o) incl += u;
            }
            const unsigned reach = __ballot_sync(0xffffffffu, incl >= kk);
            const int owner = __ffs(reach) - 1;      // (kk <= the number of keys under the prefix: always found)
            if (tid == owner) {
                uint32_t cum = incl - mine;
                int b = 0;
#pragma unroll
                for (int t = 0; t < 8; ++t) {
                    if (cum + h[t] >= kk) break;
                    cum += h[t];
                    ++b;
                }
                s_prefix = prefix | ((uint32_t)(tid * 8 + b) << shift);
                s_mask = mask | (0xFFu << shift);
                s_kk = kk - cum;
            }
        }
        __syncthreads();
    }
    return s_prefix;   // exactly the k-th smallest key
}

// the probe whose run [off[p], off[p + 1]) holds entry i (off non-decreasing, off[0] = 0, i < off[probes]; empty probes share an offset)
__device__ __forceinline__ int ss_probe_of(const int32_t* off, int probes, int i) {
    int p = 0, hi = probes;
    while (hi - p > 1) {
        const int mid = (p + hi) >> 1;
        if (off[mid] <= i) p = mid;
        else hi = mid;
    }
    return p;
}

struct SsWork {
    int64_t *lo, *hi;        // [probes] list bounds
    uint32_t *skey, *qlist;  // [cap_s] orderable slab minima, qualifying slabs
    int32_t *off, *co;       // [probes + 1] first slab of every probe, [probes] first candidate of every probe
};
__device__ __forceinline__ SsWork ss_work_layout(void* work, int64_t cap_s, int probes) {
    SsWork w;
    w.lo = reinterpret_cast<int64_t*>(work);
    w.hi = w.lo + probes;
    w.skey = reinterpret_cast<uint32_t*>(w.hi + probes);
    w.qlist = w.skey + cap_s;
    w.off = reinterpret_cast<int32_t*>(w.qlist + cap_s);
    w.co = w.off + probes + 1;
    return w;
}

// shared memory the selection needs beside cand[SS_CAND]: slab keys + the list of qualifying slabs (2 cap_s words), and
// per probe: first slab (probes + 1), candidate offset, list bounds
__host__ __device__ inline size_t ss_select_smem_bytes(int64_t cap_s, int probes) {
    return (size_t)cap_s * 8 + (size_t)(2 * probes + 2) * 4 + (size_t)probes * 16 + 16;
}

// dynamic shared memory of one CTA of launch_slab_select and of launch_list_tc_cta_refine, at most.  The batched search
// takes slab minima only where the launch that reads them stays under it (ivf_scan_topk).
constexpr size_t SS_SMEM_MAX = 200 * 1024;

// dynamic shared memory of slab_select_kernel (launch_slab_select): cand[SS_CAND] and the selection's work area
inline size_t slab_select_launch_smem(int64_t cap_s, int probes) { return (size_t)SS_CAND * 8 + ss_select_smem_bytes(cap_s, probes); }

// The candidates of query q that can be among its k nearest by d~: (1) the run's slab minima into shared memory,
// (2) radix-select tau, (3) list the qualifying slabs, then gather their candidates <= tau with every load independent
// (one candidate per thread and step), (4) sort.  Returns their number n (cand[0 .. n) sorted, n >= min(k, run length)),
// or -1 when more than SS_CAND qualify (ties by the thousand).  `work`: ss_select_smem_bytes() of shared memory, 8-byte aligned.
__device__ __forceinline__ int slab_select_cta(const float* __restrict__ dist, const float* __restrict__ smin, int probes,
                                               const int32_t* __restrict__ probe_lists, const int32_t* __restrict__ cand_off,
                                               const int64_t* __restrict__ list_off, int64_t cap, int64_t cap_s, int q, int k,
                                               uint64_t* cand, void* work) {
    __shared__ uint32_t s_count, s_nq;
    const SsWork W = ss_work_layout(work, cap_s, probes);
    int64_t *s_lo = W.lo, *s_hi = W.hi;
    uint32_t *skey = W.skey, *qlist = W.qlist;
    int32_t *s_off = W.off, *s_co = W.co;
    const int tid = threadIdx.x;
    const int32_t* co = cand_off + (int64_t)q * (probes + 1);
    const int32_t* pl = probe_lists + (int64_t)q * probes;
    // slabs per probe (the list bounds are independent loads: one thread per probe), then their prefix sums
    for (int p = tid; p < probes; p += SS_THREADS) {
        const int l = pl[p];
        int ns = 0;
        int64_t lo = 0, hi = 0;
        if (l >= 0) {
            lo = list_off[l];
            hi = list_off[l + 1];
            if (hi > lo) ns = (int)(((hi - 1) >> 5) - (lo >> 5) + 1);
        }
        s_lo[p] = lo;
        s_hi[p] = hi;
        s_co[p] = co[p];
        s_off[p + 1] = ns;
    }
    __syncthreads();
    if (tid == 0) {
        int off = 0;
        s_off[0] = 0;
        for (int p = 0; p < probes; ++p) {
            off += s_off[p + 1];
            s_off[p + 1] = off;
        }
        s_count = 0;
        s_nq = 0;
    }
    __syncthreads();
    const int S = s_off[probes];
    // slab minima of all probes at once (one independent load per thread and step)
    for (int i = tid; i < S; i += SS_THREADS) {
        const int p = ss_probe_of(s_off, probes, i);
        skey[i] = orderable_key(smin[slab_base(q, cap_s, s_co[p], p) + (i - s_off[p])]);
    }
    __syncthreads();
    // ---- tau: the k-th smallest slab minimum (everything when there are at most k slabs)
    uint32_t tau = 0xFFFFFFFFu;
    if (S > k) tau = ss_radix_kth(skey, S, k);
    // ---- the qualifying slabs, then their rows: thread t takes row t % 32 of listed slab t / 32
    for (int i = tid; i < S; i += SS_THREADS)
        if (skey[i] <= tau) qlist[atomicAdd(&s_nq, 1u)] = (uint32_t)i;
    __syncthreads();
    const int nq_rows = (int)s_nq * 32;
    const float* dq = dist + (int64_t)q * cap;
    for (int t = tid; t < nq_rows; t += SS_THREADS) {
        const int i = (int)qlist[t >> 5];
        const int p = ss_probe_of(s_off, probes, i);
        const int64_t lo = s_lo[p], hi = s_hi[p];
        const int64_t r = (((lo >> 5) + (i - s_off[p])) << 5) + (t & 31);
        if (r >= lo && r < hi) {
            const uint32_t pos = (uint32_t)(s_co[p] + (int32_t)(r - lo));
            const uint32_t ok = orderable_key(dq[pos]);
            if (ok <= tau) {
                const uint32_t slot = atomicAdd(&s_count, 1u);
                if (slot < (uint32_t)SS_CAND) cand[slot] = ((uint64_t)ok << 32) | pos;
            }
        }
    }
    __syncthreads();
    const uint32_t n = s_count;
    if (n > (uint32_t)SS_CAND) return -1;
    ss_sort_cand(cand, n);
    return (int)n;
}

// EXACTLY the min(k, n) smallest of keys[0 .. n) (shared memory, orderable keys) by (key, index), sorted, as composites
// key << 32 | index in cand (capacity: the power of two >= max(2, min(k, n)); k <= SS_CAND).  Ties across the k-th place
// are settled by index -- scan position / list number, this library's tie rule -- whatever their number (bit vectors put
// thousands of rows at one Hamming distance): the index bound is found by bisection, a counting pass per step.
// All SS_THREADS threads call it; keys must be complete (a __syncthreads() after the last write).
__device__ __forceinline__ int select_exact_cta(const uint32_t* keys, int n, int k, uint64_t* cand) {
    __shared__ uint32_t se_cnt, se_less, se_eq, se_tally;
    const int tid = threadIdx.x;
    if (n <= k) {
        for (int i = tid; i < n; i += SS_THREADS) cand[i] = ((uint64_t)keys[i] << 32) | (uint32_t)i;
        __syncthreads();
        ss_sort_cand(cand, (uint32_t)n);
        return n;
    }
    if (tid == 0) se_cnt = se_less = se_eq = 0;
    const uint32_t tau = ss_radix_kth(keys, n, k);     // (its first barrier also publishes the zeros above)
    {
        uint32_t less = 0, eq = 0;
        for (int i = tid; i < n; i += SS_THREADS) {
            const uint32_t key = keys[i];
            less += key < tau ? 1u : 0u;
            eq += key == tau ? 1u : 0u;
        }
        for (int o = 16; o > 0; o >>= 1) {
            less += __shfl_xor_sync(0xffffffffu, less, o);
            eq += __shfl_xor_sync(0xffffffffu, eq, o);
        }
        if ((tid & 31) == 0) {
            if (less) atomicAdd(&se_less, less);
            if (eq) atomicAdd(&se_eq, eq);
        }
    }
    __syncthreads();
    const uint32_t need = (uint32_t)k - se_less;       // 1 <= need <= se_eq: the equals that still fit
    uint32_t plim = 0xFFFFFFFFu;                       // equals with index <= plim are taken
    if (se_eq > need) {
        uint32_t lo = 0, hi = (uint32_t)n - 1;         // the smallest P with #{i <= P : keys[i] == tau} >= need
        while (lo < hi) {
            const uint32_t mid = lo + ((hi - lo) >> 1);
            __syncthreads();
            if (tid == 0) se_tally = 0;
            __syncthreads();
            uint32_t c = 0;
            for (int i = tid; i < n && (uint32_t)i <= mid; i += SS_THREADS) c += keys[i] == tau ? 1u : 0u;
            for (int o = 16; o > 0; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
            if ((tid & 31) == 0 && c) atomicAdd(&se_tally, c);
            __syncthreads();
            if (se_tally >= need) hi = mid;
            else lo = mid + 1;
        }
        plim = lo;
    }
    for (int i = tid; i < n; i += SS_THREADS) {
        const uint32_t key = keys[i];
        if (key < tau || (key == tau && (uint32_t)i <= plim)) {
            const uint32_t slot = atomicAdd(&se_cnt, 1u);
            cand[slot] = ((uint64_t)key << 32) | (uint32_t)i;     // (exactly k of them)
        }
    }
    __syncthreads();
    ss_sort_cand(cand, (uint32_t)k);
    return k;
}

}  // namespace vb
