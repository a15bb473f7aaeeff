// vb_ivf_one.cu -- the IVFFlat scan of ONE query (or a handful): what a backend issues.  ivfflatgettuple's first call
// runs GetScanLists and GetScanItems for a single ORDER BY value (src/ivfscan.c:47-118, 123-187, 360-414;
// amcanparallel = false, src/ivfflat.c:266), so the latency of a scan is launches and round trips, not bandwidth: 60 MB of
// rows are ~20 us of HBM time, far less than the nine launches, three memsets and four copies of the general path.
//
// Here a scan is TWO kernels, each a fused distance + select (north_star's "one-query-vs-many-candidates distance +
// top-k select as a fused kernel"):
//   one_probe_kernel  distances of the query to every centre (the CTAs split the centre table), then the LAST CTA to
//                     finish (a ticket counter) selects the `probes` nearest by (distance, list number);
//   one_scan_kernel   every CTA derives the candidate offsets of the probed lists, scores its slice of the concatenated
//                     candidate run, and the last CTA selects the k nearest by (distance, scan position), maps them to
//                     heap ids and applies the operator's epilogue (sqrt / negate, src/vector.c:591-598, 632-639).
// The per-row arithmetic is scan_kernel's (vb_scan.cu: groups of LPR lanes walk a row with 128-bit loads, RPI rows in
// flight, xor-shuffle reduction), lane for lane -- a distance does not depend on which kernel computed it.
#include "vb_common.cuh"
#include "vb_distance.cuh"
#include "vb_slab_select.cuh"

#include <algorithm>

namespace vb {

constexpr int ONE_THREADS = SS_THREADS;   // the selection helpers are written for this CTA size

// distances of the shared-memory query image to n_rows consecutive table rows -> out[0 .. n_rows)
template <int ELEM, int METRIC, int LPR, int RPI>
__device__ __forceinline__ void one_score_rows(const uint8_t* __restrict__ base, size_t stride, int V, int n_rows, const uint4* sq,
                                               float* __restrict__ out) {
    constexpr int G = ONE_THREADS / LPR;
    const int g = threadIdx.x / LPR;
    const int l = threadIdx.x % LPR;
    // trip count is uniform over the CTA (the lanes of a group must stay converged for the shuffles)
    for (int rb = 0; rb < n_rows; rb += G * RPI) {
        const int r0 = rb + g;
        Acc<ELEM, METRIC> acc[RPI];
        const uint4* rp[RPI];
#pragma unroll
        for (int i = 0; i < RPI; ++i) {
            const int r = r0 + i * G;
            rp[i] = reinterpret_cast<const uint4*>(base + (size_t)min(r, n_rows - 1) * stride);   // out-of-range: a valid row, result dropped
        }
        uint4 cur[RPI];
        if (l < V) {
#pragma unroll
            for (int i = 0; i < RPI; ++i) cur[i] = ldg_stream(rp[i] + l);
        }
#pragma unroll 2
        for (int v = l; v < V; v += LPR) {
            uint4 nxt[RPI];
            const int vn = v + LPR;
            if (vn < V) {
#pragma unroll
                for (int i = 0; i < RPI; ++i) nxt[i] = ldg_stream(rp[i] + vn);
            }
#pragma unroll
            for (int i = 0; i < RPI; ++i) acc[i].add(cur[i], sq, v);
            if (vn < V) {
#pragma unroll
                for (int i = 0; i < RPI; ++i) cur[i] = nxt[i];
            }
        }
#pragma unroll
        for (int i = 0; i < RPI; ++i) {
            acc[i].template reduce<LPR>();
            const int r = r0 + i * G;
            if (l == 0 && r < n_rows) out[r] = (float)acc[i].value();
        }
    }
}

// true in the CTA that finishes last for this query (all CTAs of the query call it once, after their global writes)
__device__ __forceinline__ bool one_last_cta(unsigned* ticket) {
    __shared__ bool s_last;
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) s_last = atomicAdd(ticket, 1u) == gridDim.x - 1;
    __syncthreads();
    if (s_last) __threadfence();
    return s_last;
}

struct OneProbeArgs {
    const uint8_t* centres;
    size_t stride;
    int V, lists;
    const uint8_t* qimg;
    size_t qstride;
    int qvec, probes;
    float* cdist;          // [nq][lists]
    unsigned* ticket;      // [nq], zero between launches
    int32_t* out_lists;    // [nq][probes]
    float* out_ldist;      // [nq][probes]
    unsigned long long* zero_me;   // the scan's running candidate total, reset here (or null)
};

// GetScanLists (src/ivfscan.c:47-118) for query blockIdx.y
template <int ELEM, int METRIC, int LPR, int RPI>
__global__ void __launch_bounds__(ONE_THREADS) one_probe_kernel(OneProbeArgs a) {
    extern __shared__ uint4 one_smem[];
    uint4* sq = one_smem;
    const int q = blockIdx.y;
    const uint4* gq = reinterpret_cast<const uint4*>(a.qimg + (size_t)q * a.qstride);
    for (int i = threadIdx.x; i < a.qvec; i += ONE_THREADS) sq[i] = gq[i];
    __syncthreads();
    constexpr int UNIT = (ONE_THREADS / LPR) * RPI;
    float* cd = a.cdist + (size_t)q * a.lists;
    for (int r0 = blockIdx.x * UNIT; r0 < a.lists; r0 += gridDim.x * UNIT)
        one_score_rows<ELEM, METRIC, LPR, RPI>(a.centres + (size_t)r0 * a.stride, a.stride, a.V, min(UNIT, a.lists - r0), sq, cd + r0);
    if (!one_last_cta(a.ticket + q)) return;
    // the nearest `probes` centres by (distance, list number)
    uint32_t* keys = reinterpret_cast<uint32_t*>(one_smem + a.qvec);
    uint64_t* cand = reinterpret_cast<uint64_t*>(keys + ((a.lists + 1) & ~1));
    for (int i = threadIdx.x; i < a.lists; i += ONE_THREADS) keys[i] = orderable_key(__ldcg(cd + i));
    __syncthreads();
    const int m = select_exact_cta(keys, a.lists, a.probes, cand);
    for (int p = threadIdx.x; p < a.probes; p += ONE_THREADS) {
        const bool have = p < m;
        a.out_lists[(size_t)q * a.probes + p] = have ? (int32_t)(uint32_t)cand[p] : -1;
        a.out_ldist[(size_t)q * a.probes + p] = have ? key_to_float((uint32_t)(cand[p] >> 32)) : __int_as_float(0x7F800000);
    }
    if (threadIdx.x == 0) {
        a.ticket[q] = 0;
        if (q == 0 && a.zero_me) *a.zero_me = 0;
    }
}

struct OneScanArgs {
    const uint8_t* rows;
    size_t stride;
    int V;
    const int64_t* list_off;
    const int64_t* ids;
    const int32_t* probe_lists;   // [nq][probes]
    int probes;
    const uint8_t* qimg;
    size_t qstride;
    int qvec, k, metric;
    int64_t cap;                  // bound of one query's candidates (stride of dist, words of the key area)
    float* dist;                  // [nq][cap]
    unsigned* ticket;             // [nq], zero between launches
    int64_t* out_ids;             // [nq][k]
    float* out_f;                 // [nq][k] or null
    double* out_d;                // [nq][k] or null
    int32_t* out_total;           // [nq] candidates scanned, or null
    unsigned long long* cand_sum; // running total of candidates scanned, or null
    int cand_store;               // 1: store this query's total instead of adding it (single query, no probe kernel before)
};

__device__ __forceinline__ double one_finish_value(int metric, float key) {
    if (metric == VB_L2) return sqrt((double)key);
    if (metric == VB_IP) return -(double)key;
    return (double)key;
}

// GetScanItems + the sort (src/ivfscan.c:123-187, 400-414) for query blockIdx.y
template <int ELEM, int METRIC, int LPR, int RPI>
__global__ void __launch_bounds__(ONE_THREADS) one_scan_kernel(OneScanArgs a) {
    extern __shared__ uint4 one_smem[];
    uint4* sq = one_smem;
    int64_t* lo = reinterpret_cast<int64_t*>(one_smem + a.qvec);           // [probes] first table row of the probed list
    int32_t* co = reinterpret_cast<int32_t*>(lo + a.probes);               // [probes + 1] candidate offsets
    uint32_t* keys = reinterpret_cast<uint32_t*>(co + ((a.probes + 2) & ~1));
    uint64_t* cand = reinterpret_cast<uint64_t*>(keys + ((a.cap + 1) & ~(int64_t)1));
    const int q = blockIdx.y;
    const uint4* gq = reinterpret_cast<const uint4*>(a.qimg + (size_t)q * a.qstride);
    for (int i = threadIdx.x; i < a.qvec; i += ONE_THREADS) sq[i] = gq[i];
    const int32_t* pl = a.probe_lists + (size_t)q * a.probes;
    for (int p = threadIdx.x; p < a.probes; p += ONE_THREADS) {
        const int l = pl[p];
        const int64_t b = l >= 0 ? a.list_off[l] : 0;
        lo[p] = b;
        co[p + 1] = l >= 0 ? (int32_t)(a.list_off[l + 1] - b) : 0;      // the length for now
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        int32_t off = 0;
        co[0] = 0;
        for (int p = 0; p < a.probes; ++p) {
            off += co[p + 1];
            co[p + 1] = off;
        }
    }
    __syncthreads();
    const int total = co[a.probes];
    float* dq = a.dist + (size_t)q * a.cap;
    {
        constexpr int UNIT = (ONE_THREADS / LPR) * RPI;
        int per = (total + (int)gridDim.x - 1) / (int)gridDim.x;
        per = max(UNIT, (per + UNIT - 1) / UNIT * UNIT);
        const int s0 = (int)blockIdx.x * per;
        const int s1 = min(total, s0 + per);
        if (s0 < s1) {
            for (int p = 0; p < a.probes; ++p) {
                const int b0 = max(s0, co[p]), b1 = min(s1, co[p + 1]);
                if (b0 < b1)
                    one_score_rows<ELEM, METRIC, LPR, RPI>(a.rows + (size_t)(lo[p] + (b0 - co[p])) * a.stride, a.stride, a.V, b1 - b0, sq, dq + b0);
            }
        }
    }
    if (!one_last_cta(a.ticket + q)) return;
    {
        // (cap is a multiple of 4 and the scratch 256-byte aligned: every query's run starts on a 16-byte boundary)
        const int t4 = total >> 2;
        const uint4* d4 = reinterpret_cast<const uint4*>(dq);
        for (int i = threadIdx.x; i < t4; i += ONE_THREADS) {
            const uint4 v = __ldcg(d4 + i);
            keys[4 * i] = orderable_key(__uint_as_float(v.x));
            keys[4 * i + 1] = orderable_key(__uint_as_float(v.y));
            keys[4 * i + 2] = orderable_key(__uint_as_float(v.z));
            keys[4 * i + 3] = orderable_key(__uint_as_float(v.w));
        }
        for (int i = (t4 << 2) + threadIdx.x; i < total; i += ONE_THREADS) keys[i] = orderable_key(__ldcg(dq + i));
    }
    __syncthreads();
    const int m = select_exact_cta(keys, total, a.k, cand);
    for (int i = threadIdx.x; i < a.k; i += ONE_THREADS) {
        int64_t id = -1;
        float key = __int_as_float(0x7F800000);
        if (i < m) {
            const int ps = (int)(uint32_t)cand[i];
            key = key_to_float((uint32_t)(cand[i] >> 32));
            int pa = 0, pb = a.probes;        // the last probe whose offset is <= ps (empty lists share an offset)
            while (pb - pa > 1) {
                const int mid = (pa + pb) >> 1;
                if (co[mid] <= ps) pa = mid;
                else pb = mid;
            }
            const int64_t row = lo[pa] + (ps - co[pa]);
            id = a.ids ? a.ids[row] : row;
        }
        const double v = one_finish_value(a.metric, key);
        a.out_ids[(size_t)q * a.k + i] = id;
        if (a.out_f) a.out_f[(size_t)q * a.k + i] = (float)v;
        if (a.out_d) a.out_d[(size_t)q * a.k + i] = v;
    }
    if (threadIdx.x == 0) {
        a.ticket[q] = 0;
        if (a.out_total) a.out_total[q] = total;
        if (a.cand_sum) {
            if (a.cand_store) *a.cand_sum = (unsigned long long)total;
            else atomicAdd(a.cand_sum, (unsigned long long)total);
        }
    }
}

// ----------------------------------------------------------------------------- host side

static int pow2_at_least(int64_t x) {
    int p = 2;
    while (p < x) p <<= 1;
    return p;
}

size_t one_probe_smem(int lists, size_t qstride, int probes) {
    return qstride + (size_t)((lists + 1) & ~1) * 4 + (size_t)pow2_at_least(std::min(probes, lists)) * 8;
}
size_t one_scan_smem(int64_t cap, size_t qstride, int probes, int64_t k) {
    return qstride + (size_t)probes * 8 + (size_t)((probes + 2) & ~1) * 4 + (size_t)((cap + 1) & ~(int64_t)1) * 4 +
           (size_t)pow2_at_least(std::min<int64_t>(k, cap)) * 8;
}
constexpr size_t ONE_SMEM_MAX = 200 * 1024;

bool one_probe_fits(int lists, size_t qstride, int probes) {
    return probes >= 1 && probes <= SS_CAND && lists >= 1 && one_probe_smem(lists, qstride, probes) <= ONE_SMEM_MAX;
}
bool one_scan_fits(int64_t cap, size_t qstride, int probes, int64_t k) {
    return probes >= 1 && probes <= 4096 && k >= 1 && k <= SS_CAND && cap >= 1 && cap < (int64_t)1 << 30 &&
           one_scan_smem(cap, qstride, probes, k) <= ONE_SMEM_MAX;
}

// lanes per row / rows in flight as launch_scan_t (vb_scan.cu) picks them -- the summation order of a distance follows
#define VB_ONE_SHAPES(X, V)        \
    do {                           \
        if ((V) >= 32) X(32, 4);   \
        else if ((V) >= 16) X(16, 4); \
        else if ((V) >= 8) X(8, 4); \
        else if ((V) >= 4) X(4, 8); \
        else if ((V) >= 2) X(2, 8); \
        else X(1, 8);              \
    } while (0)

template <int ELEM, int METRIC>
static int one_probe_t(const OneProbeArgs& a, int64_t nq) {
    const size_t smem = one_probe_smem(a.lists, a.qstride, a.probes);
    cudaStream_t s = ctx().stream;
#define VB_X(LPR, RPI)                                                                                                    \
    do {                                                                                                                  \
        auto kern = one_probe_kernel<ELEM, METRIC, LPR, RPI>;                                                             \
        if (smem > 48 * 1024) VB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); \
        const int unit = (ONE_THREADS / LPR) * RPI;                                                                       \
        const int gx = std::max(1, std::min((a.lists + unit - 1) / unit, ctx().sm_count * 4));                            \
        kern<<<dim3((unsigned)gx, (unsigned)nq), ONE_THREADS, smem, s>>>(a);                                              \
    } while (0)
    VB_ONE_SHAPES(VB_X, a.V);
#undef VB_X
    VB_CUDA(cudaGetLastError());
    count_launch();
    return VB_OK;
}

template <int ELEM, int METRIC>
static int one_scan_t(const OneScanArgs& a, int64_t nq) {
    const size_t smem = one_scan_smem(a.cap, a.qstride, a.probes, a.k);
    cudaStream_t s = ctx().stream;
#define VB_X(LPR, RPI)                                                                                                    \
    do {                                                                                                                  \
        auto kern = one_scan_kernel<ELEM, METRIC, LPR, RPI>;                                                              \
        if (smem > 48 * 1024) VB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); \
        const int unit = (ONE_THREADS / LPR) * RPI;                                                                       \
        const int64_t gx = std::max<int64_t>(1, std::min<int64_t>((a.cap + unit - 1) / unit, (int64_t)ctx().sm_count * 2)); \
        kern<<<dim3((unsigned)gx, (unsigned)nq), ONE_THREADS, smem, s>>>(a);                                              \
    } while (0)
    VB_ONE_SHAPES(VB_X, a.V);
#undef VB_X
    VB_CUDA(cudaGetLastError());
    count_launch();
    return VB_OK;
}

#define VB_ONE_DISPATCH(FN, elem, km, ...)                                                          \
    do {                                                                                            \
        if ((elem) == VB_VECTOR) {                                                                  \
            switch (km) {                                                                           \
                case VB_L2_SQUARED: return FN<VB_VECTOR, VB_L2_SQUARED>(__VA_ARGS__);               \
                case VB_NEG_IP: return FN<VB_VECTOR, VB_NEG_IP>(__VA_ARGS__);                       \
                case VB_COSINE: return FN<VB_VECTOR, VB_COSINE>(__VA_ARGS__);                       \
                case VB_L1: return FN<VB_VECTOR, VB_L1>(__VA_ARGS__);                               \
            }                                                                                       \
        } else if ((elem) == VB_HALFVEC) {                                                          \
            switch (km) {                                                                           \
                case VB_L2_SQUARED: return FN<VB_HALFVEC, VB_L2_SQUARED>(__VA_ARGS__);              \
                case VB_NEG_IP: return FN<VB_HALFVEC, VB_NEG_IP>(__VA_ARGS__);                      \
                case VB_COSINE: return FN<VB_HALFVEC, VB_COSINE>(__VA_ARGS__);                      \
                case VB_L1: return FN<VB_HALFVEC, VB_L1>(__VA_ARGS__);                              \
            }                                                                                       \
        } else {                                                                                    \
            switch (km) {                                                                           \
                case VB_HAMMING: return FN<VB_BIT, VB_HAMMING>(__VA_ARGS__);                        \
                case VB_JACCARD: return FN<VB_BIT, VB_JACCARD>(__VA_ARGS__);                        \
            }                                                                                       \
        }                                                                                           \
        set_error("unsupported metric %d for element type %d", (int)(km), (int)(elem));            \
        return VB_EINVAL;                                                                           \
    } while (0)

int launch_one_probe(const Table& centres, int km, const void* qimg, size_t qstride, int64_t nq, int probes, float* cdist,
                     unsigned* ticket, int32_t* out_lists, float* out_ldist, int64_t* zero_me) {
    OneProbeArgs a{};
    a.centres = centres.d;
    a.stride = centres.stride;
    a.V = (int)(centres.stride / 16);
    a.lists = (int)centres.n;
    a.qimg = (const uint8_t*)qimg;
    a.qstride = qstride;
    a.qvec = (int)(qstride / 16);
    a.probes = probes;
    a.cdist = cdist;
    a.ticket = ticket;
    a.out_lists = out_lists;
    a.out_ldist = out_ldist;
    a.zero_me = (unsigned long long*)zero_me;
    VB_ONE_DISPATCH(one_probe_t, centres.elem, km, a, nq);
}

int launch_one_scan(const Table& rows, int km, int metric, const int64_t* list_off, const int64_t* ids, const int32_t* probe_lists,
                    int probes, const void* qimg, size_t qstride, int64_t nq, int k, int64_t cap, float* dist, unsigned* ticket,
                    int64_t* out_ids, float* out_f, double* out_d, int32_t* out_total, int64_t* cand_sum, bool cand_store) {
    OneScanArgs a{};
    a.rows = rows.d;
    a.stride = rows.stride;
    a.V = (int)(rows.stride / 16);
    a.list_off = list_off;
    a.ids = ids;
    a.probe_lists = probe_lists;
    a.probes = probes;
    a.qimg = (const uint8_t*)qimg;
    a.qstride = qstride;
    a.qvec = (int)(qstride / 16);
    a.k = k;
    a.metric = metric;
    a.cap = cap;
    a.dist = dist;
    a.ticket = ticket;
    a.out_ids = out_ids;
    a.out_f = out_f;
    a.out_d = out_d;
    a.out_total = out_total;
    a.cand_sum = (unsigned long long*)cand_sum;
    a.cand_store = cand_store ? 1 : 0;
    VB_ONE_DISPATCH(one_scan_t, rows.elem, km, a, nq);
}

}  // namespace vb
