// vb_ivf_build.cu -- the device passes of vb_ivf_build* that the k-means and assign code does not already own:
// the sample draw, the destinations (list numbers -> list offsets and one image row per indexed row, call order kept
// inside a list: what the reference gets from its tuplesort by list number, src/ivfbuild.c:271-331), and the placement
// kernel that moves every row once.  The entry points are in vb_ivf.cu, beside the image they fill.
#include "vb_common.cuh"

#include <cub/cub.cuh>

namespace vb {

// ----------------------------------------------------------------------------- sample draw

__device__ __forceinline__ uint32_t build_round(uint64_t seed, int round, uint32_t x) {   // splitmix64 of (seed, round, x)
    uint64_t z = seed + 0x9e3779b97f4a7c15ULL * (uint64_t)(round + 1) + ((uint64_t)x << 32 | x);
    z = (z ^ (z >> 30)) * 0xbf58476d1ce4e5b9ULL;
    z = (z ^ (z >> 27)) * 0x94d049bb133111ebULL;
    return (uint32_t)((z ^ (z >> 31)) >> 16);
}

// rows_out[j] = perm(j): four Feistel rounds over 2 * half bits, walked along the permutation's cycle until the value
// is a row number.  The cycle through j < n comes back to j, so the walk ends; 2^(2 half) < 4 n keeps it short.
__global__ void build_draw_kernel(int64_t n, int64_t ns, uint64_t seed, int half, int64_t* __restrict__ rows_out) {
    const int64_t j = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (j >= ns) return;
    const uint32_t mask = (1u << half) - 1u;
    uint64_t x = (uint64_t)j;
    do {
        uint32_t l = (uint32_t)(x >> half), r = (uint32_t)x & mask;
#pragma unroll
        for (int round = 0; round < 4; ++round) {
            const uint32_t t = l ^ (build_round(seed, round, r) & mask);
            l = r;
            r = t;
        }
        x = (uint64_t)l << half | r;
    } while (x >= (uint64_t)n);
    rows_out[j] = (int64_t)x;
}

static size_t up256(size_t b) { return (b + 255) & ~(size_t)255; }

int build_draw_samples(int64_t n, int64_t ns, uint64_t seed, int64_t* rows_out) {
    cudaStream_t s = ctx().stream;
    int half = 1;
    while (((int64_t)1 << (2 * half)) < n) ++half;
    size_t tmp_bytes = 0;
    VB_CUDA(cub::DeviceRadixSort::SortKeys(nullptr, tmp_bytes, (int64_t*)nullptr, (int64_t*)nullptr, ns, 0, 2 * half, s));
    Scratch sc("ivfflat build");
    void* mem;
    VB_TRY(sc.own(up256(8 * (size_t)ns) + tmp_bytes, &mem));
    int64_t* drawn = (int64_t*)mem;
    build_draw_kernel<<<(unsigned)((ns + 255) / 256), 256, 0, s>>>(n, ns, seed, half, drawn);
    VB_CUDA(cudaGetLastError());
    VB_CUDA(cub::DeviceRadixSort::SortKeys((uint8_t*)mem + up256(8 * (size_t)ns), tmp_bytes, drawn, rows_out, ns, 0, 2 * half, s));
    count_launch(2);
    return VB_OK;
}

// ----------------------------------------------------------------------------- placement
//
// Bound by HBM: every row is read once and written once.  A row that is only copied takes as many lanes as it has
// 16-byte words, up to a warp (8 lanes and 4 rows per warp for a 128-byte bit(1024) row, a full warp for 1536 and
// 6144 bytes), each lane keeping four loads in flight.  A row that is normalised takes a warp and element-wise
// accesses: its norm must carry the bits of vb_l2_normalize_batch (the stored rows of the cosine opclasses are compared
// with it bit for bit), and an fp64 sum is only reproducible in one order -- that kernel's: lane l adds elements
// l, l + 32, ... and a butterfly adds the lanes.

template <typename T>
__global__ void __launch_bounds__(256) place_copy_kernel(const uint8_t* __restrict__ src, size_t pitch, const int64_t* __restrict__ src_ids,
                                                         const int64_t* __restrict__ src_idx, const int64_t* __restrict__ dst_idx, int64_t m,
                                                         int lane_shift, int words, int raw, uint8_t* __restrict__ out, size_t out_stride,
                                                         int64_t* __restrict__ out_ids) {
    const int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    const int64_t j = t >> lane_shift;
    const int G = 1 << lane_shift, g = (int)t & (G - 1);
    if (j >= m) return;
    const int64_t s = src_idx ? src_idx[j] : j;
    const int64_t d = dst_idx ? dst_idx[j] : j;
    if (d < 0) return;
    const T* __restrict__ sp = reinterpret_cast<const T*>(src + (size_t)s * pitch);
    T* __restrict__ op = reinterpret_cast<T*>(out + (size_t)d * out_stride);
    int w = g;
    for (; w + 3 * G < words; w += 4 * G) {
        const T a = sp[w], b = sp[w + G], c = sp[w + 2 * G], e = sp[w + 3 * G];
        op[w] = a;
        op[w + G] = b;
        op[w + 2 * G] = c;
        op[w + 3 * G] = e;
    }
    for (; w < words; w += G) op[w] = sp[w];
    uint8_t* orow = out + (size_t)d * out_stride;
    for (int b = raw + g; b < (int)out_stride; b += G) orow[b] = 0;
    if (g == 0 && out_ids) out_ids[d] = src_ids ? src_ids[s] : s;
}

template <int ELEM>
__device__ __forceinline__ float place_elem(const uint8_t* row, int i) {
    return ELEM == VB_VECTOR ? reinterpret_cast<const float*>(row)[i] : __half2float(reinterpret_cast<const __half*>(row)[i]);
}

template <int ELEM>
__global__ void __launch_bounds__(256) place_normalize_kernel(const uint8_t* __restrict__ src, size_t pitch, const int64_t* __restrict__ src_ids,
                                                              const int64_t* __restrict__ src_idx, const int64_t* __restrict__ dst_idx,
                                                              int64_t m, int dim, uint8_t* __restrict__ out, size_t out_stride,
                                                              int64_t* __restrict__ out_ids, int32_t* __restrict__ zero) {
    const int64_t j = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (j >= m) return;
    const int64_t s = src_idx ? src_idx[j] : j;
    const int64_t d = !out ? -1 : dst_idx ? dst_idx[j] : j;   // no table: only the zero flags are wanted
    if (d < 0 && !zero) return;
    const uint8_t* row = src + (size_t)s * pitch;
    double sum = 0.0;
    for (int i = lane; i < dim; i += 32) {
        const double x = (double)place_elem<ELEM>(row, i);
        sum += x * x;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
    const double norm = sqrt(sum);
    if (zero && lane == 0) zero[j] = norm > 0 ? 0 : 1;
    if (d < 0) return;
    uint8_t* orow = out + (size_t)d * out_stride;
    const int padded = (int)(out_stride / (ELEM == VB_VECTOR ? 4 : 2));
    for (int i = lane; i < padded; i += 32) {
        // the quotient in double, narrowed to float (halfvec: then to half, to nearest even); a zero row stays zero
        const float v = i < dim && norm > 0 ? (float)((double)place_elem<ELEM>(row, i) / norm) : 0.f;
        if (ELEM == VB_VECTOR) reinterpret_cast<float*>(orow)[i] = v;
        else reinterpret_cast<__half*>(orow)[i] = __float2half_rn(v);
    }
    if (lane == 0 && out_ids) out_ids[d] = src_ids ? src_ids[s] : s;
}

int launch_place_rows(int elem, int dim, bool normalize, const void* src, size_t pitch, const int64_t* src_ids, const int64_t* src_idx,
                      const int64_t* dst_idx, int64_t m, uint8_t* out, size_t out_stride, int64_t* out_ids, int32_t* zero) {
    if (m <= 0) return VB_OK;
    cudaStream_t s = ctx().stream;
    const uint8_t* sp = (const uint8_t*)src;
    VB_REQUIRE(!normalize || elem != VB_BIT, "bit rows have no norm");
    if (normalize) {
        const unsigned grid = (unsigned)((m * 32 + 255) / 256);
        if (elem == VB_VECTOR)
            place_normalize_kernel<VB_VECTOR><<<grid, 256, 0, s>>>(sp, pitch, src_ids, src_idx, dst_idx, m, dim, out, out_stride, out_ids, zero);
        else
            place_normalize_kernel<VB_HALFVEC><<<grid, 256, 0, s>>>(sp, pitch, src_ids, src_idx, dst_idx, m, dim, out, out_stride, out_ids, zero);
    } else {
        // the widest word that divides the row bytes, the row pitch and the source address
        const int raw = (int)raw_row_bytes(elem, dim);
        const size_t bits = (size_t)raw | pitch | (size_t)(uintptr_t)sp | 16;
        const int W = (int)(bits & (~bits + 1));
        const int words = raw / W;
        int lane_shift = 0;
        while ((1 << lane_shift) < words && lane_shift < 5) ++lane_shift;
        const unsigned grid = (unsigned)(((m << lane_shift) + 255) / 256);
#define VB_PLACE(T) place_copy_kernel<T><<<grid, 256, 0, s>>>(sp, pitch, src_ids, src_idx, dst_idx, m, lane_shift, words, raw, out, out_stride, out_ids)
        if (W == 16) VB_PLACE(uint4);
        else if (W == 8) VB_PLACE(uint2);
        else if (W == 4) VB_PLACE(uint32_t);
        else if (W == 2) VB_PLACE(uint16_t);
        else VB_PLACE(uint8_t);
#undef VB_PLACE
    }
    VB_CUDA(cudaGetLastError());
    count_launch();
    return VB_OK;
}

// ----------------------------------------------------------------------------- skipped rows, compaction, destinations

__global__ void build_mark_kernel(const int32_t* __restrict__ zero, int64_t m, int32_t* __restrict__ lists) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i < m && zero[i]) lists[i] = -1;
}

int build_mark_skipped(const int32_t* zero, int64_t m, int32_t* lists) {
    if (m <= 0) return VB_OK;
    build_mark_kernel<<<(unsigned)((m + 255) / 256), 256, 0, ctx().stream>>>(zero, m, lists);
    VB_CUDA(cudaGetLastError());
    count_launch();
    return VB_OK;
}

__global__ void build_compact_kernel(const int32_t* __restrict__ zero, const int64_t* __restrict__ before, int64_t m,
                                     int64_t* __restrict__ dst, int64_t* __restrict__ kept) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= m) return;
    const int64_t pos = i - before[i];   // before[i] = dropped rows in front of row i
    dst[i] = zero[i] ? -1 : pos;
    if (i == m - 1) *kept = pos + (zero[i] ? 0 : 1);
}

int build_compact_map(const int32_t* zero, int64_t m, int64_t* dst, int64_t* kept) {
    cudaStream_t s = ctx().stream;
    size_t tmp_bytes = 0;
    VB_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, tmp_bytes, (const int32_t*)nullptr, (int64_t*)nullptr, m, s));
    Scratch sc("ivfflat build");
    void* mem;
    VB_TRY(sc.own(up256(8 * (size_t)m) + up256(8) + tmp_bytes, &mem));
    int64_t* before = (int64_t*)mem;
    int64_t* d_kept = (int64_t*)((uint8_t*)mem + up256(8 * (size_t)m));
    VB_CUDA(cub::DeviceScan::ExclusiveSum((uint8_t*)d_kept + up256(8), tmp_bytes, zero, before, m, s));
    build_compact_kernel<<<(unsigned)((m + 255) / 256), 256, 0, s>>>(zero, before, m, dst, d_kept);
    VB_CUDA(cudaGetLastError());
    count_launch(2);
    VB_CUDA(cudaMemcpyAsync(kept, d_kept, sizeof(int64_t), cudaMemcpyDeviceToHost, s));
    VB_CUDA(cudaStreamSynchronize(s));
    return VB_OK;
}

// sort key of a row: its list, the rows that are not indexed behind every list
__global__ void build_keys_kernel(const int32_t* __restrict__ lists_of_row, int64_t n, int lists, uint32_t* __restrict__ key,
                                  int64_t* __restrict__ row) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int32_t l = lists_of_row[i];
    key[i] = l < 0 ? (uint32_t)lists : (uint32_t)l;
    row[i] = i;
}

// list_off[l] = first image row whose key is >= l (l <= lists: list_off[lists] = the indexed rows)
__global__ void build_offsets_kernel(const uint32_t* __restrict__ sorted_key, int64_t n, int lists, int64_t* __restrict__ list_off) {
    const int l = blockIdx.x * blockDim.x + threadIdx.x;
    if (l > lists) return;
    int64_t lo = 0, hi = n;
    while (lo < hi) {
        const int64_t mid = (lo + hi) >> 1;
        if (sorted_key[mid] < (uint32_t)l) lo = mid + 1;
        else hi = mid;
    }
    list_off[l] = lo;
}

__global__ void build_dst_kernel(const int64_t* __restrict__ order, int64_t n, const int64_t* __restrict__ list_off, int lists,
                                 int64_t* __restrict__ dst) {
    const int64_t p = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (p < n) dst[order[p]] = p < list_off[lists] ? p : -1;
}

int build_destinations(const int32_t* lists_of_row, int64_t n, int lists, int64_t* order, int64_t* dst, int64_t* list_off_host) {
    cudaStream_t s = ctx().stream;
    int end_bit = 1;
    while ((1 << end_bit) <= lists) ++end_bit;
    size_t tmp_bytes = 0;
    VB_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, tmp_bytes, (uint32_t*)nullptr, (uint32_t*)nullptr, (int64_t*)nullptr,
                                            (int64_t*)nullptr, n, 0, end_bit, s));
    // the radix sort is stable: rows of one list stay in call order
    const size_t b_key = up256(4 * (size_t)n), b_row = up256(8 * (size_t)n), b_off = up256(8 * ((size_t)lists + 1));
    Scratch sc("ivfflat build");
    void* mem;
    VB_TRY(sc.own(2 * b_key + b_row + b_off + tmp_bytes, &mem));
    uint8_t* p = (uint8_t*)mem;
    uint32_t* key = (uint32_t*)p;
    uint32_t* sorted_key = (uint32_t*)(p + b_key);
    int64_t* row = (int64_t*)(p + 2 * b_key);
    int64_t* d_off = (int64_t*)(p + 2 * b_key + b_row);
    void* tmp = p + 2 * b_key + b_row + b_off;
    const unsigned grid = (unsigned)((n + 255) / 256);
    {
        ProfScope span(VB_PROF_BUILD_DEST);
        build_keys_kernel<<<grid, 256, 0, s>>>(lists_of_row, n, lists, key, row);
        VB_CUDA(cub::DeviceRadixSort::SortPairs(tmp, tmp_bytes, key, sorted_key, row, order, n, 0, end_bit, s));
        build_offsets_kernel<<<(unsigned)(lists / 256 + 1), 256, 0, s>>>(sorted_key, n, lists, d_off);
        build_dst_kernel<<<grid, 256, 0, s>>>(order, n, d_off, lists, dst);
    }
    VB_CUDA(cudaGetLastError());
    count_launch(4);
    VB_CUDA(cudaMemcpyAsync(list_off_host, d_off, 8 * ((size_t)lists + 1), cudaMemcpyDeviceToHost, s));
    VB_CUDA(cudaStreamSynchronize(s));
    return VB_OK;
}

}  // namespace vb
