// vb_kmeans.cu -- IVFFlat build path on the device: nearest-centre assign (AddTupleToSort,
// src/ivfbuild.c:161-219), Lloyd k-means with the reference's centre-update rules
// (ComputeNewCenters, src/ivfkmeans.c:179-236) and k-means++ seeding (InitCenters, :23-91).
//
// This file holds the EXACT fp32 assign kernel: distances are accumulated as
// sum((x - c)^2) / sum(x * c) / popcount(x ^ c) in fp32 / integer, the same arithmetic
// as the reference's proc-1 functions, so argmin decisions match the CPU path up to
// fp32 reassociation.  It is compute bound on the CUDA cores (2 ops per element for L2);
// the tensor-core (wgmma) assign in vb_assign_tc.cu uses it to re-check near ties.
#include "vb_common.cuh"
#include "vb_distance.cuh"
#include <cuda_bf16.h>

#include <cub/cub.cuh>

#include <algorithm>
#include <cmath>
#include <cstring>
#include <vector>

namespace vb {

// ----------------------------------------------------------------------------- exact assign

constexpr int AT_M = 128, AT_N = 128, AT_K = 16, AT_THREADS = 256;

// four consecutive 32-bit "words" of a row starting at word w (w % 4 == 0): fp32 values, widened halves, or raw bit words
template <int ELEM>
__device__ __forceinline__ uint4 load_words4(const uint8_t* row, int w, int words) {
    if (w >= words) return make_uint4(0, 0, 0, 0);
    if (ELEM == VB_HALFVEC) {
        uint2 h = *reinterpret_cast<const uint2*>(row + (size_t)w * 2);
        float2 a = __half22float2(*reinterpret_cast<const __half2*>(&h.x));
        float2 b = __half22float2(*reinterpret_cast<const __half2*>(&h.y));
        return make_uint4(__float_as_uint(a.x), __float_as_uint(a.y), __float_as_uint(b.x), __float_as_uint(b.y));
    }
    return *reinterpret_cast<const uint4*>(row + (size_t)w * 4);
}

// KIND 0: sum (x-c)^2   1: -sum x*c   2: popcount(x ^ c)
template <int ELEM, int KIND>
__global__ void __launch_bounds__(AT_THREADS) assign_exact_kernel(const uint8_t* __restrict__ X, size_t xstride, int64_t n,
                                                                   const int32_t* __restrict__ row_sel, int64_t n_sel,
                                                                   const uint8_t* __restrict__ Cn, size_t cstride, int k_total, int words,
                                                                   int32_t* __restrict__ out_idx, float* __restrict__ out_val,
                                                                   int k_per_split, unsigned long long* __restrict__ packed,
                                                                   float* __restrict__ out_matrix, int64_t matrix_ld) {
    // blockIdx.y selects a slice of the centres (used when few rows are re-checked: keeps every SM busy);
    // slices are merged with a 64-bit atomicMin on (orderable value, centre number) = first minimum wins
    const int k_lo = blockIdx.y * k_per_split;
    const int k = min(k_total, k_lo + k_per_split);
    __shared__ uint32_t Xs[AT_K][AT_M + 4];
    __shared__ uint32_t Cs[AT_K][AT_N + 4];
    const int tid = threadIdx.x;
    const int tx = tid % 16, ty = tid / 16;
    const int64_t total = row_sel ? n_sel : n;
    const int64_t m0 = (int64_t)blockIdx.x * AT_M;

    float best_v[8];
    int best_i[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        best_v[i] = INFINITY;
        best_i[i] = 0x7fffffff;
    }
    // the two rows / centres this thread stages per K step
    const int lr = tid / 4;        // 0..63 (+64)
    const int lw = (tid % 4) * 4;  // word offset within the K step
    const uint8_t* xrow[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        int64_t r = m0 + lr + h * 64;
        if (r >= total) r = total - 1;
        if (row_sel) r = row_sel[r];
        xrow[h] = X + (size_t)r * xstride;
    }

    for (int n0 = k_lo; n0 < k; n0 += AT_N) {
        const uint8_t* crow[2];
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            int c = n0 + lr + h * 64;
            if (c >= k) c = k - 1;
            crow[h] = Cn + (size_t)c * cstride;
        }
        float acc[8][8];
        uint32_t uacc[8][8];
#pragma unroll
        for (int i = 0; i < 8; ++i)
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                acc[i][j] = 0.f;
                uacc[i][j] = 0;
            }
        for (int k0 = 0; k0 < words; k0 += AT_K) {
            uint4 xv[2], cv[2];
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                xv[h] = load_words4<ELEM>(xrow[h], k0 + lw, words);
                cv[h] = load_words4<ELEM>(crow[h], k0 + lw, words);
            }
            __syncthreads();
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                int r = lr + h * 64;
                Xs[lw + 0][r] = xv[h].x;
                Xs[lw + 1][r] = xv[h].y;
                Xs[lw + 2][r] = xv[h].z;
                Xs[lw + 3][r] = xv[h].w;
                Cs[lw + 0][r] = cv[h].x;
                Cs[lw + 1][r] = cv[h].y;
                Cs[lw + 2][r] = cv[h].z;
                Cs[lw + 3][r] = cv[h].w;
            }
            __syncthreads();
#pragma unroll
            for (int kk = 0; kk < AT_K; ++kk) {
                uint32_t a[8], b[8];
                *reinterpret_cast<uint4*>(&a[0]) = *reinterpret_cast<const uint4*>(&Xs[kk][ty * 8]);
                *reinterpret_cast<uint4*>(&a[4]) = *reinterpret_cast<const uint4*>(&Xs[kk][ty * 8 + 4]);
                *reinterpret_cast<uint4*>(&b[0]) = *reinterpret_cast<const uint4*>(&Cs[kk][tx * 8]);
                *reinterpret_cast<uint4*>(&b[4]) = *reinterpret_cast<const uint4*>(&Cs[kk][tx * 8 + 4]);
#pragma unroll
                for (int i = 0; i < 8; ++i)
#pragma unroll
                    for (int j = 0; j < 8; ++j) {
                        if (KIND == 0) {
                            float d = __uint_as_float(a[i]) - __uint_as_float(b[j]);
                            acc[i][j] = fmaf(d, d, acc[i][j]);
                        } else if (KIND == 1) {
                            acc[i][j] = fmaf(__uint_as_float(a[i]), __uint_as_float(b[j]), acc[i][j]);
                        } else {
                            uacc[i][j] += __popc(a[i] ^ b[j]);
                        }
                    }
            }
        }
        if (out_matrix) {
            // distance-matrix mode (batched centre scan of GetScanLists): write the tile, no argmin
#pragma unroll
            for (int i = 0; i < 8; ++i) {
                const int64_t r = m0 + ty * 8 + i;
                if (r >= total) continue;
                float* orow = out_matrix + r * matrix_ld;
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    const int c = n0 + tx * 8 + j;
                    if (c < k) orow[c] = KIND == 0 ? acc[i][j] : KIND == 1 ? -acc[i][j] : (float)uacc[i][j];
                }
            }
            continue;
        }
        // fold this centre tile into the running argmin: strict <, first minimum wins (src/ivfbuild.c:183-192)
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            float v = INFINITY;
            int vi = 0x7fffffff;
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                int c = n0 + tx * 8 + j;
                float d = KIND == 0 ? acc[i][j] : KIND == 1 ? -acc[i][j] : (float)uacc[i][j];
                if (c < k && d < v) {  // NaN / +Inf never win a strict <
                    v = d;
                    vi = c;
                }
            }
#pragma unroll
            for (int o = 8; o > 0; o >>= 1) {
                float ov = __shfl_xor_sync(0xffffffffu, v, o);
                int oi = __shfl_xor_sync(0xffffffffu, vi, o);
                if (ov < v || (ov == v && oi < vi)) {
                    v = ov;
                    vi = oi;
                }
            }
            if (v < best_v[i]) {
                best_v[i] = v;
                best_i[i] = vi;
            }
        }
    }
    if (out_matrix) return;
    if (tx == 0) {
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            int64_t r = m0 + ty * 8 + i;
            if (r < total) {
                if (packed) {
                    // rows that never saw a finite value keep the initial all-ones key (-> centre 0 in the finalize step)
                    if (best_i[i] != 0x7fffffff) {
                        uint32_t u = __float_as_uint(best_v[i]);
                        if (u == 0x80000000u) u = 0;
                        u = (u & 0x80000000u) ? ~u : (u | 0x80000000u);
                        atomicMin(&packed[r], ((unsigned long long)u << 32) | (unsigned)best_i[i]);
                    }
                } else {
                    int64_t dst = row_sel ? row_sel[r] : r;
                    // all-NaN / all-inf rows: closestCenter stays 0 like the reference (minDistance = DBL_MAX start)
                    out_idx[dst] = best_i[i] == 0x7fffffff ? 0 : best_i[i];
                    if (out_val) out_val[dst] = best_v[i];
                }
            }
        }
    }
}

__global__ void unpack_assign_kernel(const unsigned long long* __restrict__ packed, const int32_t* __restrict__ row_sel, int64_t total,
                                     int32_t* __restrict__ out_idx) {
    int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (r >= total) return;
    unsigned long long key = packed[r];
    int64_t dst = row_sel ? row_sel[r] : r;
    out_idx[dst] = key == ~0ull ? 0 : (int32_t)(unsigned)key;
}

static int assign_kind(int metric) {
    switch (key_metric(metric)) {
        case VB_L2_SQUARED: return 0;
        case VB_NEG_IP: return 1;
        case VB_HAMMING: return 2;
    }
    return -1;
}

// exact assign of all rows of X (or of the rows listed in row_sel) against k centres
int launch_assign_exact(const Table& X, int metric, const Table& Cn, int k, const int32_t* row_sel_dev, int64_t n_sel,
                        int32_t* out_idx, float* out_val) {
    Scratch sc;
    const int kind = assign_kind(metric);
    VB_REQUIRE(kind >= 0, "assign: unsupported metric %d", metric);
    const int64_t total = row_sel_dev ? n_sel : X.n;
    if (total <= 0 || k <= 0) return VB_OK;
    const int words = (int)(X.elem == VB_HALFVEC ? X.stride / 2 : X.stride / 4);
    const unsigned gx = (unsigned)((total + AT_M - 1) / AT_M);
    cudaStream_t s = ctx().stream;
    // few row tiles (a re-check of flagged rows): slice the centres over blockIdx.y so the grid covers the GPU
    int splits = 1;
    const int ktiles = (k + AT_N - 1) / AT_N;
    if (row_sel_dev && !out_val && (int)gx < ctx().sm_count) splits = std::min(ktiles, std::max(1, (2 * ctx().sm_count) / (int)gx));
    const int k_per_split = ((ktiles + splits - 1) / splits) * AT_N;
    splits = (k + k_per_split - 1) / k_per_split;
    unsigned long long* packed = nullptr;
    if (splits > 1) {
        void* p;
        VB_TRY(sc.take(sizeof(unsigned long long) * (size_t)total, &p));
        packed = (unsigned long long*)p;
        VB_CUDA(cudaMemsetAsync(packed, 0xFF, sizeof(unsigned long long) * (size_t)total, s));
    }
    const dim3 grid(gx, (unsigned)splits);
#define VB_ASSIGN(E, K)                                                                                                             \
    assign_exact_kernel<E, K><<<grid, AT_THREADS, 0, s>>>(X.d, X.stride, X.n, row_sel_dev, n_sel, Cn.d, Cn.stride, k, words, out_idx, \
                                                          out_val, k_per_split, packed, nullptr, 0)
    if (X.elem == VB_VECTOR) {
        if (kind == 0) VB_ASSIGN(VB_VECTOR, 0);
        else if (kind == 1) VB_ASSIGN(VB_VECTOR, 1);
        else VB_REQUIRE(false, "assign: Hamming needs bit rows");
    } else if (X.elem == VB_HALFVEC) {
        if (kind == 0) VB_ASSIGN(VB_HALFVEC, 0);
        else if (kind == 1) VB_ASSIGN(VB_HALFVEC, 1);
        else VB_REQUIRE(false, "assign: Hamming needs bit rows");
    } else {
        VB_REQUIRE(kind == 2, "assign: bit rows need the Hamming metric");
        VB_ASSIGN(VB_BIT, 2);
    }
#undef VB_ASSIGN
    VB_CUDA(cudaGetLastError());
    count_launch();
    if (packed) {
        unpack_assign_kernel<<<(unsigned)((total + 255) / 256), 256, 0, s>>>(packed, row_sel_dev, total, out_idx);
        VB_CUDA(cudaGetLastError());
        count_launch();
    }
    return VB_OK;
}

// Every row of X against every row of Cn -> out[x][c] (fp32 key metric), register-tiled: both operands are
// staged through shared memory once per 128 x 128 tile instead of once per (query, row chunk).  Used for the
// batched centre scan of GetScanLists (src/ivfscan.c:47-118) when many queries are searched at once.
int launch_distance_matrix(const Table& X, int metric, const Table& Cn, int k, float* out, int64_t ld) {
    const int kind = assign_kind(metric);
    VB_REQUIRE(kind >= 0 && X.elem == Cn.elem && X.stride == Cn.stride, "distance matrix: unsupported operands");
    if (X.n <= 0 || k <= 0) return VB_OK;
    const int words = (int)(X.elem == VB_HALFVEC ? X.stride / 2 : X.stride / 4);
    // one CTA per (128 queries, 128 centres) tile: outputs are disjoint, so centre slices need no merge
    const dim3 grid((unsigned)((X.n + AT_M - 1) / AT_M), (unsigned)((k + AT_N - 1) / AT_N));
    cudaStream_t s = ctx().stream;
    const int kps = AT_N;
#define VB_DM(E, K)                                                                                                                   \
    assign_exact_kernel<E, K><<<grid, AT_THREADS, 0, s>>>(X.d, X.stride, X.n, nullptr, 0, Cn.d, Cn.stride, k, words, nullptr, nullptr, \
                                                          kps, nullptr, out, ld)
    if (X.elem == VB_VECTOR) {
        if (kind == 0) VB_DM(VB_VECTOR, 0);
        else if (kind == 1) VB_DM(VB_VECTOR, 1);
        else VB_REQUIRE(false, "distance matrix: Hamming needs bit rows");
    } else if (X.elem == VB_HALFVEC) {
        if (kind == 0) VB_DM(VB_HALFVEC, 0);
        else if (kind == 1) VB_DM(VB_HALFVEC, 1);
        else VB_REQUIRE(false, "distance matrix: Hamming needs bit rows");
    } else {
        VB_REQUIRE(kind == 2, "distance matrix: bit rows need the Hamming metric");
        VB_DM(VB_BIT, 2);
    }
#undef VB_DM
    VB_CUDA(cudaGetLastError());
    count_launch();
    return VB_OK;
}

// Elkan only moves a sample when another centre is STRICTLY closer than its current one
// (src/ivfkmeans.c:431-444: "if (dxc < dxcx)"), so on an exact tie the sample keeps its centre,
// whereas a plain argmin would pick the lowest-numbered minimum.  After every Lloyd assign
// (except the initial one, which is a first-minimum-wins argmin in the reference as well,
// :324-344) each sample is re-scored against its previous centre and its new one with the same
// arithmetic, and stays put unless the new one is strictly closer.  Matters for Hamming (ties are
// the norm); measure-zero for float data.  One warp per sample.
template <int ELEM, int KIND>
__global__ void keep_previous_on_tie_kernel(const uint8_t* __restrict__ X, size_t xstride, int64_t n, const uint8_t* __restrict__ Cn,
                                            size_t cstride, int words, const int32_t* __restrict__ prev, int32_t* __restrict__ closest) {
    const int64_t i = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) / 32;
    const int lane = threadIdx.x % 32;
    if (i >= n) return;
    const int p = prev[i], c = closest[i];
    if (p == c) return;   // warp-uniform
    const uint8_t* x = X + (size_t)i * xstride;
    const uint8_t* cp = Cn + (size_t)p * cstride;
    const uint8_t* cc = Cn + (size_t)c * cstride;
    float fp = 0.f, fc = 0.f;
    uint32_t up = 0, uc = 0;
    for (int w = lane * 4; w < words; w += 128) {
        uint4 xv = load_words4<ELEM>(x, w, words), pv = load_words4<ELEM>(cp, w, words), cv = load_words4<ELEM>(cc, w, words);
        const uint32_t xs[4] = {xv.x, xv.y, xv.z, xv.w}, ps[4] = {pv.x, pv.y, pv.z, pv.w}, cs[4] = {cv.x, cv.y, cv.z, cv.w};
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            if (KIND == 0) {
                float a = __uint_as_float(xs[j]) - __uint_as_float(ps[j]), b = __uint_as_float(xs[j]) - __uint_as_float(cs[j]);
                fp = fmaf(a, a, fp);
                fc = fmaf(b, b, fc);
            } else if (KIND == 1) {
                fp = fmaf(__uint_as_float(xs[j]), __uint_as_float(ps[j]), fp);
                fc = fmaf(__uint_as_float(xs[j]), __uint_as_float(cs[j]), fc);
            } else {
                up += __popc(xs[j] ^ ps[j]);
                uc += __popc(xs[j] ^ cs[j]);
            }
        }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        fp += __shfl_xor_sync(0xffffffffu, fp, o);
        fc += __shfl_xor_sync(0xffffffffu, fc, o);
        up += __shfl_xor_sync(0xffffffffu, up, o);
        uc += __shfl_xor_sync(0xffffffffu, uc, o);
    }
    const float dp = KIND == 0 ? fp : KIND == 1 ? -fp : (float)up;
    const float dc = KIND == 0 ? fc : KIND == 1 ? -fc : (float)uc;
    if (lane == 0 && !(dc < dp)) closest[i] = p;
}

static int launch_keep_previous(const Table& X, int metric, const Table& Cn, const int32_t* prev, int32_t* closest) {
    const int kind = assign_kind(metric);
    if (X.n == 0) return VB_OK;
    const int words = (int)(X.elem == VB_HALFVEC ? X.stride / 2 : X.stride / 4);
    const unsigned grid = (unsigned)((X.n * 32 + 255) / 256);
    cudaStream_t s = ctx().stream;
#define VB_KEEP(E, K) keep_previous_on_tie_kernel<E, K><<<grid, 256, 0, s>>>(X.d, X.stride, X.n, Cn.d, Cn.stride, words, prev, closest)
    if (X.elem == VB_VECTOR) {
        if (kind == 0) VB_KEEP(VB_VECTOR, 0);
        else VB_KEEP(VB_VECTOR, 1);
    } else if (X.elem == VB_HALFVEC) {
        if (kind == 0) VB_KEEP(VB_HALFVEC, 0);
        else VB_KEEP(VB_HALFVEC, 1);
    } else {
        VB_KEEP(VB_BIT, 2);
    }
#undef VB_KEEP
    VB_CUDA(cudaGetLastError());
    count_launch();
    return VB_OK;
}

// ----------------------------------------------------------------------------- centre update

__global__ void count_and_diff_kernel(const int32_t* __restrict__ closest, int32_t* __restrict__ prev, int64_t n,
                                      int32_t* __restrict__ counts, int* __restrict__ changes, int first) {
    int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= n) return;
    int c = closest[i];
    atomicAdd(&counts[c], 1);
    if (!first && prev[i] != c) atomicAdd(changes, 1);
    prev[i] = c;
}

// stable counting sort of sample ids by cluster: position = start[c] + rank among equal c in index order.
// One thread per cluster walks the (small) assignment array; k threads x n reads is fine for k-means samples
// (n = 50 * k), and keeps member order = ascending sample index = the reference's summation order.
__global__ void members_kernel(const int32_t* __restrict__ closest, int64_t n, int k, const int32_t* __restrict__ start,
                               int32_t* __restrict__ members) {
    // warp per cluster: ballot-compaction keeps index order
    const int warp = (blockIdx.x * blockDim.x + threadIdx.x) / 32;
    const int lane = threadIdx.x % 32;
    if (warp >= k) return;
    int pos = start[warp];
    for (int64_t base = 0; base < n; base += 32) {
        int64_t i = base + lane;
        bool mine = i < n && closest[i] == warp;
        unsigned m = __ballot_sync(0xffffffffu, mine);
        if (mine) members[pos + __popc(m & ((1u << lane) - 1))] = (int32_t)i;
        pos += __popc(m);
    }
}

// agg[c][j] = sum over members in ascending sample order of x[j] (fp32, sequential like SumCenters, src/ivfkmeans.c:151-160)
template <int ELEM>
__global__ void sum_centers_kernel(const uint8_t* __restrict__ X, size_t xstride, int dim, const int32_t* __restrict__ members,
                                   const int32_t* __restrict__ start, const int32_t* __restrict__ counts,
                                   float* __restrict__ agg) {
    const int c = blockIdx.y;
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= dim) return;
    const int32_t* mem = members + start[c];
    const int cnt = counts[c];
    float s = 0.f;
    for (int t = 0; t < cnt; ++t) {
        const uint8_t* row = X + (size_t)mem[t] * xstride;
        float v;
        if (ELEM == VB_VECTOR) v = reinterpret_cast<const float*>(row)[j];
        else if (ELEM == VB_HALFVEC) v = __half2float(reinterpret_cast<const __half*>(row)[j]);
        else v = (float)((row[j >> 3] >> (7 - (j & 7))) & 1);   // BitSumCenter (src/ivfutils.c:363-370)
        s += v;
    }
    agg[(size_t)c * dim + j] = s;
}

__device__ __forceinline__ float hash_uniform(uint64_t seed, uint64_t a, uint64_t b) {
    // counter-based stand-in for RandomDouble() (pg_prng is PostgreSQL core; stream not reproduced)
    uint64_t z = seed + 0x9e3779b97f4a7c15ULL * (a * 0x100000001b3ULL + b + 1);
    z = (z ^ (z >> 30)) * 0xbf58476d1ce4e5b9ULL;
    z = (z ^ (z >> 27)) * 0x94d049bb133111ebULL;
    z ^= z >> 31;
    return (float)((double)(z >> 11) * (1.0 / 9007199254740992.0));
}

// divide by count, clamp +-Inf, re-seed empty clusters (src/ivfkmeans.c:203-228)
__global__ void finish_centers_kernel(float* __restrict__ agg, const int32_t* __restrict__ counts, int k, int dim,
                                      uint64_t seed, int iteration) {
    int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= (int64_t)k * dim) return;
    int c = (int)(i / dim), j = (int)(i % dim);
    int cnt = counts[c];
    float x = agg[i];
    if (cnt > 0) {
        if (isinf(x)) x = x > 0 ? 3.402823466e+38f : -3.402823466e+38f;
        x /= (float)cnt;
    } else {
        x = hash_uniform(seed, (uint64_t)iteration * k + c, j);
    }
    agg[i] = x;
}

// typed centre rows from fp32 aggregates (+ spherical renormalisation):
// {Vector,Halfvec,Bit}UpdateCenter (src/ivfutils.c:301-339), l2_normalize (src/vector.c:785-819, src/halfvec.c:725-759)
template <int ELEM>
__global__ void write_centers_kernel(const float* __restrict__ agg, int k, int dim, int spherical, uint8_t* __restrict__ Cn,
                                     size_t cstride) {
    const int c = blockIdx.x;
    const float* a = agg + (size_t)c * dim;
    uint8_t* row = Cn + (size_t)c * cstride;
    __shared__ double s_norm;
    __shared__ double red[32];
    if (ELEM == VB_BIT) {
        for (int b = threadIdx.x; b < (int)cstride; b += blockDim.x) {
            uint8_t v = 0;
            for (int t = 0; t < 8; ++t) {
                int j = b * 8 + t;
                if (j < dim && a[j] > 0.5f) v |= (uint8_t)(1u << (7 - t));
            }
            row[b] = v;
        }
        return;
    }
    double norm = 1.0;
    if (spherical) {
        // typed value first (half centres are rounded before normalising), norm accumulated in double
        double p = 0;
        for (int j = threadIdx.x; j < dim; j += blockDim.x) {
            float v = ELEM == VB_HALFVEC ? __half2float(__float2half_rn(a[j])) : a[j];
            p += (double)v * (double)v;
        }
        for (int o = 16; o > 0; o >>= 1) p += __shfl_xor_sync(0xffffffffu, p, o);
        if (threadIdx.x % 32 == 0) red[threadIdx.x / 32] = p;
        __syncthreads();
        if (threadIdx.x == 0) {
            double t = 0;
            for (int w = 0; w < (blockDim.x + 31) / 32; ++w) t += red[w];
            s_norm = sqrt(t);
        }
        __syncthreads();
        norm = s_norm;
    }
    const int padded = ELEM == VB_VECTOR ? (int)(cstride / 4) : (int)(cstride / 2);
    for (int j = threadIdx.x; j < padded; j += blockDim.x) {
        float v = j < dim ? a[j] : 0.f;
        if (ELEM == VB_HALFVEC) {
            __half h = __float2half_rn(v);
            if (spherical && j < dim) {
                // zero vector stays zero (src/halfvec.c:745)
                h = norm > 0 ? __float2half_rn((float)((double)__half2float(h) / norm)) : __float2half_rn(0.f);
            }
            reinterpret_cast<__half*>(row)[j] = h;
        } else {
            if (spherical && j < dim) v = norm > 0 ? (float)((double)v / norm) : 0.f;
            reinterpret_cast<float*>(row)[j] = v;
        }
    }
}

// device working set of one k-means run
struct KmeansState {
    Table centers;           // typed centre rows (padded)
    int32_t *closest = nullptr, *prev = nullptr, *counts = nullptr, *start = nullptr, *members = nullptr;
    float* agg = nullptr;
    int* changes = nullptr;
    void* scan_tmp = nullptr;
    size_t scan_tmp_bytes = 0;
};

static int kmeans_update_centers(const Table& X, KmeansState& st, int k, bool spherical, uint64_t seed, int iteration,
                                 vb_allreduce_fn allreduce, void* actx) {
    Context& c = ctx();
    cudaStream_t s = c.stream;
    const int dim = X.dim;
    // member lists in ascending sample order
    VB_CUDA(cub::DeviceScan::ExclusiveSum(st.scan_tmp, st.scan_tmp_bytes, st.counts, st.start, k, s));
    count_launch();
    if (X.n > 0) {
        members_kernel<<<(unsigned)((k * 32 + 255) / 256), 256, 0, s>>>(st.closest, X.n, k, st.start, st.members);
        VB_CUDA(cudaGetLastError());
        count_launch();
    }
    dim3 grid((unsigned)((dim + 127) / 128), (unsigned)k);
    if (X.elem == VB_VECTOR) sum_centers_kernel<VB_VECTOR><<<grid, 128, 0, s>>>(X.d, X.stride, dim, st.members, st.start, st.counts, st.agg);
    else if (X.elem == VB_HALFVEC) sum_centers_kernel<VB_HALFVEC><<<grid, 128, 0, s>>>(X.d, X.stride, dim, st.members, st.start, st.counts, st.agg);
    else sum_centers_kernel<VB_BIT><<<grid, 128, 0, s>>>(X.d, X.stride, dim, st.members, st.start, st.counts, st.agg);
    VB_CUDA(cudaGetLastError());
    count_launch();
    if (allreduce) {
        // sharded build: partial sums and counts of every rank are added (the only collective of the build)
        VB_CUDA(cudaStreamSynchronize(s));
        if (allreduce(st.agg, (int64_t)k * dim, 0, actx) != 0 || allreduce(st.counts, k, 1, actx) != 0) {
            set_error("allreduce hook failed");
            return VB_ESTATE;
        }
    } else if (comm_world() > 1) {
        // the library's own communicator: ncclAllReduce on the library stream, no host round trip
        VB_TRY(comm_allreduce(st.agg, (int64_t)k * dim, 0));
        VB_TRY(comm_allreduce(st.counts, k, 1));
    }
    finish_centers_kernel<<<(unsigned)(((int64_t)k * dim + 255) / 256), 256, 0, s>>>(st.agg, st.counts, k, dim, seed, iteration);
    VB_CUDA(cudaGetLastError());
    count_launch();
    if (X.elem == VB_VECTOR) write_centers_kernel<VB_VECTOR><<<k, 256, 0, s>>>(st.agg, k, dim, spherical, st.centers.d, st.centers.stride);
    else if (X.elem == VB_HALFVEC) write_centers_kernel<VB_HALFVEC><<<k, 256, 0, s>>>(st.agg, k, dim, spherical, st.centers.d, st.centers.stride);
    else write_centers_kernel<VB_BIT><<<k, 256, 0, s>>>(st.agg, k, dim, 0, st.centers.d, st.centers.stride);
    VB_CUDA(cudaGetLastError());
    count_launch();
    return VB_OK;
}


int kmeans_run(const Table& X, int kmeans_metric, void* centers_host, int k, int max_iter, uint64_t seed,
               vb_allreduce_fn allreduce, void* actx, int* iters_out) {
    Scratch sc;
    Context& c = ctx();
    cudaStream_t s = c.stream;
    const bool spherical = kmeans_metric == VB_SPHERICAL;
    int proc1;
    if (kmeans_metric == VB_L2) proc1 = VB_L2_SQUARED;           // argmin of sqrt(d2) == argmin of d2
    else if (kmeans_metric == VB_SPHERICAL) proc1 = VB_NEG_IP;   // acos(ip)/pi is decreasing in ip
    else if (kmeans_metric == VB_HAMMING) proc1 = VB_HAMMING;
    else VB_REQUIRE(false, "k-means distance must be L2, spherical or Hamming (opclass proc 3)");
    VB_REQUIRE((X.elem == VB_BIT) == (kmeans_metric == VB_HAMMING), "metric does not fit the element type");
    if (max_iter <= 0 || max_iter > 500) max_iter = 500;        // src/ivfkmeans.c:347

    KmeansState st;
    st.centers.elem = X.elem;
    st.centers.dim = X.dim;
    st.centers.stride = X.stride;
    const int64_t n = X.n;
    // The state of a run lives in ONE range of the scratch arena: nine cudaMalloc + cudaFree pairs per call cost more
    // than the five Lloyd iterations of config D on a context that holds a large table, and cudaFree synchronises the
    // device.
    size_t scan_tmp_bytes = 0;
    VB_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, scan_tmp_bytes, (int32_t*)nullptr, (int32_t*)nullptr, k, s));
    st.scan_tmp_bytes = scan_tmp_bytes;
    auto up = [](size_t b) { return (b + 255) & ~(size_t)255; };
    const size_t b_cent = up(X.stride * (size_t)k + 16), b_n = up(sizeof(int32_t) * (size_t)std::max<int64_t>(n, 1)),
                 b_k = up(sizeof(int32_t) * (size_t)k), b_agg = up(sizeof(float) * (size_t)k * X.dim), b_tmp = up(std::max<size_t>(scan_tmp_bytes, 16));
    void* arena;
    VB_TRY(sc.take(b_cent + 3 * b_n + 2 * b_k + b_agg + 256 + b_tmp, &arena));
    {
        uint8_t* p = (uint8_t*)arena;
        st.centers.d = p;                       // (table_append_host copies into it: capacity k, nothing to reserve)
        st.centers.cap = k;
        p += b_cent;
        st.closest = (int32_t*)p;
        p += b_n;
        st.prev = (int32_t*)p;
        p += b_n;
        st.members = (int32_t*)p;
        p += b_n;
        st.counts = (int32_t*)p;
        p += b_k;
        st.start = (int32_t*)p;
        p += b_k;
        st.agg = (float*)p;
        p += b_agg;
        st.changes = (int*)p;
        p += 256;
        st.scan_tmp = p;
    }
    auto cleanup = [&]() {};   // (the arena stays with the context)
    int rc = table_append_host(st.centers, centers_host, k);
    if (rc != VB_OK) return rc;

    int iteration = 0;
    rc = VB_OK;
    for (; iteration < max_iter; ++iteration) {
        prof_begin(VB_PROF_ASSIGN);
        rc = launch_assign(X, proc1, st.centers, k, st.closest);
        prof_end(VB_PROF_ASSIGN);
        if (rc != VB_OK) break;
        if (iteration > 0) {
            rc = launch_keep_previous(X, proc1, st.centers, st.prev, st.closest);
            if (rc != VB_OK) break;
        }
        cudaMemsetAsync(st.counts, 0, sizeof(int32_t) * (size_t)k, s);
        cudaMemsetAsync(st.changes, 0, sizeof(int), s);
        if (n > 0) {
            count_and_diff_kernel<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(st.closest, st.prev, n, st.counts, st.changes, iteration == 0);
            count_launch();
        }
        rc = kmeans_update_centers(X, st, k, spherical, seed, iteration, allreduce, actx);
        if (rc != VB_OK) break;
        int changes = 0;
        if (!allreduce && comm_world() > 1) {
            // every rank must take the same branch: sum the change counters on the device, before the read
            rc = comm_allreduce(st.changes, 1, 1);
            if (rc != VB_OK) break;
        }
        if (cudaMemcpyAsync(&changes, st.changes, sizeof(int), cudaMemcpyDeviceToHost, s) != cudaSuccess ||
            cudaStreamSynchronize(s) != cudaSuccess) {
            set_error("k-means: reading the change counter failed");
            rc = VB_ECUDA;
            break;
        }
        if (allreduce) {
            // every rank must take the same branch: sum the change counters
            if (cudaMemcpy(st.changes, &changes, sizeof(int), cudaMemcpyHostToDevice) != cudaSuccess ||
                allreduce(st.changes, 1, 1, actx) != 0 ||
                cudaMemcpy(&changes, st.changes, sizeof(int), cudaMemcpyDeviceToHost) != cudaSuccess) {
                set_error("k-means: change-counter allreduce failed");
                rc = VB_ESTATE;
                break;
            }
        }
        // src/ivfkmeans.c:482-483 (iteration 0 here = initial assignment + first pass of the reference)
        if (changes == 0 && iteration != 0) {
            ++iteration;
            break;
        }
    }
    if (rc == VB_OK) {
        const size_t raw = raw_row_bytes(X.elem, X.dim);
        cudaError_t ce = cudaMemcpy2DAsync(centers_host, raw, st.centers.d, st.centers.stride, raw, (size_t)k, cudaMemcpyDeviceToHost, s);
        if (ce == cudaSuccess) ce = cudaStreamSynchronize(s);
        if (ce != cudaSuccess) {
            set_error("k-means: copying centres back failed: %s", cudaGetErrorString(ce));
            rc = VB_ECUDA;
        }
    }
    if (iters_out) *iters_out = iteration;
    cleanup();
    return rc;
}

// ----------------------------------------------------------------------------- k-means++ seeding

// weight[j] = min(weight[j], d^2) with the reference's types (src/ivfkmeans.c:59-69); also emits the weights as double for the scan
__global__ void pp_weight_kernel(const float* __restrict__ key, int kmeans_metric, int64_t n, float* __restrict__ weight,
                                 double* __restrict__ wd) {
    int64_t j = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (j >= n) return;
    double distance;
    if (kmeans_metric == VB_L2) distance = sqrt((double)key[j]);
    else if (kmeans_metric == VB_SPHERICAL) {
        double d = -(double)key[j];
        if (d > 1) d = 1;
        else if (d < -1) d = -1;
        distance = acos(d) / 3.14159265358979323846;
    } else distance = (double)key[j];
    distance *= distance;
    float w = weight[j];
    if (distance < (double)w) w = (float)distance;
    weight[j] = w;
    wd[j] = (double)w;
}

// first j in [0, n-1) with choice - cumsum(w)[j] <= 0, else n-1 (src/ivfkmeans.c:77-83).  The uniform draw and the
// result stay on the device so a whole seeding run needs no host round trip per centre.
__global__ void pp_pick_kernel(const double* __restrict__ cum, int64_t n, const double* __restrict__ u, int64_t* __restrict__ picked) {
    if (blockIdx.x || threadIdx.x) return;
    double choice = cum[n - 1] * u[0];
    int64_t lo = 0, hi = n - 1;  // smallest j with cum[j] >= choice
    while (lo < hi) {
        int64_t mid = (lo + hi) >> 1;
        if (cum[mid] >= choice) hi = mid;
        else lo = mid + 1;
    }
    *picked = lo;
}

// pp_pick_kernel's search with 256 probes per step (three dependent steps for 2 * 10^5 samples instead of eighteen), then
// the picked row is copied to `row_out` (16-byte words) by the same CTA: one launch per round instead of two.
__global__ void __launch_bounds__(256) pp_pick_gather_kernel(const double* __restrict__ cum, int64_t n, const double* __restrict__ u,
                                                             int64_t* __restrict__ picked, const uint8_t* __restrict__ X, size_t stride,
                                                             uint8_t* __restrict__ row_out) {
    __shared__ int64_t s_lo, s_hi;
    __shared__ int s_first;
    const int t = threadIdx.x;
    const double choice = cum[n - 1] * u[0];
    if (t == 0) {
        s_lo = 0;
        s_hi = n - 1;
    }
    __syncthreads();
    for (;;) {
        const int64_t lo = s_lo, hi = s_hi;   // the answer (smallest j with cum[j] >= choice, else n - 1) is in [lo, hi]
        if (lo >= hi) break;
        const int64_t step = (hi - lo + 255) / 256;
        const int64_t p = min(hi, lo + (int64_t)t * step);
        const bool ge = cum[p] >= choice;
        if (t == 0) s_first = 256;
        __syncthreads();
        if (ge) atomicMin(&s_first, t);
        __syncthreads();
        const int first = s_first;
        __syncthreads();
        if (t == 0) {
            if (first == 0) {
                s_hi = lo;
            } else if (first == 256) {
                s_lo = min(hi, min(hi, lo + 255 * step) + 1);
            } else {
                s_lo = min(hi, lo + (int64_t)(first - 1) * step) + 1;
                s_hi = min(hi, lo + (int64_t)first * step);
            }
        }
        __syncthreads();
    }
    const int64_t row = s_lo;
    if (t == 0) *picked = row;
    const uint4* src = reinterpret_cast<const uint4*>(X + (size_t)row * stride);
    uint4* dst = reinterpret_cast<uint4*>(row_out);
    for (size_t v = t; v < stride / 16; v += 256) dst[v] = src[v];
}

// out[i] = first `bytes` bytes of row picks[i]; one block per picked row
__global__ void pp_gather_rows_kernel(const uint8_t* __restrict__ X, size_t stride, const int64_t* __restrict__ picks, size_t bytes,
                                      size_t out_stride, uint8_t* __restrict__ out) {
    const uint8_t* src = X + (size_t)picks[blockIdx.x] * stride;
    uint8_t* dst = out + (size_t)blockIdx.x * out_stride;
    for (size_t b = threadIdx.x; b < bytes; b += blockDim.x) dst[b] = src[b];
}

// ---- k-means++ distance pass with two exact filters (vector, L2) ------------------------------------------------------
//
// Round i needs w[j] = min(w[j], d(x_j, c_i)^2) for every sample; the reference computes all n distances
// (src/ivfkmeans.c:48-65, with a TODO to use the triangle inequality).  Here a sample is touched only when its weight
// could change:
//   1. triangle inequality over the chosen centres: d(x, c_i) >= d(c_near, c_i) - d(x, c_near), so
//      d(c_near(x), c_i) >= 2 sqrt(w(x)) leaves w(x) alone -- no row is read at all (needs near[j] and the i
//      centre-to-centre distances of the round);
//   2. a bf16 copy of the samples (half the bytes): d(x, c_i) >= d(x^, c_i) - |x - x^|, with |x - x^| stored per row.
// Only the samples that pass both are re-scored from their fp32 rows with the scan arithmetic, so the weights -- and the
// rows picked from the same draws -- are exactly those of the full pass (margins of 1e-5 cover fp32 rounding of the
// filter quantities; they only ever send a sample to the exact path, never past it).
struct PpFilter {
    __nv_bfloat16* xb = nullptr;   // [n][words] bf16 copy of the samples (words = padded dimension)
    float* ex = nullptr;           // [n] |x - x^| (upper bound)
    int32_t* near = nullptr;       // [n] chosen centre currently nearest
    float* dcc = nullptr;          // [k] distance of the newest centre to every earlier one (lower bounds)
    uint8_t* cent = nullptr;       // [k][stride] chosen centre rows
    unsigned long long* stats = nullptr;   // [3] samples skipped by (1), stopped by (2), re-scored exactly
    int words = 0;
};

__global__ void pp_prepare_bf16_kernel(const uint8_t* __restrict__ X, size_t stride, int words, int64_t n, __nv_bfloat16* __restrict__ xb,
                                       float* __restrict__ ex) {
    const int64_t j = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) / 32;
    const int lane = threadIdx.x % 32;
    if (j >= n) return;
    const float* x = reinterpret_cast<const float*>(X + (size_t)j * stride);
    __nv_bfloat16* o = xb + (size_t)j * words;
    float err = 0.f;
    for (int t = lane; t < words; t += 32) {
        const float v = x[t];
        const __nv_bfloat16 b = __float2bfloat16_rn(v);
        o[t] = b;
        const float d = v - __bfloat162float(b);
        err = fmaf(d, d, err);
    }
    for (int o2 = 16; o2 > 0; o2 >>= 1) err += __shfl_xor_sync(0xffffffffu, err, o2);
    if (lane == 0) ex[j] = sqrtf(err) * 1.0001f + 1e-30f;
}

// distance of the newest centre (fp32 row `cq`) to the earlier centres: one warp each, scan arithmetic
__global__ void pp_dcc_kernel(const uint8_t* __restrict__ cent, size_t stride, int V, const uint8_t* __restrict__ cq, int i,
                              float* __restrict__ dcc) {
    const int t = (int)((blockIdx.x * (int64_t)blockDim.x + threadIdx.x) / 32);
    const int lane = threadIdx.x % 32;
    if (t >= i) return;
    const uint4* rp = reinterpret_cast<const uint4*>(cent + (size_t)t * stride);
    const uint4* sq = reinterpret_cast<const uint4*>(cq);
    Acc<VB_VECTOR, VB_L2_SQUARED> acc;
    for (int v = lane; v < V; v += 32) acc.add(__ldg(rp + v), sq, v);
    acc.template reduce<32>();
    if (lane == 0) dcc[t] = sqrtf((float)acc.value()) * (1.f - 1e-5f);
}

constexpr int PPF_WARPS = 8;
// Persistent CTAs (the centre image is staged once per CTA, not once per 8 rows); a warp takes 32 consecutive samples at
// a time: the triangle test runs one sample per lane (coalesced reads of w / near, no row touched), the survivors are
// then visited one after the other by the whole warp for the bf16 bound and, if that cannot decide, the exact fp32
// distance.
__global__ void __launch_bounds__(PPF_WARPS * 32) pp_filtered_pass_kernel(const uint8_t* __restrict__ X, size_t stride, int V, PpFilter f,
                                                                          const uint8_t* __restrict__ cq, int i, int64_t n,
                                                                          float* __restrict__ w, double* __restrict__ wd) {
    // the newest centre twice: as it is (V vectors, for the exact pass) and, for the bf16 pass, de-interleaved into the
    // first and second float4 of every 8-element group -- lane v then reads c_a[v], c_b[v]: consecutive 16-byte words,
    // conflict-free.  (Reading c[v * 8 + t] from the plain image is an 8-way bank conflict on every load.)
    extern __shared__ uint4 ppf_sq[];
    float4* c_a = reinterpret_cast<float4*>(ppf_sq + V);
    float4* c_b = c_a + V / 2;
    for (int v = threadIdx.x; v < V; v += blockDim.x) {
        const uint4 x = reinterpret_cast<const uint4*>(cq)[v];
        ppf_sq[v] = x;
        const float4 c = make_float4(__uint_as_float(x.x), __uint_as_float(x.y), __uint_as_float(x.z), __uint_as_float(x.w));
        if (v & 1) c_b[v >> 1] = c;
        else c_a[v >> 1] = c;
    }
    __syncthreads();
    const int lane = threadIdx.x % 32;
    const int64_t gwarp = blockIdx.x * (int64_t)PPF_WARPS + threadIdx.x / 32;
    const int64_t nwarps = gridDim.x * (int64_t)PPF_WARPS;
    const int groups = f.words / 8;
    unsigned long long n_tri = 0, n_bf = 0, n_exact = 0;   // warp-uniform tallies, one atomic per warp at the end
    for (int64_t base = gwarp * 32; base < n; base += nwarps * 32) {
        const int64_t jl = base + lane;
        float wl = 0.f;
        bool pass = false;
        if (jl < n) {
            wl = w[jl];
            pass = i == 0 || !(f.dcc[f.near[jl]] >= 2.0002f * sqrtf(wl));
        }
        unsigned todo = __ballot_sync(0xffffffffu, pass);
        n_tri += (unsigned)__popc(__ballot_sync(0xffffffffu, jl < n)) - (unsigned)__popc(todo);
        while (todo) {
            const int r = __ffs(todo) - 1;
            todo &= todo - 1;
            const int64_t j = base + r;
            const float wj = __shfl_sync(0xffffffffu, wl, r);
            const float sj = sqrtf(wj);
            if (i > 0) {
                // bf16 lower bound: 8 elements per 16-byte load
                const uint4* xb = reinterpret_cast<const uint4*>(f.xb + (size_t)j * f.words);
                float acc = 0.f;
#pragma unroll 2
                for (int v = lane; v < groups; v += 32) {
                    const uint4 b = __ldg(xb + v);
                    const float4 ca = c_a[v], cb = c_b[v];
                    const float d0 = __uint_as_float(b.x << 16) - ca.x, d1 = __uint_as_float(b.x & 0xFFFF0000u) - ca.y;
                    const float d2 = __uint_as_float(b.y << 16) - ca.z, d3 = __uint_as_float(b.y & 0xFFFF0000u) - ca.w;
                    const float d4 = __uint_as_float(b.z << 16) - cb.x, d5 = __uint_as_float(b.z & 0xFFFF0000u) - cb.y;
                    const float d6 = __uint_as_float(b.w << 16) - cb.z, d7 = __uint_as_float(b.w & 0xFFFF0000u) - cb.w;
                    acc = fmaf(d0, d0, acc);
                    acc = fmaf(d1, d1, acc);
                    acc = fmaf(d2, d2, acc);
                    acc = fmaf(d3, d3, acc);
                    acc = fmaf(d4, d4, acc);
                    acc = fmaf(d5, d5, acc);
                    acc = fmaf(d6, d6, acc);
                    acc = fmaf(d7, d7, acc);
                }
                for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
                if (sqrtf(acc) * (1.f - 1e-5f) - f.ex[j] >= sj * (1.f + 1e-5f)) {
                    ++n_bf;
                    continue;
                }
            }
            // exact: the scan kernels' arithmetic (one row per warp pass), then the reference's weight rule (src/ivfkmeans.c:59-69)
            const uint4* rp = reinterpret_cast<const uint4*>(X + (size_t)j * stride);
            Acc<VB_VECTOR, VB_L2_SQUARED> a;
#pragma unroll 4
            for (int v = lane; v < V; v += 32) a.add(ldg_stream(rp + v), ppf_sq, v);
            a.template reduce<32>();
            ++n_exact;
            if (lane == 0) {
                double distance = sqrt((double)(float)a.value());
                distance *= distance;
                if (distance < (double)wj) {
                    const float nw = (float)distance;
                    w[j] = nw;
                    wd[j] = (double)nw;
                    f.near[j] = i;
                }
            }
        }
    }
    if (lane == 0) {
        if (n_tri) atomicAdd(&f.stats[0], n_tri);
        if (n_bf) atomicAdd(&f.stats[1], n_bf);
        if (n_exact) atomicAdd(&f.stats[2], n_exact);
    }
}

__global__ void pp_fill_f64_kernel(double* p, int64_t n, double v) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i < n) p[i] = v;
}

static bool pp_filter_applies(const Table& X, int kmeans_metric, int k) {
    // the filters pay off once the sample table is much larger than L2 and there are enough rounds to amortise the bf16 copy
    if (!ctx().pp_filter || X.elem != VB_VECTOR || kmeans_metric != VB_L2 || X.stride % 32 != 0) return false;
    return ctx().pp_filter == 2 || (k >= 64 && (size_t)X.n * X.stride >= ((size_t)256 << 20));   // 2 = forced (tests)
}

static int pp_filter_prepare(Scratch& sc, const Table& X, int k, double* d_wd, PpFilter* f) {
    cudaStream_t s = ctx().stream;
    const int64_t n = X.n;
    f->words = (int)(X.stride / 4);
    void *p_xb, *p_flt, *p_cent;
    VB_TRY(sc.take(sizeof(__nv_bfloat16) * (size_t)n * f->words, &p_xb));
    VB_TRY(sc.take((sizeof(float) + sizeof(int32_t)) * (size_t)n + sizeof(float) * (size_t)k + 64, &p_flt));
    VB_TRY(sc.take(X.stride * (size_t)k, &p_cent));
    f->xb = (__nv_bfloat16*)p_xb;
    f->ex = (float*)p_flt;
    f->near = (int32_t*)(f->ex + n);
    f->dcc = (float*)(f->near + n);
    f->stats = (unsigned long long*)((uint8_t*)(f->dcc + k) + ((8 - ((uintptr_t)(f->dcc + k) & 7)) & 7));
    f->cent = (uint8_t*)p_cent;
    VB_CUDA(cudaMemsetAsync(f->near, 0, sizeof(int32_t) * (size_t)n, s));
    VB_CUDA(cudaMemsetAsync(f->stats, 0, 3 * sizeof(unsigned long long), s));
    pp_prepare_bf16_kernel<<<(unsigned)((n * 32 + 255) / 256), 256, 0, s>>>(X.d, X.stride, f->words, n, f->xb, f->ex);
    pp_fill_f64_kernel<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(d_wd, n, 3.402823466e+38);
    VB_CUDA(cudaGetLastError());
    count_launch(2);
    return VB_OK;
}

// round i of the seeding on this process's samples: the newest centre's fp32 row is at crow (device, padded stride)
static int pp_filter_round(const Table& X, const PpFilter& f, const uint8_t* crow, int i, float* d_w, double* d_wd) {
    cudaStream_t s = ctx().stream;
    const int V = (int)(X.stride / 16);
    VB_CUDA(cudaMemcpyAsync(f.cent + (size_t)i * X.stride, crow, X.stride, cudaMemcpyDeviceToDevice, s));
    if (i > 0) pp_dcc_kernel<<<(unsigned)((i * 32 + 255) / 256), 256, 0, s>>>(f.cent, X.stride, V, crow, i, f.dcc);
    if (X.n > 0) {
        const size_t smem = 2 * X.stride;
        static bool attr = false;
        if (!attr && smem > 48 * 1024) {
            VB_CUDA(cudaFuncSetAttribute(pp_filtered_pass_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 64 * 1024));
            attr = true;
        }
        const int64_t want = (X.n + PPF_WARPS * 32 - 1) / (PPF_WARPS * 32);
        static int resident = 0;   // CTAs per SM at this shared-memory size (one wave: the kernel is persistent)
        if (resident == 0) {
            VB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&resident, pp_filtered_pass_kernel, PPF_WARPS * 32, smem));
            resident = std::max(1, resident);
        }
        const unsigned grid = (unsigned)std::min<int64_t>(want, (int64_t)ctx().sm_count * resident);
        pp_filtered_pass_kernel<<<grid, PPF_WARPS * 32, smem, s>>>(X.d, X.stride, V, f, crow, i, X.n, d_w,
                                                                                                          d_wd);
    }
    VB_CUDA(cudaGetLastError());
    count_launch(2);
    return VB_OK;
}

static double host_uniform(uint64_t* st) {
    uint64_t z = (*st += 0x9e3779b97f4a7c15ULL);
    z = (z ^ (z >> 30)) * 0xbf58476d1ce4e5b9ULL;
    z = (z ^ (z >> 27)) * 0x94d049bb133111ebULL;
    z ^= z >> 31;
    return (double)(z >> 11) * (1.0 / 9007199254740992.0);
}

// first_row / u: the draws of InitCenters (src/ivfkmeans.c:36, 78) when the caller supplies them (parity tests feed the
// oracle the same ones); otherwise they come from the seed.  picked_out (optional, host): the chosen sample rows.
int kmeans_pp(const Table& X, int kmeans_metric, void* centers_host, int k, uint64_t seed, int64_t first_row, const double* u_in,
              int64_t* picked_out) {
    Scratch sc;
    Context& c = ctx();
    cudaStream_t s = c.stream;
    const int64_t n = X.n;
    VB_REQUIRE(n > 0 && k > 0, "k-means++ needs samples");
    VB_REQUIRE(kmeans_metric == VB_L2 || kmeans_metric == VB_SPHERICAL || kmeans_metric == VB_HAMMING, "bad k-means metric");
    const int km = kmeans_metric == VB_L2 ? VB_L2_SQUARED : kmeans_metric == VB_SPHERICAL ? VB_NEG_IP : VB_HAMMING;
    const size_t raw = raw_row_bytes(X.elem, X.dim);
    void *d_key, *d_w, *d_wd, *d_cum, *d_picks, *d_u, *d_tmp, *d_q, *d_qraw, *d_out;
    VB_TRY(sc.take(sizeof(float) * (size_t)n, &d_key));
    VB_TRY(sc.take(sizeof(float) * (size_t)n, &d_w));
    VB_TRY(sc.take(sizeof(double) * (size_t)n, &d_wd));
    VB_TRY(sc.take(sizeof(double) * (size_t)n, &d_cum));
    VB_TRY(sc.take(sizeof(int64_t) * (size_t)k, &d_picks));
    VB_TRY(sc.take(sizeof(double) * (size_t)k, &d_u));
    VB_TRY(sc.take(X.stride, &d_qraw));
    VB_TRY(sc.take(raw * (size_t)k, &d_out));
    size_t tmp_bytes = 0;
    VB_CUDA(cub::DeviceScan::InclusiveSum(nullptr, tmp_bytes, (double*)d_wd, (double*)d_cum, (int)n, s));
    VB_TRY(sc.take(tmp_bytes, &d_tmp));
    // FLT_MAX start (src/ivfkmeans.c:39-40); every uniform draw is made up front, in the order the rounds consume them
    std::vector<float> w0((size_t)n, 3.402823466e+38f);
    uint64_t rs = seed ^ 0x5851f42d4c957f2dULL;
    int64_t first = (int64_t)(host_uniform(&rs) * (double)n);
    if (first >= n) first = n - 1;
    std::vector<double> u((size_t)k);
    for (int i = 0; i + 1 < k; ++i) u[(size_t)i] = host_uniform(&rs);
    if (first_row >= 0) first = std::min<int64_t>(first_row, n - 1);
    if (u_in)
        for (int i = 0; i + 1 < k; ++i) u[(size_t)i] = u_in[i];
    VB_CUDA(cudaMemcpyAsync(d_w, w0.data(), sizeof(float) * (size_t)n, cudaMemcpyHostToDevice, s));
    VB_CUDA(cudaMemcpyAsync(d_u, u.data(), sizeof(double) * (size_t)k, cudaMemcpyHostToDevice, s));
    VB_CUDA(cudaMemcpyAsync(d_picks, &first, sizeof(int64_t), cudaMemcpyHostToDevice, s));
    VB_CUDA(cudaStreamSynchronize(s));  // the host vectors above go out of use here
    const bool filtered = pp_filter_applies(X, kmeans_metric, k);
    PpFilter flt;
    if (filtered) VB_TRY(pp_filter_prepare(sc, X, k, (double*)d_wd, &flt));
    pp_gather_rows_kernel<<<1, 256, 0, s>>>(X.d, X.stride, (const int64_t*)d_picks, X.stride, X.stride, (uint8_t*)d_qraw);
    count_launch(1);
    for (int i = 0; i + 1 < k; ++i) {
        // distance of every sample to the newest centre (its row is in d_qraw): the scan kernel with that row as the query
        if (filtered) {
            VB_TRY(pp_filter_round(X, flt, (const uint8_t*)d_qraw, i, (float*)d_w, (double*)d_wd));
        } else {
            Scratch query;
            size_t qstride;
            VB_TRY(upload_queries(query, X.elem, X.dim, d_qraw, 1, false, &d_q, &qstride));
            VB_TRY(launch_scan_regular(X, km, d_q, qstride, 1, n, (float*)d_key, n));
            pp_weight_kernel<<<(unsigned)((n + 255) / 256), 256, 0, s>>>((const float*)d_key, kmeans_metric, n, (float*)d_w, (double*)d_wd);
        }
        VB_CUDA(cub::DeviceScan::InclusiveSum(d_tmp, tmp_bytes, (double*)d_wd, (double*)d_cum, (int)n, s));
        pp_pick_gather_kernel<<<1, 256, 0, s>>>((const double*)d_cum, n, (const double*)d_u + i, (int64_t*)d_picks + i + 1, X.d, X.stride,
                                                (uint8_t*)d_qraw);
        count_launch(3);
    }
    pp_gather_rows_kernel<<<(unsigned)k, 256, 0, s>>>(X.d, X.stride, (const int64_t*)d_picks, raw, raw, (uint8_t*)d_out);
    count_launch(1);
    VB_CUDA(cudaMemcpyAsync(centers_host, d_out, raw * (size_t)k, cudaMemcpyDeviceToHost, s));
    if (picked_out) VB_CUDA(cudaMemcpyAsync(picked_out, d_picks, sizeof(int64_t) * (size_t)k, cudaMemcpyDeviceToHost, s));
    if (filtered) VB_CUDA(cudaMemcpyAsync(c.pp_stats, flt.stats, 3 * sizeof(unsigned long long), cudaMemcpyDeviceToHost, s));
    else c.pp_stats[0] = c.pp_stats[1] = c.pp_stats[2] = 0;
    VB_CUDA(cudaStreamSynchronize(s));
    VB_CUDA(cudaGetLastError());
    return VB_OK;
}

// ----------------------------------------------------------------------------- k-means++ over row-sharded samples
//
// Every rank holds a slice of the samples (global sample order = rank order, then local order).  Per new centre:
// local distance pass + weight update + local prefix sums as in kmeans_pp; ncclAllGather of the local weight sums;
// every rank locates the owner of choice = u * total (the first rank whose running sum reaches it) on the device;
// the owner's pick kernel selects its local row, the others contribute zeros, and ncclAllReduce (uint32 sum of the
// row's bit pattern) hands the new centre to everybody -- no host round trip per centre.

__global__ void pp_pick_sharded_kernel(const double* __restrict__ cum, int64_t n_local, const double* __restrict__ sums, int world,
                                       int rank, const double* __restrict__ u, int64_t* __restrict__ picked_local,
                                       int64_t* __restrict__ picked_global, const int64_t* __restrict__ row_base) {
    if (blockIdx.x || threadIdx.x) return;
    double total = 0;
    for (int r = 0; r < world; ++r) total += sums[r];
    double choice = total * u[0];
    // owner: first rank whose running sum reaches the draw (the last rank takes what rounding leaves over)
    int owner = world - 1;
    double before = 0;
    for (int r = 0; r < world; ++r) {
        if (before + sums[r] >= choice && (sums[r] > 0 || r == world - 1)) {
            owner = r;
            break;
        }
        before += sums[r];
    }
    int64_t j = -1;
    if (owner == rank && n_local > 0) {
        const double local = choice - before;
        int64_t lo = 0, hi = n_local - 1;   // smallest j with cum[j] >= local, else the last row
        while (lo < hi) {
            int64_t mid = (lo + hi) >> 1;
            if (cum[mid] >= local) hi = mid;
            else lo = mid + 1;
        }
        j = lo;
    }
    *picked_local = j;
    if (picked_global) *picked_global = j >= 0 ? row_base[rank] + j : 0;   // summed over the ranks afterwards
}

// the picked row's bytes (owner) or zeros (everybody else), as uint32 words for the sum-allreduce
__global__ void pp_contribute_row_kernel(const uint8_t* __restrict__ X, size_t stride, const int64_t* __restrict__ picked_local,
                                         uint32_t* __restrict__ out, int words) {
    const int64_t j = *picked_local;
    const uint32_t* src = j >= 0 ? reinterpret_cast<const uint32_t*>(X + (size_t)j * stride) : nullptr;
    for (int w = blockIdx.x * blockDim.x + threadIdx.x; w < words; w += gridDim.x * blockDim.x) out[w] = src ? src[w] : 0u;
}

__global__ void pp_local_sum_kernel(const double* __restrict__ cum, int64_t n_local, double* __restrict__ out) {
    if (blockIdx.x || threadIdx.x) return;
    *out = n_local > 0 ? cum[n_local - 1] : 0.0;
}

__global__ void pp_store_centre_kernel(const uint8_t* __restrict__ row, size_t raw, uint8_t* __restrict__ out) {
    for (size_t b = threadIdx.x; b < raw; b += blockDim.x) out[b] = row[b];
}

static int kmeans_pp_sharded(const Table& X, int kmeans_metric, void* centers_host, int k, uint64_t seed, int64_t* picked_out) {
    Scratch sc;
    Context& c = ctx();
    cudaStream_t s = c.stream;
    const int world = comm_world(), rank = comm_rank();
    const int64_t n = X.n;
    VB_REQUIRE(k > 0, "k-means++ needs k > 0");
    VB_REQUIRE(kmeans_metric == VB_L2 || kmeans_metric == VB_SPHERICAL || kmeans_metric == VB_HAMMING, "bad k-means metric");
    const int km = kmeans_metric == VB_L2 ? VB_L2_SQUARED : kmeans_metric == VB_SPHERICAL ? VB_NEG_IP : VB_HAMMING;
    const size_t raw = raw_row_bytes(X.elem, X.dim);
    const int words = (int)(X.stride / 4);
    void *d_key, *d_w, *d_wd, *d_cum, *d_u, *d_tmp = nullptr, *d_q, *d_row, *d_out, *d_misc;
    VB_TRY(sc.take(sizeof(float) * (size_t)std::max<int64_t>(n, 1), &d_key));
    VB_TRY(sc.take(sizeof(float) * (size_t)std::max<int64_t>(n, 1), &d_w));
    VB_TRY(sc.take(sizeof(double) * (size_t)std::max<int64_t>(n, 1), &d_wd));
    VB_TRY(sc.take(sizeof(double) * (size_t)std::max<int64_t>(n, 1), &d_cum));
    VB_TRY(sc.take(sizeof(double) * (size_t)k, &d_u));
    VB_TRY(sc.take(X.stride, &d_row));
    VB_TRY(sc.take(raw * (size_t)k, &d_out));
    // misc: sums[world] doubles | local sum | row_base[world] | picked_local | picked_global[k]
    VB_TRY(sc.take(sizeof(double) * (size_t)(world + 1) + sizeof(int64_t) * (size_t)(world + 1 + k) + 64, &d_misc));
    double* d_sums = (double*)d_misc;
    double* d_lsum = d_sums + world;
    int64_t* d_base = (int64_t*)(d_lsum + 1);
    int64_t* d_pick = d_base + world;
    int64_t* d_gpick = d_pick + 1;
    size_t tmp_bytes = 0;
    if (n > 0) {
        VB_CUDA(cub::DeviceScan::InclusiveSum(nullptr, tmp_bytes, (double*)d_wd, (double*)d_cum, (int)n, s));
        VB_TRY(sc.take(tmp_bytes, &d_tmp));
    }
    // global row numbering: every rank learns every slice length (one exchange at the start)
    std::vector<int64_t> lens((size_t)world, 0), base((size_t)world, 0);
    {
        int64_t* d_len = d_gpick;   // borrowed before the rounds start
        VB_REQUIRE(k >= world, "k-means++ over %d ranks needs at least as many centres", world);
        VB_CUDA(cudaMemcpyAsync(d_len + rank, &n, sizeof(int64_t), cudaMemcpyHostToDevice, s));
        VB_TRY(comm_allgather(d_len + rank, d_len, sizeof(int64_t)));
        VB_CUDA(cudaMemcpyAsync(lens.data(), d_len, sizeof(int64_t) * (size_t)world, cudaMemcpyDeviceToHost, s));
        VB_CUDA(cudaStreamSynchronize(s));
    }
    int64_t n_total = 0;
    for (int r = 0; r < world; ++r) {
        base[(size_t)r] = n_total;
        n_total += lens[(size_t)r];
    }
    VB_REQUIRE(n_total > 0, "k-means++ needs samples");
    std::vector<float> w0((size_t)std::max<int64_t>(n, 1), 3.402823466e+38f);
    uint64_t rs = seed ^ 0x5851f42d4c957f2dULL;
    int64_t first = (int64_t)(host_uniform(&rs) * (double)n_total);
    if (first >= n_total) first = n_total - 1;
    std::vector<double> u((size_t)k);
    for (int i = 0; i + 1 < k; ++i) u[(size_t)i] = host_uniform(&rs);
    int64_t first_local = (first >= base[(size_t)rank] && first < base[(size_t)rank] + n) ? first - base[(size_t)rank] : -1;
    VB_CUDA(cudaMemcpyAsync(d_w, w0.data(), sizeof(float) * (size_t)std::max<int64_t>(n, 1), cudaMemcpyHostToDevice, s));
    VB_CUDA(cudaMemcpyAsync(d_u, u.data(), sizeof(double) * (size_t)k, cudaMemcpyHostToDevice, s));
    VB_CUDA(cudaMemcpyAsync(d_base, base.data(), sizeof(int64_t) * (size_t)world, cudaMemcpyHostToDevice, s));
    VB_CUDA(cudaMemcpyAsync(d_pick, &first_local, sizeof(int64_t), cudaMemcpyHostToDevice, s));
    int64_t first_contrib = first_local >= 0 ? first : 0;
    VB_CUDA(cudaMemcpyAsync(d_gpick, &first_contrib, sizeof(int64_t), cudaMemcpyHostToDevice, s));
    VB_CUDA(cudaStreamSynchronize(s));   // the host vectors above go out of use here
    // (every rank decides alike: the slices of a sharded sample set have the same shape; a rank without samples skips the pass)
    const bool filtered = n > 0 && ctx().pp_filter && X.elem == VB_VECTOR && kmeans_metric == VB_L2 && X.stride % 32 == 0 &&
                          (ctx().pp_filter == 2 || (k >= 64 && (size_t)n_total * X.stride >= ((size_t)256 << 20)));
    PpFilter flt;
    if (filtered) VB_TRY(pp_filter_prepare(sc, X, k, (double*)d_wd, &flt));
    for (int i = 0; i < k; ++i) {
        // centre i: the owner's row reaches every rank
        pp_contribute_row_kernel<<<4, 256, 0, s>>>(X.d, X.stride, d_pick, (uint32_t*)d_row, words);
        count_launch();
        VB_TRY(comm_allreduce(d_row, words, 4));
        pp_store_centre_kernel<<<1, 256, 0, s>>>((const uint8_t*)d_row, raw, (uint8_t*)d_out + (size_t)i * raw);
        count_launch();
        if (i + 1 == k) break;
        if (n > 0) {
            if (filtered) {
                VB_TRY(pp_filter_round(X, flt, (const uint8_t*)d_row, i, (float*)d_w, (double*)d_wd));
            } else {
                Scratch query;
                size_t qstride;
                VB_TRY(upload_queries(query, X.elem, X.dim, d_row, 1, false, &d_q, &qstride));
                VB_TRY(launch_scan_regular(X, km, d_q, qstride, 1, n, (float*)d_key, n));
                pp_weight_kernel<<<(unsigned)((n + 255) / 256), 256, 0, s>>>((const float*)d_key, kmeans_metric, n, (float*)d_w, (double*)d_wd);
            }
            VB_CUDA(cub::DeviceScan::InclusiveSum(d_tmp, tmp_bytes, (double*)d_wd, (double*)d_cum, (int)n, s));
            count_launch(2);
        }
        pp_local_sum_kernel<<<1, 1, 0, s>>>((const double*)d_cum, n, d_lsum);
        VB_TRY(comm_allgather(d_lsum, d_sums, sizeof(double)));
        pp_pick_sharded_kernel<<<1, 1, 0, s>>>((const double*)d_cum, n, d_sums, world, rank, (const double*)d_u + i, d_pick,
                                               d_gpick + i + 1, d_base);
        count_launch(2);
    }
    // global row numbers of the picks (each is non-zero on its owner only)
    VB_TRY(comm_allreduce(d_gpick, k, 2));
    VB_CUDA(cudaMemcpyAsync(centers_host, d_out, raw * (size_t)k, cudaMemcpyDeviceToHost, s));
    if (picked_out) VB_CUDA(cudaMemcpyAsync(picked_out, d_gpick, sizeof(int64_t) * (size_t)k, cudaMemcpyDeviceToHost, s));
    // this rank's filter tallies (vb_kmeans_pp_stats; the caller sums them over the ranks if it wants the totals)
    if (filtered) VB_CUDA(cudaMemcpyAsync(c.pp_stats, flt.stats, 3 * sizeof(unsigned long long), cudaMemcpyDeviceToHost, s));
    else c.pp_stats[0] = c.pp_stats[1] = c.pp_stats[2] = 0;
    VB_CUDA(cudaStreamSynchronize(s));
    VB_CUDA(cudaGetLastError());
    return VB_OK;
}

}  // namespace vb

using namespace vb;

extern "C" {

int vb_kmeans(vb_table* samples, int kmeans_metric, void* centers, int k, int max_iter, uint64_t seed, vb_allreduce_fn allreduce,
              void* allreduce_ctx, int* iters_out) {
    VB_TRY(require_init());
    VB_REQUIRE(samples && centers && k >= 1, "bad k-means arguments");
    return kmeans_run(samples->t, kmeans_metric, centers, k, max_iter, seed, allreduce, allreduce_ctx, iters_out);
}

int vb_kmeans_pp_init(vb_table* samples, int kmeans_metric, void* centers, int k, uint64_t seed) {
    VB_TRY(require_init());
    VB_REQUIRE(samples && centers && k >= 1, "bad k-means++ arguments");
    // with a communicator the samples are this rank's slice of a row-sharded sample set: every rank gets the same centres
    if (comm_world() > 1) return kmeans_pp_sharded(samples->t, kmeans_metric, centers, k, seed, nullptr);
    return kmeans_pp(samples->t, kmeans_metric, centers, k, seed);
}

int vb_kmeans_pp_stats(int64_t* out3) {
    VB_REQUIRE(out3, "null argument");
    for (int i = 0; i < 3; ++i) out3[i] = (int64_t)ctx().pp_stats[i];
    return VB_OK;
}

int vb_kmeans_pp_init_draws(vb_table* samples, int kmeans_metric, void* centers, int k, int64_t first_row, const double* u,
                            int64_t* picked_out) {
    VB_TRY(require_init());
    VB_REQUIRE(samples && centers && k >= 1 && first_row >= 0 && (u || k == 1), "bad k-means++ arguments");
    return kmeans_pp(samples->t, kmeans_metric, centers, k, 0, first_row, u, picked_out);
}

static int assign_impl(vb_table* rows, int metric, const void* centers, int k, bool host, int32_t* out) {
    VB_TRY(require_init());
    VB_REQUIRE(rows && centers && k >= 1 && out, "bad assign arguments");
    const Table& X = rows->t;
    VB_REQUIRE(metric == VB_L2_SQUARED || metric == VB_NEG_IP || metric == VB_HAMMING, "assign metric must be the opclass proc 1");
    VB_REQUIRE((X.elem == VB_BIT) == (metric == VB_HAMMING), "metric does not fit the element type");
    Table Cn;
    Cn.elem = X.elem;
    Cn.dim = X.dim;
    Cn.stride = X.stride;
    int rc = host ? table_append_host(Cn, centers, k) : table_append_dev(Cn, centers, k);
    int32_t* d_out = out;
    Scratch sc;
    void* ws = nullptr;
    if (rc == VB_OK && host) {
        rc = sc.take(sizeof(int32_t) * (size_t)std::max<int64_t>(X.n, 1), &ws);
        d_out = (int32_t*)ws;
    }
    if (rc == VB_OK) {
        prof_begin(VB_PROF_ASSIGN);
        rc = launch_assign(X, metric, Cn, k, d_out);
        prof_end(VB_PROF_ASSIGN);
    }
    if (rc == VB_OK && host && X.n > 0) {
        cudaError_t e = cudaMemcpyAsync(out, d_out, sizeof(int32_t) * (size_t)X.n, cudaMemcpyDeviceToHost, ctx().stream);
        if (e == cudaSuccess) e = cudaStreamSynchronize(ctx().stream);
        if (e != cudaSuccess) {
            set_error("assign: copy back failed: %s", cudaGetErrorString(e));
            rc = VB_ECUDA;
        }
    }
    if (rc == VB_OK && !host) cudaStreamSynchronize(ctx().stream);  // Cn is freed below
    table_free(Cn);
    return rc;
}

int vb_assign(vb_table* rows, int metric, const void* centers, int k, int32_t* out_list) {
    return assign_impl(rows, metric, centers, k, true, out_list);
}
int vb_assign_dev(vb_table* rows, int metric, const void* centers_dev, int k, int32_t* out_list_dev) {
    return assign_impl(rows, metric, centers_dev, k, false, out_list_dev);
}

}  // extern "C"
