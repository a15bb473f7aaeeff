// vb_assign_tc.cu -- nearest-centre assign on the Hopper tensor cores (wgmma).
//
// The assign pass (AddTupleToSort, src/ivfbuild.c:161-219) and the Lloyd assign step of
// k-means are the one GEMM-shaped part of the hot path: X[n x d] . C^T[d x k] followed by a
// row-argmin of  |c|^2 - 2 x.c  (L2 opclasses) or  -x.c  (ip / cosine opclasses).
//
// Precision.  The reference evaluates fp32 distances.  Tensor cores take bf16 operands, so
// both operands are split x = hi + lo (two bf16 planes, |lo| <= 2^-8 |hi|) and three MMAs per
// K step accumulate hi.hi + hi.lo + lo.hi in fp32 registers (the dropped lo.lo term is <= 2^-16 of
// |x||c|).  The epilogue keeps the best AND the second-best value of every row; rows whose
// margin is below a rigorous error bound are re-evaluated by the exact fp32 kernel
// (assign_exact_kernel), so the final list numbers equal the fp32 argmin.  halfvec rows are
// represented exactly by hi + lo (11-bit significand = 8 + 3).
//
// Kernel shape: CTA tile 128 rows x 256 centres, K step 64 (one 128-byte swizzle atom of bf16).
// Warps 0-7 are two consumer warpgroups, each issuing wgmma m64n256k16 for 64 rows of the tile
// (128 fp32 accumulators per thread) and then reducing its fragment to the row-argmin (each row is
// spread over the 4 lanes of a quad: one xor-shuffle merge at the end of the row tile); warp 8 is
// the bulk-copy producer feeding a 2 x 96 KB stage ring.
// Operands live in HBM already in the tiled, 128B-swizzled shared-memory image
// (pack_planes_kernel), so a stage is filled by two contiguous cp.async.bulk copies (A: 32 KB,
// B: 64 KB) that complete on an mbarrier -- TMA without tensor maps.
//
// Roofline: tensor pipe.  FLOPs = 2 n k d x 3 (three bf16 MMAs per fp32-accurate product).
#include "vb_tc.cuh"

#include <algorithm>
#include <cmath>
#include <cstring>
#include <vector>

namespace vb {

constexpr int TC_M = 128;       // rows per CTA tile (two warpgroups of 64)
constexpr int TC_N = 256;       // centres per tile (= wgmma N: 128 fp32 accumulator registers per thread)
constexpr int TC_STAGES = 2;
constexpr int TC_CONSUMERS = 256;
constexpr int TC_THREADS = TC_CONSUMERS + 32;   // + the producer warp
constexpr uint32_t A_PLANE_BYTES = TC_M * TC_K * 2;   // 16 KB
constexpr uint32_t B_PLANE_BYTES = TC_N * TC_K * 2;   // 32 KB
constexpr uint32_t A_STAGE_BYTES = 2 * A_PLANE_BYTES; // hi + lo
constexpr uint32_t B_STAGE_BYTES = 2 * B_PLANE_BYTES;
constexpr uint32_t STAGE_BYTES = A_STAGE_BYTES + B_STAGE_BYTES;  // 96 KB
constexpr size_t TC_SMEM = (size_t)TC_STAGES * STAGE_BYTES + 1024 /*align*/ + 256 /*barriers*/;

// ----------------------------------------------------------------------------- the GEMM + row-argmin kernel

struct TcArgs {
    const uint8_t* A;       // packed row planes of this slab: [m_tile][kb][2][128 x 64]
    const uint8_t* B;       // packed centre planes:            [n_tile][kb][2][256 x 64]
    const float* cn;        // |c|^2 per centre (padded centres = +inf), or zeros for inner product
    const float* xn;        // |x|^2 per row of the slab
    int n_mtiles, n_ntiles, n_kblocks;
    int64_t row0;           // first row of the slab (for output indices)
    int64_t n_rows;         // valid rows in the slab
    int k;                  // real centres
    int is_l2;              // 1: value = cn - 2 dot ; 0: value = -dot
    float cmax;             // max |c| over real centres
    float tol;              // relative error bound of the split-bf16 product
    float sum_tol;          // relative error bound of the fp32 norms / final sum (L2 form)
    int32_t* out_idx;       // [n] global
    int32_t* flagged;       // list of global row numbers needing the exact kernel
    int* n_flagged;
};

// (best, index, second best) of a row, merged across the lanes that hold other columns of it: the smaller value wins,
// the smaller centre number on equal values (the first minimum in centre order, src/ivfbuild.c:186-190)
__device__ __forceinline__ void merge_best(float& best, int& best_i, float& second, int lane_mask) {
    const float ob = __shfl_xor_sync(0xffffffffu, best, lane_mask);
    const int oi = __shfl_xor_sync(0xffffffffu, best_i, lane_mask);
    const float os = __shfl_xor_sync(0xffffffffu, second, lane_mask);
    if (ob < best || (ob == best && oi < best_i)) {
        second = fminf(best, os);
        best = ob;
        best_i = oi;
    } else {
        second = fminf(second, ob);
    }
}

__global__ void __launch_bounds__(TC_THREADS, 1) assign_tc_kernel(TcArgs a) {
    extern __shared__ uint8_t smem_raw[];
    // 1024-byte alignment for the 128B swizzle atoms
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem + (size_t)TC_STAGES * STAGE_BYTES);
    uint64_t* full_bar = bars;                    // [TC_STAGES]
    uint64_t* empty_bar = bars + TC_STAGES;       // [TC_STAGES]

    const int warp = threadIdx.x / 32, lane = threadIdx.x % 32;

    if (threadIdx.x == 0) {
        for (int s = 0; s < TC_STAGES; ++s) {
            mbar_init(&full_bar[s], 1);
            mbar_init(&empty_bar[s], TC_CONSUMERS / 32);   // one arrive per consumer warp
        }
        fence_barrier_init();
    }
    __syncthreads();

    const size_t a_tile_bytes = (size_t)a.n_kblocks * A_STAGE_BYTES;   // per m tile
    const size_t b_tile_bytes = (size_t)a.n_kblocks * B_STAGE_BYTES;   // per n tile

    if (warp == TC_CONSUMERS / 32) {
        // ===== producer: two bulk copies per stage; the warp runs converged and one elected lane issues =====
        const bool leader = elect_one();
        uint32_t it = 0;
        for (int mt = blockIdx.x; mt < a.n_mtiles; mt += gridDim.x)
            for (int nt = 0; nt < a.n_ntiles; ++nt)
                for (int kb = 0; kb < a.n_kblocks; ++kb, ++it) {
                    const int s = it % TC_STAGES;
                    const uint32_t ph = (it / TC_STAGES) & 1;
                    mbar_wait(&empty_bar[s], ph ^ 1);
                    uint8_t* sa = smem + (size_t)s * STAGE_BYTES;
                    uint8_t* sb = sa + A_STAGE_BYTES;
                    if (leader) {
                        mbar_arrive_expect_tx(&full_bar[s], STAGE_BYTES);
                        bulk_g2s(sa, a.A + (size_t)mt * a_tile_bytes + (size_t)kb * A_STAGE_BYTES, A_STAGE_BYTES, &full_bar[s]);
                        bulk_g2s(sb, a.B + (size_t)nt * b_tile_bytes + (size_t)kb * B_STAGE_BYTES, B_STAGE_BYTES, &full_bar[s]);
                    }
                    __syncwarp();
                }
    } else {
        // ===== consumers: warpgroup wg multiplies rows 64 wg .. 64 wg + 63 of the tile by all 256 centres, then keeps
        // the running best / second best of its two fragment rows over the centres it holds =====
        const int wg = warp / 4, t = threadIdx.x % 128;
        const int frag_row = 16 * (t / 32) + (t % 32) / 4;   // and frag_row + 8
        const int frag_col = 2 * (t % 4);
        uint32_t it = 0;
        for (int mt = blockIdx.x; mt < a.n_mtiles; mt += gridDim.x) {
            float best[2] = {INFINITY, INFINITY}, second[2] = {INFINITY, INFINITY};
            int best_i[2] = {0x7fffffff, 0x7fffffff};
            for (int nt = 0; nt < a.n_ntiles; ++nt) {
                float acc[TC_N / 2];
                for (int kb = 0; kb < a.n_kblocks; ++kb, ++it) {
                    const int s = it % TC_STAGES;
                    const uint32_t ph = (it / TC_STAGES) & 1;
                    mbar_wait(&full_bar[s], ph);
                    const uint32_t sa = smem_u32(smem + (size_t)s * STAGE_BYTES) + (uint32_t)wg * (64 * 128);
                    const uint32_t sb = smem_u32(smem + (size_t)s * STAGE_BYTES) + A_STAGE_BYTES;
                    const uint64_t da_hi = make_sw128_desc(sa), da_lo = make_sw128_desc(sa + A_PLANE_BYTES);
                    const uint64_t db_hi = make_sw128_desc(sb), db_lo = make_sw128_desc(sb + B_PLANE_BYTES);
                    wgmma_fence();
#pragma unroll
                    for (int k = 0; k < TC_K / 16; ++k) {
                        const uint64_t adv = (uint64_t)((k * 16 * 2) >> 4);   // 32 bytes per K step inside the atom
                        wgmma_bf16_n256(acc, da_hi + adv, db_hi + adv, (kb | k) != 0);
                        wgmma_bf16_n256(acc, da_hi + adv, db_lo + adv, 1);
                        wgmma_bf16_n256(acc, da_lo + adv, db_hi + adv, 1);
                    }
                    wgmma_commit();
                    wgmma_wait<0>();
                    __syncwarp();
                    if (lane == 0) mbar_arrive(&empty_bar[s]);   // smem stage reusable: this warp's MMAs have retired
                }
#pragma unroll
                for (int i = 0; i < TC_N / 2; ++i) {
                    const int h = (i / 2) % 2;
                    const int col = nt * TC_N + 8 * (i / 4) + frag_col + (i % 2);
                    const float dot = acc[i];
                    const float v = a.is_l2 ? fmaf(-2.f, dot, __ldg(a.cn + col)) : (col < a.k ? -dot : INFINITY);
                    if (v < best[h]) {            // strict <: first minimum wins (src/ivfbuild.c:186-190)
                        second[h] = best[h];
                        best[h] = v;
                        best_i[h] = col;
                    } else if (v < second[h]) {
                        second[h] = v;
                    }
                }
            }
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                merge_best(best[h], best_i[h], second[h], 1);
                merge_best(best[h], best_i[h], second[h], 2);
                const int64_t r_slab = (int64_t)mt * TC_M + wg * 64 + frag_row + 8 * h;
                if (t % 4 == 0 && r_slab < a.n_rows) {
                    const int64_t row = a.row0 + r_slab;
                    a.out_idx[row] = best_i[h] == 0x7fffffff ? 0 : best_i[h];
                    // error bound of the split product: |err(x.c)| <= tol |x| |c|  (both compared values carry it)
                    const float xnorm = sqrtf(a.xn[r_slab]);
                    const float eps = (a.is_l2 ? 4.f : 2.f) * a.tol * xnorm * a.cmax + (a.is_l2 ? a.sum_tol * (a.cmax * a.cmax + xnorm * xnorm) : 0.f);
                    if (!(second[h] - best[h] > eps)) {      // also catches NaN / Inf rows
                        int p = atomicAdd(a.n_flagged, 1);
                        a.flagged[p] = (int32_t)row;
                    }
                }
            }
        }
    }
}

// ----------------------------------------------------------------------------- host side

static bool g_tc_enabled = true;

int launch_assign_tc(const Table& X, int metric, const Table& Cn, int k, int32_t* out_idx) {
    Scratch sc;
    Context& c = ctx();
    cudaStream_t s = c.stream;
    const int km = key_metric(metric);
    const int is_l2 = km == VB_L2_SQUARED;
    const int dim = X.dim;
    const int n_kblocks = (dim + TC_K - 1) / TC_K;
    const int n_ntiles = (k + TC_N - 1) / TC_N;
    const int64_t n = X.n;
    if (n == 0) return VB_OK;

    // centres: packed planes + norms
    const size_t b_bytes = (size_t)n_ntiles * n_kblocks * B_STAGE_BYTES;
    void *d_B, *d_norms, *d_A, *d_flag;
    VB_TRY(sc.take(b_bytes, &d_B));
    const int64_t kpad = (int64_t)n_ntiles * TC_N;
    // slab of rows: a few tiles per SM
    const int64_t slab_tiles = (int64_t)c.sm_count * 4;
    const int64_t slab_rows = slab_tiles * TC_M;
    const size_t a_bytes = (size_t)slab_tiles * n_kblocks * A_STAGE_BYTES;
    VB_TRY(sc.take(a_bytes, &d_A));
    VB_TRY(sc.take(sizeof(float) * (size_t)(kpad + slab_rows) + 64, &d_norms));
    float* d_cn = (float*)d_norms;
    float* d_xn = d_cn + kpad;
    VB_TRY(sc.take(sizeof(int32_t) * (size_t)n + 64, &d_flag));
    int* d_nflag = (int*)d_flag;
    int32_t* d_flagged = (int32_t*)d_flag + 16;
    VB_CUDA(cudaMemsetAsync(d_nflag, 0, sizeof(int), s));

    {
        const int64_t chunks = kpad * n_kblocks * 8;
        const unsigned grid = (unsigned)((chunks + 255) / 256);
        if (X.elem == VB_VECTOR) pack_planes_kernel<VB_VECTOR><<<grid, 256, 0, s>>>(Cn.d, Cn.stride, 0, k, dim, TC_N, n_kblocks, (uint8_t*)d_B, nullptr);
        else pack_planes_kernel<VB_HALFVEC><<<grid, 256, 0, s>>>(Cn.d, Cn.stride, 0, k, dim, TC_N, n_kblocks, (uint8_t*)d_B, nullptr);
        const unsigned g2 = (unsigned)((kpad * 32 + 255) / 256);
        // padded centres get +inf so they never win; for inner product the kernel masks by index instead
        if (X.elem == VB_VECTOR) row_sqnorm_kernel<VB_VECTOR><<<g2, 256, 0, s>>>(Cn.d, Cn.stride, k, dim, d_cn, kpad, INFINITY);
        else row_sqnorm_kernel<VB_HALFVEC><<<g2, 256, 0, s>>>(Cn.d, Cn.stride, k, dim, d_cn, kpad, INFINITY);
        VB_CUDA(cudaGetLastError());
        count_launch(2);
    }
    // max |c| (host reduction of k floats; k <= 32768)
    std::vector<float> hcn((size_t)k);
    VB_CUDA(cudaMemcpyAsync(hcn.data(), d_cn, sizeof(float) * (size_t)k, cudaMemcpyDeviceToHost, s));
    VB_CUDA(cudaStreamSynchronize(s));
    float cmax2 = 0.f;
    for (float v : hcn) cmax2 = std::max(cmax2, v);

    static bool attr_set = false;
    if (!attr_set) {
        VB_CUDA(cudaFuncSetAttribute(assign_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)TC_SMEM));
        attr_set = true;
    }

    for (int64_t r0 = 0; r0 < n; r0 += slab_rows) {
        const int64_t rows = std::min(slab_rows, n - r0);
        const int n_mtiles = (int)((rows + TC_M - 1) / TC_M);
        const int64_t chunks = (int64_t)n_mtiles * TC_M * n_kblocks * 8;
        const unsigned grid = (unsigned)((chunks + 255) / 256);
        const unsigned g2 = (unsigned)((rows * 32 + 255) / 256);
        if (X.elem == VB_VECTOR) {
            pack_planes_kernel<VB_VECTOR><<<grid, 256, 0, s>>>(X.d, X.stride, r0, rows, dim, TC_M, n_kblocks, (uint8_t*)d_A, nullptr);
            row_sqnorm_kernel<VB_VECTOR><<<g2, 256, 0, s>>>(X.d + (size_t)r0 * X.stride, X.stride, rows, dim, d_xn, rows, 0.f);
        } else {
            pack_planes_kernel<VB_HALFVEC><<<grid, 256, 0, s>>>(X.d, X.stride, r0, rows, dim, TC_M, n_kblocks, (uint8_t*)d_A, nullptr);
            row_sqnorm_kernel<VB_HALFVEC><<<g2, 256, 0, s>>>(X.d + (size_t)r0 * X.stride, X.stride, rows, dim, d_xn, rows, 0.f);
        }
        TcArgs a{};
        a.A = (const uint8_t*)d_A;
        a.B = (const uint8_t*)d_B;
        a.cn = d_cn;
        a.xn = d_xn;
        a.n_mtiles = n_mtiles;
        a.n_ntiles = n_ntiles;
        a.n_kblocks = n_kblocks;
        a.row0 = r0;
        a.n_rows = rows;
        a.k = k;
        a.is_l2 = is_l2;
        a.cmax = std::sqrt(cmax2);
        // |err(x.c)| <= tol |x||c| for the split product (same derivation as lc_make_bound, vb_list_tc.cu):
        //   representation: hi.hi + hi.lo + lo.hi drops lo.lo and the two bf16 residuals: 3 * 2^-16;
        //   accumulation: one fp32 rounding of the accumulator per MMA, 3 MMAs per 16-element K step, 2^-23 each
        //     (truncation), doubled for the alignment of the 16 products inside an MMA -> 6 * (dim / 16) * 2^-23.
        // 2^-13 covers both up to ~1650 dimensions (the shapes validated in round 1); longer rows (ivfflat allows 2000
        // for vector, 4000 for halfvec) take the formula.  The fp32 norms |x|^2, |c|^2 are sums of dim / 32 terms per
        // lane plus a 5-step shuffle tree: (dim / 32 + 8) * 2^-23 relative, at least 1e-6.
        {
            const float steps = (float)(n_kblocks * (TC_K / 16));
            a.tol = std::max(1.0f / 8192.0f, 3.0f / 65536.0f + 6.0f * steps / 8388608.0f);
            a.sum_tol = std::max(1e-6f, ((float)dim / 32.0f + 8.0f) / 8388608.0f);
        }
        a.out_idx = out_idx;
        a.flagged = d_flagged;
        a.n_flagged = d_nflag;
        const int gridk = std::min(n_mtiles, c.sm_count);
        assign_tc_kernel<<<gridk, TC_THREADS, TC_SMEM, s>>>(a);
        VB_CUDA(cudaGetLastError());
        count_launch(3);
    }
    // exact re-check of the rows whose margin was inside the error bound
    int nflag = 0;
    VB_CUDA(cudaMemcpyAsync(&nflag, d_nflag, sizeof(int), cudaMemcpyDeviceToHost, s));
    VB_CUDA(cudaStreamSynchronize(s));
    if (nflag > 0) VB_TRY(launch_assign_exact(X, metric, Cn, k, d_flagged, nflag, out_idx, nullptr));
    c.last_assign_flagged = nflag;
    return VB_OK;
}

void set_tc_enabled(bool on) { g_tc_enabled = on; }

int launch_assign(const Table& X, int metric, const Table& Cn, int k, int32_t* out_idx) {
    const int km = key_metric(metric);
    const bool tc_ok = g_tc_enabled && X.elem != VB_BIT && (km == VB_L2_SQUARED || km == VB_NEG_IP) && X.n >= 1024 && k >= 16;
    if (tc_ok) return launch_assign_tc(X, metric, Cn, k, out_idx);
    // Hamming (integer popcount) and tiny problems stay on the exact CUDA-core kernel
    ctx().last_assign_flagged = -1;
    return launch_assign_exact(X, metric, Cn, k, nullptr, 0, out_idx, nullptr);
}

}  // namespace vb

extern "C" {
int vb_set_tensor_cores(int on) {
    vb::set_tc_enabled(on != 0);
    return VB_OK;
}
int64_t vb_last_assign_rechecked(void) { return vb::ctx().last_assign_flagged; }
int vb_set_option(const char* name, int64_t value) {
    if (!name) return VB_EINVAL;
    if (!strcmp(name, "scan_impl")) {
        vb::ctx().scan_impl = (int)value;
        return VB_OK;
    }
    if (!strcmp(name, "tc_level1")) {
        vb::ctx().tc_level1 = value != 0;
        return VB_OK;
    }
    if (!strcmp(name, "tc_level0")) {
        vb::ctx().tc_level0 = value != 0;
        return VB_OK;
    }
    if (!strcmp(name, "tc_levelp")) {
        vb::ctx().tc_levelp = value != 0;
        return VB_OK;
    }
    if (!strcmp(name, "pp_filter")) {
        vb::ctx().pp_filter = (int)value;
        return VB_OK;
    }
    if (!strcmp(name, "hnsw_l2_persist")) {
        vb::ctx().hnsw_l2_persist = value != 0;
        return VB_OK;
    }
    if (!strcmp(name, "one_query")) {
        vb::ctx().one_query = value != 0;
        return VB_OK;
    }
    if (!strcmp(name, "slab_select")) {
        vb::ctx().slab_select = value != 0;
        return VB_OK;
    }
    if (!strcmp(name, "hnsw_build_fraction")) {
        vb::ctx().hnsw_build_fraction = (int)std::max<int64_t>(1, value);
        return VB_OK;
    }
    if (!strcmp(name, "hnsw_build_batch")) {
        vb::ctx().hnsw_build_batch = (int)std::max<int64_t>(1, std::min<int64_t>(value, 1 << 20));
        return VB_OK;
    }
    if (!strcmp(name, "tensor_cores")) {
        vb::set_tc_enabled(value != 0);
        return VB_OK;
    }
    vb::set_error("unknown option %s", name);
    return VB_EINVAL;
}
}
