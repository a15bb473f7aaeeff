// vb_list_proj.cu -- level P of the batched IVFFlat list scan: a projection lower bound in front of level 0.
//
// For any r x dim matrix P with spectral norm ||P||_2 <= sigma, |x - q|^2 >= |P(x - q)|^2 / sigma^2 for every row x and
// query q, whatever P is.  The basis only decides how tight the bound is: with the top principal directions of the
// index's own rows it is tight on data whose spectrum decays, and a filter pass then reads 4 r bytes per row instead of
// the int8 plane's dim.  The bound takes the place of d~ in level 0's listing refine with zero per-row terms: it
// re-scores the k smallest, then every other listed candidate with LB <= T1, and certifies with LB_{k'} > T.
//
// The basis is built once per image (list_proj_prepare): subspace iteration on the Gram matrix of a row sample (GEMMs on
// the device in double, QR on the host in double), r = the smallest multiple of 16 holding at least 90 % of the sample's
// energy about the origin, at most dim / 8; none (no level P) when no such r exists.  sigma^2 >= ||P||_2^2 comes from a
// Gershgorin bound on P P^T in double, so P need not be orthonormal.  Each row's y_x = P x (accumulated in double,
// rounded to fp32) is stored in list order; the queries are projected the same way per batch, and one pass over the
// projected plane (lp_scan_kernel) computes fl(sum_j (y_x,j - y_q,j)^2) for every probed (row, query) pair, turns it into a
// rigorous lower bound and takes the slab minima the refine selects from.
#include "vb_common.cuh"

#include <algorithm>
#include <cfloat>
#include <cmath>
#include <random>
#include <vector>

namespace vb {

// C[m][n] = sum_k A[k lda + m] B[k ldb + n] in double (16 x 16 tiles): the Gram matrix of the sample rows (A = B = the
// rows, lda = the sampling step in elements) and the product G B of one subspace iteration
template <typename T>
__global__ void lp_gemm_tn_kernel(const T* __restrict__ A, int64_t lda, const T* __restrict__ B, int64_t ldb, int64_t K, int M, int N,
                                  double* __restrict__ C) {
    __shared__ double As[16][17], Bs[16][17];
    const int tx = threadIdx.x, ty = threadIdx.y;
    const int am = blockIdx.y * 16 + tx, bn = blockIdx.x * 16 + tx;
    double acc = 0.0;
    for (int64_t k0 = 0; k0 < K; k0 += 16) {
        const int64_t k = k0 + ty;
        As[ty][tx] = k < K && am < M ? (double)A[k * lda + am] : 0.0;
        Bs[ty][tx] = k < K && bn < N ? (double)B[k * ldb + bn] : 0.0;
        __syncthreads();
#pragma unroll
        for (int kk = 0; kk < 16; ++kk) acc = fma(As[kk][ty], Bs[kk][tx], acc);
        __syncthreads();
    }
    const int m = blockIdx.y * 16 + ty, n = blockIdx.x * 16 + tx;
    if (m < M && n < N) C[(int64_t)m * N + n] = acc;
}

// y[row][c LP_PC + j] = fl32(sum_i P[c LP_PC + j][i] x[row][i]), the sum in double: one warp per (row, LP_PC components),
// lane l summing i = l, l + 32, ... in order, then an xor-shuffle tree.  The loads of LP_PU consecutive steps are issued
// before their FMAs.  (With a warp per 16 components and one step at a time, a batch's queries -- a warp each -- took 79 us
// at config B: 48 round trips in a row on 15 warps per SM.)  Rows past n (up to n_out) are zero.
constexpr int LP_PC = 4;
constexpr int LP_PU = 8;
__global__ void lp_project_kernel(const uint8_t* __restrict__ rows, size_t stride, int64_t n, int dim, const float* __restrict__ P, int r,
                                  float* __restrict__ y, int64_t n_out) {
    const int64_t w = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) / 32;
    const int lane = threadIdx.x % 32;
    const int chunks = r / LP_PC;
    const int64_t row = w / chunks;
    const int c = (int)(w % chunks);
    if (row >= n_out) return;
    double acc[LP_PC];
#pragma unroll
    for (int j = 0; j < LP_PC; ++j) acc[j] = 0.0;
    if (row < n) {
        const float* x = reinterpret_cast<const float*>(rows + (size_t)row * stride);
        const float* p = P + (size_t)c * LP_PC * dim;
        int i = lane;
        for (; i + 32 * (LP_PU - 1) < dim; i += 32 * LP_PU) {
            float xv[LP_PU], pv[LP_PU][LP_PC];
#pragma unroll
            for (int u = 0; u < LP_PU; ++u) {
                xv[u] = x[i + 32 * u];
#pragma unroll
                for (int j = 0; j < LP_PC; ++j) pv[u][j] = __ldg(p + (size_t)j * dim + i + 32 * u);
            }
#pragma unroll
            for (int u = 0; u < LP_PU; ++u)
#pragma unroll
                for (int j = 0; j < LP_PC; ++j) acc[j] = fma((double)pv[u][j], (double)xv[u], acc[j]);
        }
        for (; i < dim; i += 32) {
            const double xv = x[i];
#pragma unroll
            for (int j = 0; j < LP_PC; ++j) acc[j] = fma((double)__ldg(p + (size_t)j * dim + i), xv, acc[j]);
        }
#pragma unroll
        for (int j = 0; j < LP_PC; ++j)
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) acc[j] += __shfl_xor_sync(0xffffffffu, acc[j], o);
    }
    float v = 0.f;
#pragma unroll
    for (int j = 0; j < LP_PC; ++j)
        if (lane == j) v = (float)acc[j];
    if (lane < LP_PC) y[(size_t)row * r + c * LP_PC + lane] = v;
}

// The bound, from s = fl(sum_j fl(y^x_j - y^q_j)^2) (a sequential fmaf chain over the r components, as the list-major
// fp32 kernel list_tile_kernel computes it) with y^ the stored fp32 projections, u = 2^-24:
//   the sum: each difference rounds once (factor (1 + u)^2 on its square) and the chain of r fmaf rounds r times on
//     non-negative terms, so a = |y^x - y^q| satisfies a^2 >= s / ((1 + u)^(r + 2)) >= s c1, c1 = 1 - (r + 4) u;
//   the projections: y^ = fl32(y~) with y~ the double sum, |y^_j - y~_j| <= u |y~_j| and |y~_j - (P x)_j| <= dim 2^-53
//     (1.01) |p_j| |x|, so |y^x - P x| <= |x| (u sigma (1 + u) + dim 2^-52 ||P||_F) =: c_e |x|, and the same for q;
//   then |P(x - q)| >= a - c_e (|x| + |q|) >= a - delta(q), delta(q) = c_e (xmax + |q|) (1 + 2^-10) covering the
//     fp32 norms, and |x - q|^2 >= |P(x - q)|^2 / sigma^2;
//   the distance it is compared with is the fp32 sum over dim squared differences (the refine's re-score, the oracle):
//     d_fp32 >= |x - q|^2 (1 - (dim + 8) u) in any summation order.
// So LB = (max(0, sqrt(s c1) - delta))^2 c2, c2 = (1 - (dim + 8) u) / sigma^2 rounded down, every fp32 step rounded down
// (__fmul_rd, __fsqrt_rd, __fsub_rd), is <= d_fp32.  A sum that overflowed is taken as FLT_MAX (the exact one is above it);
// NaN stays NaN (the refine re-scores it and the certificate fails).
struct LpBound {
    float c1, c2, ce, xmax;
};

constexpr int LP_ROWS = 128;             // one table tile (a ListUnit): 4 warps, each one table-aligned 32-row slab
constexpr int LP_XP = LP_ROWS + 2;       // line of one component across the tile; +2 words make the transposing stores conflict-free
constexpr int LP_QC = 32;                // queries staged per chunk

struct LpScanArgs {
    const float* y;              // [rows][r] projections of the rows, list order
    const float* yq;             // [nq][r] projections of the queries
    const ListUnit* units;
    const int64_t* list_off;
    const int32_t* grp_begin;
    const int32_t* grp_cnt;
    const int32_t* pair_q;
    const int64_t* pair_out;
    const int32_t* pair_sbase;
    const float* qn;             // |q|^2
    float* out;                  // the per-query candidate runs
    float* smin;                 // slab minima (slab_base(), vb_common.cuh)
    LpBound b;
    int r;
};

static size_t lp_scan_smem(int r) { return sizeof(float) * (size_t)r * (LP_XP + LP_QC); }

// NQ queries (columns j0 .. j0 + NQ - 1 of the staged chunk; all of them real when FULL, else the first nqt - j0) against
// the thread's row: the distance chains, then per query the bound and its store, and the slab minima, which lane j
// collects for query j0 + j and stores once.  The minimum is taken on the bit patterns: every bound is +0, positive, +inf
// or NaN (mapped to the canonical 0x7FFFFFFF, above +inf), whose unsigned order is fminf's, NaN ignored unless the whole
// slab is NaN -- and min is exact, so any reduction order gives the bits of fminf's butterfly.
template <int NQ, bool FULL>
__device__ __forceinline__ void lp_block(const float* __restrict__ Xs, const float* __restrict__ Qs, int r, int j0, int nqt, int tid,
                                         bool valid, float* const* s_outp, const float* s_delta, float* __restrict__ smin,
                                         const int32_t* s_sb, int64_t slab, const LpBound& b) {
    float s[NQ];
#pragma unroll
    for (int j = 0; j < NQ; ++j) s[j] = 0.f;
    for (int d0 = 0; d0 < r; d0 += 16) {
#pragma unroll
        for (int dd = 0; dd < 16; ++dd) {
            const int d = d0 + dd;
            const float x = Xs[d * LP_XP + tid];
            float nq[NQ];
#pragma unroll
            for (int j = 0; j < NQ; j += 4) {
                const float4 q4 = *reinterpret_cast<const float4*>(&Qs[d * LP_QC + j0 + j]);
                nq[j] = q4.x;
                nq[j + 1] = q4.y;
                nq[j + 2] = q4.z;
                nq[j + 3] = q4.w;
            }
#pragma unroll
            for (int j = 0; j < NQ; ++j) {
                const float e = __fadd_rn(x, nq[j]);
                s[j] = __fmaf_rn(e, e, s[j]);
            }
        }
    }
    const int lane = tid % 32;
    const int nv = FULL ? NQ : nqt - j0;
    unsigned mine = 0u;
#pragma unroll
    for (int j = 0; j < NQ; ++j) {
        if (!FULL && j >= nv) break;   // block-uniform
        float sj = s[j];
        if (sj > FLT_MAX) sj = FLT_MAX;
        float t = __fsub_rd(__fsqrt_rd(__fmul_rd(sj, b.c1)), s_delta[j0 + j]);
        if (t < 0.f) t = 0.f;
        const float v = __fmul_rd(__fmul_rd(t, t), b.c2);
        if (valid) s_outp[j0 + j][tid] = v;
        const unsigned key = !valid ? 0x7F800000u : v != v ? 0x7FFFFFFFu : __float_as_uint(v);
        const unsigned m = __reduce_min_sync(0xffffffffu, key);
        if (lane == j) mine = m;
    }
    if (lane < nv) smin[s_sb[j0 + lane] + slab] = __uint_as_float(mine);
}

// One CTA per (list, 128-row table tile) unit against every query probing the list: the tile's projected rows are read
// once, coalesced, into a transposed shared tile, the queries' projections follow in chunks of LP_QC, and each thread
// (one row) runs up to 8 queries at a time.  Per (row, query): s = fmaf(d, d, s) over j = 0 .. r - 1 from 0 with
// d = y_x,j + (-y_q,j) (list_tile_kernel's chain, bit for bit), then the bound above stored at pair_out + (row - lo), one
// coalesced 128-byte store per (warp, query), and the minimum over the warp's slab (rows outside the list: +inf, nothing
// stored).
__global__ void __launch_bounds__(LP_ROWS) lp_scan_kernel(LpScanArgs a) {
    const ListUnit un = a.units[blockIdx.x];
    const int cnt = a.grp_cnt[un.list];
    if (cnt == 0) return;   // list not probed by this batch

    extern __shared__ __align__(16) float lp_smem[];
    const int r = a.r, r4 = a.r / 4;
    float* Xs = lp_smem;                 // [r][LP_XP] the tile's rows, transposed
    float* Qs = lp_smem + r * LP_XP;     // [r][LP_QC] the chunk's queries, negated, transposed
    __shared__ int32_t s_q[LP_QC];
    __shared__ int32_t s_sb[LP_QC];
    __shared__ float* s_outp[LP_QC];     // the run entry of the tile's row t0 (thread 0's)
    __shared__ float s_delta[LP_QC];

    const int tid = threadIdx.x, warp = tid / 32;
    const int64_t lo = a.list_off[un.list], hi = a.list_off[un.list + 1];
    const int64_t t0 = (int64_t)un.tile * LP_ROWS, row = t0 + tid, s0 = t0 + 32 * warp;
    const bool valid = row >= lo && row < hi;
    const bool warp_rows = s0 < hi && s0 + 32 > lo;   // warp-uniform
    const int64_t slab = (s0 >> 5) - (lo >> 5);
    const int gb = a.grp_begin[un.list];
    const LpBound b = a.b;

    {
        const float4* src = reinterpret_cast<const float4*>(a.y + (size_t)t0 * r);
        for (int i = tid; i < LP_ROWS * r4; i += LP_ROWS) {
            const int rr = i / r4, c = 4 * (i - rr * r4);
            float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
            if (t0 + rr >= lo && t0 + rr < hi) v = __ldg(src + i);
            Xs[(c + 0) * LP_XP + rr] = v.x;
            Xs[(c + 1) * LP_XP + rr] = v.y;
            Xs[(c + 2) * LP_XP + rr] = v.z;
            Xs[(c + 3) * LP_XP + rr] = v.w;
        }
    }

    for (int c0 = 0; c0 < cnt; c0 += LP_QC) {
        const int nqt = min(LP_QC, cnt - c0);
        __syncthreads();   // the previous chunk is done with Qs and the pair arrays
        if (tid < LP_QC) {
            const int sl = gb + c0 + min(tid, nqt - 1);   // the chunk's last query fills the unused columns
            const int q = a.pair_q[sl];
            s_q[tid] = q;
            s_outp[tid] = a.out + a.pair_out[sl] + (t0 - lo);
            s_sb[tid] = a.pair_sbase[sl];
            s_delta[tid] = __fmul_ru(b.ce, __fadd_ru(b.xmax, __fmul_ru(__fsqrt_ru(a.qn[q]), 1.0f + 1.0f / 1024.0f)));
        }
        __syncthreads();
        for (int i = tid; i < LP_QC * r4; i += LP_ROWS) {
            const int j = i / r4, c4 = i - j * r4;
            const float4 v = __ldg(reinterpret_cast<const float4*>(a.yq + (size_t)s_q[j] * r) + c4);
            Qs[(4 * c4 + 0) * LP_QC + j] = -v.x;
            Qs[(4 * c4 + 1) * LP_QC + j] = -v.y;
            Qs[(4 * c4 + 2) * LP_QC + j] = -v.z;
            Qs[(4 * c4 + 3) * LP_QC + j] = -v.w;
        }
        __syncthreads();
        if (!warp_rows) continue;
        int j0 = 0;
        for (; j0 + 8 <= nqt; j0 += 8) lp_block<8, true>(Xs, Qs, r, j0, nqt, tid, valid, s_outp, s_delta, a.smin, s_sb, slab, b);
        if (nqt - j0 > 4) lp_block<8, false>(Xs, Qs, r, j0, nqt, tid, valid, s_outp, s_delta, a.smin, s_sb, slab, b);
        else if (nqt - j0 == 4) lp_block<4, true>(Xs, Qs, r, j0, nqt, tid, valid, s_outp, s_delta, a.smin, s_sb, slab, b);
        else if (nqt > j0) lp_block<4, false>(Xs, Qs, r, j0, nqt, tid, valid, s_outp, s_delta, a.smin, s_sb, slab, b);
    }
}

// ----------------------------------------------------------------------------- host side

static int lp_gemm(const float* A, int64_t lda, int64_t K, int M, double* C, cudaStream_t s) {
    dim3 grid((unsigned)((M + 15) / 16), (unsigned)((M + 15) / 16));
    lp_gemm_tn_kernel<float><<<grid, dim3(16, 16), 0, s>>>(A, lda, A, lda, K, M, M, C);
    VB_CUDA(cudaGetLastError());
    count_launch();
    return VB_OK;
}
static int lp_gemm(const double* G, int dim, const double* B, int N, double* C, cudaStream_t s) {
    dim3 grid((unsigned)((N + 15) / 16), (unsigned)((dim + 15) / 16));
    lp_gemm_tn_kernel<double><<<grid, dim3(16, 16), 0, s>>>(G, dim, B, N, dim, dim, N, C);
    VB_CUDA(cudaGetLastError());
    count_launch();
    return VB_OK;
}

// modified Gram-Schmidt, twice, on the columns of the dim x c block b (row-major)
static void lp_orthonormalise(std::vector<double>& b, int dim, int c) {
    for (int pass = 0; pass < 2; ++pass)
        for (int j = 0; j < c; ++j) {
            for (int i = 0; i < j; ++i) {
                double d = 0.0;
                for (int e = 0; e < dim; ++e) d += b[(size_t)e * c + i] * b[(size_t)e * c + j];
                for (int e = 0; e < dim; ++e) b[(size_t)e * c + j] -= d * b[(size_t)e * c + i];
            }
            double nrm = 0.0;
            for (int e = 0; e < dim; ++e) nrm += b[(size_t)e * c + j] * b[(size_t)e * c + j];
            nrm = std::sqrt(nrm);
            for (int e = 0; e < dim; ++e) b[(size_t)e * c + j] = nrm > 0.0 ? b[(size_t)e * c + j] / nrm : 0.0;
        }
}

int list_proj_project(const Table& rows, const ListProj& lp, int64_t first_row, int64_t n_out) {
    if (n_out <= first_row) return VB_OK;
    const int64_t m = n_out - first_row;
    const int64_t warps = m * (lp.r / LP_PC);
    lp_project_kernel<<<(unsigned)((warps * 32 + 255) / 256), 256, 0, ctx().stream>>>(rows.d + (size_t)first_row * rows.stride, rows.stride,
                                                                                  std::max<int64_t>(rows.n - first_row, 0), rows.dim, lp.P, lp.r,
                                                                                  lp.y + (size_t)first_row * lp.r, m);
    VB_CUDA(cudaGetLastError());
    count_launch();
    return VB_OK;
}

int list_proj_prepare(const Table& rows, int n_lists, ListProj* lp) {
    Context& c = ctx();
    cudaStream_t s = c.stream;
    lp->tried = true;
    const int dim = rows.dim;
    const int cap_r = (dim / 8) / 16 * 16;
    if (rows.elem != VB_VECTOR || rows.n == 0 || cap_r < 16) return VB_OK;
    // the sample: every step-th row, as many as k-means samples (src/ivfbuild.c:448-452)
    const int64_t ns_want = std::min<int64_t>(rows.n, std::max<int64_t>((int64_t)n_lists * 50, 10000));
    const int64_t step = std::max<int64_t>(1, rows.n / ns_want);
    const int64_t ns = (rows.n + step - 1) / step;
    const int cb = cap_r;
    void* dev;
    const size_t g_bytes = sizeof(double) * (size_t)dim * dim, b_bytes = sizeof(double) * (size_t)dim * cb;
    VB_CUDA(cudaMalloc(&dev, g_bytes + 2 * b_bytes));
    double* d_G = (double*)dev;
    double* d_B = d_G + (size_t)dim * dim;
    double* d_M = d_B + (size_t)dim * cb;
    int rc = lp_gemm(reinterpret_cast<const float*>(rows.d), (int64_t)(step * rows.stride / 4), ns, dim, d_G, s);
    std::vector<double> b((size_t)dim * cb), m((size_t)dim * cb), gdiag((size_t)dim);
    std::mt19937_64 rng(42);
    std::normal_distribution<double> nd;
    for (double& v : b) v = nd(rng);
    lp_orthonormalise(b, dim, cb);
    for (int it = 0; it <= 8 && rc == VB_OK; ++it) {
        if (cudaMemcpyAsync(d_B, b.data(), b_bytes, cudaMemcpyHostToDevice, s) != cudaSuccess) rc = VB_ECUDA;
        if (rc == VB_OK) rc = lp_gemm(d_G, dim, d_B, cb, d_M, s);
        if (rc == VB_OK && cudaMemcpyAsync(m.data(), d_M, b_bytes, cudaMemcpyDeviceToHost, s) != cudaSuccess) rc = VB_ECUDA;
        if (rc == VB_OK && cudaStreamSynchronize(s) != cudaSuccess) rc = VB_ECUDA;
        if (rc == VB_OK && it < 8) {
            b = m;
            lp_orthonormalise(b, dim, cb);
        }
    }
    if (rc == VB_OK && cudaMemcpy2D(gdiag.data(), sizeof(double), d_G, sizeof(double) * (dim + 1), sizeof(double), dim, cudaMemcpyDeviceToHost) != cudaSuccess)
        rc = VB_ECUDA;
    cudaFree(dev);
    if (rc != VB_OK) {
        cudaGetLastError();
        return rc;
    }
    // the energy of the sample about the origin, and the part of it each column holds (b_j^T G b_j, m = G b)
    double total = 0.0;
    for (double v : gdiag) total += v;
    if (!(total > 0.0) || !std::isfinite(total)) return VB_OK;
    int r = 0;
    double held = 0.0;
    for (int j = 0; j < cb && r == 0; ++j) {
        for (int e = 0; e < dim; ++e) held += b[(size_t)e * cb + j] * m[(size_t)e * cb + j];
        if ((j + 1) % 16 == 0 && held >= 0.9 * total) r = j + 1;
    }
    if (r == 0) return VB_OK;
    std::vector<float> P((size_t)r * dim);
    for (int j = 0; j < r; ++j)
        for (int e = 0; e < dim; ++e) P[(size_t)j * dim + e] = (float)b[(size_t)e * cb + j];
    // sigma^2 >= ||P||_2^2 = lambda_max(P P^T): Gershgorin on P P^T in double, each entry widened by its rounding bound
    // (dim products exact in double, dim additions: <= dim 2^-53 |p_i| |p_j|, taken as dim 2^-52 max |p_i|^2)
    double pmax2 = 0.0, frob2 = 0.0;
    std::vector<double> pn((size_t)r, 0.0);
    for (int i = 0; i < r; ++i) {
        for (int e = 0; e < dim; ++e) pn[(size_t)i] += (double)P[(size_t)i * dim + e] * P[(size_t)i * dim + e];
        pmax2 = std::max(pmax2, pn[(size_t)i]);
        frob2 += pn[(size_t)i];
    }
    double sigma2 = 0.0;
    for (int i = 0; i < r; ++i) {
        double row = 0.0;
        for (int j = 0; j < r; ++j) {
            double d = 0.0;
            for (int e = 0; e < dim; ++e) d += (double)P[(size_t)i * dim + e] * P[(size_t)j * dim + e];
            row += std::fabs(d) + dim * std::ldexp(pmax2, -52);
        }
        sigma2 = std::max(sigma2, row);
    }
    sigma2 *= 1.0 + std::ldexp(1.0, -40);
    const double u = std::ldexp(1.0, -24);
    lp->r = r;
    lp->sigma2 = sigma2;
    lp->c1 = std::nextafter((float)(1.0 - (r + 4) * u), 0.f);
    lp->c2 = std::nextafter((float)((1.0 - (dim + 8) * u) / sigma2), 0.f);
    lp->ce = std::nextafter((float)(u * std::sqrt(sigma2) * (1.0 + u) + dim * std::ldexp(1.0, -52) * std::sqrt(frob2) * 1.01), FLT_MAX);
    lp->ce = std::nextafter(lp->ce, FLT_MAX);
    VB_CUDA(cudaMalloc(&lp->P, sizeof(float) * P.size()));
    VB_CUDA(cudaMemcpy(lp->P, P.data(), sizeof(float) * P.size(), cudaMemcpyHostToDevice));
    lp->cap_rows = std::max<int64_t>(rows.cap, rows.n);
    VB_CUDA(cudaMalloc(&lp->y, sizeof(float) * (size_t)lp->cap_rows * r));
    VB_TRY(list_proj_project(rows, *lp, 0, rows.n));
    VB_CUDA(cudaStreamSynchronize(s));
    return VB_OK;
}

void list_proj_release(ListProj* lp) {
    if (lp->P) cudaFree(lp->P);
    if (lp->y) cudaFree(lp->y);
    *lp = ListProj{};
}

int list_proj_update(const Table& rows, ListProj* lp, int64_t first_row) {
    if (!lp->y) return VB_OK;
    if (rows.n > lp->cap_rows) {
        cudaFree(lp->y);
        lp->y = nullptr;
        lp->cap_rows = std::max(rows.n, lp->cap_rows + lp->cap_rows / 2);
        if (cudaMalloc(&lp->y, sizeof(float) * (size_t)lp->cap_rows * lp->r) != cudaSuccess) {
            cudaGetLastError();
            list_proj_release(lp);   // the level is off until the image is loaded again
            lp->tried = true;
            return VB_OK;
        }
        first_row = 0;
    }
    return list_proj_project(rows, *lp, std::min(first_row, rows.n), rows.n);
}

int launch_list_proj(Scratch& sc, const Table& rows, const ListProj& lp, const ListTcImage& im, const void* qimg, size_t qstride, int64_t nq,
                     const int32_t* d_lists, int probes, const int32_t* cand_off, int64_t cap, const int64_t* d_list_off, int n_lists,
                     float* out, const float* qn, float* smin, int64_t cap_s) {
    VB_REQUIRE(lp.r > 0 && lp.r % 16 == 0 && lp.y != nullptr, "list scan level P without its projected plane");
    // (level P's k' is level 0's, and level 0 runs only where the refine takes the slab minima at that k': ivf_scan_topk)
    VB_REQUIRE(smin != nullptr, "list scan level P without slab minima");
    if (nq <= 0 || im.n_units <= 0) return VB_OK;
    cudaStream_t s = ctx().stream;
    void* d_yq;
    VB_TRY(sc.take(sizeof(float) * (size_t)nq * lp.r, &d_yq));
    const int64_t warps = nq * (lp.r / LP_PC);
    lp_project_kernel<<<(unsigned)((warps * 32 + 255) / 256), 256, 0, s>>>((const uint8_t*)qimg, qstride, nq, rows.dim, lp.P, lp.r,
                                                                         (float*)d_yq, nq);
    VB_CUDA(cudaGetLastError());
    count_launch();
    QueryGroups g{};
    VB_TRY(build_query_groups(sc, d_lists, nq, probes, cand_off, cap, n_lists, 0, &g, cap_s));
    const size_t smem = lp_scan_smem(lp.r);
    VB_REQUIRE(smem <= 227 * 1024, "level P: r = %d needs %zu bytes of shared memory", lp.r, smem);
    if (smem > 48 * 1024) VB_CUDA(cudaFuncSetAttribute(lp_scan_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    LpScanArgs a{};
    a.y = lp.y;
    a.yq = (const float*)d_yq;
    a.units = im.units;
    a.list_off = d_list_off;
    a.grp_begin = g.begin;
    a.grp_cnt = g.cnt;
    a.pair_q = g.pair_q;
    a.pair_out = g.pair_out;
    a.pair_sbase = g.pair_sbase;
    a.qn = qn;
    a.out = out;
    a.smin = smin;
    a.b = LpBound{lp.c1, lp.c2, lp.ce, __builtin_nextafterf(im.xmax * (1.0f + 1.0f / 1024.0f), FLT_MAX)};
    a.r = lp.r;
    lp_scan_kernel<<<(unsigned)im.n_units, LP_ROWS, smem, s>>>(a);
    VB_CUDA(cudaGetLastError());
    count_launch();
    return VB_OK;
}

}  // namespace vb
