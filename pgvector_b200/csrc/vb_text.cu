// vb_text.cu -- the type I/O of vector, halfvec and sparsevec over a column: vector_in / halfvec_in / sparsevec_in
// (src/vector.c:174-281, src/halfvec.c:178-286, src/sparsevec.c:203-409) and vector_out / halfvec_out / sparsevec_out
// (src/vector.c:289-326, src/halfvec.c:294-335, src/sparsevec.c:428-476), one warp per literal or row.
#include "vb_common.cuh"
#include "vb_text.cuh"
#include "vb_typio.cuh"

#include <cub/cub.cuh>

#include <cstring>
#include <string>
#include <vector>

namespace vb {
int offsets_from_counts(const int64_t* count, int64_t n, int64_t* row_off) {
    cudaStream_t s = ctx().stream;
    VB_CUDA(cudaMemsetAsync(row_off, 0, sizeof(int64_t), s));
    if (n == 0) return VB_OK;
    size_t tb = 0;
    VB_CUDA(cub::DeviceScan::InclusiveSum(nullptr, tb, count, row_off + 1, n, s));
    Scratch sc("type I/O");
    void* tmp = nullptr;
    VB_TRY(sc.own(tb, &tmp));
    VB_CUDA(cub::DeviceScan::InclusiveSum(tmp, tb, count, row_off + 1, n, s));
    count_launch();
    return VB_OK;
}

Staging& staging() {
    static Staging st;
    return st;
}

int pinned_grow(void** buf, size_t* have, size_t bytes) {
    if (*have >= bytes) return VB_OK;
    if (*buf) VB_CUDA(cudaFreeHost(*buf));
    *buf = nullptr;
    *have = 0;
    if (cudaMallocHost(buf, bytes) != cudaSuccess) {
        set_error("cudaMallocHost(%zu) for type I/O staging failed", bytes);
        return VB_ENOMEM;
    }
    *have = bytes;
    return VB_OK;
}

void set_error_detail(const char* detail);

namespace {
using namespace text;

constexpr int kMaxDim = 16000;          // VECTOR_MAX_DIM, HALFVEC_MAX_DIM, SPARSEVEC_MAX_NNZ
constexpr int kWarps = 8;               // warps per block
constexpr int kChunk = 16;              // bytes a lane classifies per step (a warp covers 512)
constexpr uint32_t kNone = 0xffffffffu;

// Outcome keys of one literal, ordered as the reference's left-to-right scan meets them: literal-level checks below
// 16, then element k's checks at ((k + 2) << 4) | stage (k = -1: sparsevec's "{}").  The least key is the outcome.
enum : uint32_t { L_MAXNNZ = 0, L_OPEN = 1, L_EMPTY = 2 };
enum : uint32_t {               // dense element stages
    D_MAXDIM = 0, D_NUL, D_NOCONV, D_RANGE, D_NAN, D_INF, D_SEP, D_CLOSE, D_JUNK };
enum : uint32_t {               // sparsevec element stages
    S_NUL = 0, S_IDX, S_COLON, S_NOCONV, S_RANGE, S_NAN, S_INF, S_SEP, S_CLOSE, S_SLASH, S_DIM, S_JUNK };
// after a CLOSE outcome (checked on the host side of the record): CheckDim, CheckExpectedDim, CheckIndex
enum : int32_t { X_NONE = 0, X_DIM_LOW, X_DIM_HIGH, X_TYPMOD, X_IDX_BOUNDS, X_IDX_DUP };

struct Status {                          // the one small result a call reads back
    unsigned long long first_bad;        // least failing literal, ~0 when none
    uint32_t key;                        // its outcome key
    int32_t post;                        // X_* after a CLOSE outcome
    int64_t dim;                         // its dimension (after CLOSE)
    int64_t tok_begin, tok_end;          // the token of a range error (literal-relative)
    int64_t lit_begin, lit_len;          // the literal (text-relative) up to its first NUL
    unsigned long long unsorted;         // sparsevec: some row's indices need the sort
};

__device__ __forceinline__ uint32_t lanemask_lt() {
    uint32_t m;
    asm("mov.u32 %0, %%lanemask_lt;" : "=r"(m));
    return m;
}

__device__ __forceinline__ Lit literal(const char* text, const int64_t* off, int64_t r) {
    const int64_t b = off[r], e = off[r + 1];
    return Lit{reinterpret_cast<const uint8_t*>(text) + b, e > b ? e - b : 0};
}

// A warp walks the literal from `open` in 512-byte windows; each lane classifies its 16 bytes, and element k starts
// after the k-th separator (`open` itself for k = 0: commas can only follow it in a literal that passed the opening
// check).  fn(k, start) runs on the lane holding the start and returns the element's key (kNone: it ended with ',').
// Stops after the first window that produced a key, since later elements cannot beat it.  Returns the least key;
// `mine` is the calling lane's least key of that window (the owner of the outcome has mine == result).
template <typename Fn>
__device__ uint32_t walk_elements(Lit L, int64_t open, uint32_t& mine, Fn fn) {
    const int lane = threadIdx.x & 31;
    uint32_t best = kNone;
    int64_t base_k = 0;
    for (int64_t w0 = open; w0 < L.len; w0 += 32 * kChunk) {
        const int64_t c0 = w0 + (int64_t)lane * kChunk;
        uint32_t sep = 0;
        int nul = kChunk;
        for (int i = 0; i < kChunk; ++i) {
            const int64_t pos = c0 + i;
            const uint32_t ch = pos < L.len ? (uint32_t)__ldg(L.s + pos) : 1u;
            if (ch == 0 && nul == kChunk) nul = i;
            if (ch == ',' || pos == open) sep |= 1u << i;
        }
        const uint32_t nul_lanes = __ballot_sync(~0u, nul < kChunk);
        const int first_nul_lane = nul_lanes ? __ffs(nul_lanes) - 1 : 32;
        if (lane > first_nul_lane) sep = 0;
        else if (lane == first_nul_lane) sep &= (1u << nul) - 1;
        const int cnt = __popc(sep);
        int incl = cnt;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const int t = __shfl_up_sync(~0u, incl, d);
            if (lane >= d) incl += t;
        }
        int64_t k = base_k + incl - cnt;
        uint32_t key = kNone;
        while (sep) {
            const int i = __ffs(sep) - 1;
            sep &= sep - 1;
            if (k <= kMaxDim && key == kNone) key = fn(k, c0 + i + 1);   // a lane's later elements lose to its first key
            ++k;
        }
        mine = key;
        best = __reduce_min_sync(~0u, key);
        base_k += __shfl_sync(~0u, incl, 31);
        if (best != kNone || nul_lanes) break;
    }
    return best;
}

__device__ __forceinline__ int64_t skip_space(Lit L, int64_t p) {
    while (is_space(L.at(p))) ++p;
    return p;
}

// what the lane that owns the outcome knows: the token of a range error, sparsevec's dimension
struct Detail {
    int64_t tok_begin = 0, tok_end = 0, dim = 0;
};
__device__ __forceinline__ Detail owner_detail(uint32_t mine, uint32_t best, const Detail& d) {
    const uint32_t who = __ballot_sync(~0u, mine == best);
    const int src = who ? __ffs(who) - 1 : 0;
    Detail o;
    o.tok_begin = __shfl_sync(~0u, d.tok_begin, src);
    o.tok_end = __shfl_sync(~0u, d.tok_end, src);
    o.dim = __shfl_sync(~0u, d.dim, src);
    return o;
}

// vector_in / halfvec_in of one literal by one warp: values to out[k] for k < cap
template <bool HALF>
__device__ uint32_t parse_dense(Lit L, void* out, int64_t cap, Detail* det) {
    int64_t p = skip_space(L, 0);
    if (L.at(p) != '[') return L_OPEN;
    const int64_t open = p;
    if (L.at(skip_space(L, p + 1)) == ']') return L_EMPTY;
    Detail d;
    uint32_t mine = kNone;
    const uint32_t best = walk_elements(L, open, mine, [&](int64_t k, int64_t q) -> uint32_t {
        const uint32_t kk = (uint32_t)(k + 2) << 4;
        if (k == kMaxDim) return kk | D_MAXDIM;
        q = skip_space(L, q);
        if (L.at(q) == 0) return kk | D_NUL;
        const FloatParse f = parse_float4(L, q);
        if (f.end == q) return kk | D_NOCONV;
        bool range, nan, inf;
        __half h;
        if (HALF) {
            bool ovf;
            h = float_to_half_checked(f.v, &ovf);
            range = (f.erange && isinf(f.v)) || ovf;
            nan = __hisnan(h);
            inf = __hisinf(h) != 0;
        } else {
            range = f.erange && isinf(f.v);
            nan = isnan(f.v);
            inf = isinf(f.v);
        }
        if (range) { d.tok_begin = q; d.tok_end = f.end; return kk | D_RANGE; }
        if (nan || inf) return kk | (nan ? D_NAN : D_INF);
        if (k < cap) {
            if (HALF) static_cast<__half*>(out)[k] = h;
            else static_cast<float*>(out)[k] = f.v;
        }
        q = skip_space(L, f.end);
        const uint32_t c = L.at(q);
        if (c == ',') return kNone;
        if (c == ']') return kk | (L.at(skip_space(L, q + 1)) == 0 ? D_CLOSE : D_JUNK);
        return kk | D_SEP;
    });
    if (det) *det = owner_detail(mine, best, d);
    return best;
}

// sparsevec's tail after '}': "/dim" and whitespace; kk is the closing element's key base
__device__ __forceinline__ uint32_t sparse_tail(Lit L, int64_t q, uint32_t kk, int64_t* dim) {
    q = skip_space(L, q);
    if (L.at(q) != '/') return kk | S_SLASH;
    q = skip_space(L, q + 1);
    const IntParse d = parse_long(L, q, INT32_MIN, INT32_MAX);
    if (d.end == q) return kk | S_DIM;
    if (L.at(skip_space(L, d.end)) != 0) return kk | S_JUNK;
    *dim = d.v;
    return kk | S_CLOSE;
}

// sparsevec_in of one literal by one warp: entry k (index - 1, value) to slot k, zeros included (the gather drops
// them); max_nnz is the literal's comma count + 1
__device__ uint32_t parse_sparse(Lit L, int64_t max_nnz, int32_t* idx, float* val, Detail* det) {
    if (max_nnz > kMaxDim) return L_MAXNNZ;
    int64_t p = skip_space(L, 0);
    if (L.at(p) != '{') return L_OPEN;
    const int64_t open = p;
    Detail d;
    p = skip_space(L, p + 1);
    if (L.at(p) == '}') {
        const uint32_t key = sparse_tail(L, p + 1, 1u << 4, &d.dim);
        if (det) *det = d;
        return key;
    }
    uint32_t mine = kNone;
    const uint32_t best = walk_elements(L, open, mine, [&](int64_t k, int64_t q) -> uint32_t {
        const uint32_t kk = (uint32_t)(k + 2) << 4;
        q = skip_space(L, q);
        if (L.at(q) == 0) return kk | S_NUL;
        const IntParse ix = parse_long(L, q, (int64_t)INT32_MIN + 1, INT32_MAX);
        if (ix.end == q) return kk | S_IDX;
        q = skip_space(L, ix.end);
        if (L.at(q) != ':') return kk | S_COLON;
        q = skip_space(L, q + 1);
        const FloatParse f = parse_float4(L, q);
        if (f.end == q) return kk | S_NOCONV;
        if (f.erange && (f.v == 0.f || isinf(f.v))) { d.tok_begin = q; d.tok_end = f.end; return kk | S_RANGE; }
        if (isnan(f.v)) return kk | S_NAN;
        if (isinf(f.v)) return kk | S_INF;
        idx[k] = (int32_t)(ix.v - 1);
        val[k] = f.v;
        q = skip_space(L, f.end);
        const uint32_t c = L.at(q);
        if (c == ',') return kNone;
        if (c == '}') return sparse_tail(L, q + 1, kk, &d.dim);
        return kk | S_SEP;
    });
    if (det) *det = owner_detail(mine, best, d);
    return best;
}

// the elements of a literal whose outcome is a CLOSE (k + 1; 0 for "{}")
__device__ __forceinline__ int64_t close_count(uint32_t key) { return (int64_t)(key >> 4) - 1; }

// ---------------------------------------------------------------------------------------------------- count pass
// commas + 1 before the first NUL of every literal: the dense bound and sparsevec_in's maxNnz
__global__ void __launch_bounds__(kWarps * 32) text_count_kernel(const char* text, const int64_t* off, int64_t n,
                                                                 int64_t* count) {
    const int lane = threadIdx.x & 31;
    for (int64_t r = (int64_t)blockIdx.x * kWarps + (threadIdx.x >> 5); r < n; r += (int64_t)gridDim.x * kWarps) {
        const Lit L = literal(text, off, r);
        int64_t c = 0;
        for (int64_t w0 = 0; w0 < L.len; w0 += 32 * kChunk) {
            int nul = kChunk, cm = 0;
            uint32_t commas = 0;
            for (int i = 0; i < kChunk; ++i) {
                const int64_t pos = w0 + (int64_t)lane * kChunk + i;
                const uint32_t ch = pos < L.len ? (uint32_t)__ldg(L.s + pos) : 1u;
                if (ch == 0 && nul == kChunk) nul = i;
                if (ch == ',') commas |= 1u << i;
            }
            const uint32_t nul_lanes = __ballot_sync(~0u, nul < kChunk);
            const int first = nul_lanes ? __ffs(nul_lanes) - 1 : 32;
            if (lane < first) cm = __popc(commas);
            else if (lane == first) cm = __popc(commas & ((1u << nul) - 1));
            c += __reduce_add_sync(~0u, (unsigned)cm);
            if (nul_lanes) break;
        }
        if (lane == 0) count[r] = c + 1;
    }
}

__global__ void typmod_offsets_kernel(int64_t n, int64_t typmod, int64_t* row_off) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i <= n; i += (int64_t)gridDim.x * blockDim.x)
        row_off[i] = i * typmod;
}

// ---------------------------------------------------------------------------------------------------- parse
template <bool HALF>
__global__ void __launch_bounds__(kWarps * 32) text_parse_dense_kernel(const char* text, const int64_t* off, int64_t n,
                                                                       int32_t typmod, const int64_t* row_off,
                                                                       void* out, Status* st) {
    for (int64_t r = (int64_t)blockIdx.x * kWarps + (threadIdx.x >> 5); r < n; r += (int64_t)gridDim.x * kWarps) {
        const int64_t b = row_off[r];
        void* row = HALF ? (void*)(static_cast<__half*>(out) + b) : (void*)(static_cast<float*>(out) + b);
        const uint32_t key = parse_dense<HALF>(literal(text, off, r), row, row_off[r + 1] - b, nullptr);
        const bool ok = key >= 32 && (key & 15) == D_CLOSE && (typmod == -1 || typmod == close_count(key));
        if (!ok && (threadIdx.x & 31) == 0) atomicMin(&st->first_bad, (unsigned long long)r);
    }
}

// sparsevec: entries to slots (at the bound offsets), the stored count and the dimension of every literal
__global__ void __launch_bounds__(kWarps * 32) text_parse_sparse_kernel(const char* text, const int64_t* off, int64_t n,
                                                                        int32_t typmod, const int64_t* slot_off,
                                                                        int32_t* slot_idx, float* slot_val,
                                                                        int64_t* nnz, int32_t* out_dim, Status* st) {
    const int lane = threadIdx.x & 31;
    for (int64_t r = (int64_t)blockIdx.x * kWarps + (threadIdx.x >> 5); r < n; r += (int64_t)gridDim.x * kWarps) {
        const int64_t b = slot_off[r];
        Detail d;
        const uint32_t key = parse_sparse(literal(text, off, r), slot_off[r + 1] - b, slot_idx + b, slot_val + b, &d);
        const bool ok = key >= 16 && (key & 15) == S_CLOSE && d.dim >= 1 && d.dim <= 1000000000 &&
                        (typmod == -1 || typmod == d.dim);
        unsigned cnt = 0;
        if (ok)
            for (int64_t k = lane; k < close_count(key); k += 32) cnt += slot_val[b + k] != 0.f;
        cnt = __reduce_add_sync(~0u, cnt);
        if (lane == 0) {
            nnz[r] = ok ? cnt : 0;
            out_dim[r] = (int32_t)d.dim;
            if (!ok) atomicMin(&st->first_bad, (unsigned long long)r);
        }
    }
}

// the stored entries of every good literal from its slots to its row of the CSR, zeros dropped, order kept
__global__ void __launch_bounds__(kWarps * 32) sparse_gather_kernel(int64_t n, const int64_t* slot_off,
                                                                    const int32_t* slot_idx, const float* slot_val,
                                                                    const int64_t* row_off, int32_t* idx, float* val) {
    const int lane = threadIdx.x & 31;
    for (int64_t r = (int64_t)blockIdx.x * kWarps + (threadIdx.x >> 5); r < n; r += (int64_t)gridDim.x * kWarps) {
        const int64_t want = row_off[r + 1] - row_off[r];
        if (want == 0) continue;
        const int64_t b = slot_off[r], e = slot_off[r + 1];
        int64_t o = row_off[r];
        for (int64_t k0 = b; k0 < e; k0 += 32) {
            const int64_t k = k0 + lane;
            const bool keep = k < e && slot_val[k] != 0.f;
            const uint32_t m = __ballot_sync(~0u, keep);
            if (keep) {
                const int64_t at = o + __popc(m & lanemask_lt());
                idx[at] = slot_idx[k];
                val[at] = slot_val[k];
            }
            o += __popc(m);
        }
    }
}

// CheckIndex after the sort (src/sparsevec.c:107-131, 396-406) on rows in ascending order; a row not yet in order
// sets st->unsorted and is checked after the sort (final = true checks every row)
__global__ void __launch_bounds__(kWarps * 32) sparse_check_kernel(int64_t n, const int64_t* row_off, const int32_t* idx,
                                                                   const int32_t* dim, bool final, Status* st) {
    const int lane = threadIdx.x & 31;
    for (int64_t r = (int64_t)blockIdx.x * kWarps + (threadIdx.x >> 5); r < n; r += (int64_t)gridDim.x * kWarps) {
        const int64_t b = row_off[r], e = row_off[r + 1];
        bool down = false, bad = false;
        for (int64_t i = b + lane; i < e; i += 32) {
            const int32_t x = idx[i];
            if (i > b && x < idx[i - 1]) down = true;
            if (x < 0 || x >= dim[r] || (i > b && x == idx[i - 1])) bad = true;
        }
        down = __any_sync(~0u, down);
        bad = __any_sync(~0u, bad);
        if (lane == 0) {
            if (down && !final) st->unsorted = 1;
            else if (bad) atomicMin(&st->first_bad, (unsigned long long)r);
        }
    }
}

// one warp re-reads the least failing literal and records why it failed
template <int KIND>   // 0 vector, 1 halfvec, 2 sparsevec
__global__ void text_record_kernel(const char* text, const int64_t* off, int32_t typmod, const int64_t* slot_off,
                                   int32_t* slot_idx, float* slot_val, const int64_t* row_off, const int32_t* idx,
                                   Status* st) {
    const unsigned long long r = st->first_bad;
    if (r == ~0ull) return;
    const Lit L = literal(text, off, (int64_t)r);
    Detail d;
    uint32_t key;
    if (KIND == 2) {
        key = parse_sparse(L, slot_off[r + 1] - slot_off[r], slot_idx + slot_off[r], slot_val + slot_off[r], &d);
    } else {
        // the values are not needed again: cap 0 writes none
        key = parse_dense<KIND == 1>(L, nullptr, 0, &d);
        d.dim = close_count(key);
    }
    if (threadIdx.x != 0) return;
    int64_t len = 0;
    while (len < L.len && L.s[len] != 0) ++len;
    st->key = key;
    st->dim = d.dim;
    st->tok_begin = d.tok_begin;
    st->tok_end = d.tok_end;
    st->lit_begin = off[r];
    st->lit_len = len;
    int32_t post = X_NONE;
    const bool closed = KIND == 2 ? (key >= 16 && (key & 15) == S_CLOSE) : (key >= 32 && (key & 15) == D_CLOSE);
    if (closed) {
        if (KIND == 2 && d.dim < 1) post = X_DIM_LOW;
        else if (KIND == 2 && d.dim > 1000000000) post = X_DIM_HIGH;
        else if (typmod != -1 && typmod != d.dim) post = X_TYPMOD;
        else if (KIND == 2) {
            // CheckIndex in ascending order: the first entry out of bounds or equal to its predecessor
            for (int64_t i = row_off[r]; i < row_off[r + 1]; ++i) {
                const int32_t x = idx[i];
                if (x < 0 || x >= d.dim) { post = X_IDX_BOUNDS; break; }
                if (i > row_off[r] && x == idx[i - 1]) { post = X_IDX_DUP; break; }
            }
        }
    }
    st->post = post;
}

// ---------------------------------------------------------------------------------------------------- format
__device__ __forceinline__ float row_value(int elem, const void* rows, int64_t i) {
    return elem == VB_VECTOR ? static_cast<const float*>(rows)[i] : __half2float(static_cast<const __half*>(rows)[i]);
}

__device__ __forceinline__ int uint_len(uint64_t v) {
    int k = 1;
    while (v >= 10) { v /= 10; ++k; }
    return k;
}

// Two passes over the same warp loop: WRITE = false sums the text length of each row, WRITE = true places every
// element's text after a warp scan of the lengths.  dense: [x,x,...]; sparse: {i:x,...}/dim
template <bool WRITE, bool SPARSE>
__global__ void __launch_bounds__(kWarps * 32) text_format_kernel(int elem, int dim, const void* rows, int64_t n,
                                                                  const int64_t* row_off, const int32_t* sidx,
                                                                  int64_t* len_or_off, char* out) {
    const int lane = threadIdx.x & 31;
    for (int64_t r = (int64_t)blockIdx.x * kWarps + (threadIdx.x >> 5); r < n; r += (int64_t)gridDim.x * kWarps) {
        const int64_t b = SPARSE ? row_off[r] : r * (int64_t)dim;
        const int64_t cnt = SPARSE ? row_off[r + 1] - b : dim;
        int64_t pos = WRITE ? len_or_off[r] : 0;
        if (WRITE && lane == 0) out[pos] = SPARSE ? '{' : '[';
        ++pos;
        for (int64_t e0 = 0; e0 < cnt; e0 += 32) {
            const int64_t e = e0 + lane;
            char buf[28];
            int l = 0;
            if (e < cnt) {
                if (e > 0) buf[l++] = ',';
                if (SPARSE) {
                    l += put_uint(buf + l, (uint64_t)(int64_t)sidx[b + e] + 1);
                    buf[l++] = ':';
                }
                l += format_float4(row_value(elem, rows, b + e), buf + l);
            }
            int incl = l;
#pragma unroll
            for (int d = 1; d < 32; d <<= 1) {
                const int t = __shfl_up_sync(~0u, incl, d);
                if (lane >= d) incl += t;
            }
            if (WRITE)
                for (int i = 0; i < l; ++i) out[pos + incl - l + i] = buf[i];
            pos += __shfl_sync(~0u, incl, 31);
        }
        if (lane == 0) {
            if (SPARSE) {
                if (WRITE) {
                    out[pos] = '}';
                    out[pos + 1] = '/';
                    put_uint(out + pos + 2, (uint64_t)dim);
                }
                pos += 2 + uint_len((uint64_t)dim);
            } else {
                if (WRITE) out[pos] = ']';
                ++pos;
            }
            if (!WRITE) len_or_off[r] = pos;
        }
    }
}

// ---------------------------------------------------------------------------------------------------- host side
int grid_for(int64_t n) {
    const int64_t want = (n + kWarps - 1) / kWarps;
    const int64_t cap = (int64_t)ctx().sm_count * 16;
    return (int)std::max<int64_t>(1, std::min(want, cap));
}

const char* type_name(int kind) { return kind == 0 ? "vector" : kind == 1 ? "halfvec" : "sparsevec"; }

// the reference's error for a recorded failure; lit is the literal up to its first NUL
int text_error(int kind, int32_t typmod, const Status& st, const std::string& lit) {
    const char* t = type_name(kind);
    const uint32_t key = st.key;
    const uint32_t stage = key & 15;
    auto syntax = [&](const char* detail) {
        set_error("invalid input syntax for type %s: \"%s\"", t, lit.c_str());
        if (detail) set_error_detail(detail);
        return VB_EINVAL;
    };
    auto range = [&]() {
        set_error("\"%s\" is out of range for type %s",
                  lit.substr((size_t)st.tok_begin, (size_t)(st.tok_end - st.tok_begin)).c_str(), t);
        return VB_EINVAL;
    };
    if (key < 16) {
        if (key == L_MAXNNZ) { set_error("sparsevec cannot have more than %d non-zero elements", kMaxDim); return VB_EINVAL; }
        if (key == L_OPEN) return syntax(kind == 2 ? "Vector contents must start with \"{\"." : "Vector contents must start with \"[\".");
        set_error("%s must have at least 1 dimension", t);
        return VB_EINVAL;
    }
    if (kind != 2) {
        switch (stage) {
            case D_MAXDIM: set_error("%s cannot have more than %d dimensions", t, kMaxDim); return VB_EINVAL;
            case D_RANGE: return range();
            case D_NAN: set_error("NaN not allowed in %s", t); return VB_EINVAL;
            case D_INF: set_error("infinite value not allowed in %s", t); return VB_EINVAL;
            case D_JUNK: return syntax("Junk after closing right brace.");
            case D_CLOSE: break;
            default: return syntax(nullptr);
        }
    } else {
        switch (stage) {
            case S_RANGE: return range();
            case S_NAN: set_error("NaN not allowed in %s", t); return VB_EINVAL;
            case S_INF: set_error("infinite value not allowed in %s", t); return VB_EINVAL;
            case S_SLASH: return syntax("Unexpected end of input.");
            case S_JUNK: return syntax("Junk after closing.");
            case S_CLOSE: break;
            default: return syntax(nullptr);
        }
    }
    switch (st.post) {
        case X_DIM_LOW: set_error("%s must have at least 1 dimension", t); return VB_EINVAL;
        case X_DIM_HIGH: set_error("sparsevec cannot have more than %d dimensions", 1000000000); return VB_EINVAL;
        case X_TYPMOD: set_error("expected %d dimensions, not %lld", typmod, (long long)st.dim); return VB_EINVAL;
        case X_IDX_BOUNDS: set_error("sparsevec index out of bounds"); return VB_EINVAL;
        case X_IDX_DUP: set_error("sparsevec indices must not contain duplicates"); return VB_EINVAL;
        default: set_error("%s input: failure without a recorded cause", t); return VB_ECUDA;
    }
}

// reads the status back; on a failure, the literal too, and raises its error
int finish(int kind, int32_t typmod, const char* text_dev, Status* st_dev, int64_t* out_bad, int64_t bad_base) {
    Status st;
    VB_CUDA(cudaMemcpyAsync(&st, st_dev, sizeof(Status), cudaMemcpyDeviceToHost, ctx().stream));
    VB_CUDA(cudaStreamSynchronize(ctx().stream));
    if (st.first_bad == ~0ull) return VB_OK;
    std::string lit((size_t)st.lit_len, '\0');
    if (st.lit_len)
        VB_CUDA(cudaMemcpy(&lit[0], text_dev + st.lit_begin, (size_t)st.lit_len, cudaMemcpyDeviceToHost));
    if (out_bad) *out_bad = bad_base + (int64_t)st.first_bad;
    return text_error(kind, typmod, st, lit);
}

Status fresh_status() {
    Status s;
    std::memset(&s, 0, sizeof(s));
    s.first_bad = ~0ull;
    return s;
}

// a fresh Status on the device: first_bad = ~0, the rest 0 (no host memory involved)
int status_reset(Status* st) {
    VB_CUDA(cudaMemsetAsync(st, 0, sizeof(Status), ctx().stream));
    VB_CUDA(cudaMemsetAsync(&st->first_bad, 0xff, sizeof(st->first_bad), ctx().stream));
    return VB_OK;
}

// enqueue the dense parse of n literals into rows at row_off (already written) and the record of the first failure
int dense_parse_enqueue(int elem, int32_t typmod, int64_t n, const char* text, const int64_t* off, const int64_t* row_off,
                        void* out, Status* sp) {
    cudaStream_t s = ctx().stream;
    VB_TRY(status_reset(sp));
    {
        ProfScope prof(VB_PROF_TEXT_PARSE);
        if (elem == VB_VECTOR)
            text_parse_dense_kernel<false><<<grid_for(n), kWarps * 32, 0, s>>>(text, off, n, typmod, row_off, out, sp);
        else
            text_parse_dense_kernel<true><<<grid_for(n), kWarps * 32, 0, s>>>(text, off, n, typmod, row_off, out, sp);
        VB_CUDA(cudaGetLastError());
    }
    if (elem == VB_VECTOR)
        text_record_kernel<0><<<1, 32, 0, s>>>(text, off, typmod, nullptr, nullptr, nullptr, nullptr, nullptr, sp);
    else
        text_record_kernel<1><<<1, 32, 0, s>>>(text, off, typmod, nullptr, nullptr, nullptr, nullptr, nullptr, sp);
    VB_CUDA(cudaGetLastError());
    count_launch(2);
    return VB_OK;
}

int dense_parse_dev(int elem, int32_t typmod, int64_t n, const char* text, const int64_t* off, const int64_t* row_off,
                    void* out, int64_t* out_bad, int64_t bad_base) {
    Scratch sc("type I/O");
    void* st = nullptr;
    VB_TRY(sc.own(sizeof(Status), &st));
    Status* sp = static_cast<Status*>(st);
    VB_TRY(dense_parse_enqueue(elem, typmod, n, text, off, row_off, out, sp));
    return finish(elem == VB_VECTOR ? 0 : 1, typmod, text, sp, out_bad, bad_base);
}

int check_text_args(const char* fn, int64_t n, const void* text, const int64_t* off, int64_t cap) {
    VB_REQUIRE(n >= 0 && n < (int64_t)INT32_MAX, "%s: bad literal count %lld", fn, (long long)n);
    VB_REQUIRE(cap >= 0, "%s: bad cap %lld", fn, (long long)cap);
    VB_REQUIRE(n == 0 || (text && off), "%s: text and off are required", fn);
    return VB_OK;
}

// host bound of one literal: commas + 1 before its first NUL
int64_t host_count(const char* t, int64_t len) {
    const char* end = t + strnlen(t, (size_t)len);
    int64_t c = 1;
    for (const char* p = t; (p = static_cast<const char*>(std::memchr(p, ',', (size_t)(end - p)))) != nullptr; ++p) ++c;
    return c;
}


// sparsevec parse of n literals on the device: bound offsets, cap check, parse to slots, CSR, sort when needed, checks
int sparse_parse_dev(int32_t typmod, int64_t n, const char* text, const int64_t* off, int64_t cap, int32_t* out_dim,
                     int64_t* out_row_off, int32_t* out_idx, float* out_val, int64_t* out_bad, int64_t bad_base,
                     int64_t* total_out) {
    cudaStream_t s = ctx().stream;
    Scratch sc("type I/O");
    void *cnt = nullptr, *slot_off = nullptr, *st = nullptr;
    VB_TRY(sc.own(sizeof(int64_t) * (size_t)n, &cnt));
    VB_TRY(sc.own(sizeof(int64_t) * (size_t)(n + 1), &slot_off));
    VB_TRY(sc.own(sizeof(Status), &st));
    int64_t* cp = static_cast<int64_t*>(cnt);
    int64_t* so = static_cast<int64_t*>(slot_off);
    Status* sp = static_cast<Status*>(st);
    if (n) text_count_kernel<<<grid_for(n), kWarps * 32, 0, s>>>(text, off, n, cp);
    VB_CUDA(cudaGetLastError());
    VB_TRY(offsets_from_counts(cp, n, so));
    int64_t bound = 0;
    VB_CUDA(cudaMemcpyAsync(&bound, so + n, sizeof(int64_t), cudaMemcpyDeviceToHost, s));
    VB_CUDA(cudaStreamSynchronize(s));
    if (total_out) *total_out = bound;
    if (bound > cap) {
        VB_CUDA(cudaMemcpyAsync(out_row_off, so, sizeof(int64_t) * (size_t)(n + 1), cudaMemcpyDeviceToDevice, s));
        VB_CUDA(cudaStreamSynchronize(s));
        set_error("sparsevec_in: the literals need up to %lld entries, more than cap = %lld", (long long)bound, (long long)cap);
        return VB_EINVAL;
    }
    if (n == 0) {
        VB_CUDA(cudaMemsetAsync(out_row_off, 0, sizeof(int64_t), s));
        return VB_OK;
    }
    // the segmented sort counts entries in int
    VB_REQUIRE(bound <= INT32_MAX, "sparsevec_in: the literals need up to %lld entries, more than %d in one call",
               (long long)bound, INT32_MAX);
    void *sidx = nullptr, *sval = nullptr;
    VB_TRY(sc.own(sizeof(int32_t) * (size_t)bound, &sidx));
    VB_TRY(sc.own(sizeof(float) * (size_t)bound, &sval));
    int32_t* si = static_cast<int32_t*>(sidx);
    float* sv = static_cast<float*>(sval);
    const Status init = fresh_status();
    VB_CUDA(cudaMemcpyAsync(sp, &init, sizeof(Status), cudaMemcpyHostToDevice, s));
    {
        ProfScope prof(VB_PROF_TEXT_PARSE);
        text_parse_sparse_kernel<<<grid_for(n), kWarps * 32, 0, s>>>(text, off, n, typmod, so, si, sv, cp, out_dim, sp);
        VB_CUDA(cudaGetLastError());
    }
    VB_TRY(offsets_from_counts(cp, n, out_row_off));
    sparse_gather_kernel<<<grid_for(n), kWarps * 32, 0, s>>>(n, so, si, sv, out_row_off, out_idx, out_val);
    sparse_check_kernel<<<grid_for(n), kWarps * 32, 0, s>>>(n, out_row_off, out_idx, out_dim, false, sp);
    VB_CUDA(cudaGetLastError());
    count_launch(3);
    unsigned long long unsorted = 0;
    int64_t nnz = 0;
    VB_CUDA(cudaMemcpyAsync(&unsorted, &sp->unsorted, sizeof(unsorted), cudaMemcpyDeviceToHost, s));
    VB_CUDA(cudaMemcpyAsync(&nnz, out_row_off + n, sizeof(nnz), cudaMemcpyDeviceToHost, s));
    VB_CUDA(cudaStreamSynchronize(s));
    if (unsorted) {
        // qsort by index (src/sparsevec.c:396): a stable segmented sort of the rows, through the slot buffers
        VB_CUDA(cudaMemcpyAsync(si, out_idx, sizeof(int32_t) * (size_t)nnz, cudaMemcpyDeviceToDevice, s));
        VB_CUDA(cudaMemcpyAsync(sv, out_val, sizeof(float) * (size_t)nnz, cudaMemcpyDeviceToDevice, s));
        size_t tb = 0;
        VB_CUDA(cub::DeviceSegmentedSort::StableSortPairs(nullptr, tb, si, out_idx, sv, out_val, (int)nnz, (int)n,
                                                          out_row_off, out_row_off + 1, s));
        Scratch sc("type I/O");
        void* tmp = nullptr;
        VB_TRY(sc.own(tb, &tmp));
        VB_CUDA(cub::DeviceSegmentedSort::StableSortPairs(tmp, tb, si, out_idx, sv, out_val, (int)nnz, (int)n,
                                                          out_row_off, out_row_off + 1, s));
        sparse_check_kernel<<<grid_for(n), kWarps * 32, 0, s>>>(n, out_row_off, out_idx, out_dim, true, sp);
        VB_CUDA(cudaGetLastError());
        count_launch(2);
    }
    text_record_kernel<2><<<1, 32, 0, s>>>(text, off, typmod, so, si, sv, out_row_off, out_idx, sp);
    VB_CUDA(cudaGetLastError());
    count_launch();
    return finish(2, typmod, text, sp, out_bad, bad_base);
}

// the write pass alone, at offsets already in out_off (device)
int format_write(bool sparse, int elem, int dim, const void* rows, int64_t n, const int64_t* row_off, const int32_t* idx,
                 const int64_t* out_off, char* out) {
    cudaStream_t s = ctx().stream;
    ProfScope prof(VB_PROF_TEXT_FORMAT);
    if (sparse)
        text_format_kernel<true, true><<<grid_for(n), kWarps * 32, 0, s>>>(elem, dim, rows, n, row_off, idx,
                                                                          const_cast<int64_t*>(out_off), out);
    else
        text_format_kernel<true, false><<<grid_for(n), kWarps * 32, 0, s>>>(elem, dim, rows, n, row_off, idx,
                                                                           const_cast<int64_t*>(out_off), out);
    VB_CUDA(cudaGetLastError());
    count_launch();
    return VB_OK;
}

// text of n dense rows (row_off == nullptr) or sparsevec rows: sparsevec rows checked as the sparse table calls check
// them (offsets from 0, indices ascending in [0, dim)), lengths, offsets, cap check, write
int format_dev(bool sparse, int elem, int dim, const void* rows, int64_t n, const int64_t* row_off, const int32_t* idx,
               int64_t cap, int64_t* out_off, char* out, int64_t* total_out) {
    cudaStream_t s = ctx().stream;
    if (sparse && n) VB_TRY(sparse_csr_check_dev("sparsevec_out", dim, n, row_off, idx));
    Scratch sc("type I/O");
    void* len = nullptr;
    VB_TRY(sc.own(sizeof(int64_t) * (size_t)n, &len));
    int64_t* lp = static_cast<int64_t*>(len);
    {
        ProfScope prof(VB_PROF_TEXT_FORMAT);
        if (n) {
            if (sparse)
                text_format_kernel<false, true><<<grid_for(n), kWarps * 32, 0, s>>>(elem, dim, rows, n, row_off, idx, lp, nullptr);
            else
                text_format_kernel<false, false><<<grid_for(n), kWarps * 32, 0, s>>>(elem, dim, rows, n, row_off, idx, lp, nullptr);
        }
        VB_CUDA(cudaGetLastError());
        count_launch();
    }
    VB_TRY(offsets_from_counts(lp, n, out_off));
    int64_t total = 0;
    VB_CUDA(cudaMemcpyAsync(&total, out_off + n, sizeof(int64_t), cudaMemcpyDeviceToHost, s));
    VB_CUDA(cudaStreamSynchronize(s));
    if (total_out) *total_out = total;
    if (n == 0 || !out) return VB_OK;   // no output: a sizing call
    VB_REQUIRE(total <= cap, "%s: the text is %lld bytes, more than cap = %lld", sparse ? "sparsevec_out" : "vector_out",
               (long long)total, (long long)cap);
    VB_TRY(format_write(sparse, elem, dim, rows, n, row_off, idx, out_off, out));
    VB_CUDA(cudaStreamSynchronize(s));   // the text is complete when the call returns, as for the input calls
    return VB_OK;
}

constexpr int64_t kStageBytes = 64ll << 20;     // text bytes per chunk of the host variants

}  // namespace
}  // namespace vb

using namespace vb;

extern "C" {

int vb_text_to_rows_batch_dev(int elem, int32_t typmod, int64_t n, const char* text, const int64_t* off, int64_t cap,
                              int64_t* out_row_off, void* out, int64_t* out_bad) {
    if (out_bad) *out_bad = -1;
    VB_TRY(require_init());
    VB_TRY(check_text_args("vb_text_to_rows_batch_dev", n, text, off, cap));
    VB_REQUIRE(elem == VB_VECTOR || elem == VB_HALFVEC, "vb_text_to_rows_batch_dev: elem must be VB_VECTOR or VB_HALFVEC");
    VB_REQUIRE(typmod == -1 || (typmod >= 1 && typmod <= kMaxDim), "vb_text_to_rows_batch_dev: bad typmod %d", typmod);
    VB_REQUIRE(out_row_off, "vb_text_to_rows_batch_dev: out_row_off is required");
    cudaStream_t s = ctx().stream;
    if (typmod >= 1) {
        typmod_offsets_kernel<<<grid_for(n + 1), 256, 0, s>>>(n, typmod, out_row_off);
    } else {
        Scratch sc("type I/O");
        void* cnt = nullptr;
        VB_TRY(sc.own(sizeof(int64_t) * (size_t)n, &cnt));
        if (n) text_count_kernel<<<grid_for(n), kWarps * 32, 0, s>>>(text, off, n, static_cast<int64_t*>(cnt));
        VB_CUDA(cudaGetLastError());
        VB_TRY(offsets_from_counts(static_cast<int64_t*>(cnt), n, out_row_off));
    }
    VB_CUDA(cudaGetLastError());
    count_launch();
    int64_t total = 0;
    VB_CUDA(cudaMemcpyAsync(&total, out_row_off + n, sizeof(int64_t), cudaMemcpyDeviceToHost, s));
    VB_CUDA(cudaStreamSynchronize(s));
    VB_REQUIRE(total <= cap, "vb_text_to_rows_batch_dev: the literals need %lld elements, more than cap = %lld",
               (long long)total, (long long)cap);
    if (n == 0) return VB_OK;
    VB_REQUIRE(out, "vb_text_to_rows_batch_dev: out is required");
    return dense_parse_dev(elem, typmod, n, text, off, out_row_off, out, out_bad, 0);
}

int vb_text_to_rows_batch(int elem, int32_t typmod, int64_t n, const char* text, const int64_t* off, int64_t cap,
                          int64_t* out_row_off, void* out, int64_t* out_bad) {
    if (out_bad) *out_bad = -1;
    VB_TRY(require_init());
    VB_TRY(check_text_args("vb_text_to_rows_batch", n, text, off, cap));
    VB_REQUIRE(elem == VB_VECTOR || elem == VB_HALFVEC, "vb_text_to_rows_batch: elem must be VB_VECTOR or VB_HALFVEC");
    VB_REQUIRE(typmod == -1 || (typmod >= 1 && typmod <= kMaxDim), "vb_text_to_rows_batch: bad typmod %d", typmod);
    VB_REQUIRE(out_row_off, "vb_text_to_rows_batch: out_row_off is required");
    out_row_off[0] = 0;
    for (int64_t r = 0; r < n; ++r)
        out_row_off[r + 1] = out_row_off[r] + (typmod >= 1 ? typmod : host_count(text + off[r], off[r + 1] - off[r]));
    VB_REQUIRE(out_row_off[n] <= cap, "vb_text_to_rows_batch: the literals need %lld elements, more than cap = %lld",
               (long long)out_row_off[n], (long long)cap);
    if (n == 0) return VB_OK;
    VB_REQUIRE(out, "vb_text_to_rows_batch: out is required");
    const size_t esz = elem == VB_VECTOR ? 4 : 2;
    cudaStream_t s = ctx().stream;
    // chunks of literals of at most kStageBytes of text (or one longer literal), in order
    std::vector<int64_t> cuts{0};
    while (cuts.back() < n) {
        const int64_t r0 = cuts.back();
        int64_t r1 = r0 + 1;
        while (r1 < n && off[r1 + 1] - off[r0] <= kStageBytes) ++r1;
        cuts.push_back(r1);
    }
    const int64_t nch = (int64_t)cuts.size() - 1;
    int64_t max_tb = 1, max_nr = 1, max_ne = 1;
    for (int64_t c = 0; c < nch; ++c) {
        max_tb = std::max(max_tb, off[cuts[c + 1]] - off[cuts[c]]);
        max_nr = std::max(max_nr, cuts[c + 1] - cuts[c]);
        max_ne = std::max(max_ne, out_row_off[cuts[c + 1]] - out_row_off[cuts[c]]);
    }
    // two slots: while the device parses chunk c, the host finishes chunk c - 1 and stages chunk c + 1
    Staging& sg = staging();
    const size_t tb_al = ((size_t)max_tb + 15) & ~(size_t)15;
    const size_t in_bytes = tb_al + sizeof(int64_t) * 2 * (size_t)(max_nr + 1);
    const size_t out_bytes = sizeof(Status) + esz * (size_t)max_ne;
    Scratch sc("type I/O");
    void *dtext[2] = {}, *doff[2] = {}, *dout[2] = {}, *dst[2] = {};
    for (int k = 0; k < 2 && k < nch; ++k) {
        VB_TRY(pinned_grow(&sg.in[k], &sg.in_bytes[k], in_bytes));
        VB_TRY(pinned_grow(&sg.out[k], &sg.out_bytes[k], out_bytes));
        VB_TRY(sc.own((size_t)max_tb, &dtext[k]));
        VB_TRY(sc.own(sizeof(int64_t) * 2 * (size_t)(max_nr + 1), &doff[k]));
        VB_TRY(sc.own(esz * (size_t)max_ne, &dout[k]));
        VB_TRY(sc.own(sizeof(Status), &dst[k]));
    }
    auto enqueue = [&](int64_t c, int k) -> int {
        const int64_t r0 = cuts[c], r1 = cuts[c + 1];
        const int64_t tb = off[r1] - off[r0], nr = r1 - r0, ne = out_row_off[r1] - out_row_off[r0];
        char* ptext = static_cast<char*>(sg.in[k]);
        int64_t* poff = reinterpret_cast<int64_t*>(ptext + tb_al);
        std::memcpy(ptext, text + off[r0], (size_t)tb);
        for (int64_t i = 0; i <= nr; ++i) {
            poff[i] = off[r0 + i] - off[r0];
            poff[nr + 1 + i] = out_row_off[r0 + i] - out_row_off[r0];
        }
        VB_CUDA(cudaMemcpyAsync(dtext[k], ptext, (size_t)tb, cudaMemcpyHostToDevice, s));
        VB_CUDA(cudaMemcpyAsync(doff[k], poff, sizeof(int64_t) * 2 * (size_t)(nr + 1), cudaMemcpyHostToDevice, s));
        const int64_t* doffp = static_cast<int64_t*>(doff[k]);
        Status* sp = static_cast<Status*>(dst[k]);
        VB_TRY(dense_parse_enqueue(elem, typmod, nr, static_cast<char*>(dtext[k]), doffp, doffp + nr + 1, dout[k], sp));
        VB_CUDA(cudaMemcpyAsync(sg.out[k], sp, sizeof(Status), cudaMemcpyDeviceToHost, s));
        VB_CUDA(cudaMemcpyAsync(static_cast<char*>(sg.out[k]) + sizeof(Status), dout[k], esz * (size_t)ne,
                                cudaMemcpyDeviceToHost, s));
        return VB_OK;
    };
    auto finish_chunk = [&](int64_t c, int k) -> int {
        const int64_t r0 = cuts[c], r1 = cuts[c + 1];
        const Status& st = *static_cast<const Status*>(sg.out[k]);
        if (st.first_bad != ~0ull) {
            if (out_bad) *out_bad = r0 + (int64_t)st.first_bad;
            return text_error(elem == VB_VECTOR ? 0 : 1, typmod, st,
                              std::string(text + off[r0] + st.lit_begin, (size_t)st.lit_len));
        }
        std::memcpy(static_cast<char*>(out) + esz * (size_t)out_row_off[r0], static_cast<char*>(sg.out[k]) + sizeof(Status),
                    esz * (size_t)(out_row_off[r1] - out_row_off[r0]));
        return VB_OK;
    };
    return pipeline_chunks(nch, enqueue, finish_chunk);
}

int vb_text_to_sparsevec_batch_dev(int32_t typmod, int64_t n, const char* text, const int64_t* off, int64_t cap,
                                   int32_t* out_dim, int64_t* out_row_off, int32_t* out_idx, float* out_val,
                                   int64_t* out_bad) {
    if (out_bad) *out_bad = -1;
    VB_TRY(require_init());
    VB_TRY(check_text_args("vb_text_to_sparsevec_batch_dev", n, text, off, cap));
    VB_REQUIRE(typmod == -1 || (typmod >= 1 && typmod <= 1000000000), "vb_text_to_sparsevec_batch_dev: bad typmod %d", typmod);
    VB_REQUIRE(out_row_off && (n == 0 || out_dim), "vb_text_to_sparsevec_batch_dev: out_row_off and out_dim are required");
    return sparse_parse_dev(typmod, n, text, off, cap, out_dim, out_row_off, out_idx, out_val, out_bad, 0, nullptr);
}

int vb_text_to_sparsevec_batch(int32_t typmod, int64_t n, const char* text, const int64_t* off, int64_t cap,
                               int32_t* out_dim, int64_t* out_row_off, int32_t* out_idx, float* out_val,
                               int64_t* out_bad) {
    if (out_bad) *out_bad = -1;
    VB_TRY(require_init());
    VB_TRY(check_text_args("vb_text_to_sparsevec_batch", n, text, off, cap));
    VB_REQUIRE(typmod == -1 || (typmod >= 1 && typmod <= 1000000000), "vb_text_to_sparsevec_batch: bad typmod %d", typmod);
    VB_REQUIRE(out_row_off, "vb_text_to_sparsevec_batch: out_row_off is required");
    out_row_off[0] = 0;
    for (int64_t r = 0; r < n; ++r) out_row_off[r + 1] = out_row_off[r] + host_count(text + off[r], off[r + 1] - off[r]);
    VB_REQUIRE(out_row_off[n] <= cap, "sparsevec_in: the literals need up to %lld entries, more than cap = %lld",
               (long long)out_row_off[n], (long long)cap);
    if (n == 0) return VB_OK;
    VB_REQUIRE(out_dim && out_idx && out_val, "vb_text_to_sparsevec_batch: out_dim, out_idx and out_val are required");
    cudaStream_t s = ctx().stream;
    int64_t done_nnz = 0;
    for (int64_t r0 = 0; r0 < n;) {
        int64_t r1 = r0 + 1;
        while (r1 < n && off[r1 + 1] - off[r0] <= kStageBytes) ++r1;
        const int64_t tb = off[r1] - off[r0], nr = r1 - r0;
        const int64_t bound = out_row_off[r1] - out_row_off[r0];
        void* pin;
        VB_TRY(pinned_buffer((size_t)tb + sizeof(int64_t) * (size_t)(nr + 1) + 16, &pin));
        char* ptext = static_cast<char*>(pin);
        int64_t* poff = reinterpret_cast<int64_t*>(ptext + ((tb + 15) & ~(int64_t)15));
        std::memcpy(ptext, text + off[r0], (size_t)tb);
        for (int64_t i = 0; i <= nr; ++i) poff[i] = off[r0 + i] - off[r0];
        Scratch sc("type I/O");
        void *dtext = nullptr, *doff = nullptr, *ddim = nullptr, *drow = nullptr, *didx = nullptr, *dval = nullptr;
        VB_TRY(sc.own((size_t)tb, &dtext));
        VB_TRY(sc.own(sizeof(int64_t) * (size_t)(nr + 1), &doff));
        VB_TRY(sc.own(sizeof(int32_t) * (size_t)nr, &ddim));
        VB_TRY(sc.own(sizeof(int64_t) * (size_t)(nr + 1), &drow));
        VB_TRY(sc.own(sizeof(int32_t) * (size_t)bound, &didx));
        VB_TRY(sc.own(sizeof(float) * (size_t)bound, &dval));
        VB_CUDA(cudaMemcpyAsync(dtext, ptext, (size_t)tb, cudaMemcpyHostToDevice, s));
        VB_CUDA(cudaMemcpyAsync(doff, poff, sizeof(int64_t) * (size_t)(nr + 1), cudaMemcpyHostToDevice, s));
        VB_TRY(sparse_parse_dev(typmod, nr, static_cast<char*>(dtext), static_cast<int64_t*>(doff), bound,
                                static_cast<int32_t*>(ddim), static_cast<int64_t*>(drow), static_cast<int32_t*>(didx),
                                static_cast<float*>(dval), out_bad, r0, nullptr));
        std::vector<int64_t> rows((size_t)nr + 1);
        VB_CUDA(cudaMemcpy(rows.data(), drow, sizeof(int64_t) * (size_t)(nr + 1), cudaMemcpyDeviceToHost));
        const int64_t nz = rows[(size_t)nr];
        VB_CUDA(cudaMemcpy(out_dim + r0, ddim, sizeof(int32_t) * (size_t)nr, cudaMemcpyDeviceToHost));
        VB_CUDA(cudaMemcpy(out_idx + done_nnz, didx, sizeof(int32_t) * (size_t)nz, cudaMemcpyDeviceToHost));
        VB_CUDA(cudaMemcpy(out_val + done_nnz, dval, sizeof(float) * (size_t)nz, cudaMemcpyDeviceToHost));
        // out_row_off[r0] is already final (earlier chunks); the bound offsets past it become the stored ones
        for (int64_t i = 1; i <= nr; ++i) out_row_off[r0 + i] = done_nnz + rows[(size_t)i];
        done_nnz += nz;
        r0 = r1;
    }
    return VB_OK;
}

int vb_rows_to_text_batch_dev(int elem, int dim, const void* rows, int64_t n, int64_t cap, int64_t* out_off, char* out) {
    VB_TRY(require_init());
    VB_REQUIRE(elem == VB_VECTOR || elem == VB_HALFVEC, "vb_rows_to_text_batch_dev: elem must be VB_VECTOR or VB_HALFVEC");
    VB_REQUIRE(dim >= 1 && n >= 0 && n < (int64_t)INT32_MAX && cap >= 0, "vb_rows_to_text_batch_dev: bad dim %d, n %lld or cap %lld",
               dim, (long long)n, (long long)cap);
    VB_REQUIRE(out_off && (n == 0 || rows), "vb_rows_to_text_batch_dev: rows and out_off are required");
    return format_dev(false, elem, dim, rows, n, nullptr, nullptr, cap, out_off, out, nullptr);
}

int vb_sparsevec_to_text_batch_dev(int dim, int64_t n, const int64_t* row_off, const int32_t* idx, const float* val,
                                   int64_t cap, int64_t* out_off, char* out) {
    VB_TRY(require_init());
    VB_REQUIRE(dim >= 1 && n >= 0 && n < (int64_t)INT32_MAX && cap >= 0, "vb_sparsevec_to_text_batch_dev: bad dim %d, n %lld or cap %lld",
               dim, (long long)n, (long long)cap);
    VB_REQUIRE(out_off && (n == 0 || row_off), "vb_sparsevec_to_text_batch_dev: row_off and out_off are required");
    return format_dev(true, VB_VECTOR, dim, val, n, row_off, idx, cap, out_off, out, nullptr);
}

// host formats: rows in chunks through pinned staging; a length pass over all chunks sizes the text first
static int rows_to_text_host(bool sparse, int elem, int dim, const void* rows, int64_t n, const int64_t* row_off,
                             const int32_t* idx, int64_t cap, int64_t* out_off, char* out) {
    cudaStream_t s = ctx().stream;
    const size_t esz = sparse ? 4 : elem == VB_VECTOR ? 4 : 2;
    const int64_t per_row = sparse ? 0 : (int64_t)dim;
    // chunks whose text is at most kStageBytes by the reference's bound (16 bytes per element, 28 per entry), or one row
    const int64_t max_elems = kStageBytes / (sparse ? 28 : 16);
    auto first = [&](int64_t r) { return sparse ? row_off[r] : r * per_row; };
    std::vector<int64_t> cuts{0};
    while (cuts.back() < n) {
        const int64_t r0 = cuts.back();
        int64_t r1 = r0 + 1;
        while (r1 < n && first(r1 + 1) - first(r0) <= max_elems) ++r1;
        cuts.push_back(r1);
    }
    out_off[0] = 0;
    // pass 0 sizes every chunk (and checks sparsevec rows) before any text is written; pass 1 only writes
    for (int pass = 0; pass < 2; ++pass) {
        if (pass == 1)
            VB_REQUIRE(out_off[n] <= cap, "%s: the text is %lld bytes, more than cap = %lld", sparse ? "sparsevec_out" : "vector_out",
                       (long long)out_off[n], (long long)cap);
        for (size_t c = 0; c + 1 < cuts.size(); ++c) {
            const int64_t r0 = cuts[c], r1 = cuts[c + 1];
            const int64_t nr = r1 - r0, ne = first(r1) - first(r0);
            Scratch sc("type I/O");
            void *drows = nullptr, *didx = nullptr, *droff = nullptr, *doff = nullptr, *dtext = nullptr;
            VB_TRY(sc.own(esz * (size_t)ne, &drows));
            VB_CUDA(cudaMemcpyAsync(drows, static_cast<const char*>(rows) + esz * (size_t)first(r0), esz * (size_t)ne,
                                    cudaMemcpyHostToDevice, s));
            const int64_t* rp = nullptr;
            if (sparse) {
                VB_TRY(sc.own(sizeof(int32_t) * (size_t)ne, &didx));
                VB_TRY(sc.own(sizeof(int64_t) * (size_t)(nr + 1), &droff));
                std::vector<int64_t> ro((size_t)nr + 1);
                for (int64_t i = 0; i <= nr; ++i) ro[(size_t)i] = row_off[r0 + i] - row_off[r0];
                VB_CUDA(cudaMemcpyAsync(didx, idx + row_off[r0], sizeof(int32_t) * (size_t)ne, cudaMemcpyHostToDevice, s));
                VB_CUDA(cudaMemcpy(droff, ro.data(), sizeof(int64_t) * (size_t)(nr + 1), cudaMemcpyHostToDevice));
                rp = static_cast<int64_t*>(droff);
            }
            VB_TRY(sc.own(sizeof(int64_t) * (size_t)(nr + 1), &doff));
            int64_t* dop = static_cast<int64_t*>(doff);
            std::vector<int64_t> o((size_t)nr + 1);
            if (pass == 0) {
                VB_TRY(format_dev(sparse, elem, dim, drows, nr, rp, static_cast<int32_t*>(didx), INT64_MAX, dop, nullptr, nullptr));
                VB_CUDA(cudaMemcpy(o.data(), dop, sizeof(int64_t) * (size_t)(nr + 1), cudaMemcpyDeviceToHost));
                for (int64_t i = 1; i <= nr; ++i) out_off[r0 + i] = out_off[r0] + o[(size_t)i];
            } else {
                const int64_t tb = out_off[r1] - out_off[r0];
                for (int64_t i = 0; i <= nr; ++i) o[(size_t)i] = out_off[r0 + i] - out_off[r0];
                VB_CUDA(cudaMemcpy(dop, o.data(), sizeof(int64_t) * (size_t)(nr + 1), cudaMemcpyHostToDevice));
                VB_TRY(sc.own((size_t)tb, &dtext));
                VB_TRY(format_write(sparse, elem, dim, drows, nr, rp, static_cast<int32_t*>(didx), dop,
                                    static_cast<char*>(dtext)));
                void* pin;
                VB_TRY(pinned_buffer2((size_t)tb + 16, &pin));
                VB_CUDA(cudaMemcpyAsync(pin, dtext, (size_t)tb, cudaMemcpyDeviceToHost, s));
                VB_CUDA(cudaStreamSynchronize(s));
                std::memcpy(out + out_off[r0], pin, (size_t)tb);
            }
        }
    }
    return VB_OK;
}

int vb_rows_to_text_batch(int elem, int dim, const void* rows, int64_t n, int64_t cap, int64_t* out_off, char* out) {
    VB_TRY(require_init());
    VB_REQUIRE(elem == VB_VECTOR || elem == VB_HALFVEC, "vb_rows_to_text_batch: elem must be VB_VECTOR or VB_HALFVEC");
    VB_REQUIRE(dim >= 1 && n >= 0 && n < (int64_t)INT32_MAX && cap >= 0, "vb_rows_to_text_batch: bad dim %d, n %lld or cap %lld",
               dim, (long long)n, (long long)cap);
    VB_REQUIRE(out_off && (n == 0 || rows), "vb_rows_to_text_batch: rows and out_off are required");
    return rows_to_text_host(false, elem, dim, rows, n, nullptr, nullptr, cap, out_off, out);
}

int vb_sparsevec_to_text_batch(int dim, int64_t n, const int64_t* row_off, const int32_t* idx, const float* val,
                               int64_t cap, int64_t* out_off, char* out) {
    VB_TRY(require_init());
    VB_REQUIRE(dim >= 1 && n >= 0 && n < (int64_t)INT32_MAX && cap >= 0, "vb_sparsevec_to_text_batch: bad dim %d, n %lld or cap %lld",
               dim, (long long)n, (long long)cap);
    VB_REQUIRE(out_off && (n == 0 || (row_off && row_off[0] == 0)), "vb_sparsevec_to_text_batch: row_off (from 0) and out_off are required");
    return rows_to_text_host(true, VB_VECTOR, dim, val, n, row_off, idx, cap, out_off, out);
}

}  // extern "C"
