// vb_binary.cu -- the binary type I/O of vector, halfvec and sparsevec over a column: vector_recv / vector_send
// (src/vector.c:376-422), halfvec_recv / halfvec_send (src/halfvec.c:43-72, 373-419) and sparsevec_recv /
// sparsevec_send (src/sparsevec.c:514-585), 1 to 32 lanes per field or row.
//
// The wire format is big-endian and a field starts at any byte, so every kernel moves aligned 16-byte words: it loads
// the two aligned words that cover 16 payload bytes and builds each output word with one __byte_perm, which realigns
// and byte-swaps at once.  Only the few bytes before the first and after the last aligned word of a run go one by one.
#include "vb_common.cuh"
#include "vb_typio.cuh"

#include <algorithm>
#include <cstring>
#include <vector>

namespace vb {
namespace {

constexpr int kMaxDim = 16000;                  // VECTOR_MAX_DIM, HALFVEC_MAX_DIM, SPARSEVEC_MAX_NNZ
constexpr int kSparseMaxDim = 1000000000;       // SPARSEVEC_MAX_DIM
constexpr int kThreads = 256;
constexpr int64_t kStageBytes = 64ll << 20;     // payload bytes per chunk of the host variants
constexpr unsigned long long kNoError = ~0ull;

// The outcome of one field is a key (field << 32 | step): the least key of a batch is the error row-by-row execution
// raises first.  Steps follow the reference's read / check order; a read past the end of the field is the step of the
// read it stops, and bytes left over after a good decode come last.
enum : uint32_t {   // vector_recv / halfvec_recv header steps
    D_SHORT_DIM = 0, D_SHORT_UNUSED, D_DIM_LOW, D_DIM_HIGH, D_TYPMOD, D_UNUSED };
enum : uint32_t {   // sparsevec_recv header steps
    S_SHORT_DIM = 0, S_SHORT_NNZ, S_SHORT_UNUSED, S_DIM_LOW, S_DIM_HIGH, S_NNZ_NEG, S_NNZ_MAX, S_NNZ_DIM, S_TYPMOD,
    S_UNUSED };
// element e of the dense loop: ((e + 2) << 2) | kind; index i: ((i + 4) << 2) | kind; value i: ((nnz + 4 + i) << 2) | kind
enum : uint32_t { K_SHORT = 0, K_NAN = 1, K_INF = 2, K_ZERO = 3 };               // dense elements and sparsevec values
enum : uint32_t { I_SHORT = 0, I_BOUNDS = 1, I_ORDER = 2, I_DUP = 3 };           // sparsevec indices
constexpr uint32_t kTrailing = 0xFFFFFFF0u;
constexpr uint32_t kNone = 0xFFFFFFFFu;

struct Status {                     // the one small result a receive call reads back
    unsigned long long key;         // least outcome key, kNoError when every field decoded
    int32_t dim, nnz, unused, pad;  // the failing field's header (what its error text needs)
};

// __byte_perm selectors over a pair of words (bytes 0..7) starting at byte b: recv takes four consecutive wire bytes
// and reverses each element; send reverses the elements of element-aligned words and takes four consecutive bytes.
template <int ESZ>
__device__ __forceinline__ uint32_t sel_recv(uint32_t b) {
    uint32_t s = 0;
#pragma unroll
    for (int i = 0; i < 4; ++i) s |= (b + (i ^ (ESZ - 1))) << (4 * i);
    return s;
}
template <int ESZ>
__device__ __forceinline__ uint32_t sel_send(uint32_t b) {
    uint32_t s = 0;
#pragma unroll
    for (int i = 0; i < 4; ++i) s |= ((b + i) ^ (ESZ - 1)) << (4 * i);
    return s;
}

// 16 bytes from byte 4 * q0 + (selector's b) of the 32 bytes lo:hi, through sel
__device__ __forceinline__ uint4 realign(uint4 lo, uint4 hi, int q0, uint32_t sel) {
    uint32_t w0, w1, w2, w3, w4;
    switch (q0) {
        case 0: w0 = lo.x; w1 = lo.y; w2 = lo.z; w3 = lo.w; w4 = hi.x; break;
        case 1: w0 = lo.y; w1 = lo.z; w2 = lo.w; w3 = hi.x; w4 = hi.y; break;
        case 2: w0 = lo.z; w1 = lo.w; w2 = hi.x; w3 = hi.y; w4 = hi.z; break;
        default: w0 = lo.w; w1 = hi.x; w2 = hi.y; w3 = hi.z; w4 = hi.w; break;
    }
    return make_uint4(__byte_perm(w0, w1, sel), __byte_perm(w1, w2, sel), __byte_perm(w2, w3, sel),
                      __byte_perm(w3, w4, sel));
}

// the aligned 16-byte words holding p .. p + 15; the second is read only when p is unaligned, so no word without a
// byte of the run is read
__device__ __forceinline__ void load_pair(const uint8_t* p, uint4* lo, uint4* hi) {
    const uintptr_t a = reinterpret_cast<uintptr_t>(p);
    const uint4* w = reinterpret_cast<const uint4*>(a & ~(uintptr_t)15);
    *lo = __ldg(w);
    *hi = (a & 15) ? __ldg(w + 1) : make_uint4(0, 0, 0, 0);
}

// a big-endian int32 at any byte (both aligned words hold bytes of it)
__device__ __forceinline__ uint32_t load_be32(const uint8_t* p) {
    const uintptr_t a = reinterpret_cast<uintptr_t>(p);
    const uint32_t* w = reinterpret_cast<const uint32_t*>(a & ~(uintptr_t)3);
    const uint32_t b = (uint32_t)(a & 3);
    return __byte_perm(__ldg(w), b ? __ldg(w + 1) : 0u, sel_recv<4>(b));
}
__device__ __forceinline__ uint32_t load_be16(const uint8_t* p) { return ((uint32_t)__ldg(p) << 8) | __ldg(p + 1); }

// CheckElement of a float (ESZ 4) or half (ESZ 2) on its bits: 0, K_NAN or K_INF
template <int ESZ>
__device__ __forceinline__ uint32_t element_kind(uint32_t v) {
    if (ESZ == 4) return (v & 0x7f800000u) != 0x7f800000u ? 0u : (v & 0x7fffffu) ? K_NAN : K_INF;
    return (v & 0x7c00u) != 0x7c00u ? 0u : (v & 0x3ffu) ? K_NAN : K_INF;
}

// Decodes n_el big-endian elements from src (any byte) to dst (ESZ-aligned) with the g lanes of a group (lane j);
// check(e, bits) runs on every element in ascending order per lane and returns its key or kNone.  The lane's least
// key is returned.
template <int ESZ, typename Check>
__device__ __forceinline__ uint32_t recv_run(const uint8_t* src, int64_t n_el, uint8_t* dst, int j, int g, Check check) {
    const int64_t nb = n_el * ESZ;
    const int64_t hb = std::min<int64_t>(nb, (16 - (int64_t)(reinterpret_cast<uintptr_t>(dst) & 15)) & 15);
    const int64_t nw = (nb - hb) >> 4;
    const int64_t tb = nb - hb - (nw << 4);
    uint32_t best = kNone;
    // the elements before the first and after the last aligned output word
    for (int64_t t = j; t < (hb + tb) / ESZ; t += g) {
        const int64_t e = t < hb / ESZ ? t : (hb + (nw << 4)) / ESZ + (t - hb / ESZ);
        const uint32_t v = ESZ == 4 ? load_be32(src + e * 4) : load_be16(src + e * 2);
        if (ESZ == 4) reinterpret_cast<uint32_t*>(dst)[e] = v;
        else reinterpret_cast<uint16_t*>(dst)[e] = (uint16_t)v;
        best = min(best, check(e, v));
    }
    const uint32_t sh = (uint32_t)(reinterpret_cast<uintptr_t>(src + hb) & 15);
    const uint32_t sel = sel_recv<ESZ>(sh & 3);
    for (int64_t w = j; w < nw; w += g) {
        uint4 lo, hi;
        load_pair(src + hb + (w << 4), &lo, &hi);
        const uint4 o = realign(lo, hi, (int)(sh >> 2), sel);
        *reinterpret_cast<uint4*>(dst + hb + (w << 4)) = o;
        const int64_t e0 = (hb + (w << 4)) / ESZ;
        const uint32_t x[4] = {o.x, o.y, o.z, o.w};
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            if (ESZ == 4) {
                best = min(best, check(e0 + k, x[k]));
            } else {
                best = min(best, check(e0 + 2 * k, x[k] & 0xffffu));
                best = min(best, check(e0 + 2 * k + 1, x[k] >> 16));
            }
        }
    }
    return best;
}

// Encodes nb bytes of ESZ-byte elements from src (ESZ-aligned) big-endian to dst (any byte) with the g lanes of a
// group: aligned 16-byte stores inside the run, byte stores at its two ends (which may share a word with a neighbour).
template <int ESZ>
__device__ __forceinline__ void send_run(const uint8_t* src, int64_t nb, uint8_t* dst, int j, int g) {
    const int64_t hb = std::min<int64_t>(nb, (16 - (int64_t)(reinterpret_cast<uintptr_t>(dst) & 15)) & 15);
    const int64_t nw = (nb - hb) >> 4;
    const int64_t tb = nb - hb - (nw << 4);
    for (int64_t t = j; t < hb + tb; t += g) {
        const int64_t m = t < hb ? t : hb + (nw << 4) + (t - hb);
        dst[m] = __ldg(src + (m ^ (ESZ - 1)));
    }
    const uint32_t sh = (uint32_t)(reinterpret_cast<uintptr_t>(src + hb) & 15);
    const uint32_t sel = sel_send<ESZ>(sh & 3);
    for (int64_t w = j; w < nw; w += g) {
        uint4 lo, hi;
        load_pair(src + hb + (w << 4), &lo, &hi);
        *reinterpret_cast<uint4*>(dst + hb + (w << 4)) = realign(lo, hi, (int)(sh >> 2), sel);
    }
}

// the least key of a warp's lanes to st->key (one atomicMin per warp that holds an error)
__device__ __forceinline__ void warp_min_key(unsigned long long best, Status* st) {
    const uint32_t hi = __reduce_min_sync(~0u, (uint32_t)(best >> 32));
    const uint32_t lo = __reduce_min_sync(~0u, (uint32_t)(best >> 32) == hi ? (uint32_t)best : kNone);
    const unsigned long long k = ((unsigned long long)hi << 32) | lo;
    if ((threadIdx.x & 31) == 0 && k != kNoError) atomicMin(&st->key, k);
}

__device__ __forceinline__ unsigned long long field_key(int64_t r, uint32_t step) {
    return step == kNone ? kNoError : ((unsigned long long)r << 32) | step;
}

// ---------------------------------------------------------------------------------------------------- kernels
// the bound of every field: max(0, (len - hdr) / per)
__global__ void bound_kernel(const int64_t* off, int64_t n, int hdr, int per, int64_t* count) {
    for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < n; r += (int64_t)gridDim.x * blockDim.x) {
        const int64_t len = off[r + 1] - off[r];
        count[r] = len > hdr ? (len - hdr) / per : 0;
    }
}

// vector_recv / halfvec_recv: 2^lg lanes per field, elements to out at row_off (the bound offsets)
template <int ESZ>
__global__ void __launch_bounds__(kThreads) recv_dense_kernel(const uint8_t* bytes, const int64_t* off, int64_t n,
                                                              int32_t typmod, const int64_t* row_off, uint8_t* out,
                                                              int lg, Status* st) {
    const int g = 1 << lg, j = (int)(threadIdx.x & (g - 1));
    unsigned long long best = kNoError;
    for (int64_t r = ((int64_t)blockIdx.x * kThreads + threadIdx.x) >> lg; r < n; r += ((int64_t)gridDim.x * kThreads) >> lg) {
        const int64_t b = off[r], len = std::max<int64_t>(off[r + 1] - b, 0);
        const uint8_t* p = bytes + b;
        const int64_t bound = row_off[r + 1] - row_off[r];
        uint32_t key;
        int64_t dim = 0;
        if (len < 2) key = D_SHORT_DIM;
        else if (len < 4) key = D_SHORT_UNUSED;
        else {
            dim = load_be16(p);
            const uint32_t unused = load_be16(p + 2);
            if (dim < 1) key = D_DIM_LOW;
            else if (dim > kMaxDim) key = D_DIM_HIGH;
            else if (typmod != -1 && typmod != dim) key = D_TYPMOD;
            else if (unused != 0) key = D_UNUSED;
            else if (dim > bound) key = ((uint32_t)(bound + 2) << 2) | K_SHORT;   // the read of element `bound`
            else if (4 + dim * ESZ != len) key = kTrailing;
            else key = kNone;
        }
        if (key >= 8) {   // the header passed: the element loop, up to the first element past the end
            const uint32_t k = recv_run<ESZ>(p + 4, std::min(dim, bound), out + row_off[r] * ESZ, j, g,
                                             [](int64_t e, uint32_t v) -> uint32_t {
                                                 const uint32_t kind = element_kind<ESZ>(v);
                                                 return kind ? ((uint32_t)(e + 2) << 2) | kind : kNone;
                                             });
            key = min(key, k);
        }
        best = min(best, field_key(r, key));
    }
    warp_min_key(best, st);
}

// sparsevec_recv: 2^lg lanes per field, entries to the CSR at row_off (the bound offsets), dimensions to out_dim
__global__ void __launch_bounds__(kThreads) recv_sparse_kernel(const uint8_t* bytes, const int64_t* off, int64_t n,
                                                               int32_t typmod, const int64_t* row_off, int32_t* out_dim,
                                                               int32_t* out_idx, float* out_val, int lg, Status* st) {
    const int g = 1 << lg, j = (int)(threadIdx.x & (g - 1));
    unsigned long long best = kNoError;
    for (int64_t r = ((int64_t)blockIdx.x * kThreads + threadIdx.x) >> lg; r < n; r += ((int64_t)gridDim.x * kThreads) >> lg) {
        const int64_t b = off[r], len = std::max<int64_t>(off[r + 1] - b, 0);
        const uint8_t* p = bytes + b;
        const int64_t ro = row_off[r], bound = row_off[r + 1] - ro;
        uint32_t key;
        int32_t dim = 0, nnz = 0;
        if (len >= 4) dim = (int32_t)load_be32(p);
        if (len < 4) key = S_SHORT_DIM;
        else if (len < 8) key = S_SHORT_NNZ;
        else if (len < 12) key = S_SHORT_UNUSED;
        else {
            nnz = (int32_t)load_be32(p + 4);
            const int32_t unused = (int32_t)load_be32(p + 8);
            if (dim < 1) key = S_DIM_LOW;
            else if (dim > kSparseMaxDim) key = S_DIM_HIGH;
            else if (nnz < 0) key = S_NNZ_NEG;
            else if (nnz > kMaxDim) key = S_NNZ_MAX;
            else if (nnz > dim) key = S_NNZ_DIM;
            else if (typmod != -1 && typmod != dim) key = S_TYPMOD;
            else if (unused != 0) key = S_UNUSED;
            else key = kNone;
        }
        if (j == 0) out_dim[r] = dim;
        if (key == kNone) {
            // indices fit up to ib, values up to vb; a read past either stops the field there
            const int64_t ib = (len - 12) / 4;
            const int64_t vb = nnz <= ib ? (len - 12 - 4 * (int64_t)nnz) / 4 : 0;
            if (nnz > ib) key = ((uint32_t)(ib + 4) << 2) | I_SHORT;
            else if (nnz > vb) key = ((uint32_t)(nnz + 4 + vb) << 2) | K_SHORT;
            else if (12 + 8 * (int64_t)nnz != len) key = kTrailing;
            // CheckIndex of every index read (i < min(nnz, ib)); only the first `bound` can be stored
            const uint8_t* pi = p + 12;
            for (int64_t i = j; i < std::min<int64_t>(nnz, ib); i += g) {
                const int32_t x = (int32_t)load_be32(pi + 4 * i);
                uint32_t kind = 0;
                if (x < 0 || x >= dim) kind = I_BOUNDS;
                else if (i > 0) {
                    const int32_t prev = (int32_t)load_be32(pi + 4 * (i - 1));
                    kind = x < prev ? I_ORDER : x == prev ? I_DUP : 0;
                }
                if (i < bound) out_idx[ro + i] = x;
                if (kind) {
                    key = min(key, ((uint32_t)(i + 4) << 2) | kind);
                    break;
                }
            }
            if (nnz <= ib) {
                const uint32_t vbase = (uint32_t)(nnz + 4);
                const uint32_t k = recv_run<4>(pi + 4 * (int64_t)nnz, std::min<int64_t>(std::min<int64_t>(nnz, vb), bound),
                                               reinterpret_cast<uint8_t*>(out_val + ro), j, g,
                                               [vbase](int64_t i, uint32_t v) -> uint32_t {
                                                   uint32_t kind = element_kind<4>(v);
                                                   if (!kind && (v & 0x7fffffffu) == 0) kind = K_ZERO;
                                                   return kind ? ((vbase + (uint32_t)i) << 2) | kind : kNone;
                                               });
                key = min(key, k);
            }
        }
        best = min(best, field_key(r, key));
    }
    warp_min_key(best, st);
}

// the failing field's header, for its error text
__global__ void record_kernel(const uint8_t* bytes, const int64_t* off, bool sparse, Status* st) {
    const unsigned long long k = st->key;
    if (k == kNoError) return;
    const int64_t r = (int64_t)(k >> 32);
    const uint8_t* p = bytes + off[r];
    const int64_t len = off[r + 1] - off[r];
    if (sparse) {
        st->dim = len >= 4 ? (int32_t)load_be32(p) : 0;
        st->nnz = len >= 8 ? (int32_t)load_be32(p + 4) : 0;
        st->unused = len >= 12 ? (int32_t)load_be32(p + 8) : 0;
    } else {
        st->dim = len >= 2 ? (int32_t)load_be16(p) : 0;
        st->unused = len >= 4 ? (int32_t)load_be16(p + 2) : 0;
    }
}

// vector_send / halfvec_send: 2^lg lanes per row; out_off from every thread, the rows only when out is set
template <int ESZ>
__global__ void __launch_bounds__(kThreads) send_dense_kernel(const uint8_t* rows, int dim, int64_t n, int lg,
                                                              int64_t* out_off, uint8_t* out) {
    const int64_t rb = 4 + (int64_t)dim * ESZ;
    const int64_t t0 = (int64_t)blockIdx.x * kThreads + threadIdx.x, nt = (int64_t)gridDim.x * kThreads;
    for (int64_t i = t0; i <= n; i += nt) out_off[i] = i * rb;
    if (!out) return;
    const int g = 1 << lg, j = (int)(threadIdx.x & (g - 1));
    for (int64_t r = t0 >> lg; r < n; r += nt >> lg) {
        uint8_t* o = out + r * rb;
        if (j == 0) {
            o[0] = (uint8_t)(dim >> 8);
            o[1] = (uint8_t)dim;
            o[2] = 0;
            o[3] = 0;
        }
        send_run<ESZ>(rows + r * (int64_t)dim * ESZ, (int64_t)dim * ESZ, o + 4, j, g);
    }
}

// sparsevec_send of checked CSR rows (offsets from 0): out_off[i] = 12 i + 8 row_off[i]
__global__ void __launch_bounds__(kThreads) send_sparse_kernel(int dim, int64_t n, const int64_t* row_off,
                                                               const int32_t* idx, const float* val, int lg,
                                                               int64_t* out_off, uint8_t* out) {
    const int64_t t0 = (int64_t)blockIdx.x * kThreads + threadIdx.x, nt = (int64_t)gridDim.x * kThreads;
    for (int64_t i = t0; i <= n; i += nt) out_off[i] = 12 * i + 8 * row_off[i];
    if (!out) return;
    const int g = 1 << lg, j = (int)(threadIdx.x & (g - 1));
    for (int64_t r = t0 >> lg; r < n; r += nt >> lg) {
        const int64_t b = row_off[r], nnz = row_off[r + 1] - b;
        uint8_t* o = out + 12 * r + 8 * b;
        if (j == 0) {
            const uint32_t h[3] = {(uint32_t)dim, (uint32_t)nnz, 0u};
            for (int q = 0; q < 12; ++q) o[q] = (uint8_t)(h[q >> 2] >> (8 * (3 - (q & 3))));
        }
        send_run<4>(reinterpret_cast<const uint8_t*>(idx + b), 4 * nnz, o + 12, j, g);
        send_run<4>(reinterpret_cast<const uint8_t*>(val + b), 4 * nnz, o + 12 + 4 * nnz, j, g);
    }
}

// ---------------------------------------------------------------------------------------------------- host side
// 2^lg lanes per field or row of about `units` 16-byte words: up to a warp
int lanes_lg(int64_t units) {
    int lg = 0;
    while (lg < 5 && ((int64_t)1 << lg) < units) ++lg;
    return lg;
}

unsigned grid_for(int64_t n, int lg) {
    const int64_t want = ((n << lg) + kThreads - 1) / kThreads;
    const int64_t cap = (int64_t)ctx().sm_count * 16;
    return (unsigned)std::max<int64_t>(1, std::min(want, cap));
}

const char* type_name(int kind) { return kind == 0 ? "vector" : kind == 1 ? "halfvec" : "sparsevec"; }

// The reference's error for a recorded failure (kind 0 vector, 1 halfvec, 2 sparsevec).  The two texts of a read past
// the end and of bytes left over are PostgreSQL's: pq_copymsgbytes and CopyReadBinaryAttribute.
int recv_error(int kind, int32_t typmod, const Status& st) {
    const char* t = type_name(kind);
    const uint32_t step = (uint32_t)st.key;
    auto fail = [](const char* fmt, auto... a) {
        set_error(fmt, a...);
        return VB_EINVAL;
    };
    if (step == kTrailing) return fail("incorrect binary data format");
    if (kind != 2) {
        switch (step) {
            case D_SHORT_DIM: case D_SHORT_UNUSED: return fail("insufficient data left in message");
            case D_DIM_LOW: return fail("%s must have at least 1 dimension", t);
            case D_DIM_HIGH: return fail("%s cannot have more than %d dimensions", t, kMaxDim);
            case D_TYPMOD: return fail("expected %d dimensions, not %d", typmod, st.dim);
            case D_UNUSED: return fail("expected unused to be 0, not %d", st.unused);
        }
        switch (step & 3) {
            case K_SHORT: return fail("insufficient data left in message");
            case K_NAN: return fail("NaN not allowed in %s", t);
            default: return fail("infinite value not allowed in %s", t);
        }
    }
    switch (step) {
        case S_SHORT_DIM: case S_SHORT_NNZ: case S_SHORT_UNUSED: return fail("insufficient data left in message");
        case S_DIM_LOW: return fail("sparsevec must have at least 1 dimension");
        case S_DIM_HIGH: return fail("sparsevec cannot have more than %d dimensions", kSparseMaxDim);
        case S_NNZ_NEG: return fail("sparsevec cannot have negative number of elements");
        case S_NNZ_MAX: return fail("sparsevec cannot have more than %d non-zero elements", kMaxDim);
        case S_NNZ_DIM: return fail("sparsevec cannot have more elements than dimensions");
        case S_TYPMOD: return fail("expected %d dimensions, not %d", typmod, st.dim);
        case S_UNUSED: return fail("expected unused to be 0, not %d", st.unused);
    }
    if ((int64_t)(step >> 2) - 4 < (int64_t)st.nnz) {   // the index loop
        switch (step & 3) {
            case I_SHORT: return fail("insufficient data left in message");
            case I_BOUNDS: return fail("sparsevec index out of bounds");
            case I_ORDER: return fail("sparsevec indices must be in ascending order");
            default: return fail("sparsevec indices must not contain duplicates");
        }
    }
    switch (step & 3) {
        case K_SHORT: return fail("insufficient data left in message");
        case K_NAN: return fail("NaN not allowed in sparsevec");
        case K_INF: return fail("infinite value not allowed in sparsevec");
        default: return fail("binary representation of sparsevec cannot contain zero values");
    }
}

int status_reset(Status* st) {
    VB_CUDA(cudaMemsetAsync(st, 0, sizeof(Status), ctx().stream));
    VB_CUDA(cudaMemsetAsync(&st->key, 0xff, sizeof(st->key), ctx().stream));
    return VB_OK;
}

// enqueue the decode of n >= 1 fields into the bound offsets row_off (already written) and the record of the first
// failure; `units` is the average field's size in 16-byte words (lanes per field)
int recv_enqueue(int kind, int32_t typmod, int64_t n, const uint8_t* bytes, const int64_t* off, const int64_t* row_off,
                 void* out, int32_t* out_dim, int32_t* out_idx, float* out_val, int64_t units, Status* st) {
    cudaStream_t s = ctx().stream;
    VB_TRY(status_reset(st));
    const int lg = lanes_lg(units);
    {
        ProfScope prof(VB_PROF_BINARY_RECV);
        if (kind == 0)
            recv_dense_kernel<4><<<grid_for(n, lg), kThreads, 0, s>>>(bytes, off, n, typmod, row_off,
                                                                     static_cast<uint8_t*>(out), lg, st);
        else if (kind == 1)
            recv_dense_kernel<2><<<grid_for(n, lg), kThreads, 0, s>>>(bytes, off, n, typmod, row_off,
                                                                     static_cast<uint8_t*>(out), lg, st);
        else
            recv_sparse_kernel<<<grid_for(n, lg), kThreads, 0, s>>>(bytes, off, n, typmod, row_off, out_dim, out_idx,
                                                                   out_val, lg, st);
        VB_CUDA(cudaGetLastError());
    }
    record_kernel<<<1, 1, 0, s>>>(bytes, off, kind == 2, st);
    VB_CUDA(cudaGetLastError());
    count_launch(2);
    return VB_OK;
}

int check_recv_args(const char* fn, int64_t n, const void* bytes, const int64_t* off, int64_t cap, int32_t typmod,
                    bool sparse) {
    VB_REQUIRE(n >= 0 && n < (int64_t)INT32_MAX, "%s: bad field count %lld", fn, (long long)n);
    VB_REQUIRE(cap >= 0, "%s: bad cap %lld", fn, (long long)cap);
    VB_REQUIRE(n == 0 || (bytes && off), "%s: bytes and off are required", fn);
    VB_REQUIRE(typmod == -1 || (typmod >= 1 && typmod <= (sparse ? kSparseMaxDim : kMaxDim)), "%s: bad typmod %d", fn, typmod);
    return VB_OK;
}

// header bytes and bytes per stored unit of a field
void field_shape(int kind, int* hdr, int* per) {
    *hdr = kind == 2 ? 12 : 4;
    *per = kind == 2 ? 8 : kind == 0 ? 4 : 2;
}

// the receive of n fields on the device: bound offsets, cap check, decode, one read of the status
int recv_dev(int kind, int32_t typmod, int64_t n, const uint8_t* bytes, const int64_t* off, int64_t cap,
             int64_t* out_row_off, void* out, int32_t* out_dim, int32_t* out_idx, float* out_val, int64_t* out_bad) {
    const char* fn = kind == 2 ? "vb_binary_to_sparsevec_batch_dev" : "vb_binary_to_rows_batch_dev";
    cudaStream_t s = ctx().stream;
    int hdr, per;
    field_shape(kind, &hdr, &per);
    {
        Scratch sc("type I/O");
        void* cnt = nullptr;
        VB_TRY(sc.own(sizeof(int64_t) * (size_t)n, &cnt));
        if (n) bound_kernel<<<grid_for(n, 0), kThreads, 0, s>>>(off, n, hdr, per, static_cast<int64_t*>(cnt));
        VB_CUDA(cudaGetLastError());
        count_launch();
        VB_TRY(offsets_from_counts(static_cast<int64_t*>(cnt), n, out_row_off));
    }
    int64_t total = 0;
    VB_CUDA(cudaMemcpyAsync(&total, out_row_off + n, sizeof(int64_t), cudaMemcpyDeviceToHost, s));
    VB_CUDA(cudaStreamSynchronize(s));
    VB_REQUIRE(total <= cap, "%s: the fields need %lld %s, more than cap = %lld", fn, (long long)total,
               kind == 2 ? "entries" : "elements", (long long)cap);
    if (n == 0) return VB_OK;
    VB_REQUIRE(kind == 2 ? (out_dim && (total == 0 || (out_idx && out_val))) : (total == 0 || out != nullptr),
               "%s: the outputs are required", fn);
    Scratch sc("type I/O");
    void* st = nullptr;
    VB_TRY(sc.own(sizeof(Status), &st));
    Status* sp = static_cast<Status*>(st);
    VB_TRY(recv_enqueue(kind, typmod, n, bytes, off, out_row_off, out, out_dim, out_idx, out_val,
                        (total * per / n + 15) / 16, sp));
    Status h;
    VB_CUDA(cudaMemcpyAsync(&h, sp, sizeof(Status), cudaMemcpyDeviceToHost, s));
    VB_CUDA(cudaStreamSynchronize(s));
    if (h.key == kNoError) return VB_OK;
    if (out_bad) *out_bad = (int64_t)(h.key >> 32);
    return recv_error(kind, typmod, h);
}

// The receive of n host fields: bound offsets on the host, then chunks of at most kStageBytes of payload (or one
// larger field) through the two pinned slots.  Each slot carries [payload | off | row_off] in and
// [Status | rows or (dims | idx | val)] out.
int recv_host(int kind, int32_t typmod, int64_t n, const uint8_t* bytes, const int64_t* off, int64_t cap,
              int64_t* out_row_off, void* out, int32_t* out_dim, int32_t* out_idx, float* out_val, int64_t* out_bad) {
    const char* fn = kind == 2 ? "vb_binary_to_sparsevec_batch" : "vb_binary_to_rows_batch";
    int hdr, per;
    field_shape(kind, &hdr, &per);
    out_row_off[0] = 0;
    for (int64_t r = 0; r < n; ++r) {
        const int64_t len = off[r + 1] - off[r];
        out_row_off[r + 1] = out_row_off[r] + (len > hdr ? (len - hdr) / per : 0);
    }
    VB_REQUIRE(out_row_off[n] <= cap, "%s: the fields need %lld %s, more than cap = %lld", fn, (long long)out_row_off[n],
               kind == 2 ? "entries" : "elements", (long long)cap);
    if (n == 0) return VB_OK;
    VB_REQUIRE(kind == 2 ? (out_dim && (out_row_off[n] == 0 || (out_idx && out_val))) : (out_row_off[n] == 0 || out != nullptr),
               "%s: the outputs are required", fn);
    const size_t esz = kind == 2 ? 4 : (size_t)per;   // bytes per stored element (sparsevec: per array)
    const int64_t planes = kind == 2 ? 2 : 1;
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
    Staging& sg = staging();
    const size_t tb_al = ((size_t)max_tb + 15) & ~(size_t)15;
    const size_t dims_al = kind == 2 ? ((sizeof(int32_t) * (size_t)max_nr + 15) & ~(size_t)15) : 0;
    const size_t ne_al = (esz * (size_t)max_ne + 15) & ~(size_t)15;
    const size_t in_bytes = tb_al + sizeof(int64_t) * 2 * (size_t)(max_nr + 1);
    const size_t out_bytes = sizeof(Status) + dims_al + (size_t)planes * ne_al;
    Scratch sc("type I/O");
    void *dbytes[2] = {}, *doff[2] = {}, *dout[2] = {}, *dst[2] = {};
    for (int k = 0; k < 2 && k < nch; ++k) {
        VB_TRY(pinned_grow(&sg.in[k], &sg.in_bytes[k], in_bytes));
        VB_TRY(pinned_grow(&sg.out[k], &sg.out_bytes[k], out_bytes));
        VB_TRY(sc.own((size_t)max_tb, &dbytes[k]));
        VB_TRY(sc.own(sizeof(int64_t) * 2 * (size_t)(max_nr + 1), &doff[k]));
        VB_TRY(sc.own(dims_al + (size_t)planes * ne_al, &dout[k]));
        VB_TRY(sc.own(sizeof(Status), &dst[k]));
    }
    cudaStream_t s = ctx().stream;
    auto enqueue = [&](int64_t c, int k) -> int {
        const int64_t r0 = cuts[c], r1 = cuts[c + 1];
        const int64_t tb = off[r1] - off[r0], nr = r1 - r0, ne = out_row_off[r1] - out_row_off[r0];
        uint8_t* pin = static_cast<uint8_t*>(sg.in[k]);
        int64_t* poff = reinterpret_cast<int64_t*>(pin + tb_al);
        std::memcpy(pin, bytes + off[r0], (size_t)tb);
        for (int64_t i = 0; i <= nr; ++i) {
            poff[i] = off[r0 + i] - off[r0];
            poff[nr + 1 + i] = out_row_off[r0 + i] - out_row_off[r0];
        }
        VB_CUDA(cudaMemcpyAsync(dbytes[k], pin, (size_t)tb, cudaMemcpyHostToDevice, s));
        VB_CUDA(cudaMemcpyAsync(doff[k], poff, sizeof(int64_t) * 2 * (size_t)(nr + 1), cudaMemcpyHostToDevice, s));
        const int64_t* doffp = static_cast<int64_t*>(doff[k]);
        uint8_t* o = static_cast<uint8_t*>(dout[k]);
        Status* sp = static_cast<Status*>(dst[k]);
        VB_TRY(recv_enqueue(kind, typmod, nr, static_cast<uint8_t*>(dbytes[k]), doffp, doffp + nr + 1, o,
                            reinterpret_cast<int32_t*>(o), reinterpret_cast<int32_t*>(o + dims_al),
                            reinterpret_cast<float*>(o + dims_al + ne_al), (ne * per / nr + 15) / 16, sp));
        uint8_t* po = static_cast<uint8_t*>(sg.out[k]);
        VB_CUDA(cudaMemcpyAsync(po, sp, sizeof(Status), cudaMemcpyDeviceToHost, s));
        if (kind == 2) {
            VB_CUDA(cudaMemcpyAsync(po + sizeof(Status), o, sizeof(int32_t) * (size_t)nr, cudaMemcpyDeviceToHost, s));
            VB_CUDA(cudaMemcpyAsync(po + sizeof(Status) + dims_al, o + dims_al, esz * (size_t)ne, cudaMemcpyDeviceToHost, s));
            VB_CUDA(cudaMemcpyAsync(po + sizeof(Status) + dims_al + ne_al, o + dims_al + ne_al, esz * (size_t)ne,
                                    cudaMemcpyDeviceToHost, s));
        } else {
            VB_CUDA(cudaMemcpyAsync(po + sizeof(Status), o, esz * (size_t)ne, cudaMemcpyDeviceToHost, s));
        }
        return VB_OK;
    };
    auto finish = [&](int64_t c, int k) -> int {
        const int64_t r0 = cuts[c], r1 = cuts[c + 1];
        const int64_t e0 = out_row_off[r0], ne = out_row_off[r1] - e0;
        const uint8_t* po = static_cast<const uint8_t*>(sg.out[k]);
        const Status& st = *reinterpret_cast<const Status*>(po);
        if (st.key != kNoError) {
            if (out_bad) *out_bad = r0 + (int64_t)(st.key >> 32);
            return recv_error(kind, typmod, st);
        }
        po += sizeof(Status);
        if (kind == 2) {
            std::memcpy(out_dim + r0, po, sizeof(int32_t) * (size_t)(r1 - r0));
            std::memcpy(out_idx + e0, po + dims_al, esz * (size_t)ne);
            std::memcpy(out_val + e0, po + dims_al + ne_al, esz * (size_t)ne);
        } else {
            std::memcpy(static_cast<uint8_t*>(out) + esz * (size_t)e0, po, esz * (size_t)ne);
        }
        return VB_OK;
    };
    return pipeline_chunks(nch, enqueue, finish);
}

int check_send_args(const char* fn, int dim, int64_t n, int64_t cap, const int64_t* out_off, bool have_rows) {
    VB_REQUIRE(dim >= 1 && n >= 0 && n < (int64_t)INT32_MAX && cap >= 0, "%s: bad dim %d, n %lld or cap %lld", fn, dim,
               (long long)n, (long long)cap);
    VB_REQUIRE(out_off && (n == 0 || have_rows), "%s: rows and out_off are required", fn);
    return VB_OK;
}

// enqueue the offsets (and, with out, the payloads) of n dense rows; no read back
int send_dense_enqueue(int elem, int dim, const void* rows, int64_t n, int64_t* out_off, void* out) {
    const int esz = elem == VB_VECTOR ? 4 : 2;
    const int lg = out ? lanes_lg(((int64_t)dim * esz + 15) / 16) : 0;
    cudaStream_t s = ctx().stream;
    ProfScope prof(VB_PROF_BINARY_SEND);
    const unsigned grid = grid_for(n, lg);
    if (esz == 4)
        send_dense_kernel<4><<<grid, kThreads, 0, s>>>(static_cast<const uint8_t*>(rows), dim, n, lg, out_off,
                                                       static_cast<uint8_t*>(out));
    else
        send_dense_kernel<2><<<grid, kThreads, 0, s>>>(static_cast<const uint8_t*>(rows), dim, n, lg, out_off,
                                                       static_cast<uint8_t*>(out));
    VB_CUDA(cudaGetLastError());
    count_launch();
    return VB_OK;
}

// check the CSR of n >= 1 device rows (one 24-byte read), then enqueue the offsets and, when out is set and the
// payloads fit cap, the payloads
int send_sparse_dev(int dim, int64_t n, const int64_t* row_off, const int32_t* idx, const float* val, int64_t cap,
                    int64_t* out_off, void* out, const char* fn) {
    int64_t nnz = 0;
    VB_TRY(sparse_csr_check_dev("sparsevec_send", dim, n, row_off, idx, &nnz));
    const int64_t total = 12 * n + 8 * nnz;
    const bool write = out && total <= cap;
    const int lg = write ? lanes_lg((nnz * 4 / n + 15) / 16) : 0;
    {
        ProfScope prof(VB_PROF_BINARY_SEND);
        send_sparse_kernel<<<grid_for(n, lg), kThreads, 0, ctx().stream>>>(dim, n, row_off, idx, val, lg, out_off,
                                                                           write ? static_cast<uint8_t*>(out) : nullptr);
        VB_CUDA(cudaGetLastError());
        count_launch();
    }
    VB_REQUIRE(!out || total <= cap, "%s: the payloads are %lld bytes, more than cap = %lld", fn, (long long)total,
               (long long)cap);
    return VB_OK;
}

}  // namespace
}  // namespace vb

using namespace vb;

extern "C" {

int vb_binary_to_rows_batch_dev(int elem, int32_t typmod, int64_t n, const void* bytes, const int64_t* off, int64_t cap,
                                int64_t* out_row_off, void* out, int64_t* out_bad) {
    if (out_bad) *out_bad = -1;
    VB_TRY(require_init());
    VB_TRY(check_recv_args("vb_binary_to_rows_batch_dev", n, bytes, off, cap, typmod, false));
    VB_REQUIRE(elem == VB_VECTOR || elem == VB_HALFVEC, "vb_binary_to_rows_batch_dev: elem must be VB_VECTOR or VB_HALFVEC");
    VB_REQUIRE(out_row_off, "vb_binary_to_rows_batch_dev: out_row_off is required");
    return recv_dev(elem == VB_VECTOR ? 0 : 1, typmod, n, static_cast<const uint8_t*>(bytes), off, cap, out_row_off, out,
                    nullptr, nullptr, nullptr, out_bad);
}

int vb_binary_to_rows_batch(int elem, int32_t typmod, int64_t n, const void* bytes, const int64_t* off, int64_t cap,
                            int64_t* out_row_off, void* out, int64_t* out_bad) {
    if (out_bad) *out_bad = -1;
    VB_TRY(require_init());
    VB_TRY(check_recv_args("vb_binary_to_rows_batch", n, bytes, off, cap, typmod, false));
    VB_REQUIRE(elem == VB_VECTOR || elem == VB_HALFVEC, "vb_binary_to_rows_batch: elem must be VB_VECTOR or VB_HALFVEC");
    VB_REQUIRE(out_row_off, "vb_binary_to_rows_batch: out_row_off is required");
    return recv_host(elem == VB_VECTOR ? 0 : 1, typmod, n, static_cast<const uint8_t*>(bytes), off, cap, out_row_off, out,
                     nullptr, nullptr, nullptr, out_bad);
}

int vb_binary_to_sparsevec_batch_dev(int32_t typmod, int64_t n, const void* bytes, const int64_t* off, int64_t cap,
                                     int32_t* out_dim, int64_t* out_row_off, int32_t* out_idx, float* out_val,
                                     int64_t* out_bad) {
    if (out_bad) *out_bad = -1;
    VB_TRY(require_init());
    VB_TRY(check_recv_args("vb_binary_to_sparsevec_batch_dev", n, bytes, off, cap, typmod, true));
    VB_REQUIRE(out_row_off, "vb_binary_to_sparsevec_batch_dev: out_row_off is required");
    return recv_dev(2, typmod, n, static_cast<const uint8_t*>(bytes), off, cap, out_row_off, nullptr, out_dim, out_idx,
                    out_val, out_bad);
}

int vb_binary_to_sparsevec_batch(int32_t typmod, int64_t n, const void* bytes, const int64_t* off, int64_t cap,
                                 int32_t* out_dim, int64_t* out_row_off, int32_t* out_idx, float* out_val,
                                 int64_t* out_bad) {
    if (out_bad) *out_bad = -1;
    VB_TRY(require_init());
    VB_TRY(check_recv_args("vb_binary_to_sparsevec_batch", n, bytes, off, cap, typmod, true));
    VB_REQUIRE(out_row_off, "vb_binary_to_sparsevec_batch: out_row_off is required");
    return recv_host(2, typmod, n, static_cast<const uint8_t*>(bytes), off, cap, out_row_off, nullptr, out_dim, out_idx,
                     out_val, out_bad);
}

int vb_rows_to_binary_batch_dev(int elem, int dim, const void* rows, int64_t n, int64_t cap, int64_t* out_off, void* out) {
    VB_TRY(require_init());
    VB_REQUIRE(elem == VB_VECTOR || elem == VB_HALFVEC, "vb_rows_to_binary_batch_dev: elem must be VB_VECTOR or VB_HALFVEC");
    VB_TRY(check_send_args("vb_rows_to_binary_batch_dev", dim, n, cap, out_off, rows != nullptr));
    VB_REQUIRE(dim <= 65535, "vb_rows_to_binary_batch_dev: dim %d does not fit the 16-bit header", dim);
    const int64_t total = n * (4 + (int64_t)dim * (elem == VB_VECTOR ? 4 : 2));
    const bool write = out && total <= cap;
    VB_TRY(send_dense_enqueue(elem, dim, rows, n, out_off, write ? out : nullptr));
    VB_REQUIRE(!out || total <= cap, "vb_rows_to_binary_batch_dev: the payloads are %lld bytes, more than cap = %lld",
               (long long)total, (long long)cap);
    return VB_OK;
}

int vb_rows_to_binary_batch(int elem, int dim, const void* rows, int64_t n, int64_t cap, int64_t* out_off, void* out) {
    VB_TRY(require_init());
    VB_REQUIRE(elem == VB_VECTOR || elem == VB_HALFVEC, "vb_rows_to_binary_batch: elem must be VB_VECTOR or VB_HALFVEC");
    VB_TRY(check_send_args("vb_rows_to_binary_batch", dim, n, cap, out_off, rows != nullptr));
    VB_REQUIRE(dim <= 65535, "vb_rows_to_binary_batch: dim %d does not fit the 16-bit header", dim);
    const int64_t esz = elem == VB_VECTOR ? 4 : 2, rb = 4 + (int64_t)dim * esz;
    for (int64_t i = 0; i <= n; ++i) out_off[i] = i * rb;
    if (!out || n == 0) return VB_OK;
    VB_REQUIRE(n * rb <= cap, "vb_rows_to_binary_batch: the payloads are %lld bytes, more than cap = %lld",
               (long long)(n * rb), (long long)cap);
    // chunks of at most kStageBytes of payload (or one row) through the two pinned slots: [rows] in, [payloads] out
    const int64_t per = std::max<int64_t>(1, kStageBytes / rb);
    const int64_t nch = (n + per - 1) / per;
    const int64_t max_nr = std::min(n, per);
    Staging& sg = staging();
    Scratch sc("type I/O");
    void *drows[2] = {}, *dout[2] = {}, *doff[2] = {};
    for (int k = 0; k < 2 && k < nch; ++k) {
        VB_TRY(pinned_grow(&sg.in[k], &sg.in_bytes[k], (size_t)(max_nr * dim * esz)));
        VB_TRY(pinned_grow(&sg.out[k], &sg.out_bytes[k], (size_t)(max_nr * rb)));
        VB_TRY(sc.own((size_t)(max_nr * dim * esz), &drows[k]));
        VB_TRY(sc.own((size_t)(max_nr * rb), &dout[k]));
        VB_TRY(sc.own(sizeof(int64_t) * (size_t)(max_nr + 1), &doff[k]));
    }
    cudaStream_t s = ctx().stream;
    auto enqueue = [&](int64_t c, int k) -> int {
        const int64_t r0 = c * per, nr = std::min(per, n - r0);
        std::memcpy(sg.in[k], static_cast<const uint8_t*>(rows) + r0 * dim * esz, (size_t)(nr * dim * esz));
        VB_CUDA(cudaMemcpyAsync(drows[k], sg.in[k], (size_t)(nr * dim * esz), cudaMemcpyHostToDevice, s));
        VB_TRY(send_dense_enqueue(elem, dim, drows[k], nr, static_cast<int64_t*>(doff[k]), dout[k]));
        VB_CUDA(cudaMemcpyAsync(sg.out[k], dout[k], (size_t)(nr * rb), cudaMemcpyDeviceToHost, s));
        return VB_OK;
    };
    auto finish = [&](int64_t c, int k) -> int {
        const int64_t r0 = c * per, nr = std::min(per, n - r0);
        std::memcpy(static_cast<uint8_t*>(out) + r0 * rb, sg.out[k], (size_t)(nr * rb));
        return VB_OK;
    };
    return pipeline_chunks(nch, enqueue, finish);
}

int vb_sparsevec_to_binary_batch_dev(int dim, int64_t n, const int64_t* row_off, const int32_t* idx, const float* val,
                                     int64_t cap, int64_t* out_off, void* out) {
    VB_TRY(require_init());
    VB_TRY(check_send_args("vb_sparsevec_to_binary_batch_dev", dim, n, cap, out_off, row_off != nullptr));
    if (n == 0) {
        VB_CUDA(cudaMemsetAsync(out_off, 0, sizeof(int64_t), ctx().stream));
        return VB_OK;
    }
    return send_sparse_dev(dim, n, row_off, idx, val, cap, out_off, out, "vb_sparsevec_to_binary_batch_dev");
}

int vb_sparsevec_to_binary_batch(int dim, int64_t n, const int64_t* row_off, const int32_t* idx, const float* val,
                                 int64_t cap, int64_t* out_off, void* out) {
    VB_TRY(require_init());
    VB_TRY(check_send_args("vb_sparsevec_to_binary_batch", dim, n, cap, out_off, row_off != nullptr));
    VB_REQUIRE(n == 0 || row_off[0] == 0, "vb_sparsevec_to_binary_batch: row_off must start at 0");
    out_off[0] = 0;
    if (n == 0) return VB_OK;
    const int64_t total = 12 * n + 8 * row_off[n];
    const bool write = out && total <= cap;
    // chunks of rows of at most kStageBytes of payload (or one row), one after another: each chunk's CSR check reads
    // back before its payloads are written
    std::vector<int64_t> cuts{0};
    while (cuts.back() < n) {
        const int64_t r0 = cuts.back();
        int64_t r1 = r0 + 1;
        while (r1 < n && 12 * (r1 + 1 - r0) + 8 * (row_off[r1 + 1] - row_off[r0]) <= kStageBytes) ++r1;
        cuts.push_back(r1);
    }
    cudaStream_t s = ctx().stream;
    for (size_t c = 0; c + 1 < cuts.size(); ++c) {
        const int64_t r0 = cuts[c], r1 = cuts[c + 1], nr = r1 - r0;
        const int64_t e0 = row_off[r0], ne = row_off[r1] - e0;
        VB_REQUIRE(ne >= 0, "sparsevec_send: offsets must not decrease");
        Scratch sc("type I/O");
        void *droff = nullptr, *didx = nullptr, *dval = nullptr, *doff = nullptr, *dout = nullptr;
        VB_TRY(sc.own(sizeof(int64_t) * (size_t)(nr + 1), &droff));
        VB_TRY(sc.own(sizeof(int32_t) * (size_t)ne, &didx));
        VB_TRY(sc.own(sizeof(float) * (size_t)ne, &dval));
        VB_TRY(sc.own(sizeof(int64_t) * (size_t)(nr + 1), &doff));
        VB_TRY(sc.own((size_t)(12 * nr + 8 * ne), &dout));
        std::vector<int64_t> ro((size_t)nr + 1);
        for (int64_t i = 0; i <= nr; ++i) ro[(size_t)i] = row_off[r0 + i] - e0;
        VB_CUDA(cudaMemcpyAsync(droff, ro.data(), sizeof(int64_t) * (size_t)(nr + 1), cudaMemcpyHostToDevice, s));
        if (ne) VB_CUDA(cudaMemcpyAsync(didx, idx + e0, sizeof(int32_t) * (size_t)ne, cudaMemcpyHostToDevice, s));
        if (ne && write) VB_CUDA(cudaMemcpyAsync(dval, val + e0, sizeof(float) * (size_t)ne, cudaMemcpyHostToDevice, s));
        VB_TRY(send_sparse_dev(dim, nr, static_cast<int64_t*>(droff), static_cast<int32_t*>(didx),
                               static_cast<float*>(dval), INT64_MAX, static_cast<int64_t*>(doff),
                               write ? dout : nullptr, "vb_sparsevec_to_binary_batch"));
        for (int64_t i = 1; i <= nr; ++i) out_off[r0 + i] = 12 * (r0 + i) + 8 * row_off[r0 + i];
        if (write) {
            void* pin;
            VB_TRY(pinned_buffer2((size_t)(12 * nr + 8 * ne) + 16, &pin));
            VB_CUDA(cudaMemcpyAsync(pin, dout, (size_t)(12 * nr + 8 * ne), cudaMemcpyDeviceToHost, s));
            VB_CUDA(cudaStreamSynchronize(s));
            std::memcpy(static_cast<uint8_t*>(out) + out_off[r0], pin, (size_t)(12 * nr + 8 * ne));
        }
    }
    VB_REQUIRE(!out || total <= cap, "vb_sparsevec_to_binary_batch: the payloads are %lld bytes, more than cap = %lld",
               (long long)total, (long long)cap);
    return VB_OK;
}

}  // extern "C"
