// vb_common.cuh -- shared declarations for libvecb200 (sm_90a only).
#pragma once

#include <cuda_runtime.h>
#include <cuda_fp16.h>
#include <stdint.h>
#include <stddef.h>
#include <string>
#include <vector>

#include "../../include/vecb200.h"

namespace vb {

// ---------------------------------------------------------------- errors
void set_error(const char* fmt, ...);
extern thread_local int g_last_status;

#define VB_CUDA(call)                                                                    \
    do {                                                                                 \
        cudaError_t e__ = (call);                                                        \
        if (e__ != cudaSuccess) {                                                        \
            vb::set_error("%s failed: %s (%s:%d)", #call, cudaGetErrorString(e__), __FILE__, __LINE__); \
            return VB_ECUDA;                                                             \
        }                                                                                \
    } while (0)

#define VB_TRY(expr)               \
    do {                           \
        int rc__ = (expr);         \
        if (rc__ != VB_OK) return rc__; \
    } while (0)

#define VB_REQUIRE(cond, ...)        \
    do {                             \
        if (!(cond)) {               \
            vb::set_error(__VA_ARGS__); \
            return VB_EINVAL;        \
        }                            \
    } while (0)

// ---------------------------------------------------------------- context
struct Scratch;
struct Context {
    bool inited = false;
    int device = -1;
    int sm_count = 132;
    cudaStream_t stream = nullptr;
    cudaStream_t copy_stream = nullptr;
    int64_t launches = 0;
    int slab_select = 1;               // selection from the filter's slab minima (0: full radix selection of every run)
    int tc_level1 = 1;                 // batched list scan: try the hi-plane-only filter first (vb_set_option "tc_level1")
    int tc_level0 = 1;                 // ... and in front of it the int8 filter, where tc_level1 is on (vb_set_option "tc_level0")
    int tc_levelp = 1;                 // ... and in front of that the projection lower bound, where tc_level0 is on (vb_set_option "tc_levelp")
    int pp_filter = 1;                 // k-means++ on large fp32 sample tables: triangle-inequality + bf16 filters in front of the exact distances
    unsigned long long pp_stats[3] = {0, 0, 0};   // last seeding: samples skipped by the triangle rule / stopped by the bf16 bound / re-scored exactly
    int one_query = 1;                 // scans of at most 16 queries: two fused distance + select kernels (vb_ivf_one.cu); 0 = the general path
    int scan_impl = 2;                 // 0 = LDG variant (vb_scan.cu), 1 = bulk-copy / TMA variant (vb_scan_bulk.cu), 2 = by table size
    int hnsw_build_fraction = 64;      // HNSW build: a batch is at most 1/fraction of the elements already inserted
    int hnsw_build_batch = 16384;      // ... and at most this many elements
    int hnsw_l2_persist = 1;           // HNSW scans: keep the visited tables in the persisting part of L2
    int64_t last_assign_flagged = -1;  // rows re-checked by the exact kernel in the last tensor-core assign (-1: exact path)
    // the grow-only scratch arena (Scratch)
    uint8_t* arena = nullptr;
    size_t arena_bytes = 0;
    size_t arena_peak = 0;             // the most of it any call has needed
    Scratch* scratch = nullptr;        // the innermost live Scratch
    // pinned staging
    void* pinned = nullptr;
    size_t pinned_bytes = 0;
    void* pinned2 = nullptr;
    size_t pinned2_bytes = 0;
};
Context& ctx();
int require_init();

// Device scratch of one library call.  Scratch objects nest like the calls that own them: take() hands out a
// 256-byte-aligned range of the library's grow-only arena above everything the enclosing calls hold; own() a
// one-off allocation for build-sized temporaries the library must not keep.  Both are released with the Scratch.
// A function whose device pointers outlive its return takes its caller's Scratch; every other one opens its own.
// Only the innermost live Scratch may take (anything else is refused with VB_ESTATE).  A range that does not fit the
// arena is a one-off allocation, and the arena grows to the call's peak when the outermost Scratch closes, so a
// repeated call allocates nothing.  fn (optional) names the call in the allocation errors.
struct Scratch {
    explicit Scratch(const char* fn = nullptr);
    ~Scratch();
    Scratch(const Scratch&) = delete;
    Scratch& operator=(const Scratch&) = delete;
    int take(size_t bytes, void** out);
    int own(size_t bytes, void** out);

  private:
    const char* fn_;
    Scratch* outer_;
    size_t top_;                 // arena offset of the next range (past the arena's end: one-off allocations)
    std::vector<void*> owned_;
};
int pinned_buffer(size_t bytes, void** out);
int pinned_buffer2(size_t bytes, void** out);

inline void count_launch(int n = 1) { ctx().launches += n; }

// optional event brackets around a kernel class (vb_prof_enable)
void prof_begin(int which);
void prof_end(int which);
struct ProfScope {   // a bracket that is closed on every exit of its scope
    int which;
    explicit ProfScope(int w) : which(w) { prof_begin(w); }
    ~ProfScope() { prof_end(which); }
};

// ---------------------------------------------------------------- communicator (vb_comm.cu)
// world size / rank of the library's NCCL communicator (1 / 0 when none was created)
int comm_world();
int comm_rank();
// in-place sum over the ranks on the library stream; dtype 0 = fp32, 1 = int32, 2 = int64, 3 = fp64, 4 = uint32
int comm_allreduce(void* buf_dev, int64_t count, int dtype);
// recv[r * bytes .. ) = rank r's send buffer, on the library stream (a plain copy when there is one rank)
int comm_allgather(const void* send_dev, void* recv_dev, int64_t bytes_per_rank);

// ---------------------------------------------------------------- layout
inline size_t raw_row_bytes(int elem, int dim) {
    return elem == VB_VECTOR ? (size_t)dim * 4 : elem == VB_HALFVEC ? (size_t)dim * 2 : ((size_t)dim + 7) / 8;
}
// device rows are padded to 16-byte multiples so every row starts 128-bit aligned
inline size_t padded_row_bytes(int elem, int dim) { return (raw_row_bytes(elem, dim) + 15) & ~(size_t)15; }
// The LDG scan (vb_scan.cu) holds one query's image -- the padded row, halfvec widened to fp32 -- in shared memory, and
// an sm_90 CTA can opt into at most 227 KiB of it: wider rows (vector or halfvec past 58112 dimensions, bit past
// 1859584 bits) cannot be scanned, so tables and distance batches of them are refused before anything runs.
constexpr size_t SCAN_QUERY_SMEM_MAX = 227 * 1024;
inline size_t query_image_bytes(int elem, int dim) {
    return elem == VB_HALFVEC ? 2 * padded_row_bytes(elem, dim) : padded_row_bytes(elem, dim);
}
inline int require_scannable_rows(int elem, int dim) {
    VB_REQUIRE(query_image_bytes(elem, dim) <= SCAN_QUERY_SMEM_MAX,
               "rows of %d %s take a %zu-byte query image; the scan holds it in shared memory, at most %zu bytes (227 KiB)",
               dim, elem == VB_BIT ? "bits" : "dimensions", query_image_bytes(elem, dim), SCAN_QUERY_SMEM_MAX);
    return VB_OK;
}

inline bool metric_valid_for(int elem, int metric) {
    if (elem == VB_BIT) return metric == VB_HAMMING || metric == VB_JACCARD;
    return metric == VB_L2_SQUARED || metric == VB_NEG_IP || metric == VB_COSINE || metric == VB_L1 ||
           metric == VB_L2 || metric == VB_IP || metric == VB_SPHERICAL;
}
// the metric the kernels order by ("key metric"); the float8 the operator returns is derived from it
inline int key_metric(int metric) {
    switch (metric) {
        case VB_L2: return VB_L2_SQUARED;
        case VB_IP:
        case VB_SPHERICAL: return VB_NEG_IP;
        default: return metric;
    }
}

// A resident row table: n rows, padded stride.
struct Table {
    int elem = 0, dim = 0;
    size_t stride = 0;      // padded row bytes
    int64_t n = 0, cap = 0;
    uint8_t* d = nullptr;   // device
};
int table_reserve(Table& t, int64_t rows);
int table_append_host(Table& t, const void* rows, int64_t n);
int table_append_dev(Table& t, const void* rows_dev, int64_t n);
void table_free(Table& t);

// Float4ToHalf (src/halfutils.h:244-261): round to nearest even; *overflow = a finite value became infinite, which the
// reference refuses (vector_to_halfvec, sparsevec_to_halfvec)
__device__ __forceinline__ __half float_to_half_checked(float x, bool* overflow) {
    const __half h = __float2half_rn(x);
    *overflow = __hisinf(h) != 0 && !isinf(x);
    return h;
}
// Float4ToHalf's error for value v: sets "\"<v>\" is out of range for type halfvec" (v in PostgreSQL's float4 output
// style) and returns VB_EINVAL (vb_ops.cu)
int half_range_error(float v);

// Pad + (for halfvec) widen queries into the fp32 query image the kernels read.
// vector/halfvec: float[nq][qstride/4]; bit: bytes[nq][qstride]. host==true: `queries` is host memory.
int upload_queries(Scratch& sc, int elem, int dim, const void* queries, int64_t nq, bool host, void** out_dev, size_t* qstride);

// ---------------------------------------------------------------- scan primitives (vb_scan.cu)
struct Chunk {           // one unit of scan work: a run of rows against one query
    int64_t row_begin;   // row index into the table
    int64_t out_off;     // where distance[0] of this run goes in the output array
    int32_t n_rows;
    int32_t q;           // query index
};

// distances of regular work: every query against rows [0, n) ; out[q * out_stride + r]
int launch_scan_regular(const Table& t, int key_metric, const void* q_dev, size_t qstride, int64_t nq,
                        int64_t n_rows, float* out, int64_t out_stride);
// distances of chunk-list work; n_chunks_dev holds the chunk count (device int32).  ldg_only: always the LDG kernel
// (scan_kernel), whose per-row arithmetic the scans of one query share, never the bulk-copy one
int launch_scan_chunks(const Table& t, int key_metric, const void* q_dev, size_t qstride,
                       const Chunk* chunks_dev, const int* n_chunks_dev, int max_chunks, float* out, bool ldg_only = false);
// distances of chunk-list work over gathered rows: row r of a chunk is table row ids_dev[row_begin + r] (LDG kernel)
int launch_scan_gather(const Table& t, int key_metric, const void* q_dev, size_t qstride, const int64_t* ids_dev,
                       const Chunk* chunks_dev, const int* n_chunks_dev, int max_chunks, float* out);
// Jaccard needs the exact float8: out as double
int launch_scan_regular_f64(const Table& t, int key_metric, const void* q_dev, size_t qstride, int64_t nq,
                            int64_t n_rows, double* out, int64_t out_stride);

// per segment top-k of float keys with position tie-break, ascending (vb_scan.cu).
// seg_begin/seg_len: device arrays (offset into keys, length).  Host copies are only needed for
// k > 2048 (full segmented sort path).  Writes out_pos[nseg*k] (position within segment, -1 pad)
// and out_key[nseg*k].
int launch_segment_topk_v(const float* keys, const int64_t* seg_begin_dev, const int32_t* seg_len_dev,
                          const int64_t* seg_begin_host, const int32_t* seg_len_host, int64_t nseg, int k,
                          int32_t* out_pos, float* out_key);
int scan_chunk_rows(const Table& t);
// the k smallest keys of every segment strictly above floor_key[seg] (once returned[seg] > 0), ascending; then
// floor_key / returned advance past the page and count[seg] = its size.  k <= 2048 (the paged scan of vb_ivf_iter.cu)
int launch_segment_topk_floor(const float* keys, const int64_t* seg_begin_dev, const int32_t* seg_len_dev, int64_t nseg, int k,
                              uint64_t* floor_key, int32_t* returned, int32_t* count, int32_t* out_pos, float* out_key);

// exact fp32 nearest-centre assign (vb_kmeans.cu) and the default assign entry (tensor cores + exact re-check)
int launch_assign_exact(const Table& X, int metric, const Table& Cn, int k, const int32_t* row_sel_dev, int64_t n_sel,
                        int32_t* out_idx, float* out_val);
int launch_assign(const Table& X, int metric, const Table& Cn, int k, int32_t* out_idx);
// all-pairs fp32 distances X x Cn -> out[x * ld + c] (register-tiled CUDA-core kernel, vb_kmeans.cu)
int launch_distance_matrix(const Table& X, int metric, const Table& Cn, int k, float* out, int64_t ld);
void set_tc_enabled(bool on);
// the seeding and Lloyd code behind vb_kmeans_pp_init[_draws] and vb_kmeans (vb_kmeans.cu), for vb_ivf_build
int kmeans_pp(const Table& X, int kmeans_metric, void* centers_host, int k, uint64_t seed, int64_t first_row = -1,
              const double* u_in = nullptr, int64_t* picked_out = nullptr);
int kmeans_run(const Table& X, int kmeans_metric, void* centers_host, int k, int max_iter, uint64_t seed, vb_allreduce_fn allreduce,
               void* actx, int* iters_out);

// ---------------------------------------------------------------- IVFFlat build (vb_ivf_build.cu)
// ns distinct rows of [0, n) drawn from the seed, ascending (device, [ns])
int build_draw_samples(int64_t n, int64_t ns, uint64_t seed, int64_t* rows_out);
// The placement pass: work item j reads source row s = src_idx ? src_idx[j] : j (packed rows, `pitch` bytes apart) and
// writes table row d = dst_idx ? dst_idx[j] : j (d < 0: skipped) at the padded stride, pad bytes zero, with its id
// (src_ids ? src_ids[s] : s) to out_ids[d] when out_ids is given.  normalize (vector / halfvec): the row is stored
// l2-normalised, and zero (optional, [m]) receives 1 where the norm is not > 0, else 0; out == nullptr computes only zero.
int launch_place_rows(int elem, int dim, bool normalize, const void* src, size_t pitch, const int64_t* src_ids, const int64_t* src_idx,
                      const int64_t* dst_idx, int64_t m, uint8_t* out, size_t out_stride, int64_t* out_ids, int32_t* zero);
// lists[i] = -1 where zero[i]
int build_mark_skipped(const int32_t* zero, int64_t m, int32_t* lists);
// keep-order compaction map of the rows with zero[i] == 0: dst[i] = position among them, or -1; *kept = their number
int build_compact_map(const int32_t* zero, int64_t m, int64_t* dst, int64_t* kept);
// From the list numbers (-1 = not indexed) of n rows: order[p] = the row stored at image row p (lists ascending, call
// order inside a list; the rows that are not indexed follow), dst[i] = image row of row i or -1, list_off [lists + 1]
// (host).  order and dst are device arrays of n.
int build_destinations(const int32_t* lists_of_row, int64_t n, int lists, int64_t* order, int64_t* dst, int64_t* list_off_host);

// list-major batched list scan (vb_list_tile.cu): the (query, probe) pairs of a batch grouped by list, one CTA
// per static row tile of the index against every query probing that list
struct ListTile {
    int64_t row_begin;   // first row of the tile in the list-ordered table
    int32_t list;
    int32_t n_rows;      // <= list_tile_rows()
};
// (query, probe) pairs of a batch grouped by list: slots [begin[l], begin[l] + cnt[l]) belong to list l
struct QueryGroups {
    int32_t* cnt;        // [lists]
    int32_t* begin;      // [lists]
    int32_t* gt_begin;   // [lists] first query tile of each list (only when built with gt_rows > 0)
    int32_t* pair_q;     // [pairs] query number
    int32_t* pair_list;  // [pairs] list number
    int64_t* pair_out;   // [pairs] offset of the pair's candidate run in the distance buffer
    int32_t* pair_sbase; // [pairs] first entry of the pair's run in the slab-minimum array (slab_base(), cap_s > 0 only)
    int64_t n_pairs;
};
// Slab minima of the tensor-core filter: a slab = 32 table-aligned rows of one (query, probe) pair's list; the filter's
// epilogue stores min d~ over the slab next to the dense d~ array, and the selection reads only the slabs that can hold
// one of the k' nearest.  Layout: query q owns cap_s = cap / 32 + 2 probes + 2 entries; probe p's run starts at
// q cap_s + cand_off[q][p] / 32 + 2 p (a list of len rows spans at most len / 32 + 2 slabs, so runs never overlap) and
// slab (r >> 5) - (list_off[l] >> 5) of the list is entry number that of the run.
__host__ __device__ inline int64_t slab_cap(int64_t cap, int probes) { return (cap >> 5) + 2 * (int64_t)probes + 2; }
__host__ __device__ inline int64_t slab_base(int64_t q, int64_t cap_s, int32_t cand_off, int p) {
    return q * cap_s + (cand_off >> 5) + 2 * p;
}
int build_query_groups(Scratch& sc, const int32_t* d_lists, int64_t nq, int probes, const int32_t* cand_off, int64_t cap, int n_lists, int gt_rows,
                       QueryGroups* g, int64_t cap_s = 0);
// tensor-core filter of the batched list scan (vb_list_tc.cu)
struct ListUnit {
    int32_t list;
    int32_t tile;        // 128-row tile of the list-ordered table that intersects the list
};
struct ListTcImage {
    uint8_t* planes = nullptr;   // bf16 hi/lo planes of the whole table, swizzled smem image per (tile, 64-dim block)
    float* xn = nullptr;         // |row|^2
    ListUnit* units = nullptr;
    int n_units = 0;
    int n_kblocks = 0;
    int64_t n_tiles = 0;
    float xmax = 0.f;            // max |row|
    bool finite = true;          // false when a row norm is Inf / NaN (no error bound -> exact path only)
    // level 0 (int8 rows), built on first use where it fits: [tile][128-dim block][128 rows x 128 B], same swizzle
    uint8_t* planes8 = nullptr;
    float* xs = nullptr;         // per-row scale s_x = max |x_i| / 127 (x ~ s_x * x8)
    float* r8 = nullptr;         // per-row residual |x - s_x x8|, rounded up (0 on padding rows): the refine's per-row bound
    int n_kblocks8 = 0;
    float rmax = 0.f;            // max over rows of |x - s_x x8|, rounded up
    bool l0_tried = false;       // the int8 plane was built or found not to fit
};
bool list_tc_supported(int elem, int key_metric, int k);
// The per-query inputs of the filter's and the refine's error bounds for one batch of query images, owned by the batch so
// that its probe selection and list scan compute |q|^2 once: *qn = a range of sc holding |q|^2 of the batch, with room for
// what launch_list_tc adds at level 0 (t_q, eps(q)^2, per-row bound coefficients)
int list_tc_query_norms(Scratch& sc, const void* qimg, size_t qstride, int64_t nq, float** qn);
int list_tc_kp(int k, int level = 2);
// dynamic shared memory of a launch_list_tc_cta_refine launch that selects its k' nearest from the slab minima (slabs), takes
// them preselected (pre) or selects them from the whole run (neither)
size_t cta_refine_smem_bytes(int kp, size_t qstride, bool slabs, bool pre, int64_t cap, int64_t cap_s, int probes);
int list_tc_prepare(const Table& rows, ListTcImage* im);
// the int8 plane, row scales and rmax of level 0 (rows must already be prepared)
int list_tc_prepare_l0(const Table& rows, ListTcImage* im);
void list_tc_release(ListTcImage* im);
// In-place changes of the table (vb_ivf_insert / vb_ivf_delete).  list_tc_reserve, before the rows move: plane buffers
// (built ones only) that hold fewer than nt tiles are freed and allocated again with half again as many; *whole / *whole8
// say the bf16 / int8 plane must then be packed from tile 0.  When an allocation fails the image is released (the next
// batched scan rebuilds it, if it fits) and false is returned.  cap_tiles / cap_tiles8: the tiles the buffers hold.
bool list_tc_reserve(ListTcImage* im, int64_t nt, int64_t* cap_tiles, int64_t* cap_tiles8, bool* whole, bool* whole8);
// list_tc_repack, after: the planes, |x|^2 and (if built) the int8 plane, s_x and R_x re-packed from the given tiles on,
// n_tiles set, and xmax / finite / rmax recomputed over the whole table as list_tc_prepare(_l0) compute them (d_stats:
// 4 device words of scratch)
int list_tc_repack(const Table& rows, ListTcImage* im, int64_t first_tile, int64_t first_tile8, unsigned* d_stats);
int launch_list_tc(const Table& rows, const ListTcImage& im, int key_metric, const void* qimg, size_t qstride, int64_t nq,
                   const int32_t* d_lists, int probes, const int32_t* cand_off, int64_t cap, const int64_t* d_list_off, int n_lists,
                   float* out, float* qn, bool one_list_all_queries = false, int level = 2, float* smin = nullptr,
                   int64_t cap_s = 0);
// Level P of the batched list scan (vb_list_proj.cu): a projection lower bound |x - q|^2 >= |P(x - q)|^2 / sigma^2 with the
// top principal directions of the rows as P, in front of level 0.  Its runs hold rigorous lower bounds of the fp32 distance
// and go through level 0's listing refine with zero per-row terms.
constexpr int LIST_LEVEL_P = 3;
struct ListProj {
    float* P = nullptr;          // [r][dim] fp32 basis
    float* y = nullptr;          // [cap_rows][r] fp32 projections of the rows, list order
    int r = 0;                   // 0: no level P (not built, or no r <= dim / 8 holds 90 % of the sample's energy)
    int64_t cap_rows = 0;
    double sigma2 = 0.0;         // >= ||P||_2^2
    float c1 = 0.f, c2 = 0.f, ce = 0.f;   // the bound's constants (lp_scan_kernel)
    bool tried = false;          // the basis was built or found not to apply
};
// the basis and the projected plane, once per image (fp32 rows only; lp->r stays 0 where no basis applies)
int list_proj_prepare(const Table& rows, int n_lists, ListProj* lp);
void list_proj_release(ListProj* lp);
// after an in-place change: the projections re-computed from first_row on (the basis stays), the plane grown when needed
int list_proj_update(const Table& rows, ListProj* lp, int64_t first_row);
// the filter pass: the queries projected, then one pass over the (list, table tile) units of im (im.units) writes the lower
// bounds of the fp32 distance from fl(|y_x - y_q|^2) into the runs and takes the slab minima (smin, required).
// qn: |q|^2 of the batch; im.xmax: max |x| over the rows.
int launch_list_proj(Scratch& sc, const Table& rows, const ListProj& lp, const ListTcImage& im, const void* qimg, size_t qstride, int64_t nq,
                     const int32_t* d_lists, int probes, const int32_t* cand_off, int64_t cap, const int64_t* d_list_off, int n_lists,
                     float* out, const float* qn, float* smin, int64_t cap_s);
// the k' nearest of every query's candidate run from the slab minima (same output as launch_segment_topk_v)
int launch_slab_select(const float* dist, const float* smin, int64_t nq, int probes, const int32_t* probe_lists, const int32_t* cand_off,
                       const int64_t* list_off, int64_t cap, int64_t cap_s, const int64_t* seg_begin, const int32_t* seg_len, int kp,
                       int32_t* out_pos, float* out_key);
// traffic accounting of list_tc_kernel launches (profiling): enable / read-and-reset 8 counters (lists: 0-3, centres: 4-7)
int list_tc_traffic(int on, int64_t* out8);
// read-and-reset the level-0 refine's counters, kept while traffic accounting is on: rows re-scored, rows under the
// global-bound threshold (d~ <= d~_k + 2 eps(q)), queries refined
int list_tc_level0_rescored(int64_t* out3);
// the exact re-score of the k' nearest of every query's candidate run, their final order and the certificate, with one CTA
// per query.  The k' are selected in the kernel from the slab minima (smin), taken as selected (pre_pos / pre_key
// [nq][kp], sorted, -1 padded: launch_slab_select / launch_segment_topk_v), or else selected in the kernel from the whole
// run dist[q * cap ..) of seg_len[q] <= CR_RUN_MAX entries.  The number of uncertified queries is ADDED to *fail_dev
// (level 0: and they are listed in fail_list).  qn: the batch's bound inputs the filter used (list_tc_query_norms).
constexpr int CR_RUN_MAX = 4096;
// has_nan (vb_ivf_search_filtered): the runs were masked (FILTER_REJECTED marks rejected entries): marked candidates are
// not candidates, and a query with an allowed NaN d~ (has_nan[q]) counts as uncertified.
int launch_list_tc_cta_refine(const Table& rows, const ListTcImage& im, int key_metric, const void* qimg, size_t qstride, int64_t nq,
                              int k, int kp, int probes, const int32_t* d_lists, const int32_t* cand_off, const int64_t* d_list_off,
                              const float* dist, const float* smin, const int32_t* pre_pos, const float* pre_key, int64_t cap,
                              int64_t cap_s, const int32_t* seg_len, const float* qn, int32_t* out_pos, float* out_key, int* fail_dev,
                              int level = 2, int32_t* fail_list = nullptr, const int32_t* has_nan = nullptr);
// vb_ivf_one.cu: the scan of one query (or a handful) as two fused distance + select kernels
bool one_probe_fits(int lists, size_t qstride, int probes);
bool one_scan_fits(int64_t cap, size_t qstride, int probes, int64_t k);
int launch_one_probe(const Table& centres, int key_metric, const void* qimg, size_t qstride, int64_t nq, int probes, float* cdist,
                     unsigned* ticket, int32_t* out_lists, float* out_ldist, int64_t* zero_me);
int launch_one_scan(const Table& rows, int key_metric, int metric, const int64_t* list_off, const int64_t* ids,
                    const int32_t* probe_lists, int probes, const void* qimg, size_t qstride, int64_t nq, int k, int64_t cap,
                    float* dist, unsigned* ticket, int64_t* out_ids, float* out_f, double* out_d, int32_t* out_total,
                    int64_t* cand_sum, bool cand_store);
constexpr int ONE_MAX_Q = 16;   // queries per call the fused path takes
// vb_ivf_iter.cu: a query of an iterative scan whose group of lists is used up moves to its next non-empty group
int launch_ivf_iter_advance(int64_t nq, int probes, int max_probes, const int32_t* probe_lists, const int64_t* list_off,
                            int32_t* glists, int32_t* list_index, int32_t* returned, int32_t* seg_len, int32_t* active);
// a filtered iterative scan: probe_lists[q][j] = l becomes the virtual list fq[q] * lists + l (-1 stays -1), so that the
// advance, chunk and finish kernels read list l of the query's row filter from the handle's concatenated offset table
int launch_ivf_filter_lists(int64_t nq, int max_probes, int lists, const int32_t* fq_dev, int32_t* probe_lists);

// ---------------------------------------------------------------- row filters (vb_filter.cu)
// The allowed rows of one table or one IVFFlat image, ascending.  An IVFFlat image stores rows grouped by list, so the
// allowed rows of list l are one run pos[off[l] .. off[l + 1]).  The allowed elements of an HNSW image are a bitset:
// its iterative scan tests the elements a traversal returns, it never enumerates the allowed ones.
// process-wide unique stamp of a table, sparse table, IVFFlat or HNSW image: a filter matches its owner by address and
// stamp, so a filter that outlived its owner is refused even when a new owner is allocated at the same address
uint64_t next_owner_uid();
// Orders (vb_order.cu) read their table at every bounds call: owner_watch(uid) at an order's creation, owner_released(uid)
// when a table is freed, so that an order of a freed table is refused.
void owner_watch(uint64_t uid);
void owner_released(uint64_t uid);
enum FilterKind { FILTER_TABLE, FILTER_IVF, FILTER_HNSW, FILTER_SPARSE };
struct Filter {
    const void* owner = nullptr;   // the vb_table, vb_sparse_table, vb_ivf or vb_hnsw it was made for
    uint64_t owner_uid = 0;        // and that owner's stamp
    FilterKind kind = FILTER_TABLE;
    uint64_t generation = 0;       // IVFFlat / HNSW: the image's generation at creation
    int64_t n = 0;                 // rows allowed
    int lists = 0;
    void* mem = nullptr;           // one allocation: pos | ids | off (HNSW: bits)
    int64_t* pos = nullptr;        // [n] table: row numbers; IVFFlat: rows of the list-ordered image
    int64_t* ids = nullptr;        // [n] IVFFlat: the heap ids of pos
    int64_t* off = nullptr;        // [lists + 1] IVFFlat: per-list runs of pos
    std::vector<int64_t> h_off;    // host copy of off (allowed counts per list: sizes a scan handle's group buffers)
    uint32_t* bits = nullptr;      // HNSW: [words] bit e = element e is allowed
    int64_t words = 0;
};
// table: rows = row numbers (values outside [0, n_rows) ignored; the host variant validates before this call)
int filter_build_table(int64_t n_rows, const int64_t* rows, int64_t n, bool host, Filter* f);
// A filter of row numbers of a table of n_rows rows (owner, its stamp, kind FILTER_TABLE or FILTER_SPARSE): the body of
// vb_table_filter_create[_dev] and vb_sparse_table_filter_create.  fn names the entry point in the messages; owner ==
// nullptr fails ("null table").  The host variant validates every row first.
int table_filter_create(const char* fn, const void* owner, uint64_t owner_uid, int64_t n_rows, FilterKind kind, const int64_t* rows,
                        int64_t n, bool host, vb_filter** out);
// IVFFlat image of n_rows rows: image_ids = heap ids of the rows (nullptr: row positions), list_off [lists + 1] device
int filter_build_ivf(int64_t n_rows, const int64_t* image_ids, const int64_t* list_off, int lists, const int64_t* ids, int64_t n,
                     bool host, Filter* f);
// HNSW image of n_elems elements: elems = element numbers (values outside [0, n_elems) ignored; the host variant
// validates before this call)
int filter_build_hnsw(int64_t n_elems, const int64_t* elems, int64_t n, bool host, Filter* f);
void filter_release(Filter* f);
// The batched filtered IVFFlat search (vb_ivf_search_filtered) masks each query's run of candidate distances: a rejected
// entry holds these bits, a negative NaN.  orderable_key() sorts every NaN after +inf, so a rejected entry is never
// selected ahead of an allowed one; the bits tell it apart from an allowed row's NaN distance (the GPU computes NaN as
// 0x7FFFFFFF, and the mask rewrites an allowed NaN that carries these bits to that).
constexpr uint32_t FILTER_REJECTED = 0xFFFFFFFFu;

// The work lists of a filtered exact top-k (vb_exact_topk_filtered, vb_sparse_exact_topk_filtered).  Per sub-batch of
// queries: per-query arguments, the chunks of each query's allowed rows (Chunk::row_begin indexes the call's concatenated
// position arrays, one copy per filter; Chunk::out_off its distance run), and the scan launches over them.
struct FilterQuery {
    int64_t run;     // first distance of the query's run (segment begin)
    int64_t base;    // first position of its filter in the concatenated position array
    int64_t cbase;   // its first chunk: the chunks of the queries that share a filter are one block, filters in order
    int32_t len;     // rows its filter allows
    int32_t pad;
};
struct FilterBatch {
    std::vector<FilterQuery> qa;          // queries q0 .. q0 + qa.size() of the call
    std::vector<int64_t> launch_begin;    // scan launch l covers chunks [launch_begin[l], launch_begin[l] + launch_count[l])
    std::vector<int32_t> launch_count;
    int64_t run = 0;                      // distances of the sub-batch
    int64_t max_chunks = 0;
};
// The positions of the filters side by side: fbase [nfilters + 1] (host), *rows = the device array (a single filter is
// read in place, several are copied into a range of sc)
int filter_concat_positions(Scratch& sc, const vb_filter* const* filters, int nfilters, std::vector<int64_t>* fbase, const int64_t** rows);
// The next sub-batch from query q0 on: as many queries as keep its distances under ~1 GiB (at least one), at most max_q.
// A filter's queries get one block of chunks; each block gets a scan launch of its own once it fills grid_chunks chunks
// (the whole grid then reads one filter's rows, which stay in L2 for its other queries), smaller blocks share one.
int filter_batch_plan(const vb_filter* const* filters, int nfilters, const int32_t* filter_of_query, const int64_t* fbase, int64_t q0,
                      int64_t nq, int64_t max_q, int rows_per_chunk, int64_t grid_chunks, FilterBatch* b);
// filter_chunks_kernel: seg_begin / seg_len / chunks of the sub-batch's nq queries (qa_dev = FilterBatch::qa on the device)
int launch_filter_chunks(const FilterQuery* qa_dev, int64_t nq, int rows_per_chunk, int64_t* seg_begin, int32_t* seg_len, Chunk* chunks);
// rerank_prepare_kernel (vb_rerank.cu): ids[q c + j], j < seg_len[q] = the candidates of query q in [0, n), in candidate
// order; seg_begin[q] = q c; the chunks of each query's run (row_begin = out_off into ids / distances) appended at
// *n_chunks (device, zeroed by the caller)
int launch_rerank_prepare(const int64_t* cand, int64_t nq, int c, int64_t n, int rows_per_chunk, int64_t* ids, int64_t* seg_begin,
                          int32_t* seg_len, Chunk* chunks, int* n_chunks);

// ---------------------------------------------------------------- sparse CSR for the orders (vb_sparse.cu)
struct SparseCsr {
    int dim;
    int64_t n;
    const int64_t* off;   // [n + 1] device
    const int32_t* idx;
    const float* val;
};
// the resident rows of a sparse table as they are now (its buffers move when it grows), and its stamp
SparseCsr sparse_table_csr(const vb_sparse_table* h);
uint64_t sparse_table_uid(const vb_sparse_table* h);
// nq >= 1 sparse queries of a call on a table of dimension dim, checked with the sparse calls' rules and texts (CheckDims,
// then the CSR: host variant on the host, device CSR by the one checked read-back) and on the device: host CSR uploaded
// to a range of sc, device CSR used in place
int sparse_queries_on_device(Scratch& sc, int dim, int q_dim, int64_t nq, const int64_t* q_off, const int32_t* q_idx, const float* q_val, bool host,
                             SparseCsr* out);

int list_tile_rows();
bool list_major_supported(int elem, int key_metric);
int launch_list_major(const Table& rows, int key_metric, const void* qimg, size_t qstride, int64_t nq, const int32_t* d_lists,
                      int probes, const int32_t* cand_off, int64_t cap, const int64_t* d_list_off, int n_lists,
                      const ListTile* d_tiles, int n_tiles, float* out);

}  // namespace vb

// opaque handle types of the C ABI
struct vb_table {
    vb::Table t;
    uint64_t uid = vb::next_owner_uid();
};
struct vb_filter {
    vb::Filter f;
};
