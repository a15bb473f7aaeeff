/*
 * vecb200.h -- C ABI of libvecb200.so: the H100 (sm_90a) implementation of
 * pgvector's batched-distance hot path.
 *
 * This is the drop-in boundary (SURVEY.md section 8b).  Every entry point takes plain
 * pointers and sizes; there are no PostgreSQL, C++ or torch types in any
 * signature.  Each function names the reference code whose inner loop it
 * replaces (paths relative to the pgvector tree @ e48241b).  The extension-side
 * glue that calls these from the index AM is in pgvector_b200/ext/ and
 * INTEGRATION.md.
 *
 * Conventions
 *   - every function returns 0 (VB_OK) or a negative VB_E* code; the message is
 *     available from vb_last_error() (thread local).  The caller (a Postgres
 *     backend) turns it into ereport(ERROR) AFTER the call returns, so no device
 *     state is held across a longjmp.
 *   - there is NO CPU fallback: every call fails with VB_ENODEVICE when no
 *     sm_90 device is usable.
 *   - "host" pointers are ordinary process memory; "_dev" variants take device
 *     pointers valid on the library's current device.  Work is enqueued on the
 *     library stream (vb_stream()); host-buffer variants synchronise before
 *     returning.  _dev variants return with their work enqueued, with these stated
 *     exceptions: the batched vb_ivf_search*_dev read ONE 8-byte pair of certificate
 *     counters per sub-batch of queries, with up to 64 numbers of the queries filter
 *     level 0 could not certify (the tensor-core filter re-runs uncertified queries
 *     before the results may be used; a re-run synchronises again),
 *     vb_hnsw_search_dev reads one overflow flag per call (visited-table growth),
 *     vb_table_aggregate_dev reads sum's 4-byte overflow flag (float_overflow_error), and
 *     the sparsevec _dev calls read the result of their device CSR check: one copy of at
 *     most 24 bytes (first defect, largest row nnz, total nnz) before any other work
 *     (the casts: one copy of at most 32 bytes, see vb_dense_to_sparsevec_batch),
 *     vb_l2_normalize_batch_dev reads its 4-byte overflow flag (float_overflow_error), and
 *     vb_vector_to_halfvec_batch_dev reads the 8-byte index of the first value that does
 *     not fit, plus that 4-byte value only when there is one (for the error text), and
 *     vb_sparse_order_bounds_dev reads the result of its device CSR check like the other
 *     sparsevec _dev calls, and vb_arith_batch_dev and vb_array_to_rows_batch_dev read the
 *     8-byte key of the first value that fails the reference's checks, plus, for a halfvec
 *     range error only, that source element (at most 8 bytes, for the error text).
 *     The binary receive calls read the bound total (8 bytes) and a 24-byte status;
 *     vb_sparsevec_to_binary_batch_dev reads its 24-byte CSR check; vb_rows_to_binary_batch_dev
 *     reads nothing (it can be captured into a CUDA graph).
 *   - rows are row-major and contiguous in the caller's buffers (vector: dim
 *     fp32; halfvec: dim IEEE binary16; bit: (dim+7)/8 bytes, MSB first, tail
 *     bits zero -- exactly the payload of Vector.x (src/vector.h:18-24),
 *     HalfVector.x (src/halfvec.h:67-73) and VARBITS (src/bitvec.c:16-28)).
 *     Device images pad each row to a multiple of 16 bytes (zero fill).
 *   - heap TIDs are passed opaquely as int64 ids (block << 16 | offset in the glue).
 */
#ifndef VECB200_H
#define VECB200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define VB_ABI_VERSION 1

/* status codes */
#define VB_OK 0
#define VB_EINVAL (-1)			/* bad argument (dimension mismatch, unsupported metric for type, ...) */
#define VB_ENODEVICE (-2)		/* no usable sm_90 device / CUDA failure at init */
#define VB_ECUDA (-3)			/* CUDA runtime error */
#define VB_ENOMEM (-4)			/* device or host allocation failed */
#define VB_ESTATE (-5)			/* call sequence error (index not loaded, ...) */

/* element types */
#define VB_VECTOR 0				/* vector   : fp32   (src/vector.h:18-24) */
#define VB_HALFVEC 1			/* halfvec  : fp16   (src/halfvec.h:67-73) */
#define VB_BIT 2				/* bit      : packed (src/bitvec.c:16-28) */

/* metrics: what the SQL operator / opclass support function returns */
#define VB_L2_SQUARED 0			/* vector_l2_squared_distance    src/vector.c:595-605, halfvec.c:575-585 (index proc 1 of l2 opclasses) */
#define VB_NEG_IP 1				/* vector_negative_inner_product src/vector.c:637-647, halfvec.c:605-615 (<#>; proc 1 of ip and cosine opclasses) */
#define VB_COSINE 2				/* cosine_distance               src/vector.c:671-696, halfvec.c:620-645 (<=>, sequential scan only) */
#define VB_L1 3					/* l1_distance                   src/vector.c:740-750, halfvec.c:676-686 (<+>) */
#define VB_HAMMING 4			/* hamming_distance              src/bitvec.c:45-55  (<~>) */
#define VB_JACCARD 5			/* jaccard_distance              src/bitvec.c:60-70  (<%>) */
#define VB_L2 6					/* l2_distance                   src/vector.c:579-589 (<->): sqrt((double) L2^2) */
#define VB_IP 7					/* inner_product                 src/vector.c:622-632 */
#define VB_SPHERICAL 8			/* vector_spherical_distance     src/vector.c:703-722 (k-means proc 3 of ip/cosine opclasses) */

/* ------------------------------------------------------------------ runtime */

/* Bind this process to CUDA device `device` (a backend calls it once, lazily). */
int			vb_init(int device);
/* Release every device allocation made by the library in this process. */
int			vb_shutdown(void);
const char *vb_last_error(void);
/* The reference's errdetail of the last error, "" when it has none (the type input errors below have one). */
const char *vb_last_error_detail(void);
int			vb_abi_version(void);
/* cudaStream_t the library launches on (as void*), for event timing / graph capture by the host. */
void	   *vb_stream(void);
/* Kernels launched by this library since vb_init (a claim for bench.py's gpu_launches). */
int64_t		vb_launch_count(void);
int			vb_synchronize(void);
/*
 * Order the library stream after work the caller enqueued on another stream: `cuda_event` is a cudaEvent_t recorded
 * there.  Needed before a _dev call whose inputs were produced on a different stream (vb_stream() is non-blocking).
 */
int			vb_stream_wait_event(void *cuda_event);

/*
 * Optional per-kernel timing with CUDA events on vb_stream(), used by bench.py for the
 * roofline of the dominant kernel (the events add ~1 us per bracketed launch).
 * Kernels: 0 = list/candidate scan (GetScanItems) incl. query grouping / packing, 1 = centre scan (GetScanLists),
 * 2 = top-k select + exact re-score + certificate, 3 = k-means assign, 4 = HNSW search, 5 / 6 = the tensor-core filter
 * kernel alone (lists / centres).
 */
#define VB_PROF_SCAN_ITEMS 0
#define VB_PROF_SCAN_LISTS 1
#define VB_PROF_TOPK 2
#define VB_PROF_ASSIGN 3
#define VB_PROF_HNSW 4
#define VB_PROF_LIST_TC 5		/* list_tc_kernel alone (the tensor-core filter pass over the probed lists) */
#define VB_PROF_CENTRE_TC 6		/* the same kernel over the centre table (probe selection of query batches) */
#define VB_PROF_FILTER_MASK 7	/* the row-filter mask of vb_ivf_search_filtered over the candidate distances */
/* the phases of vb_ivf_build* (VB_PROF_ASSIGN stays with vb_assign and the Lloyd iterations' assign step) */
#define VB_PROF_BUILD_SAMPLE 8	/* draw, gather and (spherical) normalise + compact the samples */
#define VB_PROF_BUILD_SEED 9	/* k-means++ seeding */
#define VB_PROF_BUILD_LLOYD 10	/* Lloyd iterations */
#define VB_PROF_BUILD_DEST 11	/* list numbers -> list offsets, image order and per-row destinations */
#define VB_PROF_BUILD_PLACE 12	/* the placement kernel alone (one bracket per launch) */
#define VB_PROF_BUILD_ASSIGN 13	/* pass one: the list of every row (per chunk: padding / normalisation, assign) */
#define VB_PROF_TEXT_PARSE 14	/* the type input parse kernels (text_parse_dense_kernel, text_parse_sparse_kernel) */
#define VB_PROF_TEXT_FORMAT 15	/* the type output kernels (text_format_kernel, length and write passes) */
#define VB_PROF_BINARY_RECV 16	/* the binary receive kernels (recv_dense_kernel, recv_sparse_kernel) */
#define VB_PROF_BINARY_SEND 17	/* the binary send kernels (send_dense_kernel, send_sparse_kernel) */
int			vb_prof_enable(int on);
/* Synchronises, then returns accumulated milliseconds and bracketed launches since the last read of `kernel`. */
int			vb_prof_read(int kernel, double *total_ms, int64_t *launches);

/* ------------------------------------------------- batched distance operator */

/*
 * One query against n rows, all host buffers: out[i] = metric(rows[i], q) as the
 * float8 the fmgr wrapper returns.  Replaces n calls of
 * FunctionCall2Coll(procinfo, collation, row, q) -> l2_distance / ... / jaccard_distance
 * (src/vector.c:576-750, src/halfvec.c:557-686, src/bitvec.c:33-70).
 * dim is elements (bits for VB_BIT; 0 is a valid bit length).  q == NULL gives all zeros (ZeroDistance, src/ivfscan.c:192-196).
 */
int			vb_distance_batch(int elem, int metric, int dim, const void *q,
							  const void *rows, int64_t n, double *out);

/*
 * Batched row transforms next to the distance path (host buffers in and out):
 *   vb_norm_batch            vector_norm / l2_norm           (src/vector.c:767-780, src/halfvec.c:703-720)
 *   vb_l2_normalize_batch    l2_normalize                    (src/vector.c:785-819, src/halfvec.c:725-759); what the cosine
 *                            opclasses apply to every indexed row and to the query (src/ivfbuild.c:174-180, src/ivfscan.c:222-229);
 *                            fails with "value out of range: overflow" like float_overflow_error()
 *   vb_binary_quantize_batch binary_quantize                 (src/vector.c:952-978): out = (dim + 7) / 8 bytes per row, MSB first
 * elem = VB_VECTOR or VB_HALFVEC; norms accumulate in fp64 as in the reference.
 */
int			vb_norm_batch(int elem, int dim, const void *rows, int64_t n, double *out);
int			vb_l2_normalize_batch(int elem, int dim, const void *rows, int64_t n, void *out);
int			vb_binary_quantize_batch(int elem, int dim, const void *rows, int64_t n, uint8_t *out);
/*
 * The casts that feed halfvec / bit indexes from vector columns (README "half-precision indexing"):
 *   vb_vector_to_halfvec_batch  vector_to_halfvec (src/halfvec.c:540-555): Float4ToHalf, round to nearest even; a finite
 *                               value that overflows fails with the reference's text: "<value>" is out of range for type halfvec
 *   vb_halfvec_to_vector_batch  halfvec_to_vector (src/vector.c halfvec_to_vector): exact widening
 */
int			vb_vector_to_halfvec_batch(int dim, const void *rows, int64_t n, void *out);
int			vb_halfvec_to_vector_batch(int dim, const void *rows, int64_t n, void *out);
/*
 * subvector(v, start, count) of every row (src/vector.c:983-1025, src/halfvec.c:939-981), the value of the README's
 * "subvector indexing" recipe.  elem = VB_VECTOR or VB_HALFVEC (there is no bit subvector).  The result's dimension
 * follows the reference from the scalars alone: count < 1 is an error; end = start > dim - count ? dim + 1 :
 * start + count; start < 1 becomes 1 and start > dim is an error; out_dim = end - start must pass CheckDim (1 ..
 * 16000).  The errors are "vector must have at least 1 dimension" ("halfvec ..." for halfvec).  *out_dim is written
 * once these checks pass, before any work, and is left untouched on any error.  out receives n packed rows of
 * *out_dim elements; with n = 0, rows and out may be NULL, so such a call sizes the output.
 */
int			vb_subvector_batch(int elem, int dim, const void *rows, int64_t n, int32_t start, int32_t count, void *out,
							   int *out_dim);

/*
 * The same transforms on rows that already live on the device (a model's output, a resident column), for the
 * expression-index recipes: embedding::halfvec(n), binary_quantize(embedding)::bit(n) and subvector(embedding, 1, n)
 * under the cosine opclasses.  Rows and outputs are packed (dim elements per row, no padding; bit rows (dim + 7) / 8
 * bytes; norms one float8 per row), and each result equals its host variant's bit for bit.  Input and output must not
 * overlap, except that vb_l2_normalize_batch_dev may run in place (out_dev == rows_dev); another overlap is refused.
 * Refused before any launch (VB_EINVAL): an elem other than VB_VECTOR / VB_HALFVEC, dim <= 0, n < 0, a NULL pointer with
 * n > 0.  n = 0 launches nothing.
 * vb_norm_batch_dev, vb_binary_quantize_batch_dev, vb_halfvec_to_vector_batch_dev and vb_subvector_batch_dev are fully
 * asynchronous on vb_stream() and use no workspace (they can be captured into a CUDA graph).  The two calls that can
 * fail on the data read back a little (see the conventions above) and synchronise: vb_l2_normalize_batch_dev returns
 * VB_EINVAL "value out of range: overflow", vb_vector_to_halfvec_batch_dev the host variant's text for the first
 * offender in row-major order; on either error out_dev is unspecified.
 */
int			vb_norm_batch_dev(int elem, int dim, const void *rows_dev, int64_t n, double *out_dev);
int			vb_l2_normalize_batch_dev(int elem, int dim, const void *rows_dev, int64_t n, void *out_dev);
int			vb_binary_quantize_batch_dev(int elem, int dim, const void *rows_dev, int64_t n, uint8_t *out_dev);
int			vb_vector_to_halfvec_batch_dev(int dim, const void *rows_dev, int64_t n, void *out_dev);
int			vb_halfvec_to_vector_batch_dev(int dim, const void *rows_dev, int64_t n, void *out_dev);
int			vb_subvector_batch_dev(int elem, int dim, const void *rows_dev, int64_t n, int32_t start, int32_t count,
								   void *out_dev, int *out_dim);

/*
 * The operators + - * || of vector and halfvec over batches of rows (sql/vector.sql:274-298, :734-760), e.g. centring a
 * column (v - mean), per-dimension weights (v * w) or joining two models' embeddings (a || b):
 *   vb_arith_batch   vector_add / vector_sub / vector_mul (src/vector.c:824-921) and halfvec_add / halfvec_sub /
 *                    halfvec_mul (src/halfvec.c:766-879), chosen by op.  vector: a op b in fp32; halfvec:
 *                    Float4ToHalfUnchecked(HalfToFloat4(a) op HalfToFloat4(b)), the fp32 result rounded to nearest even.
 *                    Subnormals are kept, and a NaN operand passes through.
 *   vb_concat_batch  vector_concat (src/vector.c:928-947), halfvec_concat (src/halfvec.c:886-903): rows of dim_a + dim_b
 * elem = VB_VECTOR or VB_HALFVEC.  Rows are packed.  na and nb are equal, or one of them is 1: an operand of one row is
 * used with every row of the other (SQL's v - $1, $1 || v).  The result has nb rows (na when nb == 1); other counts are
 * refused.
 * Before any work: vb_arith_batch requires dim_a == dim_b ("different vector dimensions %d and %d", CheckDims,
 * src/vector.c:71-77); vb_concat_batch requires dim_a + dim_b <= 16000 ("vector cannot have more than 16000 dimensions",
 * CheckDim, src/vector.c:95-106), then writes *out_dim (left untouched on any error); with 0 result rows, rows and out may
 * be NULL, so such a call sizes the output.  halfvec texts say "halfvec".
 * Data errors are those the reference's row-by-row execution raises first (lowest row, then the first element its
 * checking loop reaches): "value out of range: overflow" where a result is infinite (isinf / HalfIsInf), and for *,
 * "value out of range: underflow" where it is zero (halfvec: HalfIsZero, so -0 too) while neither operand is.  || has
 * none.  On a data error out is unspecified.
 */
#define VB_ADD 0				/* vector_add / halfvec_add (+) */
#define VB_SUB 1				/* vector_sub / halfvec_sub (-) */
#define VB_MUL 2				/* vector_mul / halfvec_mul (*) */
int			vb_arith_batch(int elem, int op, int dim_a, const void *a, int64_t na, int dim_b, const void *b, int64_t nb,
						   void *out);
int			vb_concat_batch(int elem, int dim_a, const void *a, int64_t na, int dim_b, const void *b, int64_t nb, void *out,
							int *out_dim);
/*
 * The array casts array_to_vector (src/vector.c:443-512) and array_to_halfvec (src/halfvec.c:442-509): n rows of dim
 * elements of integer[], real[] or double precision[] (src) to vector / halfvec rows (elem), as (float) of the int32 or
 * double (round to nearest even) and, for halfvec, Float4ToHalf of that float.  typmod is the target's dimension, or -1.
 * Before any work, in the reference's order: CheckDim(dim) ("vector must have at least 1 dimension", "vector cannot
 * have more than 16000 dimensions"), then CheckExpectedDim ("expected %d dimensions, not %d").  Data errors, from the
 * lowest failing row:
 *   vector:  the whole row is converted, then the first NaN or infinite element gives "NaN not allowed in vector" or
 *            "infinite value not allowed in vector" (so {4e38} from double precision[] is an infinite value);
 *   halfvec: first the conversion pass: the first element whose float is finite but whose half is infinite gives
 *            "\"<float>\" is out of range for type halfvec"; only when there is none, the check pass: "NaN not allowed
 *            in halfvec" / "infinite value not allowed in halfvec".  So in one row a range error beats an earlier NaN.
 * On a data error out is unspecified.  The array structure checks ("array must be 1-D", "array must not contain
 * nulls", "unsupported array type") stay with the caller, which unpacks the ArrayType; numeric[] sources go to
 * vb_numeric_array_to_rows_batch.
 */
#define VB_ARRAY_INT4 0			/* integer[]          : (float) int32  */
#define VB_ARRAY_FLOAT4 1		/* real[]             : as is          */
#define VB_ARRAY_FLOAT8 2		/* double precision[] : (float) double */
#define VB_ARRAY_NUMERIC 3		/* numeric[]: one numeric_send field per element (vb_numeric_array_to_rows_batch,
								 * vb_array_to_sparsevec_batch; vb_array_to_rows_batch refuses it) */
int			vb_array_to_rows_batch(int elem, int src, int dim, int32_t typmod, const void *in, int64_t n, void *out);
/*
 * The numeric[] branch of array_to_vector / array_to_halfvec: n rows of dim numeric elements, element i of row r the
 * field e = r * dim + i at bytes[off[e] .. off[e + 1]) (any alignment; off[n * dim + 1], 8-byte aligned).  A field is
 * what PostgreSQL's numeric_send writes: big-endian int16 ndigits, int16 weight, uint16 sign, uint16 dscale, then
 * ndigits base-10000 int16 digits.  These rules are PostgreSQL core's (numeric.c, float.c), not pgvector's:
 *   - a field is first checked as numeric_recv reads it; a malformed one is refused with VB_EINVAL before any data
 *     error, naming the field: "insufficient data left in message" (a read past its end), "invalid sign in external
 *     "numeric" value", "invalid scale in external "numeric" value" (dscale > 0x3FFF), "invalid digit in external
 *     "numeric" value" (a digit >= 10000), "incorrect binary data format" (bytes left over, as COPY reports them);
 *   - each element becomes numeric_float4 of it: NaN and +-Infinity as themselves; a finite value is float4in of the
 *     decimal numeric_out prints (digits past dscale fraction digits truncated, zero as "0", so +0), which is glibc
 *     strtof, correctly rounded; when strtof's result is 0 or infinite from a value that is not, float4in fails with
 *     ""<numeric_out text>" is out of range for type real" (a subnormal result is kept);
 *   - vector converts the whole row, then CheckElement: a range error at element 9 beats a NaN at element 2;
 *     halfvec runs numeric_float4 and then Float4ToHalf on each element in turn (""65520" is out of range for type
 *     halfvec"), then CheckElement.
 * The dimension checks and the lowest-failing-row rule are vb_array_to_rows_batch's.  *out_bad (optional) is the failing
 * row, or -1.  The host variant streams chunks of whole rows (about 32 MB of fields and offsets; a longer row alone)
 * through pinned staging.  The _dev variant reads back 16 bytes (the first-offender key and the first malformed field)
 * and, on an error only, the offending field for its text.
 */
int			vb_numeric_array_to_rows_batch(int elem, int dim, int32_t typmod, const void *bytes, const int64_t *off, int64_t n,
										   void *out, int64_t *out_bad);
int			vb_numeric_array_to_rows_batch_dev(int elem, int dim, int32_t typmod, const void *bytes_dev, const int64_t *off_dev,
											   int64_t n, void *out_dev, int64_t *out_bad);
/*
 * The same on device rows.  Each result equals its host variant's bit for bit.  Refused before any launch (VB_EINVAL):
 * a bad elem, op or src, a dimension <= 0, a negative count, a NULL pointer for work that exists, rows or output not
 * aligned to their elements, and input and output that overlap, except that vb_arith_batch_dev may write in place
 * (out_dev == a_dev or b_dev) over an operand that is not broadcast.  Calls with 0 result rows launch nothing.
 * vb_concat_batch_dev is fully asynchronous on vb_stream() and uses no workspace (it can be captured into a CUDA graph).
 * vb_arith_batch_dev and vb_array_to_rows_batch_dev read back the 8-byte key of the first offender and synchronise;
 * a halfvec range error also reads the offending source element (at most 8 bytes) for its text.
 */
int			vb_arith_batch_dev(int elem, int op, int dim_a, const void *a_dev, int64_t na, int dim_b, const void *b_dev,
							   int64_t nb, void *out_dev);
int			vb_concat_batch_dev(int elem, int dim_a, const void *a_dev, int64_t na, int dim_b, const void *b_dev, int64_t nb,
								void *out_dev, int *out_dim);
int			vb_array_to_rows_batch_dev(int elem, int src, int dim, int32_t typmod, const void *in_dev, int64_t n,
									   void *out_dev);

/* ------------------------------------------------------ resident row tables */

typedef struct vb_table vb_table;	/* [n x dim] rows resident in HBM (exact scan, HNSW vectors, k-means samples) */

/*
 * Rows whose query image (the padded row, halfvec widened to fp32) is over the 227 KiB of shared memory the scan holds
 * it in -- vector or halfvec past 58112 dimensions, bit past 1859584 bits -- are refused with VB_EINVAL, as they are by
 * vb_distance_batch.
 */
int			vb_table_create(int elem, int dim, vb_table **out);
/* Append n rows from host memory (pinned staging + async copy inside). */
int			vb_table_append(vb_table *t, const void *rows, int64_t n);
/* Append n rows that already live on the device (packed, unpadded layout). */
int			vb_table_append_dev(vb_table *t, const void *rows_dev, int64_t n);
int64_t		vb_table_rows(const vb_table *t);
/* Read-only view of the resident rows: device pointer of row 0 and the padded row stride in bytes. */
const void *vb_table_device_rows(const vb_table *t, size_t *stride_bytes);
int			vb_table_free(vb_table *t);

/*
 * Exact (no index) top-k of nq queries over the table: the sequential-scan plan
 * "ORDER BY v <op> q LIMIT k" (operator wrapper + top-N sort; SURVEY 3.4).
 * out_ids[q*k + j] is the row number (0-based append order), -1 padded;
 * out_dist the operator's float8.  Ties on distance: smaller row number first.
 */
int			vb_exact_topk(vb_table *t, int metric, const void *queries, int64_t nq, int k,
						  int64_t *out_ids, double *out_dist);
int			vb_exact_topk_dev(vb_table *t, int metric, const void *queries_dev, int64_t nq, int k,
							  int64_t *out_ids_dev, float *out_dist_dev);

/*
 * Re-rank: for each query, the k nearest of ITS candidate rows of the table, under the SQL operator -- the outer
 * "ORDER BY v <op> q LIMIT k" over an inner index scan's result (README quantize-then-rerank flow).
 * cand[q*c + j] = a row number of t (append order); -1 = no candidate.  metric: as vb_exact_topk (VB_L2, VB_L2_SQUARED,
 * VB_IP, VB_NEG_IP, VB_COSINE, VB_L1 for vector / halfvec; VB_HAMMING, VB_JACCARD for bit).  1 <= k <= 2048, c >= 0.
 * out_ids = row numbers, -1 padded when a query has fewer than k candidates; out_dist = the operator's float8, as
 * vb_exact_topk reports it.  Ties: earlier candidate position first.  A row listed twice is scored twice.
 * Host variant: a candidate outside [-1, n) fails with VB_EINVAL naming query, position and value, nothing written.
 * _dev variant: asynchronous on vb_stream(), no host read; candidates outside [0, n) are treated as absent (never read).
 */
int			vb_table_rerank(vb_table *t, int metric, const void *queries, int64_t nq, const int64_t *cand, int c, int k,
							int64_t *out_ids, double *out_dist);
int			vb_table_rerank_dev(vb_table *t, int metric, const void *queries_dev, int64_t nq, const int64_t *cand_dev, int c,
								int k, int64_t *out_ids_dev, float *out_dist_dev);

/* ------------------------------------------------------------- row filters */

/*
 * A row filter: the allowed rows of one table or one IVFFlat image, resident on the device -- what a B-tree or bitmap
 * scan on a filter column yields for "WHERE <predicate> ORDER BY v <op> q LIMIT k" (README "Filtering").  Queries that
 * take a filter never read, score, select or copy a row it does not allow.  Sparse tables take filters of their own
 * (vb_sparse_table_filter_create, with the sparsevec calls below).
 *
 * Table filters: rows = row numbers of t (append order).  Host variant: a value outside [0, n) fails with VB_EINVAL
 * naming its position and value; _dev variant: such values are ignored.  Rows appended to t later are not in the
 * filter; the filter stays valid (row numbers do not move).
 * IVFFlat filters: ids = heap ids as given at load (row positions when the image was loaded with ids == NULL).  Ids the
 * image does not hold are ignored (a TID set from a bitmap scan of the heap may name rows this index does not hold);
 * every image row whose id is in the set is allowed, so an id the image holds on several rows allows them all.
 * The filter records the image it was made for: after vb_ivf_load*, vb_ivf_end_load or vb_ivf_replace_list, any use of
 * it fails with VB_ESTATE ("index changed since the filter was created").
 * Duplicates collapse.  n == 0 is an empty filter.  Using a filter with a table or index other than its own fails with
 * VB_EINVAL, also after its own was freed (every table and image carries a process-wide unique stamp).  The exact top-k
 * takes filters of fewer than 2^31 rows.  Creation synchronises (it reads back the number of allowed rows); the caller's arrays may be reused at once.
 * HNSW images take element filters (vb_hnsw_filter_create, with the HNSW scan below).
 */
typedef struct vb_filter vb_filter;
struct vb_ivf;	/* the IVFFlat image, below */
int			vb_table_filter_create(vb_table *t, const int64_t *rows, int64_t n, vb_filter **out);
int			vb_table_filter_create_dev(vb_table *t, const int64_t *rows_dev, int64_t n, vb_filter **out);
int			vb_ivf_filter_create(struct vb_ivf *ix, const int64_t *ids, int64_t n, vb_filter **out);
int			vb_ivf_filter_create_dev(struct vb_ivf *ix, const int64_t *ids_dev, int64_t n, vb_filter **out);
int64_t		vb_filter_rows(const vb_filter *f);	/* rows allowed (0 for NULL) */
int			vb_filter_free(vb_filter *f);

/*
 * Filtered exact top-k: for each query q, the k nearest of the rows filters[filter_of_query[q]] allows.
 * filter_of_query is host memory in both variants ([nq], entries in [0, nfilters); NULL when nfilters == 1); an entry
 * out of range fails with VB_EINVAL naming the query.  One call can batch queries with different predicates.
 * Each query's result is bit-identical, ids and distances, to vb_table_rerank(t, metric, q, cand = its filter's allowed
 * rows in ascending order, k): the same metrics, 1 <= k <= 2048, ties to the smaller row number, the same -1 padding
 * when fewer than k rows are allowed.  A filter of every row therefore gives vb_exact_topk under scan_impl = 0.
 * _dev variant: queries and outputs on the device, asynchronous on vb_stream().
 */
int			vb_exact_topk_filtered(vb_table *t, int metric, const void *queries, int64_t nq, int k,
								   const vb_filter *const *filters, int nfilters, const int32_t *filter_of_query,
								   int64_t *out_ids, double *out_dist);
int			vb_exact_topk_filtered_dev(vb_table *t, int metric, const void *queries_dev, int64_t nq, int k,
									   const vb_filter *const *filters, int nfilters, const int32_t *filter_of_query,
									   int64_t *out_ids_dev, float *out_dist_dev);

/* -------------------------------------------------------------- aggregates */

/*
 * avg(vector), sum(vector), avg(halfvec), sum(halfvec) (sql/vector.sql:163-198, 607-642) over the rows of a table, with
 * GROUP BY: "SELECT avg(v) FROM t" and "SELECT g, avg(v) FROM t GROUP BY g".  t holds VB_VECTOR or VB_HALFVEC rows
 * (VB_BIT: VB_EINVAL, the reference has no bit aggregates).
 *
 * group_of_row [n] puts row i in group group_of_row[i] in [0, ngroups), or leaves it out with -1 (a WHERE that rejects
 * it, or a NULL value); NULL puts every row in group 0 and requires ngroups == 1.
 *
 * The plan.  For each group g, S_g = its rows in ascending row number, cut into runs of R = run_rows consecutive rows
 * (the last may be short; R = 0 or R >= |S_g| is one run, the serial plan):
 *   run state    the transition function over the run's rows in order from the initial condition.  avg, INITCOND '{0}':
 *                the first row sets n = 1, s_i = (double) x_i (vector_accum's new-array branch, so a -0 survives), each
 *                later row adds (double) x_i in float8 (src/vector.c:1148-1204; halfvec widens by HalfToFloat4,
 *                src/halfvec.c:1104-1160).  sum, strict with no initcond: the first row is the state, each later row is
 *                added by vector_add (fp32 add, src/vector.c:824-852) or halfvec_add (add, round to fp16,
 *                src/halfvec.c:764-798);
 *   group state  the run states combined left to right, combine(combine(r0, r1), r2) ...: avg by vector_combine (sums and
 *                counts added, src/vector.c:1209-1284), sum by the transition's add;
 *   final        avg: (float) (s_i / n) (src/vector.c:1289-1318), Float4ToHalf of that for halfvec (src/halfvec.c:1165-1194);
 *                sum: the state.  A group with no rows has count 0 (the SQL NULL) and a zero-filled result.
 * R = 0 without groups is PostgreSQL's serial "SELECT avg(v) FROM t" in table order; R = ceil(n / W) is a Partial
 * Aggregate of W participants taking contiguous ranges.  Results depend on R only through rounding, as the reference's
 * depend on its plan; for a given R they are deterministic and independent of the launch configuration.
 *
 * Outputs: out [ngroups x dim] (fp32 for vector, IEEE binary16 for halfvec), out_counts [ngroups], and for avg optionally
 * out_state [ngroups x (dim + 1)] = n, s_1 .. s_dim: the float8 transition state vector_accum / vector_combine hold, which
 * a Partial Aggregate hands to the Finalize Aggregate (so a caller can combine it with partial states computed
 * elsewhere).  sum's state is out itself: sum requires out_state == NULL.
 *
 * Errors.  sum: a transition or combine step that produces an infinite element fails with VB_EINVAL and
 * float_overflow_error()'s text, "value out of range: overflow"; which steps exist depends on R, so whether a call fails
 * does too (the host variant then writes nothing).  avg: the float8 state cannot overflow for finite rows; what a
 * non-finite row gives is unspecified.  Validation before any kernel runs: an unknown agg, ngroups < 1, run_rows < 0, a
 * NULL group_of_row with ngroups != 1, or (host variant) a group id outside [-1, ngroups), which names the row and the
 * value, fail with VB_EINVAL; the _dev variant counts such ids as -1.  Grouped calls take tables of at most 2^31 - 1
 * rows.  VB_ENOMEM names the bytes needed (row list and sort space, run states, staged results) and allocates nothing.
 * An empty table gives every count 0.
 * _dev variant: group_of_row and the outputs on the device; asynchronous on vb_stream() except for one 4-byte read of
 * sum's overflow flag.
 */
#define VB_AGG_AVG 0
#define VB_AGG_SUM 1
int			vb_table_aggregate(vb_table *t, int agg, const int32_t *group_of_row, int ngroups, int64_t run_rows,
							   void *out, int64_t *out_counts, double *out_state);
int			vb_table_aggregate_dev(vb_table *t, int agg, const int32_t *group_of_row_dev, int ngroups, int64_t run_rows,
								   void *out_dev, int64_t *out_counts_dev, double *out_state_dev);

/* ---------------------------------------------------------------- sparsevec */

/*
 * sparsevec (src/sparsevec.h:21-32): dim, nnz, indices[nnz] (0-based, ascending), values[nnz].  A batch of rows is CSR:
 * row r = entries row_off[r] .. row_off[r+1] of idx[] / val[] (row_off[0] = 0).  The calls of this block take host
 * buffers; the resident table's calls and the casts below also have _dev variants.
 *
 *   vb_sparsevec_distance_batch      out[r] = metric(row r, q) as the float8 of sparsevec's l2_distance /
 *                                    l2_squared_distance / inner_product / negative_inner_product / cosine_distance /
 *                                    l1_distance (src/sparsevec.c:826-1057); metric = VB_L2, VB_L2_SQUARED, VB_IP, VB_NEG_IP,
 *                                    VB_COSINE, VB_L1.  dim != q_dim fails with CheckDims' text ("different sparsevec
 *                                    dimensions %d and %d", src/sparsevec.c:44-51); q_nnz < 0 = NULL query, all zeros.
 *   vb_sparsevec_norm_batch          l2_norm (src/sparsevec.c:1062-1077), fp64 sums
 *   vb_sparsevec_l2_normalize_batch  l2_normalize (src/sparsevec.c:1082-1150): quotients that round to zero are dropped, so
 *                                    the result has its own offsets; out_idx / out_val need room for row_off[n] entries;
 *                                    an infinite quotient fails with "value out of range: overflow"
 */
int			vb_sparsevec_distance_batch(int metric, int dim, int q_dim, int32_t q_nnz, const int32_t *q_idx, const float *q_val,
										int64_t n, const int64_t *row_off, const int32_t *idx, const float *val, double *out);
int			vb_sparsevec_norm_batch(int64_t n, const int64_t *row_off, const float *val, double *out);
int			vb_sparsevec_l2_normalize_batch(int64_t n, const int64_t *row_off, const int32_t *idx, const float *val,
											int64_t *out_row_off, int32_t *out_idx, float *out_val);

typedef struct vb_sparse_table vb_sparse_table;	/* n sparsevec rows resident in HBM as CSR */

int			vb_sparse_table_create(int dim, vb_sparse_table **out);
int			vb_sparse_table_append(vb_sparse_table *t, int64_t n, const int64_t *row_off, const int32_t *idx, const float *val);
/*
 * Device CSR (the _dev variants of this section): row_off_dev / q_off_dev [n + 1] int64, idx int32, val float, all device
 * pointers, checked on the device with the host variants' rules and texts -- offsets from 0 and never decreasing, at most
 * 16000 entries per row, indices inside [0, dim) and strictly ascending -- with " (row r)" naming the first bad row.
 * That check is the one read back (at most 24 bytes); everything after it is enqueued on vb_stream().  Entries of a row
 * whose offsets lie outside [0, row_off[n]] are not read (a row before it has bad offsets and is reported).
 * vb_sparse_table_append_dev appends nothing on any error; growing the table's buffers synchronises, as in the host
 * variant.
 */
int			vb_sparse_table_append_dev(vb_sparse_table *t, int64_t n, const int64_t *row_off_dev, const int32_t *idx_dev,
									   const float *val_dev);
int64_t		vb_sparse_table_rows(const vb_sparse_table *t);
int64_t		vb_sparse_table_nnz(const vb_sparse_table *t);
int			vb_sparse_table_free(vb_sparse_table *t);
/*
 * Exact (no index) top-k of nq sparsevec queries (CSR: q_off[nq+1], q_idx, q_val) over the table: the sequential-scan plan
 * "ORDER BY v <op> q LIMIT k" for <-> (VB_L2), <#> (VB_NEG_IP), <=> (VB_COSINE), <+> (VB_L1); k <= 2048.
 * out_ids = row numbers (append order, -1 padded), out_dist = the operator's float8; ties: smaller row number first.
 */
int			vb_sparse_exact_topk(vb_sparse_table *t, int metric, int q_dim, int64_t nq, const int64_t *q_off, const int32_t *q_idx,
								 const float *q_val, int k, int64_t *out_ids, double *out_dist);
/* queries and outputs on the device: ids as the host variant's, distances the float of its float8 */
int			vb_sparse_exact_topk_dev(vb_sparse_table *t, int metric, int q_dim, int64_t nq, const int64_t *q_off_dev,
										 const int32_t *q_idx_dev, const float *q_val_dev, int k, int64_t *out_ids_dev,
										 float *out_dist_dev);

/*
 * Row filters of a sparse table (see vb_filter above): rows = row numbers of t (append order).  A value outside [0, n)
 * fails with VB_EINVAL naming its position and value.  Duplicates collapse, n == 0 is an empty filter; rows appended
 * later are not in the filter, and it stays valid.  vb_filter_rows and vb_filter_free apply.  A sparse filter is refused
 * (VB_EINVAL, "made for another table or index") by any other sparse table, by its own after that was freed, and by
 * every dense, IVFFlat and HNSW call; the sparse calls refuse their filters.
 */
int			vb_sparse_table_filter_create(vb_sparse_table *t, const int64_t *rows, int64_t n, vb_filter **out);
/* rows on the device; values outside [0, n) are ignored (as vb_table_filter_create_dev) */
int			vb_sparse_table_filter_create_dev(vb_sparse_table *t, const int64_t *rows_dev, int64_t n, vb_filter **out);
/*
 * Filtered exact top-k: for each query q, the k nearest of the rows filters[filter_of_query[q]] allows -- the plan of
 * "WHERE <predicate> ORDER BY v <op> q LIMIT k" with a B-tree or bitmap scan on the filter column.  filter_of_query is a
 * host array [nq], NULL when nfilters == 1; an entry out of range fails with VB_EINVAL naming the query.  Metrics, k and
 * q_dim as vb_sparse_exact_topk (its texts).  Each query's result is bit-identical, ids and distances, to
 * vb_sparse_table_rerank with cand = its filter's allowed rows in ascending order: ties to the smaller row number, -1 /
 * +inf padding when fewer than k rows are allowed.  A filter of every row therefore gives vb_sparse_exact_topk's output.
 * Rows the filter rejects are never read, scored, selected or copied.
 *
 * Re-rank: for each query, the k nearest of ITS candidate rows -- the outer "ORDER BY v <op> q LIMIT k" over another
 * index's result (hybrid search: a dense or quantized index fetches the candidates, the sparse column orders them).
 * cand[q*c + j] = a row number of t; -1 = no candidate.  A value outside [-1, n) fails with VB_EINVAL naming the query,
 * the position and the value.  A row listed twice is scored twice; ties go to the earlier candidate position, and a NaN
 * distance (cosine against a zero-norm row) ranks before the padding.  Every distance is bit-identical to the one
 * vb_sparse_exact_topk reports for that row.  c >= 0.
 *
 * Both: everything is validated before any kernel runs, and on any error nothing is written to out_ids / out_dist.
 * Queries run in sub-batches of at most 65535 whose distance runs stay under 1 GiB; VB_ENOMEM names the bytes that could
 * not be allocated.  The filters may be freed once the call returns.
 *
 * _dev variants: queries (device CSR, above), cand and the outputs on the device, ids as the host variant's and distances
 * the float of its float8; filters and filter_of_query stay host arrays.  Candidates outside [0, n) are treated as
 * absent and never read (as vb_table_rerank_dev).  On a refused call nothing is written.
 */
int			vb_sparse_exact_topk_filtered(vb_sparse_table *t, int metric, int q_dim, int64_t nq, const int64_t *q_off,
										  const int32_t *q_idx, const float *q_val, int k, const vb_filter *const *filters,
										  int nfilters, const int32_t *filter_of_query, int64_t *out_ids, double *out_dist);
int			vb_sparse_exact_topk_filtered_dev(vb_sparse_table *t, int metric, int q_dim, int64_t nq, const int64_t *q_off_dev,
												  const int32_t *q_idx_dev, const float *q_val_dev, int k,
												  const vb_filter *const *filters, int nfilters, const int32_t *filter_of_query,
												  int64_t *out_ids_dev, float *out_dist_dev);
int			vb_sparse_table_rerank(vb_sparse_table *t, int metric, int q_dim, int64_t nq, const int64_t *q_off,
								   const int32_t *q_idx, const float *q_val, const int64_t *cand, int c, int k, int64_t *out_ids,
								   double *out_dist);
int			vb_sparse_table_rerank_dev(vb_sparse_table *t, int metric, int q_dim, int64_t nq, const int64_t *q_off_dev,
										   const int32_t *q_idx_dev, const float *q_val_dev, const int64_t *cand_dev, int c, int k,
										   int64_t *out_ids_dev, float *out_dist_dev);

/*
 * Casts between the dense types and sparsevec, batched (elem = VB_VECTOR or VB_HALFVEC; rows packed, dim elements each):
 *   vb_dense_to_sparsevec_batch  vector_to_sparsevec / halfvec_to_sparsevec (src/sparsevec.c:606-689): an element is kept
 *                                when x != 0 (halfvec: !HalfIsZero), so -0 is dropped; kept elements in ascending index
 *                                order, halfvec values widened exactly.  out_row_off [n + 1] is always written; when the
 *                                rows hold more than cap entries the call fails with VB_EINVAL naming the count and writes
 *                                no indices or values (cap = 0 sizes the output).  Errors: CheckDim's and CheckNnz's texts
 *                                ("sparsevec must have at least 1 dimension", "sparsevec cannot have more than 16000
 *                                non-zero elements (row r)").
 *   vb_sparsevec_to_dense_batch  sparsevec_to_vector / sparsevec_to_halfvec (src/vector.c:1323-1349, src/halfvec.c:1199-1225):
 *                                out [n x dim] zero-filled, then the entries scattered; halfvec by Float4ToHalf, so a
 *                                finite value that overflows fails with "\"65520\" is out of range for type halfvec" and a
 *                                value that rounds to 0 stores a zero.  dim above 16000 fails with "vector cannot have
 *                                more than 16000 dimensions" (or halfvec's).  The CSR is checked as the table's; on error
 *                                out is unspecified.
 * Host variants synchronise.  _dev variants read back one result of at most 24 bytes (to sparsevec: the nnz check and
 * the total) or 32 bytes (to dense: the CSR check and the first overflowing entry; on that error 4 more bytes, the value).
 */
/*
 * array_to_sparsevec (src/sparsevec.c:694-821), batched: n rows of dim elements of integer[], real[], double precision[]
 * (src = VB_ARRAY_INT4 / FLOAT4 / FLOAT8, rows packed and aligned to their elements, in_off NULL) or numeric[]
 * (VB_ARRAY_NUMERIC: in holds numeric_send fields at in_off, as in vb_numeric_array_to_rows_batch) to CSR, with the
 * output conventions of vb_dense_to_sparsevec_batch (out_row_off [n + 1] always written, cap = 0 sizes the output, a
 * total above cap fails with VB_EINVAL naming the total and writes no entries).  Each element becomes (float) of the
 * int32 or double (round to nearest even), a real as is, or numeric_float4 of the numeric, and is kept when v != 0: -0
 * and a double that rounds to 0 (1e-46) are dropped, NaN and the infinities are kept.  Rows may have up to 10^9
 * elements.
 * Before any work, in the reference's order: CheckDim ("sparsevec must have at least 1 dimension", "sparsevec cannot
 * have more than 1000000000 dimensions"), then CheckExpectedDim ("expected %d dimensions, not %d"; typmod -1: none).
 * numeric[]: malformed fields are refused first, as in vb_numeric_array_to_rows_batch.  Data errors, as row-by-row
 * execution raises them (the lowest failing row, then the first check its loops reach): numeric_float4's range error in
 * the count loop (the first failing element), CheckNnz after it ("sparsevec cannot have more than 16000 non-zero
 * elements"), then CheckElement over the kept values in index order ("NaN not allowed in sparsevec", "infinite value not
 * allowed in sparsevec").  A data error wins over the cap check, so a sizing call already fails with the error the full
 * call would raise.  *out_bad (optional) is the failing row, or -1.  On an error the outputs are unspecified.  The array
 * structure checks ("array must be 1-D", "array must not contain nulls", "unsupported array type") stay with the caller.
 * The host variant streams chunks of whole rows (about 32 MB of source each; a longer row is a chunk of its own)
 * through pinned staging, so the input is not bound by device memory.  The _dev variant reads back one 24-byte check
 * result, like vb_dense_to_sparsevec_batch_dev (numeric[]: 16 bytes more, and the offending field on an error).  Calls
 * with n = 0 launch nothing.
 */
int			vb_array_to_sparsevec_batch(int src, int dim, int32_t typmod, const void *in, const int64_t *in_off, int64_t n,
										int64_t cap, int64_t *out_row_off, int32_t *out_idx, float *out_val, int64_t *out_bad);
int			vb_array_to_sparsevec_batch_dev(int src, int dim, int32_t typmod, const void *in_dev, const int64_t *in_off_dev,
											int64_t n, int64_t cap, int64_t *out_row_off_dev, int32_t *out_idx_dev,
											float *out_val_dev, int64_t *out_bad);
int			vb_dense_to_sparsevec_batch(int elem, int dim, const void *rows, int64_t n, int64_t cap, int64_t *out_row_off,
										int32_t *out_idx, float *out_val);
int			vb_dense_to_sparsevec_batch_dev(int elem, int dim, const void *rows_dev, int64_t n, int64_t cap,
											int64_t *out_row_off_dev, int32_t *out_idx_dev, float *out_val_dev);
int			vb_sparsevec_to_dense_batch(int elem, int dim, int64_t n, const int64_t *row_off, const int32_t *idx, const float *val,
										void *out);
int			vb_sparsevec_to_dense_batch_dev(int elem, int dim, int64_t n, const int64_t *row_off_dev, const int32_t *idx_dev,
											const float *val_dev, void *out_dev);

/* ------------------------------------------------------------ text input and output */

/*
 * The type I/O over a column: vector_in / halfvec_in (src/vector.c:174-281, src/halfvec.c:178-286, elem = VB_VECTOR /
 * VB_HALFVEC), sparsevec_in (src/sparsevec.c:203-409) and vector_out / halfvec_out / sparsevec_out (src/vector.c:289-326,
 * src/halfvec.c:294-335, src/sparsevec.c:428-476).  Values, bytes and error texts are the reference's.
 *
 * Input literals.  Literal i is text[off[i] .. off[i + 1]), ending earlier at its first NUL byte as the cstring the fmgr
 * passes would; no terminator is needed.  Tokens are what glibc strtof / strtol (base 10) accept in the C locale,
 * correctly rounded to nearest even (decimal of any length, hex floats, inf / infinity / nan / nan(chars), any case).
 * Rows: dense values packed at out[out_row_off[i] ..) (float, or IEEE half bits); sparsevec as the CSR the sparse table
 * calls take (ascending 0-based indices, no zeros: vb_sparse_table_append_dev takes it unchanged) and the dimension of
 * each literal in out_dim.
 *
 * Sizes.  The bound of a literal is its commas before the first NUL + 1 (the dimension of every valid dense literal,
 * and sparsevec_in's maxNnz); typmod >= 1 makes the dense offsets i * typmod.  out_row_off [n + 1] is always written:
 * dense, the bound's (or typmod's) offsets; sparsevec, the stored entries' offsets on success and the bound's when
 * the call fails on cap.  A bound total above cap fails with VB_EINVAL naming the total and writes nothing else.
 * Output: text without terminators, out_off [n + 1] byte offsets, always written; cap is bytes, and a total above it
 * fails with VB_EINVAL naming the total (out = NULL sizes: offsets only, no cap check).  The reference's own buffer bound always suffices:
 * dim * 16 + 2 bytes per dense row, (12 + 16) * nnz + 15 per sparsevec row.
 *
 * Errors.  A call fails (VB_EINVAL) with the error the reference's row-by-row execution raises first: the lowest failing
 * literal, within it the first error its left-to-right scan reaches, the end-of-literal checks (CheckDim,
 * CheckExpectedDim, and after the sort CheckIndex) last.  vb_last_error() is the reference's errmsg (the literal echoed
 * in "invalid input syntax for type vector: \"...\"", the strtof token in "\"4e38\" is out of range for type vector"),
 * vb_last_error_detail() its errdetail.  *out_bad (may be NULL) is the failing literal's index, -1 otherwise.  On an
 * error the rows are unspecified.
 *
 * Host variants stream the text through pinned staging in chunks of literals of at most 64 MiB of text (one longer
 * literal makes a chunk of its own); chunks run in order and the first chunk with an error stops the call.  The dense
 * input overlaps the host's staging of the next chunk (and its copy of the previous chunk's rows) with the parse of
 * the current one through two pinned slots; sparsevec input runs chunks one after another, since each reads back its
 * stored total and sort flag before the next can start.  The bound is counted on the host first (commas before the
 * first NUL, with the C library's memchr).  Output host variants take chunks of rows whose text is at most 64 MiB by
 * the reference's bound; a length pass over all chunks sizes the text before any is written, and the write pass
 * reuses those offsets.  sparsevec output first checks the rows as the sparse table calls do (offsets from 0, indices
 * ascending inside [0, dim)), with their texts ("sparsevec index out of bounds (row r)").  _dev variants take device
 * pointers (text, off, outputs; out_bad and cap stay host values), run on vb_stream() and synchronise.  They read
 * back: dense input, the bound total (8 bytes) and a 64-byte status; sparsevec input, the bound total, the stored total
 * and the sort flag (8 bytes each) and the status (more than 2^31 - 1 bound entries in one call are refused);
 * output, the text total (8 bytes), and for sparsevec the 24-byte row check.  On an error they also read the failing
 * literal (at most its length in bytes).
 */
int			vb_text_to_rows_batch(int elem, int32_t typmod, int64_t n, const char *text, const int64_t *off, int64_t cap,
								  int64_t *out_row_off, void *out, int64_t *out_bad);
int			vb_text_to_rows_batch_dev(int elem, int32_t typmod, int64_t n, const char *text_dev, const int64_t *off_dev,
									  int64_t cap, int64_t *out_row_off_dev, void *out_dev, int64_t *out_bad);
int			vb_text_to_sparsevec_batch(int32_t typmod, int64_t n, const char *text, const int64_t *off, int64_t cap,
									   int32_t *out_dim, int64_t *out_row_off, int32_t *out_idx, float *out_val,
									   int64_t *out_bad);
int			vb_text_to_sparsevec_batch_dev(int32_t typmod, int64_t n, const char *text_dev, const int64_t *off_dev,
										   int64_t cap, int32_t *out_dim_dev, int64_t *out_row_off_dev, int32_t *out_idx_dev,
										   float *out_val_dev, int64_t *out_bad);
int			vb_rows_to_text_batch(int elem, int dim, const void *rows, int64_t n, int64_t cap, int64_t *out_off, char *out);
int			vb_rows_to_text_batch_dev(int elem, int dim, const void *rows_dev, int64_t n, int64_t cap, int64_t *out_off_dev,
									  char *out_dev);
int			vb_sparsevec_to_text_batch(int dim, int64_t n, const int64_t *row_off, const int32_t *idx, const float *val,
									   int64_t cap, int64_t *out_off, char *out);
int			vb_sparsevec_to_text_batch_dev(int dim, int64_t n, const int64_t *row_off_dev, const int32_t *idx_dev,
										   const float *val_dev, int64_t cap, int64_t *out_off_dev, char *out_dev);

/* ------------------------------------------------------------ binary input and output */

/*
 * The binary type I/O over a column, what COPY ... (FORMAT binary) and binary bind parameters run: vector_recv /
 * vector_send (src/vector.c:376-422), halfvec_recv / halfvec_send (src/halfvec.c:43-72, 373-419, elem = VB_HALFVEC),
 * sparsevec_recv / sparsevec_send (src/sparsevec.c:514-585).  Values, bytes and error texts are the reference's.
 *
 * Payloads.  Field i is bytes[off[i] .. off[i + 1]), the bytes the server hands the receive function (no length word;
 * a zero byte is data; any alignment; NULL fields are not in the batch).  vector / halfvec: uint16 dim, uint16 unused,
 * then dim big-endian float4 (halfvec: binary16 bits); sparsevec: int32 dim, nnz and unused, nnz 0-based int32
 * indices, then nnz float4 values.
 *
 * Receive.  Each field is decoded in the reference's order: the header reads, CheckDim, (sparsevec: CheckNnz),
 * CheckExpectedDim, unused != 0, then element by element the read and CheckElement (sparsevec: every index read and
 * CheckIndex, then every value read, CheckElement and the zero check).  A read past the end of the field fails where it
 * happens with PostgreSQL's "insufficient data left in message"; bytes left over after a good decode fail with COPY's
 * "incorrect binary data format".  A failing call (VB_EINVAL) raises the error row-by-row execution raises first: the
 * lowest failing field, within it the first step above.  vb_last_error() is the errmsg, vb_last_error_detail() is "",
 * *out_bad (may be NULL) the failing field's index (-1 otherwise); the rows are then unspecified.
 *
 * Sizes.  The bound of a field is max(0, (len - 4) / esz) elements (esz 4 or 2), sparsevec max(0, (len - 12) / 8)
 * entries; a field that decodes has exactly its bound, so out_row_off [n + 1], always written, is final from the
 * offsets alone.  A bound total above cap fails naming the total and writes nothing else; out = NULL (sparsevec: idx and
 * val) with cap 0 sizes.  Dense rows are packed at out_row_off (with a typmod, the n x typmod block
 * vb_table_append_dev takes); sparsevec gives the CSR the sparse table calls take and every field's dim in out_dim [n].
 *
 * Send.  Rows are written byte for byte as the reference's send writes them, bits unchanged (-0, subnormals, inf and
 * NaN payloads: send checks nothing); dense rows are n x dim, dim <= 65535.  out_off [n + 1] is always written; a total
 * above cap fails naming it, out = NULL sizes.  sparsevec rows (offsets from 0) are first checked as
 * vb_sparsevec_to_text_batch checks them, with the same texts and "(row r)".
 *
 * Host variants stream through the pinned staging of the text calls in chunks of at most 64 MiB of payload (one larger
 * field or row makes a chunk of its own).  Since sizes follow from the offsets, receive and dense send pipeline: the
 * host stages chunk c + 1 and copies out chunk c - 1 while chunk c runs.  sparsevec send runs its chunks one after
 * another (each reads back its CSR check).  _dev variants take device pointers (out_bad and cap stay host values) and
 * run on vb_stream(); what they read back is listed in the conventions above.  Receive and sparsevec send synchronise;
 * vb_rows_to_binary_batch_dev only enqueues.
 */
int			vb_binary_to_rows_batch(int elem, int32_t typmod, int64_t n, const void *bytes, const int64_t *off, int64_t cap,
									int64_t *out_row_off, void *out, int64_t *out_bad);
int			vb_binary_to_rows_batch_dev(int elem, int32_t typmod, int64_t n, const void *bytes_dev, const int64_t *off_dev,
										int64_t cap, int64_t *out_row_off_dev, void *out_dev, int64_t *out_bad);
int			vb_binary_to_sparsevec_batch(int32_t typmod, int64_t n, const void *bytes, const int64_t *off, int64_t cap,
										 int32_t *out_dim, int64_t *out_row_off, int32_t *out_idx, float *out_val,
										 int64_t *out_bad);
int			vb_binary_to_sparsevec_batch_dev(int32_t typmod, int64_t n, const void *bytes_dev, const int64_t *off_dev,
											 int64_t cap, int32_t *out_dim_dev, int64_t *out_row_off_dev,
											 int32_t *out_idx_dev, float *out_val_dev, int64_t *out_bad);
int			vb_rows_to_binary_batch(int elem, int dim, const void *rows, int64_t n, int64_t cap, int64_t *out_off, void *out);
int			vb_rows_to_binary_batch_dev(int elem, int dim, const void *rows_dev, int64_t n, int64_t cap,
										int64_t *out_off_dev, void *out_dev);
int			vb_sparsevec_to_binary_batch(int dim, int64_t n, const int64_t *row_off, const int32_t *idx, const float *val,
										 int64_t cap, int64_t *out_off, void *out);
int			vb_sparsevec_to_binary_batch_dev(int dim, int64_t n, const int64_t *row_off_dev, const int32_t *idx_dev,
											 const float *val_dev, int64_t cap, int64_t *out_off_dev, void *out_dev);

/* ------------------------------------------------------------ ordering by value */

/*
 * The btree operator classes vector_ops, halfvec_ops and sparsevec_ops (sql/vector.sql:397, 810, 1180) over a resident
 * table: ORDER BY v, SELECT DISTINCT v, GROUP BY v, the tuplesort of CREATE [UNIQUE] INDEX ON t (v), and the lookups
 * WHERE v = $1, v IN (...), v < / <= / >= / > $1.
 *
 * Comparators.  Rows are ordered by the reference's comparator of their type:
 *   vector, halfvec  element by element with < and > on float (halfvec: on HalfToFloat4), the dimension deciding only
 *                    after that (vector_cmp_internal, src/vector.c:1030-1052; halfvec_cmp_internal, src/halfvec.c:987).
 *                    Every row of a table has its dimension, so -0 and +0 are equal and +-inf are ordinary values.
 *   sparsevec        sparsevec_cmp_internal (src/sparsevec.c:1153-1188).  For rows of one dimension it is the
 *                    lexicographic order of 64-bit keys, one per stored entry (i, v): v < 0: (i << 32) | f(v), otherwise
 *                    (2 << 62) | ((2^30 - 1 - i) << 32) | f(v), each row ending with the key 1 << 62, where f is the
 *                    order-preserving map of fp32 bits with -0 made +0.  Exact with stored zeros and +-inf.
 * Ties: equal rows are ordered by ascending row number (tuplesort gives no stable order; this one is deterministic).
 * NaN: the reference's input functions refuse it, device rows can hold it.  A row containing NaN does not fail the
 * call, which still returns a permutation, but where such a row lands is unspecified.
 *
 * Results.  perm [n]: row numbers in order.  A group is a maximal run of equal rows in the order; groups are numbered
 * 0, 1, ... ascending, so group_of_row [n] is the dense rank of each row's value -- the group_of_row vb_table_aggregate
 * takes, which makes GROUP BY v two calls.  group_start [groups + 1]: the position in perm of each group's first row,
 * group_start[groups] = n.  DISTINCT v is perm[group_start[g]] for each g (the smallest row number of each group);
 * count(*) of group g is group_start[g + 1] - group_start[g].  ORDER BY v LIMIT k is perm[0 .. k).
 *
 * Bounds.  For each query q, lo = the number of ordered rows < q and hi = the number <= q; the rows equal to q are
 * perm[lo .. hi), which serves all five btree strategies.  Queries have the table's dimension (dense: packed rows of
 * dim elements; sparse: CSR as the sparse calls take it, a q_dim other than the table's fails with CheckDims' text,
 * "different sparsevec dimensions %d and %d").
 *
 * Lifetime.  An order covers the rows its table held at creation (vb_order_rows); rows appended later are not in it
 * and it stays valid, since row numbers do not move.  Bounds read the rows through the table's current buffers, so a
 * table that grew still works.  Bounds on an order whose table was freed fail with VB_EINVAL, and so does a dense order
 * given to a sparse bounds call or the reverse; reads need only the order.
 *
 * Refusals and failure.  A bit table fails with VB_EINVAL (pgvector has no btree operator class for bit; bit columns
 * use PostgreSQL's bit_ops), and so does a table of 2^31 rows or more (group_of_row is int32).  Everything is validated
 * before any launch; on any error nothing is written to the outputs.  VB_ENOMEM names the bytes needed and leaves
 * nothing allocated.  n = 0 gives an empty order with 0 groups.
 *
 * Synchronisation.  Creation synchronises: the sort is host-driven and reads back one 16-byte count per refinement
 * pass (vb_order_passes: at most the key length + 1, that is dim + 1 for vector, about dim / 2 + 1 for halfvec and
 * max nnz + 2 for sparsevec; a table of identical rows takes at most 2).  vb_order_read and the host bounds calls
 * synchronise; vb_order_read_dev and vb_order_bounds_dev are asynchronous on vb_stream() and use no workspace (they can
 * be captured into a CUDA graph); vb_sparse_order_bounds_dev reads its CSR check first (see the conventions above).
 * Each output of vb_order_read may be NULL.
 */
typedef struct vb_order vb_order;
int			vb_table_order_create(vb_table *t, vb_order **out);	/* VB_VECTOR / VB_HALFVEC tables */
int			vb_sparse_table_order_create(vb_sparse_table *t, vb_order **out);
int64_t		vb_order_rows(const vb_order *o);		/* rows ordered: the table's row count at creation */
int64_t		vb_order_groups(const vb_order *o);		/* distinct values */
int64_t		vb_order_passes(const vb_order *o);		/* refinement passes the sort took */
int			vb_order_read(const vb_order *o, int64_t *perm, int32_t *group_of_row, int64_t *group_start);
int			vb_order_read_dev(const vb_order *o, int64_t *perm_dev, int32_t *group_of_row_dev, int64_t *group_start_dev);
int			vb_order_bounds(vb_order *o, const void *queries, int64_t nq, int64_t *out_lo, int64_t *out_hi);
int			vb_order_bounds_dev(vb_order *o, const void *queries_dev, int64_t nq, int64_t *out_lo_dev, int64_t *out_hi_dev);
int			vb_sparse_order_bounds(vb_order *o, int q_dim, int64_t nq, const int64_t *q_off, const int32_t *q_idx,
								   const float *q_val, int64_t *out_lo, int64_t *out_hi);
/* device CSR checked as in the other sparse _dev calls */
int			vb_sparse_order_bounds_dev(vb_order *o, int q_dim, int64_t nq, const int64_t *q_off_dev, const int32_t *q_idx_dev,
									   const float *q_val_dev, int64_t *out_lo_dev, int64_t *out_hi_dev);
int			vb_order_free(vb_order *o);

/* ---------------------------------------------------------------- IVFFlat */

typedef struct vb_ivf vb_ivf;	/* device image of one ivfflat index: centres + rows grouped by list + ids */

/* metric = the opclass's proc 1: VB_L2_SQUARED, VB_NEG_IP (ip and cosine opclasses) or VB_HAMMING. */
int			vb_ivf_create(int elem, int metric, int dim, int lists, vb_ivf **out);
/*
 * Load the whole image from host memory: centres [lists], rows grouped by
 * list with list_offsets [lists+1] (row index prefix), ids [n] (heap TIDs).
 * This is what the packer produces from the list pages / entry pages
 * (src/ivfflat.h:251-277; readers src/ivfscan.c:62-107, 139-179).
 */
int			vb_ivf_load(vb_ivf *ix, const void *centers, const int64_t *list_offsets,
						const void *rows, const int64_t *ids);
/* Same, from device buffers (packed rows; ids may be NULL = row positions). */
int			vb_ivf_load_dev(vb_ivf *ix, const void *centers_dev, const int64_t *list_offsets_host,
							const void *rows_dev, const int64_t *ids_dev);
int64_t		vb_ivf_rows(const vb_ivf *ix);
/*
 * The same image, one list at a time -- the granularity the packer reads at (one entry-page chain per list,
 * src/ivfscan.c:139-179), so the host never stages more than one list: vb_ivf_begin_load (centres), vb_ivf_load_list
 * for the non-empty lists in ascending list order, vb_ivf_end_load.
 * vb_ivf_replace_list swaps one list of a loaded image for new contents (an insert into that list, a vacuum of it):
 * only that list crosses PCIe, the rows behind it are moved on the device, and the packed planes of the tensor-core
 * filter are rebuilt on the device by the next batched scan.
 */
int			vb_ivf_begin_load(vb_ivf *ix, const void *centers);
int			vb_ivf_load_list(vb_ivf *ix, int list, const void *rows, const int64_t *ids, int64_t n);
int			vb_ivf_end_load(vb_ivf *ix);
int			vb_ivf_replace_list(vb_ivf *ix, int list, const void *rows, const int64_t *ids, int64_t n);
/*
 * In-place inserts and deletes (ivfflatinsert, ivfflatbulkdelete) on a loaded image, without reloading or repacking it.
 *
 * vb_ivf_insert is InsertTuple (src/ivfinsert.c:72-181) for each of the n rows, in call order.  Row i goes to the list
 * FindInsertPage picks (support-1 distance to every centre, a running minimum that starts at list 0 and moves only on a
 * strict <): for every row that is vb_ivf_scan_lists(row, 1) on the same image, except that a row whose distance to
 * centre 0 is NaN (vector_ip_ops with elements near 1e38) stays in list 0.  out_lists[i] receives it.  Each row is
 * appended at the end of its list, rows of one call in call order: the reference's placement whenever the list's insert
 * page is its last page (after a build, a load, and any number of inserts).  After a VACUUM freed space on an earlier
 * page the AM fills that space first; a caller that needs that position replaces the list (vb_ivf_replace_list).
 * Position only decides exact ties, which list scans break by (distance, scan position).  Rows come as stored (cosine
 * opclasses pass l2-normalised rows, as vb_ivf_load takes them); ids are the rows' heap TIDs and must not be NULL.
 * vb_ivf_insert_dev takes device rows and ids; its out_lists (host) may be NULL.
 *
 * vb_ivf_delete is ivfflatbulkdelete (src/ivfvacuum.c:18-143): every row whose heap id is in ids[0 .. n) is removed, ids
 * the image does not hold are ignored, survivors keep their order within each list, and *out_removed (may be NULL) is
 * the reference's tuples_removed.  Lists may become empty.
 *
 * vb_ivf_list_offsets copies the image's list offsets, [lists + 1].
 *
 * Only the rows from the first changed one onward move, in place, and the derived state (list offsets, the packed
 * planes of the tensor-core filter where they were built, and the norm bounds its certificates use) is brought up to
 * date on the device; the centre planes are untouched.  A loaded table has no headroom: the first insert grows it by
 * half again (the growth allocates the new table beside the old one, releasing the packed planes first when both do
 * not fit beside them; the next batched scan rebuilds them).  A call that changes rows bumps the image's generation, as
 * vb_ivf_replace_list does: row filters and iterative scan handles made before it fail with VB_ESTATE.  n == 0 does
 * nothing.  An image that is not loaded, or was loaded without ids, fails with VB_ESTATE; a NULL pointer with
 * VB_EINVAL.  After VB_EINVAL or VB_ENOMEM (whose message names the bytes) the image is as it was: the call validates,
 * reserves and allocates before any row moves.  A CUDA error after rows started moving leaves the image unloaded (later
 * calls get VB_ESTATE until the next load).  Images of the list-sharded search (vb_ivf_search_sharded) are not
 * supported.
 */
int			vb_ivf_insert(vb_ivf *ix, const void *rows, const int64_t *ids, int64_t n, int32_t *out_lists);
int			vb_ivf_insert_dev(vb_ivf *ix, const void *rows_dev, const int64_t *ids_dev, int64_t n,
							  int32_t *out_lists /* host, may be NULL */ );
int			vb_ivf_delete(vb_ivf *ix, const int64_t *ids, int64_t n, int64_t *out_removed);
int			vb_ivf_list_offsets(const vb_ivf *ix, int64_t *out /* [lists + 1] */ );
int			vb_ivf_free(vb_ivf *ix);

/*
 * GetScanLists (src/ivfscan.c:47-118): distance from each query to every
 * centre, nearest max_probes lists, ascending.  Ties: smaller list number first.
 * out_lists [nq x max_probes] (int32), out_dist [nq x max_probes] (may be NULL).
 */
int			vb_ivf_scan_lists(vb_ivf *ix, const void *queries, int64_t nq, int max_probes,
							  int32_t *out_lists, double *out_dist);
/*
 * GetScanItems (src/ivfscan.c:123-187) for ONE query: distance to every row of
 * the given lists, fully sorted ascending (tuplesort_performsort, :182).  Writes
 * at most cap results, *n_out = number of candidates scanned.  Ties: scan order.
 * q == NULL: all distances 0 (src/ivfscan.c:207-211).
 */
int			vb_ivf_scan_items(vb_ivf *ix, const void *q, const int32_t *lists, int nlists,
							  int64_t cap, int64_t *out_ids, double *out_dist, int64_t *n_out);
/*
 * The whole first batch of ivfflatgettuple (src/ivfscan.c:360-414) for nq
 * queries at once: probe selection + list scan + top-k (k nearest of the
 * probed lists; k <= 0 is rejected here, use vb_ivf_scan_items for "all").
 * Host buffers; copies are inside the call.
 */
int			vb_ivf_search(vb_ivf *ix, const void *queries, int64_t nq, int probes, int k,
						  int64_t *out_ids, double *out_dist);
/* Same with device-resident queries and outputs (float distances), asynchronous on vb_stream(). */
int			vb_ivf_search_dev(vb_ivf *ix, const void *queries_dev, int64_t nq, int probes, int k,
							  int64_t *out_ids_dev, float *out_dist_dev);
/*
 * vb_ivf_search with a row filter per query (see vb_filter above): the plan of WHERE <predicate> ORDER BY v <op> q
 * LIMIT k with ivfflat.iterative_scan = off, for a batch of queries.
 *
 * Result.  Query q uses filters[filter_of_query[q]]; filter_of_query is a host array in both variants, NULL when
 * nfilters == 1.  For each query the result is the first k rows of vb_ivf_search's order over its probed lists (by
 * (distance, scan position); the lists are those of vb_ivf_scan_lists(q, probes)) restricted to the ids its filter
 * allows, padded with -1 / +inf when fewer than k allowed rows lie in the probed lists (where the reference returns
 * fewer rows).  An allowed row whose distance is +inf or NaN is a result, in that order's place; a rejected row never is.
 *
 * Bit identity.  An allowed row gets bit for bit the distance vb_ivf_search computes for it on the same path, so with a
 * filter that allows every row the output equals vb_ivf_search's, ids and distances, under every scan_impl, tc_level1
 * and tc_level0.  The filtered call never takes the fused one-query kernels: for calls of at most 16 queries, the
 * comparison is with vb_ivf_search under option one_query = 0.
 *
 * Reads.  Unlike the other filtered calls this one reads rejected rows: the probed lists are read whole, once per batch,
 * because the queries of a batch share them, and each query's candidate distances are masked (VB_PROF_FILTER_MASK)
 * before anything selects from them.  Rejected rows are never selected, re-scored or returned.  For very selective
 * filters, vb_exact_topk_filtered (the exact scan of the allowed rows) or the filtered iterative scan
 * (vb_ivf_scan_begin_filtered), which read the allowed rows only, move fewer bytes.
 *
 * Errors.  An index that is not loaded: VB_ESTATE.  A filter of another table, index or image, also after its owner was
 * freed: VB_EINVAL.  A filter made before a load, vb_ivf_replace_list, vb_ivf_insert or vb_ivf_delete: VB_ESTATE ("index
 * changed since the filter was created").  A filter_of_query entry out of range: VB_EINVAL naming the query.  k and
 * probes have the limits of vb_ivf_search; VB_ENOMEM names the bytes.  The host variant writes nothing on any error.
 * Images of the list-sharded search are not supported.  The filters may be freed once the call returns.
 */
int			vb_ivf_search_filtered(vb_ivf *ix, const void *queries, int64_t nq, int probes, int k,
								   const vb_filter *const *filters, int nfilters, const int32_t *filter_of_query,
								   int64_t *out_ids, double *out_dist);
int			vb_ivf_search_filtered_dev(vb_ivf *ix, const void *queries_dev, int64_t nq, int probes, int k,
									   const vb_filter *const *filters, int nfilters, const int32_t *filter_of_query,
									   int64_t *out_ids_dev, float *out_dist_dev);
/*
 * Pipelined host path.  vb_ivf_prefetch_queries starts the host->device copy of the NEXT batch of queries on a second
 * stream (slot 0 or 1; `queries` should be page-locked and must stay valid until the matching search returns) and
 * returns at once; vb_ivf_search_prefetched runs the search of a slot filled earlier (same results as vb_ivf_search)
 * and returns when its results are in `out_ids` / `out_dist`.  Alternating the two slots overlaps every copy with the
 * previous batch's compute.  vector queries with dim % 4 == 0 only; VB_EINVAL otherwise.
 */
int			vb_ivf_prefetch_queries(vb_ivf *ix, const void *queries, int64_t nq, int slot);
int			vb_ivf_search_prefetched(vb_ivf *ix, int slot, int probes, int k, int64_t *out_ids, double *out_dist);
/*
 * ivfflat.iterative_scan (src/ivfscan.c:123-187 GetScanItems, :252-283 ivfflatbeginscan, :400-406 ivfflatgettuple) for
 * nq queries at once.  The handle owns what IvfflatScanOpaqueData keeps between batches: the probe order, listIndex
 * and the position in the sorted batch.
 *
 * Begin.  p = min(probes, lists) and P = min(max(max_probes, probes), lists), as ivfflatbeginscan clamps them
 * (:268-277); max_probes = probes is iterative_scan = off.  Probe selection runs for P lists per query: the lists and
 * their order are what vb_ivf_scan_lists(q, P) returns (ties by list number).  Queries are host memory; begin
 * returns synchronised.  Cosine opclasses: the caller normalises the queries, as for vb_ivf_search.
 *
 * The sequence S_q of a query.  L[0..P) is split into groups of p consecutive lists (the last may be short).  S_q is
 * the concatenation, over the groups in order, of all rows of the group's lists sorted by (distance, scan position),
 * the scan position being the position in the concatenation of the group's lists in probe order, rows in stored
 * order: GetScanItems + tuplesort_performsort + the loop at :400-406.  Distances are the float8 vb_ivf_scan_items
 * reports; ids are the heap ids given at load, or row positions when those were NULL.
 *
 * Next.  Per query, the next <= page elements of S_q go to out_ids / out_dist [nq x page] (-1 / +inf padded) and
 * their number to out_counts[q].  A page never spans two groups: a query whose group ran dry moves to its next
 * non-empty group within the same call (empty lists and groups are skipped as the reference's while loop skips
 * them).  out_counts[q] == 0 if and only if S_q is exhausted, and stays 0.  Queries progress independently: in one
 * call some may still drain group 0 while others start group 3.  vb_ivf_scan_lists_done writes the reference's
 * so->listIndex per query [nq]: 0 before the first next, P once the sequence is exhausted.
 *
 * Limits.  1 <= page <= 2048 (the selection stays on the device), probes >= 1, max_probes >= 1, nq >= 1, queries not
 * NULL (NULL-query scans keep vb_ivf_scan_items, as for vb_ivf_search), the index loaded: VB_EINVAL / VB_ESTATE and a
 * message otherwise.
 *
 * State.  Everything a handle keeps between calls lives in device memory it owns, so other searches or handles between
 * two next calls do not change a sequence.  Begin allocates per query the query image, P probe slots, the group's
 * candidate distances (as many as the p longest lists hold), group lists and offsets, the cursor and the page staging, plus the scan chunk
 * descriptors; when that does not fit next to the index it fails with VB_ENOMEM, names the bytes per query and
 * allocates nothing.  next allocates nothing.  vb_ivf_load*, vb_ivf_begin_load, vb_ivf_end_load and
 * vb_ivf_replace_list change the image: next on a handle opened before fails with VB_ESTATE ("index changed since the
 * scan began") and writes nothing.  end always succeeds; end every handle before vb_ivf_free.
 *
 * Equivalence with the per-scan path.  For every query, S_q is bit-identical in ids and distances to what successive
 * vb_ivf_scan_items(q, L[g p ..], cap = all) calls return when those calls score with scan_kernel's per-row arithmetic:
 * the fused one-query kernels (the default for one query) and option scan_impl = 0.  The handle therefore always
 * scores with that arithmetic (the LDG chunk scan), whatever scan_impl says.  The bulk-copy scan (scan_bulk_kernel,
 * scan_impl 1, or 2 on tables above 50 MB) is not bit-identical in general: it splits every row over 32 lanes where
 * the LDG scan uses fewer for rows narrower than 512 bytes, and it scores halfvec rows against a half-precision query
 * image; for vector and bit rows of 512 bytes and more the two follow the same per-lane order.  The list-major and
 * tensor-core formulations of vb_ivf_search are not used here: a filter cannot certify a full order, and list-major
 * distances differ in the last bits.  This is what lets a caller serve the first pages of a request from a batch and
 * the rest per scan without a visible difference.
 */
typedef struct vb_ivf_scan vb_ivf_scan;
int			vb_ivf_scan_begin(vb_ivf *ix, const void *queries, int64_t nq, int probes, int max_probes, int page,
							  vb_ivf_scan **out);
/*
 * The same scan with a row filter per query (see vb_filter above): query q uses filters[filter_of_query[q]] (host
 * array; NULL when nfilters == 1; an entry out of range fails with VB_EINVAL naming the query).  Its sequence is the
 * subsequence of S_q whose ids the filter allows: same order, same float8 distances bit for bit.  A page never spans
 * two groups; a group with no allowed row is skipped like an empty one, so out_counts[q] == 0 still means exhausted.
 * vb_ivf_scan_lists_done after a page is what the unfiltered handle reports when it returns those rows, and P at
 * exhaustion.  Rows the filter rejects are never read, scored, selected or copied.  Begin copies what it needs from the
 * filters into the handle's own allocation (the filters may be freed at once) and sizes the group buffers by the p
 * largest allowed counts per list; VB_ENOMEM names the bytes the filters take too.  next, lists_done and end are the
 * unfiltered handle's.
 */
int			vb_ivf_scan_begin_filtered(vb_ivf *ix, const void *queries, int64_t nq, int probes, int max_probes, int page,
									   const vb_filter *const *filters, int nfilters, const int32_t *filter_of_query,
									   vb_ivf_scan **out);
int			vb_ivf_scan_next(vb_ivf_scan *scan, int64_t *out_ids, double *out_dist, int32_t *out_counts);
int			vb_ivf_scan_lists_done(vb_ivf_scan *scan, int32_t *out);	/* [nq]: the reference's so->listIndex */
int			vb_ivf_scan_end(vb_ivf_scan *scan);
/* algorithmic bytes of the last vb_ivf_search*: sum over queries of (lists + candidates) * dim * elem size (SURVEY 8d) */
int64_t		vb_ivf_last_scan_bytes(const vb_ivf *ix);
int64_t		vb_ivf_last_candidates(const vb_ivf *ix);
/* Queries (cumulative) whose tensor-core filter result could not be certified against the error bound and were
 * re-run on the exact fp32 kernel (option "scan_impl" = 4); 0 when that path is not in use. */
int64_t		vb_ivf_tc_fallbacks(const vb_ivf *ix);
/* Queries (cumulative) the first filter level (hi plane of the rows only, option "tc_level1") could not certify; their
 * batches were repeated with both planes.  After such a batch the level rests for 64 batches. */
int64_t		vb_ivf_tc_level1_fallbacks(const vb_ivf *ix);
/* Queries (cumulative) filter level 0 (int8 rows, option "tc_level0") could not certify.  Only those queries were
 * searched again, from level 1 on; level 0 rests for 64 batches after one whose failed queries probe, in expectation,
 * more than a quarter of the lists (1 - (1 - probes / lists)^failed > 1/4), where the re-run costs more than level 0 saved. */
int64_t		vb_ivf_tc_level0_fallbacks(const vb_ivf *ix);
/* Queries (cumulative) filter level P (a lower bound from the rows' projection on their principal directions, option
 * "tc_levelp") could not certify.  Only those queries were searched again, from level 0 on; level P rests for 64 batches
 * after one whose failed queries probe, in expectation, more than half of the lists. */
int64_t		vb_ivf_tc_levelp_fallbacks(const vb_ivf *ix);

/*
 * Traffic accounting of the tensor-core filter kernel (profiling, off by default): with on != 0 every launch also
 * sums, from the job list the kernel walks, the bytes its bulk copies request and the distinct bytes among them.
 * out8 (may be NULL): read and reset the counters -- list scan [0] bytes requested, [1] distinct row-plane bytes,
 * [2] distinct query-tile bytes, [3] launches; [4..7] the same for the centre scan (probe selection).
 */
int			vb_ivf_tc_traffic(int on, int64_t *out8);
/*
 * Counters of the level-0 refine, kept while traffic accounting is on: read and reset into out3 -- [0] rows re-scored
 * exactly (per-row bounds), [1] rows the global bound (d~ <= k-th d~ + 2 eps(q)) would have re-scored, [2] queries refined.
 */
int			vb_ivf_tc_level0_rescored(int64_t *out3);

/*
 * List-sharded search over the library's communicator (vb_comm_init): this rank's image holds its own lists under
 * the GLOBAL list numbering (every other list empty) and all centres.  Probe selection runs on this rank's slice of
 * the queries, the probe lists are all-gathered, every rank scans its lists for all queries, the per-rank k nearest
 * are all-gathered and merged by (distance, id).  All ranks call it with the same queries and get the full result.
 * Device pointers; asynchronous on vb_stream() apart from one read of the filter's certificate counters.
 */
int			vb_ivf_search_sharded_dev(vb_ivf *ix, const void *queries_dev, int64_t nq, int probes, int k,
									  int64_t *out_ids_dev, float *out_dist_dev);
/* The same with host buffers (queries in, int64 ids + float8 distances out; copies inside, synchronous). */
int			vb_ivf_search_sharded(vb_ivf *ix, const void *queries, int64_t nq, int probes, int k,
								  int64_t *out_ids, double *out_dist);

/*
 * Exact (no index) top-k over a row-sharded table: every rank scans its own rows (vb_exact_topk_dev), the per-rank k
 * nearest are all-gathered and merged by (distance, id).  id_offset = the global number of this rank's first row.
 * Collective; every rank gets the full result.
 */
int			vb_exact_topk_sharded_dev(vb_table *t, int metric, const void *queries_dev, int64_t nq, int k, int64_t id_offset,
									  int64_t *out_ids_dev, float *out_dist_dev);

/* --------------------------------------------------------------- communicator */

/*
 * One process per GPU.  vb_comm_unique_id (on one rank) fills the 128-byte NCCL id the host passes to the others
 * (the extension: through its DSM segment, like the reference's parallel-build state, src/ivfbuild.c:830-966);
 * vb_comm_init (every rank, collectively) creates the communicator on the library's device.  While it exists,
 * vb_kmeans / vb_kmeans_pp_init treat `samples` as this rank's slice of a row-sharded sample set (centre sums,
 * counts, the change counter, k-means++ weight sums and chosen rows are exchanged with ncclAllReduce /
 * ncclAllGather on vb_stream()), and vb_ivf_search_sharded_dev is available.  dtype: 0 fp32, 1 int32, 2 int64,
 * 3 fp64, 4 uint32.
 */
int			vb_comm_unique_id(void *out, size_t cap);
int			vb_comm_init(const void *id_bytes, int rank, int world);
int			vb_comm_free(void);
int			vb_comm_world(void);
int			vb_comm_rank(void);
int			vb_comm_allreduce(void *buf_dev, int64_t count, int dtype);
int			vb_comm_allgather(const void *send_dev, void *recv_dev, int64_t bytes_per_rank);

/* ------------------------------------------------------- IVFFlat build path */

/*
 * Collective hook for the sharded build: sum-reduce `count` elements of the
 * given device buffer in place across all ranks (dtype 0 = fp32, 1 = int32,
 * 2 = int64).  The extension passes an ncclAllReduce wrapper; tests pass a
 * torch.distributed one.  NULL = single process.
 */
typedef int (*vb_allreduce_fn) (void *buf_dev, int64_t count, int dtype, void *ctx);

/*
 * k-means on samples resident in `samples` (this rank's shard), replacing
 * ElkanKmeans (src/ivfkmeans.c:246-485) from given initial centres
 * (centres = in/out host buffer of k rows; k-means++ draws are host-side,
 * see vb_kmeans_pp_init).  kmeans_metric: VB_L2 (l2 opclasses), VB_SPHERICAL
 * (ip / cosine opclasses; samples must already be unit vectors,
 * src/ivfbuild.c:153-155) or VB_HAMMING (bit).  Lloyd iterations with a dense
 * assign step; centre update and stopping rule as src/ivfkmeans.c:179-236,
 * 482-483.  *iters_out = iterations executed.
 */
int			vb_kmeans(vb_table *samples, int kmeans_metric, void *centers, int k, int max_iter,
					  uint64_t seed, vb_allreduce_fn allreduce, void *allreduce_ctx, int *iters_out);
/* InitCenters (src/ivfkmeans.c:23-91): k-means++ seeding on the device, centres out (host). */
int			vb_kmeans_pp_init(vb_table *samples, int kmeans_metric, void *centers, int k, uint64_t seed);
/*
 * Same with the caller's random draws (the extension passes pg_prng's, the parity tests the oracle's): the first
 * centre is sample first_row (RandomInt() % numSamples, src/ivfkmeans.c:36); u[i], i < k - 1, is the RandomDouble()
 * of round i (src/ivfkmeans.c:78).  picked_out (may be NULL): the k chosen sample rows.
 */
/*
 * On large fp32 sample tables the seeding touches a sample only when its weight could change (triangle inequality over
 * the chosen centres, then a bf16 lower bound; exact fp32 re-score for the rest -- the weights and the picks are
 * those of the full pass).  out3: samples skipped by the triangle rule / stopped by the bf16 bound / re-scored
 * exactly during the last seeding of this process (all zero when the plain pass ran).  Option "pp_filter": 0 = never,
 * 1 = automatic (default), 2 = always.
 */
int			vb_kmeans_pp_stats(int64_t *out3);
int			vb_kmeans_pp_init_draws(vb_table *samples, int kmeans_metric, void *centers, int k, int64_t first_row,
									const double *u, int64_t *picked_out);
/*
 * AddTupleToSort's argmin (src/ivfbuild.c:161-219): out_list[i] = first centre
 * minimising the proc-1 distance (strict <).  metric = VB_L2_SQUARED / VB_NEG_IP / VB_HAMMING.
 */
int			vb_assign(vb_table *rows, int metric, const void *centers, int k, int32_t *out_list);
int			vb_assign_dev(vb_table *rows, int metric, const void *centers_dev, int k, int32_t *out_list_dev);
/*
 * The assign step runs on the tensor cores (wgmma, split-bf16 GEMM with a fused row argmin)
 * and re-checks rows whose best/second-best margin is inside the error bound with the exact
 * fp32 kernel.  vb_set_tensor_cores(0) forces the exact CUDA-core kernel for everything
 * (used by the parity tests); vb_last_assign_rechecked() = rows the last assign re-checked
 * (-1 when the exact kernel did all the work).
 */
int			vb_set_tensor_cores(int on);
int64_t		vb_last_assign_rechecked(void);
/*
 * Tuning switches.  "scan_impl" selects the list / table scan: 0 = per-query LDG.128 streaming kernel,
 * 1 = per-query cp.async.bulk (TMA) + mbarrier staged kernel for rows of at least 512 bytes, 2 (default) =
 * automatic (query batches are scanned list-major: each probed list read once per batch, fp32x2 register
 * tiles; single queries stream), 3 = list-major wherever it applies, 4 = tensor-core filter (split-bf16
 * tensor-core distances, exact fp32 re-score of k' candidates, certificate, exact fallback) wherever it applies.
 * Every setting returns the same neighbours.  "tc_level1" (default 1): the tensor-core filter first reads only the
 * hi plane of the rows (half the HBM traffic, 2^-7 relative error bound) and repeats a batch with both planes when a
 * certificate fails.  "tc_level0" (default 1, effective where "tc_level1" is on): batched searches (vb_ivf_search*,
 * not the sharded one) start one level lower, at int8 rows (a quarter of the bf16 planes' bytes, bound ~ max |x - x^| |q|,
 * k' = 128); only the queries it cannot certify are searched again, from level 1 on.  "tc_levelp" (default 1, effective
 * where "tc_level0" is on, fp32 rows with L2 distance): in front of level 0, the bound |x - q|^2 >= |P(x - q)|^2 / sigma^2
 * with P the top principal directions of a row sample (r of them, a multiple of 16 holding 90 % of its energy, at most
 * dim / 8; no level P where none does) reads 4 r bytes a row; only the queries it cannot certify are searched again, from
 * level 0 on.  It is taken with scan_impl 2, for batches of at least 256 queries over at least 128 lists, where the int8
 * bytes it saves exceed the fp32 rows its looser bound adds to the refine.  "tensor_cores" as vb_set_tensor_cores.  "one_query" (default 1): calls with at most 16 queries --
 * one backend's scan: vb_ivf_scan_lists, vb_ivf_scan_items, vb_ivf_search -- run as two fused distance + select
 * kernels (the last CTA to finish selects; csrc/vb_ivf_one.cu) instead of the general launch sequence; 0 = general path.
 */
int			vb_set_option(const char *name, int64_t value);

/*
 * CREATE INDEX ... USING ivfflat in one call (ivfflatbuild, src/ivfbuild.c): the n rows of the call become a resident,
 * searchable image of `ix` (made by vb_ivf_create; any element type and metric it accepts).  The call composes the
 * entry points above -- it equals them bit for bit on the same samples and draws -- and adds what lay between them:
 *
 *   samples   SampleRows (src/ivfbuild.c:132-156).  opts->sample_rows, in the caller's order, or n_samples distinct rows
 *             drawn on the device: row numbers perm(0 .. n_samples - 1) of a 4-round Feistel permutation of [0, 2^b)
 *             keyed by the seed (b even, 2^b >= n), cycle-walked into [0, n) -- a bijection, so the draws are distinct
 *             without a table of size n -- and sorted ascending.  The reference's block sampler and reservoir are
 *             PRNG-driven and not reproduced; parity is defined from shared sample_rows / first_row / u.  The k-means
 *             metric follows the opclass: VB_L2 (L2 squared), VB_SPHERICAL (negative inner product, i.e. the ip and the
 *             cosine opclasses), VB_HAMMING (bit).  Spherical: samples of norm 0 are dropped and the others
 *             l2-normalised (vb_l2_normalize_batch's arithmetic), keeping their order, whatever `normalize` says
 *             (AddSample, src/ivfbuild.c:66-73).  Fewer usable samples than lists is VB_EINVAL.
 *   centres   vb_kmeans_pp_init[_draws], then vb_kmeans, on those samples; they become the image's centre table
 *             (vb_ivf_centers reads it back, for CreateListPages).
 *   assign    AddTupleToSort (src/ivfbuild.c:161-219).  normalize != 0 (the cosine opclasses): a row of norm 0 is not
 *             indexed (out_lists[i] = -1) and the others are l2-normalised before the argmin and stored normalised.
 *             out_lists[i] = vb_assign's list of (normalised) row i: the first minimum wins.
 *   place     row i is stored in list out_lists[i], rows of one list in call order (the order a serial heap scan feeds
 *             the tuplesort in; list scans break exact ties by position).  out_order[p], p < vb_ivf_rows(ix), is the
 *             call's row number stored at image row p -- with vb_ivf_list_offsets, what InsertTuples walks -- and -1
 *             from there on.  The image ends as vb_ivf_load leaves it for the same centres, offsets, grouped rows and
 *             ids: generation bumped, packed tensor-core planes released (the next batched scan builds them).
 *
 * vb_ivf_build streams the host rows twice through two pinned staging buffers of chunk_rows rows (0 = 128 MB worth,
 * at least 1024 and at most 2^20 rows; a buffer is chunk_rows * (row bytes + 8) bytes, and exists twice pinned -- kept
 * by the library for later calls -- and twice on the device; caller memory that is already page-locked is read in
 * place), the copy of chunk c + 1 overlapping the
 * work on chunk c: pass one assigns and keeps 4 bytes per row, pass two scatters each chunk's rows to their final image
 * rows.  The device holds one copy of the indexed rows, their ids, 36 bytes per row of list numbers, sort buffers and
 * destinations, the samples, and the chunk buffers.  vb_ivf_build_dev reads the caller's device rows in place (assign,
 * then one gather in image order), so it holds the caller's copy and the image.  Both synchronise before returning.
 *
 * Everything that can be refused without touching the image happens first: arguments (n < 1, n >= 2^31, NULL rows or
 * ids -- an image without ids cannot take inserts --, sample_rows out of range or repeated: VB_EINVAL; an active
 * communicator, whose images are shards: VB_ESTATE), the samples, the k-means and the assign.  After such a failure a
 * loaded image is as it was.  Then the old rows are released, the new table is allocated and the rows are placed: a
 * VB_ENOMEM (its message names the bytes) or CUDA error from there on leaves the image unloaded (VB_ESTATE until the
 * next load or build).  Row filters and scan handles made before a build fail with VB_ESTATE afterwards.
 */
typedef struct vb_ivf_build_opts
{
	uint64_t	seed;			/* sample draw (sample_rows == NULL), k-means++ draws (u == NULL), empty-cluster reseed */
	int			max_iter;		/* Lloyd iterations, 0 = 500 (src/ivfkmeans.c:347) */
	const int64_t *sample_rows;	/* host, [n_samples] row numbers of this call's rows; NULL = drawn by the library */
	int64_t		n_samples;		/* with sample_rows; otherwise 0 = min(n, max(50 * lists, 10000)) (src/ivfbuild.c:448-455) */
	int64_t		first_row;		/* with u: index INTO THE USABLE SAMPLES of the first centre, as vb_kmeans_pp_init_draws */
	const double *u;			/* host, [lists - 1] RandomDouble() draws; NULL = from seed */
	int64_t		chunk_rows;		/* vb_ivf_build: rows per streamed chunk, 0 = automatic */
} vb_ivf_build_opts;

int			vb_ivf_build(vb_ivf *ix, const void *rows, const int64_t *ids, int64_t n, int normalize,
						 const vb_ivf_build_opts *opts /* NULL = defaults, seed 42 */ ,
						 int32_t *out_lists /* host [n], may be NULL */ , int64_t *out_order /* host [n], may be NULL */ ,
						 int *iters_out /* may be NULL */ );
int			vb_ivf_build_dev(vb_ivf *ix, const void *rows_dev, const int64_t *ids_dev, int64_t n, int normalize,
							 const vb_ivf_build_opts *opts, int32_t *out_lists /* host */ , int64_t *out_order /* host */ ,
							 int *iters_out);
/* The centre table of a loaded image: [lists] packed rows of the index's element type, to host memory. */
int			vb_ivf_centers(const vb_ivf *ix, void *out);

/* -------------------------------------------------------------------- HNSW */

typedef struct vb_hnsw vb_hnsw;	/* device image of one hnsw index: element vectors + neighbour tables */

/*
 * metric = opclass proc 1 (VB_L2_SQUARED, VB_NEG_IP, VB_L1, VB_HAMMING, VB_JACCARD).
 * Elements are numbered 0..n-1; levels[n]; nbr0 [n x 2m] layer-0 neighbour
 * element numbers in on-disk order (HnswSetNeighborTuple, src/hnswutils.c:455-486),
 * -1 terminated; upper layers as upper_off[n] (-1 when level 0) and
 * upper [slots x m] with layer lc of element e at slot upper_off[e] + lc - 1.
 * entry = entry point element (meta page, src/hnswutils.c:298-328).
 */
int			vb_hnsw_create(int elem, int metric, int dim, int m, vb_hnsw **out);
int			vb_hnsw_load(vb_hnsw *h, const void *rows, int64_t n, const int32_t *levels,
						 const int32_t *nbr0, const int64_t *upper_off, const int32_t *upper,
						 int64_t upper_slots, int64_t entry);
int			vb_hnsw_free(vb_hnsw *h);
/*
 * CREATE INDEX ... USING hnsw on the device: the in-memory build of src/hnswbuild.c:437-480 --
 * HnswFindElementNeighbors (src/hnswutils.c:1280-1357) with ef_construction, the SelectNeighbors heuristic
 * (:1065-1165), duplicate folding (src/hnswbuild.c:343-364) and HnswUpdateConnection (:1184-1231) -- for rows
 * inserted in batches the way the reference's parallel workers insert concurrently.  Row i becomes element i.
 * levels: the per-row level draws of HnswInitElement (src/hnswutils.c:248-254) when the caller owns the PRNG
 * (the extension passes pg_prng's), NULL = drawn from `seed`.  The index is searchable afterwards (vb_hnsw_search)
 * and vb_hnsw_export returns the graph in the layout vb_hnsw_load takes, for the page writer
 * (HnswSetNeighborTuple, src/hnswutils.c:455-486): levels [n], nbr0 [n x 2m], upper_off [n], upper
 * [vb_hnsw_upper_slots() x m], entry point, and dup_of [n] = the element a duplicate row was folded into (its heap
 * TID joins that element's, HNSW_HEAPTIDS = 10 at most, src/hnsw.h:69) or -1.  Any output may be NULL.
 */
int			vb_hnsw_build(vb_hnsw *h, const void *rows, int64_t n, int ef_construction, uint64_t seed,
						  const int32_t *levels);
int			vb_hnsw_build_dev(vb_hnsw *h, const void *rows_dev, int64_t n, int ef_construction, uint64_t seed,
							  const int32_t *levels);
/*
 * INSERT into a resident image (aminsert = HnswInsertTupleOnDisk, src/hnswinsert.c:696-743), so the image stays valid
 * across inserts and only the changed neighbour slots go to the pages.
 *
 * Element numbers: row i of the call becomes element n_old + i, a duplicate too (as in vb_hnsw_build): out_dup_of[i]
 * (may be NULL) and vb_hnsw_export's dup_of give the element the row was folded into, or -1.  A folded element gets
 * no neighbours and no incoming links.  levels: the caller's draws (the extension takes them from pg_prng), capped at
 * HnswGetMaxLevel(m) as in the build; NULL = drawn from `seed` with the build's expression.
 *
 * Semantics: HnswInsertTupleOnDisk for each row, in batches.  Rows go in in order; rows of one batch do not see each
 * other (the reference's concurrent inserters).  A batch holds at most max(1, graph size / hnsw_build_fraction) rows,
 * at most hnsw_build_batch (vb_set_option), and ends at a row that rises above the entry level; with batches of one
 * row the result is the serial reference insert.  The on-disk rules:
 *   - candidates whose element is being deleted (heap TID count 0) help the search but are removed before
 *     SelectNeighbors (RemoveElements, src/hnswutils.c:1237-1259);
 *   - a row is folded into the first equal layer-0 neighbour, in neighbour order, with 1..9 heap TIDs; 0 (being
 *     deleted) or 10 (full) is skipped (FindDuplicateOnDisk / AddDuplicateOnDisk, src/hnswinsert.c:586-663);
 *   - a neighbour's list that is not full takes the new element in its first free slot; a full list has its distances
 *     recomputed from the neighbour's own row, its first neighbour that is being deleted is replaced, and otherwise
 *     HnswUpdateConnection (src/hnswutils.c:1184-1231) replaces the pruned connection in its slot, or changes nothing
 *     when the new element is the one pruned (GetUpdateIndex, src/hnswinsert.c:409-448).  Stored distances are never
 *     read, so a loaded image and a built one behave alike;
 *   - the entry point moves only to a strictly higher level, never to a folded row; into an empty image the first
 *     row becomes the entry point, with no neighbours.
 * ef_construction is checked as by vb_hnsw_build.
 *
 * Heap TID counts drive RemoveElements, the preference for deleted neighbours and duplicate folding: after
 * vb_hnsw_load every element counts 1, after vb_hnsw_build the build's counts; folds add to them.
 * vb_hnsw_set_heaptid_counts (host [n], 0..10) passes what the glue saw on the pages (0 = being deleted).  The
 * search never reads them.
 *
 * Change records: *out_nchanges (may be NULL) of them; vb_hnsw_insert_changes copies them, sorted by (element, layer,
 * slot): one per neighbour-array slot whose value after the call differs from its value before -- every filled slot
 * of the new elements and every slot UpdateNeighborOnDisk rewrote in an existing element; slot indexes the layer's lm
 * entries (2m at layer 0, m above).  A slot rewritten twice in one call appears once, with its final value: applied
 * to a vb_hnsw_export taken before the call they give exactly the export taken after it.  cap below the count fails
 * with VB_EINVAL, writing nothing.  The records stay valid until the next insert, vacuum, load or build.
 *
 * Growth and failure: the device arrays grow geometrically (the graph is not double-buffered).  Before any kernel
 * runs, the call validates its arguments and reserves capacity, upper slots, record space and visited tables; after
 * VB_EINVAL or VB_ENOMEM (which names the bytes) the image is as it was.
 *
 * An insert bumps the image's generation, like a load: element filters made before it and filtered scan handles
 * begun before it fail with VB_ESTATE (their bitsets cover the old elements only).  Unfiltered vb_hnsw_scan handles
 * and vb_hnsw_search* work on the grown graph.
 */
typedef struct vb_hnsw_slot
{
	int32_t		element,
				layer,
				slot,
				neighbor;
} vb_hnsw_slot;
int			vb_hnsw_insert(vb_hnsw *h, const void *rows, int64_t n, int ef_construction, uint64_t seed,
						   const int32_t *levels, int32_t *out_dup_of, int64_t *out_nchanges);
int			vb_hnsw_insert_dev(vb_hnsw *h, const void *rows_dev, int64_t n, int ef_construction, uint64_t seed,
							   const int32_t *levels, int32_t *out_dup_of, int64_t *out_nchanges);
int			vb_hnsw_insert_changes(vb_hnsw *h, vb_hnsw_slot *out, int64_t cap);	/* the last insert's or vacuum's records */
int			vb_hnsw_set_heaptid_counts(vb_hnsw *h, const int32_t *counts);

/*
 * VACUUM of a resident image: the graph part of hnswbulkdelete (src/hnswvacuum.c:776-797).  counts (host [vb_hnsw_rows])
 * are the heap TIDs each element keeps after RemoveHeapTids (:35-173), which the glue runs on the pages: 0..10, 0 = the
 * element is deleted now or was deleted by an earlier vacuum; rows vb_hnsw_insert folded into another element must be
 * 0.  They replace the image's counts, as vb_hnsw_set_heaptid_counts does.  Then:
 *   1. RepairGraphEntryPoint (:279-373): the highest live point (the first live element of a strictly higher level, in
 *      element order, which is page order) -- or the fallback point when that is the entry point -- is repaired when
 *      NeedsUpdated; an entry point being deleted is replaced by the highest point (-1 when nothing is live); a live one
 *      is repaired when NeedsUpdated, searching from the highest point.
 *   2. RepairGraph (:378-502): every live element other than the entry point for which NeedsUpdated (:178-220) holds
 *      -- a slot on any layer names an element of count 0, or the last layer-0 slot is empty -- is repaired, in element
 *      order, in batches of at most max(1, live / hnsw_build_fraction) elements (capped by hnsw_build_batch), with
 *      NeedsUpdated evaluated at each batch's start.  A repair is RepairGraphElement: HnswFindElementNeighbors with
 *      existing = true (elements of count 0 do not count towards ef, ef_construction + 1, the element itself and
 *      elements of count 0 removed before SelectNeighbors) against the graph as of the batch start; its whole neighbour
 *      tuple is replaced, then HnswUpdateNeighborsOnDisk with ConnectionExists (src/hnswinsert.c:453-468) updates its
 *      neighbours.  With batches of one element the result is the serial reference's.
 *   3. MarkDeleted (:594-729): every neighbour slot of every element of count 0 is cleared.  Such elements stay in the
 *      image as unreachable tombstones; their numbers are not reused, so the image grows until it is reloaded.
 * *out_nrepaired (may be NULL) = the repairs made; change records as for vb_hnsw_insert: every slot whose value
 * differs from before the call (a cleared slot has neighbor -1), through vb_hnsw_insert_changes.
 * Arguments are validated and memory reserved before any kernel runs (VB_EINVAL / VB_ENOMEM leave the image as it
 * was).  A vacuum bumps the generation like an insert; unfiltered vb_hnsw_scan handles keep working (a tombstone they
 * return from their discarded set has count 0, so the glue hands out no heap TIDs for it).
 */
int			vb_hnsw_vacuum(vb_hnsw *h, const int32_t *counts, int ef_construction, int64_t *out_nrepaired,
						   int64_t *out_nchanges);
int64_t		vb_hnsw_rows(const vb_hnsw *h);
int64_t		vb_hnsw_upper_slots(const vb_hnsw *h);
int			vb_hnsw_export(vb_hnsw *h, int32_t *levels, int32_t *nbr0, int64_t *upper_off, int32_t *upper,
						   int64_t *entry, int32_t *dup_of);
/*
 * GetScanItems (src/hnswscan.c:25-56): greedy descent with ef = 1 through the
 * upper layers, then HnswSearchLayer (src/hnswutils.c:824-987) with ef at layer 0;
 * results nearest first (src/hnswscan.c:293-326), k <= ef of them per query,
 * -1 padded.  Every distance comparison is on the total order (distance,
 * element number).  out_ndist (may be NULL) = distance evaluations per query
 * (the reference's `tuples` counter, src/hnswutils.c:872-873, 905-906).
 */
int			vb_hnsw_search(vb_hnsw *h, const void *queries, int64_t nq, int ef, int k,
						   int64_t *out_ids, double *out_dist, int64_t *out_ndist);
int			vb_hnsw_search_dev(vb_hnsw *h, const void *queries_dev, int64_t nq, int ef, int k,
							   int64_t *out_ids_dev, float *out_dist_dev, int64_t *out_ndist_dev);

/*
 * hnsw.iterative_scan (src/hnswscan.c:62-87 ResumeScanItems, :228-340 hnswgettuple) for nq queries at once.  The
 * handle owns what the reference keeps in HnswScanOpaqueData between batches: the visited set `v`, the `discarded`
 * candidates (rejected neighbours and evicted results, src/hnswutils.c:929-937, 968-973) and the `tuples` counter.
 * vb_hnsw_scan_next returns, per query, the next batch nearest first: out_ids / out_distances [nq x ef_search]
 * (-1 / +inf padded), out_counts [nq]; the first call is GetScanItems (:25-56), every later one resumes from the
 * ef_search nearest discarded candidates on the same visited set, and once a query's tuples counter has reached
 * max_scan_tuples (hnsw.max_scan_tuples, src/hnsw.c:101-105) its remaining discarded candidates come back nearest
 * first, ef_search at a time, without searching (:247-254).  out_counts[q] == 0: that scan is exhausted.
 * The sequence is hnsw.iterative_scan = relaxed_order's; strict_order is the caller's filter on it (:316-322).
 * work_mem * hnsw.scan_mem_multiplier (:247) is not modelled: map it onto max_scan_tuples.
 */
typedef struct vb_hnsw_scan vb_hnsw_scan;
int			vb_hnsw_scan_begin(vb_hnsw *h, const void *queries, int64_t nq, int ef_search, int64_t max_scan_tuples,
							   vb_hnsw_scan **out);
int			vb_hnsw_scan_next(vb_hnsw_scan *scan, int64_t *out_ids, double *out_distances, int32_t *out_counts);
int			vb_hnsw_scan_tuples(vb_hnsw_scan *scan, int64_t *out_tuples);	/* [nq] the tuples counters */
int			vb_hnsw_scan_end(vb_hnsw_scan *scan);

/*
 * Element filters of an HNSW image (see vb_filter above): elements = element numbers in [0, n).  Host variant: a value
 * out of range fails with VB_EINVAL naming its position and value; _dev variant: such values are ignored.  Duplicates
 * collapse, n == 0 is an empty filter; vb_filter_rows and vb_filter_free apply.  The image holds no heap TIDs: the caller
 * allows an element when any of its heap TIDs passes (a row a GPU build folded into another element, dup_of, is reached
 * through that element) and withholds the rejected TIDs of an element the scan returns (INTEGRATION.md section 7c).
 * A filter is refused (VB_EINVAL) by any other index, table or IVFFlat image, also after its own was freed, and an HNSW
 * filter by their entry points; after vb_hnsw_load / vb_hnsw_build* of its image, begin fails with VB_ESTATE ("index
 * changed since the filter was created").
 */
int			vb_hnsw_filter_create(vb_hnsw *h, const int64_t *elements, int64_t n, vb_filter **out);
int			vb_hnsw_filter_create_dev(vb_hnsw *h, const int64_t *elements_dev, int64_t n, vb_filter **out);

/*
 * The iterative scan with an element filter per query: query q uses filters[filter_of_query[q]] (host array; NULL when
 * nfilters == 1; an entry out of range fails with VB_EINVAL naming the query).  Let S_q be the unfiltered handle's
 * sequence (its batches concatenated until out_counts == 0).  The filtered sequence is S_q restricted to the allowed
 * elements: same order, same element numbers, same float8 distances bit for bit.  The traversal is the unfiltered one:
 * rejected elements are visited, expanded, counted in `tuples` and kept as discarded candidates, as in the reference,
 * where the predicate is applied above the index.
 * vb_hnsw_scan_next on this handle writes out_ids / out_distances [nq x page] (1 <= page <= 2048, -1 / +inf padded):
 * the next min(page, remaining) allowed elements of each query, across underlying batches; out_counts[q] < page only
 * when the sequence is exhausted, and 0 (for good) once it is.  Underlying batches run inside the call, only while the
 * page is not full: after a call that fills its page, tuples equals the unfiltered handle's after the batch holding the
 * call's last element; after one that does not, the scan has run to its end.  Begin copies the filters' bitsets (the
 * filters may be freed at once) and counts them in the VB_ENOMEM check.  next fails with VB_ESTATE, writing nothing,
 * once the image has been loaded or built again.  vb_hnsw_scan_tuples and vb_hnsw_scan_end are shared.
 */
int			vb_hnsw_scan_begin_filtered(vb_hnsw *h, const void *queries, int64_t nq, int ef_search,
										int64_t max_scan_tuples, int page, const vb_filter *const *filters, int nfilters,
										const int32_t *filter_of_query, vb_hnsw_scan **out);

#ifdef __cplusplus
}
#endif
#endif							/* VECB200_H */
