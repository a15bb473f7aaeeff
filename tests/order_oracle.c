/*
 * order_oracle.c -- the btree comparators of vector, halfvec and sparsevec restated on the CPU, and the order the GPU's
 * vb_order is checked against.  TEST INFRASTRUCTURE ONLY.
 *
 *   vector_cmp_internal     src/vector.c:1030-1052: elements with < and >, then the dimensions
 *   halfvec_cmp_internal    src/halfvec.c:987: the same on HalfToFloat4 (pgv_half_to_float, oracle/pgv_distance.c)
 *   sparsevec_cmp_internal  src/sparsevec.c:1153-1188: entries while both rows have them (an index mismatch is decided
 *                           by the sign of the value with the smaller index), then the first extra entry of the longer
 *                           row when its index is inside the other's dimension, then the dimensions
 * All three take rows of different dimensions, as the reference does.
 *
 * The order: qsort of the row numbers on (comparator, row number); groups = maximal runs the comparator calls equal;
 * bounds by a linear scan over the rows (lo = rows < q, hi = rows <= q).
 */
#include <stdint.h>
#include <stdlib.h>

#include "pgv_oracle.h"

int
ord_vector_cmp(const float *a, int da, const float *b, int db)
{
	int			dim = da < db ? da : db;

	for (int i = 0; i < dim; i++)
	{
		if (a[i] < b[i])
			return -1;
		if (a[i] > b[i])
			return 1;
	}
	if (da < db)
		return -1;
	if (da > db)
		return 1;
	return 0;
}

int
ord_halfvec_cmp(const uint16_t *a, int da, const uint16_t *b, int db)
{
	int			dim = da < db ? da : db;

	for (int i = 0; i < dim; i++)
	{
		float		x = pgv_half_to_float(a[i]),
					y = pgv_half_to_float(b[i]);

		if (x < y)
			return -1;
		if (x > y)
			return 1;
	}
	if (da < db)
		return -1;
	if (da > db)
		return 1;
	return 0;
}

int
ord_sparsevec_cmp(int adim, int annz, const int32_t *ai, const float *ax, int bdim, int bnnz, const int32_t *bi, const float *bx)
{
	int			nnz = annz < bnnz ? annz : bnnz;

	for (int i = 0; i < nnz; i++)
	{
		if (ai[i] < bi[i])
			return ax[i] < 0 ? -1 : 1;
		if (ai[i] > bi[i])
			return bx[i] < 0 ? 1 : -1;
		if (ax[i] < bx[i])
			return -1;
		if (ax[i] > bx[i])
			return 1;
	}
	if (annz < bnnz && bi[nnz] < adim)
		return bx[nnz] < 0 ? 1 : -1;
	if (annz > bnnz && ai[nnz] < bdim)
		return ax[nnz] < 0 ? -1 : 1;
	if (adim < bdim)
		return -1;
	if (adim > bdim)
		return 1;
	return 0;
}

/* pairs of rows a[k], b[k] of one dimension (dense: packed rows; sparse: CSR with offsets into its own idx / val) */
void
ord_dense_cmp_pairs(int half, const void *a, const void *b, int64_t npairs, int dim, int32_t *out)
{
	for (int64_t k = 0; k < npairs; k++)
		out[k] = half ? ord_halfvec_cmp((const uint16_t *) a + k * dim, dim, (const uint16_t *) b + k * dim, dim)
			: ord_vector_cmp((const float *) a + k * dim, dim, (const float *) b + k * dim, dim);
}

void
ord_sparse_cmp_pairs(int dim, int64_t npairs, const int64_t *aoff, const int32_t *aidx, const float *aval, const int64_t *boff,
					 const int32_t *bidx, const float *bval, int32_t *out)
{
	for (int64_t k = 0; k < npairs; k++)
		out[k] = ord_sparsevec_cmp(dim, (int) (aoff[k + 1] - aoff[k]), aidx + aoff[k], aval + aoff[k], dim, (int) (boff[k + 1] - boff[k]),
								   bidx + boff[k], bval + boff[k]);
}

/* one table and its comparator, for qsort */
static struct
{
	int			kind;			/* 0 vector, 1 halfvec, 2 sparsevec */
	int			dim;
	const void *rows;
	const int64_t *off;
	const int32_t *idx;
	const float *val;
}			T;

static int
row_cmp(int64_t r, int64_t s)
{
	if (T.kind == 0)
		return ord_vector_cmp((const float *) T.rows + r * T.dim, T.dim, (const float *) T.rows + s * T.dim, T.dim);
	if (T.kind == 1)
		return ord_halfvec_cmp((const uint16_t *) T.rows + r * T.dim, T.dim, (const uint16_t *) T.rows + s * T.dim, T.dim);
	return ord_sparsevec_cmp(T.dim, (int) (T.off[r + 1] - T.off[r]), T.idx + T.off[r], T.val + T.off[r], T.dim,
							 (int) (T.off[s + 1] - T.off[s]), T.idx + T.off[s], T.val + T.off[s]);
}

static int
perm_cmp(const void *x, const void *y)
{
	int64_t		r = *(const int64_t *) x,
				s = *(const int64_t *) y;
	int			c = row_cmp(r, s);

	if (c)
		return c;
	return r < s ? -1 : (r > s ? 1 : 0);
}

/* kind, dim, rows (dense) or off / idx / val (sparse), n -> perm [n], group_of_row [n], group_start [n + 1]; returns groups */
int64_t
ord_order(int kind, int dim, const void *rows, const int64_t *off, const int32_t *idx, const float *val, int64_t n, int64_t *perm,
		  int32_t *gor, int64_t *gstart)
{
	int64_t		g = 0;

	T.kind = kind;
	T.dim = dim;
	T.rows = rows;
	T.off = off;
	T.idx = idx;
	T.val = val;
	for (int64_t i = 0; i < n; i++)
		perm[i] = i;
	qsort(perm, (size_t) n, sizeof(int64_t), perm_cmp);
	for (int64_t i = 0; i < n; i++)
	{
		if (i == 0 || row_cmp(perm[i - 1], perm[i]) != 0)
			gstart[g++] = i;
		gor[perm[i]] = (int32_t) (g - 1);
	}
	gstart[g] = n;
	return g;
}

/* lo / hi of nq queries (dense: packed rows of dim; sparse: CSR qoff / qidx / qval) over the table's n rows */
void
ord_bounds(int kind, int dim, const void *rows, const int64_t *off, const int32_t *idx, const float *val, int64_t n, const void *q,
		   const int64_t *qoff, const int32_t *qidx, const float *qval, int64_t nq, int64_t *lo, int64_t *hi)
{
	for (int64_t k = 0; k < nq; k++)
	{
		int64_t		l = 0,
					h = 0;

		for (int64_t r = 0; r < n; r++)
		{
			int			c;

			if (kind == 0)
				c = ord_vector_cmp((const float *) rows + r * dim, dim, (const float *) q + k * dim, dim);
			else if (kind == 1)
				c = ord_halfvec_cmp((const uint16_t *) rows + r * dim, dim, (const uint16_t *) q + k * dim, dim);
			else
				c = ord_sparsevec_cmp(dim, (int) (off[r + 1] - off[r]), idx + off[r], val + off[r], dim, (int) (qoff[k + 1] - qoff[k]),
									  qidx + qoff[k], qval + qoff[k]);
			l += c < 0;
			h += c <= 0;
		}
		lo[k] = l;
		hi[k] = h;
	}
}
