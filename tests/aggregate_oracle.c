/*
 * aggregate_oracle.c -- the reference's vector / halfvec aggregates restated in C, and the run plan of
 * vb_table_aggregate on top of them.  TEST INFRASTRUCTURE ONLY: the GPU aggregate is checked against this.
 *
 * State arrays are passed as the reference's ArrayType would hold them: ndim, the length of the first dimension, a
 * has-nulls flag and the float8 data, so that CheckStateArray's errors can be reproduced.  Every function returns 0,
 * or -1 with the reference's error text in err (ERRBUF bytes).  Halves are IEEE binary16 bit patterns, converted by the
 * CPU oracle's HalfToFloat4 / Float4ToHalfUnchecked restatements (oracle/pgv_distance.c).
 */
#include <math.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "pgv_oracle.h"

#define ERRBUF 256
#define MAX_DIM 16000			/* VECTOR_MAX_DIM (src/vector.h:11), HALFVEC_MAX_DIM (src/halfvec.h:60) */

static int
fail(char *err, const char *msg)
{
	snprintf(err, ERRBUF, "%s", msg);
	return -1;
}

/* CheckStateArray (src/vector.c:163-171) */
static int
check_state_array(int ndim, int len0, int hasnull, const char *caller, char *err)
{
	if (ndim != 1 || len0 < 1 || hasnull)
	{
		snprintf(err, ERRBUF, "%s: expected state array", caller);
		return -1;
	}
	return 0;
}

/* CheckDim (src/vector.c:95-106; halfvec's, src/halfvec.c:99-110) */
static int
check_dim(int dim, const char *type, char *err)
{
	if (dim < 1)
	{
		snprintf(err, ERRBUF, "%s must have at least 1 dimension", type);
		return -1;
	}
	if (dim > MAX_DIM)
	{
		snprintf(err, ERRBUF, "%s cannot have more than %d dimensions", type, MAX_DIM);
		return -1;
	}
	return 0;
}

/* CheckExpectedDim (src/vector.c:83-89) */
static int
check_expected_dim(int typmod, int dim, char *err)
{
	if (typmod != -1 && typmod != dim)
	{
		snprintf(err, ERRBUF, "expected %d dimensions, not %d", typmod, dim);
		return -1;
	}
	return 0;
}

/* Float4ToHalf (src/halfutils.h:244-260): Float4ToHalfUnchecked plus its overflow check (the value is printed with %g,
 * not float_to_shortest_decimal_buf: a mean of halves never reaches it) */
static int
float4_to_half(float f, uint16_t *out, char *err)
{
	uint16_t	h = pgv_float_to_half(f);

	if ((h & 0x7fff) == 0x7c00 && !isinf(f))
	{
		char		num[64];

		snprintf(num, sizeof(num), "%g", f);
		snprintf(err, ERRBUF, "\"%s\" is out of range for type halfvec", num);
		return -1;
	}
	*out = h;
	return 0;
}

/*
 * vector_accum (src/vector.c:1148-1204) and halfvec_accum (src/halfvec.c:1104-1160): out = [n + 1, s + x] (dim + 1
 * entries; dim = the row's when the state has none).  x is float[dim] (half = 0) or binary16[dim] (half = 1).
 */
int
agg_accum(int half, const double *st, int ndim, int len0, int hasnull, const void *x, int dim, double *out, char *err)
{
	int			sdim;
	int			newarr;

	if (check_state_array(ndim, len0, hasnull, half ? "halfvec_accum" : "vector_accum", err))
		return -1;
	sdim = len0 - 1;			/* STATE_DIMS */
	newarr = sdim == 0;
	if (!newarr && check_expected_dim(sdim, dim, err))
		return -1;
	out[0] = st[0] + 1.0;
	for (int i = 0; i < dim; i++)
	{
		double		xi = half ? (double) pgv_half_to_float(((const uint16_t *) x)[i]) : (double) ((const float *) x)[i];

		if (newarr)
			out[i + 1] = xi;
		else
		{
			double		v = st[i + 1] + xi;

			if (isinf(v))
				return fail(err, "value out of range: overflow");
			out[i + 1] = v;
		}
	}
	return 0;
}

/* vector_combine (src/vector.c:1209-1284), also halfvec_combine: *out_len = the result's length (dim + 1) */
int
agg_combine(const double *s1, int nd1, int l1, int hn1, const double *s2, int nd2, int l2, int hn2, double *out, int *out_len,
			char *err)
{
	int			dim1,
				dim2,
				dim;

	if (check_state_array(nd1, l1, hn1, "vector_combine", err) || check_state_array(nd2, l2, hn2, "vector_combine", err))
		return -1;
	dim1 = l1 - 1;
	dim2 = l2 - 1;
	if (dim1 == 0 && dim2 == 0)
		dim = 0;
	else if (dim1 == 0)
	{
		dim = dim2;
		if (check_dim(dim, "vector", err))
			return -1;
		for (int i = 0; i < dim; i++)
			out[i + 1] = s2[i + 1];
	}
	else if (dim2 == 0)
	{
		dim = dim1;
		if (check_dim(dim, "vector", err))
			return -1;
		for (int i = 0; i < dim; i++)
			out[i + 1] = s1[i + 1];
	}
	else
	{
		dim = dim1;
		if (check_dim(dim, "vector", err) || check_expected_dim(dim, dim2, err))
			return -1;
		for (int i = 0; i < dim; i++)
		{
			double		v = s1[i + 1] + s2[i + 1];

			if (isinf(v))
				return fail(err, "value out of range: overflow");
			out[i + 1] = v;
		}
	}
	out[0] = s1[0] + s2[0];
	*out_len = dim + 1;
	return 0;
}

/*
 * vector_avg (src/vector.c:1289-1318) and halfvec_avg (src/halfvec.c:1165-1194): *is_null = 1 when n == 0 (SQL NULL);
 * otherwise out = float[dim] or binary16[dim].  CheckElement cannot fail on a mean of finite values and is not restated.
 */
int
agg_avg(int half, const double *st, int ndim, int len0, int hasnull, void *out, int *is_null, char *err)
{
	double		n;
	int			dim;

	if (check_state_array(ndim, len0, hasnull, half ? "halfvec_avg" : "vector_avg", err))
		return -1;
	n = st[0];
	*is_null = n == 0.0;
	if (*is_null)
		return 0;
	dim = len0 - 1;
	if (check_dim(dim, half ? "halfvec" : "vector", err))
		return -1;
	for (int i = 0; i < dim; i++)
	{
		float		m = (float) (st[i + 1] / n);

		if (half)
		{
			if (float4_to_half(m, &((uint16_t *) out)[i], err))
				return -1;
		}
		else
			((float *) out)[i] = m;
	}
	return 0;
}

/* vector_add (src/vector.c:824-852) and halfvec_add (src/halfvec.c:764-798; the non-_Float16 branch, which rounds the
 * fp32 sum of the widened halves: the correctly rounded half sum) */
int
agg_add(int half, const void *a, const void *b, int dim, void *out, char *err)
{
	for (int i = 0; i < dim; i++)
	{
		if (half)
		{
			uint16_t	r = pgv_float_to_half(pgv_half_to_float(((const uint16_t *) a)[i]) + pgv_half_to_float(((const uint16_t *) b)[i]));

			((uint16_t *) out)[i] = r;
		}
		else
			((float *) out)[i] = ((const float *) a)[i] + ((const float *) b)[i];
	}
	for (int i = 0; i < dim; i++)
	{
		int			inf = half ? (((const uint16_t *) out)[i] & 0x7fff) == 0x7c00 : isinf(((const float *) out)[i]);

		if (inf)
			return fail(err, "value out of range: overflow");
	}
	return 0;
}

/*
 * The plan of vb_table_aggregate (include/vecb200.h): per group, its rows in ascending row number cut into runs of R
 * (0 = one run), each run's state from the initial condition through the transition function, the run states combined
 * left to right, then the final function.  agg 0 = avg, 1 = sum.  rows [n x dim] float or binary16; groups [n] in
 * [-1, ngroups) or NULL (every row in group 0).  Outputs as the C ABI's; on an error nothing is written.
 */
int
agg_table(int half, int agg, const void *rows, int64_t n, int dim, const int32_t *groups, int ngroups, int64_t R, void *out,
		  int64_t *counts, double *state, char *err)
{
	size_t		esize = half ? 2 : 4;
	int64_t    *cnt = calloc((size_t) ngroups + 1, sizeof(int64_t));
	int64_t    *pos = malloc(sizeof(int64_t) * ((size_t) n + 1));
	double	   *gst = malloc(sizeof(double) * ((size_t) dim + 1));	/* the group's state (avg) */
	double	   *rst = malloc(sizeof(double) * ((size_t) dim + 1));	/* the run's state (avg) */
	double	   *tmp = malloc(sizeof(double) * ((size_t) dim + 1));
	uint8_t    *gsum = malloc(esize * (size_t) dim);	/* the group's state (sum) */
	uint8_t    *rsum = malloc(esize * (size_t) dim);	/* the run's state (sum) */
	uint8_t    *vals = calloc((size_t) ngroups * dim, esize);
	int64_t    *vcnt = calloc((size_t) ngroups, sizeof(int64_t));
	double	   *vst = calloc((size_t) ngroups * (dim + 1), sizeof(double));
	int			rc = 0;

	/* each group's rows in ascending row number (a stable counting sort) */
	for (int64_t i = 0; i < n; i++)
	{
		int			g = groups ? groups[i] : 0;

		if (g >= 0)
			cnt[g + 1]++;
	}
	for (int g = 0; g < ngroups; g++)
		cnt[g + 1] += cnt[g];
	{
		int64_t    *fill = malloc(sizeof(int64_t) * ((size_t) ngroups + 1));

		memcpy(fill, cnt, sizeof(int64_t) * ((size_t) ngroups + 1));
		for (int64_t i = 0; i < n; i++)
		{
			int			g = groups ? groups[i] : 0;

			if (g >= 0)
				pos[fill[g]++] = i;
		}
		free(fill);
	}

	for (int g = 0; g < ngroups && rc == 0; g++)
	{
		int64_t		b = cnt[g],
					e = cnt[g + 1],
					len = e - b;
		int64_t		run = (R == 0 || R >= len) ? len : R;
		int			glen = 1;	/* length of the avg group state: INITCOND '{0}' */

		vcnt[g] = len;
		if (len == 0)
			continue;
		gst[0] = 0.0;
		for (int64_t r0 = b; r0 < e && rc == 0; r0 += run)
		{
			int64_t		r1 = r0 + run < e ? r0 + run : e;

			if (agg == 0)
			{
				int			rlen = 1;

				rst[0] = 0.0;	/* INITCOND '{0}' */
				for (int64_t j = r0; j < r1 && rc == 0; j++)
				{
					rc = agg_accum(half, rst, 1, rlen, 0, (const uint8_t *) rows + (size_t) pos[j] * dim * esize, dim, tmp, err);
					memcpy(rst, tmp, sizeof(double) * ((size_t) dim + 1));
					rlen = dim + 1;
				}
				if (rc == 0)
				{
					int			olen;

					rc = agg_combine(gst, 1, glen, 0, rst, 1, rlen, 0, tmp, &olen, err);
					memcpy(gst, tmp, sizeof(double) * (size_t) olen);
					glen = olen;
				}
			}
			else
			{
				memcpy(rsum, (const uint8_t *) rows + (size_t) pos[r0] * dim * esize, esize * dim);
				for (int64_t j = r0 + 1; j < r1 && rc == 0; j++)
					rc = agg_add(half, rsum, (const uint8_t *) rows + (size_t) pos[j] * dim * esize, dim, rsum, err);
				if (rc == 0)
				{
					if (r0 == b)
						memcpy(gsum, rsum, esize * dim);
					else
						rc = agg_add(half, gsum, rsum, dim, gsum, err);
				}
			}
		}
		if (rc)
			break;
		if (agg == 0)
		{
			int			is_null;

			rc = agg_avg(half, gst, 1, glen, 0, vals + (size_t) g * dim * esize, &is_null, err);
			memcpy(vst + (size_t) g * (dim + 1), gst, sizeof(double) * ((size_t) dim + 1));
		}
		else
			memcpy(vals + (size_t) g * dim * esize, gsum, esize * dim);
	}
	if (rc == 0)
	{
		memcpy(out, vals, esize * (size_t) ngroups * dim);
		memcpy(counts, vcnt, sizeof(int64_t) * (size_t) ngroups);
		if (state)
			memcpy(state, vst, sizeof(double) * (size_t) ngroups * (dim + 1));
	}
	free(cnt);
	free(pos);
	free(gst);
	free(rst);
	free(tmp);
	free(gsum);
	free(rsum);
	free(vals);
	free(vcnt);
	free(vst);
	return rc;
}
