/*
 * ivf_insert_oracle.c -- TEST INFRASTRUCTURE ONLY: FindInsertPage (src/ivfinsert.c:19-67), the list an IVFFlat insert
 * goes to, restated beside the CPU oracle's pgv_ivf_assign (which restates AddTupleToSort's choice at build time).
 * Built at test time by tests/ivf_insert_oracle.py against oracle/pgv_distance.c.
 *
 * The two differ only in where the running minimum starts: the insert takes the first list unconditionally (its insert
 * page is still invalid) and then moves on a strict <, so a NaN distance to list 0 keeps list 0 -- no distance
 * compares smaller than a NaN -- while the build's minimum starts at DBL_MAX and skips a NaN list 0.
 */
#include <float.h>

#include "pgv_oracle.h"

void
pgv_ivf_insert_lists(int elem, int metric, int dim, const void *rows, int64_t n, const void *centers, int lists,
					 int32_t *out_list)
{
	size_t		rb = pgv_row_bytes(elem, dim);

	for (int64_t r = 0; r < n; r++)
	{
		double		minDistance = DBL_MAX;
		int			insertList = -1;

		for (int i = 0; i < lists; i++)
		{
			double		distance = pgv_distance(elem, metric, dim, (const char *) rows + (size_t) r * rb,
												(const char *) centers + (size_t) i * rb);

			if (distance < minDistance || insertList < 0)
			{
				insertList = i;
				minDistance = distance;
			}
		}
		out_list[r] = insertList;
	}
}
