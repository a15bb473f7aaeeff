/*
 * hnsw_ondisk_oracle.c -- TEST INFRASTRUCTURE ONLY: the serial on-disk HNSW insert (HnswInsertTupleOnDisk,
 * src/hnswinsert.c:696-743) that vb_hnsw_insert is checked against, restated on top of the CPU oracle's HNSW
 * (oracle/pgv_hnsw.c is compiled into this translation unit unchanged, so the layer search, SelectNeighbors and
 * HnswUpdateConnection are the oracle's own).  Built at test time by tests/hnsw_ondisk_oracle.py.
 *
 * The rules that differ from the in-memory build:
 *   - RemoveElements (src/hnswutils.c:1237-1259, 1343-1344): candidates whose element is being deleted (no heap
 *     TIDs) help the search but are removed before SelectNeighbors;
 *   - FindDuplicateOnDisk / AddDuplicateOnDisk (src/hnswinsert.c:586-663): the row joins the first equal layer-0
 *     neighbour, in neighbour order, with 1..9 heap TIDs (0 = being deleted and 10 = full are skipped);
 *   - UpdateNeighborOnDisk through GetUpdateIndex (:409-448, 506-518): a list with room takes the new element in its
 *     first free slot; a full list has its distances recomputed from the target's own value (LoadElementsForInsert,
 *     :383-403) and its first element being deleted is replaced; otherwise HnswUpdateConnection replaces the pruned
 *     connection in its slot (nothing changes when the new element is the one pruned);
 *   - the entry point moves only to a strictly higher level (:688-689), never to a folded row.
 * Row i of an insert becomes element n + i; a folded row keeps its number with no neighbours and no heap TIDs.
 */
#include "pgv_hnsw.c"

/* an oracle graph plus what the on-disk insert keeps beside it: the rows it copied and the duplicate map */
typedef struct
{
	PgvHnsw    *g;
	int64_t		nrows;			/* rows in g->rows */
	void	   *own_rows;		/* rows copied by the inserts (then g->rows == own_rows) */
	int32_t    *dup_of;			/* [g->n]: element a row was folded into, or -1 */
} DiskHnsw;

DiskHnsw *
disk_hnsw_wrap(PgvHnsw *g, int64_t nrows)
{
	DiskHnsw   *d = calloc(1, sizeof(DiskHnsw));

	d->g = g;
	d->nrows = nrows;
	d->dup_of = malloc(sizeof(int32_t) * (size_t) (g->n + 1));
	for (int64_t i = 0; i < g->n; i++)
		d->dup_of[i] = -1;
	return d;
}

void
disk_hnsw_free(DiskHnsw *d)
{
	if (!d)
		return;
	pgv_hnsw_free(d->g);
	free(d->own_rows);
	free(d->dup_of);
	free(d);
}

/* HnswFindElementNeighbors (hnswutils.c:1280-1357), existing = false, with RemoveElements before SelectNeighbors */
static void
find_element_neighbors_on_disk(PgvHnsw *g, int32_t eid, int64_t entryPoint)
{
	Element    *element = &g->el[eid];
	const void *q = (const char *) g->rows + (size_t) element->row * g->rb;
	int			level = element->level;
	int			entryLevel;
	Arena		arena = {0};
	CandList	ep,
				w;

	if (entryPoint < 0)
		return;

	ep.items = malloc(sizeof(SearchCand *));
	ep.items[0] = arena_new(&arena, (int32_t) entryPoint, elem_distance(g, q, (int32_t) entryPoint));
	ep.n = 1;
	entryLevel = g->el[entryPoint].level;

	for (int lc = entryLevel; lc >= level + 1; lc--)
	{
		g->epoch++;
		w = search_layer(g, q, ep, 1, lc, 0, g->visited, g->epoch, NULL, &arena);
		free(ep.items);
		ep = w;
	}
	if (level > entryLevel)
		level = entryLevel;

	for (int lc = level; lc >= 0; lc--)
	{
		int			lm = LAYER_M(g->m, lc);
		int			lwn = 0,
					rn;
		Cand	   *lw;
		Cand	  **lwp,
				  **r;
		NbrArray   *na = &element->nbr[lc];

		g->epoch++;
		w = search_layer(g, q, ep, g->efc, lc, 0, g->visited, g->epoch, NULL, &arena);

		lw = malloc(sizeof(Cand) * (size_t) (w.n + 1));
		lwp = malloc(sizeof(Cand *) * (size_t) (w.n + 1));
		r = malloc(sizeof(Cand *) * (size_t) (w.n + 1));
		for (int i = 0; i < w.n; i++)
		{
			/* elements being deleted help the search but are removed before selecting neighbors */
			if (g->el[w.items[i]->element].heaptidsLength == 0)
				continue;
			lw[lwn].id = w.items[i]->element;
			lw[lwn].distance = (float) w.items[i]->distance;
			lw[lwn].closer = 0;
			lwp[lwn] = &lw[lwn];
			lwn++;
		}
		rn = select_neighbors(g, lwp, lwn, lm, &na->closerSet, NULL, NULL, 0, r);
		for (int i = 0; i < rn; i++)
			na->items[na->length++] = *r[i];
		free(lw);
		free(lwp);
		free(r);
		free(ep.items);
		ep = w;				/* the unfiltered W is the next layer's entry list */
	}
	free(ep.items);
	arena_free(&arena);
}

static void
update_neighbor_on_disk(PgvHnsw *g, int32_t t, int lc, int32_t newId, float distance)
{
	NbrArray   *na = &g->el[t].nbr[lc];
	int			lm = LAYER_M(g->m, lc);

	if (na->length < lm)
	{
		na->items[na->length].id = newId;
		na->items[na->length].distance = distance;
		na->items[na->length].closer = 0;
		na->length++;
		return;
	}
	for (int i = 0; i < na->length; i++)
	{
		na->items[i].distance = pair_distance(g, t, na->items[i].id);
		na->items[i].closer = 0;
		if (g->el[na->items[i].id].heaptidsLength == 0)
		{
			na->items[i].id = newId;
			na->items[i].distance = distance;
			return;
		}
	}
	na->closerSet = 0;			/* a list loaded from its page carries no closer flags */
	update_connection(g, na, newId, distance, lm);
}

static void
insert_row_on_disk(DiskHnsw *d, int64_t row, int level)
{
	PgvHnsw    *g = d->g;
	int32_t		eid = (int32_t) g->n;
	Element    *e = &g->el[eid];
	int64_t		entryPoint = g->entry;

	if (level > g->maxLevel)
		level = g->maxLevel;
	memset(e, 0, sizeof(*e));
	e->level = level;
	e->row = row;
	e->heaptids[e->heaptidsLength++] = row;
	init_neighbors(g, e);
	d->dup_of[eid] = -1;
	g->n++;

	find_element_neighbors_on_disk(g, eid, entryPoint);

	/* FindDuplicateOnDisk / AddDuplicateOnDisk */
	{
		NbrArray   *na = &e->nbr[0];

		for (int i = 0; i < na->length; i++)
		{
			Element    *ne = &g->el[na->items[i].id];

			if (!rows_equal(g, e->row, ne->row))
				break;
			if (ne->heaptidsLength == 0 || ne->heaptidsLength == HNSW_HEAPTIDS)
				continue;
			ne->heaptids[ne->heaptidsLength++] = row;
			for (int lc = 0; lc <= e->level; lc++)
				e->nbr[lc].length = 0;
			e->heaptidsLength = 0;
			d->dup_of[eid] = na->items[i].id;
			return;
		}
	}

	/* HnswUpdateNeighborsOnDisk */
	for (int lc = e->level; lc >= 0; lc--)
	{
		NbrArray   *na = &e->nbr[lc];

		for (int i = 0; i < na->length; i++)
			update_neighbor_on_disk(g, na->items[i].id, lc, eid, na->items[i].distance);
	}
	if (entryPoint < 0 || e->level > g->el[entryPoint].level)
		g->entry = eid;
}

/* n rows inserted one at a time; levels NULL = drawn from the oracle's PRNG */
void
disk_hnsw_insert(DiskHnsw *d, const void *rows, int64_t n, const int32_t *levels)
{
	PgvHnsw    *g = d->g;
	int64_t		n0 = g->n;
	char	   *all = malloc(g->rb * (size_t) (d->nrows + n) + 1);

	if (d->nrows > 0)
		memcpy(all, g->rows, g->rb * (size_t) d->nrows);
	if (n > 0)
		memcpy(all + g->rb * (size_t) d->nrows, rows, g->rb * (size_t) n);
	free(d->own_rows);
	d->own_rows = all;
	g->rows = all;
	g->el = realloc(g->el, sizeof(Element) * (size_t) (n0 + n + 1));
	d->dup_of = realloc(d->dup_of, sizeof(int32_t) * (size_t) (n0 + n + 1));
	g->visited = realloc(g->visited, sizeof(uint32_t) * (size_t) (n0 + n + 1));
	memset(g->visited, 0, sizeof(uint32_t) * (size_t) (n0 + n + 1));
	g->epoch = 0;
	for (int64_t i = 0; i < n; i++)
	{
		int			level = levels ? levels[i] : (int) (-log(rnd_double(g)) * g->ml);

		insert_row_on_disk(d, d->nrows + i, level);
	}
	d->nrows += n;
}

/* heap TID count of every element (0 = being deleted, 10 = full) */
void
disk_hnsw_set_heaptid_counts(DiskHnsw *d, const int32_t *counts)
{
	for (int64_t i = 0; i < d->g->n; i++)
	{
		d->g->el[i].heaptidsLength = counts[i];
		for (int j = 0; j < counts[i]; j++)
			d->g->el[i].heaptids[j] = d->g->el[i].row;
	}
}

void
disk_hnsw_dup_of(const DiskHnsw *d, int32_t *dup_of)
{
	memcpy(dup_of, d->dup_of, sizeof(int32_t) * (size_t) d->g->n);
}

PgvHnsw *
disk_hnsw_graph(const DiskHnsw *d)
{
	return d->g;
}
