/*
 * hnsw_vacuum_oracle.c -- TEST INFRASTRUCTURE ONLY: the serial graph work of hnswbulkdelete (src/hnswvacuum.c) that
 * vb_hnsw_vacuum is checked against, restated on top of the serial on-disk insert (tests/hnsw_ondisk_oracle.c, which
 * compiles the CPU oracle's oracle/pgv_hnsw.c; both are included here unchanged, so SelectNeighbors, the on-disk
 * neighbour update and the export are theirs).  Built at test time by tests/hnsw_vacuum_oracle.py.
 *
 * What the vacuum adds:
 *   - the layer search with a skip element (CountElement): elements with no heap TIDs do not count towards ef;
 *   - RepairGraphElement: HnswFindElementNeighbors with existing = true, then HnswUpdateNeighborsOnDisk with
 *     ConnectionExists;
 *   - RemoveHeapTids' highest and fallback points, RepairGraphEntryPoint, RepairGraph with NeedsUpdated at each
 *     element's turn, and MarkDeleted.
 */
#include "hnsw_ondisk_oracle.c"


/*
 * HnswSearchLayer (hnswutils.c:824-987) with a skip element (existing = true, the vacuum's repairs): elements with no
 * heap TIDs do not count towards ef (CountElement, :713-728, 879-885, 957-974).  wlen counts the counted additions and
 * is never decremented; once it passes ef, every counted addition removes the furthest element of W, counted or not,
 * so W can hold more than ef elements.  Ties are not broken by element number (tie_total = 0), as in the insert.
 */
static CandList
search_layer_vacuum(const PgvHnsw *g, const void *q, CandList ep, int ef, int lc, uint32_t *visited, uint32_t epoch, Arena *arena)
{
	ph_heap		C,
				W;
	int			wlen = 0,
				wn = 0;
	int			lm = LAYER_M(g->m, lc);
	int			total = 0;
	int32_t    *unvisited = malloc(sizeof(int32_t) * (size_t) lm);
	CandList	w;

	ph_init(&C, cmp_nearest, &total);
	ph_init(&W, cmp_furthest, &total);
	for (int i = 0; i < ep.n; i++)
	{
		SearchCand *sc = ep.items[i];

		visited[sc->element] = epoch;
		ph_add(&C, &sc->c_node);
		ph_add(&W, &sc->w_node);
		wn++;
		if (g->el[sc->element].heaptidsLength != 0)
			wlen++;
	}
	while (!ph_is_empty(&C))
	{
		SearchCand *c = ph_container(SearchCand, c_node, ph_remove_first(&C));
		SearchCand *f = ph_container(SearchCand, w_node, ph_first(&W));
		const Element *ce;
		int			unvisitedLength = 0;

		if (key_cmp(c->distance, c->element, f->distance, f->element, total) > 0)
			break;
		ce = &g->el[c->element];
		if (lc <= ce->level)
		{
			const NbrArray *na = &ce->nbr[lc];

			for (int i = 0; i < na->length; i++)
			{
				int32_t		nid = na->items[i].id;

				if (visited[nid] != epoch)
				{
					visited[nid] = epoch;
					unvisited[unvisitedLength++] = nid;
				}
			}
		}
		for (int i = 0; i < unvisitedLength; i++)
		{
			int32_t		eid = unvisited[i];
			double		eDistance;
			int			alwaysAdd = wlen < ef;
			SearchCand *e;

			f = ph_container(SearchCand, w_node, ph_first(&W));
			eDistance = elem_distance(g, q, eid);
			if (!(key_cmp(eDistance, eid, f->distance, f->element, total) < 0 || alwaysAdd))
				continue;
			if (g->el[eid].level < lc)
				continue;
			e = arena_new(arena, eid, eDistance);
			ph_add(&C, &e->c_node);
			ph_add(&W, &e->w_node);
			wn++;
			if (g->el[eid].heaptidsLength != 0)
			{
				wlen++;
				if (wlen > ef)
				{
					ph_remove_first(&W);
					wn--;
				}
			}
		}
	}
	w.items = malloc(sizeof(SearchCand *) * (size_t) (wn + 1));
	w.n = 0;
	while (!ph_is_empty(&W))
		w.items[w.n++] = ph_container(SearchCand, w_node, ph_remove_first(&W));
	free(unvisited);
	return w;
}

/* HnswFindElementNeighbors (hnswutils.c:1280-1357), existing = true: ef_construction + 1, the element itself and the
 * elements with no heap TIDs removed before SelectNeighbors.  The new lists go to out[lc] / outn[lc]: the searches read
 * the element's lists as they stand on the pages, which RepairGraphElement overwrites only afterwards. */
static void
find_element_neighbors_existing(PgvHnsw *g, int32_t eid, int64_t entryPoint, Cand **out, int *outn)
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
		w = search_layer_vacuum(g, q, ep, 1, lc, g->visited, g->epoch, &arena);
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
		uint8_t		closerSet = 0;

		g->epoch++;
		w = search_layer_vacuum(g, q, ep, g->efc + 1, lc, g->visited, g->epoch, &arena);
		lw = malloc(sizeof(Cand) * (size_t) (w.n + 1));
		lwp = malloc(sizeof(Cand *) * (size_t) (w.n + 1));
		r = malloc(sizeof(Cand *) * (size_t) (w.n + 1));
		for (int i = 0; i < w.n; i++)
		{
			int32_t		id = w.items[i]->element;

			/* RemoveElements (hnswutils.c:1237-1259): the element itself and elements being deleted */
			if (id == eid || g->el[id].heaptidsLength == 0)
				continue;
			lw[lwn].id = id;
			lw[lwn].distance = (float) w.items[i]->distance;
			lw[lwn].closer = 0;
			lwp[lwn] = &lw[lwn];
			lwn++;
		}
		rn = select_neighbors(g, lwp, lwn, lm, &closerSet, NULL, NULL, 0, r);
		for (int i = 0; i < rn; i++)
			out[lc][i] = *r[i];
		outn[lc] = rn;
		free(lw);
		free(lwp);
		free(r);
		free(ep.items);
		ep = w;
	}
	free(ep.items);
	arena_free(&arena);
}

/* NeedsUpdated (hnswvacuum.c:178-220): a neighbour on any layer is being deleted, or the layer-0 list is not full */
static int
needs_updated(const PgvHnsw *g, int32_t e)
{
	const Element *el = &g->el[e];

	for (int lc = 0; lc <= el->level; lc++)
		for (int i = 0; i < el->nbr[lc].length; i++)
			if (g->el[el->nbr[lc].items[i].id].heaptidsLength == 0)
				return 1;
	return el->nbr[0].length < 2 * g->m;
}

/* RepairGraphElement (hnswvacuum.c:225-274): the whole neighbour tuple is replaced, then HnswUpdateNeighborsOnDisk with
 * ConnectionExists (hnswinsert.c:453-468, 503-505): a neighbour that already links to the element is left as it is */
static void
repair_graph_element(PgvHnsw *g, int32_t eid, int64_t entryPoint)
{
	Element    *e = &g->el[eid];
	Cand	  **out = malloc(sizeof(Cand *) * (size_t) (e->level + 1));
	int		   *outn = calloc((size_t) e->level + 1, sizeof(int));

	for (int lc = 0; lc <= e->level; lc++)
		out[lc] = malloc(sizeof(Cand) * (size_t) LAYER_M(g->m, lc));
	find_element_neighbors_existing(g, eid, entryPoint, out, outn);
	for (int lc = 0; lc <= e->level; lc++)
	{
		memcpy(e->nbr[lc].items, out[lc], sizeof(Cand) * (size_t) outn[lc]);
		e->nbr[lc].length = outn[lc];
		e->nbr[lc].closerSet = 0;
		free(out[lc]);
	}
	free(out);
	free(outn);
	for (int lc = e->level; lc >= 0; lc--)
	{
		NbrArray   *na = &e->nbr[lc];

		for (int i = 0; i < na->length; i++)
		{
			int32_t		t = na->items[i].id;
			const NbrArray *tn = &g->el[t].nbr[lc];
			int			exists = 0;

			for (int j = 0; j < tn->length && !exists; j++)
				exists = tn->items[j].id == eid;
			if (!exists)
				update_neighbor_on_disk(g, t, lc, eid, na->items[i].distance);
		}
	}
}

/*
 * hnswbulkdelete's graph work on heap TID counts already reduced by RemoveHeapTids (0 = being deleted or deleted by an
 * earlier vacuum; such elements hold no neighbours once this returns): RepairGraphEntryPoint, RepairGraph with
 * NeedsUpdated at each element's turn, MarkDeleted.  Returns the number of repairs made.
 */
int64_t
disk_hnsw_vacuum(DiskHnsw *d, const int32_t *counts)
{
	PgvHnsw    *g = d->g;
	int64_t		highest = -1,
				fallback = -1,
				nrep = 0;
	int			highestLevel = -1,
				fallbackLevel = -1;
	int64_t		entry;

	disk_hnsw_set_heaptid_counts(d, counts);
	/* RemoveHeapTids (hnswvacuum.c:133-157): the highest and the fallback point, in element (page) order */
	for (int64_t i = 0; i < g->n; i++)
	{
		if (g->el[i].heaptidsLength == 0)
			continue;
		if (g->el[i].level > highestLevel)
		{
			fallback = highest;
			fallbackLevel = highestLevel;
			highest = i;
			highestLevel = g->el[i].level;
		}
		else if (g->el[i].level > fallbackLevel)
		{
			fallback = i;
			fallbackLevel = g->el[i].level;
		}
	}
	/* RepairGraphEntryPoint (hnswvacuum.c:279-373) */
	entry = g->entry;
	if (highest >= 0)
	{
		int64_t		hp = highest == entry ? fallback : highest;

		if (hp >= 0 && needs_updated(g, (int32_t) hp))
		{
			repair_graph_element(g, (int32_t) hp, entry);
			nrep++;
		}
		highest = hp;
	}
	if (entry >= 0)
	{
		if (g->el[entry].heaptidsLength == 0)
			g->entry = highest;
		else if (needs_updated(g, (int32_t) entry))
		{
			repair_graph_element(g, (int32_t) entry, highest);
			nrep++;
		}
	}
	/* RepairGraph (hnswvacuum.c:378-502) */
	entry = g->entry;
	for (int64_t i = 0; i < g->n; i++)
	{
		if (g->el[i].heaptidsLength == 0 || i == entry || !needs_updated(g, (int32_t) i))
			continue;
		repair_graph_element(g, (int32_t) i, entry);
		nrep++;
	}
	/* MarkDeleted (hnswvacuum.c:594-729) */
	for (int64_t i = 0; i < g->n; i++)
		if (g->el[i].heaptidsLength == 0)
			for (int lc = 0; lc <= g->el[i].level; lc++)
				g->el[i].nbr[lc].length = 0;
	return nrep;
}
