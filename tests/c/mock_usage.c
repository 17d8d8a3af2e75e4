/* The CPU stand-in engine with pins (mock_pin.c) and the usage calls, TEST INFRASTRUCTURE ONLY
 * (tests/test_usage_logic.py).  cmb200_residency marks every record of {u, l} in the interval (all in the
 * arena: the stand-in has no tier); cmb200_usage_set groups every engine's records by (u, genid) with the
 * stand-in's record length, 24 + the page (pages are kept raw), and orders the rows as the engine does.
 * cmb200_invalidate removes an interval's records, as the engine does.  mock_usage_fail(e) makes both usage
 * calls fail on engine e (NULL: none).  Nothing of the product links against this file. */
#include "mock_pin.c"

static cmb200_engine *usage_fail;

void mock_usage_fail(cmb200_engine *e) { __atomic_store_n(&usage_fail, e, __ATOMIC_RELEASE); }

static int fails(cmb200_engine *e) {
	if (__atomic_load_n(&usage_fail, __ATOMIC_ACQUIRE) != e) return 0;
	snprintf(err_buf, sizeof(err_buf), "mock: this engine cannot answer");
	return 1;
}

int cmb200_invalidate(cmb200_engine *e, uint64_t u, uint64_t l_first, uint64_t l_last, uint64_t *removed_out) {
	uint64_t n = 0;
	pthread_mutex_lock(&e->mu);
	for (uint32_t i = 0; i < SLOTS; i++) {
		struct entry *s = &e->tab[i];
		if (s->used == 1 && s->a.u == u && s->a.l >= l_first && s->a.l <= l_last) {
			s->used = 2;
			e->entries--;
			n++;
		}
	}
	pthread_mutex_unlock(&e->mu);
	if (removed_out) *removed_out = n;
	return 0;
}

int cmb200_residency(cmb200_engine *e, uint64_t u, uint64_t l_first, uint64_t l_last, uint8_t *out) {
	if (l_first > l_last || fails(e)) return -1;
	pthread_mutex_lock(&e->mu);
	for (uint32_t i = 0; i < SLOTS; i++) {
		const struct entry *s = &e->tab[i];
		if (s->used == 1 && s->a.u == u && s->a.l >= l_first && s->a.l <= l_last) out[s->a.l - l_first] = 1;
	}
	pthread_mutex_unlock(&e->mu);
	return 0;
}

static int row_key_cmp(const void *a, const void *b) {
	const cmb200_object_usage *x = a, *y = b;
	if (x->u != y->u) return x->u < y->u ? -1 : 1;
	return x->genid < y->genid ? -1 : x->genid > y->genid;
}

static int row_order_cmp(const void *a, const void *b) {
	const cmb200_object_usage *x = a, *y = b;
	if (x->stored_bytes != y->stored_bytes) return x->stored_bytes > y->stored_bytes ? -1 : 1;
	return row_key_cmp(a, b);
}

int cmb200_usage_set(cmb200_engine *const *engines, int g, size_t max, cmb200_object_usage *out, uint64_t *objects_out) {
	for (int k = 0; k < g; k++)
		if (fails(engines[k])) return -1;
	size_t n = 0, cap = 1024;
	cmb200_object_usage *r = malloc(cap * sizeof(*r));
	for (int k = 0; k < g; k++) {
		cmb200_engine *e = engines[k];
		pthread_mutex_lock(&pin_mu);
		pthread_mutex_lock(&e->mu);
		const struct pins *p = pins_of(e);
		for (uint32_t i = 0; i < SLOTS; i++) {
			const struct entry *s = &e->tab[i];
			if (s->used != 1) continue;
			if (n == cap) r = realloc(r, (cap *= 2) * sizeof(*r));
			const uint64_t page = s->a.l & ((1ull << 44) - 1);
			r[n++] = (cmb200_object_usage){ s->a.u, (uint32_t)(s->a.l >> 44), 0, 1, 0, (uint64_t)pinned(p, &s->a),
			    24u + e->bsize, page, page, s->ts, s->ts };
		}
		pthread_mutex_unlock(&e->mu);
		pthread_mutex_unlock(&pin_mu);
	}
	qsort(r, n, sizeof(*r), row_key_cmp);
	size_t m = 0;
	for (size_t i = 0; i < n; i++) {
		if (m && row_key_cmp(&r[m - 1], &r[i]) == 0) {
			cmb200_object_usage *a = &r[m - 1];
			a->pages += r[i].pages; a->tier_pages += r[i].tier_pages; a->pinned_pages += r[i].pinned_pages;
			a->stored_bytes += r[i].stored_bytes;
			if (r[i].first_page < a->first_page) a->first_page = r[i].first_page;
			if (r[i].last_page > a->last_page) a->last_page = r[i].last_page;
			if (r[i].oldest_ts < a->oldest_ts) a->oldest_ts = r[i].oldest_ts;
			if (r[i].newest_ts > a->newest_ts) a->newest_ts = r[i].newest_ts;
		} else {
			r[m++] = r[i];
		}
	}
	qsort(r, m, sizeof(*r), row_order_cmp);
	memcpy(out, r, (max < m ? max : m) * sizeof(*r));
	free(r);
	if (objects_out) *objects_out = m;
	return 0;
}
