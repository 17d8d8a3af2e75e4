/* The CPU stand-in engine of mock_invalidate.c with cmb200_rename_set, TEST INFRASTRUCTURE ONLY
 * (tests/test_rename_logic.py).  cmb200_rename_set logs its arguments ("ren <g> <u_from> <u_to> <l_first>
 * <l_last>"), waits MOCK_RENAME_PAUSE_US microseconds and logs "ren-overlap" if any engine took a put
 * meanwhile, then takes every record stored at {u_from, l}, l in the interval, out of each engine under
 * that engine's lock and puts its page at {u_to, l} into engine cmb200_owner(key, g), and logs "ren-done
 * <moved>".  MOCK_RENAME_FAIL=1 makes it fail before anything changes.  Built with -DMOCK_NO_RENAME it is
 * left out, so that the drop-in sees the weak symbol absent.  Nothing of the product links this file. */
#include "mock_invalidate.c"

#ifndef MOCK_NO_RENAME
static uint64_t puts_of(cmb200_engine *const *engines, int g) {
	uint64_t n = 0;
	for (int i = 0; i < g; i++) {
		pthread_mutex_lock(&engines[i]->mu);
		n += engines[i]->puts;
		pthread_mutex_unlock(&engines[i]->mu);
	}
	return n;
}

int cmb200_rename_set(cmb200_engine *const *engines, int g, uint64_t u_from, uint64_t u_to,
    uint64_t l_first, uint64_t l_last, uint64_t *moved_out, uint64_t *dropped_out) {
	if (moved_out) *moved_out = 0;
	if (dropped_out) *dropped_out = 0;
	if (g < 1 || l_first > l_last) { snprintf(err_buf, sizeof(err_buf), "mock: bad rename"); return -1; }
	char line[200];
	snprintf(line, sizeof(line), "ren %d %llu %llu %llu %llu", g, (unsigned long long)u_from,
	    (unsigned long long)u_to, (unsigned long long)l_first, (unsigned long long)l_last);
	log_line(line);
	const char *fail = getenv("MOCK_RENAME_FAIL");
	if (fail && atoi(fail)) { snprintf(err_buf, sizeof(err_buf), "mock: rename fails"); return -1; }
	const char *pause = getenv("MOCK_RENAME_PAUSE_US");
	if (pause && atoi(pause)) {
		const uint64_t before = puts_of(engines, g);
		usleep((useconds_t)atoi(pause));
		if (puts_of(engines, g) != before) log_line("ren-overlap");
	}
	if (u_from == u_to) { log_line("ren-done 0"); return 0; }
	uint64_t moved = 0;
	const uint32_t bsize = engines[0]->bsize;
	for (int i = 0; i < g; i++) {
		cmb200_engine *e = engines[i];
		size_t n = 0, cap = 16;
		cmb200_addr *to = malloc(cap * sizeof(*to));
		uint8_t *pages = malloc(cap * bsize);
		uint64_t *ts = malloc(cap * sizeof(*ts));
		pthread_mutex_lock(&e->mu);
		for (uint32_t k = 0; k < SLOTS; k++) {
			struct entry *s = &e->tab[k];
			if (s->used != 1 || s->a.u != u_from || s->a.l < l_first || s->a.l > l_last) continue;
			if (n == cap) {
				cap *= 2;
				to = realloc(to, cap * sizeof(*to));
				pages = realloc(pages, cap * bsize);
				ts = realloc(ts, cap * sizeof(*ts));
			}
			to[n] = (cmb200_addr){ u_to, s->a.l };
			memcpy(pages + n * bsize, s->page, bsize);
			ts[n] = s->ts;
			n++;
			s->used = 2;
			e->entries--;
		}
		pthread_mutex_unlock(&e->mu);
		for (size_t k = 0; k < n; k++)
			cmb200_put_batch(engines[cmb200_owner(addr_key(&to[k]), g)], 1, &to[k], NULL, pages + k * bsize, &ts[k], NULL);
		moved += n;
		free(to);
		free(pages);
		free(ts);
	}
	snprintf(line, sizeof(line), "ren-done %llu", (unsigned long long)moved);
	log_line(line);
	if (moved_out) *moved_out = moved;
	return 0;
}
#endif
