/* The CPU stand-in engine (mock_engine.c) with cmb200_invalidate and snapshot set calls, TEST
 * INFRASTRUCTURE ONLY (tests/test_invalidate_logic.py).  cmb200_invalidate removes, under the engine's
 * lock, every record whose stored address has u == u and l_first <= l <= l_last, and logs the interval
 * it was given ("inv <engine> <u> <l_first> <l_last> <removed>").  cmb200_save_set logs "save" and writes
 * a small file through <path>.tmp and a rename; cmb200_load_set logs "load" and puts MOCK_LOAD_PAGES
 * pages of object MOCK_LOAD_NHID, genid 0, pages 0.., into the engines (each page to the engine of its
 * key), so that a driver can see whether a call was applied to the loaded store or overwritten by it.
 * Nothing of the product links against this file. */
#include "mock_engine.c"

static pthread_mutex_t log_mu = PTHREAD_MUTEX_INITIALIZER;
static char inv_log[1 << 16];
static int engine_ids;

static void log_line(const char *line) {
	pthread_mutex_lock(&log_mu);
	if (strlen(inv_log) + strlen(line) + 2 < sizeof(inv_log)) {
		strcat(inv_log, line);
		strcat(inv_log, "\n");
	}
	pthread_mutex_unlock(&log_mu);
}

/* engines are numbered in creation order, which is CMB200_DEVICES order */
static int engine_id(cmb200_engine *e) {
	static cmb200_engine *seen[64];
	pthread_mutex_lock(&log_mu);
	int i = 0;
	while (i < engine_ids && seen[i] != e) i++;
	if (i == engine_ids && i < 64) seen[engine_ids++] = e;
	pthread_mutex_unlock(&log_mu);
	return i;
}

int cmb200_invalidate(cmb200_engine *e, uint64_t u, uint64_t l_first, uint64_t l_last, uint64_t *removed_out) {
	if (l_first > l_last) { snprintf(err_buf, sizeof(err_buf), "mock: l_first > l_last"); return -1; }
	uint64_t removed = 0;
	pthread_mutex_lock(&e->mu);
	for (uint32_t i = 0; i < SLOTS; i++) {
		struct entry *s = &e->tab[i];
		if (s->used == 1 && s->a.u == u && s->a.l >= l_first && s->a.l <= l_last) { s->used = 2; e->entries--; removed++; }
	}
	pthread_mutex_unlock(&e->mu);
	char line[160];
	snprintf(line, sizeof(line), "inv %d %llu %llu %llu %llu", engine_id(e), (unsigned long long)u,
	    (unsigned long long)l_first, (unsigned long long)l_last, (unsigned long long)removed);
	log_line(line);
	if (removed_out) *removed_out = removed;
	return 0;
}

int cmb200_save_set(cmb200_engine *const *engines, int g, const char *path, uint64_t *records_out) {
	(void)engines; (void)g;
	log_line("save");
	if (records_out) *records_out = 0;
	char tmp[2400];
	snprintf(tmp, sizeof(tmp), "%s.tmp", path);
	FILE *f = fopen(tmp, "wb");
	if (!f) return -1;
	const int ok = fputs("mock snapshot\n", f) >= 0;
	if (fclose(f) != 0 || !ok) return -1;
	return rename(tmp, path) == 0 ? 0 : -1;
}

int cmb200_load_set(cmb200_engine *const *engines, int g, const char *path, uint64_t *records_out) {
	(void)path;
	log_line("load");
	const char *v = getenv("MOCK_LOAD_PAGES");
	const uint64_t n = v ? strtoull(v, NULL, 0) : 0;
	const char *h = getenv("MOCK_LOAD_NHID");
	const uint64_t nhid = h ? strtoull(h, NULL, 0) : 7;
	uint8_t *page = calloc(1, engines[0]->bsize);
	for (uint64_t p = 0; p < n; p++) {
		cmb200_addr a = { nhid, p };
		memset(page, (int)(p + 1), engines[0]->bsize);
		cmb200_put_batch(engines[cmb200_owner(addr_key(&a), g)], 1, &a, NULL, page, NULL, NULL);
	}
	free(page);
	if (records_out) *records_out = n;
	return 0;
}

/* the calls logged so far, one per line */
void mock_invalidate_log(char *out, size_t cap) {
	pthread_mutex_lock(&log_mu);
	snprintf(out, cap, "%s", inv_log);
	pthread_mutex_unlock(&log_mu);
}
