/* The CPU stand-in engine (mock_engine.c) with cmb200_patch_batch and the snapshot set calls, TEST
 * INFRASTRUCTURE ONLY (tests/test_patch_logic.py).  cmb200_patch_batch applies each patch in array order,
 * under the engine's lock, to the record its address holds, and logs it ("patch <engine> <u> <l>
 * <page_off> <len> <status>").  cmb200_save_set logs "save" and writes a small file through <path>.tmp and
 * a rename; cmb200_load_set finds nothing to load.  Nothing of the product links against this file. */
#include "mock_engine.c"

static pthread_mutex_t log_mu = PTHREAD_MUTEX_INITIALIZER;
static char patch_log[1 << 20];
static int engine_ids;

static void log_line(const char *line) {
	pthread_mutex_lock(&log_mu);
	const size_t used = strlen(patch_log), add = strlen(line);
	if (used + add + 2 < sizeof(patch_log)) {
		memcpy(patch_log + used, line, add);
		patch_log[used + add] = '\n';
		patch_log[used + add + 1] = '\0';
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

int cmb200_patch_batch(cmb200_engine *e, size_t n, const cmb200_addr *addr, const uint32_t *page_off,
    const uint32_t *len, const void *bytes_host, const uint64_t *ts, int32_t *status_out) {
	for (size_t i = 0; i < n; i++)
		if (len[i] == 0 || (uint64_t)page_off[i] + len[i] > e->bsize) { snprintf(err_buf, sizeof(err_buf), "mock: bad extent"); return -1; }
	const int id = engine_id(e);
	usleep(30);                                                   /* a launch and a copy take a while */
	const uint8_t *src = bytes_host;
	pthread_mutex_lock(&e->mu);
	for (size_t i = 0; i < n; i++) {
		struct entry *s;
		status_out[i] = lookup(e, &addr[i], &s);
		if (s) {
			memcpy(s->page + page_off[i], src, len[i]);
			s->ts = ts ? ts[i] : 0;
			e->puts++;
		}
		src += len[i];
		char line[160];
		snprintf(line, sizeof(line), "patch %d %llu %llu %u %u %d", id, (unsigned long long)addr[i].u,
		    (unsigned long long)addr[i].l, page_off[i], len[i], status_out[i]);
		log_line(line);
	}
	pthread_mutex_unlock(&e->mu);
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
	(void)engines; (void)g; (void)path;
	if (records_out) *records_out = 0;
	return 0;
}

/* the calls logged so far, one per line */
void mock_patch_log(char *out, size_t cap) {
	pthread_mutex_lock(&log_mu);
	snprintf(out, cap, "%s", patch_log);
	pthread_mutex_unlock(&log_mu);
}
