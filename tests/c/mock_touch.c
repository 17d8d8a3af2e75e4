/* The CPU stand-in engine (mock_engine.c) with CMB200_TOUCH, TEST INFRASTRUCTURE ONLY
 * (tests/test_evict_logic.py).  An engine created with the flag raises the ts of every record a get
 * answers CMB200_HIT to CLOCK_REALTIME_COARSE in ns, as the engine's kernels do: cmb200_get_batch and
 * cmb200_get_small_end stamp their hits once the answers are in.  mock_engine_flags and mock_record_ts let a
 * test see the config flags an engine was created with and a record's ts.
 * Nothing of the product links against this file. */
#define cmb200_engine_create mock_base_engine_create
#define cmb200_engine_destroy mock_base_engine_destroy
#define cmb200_get_batch mock_base_get_batch
#define cmb200_get_small_end mock_base_get_small_end
#include "mock_engine.c"
#undef cmb200_engine_create
#undef cmb200_engine_destroy
#undef cmb200_get_batch
#undef cmb200_get_small_end

#include <time.h>

#define MAX_ENGINES 64

static pthread_mutex_t flags_mu = PTHREAD_MUTEX_INITIALIZER;
static cmb200_engine *flag_engine[MAX_ENGINES];
static uint32_t flag_value[MAX_ENGINES];

uint32_t mock_engine_flags(cmb200_engine *e) {
	uint32_t f = 0;
	pthread_mutex_lock(&flags_mu);
	for (int i = 0; i < MAX_ENGINES; i++)
		if (flag_engine[i] == e) f = flag_value[i];
	pthread_mutex_unlock(&flags_mu);
	return f;
}

cmb200_engine *cmb200_engine_create(const cmb200_config *cfg) {
	cmb200_engine *e = mock_base_engine_create(cfg);
	pthread_mutex_lock(&flags_mu);
	for (int i = 0; i < MAX_ENGINES; i++)
		if (!flag_engine[i]) { flag_engine[i] = e; flag_value[i] = cfg->flags; break; }
	pthread_mutex_unlock(&flags_mu);
	return e;
}

void cmb200_engine_destroy(cmb200_engine *e) {
	pthread_mutex_lock(&flags_mu);
	for (int i = 0; i < MAX_ENGINES; i++)
		if (flag_engine[i] == e) flag_engine[i] = NULL;
	pthread_mutex_unlock(&flags_mu);
	mock_base_engine_destroy(e);
}

/* raises the ts of the records of the requests answered CMB200_HIT (CMB200_TOUCH engines only) */
static void touch_hits(cmb200_engine *e, size_t n, const cmb200_addr *addr, const int32_t *status) {
	if (!(mock_engine_flags(e) & CMB200_TOUCH)) return;
	struct timespec tp;
	clock_gettime(CLOCK_REALTIME_COARSE, &tp);
	const uint64_t now = (uint64_t)tp.tv_sec * 1000000000ull + (uint64_t)tp.tv_nsec;
	pthread_mutex_lock(&e->mu);
	for (size_t i = 0; i < n; i++) {
		struct entry *s;
		if (status[i] == CMB200_HIT && lookup(e, &addr[i], &s) == CMB200_HIT && now > s->ts) s->ts = now;
	}
	pthread_mutex_unlock(&e->mu);
}

int cmb200_get_batch(cmb200_engine *e, size_t n, const cmb200_addr *addr, const uint8_t *valid, void *pages_out, int32_t *status_out) {
	const int rc = mock_base_get_batch(e, n, addr, valid, pages_out, status_out);
	if (rc == 0) touch_hits(e, n, addr, status_out);
	return rc;
}

int cmb200_get_small_end(cmb200_engine *e, cmb200_small_ticket *t, int32_t *status_out) {
	if (!t || t->lane < 0) return mock_base_get_small_end(e, t, status_out);
	/* the lane's addresses and statuses belong to this ticket until the base call frees the lane */
	const uint32_t n = t->n;
	cmb200_addr *addr = malloc((size_t)n * sizeof(cmb200_addr));
	int32_t *st = malloc((size_t)n * sizeof(int32_t));
	if (!addr || !st) { free(addr); free(st); return mock_base_get_small_end(e, t, status_out); }
	memcpy(addr, e->lane_addr[t->lane], (size_t)n * sizeof(cmb200_addr));
	const int rc = mock_base_get_small_end(e, t, st);
	if (rc == 0) {
		touch_hits(e, n, addr, st);
		if (status_out) memcpy(status_out, st, (size_t)n * sizeof(int32_t));
	}
	free(addr);
	free(st);
	return rc;
}

/* 1 and the ts of a's record, or 0 when a has none */
int mock_record_ts(cmb200_engine *e, const cmb200_addr *a, uint64_t *ts) {
	pthread_mutex_lock(&e->mu);
	struct entry *s;
	const int ok = lookup(e, a, &s) == CMB200_HIT;
	if (ok) *ts = s->ts;
	pthread_mutex_unlock(&e->mu);
	return ok;
}
