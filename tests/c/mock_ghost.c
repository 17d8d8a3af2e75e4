/* The CPU stand-in engine (mock_engine.c) with CMB200_GHOST, TEST INFRASTRUCTURE ONLY
 * (tests/test_ghost_logic.py).  It counts, per engine, the addresses that reach it through
 * cmb200_evict_batch (an engine created with the flag; -1 otherwise) and through cmb200_unset_batch;
 * both remove as cmb200_unset_batch does.  cmb200_ghost_stats answers a table of 256 entries (buckets of
 * 4) whose histogram and probe count a test sets with mock_ghost_set_hist.  For CMB200_ADMIT=freq,
 * cmb200_freq_estimate answers 15 for pages l >= MOCK_HOT_FROM and 0 below.
 * mock_engine_flags lets a test see the config flags an engine was created with.
 * Nothing of the product links against this file. */
#define cmb200_engine_create mock_base_engine_create
#define cmb200_engine_destroy mock_base_engine_destroy
#define cmb200_unset_batch mock_base_unset_batch
#include "mock_engine.c"
#undef cmb200_engine_create
#undef cmb200_engine_destroy
#undef cmb200_unset_batch

#define MAX_ENGINES 64
#define MOCK_HOT_FROM 5000

struct ghosts {
	cmb200_engine *e;
	uint32_t flags;
	uint64_t evicted, unset, probes;
	uint64_t hist[64];
};

static pthread_mutex_t gh_mu = PTHREAD_MUTEX_INITIALIZER;
static struct ghosts gh[MAX_ENGINES];

static struct ghosts *ghosts_of(cmb200_engine *e) {
	for (int i = 0; i < MAX_ENGINES; i++)
		if (gh[i].e == e) return &gh[i];
	return NULL;
}

uint32_t mock_engine_flags(cmb200_engine *e) {
	pthread_mutex_lock(&gh_mu);
	struct ghosts *g = ghosts_of(e);
	const uint32_t f = g ? g->flags : 0;
	pthread_mutex_unlock(&gh_mu);
	return f;
}

void mock_ghost_counts(cmb200_engine *e, uint64_t *evicted, uint64_t *unset) {
	pthread_mutex_lock(&gh_mu);
	struct ghosts *g = ghosts_of(e);
	*evicted = g ? g->evicted : 0;
	*unset = g ? g->unset : 0;
	pthread_mutex_unlock(&gh_mu);
}

void mock_ghost_set_hist(cmb200_engine *e, const uint64_t *hist, uint64_t probes) {
	pthread_mutex_lock(&gh_mu);
	struct ghosts *g = ghosts_of(e);
	if (g) { memcpy(g->hist, hist, sizeof(g->hist)); g->probes = probes; }
	pthread_mutex_unlock(&gh_mu);
}

cmb200_engine *cmb200_engine_create(const cmb200_config *cfg) {
	cmb200_engine *e = mock_base_engine_create(cfg);
	if (!e) return NULL;
	pthread_mutex_lock(&gh_mu);
	struct ghosts *g = ghosts_of(NULL);
	if (g) { memset(g, 0, sizeof(*g)); g->e = e; g->flags = cfg->flags; }
	pthread_mutex_unlock(&gh_mu);
	return e;
}

void cmb200_engine_destroy(cmb200_engine *e) {
	pthread_mutex_lock(&gh_mu);
	struct ghosts *g = ghosts_of(e);
	if (g) memset(g, 0, sizeof(*g));
	pthread_mutex_unlock(&gh_mu);
	mock_base_engine_destroy(e);
}

int cmb200_unset_batch(cmb200_engine *e, size_t n, const cmb200_addr *addr) {
	pthread_mutex_lock(&gh_mu);
	struct ghosts *g = ghosts_of(e);
	if (g) g->unset += n;
	pthread_mutex_unlock(&gh_mu);
	return mock_base_unset_batch(e, n, addr);
}

int cmb200_evict_batch(cmb200_engine *e, size_t n, const cmb200_addr *addr, uint64_t *evicted_out) {
	pthread_mutex_lock(&gh_mu);
	struct ghosts *g = ghosts_of(e);
	const int ok = g && (g->flags & CMB200_GHOST);
	if (ok) g->evicted += n;
	pthread_mutex_unlock(&gh_mu);
	if (!ok) { snprintf(err_buf, sizeof(err_buf), "mock: no CMB200_GHOST"); return -1; }
	if (evicted_out) *evicted_out = n;
	return mock_base_unset_batch(e, n, addr);
}

int cmb200_ghost_stats(cmb200_engine *e, struct cmb200_ghost_stats *out) {
	pthread_mutex_lock(&gh_mu);
	struct ghosts *g = ghosts_of(e);
	const int ok = g && (g->flags & CMB200_GHOST);
	if (ok) {
		memset(out, 0, sizeof(*out));
		out->entries = 256;
		out->bucket_width = 4;
		out->clock = out->inserted = g->evicted;
		out->probes = g->probes;
		memcpy(out->hist, g->hist, sizeof(out->hist));
		for (int k = 0; k < 64; k++) out->refaults += g->hist[k];
	}
	pthread_mutex_unlock(&gh_mu);
	return ok ? 0 : -1;
}

int cmb200_freq_estimate(cmb200_engine *e, size_t n, const cmb200_addr *addr, uint8_t *est_out) {
	if (!(mock_engine_flags(e) & CMB200_FREQ)) { snprintf(err_buf, sizeof(err_buf), "mock: no CMB200_FREQ"); return -1; }
	for (size_t i = 0; i < n; i++) est_out[i] = (addr[i].l & ((1ull << 44) - 1)) >= MOCK_HOT_FROM ? 15 : 0;
	return 0;
}
