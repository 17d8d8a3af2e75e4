/* The CPU stand-in engine (mock_engine.c) with a host tier, TEST INFRASTRUCTURE ONLY
 * (tests/test_host_tier_logic.py).  It compiles mock_engine.c into this file with its put, unset,
 * create and stats entry points renamed, and wraps them: the engine gets an arena of cfg->arena_bytes
 * whose arena_used counts the pages outside the tier, so that the drop-in's arena check demotes, and
 * a tier that is a ring of tier_bytes / bsize pages which unsets the oldest demoted key still in it
 * when it comes round.  One engine per process (host_stress makes one).  Nothing of the product
 * links against this file. */
#define cmb200_engine_create mock_base_engine_create
#define cmb200_engine_destroy mock_base_engine_destroy
#define cmb200_put_batch mock_base_put_batch
#define cmb200_unset_batch mock_base_unset_batch
#define cmb200_get_stats mock_base_get_stats
#include "mock_engine.c"
#undef cmb200_engine_create
#undef cmb200_engine_destroy
#undef cmb200_put_batch
#undef cmb200_unset_batch
#undef cmb200_get_stats

static struct {
	uint64_t arena_bytes;
	uint8_t *in_tier;               /* per slot of the stand-in's table */
	uint64_t *tier_pos;
	cmb200_addr *ring;              /* ring[pos % tier_n] = key demoted at position pos */
	uint64_t tier_n, tier_head, records, demoted, retired;
} tier;

cmb200_engine *cmb200_engine_create(const cmb200_config *cfg) {
	tier.arena_bytes = cfg->arena_bytes ? cfg->arena_bytes : 1ull << 40;
	tier.in_tier = calloc(SLOTS, 1);
	tier.tier_pos = calloc(SLOTS, sizeof(uint64_t));
	return mock_base_engine_create(cfg);
}

void cmb200_engine_destroy(cmb200_engine *e) {
	if (tier.ring) fprintf(stderr, "mock host tier: demoted %lu retired %lu\n", (unsigned long)tier.demoted, (unsigned long)tier.retired);
	mock_base_engine_destroy(e);
	free(tier.ring); free(tier.in_tier); free(tier.tier_pos);
	memset(&tier, 0, sizeof(tier));
}

/* a key that leaves the tier (put again: the new record goes to the arena; or unset) */
static void leave_tier(cmb200_engine *e, const cmb200_addr *a) {
	int present;
	struct entry *s = find(e, a, &present);
	if (s && tier.in_tier[s - e->tab]) { tier.in_tier[s - e->tab] = 0; tier.records--; }
}

int cmb200_put_batch(cmb200_engine *e, size_t n, const cmb200_addr *addr, const uint8_t *valid, const void *pages,
    const uint64_t *ts, int32_t *lens_out) {
	const int rc = mock_base_put_batch(e, n, addr, valid, pages, ts, lens_out);
	pthread_mutex_lock(&e->mu);
	for (size_t i = 0; i < n; i++)
		if (!valid || valid[i]) leave_tier(e, &addr[i]);
	pthread_mutex_unlock(&e->mu);
	return rc;
}

int cmb200_unset_batch(cmb200_engine *e, size_t n, const cmb200_addr *addr) {
	pthread_mutex_lock(&e->mu);
	for (size_t i = 0; i < n; i++) leave_tier(e, &addr[i]);
	pthread_mutex_unlock(&e->mu);
	return mock_base_unset_batch(e, n, addr);
}

int cmb200_get_stats(cmb200_engine *e, cmb200_stats *out) {
	mock_base_get_stats(e, out);
	pthread_mutex_lock(&e->mu);
	out->arena_bytes = tier.arena_bytes;
	out->arena_used = (e->entries - tier.records) * (uint64_t)e->bsize;
	pthread_mutex_unlock(&e->mu);
	return 0;
}

int cmb200_host_tier_enable(cmb200_engine *e, uint64_t bytes) {
	pthread_mutex_lock(&e->mu);
	int rc = -1;
	if (!tier.ring && bytes / e->bsize >= 4) {
		tier.tier_n = bytes / e->bsize;
		tier.ring = calloc(tier.tier_n, sizeof(cmb200_addr));
		rc = tier.ring ? 0 : -1;
	}
	pthread_mutex_unlock(&e->mu);
	return rc;
}

int cmb200_demote_batch(cmb200_engine *e, size_t n, const cmb200_addr *addr, uint64_t *demoted_out) {
	if (demoted_out) *demoted_out = 0;
	pthread_mutex_lock(&e->mu);
	if (!tier.ring) { pthread_mutex_unlock(&e->mu); return -1; }
	uint64_t done = 0;
	for (size_t i = 0; i < n; i++) {
		int present;
		struct entry *s = find(e, &addr[i], &present);
		if (!present || tier.in_tier[s - e->tab]) continue;
		if (tier.tier_head >= tier.tier_n) {                      /* the ring comes round: retire the oldest */
			const uint64_t pos = tier.tier_head - tier.tier_n;
			int there;
			struct entry *o = find(e, &tier.ring[pos % tier.tier_n], &there);
			if (there && tier.in_tier[o - e->tab] && tier.tier_pos[o - e->tab] == pos) {
				o->used = 2; tier.in_tier[o - e->tab] = 0; e->entries--; tier.records--; tier.retired++;
			}
		}
		tier.ring[tier.tier_head % tier.tier_n] = addr[i];
		tier.in_tier[s - e->tab] = 1; tier.tier_pos[s - e->tab] = tier.tier_head++;
		tier.records++; done++;
	}
	tier.demoted += done;
	pthread_mutex_unlock(&e->mu);
	if (demoted_out) *demoted_out = done;
	return 0;
}

int cmb200_host_tier_stats(cmb200_engine *e, struct cmb200_host_tier_stats *out) {
	memset(out, 0, sizeof(*out));
	pthread_mutex_lock(&e->mu);
	if (tier.ring) {
		out->bytes = tier.tier_n * e->bsize;
		out->used = (tier.tier_head < tier.tier_n ? tier.tier_head : tier.tier_n) * e->bsize;
		out->records = tier.records;
		out->demoted_records = tier.demoted; out->demoted_bytes = tier.demoted * e->bsize;
		out->retired_records = tier.retired;
	}
	pthread_mutex_unlock(&e->mu);
	return 0;
}
