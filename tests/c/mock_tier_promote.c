/* The CPU stand-in engine with a host tier (mock_host_tier.c) that can also promote, TEST
 * INFRASTRUCTURE ONLY (tests/test_tier_promote_logic.py).  It compiles mock_host_tier.c into this file
 * with the stand-in's two get entry points renamed and wraps them: a get of a key that is in the tier
 * logs the key, as the engine's kernels log tier hits.  cmb200_host_tier_hot drains that log and
 * cmb200_promote_batch moves tier keys back to the arena while the arena has room for a page.  The
 * totals are printed when the process exits.  Nothing of the product links against this file. */
#define cmb200_get_small_begin mock_base_get_small_begin
#define cmb200_get_batch mock_base_get_batch
#include "mock_host_tier.c"
#undef cmb200_get_small_begin
#undef cmb200_get_batch

#define HOT_N 4096

static struct {
	cmb200_addr log[HOT_N];
	uint64_t head, drained;
	uint64_t promoted, hot_drains;
} promo;

/* the tier keys among addr (e->mu held) */
static void log_tier_hits(cmb200_engine *e, size_t n, const cmb200_addr *addr) {
	for (size_t i = 0; i < n; i++) {
		int present;
		struct entry *s = find(e, &addr[i], &present);
		if (present && tier.in_tier[s - e->tab]) promo.log[promo.head++ % HOT_N] = addr[i];
	}
}

int cmb200_get_small_begin(cmb200_engine *e, size_t n, const cmb200_addr *addr, void *pages_out, cmb200_small_ticket *t) {
	pthread_mutex_lock(&e->mu);
	log_tier_hits(e, n, addr);
	pthread_mutex_unlock(&e->mu);
	return mock_base_get_small_begin(e, n, addr, pages_out, t);
}

int cmb200_get_batch(cmb200_engine *e, size_t n, const cmb200_addr *addr, const uint8_t *valid, void *pages_out, int32_t *status_out) {
	pthread_mutex_lock(&e->mu);
	log_tier_hits(e, n, addr);
	pthread_mutex_unlock(&e->mu);
	return mock_base_get_batch(e, n, addr, valid, pages_out, status_out);
}

int cmb200_host_tier_hot(cmb200_engine *e, size_t max, cmb200_addr *addr_out, size_t *n_out, uint64_t *lost_out) {
	pthread_mutex_lock(&e->mu);
	const uint64_t since = promo.head - promo.drained, from = since > HOT_N ? promo.head - HOT_N : promo.drained;
	if (lost_out) *lost_out = since > HOT_N ? since - HOT_N : 0;
	size_t k = 0;
	for (uint64_t p = promo.head; p > from && k < max; p--) {          /* newest first, distinct */
		const cmb200_addr a = promo.log[(p - 1) % HOT_N];
		int dup = 0;
		for (size_t j = 0; j < k && !dup; j++) dup = addr_out[j].u == a.u && addr_out[j].l == a.l;
		if (!dup) addr_out[k++] = a;
	}
	promo.drained = promo.head;
	promo.hot_drains++;
	pthread_mutex_unlock(&e->mu);
	*n_out = k;
	return 0;
}

int cmb200_promote_batch(cmb200_engine *e, size_t n, const cmb200_addr *addr, uint64_t *promoted_out) {
	if (promoted_out) *promoted_out = 0;
	pthread_mutex_lock(&e->mu);
	if (!tier.ring) { pthread_mutex_unlock(&e->mu); return -1; }
	uint64_t done = 0;
	for (size_t i = 0; i < n; i++) {
		int present;
		struct entry *s = find(e, &addr[i], &present);
		if (!present || !tier.in_tier[s - e->tab]) continue;
		if ((e->entries - tier.records + 1) * (uint64_t)e->bsize > tier.arena_bytes) break;   /* no free arena bytes */
		tier.in_tier[s - e->tab] = 0; tier.records--; done++;
	}
	promo.promoted += done;
	pthread_mutex_unlock(&e->mu);
	if (promoted_out) *promoted_out = done;
	return 0;
}

__attribute__((destructor)) static void promo_report(void) {
	fprintf(stderr, "mock tier promote: promoted %lu drains %lu\n", (unsigned long)promo.promoted, (unsigned long)promo.hot_drains);
}
