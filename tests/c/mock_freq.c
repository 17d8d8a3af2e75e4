/* The CPU stand-in engine (mock_engine.c) with CMB200_FREQ, TEST INFRASTRUCTURE ONLY
 * (tests/test_admit_logic.py).  An engine created with the flag keeps the count-min sketch of
 * cachemap_b200.h with the header's index function: cmb200_get_batch counts every request with a valid
 * address, cmb200_get_small_begin every request, and the call that takes the count since the last halving
 * to 10 x capacity halves every counter; cmb200_freq_estimate, _read and _stats read it.
 * mock_engine_flags lets a test see the config flags an engine was created with.
 * Nothing of the product links against this file. */
#define cmb200_engine_create mock_base_engine_create
#define cmb200_engine_destroy mock_base_engine_destroy
#define cmb200_get_batch mock_base_get_batch
#define cmb200_get_small_begin mock_base_get_small_begin
#include "mock_engine.c"
#undef cmb200_engine_create
#undef cmb200_engine_destroy
#undef cmb200_get_batch
#undef cmb200_get_small_begin

#define MAX_ENGINES 64

struct sketch {
	cmb200_engine *e;
	uint32_t flags;
	uint8_t *c;             /* 4 x width counters, one byte each */
	int log2w;
	uint64_t width, period, increments, since, halvings;
};

static pthread_mutex_t sk_mu = PTHREAD_MUTEX_INITIALIZER;
static struct sketch sk[MAX_ENGINES];

static struct sketch *sketch_of(cmb200_engine *e) {
	for (int i = 0; i < MAX_ENGINES; i++)
		if (sk[i].e == e) return &sk[i];
	return NULL;
}

uint32_t mock_engine_flags(cmb200_engine *e) {
	pthread_mutex_lock(&sk_mu);
	struct sketch *s = sketch_of(e);
	const uint32_t f = s ? s->flags : 0;
	pthread_mutex_unlock(&sk_mu);
	return f;
}

cmb200_engine *cmb200_engine_create(const cmb200_config *cfg) {
	cmb200_engine *e = mock_base_engine_create(cfg);
	if (!e) return NULL;
	pthread_mutex_lock(&sk_mu);
	struct sketch *s = sketch_of(NULL);
	if (s) {
		memset(s, 0, sizeof(*s));
		s->e = e;
		s->flags = cfg->flags;
		if (cfg->flags & CMB200_FREQ) {
			uint64_t w = 16;
			while (w < cfg->capacity) w <<= 1;
			while ((1ull << s->log2w) < w) s->log2w++;
			s->width = w;
			s->period = 10 * cfg->capacity;
			s->c = calloc(4, w);
		}
	}
	pthread_mutex_unlock(&sk_mu);
	return e;
}

void cmb200_engine_destroy(cmb200_engine *e) {
	pthread_mutex_lock(&sk_mu);
	struct sketch *s = sketch_of(e);
	if (s) { free(s->c); memset(s, 0, sizeof(*s)); }
	pthread_mutex_unlock(&sk_mu);
	mock_base_engine_destroy(e);
}

/* one counting launch of n requests */
static void count(cmb200_engine *e, size_t n, const cmb200_addr *addr, const uint8_t *valid) {
	pthread_mutex_lock(&sk_mu);
	struct sketch *s = sketch_of(e);
	if (s && s->c) {
		uint64_t k = 0;
		for (size_t i = 0; i < n; i++) {
			if (valid && !valid[i]) continue;
			const uint64_t key = addr_key(&addr[i]);
			for (int r = 0; r < 4; r++) {
				uint8_t *c = &s->c[(uint64_t)r * s->width + cmb200_freq_index(key, r, s->log2w)];
				if (*c < 15) (*c)++;
			}
			k++;
		}
		s->increments += k;
		s->since += k;
		if (s->since >= s->period) {
			for (uint64_t j = 0; j < 4 * s->width; j++) s->c[j] >>= 1;
			s->since = 0;
			s->halvings++;
		}
	}
	pthread_mutex_unlock(&sk_mu);
}

int cmb200_get_batch(cmb200_engine *e, size_t n, const cmb200_addr *addr, const uint8_t *valid, void *pages_out, int32_t *status_out) {
	count(e, n, addr, valid);
	return mock_base_get_batch(e, n, addr, valid, pages_out, status_out);
}

int cmb200_get_small_begin(cmb200_engine *e, size_t n, const cmb200_addr *addr, void *pages_out, cmb200_small_ticket *t) {
	const int rc = mock_base_get_small_begin(e, n, addr, pages_out, t);
	if (rc == 0) count(e, n, addr, NULL);
	return rc;
}

int cmb200_freq_estimate(cmb200_engine *e, size_t n, const cmb200_addr *addr, uint8_t *est_out) {
	pthread_mutex_lock(&sk_mu);
	struct sketch *s = sketch_of(e);
	const int ok = s && s->c;
	for (size_t i = 0; ok && i < n; i++) {
		const uint64_t key = addr_key(&addr[i]);
		uint8_t m = 15;
		for (int r = 0; r < 4; r++) {
			const uint8_t c = s->c[(uint64_t)r * s->width + cmb200_freq_index(key, r, s->log2w)];
			if (c < m) m = c;
		}
		est_out[i] = m;
	}
	pthread_mutex_unlock(&sk_mu);
	if (!ok) snprintf(err_buf, sizeof(err_buf), "mock: no CMB200_FREQ");
	return ok ? 0 : -1;
}

int cmb200_freq_stats(cmb200_engine *e, struct cmb200_freq_stats *out) {
	pthread_mutex_lock(&sk_mu);
	struct sketch *s = sketch_of(e);
	const int ok = s && s->c;
	if (ok) *out = (struct cmb200_freq_stats){ s->width, s->period, s->increments, s->since, s->halvings };
	pthread_mutex_unlock(&sk_mu);
	return ok ? 0 : -1;
}
