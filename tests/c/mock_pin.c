/* The CPU stand-in engine (mock_engine.c) with pins, TEST INFRASTRUCTURE ONLY (tests/test_pin_logic.py).
 * cmb200_pin_set keeps each engine's list (and refuses unsorted or overlapping ranges, as the engine does);
 * cmb200_sample passes over pinned records; cmb200_pin_count counts the pinned records (none is in a tier);
 * cmb200_pin_promote moves nothing.  mock_pin_list lets a test read an engine's list and how many lists
 * it was given.  cmb200_aead_seal_batch is a keyed FNV-1a stand-in with the real call's shape:
 * the drop-in's framing of a sealed pins file is what is tested here, the cipher on the GPU.  For
 * CMB200_ADMIT=freq, cmb200_freq_estimate answers 15 for pages l >= MOCK_HOT_FROM and 0 below.
 * Nothing of the product links against this file. */
#define cmb200_sample mock_base_sample
#define cmb200_engine_destroy mock_base_engine_destroy
#include "mock_engine.c"
#undef cmb200_sample
#undef cmb200_engine_destroy

#define MAX_ENGINES 64
#define MOCK_HOT_FROM 5000

struct pins {
	cmb200_engine *e;
	size_t n;
	uint64_t sets;
	cmb200_pin_range r[CMB200_PIN_RANGES];
};

static pthread_mutex_t pin_mu = PTHREAD_MUTEX_INITIALIZER;
static struct pins pn[MAX_ENGINES];

static struct pins *pins_of(cmb200_engine *e) {
	for (int i = 0; i < MAX_ENGINES; i++)
		if (pn[i].e == e) return &pn[i];
	return NULL;
}

static int pinned(const struct pins *p, const cmb200_addr *a) {
	for (size_t k = 0; p && k < p->n; k++)
		if (p->r[k].u == a->u && p->r[k].l_first <= a->l && a->l <= p->r[k].l_last) return 1;
	return 0;
}

void cmb200_engine_destroy(cmb200_engine *e) {
	pthread_mutex_lock(&pin_mu);
	struct pins *p = pins_of(e);
	if (p) p->e = NULL;
	pthread_mutex_unlock(&pin_mu);
	mock_base_engine_destroy(e);
}

int cmb200_pin_set(cmb200_engine *e, size_t n, const cmb200_pin_range *r) {
	if (n > CMB200_PIN_RANGES) return -1;
	for (size_t k = 0; k < n; k++)
		if (r[k].l_first > r[k].l_last ||
		    (k && !(r[k].u > r[k - 1].u || (r[k].u == r[k - 1].u && r[k].l_first > r[k - 1].l_last)))) {
			snprintf(err_buf, sizeof(err_buf), "mock: ranges not sorted and disjoint");
			return -1;
		}
	pthread_mutex_lock(&pin_mu);
	struct pins *p = pins_of(e);
	if (!p && (p = pins_of(NULL))) { p->e = e; p->sets = 0; }
	if (p) { memcpy(p->r, r, n * sizeof(*r)); p->n = n; p->sets++; }
	pthread_mutex_unlock(&pin_mu);
	return p ? 0 : -1;
}

size_t mock_pin_list(cmb200_engine *e, cmb200_pin_range *out, size_t max, uint64_t *sets) {
	pthread_mutex_lock(&pin_mu);
	struct pins *p = pins_of(e);
	const size_t n = p ? (p->n < max ? p->n : max) : 0;
	if (p) memcpy(out, p->r, n * sizeof(*out));
	if (sets) *sets = p ? p->sets : 0;
	pthread_mutex_unlock(&pin_mu);
	return n;
}

int cmb200_sample(cmb200_engine *e, size_t n, const uint64_t *r, cmb200_addr *addr_out, uint64_t *ts_out, int32_t *ok_out) {
	pthread_mutex_lock(&pin_mu);
	pthread_mutex_lock(&e->mu);
	const struct pins *p = pins_of(e);
	for (size_t k = 0; k < n; k++) {
		ok_out[k] = 0;
		uint64_t i = r[k] & (SLOTS - 1);
		for (uint32_t step = 0; step < SLOTS; step++, i = (i + 1) & (SLOTS - 1))
			if (e->tab[i].used == 1 && !pinned(p, &e->tab[i].a)) {
				addr_out[k] = e->tab[i].a; ts_out[k] = e->tab[i].ts; ok_out[k] = 1;
				break;
			}
	}
	pthread_mutex_unlock(&e->mu);
	pthread_mutex_unlock(&pin_mu);
	return 0;
}

int cmb200_pin_count(cmb200_engine *e, uint64_t *in_arena, uint64_t *in_tier) {
	uint64_t c = 0;
	pthread_mutex_lock(&pin_mu);
	pthread_mutex_lock(&e->mu);
	const struct pins *p = pins_of(e);
	for (uint32_t i = 0; i < SLOTS; i++)
		if (e->tab[i].used == 1 && pinned(p, &e->tab[i].a)) c++;
	pthread_mutex_unlock(&e->mu);
	pthread_mutex_unlock(&pin_mu);
	*in_arena = c;
	*in_tier = 0;
	return 0;
}

int cmb200_pin_promote(cmb200_engine *e, uint64_t *promoted_out) {
	(void)e;
	if (promoted_out) *promoted_out = 0;
	return 0;
}

int cmb200_set_file_key(cmb200_engine *e, const uint8_t *key) { (void)e; (void)key; return 0; }

int cmb200_aead_seal_batch(int device, const uint8_t *key, size_t n, const uint8_t *nonces,
    const uint8_t *const *aad, const size_t *aad_len, const uint8_t *const *msg, const size_t *msg_len,
    uint8_t *const *out) {
	(void)device; (void)msg;
	for (size_t i = 0; i < n; i++) {
		if (msg_len[i]) return -1;
		uint64_t h[2] = { 0xcbf29ce484222325ull, 0x84222325cbf29ce4ull };
		for (int w = 0; w < 2; w++) {
			for (int k = 0; k < 32; k++) h[w] = (h[w] ^ key[k]) * 0x100000001b3ull;
			for (int k = 0; k < 12; k++) h[w] = (h[w] ^ nonces[12 * i + k]) * 0x100000001b3ull;
			for (size_t k = 0; k < aad_len[i]; k++) h[w] = (h[w] ^ aad[i][k]) * 0x100000001b3ull;
		}
		memcpy(out[i], h, 16);
	}
	return 0;
}

int cmb200_freq_estimate(cmb200_engine *e, size_t n, const cmb200_addr *addr, uint8_t *est_out) {
	(void)e;
	for (size_t i = 0; i < n; i++) est_out[i] = (addr[i].l & ((1ull << 44) - 1)) >= MOCK_HOT_FROM ? 15 : 0;
	return 0;
}
