/* A CPU stand-in for the GPU engine (include/cachemap_b200.h), TEST INFRASTRUCTURE ONLY: it lets the
 * host layer of the drop-in (edge_fuse_b200/csrc/cachemap_api.c: write-behind ring + flusher, the
 * combining queue of single-page gets with per-request completion, eviction bookkeeping) run and be
 * stressed from many threads on a machine without a GPU, under ThreadSanitizer if wanted
 * (tests/test_host_logic.py).  It keeps pages uncompressed in a hash map and imitates what the
 * engine promises the host layer, including the asynchronous part: cmb200_get_small_begin returns at
 * once and worker threads answer the requests one by one, in shuffled order, after short random
 * delays — page first, then the status word (release) — exactly the order the kernel keeps.
 * Like the engine it keeps one record per store key (FNV-1a-64 of the 16 address bytes, filemap.c:18-24):
 * a put replaces the key's record whatever address it held, a get of a key that holds another address
 * answers CMB200_BAD_ENTRY, and an unset deletes the key's record.  mock_hold_puts(1) makes every put
 * wait until mock_hold_puts(0), so that a test can keep pages in the drop-in's write-behind ring.
 * A put of a page that begins with the 8 bytes MOCK_DROP finds no room, as a put into a full arena:
 * lens_out is -1 and the key keeps the record it had.
 * Nothing of the product links against this file. */
#include <pthread.h>
#include <sched.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <unistd.h>

#include "../../include/cachemap_b200.h"
#include "../../include/uint128.h"

#define SLOTS (1u << 17)
#define LANES 32
#define LANE_MAX 1024
#define WORKERS 6
#define MOCK_DROP "MOCKDROP"

struct entry { int used; uint64_t key; cmb200_addr a; uint64_t ts; uint8_t *page; };

struct job { int lane; uint32_t n; uint8_t *out; };

struct cmb200_engine {
	uint32_t bsize;
	pthread_mutex_t mu;             /* the map */
	struct entry *tab;
	uint64_t entries, puts, gets, hits, launches;
	/* small gets */
	int lane_busy[LANES];
	int32_t *lane_status[LANES];
	cmb200_addr *lane_addr[LANES];
	pthread_mutex_t jq_mu;
	pthread_cond_t jq_cv;
	struct job jq[LANES];
	int jq_n, stop;
	pthread_t worker[WORKERS];
};

static __thread char err_buf[128];
const char *cmb200_last_error(void) { return err_buf[0] ? err_buf : "mock engine"; }
int cmb200_device_count(void) { return 1; }
void *cmb200_host_alloc(size_t bytes) { return malloc(bytes ? bytes : 1); }
void cmb200_host_free(void *p) { free(p); }

static uint64_t addr_key(const cmb200_addr *a) {
	uint64_t key;
	FNV_hash(a, (int)sizeof(*a), &key);
	return key;
}
/* slot of the key of `a` (whatever address its record holds), or the free slot where it would go (mu held) */
static struct entry *find(cmb200_engine *e, const cmb200_addr *a, int *present) {
	const uint64_t key = addr_key(a);
	uint64_t i = (key ^ (key >> 29)) & (SLOTS - 1);
	struct entry *hole = NULL;
	for (uint32_t n = 0; n < SLOTS; n++, i = (i + 1) & (SLOTS - 1)) {
		struct entry *s = &e->tab[i];
		if (s->used == 1 && s->key == key) { *present = 1; return s; }
		if (s->used == 2 && !hole) hole = s;                 /* deleted */
		if (s->used == 0) { *present = 0; return hole ? hole : s; }
	}
	*present = 0;
	return hole;
}
/* HIT, BAD_ENTRY (the key holds another address) or MISS for `a`, and its entry on a hit (mu held) */
static int32_t lookup(cmb200_engine *e, const cmb200_addr *a, struct entry **hit) {
	int present;
	struct entry *s = find(e, a, &present);
	*hit = NULL;
	if (!present) return CMB200_MISS;
	if (s->a.u != a->u || s->a.l != a->l) return CMB200_BAD_ENTRY;
	*hit = s;
	return CMB200_HIT;
}

static pthread_mutex_t hold_mu = PTHREAD_MUTEX_INITIALIZER;
static pthread_cond_t hold_cv = PTHREAD_COND_INITIALIZER;
static int hold_puts;
void mock_hold_puts(int on) {
	pthread_mutex_lock(&hold_mu);
	hold_puts = on;
	pthread_cond_broadcast(&hold_cv);
	pthread_mutex_unlock(&hold_mu);
}

static void *worker(void *arg) {
	cmb200_engine *e = arg;
	unsigned seed = (unsigned)(uintptr_t)pthread_self();
	for (;;) {
		pthread_mutex_lock(&e->jq_mu);
		while (!e->jq_n && !e->stop) pthread_cond_wait(&e->jq_cv, &e->jq_mu);
		if (!e->jq_n && e->stop) { pthread_mutex_unlock(&e->jq_mu); return NULL; }
		struct job j = e->jq[--e->jq_n];
		pthread_mutex_unlock(&e->jq_mu);
		/* answer in a shuffled order with small pauses, like CTAs finishing at different times */
		uint32_t order[LANE_MAX];
		for (uint32_t i = 0; i < j.n; i++) order[i] = i;
		for (uint32_t i = j.n; i > 1; i--) { uint32_t k = rand_r(&seed) % i, t = order[i - 1]; order[i - 1] = order[k]; order[k] = t; }
		for (uint32_t q = 0; q < j.n; q++) {
			const uint32_t i = order[q];
			if ((rand_r(&seed) & 3) == 0) usleep(rand_r(&seed) % 40);
			pthread_mutex_lock(&e->mu);
			struct entry *s;
			const int32_t st = lookup(e, &e->lane_addr[j.lane][i], &s);
			if (s) memcpy(j.out + (size_t)i * e->bsize, s->page, e->bsize);
			pthread_mutex_unlock(&e->mu);
			__atomic_store_n(&e->lane_status[j.lane][i], st, __ATOMIC_RELEASE);    /* the page first, then its status */
		}
	}
}

cmb200_engine *cmb200_engine_create(const cmb200_config *cfg) {
	cmb200_engine *e = calloc(1, sizeof(*e));
	e->bsize = 1u << cfg->pshift;
	e->tab = calloc(SLOTS, sizeof(struct entry));
	pthread_mutex_init(&e->mu, NULL);
	pthread_mutex_init(&e->jq_mu, NULL);
	pthread_cond_init(&e->jq_cv, NULL);
	for (int i = 0; i < LANES; i++) {
		e->lane_status[i] = malloc(LANE_MAX * sizeof(int32_t));
		e->lane_addr[i] = malloc(LANE_MAX * sizeof(cmb200_addr));
	}
	for (int i = 0; i < WORKERS; i++) pthread_create(&e->worker[i], NULL, worker, e);
	return e;
}

void cmb200_engine_destroy(cmb200_engine *e) {
	if (!e) return;
	pthread_mutex_lock(&e->jq_mu);
	e->stop = 1;
	pthread_cond_broadcast(&e->jq_cv);
	pthread_mutex_unlock(&e->jq_mu);
	for (int i = 0; i < WORKERS; i++) pthread_join(e->worker[i], NULL);
	for (uint32_t i = 0; i < SLOTS; i++) free(e->tab[i].page);
	for (int i = 0; i < LANES; i++) { free(e->lane_status[i]); free(e->lane_addr[i]); }
	free(e->tab);
	free(e);
}

int cmb200_put_batch(cmb200_engine *e, size_t n, const cmb200_addr *addr, const uint8_t *valid, const void *pages,
    const uint64_t *ts, int32_t *lens_out) {
	pthread_mutex_lock(&hold_mu);
	while (hold_puts) pthread_cond_wait(&hold_cv, &hold_mu);
	pthread_mutex_unlock(&hold_mu);
	usleep(30 + n / 8);                                           /* a launch and a copy take a while */
	pthread_mutex_lock(&e->mu);
	for (size_t i = 0; i < n; i++) {
		if (valid && !valid[i]) { if (lens_out) lens_out[i] = -1; continue; }
		if (memcmp((const uint8_t *)pages + i * e->bsize, MOCK_DROP, 8) == 0) { if (lens_out) lens_out[i] = -1; continue; }
		int present;
		struct entry *s = find(e, &addr[i], &present);
		if (!s) continue;                                         /* map full: dropped */
		if (!present) { s->used = 1; s->key = addr_key(&addr[i]); if (!s->page) s->page = malloc(e->bsize); e->entries++; }
		s->a = addr[i];                                           /* the key's record, whatever address it held */
		memcpy(s->page, (const uint8_t *)pages + i * e->bsize, e->bsize);
		s->ts = ts ? ts[i] : 0;
		if (lens_out) lens_out[i] = (int32_t)e->bsize;
		e->puts++;
	}
	pthread_mutex_unlock(&e->mu);
	return 0;
}
int cmb200_put_batch_async(cmb200_engine *e, size_t n, const cmb200_addr *addr, const uint8_t *valid, const void *pages,
    const uint64_t *ts, int32_t *lens_out, uint64_t *ticket) {
	if (ticket) *ticket = 0;
	return cmb200_put_batch(e, n, addr, valid, pages, ts, lens_out);
}
int cmb200_wait(cmb200_engine *e, uint64_t ticket) { (void)e; (void)ticket; return 0; }
int cmb200_put_batch_dev(cmb200_engine *e, size_t n, const cmb200_addr *a, const uint8_t *v, const void *p, const uint64_t *t, int32_t *l) {
	(void)e; (void)n; (void)a; (void)v; (void)p; (void)t; (void)l; snprintf(err_buf, sizeof(err_buf), "mock: no device memory"); return -1;
}
int cmb200_get_batch_dev(cmb200_engine *e, size_t n, const cmb200_addr *a, const uint8_t *v, void *p, int32_t *s) {
	(void)e; (void)n; (void)a; (void)v; (void)p; (void)s; snprintf(err_buf, sizeof(err_buf), "mock: no device memory"); return -1;
}

int cmb200_get_batch(cmb200_engine *e, size_t n, const cmb200_addr *addr, const uint8_t *valid, void *pages_out, int32_t *status_out) {
	usleep(30);
	pthread_mutex_lock(&e->mu);
	for (size_t i = 0; i < n; i++) {
		if (valid && !valid[i]) { status_out[i] = CMB200_INVALID; continue; }
		struct entry *s;
		status_out[i] = lookup(e, &addr[i], &s);
		if (s) memcpy((uint8_t *)pages_out + i * e->bsize, s->page, e->bsize);
		e->gets++; e->hits += s != NULL;
	}
	pthread_mutex_unlock(&e->mu);
	return 0;
}

int cmb200_get_small_begin(cmb200_engine *e, size_t n, const cmb200_addr *addr, void *pages_out, cmb200_small_ticket *t) {
	t->lane = -1; t->n = 0; t->status = NULL;
	if (n == 0) return 0;
	if (n > LANE_MAX) return -1;
	if (e->bsize > 65536) return -2;                              /* like the fused kernel: pages above 64 KiB are not served */
	int li = -1;
	while (li < 0) {
		for (int c = 0; c < LANES && li < 0; c++) {
			int idle = 0;
			if (__atomic_compare_exchange_n(&e->lane_busy[c], &idle, 1, 0, __ATOMIC_ACQ_REL, __ATOMIC_RELAXED)) li = c;
		}
		if (li < 0) sched_yield();
	}
	memcpy(e->lane_addr[li], addr, n * sizeof(cmb200_addr));
	for (size_t i = 0; i < n; i++) __atomic_store_n(&e->lane_status[li][i], CMB200_SMALL_PENDING, __ATOMIC_RELAXED);
	usleep(5);                                                    /* the launch */
	pthread_mutex_lock(&e->jq_mu);
	e->jq[e->jq_n++] = (struct job){ li, (uint32_t)n, pages_out };
	pthread_cond_signal(&e->jq_cv);
	pthread_mutex_unlock(&e->jq_mu);
	t->lane = li; t->n = (uint32_t)n; t->status = e->lane_status[li];
	return 0;
}

int cmb200_get_small_end(cmb200_engine *e, cmb200_small_ticket *t, int32_t *status_out) {
	if (!t || t->lane < 0) return 0;
	uint64_t hits = 0;
	for (uint32_t i = 0; i < t->n; i++) {
		int32_t st;
		while ((st = __atomic_load_n(&e->lane_status[t->lane][i], __ATOMIC_ACQUIRE)) == CMB200_SMALL_PENDING) sched_yield();
		if (status_out) status_out[i] = st;
		hits += st == CMB200_HIT;
	}
	__atomic_fetch_add(&e->gets, t->n, __ATOMIC_RELAXED);
	__atomic_fetch_add(&e->hits, hits, __ATOMIC_RELAXED);
	__atomic_fetch_add(&e->launches, 1, __ATOMIC_RELAXED);
	const int li = t->lane;
	t->lane = -1;
	__atomic_store_n(&e->lane_busy[li], 0, __ATOMIC_RELEASE);
	return 0;
}

int cmb200_unset_batch(cmb200_engine *e, size_t n, const cmb200_addr *addr) {
	pthread_mutex_lock(&e->mu);
	for (size_t i = 0; i < n; i++) {
		int present;
		struct entry *s = find(e, &addr[i], &present);
		if (present) { s->used = 2; e->entries--; }
	}
	pthread_mutex_unlock(&e->mu);
	return 0;
}
uint64_t cmb200_entries(cmb200_engine *e) {
	pthread_mutex_lock(&e->mu);
	const uint64_t n = e->entries;
	pthread_mutex_unlock(&e->mu);
	return n;
}
int cmb200_sample(cmb200_engine *e, size_t n, const uint64_t *r, cmb200_addr *addr_out, uint64_t *ts_out, int32_t *ok_out) {
	pthread_mutex_lock(&e->mu);
	for (size_t k = 0; k < n; k++) {
		ok_out[k] = 0;
		uint64_t i = r[k] & (SLOTS - 1);
		for (uint32_t step = 0; step < SLOTS; step++, i = (i + 1) & (SLOTS - 1))
			if (e->tab[i].used == 1) { addr_out[k] = e->tab[i].a; ts_out[k] = e->tab[i].ts; ok_out[k] = 1; break; }
	}
	pthread_mutex_unlock(&e->mu);
	return 0;
}
int cmb200_get_stats(cmb200_engine *e, cmb200_stats *out) {
	memset(out, 0, sizeof(*out));
	pthread_mutex_lock(&e->mu);
	out->entries = e->entries; out->table_slots = SLOTS;
	out->arena_bytes = 1ull << 40; out->arena_used = e->entries * (uint64_t)e->bsize;
	out->put_chunks = e->puts;
	pthread_mutex_unlock(&e->mu);
	out->get_requests = __atomic_load_n(&e->gets, __ATOMIC_RELAXED);
	out->get_hits = __atomic_load_n(&e->hits, __ATOMIC_RELAXED);
	out->kernel_launches = __atomic_load_n(&e->launches, __ATOMIC_RELAXED);
	return 0;
}
int cmb200_compact(cmb200_engine *e, uint64_t *reclaimed_out) { (void)e; if (reclaimed_out) *reclaimed_out = 0; return 0; }
int cmb200_save(cmb200_engine *e, const char *path, uint64_t *records_out) { (void)e; (void)path; if (records_out) *records_out = 0; return -1; }
int cmb200_load(cmb200_engine *e, const char *path, uint64_t *records_out) { (void)e; (void)path; if (records_out) *records_out = 0; return -1; }
