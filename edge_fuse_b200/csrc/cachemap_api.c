/*
 * cachemap_api.c — the reference's C API (include/cachemap.h, include/filemap.h) over the H100
 * engine.  Host code stays C; everything heavy happens in the engine's kernels.
 *
 * What each reference function became:
 *   filemap_create/free        cachemap/filemap.c:35-110   -> config only; engine built lazily
 *   filemap_set                cachemap/filemap.c:112-158  -> WRITE-BEHIND: the page is copied into a
 *                              page-locked ring and the call returns; one flusher thread hands the
 *                              ring to the GPU in batches.  A single chunk takes the GPU 0.2-3 ms
 *                              to encode (the LZ4 parse is serial), which no caller should wait
 *                              for; what the reference guarantees to its callers — a get after a
 *                              put returns that page — is kept by looking in the ring first.
 *   filemap_get                cachemap/filemap.c:217-262  -> ring hit, else one request in a
 *                              combining queue: whichever caller finds no batch in flight becomes
 *                              the leader and runs every queued request as one GPU batch
 *   filemap_unset/get_rand/entries  filemap.c:188-330     -> drain the ring, then engine calls
 *   cachemap_*                 cachemap/cachemap.c:107-239 -> same logic: address composition,
 *                              timestamps, counters; evict-oldest-of-3 runs in the flusher before
 *                              each batch; put_async == put (both are write-behind now)
 * There is no CPU fallback: if the engine cannot be created the process stops with a message
 * (set CMB200_SOFT_FAIL=1 to degrade to "every put dropped, every get a miss" instead).
 */
#define _GNU_SOURCE
#include <pthread.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <sys/stat.h>
#include <time.h>
#include <sched.h>
#include <semaphore.h>
#include <unistd.h>

#include "../../include/cachemap.h"
#include "../../include/cachemap_b200.h"

/* The host tier is optional in the engine this layer links against: libcachemap's engine defines
 * these, an engine without a tier (such as the CPU stand-in the host-layer tests link) does not, and
 * then they are null and CMB200_HOST_TIER_MB is refused. */
#pragma weak cmb200_host_tier_enable
#pragma weak cmb200_demote_batch
#pragma weak cmb200_host_tier_stats
#pragma weak cmb200_promote_batch
#pragma weak cmb200_host_tier_hot

#define COMBINE_MAX 32          /* get/unset requests one leader takes per GPU batch */
#define LEADERS 32              /* batches of gets that may be in flight at once, each on its own engine lane
                                 * (<= the engine's GET_LANES); see the combining queue below */
#define GET_CALLERS 32          /* callers inside the combining queue at once; the rest sleep at its door */
#define FLUSH_MAX 4096          /* pages the flusher hands over per GPU batch */
#define PNUM_SHIFT 44           /* cachemap.c:155 */
#define PROMOTE_EVERY_MS 100    /* CMB200_TIER_PROMOTE: at most one promotion round this often */

enum req_kind { REQ_GET, REQ_UNSET };
enum wb_state { WB_FREE = 0, WB_FILLING, WB_READY, WB_FLUSHING };

struct fm_req {
	enum req_kind kind;
	cmb200_addr addr;
	void *out;              /* REQ_GET: malloc()ed page (or dst) on a hit, else NULL */
	void *dst;              /* REQ_GET: caller's buffer to fill instead of malloc()ing one */
	const volatile int32_t *status; /* where this request's answer appears (set, under q_mu, when its batch is launched) */
	int slot, pos;          /* leader slot of its batch and position in that batch's stage buffer */
	int bad_entry;
	struct fm_req *next;
};

struct wb_slot {
	cmb200_addr addr;
	uint64_t ts;
	int state;
};

struct filemap {
	uint64_t n;
	int compress;
	int bsize;
	int pshift;
	char destdir[2048];
	uint64_t capacity;      /* eviction threshold (set by cachemap_create), 0 = none */
	/* engine, built on first use (fork safety, SURVEY.md §3.1) */
	pthread_mutex_t init_mu;
	int init_state;         /* 0 = not yet, 1 = ready, -1 = failed */
	cmb200_engine *eng;
	int host_tier;          /* the engine has a host tier (CMB200_HOST_TIER_MB): a full arena demotes instead of evicting */
	/* promotion of hot tier records back to the arena (CMB200_TIER_PROMOTE), run by the flusher */
	uint64_t tier_promote;  /* pages per round, 0 = off */
	cmb200_addr *promo_hot; /* tier_promote entries: the round's drained hot addresses */
	pthread_mutex_t promo_mu;       /* the guard below (demotion runs in callers of cachemap_put_batch too) */
	cmb200_addr *promo_guard;       /* FIFO of the last 4 x tier_promote promoted addresses: not demoted again */
	uint64_t promo_guard_n;         /* addresses ever added; slot = index % (4 x tier_promote) */
	struct timespec promo_last;     /* CLOCK_MONOTONIC of the last round */
	uint8_t *h_stage;       /* page-locked, LEADERS x COMBINE_MAX pages: the stage buffer of each leader slot */
	int leader_busy[LEADERS];       /* a batch is in flight in this slot (under q_mu) */
	int batch_left[LEADERS];        /* its requesters that have not taken their answer yet (atomic) */
	cmb200_small_ticket ticket[LEADERS];    /* the slot's launch (lane < 0: the batch was answered synchronously) */
	int32_t sync_status[LEADERS][COMBINE_MAX];      /* answers of a synchronously run batch */
	int launching;                  /* a caller is inside a launch: arrivals meanwhile form the next batch (set under q_mu) */
	sem_t q_door;                   /* GET_CALLERS permits: the queue is built on watching, not sleeping, and that only
	                                 * works while the watchers have cores of their own */
	int busy_slots;                 /* slots with a batch in flight (atomic; changes under q_mu) */
	int q_len;                      /* requests queued and not yet launched (atomic; changes under q_mu) */
	/* combining queue (gets, unsets) */
	pthread_mutex_t q_mu;
	struct fm_req *q_head, *q_tail;
	/* write-behind ring: slots [wb_tail, wb_head) are in use, numbered modulo wb_n */
	pthread_mutex_t wb_mu;
	pthread_cond_t wb_space, wb_work, wb_idle;
	uint8_t *wb_pages;      /* page-locked, wb_n pages */
	struct wb_slot *wb_slot;
	uint64_t wb_n, wb_head, wb_tail;
	pthread_t wb_thread;
	int wb_started, wb_stop;
	int wb_flusher_asleep;  /* the flusher waits on wb_work (under wb_mu) */
	/* persistence: <destdir>/cachemap_b200.snap (cmb200_save / cmb200_load) */
	int persist;
	long checkpoint_sec;    /* > 0: the flusher saves a snapshot this often when puts have arrived */
	uint64_t puts_seen, puts_saved;
	pthread_mutex_t snap_mu;
};

#define SNAPSHOT_NAME "cachemap_b200.snap"

static int
filemap_snapshot_path(struct filemap *m, char *out, size_t cap)
{
	return snprintf(out, cap, "%s/%s", m->destdir, SNAPSHOT_NAME) < (int)cap;
}

static long
env_long(const char *name, long dflt)
{
	const char *v = getenv(name);
	return (v && *v) ? strtol(v, NULL, 0) : dflt;
}

static void *filemap_flusher(void *arg);

static int
filemap_engine_ready(struct filemap *m)
{
	if (__atomic_load_n(&m->init_state, __ATOMIC_ACQUIRE) == 1)
		return 1;
	pthread_mutex_lock(&m->init_mu);
	if (m->init_state == 0) {
		cmb200_config cfg;
		memset(&cfg, 0, sizeof(cfg));
		cfg.device = (int)env_long("CMB200_DEVICE", -1);
		cfg.pshift = m->pshift;
		cfg.accel = m->compress;
		cfg.capacity = m->n;
		cfg.arena_bytes = (uint64_t)env_long("CMB200_ARENA_MB", 0) << 20;
		cfg.table_slots = (uint64_t)env_long("CMB200_TABLE_SLOTS", 0);
		cfg.max_batch = (uint32_t)env_long("CMB200_MAX_BATCH", 0);
		cfg.flags = env_long("CMB200_FINGERPRINT", 0) ? CMB200_FINGERPRINT : 0;
		m->eng = cmb200_engine_create(&cfg);
		const long tier_mb = env_long("CMB200_HOST_TIER_MB", 0);
		if (m->eng && tier_mb > 0) {
			if (!cmb200_host_tier_enable)
				fprintf(stderr, "cachemap_b200: no host tier of %ld MiB: the engine has none\n", tier_mb);
			else if (cmb200_host_tier_enable(m->eng, (uint64_t)tier_mb << 20) == 0)
				m->host_tier = 1;
			else
				fprintf(stderr, "cachemap_b200: no host tier of %ld MiB: %s\n", tier_mb, cmb200_last_error());
		}
		const long promote = env_long("CMB200_TIER_PROMOTE", 0);
		if (m->host_tier && promote > 0) {
			if (!cmb200_promote_batch || !cmb200_host_tier_hot)
				fprintf(stderr, "cachemap_b200: CMB200_TIER_PROMOTE ignored: the engine cannot promote\n");
			else {
				m->promo_hot = malloc((size_t)promote * sizeof(cmb200_addr));
				m->promo_guard = malloc(4 * (size_t)promote * sizeof(cmb200_addr));
				if (m->promo_hot && m->promo_guard)
					m->tier_promote = (uint64_t)promote;
			}
		}
		if (m->eng) {
			m->h_stage = cmb200_host_alloc((size_t)LEADERS * COMBINE_MAX * m->bsize);
			/* ring of 256 MiB by default, at least 64 pages.  The size sets the batch the flusher can form
			 * (half the ring), and a batch below ~2 000 chunks leaves the encode kernel a partial wave
			 * whose duration is one chunk's latency (~2 ms for a text-like page) whatever its size */
			long slots = env_long("CMB200_WB_SLOTS", (256L << 20) / m->bsize);
			if (slots > 0 && slots < 64)
				slots = 64;
			if (slots > 0) {
				m->wb_pages = cmb200_host_alloc((size_t)slots * m->bsize);
				m->wb_slot = calloc((size_t)slots, sizeof(struct wb_slot));
				m->wb_n = (m->wb_pages && m->wb_slot) ? (uint64_t)slots : 0;
			}
		}
		if (!m->eng || !m->h_stage) {
			fprintf(stderr, "cachemap_b200: cannot start the GPU engine: %s\n", cmb200_last_error());
			if (!env_long("CMB200_SOFT_FAIL", 0)) {
				fprintf(stderr, "cachemap_b200: no CPU fallback exists; aborting "
				    "(CMB200_SOFT_FAIL=1 turns this into dropped puts / misses)\n");
				abort();
			}
			__atomic_store_n(&m->init_state, -1, __ATOMIC_RELEASE);
		} else {
			/* what the cache directory holds from an earlier run comes back first: the reference's
			 * store is persistent (LMDB files under destdir, filemap.c:57,71-72) */
			m->persist = (int)env_long("CMB200_PERSIST", 1);
			m->checkpoint_sec = env_long("CMB200_CHECKPOINT_SEC", 0);
			char snap[2200];
			if (m->persist && filemap_snapshot_path(m, snap, sizeof(snap)) && access(snap, R_OK) == 0) {
				uint64_t got = 0;
				if (cmb200_load(m->eng, snap, &got) != 0)
					fprintf(stderr, "cachemap_b200: %s ignored: %s\n", snap, cmb200_last_error());
			}
			/* the flusher starts here, i.e. in the process that actually caches (after any fork) */
			if (m->wb_n && pthread_create(&m->wb_thread, NULL, filemap_flusher, m) == 0)
				m->wb_started = 1;
			else
				m->wb_n = 0;
			__atomic_store_n(&m->init_state, 1, __ATOMIC_RELEASE);
		}
	}
	pthread_mutex_unlock(&m->init_mu);
	return m->init_state == 1;
}

struct filemap *
filemap_create(char *destdir, uint64_t n, int compress_accel, int pshift)
{
	if (!destdir || strlen(destdir) >= sizeof(((struct filemap *)0)->destdir))
		return NULL;
	if (n < FILEMAP_SHARD_FACTOR)           /* filemap.c:51 */
		return NULL;
	if (pshift < 6 || pshift > 20)
		return NULL;
	struct filemap *m = calloc(1, sizeof(*m));
	if (!m)
		return NULL;
	m->n = n;
	m->compress = compress_accel;
	m->bsize = 1 << pshift;
	m->pshift = pshift;
	strcpy(m->destdir, destdir);
	pthread_mutex_init(&m->init_mu, NULL);
	pthread_mutex_init(&m->q_mu, NULL);
	sem_init(&m->q_door, 0, GET_CALLERS);
	pthread_mutex_init(&m->wb_mu, NULL);
	pthread_cond_init(&m->wb_space, NULL);
	pthread_cond_init(&m->wb_work, NULL);
	pthread_cond_init(&m->wb_idle, NULL);
	pthread_mutex_init(&m->snap_mu, NULL);
	pthread_mutex_init(&m->promo_mu, NULL);
	return m;
}

/* Saves the store to <destdir>/cachemap_b200.snap.  0 = saved, -1 = not (disabled, engine never
 * started, or I/O error). */
static int
filemap_save(struct filemap *m)
{
	char snap[2200];
	if (__atomic_load_n(&m->init_state, __ATOMIC_ACQUIRE) != 1 || !m->persist ||
	    !filemap_snapshot_path(m, snap, sizeof(snap)))
		return -1;
	pthread_mutex_lock(&m->snap_mu);
	uint64_t seen = __atomic_load_n(&m->puts_seen, __ATOMIC_RELAXED);
	int rc = cmb200_save(m->eng, snap, NULL);
	if (rc == 0)
		m->puts_saved = seen;
	else
		fprintf(stderr, "cachemap_b200: snapshot not written: %s\n", cmb200_last_error());
	pthread_mutex_unlock(&m->snap_mu);
	return rc;
}

/* Waits until every page accepted so far is in the GPU store. */
static void
filemap_drain(struct filemap *m)
{
	if (!m->wb_n)
		return;
	pthread_mutex_lock(&m->wb_mu);
	/* everything accepted before this call, not "until the ring is empty": with other threads
	 * still putting the ring may never be empty (the flusher broadcasts after every batch) */
	const uint64_t target = m->wb_head;
	while (m->wb_tail < target)
		pthread_cond_wait(&m->wb_idle, &m->wb_mu);
	pthread_mutex_unlock(&m->wb_mu);
}

void
filemap_free(struct filemap *m)
{
	if (!m)
		return;
	if (m->wb_started) {
		pthread_mutex_lock(&m->wb_mu);
		m->wb_stop = 1;
		pthread_cond_broadcast(&m->wb_work);
		pthread_mutex_unlock(&m->wb_mu);
		pthread_join(m->wb_thread, NULL);      /* drains the ring first */
	}
	filemap_save(m);                                /* the cache directory outlives the process */
	if (m->wb_pages)
		cmb200_host_free(m->wb_pages);
	free(m->wb_slot);
	if (m->h_stage)
		cmb200_host_free(m->h_stage);
	if (m->eng)
		cmb200_engine_destroy(m->eng);
	free(m->promo_hot);
	free(m->promo_guard);
	pthread_mutex_destroy(&m->promo_mu);
	pthread_mutex_destroy(&m->snap_mu);
	pthread_mutex_destroy(&m->init_mu);
	pthread_mutex_destroy(&m->q_mu);
	sem_destroy(&m->q_door);
	pthread_mutex_destroy(&m->wb_mu);
	pthread_cond_destroy(&m->wb_space);
	pthread_cond_destroy(&m->wb_work);
	pthread_cond_destroy(&m->wb_idle);
	free(m);
}

/* Retires up to `want` records, each the oldest of three random live ones (cachemap.c:17-45).
 * Statistically the reference's policy; bitwise parity is undefined there (wall-clock
 * timestamps, rand()).  Returns how many entries actually went away. */
static uint64_t
filemap_evict_n(struct filemap *m, uint64_t want)
{
	uint64_t before = cmb200_entries(m->eng), gone = 0;
	while (gone < want && before > 0) {
		uint64_t need = want - gone;
		if (need > before)
			need = before;
		if (need > 4096)
			need = 4096;    /* per round; the loop continues */
		uint64_t *draws = malloc(3 * need * sizeof(uint64_t));
		uint64_t *ts = malloc(3 * need * sizeof(uint64_t));
		int32_t *ok = malloc(3 * need * sizeof(int32_t));
		cmb200_addr *cand = malloc(3 * need * sizeof(cmb200_addr));
		cmb200_addr *victim = malloc(need * sizeof(cmb200_addr));
		uint64_t nv = 0;
		if (draws && ts && ok && cand && victim) {
			for (uint64_t i = 0; i < 3 * need; i++) {
				uint64_t r = 0;
				for (int b = 0; b < 64; b += 30)        /* filemap.c:271-274 */
					r = r * ((uint64_t)RAND_MAX + 1) + (uint64_t)rand();
				draws[i] = r;
			}
			if (cmb200_sample(m->eng, (size_t)(3 * need), draws, cand, ts, ok) == 0) {
				for (uint64_t i = 0; i < need; i++) {
					uint64_t a = ts[3 * i], b = ts[3 * i + 1], c = ts[3 * i + 2];
					int pick;
					if (a < b)
						pick = (a > c) ? 2 : 0;         /* cachemap.c:29-41 */
					else
						pick = (b > c) ? 2 : 1;
					if (ok[3 * i + pick] > 0)
						victim[nv++] = cand[3 * i + pick];
				}
				if (nv)
					cmb200_unset_batch(m->eng, (size_t)nv, victim);
			} else {
				fprintf(stderr, "cachemap_b200: eviction could not sample the store: %s\n", cmb200_last_error());
			}
		}
		free(draws); free(ts); free(ok); free(cand); free(victim);
		/* two draws may have picked the same victim: count what really left the table */
		uint64_t after = cmb200_entries(m->eng);
		if (nv == 0 || after >= before)
			break;          /* no progress */
		gone += before - after;
		before = after;
	}
	return gone;
}

struct aged { uint64_t ts; cmb200_addr a; };

static int
aged_cmp(const void *x, const void *y)
{
	const uint64_t a = ((const struct aged *)x)->ts, b = ((const struct aged *)y)->ts;
	return a < b ? -1 : a > b;
}

static int
addr_cmp(const void *x, const void *y)
{
	const cmb200_addr *a = x, *b = y;
	if (a->u != b->u)
		return a->u < b->u ? -1 : 1;
	return a->l < b->l ? -1 : a->l > b->l;
}

/* Sorted copy of the addresses the last promotion rounds offered (CMB200_TIER_PROMOTE), or NULL.  A
 * promoted record keeps its old put timestamp, so without this the next demotion, which takes the
 * oldest of what it samples, would send it straight back to the tier. */
static cmb200_addr *
filemap_promo_guard(struct filemap *m, size_t *n)
{
	*n = 0;
	if (!m->tier_promote)
		return NULL;
	pthread_mutex_lock(&m->promo_mu);
	const uint64_t cap = 4 * m->tier_promote;
	const size_t k = (size_t)(m->promo_guard_n < cap ? m->promo_guard_n : cap);
	cmb200_addr *g = k ? malloc(k * sizeof(cmb200_addr)) : NULL;
	if (g) {
		memcpy(g, m->promo_guard, k * sizeof(cmb200_addr));
		*n = k;
	}
	pthread_mutex_unlock(&m->promo_mu);
	if (g)
		qsort(g, *n, sizeof(cmb200_addr), addr_cmp);
	return g;
}

/* Moves up to `want` arena records to the host tier.  The candidates are drawn as filemap_evict_n
 * draws them (3 per record wanted) and go oldest first; keys already in the tier, and keys promotion
 * has just brought back (filemap_promo_guard), are passed over, so a round goes on down its candidates
 * until `want` have moved.  When few records are left in the arena a round may find none: it draws
 * again, up to 16 times in a row.  Returns how many moved. */
static uint64_t
filemap_demote_n(struct filemap *m, uint64_t want)
{
	uint64_t moved = 0;
	int idle = 0;
	size_t ng = 0;
	cmb200_addr *guard = filemap_promo_guard(m, &ng);
	while (moved < want && idle < 16) {
		uint64_t need = want - moved;
		if (need > 4096)
			need = 4096;
		const uint64_t nd = 3 * need;
		uint64_t *draws = malloc(nd * sizeof(uint64_t));
		uint64_t *ts = malloc(nd * sizeof(uint64_t));
		int32_t *ok = malloc(nd * sizeof(int32_t));
		cmb200_addr *cand = malloc(nd * sizeof(cmb200_addr));
		struct aged *old = malloc(nd * sizeof(struct aged));
		cmb200_addr *victim = malloc(nd * sizeof(cmb200_addr));
		uint64_t round = 0;
		if (draws && ts && ok && cand && old && victim) {
			for (uint64_t i = 0; i < nd; i++) {
				uint64_t r = 0;
				for (int b = 0; b < 64; b += 30)        /* filemap.c:271-274 */
					r = r * ((uint64_t)RAND_MAX + 1) + (uint64_t)rand();
				draws[i] = r;
			}
			if (cmb200_sample(m->eng, (size_t)nd, draws, cand, ts, ok) == 0) {
				uint64_t nv = 0;
				for (uint64_t i = 0; i < nd; i++)
					if (ok[i] > 0 && !(guard && bsearch(&cand[i], guard, ng, sizeof(cmb200_addr), addr_cmp)))
						old[nv++] = (struct aged){ ts[i], cand[i] };
				qsort(old, (size_t)nv, sizeof(struct aged), aged_cmp);
				for (uint64_t k = 0; k < nv && moved < want;) {
					uint64_t take = want - moved < nv - k ? want - moved : nv - k, got = 0;
					for (uint64_t j = 0; j < take; j++)
						victim[j] = old[k + j].a;
					if (cmb200_demote_batch(m->eng, (size_t)take, victim, &got) != 0) {
						fprintf(stderr, "cachemap_b200: demotion to the host tier failed: %s\n", cmb200_last_error());
						break;
					}
					moved += got;
					round += got;
					k += take;
				}
			} else {
				fprintf(stderr, "cachemap_b200: demotion could not sample the store: %s\n", cmb200_last_error());
			}
		}
		free(draws); free(ts); free(ok); free(cand); free(old); free(victim);
		idle = round ? 0 : idle + 1;
	}
	free(guard);
	return moved;
}

/* Before `incoming` puts: while entries + incoming > capacity, evict (cachemap.c:17-45); loops
 * until the count fits or nothing more can be retired. */
static void
filemap_evict(struct filemap *m, uint64_t incoming)
{
	if (!m->capacity)
		return;
	for (;;) {
		uint64_t entries = cmb200_entries(m->eng);
		if (entries + incoming <= m->capacity || entries == 0)
			return;
		uint64_t need = entries + incoming - m->capacity;
		if (incoming == 1)
			need = 1;       /* the reference evicts exactly one per put */
		if (filemap_evict_n(m, need) == 0 || incoming == 1)
			return;
	}
}

/* The arena is a bump allocator; deleted and outgrown records stay behind as garbage until
 * cmb200_compact slides the live ones down.  When `incoming` worst-case records would not fit:
 * compact if that frees enough; otherwise the live data itself fills the arena (the store was
 * sized in pages, the arena is bytes).  With a host tier that can take what must move, the oldest
 * records are demoted to it and the arena compacted, so the store keeps `capacity` pages as the
 * reference's LMDB files do; otherwise evict by bytes as well and compact what that frees.
 * Only when even that fails does a put get dropped, as a full LMDB map drops it
 * (filemap.c:143-145,154-157).  may_evict = 0 (room for promotion): demotion and compaction only. */
static void
filemap_arena_room(struct filemap *m, uint64_t incoming, int may_evict)
{
	const uint64_t need = incoming * ((uint64_t)m->bsize + 1056);
	int evicted = 0;
	for (int attempt = 0; attempt < 6; attempt++) {
		cmb200_stats st;
		if (cmb200_get_stats(m->eng, &st) != 0)
			return;
		if (st.arena_used + need <= st.arena_bytes)
			return;
		const uint64_t free_b = st.arena_bytes - st.arena_used;
		if (st.arena_garbage > 0 && (free_b + st.arena_garbage >= need || evicted)) {
			uint64_t got = 0;
			if (cmb200_compact(m->eng, &got) != 0) {
				fprintf(stderr, "cachemap_b200: arena compaction failed: %s\n", cmb200_last_error());
				return;
			}
			evicted = 0;
			continue;
		}
		if (st.entries == 0)
			return;
		/* live records fill the arena: move or retire enough of them (average record size, plus a margin) */
		const uint64_t live = st.arena_used > st.arena_garbage ? st.arena_used - st.arena_garbage : 1;
		const uint64_t shortfall = need - (free_b + st.arena_garbage < need ? free_b + st.arena_garbage : need);
		struct cmb200_host_tier_stats ht;
		if (m->host_tier && cmb200_host_tier_stats(m->eng, &ht) == 0 && shortfall <= ht.bytes) {
			if (st.entries <= ht.records)
				return;         /* every live record is in the tier already: evicting frees no arena bytes */
			const uint64_t in_arena = st.entries - ht.records;
			const uint64_t avg = live / in_arena ? live / in_arena : 1;
			uint64_t victims = shortfall / avg + shortfall / avg / 8 + 16;
			if (victims > in_arena)
				victims = in_arena;
			if (filemap_demote_n(m, victims) == 0)
				return;
			evicted = 1;
			continue;
		}
		if (!may_evict)
			return;
		const uint64_t avg = live / st.entries ? live / st.entries : 1;
		uint64_t victims = shortfall / avg + shortfall / avg / 8 + 16;
		if (victims > st.entries)
			victims = st.entries;
		if (filemap_evict_n(m, victims) == 0)
			return;
		evicted = 1;
	}
}

static void
filemap_check_arena(struct filemap *m, uint64_t incoming)
{
	filemap_arena_room(m, incoming, 1);
}

/* One promotion round (CMB200_TIER_PROMOTE = N): up to N addresses that gets answered from the host
 * tier since the last round, newest first, go back to the arena.  Room is made only by demoting the
 * oldest arena records and compacting, never by evicting; when that frees too little, the round
 * promotes what fits.  The addresses join the guard FIFO that demotion passes over. */
static void
filemap_promote_round(struct filemap *m)
{
	clock_gettime(CLOCK_MONOTONIC, &m->promo_last);
	size_t n = 0;
	if (cmb200_host_tier_hot(m->eng, (size_t)m->tier_promote, m->promo_hot, &n, NULL) != 0) {
		fprintf(stderr, "cachemap_b200: the host tier's hot log could not be read: %s\n", cmb200_last_error());
		return;
	}
	if (n == 0)
		return;
	filemap_arena_room(m, n, 0);
	uint64_t got = 0;
	if (cmb200_promote_batch(m->eng, n, m->promo_hot, &got) != 0) {
		fprintf(stderr, "cachemap_b200: promotion from the host tier failed: %s\n", cmb200_last_error());
		return;
	}
	pthread_mutex_lock(&m->promo_mu);
	const uint64_t cap = 4 * m->tier_promote;
	for (size_t i = 0; i < n; i++)
		m->promo_guard[m->promo_guard_n++ % cap] = m->promo_hot[i];
	pthread_mutex_unlock(&m->promo_mu);
}

/* A promotion round is due: the knob is on and PROMOTE_EVERY_MS have passed since the last one. */
static int
filemap_promote_due(struct filemap *m)
{
	if (!m->tier_promote)
		return 0;
	struct timespec now;
	clock_gettime(CLOCK_MONOTONIC, &now);
	const int64_t ms = (int64_t)(now.tv_sec - m->promo_last.tv_sec) * 1000 + (now.tv_nsec - m->promo_last.tv_nsec) / 1000000;
	return ms >= PROMOTE_EVERY_MS;
}

/* Before a batch of `incoming` puts: evict down to capacity, then make sure the arena has room
 * (what eviction frees is garbage until the arena is compacted). */
static void
filemap_make_room(struct filemap *m, uint64_t incoming)
{
	filemap_evict(m, incoming);
	filemap_check_arena(m, incoming);
}

static void
timespec_add_ms(struct timespec *t, long ms)
{
	t->tv_nsec += ms * 1000000L;
	t->tv_sec += t->tv_nsec / 1000000000L;
	t->tv_nsec %= 1000000000L;
}

/* The flusher: takes the longest run of finished slots from the tail of the ring and puts it
 * into the GPU store as one batch (two calls when the run wraps around the ring). */
static void *
filemap_flusher(void *arg)
{
	struct filemap *m = arg;
	cmb200_addr *addr = malloc(FLUSH_MAX * sizeof(cmb200_addr));
	uint64_t *ts = malloc(FLUSH_MAX * sizeof(uint64_t));
	time_t last_save = time(NULL);
	pthread_mutex_lock(&m->wb_mu);
	for (;;) {
		uint64_t count = 0;
		/* at most half the ring per batch: callers keep filling the other half while this one is on the GPU */
		const uint64_t flush_cap = m->wb_n / 2 < FLUSH_MAX ? (m->wb_n / 2 ? m->wb_n / 2 : 1) : FLUSH_MAX;
		while (m->wb_tail + count < m->wb_head && count < flush_cap &&
		    m->wb_slot[(m->wb_tail + count) % m->wb_n].state == WB_READY)
			count++;
		if (count == 0) {
			if (m->wb_stop && m->wb_tail == m->wb_head)
				break;
			if (filemap_promote_due(m)) {
				pthread_mutex_unlock(&m->wb_mu);
				filemap_promote_round(m);
				pthread_mutex_lock(&m->wb_mu);
				continue;
			}
			if (m->checkpoint_sec > 0 && m->persist) {
				struct timespec now, until;
				clock_gettime(CLOCK_REALTIME, &now);
				if (m->puts_seen != m->puts_saved && now.tv_sec - last_save >= m->checkpoint_sec) {
					pthread_mutex_unlock(&m->wb_mu);
					filemap_save(m);
					pthread_mutex_lock(&m->wb_mu);
					last_save = now.tv_sec;
					continue;
				}
				until = now;
				if (m->tier_promote)
					timespec_add_ms(&until, PROMOTE_EVERY_MS);
				else
					until.tv_sec += 1;
				m->wb_flusher_asleep = 1;
				pthread_cond_timedwait(&m->wb_work, &m->wb_mu, &until);
				m->wb_flusher_asleep = 0;
			} else if (m->tier_promote) {
				/* woken for the next promotion round at the latest */
				struct timespec until;
				clock_gettime(CLOCK_REALTIME, &until);
				timespec_add_ms(&until, PROMOTE_EVERY_MS);
				m->wb_flusher_asleep = 1;
				pthread_cond_timedwait(&m->wb_work, &m->wb_mu, &until);
				m->wb_flusher_asleep = 0;
			} else {
				m->wb_flusher_asleep = 1;
				pthread_cond_wait(&m->wb_work, &m->wb_mu);
				m->wb_flusher_asleep = 0;
			}
			continue;
		}
		for (uint64_t i = 0; i < count; i++) {
			struct wb_slot *s = &m->wb_slot[(m->wb_tail + i) % m->wb_n];
			s->state = WB_FLUSHING;
			addr[i] = s->addr;
			ts[i] = s->ts;
		}
		const uint64_t first = m->wb_tail % m->wb_n;
		pthread_mutex_unlock(&m->wb_mu);

		if (addr && ts) {
			filemap_make_room(m, count);
			uint64_t run1 = count < m->wb_n - first ? count : m->wb_n - first;
			cmb200_put_batch(m->eng, (size_t)run1, addr, NULL, m->wb_pages + first * (size_t)m->bsize, ts, NULL);
			if (run1 < count)
				cmb200_put_batch(m->eng, (size_t)(count - run1), addr + run1, NULL, m->wb_pages, ts + run1, NULL);
		}

		pthread_mutex_lock(&m->wb_mu);
		__atomic_fetch_add(&m->puts_seen, count, __ATOMIC_RELAXED);
		for (uint64_t i = 0; i < count; i++)
			m->wb_slot[(m->wb_tail + i) % m->wb_n].state = WB_FREE;
		m->wb_tail += count;
		pthread_cond_broadcast(&m->wb_space);
		pthread_cond_broadcast(&m->wb_idle);            /* waiters compare wb_tail with their own target */
		if (filemap_promote_due(m)) {
			pthread_mutex_unlock(&m->wb_mu);
			filemap_promote_round(m);
			pthread_mutex_lock(&m->wb_mu);
		}
	}
	pthread_mutex_unlock(&m->wb_mu);
	free(addr);
	free(ts);
	return NULL;
}

/* Newest copy of `addr` still in the ring -> malloc()ed page, else NULL. */
static void *
filemap_ring_lookup(struct filemap *m, const cmb200_addr *addr, void *dst)
{
	void *page = NULL;
	if (!m->wb_n)
		return NULL;
	pthread_mutex_lock(&m->wb_mu);
	for (uint64_t s = m->wb_head; s > m->wb_tail; s--) {
		struct wb_slot *w = &m->wb_slot[(s - 1) % m->wb_n];
		if (w->state >= WB_READY && w->addr.u == addr->u && w->addr.l == addr->l) {
			page = dst ? dst : malloc((size_t)m->bsize);
			if (page)
				memcpy(page, m->wb_pages + ((s - 1) % m->wb_n) * (size_t)m->bsize, (size_t)m->bsize);
			break;
		}
	}
	pthread_mutex_unlock(&m->wb_mu);
	return page;
}

/* Combining queue of the single-page calls (cachemap_get / filemap_unset from FUSE worker threads).
 *
 * A get's latency is one page's decode on one SM and an H100 decodes 132 pages at a time, so a
 * request is launched at once when it can be: whoever finds a free leader slot and nobody else
 * inside a launch takes everything queued (<= COMBINE_MAX) and launches it as ONE fused kernel
 * (cmb200_get_small_begin).  Kernel launches are what limits the rate with many callers (~100 k
 * launches/s whatever the number of threads), and only one caller launches at a time, so under load
 * the requests that arrive during a launch ride together in the next one.
 * Nobody waits for a batch: the kernel answers each request in its own status word (page-locked
 * memory) and every requester watches ITS word, copies ITS page out of the slot's stage buffer and
 * leaves; the last one out ends the launch (cmb200_get_small_end) and frees the slot.
 */
static const int32_t fm_answered = CMB200_MISS;         /* status word of requests that have no page to wait for */

/* Takes up to COMBINE_MAX queued requests into leader slot `ls` and launches them.  Called with q_mu
 * held and m->launching set; returns with q_mu held. */
static void
filemap_lead(struct filemap *m, int ls)
{
	struct fm_req *batch[COMBINE_MAX];
	cmb200_addr addr[COMBINE_MAX];
	int idx[COMBINE_MAX];
	int nb = 0, k;

	while (m->q_head && nb < COMBINE_MAX) {
		batch[nb++] = m->q_head;
		m->q_head = m->q_head->next;
	}
	if (!m->q_head)
		m->q_tail = NULL;
	__atomic_fetch_sub(&m->q_len, nb, __ATOMIC_RELAXED);
	pthread_mutex_unlock(&m->q_mu);

	k = 0;
	for (int i = 0; i < nb; i++)
		if (batch[i]->kind == REQ_UNSET)
			addr[k++] = batch[i]->addr;
	if (k)
		cmb200_unset_batch(m->eng, (size_t)k, addr);    /* unsets first: they change the table the gets read by key */

	k = 0;
	for (int i = 0; i < nb; i++) {
		if (batch[i]->kind != REQ_GET)
			continue;
		addr[k] = batch[i]->addr;
		idx[k] = i;
		k++;
	}
	uint8_t *stage = m->h_stage + (size_t)ls * COMBINE_MAX * (size_t)m->bsize;
	const volatile int32_t *answers = m->sync_status[ls];
	m->ticket[ls].lane = -1;
	if (k) {
		/* the fused small-batch get: one kernel on a stream of its own, pages land in the page-locked
		 * stage buffer directly; page sizes it does not serve (> 64 KiB) take the two-kernel batch path,
		 * synchronously */
		int rc = cmb200_get_small_begin(m->eng, (size_t)k, addr, stage, &m->ticket[ls]);
		if (rc == 0) {
			answers = m->ticket[ls].status;
		} else {
			m->ticket[ls].lane = -1;
			if (rc == -2)
				rc = cmb200_get_batch(m->eng, (size_t)k, addr, NULL, stage, m->sync_status[ls]);
			if (rc != 0)
				for (int j = 0; j < k; j++)
					m->sync_status[ls][j] = CMB200_MISS;
		}
	}

	pthread_mutex_lock(&m->q_mu);
	__atomic_store_n(&m->batch_left[ls], nb, __ATOMIC_RELEASE);
	for (int j = 0; j < k; j++)
		batch[idx[j]]->pos = j;
	k = 0;
	for (int i = 0; i < nb; i++) {
		/* slot and position first: the requester goes on as soon as it sees its status pointer, and
		 * may be gone (its request with it) right after */
		struct fm_req *r = batch[i];
		r->slot = ls;
		__atomic_store_n(&r->status, r->kind == REQ_GET ? answers + k++ : &fm_answered, __ATOMIC_RELEASE);
	}
}

/* Queues `count` requests (an array) and returns when all of them have been answered.  A requester
 * takes q_mu once to queue; after that it only takes it again to launch a batch itself or to sleep
 * when every slot is busy — watching for its launch and for its answer needs no lock. */
static void
filemap_submit_many(struct filemap *m, struct fm_req *reqs, int count)
{
	for (int i = 0; i < count; i++) {
		reqs[i].status = NULL;
		reqs[i].slot = -1;
		reqs[i].pos = 0;
		reqs[i].next = i + 1 < count ? &reqs[i + 1] : NULL;
	}
	while (sem_wait(&m->q_door) != 0)
		;
	pthread_mutex_lock(&m->q_mu);
	if (m->q_tail)
		m->q_tail->next = &reqs[0];
	else
		m->q_head = &reqs[0];
	m->q_tail = &reqs[count - 1];
	__atomic_fetch_add(&m->q_len, count, __ATOMIC_RELAXED);
	pthread_mutex_unlock(&m->q_mu);

	for (int i = 0; i < count; i++) {
		struct fm_req *r = &reqs[i];
		const volatile int32_t *answer;
		unsigned waited = 0;
		while (!(answer = __atomic_load_n(&r->status, __ATOMIC_ACQUIRE))) {
			/* Watch without the lock while somebody is inside a launch (microseconds: it either has this
			 * request with it or leaves it to the next launch), while every slot is busy, and — for a
			 * short while — when a launch now would carry very few requests into one of the last free
			 * slots: with many callers the slots are what runs out, and batches of 1 use them up. */
			const int busy = __atomic_load_n(&m->busy_slots, __ATOMIC_RELAXED);
			if (__atomic_load_n(&m->launching, __ATOMIC_ACQUIRE) || busy >= LEADERS ||
			    (busy >= LEADERS / 2 && waited < 256u && 4 * __atomic_load_n(&m->q_len, __ATOMIC_RELAXED) < busy)) {
#if defined(__x86_64__)
				__builtin_ia32_pause();
#endif
				if ((++waited & 1023u) == 0u)
					sched_yield();
				continue;
			}
			pthread_mutex_lock(&m->q_mu);
			if (!r->status && !__atomic_load_n(&m->launching, __ATOMIC_RELAXED)) {
				int ls = -1;
				for (int k = 0; k < LEADERS; k++)
					if (!m->leader_busy[k]) { ls = k; break; }
				if (ls >= 0) {
					__atomic_store_n(&m->launching, 1, __ATOMIC_RELAXED);  /* (read by watchers that hold no lock) */
					m->leader_busy[ls] = 1;
					__atomic_fetch_add(&m->busy_slots, 1, __ATOMIC_RELAXED);
					filemap_lead(m, ls);                    /* (drops and retakes q_mu around the launch) */
					__atomic_store_n(&m->launching, 0, __ATOMIC_RELEASE);
				}
			}
			pthread_mutex_unlock(&m->q_mu);
		}
		const int ls = r->slot;

		/* my answer: the kernel writes the page, fences, then the status word */
		int32_t st;
		for (unsigned spins = 0; (st = __atomic_load_n(answer, __ATOMIC_ACQUIRE)) == CMB200_SMALL_PENDING; spins++) {
#if defined(__x86_64__)
			__builtin_ia32_pause();
#endif
			if ((spins & 4095u) == 4095u)
				sched_yield();
		}
		/* (the acquire load above orders the page bytes after the status word) */
		if (r->kind == REQ_GET) {
			if (st == CMB200_HIT) {
				r->out = r->dst ? r->dst : malloc((size_t)m->bsize);    /* filemap.c:242 */
				if (r->out)
					memcpy(r->out, m->h_stage + ((size_t)ls * COMBINE_MAX + (size_t)r->pos) * (size_t)m->bsize,
					    (size_t)m->bsize);
			} else if (st == CMB200_BAD_ENTRY) {
				r->bad_entry = 1;
			}
		}

		if (__atomic_sub_fetch(&m->batch_left[ls], 1, __ATOMIC_ACQ_REL) == 0) {
			/* last one out: every status word of the launch has been seen answered, so ending it does
			 * not wait; then the slot and its stage buffer are free again */
			if (m->ticket[ls].lane >= 0)
				cmb200_get_small_end(m->eng, &m->ticket[ls], NULL);
			pthread_mutex_lock(&m->q_mu);
			m->leader_busy[ls] = 0;
			__atomic_fetch_sub(&m->busy_slots, 1, __ATOMIC_RELEASE);
			pthread_mutex_unlock(&m->q_mu);
		}
	}
	sem_post(&m->q_door);
}

static void
filemap_submit(struct filemap *m, struct fm_req *req)
{
	filemap_submit_many(m, req, 1);
}

void
filemap_set(struct filemap *m, uint128_t *key, void *value, uint64_t attr)
{
	if (!filemap_engine_ready(m))
		return;
	cmb200_addr a = { key->u, key->l };
	if (!m->wb_n) {                         /* write-behind disabled: one synchronous GPU put */
		filemap_make_room(m, 1);
		cmb200_put_batch(m->eng, 1, &a, NULL, value, &attr, NULL);
		__atomic_fetch_add(&m->puts_seen, 1, __ATOMIC_RELAXED);
		return;
	}
	pthread_mutex_lock(&m->wb_mu);
	while (m->wb_head - m->wb_tail == m->wb_n)
		pthread_cond_wait(&m->wb_space, &m->wb_mu);     /* back-pressure: the ring is full */
	const uint64_t s = m->wb_head++;
	struct wb_slot *w = &m->wb_slot[s % m->wb_n];
	w->addr = a;
	w->ts = attr;
	w->state = WB_FILLING;
	pthread_mutex_unlock(&m->wb_mu);
	memcpy(m->wb_pages + (s % m->wb_n) * (size_t)m->bsize, value, (size_t)m->bsize);
	pthread_mutex_lock(&m->wb_mu);
	w->state = WB_READY;
	if (m->wb_flusher_asleep)               /* a busy flusher finds the page by itself when it comes back: no wake-up call per put */
		pthread_cond_signal(&m->wb_work);
	pthread_mutex_unlock(&m->wb_mu);
}

void
filemap_unset(struct filemap *m, uint128_t *key)
{
	if (!filemap_engine_ready(m))
		return;
	filemap_drain(m);
	struct fm_req r;
	memset(&r, 0, sizeof(r));
	r.kind = REQ_UNSET;
	r.addr.u = key->u;
	r.addr.l = key->l;
	filemap_submit(m, &r);
}

void *
filemap_get(struct filemap *m, uint128_t *key)
{
	if (!filemap_engine_ready(m))
		return NULL;
	struct fm_req r;
	memset(&r, 0, sizeof(r));
	r.kind = REQ_GET;
	r.addr.u = key->u;
	r.addr.l = key->l;
	/* a page accepted by filemap_set but not flushed yet is served from the ring; a slot leaves
	 * the ring only after the GPU put of its batch has completed, so nothing falls between */
	void *page = filemap_ring_lookup(m, &r.addr, NULL);
	if (page)
		return page;
	filemap_submit(m, &r);
	if (r.bad_entry)
		printf("bad entry\n");          /* filemap.c:237 */
	return r.out;
}

int
filemap_get_rand(struct filemap *m, uint128_t *key, uint64_t *ts)
{
	if (!filemap_engine_ready(m))
		return 0;
	filemap_drain(m);
	/* filemap.c:271-274: a 64-bit draw built from rand() */
	uint64_t r = 0;
	for (int i = 0; i < 64; i += 30)
		r = r * ((uint64_t)RAND_MAX + 1) + (uint64_t)rand();
	cmb200_addr a;
	int32_t ok = 0;
	if (cmb200_sample(m->eng, 1, &r, &a, ts, &ok) != 0 || !ok)
		return 0;
	key->u = a.u;
	key->l = a.l;
	return 1;
}

uint64_t
filemap_entries(struct filemap *m)
{
	if (!filemap_engine_ready(m))
		return 0;
	filemap_drain(m);
	return cmb200_entries(m->eng);
}

/* ------------------------------------------------------------------------------------------ */

struct cachemap {
	struct filemap *pages;  /* first member, as in the reference (cachemap.h:20-21) */
	uint64_t capacity;
	uint64_t requests;
	uint64_t hits;
};

static uint64_t
now_ns(void)
{
	struct timespec tp;
	(void)clock_gettime(CLOCK_REALTIME_COARSE, &tp);        /* cachemap.c:10-15 */
	return (uint64_t)tp.tv_sec * 1000000000ULL + (uint64_t)tp.tv_nsec;
}

/* cachemap.c:151-166 */
static int
compose_addr(struct cachemap *cm, uint64_t offset, uint64_t nhid_small, uint32_t genid, cmb200_addr *out)
{
	uint64_t page = offset >> cm->pages->pshift;
	if (page >> PNUM_SHIFT)
		return -1;
	out->l = page | ((uint64_t)genid << PNUM_SHIFT);
	out->u = nhid_small;
	return 0;
}

struct cachemap *
cachemap_create(char *destdir, uint64_t capacity, int comp_accel, int pshift)
{
	struct stat sb;
	if (!destdir || stat(destdir, &sb) != 0 || !S_ISDIR(sb.st_mode))   /* cachemap.c:113-114 */
		return NULL;
	struct cachemap *cm = calloc(1, sizeof(*cm));
	if (!cm)
		return NULL;
	cm->pages = filemap_create(destdir, capacity, comp_accel, pshift);
	if (!cm->pages) {
		free(cm);
		return NULL;
	}
	cm->capacity = capacity;
	cm->pages->capacity = capacity;         /* the flusher evicts before each batch (cachemap.c:17-45) */
	return cm;
}

void *
cachemap_get(struct cachemap *cm, uint64_t offset, uint64_t nhid_small, uint32_t genid)
{
	cmb200_addr a;
	if (compose_addr(cm, offset, nhid_small, genid, &a) != 0)
		return NULL;
	__atomic_fetch_add(&cm->requests, 1, __ATOMIC_RELAXED);         /* cachemap.c:176 */
	uint128_t key = { a.u, a.l };
	void *page = filemap_get(cm->pages, &key);
	if (page)
		__atomic_fetch_add(&cm->hits, 1, __ATOMIC_RELAXED);     /* cachemap.c:181 */
	return page;
}

void
cachemap_put(struct cachemap *cm, uint64_t offset, uint64_t nhid_small, uint32_t genid, const void *page)
{
	cmb200_addr a;
	if (compose_addr(cm, offset, nhid_small, genid, &a) != 0)
		return;
	uint128_t key = { a.u, a.l };
	filemap_set(cm->pages, &key, (void *)page, now_ns());   /* copies the page before returning */
}

/* The reference copies the page and queues it for 4 worker threads (cachemap.c:199-216); here
 * every put is already write-behind, so the two entry points are the same. */
void
cachemap_put_async(struct cachemap *cm, uint64_t offset, uint64_t nhid_small, uint32_t genid, const void *page)
{
	cachemap_put(cm, offset, nhid_small, genid, page);
}

void
cachemap_free(struct cachemap *cm)
{
	if (!cm)
		return;
	filemap_free(cm->pages);                /* drains the write-behind ring (cachemap.c:218-232) */
	free(cm);
}

void
cachemap_print_stats(struct cachemap *cm)
{
	uint64_t rq = __atomic_load_n(&cm->requests, __ATOMIC_RELAXED);
	uint64_t ht = __atomic_load_n(&cm->hits, __ATOMIC_RELAXED);
	printf("requests: %lu, hits: %lu, ratio: %5.2f\n",              /* cachemap.c:237-238 */
	    (unsigned long)rq, (unsigned long)ht, ht * 100 / (float)rq);
}

/* ---- batch extension ---------------------------------------------------------------------- */

struct batch_keys {
	cmb200_addr *addr;
	uint8_t *valid;
	uint64_t *ts;
};

static int
batch_keys_build(struct cachemap *cm, uint64_t n, const uint64_t *offset, const uint64_t *nhid,
    const uint32_t *genid, int want_ts, struct batch_keys *bk)
{
	bk->addr = malloc((size_t)n * sizeof(cmb200_addr));
	bk->valid = malloc((size_t)n);
	bk->ts = want_ts ? malloc((size_t)n * 8) : NULL;
	if (!bk->addr || !bk->valid || (want_ts && !bk->ts)) {
		free(bk->addr); free(bk->valid); free(bk->ts);
		return -1;
	}
	uint64_t ts = want_ts ? now_ns() : 0;
	for (uint64_t i = 0; i < n; i++) {
		bk->valid[i] = compose_addr(cm, offset[i], nhid[i], genid ? genid[i] : 0, &bk->addr[i]) == 0;
		if (!bk->valid[i])
			memset(&bk->addr[i], 0, sizeof(cmb200_addr));
		if (want_ts)
			bk->ts[i] = ts;
	}
	return 0;
}

static void
batch_keys_free(struct batch_keys *bk)
{
	free(bk->addr); free(bk->valid); free(bk->ts);
}

static void
put_batch_common(struct cachemap *cm, uint64_t n, const uint64_t *offset, const uint64_t *nhid,
    const uint32_t *genid, const void *pages, int on_dev)
{
	struct batch_keys bk;
	if (n == 0 || !filemap_engine_ready(cm->pages))
		return;
	if (batch_keys_build(cm, n, offset, nhid, genid, 1, &bk) != 0)
		return;
	filemap_drain(cm->pages);               /* earlier single puts land first */
	__atomic_fetch_add(&cm->pages->puts_seen, n, __ATOMIC_RELAXED);
	/* One GPU batch when the store has room for all of it; at capacity the batch goes in slices
	 * with eviction before each, so that entries never run past capacity by more than a slice
	 * (the reference evicts before every single put, cachemap.c:186-197). */
	uint64_t slice = n;
	if (cm->capacity && cmb200_entries(cm->pages->eng) + n > cm->capacity) {
		slice = cm->capacity / 4;
		if (slice > 4096)
			slice = 4096;
		if (slice < 1)
			slice = 1;
	}
	const size_t bsize = (size_t)cm->pages->bsize;
	for (uint64_t at = 0; at < n; at += slice) {
		const uint64_t m = n - at < slice ? n - at : slice;
		const uint8_t *pg = (const uint8_t *)pages + at * bsize;
		filemap_make_room(cm->pages, m);
		if (on_dev)
			cmb200_put_batch_dev(cm->pages->eng, (size_t)m, bk.addr + at, bk.valid + at, pg, bk.ts + at, NULL);
		else {
			/* write-behind like cachemap_put: back when the pages have crossed to the GPU and the
			 * caller may reuse them; whatever is called next is ordered after the encode */
			uint64_t ticket;
			cmb200_put_batch_async(cm->pages->eng, (size_t)m, bk.addr + at, bk.valid + at, pg, bk.ts + at, NULL, &ticket);
		}
	}
	batch_keys_free(&bk);
}

static void
get_batch_common(struct cachemap *cm, uint64_t n, const uint64_t *offset, const uint64_t *nhid,
    const uint32_t *genid, void *pages_out, uint8_t *hit_out, int on_dev)
{
	struct batch_keys bk;
	memset(hit_out, 0, (size_t)n);
	if (n == 0 || !filemap_engine_ready(cm->pages))
		return;
	if (batch_keys_build(cm, n, offset, nhid, genid, 0, &bk) != 0)
		return;
	filemap_drain(cm->pages);
	int32_t *status = malloc((size_t)n * 4);
	int rc = -1;
	if (status)
		rc = on_dev ? cmb200_get_batch_dev(cm->pages->eng, (size_t)n, bk.addr, bk.valid, pages_out, status)
			    : cmb200_get_batch(cm->pages->eng, (size_t)n, bk.addr, bk.valid, pages_out, status);
	uint64_t rq = 0, ht = 0;
	for (uint64_t i = 0; i < n; i++) {
		if (!bk.valid[i])
			continue;                       /* cachemap.c:173-174: not a request */
		rq++;
		if (rc == 0 && status[i] == CMB200_HIT) {
			hit_out[i] = 1;
			ht++;
		} else if (rc == 0 && status[i] == CMB200_BAD_ENTRY) {
			printf("bad entry\n");
		}
	}
	__atomic_fetch_add(&cm->requests, rq, __ATOMIC_RELAXED);
	__atomic_fetch_add(&cm->hits, ht, __ATOMIC_RELAXED);
	free(status);
	batch_keys_free(&bk);
}

void
cachemap_put_batch(struct cachemap *cm, uint64_t n, const uint64_t *offset, const uint64_t *nhid_small,
    const uint32_t *genid, const void *pages)
{
	put_batch_common(cm, n, offset, nhid_small, genid, pages, 0);
}

void
cachemap_put_batch_dev(struct cachemap *cm, uint64_t n, const uint64_t *offset, const uint64_t *nhid_small,
    const uint32_t *genid, const void *pages_dev)
{
	put_batch_common(cm, n, offset, nhid_small, genid, pages_dev, 1);
}

void
cachemap_get_batch(struct cachemap *cm, uint64_t n, const uint64_t *offset, const uint64_t *nhid_small,
    const uint32_t *genid, void *pages_out, uint8_t *hit_out)
{
	get_batch_common(cm, n, offset, nhid_small, genid, pages_out, hit_out, 0);
}

void
cachemap_get_batch_dev(struct cachemap *cm, uint64_t n, const uint64_t *offset, const uint64_t *nhid_small,
    const uint32_t *genid, void *pages_out_dev, uint8_t *hit_out)
{
	get_batch_common(cm, n, offset, nhid_small, genid, pages_out_dev, hit_out, 1);
}

/* ---- request ranges (edgefs.c:1159-1195, 1216-1228) ------------------------------------------ */

int
cachemap_read_range(struct cachemap *cm, uint64_t nhid_small, uint32_t genid, uint64_t off, size_t size,
    void *out_buf)
{
	const int pshift = cm->pages->pshift;
	const uint64_t page_size = 1ULL << pshift;
	if ((off & (page_size - 1)) || ((off + (uint64_t)size) & (page_size - 1)))     /* edgefs.c:192-203 */
		return 0;
	const uint64_t n = (uint64_t)size >> pshift;
	if (n == 0)
		return 1;
	if (!filemap_engine_ready(cm->pages))
		return 0;
	struct fm_req *reqs = calloc((size_t)n, sizeof(*reqs));
	int *which = malloc((size_t)n * sizeof(int));
	uint8_t *state = calloc((size_t)n, 1);          /* 0 miss, 1 hit, 2 invalid address */
	if (!reqs || !which || !state) {
		free(reqs); free(which); free(state);
		return 0;
	}
	/* pages still in the write-behind ring are served from it, the rest go to the GPU as one
	 * chain of requests (one batch unless the chain is longer than COMBINE_MAX) */
	int k = 0;
	for (uint64_t i = 0; i < n; i++) {
		cmb200_addr a;
		uint8_t *dst = (uint8_t *)out_buf + (i << pshift);
		if (compose_addr(cm, off + (i << pshift), nhid_small, genid, &a) != 0) {
			state[i] = 2;
			continue;
		}
		if (filemap_ring_lookup(cm->pages, &a, dst)) {
			state[i] = 1;
			continue;
		}
		reqs[k].kind = REQ_GET;
		reqs[k].addr = a;
		reqs[k].dst = dst;
		which[k] = (int)i;
		k++;
	}
	if (k)
		filemap_submit_many(cm->pages, reqs, k);
	for (int j = 0; j < k; j++) {
		if (reqs[j].out)
			state[which[j]] = 1;
	}
	/* counters as the reference's loop leaves them: it stops at the first page that is not a
	 * hit; an invalid address returns NULL without counting a request (cachemap.c:173-174) */
	uint64_t rq = 0, ht = 0, i = 0;
	for (; i < n; i++) {
		if (state[i] == 2)
			break;
		rq++;
		if (state[i] != 1)
			break;
		ht++;
	}
	for (int j = 0; j < k; j++)
		if (reqs[j].bad_entry && (uint64_t)which[j] <= i)
			printf("bad entry\n");                  /* filemap.c:237 */
	__atomic_fetch_add(&cm->requests, rq, __ATOMIC_RELAXED);
	__atomic_fetch_add(&cm->hits, ht, __ATOMIC_RELAXED);
	free(reqs); free(which); free(state);
	return i == n;
}

void
cachemap_write_range(struct cachemap *cm, uint64_t nhid_small, uint32_t genid, uint64_t off, size_t size,
    const void *data)
{
	const int pshift = cm->pages->pshift;
	const uint64_t page_size = 1ULL << pshift;
	if ((off & (page_size - 1)) || ((off + (uint64_t)size) & (page_size - 1)))     /* edgefs.c:192-203 */
		return;
	/* every put is write-behind (one memcpy into the page-locked ring), so the loop of
	 * edgefs.c:1186-1190 / 1219-1223 already hands the GPU one batch */
	for (uint64_t i = 0; i < ((uint64_t)size >> pshift); i++)
		cachemap_put(cm, off + (i << pshift), nhid_small, genid, (const uint8_t *)data + (i << pshift));
}

int
cachemap_checkpoint(struct cachemap *cm)
{
	if (!filemap_engine_ready(cm->pages))
		return -1;
	filemap_drain(cm->pages);
	return filemap_save(cm->pages);
}

void
cachemap_get_counters(struct cachemap *cm, uint64_t *requests, uint64_t *hits)
{
	*requests = __atomic_load_n(&cm->requests, __ATOMIC_RELAXED);
	*hits = __atomic_load_n(&cm->hits, __ATOMIC_RELAXED);
}

struct cmb200_engine *
cachemap_engine(struct cachemap *cm)
{
	if (!filemap_engine_ready(cm->pages))
		return NULL;
	filemap_drain(cm->pages);               /* callers of the engine see every accepted put */
	return cm->pages->eng;
}
