/*
 * cachemap_api.c — the reference's C API (include/cachemap.h, include/filemap.h) over the H100
 * engine.  Host code stays C; everything heavy happens in the engine's kernels.
 *
 * What each reference function became:
 *   filemap_create/free        cachemap/filemap.c:35-110   -> config only; engines built lazily
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
 *
 * One map, several GPUs (CMB200_DEVICES): the reference already splits its store into 32 shards by
 * key and no call but filemap_entries crosses shards (filemap.c:26-33).  Here the map owns one engine
 * per listed device and every key lives on exactly one of them, cmb200_owner(key, G).  Each engine
 * has its own write-behind ring and flusher, combining queue, host tier and promotion state (struct
 * fm_dev); the map keeps the capacity, the counters, the eviction decision and persistence.  Without
 * CMB200_DEVICES there is one engine on CMB200_DEVICE: G = 1 of the same code.
 *
 * There is no CPU fallback: if an engine cannot be created the process stops with a message
 * (set CMB200_SOFT_FAIL=1 to degrade to "every put dropped, every get a miss" instead).
 */
#define _GNU_SOURCE
#include <dirent.h>
#include <errno.h>
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

/* the library's external definition of the header's inline cmb200_owner */
extern int cmb200_owner(uint64_t key, int g);

/* The host tier is optional in the engine this layer links against: libcachemap's engine defines
 * these, an engine without a tier (such as the CPU stand-in the host-layer tests link) does not, and
 * then they are null and CMB200_HOST_TIER_MB is refused.  The same holds for the calls of a sharded
 * store: without the snapshot set calls a map does not persist, without the page moves and device
 * memory the _dev batch calls serve G = 1 only. */
#pragma weak cmb200_host_tier_enable
#pragma weak cmb200_demote_batch
#pragma weak cmb200_host_tier_stats
#pragma weak cmb200_promote_batch
#pragma weak cmb200_host_tier_hot
#pragma weak cmb200_save_set
#pragma weak cmb200_load_set
#pragma weak cmb200_chain_begin
#pragma weak cmb200_snapshot_finish
#pragma weak cmb200_load_chain
#pragma weak cmb200_move_pages
#pragma weak cmb200_copy_peer
#pragma weak cmb200_dev_alloc
#pragma weak cmb200_dev_free
#pragma weak cmb200_invalidate
#pragma weak cmb200_patch_batch

#define COMBINE_MAX 32          /* get/unset requests one leader takes per GPU batch */
#define LEADERS 32              /* batches of gets that may be in flight at once, each on its own engine lane
                                 * (<= the engine's GET_LANES); see the combining queue below */
#define GET_CALLERS 32          /* callers inside the combining queue at once; the rest sleep at its door */
#define FLUSH_MAX 4096          /* pages the flusher hands over per GPU batch */
#define PNUM_SHIFT 44           /* cachemap.c:155 */
#define PROMOTE_EVERY_MS 100    /* CMB200_TIER_PROMOTE: at most one promotion round this often */
#define MAX_DEVICES 64          /* engines one map may own (CMB200_DEVICES) */

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
	uint64_t key;           /* store key of addr (addr_key): ring lookups go by key, as the store does */
	uint64_t ts;
	int state;
};

/* One engine of the map and everything that feeds it: the keys with cmb200_owner(key, G) == index. */
struct fm_dev {
	struct filemap *m;
	int index;              /* position in CMB200_DEVICES */
	int device;             /* CUDA ordinal (-1 = the current device: CMB200_DEVICES unset, CMB200_DEVICE unset) */
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
	pthread_mutex_t land_mu;        /* held while a put batch lands in this engine (filemap_land_begin) */
	/* staging of this engine's share of batch calls that span engines (stage_mu): page-locked host
	 * pages, and device buffers on the first engine's GPU and on this engine's, grown as needed */
	pthread_mutex_t stage_mu;
	uint8_t *h_put;
	void *d_first, *d_own;
	size_t d_first_bytes, d_own_bytes;
};

struct filemap {
	uint64_t n;
	int compress;
	int bsize;
	int pshift;
	char destdir[2048];
	uint64_t capacity;      /* eviction threshold (set by cachemap_create), 0 = none */
	/* engines, built on first use (fork safety, SURVEY.md §3.1) */
	pthread_mutex_t init_mu;
	int init_state;         /* 0 = not yet, 1 = ready, -1 = failed */
	int g;                  /* engines (G) */
	struct fm_dev *dev[MAX_DEVICES];
	cmb200_engine *engs[MAX_DEVICES];
	/* eviction by count is one decision over all engines, taken under evict_mu: a batch reserves its
	 * pages (filemap_evict) until they have landed in their engine (filemap_land_end), so that two
	 * flushers never evict for the same excess nor both fill the same room */
	pthread_mutex_t evict_mu;
	uint64_t reserved;      /* (atomic) */
	/* persistence: <destdir>/cachemap_b200.snap (cmb200_save_set / cmb200_load_set) */
	int persist;
	long checkpoint_sec;    /* > 0: the checkpoint thread saves a snapshot this often when puts have landed */
	long checkpoint_deltas; /* CMB200_CHECKPOINT_DELTAS: > 0 = its ticks write deltas of a chain, at most this many per base */
	int chain_deltas;       /* deltas of the chain at the snapshot path, -1 = no chain open (under snap_mu) */
	uint64_t puts_seen, puts_saved; /* (atomic) */
	pthread_mutex_t snap_mu;
	/* the checkpoint thread (CMB200_CHECKPOINT_SEC): sleeps on ckpt_cv, so that filemap_free can wake it */
	pthread_mutex_t ckpt_mu;
	pthread_cond_t ckpt_cv;
	pthread_t ckpt_thread;
	int ckpt_started, ckpt_stop;
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

/* The store key of `a`: the store keeps one record per key, not per address. */
static uint64_t
addr_key(const cmb200_addr *a)
{
	uint64_t key;
	FNV_hash(a, (int)sizeof(*a), &key);                     /* filemap.c:18-24 */
	return key;
}

/* The engine that owns `a`. */
static struct fm_dev *
filemap_owner(struct filemap *m, const cmb200_addr *a)
{
	return m->dev[cmb200_owner(addr_key(a), m->g)];
}

/* CMB200_DEVICES: "all", or a comma-separated list of CUDA ordinals (one may repeat: two engines on
 * one GPU).  Unset: one engine on CMB200_DEVICE.  Returns how many, 0 for a list that names none. */
static int
filemap_device_list(int *out)
{
	const char *v = getenv("CMB200_DEVICES");
	if (!v || !*v) {
		out[0] = (int)env_long("CMB200_DEVICE", -1);
		return 1;
	}
	if (strcmp(v, "all") == 0) {
		int n = cmb200_device_count();
		if (n > MAX_DEVICES)
			n = MAX_DEVICES;
		for (int i = 0; i < n; i++)
			out[i] = i;
		return n > 0 ? n : 0;
	}
	int n = 0;
	const char *p = v;
	for (;;) {
		char *end;
		const long d = strtol(p, &end, 10);
		if (end == p || d < 0 || d > 1023 || n == MAX_DEVICES)
			return 0;
		out[n++] = (int)d;
		while (*end == ' ')
			end++;
		if (*end == '\0')
			return n;
		if (*end != ',')
			return 0;
		p = end + 1;
	}
}

static void *filemap_flusher(void *arg);
static void *filemap_checkpointer(void *arg);

static void
fm_dev_free(struct fm_dev *d)
{
	if (!d)
		return;
	if (d->wb_pages)
		cmb200_host_free(d->wb_pages);
	free(d->wb_slot);
	if (d->h_stage)
		cmb200_host_free(d->h_stage);
	if (d->eng)
		cmb200_engine_destroy(d->eng);
	free(d->promo_hot);
	free(d->promo_guard);
	pthread_mutex_destroy(&d->promo_mu);
	pthread_mutex_destroy(&d->land_mu);
	pthread_mutex_destroy(&d->stage_mu);
	pthread_mutex_destroy(&d->q_mu);
	sem_destroy(&d->q_door);
	pthread_mutex_destroy(&d->wb_mu);
	pthread_cond_destroy(&d->wb_space);
	pthread_cond_destroy(&d->wb_work);
	pthread_cond_destroy(&d->wb_idle);
	free(d);
}

/* CMB200_EVICT: what a record's timestamp means to eviction and demotion, which take the oldest of what
 * they sample.  "put" (or unset): the put time, the reference's policy.  "access": the last hit as well
 * (CMB200_TOUCH), so pages that are read stay.  Reads alone are not changes for a checkpoint (puts_seen):
 * a full snapshot saves the touched timestamps, a chain delta carries only the records put since the last
 * tick, each with the timestamp it had then.  Any other value warns (once, with `warn`) and keeps "put". */
static uint32_t
evict_flags(int warn)
{
	const char *v = getenv("CMB200_EVICT");
	if (!v || !*v || strcmp(v, "put") == 0)
		return 0;
	if (strcmp(v, "access") == 0)
		return CMB200_TOUCH;
	if (warn)
		fprintf(stderr, "cachemap_b200: CMB200_EVICT=%s is neither put nor access; evicting by put time\n", v);
	return 0;
}

/* Engine `index` of the map on CUDA device `device`, with its buffers; NULL if it cannot start.
 * The knobs apply per engine; the table and the default arena are sized for its share of the
 * capacity, ceil(n / G). */
static struct fm_dev *
fm_dev_start(struct filemap *m, int index, int device, int g)
{
	struct fm_dev *d = calloc(1, sizeof(*d));
	if (!d)
		return NULL;
	d->m = m;
	d->index = index;
	d->device = device;
	pthread_mutex_init(&d->q_mu, NULL);
	sem_init(&d->q_door, 0, GET_CALLERS);
	pthread_mutex_init(&d->wb_mu, NULL);
	pthread_cond_init(&d->wb_space, NULL);
	pthread_cond_init(&d->wb_work, NULL);
	pthread_cond_init(&d->wb_idle, NULL);
	pthread_mutex_init(&d->promo_mu, NULL);
	pthread_mutex_init(&d->land_mu, NULL);
	pthread_mutex_init(&d->stage_mu, NULL);

	cmb200_config cfg;
	memset(&cfg, 0, sizeof(cfg));
	cfg.device = device;
	cfg.pshift = m->pshift;
	cfg.accel = m->compress;
	cfg.capacity = (m->n + (uint64_t)g - 1) / (uint64_t)g;
	cfg.arena_bytes = (uint64_t)env_long("CMB200_ARENA_MB", 0) << 20;
	cfg.table_slots = (uint64_t)env_long("CMB200_TABLE_SLOTS", 0);
	cfg.max_batch = (uint32_t)env_long("CMB200_MAX_BATCH", 0);
	cfg.flags = env_long("CMB200_FINGERPRINT", 0) ? CMB200_FINGERPRINT : 0;
	/* every get compared with its page's EF128 on the GPU; a page that differs is a miss */
	if (env_long("CMB200_VERIFY", 0)) cfg.flags |= CMB200_VERIFY;
	cfg.flags |= evict_flags(index == 0);
	d->eng = cmb200_engine_create(&cfg);
	const long tier_mb = env_long("CMB200_HOST_TIER_MB", 0);
	if (d->eng && tier_mb > 0) {
		if (!cmb200_host_tier_enable)
			fprintf(stderr, "cachemap_b200: no host tier of %ld MiB: the engine has none\n", tier_mb);
		else if (cmb200_host_tier_enable(d->eng, (uint64_t)tier_mb << 20) == 0)
			d->host_tier = 1;
		else
			fprintf(stderr, "cachemap_b200: no host tier of %ld MiB: %s\n", tier_mb, cmb200_last_error());
	}
	const long promote = env_long("CMB200_TIER_PROMOTE", 0);
	if (d->host_tier && promote > 0) {
		if (!cmb200_promote_batch || !cmb200_host_tier_hot)
			fprintf(stderr, "cachemap_b200: CMB200_TIER_PROMOTE ignored: the engine cannot promote\n");
		else {
			d->promo_hot = malloc((size_t)promote * sizeof(cmb200_addr));
			d->promo_guard = malloc(4 * (size_t)promote * sizeof(cmb200_addr));
			if (d->promo_hot && d->promo_guard)
				d->tier_promote = (uint64_t)promote;
		}
	}
	if (d->eng) {
		d->h_stage = cmb200_host_alloc((size_t)LEADERS * COMBINE_MAX * m->bsize);
		/* ring of 256 MiB by default, at least 64 pages.  The size sets the batch the flusher can form
		 * (half the ring), and a batch below ~2 000 chunks leaves the encode kernel a partial wave
		 * whose duration is one chunk's latency (~2 ms for a text-like page) whatever its size */
		long slots = env_long("CMB200_WB_SLOTS", (256L << 20) / m->bsize);
		if (slots > 0 && slots < 64)
			slots = 64;
		if (slots > 0) {
			d->wb_pages = cmb200_host_alloc((size_t)slots * m->bsize);
			d->wb_slot = calloc((size_t)slots, sizeof(struct wb_slot));
			d->wb_n = (d->wb_pages && d->wb_slot) ? (uint64_t)slots : 0;
		}
	}
	if (!d->eng || !d->h_stage) {
		fprintf(stderr, "cachemap_b200: cannot start the GPU engine on device %d: %s\n", device, cmb200_last_error());
		fm_dev_free(d);
		return NULL;
	}
	return d;
}

static int
filemap_engine_ready(struct filemap *m)
{
	if (__atomic_load_n(&m->init_state, __ATOMIC_ACQUIRE) == 1)
		return 1;
	pthread_mutex_lock(&m->init_mu);
	if (m->init_state == 0) {
		int devs[MAX_DEVICES];
		const int g = filemap_device_list(devs);
		int started = 0;
		if (g == 0)
			fprintf(stderr, "cachemap_b200: CMB200_DEVICES=%s names no device\n", getenv("CMB200_DEVICES"));
		/* all engines or none */
		while (started < g && (m->dev[started] = fm_dev_start(m, started, devs[started], g)) != NULL)
			started++;
		if (g == 0 || started < g) {
			for (int i = 0; i < started; i++) {
				fm_dev_free(m->dev[i]);
				m->dev[i] = NULL;
			}
			if (!env_long("CMB200_SOFT_FAIL", 0)) {
				fprintf(stderr, "cachemap_b200: no CPU fallback exists; aborting "
				    "(CMB200_SOFT_FAIL=1 turns this into dropped puts / misses)\n");
				abort();
			}
			__atomic_store_n(&m->init_state, -1, __ATOMIC_RELEASE);
		} else {
			m->g = g;
			for (int i = 0; i < g; i++)
				m->engs[i] = m->dev[i]->eng;
			/* what the cache directory holds from an earlier run comes back first: the reference's
			 * store is persistent (LMDB files under destdir, filemap.c:57,71-72).  A file saved with
			 * any number of engines loads into this one's. */
			m->persist = (int)env_long("CMB200_PERSIST", 1);
			m->checkpoint_sec = env_long("CMB200_CHECKPOINT_SEC", 0);
			m->checkpoint_deltas = env_long("CMB200_CHECKPOINT_DELTAS", 0);
			m->chain_deltas = -1;
			char snap[2200], d1[2300];
			if (m->persist && filemap_snapshot_path(m, snap, sizeof(snap)) && access(snap, R_OK) == 0) {
				uint64_t got = 0;
				uint32_t k = 0;
				snprintf(d1, sizeof(d1), "%s.d1", snap);
				/* a chain next to the base is never ignored, whatever CMB200_CHECKPOINT_DELTAS says now;
				 * a base whose deltas do not match it loads alone */
				if (cmb200_load_chain && (m->checkpoint_deltas > 0 || access(d1, R_OK) == 0)) {
					if (cmb200_load_chain(m->engs, g, snap, &got, &k) != 0)
						fprintf(stderr, "cachemap_b200: %s ignored: %s\n", snap, cmb200_last_error());
					else
						m->chain_deltas = (int)k;
				} else if (!cmb200_load_set)
					fprintf(stderr, "cachemap_b200: %s ignored: the engine cannot load snapshots\n", snap);
				else if (cmb200_load_set(m->engs, g, snap, &got) != 0)
					fprintf(stderr, "cachemap_b200: %s ignored: %s\n", snap, cmb200_last_error());
			}
			/* the flushers start here, i.e. in the process that actually caches (after any fork) */
			for (int i = 0; i < g; i++) {
				struct fm_dev *d = m->dev[i];
				if (d->wb_n && pthread_create(&d->wb_thread, NULL, filemap_flusher, d) == 0)
					d->wb_started = 1;
				else
					d->wb_n = 0;
			}
			if (m->persist && m->checkpoint_sec > 0 &&
			    pthread_create(&m->ckpt_thread, NULL, filemap_checkpointer, m) == 0)
				m->ckpt_started = 1;
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
	pthread_mutex_init(&m->evict_mu, NULL);
	pthread_mutex_init(&m->snap_mu, NULL);
	pthread_mutex_init(&m->ckpt_mu, NULL);
	pthread_cond_init(&m->ckpt_cv, NULL);
	return m;
}

/* Removes the deltas (and half-written deltas) of any chain next to the base at `snap`: a base that
 * was just renamed into place has a chain id of its own, or none. */
static void
filemap_remove_deltas(struct filemap *m)
{
	DIR *dir = opendir(m->destdir);
	if (!dir)
		return;
	const char *stem = SNAPSHOT_NAME ".d";
	struct dirent *ent;
	char path[2600];
	while ((ent = readdir(dir)) != NULL)
		if (strncmp(ent->d_name, stem, strlen(stem)) == 0 &&
		    snprintf(path, sizeof(path), "%s/%s", m->destdir, ent->d_name) < (int)sizeof(path))
			unlink(path);
	closedir(dir);
}

static long long
file_bytes(const char *path)
{
	struct stat st;
	return stat(path, &st) == 0 ? (long long)st.st_size : -1;
}

/* CMB200_CHECKPOINT_DELTAS: one tick of the chain at `snap` (under snap_mu).  A tick of the checkpoint
 * thread writes the chain's next delta; it writes a base instead when no chain is open (none yet, or a
 * load left the engines without chain state), when the chain already has checkpoint_deltas deltas, or
 * when its deltas together are as large as its base, so that a chain stays within about twice the store.
 * cachemap_checkpoint and cachemap_free always write a base. */
static int
filemap_save_chain(struct filemap *m, const char *snap, int tick)
{
	int delta = tick && m->chain_deltas >= 0 && m->chain_deltas < m->checkpoint_deltas;
	if (delta) {
		long long sum = 0;
		char path[2300];
		for (int k = 1; k <= m->chain_deltas; k++) {
			snprintf(path, sizeof(path), "%s.d%d", snap, k);
			const long long b = file_bytes(path);
			sum += b > 0 ? b : 0;
		}
		delta = sum < file_bytes(snap);
	}
	cmb200_snapshot *s = delta ? cmb200_chain_begin(m->engs, m->g, snap, 1) : NULL;
	if (!s) {
		delta = 0;
		s = cmb200_chain_begin(m->engs, m->g, snap, 0);
	}
	const int rc = s ? cmb200_snapshot_finish(s, NULL) : -1;
	if (rc == 0 && delta)
		m->chain_deltas++;
	else if (rc == 0) {
		m->chain_deltas = 0;
		filemap_remove_deltas(m);
	}
	return rc;
}

/* Saves the store to <destdir>/cachemap_b200.snap (tick: a save of the checkpoint thread, which may
 * write a delta instead).  0 = saved, -1 = not (disabled, engine never started, or I/O error). */
static int
filemap_save(struct filemap *m, int tick)
{
	char snap[2200];
	if (__atomic_load_n(&m->init_state, __ATOMIC_ACQUIRE) != 1 || !m->persist ||
	    !filemap_snapshot_path(m, snap, sizeof(snap)))
		return -1;
	const int chain = m->checkpoint_deltas > 0 && cmb200_chain_begin && cmb200_snapshot_finish;
	if (!chain && !cmb200_save_set) {
		fprintf(stderr, "cachemap_b200: snapshot not written: the engine cannot save snapshots\n");
		return -1;
	}
	pthread_mutex_lock(&m->snap_mu);
	uint64_t seen = __atomic_load_n(&m->puts_seen, __ATOMIC_RELAXED);
	int rc;
	if (chain)
		rc = filemap_save_chain(m, snap, tick);
	else if ((rc = cmb200_save_set(m->engs, m->g, snap, NULL)) == 0 && m->chain_deltas >= 0) {
		/* a chain loaded at start is folded into this base */
		m->chain_deltas = -1;
		filemap_remove_deltas(m);
	}
	if (rc == 0)
		__atomic_store_n(&m->puts_saved, seen, __ATOMIC_RELAXED);
	else
		fprintf(stderr, "cachemap_b200: snapshot not written: %s\n", cmb200_last_error());
	pthread_mutex_unlock(&m->snap_mu);
	return rc;
}

/* CMB200_CHECKPOINT_SEC: every checkpoint_sec seconds, a snapshot if puts have landed since the last
 * one.  The engines list their records under their locks and write them outside, so neither the
 * flushers nor the callers of the map wait for the file. */
static void *
filemap_checkpointer(void *arg)
{
	struct filemap *m = arg;
	pthread_mutex_lock(&m->ckpt_mu);
	while (!m->ckpt_stop) {
		struct timespec until;
		clock_gettime(CLOCK_REALTIME, &until);
		until.tv_sec += m->checkpoint_sec;
		while (!m->ckpt_stop && pthread_cond_timedwait(&m->ckpt_cv, &m->ckpt_mu, &until) != ETIMEDOUT)
			;
		if (m->ckpt_stop)
			break;
		pthread_mutex_unlock(&m->ckpt_mu);
		if (__atomic_load_n(&m->puts_seen, __ATOMIC_RELAXED) != __atomic_load_n(&m->puts_saved, __ATOMIC_RELAXED))
			filemap_save(m, 1);
		pthread_mutex_lock(&m->ckpt_mu);
	}
	pthread_mutex_unlock(&m->ckpt_mu);
	return NULL;
}

/* Waits until every page accepted by this engine's ring so far is in its store. */
static void
fm_dev_drain(struct fm_dev *d)
{
	if (!d->wb_n)
		return;
	pthread_mutex_lock(&d->wb_mu);
	/* everything accepted before this call, not "until the ring is empty": with other threads
	 * still putting the ring may never be empty (the flusher broadcasts after every batch) */
	const uint64_t target = d->wb_head;
	while (d->wb_tail < target)
		pthread_cond_wait(&d->wb_idle, &d->wb_mu);
	pthread_mutex_unlock(&d->wb_mu);
}

/* Waits until every page accepted so far is in the GPU store. */
static void
filemap_drain(struct filemap *m)
{
	for (int i = 0; i < m->g; i++)
		fm_dev_drain(m->dev[i]);
}

/* Live entries over all engines. */
static uint64_t
filemap_count(struct filemap *m)
{
	uint64_t n = 0;
	for (int i = 0; i < m->g; i++)
		n += cmb200_entries(m->dev[i]->eng);
	return n;
}

void
filemap_free(struct filemap *m)
{
	if (!m)
		return;
	if (m->ckpt_started) {
		pthread_mutex_lock(&m->ckpt_mu);
		m->ckpt_stop = 1;
		pthread_cond_broadcast(&m->ckpt_cv);
		pthread_mutex_unlock(&m->ckpt_mu);
		pthread_join(m->ckpt_thread, NULL);     /* a save in progress ends first */
	}
	for (int i = 0; i < m->g; i++) {
		struct fm_dev *d = m->dev[i];
		if (!d->wb_started)
			continue;
		pthread_mutex_lock(&d->wb_mu);
		d->wb_stop = 1;
		pthread_cond_broadcast(&d->wb_work);
		pthread_mutex_unlock(&d->wb_mu);
		pthread_join(d->wb_thread, NULL);      /* drains the ring first */
	}
	filemap_save(m, 0);                             /* the cache directory outlives the process */
	for (int i = 0; i < m->g; i++) {
		/* staging first, while every engine that allocated it is alive */
		struct fm_dev *d = m->dev[i];
		if (d->h_put)
			cmb200_host_free(d->h_put);
		if (d->d_first)
			cmb200_dev_free(m->dev[0]->eng, d->d_first);
		if (d->d_own)
			cmb200_dev_free(d->eng, d->d_own);
	}
	for (int i = 0; i < m->g; i++)
		fm_dev_free(m->dev[i]);
	pthread_mutex_destroy(&m->snap_mu);
	pthread_cond_destroy(&m->ckpt_cv);
	pthread_mutex_destroy(&m->ckpt_mu);
	pthread_mutex_destroy(&m->evict_mu);
	pthread_mutex_destroy(&m->init_mu);
	free(m);
}

/* Counting sort of n items by engine: order[] lists the items of engine 0, then of engine 1, ...,
 * each in array order; engine k's are order[start[k] .. start[k+1]).  own[i] = engine of item i. */
static void
group_by_owner(int g, size_t n, const int *own, size_t *order, size_t *start)
{
	for (int k = 0; k <= g; k++)
		start[k] = 0;
	for (size_t i = 0; i < n; i++)
		start[own[i] + 1]++;
	for (int k = 0; k < g; k++)
		start[k + 1] += start[k];
	size_t fill[MAX_DEVICES];
	for (int k = 0; k < g; k++)
		fill[k] = start[k];
	for (size_t i = 0; i < n; i++)
		order[fill[own[i]]++] = i;
}

static uint64_t
rand64(void)
{
	uint64_t r = 0;
	for (int b = 0; b < 64; b += 30)        /* filemap.c:271-274 */
		r = r * ((uint64_t)RAND_MAX + 1) + (uint64_t)rand();
	return r;
}

/* cmb200_sample of n draws: on engine `only`, or (only = NULL) each draw on engine cmb200_owner(r, G).
 * own_out[i] = the engine that answered draw i.  0 = sampled, -1 = an engine failed. */
static int
filemap_sample(struct filemap *m, struct fm_dev *only, size_t n, const uint64_t *draws, cmb200_addr *cand,
    uint64_t *ts, int32_t *ok, int *own_out)
{
	if (only) {
		for (size_t i = 0; i < n; i++)
			own_out[i] = only->index;
		return cmb200_sample(only->eng, n, draws, cand, ts, ok);
	}
	size_t *order = malloc(n * sizeof(size_t));
	uint64_t *r = malloc(n * sizeof(uint64_t)), *t = malloc(n * sizeof(uint64_t));
	cmb200_addr *a = malloc(n * sizeof(cmb200_addr));
	int32_t *o = malloc(n * sizeof(int32_t));
	size_t start[MAX_DEVICES + 1];
	int rc = (order && r && t && a && o) ? 0 : -1;
	if (rc == 0) {
		for (size_t i = 0; i < n; i++)
			own_out[i] = cmb200_owner(draws[i], m->g);
		group_by_owner(m->g, n, own_out, order, start);
		for (size_t j = 0; j < n; j++)
			r[j] = draws[order[j]];
		for (int k = 0; k < m->g && rc == 0; k++)
			if (start[k + 1] > start[k])
				rc = cmb200_sample(m->dev[k]->eng, start[k + 1] - start[k], r + start[k], a + start[k], t + start[k],
				    o + start[k]);
		for (size_t j = 0; rc == 0 && j < n; j++) {
			cand[order[j]] = a[j];
			ts[order[j]] = t[j];
			ok[order[j]] = o[j];
		}
	}
	free(order); free(r); free(t); free(a); free(o);
	return rc;
}

/* Unsets n victims, each on its engine own[i]. */
static void
filemap_unset_victims(struct filemap *m, size_t n, const cmb200_addr *victim, const int *own)
{
	cmb200_addr *v = malloc(n * sizeof(cmb200_addr));
	if (!v)
		return;
	for (int k = 0; k < m->g; k++) {
		size_t c = 0;
		for (size_t i = 0; i < n; i++)
			if (own[i] == k)
				v[c++] = victim[i];
		if (c)
			cmb200_unset_batch(m->dev[k]->eng, c, v);
	}
	free(v);
}

/* Retires up to `want` records, each the oldest of three random live ones (cachemap.c:17-45): on
 * engine `only` (arena pressure), or over the whole map (only = NULL, eviction by count; each draw on
 * the engine its r names).  Statistically the reference's policy; bitwise parity is undefined there
 * (wall-clock timestamps, rand()).  Returns how many entries actually went away. */
static uint64_t
filemap_evict_n(struct filemap *m, struct fm_dev *only, uint64_t want)
{
	uint64_t before = only ? cmb200_entries(only->eng) : filemap_count(m), gone = 0;
	while (gone < want && before > 0) {
		uint64_t need = want - gone;
		if (need > before)
			need = before;
		if (need > 4096)
			need = 4096;    /* per round; the loop continues */
		uint64_t *draws = malloc(3 * need * sizeof(uint64_t));
		uint64_t *ts = malloc(3 * need * sizeof(uint64_t));
		int32_t *ok = malloc(3 * need * sizeof(int32_t));
		int *own = malloc(3 * need * sizeof(int));
		cmb200_addr *cand = malloc(3 * need * sizeof(cmb200_addr));
		cmb200_addr *victim = malloc(need * sizeof(cmb200_addr));
		int *vown = malloc(need * sizeof(int));
		uint64_t nv = 0;
		if (draws && ts && ok && own && cand && victim && vown) {
			for (uint64_t i = 0; i < 3 * need; i++)
				draws[i] = rand64();
			if (filemap_sample(m, only, (size_t)(3 * need), draws, cand, ts, ok, own) == 0) {
				for (uint64_t i = 0; i < need; i++) {
					uint64_t a = ts[3 * i], b = ts[3 * i + 1], c = ts[3 * i + 2];
					int pick;
					if (a < b)
						pick = (a > c) ? 2 : 0;         /* cachemap.c:29-41 */
					else
						pick = (b > c) ? 2 : 1;
					if (ok[3 * i + pick] > 0) {
						victim[nv] = cand[3 * i + pick];
						vown[nv++] = own[3 * i + pick];
					}
				}
				if (nv)
					filemap_unset_victims(m, (size_t)nv, victim, vown);
			} else {
				fprintf(stderr, "cachemap_b200: eviction could not sample the store: %s\n", cmb200_last_error());
			}
		}
		free(draws); free(ts); free(ok); free(own); free(cand); free(victim); free(vown);
		/* two draws may have picked the same victim: count what really left the table */
		uint64_t after = only ? cmb200_entries(only->eng) : filemap_count(m);
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
filemap_promo_guard(struct fm_dev *d, size_t *n)
{
	*n = 0;
	if (!d->tier_promote)
		return NULL;
	pthread_mutex_lock(&d->promo_mu);
	const uint64_t cap = 4 * d->tier_promote;
	const size_t k = (size_t)(d->promo_guard_n < cap ? d->promo_guard_n : cap);
	cmb200_addr *g = k ? malloc(k * sizeof(cmb200_addr)) : NULL;
	if (g) {
		memcpy(g, d->promo_guard, k * sizeof(cmb200_addr));
		*n = k;
	}
	pthread_mutex_unlock(&d->promo_mu);
	if (g)
		qsort(g, *n, sizeof(cmb200_addr), addr_cmp);
	return g;
}

/* Moves up to `want` arena records of engine d to its host tier.  The candidates are drawn as
 * filemap_evict_n draws them (3 per record wanted, on this engine only) and go oldest first; keys
 * already in the tier, and keys promotion has just brought back (filemap_promo_guard), are passed
 * over, so a round goes on down its candidates until `want` have moved.  When few records are left in
 * the arena a round may find none: it draws again, up to 16 times in a row.  Returns how many moved. */
static uint64_t
filemap_demote_n(struct fm_dev *d, uint64_t want)
{
	uint64_t moved = 0;
	int idle = 0;
	size_t ng = 0;
	cmb200_addr *guard = filemap_promo_guard(d, &ng);
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
			for (uint64_t i = 0; i < nd; i++)
				draws[i] = rand64();
			if (cmb200_sample(d->eng, (size_t)nd, draws, cand, ts, ok) == 0) {
				uint64_t nv = 0;
				for (uint64_t i = 0; i < nd; i++)
					if (ok[i] > 0 && !(guard && bsearch(&cand[i], guard, ng, sizeof(cmb200_addr), addr_cmp)))
						old[nv++] = (struct aged){ ts[i], cand[i] };
				qsort(old, (size_t)nv, sizeof(struct aged), aged_cmp);
				for (uint64_t k = 0; k < nv && moved < want;) {
					uint64_t take = want - moved < nv - k ? want - moved : nv - k, got = 0;
					for (uint64_t j = 0; j < take; j++)
						victim[j] = old[k + j].a;
					if (cmb200_demote_batch(d->eng, (size_t)take, victim, &got) != 0) {
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

/* Before a batch of `incoming` puts: while entries + incoming > capacity over all engines, evict
 * (cachemap.c:17-45); loops until the count fits or nothing more can be retired.  Then the batch's
 * pages are reserved until they have landed in their engine (filemap_land_end): a batch that has made
 * its room but is not in its engine yet counts for every other batch's decision, so two flushers
 * neither evict for the same excess nor fill the same room.  The estimate (entries + reserved) can
 * count a batch twice, after it has landed and before its reservation is released; so when the
 * estimate says evict, the decision takes every engine's land_mu and counts again: no batch is
 * between the two then, and no more is evicted than the count needs. */
static void
filemap_evict(struct filemap *m, uint64_t incoming)
{
	if (!m->capacity)
		return;
	pthread_mutex_lock(&m->evict_mu);
	uint64_t entries = filemap_count(m) + __atomic_load_n(&m->reserved, __ATOMIC_RELAXED);
	if (entries + incoming > m->capacity && entries > 0) {
		for (int k = 0; k < m->g; k++)
			pthread_mutex_lock(&m->dev[k]->land_mu);
		for (;;) {
			entries = filemap_count(m) + __atomic_load_n(&m->reserved, __ATOMIC_RELAXED);
			if (entries + incoming <= m->capacity || entries == 0)
				break;
			uint64_t need = entries + incoming - m->capacity;
			if (incoming == 1)
				need = 1;       /* the reference evicts exactly one per put */
			if (filemap_evict_n(m, NULL, need) == 0 || incoming == 1)
				break;
		}
		for (int k = m->g - 1; k >= 0; k--)
			pthread_mutex_unlock(&m->dev[k]->land_mu);
	}
	__atomic_fetch_add(&m->reserved, incoming, __ATOMIC_RELAXED);
	pthread_mutex_unlock(&m->evict_mu);
}

/* Puts land in an engine under its land_mu, and their reservation (filemap_evict) is released before
 * land_mu is: a decision that holds every land_mu sees each batch either reserved or in its engine,
 * never both. */
static void
filemap_land_begin(struct fm_dev *d)
{
	pthread_mutex_lock(&d->land_mu);
}

static void
filemap_land_end(struct fm_dev *d, uint64_t pages)
{
	if (d->m->capacity)
		__atomic_fetch_sub(&d->m->reserved, pages, __ATOMIC_RELAXED);
	pthread_mutex_unlock(&d->land_mu);
}

/* The arena is a bump allocator; deleted and outgrown records stay behind as garbage until
 * cmb200_compact slides the live ones down.  When `incoming` worst-case records would not fit:
 * compact if that frees enough; otherwise the live data itself fills the arena (the store was
 * sized in pages, the arena is bytes).  With a host tier that can take what must move, the oldest
 * records are demoted to it and the arena compacted, so the store keeps `capacity` pages as the
 * reference's LMDB files do; otherwise evict by bytes as well and compact what that frees.
 * Only when even that fails does a put get dropped, as a full LMDB map drops it
 * (filemap.c:143-145,154-157).  may_evict = 0 (room for promotion): demotion and compaction only.
 * All of it happens on engine d, the one whose arena is full. */
static void
filemap_arena_room(struct fm_dev *d, uint64_t incoming, int may_evict)
{
	const uint64_t need = incoming * ((uint64_t)d->m->bsize + 1056);
	int evicted = 0;
	for (int attempt = 0; attempt < 6; attempt++) {
		cmb200_stats st;
		if (cmb200_get_stats(d->eng, &st) != 0)
			return;
		if (st.arena_used + need <= st.arena_bytes)
			return;
		const uint64_t free_b = st.arena_bytes - st.arena_used;
		if (st.arena_garbage > 0 && (free_b + st.arena_garbage >= need || evicted)) {
			uint64_t got = 0;
			if (cmb200_compact(d->eng, &got) != 0) {
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
		if (d->host_tier && cmb200_host_tier_stats(d->eng, &ht) == 0 && shortfall <= ht.bytes) {
			if (st.entries <= ht.records)
				return;         /* every live record is in the tier already: evicting frees no arena bytes */
			const uint64_t in_arena = st.entries - ht.records;
			const uint64_t avg = live / in_arena ? live / in_arena : 1;
			uint64_t victims = shortfall / avg + shortfall / avg / 8 + 16;
			if (victims > in_arena)
				victims = in_arena;
			if (filemap_demote_n(d, victims) == 0)
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
		if (filemap_evict_n(d->m, d, victims) == 0)
			return;
		evicted = 1;
	}
}

static void
filemap_check_arena(struct fm_dev *d, uint64_t incoming)
{
	filemap_arena_room(d, incoming, 1);
}

/* One promotion round (CMB200_TIER_PROMOTE = N): up to N addresses that gets answered from the host
 * tier since the last round, newest first, go back to the arena.  Room is made only by demoting the
 * oldest arena records and compacting, never by evicting; when that frees too little, the round
 * promotes what fits.  The addresses join the guard FIFO that demotion passes over. */
static void
filemap_promote_round(struct fm_dev *d)
{
	clock_gettime(CLOCK_MONOTONIC, &d->promo_last);
	size_t n = 0;
	if (cmb200_host_tier_hot(d->eng, (size_t)d->tier_promote, d->promo_hot, &n, NULL) != 0) {
		fprintf(stderr, "cachemap_b200: the host tier's hot log could not be read: %s\n", cmb200_last_error());
		return;
	}
	if (n == 0)
		return;
	filemap_arena_room(d, n, 0);
	uint64_t got = 0;
	if (cmb200_promote_batch(d->eng, n, d->promo_hot, &got) != 0) {
		fprintf(stderr, "cachemap_b200: promotion from the host tier failed: %s\n", cmb200_last_error());
		return;
	}
	pthread_mutex_lock(&d->promo_mu);
	const uint64_t cap = 4 * d->tier_promote;
	for (size_t i = 0; i < n; i++)
		d->promo_guard[d->promo_guard_n++ % cap] = d->promo_hot[i];
	pthread_mutex_unlock(&d->promo_mu);
}

/* A promotion round is due: the knob is on and PROMOTE_EVERY_MS have passed since the last one. */
static int
filemap_promote_due(struct fm_dev *d)
{
	if (!d->tier_promote)
		return 0;
	struct timespec now;
	clock_gettime(CLOCK_MONOTONIC, &now);
	const int64_t ms = (int64_t)(now.tv_sec - d->promo_last.tv_sec) * 1000 + (now.tv_nsec - d->promo_last.tv_nsec) / 1000000;
	return ms >= PROMOTE_EVERY_MS;
}

/* Before a batch of `incoming` puts into engine d: evict the map down to capacity (and reserve the
 * batch, see filemap_evict), then make sure d's arena has room (what eviction frees is garbage until
 * the arena is compacted).  The put follows between filemap_land_begin and filemap_land_end. */
static void
filemap_make_room(struct fm_dev *d, uint64_t incoming)
{
	filemap_evict(d->m, incoming);
	filemap_check_arena(d, incoming);
}

static void
timespec_add_ms(struct timespec *t, long ms)
{
	t->tv_nsec += ms * 1000000L;
	t->tv_sec += t->tv_nsec / 1000000000L;
	t->tv_nsec %= 1000000000L;
}

/* The flusher of one engine: takes the longest run of finished slots from the tail of its ring and
 * puts it into the engine as one batch (two calls when the run wraps around the ring). */
static void *
filemap_flusher(void *arg)
{
	struct fm_dev *d = arg;
	struct filemap *m = d->m;
	cmb200_addr *addr = malloc(FLUSH_MAX * sizeof(cmb200_addr));
	uint64_t *ts = malloc(FLUSH_MAX * sizeof(uint64_t));
	pthread_mutex_lock(&d->wb_mu);
	for (;;) {
		uint64_t count = 0;
		/* at most half the ring per batch: callers keep filling the other half while this one is on the GPU */
		uint64_t flush_cap = d->wb_n / 2 < FLUSH_MAX ? (d->wb_n / 2 ? d->wb_n / 2 : 1) : FLUSH_MAX;
		/* and at most this engine's share of the capacity: the batches of all flushers in flight at once
		 * then fit the store together */
		if (m->capacity && flush_cap > m->capacity / (uint64_t)m->g)
			flush_cap = m->capacity / (uint64_t)m->g ? m->capacity / (uint64_t)m->g : 1;
		while (d->wb_tail + count < d->wb_head && count < flush_cap &&
		    d->wb_slot[(d->wb_tail + count) % d->wb_n].state == WB_READY)
			count++;
		if (count == 0) {
			if (d->wb_stop && d->wb_tail == d->wb_head)
				break;
			if (filemap_promote_due(d)) {
				pthread_mutex_unlock(&d->wb_mu);
				filemap_promote_round(d);
				pthread_mutex_lock(&d->wb_mu);
				continue;
			}
			if (d->tier_promote) {
				/* woken for the next promotion round at the latest */
				struct timespec until;
				clock_gettime(CLOCK_REALTIME, &until);
				timespec_add_ms(&until, PROMOTE_EVERY_MS);
				d->wb_flusher_asleep = 1;
				pthread_cond_timedwait(&d->wb_work, &d->wb_mu, &until);
				d->wb_flusher_asleep = 0;
			} else {
				d->wb_flusher_asleep = 1;
				pthread_cond_wait(&d->wb_work, &d->wb_mu);
				d->wb_flusher_asleep = 0;
			}
			continue;
		}
		for (uint64_t i = 0; i < count; i++) {
			struct wb_slot *s = &d->wb_slot[(d->wb_tail + i) % d->wb_n];
			s->state = WB_FLUSHING;
			addr[i] = s->addr;
			ts[i] = s->ts;
		}
		const uint64_t first = d->wb_tail % d->wb_n;
		pthread_mutex_unlock(&d->wb_mu);

		if (addr && ts) {
			filemap_make_room(d, count);
			filemap_land_begin(d);
			uint64_t run1 = count < d->wb_n - first ? count : d->wb_n - first;
			cmb200_put_batch(d->eng, (size_t)run1, addr, NULL, d->wb_pages + first * (size_t)m->bsize, ts, NULL);
			if (run1 < count)
				cmb200_put_batch(d->eng, (size_t)(count - run1), addr + run1, NULL, d->wb_pages, ts + run1, NULL);
			filemap_land_end(d, count);
		}

		pthread_mutex_lock(&d->wb_mu);
		__atomic_fetch_add(&m->puts_seen, count, __ATOMIC_RELAXED);
		for (uint64_t i = 0; i < count; i++)
			d->wb_slot[(d->wb_tail + i) % d->wb_n].state = WB_FREE;
		d->wb_tail += count;
		pthread_cond_broadcast(&d->wb_space);
		pthread_cond_broadcast(&d->wb_idle);            /* waiters compare wb_tail with their own target */
		if (filemap_promote_due(d)) {
			pthread_mutex_unlock(&d->wb_mu);
			filemap_promote_round(d);
			pthread_mutex_lock(&d->wb_mu);
		}
	}
	pthread_mutex_unlock(&d->wb_mu);
	free(addr);
	free(ts);
	return NULL;
}

/* The newest page of `key` (the store key of `addr`) still in its engine's ring decides, as it will
 * once it has landed: CMB200_HIT when it is of `addr` (*page = a malloc()ed copy, or dst; NULL if malloc fails),
 * CMB200_BAD_ENTRY when it is of another address with the same key (that put replaces the record of
 * `addr`, filemap.c:236-240), CMB200_MISS when the ring holds no page of the key: ask the engine. */
static int32_t
filemap_ring_lookup(struct fm_dev *d, const cmb200_addr *addr, uint64_t key, void *dst, void **page)
{
	int32_t st = CMB200_MISS;
	*page = NULL;
	if (!d->wb_n)
		return st;
	const size_t bsize = (size_t)d->m->bsize;
	pthread_mutex_lock(&d->wb_mu);
	for (uint64_t s = d->wb_head; s > d->wb_tail; s--) {
		struct wb_slot *w = &d->wb_slot[(s - 1) % d->wb_n];
		if (w->state < WB_READY || w->key != key)
			continue;
		if (w->addr.u != addr->u || w->addr.l != addr->l) {
			st = CMB200_BAD_ENTRY;
			break;
		}
		st = CMB200_HIT;
		*page = dst ? dst : malloc(bsize);
		if (*page)
			memcpy(*page, d->wb_pages + ((s - 1) % d->wb_n) * bsize, bsize);
		break;
	}
	pthread_mutex_unlock(&d->wb_mu);
	return st;
}

/* Combining queue of the single-page calls (cachemap_get / filemap_unset from FUSE worker threads),
 * one per engine.
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
 * held and d->launching set; returns with q_mu held. */
static void
filemap_lead(struct fm_dev *d, int ls)
{
	struct fm_req *batch[COMBINE_MAX];
	cmb200_addr addr[COMBINE_MAX];
	int idx[COMBINE_MAX];
	int nb = 0, k;

	while (d->q_head && nb < COMBINE_MAX) {
		batch[nb++] = d->q_head;
		d->q_head = d->q_head->next;
	}
	if (!d->q_head)
		d->q_tail = NULL;
	__atomic_fetch_sub(&d->q_len, nb, __ATOMIC_RELAXED);
	pthread_mutex_unlock(&d->q_mu);

	k = 0;
	for (int i = 0; i < nb; i++)
		if (batch[i]->kind == REQ_UNSET)
			addr[k++] = batch[i]->addr;
	if (k)
		cmb200_unset_batch(d->eng, (size_t)k, addr);    /* unsets first: they change the table the gets read by key */

	k = 0;
	for (int i = 0; i < nb; i++) {
		if (batch[i]->kind != REQ_GET)
			continue;
		addr[k] = batch[i]->addr;
		idx[k] = i;
		k++;
	}
	uint8_t *stage = d->h_stage + (size_t)ls * COMBINE_MAX * (size_t)d->m->bsize;
	const volatile int32_t *answers = d->sync_status[ls];
	d->ticket[ls].lane = -1;
	if (k) {
		/* the fused small-batch get: one kernel on a stream of its own, pages land in the page-locked
		 * stage buffer directly; page sizes it does not serve (> 128 KiB) take the two-kernel batch path,
		 * synchronously */
		int rc = cmb200_get_small_begin(d->eng, (size_t)k, addr, stage, &d->ticket[ls]);
		if (rc == 0) {
			answers = d->ticket[ls].status;
		} else {
			d->ticket[ls].lane = -1;
			if (rc == -2)
				rc = cmb200_get_batch(d->eng, (size_t)k, addr, NULL, stage, d->sync_status[ls]);
			if (rc != 0)
				for (int j = 0; j < k; j++)
					d->sync_status[ls][j] = CMB200_MISS;
		}
	}

	pthread_mutex_lock(&d->q_mu);
	__atomic_store_n(&d->batch_left[ls], nb, __ATOMIC_RELEASE);
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

/* Queues `count` requests (an array) on engine d.  filemap_await must follow with the same array. */
static void
filemap_enqueue(struct fm_dev *d, struct fm_req *reqs, int count)
{
	for (int i = 0; i < count; i++) {
		reqs[i].status = NULL;
		reqs[i].slot = -1;
		reqs[i].pos = 0;
		reqs[i].next = i + 1 < count ? &reqs[i + 1] : NULL;
	}
	while (sem_wait(&d->q_door) != 0)
		;
	pthread_mutex_lock(&d->q_mu);
	if (d->q_tail)
		d->q_tail->next = &reqs[0];
	else
		d->q_head = &reqs[0];
	d->q_tail = &reqs[count - 1];
	__atomic_fetch_add(&d->q_len, count, __ATOMIC_RELAXED);
	pthread_mutex_unlock(&d->q_mu);
}

/* Returns when all `count` requests queued by filemap_enqueue have been answered.  A requester
 * takes q_mu once to queue; after that it only takes it again to launch a batch itself or to sleep
 * when every slot is busy — watching for its launch and for its answer needs no lock. */
static void
filemap_await(struct fm_dev *d, struct fm_req *reqs, int count)
{
	for (int i = 0; i < count; i++) {
		struct fm_req *r = &reqs[i];
		const volatile int32_t *answer;
		unsigned waited = 0;
		while (!(answer = __atomic_load_n(&r->status, __ATOMIC_ACQUIRE))) {
			/* Watch without the lock while somebody is inside a launch (microseconds: it either has this
			 * request with it or leaves it to the next launch), while every slot is busy, and — for a
			 * short while — when a launch now would carry very few requests into one of the last free
			 * slots: with many callers the slots are what runs out, and batches of 1 use them up. */
			const int busy = __atomic_load_n(&d->busy_slots, __ATOMIC_RELAXED);
			if (__atomic_load_n(&d->launching, __ATOMIC_ACQUIRE) || busy >= LEADERS ||
			    (busy >= LEADERS / 2 && waited < 256u && 4 * __atomic_load_n(&d->q_len, __ATOMIC_RELAXED) < busy)) {
#if defined(__x86_64__)
				__builtin_ia32_pause();
#endif
				if ((++waited & 1023u) == 0u)
					sched_yield();
				continue;
			}
			pthread_mutex_lock(&d->q_mu);
			if (!r->status && !__atomic_load_n(&d->launching, __ATOMIC_RELAXED)) {
				int ls = -1;
				for (int k = 0; k < LEADERS; k++)
					if (!d->leader_busy[k]) { ls = k; break; }
				if (ls >= 0) {
					__atomic_store_n(&d->launching, 1, __ATOMIC_RELAXED);  /* (read by watchers that hold no lock) */
					d->leader_busy[ls] = 1;
					__atomic_fetch_add(&d->busy_slots, 1, __ATOMIC_RELAXED);
					filemap_lead(d, ls);                    /* (drops and retakes q_mu around the launch) */
					__atomic_store_n(&d->launching, 0, __ATOMIC_RELEASE);
				}
			}
			pthread_mutex_unlock(&d->q_mu);
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
				const size_t bsize = (size_t)d->m->bsize;
				r->out = r->dst ? r->dst : malloc(bsize);    /* filemap.c:242 */
				if (r->out)
					memcpy(r->out, d->h_stage + ((size_t)ls * COMBINE_MAX + (size_t)r->pos) * bsize, bsize);
			} else if (st == CMB200_BAD_ENTRY) {
				r->bad_entry = 1;
			}
		}

		if (__atomic_sub_fetch(&d->batch_left[ls], 1, __ATOMIC_ACQ_REL) == 0) {
			/* last one out: every status word of the launch has been seen answered, so ending it does
			 * not wait; then the slot and its stage buffer are free again */
			if (d->ticket[ls].lane >= 0)
				cmb200_get_small_end(d->eng, &d->ticket[ls], NULL);
			pthread_mutex_lock(&d->q_mu);
			d->leader_busy[ls] = 0;
			__atomic_fetch_sub(&d->busy_slots, 1, __ATOMIC_RELEASE);
			pthread_mutex_unlock(&d->q_mu);
		}
	}
	sem_post(&d->q_door);
}

static void
filemap_submit(struct fm_dev *d, struct fm_req *req)
{
	filemap_enqueue(d, req, 1);
	filemap_await(d, req, 1);
}

void
filemap_set(struct filemap *m, uint128_t *key, void *value, uint64_t attr)
{
	if (!filemap_engine_ready(m))
		return;
	cmb200_addr a = { key->u, key->l };
	const uint64_t k = addr_key(&a);
	struct fm_dev *d = m->dev[cmb200_owner(k, m->g)];
	if (!d->wb_n) {                         /* write-behind disabled: one synchronous GPU put */
		filemap_make_room(d, 1);
		filemap_land_begin(d);
		cmb200_put_batch(d->eng, 1, &a, NULL, value, &attr, NULL);
		filemap_land_end(d, 1);
		__atomic_fetch_add(&m->puts_seen, 1, __ATOMIC_RELAXED);
		return;
	}
	pthread_mutex_lock(&d->wb_mu);
	while (d->wb_head - d->wb_tail == d->wb_n)
		pthread_cond_wait(&d->wb_space, &d->wb_mu);     /* back-pressure: the ring is full */
	const uint64_t s = d->wb_head++;
	struct wb_slot *w = &d->wb_slot[s % d->wb_n];
	w->addr = a;
	w->key = k;
	w->ts = attr;
	w->state = WB_FILLING;
	pthread_mutex_unlock(&d->wb_mu);
	memcpy(d->wb_pages + (s % d->wb_n) * (size_t)m->bsize, value, (size_t)m->bsize);
	pthread_mutex_lock(&d->wb_mu);
	w->state = WB_READY;
	if (d->wb_flusher_asleep)               /* a busy flusher finds the page by itself when it comes back: no wake-up call per put */
		pthread_cond_signal(&d->wb_work);
	pthread_mutex_unlock(&d->wb_mu);
}

void
filemap_unset(struct filemap *m, uint128_t *key)
{
	if (!filemap_engine_ready(m))
		return;
	struct fm_req r;
	memset(&r, 0, sizeof(r));
	r.kind = REQ_UNSET;
	r.addr.u = key->u;
	r.addr.l = key->l;
	struct fm_dev *d = filemap_owner(m, &r.addr);
	fm_dev_drain(d);
	filemap_submit(d, &r);
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
	const uint64_t k = addr_key(&r.addr);
	struct fm_dev *d = m->dev[cmb200_owner(k, m->g)];
	/* a page accepted by filemap_set but not flushed yet is served from the ring; a slot leaves
	 * the ring only after the GPU put of its batch has completed, so nothing falls between */
	void *page;
	const int32_t st = filemap_ring_lookup(d, &r.addr, k, NULL, &page);
	if (st == CMB200_HIT)
		return page;
	if (st == CMB200_BAD_ENTRY) {
		printf("bad entry\n");          /* filemap.c:237 */
		return NULL;
	}
	filemap_submit(d, &r);
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
	/* filemap.c:271-274: a 64-bit draw built from rand(), sampled on the engine it names */
	uint64_t r = rand64();
	cmb200_addr a;
	int32_t ok = 0;
	if (cmb200_sample(m->dev[cmb200_owner(r, m->g)]->eng, 1, &r, &a, ts, &ok) != 0 || !ok)
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
	return filemap_count(m);
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
	filemap_free(cm->pages);                /* drains the write-behind rings (cachemap.c:218-232) */
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
	int *own;               /* engine of each page (an invalid address goes to engine 0, which skips it) */
};

static int
batch_keys_build(struct cachemap *cm, uint64_t n, const uint64_t *offset, const uint64_t *nhid,
    const uint32_t *genid, int want_ts, struct batch_keys *bk)
{
	bk->addr = malloc((size_t)n * sizeof(cmb200_addr));
	bk->valid = malloc((size_t)n);
	bk->ts = want_ts ? malloc((size_t)n * 8) : NULL;
	bk->own = malloc((size_t)n * sizeof(int));
	if (!bk->addr || !bk->valid || (want_ts && !bk->ts) || !bk->own) {
		free(bk->addr); free(bk->valid); free(bk->ts); free(bk->own);
		return -1;
	}
	uint64_t ts = want_ts ? now_ns() : 0;
	for (uint64_t i = 0; i < n; i++) {
		bk->valid[i] = compose_addr(cm, offset[i], nhid[i], genid ? genid[i] : 0, &bk->addr[i]) == 0;
		if (!bk->valid[i])
			memset(&bk->addr[i], 0, sizeof(cmb200_addr));
		bk->own[i] = bk->valid[i] ? filemap_owner(cm->pages, &bk->addr[i])->index : 0;
		if (want_ts)
			bk->ts[i] = ts;
	}
	return 0;
}

static void
batch_keys_free(struct batch_keys *bk)
{
	free(bk->addr); free(bk->valid); free(bk->ts); free(bk->own);
}

/* One engine's share of a batch call when the batch spans engines: its pages' keys gathered, and
 * where its pages are in the caller's buffer.  The shares of a call run concurrently, one thread per
 * engine, each through its engine's reusable staging buffers (struct fm_dev, stage_mu). */
struct batch_part {
	struct filemap *m;
	struct fm_dev *d;
	size_t c;
	cmb200_addr *addr;
	uint8_t *valid;
	uint64_t *ts;
	uint32_t *idx;          /* page of the caller's buffer of each */
	int32_t *status;        /* get: status of each */
	const uint8_t *src;     /* put: the caller's pages (host, or the first engine's GPU) */
	uint8_t *dst;           /* get: the caller's output (host, or the first engine's GPU) */
	int on_dev;
	pthread_t th;
};

/* The pages order[0..c) of the batch keys, from position `at` on. */
static int
batch_part_gather(struct batch_part *p, const struct batch_keys *bk, const size_t *order, size_t c, uint64_t at)
{
	p->c = c;
	p->addr = malloc(c * sizeof(cmb200_addr));
	p->valid = malloc(c);
	p->ts = bk->ts ? malloc(c * 8) : NULL;
	p->idx = malloc(c * sizeof(uint32_t));
	p->status = bk->ts ? NULL : malloc(c * sizeof(int32_t));
	if (!p->addr || !p->valid || (bk->ts && !p->ts) || !p->idx || (!bk->ts && !p->status))
		return -1;
	for (size_t j = 0; j < c; j++) {
		p->addr[j] = bk->addr[at + order[j]];
		p->valid[j] = bk->valid[at + order[j]];
		if (p->ts)
			p->ts[j] = bk->ts[at + order[j]];
		p->idx[j] = (uint32_t)order[j];
	}
	return 0;
}

static void
batch_part_free(struct batch_part *p)
{
	free(p->addr); free(p->valid); free(p->ts); free(p->idx); free(p->status);
}

/* Host pages a share moves per engine call: 64 MiB of page-locked staging per engine, at most 4096
 * pages (the engine's sub-batch). */
static size_t
stage_pages(const struct filemap *m)
{
	size_t k = ((size_t)64 << 20) / (size_t)m->bsize;
	return k < 1 ? 1 : k > 4096 ? 4096 : k;
}

/* d->h_put, allocated on first use (stage_mu held). */
static uint8_t *
stage_host(struct fm_dev *d)
{
	if (!d->h_put)
		d->h_put = cmb200_host_alloc(stage_pages(d->m) * (size_t)d->m->bsize);
	return d->h_put;
}

/* A device buffer of at least `bytes` on engine e's GPU in *p, kept in the share's engine and grown as
 * needed (stage_mu held): no allocation, and no device-wide cudaFree, per call. */
static void *
stage_dev(cmb200_engine *e, void **p, size_t *cap, size_t bytes)
{
	if (*p && *cap >= bytes)
		return *p;
	if (*p)
		cmb200_dev_free(e, *p);
	*p = cmb200_dev_alloc(e, bytes);
	*cap = *p ? bytes : 0;
	return *p;
}

/* Device-resident pages (the _dev calls) are on the first engine's GPU.  Engine k's pages cross to
 * its GPU in one contiguous buffer and one peer copy: gathered on the first GPU by k_move_pages
 * (cmb200_move_pages), then copied; nothing is copied when engine k is on the first GPU. */
static int
same_gpu(struct filemap *m, int k)
{
	return m->dev[k]->device == m->dev[0]->device;
}

static int
dev_calls_present(void)
{
	return cmb200_move_pages && cmb200_copy_peer && cmb200_dev_alloc && cmb200_dev_free;
}

/* One engine's share of a put: host pages are copied into the engine's page-locked staging buffer in
 * runs of stage_pages(); device pages are gathered on the first GPU by k_move_pages and cross in one
 * peer copy. */
static void *
put_part(void *arg)
{
	struct batch_part *p = arg;
	struct filemap *m = p->m;
	struct fm_dev *d = p->d, *d0 = m->dev[0];
	const size_t bsize = (size_t)m->bsize, bytes = p->c * bsize;
	int rc = -1;
	pthread_mutex_lock(&d->stage_mu);
	filemap_check_arena(d, p->c);
	filemap_land_begin(d);
	if (!p->on_dev) {
		uint8_t *h = stage_host(d);
		const size_t sp = stage_pages(m);
		rc = h ? 0 : -1;
		for (size_t at = 0; rc == 0 && at < p->c; at += sp) {
			const size_t k = p->c - at < sp ? p->c - at : sp;
			for (size_t j = 0; j < k; j++)
				memcpy(h + j * bsize, p->src + (size_t)p->idx[at + j] * bsize, bsize);
			/* back when the pages have crossed to the GPU: the buffer is free for the next run */
			uint64_t ticket;
			rc = cmb200_put_batch_async(d->eng, k, p->addr + at, p->valid + at, h, p->ts + at, NULL, &ticket);
		}
	} else if (dev_calls_present()) {
		void *g0 = stage_dev(d0->eng, &d->d_first, &d->d_first_bytes, bytes), *buf = g0;
		rc = g0 ? cmb200_move_pages(d0->eng, p->c, g0, NULL, p->src, p->idx) : -1;
		if (rc == 0 && !same_gpu(m, d->index)) {
			buf = stage_dev(d->eng, &d->d_own, &d->d_own_bytes, bytes);
			rc = buf ? cmb200_copy_peer(d->eng, buf, d0->eng, g0, bytes) : -1;
		}
		if (rc == 0)
			rc = cmb200_put_batch_dev(d->eng, p->c, p->addr, p->valid, buf, p->ts, NULL);
	}
	filemap_land_end(d, p->c);
	pthread_mutex_unlock(&d->stage_mu);
	if (rc != 0)
		fprintf(stderr, "cachemap_b200: %zu pages not stored on engine %d: %s\n", p->c, d->index, cmb200_last_error());
	return NULL;
}

/* One engine's share of a get: decoded into the engine's staging buffer (host: in runs of
 * stage_pages(); device: on the engine's GPU, then one peer copy to the first GPU), and the hits
 * scattered to their places in the caller's output; a miss leaves its page untouched.  p->status
 * stays CMB200_MISS where the engine could not answer. */
static void *
get_part(void *arg)
{
	struct batch_part *p = arg;
	struct filemap *m = p->m;
	struct fm_dev *d = p->d, *d0 = m->dev[0];
	const size_t bsize = (size_t)m->bsize, bytes = p->c * bsize;
	for (size_t j = 0; j < p->c; j++)
		p->status[j] = CMB200_MISS;
	pthread_mutex_lock(&d->stage_mu);
	if (!p->on_dev) {
		uint8_t *h = stage_host(d);
		const size_t sp = stage_pages(m);
		for (size_t at = 0; h && at < p->c; at += sp) {
			const size_t k = p->c - at < sp ? p->c - at : sp;
			if (cmb200_get_batch(d->eng, k, p->addr + at, p->valid + at, h, p->status + at) != 0) {
				for (size_t j = 0; j < k; j++)
					p->status[at + j] = CMB200_MISS;
				continue;
			}
			for (size_t j = 0; j < k; j++)
				if (p->status[at + j] == CMB200_HIT)
					memcpy(p->dst + (size_t)p->idx[at + j] * bsize, h + j * bsize, bsize);
		}
	} else if (dev_calls_present()) {
		uint32_t *src = malloc(p->c * sizeof(uint32_t)), *dst = malloc(p->c * sizeof(uint32_t));
		void *gk = stage_dev(d->eng, &d->d_own, &d->d_own_bytes, bytes), *buf = gk;
		int rc = gk && src && dst ? cmb200_get_batch_dev(d->eng, p->c, p->addr, p->valid, gk, p->status) : -1;
		if (rc == 0 && !same_gpu(m, d->index)) {
			buf = stage_dev(d0->eng, &d->d_first, &d->d_first_bytes, bytes);
			rc = buf ? cmb200_copy_peer(d0->eng, buf, d->eng, gk, bytes) : -1;
		}
		if (rc == 0) {
			size_t h = 0;
			for (size_t j = 0; j < p->c; j++)
				if (p->status[j] == CMB200_HIT) {
					src[h] = (uint32_t)j;
					dst[h++] = p->idx[j];
				}
			rc = cmb200_move_pages(d0->eng, h, p->dst, dst, buf, src);
		}
		if (rc != 0)
			for (size_t j = 0; j < p->c; j++)
				p->status[j] = CMB200_MISS;
		free(src); free(dst);
	}
	pthread_mutex_unlock(&d->stage_mu);
	return NULL;
}

/* Runs the np shares of a call at once: one thread each, the first on the caller's thread. */
static void
run_parts(struct batch_part *parts, int np, void *(*fn)(void *))
{
	int started[MAX_DEVICES];
	for (int i = 1; i < np; i++)
		started[i] = pthread_create(&parts[i].th, NULL, fn, &parts[i]) == 0;
	if (np > 0)
		fn(&parts[0]);
	for (int i = 1; i < np; i++) {
		if (started[i])
			pthread_join(parts[i].th, NULL);
		else
			fn(&parts[i]);
	}
}

static void
put_batch_common(struct cachemap *cm, uint64_t n, const uint64_t *offset, const uint64_t *nhid,
    const uint32_t *genid, const void *pages, int on_dev)
{
	struct filemap *fm = cm->pages;
	struct batch_keys bk;
	if (n == 0 || !filemap_engine_ready(fm))
		return;
	if (batch_keys_build(cm, n, offset, nhid, genid, 1, &bk) != 0)
		return;
	size_t *order = malloc((size_t)n * sizeof(size_t));
	if (!order) {
		batch_keys_free(&bk);
		return;
	}
	filemap_drain(fm);                      /* earlier single puts land first */
	__atomic_fetch_add(&fm->puts_seen, n, __ATOMIC_RELAXED);
	/* One GPU batch per engine when the store has room for all of it; at capacity the batch goes in
	 * slices with eviction before each, so that entries never run past capacity by more than a slice
	 * (the reference evicts before every single put, cachemap.c:186-197). */
	uint64_t slice = n;
	if (cm->capacity && filemap_count(fm) + n > cm->capacity) {
		slice = cm->capacity / 4;
		if (slice > 4096)
			slice = 4096;
		if (slice < 1)
			slice = 1;
	}
	const size_t bsize = (size_t)fm->bsize;
	for (uint64_t at = 0; at < n; at += slice) {
		const uint64_t m = n - at < slice ? n - at : slice;
		const uint8_t *pg = (const uint8_t *)pages + at * bsize;
		size_t start[MAX_DEVICES + 1];
		group_by_owner(fm->g, (size_t)m, bk.own + at, order, start);
		filemap_evict(fm, m);
		struct batch_part parts[MAX_DEVICES];
		int np = 0;
		for (int k = 0; k < fm->g; k++) {
			const size_t c = start[k + 1] - start[k];
			if (c == 0)
				continue;
			struct fm_dev *d = fm->dev[k];
			if (c == m && (k == 0 || !on_dev)) {
				/* the whole slice is this engine's (always so with one engine): the caller's arrays as they are */
				filemap_check_arena(d, c);
				filemap_land_begin(d);
				if (on_dev)
					cmb200_put_batch_dev(d->eng, (size_t)m, bk.addr + at, bk.valid + at, pg, bk.ts + at, NULL);
				else {
					/* write-behind like cachemap_put: back when the pages have crossed to the GPU and the
					 * caller may reuse them; whatever is called next is ordered after the encode */
					uint64_t ticket;
					cmb200_put_batch_async(d->eng, (size_t)m, bk.addr + at, bk.valid + at, pg, bk.ts + at, NULL, &ticket);
				}
				filemap_land_end(d, m);
				continue;
			}
			struct batch_part *p = &parts[np];
			memset(p, 0, sizeof(*p));
			p->m = fm;
			p->d = d;
			p->src = pg;
			p->on_dev = on_dev;
			if (batch_part_gather(p, &bk, order + start[k], c, at) != 0) {
				batch_part_free(p);
				filemap_land_begin(d);
				filemap_land_end(d, c);         /* (what a share cannot store gives its reservation back) */
				continue;
			}
			np++;
		}
		run_parts(parts, np, put_part);
		for (int i = 0; i < np; i++)
			batch_part_free(&parts[i]);
	}
	free(order);
	batch_keys_free(&bk);
}

static void
get_batch_common(struct cachemap *cm, uint64_t n, const uint64_t *offset, const uint64_t *nhid,
    const uint32_t *genid, void *pages_out, uint8_t *hit_out, int on_dev)
{
	struct filemap *fm = cm->pages;
	struct batch_keys bk;
	memset(hit_out, 0, (size_t)n);
	if (n == 0 || !filemap_engine_ready(fm))
		return;
	if (batch_keys_build(cm, n, offset, nhid, genid, 0, &bk) != 0)
		return;
	filemap_drain(fm);
	int32_t *status = malloc((size_t)n * 4);
	size_t *order = malloc((size_t)n * sizeof(size_t));
	size_t start[MAX_DEVICES + 1];
	struct batch_part parts[MAX_DEVICES];
	int np = 0;
	if (status && order) {
		for (uint64_t i = 0; i < n; i++)
			status[i] = CMB200_MISS;        /* what an engine that fails leaves: no hit, no bad entry */
		group_by_owner(fm->g, (size_t)n, bk.own, order, start);
		for (int k = 0; k < fm->g; k++) {
			const size_t c = start[k + 1] - start[k];
			if (c == 0)
				continue;
			struct fm_dev *d = fm->dev[k];
			if (c == n && (k == 0 || !on_dev)) {
				/* all of it on this engine (always so with one engine): straight into the caller's arrays */
				int rc = on_dev ? cmb200_get_batch_dev(d->eng, (size_t)n, bk.addr, bk.valid, pages_out, status)
				                : cmb200_get_batch(d->eng, (size_t)n, bk.addr, bk.valid, pages_out, status);
				if (rc != 0)
					for (uint64_t i = 0; i < n; i++)
						status[i] = CMB200_MISS;
				continue;
			}
			struct batch_part *p = &parts[np];
			memset(p, 0, sizeof(*p));
			p->m = fm;
			p->d = d;
			p->dst = pages_out;
			p->on_dev = on_dev;
			if (batch_part_gather(p, &bk, order + start[k], c, 0) != 0) {
				batch_part_free(p);
				continue;
			}
			np++;
		}
		run_parts(parts, np, get_part);
		for (int i = 0; i < np; i++) {
			for (size_t j = 0; j < parts[i].c; j++)
				status[parts[i].idx[j]] = parts[i].status[j];
			batch_part_free(&parts[i]);
		}
	}
	uint64_t rq = 0, ht = 0;
	for (uint64_t i = 0; i < n; i++) {
		if (!bk.valid[i])
			continue;                       /* cachemap.c:173-174: not a request */
		rq++;
		if (status && status[i] == CMB200_HIT) {
			hit_out[i] = 1;
			ht++;
		} else if (status && status[i] == CMB200_BAD_ENTRY) {
			printf("bad entry\n");
		}
	}
	__atomic_fetch_add(&cm->requests, rq, __ATOMIC_RELAXED);
	__atomic_fetch_add(&cm->hits, ht, __ATOMIC_RELAXED);
	free(status);
	free(order);
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

/* Where page i of n goes in a read of the pages from a page-aligned offset: into first (i == 0) or last
 * (i == n - 1) when those are given, else into out, which holds the read from `skew` bytes into page 0. */
static uint8_t *
page_dst(uint64_t i, uint64_t n, int pshift, uint8_t *out, size_t skew, uint8_t *first, uint8_t *last)
{
	if (i == 0 && first)
		return first;
	if (i == n - 1 && last)
		return last;
	return out + ((i << pshift) - skew);
}

/* The page loop of edgefs_read over n >= 1 pages from the page-aligned offset off, each page to its
 * page_dst.  1 when every page hits; requests / hits advance as the reference's loop advances them. */
static int
read_pages(struct cachemap *cm, uint64_t nhid_small, uint32_t genid, uint64_t off, uint64_t n, uint8_t *out,
    size_t skew, uint8_t *first, uint8_t *last)
{
	struct filemap *fm = cm->pages;
	const int pshift = fm->pshift;
	if (!filemap_engine_ready(fm))
		return 0;
	struct fm_req *reqs = calloc((size_t)n, sizeof(*reqs));
	cmb200_addr *addr = malloc((size_t)n * sizeof(cmb200_addr));
	int *own = malloc((size_t)n * sizeof(int));
	size_t *order = malloc((size_t)n * sizeof(size_t));
	uint8_t *state = calloc((size_t)n, 1);          /* 0 miss, 1 hit, 2 invalid address, 3 asked of an engine,
	                                                 * 4 bad entry in a ring */
	if (!reqs || !addr || !own || !order || !state) {
		free(reqs); free(addr); free(own); free(order); free(state);
		return 0;
	}
	/* pages still in a write-behind ring are served from it; the rest go to their engines, one chain
	 * of requests per engine (one batch unless the chain is longer than COMBINE_MAX) */
	size_t ask = 0;
	for (uint64_t i = 0; i < n; i++) {
		uint8_t *dst = page_dst(i, n, pshift, out, skew, first, last);
		if (compose_addr(cm, off + (i << pshift), nhid_small, genid, &addr[ask]) != 0) {
			state[i] = 2;
			continue;
		}
		const uint64_t k = addr_key(&addr[ask]);
		struct fm_dev *d = fm->dev[cmb200_owner(k, fm->g)];
		void *page;
		const int32_t rs = filemap_ring_lookup(d, &addr[ask], k, dst, &page);
		if (rs != CMB200_MISS) {
			state[i] = rs == CMB200_HIT ? 1 : 4;
			continue;
		}
		state[i] = 3;
		own[ask] = d->index;
		order[ask] = i;         /* (page of each asked request, until grouped below) */
		ask++;
	}
	size_t start[MAX_DEVICES + 1], *page_of = malloc((ask ? ask : 1) * sizeof(size_t));
	if (!page_of) {
		free(reqs); free(addr); free(own); free(order); free(state);
		return 0;
	}
	memcpy(page_of, order, ask * sizeof(size_t));
	group_by_owner(fm->g, ask, own, order, start);
	for (size_t j = 0; j < ask; j++) {
		reqs[j].kind = REQ_GET;
		reqs[j].addr = addr[order[j]];
		reqs[j].dst = page_dst(page_of[order[j]], n, pshift, out, skew, first, last);
	}
	/* every engine's chain is queued before any is waited for, in engine order (so that two callers
	 * never hold the door of one engine while they wait for the other's) */
	for (int k = 0; k < fm->g; k++)
		if (start[k + 1] > start[k])
			filemap_enqueue(fm->dev[k], reqs + start[k], (int)(start[k + 1] - start[k]));
	for (int k = 0; k < fm->g; k++)
		if (start[k + 1] > start[k])
			filemap_await(fm->dev[k], reqs + start[k], (int)(start[k + 1] - start[k]));
	for (size_t j = 0; j < ask; j++)
		state[page_of[order[j]]] = reqs[j].out ? 1 : 0;
	/* counters as the reference's loop leaves them, in page order whatever engine answered which page:
	 * it stops at the first page that is not a hit; an invalid address returns NULL without counting a
	 * request (cachemap.c:173-174) */
	uint64_t rq = 0, ht = 0, i = 0;
	for (; i < n; i++) {
		if (state[i] == 2)
			break;
		rq++;
		if (state[i] != 1)
			break;
		ht++;
	}
	for (size_t j = 0; j < ask; j++)
		if (reqs[j].bad_entry && (uint64_t)page_of[order[j]] <= i)
			printf("bad entry\n");                  /* filemap.c:237 */
	if (i < n && state[i] == 4)
		printf("bad entry\n");
	__atomic_fetch_add(&cm->requests, rq, __ATOMIC_RELAXED);
	__atomic_fetch_add(&cm->hits, ht, __ATOMIC_RELAXED);
	free(reqs); free(addr); free(own); free(order); free(state); free(page_of);
	return i == n;
}

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
	return read_pages(cm, nhid_small, genid, off, n, out_buf, 0, NULL, NULL);
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
cachemap_pread(struct cachemap *cm, uint64_t nhid_small, uint32_t genid, uint64_t off, size_t size, void *out_buf)
{
	const int pshift = cm->pages->pshift;
	const uint64_t page_size = 1ULL << pshift;
	if (size == 0)
		return 1;
	if ((uint64_t)size - 1 > UINT64_MAX - off)
		return 0;
	const uint64_t end = off + size;
	const size_t skew = off & (page_size - 1), tail = end & (page_size - 1);
	if (!skew && !tail)
		return cachemap_read_range(cm, nhid_small, genid, off, size, out_buf);
	/* the pages in between go straight to out_buf, the partial ones at the ends through whole pages */
	const uint64_t n = ((end - 1) >> pshift) - (off >> pshift) + 1;
	uint8_t *edge = malloc(2 * page_size);
	if (!edge)
		return 0;
	uint8_t *first = skew || n == 1 ? edge : NULL;
	uint8_t *last = tail && n > 1 ? edge + page_size : NULL;
	const int ok = read_pages(cm, nhid_small, genid, off - skew, n, out_buf, skew, first, last);
	if (ok) {
		if (first)
			memcpy(out_buf, first + skew, n == 1 ? size : page_size - skew);
		if (last)
			memcpy((uint8_t *)out_buf + (((n - 1) << pshift) - skew), last, tail);
	}
	free(edge);
	return ok;
}

/* Writes len bytes at byte page_off of the cached page of `a` (filemap level, ts = the put time the
 * patched page takes).  The newest page of the key in the engine's write-behind ring decides, as it
 * decides a get: a page of `a` is copied into a new slot with the bytes applied, all under wb_mu, so that
 * concurrent writers of one page each patch the other's result; a page of another address replaces the
 * key's record anyway.  Without a ring page the engine patches its stored page (cmb200_patch_batch), or,
 * if it cannot, drops it: no get returns the page's old bytes afterwards. */
static void
filemap_patch(struct filemap *m, const cmb200_addr *a, uint32_t page_off, uint32_t len, const void *bytes, uint64_t ts)
{
	const uint64_t k = addr_key(a);
	struct fm_dev *d = m->dev[cmb200_owner(k, m->g)];
	const size_t bsize = (size_t)m->bsize;
	if (d->wb_n) {
		pthread_mutex_lock(&d->wb_mu);
		for (;;) {
			uint64_t s = d->wb_head;
			while (s > d->wb_tail && d->wb_slot[(s - 1) % d->wb_n].key != k)
				s--;
			if (s == d->wb_tail)
				break;
			struct wb_slot *w = &d->wb_slot[(s - 1) % d->wb_n];
			if (w->state == WB_FILLING) {           /* a put of the key is copying its page in: take that one */
				pthread_mutex_unlock(&d->wb_mu);
				sched_yield();
				pthread_mutex_lock(&d->wb_mu);
				continue;
			}
			if (w->addr.u != a->u || w->addr.l != a->l) {
				pthread_mutex_unlock(&d->wb_mu);
				return;
			}
			if (d->wb_head - d->wb_tail == d->wb_n) {
				pthread_cond_wait(&d->wb_space, &d->wb_mu);     /* the ring may have moved on: look again */
				continue;
			}
			const uint64_t t = d->wb_head++;
			struct wb_slot *nw = &d->wb_slot[t % d->wb_n];
			uint8_t *page = d->wb_pages + (t % d->wb_n) * bsize;
			memcpy(page, d->wb_pages + ((s - 1) % d->wb_n) * bsize, bsize);
			memcpy(page + page_off, bytes, len);
			nw->addr = *a;
			nw->key = k;
			nw->ts = ts;
			nw->state = WB_READY;
			if (d->wb_flusher_asleep)
				pthread_cond_signal(&d->wb_work);
			pthread_mutex_unlock(&d->wb_mu);
			return;
		}
		pthread_mutex_unlock(&d->wb_mu);
	}
	/* a patch adds no entry, so only the arena needs room: no eviction by count */
	filemap_check_arena(d, 1);
	int32_t st = CMB200_MISS;
	if (!cmb200_patch_batch || cmb200_patch_batch(d->eng, 1, a, &page_off, &len, bytes, &ts, &st) != 0) {
		if (cmb200_patch_batch)
			fprintf(stderr, "cachemap_b200: a page could not be patched, it is dropped: %s\n", cmb200_last_error());
		cmb200_unset_batch(d->eng, 1, a);
		st = CMB200_DROPPED;
	}
	/* a patched page and a removed one are changes of the store: the next checkpoint must write them */
	if (st != CMB200_MISS && st != CMB200_BAD_ENTRY)
		__atomic_fetch_add(&m->puts_seen, 1, __ATOMIC_RELAXED);
}

void
cachemap_pwrite(struct cachemap *cm, uint64_t nhid_small, uint32_t genid, uint64_t off, size_t size, const void *data)
{
	struct filemap *fm = cm->pages;
	const int pshift = fm->pshift;
	const uint64_t page_size = 1ULL << pshift;
	if (size == 0 || (uint64_t)size - 1 > UINT64_MAX - off)
		return;
	const uint64_t end = off + size;
	const size_t skew = off & (page_size - 1), tail = end & (page_size - 1);
	if (!skew && !tail) {
		cachemap_write_range(cm, nhid_small, genid, off, size, data);
		return;
	}
	const uint8_t *src = data;
	const uint64_t p0 = off >> pshift, p1 = (end - 1) >> pshift;
	/* pages the range covers whole are put */
	for (uint64_t p = skew ? p0 + 1 : p0; p < (tail ? p1 : p1 + 1); p++)
		cachemap_put(cm, p << pshift, nhid_small, genid, src + ((p << pshift) - off));
	if (!filemap_engine_ready(fm))
		return;
	/* the one or two pages it covers in part are patched where cached */
	const uint64_t ts = now_ns();
	cmb200_addr a;
	if (skew && compose_addr(cm, off, nhid_small, genid, &a) == 0)
		filemap_patch(fm, &a, (uint32_t)skew, (uint32_t)(p1 == p0 ? size : page_size - skew), src, ts);
	if (tail && (p1 != p0 || !skew) && compose_addr(cm, p1 << pshift, nhid_small, genid, &a) == 0)
		filemap_patch(fm, &a, 0, (uint32_t)tail, src + ((p1 << pshift) - off), ts);
}

uint64_t
cachemap_invalidate(struct cachemap *cm, uint64_t nhid_small, uint32_t genid, uint64_t off, uint64_t size)
{
	struct filemap *fm = cm->pages;
	if (size == 0 || !cmb200_invalidate)
		return 0;
	/* a call before the first get applies to the loaded snapshot, not before it */
	if (!filemap_engine_ready(fm))
		return 0;
	filemap_drain(fm);                      /* every page accepted before the call is in a store */
	cmb200_addr first, last;
	if (compose_addr(cm, off, nhid_small, genid, &first) != 0)
		return 0;                       /* put ignores such a page: none is cached */
	/* the last byte, off + size - 1, saturating: TO_END and an overflowing end both mean "to the end" */
	const uint64_t end = size - 1 > UINT64_MAX - off ? UINT64_MAX : off + (size - 1);
	if (compose_addr(cm, end, nhid_small, genid, &last) != 0)
		last.l = ((1ULL << PNUM_SHIFT) - 1) | ((uint64_t)genid << PNUM_SHIFT);
	uint64_t removed = 0;
	for (int i = 0; i < fm->g; i++) {       /* the object's pages are spread over the engines by key */
		uint64_t r = 0;
		if (cmb200_invalidate(fm->dev[i]->eng, nhid_small, first.l, last.l, &r) == 0)
			removed += r;
		else
			fprintf(stderr, "cachemap_b200: cachemap_invalidate: %s\n", cmb200_last_error());
	}
	/* a removal is a change of the store: the next checkpoint must write it */
	__atomic_fetch_add(&fm->puts_seen, removed, __ATOMIC_RELAXED);
	return removed;
}

int
cachemap_checkpoint(struct cachemap *cm)
{
	if (!filemap_engine_ready(cm->pages))
		return -1;
	filemap_drain(cm->pages);
	return filemap_save(cm->pages, 0);
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
	return cm->pages->dev[0]->eng;
}

int
cachemap_engines(struct cachemap *cm, struct cmb200_engine **out, int max)
{
	if (!filemap_engine_ready(cm->pages))
		return 0;
	filemap_drain(cm->pages);
	for (int i = 0; i < cm->pages->g && i < max; i++)
		out[i] = cm->pages->dev[i]->eng;
	return cm->pages->g;
}
