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
#include <stddef.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <sys/random.h>
#include <sys/stat.h>
#include <time.h>
#include <sched.h>
#include <semaphore.h>
#include <unistd.h>

#include "../../include/cachemap.h"
#include "../../include/cachemap_b200.h"

/* the library's external definition of the header's inline cmb200_owner */
extern int cmb200_owner(uint64_t key, int g);
/* ... and of cmb200_freq_index */
extern uint32_t cmb200_freq_index(uint64_t key, int row, int log2_width);
/* ... and of cmb200_ghost_set */
extern uint32_t cmb200_ghost_set(uint64_t key, int log2_sets);

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
#pragma weak cmb200_rename_set
#pragma weak cmb200_patch_batch
#pragma weak cmb200_freq_estimate
#pragma weak cmb200_load_open
#pragma weak cmb200_load_step
#pragma weak cmb200_load_total
#pragma weak cmb200_load_close
#pragma weak cmb200_set_file_key
#pragma weak cmb200_evict_batch
#pragma weak cmb200_ghost_stats
#pragma weak cmb200_pin_set
#pragma weak cmb200_pin_count
#pragma weak cmb200_pin_promote
#pragma weak cmb200_residency
#pragma weak cmb200_usage_set
#pragma weak cmb200_aead_seal_batch

#define COMBINE_MAX 32          /* get/unset requests one leader takes per GPU batch */
#define LEADERS 32              /* batches of gets that may be in flight at once, each on its own engine lane
                                 * (<= the engine's GET_LANES); see the combining queue below */
#define GET_CALLERS 32          /* callers inside the combining queue at once; the rest sleep at its door */
#define FLUSH_MAX 4096          /* pages the flusher hands over per GPU batch */
#define PNUM_SHIFT 44           /* cachemap.c:155 */
#define PROMOTE_EVERY_MS 100    /* CMB200_TIER_PROMOTE: at most one promotion round this often */
#define MAX_DEVICES 64          /* engines one map may own (CMB200_DEVICES) */
#define LOAD_STEP 4096          /* CMB200_LOAD=background: records per step of the loader thread */

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
	/* held from making arena room until the call that uses it is done (a put batch, a patch, a promotion
	 * round), so that no other call on this engine takes the room in between and the put drops pages */
	pthread_mutex_t room_mu;
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
	/* CMB200_ADMIT=freq: count eviction admits a page only if it is asked for more often than its victim
	 * (filemap_admit_n); set while the engines start, read after */
	int admit;
	uint64_t admitted, rejected;    /* (atomic) pages admitted over a victim / rejected */
	/* CMB200_GHOST=1: every engine keeps ghosts of what it evicts (CMB200_GHOST), and the victims of eviction
	 * by count and by arena pressure, and of admission, go through cmb200_evict_batch; set while the engines
	 * start, read after */
	int ghost;
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
	/* CMB200_LOAD=background: the loader thread runs the steps of `loader` while the map serves.  loading
	 * is 1 from the load's open until its close (under load_mu, read atomically); load_cv is broadcast when
	 * it ends.  load_chain: the load stands for cmb200_load_chain (chain_deltas follows it) rather than
	 * cmb200_load_set. */
	cmb200_loader *loader;
	pthread_t load_thread;
	int load_started, loading, load_chain;
	uint64_t load_loaded, load_total;       /* (atomic) */
	pthread_mutex_t load_mu;
	pthread_cond_t load_cv;
	/* pins (cachemap_pin): pin_n ranges sorted by (u, l_first), disjoint and not touching, the same list on
	 * every engine (cmb200_pin_set), naming pin_pages pages, at most pin_max (CMB200_PIN_MAX, set while the
	 * engines start).  Under pin_mu, which also orders the writes of <destdir>/cachemap_b200.pins.  pin_sealed:
	 * CMB200_KEY_FILE's key is in pin_key and seals the file. */
	pthread_mutex_t pin_mu;
	cmb200_pin_range *pins;
	size_t pin_n;
	uint64_t pin_pages, pin_max;
	int pin_sealed;
	uint8_t pin_key[32];
};

#define SNAPSHOT_NAME "cachemap_b200.snap"
#define PINS_NAME "cachemap_b200.pins"

static int
filemap_snapshot_path(struct filemap *m, char *out, size_t cap)
{
	return snprintf(out, cap, "%s/%s", m->destdir, SNAPSHOT_NAME) < (int)cap;
}

/* CMB200_KEY_FILE: the 32-byte file key, as 32 raw bytes or 64 hex digits (surrounding white space
 * allowed), into key[32].  1 = a key was read, 0 = the variable is unset, -1 = it is set and the file is
 * missing, unreadable or malformed (warned). */
static int
read_key_file(uint8_t key[32])
{
	const char *path = getenv("CMB200_KEY_FILE");
	if (!path || !*path)
		return 0;
	uint8_t buf[160];
	size_t n = 0;
	FILE *f = fopen(path, "rb");
	if (f) {
		n = fread(buf, 1, sizeof(buf), f);
		fclose(f);
	}
	int ok = f && n == 32;
	if (f && !ok) {
		/* 64 hex digits */
		size_t a = 0, b = n;
		while (a < b && (buf[a] == ' ' || buf[a] == '\t' || buf[a] == '\n' || buf[a] == '\r'))
			a++;
		while (b > a && (buf[b - 1] == ' ' || buf[b - 1] == '\t' || buf[b - 1] == '\n' || buf[b - 1] == '\r'))
			b--;
		ok = b - a == 64 && n < sizeof(buf);
		for (size_t i = 0; ok && i < 32; i++) {
			unsigned v;
			char hx[3] = {(char)buf[a + 2 * i], (char)buf[a + 2 * i + 1], 0};
			char *end;
			v = (unsigned)strtoul(hx, &end, 16);
			ok = *end == 0 && hx[0] != '+' && hx[0] != '-' && hx[0] != ' ' && hx[1] != ' ';
			key[i] = (uint8_t)v;
		}
	} else if (ok) {
		memcpy(key, buf, 32);
	}
	explicit_bzero(buf, sizeof(buf));
	if (ok)
		return 1;
	explicit_bzero(key, 32);
	fprintf(stderr, "cachemap_b200: CMB200_KEY_FILE=%s is %s; the cache directory is neither read nor written\n",
	    path, f ? "neither 32 raw bytes nor 64 hex digits" : "missing or unreadable");
	return -1;
}

/* The first 8 bytes of the file at path are a sealed base's magic. */
static int
snapshot_sealed(const char *path)
{
	char magic[8] = {0};
	FILE *f = fopen(path, "rb");
	if (!f)
		return 0;
	const int ok = fread(magic, 8, 1, f) == 1 && memcmp(magic, "CMB200E1", 8) == 0;
	fclose(f);
	return ok;
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
static void *filemap_loader(void *arg);

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
	pthread_mutex_destroy(&d->room_mu);
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

/* CMB200_ADMIT: "freq" gives every engine a frequency sketch (CMB200_FREQ) that counts every get the GPU
 * looks up, and eviction by count admits an incoming page only if its key has been asked for more often
 * than the victim it would replace (filemap_admit_n).  It combines with CMB200_EVICT, which still chooses
 * the victims.  "all" (or unset): every page is admitted, today's behaviour.  Any other value warns (once,
 * with `warn`) and admits all. */
static uint32_t
admit_flags(int warn)
{
	const char *v = getenv("CMB200_ADMIT");
	if (!v || !*v || strcmp(v, "all") == 0)
		return 0;
	if (strcmp(v, "freq") == 0)
		return CMB200_FREQ;
	if (warn)
		fprintf(stderr, "cachemap_b200: CMB200_ADMIT=%s is neither freq nor all; admitting every page\n", v);
	return 0;
}

/* CMB200_LOAD: how the first call after cachemap_create reads the cache directory back.  "wait" (or unset):
 * the call returns once every record is in HBM.  "background": the engines serve at once while a thread
 * loads the file in steps (filemap_loader).  Any other value warns and waits.  1 = background. */
static int
load_background(void)
{
	const char *v = getenv("CMB200_LOAD");
	if (!v || !*v || strcmp(v, "wait") == 0)
		return 0;
	if (strcmp(v, "background") == 0)
		return 1;
	fprintf(stderr, "cachemap_b200: CMB200_LOAD=%s is neither wait nor background; loading before serving\n", v);
	return 0;
}

/* ---- pin list ------------------------------------------------------------------------------------ */

static int
pin_cmp(const void *x, const void *y)
{
	const cmb200_pin_range *a = x, *b = y;
	if (a->u != b->u)
		return a->u < b->u ? -1 : 1;
	return a->l_first < b->l_first ? -1 : a->l_first > b->l_first;
}

/* Sorts the n ranges of r and merges those of one u that overlap or touch.  Returns how many are left. */
static size_t
pin_normalize(cmb200_pin_range *r, size_t n)
{
	if (n == 0)
		return 0;
	qsort(r, n, sizeof(*r), pin_cmp);
	size_t k = 0;
	for (size_t i = 1; i < n; i++) {
		cmb200_pin_range *p = &r[k];
		if (r[i].u == p->u && (r[i].l_first <= p->l_last || r[i].l_first - 1 == p->l_last)) {
			if (r[i].l_last > p->l_last)
				p->l_last = r[i].l_last;
		} else {
			r[++k] = r[i];
		}
	}
	return k + 1;
}

/* Copies the n ranges of cur to out (room for n + 1) without the pages {u, l}, lf <= l <= ll: a range
 * that holds some of them keeps the rest, split in two when they lie inside it.  The pages taken go to
 * cut (room for n, nullable) as ranges, *n_cut of them.  Returns the length of out. */
static size_t
pin_cut(const cmb200_pin_range *cur, size_t n, uint64_t u, uint64_t lf, uint64_t ll, cmb200_pin_range *out,
    cmb200_pin_range *cut, size_t *n_cut)
{
	size_t k = 0, c = 0;
	for (size_t i = 0; i < n; i++) {
		const cmb200_pin_range r = cur[i];
		if (r.u != u || r.l_last < lf || r.l_first > ll) {
			out[k++] = r;
			continue;
		}
		if (r.l_first < lf)
			out[k++] = (cmb200_pin_range){ r.u, r.l_first, lf - 1 };
		if (r.l_last > ll)
			out[k++] = (cmb200_pin_range){ r.u, ll + 1, r.l_last };
		if (cut)
			cut[c++] = (cmb200_pin_range){ r.u, r.l_first > lf ? r.l_first : lf, r.l_last < ll ? r.l_last : ll };
	}
	if (n_cut)
		*n_cut = c;
	return k;
}

static uint64_t
pin_total(const cmb200_pin_range *r, size_t n)
{
	uint64_t pages = 0;
	for (size_t i = 0; i < n; i++)
		pages += r[i].l_last - r[i].l_first + 1;
	return pages;
}

/* {u, l} is pinned (pin_mu held). */
static int
pin_has(const struct filemap *m, const cmb200_addr *a)
{
	size_t lo = 0, hi = m->pin_n;                   /* the first range that starts after a */
	while (lo < hi) {
		const size_t mid = (lo + hi) / 2;
		const cmb200_pin_range *r = &m->pins[mid];
		if (r->u < a->u || (r->u == a->u && r->l_first <= a->l))
			lo = mid + 1;
		else
			hi = mid;
	}
	return lo > 0 && m->pins[lo - 1].u == a->u && a->l <= m->pins[lo - 1].l_last;
}

/* The tag of a sealed pins file: one ChaCha20-Poly1305 seal of an empty text with the file before the tag
 * as AAD, nonce {file nonce, 0}. */
static int
pins_tag(struct filemap *m, const uint8_t *aad, size_t aad_len, uint64_t nonce, uint8_t tag[16])
{
	if (!cmb200_aead_seal_batch)
		return -1;
	uint8_t nc[12] = {0};
	memcpy(nc, &nonce, 8);
	const uint8_t *a[1] = { aad }, *msg[1] = { aad };
	const size_t al[1] = { aad_len }, ml[1] = { 0 };
	uint8_t *out[1] = { tag };
	return cmb200_aead_seal_batch(m->dev[0]->device, m->pin_key, 1, nc, a, al, msg, ml, out);
}

/* Rewrites <destdir>/cachemap_b200.pins with the list (pin_mu held): "CMB200P1" (sealed: "CMB200Q1") |
 * u32 version 1 | u32 pshift | u64 ranges | u64 file nonce | ranges x {u64 u, l_first, l_last} (| the
 * 16-byte tag), little-endian, written to a temporary file and renamed over the old one. */
static void
filemap_pins_write(struct filemap *m)
{
	char path[2200], tmp[2300];
	if (!m->persist || snprintf(path, sizeof(path), "%s/%s", m->destdir, PINS_NAME) >= (int)sizeof(path))
		return;
	snprintf(tmp, sizeof(tmp), "%s.tmp", path);
	const size_t body = 32 + 24 * m->pin_n, len = body + (m->pin_sealed ? 16 : 0);
	uint8_t *buf = malloc(len);
	if (!buf)
		return;
	const uint32_t head[2] = { 1, (uint32_t)m->pshift };
	const uint64_t nr = m->pin_n;
	uint64_t nonce = 0;
	memcpy(buf, m->pin_sealed ? "CMB200Q1" : "CMB200P1", 8);
	memcpy(buf + 8, head, 8);
	memcpy(buf + 16, &nr, 8);
	const char *why = NULL;
	if (m->pin_sealed && getrandom(&nonce, sizeof(nonce), 0) != (ssize_t)sizeof(nonce))
		why = "no random file nonce";
	memcpy(buf + 24, &nonce, 8);
	for (size_t k = 0; k < m->pin_n; k++)
		memcpy(buf + 32 + 24 * k, &m->pins[k], 24);
	if (!why && m->pin_sealed && pins_tag(m, buf, body, nonce, buf + body) != 0)
		why = cmb200_aead_seal_batch ? cmb200_last_error() : "the engine cannot seal";
	FILE *f = why ? NULL : fopen(tmp, "wb");
	if (!why && !f)
		why = strerror(errno);
	if (f) {
		const int ok = fwrite(buf, 1, len, f) == len;
		if (fclose(f) != 0 || !ok || rename(tmp, path) != 0) {
			why = "cannot write it";
			unlink(tmp);
		}
	}
	if (why)
		fprintf(stderr, "cachemap_b200: %s not written: %s\n", path, why);
	free(buf);
}

/* Reads <destdir>/cachemap_b200.pins into the list, which is empty (as the engines start).  A file that is
 * not a pins file of this version and page size, whose tag fails, or that is sealed while no key is set is
 * ignored with a warning.  Otherwise its ranges are taken in file order up to the first one that is
 * malformed, out of order, missing from a short file, or would take the list past CMB200_PIN_MAX pages or
 * CMB200_PIN_RANGES ranges; a file not taken whole is warned about. */
static void
filemap_pins_read(struct filemap *m)
{
	char path[2200];
	if (snprintf(path, sizeof(path), "%s/%s", m->destdir, PINS_NAME) >= (int)sizeof(path))
		return;
	FILE *f = fopen(path, "rb");
	if (!f)
		return;
	const size_t cap = 32 + 24 * (size_t)CMB200_PIN_RANGES + 16 + 1;
	uint8_t *buf = malloc(cap);
	const size_t len = buf ? fread(buf, 1, cap, f) : 0;
	fclose(f);
	const char *why = NULL;
	uint32_t head[2] = {0};
	uint64_t nr = 0, nonce = 0;
	int sealed = 0;
	if (len < 32 || (memcmp(buf, "CMB200P1", 8) != 0 && !(sealed = memcmp(buf, "CMB200Q1", 8) == 0)))
		why = "not a pins file";
	if (!why) {
		memcpy(head, buf + 8, 8);
		memcpy(&nr, buf + 16, 8);
		memcpy(&nonce, buf + 24, 8);
		if (head[0] != 1)
			why = "of another version";
		else if (head[1] != (uint32_t)m->pshift)
			why = "of another page size";
	}
	if (!why && sealed) {
		uint8_t tag[16];
		if (!m->pin_sealed)
			why = "sealed, and no CMB200_KEY_FILE is set";
		else if (nr > CMB200_PIN_RANGES || len != 32 + 24 * nr + 16)
			why = "damaged";
		else if (pins_tag(m, buf, len - 16, nonce, tag) != 0)
			why = "not checked: the engine cannot open it";
		else {
			uint8_t diff = 0;
			for (int i = 0; i < 16; i++)
				diff |= tag[i] ^ buf[len - 16 + i];
			if (diff)
				why = "damaged or sealed with another key (its tag fails)";
		}
	}
	if (why) {
		fprintf(stderr, "cachemap_b200: %s ignored: the file is %s\n", path, why);
		free(buf);
		return;
	}
	const size_t avail = (len - 32 - (sealed ? 16 : 0)) / 24;
	const size_t want = nr < avail ? (size_t)nr : avail;
	m->pins = malloc((want ? want : 1) * sizeof(cmb200_pin_range));
	size_t k = 0;
	uint64_t pages = 0;
	for (; m->pins && k < want && k < CMB200_PIN_RANGES; k++) {
		cmb200_pin_range r;
		memcpy(&r, buf + 32 + 24 * k, 24);
		const cmb200_pin_range *p = k ? &m->pins[k - 1] : NULL;
		if (r.l_first > r.l_last || (p && (r.u < p->u || (r.u == p->u && r.l_first <= p->l_last))) ||
		    r.l_last - r.l_first >= m->pin_max - pages)
			break;
		m->pins[k] = r;
		pages += r.l_last - r.l_first + 1;
	}
	m->pin_n = k;
	m->pin_pages = pages;
	if (k < nr)
		fprintf(stderr, "cachemap_b200: %s: %zu of its %llu ranges kept (%s)\n", path, k, (unsigned long long)nr,
		    k == want && want < nr ? "the file is short" : "the next one is malformed or over CMB200_PIN_MAX");
	free(buf);
}

/* Sends the list to every engine (pin_mu held, or the engines starting). */
static void
filemap_pins_send(struct filemap *m)
{
	for (int i = 0; i < m->g; i++)
		if (cmb200_pin_set(m->engs[i], m->pin_n, m->pins) != 0)
			fprintf(stderr, "cachemap_b200: pins not set on engine %d: %s\n", i, cmb200_last_error());
}

/* Makes `next` (n ranges, normalized) the list: on every engine, then in the file (pin_mu held).  The old
 * list is freed. */
static void
filemap_pins_install(struct filemap *m, cmb200_pin_range *next, size_t n)
{
	free(m->pins);
	m->pins = next;
	m->pin_n = n;
	m->pin_pages = pin_total(next, n);
	filemap_pins_send(m);
	filemap_pins_write(m);
}

/* The pinned records of each engine's host tier go back to its arena while free bytes hold them; under the
 * engine's room lock, so that no put's room is taken. */
static void
filemap_pins_promote(struct filemap *m)
{
	for (int i = 0; i < m->g && cmb200_pin_promote; i++) {
		struct fm_dev *d = m->dev[i];
		if (!d->host_tier)
			continue;
		pthread_mutex_lock(&d->room_mu);
		if (cmb200_pin_promote(d->eng, NULL) != 0)
			fprintf(stderr, "cachemap_b200: pinned records not promoted: %s\n", cmb200_last_error());
		pthread_mutex_unlock(&d->room_mu);
	}
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
	pthread_mutex_init(&d->room_mu, NULL);
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
	const uint32_t admit = admit_flags(index == 0);
	cfg.flags |= admit;
	if (admit && cmb200_freq_estimate)
		m->admit = 1;
	if (env_long("CMB200_GHOST", 0)) {
		if (!cmb200_evict_batch || !cmb200_ghost_stats) {
			if (index == 0)
				fprintf(stderr, "cachemap_b200: CMB200_GHOST ignored: the engine keeps no ghosts\n");
		} else {
			cfg.flags |= CMB200_GHOST;
			m->ghost = 1;
		}
	}
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
			if (m->persist) {
				/* a misconfigured key must never replace an encrypted cache with a plaintext one */
				uint8_t key[32];
				const int have = read_key_file(key);
				if (have < 0)
					m->persist = 0;
				else if (have && !cmb200_set_file_key) {
					fprintf(stderr, "cachemap_b200: CMB200_KEY_FILE ignored: the engine cannot encrypt; the cache "
					    "directory is neither read nor written\n");
					m->persist = 0;
				}
				for (int i = 0; have > 0 && m->persist && i < g; i++)
					if (cmb200_set_file_key(m->engs[i], key) != 0) {
						fprintf(stderr, "cachemap_b200: no file key: %s; the cache directory is neither read nor "
						    "written\n", cmb200_last_error());
						m->persist = 0;
					}
				if (have > 0 && m->persist) {
					memcpy(m->pin_key, key, sizeof(key));
					m->pin_sealed = 1;
				}
				explicit_bzero(key, sizeof(key));
			}
			/* CMB200_PIN_MAX: pages the pins may name, capacity / 4 by default, at most half the capacity so
			 * that at capacity at least half the entries stay evictable; 0 = no pins */
			const long pin_max = env_long("CMB200_PIN_MAX", -1);
			m->pin_max = pin_max < 0 ? m->n / 4 : (uint64_t)pin_max;
			if (m->pin_max > m->n / 2) {
				fprintf(stderr, "cachemap_b200: CMB200_PIN_MAX=%ld is above half the capacity; pinning at most "
				    "%llu pages\n", pin_max, (unsigned long long)(m->n / 2));
				m->pin_max = m->n / 2;
			}
			/* the pins are in force before any record is loaded */
			if (m->persist && cmb200_pin_set) {
				filemap_pins_read(m);
				if (m->pin_n)
					filemap_pins_send(m);
			}
			char snap[2200], d1[2300];
			if (m->persist && filemap_snapshot_path(m, snap, sizeof(snap)) && access(snap, R_OK) == 0) {
				uint64_t got = 0;
				uint32_t k = 0;
				int load_rc = 0;
				snprintf(d1, sizeof(d1), "%s.d1", snap);
				/* a chain next to the base is never ignored, whatever CMB200_CHECKPOINT_DELTAS says now;
				 * a base whose deltas do not match it loads alone */
				const int chain = cmb200_load_chain && (m->checkpoint_deltas > 0 || access(d1, R_OK) == 0);
				if (load_background() && cmb200_load_open && cmb200_load_step && cmb200_load_total && cmb200_load_close) {
					/* the loader thread starts with the flushers below */
					m->loader = cmb200_load_open(m->engs, g, snap);
					if (!m->loader)
						fprintf(stderr, "cachemap_b200: %s: no background load (%s); loading before serving\n", snap,
						    cmb200_last_error());
				}
				if (m->loader) {
					m->load_chain = chain;
					m->load_total = cmb200_load_total(m->loader);
					m->loading = 1;
				} else if (chain) {
					if ((load_rc = cmb200_load_chain(m->engs, g, snap, &got, &k)) != 0)
						fprintf(stderr, "cachemap_b200: %s ignored: %s\n", snap, cmb200_last_error());
					else
						m->chain_deltas = (int)k;
				} else if (!cmb200_load_set)
					fprintf(stderr, "cachemap_b200: %s ignored: the engine cannot load snapshots\n", snap);
				else if ((load_rc = cmb200_load_set(m->engs, g, snap, &got)) != 0)
					fprintf(stderr, "cachemap_b200: %s ignored: %s\n", snap, cmb200_last_error());
				/* an encrypted base that does not load (no key, another key, a damaged file) is left as it is:
				 * the map starts empty and never writes the directory, not even at cachemap_free */
				if (load_rc != 0 && snapshot_sealed(snap)) {
					fprintf(stderr, "cachemap_b200: %s is encrypted and did not load; the cache directory is left "
					    "as it is and not written\n", snap);
					m->persist = 0;
				}
				if (!m->loader && m->pin_n)
					filemap_pins_promote(m);
			}
			/* the flushers start here, i.e. in the process that actually caches (after any fork) */
			for (int i = 0; i < g; i++) {
				struct fm_dev *d = m->dev[i];
				if (d->wb_n && pthread_create(&d->wb_thread, NULL, filemap_flusher, d) == 0)
					d->wb_started = 1;
				else
					d->wb_n = 0;
			}
			if (m->loader) {
				if (pthread_create(&m->load_thread, NULL, filemap_loader, m) == 0)
					m->load_started = 1;
				else
					filemap_loader(m);      /* no thread: the load runs here, as a blocking one */
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
	pthread_mutex_init(&m->load_mu, NULL);
	pthread_cond_init(&m->load_cv, NULL);
	pthread_mutex_init(&m->pin_mu, NULL);
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

/* CMB200_LOAD=background: runs the load's steps to the end, then closes it.  The engines refuse
 * snapshots while the load is open; chain_deltas takes the load's outcome under snap_mu, as a load before
 * serving sets it. */
static void *
filemap_loader(void *arg)
{
	struct filemap *m = arg;
	uint64_t loaded = 0, records = 0;
	uint32_t k = 0;
	int r;
	char snap[2200];
	filemap_snapshot_path(m, snap, sizeof(snap));
	while ((r = cmb200_load_step(m->loader, LOAD_STEP, &loaded)) == 1)
		__atomic_store_n(&m->load_loaded, loaded, __ATOMIC_RELAXED);
	__atomic_store_n(&m->load_loaded, loaded, __ATOMIC_RELAXED);
	if (r < 0)
		fprintf(stderr, "cachemap_b200: %s: the load stopped: %s\n", snap, cmb200_last_error());
	pthread_mutex_lock(&m->snap_mu);
	if (cmb200_load_close(m->loader, &records, &k) == 0 && r == 0 && m->load_chain)
		m->chain_deltas = (int)k;
	pthread_mutex_unlock(&m->snap_mu);
	m->loader = NULL;
	/* the pinned records the load put in a host tier */
	pthread_mutex_lock(&m->pin_mu);
	const size_t pinned = m->pin_n;
	pthread_mutex_unlock(&m->pin_mu);
	if (pinned)
		filemap_pins_promote(m);
	pthread_mutex_lock(&m->load_mu);
	__atomic_store_n(&m->loading, 0, __ATOMIC_RELEASE);
	pthread_cond_broadcast(&m->load_cv);
	pthread_mutex_unlock(&m->load_mu);
	return NULL;
}

/* Waits until a background load has ended. */
static void
filemap_load_wait(struct filemap *m)
{
	pthread_mutex_lock(&m->load_mu);
	while (m->loading)
		pthread_cond_wait(&m->load_cv, &m->load_mu);
	pthread_mutex_unlock(&m->load_mu);
}

/* CMB200_CHECKPOINT_SEC: every checkpoint_sec seconds, a snapshot if puts have landed since the last
 * one.  The engines list their records under their locks and write them outside, so neither the
 * flushers nor the callers of the map wait for the file.  No tick while a background load runs: a file
 * of the half-loaded store would replace the one it is loaded from with less. */
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
		if (!__atomic_load_n(&m->loading, __ATOMIC_ACQUIRE) &&
		    __atomic_load_n(&m->puts_seen, __ATOMIC_RELAXED) != __atomic_load_n(&m->puts_saved, __ATOMIC_RELAXED))
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
	/* a background load runs to its end: the base written below must hold the pages not loaded yet, and
	 * not those this session removed */
	if (m->load_started)
		pthread_join(m->load_thread, NULL);
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
	pthread_mutex_destroy(&m->pin_mu);
	free(m->pins);
	explicit_bzero(m->pin_key, sizeof(m->pin_key));
	pthread_cond_destroy(&m->load_cv);
	pthread_mutex_destroy(&m->load_mu);
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

/* One array of a fan-out: `elem` bytes per item; out = the engines write it, else they read it. */
struct fan { void *p; size_t elem; int out; };

/* What a fan-out calls on one engine: its n items, element j of each in p[j]. */
typedef int (*fan_call)(struct fm_dev *d, size_t n, void *const *p);

/* Calls `call` on each engine that has items, in engine order, with that engine's items in array order:
 * item i of n is on engine own[i], and its values are element i of each of the na (<= 4) arrays a[].
 * With one engine the caller's arrays go through as they are (own is not read).  Otherwise each engine's
 * items are gathered by group_by_owner and, once every call has returned 0, the outputs scattered back.
 * 0 = every call returned 0; -1 = no memory, or a call failed (the engines after it are not called). */
static int
filemap_fan_out(struct filemap *m, size_t n, const int *own, int na, const struct fan *a, fan_call call)
{
	void *p[4], *q[4];
	for (int j = 0; j < na; j++)
		p[j] = a[j].p;
	if (n == 0 || m->g == 1)
		return n ? call(m->dev[0], n, p) : 0;
	size_t bytes = n * sizeof(size_t), start[MAX_DEVICES + 1];
	for (int j = 0; j < na; j++)
		bytes += (n * a[j].elem + 7) & ~(size_t)7;      /* each gathered array 8-byte aligned */
	size_t *order = malloc(bytes);
	if (!order)
		return -1;
	group_by_owner(m->g, n, own, order, start);
	uint8_t *at = (uint8_t *)(order + n);
	for (int j = 0; j < na; j++) {
		p[j] = at;
		at += (n * a[j].elem + 7) & ~(size_t)7;
		for (size_t i = 0; !a[j].out && i < n; i++)
			memcpy((uint8_t *)p[j] + i * a[j].elem, (const uint8_t *)a[j].p + order[i] * a[j].elem, a[j].elem);
	}
	int rc = 0;
	for (int k = 0; k < m->g && rc == 0; k++) {
		for (int j = 0; j < na; j++)
			q[j] = (uint8_t *)p[j] + start[k] * a[j].elem;
		if (start[k + 1] > start[k])
			rc = call(m->dev[k], start[k + 1] - start[k], q);
	}
	for (int j = 0; rc == 0 && j < na; j++)
		for (size_t i = 0; a[j].out && i < n; i++)
			memcpy((uint8_t *)a[j].p + order[i] * a[j].elem, (const uint8_t *)p[j] + i * a[j].elem, a[j].elem);
	free(order);
	return rc;
}

static uint64_t
rand64(void)
{
	uint64_t r = 0;
	for (int b = 0; b < 64; b += 30)        /* filemap.c:271-274 */
		r = r * ((uint64_t)RAND_MAX + 1) + (uint64_t)rand();
	return r;
}

#define ROUND_MAX 4096          /* records one round of eviction, admission or demotion goes for, 3 draws each */

/* One round of candidate draws: draw i from rand64(), and what engine own[i] answered for it
 * (cmb200_sample: cand[i], ts[i], ok[i]).  One allocation, at cand. */
struct round {
	cmb200_addr *cand;
	uint64_t *draw, *ts;
	int32_t *ok;
	int *own;
};

static int
sample_call(struct fm_dev *d, size_t n, void *const *p)
{
	return cmb200_sample(d->eng, n, p[0], p[1], p[2], p[3]);
}

/* Takes n draws from rand64() and samples each on engine `only`, or (only = NULL) on engine
 * cmb200_owner(r, G); r holds them in draw order.  0 = sampled; -1 = nothing was drawn (no memory) or an
 * engine failed (said on stderr for `who`).  The caller frees r->cand either way. */
static int
round_draw(struct filemap *m, struct fm_dev *only, size_t n, const char *who, struct round *r)
{
	r->cand = malloc(n * (sizeof(cmb200_addr) + 2 * sizeof(uint64_t) + sizeof(int32_t) + sizeof(int)));
	if (!r->cand)
		return -1;
	r->draw = (uint64_t *)(r->cand + n);
	r->ts = r->draw + n;
	r->ok = (int32_t *)(r->ts + n);
	r->own = (int *)(r->ok + n);
	for (size_t i = 0; i < n; i++) {
		r->draw[i] = rand64();
		r->own[i] = only ? only->index : cmb200_owner(r->draw[i], m->g);
	}
	const struct fan a[] = { { r->draw, sizeof(uint64_t), 0 }, { r->cand, sizeof(cmb200_addr), 1 },
	                         { r->ts, sizeof(uint64_t), 1 }, { r->ok, sizeof(int32_t), 1 } };
	const int rc = only ? cmb200_sample(only->eng, n, r->draw, r->cand, r->ts, r->ok)
	                    : filemap_fan_out(m, n, r->own, 4, a, sample_call);
	if (rc != 0)
		fprintf(stderr, "cachemap_b200: %s could not sample the store: %s\n", who, cmb200_last_error());
	return rc;
}

/* The oldest of draws 3i .. 3i+2 by the reference's rule (cachemap.c:29-41), as its index in the round;
 * -1 when that draw found no record. */
static long
oldest_of_three(const struct round *r, size_t i)
{
	const uint64_t a = r->ts[3 * i], b = r->ts[3 * i + 1], c = r->ts[3 * i + 2];
	const size_t k = 3 * i + (a < b ? (a > c ? 2 : 0) : (b > c ? 2 : 1));
	return r->ok[k] > 0 ? (long)k : -1;
}

/* Moves the oldest of each of the first `need` triples of draws to the front of the round, in order, and
 * returns how many there are: victim v comes from draw 3i or later, i >= v, so none is overwritten unread. */
static size_t
round_victims(struct round *r, size_t need)
{
	size_t nv = 0;
	for (size_t i = 0; i < need; i++) {
		const long k = oldest_of_three(r, i);
		if (k >= 0) {
			r->cand[nv] = r->cand[k];
			r->own[nv++] = r->own[k];
		}
	}
	return nv;
}

/* Removals ignore what each engine answers: one engine's failure does not keep the others' victims. */
static int
evict_call(struct fm_dev *d, size_t n, void *const *p)
{
	cmb200_evict_batch(d->eng, n, p[0], NULL);
	return 0;
}

static int
unset_call(struct fm_dev *d, size_t n, void *const *p)
{
	cmb200_unset_batch(d->eng, n, p[0]);
	return 0;
}

/* Unsets n victims, each on its engine own[i].  evict: they are evictions, which leave ghosts under
 * CMB200_GHOST (cmb200_evict_batch); other removals do not. */
static void
filemap_unset_victims(struct filemap *m, size_t n, const cmb200_addr *victim, const int *own, int evict)
{
	const struct fan a[] = { { (void *)victim, sizeof(cmb200_addr), 0 } };
	filemap_fan_out(m, n, own, 1, a, evict && m->ghost ? evict_call : unset_call);
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
		if (need > ROUND_MAX)
			need = ROUND_MAX;       /* per round; the loop continues */
		struct round r;
		size_t nv = 0;
		if (round_draw(m, only, (size_t)(3 * need), "eviction", &r) == 0) {
			nv = round_victims(&r, (size_t)need);
			filemap_unset_victims(m, nv, r.cand, r.own, 1);
		}
		free(r.cand);
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
		if (need > ROUND_MAX)
			need = ROUND_MAX;
		const size_t nd = (size_t)(3 * need);
		struct aged *old = malloc(nd * sizeof(struct aged));
		struct round r = { NULL };
		uint64_t round = 0;
		if (old && round_draw(d->m, d, nd, "demotion", &r) == 0) {
			size_t nv = 0;
			for (size_t i = 0; i < nd; i++)
				if (r.ok[i] > 0 && !(guard && bsearch(&r.cand[i], guard, ng, sizeof(cmb200_addr), addr_cmp)))
					old[nv++] = (struct aged){ r.ts[i], r.cand[i] };
			qsort(old, nv, sizeof(struct aged), aged_cmp);
			for (size_t k = 0; k < nv; k++)
				r.cand[k] = old[k].a;           /* oldest first */
			for (size_t k = 0; k < nv && moved < want;) {
				uint64_t take = want - moved < nv - k ? want - moved : nv - k, got = 0;
				if (cmb200_demote_batch(d->eng, (size_t)take, r.cand + k, &got) != 0) {
					fprintf(stderr, "cachemap_b200: demotion to the host tier failed: %s\n", cmb200_last_error());
					break;
				}
				moved += got;
				round += got;
				k += take;
			}
		}
		free(old);
		free(r.cand);
		idle = round ? 0 : idle + 1;
	}
	free(guard);
	return moved;
}

static int
estimate_call(struct fm_dev *d, size_t n, void *const *p)
{
	return cmb200_freq_estimate(d->eng, n, p[0], p[1]);
}

/* est_out[i] = the frequency estimate of addr[i]'s key, from the sketch of the engine that owns it.  -1 if
 * an engine cannot give one. */
static int
filemap_estimate(struct filemap *m, size_t n, const cmb200_addr *addr, uint8_t *est_out)
{
	int *own = NULL;
	if (m->g > 1) {
		if (!(own = malloc(n * sizeof(*own))))
			return -1;
		for (size_t i = 0; i < n; i++)
			own[i] = cmb200_owner(addr_key(&addr[i]), m->g);
	}
	const struct fan a[] = { { (void *)addr, sizeof(cmb200_addr), 0 }, { est_out, 1, 1 } };
	const int rc = filemap_fan_out(m, n, own, 2, a, estimate_call);
	free(own);
	return rc;
}

struct drawn { cmb200_addr a; size_t k; };

static int
drawn_cmp(const void *x, const void *y)
{
	const struct drawn *p = x, *q = y;
	const int c = addr_cmp(&p->a, &q->a);
	return c ? c : (p->k < q->k ? -1 : p->k > q->k);
}

/* Admission by frequency (CMB200_ADMIT=freq) for the `want` pages that overflow the store, pages[0..want):
 * victim k, drawn as filemap_evict_n draws it (the oldest of three), is paired with page k.  The page is
 * admitted if its key's estimate is strictly greater than its victim's, and the victim is unset; otherwise
 * reject[k] = 1 and the victim stays.  With want = 1 this is TinyLFU over the reference's sampler.  A
 * victim drawn twice in a round is paired once, with the first page: the pages after it take the next
 * victims, so every admitted page evicts a record of its own.  Pages left unpaired when the draws find
 * nothing are admitted, as eviction that makes no progress admits them. */
static void
filemap_admit_n(struct filemap *m, uint64_t want, const cmb200_addr *pages, uint8_t *reject)
{
	static int warned;
	uint64_t done = 0;
	int idle = 0;
	while (done < want && idle < 16) {
		uint64_t need = want - done;
		if (need > ROUND_MAX)
			need = ROUND_MAX;
		struct drawn *dr = malloc(need * sizeof(struct drawn));
		uint8_t *ev = malloc(2 * need);        /* estimates: the victims', then the pages' (ep) */
		struct round r = { NULL };
		size_t nv = 0;
		if (dr && ev && round_draw(m, NULL, (size_t)(3 * need), "eviction", &r) == 0) {
			size_t nd = 0;
			for (size_t i = 0; i < need; i++) {
				const long k = oldest_of_three(&r, i);
				if (k >= 0)
					dr[nd++] = (struct drawn){ r.cand[k], (size_t)k };
			}
			qsort(dr, nd, sizeof(*dr), drawn_cmp);
			for (size_t j = 1; j < nd; j++)
				if (addr_cmp(&dr[j].a, &dr[j - 1].a) == 0)
					r.ok[dr[j].k] = 0;              /* drawn before in this round: no victim */
			nv = round_victims(&r, (size_t)need);
			/* victims and pages in one call per engine */
			uint8_t *ep = ev + nv;
			memcpy(r.cand + nv, pages + done, nv * sizeof(cmb200_addr));
			if (nv && filemap_estimate(m, 2 * nv, r.cand, ev) != 0) {
				if (!__atomic_exchange_n(&warned, 1, __ATOMIC_RELAXED))
					fprintf(stderr, "cachemap_b200: admission has no estimates (%s); admitting every page\n",
					    cmb200_last_error());
				memset(ev, 0, nv);
				memset(ep, 1, nv);
			}
			/* a pinned page is always admitted: 16 is above every 4-bit counter */
			pthread_mutex_lock(&m->pin_mu);
			for (size_t k = 0; k < nv && m->pin_n; k++)
				if (pin_has(m, &r.cand[nv + k]))
					ep[k] = 16;
			pthread_mutex_unlock(&m->pin_mu);
			uint64_t ng = 0, nr = 0;
			for (size_t k = 0; k < nv; k++) {
				if (ep[k] > ev[k]) {
					r.cand[ng] = r.cand[k];
					r.own[ng++] = r.own[k];
				} else {
					reject[done + k] = 1;
					nr++;
				}
			}
			filemap_unset_victims(m, (size_t)ng, r.cand, r.own, 1);
			__atomic_fetch_add(&m->admitted, ng, __ATOMIC_RELAXED);
			__atomic_fetch_add(&m->rejected, nr, __ATOMIC_RELAXED);
		}
		free(dr);
		free(ev);
		free(r.cand);
		done += nv;
		idle = nv ? 0 : idle + 1;
	}
}

/* Before a batch of `incoming` puts: while entries + incoming > capacity over all engines, evict
 * (cachemap.c:17-45); loops until the count fits or nothing more can be retired.  Then the batch's
 * pages are reserved until they have landed in their engine (filemap_land_end): a batch that has made
 * its room but is not in its engine yet counts for every other batch's decision, so two flushers
 * neither evict for the same excess nor fill the same room.  The estimate (entries + reserved) can
 * count a batch twice, after it has landed and before its reservation is released; so when the
 * estimate says evict, the decision takes every engine's land_mu and counts again: no batch is
 * between the two then, and no more is evicted than the count needs.
 * With CMB200_ADMIT=freq and the batch's addresses given (addr, nullable), the pages that overflow, the last
 * `need` of the batch (the first ones fill the room that is free), go through filemap_admit_n instead:
 * reject[i] = 1 marks a page that must not be stored (the caller zeroes reject). */
static void
filemap_evict(struct filemap *m, uint64_t incoming, const cmb200_addr *addr, uint8_t *reject)
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
			if (m->admit && addr) {
				/* an excess beyond the batch (the store over capacity already) is evicted as before */
				const uint64_t paired = need < incoming ? need : incoming;
				if (need > paired)
					filemap_evict_n(m, NULL, need - paired);
				filemap_admit_n(m, paired, addr + incoming - paired, reject + incoming - paired);
				break;
			}
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
	pthread_mutex_lock(&d->room_mu);
	filemap_arena_room(d, n, 0);
	uint64_t got = 0;
	const int rc = cmb200_promote_batch(d->eng, n, d->promo_hot, &got);
	pthread_mutex_unlock(&d->room_mu);
	if (rc != 0) {
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
 * the arena is compacted).  The put follows between filemap_land_begin and filemap_land_end.  addr and
 * reject: the batch's pages and the admission's verdicts (filemap_evict). */
static void
filemap_make_room(struct fm_dev *d, uint64_t incoming, const cmb200_addr *addr, uint8_t *reject)
{
	filemap_evict(d->m, incoming, addr, reject);
	filemap_arena_room(d, incoming, 1);
}

/* Row i is the last of its key in addr[0..n): a batch's newest page of a key decides for the key. */
static int
last_of_key(size_t n, const cmb200_addr *addr, size_t i)
{
	const uint64_t k = addr_key(&addr[i]);
	for (size_t j = i + 1; j < n; j++)
		if (addr_key(&addr[j]) == k)
			return 0;
	return 1;
}

/* After a put of n pages whose stored lengths are lens (-1: nothing stored): the keys whose newest page
 * in the batch found no arena room are unset.  The engine leaves such a key's record as it was, and
 * that record holds bytes older than the page just written; served, it would be stale. */
static void
filemap_unset_dropped(struct fm_dev *d, size_t n, const cmb200_addr *addr, const int32_t *lens)
{
	cmb200_addr *v = NULL;
	size_t nv = 0;
	for (size_t i = 0; i < n; i++) {
		if (lens[i] >= 0 || !last_of_key(n, addr, i))
			continue;       /* a later row of the same key supersedes this one (its lens is -1 too) */
		if (!v && !(v = malloc(n * sizeof(*v))))
			return;
		v[nv++] = addr[i];
	}
	if (nv)
		cmb200_unset_batch(d->eng, nv, v);
	free(v);
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
	int32_t *lens = malloc(FLUSH_MAX * sizeof(int32_t));
	uint8_t *reject = malloc(FLUSH_MAX);    /* admission's verdicts, then the put's valid flags */
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

		if (addr && ts && lens && reject) {
			pthread_mutex_lock(&d->room_mu);
			memset(reject, 0, (size_t)count);
			filemap_make_room(d, count, addr, reject);
			filemap_land_begin(d);
			uint64_t run1 = count < d->wb_n - first ? count : d->wb_n - first;
			uint8_t *valid = NULL;
			if (m->admit) {                 /* a rejected page is not stored; its lens -1 unsets its key below */
				for (uint64_t i = 0; i < count; i++)
					reject[i] = !reject[i];
				valid = reject;
			}
			for (uint64_t i = 0; i < count; i++)
				lens[i] = 0;
			cmb200_put_batch(d->eng, (size_t)run1, addr, valid, d->wb_pages + first * (size_t)m->bsize, ts, lens);
			if (run1 < count)
				cmb200_put_batch(d->eng, (size_t)(count - run1), addr + run1, valid ? valid + run1 : NULL, d->wb_pages,
				    ts + run1, lens + run1);
			/* while the slots are still in the ring, which answers gets of their keys */
			filemap_unset_dropped(d, (size_t)count, addr, lens);
			filemap_land_end(d, count);
			pthread_mutex_unlock(&d->room_mu);
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
	free(lens);
	free(reject);
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
		pthread_mutex_lock(&d->room_mu);
		uint8_t reject = 0;
		filemap_make_room(d, 1, &a, &reject);
		filemap_land_begin(d);
		int32_t len = 0;
		const uint8_t valid = !reject;
		cmb200_put_batch(d->eng, 1, &a, &valid, value, &attr, &len);
		filemap_unset_dropped(d, 1, &a, &len);
		filemap_land_end(d, 1);
		pthread_mutex_unlock(&d->room_mu);
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
	pthread_mutex_lock(&d->room_mu);
	filemap_arena_room(d, p->c, 1);
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
	pthread_mutex_unlock(&d->room_mu);
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

/* The admission's verdicts on a slice of a batch call (filemap_evict): a key whose newest page in the
 * slice was rejected stores none of the slice's pages (valid = 0) and is unset now, before the put, so
 * that no older page of it is served.  reject is zeroed again for the next slice. */
static void
filemap_reject_batch(struct filemap *m, size_t n, const cmb200_addr *addr, uint8_t *valid, uint8_t *reject)
{
	cmb200_addr *v = NULL;
	int *own = NULL;
	size_t nv = 0;
	for (size_t i = 0; i < n; i++) {
		if (!reject[i] || !last_of_key(n, addr, i))
			continue;               /* a later page of the key decides */
		const uint64_t k = addr_key(&addr[i]);
		for (size_t j = 0; j <= i; j++)
			if (addr_key(&addr[j]) == k)
				valid[j] = 0;
		if (!v && (!(v = malloc(n * sizeof(*v))) || !(own = malloc(n * sizeof(*own)))))
			break;
		own[nv] = cmb200_owner(k, m->g);
		v[nv++] = addr[i];
	}
	filemap_unset_victims(m, nv, v, own, 0);
	free(v);
	free(own);
	memset(reject, 0, n);
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
	uint8_t *reject = calloc((size_t)n, 1);
	if (!order || !reject) {
		free(order);
		free(reject);
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
		filemap_evict(fm, m, bk.addr + at, reject);
		if (fm->admit)
			filemap_reject_batch(fm, (size_t)m, bk.addr + at, bk.valid + at, reject);
		struct batch_part parts[MAX_DEVICES];
		int np = 0;
		for (int k = 0; k < fm->g; k++) {
			const size_t c = start[k + 1] - start[k];
			if (c == 0)
				continue;
			struct fm_dev *d = fm->dev[k];
			if (c == m && (k == 0 || !on_dev)) {
				/* the whole slice is this engine's (always so with one engine): the caller's arrays as they are */
				pthread_mutex_lock(&d->room_mu);
				filemap_arena_room(d, c, 1);
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
				pthread_mutex_unlock(&d->room_mu);
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
	free(reject);
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
	pthread_mutex_lock(&d->room_mu);
	filemap_arena_room(d, 1, 1);
	int32_t st = CMB200_MISS;
	if (!cmb200_patch_batch || cmb200_patch_batch(d->eng, 1, a, &page_off, &len, bytes, &ts, &st) != 0) {
		if (cmb200_patch_batch)
			fprintf(stderr, "cachemap_b200: a page could not be patched, it is dropped: %s\n", cmb200_last_error());
		cmb200_unset_batch(d->eng, 1, a);
		st = CMB200_DROPPED;
	}
	pthread_mutex_unlock(&d->room_mu);
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

/* The addresses of the first and the last page of object (nhid_small, genid) that bytes [off, off + size)
 * overlap, size >= 1.  The last byte, off + size - 1, saturates: TO_END and an overflowing end both mean
 * "to the end", the page 2^44 - 1.  -1 when the first page does not fit 44 bits. */
static int
compose_span(struct cachemap *cm, uint64_t nhid_small, uint32_t genid, uint64_t off, uint64_t size,
    cmb200_addr *first, cmb200_addr *last)
{
	if (compose_addr(cm, off, nhid_small, genid, first) != 0)
		return -1;
	const uint64_t end = size - 1 > UINT64_MAX - off ? UINT64_MAX : off + (size - 1);
	if (compose_addr(cm, end, nhid_small, genid, last) != 0)
		last->l = ((1ULL << PNUM_SHIFT) - 1) | ((uint64_t)genid << PNUM_SHIFT);
	return 0;
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
	if (compose_span(cm, nhid_small, genid, off, size, &first, &last) != 0)
		return 0;                       /* put ignores such a page: none is cached */
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

/* Every page of (nhid_small, genid) leaves every engine.  Returns the pages removed. */
static uint64_t
filemap_invalidate_all(struct filemap *fm, uint64_t nhid_small, uint32_t genid)
{
	const uint64_t first = (uint64_t)genid << PNUM_SHIFT, last = first | ((1ULL << PNUM_SHIFT) - 1);
	uint64_t removed = 0;
	for (int i = 0; i < fm->g; i++) {
		uint64_t r = 0;
		if (cmb200_invalidate && cmb200_invalidate(fm->dev[i]->eng, nhid_small, first, last, &r) == 0)
			removed += r;
		else
			fprintf(stderr, "cachemap_b200: cachemap_rename: %s\n",
			    cmb200_invalidate ? cmb200_last_error() : "the engine cannot invalidate");
	}
	return removed;
}

/* cachemap_rename's pins: those of `to` for genid are dropped and those of `from` become pins of `to`. */
static void
filemap_pins_rename(struct filemap *m, uint64_t from, uint64_t to, uint32_t genid)
{
	const uint64_t first = (uint64_t)genid << PNUM_SHIFT, last = first | ((1ULL << PNUM_SHIFT) - 1);
	pthread_mutex_lock(&m->pin_mu);
	const size_t n = m->pin_n;
	/* room: each cut splits at most one range in two; the moved ranges come back at the end */
	cmb200_pin_range *a = n ? malloc((2 * n + 2) * sizeof(*a)) : NULL, *b = n ? malloc((2 * n + 2) * sizeof(*b)) : NULL;
	if (a && b) {
		size_t moved = 0;
		const size_t k = pin_cut(m->pins, n, to, first, last, a, NULL, NULL);
		size_t j = pin_cut(a, k, from, first, last, b, a, &moved);
		for (size_t i = 0; i < moved; i++)
			b[j++] = (cmb200_pin_range){ to, a[i].l_first, a[i].l_last };
		j = pin_normalize(b, j);
		if (j != n || memcmp(b, m->pins, n * sizeof(*b)) != 0) {
			if (j <= CMB200_PIN_RANGES) {
				filemap_pins_install(m, b, j);
				b = NULL;
			} else {
				fprintf(stderr, "cachemap_b200: cachemap_rename: the pins would need more than %d ranges; they "
				    "stay as they are\n", CMB200_PIN_RANGES);
			}
		}
	}
	free(a);
	free(b);
	pthread_mutex_unlock(&m->pin_mu);
}

uint64_t
cachemap_rename(struct cachemap *cm, uint64_t nhid_from, uint64_t nhid_to, uint32_t genid)
{
	struct filemap *fm = cm->pages;
	if (nhid_from == nhid_to)
		return 0;
	/* a call before the first get applies to the loaded snapshot, not before it */
	if (!filemap_engine_ready(fm))
		return 0;
	filemap_drain(fm);                      /* every page accepted before the call is in a store */
	/* the pins first, so that the moved pages are pinned on the engines before they arrive */
	filemap_pins_rename(fm, nhid_from, nhid_to, genid);
	/* the old pages of `to` go first: the move replaces only the pages `from` has */
	uint64_t removed = filemap_invalidate_all(fm, nhid_to, genid);
	const uint64_t first = (uint64_t)genid << PNUM_SHIFT, last = first | ((1ULL << PNUM_SHIFT) - 1);
	uint64_t moved = 0, dropped = 0;
	int rc = -1;
	if (cmb200_rename_set) {
		/* every engine's room lock, in index order, so that no flusher's room-making is eaten by the
		 * moved records; the engine call takes each engine's own lock in turn */
		for (int i = 0; i < fm->g; i++)
			pthread_mutex_lock(&fm->dev[i]->room_mu);
		rc = cmb200_rename_set(fm->engs, fm->g, nhid_from, nhid_to, first, last, &moved, &dropped);
		for (int i = fm->g - 1; i >= 0; i--)
			pthread_mutex_unlock(&fm->dev[i]->room_mu);
		if (rc != 0)
			fprintf(stderr, "cachemap_b200: cachemap_rename: %s\n", cmb200_last_error());
	}
	/* without the move, what is left of `from` must not be served under its old name either */
	if (rc != 0)
		removed += filemap_invalidate_all(fm, nhid_from, genid);
	/* moves and removals are changes of the store: the next checkpoint must write them */
	__atomic_fetch_add(&fm->puts_seen, moved + dropped + removed, __ATOMIC_RELAXED);
	return moved;
}

int64_t
cachemap_pin(struct cachemap *cm, uint64_t nhid_small, uint32_t genid, uint64_t off, uint64_t size)
{
	struct filemap *m = cm->pages;
	cmb200_addr first, last;
	if (size == 0 || size == CACHEMAP_TO_END || compose_span(cm, nhid_small, genid, off, size, &first, &last) != 0)
		return -1;
	if (!cmb200_pin_set || !filemap_engine_ready(m))
		return -1;
	int64_t added = -1;
	pthread_mutex_lock(&m->pin_mu);
	cmb200_pin_range *next = malloc((m->pin_n + 1) * sizeof(*next));
	if (next && m->pin_max) {
		memcpy(next, m->pins, m->pin_n * sizeof(*next));
		next[m->pin_n] = (cmb200_pin_range){ nhid_small, first.l, last.l };
		const size_t n = pin_normalize(next, m->pin_n + 1);
		const uint64_t pages = pin_total(next, n);
		if (n <= CMB200_PIN_RANGES && pages <= m->pin_max) {
			added = (int64_t)(pages - m->pin_pages);
			if (added > 0)
				filemap_pins_install(m, next, n);
			else
				free(next);
			next = NULL;
		}
	}
	free(next);
	pthread_mutex_unlock(&m->pin_mu);
	if (added > 0)
		filemap_pins_promote(m);
	return added;
}

uint64_t
cachemap_unpin(struct cachemap *cm, uint64_t nhid_small, uint32_t genid, uint64_t off, uint64_t size)
{
	struct filemap *m = cm->pages;
	cmb200_addr first, last;
	if (size == 0 || compose_span(cm, nhid_small, genid, off, size, &first, &last) != 0)
		return 0;
	if (!cmb200_pin_set || !filemap_engine_ready(m))
		return 0;
	uint64_t removed = 0;
	pthread_mutex_lock(&m->pin_mu);
	cmb200_pin_range *next = malloc((m->pin_n + 1) * sizeof(*next));
	if (next) {
		const size_t n = pin_cut(m->pins, m->pin_n, nhid_small, first.l, last.l, next, NULL, NULL);
		removed = m->pin_pages - pin_total(next, n);
		if (n > CMB200_PIN_RANGES) {
			fprintf(stderr, "cachemap_b200: cachemap_unpin: the pins would need more than %d ranges; nothing "
			    "is unpinned\n", CMB200_PIN_RANGES);
			removed = 0;
		} else if (removed) {
			filemap_pins_install(m, next, n);
			next = NULL;
		}
	}
	free(next);
	pthread_mutex_unlock(&m->pin_mu);
	return removed;
}

void
cachemap_pin_stats(struct cachemap *cm, uint64_t *pinned, uint64_t *in_hbm, uint64_t *in_tier)
{
	struct filemap *m = cm->pages;
	uint64_t p = 0, a = 0, t = 0;
	if (filemap_engine_ready(m)) {
		filemap_drain(m);               /* every page accepted before the call is counted */
		pthread_mutex_lock(&m->pin_mu);
		p = m->pin_pages;
		pthread_mutex_unlock(&m->pin_mu);
		for (int i = 0; i < m->g && cmb200_pin_count && p; i++) {
			uint64_t x = 0, y = 0;
			if (cmb200_pin_count(m->dev[i]->eng, &x, &y) == 0) {
				a += x;
				t += y;
			}
		}
	}
	if (pinned)
		*pinned = p;
	if (in_hbm)
		*in_hbm = a;
	if (in_tier)
		*in_tier = t;
}

_Static_assert(sizeof(struct cachemap_object_usage) == sizeof(cmb200_object_usage) &&
    offsetof(struct cachemap_object_usage, genid) == offsetof(cmb200_object_usage, genid) &&
    offsetof(struct cachemap_object_usage, pages) == offsetof(cmb200_object_usage, pages) &&
    offsetof(struct cachemap_object_usage, stored_bytes) == offsetof(cmb200_object_usage, stored_bytes) &&
    offsetof(struct cachemap_object_usage, newest_ts) == offsetof(cmb200_object_usage, newest_ts),
    "struct cachemap_object_usage is cmb200_object_usage");

int64_t
cachemap_residency(struct cachemap *cm, uint64_t nhid_small, uint32_t genid, uint64_t off, uint64_t size,
    uint8_t *vec)
{
	struct filemap *m = cm->pages;
	cmb200_addr first, last;
	if (size == 0 || size == CACHEMAP_TO_END || size - 1 > UINT64_MAX - off)
		return -1;
	if (compose_addr(cm, off, nhid_small, genid, &first) != 0 ||
	    compose_addr(cm, off + (size - 1), nhid_small, genid, &last) != 0)
		return -1;
	/* a call before the first get answers for the loaded snapshot, not before it */
	if (!cmb200_residency || !filemap_engine_ready(m))
		return -1;
	filemap_drain(m);                       /* every page accepted before the call is in a store */
	const uint64_t n = last.l - first.l + 1;
	uint8_t *v = calloc(n, 1);              /* vec stays untouched unless every engine answers */
	if (!v)
		return -1;
	for (int i = 0; i < m->g; i++)          /* the object's pages are spread over the engines by key */
		if (cmb200_residency(m->dev[i]->eng, nhid_small, first.l, last.l, v) != 0) {
			fprintf(stderr, "cachemap_b200: cachemap_residency: %s\n", cmb200_last_error());
			free(v);
			return -1;
		}
	int64_t cached = 0;
	for (uint64_t k = 0; k < n; k++)
		cached += v[k] != 0;
	pthread_mutex_lock(&m->pin_mu);
	for (size_t k = 0; k < m->pin_n; k++) {
		const cmb200_pin_range *r = &m->pins[k];
		if (r->u != nhid_small || r->l_last < first.l || r->l_first > last.l)
			continue;
		const uint64_t a = r->l_first > first.l ? r->l_first : first.l, b = r->l_last < last.l ? r->l_last : last.l;
		for (uint64_t l = a; l <= b; l++)
			v[l - first.l] |= CACHEMAP_PINNED;
	}
	pthread_mutex_unlock(&m->pin_mu);
	memcpy(vec, v, n);
	free(v);
	return cached;
}

int64_t
cachemap_usage(struct cachemap *cm, size_t max, struct cachemap_object_usage *out)
{
	struct filemap *m = cm->pages;
	/* a call before the first get answers for the loaded snapshot, not before it */
	if (!cmb200_usage_set || !filemap_engine_ready(m))
		return -1;
	filemap_drain(m);                       /* every page accepted before the call is counted */
	uint64_t objects = 0;
	if (cmb200_usage_set(m->engs, m->g, max, (cmb200_object_usage *)out, &objects) != 0) {
		fprintf(stderr, "cachemap_b200: cachemap_usage: %s\n", cmb200_last_error());
		return -1;
	}
	return (int64_t)objects;
}

int
cachemap_checkpoint(struct cachemap *cm)
{
	if (!filemap_engine_ready(cm->pages))
		return -1;
	filemap_load_wait(cm->pages);
	filemap_drain(cm->pages);
	return filemap_save(cm->pages, 0);
}

int
cachemap_load_progress(struct cachemap *cm, uint64_t *loaded, uint64_t *total)
{
	struct filemap *m = cm->pages;
	const int loading = __atomic_load_n(&m->loading, __ATOMIC_ACQUIRE);
	if (loaded)
		*loaded = __atomic_load_n(&m->load_loaded, __ATOMIC_RELAXED);
	if (total)
		*total = __atomic_load_n(&m->load_total, __ATOMIC_RELAXED);
	return loading;
}

void
cachemap_get_counters(struct cachemap *cm, uint64_t *requests, uint64_t *hits)
{
	*requests = __atomic_load_n(&cm->requests, __ATOMIC_RELAXED);
	*hits = __atomic_load_n(&cm->hits, __ATOMIC_RELAXED);
}

void
cachemap_get_admission(struct cachemap *cm, uint64_t *admitted, uint64_t *rejected)
{
	*admitted = __atomic_load_n(&cm->pages->admitted, __ATOMIC_RELAXED);
	*rejected = __atomic_load_n(&cm->pages->rejected, __ATOMIC_RELAXED);
}

/* With G engines each engine's clock counts its own evictions, and keys split evenly over the engines
 * (cmb200_owner), so Δ more pages for the map are Δ / G more for each engine.  A refault at distance d
 * would have hit when d < Δ / G; Δ / G is rounded down to a bucket boundary, so that no refault at or beyond
 * it is counted. */
int
cachemap_hit_curve(struct cachemap *cm, size_t n, const uint64_t *extra_pages, uint64_t *would_hit, uint64_t *misses)
{
	struct filemap *m = cm->pages;
	if (!filemap_engine_ready(m) || !m->ghost)
		return -1;
	for (size_t i = 0; i < n; i++)
		would_hit[i] = 0;
	uint64_t probes = 0;
	for (int k = 0; k < m->g; k++) {
		struct cmb200_ghost_stats st;
		if (cmb200_ghost_stats(m->dev[k]->eng, &st) != 0)
			return -1;
		probes += st.probes;
		for (size_t i = 0; i < n; i++) {
			uint64_t b = extra_pages[i] / (uint64_t)m->g / st.bucket_width;
			if (b > 64)
				b = 64;
			for (uint64_t j = 0; j < b; j++)
				would_hit[i] += st.hist[j];
		}
	}
	if (misses)
		*misses = probes;
	return 0;
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
