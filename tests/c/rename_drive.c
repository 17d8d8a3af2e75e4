/* Drives cachemap_rename over the stand-in of mock_rename.c.  usage:
 *   rename_drive basic <dir>     `to` (nhid 50, 32 pages) is replaced by `from` (nhid 51, 20 pages)
 *   rename_drive ring <dir>      as basic, with a page of `from` still held in the write-behind ring
 *   rename_drive room <dir>      a thread keeps putting another object while the call runs
 *   rename_drive ckpt <dir>      checkpoint ticks (CMB200_CHECKPOINT_SEC=1) before and after a rename
 *   rename_drive stress <dir> <threads> <seconds>
 *                                puts, gets and renames among four names from many threads at once
 * basic, ring and room print "moved <n> right <to pages with from's bytes> gone <pages that miss>";
 * every mode ends with "log:" and the stand-in's call log, one call per line. */
#include <pthread.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <unistd.h>

#include "../../include/cachemap.h"
#include "../../include/cachemap_b200.h"

void mock_invalidate_log(char *out, size_t cap);
void mock_hold_puts(int on);

static struct cachemap *cm;
static const int pshift = 12;
enum { TO = 50, FROM = 51, TO_PAGES = 32, FROM_PAGES = 20 };

static void fill(uint8_t *page, uint64_t nhid, uint64_t pg, uint64_t version) {
	memset(page, (int)(version & 0xff), (size_t)1 << pshift);
	memcpy(page, &nhid, 8);
	memcpy(page + 8, &pg, 8);
	memcpy(page + 16, &version, 8);
}

/* 1 when page pg of nhid is cached with exactly the bytes fill(.., want_nhid, pg, version) made */
static int holds(uint64_t nhid, uint64_t pg, uint64_t want_nhid, uint64_t version) {
	uint8_t *p = cachemap_get(cm, pg << pshift, nhid, 0);
	if (!p) return 0;
	uint8_t *want = malloc((size_t)1 << pshift);
	fill(want, want_nhid, pg, version);
	const int same = memcmp(p, want, (size_t)1 << pshift) == 0;
	free(want);
	free(p);
	return same;
}

static int misses(uint64_t nhid, uint64_t pg) {
	void *p = cachemap_get(cm, pg << pshift, nhid, 0);
	free(p);
	return p == NULL;
}

static int saves(void) {
	static char log[1 << 16];
	mock_invalidate_log(log, sizeof(log));
	int n = 0;
	for (const char *p = log; (p = strstr(p, "save\n")) != NULL; p++) n++;
	return n;
}

static void *release_puts(void *arg) {
	(void)arg;
	usleep(100000);
	mock_hold_puts(0);
	return NULL;
}

static int stop;

static void *other_puts(void *arg) {
	uint8_t *page = arg;
	for (uint64_t i = 0; !__atomic_load_n(&stop, __ATOMIC_RELAXED); i++) {
		fill(page, 60, i % 64, 9);
		cachemap_put(cm, (i % 64) << pshift, 60, 0, page);
	}
	return NULL;
}

static void write_both(uint8_t *page, int hold_one) {
	for (uint64_t p = 0; p < TO_PAGES; p++) {
		fill(page, TO, p, 1);
		cachemap_put(cm, p << pshift, TO, 0, page);
	}
	for (uint64_t p = 0; p < FROM_PAGES; p++) {
		if (hold_one && p == 2) mock_hold_puts(1);
		fill(page, FROM, p, 2);
		cachemap_put(cm, p << pshift, FROM, 0, page);
	}
}

static void report(uint64_t moved) {
	int right = 0, gone = 0;
	for (uint64_t p = 0; p < FROM_PAGES; p++) right += holds(TO, p, FROM, 2);
	for (uint64_t p = FROM_PAGES; p < TO_PAGES; p++) gone += misses(TO, p);
	for (uint64_t p = 0; p < FROM_PAGES; p++) gone += misses(FROM, p);
	printf("moved %llu right %d gone %d\n", (unsigned long long)moved, right, gone);
}

struct stress_arg { unsigned seed; long errors, ops; };

static void *stress(void *arg) {
	struct stress_arg *a = arg;
	uint8_t *page = malloc((size_t)1 << pshift);
	while (!__atomic_load_n(&stop, __ATOMIC_RELAXED)) {
		const unsigned r = rand_r(&a->seed);
		const uint64_t nhid = 100 + r % 4, pg = (r >> 2) % 32;
		const unsigned op = (r >> 8) % 8;
		if (op < 4) {
			fill(page, nhid, pg, r);
			cachemap_put(cm, pg << pshift, nhid, 0, page);
		} else if (op < 7) {
			uint8_t *p = cachemap_get(cm, pg << pshift, nhid, 0);
			uint64_t l;
			if (p) {
				/* a page moves between names, never between page numbers */
				memcpy(&l, p + 8, 8);
				if (l != pg) a->errors++;
				free(p);
			}
		} else {
			cachemap_rename(cm, nhid, 100 + (r >> 12) % 4, 0);
		}
		a->ops++;
	}
	free(page);
	return NULL;
}

int main(int argc, char **argv) {
	if (argc < 3) { fprintf(stderr, "usage: %s mode dir ...\n", argv[0]); return 2; }
	const char *mode = argv[1];
	cm = cachemap_create(argv[2], 1 << 16, 12, pshift);
	if (!cm) { fprintf(stderr, "cachemap_create failed\n"); return 1; }
	uint8_t *page = malloc((size_t)1 << pshift);
	if (strcmp(mode, "basic") == 0) {
		write_both(page, 0);
		report(cachemap_rename(cm, FROM, TO, 0));
		printf("same %llu\n", (unsigned long long)cachemap_rename(cm, TO, TO, 0));
	} else if (strcmp(mode, "ring") == 0) {
		write_both(page, 1);                                   /* page 2 of `from` and after: held */
		pthread_t t;
		pthread_create(&t, NULL, release_puts, NULL);
		const uint64_t moved = cachemap_rename(cm, FROM, TO, 0);
		pthread_join(t, NULL);
		report(moved);
	} else if (strcmp(mode, "room") == 0) {
		write_both(page, 0);
		uint8_t *other = malloc((size_t)1 << pshift);
		pthread_t t;
		pthread_create(&t, NULL, other_puts, other);
		usleep(20000);
		const uint64_t moved = cachemap_rename(cm, FROM, TO, 0);
		__atomic_store_n(&stop, 1, __ATOMIC_RELAXED);
		pthread_join(t, NULL);
		free(other);
		report(moved);
	} else if (strcmp(mode, "ckpt") == 0) {
		for (uint64_t p = 0; p < 8; p++) {
			fill(page, FROM, p, 1);
			cachemap_put(cm, p << pshift, FROM, 0, page);
		}
		usleep(2500000);                                       /* a tick saves the puts */
		const int after_puts = saves();
		usleep(2200000);                                       /* nothing changed: no save */
		const int idle = saves();
		const uint64_t moved = cachemap_rename(cm, FROM, TO, 0);
		usleep(2500000);                                       /* a tick saves the move */
		printf("moved %llu saves %d %d %d\n", (unsigned long long)moved, after_puts, idle, saves());
	} else if (strcmp(mode, "stress") == 0 && argc > 4) {
		const int n = atoi(argv[3]);
		struct stress_arg *a = calloc((size_t)n, sizeof(*a));
		pthread_t *t = calloc((size_t)n, sizeof(*t));
		for (int i = 0; i < n; i++) {
			a[i].seed = 4321u + (unsigned)i;
			pthread_create(&t[i], NULL, stress, &a[i]);
		}
		usleep((useconds_t)(atof(argv[4]) * 1e6));
		__atomic_store_n(&stop, 1, __ATOMIC_RELAXED);
		long errors = 0, ops = 0;
		for (int i = 0; i < n; i++) {
			pthread_join(t[i], NULL);
			errors += a[i].errors;
			ops += a[i].ops;
		}
		/* quiet now: every name moves to 104, which then holds each page at most once */
		uint64_t moved = 0;
		for (uint64_t nhid = 100; nhid < 104; nhid++) moved += cachemap_rename(cm, nhid, 104, 0);
		int h = 0;
		for (uint64_t nhid = 100; nhid < 104; nhid++)
			for (uint64_t p = 0; p < 32; p++) h += !misses(nhid, p);
		printf("errors %ld ops %ld hits %d\n", errors, ops, h);
		free(a);
		free(t);
	} else {
		fprintf(stderr, "unknown mode %s\n", mode);
		return 2;
	}
	free(page);
	cachemap_free(cm);
	static char log[1 << 16];
	mock_invalidate_log(log, sizeof(log));
	printf("log:\n%s", log);
	return 0;
}
