/* Drives cachemap_invalidate over the stand-in of mock_invalidate.c.  usage:
 *   invalidate_drive convert <dir> <pshift> [<off> <size>]...
 *       for each case: puts pages 0..15 and page 2^44-1 of object (5, genid 3), invalidates
 *       [off, off + size) and prints "ret <pages removed>"
 *   invalidate_drive ring <dir>      a page still in the write-behind ring when the call comes is
 *                                    dropped, a page put after the call is kept
 *   invalidate_drive multi <dir>     every engine of CMB200_DEVICES is called and the counts add up
 *   invalidate_drive ckpt <dir>      checkpoint ticks (CMB200_CHECKPOINT_SEC=1) before and after an
 *                                    invalidation-only change
 *   invalidate_drive load <dir>      the first call of the map, with a snapshot in the directory
 *   invalidate_drive stress <dir> <threads> <seconds>
 *                                    puts, gets and invalidations from many threads at once
 * Every mode ends with "log:" and the stand-in's call log, one call per line. */
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
static int pshift = 12;

static void fill(uint8_t *page, uint64_t nhid, uint64_t pg, uint64_t version) {
	memset(page, (int)(version & 0xff), (size_t)1 << pshift);
	memcpy(page, &nhid, 8);
	memcpy(page + 8, &pg, 8);
	memcpy(page + 16, &version, 8);
}

static int hits(uint64_t nhid, uint32_t genid, uint64_t pg) {
	void *p = cachemap_get(cm, pg << pshift, nhid, genid);
	free(p);
	return p != NULL;
}

/* snapshot saves the stand-in has logged so far */
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

struct stress_arg { unsigned seed; long errors, ops; };
static int stress_stop;

static void *stress(void *arg) {
	struct stress_arg *a = arg;
	uint8_t *page = malloc((size_t)1 << pshift);
	while (!__atomic_load_n(&stress_stop, __ATOMIC_RELAXED)) {
		const unsigned r = rand_r(&a->seed);
		const uint64_t nhid = 100 + r % 4, pg = (r >> 2) % 32;
		const unsigned op = (r >> 8) % 8;
		if (op < 4) {
			fill(page, nhid, pg, r);
			cachemap_put(cm, pg << pshift, nhid, 0, page);
		} else if (op < 7) {
			uint8_t *p = cachemap_get(cm, pg << pshift, nhid, 0);
			uint64_t u, l;
			if (p) {
				memcpy(&u, p, 8);
				memcpy(&l, p + 8, 8);
				if (u != nhid || l != pg) a->errors++;
				free(p);
			}
		} else {
			const uint64_t first = (r >> 12) % 32;
			cachemap_invalidate(cm, nhid, 0, first << pshift, (r >> 20) & 1 ? CACHEMAP_TO_END : (uint64_t)3 << pshift);
		}
		a->ops++;
	}
	free(page);
	return NULL;
}

int main(int argc, char **argv) {
	if (argc < 3) { fprintf(stderr, "usage: %s mode dir ...\n", argv[0]); return 2; }
	const char *mode = argv[1];
	if (strcmp(mode, "convert") == 0 && argc > 3) pshift = atoi(argv[3]);
	cm = cachemap_create(argv[2], 1 << 16, 12, pshift);
	if (!cm) { fprintf(stderr, "cachemap_create failed\n"); return 1; }
	uint8_t *page = malloc((size_t)1 << pshift);
	if (strcmp(mode, "convert") == 0) {
		for (int c = 4; c + 1 < argc; c += 2) {
			for (uint64_t p = 0; p < 16; p++) {
				fill(page, 5, p, 1);
				cachemap_put(cm, p << pshift, 5, 3, page);
			}
			fill(page, 5, (1ULL << 44) - 1, 1);
			cachemap_put(cm, ((1ULL << 44) - 1) << pshift, 5, 3, page);
			const uint64_t off = strtoull(argv[c], NULL, 0), size = strtoull(argv[c + 1], NULL, 0);
			printf("ret %llu\n", (unsigned long long)cachemap_invalidate(cm, 5, 3, off, size));
		}
	} else if (strcmp(mode, "ring") == 0) {
		fill(page, 9, 1, 1);
		cachemap_put(cm, 1ULL << pshift, 9, 0, page);            /* lands in the store */
		cachemap_invalidate(cm, 9, 0, 0, 0);                      /* size 0: nothing */
		mock_hold_puts(1);
		fill(page, 9, 2, 1);
		cachemap_put(cm, 2ULL << pshift, 9, 0, page);            /* held in the ring */
		pthread_t t;
		pthread_create(&t, NULL, release_puts, NULL);
		const uint64_t removed = cachemap_invalidate(cm, 9, 0, 0, CACHEMAP_TO_END);
		pthread_join(t, NULL);
		printf("removed %llu\n", (unsigned long long)removed);
		printf("after %d %d\n", hits(9, 0, 1), hits(9, 0, 2));
		fill(page, 9, 2, 2);
		cachemap_put(cm, 2ULL << pshift, 9, 0, page);            /* after the call: kept */
		uint8_t *p = cachemap_get(cm, 2ULL << pshift, 9, 0);
		uint64_t version = 0;
		if (p) memcpy(&version, p + 16, 8);
		free(p);
		printf("later %d %llu\n", p != NULL, (unsigned long long)version);
	} else if (strcmp(mode, "multi") == 0) {
		for (uint64_t p = 0; p < 96; p++) {
			fill(page, 21, p, 1);
			cachemap_put(cm, p << pshift, 21, 0, page);
		}
		for (uint64_t p = 0; p < 10; p++) {
			fill(page, 22, p, 1);
			cachemap_put(cm, p << pshift, 22, 0, page);
		}
		const uint64_t removed = cachemap_invalidate(cm, 21, 0, 0, CACHEMAP_TO_END);
		int h21 = 0, h22 = 0;
		for (uint64_t p = 0; p < 96; p++) h21 += hits(21, 0, p);
		for (uint64_t p = 0; p < 10; p++) h22 += hits(22, 0, p);
		struct cmb200_engine *eng[8];
		const int g = cachemap_engines(cm, eng, 8);
		uint64_t entries = 0;
		for (int i = 0; i < g; i++) entries += cmb200_entries(eng[i]);
		printf("removed %llu engines %d entries %llu hits %d %d\n", (unsigned long long)removed, g,
		    (unsigned long long)entries, h21, h22);
	} else if (strcmp(mode, "ckpt") == 0) {
		for (uint64_t p = 0; p < 8; p++) {
			fill(page, 31, p, 1);
			cachemap_put(cm, p << pshift, 31, 0, page);
		}
		usleep(2500000);                                          /* a tick saves the puts */
		const int after_puts = saves();
		usleep(2200000);                                          /* nothing changed: no save */
		const int idle = saves();
		const uint64_t removed = cachemap_invalidate(cm, 31, 0, 0, (uint64_t)4 << pshift);
		usleep(2500000);                                          /* a tick saves the removal */
		printf("removed %llu saves %d %d %d\n", (unsigned long long)removed, after_puts, idle, saves());
	} else if (strcmp(mode, "load") == 0) {
		const uint64_t removed = cachemap_invalidate(cm, 7, 0, 0, CACHEMAP_TO_END);   /* the first call of the map */
		int h = 0;
		for (uint64_t p = 0; p < 8; p++) h += hits(7, 0, p);
		printf("removed %llu hits %d\n", (unsigned long long)removed, h);
	} else if (strcmp(mode, "stress") == 0 && argc > 4) {
		const int n = atoi(argv[3]);
		struct stress_arg *a = calloc((size_t)n, sizeof(*a));
		pthread_t *t = calloc((size_t)n, sizeof(*t));
		for (int i = 0; i < n; i++) {
			a[i].seed = 1234u + (unsigned)i;
			pthread_create(&t[i], NULL, stress, &a[i]);
		}
		usleep((useconds_t)(atof(argv[4]) * 1e6));
		__atomic_store_n(&stress_stop, 1, __ATOMIC_RELAXED);
		long errors = 0, ops = 0;
		for (int i = 0; i < n; i++) {
			pthread_join(t[i], NULL);
			errors += a[i].errors;
			ops += a[i].ops;
		}
		/* quiet now: an invalidation of everything leaves nothing */
		for (uint64_t nhid = 100; nhid < 104; nhid++) cachemap_invalidate(cm, nhid, 0, 0, CACHEMAP_TO_END);
		int h = 0;
		for (uint64_t nhid = 100; nhid < 104; nhid++)
			for (uint64_t p = 0; p < 32; p++) h += hits(nhid, 0, p);
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
