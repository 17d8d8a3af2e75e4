/* Drives cachemap_residency and cachemap_usage over the CPU stand-in of mock_usage.c.
 * usage: usage_drive <dir> <capacity> <step>...  Each step is one word, run in order:
 *   put:<u>:<genid>:<first>:<n>    -> "put"                 pages first .. first+n-1 of (u, genid), one batch
 *   held:<u>:<genid>:<page>        -> "held"                one cachemap_put while the stand-in holds every put;
 *                                                           a thread lets the puts go 50 ms later
 *   res:<u>:<genid>:<off>:<size>   -> "res <rc> <vec>"      cachemap_residency, vec as one digit per page (size
 *                                                           may be "end": CACHEMAP_TO_END)
 *   usage:<max>                    -> "usage <rc>" then "row <nhid> <genid> <pages> <tier> <pinned> <bytes>
 *                                     <first> <last>" per row returned
 *   pin:<u>:<genid>:<off>:<size>   -> "pin <rc>"            cachemap_pin
 *   inval:<u>:<genid>              -> "inval <removed>"     cachemap_invalidate of every page from 0 on
 *   fail:<k>                       -> "fail"                engine k cannot answer the usage calls (k < 0: all can)
 *   race:<threads>                 -> "race"                threads calling both race puts, pins and invalidations
 * Pages are 4 KiB. */
#include <pthread.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <unistd.h>

#include "../../include/cachemap.h"
#include "../../include/cachemap_b200.h"

void mock_usage_fail(cmb200_engine *e);
void mock_hold_puts(int on);

#define PSHIFT 12

static void put(struct cachemap *cm, uint64_t u, uint32_t genid, uint64_t first, uint64_t n) {
	uint64_t *off = calloc(n, 8), *nh = calloc(n, 8);
	uint32_t *gen = calloc(n, 4);
	uint8_t *pages = calloc(n, 1 << PSHIFT);
	for (uint64_t i = 0; i < n; i++) {
		off[i] = (first + i) << PSHIFT;
		nh[i] = u;
		gen[i] = genid;
		memcpy(pages + (i << PSHIFT), &off[i], 8);
	}
	cachemap_put_batch(cm, n, off, nh, gen, pages);
	free(off); free(nh); free(gen); free(pages);
}

static void *release(void *arg) {
	(void)arg;
	usleep(50000);
	mock_hold_puts(0);
	return NULL;
}

struct racer { struct cachemap *cm; int k; };

static void *reader(void *arg) {
	struct racer *r = arg;
	static __thread uint8_t vec[256];
	struct cachemap_object_usage rows[16];
	for (int i = 0; i < 200; i++) {
		if (cachemap_residency(r->cm, 1 + i % 2, 0, 0, 256 << PSHIFT, vec) < 0) abort();
		if (cachemap_usage(r->cm, 16, rows) < 0) abort();
	}
	return NULL;
}

static void *writer(void *arg) {
	struct racer *r = arg;
	for (int i = 0; i < 40; i++) {
		put(r->cm, 1 + i % 2, 0, (uint64_t)((i * 13 + r->k) % 200), 32);
		if (i % 4 == 0) cachemap_pin(r->cm, 1, 0, (uint64_t)(i % 64) << PSHIFT, 3 << PSHIFT);
		if (i % 5 == 0) cachemap_invalidate(r->cm, 2, 0, (uint64_t)(i % 100) << PSHIFT, 16 << PSHIFT);
	}
	return NULL;
}

int main(int argc, char **argv) {
	if (argc < 3) return 2;
	struct cachemap *cm = cachemap_create(argv[1], strtoull(argv[2], NULL, 0), 12, PSHIFT);
	if (!cm) return 1;
	for (int s = 3; s < argc; s++) {
		char w[256];
		snprintf(w, sizeof(w), "%s", argv[s]);
		char *f[6] = {0};
		int nf = 0;
		for (char *t = strtok(w, ":"); t && nf < 6; t = strtok(NULL, ":")) f[nf++] = t;
		uint64_t a[5] = {0};
		for (int i = 1; i < nf; i++) a[i - 1] = strcmp(f[i], "end") == 0 ? CACHEMAP_TO_END : strtoull(f[i], NULL, 0);
		if (strcmp(f[0], "put") == 0) {
			put(cm, a[0], (uint32_t)a[1], a[2], a[3]);
			printf("put\n");
		} else if (strcmp(f[0], "held") == 0) {
			static uint8_t page[1 << PSHIFT];
			pthread_t t;
			mock_hold_puts(1);
			cachemap_put(cm, a[2] << PSHIFT, a[0], (uint32_t)a[1], page);
			pthread_create(&t, NULL, release, NULL);
			pthread_detach(t);
			printf("held\n");
		} else if (strcmp(f[0], "res") == 0) {
			/* the vector's length as the call counts it, with a canary past it; 1 when refused */
			const uint64_t off = a[2], size = a[3];
			uint64_t n = 1;
			if (size && size != CACHEMAP_TO_END && size - 1 <= UINT64_MAX - off)
				n = ((off + size - 1) >> PSHIFT) - (off >> PSHIFT) + 1;
			if (n > (1u << 20)) n = 1;
			uint8_t *vec = malloc(n + 1);
			memset(vec, 0xee, n + 1);
			const int64_t rc = cachemap_residency(cm, a[0], (uint32_t)a[1], off, size, vec);
			printf("res %lld ", (long long)rc);
			for (uint64_t k = 0; k < n + 1; k++) printf("%c", vec[k] == 0xee ? '.' : '0' + vec[k]);
			printf("\n");
			free(vec);
		} else if (strcmp(f[0], "usage") == 0) {
			struct cachemap_object_usage rows[64];
			memset(rows, 0xee, sizeof(rows));
			const int64_t rc = cachemap_usage(cm, a[0] < 64 ? a[0] : 64, rows);
			printf("usage %lld\n", (long long)rc);
			for (int64_t k = 0; k < rc && k < (int64_t)a[0] && k < 64; k++)
				printf("row %llu %u %llu %llu %llu %llu %llu %llu\n", (unsigned long long)rows[k].nhid_small, rows[k].genid,
				    (unsigned long long)rows[k].pages, (unsigned long long)rows[k].tier_pages,
				    (unsigned long long)rows[k].pinned_pages, (unsigned long long)rows[k].stored_bytes,
				    (unsigned long long)rows[k].first_page, (unsigned long long)rows[k].last_page);
			if (rc >= 0 && (uint64_t)rc < a[0] && rc < 64)
				printf("untouched %d\n", rows[rc].pages == 0xeeeeeeeeeeeeeeeeull);
		} else if (strcmp(f[0], "pin") == 0) {
			printf("pin %lld\n", (long long)cachemap_pin(cm, a[0], (uint32_t)a[1], a[2], a[3]));
		} else if (strcmp(f[0], "inval") == 0) {
			printf("inval %llu\n", (unsigned long long)cachemap_invalidate(cm, a[0], (uint32_t)a[1], 0, CACHEMAP_TO_END));
		} else if (strcmp(f[0], "fail") == 0) {
			struct cmb200_engine *eng[64];
			const int g = cachemap_engines(cm, eng, 64);
			const long k = strtol(f[1], NULL, 0);
			mock_usage_fail(k >= 0 && k < g ? eng[k] : NULL);
			printf("fail\n");
		} else if (strcmp(f[0], "race") == 0) {
			const int t = (int)a[0];
			pthread_t th[32];
			struct racer rr[32];
			for (int i = 0; i < 2 * t && i < 32; i++) {
				rr[i] = (struct racer){ cm, i };
				pthread_create(&th[i], NULL, i % 2 ? writer : reader, &rr[i]);
			}
			for (int i = 0; i < 2 * t && i < 32; i++) pthread_join(th[i], NULL);
			printf("race\n");
		} else {
			return 3;
		}
		fflush(stdout);
	}
	cachemap_free(cm);
	return 0;
}
