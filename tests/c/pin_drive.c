/* Drives cachemap_pin over the CPU stand-in of mock_pin.c.  usage: pin_drive <dir> <capacity> <step>...
 * Each step is one word, run in order, and prints one line:
 *   pin:<u>:<genid>:<off>:<size>    -> "pin <rc>"        cachemap_pin (size may be "end": CACHEMAP_TO_END)
 *   unpin:<u>:<genid>:<off>:<size>  -> "unpin <rc>"      cachemap_unpin
 *   rename:<from>:<to>:<genid>      -> "rename <moved>"  cachemap_rename
 *   inval:<u>:<genid>               -> "inval <removed>" cachemap_invalidate of every page from 0 on
 *   put:<u>:<first>:<n>             -> "put"             pages first .. first+n-1 of (u, 0), one batch
 *   read:<u>:<first>:<n>            -> "read <hits>"     cachemap_get_batch of those pages
 *   stats                           -> "stats <pinned> <in_hbm> <in_tier>"
 *   admission                       -> "admission <admitted> <rejected>"
 *   lists                           -> "lists <g> <sets>" then, per engine, "list <k> <u>:<l_first>:<l_last> ..."
 *   race:<threads>                  -> "race"  threads that pin and unpin race threads that put past capacity
 * Pages are 4 KiB; page p of u holds p in its first 8 bytes. */
#include <pthread.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "../../include/cachemap.h"
#include "../../include/cachemap_b200.h"

size_t mock_pin_list(cmb200_engine *e, cmb200_pin_range *out, size_t max, uint64_t *sets);

#define PSHIFT 12

static void batch(struct cachemap *cm, uint64_t u, uint64_t first, uint64_t n, int put, uint64_t *hits) {
	uint64_t *off = calloc(n, 8), *nh = calloc(n, 8);
	uint32_t *gen = calloc(n, 4);
	uint8_t *pages = calloc(n, 1 << PSHIFT), *hit = calloc(n, 1);
	for (uint64_t i = 0; i < n; i++) {
		const uint64_t p = first + i;
		off[i] = p << PSHIFT;
		nh[i] = u;
		memcpy(pages + (i << PSHIFT), &p, 8);
	}
	if (put)
		cachemap_put_batch(cm, n, off, nh, gen, pages);
	else {
		cachemap_get_batch(cm, n, off, nh, gen, pages, hit);
		*hits = 0;
		for (uint64_t i = 0; i < n; i++) *hits += hit[i];
	}
	free(off); free(nh); free(gen); free(pages); free(hit);
}

struct racer { struct cachemap *cm; int k; };

static void *pinner(void *arg) {
	struct racer *r = arg;
	for (int i = 0; i < 200; i++) {
		const uint64_t off = (uint64_t)((i * 7 + r->k) % 64) << PSHIFT;
		if (cachemap_pin(r->cm, 1, 0, off, 3 << PSHIFT) < -1) abort();
		if (i % 3 == 0) cachemap_unpin(r->cm, 1, 0, off, 1 << PSHIFT);
		uint64_t p, a, t;
		cachemap_pin_stats(r->cm, &p, &a, &t);
	}
	return NULL;
}

static void *putter(void *arg) {
	struct racer *r = arg;
	for (int i = 0; i < 20; i++) batch(r->cm, 1, (uint64_t)(r->k * 20 + i) * 64, 64, 1, NULL);
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
		if (strcmp(f[0], "pin") == 0)
			printf("pin %lld\n", (long long)cachemap_pin(cm, a[0], (uint32_t)a[1], a[2], a[3]));
		else if (strcmp(f[0], "unpin") == 0)
			printf("unpin %llu\n", (unsigned long long)cachemap_unpin(cm, a[0], (uint32_t)a[1], a[2], a[3]));
		else if (strcmp(f[0], "rename") == 0)
			printf("rename %llu\n", (unsigned long long)cachemap_rename(cm, a[0], a[1], (uint32_t)a[2]));
		else if (strcmp(f[0], "inval") == 0)
			printf("inval %llu\n", (unsigned long long)cachemap_invalidate(cm, a[0], (uint32_t)a[1], 0, CACHEMAP_TO_END));
		else if (strcmp(f[0], "put") == 0) {
			batch(cm, a[0], a[1], a[2], 1, NULL);
			printf("put\n");
		} else if (strcmp(f[0], "read") == 0) {
			uint64_t h = 0;
			batch(cm, a[0], a[1], a[2], 0, &h);
			printf("read %llu\n", (unsigned long long)h);
		} else if (strcmp(f[0], "stats") == 0) {
			uint64_t p, x, t;
			cachemap_pin_stats(cm, &p, &x, &t);
			printf("stats %llu %llu %llu\n", (unsigned long long)p, (unsigned long long)x, (unsigned long long)t);
		} else if (strcmp(f[0], "admission") == 0) {
			uint64_t x, y;
			cachemap_get_admission(cm, &x, &y);
			printf("admission %llu %llu\n", (unsigned long long)x, (unsigned long long)y);
		} else if (strcmp(f[0], "lists") == 0) {
			struct cmb200_engine *eng[64];
			const int g = cachemap_engines(cm, eng, 64);
			static cmb200_pin_range r[CMB200_PIN_RANGES];
			uint64_t sets = 0, total = 0;
			for (int i = 0; i < g; i++) {
				mock_pin_list(eng[i], r, CMB200_PIN_RANGES, &sets);
				total += sets;
			}
			printf("lists %d %llu\n", g, (unsigned long long)total);
			for (int i = 0; i < g; i++) {
				const size_t n = mock_pin_list(eng[i], r, CMB200_PIN_RANGES, NULL);
				printf("list %zu", n);
				for (size_t k = 0; k < n; k++)
					printf(" %llu:%llu:%llu", (unsigned long long)r[k].u, (unsigned long long)r[k].l_first,
					    (unsigned long long)r[k].l_last);
				printf("\n");
			}
		} else if (strcmp(f[0], "race") == 0) {
			const int t = (int)a[0];
			pthread_t th[32];
			struct racer rr[32];
			for (int i = 0; i < 2 * t && i < 32; i++) {
				rr[i] = (struct racer){ cm, i };
				pthread_create(&th[i], NULL, i % 2 ? putter : pinner, &rr[i]);
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
