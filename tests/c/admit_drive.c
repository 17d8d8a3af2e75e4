/* Drives CMB200_ADMIT over the CPU stand-in of mock_freq.c.  usage:
 *   admit_drive flags <dir>    starts the map (CMB200_DEVICES as set) and prints
 *                              "engines <g> flags <f0> <f1> ..." with each engine's config flags
 *   admit_drive reject <dir>   fills a map of 1024 pages (4 KiB) and reads pages 0..511 twice; then puts a
 *                              new page whose estimate is 0, then a new version of a page p >= 512 whose
 *                              estimate is 0, both at capacity, where every victim's estimate is >= 0.
 *                              Prints "old <0|1>" (a get of p hits), "new <0|1>", "entries <n>" and
 *                              "admission <admitted> <rejected>"
 *   admit_drive admit <dir>    fills a map of 1024 pages that are never read; reads a new page three times
 *                              (misses) and puts it at capacity.  Prints "new <0|1>" (a get returns its
 *                              bytes), "entries <n>" and "admission <admitted> <rejected>" */
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "../../include/cachemap.h"
#include "../../include/cachemap_b200.h"
#include "../../include/uint128.h"

uint32_t mock_engine_flags(cmb200_engine *e);

#define PSHIFT 12
#define CAP 1024

static int cached(struct cachemap *cm, uint64_t pg) {
	void *p = cachemap_get(cm, pg << PSHIFT, 1, 0);
	const int hit = p != NULL;
	free(p);
	return hit;
}

static uint64_t entries(struct cachemap *cm) {
	struct cmb200_engine *eng[8];
	const int g = cachemap_engines(cm, eng, 8);       /* every put is in its engine */
	uint64_t n = 0;
	for (int i = 0; i < g; i++) n += cmb200_entries(eng[i]);
	return n;
}

/* the first page >= from whose key's estimate, on the engine that owns it, is 0 */
static uint64_t first_unread(struct cachemap *cm, uint64_t from) {
	struct cmb200_engine *eng[8];
	const int g = cachemap_engines(cm, eng, 8);
	for (uint64_t p = from;; p++) {
		uint128_t a = { 1, p };
		uint64_t key;
		FNV_hash(&a, (int)sizeof(a), &key);
		const cmb200_addr ca = { 1, p };
		uint8_t est = 1;
		if (cmb200_freq_estimate(eng[cmb200_owner(key, g)], 1, &ca, &est) != 0) return from;
		if (est == 0) return p;
	}
}

static void put(struct cachemap *cm, uint8_t *page, uint64_t pg, uint64_t version) {
	memcpy(page, &pg, 8);
	memcpy(page + 8, &version, 8);
	cachemap_put(cm, pg << PSHIFT, 1, 0, page);
	struct cmb200_engine *eng[8];
	cachemap_engines(cm, eng, 8);                     /* landed: the next put sees it */
}

int main(int argc, char **argv) {
	if (argc < 3) { fprintf(stderr, "usage: %s mode dir\n", argv[0]); return 2; }
	struct cachemap *cm = cachemap_create(argv[2], CAP, 12, PSHIFT);
	if (!cm) { fprintf(stderr, "cachemap_create failed\n"); return 1; }
	uint8_t *page = calloc(1, 1u << PSHIFT);
	uint64_t adm = 0, rej = 0;
	if (strcmp(argv[1], "flags") == 0) {
		cachemap_put(cm, 0, 1, 0, page);
		struct cmb200_engine *eng[8];
		const int g = cachemap_engines(cm, eng, 8);
		printf("engines %d flags", g);
		for (int i = 0; i < g; i++) printf(" %u", mock_engine_flags(eng[i]));
		printf("\n");
	} else if (strcmp(argv[1], "reject") == 0) {
		for (uint64_t p = 0; p < CAP; p++) put(cm, page, p, 1);
		for (int k = 0; k < 2; k++)
			for (uint64_t p = 0; p < CAP / 2; p++) cached(cm, p);
		const uint64_t old = first_unread(cm, CAP / 2), fresh = first_unread(cm, 2 * CAP);
		put(cm, page, fresh, 1);                      /* first: the store is at capacity for both */
		put(cm, page, old, 2);
		printf("old %d\nnew %d\nentries %llu\n", cached(cm, old), cached(cm, fresh), (unsigned long long)entries(cm));
		cachemap_get_admission(cm, &adm, &rej);
		printf("admission %llu %llu\n", (unsigned long long)adm, (unsigned long long)rej);
	} else if (strcmp(argv[1], "admit") == 0) {
		for (uint64_t p = 0; p < CAP; p++) put(cm, page, p, 1);
		for (int k = 0; k < 3; k++) cached(cm, CAP + 7);
		put(cm, page, CAP + 7, 1);
		const uint64_t n = entries(cm);
		void *got = cachemap_get(cm, (uint64_t)(CAP + 7) << PSHIFT, 1, 0);
		const int ok = got && memcmp(got, page, 1u << PSHIFT) == 0;
		free(got);
		printf("new %d\nentries %llu\n", ok, (unsigned long long)n);
		cachemap_get_admission(cm, &adm, &rej);
		printf("admission %llu %llu\n", (unsigned long long)adm, (unsigned long long)rej);
	} else {
		fprintf(stderr, "unknown mode %s\n", argv[1]);
		return 2;
	}
	free(page);
	cachemap_free(cm);
	return 0;
}
