/* Drives CMB200_GHOST over the CPU stand-in of mock_ghost.c.  usage:
 *   ghost_drive flags <dir>    starts the map (CMB200_DEVICES as set) and prints
 *                              "engines <g> flags <f0> <f1> ..." with each engine's config flags
 *   ghost_drive evict <dir>    puts 1056 distinct pages, one by one, into a map of 1024 (4 KiB) from `threads`
 *                              threads (argv[3], default 1: 1, 2, 4 or 8), each its own pages; then puts a page that finds no
 *                              arena room (a dropped put), "counts ...", and unsets one page (filemap_unset).  Prints "counts <evicted>
 *                              <unset>": the addresses that reached cmb200_evict_batch and cmb200_unset_batch
 *   ghost_drive admit <dir>    CMB200_ADMIT=freq: 1024 pages below MOCK_HOT_FROM (estimate 0), then one batch
 *                              of new versions of 8 of them (rejected: their old versions are unset), "counts
 *                              ..."; then one batch of 16 pages at MOCK_HOT_FROM and above: 8 fill the room the
 *                              rejections left, 8 are admitted over their victims, "counts ..."
 *   ghost_drive curve <dir>    gives engine k the histogram hist[j] = (k + 1) (j + 1) and 1000 (k + 1) probes, and
 *                              prints "curve <rc> <misses> <would_hit...>" of cachemap_hit_curve at the extras
 *                              given after the directory */
#include <pthread.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "../../include/cachemap.h"
#include "../../include/cachemap_b200.h"
#include "../../include/filemap.h"

uint32_t mock_engine_flags(cmb200_engine *e);
void mock_ghost_counts(cmb200_engine *e, uint64_t *evicted, uint64_t *unset);
void mock_ghost_set_hist(cmb200_engine *e, const uint64_t *hist, uint64_t probes);

#define PSHIFT 12
#define CAP 1024
#define PUTS (CAP + 32)

static void counts(struct cachemap *cm) {
	struct cmb200_engine *eng[8];
	const int g = cachemap_engines(cm, eng, 8);       /* every put is in its engine */
	uint64_t ev = 0, un = 0;
	for (int i = 0; i < g; i++) {
		uint64_t a, b;
		mock_ghost_counts(eng[i], &a, &b);
		ev += a;
		un += b;
	}
	printf("counts %llu %llu\n", (unsigned long long)ev, (unsigned long long)un);
}

struct job { struct cachemap *cm; int first, n; };

static void *putter(void *arg) {
	struct job *j = arg;
	uint8_t page[1 << PSHIFT];
	memset(page, 0, sizeof(page));
	for (int p = j->first; p < j->first + j->n; p++) {
		memcpy(page, &p, sizeof(p));
		cachemap_put(j->cm, (uint64_t)p << PSHIFT, 1, 0, page);
	}
	return NULL;
}

int main(int argc, char **argv) {
	if (argc < 3) return 2;
	struct cachemap *cm = cachemap_create(argv[2], CAP, 12, PSHIFT);
	if (!cm) return 1;
	uint8_t page[1 << PSHIFT];
	memset(page, 0, sizeof(page));
	if (strcmp(argv[1], "flags") == 0) {
		struct cmb200_engine *eng[64];
		const int g = cachemap_engines(cm, eng, 64);
		printf("engines %d flags", g);
		for (int i = 0; i < g; i++) printf(" %u", mock_engine_flags(eng[i]));
		printf("\n");
	} else if (strcmp(argv[1], "evict") == 0) {
		const int threads = argc > 3 ? atoi(argv[3]) : 1;
		pthread_t th[16];
		struct job jobs[16];
		for (int t = 0; t < threads; t++) {
			jobs[t] = (struct job){ cm, t * (PUTS / threads), PUTS / threads };
			pthread_create(&th[t], NULL, putter, &jobs[t]);
		}
		for (int t = 0; t < threads; t++) pthread_join(th[t], NULL);
		counts(cm);
		memcpy(page, "MOCKDROP", 8);
		cachemap_put(cm, (uint64_t)9000 << PSHIFT, 1, 0, page);
		counts(cm);
		uint128_t a = { 1, 95 };                         /* struct cachemap begins with its filemap */
		filemap_unset(*(struct filemap **)cm, &a);
		counts(cm);
	} else if (strcmp(argv[1], "admit") == 0) {
		for (uint64_t p = 0; p < CAP; p++) {
			memcpy(page, &p, sizeof(p));
			cachemap_put(cm, p << PSHIFT, 1, 0, page);
		}
		counts(cm);
		uint64_t off[8], nh[8];
		uint32_t gen[8];
		uint8_t *pages = calloc(8, 1 << PSHIFT);
		for (int i = 0; i < 8; i++) { off[i] = (uint64_t)(2 * i) << PSHIFT; nh[i] = 1; gen[i] = 0; }
		cachemap_put_batch(cm, 8, off, nh, gen, pages);
		counts(cm);
		uint64_t off2[16], nh2[16];
		uint32_t gen2[16];
		uint8_t *pages2 = calloc(16, 1 << PSHIFT);
		for (int i = 0; i < 16; i++) { off2[i] = (uint64_t)(5000 + i) << PSHIFT; nh2[i] = 1; gen2[i] = 0; }
		cachemap_put_batch(cm, 16, off2, nh2, gen2, pages2);
		free(pages2);
		counts(cm);
		free(pages);
	} else if (strcmp(argv[1], "curve") == 0) {
		struct cmb200_engine *eng[64];
		const int g = cachemap_engines(cm, eng, 64);
		for (int k = 0; k < g; k++) {
			uint64_t h[64];
			for (int j = 0; j < 64; j++) h[j] = (uint64_t)(k + 1) * (j + 1);
			mock_ghost_set_hist(eng[k], h, 1000 * (uint64_t)(k + 1));
		}
		const int n = argc - 3;
		uint64_t extra[32], hit[32], misses = 0;
		for (int i = 0; i < n && i < 32; i++) extra[i] = strtoull(argv[3 + i], NULL, 0);
		const int rc = cachemap_hit_curve(cm, (size_t)n, extra, hit, &misses);
		printf("curve %d %llu", rc, (unsigned long long)misses);
		for (int i = 0; rc == 0 && i < n; i++) printf(" %llu", (unsigned long long)hit[i]);
		printf("\n");
	}
	cachemap_free(cm);
	return 0;
}
