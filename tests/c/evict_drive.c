/* Drives CMB200_EVICT over the CPU stand-in of mock_touch.c.  usage:
 *   evict_drive flags <dir>    starts the map (CMB200_DEVICES as set) and prints
 *                              "engines <g> flags <f0> <f1> ..." with each engine's config flags
 *   evict_drive victim <dir>   fills a map of 1024 pages (4 KiB), reads 8 of the oldest pages past a
 *                              clock tick, then puts 8 new pages past another tick, each a put at
 *                              capacity that evicts.  Prints "raised <n>" (read pages whose ts the
 *                              read raised) and "kept <n>" (read pages still cached at the end). */
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <unistd.h>

#include "../../include/cachemap.h"
#include "../../include/cachemap_b200.h"

uint32_t mock_engine_flags(cmb200_engine *e);
int mock_record_ts(cmb200_engine *e, const cmb200_addr *a, uint64_t *ts);

#define PSHIFT 12
#define CAP 1024
#define READ 8

/* ts of {nhid, page} in whichever engine holds it, 0 when none does */
static uint64_t record_ts(struct cachemap *cm, uint64_t nhid, uint64_t pg) {
	struct cmb200_engine *eng[8];
	const int g = cachemap_engines(cm, eng, 8);
	const cmb200_addr a = { nhid, pg };
	uint64_t ts = 0;
	for (int i = 0; i < g; i++)
		if (mock_record_ts(eng[i], &a, &ts)) return ts;
	return 0;
}

int main(int argc, char **argv) {
	if (argc < 3) { fprintf(stderr, "usage: %s mode dir\n", argv[0]); return 2; }
	struct cachemap *cm = cachemap_create(argv[2], CAP, 12, PSHIFT);
	if (!cm) { fprintf(stderr, "cachemap_create failed\n"); return 1; }
	uint8_t *page = calloc(1, 1u << PSHIFT);
	if (strcmp(argv[1], "flags") == 0) {
		cachemap_put(cm, 0, 1, 0, page);
		struct cmb200_engine *eng[8];
		const int g = cachemap_engines(cm, eng, 8);
		printf("engines %d flags", g);
		for (int i = 0; i < g; i++) printf(" %u", mock_engine_flags(eng[i]));
		printf("\n");
	} else if (strcmp(argv[1], "victim") == 0) {
		for (uint64_t p = 0; p < CAP; p++) {
			memcpy(page, &p, 8);
			cachemap_put(cm, p << PSHIFT, 1, 0, page);
		}
		struct cmb200_engine *eng[8];
		cachemap_engines(cm, eng, 8);                 /* every put is in its engine */
		uint64_t before[READ];
		for (uint64_t p = 0; p < READ; p++) before[p] = record_ts(cm, 1, p);
		usleep(20000);                                /* past the coarse clock's tick */
		for (uint64_t p = 0; p < READ; p++) free(cachemap_get(cm, p << PSHIFT, 1, 0));
		int raised = 0;
		for (uint64_t p = 0; p < READ; p++) raised += record_ts(cm, 1, p) > before[p];
		usleep(20000);
		for (uint64_t p = 0; p < READ; p++) {
			const uint64_t q = CAP + p;
			memcpy(page, &q, 8);
			cachemap_put(cm, q << PSHIFT, 1, 0, page);
		}
		cachemap_engines(cm, eng, 8);
		int kept = 0;
		for (uint64_t p = 0; p < READ; p++) kept += record_ts(cm, 1, p) != 0;
		printf("raised %d\nkept %d\n", raised, kept);
	} else {
		fprintf(stderr, "unknown mode %s\n", argv[1]);
		return 2;
	}
	free(page);
	cachemap_free(cm);
	return 0;
}
