/* Replays the trace of tests/golden/key_edges.json (addresses that share a store key, and addresses of
 * the table's sentinel keys) through the drop-in's single-page calls over the CPU stand-in of
 * mock_engine.c, which keys its records by FNV-1a as the engine does.  TEST INFRASTRUCTURE ONLY
 * (tests/test_key_edges.py).
 *
 *   key_edges_drive <cachedir> <pshift> <ops file> <pages file> <get|range> <held|one|off>
 *
 * ops file: one op per line, "p <u> <l> <page index>" (cachemap_put), "g <u> <l>" (cachemap_get, or a
 * one-page cachemap_read_range), "u <u> <l>" (filemap_unset); u and l in hex.  pages file: the put
 * pages, 1 << pshift bytes each.  The address {u, l} is offset (l & (2^44 - 1)) << pshift, nhid u,
 * genid l >> 44.
 * ring: held = the stand-in holds every put, so that each page stays in the write-behind ring until an
 * unset drains it; one = the same, but the ring is drained before each put, so that it holds the newest
 * page only; off = no hold (for CMB200_WB_SLOTS=0, where puts are synchronous).
 * Prints, for each op, "op <i> <answer>" after whatever the drop-in printed for it (`bad entry`): the
 * answer is "-" for a put or unset, and "miss" or the page's FNV-1a-64 for a get; then
 * "entries <n> requests <r> hits <h>". */
#include <inttypes.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "../../include/cachemap.h"

void mock_hold_puts(int on);

#define PNUM_MASK ((1ull << 44) - 1)

struct cachemap_head { struct filemap *pages; };         /* the drop-in's struct cachemap starts so */

int main(int argc, char **argv) {
	if (argc != 7) {
		fprintf(stderr, "usage: key_edges_drive <cachedir> <pshift> <ops> <pages> <get|range> <held|one|off>\n");
		return 2;
	}
	const int pshift = atoi(argv[2]);
	const size_t bsize = (size_t)1 << pshift;
	const int by_range = strcmp(argv[5], "range") == 0;
	const int one = strcmp(argv[6], "one") == 0, held = one || strcmp(argv[6], "held") == 0;
	FILE *ops = fopen(argv[3], "r"), *pf = fopen(argv[4], "rb");
	if (!ops || !pf) { perror("open"); return 2; }
	fseek(pf, 0, SEEK_END);
	const long pbytes = ftell(pf);
	fseek(pf, 0, SEEK_SET);
	uint8_t *pages = malloc((size_t)pbytes), *buf = malloc(bsize);
	if (!pages || !buf || fread(pages, 1, (size_t)pbytes, pf) != (size_t)pbytes) { fprintf(stderr, "pages\n"); return 2; }
	fclose(pf);

	struct cachemap *cm = cachemap_create(argv[1], 1024, 12, pshift);
	if (!cm) { fprintf(stderr, "cachemap_create failed\n"); return 2; }
	struct filemap *fm = ((struct cachemap_head *)cm)->pages;
	filemap_entries(fm);                                    /* start the engine before the first hold */
	if (held)
		mock_hold_puts(1);
	char kind;
	uint64_t u, l;
	for (int i = 0; fscanf(ops, " %c %" SCNx64 " %" SCNx64, &kind, &u, &l) == 3; i++) {
		const uint64_t off = (l & PNUM_MASK) << pshift;
		const uint32_t genid = (uint32_t)(l >> 44);
		if (kind == 'p') {
			long idx;
			if (fscanf(ops, " %ld", &idx) != 1 || (idx + 1) * (long)bsize > pbytes) { fprintf(stderr, "bad op %d\n", i); return 2; }
			if (one) {
				mock_hold_puts(0);
				filemap_entries(fm);                    /* lands every page the ring holds */
				mock_hold_puts(1);
			}
			cachemap_put(cm, off, u, genid, pages + (size_t)idx * bsize);
			printf("op %d -\n", i);
		} else if (kind == 'u') {
			uint128_t a = { u, l };
			if (held)
				mock_hold_puts(0);                      /* filemap_unset lands the ring first */
			filemap_unset(fm, &a);
			if (held)
				mock_hold_puts(1);
			printf("op %d -\n", i);
		} else {
			void *p = NULL;
			if (by_range)
				p = cachemap_read_range(cm, u, genid, off, bsize, buf) ? buf : NULL;
			else
				p = cachemap_get(cm, off, u, genid);
			if (p) {
				uint64_t h;
				FNV_hash(p, (int)bsize, &h);
				printf("op %d %016" PRIx64 "\n", i, h);
				if (p != buf)
					free(p);
			} else {
				printf("op %d miss\n", i);
			}
		}
	}
	fclose(ops);
	if (held)
		mock_hold_puts(0);
	uint64_t rq, ht;
	cachemap_get_counters(cm, &rq, &ht);
	printf("entries %" PRIu64 " requests %" PRIu64 " hits %" PRIu64 "\n", filemap_entries(fm), rq, ht);
	cachemap_free(cm);
	free(pages);
	free(buf);
	return 0;
}
