/* Checks of the drop-in's sharding over several engines (CMB200_DEVICES) on the CPU stand-in
 * (mock_multidev.c), TEST INFRASTRUCTURE ONLY (tests/test_multidevice_logic.py).
 * usage: multidev_check <cachedir> share   65 536 keys through the batch calls: every engine holds
 *                                          keys, each holds 1/G of them within 3 %, every page comes
 *                                          back, a range across engines counts in page order
 *        multidev_check <cachedir> fail    an engine that cannot start: none is kept (CMB200_SOFT_FAIL)
 *        multidev_check - owner            stdin: "u l" in hex per line; stdout: the FNV-1a-64 key and
 *                                          cmb200_owner(key, G) for G = 1..8 */
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "../../include/cachemap.h"
#include "../../include/cachemap_b200.h"

int mock_engine_config(cmb200_engine *e, int *device, uint64_t *capacity);
int mock_engines_alive(void);

#define KEYS 65536
#define PSHIFT 9
#define CAPACITY (1u << 17)

static int share(const char *dir) {
	const size_t bsize = (size_t)1 << PSHIFT;
	struct cachemap *cm = cachemap_create((char *)dir, CAPACITY, 12, PSHIFT);
	if (!cm) { fprintf(stderr, "cachemap_create failed\n"); return 1; }
	uint64_t *off = malloc(KEYS * 8), *nhid = malloc(KEYS * 8);
	uint32_t *gen = malloc(KEYS * 4);
	uint8_t *pages = malloc(KEYS * bsize), *back = malloc(KEYS * bsize), *hit = malloc(KEYS);
	for (uint64_t i = 0; i < KEYS; i++) {
		off[i] = (i % 4096) << PSHIFT;
		nhid[i] = 0x5eed0000u + i / 4096;
		gen[i] = 3;
		memset(pages + i * bsize, 0, bsize);
		memcpy(pages + i * bsize, &i, 8);
		memcpy(pages + (i + 1) * bsize - 8, &i, 8);
	}
	cachemap_put_batch(cm, KEYS, off, nhid, gen, pages);
	int bad = 0;
	cmb200_engine *eng[64];
	const int g = cachemap_engines(cm, eng, 64);
	const double share = (double)KEYS / g;
	const uint64_t cap = (CAPACITY + (uint64_t)g - 1) / (uint64_t)g;
	uint64_t total = 0;
	printf("engines %d\n", g);
	for (int k = 0; k < g; k++) {
		int dev = -2;
		uint64_t c = 0;
		const uint64_t n = cmb200_entries(eng[k]);
		mock_engine_config(eng[k], &dev, &c);
		printf("engine %d device %d capacity %lu entries %lu\n", k, dev, (unsigned long)c, (unsigned long)n);
		total += n;
		if (n == 0 || n < 0.97 * share || n > 1.03 * share) { fprintf(stderr, "engine %d holds %lu of %d keys\n", k, (unsigned long)n, KEYS); bad = 1; }
		if (c != cap) { fprintf(stderr, "engine %d capacity %lu, want %lu\n", k, (unsigned long)c, (unsigned long)cap); bad = 1; }
	}
	if (g < 1 || total != KEYS || cachemap_engine(cm) != eng[0]) {
		fprintf(stderr, "entries do not add up: %lu\n", (unsigned long)total);
		bad = 1;
	}
	/* every page back from its engine, in the caller's order */
	cachemap_get_batch(cm, KEYS, off, nhid, gen, back, hit);
	for (uint64_t i = 0; i < KEYS; i++)
		if (!hit[i] || memcmp(back + i * bsize, pages + i * bsize, bsize)) { fprintf(stderr, "page %lu not back\n", (unsigned long)i); bad = 1; break; }
	/* a range over 64 pages of one object, its pages spread over the engines: all hit and counted; then a
	 * range over an object whose page 40 was never put, so the range stops counting there whichever
	 * engine answered first */
	uint64_t rq0, ht0, rq1, ht1;
	for (uint64_t i = 0; i < 64; i++)
		nhid[i] = 0x401e;
	memmove(off + 40, off + 41, 23 * 8);
	cachemap_put_batch(cm, 63, off, nhid, gen, pages);
	cachemap_get_counters(cm, &rq0, &ht0);
	uint8_t *buf = malloc(64 * bsize);
	if (cachemap_read_range(cm, 0x5eed0000u, 3, 0, 64 * bsize, buf) != 1 || memcmp(buf, pages, 64 * bsize)) { fprintf(stderr, "range not read\n"); bad = 1; }
	if (cachemap_read_range(cm, 0x401e, 3, 0, 64 * bsize, buf) != 0) { fprintf(stderr, "range with a hole read\n"); bad = 1; }
	cachemap_get_counters(cm, &rq1, &ht1);
	if (rq1 - rq0 != 64 + 41 || ht1 - ht0 != 64 + 40) {
		fprintf(stderr, "range counters %lu/%lu\n", (unsigned long)(rq1 - rq0), (unsigned long)(ht1 - ht0));
		bad = 1;
	}
	cachemap_free(cm);
	free(off); free(nhid); free(gen); free(pages); free(back); free(hit); free(buf);
	printf(bad ? "multidev_check FAILED\n" : "multidev_check ok\n");
	return bad;
}

static int fail(const char *dir) {
	struct cachemap *cm = cachemap_create((char *)dir, CAPACITY, 12, PSHIFT);
	if (!cm) return 1;
	cmb200_engine *eng[64];
	void *p = cachemap_get(cm, 0, 1, 1);
	const int g = cachemap_engines(cm, eng, 64), alive = mock_engines_alive();
	printf("engines %d alive %d\n", g, alive);
	cachemap_free(cm);
	const int bad = p != NULL || g != 0 || alive != 0;
	printf(bad ? "multidev_check FAILED\n" : "multidev_check ok\n");
	return bad;
}

static int owner(void) {
	unsigned long long u, l;
	while (scanf("%llx %llx", &u, &l) == 2) {
		uint128_t a = { u, l };
		uint64_t key;
		FNV_hash(&a, (int)sizeof(a), &key);
		printf("%016llx", (unsigned long long)key);
		for (int g = 1; g <= 8; g++)
			printf(" %d", cmb200_owner(key, g));
		printf("\n");
	}
	return 0;
}

int main(int argc, char **argv) {
	if (argc < 3) { fprintf(stderr, "usage: %s cachedir share|fail|owner\n", argv[0]); return 2; }
	if (!strcmp(argv[2], "share")) return share(argv[1]);
	if (!strcmp(argv[2], "fail")) return fail(argv[1]);
	if (!strcmp(argv[2], "owner")) return owner();
	return 2;
}
