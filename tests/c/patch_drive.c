/* Drives cachemap_pwrite / cachemap_pread over the stand-in of mock_patch.c (or plain mock_engine.c,
 * which has no cmb200_patch_batch).  Every mode keeps a model of the object's bytes and checks each page a
 * get returns against it.  usage:
 *   patch_drive split <dir> <pshift> [<off> <size>]...
 *       for each case: puts pages 0..15 of object (5, genid 0), pwrites [off, off + size), then prints
 *       "case <pages put by the pwrite> <pages cached> <pages that differ from the model>" and, when
 *       pread of the range succeeds, "pread <1 if its bytes equal the model's>"
 *   patch_drive ring <dir>      a page still in the write-behind ring is patched there, a later put kept
 *   patch_drive multi <dir>     patches reach the engine that owns the page's key (CMB200_DEVICES)
 *   patch_drive ckpt <dir>      checkpoint ticks (CMB200_CHECKPOINT_SEC=1) before and after a patch-only change
 *   patch_drive fallback <dir>  without cmb200_patch_batch a page covered in part is dropped
 *   patch_drive stress <dir> <threads> <seconds>
 *                               threads pwrite disjoint bytes of one page while its puts are held back
 *                               for a while and others read it; every thread's last bytes must land
 * Every mode ends with "log:" and the stand-in's call log, one call per line. */
#include <pthread.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <unistd.h>

#include "../../include/cachemap.h"
#include "../../include/cachemap_b200.h"
#include "../../include/uint128.h"

void mock_patch_log(char *out, size_t cap) __attribute__((weak));
void mock_hold_puts(int on);

#define PAGES 16

static struct cachemap *cm;
static int pshift = 12;
static uint8_t *model;                  /* 2 x PAGES pages of object (5, 0); pages 0 .. PAGES - 1 are put */

static size_t page_size(void) { return (size_t)1 << pshift; }

static uint64_t put_chunks(void) {
	struct cmb200_engine *eng[8];
	const int g = cachemap_engines(cm, eng, 8);
	uint64_t n = 0;
	for (int i = 0; i < g; i++) {
		cmb200_stats st;
		cmb200_get_stats(eng[i], &st);
		n += st.put_chunks;
	}
	return n;
}

/* pages of (5, 0) cached, and those among them whose bytes differ from the model */
static void check_pages(int *cached, int *wrong) {
	*cached = *wrong = 0;
	for (uint64_t p = 0; p < PAGES; p++) {
		uint8_t *got = cachemap_get(cm, p << pshift, 5, 0);
		if (!got) continue;
		(*cached)++;
		*wrong += memcmp(got, model + (p << pshift), page_size()) != 0;
		free(got);
	}
}

static void put_all(uint64_t nhid, int version) {
	for (uint64_t p = 0; p < PAGES; p++) {
		for (size_t b = 0; b < page_size(); b++) model[(p << pshift) + b] = (uint8_t)(p * 31 + b * 7 + (size_t)version);
		cachemap_put(cm, p << pshift, nhid, 0, model + (p << pshift));
	}
	free(cachemap_get(cm, 0, 99, 0));           /* (a get of nothing: the engines are up) */
}

static void *release_puts(void *arg) {
	(void)arg;
	usleep(100000);
	mock_hold_puts(0);
	return NULL;
}

/* stress: thread t owns bytes [24 t + 8, 24 t + 32) of page 1 */
#define REGION 24
struct stress_arg { int t; unsigned seed; long ops, errors; uint8_t last; };
static int stress_stop;

static void *stress(void *arg) {
	struct stress_arg *a = arg;
	uint8_t buf[REGION];
	const uint64_t off = (1ull << pshift) + 8 + (uint64_t)REGION * (uint64_t)a->t;
	while (!__atomic_load_n(&stress_stop, __ATOMIC_RELAXED)) {
		const unsigned r = rand_r(&a->seed);
		if (r % 4 == 0) {
			uint8_t *p = cachemap_get(cm, 1ull << pshift, 5, 0);
			if (p) {
				/* my region holds one value throughout: a page is never a mix of two versions of it */
				for (int b = 1; b < REGION; b++) a->errors += p[off - (1ull << pshift) + (size_t)b] != p[off - (1ull << pshift)];
				free(p);
			}
		} else {
			a->last = (uint8_t)(r >> 8);
			memset(buf, a->last, REGION);
			cachemap_pwrite(cm, 5, 0, off, REGION, buf);
		}
		a->ops++;
	}
	return NULL;
}

int main(int argc, char **argv) {
	if (argc < 3) { fprintf(stderr, "usage: %s mode dir ...\n", argv[0]); return 2; }
	const char *mode = argv[1];
	if (strcmp(mode, "split") == 0 && argc > 3) pshift = atoi(argv[3]);
	cm = cachemap_create(argv[2], 1 << 16, 12, pshift);
	if (!cm) { fprintf(stderr, "cachemap_create failed\n"); return 1; }
	model = calloc(2 * PAGES, (size_t)1 << pshift);
	const size_t P = page_size();
	if (strcmp(mode, "split") == 0) {
		for (int c = 4; c + 1 < argc; c += 2) {
			put_all(5, c);
			struct cmb200_engine *e;
			cachemap_engines(cm, &e, 1);            /* every put is in the store */
			const uint64_t off = strtoull(argv[c], NULL, 0), size = strtoull(argv[c + 1], NULL, 0);
			uint8_t *data = malloc(size ? size : 1);
			for (uint64_t b = 0; b < size; b++) data[b] = (uint8_t)(0x80 + c + b * 13);
			const uint64_t before = put_chunks();
			cachemap_pwrite(cm, 5, 0, off, size, data);
			cachemap_engines(cm, &e, 1);
			memcpy(model + off, data, size);
			int cached, wrong;
			check_pages(&cached, &wrong);
			printf("case %llu %d %d\n", (unsigned long long)(put_chunks() - before), cached, wrong);
			uint8_t *back = malloc(size ? size : 1);
			if (cachemap_pread(cm, 5, 0, off, size, back))
				printf("pread %d\n", memcmp(back, model + off, size) == 0);
			free(back);
			free(data);
		}
	} else if (strcmp(mode, "ring") == 0) {
		put_all(5, 1);
		struct cmb200_engine *e;
		cachemap_engines(cm, &e, 1);
		mock_hold_puts(1);
		for (size_t b = 0; b < P; b++) model[2 * P + b] = (uint8_t)(b * 3 + 1);
		cachemap_put(cm, 2 * P, 5, 0, model + 2 * P);                       /* held in the ring */
		const uint8_t a[5] = {1, 2, 3, 4, 5}, b[7] = {9, 9, 9, 9, 9, 9, 9};
		cachemap_pwrite(cm, 5, 0, 2 * P + 100, sizeof(a), a);                /* patched in the ring */
		memcpy(model + 2 * P + 100, a, sizeof(a));
		cachemap_pwrite(cm, 5, 0, 2 * P + 102, sizeof(b), b);                /* on top of the first one */
		memcpy(model + 2 * P + 102, b, sizeof(b));
		uint8_t *got = cachemap_get(cm, 2 * P, 5, 0);
		printf("held %d\n", got && memcmp(got, model + 2 * P, P) == 0);
		free(got);
		pthread_t t;
		pthread_create(&t, NULL, release_puts, NULL);
		pthread_join(t, NULL);
		cachemap_engines(cm, &e, 1);
		int cached, wrong;
		check_pages(&cached, &wrong);
		printf("landed %d %d\n", cached, wrong);
		for (size_t x = 0; x < P; x++) model[2 * P + x] = 0x77;
		cachemap_put(cm, 2 * P, 5, 0, model + 2 * P);                       /* a later put is kept */
		check_pages(&cached, &wrong);
		printf("later %d %d\n", cached, wrong);
	} else if (strcmp(mode, "multi") == 0) {
		put_all(5, 1);
		struct cmb200_engine *e;
		cachemap_engines(cm, &e, 1);
		uint8_t data[3 * 4096];
		for (size_t b = 0; b < sizeof(data); b++) data[b] = (uint8_t)(b * 5 + 1);
		/* 15 ranges from byte 100 of page p to byte 100 of page p + 1: two edge pages each */
		for (uint64_t p = 0; p + 1 < PAGES; p++) {
			cachemap_pwrite(cm, 5, 0, p * P + 100, P, data);
			memcpy(model + p * P + 100, data, P);
		}
		int cached, wrong;
		check_pages(&cached, &wrong);
		struct cmb200_engine *eng[8];
		const int g = cachemap_engines(cm, eng, 8);
		printf("engines %d cached %d wrong %d\n", g, cached, wrong);
	} else if (strcmp(mode, "ckpt") == 0) {
		put_all(5, 1);
		usleep(2500000);                                                     /* a tick saves the puts */
		static char log[1 << 20];
		int saves[3];
		for (int k = 0; k < 3; k++) {
			if (k == 1) usleep(2200000);                                     /* nothing changed: no save */
			if (k == 2) {
				const uint8_t a[3] = {7, 7, 7};
				cachemap_pwrite(cm, 5, 0, 3 * P + 11, sizeof(a), a);          /* a patch and nothing else */
				usleep(2500000);
			}
			mock_patch_log(log, sizeof(log));
			saves[k] = 0;
			for (const char *q = log; (q = strstr(q, "save\n")) != NULL; q++) saves[k]++;
		}
		printf("saves %d %d %d\n", saves[0], saves[1], saves[2]);
	} else if (strcmp(mode, "fallback") == 0) {
		put_all(5, 1);
		struct cmb200_engine *e;
		cachemap_engines(cm, &e, 1);
		uint8_t data[3 * 4096];
		memset(data, 0x55, sizeof(data));
		cachemap_pwrite(cm, 5, 0, 2 * P + 10, 2 * P, data);                  /* page 3 whole, pages 2 and 4 in part */
		memcpy(model + 2 * P + 10, data, 2 * P);
		cachemap_engines(cm, &e, 1);
		int hit[PAGES], cached, wrong;
		for (uint64_t p = 0; p < PAGES; p++) { void *q = cachemap_get(cm, p << pshift, 5, 0); hit[p] = q != NULL; free(q); }
		check_pages(&cached, &wrong);
		printf("fallback %d %d %d cached %d wrong %d\n", hit[2], hit[3], hit[4], cached, wrong);
	} else if (strcmp(mode, "stress") == 0 && argc > 4) {
		const int n = atoi(argv[3]);
		if ((size_t)(8 + REGION * n) > P) { fprintf(stderr, "too many threads for the page\n"); return 2; }
		put_all(5, 1);
		struct cmb200_engine *e;
		cachemap_engines(cm, &e, 1);
		mock_hold_puts(1);
		memset(model + P, 0, P);
		cachemap_put(cm, P, 5, 0, model + P);                                /* page 1 starts in the ring */
		pthread_t rel;
		pthread_create(&rel, NULL, release_puts, NULL);
		struct stress_arg *a = calloc((size_t)n, sizeof(*a));
		pthread_t *t = calloc((size_t)n, sizeof(*t));
		for (int i = 0; i < n; i++) {
			a[i].t = i;
			a[i].seed = 777u + (unsigned)i;
			a[i].last = model[P + 8 + (size_t)REGION * (size_t)i];
			pthread_create(&t[i], NULL, stress, &a[i]);
		}
		usleep((useconds_t)(atof(argv[4]) * 1e6));
		__atomic_store_n(&stress_stop, 1, __ATOMIC_RELAXED);
		long ops = 0, errors = 0, lost = 0;
		for (int i = 0; i < n; i++) {
			pthread_join(t[i], NULL);
			ops += a[i].ops;
			errors += a[i].errors;
		}
		pthread_join(rel, NULL);
		cachemap_engines(cm, &e, 1);
		uint8_t *p = cachemap_get(cm, P, 5, 0);
		for (int i = 0; i < n && p; i++)
			for (int b = 0; b < REGION; b++) lost += p[8 + REGION * i + b] != a[i].last;
		printf("stress errors %ld ops %ld lost %ld page %d\n", errors, ops, lost, p != NULL);
		free(p);
		free(a);
		free(t);
	} else {
		fprintf(stderr, "unknown mode %s\n", mode);
		return 2;
	}
	cachemap_free(cm);
	free(model);
	static char log[1 << 20];
	log[0] = '\0';
	if (mock_patch_log) mock_patch_log(log, sizeof(log));
	printf("log:\n%s", log);
	return 0;
}
