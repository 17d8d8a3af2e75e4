/* cachemap_get latency from T native threads, with or without a thread that calls cachemap_usage back to
 * back meanwhile (tools/usage_bench.py builds and runs it against the library).
 *   usage_serve <cachedir> <pages> <threads> <gets-per-thread> <usage: 0|1>
 * The map holds <pages> 4 KiB pages of objects of 16 pages.  Prints one JSON line: get p50 / p99 in
 * microseconds over every call of every thread, hits, and the usage calls made while the gets ran. */
#include <pthread.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <time.h>

#include "../include/cachemap.h"

static struct cachemap *cm;
static uint64_t npages;
static int per, stop;
static double *lat;
static long hits, usage_calls;

static double now(void) { struct timespec t; clock_gettime(CLOCK_MONOTONIC, &t); return t.tv_sec + 1e-9 * t.tv_nsec; }

static void *reader(void *arg) {
	const long k = (long)arg;
	uint64_t x = 0x9E3779B97F4A7C15ull * (uint64_t)(k + 1);
	long h = 0;
	for (int i = 0; i < per; i++) {
		x ^= x << 13; x ^= x >> 7; x ^= x << 17;
		const uint64_t p = x % npages;
		const double t0 = now();
		void *page = cachemap_get(cm, (p % 16) << 12, 1000 + p / 16, 0);
		lat[k * per + i] = now() - t0;
		if (page) { h++; free(page); }
	}
	__atomic_fetch_add(&hits, h, __ATOMIC_RELAXED);
	return NULL;
}

static void *scanner(void *arg) {
	(void)arg;
	struct cachemap_object_usage rows[16];
	while (!__atomic_load_n(&stop, __ATOMIC_ACQUIRE)) {
		if (cachemap_usage(cm, 16, rows) < 0) abort();
		usage_calls++;
	}
	return NULL;
}

static int cmp(const void *a, const void *b) {
	const double x = *(const double *)a, y = *(const double *)b;
	return x < y ? -1 : x > y;
}

int main(int argc, char **argv) {
	if (argc < 6) return 2;
	npages = strtoull(argv[2], NULL, 0);
	const int threads = atoi(argv[3]);
	per = atoi(argv[4]);
	const int with_usage = atoi(argv[5]);
	cm = cachemap_create(argv[1], 2 * npages, 12, 12);
	if (!cm) return 1;
	const uint64_t batch = 4096;
	uint8_t *pages = calloc(batch, 4096);
	uint64_t *off = calloc(batch, 8), *nh = calloc(batch, 8);
	uint32_t *gen = calloc(batch, 4);
	for (uint64_t at = 0; at < npages; at += batch) {
		const uint64_t m = npages - at < batch ? npages - at : batch;
		for (uint64_t i = 0; i < m; i++) {
			const uint64_t p = at + i;
			off[i] = (p % 16) << 12;
			nh[i] = 1000 + p / 16;
			memcpy(pages + i * 4096, &p, 8);
		}
		cachemap_put_batch(cm, m, off, nh, gen, pages);
	}
	struct cachemap_object_usage one;
	if (cachemap_usage(cm, 1, &one) < 0) return 1;      /* every put has landed */
	lat = calloc((size_t)threads * per, sizeof(double));
	pthread_t th[256], sc;
	if (with_usage) pthread_create(&sc, NULL, scanner, NULL);
	for (long k = 0; k < threads; k++) pthread_create(&th[k], NULL, reader, (void *)k);
	for (int k = 0; k < threads; k++) pthread_join(th[k], NULL);
	__atomic_store_n(&stop, 1, __ATOMIC_RELEASE);
	if (with_usage) pthread_join(sc, NULL);
	const size_t n = (size_t)threads * per;
	qsort(lat, n, sizeof(double), cmp);
	printf("{\"threads\": %d, \"usage_running\": %d, \"gets\": %zu, \"hits\": %ld, \"get_p50_us\": %.1f, "
	    "\"get_p99_us\": %.1f, \"usage_calls_meanwhile\": %ld}\n", threads, with_usage, n, hits,
	    lat[n / 2] * 1e6, lat[(size_t)(n * 0.99)] * 1e6, usage_calls);
	cachemap_free(cm);
	return 0;
}
