/* cachemap_put of 64 KiB pages from T native threads for S seconds, against any libcachemap.so loaded
 * by path: the drop-in's put rate with and without CMB200_CHECKPOINT_SEC (tools/snapshot_bench.py).
 * Each thread rewrites its own 2048 keys round after round, so the store stays at a fixed size.
 *   checkpoint_puts <libcachemap.so> <cachedir> <pages.bin> <threads> <seconds>
 * Prints one JSON line. */
#include <dlfcn.h>
#include <pthread.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <time.h>
#include <unistd.h>

#define CH 65536
#define KEYS_PER_THREAD 2048
typedef void *(*create_fn)(const char *, uint64_t, int, int);
typedef void (*put_fn)(void *, uint64_t, uint64_t, uint32_t, void *);
typedef void (*free_fn)(void *);

static put_fn f_put;
static void *cm;
static uint8_t *pages;
static int npages;
static double seconds;
static uint64_t calls, worst_ns;

static uint64_t now_ns(void) { struct timespec t; clock_gettime(CLOCK_MONOTONIC, &t); return (uint64_t)t.tv_sec * 1000000000ull + (uint64_t)t.tv_nsec; }

static void *worker(void *arg) {
	const long t = (long)arg;
	const uint64_t end = now_ns() + (uint64_t)(seconds * 1e9);
	uint64_t n = 0, worst = 0;
	while (now_ns() < end) {
		const uint64_t k = (uint64_t)t * KEYS_PER_THREAD + n % KEYS_PER_THREAD;
		const uint64_t t0 = now_ns();
		f_put(cm, k << 16, 0x78, 0, pages + ((k + n / KEYS_PER_THREAD) % (uint64_t)npages) * CH);
		const uint64_t dt = now_ns() - t0;
		if (dt > worst) worst = dt;
		n++;
	}
	__atomic_fetch_add(&calls, n, __ATOMIC_RELAXED);
	uint64_t cur = __atomic_load_n(&worst_ns, __ATOMIC_RELAXED);
	while (worst > cur && !__atomic_compare_exchange_n(&worst_ns, &cur, worst, 0, __ATOMIC_RELAXED, __ATOMIC_RELAXED))
		;
	return NULL;
}

int main(int argc, char **argv) {
	if (argc < 6) { fprintf(stderr, "usage: %s lib cachedir pages.bin threads seconds\n", argv[0]); return 2; }
	void *h = dlopen(argv[1], RTLD_NOW | RTLD_LOCAL);
	if (!h) { fprintf(stderr, "%s\n", dlerror()); return 1; }
	create_fn f_create = (create_fn)dlsym(h, "cachemap_create");
	free_fn f_free = (free_fn)dlsym(h, "cachemap_free");
	f_put = (put_fn)dlsym(h, "cachemap_put");
	FILE *f = fopen(argv[3], "rb");
	if (!f) { perror(argv[3]); return 1; }
	fseek(f, 0, SEEK_END); long sz = ftell(f); fseek(f, 0, SEEK_SET);
	npages = (int)(sz / CH);
	pages = malloc((size_t)sz);
	if (fread(pages, 1, (size_t)sz, f) != (size_t)sz) return 1;
	fclose(f);
	int threads = atoi(argv[4]);
	seconds = atof(argv[5]);
	if (threads < 1 || threads > 256) threads = 8;
	cm = f_create(argv[2], 1 << 16, 12, 16);
	if (!cm) { fprintf(stderr, "cachemap_create failed\n"); return 1; }
	f_put(cm, 1ull << 40, 1, 0, pages);              /* engine start outside the clock */
	pthread_t th[256];
	const uint64_t t0 = now_ns();
	for (long t = 0; t < threads; t++) pthread_create(&th[t], NULL, worker, (void *)t);
	for (int t = 0; t < threads; t++) pthread_join(th[t], NULL);
	const double el = (double)(now_ns() - t0) * 1e-9;
	printf("{\"threads\": %d, \"seconds\": %.2f, \"put_gibs\": %.3f, \"put_kops\": %.1f, \"max_put_ms\": %.2f}\n", threads, el,
	    (double)calls * CH / el / (1 << 30), (double)calls / el / 1e3, (double)worst_ns * 1e-6);
	fflush(stdout);
	f_free(cm);
	return 0;
}
