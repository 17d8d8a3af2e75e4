/* Drives the drop-in's CMB200_CHECKPOINT_SEC thread over the stand-in of mock_checkpoint.c, whose
 * cmb200_save_set sleeps for a second: T threads call cachemap_put back to back for S seconds (a small
 * write-behind ring stays busy throughout), each timing its slowest call.  Then cachemap_free.  Prints
 *   saves_during <saves begun while the puts ran> max_put_us <slowest cachemap_put> puts <calls>
 *   begun_before_free <saves begun before cachemap_free> begun_by_free <when it returned>
 *   ended_by_free <saves ended when it returned> saves_later <begun in the second after it>
 * usage: checkpoint_drive <cachedir> <threads> <seconds> */
#include <pthread.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <time.h>
#include <unistd.h>

#include "../../include/cachemap.h"

void mock_save_counts(int *started, int *done);

#define PSHIFT 12

static struct cachemap *cm;
static double seconds;
static uint64_t max_put_ns, put_calls;

static uint64_t now_ns(void) {
	struct timespec t;
	clock_gettime(CLOCK_MONOTONIC, &t);
	return (uint64_t)t.tv_sec * 1000000000ull + (uint64_t)t.tv_nsec;
}

static void *putter(void *arg) {
	const long t = (long)arg;
	uint8_t page[1 << PSHIFT];
	const uint64_t end = now_ns() + (uint64_t)(seconds * 1e9);
	uint64_t worst = 0, n = 0;
	for (uint64_t i = 0; now_ns() < end; i++, n++) {
		const uint64_t key = (uint64_t)t * 4096u + i % 4096u;
		memset(page, (int)(key + i), sizeof(page));
		const uint64_t t0 = now_ns();
		cachemap_put(cm, key << PSHIFT, 11, 1, page);
		const uint64_t dt = now_ns() - t0;
		if (dt > worst) worst = dt;
	}
	uint64_t cur = __atomic_load_n(&max_put_ns, __ATOMIC_RELAXED);
	while (worst > cur && !__atomic_compare_exchange_n(&max_put_ns, &cur, worst, 0, __ATOMIC_RELAXED, __ATOMIC_RELAXED))
		;
	__atomic_fetch_add(&put_calls, n, __ATOMIC_RELAXED);
	return NULL;
}

int main(int argc, char **argv) {
	if (argc < 4) { fprintf(stderr, "usage: %s cachedir threads seconds\n", argv[0]); return 2; }
	int threads = atoi(argv[2]);
	seconds = atof(argv[3]);
	if (threads < 1 || threads > 64) threads = 8;
	cm = cachemap_create(argv[1], 1 << 20, 12, PSHIFT);
	if (!cm) { fprintf(stderr, "cachemap_create failed\n"); return 1; }
	int begun0, begun1, begun2, begun3, ended;
	mock_save_counts(&begun0, &ended);
	pthread_t th[64];
	for (long t = 0; t < threads; t++) pthread_create(&th[t], NULL, putter, (void *)t);
	for (int t = 0; t < threads; t++) pthread_join(th[t], NULL);
	mock_save_counts(&begun1, &ended);
	cachemap_free(cm);
	mock_save_counts(&begun2, &ended);
	const int ended_by_free = ended;
	sleep(1);
	mock_save_counts(&begun3, &ended);
	printf("saves_during %d max_put_us %lu puts %lu begun_before_free %d begun_by_free %d ended_by_free %d saves_later %d\n",
	    begun1 - begun0, (unsigned long)(max_put_ns / 1000), (unsigned long)put_calls, begun1, begun2, ended_by_free,
	    begun3 - begun2);
	return 0;
}
