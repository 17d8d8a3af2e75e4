/* Drives the drop-in's background load over the stand-in of mock_load.c (or mock_chain.c alone, which
 * has no background-load calls).  The cache directory must hold a base already.  The map is created and
 * one page is put and read back while the stand-in's first load step is held; then, by mode:
 *   ticks       hold the load for 2.5 s while CMB200_CHECKPOINT_SEC ticks, release it, put for 1.5 s more
 *   checkpoint  call cachemap_checkpoint on a thread while the load is held, release it after 0.5 s
 *   free        call cachemap_free on a thread while the load is held, release it after 0.5 s
 * then cachemap_free (unless the mode freed already).  Prints
 *   served: <1 if the put and the get returned, and the get hit, while the load was held>
 *   loading: <cachemap_load_progress during the hold> <loaded> <total>
 *   waited: <1 if the checkpoint / free thread had not returned before the release>
 *   calls: <every snapshot and load call, and the driver's marks, in order>
 * usage: load_drive <cachedir> <ticks|checkpoint|free> */
#include <pthread.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <unistd.h>

#include "../../include/cachemap.h"

void mock_chain_log(char *out, size_t cap);
#pragma weak mock_load_release
#pragma weak mock_log_mark
void mock_load_release(void);
void mock_log_mark(const char *what);

#define PSHIFT 12

static struct cachemap *cm;
static volatile int returned;

static void *checkpoint_thread(void *arg) { (void)arg; cachemap_checkpoint(cm); __atomic_store_n(&returned, 1, __ATOMIC_RELEASE); return NULL; }
static void *free_thread(void *arg) { (void)arg; cachemap_free(cm); __atomic_store_n(&returned, 1, __ATOMIC_RELEASE); return NULL; }

static void mark(const char *what) { if (mock_log_mark) mock_log_mark(what); }
static void release(void) { mark("release"); if (mock_load_release) mock_load_release(); }

int main(int argc, char **argv) {
	if (argc < 3) { fprintf(stderr, "usage: %s cachedir ticks|checkpoint|free\n", argv[0]); return 2; }
	const char *mode = argv[2];
	cm = cachemap_create(argv[1], 1 << 16, 12, PSHIFT);
	if (!cm) { fprintf(stderr, "cachemap_create failed\n"); return 1; }
	static uint8_t page[1 << PSHIFT];
	memset(page, 7, sizeof(page));
	cachemap_put(cm, 0, 11, 1, page);
	void *got = cachemap_get(cm, 0, 11, 1);
	const int hit = got && memcmp(got, page, sizeof(page)) == 0;
	free(got);
	uint64_t loaded = 0, total = 0;
	const int loading = cachemap_load_progress(cm, &loaded, &total);
	printf("served: %d\n", hit);
	printf("loading: %d %llu %llu\n", loading, (unsigned long long)loaded, (unsigned long long)total);
	int waited = 0, freed = 0;
	if (strcmp(mode, "ticks") == 0) {
		for (int i = 0; i < 125; i++) {          /* 2.5 s of puts while the load is held */
			memset(page, i, sizeof(page));
			cachemap_put(cm, (uint64_t)(i % 64) << PSHIFT, 11, 1, page);
			usleep(20000);
		}
		release();
		for (int i = 0; i < 75; i++) {
			memset(page, i, sizeof(page));
			cachemap_put(cm, (uint64_t)(i % 64) << PSHIFT, 11, 1, page);
			usleep(20000);
		}
		mark("end");
	} else {
		pthread_t th;
		pthread_create(&th, NULL, strcmp(mode, "free") == 0 ? free_thread : checkpoint_thread, NULL);
		usleep(500000);
		waited = !__atomic_load_n(&returned, __ATOMIC_ACQUIRE);
		release();
		pthread_join(th, NULL);
		freed = strcmp(mode, "free") == 0;
		mark("end");
	}
	printf("waited: %d\n", waited);
	if (!freed)
		cachemap_free(cm);
	static char log[16384];
	mock_chain_log(log, sizeof(log));
	printf("calls: %s\n", log);
	return 0;
}
