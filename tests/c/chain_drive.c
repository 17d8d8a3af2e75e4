/* Drives the drop-in's checkpoint policy over the stand-in of mock_chain.c: one thread puts a page every
 * 20 ms for S seconds while the CMB200_CHECKPOINT_SEC thread ticks, then cachemap_free.  Prints
 *   calls: <every snapshot call, in order>
 *   files: <the files the cache directory holds afterwards, sorted>
 * usage: chain_drive <cachedir> <seconds> */
#include <dirent.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <time.h>
#include <unistd.h>

#include "../../include/cachemap.h"

void mock_chain_log(char *out, size_t cap);

#define PSHIFT 12

static int cmp(const void *a, const void *b) { return strcmp(*(char *const *)a, *(char *const *)b); }

int main(int argc, char **argv) {
	if (argc < 3) { fprintf(stderr, "usage: %s cachedir seconds\n", argv[0]); return 2; }
	struct cachemap *cm = cachemap_create(argv[1], 1 << 16, 12, PSHIFT);
	if (!cm) { fprintf(stderr, "cachemap_create failed\n"); return 1; }
	uint8_t page[1 << PSHIFT];
	const long steps = (long)(atof(argv[2]) * 50);
	for (long i = 0; i < steps; i++) {
		memset(page, (int)i, sizeof(page));
		cachemap_put(cm, (uint64_t)(i % 512) << PSHIFT, 11, 1, page);
		usleep(20000);
	}
	cachemap_free(cm);
	static char log[16384];
	mock_chain_log(log, sizeof(log));
	printf("calls: %s\n", log);
	char *names[256];
	int n = 0;
	DIR *d = opendir(argv[1]);
	for (struct dirent *e; d && (e = readdir(d)) != NULL;)
		if (e->d_name[0] != '.' && n < 256) names[n++] = strdup(e->d_name);
	if (d) closedir(d);
	qsort(names, n, sizeof(names[0]), cmp);
	printf("files:");
	for (int i = 0; i < n; i++) printf(" %s", names[i]);
	printf("\n");
	return 0;
}
