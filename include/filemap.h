/*
 * filemap.h — keyed page store, H100 edition.  Same seven entry points as the reference's
 * cachemap/filemap.h:19-29; behind them the 32 LMDB environments are replaced by one HBM key
 * table + record arena per GPU (include/cachemap_b200.h, DESIGN.md §2).
 *
 * struct filemap is opaque here: cachemap.c and the tests only ever hold the pointer.
 */
#ifndef FILEMAP_H
#define FILEMAP_H

#include <stdint.h>
#include "uint128.h"

#ifdef __cplusplus
extern "C" {
#endif

#define FILEMAP_SHARD_NUM	32      /* reference shard count; here only `key & 31` reporting */
#define FILEMAP_SHARD_FACTOR	1024    /* smallest legal `n` (reference filemap.c:51) */

struct filemap;

/* n = capacity in pages (>= FILEMAP_SHARD_FACTOR or NULL), compress_accel = LZ4 acceleration
 * (0 stores raw pages), pshift = log2(page bytes).  No GPU work happens here: the device is
 * initialised on the first set/get so that a daemon may fork() after creating the map
 * (edgefs.c:2114-2169). */
struct filemap *filemap_create(char *destdir, uint64_t n, int compress_accel, int pshift);
void filemap_free(struct filemap *m);

/* value: one page, borrowed for the call.  attr: the put timestamp kept for eviction. */
void filemap_set(struct filemap *m, uint128_t *key, void *value, uint64_t attr);
void filemap_unset(struct filemap *m, uint128_t *key);

/* Returns a malloc()ed page the caller frees, or NULL on a miss. */
void *filemap_get(struct filemap *m, uint128_t *key);

/* One live entry picked from a random point of the key space (1), or 0 when none. */
int filemap_get_rand(struct filemap *m, uint128_t *key, uint64_t *ts);

uint64_t filemap_entries(struct filemap *m);

#ifdef __cplusplus
}
#endif
#endif
