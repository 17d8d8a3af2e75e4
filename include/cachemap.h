/*
 * cachemap.h — L2 page cache front end, H100 edition.  Drop-in for the reference's
 * cachemap/cachemap.h:33-47: the same six functions with the same meaning, so edgefs.c's
 * FUSE read()/write() callbacks (edgefs.c:1165,1191,1224) and its cachemap_create call
 * (edgefs.c:2115) compile and link against this library unchanged.
 *
 * Behaviour kept from the reference (SURVEY.md §8b):
 *   - cachemap_create returns NULL unless destdir is an existing directory and
 *     capacity >= 1024 pages;
 *   - cachemap_get returns a malloc()ed page of 1<<pshift bytes that the caller free()s, or NULL;
 *     `requests` counts only valid addresses, `hits` counts non-NULL returns;
 *   - cachemap_put borrows `page` for the duration of the call (it is copied into a page-locked
 *     write-behind ring before the call returns; a get that follows returns it from there until
 *     the batch it belongs to is in the GPU store); cachemap_put_async is the same call;
 *   - a page number that does not fit 44 bits is ignored (put) / NULL without counting (get);
 *   - no error codes: any internal failure is a dropped put or a miss.
 * New: all calls are thread-safe, and concurrent callers are combined into one GPU batch.
 * With CMB200_VERIFY=1 in the environment every engine checks each page it serves against the
 * page's stored EF128 fingerprint (cachemap_b200.h, CMB200_VERIFY): a page that differs is a miss,
 * counted in `requests` and not in `hits`, so the caller fetches and puts it again.
 * With CMB200_EVICT=access, eviction (and demotion into a host tier) takes the pages read least
 * recently instead of those put longest ago: every page a get serves has its timestamp raised to the time
 * of the get (cachemap_b200.h, CMB200_TOUCH).  CMB200_EVICT=put, the default, is the reference's policy.
 * struct cachemap is opaque (edgefs.c never looks inside it).
 */
#ifndef CACHEMAP_H
#define CACHEMAP_H

#include <stdint.h>
#include "filemap.h"

#ifdef __cplusplus
extern "C" {
#endif

#define PUT_THREADS	4       /* reference async worker count; here one write-behind flusher */

struct cachemap;

struct cachemap *cachemap_create(char *destdir, uint64_t capacity, int comp_accel, int pshift);
void cachemap_free(struct cachemap *cm);

void *cachemap_get(struct cachemap *cm, uint64_t offset, uint64_t nhid_small, uint32_t genid);
void cachemap_put(struct cachemap *cm, uint64_t offset, uint64_t nhid_small, uint32_t genid,
    const void *page);
void cachemap_put_async(struct cachemap *cm, uint64_t offset, uint64_t nhid_small, uint32_t genid,
    const void *page);

void cachemap_print_stats(struct cachemap *cm);

/* ---- batch extension (not in the reference): n pages per call, see cachemap_b200.h ---- */

/* pages: n x (1<<pshift) bytes, host memory.  Equivalent to n cachemap_put calls in order. */
void cachemap_put_batch(struct cachemap *cm, uint64_t n, const uint64_t *offset,
    const uint64_t *nhid_small, const uint32_t *genid, const void *pages);
/* pages_out: n x (1<<pshift) bytes; hit_out[i] = 1 and the page is filled on a hit, else 0.
 * Counts requests / hits like n cachemap_get calls. */
void cachemap_get_batch(struct cachemap *cm, uint64_t n, const uint64_t *offset,
    const uint64_t *nhid_small, const uint32_t *genid, void *pages_out, uint8_t *hit_out);
/* Same with the pages resident in HBM (device pointers of the cachemap's GPU). */
void cachemap_put_batch_dev(struct cachemap *cm, uint64_t n, const uint64_t *offset,
    const uint64_t *nhid_small, const uint32_t *genid, const void *pages_dev);
void cachemap_get_batch_dev(struct cachemap *cm, uint64_t n, const uint64_t *offset,
    const uint64_t *nhid_small, const uint32_t *genid, void *pages_out_dev, uint8_t *hit_out);

/*
 * ---- request-range calls: the page loops of the FUSE callbacks as one call -----------------
 * edgefs_read (edgefs.c:1159-1178) walks the pages of a request with cachemap_get and gives up at
 * the first miss; its miss path and edgefs_write (edgefs.c:1183-1195, 1216-1228) put every page
 * of the request.  These two calls do the same for a whole request at once — the gets as ONE GPU
 * batch — after applying the gate of edgefs.c:192-203 (both ends page-aligned, see
 * edgefs_glue.h).
 *
 * cachemap_read_range: returns 1 and fills out_buf[0..size) when the range passes the gate and
 * every page hits; returns 0 otherwise (out_buf contents are then unspecified, as after the
 * reference's partial loop).  requests / hits advance exactly as the reference's loop advances
 * them: pages after the first miss are not counted.  size 0 returns 1 (the loop body never runs).
 * cachemap_write_range: puts every page of the range if it passes the gate, else does nothing.
 */
int cachemap_read_range(struct cachemap *cm, uint64_t nhid_small, uint32_t genid, uint64_t off,
    size_t size, void *out_buf);
void cachemap_write_range(struct cachemap *cm, uint64_t nhid_small, uint32_t genid, uint64_t off,
    size_t size, const void *data);

/*
 * Any byte range [off, off + size) of object (nhid_small, genid), for requests whose ends are not
 * page-aligned (INTEGRATION.md).
 * cachemap_pread: 1 and out_buf[0..size) filled when every page overlapping the range hits (ring or
 * store), else 0.  requests / hits advance over those pages as cachemap_read_range's do (page order,
 * stop at the first miss).  An aligned range behaves exactly as cachemap_read_range; size 0 returns 1.
 * cachemap_pwrite: pages the range covers whole are put (cachemap_put).  A page it covers in part is
 * patched if it is cached (on the GPU, cmb200_patch_batch: only the written bytes cross PCIe), and left
 * uncached otherwise.  Afterwards no get returns the page's old bytes.  Concurrent writes of disjoint
 * bytes of one page all land.  An aligned range behaves exactly as cachemap_write_range.
 */
int cachemap_pread(struct cachemap *cm, uint64_t nhid_small, uint32_t genid, uint64_t off, size_t size,
    void *out_buf);
void cachemap_pwrite(struct cachemap *cm, uint64_t nhid_small, uint32_t genid, uint64_t off, size_t size,
    const void *data);

/*
 * Persistence.  The reference's cache survives a restart because its store is a set of LMDB files
 * in destdir (cachemap/filemap.c:57,71-72).  Here the store is in HBM: it is written to
 * destdir/cachemap_b200.snap by cachemap_free, by cachemap_checkpoint, and every
 * CMB200_CHECKPOINT_SEC seconds if that variable is set (edgefs never calls cachemap_free), and
 * read back on the first put/get after cachemap_create on the same directory
 * (CMB200_PERSIST=0 turns all of it off).  Returns 0 when a snapshot was written.
 */
int cachemap_checkpoint(struct cachemap *cm);

/*
 * Invalidation.  The key of a page is its object's nhid_small and generation plus the page number,
 * so a file that is replaced (rename over it), deleted and created again under the same name, or
 * truncated, would be served its old pages; the file system calls this at those points
 * (INTEGRATION.md, "Invalidation").
 * Drops every cached page of object (nhid_small, genid) that overlaps bytes [off, off + size);
 * size = CACHEMAP_TO_END (UINT64_MAX) drops every page from off on.  Partial pages at either end are
 * dropped.  Pages accepted by cachemap_put before the call are dropped; pages put after it returns
 * are kept.  Returns the pages removed.  A removal counts as a change for the next checkpoint, so a
 * restart does not bring the pages back.
 */
#define CACHEMAP_TO_END UINT64_MAX
uint64_t cachemap_invalidate(struct cachemap *cm, uint64_t nhid_small, uint32_t genid, uint64_t off, uint64_t size);

/* requests / hits counters (cachemap.c:176,181) and the engine under the map. */
void cachemap_get_counters(struct cachemap *cm, uint64_t *requests, uint64_t *hits);
struct cmb200_engine *cachemap_engine(struct cachemap *cm);
/* Every engine under the map, in CMB200_DEVICES order (cachemap_engine is out[0]): stores up to max
 * of them in out and returns how many there are, 0 if none could be started.  Like cachemap_engine,
 * returns after every accepted put is in its engine. */
int cachemap_engines(struct cachemap *cm, struct cmb200_engine **out, int max);

#ifdef __cplusplus
}
#endif
#endif
