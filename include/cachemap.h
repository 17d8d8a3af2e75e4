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
 * With CMB200_ADMIT=freq, a page that would evict another is stored only if its key has been asked for
 * more often than the victim's, counted by every get the GPU looks up (cachemap_b200.h, CMB200_FREQ), so a
 * one-time scan of many pages does not flush the pages read often.  CMB200_ADMIT=all, the default, admits all.
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
 *
 * CMB200_LOAD says how that first call reads the file back.  "wait" (or unset): the call returns once
 * the whole store is in HBM.  "background": it starts the engines and returns; a thread loads the file
 * in steps while the map serves.  A page not loaded yet is a miss, and the file never overrides a change
 * made since the restart: a get returns either the page that loading the whole file first and then
 * making every later call would leave, or a miss (cmb200_load_open in cachemap_b200.h).  While the load
 * runs, checkpoint ticks are skipped; cachemap_checkpoint and cachemap_free wait for the load to end and
 * then write a base.  If the engine cannot load in steps, the call waits as with "wait".  Any other
 * value warns and waits.
 *
 * CMB200_KEY_FILE=<path> encrypts the directory at rest: a file of 32 raw bytes or 64 hex digits, read
 * once when the engines start (after any fork) and set on every engine (cmb200_set_file_key).  Every
 * file the map writes is then sealed with ChaCha20-Poly1305, and a plaintext directory still loads (the
 * next file written is sealed).  If the variable is set and the file is missing, unreadable or
 * malformed, the map warns on stderr and runs without persistence: it neither reads nor writes the
 * directory.  If the directory's base is sealed and does not load (no key, another key, a damaged
 * file), the map warns, starts empty and never writes the directory, not even at cachemap_free, so
 * that the sealed file stays as it was for a restart with the right key.  Records whose tag fails are
 * left out and counted (cmb200_load_rejected); the rest loads.
 */
int cachemap_checkpoint(struct cachemap *cm);
/* 1 while a background load runs (*loaded = records stored so far, *total = records the files hold by
 * their headers, an upper bound), 0 otherwise. */
int cachemap_load_progress(struct cachemap *cm, uint64_t *loaded, uint64_t *total);

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

/*
 * Rename.  edgefs_rename has the server copy `from` to `to` and delete `from`, after which `to` holds
 * exactly the bytes `from` held; the file system calls this at that point (INTEGRATION.md, "Invalidation")
 * with the nhid_small of each name.  Every cached page of `to` for genid is dropped, then every cached
 * page of `from` moves to `to` on the GPU, without a decode or an encode; afterwards no page of `from` is
 * cached.  Pages accepted by cachemap_put before the call are part of it.  A page the store has no room
 * for is dropped; if the engine cannot move pages at all, the pages of `from` are dropped instead, so that
 * nothing is served stale under either name.  Returns the pages moved.  The change counts for the next
 * checkpoint.
 */
uint64_t cachemap_rename(struct cachemap *cm, uint64_t nhid_from, uint64_t nhid_to, uint32_t genid);

/*
 * Pins.  A pinned page is never evicted (by count or by arena bytes), never paired as a victim by
 * admission and never demoted to the host tier: every victim the map draws comes from a sampler that
 * passes over pinned pages (cmb200_sample).  Under CMB200_ADMIT=freq a put of a pinned page is always
 * admitted.  A pin names stored addresses {nhid_small, genid << 44 | page}, as cachemap_invalidate does,
 * not keys: another object's page that shares a page's key is not pinned.  It holds whether the page is
 * cached now or put later.  A pinned page still leaves when it is unset, invalidated, renamed away or
 * over, and when a put or a patch of it finds no arena room, which happens only when pinned pages fill
 * the arena, or when a background load (which never evicts) finds no room for it.
 * Pins the pages of object (nhid_small, genid) that overlap bytes [off, off + size), partial pages at
 * both ends included.  Returns the pages newly pinned (already pinned ones are not counted again), or -1,
 * pinning nothing, when size is 0 or CACHEMAP_TO_END, when the first page does not fit 44 bits, when the
 * map's pinned pages would exceed CMB200_PIN_MAX, or when the pins would need more than CMB200_PIN_RANGES
 * disjoint ranges.  CMB200_PIN_MAX counts pages over the whole map: capacity / 4 by default, at most
 * capacity / 2 (a larger value warns and is clamped), 0 = no pins.  Pinned records already in the host
 * tier go back to HBM as far as free arena bytes hold them; the rest stay in the tier, counted in
 * *in_tier, where a lap of the tier's ring may retire them before a later pin call moves them.
 * Pins survive a restart in destdir/cachemap_b200.pins (sealed under CMB200_KEY_FILE; nothing is read or
 * written with CMB200_PERSIST=0), read before any snapshot record is loaded.  cachemap_invalidate leaves
 * pins alone, so a truncated file that is written again stays pinned; cachemap_rename drops the pins of
 * `to` and moves those of `from` to `to` before it moves the pages.
 */
int64_t cachemap_pin(struct cachemap *cm, uint64_t nhid_small, uint32_t genid, uint64_t off, uint64_t size);
/* Unpins the pages overlapping [off, off + size); CACHEMAP_TO_END is allowed.  Returns the pages
 * unpinned; 0, unpinning nothing, when the pins would need more than CMB200_PIN_RANGES ranges. */
uint64_t cachemap_unpin(struct cachemap *cm, uint64_t nhid_small, uint32_t genid, uint64_t off, uint64_t size);
/* pinned = pages named by pins; in_hbm / in_tier = pinned pages cached in the arena / the host tier. */
void cachemap_pin_stats(struct cachemap *cm, uint64_t *pinned, uint64_t *in_hbm, uint64_t *in_tier);

/*
 * What the cache holds, read off the key table on the GPU (DESIGN.md §2, *Usage and residency*).
 * Both calls answer for every page cachemap_put accepted before the call (the write-behind rings are
 * drained first), and count only records stored on this map's engines, in HBM or in the host tier.
 * A page not loaded yet by a CMB200_LOAD=background load is not cached, as a get would answer.  A call
 * before the first get starts the engines and answers for the loaded snapshot, as cachemap_invalidate
 * does.  Neither call changes anything else: the request and hit counters, the frequency sketch, ghost
 * entries, record timestamps, the host tier's hot log and promotion, and the checkpoint change count all
 * stay as they were.  A small get that touches a record (CMB200_EVICT=access) while a usage scan runs may
 * or may not show in newest_ts: the benign race of touches (cmb200_get_small).
 *
 * cachemap_residency: vec gets one byte per page of object (nhid_small, genid) that overlaps bytes
 * [off, off + size), partial pages at both ends included, as cachemap_pin counts them: CACHEMAP_IN_HBM or
 * CACHEMAP_IN_TIER if the page is cached, 0 if it is not, with CACHEMAP_PINNED ORed in when the address is
 * pinned, cached or not.  Returns the pages cached, or -1, leaving vec untouched, when size is 0 or
 * CACHEMAP_TO_END, when the first or the last page does not fit 44 bits, or when an engine cannot answer.
 *
 * cachemap_usage: returns the number of objects (nhid_small, genid) with at least one cached page, or -1
 * if any engine cannot answer (nothing partial is returned).  out gets the first min(max, count) of them
 * ordered by stored_bytes descending, then nhid_small ascending, then genid ascending; max = 0 counts
 * only.
 */
#define CACHEMAP_IN_HBM  1u
#define CACHEMAP_IN_TIER 2u
#define CACHEMAP_PINNED  4u
int64_t cachemap_residency(struct cachemap *cm, uint64_t nhid_small, uint32_t genid, uint64_t off, uint64_t size,
    uint8_t *vec);

struct cachemap_object_usage {
	uint64_t nhid_small;
	uint32_t genid, reserved;          /* reserved = 0 */
	uint64_t pages;                    /* cached pages: HBM + host tier */
	uint64_t tier_pages;               /* of those, in the host tier */
	uint64_t pinned_pages;             /* of those, at pinned addresses */
	uint64_t stored_bytes;             /* sum of record lengths: 24-byte prefix + LZ4 block or raw page */
	uint64_t first_page, last_page;    /* lowest / highest cached page number */
	uint64_t oldest_ts, newest_ts;     /* lowest / highest record ts (put time, or last hit under CMB200_EVICT=access) */
};
int64_t cachemap_usage(struct cachemap *cm, size_t max, struct cachemap_object_usage *out);

/* requests / hits counters (cachemap.c:176,181) and the engine under the map. */
void cachemap_get_counters(struct cachemap *cm, uint64_t *requests, uint64_t *hits);
/* CMB200_ADMIT=freq: pages admitted over the victim they were paired with, and pages rejected (not stored,
 * their key unset) since cachemap_create.  Both 0 without admission. */
void cachemap_get_admission(struct cachemap *cm, uint64_t *admitted, uint64_t *rejected);
/* CMB200_GHOST=1: for each extra_pages[i], would_hit[i] = the GPU misses since cachemap_create that a map of
 * capacity + extra_pages[i] pages would have served, estimated from the refault distances of evicted pages
 * (cmb200_ghost_stats); *misses (nullable) = the GPU misses looked up.  It counts only the refaults whose
 * distance lies below extra_pages[i] / G (G engines) rounded down to a bucket of the ghost table; that
 * rounding, ghosts displaced from a full set, and renames make it low.  The eviction policy can make it high:
 * under random oldest-of-three eviction a page read in a cycle that refaulted at distance d often would not
 * have lasted d more evictions in the larger map either, and on such a workload the curve overestimates the
 * hit ratio by up to 0.24 (DESIGN.md §2, *Ghost entries*).  -1 without CMB200_GHOST. */
int cachemap_hit_curve(struct cachemap *cm, size_t n, const uint64_t *extra_pages, uint64_t *would_hit,
    uint64_t *misses);
struct cmb200_engine *cachemap_engine(struct cachemap *cm);
/* Every engine under the map, in CMB200_DEVICES order (cachemap_engine is out[0]): stores up to max
 * of them in out and returns how many there are, 0 if none could be started.  Like cachemap_engine,
 * returns after every accepted put is in its engine. */
int cachemap_engines(struct cachemap *cm, struct cmb200_engine **out, int max);

#ifdef __cplusplus
}
#endif
#endif
