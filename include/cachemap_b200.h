/*
 * cachemap_b200.h — C ABI of the H100 cachemap engine (batch extension + kernel-level entries).
 *
 * The drop-in surface is include/cachemap.h + include/filemap.h (same prototypes as the
 * reference's cachemap/cachemap.h:33-47 and cachemap/filemap.h:19-29).  This header is the layer
 * under it: batched put/get over many chunks per call (the reference's API moves one page per
 * call — edgefs.c:1165,1191,1224 — which cannot feed a GPU; SURVEY.md §7 H3), plus direct entry
 * points to the individual kernels so that parity tests can compare each one with the oracle.
 *
 * Plain C: pointers and sizes only, no CUDA or torch types.  "host" pointers may be pageable or
 * page-locked (cmb200_host_alloc gives page-locked memory; transfers from it run at full PCIe
 * rate).  "dev" pointers are device addresses in the engine's CUDA device.
 * All functions return 0 on success and -1 on failure unless stated; cmb200_last_error() then
 * describes the failure.  There is no CPU fallback anywhere: without a usable CUDA device every
 * entry point fails.
 */
#ifndef CACHEMAP_B200_H
#define CACHEMAP_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct cmb200_engine cmb200_engine;

/* 16-byte page address, {u = nhid_small, l = page | genid << 44} (cachemap/uint128.h:4,
 * cachemap/cachemap.c:151-166). */
typedef struct { uint64_t u; uint64_t l; } cmb200_addr;

#define CMB200_FINGERPRINT 1u   /* compute + keep the EF128 content fingerprint of every put */
/* Verified reads (implies CMB200_FINGERPRINT): every hit of cmb200_get_batch, cmb200_get_batch_dev,
 * cmb200_get_small and cmb200_get_small_begin / _end has its decoded page's EF128 compared on the GPU
 * with the fingerprint stored for that record version; a page that differs is answered
 * CMB200_CORRUPT instead of CMB200_HIT.  A hit whose record has no fingerprint (imported from another
 * rank, read from a peer's arena, or loaded from a snapshot written without fingerprints) is served
 * as CMB200_HIT and counted unverified.  See cmb200_verify_stats and cmb200_verify_store. */
#define CMB200_VERIFY 2u
/* Eviction by last access: every get of cmb200_get_small, cmb200_get_small_begin / _end, cmb200_get_batch
 * and cmb200_get_batch_dev that answers CMB200_HIT for a LOCAL record (in the arena or the host tier)
 * raises that record's timestamp attribute — the ts that cmb200_sample reports and eviction and demotion
 * compare — to a stamp taken when the get is launched: CLOCK_REALTIME_COARSE in ns, the clock the
 * reference's cachemap_put stamps with (cachemap.c:10-15).  The update is an atomic maximum, so ts never
 * goes backwards whichever of two gets lands first.  Without the flag ts is the put time, as in the
 * reference, and no get changes it.
 * Nothing else touches: misses, CMB200_BAD_ENTRY, _BAD_DECODE, _CORRUPT, _INVALID and _REMOTE answers, hits
 * served from a peer's arena (the slot is a replica; the owner's is in another process), and
 * cmb200_locate_batch, cmb200_read_records, cmb200_verify_store, cmb200_sample, snapshots, compaction,
 * demotion and promotion (which keep ts as it is).
 * The stamps compare only with put timestamps of the same clock: the drop-in's puts use it; an engine
 * level put with ts = NULL stores 0, older than any stamp.
 * Two races are benign, because ts is eviction metadata and never decides which bytes a get returns: a
 * touch that lands on a slot a put of the same key has just rewritten raises the new record's ts to about
 * now, and a touch that races a table rebuild may be lost. */
#define CMB200_TOUCH 4u

typedef struct cmb200_config {
	int device;             /* CUDA ordinal, -1 = current device */
	int pshift;             /* page shift: chunk = 1 << pshift bytes (edgefs -p, edgefs.c:2043-2048) */
	int accel;              /* LZ4 acceleration, 0 = store raw (cachemap_create comp_accel) */
	uint64_t capacity;      /* entries before eviction starts (cachemap_create capacity) */
	uint64_t arena_bytes;   /* HBM arena for records, 0 = sized from capacity and free memory */
	uint64_t table_slots;   /* key-table slots (power of two), 0 = 4 x capacity rounded up */
	uint32_t max_batch;     /* chunks per kernel launch, 0 = 4096 (host pages are pipelined in
	                         * steps of min(max_batch, 4096) chunks) */
	uint32_t flags;
} cmb200_config;

/* per-request result of a get */
enum {
	CMB200_MISS = 0,
	CMB200_HIT = 1,
	CMB200_INVALID = 2,     /* address rejected: not counted as a request (cachemap.c:173-174) */
	CMB200_BAD_ENTRY = 3,   /* key present under another address: a miss (filemap.c:236-240) */
	CMB200_BAD_DECODE = 4,  /* decoded length != stored length: a miss (filemap.c:244-248) */
	CMB200_REMOTE = 5,      /* multi-GPU: the newest record of this key lives on another rank */
	CMB200_CORRUPT = 6,     /* CMB200_VERIFY: the decoded page differs from the stored EF128: a miss.
	                         * The page is not written by cmb200_get_small; cmb200_get_batch(_dev) may
	                         * have written it, as for CMB200_BAD_DECODE. */
	CMB200_DROPPED = 7      /* cmb200_patch_batch: the patched page did not fit the arena */
};

const char *cmb200_last_error(void);
int cmb200_device_count(void);

cmb200_engine *cmb200_engine_create(const cmb200_config *cfg);
void cmb200_engine_destroy(cmb200_engine *e);

void *cmb200_host_alloc(size_t bytes);        /* page-locked host memory */
void cmb200_host_free(void *p);
void *cmb200_dev_alloc(cmb200_engine *e, size_t bytes);
void cmb200_dev_free(cmb200_engine *e, void *p);
int cmb200_memcpy_h2d(cmb200_engine *e, void *dev, const void *host, size_t bytes);
int cmb200_memcpy_d2h(cmb200_engine *e, void *host, const void *dev, size_t bytes);
void *cmb200_stream(cmb200_engine *e);        /* the engine's compute cudaStream_t, for event timing */
int cmb200_sync(cmb200_engine *e);

/* filemap_set for n chunks (cachemap/filemap.c:112-158): pages = n x (1<<pshift) bytes.
 * valid (nullable) = per-chunk flag, 0 skips the chunk (rejected address).  ts (nullable) = the
 * LMDB attribute.  Chunks are applied in array order: a later chunk with the same key wins.
 * lens_out (nullable, host) receives each stored compressed_length, or -1 for skipped chunks.
 * pages_dev (cmb200_put_batch_dev) must be 16-byte aligned, as cmb200_dev_alloc and cudaMalloc
 * memory is; any other pointer fails with -1 before anything is stored. */
int cmb200_put_batch(cmb200_engine *e, size_t n, const cmb200_addr *addr, const uint8_t *valid,
    const void *pages_host, const uint64_t *ts, int32_t *lens_out);
int cmb200_put_batch_dev(cmb200_engine *e, size_t n, const cmb200_addr *addr, const uint8_t *valid,
    const void *pages_dev, const uint64_t *ts, int32_t *lens_out);

/* Write-behind form of cmb200_put_batch, the batch analogue of cachemap_put_async
 * (cachemap/cachemap.c:199-216): returns as soon as addr / valid / pages_host / ts have crossed to
 * the device and may be reused by the caller, like the borrowed page of cachemap_put; the encode of
 * the last sub-batch completes behind *ticket.  Every later call on this engine (gets included)
 * is ordered after the put, so waiting is needed only before reading lens_out, which must then be
 * page-locked (cmb200_host_alloc) and stay valid until cmb200_wait(ticket) has returned.
 * Submitting batch k+1 before waiting for batch k overlaps its host-to-device copy with the tail
 * of batch k's encode. */
int cmb200_put_batch_async(cmb200_engine *e, size_t n, const cmb200_addr *addr, const uint8_t *valid,
    const void *pages_host, const uint64_t *ts, int32_t *lens_out, uint64_t *ticket);
int cmb200_wait(cmb200_engine *e, uint64_t ticket);

/* filemap_get for n requests (cachemap/filemap.c:217-262).  status_out[i] is one of CMB200_*;
 * pages_out receives 1<<pshift bytes per request (untouched for non-hits). */
int cmb200_get_batch(cmb200_engine *e, size_t n, const cmb200_addr *addr, const uint8_t *valid,
    void *pages_out_host, int32_t *status_out);
int cmb200_get_batch_dev(cmb200_engine *e, size_t n, const cmb200_addr *addr, const uint8_t *valid,
    void *pages_out_dev, int32_t *status_out);

/* filemap_unset (filemap.c:188-215), filemap_entries (filemap.c:316-330),
 * filemap_get_rand (filemap.c:264-314; policy-equivalent: first live record at or after r). */
int cmb200_unset_batch(cmb200_engine *e, size_t n, const cmb200_addr *addr);
/* Removes every live local record whose stored address has u == u and l_first <= l <= l_last
 * (one generation's pages p..q of one object: l = genid << 44 | page).  Unlike cmb200_unset_batch it
 * goes by stored address, never by key alone: a record of another address that shares a key stays.
 * Ordered after everything enqueued on the engine before the call, async puts included; runs under the
 * engine lock on its stream, as cmb200_unset_batch does.  A short interval is looked up page by page,
 * a long one by a scan of the table; both leave the same store.  Records of the host tier leave it as
 * if unset.  The table only changes, so a snapshot begun before the call still holds the records, and
 * the next delta of a chain names them as tombstones.  When the removals leave more than cap/8
 * tombstones the table is rebuilt, as cmb200_compact does.  *removed_out = records removed.  -1 if
 * l_first > l_last, or on an engine that has made a multi-GPU call (its index holds other ranks'
 * records). */
int cmb200_invalidate(cmb200_engine *e, uint64_t u, uint64_t l_first, uint64_t l_last, uint64_t *removed_out);
/* Moves every live local record stored at {u_from, l}, l_first <= l <= l_last, to {u_to, l} on engine
 * cmb200_owner(FNV(u_to, l), g), with the same block, ts and fingerprint (a fingerprint only where the
 * record had one for that version).  After a 0 return no record is stored at {u_from, l} in the interval on
 * any engine; each one that was is stored at {u_to, l}, byte for byte what a put of the same page there
 * stores, its parse checkpoints rebuilt as a load rebuilds them, or was dropped for lack of arena room
 * (counted in *dropped_out and in the `dropped` statistic, as a put is).  Only the moved pages' slots
 * change: a {u_to, l} whose key another address holds replaces that record as a put would; a key of the
 * interval that holds another object's address is left alone; the rest of u_to is not cleared (invalidate
 * it first).  Selection goes key by key or by a scan of the table on cmb200_invalidate's threshold.
 * The records move in slices (<= max_batch records, one page-ring buffer of bytes): under the source
 * engine's lock they are copied out and retired, then under the destination's lock they are stored,
 * after one compaction if the slice does not fit and garbage covers the shortfall; nothing is evicted or
 * demoted.  Ordered after everything enqueued on each engine before the call, async puts included; never
 * holds two engine locks at once, and one rename runs at a time.  Small gets on other streams may overlap
 * and get the right page or a miss.  Records of the host tier move into the arena; retired bytes become
 * garbage of their tier.  The next chain delta holds the moved records and tombstones for the old
 * addresses.  u_from == u_to: 0, nothing changes.  -1 if l_first > l_last, g < 1, the engines' page sizes
 * differ, or an engine has made a multi-GPU call (checked before anything changes). */
int cmb200_rename_set(cmb200_engine *const *engines, int g, uint64_t u_from, uint64_t u_to,
    uint64_t l_first, uint64_t l_last, uint64_t *moved_out, uint64_t *dropped_out);
/* cmb200_rename_set with g = 1 */
int cmb200_rename(cmb200_engine *e, uint64_t u_from, uint64_t u_to, uint64_t l_first, uint64_t l_last,
    uint64_t *moved_out, uint64_t *dropped_out);
/* Read-modify-write of stored pages.  Patch i writes len[i] >= 1 bytes at byte page_off[i] of the page
 * stored at addr[i] (page_off[i] + len[i] <= 1 << pshift).  bytes_host holds the patches' bytes back to
 * back in array order.  ts (nullable) as for cmb200_put_batch; a page patched more than once in the call
 * takes the ts of its last patch.  status_out[i]:
 *   CMB200_HIT        the new page (old page, patches applied) is stored, exactly as a put of it would
 *                     store it: same record bytes, fingerprint, parse checkpoints, ts, sequence
 *   CMB200_MISS       no record of addr[i]: nothing is stored (the rest of the page is unknown)
 *   CMB200_BAD_ENTRY  the key holds another address: nothing changes
 *   CMB200_BAD_DECODE / CMB200_CORRUPT   the stored record cannot be trusted: it is removed
 *   CMB200_DROPPED    the new record did not fit the arena: the old record is removed
 * After the call, a get of addr[i] returns the patched page or misses.  It never returns the old page.
 * Patches of one address in one call are applied in array order to one page and stored once; they all
 * get the same status.  Ordered after everything enqueued on the engine before the call, async puts
 * included; runs under the engine lock on its stream, as cmb200_invalidate does.  A concurrent
 * cmb200_get_small returns the old or the new page, never a mix.  A patch is a put, not a get: the get
 * counters, the verified-read counters, tier hits, the tier's hot log and CMB200_TOUCH stamps do not move;
 * put_chunks counts the pages stored.  A patched host-tier record is stored again in the arena and its
 * tier bytes become tier garbage.  -1 before anything is applied if an extent is out of the page or len
 * is 0, and on an engine that has made a multi-GPU call. */
int cmb200_patch_batch(cmb200_engine *e, size_t n, const cmb200_addr *addr, const uint32_t *page_off,
    const uint32_t *len, const void *bytes_host, const uint64_t *ts, int32_t *status_out);
uint64_t cmb200_entries(cmb200_engine *e);
int cmb200_sample(cmb200_engine *e, size_t n, const uint64_t *r, cmb200_addr *addr_out,
    uint64_t *ts_out, int32_t *ok_out);

/* Copies the stored record of each address — the bytes the reference keeps in LMDB:
 * 24-byte data_prefix + payload (filemap.c:9-12,140-147) — into out (stride bytes apart) and its
 * total length into len_out (-1 = absent). */
int cmb200_read_records(cmb200_engine *e, size_t n, const cmb200_addr *addr, void *out_host,
    size_t stride, int32_t *len_out);
/* EF128 of the stored records (engine created with CMB200_FINGERPRINT): fp_out[2i]=hi, [2i+1]=lo. */
int cmb200_read_fingerprints(cmb200_engine *e, size_t n, const cmb200_addr *addr, uint64_t *fp_out,
    int32_t *ok_out);

typedef struct cmb200_stats {
	uint64_t entries, table_slots, tombstones;
	uint64_t arena_bytes, arena_used, arena_garbage, dropped_puts;
	uint64_t remote_entries;  /* keys whose newest record is on another GPU (multi-GPU index) */
	uint64_t put_chunks, get_requests, get_hits, kernel_launches;
	/* summed CUDA-event durations of the encode / decode kernel launches (last 64 per call) */
	uint64_t encode_kernel_ns, encode_kernel_launches, decode_kernel_ns, decode_kernel_launches;
	uint64_t fingerprint_kernel_ns;
} cmb200_stats;
int cmb200_get_stats(cmb200_engine *e, cmb200_stats *out);

/* One put step of a sharded stream with everything that follows it kept on the device and
 * asynchronous.  Like cmb200_put_batch_async (pages on the host, pages_on_dev = 0), or with the
 * pages in page-locked host memory that the caller leaves untouched until the ticket is done
 * (pages_on_dev = 2: the call returns without waiting for its own copies, so the next step can be
 * queued behind them at once), or device resident (pages_on_dev = 1, same lifetime rule, and
 * 16-byte aligned as for cmb200_put_batch_dev),
 * and additionally writes one 32-byte exchange record per chunk — {u, l, global stream position,
 * rank << 56 | arena offset / 16 << 22 | stored length + 1 (0: nothing stored)} — to records_dev_out
 * (device memory, n x 32 bytes) on the engine's stream.  The caller all-gathers those records (NCCL,
 * on that stream) and hands the result to cmb200_import_records_dev, which imports the rows of the
 * other ranks into the index replica, again without a host round trip.  n <= 262144.
 * cmb200_import_records_dev reads n_total such records from device memory, skips the rows of my_rank
 * and the rows that stored nothing, and is asynchronous on the engine's stream.  The arena offset
 * lets cmb200_get_small read a record over NVLink once cmb200_open_peer has mapped its owner's arena. */
int cmb200_put_step(cmb200_engine *e, size_t n, const cmb200_addr *addr, const uint8_t *valid,
    const void *pages, int pages_on_dev, const uint64_t *ts, uint32_t rank, void *records_dev_out,
    int32_t *lens_out, uint64_t *ticket);
int cmb200_import_records_dev(cmb200_engine *e, size_t n_total, const void *records_dev, uint32_t my_rank);

/* Slides the live records to the start of the arena so that the space of deleted and outgrown
 * records (stats.arena_garbage, and the unused remainders of per-warp segments) can be allocated
 * again; *reclaimed_out = bytes by which stats.arena_used went down.  Blocks the engine while it
 * runs (HBM speed).  The cachemap layer calls it by itself when the arena is about to overflow.
 * While a snapshot's section of this engine is not written yet, it first waits for the writer
 * (cmb200_snapshot_begin). */
int cmb200_compact(cmb200_engine *e, uint64_t *reclaimed_out);

/* ---- snapshot: what makes the cache directory persistent (SURVEY.md §8 f3) --------------------
 * The reference's store is its LMDB files under <cachedir> (cachemap/filemap.c:57,71-72) and so
 * survives a restart.  cmb200_save writes every live local record — byte for byte the LMDB value
 * of the reference, 24-byte data_prefix + payload (filemap.c:140-147), with its timestamp
 * attribute and fingerprint — to one file (written to path.tmp, then renamed); cmb200_load puts
 * the records of such a file into the store as if they had been put in file order (existing keys
 * are overwritten).  The format (engine.cu) is independent of capacity and arena size; the page
 * size must match.  The file holds no parse checkpoints: cmb200_load rebuilds them from each LZ4
 * block, so a loaded record is read by cmb200_get_small as fast as a freshly put one (a block whose
 * token chain does not add up to the page gets none and is walked by one warp).
 * Both return 0 on success, -1 with cmb200_last_error() otherwise. */
int cmb200_save(cmb200_engine *e, const char *path, uint64_t *records_out);
int cmb200_load(cmb200_engine *e, const char *path, uint64_t *records_out);

/* ---- a store sharded by key over several engines (CMB200_DEVICES, one engine per listed GPU) -------
 * key = FNV-1a-64 of the 16 address bytes (FNV_hash in uint128.h; the key of filemap.c:18-24).  Of g
 * engines, the key belongs to engine cmb200_owner(key, g): the high 32 bits of the key scaled to g, so
 * the split is even for any g and independent of the low bits the reference's 32 shards use
 * (filemap.c:26-33).  This is the only definition; the drop-in and the snapshot code both call it.
 * (C99 inline: cachemap_api.c emits the external definition, so the library exports it as well.) */
inline int cmb200_owner(uint64_t key, int g) { return (int)(((key >> 32) * (uint64_t)g) >> 32); }

/* cmb200_save / cmb200_load over g engines that split the keys by cmb200_owner.  The file is the one
 * cmb200_save writes: one header, then the records of engine 0, 1, ...  Each engine's section is a
 * point-in-time copy of that engine (its records as they were when its list was taken, see
 * cmb200_snapshot_begin); the engines hold disjoint keys, so the union is a valid store.
 * cmb200_load_set reads the file once and puts each record into engine cmb200_owner(key, g), whatever g
 * the file was written with.  cmb200_save_set is cmb200_snapshot_begin followed by
 * cmb200_snapshot_finish; cmb200_save and cmb200_load are these calls with g = 1. */
int cmb200_save_set(cmb200_engine *const *engines, int g, const char *path, uint64_t *records_out);
int cmb200_load_set(cmb200_engine *const *engines, int g, const char *path, uint64_t *records_out);

typedef struct cmb200_snapshot cmb200_snapshot;
/* Starts a snapshot of g engines (the cmb200_save_set file, written to path.tmp).  Each engine is
 * locked only while its live records (both tiers) are listed, after its stream has been synchronised,
 * so every put enqueued before the call (asynchronous ones included) is in the list.  The listed
 * records are then written by a thread of the snapshot while the engines keep serving.  The file holds
 * exactly the records that were live when each engine's list was taken: puts, unsets, demotions and
 * promotions after that do not change it.  Until an engine's section is written, the two operations
 * that reuse record bytes (compaction, and a host-tier lap that overwrites records) wait for the
 * writer.  Nothing else waits.  A begin on an engine whose previous snapshot is still writing waits for
 * it.  Destroying an engine while a snapshot of it is open is a caller error, as destroying an engine
 * whose peers are mapped is.  An engine may appear once per call.
 * NULL on failure (cmb200_last_error); a failed begin leaves no file behind. */
cmb200_snapshot *cmb200_snapshot_begin(cmb200_engine *const *engines, int g, const char *path);
/* Waits for the writer, renames path.tmp to path (on failure removes it), frees s.  0 / -1. */
int cmb200_snapshot_finish(cmb200_snapshot *s, uint64_t *records_out);

/* ---- snapshot chains: checkpoints whose cost follows how much the store changed -------------------
 * A chain is a base, the cmb200_save_set file with a nonzero 64-bit chain id in header bytes 40..47
 * (zero in files written by cmb200_save_set), and deltas base_path.d1, .d2, ...  Delta k holds the
 * addresses that were live at tick k-1 and are not at tick k (tombstones), then every live local record
 * put between the two ticks, in the base's record format.  A record that only moved (compaction,
 * demotion, promotion, a table rebuild) is not in a delta.  The store a chain describes is the base,
 * then for each delta in order its tombstones removed and its records put.
 *
 * cmb200_chain_begin starts one tick over g engines, finished by cmb200_snapshot_finish, with the
 * contract of cmb200_snapshot_begin (engines locked only while listed, file written to .tmp and renamed,
 * the file holds the records as of begin).  delta = 0 writes a base at base_path with a fresh chain id.
 * delta = 1 writes the next delta of the chain whose base lies at base_path; it fails (NULL, error set)
 * unless every engine holds chain state for that base's id.  An engine holds chain state once a tick of
 * it has been finished successfully, or after a complete cmb200_load_chain; the state is that tick's
 * watermark (records put since have a higher sequence) and its live addresses, kept in page-locked host
 * memory.  Only one chain tick of an engine may be open at a time.
 *
 * cmb200_load_chain loads the base plus the longest run of deltas 1, 2, ... that are present, complete,
 * of the base's chain id and in sequence; the first that is not ends the run without failing the load,
 * and nothing after it is applied (*deltas_out = deltas applied, *records_out = records put).  Files are
 * read newest first and each address is decided by the newest file that names it, so each record is put
 * once.  Records route by cmb200_owner, so a chain written by any number of engines loads into g.  When
 * the engines were empty, every record the chain names is live afterwards and no base_path.d<j> lies
 * beyond the run (a missing or damaged delta ended it early), each engine takes chain
 * state from the load, so that the next delta tick continues the chain; otherwise none holds any and
 * the next tick must write a base.  Load before the engines serve.  0 / -1. */
cmb200_snapshot *cmb200_chain_begin(cmb200_engine *const *engines, int g, const char *base_path, int delta);
int cmb200_load_chain(cmb200_engine *const *engines, int g, const char *base_path, uint64_t *records_out,
    uint32_t *deltas_out);

/* Moves n pages of the engine's page size within the engine's device memory:
 * dst[dst_idx ? dst_idx[i] : i] = src[src_idx ? src_idx[i] : i] (one warp per page, 16-byte loads and
 * stores; dst and src 16-byte aligned and not overlapping; the index arrays are host memory).  Returns
 * when the pages have moved. */
int cmb200_move_pages(cmb200_engine *e, size_t n, void *dst_dev, const uint32_t *dst_idx, const void *src_dev,
    const uint32_t *src_idx);
/* Copies `bytes` from device memory of engine src_e to device memory of engine dst_e (one
 * cudaMemcpyPeerAsync; the two may be on the same GPU).  Returns when the bytes have arrived. */
int cmb200_copy_peer(cmb200_engine *dst_e, void *dst_dev, cmb200_engine *src_e, const void *src_dev, size_t bytes);

/* ---- host tier: records beyond the HBM arena ----------------------------------------------------
 * The reference keeps `capacity` pages in LMDB files on SSD; here the store is an HBM arena, which can
 * be far smaller than what `capacity` pages need.  A host tier is page-locked, device-mapped host
 * memory that holds records demoted from the arena, byte for byte in the same format (24-byte
 * data_prefix + payload).  Gets read them over PCIe and answer CMB200_HIT as for any record; keys,
 * records, statuses and counters do not depend on the tier a record is in.
 * cmb200_host_tier_enable allocates `bytes` of it: once, before the first put, and never on an engine
 * that has made a multi-GPU call (cmb200_set_stream_order, cmb200_put_step, cmb200_import_records_dev,
 * cmb200_arena_ipc_handle, cmb200_open_peer); those calls in turn fail on an engine with a tier.
 * cmb200_demote_batch moves the arena records of the named keys to the tier (*demoted_out = how many);
 * keys that are absent, remote or already in the tier are skipped.  Their arena bytes become
 * arena_garbage.  The tier is a ring in demotion order: when it comes round, the keys whose records
 * it overwrites are unset, an eviction like cmb200_unset_batch (retired_records).  A record leaves
 * the tier when it is unset, overwritten, retired or promoted back to the arena (cmb200_promote_batch).
 * A promoted record's tier bytes become tier garbage until the ring laps them; its key is not retired
 * then.  Promotion keeps the record's timestamp, which the eviction policy reads: the put time, or with
 * CMB200_TOUCH the last hit, tier hits included. */
struct cmb200_host_tier_stats {
	uint64_t bytes, used, records, garbage;     /* tier size; bytes between oldest and newest record; live records; dead bytes */
	uint64_t demoted_records, demoted_bytes;    /* moved from the arena so far (bytes = record lengths) */
	uint64_t retired_records;                   /* keys unset because the ring overwrote their records */
	uint64_t hits;                              /* gets answered from the tier */
	uint64_t promoted_records, promoted_bytes;  /* moved back to the arena so far (bytes = record lengths) */
};
int cmb200_host_tier_enable(cmb200_engine *e, uint64_t bytes);
int cmb200_demote_batch(cmb200_engine *e, size_t n, const cmb200_addr *addr, uint64_t *demoted_out);
/* all zero for an engine without a tier */
int cmb200_host_tier_stats(cmb200_engine *e, struct cmb200_host_tier_stats *out);
/* Moves the host-tier records of the named keys back into the HBM arena (*promoted_out = how many).
 * Keys that are absent, remote or already in the arena are skipped; a key named twice moves once.
 * Only free arena bytes are used: keys are taken in array order while their records fit between the
 * bump pointer and the end of the arena; the rest stay in the tier (no eviction, demotion or
 * compaction happens inside this call).  Keys, records, statuses and counters are unchanged. */
int cmb200_promote_batch(cmb200_engine *e, size_t n, const cmb200_addr *addr, uint64_t *promoted_out);
/* Addresses read from the host tier since the last call, newest first, distinct, at most max
 * (*n_out); *lost_out (nullable) = hits that the log overwrote before they were drained.  The engine
 * logs the last 4096 tier hits of cmb200_get_batch and cmb200_get_small in a device ring without a
 * lock, so an address may be stale; cmb200_promote_batch checks every address it is given.  Empty
 * for an engine without a tier. */
int cmb200_host_tier_hot(cmb200_engine *e, size_t max, cmb200_addr *addr_out, size_t *n_out, uint64_t *lost_out);

/* ---- multi-GPU: chunks sharded round-robin over ranks, one replicated key index per GPU ----
 * Each rank puts its own shard with the chunks' GLOBAL stream positions as sequence numbers
 * (next_seq = position of the rank's next chunk, stride = world size), then the ranks all-gather
 * {address, owner rank, sequence} of what they stored (NCCL, done by the caller) and import the
 * others' records: per key the highest sequence wins, exactly as sequential puts would resolve
 * (SURVEY.md §8e "ordering caveat"); a local record that loses is retired. */
int cmb200_set_stream_order(cmb200_engine *e, uint64_t next_seq, uint64_t stride);
/* The other ranks' arenas as NVLink peer memory.  Every rank exports the CUDA IPC handle of its
 * arena (64 bytes; exchange them with one all-gather), and opens the handles of the ranks it wants
 * to read from.  A cmb200_get_small of a key whose newest record lives on rank r then copies the
 * record straight out of rank r's arena (the location travelled with the exchange record) and
 * decodes it locally: replaces cachemap_get's LMDB read (cachemap.c:168-184, filemap.c:217-262) on
 * a box-global index.  Without a mapped peer such a get reports CMB200_REMOTE.  A location that no
 * longer holds the record (the owner compacted its arena since the exchange) is a miss. */
int cmb200_arena_ipc_handle(cmb200_engine *e, void *handle64_out, uint64_t *arena_bytes_out);
int cmb200_open_peer(cmb200_engine *e, uint32_t rank, const void *handle64, uint64_t arena_bytes);
/* Unmaps every peer arena (call on all ranks, then synchronise the ranks, before any of them
 * destroys its engine: an arena must not be freed while another process still maps it). */
int cmb200_close_peers(cmb200_engine *e);

/* Small batches of gets (cachemap_get from FUSE worker threads, n <= a few hundred): ONE fused
 * kernel per call — key lookup, record staged in shared memory by TMA, LZ4 decode shared -> shared,
 * page written with 16-byte stores — on a stream and a lock of its own, so a get neither waits for
 * a put batch in flight nor copies its result a second time: pages_out must be page-locked host
 * memory (cmb200_host_alloc; the kernel writes it directly) or device memory.  Records are
 * immutable and every rewrite goes to fresh arena space, so a get that overlaps a put of the same
 * key returns the old or the new page, never a mix (the reference's LMDB snapshot reads,
 * filemap.c:223-231).  Pages of 128 KiB (pshift 17) are decoded by a cluster of two CTAs per
 * request, record in one and page in the other, with the same contract.  Page sizes above 128 KiB
 * are not served by this call (-2): use cmb200_get_batch.  status_out as cmb200_get_batch. */
int cmb200_get_small(cmb200_engine *e, size_t n, const cmb200_addr *addr, void *pages_out, int32_t *status_out);

/* The same get in two halves, for callers that combine the requests of several threads into one
 * launch (the drop-in's combining queue, cachemap_api.c): begin (n <= 1024) launches and returns;
 * ticket.status[i] — page-locked host memory the kernel writes — holds CMB200_SMALL_PENDING until
 * request i is answered, and page i is complete in pages_out once its status is (read the status
 * with acquire semantics), so every requester can leave when ITS page is there instead of when
 * the slowest page of the batch is.  end waits for the rest, copies the statuses (status_out may
 * be NULL), books the statistics and releases the ticket's engine lane; it may be called from
 * another thread than begin, exactly once per successful begin. */
#define CMB200_SMALL_PENDING (-1)
typedef struct cmb200_small_ticket {
	int lane;                        /* engine lane the launch runs on, -1 = nothing in flight */
	uint32_t n;
	const volatile int32_t *status;
} cmb200_small_ticket;
int cmb200_get_small_begin(cmb200_engine *e, size_t n, const cmb200_addr *addr, void *pages_out, cmb200_small_ticket *ticket);
int cmb200_get_small_end(cmb200_engine *e, cmb200_small_ticket *ticket, int32_t *status_out);

/* ---- verified reads (CMB200_VERIFY) -------------------------------------------------------------
 * Counters of the engine's verified gets: hits whose page matched the stored EF128, hits without a
 * fingerprint for their record version, pages answered CMB200_CORRUPT; and of cmb200_verify_store:
 * records decoded by the scans so far, and those among them that failed.  All zero without the flag.
 * A call of its own rather than more fields of cmb200_stats, so that code built against an older
 * header keeps passing the struct size it knows. */
struct cmb200_verify_stats {
	uint64_t verified, unverified, corrupt;
	uint64_t scanned, scan_corrupt;
};
int cmb200_verify_stats(cmb200_engine *e, struct cmb200_verify_stats *out);
/* At-rest check of every live local record, in HBM and in the host tier, including records nobody
 * reads: each one is decoded on the GPU and its page compared with the stored EF128.  Runs on the
 * engine's stream under its lock, as cmb200_compact does, and repairs nothing.  *n_bad = records whose
 * page differs from its fingerprint or whose block does not decode; the first `max` of their addresses
 * go to bad_out (the caller may cmb200_unset_batch them).  *checked = records that had a fingerprint
 * to compare with; the others are unverified.  -1 for an engine created without CMB200_VERIFY. */
int cmb200_verify_store(cmb200_engine *e, size_t max, cmb200_addr *bad_out, size_t *n_bad, uint64_t *checked);

/* Lookup only: status_out[i] in CMB200_{MISS,HIT,BAD_ENTRY,REMOTE}; owner_out[i] = owning rank for
 * CMB200_REMOTE. */
int cmb200_locate_batch(cmb200_engine *e, size_t n, const cmb200_addr *addr, int32_t *status_out,
    uint64_t *owner_out);

/* ---- kernel-level entry points (parity tests, benchmarks); device = CUDA ordinal or -1 ---- */

/* cachemap.c:151-166 + filemap.c:18-24 on the device. */
int cmb200_compose_keys(int device, size_t n, const uint64_t *offset, const uint64_t *nhid,
    const uint32_t *genid, int pshift, cmb200_addr *addr_out, uint8_t *valid_out, uint64_t *key_out);

/* LZ4_compress_fast(page, dst, nbytes, nbytes+1024, accel) for n pages `stride` bytes apart
 * (stride multiple of 16); blocks_out rows are out_stride apart (>= nbytes + nbytes/255 + 16).
 * fp_out nullable: EF128 {hi,lo} per page from the same (fused) kernel. */
int cmb200_lz4_encode_batch(int device, const void *pages_host, size_t n, uint32_t nbytes,
    size_t stride, int accel, void *blocks_out_host, size_t out_stride, int32_t *lens_out,
    uint64_t *fp_out);
/* LZ4_decompress_fast(block, page, nbytes): consumed_out[i] = bytes consumed or < 0. */
int cmb200_lz4_decode_batch(int device, const void *blocks_host, size_t in_stride, const int32_t *lens,
    size_t n, uint32_t nbytes, void *pages_out_host, int32_t *consumed_out);
int cmb200_fingerprint_batch(int device, const void *pages_host, size_t n, uint32_t nbytes,
    size_t stride, uint64_t *fp_out);
/* EF128 of n pages resident in the engine's HBM (1<<pshift bytes each); fp_out on the host. */
int cmb200_fingerprint_dev(cmb200_engine *e, size_t n, const void *pages_dev, uint64_t *fp_out_host);
/* Parse checkpoints of the stored records: words_out[16 i + k] = word k (word 0 = tag as stored).
 * ok_out[i] = 1: the key's record is local and word 0 names its location and length;
 * 0: the key has a record without valid checkpoints; -1: absent, remote, or no side table. */
int cmb200_read_checkpoints(cmb200_engine *e, size_t n, const cmb200_addr *addr, uint32_t *words_out, int32_t *ok_out);

/* ---- synthetic streams (SURVEY.md §8d), same definition on host and device ---- */
void cmb200_gen_chunk_host(uint64_t seed, uint64_t cid, uint32_t bsize, void *out);
int cmb200_gen_chunks_dev(cmb200_engine *e, uint64_t seed, const uint64_t *cids_host, size_t n,
    void *out_dev);
/* cid[k] for a stream of n chunks with duplicate fraction dup (same-address repeats);
 * returns the number of distinct chunks. */
uint64_t cmb200_gen_stream_ids(uint64_t seed2, size_t n, double dup, uint64_t first_cid, uint64_t *cid_out);
void cmb200_gen_addr(uint64_t seed, uint64_t cid, int pshift, uint64_t *offset_out, uint64_t *nhid_out);

#ifdef __cplusplus
}
#endif
#endif
