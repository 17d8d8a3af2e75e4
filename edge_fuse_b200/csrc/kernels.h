// kernels.h — launch interface between the engine (host C++) and the sm_90a kernels.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace cmb {

// One record of the HBM key table (64 bytes).  Replaces the reference's LMDB B+tree entry:
// key = FNV-1a-64 of the 16 address bytes (cachemap/filemap.c:18-24), one record per key
// (mdb_put_attr overwrite, filemap.c:143), attr = put timestamp (filemap.c:143, cachemap.c:195).
struct Slot {
	unsigned long long key;      // 0 = never used, ~0 = deleted; those two key values live in side slots
	unsigned long long addr_u;   // stored address, verified on get (filemap.c:236-240)
	unsigned long long addr_l;
	unsigned long long rec_off;  // location of {24-byte data_prefix, payload} (filemap.c:140-147): arena
	                             // offset, or REC_HOST | offset in the host tier
	uint32_t vlen;               // 0 = no valid record, else compressed_length + 1 (0+1 = raw page)
	uint32_t alloc;              // bytes reserved at rec_off (arena or host tier)
	unsigned long long ts;       // LMDB node attribute of the reference
	unsigned long long seq;      // stream order of the last put that claimed this key
	unsigned long long owner;    // 0 = record (if any) is in this GPU's arena; r+1 = key last written on rank r
};
static_assert(sizeof(Slot) == 64, "slot layout");

constexpr unsigned long long KEY_EMPTY = 0ull;
constexpr unsigned long long KEY_TOMB = ~0ull;

// Bit 63 of Slot::rec_off: the record lives in the host tier (page-locked, device-mapped host memory)
// at offset rec_off & ~REC_HOST, in the same format as in the arena.  A record moves between the
// tiers by one 8-byte store of rec_off: to the host tier by cmb200_demote_batch, back to the arena by
// cmb200_promote_batch.
constexpr unsigned long long REC_HOST = 1ull << 63;

// The log of host-tier hits: a ring of the last HOT_LOG_N addresses {u, l} that a get answered from the
// tier, appended by k_decode / k_get_small / k_get_small_pair (slot = atomicAdd(head, 1) % HOT_LOG_N,
// one 16-byte store) and drained by cmb200_host_tier_hot.
constexpr uint32_t HOT_LOG_N = 4096;
struct HotLog {
	unsigned long long *head;     // appends so far (64-bit, never wraps)
	ulonglong2 *ring;             // HOT_LOG_N entries {u, l}
};

struct TableView {
	Slot *slots;                 // cap + 2 entries; [cap] holds key 0, [cap+1] holds key ~0
	uint64_t cap;                // power of two
	unsigned long long *entries; // live records
	unsigned long long *tombs;   // deleted main-table slots (rebuild trigger)
	unsigned long long *remote;  // keys whose newest record lives on another GPU
	uint64_t *fp;                // optional, 2 x u64 per slot {hi, lo}
	uint32_t *ckpt;              // optional, CKPT_WORDS per slot: parse checkpoints of the slot's record
	uint32_t *fp_tag;            // CMB200_VERIFY only, one per slot: ckpt_tag of the record version fp
	                             // belongs to (0 = none); gets compare a page with fp only under it
};

// Parse checkpoints (lz4_decode_cta.cuh): word 0 = tag naming the record version (0 = none), word k
// (1..15) = where the first LZ4 sequence at or after k/16 of the page starts:
// block offset << CKPT_POS_BITS | (output position - k * n/16), or ~0 when no sequence starts in
// that sixteenth.  Written by the encoder (kernels.cu:ckpt_store), read by k_get_small.
constexpr uint32_t CKPT_WORDS = 16;
constexpr uint32_t CKPT_POS_BITS = 13;       // n/16 <= 8192 for pages up to 128 KiB
// Bit 30 of the tag is the record's tier, so a tag never names a record in the other tier.
__host__ __device__ inline uint32_t ckpt_tag(unsigned long long rec_off, uint32_t clen) {
	return 0x80000000u | ((uint32_t)(rec_off >> 33) & 0x40000000u) |
	    (((uint32_t)(rec_off >> 4) ^ (clen * 0x9E3779B1u)) & 0x3fffffffu);
}

#define ARENA_SEG_SLOTS 4096u    // resident encoder warps that can own an arena segment

struct ArenaView {
	uint8_t *base;
	uint64_t size;
	unsigned long long *head;     // bump pointer
	unsigned long long *garbage;  // bytes orphaned by relocated / deleted records
	unsigned long long *dropped;  // puts dropped because the arena was full (filemap.c:154-157 analogue)
	unsigned long long *tier;     // host tier: [0] = garbage bytes, [1] = live records
	// direct encode (large arenas): every resident encoder warp owns a segment of the arena and
	// writes blocks straight into it; seg[2w] = cursor, seg[2w+1] = end of warp slot w's segment
	unsigned long long *seg;
	uint32_t seg_bytes;           // segment size, 0 = blocks go through the stage buffer instead
};

enum LookupStatus : int32_t {
	ST_MISS = 0,
	ST_HIT = 1,
	ST_INVALID = 2,      // page number overflowed 44 bits: not counted as a request (cachemap.c:173-174)
	ST_BAD_ENTRY = 3,    // key present with another address (filemap.c:236-240)
	ST_BAD_DECODE = 4,   // decoder consumed != stored length (filemap.c:244-248)
	ST_REMOTE = 5,       // multi-GPU: the key's newest record is on another rank (status - 5 is not encoded; see owner_out)
	ST_CORRUPT = 6,      // CMB200_VERIFY: the decoded page's EF128 differs from the one stored with the record
};

// Counters of the verified gets (CMB200_VERIFY), device words: [VS_VERIFIED] hits whose page matched
// the stored EF128, [VS_UNVERIFIED] hits without a fingerprint for that record version, [VS_CORRUPT]
// pages that did not match.
enum : uint32_t { VS_VERIFIED = 0, VS_UNVERIFIED = 1, VS_CORRUPT = 2, VS_WORDS = 3 };

struct EncodeJob {
	const uint8_t *pages;    // n chunks, `page_stride` apart, 16-byte aligned
	uint64_t page_stride;    // a multiple of 16
	uint32_t nbytes;         // chunk length
	uint32_t n;
	uint32_t accel;          // 0 = store raw (cachemap.h comp_accel==0)
	uint8_t *stage;          // n x stage_stride scratch for blocks
	uint64_t stage_stride;
	int32_t *lens;           // out: block length, -1 = chunk skipped (superseded inside the batch)
	unsigned long long *rec_out; // out, optional: arena offset of the stored record per chunk (~0 = dropped)
	uint64_t *fps;           // out, optional: 2 x u64 per chunk {hi, lo}
	unsigned int *work;      // 1 + ENC_BUCKETS words: the ticket counter, then the bucket sizes (zeroed by the launcher)
	uint32_t *order;         // scratch of encode_order_words(n): chunk lists of the longest-first handout (launch_encode)
	// store mode (all null/0 for codec-only use)
	const uint32_t *slot_idx; // per chunk, from the upsert kernel; 0xffffffff = invalid address
	const unsigned long long *addr; // per chunk {u,l}
	const unsigned long long *ts;   // per chunk
	unsigned long long seq0;  // sequence of chunk 0
	unsigned long long seq_stride;  // sequence step between chunks (world size when chunks are sharded round-robin)
	TableView table;
	ArenaView arena;
};

// Longest-first handout (DESIGN.md §4): when a launch has more chunks than resident encoder warps,
// k_cost rates every chunk from a sample of its bytes and appends it to the list of its cost bucket;
// the tickets of k_encode then walk the buckets from the costliest down.
constexpr uint32_t ENC_BUCKETS = 8;
inline size_t encode_order_words(uint32_t n) { return (size_t)ENC_BUCKETS * n; }
int launch_encode(const EncodeJob &job, cudaStream_t st);   // -> kernels launched (0..2), < 0 on error

struct DecodeJob {
	uint32_t n;
	uint32_t nbytes;
	uint8_t *pages;              // n x nbytes out
	int32_t *status;             // in/out (store mode) or out consumed (codec mode)
	// codec mode
	const uint8_t *blocks;       // n blocks, block_stride apart
	uint64_t block_stride;
	const int32_t *lens;
	// store mode
	const uint64_t *rec_off;     // per request, from lookup
	const uint32_t *vlen;
	const uint8_t *arena;
	const uint8_t *host;         // device address of the host tier (null: no tier)
	unsigned long long *host_hits;
	HotLog hot;                  // where tier hits are logged (null: no tier)
	const unsigned long long *addr;   // n x {u, l}, the requests' addresses (for the log)
};
// Store mode with CMB200_VERIFY: every decoded page is compared with its record's EF128 (k_decode_verify).
struct DecodeVerify {
	const uint32_t *idx;              // per request, the key's slot (from lookup)
	const uint64_t *fp;               // the table's fingerprints and their tags
	const uint32_t *fp_tag;
	unsigned long long *vstat;        // VS_WORDS counters
};
// Store mode with CMB200_TOUCH: every request answered ST_HIT raises its slot's ts to `ts`
// (k_decode_touch, k_decode_verify_touch).
struct DecodeTouch {
	const uint32_t *idx;              // per request, the key's slot (from lookup)
	Slot *slots;
	unsigned long long ts;
};
int launch_decode(const DecodeJob &job, cudaStream_t st, const DecodeVerify *verify = nullptr,
    const DecodeTouch *touch = nullptr);

// Fused small-batch get (one CTA per request): key lookup, record staged in shared memory by TMA,
// LZ4 decode shared -> shared, page written out with 16-byte stores (device memory or page-locked
// host memory).  Safe to run on its own stream while puts run on another: records are immutable
// and the record's own prefix is checked against the request.  peer[r] = base of rank r's arena
// mapped into this process (NVLink peer memory), for keys whose newest record lives on rank r.
#define GET_MAX_PEERS 16
struct GetJob {
	TableView table;
	const uint8_t *arena;
	uint64_t arena_size;
	const uint8_t *host;              // device address of the host tier (null: no tier)
	uint64_t host_size;
	unsigned long long *host_hits;
	const unsigned long long *addr;   // n x {u, l}
	const uint8_t *valid;             // optional
	uint32_t n;
	uint32_t nbytes;                  // page size, <= 131072; above 65536 a cluster of two CTAs per request
	uint8_t *out;                     // n x nbytes
	int32_t *status;                  // n
	const uint8_t *peer[GET_MAX_PEERS];
	uint64_t peer_size[GET_MAX_PEERS];
	uint4 *scratch;                   // pool_n regions of region_entries sequence descriptors (16 bytes each)
	uint32_t region_entries;
	uint32_t *pool_bits;              // bitmap of the regions in use
	uint32_t pool_n;
	HotLog hot;                       // where tier hits are logged (null: no tier); last, so that the
	                                  // other members keep their parameter offsets
	unsigned long long *vstat;        // CMB200_VERIFY (table.fp_tag set): VS_WORDS counters
	unsigned long long touch_ts;      // CMB200_TOUCH: a local hit raises its slot's ts to this; 0 = no touch
};
bool get_small_supports(uint32_t nbytes);
size_t get_small_smem(uint32_t nbytes, bool verify);
uint32_t get_small_region_entries(uint32_t nbytes);
// requests resident on the device at once, < 0 on error
int get_small_residency(uint32_t nbytes, bool verify, bool touch);
int launch_get_small(const GetJob &job, int device, cudaStream_t st);   // device: CUDA ordinal the launch runs on

int launch_fingerprint(const uint8_t *pages, uint64_t stride, uint32_t nbytes, uint32_t n,
    uint64_t *fps, cudaStream_t st);

// addr[2i],addr[2i+1] = {u,l}; valid[i] = 0 marks a rejected address (cachemap.c:160-161).
int launch_compose(const uint64_t *offset, const uint64_t *nhid, const uint32_t *genid, int pshift,
    uint32_t n, unsigned long long *addr, uint8_t *valid, unsigned long long *key, cudaStream_t st);

int launch_upsert(TableView t, const unsigned long long *addr, const uint8_t *valid, uint32_t n,
    unsigned long long seq0, unsigned long long seq_stride, uint32_t *slot_idx, cudaStream_t st);

// Multi-GPU index replication, the records staying on the device: pack one 32-byte record per chunk
// of a put step, import all-gathered records written on other GPUs (rows of my_rank / rows that stored
// nothing are skipped).  Newest sequence per key wins; a local record that loses is retired.
// Record = {u, l, global stream position, tail}; tail = owner rank << 56 | arena offset / 16 << 22 |
// stored length + 1 (0 = the chunk stored nothing).  The location lets another GPU read the record
// from the owner's arena over NVLink (k_get_small).
#define XREC_LEN_BITS 22
#define XREC_OFF_BITS 34
__host__ __device__ inline unsigned long long xrec_tail(uint32_t owner, unsigned long long rec_off, int32_t len) {
	return ((unsigned long long)owner << 56) | (((rec_off >> 4) & ((1ull << XREC_OFF_BITS) - 1)) << XREC_LEN_BITS) |
	    (unsigned long long)(len < 0 ? 0u : (uint32_t)len + 1u);
}
__host__ __device__ inline uint32_t xrec_owner(unsigned long long tail) { return (uint32_t)(tail >> 56); }
__host__ __device__ inline unsigned long long xrec_off(unsigned long long tail) {
	return ((tail >> XREC_LEN_BITS) & ((1ull << XREC_OFF_BITS) - 1)) << 4;
}
__host__ __device__ inline uint32_t xrec_len1(unsigned long long tail) { return (uint32_t)(tail & ((1u << XREC_LEN_BITS) - 1)); }
int launch_pack_records(const unsigned long long *addr, const int32_t *lens, const unsigned long long *rec_off, uint32_t n,
    unsigned long long seq0, unsigned long long stride, uint32_t rank, unsigned long long *out, cudaStream_t st);
int launch_import_records(TableView t, ArenaView a, const unsigned long long *rec, uint32_t n, uint32_t my_rank,
    uint32_t *slot_idx, cudaStream_t st);

int launch_lookup(TableView t, const unsigned long long *addr, const uint8_t *valid, uint32_t n,
    int32_t *status, uint64_t *rec_off, uint32_t *vlen, unsigned long long *ts_out, cudaStream_t st,
    uint32_t *idx_out = nullptr);
// After launch_lookup: status ST_REMOTE entries have their owner rank in rec_off[i]; idx_out (optional)
// gets the key's slot of every ST_HIT.

int launch_unset(TableView t, ArenaView a, const unsigned long long *addr, uint32_t n, cudaStream_t st);
// cmb200_invalidate: retires every live local record whose stored address is {u, l} with
// l_first <= l <= l_last, adding the count to *removed.  scan: k_invalidate_scan, one thread per slot;
// otherwise k_invalidate_keys, one thread per l (the caller keeps l_last - l_first + 1 small).
int launch_invalidate(TableView t, ArenaView a, unsigned long long u, unsigned long long l_first,
    unsigned long long l_last, bool scan, unsigned long long *removed, cudaStream_t st);

// cmb200_rename: the records of one slice, in the order they were taken.  Record k lies at loc[k] (slot
// slot[k], len[k] bytes with the 16-byte padding) and is staged at off[k]; it is stored again at addr[k]
// with ts[k] and fingerprint fp[k] ({0, 0} = none).  addr, ts, off and fp are what launch_restore reads.
struct RenameList {
	unsigned long long *cursor;       // [0] candidates counted by the select (zeroed before it), [1] records
	                                  // of the slice, [2] its staged bytes (both written by the placement)
	unsigned long long *addr, *ts, *off, *loc;
	uint64_t *fp;
	uint32_t *slot, *len;
	uint32_t max_n;
	unsigned long long max_bytes;
};
// k_rename_select: lists every live local record of {u_from, l}, l_first <= l <= l_last, whose {u_to, l}
// belongs to engine dst of g, while the list has room (scan: one thread per slot, as k_invalidate_scan;
// otherwise one thread per l, as k_invalidate_keys); then k_rename_place gives the listed records their
// staging offsets and cuts the slice at max_bytes (cursor[1], cursor[2]).
int launch_rename_select(TableView t, const RenameList &r, unsigned long long u_from, unsigned long long u_to,
    unsigned long long l_first, unsigned long long l_last, bool scan, int g, int dst, uint32_t bsize, cudaStream_t st);
// k_rename_gather: copies the n taken records to stage + off[k] (arena or mapped host tier `host`) and
// retires each slot that still holds its record.
int launch_rename_gather(TableView t, ArenaView a, const uint8_t *host, const RenameList &r, uint32_t n, uint8_t *stage,
    cudaStream_t st);

// Policy-equivalent of filemap_get_rand (filemap.c:264-314): first live slot at or after r.
int launch_sample(TableView t, const unsigned long long *r, uint32_t n, unsigned long long *addr_out,
    unsigned long long *ts_out, int32_t *ok, cudaStream_t st);

int launch_read_fp(TableView t, const unsigned long long *addr, uint32_t n, uint64_t *fp_out, int32_t *ok,
    cudaStream_t st);
// words_out[CKPT_WORDS i + k] = checkpoint word k of the key's slot (t.ckpt must be set); ok[i] = 1: a local
// record whose tag names it, 0: a local record without valid checkpoints, -1: absent or remote.
int launch_read_ckpt(TableView t, const unsigned long long *addr, uint32_t n, uint32_t *words_out, int32_t *ok,
    cudaStream_t st);

int launch_streamgen(const uint64_t *cids, uint32_t n, uint64_t seed, uint32_t bsize, uint8_t *out,
    cudaStream_t st);

// ---- snapshot of the store (persistence of the cache directory, SURVEY.md 8 f3) ----
// One entry per live local record, written by launch_export_list in arbitrary order.
struct ExportEntry {
	unsigned long long rec_off;  // arena offset of {data_prefix, payload}
	unsigned long long ts;
	unsigned long long fp_hi, fp_lo;
	uint32_t len;                // 24 + payload bytes
	uint32_t slot;
};
static_assert(sizeof(ExportEntry) == 40, "export entry layout");
// arena_only: leave out the records of the host tier (compaction moves arena records only).
// seq_min: list only records whose slot's seq is at least this (a delta of a snapshot chain).
// addr_out (nullable): also receives the address {u, l} of every live local record, whatever its seq,
// counted in count[1] (then count has two words); at most max_out of either are written.
int launch_export_list(TableView t, uint32_t bsize, ExportEntry *out, unsigned long long *count,
    unsigned long long max_out, bool arena_only, cudaStream_t st, unsigned long long seq_min = 0,
    ulonglong2 *addr_out = nullptr);
// Snapshot chains: the addresses among base[0 .. n) that no longer hold a live local record (absent,
// no record, owned by another GPU, or the key holds another address) go to out, counted in *count.
int launch_delta_gone(TableView t, const ulonglong2 *base, uint64_t n, ulonglong2 *out, unsigned long long *count,
    cudaStream_t st);
// cmb200_verify_store: turns n export entries into the lookup results of their keys (status ST_HIT,
// location, vlen, slot, address), the input k_decode's verified store mode reads.
int launch_scan_prep(TableView t, const ExportEntry *list, uint32_t n, int32_t *status, uint64_t *rec_off,
    uint32_t *vlen, uint32_t *idx, unsigned long long *addr, cudaStream_t st);
// Restores n records {24-byte prefix, payload} lying at blob + off[i]; slot_idx from launch_upsert
// on the records' addresses (job.addr / job.ts / job.table / job.arena / job.seq0 as for a put).
int launch_restore(const EncodeJob &job, const uint8_t *blob, const unsigned long long *off,
    const uint64_t *fps, uint32_t bsize, cudaStream_t st);

// ---- arena compaction (SURVEY.md 8 f2: space of deleted / outgrown records comes back) ----
// Moves n records (sorted by old offset, new offset <= old offset) down in two steps per window so
// that no record is overwritten before it has been read: gather into `bounce`, then scatter to the
// new offsets and repoint the slots.
struct MoveEntry { unsigned long long old_off, new_off; uint32_t len, slot; };
static_assert(sizeof(MoveEntry) == 24, "move entry layout");
int launch_compact_window(TableView t, ArenaView a, const MoveEntry *moves, uint32_t n, uint8_t *bounce,
    cudaStream_t st);

// ---- host tier (cmb200_demote_batch) ----
// One record moving from the arena to the host tier: gathered from the arena into the bounce buffer at
// bounce_off, copied to the tier by the copy engine, then published at host_off.
struct DemoteEntry { unsigned long long old_off, host_off, bounce_off; uint32_t len, pad; };
static_assert(sizeof(DemoteEntry) == 32, "demote entry layout");
int launch_demote_gather(ArenaView a, const DemoteEntry *d, uint32_t n, uint8_t *bounce, cudaStream_t st);
// Repoints each slot that still holds old_off to REC_HOST | host_off and moves its bytes from arena
// garbage accounting to the tier's.
int launch_demote_publish(TableView t, ArenaView a, const DemoteEntry *d, uint32_t n, cudaStream_t st);
// ---- host tier (cmb200_promote_batch) ----
// One record moving from the host tier back to the arena: copied from host_off (one warp, 16-byte
// loads from the mapped tier) to new_off, free arena bytes above the bump pointer.  The slot that
// still holds REC_HOST | host_off then points at new_off and its bytes go from the tier's accounting
// to the arena's; a slot that no longer holds it leaves the copy as arena garbage.
struct PromoteEntry { unsigned long long host_off, new_off; uint32_t len, pad; };
static_assert(sizeof(PromoteEntry) == 24, "promote entry layout");
int launch_promote(TableView t, ArenaView a, const PromoteEntry *p, uint32_t n, const uint8_t *host, cudaStream_t st);
// Records of the tier that are about to be overwritten: {u, l, REC_HOST | offset, bytes}.  A key whose
// slot still points at that exact location is unset (an eviction); otherwise the bytes leave the
// tier's garbage.  *retired counts the unset keys.
int launch_tier_retire(TableView t, ArenaView a, const unsigned long long *rec, uint32_t n,
    unsigned long long *retired, cudaStream_t st);

// Re-inserts every live slot of `from` into the (zeroed) table `to` of the same geometry.
int launch_rehash(TableView from, TableView to, cudaStream_t st);

// dst[dst_idx ? dst_idx[i] : i] = src[src_idx ? src_idx[i] : i] for n pages of nbytes (a multiple of
// 16; pages 16-byte aligned; index arrays in device memory).  One warp per page.
int launch_move_pages(void *dst, const uint32_t *dst_idx, const void *src, const uint32_t *src_idx, uint32_t n,
    uint32_t nbytes, cudaStream_t st);

// ---- read-modify-write of stored pages (cmb200_patch_batch) ----
// Span k of a row: len bytes at bytes + src_off go to byte page_off of the row's decoded page.
struct PatchSpan { uint32_t page_off, len; unsigned long long src_off; };
static_assert(sizeof(PatchSpan) == 16, "patch span layout");
// For each of `rows` pages (nbytes apart, 16-byte aligned): valid[r] = status[r] == ST_HIT, and on a hit
// spans first[r] .. first[r + 1] - 1 are applied in order.  bytes is 16-byte aligned.
int launch_patch(uint8_t *pages, uint32_t nbytes, uint32_t rows, const int32_t *status, const uint32_t *first,
    const PatchSpan *spans, const uint8_t *bytes, uint8_t *valid, cudaStream_t st);

int sm_count();

}  // namespace cmb
