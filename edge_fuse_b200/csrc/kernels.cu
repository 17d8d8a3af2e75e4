// kernels.cu — sm_90a kernels of the cachemap hot path and their launchers.
//
//   k_encode      fingerprint + LZ4 block encode + arena commit, one warp per chunk  (HBM: §4)
//   k_decode      table record -> LZ4 decode -> page, one warp per request
//   k_fingerprint EF128 alone
//   k_compose / k_upsert / k_lookup / k_unset / k_sample / k_invalidate_*   the HBM key table
//   k_streamgen   synthetic benchmark input
#include "kernels.h"
#include "common.cuh"
#include "fingerprint.cuh"
#include "lz4_encode.cuh"
#include "lz4_encode_ring.cuh"
#include <type_traits>
#include "lz4_decode.cuh"
#include "lz4_decode_cta.cuh"
#include "streamgen.cuh"

namespace cmb {

// ------------------------------------------------------------------------------------------
// key table primitives
// ------------------------------------------------------------------------------------------

// FNV-1a-64 over the 16 in-memory bytes of {u,l} (cachemap/uint128.h:6-21, filemap.c:18-24).
__host__ __device__ __forceinline__ unsigned long long fnv_addr(unsigned long long u, unsigned long long l) {
	unsigned long long h = 14695981039346656037ULL;
#pragma unroll
	for (int i = 0; i < 8; i++) { h = (h ^ ((u >> (8 * i)) & 0xFF)) * 0x100000001b3ULL; }
#pragma unroll
	for (int i = 0; i < 8; i++) { h = (h ^ ((l >> (8 * i)) & 0xFF)) * 0x100000001b3ULL; }
	return h;
}

// Home slot: the low bits of an FNV key are its weakest, so remix before masking.
__device__ __forceinline__ uint64_t home_slot(unsigned long long key, uint64_t cap) {
	unsigned long long z = key;
	z = (z ^ (z >> 32)) * 0xD6E8FEB86659FD93ULL;
	z ^= z >> 32;
	return z & (cap - 1);
}

__device__ __forceinline__ unsigned long long ld_key(const Slot *s) {
	return *reinterpret_cast<const volatile unsigned long long *>(&s->key);
}

// Finds the slot holding `key`, claiming one if absent.  Returns the slot index, or 0xffffffff
// when the table is full.  A deleted slot (tombstone) met on the way is reused, but only after the
// whole probe chain has been searched for the key, and by CAS, so that concurrent claimers of the
// same key inside one kernel converge on one slot: they walk the same chain, so they either agree
// on the first tombstone, or the loser of a CAS rescans and finds the winner's entry.
__device__ uint32_t table_find_or_claim(const TableView &t, unsigned long long key) {
	if (key == KEY_EMPTY) return (uint32_t)t.cap;
	if (key == KEY_TOMB) return (uint32_t)t.cap + 1;
	for (int attempt = 0; attempt < 64; attempt++) {
		uint64_t i = home_slot(key, t.cap);
		uint64_t tomb = ~0ull;
		bool retry = false;
		for (uint64_t n = 0; n < t.cap; n++, i = (i + 1) & (t.cap - 1)) {
			unsigned long long cur = ld_key(&t.slots[i]);
			if (cur == key) return (uint32_t)i;
			if (cur == KEY_TOMB) { if (tomb == ~0ull) tomb = i; continue; }
			if (cur == KEY_EMPTY) {
				if (tomb != ~0ull) {
					unsigned long long old = atomicCAS(&t.slots[tomb].key, KEY_TOMB, key);
					if (old == KEY_TOMB) { atomicAdd(t.tombs, (unsigned long long)-1ll); return (uint32_t)tomb; }
					if (old == key) return (uint32_t)tomb;
					retry = true;           // someone else took that tombstone: rescan
					break;
				}
				unsigned long long old = atomicCAS(&t.slots[i].key, KEY_EMPTY, key);
				if (old == KEY_EMPTY || old == key) return (uint32_t)i;
				// lost the empty slot to another key: keep walking from here
			}
		}
		if (retry) continue;
		if (tomb != ~0ull) {        // chain wrapped without an empty slot: still may reuse a tombstone
			unsigned long long old = atomicCAS(&t.slots[tomb].key, KEY_TOMB, key);
			if (old == KEY_TOMB) { atomicAdd(t.tombs, (unsigned long long)-1ll); return (uint32_t)tomb; }
			if (old == key) return (uint32_t)tomb;
			continue;
		}
		break;
	}
	return 0xffffffffu;
}

__device__ uint32_t table_find(const TableView &t, unsigned long long key) {
	if (key == KEY_EMPTY) return (uint32_t)t.cap;
	if (key == KEY_TOMB) return (uint32_t)t.cap + 1;
	uint64_t i = home_slot(key, t.cap);
	for (uint64_t n = 0; n < t.cap; n++, i = (i + 1) & (t.cap - 1)) {
		unsigned long long cur = ld_key(&t.slots[i]);
		if (cur == key) return (uint32_t)i;
		if (cur == KEY_EMPTY) break;
	}
	return 0xffffffffu;
}

// cachemap/cachemap.c:151-166 + filemap.c:18-24, one thread per request.
__global__ void k_compose(const uint64_t *offset, const uint64_t *nhid, const uint32_t *genid, int pshift,
    uint32_t n, unsigned long long *addr, uint8_t *valid, unsigned long long *key) {
	uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= n) return;
	unsigned long long page = offset[i] >> pshift;
	bool ok = (page >> 44) == 0;
	unsigned long long l = page | ((unsigned long long)genid[i] << 44);
	unsigned long long u = nhid[i];
	addr[2 * i] = u;
	addr[2 * i + 1] = l;
	valid[i] = ok;
	if (key) key[i] = fnv_addr(u, l);
}

// Claims the slot of every chunk of a put batch and records stream order: the chunk with the
// highest sequence per key is the one whose record survives (sequential last-writer-wins,
// SURVEY.md App. B rule 4).
__global__ void k_upsert(TableView t, const unsigned long long *addr, const uint8_t *valid, uint32_t n,
    unsigned long long seq0, unsigned long long seq_stride, uint32_t *slot_idx) {
	uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= n) return;
	uint32_t idx = 0xffffffffu;
	if (!valid || valid[i]) {
		unsigned long long key = fnv_addr(addr[2 * i], addr[2 * i + 1]);
		idx = table_find_or_claim(t, key);
		if (idx != 0xffffffffu) atomicMax(&t.slots[idx].seq, seq0 + seq_stride * i);
	}
	slot_idx[i] = idx;
}

__global__ void k_lookup(TableView t, const unsigned long long *addr, const uint8_t *valid, uint32_t n,
    int32_t *status, uint64_t *rec_off, uint32_t *vlen, unsigned long long *ts_out, uint32_t *idx_out) {
	uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= n) return;
	int32_t st = ST_MISS;
	uint64_t off = 0;
	uint32_t vl = 0;
	unsigned long long ts = 0;
	uint32_t idx = 0xffffffffu;
	if (valid && !valid[i]) {
		st = ST_INVALID;
	} else {
		unsigned long long u = addr[2 * i], l = addr[2 * i + 1];
		idx = table_find(t, fnv_addr(u, l));
		if (idx != 0xffffffffu) {
			const Slot &s = t.slots[idx];
			if (s.vlen != 0) {
				if (s.addr_u == u && s.addr_l == l) {
					st = ST_HIT; off = s.rec_off; vl = s.vlen; ts = s.ts;
				} else {
					st = ST_BAD_ENTRY;
				}
			} else if (s.owner != 0 && s.addr_u == u && s.addr_l == l) {
				st = ST_REMOTE; off = s.owner - 1;
			}
		}
	}
	status[i] = st;
	if (rec_off) rec_off[i] = off;
	if (vlen) vlen[i] = vl;
	if (ts_out) ts_out[i] = ts;
	if (idx_out) idx_out[i] = idx;
}

// The bytes a slot's record held (s.alloc) become garbage of the tier they are in.
__device__ __forceinline__ void slot_release(const ArenaView &a, const Slot &s) {
	if (s.rec_off & REC_HOST) {
		atomicAdd(a.tier, (unsigned long long)s.alloc);
		atomicAdd(a.tier + 1, (unsigned long long)-1ll);
	} else {
		atomicAdd(a.garbage, (unsigned long long)s.alloc);
	}
}

// Appends the address of a get answered from the host tier to the hot log (one thread).  The log is
// written without a lock: an entry read while it is being written, or one a later lap has replaced, is
// only a hint, since cmb200_promote_batch looks every address up again and checks the record's prefix.
__device__ __forceinline__ void hot_log(const HotLog &h, unsigned long long u, unsigned long long l) {
	const unsigned long long k = atomicAdd(h.head, 1ull);
	h.ring[k % HOT_LOG_N] = make_ulonglong2(u, l);
}

// CMB200_TOUCH: a hit on {u, l} raises the ts of its slot idx to `stamp` (one thread).  The slot is
// re-checked for the key first, so a slot that a table rebuild or a tombstone reuse gave to another key
// keeps its ts; the side slots of keys 0 and ~0 belong to their key alone.  atomicMax: a stamp never
// lowers ts, whichever of two gets (or a put and a get) lands first.
__device__ __forceinline__ void slot_touch(Slot *slots, uint32_t idx, unsigned long long u, unsigned long long l,
    unsigned long long stamp) {
	Slot &s = slots[idx];
	const unsigned long long key = fnv_addr(u, l);
	if (key == KEY_EMPTY || key == KEY_TOMB || ld_key(&s) == key) atomicMax(&s.ts, stamp);
}

// Retires the record of slot idx: the slot becomes a tombstone (the side slots of keys 0 and ~0 stay
// empty slots) and the record's bytes garbage.  Returns false when the slot held no record, so that
// of two threads naming the same slot exactly one retires it.
__device__ __forceinline__ bool slot_retire(const TableView &t, const ArenaView &a, uint32_t idx) {
	Slot &s = t.slots[idx];
	uint32_t old = atomicExch(&s.vlen, 0u);
	if (old == 0) return false;
	atomicAdd(t.entries, (unsigned long long)-1ll);
	slot_release(a, s);
	s.alloc = 0;
	s.owner = 0;
	if (t.fp_tag) t.fp_tag[idx] = 0u;
	if (idx < t.cap) {
		s.key = KEY_TOMB;
		atomicAdd(t.tombs, 1ull);
	}
	return true;
}

// filemap_unset (filemap.c:188-215): delete by key, whatever address the record holds.
__global__ void k_unset(TableView t, ArenaView a, const unsigned long long *addr, uint32_t n) {
	uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= n) return;
	uint32_t idx = table_find(t, fnv_addr(addr[2 * i], addr[2 * i + 1]));
	if (idx == 0xffffffffu) return;
	// Two requests of one batch may name the same key: let exactly one retire the record.
	slot_retire(t, a, idx);
}

// cmb200_invalidate: retire every live local record whose stored address is {u, l}, l in
// [l_first, l_last].  Two paths that leave the same store, chosen by the engine from the interval's
// length (DESIGN.md §2, *Invalidation*).  Removals are counted once per warp.
__device__ __forceinline__ void count_warp(bool hit, unsigned long long *removed) {
	const unsigned m = __ballot_sync(0xffffffffu, hit);
	if (m && (threadIdx.x & 31) == 0) atomicAdd(removed, (unsigned long long)__popc(m));
}

// One thread per slot (cap + 2 of them).  Only the first 16 bytes {key, addr_u} are read for every
// slot, by one streaming load, so that a scan of a large table does not push the encoder's and the
// small gets' lines out of L2; the rest of the slot is read only where addr_u matches.  A dead slot
// keeps its old address, hence the liveness test of k_export_list.
__global__ void __launch_bounds__(256) k_invalidate_scan(TableView t, ArenaView a, unsigned long long u,
    unsigned long long l_first, unsigned long long l_last, unsigned long long *removed) {
	const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
	bool hit = false;
	if (i < t.cap + 2) {
		const ulonglong2 ku = __ldcs(reinterpret_cast<const ulonglong2 *>(t.slots + i));
		if (ku.y == u && (i >= t.cap || (ku.x != KEY_EMPTY && ku.x != KEY_TOMB))) {
			const Slot &s = t.slots[i];
			const unsigned long long l = s.addr_l;
			if (l >= l_first && l <= l_last && s.vlen != 0 && s.owner == 0) hit = slot_retire(t, a, (uint32_t)i);
		}
	}
	count_warp(hit, removed);
}

// One thread per l of the interval: the thread builds its address, finds the key's slot and retires
// it only when the slot holds exactly that address.  A key names one record, not one address: another
// object's page may hold it, and that page stays.
__global__ void __launch_bounds__(256) k_invalidate_keys(TableView t, ArenaView a, unsigned long long u,
    unsigned long long l_first, uint64_t n, unsigned long long *removed) {
	const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
	bool hit = false;
	if (i < n) {
		const unsigned long long l = l_first + i;
		const uint32_t idx = table_find(t, fnv_addr(u, l));
		if (idx != 0xffffffffu) {
			const Slot &s = t.slots[idx];
			if (s.addr_u == u && s.addr_l == l && s.owner == 0) hit = slot_retire(t, a, idx);
		}
	}
	count_warp(hit, removed);
}

// filemap_get_rand (filemap.c:264-314) picks the first key at or after a random 64-bit draw; the
// policy-equivalent here is the first live slot at or after a random slot.  One thread per draw
// walks at most SAMPLE_WALK slots (a table at its eviction threshold is >= 1/8 full, so this
// almost always ends within a few slots) and redraws a few times; whatever is still unresolved
// (a nearly empty table) is finished by k_sample_scan, one CTA per draw, 256 slots per step.
constexpr uint32_t SAMPLE_WALK = 128, SAMPLE_REDRAWS = 8;
__device__ __forceinline__ bool slot_live(const Slot &s) { return s.vlen != 0; }
__global__ void k_sample(TableView t, const unsigned long long *r, uint32_t n, unsigned long long *addr_out,
    unsigned long long *ts_out, int32_t *ok) {
	uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= n) return;
	unsigned long long draw = r[i];
	int32_t found = -1;                                   // -1 = left to k_sample_scan
	for (uint32_t a = 0; a < SAMPLE_REDRAWS && found < 0; a++) {
		const uint64_t start = home_slot(draw, t.cap);
		for (uint32_t k = 0; k < SAMPLE_WALK; k++) {
			const uint64_t j = (start + k) % (t.cap + 2);
			const Slot &s = t.slots[j];
			if (slot_live(s)) {
				addr_out[2 * i] = s.addr_u; addr_out[2 * i + 1] = s.addr_l; ts_out[i] = s.ts;
				found = 1;
				break;
			}
		}
		draw = draw * 0x9E3779B97F4A7C15ULL + 0xD1B54A32D192ED03ULL;
	}
	ok[i] = found;
}
__global__ void __launch_bounds__(256) k_sample_scan(TableView t, const unsigned long long *r, uint32_t n,
    unsigned long long *addr_out, unsigned long long *ts_out, int32_t *ok) {
	__shared__ unsigned long long first;
	for (uint32_t i = blockIdx.x; i < n; i += gridDim.x) {
		if (ok[i] >= 0) continue;                         // uniform across the CTA
		const uint64_t total = t.cap + 2, start = home_slot(r[i], t.cap);
		if (threadIdx.x == 0) first = ~0ull;
		__syncthreads();
		for (uint64_t base = 0; base < total; base += blockDim.x) {
			const uint64_t k = base + threadIdx.x;
			if (k < total && slot_live(t.slots[(start + k) % total])) atomicMin(&first, (unsigned long long)k);
			__syncthreads();
			if (first != ~0ull) break;
			__syncthreads();
		}
		if (threadIdx.x == 0) {
			if (first != ~0ull) {
				const Slot &s = t.slots[(start + first) % total];
				addr_out[2 * i] = s.addr_u; addr_out[2 * i + 1] = s.addr_l; ts_out[i] = s.ts;
				ok[i] = 1;
			} else {
				ok[i] = 0;
			}
		}
		__syncthreads();
	}
}

// ------------------------------------------------------------------------------------------
// fused fingerprint -> LZ4 encode -> arena commit
// ------------------------------------------------------------------------------------------

// Points the slot at a finished record (one thread).  Order: location first, then the length that
// makes the slot valid; readers on other streams take the length and the address from the record's
// own prefix and only the location from the slot (k_get_small).
// Invariant: rec_off is the only word of a slot that such a reader trusts, and it is always written
// with ONE 8-byte store.  Demotion to the host tier (k_demote_publish) changes nothing else (vlen,
// addr and ts stay), so a reader sees the old arena location or the new host location, never a mix;
// the arena bytes stay intact until the next compaction, which closes get_gate.
// Promotion back to the arena (k_promote) is the same store in the other direction and needs no
// get_gate either: a reader sees the tier location or the arena location, and both hold the same bytes.
// The tier bytes stay intact until the ring laps them, and that lap closes get_gate (demote_group).
// The arena bytes lie above the bump pointer as it was before the promotion, where no slot pointed, so
// no reader can reach them before the rec_off store, which k_promote makes after a fence.
// With CMB200_VERIFY the fingerprint is guarded like the checkpoints (ckpt_store): its tag is zeroed
// before fp changes and names the new record only once rec_off and vlen are out, so a get on another
// stream that staged the old record never compares it with the new fingerprint.  has_fp = false (a
// snapshot written without fingerprints) leaves the tag zero: the record is served unverified.
__device__ __forceinline__ void slot_publish(const EncodeJob &job, Slot &s, uint32_t i, uint32_t idx, unsigned long long off,
    uint32_t need, uint32_t clen, unsigned long long au, unsigned long long al, uint64_t fp_hi, uint64_t fp_lo,
    bool has_fp = true) {
	// whatever checkpoints the slot has describe the record it is leaving (ckpt_store renews them)
	if (job.table.ckpt) *reinterpret_cast<volatile uint32_t *>(&job.table.ckpt[(size_t)idx * CKPT_WORDS]) = 0u;
	if (job.table.fp_tag) { *reinterpret_cast<volatile uint32_t *>(&job.table.fp_tag[idx]) = 0u; __threadfence(); }
	if (s.owner) { atomicAdd(job.table.remote, (unsigned long long)-1ll); s.owner = 0; }   // now newest here (alloc held the remote length)
	else if (s.alloc) slot_release(job.arena, s);                                          // the record this one replaces
	s.addr_u = au; s.addr_l = al;
	s.ts = job.ts ? job.ts[i] : 0;
	if (job.table.fp) { job.table.fp[2 * (size_t)idx] = fp_hi; job.table.fp[2 * (size_t)idx + 1] = fp_lo; }
	s.alloc = need;
	*reinterpret_cast<volatile unsigned long long *>(&s.rec_off) = off;
	__threadfence();
	if (s.vlen == 0) atomicAdd(job.table.entries, 1ull);
	*reinterpret_cast<volatile uint32_t *>(&s.vlen) = clen + 1u;
	if (job.rec_out) job.rec_out[i] = off;
	if (job.table.fp_tag && has_fp) { __threadfence(); *reinterpret_cast<volatile uint32_t *>(&job.table.fp_tag[idx]) = ckpt_tag(off, clen); }
}

// Parse checkpoints of the record just published in slot idx (whole warp; lane k holds word k, see
// lz4_encode_lean).  slot_publish has zeroed the tag and fenced; the words go in, then the tag that
// names this record version — a reader takes the words only between two equal reads of that tag.
__device__ __forceinline__ void ckpt_store(const EncodeJob &job, uint32_t idx, unsigned long long off, uint32_t clen,
    uint32_t ck, int lane) {
	if (!job.table.ckpt) return;
	uint32_t *w = job.table.ckpt + (size_t)idx * CKPT_WORDS;
	__syncwarp();
	if (lane >= 1 && lane < (int)CKPT_WORDS) *reinterpret_cast<volatile uint32_t *>(w + lane) = ck;
	__threadfence();
	__syncwarp();
	if (lane == 0) *reinterpret_cast<volatile uint32_t *>(w) = ckpt_tag(off, clen);
}

// The record of slot idx moved from old_loc to new_loc with its block unchanged (compaction, demotion,
// promotion), so its checkpoints and its fingerprint still hold and only their tags move.  A tag that
// names another record version (or none) is left alone.  The fence orders the caller's rec_off store
// before the new tag, so a reader that sees the tag also sees the location it names.  (one thread)
__device__ __forceinline__ void ckpt_retag(const TableView &t, uint32_t idx, unsigned long long old_loc,
    unsigned long long new_loc, uint32_t clen) {
	uint32_t *tags[2] = {t.ckpt ? t.ckpt + (size_t)idx * CKPT_WORDS : nullptr, t.fp_tag ? t.fp_tag + idx : nullptr};
	for (uint32_t *w : tags) {
		if (w && *reinterpret_cast<volatile uint32_t *>(w) == ckpt_tag(old_loc, clen)) {
			__threadfence();
			*reinterpret_cast<volatile uint32_t *>(w) = ckpt_tag(new_loc, clen);
		}
	}
}

// Stores the finished block as a filemap record {data_prefix, block} (filemap.c:140-147) and
// publishes it in the key table.  Called by the whole warp; lane 0 owns the bookkeeping.
__device__ unsigned long long commit_record(const EncodeJob &job, uint32_t i, uint32_t idx, const uint8_t *payload,
    uint32_t plen, int32_t clen, bool payload_ro, uint64_t fp_hi, uint64_t fp_lo, int lane, bool has_fp = true) {
	Slot &s = job.table.slots[idx];
	const uint32_t need = (24u + plen + 15u) & ~15u;
	unsigned long long off = 0;
	int ok = 1;
	if (lane == 0) {
		// Records are immutable once published and a rewrite never reuses the old record's bytes:
		// a get that runs concurrently on another stream (k_get_small) decodes either the old or the
		// new record, never a torn one (LMDB gives the reference's readers a snapshot, filemap.c:223).
		// The old bytes become garbage until the arena is compacted.
		off = atomicAdd(job.arena.head, (unsigned long long)need);
		if (off + need > job.arena.size) {
			// arena full: the put is dropped silently, as a full LMDB map drops it
			// (filemap.c:143-145,154-157).  The bump pointer is never rolled back (a rollback
			// races with allocations that succeeded in between and would hand their bytes out
			// twice): it stays saturated until cmb200_compact resets it.
			// The slot is left as it is: a record the key already has stays readable, as the
			// reference's store keeps the old value when mdb_put fails.
			atomicAdd(job.arena.dropped, 1ull);
			ok = 0;
		}
	}
	ok = __shfl_sync(CMB_FULL, ok, 0);
	if (!ok) {
		// nothing was stored: lens_out says so (-1), as for a skipped chunk (cachemap_b200.h)
		if (lane == 0 && job.rec_out) job.rec_out[i] = ~0ull;
		if (lane == 0 && job.lens) job.lens[i] = -1;
		return ~0ull;
	}
	off = __shfl_sync(CMB_FULL, off, 0);
	uint8_t *rec = job.arena.base + off;
	const unsigned long long au = job.addr[2 * i], al = job.addr[2 * i + 1];
	if (lane < 6) {
		uint32_t w;
		switch (lane) {
		case 0: w = (uint32_t)au; break;
		case 1: w = (uint32_t)(au >> 32); break;
		case 2: w = (uint32_t)al; break;
		case 3: w = (uint32_t)(al >> 32); break;
		case 4: w = (uint32_t)clen; break;
		default: w = 0; break;                   // the reference leaves these 4 pad bytes unspecified
		}
		reinterpret_cast<uint32_t *>(rec)[lane] = w;
	}
	if (payload_ro) warp_copy_ro(rec + 24, payload, plen, lane);
	else warp_copy_rw(rec + 24, payload, plen, lane);
	__threadfence();                                 // the record is complete before the slot points to it
	__syncwarp();
	if (lane == 0) slot_publish(job, s, i, idx, off, need, (uint32_t)clen, au, al, fp_hi, fp_lo, has_fp);
	return off;                                      // arena offset of the record (~0: dropped)
}

// Direct variant of commit_record: the block already sits in the arena at `base + 24` (this warp's
// segment cursor) and stays there.  Returns the bytes of the segment consumed.
__device__ uint32_t commit_direct(const EncodeJob &job, uint32_t i, uint32_t idx, unsigned long long base,
    uint32_t clen, uint64_t fp_hi, uint64_t fp_lo, int lane) {
	Slot &s = job.table.slots[idx];
	const uint32_t need = (24u + clen + 15u) & ~15u;
	uint8_t *r = job.arena.base + base;
	const unsigned long long au = job.addr[2 * i], al = job.addr[2 * i + 1];
	if (lane < 6) {
		const uint32_t w = lane == 0 ? (uint32_t)au : lane == 1 ? (uint32_t)(au >> 32) : lane == 2 ? (uint32_t)al
		    : lane == 3 ? (uint32_t)(al >> 32) : lane == 4 ? clen : 0u;
		reinterpret_cast<uint32_t *>(r)[lane] = w;
	}
	__threadfence();                                 // block (written by all lanes) and prefix before the slot
	__syncwarp();
	if (lane == 0) slot_publish(job, s, i, idx, base, need, clen, au, al, fp_hi, fp_lo);
	return need;
}

// ---- longest-first handout ---------------------------------------------------------------------
// A launch ends when its last chunk does, and chunk costs differ by about 10x (DESIGN.md §4): with
// chunks taken in index order, the warps that run dry wait for whoever drew a costly chunk last.
// k_cost rates each chunk before the encode and puts it in one of ENC_BUCKETS lists; k_encode's
// tickets then walk the lists from the costliest down, so the launch ends on cheap chunks.
//
// The rate comes from a 1 KiB sample, 8 windows of 128 bytes spread over the page (lane L holds
// bytes [32 (L & 3), +32) of window L >> 2), scanned like the encoder scans the page: a 4-byte
// sequence that occurs elsewhere in the sample is a match, and a match whose previous byte also
// matches at the same distance continues a sequence instead of starting one.  Estimated LZ4 loop
// iterations = sequence starts + match-less positions / (COST_LIT x accel).  Zero pages and repeats
// rate cheap (few starts), incompressible pages too (the probe step skips through them).  A page
// whose sequences are all further apart than the sample sees (source text) rates low; that costs
// balance, never a result.  Only page bytes and slot liveness go into it; a chunk that a later
// chunk of the batch rewrites is not encoded at all and goes last.
// COST_LIT and COST_FULL: least-squares fit of the per-chunk durations of tools/encode_timeline.py
// on an H100 80GB HBM3 (400 W), bench stream and tree files (DESIGN.md §4).
constexpr uint32_t COST_WARPS = 8, COST_TAB = 2048, COST_POS = 125;   // positions rated per window
constexpr float COST_LIT = 1.0f / 14.0f;       // a match-less position weighs 1 / (14 accel) sequence starts
constexpr float COST_FULL = 160.0f;            // estimate at and above which a chunk goes in the top bucket
#ifdef CMB_ENC_TIMELINE        /* diagnostic builds only (tools/encode_timeline.py) */
__device__ unsigned long long *g_enc_timeline;   // per chunk {warp slot, start ns, end ns, estimate}
__device__ __forceinline__ unsigned long long enc_clock() {
	unsigned long long t;
	asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
	return t;
}
#endif
__global__ void __launch_bounds__(COST_WARPS * 32, 4) k_cost(EncodeJob job) {
	__shared__ __align__(16) uint32_t smp[COST_WARPS][256 + 4];           // the sample (+ the word a gram may touch past it)
	// gram hash -> a sample position with that hash; whatever an entry holds (another gram, a position
	// of the previous chunk) is checked against the sample itself, so the table is never cleared
	__shared__ uint16_t tab[COST_WARPS][COST_TAB];
	const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
	uint32_t *s = smp[warp];
	uint16_t *h = tab[warp];
	const uint8_t *sb = reinterpret_cast<const uint8_t *>(s);
	const uint32_t o0 = ((uint32_t)lane & 3u) * 32u;                      // offset of this lane's bytes in its window
	const uint32_t win_stride = (job.nbytes / 8u) & ~15u;
	for (uint32_t i = blockIdx.x * COST_WARPS + warp; i < job.n; i += gridDim.x * COST_WARPS) {
		// the sample is loaded before liveness is known: the two round trips overlap
		const uint4 *src = reinterpret_cast<const uint4 *>(job.pages + (size_t)i * job.page_stride + (lane >> 2) * win_stride + o0);
		const uint4 a = __ldg(src), c = __ldg(src + 1);
		bool live = true;
		if (job.slot_idx) {
			const uint32_t idx = job.slot_idx[i];
			live = idx != 0xffffffffu && job.table.slots[idx].seq == job.seq0 + job.seq_stride * i;
		}
		uint32_t bucket = 0;
		[[maybe_unused]] uint32_t est = 0;                                 // {starts, match-less positions}, timeline builds report it
		if (live) {
			const uint32_t w[9] = {a.x, a.y, a.z, a.w, c.x, c.y, c.z, c.w, __shfl_down_sync(CMB_FULL, a.x, 1)};
			__syncwarp();                                             // the previous chunk's reads of s and h are done
			reinterpret_cast<uint4 *>(s)[2 * lane] = a;
			reinterpret_cast<uint4 *>(s)[2 * lane + 1] = c;
			// every position enters the table (one writer per entry survives), then every position looks
			// its gram up: a gram seen r times finds r - 1 partners, as a serial scan would
#pragma unroll
			for (uint32_t k = 0; k < 32; k++) {
				if (o0 + k >= COST_POS) break;
				const uint32_t g = __funnelshift_r(w[k >> 2], w[(k >> 2) + 1], (k & 3u) * 8u);
				h[(g * 2654435761u) >> 21] = (uint16_t)((uint32_t)lane * 32u + k);
			}
			__syncwarp();
			uint32_t starts = 0, lits = 0;
#pragma unroll
			for (uint32_t k = 0; k < 32; k++) {
				if (o0 + k >= COST_POS) break;
				const uint32_t p = (uint32_t)lane * 32u + k;
				const uint32_t g = __funnelshift_r(w[k >> 2], w[(k >> 2) + 1], (k & 3u) * 8u);
				const uint32_t q = h[(g * 2654435761u) >> 21] & 1023u;
				const bool m = q != p && (q & 127u) < COST_POS && __funnelshift_r(s[q >> 2], s[(q >> 2) + 1], (q & 3u) * 8u) == g;
				const bool cont = m && o0 + k > 0u && (q & 127u) > 0u && sb[p - 1] == sb[q - 1];
				starts += m && !cont;
				lits += !m;
			}
#pragma unroll
			for (int d = 16; d > 0; d >>= 1) {
				starts += __shfl_xor_sync(CMB_FULL, starts, d);
				lits += __shfl_xor_sync(CMB_FULL, lits, d);
			}
			const float cost = (float)starts + COST_LIT * (float)lits / (float)job.accel;
			bucket = min(ENC_BUCKETS - 1u, (uint32_t)(cost * ((float)ENC_BUCKETS / COST_FULL)));
			est = starts << 16 | lits;
		}
		if (lane == 0) {
			const uint32_t pos = atomicAdd(&job.work[1 + bucket], 1u);
			job.order[(size_t)bucket * job.n + pos] = i;
#ifdef CMB_ENC_TIMELINE
			if (g_enc_timeline) g_enc_timeline[4 * (size_t)i + 3] = (unsigned long long)bucket << 32 | est;
#endif
		}
	}
}

// Ticket t of an ordered launch -> chunk: the buckets' sizes in descending cost order, prefix-summed
// across lanes 0..ENC_BUCKETS-1, tell which list t falls in (once per chunk, out of the parse loop).
__device__ __noinline__ uint32_t enc_ticket_chunk(const unsigned int *work, const uint32_t *order, uint32_t n, uint32_t t, int lane) {
	uint32_t cum = lane < (int)ENC_BUCKETS ? work[ENC_BUCKETS - lane] : 0u;   // lane k: bucket ENC_BUCKETS-1-k
#pragma unroll
	for (int d = 1; d < (int)ENC_BUCKETS; d <<= 1) {
		const uint32_t v = __shfl_up_sync(CMB_FULL, cum, d);
		if (lane >= d) cum += v;
	}
	const int k = __ffs(__ballot_sync(CMB_FULL, lane < (int)ENC_BUCKETS && t < cum)) - 1;   // t < n = the sum
	const uint32_t before = __shfl_sync(CMB_FULL, cum, (k + 31) & 31);
	return order[(size_t)(ENC_BUCKETS - 1 - k) * n + (t - (k ? before : 0u))];
}

// ENC 0: page read through the L1.  ENC 1: parse frontier staged in a per-warp shared-memory ring
// by TMA (lz4_encode_ring.cuh); shared memory = tables | rings | mbarriers.
// Launch bounds = the real launch shapes (2 CTAs x 7 warps, or 1 CTA x 13 warps with the ring), so
// that the register allocator may use what the SM has (up to 146 / 152 registers per thread) instead
// of rematerialising loop invariants inside the parse loop.
constexpr int ENC_PLAIN_WARPS = 7, ENC_PLAIN_CTAS = 2, ENC_RING_WARPS = 13;
template <bool WIDE, int ENC>
__global__ void __launch_bounds__(ENC == 1 ? ENC_RING_WARPS * 32 : ENC_PLAIN_WARPS * 32, ENC == 1 ? 1 : ENC_PLAIN_CTAS) k_encode(EncodeJob job) {
	extern __shared__ __align__(128) uint8_t smem[];
	const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
	const uint32_t nwarps = blockDim.x >> 5;
	uint8_t *wsm = smem + (size_t)warp * LZ4_TABLE_BYTES;
	PageRing ring;
	if (ENC == 1)
		ring_setup(ring, smem + (size_t)nwarps * LZ4_TABLE_BYTES + (size_t)warp * RING_ALLOC,
		    smem + (size_t)nwarps * (LZ4_TABLE_BYTES + RING_ALLOC) + (size_t)warp * RING_MBAR_BYTES, lane);
	const uint32_t gw = blockIdx.x * (blockDim.x >> 5) + warp;         // resident warp slot
	const bool direct = job.slot_idx != nullptr && job.arena.seg_bytes != 0u && job.accel != 0u && gw < ARENA_SEG_SLOTS;
	// room one chunk may need while it is being encoded: prefix + a stage row (>= LZ4_compressBound)
	const uint32_t worst = (uint32_t)((24u + job.stage_stride + 15u) & ~15ull);
	unsigned long long seg_cur = 0, seg_end = 0;                         // lane 0's copy is the truth
	if (direct && lane == 0) { seg_cur = job.arena.seg[2 * gw]; seg_end = job.arena.seg[2 * gw + 1]; }
#ifdef CMB_ENC_TIMELINE
	uint32_t prev = ~0u;
#endif
	for (;;) {
		uint32_t i = 0;
		if (lane == 0) i = atomicAdd(job.work, 1u);
		i = __shfl_sync(CMB_FULL, i, 0);
		if (i < job.n && job.order) i = enc_ticket_chunk(job.work, job.order, job.n, i, lane);
#ifdef CMB_ENC_TIMELINE
		if (lane == 0 && g_enc_timeline) {               // a chunk ends where the warp draws its next ticket
			const unsigned long long t = enc_clock();
			if (prev != ~0u) g_enc_timeline[4 * (size_t)prev + 2] = t;
			if (i < job.n) { g_enc_timeline[4 * (size_t)i] = gw; g_enc_timeline[4 * (size_t)i + 1] = t; }
			prev = i;
		}
#endif
		if (i >= job.n) break;
		const bool store = job.slot_idx != nullptr;
		uint32_t idx = 0;
		if (store) {
			idx = job.slot_idx[i];
			// invalid address, or a later chunk of this batch rewrites the same key
			bool live = idx != 0xffffffffu && job.table.slots[idx].seq == job.seq0 + job.seq_stride * i;
			if (!live) { if (lane == 0) job.lens[i] = -1; continue; }
		}
		const uint8_t *src = job.pages + (size_t)i * job.page_stride;
		uint64_t fp_hi = 0, fp_lo = 0;
		if (job.accel == 0) {           // comp_accel == 0: raw page, compressed_length 0 (filemap.c:129-133)
			if (job.fps) {
				warp_fingerprint128(src, job.nbytes, lane, fp_hi, fp_lo);
				if (lane == 0) { job.fps[2 * (size_t)i] = fp_hi; job.fps[2 * (size_t)i + 1] = fp_lo; }
			}
			if (lane == 0) job.lens[i] = 0;
			if (store) commit_record(job, i, idx, src, job.nbytes, 0, true, fp_hi, fp_lo, lane);
			continue;
		}
		// store mode: the block only passes through the stage on its way into the arena, so each warp
		// reuses ONE stage row instead of a row per chunk; with a large arena it does not even do
		// that: the block is encoded straight into this warp's arena segment
		uint8_t *dst = job.stage + (size_t)(store ? gw : i) * job.stage_stride;
		unsigned long long base = 0;
		int in_arena = 0;
		if (direct) {
			if (lane == 0) {
				if (seg_cur + worst > seg_end) {             // segment exhausted: take the next one
					if (seg_end > seg_cur) atomicAdd(job.arena.garbage, seg_end - seg_cur);
					const unsigned long long off = atomicAdd(job.arena.head, (unsigned long long)job.arena.seg_bytes);
					if (off + job.arena.seg_bytes <= job.arena.size) { seg_cur = off; seg_end = off + job.arena.seg_bytes; }
					else { seg_cur = seg_end = 0; }       // no rollback (see commit_record): saturated until compaction
				}
				in_arena = seg_cur + worst <= seg_end;
				base = seg_cur;
			}
			in_arena = __shfl_sync(CMB_FULL, in_arena, 0);
			base = __shfl_sync(CMB_FULL, base, 0);
			if (in_arena) dst = job.arena.base + base + 24;
		}
		uint32_t clen, ck = 0xffffffffu;
#ifdef CMB_ENC_PHASES
		if (lane == 0) s_enc_phase_row[warp] = g_enc_phases && gw % 4u == 0u ? g_enc_phases + 2u * ENC_PH_N * (size_t)i : nullptr;
		__syncwarp();
#endif
		if (job.fps) {                  // fingerprint along the parse frontier: the page is read once
			clen = lz4_encode_lean<WIDE, true, ENC == 1>(src, job.nbytes, dst, job.accel, wsm, ring, lane, fp_hi, fp_lo, ck);
			if (lane == 0) { job.fps[2 * (size_t)i] = fp_hi; job.fps[2 * (size_t)i + 1] = fp_lo; }
		} else {
			clen = lz4_encode_lean<WIDE, false, ENC == 1>(src, job.nbytes, dst, job.accel, wsm, ring, lane, fp_hi, fp_lo, ck);
		}
		// A store keeps at most bsize + 1024 block bytes (filemap.c:126, dstCapacity): above that,
		// LZ4_compress_fast returns 0 (only incompressible pages of more than 128 KiB get there) and
		// the page is stored raw, as with comp_accel == 0.  The block in the stage row or the segment
		// is dropped; a direct segment's cursor stays where it was.
		const bool raw = store && clen > job.nbytes + 1024u;
		if (lane == 0) job.lens[i] = raw ? 0 : (int32_t)clen;
		if (raw) {
			__syncwarp();
			commit_record(job, i, idx, src, job.nbytes, 0, true, fp_hi, fp_lo, lane);
		} else if (store) {
			__syncwarp();
			if (in_arena) {
				const uint32_t used = commit_direct(job, i, idx, base, clen, fp_hi, fp_lo, lane);
				if (lane == 0) seg_cur += used;
				ckpt_store(job, idx, base, clen, ck, lane);
			} else {
				const unsigned long long at = commit_record(job, i, idx, dst, clen, (int32_t)clen, false, fp_hi, fp_lo, lane);
				if (at != ~0ull) ckpt_store(job, idx, at, clen, ck, lane);
			}
		}
	}
	if (direct && lane == 0) { job.arena.seg[2 * gw] = seg_cur; job.arena.seg[2 * gw + 1] = seg_end; }
}

static int g_sm_count = 0;
int sm_count() {
	if (!g_sm_count) {
		int dev = 0;
		cudaGetDevice(&dev);
		cudaDeviceGetAttribute(&g_sm_count, cudaDevAttrMultiProcessorCount, dev);
		if (g_sm_count <= 0) g_sm_count = 132;          // H100 SXM
	}
	return g_sm_count;
}

// Launches k_encode in one of its two organisations (chunks handed out dynamically in both):
//   plain: residency is bounded by shared memory, one 16 KiB position table per chunk, 14 of them in
//          the 227 KiB of an SM (2 CTAs x 7 warps);
//   ring (lz4_encode_ring.cuh): table + 1 KiB TMA ring + mbarriers per warp, 13 chunks per SM in one CTA.
static int launch_encode_kernel(const EncodeJob &job, bool ring, cudaStream_t st) {
	const bool wide = job.nbytes >= LZ4_NARROW_LIMIT;
	void (*const kern)(EncodeJob) = ring ? (wide ? k_encode<true, 1> : k_encode<false, 1>)
	                                     : (wide ? k_encode<true, 0> : k_encode<false, 0>);
	const int warps = ring ? ENC_RING_WARPS : ENC_PLAIN_WARPS, ctas_per_sm = ring ? 1 : ENC_PLAIN_CTAS;
	const size_t smem = (size_t)warps * (ring ? RING_WARP_SMEM : LZ4_TABLE_BYTES);
	CMB_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
	uint32_t grid = (uint32_t)(sm_count() * ctas_per_sm);
	uint32_t need = (job.n + warps - 1) / warps;
	if (grid > need) grid = need;
	kern<<<grid, warps * 32, smem, st>>>(job);
	CMB_CHECK(cudaGetLastError());
	return 0;
}

int launch_encode(const EncodeJob &job_in, cudaStream_t st) {
	if (job_in.n == 0) return 0;
	// One encoder loop (lz4_encode_lean), two data paths with identical output: the ring, where it
	// holds what 30 probes reach (accel <= 12), and the page read through the L1 for every other
	// acceleration.  Both need the 16-byte aligned pages EncodeJob asks for (TMA, fingerprint loads).
	EncodeJob job = job_in;
	const bool ring = job.accel >= 1 && job.accel <= RING_MAX_ACCEL && job.nbytes < (1u << 24);
	// Longest-first handout when chunks wait for a warp at all (more chunks than resident warps) and
	// are encoded (a raw store costs the same per chunk); the sample wants >= 1 KiB pages.
	const uint32_t resident = (uint32_t)sm_count() * (ring ? ENC_RING_WARPS : ENC_PLAIN_CTAS * ENC_PLAIN_WARPS);
	if (job.n <= resident || job.accel == 0 || job.nbytes < 1024u) job.order = nullptr;
	CMB_CHECK(cudaMemsetAsync(job.work, 0, (job.order ? 1 + ENC_BUCKETS : 1) * sizeof(unsigned int), st));
	if (job.order) {
		k_cost<<<(job.n + COST_WARPS - 1) / COST_WARPS, COST_WARPS * 32, 0, st>>>(job);   // a warp per chunk
		CMB_CHECK(cudaGetLastError());
	}
	if (launch_encode_kernel(job, ring, st) != 0) return -1;
	return job.order ? 2 : 1;
}

#ifdef CMB_ENC_TIMELINE
extern "C" int cmb200_enc_timeline(void *buf) {       // n x 4 u64, see g_enc_timeline; null = off
	return cudaMemcpyToSymbol(g_enc_timeline, &buf, sizeof(buf)) == cudaSuccess ? 0 : -1;
}
#endif
#ifdef CMB_ENC_PHASES
extern "C" int cmb200_enc_phases(void *buf, uint32_t *nphases) {   // n x 2 x ENC_PH_N u64, see g_enc_phases; null = off
	if (nphases) *nphases = ENC_PH_N;
	return cudaMemcpyToSymbol(g_enc_phases, &buf, sizeof(buf)) == cudaSuccess ? 0 : -1;
}
#endif

// ------------------------------------------------------------------------------------------
// decode
// ------------------------------------------------------------------------------------------

// VERIFY (CMB200_VERIFY): the warp fingerprints the page it has just written and compares it with the
// record's EF128 when the slot's tag names this record version (the engine stream orders this kernel
// after every put, so no writer races it); a mismatch is ST_CORRUPT.  host_hits null: a scan of the
// store (cmb200_verify_store), which is not a get and books no tier hit.
// The verify state is a parameter of k_decode_verify alone, so that k_decode's parameter block (and with
// it its register allocation) stays what it is without the flag.
// TOUCH (CMB200_TOUCH): lane 0 raises the slot's ts once the request's answer is ST_HIT (after the
// fingerprint comparison under VERIFY); the state is, likewise, a parameter of the touching kernels alone.
template <bool TOUCH>
__device__ __forceinline__ void decode_touch(const DecodeJob &job, const DecodeTouch &t, uint32_t i, int lane) {
	if constexpr (TOUCH) {
		if (lane == 0) slot_touch(t.slots, t.idx[i], job.addr[2 * (size_t)i], job.addr[2 * (size_t)i + 1], t.ts);
	}
}

template <bool VERIFY, bool TOUCH>
__device__ __forceinline__ void decode_request(const DecodeJob &job, const DecodeVerify &v, const DecodeTouch &t) {
	const int lane = threadIdx.x & 31;
	const uint32_t i = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
	if (i >= job.n) return;
	uint8_t *out = job.pages + (size_t)i * job.nbytes;
	if (job.rec_off) {                                  // store mode
		if (job.status[i] != ST_HIT) return;
		const unsigned long long off = job.rec_off[i];
		// host tier: mapped host memory, read over PCIe
		const uint8_t *rec = (off & REC_HOST) ? job.host + (off & ~REC_HOST) : job.arena + off;
		if ((off & REC_HOST) && lane == 0 && (!VERIFY || job.host_hits)) {
			atomicAdd(job.host_hits, 1ull);
			hot_log(job.hot, job.addr[2 * (size_t)i], job.addr[2 * (size_t)i + 1]);
		}
		uint32_t clen = job.vlen[i] - 1u;
		if constexpr (!VERIFY) {
			if (clen == 0) {                            // raw page (filemap.c:249-251)
				warp_copy_ro(out, rec + 24, job.nbytes, lane);
				decode_touch<TOUCH>(job, t, i, lane);
				return;
			}
			int used = lz4_decode_warp(rec + 24, clen, out, job.nbytes, lane);
			if (used != (int)clen && lane == 0) job.status[i] = ST_BAD_DECODE;   // filemap.c:244-248
			if (used == (int)clen) decode_touch<TOUCH>(job, t, i, lane);
		} else {
			if (clen == 0) {
				warp_copy_ro(out, rec + 24, job.nbytes, lane);
			} else if (lz4_decode_warp(rec + 24, clen, out, job.nbytes, lane) != (int)clen) {
				if (lane == 0) job.status[i] = ST_BAD_DECODE;
				return;
			}
			const uint32_t idx = v.idx[i];
			if (v.fp_tag[idx] != ckpt_tag(off, clen)) {
				if (lane == 0) atomicAdd(&v.vstat[VS_UNVERIFIED], 1ull);
				decode_touch<TOUCH>(job, t, i, lane);
				return;
			}
			__syncwarp();                           // every lane's stores of the page are visible to the warp
			uint64_t hi, lo;
			warp_fingerprint128<true>(out, job.nbytes, lane, hi, lo);
			const bool match = hi == v.fp[2 * (size_t)idx] && lo == v.fp[2 * (size_t)idx + 1];
			if (lane == 0) {
				atomicAdd(&v.vstat[match ? VS_VERIFIED : VS_CORRUPT], 1ull);
				if (!match) job.status[i] = ST_CORRUPT;
			}
			if (match) decode_touch<TOUCH>(job, t, i, lane);
		}
	} else {
		int used = lz4_decode_warp(job.blocks + (size_t)i * job.block_stride, (uint32_t)job.lens[i], out,
		    job.nbytes, lane);
		if (lane == 0) job.status[i] = used;
	}
}

__global__ void __launch_bounds__(256, 8) k_decode(DecodeJob job) {
	decode_request<false, false>(job, DecodeVerify{}, DecodeTouch{});
}
// 4 CTAs per SM rather than 8: the fingerprint's 16 loads in flight per lane need the registers that 8
// would leave to spills.
__global__ void __launch_bounds__(256, 4) k_decode_verify(DecodeJob job, DecodeVerify v) {
	decode_request<true, false>(job, v, DecodeTouch{});
}
__global__ void __launch_bounds__(256, 8) k_decode_touch(DecodeJob job, DecodeTouch t) {
	decode_request<false, true>(job, DecodeVerify{}, t);
}
__global__ void __launch_bounds__(256, 4) k_decode_verify_touch(DecodeJob job, DecodeVerify v, DecodeTouch t) {
	decode_request<true, true>(job, v, t);
}

int launch_decode(const DecodeJob &job, cudaStream_t st, const DecodeVerify *verify, const DecodeTouch *touch) {
	if (job.n == 0) return 0;
	const int warps = 8;
	const uint32_t grid = (job.n + warps - 1) / warps;
	if (job.rec_off && touch) {
		if (verify) k_decode_verify_touch<<<grid, warps * 32, 0, st>>>(job, *verify, *touch);
		else k_decode_touch<<<grid, warps * 32, 0, st>>>(job, *touch);
	} else if (job.rec_off && verify) {
		k_decode_verify<<<grid, warps * 32, 0, st>>>(job, *verify);
	} else {
		k_decode<<<grid, warps * 32, 0, st>>>(job);
	}
	CMB_CHECK(cudaGetLastError());
	return 0;
}

// ------------------------------------------------------------------------------------------
// fused small-batch get: lookup + record staging (TMA) + decode in shared memory + page out
// ------------------------------------------------------------------------------------------

constexpr uint32_t GS_THREADS = DC_THREADS;       // 16 warps: one per parse section (lz4_decode_cta.cuh)
constexpr uint32_t GS_CTRL = 128 + 1152;          // control block + decoder state at the start of the shared memory
static_assert(sizeof(DecodeCta) <= 1152, "decoder state fits its slot");
constexpr uint32_t GS_MAX_PAGE = 65536;           // record buffer + page buffer must fit 227 KiB
constexpr uint32_t GS_PAIR_MAX_PAGE = 131072;     // k_get_small_pair: one buffer per CTA of a cluster of two
struct GetShared {
	unsigned long long bar;                   // mbarrier of the record copy
	unsigned long long off;                   // arena offset of the record
	int32_t st;
	uint32_t clen;                            // expected compressed_length (0 = raw page)
	uint32_t owner;                           // rank + 1 when the record is in a peer's arena
	uint32_t idx;                             // slot of the key
	uint32_t region;                          // scratch region this CTA holds (~0: none)
	uint32_t sections;                        // 1 = one warp walks the block, 16 = the record's checkpoints are used
	uint32_t ck[CKPT_WORDS];
	unsigned long long fp[2];                 // VERIFY: the record's stored EF128 {hi, lo} ...
	uint32_t fp_ok;                           // ... 1 = taken under a tag naming the staged record
	uint32_t match;                           // gs_page_matches' answer
};
static_assert(sizeof(GetShared) <= 128, "control block");
__host__ __device__ inline uint32_t gs_recbuf(uint32_t nbytes) { return (24u + nbytes + 1024u + 31u) & ~15u; }
bool get_small_supports(uint32_t nbytes) { return nbytes >= 64u && nbytes <= GS_PAIR_MAX_PAGE && (nbytes & 15u) == 0; }
// Shared memory per CTA: control block, record buffer, page buffer (one CTA per request); with VERIFY
// the EF128 lane sums of the page's 16-stripe groups follow (gs_page_matches).
__host__ __device__ inline uint32_t gs_sums_at(uint32_t nbytes) {
	return nbytes > GS_MAX_PAGE ? GS_CTRL + gs_recbuf(nbytes) : GS_CTRL + gs_recbuf(nbytes) + nbytes;
}
size_t get_small_smem(uint32_t nbytes, bool verify) {
	return gs_sums_at(nbytes) + (verify ? ef_groups(nbytes) * 32u * sizeof(ulonglong2) : 0u);
}
uint32_t get_small_region_entries(uint32_t nbytes) { return dc_region(nbytes); }

__device__ __forceinline__ unsigned long long ldv64(const unsigned long long *p) { return *reinterpret_cast<const volatile unsigned long long *>(p); }
__device__ __forceinline__ uint32_t ldv32(const uint32_t *p) { return *reinterpret_cast<const volatile uint32_t *>(p); }

// Reads the slot of {u, l}.  Readers never block writers: the location is a single 8-byte load and
// everything else about the record (address, length) is taken from the record's own prefix later.
__device__ void gs_lookup(const GetJob &job, unsigned long long u, unsigned long long l, GetShared *sh) {
	int32_t st = ST_MISS;
	uint32_t clen = 0, owner = 0;
	unsigned long long off = 0;
	const uint32_t idx = table_find(job.table, fnv_addr(u, l));
	if (idx != 0xffffffffu) {
		const Slot *s = &job.table.slots[idx];
		const uint32_t vlen = ldv32(&s->vlen);
		const unsigned long long au = ldv64(&s->addr_u), al = ldv64(&s->addr_l);
		if (vlen != 0u) {
			if (au == u && al == l) { st = ST_HIT; __threadfence(); off = ldv64(&s->rec_off); clen = vlen - 1u; }
			else st = ST_BAD_ENTRY;                              // filemap.c:236-240
		} else {
			const unsigned long long ow = ldv64(&s->owner);
			if (ow != 0ull && au == u && al == l) {
				st = ST_REMOTE; owner = (uint32_t)ow;
				__threadfence();
				off = ldv64(&s->rec_off);
				const uint32_t len1 = ldv32(&s->alloc);             // remote stored length + 1, 0 = unknown
				clen = len1 ? len1 - 1u : 0xffffffffu;
			}
		}
	}
	sh->st = st; sh->clen = clen; sh->off = off; sh->owner = owner; sh->idx = idx;
}

// Scratch regions for the sequence descriptors: one per resident CTA, handed out through a bitmap
// (the pool has as many regions as CTAs of this kernel can be resident, so a free one exists).
__device__ uint32_t gs_region_take(const GetJob &job) {
	uint32_t smid;
	asm volatile("mov.u32 %0, %%smid;" : "=r"(smid));
	const uint32_t words = (job.pool_n + 31u) / 32u;
	for (uint32_t probe = 0; probe < (1u << 22); probe++) {
		const uint32_t w = (smid + probe) % words;
		const uint32_t live = w + 1u == words && (job.pool_n & 31u) ? (1u << (job.pool_n & 31u)) - 1u : 0xffffffffu;
		const uint32_t vacant = ~ldv32(&job.pool_bits[w]) & live;
		if (!vacant) continue;
		const uint32_t b = (uint32_t)__ffs(vacant) - 1u;
		if (!((atomicOr(&job.pool_bits[w], 1u << b) >> b) & 1u)) return w * 32u + b;
	}
	return 0xffffffffu;
}
__device__ void gs_region_give(const GetJob &job, uint32_t r) { atomicAnd(&job.pool_bits[r / 32u], ~(1u << (r & 31u))); }

// The record's checkpoints (ckpt_store) -> section table.  Seqlock: tag, words, tag again; the tag
// names the record (arena offset + length), so words of another record version never pass.
__device__ void gs_sections(const GetJob &job, GetShared *sh, DecodeCta *dc, uint32_t clen, bool local) {
	const uint32_t n = job.nbytes, S = n / DC_CHAINS;
	bool use = false;
	if (local && job.table.ckpt) {
		const uint32_t *ck = job.table.ckpt + (size_t)sh->idx * CKPT_WORDS;
		const uint32_t want = ckpt_tag(sh->off, clen);
		if (ldv32(ck) == want) {
			__threadfence();
			for (uint32_t k = 1; k < CKPT_WORDS; k++) sh->ck[k] = ldv32(ck + k);
			__threadfence();
			use = ldv32(ck) == want;
		}
	}
	for (uint32_t c = 0; c < DC_CHAINS; c++) { dc->ip0[c] = 0xffffffffu; dc->op0[c] = 0; dc->op_end[c] = 0; dc->cnt[c] = 0; dc->ip1[c] = 0; dc->op1[c] = 0; }
	dc->err = 0;
	dc->ip0[0] = 0; dc->op0[0] = 0;
	uint32_t prev = 0;
	if (use) {
		for (uint32_t k = 1; k < DC_CHAINS; k++) {
			const uint32_t v = sh->ck[k];
			if (v == 0xffffffffu) continue;                      // no sequence starts in this section
			const uint32_t ip = v >> CKPT_POS_BITS, op = k * S + (v & ((1u << CKPT_POS_BITS) - 1u));
			if (ip >= clen || op >= n || op >= (k + 1u) * S || ip <= dc->ip0[prev]) { use = false; break; }
			dc->ip0[k] = ip; dc->op0[k] = op;
			dc->op_end[prev] = op;
			prev = k;
		}
	}
	if (!use) {
		for (uint32_t c = 1; c < DC_CHAINS; c++) dc->ip0[c] = 0xffffffffu;
		prev = 0;
	}
	dc->op_end[prev] = n;
	sh->sections = use ? DC_CHAINS : 1u;
}

// CMB200_VERIFY: the stored EF128 of the record this CTA staged (slot sh->idx, location off, length
// clen), taken between two equal reads of the slot's fingerprint tag, and only when the tag names that
// location and length.  Otherwise sh->fp_ok = 0 and the page is served unverified: a put of the key on
// another stream may have replaced the fingerprint after the record was staged.  (one thread)
__device__ void gs_fp_take(const GetJob &job, GetShared *sh, unsigned long long off, uint32_t clen, bool local) {
	sh->fp_ok = 0u;
	if (!local) return;                                      // a peer's record: no fingerprint travels with it
	const uint32_t *tag = job.table.fp_tag + sh->idx;
	const uint32_t want = ckpt_tag(off, clen);
	if (ldv32(tag) != want) return;
	__threadfence();
	const unsigned long long *fp = reinterpret_cast<const unsigned long long *>(job.table.fp) + 2 * (size_t)sh->idx;
	sh->fp[0] = ldv64(fp);
	sh->fp[1] = ldv64(fp + 1);
	__threadfence();
	sh->fp_ok = ldv32(tag) == want ? 1u : 0u;
}

// Whole CTA: does the n-byte page at `src` (shared memory, 8-byte aligned) have the EF128 {hi, lo}?
// The 16 warps take the lane sums of the page's 16-stripe groups (fingerprint.cuh: ef_group_sum) into
// `sums`, warp 0 chains and folds them.  The answer passes through *flag and the barrier.
__device__ bool gs_page_matches(const uint8_t *src, uint32_t n, ulonglong2 *sums, unsigned long long hi,
    unsigned long long lo, uint32_t *flag, uint32_t warp, int lane) {
	for (uint32_t g = warp; g < ef_groups(n); g += GS_THREADS / 32u) sums[32u * g + (uint32_t)lane] = ef_group_sum(src, n, g, lane);
	__syncthreads();
	if (warp == 0) {
		uint64_t h, l;
		ef_group_finish(sums, n, lane, h, l);
		if (lane == 0) *flag = h == hi && l == lo ? 1u : 0u;
	}
	__syncthreads();
	return *flag != 0u;
}

// Do the sections add up to the serial parse?  (one thread)
__device__ bool gs_sections_fit(const DecodeCta *dc, uint32_t clen, uint32_t n) {
	if (dc->err) return false;
	uint32_t prev = 0;
	for (uint32_t c = 1; c < DC_CHAINS; c++) {
		if (dc->ip0[c] == 0xffffffffu) continue;
		if (dc->ip1[prev] != dc->ip0[c] || dc->op1[prev] != dc->op0[c]) return false;
		prev = c;
	}
	return dc->ip1[prev] == clen && dc->op1[prev] == n;          // filemap.c:244-248: consumed == compressed_length
}

// The request's answer, by thread 0 of the CTA that answers (k_get_small; the page CTA of
// k_get_small_pair), after a barrier that follows the page's last store.  The status may live in
// page-locked host memory that the caller polls: the page first, then the status (every thread's
// stores happen before the barrier, this thread's system-wide fence after it is cumulative).
// TOUCH (CMB200_TOUCH): a hit on a local record (touch_idx = its slot; ~0 for a peer's record) raises the
// slot's ts to job.touch_ts before the status is stored, so a caller that has seen the status sees the ts.
template <bool VERIFY, bool TOUCH>
__device__ __forceinline__ void gs_answer(const GetJob &job, uint32_t i, int32_t result, uint32_t region, bool from_host,
    uint32_t fp_ok, uint32_t touch_idx) {
	if (region != 0xffffffffu) gs_region_give(job, region);
	if (result == ST_HIT && from_host) {
		atomicAdd(job.host_hits, 1ull);
		// loaded again rather than kept from the top: u and l live past the loop would cost registers
		hot_log(job.hot, job.addr[2 * (size_t)i], job.addr[2 * (size_t)i + 1]);
	}
	if (VERIFY && (result == ST_HIT || result == ST_CORRUPT))
		atomicAdd(&job.vstat[result == ST_CORRUPT ? VS_CORRUPT : fp_ok ? VS_VERIFIED : VS_UNVERIFIED], 1ull);
	if (TOUCH && result == ST_HIT && touch_idx != 0xffffffffu)
		slot_touch(job.table.slots, touch_idx, job.addr[2 * (size_t)i], job.addr[2 * (size_t)i + 1], job.touch_ts);
	__threadfence_system();
	*reinterpret_cast<volatile int32_t *>(&job.status[i]) = result;
}

// VERIFY (CMB200_VERIFY): the page, decoded or raw, is compared with the record's stored EF128 while it
// is still in shared memory (gs_page_matches), so a page that does not match is never written out and
// is answered ST_CORRUPT.
template <bool VERIFY, bool TOUCH>
__global__ void __launch_bounds__(GS_THREADS, 1) k_get_small(GetJob job) {
	extern __shared__ __align__(128) uint8_t smem[];
	GetShared *sh = reinterpret_cast<GetShared *>(smem);
	DecodeCta *dc = reinterpret_cast<DecodeCta *>(smem + 128);
	uint8_t *rec = smem + GS_CTRL;
	uint8_t *page = rec + gs_recbuf(job.nbytes);
	const uint32_t i = blockIdx.x, tid = threadIdx.x;
	const int lane = tid & 31;
	const uint32_t warp = tid >> 5;
	const unsigned long long u = job.addr[2 * (size_t)i], l = job.addr[2 * (size_t)i + 1];
	uint8_t *out = job.out + (size_t)i * job.nbytes;
	const uint32_t s_bar = smem_addr(&sh->bar);
	if (job.valid && !job.valid[i]) { if (tid == 0) job.status[i] = ST_INVALID; return; }
	if (tid == 0) {
		sh->region = 0xffffffffu;
		mbar_init(s_bar, 1u);
		asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
		asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
	}
	uint32_t phase = 0;
	int32_t result = ST_MISS;
	bool from_host = false;                                     // the record read last came from the host tier
	for (int attempt = 0; attempt < 4; attempt++) {
		if (tid == 0) gs_lookup(job, u, l, sh);
		__syncthreads();
		const int32_t st = sh->st;
		const uint32_t clen = sh->clen, owner = sh->owner;
		const unsigned long long off = sh->off;
		result = st;
		if (st != ST_HIT && st != ST_REMOTE) break;
		const uint32_t plen = clen ? clen : job.nbytes;           // payload bytes (raw page when compressed_length is 0)
		const uint32_t tx = (24u + plen + 15u) & ~15u;
		const uint8_t *base = job.arena;
		uint64_t limit = job.arena_size + 256u;                  // every arena is allocated with 256 bytes of slack
		from_host = st == ST_HIT && (off & REC_HOST);
		if (from_host) { base = job.host; limit = job.host_size; }
		const unsigned long long roff = off & ~REC_HOST;
		bool ok = clen <= job.nbytes + 1024u && (off & 15u) == 0;
		if (st == ST_REMOTE) {
			base = owner - 1u < GET_MAX_PEERS ? job.peer[owner - 1u] : nullptr;
			limit = owner - 1u < GET_MAX_PEERS ? job.peer_size[owner - 1u] + 256u : 0;
			ok = ok && base != nullptr && clen != 0xffffffffu;
			if (!ok) break;                                      // no path to the owner's arena: REMOTE is the answer
		}
		if (!ok || roff + tx > limit) { result = ST_MISS; break; }
		if (st == ST_HIT && !from_host) {
			if (tid == 0) { mbar_expect_tx(s_bar, tx); tma_load_1d(smem_addr(rec), base + off, tx, s_bar); }
			while (!mbar_try_wait(s_bar, phase)) {}
			phase ^= 1u;
		} else {
			// the owner's arena over NVLink, or the host tier over PCIe: plain 16-byte loads (TMA is not
			// used on mapped host memory), no local L2 (peer lines are not cached there)
			const uint4 *src = reinterpret_cast<const uint4 *>(base + roff);
			for (uint32_t k = tid; k < tx / 16u; k += GS_THREADS) reinterpret_cast<uint4 *>(rec)[k] = __ldcg(src + k);
			__syncthreads();
		}
		// the record's own prefix decides (filemap.c:9-12): address and compressed_length
		const unsigned long long pu = *reinterpret_cast<const unsigned long long *>(rec);
		const unsigned long long pl = *reinterpret_cast<const unsigned long long *>(rec + 8);
		const uint32_t pclen = *reinterpret_cast<const uint32_t *>(rec + 16);
		if (pu != u || pl != l || pclen != clen) {
			// the slot moved on between the two reads (a put or a compaction on another stream / GPU):
			// look again; a remote location that no longer holds the record is a miss
			result = ST_MISS;
			__syncthreads();
			if (st == ST_REMOTE) break;
			continue;
		}
		if (VERIFY) {
			if (tid == 0) gs_fp_take(job, sh, off, clen, st == ST_HIT);
			__syncthreads();
		}
		if (clen == 0u) {
			if (VERIFY && sh->fp_ok &&
			    !gs_page_matches(rec + 24, job.nbytes, reinterpret_cast<ulonglong2 *>(smem + gs_sums_at(job.nbytes)),
			        sh->fp[0], sh->fp[1], &sh->match, warp, lane)) { result = ST_CORRUPT; break; }
			// raw page (filemap.c:249-251); 8-byte granularity: rec + 24 is not 16-byte aligned
			for (uint32_t k = tid; k < job.nbytes / 8u; k += GS_THREADS)
				reinterpret_cast<unsigned long long *>(out)[k] = reinterpret_cast<const unsigned long long *>(rec + 24)[k];
			result = ST_HIT;
			break;
		}
		// ---- LZ4 block -> page, both in shared memory (lz4_decode_cta.cuh) ----
		if (tid == 0) {
			if (sh->region == 0xffffffffu) sh->region = gs_region_take(job);
			gs_sections(job, sh, dc, clen, st == ST_HIT);
		}
		__syncthreads();
		if (sh->region == 0xffffffffu) { result = ST_BAD_DECODE; break; }           // cannot happen with a pool sized to residency
		uint4 *desc = job.scratch + (size_t)sh->region * job.region_entries;
		const uint32_t stride = dc_stride(job.nbytes);
		const uint32_t blk_s = smem_addr(rec + 24), page_s = smem_addr(page);
		bool good = false;
		for (int pass = 0; pass < 2 && !good; pass++) {
			const bool many = sh->sections > 1u;
			if (dc->ip0[warp] != 0xffffffffu)
				dc_parse_chain<false>(dc, warp, blk_s, clen, job.nbytes, desc + (size_t)warp * stride,
				    many ? stride : job.region_entries, lane);
			__syncthreads();
			good = gs_sections_fit(dc, clen, job.nbytes);
			if (good || !many) break;
			// checkpoints that do not describe this block (never seen; the record is what counts): one walk
			__syncthreads();
			if (tid == 0) gs_sections(job, sh, dc, clen, false);
			__syncthreads();
		}
		if (!good) { result = ST_BAD_DECODE; break; }             // filemap.c:244-248
		dc_literals<false>(dc, desc, stride, blk_s, page_s, rec + 24, page, warp, lane);
		__syncthreads();
		if (warp == 0) dc_matches<false>(dc, desc, stride, page_s, lane);
		__syncthreads();
		if (VERIFY && sh->fp_ok &&
		    !gs_page_matches(page, job.nbytes, reinterpret_cast<ulonglong2 *>(smem + gs_sums_at(job.nbytes)),
		        sh->fp[0], sh->fp[1], &sh->match, warp, lane)) { result = ST_CORRUPT; break; }
		for (uint32_t k = tid; k < job.nbytes / 16u; k += GS_THREADS)
			reinterpret_cast<uint4 *>(out)[k] = reinterpret_cast<const uint4 *>(page)[k];
		result = ST_HIT;
		break;
	}
	__syncthreads();
	// the last lookup decided the answer: owner 0 is a local record, which a hit may touch
	if (tid == 0)
		gs_answer<VERIFY, TOUCH>(job, i, result, sh->region, from_host, sh->fp_ok,
		    TOUCH && sh->owner == 0u ? sh->idx : 0xffffffffu);
}

// ---- pages above 64 KiB: one request per cluster of two CTAs ----------------------------------------
// The record and the page together (264 KiB at 128 KiB pages) exceed the 227 KiB one CTA may have, so
// the request is split over a cluster of two with the same shared-memory layout (DESIGN.md §5):
//   rank 0, the RECORD CTA: lookup, staging, prefix check and retries exactly as k_get_small, the parse
//           on the block in its own shared memory, then the literal phase, which stores the runs into
//           the page CTA over DSMEM.  Raw pages go straight to `out`.  Every decision is taken here.
//   rank 1, the PAGE CTA: holds the page at the record buffer's offset.  Given the record CTA's
//           verdict it runs the match phase on its own shared memory, writes the page out, then the
//           status.  It is the one CTA that answers (gs_answer): region release, host-tier hit, status word.
// Two cluster barrier phases.  A: both CTAs arrive at entry, and the record CTA waits for A before
// its first remote store, so the page CTA has started.  B: the record CTA arrives with release after
// its last remote store and global write, the page CTA waits with acquire: literals, descriptors,
// counts and verdict are visible before the match phase.  Only the page CTA's shared memory is
// accessed remotely, and it waits for B, so no CTA exits while its partner can still reach it.
struct PairVerdict {                              // the page CTA's control block, written by the record CTA
	int32_t result;
	uint32_t region;                          // scratch region of the descriptors (~0: none)
	uint32_t decode;                          // 1: the literals are in the page, the matches are not
	uint32_t from_host;                       // the record came from the host tier
	uint32_t fp_ok;                           // VERIFY: fp holds the record's stored EF128 (GetShared::fp_ok)
	uint32_t match;                           // the page CTA's gs_page_matches answer
	uint32_t fp[4];                           // {hi, lo} as 32-bit halves (DSMEM stores are 32-bit)
	uint32_t touch_idx;                       // TOUCH: slot of a local record, ~0 otherwise
};
static_assert(sizeof(PairVerdict) <= 128, "control block");

__device__ __forceinline__ uint32_t cluster_rank() { uint32_t r; asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r)); return r; }
__device__ __forceinline__ void cluster_arrive_relaxed() { asm volatile("barrier.cluster.arrive.relaxed;" ::: "memory"); }
__device__ __forceinline__ void cluster_arrive_release() { asm volatile("barrier.cluster.arrive.release;" ::: "memory"); }
__device__ __forceinline__ void cluster_wait() { asm volatile("barrier.cluster.wait.acquire;" ::: "memory"); }
// shared::cluster address / generic address of the same location in CTA `rank` of the cluster
__device__ __forceinline__ uint32_t dsmem_map(uint32_t a, uint32_t rank) {
	uint32_t r;
	asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(rank));
	return r;
}
__device__ __forceinline__ uint8_t *dsmem_map_generic(uint8_t *p, uint32_t rank) {
	uint64_t r;
	asm volatile("mapa.u64 %0, %1, %2;" : "=l"(r) : "l"(p), "r"(rank));
	return reinterpret_cast<uint8_t *>(r);
}
__device__ __forceinline__ void dsmem_st32(uint32_t a, uint32_t v) { asm volatile("st.shared::cluster.u32 [%0], %1;" ::"r"(a), "r"(v) : "memory"); }

// VERIFY: the CTA that holds the page compares it with the record's stored EF128 before writing it out
// (gs_page_matches): the page CTA for a decoded page, the record CTA for a raw one.
template <bool VERIFY, bool TOUCH>
__global__ void __cluster_dims__(2, 1, 1) __launch_bounds__(GS_THREADS, 1) k_get_small_pair(GetJob job) {
	extern __shared__ __align__(128) uint8_t smem[];
	DecodeCta *dc = reinterpret_cast<DecodeCta *>(smem + 128);
	uint8_t *buf = smem + GS_CTRL;                              // record CTA: the record; page CTA: the page
	const uint32_t i = blockIdx.x >> 1, tid = threadIdx.x, rank = cluster_rank();
	const int lane = tid & 31;
	const uint32_t warp = tid >> 5;
	uint8_t *out = job.out + (size_t)i * job.nbytes;
	const uint32_t stride = dc_stride(job.nbytes);
	if (job.valid && !job.valid[i]) { if (rank == 1u && tid == 0) job.status[i] = ST_INVALID; return; }
	cluster_arrive_relaxed();                                   // A
	if (rank == 1u) {
		const PairVerdict *v = reinterpret_cast<const PairVerdict *>(smem);
		cluster_wait();                                     // A
		cluster_arrive_relaxed();                           // B
		cluster_wait();                                     // B: the record CTA is done with this CTA
		if (v->decode) {
			if (warp == 0) dc_matches<true>(dc, job.scratch + (size_t)v->region * job.region_entries, stride, smem_addr(buf), lane);
			__syncthreads();
			bool write = true;
			if constexpr (VERIFY) {
				PairVerdict *vw = reinterpret_cast<PairVerdict *>(smem);
				if (v->fp_ok &&
				    !gs_page_matches(buf, job.nbytes, reinterpret_cast<ulonglong2 *>(smem + gs_sums_at(job.nbytes)),
				        (unsigned long long)v->fp[1] << 32 | v->fp[0], (unsigned long long)v->fp[3] << 32 | v->fp[2],
				        &vw->match, warp, lane)) {
					write = false;
					if (tid == 0) vw->result = ST_CORRUPT;      // read below by this thread only
				}
			}
			if (write)
				for (uint32_t k = tid; k < job.nbytes / 16u; k += GS_THREADS)
					reinterpret_cast<uint4 *>(out)[k] = reinterpret_cast<const uint4 *>(buf)[k];
		}
		// the page first, then the status (a raw page was written by the record CTA before it arrived
		// at B, and this thread acquired B)
		__syncthreads();
		if (tid == 0) gs_answer<VERIFY, TOUCH>(job, i, v->result, v->region, v->from_host, v->fp_ok, TOUCH ? v->touch_idx : 0u);
		return;
	}
	GetShared *sh = reinterpret_cast<GetShared *>(smem);
	uint8_t *rec = buf;
	const unsigned long long u = job.addr[2 * (size_t)i], l = job.addr[2 * (size_t)i + 1];
	const uint32_t s_bar = smem_addr(&sh->bar);
	if (tid == 0) {
		sh->region = 0xffffffffu;
		mbar_init(s_bar, 1u);
		asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
		asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
	}
	uint32_t phase = 0;
	int32_t result = ST_MISS;
	bool from_host = false, decode = false;
	for (int attempt = 0; attempt < 4; attempt++) {
		if (tid == 0) gs_lookup(job, u, l, sh);
		__syncthreads();
		const int32_t st = sh->st;
		const uint32_t clen = sh->clen, owner = sh->owner;
		const unsigned long long off = sh->off;
		result = st;
		if (st != ST_HIT && st != ST_REMOTE) break;
		const uint32_t plen = clen ? clen : job.nbytes;
		const uint32_t tx = (24u + plen + 15u) & ~15u;
		const uint8_t *base = job.arena;
		uint64_t limit = job.arena_size + 256u;
		from_host = st == ST_HIT && (off & REC_HOST);
		if (from_host) { base = job.host; limit = job.host_size; }
		const unsigned long long roff = off & ~REC_HOST;
		bool ok = clen <= job.nbytes + 1024u && (off & 15u) == 0;
		if (st == ST_REMOTE) {
			base = owner - 1u < GET_MAX_PEERS ? job.peer[owner - 1u] : nullptr;
			limit = owner - 1u < GET_MAX_PEERS ? job.peer_size[owner - 1u] + 256u : 0;
			ok = ok && base != nullptr && clen != 0xffffffffu;
			if (!ok) break;
		}
		if (!ok || roff + tx > limit) { result = ST_MISS; break; }
		if (st == ST_HIT && !from_host) {
			if (tid == 0) { mbar_expect_tx(s_bar, tx); tma_load_1d(smem_addr(rec), base + off, tx, s_bar); }
			while (!mbar_try_wait(s_bar, phase)) {}
			phase ^= 1u;
		} else {
			const uint4 *src = reinterpret_cast<const uint4 *>(base + roff);
			for (uint32_t k = tid; k < tx / 16u; k += GS_THREADS) reinterpret_cast<uint4 *>(rec)[k] = __ldcg(src + k);
			__syncthreads();
		}
		const unsigned long long pu = *reinterpret_cast<const unsigned long long *>(rec);
		const unsigned long long pl = *reinterpret_cast<const unsigned long long *>(rec + 8);
		const uint32_t pclen = *reinterpret_cast<const uint32_t *>(rec + 16);
		if (pu != u || pl != l || pclen != clen) {
			result = ST_MISS;
			__syncthreads();
			if (st == ST_REMOTE) break;
			continue;
		}
		if (VERIFY) {
			if (tid == 0) gs_fp_take(job, sh, off, clen, st == ST_HIT);
			__syncthreads();
		}
		if (clen == 0u) {
			if (VERIFY && sh->fp_ok &&
			    !gs_page_matches(rec + 24, job.nbytes, reinterpret_cast<ulonglong2 *>(smem + gs_sums_at(job.nbytes)),
			        sh->fp[0], sh->fp[1], &sh->match, warp, lane)) { result = ST_CORRUPT; break; }
			for (uint32_t k = tid; k < job.nbytes / 8u; k += GS_THREADS)
				reinterpret_cast<unsigned long long *>(out)[k] = reinterpret_cast<const unsigned long long *>(rec + 24)[k];
			result = ST_HIT;
			break;
		}
		if (tid == 0) {
			if (sh->region == 0xffffffffu) sh->region = gs_region_take(job);
			gs_sections(job, sh, dc, clen, st == ST_HIT);
		}
		__syncthreads();
		if (sh->region == 0xffffffffu) { result = ST_BAD_DECODE; break; }
		uint4 *desc = job.scratch + (size_t)sh->region * job.region_entries;
		const uint32_t blk_s = smem_addr(rec + 24);
		bool good = false;
		for (int pass = 0; pass < 2 && !good; pass++) {
			const bool many = sh->sections > 1u;
			if (dc->ip0[warp] != 0xffffffffu)
				dc_parse_chain<true>(dc, warp, blk_s, clen, job.nbytes, desc + (size_t)warp * stride,
				    many ? stride : job.region_entries, lane);
			__syncthreads();
			good = gs_sections_fit(dc, clen, job.nbytes);
			if (good || !many) break;
			__syncthreads();
			if (tid == 0) gs_sections(job, sh, dc, clen, false);
			__syncthreads();
		}
		result = good ? ST_HIT : ST_BAD_DECODE;
		decode = good;
		break;
	}
	cluster_wait();                                             // A: the page CTA has started
	const uint32_t region = sh->region;
	if (decode) {
		dc_literals<true>(dc, job.scratch + (size_t)region * job.region_entries, stride, smem_addr(rec + 24),
		    dsmem_map(smem_addr(buf), 1u), rec + 24, dsmem_map_generic(buf, 1u), warp, lane);
		if (tid < DC_CHAINS) dsmem_st32(dsmem_map(smem_addr(&dc->cnt[tid]), 1u), dc->cnt[tid]);
	}
	if (tid == 0) {
		const uint32_t v = dsmem_map(smem_addr(smem), 1u);
		dsmem_st32(v + offsetof(PairVerdict, result), (uint32_t)result);
		dsmem_st32(v + offsetof(PairVerdict, region), region);
		dsmem_st32(v + offsetof(PairVerdict, decode), decode ? 1u : 0u);
		dsmem_st32(v + offsetof(PairVerdict, from_host), from_host ? 1u : 0u);
		if (VERIFY) {
			// a raw page was checked here; fp_ok also tells the page CTA which counter the hit goes to
			const uint32_t fp_ok = (result == ST_HIT || result == ST_CORRUPT) ? sh->fp_ok : 0u;
			dsmem_st32(v + offsetof(PairVerdict, fp_ok), fp_ok);
			for (uint32_t k = 0; k < 4; k++)
				dsmem_st32(v + offsetof(PairVerdict, fp) + 4u * k, (uint32_t)(sh->fp[k >> 1] >> (32u * (k & 1u))));
		}
		if (TOUCH) dsmem_st32(v + offsetof(PairVerdict, touch_idx), sh->owner == 0u ? sh->idx : 0xffffffffu);
	}
	cluster_arrive_release();                                   // B
	cluster_wait();
}

template <bool VERIFY, bool TOUCH>
static int launch_get_small_kernel(const GetJob &job, int device, cudaStream_t st) {
	const size_t smem = get_small_smem(job.nbytes, VERIFY);
	// the attribute belongs to the device: engines on several GPUs (CMB200_DEVICES) each set their own
	constexpr int MAX_DEV = 64;
	const int dev = device >= 0 && device < MAX_DEV ? device : 0;
	if (job.nbytes > GS_MAX_PAGE) {
		static size_t configured_pair[MAX_DEV] = {};
		if (smem > configured_pair[dev]) {
			CMB_CHECK(cudaFuncSetAttribute(k_get_small_pair<VERIFY, TOUCH>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
			configured_pair[dev] = smem;
		}
		k_get_small_pair<VERIFY, TOUCH><<<2u * job.n, GS_THREADS, smem, st>>>(job);
		CMB_CHECK(cudaGetLastError());
		return 0;
	}
	static size_t configured[MAX_DEV] = {};
	if (smem > configured[dev]) {
		CMB_CHECK(cudaFuncSetAttribute(k_get_small<VERIFY, TOUCH>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
		configured[dev] = smem;
	}
	k_get_small<VERIFY, TOUCH><<<job.n, GS_THREADS, smem, st>>>(job);
	CMB_CHECK(cudaGetLastError());
	return 0;
}
int launch_get_small(const GetJob &job, int device, cudaStream_t st) {
	if (job.n == 0) return 0;
	if (job.touch_ts)
		return job.table.fp_tag ? launch_get_small_kernel<true, true>(job, device, st) : launch_get_small_kernel<false, true>(job, device, st);
	return job.table.fp_tag ? launch_get_small_kernel<true, false>(job, device, st) : launch_get_small_kernel<false, false>(job, device, st);
}

// Requests of k_get_small (CTAs) or k_get_small_pair (clusters) that can be resident on the device at
// once (= scratch regions needed).  Clusters of two need two SMs of one GPC.
template <bool VERIFY, bool TOUCH>
static int get_small_residency_of(uint32_t nbytes) {
	const size_t smem = get_small_smem(nbytes, VERIFY);
	if (nbytes > GS_MAX_PAGE) {
		if (cudaFuncSetAttribute(k_get_small_pair<VERIFY, TOUCH>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess) return -1;
		cudaLaunchConfig_t cfg = {};
		cfg.gridDim = dim3(2u * (uint32_t)sm_count());
		cfg.blockDim = dim3(GS_THREADS);
		cfg.dynamicSmemBytes = smem;
		int clusters = 0;
		if (cudaOccupancyMaxActiveClusters(&clusters, k_get_small_pair<VERIFY, TOUCH>, &cfg) != cudaSuccess) return -1;
		return clusters;
	}
	if (cudaFuncSetAttribute(k_get_small<VERIFY, TOUCH>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess) return -1;
	int per_sm = 0;
	if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_get_small<VERIFY, TOUCH>, (int)GS_THREADS, smem) != cudaSuccess) return -1;
	return per_sm * sm_count();
}
int get_small_residency(uint32_t nbytes, bool verify, bool touch) {
	if (touch) return verify ? get_small_residency_of<true, true>(nbytes) : get_small_residency_of<false, true>(nbytes);
	return verify ? get_small_residency_of<true, false>(nbytes) : get_small_residency_of<false, false>(nbytes);
}

// ------------------------------------------------------------------------------------------
// fingerprint alone, stream generator, small launchers
// ------------------------------------------------------------------------------------------

__global__ void __launch_bounds__(256) k_fingerprint(const uint8_t *pages, uint64_t stride, uint32_t nbytes,
    uint32_t n, uint64_t *fps) {
	const int lane = threadIdx.x & 31;
	const uint32_t i = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
	if (i >= n) return;
	uint64_t hi, lo;
	warp_fingerprint128(pages + (size_t)i * stride, nbytes, lane, hi, lo);
	if (lane == 0) { fps[2 * (size_t)i] = hi; fps[2 * (size_t)i + 1] = lo; }
}

int launch_fingerprint(const uint8_t *pages, uint64_t stride, uint32_t nbytes, uint32_t n, uint64_t *fps,
    cudaStream_t st) {
	if (n == 0) return 0;
	const int warps = 8;
	k_fingerprint<<<(n + warps - 1) / warps, warps * 32, 0, st>>>(pages, stride, nbytes, n, fps);
	CMB_CHECK(cudaGetLastError());
	return 0;
}

__global__ void k_streamgen(const uint64_t *cids, uint32_t n, uint64_t seed, uint32_t bsize, uint8_t *out) {
	const uint32_t words = bsize / 8;
	const uint64_t total = (uint64_t)n * words;
	for (uint64_t g = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; g < total;
	     g += (uint64_t)gridDim.x * blockDim.x) {
		uint32_t c = (uint32_t)(g / words), w = (uint32_t)(g % words);
		reinterpret_cast<uint64_t *>(out)[g] = sg_chunk_word(seed, cids[c], bsize, w);
	}
}

int launch_streamgen(const uint64_t *cids, uint32_t n, uint64_t seed, uint32_t bsize, uint8_t *out,
    cudaStream_t st) {
	if (n == 0) return 0;
	k_streamgen<<<sm_count() * 8, 256, 0, st>>>(cids, n, seed, bsize, out);
	CMB_CHECK(cudaGetLastError());
	return 0;
}

#define GRID1D(n) (((n) + 255u) / 256u), 256

int launch_compose(const uint64_t *offset, const uint64_t *nhid, const uint32_t *genid, int pshift,
    uint32_t n, unsigned long long *addr, uint8_t *valid, unsigned long long *key, cudaStream_t st) {
	if (n == 0) return 0;
	k_compose<<<GRID1D(n), 0, st>>>(offset, nhid, genid, pshift, n, addr, valid, key);
	CMB_CHECK(cudaGetLastError());
	return 0;
}
// ---- multi-GPU exchange records, device resident ------------------------------------------------
// One 32-byte record per chunk of a put step: {u, l, global stream position, tail}; tail is
// xrec_tail(owner rank, arena offset, stored length) (kernels.h; edge_fuse_b200/sharding.py has the
// same layout).
__global__ void k_pack_records(const unsigned long long *addr, const int32_t *lens, const unsigned long long *rec_off,
    uint32_t n, unsigned long long seq0, unsigned long long stride, uint32_t rank, unsigned long long *out) {
	uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= n) return;
	ulonglong2 a = *reinterpret_cast<const ulonglong2 *>(addr + 2 * (size_t)i);
	ulonglong2 b;
	b.x = seq0 + stride * i;
	int32_t len = lens[i];
	unsigned long long off = (len >= 0 && rec_off) ? rec_off[i] : 0ull;
	if (off == ~0ull) { len = -1; off = 0; }        // the put was dropped (arena full)
	b.y = xrec_tail(rank, off, len);
	reinterpret_cast<ulonglong2 *>(out)[2 * (size_t)i] = a;
	reinterpret_cast<ulonglong2 *>(out)[2 * (size_t)i + 1] = b;
}
int launch_pack_records(const unsigned long long *addr, const int32_t *lens, const unsigned long long *rec_off, uint32_t n,
    unsigned long long seq0, unsigned long long stride, uint32_t rank, unsigned long long *out, cudaStream_t st) {
	if (n == 0) return 0;
	k_pack_records<<<GRID1D(n), 0, st>>>(addr, lens, rec_off, n, seq0, stride, rank, out);
	CMB_CHECK(cudaGetLastError());
	return 0;
}
// Import straight from all-gathered records: rows of `my_rank` and rows that stored nothing are skipped.
// Phase 1 claims the slot and records stream order; phase 2: the newest sequence per key applies
// itself (a key may appear several times in one import).
__global__ void k_import_claim_rec(TableView t, const unsigned long long *rec, uint32_t n, uint32_t my_rank,
    uint32_t *slot_idx) {
	uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= n) return;
	const unsigned long long tail = rec[4 * (size_t)i + 3];
	uint32_t idx = 0xffffffffu;
	if (xrec_owner(tail) != my_rank && xrec_len1(tail) != 0u) {
		idx = table_find_or_claim(t, fnv_addr(rec[4 * (size_t)i], rec[4 * (size_t)i + 1]));
		if (idx != 0xffffffffu) atomicMax(&t.slots[idx].seq, rec[4 * (size_t)i + 2]);
	}
	slot_idx[i] = idx;
}
__global__ void k_import_apply_rec(TableView t, ArenaView a, const unsigned long long *rec, uint32_t n,
    const uint32_t *slot_idx) {
	uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= n) return;
	uint32_t idx = slot_idx[i];
	if (idx == 0xffffffffu) return;
	Slot &s = t.slots[idx];
	if (s.seq != rec[4 * (size_t)i + 2]) return;  // an even newer put (local or imported) owns the key
	if (s.vlen) {                                 // our local record is superseded
		atomicAdd(t.entries, (unsigned long long)-1ll);
		atomicAdd(a.garbage, (unsigned long long)s.alloc);
		s.vlen = 0; s.alloc = 0;
	}
	if (s.owner == 0) atomicAdd(t.remote, 1ull);
	const unsigned long long tail = rec[4 * (size_t)i + 3];
	s.addr_u = rec[4 * (size_t)i]; s.addr_l = rec[4 * (size_t)i + 1];
	// where the record lies in the owner's arena (vlen stays 0: no local record)
	s.rec_off = xrec_off(tail); s.alloc = xrec_len1(tail);
	if (t.fp_tag) t.fp_tag[idx] = 0u;                 // the exchange record carries no fingerprint
	__threadfence();
	s.owner = (unsigned long long)xrec_owner(tail) + 1;
}
int launch_import_records(TableView t, ArenaView a, const unsigned long long *rec, uint32_t n, uint32_t my_rank,
    uint32_t *slot_idx, cudaStream_t st) {
	if (n == 0) return 0;
	k_import_claim_rec<<<GRID1D(n), 0, st>>>(t, rec, n, my_rank, slot_idx);
	CMB_CHECK(cudaGetLastError());
	k_import_apply_rec<<<GRID1D(n), 0, st>>>(t, a, rec, n, slot_idx);
	CMB_CHECK(cudaGetLastError());
	return 0;
}

int launch_upsert(TableView t, const unsigned long long *addr, const uint8_t *valid, uint32_t n,
    unsigned long long seq0, unsigned long long seq_stride, uint32_t *slot_idx, cudaStream_t st) {
	if (n == 0) return 0;
	k_upsert<<<GRID1D(n), 0, st>>>(t, addr, valid, n, seq0, seq_stride, slot_idx);
	CMB_CHECK(cudaGetLastError());
	return 0;
}
int launch_lookup(TableView t, const unsigned long long *addr, const uint8_t *valid, uint32_t n,
    int32_t *status, uint64_t *rec_off, uint32_t *vlen, unsigned long long *ts_out, cudaStream_t st, uint32_t *idx_out) {
	if (n == 0) return 0;
	k_lookup<<<GRID1D(n), 0, st>>>(t, addr, valid, n, status, rec_off, vlen, ts_out, idx_out);
	CMB_CHECK(cudaGetLastError());
	return 0;
}
int launch_unset(TableView t, ArenaView a, const unsigned long long *addr, uint32_t n, cudaStream_t st) {
	if (n == 0) return 0;
	k_unset<<<GRID1D(n), 0, st>>>(t, a, addr, n);
	CMB_CHECK(cudaGetLastError());
	return 0;
}
int launch_invalidate(TableView t, ArenaView a, unsigned long long u, unsigned long long l_first,
    unsigned long long l_last, bool scan, unsigned long long *removed, cudaStream_t st) {
	if (scan) {
		const uint64_t n = t.cap + 2;
		k_invalidate_scan<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(t, a, u, l_first, l_last, removed);
	} else {
		const uint64_t n = l_last - l_first + 1;
		k_invalidate_keys<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(t, a, u, l_first, n, removed);
	}
	CMB_CHECK(cudaGetLastError());
	return 0;
}
__global__ void k_read_fp(TableView t, const unsigned long long *addr, uint32_t n, uint64_t *fp_out, int32_t *ok) {
	uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= n) return;
	unsigned long long u = addr[2 * i], l = addr[2 * i + 1];
	uint32_t idx = table_find(t, fnv_addr(u, l));
	int32_t found = 0;
	if (idx != 0xffffffffu && t.slots[idx].vlen != 0 && t.slots[idx].addr_u == u && t.slots[idx].addr_l == l) {
		fp_out[2 * i] = t.fp[2 * (size_t)idx]; fp_out[2 * i + 1] = t.fp[2 * (size_t)idx + 1];
		found = 1;
	}
	ok[i] = found;
}
int launch_read_fp(TableView t, const unsigned long long *addr, uint32_t n, uint64_t *fp_out, int32_t *ok,
    cudaStream_t st) {
	if (n == 0) return 0;
	k_read_fp<<<GRID1D(n), 0, st>>>(t, addr, n, fp_out, ok);
	CMB_CHECK(cudaGetLastError());
	return 0;
}
__global__ void k_read_ckpt(TableView t, const unsigned long long *addr, uint32_t n, uint32_t *words_out, int32_t *ok) {
	uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= n) return;
	unsigned long long u = addr[2 * i], l = addr[2 * i + 1];
	uint32_t idx = table_find(t, fnv_addr(u, l));
	int32_t found = -1;
	uint32_t *w = words_out + (size_t)i * CKPT_WORDS;
	for (uint32_t k = 0; k < CKPT_WORDS; k++) w[k] = 0;
	if (idx != 0xffffffffu) {
		const Slot &s = t.slots[idx];
		if (s.vlen != 0 && s.owner == 0 && s.addr_u == u && s.addr_l == l) {
			for (uint32_t k = 0; k < CKPT_WORDS; k++) w[k] = t.ckpt[(size_t)idx * CKPT_WORDS + k];
			found = w[0] == ckpt_tag(s.rec_off, s.vlen - 1u) ? 1 : 0;
		}
	}
	ok[i] = found;
}
int launch_read_ckpt(TableView t, const unsigned long long *addr, uint32_t n, uint32_t *words_out, int32_t *ok,
    cudaStream_t st) {
	if (n == 0) return 0;
	k_read_ckpt<<<GRID1D(n), 0, st>>>(t, addr, n, words_out, ok);
	CMB_CHECK(cudaGetLastError());
	return 0;
}
// ---- snapshot -----------------------------------------------------------------------------
__global__ void k_export_list(TableView t, uint32_t bsize, ExportEntry *out, unsigned long long *count,
    unsigned long long max_out, bool arena_only, unsigned long long seq_min, ulonglong2 *addr_out) {
	const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= t.cap + 2) return;
	const Slot &s = t.slots[i];
	if (s.vlen == 0 || s.owner != 0) return;        // empty / deleted / the record lives on another GPU
	if (arena_only && (s.rec_off & REC_HOST)) return;
	if (i < t.cap && (s.key == KEY_EMPTY || s.key == KEY_TOMB)) return;
	if (addr_out) {
		const unsigned long long k = atomicAdd(count + 1, 1ull);
		if (k < max_out) addr_out[k] = make_ulonglong2(s.addr_u, s.addr_l);
	}
	if (s.seq < seq_min) return;                    // put before the watermark: in an earlier file of the chain
	const unsigned long long j = atomicAdd(count, 1ull);
	if (j >= max_out) return;
	ExportEntry e;
	e.rec_off = s.rec_off; e.ts = s.ts;
	// {0, 0} = no fingerprint: a record loaded without one keeps none (with CMB200_VERIFY its tag says
	// whether fp belongs to this record; without it, fp of such a record is {0, 0} already)
	const bool has_fp = t.fp && (!t.fp_tag || t.fp_tag[i] == ckpt_tag(s.rec_off, s.vlen - 1u));
	e.fp_hi = has_fp ? t.fp[2 * i] : 0ull; e.fp_lo = has_fp ? t.fp[2 * i + 1] : 0ull;
	e.len = 24u + (s.vlen > 1u ? s.vlen - 1u : bsize);
	e.slot = (uint32_t)i;
	out[j] = e;
}
int launch_export_list(TableView t, uint32_t bsize, ExportEntry *out, unsigned long long *count,
    unsigned long long max_out, bool arena_only, cudaStream_t st, unsigned long long seq_min, ulonglong2 *addr_out) {
	const uint64_t n = t.cap + 2;
	k_export_list<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(t, bsize, out, count, max_out, arena_only, seq_min, addr_out);
	CMB_CHECK(cudaGetLastError());
	return 0;
}
// One thread per address of the previous tick's baseline (page-locked host memory read over PCIe, so
// 16-byte loads that bypass L1): a tombstone for each address that no longer holds a live local record.
__global__ void k_delta_gone(TableView t, const ulonglong2 *base, uint64_t n, ulonglong2 *out, unsigned long long *count) {
	const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= n) return;
	const ulonglong2 a = __ldcg(base + i);
	const uint32_t idx = table_find(t, fnv_addr(a.x, a.y));
	if (idx != 0xffffffffu) {
		const Slot &s = t.slots[idx];
		if (s.vlen != 0 && s.owner == 0 && s.addr_u == a.x && s.addr_l == a.y) return;
	}
	out[atomicAdd(count, 1ull)] = a;
}
int launch_delta_gone(TableView t, const ulonglong2 *base, uint64_t n, ulonglong2 *out, unsigned long long *count,
    cudaStream_t st) {
	if (n == 0) return 0;
	k_delta_gone<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(t, base, n, out, count);
	CMB_CHECK(cudaGetLastError());
	return 0;
}
__global__ void k_scan_prep(TableView t, const ExportEntry *list, uint32_t n, int32_t *status, uint64_t *rec_off,
    uint32_t *vlen, uint32_t *idx, unsigned long long *addr) {
	const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= n) return;
	const ExportEntry x = list[i];
	const Slot &s = t.slots[x.slot];
	status[i] = ST_HIT; rec_off[i] = x.rec_off; vlen[i] = s.vlen; idx[i] = x.slot;
	addr[2 * (size_t)i] = s.addr_u; addr[2 * (size_t)i + 1] = s.addr_l;
}
int launch_scan_prep(TableView t, const ExportEntry *list, uint32_t n, int32_t *status, uint64_t *rec_off,
    uint32_t *vlen, uint32_t *idx, unsigned long long *addr, cudaStream_t st) {
	if (n == 0) return 0;
	k_scan_prep<<<GRID1D(n), 0, st>>>(t, list, n, status, rec_off, vlen, idx, addr);
	CMB_CHECK(cudaGetLastError());
	return 0;
}

// Parse checkpoints of a block that arrives without them (a snapshot record), by walking its token
// chain: the same words as the encoder's (lz4_encode_lean), lane k gets word k.  Every lane walks
// the same chain out of a per-warp window of the block in shared memory, which the warp refills
// when the walk leaves it; only [blk, blk + clen) is read.  The block is untrusted: a chain that
// does not end exactly at (consumed == clen, output == n), or whose runs pass the page end, gives
// false and no checkpoints.
constexpr uint32_t RESTORE_WARPS = 8, RESTORE_WIN = 1024;
__device__ bool restore_ckpt_walk(const uint8_t *blk, uint32_t clen, uint32_t n, uint8_t *win, int lane, uint32_t &ck) {
	const uint32_t S = n / CKPT_WORDS;
	uint32_t ip = 0, op = 0, k = 1, wb = 0, we = 0;
	ck = 0xffffffffu;
	// byte p of the block, p < clen; positions only grow along the chain
	auto at = [&](uint32_t p) -> uint32_t {
		if (p >= we) {
			__syncwarp();
			wb = p; we = min(p + RESTORE_WIN, clen);
			for (uint32_t q = wb + (uint32_t)lane; q < we; q += 32u) win[q - wb] = blk[q];
			__syncwarp();
		}
		return win[p - wb];
	};
	for (;;) {
		// a sequence starts at token ip, its literals at output position op
		for (; k < CKPT_WORDS && op >= k * S; k++)
			if ((uint32_t)lane == k) ck = op - k * S < S ? (ip << CKPT_POS_BITS) | (op - k * S) : 0xffffffffu;
		if (ip >= clen) return false;
		const uint32_t tok = at(ip++);
		uint32_t lit = tok >> 4;
		if (lit == 15u) {
			uint32_t b;
			do {
				if (ip >= clen) return false;
				b = at(ip++);
				lit += b;
			} while (b == 255u && lit <= n);
		}
		if (lit > n - op || lit > clen - ip) return false;
		ip += lit; op += lit;
		if (ip == clen) break;                              // the last literals
		if (clen - ip < 2u) return false;
		ip += 2;                                            // match offset
		uint32_t mlen = tok & 15u;
		if (mlen == 15u) {
			uint32_t b;
			do {
				if (ip >= clen) return false;
				b = at(ip++);
				mlen += b;
			} while (b == 255u && mlen <= n);
		}
		if (mlen + 4u > n - op) return false;
		op += mlen + 4u;
	}
	if (op != n) return false;
	for (; k < CKPT_WORDS; k++) if ((uint32_t)lane == k) ck = 0xffffffffu;   // no sequence starts at or after k * S
	return true;
}

__global__ void __launch_bounds__(RESTORE_WARPS * 32) k_restore(EncodeJob job, const uint8_t *blob, const unsigned long long *off,
    const uint64_t *fps, uint32_t bsize) {
	__shared__ uint8_t win[RESTORE_WARPS][RESTORE_WIN];
	const int lane = threadIdx.x & 31;
	const uint32_t i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
	if (i >= job.n) return;
	const uint32_t idx = job.slot_idx[i];
	if (idx == 0xffffffffu || job.table.slots[idx].seq != job.seq0 + job.seq_stride * i) return;
	const uint8_t *rec = blob + off[i];
	const int32_t clen = *reinterpret_cast<const int32_t *>(rec + 16);   // data_prefix.compressed_length (filemap.c:9-12); off[] is 16-aligned
	const uint32_t plen = clen > 0 ? (uint32_t)clen : bsize;
	// a record saved without a fingerprint carries {0, 0} even in a file whose header says it has them
	// (cmb200_save writes every record of the store): it stays unverified
	const uint64_t fp_hi = fps ? fps[2 * i] : 0ull, fp_lo = fps ? fps[2 * i + 1] : 0ull;
	const unsigned long long at =
	    commit_record(job, i, idx, rec + 24, plen, clen, true, fp_hi, fp_lo, lane, (fp_hi | fp_lo) != 0ull);
	// the encoder's checkpoints, rebuilt from the block (raw pages have none); slot_publish has zeroed
	// the tag, so a block that does not walk leaves the record to the one-warp parse of k_get_small
	if (at == ~0ull || clen <= 0 || !job.table.ckpt) return;
	uint32_t ck;
	if (restore_ckpt_walk(rec + 24, (uint32_t)clen, bsize, win[threadIdx.x >> 5], lane, ck))
		ckpt_store(job, idx, at, (uint32_t)clen, ck, lane);
}
int launch_restore(const EncodeJob &job, const uint8_t *blob, const unsigned long long *off,
    const uint64_t *fps, uint32_t bsize, cudaStream_t st) {
	if (job.n == 0) return 0;
	k_restore<<<(job.n + RESTORE_WARPS - 1) / RESTORE_WARPS, RESTORE_WARPS * 32, 0, st>>>(job, blob, off, fps, bsize);
	CMB_CHECK(cudaGetLastError());
	return 0;
}

// ---- arena compaction ---------------------------------------------------------------------
// moves[i].new_off - moves[0].new_off is also the record's place in the bounce buffer (records are
// packed in the same order and with the same 16-byte rounding in both).
__global__ void __launch_bounds__(256) k_compact_gather(ArenaView a, const MoveEntry *moves, uint32_t n, uint8_t *bounce) {
	const int lane = threadIdx.x & 31;
	const uint32_t i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
	if (i >= n) return;
	const MoveEntry m = moves[i];
	warp_copy_rw(bounce + (m.new_off - moves[0].new_off), a.base + m.old_off, m.len, lane);
}
__global__ void __launch_bounds__(256) k_compact_scatter(TableView t, ArenaView a, const MoveEntry *moves, uint32_t n,
    const uint8_t *bounce) {
	const int lane = threadIdx.x & 31;
	const uint32_t i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
	if (i >= n) return;
	const MoveEntry m = moves[i];
	warp_copy_rw(a.base + m.new_off, bounce + (m.new_off - moves[0].new_off), m.len, lane);
	if (lane == 0) {
		Slot &s = t.slots[m.slot];
		s.rec_off = m.new_off;
		s.alloc = (m.len + 15u) & ~15u;
		ckpt_retag(t, m.slot, m.old_off, m.new_off, s.vlen - 1u);
	}
}
int launch_compact_window(TableView t, ArenaView a, const MoveEntry *moves, uint32_t n, uint8_t *bounce,
    cudaStream_t st) {
	if (n == 0) return 0;
	k_compact_gather<<<(n * 32 + 255) / 256, 256, 0, st>>>(a, moves, n, bounce);
	CMB_CHECK(cudaGetLastError());
	k_compact_scatter<<<(n * 32 + 255) / 256, 256, 0, st>>>(t, a, moves, n, bounce);
	CMB_CHECK(cudaGetLastError());
	return 0;
}

// ---- host tier ---------------------------------------------------------------------------------
// Demotion: gather the records into the bounce buffer in tier order (one warp per record), let the copy
// engine move the buffer to the tier, then repoint the slots.
__global__ void __launch_bounds__(256) k_demote_gather(ArenaView a, const DemoteEntry *d, uint32_t n, uint8_t *bounce) {
	const int lane = threadIdx.x & 31;
	const uint32_t i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
	if (i >= n) return;
	const DemoteEntry m = d[i];
	warp_copy_rw(bounce + m.bounce_off, a.base + m.old_off, m.len, lane);
}
__global__ void k_demote_publish(TableView t, ArenaView a, const DemoteEntry *d, uint32_t n) {
	const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= n) return;
	const DemoteEntry m = d[i];
	// the arena copy is intact until the next compaction: its prefix names the key
	const unsigned long long *pre = reinterpret_cast<const unsigned long long *>(a.base + m.old_off);
	const uint32_t idx = table_find(t, fnv_addr(pre[0], pre[1]));
	if (idx == 0xffffffffu) return;
	Slot &s = t.slots[idx];
	if (s.vlen == 0 || s.owner != 0 || s.rec_off != m.old_off) return;   // not the record that was copied
	const uint32_t clen = s.vlen - 1u;
	const unsigned long long loc = REC_HOST | m.host_off;
	atomicAdd(a.garbage, (unsigned long long)s.alloc);
	atomicAdd(a.tier + 1, 1ull);
	s.alloc = (m.len + 15u) & ~15u;
	*reinterpret_cast<volatile unsigned long long *>(&s.rec_off) = loc;      // the one store readers trust
	ckpt_retag(t, idx, m.old_off, loc, clen);
}
int launch_demote_gather(ArenaView a, const DemoteEntry *d, uint32_t n, uint8_t *bounce, cudaStream_t st) {
	if (n == 0) return 0;
	k_demote_gather<<<(n * 32 + 255) / 256, 256, 0, st>>>(a, d, n, bounce);
	CMB_CHECK(cudaGetLastError());
	return 0;
}
int launch_demote_publish(TableView t, ArenaView a, const DemoteEntry *d, uint32_t n, cudaStream_t st) {
	if (n == 0) return 0;
	k_demote_publish<<<GRID1D(n), 0, st>>>(t, a, d, n);
	CMB_CHECK(cudaGetLastError());
	return 0;
}

// Promotion: one warp per record copies it from the mapped tier into the arena above the old bump
// pointer (16-byte loads past the L1, as k_get_small reads the tier), then lane 0 repoints the slot.
__global__ void __launch_bounds__(256) k_promote(TableView t, ArenaView a, const PromoteEntry *p, uint32_t n,
    const uint8_t *host) {
	const int lane = threadIdx.x & 31;
	const uint32_t i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
	if (i >= n) return;
	const PromoteEntry m = p[i];
	const uint32_t need = (m.len + 15u) & ~15u;
	const uint4 *src = reinterpret_cast<const uint4 *>(host + m.host_off);
	uint4 *dst = reinterpret_cast<uint4 *>(a.base + m.new_off);
	for (uint32_t k = lane; k < need / 16u; k += 32) dst[k] = __ldcg(src + k);
	__threadfence();                                 // the record is complete before the slot points to it
	__syncwarp();
	if (lane != 0) return;
	// the record's own prefix names the key, as in k_demote_publish
	const unsigned long long *pre = reinterpret_cast<const unsigned long long *>(a.base + m.new_off);
	const unsigned long long loc = REC_HOST | m.host_off;
	const uint32_t idx = table_find(t, fnv_addr(pre[0], pre[1]));
	Slot *s = idx == 0xffffffffu ? nullptr : &t.slots[idx];
	if (!s || s->vlen == 0 || s->owner != 0 || s->rec_off != loc) {
		atomicAdd(a.garbage, (unsigned long long)need);          // not the record that was copied
		return;
	}
	const uint32_t clen = s->vlen - 1u;
	atomicAdd(a.tier, (unsigned long long)s->alloc);           // the tier copy is dead bytes until the ring laps it
	atomicAdd(a.tier + 1, (unsigned long long)-1ll);
	s->alloc = need;
	*reinterpret_cast<volatile unsigned long long *>(&s->rec_off) = m.new_off;   // the one store readers trust
	ckpt_retag(t, idx, loc, m.new_off, clen);
}
int launch_promote(TableView t, ArenaView a, const PromoteEntry *p, uint32_t n, const uint8_t *host, cudaStream_t st) {
	if (n == 0) return 0;
	k_promote<<<(n * 32 + 255) / 256, 256, 0, st>>>(t, a, p, n, host);
	CMB_CHECK(cudaGetLastError());
	return 0;
}

// Conditional unset of the records a wrap of the tier overwrites: rec[4i..4i+3] = {u, l, location, bytes}.
__global__ void k_tier_retire(TableView t, ArenaView a, const unsigned long long *rec, uint32_t n,
    unsigned long long *retired) {
	const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= n) return;
	const unsigned long long loc = rec[4 * (size_t)i + 2], bytes = rec[4 * (size_t)i + 3];
	const uint32_t idx = table_find(t, fnv_addr(rec[4 * (size_t)i], rec[4 * (size_t)i + 1]));
	if (idx != 0xffffffffu) {
		Slot &s = t.slots[idx];
		// a location names one record, so no two requests of a batch can both match
		if (s.vlen != 0 && s.rec_off == loc) {
			s.vlen = 0;
			atomicAdd(t.entries, (unsigned long long)-1ll);        // an eviction, counted as k_unset counts it
			atomicAdd(a.tier + 1, (unsigned long long)-1ll);
			s.alloc = 0;
			s.owner = 0;
			if (t.fp_tag) t.fp_tag[idx] = 0u;
			if (idx < t.cap) {
				s.key = KEY_TOMB;
				atomicAdd(t.tombs, 1ull);
			}
			atomicAdd(retired, 1ull);
			return;
		}
	}
	atomicAdd(a.tier, 0ull - bytes);                         // a dead record: its bytes leave the tier's garbage
}
int launch_tier_retire(TableView t, ArenaView a, const unsigned long long *rec, uint32_t n,
    unsigned long long *retired, cudaStream_t st) {
	if (n == 0) return 0;
	k_tier_retire<<<GRID1D(n), 0, st>>>(t, a, rec, n, retired);
	CMB_CHECK(cudaGetLastError());
	return 0;
}

// ---- table rebuild ---------------------------------------------------------------------------
// Linear probing never gives a slot back: a deleted key leaves a tombstone and a key whose put was
// dropped leaves a claimed slot without a record, so over a long run the EMPTY slots only shrink and
// miss probes walk ever longer chains.  The rebuild re-inserts what is alive (a local record or a
// remote owner) into a fresh table of the same size; everything else disappears.
__global__ void k_rehash(TableView from, TableView to) {
	const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= from.cap + 2) return;
	const Slot s = from.slots[i];
	if (s.vlen == 0 && s.owner == 0) return;
	if (i < from.cap && (s.key == KEY_EMPTY || s.key == KEY_TOMB)) return;
	const unsigned long long key = i < from.cap ? s.key : (i == from.cap ? KEY_EMPTY : KEY_TOMB);
	const uint32_t idx = table_find_or_claim(to, key);
	if (idx == 0xffffffffu) return;                     // cannot happen: same size, fewer keys
	Slot d = s;
	d.key = idx < to.cap ? key : 0ull;
	// the key word was written by the claim; copy the rest field by field so that it is not torn
	Slot &t = to.slots[idx];
	t.addr_u = d.addr_u; t.addr_l = d.addr_l; t.rec_off = d.rec_off; t.vlen = d.vlen; t.alloc = d.alloc;
	t.ts = d.ts; t.seq = d.seq; t.owner = d.owner;
	if (from.fp && to.fp) { to.fp[2 * (size_t)idx] = from.fp[2 * i]; to.fp[2 * (size_t)idx + 1] = from.fp[2 * i + 1]; }
	// the tag names rec_off and the length, which stay: the parse checkpoints move with the slot
	if (from.ckpt && to.ckpt)
		for (uint32_t k = 0; k < CKPT_WORDS; k++) to.ckpt[(size_t)idx * CKPT_WORDS + k] = from.ckpt[i * CKPT_WORDS + k];
	if (from.fp_tag && to.fp_tag) to.fp_tag[idx] = from.fp_tag[i];
}
int launch_rehash(TableView from, TableView to, cudaStream_t st) {
	const uint64_t n = from.cap + 2;
	k_rehash<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(from, to);
	CMB_CHECK(cudaGetLastError());
	return 0;
}

int launch_sample(TableView t, const unsigned long long *r, uint32_t n, unsigned long long *addr_out,
    unsigned long long *ts_out, int32_t *ok, cudaStream_t st) {
	if (n == 0) return 0;
	k_sample<<<GRID1D(n), 0, st>>>(t, r, n, addr_out, ts_out, ok);
	CMB_CHECK(cudaGetLastError());
	k_sample_scan<<<n < 1024u ? n : 1024u, 256, 0, st>>>(t, r, n, addr_out, ts_out, ok);
	CMB_CHECK(cudaGetLastError());
	return 0;
}

// ---- page moves between the engines of a sharded store (cmb200_move_pages) --------------------
// One warp per page: 32 lanes x 16 bytes per step, so a page of nbytes takes ceil(nbytes / 512) steps.
// The pages of one owner are gathered into a contiguous buffer before a peer copy, or scattered
// from one after it.
__global__ void __launch_bounds__(256) k_move_pages(uint4 *dst, const uint32_t *dst_idx, const uint4 *src,
    const uint32_t *src_idx, uint32_t n, uint32_t nbytes) {
	const int lane = threadIdx.x & 31;
	const uint32_t i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
	if (i >= n) return;
	const size_t words = nbytes >> 4;
	uint4 *d = dst + (size_t)(dst_idx ? dst_idx[i] : i) * words;
	const uint4 *s = src + (size_t)(src_idx ? src_idx[i] : i) * words;
	for (size_t w = lane; w < words; w += 32) d[w] = s[w];
}
int launch_move_pages(void *dst, const uint32_t *dst_idx, const void *src, const uint32_t *src_idx, uint32_t n,
    uint32_t nbytes, cudaStream_t st) {
	if (n == 0) return 0;
	k_move_pages<<<(n * 32 + 255) / 256, 256, 0, st>>>((uint4 *)dst, dst_idx, (const uint4 *)src, src_idx, n, nbytes);
	CMB_CHECK(cudaGetLastError());
	return 0;
}

// ---- read-modify-write of stored pages (cmb200_patch_batch) ------------------------------------
// One CTA per page-ring row.  A row that lookup and decode did not answer ST_HIT is left out of the
// upsert (valid = 0); the spans of every other row are copied over its decoded page in array order,
// with a barrier after each, since a later span may overwrite bytes of an earlier one.  The part of a
// span between the 16-byte boundaries of source and destination moves in 16-byte words when the two are
// congruent modulo 16 (the engine lays the bytes out so that they are), the ragged ends byte by byte.
__global__ void __launch_bounds__(256) k_patch(uint8_t *pages, uint32_t nbytes, const int32_t *status,
    const uint32_t *first, const PatchSpan *spans, const uint8_t *bytes, uint8_t *valid) {
	const uint32_t row = blockIdx.x;
	const bool hit = status[row] == ST_HIT;
	if (threadIdx.x == 0) valid[row] = hit;
	if (!hit) return;
	uint8_t *page = pages + (size_t)row * nbytes;
	for (uint32_t k = first[row]; k < first[row + 1]; k++) {
		const PatchSpan s = spans[k];
		uint8_t *dst = page + s.page_off;
		const uint8_t *src = bytes + s.src_off;
		const bool wide = ((s.page_off ^ s.src_off) & 15u) == 0;
		const uint32_t lead = wide ? min((0u - s.page_off) & 15u, s.len) : s.len;
		const uint32_t words = (s.len - lead) >> 4;
		const uint32_t tail = lead + (words << 4);
		for (uint32_t j = threadIdx.x; j < lead; j += blockDim.x) dst[j] = src[j];
		for (uint32_t j = threadIdx.x; j < words; j += blockDim.x)
			reinterpret_cast<uint4 *>(dst + lead)[j] = reinterpret_cast<const uint4 *>(src + lead)[j];
		for (uint32_t j = tail + threadIdx.x; j < s.len; j += blockDim.x) dst[j] = src[j];
		__syncthreads();
	}
}
int launch_patch(uint8_t *pages, uint32_t nbytes, uint32_t rows, const int32_t *status, const uint32_t *first,
    const PatchSpan *spans, const uint8_t *bytes, uint8_t *valid, cudaStream_t st) {
	if (rows == 0) return 0;
	k_patch<<<rows, 256, 0, st>>>(pages, nbytes, status, first, spans, bytes, valid);
	CMB_CHECK(cudaGetLastError());
	return 0;
}

}  // namespace cmb
