// lz4_encode.cuh — byte-exact LZ4 1.8.1 block encoder, one warp per chunk (sm_90a): tables, probe
// neighbourhoods and the out-of-line paths; the loop is lz4_encode_lean in lz4_encode_ring.cuh.
//
// Emits exactly the bytes the reference's filemap_set stores:
//   LZ4_compress_fast(page, dst, n, n+1024, accel)            cachemap/filemap.c:124-128
//   -> LZ4_compress_generic<notLimited, byU16|byU32, noDict>   cachemap/lz4.c:532-733,736-771
// (byU16 + 13-bit hash4 for n < 65547, byU32 + 12-bit hash5 + MAX_DISTANCE test otherwise).
//
// The greedy parse is a serial dependency chain per chunk (every probe reads then writes the
// position table), so throughput = chunks in flight / latency per LZ4 sequence.
//   * Chunks in flight: one independent chunk per warp; the 16 KiB position table lives in shared
//     memory (13-14 chunks per SM) and, by default, a 1 KiB window of the page at the parse
//     frontier, kept filled by TMA (lz4_encode_ring.cuh); candidates are read through the
//     read-only L1 path (ld.global.nc).  Staging the whole 64 KiB page in shared memory would cap
//     residency at two chunks per SM (DESIGN.md §4).
//   * Latency per sequence: the warp runs the reference's loop speculatively, one LZ4 sequence
//     per iteration with ONE table round trip and ONE page round trip:
//       "unified batch": lane 0 replays the table refill of position end-2 (lz4.c:691), lane 1
//         the immediate re-test at `end` (lz4.c:694-707), lanes 2.. the first 30 probes of the
//         following search (lz4.c:593-619; probe positions are a closed form of the probe index:
//         +1, then +accel for 64 probes, +accel+1 for the next 64, ...).  All are "read slot,
//         write slot, compare 4 bytes" in program order.  Every lane stores its position
//         speculatively and reads the slot back; lanes that see a foreign value share a slot
//         with another lane.  Below the lowest such lane program order is irrelevant, so if the
//         first hit (ballot) lies there it wins and the later lanes put the old values back.
//         Otherwise (a true intra-batch dependency, or 30 probes were not enough) the general
//         search lz4_search_slow resolves program order with __match_any_sync.
//       Each lane fetches 12 bytes around its probe and around its candidate in that same round
//         trip, so the winner already knows the match extension up to 4 bytes forward
//         (lz4.c:415-439) and 4 bytes backward (lz4.c:622); longer ones go out of line.
//   * The hot loop is kept small on purpose (the profile of the first version showed a third of
//     the stall samples waiting on instruction fetch): rare paths are __noinline__.
#pragma once
#include "common.cuh"
#include "fingerprint.cuh"

namespace cmb {

constexpr uint32_t LZ4_MIN_MATCH = 4;
constexpr uint32_t LZ4_TAIL_LITERALS = 5;      // lz4.c:296
constexpr uint32_t LZ4_MATCH_FIND_MARGIN = 12; // lz4.c:297
constexpr uint32_t LZ4_MIN_INPUT = 13;         // lz4.c:298
constexpr uint32_t LZ4_NARROW_LIMIT = 65536 + 11;  // lz4.c:446
constexpr uint32_t LZ4_FAR = 65535;            // lz4.c:304-305
constexpr uint32_t LZ4_TABLE_BYTES = 16384;    // lz4.h:120

__device__ __forceinline__ uint32_t lz4_hash4(uint32_t v) { return (v * 2654435761u) >> 19; }
__device__ __forceinline__ uint32_t lz4_hash5(uint64_t v) {
	return (uint32_t)(((v << 24) * 889523592379ULL) >> 52);
}

// Offset of probe k of a search from its first probe position (lz4.c:594-600).
__device__ __forceinline__ uint32_t lz4_probe_off(uint32_t k, uint32_t accel) {
	if (k == 0) return 0;
	uint32_t m = k - 1, q = m >> 6, r = m & 63u;
	return 1u + accel * m + 32u * q * (q - 1u) + q * r;
}

template <bool WIDE> struct Lz4Table;
template <> struct Lz4Table<false> {
	uint16_t *t;
	__device__ __forceinline__ uint32_t get(uint32_t h) const { return t[h]; }
	__device__ __forceinline__ void put(uint32_t h, uint32_t pos) const { t[h] = (uint16_t)pos; }
};
template <> struct Lz4Table<true> {
	uint32_t *t;
	__device__ __forceinline__ uint32_t get(uint32_t h) const { return t[h]; }
	__device__ __forceinline__ void put(uint32_t h, uint32_t pos) const { t[h] = pos; }
};

// The 12 bytes [p-4, p+8) of the page as three little-endian words {before, at, next}: four
// aligned loads (page buffers are padded past their end; the word before the page start is never
// needed because backward extension is capped by the position itself).
struct Lz4Around { uint32_t before, at, next; };
// The same in two halves, the loads and the byte alignment, for a caller that has other work to
// do while the loads are in flight.
struct Lz4Words { uint32_t w0, w1, w2, w3, sh; };
__device__ __forceinline__ Lz4Words lz4_around_load(const uint8_t *src, uint32_t p) {
	const uint32_t a = p & ~3u;
	const uint32_t *q = reinterpret_cast<const uint32_t *>(src + a);
	// p < 4: the word before the page does not exist and is not needed (backward extension is capped
	// by the position), so the first word is read twice instead of branching
	Lz4Words w;
	w.w0 = __ldg(q - (a != 0u));
	w.w1 = __ldg(q); w.w2 = __ldg(q + 1); w.w3 = __ldg(q + 2);
	w.sh = (p & 3u) * 8u;
	return w;
}
__device__ __forceinline__ Lz4Around lz4_around_align(const Lz4Words &w) {
	Lz4Around r;
	r.before = __funnelshift_r(w.w0, w.w1, w.sh);
	r.at = __funnelshift_r(w.w1, w.w2, w.sh);
	r.next = __funnelshift_r(w.w2, w.w3, w.sh);
	return r;
}
__device__ __forceinline__ Lz4Around lz4_around(const uint8_t *src, uint32_t p) {
	return lz4_around_align(lz4_around_load(src, p));
}

// ---- rare paths, kept out of line ------------------------------------------------------------

// Emits `count` as LZ4 length-extension bytes at dst[op..): count/255 bytes of 0xFF then count%255.
__device__ __noinline__ uint32_t lz4_emit_len(uint8_t *dst, uint32_t op, uint32_t count, int lane) {
	uint32_t nff = count / 255u;
	for (uint32_t i = lane; i < nff; i += 32) dst[op + i] = 0xFF;
	if (lane == 0) dst[op + nff] = (uint8_t)(count - nff * 255u);
	return op + nff + 1;
}
// The number of bytes lz4_emit_len writes for a token field that holds `count` (none below 15).
__device__ __forceinline__ uint32_t lz4_len_bytes(uint32_t count) { return count >= 15u ? (count - 15u) / 255u + 1u : 0u; }
// Size of a whole sequence: token, literal length bytes, literals, offset, match length bytes.
__device__ __forceinline__ uint32_t lz4_seq_bytes(uint32_t lit, uint32_t mc) {
	return 3u + lit + lz4_len_bytes(lit) + lz4_len_bytes(mc);
}

__device__ __noinline__ void lz4_copy_literals(uint8_t *dst, const uint8_t *src, uint32_t len, int lane) {
	warp_copy_ro(dst, src, len, lane);
}

// Common prefix length of src[a..) and src[b..), the a side capped at `lim` (lz4.c:415-439);
// 512 bytes per step for the long matches of repetitive pages.
__device__ __noinline__ uint32_t lz4_count_long(const uint8_t *src, uint32_t a, uint32_t b, uint32_t lim,
    uint32_t lim4, int lane) {
	// most matches that outgrow the neighbourhoods end within the next few bytes: one byte per lane first
	{
		const uint32_t pa = a + (uint32_t)lane;
		const bool same = pa < lim && ldg8(src + pa) == ldg8(src + b + (uint32_t)lane);
		const uint32_t stop = __ballot_sync(CMB_FULL, !same);
		if (stop) return (uint32_t)(__ffs(stop) - 1);
	}
	uint32_t total = 32;
	for (;;) {
		const uint32_t pa = a + total + 16u * lane;
		uint32_t nb = 0;                                  // equal bytes in this lane's 16
		if (pa < lim) {
			const uint32_t avail = min(16u, lim - pa);
			const uint32_t pb = b + total + 16u * lane;
			// both 16-byte windows are loaded at once (one L2 round trip per step), then compared
			uint32_t wa[5], wb[5];
			const uint32_t qa = pa & ~3u, qb = pb & ~3u;
#pragma unroll
			for (uint32_t k = 0; k < 5; k++) {
				wa[k] = qa + 4u * k < lim4 ? ldg32(src + qa + 4u * k) : 0u;
				wb[k] = qb + 4u * k < lim4 ? ldg32(src + qb + 4u * k) : 0u;
			}
#pragma unroll
			for (uint32_t j = 0; j < 4; j++) {
				if (nb == 4u * j) {
					const uint32_t x = __funnelshift_r(wa[j], wa[j + 1], (pa & 3u) * 8u) ^
					    __funnelshift_r(wb[j], wb[j + 1], (pb & 3u) * 8u);
					nb += x ? (uint32_t)(__ffs(x) - 1) >> 3 : 4u;
				}
			}
			nb = min(nb, avail);
		}
		const uint32_t stop = __ballot_sync(CMB_FULL, nb < 16u);
		if (stop) {
			int f = __ffs(stop) - 1;
			return total + 16u * f + __shfl_sync(CMB_FULL, nb, f);
		}
		total += 512u;
	}
}

// Backward extension (lz4.c:622) continuing from (ip, match): returns extra steps.
__device__ __noinline__ uint32_t lz4_catchup_long(const uint8_t *src, uint32_t ip, uint32_t match,
    uint32_t anchor, int lane) {
	uint32_t total = 0;
	for (;;) {
		uint32_t k = total + lane + 1;
		bool ok = ip >= anchor + k && match >= k && ldg8(src + ip - k) == ldg8(src + match - k);
		uint32_t fail = __ballot_sync(CMB_FULL, !ok);
		if (fail) return total + (uint32_t)(__ffs(fail) - 1);
		total += 32;
	}
}

// Result of a search, packed so that the out-of-line function returns in registers:
// bit 63 found, bit 62 hit was the re-test lane, bits 32..61 ip, bits 0..31 match.
__device__ __forceinline__ uint64_t lz4_pack(bool found, bool retest, uint32_t ip, uint32_t match) {
	return ((uint64_t)found << 63) | ((uint64_t)retest << 62) | ((uint64_t)ip << 32) | match;
}

// The general search (any number of probes, any hash clashes).  Slot g of the search is the
// refill (g = 0) / re-test (g = 1) when g < shift, else probe g - shift; starts at slot g0.
// specials = false: the two special slots exist in the numbering but do nothing (first search of
// a chunk in the ring encoder, which keeps one lane layout for every batch).
template <bool WIDE>
__device__ __noinline__ uint64_t lz4_search_slow(const uint8_t *src, uint32_t lim4, Lz4Table<WIDE> tab,
    uint32_t anchor, uint32_t shift, uint32_t accel, uint32_t mflimit, uint32_t g0, int lane, bool specials = true) {
	const uint32_t p0 = anchor + 1;
	for (;; g0 += 32) {
		const uint32_t g = g0 + lane;
		const bool special = g < shift;
		const uint32_t k = g - shift;
		uint32_t pos = p0 + lz4_probe_off(k, accel);
		const uint32_t nxt = p0 + lz4_probe_off(k + 1, accel);
		bool en = nxt <= mflimit;
		if (special) { pos = anchor - 2u + 2u * g; en = specials; }
		uint32_t h = 0x10000u + lane, pseq = 0, cand = 0;
		if (en) {
			if (WIDE) { uint64_t v = read64u(src, pos, lim4); pseq = (uint32_t)v; h = lz4_hash5(v); }
			else { pseq = read32u(src, pos, lim4); h = lz4_hash4(pseq); }
			cand = tab.get(h);
		}
		const uint32_t peers = __match_any_sync(CMB_FULL, h);
		const uint32_t lower = peers & ((1u << lane) - 1u);
		const uint32_t prev_pos = __shfl_sync(CMB_FULL, pos, lower ? 31 - __clz(lower) : lane);
		if (lower) cand = prev_pos;          // what the serial loop would have stored by then
		bool hit = false;
		if (en && !(special && g == 0) && cand + LZ4_FAR >= pos)
			hit = read32u(src, cand, lim4) == pseq;
		const uint32_t hits = __ballot_sync(CMB_FULL, hit);
		const uint32_t enmask = __ballot_sync(CMB_FULL, en);
		const int w = hits ? __ffs(hits) - 1 : 31;
		const uint32_t commit = hits ? (0xffffffffu >> (31 - w)) & enmask : enmask;
		if ((commit >> lane) & 1u) {
			const uint32_t pc = peers & commit;
			if (31 - __clz(pc) == lane) tab.put(h, pos);     // last writer per slot wins
		}
		__syncwarp();
		if (hits)
			return lz4_pack(true, g0 + (uint32_t)w < shift, __shfl_sync(CMB_FULL, pos, w),
			    __shfl_sync(CMB_FULL, cand, w));
		if (__ballot_sync(CMB_FULL, en || special) != CMB_FULL) return 0;   // a probe ran into the end margin
	}
}

// Everything after a found match that does not fit the straight-line emitter: long literal runs,
// length bytes beyond one.  Returns the new output offset.
__device__ __noinline__ uint32_t lz4_emit_general(uint8_t *dst, uint32_t op, const uint8_t *src, uint32_t anchor,
    uint32_t lit, uint32_t off, uint32_t mc, int lane) {
	if (lane == 0) dst[op] = (uint8_t)((min(lit, 15u) << 4) | min(mc, 15u));
	op++;
	if (lit >= 15u) op = lz4_emit_len(dst, op, lit - 15u, lane);
	if (lit <= 256u) {           // the usual case here is a run of 129..256 bytes: bytes, no alignment work
		for (uint32_t i = lane; i < lit; i += 32) st_out8(dst + op + i, ldg8(src + anchor + i));
	} else {
		warp_copy_ro(dst + op, src + anchor, lit, lane);
	}
	op += lit;
	if (lane == 0) { dst[op] = (uint8_t)off; dst[op + 1] = (uint8_t)(off >> 8); }
	op += 2;
	if (mc >= 15u) op = lz4_emit_len(dst, op, mc - 15u, lane);
	return op;
}

// Byte store of encoder output (global memory) as ONE predicated instruction.  Inside the encoder
// loop's conditional emit the compiler otherwise branches around each store and recomputes its
// address behind the branch.
__device__ __forceinline__ void st_out8_if(bool p, uint8_t *ptr, uint32_t v) {
	asm volatile("{\n\t.reg .pred q;\n\tsetp.ne.u32 q, %2, 0;\n\t@q st.global.u8 [%0], %1;\n\t}" ::"l"(
	                 __cvta_generic_to_global(ptr)), "r"(v), "r"((uint32_t)p)
	             : "memory");
}

// Writes one sequence — token, literal run, offset and match length (lz4.c:625-683) — at dst[op..),
// lz4_seq_bytes(lit, mc) bytes.  A run of at most LZ4_LIT_REG literals comes from a register (lw =
// src[from + 4 lane .. + 4), little-endian, loaded by the batch that found the match) and is written
// by predicated lane stores; longer runs and long lengths go to lz4_emit_general, which reads the
// literals from the page in global memory (an L2 round trip on the parse's path).
constexpr uint32_t LZ4_LIT_REG = 128;
__device__ __forceinline__ void lz4_emit_seq(uint8_t *dst, const uint8_t *src, uint32_t op, uint32_t from, uint32_t lit,
    uint32_t off, uint32_t mc, uint32_t lw, int lane) {
	if (lit <= LZ4_LIT_REG && mc < 15u + 255u) {
		uint8_t *o = dst + op;
		const uint32_t lext = lit >= 15u, mext = mc >= 15u;
		const uint32_t hl = 1u + lext;
		const uint32_t l4 = 4u * (uint32_t)lane;
#pragma unroll
		for (uint32_t k = 0; k < 4; k++) st_out8_if(l4 + k < lit, o + hl + l4 + k, lw >> (8u * k));
		const uint32_t tail = hl + lit;
		const uint32_t head4 = (min(lit, 15u) << 4) | min(mc, 15u) | (((lit - 15u) & 0xffu) << 8) | (off << 16);
		const uint32_t val = lane < 4 ? head4 >> (8u * (uint32_t)lane) : mc - 15u;
		const uint32_t at = lane < 2 ? (uint32_t)lane : tail + (uint32_t)lane - 2u;
		const uint32_t owners = 0x0du | (lext << 1) | (mext << 4);
		st_out8_if((owners >> lane) & 1u, o + at, val);
	} else {
		lz4_emit_general(dst, op, src, from, lit, off, mc, lane);
	}
}

// The encoder loop itself is lz4_encode_lean (lz4_encode_ring.cuh).

}  // namespace cmb
