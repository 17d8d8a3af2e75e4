// lz4_decode_cta.cuh — one CTA decodes one LZ4 block that sits in shared memory (k_get_small; for
// 128 KiB pages the page sits in a second CTA of a cluster, k_get_small_pair, see PAIR below).
//
// Same result as LZ4_decompress_fast (cachemap/lz4.c:1169-1344,1360-1363): exactly n bytes decoded,
// `consumed` = bytes of the block read (lz4.c:1339), which filemap_get compares with the stored
// compressed_length (filemap.c:243-248); a malformed block is an error, never an out-of-bounds access.
//
// A latency problem, not a throughput one: a single page, a caller waiting.  What is serial in an
// LZ4 block is (a) the token chain — where sequence k+1 starts is known only after sequence k's
// lengths — and (b) the matches, which read output that earlier sequences wrote.  The decoder
// therefore runs in phases, CTA barriers between them and no flags to poll:
//
//   1. PARSE    up to 16 warps walk 16 sections of the token chain at once.  Where a section starts
//               cannot be found without walking — so the ENCODER leaves 15 checkpoints per record
//               (block offset + output position of the first sequence at or after k/16 of the page;
//               a side table indexed by slot, kernels.cu:ckpt_store; rebuilt from the block when a
//               snapshot is loaded, kernels.cu:restore_ckpt_walk; kept by compaction and table
//               rebuilds) and a record without usable checkpoints (a raw page, another GPU's, a
//               loaded block whose chain does not fit) is walked by one warp.  Each sequence becomes a 16-byte descriptor in a scratch
//               region in global memory (L2): {literal source, output position, literal length,
//               offset | (match length - 4) << 16}; offset 0 marks the last sequence.
//               Every section must end exactly where the next one starts, the last at
//               (consumed == block length, output == n): together the sections then ARE the serial
//               parse, and anything else falls back to one warp walking the whole block.
//   2. LITERALS all warps, batches of 32 sequences dealt round-robin; literal runs depend on nothing.
//               A lane copies the run of one sequence word by word (runs are short: ~20 bytes on
//               text-like pages), long runs are copied by the warp.  The warp that holds a batch
//               also works out the ORDER OF ITS MATCHES here, where 16 warps share the batches:
//               wave(j) = 1 + the highest wave of an earlier match of the batch whose destination
//               match j's source touches (1 if none); matches of one wave are independent.  The
//               number goes into the descriptor.
//   3. MATCHES  one warp walks all batches, 32 sequences at a time, and only executes: wave by
//               wave, a lane per match (2-3 waves per batch on text, 8 bytes per lane and step);
//               matches longer than 16 bytes are copied by the whole warp when their wave is up.
//               Everything this one warp need not do itself counts: with the dependency analysis
//               inside this phase it took 130 k cycles on a text page, without 78 k.
#pragma once
#include "common.cuh"
#include "lz4_decode.cuh"

namespace cmb {

constexpr uint32_t DC_CHAINS = 16;                 // parse sections = warps of the CTA
constexpr uint32_t DC_THREADS = DC_CHAINS * 32;
constexpr uint32_t DC_LANE_LIT = 64;               // literal runs up to this are copied by one lane
constexpr uint32_t DC_LANE_MATCH = 16;             // matches up to this are copied by one lane

struct DecodeCta {                                 // shared memory
	uint32_t ip0[DC_CHAINS], op0[DC_CHAINS];   // section start: block offset of its first token, output position; ip0 = ~0: empty
	uint32_t op_end[DC_CHAINS];                // the section takes the sequences that start below this output position
	uint32_t cnt[DC_CHAINS];                   // sequences it found
	uint32_t ip1[DC_CHAINS], op1[DC_CHAINS];   // where it stopped
	int32_t err;                               // nonzero: malformed block, or checkpoints that do not fit it
};

// descriptors per section for a page of n bytes: a sequence that is not the last one produces at
// least 4 bytes (its match), so at most S/4 of them start inside S bytes, + the last sequence
__host__ __device__ inline uint32_t dc_stride(uint32_t n) { return n / DC_CHAINS / 4u + 2u; }
__host__ __device__ inline uint32_t dc_region(uint32_t n) { return DC_CHAINS * dc_stride(n); }   // entries of 16 bytes

__device__ __forceinline__ uint32_t dcs_ld8(uint32_t a) { uint32_t v; asm volatile("ld.shared.u8 %0, [%1];" : "=r"(v) : "r"(a)); return v; }
__device__ __forceinline__ uint32_t dcs_ld32(uint32_t a) { uint32_t v; asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(a)); return v; }
__device__ __forceinline__ void dcs_st32(uint32_t a, uint32_t v) { asm volatile("st.shared.u32 [%0], %1;" ::"r"(a), "r"(v)); }
__device__ __forceinline__ void dcs_st8(uint32_t a, uint32_t v) { asm volatile("st.shared.u8 [%0], %1;" ::"r"(a), "r"(v)); }

// PAIR = the two-CTA decoder of 128 KiB pages (kernels.cu:k_get_small_pair): the record and the page
// do not fit one CTA's shared memory, so the page lives in the partner CTA of a cluster of two and
// the literal phase stores into it over DSMEM.  Its descriptors need 17 bits for match length - 4 (a
// zero page is ONE match of ~131 060 bytes): the low 16 stay in the top half of the last word, bit 16
// goes to bit 31 of the literal length (at most 131 072, so bits 18-31 are free).  Literal source,
// output position and offset (< 65 536, the encoder's MAX_DISTANCE) keep their fields.
template <bool PAIR> __device__ __forceinline__ uint32_t dc_lit_len(uint4 d) { return PAIR ? d.z & 0x7fffffffu : d.z; }
template <bool PAIR> __device__ __forceinline__ uint32_t dc_match_len(uint4 d) {
	return PAIR ? ((d.w >> 16) | (d.z >> 31) << 16) + 4u : (d.w >> 16) + 4u;
}
template <bool PAIR> __device__ __forceinline__ void dc_put8(uint32_t a, uint32_t v) {
	if (PAIR) asm volatile("st.shared::cluster.u8 [%0], %1;" ::"r"(a), "r"(v));
	else dcs_st8(a, v);
}
template <bool PAIR> __device__ __forceinline__ void dc_put32(uint32_t a, uint32_t v) {
	if (PAIR) asm volatile("st.shared::cluster.u32 [%0], %1;" ::"r"(a), "r"(v));
	else dcs_st32(a, v);
}

// LZ4 255-run length extension at shared address blk + ip; cap = block length
__device__ __forceinline__ bool dcs_ext(uint32_t blk, uint32_t cap, uint32_t &ip, uint32_t &len, int lane) {
	for (;;) {
		const bool in = ip + lane < cap;
		const uint32_t b = in ? dcs_ld8(blk + ip + lane) : 0u;
		const uint32_t stop = __ballot_sync(CMB_FULL, !in || b != 255u);
		if (stop) {
			const int f = __ffs(stop) - 1;
			if (ip + f >= cap) return false;
			len += 255u * f + __shfl_sync(CMB_FULL, b, f);
			ip += f + 1;
			return true;
		}
		len += 255u * 32u;
		ip += 32;
	}
}

// Phase 1, one warp per section.  blk = shared address of the block (padded: reads up to ~300 bytes
// past `cap` stay inside the CTA's shared memory and every use is bounds-checked).  The walk is one
// shared-memory round trip per sequence: the token and the byte after it fix where the offset, the
// match-length byte and the NEXT token lie, so those five bytes are requested together.
template <bool PAIR>
__device__ void dc_parse_chain(DecodeCta *dc, uint32_t c, uint32_t blk, uint32_t cap, uint32_t n, uint4 *desc,
    uint32_t max_desc, int lane) {
	uint32_t ip = dc->ip0[c], op = dc->op0[c];
	const uint32_t op_end = dc->op_end[c];
	uint32_t cnt = 0;
	uint4 *dnext = desc;
	int32_t err = 0;
	if (ip >= cap) err = -1;
	uint32_t tok = err ? 0u : dcs_ld8(blk + ip), b0 = err ? 0u : dcs_ld8(blk + ip + 1u);
	while (!err && op < op_end) {
		{
			// the common sequence, straight line: at most one extension byte per length, everything inside
			// the block and the page.  Anything else is ONE rarely taken branch to the general code.
			const uint32_t l4 = tok >> 4, m4 = tok & 15u;
			const uint32_t lx = l4 == 15u ? 1u : 0u, mx = m4 == 15u ? 1u : 0u;
			const uint32_t flen = l4 + (lx ? b0 : 0u);
			const uint32_t fsrc = ip + 1u + lx;
			const uint32_t ip2 = fsrc + flen, op2 = op + flen;
			// offset (2 bytes), match-length byte, and the next token with its follower are the five bytes
			// at ip2 (the token follows the offset directly when there is no match-length byte): two
			// aligned words cover them, so everything the next iteration needs arrives in ONE round trip
			const uint32_t a = blk + ip2, s8 = (a & 3u) * 8u;
			const uint32_t lo = dcs_ld32(a & ~3u), hi = dcs_ld32((a & ~3u) + 4u);
			const uint32_t w = __funnelshift_r(lo, hi, s8);          // bytes ip2 .. ip2 + 3
			const uint32_t b4 = (hi >> s8) & 0xffu;                 // byte ip2 + 4
			const uint32_t m0 = (w >> 16) & 0xffu, b3 = w >> 24;
			const uint32_t nip = ip2 + 2u + mx;
			const uint32_t t1 = mx ? b3 : m0, t2 = mx ? b4 : b3;
			const uint32_t off = w & 0xffffu;
			const uint32_t fm = m4 + (mx ? m0 : 0u);
			const uint32_t op3 = op2 + fm + 4u;
			// nip <= cap covers ip + 2 < cap; op3 + 5 <= n covers "not the last literals" (op2 + 8 <= n);
			// flen / fm == 270 <=> an extension byte of 255; off - 1 >= op2 <=> off == 0 or off > op2
			const bool rare = nip > cap || flen == 270u || fm == 270u || off - 1u >= op2 || op3 + 5u > n || cnt >= max_desc;
			if (!rare) {
				if (lane == 0) *dnext = make_uint4(fsrc, op, flen, off | (fm << 16));
				dnext++;
				cnt++;
				ip = nip; op = op3; tok = t1; b0 = t2;
				continue;
			}
		}
		if (ip >= cap || cnt >= max_desc) { err = -1; break; }
		uint32_t len = tok >> 4, mlen = tok & 15u;
		uint32_t lit_src = ip + 1u;
		if (len == 15u) {
			if (b0 != 255u && ip + 1u < cap) { len += b0; lit_src = ip + 2u; }
			else { uint32_t q = ip + 1u; if (!dcs_ext(blk, cap, q, len, lane)) { err = -1; break; } lit_src = q; }
		}
		const bool last = op + len + 8u > n;                 // lz4.c:1242-1256: last literals
		if (len > n - op || len > cap - lit_src || (last && op + len != n)) { err = -1; break; }
		const uint32_t out_pos = op;
		uint32_t off = 0;
		ip = lit_src + len; op += len;
		if (!last) {
			if (ip + 2u > cap) { err = -1; break; }
			const uint32_t o0 = dcs_ld8(blk + ip), o1 = dcs_ld8(blk + ip + 1u), m0 = dcs_ld8(blk + ip + 2u);
			uint32_t nip = ip + 2u + (mlen == 15u ? 1u : 0u);
			const uint32_t t1 = dcs_ld8(blk + nip), t2 = dcs_ld8(blk + nip + 1u);
			off = o0 | (o1 << 8);
			if (mlen == 15u) {
				if (m0 != 255u && ip + 2u < cap) { mlen += m0; tok = t1; b0 = t2; }
				else {
					uint32_t q = ip + 2u;
					if (!dcs_ext(blk, cap, q, mlen, lane)) { err = -1; break; }
					nip = q; tok = dcs_ld8(blk + nip); b0 = dcs_ld8(blk + nip + 1u);
				}
			} else { tok = t1; b0 = t2; }
			ip = nip;
			if (off == 0u || off > op || op + mlen + 9u > n) { err = -1; break; }   // lz4.c:1319: op + (mlen + 4) + 5 > n
			op += mlen + 4u;
		} else {
			mlen = 0;
		}
		if (lane == 0) *dnext = make_uint4(lit_src, out_pos, PAIR ? len | (mlen >> 16) << 31 : len, off | (mlen << 16));
		dnext++;
		cnt++;
		if (last) break;                                     // op == n, ip == bytes consumed (lz4.c:1339)
	}
	if (lane == 0) {
		dc->cnt[c] = cnt; dc->ip1[c] = ip; dc->op1[c] = op;
		if (err) dc->err = err;
	}
}

// Phase 2, all warps: batches of 32 descriptors, dealt round-robin.  PAIR: `out` / `out_g` is the
// page in the partner CTA of the cluster (a shared::cluster address / a generic address).
template <bool PAIR>
__device__ void dc_literals(const DecodeCta *dc, uint4 *desc, uint32_t stride, uint32_t blk, uint32_t out,
    const uint8_t *blk_g, uint8_t *out_g, uint32_t warp, int lane) {
	uint32_t turn = 0;
	for (uint32_t c = 0; c < DC_CHAINS; c++) {
		const uint32_t cnt = dc->cnt[c];
		for (uint32_t b = 0; b < cnt; b += 32u, turn++) {
			if (turn % DC_CHAINS != warp) continue;
			const bool valid = b + lane < cnt;
			uint4 d = make_uint4(0, 0, 0, 0);
			if (valid) d = __ldcg(desc + (size_t)c * stride + b + lane);
			const uint32_t len = dc_lit_len<PAIR>(d);
			const uint32_t mine = len <= DC_LANE_LIT ? len : 0u;
			const uint32_t most = __reduce_max_sync(CMB_FULL, mine);
			const uint32_t src = blk + d.x, dst = out + d.y;
			{
				// a lane's run word by word: up to 3 bytes until the destination is 4-byte aligned, then
				// words put together from the two aligned source words around them, then up to 3 bytes
				// (byte copies of 32 scattered runs are mostly shared-memory wavefronts; this is a third of them)
				const uint32_t head = min(mine, (4u - (dst & 3u)) & 3u);
				const uint32_t words = (mine - head) / 4u, tail = head + 4u * words;
#pragma unroll
				for (uint32_t j = 0; j < 3u; j++) if (j < head) dc_put8<PAIR>(dst + j, dcs_ld8(src + j));
				const uint32_t mostw = __reduce_max_sync(CMB_FULL, words);
				const uint32_t sa = src + head, s8 = (sa & 3u) * 8u;
				for (uint32_t t = 0; t < mostw; t++) {
					if (t < words) {
						const uint32_t a = (sa & ~3u) + 4u * t;
						dc_put32<PAIR>(dst + head + 4u * t, __funnelshift_r(dcs_ld32(a), dcs_ld32(a + 4u), s8));
					}
				}
#pragma unroll
				for (uint32_t j = 0; j < 3u; j++) if (tail + j < mine) dc_put8<PAIR>(dst + tail + j, dcs_ld8(src + tail + j));
			}
			(void)most;
			uint32_t wide = __ballot_sync(CMB_FULL, len > DC_LANE_LIT);
			while (wide) {
				const int j = __ffs(wide) - 1;
				wide &= wide - 1u;
				const uint32_t x = __shfl_sync(CMB_FULL, d.x, j), y = __shfl_sync(CMB_FULL, d.y, j), z = __shfl_sync(CMB_FULL, len, j);
				warp_copy_rw(out_g + y, blk_g + x, z, lane);     // 16 bytes per lane per step
			}
			// ---- the order of this batch's MATCHES, worked out here where 16 warps share the batches:
			// the match phase is one warp walking all batches, so whatever it need not do itself counts.
			// wave(j) = 1 + the highest wave of an earlier match of the batch whose destination my source
			// touches (1 if none): matches of equal wave are independent of each other.  Lane i's wave is
			// final when the loop reaches i.  The number replaces the literal source in the descriptor.
			const uint32_t off = d.w & 0xffffu;
			const bool has = valid && off != 0u;
			const uint32_t mlen = has ? dc_match_len<PAIR>(d) : 0u;
			const uint32_t to = has ? d.y + len : 0xffffffffu, from = to - off, fe = from + mlen;
			uint32_t wave = has ? 1u : 0u;
			const uint32_t to0 = __shfl_sync(CMB_FULL, to, 0);             // (every lane takes part in the shuffle)
			if (__any_sync(CMB_FULL, has && fe > to0)) {                  // somebody reads inside the batch
				if (PAIR) {
					// destinations and lengths reach 17 bits: they travel in two words
#pragma unroll
					for (int i = 0; i < 31; i++) {
						const uint32_t ti = __shfl_sync(CMB_FULL, to, i), li = __shfl_sync(CMB_FULL, mlen, i);
						const uint32_t wi = __shfl_sync(CMB_FULL, wave, i);
						if (lane > i && has && ti < fe && ti + li > from) wave = max(wave, wi + 1u);
					}
				} else {
					// destination and length travel in one word (both < 65 536); only the wave is a chain
					const uint32_t key = has ? to | (mlen << 16) : 0xffffu;
#pragma unroll
					for (int i = 0; i < 31; i++) {
						const uint32_t ki = __shfl_sync(CMB_FULL, key, i), wi = __shfl_sync(CMB_FULL, wave, i);
						const uint32_t ti = ki & 0xffffu, li = ki >> 16;
						if (lane > i && has && ti < fe && ti + li > from) wave = max(wave, wi + 1u);
					}
				}
			}
			if (valid) desc[(size_t)c * stride + b + lane].x = wave;
		}
	}
}

__device__ __forceinline__ uint4 dcs_ld128(uint32_t a) {
	uint4 v;
	asm volatile("ld.shared.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(a));
	return v;
}
__device__ __forceinline__ void dcs_st128(uint32_t a, uint4 v) {
	asm volatile("st.shared.v4.u32 [%0], {%1, %2, %3, %4};" ::"r"(a), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w));
}

// Bytes [k0, k1) of a match that repeats the `off` bytes before it (off < 32): byte k = from[k mod off].
// Lanes only read bytes that were complete before the sequence began.
__device__ __forceinline__ void dc_periodic_bytes(uint32_t to, uint32_t from, uint32_t off, uint32_t k0, uint32_t k1, int lane) {
	uint32_t r = (k0 + (uint32_t)lane) % off;
	const uint32_t step = 32u % off;
	for (uint32_t k = k0 + lane; k < k1; k += 32u) {
		dcs_st8(to + k, dcs_ld8(from + r));
		r += step;
		if (r >= off) r -= off;
	}
}

// A match longer than a lane should copy: all 32 lanes.  to / from = shared addresses.
__device__ __forceinline__ void dc_match_wide(uint32_t to, uint32_t from, uint32_t off, uint32_t len, int lane) {
	if (off >= 136u && len >= 64u) {
		// 128 bytes per step: a 4-byte word per lane, destination aligned (up to 3 bytes go first), source
		// word put together from the two aligned words around it; a step reads at most 132 bytes from its
		// source position, all of them below what the step writes
		const uint32_t head = (4u - (to & 3u)) & 3u;
		if ((uint32_t)lane < head) dcs_st8(to + lane, dcs_ld8(from + lane));
		uint32_t k = head;
		for (; k + 128u <= len; k += 128u) {
			const uint32_t a = from + k + 4u * lane, s8 = (a & 3u) * 8u;
			const uint32_t lo = dcs_ld32(a & ~3u), hi = dcs_ld32((a & ~3u) + 4u);
			dcs_st32(to + k + 4u * lane, __funnelshift_r(lo, hi, s8));
			__syncwarp();
		}
		for (; k < len; k += 32u) {
			if (k + lane < len) dcs_st8(to + k + lane, dcs_ld8(from + k + lane));
			__syncwarp();
		}
	} else if (off >= 32u) {
		// a step of 32 bytes only reads bytes that earlier steps (or earlier sequences) wrote
		for (uint32_t k0 = 0; k0 < len; k0 += 32u) {
			if (k0 + lane < len) dcs_st8(to + k0 + lane, dcs_ld8(from + k0 + lane));
			__syncwarp();
		}
	} else if (len < 4096u) {
		dc_periodic_bytes(to, from, off, 0u, len, lane);
	} else {
		// A long run of a short pattern (a zero page is ONE such match): the first `head + period` bytes
		// byte by byte, where period = a multiple of both off and 16 that is >= 512 and head aligns the
		// rest to 16 bytes; from there every 16-byte word equals the one `period` bytes before it, and a
		// step of 32 lanes x 16 bytes only reads what earlier steps wrote.
		const uint32_t period = 16u * off * ((512u + 16u * off - 1u) / (16u * off));
		const uint32_t first = ((16u - (to & 15u)) & 15u) + period;
		dc_periodic_bytes(to, from, off, 0u, first, lane);
		__syncwarp();
		uint32_t k = first;
		for (; k + 512u <= len; k += 512u) {
			dcs_st128(to + k + 16u * lane, dcs_ld128(to + k + 16u * lane - period));
			__syncwarp();
		}
		dc_periodic_bytes(to, from, off, k, len, lane);
	}
	__syncwarp();
}

// Phase 3, one warp.  out = shared address of the page (in this CTA also for PAIR).  Every descriptor carries the wave of its
// match within its batch of 32 (dc_literals): the matches of one wave are copied together, a lane
// each; long ones by the whole warp, one after the other.
template <bool PAIR>
__device__ void dc_matches(const DecodeCta *dc, const uint4 *desc, uint32_t stride, uint32_t out, int lane) {
	for (uint32_t c = 0; c < DC_CHAINS; c++) {
		const uint32_t cnt = dc->cnt[c];
		const uint4 *dq = desc + (size_t)c * stride;
		uint4 nxt = make_uint4(0, 0, 0, 0);
		if ((uint32_t)lane < cnt) nxt = __ldcg(dq + lane);
		for (uint32_t b = 0; b < cnt; b += 32u) {
			const uint4 d = nxt;
			if (b + 32u + lane < cnt) nxt = __ldcg(dq + b + 32u + lane);      // next batch while this one is copied
			const uint32_t off = d.w & 0xffffu;
			const bool valid = b + lane < cnt && off != 0u;
			const uint32_t len = valid ? dc_match_len<PAIR>(d) : 0u;
			const uint32_t to = d.y + dc_lit_len<PAIR>(d), from = to - off;
			const uint32_t wave = valid ? d.x : 0u;
			const bool wide = len > DC_LANE_MATCH;
			const uint32_t waves = __reduce_max_sync(CMB_FULL, wave);
			const uint32_t src = out + from, dst = out + to;
			for (uint32_t w = 1; w <= waves; w++) {
				const bool run = wave == w && !wide;
				const uint32_t mine = run ? len : 0u;
				const uint32_t most = __reduce_max_sync(CMB_FULL, mine);
				if (!__any_sync(CMB_FULL, run && off < len)) {
					// nothing in this wave overlaps itself (the usual case; matches are 4-5 bytes on text):
					// eight loads, then eight stores per step
					for (uint32_t k = 0; k < most; k += 8u) {
						uint32_t v[8];
#pragma unroll
						for (uint32_t j = 0; j < 8u; j++) { v[j] = 0; if (k + j < mine) v[j] = dcs_ld8(src + k + j); }
#pragma unroll
						for (uint32_t j = 0; j < 8u; j++) if (k + j < mine) dcs_st8(dst + k + j, v[j]);
					}
				} else {
					// Byte k of a match is byte k mod off of the `off` bytes before it (a match that overlaps
					// itself repeats them), all of which exist before the match starts: four loads, then four
					// stores, no load waits for a store of its own match.
					uint32_t r = 0;
					for (uint32_t k = 0; k < most; k += 4u) {
						const uint32_t r0 = r, r1 = r0 + 1u == off ? 0u : r0 + 1u, r2 = r1 + 1u == off ? 0u : r1 + 1u,
						    r3 = r2 + 1u == off ? 0u : r2 + 1u;
						r = r3 + 1u == off ? 0u : r3 + 1u;
						uint32_t v0 = 0, v1 = 0, v2 = 0, v3 = 0;
						if (k < mine) v0 = dcs_ld8(src + r0);
						if (k + 1u < mine) v1 = dcs_ld8(src + r1);
						if (k + 2u < mine) v2 = dcs_ld8(src + r2);
						if (k + 3u < mine) v3 = dcs_ld8(src + r3);
						if (k < mine) dcs_st8(dst + k, v0);
						if (k + 1u < mine) dcs_st8(dst + k + 1u, v1);
						if (k + 2u < mine) dcs_st8(dst + k + 2u, v2);
						if (k + 3u < mine) dcs_st8(dst + k + 3u, v3);
					}
				}
				uint32_t wides = __ballot_sync(CMB_FULL, wave == w && wide);
				while (wides) {
					const int j = __ffs(wides) - 1;
					wides &= wides - 1u;
					dc_match_wide(out + __shfl_sync(CMB_FULL, to, j), out + __shfl_sync(CMB_FULL, from, j),
					    __shfl_sync(CMB_FULL, off, j), __shfl_sync(CMB_FULL, len, j), lane);
				}
				__syncwarp();
			}
		}
	}
}

}  // namespace cmb
