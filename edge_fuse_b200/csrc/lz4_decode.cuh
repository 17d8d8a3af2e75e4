// lz4_decode.cuh — LZ4 block decoder with LZ4_decompress_fast semantics, one warp per chunk.
//
// Replaces filemap_get's LZ4_decompress_fast(block, page, bsize) (cachemap/filemap.c:243-248 ->
// cachemap/lz4.c:1360-1363,1169-1344): decodes exactly n bytes and returns the number of
// compressed bytes consumed, which filemap_get compares with the stored compressed_length.
// Unlike the reference's trusting variant this one is bounds-checked and returns <0 on a
// malformed block (SURVEY.md App. A "Decoder freedom": any correct decoder yields the same page).
//
// The token chain is serial; literal and match copies are warp-parallel.  Match bytes are read
// back from the page being written (global memory, coherent loads, __syncwarp between
// sequences); an overlapping match (offset < length) is expanded as out[i] = out[base + i % offset]
// so that every lane only reads bytes finished before this sequence began.
#pragma once
#include "common.cuh"

namespace cmb {

// Reads an LZ4 length extension at blk[ip..cap): sum of bytes up to and including the first
// non-0xFF one, 32 bytes per step.  Returns false when the block ends first.
__device__ __forceinline__ bool lz4_read_ext(const uint8_t *blk, uint32_t cap, uint32_t &ip,
    uint32_t &len, int lane) {
	for (;;) {
		bool in = ip + lane < cap;
		uint32_t b = in ? ldg8(blk + ip + lane) : 0u;
		uint32_t stop = __ballot_sync(CMB_FULL, !in || b != 255u);
		if (stop) {
			int f = __ffs(stop) - 1;
			if (ip + f >= cap) return false;
			len += 255u * f + __shfl_sync(CMB_FULL, b, f);
			ip += f + 1;
			return true;
		}
		len += 255u * 32u;
		ip += 32;
	}
}

// Returns bytes consumed (>0) or a negative error; uniform across the warp.
// The kernel is issue-bound (64 warps per SM), so the loop is
// written for few instructions per sequence: the common sequence — up to 32 literals with at most one
// length byte, a match of up to 32 bytes that does not overlap itself — is one predicated byte load
// and store per lane for the literals and one for the match; the token of the NEXT sequence and the
// byte after it are requested together with the offset bytes (their position is known as soon as
// the literal length is), so a sequence costs one block round trip, not two.  Reads past `cap` are
// harmless prefetches (blocks lie in padded buffers) and every use is bounds-checked.
__device__ int lz4_decode_warp(const uint8_t *__restrict__ blk, uint32_t cap, uint8_t *out,
    uint32_t n, int lane) {
	uint32_t ip = 0, op = 0;
	if (n == 0 || cap == 0) return -1;
	uint32_t tok = ldg8(blk), b0 = ldg8(blk + 1);
	for (;;) {
		if (ip >= cap) return -1;
		uint32_t len = tok >> 4, mlen = tok & 15u;
		uint32_t lit_src = ip + 1u;
		if (len == 15u) {
			if (b0 != 255u && ip + 1u < cap) { len += b0; lit_src = ip + 2u; }
			else { uint32_t q = ip + 1u; if (!lz4_read_ext(blk, cap, q, len, lane)) return -1; lit_src = q; }
		}
		if (len > n - op || len > cap - lit_src) return -1;
		const bool last = op + len + 8u > n;                 // lz4.c:1242-1256: last literals
		if (last && op + len != n) return -1;
		if (len <= 32u) { if ((uint32_t)lane < len) out[op + lane] = (uint8_t)ldg8(blk + lit_src + lane); }
		else warp_copy_ro(out + op, blk + lit_src, len, lane);
		if (last) return (int)(lit_src + len);              // lz4.c:1339
		ip = lit_src + len; op += len;
		if (ip + 2u > cap) return -1;
		const uint32_t o0 = ldg8(blk + ip), o1 = ldg8(blk + ip + 1u), m0 = ldg8(blk + ip + 2u);
		uint32_t nip = ip + 2u + (mlen == 15u ? 1u : 0u);
		const uint32_t t1 = ldg8(blk + nip), t2 = ldg8(blk + nip + 1u);
		const uint32_t off = o0 | (o1 << 8);
		if (mlen == 15u) {
			if (m0 != 255u && ip + 2u < cap) { mlen += m0; tok = t1; b0 = t2; }
			else {
				uint32_t q = ip + 2u;
				if (!lz4_read_ext(blk, cap, q, mlen, lane)) return -1;
				nip = q; tok = ldg8(blk + nip); b0 = ldg8(blk + nip + 1u);
			}
		} else { tok = t1; b0 = t2; }
		ip = nip;
		mlen += 4u;
		if (off == 0u || off > op || op + mlen + 5u > n) return -1;   // lz4.c:1319
		__syncwarp();                                // literals above are now visible to all lanes
		const uint8_t *from = out + op - off;
		if (off >= mlen) {
			if (mlen <= 32u) { if ((uint32_t)lane < mlen) out[op + lane] = from[lane]; }
			else warp_copy_rw(out + op, from, mlen, lane);
		} else {
			for (uint32_t i = lane; i < mlen; i += 32) out[op + i] = from[i % off];
		}
		op += mlen;
		__syncwarp();
	}
}

}  // namespace cmb
