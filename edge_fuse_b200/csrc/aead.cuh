// aead.cuh — ChaCha20-Poly1305 (RFC 8439 §2.8) on the GPU, one warp per message.
//
// Layout: lane j makes the 64-byte ChaCha20 blocks j, j + 32, ... of the text (block b uses counter
// 1 + b), xors them into the text with 8-byte loads and stores (a sealed record's text starts 24 bytes
// into the record, so 8 bytes is the widest alignment every message shares), and feeds the 64 bytes of
// ciphertext it made or read to its own Poly1305 accumulator as four 16-byte blocks.  So a lane
// authenticates exactly the bytes it wrote and no lane waits for another.  Each lane runs Horner over
// its blocks (r between the four blocks of one ChaCha20 block, r^125 to its next one, 128 blocks on),
// then multiplies its sum by r^(C - last block) and the warp adds the 32 sums with shuffles.  The AAD is
// summed the same way.  The tag is (H(AAD) r^C + H(CT) + lengths) r + s, with H(X) the Poly1305
// polynomial of X's padded blocks: the same value as the RFC's serial loop.
//
// Arithmetic mod 2^130 - 5 is exact, in five 26-bit limbs with 32 x 32 -> 64-bit products
// (poly1305-donna's representation), including the final carry and the h >= p reduction.
#pragma once
#include <stdint.h>

namespace cmb {

struct P130 { uint32_t v[5]; };

__device__ __forceinline__ uint32_t rotl32(uint32_t x, int n) { return __funnelshift_l(x, x, n); }

#define CMB_QR(a, b, c, d) \
	a += b; d ^= a; d = rotl32(d, 16); c += d; b ^= c; b = rotl32(b, 12); \
	a += b; d ^= a; d = rotl32(d, 8);  c += d; b ^= c; b = rotl32(b, 7);

// One ChaCha20 block (RFC 8439 §2.3): out = state after 20 rounds + input state.
__device__ __forceinline__ void chacha20_block(const uint32_t key[8], uint32_t counter, const uint32_t nonce[3], uint32_t out[16]) {
	uint32_t x[16] = {0x61707865u, 0x3320646eu, 0x79622d32u, 0x6b206574u, key[0], key[1], key[2], key[3],
	                  key[4], key[5], key[6], key[7], counter, nonce[0], nonce[1], nonce[2]};
#pragma unroll
	for (int i = 0; i < 16; i++) out[i] = x[i];
#pragma unroll 1
	for (int r = 0; r < 10; r++) {
		CMB_QR(out[0], out[4], out[8], out[12]) CMB_QR(out[1], out[5], out[9], out[13])
		CMB_QR(out[2], out[6], out[10], out[14]) CMB_QR(out[3], out[7], out[11], out[15])
		CMB_QR(out[0], out[5], out[10], out[15]) CMB_QR(out[1], out[6], out[11], out[12])
		CMB_QR(out[2], out[7], out[8], out[13]) CMB_QR(out[3], out[4], out[9], out[14])
	}
#pragma unroll
	for (int i = 0; i < 16; i++) out[i] += x[i];
}
#undef CMB_QR

// a * b mod 2^130 - 5, partially reduced (limbs < 2^26 except limb 1, < 2^26 + 2^12).  Inputs: limbs < 2^27.
__device__ __forceinline__ P130 p130_mul(const P130 &a, const P130 &b) {
	const uint64_t a0 = a.v[0], a1 = a.v[1], a2 = a.v[2], a3 = a.v[3], a4 = a.v[4];
	const uint64_t b0 = b.v[0], b1 = b.v[1], b2 = b.v[2], b3 = b.v[3], b4 = b.v[4];
	const uint64_t s1 = b1 * 5, s2 = b2 * 5, s3 = b3 * 5, s4 = b4 * 5;
	uint64_t d0 = a0 * b0 + a1 * s4 + a2 * s3 + a3 * s2 + a4 * s1;
	uint64_t d1 = a0 * b1 + a1 * b0 + a2 * s4 + a3 * s3 + a4 * s2;
	uint64_t d2 = a0 * b2 + a1 * b1 + a2 * b0 + a3 * s4 + a4 * s3;
	uint64_t d3 = a0 * b3 + a1 * b2 + a2 * b1 + a3 * b0 + a4 * s4;
	uint64_t d4 = a0 * b4 + a1 * b3 + a2 * b2 + a3 * b1 + a4 * b0;
	const uint64_t M = 0x3ffffff;
	d1 += d0 >> 26; d2 += d1 >> 26; d3 += d2 >> 26; d4 += d3 >> 26;
	uint64_t h0 = (d0 & M) + (d4 >> 26) * 5;
	P130 r;
	r.v[0] = (uint32_t)(h0 & M);
	r.v[1] = (uint32_t)((d1 & M) + (h0 >> 26));
	r.v[2] = (uint32_t)(d2 & M); r.v[3] = (uint32_t)(d3 & M); r.v[4] = (uint32_t)(d4 & M);
	return r;
}

// a + b with the carries propagated (limbs < 2^26 except limb 1).
__device__ __forceinline__ P130 p130_add(const P130 &a, const P130 &b) {
	uint32_t c, h[5];
#pragma unroll
	for (int i = 0; i < 5; i++) h[i] = a.v[i] + b.v[i];
	c = h[0] >> 26; h[0] &= 0x3ffffff; h[1] += c;
	c = h[1] >> 26; h[1] &= 0x3ffffff; h[2] += c;
	c = h[2] >> 26; h[2] &= 0x3ffffff; h[3] += c;
	c = h[3] >> 26; h[3] &= 0x3ffffff; h[4] += c;
	c = h[4] >> 26; h[4] &= 0x3ffffff; h[0] += c * 5;
	c = h[0] >> 26; h[0] &= 0x3ffffff; h[1] += c;
	P130 r;
#pragma unroll
	for (int i = 0; i < 5; i++) r.v[i] = h[i];
	return r;
}

// h + (16 bytes w0..w3, little-endian) + hibit * 2^128
__device__ __forceinline__ void p130_add_block(P130 &h, uint32_t w0, uint32_t w1, uint32_t w2, uint32_t w3, uint32_t hibit) {
	h.v[0] += w0 & 0x3ffffff;
	h.v[1] += ((w0 >> 26) | (w1 << 6)) & 0x3ffffff;
	h.v[2] += ((w1 >> 20) | (w2 << 12)) & 0x3ffffff;
	h.v[3] += ((w2 >> 14) | (w3 << 18)) & 0x3ffffff;
	h.v[4] += (w3 >> 8) | (hibit << 24);
}

__device__ __forceinline__ P130 p130_pow(P130 r, uint64_t e) {
	P130 acc = {{1, 0, 0, 0, 0}};
	while (e) {
		if (e & 1) acc = p130_mul(acc, r);
		e >>= 1;
		if (e) r = p130_mul(r, r);
	}
	return acc;
}

__device__ __forceinline__ P130 p130_warp_sum(P130 h) {
#pragma unroll
	for (int o = 16; o > 0; o >>= 1) {
		P130 x;
#pragma unroll
		for (int i = 0; i < 5; i++) x.v[i] = __shfl_xor_sync(0xffffffffu, h.v[i], o);
		h = p130_add(h, x);
	}
	return h;
}

// (h mod 2^130 - 5) + s mod 2^128, as four little-endian words: the tag.
__device__ __forceinline__ void p130_finish(P130 h, const uint32_t s[4], uint32_t tag[4]) {
	h = p130_add(h, P130{{0, 0, 0, 0, 0}});
	uint32_t h0 = h.v[0], h1 = h.v[1], h2 = h.v[2], h3 = h.v[3], h4 = h.v[4], c;
	c = h1 >> 26; h1 &= 0x3ffffff; h2 += c;
	c = h2 >> 26; h2 &= 0x3ffffff; h3 += c;
	c = h3 >> 26; h3 &= 0x3ffffff; h4 += c;
	c = h4 >> 26; h4 &= 0x3ffffff; h0 += c * 5;
	c = h0 >> 26; h0 &= 0x3ffffff; h1 += c;
	// g = h + 5 - 2^130: if it does not borrow, h >= p and g is the reduced value
	uint32_t g0 = h0 + 5; c = g0 >> 26; g0 &= 0x3ffffff;
	uint32_t g1 = h1 + c; c = g1 >> 26; g1 &= 0x3ffffff;
	uint32_t g2 = h2 + c; c = g2 >> 26; g2 &= 0x3ffffff;
	uint32_t g3 = h3 + c; c = g3 >> 26; g3 &= 0x3ffffff;
	uint32_t g4 = h4 + c - (1u << 26);
	const uint32_t take_g = (g4 >> 31) - 1;           // all ones when g4 did not borrow
	h0 = (h0 & ~take_g) | (g0 & take_g); h1 = (h1 & ~take_g) | (g1 & take_g);
	h2 = (h2 & ~take_g) | (g2 & take_g); h3 = (h3 & ~take_g) | (g3 & take_g);
	h4 = (h4 & ~take_g) | (g4 & take_g);
	const uint32_t w0 = h0 | (h1 << 26), w1 = (h1 >> 6) | (h2 << 20), w2 = (h2 >> 12) | (h3 << 14), w3 = (h3 >> 18) | (h4 << 8);
	uint64_t f = (uint64_t)w0 + s[0]; tag[0] = (uint32_t)f;
	f = (uint64_t)w1 + s[1] + (f >> 32); tag[1] = (uint32_t)f;
	f = (uint64_t)w2 + s[2] + (f >> 32); tag[2] = (uint32_t)f;
	f = (uint64_t)w3 + s[3] + (f >> 32); tag[3] = (uint32_t)f;
}

// The first min(avail, 8) bytes at p as a little-endian word, zeros above; and the store of as many.
__device__ __forceinline__ uint64_t load_tail(const uint8_t *p, uint64_t avail) {
	uint64_t v = 0;
	for (uint64_t k = 0; k < avail && k < 8; k++) v |= (uint64_t)p[k] << (8 * k);
	return v;
}
__device__ __forceinline__ void store_tail(uint8_t *p, uint64_t v, uint64_t avail) {
	for (uint64_t k = 0; k < avail && k < 8; k++) p[k] = (uint8_t)(v >> (8 * k));
}

// The per-lane Poly1305 sum of a run of 64-byte groups: blocks (in 16-byte units) 4g .. 4g + 3 of
// group g (those below nblk) are folded into h, r between blocks, rgap before the group's first block
// when h already holds earlier groups.  last: the index of the last block folded so far (or -1).
__device__ __forceinline__ void poly_group(P130 &h, long long &last, const uint64_t q[8], uint64_t g, uint64_t nblk,
    const P130 &r, const P130 &rgap) {
#pragma unroll
	for (int k = 0; k < 4; k++) {
		const uint64_t blk = 4 * g + k;
		if (blk >= nblk) break;
		if (last >= 0) h = p130_mul(h, k == 0 ? rgap : r);
		p130_add_block(h, (uint32_t)q[2 * k], (uint32_t)(q[2 * k] >> 32), (uint32_t)q[2 * k + 1],
		               (uint32_t)(q[2 * k + 1] >> 32), 1u);
		last = (long long)blk;
	}
}

// h * r^(nblk - last) on every lane that holds blocks, summed over the warp: the Poly1305 polynomial of a
// run of nblk padded blocks (each block times r^(nblk - index)).
__device__ __forceinline__ P130 poly_close(P130 h, long long last, uint64_t nblk, const P130 &r) {
	if (last >= 0) h = p130_mul(h, p130_pow(r, nblk - (uint64_t)last));
	else h = P130{{0, 0, 0, 0, 0}};
	return p130_warp_sum(h);
}

// Poly1305 of aad (any alignment, aad_len bytes) over the warp.
__device__ __forceinline__ P130 poly_aad(const uint8_t *aad, uint64_t aad_len, const P130 &r, const P130 &rgap, int lane) {
	const uint64_t nblk = (aad_len + 15) / 16, ngrp = (aad_len + 63) / 64;
	P130 h = {{0, 0, 0, 0, 0}};
	long long last = -1;
	for (uint64_t g = lane; g < ngrp; g += 32) {
		uint64_t q[8];
#pragma unroll
		for (int w = 0; w < 8; w++) {
			const uint64_t at = 64 * g + 8 * w;
			q[w] = at < aad_len ? load_tail(aad + at, aad_len - at) : 0;
		}
		poly_group(h, last, q, g, nblk, r, rgap);
	}
	return poly_close(h, last, nblk, r);
}

// The message a warp seals or opens.  The text is `len` bytes: word k (bytes 8k .. 8k + 7) is head[k] for
// k < head_words, else the 8 bytes at src + 8k (src + 8k is 8-aligned for every whole word).  The result
// goes to dst (8-aligned); the tag is compared with, or written to, tag.
struct AeadText {
	const uint8_t *src;
	uint8_t *dst;
	uint64_t len;
	uint64_t head[3];
	int head_words;
};

// Seals (OPEN = false: dst gets ciphertext, tag_io the tag) or opens (dst gets plaintext; returns whether
// tag_io holds the right tag) one message on a whole warp.  Every lane returns the same value.
template <bool OPEN>
__device__ bool aead_warp(const uint32_t key[8], const uint32_t nonce[3], const uint8_t *aad, uint64_t aad_len,
    const AeadText &t, uint8_t *tag_io, int lane) {
	uint32_t ks[16];
	chacha20_block(key, 0, nonce, ks);
	// r clamped (RFC 8439 §2.5), in 26-bit limbs
	const uint32_t r0 = ks[0] & 0x0fffffffu, r1 = ks[1] & 0x0ffffffcu, r2 = ks[2] & 0x0ffffffcu, r3 = ks[3] & 0x0ffffffcu;
	const P130 r = {{r0 & 0x3ffffff, ((r0 >> 26) | (r1 << 6)) & 0x3ffffff, ((r1 >> 20) | (r2 << 12)) & 0x3ffffff,
	                 ((r2 >> 14) | (r3 << 18)) & 0x3ffffff, r3 >> 8}};
	const uint32_t s[4] = {ks[4], ks[5], ks[6], ks[7]};
	const P130 rgap = p130_pow(r, 125);
	const P130 ha = poly_aad(aad, aad_len, r, rgap, lane);

	const uint64_t nblk = (t.len + 15) / 16, ngrp = (t.len + 63) / 64;
	P130 h = {{0, 0, 0, 0, 0}};
	long long last = -1;
	for (uint64_t g = lane; g < ngrp; g += 32) {
		chacha20_block(key, (uint32_t)(1 + g), nonce, ks);
		uint64_t in[8], out[8];
#pragma unroll
		for (int w = 0; w < 8; w++) {
			const uint64_t k = 8 * g + w, at = 8 * k;
			if (at >= t.len) { in[w] = 0; continue; }
			if ((long long)k < t.head_words) in[w] = t.head[k];
			else if (at + 8 <= t.len) in[w] = *reinterpret_cast<const uint64_t *>(t.src + at);
			else in[w] = load_tail(t.src + at, t.len - at);
		}
#pragma unroll
		for (int w = 0; w < 8; w++) {
			const uint64_t at = 64 * g + 8 * w;
			const uint64_t kw = (uint64_t)ks[2 * w] | ((uint64_t)ks[2 * w + 1] << 32);
			// ciphertext bytes past the end are the zero padding Poly1305 reads
			if (at >= t.len) { out[w] = 0; continue; }
			if (at + 8 <= t.len) {
				out[w] = in[w] ^ kw;
				*reinterpret_cast<uint64_t *>(t.dst + at) = out[w];
			} else {
				out[w] = (in[w] ^ kw) & ((1ull << (8 * (t.len - at))) - 1);
				store_tail(t.dst + at, out[w], t.len - at);
			}
		}
		if (OPEN) {
#pragma unroll
			for (int w = 0; w < 8; w++) if (64 * g + 8 * w >= t.len) in[w] = 0;
		}
		poly_group(h, last, OPEN ? in : out, g, nblk, r, rgap);
	}
	const P130 hc = poly_close(h, last, nblk, r);
	P130 acc = p130_add(p130_mul(ha, p130_pow(r, nblk)), hc);
	p130_add_block(acc, (uint32_t)aad_len, (uint32_t)(aad_len >> 32), (uint32_t)t.len, (uint32_t)(t.len >> 32), 1u);
	acc = p130_mul(acc, r);
	uint32_t tag[4];
	p130_finish(acc, s, tag);
	if (!OPEN) {
		if (lane < 16) tag_io[lane] = (uint8_t)(tag[lane >> 2] >> (8 * (lane & 3)));
		return true;
	}
	uint32_t diff = 0;
#pragma unroll
	for (int k = 0; k < 16; k++) diff |= ((tag[k >> 2] >> (8 * (k & 3))) & 0xffu) ^ tag_io[k];
	return diff == 0;
}

}  // namespace cmb
