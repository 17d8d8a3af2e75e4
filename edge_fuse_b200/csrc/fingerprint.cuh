// fingerprint.cuh — EF128 content fingerprint, warp-level device routine (spec: DESIGN.md §5).
//
// NEW definition: the reference has no content hash (its uint128 is an address, SURVEY.md §0 R1).
// One warp fingerprints one chunk: each lane streams 16-byte vectors (ld.global.nc.v4, 512
// contiguous bytes per warp instruction, fully coalesced), keeps two 64-bit accumulators fed by
// one 32x32->64 multiply per 8 input bytes, and the 32 lane digests are folded with a shuffle
// butterfly.  HBM-bound: 65 536 B read + 16 B written per chunk.
#pragma once
#include "common.cuh"

namespace cmb {

__host__ __device__ __forceinline__ uint64_t ef_secret(unsigned i) {
	uint64_t z = 0x4544474546555345ULL + (uint64_t)(i + 1) * 0x9E3779B97F4A7C15ULL;
	z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ULL;
	z = (z ^ (z >> 27)) * 0x94D049BB133111EBULL;
	return z ^ (z >> 31);
}

__device__ __forceinline__ uint64_t ef_fold(uint64_t x, uint64_t y) {
	return (x * y) ^ __umul64hi(x, y);
}
__device__ __forceinline__ uint64_t ef_av(uint64_t h) {
	h ^= h >> 37; h *= 0x165667919E3779F9ULL; h ^= h >> 32; return h;
}

struct EfLane { uint64_t a, b, s0, s1, s2, s3; };

// 16-byte page load of the fused fingerprint.  Every page byte is absorbed exactly once, so in the
// encoder the stripes are pure streaming traffic: they stay out of the L1, which the parse needs for
// its match-candidate reads (ld.global.nc.L1::no_allocate).
__device__ __forceinline__ uint4 ef_ld16(const uint4 *p) {
	uint4 v;
	asm("ld.global.nc.L1::no_allocate.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p));
	return v;
}

__device__ __forceinline__ void ef_init(EfLane &L, int lane) {
	L.s0 = ef_secret(4 * lane); L.s1 = ef_secret(4 * lane + 1);
	L.s2 = ef_secret(4 * lane + 2); L.s3 = ef_secret(4 * lane + 3);
	L.a = L.s2; L.b = L.s3;
}
__device__ __forceinline__ void ef_absorb(EfLane &L, uint64_t x0, uint64_t x1) {
	uint64_t d0 = x0 ^ L.s0, d1 = x1 ^ L.s1;
	L.a += (uint64_t)(uint32_t)d0 * (uint64_t)(uint32_t)(d0 >> 32) + x1;
	L.b += (uint64_t)(uint32_t)d1 * (uint64_t)(uint32_t)(d1 >> 32) + x0;
}
__device__ __forceinline__ void ef_scramble(EfLane &L) {
	L.a = ((L.a ^ (L.a >> 47)) ^ L.s2) * 0x9E3779B1ULL;
	L.b = ((L.b ^ (L.b >> 47)) ^ L.s3) * 0x85EBCA77ULL;
}

// Whole-warp call.  `src` 16-byte aligned; bytes at or beyond n read as zero.  Result on all lanes.
// COHERENT: the page was written by the calling kernel, so it is read through the L2
// (ld.global.cg) and never through the read-only path, which may hold stale lines.
template <bool COHERENT = false>
__device__ __forceinline__ void warp_fingerprint128(const uint8_t *src, uint32_t n, int lane,
    uint64_t &hi, uint64_t &lo) {
	EfLane L;
	ef_init(L, lane);
	const uint32_t full = n >> 9;             // stripes made only of real bytes
	const uint32_t stripes = (n + 511) >> 9;
	const uint4 *v = reinterpret_cast<const uint4 *>(src) + lane;
	uint32_t s = 0;
	// 16-stripe groups: 16 independent 16-byte loads in flight per lane, one scramble per group.
	for (; s + 16 <= full; s += 16) {
		uint4 x[16];
#pragma unroll
		for (int k = 0; k < 16; k++) x[k] = COHERENT ? __ldcg(v + (size_t)(s + k) * 32) : __ldg(v + (size_t)(s + k) * 32);
#pragma unroll
		for (int k = 0; k < 16; k++)
			ef_absorb(L, (uint64_t)x[k].x | ((uint64_t)x[k].y << 32),
			    (uint64_t)x[k].z | ((uint64_t)x[k].w << 32));
		ef_scramble(L);
	}
	for (; s < stripes; s++) {
		uint32_t off = s * 512 + lane * 16;
		uint64_t x0 = 0, x1 = 0;
		if (off + 16 <= n) {
			uint4 x = COHERENT ? __ldcg(v + (size_t)s * 32) : __ldg(v + (size_t)s * 32);
			x0 = (uint64_t)x.x | ((uint64_t)x.y << 32);
			x1 = (uint64_t)x.z | ((uint64_t)x.w << 32);
		} else {
			for (uint32_t k = 0; k < 16 && off + k < n; k++) {
				uint64_t byte = COHERENT ? (uint64_t)__ldcg(src + off + k) : ldg8(src + off + k);
				if (k < 8) x0 |= byte << (8 * k); else x1 |= byte << (8 * (k - 8));
			}
		}
		ef_absorb(L, x0, x1);
		if ((s & 15u) == 15u) ef_scramble(L);
	}
	uint64_t u = ef_fold(L.a ^ L.s0, L.b ^ L.s1);
	uint64_t w = ef_fold(L.a ^ L.s3, L.b ^ L.s2);
	u = warp_sum_u64(u);
	w = warp_sum_u64(w);
	lo = ef_av((uint64_t)n * 0x9E3779B185EBCA87ULL + u);
	hi = ef_av(~((uint64_t)n * 0xC2B2AE3D27D4EB4FULL) + w);
}

// EF128 split by 16-stripe groups, for a page that a whole CTA holds (k_get_small's shared memory).
// Inside a group the absorb step only adds to a and b (mod 2^64), and what it adds depends on the
// input and the lane's secrets alone, so with A_g = lane l's sum over group g,
//   a after group g = scramble(a before + A_g),
// and the groups' sums can be taken by different warps at once.  One warp then chains them: a group
// that reaches its 16th stripe is followed by a scramble, a trailing shorter group is added without one.
// Same result as warp_fingerprint128 for every n.
constexpr uint32_t EF_GROUP_BYTES = 16u * 512u;
__host__ __device__ __forceinline__ uint32_t ef_groups(uint32_t n) { return (n + EF_GROUP_BYTES - 1u) / EF_GROUP_BYTES; }

// Lane sums {A, B} of group g of the n bytes at `src` (8-byte aligned, any state space the generic
// address reaches; bytes at or beyond n read as zero).
__device__ __forceinline__ ulonglong2 ef_group_sum(const uint8_t *src, uint32_t n, uint32_t g, int lane) {
	EfLane G;
	G.s0 = ef_secret(4 * lane); G.s1 = ef_secret(4 * lane + 1);
	G.a = 0; G.b = 0;
	const uint32_t stripes = (n + 511u) >> 9, end = min(stripes, 16u * g + 16u);
	for (uint32_t s = 16u * g; s < end; s++) {
		const uint32_t off = s * 512u + (uint32_t)lane * 16u;
		uint64_t x0 = 0, x1 = 0;
		if (off + 16u <= n) {
			x0 = *reinterpret_cast<const uint64_t *>(src + off);
			x1 = *reinterpret_cast<const uint64_t *>(src + off + 8u);
		} else {
			for (uint32_t k = 0; k < 16u && off + k < n; k++) {
				const uint64_t byte = src[off + k];
				if (k < 8) x0 |= byte << (8 * k); else x1 |= byte << (8 * (k - 8));
			}
		}
		ef_absorb(G, x0, x1);
	}
	return make_ulonglong2(G.a, G.b);
}

// Whole-warp call: chains the lane sums sums[32 g + lane] of every group of an n-byte page and folds
// them.  Result on all lanes.
__device__ __forceinline__ void ef_group_finish(const ulonglong2 *sums, uint32_t n, int lane, uint64_t &hi, uint64_t &lo) {
	EfLane L;
	ef_init(L, lane);
	const uint32_t groups = ef_groups(n), full = ((n + 511u) >> 9) >> 4;   // groups that reach their 16th stripe
	for (uint32_t g = 0; g < groups; g++) {
		const ulonglong2 s = sums[32u * g + (uint32_t)lane];
		L.a += s.x; L.b += s.y;
		if (g < full) ef_scramble(L);
	}
	uint64_t u = ef_fold(L.a ^ L.s0, L.b ^ L.s1);
	uint64_t w = ef_fold(L.a ^ L.s3, L.b ^ L.s2);
	u = warp_sum_u64(u);
	w = warp_sum_u64(w);
	lo = ef_av((uint64_t)n * 0x9E3779B185EBCA87ULL + u);
	hi = ef_av(~((uint64_t)n * 0xC2B2AE3D27D4EB4FULL) + w);
}

// EF128 computed along the frontier of another pass over the same page (the LZ4 parse): stripes
// are absorbed in order as the caller's position advances, one stripe requested ahead of need, so
// the page crosses HBM once and the stripe loads double as a prefetch for the parse that follows
// them.  Same result as warp_fingerprint128; `src` 16-byte aligned.
struct EfFrontier {
	EfLane L;
	uint4 ahead;          // stripe `next`, already requested
	uint32_t next;        // next stripe to absorb
	uint32_t full;        // stripes made only of real bytes

	__device__ __forceinline__ void start(const uint8_t *src, uint32_t n, int lane) {
		ef_init(L, lane);
		next = 0;
		full = n >> 9;
		ahead = full ? ef_ld16(reinterpret_cast<const uint4 *>(src) + lane) : make_uint4(0, 0, 0, 0);
	}
	__device__ __forceinline__ void take(const uint4 &x) {
		ef_absorb(L, (uint64_t)x.x | ((uint64_t)x.y << 32), (uint64_t)x.z | ((uint64_t)x.w << 32));
		if ((next & 15u) == 15u) ef_scramble(L);
		next++;
	}
	// absorb every full stripe that starts below `pos`
	__device__ __forceinline__ void upto(const uint8_t *src, uint32_t pos, int lane) {
		const uint32_t target = min(full, (pos + 511u) >> 9);
		if (next >= target) return;
		const uint4 *v = reinterpret_cast<const uint4 *>(src) + lane;
		take(ahead);
		// a long match jumped ahead: single stripes up to a scramble boundary, then 16 stripes per
		// step with 16 loads in flight, then the remainder
		while (next < target && (next & 15u)) { const uint4 x = ef_ld16(v + (size_t)next * 32); take(x); }
		while (target - next >= 16u) {
			uint4 x[16];
#pragma unroll
			for (int k = 0; k < 16; k++) x[k] = ef_ld16(v + (size_t)(next + k) * 32);
#pragma unroll
			for (int k = 0; k < 16; k++)
				ef_absorb(L, (uint64_t)x[k].x | ((uint64_t)x[k].y << 32), (uint64_t)x[k].z | ((uint64_t)x[k].w << 32));
			ef_scramble(L);
			next += 16;
		}
		while (next < target) { const uint4 x = ef_ld16(v + (size_t)next * 32); take(x); }
		if (next < full) ahead = ef_ld16(v + (size_t)next * 32);
	}
	// absorb the rest of the page (incl. a zero-padded partial stripe) and fold the lanes
	__device__ __forceinline__ void finish(const uint8_t *src, uint32_t n, int lane, uint64_t &hi, uint64_t &lo) {
		upto(src, n, lane);                               // all full stripes
		const uint32_t stripes = (n + 511u) >> 9;
		if (next < stripes) {                             // partial last stripe
			const uint32_t off = next * 512u + lane * 16u;
			uint64_t x0 = 0, x1 = 0;
			for (uint32_t k = 0; k < 16 && off + k < n; k++) {
				const uint64_t byte = ldg8(src + off + k);
				if (k < 8) x0 |= byte << (8 * k); else x1 |= byte << (8 * (k - 8));
			}
			ef_absorb(L, x0, x1);
			if ((next & 15u) == 15u) ef_scramble(L);
			next++;
		}
		uint64_t u = ef_fold(L.a ^ L.s0, L.b ^ L.s1);
		uint64_t w = ef_fold(L.a ^ L.s3, L.b ^ L.s2);
		u = warp_sum_u64(u);
		w = warp_sum_u64(w);
		lo = ef_av((uint64_t)n * 0x9E3779B185EBCA87ULL + u);
		hi = ef_av(~((uint64_t)n * 0xC2B2AE3D27D4EB4FULL) + w);
	}
};

}  // namespace cmb
