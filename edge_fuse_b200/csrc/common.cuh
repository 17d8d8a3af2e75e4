// common.cuh — device helpers shared by the cachemap kernels (sm_90a).
//
// Everything on this path is byte / integer work on 64 KiB chunks that live in HBM; the helpers
// here are the unaligned-access and warp-collective building blocks the LZ4 and fingerprint
// kernels are written in.  No tensor cores are involved anywhere (see DESIGN.md §3).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#define CMB_FULL 0xffffffffu
#define CMB_CHECK(expr)                                                         \
	do {                                                                    \
		cudaError_t e_ = (expr);                                        \
		if (e_ != cudaSuccess) {                                        \
			cmb_set_error(#expr, e_, __FILE__, __LINE__);           \
			return -1;                                              \
		}                                                               \
	} while (0)

void cmb_set_error(const char *what, cudaError_t e, const char *file, int line);

namespace cmb {

// Read-only (non-coherent, L1-cached) loads of input pages.  Pages are immutable for the life of
// the kernel, so ld.global.nc is legal and lets the 128-byte L1 line absorb the probe / verify /
// literal-copy re-reads of the same neighbourhood.
__device__ __forceinline__ uint32_t ldg32(const uint8_t *p) {
	return __ldg(reinterpret_cast<const uint32_t *>(p));
}
__device__ __forceinline__ uint32_t ldg8(const uint8_t *p) { return __ldg(p); }

// Byte store of encoder output.
__device__ __forceinline__ void st_out8(uint8_t *p, uint32_t v) { *p = (uint8_t)v; }

// Little-endian 32-bit read at an arbitrary byte offset `pos` of a 4-byte-aligned base.
// `lim4` is the chunk length rounded up to 4: the second word is only touched when it lies
// inside the chunk, so nothing past the rounded end is ever read.
__device__ __forceinline__ uint32_t read32u(const uint8_t *base, uint32_t pos, uint32_t lim4) {
	uint32_t a = pos & ~3u;
	uint32_t w0 = ldg32(base + a);
	uint32_t w1 = (a + 4 < lim4) ? ldg32(base + a + 4) : 0u;
	return __funnelshift_r(w0, w1, (pos & 3u) * 8u);
}
__device__ __forceinline__ uint64_t read64u(const uint8_t *base, uint32_t pos, uint32_t lim4) {
	uint32_t a = pos & ~3u;
	uint32_t w0 = ldg32(base + a);
	uint32_t w1 = (a + 4 < lim4) ? ldg32(base + a + 4) : 0u;
	uint32_t w2 = (a + 8 < lim4) ? ldg32(base + a + 8) : 0u;
	uint32_t sh = (pos & 3u) * 8u;
	return (uint64_t)__funnelshift_r(w0, w1, sh) | ((uint64_t)__funnelshift_r(w1, w2, sh) << 32);
}

// Warp-cooperative copy global -> global, arbitrary alignment on both sides, src read through
// the read-only path.  16-byte stores once dst is aligned; each lane funnels five aligned source
// words into one 16-byte vector.  Requires the source allocation to be readable up to the next
// 4-byte boundary past src+len (true for every page / record buffer in this library).
__device__ __forceinline__ void warp_copy_ro(uint8_t *dst, const uint8_t *src, uint32_t len, int lane) {
	if (len <= 32) {
		if ((uint32_t)lane < len) dst[lane] = (uint8_t)ldg8(src + lane);
		return;
	}
	uint32_t head = (16u - (uint32_t)(reinterpret_cast<uintptr_t>(dst) & 15u)) & 15u;
	if ((uint32_t)lane < head) dst[lane] = (uint8_t)ldg8(src + lane);
	dst += head; src += head; len -= head;
	uint32_t nvec = len >> 4;
	uint32_t sh = (uint32_t)(reinterpret_cast<uintptr_t>(src) & 3u) * 8u;
	const uint8_t *s4 = src - (reinterpret_cast<uintptr_t>(src) & 3u);
	for (uint32_t i = lane; i < nvec; i += 32) {
		const uint8_t *q = s4 + (size_t)i * 16;
		uint32_t w0 = ldg32(q), w1 = ldg32(q + 4), w2 = ldg32(q + 8), w3 = ldg32(q + 12);
		uint32_t w4 = sh ? ldg32(q + 16) : 0u;
		uint4 v;
		v.x = __funnelshift_r(w0, w1, sh);
		v.y = __funnelshift_r(w1, w2, sh);
		v.z = __funnelshift_r(w2, w3, sh);
		v.w = __funnelshift_r(w3, w4, sh);
		*reinterpret_cast<uint4 *>(dst + (size_t)i * 16) = v;
	}
	uint32_t rem = len & 15u;
	if ((uint32_t)lane < rem) dst[nvec * 16 + lane] = (uint8_t)ldg8(src + nvec * 16 + lane);
}

// Same shape for a source that this warp itself may have written (coherent loads).
__device__ __forceinline__ void warp_copy_rw(uint8_t *dst, const uint8_t *src, uint32_t len, int lane) {
	uint32_t head = (16u - (uint32_t)(reinterpret_cast<uintptr_t>(dst) & 15u)) & 15u;
	if (head > len) head = len;
	if ((uint32_t)lane < head) dst[lane] = src[lane];
	dst += head; src += head; len -= head;
	uint32_t nvec = len >> 4;
	if ((reinterpret_cast<uintptr_t>(src) & 15u) == 0) {
		for (uint32_t i = lane; i < nvec; i += 32)
			*reinterpret_cast<uint4 *>(dst + (size_t)i * 16) =
			    *reinterpret_cast<const uint4 *>(src + (size_t)i * 16);
	} else {
		uint32_t sh = (uint32_t)(reinterpret_cast<uintptr_t>(src) & 3u) * 8u;
		const uint8_t *s4 = src - (reinterpret_cast<uintptr_t>(src) & 3u);
		for (uint32_t i = lane; i < nvec; i += 32) {
			const uint32_t *q = reinterpret_cast<const uint32_t *>(s4 + (size_t)i * 16);
			uint32_t w0 = q[0], w1 = q[1], w2 = q[2], w3 = q[3];
			uint32_t w4 = sh ? q[4] : 0u;
			uint4 v;
			v.x = __funnelshift_r(w0, w1, sh);
			v.y = __funnelshift_r(w1, w2, sh);
			v.z = __funnelshift_r(w2, w3, sh);
			v.w = __funnelshift_r(w3, w4, sh);
			*reinterpret_cast<uint4 *>(dst + (size_t)i * 16) = v;
		}
	}
	uint32_t rem = len & 15u;
	if ((uint32_t)lane < rem) dst[nvec * 16 + lane] = src[nvec * 16 + lane];
}

__device__ __forceinline__ uint64_t warp_sum_u64(uint64_t v) {
#pragma unroll
	for (int d = 16; d > 0; d >>= 1) v += __shfl_xor_sync(CMB_FULL, v, d);
	return v;
}

}  // namespace cmb
