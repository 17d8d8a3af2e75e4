// lz4_encode_ring.cuh — the warp-per-chunk LZ4 1.8.1 encoder of lz4_encode.cuh with the page's
// sliding window staged in shared memory by TMA (sm_90a: cp.async.bulk + mbarrier).
//
// Output bytes: LZ4_compress_fast of the reference (cachemap/lz4.c:532-733 behind filemap.c:124-128); what
// changes is where the parse frontier reads the page from.  Profile of the plain kernel (round 1,
// T-class pages): 46 % of the stall samples are long-scoreboard waits on the two dependent page
// reads of a batch — the probe neighbourhoods (30 lanes x 12 bytes spread over ~350 bytes ahead of
// the anchor) and the candidate neighbourhoods (anywhere earlier in the page).  Both go through an
// L1 of ~28 KB that 14 warps share and that the fingerprint's streaming loads keep flushing, so a
// warp-wide load almost always waits for an L2 round trip (a load is as slow as its slowest lane).
//
// Here every warp owns a 1 KiB ring of the page around its parse frontier:
//   * four 256-byte buffers; buffer g & 3 holds page bytes [256 g, 256 g + 256);
//   * ONE lane issues cp.async.bulk (global -> shared, 256 B, no registers, no L1 allocation) for
//     the buffers ahead of the frontier and arms the buffer's mbarrier with the byte count; the warp
//     waits on the mbarrier (try_wait.parity) only when the frontier first enters a buffer, i.e. once
//     per 256 bytes of parse (~10 LZ4 sequences on text-like pages), by which time the copy issued
//     256-768 bytes earlier has long landed;
//   * a batch (refill + re-test + 30 probes) reads bytes [anchor - 4, anchor + 376): at most three
//     buffers, so the fourth is always free to prefetch into;
//   * the probe neighbourhoods and the speculative literal bytes then come from shared memory
//     (29-cycle LDS, conflict-free: lanes are 12 bytes = 3 banks apart), which removes the first of
//     the two page round trips from the per-sequence chain and leaves the L1 to the candidate reads
//     (the fingerprint frontier loads with L1::no_allocate).
// The ring needs 1 KiB + 4 mbarriers per warp next to the 16 KiB position table: 13 chunks per SM
// instead of 14 (one CTA of 13 warps).  It serves accel <= 12 (the reference's setting,
// edgefs.c:168; a larger accel spreads 30 probes over more than the ring holds) — other
// accelerations use the plain kernel.
#pragma once
#include "lz4_encode.cuh"
#include "kernels.h"

namespace cmb {

constexpr uint32_t RING_BYTES = 1024, RING_BUF = 256, RING_BUFS = 4;
constexpr uint32_t RING_MIRROR = 16;       // the ring's first 16 bytes again behind its end: a 16-byte read never wraps
constexpr uint32_t RING_ALLOC = RING_BYTES + 64;   // per-warp allocation (ring + mirror, keeps 64-byte alignment)
constexpr uint32_t RING_AHEAD = 376;      // a batch reads page bytes [anchor - 4, anchor + RING_AHEAD)
constexpr uint32_t RING_MAX_ACCEL = 12;   // 2 + accel * 29 + 12 <= RING_AHEAD, first batch 2 + accel * 30 + 12
constexpr uint32_t RING_MBAR_BYTES = 64;  // 4 x 8-byte mbarriers, padded
constexpr uint32_t RING_WARP_SMEM = LZ4_TABLE_BYTES + RING_ALLOC + RING_MBAR_BYTES;

__device__ __forceinline__ uint32_t smem_addr(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t arrivals) {
	asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(arrivals) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
	asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
// TMA 1-D bulk copy global -> shared, completion counted in bytes on `bar` (SASS: UBLKCP).
__device__ __forceinline__ void tma_load_1d(uint32_t dst, const void *src, uint32_t bytes, uint32_t bar) {
	asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst),
	    "l"(src), "r"(bytes), "r"(bar)
	    : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint32_t bar, uint32_t parity) {
	uint32_t ok;
	asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
	    : "=r"(ok)
	    : "r"(bar), "r"(parity)
	    : "memory");
	return ok != 0;
}

// One warp's window of the page it is encoding.  All members are warp-uniform and stay in
// registers: the cold part (ring_advance) is an out-of-line function that takes and returns them
// by value, so nothing of the ring state lives in local memory.
struct PageRing {
	const uint8_t *bytes;  // RING_BYTES of shared memory, 128-byte aligned
	uint32_t s_bytes;      // the same as a shared-space address
	uint32_t s_bar;        // shared-space address of the RING_BUFS mbarriers
	uint32_t issued;       // page buffers [.., issued) have been requested from TMA
	uint32_t ready;        // page buffers [.., ready) have landed and been waited for
	uint32_t parity;       // bit r: phase of ring buffer r's mbarrier that the next wait expects
};

__device__ __forceinline__ void ring_wait_buf(uint32_t s_bar, uint32_t &parity, uint32_t g) {
	const uint32_t r = g & (RING_BUFS - 1u);
	while (!mbar_try_wait(s_bar + 8u * r, (parity >> r) & 1u)) {}
	parity ^= 1u << r;
}

// once per warp, before the first page
__device__ __forceinline__ void ring_setup(PageRing &ring, uint8_t *ring_smem, uint8_t *bar_smem, int lane) {
	ring.bytes = ring_smem;
	ring.s_bytes = smem_addr(ring_smem);
	ring.s_bar = smem_addr(bar_smem);
	ring.issued = ring.ready = 0;
	ring.parity = 0;
	if (lane == 0) {
#pragma unroll
		for (uint32_t r = 0; r < RING_BUFS; r++) mbar_init(ring.s_bar + 8u * r, 1u);
		asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
		asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
	}
	__syncwarp();
}

// Called when the parse frontier enters page buffer g_lo (and once at the start of a page): makes
// buffers [g_lo, g_lo + 2] resident — a batch reads bytes [anchor - 4, anchor + RING_AHEAD), which
// never reach past g_lo + 2 — and requests g_lo + 3.  In the steady state that is one wait (for
// the buffer requested two crossings ago) and one request.  Every buffer that was requested is
// waited for exactly once and in order, also those a long match jumped over, so a ring buffer is
// never handed to TMA again while an earlier copy into it is in flight.
// state = issued | ready << 16 | parity << 32, in and out (page sizes up to 2^20: < 2^16 buffers).
__device__ __noinline__ uint64_t ring_advance(uint32_t s_bytes, uint32_t s_bar, uint64_t state, const uint8_t *src,
    uint32_t n, uint32_t nbufs, uint32_t g_lo, int lane) {
	uint32_t issued = (uint32_t)state & 0xffffu, ready = (uint32_t)(state >> 16) & 0xffffu, parity = (uint32_t)(state >> 32);
	const uint32_t g_hi = min(g_lo + 2u, nbufs - 1u);
	// (1) requested buffers that are needed, or that the parse has already left behind (a long match
	//     jumped over them), must have landed before their ring buffer can be reused
	const uint32_t upto = min(issued, g_hi + 1u);
	while (ready < upto) { ring_wait_buf(s_bar, parity, ready); ready++; }
	// (2) the jump went past everything requested so far: restart at g_lo
	if (issued < g_lo) { issued = g_lo; ready = g_lo; }
	// (3) request what the ring has room for: buffers below g_lo are dead, so [g_lo, g_lo + 4) fit
	const uint32_t want = min(g_lo + RING_BUFS, nbufs);
	__syncwarp();                                   // every lane is done reading the buffers being replaced
	if (lane == 0) {
		for (uint32_t g = issued; g < want; g++) {
			const uint32_t r = g & (RING_BUFS - 1u);
			// whole 16-byte units; the last buffer of a ragged page reads < 16 bytes past its end
			// (page buffers are padded: src is readable up to 16 bytes past src + n)
			const uint32_t nb = min(RING_BUF, (n - g * RING_BUF + 15u) & ~15u);
			const uint8_t *from = src + (size_t)g * RING_BUF;
			mbar_expect_tx(s_bar + 8u * r, nb + (r == 0u ? RING_MIRROR : 0u));
			tma_load_1d(s_bytes + r * RING_BUF, from, nb, s_bar + 8u * r);
			if (r == 0u) tma_load_1d(s_bytes + RING_BYTES, from, RING_MIRROR, s_bar);   // the mirror of the ring's head
		}
	}
	if (issued < want) issued = want;
	// (4) what the batches in this buffer read
	while (ready <= g_hi) { ring_wait_buf(s_bar, parity, ready); ready++; }
	return (uint64_t)issued | ((uint64_t)ready << 16) | ((uint64_t)parity << 32);
}
__device__ __forceinline__ void ring_step(PageRing &ring, const uint8_t *src, uint32_t n, uint32_t nbufs, uint32_t g_lo,
    int lane) {
	const uint64_t st = ring_advance(ring.s_bytes, ring.s_bar,
	    (uint64_t)ring.issued | ((uint64_t)ring.ready << 16) | ((uint64_t)ring.parity << 32), src, n, nbufs, g_lo, lane);
	ring.issued = (uint32_t)st & 0xffffu; ring.ready = (uint32_t)(st >> 16) & 0xffffu; ring.parity = (uint32_t)(st >> 32);
}
// nothing may be in flight when the page (or the kernel) ends
__device__ __forceinline__ void ring_drain(PageRing &ring) {
	while (ring.ready < ring.issued) { ring_wait_buf(ring.s_bar, ring.parity, ring.ready); ring.ready++; }
}

// The 12 page bytes [p-4, p+8) from the ring (p inside the resident window), as lz4_around: one
// address, four shared-memory words at fixed offsets (the mirrored tail absorbs the wrap).
__device__ __forceinline__ Lz4Around ring_around(const uint8_t *ring, uint32_t p) {
	const uint32_t sh = (p & 3u) * 8u;
	const uint32_t *q = reinterpret_cast<const uint32_t *>(ring + (((p & ~3u) - 4u) & (RING_BYTES - 1u)));
	const uint32_t w0 = q[0], w1 = q[1], w2 = q[2], w3 = q[3];     // p < 4: w0 is not page data, and is never used
	Lz4Around r;
	r.before = __funnelshift_r(w0, w1, sh);
	r.at = __funnelshift_r(w1, w2, sh);
	r.next = __funnelshift_r(w2, w3, sh);
	return r;
}

#ifdef CMB_ENC_PHASES   /* diagnostic builds only (tools/encode_phases.py) */
// Where the cycles of one parse iteration go.  Lane 0 of every fourth resident warp slot stamps
// clock64() at fixed points of each iteration and adds the cycles since its previous stamp to the
// phase that has just ended (a warp issues in order, so a stamp counts every stall of the
// instructions before it).  Row per chunk: ENC_PH_N cycle sums, then ENC_PH_N counts.
enum : uint32_t {
	ENC_PH_HEAD,           // end of the previous iteration -> past the loop-head test (events excluded)
	ENC_PH_EVENTS,         // checkpoint / ring / fingerprint events
	ENC_PH_TABLE,          // ring read, hash, table get / put, candidate-load issue, read-back
	ENC_PH_EMIT,           // deferred emit, fast path
	ENC_PH_WAIT,           // literal bytes, candidate bytes' first use, the two ballots
	ENC_PH_RESOLVE,        // winner, shuffles, undo stores, next anchor
	ENC_PH_SEARCH_SLOW,    // lz4_search_slow
	ENC_PH_COUNT_LONG,     // lz4_count_long
	ENC_PH_CATCHUP_LONG,   // lz4_catchup_long
	ENC_PH_EMIT_GENERAL,   // lz4_emit_general (deferred emit, long runs)
	ENC_PH_N
};
__device__ unsigned long long *g_enc_phases;   // null = off
__shared__ unsigned long long *s_enc_phase_row[32];   // per warp of the CTA: its chunk's row, or null
struct EncPhaseClock {
	unsigned long long *row;
	unsigned long long t;
	__device__ __forceinline__ void start(int lane) {
		row = lane == 0 ? s_enc_phase_row[threadIdx.x >> 5] : nullptr;
		t = clock64();
	}
	__device__ __forceinline__ void mark(uint32_t ph) {
		const unsigned long long now = clock64();
		if (row) { atomicAdd(row + ph, now - t); atomicAdd(row + ENC_PH_N + ph, 1ull); }
		t = now;
	}
};
#define ENC_PHASE(ph) phc.mark(ph)
#else
#define ENC_PHASE(ph) do {} while (0)
#endif

// Encodes src[0,n) into dst; returns the block length (uniform across the warp).  tab_smem = this
// warp's LZ4_TABLE_BYTES of shared memory; src must be 4-byte aligned and readable up to 16 bytes
// past src + n (the library's page buffers are contiguous and padded); with FP, 16-byte aligned.  With FP the EF128
// fingerprint of the page is computed along the way (EfFrontier): parse and fingerprint then read
// the page from HBM once.  RING: the probe neighbourhoods and literal bytes come from the warp's TMA ring
// (accel <= RING_MAX_ACCEL, src 16-byte aligned, `ring` set up by this warp); otherwise from global
// memory through the L1.
// One lane layout for every batch: lane 0 refills the slot of end-2 (lz4.c:691), lane 1 re-tests
// `end` (lz4.c:694-707), lane j >= 2 is probe j-2 of the search that starts at end+1
// (lz4.c:593-619).  The first search of a page (lz4.c:583-584: from position 1, nothing before it)
// is the same batch with end = 0 and the two special lanes switched off.
// The loop is written for a short in-order instruction stream (a warp issues in order; with one
// chain per warp every instruction of the body costs issue time whether or not the next sequence
// depends on it): everything that changes only every few hundred bytes — the fingerprint frontier,
// the ring — hangs off ONE comparison of the anchor with the position of the next such event.
template <bool WIDE, bool FP, bool RING>
__device__ uint32_t lz4_encode_lean(const uint8_t *__restrict__ src, uint32_t n, uint8_t *__restrict__ dst,
    uint32_t accel, uint8_t *tab_smem, PageRing &ring, int lane, uint64_t &fp_hi, uint64_t &fp_lo, uint32_t &ck) {
	Lz4Table<WIDE> tab;
	tab.t = reinterpret_cast<decltype(tab.t)>(tab_smem);
	const uint32_t lim4 = (n + 3u) & ~3u;
	uint32_t op = 0, anchor = 0;
	// Parse checkpoints for the CTA decoder (lz4_decode_cta.cuh): lane k (1..15) keeps where the first
	// sequence at or after k * n/16 starts — block offset << CKPT_POS_BITS | distance past that
	// position — or ~0 if none starts inside that sixteenth.  ck_at = the position the next one waits for.
	const uint32_t ck_span = n / CKPT_WORDS;
	uint32_t ck_k = 1, ck_at = ck_span ? ck_span : 0xffffffffu;
	ck = 0xffffffffu;
	EfFrontier fp;
	if (FP) fp.start(src, n, lane);

	// lz4.c:739 — table cleared per call: an untouched slot aliases position 0.
	{
		uint4 z = make_uint4(0, 0, 0, 0);
		uint4 *t4 = reinterpret_cast<uint4 *>(tab_smem);
#pragma unroll 4
		for (uint32_t i = lane; i < LZ4_TABLE_BYTES / 16; i += 32) t4[i] = z;
	}
	__syncwarp();

	if (n >= LZ4_MIN_INPUT) {
		const uint32_t mflimit = n - LZ4_MATCH_FIND_MARGIN;
		const uint32_t mlimit = n - LZ4_TAIL_LITERALS;
		const uint32_t nbufs = (n + RING_BUF - 1u) / RING_BUF;
		const uint8_t *const rb = ring.bytes;
		if (RING) ring.issued = ring.ready = 0;
		const bool special = lane < 2;
		const uint32_t kk = (uint32_t)lane - 2u;
		uint32_t delta2 = special ? 2u * (uint32_t)lane - 2u : 1u + (kk ? 1u + accel * (kk - 1u) : 0u);
		// A lane takes part while anchor < en_below: the probe after its own must stay <= mflimit
		// (lz4.c:601), i.e. anchor + need2 <= mflimit; the special lanes take part once a match has
		// ended (0 until then, everything afterwards).
		const uint32_t need2 = 2u + accel * kk;
		uint32_t en_below = special ? 0u : (mflimit >= need2 ? mflimit - need2 + 1u : 0u);
		const uint32_t special_on = special ? 0xffffffffu : 0u;
		// the two per-lane values the loop uses stay in registers (the compiler otherwise recomputes
		// them from the lane number on the critical path of every iteration)
		asm volatile("" : "+r"(delta2), "+r"(en_below));
		bool started = false;                                              // a match has ended (uniform)
		// Batch width.  Only the lanes up to the first hit matter; the rest of the 30 speculative probes
		// are table traffic and — worse — scattered candidate reads, most of which miss the L1 and
		// occupy the SM's outstanding-request slots (text-like pages find their match within the first
		// few probes).  So a chunk whose recent batches all hit early runs 16-lane batches (refill,
		// re-test, 14 probes); a 16-lane batch that finds nothing continues in lz4_search_slow from slot
		// 16 and the chunk goes back to 32 lanes for a while.  Same probes in the same order either way.
		constexpr uint32_t NARROW_W = 16u;                                 // lanes of a narrow batch
		constexpr int NARROW_HIT = 12;                                     // a hit at or above this lane widens the batch again
		uint32_t width = 32u, calm = 0u;                                    // lanes per batch; batches in a row that hit below NARROW_HIT
		uint32_t next_event = 0, ring_next = 0;                            // anchor at which the frontiers move next / a checkpoint is due
		// The sequence a batch resolves is written by the NEXT iteration, behind that batch's candidate
		// reads: the emit's stores and arithmetic (its size included) then fill the L2 round trip instead
		// of standing between one batch and the next.  From the top of an iteration to its deferred
		// emit, if `started`, one sequence is pending: it starts at dst[op] and at page position
		// anchor - LZ4_MIN_MATCH - p_mc - p_lit, and its first LZ4_LIT_REG literal bytes are in litw.
		uint32_t p_lit = 0, p_off = 0, p_mc = 0, litw = 0;
#ifdef CMB_ENC_PHASES
		EncPhaseClock phc;
		phc.start(lane);
#endif
		for (;;) {
			if (anchor >= next_event) {
				ENC_PHASE(ENC_PH_HEAD);
				// a sequence starts at or after the next checkpoint position: this is the one to note
				while (anchor >= ck_at) {
					const uint32_t rel = anchor - ck_at;
					const uint32_t at = op + (started ? lz4_seq_bytes(p_lit, p_mc) : 0u);   // behind the pending one
					if ((uint32_t)lane == ck_k) ck = rel < ck_span ? (at << CKPT_POS_BITS) | rel : 0xffffffffu;
					ck_k++;
					ck_at = ck_k < CKPT_WORDS ? ck_at + ck_span : 0xffffffffu;
				}
				if (anchor >= ring_next) {
				// every 256 bytes: ring buffers, then fingerprint stripes up to the probes (in this order:
				// the ring's out-of-line path would otherwise wait for the stripe the fingerprint prefetches)
				if (RING) {
					const uint32_t g_lo = (max(anchor, 4u) - 4u) / RING_BUF;
					if (ring.ready == g_lo + 2u && ring.issued == g_lo + 3u && g_lo + 3u < nbufs) {
						// steady state: the frontier moved on by one buffer.  Request g_lo + 3 into the buffer
						// g_lo - 1 has just left, wait for g_lo + 2 (requested two buffers ago).
						__syncwarp();
						if (lane == 0) {
							const uint32_t g = g_lo + 3u, r = g & (RING_BUFS - 1u);
							const uint32_t nb = min(RING_BUF, (n - g * RING_BUF + 15u) & ~15u);
							const uint8_t *from = src + (size_t)g * RING_BUF;
							mbar_expect_tx(ring.s_bar + 8u * r, nb + (r == 0u ? RING_MIRROR : 0u));
							tma_load_1d(ring.s_bytes + r * RING_BUF, from, nb, ring.s_bar + 8u * r);
							if (r == 0u) tma_load_1d(ring.s_bytes + RING_BYTES, from, RING_MIRROR, ring.s_bar);
						}
						ring.issued = g_lo + 4u;
						ring_wait_buf(ring.s_bar, ring.parity, g_lo + 2u);
						ring.ready = g_lo + 3u;
					} else {
						ring_step(ring, src, n, nbufs, g_lo, lane);
					}
					ring_next = (g_lo + 1u) * RING_BUF + 4u;
				} else {
					ring_next = (anchor | 255u) + 1u;
				}
				if (FP) fp.upto(src, anchor + 512u, lane);
				}
				next_event = min(ring_next, ck_at);
				ENC_PHASE(ENC_PH_EVENTS);
			}
			ENC_PHASE(ENC_PH_HEAD);
			const bool en = anchor < en_below && (uint32_t)lane < width;
			const uint32_t pos = en ? anchor + delta2 : 0u;        // disabled lanes read (and ignore) position 0 / ring offset 0
			const Lz4Around ai = RING ? ring_around(rb, pos) : lz4_around(src, pos);

			// ---- unified batch ----
			const uint32_t pseq = ai.at;
			const uint32_t h = WIDE ? lz4_hash5((uint64_t)ai.at | ((uint64_t)ai.next << 32)) : lz4_hash4(ai.at);
			const uint32_t cand = tab.get(h);
			__syncwarp();
			if (en) tab.put(h, pos);                                // speculative commit
			__syncwarp();
			Lz4Words acw = lz4_around_load(src, cand);   // latency overlaps the read-back and the emit below
			const uint32_t seen = tab.get(h);
			__syncwarp();                                           // read-backs done before any undo store
			ENC_PHASE(ENC_PH_TABLE);

			// ---- deferred emit of the pending sequence, while the candidate reads are in flight ----
			// It needs nothing of this batch: the fast path stores registers only, lz4_emit_general reads
			// the page from global memory (never from the ring, whose buffers the loop head recycles).
			if (started) {
				lz4_emit_seq(dst, src, op, anchor - LZ4_MIN_MATCH - p_mc - p_lit, p_lit, p_off, p_mc, litw, lane);
				op += lz4_seq_bytes(p_lit, p_mc);
				ENC_PHASE(p_lit <= LZ4_LIT_REG && p_mc < 15u + 255u ? ENC_PH_EMIT : ENC_PH_EMIT_GENERAL);
			}
			// speculative literal bytes of the sequence this batch resolves: src[anchor + 4 lane .. + 4)
			// (used when the run is <= LZ4_LIT_REG bytes; never stored beyond the literal run, so what a
			// lane reads past the page end does not matter).  In the ring: two aligned words inside the
			// resident [anchor - 4, anchor + RING_AHEAD), the mirror absorbing the wrap; from the page: a
			// lane past the end reads the last word instead (pages are padded by 16 bytes).
			{
				const uint32_t sh = (anchor & 3u) * 8u;
				if (RING) {
					const uint32_t *q = reinterpret_cast<const uint32_t *>(rb + (((anchor & ~3u) + 4u * (uint32_t)lane) & (RING_BYTES - 1u)));
					litw = __funnelshift_r(q[0], q[1], sh);
				} else {
					const uint32_t a = min((anchor & ~3u) + 4u * (uint32_t)lane, (n - 1u) & ~3u);
					litw = __funnelshift_r(ldg32(src + a), ldg32(src + a + 4u), sh);
				}
			}
			// The candidate words are first used here, behind the emit (the compiler would otherwise align
			// them right after the loads, and the warp would wait for the L2 before emitting).
			asm volatile("" : "+r"(acw.w0), "+r"(acw.w1), "+r"(acw.w2), "+r"(acw.w3));
			const Lz4Around ac = lz4_around_align(acw);
			const bool foreign = en && seen != (WIDE ? pos : (pos & 0xffffu));
			bool hit = en && lane != 0 && ac.at == pseq;
			if (WIDE) hit = hit && cand + LZ4_FAR >= pos;           // byU16: every distance fits (lz4.c:617)
			const uint32_t foreigns = __ballot_sync(CMB_FULL, foreign);
			const uint32_t hits = __ballot_sync(CMB_FULL, hit);
			uint32_t nf, nb;
			{
				const uint32_t xf = ai.next ^ ac.next;
				nf = xf ? (uint32_t)(__ffs(xf) - 1) >> 3 : 4u;
				nf = min(nf, mlimit - min(pos + LZ4_MIN_MATCH, mlimit));
				const uint32_t xb = ai.before ^ ac.before;
				nb = xb ? (uint32_t)__clz(xb) >> 3 : 4u;
				nb = min(nb, min(pos - min(anchor, pos), cand));
				if (special) nb = 0;                               // the re-test starts a sequence as is
			}
			const uint32_t low_hit = hits & (0u - hits), low_for = foreigns & (0u - foreigns);
			uint32_t ip, match, fwd, back;
			bool retest_hit;
			if (low_hit - 1u < low_for - 1u) {
				ENC_PHASE(ENC_PH_WAIT);
				const int w = __ffs(hits) - 1;
				const uint32_t pos_w = __shfl_sync(CMB_FULL, pos, w);
				if (en && lane > w && !(foreign && seen <= (WIDE ? pos_w : (pos_w & 0xffffu)))) tab.put(h, cand);
				__syncwarp();
				ip = pos_w;
				match = __shfl_sync(CMB_FULL, cand, w);
				fwd = __shfl_sync(CMB_FULL, nf, w);
				back = __shfl_sync(CMB_FULL, nb, w);
				retest_hit = w == 1;
				calm = w < NARROW_HIT ? calm + 1u : 0u;
				if (w >= NARROW_HIT) width = 32u; else if (calm >= 8u) width = NARROW_W;
				if (fwd == 4u || back == 4u) {                      // longer than the neighbourhoods show: rare
					ENC_PHASE(ENC_PH_RESOLVE);
					if (fwd == 4u) {
						fwd = 4u + lz4_count_long(src, ip + 8u, match + 8u, mlimit, lim4, lane);
						ENC_PHASE(ENC_PH_COUNT_LONG);
					}
					if (back == 4u && ip >= anchor + 5u && match >= 5u) {
						back = 4u + lz4_catchup_long(src, ip - 4u, match - 4u, anchor, lane);
						ENC_PHASE(ENC_PH_CATCHUP_LONG);
					}
				}
			} else {
				ENC_PHASE(ENC_PH_WAIT);
				uint64_t res = 0;
				// lanes of this batch that were held back only by the end margin (not by the batch width)
				const uint32_t enmask = __ballot_sync(CMB_FULL, en || special || (uint32_t)lane >= width);
				const uint32_t w0 = width;
				width = 32u; calm = 0u;
				if (foreigns) {
					if (en) tab.put(h, cand);
					__syncwarp();
					res = lz4_search_slow<WIDE>(src, lim4, tab, anchor, 2u, accel, mflimit, 0, lane, started);
				} else if (enmask == CMB_FULL) {                     // the probes of this batch were not enough
					res = lz4_search_slow<WIDE>(src, lim4, tab, anchor, 2u, accel, mflimit, w0, lane, started);
				}
				ENC_PHASE(ENC_PH_SEARCH_SLOW);
				if (!(res >> 63)) break;                             // -> last literals (nothing pending)
				retest_hit = (res >> 62) & 1u;
				ip = (uint32_t)(res >> 32) & 0x3fffffffu;
				match = (uint32_t)res;
				fwd = lz4_count_long(src, ip + LZ4_MIN_MATCH, match + LZ4_MIN_MATCH, mlimit, lim4, lane);
				ENC_PHASE(ENC_PH_COUNT_LONG);
				back = retest_hit ? 0u : lz4_catchup_long(src, ip, match, anchor, lane);
				ENC_PHASE(ENC_PH_CATCHUP_LONG);
			}
			// ---- the sequence becomes the pending one (emitted by the next iteration) ----
			p_off = ip - match;
			p_mc = back + fwd;                            // lz4.c:660 matchCode
			p_lit = ip - back - anchor;
			const uint32_t end = ip + LZ4_MIN_MATCH + fwd;

			anchor = end;
			started = true;
			en_below |= special_on;
			ENC_PHASE(ENC_PH_RESOLVE);
			if (end > mflimit) break;                     // lz4.c:688
		}
		// Still pending when the loop stopped at the end margin (anchor = end > mflimit).  A search that
		// ran into the margin has already emitted its predecessor (its anchor is <= mflimit).  Either way
		// the whole block is written before this function returns (and dst may be the arena).
		if (started && anchor > mflimit) {
			lz4_emit_seq(dst, src, op, anchor - LZ4_MIN_MATCH - p_mc - p_lit, p_lit, p_off, p_mc, litw, lane);
			op += lz4_seq_bytes(p_lit, p_mc);
		}
		if (RING) ring_drain(ring);
	}

	// the last literals are a sequence start like any other
	while (ck_k < CKPT_WORDS && ck_span) {
		const uint32_t rel = anchor - ck_at;
		if ((uint32_t)lane == ck_k) ck = (anchor >= ck_at && rel < ck_span) ? (op << CKPT_POS_BITS) | rel : 0xffffffffu;
		ck_k++;
		ck_at += ck_span;
	}

	// ---- last literals (lz4.c:713-729) ----
	uint32_t run = n - anchor;
	if (lane == 0) dst[op] = (uint8_t)(min(run, 15u) << 4);
	op++;
	if (run >= 15u) op = lz4_emit_len(dst, op, run - 15u, lane);
	lz4_copy_literals(dst + op, src + anchor, run, lane);
	op += run;
	if (FP) fp.finish(src, n, lane, fp_hi, fp_lo);
	return op;
}

}  // namespace cmb
