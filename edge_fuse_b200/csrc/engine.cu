// engine.cu — host side of the H100 cachemap engine: HBM layout, batch pipelines, C ABI.
//
// HBM layout per engine (one engine per GPU):
//   key table   (slots+2) x 64 B          replaces the 32 LMDB environments (filemap.c:54-90)
//   arena       bump-allocated records    {24-byte data_prefix, LZ4 block | raw page}
//   page ring   2 x max_batch x bsize     double-buffered landing zone for host pages
//   stage       one max(bsize+1024, LZ4_compressBound) row per resident encoder warp: block before it is packed into the arena
// Host tier (optional, cmb200_host_tier_enable): page-locked, device-mapped host memory holding records
// demoted from the arena, a ring in demotion order (DESIGN.md §2).
// A put batch is: H2D copy (copy stream)  ->  k_upsert  ->  k_encode (fingerprint + LZ4 + arena
// commit + table publish), sub-batch k+1's copy overlapping sub-batch k's kernels.
// A get batch is: k_lookup -> k_decode -> D2H copy.
#include <algorithm>
#include <atomic>
#include <condition_variable>
#include <deque>
#include <dirent.h>
#include <mutex>
#include <set>
#include <shared_mutex>
#include <sched.h>
#include <string>
#include <new>
#include <thread>
#include <unordered_map>
#include <unordered_set>
#include <utility>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <time.h>
#include <unistd.h>
#include <vector>
#include "../../include/cachemap_b200.h"
#include "../../include/uint128.h"
#include "kernels.h"
#include "common.cuh"
#include "streamgen.cuh"

static thread_local char g_err[512];

void cmb_set_error(const char *what, cudaError_t e, const char *file, int line) {
	snprintf(g_err, sizeof(g_err), "%s:%d: %s: %s", file, line, what, cudaGetErrorString(e));
}
static void set_error_msg(const char *msg) { snprintf(g_err, sizeof(g_err), "%s", msg); }

using namespace cmb;

// ---- owners of CUDA resources ------------------------------------------------------------------
// Each owner frees its resource in its destructor on the device it was made on, and leaves the
// calling thread's current device as it found it: a load or a snapshot of several engines releases
// one engine's buffers on a thread that often has another engine's device current.
template <class H, cudaError_t (*Release)(H)>
class Owned {
public:
	Owned() = default;
	Owned(Owned &&o) noexcept { *this = std::move(o); }
	Owned &operator=(Owned &&o) noexcept {
		if (this != &o) { reset(); std::swap(h_, o.h_); std::swap(dev_, o.dev_); std::swap(bytes_, o.bytes_); }
		return *this;
	}
	~Owned() { reset(); }
	void reset() {
		if (!h_) return;
		int cur = dev_;
		cudaGetDevice(&cur);
		if (cur != dev_) cudaSetDevice(dev_);
		Release(h_);
		if (cur != dev_) cudaSetDevice(cur);
		h_ = nullptr; bytes_ = 0;
	}
	H get() const { return h_; }
protected:
	int adopt(H h, size_t bytes = 0) {                   // h was just made on the current device
		reset();
		h_ = h; bytes_ = bytes;
		cudaGetDevice(&dev_);
		return 0;
	}
	H h_ = nullptr;
	int dev_ = 0;
	size_t bytes_ = 0;
};

template <class T = uint8_t>
struct DevMem : Owned<void *, cudaFree> {
	operator T *() const { return (T *)h_; }
	int alloc(size_t bytes) {
		reset();                                         // first: the old and the new never coexist
		void *p;
		CMB_CHECK(cudaMalloc(&p, bytes));
		return adopt(p, bytes);
	}
	// Scratch kept across calls: grown to the largest request, never shrunk (a cudaFree per call would
	// synchronise the whole device); the work on `st` that may still read it is waited for first.
	int grow(size_t bytes, cudaStream_t st) {
		if (bytes <= bytes_) return 0;
		CMB_CHECK(cudaStreamSynchronize(st));
		return alloc(bytes);
	}
};

template <class T = uint8_t>
struct HostMem : Owned<void *, cudaFreeHost> {            // page-locked
	operator T *() const { return (T *)h_; }
	int alloc(size_t bytes, bool mapped = false) {
		void *p;
		CMB_CHECK(cudaHostAlloc(&p, bytes, mapped ? cudaHostAllocMapped : cudaHostAllocDefault));
		return adopt(p);
	}
};

struct Stream : Owned<cudaStream_t, cudaStreamDestroy> {
	operator cudaStream_t() const { return h_; }
	int create() { cudaStream_t s; CMB_CHECK(cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking)); return adopt(s); }
};

struct Event : Owned<cudaEvent_t, cudaEventDestroy> {
	operator cudaEvent_t() const { return h_; }
	int create(unsigned flags) { cudaEvent_t ev; CMB_CHECK(cudaEventCreateWithFlags(&ev, flags)); return adopt(ev); }
};

// The key table's memory: cap + 2 slots and the side tables the engine's flags call for.  The kernels
// get it as a TableView, refreshed by view() whenever the table is replaced.
struct TableMem {
	DevMem<Slot> slots;
	DevMem<uint64_t> fp;
	DevMem<uint32_t> fp_tag, ckpt;
	void view(TableView &t) const { t.slots = slots; t.fp = fp; t.fp_tag = fp_tag; t.ckpt = ckpt; }
};

// Allocates the slots and each side table asked for, zeroed on st.  0 = done; 1 = a table found no
// room (error set, CUDA's cleared; m is left empty); -1 = another CUDA call failed (error set).
static int table_alloc(TableMem &m, uint64_t cap, bool fp, bool fp_tag, bool ckpt, cudaStream_t st) {
	const size_t n = cap + 2;
	if (m.slots.alloc(n * sizeof(Slot)) || (fp && m.fp.alloc(n * 16)) || (fp_tag && m.fp_tag.alloc(n * 4)) ||
	    (ckpt && m.ckpt.alloc(n * CKPT_WORDS * 4))) {
		(void)cudaGetLastError();
		m = TableMem{};
		return 1;
	}
	CMB_CHECK(cudaMemsetAsync(m.slots, 0, n * sizeof(Slot), st));
	if (fp) CMB_CHECK(cudaMemsetAsync(m.fp, 0, n * 16, st));
	if (fp_tag) CMB_CHECK(cudaMemsetAsync(m.fp_tag, 0, n * 4, st));
	if (ckpt) CMB_CHECK(cudaMemsetAsync(m.ckpt, 0, n * CKPT_WORDS * 4, st));
	return 0;
}

struct cmb200_engine {
	int device = 0;
	int pshift = 16;
	uint32_t bsize = 65536;
	int accel = 12;
	uint64_t capacity = 0;
	uint32_t max_batch = 4096;   // chunks per kernel launch (stage buffer size)
	uint32_t host_batch = 4096;  // chunks per H2D/D2H pipeline step (page ring size), <= max_batch
	uint32_t flags = 0;
	Stream st, copy;
	// small gets (cmb200_get_small) have their own stream, lock and buffers: they neither queue behind
	// a put batch on `st` nor take `mu`
	// Several small gets may be in flight at once (two leader threads of the combining queue, or any
	// callers of cmb200_get_small): each takes one LANE — a stream plus page-locked request / status
	// words — and the open side of get_gate; what moves records or peer mappings (compaction, peers,
	// destroy) closes get_gate.
	static constexpr int GET_LANES = 32;
	struct GetLane { std::atomic<int> busy{0}; Stream st; HostMem<int32_t> h_status; HostMem<cmb200_addr> h_addr; };
	GetLane lane[GET_LANES];
	// A small get may be begun by one thread and ended by another (cmb200_get_small_begin / _end), so
	// the "no small get in flight" condition is a counter and a closing flag, not a lock a thread owns.
	struct GetGate {
		std::atomic<int> active{0}, closed{0};
		void enter() {
			for (;;) {
				while (closed.load(std::memory_order_acquire)) sched_yield();
				active.fetch_add(1, std::memory_order_acq_rel);
				if (!closed.load(std::memory_order_acquire)) return;
				active.fetch_sub(1, std::memory_order_acq_rel);
			}
		}
		void leave() { active.fetch_sub(1, std::memory_order_acq_rel); }
		void close() {                        // exclusive: waits for the gets in flight, holds new ones off
			int open = 0;
			while (!closed.compare_exchange_weak(open, 1, std::memory_order_acq_rel)) { open = 0; sched_yield(); }
			while (active.load(std::memory_order_acquire)) sched_yield();
		}
		void reopen() { closed.store(0, std::memory_order_release); }
	} get_gate;
	struct GateClosed {                           // scope guard of the exclusive side
		GetGate &g;
		explicit GateClosed(GetGate &gate) : g(gate) { g.close(); }
		~GateClosed() { g.reopen(); }
	};
	std::atomic<uint32_t> lane_turn{0};
	static constexpr size_t GET_SMALL_MAX = 1024;
	const uint8_t *peer_base[GET_MAX_PEERS] = {};
	uint64_t peer_size[GET_MAX_PEERS] = {};
	std::atomic<uint64_t> small_get_requests{0}, small_get_hits{0}, small_get_launches{0};
	DevMem<unsigned long long> d_recoff_out;     // arena offset per chunk of the current put slice (exchange records)
	// k_get_small's sequence descriptors: one scratch region per CTA that can be resident (kernels.cu:gs_region_take)
	DevMem<uint4> d_scratch;
	DevMem<uint32_t> d_pool_bits;
	uint32_t pool_n = 0, region_entries = 0;
	Event landed[2], consumed[2];
	TableMem table_mem;
	TableView table{};
	DevMem<uint8_t> arena_base;
	DevMem<unsigned long long> arena_seg;
	ArenaView arena{};
	DevMem<unsigned long long> d_counters;      // entries, tombs, head, garbage, dropped
	DevMem<uint8_t> d_pages[2];
	DevMem<uint8_t> d_stage;
	uint64_t stage_stride = 0;
	DevMem<unsigned long long> d_addr, d_ts;
	DevMem<uint8_t> d_valid;
	DevMem<uint32_t> d_slot, d_vlen;
	DevMem<int32_t> d_lens, d_status;
	DevMem<uint64_t> d_fps, d_recoff;
	DevMem<unsigned int> d_work;
	DevMem<uint32_t> d_order;            // the encoder's longest-first chunk lists (encode_order_words(max_batch))
	DevMem<uint32_t> d_import_slot;      // slot scratch of cmb200_import_records_dev, grown, never shrunk
	DevMem<uint32_t> d_move_idx;         // index scratch of cmb200_move_pages (destination, then source), grown, never shrunk
	DevMem<unsigned long long> d_removed; // records removed by cmb200_invalidate, allocated by its first call
	// cmb200_rename: a slice's list and staged records, on the engine they leave and on the one they enter,
	// grown, never shrunk (rename_mu: one rename call at a time uses them)
	DevMem<uint8_t> d_ren_list, d_ren_bytes;
	// cmb200_patch_batch: the call's rows, spans and bytes, staged page-locked and copied over in one piece,
	// grown, never shrunk; and the tier-hit counter and hot log its decode books into instead of the gets'
	HostMem<uint8_t> h_patch;
	size_t h_patch_bytes = 0;
	DevMem<uint8_t> d_patch;
	DevMem<unsigned long long> d_patch_hot;
	// page-locked staging for the small per-chunk arrays, so that no copy ever blocks the host
	// thread that is feeding the pipeline (a pageable cudaMemcpyAsync waits for the stream)
	static constexpr size_t META_CAP = 1u << 18;   // chunks per outer slice of a call
	HostMem<uint8_t> h_meta;                       // META_CAP x (16 addr + 8 ts + 4 lens + 4 status + 1 valid)
	unsigned long long seq = 1;          // sequence of the next chunk
	unsigned long long seq_stride = 1;   // > 1 when the global stream is sharded round-robin over ranks
	// per-launch device timing of the dominant kernels (roofline evidence for bench.py)
	static constexpr int RING = 64;
	Event t0[RING], t1[RING];
	// asynchronous puts (cmb200_put_batch_async): kernel timing events not harvested yet are
	// p0/p1[pend_tail .. pend_head), completion tickets are events on the compute stream
	Event p0[RING], p1[RING];
	uint64_t pend_head = 0, pend_tail = 0;
	static constexpr int TICKETS = 8;
	Event ticket_ev[TICKETS];
	uint64_t tickets = 0;
	Event meta_done, meta_free[2];
	uint64_t ring_pos = 0;               // page ring buffer in turn, kept across calls
	uint64_t meta_pos = 0;               // same for the two copies of d_addr / d_ts / d_valid (host puts)
	size_t meta_cap = 0;                 // entries per copy
	std::mutex mu;
	cmb200_stats stats{};
	// host tier: a ring of records in demotion order.  Log position p lies at tier offset p % size; a
	// record never straddles the end of the ring (the rest of the lap is skipped).
	struct HostTier {
		HostMem<uint8_t> host;               // mapped; null = no tier
		uint8_t *dev = nullptr;              // its device address
		uint64_t size = 0;
		uint64_t head = 0;                   // log position of the next record
		std::deque<std::pair<uint64_t, uint32_t>> log;   // {position, bytes} of each record not yet overwritten, oldest first
		uint64_t demoted_records = 0, demoted_bytes = 0;
		uint64_t promoted_records = 0, promoted_bytes = 0;
		DevMem<unsigned long long> d_ctr;    // device: [0] records retired by wrap-around, [1] host-tier hits,
		                                     // [2] head of the hot log
		DevMem<ulonglong2> d_hot;            // the hot log: HOT_LOG_N addresses of tier hits
		uint64_t hot_drained = 0;            // hot-log head at the last cmb200_host_tier_hot
		DevMem<unsigned long long> d_retire; // {u, l, location, bytes} per record a wrap overwrites, grown, never shrunk
		DevMem<DemoteEntry> d_moves;         // max_batch entries
		DevMem<PromoteEntry> d_promote;      // max_batch entries
		HotLog hot() const { return HotLog{d_ctr ? d_ctr + 2 : nullptr, d_hot}; }
	} tier;
	std::atomic<bool> multi_gpu{false};  // a multi-GPU call was made: no host tier from then on
	// CMB200_VERIFY: device counters, VS_WORDS of the gets, then VS_WORDS of the running store scan
	DevMem<unsigned long long> d_vstat;
	DevMem<uint32_t> d_vidx;             // slot of each request of a verified or touching get batch (max_batch)
	uint64_t scanned = 0, scan_corrupt = 0;
	// snapshots (cmb200_snapshot_begin): SNAP_FREE, SNAP_CLAIMED by a snapshot that has not listed this
	// engine's records yet, or SNAP_PENDING: listed, section not written yet.  snap_state changes under
	// snap_mu and every change is broadcast on snap_cv.  Lock order: mu before snap_mu.  The snapshot's
	// writer takes snap_mu only, never mu, so a holder of mu may wait on snap_cv for the writer.
	enum { SNAP_FREE = 0, SNAP_CLAIMED, SNAP_PENDING };
	int snap_state = SNAP_FREE;
	std::mutex snap_mu;
	std::condition_variable snap_cv;
	HostMem<uint8_t> snap_win;           // page-locked window of the writer, kept from the first snapshot on
	Stream snap_st;                      // the writer's copies: they do not queue behind encodes on st
	// snapshot chains (cmb200_chain_begin): the file `id` and its `k` deltas describe this engine's
	// records as of the last tick, whose watermark was w (every record version put since has seq >= w)
	// and whose live addresses are the baseline base[cur][0 .. n).  The baseline is page-locked,
	// device-mapped host memory, double-buffered: a tick's export writes the next one into the other
	// half.  A tick that is listed and not finished keeps its results in the *_next fields until
	// cmb200_snapshot_finish commits them (the file is in place) or drops them.  Under mu.
	struct Chain {
		uint64_t id = 0;                 // 0 = no chain state: the next tick must write a base
		uint32_t k = 0;
		unsigned long long w = 0;
		HostMem<ulonglong2> base[2];
		ulonglong2 *base_dev[2] = {};
		uint64_t cap[2] = {}, n = 0;
		int cur = 0;
		bool pending = false;
		uint64_t id_next = 0, n_next = 0;
		uint32_t k_next = 0;
		unsigned long long w_next = 0;
	} chain;
};

// CMB200_TOUCH: the stamp a get raises its hits' ts to, taken at launch from the clock the drop-in's puts
// stamp with (cachemap_api.c:now_ns, the reference's cachemap.c:10-15).  Never 0 (GetJob::touch_ts).
static unsigned long long touch_stamp() {
	struct timespec tp;
	clock_gettime(CLOCK_REALTIME_COARSE, &tp);
	const unsigned long long ns = (unsigned long long)tp.tv_sec * 1000000000ull + (unsigned long long)tp.tv_nsec;
	return ns ? ns : 1ull;
}

static uint64_t next_pow2(uint64_t v) {
	uint64_t p = 1;
	while (p < v) p <<= 1;
	return p;
}

extern "C" const char *cmb200_last_error(void) { return g_err; }

extern "C" int cmb200_device_count(void) {
	int n = 0;
	cudaError_t e = cudaGetDeviceCount(&n);
	if (e != cudaSuccess) { cmb_set_error("cudaGetDeviceCount", e, __FILE__, __LINE__); return 0; }
	return n;
}

static int select_device(int device) {
	if (device >= 0) CMB_CHECK(cudaSetDevice(device));
	int n = 0;
	CMB_CHECK(cudaGetDeviceCount(&n));
	if (n == 0) { set_error_msg("no CUDA device"); return -1; }
	return 0;
}

extern "C" void cmb200_engine_destroy(cmb200_engine *e) {
	if (!e) return;
	cudaSetDevice(e->device);
	if (e->st) cudaStreamSynchronize(e->st);
	if (e->copy) cudaStreamSynchronize(e->copy);
	for (auto &ln : e->lane) if (ln.st) cudaStreamSynchronize(ln.st);
	for (int r = 0; r < GET_MAX_PEERS; r++) if (e->peer_base[r]) cudaIpcCloseMemHandle((void *)e->peer_base[r]);
	delete e;
}

static int engine_init(cmb200_engine *e, const cmb200_config *cfg) {
	cudaGetDevice(&e->device);
	e->pshift = cfg->pshift;
	e->bsize = 1u << cfg->pshift;
	e->accel = cfg->accel < 0 ? 1 : (cfg->accel > (1 << 20) ? (1 << 20) : cfg->accel);   // lz4.c:740
	e->capacity = cfg->capacity;
	e->max_batch = cfg->max_batch ? cfg->max_batch : 4096;
	// host pages are pipelined in smaller steps than a resident batch is launched in: the first
	// copy of a call cannot overlap anything, while a launch wants many chunks per warp
	e->host_batch = e->max_batch < 4096u ? e->max_batch : 4096u;
	e->flags = cfg->flags;
	if (e->flags & CMB200_VERIFY) e->flags |= CMB200_FINGERPRINT;
	const uint64_t B = e->max_batch;
	uint64_t slots = cfg->table_slots ? next_pow2(cfg->table_slots) : next_pow2(4 * (cfg->capacity ? cfg->capacity : 1024));
	if (slots < 1024) slots = 1024;
	if (slots > (1ull << 27)) slots = 1ull << 27;
	e->table.cap = slots;
	if (e->st.create() || e->copy.create()) return -1;
	for (auto &ln : e->lane) if (ln.st.create()) return -1;
	for (int i = 0; i < 2; i++)
		if (e->landed[i].create(cudaEventDisableTiming) || e->consumed[i].create(cudaEventDisableTiming)) return -1;
	for (int i = 0; i < cmb200_engine::RING; i++)
		if (e->t0[i].create(cudaEventDefault) || e->t1[i].create(cudaEventDefault) ||
		    e->p0[i].create(cudaEventDefault) || e->p1[i].create(cudaEventDefault)) return -1;
	for (Event &ev : e->ticket_ev) if (ev.create(cudaEventDisableTiming)) return -1;
	if (e->meta_done.create(cudaEventDisableTiming) || e->meta_free[0].create(cudaEventDisableTiming) ||
	    e->meta_free[1].create(cudaEventDisableTiming)) return -1;
	// parse checkpoints per slot (64 bytes) when the fused single-page get serves this page size
	const char *ck = getenv("CMB200_CKPT");
	const bool ckpt = get_small_supports(e->bsize) && (!ck || atoi(ck) != 0);
	if (table_alloc(e->table_mem, slots, e->flags & CMB200_FINGERPRINT, e->flags & CMB200_VERIFY, ckpt, e->st)) return -1;
	e->table_mem.view(e->table);
	if (e->flags & CMB200_VERIFY) {
		if (e->d_vstat.alloc(2 * VS_WORDS * sizeof(unsigned long long))) return -1;
		CMB_CHECK(cudaMemsetAsync(e->d_vstat, 0, 2 * VS_WORDS * sizeof(unsigned long long), e->st));
	}
	if ((e->flags & (CMB200_VERIFY | CMB200_TOUCH)) && e->d_vidx.alloc(B * 4)) return -1;
	if (get_small_supports(e->bsize)) {
		// the descriptor scratch of the fused single-page get
		const int resident = get_small_residency(e->bsize, e->table.fp_tag != nullptr, e->flags & CMB200_TOUCH);
		if (resident <= 0) { set_error_msg("k_get_small does not fit this device"); return -1; }
		e->pool_n = (uint32_t)resident;
		e->region_entries = get_small_region_entries(e->bsize);
		if (e->d_scratch.alloc((size_t)e->pool_n * e->region_entries * sizeof(uint4)) ||
		    e->d_pool_bits.alloc(((size_t)e->pool_n + 31) / 32 * 4)) return -1;
		CMB_CHECK(cudaMemsetAsync(e->d_pool_bits, 0, ((size_t)e->pool_n + 31) / 32 * 4, e->st));
	}
	if (e->d_counters.alloc(8 * sizeof(unsigned long long))) return -1;
	CMB_CHECK(cudaMemsetAsync(e->d_counters, 0, 8 * sizeof(unsigned long long), e->st));
	e->table.entries = e->d_counters + 0;
	e->table.tombs = e->d_counters + 1;
	e->arena.head = e->d_counters + 2;
	e->arena.garbage = e->d_counters + 3;
	e->arena.dropped = e->d_counters + 4;
	e->table.remote = e->d_counters + 5;
	e->arena.tier = e->d_counters + 6;

	// filemap.c:120 dest[bsize+1024], but never below LZ4_compressBound: the encoder has no output
	// limit, and above 128 KiB pages an incompressible block is longer than bsize + 1024 (k_encode
	// then stores the page raw, as LZ4_compress_fast's 0 would make filemap_set do)
	{
		const uint64_t bound = (uint64_t)e->bsize + e->bsize / 255 + 16;
		const uint64_t row = (uint64_t)e->bsize + 1024 > bound ? (uint64_t)e->bsize + 1024 : bound;
		e->stage_stride = (row + 15) & ~15ull;
	}
	if (e->d_pages[0].alloc((uint64_t)e->host_batch * e->bsize + 256) ||
	    e->d_pages[1].alloc((uint64_t)e->host_batch * e->bsize + 256)) return -1;
	// one stage row per resident warp / group of the encode kernels (store mode), not per chunk
	if (e->d_stage.alloc((uint64_t)16384 * e->stage_stride + 256)) return -1;
	// small per-chunk arrays are sized for a whole slice of a call (META_CAP chunks) so that
	// they cross PCIe once, outside the page pipeline
	const uint64_t M = cmb200_engine::META_CAP > B ? cmb200_engine::META_CAP : B;
	// two copies: a host put stages the next call's arrays while the kernels of the previous
	// one still read theirs (cmb200_put_batch_async)
	e->meta_cap = M;
	if (e->d_addr.alloc(2 * M * 16) || e->d_ts.alloc(2 * M * 8) || e->d_valid.alloc(2 * M) ||
	    e->d_slot.alloc(B * 4) || e->d_vlen.alloc(B * 4) || e->d_lens.alloc(M * 4) || e->d_status.alloc(M * 4) ||
	    e->d_fps.alloc(B * 16) || e->d_recoff.alloc(B * 8) || e->d_work.alloc(64) ||
	    e->d_order.alloc(encode_order_words((uint32_t)B) * 4) || e->h_meta.alloc(cmb200_engine::META_CAP * 33)) return -1;
	for (auto &ln : e->lane)
		if (ln.h_status.alloc(cmb200_engine::GET_SMALL_MAX * 4) || ln.h_addr.alloc(cmb200_engine::GET_SMALL_MAX * 16)) return -1;
	if (e->d_recoff_out.alloc(M * 8)) return -1;

	uint64_t arena = cfg->arena_bytes;
	if (!arena) {
		size_t free_b = 0, total_b = 0;
		CMB_CHECK(cudaMemGetInfo(&free_b, &total_b));
		// capacity worst-case records (24 + a stage row: a stored record is never longer, since a
		// block longer than bsize + 1024 is stored as the raw page) plus 1/8 headroom, so that a
		// store at capacity still has garbage worth compacting
		uint64_t want = (cfg->capacity ? cfg->capacity : 1024) * (e->stage_stride + 32);
		want += want / 8;
		uint64_t lim = (uint64_t)(free_b * 0.8);
		arena = want < lim ? want : lim;
	}
	arena = (arena + 255) & ~255ull;
	if (e->arena_base.alloc(arena + 256)) return -1;
	e->arena.base = e->arena_base;
	e->arena.size = arena;
	{
		// direct encode into per-warp arena segments when the arena is large enough that
		// 4096 segments of >= 4 worst-case records stay a small part of it
		// (CMB200_SEG_KB overrides: 0 = always through the stage buffer)
		const uint64_t worst = (24 + e->stage_stride + 15) & ~15ull;
		uint64_t seg = arena / (8ull * 2072ull);
		if (seg > (2ull << 20)) seg = 2ull << 20;
		if (seg < 4 * worst) seg = 0;
		const char *kb = getenv("CMB200_SEG_KB");
		if (kb && *kb) { seg = strtoull(kb, nullptr, 10) << 10; if (seg && seg < worst) seg = worst; }
		seg = (seg + 255) & ~255ull;
		e->arena.seg_bytes = (uint32_t)seg;
		if (e->arena_seg.alloc(ARENA_SEG_SLOTS * 2 * sizeof(unsigned long long))) return -1;
		CMB_CHECK(cudaMemsetAsync(e->arena_seg, 0, ARENA_SEG_SLOTS * 2 * sizeof(unsigned long long), e->st));
		e->arena.seg = e->arena_seg;
	}
	CMB_CHECK(cudaStreamSynchronize(e->st));
	return 0;
}

extern "C" cmb200_engine *cmb200_engine_create(const cmb200_config *cfg) {
	if (!cfg || cfg->pshift < 6 || cfg->pshift > 20) { set_error_msg("bad config: pshift must be 6..20"); return nullptr; }
	if (select_device(cfg->device) != 0) return nullptr;
	cmb200_engine *e = new (std::nothrow) cmb200_engine();
	if (!e) return nullptr;
	if (engine_init(e, cfg) == 0) return e;
	cmb200_engine_destroy(e);
	return nullptr;
}

extern "C" void *cmb200_host_alloc(size_t bytes) {
	void *p = nullptr;
	cudaError_t er = cudaMallocHost(&p, bytes);
	if (er != cudaSuccess) { cmb_set_error("cudaMallocHost", er, __FILE__, __LINE__); return nullptr; }
	return p;
}
extern "C" void cmb200_host_free(void *p) { if (p) cudaFreeHost(p); }
extern "C" void *cmb200_dev_alloc(cmb200_engine *e, size_t bytes) {
	void *p = nullptr;
	if (e) cudaSetDevice(e->device);
	cudaError_t er = cudaMalloc(&p, bytes + 256);
	if (er != cudaSuccess) { cmb_set_error("cudaMalloc", er, __FILE__, __LINE__); return nullptr; }
	return p;
}
extern "C" void cmb200_dev_free(cmb200_engine *e, void *p) { if (e) cudaSetDevice(e->device); if (p) cudaFree(p); }
extern "C" int cmb200_memcpy_h2d(cmb200_engine *e, void *dev, const void *host, size_t bytes) {
	cudaSetDevice(e->device);
	CMB_CHECK(cudaMemcpyAsync(dev, host, bytes, cudaMemcpyHostToDevice, e->st));
	CMB_CHECK(cudaStreamSynchronize(e->st));
	return 0;
}
extern "C" int cmb200_memcpy_d2h(cmb200_engine *e, void *host, const void *dev, size_t bytes) {
	cudaSetDevice(e->device);
	CMB_CHECK(cudaMemcpyAsync(host, dev, bytes, cudaMemcpyDeviceToHost, e->st));
	CMB_CHECK(cudaStreamSynchronize(e->st));
	return 0;
}
extern "C" void *cmb200_stream(cmb200_engine *e) { return (void *)e->st; }
extern "C" int cmb200_sync(cmb200_engine *e) {
	cudaSetDevice(e->device);
	CMB_CHECK(cudaStreamSynchronize(e->copy));
	CMB_CHECK(cudaStreamSynchronize(e->st));
	return 0;
}

// ---- put ---------------------------------------------------------------------------------

// Adds the kernel times of asynchronous puts whose events have completed to the statistics;
// wait = true blocks until every pending one has.
static void harvest_pending(cmb200_engine *e, bool wait) {
	while (e->pend_tail < e->pend_head) {
		const int k = (int)(e->pend_tail % cmb200_engine::RING);
		if (wait) cudaEventSynchronize(e->p1[k]);
		else if (cudaEventQuery(e->p1[k]) != cudaSuccess) { (void)cudaGetLastError(); break; }
		float ms = 0;
		if (cudaEventElapsedTime(&ms, e->p0[k], e->p1[k]) == cudaSuccess) {
			e->stats.encode_kernel_ns += (uint64_t)(ms * 1e6);
			e->stats.encode_kernel_launches++;
		}
		e->pend_tail++;
	}
}

// One slice (<= META_CAP chunks) of a put.  ticket == nullptr: returns when the chunks are stored.
// ticket != nullptr (host pages only): returns as soon as the caller's arrays have crossed to the
// device; the encode of the last sub-batch (and the copy of lens_out, which must then be
// page-locked and stay valid) completes behind the ticket.
// device-resident exchange records of a step; keep_pages: the caller keeps the host pages untouched
// until the ticket is done, so the call need not wait for its own copies
struct StepRecords { uint32_t rank; unsigned long long *out; bool keep_pages; };

static int put_slice(cmb200_engine *e, size_t n, const cmb200_addr *addr, const uint8_t *valid,
    const uint8_t *pages, bool pages_on_dev, const uint64_t *ts, int32_t *lens_out, uint64_t *ticket,
    const StepRecords *recs = nullptr) {
	const size_t B = pages_on_dev ? e->max_batch : e->host_batch;
	const bool deferred = ticket != nullptr;
	const bool copy_meta = !pages_on_dev || deferred;      // small arrays travel on the copy stream
	const unsigned long long seq_first = e->seq;
	// stage the small arrays in page-locked memory once; every copy below is then truly async
	cmb200_addr *h_addr = (cmb200_addr *)e->h_meta.get();
	uint64_t *h_ts = (uint64_t *)(e->h_meta + cmb200_engine::META_CAP * 16);
	int32_t *h_lens = (int32_t *)(e->h_meta + cmb200_engine::META_CAP * 24);
	uint8_t *h_valid = e->h_meta + cmb200_engine::META_CAP * 32;
	harvest_pending(e, !deferred);
	memcpy(h_addr, addr, n * 16);
	if (ts) memcpy(h_ts, ts, n * 8);
	if (valid) memcpy(h_valid, valid, n);
	// The small arrays go over once, before the page pipeline starts: a small copy issued between
	// two page copies would queue behind the next 256 MiB transfer in the copy engine and stall
	// the kernels that wait for it.  For host pages they travel on the copy stream into the copy of
	// the arrays that the previous call is not using: on the compute stream they would wait for
	// the previous call's last encode, and the page copies issued after them would wait with them
	// in the copy engine's queue.
	const int mb = copy_meta ? (int)(e->meta_pos++ & 1) : 0;
	unsigned long long *d_addr = e->d_addr + (size_t)mb * e->meta_cap * 2;
	unsigned long long *d_ts = e->d_ts + (size_t)mb * e->meta_cap;
	uint8_t *d_valid = e->d_valid + (size_t)mb * e->meta_cap;
	cudaStream_t ms = copy_meta ? e->copy : e->st;
	if (copy_meta) CMB_CHECK(cudaStreamWaitEvent(e->copy, e->meta_free[mb], 0));
	CMB_CHECK(cudaMemcpyAsync(d_addr, h_addr, n * 16, cudaMemcpyHostToDevice, ms));
	if (valid) CMB_CHECK(cudaMemcpyAsync(d_valid, h_valid, n, cudaMemcpyHostToDevice, ms));
	if (ts) CMB_CHECK(cudaMemcpyAsync(d_ts, h_ts, n * 8, cudaMemcpyHostToDevice, ms));
	if (copy_meta) {
		CMB_CHECK(cudaEventRecord(e->meta_done, e->copy));
		CMB_CHECK(cudaStreamWaitEvent(e->st, e->meta_done, 0));
	}
	size_t nb = 0;
	int last_buf = 0;
	for (size_t at = 0; at < n; at += B, nb++) {
		// (splitting the last step into smaller ones to shorten the un-overlapped tail was tried:
		// launches below ~4096 chunks run below PCIe rate, so the tail got longer, not shorter)
		const uint32_t m = (uint32_t)((n - at < B) ? n - at : B);
		const int buf = (int)(e->ring_pos & 1);
		const uint8_t *d_in;
		if (pages_on_dev) {
			d_in = pages + at * e->bsize;
		} else {
			// land the pages in ring buffer `buf` once the kernels that last read it are done
			e->ring_pos++;
			last_buf = buf;
			CMB_CHECK(cudaStreamWaitEvent(e->copy, e->consumed[buf], 0));
			CMB_CHECK(cudaMemcpyAsync(e->d_pages[buf], pages + at * e->bsize, (size_t)m * e->bsize,
			    cudaMemcpyHostToDevice, e->copy));
			CMB_CHECK(cudaEventRecord(e->landed[buf], e->copy));
			CMB_CHECK(cudaStreamWaitEvent(e->st, e->landed[buf], 0));
			d_in = e->d_pages[buf];
		}
		if (launch_upsert(e->table, d_addr + 2 * at, valid ? d_valid + at : nullptr, m, e->seq, e->seq_stride, e->d_slot, e->st)) return -1;
		EncodeJob job{};
		job.pages = d_in; job.page_stride = e->bsize; job.nbytes = e->bsize; job.n = m;
		job.accel = (uint32_t)e->accel;
		job.stage = e->d_stage; job.stage_stride = e->stage_stride;
		job.lens = e->d_lens + at;
		job.rec_out = e->d_recoff_out + at;
		job.fps = (e->flags & CMB200_FINGERPRINT) ? (uint64_t *)e->d_fps : nullptr;
		job.work = e->d_work;
		job.order = e->d_order;
		job.slot_idx = e->d_slot;
		job.addr = d_addr + 2 * at;
		job.ts = ts ? d_ts + at : nullptr;
		job.seq0 = e->seq; job.seq_stride = e->seq_stride;
		job.table = e->table; job.arena = e->arena;
		cudaEvent_t ev0, ev1;
		if (deferred) {
			if (e->pend_head - e->pend_tail >= (uint64_t)cmb200_engine::RING) harvest_pending(e, true);
			ev0 = e->p0[e->pend_head % cmb200_engine::RING]; ev1 = e->p1[e->pend_head % cmb200_engine::RING];
			e->pend_head++;
		} else {
			ev0 = e->t0[nb % e->RING]; ev1 = e->t1[nb % e->RING];
		}
		CMB_CHECK(cudaEventRecord(ev0, e->st));
		const int encode_kernels = launch_encode(job, e->st);
		if (encode_kernels < 0) return -1;
		CMB_CHECK(cudaEventRecord(ev1, e->st));
		if (!pages_on_dev) CMB_CHECK(cudaEventRecord(e->consumed[buf], e->st));
		e->seq += (unsigned long long)m * e->seq_stride;
		e->stats.kernel_launches += 1 + encode_kernels;
	}
	e->stats.put_chunks += n;
	if (recs && recs->out) {
		if (launch_pack_records(d_addr, e->d_lens, e->d_recoff_out, (uint32_t)n, seq_first, e->seq_stride, recs->rank, recs->out, e->st)) return -1;
		e->stats.kernel_launches++;
	}
	if (copy_meta) CMB_CHECK(cudaEventRecord(e->meta_free[mb], e->st));
	if (deferred) {
		if (lens_out) CMB_CHECK(cudaMemcpyAsync(lens_out, e->d_lens, n * 4, cudaMemcpyDeviceToHost, e->st));
		CMB_CHECK(cudaEventRecord(e->ticket_ev[e->tickets % cmb200_engine::TICKETS], e->st));
		*ticket = ++e->tickets;
		// the caller may reuse addr / valid / ts / pages once they have crossed
		CMB_CHECK(cudaEventSynchronize(e->meta_done));
		if (nb && !pages_on_dev && !(recs && recs->keep_pages)) CMB_CHECK(cudaEventSynchronize(e->landed[last_buf]));
		harvest_pending(e, false);
		return 0;
	}
	if (lens_out) CMB_CHECK(cudaMemcpyAsync(h_lens, e->d_lens, n * 4, cudaMemcpyDeviceToHost, e->st));
	CMB_CHECK(cudaStreamSynchronize(e->st));
	if (lens_out) memcpy(lens_out, h_lens, n * 4);
	for (size_t k = 0; k < nb && k < (size_t)e->RING; k++) {
		float ms = 0;
		CMB_CHECK(cudaEventElapsedTime(&ms, e->t0[k], e->t1[k]));
		e->stats.encode_kernel_ns += (uint64_t)(ms * 1e6);
		e->stats.encode_kernel_launches++;
	}
	return 0;
}

// The encoder reads device pages with 16-byte loads (TMA ring, fingerprint stripes): a device page
// pointer is checked before anything is queued.  Page strides (1 << pshift, pshift >= 6) are multiples of 64.
static int check_dev_pages(const void *pages, const char *what) {
	if (reinterpret_cast<uintptr_t>(pages) & 15u) {
		snprintf(g_err, sizeof(g_err), "%s: device pages must be 16-byte aligned", what);
		return -1;
	}
	return 0;
}

// The multi-GPU calls and the host tier exclude each other: the exchange records and peer reads know
// arena locations only.
static int multi_gpu_call(cmb200_engine *e, const char *what) {
	if (e->tier.host) {
		snprintf(g_err, sizeof(g_err), "%s: not available on an engine with a host tier", what);
		return -1;
	}
	e->multi_gpu = true;
	return 0;
}

static int put_impl(cmb200_engine *e, size_t n, const cmb200_addr *addr, const uint8_t *valid,
    const uint8_t *pages, bool pages_on_dev, const uint64_t *ts, int32_t *lens_out, uint64_t *ticket) {
	std::lock_guard<std::mutex> g(e->mu);
	CMB_CHECK(cudaSetDevice(e->device));
	if (ticket) *ticket = e->tickets;       // nothing to wait for unless the last slice is deferred
	for (size_t at = 0; at < n; at += cmb200_engine::META_CAP) {
		size_t m = n - at < cmb200_engine::META_CAP ? n - at : cmb200_engine::META_CAP;
		const bool last = at + m == n;
		if (put_slice(e, m, addr + at, valid ? valid + at : nullptr, pages + at * e->bsize, pages_on_dev,
			ts ? ts + at : nullptr, lens_out ? lens_out + at : nullptr, last ? ticket : nullptr)) return -1;
	}
	return 0;
}

extern "C" int cmb200_put_batch(cmb200_engine *e, size_t n, const cmb200_addr *addr, const uint8_t *valid,
    const void *pages_host, const uint64_t *ts, int32_t *lens_out) {
	return put_impl(e, n, addr, valid, (const uint8_t *)pages_host, false, ts, lens_out, nullptr);
}
extern "C" int cmb200_put_batch_async(cmb200_engine *e, size_t n, const cmb200_addr *addr, const uint8_t *valid,
    const void *pages_host, const uint64_t *ts, int32_t *lens_out, uint64_t *ticket) {
	uint64_t t = 0;
	const int rc = put_impl(e, n, addr, valid, (const uint8_t *)pages_host, false, ts, lens_out, &t);
	if (ticket) *ticket = t;
	return rc;
}
extern "C" int cmb200_put_step(cmb200_engine *e, size_t n, const cmb200_addr *addr, const uint8_t *valid,
    const void *pages, int pages_on_dev, const uint64_t *ts, uint32_t rank, void *records_dev_out,
    int32_t *lens_out, uint64_t *ticket) {
	if (multi_gpu_call(e, "cmb200_put_step")) return -1;
	if (n > cmb200_engine::META_CAP) { set_error_msg("cmb200_put_step: more than 262144 chunks in one step"); return -1; }
	if (pages_on_dev == 1 && check_dev_pages(pages, "cmb200_put_step")) return -1;
	std::lock_guard<std::mutex> g(e->mu);
	CMB_CHECK(cudaSetDevice(e->device));
	uint64_t t = e->tickets;
	StepRecords r{rank, (unsigned long long *)records_dev_out, pages_on_dev == 2};
	const int rc = n ? put_slice(e, n, addr, valid, (const uint8_t *)pages, pages_on_dev == 1, ts, lens_out, &t, &r) : 0;
	if (ticket) *ticket = t;
	return rc;
}

extern "C" int cmb200_import_records_dev(cmb200_engine *e, size_t n_total, const void *records_dev, uint32_t my_rank) {
	std::lock_guard<std::mutex> g(e->mu);
	if (multi_gpu_call(e, "cmb200_import_records_dev")) return -1;
	CMB_CHECK(cudaSetDevice(e->device));
	if (n_total == 0) return 0;
	if (n_total > 0xffffffffull) { set_error_msg("cmb200_import_records_dev: too many records"); return -1; }
	// the whole gathered buffer in one claim + one apply launch (the slot scratch grows on demand)
	if (e->d_import_slot.grow(n_total * sizeof(uint32_t), e->st)) return -1;
	if (launch_import_records(e->table, e->arena, (const unsigned long long *)records_dev, (uint32_t)n_total, my_rank,
		e->d_import_slot, e->st)) return -1;
	e->stats.kernel_launches += 2;
	return 0;                                               // asynchronous: ordered on the engine's stream
}

extern "C" int cmb200_wait(cmb200_engine *e, uint64_t ticket) {
	cudaEvent_t ev = nullptr;
	{
		std::lock_guard<std::mutex> g(e->mu);
		if (ticket == 0 || ticket > e->tickets) return 0;
		// a ticket whose event has been recorded again waits for the later put: the stream is in order
		ev = e->ticket_ev[(ticket - 1) % cmb200_engine::TICKETS];
		if (cudaSetDevice(e->device) != cudaSuccess) return -1;
	}
	CMB_CHECK(cudaEventSynchronize(ev));
	return 0;
}
extern "C" int cmb200_put_batch_dev(cmb200_engine *e, size_t n, const cmb200_addr *addr, const uint8_t *valid,
    const void *pages_dev, const uint64_t *ts, int32_t *lens_out) {
	if (check_dev_pages(pages_dev, "cmb200_put_batch_dev")) return -1;
	return put_impl(e, n, addr, valid, (const uint8_t *)pages_dev, true, ts, lens_out, nullptr);
}

// ---- get ---------------------------------------------------------------------------------

static int get_slice(cmb200_engine *e, size_t n, const cmb200_addr *addr, const uint8_t *valid,
    uint8_t *pages_out, bool out_on_dev, int32_t *status_out) {
	const size_t B = out_on_dev ? e->max_batch : e->host_batch;
	cmb200_addr *h_addr = (cmb200_addr *)e->h_meta.get();
	int32_t *h_status = (int32_t *)(e->h_meta + cmb200_engine::META_CAP * 28);
	uint8_t *h_valid = e->h_meta + cmb200_engine::META_CAP * 32;
	memcpy(h_addr, addr, n * 16);
	if (valid) memcpy(h_valid, valid, n);
	CMB_CHECK(cudaMemcpyAsync(e->d_addr, h_addr, n * 16, cudaMemcpyHostToDevice, e->st));
	if (valid) CMB_CHECK(cudaMemcpyAsync(e->d_valid, h_valid, n, cudaMemcpyHostToDevice, e->st));
	size_t nb = 0;
	for (size_t at = 0; at < n; at += B, nb++) {
		const uint32_t m = (uint32_t)((n - at < B) ? n - at : B);
		const int buf = (int)(nb & 1);
		uint8_t *d_out = out_on_dev ? pages_out + at * e->bsize : e->d_pages[buf];
		if (!out_on_dev) CMB_CHECK(cudaStreamWaitEvent(e->st, e->consumed[buf], 0));   // D2H of buf finished
		if (launch_lookup(e->table, e->d_addr + 2 * at, valid ? e->d_valid + at : nullptr, m, e->d_status + at, e->d_recoff,
			e->d_vlen, nullptr, e->st, e->d_vidx)) return -1;
		DecodeJob job{};
		job.n = m; job.nbytes = e->bsize; job.pages = d_out; job.status = e->d_status + at;
		job.rec_off = e->d_recoff; job.vlen = e->d_vlen; job.arena = e->arena.base;
		job.host = e->tier.dev; job.host_hits = e->tier.d_ctr + 1;
		job.hot = e->tier.hot(); job.addr = e->d_addr + 2 * at;
		const DecodeVerify ver{e->d_vidx, e->table.fp, e->table.fp_tag, e->d_vstat};
		const DecodeTouch touch{e->d_vidx, e->table.slots, (e->flags & CMB200_TOUCH) ? touch_stamp() : 0ull};
		CMB_CHECK(cudaEventRecord(e->t0[nb % e->RING], e->st));
		if (launch_decode(job, e->st, e->table.fp_tag ? &ver : nullptr, touch.ts ? &touch : nullptr)) return -1;
		CMB_CHECK(cudaEventRecord(e->t1[nb % e->RING], e->st));
		if (!out_on_dev) {
			CMB_CHECK(cudaEventRecord(e->landed[buf], e->st));
			CMB_CHECK(cudaStreamWaitEvent(e->copy, e->landed[buf], 0));
			CMB_CHECK(cudaMemcpyAsync(pages_out + at * e->bsize, d_out, (size_t)m * e->bsize,
			    cudaMemcpyDeviceToHost, e->copy));
			CMB_CHECK(cudaEventRecord(e->consumed[buf], e->copy));
		}
		e->stats.kernel_launches += 2;
	}
	CMB_CHECK(cudaMemcpyAsync(h_status, e->d_status, n * 4, cudaMemcpyDeviceToHost, e->st));
	CMB_CHECK(cudaStreamSynchronize(e->st));
	CMB_CHECK(cudaStreamSynchronize(e->copy));
	memcpy(status_out, h_status, n * 4);
	for (size_t k = 0; k < nb && k < (size_t)e->RING; k++) {
		float ms = 0;
		CMB_CHECK(cudaEventElapsedTime(&ms, e->t0[k], e->t1[k]));
		e->stats.decode_kernel_ns += (uint64_t)(ms * 1e6);
		e->stats.decode_kernel_launches++;
	}
	for (size_t i = 0; i < n; i++) {
		if (status_out[i] != CMB200_INVALID) e->stats.get_requests++;
		if (status_out[i] == CMB200_HIT) e->stats.get_hits++;
	}
	return 0;
}

static int get_impl(cmb200_engine *e, size_t n, const cmb200_addr *addr, const uint8_t *valid,
    uint8_t *pages_out, bool out_on_dev, int32_t *status_out) {
	std::lock_guard<std::mutex> g(e->mu);
	CMB_CHECK(cudaSetDevice(e->device));
	for (size_t at = 0; at < n; at += cmb200_engine::META_CAP) {
		size_t m = n - at < cmb200_engine::META_CAP ? n - at : cmb200_engine::META_CAP;
		if (get_slice(e, m, addr + at, valid ? valid + at : nullptr, pages_out + at * e->bsize, out_on_dev,
			status_out + at)) return -1;
	}
	return 0;
}

extern "C" int cmb200_get_batch(cmb200_engine *e, size_t n, const cmb200_addr *addr, const uint8_t *valid,
    void *pages_out_host, int32_t *status_out) {
	return get_impl(e, n, addr, valid, (uint8_t *)pages_out_host, false, status_out);
}
// Looks up m <= max_batch host addresses and brings each one's status, location and vlen (stored
// length + 1; nullable) to the host.  For ST_REMOTE the location is the owner rank (k_lookup).  The
// callers count the launch.  (e->mu held)
static int lookup_chunk(cmb200_engine *e, const cmb200_addr *addr, uint32_t m, int32_t *status, uint64_t *loc,
    uint32_t *vlen) {
	CMB_CHECK(cudaMemcpyAsync(e->d_addr, addr, (size_t)m * 16, cudaMemcpyHostToDevice, e->st));
	if (launch_lookup(e->table, e->d_addr, nullptr, m, e->d_status, e->d_recoff, e->d_vlen, nullptr, e->st)) return -1;
	CMB_CHECK(cudaMemcpyAsync(status, e->d_status, (size_t)m * 4, cudaMemcpyDeviceToHost, e->st));
	CMB_CHECK(cudaMemcpyAsync(loc, e->d_recoff, (size_t)m * 8, cudaMemcpyDeviceToHost, e->st));
	if (vlen) CMB_CHECK(cudaMemcpyAsync(vlen, e->d_vlen, (size_t)m * 4, cudaMemcpyDeviceToHost, e->st));
	CMB_CHECK(cudaStreamSynchronize(e->st));
	return 0;
}

extern "C" int cmb200_locate_batch(cmb200_engine *e, size_t n, const cmb200_addr *addr, int32_t *status_out,
    uint64_t *owner_out) {
	// lookup only: which requests hit here, miss, or live on another rank (owner_out = rank)
	std::lock_guard<std::mutex> g(e->mu);
	CMB_CHECK(cudaSetDevice(e->device));
	for (size_t at = 0; at < n; at += e->max_batch) {
		uint32_t m = (uint32_t)((n - at < e->max_batch) ? n - at : e->max_batch);
		if (lookup_chunk(e, addr + at, m, status_out + at, owner_out + at, nullptr)) return -1;
		e->stats.kernel_launches++;
	}
	return 0;
}
extern "C" int cmb200_get_batch_dev(cmb200_engine *e, size_t n, const cmb200_addr *addr, const uint8_t *valid,
    void *pages_out_dev, int32_t *status_out) {
	return get_impl(e, n, addr, valid, (uint8_t *)pages_out_dev, true, status_out);
}

// ---- multi-GPU index replication -------------------------------------------------------------

extern "C" int cmb200_set_stream_order(cmb200_engine *e, uint64_t next_seq, uint64_t stride) {
	std::lock_guard<std::mutex> g(e->mu);
	if (multi_gpu_call(e, "cmb200_set_stream_order")) return -1;
	if (stride == 0) { set_error_msg("stream order: stride must be >= 1"); return -1; }
	e->seq = next_seq; e->seq_stride = stride;
	return 0;
}

// ---- small gets: one fused kernel on their own stream ------------------------------------------

// Begin / end halves of a small get.  begin launches the kernel on a free lane and returns at once;
// the answers appear in t->status (page-locked host memory the kernel writes: a page, a system-wide
// fence, then its status word), so every requester of a combined batch can watch ITS word and leave
// as soon as its own page is there — a batch costs each caller its own page's decode, not the
// slowest one's.  end waits for whatever is still pending, books the statistics and frees the lane;
// it may run on another thread than begin.
static const int32_t SMALL_PENDING = -1;

extern "C" int cmb200_get_small_begin(cmb200_engine *e, size_t n, const cmb200_addr *addr, void *pages_out, cmb200_small_ticket *t) {
	if (!t) return -1;
	t->lane = -1; t->n = 0; t->status = nullptr;
	if (n == 0) return 0;
	if (n > cmb200_engine::GET_SMALL_MAX) { set_error_msg("cmb200_get_small_begin: more than 1024 requests"); return -1; }
	if (!get_small_supports(e->bsize)) { set_error_msg("cmb200_get_small: page size not supported by the fused kernel"); return -2; }
	e->get_gate.enter();
	// a free lane if there is one, else wait for one
	cmb200_engine::GetLane *ln = nullptr;
	int li = -1;
	const uint32_t first = e->lane_turn.fetch_add(1, std::memory_order_relaxed);
	for (uint64_t spins = 0; !ln; spins++) {
		for (int k = 0; k < cmb200_engine::GET_LANES && !ln; k++) {
			const int c = (int)((first + k) % cmb200_engine::GET_LANES);
			int idle = 0;
			if (e->lane[c].busy.compare_exchange_strong(idle, 1, std::memory_order_acq_rel)) { ln = &e->lane[c]; li = c; }
		}
		if (!ln) sched_yield();
	}
	if (cudaSetDevice(e->device) != cudaSuccess) { ln->busy.store(0, std::memory_order_release); e->get_gate.leave(); return -1; }
	// Requests and answers travel through page-locked host memory that the kernel reads and writes
	// directly: no copy is queued before or after the launch, and the end is seen by watching the
	// status words flip, which costs a few microseconds where a stream synchronisation costs tens.
	memcpy(ln->h_addr, addr, n * 16);
	volatile int32_t *hs = ln->h_status;
	for (size_t i = 0; i < n; i++) hs[i] = SMALL_PENDING;
	GetJob job{};
	job.table = e->table; job.arena = e->arena.base; job.arena_size = e->arena.size;
	job.host = e->tier.dev; job.host_size = e->tier.size; job.host_hits = e->tier.d_ctr + 1;
	job.addr = (const unsigned long long *)ln->h_addr.get(); job.valid = nullptr; job.n = (uint32_t)n; job.nbytes = e->bsize;
	job.out = (uint8_t *)pages_out;                          // device memory or page-locked host memory (UVA)
	job.status = ln->h_status;
	for (int r = 0; r < GET_MAX_PEERS; r++) { job.peer[r] = e->peer_base[r]; job.peer_size[r] = e->peer_size[r]; }
	job.scratch = e->d_scratch; job.region_entries = e->region_entries; job.pool_bits = e->d_pool_bits; job.pool_n = e->pool_n;
	job.hot = e->tier.hot();
	job.vstat = e->d_vstat;
	job.touch_ts = (e->flags & CMB200_TOUCH) ? touch_stamp() : 0ull;
	if (launch_get_small(job, e->device, ln->st)) { ln->busy.store(0, std::memory_order_release); e->get_gate.leave(); return -1; }
	t->lane = li; t->n = (uint32_t)n; t->status = ln->h_status;
	return 0;
}

extern "C" int cmb200_get_small_end(cmb200_engine *e, cmb200_small_ticket *t, int32_t *status_out) {
	if (!t || t->lane < 0) return 0;
	cmb200_engine::GetLane *ln = &e->lane[t->lane];
	volatile int32_t *hs = ln->h_status;
	int rc = 0;
	uint32_t done = 0;
	for (uint64_t spins = 0; done < t->n;) {
		if (hs[done] != SMALL_PENDING) { done++; continue; }
#if defined(__x86_64__)
		__builtin_ia32_pause();
#endif
		if (++spins > 20000) {                                // ~1 ms of polling: a large batch, let the driver wait
			if (cudaSetDevice(e->device) != cudaSuccess || cudaStreamSynchronize(ln->st) != cudaSuccess) {
				cmb_set_error("cudaStreamSynchronize(small get)", cudaGetLastError(), __FILE__, __LINE__);
				rc = -1; break;
			}
			spins = 0;
			if (hs[done] == SMALL_PENDING) { set_error_msg("cmb200_get_small: kernel finished without an answer"); rc = -1; break; }
		}
	}
	__atomic_thread_fence(__ATOMIC_ACQUIRE);
	if (rc == 0) {
		uint64_t rq = 0, ht = 0;
		for (uint32_t i = 0; i < t->n; i++) {
			const int32_t st = hs[i];
			if (status_out) status_out[i] = st;
			if (st != CMB200_INVALID) rq++;
			if (st == CMB200_HIT) ht++;
		}
		e->small_get_launches++;
		e->small_get_requests += rq; e->small_get_hits += ht;
	}
	t->lane = -1;
	ln->busy.store(0, std::memory_order_release);
	e->get_gate.leave();
	return rc;
}

extern "C" int cmb200_get_small(cmb200_engine *e, size_t n, const cmb200_addr *addr, void *pages_out, int32_t *status_out) {
	for (size_t at = 0; at < n; at += cmb200_engine::GET_SMALL_MAX) {
		const size_t m = n - at < cmb200_engine::GET_SMALL_MAX ? n - at : cmb200_engine::GET_SMALL_MAX;
		cmb200_small_ticket t;
		const int rc = cmb200_get_small_begin(e, m, addr + at, (uint8_t *)pages_out + at * e->bsize, &t);
		if (rc) return rc;
		if (cmb200_get_small_end(e, &t, status_out + at)) return -1;
	}
	return 0;
}

// ---- peers: the other ranks' arenas, mapped for NVLink reads -------------------------------------

extern "C" int cmb200_close_peers(cmb200_engine *e) {
	cmb200_engine::GateClosed g(e->get_gate);             // no small get in flight
	CMB_CHECK(cudaSetDevice(e->device));
	for (int r = 0; r < GET_MAX_PEERS; r++) {
		if (e->peer_base[r]) cudaIpcCloseMemHandle((void *)e->peer_base[r]);
		e->peer_base[r] = nullptr; e->peer_size[r] = 0;
	}
	return 0;
}

extern "C" int cmb200_arena_ipc_handle(cmb200_engine *e, void *handle64, uint64_t *arena_bytes_out) {
	{
		std::lock_guard<std::mutex> g(e->mu);
		if (multi_gpu_call(e, "cmb200_arena_ipc_handle")) return -1;
	}
	CMB_CHECK(cudaSetDevice(e->device));
	cudaIpcMemHandle_t h;
	static_assert(sizeof(h) == 64, "cudaIpcMemHandle_t is 64 bytes");
	CMB_CHECK(cudaIpcGetMemHandle(&h, e->arena.base));
	memcpy(handle64, &h, 64);
	if (arena_bytes_out) *arena_bytes_out = e->arena.size;
	return 0;
}

extern "C" int cmb200_open_peer(cmb200_engine *e, uint32_t rank, const void *handle64, uint64_t arena_bytes) {
	{
		std::lock_guard<std::mutex> g(e->mu);
		if (multi_gpu_call(e, "cmb200_open_peer")) return -1;
	}
	if (rank >= GET_MAX_PEERS) { set_error_msg("cmb200_open_peer: rank out of range"); return -1; }
	cmb200_engine::GateClosed g(e->get_gate);
	CMB_CHECK(cudaSetDevice(e->device));
	cudaIpcMemHandle_t h;
	memcpy(&h, handle64, 64);
	void *p = nullptr;
	CMB_CHECK(cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess));
	if (e->peer_base[rank]) cudaIpcCloseMemHandle((void *)e->peer_base[rank]);
	e->peer_base[rank] = (const uint8_t *)p;
	e->peer_size[rank] = arena_bytes;
	return 0;
}

// ---- unset / entries / sample / records ----------------------------------------------------

extern "C" int cmb200_unset_batch(cmb200_engine *e, size_t n, const cmb200_addr *addr) {
	std::lock_guard<std::mutex> g(e->mu);
	CMB_CHECK(cudaSetDevice(e->device));
	for (size_t at = 0; at < n; at += e->max_batch) {
		uint32_t m = (uint32_t)((n - at < e->max_batch) ? n - at : e->max_batch);
		CMB_CHECK(cudaMemcpyAsync(e->d_addr, addr + at, (size_t)m * 16, cudaMemcpyHostToDevice, e->st));
		if (launch_unset(e->table, e->arena, e->d_addr, m, e->st)) return -1;
		e->stats.kernel_launches++;
	}
	CMB_CHECK(cudaStreamSynchronize(e->st));
	return 0;
}

static int read_counters(cmb200_engine *e, unsigned long long out[8]) {
	CMB_CHECK(cudaSetDevice(e->device));
	CMB_CHECK(cudaMemcpyAsync(out, e->d_counters, 8 * sizeof(unsigned long long), cudaMemcpyDeviceToHost, e->st));
	CMB_CHECK(cudaStreamSynchronize(e->st));
	return 0;
}

extern "C" uint64_t cmb200_entries(cmb200_engine *e) {
	std::lock_guard<std::mutex> g(e->mu);
	unsigned long long c[8];
	if (read_counters(e, c)) return 0;
	return c[0];
}

extern "C" int cmb200_get_stats(cmb200_engine *e, cmb200_stats *out) {
	std::lock_guard<std::mutex> g(e->mu);
	unsigned long long c[8];
	if (read_counters(e, c)) return -1;
	harvest_pending(e, true);
	*out = e->stats;
	out->get_requests += e->small_get_requests.load(); out->get_hits += e->small_get_hits.load();
	out->kernel_launches += e->small_get_launches.load();
	out->entries = c[0]; out->tombstones = c[1];
	out->arena_used = c[2] < e->arena.size ? c[2] : e->arena.size;   // the bump pointer saturates past the end (no rollback)
	out->arena_garbage = c[3];
	out->dropped_puts = c[4]; out->remote_entries = c[5];
	out->table_slots = e->table.cap; out->arena_bytes = e->arena.size;
	return 0;
}

extern "C" int cmb200_sample(cmb200_engine *e, size_t n, const uint64_t *r, cmb200_addr *addr_out,
    uint64_t *ts_out, int32_t *ok_out) {
	std::lock_guard<std::mutex> g(e->mu);
	CMB_CHECK(cudaSetDevice(e->device));
	for (size_t at = 0; at < n; at += e->max_batch) {
		const uint32_t m = (uint32_t)((n - at < e->max_batch) ? n - at : e->max_batch);
		CMB_CHECK(cudaMemcpyAsync(e->d_recoff, r + at, (size_t)m * 8, cudaMemcpyHostToDevice, e->st));
		if (launch_sample(e->table, (const unsigned long long *)e->d_recoff.get(), m, e->d_addr, e->d_ts, e->d_status, e->st)) return -1;
		CMB_CHECK(cudaMemcpyAsync(addr_out + at, e->d_addr, (size_t)m * 16, cudaMemcpyDeviceToHost, e->st));
		CMB_CHECK(cudaMemcpyAsync(ts_out + at, e->d_ts, (size_t)m * 8, cudaMemcpyDeviceToHost, e->st));
		CMB_CHECK(cudaMemcpyAsync(ok_out + at, e->d_status, (size_t)m * 4, cudaMemcpyDeviceToHost, e->st));
		CMB_CHECK(cudaStreamSynchronize(e->st));
		e->stats.kernel_launches++;
	}
	return 0;
}

extern "C" int cmb200_read_records(cmb200_engine *e, size_t n, const cmb200_addr *addr, void *out_host,
    size_t stride, int32_t *len_out) {
	std::lock_guard<std::mutex> g(e->mu);
	CMB_CHECK(cudaSetDevice(e->device));
	std::vector<int32_t> st(e->max_batch);
	std::vector<uint64_t> off(e->max_batch);
	std::vector<uint32_t> vl(e->max_batch);
	for (size_t at = 0; at < n; at += e->max_batch) {
		uint32_t m = (uint32_t)((n - at < e->max_batch) ? n - at : e->max_batch);
		if (lookup_chunk(e, addr + at, m, st.data(), off.data(), vl.data())) return -1;
		for (uint32_t i = 0; i < m; i++) {
			if (st[i] != ST_HIT) { len_out[at + i] = -1; continue; }
			uint32_t clen = vl[i] - 1;
			size_t total = 24 + (clen ? clen : e->bsize);
			if (total > stride) { set_error_msg("cmb200_read_records: stride too small"); return -1; }
			if (off[i] & REC_HOST) memcpy((uint8_t *)out_host + (at + i) * stride, e->tier.host + (off[i] & ~REC_HOST), total);
			else CMB_CHECK(cudaMemcpyAsync((uint8_t *)out_host + (at + i) * stride, e->arena.base + off[i], total,
			    cudaMemcpyDeviceToHost, e->st));
			len_out[at + i] = (int32_t)total;
		}
		CMB_CHECK(cudaStreamSynchronize(e->st));
	}
	return 0;
}

extern "C" int cmb200_read_fingerprints(cmb200_engine *e, size_t n, const cmb200_addr *addr, uint64_t *fp_out,
    int32_t *ok_out) {
	std::lock_guard<std::mutex> g(e->mu);
	CMB_CHECK(cudaSetDevice(e->device));
	if (!e->table.fp) { set_error_msg("engine created without CMB200_FINGERPRINT"); return -1; }
	for (size_t at = 0; at < n; at += e->max_batch) {
		uint32_t m = (uint32_t)((n - at < e->max_batch) ? n - at : e->max_batch);
		CMB_CHECK(cudaMemcpyAsync(e->d_addr, addr + at, (size_t)m * 16, cudaMemcpyHostToDevice, e->st));
		if (launch_read_fp(e->table, e->d_addr, m, e->d_fps, e->d_status, e->st)) return -1;
		CMB_CHECK(cudaMemcpyAsync(fp_out + 2 * at, e->d_fps, (size_t)m * 16, cudaMemcpyDeviceToHost, e->st));
		CMB_CHECK(cudaMemcpyAsync(ok_out + at, e->d_status, (size_t)m * 4, cudaMemcpyDeviceToHost, e->st));
		CMB_CHECK(cudaStreamSynchronize(e->st));
	}
	return 0;
}

extern "C" int cmb200_read_checkpoints(cmb200_engine *e, size_t n, const cmb200_addr *addr, uint32_t *words_out,
    int32_t *ok_out) {
	std::lock_guard<std::mutex> g(e->mu);
	CMB_CHECK(cudaSetDevice(e->device));
	if (!e->table.ckpt) {                                // no side table: nothing has checkpoints
		memset(words_out, 0, n * CKPT_WORDS * 4);
		for (size_t i = 0; i < n; i++) ok_out[i] = -1;
		return 0;
	}
	DevMem<uint32_t> d_words;
	if (n && d_words.alloc((size_t)e->max_batch * CKPT_WORDS * 4 + 256)) return -1;
	for (size_t at = 0; at < n; at += e->max_batch) {
		uint32_t m = (uint32_t)((n - at < e->max_batch) ? n - at : e->max_batch);
		CMB_CHECK(cudaMemcpyAsync(e->d_addr, addr + at, (size_t)m * 16, cudaMemcpyHostToDevice, e->st));
		if (launch_read_ckpt(e->table, e->d_addr, m, d_words, e->d_status, e->st)) return -1;
		CMB_CHECK(cudaMemcpyAsync(words_out + at * CKPT_WORDS, d_words, (size_t)m * CKPT_WORDS * 4, cudaMemcpyDeviceToHost, e->st));
		CMB_CHECK(cudaMemcpyAsync(ok_out + at, e->d_status, (size_t)m * 4, cudaMemcpyDeviceToHost, e->st));
		CMB_CHECK(cudaStreamSynchronize(e->st));
	}
	return 0;
}

// Every live local record (arena_only: leave out the host tier's), sorted by offset, and the counters
// read just before the export.  (e->mu held)  0 = listed, -1 = a CUDA call failed (error set), 1 = more
// than c[0] + 16 records were found (the store changed since the counters were read): the list holds
// c[0] + 16 of them.  seq_min and addr_out as for launch_export_list; addr_out (device address, room for
// c[0] + 16) then gets every live local address and *n_addr their number.
static int live_records(cmb200_engine *e, bool arena_only, std::vector<ExportEntry> &list, unsigned long long c[8],
    unsigned long long seq_min = 0, ulonglong2 *addr_out = nullptr, uint64_t *n_addr = nullptr) {
	if (read_counters(e, c)) return -1;
	const unsigned long long cap_out = c[0] + 16;
	DevMem<ExportEntry> d_list;
	DevMem<unsigned long long> d_count;
	if (d_list.alloc(cap_out * sizeof(ExportEntry) + 256) || d_count.alloc(16 + 256)) return -1;
	CMB_CHECK(cudaMemsetAsync(d_count, 0, 16, e->st));
	if (launch_export_list(e->table, e->bsize, d_list, d_count, cap_out, arena_only, e->st, seq_min, addr_out)) return -1;
	unsigned long long counts[2] = {0, 0};
	CMB_CHECK(cudaMemcpyAsync(counts, d_count, 16, cudaMemcpyDeviceToHost, e->st));
	CMB_CHECK(cudaStreamSynchronize(e->st));
	unsigned long long count = counts[0];
	int over = count > cap_out || counts[1] > cap_out;
	if (count > cap_out) count = cap_out;
	if (n_addr) *n_addr = counts[1] < cap_out ? counts[1] : cap_out;
	list.resize(count);
	if (count) CMB_CHECK(cudaMemcpy(list.data(), d_list, count * sizeof(ExportEntry), cudaMemcpyDeviceToHost));
	std::sort(list.begin(), list.end(), [](const ExportEntry &a, const ExportEntry &b) { return a.rec_off < b.rec_off; });
	return over;
}

// ---- snapshot: persistence of the cache directory (SURVEY.md 8 f3) ---------------------------
//
// The reference's store is persistent because it IS a set of LMDB files under <cachedir>
// (filemap.c:57,71-72).  Here the store lives in HBM, so it is saved to / restored from one file of
// records, each exactly the LMDB value of the reference (24-byte data_prefix + payload,
// filemap.c:140-147) preceded by {ts (the LMDB attribute), length, fingerprint}:
//
//   header   "CMB200S1" | u32 version=1 | u32 pshift | u64 records | u64 payload bytes | u32 flags | pad to 64
//   record   u64 ts | u64 fp_hi | u64 fp_lo | u32 len | u32 0 | len bytes {u, l, compressed_length, pad, payload} | pad to 16
//
// It does not depend on the table geometry or the arena layout, so a snapshot loads into an engine
// of any capacity (records that do not fit are dropped like puts into a full store).
struct SnapHeader {
	char magic[8];
	uint32_t version, pshift;
	uint64_t records, bytes;
	uint32_t flags, pad[7];
};
static_assert(sizeof(SnapHeader) == 64, "snapshot header");
struct SnapRecord { uint64_t ts, fp_hi, fp_lo; uint32_t len, zero; };
static_assert(sizeof(SnapRecord) == 32, "snapshot record header");
static const size_t SNAP_WINDOW = 64u << 20;

// A snapshot lists each engine's live records under its lock and writes them from a thread of its own
// while the engines keep serving.  That is sound because records are immutable (DESIGN.md §2): only
// compaction (which slides records down) and a host-tier lap (which overwrites the tier's oldest
// records) reuse the bytes of a record, and both wait in snap_wait_written until the engine's section
// is written.  Every other writer of arena or tier bytes writes bytes no listed record occupies.

// Waits until no snapshot holds a list of e's records that it has not written yet.  (e->mu held; the
// writer never takes it, see cmb200_engine::snap_state)
static void snap_wait_written(cmb200_engine *e) {
	std::unique_lock<std::mutex> lk(e->snap_mu);
	e->snap_cv.wait(lk, [e] { return e->snap_state != cmb200_engine::SNAP_PENDING; });
}

static void snap_set_state(cmb200_engine *e, int state) {
	std::lock_guard<std::mutex> lk(e->snap_mu);
	e->snap_state = state;
	e->snap_cv.notify_all();
}

// Writes the listed records of e to f through the engine's page-locked window, copying arena windows on
// the writer's stream.  A window may also hold garbage or records put after the list was taken; only
// listed records are written, and their bytes do not change until the section is released.  (runs
// without e->mu)  0 = written, -1 = a CUDA call failed (error set), -2 = a write failed.
static int write_section(cmb200_engine *e, FILE *f, const std::vector<ExportEntry> &list) {
	uint8_t *win = e->snap_win;
	bool ok = true;
	static const uint8_t zeros[16] = {0};
	size_t k = 0;
	while (ok && k < list.size()) {
		if (list[k].rec_off & REC_HOST) {
			// host-tier records sort last and are written straight from the tier
			const ExportEntry &x = list[k++];
			SnapRecord r{x.ts, x.fp_hi, x.fp_lo, x.len, 0};
			const size_t padn = (16 - (x.len & 15)) & 15;
			ok = fwrite(&r, sizeof(r), 1, f) == 1 && fwrite(e->tier.host + (x.rec_off & ~REC_HOST), x.len, 1, f) == 1 &&
			    (padn == 0 || fwrite(zeros, padn, 1, f) == 1);
			continue;
		}
		// one window of the arena starting at record k; the records wholly inside it are written out
		const unsigned long long w0 = list[k].rec_off;
		unsigned long long w1 = w0 + SNAP_WINDOW;
		if (w1 > e->arena.size + 256) w1 = e->arena.size + 256;
		CMB_CHECK(cudaMemcpyAsync(win, e->arena.base + w0, (size_t)(w1 - w0), cudaMemcpyDeviceToHost, e->snap_st));
		CMB_CHECK(cudaStreamSynchronize(e->snap_st));
		for (; k < list.size() && list[k].rec_off + list[k].len <= w1; k++) {
			const ExportEntry &x = list[k];
			SnapRecord r{x.ts, x.fp_hi, x.fp_lo, x.len, 0};
			const size_t padn = (16 - (x.len & 15)) & 15;
			ok = ok && fwrite(&r, sizeof(r), 1, f) == 1 && fwrite(win + (x.rec_off - w0), x.len, 1, f) == 1 &&
			    (padn == 0 || fwrite(zeros, padn, 1, f) == 1);
		}
	}
	return ok ? 0 : -2;
}

// ---- snapshot chains (cmb200_chain_begin / cmb200_load_chain) ----
// A base is the file above with a nonzero 64-bit chain id in bytes 40..47 (pad[1..2], zero in a file
// written by cmb200_save_set).  Delta k of that chain, <base>.d<k>, holds what changed between tick k-1
// (tick 0 = the base) and tick k:
//
//   header      "CMB200D1" | u32 version=1 | u32 pshift | u64 chain id | u32 k | u32 flags |
//               u64 tombstones | u64 records | u64 record bytes | pad to 64
//   tombstones  16-byte addresses that were live at tick k-1 and are not at tick k
//   records     every live local record put since tick k-1, in the base's record format
//
// The store of a chain is the base, then for each delta in order its tombstones removed and its records
// put.  "Put since tick k-1" is Slot::seq >= the engine's seq at tick k-1: every put raises the slot's
// seq (k_upsert), a table rebuild copies it, and compaction, demotion and promotion leave it alone, so
// a record that only moved is not in the delta.
struct DeltaHeader {
	char magic[8];
	uint32_t version, pshift;
	uint64_t chain;
	uint32_t index, flags;
	uint64_t tombstones, records, bytes, pad;
};
static_assert(sizeof(DeltaHeader) == 64, "delta header");

static uint64_t snap_chain_id(const SnapHeader &h) {
	uint64_t id;
	memcpy(&id, &h.pad[1], 8);
	return id;
}

enum { CHAIN_NONE = 0, CHAIN_BASE, CHAIN_DELTA };

struct cmb200_snapshot {
	std::vector<cmb200_engine *> engines;                 // in file order
	std::vector<std::vector<ExportEntry>> lists;          // each engine's live records at begin, by offset
	std::string tmp;
	FILE *f = nullptr;
	SnapHeader h{};
	std::thread writer;
	int rc = 0;                                           // the writer's: 0, -1 CUDA, -2 file
	std::string err;                                      // the writer's error text (g_err is per thread)
	int chain = CHAIN_NONE;
	DeltaHeader dh{};                                     // CHAIN_DELTA: the header written instead of h
	std::vector<ulonglong2> tombs;                        // CHAIN_DELTA: every engine's tombstones
};

// The writer thread: header, then each engine's section; an engine is released as soon as its section
// is written (or the write has failed), so that its compactions and tier laps go ahead.
static void snapshot_write(cmb200_snapshot *s) {
	bool ok = s->chain == CHAIN_DELTA
	    ? fwrite(&s->dh, sizeof(s->dh), 1, s->f) == 1 &&
	      (s->tombs.empty() || fwrite(s->tombs.data(), 16, s->tombs.size(), s->f) == s->tombs.size())
	    : fwrite(&s->h, sizeof(s->h), 1, s->f) == 1;
	int rc = ok ? 0 : -2;
	for (size_t i = 0; i < s->engines.size(); i++) {
		cmb200_engine *e = s->engines[i];
		if (rc == 0) {
			if (cudaSetDevice(e->device) != cudaSuccess) { cmb_set_error("cudaSetDevice", cudaGetLastError(), __FILE__, __LINE__); rc = -1; }
			else rc = write_section(e, s->f, s->lists[i]);
		}
		std::vector<ExportEntry>().swap(s->lists[i]);
		snap_set_state(e, cmb200_engine::SNAP_FREE);
	}
	if (rc == 0 && fflush(s->f) != 0) rc = -2;
	if (fclose(s->f) != 0 && rc == 0) rc = -2;
	s->f = nullptr;
	if (rc == -2) set_error_msg("cmb200_save: write failed");
	if (rc) s->err = g_err;
	s->rc = rc;
}

// Makes room for c0 + 16 addresses in the half of e's baseline that the next tick writes.  (e->mu held)
static int chain_room(cmb200_engine *e, unsigned long long c0) {
	cmb200_engine::Chain &ch = e->chain;
	const int nx = ch.cur ^ 1;
	const uint64_t need = c0 + 16;
	if (ch.cap[nx] >= need) return 0;
	const uint64_t cap = need + need / 4 + 1024;
	ch.cap[nx] = 0; ch.base_dev[nx] = nullptr;
	if (ch.base[nx].alloc(cap * 16, true)) return -1;
	void *dev = nullptr;
	CMB_CHECK(cudaHostGetDevicePointer(&dev, (void *)ch.base[nx], 0));
	ch.base_dev[nx] = (ulonglong2 *)dev;
	ch.cap[nx] = cap;
	return 0;
}

// Lists engine i of a chain tick (e->mu held): the tombstones against the previous baseline (a delta),
// then the records put since the previous watermark (a delta) or all of them (a base), with the next
// baseline exported by the same pass.  The results wait in the *_next fields for cmb200_snapshot_finish.
static int chain_list(cmb200_engine *e, cmb200_snapshot *s, int i) {
	cmb200_engine::Chain &ch = e->chain;
	const bool delta = s->chain == CHAIN_DELTA;
	if (ch.pending) { set_error_msg("cmb200_chain_begin: a chain tick of this engine is not finished"); return -1; }
	if (delta && (ch.id != s->dh.chain || ch.k + 1 != s->dh.index)) {
		set_error_msg("cmb200_chain_begin: an engine holds no chain state for this base: write a base first");
		return -1;
	}
	unsigned long long c[8];
	if (read_counters(e, c) || chain_room(e, c[0])) return -1;
	if (delta && ch.n) {
		DevMem<ulonglong2> d_out;
		DevMem<unsigned long long> d_cnt;
		if (d_out.alloc(ch.n * 16 + 256) || d_cnt.alloc(8 + 256)) return -1;
		CMB_CHECK(cudaMemsetAsync(d_cnt, 0, 8, e->st));
		if (launch_delta_gone(e->table, ch.base_dev[ch.cur], ch.n, d_out, d_cnt, e->st)) return -1;
		unsigned long long nt = 0;
		CMB_CHECK(cudaMemcpyAsync(&nt, d_cnt, 8, cudaMemcpyDeviceToHost, e->st));
		CMB_CHECK(cudaStreamSynchronize(e->st));
		const size_t at = s->tombs.size();
		s->tombs.resize(at + nt);
		if (nt) CMB_CHECK(cudaMemcpy(s->tombs.data() + at, d_out, nt * 16, cudaMemcpyDeviceToHost));
	}
	uint64_t n_next = 0;
	if (live_records(e, false, s->lists[i], c, delta ? ch.w : 0, ch.base_dev[ch.cur ^ 1], &n_next) < 0) return -1;
	// the stream is synchronised and mu held: every record version put so far has seq < e->seq, every later one >=
	ch.w_next = e->seq; ch.n_next = n_next; ch.id_next = s->dh.chain; ch.k_next = s->dh.index;
	ch.pending = true;
	return 0;
}

static cmb200_snapshot *snapshot_start(cmb200_engine *const *engines, int g, const char *path, int chain,
    uint64_t chain_id, uint32_t k) {
	if (g < 1 || !engines || !path) { set_error_msg("cmb200_snapshot_begin: no engines"); return nullptr; }
	for (int i = 1; i < g; i++)
		if (engines[i]->pshift != engines[0]->pshift) { set_error_msg("cmb200_save_set: engines of different page sizes"); return nullptr; }
	// engines are claimed in address order, so that two snapshots of overlapping sets never each hold
	// an engine the other one waits for
	std::vector<cmb200_engine *> order(engines, engines + g);
	std::sort(order.begin(), order.end());
	if (std::adjacent_find(order.begin(), order.end()) != order.end()) { set_error_msg("cmb200_snapshot_begin: an engine is listed twice"); return nullptr; }
	cmb200_snapshot *s = new (std::nothrow) cmb200_snapshot();
	if (!s) { set_error_msg("cmb200_snapshot_begin: out of memory"); return nullptr; }
	s->engines.assign(engines, engines + g);
	s->lists.resize(g);
	s->tmp = std::string(path) + ".tmp";
	s->f = fopen(s->tmp.c_str(), "wb");
	if (!s->f) { set_error_msg("cmb200_save: cannot create the snapshot file"); delete s; return nullptr; }
	for (cmb200_engine *e : order) {
		std::unique_lock<std::mutex> lk(e->snap_mu);
		e->snap_cv.wait(lk, [e] { return e->snap_state == cmb200_engine::SNAP_FREE; });
		e->snap_state = cmb200_engine::SNAP_CLAIMED;
	}
	int rc = 0;
	for (cmb200_engine *e : order) {
		// allocated once: cudaFreeHost may synchronise the device
		if (cudaSetDevice(e->device) != cudaSuccess ||
		    (!e->snap_win && e->snap_win.alloc(SNAP_WINDOW)) || (!e->snap_st && e->snap_st.create())) {
			cmb_set_error("cmb200_snapshot_begin: no page-locked window or stream", cudaGetLastError(), __FILE__, __LINE__);
			rc = -1;
			break;
		}
	}
	s->h = SnapHeader{};
	memcpy(s->h.magic, "CMB200S1", 8);
	s->h.version = 1; s->h.pshift = (uint32_t)engines[0]->pshift;
	s->chain = chain;
	s->dh.chain = chain_id; s->dh.index = k;
	if (chain == CHAIN_BASE) memcpy(&s->h.pad[1], &chain_id, 8);
	int listed = 0;                                       // engines whose chain tick is pending
	for (int i = 0; i < g && rc == 0; i++) {
		cmb200_engine *e = engines[i];
		std::lock_guard<std::mutex> lk(e->mu);
		if (i == 0) s->h.flags = e->table.fp ? 1u : 0u;
		unsigned long long c[8];
		// live_records synchronises the stream first: every put enqueued before now is listed
		if (chain != CHAIN_NONE ? chain_list(e, s, i) : live_records(e, false, s->lists[i], c) < 0) { rc = -1; break; }
		listed++;
		snap_set_state(e, cmb200_engine::SNAP_PENDING);
		s->h.records += s->lists[i].size();
		for (const ExportEntry &x : s->lists[i]) s->h.bytes += x.len;
	}
	if (chain == CHAIN_DELTA) {
		memcpy(s->dh.magic, "CMB200D1", 8);
		s->dh.version = 1; s->dh.pshift = s->h.pshift; s->dh.flags = s->h.flags;
		s->dh.tombstones = s->tombs.size(); s->dh.records = s->h.records; s->dh.bytes = s->h.bytes;
	}
	if (rc == 0) {
		try {
			s->writer = std::thread(snapshot_write, s);
		} catch (...) {
			set_error_msg("cmb200_snapshot_begin: cannot start the writer thread");
			rc = -1;
		}
	}
	if (rc == 0) return s;
	for (cmb200_engine *e : order) snap_set_state(e, cmb200_engine::SNAP_FREE);
	for (int i = 0; i < listed && chain != CHAIN_NONE; i++) {
		std::lock_guard<std::mutex> lk(engines[i]->mu);
		engines[i]->chain.pending = false;
	}
	fclose(s->f);
	remove(s->tmp.c_str());
	delete s;
	return nullptr;
}

extern "C" cmb200_snapshot *cmb200_snapshot_begin(cmb200_engine *const *engines, int g, const char *path) {
	return snapshot_start(engines, g, path, CHAIN_NONE, 0, 0);
}

extern "C" cmb200_snapshot *cmb200_chain_begin(cmb200_engine *const *engines, int g, const char *base_path, int delta) {
	if (g < 1 || !engines || !base_path) { set_error_msg("cmb200_chain_begin: no engines"); return nullptr; }
	if (!delta) {
		// a fresh id: the deltas of any earlier chain next to this base stop matching it
		uint64_t id = 0;
		while (id == 0) {
			struct timespec ts;
			clock_gettime(CLOCK_REALTIME, &ts);
			static std::atomic<uint64_t> calls{0};
			const uint64_t seed[2] = {(uint64_t)ts.tv_sec * 1000000000ull + (uint64_t)ts.tv_nsec,
			    ((uint64_t)getpid() << 32) ^ (uint64_t)(uintptr_t)engines[0] ^ calls.fetch_add(1)};
			FNV_hash(seed, 16, &id);
		}
		return snapshot_start(engines, g, base_path, CHAIN_BASE, id, 0);
	}
	SnapHeader h{};
	FILE *f = fopen(base_path, "rb");
	const bool ok = f && fread(&h, sizeof(h), 1, f) == 1 && memcmp(h.magic, "CMB200S1", 8) == 0 && h.version == 1;
	if (f) fclose(f);
	if (!ok || snap_chain_id(h) == 0) { set_error_msg("cmb200_chain_begin: no chain base at this path"); return nullptr; }
	uint32_t k;
	{
		// checked against every engine under its lock when the tick lists it
		std::lock_guard<std::mutex> lk(engines[0]->mu);
		k = engines[0]->chain.k + 1;
	}
	const std::string path = std::string(base_path) + ".d" + std::to_string(k);
	return snapshot_start(engines, g, path.c_str(), CHAIN_DELTA, snap_chain_id(h), k);
}

extern "C" int cmb200_snapshot_finish(cmb200_snapshot *s, uint64_t *records_out) {
	if (!s) { set_error_msg("cmb200_snapshot_finish: no snapshot"); return -1; }
	s->writer.join();
	const std::string path = s->tmp.substr(0, s->tmp.size() - 4);
	int rc = 0;
	if (s->rc != 0) {
		set_error_msg(s->err.c_str());
		rc = -1;
	} else if (rename(s->tmp.c_str(), path.c_str()) != 0) {
		set_error_msg("cmb200_save: write failed");
		rc = -1;
	}
	if (rc) remove(s->tmp.c_str());
	else if (records_out) *records_out = s->h.records;
	// a chain tick becomes the engines' chain state only once its file is in place
	for (size_t i = 0; i < s->engines.size() && s->chain != CHAIN_NONE; i++) {
		cmb200_engine *e = s->engines[i];
		std::lock_guard<std::mutex> lk(e->mu);
		cmb200_engine::Chain &ch = e->chain;
		if (rc == 0) {
			ch.cur ^= 1; ch.n = ch.n_next; ch.w = ch.w_next; ch.id = ch.id_next; ch.k = ch.k_next;
		}
		ch.pending = false;
	}
	delete s;
	return rc;
}

extern "C" int cmb200_save_set(cmb200_engine *const *engines, int g, const char *path, uint64_t *records_out) {
	cmb200_snapshot *s = cmb200_snapshot_begin(engines, g, path);
	return s ? cmb200_snapshot_finish(s, records_out) : -1;
}

extern "C" int cmb200_save(cmb200_engine *e, const char *path, uint64_t *records_out) {
	return cmb200_save_set(&e, 1, path, records_out);
}

static int demote_arena_all(cmb200_engine *e);

// One engine's share of a load: its records are staged in page-locked memory until the batch is full
// (<= max_batch records and <= one page-ring buffer of bytes), then put in as one upsert + k_restore.
struct LoadBatch {
	cmb200_engine *e = nullptr;
	HostMem<uint8_t> blob;
	size_t cap = 0, B = 0, used = 0, m = 0;
	std::vector<unsigned long long> off, ts, fps;
	std::vector<cmb200_addr> addr;
	DevMem<unsigned long long> d_off;
	DevMem<uint64_t> d_fp;
	int setup(cmb200_engine *eng) {
		e = eng;
		CMB_CHECK(cudaSetDevice(e->device));
		cap = (size_t)e->host_batch * e->bsize;
		B = e->max_batch < cmb200_engine::META_CAP ? e->max_batch : cmb200_engine::META_CAP;
		off.resize(B); ts.resize(B); fps.resize(2 * B); addr.resize(B);
		return blob.alloc(cap) || d_off.alloc(B * 8) || d_fp.alloc(B * 16) ? -1 : 0;
	}
};

// The device half of a load and of a rename: m records {24-byte prefix, payload} at blob + off[i] (device
// memory of e, 16-byte aligned) are stored at addr[i] with ts[i] and fingerprint fps[i] ({0, 0} or
// fps = nullptr: none), as if put in this order: k_upsert claims the keys and raises seq, k_restore writes
// each record under its new prefix and rebuilds its parse checkpoints.  A record the arena has no room
// for is dropped, as a put is.  Enqueued on e->st.  (e->mu held; m <= max_batch)
static int restore_records(cmb200_engine *e, const uint8_t *blob, const unsigned long long *addr,
    const unsigned long long *ts, const unsigned long long *off, const uint64_t *fps, size_t m) {
	if (launch_upsert(e->table, addr, nullptr, (uint32_t)m, e->seq, e->seq_stride, e->d_slot, e->st)) return -1;
	EncodeJob job{};
	job.n = (uint32_t)m; job.nbytes = e->bsize;
	job.slot_idx = e->d_slot; job.addr = addr; job.ts = ts;
	job.seq0 = e->seq; job.seq_stride = e->seq_stride;
	job.table = e->table; job.arena = e->arena;
	if (launch_restore(job, blob, off, fps, e->bsize, e->st)) return -1;
	e->seq += (unsigned long long)m * e->seq_stride;
	e->stats.kernel_launches += 2;
	return 0;
}

// Puts the staged records into their engine as if they had been put in file order.  Returns how many
// (>= 0) or -1.
static long long load_flush(LoadBatch &b, bool with_fp) {
	if (b.m == 0) return 0;
	cmb200_engine *e = b.e;
	std::lock_guard<std::mutex> g(e->mu);
	CMB_CHECK(cudaSetDevice(e->device));
	const size_t m = b.m;
	if (e->tier.host) {
		unsigned long long c[8];
		if (read_counters(e, c)) return -1;
		if (c[2] + b.used > e->arena.size && demote_arena_all(e)) return -1;
	}
	CMB_CHECK(cudaMemcpyAsync(e->d_pages[0], b.blob, b.used, cudaMemcpyHostToDevice, e->st));
	CMB_CHECK(cudaMemcpyAsync(e->d_addr, b.addr.data(), m * 16, cudaMemcpyHostToDevice, e->st));
	CMB_CHECK(cudaMemcpyAsync(e->d_ts, b.ts.data(), m * 8, cudaMemcpyHostToDevice, e->st));
	CMB_CHECK(cudaMemcpyAsync(b.d_off, b.off.data(), m * 8, cudaMemcpyHostToDevice, e->st));
	CMB_CHECK(cudaMemcpyAsync(b.d_fp, b.fps.data(), m * 16, cudaMemcpyHostToDevice, e->st));
	if (restore_records(e, e->d_pages[0], e->d_addr, e->d_ts, b.d_off, with_fp ? (uint64_t *)b.d_fp : nullptr, m)) return -1;
	CMB_CHECK(cudaStreamSynchronize(e->st));
	b.m = 0; b.used = 0;
	return (long long)m;
}

struct AddrHash {
	size_t operator()(const std::pair<uint64_t, uint64_t> &a) const { return (size_t)(a.first * 0x9E3779B97F4A7C15ull ^ a.second); }
};
typedef std::unordered_set<std::pair<uint64_t, uint64_t>, AddrHash> AddrSet;

// Opens a snapshot file (a base) for a load into g engines and reads its header.  nullptr on failure
// (error set).
static FILE *open_snapshot(cmb200_engine *const *engines, int g, const char *path, SnapHeader &h) {
	FILE *f = fopen(path, "rb");
	if (!f) { set_error_msg("cmb200_load: no snapshot file"); return nullptr; }
	if (fread(&h, sizeof(h), 1, f) != 1 || memcmp(h.magic, "CMB200S1", 8) != 0 || h.version != 1) {
		fclose(f); set_error_msg("cmb200_load: not a snapshot of this library"); return nullptr;
	}
	for (int i = 0; i < g; i++)
		if ((int)h.pshift != engines[i]->pshift) { fclose(f); set_error_msg("cmb200_load: snapshot has another page size"); return nullptr; }
	return f;
}

// Stages the next n records of f into the load batches of their engines (cmb200_owner), flushing a batch
// when it is full; *loaded += records put.  skip (nullable): addresses a newer file of a chain has
// decided, whose records are passed over unread; decide (nullable) gets every address read.  The
// batches are not flushed at the end.  0 / -1 (error set).
static int load_records(FILE *f, uint64_t n, std::vector<LoadBatch> &bs, int g, bool with_fp, const AddrSet *skip,
    AddrSet *decide, uint64_t *loaded) {
	const uint32_t bsize = bs[0].e->bsize;
	int rc = 0;
	uint64_t done = 0;
	while (rc == 0 && done < n) {
		// record header and address first: the address names the engine whose batch takes the bytes
		SnapRecord r;
		cmb200_addr a;
		if (fread(&r, sizeof(r), 1, f) != 1 || r.len < 24 || r.len > 24u + bsize + 1024u || fread(&a, 16, 1, f) != 1) {
			rc = -1; set_error_msg("cmb200_load: truncated or corrupt snapshot"); break;
		}
		const size_t padded = ((size_t)r.len + 15) & ~(size_t)15;
		if (skip || decide) {
			const std::pair<uint64_t, uint64_t> ul(a.u, a.l);
			const bool decided = skip && skip->count(ul);
			if (decide && !decided) decide->insert(ul);
			if (decided) {
				if (fseeko(f, (off_t)(padded - 16), SEEK_CUR) != 0) { rc = -1; set_error_msg("cmb200_load: truncated or corrupt snapshot"); }
				done++;
				continue;
			}
		}
		uint64_t key;
		FNV_hash(&a, 16, &key);
		LoadBatch &b = bs[cmb200_owner(key, g)];
		if (padded > b.cap) { rc = -1; set_error_msg("cmb200_load: record larger than the staging buffer"); break; }
		if (b.m == b.B || b.used + padded > b.cap) {
			const long long got = load_flush(b, with_fp);
			if (got < 0) { rc = -1; break; }
			*loaded += (uint64_t)got;
		}
		uint8_t *rec = b.blob + b.used;
		memcpy(rec, &a, 16);
		if (fread(rec + 16, padded - 16, 1, f) != 1) { rc = -1; set_error_msg("cmb200_load: truncated or corrupt snapshot"); break; }
		{
			// the record must be what filemap_set would have stored (filemap.c:124-147): a foreign or
			// corrupt file must not reach k_restore, which trusts compressed_length
			int32_t clen;
			memcpy(&clen, rec + 16, 4);
			if (clen < 0 || (uint32_t)clen > bsize + 1024u || r.len != 24u + (clen ? (uint32_t)clen : bsize)) {
				rc = -1; set_error_msg("cmb200_load: truncated or corrupt snapshot"); break;
			}
		}
		b.addr[b.m] = a;
		b.off[b.m] = b.used; b.ts[b.m] = r.ts; b.fps[2 * b.m] = r.fp_hi; b.fps[2 * b.m + 1] = r.fp_lo;
		b.used += padded; b.m++;
		done++;
	}
	return rc;
}

static int load_flush_all(std::vector<LoadBatch> &bs, bool with_fp, uint64_t *loaded) {
	for (LoadBatch &b : bs) {
		const long long got = load_flush(b, with_fp);
		if (got < 0) return -1;
		*loaded += (uint64_t)got;
	}
	return 0;
}

static int load_setup(std::vector<LoadBatch> &bs, cmb200_engine *const *engines, int g) {
	bs.resize(g);
	for (int i = 0; i < g; i++)
		if (bs[i].setup(engines[i])) { set_error_msg("cmb200_load: no staging buffers"); return -1; }
	return 0;
}

extern "C" int cmb200_load_set(cmb200_engine *const *engines, int g, const char *path, uint64_t *records_out) {
	if (records_out) *records_out = 0;
	if (g < 1 || !engines) { set_error_msg("cmb200_load_set: no engines"); return -1; }
	SnapHeader h{};
	FILE *f = open_snapshot(engines, g, path, h);
	if (!f) return -1;
	std::vector<LoadBatch> bs;
	uint64_t loaded = 0;
	int rc = load_setup(bs, engines, g);
	if (rc == 0) rc = load_records(f, h.records, bs, g, h.flags & 1u, nullptr, nullptr, &loaded);
	if (rc == 0) rc = load_flush_all(bs, h.flags & 1u, &loaded);
	fclose(f);
	if (records_out) *records_out = loaded;
	return rc;
}

// Opens delta k of chain `id` and checks it whole before anything of it is applied: header, then the
// bounds of every record header and the file's exact length (the record bytes are not read).  Leaves
// the file at its first tombstone.  nullptr when the delta is missing, from another chain, out of
// sequence, truncated or corrupt: the chain's valid run ends before it.
static FILE *open_delta(const std::string &path, uint64_t id, uint32_t k, uint32_t pshift, uint32_t bsize, DeltaHeader &dh) {
	FILE *f = fopen(path.c_str(), "rb");
	if (!f) return nullptr;
	bool ok = fread(&dh, sizeof(dh), 1, f) == 1 && memcmp(dh.magic, "CMB200D1", 8) == 0 && dh.version == 1 &&
	    dh.pshift == pshift && dh.chain == id && dh.index == k && fseeko(f, 0, SEEK_END) == 0;
	const uint64_t size = ok ? (uint64_t)ftello(f) : 0;
	uint64_t pos = sizeof(dh) + 16 * dh.tombstones, bytes = 0;
	ok = ok && dh.tombstones <= size / 16 && pos <= size;
	for (uint64_t i = 0; ok && i < dh.records; i++) {
		SnapRecord r;
		ok = pos + sizeof(r) <= size && fseeko(f, (off_t)pos, SEEK_SET) == 0 && fread(&r, sizeof(r), 1, f) == 1 &&
		    r.len >= 24 && r.len <= 24u + bsize + 1024u;
		pos += sizeof(r) + (((uint64_t)r.len + 15) & ~15ull);
		bytes += r.len;
	}
	ok = ok && pos == size && bytes == dh.bytes && fseeko(f, sizeof(dh), SEEK_SET) == 0;
	if (!ok) { fclose(f); return nullptr; }
	return f;
}

// Whether a file <base_path>.d<j> with j > k exists.
static bool delta_beyond(const char *base_path, uint32_t k) {
	const std::string path(base_path);
	const size_t slash = path.rfind('/');
	const std::string dir = slash == std::string::npos ? "." : path.substr(0, slash + 1);
	const std::string stem = (slash == std::string::npos ? path : path.substr(slash + 1)) + ".d";
	DIR *d = opendir(dir.c_str());
	if (!d) return true;
	bool found = false;
	while (struct dirent *ent = readdir(d)) {
		const char *name = ent->d_name;
		if (strncmp(name, stem.c_str(), stem.size()) != 0) continue;
		const char *num = name + stem.size();
		char *end = nullptr;
		const unsigned long long j = strtoull(num, &end, 10);
		if (*num >= '0' && *num <= '9' && *end == '\0' && j > k) found = true;
	}
	closedir(d);
	return found;
}

extern "C" int cmb200_load_chain(cmb200_engine *const *engines, int g, const char *base_path, uint64_t *records_out,
    uint32_t *deltas_out) {
	if (records_out) *records_out = 0;
	if (deltas_out) *deltas_out = 0;
	if (g < 1 || !engines || !base_path) { set_error_msg("cmb200_load_chain: no engines"); return -1; }
	SnapHeader h{};
	FILE *base = open_snapshot(engines, g, base_path, h);
	if (!base) return -1;
	const uint64_t id = snap_chain_id(h);
	std::vector<FILE *> ds;
	std::vector<DeltaHeader> dhs;
	for (uint32_t k = 1; id != 0; k++) {
		DeltaHeader dh{};
		FILE *f = open_delta(std::string(base_path) + ".d" + std::to_string(k), id, k, h.pshift, engines[0]->bsize, dh);
		if (!f) break;
		ds.push_back(f); dhs.push_back(dh);
	}
	uint64_t before = 0;
	for (int i = 0; i < g; i++) before += cmb200_entries(engines[i]);
	std::vector<LoadBatch> bs;
	uint64_t loaded = 0;
	int rc = load_setup(bs, engines, g);
	// newest first: an address a newer file names (a record or a tombstone) is decided there, so every
	// record is put once, and none an older file names in vain takes arena space
	AddrSet decided;
	std::vector<ulonglong2> tombs;
	for (size_t j = ds.size(); j-- > 0 && rc == 0;) {
		FILE *f = ds[j];
		const DeltaHeader &dh = dhs[j];
		tombs.resize(dh.tombstones);
		if (dh.tombstones && fread(tombs.data(), 16, tombs.size(), f) != tombs.size()) { rc = -1; set_error_msg("cmb200_load: truncated or corrupt snapshot"); break; }
		rc = load_records(f, dh.records, bs, g, dh.flags & 1u, &decided, &decided, &loaded);
		if (rc == 0) rc = load_flush_all(bs, dh.flags & 1u, &loaded);
		// the records of a delta apply after its tombstones, so its records decide first
		for (const ulonglong2 &a : tombs) decided.insert(std::make_pair((uint64_t)a.x, (uint64_t)a.y));
	}
	if (rc == 0) rc = load_records(base, h.records, bs, g, h.flags & 1u, &decided, nullptr, &loaded);
	if (rc == 0) rc = load_flush_all(bs, h.flags & 1u, &loaded);
	for (FILE *f : ds) fclose(f);
	fclose(base);
	if (rc) return -1;
	// The engines continue the chain only if they hold exactly the store it describes: they were empty
	// and every record put is live (none dropped for lack of space, none retired by a host-tier lap),
	// and no delta file lies beyond the run (a tick that continued it would leave that file in a valid
	// position).  Otherwise they hold no chain state, and the next tick writes a base.
	bool whole = id != 0 && before == 0 && !delta_beyond(base_path, (uint32_t)ds.size());
	uint64_t live = 0;
	for (int i = 0; i < g && rc == 0; i++) {
		cmb200_engine *e = engines[i];
		std::lock_guard<std::mutex> lk(e->mu);
		cmb200_engine::Chain &ch = e->chain;
		if (ch.pending) { whole = false; continue; }
		unsigned long long c[8];
		std::vector<ExportEntry> none;
		if (read_counters(e, c) || chain_room(e, c[0]) ||
		    live_records(e, false, none, c, ~0ull, ch.base_dev[ch.cur ^ 1], &ch.n_next) < 0) { rc = -1; break; }
		ch.w_next = e->seq;
		live += ch.n_next;
	}
	whole = whole && rc == 0 && live == loaded;
	for (int i = 0; i < g; i++) {
		cmb200_engine *e = engines[i];
		std::lock_guard<std::mutex> lk(e->mu);
		cmb200_engine::Chain &ch = e->chain;
		if (ch.pending) continue;
		if (whole) { ch.cur ^= 1; ch.n = ch.n_next; ch.w = ch.w_next; ch.id = id; ch.k = (uint32_t)ds.size(); }
		else ch.id = 0;
	}
	if (records_out) *records_out = loaded;
	if (deltas_out) *deltas_out = (uint32_t)ds.size();
	return rc;
}

extern "C" int cmb200_load(cmb200_engine *e, const char *path, uint64_t *records_out) {
	return cmb200_load_set(&e, 1, path, records_out);
}

// ---- pages of a sharded store (CMB200_DEVICES): gather / scatter and peer copies ----------------

extern "C" int cmb200_move_pages(cmb200_engine *e, size_t n, void *dst_dev, const uint32_t *dst_idx, const void *src_dev,
    const uint32_t *src_idx) {
	if (n == 0) return 0;
	if (check_dev_pages(dst_dev, "cmb200_move_pages") || check_dev_pages(src_dev, "cmb200_move_pages")) return -1;
	if (n > 0xffffffffu) { set_error_msg("cmb200_move_pages: too many pages"); return -1; }
	std::lock_guard<std::mutex> g(e->mu);
	CMB_CHECK(cudaSetDevice(e->device));
	if ((dst_idx || src_idx) && e->d_move_idx.grow(n * 8, e->st)) return -1;
	uint32_t *d_dst_idx = dst_idx ? (uint32_t *)e->d_move_idx : nullptr;
	uint32_t *d_src_idx = src_idx ? e->d_move_idx + n : nullptr;
	if (dst_idx) CMB_CHECK(cudaMemcpyAsync(d_dst_idx, dst_idx, n * 4, cudaMemcpyHostToDevice, e->st));
	if (src_idx) CMB_CHECK(cudaMemcpyAsync(d_src_idx, src_idx, n * 4, cudaMemcpyHostToDevice, e->st));
	if (launch_move_pages(dst_dev, d_dst_idx, src_dev, d_src_idx, (uint32_t)n, e->bsize, e->st)) return -1;
	e->stats.kernel_launches++;
	CMB_CHECK(cudaStreamSynchronize(e->st));
	return 0;
}

extern "C" int cmb200_copy_peer(cmb200_engine *dst_e, void *dst_dev, cmb200_engine *src_e, const void *src_dev, size_t bytes) {
	if (bytes == 0) return 0;
	std::lock_guard<std::mutex> g(src_e->mu);
	CMB_CHECK(cudaSetDevice(src_e->device));
	CMB_CHECK(cudaMemcpyPeerAsync(dst_dev, dst_e->device, src_dev, src_e->device, bytes, src_e->st));
	CMB_CHECK(cudaStreamSynchronize(src_e->st));
	return 0;
}

// ---- table rebuild ----------------------------------------------------------------------------
// The table is rebuilt when deleted keys (`tombs` tombstones; slots of dropped puts go with them) have
// eaten a good part of its empty slots: miss probes end at an EMPTY slot, and linear probing never
// frees one by itself.  Slots move, records do not, so a snapshot's writer need not be waited for.
// (e->mu held, get_gate closed: small gets read slots)
static int rebuild_table_locked(cmb200_engine *e, unsigned long long tombs) {
	if (tombs <= e->table.cap / 8) return 0;
	// parse checkpoints move with their slots (k_rehash); without room for a second side table
	// they are dropped instead, and those records are walked by one warp until rewritten
	const bool ckpt = e->table.ckpt != nullptr;
	TableMem mem;
	int got = table_alloc(mem, e->table.cap, e->table.fp != nullptr, e->table.fp_tag != nullptr, ckpt, e->st);
	if (got > 0 && ckpt) got = table_alloc(mem, e->table.cap, e->table.fp != nullptr, e->table.fp_tag != nullptr, false, e->st);
	if (got < 0) return -1;
	if (got > 0) return 0;                           // no room for a second table: keep the old one
	TableView fresh = e->table;
	mem.view(fresh);
	if (launch_rehash(e->table, fresh, e->st)) return -1;
	if (ckpt && !fresh.ckpt) CMB_CHECK(cudaMemsetAsync(e->table.ckpt, 0, (e->table.cap + 2) * CKPT_WORDS * 4, e->st));
	CMB_CHECK(cudaMemsetAsync(e->d_counters + 1, 0, sizeof(unsigned long long), e->st));   // tombstones
	CMB_CHECK(cudaStreamSynchronize(e->st));
	if (!mem.ckpt) mem.ckpt = std::move(e->table_mem.ckpt);
	e->table_mem = std::move(mem);
	e->table_mem.view(e->table);
	e->stats.kernel_launches++;
	return 0;
}

// ---- invalidation of an object's pages ----------------------------------------------------------
// An interval of at most this many addresses is looked up key by key (k_invalidate_keys), a longer
// one by a scan of the whole table (k_invalidate_scan).  On an H100 the two cost the same at 1/58 of
// the slots of a 2^25-slot table and 1/38 of a 2^27-slot one (DESIGN.md §2, *Invalidation*): 1/64
// keeps the keyed path where it was measured cheaper.
static uint64_t invalidate_keyed_max(uint64_t cap) { return (cap + 2) / 64; }

extern "C" int cmb200_invalidate(cmb200_engine *e, uint64_t u, uint64_t l_first, uint64_t l_last, uint64_t *removed_out) {
	if (l_first > l_last) { set_error_msg("cmb200_invalidate: l_first > l_last"); return -1; }
	std::lock_guard<std::mutex> g(e->mu);
	if (e->multi_gpu) {
		set_error_msg("cmb200_invalidate: not available after a multi-GPU call (the index holds other ranks' records)");
		return -1;
	}
	CMB_CHECK(cudaSetDevice(e->device));
	if (!e->d_removed && e->d_removed.alloc(sizeof(unsigned long long))) return -1;
	CMB_CHECK(cudaMemsetAsync(e->d_removed, 0, sizeof(unsigned long long), e->st));
	// l_last - l_first + 1 overflows for the full interval: compare the difference instead
	const bool scan = l_last - l_first >= invalidate_keyed_max(e->table.cap);
	if (launch_invalidate(e->table, e->arena, u, l_first, l_last, scan, e->d_removed, e->st)) return -1;
	e->stats.kernel_launches++;
	unsigned long long removed = 0;
	CMB_CHECK(cudaMemcpyAsync(&removed, e->d_removed, sizeof(removed), cudaMemcpyDeviceToHost, e->st));
	unsigned long long c[8];
	if (read_counters(e, c)) return -1;
	if (removed_out) *removed_out = removed;
	if (c[1] > e->table.cap / 8) {
		cmb200_engine::GateClosed gg(e->get_gate);
		return rebuild_table_locked(e, c[1]);
	}
	return 0;
}

// ---- read-modify-write of stored pages ----------------------------------------------------------
// The patches are grouped by address into rows of the page ring.  Rows, spans and bytes cross to the
// device in one copy; then each slice of host_batch rows runs a get's lookup and decode into the ring,
// k_patch, and a put's upsert and encode from the ring, so that only the written bytes cross PCIe.
// The decode is a put's read, not a get: verified, it books into the store scan's counters (which
// cmb200_verify_store zeroes before it reads them); otherwise its tier hits and hot-log entries go to
// scratch words.  It never touches.
static size_t align16(size_t v) { return (v + 15) & ~(size_t)15; }

extern "C" int cmb200_patch_batch(cmb200_engine *e, size_t n, const cmb200_addr *addr, const uint32_t *page_off,
    const uint32_t *len, const void *bytes_host, const uint64_t *ts, int32_t *status_out) {
	for (size_t i = 0; i < n; i++)
		if (len[i] == 0 || (uint64_t)page_off[i] + len[i] > e->bsize) {
			set_error_msg("cmb200_patch_batch: a patch is empty or reaches past the page");
			return -1;
		}
	if (n >= 0xffffffffull) { set_error_msg("cmb200_patch_batch: too many patches"); return -1; }
	std::lock_guard<std::mutex> g(e->mu);
	if (e->multi_gpu) {
		set_error_msg("cmb200_patch_batch: not available after a multi-GPU call (the index holds other ranks' records)");
		return -1;
	}
	if (n == 0) return 0;
	CMB_CHECK(cudaSetDevice(e->device));
	// rows in order of first appearance; each patch's span goes to its row, in array order
	std::unordered_map<std::pair<uint64_t, uint64_t>, uint32_t, AddrHash> row_of;
	std::vector<uint32_t> row(n);
	for (size_t i = 0; i < n; i++)
		row[i] = row_of.emplace(std::make_pair(addr[i].u, addr[i].l), (uint32_t)row_of.size()).first->second;
	const size_t R = row_of.size();
	std::vector<uint32_t> first(R + 1, 0);                  // first span of each row
	for (size_t i = 0; i < n; i++) first[row[i] + 1]++;
	for (size_t r = 0; r < R; r++) first[r + 1] += first[r];
	// staging: addr (16 / row), ts (8 / row), first (4 / row + 4), spans (16 / patch), bytes (each span
	// placed congruent to its page offset modulo 16, so that k_patch moves it in 16-byte words), then the
	// device-only valid flags (1 / row)
	const size_t o_ts = R * 16, o_first = align16(o_ts + R * 8), o_spans = align16(o_first + (R + 1) * 4);
	const size_t o_bytes = align16(o_spans + n * sizeof(PatchSpan));
	size_t nbytes = 0;
	for (size_t i = 0; i < n; i++) nbytes += len[i] + 15;
	const size_t o_valid = align16(o_bytes + nbytes), total = o_valid + align16(R);
	if (e->h_patch_bytes < o_valid) {
		e->h_patch_bytes = 0;
		if (e->h_patch.alloc(o_valid)) return -1;
		e->h_patch_bytes = o_valid;
	}
	if (e->d_patch.grow(total, e->st)) return -1;
	uint8_t *h = e->h_patch;
	unsigned long long *h_addr = (unsigned long long *)h, *h_ts = (unsigned long long *)(h + o_ts);
	PatchSpan *h_spans = (PatchSpan *)(h + o_spans);
	std::vector<uint32_t> fill(first.begin(), first.end() - 1);
	const uint8_t *src = (const uint8_t *)bytes_host;
	size_t at = 0;                                          // next free byte of the bytes region
	for (size_t i = 0; i < n; i++) {
		const uint32_t r = row[i];
		h_addr[2 * r] = addr[i].u; h_addr[2 * r + 1] = addr[i].l;
		h_ts[r] = ts ? ts[i] : 0;                           // the last patch of the row wins
		at += (page_off[i] - at) & 15u;
		h_spans[fill[r]++] = PatchSpan{page_off[i], len[i], (unsigned long long)at};
		memcpy(h + o_bytes + at, src, len[i]);
		src += len[i];
		at += len[i];
	}
	memcpy(h + o_first, first.data(), (R + 1) * 4);
	uint8_t *d = e->d_patch;
	CMB_CHECK(cudaMemcpyAsync(d, h, o_valid, cudaMemcpyHostToDevice, e->st));
	const bool verify = e->table.fp_tag != nullptr;
	if (!verify && e->tier.dev && !e->d_patch_hot) {
		if (e->d_patch_hot.alloc((2 + 2 * (size_t)HOT_LOG_N) * sizeof(unsigned long long))) return -1;
		CMB_CHECK(cudaMemsetAsync(e->d_patch_hot, 0, 2 * sizeof(unsigned long long), e->st));
	}
	std::vector<int32_t> st(R), lens(R);
	std::vector<cmb200_addr> drop;
	uint64_t stored = 0;
	for (size_t r0 = 0; r0 < R; r0 += e->host_batch) {
		const uint32_t m = (uint32_t)(R - r0 < e->host_batch ? R - r0 : e->host_batch);
		const unsigned long long *d_addr = (const unsigned long long *)d + 2 * r0;
		uint8_t *d_valid = d + o_valid + r0;
		uint8_t *ring = e->d_pages[(r0 / e->host_batch) & 1];
		if (launch_lookup(e->table, d_addr, nullptr, m, e->d_status, e->d_recoff, e->d_vlen, nullptr, e->st,
			verify ? (uint32_t *)e->d_vidx : nullptr)) return -1;
		DecodeJob job{};
		job.n = m; job.nbytes = e->bsize; job.pages = ring; job.status = e->d_status;
		job.rec_off = e->d_recoff; job.vlen = e->d_vlen; job.arena = e->arena.base; job.host = e->tier.dev;
		job.addr = d_addr;
		if (verify) {
			const DecodeVerify ver{e->d_vidx, e->table.fp, e->table.fp_tag, e->d_vstat + VS_WORDS};
			if (launch_decode(job, e->st, &ver)) return -1;
		} else {
			if (e->d_patch_hot) {
				job.host_hits = e->d_patch_hot;
				job.hot = HotLog{e->d_patch_hot + 1, (ulonglong2 *)(e->d_patch_hot + 2)};
			}
			if (launch_decode(job, e->st)) return -1;
		}
		if (launch_patch(ring, e->bsize, m, e->d_status, (const uint32_t *)(d + o_first) + r0,
			(const PatchSpan *)(d + o_spans), d + o_bytes, d_valid, e->st)) return -1;
		if (launch_upsert(e->table, d_addr, d_valid, m, e->seq, e->seq_stride, e->d_slot, e->st)) return -1;
		EncodeJob enc{};
		enc.pages = ring; enc.page_stride = e->bsize; enc.nbytes = e->bsize; enc.n = m;
		enc.accel = (uint32_t)e->accel;
		enc.stage = e->d_stage; enc.stage_stride = e->stage_stride;
		enc.lens = e->d_lens;
		enc.rec_out = e->d_recoff_out;
		enc.fps = (e->flags & CMB200_FINGERPRINT) ? (uint64_t *)e->d_fps : nullptr;
		enc.work = e->d_work;
		enc.order = e->d_order;
		enc.slot_idx = e->d_slot;
		enc.addr = d_addr;
		enc.ts = ts ? (const unsigned long long *)(d + o_ts) + r0 : nullptr;
		enc.seq0 = e->seq; enc.seq_stride = e->seq_stride;
		enc.table = e->table; enc.arena = e->arena;
		const int encode_kernels = launch_encode(enc, e->st);
		if (encode_kernels < 0) return -1;
		e->seq += (unsigned long long)m * e->seq_stride;
		e->stats.kernel_launches += 4 + encode_kernels;
		CMB_CHECK(cudaMemcpyAsync(st.data() + r0, e->d_status, m * 4, cudaMemcpyDeviceToHost, e->st));
		CMB_CHECK(cudaMemcpyAsync(lens.data() + r0, e->d_lens, m * 4, cudaMemcpyDeviceToHost, e->st));
		CMB_CHECK(cudaStreamSynchronize(e->st));
		for (size_t r = r0; r < r0 + m; r++) {
			// a hit that stored nothing was dropped for lack of arena space (the encoder leaves the slot as it was)
			if (st[r] == CMB200_HIT && lens[r] < 0) st[r] = CMB200_DROPPED;
			if (st[r] == CMB200_HIT) stored++;
			if (st[r] == CMB200_DROPPED || st[r] == CMB200_BAD_DECODE || st[r] == CMB200_CORRUPT)
				drop.push_back(cmb200_addr{h_addr[2 * r], h_addr[2 * r + 1]});
		}
	}
	// records that cannot be trusted, and old pages whose patched version found no room, leave the store
	for (size_t k = 0; k < drop.size(); k += e->max_batch) {
		const uint32_t m = (uint32_t)(drop.size() - k < e->max_batch ? drop.size() - k : e->max_batch);
		CMB_CHECK(cudaMemcpyAsync(e->d_addr, drop.data() + k, (size_t)m * 16, cudaMemcpyHostToDevice, e->st));
		if (launch_unset(e->table, e->arena, e->d_addr, m, e->st)) return -1;
		e->stats.kernel_launches++;
	}
	CMB_CHECK(cudaStreamSynchronize(e->st));
	e->stats.put_chunks += stored;
	for (size_t i = 0; i < n; i++) status_out[i] = st[row[i]];
	return 0;
}

// ---- arena compaction -------------------------------------------------------------------------
// The arena is a bump allocator: a deleted record, or one that outgrew its place, leaves its bytes
// behind as garbage.  Compaction slides the live records down to the start of the arena (sorted by
// offset, so every record moves to a lower or equal address), window by window through one of the
// page-ring buffers, repoints the slots and resets the bump pointer and the per-warp segments.
// Stop-the-world on the engine's stream, at HBM speed; callers trigger it when the arena is about
// to overflow although a good part of it is garbage (filemap_make_room, cmb200_compact).
// (e->mu held)
static int compact_locked(cmb200_engine *e, uint64_t *reclaimed_out) {
	snap_wait_written(e);                                // records move over listed ones; small gets go on meanwhile
	cmb200_engine::GateClosed gg(e->get_gate);          // records move: no small get may be reading the arena
	harvest_pending(e, true);
	unsigned long long c[8];
	std::vector<ExportEntry> list;
	// arena records only: the host tier is a ring and is never compacted
	const int listed = live_records(e, true, list, c);
	if (listed < 0) return -1;
	if (listed > 0) { set_error_msg("cmb200_compact: the store changed under the compaction"); return -1; }
	const unsigned long long head_before = c[2];
	const size_t count = list.size();
	DevMem<MoveEntry> d_moves;
	std::vector<MoveEntry> moves(count);
	unsigned long long at = 0;
	for (size_t i = 0; i < count; i++) {
		moves[i] = MoveEntry{list[i].rec_off, at, list[i].len, list[i].slot};
		at += ((unsigned long long)list[i].len + 15ull) & ~15ull;
	}
	if (count && d_moves.alloc(count * sizeof(MoveEntry) + 256)) return -1;
	if (count) CMB_CHECK(cudaMemcpyAsync(d_moves, moves.data(), count * sizeof(MoveEntry), cudaMemcpyHostToDevice, e->st));
	// windows: as many records as fit the bounce buffer (one page-ring buffer)
	const unsigned long long bounce_cap = (unsigned long long)e->host_batch * e->bsize;
	size_t k = 0;
	while (k < count) {
		size_t j = k;
		while (j < count && moves[j].new_off + (((unsigned long long)moves[j].len + 15ull) & ~15ull) - moves[k].new_off <= bounce_cap) j++;
		if (j == k) { set_error_msg("cmb200_compact: record larger than the bounce buffer"); return -1; }
		if (launch_compact_window(e->table, e->arena, d_moves + k, (uint32_t)(j - k), e->d_pages[0], e->st)) return -1;
		e->stats.kernel_launches += 2;
		k = j;
	}
	// bump pointer back to the end of the live records, no garbage, no half-used segments
	unsigned long long fresh[2] = {at, 0};
	CMB_CHECK(cudaMemcpyAsync(e->d_counters + 2, fresh, 16, cudaMemcpyHostToDevice, e->st));
	CMB_CHECK(cudaMemsetAsync(e->arena.seg, 0, ARENA_SEG_SLOTS * 2 * sizeof(unsigned long long), e->st));
	CMB_CHECK(cudaStreamSynchronize(e->st));
	if (reclaimed_out) *reclaimed_out = head_before > at ? head_before - at : 0;
	// the table is rebuilt on the same occasion
	return rebuild_table_locked(e, c[1]);
}

extern "C" int cmb200_compact(cmb200_engine *e, uint64_t *reclaimed_out) {
	std::lock_guard<std::mutex> g(e->mu);
	return compact_locked(e, reclaimed_out);
}

// ---- rename: an object's records move to another object's addresses ----------------------------
// A record's prefix names its address and k_get_small trusts that prefix, so a record cannot be aliased
// under a new key: it is copied under the new prefix and the old one is retired.  The LZ4 block does not
// depend on the address, so nothing is encoded again.  The work goes in slices that are bounded as a
// load's batches are (<= min(max_batch, META_CAP) records, one page-ring buffer of bytes plus one
// record), per pair (source engine, destination engine):
//   1. under the source's lock: k_rename_select lists the records whose new key the destination owns,
//      k_rename_gather copies them to the source's staging buffer and retires their slots;
//   2. the slice crosses to the destination (a peer copy, or none when both are one engine);
//   3. under the destination's lock: a compaction if the slice does not fit above the bump pointer and
//      garbage covers the shortfall, then restore_records, as a load stores its records.
// No list of arena offsets outlives step 1, so a compaction in step 3 moves nothing a later step reads.
// One call at a time uses the staging buffers; the call never holds two engine locks at once.
static std::mutex rename_mu;

// The list of a slice inside an engine's d_ren_list, for n entries: cursor (4 words), addr, ts, off, fp
// (the part a destination reads, contiguous), then loc, slot, len.
static size_t rename_list_bytes(size_t n) { return 32 + n * 64; }
static size_t rename_list_head(size_t n) { return 32 + n * 48; }
static RenameList rename_list_view(uint8_t *base, size_t n, unsigned long long max_bytes) {
	RenameList r{};
	r.cursor = (unsigned long long *)base;
	r.addr = (unsigned long long *)(base + 32);
	r.ts = r.addr + 2 * n;
	r.off = r.ts + n;
	r.fp = (uint64_t *)(r.off + n);
	r.loc = (unsigned long long *)(r.fp + 2 * n);
	r.slot = (uint32_t *)(r.loc + n);
	r.len = r.slot + n;
	r.max_n = (uint32_t)n;
	r.max_bytes = max_bytes;
	return r;
}

// Step 3 on engine e, whose d_ren_list / d_ren_bytes hold the slice (m records, `bytes` staged).
// (e->mu held)
static int rename_store(cmb200_engine *e, size_t n, size_t m, unsigned long long bytes, uint64_t *moved,
    uint64_t *dropped) {
	unsigned long long c[8];
	if (read_counters(e, c)) return -1;
	// room: compact once if the garbage covers what the slice needs beyond the bump pointer (with per-warp
	// arena segments the unused ends of segments come back too, and are not counted as garbage); never
	// evict or demote here, so whatever still does not fit is dropped by k_restore
	if (c[2] + bytes > e->arena.size && (c[3] >= c[2] + bytes - e->arena.size || e->arena.seg_bytes != 0)) {
		if (compact_locked(e, nullptr)) return -1;
		if (read_counters(e, c)) return -1;
	}
	const unsigned long long dropped_before = c[4];
	const RenameList r = rename_list_view(e->d_ren_list, n, 0);
	if (restore_records(e, e->d_ren_bytes, r.addr, r.ts, r.off, r.fp, m)) return -1;
	if (read_counters(e, c)) return -1;
	const uint64_t lost = c[4] - dropped_before;
	*moved += m - lost;
	*dropped += lost;
	return 0;
}

// One slice from engine s to engine d (index di of g).  Returns the records taken (0: none left), -1.
// An engine that has made a multi-GPU call holds other ranks' records in its index.  (e->mu held)
static bool rename_refused(cmb200_engine *e) {
	if (!e->multi_gpu) return false;
	set_error_msg("cmb200_rename: not available after a multi-GPU call (the index holds other ranks' records)");
	return true;
}

static long long rename_slice(cmb200_engine *s, cmb200_engine *d, int g, int di, uint64_t u_from, uint64_t u_to,
    uint64_t l_first, uint64_t l_last, size_t n, unsigned long long max_bytes, uint64_t *moved, uint64_t *dropped) {
	size_t m;
	unsigned long long bytes;
	{
		std::unique_lock<std::mutex> lk(s->mu);
		if (rename_refused(s)) return -1;
		CMB_CHECK(cudaSetDevice(s->device));
		if (s->d_ren_list.grow(rename_list_bytes(n), s->st)) return -1;
		const RenameList r = rename_list_view(s->d_ren_list, n, max_bytes);
		CMB_CHECK(cudaMemsetAsync(r.cursor, 0, 8, s->st));
		// l_last - l_first + 1 overflows for the full interval: compare the difference instead
		const bool scan = l_last - l_first >= invalidate_keyed_max(s->table.cap);
		if (launch_rename_select(s->table, r, u_from, u_to, l_first, l_last, scan, g, di, s->bsize, s->st)) return -1;
		unsigned long long cur[3] = {};
		CMB_CHECK(cudaMemcpyAsync(cur, r.cursor, sizeof(cur), cudaMemcpyDeviceToHost, s->st));
		CMB_CHECK(cudaStreamSynchronize(s->st));
		s->stats.kernel_launches += 2;
		if (cur[0] == 0) return 0;                           // nothing left to move to engine di
		m = (size_t)cur[1];
		bytes = cur[2];
		// grown to the largest slice so far, never past one page-ring buffer plus one record
		if (s->d_ren_bytes.grow(bytes, s->st)) return -1;
		if (launch_rename_gather(s->table, s->arena, s->tier.dev, r, (uint32_t)m, s->d_ren_bytes, s->st)) return -1;
		s->stats.kernel_launches++;
		if (s == d) {
			if (rename_store(s, n, m, bytes, moved, dropped)) return -1;
		} else {
			CMB_CHECK(cudaStreamSynchronize(s->st));
		}
		// the retired slots are tombstones: rebuild the table when they have eaten its empty slots
		unsigned long long c[8];
		if (read_counters(s, c)) return -1;
		if (c[1] > s->table.cap / 8) {
			cmb200_engine::GateClosed gg(s->get_gate);
			if (rebuild_table_locked(s, c[1])) return -1;
		}
		if (s == d) return (long long)m;
	}
	std::lock_guard<std::mutex> lk(d->mu);
	// the slice is out of the source already: a refusal here loses it, as a drop would, and never serves it stale
	if (rename_refused(d)) return -1;
	CMB_CHECK(cudaSetDevice(d->device));
	if (d->d_ren_list.grow(rename_list_bytes(n), d->st) || d->d_ren_bytes.grow(bytes, d->st)) return -1;
	// the list's cursor, addr, ts, off and fp, then the staged records
	const size_t head = rename_list_head(n);
	if (s->device == d->device) {
		CMB_CHECK(cudaMemcpyAsync(d->d_ren_list, s->d_ren_list, head, cudaMemcpyDeviceToDevice, d->st));
		CMB_CHECK(cudaMemcpyAsync(d->d_ren_bytes, s->d_ren_bytes, bytes, cudaMemcpyDeviceToDevice, d->st));
	} else {
		CMB_CHECK(cudaMemcpyPeerAsync(d->d_ren_list, d->device, s->d_ren_list, s->device, head, d->st));
		CMB_CHECK(cudaMemcpyPeerAsync(d->d_ren_bytes, d->device, s->d_ren_bytes, s->device, bytes, d->st));
	}
	if (rename_store(d, n, m, bytes, moved, dropped)) return -1;
	return (long long)m;
}

extern "C" int cmb200_rename_set(cmb200_engine *const *engines, int g, uint64_t u_from, uint64_t u_to,
    uint64_t l_first, uint64_t l_last, uint64_t *moved_out, uint64_t *dropped_out) {
	if (moved_out) *moved_out = 0;
	if (dropped_out) *dropped_out = 0;
	if (!engines || g < 1) { set_error_msg("cmb200_rename_set: no engines"); return -1; }
	if (l_first > l_last) { set_error_msg("cmb200_rename: l_first > l_last"); return -1; }
	for (int i = 0; i < g; i++) {
		if (engines[i]->pshift != engines[0]->pshift) { set_error_msg("cmb200_rename_set: engines of different page sizes"); return -1; }
		// under each engine's lock in turn, as cmb200_invalidate reads the flag; rename_slice reads it
		// again under the lock it works under
		std::lock_guard<std::mutex> lk(engines[i]->mu);
		if (rename_refused(engines[i])) return -1;
	}
	if (u_from == u_to) return 0;
	std::lock_guard<std::mutex> call(rename_mu);
	// slice bounds common to every engine of the call, as a load's batches are bounded
	size_t n = cmb200_engine::META_CAP;
	unsigned long long max_bytes = ~0ull;
	for (int i = 0; i < g; i++) {
		if (engines[i]->max_batch < n) n = engines[i]->max_batch;
		const unsigned long long ring = (unsigned long long)engines[i]->host_batch * engines[i]->bsize;
		if (ring < max_bytes) max_bytes = ring;
	}
	uint64_t moved = 0, dropped = 0;
	int rc = 0;
	for (int si = 0; si < g && rc == 0; si++)
		for (int di = 0; di < g && rc == 0; di++)
			for (;;) {
				const long long took = rename_slice(engines[si], engines[di], g, di, u_from, u_to, l_first, l_last, n,
				    max_bytes, &moved, &dropped);
				if (took < 0) rc = -1;
				if (took <= 0) break;
			}
	if (moved_out) *moved_out = moved;
	if (dropped_out) *dropped_out = dropped;
	return rc;
}

extern "C" int cmb200_rename(cmb200_engine *e, uint64_t u_from, uint64_t u_to, uint64_t l_first, uint64_t l_last,
    uint64_t *moved_out, uint64_t *dropped_out) {
	return cmb200_rename_set(&e, 1, u_from, u_to, l_first, l_last, moved_out, dropped_out);
}

// ---- verified reads (CMB200_VERIFY) ------------------------------------------------------------

extern "C" int cmb200_verify_stats(cmb200_engine *e, struct cmb200_verify_stats *out) {
	std::lock_guard<std::mutex> g(e->mu);
	memset(out, 0, sizeof(*out));
	if (!e->d_vstat) return 0;
	unsigned long long v[VS_WORDS];
	CMB_CHECK(cudaSetDevice(e->device));
	CMB_CHECK(cudaMemcpyAsync(v, e->d_vstat, sizeof(v), cudaMemcpyDeviceToHost, e->st));
	CMB_CHECK(cudaStreamSynchronize(e->st));
	out->verified = v[VS_VERIFIED]; out->unverified = v[VS_UNVERIFIED]; out->corrupt = v[VS_CORRUPT];
	out->scanned = e->scanned; out->scan_corrupt = e->scan_corrupt;
	return 0;
}

// Every live local record, both tiers, decoded batch by batch into the first page-ring buffer by the
// verified k_decode (host_hits null: a scan books no tier hit), whose counters go to the second half of
// d_vstat.  The records do not move while the engine lock is held, and small gets only read them.
extern "C" int cmb200_verify_store(cmb200_engine *e, size_t max, cmb200_addr *bad_out, size_t *n_bad,
    uint64_t *checked) {
	std::lock_guard<std::mutex> g(e->mu);
	if (n_bad) *n_bad = 0;
	if (checked) *checked = 0;
	if (!e->table.fp_tag) { set_error_msg("cmb200_verify_store: engine created without CMB200_VERIFY"); return -1; }
	CMB_CHECK(cudaSetDevice(e->device));
	harvest_pending(e, true);
	unsigned long long c[8];
	std::vector<ExportEntry> list;
	const int listed = live_records(e, false, list, c);
	if (listed < 0) return -1;
	if (listed > 0) { set_error_msg("cmb200_verify_store: the store changed under the scan"); return -1; }
	unsigned long long *scan = e->d_vstat + VS_WORDS;
	CMB_CHECK(cudaMemsetAsync(scan, 0, VS_WORDS * sizeof(unsigned long long), e->st));
	const size_t B = e->host_batch;
	DevMem<ExportEntry> d_list;
	if (!list.empty() && d_list.alloc(B * sizeof(ExportEntry) + 256)) return -1;
	std::vector<int32_t> st(B);
	std::vector<cmb200_addr> addr(B);
	size_t bad = 0;
	for (size_t at = 0; at < list.size(); at += B) {
		const uint32_t m = (uint32_t)(list.size() - at < B ? list.size() - at : B);
		CMB_CHECK(cudaMemcpyAsync(d_list, list.data() + at, m * sizeof(ExportEntry), cudaMemcpyHostToDevice, e->st));
		if (launch_scan_prep(e->table, d_list, m, e->d_status, e->d_recoff, e->d_vlen, e->d_vidx,
			e->d_addr, e->st)) return -1;
		DecodeJob job{};
		job.n = m; job.nbytes = e->bsize; job.pages = e->d_pages[0]; job.status = e->d_status;
		job.rec_off = e->d_recoff; job.vlen = e->d_vlen; job.arena = e->arena.base; job.host = e->tier.dev;
		const DecodeVerify ver{e->d_vidx, e->table.fp, e->table.fp_tag, scan};
		if (launch_decode(job, e->st, &ver)) return -1;
		e->stats.kernel_launches += 2;
		CMB_CHECK(cudaMemcpyAsync(st.data(), e->d_status, m * 4, cudaMemcpyDeviceToHost, e->st));
		CMB_CHECK(cudaMemcpyAsync(addr.data(), e->d_addr, m * 16, cudaMemcpyDeviceToHost, e->st));
		CMB_CHECK(cudaStreamSynchronize(e->st));
		for (uint32_t i = 0; i < m; i++) {
			if (st[i] != CMB200_CORRUPT && st[i] != CMB200_BAD_DECODE) continue;
			if (bad < max && bad_out) bad_out[bad] = addr[i];
			bad++;
		}
	}
	unsigned long long v[VS_WORDS];
	CMB_CHECK(cudaMemcpyAsync(v, scan, sizeof(v), cudaMemcpyDeviceToHost, e->st));
	CMB_CHECK(cudaStreamSynchronize(e->st));
	e->scanned += list.size();
	e->scan_corrupt += bad;
	if (n_bad) *n_bad = bad;
	if (checked) *checked = v[VS_VERIFIED] + v[VS_CORRUPT];
	return 0;
}

// ---- host tier ---------------------------------------------------------------------------------
// Records demoted from the arena live in page-locked, device-mapped host memory, in the arena's
// record format.  The tier is a ring in demotion order: it is never compacted, and a lap that comes
// round again first retires (unsets) the keys whose records it overwrites.

extern "C" int cmb200_host_tier_enable(cmb200_engine *e, uint64_t bytes) {
	std::lock_guard<std::mutex> g(e->mu);
	if (e->tier.host) { set_error_msg("cmb200_host_tier_enable: the engine already has a host tier"); return -1; }
	if (e->multi_gpu) { set_error_msg("cmb200_host_tier_enable: not available after a multi-GPU call"); return -1; }
	if (e->seq != 1) { set_error_msg("cmb200_host_tier_enable: must be called before the first put"); return -1; }
	bytes = (bytes + 4095) & ~4095ull;
	if (bytes < 4ull * e->stage_stride) { set_error_msg("cmb200_host_tier_enable: fewer bytes than four worst-case records"); return -1; }
	CMB_CHECK(cudaSetDevice(e->device));
	cmb200_engine::HostTier t;                          // built aside: the engine gets all of it or nothing
	if (t.d_ctr.alloc(3 * sizeof(unsigned long long)) || t.d_moves.alloc((size_t)e->max_batch * sizeof(DemoteEntry)) ||
	    t.d_promote.alloc((size_t)e->max_batch * sizeof(PromoteEntry)) || t.d_hot.alloc(HOT_LOG_N * sizeof(ulonglong2)) ||
	    cudaMemsetAsync(t.d_ctr, 0, 3 * sizeof(unsigned long long), e->st) != cudaSuccess ||
	    cudaMemsetAsync(t.d_hot, 0, HOT_LOG_N * sizeof(ulonglong2), e->st) != cudaSuccess ||
	    cudaStreamSynchronize(e->st) != cudaSuccess ||
	    t.host.alloc(bytes, true) || cudaHostGetDevicePointer(&t.dev, t.host, 0) != cudaSuccess) {
		cmb_set_error("cmb200_host_tier_enable", cudaGetLastError(), __FILE__, __LINE__);
		return -1;
	}
	t.size = bytes;
	e->tier = std::move(t);
	return 0;
}

// Moves one group of records (their tier region [start, end) is at most one lap and fits the bounce
// buffer) to the tier: gather -> retire what the region overwrites -> one or two D2H copies -> publish.
static int demote_group(cmb200_engine *e, const std::vector<DemoteEntry> &grp,
    const std::vector<std::pair<uint64_t, uint32_t>> &placed, uint64_t start, uint64_t end) {
	cmb200_engine::HostTier &t = e->tier;
	uint8_t *bounce = e->d_pages[0];
	const uint32_t n = (uint32_t)grp.size();
	CMB_CHECK(cudaMemcpyAsync(t.d_moves, grp.data(), n * sizeof(DemoteEntry), cudaMemcpyHostToDevice, e->st));
	if (launch_demote_gather(e->arena, t.d_moves, n, bounce, e->st)) return -1;
	// every record that starts before end - size lies where this region is about to be written
	std::vector<unsigned long long> ret;
	while (!t.log.empty() && t.log.front().first + t.size < end) {
		const uint64_t p = t.log.front().first, at = p % t.size;
		const unsigned long long *pre = reinterpret_cast<const unsigned long long *>(t.host + at);
		ret.insert(ret.end(), {pre[0], pre[1], REC_HOST | at, t.log.front().second});
		t.log.pop_front();
	}
	const bool overwrite = end > t.size;        // the region holds bytes of an earlier lap
	if (overwrite) {
		snap_wait_written(e);                    // nor a snapshot that has listed them
		e->get_gate.close();                     // no small get may be reading what is overwritten
	}
	int rc = 0;
	const size_t nr = ret.size() / 4;
	if (t.d_retire.grow(nr * 32, e->st)) rc = -1;
	const uint64_t a0 = start % t.size, bytes = end - start, first = std::min(bytes, t.size - a0);
	if (rc == 0 && nr) {
		rc = cudaMemcpyAsync(t.d_retire, ret.data(), nr * 32, cudaMemcpyHostToDevice, e->st) != cudaSuccess ||
		    launch_tier_retire(e->table, e->arena, t.d_retire, (uint32_t)nr, t.d_ctr, e->st) ? -1 : 0;
		e->stats.kernel_launches++;
	}
	if (rc == 0 && (cudaMemcpyAsync(t.host + a0, bounce, first, cudaMemcpyDeviceToHost, e->st) != cudaSuccess ||
	    (bytes > first && cudaMemcpyAsync(t.host, bounce + first, bytes - first, cudaMemcpyDeviceToHost, e->st) != cudaSuccess)))
		rc = -1;
	if (rc == 0 && launch_demote_publish(e->table, e->arena, t.d_moves, n, e->st)) rc = -1;
	if (cudaStreamSynchronize(e->st) != cudaSuccess) rc = -1;
	if (overwrite) e->get_gate.reopen();
	if (rc) { cmb_set_error("host tier demotion", cudaGetLastError(), __FILE__, __LINE__); return -1; }
	t.log.insert(t.log.end(), placed.begin(), placed.end());
	t.head = end;
	t.demoted_records += n;
	for (const DemoteEntry &d : grp) t.demoted_bytes += d.len;
	e->stats.kernel_launches += 2;
	return 0;
}

// Demotes the arena records {offset, length} (distinct, e->mu held) in the given order.
static int demote_records(cmb200_engine *e, const std::vector<std::pair<unsigned long long, uint32_t>> &recs) {
	cmb200_engine::HostTier &t = e->tier;
	const uint64_t cap = std::min<uint64_t>(t.size, (uint64_t)e->host_batch * e->bsize);   // bounce = one page-ring buffer
	size_t k = 0;
	std::vector<DemoteEntry> grp;
	std::vector<std::pair<uint64_t, uint32_t>> placed;
	while (k < recs.size()) {
		grp.clear(); placed.clear();
		const uint64_t start = t.head;
		uint64_t pos = start;
		while (k < recs.size() && grp.size() < e->max_batch) {
			const uint32_t len = recs[k].second, need = (len + 15u) & ~15u;
			uint64_t p = pos;
			if (p % t.size + need > t.size) p += t.size - p % t.size;     // no record straddles the end of the ring
			if (p + need - start > cap) break;
			grp.push_back(DemoteEntry{recs[k].first, p % t.size, p - start, len, 0});
			placed.emplace_back(p, need);
			pos = p + need;
			k++;
		}
		if (grp.empty()) { set_error_msg("cmb200_demote_batch: record larger than the bounce buffer"); return -1; }
		if (demote_group(e, grp, placed, start, pos)) return -1;
	}
	return 0;
}

extern "C" int cmb200_demote_batch(cmb200_engine *e, size_t n, const cmb200_addr *addr, uint64_t *demoted_out) {
	std::lock_guard<std::mutex> g(e->mu);
	if (demoted_out) *demoted_out = 0;
	if (!e->tier.host) { set_error_msg("cmb200_demote_batch: the engine has no host tier"); return -1; }
	CMB_CHECK(cudaSetDevice(e->device));
	harvest_pending(e, true);
	std::vector<int32_t> st(e->max_batch);
	std::vector<uint64_t> off(e->max_batch);
	std::vector<uint32_t> vl(e->max_batch);
	std::vector<std::pair<unsigned long long, uint32_t>> recs;
	uint64_t done = 0;
	for (size_t at = 0; at < n; at += e->max_batch) {
		const uint32_t m = (uint32_t)((n - at < e->max_batch) ? n - at : e->max_batch);
		if (lookup_chunk(e, addr + at, m, st.data(), off.data(), vl.data())) return -1;
		e->stats.kernel_launches++;
		// absent, remote and host-tier keys are skipped; a key named twice moves once
		recs.clear();
		std::unordered_set<uint64_t> seen;
		for (uint32_t i = 0; i < m; i++) {
			if (st[i] != ST_HIT || (off[i] & REC_HOST) || !seen.insert(off[i]).second) continue;
			const uint32_t clen = vl[i] - 1u;
			recs.emplace_back(off[i], 24u + (clen ? clen : e->bsize));
		}
		if (demote_records(e, recs)) return -1;
		done += recs.size();
	}
	if (demoted_out) *demoted_out = done;
	return 0;
}

// Moves every arena record to the host tier and compacts the arena (e->mu held): a snapshot that does
// not fit the arena continues into the tier.
static int demote_arena_all(cmb200_engine *e) {
	unsigned long long c[8];
	std::vector<ExportEntry> list;
	if (live_records(e, true, list, c) < 0) return -1;
	std::vector<std::pair<unsigned long long, uint32_t>> recs;
	for (const ExportEntry &x : list) recs.emplace_back(x.rec_off, x.len);
	if (demote_records(e, recs)) return -1;
	return compact_locked(e, nullptr);
}

// Promotion: the tier records of the named keys go back to free arena bytes above the bump pointer, in
// array order while they fit.  Nothing is evicted, demoted or compacted to make room; the caller does
// that first if it wants to (the drop-in's CMB200_TIER_PROMOTE).  See slot_publish in kernels.cu for
// why readers on other streams need no get_gate.
extern "C" int cmb200_promote_batch(cmb200_engine *e, size_t n, const cmb200_addr *addr, uint64_t *promoted_out) {
	std::lock_guard<std::mutex> g(e->mu);
	if (promoted_out) *promoted_out = 0;
	cmb200_engine::HostTier &t = e->tier;
	if (!t.host) { set_error_msg("cmb200_promote_batch: the engine has no host tier"); return -1; }
	CMB_CHECK(cudaSetDevice(e->device));
	harvest_pending(e, true);
	unsigned long long c[8];
	if (read_counters(e, c)) return -1;
	unsigned long long head = c[2];                  // a multiple of 16; past the end when a put overflowed
	std::vector<int32_t> st(e->max_batch);
	std::vector<uint64_t> off(e->max_batch);
	std::vector<uint32_t> vl(e->max_batch);
	std::vector<PromoteEntry> plan;
	uint64_t done = 0;
	bool full = false;
	for (size_t at = 0; at < n && !full; at += e->max_batch) {
		const uint32_t m = (uint32_t)((n - at < e->max_batch) ? n - at : e->max_batch);
		if (lookup_chunk(e, addr + at, m, st.data(), off.data(), vl.data())) return -1;
		e->stats.kernel_launches++;
		// absent, remote and arena keys are skipped; a key named twice moves once (a later chunk's
		// lookup runs after this chunk's promotion on the stream and finds it in the arena)
		plan.clear();
		std::unordered_set<uint64_t> seen;
		for (uint32_t i = 0; i < m; i++) {
			if (st[i] != ST_HIT || !(off[i] & REC_HOST) || !seen.insert(off[i]).second) continue;
			const uint32_t clen = vl[i] - 1u, len = 24u + (clen ? clen : e->bsize), need = (len + 15u) & ~15u;
			if (head + need > e->arena.size) { full = true; break; }
			plan.push_back(PromoteEntry{off[i] & ~REC_HOST, head, len, 0});
			head += need;
		}
		if (plan.empty()) continue;
		// the bump pointer moves past the new records before any of them is published
		CMB_CHECK(cudaMemcpyAsync(e->d_counters + 2, &head, 8, cudaMemcpyHostToDevice, e->st));
		CMB_CHECK(cudaMemcpyAsync(t.d_promote, plan.data(), plan.size() * sizeof(PromoteEntry), cudaMemcpyHostToDevice, e->st));
		if (launch_promote(e->table, e->arena, t.d_promote, (uint32_t)plan.size(), t.dev, e->st)) return -1;
		CMB_CHECK(cudaStreamSynchronize(e->st));
		e->stats.kernel_launches++;
		done += plan.size();
		t.promoted_records += plan.size();
		for (const PromoteEntry &p : plan) t.promoted_bytes += p.len;
	}
	if (promoted_out) *promoted_out = done;
	return 0;
}

// The hot log is read while gets go on appending to it, without the lock that puts take.  An entry
// read half-written, or one overwritten by a later lap, yields an address that is wrong or stale;
// that is harmless, since cmb200_promote_batch looks every address up again and checks its record.
extern "C" int cmb200_host_tier_hot(cmb200_engine *e, size_t max, cmb200_addr *addr_out, size_t *n_out, uint64_t *lost_out) {
	std::lock_guard<std::mutex> g(e->mu);
	*n_out = 0;
	if (lost_out) *lost_out = 0;
	cmb200_engine::HostTier &t = e->tier;
	if (!t.host) return 0;
	CMB_CHECK(cudaSetDevice(e->device));
	unsigned long long head = 0;
	std::vector<ulonglong2> ring(HOT_LOG_N);
	CMB_CHECK(cudaMemcpyAsync(&head, t.d_ctr + 2, 8, cudaMemcpyDeviceToHost, e->st));
	CMB_CHECK(cudaMemcpyAsync(ring.data(), t.d_hot, HOT_LOG_N * sizeof(ulonglong2), cudaMemcpyDeviceToHost, e->st));
	CMB_CHECK(cudaStreamSynchronize(e->st));
	const uint64_t since = head - t.hot_drained;
	const uint64_t from = since > HOT_LOG_N ? head - HOT_LOG_N : t.hot_drained;
	if (lost_out) *lost_out = since > HOT_LOG_N ? since - HOT_LOG_N : 0;
	t.hot_drained = head;
	std::set<std::pair<uint64_t, uint64_t>> seen;
	size_t k = 0;
	for (uint64_t p = head; p > from && k < max; p--) {        // newest first
		const ulonglong2 a = ring[(p - 1) % HOT_LOG_N];
		if (!seen.insert({a.x, a.y}).second) continue;
		addr_out[k].u = a.x; addr_out[k].l = a.y;
		k++;
	}
	*n_out = k;
	return 0;
}

extern "C" int cmb200_host_tier_stats(cmb200_engine *e, struct cmb200_host_tier_stats *out) {
	std::lock_guard<std::mutex> g(e->mu);
	memset(out, 0, sizeof(*out));
	const cmb200_engine::HostTier &t = e->tier;
	if (!t.host) return 0;
	unsigned long long c[8], d[2];
	if (read_counters(e, c)) return -1;
	CMB_CHECK(cudaMemcpy(d, t.d_ctr, sizeof(d), cudaMemcpyDeviceToHost));
	out->bytes = t.size;
	out->used = t.log.empty() ? 0 : t.head - t.log.front().first;
	out->records = c[7]; out->garbage = c[6];
	out->demoted_records = t.demoted_records; out->demoted_bytes = t.demoted_bytes;
	out->retired_records = d[0]; out->hits = d[1];
	out->promoted_records = t.promoted_records; out->promoted_bytes = t.promoted_bytes;
	return 0;
}

// ---- kernel-level entry points -------------------------------------------------------------
// Their device buffers, like the engine's page and stage buffers, end in 256 bytes of slack.

extern "C" int cmb200_compose_keys(int device, size_t n, const uint64_t *offset, const uint64_t *nhid,
    const uint32_t *genid, int pshift, cmb200_addr *addr_out, uint8_t *valid_out, uint64_t *key_out) {
	if (select_device(device)) return -1;
	DevMem<uint64_t> d_off, d_nh;
	DevMem<uint32_t> d_g;
	DevMem<unsigned long long> d_addr, d_key;
	DevMem<uint8_t> d_valid;
	if (d_off.alloc(n * 8 + 256) || d_nh.alloc(n * 8 + 256) || d_g.alloc(n * 4 + 256) || d_addr.alloc(n * 16 + 256) ||
	    d_valid.alloc(n + 256) || d_key.alloc(n * 8 + 256)) return -1;
	CMB_CHECK(cudaMemcpy(d_off, offset, n * 8, cudaMemcpyHostToDevice));
	CMB_CHECK(cudaMemcpy(d_nh, nhid, n * 8, cudaMemcpyHostToDevice));
	CMB_CHECK(cudaMemcpy(d_g, genid, n * 4, cudaMemcpyHostToDevice));
	if (launch_compose(d_off, d_nh, d_g, pshift, (uint32_t)n, d_addr, d_valid, d_key, 0)) return -1;
	CMB_CHECK(cudaMemcpy(addr_out, d_addr, n * 16, cudaMemcpyDeviceToHost));
	CMB_CHECK(cudaMemcpy(valid_out, d_valid, n, cudaMemcpyDeviceToHost));
	CMB_CHECK(cudaMemcpy(key_out, d_key, n * 8, cudaMemcpyDeviceToHost));
	return 0;
}

extern "C" int cmb200_lz4_encode_batch(int device, const void *pages_host, size_t n, uint32_t nbytes,
    size_t stride, int accel, void *blocks_out_host, size_t out_stride, int32_t *lens_out, uint64_t *fp_out) {
	if (select_device(device)) return -1;
	if (stride % 16 || stride < nbytes) { set_error_msg("encode_batch: stride must be a multiple of 16 and >= nbytes"); return -1; }
	size_t bound = (size_t)nbytes + nbytes / 255 + 16;
	size_t sstride = (bound + 15) & ~(size_t)15;
	if (out_stride < bound) { set_error_msg("encode_batch: out_stride below LZ4_compressBound"); return -1; }
	DevMem<uint8_t> d_in, d_stage;
	DevMem<int32_t> d_lens;
	DevMem<uint64_t> d_fps;
	DevMem<unsigned int> d_work;
	DevMem<uint32_t> d_order;
	if (d_in.alloc(n * stride + 256) || d_stage.alloc(n * sstride + 256) || d_lens.alloc(n * 4 + 256) ||
	    d_fps.alloc(n * 16 + 256) || d_work.alloc(64 + 256) || d_order.alloc(encode_order_words((uint32_t)n) * 4 + 256)) return -1;
	CMB_CHECK(cudaMemcpy(d_in, pages_host, n * stride, cudaMemcpyHostToDevice));
	EncodeJob job{};
	job.pages = d_in; job.page_stride = stride; job.nbytes = nbytes; job.n = (uint32_t)n;
	job.accel = accel < 0 ? 1u : (uint32_t)(accel > (1 << 20) ? (1 << 20) : accel);
	if (accel == 0) job.accel = 1;   // LZ4_compress_fast(accel<1) -> 1 (lz4.c:740); raw mode is a store-level notion
	job.stage = d_stage; job.stage_stride = sstride;
	job.lens = d_lens;
	job.fps = fp_out ? (uint64_t *)d_fps : nullptr;
	job.work = d_work;
	job.order = d_order;
	if (launch_encode(job, 0) < 0) return -1;
	CMB_CHECK(cudaMemcpy(lens_out, d_lens, n * 4, cudaMemcpyDeviceToHost));
	if (fp_out) CMB_CHECK(cudaMemcpy(fp_out, d_fps, n * 16, cudaMemcpyDeviceToHost));
	CMB_CHECK(cudaMemcpy2D(blocks_out_host, out_stride, d_stage, sstride, bound < out_stride ? bound : out_stride, n,
	    cudaMemcpyDeviceToHost));
	return 0;
}

extern "C" int cmb200_lz4_decode_batch(int device, const void *blocks_host, size_t in_stride, const int32_t *lens,
    size_t n, uint32_t nbytes, void *pages_out_host, int32_t *consumed_out) {
	if (select_device(device)) return -1;
	DevMem<uint8_t> d_blk, d_out;
	DevMem<int32_t> d_lens, d_used;
	if (d_blk.alloc(n * in_stride + 256) || d_lens.alloc(n * 4 + 256) || d_out.alloc(n * (size_t)nbytes + 256) ||
	    d_used.alloc(n * 4 + 256)) return -1;
	CMB_CHECK(cudaMemcpy(d_blk, blocks_host, n * in_stride, cudaMemcpyHostToDevice));
	CMB_CHECK(cudaMemcpy(d_lens, lens, n * 4, cudaMemcpyHostToDevice));
	CMB_CHECK(cudaMemset(d_out, 0, n * (size_t)nbytes));
	DecodeJob job{};
	job.n = (uint32_t)n; job.nbytes = nbytes; job.pages = d_out; job.status = d_used;
	job.blocks = d_blk; job.block_stride = in_stride; job.lens = d_lens;
	if (launch_decode(job, 0)) return -1;
	CMB_CHECK(cudaMemcpy(consumed_out, d_used, n * 4, cudaMemcpyDeviceToHost));
	CMB_CHECK(cudaMemcpy(pages_out_host, d_out, n * (size_t)nbytes, cudaMemcpyDeviceToHost));
	return 0;
}

extern "C" int cmb200_fingerprint_batch(int device, const void *pages_host, size_t n, uint32_t nbytes,
    size_t stride, uint64_t *fp_out) {
	if (select_device(device)) return -1;
	if (stride % 16) { set_error_msg("fingerprint_batch: stride must be a multiple of 16"); return -1; }
	DevMem<uint8_t> d_in;
	DevMem<uint64_t> d_fps;
	if (d_in.alloc(n * stride + 256) || d_fps.alloc(n * 16 + 256)) return -1;
	CMB_CHECK(cudaMemcpy(d_in, pages_host, n * stride, cudaMemcpyHostToDevice));
	if (launch_fingerprint(d_in, stride, nbytes, (uint32_t)n, d_fps, 0)) return -1;
	CMB_CHECK(cudaMemcpy(fp_out, d_fps, n * 16, cudaMemcpyDeviceToHost));
	return 0;
}

// EF128 of n resident pages (stand-alone form of the pass that k_encode fuses); the kernel's
// CUDA-event time is added to stats.fingerprint_kernel_ns.
extern "C" int cmb200_fingerprint_dev(cmb200_engine *e, size_t n, const void *pages_dev, uint64_t *fp_out_host) {
	std::lock_guard<std::mutex> g(e->mu);
	CMB_CHECK(cudaSetDevice(e->device));
	DevMem<uint64_t> d_fps;
	if (d_fps.alloc(n * 16 + 256)) return -1;
	CMB_CHECK(cudaEventRecord(e->t0[0], e->st));
	if (launch_fingerprint((const uint8_t *)pages_dev, e->bsize, e->bsize, (uint32_t)n, d_fps, e->st)) return -1;
	CMB_CHECK(cudaEventRecord(e->t1[0], e->st));
	CMB_CHECK(cudaMemcpyAsync(fp_out_host, d_fps, n * 16, cudaMemcpyDeviceToHost, e->st));
	CMB_CHECK(cudaStreamSynchronize(e->st));
	float ms = 0;
	CMB_CHECK(cudaEventElapsedTime(&ms, e->t0[0], e->t1[0]));
	e->stats.fingerprint_kernel_ns += (uint64_t)(ms * 1e6);
	e->stats.kernel_launches++;
	return 0;
}

// ---- synthetic streams -----------------------------------------------------------------------

extern "C" void cmb200_gen_chunk_host(uint64_t seed, uint64_t cid, uint32_t bsize, void *out) {
	uint64_t *w = (uint64_t *)out;
	for (uint32_t i = 0; i < bsize / 8; i++) w[i] = sg_chunk_word(seed, cid, bsize, i);
}

extern "C" int cmb200_gen_chunks_dev(cmb200_engine *e, uint64_t seed, const uint64_t *cids_host, size_t n, void *out_dev) {
	std::lock_guard<std::mutex> g(e->mu);
	CMB_CHECK(cudaSetDevice(e->device));
	DevMem<uint64_t> d_c;
	if (d_c.alloc(n * 8 + 256)) return -1;
	CMB_CHECK(cudaMemcpyAsync(d_c, cids_host, n * 8, cudaMemcpyHostToDevice, e->st));
	if (launch_streamgen(d_c, (uint32_t)n, seed, e->bsize, (uint8_t *)out_dev, e->st)) return -1;
	CMB_CHECK(cudaStreamSynchronize(e->st));
	return 0;
}

extern "C" uint64_t cmb200_gen_stream_ids(uint64_t seed2, size_t n, double dup, uint64_t first_cid, uint64_t *cid_out) {
	uint64_t state = seed2, distinct = 0;
	for (size_t k = 0; k < n; k++) {
		state += SG_GOLDEN;
		uint64_t r = sg_mix(state);
		bool repeat = distinct > 0 && (double)(r >> 11) * (1.0 / 9007199254740992.0) < dup;
		if (repeat) {
			state += SG_GOLDEN;
			cid_out[k] = first_cid + sg_mix(state) % distinct;
		} else {
			cid_out[k] = first_cid + distinct++;
		}
	}
	return distinct;
}

extern "C" void cmb200_gen_addr(uint64_t seed, uint64_t cid, int pshift, uint64_t *offset_out, uint64_t *nhid_out) {
	*offset_out = sg_offset(cid, pshift);
	*nhid_out = sg_nhid(seed, cid);
}
