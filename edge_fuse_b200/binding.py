"""ctypes binding of libcachemap.so.0.0 (include/cachemap.h, include/filemap.h,
include/cachemap_b200.h).  Mirrors the C API one to one; numpy arrays carry the buffers."""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None

MISS, HIT, INVALID, BAD_ENTRY, BAD_DECODE, REMOTE, CORRUPT, DROPPED = 0, 1, 2, 3, 4, 5, 6, 7
FINGERPRINT = 1
VERIFY = 2
TOUCH = 4       # a hit raises its record's timestamp: eviction by last access (CMB200_EVICT=access)

# every symbol the headers in include/ declare (checked by tests/test_abi.py)
EXPORTED_SYMBOLS = [
    # cachemap.h — reference cachemap/cachemap.h:33-47 + batch extension
    "cachemap_create", "cachemap_free", "cachemap_get", "cachemap_put", "cachemap_put_async",
    "cachemap_print_stats", "cachemap_put_batch", "cachemap_get_batch", "cachemap_put_batch_dev",
    "cachemap_get_batch_dev", "cachemap_get_counters", "cachemap_engine", "cachemap_engines",
    "cachemap_read_range", "cachemap_write_range", "cachemap_checkpoint", "cachemap_invalidate",
    "cachemap_pread", "cachemap_pwrite", "cachemap_rename",
    # filemap.h — reference cachemap/filemap.h:19-29
    "filemap_create", "filemap_free", "filemap_set", "filemap_unset", "filemap_get",
    "filemap_get_rand", "filemap_entries",
    # cachemap_b200.h
    "cmb200_last_error", "cmb200_device_count", "cmb200_engine_create", "cmb200_engine_destroy",
    "cmb200_host_alloc", "cmb200_host_free", "cmb200_dev_alloc", "cmb200_dev_free",
    "cmb200_memcpy_h2d", "cmb200_memcpy_d2h", "cmb200_stream", "cmb200_sync",
    "cmb200_put_batch", "cmb200_put_batch_dev", "cmb200_put_batch_async", "cmb200_wait", "cmb200_get_batch", "cmb200_get_batch_dev",
    "cmb200_unset_batch", "cmb200_entries", "cmb200_sample", "cmb200_read_records",
    "cmb200_read_fingerprints", "cmb200_get_stats", "cmb200_compose_keys",
    "cmb200_set_stream_order", "cmb200_locate_batch", "cmb200_save", "cmb200_load",
    "cmb200_put_step", "cmb200_import_records_dev", "cmb200_compact",
    "cmb200_get_small", "cmb200_get_small_begin", "cmb200_get_small_end", "cmb200_arena_ipc_handle", "cmb200_open_peer", "cmb200_close_peers",
    "cmb200_lz4_encode_batch", "cmb200_lz4_decode_batch", "cmb200_fingerprint_batch", "cmb200_fingerprint_dev",
    "cmb200_gen_chunk_host", "cmb200_gen_chunks_dev", "cmb200_gen_stream_ids", "cmb200_gen_addr",
    "cmb200_host_tier_enable", "cmb200_demote_batch", "cmb200_host_tier_stats",
    "cmb200_promote_batch", "cmb200_host_tier_hot", "cmb200_read_checkpoints",
    "cmb200_owner", "cmb200_save_set", "cmb200_load_set", "cmb200_move_pages", "cmb200_copy_peer",
    "cmb200_verify_stats", "cmb200_verify_store", "cmb200_snapshot_begin", "cmb200_snapshot_finish",
    "cmb200_chain_begin", "cmb200_load_chain", "cmb200_invalidate", "cmb200_patch_batch",
    "cmb200_rename", "cmb200_rename_set",
]


class Config(C.Structure):
    _fields_ = [("device", C.c_int), ("pshift", C.c_int), ("accel", C.c_int),
                ("capacity", C.c_uint64), ("arena_bytes", C.c_uint64), ("table_slots", C.c_uint64),
                ("max_batch", C.c_uint32), ("flags", C.c_uint32)]


class Stats(C.Structure):
    _fields_ = [(n, C.c_uint64) for n in (
        "entries", "table_slots", "tombstones", "arena_bytes", "arena_used", "arena_garbage",
        "dropped_puts", "remote_entries", "put_chunks", "get_requests", "get_hits", "kernel_launches",
        "encode_kernel_ns", "encode_kernel_launches", "decode_kernel_ns", "decode_kernel_launches",
        "fingerprint_kernel_ns")]


class HostTierStats(C.Structure):
    _fields_ = [(n, C.c_uint64) for n in (
        "bytes", "used", "records", "garbage", "demoted_records", "demoted_bytes", "retired_records", "hits",
        "promoted_records", "promoted_bytes")]


class VerifyStats(C.Structure):
    _fields_ = [(n, C.c_uint64) for n in ("verified", "unverified", "corrupt", "scanned", "scan_corrupt")]


def library_path() -> str:
    # CMB200_LIB: a differently tuned build of the same library (tools/build_variant.py)
    return os.environ.get("CMB200_LIB") or os.path.join(_HERE, "libcachemap.so.0.0")


def lib() -> C.CDLL:
    """Loads the library; raises if it has not been built (no fallback of any kind)."""
    global _LIB
    if _LIB is not None:
        return _LIB
    path = library_path()
    if not os.path.exists(path):
        raise RuntimeError(
            f"{path} is missing: build it with `python -m edge_fuse_b200.build` "
            "(the cachemap path is CUDA-only; there is no CPU fallback)")
    L = C.CDLL(path)
    vp, u64, u32, i32, sz = C.c_void_p, C.c_uint64, C.c_uint32, C.c_int, C.c_size_t
    sig = {
        "cachemap_create": (vp, [C.c_char_p, u64, i32, i32]),
        "cachemap_free": (None, [vp]),
        "cachemap_get": (vp, [vp, u64, u64, u32]),
        "cachemap_put": (None, [vp, u64, u64, u32, vp]),
        "cachemap_put_async": (None, [vp, u64, u64, u32, vp]),
        "cachemap_print_stats": (None, [vp]),
        "cachemap_put_batch": (None, [vp, u64, vp, vp, vp, vp]),
        "cachemap_get_batch": (None, [vp, u64, vp, vp, vp, vp, vp]),
        "cachemap_put_batch_dev": (None, [vp, u64, vp, vp, vp, vp]),
        "cachemap_get_batch_dev": (None, [vp, u64, vp, vp, vp, vp, vp]),
        "cachemap_get_counters": (None, [vp, vp, vp]),
        "cachemap_engine": (vp, [vp]),
        "cachemap_engines": (i32, [vp, vp, i32]),
        "cachemap_checkpoint": (i32, [vp]),
        "cachemap_invalidate": (u64, [vp, u64, u32, u64, u64]),
        "cachemap_rename": (u64, [vp, u64, u64, u32]),
        "cachemap_read_range": (i32, [vp, u64, u32, u64, sz, vp]),
        "cachemap_write_range": (None, [vp, u64, u32, u64, sz, vp]),
        "cachemap_pread": (i32, [vp, u64, u32, u64, sz, vp]),
        "cachemap_pwrite": (None, [vp, u64, u32, u64, sz, vp]),
        "filemap_create": (vp, [C.c_char_p, u64, i32, i32]),
        "filemap_free": (None, [vp]),
        "filemap_set": (None, [vp, vp, vp, u64]),
        "filemap_unset": (None, [vp, vp]),
        "filemap_get": (vp, [vp, vp]),
        "filemap_get_rand": (i32, [vp, vp, vp]),
        "filemap_entries": (u64, [vp]),
        "cmb200_last_error": (C.c_char_p, []),
        "cmb200_device_count": (i32, []),
        "cmb200_engine_create": (vp, [vp]),
        "cmb200_engine_destroy": (None, [vp]),
        "cmb200_host_alloc": (vp, [sz]),
        "cmb200_host_free": (None, [vp]),
        "cmb200_dev_alloc": (vp, [vp, sz]),
        "cmb200_dev_free": (None, [vp, vp]),
        "cmb200_memcpy_h2d": (i32, [vp, vp, vp, sz]),
        "cmb200_memcpy_d2h": (i32, [vp, vp, vp, sz]),
        "cmb200_stream": (vp, [vp]),
        "cmb200_sync": (i32, [vp]),
        "cmb200_put_batch": (i32, [vp, sz, vp, vp, vp, vp, vp]),
        "cmb200_put_batch_dev": (i32, [vp, sz, vp, vp, vp, vp, vp]),
        "cmb200_put_batch_async": (i32, [vp, sz, vp, vp, vp, vp, vp, vp]),
        "cmb200_wait": (i32, [vp, u64]),
        "cmb200_put_step": (i32, [vp, sz, vp, vp, vp, i32, vp, u32, vp, vp, vp]),
        "cmb200_import_records_dev": (i32, [vp, sz, vp, u32]),
        "cmb200_compact": (i32, [vp, vp]),
        "cmb200_save": (i32, [vp, C.c_char_p, vp]),
        "cmb200_load": (i32, [vp, C.c_char_p, vp]),
        "cmb200_get_batch": (i32, [vp, sz, vp, vp, vp, vp]),
        "cmb200_get_batch_dev": (i32, [vp, sz, vp, vp, vp, vp]),
        "cmb200_unset_batch": (i32, [vp, sz, vp]),
        "cmb200_invalidate": (i32, [vp, u64, u64, u64, vp]),
        "cmb200_rename": (i32, [vp, u64, u64, u64, u64, vp, vp]),
        "cmb200_rename_set": (i32, [vp, i32, u64, u64, u64, u64, vp, vp]),
        "cmb200_patch_batch": (i32, [vp, sz, vp, vp, vp, vp, vp, vp]),
        "cmb200_entries": (u64, [vp]),
        "cmb200_sample": (i32, [vp, sz, vp, vp, vp, vp]),
        "cmb200_read_records": (i32, [vp, sz, vp, vp, sz, vp]),
        "cmb200_read_fingerprints": (i32, [vp, sz, vp, vp, vp]),
        "cmb200_get_stats": (i32, [vp, vp]),
        "cmb200_set_stream_order": (i32, [vp, u64, u64]),
        "cmb200_get_small": (i32, [vp, sz, vp, vp, vp]),
        "cmb200_get_small_begin": (i32, [vp, sz, vp, vp, vp]),
        "cmb200_get_small_end": (i32, [vp, vp, vp]),
        "cmb200_arena_ipc_handle": (i32, [vp, vp, vp]),
        "cmb200_open_peer": (i32, [vp, C.c_uint32, vp, C.c_uint64]),
        "cmb200_close_peers": (i32, [vp]),
        "cmb200_locate_batch": (i32, [vp, sz, vp, vp, vp]),
        "cmb200_compose_keys": (i32, [i32, sz, vp, vp, vp, i32, vp, vp, vp]),
        "cmb200_lz4_encode_batch": (i32, [i32, vp, sz, u32, sz, i32, vp, sz, vp, vp]),
        "cmb200_lz4_decode_batch": (i32, [i32, vp, sz, vp, sz, u32, vp, vp]),
        "cmb200_fingerprint_batch": (i32, [i32, vp, sz, u32, sz, vp]),
        "cmb200_fingerprint_dev": (i32, [vp, sz, vp, vp]),
        "cmb200_gen_chunk_host": (None, [u64, u64, u32, vp]),
        "cmb200_gen_chunks_dev": (i32, [vp, u64, vp, sz, vp]),
        "cmb200_gen_stream_ids": (u64, [u64, sz, C.c_double, u64, vp]),
        "cmb200_gen_addr": (None, [u64, u64, i32, vp, vp]),
        "cmb200_host_tier_enable": (i32, [vp, u64]),
        "cmb200_demote_batch": (i32, [vp, sz, vp, vp]),
        "cmb200_host_tier_stats": (i32, [vp, vp]),
        "cmb200_promote_batch": (i32, [vp, sz, vp, vp]),
        "cmb200_host_tier_hot": (i32, [vp, sz, vp, vp, vp]),
        "cmb200_read_checkpoints": (i32, [vp, sz, vp, vp, vp]),
        "cmb200_owner": (i32, [u64, i32]),
        "cmb200_save_set": (i32, [vp, i32, C.c_char_p, vp]),
        "cmb200_load_set": (i32, [vp, i32, C.c_char_p, vp]),
        "cmb200_move_pages": (i32, [vp, sz, vp, vp, vp, vp]),
        "cmb200_copy_peer": (i32, [vp, vp, vp, vp, sz]),
        "cmb200_verify_stats": (i32, [vp, vp]),
        "cmb200_verify_store": (i32, [vp, sz, vp, vp, vp]),
        "cmb200_snapshot_begin": (vp, [vp, i32, C.c_char_p]),
        "cmb200_snapshot_finish": (i32, [vp, vp]),
        "cmb200_chain_begin": (vp, [vp, i32, C.c_char_p, i32]),
        "cmb200_load_chain": (i32, [vp, i32, C.c_char_p, vp, vp]),
    }
    for name, (res, args) in sig.items():
        fn = getattr(L, name)
        fn.restype = res
        fn.argtypes = args
    _LIB = L
    return L


def last_error() -> str:
    return (lib().cmb200_last_error() or b"").decode()


def device_count() -> int:
    return int(lib().cmb200_device_count())


def _check(rc: int, what: str) -> None:
    if rc != 0:
        raise RuntimeError(f"{what} failed: {last_error()}")


def _ptr(a):
    if a is None:
        return None
    if isinstance(a, np.ndarray):
        assert a.flags["C_CONTIGUOUS"]
        return a.ctypes.data
    return a  # raw integer address (device or pinned pointer)


def _addr_array(u, l) -> np.ndarray:
    a = np.empty((len(u), 2), dtype=np.uint64)
    a[:, 0] = u
    a[:, 1] = l
    return a


# ---- kernel-level entry points ------------------------------------------------------------------

def compose_keys(offset, nhid, genid, pshift: int, device: int = -1):
    """cachemap.c:151-166 + filemap.c:18-24 on the GPU -> (addr[n,2], valid[n], key[n])."""
    offset = np.ascontiguousarray(offset, dtype=np.uint64)
    nhid = np.ascontiguousarray(nhid, dtype=np.uint64)
    genid = np.ascontiguousarray(genid, dtype=np.uint32)
    n = len(offset)
    addr = np.zeros((n, 2), dtype=np.uint64)
    valid = np.zeros(n, dtype=np.uint8)
    key = np.zeros(n, dtype=np.uint64)
    _check(lib().cmb200_compose_keys(device, n, _ptr(offset), _ptr(nhid), _ptr(genid), pshift,
                                     _ptr(addr), _ptr(valid), _ptr(key)), "cmb200_compose_keys")
    return addr, valid, key


def lz4_encode_batch(pages: np.ndarray, nbytes: int | None = None, accel: int = 12,
                     fingerprints: bool = False, device: int = -1):
    """pages[n, stride] uint8 -> (list of block bytes, fp[n,2] or None)."""
    pages = np.ascontiguousarray(pages, dtype=np.uint8)
    n, stride = pages.shape
    nbytes = stride if nbytes is None else nbytes
    out_stride = (nbytes + nbytes // 255 + 16 + 15) // 16 * 16
    blocks = np.zeros((n, out_stride), dtype=np.uint8)
    lens = np.zeros(n, dtype=np.int32)
    fps = np.zeros((n, 2), dtype=np.uint64) if fingerprints else None
    _check(lib().cmb200_lz4_encode_batch(device, _ptr(pages), n, nbytes, stride, accel, _ptr(blocks),
                                         out_stride, _ptr(lens), _ptr(fps)), "cmb200_lz4_encode_batch")
    return [blocks[i, :lens[i]].tobytes() for i in range(n)], fps


def lz4_decode_batch(blocks: list[bytes], nbytes: int, device: int = -1):
    """-> (pages[n, nbytes], consumed[n])."""
    n = len(blocks)
    stride = (max(len(b) for b in blocks) + 15) // 16 * 16 if n else 16
    buf = np.zeros((n, stride), dtype=np.uint8)
    lens = np.zeros(n, dtype=np.int32)
    for i, b in enumerate(blocks):
        buf[i, :len(b)] = np.frombuffer(b, dtype=np.uint8)
        lens[i] = len(b)
    pages = np.zeros((n, nbytes), dtype=np.uint8)
    used = np.zeros(n, dtype=np.int32)
    _check(lib().cmb200_lz4_decode_batch(device, _ptr(buf), stride, _ptr(lens), n, nbytes, _ptr(pages),
                                         _ptr(used)), "cmb200_lz4_decode_batch")
    return pages, used


def fingerprint_batch(pages: np.ndarray, nbytes: int | None = None, device: int = -1) -> np.ndarray:
    pages = np.ascontiguousarray(pages, dtype=np.uint8)
    n, stride = pages.shape
    nbytes = stride if nbytes is None else nbytes
    fps = np.zeros((n, 2), dtype=np.uint64)
    _check(lib().cmb200_fingerprint_batch(device, _ptr(pages), n, nbytes, stride, _ptr(fps)),
           "cmb200_fingerprint_batch")
    return fps


# ---- synthetic streams --------------------------------------------------------------------------

def gen_chunk_host(seed: int, cid: int, bsize: int) -> np.ndarray:
    out = np.empty(bsize, dtype=np.uint8)
    lib().cmb200_gen_chunk_host(seed, cid, bsize, _ptr(out))
    return out


def gen_stream_ids(n: int, dup: float, seed2: int = 43, first_cid: int = 0):
    cids = np.zeros(n, dtype=np.uint64)
    distinct = lib().cmb200_gen_stream_ids(seed2, n, dup, first_cid, _ptr(cids))
    return cids, int(distinct)


def gen_addr(seed: int, cids, pshift: int):
    cids = np.asarray(cids, dtype=np.uint64)
    off = np.zeros(len(cids), dtype=np.uint64)
    nh = np.zeros(len(cids), dtype=np.uint64)
    o, h = C.c_uint64(), C.c_uint64()
    for i, c in enumerate(cids):
        lib().cmb200_gen_addr(seed, int(c), pshift, C.byref(o), C.byref(h))
        off[i], nh[i] = o.value, h.value
    return off, nh


# ---- engine -------------------------------------------------------------------------------------

def engine_stats(handle) -> dict:
    """cmb200_get_stats of an engine handle (Engine.h, or cachemap_engine(cm) of the drop-in)."""
    st = Stats()
    _check(lib().cmb200_get_stats(handle, C.byref(st)), "cmb200_get_stats")
    return {n: int(getattr(st, n)) for n, _ in Stats._fields_}


def host_tier_stats(handle) -> dict:
    """cmb200_host_tier_stats of an engine handle (all zero without a tier)."""
    st = HostTierStats()
    _check(lib().cmb200_host_tier_stats(handle, C.byref(st)), "cmb200_host_tier_stats")
    return {n: int(getattr(st, n)) for n, _ in HostTierStats._fields_}


def verify_stats(handle) -> dict:
    """cmb200_verify_stats of an engine handle (all zero for an engine created without VERIFY)."""
    st = VerifyStats()
    _check(lib().cmb200_verify_stats(handle, C.byref(st)), "cmb200_verify_stats")
    return {n: int(getattr(st, n)) for n, _ in VerifyStats._fields_}


def read_checkpoints(handle, u, l):
    """cmb200_read_checkpoints of an engine handle -> (words [n, 16] uint32, ok [n] int32): word 0 is
    the tag as stored; ok 1 = valid checkpoints, 0 = a record without them, -1 = absent, remote or
    no side table."""
    addr = _addr_array(u, l)
    n = len(addr)
    words = np.zeros((n, 16), dtype=np.uint32)
    ok = np.zeros(n, dtype=np.int32)
    _check(lib().cmb200_read_checkpoints(handle, n, _ptr(addr), _ptr(words), _ptr(ok)), "cmb200_read_checkpoints")
    return words, ok


class Engine:
    """cmb200_engine: the filemap-level batch API (addresses are (u, l) pairs).  host_tier_bytes > 0
    gives the engine a host tier of that size (cmb200_host_tier_enable)."""

    def __init__(self, pshift: int = 16, accel: int = 12, capacity: int = 1024, arena_bytes: int = 0,
                 table_slots: int = 0, max_batch: int = 0, flags: int = 0, device: int = -1,
                 host_tier_bytes: int = 0):
        cfg = Config(device, pshift, accel, capacity, arena_bytes, table_slots, max_batch, flags)
        self.h = lib().cmb200_engine_create(C.byref(cfg))
        if not self.h:
            raise RuntimeError(f"cmb200_engine_create failed: {last_error()}")
        self.bsize = 1 << pshift
        if host_tier_bytes:
            try:
                self.enable_host_tier(host_tier_bytes)
            except RuntimeError:
                self.close()
                raise

    def enable_host_tier(self, nbytes: int):
        _check(lib().cmb200_host_tier_enable(self.h, nbytes), "cmb200_host_tier_enable")

    def demote(self, u, l) -> int:
        """cmb200_demote_batch: moves the keys' arena records to the host tier -> how many moved."""
        addr = _addr_array(u, l)
        n = C.c_uint64(0)
        _check(lib().cmb200_demote_batch(self.h, len(addr), _ptr(addr), C.byref(n)), "cmb200_demote_batch")
        return n.value

    def promote(self, u, l) -> int:
        """cmb200_promote_batch: moves the keys' host-tier records back to free arena bytes, in order
        while they fit -> how many moved."""
        addr = _addr_array(u, l)
        n = C.c_uint64(0)
        _check(lib().cmb200_promote_batch(self.h, len(addr), _ptr(addr), C.byref(n)), "cmb200_promote_batch")
        return n.value

    def tier_hot(self, max_n: int = 4096):
        """cmb200_host_tier_hot -> (u, l, lost): addresses read from the host tier since the last call,
        newest first, distinct, at most max_n; lost = hits the log overwrote before this drain."""
        addr = np.zeros((max(1, max_n), 2), dtype=np.uint64)
        n, lost = C.c_size_t(0), C.c_uint64(0)
        _check(lib().cmb200_host_tier_hot(self.h, max_n, _ptr(addr), C.byref(n), C.byref(lost)), "cmb200_host_tier_hot")
        return addr[:n.value, 0].copy(), addr[:n.value, 1].copy(), lost.value

    def host_tier_stats(self) -> dict:
        return host_tier_stats(self.h)

    def verify_stats(self) -> dict:
        return verify_stats(self.h)

    def verify_store(self, max_bad: int = 4096):
        """cmb200_verify_store -> (u, l, n_bad, checked): the addresses of the first max_bad records
        whose page does not match its stored EF128 or does not decode, how many such records there
        are, and how many records had a fingerprint to compare with."""
        addr = np.zeros((max(1, max_bad), 2), dtype=np.uint64)
        n, checked = C.c_size_t(0), C.c_uint64(0)
        _check(lib().cmb200_verify_store(self.h, max_bad, _ptr(addr), C.byref(n), C.byref(checked)),
               "cmb200_verify_store")
        k = min(n.value, max_bad)
        return addr[:k, 0].copy(), addr[:k, 1].copy(), int(n.value), int(checked.value)

    def close(self):
        if self.h:
            lib().cmb200_engine_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def put(self, u, l, pages, ts=None, valid=None, on_dev=False):
        addr = _addr_array(u, l)
        n = len(addr)
        lens = np.zeros(n, dtype=np.int32)
        ts = None if ts is None else np.ascontiguousarray(ts, dtype=np.uint64)
        valid = None if valid is None else np.ascontiguousarray(valid, dtype=np.uint8)
        fn = lib().cmb200_put_batch_dev if on_dev else lib().cmb200_put_batch
        _check(fn(self.h, n, _ptr(addr), _ptr(valid), _ptr(pages), _ptr(ts), _ptr(lens)), "cmb200_put_batch")
        return lens

    def put_async(self, u, l, pages, ts=None, valid=None, lens=None) -> int:
        """cmb200_put_batch_async -> ticket for wait().  pages are host memory; `lens`, if given,
        must be page-locked int32 storage that stays alive until wait(ticket)."""
        addr = _addr_array(u, l)
        ts = None if ts is None else np.ascontiguousarray(ts, dtype=np.uint64)
        valid = None if valid is None else np.ascontiguousarray(valid, dtype=np.uint8)
        t = C.c_uint64(0)
        _check(lib().cmb200_put_batch_async(self.h, len(addr), _ptr(addr), _ptr(valid), _ptr(pages), _ptr(ts),
                                            _ptr(lens), C.byref(t)), "cmb200_put_batch_async")
        return t.value

    def put_step(self, u, l, pages, ts=None, valid=None, on_dev=False, rank=0, records_dev=None, lens=None) -> int:
        """cmb200_put_step: asynchronous put of one step of a sharded stream; exchange records are
        written to the device buffer `records_dev` (n x 32 bytes).  on_dev: False = host pages,
        reusable on return; True = device pages; 2 = page-locked host pages the caller keeps
        untouched until wait(ticket).  -> ticket."""
        addr = _addr_array(u, l)
        ts = None if ts is None else np.ascontiguousarray(ts, dtype=np.uint64)
        valid = None if valid is None else np.ascontiguousarray(valid, dtype=np.uint8)
        t = C.c_uint64(0)
        _check(lib().cmb200_put_step(self.h, len(addr), _ptr(addr), _ptr(valid), _ptr(pages), int(on_dev), _ptr(ts),
                                     rank, _ptr(records_dev), _ptr(lens), C.byref(t)), "cmb200_put_step")
        return t.value

    def import_records_dev(self, n_total: int, records_dev, my_rank: int):
        _check(lib().cmb200_import_records_dev(self.h, n_total, _ptr(records_dev), my_rank), "cmb200_import_records_dev")

    def wait(self, ticket: int):
        _check(lib().cmb200_wait(self.h, ticket), "cmb200_wait")

    def get(self, u, l, valid=None, out=None, on_dev=False):
        addr = _addr_array(u, l)
        n = len(addr)
        status = np.zeros(n, dtype=np.int32)
        valid = None if valid is None else np.ascontiguousarray(valid, dtype=np.uint8)
        if out is None:
            out = np.zeros((n, self.bsize), dtype=np.uint8)
        fn = lib().cmb200_get_batch_dev if on_dev else lib().cmb200_get_batch
        _check(fn(self.h, n, _ptr(addr), _ptr(valid), _ptr(out), _ptr(status)), "cmb200_get_batch")
        return out, status

    def get_small(self, u, l, out=None):
        """cmb200_get_small: the fused small-batch get.  `out` = page-locked host pointer / device
        pointer (int) or None (a page-locked buffer is allocated and copied into a numpy array)."""
        addr = _addr_array(u, l)
        n = len(addr)
        status = np.zeros(n, dtype=np.int32)
        own = None
        if out is None:
            own = lib().cmb200_host_alloc(max(1, n) * self.bsize)
            if not own:
                raise RuntimeError("cmb200_host_alloc failed")
            out = own
        try:
            _check(lib().cmb200_get_small(self.h, n, _ptr(addr), _ptr(out), _ptr(status)), "cmb200_get_small")
            if own:
                arr = np.ctypeslib.as_array((C.c_uint8 * (n * self.bsize)).from_address(own)).reshape(n, self.bsize).copy()
                return arr, status
            return out, status
        finally:
            if own:
                lib().cmb200_host_free(own)

    def arena_ipc_handle(self):
        h = (C.c_uint8 * 64)()
        size = C.c_uint64(0)
        _check(lib().cmb200_arena_ipc_handle(self.h, h, C.byref(size)), "cmb200_arena_ipc_handle")
        return bytes(h), int(size.value)

    def open_peer(self, rank: int, handle: bytes, arena_bytes: int):
        buf = (C.c_uint8 * 64).from_buffer_copy(handle)
        _check(lib().cmb200_open_peer(self.h, rank, buf, arena_bytes), "cmb200_open_peer")

    def close_peers(self):
        _check(lib().cmb200_close_peers(self.h), "cmb200_close_peers")

    def unset(self, u, l):
        addr = _addr_array(u, l)
        _check(lib().cmb200_unset_batch(self.h, len(addr), _ptr(addr)), "cmb200_unset_batch")

    def invalidate(self, u: int, l_first: int, l_last: int) -> int:
        """Removes every live record stored at {u, l} with l_first <= l <= l_last -> records removed."""
        removed = C.c_uint64()
        _check(lib().cmb200_invalidate(self.h, u, l_first, l_last, C.byref(removed)), "cmb200_invalidate")
        return removed.value

    def rename(self, u_from: int, u_to: int, l_first: int, l_last: int):
        """Moves every live record stored at {u_from, l}, l_first <= l <= l_last, to {u_to, l}
        -> (records moved, records dropped for lack of arena room)."""
        moved, dropped = C.c_uint64(), C.c_uint64()
        _check(lib().cmb200_rename(self.h, u_from, u_to, l_first, l_last, C.byref(moved), C.byref(dropped)),
               "cmb200_rename")
        return moved.value, dropped.value

    def patch(self, u, l, page_off, data, ts=None):
        """cmb200_patch_batch: patch i writes data[i] (bytes) at byte page_off[i] of the page stored at
        {u[i], l[i]}, in array order -> status per patch (HIT, MISS, BAD_ENTRY, BAD_DECODE, CORRUPT, DROPPED)."""
        addr = _addr_array(u, l)
        n = len(addr)
        off = np.ascontiguousarray(page_off, dtype=np.uint32)
        lens = np.array([len(d) for d in data], dtype=np.uint32)
        blob = np.frombuffer(b"".join(bytes(d) for d in data) or b"\0", dtype=np.uint8)
        ts = None if ts is None else np.ascontiguousarray(ts, dtype=np.uint64)
        status = np.zeros(n, dtype=np.int32)
        _check(lib().cmb200_patch_batch(self.h, n, _ptr(addr), _ptr(off), _ptr(lens), _ptr(blob), _ptr(ts),
                                        _ptr(status)), "cmb200_patch_batch")
        return status

    def entries(self) -> int:
        return int(lib().cmb200_entries(self.h))

    def sample(self, r):
        r = np.ascontiguousarray(r, dtype=np.uint64)
        n = len(r)
        addr = np.zeros((n, 2), dtype=np.uint64)
        ts = np.zeros(n, dtype=np.uint64)
        ok = np.zeros(n, dtype=np.int32)
        _check(lib().cmb200_sample(self.h, n, _ptr(r), _ptr(addr), _ptr(ts), _ptr(ok)), "cmb200_sample")
        return addr, ts, ok

    def read_records_raw(self, u, l):
        """-> (records [n, 24 + bsize + 1024] uint8, lens [n] int32; -1 = no record): the stored
        filemap records {data_prefix, payload} as they lie in the arena."""
        addr = _addr_array(u, l)
        n = len(addr)
        stride = 24 + self.bsize + 1024
        out = np.zeros((n, stride), dtype=np.uint8)
        lens = np.zeros(n, dtype=np.int32)
        _check(lib().cmb200_read_records(self.h, n, _ptr(addr), _ptr(out), stride, _ptr(lens)),
               "cmb200_read_records")
        return out, lens

    def read_records(self, u, l):
        out, lens = self.read_records_raw(u, l)
        return [out[i, :lens[i]].tobytes() if lens[i] >= 0 else None for i in range(len(lens))]

    def read_fingerprints(self, u, l):
        addr = _addr_array(u, l)
        n = len(addr)
        fps = np.zeros((n, 2), dtype=np.uint64)
        ok = np.zeros(n, dtype=np.int32)
        _check(lib().cmb200_read_fingerprints(self.h, n, _ptr(addr), _ptr(fps), _ptr(ok)),
               "cmb200_read_fingerprints")
        return fps, ok

    def read_checkpoints(self, u, l):
        return read_checkpoints(self.h, u, l)

    def compact(self) -> int:
        """cmb200_compact -> bytes of arena reclaimed."""
        n = C.c_uint64(0)
        _check(lib().cmb200_compact(self.h, C.byref(n)), "cmb200_compact")
        return n.value

    def save(self, path: str) -> int:
        n = C.c_uint64(0)
        _check(lib().cmb200_save(self.h, path.encode(), C.byref(n)), "cmb200_save")
        return n.value

    def load(self, path: str) -> int:
        n = C.c_uint64(0)
        _check(lib().cmb200_load(self.h, path.encode(), C.byref(n)), "cmb200_load")
        return n.value

    def snapshot_begin(self, path: str) -> int:
        """cmb200_snapshot_begin of this engine alone -> handle for snapshot_finish."""
        return snapshot_begin([self.h], path)

    def move_pages(self, n: int, dst_dev: int, src_dev: int, dst_idx=None, src_idx=None):
        """cmb200_move_pages: dst[dst_idx[i] or i] = src[src_idx[i] or i], n pages in this engine's HBM."""
        di = None if dst_idx is None else np.ascontiguousarray(dst_idx, dtype=np.uint32)
        si = None if src_idx is None else np.ascontiguousarray(src_idx, dtype=np.uint32)
        _check(lib().cmb200_move_pages(self.h, n, dst_dev, _ptr(di), src_dev, _ptr(si)), "cmb200_move_pages")

    def set_stream_order(self, next_seq: int, stride: int):
        _check(lib().cmb200_set_stream_order(self.h, next_seq, stride), "cmb200_set_stream_order")

    def locate(self, u, l):
        addr = _addr_array(u, l)
        status = np.zeros(len(addr), dtype=np.int32)
        owner = np.zeros(len(addr), dtype=np.uint64)
        _check(lib().cmb200_locate_batch(self.h, len(addr), _ptr(addr), _ptr(status), _ptr(owner)),
               "cmb200_locate_batch")
        return status, owner

    def fingerprint_dev(self, n: int, pages_dev: int) -> np.ndarray:
        fps = np.zeros((n, 2), dtype=np.uint64)
        _check(lib().cmb200_fingerprint_dev(self.h, n, pages_dev, _ptr(fps)), "cmb200_fingerprint_dev")
        return fps

    def stats(self) -> dict:
        return engine_stats(self.h)

    def stream(self) -> int:
        return int(lib().cmb200_stream(self.h) or 0)

    def sync(self):
        _check(lib().cmb200_sync(self.h), "cmb200_sync")

    def dev_alloc(self, nbytes: int) -> int:
        p = lib().cmb200_dev_alloc(self.h, nbytes)
        if not p:
            raise RuntimeError(f"cmb200_dev_alloc({nbytes}) failed: {last_error()}")
        return int(p)

    def dev_free(self, p: int):
        lib().cmb200_dev_free(self.h, p)

    def h2d(self, dev: int, host: np.ndarray):
        _check(lib().cmb200_memcpy_h2d(self.h, dev, _ptr(host), host.nbytes), "cmb200_memcpy_h2d")

    def d2h(self, host: np.ndarray, dev: int):
        _check(lib().cmb200_memcpy_d2h(self.h, _ptr(host), dev, host.nbytes), "cmb200_memcpy_d2h")

    def gen_chunks_dev(self, seed: int, cids, out_dev: int):
        cids = np.ascontiguousarray(cids, dtype=np.uint64)
        _check(lib().cmb200_gen_chunks_dev(self.h, seed, _ptr(cids), len(cids), out_dev), "cmb200_gen_chunks_dev")


def owner(key: int, g: int) -> int:
    """cmb200_owner: which of g engines holds the store key `key` (FNV-1a-64 of the address)."""
    return int(lib().cmb200_owner(key, g))


def _handles(handles):
    arr = (C.c_void_p * len(handles))(*handles)
    return arr, len(handles)


def save_set(handles, path: str) -> int:
    """cmb200_save_set over engine handles -> records written."""
    arr, g = _handles(handles)
    n = C.c_uint64(0)
    _check(lib().cmb200_save_set(arr, g, path.encode(), C.byref(n)), "cmb200_save_set")
    return n.value


def rename_set(handles, u_from: int, u_to: int, l_first: int, l_last: int):
    """cmb200_rename_set over engine handles that split the keys by cmb200_owner -> (moved, dropped)."""
    arr, g = _handles(handles)
    moved, dropped = C.c_uint64(), C.c_uint64()
    _check(lib().cmb200_rename_set(arr, g, u_from, u_to, l_first, l_last, C.byref(moved), C.byref(dropped)),
           "cmb200_rename_set")
    return moved.value, dropped.value


def snapshot_begin(handles, path: str) -> int:
    """cmb200_snapshot_begin over engine handles -> snapshot handle.  The engines' live records are
    listed now and written by a thread of the snapshot while the engines keep serving."""
    arr, g = _handles(handles)
    s = lib().cmb200_snapshot_begin(arr, g, path.encode())
    if not s:
        raise RuntimeError(f"cmb200_snapshot_begin failed: {last_error()}")
    return int(s)


def snapshot_finish(s: int) -> int:
    """cmb200_snapshot_finish: waits for the writer and renames the file into place -> records written.
    The handle is freed, whatever the outcome."""
    n = C.c_uint64(0)
    _check(lib().cmb200_snapshot_finish(s, C.byref(n)), "cmb200_snapshot_finish")
    return n.value


def load_set(handles, path: str) -> int:
    """cmb200_load_set over engine handles -> records loaded."""
    arr, g = _handles(handles)
    n = C.c_uint64(0)
    _check(lib().cmb200_load_set(arr, g, path.encode(), C.byref(n)), "cmb200_load_set")
    return n.value


def chain_begin(handles, base_path: str, delta: bool) -> int:
    """cmb200_chain_begin over engine handles -> snapshot handle for snapshot_finish.  delta=False
    writes a base at base_path with a fresh chain id, delta=True the chain's next base_path.d<k>."""
    arr, g = _handles(handles)
    s = lib().cmb200_chain_begin(arr, g, base_path.encode(), int(bool(delta)))
    if not s:
        raise RuntimeError(f"cmb200_chain_begin failed: {last_error()}")
    return int(s)


def load_chain(handles, base_path: str):
    """cmb200_load_chain over engine handles -> (records loaded, deltas applied)."""
    arr, g = _handles(handles)
    n = C.c_uint64(0)
    k = C.c_uint32(0)
    _check(lib().cmb200_load_chain(arr, g, base_path.encode(), C.byref(n), C.byref(k)), "cmb200_load_chain")
    return n.value, k.value


class Cachemap:
    """The reference's cachemap API (cachemap/cachemap.h:33-47) plus the batch extension.  The engine
    starts on first use and reads its settings from the environment then, the host tier included
    (CMB200_HOST_TIER_MB, INTEGRATION.md)."""

    def __init__(self, destdir: str, capacity: int, comp_accel: int = 12, pshift: int = 16):
        self.h = lib().cachemap_create(destdir.encode(), capacity, comp_accel, pshift)
        self.bsize = 1 << pshift
        self.pshift = pshift

    @property
    def ok(self) -> bool:
        return bool(self.h)

    def free(self):
        if self.h:
            lib().cachemap_free(self.h)
            self.h = None

    def put(self, offset: int, nhid: int, genid: int, page: np.ndarray, async_: bool = False):
        page = np.ascontiguousarray(page, dtype=np.uint8)
        assert page.size == self.bsize
        (lib().cachemap_put_async if async_ else lib().cachemap_put)(self.h, offset, nhid, genid, _ptr(page))

    def get(self, offset: int, nhid: int, genid: int):
        """-> page bytes or None; the malloc()ed buffer of the C API is freed here."""
        p = lib().cachemap_get(self.h, offset, nhid, genid)
        if not p:
            return None
        data = C.string_at(p, self.bsize)
        _libc().free(C.c_void_p(p))
        return data

    def put_batch(self, offset, nhid, genid, pages, on_dev=False):
        offset = np.ascontiguousarray(offset, dtype=np.uint64)
        nhid = np.ascontiguousarray(nhid, dtype=np.uint64)
        genid = np.ascontiguousarray(genid, dtype=np.uint32)
        fn = lib().cachemap_put_batch_dev if on_dev else lib().cachemap_put_batch
        fn(self.h, len(offset), _ptr(offset), _ptr(nhid), _ptr(genid), _ptr(pages))

    def get_batch(self, offset, nhid, genid, out=None, on_dev=False):
        offset = np.ascontiguousarray(offset, dtype=np.uint64)
        nhid = np.ascontiguousarray(nhid, dtype=np.uint64)
        genid = np.ascontiguousarray(genid, dtype=np.uint32)
        n = len(offset)
        hit = np.zeros(n, dtype=np.uint8)
        if out is None:
            out = np.zeros((n, self.bsize), dtype=np.uint8)
        fn = lib().cachemap_get_batch_dev if on_dev else lib().cachemap_get_batch
        fn(self.h, n, _ptr(offset), _ptr(nhid), _ptr(genid), _ptr(out), _ptr(hit))
        return out, hit

    def read_range(self, nhid: int, genid: int, off: int, size: int):
        """The page loop of edgefs_read (edgefs.c:1159-1178) as one call -> bytes or None."""
        out = np.zeros(max(size, 1), dtype=np.uint8)
        ok = lib().cachemap_read_range(self.h, nhid, genid, off, size, _ptr(out))
        return out[:size].tobytes() if ok else None

    def write_range(self, nhid: int, genid: int, off: int, data):
        """The put loop of edgefs_read's miss path / edgefs_write (edgefs.c:1183-1195,1216-1228)."""
        data = np.ascontiguousarray(np.frombuffer(data, dtype=np.uint8) if isinstance(data, (bytes, bytearray)) else data)
        lib().cachemap_write_range(self.h, nhid, genid, off, data.size, _ptr(data))

    def pread(self, nhid: int, genid: int, off: int, size: int):
        """Any byte range [off, off + size) -> bytes when every page it overlaps hits, else None."""
        out = np.zeros(max(size, 1), dtype=np.uint8)
        ok = lib().cachemap_pread(self.h, nhid, genid, off, size, _ptr(out))
        return out[:size].tobytes() if ok else None

    def pwrite(self, nhid: int, genid: int, off: int, data):
        """Any byte range: whole pages put, cached pages covered in part patched, the rest left uncached."""
        data = np.ascontiguousarray(np.frombuffer(data, dtype=np.uint8) if isinstance(data, (bytes, bytearray)) else data)
        lib().cachemap_pwrite(self.h, nhid, genid, off, data.size, _ptr(data))

    def checkpoint(self) -> int:
        return int(lib().cachemap_checkpoint(self.h))

    TO_END = (1 << 64) - 1

    def invalidate(self, nhid: int, genid: int, off: int, size: int) -> int:
        """Drops the cached pages of (nhid, genid) overlapping bytes [off, off + size) -> pages removed;
        size = Cachemap.TO_END drops every page from off on."""
        return int(lib().cachemap_invalidate(self.h, nhid, genid, off, size))

    def rename(self, nhid_from: int, nhid_to: int, genid: int) -> int:
        """edgefs_rename: the cached pages of (nhid_to, genid) are dropped and those of (nhid_from, genid)
        move to nhid_to -> pages moved."""
        return int(lib().cachemap_rename(self.h, nhid_from, nhid_to, genid))

    def counters(self):
        rq, ht = C.c_uint64(), C.c_uint64()
        lib().cachemap_get_counters(self.h, C.byref(rq), C.byref(ht))
        return rq.value, ht.value

    def engine_handle(self) -> int:
        return int(lib().cachemap_engine(self.h) or 0)

    def engine_handles(self) -> list:
        """Every engine of the map (one per CMB200_DEVICES entry), first = engine_handle()."""
        out = (C.c_void_p * 64)()
        n = lib().cachemap_engines(self.h, out, 64)
        return [int(out[i]) for i in range(min(n, 64))]


_LIBC = None


def _libc():
    global _LIBC
    if _LIBC is None:
        _LIBC = C.CDLL(None)
        _LIBC.free.argtypes = [C.c_void_p]
        _LIBC.free.restype = None
    return _LIBC
