"""ctypes face of the CPU oracle.  TEST INFRASTRUCTURE ONLY.

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may
import this module (see oracle/ef_oracle.h).  It wraps

* ``liboracle.so``  — the restatement of the reference path (lz4_block.c, keys.c, fingerprint.c);
* ``_ref/libcachemap_ref.so`` — the reference's own cachemap/ sources compiled by oracle/Makefile
  (present when it was built in the authoring container; ``ref()`` returns None otherwise);
* ``StoreModel`` — the keyed-store semantics of filemap/cachemap (SURVEY.md Appendix B) as a dict.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None
_REF = None
_REF_TRIED = False


def build(quiet: bool = True) -> None:
    """Compile liboracle.so (and _ref when /root/reference is present)."""
    subprocess.run(["make", "-C", _HERE], check=True,
                   stdout=subprocess.DEVNULL if quiet else None)


def lib() -> C.CDLL:
    global _LIB
    if _LIB is None:
        path = os.path.join(_HERE, "liboracle.so")
        if not os.path.exists(path):
            build()
        L = C.CDLL(path)
        L.ef_fnv1a64.restype = C.c_uint64
        L.ef_fnv1a64.argtypes = [C.c_void_p, C.c_size_t]
        L.ef_addr_compose.restype = C.c_int
        L.ef_addr_compose.argtypes = [C.c_uint64, C.c_uint64, C.c_uint32, C.c_int, C.c_void_p]
        L.ef_addr_key.restype = C.c_uint64
        L.ef_addr_key.argtypes = [C.c_void_p]
        L.ef_lz4_encode.restype = C.c_int
        L.ef_lz4_encode.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int]
        L.ef_lz4_decode.restype = C.c_int
        L.ef_lz4_decode.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int]
        L.ef_lz4_bound.restype = C.c_int
        L.ef_lz4_bound.argtypes = [C.c_int]
        L.ef_record_prefix.argtypes = [C.c_void_p, C.c_int32, C.c_void_p]
        L.ef_fingerprint128.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p]
        L.ef_cache_check.restype = C.c_int
        L.ef_cache_check.argtypes = [C.c_int, C.c_int, C.c_uint64, C.c_uint64, C.c_void_p, C.c_void_p]
        L.ef_build_nhid.restype = C.c_uint64
        L.ef_build_nhid.argtypes = [C.c_char_p, C.c_char_p]
        L.ef_cpu_bench_codec.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_int,
                                         C.c_int, C.c_int, C.c_void_p]
        L.ef_cpu_bench_store.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                         C.c_size_t, C.c_int, C.c_void_p, C.c_void_p, C.c_int,
                                         C.c_int, C.c_void_p]
        L.ef_gen_chunk.argtypes = [C.c_uint64, C.c_uint64, C.c_uint32, C.c_void_p]
        L.ef_gen_chunks.argtypes = [C.c_uint64, C.c_void_p, C.c_size_t, C.c_uint32, C.c_void_p, C.c_int]
        L.ef_gen_addr.argtypes = [C.c_uint64, C.c_void_p, C.c_size_t, C.c_int, C.c_void_p, C.c_void_p]
        L.ef_gen_stream_ids.restype = C.c_uint64
        L.ef_gen_stream_ids.argtypes = [C.c_uint64, C.c_size_t, C.c_double, C.c_uint64, C.c_void_p]
        L.ef_parity_records.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_int, C.c_int, C.c_void_p,
                                        C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p]
        _LIB = L
    return _LIB


def ref():
    """The compiled reference (libcachemap_ref.so) or None when it was never built."""
    global _REF, _REF_TRIED
    if not _REF_TRIED:
        _REF_TRIED = True
        path = os.path.join(_HERE, "_ref", "libcachemap_ref.so")
        if not os.path.exists(path) and os.path.isdir("/root/reference/cachemap"):
            build()
        if os.path.exists(path):
            R = C.CDLL(path)
            R.LZ4_compress_fast.restype = C.c_int
            R.LZ4_compress_fast.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int]
            R.LZ4_decompress_fast.restype = C.c_int
            R.LZ4_decompress_fast.argtypes = [C.c_void_p, C.c_void_p, C.c_int]
            R.LZ4_versionString.restype = C.c_char_p
            R.cachemap_create.restype = C.c_void_p
            R.cachemap_create.argtypes = [C.c_char_p, C.c_uint64, C.c_int, C.c_int]
            R.cachemap_get.restype = C.c_void_p
            R.cachemap_get.argtypes = [C.c_void_p, C.c_uint64, C.c_uint64, C.c_uint32]
            R.cachemap_put.restype = None
            R.cachemap_put.argtypes = [C.c_void_p, C.c_uint64, C.c_uint64, C.c_uint32, C.c_void_p]
            R.filemap_entries.restype = C.c_uint64
            R.filemap_entries.argtypes = [C.c_void_p]
            _REF = R
    return _REF


def gen_chunks(seed: int, cids, bsize: int = 65536, threads: int = 0, out: np.ndarray | None = None) -> np.ndarray:
    """[n, bsize] uint8 pages of the synthetic stream (oracle/streamgen.c), `threads` pthreads."""
    cids = np.ascontiguousarray(cids, dtype=np.uint64)
    if out is None:
        out = np.empty((len(cids), bsize), dtype=np.uint8)
    assert out.flags.c_contiguous and out.size == len(cids) * bsize
    lib().ef_gen_chunks(seed, cids.ctypes.data, len(cids), bsize, out.ctypes.data, threads or (os.cpu_count() or 1))
    return out


def gen_addr(seed: int, cids, pshift: int = 16):
    """-> (offset, nhid_small) arrays of the stream's addresses."""
    cids = np.ascontiguousarray(cids, dtype=np.uint64)
    off = np.empty(len(cids), dtype=np.uint64)
    nh = np.empty(len(cids), dtype=np.uint64)
    lib().ef_gen_addr(seed, cids.ctypes.data, len(cids), pshift, off.ctypes.data, nh.ctypes.data)
    return off, nh


def gen_stream_ids(n: int, dup: float, seed2: int = 43, first_cid: int = 0):
    """-> (cids, distinct): stream with a fraction `dup` of same-address repeats (SURVEY.md §8d)."""
    cids = np.empty(n, dtype=np.uint64)
    distinct = lib().ef_gen_stream_ids(seed2, n, float(dup), first_cid, cids.ctypes.data)
    return cids, int(distinct)


def parity_records(pages: np.ndarray, u, l, recs: np.ndarray, rec_lens, put_lens=None, accel: int = 12,
                   threads: int = 0) -> dict:
    """The parity gate of a measured run: every stored record must be the 24-byte prefix + the LZ4
    block that the reference's LZ4_compress_fast (oracle/_ref; the port when it is absent) makes of
    the page.  recs = [n, stride] uint8 as read back from the GPU store."""
    R = ref()
    enc = C.cast(R.LZ4_compress_fast, C.c_void_p) if R is not None else C.cast(lib().ef_port_compress_fast, C.c_void_p)
    pages = np.ascontiguousarray(pages, dtype=np.uint8)
    n, bsize = pages.shape
    addr = np.empty((n, 2), dtype=np.uint64)
    addr[:, 0], addr[:, 1] = u, l
    rec_lens = np.ascontiguousarray(rec_lens, dtype=np.int32)
    pl = None if put_lens is None else np.ascontiguousarray(put_lens, dtype=np.int32)
    recs = np.ascontiguousarray(recs, dtype=np.uint8)
    out = (C.c_double * 3)()
    lib().ef_parity_records(enc, pages.ctypes.data, n, bsize, accel, addr.ctypes.data, recs.ctypes.data,
                            recs.strides[0], rec_lens.ctypes.data, pl.ctypes.data if pl is not None else None,
                            threads or (os.cpu_count() or 1), out)
    return {"chunks": int(n), "mismatches": int(out[0]), "first_mismatch": int(out[1]),
            "against": "oracle/_ref (reference LZ4_compress_fast + data_prefix)" if R is not None else "oracle port",
            "block_bytes": int(out[2])}


def _u8(a) -> np.ndarray:
    if isinstance(a, (bytes, bytearray, memoryview)):
        a = np.frombuffer(a, dtype=np.uint8)
    a = np.ascontiguousarray(a, dtype=np.uint8)
    return a


def fnv1a64(data: bytes) -> int:
    buf = (C.c_char * max(len(data), 1)).from_buffer_copy(data or b"\0")
    return int(lib().ef_fnv1a64(buf, len(data)))


def cache_check(have_cache: bool, pshift: int, off: int, size: int):
    """edgefs.c:192-203 -> (do_cache, page_size, aligned_off)."""
    ps, ao = C.c_uint64(), C.c_uint64()
    ok = lib().ef_cache_check(int(have_cache), pshift, off, size, C.byref(ps), C.byref(ao))
    return bool(ok), ps.value, ao.value


def build_nhid(name: bytes, bucket_path: bytes) -> int:
    """edgefs.c:205-212 with bhid_small = FNV(url path) (edgefs.c:1911)."""
    return int(lib().ef_build_nhid(name, bucket_path))


def addr_compose(offset: int, nhid: int, genid: int, pshift: int):
    """-> (u, l) or None when the page number overflows 44 bits (cachemap.c:151-166)."""
    out = (C.c_uint64 * 2)()
    if lib().ef_addr_compose(offset, nhid, genid, pshift, out) != 0:
        return None
    return int(out[0]), int(out[1])


def addr_key(u: int, l: int) -> int:
    a = (C.c_uint64 * 2)(u, l)
    return int(lib().ef_addr_key(a))


def lz4_encode(page, accel: int = 12) -> bytes:
    src = _u8(page)
    dst = np.empty(int(lib().ef_lz4_bound(src.size)) + 8, dtype=np.uint8)
    n = lib().ef_lz4_encode(src.ctypes.data, src.size, dst.ctypes.data, accel)
    return dst[:n].tobytes()


def lz4_decode(block, n_out: int):
    """-> (page bytes, consumed) ; consumed < 0 on malformed input."""
    src = _u8(np.frombuffer(block, dtype=np.uint8) if isinstance(block, (bytes, bytearray)) else block)
    dst = np.zeros(n_out, dtype=np.uint8)
    used = lib().ef_lz4_decode(src.ctypes.data, src.size, dst.ctypes.data, n_out)
    return dst.tobytes(), int(used)


def record_prefix(u: int, l: int, clen: int) -> bytes:
    a = (C.c_uint64 * 2)(u, l)
    out = (C.c_uint8 * 24)()
    lib().ef_record_prefix(a, clen, out)
    return bytes(out)


def fingerprint128(data) -> tuple[int, int]:
    src = _u8(np.frombuffer(data, dtype=np.uint8) if isinstance(data, (bytes, bytearray)) else data)
    out = (C.c_uint64 * 2)()
    lib().ef_fingerprint128(src.ctypes.data if src.size else None, src.size, out)
    return int(out[0]), int(out[1])


def ref_lz4_encode(page, accel: int = 12) -> bytes:
    """The reference's own LZ4_compress_fast, called the way filemap_set does (filemap.c:126)."""
    R = ref()
    src = _u8(page)
    dst = np.empty(src.size + 1024, dtype=np.uint8)
    n = R.LZ4_compress_fast(src.ctypes.data, dst.ctypes.data, src.size, src.size + 1024, accel)
    return dst[:n].tobytes()


def ref_lz4_decode(block: bytes, n_out: int):
    R = ref()
    src = np.frombuffer(block + b"\0" * 64, dtype=np.uint8)
    # LZ4_decompress_fast is the withPrefix64k variant; give it slack on both sides.
    buf = np.zeros(n_out + 65536 + 64, dtype=np.uint8)
    dst = buf[65536:65536 + n_out]
    used = R.LZ4_decompress_fast(src.ctypes.data, dst.ctypes.data, n_out)
    return dst.tobytes(), int(used)


class StoreModel:
    """Keyed-store semantics of filemap + the counters of cachemap, no eviction
    (SURVEY.md Appendix B rules 1-4; cachemap.c:168-197; filemap.c:112-158,217-262).

    One record per 64-bit key; a put replaces whatever record has that key; a get hits only
    when the stored 16-byte address equals the requested one and the block decodes to its
    stored length.  requests++ only for valid addresses, hits++ on non-NULL.
    """

    def __init__(self, pshift: int = 16, accel: int = 12):
        self.pshift, self.accel, self.bsize = pshift, accel, 1 << pshift
        self.rec: dict[int, tuple[tuple[int, int], int, bytes]] = {}
        self.requests = 0
        self.hits = 0
        self.bad_entries = 0

    def put(self, offset: int, nhid: int, genid: int, page) -> None:
        a = addr_compose(offset, nhid, genid, self.pshift)
        if a is None:
            return
        key = addr_key(*a)
        blk = lz4_encode(page, self.accel) if self.accel else None
        # filemap_set's dstCapacity is bsize + 1024 (filemap.c:126): LZ4_compress_fast returns 0 for a
        # longer block, and this store keeps such a page raw (DESIGN.md, f1)
        if blk is not None and len(blk) <= self.bsize + 1024:
            self.rec[key] = (a, len(blk), blk)
        else:
            self.rec[key] = (a, 0, bytes(_u8(page)))

    def get(self, offset: int, nhid: int, genid: int):
        return self.get_status(offset, nhid, genid)[1]

    def get_status(self, offset: int, nhid: int, genid: int):
        """-> (status, page or None); status "hit", "miss", or "bad entry" when the key holds a record
        of another address (the reference prints `bad entry` then, filemap.c:236-240)."""
        a = addr_compose(offset, nhid, genid, self.pshift)
        if a is None:
            return "miss", None
        self.requests += 1
        r = self.rec.get(addr_key(*a))
        if r is None:
            return "miss", None
        if r[0] != a:
            self.bad_entries += 1
            return "bad entry", None
        if r[1]:
            page, used = lz4_decode(r[2], self.bsize)
            if used != r[1]:
                return "miss", None
        else:
            page = r[2]
        self.hits += 1
        return "hit", page

    def unset(self, u: int, l: int) -> None:
        self.rec.pop(addr_key(u, l), None)

    def read_range(self, nhid: int, genid: int, off: int, size: int):
        """The cache part of edgefs_read (edgefs.c:1150-1178): gate, then get page after page
        until the first miss.  -> bytes or None."""
        do_cache, page_size, aligned = cache_check(True, self.pshift, off, size)
        if not do_cache:
            return None
        out = b""
        i = aligned
        while i < off + size:
            page = self.get(i, nhid, genid)
            if page is None:
                return None
            out += bytes(page)
            i += page_size
        return out

    def write_range(self, nhid: int, genid: int, off: int, data: bytes) -> None:
        """The put loop of edgefs.c:1183-1195 / 1216-1228."""
        do_cache, page_size, aligned = cache_check(True, self.pshift, off, len(data))
        if not do_cache:
            return
        i, b = aligned, 0
        while i < off + len(data):
            self.put(i, nhid, genid, data[b:b + page_size])
            i += page_size
            b += page_size

    def entries(self) -> int:
        return len(self.rec)

    def record_bytes(self, u: int, l: int):
        """The 24-byte prefix + payload the reference would hold in LMDB for this address."""
        r = self.rec.get(addr_key(u, l))
        if r is None:
            return None
        return record_prefix(r[0][0], r[0][1], r[1]) + r[2]
