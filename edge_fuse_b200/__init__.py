"""edge_fuse_b200 — H100-native cachemap (hash -> LZ4 -> keyed lookup) behind the reference's C API.

The product is the shared library ``libcachemap.so.0.0`` built from ``csrc/`` (CUDA kernels for
sm_90a + a C host layer exporting the reference's cachemap.h / filemap.h functions).  This Python
package is only a ctypes face over that C ABI for tests and benchmarks: it never computes
anything itself and raises if the library or a CUDA device is missing — there is no CPU fallback.
"""
from .binding import (  # noqa: F401
    Cachemap, Engine, lib, library_path, compose_keys, lz4_encode_batch, lz4_decode_batch,
    fingerprint_batch, gen_chunk_host, gen_stream_ids, gen_addr, device_count, last_error,
    HIT, MISS, INVALID, BAD_ENTRY, BAD_DECODE, REMOTE, FINGERPRINT, EXPORTED_SYMBOLS, engine_stats,
    host_tier_stats, read_checkpoints, VERIFY, CORRUPT, verify_stats, owner, save_set, load_set,
    snapshot_begin, snapshot_finish, chain_begin, load_chain, TOUCH, DROPPED,
)
