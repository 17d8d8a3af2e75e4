#!/usr/bin/env python
"""A small pass over every hot kernel (ring encoder incl. long matches and ragged sizes, k_decode,
k_get_small with its decode pipeline, eviction sampling, compaction + table rebuild) meant to be
run under `compute-sanitizer --tool memcheck`."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))
import numpy as np
import datagen
import edge_fuse_b200 as E
from oracle import ef_oracle as O

for pshift, n in ((12, 24), (16, 8)):
    bs = 1 << pshift
    eng = E.Engine(pshift=pshift, accel=12, capacity=2048, table_slots=4096, arena_bytes=32 << 20, max_batch=64, flags=E.FINGERPRINT)
    pages = np.stack([datagen.make_page("RTZMPAX"[i % 7], bs, 40 + i) for i in range(n)])
    u = np.full(n, 5, dtype=np.uint64); l = np.arange(n, dtype=np.uint64)
    lens = eng.put(u, l, pages)
    recs = eng.read_records(u, l)
    for i in range(n):
        blk = O.lz4_encode(pages[i], 12)
        assert lens[i] == len(blk) and recs[i][24:] == blk, (pshift, i)
    out, st = eng.get(u, l)
    assert (st == E.HIT).all() and (out == pages).all()
    out, st = eng.get_small(u, l)
    assert (st == E.HIT).all() and (out == pages).all()
    eng.put(u[:4], l[:4], pages[4:8])                       # rewrites -> garbage
    eng.unset(u[8:12], l[8:12])                             # tombstones
    eng.sample(datagen.words(3, 16))
    eng.compact()
    out, st = eng.get_small(u[:8], l[:8])
    assert (st == E.HIT).all() and (out[:4] == pages[4:8]).all() and (out[4:] == pages[4:8]).all()
    eng.close()
# ragged codec sizes through the ring (TMA tail buffers < 256 bytes, sizes not a multiple of 16)
for nbytes in (13, 100, 255, 257, 4095, 65535):
    pg = np.stack([datagen.make_page("T", nbytes, 7), datagen.make_page("M", nbytes, 8)])
    pad = np.zeros((2, (nbytes + 15) // 16 * 16), dtype=np.uint8); pad[:, :nbytes] = pg
    blocks, _ = E.lz4_encode_batch(pad, nbytes=nbytes, accel=12)
    for i in range(2):
        assert blocks[i] == O.lz4_encode(pg[i], 12), nbytes
print("sanitize_small ok")
