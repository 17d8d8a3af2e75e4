"""One rank of a replicated index in its own process, for the peer-read tests on one GPU.

    python tests/peer_owner.py

reads one JSON command per line on stdin and answers one JSON line on stdout: {"ok": true, ...} or
{"ok": false, "error": "..."}.  Arrays travel as .npy files: a command names its inputs by path
(fields ending in "_npy"), and an answer names the files it wrote in the directory `dir` of the command.

    create    pshift, accel, flags, arena_bytes, device, capacity          -> {}
    put_step  u_npy, l_npy, [valid_npy], pages, rank, base, stride, dir    -> records_npy ([n, 4] int64), lens
    put       u_npy, l_npy, pages                                          -> lens
    unset     u_npy, l_npy                                                 -> {}
    compact                                                                -> reclaimed
    locate    u_npy, l_npy, dir   -> status_npy, where_npy (owner rank of a REMOTE answer, the record's current
                                     rec_off of a HIT), clen_npy (the stored length in the record's prefix, -1: none)
    handle                        -> handle (hex of the arena's 64-byte CUDA IPC handle), size
    stats                         -> the engine's counters
    close                         -> frees the engine and its arena

`pages` is either {"npy": path} or {"gen": [[kind, seed], ...]}: datagen.make_page(kind, bsize, seed).  The
engine, and the arena a parent may have mapped, live until `close`; at EOF on stdin the process closes its
engine and exits, so a parent that dies leaves nothing running.  A parent unmaps this arena (close_peers)
before it sends `close`.
"""
from __future__ import annotations

import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)

import numpy as np  # noqa: E402

import datagen  # noqa: E402
import edge_fuse_b200 as E  # noqa: E402


class Owner:
    def __init__(self):
        self.eng = None

    def _pages(self, spec, n):
        if "npy" in spec:
            pages = np.load(spec["npy"])
        else:
            pages = np.stack([datagen.make_page(k, self.eng.bsize, int(s)) for k, s in spec["gen"]])
        assert pages.shape == (n, self.eng.bsize) and pages.dtype == np.uint8, pages.shape
        return np.ascontiguousarray(pages)

    def _save(self, c, name, a):
        path = os.path.join(c["dir"], f"{name}.npy")
        np.save(path, a)
        return path

    def create(self, c):
        assert self.eng is None, "an engine is open"
        self.eng = E.Engine(pshift=c["pshift"], accel=c["accel"], capacity=c.get("capacity", 1024),
                            arena_bytes=c["arena_bytes"], max_batch=c.get("max_batch", 256),
                            flags=c.get("flags", 0), device=c.get("device", -1))
        return {}

    def put_step(self, c):
        u, l = np.load(c["u_npy"]), np.load(c["l_npy"])
        n = len(u)
        valid = np.load(c["valid_npy"]) if c.get("valid_npy") else None
        pages = self._pages(c["pages"], n)
        self.eng.set_stream_order(c["base"], c["stride"])
        d_rec = self.eng.dev_alloc(max(n, 1) * 32)
        try:
            self.eng.wait(self.eng.put_step(u, l, pages, valid=valid, rank=c["rank"], records_dev=d_rec))
            self.eng.sync()
            rec = np.zeros((n, 4), dtype=np.int64)
            self.eng.d2h(rec, d_rec)
        finally:
            self.eng.dev_free(d_rec)
        from edge_fuse_b200 import sharding
        return {"records_npy": self._save(c, "records", rec),
                "lens": [int(x) for x in sharding.unpack_records(rec)[4]]}

    def put(self, c):
        u, l = np.load(c["u_npy"]), np.load(c["l_npy"])
        return {"lens": [int(x) for x in self.eng.put(u, l, self._pages(c["pages"], len(u)))]}

    def unset(self, c):
        self.eng.unset(np.load(c["u_npy"]), np.load(c["l_npy"]))
        return {}

    def compact(self, c):
        return {"reclaimed": int(self.eng.compact())}

    def locate(self, c):
        u, l = np.load(c["u_npy"]), np.load(c["l_npy"])
        status, where = self.eng.locate(u, l)
        recs, lens = self.eng.read_records_raw(u, l)
        clen = np.where(lens >= 24, recs[:, 16:20].copy().view(np.uint32)[:, 0].astype(np.int64), -1)
        return {"status_npy": self._save(c, "status", status), "where_npy": self._save(c, "where", where),
                "clen_npy": self._save(c, "clen", clen)}

    def handle(self, c):
        h, size = self.eng.arena_ipc_handle()
        return {"handle": h.hex(), "size": size}

    def stats(self, c):
        return self.eng.stats()

    def close(self, c):
        if self.eng is not None:
            self.eng.close()
            self.eng = None
        return {}


def main() -> int:
    owner = Owner()
    try:
        for line in sys.stdin:
            if not line.strip():
                continue
            c = json.loads(line)
            try:
                ans = {"ok": True, **getattr(owner, c["cmd"])(c)}
            except Exception as e:                      # the parent decides what a failure means
                ans = {"ok": False, "error": f"{type(e).__name__}: {e}"}
            sys.stdout.write(json.dumps(ans) + "\n")
            sys.stdout.flush()
    finally:
        owner.close({})
    return 0


if __name__ == "__main__":
    sys.exit(main())
