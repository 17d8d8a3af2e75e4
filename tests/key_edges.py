"""tests/golden/key_edges.json (tools/gen_golden.py key_edges): addresses that share a store key (the
FNV-1a-64 of the 16 address bytes), addresses of the table's empty (0) and tombstone (~0) keys, and the
reference's answers to a trace over them.  Shared by the CPU and the GPU tests of those edges."""
from __future__ import annotations

import hashlib
import json
import os

import numpy as np

import datagen

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
PNUM_MASK = (1 << 44) - 1
SENTINEL_KEYS = {"key0": 0, "key_ones": (1 << 64) - 1}


def load() -> dict:
    with open(os.path.join(GOLD, "key_edges.json")) as f:
        fx = json.load(f)
    fx["groups"] = {k: [tuple(a) for a in v] for k, v in fx["groups"].items()}
    fx["ordinary"] = [tuple(a) for a in fx["ordinary"]]
    return fx


def cachemap_args(u: int, l: int, pshift: int):
    """-> (offset, nhid, genid) of cachemap_put / cachemap_get that compose the address {u, l}."""
    return (l & PNUM_MASK) << pshift, u, l >> 44


def page(content, pshift: int) -> np.ndarray:
    return datagen.make_page(content[0], 1 << pshift, content[1])


def sha(b) -> str:
    return hashlib.sha256(bytes(b)).hexdigest()


def model_replay(O, fx: dict, pshift: int):
    """The trace through oracle StoreModel -> (answers in the fixture's form, model)."""
    m = O.StoreModel(pshift=pshift, accel=fx["accel"])
    answers = []
    for kind, u, l, content in fx["ops"]:
        off, nh, gen = cachemap_args(u, l, pshift)
        if kind == "put":
            m.put(off, nh, gen, page(content, pshift))
        elif kind == "unset":
            m.unset(u, l)
        else:
            st, pg = m.get_status(off, nh, gen)
            answers.append(sha(pg) if st == "hit" else st)
    return answers, m
