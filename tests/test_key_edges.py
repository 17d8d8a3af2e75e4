"""Addresses that share a store key, and addresses whose key is the table's empty (0) or tombstone (~0)
marker, without a GPU (tests/golden/key_edges.json, recorded against the reference).

The store keeps one record per 64-bit FNV-1a key of the 16-byte address, not one per address
(filemap.c:18-24,143,188-215,236-240): a put replaces the key's record whatever address it held, a get
of a key that holds another address prints `bad entry` and misses, and an unset deletes by key.  Checked
here: the fixture's keys under both FNV implementations, the oracle's StoreModel against the reference's
answers, and the drop-in's host layer (edge_fuse_b200/csrc/cachemap_api.c: write-behind ring, combining
queue, range reads) over the CPU stand-in of tests/c/mock_engine.c, which keys its records as the
engine does."""
import os
import re
import subprocess

import numpy as np
import pytest

import key_edges as K

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PSHIFTS = (12, 16, 17)


@pytest.fixture(scope="module")
def fx():
    return K.load()


def _all_addrs(fx):
    return [(name, a) for name, g in fx["groups"].items() for a in g] + [("ordinary", a) for a in fx["ordinary"]]


def test_fixture_addresses_have_the_keys_they_claim(fx, oracle, tmp_path):
    """Every group shares one key (0 and ~0 for the sentinel groups), distinct from every other key, by
    the oracle's addr_key and by the FNV_hash that include/uint128.h inlines into C callers."""
    addrs = _all_addrs(fx)
    src = tmp_path / "keys.c"
    src.write_text('#include <stdio.h>\n#include <inttypes.h>\n#include "uint128.h"\n'
                   'int main(void){uint128_t a; uint64_t h;\n'
                   ' while (scanf("%" SCNx64 " %" SCNx64, &a.u, &a.l) == 2) {FNV_hash(&a, sizeof a, &h); printf("%016" PRIx64 "\\n", h);}\n'
                   ' return 0;}\n')
    exe = tmp_path / "keys"
    subprocess.run(["gcc", "-std=c99", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    out = subprocess.run([str(exe)], input="".join(f"{u:x} {l:x}\n" for _, (u, l) in addrs), capture_output=True,
                         text=True, check=True).stdout.split()
    inline = [int(x, 16) for x in out]
    assert inline == [oracle.addr_key(u, l) for _, (u, l) in addrs]
    keys = {}
    for (name, _), k in zip(addrs, inline):
        keys.setdefault(name, set()).add(k)
    assert len(fx["groups"]["quad"]) == 4 and all(len(g) >= 2 for g in fx["groups"].values())
    for name, ks in keys.items():
        if name != "ordinary":
            assert len(ks) == 1, name
    for name, k in K.SENTINEL_KEYS.items():
        assert keys[name] == {k}
    flat = [k for name, ks in keys.items() for k in ks]
    assert len(flat) == len(set(flat)) == len(fx["groups"]) + len(fx["ordinary"])


@pytest.mark.parametrize("pshift", PSHIFTS)
def test_model_answers_like_the_reference(fx, oracle, pshift):
    """StoreModel replays the trace with the reference's answers: page, plain miss, or bad entry per
    get, and the same counters and entries."""
    run = fx["runs"][str(pshift)]
    answers, m = K.model_replay(oracle, fx, pshift)
    assert answers == run["gets"]
    assert (m.requests, m.hits, len(m.rec), m.bad_entries) == (run["requests"], run["hits"], run["entries"],
                                                                run["bad_entries"])
    assert run["bad_entries"] > 0 and run["gets"].count("miss") > 0


def _build_drive(tmp_path):
    exe = str(tmp_path / "key_edges_drive")
    src = [os.path.join(ROOT, "edge_fuse_b200", "csrc", "cachemap_api.c"), os.path.join(ROOT, "tests", "c", "mock_engine.c"),
           os.path.join(ROOT, "tests", "c", "key_edges_drive.c")]
    r = subprocess.run(["gcc", "-std=gnu11", "-O1", "-g", "-pthread", *src, "-o", exe], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return exe


def parse_answers(lines, ops):
    """`op <i> <answer>` lines with the `bad entry` lines printed before them -> the answer of each get,
    "bad entry" for a miss that printed one."""
    gets, bad = [], 0
    for line in lines:
        if line == "bad entry":
            bad += 1
            continue
        m = re.fullmatch(r"op (\d+) (\S+)", line)
        assert m, line
        i, ans = int(m.group(1)), m.group(2)
        assert bad <= (ops[i][0] == "get" and ans == "miss"), f"op {i} {ops[i]}: {bad} bad entry lines, answer {ans}"
        if ops[i][0] == "get":
            gets.append("bad entry" if bad else ans)
        bad = 0
    return gets


@pytest.fixture(scope="module")
def drive(tmp_path_factory):
    return _build_drive(tmp_path_factory.mktemp("key_edges_drive"))


@pytest.mark.parametrize("pshift", PSHIFTS)
@pytest.mark.parametrize("how,ring,slots", [("get", "held", None), ("get", "one", None), ("get", "off", "0"),
                                            ("range", "held", None)])
def test_drop_in_answers_by_key(fx, oracle, drive, tmp_path, pshift, how, ring, slots):
    """The drop-in's host layer answers the trace as the reference does: with every page held in the
    write-behind ring, with only the newest page in it, with no ring, and through cachemap_read_range.
    The ring goes by key like the store: its newest page of a key decides, and a page of another
    address there is a bad entry, never a stale page of the asked address."""
    ops = fx["ops"]
    run = fx["runs"][str(pshift)]
    pages, fnv_of = [], {}
    lines = []
    for kind, u, l, content in ops:
        if kind == "put":
            p = K.page(content, pshift)
            fnv_of[K.sha(p)] = f"{oracle.fnv1a64(p.tobytes()):016x}"
            lines.append(f"p {u:x} {l:x} {len(pages)}")
            pages.append(p)
        else:
            lines.append(f"{kind[0]} {u:x} {l:x}")
    (tmp_path / "ops").write_text("\n".join(lines) + "\n")
    np.stack(pages).tofile(tmp_path / "pages")
    cache = tmp_path / "cache"
    cache.mkdir()
    env = dict(os.environ, CMB200_PERSIST="0")
    for k in ("CMB200_DEVICES", "CMB200_DEVICE", "CMB200_HOST_TIER_MB", "CMB200_TIER_PROMOTE", "CMB200_WB_SLOTS"):
        env.pop(k, None)
    if slots is not None:
        env["CMB200_WB_SLOTS"] = slots
    out = subprocess.run([drive, str(cache), str(pshift), str(tmp_path / "ops"), str(tmp_path / "pages"), how, ring],
                         capture_output=True, text=True, timeout=120, env=env)
    assert out.returncode == 0, out.stdout[-2000:] + out.stderr[-2000:]
    lines = out.stdout.splitlines()
    tail = re.fullmatch(r"entries (\d+) requests (\d+) hits (\d+)", lines[-1])
    assert tail, lines[-1]
    got = parse_answers(lines[:-1], ops)
    want = [fnv_of.get(a, a) for a in run["gets"]]
    get_ops = [op for op in ops if op[0] == "get"]
    for i, (g, w) in enumerate(zip(got, want)):
        assert g == w, f"get #{i} of {get_ops[i][1]:#x}/{get_ops[i][2]:#x}: answered {g}, the reference {w}"
    assert len(got) == len(want)
    assert [int(x) for x in tail.groups()] == [run["entries"], run["requests"], run["hits"]]
