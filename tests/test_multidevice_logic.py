"""One map over several engines (CMB200_DEVICES) without a GPU: edge_fuse_b200/csrc/cachemap_api.c over
the CPU stand-in (tests/c/mock_multidev.c, built on tests/c/mock_engine.c) with three engines, stressed
by the unchanged tests/c/host_stress.c — read-your-writes per key through the owner's ring, whole pages,
counters, eviction by count over all engines, a tiny ring, ThreadSanitizer — and checked by
tests/c/multidev_check.c: every engine holds its share of the keys, a range across engines counts in
page order, an engine that cannot start leaves none behind, and cmb200_owner is the rule pinned below on
tests/golden/keys.json.  Test infrastructure only: nothing of the product links the stand-in."""
import json
import os
import re
import shutil
import subprocess
import tempfile

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
API = os.path.join(ROOT, "edge_fuse_b200", "csrc", "cachemap_api.c")
MOCK = os.path.join(ROOT, "tests", "c", "mock_multidev.c")
STRESS = os.path.join(ROOT, "tests", "c", "host_stress.c")
CHECK = os.path.join(ROOT, "tests", "c", "multidev_check.c")
GOLD = os.path.join(ROOT, "tests", "golden", "keys.json")


def owner(key, g):
    """Engine of a key among g: the high 32 bits of the key scaled to g (cmb200_owner)."""
    return ((key >> 32) * g) >> 32


def _build(tmp_path, name, main, extra=()):
    exe = str(tmp_path / name)
    r = subprocess.run(["gcc", "-std=gnu11", "-O1", "-g", "-pthread", *extra, API, MOCK, main, "-o", exe],
                       capture_output=True, text=True)
    return exe if r.returncode == 0 else None, r.stderr


def _env(devices, **extra):
    env = dict(os.environ, CMB200_PERSIST="0", CMB200_DEVICES=devices,
               TSAN_OPTIONS="halt_on_error=0 report_signal_unsafe=0", **extra)
    for k in ("CMB200_DEVICE", "CMB200_HOST_TIER_MB", "CMB200_TIER_PROMOTE", "CMB200_ARENA_MB"):
        env.pop(k, None)
    return env


def _stress(exe, threads, ops, pshift, limit, *mode, devices="0,1,2", **extra):
    d = tempfile.mkdtemp()
    try:
        return subprocess.run([exe, d, str(threads), str(ops), str(pshift), str(limit), *mode], capture_output=True,
                              text=True, timeout=limit + 30, env=_env(devices, **extra))
    finally:
        shutil.rmtree(d, ignore_errors=True)


@pytest.mark.parametrize("threads", [1, 16, 48])
def test_three_engines_under_many_callers(tmp_path, threads):
    exe, err = _build(tmp_path, "host_stress", STRESS)
    assert exe, err
    out = _stress(exe, threads, 1500, 12, 150)
    assert out.returncode == 0 and "host_stress ok" in out.stdout, out.stdout + out.stderr


def test_two_engines_on_one_device(tmp_path):
    exe, err = _build(tmp_path, "host_stress", STRESS)
    assert exe, err
    out = _stress(exe, 16, 1000, 12, 150, devices="0,0")
    assert out.returncode == 0 and "host_stress ok" in out.stdout, out.stdout + out.stderr


def test_three_engines_with_tiny_rings(tmp_path):
    exe, err = _build(tmp_path, "host_stress", STRESS)
    assert exe, err
    out = _stress(exe, 24, 1200, 12, 150, CMB200_WB_SLOTS="64")
    assert out.returncode == 0 and "host_stress ok" in out.stdout, out.stdout + out.stderr


@pytest.mark.parametrize("threads", [16, 48])
def test_eviction_over_three_engines_ends_at_capacity(tmp_path, threads):
    """Far more keys than the capacity, three flushers deciding at once: the total over the engines
    never passes the capacity and, once the store is full, stays at it (no decision evicts more than
    the count needs)."""
    exe, err = _build(tmp_path, "host_stress", STRESS)
    assert exe, err
    out = _stress(exe, threads, 4000, 12, 150, "evict")
    assert out.returncode == 0 and "host_stress ok" in out.stdout, out.stdout + out.stderr
    m = re.search(r"entries (\d+) capacity (\d+)", out.stdout)
    assert m and int(m.group(1)) == int(m.group(2)), out.stdout


def test_three_engines_have_no_data_race(tmp_path):
    exe, err = _build(tmp_path, "host_stress_tsan", STRESS, ["-fsanitize=thread"])
    if not exe:
        pytest.skip("gcc cannot link -fsanitize=thread here: " + err[-200:])
    out = _stress(exe, 12, 600, 12, 400)
    assert out.returncode == 0 and "host_stress ok" in out.stdout, out.stdout[-2000:] + out.stderr[-2000:]
    assert "ThreadSanitizer" not in out.stderr, out.stderr[-3000:]


@pytest.mark.parametrize("devices", ["0", "0,1", "0,1,2", "3,1,4,1,5", "0,0"])
def test_every_engine_holds_its_share(tmp_path, devices):
    exe, err = _build(tmp_path, "multidev_check", CHECK)
    assert exe, err
    out = subprocess.run([exe, str(tmp_path), "share"], capture_output=True, text=True, timeout=120, env=_env(devices))
    assert out.returncode == 0 and "multidev_check ok" in out.stdout, out.stdout + out.stderr
    listed = [int(x) for x in devices.split(",")]
    got = [int(m.group(1)) for m in re.finditer(r"engine \d+ device (-?\d+)", out.stdout)]
    assert got == listed, out.stdout


def test_an_engine_that_cannot_start_leaves_none(tmp_path):
    exe, err = _build(tmp_path, "multidev_check", CHECK)
    assert exe, err
    out = subprocess.run([exe, str(tmp_path), "fail"], capture_output=True, text=True, timeout=60,
                         env=_env("0,9", CMB200_SOFT_FAIL="1"))
    assert out.returncode == 0 and "multidev_check ok" in out.stdout, out.stdout + out.stderr


def test_owner_rule_on_golden_keys(tmp_path):
    gold = json.load(open(GOLD))["addrs"]
    exe, err = _build(tmp_path, "multidev_check", CHECK)
    assert exe, err
    stdin = "".join(f"{u} {l}\n" for u, l, _ in gold)
    out = subprocess.run([exe, "-", "owner"], input=stdin, capture_output=True, text=True, timeout=60, check=True)
    lines = out.stdout.split("\n")[:len(gold)]
    assert len(lines) == len(gold)
    for (u, l, key), line in zip(gold, lines):
        got = line.split()
        k = int(key, 16)
        assert int(got[0], 16) == k, (u, l)
        assert [int(x) for x in got[1:]] == [owner(k, g) for g in range(1, 9)], (u, l, key)
    # the rule uses the high half of the key: the low bits that pick the reference's shard do not matter
    assert owner(0x00000000ffffffff, 8) == 0 and owner(0xffffffff00000000, 8) == 7
    assert {owner(k << 32, 3) for k in range(0, 1 << 32, 1 << 20)} == {0, 1, 2}
