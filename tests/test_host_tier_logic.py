"""The drop-in's host-tier path without a GPU: edge_fuse_b200/csrc/cachemap_api.c over a CPU stand-in
of the engine with a host tier (tests/c/mock_host_tier.c, built on tests/c/mock_engine.c), whose arena
is CMB200_ARENA_MB and whose host tier is CMB200_HOST_TIER_MB, stressed by tests/c/host_stress.c.  A
full arena must demote records to the tier instead of evicting them: read-your-writes holds for every
key although the live pages are many times the arena, and the eviction run still ends at capacity."""
import os
import re
import shutil
import subprocess
import tempfile

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = [os.path.join(ROOT, "edge_fuse_b200", "csrc", "cachemap_api.c"),
       os.path.join(ROOT, "tests", "c", "mock_host_tier.c"),
       os.path.join(ROOT, "tests", "c", "host_stress.c")]
# a 4 MiB arena holds 64 pages of 64 KiB or 1024 of 4 KiB; the tier is large enough never to wrap
TIER_ENV = dict(CMB200_PERSIST="0", CMB200_WB_SLOTS="64", CMB200_ARENA_MB="4", CMB200_HOST_TIER_MB="1024")


def _build(tmp_path, name, extra):
    exe = str(tmp_path / name)
    r = subprocess.run(["gcc", "-std=gnu11", "-O1", "-g", "-pthread", *extra, *SRC, "-o", exe], capture_output=True, text=True)
    return exe if r.returncode == 0 else None, r.stderr


def _run(exe, threads, ops, pshift, limit, *mode):
    d = tempfile.mkdtemp()
    try:
        env = dict(os.environ, TSAN_OPTIONS="halt_on_error=0 report_signal_unsafe=0", **TIER_ENV)
        return subprocess.run([exe, d, str(threads), str(ops), str(pshift), str(limit), *mode], capture_output=True, text=True,
                              timeout=limit + 30, env=env)
    finally:
        shutil.rmtree(d, ignore_errors=True)


def _demoted(stderr):
    m = re.search(r"mock host tier: demoted (\d+) retired (\d+)", stderr)
    assert m, stderr[-2000:]
    return int(m.group(1)), int(m.group(2))


@pytest.mark.parametrize("threads,pshift,ops", [(48, 12, 1500), (8, 16, 400), (1, 16, 800)])
def test_full_arena_demotes_and_keeps_read_your_writes(tmp_path, threads, pshift, ops):
    exe, err = _build(tmp_path, "host_stress", [])
    assert exe, err
    out = _run(exe, threads, ops, pshift, 150)
    assert out.returncode == 0 and "host_stress ok" in out.stdout, out.stdout + out.stderr
    demoted, retired = _demoted(out.stderr)
    assert demoted > 0 and retired == 0


def test_eviction_with_a_tier_still_ends_at_capacity(tmp_path):
    exe, err = _build(tmp_path, "host_stress", [])
    assert exe, err
    out = _run(exe, 16, 4000, 16, 150, "evict")
    assert out.returncode == 0 and "host_stress ok" in out.stdout, out.stdout + out.stderr
    assert _demoted(out.stderr)[0] > 0


def test_demotion_path_has_no_data_race(tmp_path):
    exe, err = _build(tmp_path, "host_stress_tsan", ["-fsanitize=thread"])
    if not exe:
        pytest.skip("gcc cannot link -fsanitize=thread here: " + err[-200:])
    out = _run(exe, 12, 600, 16, 400)
    assert out.returncode == 0 and "host_stress ok" in out.stdout, out.stdout[-2000:] + out.stderr[-2000:]
    assert "ThreadSanitizer" not in out.stderr, out.stderr[-3000:]
    assert _demoted(out.stderr)[0] > 0
