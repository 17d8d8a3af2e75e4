"""The drop-in's promotion policy (CMB200_TIER_PROMOTE) without a GPU: edge_fuse_b200/csrc/cachemap_api.c
over the CPU stand-in of an engine whose host tier can promote (tests/c/mock_tier_promote.c, built on
tests/c/mock_host_tier.c), stressed by tests/c/host_stress.c.  The arena holds far fewer pages than the
threads keep re-reading, so their keys go to the tier, the gets log them as hot, and the flusher's
rounds bring them back while puts, gets and demotions go on: read-your-writes must hold throughout, the
eviction run must still end at capacity, and ThreadSanitizer must find no race."""
import os
import re
import shutil
import subprocess
import tempfile

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = [os.path.join(ROOT, "edge_fuse_b200", "csrc", "cachemap_api.c"),
       os.path.join(ROOT, "tests", "c", "mock_tier_promote.c"),
       os.path.join(ROOT, "tests", "c", "host_stress.c")]
# a 4 MiB arena holds 64 pages of 64 KiB or 1024 of 4 KiB; the tier is large enough never to wrap
TIER_ENV = dict(CMB200_PERSIST="0", CMB200_WB_SLOTS="64", CMB200_ARENA_MB="4", CMB200_HOST_TIER_MB="1024")


def _build(tmp_path, name, extra):
    exe = str(tmp_path / name)
    r = subprocess.run(["gcc", "-std=gnu11", "-O1", "-g", "-pthread", *extra, *SRC, "-o", exe], capture_output=True, text=True)
    return exe if r.returncode == 0 else None, r.stderr


def _run(exe, threads, ops, pshift, limit, promote, *mode):
    d = tempfile.mkdtemp()
    try:
        env = dict(os.environ, TSAN_OPTIONS="halt_on_error=0 report_signal_unsafe=0", **TIER_ENV)
        env.pop("CMB200_TIER_PROMOTE", None)
        if promote:
            env["CMB200_TIER_PROMOTE"] = str(promote)
        return subprocess.run([exe, d, str(threads), str(ops), str(pshift), str(limit), *mode], capture_output=True,
                              text=True, timeout=limit + 30, env=env)
    finally:
        shutil.rmtree(d, ignore_errors=True)


def _counts(stderr):
    t = re.search(r"mock host tier: demoted (\d+) retired (\d+)", stderr)
    p = re.search(r"mock tier promote: promoted (\d+) drains (\d+)", stderr)
    assert t and p, stderr[-2000:]
    return int(t.group(1)), int(p.group(1)), int(p.group(2))


@pytest.mark.parametrize("threads,pshift,ops", [(48, 12, 1500), (8, 16, 600)])
def test_promotion_keeps_read_your_writes(tmp_path, threads, pshift, ops):
    exe, err = _build(tmp_path, "promote_stress", [])
    assert exe, err
    out = _run(exe, threads, ops, pshift, 150, 64)
    assert out.returncode == 0 and "host_stress ok" in out.stdout, out.stdout + out.stderr
    demoted, promoted, drains = _counts(out.stderr)
    assert demoted > 0 and promoted > 0 and drains > 0, (demoted, promoted, drains)


def test_promotion_is_off_unless_asked_for(tmp_path):
    exe, err = _build(tmp_path, "promote_stress", [])
    assert exe, err
    out = _run(exe, 8, 600, 16, 150, 0)
    assert out.returncode == 0 and "host_stress ok" in out.stdout, out.stdout + out.stderr
    demoted, promoted, drains = _counts(out.stderr)
    assert demoted > 0 and promoted == 0 and drains == 0


def test_eviction_with_promotion_still_ends_at_capacity(tmp_path):
    exe, err = _build(tmp_path, "promote_stress", [])
    assert exe, err
    out = _run(exe, 16, 4000, 16, 150, 64, "evict")
    assert out.returncode == 0 and "host_stress ok" in out.stdout, out.stdout + out.stderr
    assert _counts(out.stderr)[0] > 0


def test_promotion_path_has_no_data_race(tmp_path):
    exe, err = _build(tmp_path, "promote_stress_tsan", ["-fsanitize=thread"])
    if not exe:
        pytest.skip("gcc cannot link -fsanitize=thread here: " + err[-200:])
    out = _run(exe, 12, 600, 16, 400, 64)
    assert out.returncode == 0 and "host_stress ok" in out.stdout, out.stdout[-2000:] + out.stderr[-2000:]
    assert "ThreadSanitizer" not in out.stderr, out.stderr[-3000:]
    demoted, promoted, _ = _counts(out.stderr)
    assert demoted > 0 and promoted > 0
