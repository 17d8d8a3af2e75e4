"""The drop-in's CMB200_CHECKPOINT_SEC thread without a GPU: edge_fuse_b200/csrc/cachemap_api.c over the
CPU stand-in of tests/c/mock_checkpoint.c, whose snapshot call sleeps for a second, driven by
tests/c/checkpoint_drive.c — eight threads of back-to-back cachemap_put into a 64-slot write-behind ring
for four seconds.  Saves must run while the ring is busy, no put may wait for one, and cachemap_free must
stop the thread and save once more.  Test infrastructure only: nothing of the product links the
stand-in."""
import os
import re
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = [os.path.join(ROOT, "edge_fuse_b200", "csrc", "cachemap_api.c"),
       os.path.join(ROOT, "tests", "c", "mock_checkpoint.c"),
       os.path.join(ROOT, "tests", "c", "checkpoint_drive.c")]
SAVE_US = 1_000_000             # MOCK_SAVE_US of the stand-in


def _build(tmp_path, name, extra):
    exe = str(tmp_path / name)
    r = subprocess.run(["gcc", "-std=gnu11", "-O1", "-g", "-pthread", *extra, *SRC, "-o", exe], capture_output=True, text=True)
    return exe if r.returncode == 0 else None, r.stderr


def _drive(exe, tmp_path):
    env = dict(os.environ, CMB200_PERSIST="1", CMB200_CHECKPOINT_SEC="1", CMB200_WB_SLOTS="64",
               TSAN_OPTIONS="halt_on_error=0 report_signal_unsafe=0")
    for k in ("CMB200_DEVICES", "CMB200_DEVICE", "CMB200_HOST_TIER_MB", "CMB200_TIER_PROMOTE"):
        env.pop(k, None)
    d = tmp_path / "cache"
    d.mkdir()
    out = subprocess.run([exe, str(d), "8", "4"], capture_output=True, text=True, timeout=120, env=env)
    m = re.search(r"saves_during (\d+) max_put_us (\d+) puts (\d+) begun_before_free (\d+) begun_by_free (\d+) "
                  r"ended_by_free (\d+) saves_later (\d+)", out.stdout)
    assert out.returncode == 0 and m, out.stdout + out.stderr
    return out, [int(x) for x in m.groups()]


def _check(fields, out):
    during, max_put_us, puts, begun_before, begun_by_free, ended_by_free, later = fields
    msg = out.stdout + out.stderr[-3000:]
    assert puts > 1000, msg
    # a one-second save every second while the ring never empties: two of them start within four seconds
    assert during >= 2, msg
    # the callers never wait for a save: at the parent the flusher sleeps inside it and the ring fills
    assert max_put_us < SAVE_US // 4, msg
    # cachemap_free stops the thread (a save it is in finishes first), then saves once more, and nothing
    # saves after it returned
    assert begun_by_free >= begun_before + 1 and ended_by_free == begun_by_free and later == 0, msg


def test_checkpoints_run_while_puts_keep_the_ring_busy(tmp_path):
    exe, err = _build(tmp_path, "checkpoint_drive", [])
    assert exe, err
    out, fields = _drive(exe, tmp_path)
    _check(fields, out)


def test_checkpoint_thread_has_no_data_race(tmp_path):
    exe, err = _build(tmp_path, "checkpoint_drive_tsan", ["-fsanitize=thread"])
    if not exe:
        pytest.skip("gcc cannot link -fsanitize=thread here: " + err[-200:])
    out, fields = _drive(exe, tmp_path)
    assert "ThreadSanitizer" not in out.stderr, out.stderr[-3000:]
    _check(fields, out)
