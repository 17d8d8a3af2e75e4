"""cachemap_invalidate without a GPU: edge_fuse_b200/csrc/cachemap_api.c over the CPU stand-in of
tests/c/mock_invalidate.c, which removes records by stored address and logs the interval of every
cmb200_invalidate call, driven by tests/c/invalidate_drive.c.  Test infrastructure only: nothing of
the product links the stand-in."""
import os
import re
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = [os.path.join(ROOT, "edge_fuse_b200", "csrc", "cachemap_api.c"),
       os.path.join(ROOT, "tests", "c", "mock_invalidate.c"),
       os.path.join(ROOT, "tests", "c", "invalidate_drive.c")]
TO_END = (1 << 64) - 1
PNUM = 44
LAST_PAGE = (1 << PNUM) - 1
PUT_PAGES = set(range(16)) | {LAST_PAGE}          # what the convert mode holds before each case
GENID = 3


def _build(tmp_path, name, extra):
    exe = str(tmp_path / name)
    r = subprocess.run(["gcc", "-std=gnu11", "-O1", "-g", "-Wall", "-pthread", *extra, *SRC, "-o", exe],
                       capture_output=True, text=True)
    return exe if r.returncode == 0 else None, r.stderr


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    path, err = _build(tmp_path_factory.mktemp("inv"), "invalidate_drive", [])
    assert path, err
    return path


def _drive(exe, d, *args, **env_extra):
    env = dict(os.environ, CMB200_PERSIST="1", CMB200_WB_SLOTS="64",
               TSAN_OPTIONS="halt_on_error=0 report_signal_unsafe=0", **env_extra)
    for k in ("CMB200_DEVICES", "CMB200_DEVICE", "CMB200_HOST_TIER_MB", "CMB200_TIER_PROMOTE",
              "CMB200_CHECKPOINT_SEC", "CMB200_CHECKPOINT_DELTAS"):
        if k not in env_extra:
            env.pop(k, None)
    os.makedirs(d, exist_ok=True)
    out = subprocess.run([exe, args[0], str(d), *map(str, args[1:])], capture_output=True, text=True,
                         timeout=300, env=env)
    assert out.returncode == 0 and "\nlog:\n" in out.stdout, out.stdout + out.stderr
    head, log = out.stdout.split("\nlog:\n", 1)
    calls = [tuple(int(x) for x in ln.split()[1:]) for ln in log.splitlines() if ln.startswith("inv ")]
    return head, calls, log, out


def _interval(off, size, pshift):
    """[l_first, l_last] of the pages overlapping [off, off + size), or None when no call is due."""
    if size == 0 or (off >> pshift) >> PNUM:
        return None
    end = min(off + size - 1, TO_END)
    last = min(end >> pshift, LAST_PAGE)
    return (off >> pshift) | GENID << PNUM, last | GENID << PNUM


def _cases(p):
    P = 1 << p
    return [
        (0, 1),                          # one byte: its page
        (P + 1, P),                      # partial first and last pages: both dropped
        (P, 2 * P),                      # exactly pages 1 and 2
        (P - 1, 2),                      # two bytes across a page boundary
        (3 * P, TO_END),                 # from page 3 on
        (5 * P, TO_END - 5 * P + 10),    # off + size overflows: to the end
        (0, TO_END),                     # the whole object
        (LAST_PAGE * P, P),              # the last page a put accepts
        (LAST_PAGE * P + 7, TO_END),
        (14 * P, (1 << 63)),             # an end past 44 bits is clamped to the last page
        ((LAST_PAGE + 1) * P, TO_END),   # first page past 44 bits: nothing is cached there
        (0, 0),                          # empty range
    ]


@pytest.mark.parametrize("pshift", [12, 16])
def test_offset_and_size_become_one_interval_of_pages(exe, tmp_path, pshift):
    cases = _cases(pshift)
    flat = [str(x) for c in cases for x in c]
    head, calls, _log, out = _drive(exe, tmp_path / "c", "convert", pshift, *flat)
    rets = [int(x) for x in re.findall(r"^ret (\d+)$", head, re.M)]
    assert len(rets) == len(cases), out.stdout
    expect_calls = []
    for (off, size), ret in zip(cases, rets):
        iv = _interval(off, size, pshift)
        if iv is None:
            assert ret == 0, (off, size)
            continue
        expect_calls.append((0, 5, *iv))
        lo, hi = iv[0] & LAST_PAGE, iv[1] & LAST_PAGE
        assert ret == sum(lo <= p <= hi for p in PUT_PAGES), (off, size, iv)
    assert [c[:4] for c in calls] == expect_calls, out.stdout
    assert [c[4] for c in calls] == [r for (o, s), r in zip(cases, rets) if _interval(o, s, pshift)]


def test_a_page_in_the_ring_is_dropped_and_a_later_put_kept(exe, tmp_path):
    head, calls, _log, out = _drive(exe, tmp_path / "c", "ring")
    # page 1 had landed, page 2 was still held in the write-behind ring when the call came
    assert "removed 2" in head and "after 0 0" in head, out.stdout
    # the page put after the call returned is served, with its new content
    assert "later 1 2" in head, out.stdout
    assert calls == [(0, 9, 0, LAST_PAGE, 2)], out.stdout


def test_every_engine_is_called_and_the_counts_add_up(exe, tmp_path):
    head, calls, _log, out = _drive(exe, tmp_path / "c", "multi", CMB200_DEVICES="0,0,0")
    m = re.search(r"removed (\d+) engines (\d+) entries (\d+) hits (\d+) (\d+)", head)
    assert m, out.stdout
    removed, g, entries, h21, h22 = map(int, m.groups())
    assert (removed, g, entries, h21, h22) == (96, 3, 10, 0, 10), out.stdout
    assert sorted(c[0] for c in calls) == [0, 1, 2], out.stdout
    assert all(c[1:4] == (21, 0, LAST_PAGE) for c in calls), out.stdout
    assert sum(c[4] for c in calls) == 96 and all(c[4] > 0 for c in calls), out.stdout


def test_a_checkpoint_tick_writes_an_invalidation_only_change(exe, tmp_path):
    head, _calls, _log, out = _drive(exe, tmp_path / "c", "ckpt", CMB200_CHECKPOINT_SEC="1")
    m = re.search(r"removed (\d+) saves (\d+) (\d+) (\d+)", head)
    assert m, out.stdout
    removed, after_puts, idle, after_inv = map(int, m.groups())
    assert removed == 4 and after_puts >= 1, out.stdout
    assert idle == after_puts, out.stdout              # no change, no save
    assert after_inv == idle + 1, out.stdout           # the removal alone is saved
    assert (tmp_path / "c" / "cachemap_b200.snap").exists()


def test_a_call_before_the_engine_started_loads_the_snapshot_first(exe, tmp_path):
    d = tmp_path / "c"
    d.mkdir()
    (d / "cachemap_b200.snap").write_bytes(b"mock snapshot\n")
    head, calls, log, out = _drive(exe, d, "load", MOCK_LOAD_PAGES="8", MOCK_LOAD_NHID="7")
    assert "removed 8 hits 0" in head, out.stdout
    assert log.split()[:2] == ["load", "inv"], out.stdout
    assert calls == [(0, 7, 0, LAST_PAGE, 8)], out.stdout


@pytest.mark.parametrize("threads", [1, 8, 48])
def test_concurrent_puts_gets_and_invalidations(exe, tmp_path, threads):
    head, _calls, _log, out = _drive(exe, tmp_path / "c", "stress", threads, 1.5)
    m = re.search(r"errors (\d+) ops (\d+) hits (\d+)", head)
    assert m, out.stdout
    errors, ops, hits = map(int, m.groups())
    assert errors == 0 and ops > 100 and hits == 0, out.stdout


def test_concurrent_invalidations_have_no_data_race(tmp_path):
    exe, err = _build(tmp_path, "invalidate_drive_tsan", ["-fsanitize=thread"])
    if not exe:
        pytest.skip("gcc cannot link -fsanitize=thread here: " + err[-200:])
    head, _calls, _log, out = _drive(exe, tmp_path / "c", "stress", 16, 2)
    assert "ThreadSanitizer" not in out.stderr, out.stderr[-3000:]
    assert re.search(r"errors 0 ops \d+ hits 0", head), out.stdout
