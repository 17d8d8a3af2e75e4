"""cachemap_rename without a GPU: edge_fuse_b200/csrc/cachemap_api.c over the CPU stand-in of
tests/c/mock_rename.c, which moves records by stored address and logs every cmb200_invalidate and
cmb200_rename_set call, driven by tests/c/rename_drive.c.  Test infrastructure only: nothing of the
product links the stand-in."""
import os
import re
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = [os.path.join(ROOT, "edge_fuse_b200", "csrc", "cachemap_api.c"),
       os.path.join(ROOT, "tests", "c", "mock_rename.c"),
       os.path.join(ROOT, "tests", "c", "rename_drive.c")]
LAST = (1 << 44) - 1                               # genid 0: the whole page range
TO, FROM = 50, 51


def _build(tmp_path, name, extra):
    exe = str(tmp_path / name)
    r = subprocess.run(["gcc", "-std=gnu11", "-O1", "-g", "-Wall", "-pthread", *extra, *SRC, "-o", exe],
                       capture_output=True, text=True)
    return exe if r.returncode == 0 else None, r.stderr


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    path, err = _build(tmp_path_factory.mktemp("ren"), "rename_drive", [])
    assert path, err
    return path


@pytest.fixture(scope="module")
def exe_without_rename(tmp_path_factory):
    path, err = _build(tmp_path_factory.mktemp("ren0"), "rename_drive0", ["-DMOCK_NO_RENAME"])
    assert path, err
    return path


def _drive(exe, d, *args, ring=True, **env_extra):
    env = dict(os.environ, CMB200_PERSIST="1", CMB200_WB_SLOTS="64" if ring else "0",
               TSAN_OPTIONS="halt_on_error=0 report_signal_unsafe=0", **env_extra)
    for k in ("CMB200_DEVICES", "CMB200_DEVICE", "CMB200_HOST_TIER_MB", "CMB200_TIER_PROMOTE",
              "CMB200_CHECKPOINT_SEC", "CMB200_CHECKPOINT_DELTAS", "MOCK_RENAME_FAIL", "MOCK_RENAME_PAUSE_US"):
        if k not in env_extra:
            env.pop(k, None)
    os.makedirs(d, exist_ok=True)
    out = subprocess.run([exe, args[0], str(d), *map(str, args[1:])], capture_output=True, text=True,
                         timeout=300, env=env)
    assert out.returncode == 0 and "\nlog:\n" in out.stdout, out.stdout + out.stderr
    head, log = out.stdout.split("\nlog:\n", 1)
    calls = [ln.split() for ln in log.splitlines() if ln.startswith(("inv ", "ren"))]
    return head, calls, out


def _result(head):
    m = re.search(r"moved (\d+) right (\d+) gone (\d+)", head)
    assert m, head
    return tuple(map(int, m.groups()))


@pytest.mark.parametrize("ring", [True, False])
@pytest.mark.parametrize("devices", [None, "0,0,0"])
def test_to_is_dropped_then_from_moves(exe, tmp_path, ring, devices):
    extra = {"CMB200_DEVICES": devices} if devices else {}
    g = 3 if devices else 1
    head, calls, out = _drive(exe, tmp_path / "c", "basic", ring=ring, **extra)
    # 20 pages of `from` now answer as `to`; the 12 pages of `to` beyond them and all of `from` miss
    assert _result(head) == (20, 20, 32), out.stdout
    assert "same 0" in head
    # in order: every engine drops the pages of `to`, then one move over all engines
    inv = [c for c in calls if c[0] == "inv"]
    assert [c[0] for c in calls] == ["inv"] * g + ["ren", "ren-done"], out.stdout
    assert sorted(int(c[1]) for c in inv) == list(range(g))
    assert all(c[2:5] == [str(TO), "0", str(LAST)] for c in inv), out.stdout
    assert sum(int(c[5]) for c in inv) == 32
    assert calls[g] == ["ren", str(g), str(FROM), str(TO), "0", str(LAST)], out.stdout
    assert calls[g + 1] == ["ren-done", "20"]


def test_a_page_of_from_in_the_ring_is_moved(exe, tmp_path):
    head, calls, out = _drive(exe, tmp_path / "c", "ring")
    # pages 2.. of `from` were still held in the write-behind ring when the call came
    assert _result(head) == (20, 20, 32), out.stdout
    assert [c[0] for c in calls] == ["inv", "ren", "ren-done"], out.stdout


@pytest.mark.parametrize("ring", [True, False])
def test_room_locks_are_held_around_the_move(exe, tmp_path, ring):
    head, calls, out = _drive(exe, tmp_path / "c", "room", ring=ring, MOCK_RENAME_PAUSE_US="200000")
    assert _result(head) == (20, 20, 32), out.stdout
    # a put of another object that came during the call waited for it
    assert ["ren-overlap"] not in calls, out.stdout


@pytest.mark.parametrize("how", ["missing", "failing"])
@pytest.mark.parametrize("devices", [None, "0,0,0"])
def test_without_the_move_from_is_dropped(exe, exe_without_rename, tmp_path, how, devices):
    extra = {"CMB200_DEVICES": devices} if devices else {}
    g = 3 if devices else 1
    if how == "missing":
        head, calls, out = _drive(exe_without_rename, tmp_path / "c", "basic", **extra)
    else:
        head, calls, out = _drive(exe, tmp_path / "c", "basic", MOCK_RENAME_FAIL="1", **extra)
    # nothing moved: every page of both names misses, none is served stale
    assert _result(head) == (0, 0, 32), out.stdout
    names = [c[0] for c in calls]
    want = ["inv"] * g + (["ren"] if how == "failing" else []) + ["inv"] * g
    assert names == want, out.stdout
    inv = [c for c in calls if c[0] == "inv"]
    assert [c[2] for c in inv] == [str(TO)] * g + [str(FROM)] * g
    assert sum(int(c[5]) for c in inv[g:]) == 20


def test_a_checkpoint_tick_writes_a_rename_only_change(exe, tmp_path):
    head, _calls, out = _drive(exe, tmp_path / "c", "ckpt", CMB200_CHECKPOINT_SEC="1")
    m = re.search(r"moved (\d+) saves (\d+) (\d+) (\d+)", head)
    assert m, out.stdout
    moved, after_puts, idle, after = map(int, m.groups())
    assert moved == 8 and after_puts >= 1, out.stdout
    assert idle == after_puts, out.stdout              # no change, no save
    assert after == idle + 1, out.stdout               # the move alone is saved


@pytest.mark.parametrize("threads", [1, 8, 32])
def test_concurrent_puts_gets_and_renames(exe, tmp_path, threads):
    head, _calls, out = _drive(exe, tmp_path / "c", "stress", threads, 1.5, CMB200_DEVICES="0,0")
    m = re.search(r"errors (\d+) ops (\d+) hits (\d+)", head)
    assert m, out.stdout
    errors, ops, hits = map(int, m.groups())
    assert errors == 0 and ops > 100 and hits == 0, out.stdout


def test_concurrent_renames_have_no_data_race(tmp_path):
    exe, err = _build(tmp_path, "rename_drive_tsan", ["-fsanitize=thread"])
    if not exe:
        pytest.skip("gcc cannot link -fsanitize=thread here: " + err[-200:])
    head, _calls, out = _drive(exe, tmp_path / "c", "stress", 16, 2, CMB200_DEVICES="0,0")
    assert "ThreadSanitizer" not in out.stderr, out.stderr[-3000:]
    assert re.search(r"errors 0 ops \d+ hits 0", head), out.stdout
