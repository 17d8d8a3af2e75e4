"""CMB200_GHOST without a GPU: edge_fuse_b200/csrc/cachemap_api.c over tests/c/mock_ghost.c, the CPU stand-in of
tests/c/mock_engine.c that counts what reaches cmb200_evict_batch and cmb200_unset_batch and answers
cmb200_ghost_stats from a histogram the driver sets, driven by tests/c/ghost_drive.c.  Test infrastructure
only: nothing of the product links the stand-in."""
import os
import re
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = [os.path.join(ROOT, "edge_fuse_b200", "csrc", "cachemap_api.c"),
       os.path.join(ROOT, "tests", "c", "mock_ghost.c"),
       os.path.join(ROOT, "tests", "c", "ghost_drive.c")]
GHOST, FREQ = 16, 8


def _build(tmp_path, name, extra=()):
    exe = str(tmp_path / name)
    r = subprocess.run(["gcc", "-std=gnu11", "-O1", "-g", "-Wall", "-pthread", *extra, *SRC, "-o", exe],
                       capture_output=True, text=True)
    return exe, r


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    path, r = _build(tmp_path_factory.mktemp("ghost"), "ghost_drive")
    assert r.returncode == 0, r.stderr
    return path


def _drive(exe, d, mode, *args, ring=True, **env_extra):
    env = dict(os.environ, CMB200_PERSIST="0", CMB200_WB_SLOTS="64" if ring else "0",
               TSAN_OPTIONS="halt_on_error=1 report_signal_unsafe=0", **env_extra)
    for k in ("CMB200_DEVICES", "CMB200_DEVICE", "CMB200_EVICT", "CMB200_ADMIT", "CMB200_GHOST", "CMB200_HOST_TIER_MB",
              "CMB200_TIER_PROMOTE", "CMB200_CHECKPOINT_SEC", "CMB200_CHECKPOINT_DELTAS", "CMB200_VERIFY",
              "CMB200_FINGERPRINT"):
        if k not in env_extra:
            env.pop(k, None)
    os.makedirs(d, exist_ok=True)
    out = subprocess.run([exe, mode, str(d), *map(str, args)], capture_output=True, text=True, timeout=300, env=env)
    assert out.returncode == 0, out.stdout + out.stderr
    return out


def _counts(out):
    return [tuple(int(x) for x in m.groups()) for m in re.finditer(r"^counts (\d+) (\d+)$", out.stdout, re.M)]


@pytest.mark.parametrize("devices,g", [(None, 1), ("0,0,0", 3)])
def test_the_variable_sets_the_flag_on_every_engine(exe, tmp_path, devices, g):
    extra = {"CMB200_DEVICES": devices} if devices else {}
    out = _drive(exe, tmp_path / "c", "flags", CMB200_GHOST="1", **extra)
    m = re.search(r"engines (\d+) flags((?: \d+)*)", out.stdout)
    flags = [int(x) for x in m.group(2).split()]
    assert int(m.group(1)) == g and all(f & GHOST for f in flags), flags
    out = _drive(exe, tmp_path / "d", "flags", **extra)
    assert not any(int(x) & GHOST for x in re.search(r"flags((?: \d+)*)", out.stdout).group(1).split())


@pytest.mark.parametrize("ring", [True, False])
@pytest.mark.parametrize("devices", [None, "0,0,0"])
@pytest.mark.parametrize("ghost", [True, False])
def test_count_eviction_goes_through_evict_batch_only_with_the_flag(exe, tmp_path, ring, devices, ghost):
    """1056 pages into a map of 1024: 32 victims.  With the flag they reach cmb200_evict_batch and nothing is
    unset; a dropped put and a filemap_unset still go through cmb200_unset_batch.  Without it, every victim
    is unset, as before."""
    extra = {"CMB200_DEVICES": devices} if devices else {}
    if ghost:
        extra["CMB200_GHOST"] = "1"
    c = _counts(_drive(exe, tmp_path / "c", "evict", ring=ring, **extra))
    evicted, unset = c[0]
    # the dropped put is a new page at capacity: one more victim first, then its key is unset; then the unset
    if ghost:
        assert evicted >= 32 and unset == 0, c
        assert c[1] == (evicted + 1, 1) and c[2] == (evicted + 1, 2), c
    else:
        assert evicted == 0 and unset >= 32, c
        assert c[1] == (0, unset + 2) and c[2] == (0, unset + 3), c


@pytest.mark.parametrize("devices", [None, "0,0,0"])
def test_admission_victims_are_evictions_and_rejections_are_not(exe, tmp_path, devices):
    extra = {"CMB200_DEVICES": devices} if devices else {}
    c = _counts(_drive(exe, tmp_path / "c", "admit", CMB200_GHOST="1", CMB200_ADMIT="freq", **extra))
    assert c[0] == (0, 0), c                        # the map fills: nothing leaves
    assert c[1] == (0, 8), c                        # 8 rejected versions: their old records unset, no ghosts
    assert c[2] == (8, 8), c                        # 16 new pages: 8 fill the room, 8 evict a victim each


@pytest.mark.parametrize("devices,g", [(None, 1), ("0,0,0", 3)])
def test_the_curve_sums_each_engines_buckets_below_its_share(exe, tmp_path, devices, g):
    extras = [0, 3, 4, 4 * g, 4 * g + 3, 8 * g + 1, 200 * g, 256 * g, 10 ** 9]
    extra = {"CMB200_DEVICES": devices} if devices else {}
    out = _drive(exe, tmp_path / "c", "curve", *extras, CMB200_GHOST="1", **extra)
    m = re.search(r"^curve (-?\d+) (\d+)((?: \d+)*)$", out.stdout, re.M)
    assert int(m.group(1)) == 0, out.stdout
    assert int(m.group(2)) == sum(1000 * (k + 1) for k in range(g))
    got = [int(x) for x in m.group(3).split()]
    want = []
    for x in extras:
        b = min(64, x // g // 4)                    # the engine's share, rounded down to a bucket of 4
        want.append(sum((k + 1) * (j + 1) for k in range(g) for j in range(b)))
    assert got == want


def test_the_curve_needs_the_flag(exe, tmp_path):
    out = _drive(exe, tmp_path / "c", "curve", 100)
    assert re.search(r"^curve -1 ", out.stdout, re.M), out.stdout


def test_ghosts_under_thread_sanitizer(tmp_path):
    exe, r = _build(tmp_path, "ghost_drive_tsan", ["-fsanitize=thread"])
    if r.returncode != 0:
        pytest.skip("gcc cannot link -fsanitize=thread here: " + r.stderr[-200:])
    for mode, args, env in (("evict", (4,), {}), ("admit", (), {"CMB200_ADMIT": "freq"})):
        out = _drive(exe, tmp_path / mode, mode, *args, CMB200_GHOST="1", CMB200_DEVICES="0,0", **env)
        assert "ThreadSanitizer" not in out.stderr, out.stderr[-2000:]
        assert _counts(out), out.stdout
