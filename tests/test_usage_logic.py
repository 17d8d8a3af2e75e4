"""cachemap_residency and cachemap_usage without a GPU: edge_fuse_b200/csrc/cachemap_api.c over
tests/c/mock_usage.c, the CPU stand-in with pins and the usage calls, driven by tests/c/usage_drive.c and
checked against tests/usage_model.py.  Test infrastructure only: nothing of the product links the stand-in."""
import os
import subprocess

import pytest

import usage_model as UM

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = [os.path.join(ROOT, "edge_fuse_b200", "csrc", "cachemap_api.c"),
       os.path.join(ROOT, "tests", "c", "mock_usage.c"),
       os.path.join(ROOT, "tests", "c", "usage_drive.c")]
PAGE = 4096
REC = 24 + PAGE
G44 = 1 << 44


def _build(tmp_path, name, extra=()):
    exe = str(tmp_path / name)
    r = subprocess.run(["gcc", "-std=gnu11", "-O1", "-g", "-Wall", "-pthread", *extra, *SRC, "-o", exe],
                       capture_output=True, text=True)
    return exe, r


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    path, r = _build(tmp_path_factory.mktemp("usage"), "usage_drive")
    assert r.returncode == 0, r.stderr
    return path


def _drive(exe, d, cap, *steps, **env_extra):
    env = dict(os.environ, CMB200_WB_SLOTS="64", TSAN_OPTIONS="halt_on_error=1 report_signal_unsafe=0")
    for k in ("CMB200_DEVICES", "CMB200_DEVICE", "CMB200_EVICT", "CMB200_ADMIT", "CMB200_GHOST", "CMB200_HOST_TIER_MB",
              "CMB200_TIER_PROMOTE", "CMB200_CHECKPOINT_SEC", "CMB200_CHECKPOINT_DELTAS", "CMB200_PIN_MAX",
              "CMB200_KEY_FILE", "CMB200_LOAD"):
        env.pop(k, None)
    env["CMB200_PERSIST"] = "0"
    env.update(env_extra)
    os.makedirs(d, exist_ok=True)
    out = subprocess.run([exe, str(d), str(cap), *steps], capture_output=True, text=True, timeout=300, env=env)
    assert out.returncode == 0, out.stdout + out.stderr
    return out


def _res(out):
    return [(int(l.split()[1]), l.split()[2]) for l in out.stdout.splitlines() if l.startswith("res ")]


def _usages(out):
    """-> [(rc, [row tuples without the ts])] per usage step."""
    res = []
    for line in out.stdout.splitlines():
        w = line.split()
        if w[0] == "usage":
            res.append((int(w[1]), []))
        elif w[0] == "row":
            res[-1][1].append((int(w[1]), int(w[2]), 0, *(int(x) for x in w[3:])))
    return res


def _records(puts):
    """The model's records of put steps (u, genid, first, n); the stand-in keeps pages raw."""
    return {(u, g << 44 | p): (REC, False, 0) for u, g, f, n in puts for p in range(f, f + n)}


def _vec(v):
    return "".join(str(x) for x in v)


def test_argument_refusals_and_partial_pages(exe, tmp_path):
    steps = ["put:5:0:0:10", "res:5:0:0:0", f"res:5:0:0:{2 ** 64 - 1}", f"res:5:0:{G44 * PAGE}:1",
             f"res:5:0:{(G44 - 1) * PAGE}:{2 * PAGE}", f"res:5:0:{2 ** 64 - 2}:4",
             "res:5:0:4095:2", "res:5:0:100:40000", "res:5:1:0:4096", "res:6:0:0:8192"]
    got = _res(_drive(exe, tmp_path / "a", 4096, *steps))
    recs = _records([(5, 0, 0, 10)])
    # a refusal writes nothing: the vector stays as it was
    assert [rc for rc, _ in got[:5]] == [-1] * 5 and all(set(v) == {"."} for _, v in got[:5])
    assert all(UM.span(12, 0, *(int(x) for x in s.split(":")[3:])) is None for s in steps[1:6])
    want = [UM.residency(recs, [], 12, 5, 0, 4095, 2), UM.residency(recs, [], 12, 5, 0, 100, 40000),
            UM.residency(recs, [], 12, 5, 1, 0, 4096), UM.residency(recs, [], 12, 6, 0, 0, 8192)]
    # the vector's length is the pages the range overlaps: the canary right past it is untouched
    assert got[5:] == [(n, _vec(v) + ".") for n, v in want]
    assert got[5] == (2, "11.") and got[6] == (10, "1111111111.")


def test_a_page_put_just_before_the_call_is_counted(exe, tmp_path):
    out = _drive(exe, tmp_path / "a", 4096, "held:5:0:3", "res:5:0:0:16384", "held:5:0:4", "usage:4")
    assert _res(out) == [(1, "0001.")]
    assert _usages(out) == [(1, [(5, 0, 0, 2, 0, 0, 2 * REC, 3, 4)])]


def test_the_pinned_bit_on_cached_and_uncached_pages(exe, tmp_path):
    out = _drive(exe, tmp_path / "a", 4096, "put:5:0:0:6", "pin:5:0:16384:16384", "res:5:0:0:40960", "usage:4")
    recs = _records([(5, 0, 0, 6)])
    pins = [(5, 4, 7)]
    n, v = UM.residency(recs, pins, 12, 5, 0, 0, 40960)
    assert _res(out) == [(n, _vec(v) + ".")]
    assert _res(out)[0][1] == "1111554400."
    assert _usages(out) == [(1, [r[:9] for r in UM.usage(recs, pins, 4)[1]])]


PUTS = [(1, 0, 0, 40), (2, 0, 10, 40), (1, 1, 0, 20), (3, 0, 0, 60), (4, 0, 5, 40), (2, 1, 0, 40)]


@pytest.mark.parametrize("devices,g", [(None, 1), ("0,0,0", 3)])
def test_one_and_three_engines(exe, tmp_path, devices, g):
    extra = {"CMB200_DEVICES": devices} if devices else {}
    steps = [f"put:{u}:{gn}:{f}:{n}" for u, gn, f, n in PUTS] + ["usage:64", "usage:3", "usage:0", "res:3:0:0:409600"]
    out = _drive(exe, tmp_path / "a", 4096, *steps, **extra)
    recs = _records(PUTS)
    count, rows = UM.usage(recs, [], 64)
    want = [r[:9] for r in rows]
    u = _usages(out)
    assert u[0] == (count, want)
    # ties on 40 pages: nhid 1, 2 (genid 0 before 1) and 4 in order
    assert [(r[0], r[1]) for r in want] == [(3, 0), (1, 0), (2, 0), (2, 1), (4, 0), (1, 1)]
    assert u[1] == (count, want[:3])                     # max below the count
    assert u[2] == (count, [])                           # max = 0 counts only
    n, v = UM.residency(recs, [], 12, 3, 0, 0, 409600)
    assert _res(out) == [(n, _vec(v) + ".")] and n == 60
    assert "untouched 1" in out.stdout                 # rows past the count are not written


def test_an_object_spread_over_three_engines_sums_exactly(exe, tmp_path):
    out = _drive(exe, tmp_path / "a", 8192, "put:9:0:0:3000", "usage:4", CMB200_DEVICES="0,0,0")
    assert _usages(out) == [(1, [(9, 0, 0, 3000, 0, 0, 3000 * REC, 0, 2999)])]


@pytest.mark.parametrize("devices,k", [(None, 0), ("0,0,0", 2)])
def test_minus_one_when_an_engine_fails(exe, tmp_path, devices, k):
    extra = {"CMB200_DEVICES": devices} if devices else {}
    out = _drive(exe, tmp_path / "a", 4096, "put:5:0:0:30", f"fail:{k}", "usage:8", "res:5:0:0:8192", "fail:-1",
                 "usage:8", "res:5:0:0:8192", **extra)
    u = _usages(out)
    assert u[0] == (-1, []) and u[1][0] == 1
    assert _res(out) == [(-1, "..."), (2, "11.")]          # vec untouched while an engine fails


def test_both_calls_under_thread_sanitizer(tmp_path):
    exe, r = _build(tmp_path, "usage_drive_tsan", ["-fsanitize=thread"])
    if r.returncode != 0:
        pytest.skip("gcc cannot link -fsanitize=thread here: " + r.stderr[-200:])
    out = _drive(exe, tmp_path / "c", 1024, "race:4", "usage:8", CMB200_DEVICES="0,0")
    assert "WARNING: ThreadSanitizer" not in out.stderr, out.stderr[-4000:]
    assert out.stdout.splitlines()[0] == "race"
