"""cachemap_pin without a GPU: edge_fuse_b200/csrc/cachemap_api.c over tests/c/mock_pin.c, the CPU stand-in of
tests/c/mock_engine.c that keeps each engine's pin list and passes over pinned records when it samples,
driven by tests/c/pin_drive.c and checked against tests/pin_model.py.  Test infrastructure only: nothing of
the product links the stand-in."""
import os
import struct
import subprocess

import pytest

import pin_model as PM

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = [os.path.join(ROOT, "edge_fuse_b200", "csrc", "cachemap_api.c"),
       os.path.join(ROOT, "tests", "c", "mock_pin.c"),
       os.path.join(ROOT, "tests", "c", "pin_drive.c")]
PAGE = 4096
G44 = 1 << 44


def _build(tmp_path, name, extra=()):
    exe = str(tmp_path / name)
    r = subprocess.run(["gcc", "-std=gnu11", "-O1", "-g", "-Wall", "-pthread", *extra, *SRC, "-o", exe],
                       capture_output=True, text=True)
    return exe, r


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    path, r = _build(tmp_path_factory.mktemp("pin"), "pin_drive")
    assert r.returncode == 0, r.stderr
    return path


def _drive(exe, d, cap, *steps, **env_extra):
    env = dict(os.environ, CMB200_WB_SLOTS="64", TSAN_OPTIONS="halt_on_error=1 report_signal_unsafe=0")
    for k in ("CMB200_DEVICES", "CMB200_DEVICE", "CMB200_EVICT", "CMB200_ADMIT", "CMB200_GHOST", "CMB200_HOST_TIER_MB",
              "CMB200_TIER_PROMOTE", "CMB200_CHECKPOINT_SEC", "CMB200_CHECKPOINT_DELTAS", "CMB200_PIN_MAX",
              "CMB200_KEY_FILE", "CMB200_PERSIST", "CMB200_LOAD"):
        env.pop(k, None)
    env.update(env_extra)
    os.makedirs(d, exist_ok=True)
    out = subprocess.run([exe, str(d), str(cap), *steps], capture_output=True, text=True, timeout=300, env=env)
    assert out.returncode == 0, out.stdout + out.stderr
    return out


def _lines(out, word):
    return [l.split()[1:] for l in out.stdout.splitlines() if l.split()[0] == word]


def _lists(out):
    lines = out.stdout.splitlines()
    k = max(i for i, l in enumerate(lines) if l.startswith("lists "))
    g = int(lines[k].split()[1])
    res = []
    for l in lines[k + 1:k + 1 + g]:
        res.append([tuple(int(x) for x in r.split(":")) for r in l.split()[2:]])
    return res


def _run_model(cap, steps, pin_max=None):
    m = PM.Pins(cap, 12, pin_max)
    want = []
    for s in steps:
        f = s.split(":")
        a = [PM.TO_END if x == "end" else int(x) for x in f[1:]]
        if f[0] == "pin":
            want.append(["pin", m.pin(*a)])
        elif f[0] == "unpin":
            want.append(["unpin", m.unpin(*a)])
        elif f[0] == "rename":
            m.rename(*a)
    return m, want


STEPS = ["pin:5:0:0:40960", "pin:5:0:40960:8192", "pin:5:0:16384:4096", "pin:6:0:100:1", "pin:5:1:0:4096",
         "unpin:5:0:8192:8192", "unpin:5:0:0:1", "pin:5:0:4095:2", "unpin:6:0:0:end", "pin:5:0:0:0",
         "pin:5:0:0:end", f"pin:5:0:{G44 * PAGE}:4096", f"pin:7:0:{(G44 - 2) * PAGE}:{1 << 62}", "unpin:7:0:0:end",
         "pin:5:2:4096:2"]


@pytest.mark.parametrize("devices,g", [(None, 1), ("0,0,0", 3)])
def test_merge_split_refusals_and_the_list_on_every_engine(exe, tmp_path, devices, g):
    extra = {"CMB200_DEVICES": devices} if devices else {}
    out = _drive(exe, tmp_path / "c", 4096, *STEPS, "lists", CMB200_PERSIST="0", **extra)
    m, want = _run_model(4096, STEPS)
    got = [[w, int(v[0])] for w, v in ((l.split()[0], l.split()[1:]) for l in out.stdout.splitlines())
           if w in ("pin", "unpin")]
    assert got == want
    lists = _lists(out)
    assert len(lists) == g and all(l == m.ranges for l in lists), (lists, m.ranges)
    assert m.ranges and len(m.ranges) > 2


def test_the_budget_refuses_and_clamps(exe, tmp_path):
    steps = ["pin:5:0:0:4096000", "pin:5:0:0:2097152", "pin:5:0:2093056:8192", "stats"]
    out = _drive(exe, tmp_path / "a", 4096, *steps, CMB200_PERSIST="0", CMB200_PIN_MAX="3000")
    m, want = _run_model(4096, steps[:3], 3000)
    assert [["pin", int(v[0])] for v in _lines(out, "pin")] == want
    assert "above half the capacity" in out.stderr
    out = _drive(exe, tmp_path / "b", 4096, "pin:5:0:0:4096", CMB200_PERSIST="0", CMB200_PIN_MAX="0")
    assert _lines(out, "pin") == [["-1"]]


def test_too_many_ranges_are_refused(exe, tmp_path):
    steps = [f"pin:5:0:{2 * k * PAGE}:{PAGE}" for k in range(PM.PIN_RANGES + 1)]
    out = _drive(exe, tmp_path / "c", 1 << 16, *steps, "stats", CMB200_PERSIST="0")
    got = [int(v[0]) for v in _lines(out, "pin")]
    assert got == [1] * PM.PIN_RANGES + [-1]
    assert _lines(out, "stats") == [[str(PM.PIN_RANGES), "0", "0"]]


def test_a_rename_moves_the_pins_before_the_pages(exe, tmp_path):
    # the stand-in cannot move pages, so the drop-in drops those of `from`; the pins move all the same
    steps = ["pin:5:0:0:65536", "pin:5:1:0:4096", "pin:6:0:0:8192", "put:5:0:16", "lists", "rename:5:6:0", "lists",
             "stats"]
    out = _drive(exe, tmp_path / "c", 4096, *steps, CMB200_PERSIST="0", CMB200_DEVICES="0,0")
    m, _ = _run_model(4096, steps)
    assert all(l == m.ranges for l in _lists(out))
    assert m.ranges == [(5, G44, G44), (6, 0, 15)]
    assert _lines(out, "rename") == [["0"]]
    assert _lines(out, "stats") == [["17", "0", "0"]]
    assert "lists 2 6" in out.stdout and "lists 2 8" in out.stdout   # one more list per engine: before the move


@pytest.mark.parametrize("devices", [None, "0,0,0"])
def test_pinned_pages_survive_a_flood(exe, tmp_path, devices):
    extra = {"CMB200_DEVICES": devices} if devices else {}
    steps = ["pin:1:0:0:262144", "put:1:0:64", "put:9:0:4096", "read:1:0:64", "stats", "unpin:1:0:0:end",
             "put:9:5000:4096", "read:1:0:64"]
    out = _drive(exe, tmp_path / "c", 1024, *steps, CMB200_PERSIST="0", **extra)
    assert _lines(out, "read")[0] == ["64"] and int(_lines(out, "read")[1][0]) < 64
    assert _lines(out, "stats") == [["64", "64", "0"]]


def test_a_pinned_page_is_always_admitted(exe, tmp_path):
    # 1024 cold pages fill the map; then pinned cold pages of another object are put: estimate 0 against
    # victims of 0 would reject them, the pin admits them all
    steps = ["put:9:0:1024", "pin:1:0:0:131072", "put:1:0:32", "admission", "read:1:0:32", "stats"]
    out = _drive(exe, tmp_path / "c", 1024, *steps, CMB200_PERSIST="0", CMB200_ADMIT="freq")
    assert _lines(out, "admission") == [["32", "0"]]
    assert _lines(out, "read") == [["32"]]
    out = _drive(exe, tmp_path / "d", 1024, *[s for s in steps if not s.startswith("pin")], CMB200_PERSIST="0",
                 CMB200_ADMIT="freq")
    assert _lines(out, "admission") == [["0", "32"]]


def _pins_file(d):
    return open(os.path.join(d, "cachemap_b200.pins"), "rb").read()


def _parse(raw):
    magic, ver, pshift, n, nonce = struct.unpack_from("<8sIIQQ", raw)
    ranges = [struct.unpack_from("<QQQ", raw, 32 + 24 * k) for k in range(n)]
    return magic, ver, pshift, nonce, ranges


@pytest.mark.parametrize("sealed", [False, True])
def test_the_pins_file_round_trip(exe, tmp_path, sealed):
    d = tmp_path / "c"
    env = {}
    if sealed:
        (tmp_path / "key").write_bytes(bytes(range(32)))
        env["CMB200_KEY_FILE"] = str(tmp_path / "key")
    _drive(exe, d, 4096, "pin:5:0:0:40960", "pin:6:2:0:4096", "unpin:5:0:8192:4096", **env)
    raw = _pins_file(d)
    magic, ver, pshift, nonce, ranges = _parse(raw)
    assert magic == (b"CMB200Q1" if sealed else b"CMB200P1") and ver == 1 and pshift == 12
    assert ranges == [(5, 0, 1), (5, 3, 9), (6, 2 * G44, 2 * G44)]
    assert len(raw) == 32 + 24 * 3 + (16 if sealed else 0) and (nonce != 0) == sealed
    out = _drive(exe, d, 4096, "stats", "lists", **env)
    assert _lines(out, "stats")[0][0] == "10" and _lists(out)[0] == ranges
    if sealed:
        # a plaintext file loads under a key and the next write seals it
        _drive(exe, tmp_path / "p", 4096, "pin:5:0:0:4096")
        assert _pins_file(tmp_path / "p")[:8] == b"CMB200P1"
        out = _drive(exe, tmp_path / "p", 4096, "stats", "pin:5:0:4096:4096", **env)
        assert _lines(out, "stats") == [["1", "0", "0"]]
        assert _pins_file(tmp_path / "p")[:8] == b"CMB200Q1"
        # without the key a sealed file is ignored
        out = _drive(exe, d, 4096, "stats")
        assert _lines(out, "stats") == [["0", "0", "0"]] and "ignored" in out.stderr


def _rewrite(d, raw):
    with open(os.path.join(d, "cachemap_b200.pins"), "wb") as f:
        f.write(raw)


def test_damaged_wrong_size_and_over_budget_files(exe, tmp_path):
    d = tmp_path / "c"
    _drive(exe, d, 4096, "pin:5:0:0:40960", "pin:6:0:0:40960", "pin:7:0:0:40960")
    raw = _pins_file(d)
    magic, ver, pshift, nonce, ranges = _parse(raw)
    # another page size: ignored
    _rewrite(d, raw[:12] + struct.pack("<I", 16) + raw[16:])
    out = _drive(exe, d, 4096, "stats")
    assert _lines(out, "stats") == [["0", "0", "0"]] and "another page size" in out.stderr
    # a short file keeps its whole ranges
    _rewrite(d, raw[:32 + 24 + 10])
    out = _drive(exe, d, 4096, "stats", "lists")
    assert _lines(out, "stats") == [["10", "0", "0"]] and "short" in out.stderr
    # out of order: the ranges before it
    bad = bytearray(raw)
    bad[32 + 48:32 + 72] = struct.pack("<QQQ", 5, 3, 4)
    _rewrite(d, bytes(bad))
    out = _drive(exe, d, 4096, "stats")
    assert _lines(out, "stats") == [["20", "0", "0"]]
    # over the budget: file order while it allows
    _rewrite(d, raw)
    out = _drive(exe, d, 4096, "stats", "lists", CMB200_PIN_MAX="25")
    m = PM.Pins(4096, 12, 25)
    m.load(ranges)
    assert _lines(out, "stats") == [[str(PM.pages(m.ranges)), "0", "0"]] and _lists(out)[0] == m.ranges
    # garbage
    _rewrite(d, b"nonsense")
    out = _drive(exe, d, 4096, "stats")
    assert _lines(out, "stats") == [["0", "0", "0"]] and "not a pins file" in out.stderr


def test_a_tampered_sealed_file_is_ignored(exe, tmp_path):
    d = tmp_path / "c"
    (tmp_path / "key").write_bytes(bytes(range(32)))
    env = {"CMB200_KEY_FILE": str(tmp_path / "key")}
    _drive(exe, d, 4096, "pin:5:0:0:40960", **env)
    raw = bytearray(_pins_file(d))
    raw[33] ^= 1
    _rewrite(d, bytes(raw))
    out = _drive(exe, d, 4096, "stats", **env)
    assert _lines(out, "stats") == [["0", "0", "0"]] and "tag fails" in out.stderr


def test_persist_off_reads_and_writes_nothing(exe, tmp_path):
    d = tmp_path / "c"
    _drive(exe, d, 4096, "pin:5:0:0:40960", CMB200_PERSIST="0")
    assert not os.path.exists(d / "cachemap_b200.pins")
    _drive(exe, d, 4096, "pin:5:0:0:40960")
    out = _drive(exe, d, 4096, "stats", CMB200_PERSIST="0")
    assert _lines(out, "stats") == [["0", "0", "0"]]


def test_pins_under_thread_sanitizer(tmp_path):
    exe, r = _build(tmp_path, "pin_drive_tsan", ["-fsanitize=thread"])
    if r.returncode != 0:
        pytest.skip("gcc cannot link -fsanitize=thread here: " + r.stderr[-200:])
    out = _drive(exe, tmp_path / "c", 1024, "race:4", "stats", CMB200_DEVICES="0,0", CMB200_PERSIST="0")
    assert "ThreadSanitizer" not in out.stderr, out.stderr[-2000:]
    assert _lines(out, "race") == [[]]
