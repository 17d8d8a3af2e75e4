"""CMB200_ADMIT without a GPU: edge_fuse_b200/csrc/cachemap_api.c over tests/c/mock_freq.c, the CPU stand-in
of tests/c/mock_engine.c that keeps the CMB200_FREQ sketch with the header's cmb200_freq_index, driven by
tests/c/admit_drive.c.  Test infrastructure only: nothing of the product links the stand-in."""
import os
import re
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = [os.path.join(ROOT, "edge_fuse_b200", "csrc", "cachemap_api.c"),
       os.path.join(ROOT, "tests", "c", "mock_freq.c"),
       os.path.join(ROOT, "tests", "c", "admit_drive.c")]
FREQ = 8


def _build(tmp_path, name, extra=()):
    exe = str(tmp_path / name)
    r = subprocess.run(["gcc", "-std=gnu11", "-O1", "-g", "-Wall", "-pthread", *extra, *SRC, "-o", exe],
                       capture_output=True, text=True)
    return exe, r


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    path, r = _build(tmp_path_factory.mktemp("admit"), "admit_drive")
    assert r.returncode == 0, r.stderr
    return path


def _drive(exe, d, mode, ring=True, **env_extra):
    env = dict(os.environ, CMB200_PERSIST="0", CMB200_WB_SLOTS="64" if ring else "0",
               TSAN_OPTIONS="halt_on_error=1 report_signal_unsafe=0", **env_extra)
    for k in ("CMB200_DEVICES", "CMB200_DEVICE", "CMB200_EVICT", "CMB200_ADMIT", "CMB200_HOST_TIER_MB",
              "CMB200_TIER_PROMOTE", "CMB200_CHECKPOINT_SEC", "CMB200_CHECKPOINT_DELTAS", "CMB200_VERIFY",
              "CMB200_FINGERPRINT"):
        if k not in env_extra:
            env.pop(k, None)
    os.makedirs(d, exist_ok=True)
    out = subprocess.run([exe, mode, str(d)], capture_output=True, text=True, timeout=300, env=env)
    assert out.returncode == 0, out.stdout + out.stderr
    return out


def _values(out):
    return {m.group(1): [int(x) for x in m.group(2).split()]
            for m in re.finditer(r"^(\w+) ([\d ]+)$", out.stdout, re.M)}


def _flags(out):
    m = re.search(r"engines (\d+) flags((?: \d+)*)", out.stdout)
    assert m, out.stdout
    return int(m.group(1)), [int(x) for x in m.group(2).split()]


@pytest.mark.parametrize("devices,g", [(None, 1), ("0,0,0", 3)])
def test_freq_sets_the_sketch_flag_on_every_engine(exe, tmp_path, devices, g):
    extra = {"CMB200_DEVICES": devices} if devices else {}
    n, flags = _flags(_drive(exe, tmp_path / "c", "flags", CMB200_ADMIT="freq", **extra))
    assert n == g and len(flags) == g
    assert all(f & FREQ for f in flags), flags


def test_freq_combines_with_access(exe, tmp_path):
    _g, flags = _flags(_drive(exe, tmp_path / "c", "flags", CMB200_ADMIT="freq", CMB200_EVICT="access",
                              CMB200_DEVICES="0,0,0"))
    assert all(f & FREQ and f & 4 for f in flags), flags


@pytest.mark.parametrize("value", [None, "all"])
def test_all_or_unset_admits_every_page(exe, tmp_path, value):
    extra = {"CMB200_ADMIT": value} if value else {}
    out = _drive(exe, tmp_path / "c", "flags", CMB200_DEVICES="0,0", **extra)
    _g, flags = _flags(out)
    assert not any(f & FREQ for f in flags), flags
    assert "CMB200_ADMIT" not in out.stderr
    v = _values(_drive(exe, tmp_path / "r", "reject", **extra))
    assert v["old"] == [1] and v["new"] == [1] and v["admission"] == [0, 0], v


def test_an_unknown_value_warns_once_and_admits_all(exe, tmp_path):
    out = _drive(exe, tmp_path / "c", "flags", CMB200_DEVICES="0,0", CMB200_ADMIT="lfu")
    _g, flags = _flags(out)
    assert not any(f & FREQ for f in flags), flags
    assert out.stderr.count("CMB200_ADMIT=lfu") == 1, out.stderr


@pytest.mark.parametrize("ring", [True, False])
@pytest.mark.parametrize("devices", [None, "0,0,0"])
def test_a_rejected_page_is_not_stored_and_its_old_record_is_unset(exe, tmp_path, ring, devices):
    """Pages whose estimate is 0 never beat a victim: the new version of a cached page is rejected and the
    old version is unset with it; a new page is not stored."""
    extra = {"CMB200_DEVICES": devices} if devices else {}
    v = _values(_drive(exe, tmp_path / "c", "reject", ring=ring, CMB200_ADMIT="freq", **extra))
    assert v["old"] == [0] and v["new"] == [0], v
    assert v["admission"] == [0, 2], v
    assert v["entries"] == [1023], v


@pytest.mark.parametrize("ring", [True, False])
@pytest.mark.parametrize("devices", [None, "0,0,0"])
def test_an_admitted_page_evicts_its_victim(exe, tmp_path, ring, devices):
    """A page read three times beats a victim nobody read: it is stored and one record leaves."""
    extra = {"CMB200_DEVICES": devices} if devices else {}
    v = _values(_drive(exe, tmp_path / "c", "admit", ring=ring, CMB200_ADMIT="freq", **extra))
    assert v["new"] == [1] and v["entries"] == [1024], v
    assert v["admission"] == [1, 0], v


def test_admission_under_thread_sanitizer(tmp_path):
    exe, r = _build(tmp_path, "admit_drive_tsan", ["-fsanitize=thread"])
    if r.returncode != 0:
        pytest.skip("gcc cannot link -fsanitize=thread here: " + r.stderr[-200:])
    for mode in ("reject", "admit"):
        out = _drive(exe, tmp_path / mode, mode, CMB200_ADMIT="freq", CMB200_DEVICES="0,0")
        assert "ThreadSanitizer" not in out.stderr, out.stderr[-2000:]
