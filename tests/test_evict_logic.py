"""CMB200_EVICT without a GPU: edge_fuse_b200/csrc/cachemap_api.c over tests/c/mock_touch.c, the CPU
stand-in of tests/c/mock_engine.c whose gets raise a record's ts on a hit when the engine was created with
CMB200_TOUCH, driven by tests/c/evict_drive.c.  Test infrastructure only: nothing of the product links
the stand-in."""
import os
import re
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = [os.path.join(ROOT, "edge_fuse_b200", "csrc", "cachemap_api.c"),
       os.path.join(ROOT, "tests", "c", "mock_touch.c"),
       os.path.join(ROOT, "tests", "c", "evict_drive.c")]
TOUCH = 4


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    path = str(tmp_path_factory.mktemp("evict") / "evict_drive")
    r = subprocess.run(["gcc", "-std=gnu11", "-O1", "-g", "-Wall", "-pthread", *SRC, "-o", path],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return path


def _drive(exe, d, mode, **env_extra):
    env = dict(os.environ, CMB200_PERSIST="0", CMB200_WB_SLOTS="64", **env_extra)
    for k in ("CMB200_DEVICES", "CMB200_DEVICE", "CMB200_EVICT", "CMB200_HOST_TIER_MB", "CMB200_TIER_PROMOTE",
              "CMB200_CHECKPOINT_SEC", "CMB200_CHECKPOINT_DELTAS", "CMB200_VERIFY", "CMB200_FINGERPRINT"):
        if k not in env_extra:
            env.pop(k, None)
    os.makedirs(d, exist_ok=True)
    out = subprocess.run([exe, mode, str(d)], capture_output=True, text=True, timeout=120, env=env)
    assert out.returncode == 0, out.stdout + out.stderr
    return out


def _flags(out):
    m = re.search(r"engines (\d+) flags((?: \d+)*)", out.stdout)
    assert m, out.stdout
    return int(m.group(1)), [int(x) for x in m.group(2).split()]


@pytest.mark.parametrize("devices", [None, "0,0"])
def test_access_sets_the_touch_flag_on_every_engine(exe, tmp_path, devices):
    extra = {"CMB200_DEVICES": devices} if devices else {}
    g, flags = _flags(_drive(exe, tmp_path / "c", "flags", CMB200_EVICT="access", **extra))
    assert g == (2 if devices else 1) and len(flags) == g
    assert all(f & TOUCH for f in flags), flags


@pytest.mark.parametrize("value", [None, "put"])
def test_put_or_unset_keeps_the_reference_policy(exe, tmp_path, value):
    extra = {"CMB200_EVICT": value} if value else {}
    out = _drive(exe, tmp_path / "c", "flags", CMB200_DEVICES="0,0", **extra)
    _g, flags = _flags(out)
    assert not any(f & TOUCH for f in flags), flags
    assert "CMB200_EVICT" not in out.stderr


def test_an_unknown_value_warns_once_and_keeps_put(exe, tmp_path):
    out = _drive(exe, tmp_path / "c", "flags", CMB200_DEVICES="0,0", CMB200_EVICT="lru")
    _g, flags = _flags(out)
    assert not any(f & TOUCH for f in flags), flags
    assert out.stderr.count("CMB200_EVICT=lru") == 1, out.stderr


def test_a_page_that_is_read_is_not_the_victim(exe, tmp_path):
    """Under access the 8 read pages are newer than every other record but the 8 put after them, so a put
    at capacity evicts one of them only if all three draws fall on those 16 of 1024 records."""
    out = _drive(exe, tmp_path / "c", "victim", CMB200_EVICT="access")
    assert "raised 8\n" in out.stdout and "kept 8\n" in out.stdout, out.stdout


def test_without_access_a_read_leaves_the_put_time(exe, tmp_path):
    out = _drive(exe, tmp_path / "c", "victim", CMB200_EVICT="put")
    assert "raised 0\n" in out.stdout, out.stdout
