"""The drop-in's CMB200_KEY_FILE without a GPU: edge_fuse_b200/csrc/cachemap_api.c over the CPU stand-in of
tests/c/mock_key.c, driven by tests/c/chain_drive.c (puts, then cachemap_free).  A key file that is
missing or malformed turns persistence off: the directory is neither read nor written.  A good one, as
32 raw bytes or 64 hex digits, is set on every engine of CMB200_DEVICES before the directory is read.
Test infrastructure only: nothing of the product links the stand-ins."""
import os
import re
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
API = os.path.join(ROOT, "edge_fuse_b200", "csrc", "cachemap_api.c")
KEY = bytes(range(0xA0, 0xC0))


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    path = str(tmp_path_factory.mktemp("key") / "key_drive")
    r = subprocess.run(["gcc", "-std=gnu11", "-O1", "-g", "-pthread", API, os.path.join(ROOT, "tests", "c", "mock_key.c"),
                        os.path.join(ROOT, "tests", "c", "chain_drive.c"), "-o", path], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return path


def _drive(exe, d, **env_extra):
    env = dict(os.environ, CMB200_PERSIST="1", CMB200_WB_SLOTS="64")
    for k in ("CMB200_DEVICES", "CMB200_DEVICE", "CMB200_HOST_TIER_MB", "CMB200_TIER_PROMOTE", "CMB200_KEY_FILE",
              "CMB200_CHECKPOINT_SEC", "CMB200_CHECKPOINT_DELTAS", "CMB200_LOAD"):
        env.pop(k, None)
    env.update(env_extra)
    os.makedirs(d, exist_ok=True)
    base = d / "cachemap_b200.snap"
    if not base.exists():
        base.write_bytes(b"\0" * 4096)
    out = subprocess.run([exe, str(d), "0.1"], capture_output=True, text=True, timeout=120, env=env)
    m = re.search(r"^calls: ?(.*)$", out.stdout, re.M)
    assert out.returncode == 0 and m, out.stdout + out.stderr
    return m.group(1).split(), out.stderr


def test_no_key_file_sets_no_key(exe, tmp_path):
    calls, _ = _drive(exe, tmp_path / "d")
    assert not any(c.startswith("key:") for c in calls)
    assert "load_set" in calls and "save_set" in calls


@pytest.mark.parametrize("form", ["raw", "hex", "hex-newline"])
def test_a_good_key_is_set_on_every_engine_before_the_load(exe, tmp_path, form):
    kf = tmp_path / "key"
    kf.write_bytes(KEY if form == "raw" else (KEY.hex().upper() if form == "hex" else KEY.hex() + "\n").encode())
    calls, _ = _drive(exe, tmp_path / "d", CMB200_KEY_FILE=str(kf), CMB200_DEVICES="0,0,0")
    keys = [c for c in calls if c.startswith("key:")]
    assert keys == ["key:" + KEY.hex()] * 3
    assert calls.index("load_set") > max(i for i, c in enumerate(calls) if c.startswith("key:"))
    assert "save_set" in calls


@pytest.mark.parametrize("content", [None, b"", KEY[:31], KEY + b"x", b"zz" * 32, (KEY.hex() + "0").encode()])
def test_a_bad_or_missing_key_file_turns_persistence_off(exe, tmp_path, content):
    kf = tmp_path / "key"
    if content is not None:
        kf.write_bytes(content)
    calls, err = _drive(exe, tmp_path / "d", CMB200_KEY_FILE=str(kf))
    assert not any(c.startswith("key:") for c in calls)
    assert not any(c in ("load_set", "load_chain", "save_set", "base") for c in calls), calls
    assert "CMB200_KEY_FILE" in err
