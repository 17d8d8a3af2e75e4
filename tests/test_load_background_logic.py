"""The drop-in's CMB200_LOAD=background without a GPU: edge_fuse_b200/csrc/cachemap_api.c over the CPU stand-in
of tests/c/mock_load.c, whose cmb200_load_step blocks until the driver tests/c/load_drive.c releases it.
The same driver over tests/c/mock_chain.c alone stands for an engine without the background-load calls.
Test infrastructure only: nothing of the product links the stand-ins."""
import os
import re
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
API = os.path.join(ROOT, "edge_fuse_b200", "csrc", "cachemap_api.c")
DRIVE = os.path.join(ROOT, "tests", "c", "load_drive.c")


def _build(tmp_path, name, mock, extra=()):
    exe = str(tmp_path / name)
    src = [API, os.path.join(ROOT, "tests", "c", mock), DRIVE]
    r = subprocess.run(["gcc", "-std=gnu11", "-O1", "-g", "-pthread", *extra, *src, "-o", exe],
                       capture_output=True, text=True)
    return exe if r.returncode == 0 else None, r.stderr


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    path, err = _build(tmp_path_factory.mktemp("load"), "load_drive", "mock_load.c")
    assert path, err
    return path


@pytest.fixture(scope="module")
def exe_without(tmp_path_factory):
    path, err = _build(tmp_path_factory.mktemp("load_chain"), "load_drive_chain", "mock_chain.c")
    assert path, err
    return path


def _drive(exe, d, mode, **env_extra):
    env = dict(os.environ, CMB200_PERSIST="1", CMB200_CHECKPOINT_SEC="1", CMB200_WB_SLOTS="64",
               TSAN_OPTIONS="halt_on_error=0 report_signal_unsafe=0")
    env.update(env_extra)
    for k in ("CMB200_DEVICES", "CMB200_DEVICE", "CMB200_HOST_TIER_MB", "CMB200_TIER_PROMOTE"):
        env.pop(k, None)
    for k in ("CMB200_CHECKPOINT_DELTAS", "CMB200_LOAD"):
        if k not in env_extra:
            env.pop(k, None)
    os.makedirs(d, exist_ok=True)
    base = d / "cachemap_b200.snap"
    if not base.exists():
        base.write_bytes((7).to_bytes(8, "little") + b"\0" * 4088)
    out = subprocess.run([exe, str(d), mode], capture_output=True, text=True, timeout=120, env=env)
    fields = {}
    for name in ("served", "loading", "waited", "calls"):
        m = re.search(rf"^{name}: ?(.*)$", out.stdout, re.M)
        assert out.returncode == 0 and m, out.stdout + out.stderr
        fields[name] = m.group(1).split()
    return fields, out


def test_the_map_serves_while_the_load_is_held(exe, tmp_path):
    f, out = _drive(exe, tmp_path / "c", "free", CMB200_LOAD="background")
    assert f["served"] == ["1"], out.stdout
    assert f["loading"] == ["1", "0", "100"], out.stdout
    assert f["calls"][:2] == ["load_open", "load_step"], out.stdout


def test_ticks_are_skipped_during_the_load_and_resume_after_it(exe, tmp_path):
    f, out = _drive(exe, tmp_path / "c", "ticks", CMB200_LOAD="background")
    calls = f["calls"]
    held = calls[:calls.index("release")]
    assert held == ["load_open", "load_step"], out.stdout
    after = calls[calls.index("release") + 1:calls.index("end")]
    assert after[0] == "load_close" and "save_set" in after, out.stdout


@pytest.mark.parametrize("deltas", [None, "3"])
def test_checkpoint_waits_for_the_load_then_writes_a_base(exe, tmp_path, deltas):
    extra = {"CMB200_CHECKPOINT_DELTAS": deltas} if deltas else {}
    f, out = _drive(exe, tmp_path / "c", "checkpoint", CMB200_LOAD="background", CMB200_CHECKPOINT_SEC="0", **extra)
    assert f["waited"] == ["1"], out.stdout
    written = "base" if deltas else "save_set"
    assert f["calls"][:6] == ["load_open", "load_step", "release", "load_close", written, "end"], out.stdout


@pytest.mark.parametrize("deltas", [None, "3"])
def test_free_finishes_the_load_then_writes_a_base(exe, tmp_path, deltas):
    extra = {"CMB200_CHECKPOINT_DELTAS": deltas} if deltas else {}
    f, out = _drive(exe, tmp_path / "c", "free", CMB200_LOAD="background", CMB200_CHECKPOINT_SEC="0", **extra)
    assert f["waited"] == ["1"], out.stdout
    written = "base" if deltas else "save_set"
    assert f["calls"] == ["load_open", "load_step", "release", "load_close", written, "end"], out.stdout


@pytest.mark.parametrize("env", [{}, {"CMB200_LOAD": "wait"}, {"CMB200_LOAD": "later"}, {"MOCK_LOAD_OPEN_FAIL": "1"}],
                         ids=["unset", "wait", "unknown", "open-fails"])
def test_otherwise_the_first_call_loads_before_serving(exe, tmp_path, env):
    env = dict(env)
    if env.get("MOCK_LOAD_OPEN_FAIL"):
        env["CMB200_LOAD"] = "background"
    f, out = _drive(exe, tmp_path / "c", "checkpoint", CMB200_CHECKPOINT_SEC="0", CMB200_CHECKPOINT_DELTAS="3", **env)
    calls = f["calls"]
    assert calls[0] == "load_chain" and "load_open" not in calls, out.stdout
    assert f["loading"][0] == "0" and f["waited"] == ["0"], out.stdout
    if env.get("CMB200_LOAD") == "later":
        assert "CMB200_LOAD=later" in out.stderr, out.stderr
    if env.get("MOCK_LOAD_OPEN_FAIL"):
        assert "no background load" in out.stderr, out.stderr


@pytest.mark.parametrize("deltas", [None, "3"])
def test_without_the_load_calls_the_load_is_todays(exe_without, tmp_path, deltas):
    extra = {"CMB200_CHECKPOINT_DELTAS": deltas} if deltas else {}
    f, out = _drive(exe_without, tmp_path / "c", "checkpoint", CMB200_LOAD="background", CMB200_CHECKPOINT_SEC="0",
                    **extra)
    calls = f["calls"]
    assert calls[0] == ("load_chain" if deltas else "load_set"), out.stdout
    assert calls[1] == ("base" if deltas else "save_set"), out.stdout
    assert f["loading"][0] == "0", out.stdout


def test_background_load_has_no_data_race(tmp_path):
    exe, err = _build(tmp_path, "load_drive_tsan", "mock_load.c", ["-fsanitize=thread"])
    if not exe:
        pytest.skip("gcc cannot link -fsanitize=thread here: " + err[-200:])
    for mode in ("ticks", "checkpoint", "free"):
        f, out = _drive(exe, tmp_path / mode, mode, CMB200_LOAD="background", CMB200_CHECKPOINT_DELTAS="2")
        assert "ThreadSanitizer" not in out.stderr, out.stderr[-3000:]
        assert f["calls"][:2] == ["load_open", "load_step"], out.stdout
