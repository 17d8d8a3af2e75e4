"""The drop-in's CMB200_CHECKPOINT_DELTAS policy without a GPU: edge_fuse_b200/csrc/cachemap_api.c over the
CPU stand-in of tests/c/mock_chain.c, which logs every snapshot call and writes small files, driven by
tests/c/chain_drive.c — puts every 20 ms while the checkpoint thread ticks every second, then
cachemap_free.  Test infrastructure only: nothing of the product links the stand-in."""
import os
import re
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = [os.path.join(ROOT, "edge_fuse_b200", "csrc", "cachemap_api.c"),
       os.path.join(ROOT, "tests", "c", "mock_chain.c"),
       os.path.join(ROOT, "tests", "c", "chain_drive.c")]


def _build(tmp_path, name, extra):
    exe = str(tmp_path / name)
    r = subprocess.run(["gcc", "-std=gnu11", "-O1", "-g", "-pthread", *extra, *SRC, "-o", exe], capture_output=True, text=True)
    return exe if r.returncode == 0 else None, r.stderr


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    path, err = _build(tmp_path_factory.mktemp("chain"), "chain_drive", [])
    assert path, err
    return path


def _drive(exe, d, seconds, **env_extra):
    env = dict(os.environ, CMB200_PERSIST="1", CMB200_CHECKPOINT_SEC="1", CMB200_WB_SLOTS="64",
               TSAN_OPTIONS="halt_on_error=0 report_signal_unsafe=0", **env_extra)
    for k in ("CMB200_DEVICES", "CMB200_DEVICE", "CMB200_HOST_TIER_MB", "CMB200_TIER_PROMOTE"):
        env.pop(k, None)
    if "CMB200_CHECKPOINT_DELTAS" not in env_extra:
        env.pop("CMB200_CHECKPOINT_DELTAS", None)
    os.makedirs(d, exist_ok=True)
    out = subprocess.run([exe, str(d), str(seconds)], capture_output=True, text=True, timeout=120, env=env)
    calls = re.search(r"^calls: (.*)$", out.stdout, re.M)
    files = re.search(r"^files:(.*)$", out.stdout, re.M)
    assert out.returncode == 0 and calls and files, out.stdout + out.stderr
    return calls.group(1).split(), files.group(1).split(), out


def test_ticks_write_deltas_up_to_the_limit_then_a_base(exe, tmp_path):
    calls, files, out = _drive(exe, tmp_path / "c", 6.5, CMB200_CHECKPOINT_DELTAS="3")
    assert calls[:5] == ["base", "d1", "d2", "d3", "base"], out.stdout
    # cachemap_free writes a base, and the deltas of the chain it ends are removed
    assert calls[-1] == "base" and files == ["cachemap_b200.snap"], out.stdout


def test_deltas_as_large_as_the_base_force_a_base(exe, tmp_path):
    calls, _files, out = _drive(exe, tmp_path / "c", 4.5, CMB200_CHECKPOINT_DELTAS="10",
                                MOCK_BASE_BYTES="4096", MOCK_DELTA_BYTES="2049")
    assert calls[:4] == ["base", "d1", "d2", "base"], out.stdout


def test_without_the_option_the_calls_are_a_full_save_each_time(exe, tmp_path):
    calls, files, out = _drive(exe, tmp_path / "c", 2.5)
    assert calls and set(calls) == {"save_set"} and files == ["cachemap_b200.snap"], out.stdout


def test_a_chain_in_the_directory_is_loaded_and_continued_or_folded(exe, tmp_path):
    d = tmp_path / "c"
    calls, _files, out = _drive(exe, d, 2.5, CMB200_CHECKPOINT_DELTAS="5")
    assert calls[:2] == ["base", "d1"], out.stdout
    for k in (1, 2):                                     # the deltas a crash left behind
        (d / f"cachemap_b200.snap.d{k}").write_bytes(b"\0" * 64)
    # a complete load: the next tick continues the chain
    calls, _files, out = _drive(exe, d, 1.5, CMB200_CHECKPOINT_DELTAS="5", MOCK_LOAD_WHOLE="1")
    assert calls[:2] == ["load_chain", "d3"], out.stdout
    (d / "cachemap_b200.snap.d1").write_bytes(b"\0" * 64)
    # a load that left no chain state: the next tick writes a base
    calls, _files, out = _drive(exe, d, 1.5, CMB200_CHECKPOINT_DELTAS="5")
    assert calls[:3] == ["load_chain", "refused", "base"], out.stdout
    (d / "cachemap_b200.snap.d1").write_bytes(b"\0" * 64)
    # the option off: the chain is still loaded, then folded into a full save that removes its deltas
    calls, files, out = _drive(exe, d, 1.5)
    assert calls[0] == "load_chain" and set(calls[1:]) == {"save_set"}, out.stdout
    assert files == ["cachemap_b200.snap"], out.stdout


def test_checkpoint_policy_has_no_data_race(tmp_path):
    exe, err = _build(tmp_path, "chain_drive_tsan", ["-fsanitize=thread"])
    if not exe:
        pytest.skip("gcc cannot link -fsanitize=thread here: " + err[-200:])
    calls, files, out = _drive(exe, tmp_path / "c", 4.5, CMB200_CHECKPOINT_DELTAS="2")
    assert "ThreadSanitizer" not in out.stderr, out.stderr[-3000:]
    assert calls[:4] == ["base", "d1", "d2", "base"], out.stdout
