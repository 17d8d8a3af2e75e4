"""cachemap_pwrite / cachemap_pread without a GPU: edge_fuse_b200/csrc/cachemap_api.c over the CPU
stand-in of tests/c/mock_patch.c, which applies cmb200_patch_batch under its lock and logs every patch,
driven by tests/c/patch_drive.c.  Linked against plain tests/c/mock_engine.c instead, the drop-in has no
cmb200_patch_batch and must drop the pages it cannot patch.  Test infrastructure only: nothing of the
product links the stand-ins."""
import os
import re
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
API = os.path.join(ROOT, "edge_fuse_b200", "csrc", "cachemap_api.c")
DRIVE = os.path.join(ROOT, "tests", "c", "patch_drive.c")
PAGES = 16


def _build(tmp_path, name, mock, extra=()):
    exe = str(tmp_path / name)
    r = subprocess.run(["gcc", "-std=gnu11", "-O1", "-g", "-Wall", "-pthread", *extra, API,
                        os.path.join(ROOT, "tests", "c", mock), DRIVE, "-o", exe], capture_output=True, text=True)
    return exe if r.returncode == 0 else None, r.stderr


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    path, err = _build(tmp_path_factory.mktemp("patch"), "patch_drive", "mock_patch.c")
    assert path, err
    return path


def _drive(exe, d, *args, **env_extra):
    env = dict(os.environ, CMB200_PERSIST="1", CMB200_WB_SLOTS="64",
               TSAN_OPTIONS="halt_on_error=0 report_signal_unsafe=0")
    env.update(env_extra)
    for k in ("CMB200_DEVICES", "CMB200_DEVICE", "CMB200_HOST_TIER_MB", "CMB200_TIER_PROMOTE",
              "CMB200_CHECKPOINT_SEC", "CMB200_CHECKPOINT_DELTAS"):
        if k not in env_extra:
            env.pop(k, None)
    os.makedirs(d, exist_ok=True)
    out = subprocess.run([exe, args[0], str(d), *map(str, args[1:])], capture_output=True, text=True,
                         timeout=300, env=env)
    assert out.returncode == 0 and "\nlog:\n" in out.stdout, out.stdout + out.stderr
    head, log = out.stdout.split("\nlog:\n", 1)
    patches = [tuple(int(x) for x in ln.split()[1:]) for ln in log.splitlines() if ln.startswith("patch ")]
    return head, patches, log, out


def _split(off, size, pshift):
    """(pages put whole, [(page, page_off, len)] patched) of a pwrite of [off, off + size)."""
    P = 1 << pshift
    if size == 0:
        return [], []
    end = off + size
    p0, p1 = off >> pshift, (end - 1) >> pshift
    skew, tail = off % P, end % P
    if not skew and not tail:
        return list(range(p0, p1 + 1)), []
    puts = list(range(p0 + 1 if skew else p0, p1 if tail else p1 + 1))
    patches = []
    if skew:
        patches.append((p0, skew, size if p0 == p1 else P - skew))
    if tail and (p1 != p0 or not skew):
        patches.append((p1, 0, tail))
    return puts, patches


def _cases(p):
    P = 1 << p
    return [
        (0, 1),                  # byte 0
        (P - 1, 1),              # the last byte of a page
        (5, 100),                # inside one page
        (P - 1, 2),              # two bytes across a page boundary
        (P + 1, P),              # the ends of two neighbouring pages
        (100, 5 * P),            # a partial page, four whole ones, a partial page
        (3 * P, 2 * P),          # aligned: two puts and nothing else
        (2 * P, P + 7),          # a whole page, then the head of the next
        (15 * P + 9, 3 * P),     # past the cached pages: the last edge is not cached and stays so
        (7 * P + 3, 0),          # empty
    ]


@pytest.mark.parametrize("pshift", [12, 13, 16])
def test_a_range_splits_into_puts_and_edge_patches(exe, tmp_path, pshift):
    cases = _cases(pshift)
    flat = [str(x) for c in cases for x in c]
    head, patches, _log, out = _drive(exe, tmp_path / "c", "split", pshift, *flat)
    rows = re.findall(r"^case (\d+) (\d+) (\d+)$", head, re.M)
    assert len(rows) == len(cases), out.stdout
    want_patches, cached_pages, want_preads = [], set(range(PAGES)), 0
    for (off, size), (stored, cached, wrong) in zip(cases, rows):
        puts, edge = _split(off, size, pshift)
        assert (int(cached), int(wrong)) == (PAGES, 0), (off, size)
        assert int(stored) == len(puts) + sum(p < PAGES for p, _, _ in edge), (off, size)
        want_patches += [(0, 5, p, o, n, 1 if p < PAGES else 0) for p, o, n in edge]
        cached_pages |= set(puts)
        overlapped = range(off >> pshift, ((off + size - 1) >> pshift) + 1) if size else []
        want_preads += all(p in cached_pages for p in overlapped)
    assert patches == want_patches, out.stdout
    # pread of each range succeeds when every page it overlaps is cached, with the bytes just written
    preads = re.findall(r"^pread (\d)$", head, re.M)
    assert preads == ["1"] * want_preads, out.stdout


def test_a_page_in_the_ring_is_patched_there_and_a_later_put_kept(exe, tmp_path):
    head, patches, _log, out = _drive(exe, tmp_path / "c", "ring")
    assert "held 1" in head, out.stdout               # served from the ring, both patches applied
    assert "landed 16 0" in head and "later 16 0" in head, out.stdout
    assert patches == [], out.stdout                  # the engine was never asked


def _owner(u, l, g):
    h = 0xcbf29ce484222325
    for b in u.to_bytes(8, "little") + l.to_bytes(8, "little"):
        h = ((h ^ b) * 0x100000001b3) & (2**64 - 1)
    return ((h >> 32) * g) >> 32


def test_patches_reach_the_engine_that_owns_the_key(exe, tmp_path):
    head, patches, _log, out = _drive(exe, tmp_path / "c", "multi", CMB200_DEVICES="0,0,0")
    assert "engines 3 cached 16 wrong 0" in head, out.stdout
    assert len(patches) == 2 * (PAGES - 1), out.stdout
    assert all(st == 1 for *_, st in patches), out.stdout
    # the stand-in numbers engines in the order of their first patch: one engine per owner, and back
    engine_of = {}
    for eng, u, l, *_ in patches:
        assert engine_of.setdefault(_owner(u, l, 3), eng) == eng, out.stdout
    assert len(set(engine_of.values())) == len(engine_of) > 1, out.stdout


def test_a_checkpoint_tick_writes_a_patch_only_change(exe, tmp_path):
    head, patches, _log, out = _drive(exe, tmp_path / "c", "ckpt", CMB200_CHECKPOINT_SEC="1")
    m = re.search(r"saves (\d+) (\d+) (\d+)", head)
    assert m, out.stdout
    after_puts, idle, after_patch = map(int, m.groups())
    assert after_puts >= 1 and idle == after_puts, out.stdout
    assert after_patch == idle + 1, out.stdout
    assert [p[3:] for p in patches] == [(11, 3, 1)], out.stdout


def test_without_the_engine_call_partial_pages_are_dropped(tmp_path):
    exe, err = _build(tmp_path, "patch_drive_plain", "mock_engine.c")
    assert exe, err
    head, _patches, _log, out = _drive(exe, tmp_path / "c", "fallback")
    # pages 2 and 4 are written in part: dropped, never served stale; page 3 is put whole
    assert "fallback 0 1 0 cached 14 wrong 0" in head, out.stdout


@pytest.mark.parametrize("wb_slots", ["64", "0"])
def test_a_dropped_put_leaves_no_old_page(exe, tmp_path, wb_slots):
    """A put the store drops for lack of arena room (the engine keeps the key's old record) removes the
    key: the old page would be stale.  In one flush batch only a key's newest page decides: a drop
    followed by a stored put of the key keeps it."""
    head, _patches, _log, out = _drive(exe, tmp_path / "c", "dropped", CMB200_WB_SLOTS=wb_slots)
    assert "dropped 14 0" in head, out.stdout             # pages 2 and 3 miss, no page is stale
    if wb_slots != "0":
        assert "batch 1 13 0" in head, out.stdout         # page 4 holds its last put, page 5 misses


@pytest.mark.parametrize("threads", [4, 16])
def test_concurrent_writers_of_one_page_all_land(exe, tmp_path, threads):
    head, _patches, _log, out = _drive(exe, tmp_path / "c", "stress", threads, 1.0)
    m = re.search(r"stress errors (\d+) ops (\d+) lost (\d+) page (\d)", head)
    assert m, out.stdout
    errors, ops, lost, page = map(int, m.groups())
    assert (errors, lost, page) == (0, 0, 1) and ops > 100, out.stdout


def test_concurrent_writers_have_no_data_race(tmp_path):
    exe, err = _build(tmp_path, "patch_drive_tsan", "mock_patch.c", ["-fsanitize=thread"])
    if not exe:
        pytest.skip("gcc cannot link -fsanitize=thread here: " + err[-200:])
    head, _patches, _log, out = _drive(exe, tmp_path / "c", "stress", 16, 1.5)
    assert "ThreadSanitizer" not in out.stderr, out.stderr[-3000:]
    assert re.search(r"stress errors 0 ops \d+ lost 0 page 1", head), out.stdout
