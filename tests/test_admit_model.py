"""tests/admit_model.py: the sketch (saturation, halving, index function against the C header) and the
admission rule, and what admission does to the hot/cold and scan workloads.  CPU only."""
import os
import subprocess

import numpy as np
import pytest

import admit_model as A
from oracle import evict_model

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KEYS = [0, 1, 0xFFFFFFFFFFFFFFFF, 0xCBF29CE484222325, A.fnv_addr(1000, 5), A.fnv_addr(2000, 1 << 40), 0x8000000000000000]


def test_index_function_is_the_headers(tmp_path):
    src = tmp_path / "t.c"
    keys = ",".join(f"0x{k:016x}ull" for k in KEYS)
    src.write_text('#include <stdio.h>\n#include "cachemap_b200.h"\n'
                   f'static const uint64_t K[] = {{{keys}}};\n'
                   'extern inline uint32_t cmb200_freq_index(uint64_t key, int row, int log2_width);\n'
                   'int main(void){for(unsigned i=0;i<sizeof K/8;i++)for(int r=0;r<4;r++)for(int w=4;w<=32;w+=7)'
                   'printf("%u\\n",cmb200_freq_index(K[i],r,w));return 0;}\n')
    exe = tmp_path / "t"
    r = subprocess.run(["gcc", "-std=c99", "-O1", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    got = [int(x) for x in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    want = [A.freq_index(k, r, w) for k in KEYS for r in range(4) for w in range(4, 33, 7)]
    assert got == want
    assert all(0 <= x < (1 << w) for x, (_k, _r, w) in
               zip(want, [(k, r, w) for k in KEYS for r in range(4) for w in range(4, 33, 7)]))


def test_fnv_key_is_the_stores():
    # FNV-1a-64 over u, l as 16 little-endian bytes (filemap.c:18-24)
    import struct
    h = 14695981039346656037
    for b in struct.pack("<QQ", 7, 9):
        h = ((h ^ b) * 0x100000001B3) & A.M64
    assert A.fnv_addr(7, 9) == h


def test_width_and_period_follow_the_capacity():
    s = A.Sketch(1000)
    assert (s.width, s.log2w, s.period) == (1024, 10, 10000)
    assert A.Sketch(1).width == 16 and A.Sketch(1).period == 10
    s0 = A.Sketch(0)                  # capacity 0: table_slots / 4 (default table 4 x 1024 slots)
    assert s0.width == 1024 and s0.period == 10 * 1024
    assert A.Sketch(0, table_slots=1 << 20).width == 1 << 18


def test_counters_saturate_at_15():
    s = A.Sketch(1 << 10)
    k = A.fnv_addr(1, 2)
    s.launch([k] * 40)
    assert s.estimate(k) == 15
    for r in range(4):
        assert s.c[r][s.index(k, r)] == 15


def test_halving_happens_at_exactly_the_period():
    s = A.Sketch(16)                 # period 160
    keys = [A.fnv_addr(3, i) for i in range(8)]
    for t in range(159):
        s.launch([keys[t % 8]])
    assert s.halvings == 0 and s.since == 159
    before = [bytearray(r) for r in s.c]
    s.launch([keys[159 % 8]])
    assert s.halvings == 1 and s.since == 0 and s.increments == 160
    k = keys[159 % 8]
    for r in range(4):
        j = s.index(k, r)
        want = bytearray(before[r])
        want[j] = min(15, want[j] + 1)
        assert s.c[r] == bytearray(x >> 1 for x in want)


def test_a_launch_that_crosses_the_period_halves_after_all_its_increments():
    s = A.Sketch(16)
    s.launch([A.fnv_addr(4, i) for i in range(150)])
    s.launch([A.fnv_addr(5, 0)] * 20)   # 170 >= 160: halved once, count from 0
    assert s.halvings == 1 and s.since == 0 and s.increments == 170
    assert s.estimate(A.fnv_addr(5, 0)) >= 7


def test_words_pack_nibbles_in_row_order():
    s = A.Sketch(32)                 # 2 words per row
    s.c[0][0] = 1
    s.c[0][15] = 15
    s.c[3][17] = 5
    w = s.words()
    assert w.dtype == np.uint64 and len(w) == 8
    assert int(w[0]) == 1 | (15 << 60) and int(w[7]) == 5 << 4
    assert not any(int(x) for x in w[1:7])


def test_rule_is_strictly_greater():
    assert A.admits(3, 2) and not A.admits(2, 2) and not A.admits(0, 0) and not A.admits(1, 5)


@pytest.mark.parametrize("table", [False, True])
def test_the_page_asked_for_more_often_wins_and_ties_reject(table):
    s = (A.AdmitTableStore if table else A.AdmitStore)(4, False, True, seed=3)
    for p in range(4):
        s.put((1, p))
    for p in range(4):
        s.get((1, p))               # every record asked for once
    s.put((2, 0))                   # never asked for: loses to any victim
    assert (2, 0) not in s.ts and len(s) == 4 and s.rejected == 1
    s.get((2, 1))                   # asked for once: ties every victim, rejected
    s.put((2, 1))
    assert (2, 1) not in s.ts and s.rejected == 2
    s.get((2, 1))                   # twice: beats a victim asked for once
    s.put((2, 1))
    assert (2, 1) in s.ts and len(s) == 4 and s.admitted == 1 and len(s.evicted) == 1


@pytest.mark.parametrize("table", [False, True])
def test_a_rejected_page_removes_its_older_version(table):
    s = (A.AdmitTableStore if table else A.AdmitStore)(4, False, True, seed=5)
    for p in range(4):
        s.put((1, p))
        s.get((1, p))
        s.get((1, p))
    s.put((1, 2))                   # a new version at capacity, asked for 2 times like every victim: rejected
    assert (1, 2) not in s.ts and len(s) == 3


@pytest.mark.parametrize("table", [False, True])
@pytest.mark.parametrize("touch", [False, True])
def test_without_admission_hot_cold_is_evict_models(table, touch):
    kw = dict(capacity=512, hot=128, steps=6000, warmup=2000, seed=2, table=table)
    assert A.hot_cold(touch, False, **kw) == evict_model.hot_cold(touch, **kw)


@pytest.mark.parametrize("table", [False, True])
@pytest.mark.parametrize("touch", [False, True])
def test_admission_keeps_the_hot_set_through_a_scan(table, touch):
    kw = dict(capacity=1024, hot=512, steps=12000, warmup=6000, seed=1, table=table)
    off = A.scan(touch, False, **kw)
    on = A.scan(touch, True, **kw)
    assert on > off + 0.15, (off, on)
    assert on > 0.85, on
