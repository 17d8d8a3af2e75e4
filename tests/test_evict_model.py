"""oracle/evict_model.py, the eviction policy on a logical clock that the GPU test of CMB200_EVICT
compares the drop-in with: the victim is the reference's pick (cachemap.c:29-41), ties included, and the
two policies differ only in what a hit does."""
import itertools
import random

import pytest

from oracle.evict_model import Store, TableStore, hot_cold, pick


def _reference_pick(a, b, c):
    # cachemap.c:29-41, branch by branch
    if a < b:
        if a > c:
            return 2
        return 0
    if b > c:
        return 2
    return 1


@pytest.mark.parametrize("a,b,c", list(itertools.product(range(3), repeat=3)))
def test_pick_is_the_reference_comparison(a, b, c):
    assert pick(a, b, c) == _reference_pick(a, b, c)


@pytest.mark.parametrize("ts,victim", [
    ((1, 2, 3), 0), ((2, 1, 3), 1), ((3, 2, 1), 2),
    ((1, 1, 2), 1),          # a == b: the second
    ((1, 2, 1), 0),          # a == c < b: the first
    ((2, 1, 1), 1),          # b == c < a: the second
    ((1, 1, 1), 1),          # all equal: the second
    ((2, 2, 1), 2),
])
def test_pick_on_ties(ts, victim):
    assert pick(*ts) == victim


def _scripted(draws):
    it = iter(draws)
    return lambda n: next(it) % n


def test_the_victim_is_the_oldest_of_the_drawn_records():
    s = Store(4, touch=False, draw=_scripted([3, 1, 2]))
    for a in "abcd":
        s.put(a)                        # ts a=1 b=2 c=3 d=4
    s.put("e")                          # draws d, b, c: b is the oldest
    assert s.evicted == ["b"] and sorted(s.ts) == ["a", "c", "d", "e"]


def test_a_hit_refreshes_only_under_touch():
    for touch, victim in ((False, "a"), (True, "b")):
        s = Store(3, touch=touch, draw=_scripted([0, 1, 2]))
        for a in "abc":
            s.put(a)
        assert s.get("a") and not s.get("z")
        s.put("d")                      # draws a, b, c
        assert s.evicted == [victim], touch


def test_a_record_drawn_twice_against_an_older_one():
    s = Store(3, touch=False, draw=_scripted([1, 1, 0]))
    for a in "abc":
        s.put(a)
    s.put("d")                          # draws b, b, a: a is older than b
    assert s.evicted == ["a"]


def test_eviction_comes_before_every_put_at_capacity_even_a_rewrite():
    s = Store(2, touch=False, draw=_scripted([0, 0, 0]))
    s.put("a")
    s.put("b")
    s.put("b")                          # at capacity: the reference evicts first (cachemap.c:22)
    assert s.evicted == ["a"] and len(s) == 1


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_the_policies_agree_when_nothing_is_read_twice(seed):
    rng = random.Random(seed)
    draws = [rng.randrange(1 << 30) for _ in range(30000)]
    runs = []
    for touch in (False, True):
        s = Store(256, touch=touch, draw=_scripted(draws))
        hits = 0
        for t in range(4000):
            a = ("p", t)
            hits += s.get(a)            # every page is read once, before its put: a miss
            s.put(a)
        runs.append((hits, s.evicted, dict(s.ts)))
    assert runs[0] == runs[1] and runs[0][0] == 0 and len(runs[0][1]) == 4000 - 256


def test_the_hot_and_cold_workload():
    """Hot set 1024 pages read round-robin and put on a miss, one cold page put per step, capacity 4096:
    refreshing ts on a hit keeps the hot set cached."""
    put = hot_cold(touch=False, steps=32768, warmup=16384)
    access = hot_cold(touch=True, steps=32768, warmup=16384)
    assert 0.70 < put < 0.75 and 0.92 < access < 0.95, (put, access)


def test_the_table_sampler_draws_the_first_live_slot_at_or_after_a_uniform_one():
    homes = {"a": 2, "b": 2, "c": 6, "d": 0, "e": 2}
    s = TableStore(3, touch=False, draw=_scripted([3, 7, 1, 6, 6, 6]), slots=8, home=homes.__getitem__)
    for a in "abc":
        s.put(a)                        # a at 2, b at 3 (probed past a), c at 6
    assert s.table[2:4] == ["a", "b"] and s.table[6] == "c"
    s.put("d")                          # draws from 3, 7 (wraps), 1: b, a, a; a is older than b
    assert s.evicted == ["a"] and s.table[0] == "d" and s.table[2] is not None and s.table[2] != "a"
    s.put("e")                          # draws c three times; e's chain reuses a's tombstone at 2
    assert s.evicted == ["a", "c"] and s.table[2] == "e" and sorted(s.ts) == ["b", "d", "e"]


def test_the_store_sampler_costs_access_part_of_its_gain():
    """With the store's draws the hot set keeps less under access than with uniform draws; put changes
    little.  These are the values the drop-in is compared with on the GPU."""
    kw = dict(capacity=4096, hot=1024, steps=12288, warmup=8192)
    put = [hot_cold(False, seed=s, table=True, **kw) for s in (1, 2, 3)]
    access = [hot_cold(True, seed=s, table=True, **kw) for s in (1, 2, 3)]
    assert 0.67 < sum(put) / 3 < 0.74 and 0.83 < sum(access) / 3 < 0.90, (put, access)
    assert sum(access) / 3 - sum(put) / 3 > 0.12
