"""The rules of tests/pin_model.py: the range algebra of cachemap_pin's list and the sampler that passes over
pinned records."""
import random

import pin_model as PM

G44 = 1 << 44


def _pages_set(ranges):
    return {(u, l) for u, f, l_ in ranges for l in range(f, l_ + 1)}


def test_pin_and_unpin_agree_with_a_set_of_pages():
    rng = random.Random(1)
    m = PM.Pins(1 << 20, 12)
    want: set = set()
    for _ in range(400):
        u, a = rng.randrange(3), rng.randrange(200)
        n = rng.randrange(1, 20)
        if rng.random() < 0.6:
            new = {(u, l) for l in range(a, a + n)} - want
            assert m.pin(u, 0, a << 12, n << 12) == len(new)
            want |= new
        else:
            gone = {(u, l) for l in range(a, a + n)} & want
            assert m.unpin(u, 0, a << 12, n << 12) == len(gone)
            want -= gone
        assert _pages_set(m.ranges) == want
        assert m.ranges == PM.normalize(m.ranges)
        for x, y in zip(m.ranges, m.ranges[1:]):      # sorted, disjoint and never touching
            assert x[0] < y[0] or x[2] + 1 < y[1]


def test_partial_pages_and_the_end_saturate_as_invalidation_does():
    assert PM.span(12, 0, 4095, 2) == (0, 1)
    assert PM.span(12, 3, 0, PM.TO_END) == (3 * G44, 3 * G44 + G44 - 1)
    assert PM.span(12, 0, G44 << 12, 1) is None
    m = PM.Pins(1 << 20, 12)
    assert m.pin(5, 0, 0, 0) == -1 and m.pin(5, 0, 0, PM.TO_END) == -1
    assert m.unpin(5, 0, 0, PM.TO_END) == 0


def test_the_budget_and_the_range_count_refuse_without_pinning():
    m = PM.Pins(4096, 12, pin_max=3000)
    assert m.max == 2048                                  # clamped at half the capacity
    assert m.pin(5, 0, 0, 2049 << 12) == -1 and m.ranges == []
    assert m.pin(5, 0, 0, 2048 << 12) == 2048
    assert PM.Pins(4096, 12, pin_max=0).pin(5, 0, 0, 4096) == -1
    m = PM.Pins(1 << 20, 12)
    for k in range(PM.PIN_RANGES):
        assert m.pin(5, 0, (2 * k) << 12, 4096) == 1
    assert m.pin(5, 0, (2 * PM.PIN_RANGES) << 12, 4096) == -1
    assert m.pin(5, 0, 1 << 12, 4096) == 1               # fills a gap: one range fewer


def test_a_rename_drops_the_pins_of_to_and_moves_those_of_from_in_that_generation():
    m = PM.Pins(1 << 20, 12)
    m.pin(5, 0, 0, 10 << 12)
    m.pin(5, 1, 0, 1 << 12)
    m.pin(6, 0, 20 << 12, 1 << 12)
    m.rename(5, 6, 0)
    assert m.ranges == [(5, G44, G44), (6, 0, 9)]


def test_a_load_keeps_the_file_order_while_the_budget_allows():
    m = PM.Pins(4096, 12, pin_max=25)
    m.load([(5, 0, 9), (6, 0, 9), (7, 0, 9)])
    assert m.ranges == [(5, 0, 9), (6, 0, 9)]
    m.load([(5, 0, 9), (5, 5, 6), (7, 0, 0)])
    assert m.ranges == [(5, 0, 9)]
    m.load([(5, 3, 1)])
    assert m.ranges == []


def test_the_pinned_sampler_never_evicts_a_pinned_page():
    pinned = [(0, 0, 63)]
    s = PM.PinnedTableStore(256, False, seed=3, pinned=pinned)
    for l in range(64):
        s.put((0, l))
    for l in range(10000):
        s.put((1, l))
    assert all((0, l) in s.at for l in range(64))
    assert len(s) == 256 and not any(PM.has(pinned, v) for v in s.evicted)


def test_with_every_record_pinned_nothing_is_evicted():
    s = PM.PinnedTableStore(4, False, seed=1, pinned=[(0, 0, 100)])
    for l in range(6):
        s.put((0, l))
    assert len(s) == 6 and s.evicted == []
