"""The rules of tests/usage_model.py: page arithmetic of partial ends, refusals, the PINNED bit, grouping by
genid, the order and its ties, and the merge of rows spread over engines."""
import numpy as np

import usage_model as UM

G = 1 << UM.PNUM


def test_span_counts_partial_pages_at_both_ends():
    assert UM.span(12, 0, 0, 1) == (0, 0)
    assert UM.span(12, 0, 4095, 2) == (0, 1)
    assert UM.span(12, 0, 4096, 4096) == (1, 1)
    assert UM.span(12, 3, 100, 8192) == (3 * G, 3 * G + 2)
    assert UM.span(16, 1, 65535, 65538) == (G, G + 2)


def test_span_refusals():
    assert UM.span(12, 0, 0, 0) is None
    assert UM.span(12, 0, 0, UM.TO_END) is None
    assert UM.span(12, 0, G << 12, 1) is None                    # first page past 44 bits
    assert UM.span(12, 0, (G - 1) << 12, 8192) is None           # last page past 44 bits
    assert UM.span(12, 0, UM.TO_END, 2) is None                  # end past 2^64
    assert UM.span(12, 0, (G - 1) << 12, 4096) == (G - 1, G - 1)


def test_residency_bits_and_count():
    recs = {(5, 0): (100, False, 10), (5, 2): (200, True, 11), (5, G): (100, False, 12), (6, 1): (100, False, 13)}
    pins = [(5, 1, 3)]
    n, v = UM.residency(recs, pins, 12, 5, 0, 0, 4 * 4096)
    assert n == 2
    assert v.tolist() == [UM.IN_HBM, UM.PINNED, UM.IN_TIER | UM.PINNED, UM.PINNED]
    assert UM.residency(recs, pins, 12, 5, 0, 0, 0) == (-1, None)
    n, v = UM.residency(recs, pins, 12, 5, 1, 0, 1)             # genid 1 is another object
    assert n == 1 and v.tolist() == [UM.IN_HBM]


def test_engine_residency_marks_only_the_interval():
    recs = {(5, 3): (1, False, 0), (5, 9): (1, True, 0), (5, 20): (1, False, 0)}
    assert UM.engine_residency(recs, 5, 3, 9).tolist() == [1, 0, 0, 0, 0, 0, 2]


def test_usage_groups_by_genid_and_orders_with_ties():
    recs = {(5, 0): (100, False, 7), (5, 1): (50, True, 3), (5, G | 4): (150, False, 9),
            (4, 2): (150, False, 1), (9, 0): (40, False, 2)}
    n, rs = UM.usage(recs, [(5, 1, 1)], 10)
    assert n == 4
    # ties on 150 bytes: nhid 4 before nhid 5; then (5, genid 0) has 150 too, and genid 0 < 1 orders it
    assert [(r[0], r[1], r[6]) for r in rs] == [(4, 0, 150), (5, 0, 150), (5, 1, 150), (9, 0, 40)]
    r = rs[1]
    assert r == (5, 0, 0, 2, 1, 1, 150, 0, 1, 3, 7)
    assert rs[2][7:9] == (4, 4)
    assert UM.usage(recs, [(5, 1, 1)], 2) == (4, rs[:2])
    assert UM.usage(recs, [], 0) == (4, [])
    assert UM.usage({}, [], 5) == (0, [])


def test_merge_sums_an_object_spread_over_engines():
    a = {(5, 0): (100, False, 7), (5, 3): (30, True, 1)}
    b = {(5, 1): (50, False, 9), (6, 0): (10, False, 4)}
    merged = UM.order(UM.merge([UM.rows(a, []), UM.rows(b, [])]))
    assert merged == UM.usage({**a, **b}, [], 10)[1]
    assert merged[0] == (5, 0, 0, 3, 1, 0, 180, 0, 3, 1, 9)


def test_as_tuples_reads_the_dtype_fields():
    dt = np.dtype([(f, "<u8") if f not in ("genid", "reserved") else (f, "<u4") for f in UM.FIELDS])
    arr = np.zeros(1, dtype=dt)
    arr[0] = (1, 2, 0, 3, 4, 5, 6, 7, 8, 9, 10)
    assert UM.as_tuples(arr) == [(1, 2, 0, 3, 4, 5, 6, 7, 8, 9, 10)]
