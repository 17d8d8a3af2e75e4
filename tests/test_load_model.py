"""The as-if model of tests/load_model.py on its known cases, without a GPU."""
import load_model as LM
import store_machine as SM

HIT, MISS, BAD_ENTRY = LM.HIT, LM.MISS, LM.BAD_ENTRY


def _key(a):
    # two addresses share a key when their l is equal modulo 1000: a stand-in for an FNV collision
    return (a[0], a[1] % 1000)


def _model():
    return LM.AsIfModel(_key, {(1, 0): b"a0", (1, 1): b"a1", (1, 2): b"a2", (2, 5): b"b5"})


def _ok(m, a, page):
    return m.check([a], [HIT], [page]) is None


def test_file_pages_hit_and_misses_are_always_allowed():
    m = _model()
    assert _ok(m, (1, 0), b"a0")
    assert not _ok(m, (1, 0), b"zz")
    assert not _ok(m, (1, 7), b"a0")
    assert m.check([(1, 0), (3, 3)], [MISS, BAD_ENTRY], [b"", b""]) is None
    assert m.check([(1, 0)], [SM.DROPPED], [b""]) is not None


def test_a_stored_put_replaces_its_key_and_a_dropped_one_keeps_the_older():
    m = _model()
    m.put([(1, 0), (1, 1001), (1, 2)], [b"n0", b"n1", b"n2"], None, [10, 10, -1])
    assert _ok(m, (1, 0), b"n0") and not _ok(m, (1, 0), b"a0")
    assert _ok(m, (1, 1001), b"n1") and not _ok(m, (1, 1), b"a1")       # the key's other address is gone
    assert _ok(m, (1, 2), b"a2")                                         # dropped: the older page stays
    m.put([(2, 5)], [b"x"], [0], [-1])                                  # an invalid row stores nothing
    assert _ok(m, (2, 5), b"b5")


def test_unset_deletes_by_key_and_invalidate_by_interval():
    m = _model()
    m.unset([(1, 1000)])
    assert not _ok(m, (1, 0), b"a0")
    m.invalidate(1, 1, 1)
    assert not _ok(m, (1, 1), b"a1") and _ok(m, (1, 2), b"a2")


def test_rename_moves_and_keeps_the_older_destination_only_with_drops():
    m = _model()
    m.rename(1, 2, 0, 5, dropped=0)
    assert not _ok(m, (1, 0), b"a0") and _ok(m, (2, 0), b"a0")
    assert _ok(m, (2, 5), b"b5")                                         # no source at l = 5: kept
    m = LM.AsIfModel(_key, {(1, 5): b"a5", (2, 5): b"b5"})
    m.rename(1, 2, 5, 5, dropped=0)
    assert _ok(m, (2, 5), b"a5") and not _ok(m, (2, 5), b"b5")
    m = LM.AsIfModel(_key, {(1, 5): b"a5", (2, 5): b"b5"})
    m.rename(1, 2, 5, 5, dropped=1)
    assert _ok(m, (2, 5), b"a5") and _ok(m, (2, 5), b"b5")


def test_patch_hits_apply_their_spans_and_other_answers_drop_the_address():
    m = LM.AsIfModel(_key, {(1, 0): b"\0" * 32, (1, 1): b"\1" * 32})
    spans = [(0, 4, "0", 1), (30, 2, "R", 2)]
    m.patch([(1, 0), (1, 0), (1, 1)], spans + [(0, 1, "0", 3)], [HIT, HIT, MISS])
    want = bytearray(b"\0" * 32)
    want[30:32] = SM.span_bytes(spans[1])
    assert _ok(m, (1, 0), bytes(want)) and not _ok(m, (1, 0), b"\0" * 32)
    assert not _ok(m, (1, 1), b"\1" * 32)


def test_generated_logs_step_before_every_operation():
    cfg = SM.CONFIGS["A"]
    ops = LM.gen_load_ops(cfg, 11)
    assert ops == LM.gen_load_ops(cfg, 11)
    assert all(op[0] != "load" for op in ops)
    kinds = [op[0] for op in ops]
    assert kinds[0] == "step" and "rename" in kinds
    for i, op in enumerate(ops):
        if op[0] not in ("step", "rename"):
            assert ops[i - 1][0] in ("step", "rename")
    main = {(u, l) for u in cfg.us for l in range(cfg.nl)}
    first = next(op for op in ops if op[0] in ("put", "put_async"))
    assert not set(first[1]) >= main                                    # the fill is the file's, not an op
