"""The sequential model of a replicated index (tests/replica_model.py) on hand-worked cases and seeded
logs, without a GPU."""
import random

import key_edges
import replica_model as RM

HIT, MISS, BAD_ENTRY, REMOTE = RM.HIT, RM.MISS, RM.BAD_ENTRY, RM.REMOTE
A, B, C = (1, 0), (1, 1), (1, 2)


def test_fnv_key_matches_the_fixture():
    """The key-sharing pairs of tests/golden/key_edges.json share a key; the sentinel addresses hash to 0
    and ~0."""
    fx = key_edges.load()
    for name, group in fx["groups"].items():
        keys = {RM.fnv_key(*a) for a in group}
        if name in key_edges.SENTINEL_KEYS:
            assert keys == {key_edges.SENTINEL_KEYS[name]}
        else:
            assert len(keys) == 1
    assert len({RM.fnv_key(*a) for a in fx["ordinary"]}) == len(fx["ordinary"])


def test_the_highest_position_wins_whatever_the_arrival_order():
    m = RM.ReplicaModel(1)
    m.put([(A, 10, True, b"a"), (B, 13, True, b"b")])
    m.import_rows([(A, 12, 0, True), (B, 11, 2, True), (C, 9, 2, True)])
    assert m.lookup(A) == (REMOTE, 0, None)                 # the row is newer than the put
    assert m.lookup(B) == (HIT, -1, b"b")                   # the put is newer than the row
    assert m.lookup(C) == (REMOTE, 2, None)
    m.import_rows([(A, 11, 2, True), (A, 14, 2, True), (A, 5, 0, True)])   # late rows, out of order
    assert m.lookup(A) == (REMOTE, 2, None)
    assert (m.entries(), m.remote_entries()) == (1, 2)


def test_rows_of_this_rank_and_rows_that_stored_nothing_are_skipped():
    m = RM.ReplicaModel(1)
    m.import_rows([(A, 12, 1, True), (B, 12, 0, False)])
    assert m.lookup(A)[0] == MISS and m.lookup(B)[0] == MISS
    m.put([(A, 3, True, b"a")])
    m.import_rows([(A, 30, 0, False)])                      # stored nothing: the local record stays
    assert m.lookup(A) == (HIT, -1, b"a")


def test_a_put_below_the_floor_changes_nothing():
    m = RM.ReplicaModel(1)
    m.import_rows([(A, 20, 2, True)])
    m.put([(A, 19, True, b"late")])
    assert m.lookup(A) == (REMOTE, 2, None) and m.entries() == 0


def test_a_dropped_put_raises_the_floor_and_keeps_the_older_winner():
    m = RM.ReplicaModel(1)
    m.put([(A, 4, True, b"old")])
    m.put([(A, 7, False, b"new")])                          # the arena dropped it
    assert m.lookup(A) == (HIT, -1, b"old")
    m.import_rows([(A, 6, 0, True)])                        # below the dropped put's position
    assert m.lookup(A) == (HIT, -1, b"old")
    m.import_rows([(A, 8, 0, True)])
    assert m.lookup(A) == (REMOTE, 0, None) and m.entries() == 0


def test_in_batch_duplicates_and_invalid_addresses():
    m = RM.ReplicaModel(0)
    m.put([(A, 1, False, b"x"), (None, 4, False, b"bad"), (A, 7, True, b"y")])
    assert m.lookup(A) == (HIT, -1, b"y") and m.entries() == 1


def test_key_sharing_addresses():
    fx = key_edges.load()
    p, q = fx["groups"]["pair0"]
    m = RM.ReplicaModel(1)
    m.put([(p, 5, True, b"p")])
    assert m.lookup(q) == (BAD_ENTRY, -1, None)             # local winner of another address
    m.import_rows([(q, 8, 2, True)])
    assert m.lookup(q) == (REMOTE, 2, None)
    assert m.lookup(p) == (MISS, -1, None)                  # remote winner of another address
    assert (m.entries(), m.remote_entries()) == (0, 1)
    m.unset([p])                                            # by key: the remote winner stays
    assert m.lookup(q) == (REMOTE, 2, None)


def test_unset_removes_a_local_winner_and_leaves_a_remote_one():
    m = RM.ReplicaModel(1)
    m.put([(A, 1, True, b"a"), (B, 4, True, b"b")])
    m.import_rows([(B, 6, 0, True)])
    m.unset([A, B, C])
    assert m.lookup(A)[0] == MISS and m.lookup(B) == (REMOTE, 0, None)
    assert (m.entries(), m.remote_entries()) == (0, 1)
    m.put([(A, 9, True, b"a2")])                            # a removed key starts again
    assert m.lookup(A) == (HIT, -1, b"a2")


def test_a_loaded_rank_holds_the_local_winners_only():
    m = RM.ReplicaModel(1)
    m.put([(A, 1, True, b"a"), (B, 4, True, b"b")])
    m.import_rows([(B, 6, 0, True), (C, 2, 2, True)])
    f = RM.ReplicaModel.loaded(1, m.local_records())
    assert f.lookup(A) == (HIT, -1, b"a") and f.lookup(B)[0] == MISS and f.lookup(C)[0] == MISS
    assert (f.entries(), f.remote_entries()) == (1, 0)


def _brute(rank, log):
    """The winner of each key straight from its definition: the highest position among this rank's own
    stored puts and the other ranks' rows that stored something."""
    best = {}
    for kind, addr, pos, owner, stored in log:
        if addr is None or not stored or (kind == "row" and owner == rank):
            continue
        key = RM.fnv_key(*addr)
        if key not in best or pos > best[key][0]:
            best[key] = (pos, addr, rank if kind == "put" else owner)
    return best


def test_seeded_logs_against_the_definition():
    """Puts and imports in random batches, positions in any order (no unsets): the model's winner of every
    key is the definition's, except where a put the arena dropped holds the floor above it."""
    fx = key_edges.load()
    pool = [(7, i) for i in range(12)] + list(fx["groups"]["pair0"]) + list(fx["groups"]["key0"])
    for seed in range(200):
        rng = random.Random(seed)
        rank = rng.randrange(3)
        m = RM.ReplicaModel(rank)
        log, positions = [], rng.sample(range(10_000), 120)
        dropped_top = {}
        while positions:
            k = min(len(positions), rng.randrange(1, 9))
            batch, positions = positions[:k], positions[k:]
            if rng.random() < 0.5:
                chunks = [(rng.choice(pool) if rng.random() > 0.1 else None, p, rng.random() > 0.15, b"")
                          for p in batch]
                m.put(chunks)
                for a, p, s, _ in chunks:
                    log.append(("put", a, p, rank, s))
                    if a is not None and not s:
                        key = RM.fnv_key(*a)
                        dropped_top[key] = max(dropped_top.get(key, -1), p)
            else:
                rows = [(rng.choice(pool), p, rng.randrange(3), rng.random() > 0.15) for p in batch]
                m.import_rows(rows)
                log.extend(("row", a, p, o, s) for a, p, o, s in rows)
        best = _brute(rank, log)
        for key in set(best) | set(m.winner):
            w = m.winner.get(key)
            if key in dropped_top and dropped_top[key] > best.get(key, (-1,))[0]:
                continue                                    # a dropped put holds the floor above the winner
            assert w is not None and (w.pos, w.addr, w.owner) == best[key], (seed, key, w, best.get(key))
        assert m.entries() + m.remote_entries() == len(m.winner)
