"""The store machine's model and generator without a GPU (tests/store_machine.py): the model agrees
with oracle StoreModel and with the key-edge trace, the generator is deterministic, and the committed
seeds reach every rare event of their configuration."""
import pytest

import key_edges
import store_machine as SM


@pytest.mark.parametrize("name", sorted(SM.CONFIGS))
def test_generator_is_deterministic(name):
    cfg = SM.CONFIGS[name]
    for seed in cfg.seeds:
        a, b = SM.gen_ops(cfg, seed), SM.gen_ops(cfg, seed)
        assert a == b
    assert SM.gen_ops(cfg, cfg.seeds[0]) != SM.gen_ops(cfg, cfg.seeds[1])


@pytest.mark.parametrize("name", sorted(SM.CONFIGS))
def test_model_agrees_with_store_model_on_put_get_unset(name, oracle):
    """The put / get / unset part of a generated log through the machine's model and through a plain
    oracle StoreModel: the same answers, pages, records and counters."""
    cfg = SM.CONFIGS[name]
    m = SM.Model(cfg, oracle)
    ref = oracle.StoreModel(cfg.pshift, cfg.accel)
    for op in SM.gen_ops(cfg, cfg.seeds[0])[:40]:
        k = op[0]
        if k in ("put", "put_async"):
            pages = SM.pages_of(cfg, op[2])
            m.put(op[1], pages, op[3], op[4], set())
            for i in m.put_rows(op[1], op[4]):
                ref.put(*key_edges.cachemap_args(*op[1][i], cfg.pshift), pages[i])
        elif k in ("get", "get_small"):
            got = m.get(op[1], op[2])
            for i, a in enumerate(op[1]):
                if op[2] is not None and not op[2][i]:
                    assert got[i] == (SM.INVALID, None)
                    continue
                st, pg = ref.get_status(*key_edges.cachemap_args(*a, cfg.pshift))
                want = {"hit": SM.HIT, "miss": SM.MISS, "bad entry": SM.BAD_ENTRY}[st]
                assert got[i] == (want, pg), (op, i)
        elif k == "unset":
            m.unset(op[1])
            for a in op[1]:
                ref.unset(*a)
        assert m.sm.entries() == ref.entries() == len(m.rec)
        for a in SM.universe(cfg):
            r = m.live(a)
            assert (r and oracle.record_prefix(*a, r.clen) + r.block) == ref.record_bytes(*a) if r else True
    assert (m.ctr.requests, m.ctr.hits) == (ref.requests, ref.hits)


@pytest.mark.parametrize("pshift", [12, 16, 17])
def test_model_replays_the_key_edge_trace(pshift, oracle):
    """The reference's answers to the key-edge trace (tests/golden/key_edges.json), from the machine's model."""
    fx = key_edges.load()
    cfg = SM.MachineConfig("edges", pshift, fx["accel"], 0, 0, 1024, 1 << 30, 1024, 1 << 30, (), (1,), 1, 1, 1,
                           (0,), False, ())
    m = SM.Model(cfg, oracle)
    answers = []
    for kind, u, l, content in fx["ops"]:
        if kind == "put":
            m.put([(u, l)], [key_edges.page(content, pshift)], None, None, set())
        elif kind == "unset":
            m.unset([(u, l)])
        else:
            (st, pg), = m.get([(u, l)], None)
            answers.append(key_edges.sha(pg) if st == SM.HIT else {SM.MISS: "miss", SM.BAD_ENTRY: "bad entry"}[st])
    run = fx["runs"][str(pshift)]
    assert answers == run["gets"] == key_edges.model_replay(oracle, fx, pshift)[0]
    assert (len(m.rec), m.ctr.requests, m.ctr.hits) == (run["entries"], run["requests"], run["hits"])


@pytest.mark.parametrize("name", sorted(SM.CONFIGS))
def test_census_every_event_reached(name, oracle):
    """Each seed of a configuration reaches every event the configuration exercises, as far as the
    model alone can prove it."""
    cfg = SM.CONFIGS[name]
    for seed in cfg.seeds:
        ev = SM.census(cfg, seed, oracle)
        missing = [e for e in cfg.events if not ev.get(e)]
        assert not missing, (name, seed, missing, ev)
