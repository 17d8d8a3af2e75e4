"""CPU checks of tests/flag_model.py and of the flag matrix tests/test_gpu_flag_matrix.py runs.

Reach: the model over every case's script answers every status the case's flags allow, on every get path,
and HIT, BAD_DECODE and CORRUPT from records in both tiers.  Coverage: the matrix launches every compiled
k_get_small / k_get_small_pair instantiation and every k_decode variant, so trimming it cannot silently drop
one."""
import pytest

import flag_model as M


def _allowed(case):
    verify = bool(case["flags"] & M.VERIFY)
    want = set()
    for path in M.PATHS:
        for st in (M.MISS, M.BAD_ENTRY):
            want.add((path, st, "-"))
        if path in ("batch", "dev"):
            want.add((path, M.INVALID, "-"))
        for st in (M.HIT, M.BAD_DECODE) + ((M.CORRUPT,) if verify else ()):
            for tier in ("arena", "host"):
                want.add((path, st, tier))
    return want


@pytest.mark.parametrize("case", M.CASES, ids=[c["id"] for c in M.CASES])
def test_every_case_reaches_every_answer_on_every_path_from_both_tiers(oracle, case):
    census = set()
    m = M.run(case, census=census)
    missing = _allowed(case) - census
    assert not missing, sorted(missing)
    if not case["flags"] & M.VERIFY:
        assert not any(s == M.CORRUPT for _p, s, _t in census)
    if m.ghosts is not None:
        g = m.ghosts
        assert g.inserted > 5 and g.refaults > 0 and g.removed > 0, g.stats()
    if m.sketch is not None:
        assert m.sketch.halvings >= 1, vars(m.sketch)
    if case["flags"] & M.VERIFY:
        assert all(v > 0 for v in m.vstat.values()), m.vstat
    assert m.tier_hits > 0


GHOST_CASES = [c for c in M.CASES if c["flags"] & M.GHOST]


@pytest.mark.parametrize("case", GHOST_CASES, ids=[c["id"] for c in GHOST_CASES])
def test_a_ghost_behind_a_bad_entry_survives(oracle, case):
    """Every GHOST case's script evicts pair0[0] (a ghost), stores pair0[1] under the same key, and asks for
    pair0[0]: the answer is BAD_ENTRY, which does not probe, so the ghost is still there."""
    a0 = M._edges()[0]
    files, ops = M.script(case)
    m = M.FlagModel(case["flags"], case["pshift"])
    for recs, fp in files:
        m.load(recs, fp)
    seen = 0
    for op in ops:
        if op[0] == "get" and any(a0 in part for part in op[2]) and m.status(a0)[0] == M.BAD_ENTRY:
            before = [w[:] for w in m.ghosts.tab if (w[0], w[1]) == a0 and w[2]]
            if before:
                M.apply(m, op)
                assert [w for w in m.ghosts.tab if (w[0], w[1]) == a0 and w[2]] == before
                seen += 1
                continue
        M.apply(m, op)
    assert seen >= 2, seen          # the batch get and the fused get that follow pair0[1]'s put


def test_the_matrix_launches_every_get_kernel():
    small = {f"{k}<{v},{t},{f}>" for k in ("k_get_small", "k_get_small_pair")
             for v in ("false", "true") for t in ("false", "true") for f in ("false", "true")}
    decode = {"k_decode", "k_decode_verify", "k_decode_touch", "k_decode_verify_touch"}
    got = set().union(*(M.kernels(c) for c in M.CASES))
    assert small | decode <= got, sorted((small | decode) - got)
    assert len(small) == 16


@pytest.mark.parametrize("case", [c for c in M.CASES if c["flags"] & M.FREQ],
                         ids=[c["id"] for c in M.CASES if c["flags"] & M.FREQ])
def test_the_concurrent_lane_step_crosses_no_halving(oracle, case):
    """The "lanes" step runs its gets from two threads in no fixed order.  Its answers, the ghost table and the
    sketch do not depend on that order as long as no halving falls inside the step."""
    files, ops = M.script(case)
    m = M.FlagModel(case["flags"], case["pshift"])
    for recs, fp in files:
        m.load(recs, fp)
    lanes = [op for op in ops if op[0] == "get" and op[1] == "lanes"]
    assert len(lanes) == 1
    for op in ops:
        before = m.sketch.halvings
        M.apply(m, op)
        if op is lanes[0]:
            assert m.sketch.halvings == before
