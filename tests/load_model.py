"""The "as-if store" of a background load (cmb200_load_open) and seeded logs that interleave load steps
with every store operation.  It extends tests/store_machine.py without editing it.

The as-if store is the whole file loaded at open, then every call made since, in order.  A get during
or after the load must return the as-if page or a miss.  Some outcomes only the engine decides: a put
that found no arena room, or a record moved by a rename that found none.  So the model keeps, per store
key, the set of (address, page) answers that are allowed.  It checks a get by that rule alone: a hit
must be one of its key's allowed answers.  The engine's record bytes, placement and counters are
store_machine.Model's concern, not this model's.
CPU only: tests/test_gpu_load_background.py drives an engine and this model side by side.
"""
from __future__ import annotations

import store_machine as SM

HIT, MISS, BAD_ENTRY = SM.HIT, SM.MISS, SM.BAD_ENTRY


def apply_spans(page: bytes, spans) -> bytes:
    p = bytearray(page)
    for sp in spans:
        o, n = sp[0], sp[1]
        p[o:o + n] = SM.span_bytes(sp)
    return bytes(p)


class AsIfModel:
    """Allowed answers by store key: {key: {(address, page bytes)}}.  `file_pages` is {address: page} of
    the store the chain describes (one address per key, as the engine that wrote it held them)."""

    def __init__(self, key_of, file_pages: dict):
        self.key_of = key_of
        self.allowed = {}
        for a, p in file_pages.items():
            self.allowed[key_of(a)] = {(tuple(a), bytes(p))}

    def _drop_addr(self, a):
        k = self.key_of(a)
        self.allowed[k] = {x for x in self.allowed.get(k, ()) if x[0] != tuple(a)}

    def put(self, addrs, pages, valid, lens):
        """A put as the engine reported it: rows with lens >= 0 were stored; a row that stored nothing
        (superseded in its batch, invalid, or dropped for lack of room) leaves its key's older record."""
        for i, a in enumerate(addrs):
            if (valid is None or valid[i]) and lens[i] >= 0:
                self.allowed[self.key_of(a)] = {(tuple(a), bytes(pages[i]))}

    def unset(self, addrs):
        for a in addrs:
            self.allowed[self.key_of(a)] = set()

    def invalidate(self, u, lf, ll):
        for k, xs in self.allowed.items():
            self.allowed[k] = {x for x in xs if not (x[0][0] == u and lf <= x[0][1] <= ll)}

    def rename(self, uf, ut, lf, ll, dropped):
        """Every allowed answer of {uf, l}, l in [lf, ll], moves to {ut, l}.  With drops the destination
        keeps its older answers too, since a record the move found no room for leaves them in place."""
        moved = [((ut, x[0][1]), x[1]) for xs in self.allowed.values() for x in xs
                 if x[0][0] == uf and lf <= x[0][1] <= ll]
        self.invalidate(uf, lf, ll)
        for a, p in moved:
            k = self.key_of(a)
            self.allowed[k] = ({(a, p)} | self.allowed.get(k, set())) if dropped else {(a, p)}

    def patch(self, addrs, spans, status):
        """A patch call as the engine answered it.  A row answered HIT now holds its allowed page with the
        row's spans applied in array order.  Any other answer leaves no page at that address: the engine
        unsets what it could not patch, and an open load passes over the address."""
        rows = {}
        for i, a in enumerate(addrs):
            rows.setdefault(tuple(a), []).append(i)
        for a, idx in rows.items():
            k = self.key_of(a)
            if status[idx[0]] == HIT:
                sp = [spans[i] for i in idx]
                self.allowed[k] = {(a, apply_spans(p, sp)) for (b, p) in self.allowed.get(k, ()) if b == a}
            else:
                self._drop_addr(a)

    def check(self, addrs, status, pages):
        """-> the first violation as text, or None: a hit that is not one of its key's allowed answers,
        or an answer that is neither a hit nor a miss (BAD_ENTRY is a miss of a shared key)."""
        for i, a in enumerate(addrs):
            if status[i] == HIT:
                if (tuple(a), bytes(pages[i])) not in self.allowed.get(self.key_of(a), ()):
                    return f"{a}: a hit on a page the as-if store does not hold"
            elif status[i] not in (MISS, BAD_ENTRY):
                return f"{a}: status {status[i]}"
        return None


def gen_load_ops(cfg: SM.MachineConfig, seed: int) -> list:
    """store_machine.gen_ops without its fill and its load, with renames added and a load step
    ("step", max records) before every operation.  The fill is what the file holds already."""
    R = SM._Rng(seed * 7 + 3)
    ops = SM.gen_ops(cfg, seed)
    main = [(u, l) for u in cfg.us for l in range(cfg.nl)]
    fill = (len(main) + cfg.batch - 1) // cfg.batch + 1          # the fill's puts: main in batches, then edges
    out = []
    for op in ops[fill:]:
        if op[0] == "load":
            continue
        out.append(("step", 1 + R.below(2 * cfg.max_batch)))
        if R.chance(0.08):
            uf, ut = cfg.us[R.below(len(cfg.us))], cfg.us[R.below(len(cfg.us))]
            lf = R.below(cfg.nl)
            out.append(("rename", uf, ut, lf, lf + R.below(cfg.nl)))
        out.append(op)
    return out
