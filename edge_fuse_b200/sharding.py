"""Multi-GPU plumbing for the cachemap put path (SURVEY.md §8e, option B).

Chunk k of the global stream belongs to rank k mod world (round-robin); every rank encodes and
stores its own chunks with no data-path collective.  What is replicated is the key index: after
each batch the ranks all-gather one fixed-size record per stored chunk — {address u, address l,
global stream position, owner rank | stored length} = 32 bytes — over NCCL (NVLink / NVSwitch) and
import the other ranks' records into their table replica (cmb200_import_records_dev, straight from
the gathered records), where the highest stream position per key wins, i.e. the outcome of the
sequential reference.  torch.distributed is only the transport; the table logic is in the CUDA
library.
"""
from __future__ import annotations

import numpy as np

REC_WORDS = 4   # int64 words per record


def shard_positions(rank: int, world: int, n_local: int, base: int = 0) -> np.ndarray:
    """Global stream positions of this rank's chunks: base + rank, base + rank + world, ..."""
    return (np.uint64(base) + np.uint64(rank) + np.uint64(world) * np.arange(n_local, dtype=np.uint64))


LEN_BITS, OFF_BITS = 22, 34   # word 3: owner rank << 56 | arena offset / 16 << 22 | stored length + 1


def pack_records(u, l, seq, rank: int, lens, rec_off=None) -> np.ndarray:
    """[n, 4] int64: u, l, seq, tail.  tail = rank << 56 | (arena offset / 16) << 22 | (len + 1)
    (csrc/kernels.h xrec_tail): len < 0 marks a chunk that stored nothing (rejected address,
    superseded inside its batch, dropped) — its low 22 bits are 0 and importers ignore the row;
    rec_off = where the record lies in the owner's arena (0 when unknown), for NVLink reads."""
    n = len(u)
    rec = np.empty((n, REC_WORDS), dtype=np.int64)
    rec[:, 0] = np.asarray(u, dtype=np.uint64).view(np.int64)
    rec[:, 1] = np.asarray(l, dtype=np.uint64).view(np.int64)
    rec[:, 2] = np.asarray(seq, dtype=np.uint64).view(np.int64)
    ln = np.asarray(lens, dtype=np.int64)
    len1 = np.where(ln < 0, 0, ln + 1).astype(np.uint64)
    off = np.zeros(n, dtype=np.uint64) if rec_off is None else np.asarray(rec_off, dtype=np.uint64)
    off = np.where(ln < 0, np.uint64(0), off)
    tail = (np.uint64(rank) << np.uint64(56)) | (((off >> np.uint64(4)) & np.uint64((1 << OFF_BITS) - 1)) << np.uint64(LEN_BITS)) | len1
    rec[:, 3] = tail.view(np.int64)
    return rec


def unpack_records(rec):
    """-> u, l, seq, owner, length (arrays; works on numpy arrays and torch tensors alike);
    length = -1 for rows that stored nothing."""
    u, l, seq, tail = rec[..., 0], rec[..., 1], rec[..., 2], rec[..., 3]
    owner = (tail >> 56) & 0xFF
    length = (tail & ((1 << LEN_BITS) - 1)) - 1
    return u, l, seq, owner, length


def unpack_locations(rec):
    """-> arena offset of each row's record in its owner's arena (bytes)."""
    tail = rec[..., 3]
    return ((tail >> LEN_BITS) & ((1 << OFF_BITS) - 1)) << 4


def all_gather_records(rec_tensor, group=None):
    """One all-gather of this rank's [n, 4] int64 records -> [world * n, 4] (same device)."""
    import torch
    import torch.distributed as dist
    world = dist.get_world_size(group)
    out = torch.empty((world * rec_tensor.shape[0], REC_WORDS), dtype=torch.int64, device=rec_tensor.device)
    try:
        dist.all_gather_into_tensor(out, rec_tensor.contiguous(), group=group)
    except (RuntimeError, NotImplementedError):                    # backends without the flat form
        parts = [torch.empty_like(rec_tensor) for _ in range(world)]
        dist.all_gather(parts, rec_tensor.contiguous(), group=group)
        out = torch.cat(parts, dim=0)
    return out


def remote_rows(gathered, rank: int):
    """Rows written by other ranks that actually stored something (torch tensor or numpy array)."""
    _, _, _, owner, length = unpack_records(gathered)
    keep = (owner != rank) & (length >= 0)
    return gathered[keep]


def resolve_newest(records: np.ndarray) -> dict:
    """Reference resolution on the host (tests): key (u, l) -> (seq, owner) of the highest seq."""
    best = {}
    u, l, seq, owner, length = unpack_records(records)
    for i in range(len(records)):
        if length[i] < 0:
            continue
        k = (int(np.uint64(u[i])), int(np.uint64(l[i])))
        s = int(np.uint64(seq[i]))
        if k not in best or s > best[k][0]:
            best[k] = (s, int(owner[i]))
    return best


def import_gathered(engine, gathered, rank: int) -> int:
    """Imports the other ranks' rows of an all-gathered [n, 4] int64 record tensor into `engine`'s
    index replica (cmb200_import_records_dev, which skips the rows of `rank` and the rows that stored
    nothing).  A CUDA tensor must be on the engine's device; a CPU tensor is copied there first.  The
    import is complete on return.  Returns the number of rows imported."""
    _, _, _, owner, length = unpack_records(gathered)
    n = int(((owner != rank) & (length >= 0)).sum())
    if n == 0:
        return 0
    rows = gathered.contiguous()
    if rows.is_cuda:
        import torch
        torch.cuda.current_stream(rows.device).synchronize()      # the gather has landed before the engine reads it
        engine.import_records_dev(rows.shape[0], rows.data_ptr(), rank)
        engine.sync()
        return n
    d = engine.dev_alloc(rows.numel() * 8)
    try:
        engine.h2d(d, rows.numpy())
        engine.import_records_dev(rows.shape[0], d, rank)
        engine.sync()
    finally:
        engine.dev_free(d)
    return n


def open_peers(engine, rank: int, world: int, group=None) -> None:
    """Maps every other rank's arena into this process (CUDA IPC -> NVLink peer memory) so that
    cmb200_get_small serves keys whose newest record lives on another GPU.  One all-gather of the
    64-byte IPC handles; ranks must be processes on one box."""
    import torch
    import torch.distributed as dist
    handle, size = engine.arena_ipc_handle()
    mine = torch.tensor(list(handle) + list(int(size).to_bytes(8, "little")), dtype=torch.uint8)
    dev = torch.device("cuda", torch.cuda.current_device()) if dist.get_backend(group) == "nccl" else torch.device("cpu")
    mine = mine.to(dev)
    allh = [torch.empty_like(mine) for _ in range(world)]
    dist.all_gather(allh, mine, group=group)
    for r in range(world):
        if r == rank:
            continue
        raw = bytes(allh[r].cpu().tolist())
        engine.open_peer(r, raw[:64], int.from_bytes(raw[64:72], "little"))


class StepExchange:
    """The sharded put step as the product runs it (SURVEY.md §8e option B), device resident:

        engine stream   put_step(k)  [upsert, encode, pack records] | import(k-1) | put_step(k+1) | ...
        side stream                  all_gather(k)  ------------------^ (event)

    `step()` enqueues one step of this rank's shard (cmb200_put_step: asynchronous, the 32-byte
    exchange records are packed on the device), starts ONE all-gather of those records (NCCL over
    NVLink) on a side stream, and imports the previous step's gathered records into the index replica
    (cmb200_import_records_dev, one claim + one apply launch).  The all-gather of step k therefore
    overlaps the encode of step k+1; nothing in the sequence waits on the host.  Importing a step's
    records after the next local put is harmless: last-writer-wins is decided by the global stream
    position each record carries, not by arrival order (SURVEY.md App. B rule 4).  With one rank
    there is no exchange and `step()` is cmb200_put_step alone.  Call `flush()` after the last step.
    """

    def __init__(self, engine, n_per_step: int, rank: int, world: int, device, timing: bool = False):
        import torch
        self.torch = torch
        self.eng, self.n, self.rank, self.world = engine, n_per_step, rank, world
        self.dev = torch.device(device)
        self.main = torch.cuda.ExternalStream(engine.stream(), device=self.dev)
        self.rec = [torch.empty((n_per_step, REC_WORDS), dtype=torch.int64, device=self.dev) for _ in range(2)]
        self.count = 0
        self.pending = None
        self.timing = timing
        self.times = {"allgather": [], "import": []}      # lists of (start, end) event pairs
        if world > 1:
            self.side = torch.cuda.Stream(device=self.dev)
            self.gath = [torch.empty((world * n_per_step, REC_WORDS), dtype=torch.int64, device=self.dev) for _ in range(2)]
            self.put_done = [torch.cuda.Event() for _ in range(2)]
            self.gathered = [torch.cuda.Event() for _ in range(2)]
        torch.cuda.synchronize(self.dev)

    def _timed(self, stream):
        if not self.timing:
            return None
        e = self.torch.cuda.Event(enable_timing=True)
        e.record(stream)
        return e

    def _import(self, k: int):
        self.main.wait_event(self.gathered[k])
        a = self._timed(self.main)
        self.eng.import_records_dev(self.world * self.n, self.gath[k].data_ptr(), self.rank)
        b = self._timed(self.main)
        if a is not None:
            self.times["import"].append((a, b))

    def step(self, u, l, pages, on_dev, ts=None, lens=None, next_seq=None) -> int:
        """One step: chunk i of this rank is global stream position next_seq + world * i
        (set_stream_order is applied when next_seq is given).  -> ticket for engine.wait()."""
        import torch.distributed as dist
        torch = self.torch
        k = self.count & 1
        self.count += 1
        if next_seq is not None:
            self.eng.set_stream_order(int(next_seq), self.world)
        with torch.cuda.stream(self.main):
            ticket = self.eng.put_step(u, l, pages, ts=ts, on_dev=on_dev, rank=self.rank,
                                       records_dev=self.rec[k].data_ptr(), lens=lens)
        if self.world > 1:
            self.put_done[k].record(self.main)
            self.side.wait_event(self.put_done[k])
            with torch.cuda.stream(self.side):
                a = self._timed(self.side)
                dist.all_gather_into_tensor(self.gath[k], self.rec[k])
                b = self._timed(self.side)
            if a is not None:
                self.times["allgather"].append((a, b))
            self.gathered[k].record(self.side)
            if self.pending is not None:
                self._import(self.pending)
            self.pending = k
        return ticket

    def flush(self):
        """Imports the last step's records (enqueued on the engine's stream; not a host sync)."""
        if self.world > 1 and self.pending is not None:
            self._import(self.pending)
            self.pending = None

    def last_lens(self) -> np.ndarray:
        """Stored block lengths of the most recent step (-1 = stored nothing), from its records."""
        k = (self.count - 1) & 1
        self.torch.cuda.synchronize(self.dev)
        tail = self.rec[k][:, 3].cpu().numpy()
        return ((tail & ((1 << LEN_BITS) - 1)) - 1).astype(np.int64)

    def breakdown_ms(self) -> dict:
        """Mean device time of the exchange stages (needs timing=True and a synchronized device)."""
        out = {}
        for key, pairs in self.times.items():
            if pairs:
                out[key + "_ms"] = float(np.mean([a.elapsed_time(b) for a, b in pairs]))
        return out
