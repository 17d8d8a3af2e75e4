#!/usr/bin/env python
"""2+ GPU functional check of the sharded put path and the cross-GPU read path (run under torchrun,
e.g. python -m torch.distributed.run --nproc-per-node 2 --master-addr 127.0.0.1 tools/multigpu_check.py):
every rank puts its round-robin shard of a stream with 30 % same-address repeats, the ranks
exchange key records, and afterwards every rank's index must agree with a sequential pass:
the newest writer of each key is HIT on its owner and REMOTE(owner) everywhere else.
Runs twice: with the exchange records built and imported through the host (sharding.py), and with
the device-resident form (cmb200_put_step + all-gather on the engine's stream +
cmb200_import_records_dev, no host round trip)."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch
import torch.distributed as dist

import edge_fuse_b200 as E
from edge_fuse_b200 import sharding

rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
torch.cuda.set_device(local)
dist.init_process_group("nccl", device_id=torch.device("cuda", local))
n_total, bs = 4096 * world, 65536
cids, distinct = E.gen_stream_ids(n_total, 0.3)
off, nh = E.gen_addr(42, cids, 16)
mine = np.arange(rank, n_total, world)
u, l = nh[mine], off[mine] >> np.uint64(16)
# expectation from a sequential pass over the global stream
last = {}
for k in range(n_total):
    last[int(cids[k])] = k
qc = np.array(sorted(last), dtype=np.uint64)
qo, qn = E.gen_addr(42, qc, 16)
exp_owner = np.array([last[int(c)] % world for c in qc])
all_ok = True
for mode in ("host", "device"):
    eng = E.Engine(pshift=16, accel=12, capacity=4 * n_total, arena_bytes=n_total * bs // world + (256 << 20),
                   max_batch=1024, device=local)
    d = eng.dev_alloc(len(mine) * bs)
    eng.gen_chunks_dev(42, cids[mine], d)
    stream = torch.cuda.ExternalStream(eng.stream(), device=torch.device("cuda", local))
    rec_d = [torch.empty((1024, 4), dtype=torch.int64, device="cuda") for _ in range(2)]
    gat_d = [torch.empty((1024 * world, 4), dtype=torch.int64, device="cuda") for _ in range(2)]
    torch.cuda.synchronize()
    for bi, b0 in enumerate(range(0, len(mine), 1024)):        # several batches, one exchange each
        sl = slice(b0, b0 + 1024)
        pos = (1 + mine[sl]).astype(np.uint64)
        eng.set_stream_order(int(pos[0]), world)
        if mode == "host":
            lens = eng.put(u[sl], l[sl], d + b0 * bs, on_dev=True)
            rec = torch.from_numpy(sharding.pack_records(u[sl], l[sl], pos, rank, lens)).cuda()
            gathered = sharding.all_gather_records(rec)
            sharding.import_gathered(eng, gathered, rank)
        else:
            k = bi & 1
            with torch.cuda.stream(stream):
                eng.put_step(u[sl], l[sl], d + b0 * bs, on_dev=True, rank=rank, records_dev=rec_d[k].data_ptr())
                dist.all_gather_into_tensor(gat_d[k], rec_d[k])
                eng.import_records_dev(1024 * world, gat_d[k].data_ptr(), rank)
    eng.sync()
    torch.cuda.synchronize()
    status, owner = eng.locate(qn, qo >> np.uint64(16))
    ok = ((status == E.HIT) == (exp_owner == rank)).all() and (owner[status == E.REMOTE] == exp_owner[status == E.REMOTE]).all() \
        and ((status == E.HIT) | (status == E.REMOTE)).all()
    st = eng.stats()
    tot = torch.tensor([st["entries"]], device="cuda")
    dist.all_reduce(tot)
    ok = ok and int(tot.item()) == distinct and st["entries"] + st["remote_entries"] == distinct
    remote_ok = None
    if mode == "device":
        # cross-GPU read path: map the other ranks' arenas (CUDA IPC -> NVLink peer memory); a get of a key
        # whose newest record lives elsewhere then reads that record out of its owner's arena and decodes it here
        sharding.open_peers(eng, rank, world)
        dist.barrier()
        pick = np.arange(0, len(qc), max(1, len(qc) // 1024))[:1024]
        out, gst = eng.get_small(qn[pick], (qo >> np.uint64(16))[pick])
        want = np.stack([E.gen_chunk_host(42, int(c), bs) for c in qc[pick]])
        remote_ok = bool((gst == E.HIT).all() and (out == want).all())
        n_remote = int((exp_owner[pick] != rank).sum())
        ok = ok and remote_ok and n_remote > 0
        eng.close_peers()
        dist.barrier()                                  # nobody frees its arena while a peer still maps it
    print(f"rank {rank} [{mode} exchange]: ok={bool(ok)} local={st['entries']} remote={st['remote_entries']} distinct={distinct}"
          + (f" remote_gets_ok={remote_ok}" if remote_ok is not None else ""), flush=True)
    all_ok = all_ok and bool(ok)
    eng.dev_free(d)
    eng.close()
ok = all_ok
flag = torch.tensor([int(ok)], device="cuda")
dist.all_reduce(flag, op=dist.ReduceOp.MIN)
dist.destroy_process_group()
sys.exit(0 if flag.item() == 1 else 1)
