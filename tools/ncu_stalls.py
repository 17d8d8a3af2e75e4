#!/usr/bin/env python
"""Stall-reason totals and hottest SASS instructions of an .ncu-rep (source page, SASS view only).
    python tools/ncu_stalls.py x.ncu-rep [top] [min_exec_for_hot_loop]"""
import csv, io, subprocess, sys
rep = sys.argv[1]; top = int(sys.argv[2]) if len(sys.argv) > 2 else 20
hot_thr = int(sys.argv[3]) if len(sys.argv) > 3 else 0
out = subprocess.run(["ncu", "-i", rep, "--page", "source", "--csv", "--print-source", "sass"], capture_output=True, text=True).stdout
hdr, data = None, []
for r in csv.reader(io.StringIO(out)):
    if r and r[0] == "Address": hdr = r; continue
    if hdr and len(r) == len(hdr): data.append(r)
ix = {h: i for i, h in enumerate(hdr)}
S = lambda r, c: int(r[ix[c]])
tot = sum(S(r, "# Samples") for r in data); inst = sum(S(r, "Instructions Executed") for r in data)
print(f"samples {tot}  warp-instructions {inst}  SASS instructions {len(data)}")
cols = [c for c in hdr if c.startswith("stall_") and "Not Issued" not in c]
for c, v in sorted(((c, sum(S(r, c) for r in data)) for c in cols), key=lambda x: -x[1])[:9]:
    print(f"  {c:26s}{100 * v / tot:5.1f}%")
if hot_thr:
    hot = [r for r in data if S(r, "Instructions Executed") > hot_thr]
    it = max(S(r, "Instructions Executed") for r in data)
    print(f"hot loop: {len(hot)} SASS instructions, {sum(S(r, 'Instructions Executed') for r in hot) / it:.1f} executed per iteration, "
          f"{100 * sum(S(r, '# Samples') for r in hot) / tot:.1f}% of samples; whole kernel {inst / it:.1f} per iteration")
print("--- top SASS by samples")
for i, r in sorted(enumerate(data), key=lambda x: -S(x[1], "# Samples"))[:top]:
    print(f"{i:5d} {100 * S(r, '# Samples') / tot:5.1f}% x{S(r, 'Instructions Executed'):9d} {r[1].strip()[:64]:64s} long {S(r, 'stall_long_sb')} short {S(r, 'stall_short_sb')} wait {S(r, 'stall_wait')} br {S(r, 'stall_branch_resolving')}")
