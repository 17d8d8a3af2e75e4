#!/usr/bin/env python
"""Summarises an .ncu-rep: stall reasons, hottest CUDA source lines and SASS instructions.
    python tools/ncu_lines.py x.ncu-rep [top]"""
import csv, subprocess, sys, io, os
rep = sys.argv[1]; top = int(sys.argv[2]) if len(sys.argv) > 2 else 30
out = subprocess.run(["ncu", "-i", rep, "--page", "source", "--csv", "--print-source", "cuda,sass"], capture_output=True, text=True).stdout
rows = list(csv.reader(io.StringIO(out)))
cur, hdr, lines, sass = None, None, [], []
for r in rows:
    if not r: continue
    if r[0] == "File Path": cur = os.path.basename(r[1]); continue
    if r[0] == "Function Name": continue
    if r[0] == "Line No": hdr = r; continue
    if hdr is None or len(r) < len(hdr) - 2: continue
    (lines if r[0] else sass).append((cur, r))
ix = {}
for i, h in enumerate(hdr):
    ix.setdefault(h, i)
def S(r, c):
    try:
        return int(float(r[ix[c]]))
    except Exception:
        return 0
tot = sum(S(r, "# Samples") for _, r in lines); inst = sum(S(r, "Instructions Executed") for _, r in lines)
print(f"samples {tot}  warp-instructions {inst}")
cols = [c for c in hdr if c.startswith("stall_") and "Not Issued" not in c]
for c, v in sorted(((c, sum(S(r, c) for _, r in lines)) for c in cols), key=lambda x: -x[1])[:8]:
    print(f"  {c:26s}{100 * v / tot:5.1f}%")
print("--- top source lines: samples%  instr%  file:line")
for f, r in sorted(lines, key=lambda x: -S(x[1], "# Samples"))[:top]:
    print(f"{100*S(r,'# Samples')/tot:5.1f}% {100*S(r,'Instructions Executed')/inst:5.1f}%  {f}:{r[0]:>4s}  {r[1].strip()[:95]}")
print("--- top SASS")
for f, r in sorted(sass, key=lambda x: -S(x[1], "# Samples"))[:top // 2]:
    print(f"{100*S(r,'# Samples')/tot:5.1f}% x{S(r,'Instructions Executed'):9d} {r[3].strip()[:70]:70s} long {S(r,'stall_long_sb')} short {S(r,'stall_short_sb')} wait {S(r,'stall_wait')}")
if len(sys.argv) > 3:
    print("--- by line of", sys.argv[3])
    for f, r in sorted([x for x in lines if x[0] == sys.argv[3]], key=lambda x: int(x[1][0])):
        if S(r, "Instructions Executed") * 1000 > inst:
            print(f"{r[0]:>4s} smp {100*S(r,'# Samples')/tot:5.1f}% ins {100*S(r,'Instructions Executed')/inst:5.1f}%  {r[1].strip()[:100]}")
