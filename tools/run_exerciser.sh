#!/bin/bash
# tests/c/exerciser.c against the drop-in, bounded (debugging aid): run_exerciser.sh [count] [pshift] [seed]
cd "$(dirname "$0")/.."
gcc -O2 -I include tests/c/exerciser.c -o /tmp/exer_ours -L edge_fuse_b200 -lcachemap -Wl,-rpath,$PWD/edge_fuse_b200 -lpthread || exit 1
d=$(mktemp -d)
CMB200_ARENA_MB=2048 CMB200_PERSIST=0 timeout ${T:-60} /tmp/exer_ours $d ${1:-32768} ${2:-15} ${3:-1}
echo "rc=$?"
rm -rf $d
