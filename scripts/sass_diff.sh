#!/bin/bash
# Per-kernel SASS of two builds of libnrnerf_b200.so, compared instruction by instruction (anonymous-namespace hashes,
# which depend on the build directory, normalised; so are runs of blanks, since cuobjdump pads every instruction of a cubin
# to the widest one in it): which kernels are identical, which differ, which exist in one only.
#   scripts/sass_diff.sh parent/libnrnerf_b200.so nonrigid_nerf_b200/libnrnerf_b200.so
set -e
tmp=$(mktemp -d)
trap 'rm -rf "$tmp"' EXIT
dump() { mkdir -p "$2"; cuobjdump -sass "$1" | awk -v out="$2" '/Function :/ {fn=$3; gsub(/_GLOBAL__N__[0-9a-f]+_[0-9]+_[a-z_]+cu_[0-9a-f]+/, "ANON", fn); next} fn!="" && /\/\*[0-9a-f]+\*\// {gsub(/[ \t]+/, " "); print > (out "/" fn ".sass")}'; }
dump "$1" "$tmp/a"; dump "$2" "$tmp/b"
same=0; diff=0
for f in "$tmp"/a/*.sass; do n=$(basename "$f"); if [ -f "$tmp/b/$n" ]; then if cmp -s "$f" "$tmp/b/$n"; then same=$((same+1)); else diff=$((diff+1)); echo "DIFFERENT $n"; fi; else echo "ONLY-FIRST $n"; fi; done
for f in "$tmp"/b/*.sass; do n=$(basename "$f"); [ -f "$tmp/a/$n" ] || echo "ONLY-SECOND $n"; done
echo "identical: $same  different: $diff"
