#!/bin/bash
# SASS opcode summary per kernel of libnrnerf_b200.so: proves the wgmma / bulk-TMA / mbarrier instructions are in the binary.
#   scripts/sass_summary.sh > sass_summary.txt
set -e
SO=${1:-nonrigid_nerf_b200/libnrnerf_b200.so}
echo "# cuobjdump -sass $SO  (sm_90a) -- instruction counts per kernel"
echo "# HGMMA = wgmma.mma_async, UBLKCP = cp.async.bulk (G.S load / S.G store), UBLKPF = bulk L2 prefetch, SYNCS = mbarrier"
cuobjdump -sass "$SO" | awk '
/Function :/ { fn=$3; next }
{
  if (fn == "") next;
  n[fn]++;
  if ($0 ~ /HGMMA/) c[fn,"HGMMA"]++;
  if ($0 ~ /UBLKCP\.S\.G|UBLKCP.*\.S\.G/) c[fn,"UBLKCP.S.G"]++; else if ($0 ~ /UBLKCP/) c[fn,"UBLKCP.G.S"]++;
  if ($0 ~ /UBLKPF/) c[fn,"UBLKPF"]++;
  if ($0 ~ /SYNCS/) c[fn,"SYNCS"]++;
  if ($0 ~ /HMMA|IMMA/ && $0 !~ /HGMMA/) c[fn,"legacy-MMA"]++;
  if ($0 ~ /MUFU/) c[fn,"MUFU"]++;
  if ($0 ~ /ATOM|RED\./) c[fn,"ATOM/RED"]++;
  if ($0 ~ /LD\.E.*SYS|ST\.E.*SYS|\.STRONG\.SYS/) c[fn,"sys-scope ld/st"]++;
}
END {
  split("HGMMA UBLKCP.G.S UBLKCP.S.G UBLKPF SYNCS MUFU ATOM/RED sys-scope_ld/st legacy-MMA", cols, " ");
  printf "%-62s %8s", "kernel", "instrs";
  for (i = 1; i <= 9; i++) printf " %12s", cols[i];
  printf "\n";
  for (f in n) {
    g = f; gsub(/^_ZN3nrn[0-9]*/, "", g); gsub(/_GLOBAL__N__[0-9a-f_]*/, "", g);
    printf "%-62s %8d", substr(g, 1, 62), n[f];
    for (i = 1; i <= 9; i++) { k = cols[i]; gsub(/_/, " ", k); printf " %12d", c[f,k] + 0; }
    printf "\n";
  }
}' | (read -r hdr; echo "$hdr"; sort)
