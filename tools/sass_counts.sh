#!/usr/bin/env bash
# Counts, per shipped object (sm_90a), the SASS mnemonics that show wgmma / TMA use:
#   HGMMA = wgmma.mma_async, UTMALDG / UTMASTG = TMA tensor load / store, SYNCS = mbarrier operations,
#   HMMA = mma.sync, LDGSTS = cp.async, LDSM = ldmatrix. CPU-only (cuobjdump).   usage: tools/sass_counts.sh
set -euo pipefail
cd "$(dirname "$0")/../vilbert-multi-task_b200/csrc"
echo "# cuobjdump -sass of the shipped objects (sm_90a): counts of the mnemonics that show wgmma / TMA use"
for o in vb_*.o; do
  echo "## $o"
  s=$(/usr/local/cuda/bin/cuobjdump -sass "$o")
  for m in HGMMA UTMALDG UTMASTG SYNCS HMMA LDGSTS LDSM 'ATOMS\|RED'; do
    printf "  %-14s %6d\n" "$m" "$(printf '%s\n' "$s" | grep -c "$m" || true)"
  done
done
