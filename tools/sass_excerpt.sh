#!/bin/bash
# SASS evidence (no GPU needed): which Hopper-era instructions the built library contains.
# usage: tools/sass_excerpt.sh > sass_excerpt.txt
SO=aprilsam_b200/lib/libaprilsam_b200.so
echo "# cuobjdump -sass $SO  ($(date -u +%F), nvcc $(nvcc --version | grep release | sed 's/.*release //'))"
echo "# sm_90a cubin; counts of the instructions that matter (per kernel: the function the line belongs to)"
cuobjdump -sass $SO | awk '
/Function :/ { fn=$3 }
/DMMA/ { dmma[fn]++ }
/UBLKCP/ { ublk[fn]++ }
/SYNCS\./ { syncs[fn]++ }
/UTMALDG|UTMASTG/ { utma[fn]++ }
/DFMA/ { dfma[fn]++ }
/UTC[A-Z]*MMA|LDTM|STTM/ { tc[fn]++ }
END {
  printf("%-70s %6s %6s %6s %6s %6s %6s\n", "function", "DFMA", "DMMA", "UBLKCP", "SYNCS", "UTMA*", "tcgen05");
  for (f in dfma) all[f]=1; for (f in dmma) all[f]=1; for (f in ublk) all[f]=1;
  for (f in all) printf("%-70s %6d %6d %6d %6d %6d %6d\n", f, dfma[f], dmma[f], ublk[f], syncs[f], utma[f], tc[f]);
}' | sort
echo
echo "# excerpt from k_factor (tile_rm / tile_mma are non-inlined device functions inside it): mbarrier arm + bulk asynchronous"
echo "# copies (cp.async.bulk -> UBLKCP.S.G, expect_tx -> SYNCS.ARRIVE.TRANS64, try_wait -> SYNCS.PHASECHK) and the FP64 tensor-pipe"
echo "# instructions (mma.sync.m8n8k4.f64 -> DMMA.8x8x4)"
cuobjdump -sass $SO | awk '/Function : _Z8k_factor7FacArgs/ {p=1; next} p && /Function :/ {p=0} p' | grep -E "UBLKCP|SYNCS|DMMA|FENCE\.VIEW|MEMBAR" | sed 's/^ *//' | awk '!seen[$2" "$3]++' | head -40
