#!/bin/bash
# Nsight Compute evidence on one GPU: launch list of one fit + 10^4-candidate query, and --set full captures of the dominant
# kernels, each summarised next to its capture (the .ncu-rep files are large; the text summaries are what to keep).
# usage: bash tools/ncu_capture.sh [OUT]     (default OUT = ncu_out; outputs: OUT/launches.txt, OUT/ncu_<kernel>.txt, OUT/*.ncu-rep)
#        LB_NCU_ONLY="panel_update syrk" bash tools/ncu_capture.sh     (launch list + only the named captures)
set -u
OUT=${1:-ncu_out}
mkdir -p "$OUT"
NCU="ncu --set full --clock-control none --import-source on -f"
ncu --metrics gpu__time_duration.sum --clock-control none -c 700 --csv --log-file "$OUT/launches.csv" python tools/profile_step.py 16384 10000 > "$OUT/launches.log" 2>&1
python tools/ncu_summary.py launches "$OUT/launches.csv" > "$OUT/launches.txt" 2>&1
cap() { # name, kernel regex, skip, command...
  local name=$1 rx=$2 skip=$3; shift 3
  if [ -n "${LB_NCU_ONLY:-}" ] && [[ " $LB_NCU_ONLY " != *" $name "* ]]; then return; fi
  $NCU -k regex:$rx -s $skip -c 1 -o "$OUT/$name" "$@" > "$OUT/$name.log" 2>&1
  python tools/ncu_summary.py kernel "$OUT/$name.ncu-rep" > "$OUT/ncu_$name.txt" 2>&1
}
# at 10^4 candidates the panel path walks the super-blocks on one stream: launch 4 = super-block 4
cap panel_update panel_update_kernel 4 python tools/profile_step.py 16384 10000     # super-block 4: K = 8192
cap panel_solve panel_solve_kernel 4 python tools/profile_step.py 16384 10000
# syrk_kernel launches of quad 0: column updates inside the two pair panels (0, 2), the K = 256 update of pair 1's columns (1), a(0) (3), b(0) (4)
cap syrk syrk_kernel 4 python tools/profile_step.py 16384 0                          # b(0): first K = 512 trailing update
cap kbuild_se_ard kbuild_kernel 0 python tools/profile_step.py 16384 0
cap trsv_fwd trsv_fwd_kernel 0 python tools/profile_step.py 16384 0
cap trsv_bwd trsv_bwd_kernel 0 python tools/profile_step.py 16384 0
cap grad grad_kernel 0 python tools/profile_step.py 16384 0 --grad
cap kbuild_matern52 kbuild_kernel 3 python tools/kbuild_timing.py 16384 6 MaternFiveHalves
cap kstar kstar_kernel 0 python tools/profile_step.py 16384 10000
ls -la "$OUT"
