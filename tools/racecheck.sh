#!/bin/bash
# compute-sanitizer --tool racecheck over the wavefront kernel's shared-memory protocol (ring queues, slot
# state hand-over) in every scheduler variant x CTA size, on tiny workloads.
#   tools/racecheck.sh OUTDIR
# Prints per-run hazard summaries (also OUTDIR/racecheck.txt); the full log goes to OUTDIR/racecheck_full.log.
OUTDIR=${1:?usage: tools/racecheck.sh OUTDIR}
mkdir -p "$OUTDIR"
OUT=$OUTDIR/racecheck.txt
: > "$OUT"; : > "$OUTDIR/racecheck_full.log"
run() {  # name, env..., scene w h spp
  local name=$1; shift
  echo "== racecheck $name: $*" | tee -a "$OUT"
  ( env "$@" timeout 280 compute-sanitizer --tool racecheck --racecheck-report analysis --print-limit 20 python tools/profile_run.py $SCENE 2>&1 ) > "$OUTDIR/rc_one.log"
  cat "$OUTDIR/rc_one.log" >> "$OUTDIR/racecheck_full.log"
  grep -E "RACECHECK SUMMARY|ERROR SUMMARY|hazard|Msamples|Error" "$OUTDIR/rc_one.log" | sort | uniq -c | sort -rn | head -8 | tee -a "$OUT"
}
SCENE="cornell 64 48 1 1";   run "free 512 (wf2_smem generic)" TINSEL_B200_SCHED=free TINSEL_B200_CTA=512
SCENE="cornell 64 48 1 1";   run "lanes 512 (wf2_lq generic)" TINSEL_B200_SCHED=free TINSEL_B200_QUEUES=lanes TINSEL_B200_CTA=512
SCENE="veach 64 48 1 1";     run "hard 512 (wf2_smem hard)" TINSEL_B200_SCHED=hard TINSEL_B200_CTA=512
SCENE="meshlight 64 48 1 1"; run "split 512 (wf2_smem split)" TINSEL_B200_SCHED=free TINSEL_B200_SPLIT=1 TINSEL_B200_CTA=512
SCENE="meshlight 64 48 1 1"; run "free 768 (wf2_l2 generic)" TINSEL_B200_SCHED=free TINSEL_B200_SPLIT=0 TINSEL_B200_CTA=768
SCENE="veach 64 48 1 1";     run "hard 768 (wf2_l2 generic, hard flag)" TINSEL_B200_SCHED=hard TINSEL_B200_CTA=768
SCENE="meshlight 64 48 1 1"; run "split 768 (wf2_l2 split)" TINSEL_B200_SCHED=free TINSEL_B200_SPLIT=1 TINSEL_B200_CTA=768
