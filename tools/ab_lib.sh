#!/bin/bash
# Compares two builds of libttsb.so (TTSB_LIB) on one GPU, in one run:
#   tools/ab_lib.sh <lib A> <lib B> <out dir> <reps> [bench.py arguments...]
# - the card's name, power limit and top SM clock;
# - `bench.py --no-train --no-cpu-baseline [arguments]` <reps> times per library, alternating A and B so that both see the
#   same host and clock conditions; the first run of each also dumps the outputs of its last timed step;
# - `bench.py --mode train` and `--mode aligner` once per library;
# - the vocode_batch waveforms of MelGAN and HiFi-GAN V1 on the workload of tools/vocoder_bench.py per library;
# - the dumped outputs and waveforms of A and B compared element by element, and the range of each arm's results.
# Everything goes to <out dir>; the exit code is that of the comparison (0: bit-identical outputs).
set -u
if [ $# -lt 4 ]; then
  echo "usage: $0 <lib A> <lib B> <out dir> <reps> [bench.py arguments...]" >&2
  exit 2
fi
A=$(realpath "$1"); B=$(realpath "$2"); OUT=$(realpath -m "$3"); REPS=$4
shift 4
cd "$(dirname "$0")/.."
mkdir -p "$OUT"
nvidia-smi --query-gpu=name,power.limit,clocks.max.sm --format=csv,noheader > "$OUT/card.txt"
lib_of() { if [ "$1" = A ]; then echo "$A"; else echo "$B"; fi; }
for i in $(seq 1 "$REPS"); do
  for arm in A B; do
    dump=()
    [ "$i" = 1 ] && dump=(--dump-outputs "$OUT/dump_$arm")
    TTSB_LIB=$(lib_of $arm) python bench.py --no-train --no-cpu-baseline "${dump[@]}" "$@" >> "$OUT/infer_$arm.jsonl" 2>> "$OUT/stderr_$arm.log"
  done
done
for mode in train aligner; do
  for arm in A B; do
    TTSB_LIB=$(lib_of $arm) python bench.py --mode $mode --no-cpu-baseline >> "$OUT/${mode}_$arm.jsonl" 2>> "$OUT/stderr_$arm.log"
  done
done
for arm in A B; do
  TTSB_LIB=$(lib_of $arm) python tools/ab_compare.py vocode "$OUT/vocode_$arm" 2>> "$OUT/stderr_$arm.log"
done
python tools/ab_compare.py summary "$OUT" | tee "$OUT/summary.json"
python tools/ab_compare.py compare "$OUT/dump_A" "$OUT/dump_B" | tee "$OUT/compare_dump.txt"
rc=${PIPESTATUS[0]}
python tools/ab_compare.py compare "$OUT/vocode_A" "$OUT/vocode_B" | tee "$OUT/compare_vocode.txt"
[ "${PIPESTATUS[0]}" = 0 ] || rc=1
exit $rc
