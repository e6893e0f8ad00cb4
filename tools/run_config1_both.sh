#!/bin/bash
# BASELINE config 1 four ways through the UNMODIFIED bin/speedseq: oracle CLI (CPU), the GPU shims, the GPU shims with the fused
# samblaster stage, those with the main records as BAM runs into the `sambamba` shim, and those with the sorted BAM compressed on the device; then the three BAMs of each GPU run against
# the oracle run's: records (sambamba view) and header minus the @PG
# lines (they carry executable paths) must be identical, and each BAM's .bai must be the staged sambamba's index of that BAM.  usage: tools/run_config1_both.sh [staged-reference] [workdir]
ROOT=$(cd "$(dirname "$0")/.." && pwd); REF=${1:-$ROOT/oracle/_ref/stage}; W=${2:-/tmp/ssq_config1}
REF=$(cd "$REF" && pwd); SB=$REF/src/sambamba; rc=0
run() { local t0=$(date +%s%N); timeout ${SSQ_C1_TIMEOUT:-150} bash "$ROOT/tools/run_config1.sh" "$1" "$REF" "$W/$2" > "$W/$2.log" 2>&1 || { echo "$2: FAILED"; tail -5 "$W/$2.log"; rc=1; }; echo "$2: $(( ($(date +%s%N) - t0) / 1000000 )) ms wall"; }
mkdir -p "$W"
run oracle oracle
MODES=${SSQ_C1_MODES:-b200 b200_fused b200_bam b200_bamz}
for m in $MODES; do run $m $m; done
for m in $MODES; do for f in example.bam example.splitters.bam example.discordants.bam; do
	a=$("$SB" view "$W/oracle/$f" | md5sum | cut -d' ' -f1); b=$("$SB" view "$W/$m/$f" | md5sum | cut -d' ' -f1)
	ha=$("$SB" view -H "$W/oracle/$f" | grep -v '^@PG' | md5sum | cut -d' ' -f1); hb=$("$SB" view -H "$W/$m/$f" | grep -v '^@PG' | md5sum | cut -d' ' -f1)
	n=$("$SB" view -c "$W/$m/$f")
	if [ -n "$n" ] && [ "$n" -gt 0 ] && [ "$a" = "$b" ] && [ "$ha" = "$hb" ]; then echo "$m/$f: $n records, identical to the oracle run ($a)"; else echo "$m/$f: DIFFERS"; rc=1; fi
	# the .bai the run wrote (speedseq:486-494) against the staged sambamba's index of the same BAM (a fresh file: sambamba 0.5.9
	# does not truncate an existing one)
	mkdir -p "$W/bai_check"; rm -f "$W/bai_check/x.bam" "$W/bai_check/x.bam.bai"; cp "$W/$m/$f" "$W/bai_check/x.bam"
	if "$SB" index "$W/bai_check/x.bam" 2>/dev/null && cmp -s "$W/$m/$f.bai" "$W/bai_check/x.bam.bai"; then echo "$m/$f.bai: identical to sambamba's index"; else echo "$m/$f.bai: DIFFERS from sambamba's index"; rc=1; fi
done; done
exit $rc
