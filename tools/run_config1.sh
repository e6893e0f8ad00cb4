#!/bin/bash
# BASELINE config 1: the reference's own example (`example/run_speedseq.sh` step 1) through the UNMODIFIED bin/speedseq with a
# private config.  usage: tools/run_config1.sh <oracle|b200|b200_fused|b200_bam|b200_bamz|b200_view> <reference-checkout> <workdir>
#   oracle     : $BWA/$SAMBLASTER = oracle/ssqo (CPU)
#   b200       : $BWA/$SAMBLASTER = speedseq_b200/bin/{bwa,samblaster} (needs an H100; the reference checkout may be the staged one
#                of oracle/stage_config1.sh)
#   b200_fused : + the config stanza of INTEGRATION.md §2: samblaster's stage runs on the device inside `bwa mem`
#   b200_bam   : + SSQ_FUSE_BAM and $SAMBAMBA = speedseq_b200/bin/sambamba: the main records never exist as text
#   b200_bamz  : b200_bam + SSQ_BGZF_GPU=1: the shim's sort compresses the sorted BAM on the device
#   b200_view  : the default unfused shims, $SAMBAMBA = speedseq_b200/bin/sambamba with SSQ_SAM2BAM_GPU=1: every `view -S` (main and
#                both side streams) converts its SAM on the device into sorted runs for the shim's sort; `index` runs on the device too
set -e
MODE=${1:-oracle}; REF=${2:?usage: tools/run_config1.sh MODE SPEEDSEQ_CHECKOUT [WORKDIR]}; W=${3:-/tmp/ssq_config1}
ROOT=$(cd "$(dirname "$0")/.." && pwd)
mkdir -p "$W/bin"; cd "$W"
if [ "${MODE#b200}" != "$MODE" ]; then BWA=$ROOT/speedseq_b200/bin/bwa; SB=$ROOT/speedseq_b200/bin/samblaster
else printf '#!/bin/bash\nexec %s "$@"\n' "$ROOT/oracle/ssqo" > bin/bwa; chmod +x bin/bwa; ln -sf "$ROOT/oracle/ssqo" bin/samblaster; BWA=$W/bin/bwa; SB=$W/bin/samblaster; fi
command -v parallel >/dev/null || { cat > bin/parallel <<'P'
#!/bin/bash
while [ $# -gt 0 ]; do case "$1" in -j) shift 2;; *) shift;; esac; done
pids=(); rc=0
while IFS= read -r cmd; do [ -z "$cmd" ] && continue; bash -c "$cmd" & pids+=($!); done
for p in "${pids[@]}"; do wait $p || rc=$((rc+1)); done
exit $rc
P
chmod +x bin/parallel; }
command -v gawk >/dev/null || { printf '#!/bin/bash\nexec awk "$@"\n' > bin/gawk; chmod +x bin/gawk; }
export PATH=$W/bin:$PATH
cat > speedseq.b200.config <<C
SPEEDSEQ_HOME=$W
SAMBAMBA=$REF/src/sambamba
PARALLEL=$(command -v parallel)
BWA=$BWA
SAMBLASTER=$SB
C
if [ "$MODE" = b200_fused ] || [ "$MODE" = b200_bam ] || [ "$MODE" = b200_bamz ]; then cat >> speedseq.b200.config <<'C'
if [ -z "${REALIGN_RG_LIST+x}" ]; then
    export SSQ_FUSE_SAMBLASTER="$INCLUDE_DUPS --addMateTags --maxSplitCount $MAX_SPLIT_COUNT --minNonOverlap $MIN_NON_OVERLAP"
fi
C
fi
if [ "$MODE" = b200_bam ] || [ "$MODE" = b200_bamz ]; then cat >> speedseq.b200.config <<C
export SSQ_FUSE_BAM=1
export SSQ_SAMBAMBA_REAL=$REF/src/sambamba
SAMBAMBA=$ROOT/speedseq_b200/bin/sambamba
C
fi
[ "$MODE" = b200_bamz ] && echo "export SSQ_BGZF_GPU=1" >> speedseq.b200.config
if [ "$MODE" = b200_view ]; then cat >> speedseq.b200.config <<C
export SSQ_SAM2BAM_GPU=1
export SSQ_SAMBAMBA_REAL=$REF/src/sambamba
SAMBAMBA=$ROOT/speedseq_b200/bin/sambamba
C
fi
cp "$REF/example/data/human_g1k_v37_20_42220611-42542245.fasta" ref.fa
bash "$REF/bin/speedseq" align -o example -M 3 -p -t 4 -K "$W/speedseq.b200.config" -R "@RG\tID:NA12878\tSM:NA12878\tLB:lib1" ref.fa "$REF/example/data/NA12878.20slice.30X.fastq.gz"
for f in example.bam example.splitters.bam example.discordants.bam; do echo "$f $("$REF/src/sambamba" view -c $f) records"; done
