#!/bin/bash
# Stage what BASELINE config 1 needs from a speedseq checkout (its unmodified bin/speedseq, its sambamba binary, its example data)
# under oracle/_ref/stage — git-ignored, never part of the history — so that tools/run_config1_both.sh and the tests that compare
# with speedseq's own sambamba can run on a machine that has no speedseq checkout.  usage: oracle/stage_config1.sh <speedseq-checkout>
set -e
REF=${1:?usage: oracle/stage_config1.sh <speedseq-checkout>}; ROOT=$(cd "$(dirname "$0")/.." && pwd); S=$ROOT/oracle/_ref/stage
rm -rf "$S"; mkdir -p "$S/bin" "$S/src" "$S/example/data"
cp "$REF/bin/speedseq" "$S/bin/"; cp "$REF/src/sambamba" "$S/src/"
cp "$REF"/example/data/NA12878.20slice.30X.fastq.gz "$REF"/example/data/human_g1k_v37_20_42220611-42542245.fasta "$S/example/data/"
chmod -R u+w "$S"; du -sh "$S"
