"""Generates tests/golden/wgsim_r{1,2}.fq.gz with the REFERENCE'S OWN read simulator: speedseq/src/samtools-1.3.1/misc/wgsim.c
(v0.3.2) compiled from the reference tree (gcc on that one file, an empty config.h on the include path), run on the example reference with
the parameters SURVEY.md §8d names for the bench reads (seed 11, 2 x 150 bp, insert 500 +- 50, 0.5 % errors, 0.1 % mutations of which
15 % indels):  wgsim -S 11 -N 1500 -1 150 -2 150 -d 500 -s 50 -e 0.005 -r 0.001 -R 0.15 -X 0.3 ref.fa r1.fq r2.fq
Read names carry the true fragment coordinates (wgsim.c:390: contig_start_end_e1:s1:i1_e2:s2:i2_id), so mapping accuracy can be scored
without bwa.  Needs a speedseq checkout (its path in SPEEDSEQ_CHECKOUT); the tests only read the fixtures."""
import gzip
import os
import subprocess
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(os.environ["SPEEDSEQ_CHECKOUT"], "src", "samtools-1.3.1")
with tempfile.TemporaryDirectory() as d:
    open(os.path.join(d, "config.h"), "w").close()
    exe = os.path.join(d, "wgsim")
    subprocess.check_call(["gcc", "-O2", "-o", exe, os.path.join(SRC, "misc", "wgsim.c"), "-I" + d, "-I" + os.path.join(SRC, "htslib-1.3.1"), "-lz", "-lm"])
    fa = os.path.join(d, "ex.fa")
    open(fa, "wb").write(gzip.open(os.path.join(HERE, "ex_ref.fa.gz")).read())
    r1, r2 = os.path.join(d, "r1.fq"), os.path.join(d, "r2.fq")
    subprocess.check_call([exe, "-S", "11", "-N", "1500", "-1", "150", "-2", "150", "-d", "500", "-s", "50", "-e", "0.005", "-r", "0.001", "-R", "0.15", "-X", "0.3", fa, r1, r2],
                          stdout=subprocess.DEVNULL, stderr=subprocess.DEVNULL)
    for src, name in ((r1, "wgsim_r1.fq.gz"), (r2, "wgsim_r2.fq.gz")):
        with gzip.GzipFile(os.path.join(HERE, name), "wb", mtime=0) as f:
            f.write(open(src, "rb").read())
        print(name, sum(1 for _ in open(src)) // 4, "reads")
