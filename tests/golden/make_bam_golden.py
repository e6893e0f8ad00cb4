"""Generates tests/golden/ex_bam_{main,spl,disc}.records.gz: the decompressed, coordinate-sorted BAM RECORDS (everything after the
header and reference table) that speedseq's own tool src/sambamba (v0.5.9) produces with the commands of
speedseq/bin/speedseq:440-448 —  `sambamba view -S -f bam -l 0 /dev/stdin | sambamba sort` — from the oracle's
`bwa mem -p -R RG | samblaster --excludeDups --addMateTags --maxSplitCount 2 --minNonOverlap 20` over tests/golden/ex_reads_2k.fq.gz
(the two side streams go through speedseq's gawk step first: SEQ and QUAL become '*', speedseq:443,446; gawk is not installed here, the
one-line awk program is restated below).  Also writes ex_bam_header.txt: sambamba's rewritten header text.
Needs a speedseq checkout (its path in SPEEDSEQ_CHECKOUT); the tests only read the fixtures."""
import gzip
import os
import struct
import subprocess
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
import ssq_testlib as T

SB = os.path.join(os.environ["SPEEDSEQ_CHECKOUT"], "src", "sambamba")
RG = r"@RG\tID:NA12878\tSM:NA12878\tLB:lib1"


def records(bam_path):
    d = gzip.open(bam_path).read()
    assert d[:4] == b"BAM\x01"
    l_text = struct.unpack("<i", d[4:8])[0]
    text = d[8:8 + l_text]
    p = 8 + l_text
    n_ref = struct.unpack("<i", d[p:p + 4])[0]
    p += 4
    for _ in range(n_ref):
        l = struct.unpack("<i", d[p:p + 4])[0]
        p += 8 + l
    return text, d[p:]


def make(prefix, fa, fq, d, o):
    sam = subprocess.run([T.ORACLE_BIN, "mem", "-t", "4", "-p", "-R", RG, fa, fq], check=True, stdout=subprocess.PIPE, stderr=subprocess.DEVNULL).stdout
    spl, disc = os.path.join(d, "spl.sam"), os.path.join(d, "disc.sam")
    main = subprocess.run([T.ORACLE_BIN, "samblaster", "--excludeDups", "--addMateTags", "--maxSplitCount", "2", "--minNonOverlap", "20", "--splitterFile", spl, "--discordantFile", disc],
                          input=sam, check=True, stdout=subprocess.PIPE, stderr=subprocess.DEVNULL).stdout
    blank = lambda b: b"".join(l if l.startswith(b"@") else b"\t".join(f if i not in (9, 10) else b"*" for i, f in enumerate(l.rstrip(b"\n").split(b"\t"))) + b"\n" for l in b.splitlines(True))
    for tag, text in (("main", main), ("spl", blank(open(spl, "rb").read())), ("disc", blank(open(disc, "rb").read()))):
        unsorted = subprocess.run([SB, "view", "-S", "-f", "bam", "-l", "0", "/dev/stdin"], input=text, check=True, stdout=subprocess.PIPE, stderr=subprocess.DEVNULL).stdout
        out = os.path.join(d, tag + ".bam")
        subprocess.run([SB, "sort", "-t", "2", "-m", "1G", "--tmpdir=" + d, "-o", out, "/dev/stdin"], input=unsorted, check=True, stderr=subprocess.DEVNULL)
        hdr, recs = records(out)
        with gzip.GzipFile(os.path.join(HERE, "%s_bam_%s.records.gz" % (prefix, tag)), "wb", mtime=0) as f:
            f.write(recs)
        if tag == "main" and prefix == "ex":
            open(os.path.join(HERE, "ex_bam_header.txt"), "wb").write(hdr)  # sambamba's rewritten header ...
            open(os.path.join(HERE, "ex_sam_header.txt"), "wb").write(b"".join(l for l in text.splitlines(True) if l.startswith(b"@")))  # ... of this SAM header
        print(prefix, tag, len(recs), "bytes of records")


with tempfile.TemporaryDirectory() as d:
    o = T.Oracle()
    fa = os.path.join(d, "ex.fa")
    open(fa, "wb").write(gzip.open(os.path.join(T.GOLDEN, "ex_ref.fa.gz")).read())
    o.index_build(fa)
    make("ex", fa, os.path.join(T.GOLDEN, "ex_reads_2k.fq.gz"), d, o)
    # a seeded synthetic stress set: 3 contigs, duplicates, chimeric reads (SA tags, splitters), junk pairs, orphans, improper pairs, XA hits
    from test_hostsim_pipe import stress_reads
    g, bounds = T.synth_genome(400000, 7, n_contigs=3)
    fa2 = os.path.join(d, "syn.fa")
    T.write_fasta(fa2, g, bounds)
    o.index_build(fa2)
    names, seqs, quals = stress_reads(g, bounds, 700, 150, 5, err=0.01, indel=0.002)
    fq2 = os.path.join(d, "syn.fq")
    T.write_fastq(fq2, names, seqs, quals)
    make("syn", fa2, fq2, d, o)
    # the same reads as a run of three batches (`bwa mem -t 1` closes a batch at 10 Mbp; here the cuts are made explicitly through the oracle's
    # library entry so that the fixture stays small): per-batch insert-size statistics, duplicates across batches, one global coordinate sort
    idx = o.load(fa2)
    cuts = [0, 1000, 2100, len(names)]
    body = "".join(o.mem_pe(idx, names[a:b], seqs[a:b], quals[a:b], a, 4, b"NA12878") for a, b in zip(cuts, cuts[1:]))
    hdr = "@SQ\tSN:ctg1\tLN:%d\n@SQ\tSN:ctg2\tLN:%d\n@SQ\tSN:ctg3\tLN:%d\n" % tuple(int(bounds[i + 1] - bounds[i]) for i in range(3))
    main = subprocess.run([T.ORACLE_BIN, "samblaster", "--excludeDups", "--addMateTags", "--maxSplitCount", "2", "--minNonOverlap", "20"], input=(hdr + body).encode(), check=True,
                          stdout=subprocess.PIPE, stderr=subprocess.DEVNULL).stdout
    unsorted = subprocess.run([SB, "view", "-S", "-f", "bam", "-l", "0", "/dev/stdin"], input=main, check=True, stdout=subprocess.PIPE, stderr=subprocess.DEVNULL).stdout
    out = os.path.join(d, "syn3.bam")
    subprocess.run([SB, "sort", "-t", "2", "-m", "1G", "--tmpdir=" + d, "-o", out, "/dev/stdin"], input=unsorted, check=True, stderr=subprocess.DEVNULL)
    with gzip.GzipFile(os.path.join(HERE, "syn3_bam_main.records.gz"), "wb", mtime=0) as f:
        f.write(records(out)[1])
    print("syn3 main (3 batches)", len(records(out)[1]), "bytes of records")
