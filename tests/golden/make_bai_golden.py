"""Generates the BAI fixtures: small coordinate-sorted BAM files written here with Python's zlib (BGZF member sizes chosen on
purpose) and the index speedseq's own tool src/sambamba (v0.5.9) writes for each (`sambamba index x.bam` -> x.bam.bai), the call
of speedseq/bin/speedseq:486-494.  Also the syn / syn3 record goldens (syn_bam_main.records.gz, syn3_bam_main.records.gz) put
through `sambamba sort -o`, which writes the sorted BAM and its .bai.  Fixtures (tests/golden/bai_*.bam and .bam.bai):
  bai_refs       several references, two of them empty (one between, one at the end); unmapped reads placed at their mate's
                 position; unmapped reads without coordinates at the end; records across 16 KB windows; CIGARs with long N / D
                 ops that reach the upper bin levels; a stored bin that disagrees with the CIGAR; a mapped record with no
                 reference-consuming op; 3000-byte members, so records cross member borders
  bai_bigrec     a record larger than a BGZF member (about 150 KB), between ordinary ones; 0xff00-byte members
  bai_bins       some 2000 records over 100 Mb of one reference: several hundred bins, so the bin order is that of sambamba's
                 hash table after several resizes; 0xff00-byte members, and chunks merged within a block
  bai_noeof      a file without the empty EOF member: offsets at the end of the text are the file's length
  bai_header     a header-only BAM
  bai_pos0       records of reference length 0 (soft clips only, CIGAR `*`) first in their references: at position 0 (window 0,
                 from sambamba's truncating division), at 16384 (no window) and at 16390 (its own window)
  bai_syn, bai_syn3  the syn / syn3 records, sorted by sambamba itself
Needs a speedseq checkout (its path in SPEEDSEQ_CHECKOUT); the tests only read the fixtures."""
import gzip
import os
import random
import re
import struct
import subprocess
import tempfile
import zlib

HERE = os.path.dirname(os.path.abspath(__file__))
OPS = "MIDNSHP=X"


def reg2bin(beg, end):
    end -= 1
    for shift, base in ((14, 4681), (17, 585), (20, 73), (23, 9), (26, 1)):
        if beg >> shift == end >> shift:
            return base + (beg >> shift)
    return 0


def record(name, flag, ref, pos, cigar="10M", seqlen=None, bin=None, mapq=60):
    c = [(int(n), OPS.index(o)) for n, o in re.findall(r"(\d+)([MIDNSHP=X])", cigar)]
    rl = sum(n for n, o in c if o in (0, 2, 3, 7, 8))
    if seqlen is None:
        seqlen = sum(n for n, o in c if o in (0, 1, 4, 7, 8))
    if bin is None:
        bin = reg2bin(pos, pos + (rl if rl and not flag & 4 else 1)) if pos >= 0 else 4680
    nm = name.encode() + b"\0"
    body = struct.pack("<iiBBHHHiiii", ref, pos, len(nm), mapq, bin, len(c), flag, seqlen, -1, -1, 0)
    body += nm + b"".join(struct.pack("<I", n << 4 | o) for n, o in c) + bytes((seqlen + 1) // 2) + b"\xff" * seqlen
    return struct.pack("<i", len(body)) + body


def header(refs):
    text = b"@HD\tVN:1.3\tSO:coordinate\n" + b"".join(b"@SQ\tSN:%s\tLN:%d\n" % (n.encode(), l) for n, l in refs)
    h = b"BAM\1" + struct.pack("<i", len(text)) + text + struct.pack("<i", len(refs))
    return h + b"".join(struct.pack("<i", len(n) + 1) + n.encode() + b"\0" + struct.pack("<i", l) for n, l in refs)


def member(data):
    co = zlib.compressobj(6, zlib.DEFLATED, -15)
    d = co.compress(data) + co.flush()
    return b"\x1f\x8b\x08\x04\0\0\0\0\0\xff\x06\0BC\x02\0" + struct.pack("<H", 25 + len(d)) + d + struct.pack("<II", zlib.crc32(data), len(data))


def bgzf(text, size, eof=True):
    pts = list(range(0, len(text), size)) + [len(text)]
    return b"".join(member(text[a:b]) for a, b in zip(pts, pts[1:])) + (member(b"") if eof else b"")


def corpus():
    out = {}
    refs = [("chr1", 249250621), ("chrE", 1000), ("chr2", 243199373), ("chr3", 198022430), ("chrZ", 5000)]
    recs = [record("a0", 99, 0, 10), record("a1", 0, 0, 16380, "20M"), record("u_placed", 133, 0, 16390, "*"),  # placed at its mate
            record("a2", 0, 0, 16400, "50M300000N50M"), record("a3", 16, 0, 20000, "10M40000D10M"),
            record("wrongbin", 0, 0, 30000, "30M", bin=4700), record("softonly", 0, 0, 32768, "8S"),
            record("a4", 0, 0, 32770, "5M9000000N5M"), record("a5", 0, 0, 140000, "100M"), record("a6", 0, 0, 140001, "100M2000000D1M")]
    for k in range(60):
        recs.append(record("w%d" % k, 0 if k % 3 else 16, 0, 150000 + 9000 * k, "%dM" % (50 + k)))
    recs += [record("c2_%d" % k, 0, 2, 5000 * k + 7, "36M") for k in range(40)]
    recs += [record("c2_unm", 69, 2, 300000, "*"), record("c2_end", 0, 2, 300010, "60M70000000N60M")]
    recs += [record("c3_only_unmapped", 4, 3, 123456, "*")]
    recs += [record("nocoor%d" % k, 77 if k % 2 else 141, -1, -1, "*") for k in range(5)]
    out["bai_refs"] = bgzf(header(refs) + b"".join(recs), 3000)
    big = [record("b0", 0, 0, 100), record("big", 0, 0, 200, "100000M"), record("b1", 0, 0, 300), record("b2", 0, 0, 70000)]
    out["bai_bigrec"] = bgzf(header(refs[:1]) + b"".join(big), 0xff00)
    R = random.Random(11)
    recs = []
    for p in sorted(R.randrange(0, 100000000) for _ in range(2000)):
        k = R.random()
        cg = "20M%dN20M" % R.choice([100, 20000, 300000, 3000000]) if k < 0.2 else "%dM" % R.randint(20, 150)
        recs.append(record("r%d" % p, 4 | 1 if k > 0.95 else 0, 0, p, "*" if k > 0.95 else cg))
    out["bai_bins"] = bgzf(header(refs[:1]) + b"".join(recs), 0xff00)
    out["bai_noeof"] = bgzf(header(refs[:2]) + record("n0", 0, 0, 5) + record("n1", 0, 1, 7), 0xff00, eof=False)
    out["bai_header"] = bgzf(header(refs), 0xff00)
    out["bai_pos0"] = bgzf(header(refs[:4]) + record("s", 0, 0, 0, "8S") + record("b", 0, 0, 10) + record("t", 0, 1, 0, "*", seqlen=4) +
                           record("c", 0, 1, 40000) + record("u", 0, 2, 16384, "5S") + record("d", 0, 2, 16500) +
                           record("v", 0, 3, 16390, "3S") + record("e", 0, 3, 16400), 0xff00)
    return out


def records_bam(records_gz, n_ref):
    refs = [("syn%d" % i, 2 ** 29 - 1) for i in range(n_ref)]
    return bgzf(header(refs) + gzip.open(records_gz).read(), 0xff00)


def main():
    sb = os.path.join(os.environ["SPEEDSEQ_CHECKOUT"], "src", "sambamba")
    with tempfile.TemporaryDirectory() as d:
        for name, data in corpus().items():
            p = os.path.join(HERE, name + ".bam")
            open(p, "wb").write(data)
            if os.path.exists(p + ".bai"):  # sambamba 0.5.9 does not truncate an existing output: a longer old index keeps its tail
                os.unlink(p + ".bai")
            subprocess.run([sb, "index", p, p + ".bai"], check=True)
            print(name, len(data), os.path.getsize(p + ".bai"))
        for name in ("syn", "syn3"):
            rec = gzip.open(os.path.join(HERE, name + "_bam_main.records.gz")).read()
            n_ref, at = 0, 0
            while at < len(rec):  # the references the records name
                n_ref = max(n_ref, struct.unpack_from("<i", rec, at + 4)[0] + 1)
                at += 4 + struct.unpack_from("<i", rec, at)[0]
            src = os.path.join(d, name + ".bam")
            open(src, "wb").write(records_bam(os.path.join(HERE, name + "_bam_main.records.gz"), n_ref))
            p = os.path.join(HERE, "bai_%s.bam" % name)
            for f in (p, p + ".bai"):
                if os.path.exists(f):
                    os.unlink(f)
            subprocess.run([sb, "sort", "-o", p, src], check=True)
            print("bai_" + name, os.path.getsize(p), os.path.getsize(p + ".bai"))


if __name__ == "__main__":
    main()
