"""Generates the merge fixtures: small coordinate-sorted BAM inputs written here with Python's zlib (the BAM writers of
make_bai_golden.py) and what speedseq's own tool src/sambamba (v0.5.9) makes of them: `sambamba merge out.bam in1.bam ...` (the
call of speedseq/bin/speedseq:2002-2009) in several argument orders, and `sambamba merge -H`.  Per case and order:
  merge_<case>_<order>.records.gz   the merged file's records, decompressed
  merge_<case>_<order>.header.txt   its header text
  merge_<case>_<order>.H.txt        what `merge -H` prints
Inputs: merge_<case>_<k>.bam; an order names its inputs by k, in argument order.  Cases:
  ties      the three inputs of the order rule (x = 4 x 10, 1 x 20, 3 x 30; y = 4 x 10, 3 x 30; z = 1 x 5, 4 x 10, 3 x 30; all
            forward on one reference), in the orders xyz, zyx and yxz
  many      8 inputs with many equal keys over two references and unmapped tails; 2, 3 and 8 of them in several orders
  holes     inputs without records (one with its EOF block, one without it and its header spread over tiny members) and one
            with a single record, among inputs with equal keys
  unmapped  unmapped records placed at their mate's position, and tails without a reference, in every input
  bigrec    3000-byte members, so records cross member borders, and a record larger than a member
  ids       more than 16 distinct @RG and @PG IDs (the hash table grows), an identical @PG line in every input, @CO lines (two
            identical), tags out of sambamba's order
  hd14      inputs whose @HD says VN:1.4
Needs a speedseq checkout (its path in SPEEDSEQ_CHECKOUT); the tests only read the fixtures."""
import gzip
import os
import random
import struct
import subprocess
import tempfile

try:
    from make_bai_golden import bgzf, member, record
except ImportError:  # imported by the tests as golden.make_merge_golden
    from golden.make_bai_golden import bgzf, member, record

HERE = os.path.dirname(os.path.abspath(__file__))
REFS = [("m1", 5000000), ("m2", 300000)]
HD = b"@HD\tVN:1.3\tSO:coordinate\n"


def bam_header(text, refs=REFS):
    text = text + b"".join(b"@SQ\tSN:%s\tLN:%d\n" % (n.encode(), l) for n, l in refs) if b"@SQ" not in text else text
    h = b"BAM\1" + struct.pack("<i", len(text)) + text + struct.pack("<i", len(refs))
    return h + b"".join(struct.pack("<i", len(n) + 1) + n.encode() + b"\0" + struct.pack("<i", l) for n, l in refs)


def sq():
    return b"".join(b"@SQ\tSN:%s\tLN:%d\n" % (n.encode(), l) for n, l in REFS)


def sort_key(r):
    ref, pos = struct.unpack_from("<ii", r, 4)
    return (1 << 40 if ref < 0 else ref << 32 | pos + 1)


def bam(recs, text=None, size=0xff00, eof=True):
    recs = sorted(recs, key=sort_key)  # stable: equal keys keep their order
    return bgzf(bam_header(text if text is not None else HD + sq()) + b"".join(recs), size, eof)


def cases():
    """{case: ([input bytes], [orders])}"""
    out = {}
    x = [record("x%d" % i, 0, 0, p) for i, p in enumerate([10] * 4 + [20] + [30] * 3)]
    y = [record("y%d" % i, 0, 0, p) for i, p in enumerate([10] * 4 + [30] * 3)]
    z = [record("z%d" % i, 0, 0, p) for i, p in enumerate([5] + [10] * 4 + [30] * 3)]
    out["ties"] = ([bam(x), bam(y), bam(z)], ["012", "210", "102"])
    R = random.Random(5)
    many = []
    for k in range(8):
        recs = []
        for i in range(R.randint(20, 60)):
            ref = R.choice([0, 0, 1])
            recs.append(record("k%d_%d" % (k, i), R.choice([0, 16, 99, 147]), ref, R.choice([100, 100, 250, 4000, 4000, 4001, 70000])))
        recs += [record("k%d_u%d" % (k, i), 77, -1, -1, "*") for i in range(R.randint(0, 4))]
        many.append(bam(recs))
    out["many"] = (many, ["01234567", "76543210", "31570246", "05", "50", "257", "614"])
    a = [record("a%d" % i, 0, 0, p) for i, p in enumerate([7, 7, 9, 9, 9])]
    b = [record("b%d" % i, 0, 0, p) for i, p in enumerate([7, 9, 9])]
    s = [record("s0", 0, 0, 9)]
    hdr_only_split = b"".join(member(c) for c in (lambda t: [t[i:i + 11] for i in range(0, len(t), 11)])(bam_header(HD + b"@CO\tsplit header\n" + sq())))
    out["holes"] = ([bam(a), bam([]), bam(s), hdr_only_split, bam(b)], ["01234", "31024", "02143", "0124"])
    un = []
    for k in range(3):
        recs = [record("p%d_%d" % (k, i), 99, 0, 1000 * i + 5 * k) for i in range(6)]
        recs += [record("p%d_m%d" % (k, i), 133 | 8 * 0, 0, 1000 * i + 5 * k, "*") for i in range(0, 6, 2)]  # unmapped, placed at the mate
        recs += [record("p%d_c2_%d" % (k, i), 0, 1, 200 * i) for i in range(3)]
        recs += [record("p%d_n%d" % (k, i), 77 if i % 2 else 141, -1, -1, "*") for i in range(2 + k)]
        un.append(bam(recs))
    out["unmapped"] = (un, ["012", "210"])
    big0 = [record("g0_%d" % i, 0, 0, 37 * i) for i in range(150)] + [record("huge", 0, 0, 2000, "30000M")]
    big1 = [record("g1_%d" % i, 16, 0, 41 * i) for i in range(150)]
    out["bigrec"] = ([bam(big0, size=3000), bam(big1, size=3000), bam(big0[::3], size=1500)], ["01", "10", "021"])
    ids = []
    for k in range(3):
        t = HD + sq()
        for i in range(9):
            t += b"@RG\tSM:s%d\tID:rg%d_%d\tLB:lib%d\n" % (k, k, i, i % 2)
        t += b"@PG\tID:bwa\tPN:bwa\tVN:0.7.10\tCL:bwa mem ref.fa\n"
        for i in range(7):
            t += b"@PG\tVN:%d\tID:prog%d.%d\tPN:p\n" % (i, k, i)
        t += b"@CO\tcomment of file %d\n@CO\tthe same comment\n" % k
        ids.append(bam([record("i%d_%d" % (k, i), 0, 0, 3 * i + k) for i in range(10)], t))
    out["ids"] = (ids, ["012", "201"])
    hd = b"@HD\tVN:1.4\tSO:coordinate\n"
    out["hd14"] = ([bam([record("h0", 0, 0, 5)], hd + sq()), bam([record("h1", 0, 0, 5)], hd + sq())], ["01", "10"])
    return out


def body(path):
    d = gzip.open(path).read()
    lt = struct.unpack_from("<i", d, 4)[0]
    at = 8 + lt
    n_ref = struct.unpack_from("<i", d, at)[0]
    at += 4
    for _ in range(n_ref):
        at += 8 + struct.unpack_from("<i", d, at)[0]
    return d[8:8 + lt].split(b"\0")[0], d[at:]


def main():
    sb = os.path.join(os.environ["SPEEDSEQ_CHECKOUT"], "src", "sambamba")
    with tempfile.TemporaryDirectory() as d:
        for name, (inputs, orders) in cases().items():
            paths = []
            for k, data in enumerate(inputs):
                p = os.path.join(HERE, "merge_%s_%d.bam" % (name, k))
                open(p, "wb").write(data)
                paths.append(p)
            for o in orders:
                args = [paths[int(c)] for c in o]
                out = os.path.join(d, "out.bam")
                for f in (out, out + ".bai"):
                    if os.path.exists(f):
                        os.unlink(f)
                subprocess.run([sb, "merge", out] + args, check=True)
                h = subprocess.run([sb, "merge", "-H", out] + args, check=True, stdout=subprocess.PIPE).stdout
                text, recs = body(out)
                base = os.path.join(HERE, "merge_%s_%s" % (name, o))
                open(base + ".header.txt", "wb").write(text)
                open(base + ".H.txt", "wb").write(h)
                with gzip.GzipFile(base + ".records.gz", "wb", mtime=0) as g:
                    g.write(recs)
                print(name, o, len(recs))


if __name__ == "__main__":
    main()
