"""The product's `bwa mem` path (ssq_mem_batch_sam + the CLI shims speedseq_b200/bin/{bwa,samblaster}) against the oracle:
SAM records, dup flags, MC/MQ tags, discordant and splitter streams must be identical byte for byte (everything except
the @PG header lines, which carry program paths)."""
import ctypes as C
import gzip
import os
import subprocess

import numpy as np
import pytest

import ssq_testlib as T

pytestmark = pytest.mark.gpu
BWA = os.path.join(T.ROOT, "speedseq_b200", "bin", "bwa")
SAMBLASTER = os.path.join(T.ROOT, "speedseq_b200", "bin", "samblaster")
RG = r"@RG\tID:NA12878\tSM:NA12878\tLB:lib1"


def _strip_pg(b):
    return b"".join(l for l in b.splitlines(True) if not l.startswith(b"@PG"))


def _mem_batch(ssq, idx, names, seqs, quals, n_processed, paired, rg):
    n = len(names)
    arr = lambda xs: (C.c_char_p * n)(*[x.encode() for x in xs])
    out, ln = C.c_char_p(), C.c_size_t(0)
    rc = ssq.lib.ssq_mem_batch_sam(idx, ssq.opts, C.c_int(n), arr(names), arr(seqs), arr(quals), None, C.c_int64(n_processed), C.c_int(paired), None, rg, C.c_int(0),
                                   C.byref(out), C.byref(ln), None)
    ssq.ck(rc, "ssq_mem_batch_sam")
    s = C.string_at(out, ln.value).decode()
    ssq.lib.ssq_free(out)
    return s


def test_mem_batch_sam_example_reads(ssq, oracle, ex_index, ex_reads):
    idx = oracle.load(ex_index)
    h = ssq.index_load(ex_index)
    names, seqs, quals = ex_reads
    a = oracle.mem_pe(idx, names, seqs, quals, 0, 8, b"NA12878")
    b = _mem_batch(ssq, h, names, seqs, quals, 0, 1, b"NA12878")
    assert a == b
    ssq.index_free(h)


@pytest.mark.parametrize("rl,seed,kw", [(75, 1, {}), (150, 2, dict(err=0.02, indel=0.004, n_frac=0.004)), (250, 3, dict(err=0.01, indel=0.003)), (101, 4, dict(ins_mean=250, ins_sd=80))])
def test_mem_batch_sam_synthetic_stress(ssq, oracle, syn_index, rl, seed, kw):
    fa, g, bounds = syn_index
    idx = oracle.load(fa)
    h = ssq.index_load(fa)
    names, seqs, quals = T.simulate_pairs(g, bounds, 1200, rl, seed, **kw)
    rng = np.random.default_rng(seed)
    for k in range(0, len(seqs), 40):   # unmappable mates: orphans / mate rescue
        seqs[k + 1] = "".join("ACGT"[x] for x in rng.integers(0, 4, rl))
    for k in range(10, len(seqs), 50):  # chimeric reads: supplementary lines, SA tags, splitters
        seqs[k] = seqs[k][: rl // 2] + seqs[(k + 200) % len(seqs)][rl // 2:]
    a = oracle.mem_pe(idx, names, seqs, quals, 1000, 8, b"rg1")
    b = _mem_batch(ssq, h, names, seqs, quals, 1000, 1, b"rg1")
    assert a == b
    ssq.index_free(h)


def test_cli_pipeline_matches_oracle_cli(ssq, tmp_path):
    """config 1 in miniature: bwa index + bwa mem -p | samblaster with FIFOs, product shims vs oracle CLI"""
    assert os.path.exists(BWA) and os.path.exists(SAMBLASTER), "run `make -C speedseq_b200/csrc cli`"
    fq = os.path.join(T.GOLDEN, "ex_reads_2k.fq.gz")
    outs = {}
    for tag, bwa, sb in (("oracle", [T.ORACLE_BIN], [T.ORACLE_BIN, "samblaster"]), ("b200", [BWA], [SAMBLASTER])):
        d = tmp_path / tag
        d.mkdir()
        fa = str(d / "ex.fa")
        open(fa, "wb").write(gzip.open(os.path.join(T.GOLDEN, "ex_ref.fa.gz")).read())
        subprocess.check_call(bwa + ["index", fa], stderr=subprocess.DEVNULL)
        sam = subprocess.run(bwa + ["mem", "-t", "2", "-p", "-R", RG, fa, fq], check=True, stdout=subprocess.PIPE, stderr=subprocess.DEVNULL).stdout
        spl, disc = str(d / "spl.sam"), str(d / "disc.sam")
        out = subprocess.run(sb + ["--excludeDups", "--addMateTags", "--maxSplitCount", "2", "--minNonOverlap", "20", "--splitterFile", spl, "--discordantFile", disc],
                             input=sam, check=True, stdout=subprocess.PIPE, stderr=subprocess.DEVNULL).stdout
        outs[tag] = (sam, out, open(spl, "rb").read(), open(disc, "rb").read(), [open(fa + "." + e, "rb").read() for e in ("amb", "ann", "pac", "bwt", "sa")])
    for i, what in enumerate(("bwa mem SAM", "samblaster SAM", "splitters", "discordants")):
        assert _strip_pg(outs["oracle"][i]) == _strip_pg(outs["b200"][i]), what
    assert outs["oracle"][4] == outs["b200"][4]
    assert outs["b200"][1].count(b"\n") > 4000


def test_samblaster_shim_dups_across_chunks(ssq, oracle, ex_index, ex_reads, tmp_path):
    """duplicates whose first occurrence lies many records earlier; also exercises ssq_dupset_mark across several calls"""
    idx = oracle.load(ex_index)
    names, seqs, quals = ex_reads
    names = names + ["dup_" + n for n in names[:1000]]
    seqs = seqs + seqs[:1000]
    quals = quals + quals[:1000]
    body = oracle.mem_pe(idx, names, seqs, quals, 0, 8, b"")
    sam = ("@SQ\tSN:20_slice\tLN:321635\n" + body).encode()
    res = {}
    for tag, cmd in (("oracle", [T.ORACLE_BIN, "samblaster"]), ("b200", [SAMBLASTER])):
        res[tag] = subprocess.run(cmd + ["--addMateTags"], input=sam, check=True, stdout=subprocess.PIPE, stderr=subprocess.DEVNULL).stdout
    assert _strip_pg(res["oracle"]) == _strip_pg(res["b200"])
    assert res["b200"].count(b"\t1187\t") + res["b200"].count(b"\t1171\t") > 100  # flagged duplicates exist


def test_dupset_streaming_equals_one_shot(ssq, oracle):
    rng = np.random.default_rng(3)
    n = 60000
    sig = np.zeros(n, T.DUPSIG_DT)
    sig["pos1"] = rng.integers(0, 3000, n); sig["pos2"] = sig["pos1"] + rng.integers(0, 40, n)
    sig["strand1"] = rng.integers(0, 2, n); sig["strand2"] = rng.integers(0, 2, n); sig["valid"] = rng.random(n) > 0.03
    ref = oracle.dupmark(sig)
    h = C.c_void_p()
    ssq.ck(ssq.lib.ssq_dupset_create(0, C.byref(h)), "ssq_dupset_create")
    got = np.zeros(n, np.uint8)
    for lo in range(0, n, 7001):
        part = sig[lo:lo + 7001].copy()
        d = np.zeros(len(part), np.uint8)
        ssq.ck(ssq.lib.ssq_dupset_mark(h, C.c_uint64(len(part)), part.ctypes.data_as(C.c_void_p), d.ctypes.data_as(C.c_void_p)), "ssq_dupset_mark")
        got[lo:lo + 7001] = d
    ssq.lib.ssq_dupset_size.restype = C.c_uint64
    assert np.array_equal(got, ref)
    assert int(ssq.lib.ssq_dupset_size(h)) == int(((ref == 0) & (sig["valid"] == 1)).sum())
    ssq.lib.ssq_dupset_free(h)


# ------------------------------------------------------------------------------------------------------------------------------
# the invocation modes of speedseq/bin/speedseq that one interleaved single-batch run does not reach: two FASTQ files
# (:468, the default), -I (:286), -C (:1961), several batches (per-batch insert-size statistics + global read ordinals), smart
# pairing with unpaired reads, gz input, and the fused samblaster stage behind the same two executables
def _records(b):
    return b"".join(l for l in b.splitlines(True) if not l.startswith(b"@"))


def _both(args, stdin=None):
    return [subprocess.run(exe + args, input=stdin, check=True, stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, timeout=300).stdout for exe in ([T.ORACLE_BIN], [BWA])]


@pytest.fixture(scope="module")
def cli_ref(tmp_path_factory):
    d = tmp_path_factory.mktemp("cliref")
    g, bounds = T.synth_genome(600000, 31, n_contigs=4)
    fa = str(d / "ref.fa")
    T.write_fasta(fa, g, bounds)
    subprocess.check_call([BWA, "index", fa], stderr=subprocess.DEVNULL)
    return d, fa, g, bounds


def test_cli_two_files_insert_override_and_comments(ssq, cli_ref):
    from test_hostsim_pipe import stress_reads
    d, fa, g, bounds = cli_ref
    names, seqs, quals = stress_reads(g, bounds, 1500, 150, 3)
    fq1, fq2 = str(d / "r1.fq.gz"), str(d / "r2.fq")
    with gzip.open(fq1, "wt") as f1, open(fq2, "w") as f2:
        for i, (n, s, q) in enumerate(zip(names, seqs, quals)):
            (f2 if i & 1 else f1).write("@%s/%d BC:Z:x%d\n%s\n+\n%s\n" % (n, 1 + (i & 1), i % 5, s, q))
    for extra in ([], ["-I", "300,30"], ["-C"], ["-I", "420,60,900,50", "-C"]):
        a, b = _both(["mem", "-t", "3", "-R", RG] + extra + [fa, fq1, fq2])
        assert _records(a) == _records(b), extra
        assert _records(b).count(b"\n") >= 3000
        assert (b"BC:Z:x" in b) == ("-C" in extra)


def test_cli_several_batches_and_smart_pairing(ssq, cli_ref):
    """-t 1: a batch closes at 10 Mbp (67 k reads of 150 bp), so 150 k reads make three batches — each with its own insert-size
    statistics, read ordinals continuing across them; the interleaved file also holds unpaired reads (smart pairing)"""
    d, fa, g, bounds = cli_ref
    names, seqs, quals = T.simulate_pairs(g, bounds, 75000, 150, 5)
    fq = str(d / "big.fq")
    with open(fq, "w") as f:
        for i, (n, s, q) in enumerate(zip(names, seqs, quals)):
            if i % 9001 == 17:  # drop one end now and then: its mate becomes a single-end read in the middle of the stream
                continue
            f.write("@%s/%d\n%s\n+\n%s\n" % (n, 1 + (i & 1), s, q))
    a, b = _both(["mem", "-t", "1", "-p", fa, fq])
    assert _records(a) == _records(b)
    a, b = _both(["mem", "-t", "1", fa, fq])  # the same file as single-end reads
    assert _records(a) == _records(b)


def test_cli_fused_samblaster_stage(ssq, cli_ref, tmp_path, monkeypatch):
    """SSQ_FUSE_SAMBLASTER: `bwa mem | samblaster` with samblaster's stage executed on the device inside `bwa mem`; the three streams
    must equal the oracle's pipe, and the unfused product pipe, byte for byte (minus @PG)"""
    from test_hostsim_pipe import stress_reads
    d, fa, g, bounds = cli_ref
    names, seqs, quals = stress_reads(g, bounds, 40000, 150, 8)  # -t 1: two batches (dups across them)
    fq = str(d / "fused.fq")
    T.write_fastq(fq, names, seqs, quals)
    sb_args = ["--excludeDups", "--addMateTags", "--maxSplitCount", "2", "--minNonOverlap", "20"]
    outs = {}
    for tag, bwa, sb, env in (("oracle", [T.ORACLE_BIN], [T.ORACLE_BIN, "samblaster"], {}), ("unfused", [BWA], [SAMBLASTER], {}),
                              ("fused", [BWA], [SAMBLASTER], {"SSQ_FUSE_SAMBLASTER": " ".join(sb_args)})):
        e = dict(os.environ); e.update(env)
        spl, disc = str(tmp_path / (tag + ".spl")), str(tmp_path / (tag + ".disc"))
        p1 = subprocess.Popen(bwa + ["mem", "-t", "1", "-p", "-R", RG, fa, fq], stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, env=e)
        p2 = subprocess.run(sb + sb_args + ["--splitterFile", spl, "--discordantFile", disc], stdin=p1.stdout, stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, env=e, check=True, timeout=300)
        assert p1.wait(timeout=60) == 0
        outs[tag] = (_strip_pg(p2.stdout), _strip_pg(open(spl, "rb").read()), _strip_pg(open(disc, "rb").read()))
    for i, what in enumerate(("main", "splitters", "discordants")):
        assert outs["oracle"][i] == outs["unfused"][i], what
        assert outs["oracle"][i] == outs["fused"][i], what
    assert outs["fused"][0].count(b"\n") > 80000 and outs["fused"][1].count(b"\n") > 100 and outs["fused"][2].count(b"\n") > 500


def _bam_to_sam(d):
    """records of a decompressed BAM file as SAM lines + their (reference, position, strand) keys (htslib sam.c:443-467 layout)"""
    import struct
    assert d[:4] == b"BAM\x01"
    l_text = struct.unpack("<i", d[4:8])[0]
    text = d[8:8 + l_text]
    p = 8 + l_text
    n_ref = struct.unpack("<i", d[p:p + 4])[0]
    p += 4
    refs = []
    for _ in range(n_ref):
        l = struct.unpack("<i", d[p:p + 4])[0]
        refs.append(d[p + 4:p + 4 + l - 1]); p += 8 + l
    lines, keys = [], []
    while p < len(d):
        bs, tid, pos, l_name, mapq, _bin, n_cig, flag, l_seq, mtid, mpos, tlen = struct.unpack("<iiiBBHHHiiii", d[p:p + 36])
        q = p + 36
        name = d[q:q + l_name - 1]; q += l_name
        cig = b"".join(b"%d%c" % (v >> 4, b"MIDNSHP=X"[v & 15]) for v in struct.unpack("<%dI" % n_cig, d[q:q + 4 * n_cig])) or b"*"; q += 4 * n_cig
        sq = d[q:q + (l_seq + 1) // 2]; q += (l_seq + 1) // 2
        seq = bytes(b"=ACMGRSVTWYHKDBN"[(sq[i >> 1] >> (4 if i % 2 == 0 else 0)) & 15] for i in range(l_seq)) or b"*"
        ql = d[q:q + l_seq]; q += l_seq
        qual = b"*" if (l_seq == 0 or ql[0] == 0xff) else bytes(c + 33 for c in ql)
        tags = []
        end = p + 4 + bs
        while q < end:
            tg, ty = d[q:q + 2], d[q + 2:q + 3]; q += 3
            if ty == b"Z":
                e = d.index(b"\0", q); tags.append(tg + b":Z:" + d[q:e]); q = e + 1
            elif ty == b"A":
                tags.append(tg + b":A:" + d[q:q + 1]); q += 1
            else:
                fmt, n = {b"c": ("<b", 1), b"C": ("<B", 1), b"s": ("<h", 2), b"S": ("<H", 2), b"i": ("<i", 4), b"I": ("<I", 4)}[ty]
                tags.append(tg + b":i:%d" % struct.unpack(fmt, d[q:q + n])[0]); q += n
        rn = refs[tid] if tid >= 0 else b"*"
        mrn = b"*" if mtid < 0 else (b"=" if mtid == tid else refs[mtid])
        lines.append(b"\t".join([name, b"%d" % flag, rn, b"%d" % (pos + 1), b"%d" % mapq, cig, mrn, b"%d" % (mpos + 1), b"%d" % tlen, seq, qual] + tags))
        keys.append((tid if tid >= 0 else 1 << 40, pos, (flag >> 4) & 1))
        p = end
    return text, lines, keys


def test_cli_bam_mode_main_records_leave_as_sorted_runs(ssq, cli_ref, tmp_path):
    """SSQ_FUSE_BAM: `bwa mem | samblaster | sambamba view -S -f bam -l 0 | sambamba sort` (speedseq:438-441) with the three shims; the
    main records are encoded and coordinate-sorted on the device per batch and merged by the `sambamba` shim — no SAM text of them
    exists anywhere.  out.bam decoded must hold exactly the records of the (oracle-identical) fused text pipe, ordered by (reference,
    position, strand) with ties in input order — the order pinned on the reference's sambamba in tests/test_bam_golden.py; the side
    streams stay the text they were."""
    import gzip
    from test_hostsim_pipe import stress_reads
    SAMBAMBA = os.path.join(T.ROOT, "speedseq_b200", "bin", "sambamba")
    d, fa, g, bounds = cli_ref
    names, seqs, quals = stress_reads(g, bounds, 40000, 150, 8)  # -t 1: two batches = two runs
    fq = str(d / "bam_mode.fq")
    T.write_fastq(fq, names, seqs, quals)
    sb_args = ["--excludeDups", "--addMateTags", "--maxSplitCount", "2", "--minNonOverlap", "20"]
    res = {}
    for tag, extra in (("text", {}), ("bam", {"SSQ_FUSE_BAM": "1"})):
        e = dict(os.environ, SSQ_FUSE_SAMBLASTER=" ".join(sb_args), **extra)
        spl, disc = str(tmp_path / (tag + ".spl")), str(tmp_path / (tag + ".disc"))
        p1 = subprocess.Popen([BWA, "mem", "-t", "1", "-p", "-R", RG, fa, fq], stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, env=e)
        p2 = subprocess.run([SAMBLASTER] + sb_args + ["--splitterFile", spl, "--discordantFile", disc], stdin=p1.stdout, stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, env=e, check=True, timeout=300)
        assert p1.wait(timeout=60) == 0
        res[tag] = (p2.stdout, open(spl, "rb").read(), open(disc, "rb").read())
    assert _strip_pg(res["bam"][1]) == _strip_pg(res["text"][1]) and _strip_pg(res["bam"][2]) == _strip_pg(res["text"][2])
    assert b"@CO\tssq-bam-runs-v1\n" in res["bam"][0][:4096] and res["bam"][0].count(b"SSQFRAME") >= 2
    out = str(tmp_path / "out.bam")
    v = subprocess.run([SAMBAMBA, "view", "-S", "-f", "bam", "-l", "0", "/dev/stdin"], input=res["bam"][0], stdout=subprocess.PIPE, check=True, timeout=120).stdout
    subprocess.run([SAMBAMBA, "sort", "-t", "4", "-m", "1G", "--tmpdir=" + str(tmp_path), "-o", out, "/dev/stdin"], input=v, check=True, timeout=120)
    text, lines, keys = _bam_to_sam(gzip.decompress(open(out, "rb").read()))
    want = _records(res["text"][0]).splitlines()
    assert len(lines) == len(want) > 80000
    assert text.startswith(b"@HD\tVN:1.3\tSO:coordinate\n@SQ\t") and b"\n@RG\tID:NA12878\tLB:lib1\tSM:NA12878\n" in text and b"ssq-" not in text
    assert keys == sorted(keys)
    order = {}
    for i, l in enumerate(want):
        order.setdefault(l, []).append(i)
    at = {}
    idx = []
    for l in lines:  # every BAM record is one text record (identical lines: in their input order)
        k = at.get(l, 0)
        assert l in order and k < len(order[l]), l
        idx.append(order[l][k]); at[l] = k + 1
    assert sorted(idx) == list(range(len(want)))
    for a in range(1, len(idx)):
        if keys[a] == keys[a - 1]:
            assert idx[a] > idx[a - 1], (a, lines[a])


def test_cli_fastq_ingest_on_the_device_and_its_fallbacks(ssq, cli_ref):
    """the `bwa` shim hands the FASTQ text to the device tokeniser (ssq_aligner_upload_fastq); layouts it does not take — multi-line
    records, FASTA, blank lines — must silently go through the host tokeniser with identical results; CRLF line ends and a last line
    without newline are the device tokeniser's business"""
    d, fa, g, bounds = cli_ref
    names, seqs, quals = T.simulate_pairs(g, bounds, 1200, 150, 13)
    quals = ["".join(chr(33 + (7 * i + k) % 40) for k in range(len(s))) for i, s in enumerate(seqs)]  # real-looking qualities incl. '@' and '+' at line starts
    quals[4] = "@" + quals[4][1:]; quals[7] = "+" + quals[7][1:]
    rec = lambda i, nl="\n": "@%s/%d cm:Z:%d%s%s%s+%s%s" % (names[i], 1 + (i & 1), i, nl, seqs[i], nl, nl, quals[i])
    variants = {
        "plain": "".join(rec(i) + "\n" for i in range(len(names))),
        "crlf": "".join(rec(i, "\r\n") + "\r\n" for i in range(len(names))),
        "no_final_newline": "".join(rec(i) + "\n" for i in range(len(names)))[:-1],
        "multiline": "".join("@%s/%d\n%s\n%s\n+\n%s\n%s\n" % (names[i], 1 + (i & 1), seqs[i][:70], seqs[i][70:], quals[i][:70], quals[i][70:]) for i in range(len(names))),
        "fasta": "".join(">%s/%d\n%s\n" % (names[i], 1 + (i & 1), seqs[i]) for i in range(len(names))),
        "blank_lines": "".join(rec(i) + "\n" + ("\n" if i % 50 == 0 else "") for i in range(len(names))),
    }
    for tag, text in variants.items():
        fq = str(d / ("ing_%s.fq" % tag))
        open(fq, "w", newline="").write(text)
        for extra in (["-p"], ["-p", "-C"]):
            a, b = _both(["mem", "-t", "1"] + extra + [fa, fq])
            assert _records(a) == _records(b), (tag, extra)
            assert _records(b).count(b"\n") >= 2400
    # the device path is really taken for the plain layouts (and really left for the others)
    for tag, want in (("plain", False), ("crlf", False), ("no_final_newline", False), ("multiline", True), ("fasta", True), ("blank_lines", True)):
        e = dict(os.environ, SSQ_VERBOSE_INGEST="1")
        err = subprocess.run([BWA, "mem", "-t", "1", "-p", fa, str(d / ("ing_%s.fq" % tag))], stdout=subprocess.DEVNULL, stderr=subprocess.PIPE, env=e, check=True).stderr
        assert (b"host tokeniser takes over" in err) == want, tag
