"""gzip decoding on the device (ssq_gunzip_*, csrc/ssq_gunzip.cu): zlib's text and the host restatement's stats for the corpus of
tests/test_gunzip_cpu.py at several chunk sizes, the streaming call fed in pieces, a stream of several windows, SSQ_ECAP, the
example FASTQ; and the `bwa` shim, which reads every gzipped input through it, against the oracle CLI (which reads with zlib)."""
import gzip
import os
import random
import subprocess
import zlib

import numpy as np
import pytest

try:  # before anything loads libssq: torch must bring in its own NCCL first
    import torch
except ImportError:
    torch = None

import ssq_testlib as T
from test_gunzip_cpu import CHUNKS, EDATA, bgzf_file, corpus, fastq_text, gunzip_host, gz, hostsim_gunzip, member, zlib_text  # noqa: F401  (fixture)
from test_gpu_cli import BWA, RG, _both, _records, cli_ref  # noqa: F401  (fixture)

pytestmark = pytest.mark.gpu
EXAMPLE = os.path.join(T.ROOT, "oracle", "_ref", "stage", "example", "data", "NA12878.20slice.30X.fastq.gz")


@pytest.fixture(scope="module")
def gzs(ssq):
    """one decoder per chunk size"""
    g = {c: ssq.gunzip_create(0, c) for c in CHUNKS}
    yield g
    for h in g.values():
        ssq.gunzip_free(h)


def inflate_dev(ssq, g, z, cap=None):
    """-> (rc, text, out_len, stats of this call)"""
    d_in = torch.frombuffer(bytearray(z) or bytearray(1), dtype=torch.uint8).cuda()
    out = torch.empty(max(cap if cap is not None else 1, 1), dtype=torch.uint8, device="cuda")
    if cap is None:  # sized by a first call that reports the size
        rc, n = ssq.gunzip_inflate_dev(g, d_in.data_ptr(), len(z), out.data_ptr(), 0)
        if rc == -5:
            out = torch.empty(n, dtype=torch.uint8, device="cuda")
            cap = n
        else:
            cap = 0
    s0 = ssq.gunzip_stats(g)
    rc, n = ssq.gunzip_inflate_dev(g, d_in.data_ptr(), len(z), out.data_ptr(), cap)
    s1 = ssq.gunzip_stats(g)
    text = out[:n].cpu().numpy().tobytes() if rc == 0 else b""
    return rc, text, n, tuple(b - a for a, b in zip(s0, s1))


def test_device_equals_zlib_and_the_host_restatement(ssq, gzs, gunzip_host, ssq_lib_cpu):  # noqa: F811
    items = dict(corpus())
    items["bgzf"] = bgzf_file(ssq_lib_cpu, fastq_text())
    for name, z in items.items():
        want = zlib_text(z)
        for c in CHUNKS:
            rc, text, n, st = inflate_dev(ssq, gzs[c], z)
            hrc, htext, hst, _ = hostsim_gunzip(gunzip_host, z, c)
            assert rc == 0 and n == len(want) and text == want, (name, c)
            assert st == hst, (name, c, st, hst)


def test_corrupt_stream_is_edata(ssq, gzs):
    fq = fastq_text()
    z = member(fq[:300000]) + member(fq[250000:400000], zdict=fq[300000 - 32768:300000])
    assert inflate_dev(ssq, gzs[4096], z, cap=1 << 20)[0] == EDATA
    z6 = gz(fq)
    assert inflate_dev(ssq, gzs[0], z6[:len(z6) // 2], cap=4 << 20)[0] == EDATA
    rc, _ = ssq.gunzip(gzs[0], z6[:-3])
    assert rc == EDATA and "compressed byte" in ssq.err()
    assert ssq.gunzip(gzs[0], z6) == (0, fq)  # after an error the next call starts a new stream


def big_fastq(mb):
    """about mb MB of FASTQ: the golden reads with every copy's bases slightly altered"""
    recs = np.frombuffer(fastq_text(), np.uint8)
    rng = np.random.default_rng(9)
    acgt = np.frombuffer(b"ACGT", np.uint8)
    isbase = np.isin(recs, acgt)
    parts, n = [], 0
    while n < mb << 20:
        c = recs.copy()
        k = rng.integers(0, len(c), 4000)
        k = k[isbase[k]]
        c[k] = acgt[rng.integers(0, 4, len(k))]
        parts.append(c)
        n += len(c)
    return np.concatenate(parts).tobytes()


def stream(ssq, g, z, pieces, out_cap):
    """the streaming call fed by the piece sizes in `pieces` (cycled), each call after the unconsumed rest"""
    pend, at, text, out, i = bytearray(), 0, [], np.empty(out_cap, np.uint8), 0
    while True:
        if at < len(z):
            k = pieces[i % len(pieces)]
            i += 1
            pend += z[at:at + k]
            at += k
        rc, used, t, done = ssq.gunzip_inflate(g, pend, int(at >= len(z)), out)
        assert rc == 0, ssq.err()
        text.append(t)
        del pend[:used]
        if done:
            return b"".join(text)


def test_streaming_in_pieces(ssq, gzs):
    small = corpus()["multi_member"] + b"trailing"
    want = zlib_text(small)
    for piece in (1, 7, 4099):
        assert stream(ssq, gzs[4096], small, [piece], 1 << 20) == want, piece
    text = big_fastq(96)
    z = gz(text, 1)
    assert len(z) > 3 * (4096 * 1024 + (1 << 20))  # several windows of a 4 KB-chunk decoder come from non-final calls
    rnd = random.Random(4)
    for pieces, cap in (([4099], 1 << 20), ([1 << 20], 64 << 20), ([rnd.randrange(1, 3 << 20) for _ in range(50)], 100003)):
        assert stream(ssq, gzs[4096], z, pieces, cap) == text
    assert stream(ssq, gzs[0], z, [1 << 20], 8 << 20) == text


def test_stream_of_several_windows(ssq, gzs):
    text = big_fastq(300)
    z = gz(text, 1)
    rc, got, n, st = inflate_dev(ssq, gzs[0], z, cap=len(text))
    assert rc == 0 and n == len(text) and got == text
    assert st[3] >= 2, st
    rc, n = ssq.gunzip_inflate_dev(gzs[0], torch.frombuffer(bytearray(z), dtype=torch.uint8).cuda().data_ptr(), len(z), torch.empty(len(text) - 1, dtype=torch.uint8, device="cuda").data_ptr(), len(text) - 1)
    assert rc == -5 and n == len(text)


@pytest.mark.skipif(not os.path.exists(EXAMPLE), reason="the example FASTQ is not staged under oracle/_ref")
def test_example_fastq(ssq, gzs):
    z = open(EXAMPLE, "rb").read()
    rc, text, n, st = inflate_dev(ssq, gzs[0], z)
    assert rc == 0 and text == zlib_text(z)
    assert stream(ssq, gzs[0], z, [1 << 20], 16 << 20) == text


# ---- the bwa shim on gzipped input ----
def _write_fastq(path, names, seqs, quals, opener=open):
    with opener(path, "wt") as f:
        for n, s, q in zip(names, seqs, quals):
            f.write("@%s\n%s\n+\n%s\n" % (n, s, q))


def test_cli_gzipped_inputs(ssq, cli_ref, ssq_lib_cpu):  # noqa: F811
    d, fa, g, bounds = cli_ref
    names, seqs, quals = T.simulate_pairs(g, bounds, 6000, 150, 21)
    names = ["%s/%d" % (n, 1 + (i & 1)) for i, n in enumerate(names)]
    inter = str(d / "gz_inter.fq")
    _write_fastq(inter, names, seqs, quals)
    text = open(inter, "rb").read()
    r1, r2 = str(d / "gz_r1.fq.gz"), str(d / "gz_r2.fq.gz")
    _write_fastq(r1, names[0::2], seqs[0::2], quals[0::2], opener=gzip.open)
    _write_fastq(r2, names[1::2], seqs[1::2], quals[1::2], opener=gzip.open)
    a, b = _both(["mem", "-t", "2", "-R", RG, fa, r1, r2])
    assert _records(a) == _records(b) and _records(b).count(b"\n") >= 12000
    cut = [0, len(text) // 3, len(text) // 3 + 10, 2 * len(text) // 3, len(text)]
    files = {"p": gz(text), "multi": b"".join(member(text[cut[i]:cut[i + 1]], 8 * (i & 1)) for i in range(4)), "bgzf": bgzf_file(ssq_lib_cpu, text)}
    ref = None
    for tag, z in files.items():
        p = str(d / ("gz_%s.fq.gz" % tag))
        open(p, "wb").write(z)
        a, b = _both(["mem", "-t", "2", "-p", fa, p])
        assert _records(a) == _records(b), tag
        ref = ref or _records(b)
        assert _records(b) == ref, tag
    p = str(d / "gz_p.fq.gz")
    b = subprocess.run([BWA, "mem", "-t", "2", "-p", fa, "-"], stdin=open(p, "rb"), check=True, stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, timeout=300).stdout
    assert _records(b) == ref  # gzipped stdin


def test_cli_host_tokeniser_takes_over_gzipped_text(ssq, cli_ref):  # noqa: F811
    """-t 1: the first batch (10 Mbp) is four-line FASTQ for the device tokeniser; multi-line records follow, so the host tokeniser
    continues from the device-inflated text and then reads the rest of the file through the decoder"""
    d, fa, g, bounds = cli_ref
    names, seqs, quals = T.simulate_pairs(g, bounds, 45000, 150, 23)
    names = ["%s/%d" % (n, 1 + (i & 1)) for i, n in enumerate(names)]
    ml = str(d / "gz_multiline.fq.gz")
    with gzip.open(ml, "wt") as f:
        for k, (n, s, q) in enumerate(zip(names, seqs, quals)):
            w = 60 if k >= 80000 else 1000
            f.write("@%s\n%s\n+\n%s\n" % (n, "\n".join(s[i:i + w] for i in range(0, len(s), w)), "\n".join(q[i:i + w] for i in range(0, len(q), w))))
    a, b = _both(["mem", "-t", "1", "-p", fa, ml])
    assert _records(a) == _records(b) and _records(b).count(b"\n") >= 90000


def test_cli_truncated_gzip_fails_with_the_file_name(ssq, cli_ref):  # noqa: F811
    d, fa, g, bounds = cli_ref
    names, seqs, quals = T.simulate_pairs(g, bounds, 1000, 150, 22)
    z = gz("".join("@%s/%d\n%s\n+\n%s\n" % (n, 1 + (i & 1), s, q) for i, (n, s, q) in enumerate(zip(names, seqs, quals))).encode())
    p = str(d / "truncated.fq.gz")
    open(p, "wb").write(z[:len(z) * 2 // 3])
    r = subprocess.run([BWA, "mem", "-t", "2", "-p", fa, p], stdout=subprocess.PIPE, stderr=subprocess.PIPE, timeout=300)
    assert r.returncode != 0 and b"truncated.fq.gz" in r.stderr and b"corrupt or truncated" in r.stderr
