"""The BAI builder on the device (ssq_bai_*, csrc/ssq_bai.cu) and the member-parallel BGZF entry (ssq_gunzip_inflate_bgzf_dev):
every golden .bai of tests/golden (written by the reference's sambamba), byte for byte, at several walker segment sizes; the same
refusals and messages as the host restatement (tests/test_bai_cpu.py); zlib's text and the member table; the `sambamba` shim's
`index`; `sort -o` writing out.bam.bai equal to the staged sambamba's index of the same file, with host and device BGZF; a 100 MB
BAM against the staged sambamba; a member table that has to grow; and a bench-sized BAM (about 2 GB of `bwa mem -p` SAM, the input
of tools/sam2bam_bench.py, through the shim chain `view -S | sort -o`) whose .bai equals the staged sambamba's index of it."""
import gzip
import os
import random
import shutil
import struct
import subprocess

import pytest

try:  # before anything loads libssq: torch must bring in its own NCCL first
    import torch
except ImportError:
    torch = None

import ssq_testlib as T
from golden.make_bai_golden import header, record
from test_bai_cpu import GOLDEN, SHIM, bai_host, hostsim_bai, refused  # noqa: F401  (fixture)

pytestmark = pytest.mark.gpu
REAL = os.path.join(T.ROOT, "oracle", "_ref", "stage", "src", "sambamba")
need_real = pytest.mark.skipif(not os.access(REAL, os.X_OK), reason="speedseq's own sambamba is not staged under oracle/_ref (build() stages it from a speedseq checkout)")


@pytest.fixture(scope="module")
def bais(ssq):
    h = {s: ssq.bai_create(0, s) for s in (0, 97, 4096)}
    yield h
    for b in h.values():
        ssq.bai_free(b)


def test_device_gives_the_goldens(ssq, bais):
    for p in GOLDEN:
        bam, want = open(p, "rb").read(), open(p + ".bai", "rb").read()
        for s, b in bais.items():
            rc, got = ssq.bai_build(b, bam)
            assert rc == 0, (p, s, ssq.err())
            assert got == want, (p, s)


def test_device_refuses_what_the_host_refuses(ssq, bais, bai_host):  # noqa: F811
    for name, bam, code, msg in refused():
        rc, _, herr = hostsim_bai(bai_host, bam, 97)
        drc, _ = ssq.bai_build(bais[97], bam)
        derr = ssq.err()
        assert drc == rc == code and msg in derr and herr in derr, (name, drc, derr, herr)
    # the object is still good after refusals
    rc, got = ssq.bai_build(bais[97], open(GOLDEN[0], "rb").read())
    assert rc == 0 and got == open(GOLDEN[0] + ".bai", "rb").read()


def members_of(z):
    out, c, t = [], 0, 0
    while c < len(z):
        bsize = struct.unpack_from("<H", z, c + 16)[0]
        out.append((c, t))
        t += struct.unpack_from("<I", z, c + bsize + 1 - 4)[0]
        c += bsize + 1
    return out


def test_bgzf_entry_gives_zlib_text_and_the_member_table(ssq):
    g = ssq.gunzip_create(0, 0)
    s0 = ssq.gunzip_stats(g)
    for p in GOLDEN:
        z = open(p, "rb").read()
        d_in = torch.frombuffer(bytearray(z), dtype=torch.uint8).cuda()
        rc, n, _ = ssq.gunzip_inflate_bgzf_dev(g, d_in.data_ptr(), len(z), 0, 0, 0)
        assert rc == -5
        out = torch.empty(max(n, 1), dtype=torch.uint8, device="cuda")
        rc, n2, mt = ssq.gunzip_inflate_bgzf_dev(g, d_in.data_ptr(), len(z), out.data_ptr(), n, len(z) // 28 + 1)
        assert rc == 0 and n2 == n
        assert out[:n].cpu().numpy().tobytes() == gzip.decompress(z)
        assert mt == members_of(z)
    assert ssq.gunzip_stats(g) == s0  # the chunked decoder's statistics are left alone
    ssq.gunzip_free(g)


def test_shim_index_equals_the_goldens(tmp_path):
    for p in GOLDEN:
        q = str(tmp_path / os.path.basename(p))
        shutil.copy(p, q)
        r = subprocess.run([SHIM, "index", "-t", "8", q], capture_output=True, text=True, timeout=300)
        assert r.returncode == 0 and r.stderr == "", r.stderr
        assert open(q + ".bai", "rb").read() == open(p + ".bai", "rb").read(), p
        r = subprocess.run([SHIM, "index", "-p", q, q + ".other"], capture_output=True, text=True, timeout=300)
        assert r.returncode == 0 and open(q + ".other", "rb").read() == open(p + ".bai", "rb").read()


def _env(**kw):
    env = {k: v for k, v in os.environ.items() if k not in ("SSQ_SAMBAMBA_REAL", "SSQ_SAM2BAM_GPU", "SSQ_SAM2BAM_CHUNK", "SSQ_BGZF_GPU")}
    env.update(kw)
    return env


@need_real
@pytest.mark.parametrize("bgzf_gpu", ["0", "1"])
def test_sort_writes_the_index_sambamba_writes(tmp_path, bgzf_gpu):
    # without the lines with an RNAME and POS 0: a record with a reference and no position is refused by the device (its index
    # then comes from the real sambamba)
    sam = b"".join(l for l in open(os.path.join(T.GOLDEN, "sam2bam_edge.sam"), "rb") if l.startswith(b"@") or not (l.split(b"\t")[2] != b"*" and l.split(b"\t")[3] == b"0"))
    out = str(tmp_path / "s.bam")
    v = subprocess.run([SHIM, "view", "-S", "-f", "bam", "-l", "0", "/dev/stdin"], input=sam, stdout=subprocess.PIPE, check=True, timeout=600,
                       env=_env(SSQ_SAM2BAM_GPU="1"))
    s = subprocess.run([SHIM, "sort", "-t", "4", "-o", out, "/dev/stdin"], input=v.stdout, stderr=subprocess.PIPE, timeout=600, env=_env(SSQ_BGZF_GPU=bgzf_gpu))
    assert s.returncode == 0 and s.stderr == b"", s.stderr
    ref = str(tmp_path / "copy.bam")
    shutil.copy(out, ref)
    subprocess.run([REAL, "index", ref], check=True, timeout=600)
    assert open(out + ".bai", "rb").read() == open(ref + ".bai", "rb").read()


@need_real
def test_a_100mb_bam_equals_sambambas_index(ssq, bais, tmp_path):
    """some 400,000 sorted records over 25 references (two empty), about 100 MB of text, compressed on the device"""
    R = random.Random(5)
    refs = [("r%d" % i, 250000000) for i in range(25)]
    recs = []
    for ref in range(25):
        if ref in (3, 17):
            continue
        for p in sorted(R.randrange(0, 250000000) for _ in range(17000)):
            k = R.random()
            cg = "100M%dN50M" % R.choice([500, 30000, 2000000]) if k < 0.05 else "150M"
            recs.append(record("q%d" % p, 4 | 1 if k > 0.97 else 99, ref, p, "*" if k > 0.97 else cg, seqlen=150))
    recs += [record("nc%d" % i, 77, -1, -1, "*", seqlen=150) for i in range(1000)]
    text = header(refs) + b"".join(recs)
    z = ssq.bgzf_create(0)
    bam = ssq.bgzf_deflate(z, text, 1, 1)
    ssq.bgzf_free(z)
    p = str(tmp_path / "big.bam")
    open(p, "wb").write(bam)
    subprocess.run([REAL, "index", "-t", "8", p], check=True, timeout=900)
    want = open(p + ".bai", "rb").read()
    for s in (0, 4096):
        rc, got = ssq.bai_build(bais[s], bam)
        assert rc == 0 and got == want, s
    del text, bam


def test_member_table_grows_for_small_members(ssq, bais, bai_host):  # noqa: F811
    """one record per BGZF member: more members than the first table holds (room for 8 KB members)"""
    from golden.make_bai_golden import bgzf
    recs = [record("m%d" % i, 0, 0, 100 * i) for i in range(3000)]
    bam = bgzf(header([("c1", 10000000)]) + b"".join(recs), 57)
    hrc, want, herr = hostsim_bai(bai_host, bam)
    assert hrc == 0, herr
    rc, got = ssq.bai_build(bais[0], bam)
    assert rc == 0 and got == want, ssq.err()


@need_real
def test_bench_sized_bam_through_the_shim_chain(ssq, tmp_path_factory):
    """tools/sam2bam_bench.py's input (tools/sbtext_bench.py: about 2 GB of name-grouped `bwa mem -p` SAM on a 63 Mbp synthetic
    genome, made by the `bwa` shim in SSQ_BENCH_CACHE when set, else in a temporary directory), through `view -S -f bam -l 0 |
    sort -t 16 -o` with SSQ_SAM2BAM_GPU=1: the .bai the shim's sort writes is the staged sambamba's index of the same file"""
    import sys
    sys.path.insert(0, os.path.join(T.ROOT, "tools"))
    import bench
    import sbtext_bench as SB
    d = tmp_path_factory.mktemp("bench_bai")
    cache = os.environ.get("SSQ_BENCH_CACHE") or str(d)
    fa, g = bench.ensure_reference(cache, SB.GLEN, lambda f: ssq.index_build(f, None, 0))
    sam = os.path.join(cache, "sbtext_2.sam")
    if not os.path.exists(sam):
        SB.make_sam(sam, fa, g, 2.0)
    out = str(d / "bench.bam")
    with open(sam, "rb") as fi:
        v = subprocess.Popen([SHIM, "view", "-S", "-f", "bam", "-l", "0", "/dev/stdin"], stdin=fi, stdout=subprocess.PIPE, env=_env(SSQ_SAM2BAM_GPU="1"))
        s = subprocess.run([SHIM, "sort", "-t", "16", "-m", "8G", "--tmpdir=" + str(d / "tmp"), "-o", out, "/dev/stdin"], stdin=v.stdout, stderr=subprocess.PIPE,
                           timeout=900, env=_env(SSQ_BGZF_GPU="1"))
        v.stdout.close()
        assert v.wait(timeout=900) == 0
    assert s.returncode == 0 and s.stderr == b"", s.stderr
    assert os.path.getsize(out) > 200 << 20
    ref = str(d / "copy.bam")
    shutil.copy(out, ref)
    subprocess.run([REAL, "index", "-t", "16", ref], check=True, timeout=900)
    assert open(out + ".bai", "rb").read() == open(ref + ".bai", "rb").read()
