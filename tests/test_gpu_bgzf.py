"""BGZF compression on the device (ssq_bgzf_*, csrc/ssq_bgzf.cu): byte for byte what the host restatement of its kernels makes
(tests/test_bgzf_cpu.py checks that those files are valid BGZF), from host and from device buffers, for small and large inputs;
and the `sambamba` shim with SSQ_BGZF_GPU=1 writing sorted BAM files that hold the same records as without it."""
import gzip
import os
import struct
import subprocess

import numpy as np
import pytest

try:  # before anything loads libssq: torch must bring in its own NCCL first
    import torch
except ImportError:
    torch = None

import ssq_testlib as T
from test_bgzf_cpu import REAL_SAMBAMBA, bgzf_host, check_file, hostsim_bgzf, inputs, zlib_bgzf  # noqa: F401  (fixture)
from test_gpu_cli import BWA, RG, SAMBLASTER, cli_ref  # noqa: F401  (fixture)

pytestmark = pytest.mark.gpu
SHIM = os.path.join(T.ROOT, "speedseq_b200", "bin", "sambamba")


@pytest.fixture(scope="module")
def bz(ssq):
    z = ssq.bgzf_create(0)
    yield z
    ssq.bgzf_free(z)


def test_device_output_equals_the_host_restatement(ssq, bz, bgzf_host, ssq_lib_cpu):  # noqa: F811
    for name, data in inputs().items():
        for level in (6, 1, 0):
            got = ssq.bgzf_deflate(bz, data, level)
            assert got == hostsim_bgzf(bgzf_host, data, level), (name, level)
        check_file(got, data, zlib_bgzf(ssq_lib_cpu, data, 0))
        assert ssq.bgzf_deflate(bz, data, 6, 0) == hostsim_bgzf(bgzf_host, data, 6, 0), name


def big_input(mb=288):
    """several launches' worth of BAM records with some noise: the golden records, every copy slightly altered"""
    rec = np.frombuffer(gzip.open(os.path.join(T.GOLDEN, "ex_bam_main.records.gz")).read(), np.uint8)
    rng = np.random.default_rng(5)
    parts, n = [], 0
    while n < mb << 20:
        c = rec.copy()
        c[rng.integers(0, len(c), 2000)] = rng.integers(0, 256, 2000, dtype=np.uint8)
        parts.append(c); n += len(c)
    return np.concatenate(parts)[: mb << 20].tobytes()


def test_large_input_is_deterministic_and_equals_the_host_restatement(ssq, bz, bgzf_host):  # noqa: F811
    data = big_input()
    a = ssq.bgzf_deflate(bz, data, 6)
    assert a == ssq.bgzf_deflate(bz, data, 6)
    assert a == hostsim_bgzf(bgzf_host, data, 6)
    assert gzip.decompress(a) == data
    cut = 0xff00 * 3001  # any split on block boundaries gives the same members
    b = ssq.bgzf_deflate(bz, data[:cut], 6, 0) + ssq.bgzf_deflate(bz, data[cut:], 6)
    assert a == b


@pytest.mark.skipif(torch is None, reason="needs torch")
def test_device_buffers_and_capacity(ssq, bz, bgzf_host):  # noqa: F811
    for name in ("ex_bam_main", "random_1MB", "one_byte", "empty"):
        data = inputs()[name]
        want = hostsim_bgzf(bgzf_host, data, 6)
        d_in = torch.tensor(np.frombuffer(data, np.uint8) if data else np.zeros(1, np.uint8), device="cuda")
        d_out = torch.zeros(len(data) + 31 * (len(data) // 0xff00 + 1) + 64, dtype=torch.uint8, device="cuda")
        torch.cuda.synchronize()
        rc, n, need = ssq.bgzf_deflate_dev(bz, d_in.data_ptr(), len(data), d_out.data_ptr(), d_out.numel(), 6, 1)
        assert rc == 0 and n == need == len(want), name
        assert bytes(d_out[:n].cpu().numpy()) == want, name
        rc, n2, need2 = ssq.bgzf_deflate_dev(bz, d_in.data_ptr(), len(data), d_out.data_ptr(), 16, 6, 1)
        assert rc == -5 and need2 == len(want), name


def test_sambamba_shim_compresses_on_the_device(ssq, oracle, hostsim, syn_index, ssq_lib_cpu, tmp_path):
    """the run stream of test_bam_golden's shim test through `sambamba sort` with SSQ_BGZF_GPU=1: the golden records, the rewritten
    header, the same file for any -t and with spills; the reference's sambamba counts, indexes and queries it like the zlib file"""
    import ctypes as C
    from test_bam_golden import _bam_file, contigs_of, golden, split_records, syn_reads
    idx = oracle.load(syn_index[0])
    names, seqs, quals = syn_reads(syn_index)
    cuts = [0, 1000, 2100, len(names)]
    hdr = b"".join(b"@SQ\tSN:%s\tLN:%d\n" % (n, l) for n, l in contigs_of(syn_index)) + b"@RG\tID:NA12878\tSM:NA12878\tLB:lib1\n"
    stream = hdr + b"@CO\tssq-bam-runs-v1\n"
    for k, (a, b) in enumerate(zip(cuts, cuts[1:])):
        txt, bams = hostsim.pipe_bam(idx, names[a:b], seqs[a:b], quals[a:b], a, b"NA12878", 1, (1, 1, 2, 20, 0), reset=1 if k == 0 else 0)
        stream += b"SSQFRAME" + struct.pack("<QQ", 3, len(bams[0])) + bams[0]
    L = ssq_lib_cpu
    L.ssq_bam_header_text.argtypes = [C.c_char_p, C.c_int, C.c_void_p]
    out = C.c_void_p()
    assert L.ssq_bam_header_text(hdr, 1, C.byref(out)) == 0
    want_text = C.string_at(out)
    L.ssq_free(out)
    files = {}
    for tag, env, t, lvl in (("plain_t4", {}, 4, "6"), ("plain_t1", {}, 1, "6"), ("spill_t1", {"SSQ_SORT_SPILL_BYTES": "200000"}, 1, "6"),
                             ("spill_t4", {"SSQ_SORT_SPILL_BYTES": "200000"}, 4, "6"), ("zlib", {}, 4, "6"), ("level0", {}, 2, "0")):
        o = str(tmp_path / (tag + ".bam"))
        e = dict(os.environ, **env)
        if tag != "zlib":
            e["SSQ_BGZF_GPU"] = "1"
        subprocess.run([SHIM, "sort", "-t", str(t), "-l", lvl, "-m", "1G", "--tmpdir=" + str(tmp_path), "-o", o, "/dev/stdin"], input=stream, check=True, timeout=120, env=e)
        text, refs, recs = _bam_file(o)
        assert text == want_text and refs == list(contigs_of(syn_index)) and recs == golden("main", "syn3"), tag
        files[tag] = open(o, "rb").read()
    assert files["plain_t4"] == files["plain_t1"] == files["spill_t1"] == files["spill_t4"]
    assert files["plain_t4"] != files["zlib"] and gzip.decompress(files["plain_t4"]) == gzip.decompress(files["zlib"]) == gzip.decompress(files["level0"])
    assert {(m[0][0] >> 1) & 3 for m in __import__("test_bgzf_cpu").members(files["level0"])[:-1]} == {0}
    if os.access(REAL_SAMBAMBA, os.X_OK):
        n = int(subprocess.run([REAL_SAMBAMBA, "view", "-c", str(tmp_path / "plain_t4.bam")], stdout=subprocess.PIPE, check=True).stdout)
        assert n == len(split_records(golden("main", "syn3")))
        got = {}
        for tag in ("plain_t4", "zlib"):
            f = str(tmp_path / (tag + ".bam"))
            subprocess.run([REAL_SAMBAMBA, "index", f], check=True, stdout=subprocess.DEVNULL, stderr=subprocess.DEVNULL)
            got[tag] = [subprocess.run([REAL_SAMBAMBA, "view", f, reg], stdout=subprocess.PIPE, check=True).stdout for reg in ("ctg2:20000-90000", "ctg3", "ctg1")]
        assert got["plain_t4"] == got["zlib"] and all(got["zlib"]) and got["zlib"][0].count(b"\n") > 50


def test_three_shim_chain_with_device_bgzf(ssq, cli_ref, tmp_path):  # noqa: F811
    """`bwa mem | samblaster | sambamba view | sambamba sort` in BAM mode: out.bam with SSQ_BGZF_GPU=1 decompresses to the same bytes
    as without it (the bwa and sambamba processes share the GPU)"""
    from test_hostsim_pipe import stress_reads
    d, fa, g, bounds = cli_ref
    names, seqs, quals = stress_reads(g, bounds, 40000, 150, 8)
    fq = str(d / "bgzf_chain.fq")
    T.write_fastq(fq, names, seqs, quals)
    sb_args = ["--excludeDups", "--addMateTags", "--maxSplitCount", "2", "--minNonOverlap", "20"]
    res = {}
    for tag, extra in (("zlib", {}), ("device", {"SSQ_BGZF_GPU": "1"})):
        e = dict(os.environ, SSQ_FUSE_SAMBLASTER=" ".join(sb_args), SSQ_FUSE_BAM="1", **extra)
        out = str(tmp_path / (tag + ".bam"))
        p1 = subprocess.Popen([BWA, "mem", "-t", "1", "-p", "-R", RG, fa, fq], stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, env=e)
        p2 = subprocess.Popen([SAMBLASTER] + sb_args + ["--splitterFile", str(tmp_path / "spl"), "--discordantFile", str(tmp_path / "disc")], stdin=p1.stdout,
                              stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, env=e)
        p3 = subprocess.Popen([SHIM, "view", "-S", "-f", "bam", "-l", "0", "/dev/stdin"], stdin=p2.stdout, stdout=subprocess.PIPE, env=e)
        p4 = subprocess.run([SHIM, "sort", "-t", "4", "-m", "1G", "--tmpdir=" + str(tmp_path), "-o", out, "/dev/stdin"], stdin=p3.stdout, env=e, timeout=300)
        assert p4.returncode == 0 and p3.wait(timeout=60) == 0 and p2.wait(timeout=60) == 0 and p1.wait(timeout=60) == 0, tag
        res[tag] = open(out, "rb").read()
    assert res["device"] != res["zlib"]
    assert gzip.decompress(res["device"]) == gzip.decompress(res["zlib"]) and len(gzip.decompress(res["zlib"])) > 10 << 20
