"""The BAI builder (speedseq_b200/csrc/ssq_bai.cuh, with the BGZF member path of ssq_gunzip.cuh) run on the host by
tests/hostsim/bai_host.cpp (the same SSQ_HD phases and host logic, host loops in place of the kernels), and the oracle's
independent sequential restatement of sambamba's indexer (oracle/ssqo_bai.c), each compiled into a temporary directory: every
tests/golden/bai_*.bam gives the .bai the reference's sambamba wrote for it, byte for byte — from the oracle, and from the host
builder whatever the walker segment size (so that segment guesses fail, records span several segments and links are walked
again).  Each refusal gives its message, and the oracle refuses the same files.  The `sambamba` shim's `index` without a GPU hands the call to the real sambamba after one stderr line."""
import ctypes as C
import glob
import os
import struct
import subprocess

import pytest

import ssq_testlib as T
from golden.make_bai_golden import bgzf, header, member, record

EDATA, EFORMAT = -9, -8
SEGS = (0, 64, 97, 1000, 70000)
GOLDEN = sorted(glob.glob(os.path.join(T.GOLDEN, "bai_*.bam")))


def build_bai_host(d):
    so = os.path.join(str(d), "libbai_host.so")
    subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-w", "-I", os.path.join(T.ROOT, "include"), "-o", so,
                    os.path.join(T.ROOT, "tests", "hostsim", "bai_host.cpp")], check=True)
    lib = C.CDLL(so)
    lib.hostsim_bai.argtypes = [C.c_char_p, C.c_size_t, C.c_size_t, C.c_void_p, C.c_void_p, C.c_char_p, C.c_size_t]
    lib.hostsim_bai_free.argtypes = [C.c_void_p]
    return lib


@pytest.fixture(scope="module")
def bai_host(tmp_path_factory):
    return build_bai_host(tmp_path_factory.mktemp("bai_host"))


@pytest.fixture(scope="module")
def bai_oracle(tmp_path_factory):
    so = os.path.join(str(tmp_path_factory.mktemp("bai_oracle")), "libssqo_bai.so")
    subprocess.run(["gcc", "-O2", "-fPIC", "-shared", "-w", "-o", so, os.path.join(T.ROOT, "oracle", "ssqo_bai.c"), "-lz"], check=True)
    lib = C.CDLL(so)
    lib.ssqo_bai.argtypes = [C.c_char_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_char_p, C.c_size_t]
    return lib


def oracle_bai(lib, bam):
    """-> (rc, index bytes, message); the index is malloc'd by the oracle and left to the process (test sizes)"""
    out, n, err = C.c_void_p(), C.c_size_t(0), C.create_string_buffer(512)
    rc = lib.ssqo_bai(bam, len(bam), C.byref(out), C.byref(n), err, 512)
    return rc, C.string_at(out, n.value) if rc == 0 else b"", err.value.decode()


def hostsim_bai(lib, bam, seg=0):
    """-> (rc, index bytes, message)"""
    out, n, err = C.c_void_p(), C.c_size_t(0), C.create_string_buffer(512)
    rc = lib.hostsim_bai(bam, len(bam), seg, C.byref(out), C.byref(n), err, 512)
    data = C.string_at(out, n.value) if rc == 0 else b""
    if rc == 0:
        lib.hostsim_bai_free(out)
    return rc, data, err.value.decode()


def test_goldens_exist():
    names = {os.path.basename(p) for p in GOLDEN}
    assert {"bai_refs.bam", "bai_bigrec.bam", "bai_bins.bam", "bai_noeof.bam", "bai_header.bam", "bai_syn.bam", "bai_syn3.bam", "bai_pos0.bam"} <= names
    for p in GOLDEN:
        assert os.path.exists(p + ".bai")


@pytest.mark.parametrize("seg", SEGS)
@pytest.mark.parametrize("path", GOLDEN, ids=os.path.basename)
def test_host_builder_gives_sambambas_index(bai_host, path, seg):
    bam = open(path, "rb").read()
    rc, bai, err = hostsim_bai(bai_host, bam, seg)
    assert rc == 0, err
    assert bai == open(path + ".bai", "rb").read()


@pytest.mark.parametrize("path", GOLDEN, ids=os.path.basename)
def test_oracle_gives_sambambas_index(bai_oracle, path):
    rc, bai, err = oracle_bai(bai_oracle, open(path, "rb").read())
    assert rc == 0, err
    assert bai == open(path + ".bai", "rb").read()


REFS = [("c1", 100000000), ("c2", 1000)]


def refused():
    """(name, file, code, part of the message)"""
    H = header(REFS)
    ok = record("a", 0, 0, 500)
    yield "unsorted", bgzf(H + ok + record("b", 0, 0, 200), 0xff00), EFORMAT, "not coordinate-sorted"
    yield "unsorted_ref", bgzf(H + record("a", 0, 1, 5) + record("b", 0, 0, 200), 0xff00), EFORMAT, "not coordinate-sorted"
    yield "ref_beyond", bgzf(H + ok + record("b", 0, 2, 200), 0xff00), EFORMAT, "not a reference of the header"
    yield "ref_below", bgzf(H + ok + record("b", 0, -2, 200), 0xff00), EFORMAT, "not a reference of the header"
    yield "no_pos", bgzf(H + ok + record("b", 4, 1, -1, "*"), 0xff00), EFORMAT, "no position"
    yield "pos_2_29", bgzf(H + ok + record("b", 0, 0, 1 << 29, bin=4680), 0xff00), EFORMAT, "2^29"
    yield "end_2_29", bgzf(H + ok + record("b", 0, 0, (1 << 29) - 5, "20M", bin=4680), 0xff00), EFORMAT, "2^29"
    yield "nocoor_first", bgzf(H + record("n", 4, -1, -1, "*") + ok, 0xff00), EFORMAT, "without a reference comes before"
    t = H + ok + ok
    yield "empty_member_inside", member(t[:len(H)]) + member(b"") + member(t[len(H):]) + member(b""), EFORMAT, "empty BGZF member"
    yield "truncated_record", bgzf(H + ok[:-3], 0xff00), EFORMAT, "not a BAM record"
    yield "bad_block_size", bgzf(H + ok + struct.pack("<i", 8) + b"\0" * 8, 0xff00), EFORMAT, "not a BAM record"
    yield "not_bam", bgzf(b"hello world, not BAM at all", 0xff00), EFORMAT, "no BAM magic"
    yield "short_header", bgzf(b"BAM\1" + struct.pack("<i", 100) + b"@HD", 0xff00), EFORMAT, "header is truncated"
    good = bgzf(H + ok, 0xff00)
    yield "plain_gzip", b"\x1f\x8b\x08\x00" + good[4:], EDATA, "without a BGZF BSIZE"
    yield "truncated_member", good[:-40], EDATA, "truncated member"
    yield "trailing_bytes", good + b"junk after the last member", EDATA, "no gzip member header"
    yield "trailing_short", good + b"junk", EDATA, "truncated member"
    first = len(member(H + ok))
    bad = bytearray(good)
    bad[first // 2] ^= 0x55  # inside the first member's deflate data
    yield "corrupt_member", bytes(bad), EDATA, "corrupt BGZF member at compressed byte 0"
    big = bytearray(good)
    big[first - 2] = 1  # ISIZE over 64 KB
    yield "isize_big", bytes(big), EDATA, "more than 64 KB"
    crc = bytearray(good)
    crc[first - 8] ^= 1  # the first member's CRC-32
    yield "crc", bytes(crc), EDATA, "corrupt BGZF member at compressed byte 0"
    isz = bytearray(good)
    isz[first - 4] ^= 1  # its ISIZE
    yield "isize", bytes(isz), EDATA, "compressed byte 0"


@pytest.mark.parametrize("name,bam,code,msg", list(refused()), ids=[r[0] for r in refused()])
def test_refusals(bai_host, bai_oracle, name, bam, code, msg):
    for seg in (0, 97):
        rc, _, err = hostsim_bai(bai_host, bam, seg)
        assert rc == code and msg in err, (name, seg, rc, err)
    assert oracle_bai(bai_oracle, bam)[0] != 0, name


SHIM = os.path.join(T.ROOT, "speedseq_b200", "bin", "sambamba")


@pytest.mark.skipif(not os.path.exists(SHIM), reason="the CLI shims are built by build()")
def test_shim_index_without_gpu_goes_to_the_real_sambamba(tmp_path):
    """no usable GPU, -c, -C: one stderr line naming the reason, then the real sambamba with the same arguments"""
    if T.gpu_visible():
        pytest.skip("a GPU is visible: the shim indexes on it (tests/test_gpu_bai.py)")
    real = tmp_path / "real.sh"
    real.write_text("#!/bin/sh\necho \"real $*\"\n")
    real.chmod(0o755)
    env = dict(os.environ, SSQ_SAMBAMBA_REAL=str(real))
    bam = GOLDEN[0]
    for args, why in ((["index", "-t", "4", bam], "no usable GPU"), (["index", "-c", bam], "bin check"), (["index", "-C", bam], "CRAM")):
        r = subprocess.run([SHIM] + args, env=env, capture_output=True, text=True)
        assert r.returncode == 0 and r.stdout.strip() == "real " + " ".join(args), r
        assert len(r.stderr.strip().splitlines()) == 1 and why in r.stderr, r.stderr
    notbgzf = tmp_path / "x.bam"
    notbgzf.write_bytes(b"plain")
    r = subprocess.run([SHIM, "index", str(notbgzf)], env=env, capture_output=True, text=True)
    assert r.stdout.strip() == "real index %s" % notbgzf and "not BGZF" in r.stderr
