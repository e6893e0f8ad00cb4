"""The device BGZF encoder (speedseq_b200/csrc/ssq_bgzf.cuh) run on the host by tests/hostsim/bgzf_host.cpp (same SSQ_HD phases,
thread loops in place of the CTA; compiled into a temporary directory): every file it makes is a well-formed BGZF file that
decompresses to the input, cut into the same blocks as ssq_bgzf_compress, and no more than 10 % larger than zlib level 1 on real
BAM records."""
import ctypes as C
import gzip
import os
import random
import struct
import subprocess
import zlib

import pytest

import ssq_testlib as T

REAL_SAMBAMBA = os.path.join(T.ROOT, "oracle", "_ref", "stage", "src", "sambamba")


def de_bruijn_text():
    """every 3-byte window distinct (de Bruijn sequence over 26 letters): deflate finds no match in it"""
    k, n, a, seq = 26, 3, [0] * 78, []

    def db(t, p):
        if t > n:
            if n % p == 0:
                seq.extend(a[1:p + 1])
        else:
            a[t] = a[t - p]
            db(t + 1, p)
            for j in range(a[t - p] + 1, k):
                a[t] = j
                db(t + 1, t)
    db(1, 1)
    s = bytes(97 + x for x in seq)
    return s + s[:2]


def inputs():
    rnd = random.Random(11)
    ex = gzip.open(os.path.join(T.GOLDEN, "ex_bam_main.records.gz")).read()
    return {
        "empty": b"", "one_byte": b"\x07", "exactly_ff00": ex[:0xff00], "ff00_plus_1": ex[:0xff01],
        "zeros_1MB": bytes(1 << 20), "random_1MB": bytes(rnd.getrandbits(8) for _ in range(1 << 20)),
        "no_3byte_repeats": de_bruijn_text(), "one_symbol": b"Q" * 300001,
        "ex_bam_main": ex, "syn_bam_main": gzip.open(os.path.join(T.GOLDEN, "syn_bam_main.records.gz")).read(),
    }


def build_bgzf_host(d):
    """tests/hostsim/bgzf_host.cpp -> a shared library in directory d (the encoder's SSQ_HD phases compiled for the host)"""
    so = os.path.join(str(d), "libbgzf_host.so")
    subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-w", "-I", os.path.join(T.ROOT, "include"), "-o", so,
                    os.path.join(T.ROOT, "tests", "hostsim", "bgzf_host.cpp")], check=True)
    return C.CDLL(so)


@pytest.fixture(scope="session")
def bgzf_host(tmp_path_factory):
    return build_bgzf_host(tmp_path_factory.mktemp("bgzf_host"))


def hostsim_bgzf(lib, data, level=6, with_eof=1):
    lib.hostsim_bgzf.argtypes = [C.c_char_p, C.c_size_t, C.c_int, C.c_int, C.c_void_p, C.c_void_p]
    lib.hostsim_free.argtypes = [C.c_void_p]
    out, n = C.c_void_p(), C.c_size_t(0)
    assert lib.hostsim_bgzf(data, len(data), level, with_eof, C.byref(out), C.byref(n)) == 0
    r = C.string_at(out, n.value)
    lib.hostsim_free(out)
    return r


def zlib_bgzf(lib_cpu, data, level, with_eof=1):
    out, n = C.c_void_p(), C.c_size_t(0)
    assert lib_cpu.ssq_bgzf_compress(data, len(data), level, with_eof, C.byref(out), C.byref(n)) == 0
    r = C.string_at(out, n.value)
    lib_cpu.ssq_free(out)
    return r


def members(f):
    """[(deflate bytes, payload CRC-32, ISIZE)] of a BGZF file; asserts every member is well formed"""
    out, p = [], 0
    while p < len(f):
        assert f[p:p + 4] == b"\x1f\x8b\x08\x04" and f[p + 10:p + 12] == b"\x06\x00" and f[p + 12:p + 16] == b"BC\x02\x00", p
        bsize = struct.unpack("<H", f[p + 16:p + 18])[0] + 1
        assert bsize <= 65536 and p + bsize <= len(f)
        crc, isize = struct.unpack("<II", f[p + bsize - 8:p + bsize])
        out.append((f[p + 18:p + bsize - 8], crc, isize))
        p += bsize
    assert p == len(f)
    return out


def check_file(f, data, ref):
    """f decompresses to data, every member's CRC-32 is that of its payload, the block sizes are those of ref (zlib framing)"""
    assert gzip.decompress(f) == data
    ms, at = members(f), 0
    for d, crc, isize in ms:
        payload = zlib.decompress(d, -15)
        assert len(payload) == isize and zlib.crc32(payload) == crc
        at += isize
    assert at == len(data)
    assert [m[2] for m in ms] == [m[2] for m in members(ref)]
    assert f[-28:] == ref[-28:] and ms[-1][2] == 0  # the EOF block
    return ms


@pytest.mark.parametrize("name", list(inputs()))
def test_hostsim_encoder_makes_valid_bgzf(bgzf_host, ssq_lib_cpu, name):
    data = inputs()[name]
    f = hostsim_bgzf(bgzf_host, data)
    ms = check_file(f, data, zlib_bgzf(ssq_lib_cpu, data, 6))
    btypes = {(m[0][0] >> 1) & 3 for m in ms[:-1]}
    if name == "random_1MB":
        assert btypes == {0} and len(f) <= len(data) + 31 * len(ms) + 28  # stored: random bytes never expand beyond the framing
    if name == "no_3byte_repeats":
        assert btypes == {2}  # a dynamic block whose distance tree declares one unused code
    if name in ("zeros_1MB", "one_symbol"):
        assert len(f) < len(data) // 100
    assert hostsim_bgzf(bgzf_host, data, level=0) == hostsim_bgzf(bgzf_host, data, level=0)
    f0 = hostsim_bgzf(bgzf_host, data, level=0)
    assert {(m[0][0] >> 1) & 3 for m in check_file(f0, data, zlib_bgzf(ssq_lib_cpu, data, 0))[:-1]} <= {0}
    assert hostsim_bgzf(bgzf_host, data, level=1) == f == hostsim_bgzf(bgzf_host, data, level=9)  # one effort level for 1-9


@pytest.mark.parametrize("prefix", ["ex", "syn"])
def test_ratio_on_bam_records_against_zlib(bgzf_host, ssq_lib_cpu, prefix):
    data = gzip.open(os.path.join(T.GOLDEN, "%s_bam_main.records.gz" % prefix)).read()
    n = len(hostsim_bgzf(bgzf_host, data))
    z1, z6 = len(zlib_bgzf(ssq_lib_cpu, data, 1)), len(zlib_bgzf(ssq_lib_cpu, data, 6))
    print("%s_bam_main: %d bytes -> device encoder %d (%.3f), zlib -1 %d (%.3f), zlib -6 %d (%.3f); %.3f x level 1, %.3f x level 6"
          % (prefix, len(data), n, n / len(data), z1, z1 / len(data), z6, z6 / len(data), n / z1, n / z6))
    assert n <= 1.10 * z1


@pytest.mark.skipif(not os.access(REAL_SAMBAMBA, os.X_OK), reason="the reference's sambamba is not staged under oracle/_ref")
def test_reference_sambamba_reads_the_encoded_bam(bgzf_host, ssq_lib_cpu, tmp_path):
    """header + golden records encoded by the device encoder's bodies: speedseq's own sambamba counts every record"""
    from test_bam_golden import golden, split_records
    text = open(os.path.join(T.GOLDEN, "ex_bam_header.txt"), "rb").read()
    refs = [l.split(b"\t") for l in text.splitlines() if l.startswith(b"@SQ")]
    hdr = b"BAM\x01" + struct.pack("<i", len(text)) + text + struct.pack("<i", len(refs))
    for r in refs:
        nm = next(f[3:] for f in r if f.startswith(b"SN:")) + b"\0"
        hdr += struct.pack("<i", len(nm)) + nm + struct.pack("<i", int(next(f[3:] for f in r if f.startswith(b"LN:"))))
    recs = golden("main")
    path = str(tmp_path / "dev.bam")
    open(path, "wb").write(hostsim_bgzf(bgzf_host, hdr + recs))
    n = subprocess.run([REAL_SAMBAMBA, "view", "-c", path], stdout=subprocess.PIPE, check=True).stdout
    assert int(n) == len(split_records(recs))


@pytest.mark.skipif(T.gpu_visible(), reason="box has a GPU")
def test_no_gpu_no_device_bgzf(ssq_lib_cpu, tmp_path):
    h = C.c_void_p()
    ssq_lib_cpu.ssq_last_error.restype = C.c_char_p
    assert ssq_lib_cpu.ssq_bgzf_create(0, C.byref(h)) == -1 and b"no CPU path" in ssq_lib_cpu.ssq_last_error()
    shim = os.path.join(T.ROOT, "speedseq_b200", "bin", "sambamba")
    stream = b"@SQ\tSN:c1\tLN:100\n@CO\tssq-bam-runs-v1\n"
    p = subprocess.run([shim, "sort", "-t", "2", "-o", str(tmp_path / "o.bam"), "/dev/stdin"], input=stream, stdout=subprocess.PIPE, stderr=subprocess.PIPE,
                       env=dict(os.environ, SSQ_BGZF_GPU="1"), timeout=60)
    assert p.returncode != 0 and b"SSQ_BGZF_GPU" in p.stderr
    p = subprocess.run([shim, "sort", "-t", "2", "-o", str(tmp_path / "o.bam"), "/dev/stdin"], input=stream, stdout=subprocess.PIPE, stderr=subprocess.PIPE, timeout=60)
    assert p.returncode == 0  # without the variable nothing needs a GPU
