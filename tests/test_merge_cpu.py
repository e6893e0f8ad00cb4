"""The merge of sorted BAM files (speedseq_b200/csrc/ssq_merge.cuh, with the BGZF member path of ssq_gunzip.cuh) run on the host
by tests/hostsim/merge_host.cpp (the same SSQ_HD phases, windowing and heap, host loops in place of the kernels), and the
oracle's independent sequential restatement (oracle/ssqo_merge.c), each compiled into a temporary directory: every fixture of
tests/golden/make_merge_golden.py gives the records and header the reference's sambamba wrote — from the oracle, and from the
host merge whatever the window size (one member per window, so records and headers are cut by window ends; a few members; the
whole file) and walker segment size.  The host's merged header (ssq_merge_header, no GPU needed) equals `merge -H`.  Each
refusal gives its message and the oracle refuses the same inputs.  The `sambamba` shim's `merge` without SSQ_MERGE_GPU=1, or
without a GPU, hands the call to the real sambamba with its arguments unchanged."""
import ctypes as C
import glob
import gzip
import os
import struct
import subprocess

import pytest

import ssq_testlib as T
from golden.make_bai_golden import bgzf, member, record
from golden.make_merge_golden import HD, bam, bam_header, sq

EDATA, EFORMAT, EINVAL = -9, -8, -4
RUNS = sorted(os.path.basename(p)[len("merge_"):-len(".records.gz")] for p in glob.glob(os.path.join(T.GOLDEN, "merge_*.records.gz")))
SHIM = os.path.join(T.ROOT, "speedseq_b200", "bin", "sambamba")


def inputs(run):
    case, order = run.rsplit("_", 1)
    return [os.path.join(T.GOLDEN, "merge_%s_%s.bam" % (case, c)) for c in order]


def want(run):
    base = os.path.join(T.GOLDEN, "merge_" + run)
    return open(base + ".header.txt", "rb").read(), gzip.open(base + ".records.gz").read(), open(base + ".H.txt", "rb").read()


def split(body):
    """uncompressed BAM -> (header text, records)"""
    lt = struct.unpack_from("<i", body, 4)[0]
    at = 8 + lt
    n_ref = struct.unpack_from("<i", body, at)[0]
    at += 4
    for _ in range(n_ref):
        at += 8 + struct.unpack_from("<i", body, at)[0]
    return body[8:8 + lt], body[at:]


def names(records):
    out, at = [], 0
    while at < len(records):
        out.append(records[at + 36:at + 36 + records[at + 12] - 1].decode())
        at += 4 + struct.unpack_from("<i", records, at)[0]
    return out


def cpaths(paths):
    return (C.c_char_p * len(paths))(*[os.fsencode(p) for p in paths])


@pytest.fixture(scope="module")
def merge_host(tmp_path_factory):
    so = os.path.join(str(tmp_path_factory.mktemp("merge_host")), "libmerge_host.so")
    subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-w", "-I", os.path.join(T.ROOT, "include"), "-o", so,
                    os.path.join(T.ROOT, "tests", "hostsim", "merge_host.cpp"), "-lz"], check=True)
    lib = C.CDLL(so)
    lib.hostsim_merge.argtypes = [C.c_void_p, C.c_int, C.c_size_t, C.c_size_t, C.c_void_p, C.c_void_p, C.c_char_p, C.c_size_t]
    lib.hostsim_merge_free.argtypes = [C.c_void_p]
    return lib


@pytest.fixture(scope="module")
def merge_oracle(tmp_path_factory):
    so = os.path.join(str(tmp_path_factory.mktemp("merge_oracle")), "libssqo_merge.so")
    subprocess.run(["gcc", "-O2", "-fPIC", "-shared", "-w", "-o", so, os.path.join(T.ROOT, "oracle", "ssqo_merge.c"), "-lz"], check=True)
    lib = C.CDLL(so)
    lib.ssqo_merge.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_char_p, C.c_size_t]
    return lib


def hostsim_merge(lib, paths, window=0, seg=0):
    """-> (rc, uncompressed merged file, message)"""
    out, n, err = C.c_void_p(), C.c_size_t(0), C.create_string_buffer(512)
    rc = lib.hostsim_merge(cpaths(paths), len(paths), window, seg, C.byref(out), C.byref(n), err, 512)
    data = C.string_at(out, n.value) if rc == 0 else b""
    if rc == 0:
        lib.hostsim_merge_free(out)
    return rc, data, err.value.decode()


def oracle_merge(lib, paths):
    """-> (rc, uncompressed merged file, message); the file is left to the process (test sizes)"""
    out, n, err = C.c_void_p(), C.c_size_t(0), C.create_string_buffer(512)
    rc = lib.ssqo_merge(cpaths(paths), len(paths), C.byref(out), C.byref(n), err, 512)
    return rc, C.string_at(out, n.value) if rc == 0 else b"", err.value.decode()


def test_fixtures_exist():
    cases = {r.rsplit("_", 1)[0] for r in RUNS}
    assert {"ties", "many", "holes", "unmapped", "bigrec", "ids", "hd14"} <= cases
    assert {"ties_012", "ties_210", "ties_102", "many_05", "many_257", "many_01234567"} <= set(RUNS)


@pytest.mark.parametrize("window,seg", [(0, 0), (1, 0), (1, 64), (2000, 97), (40000, 0)])
@pytest.mark.parametrize("run", RUNS)
def test_host_merge_gives_sambambas(merge_host, run, window, seg):
    rc, body, err = hostsim_merge(merge_host, inputs(run), window, seg)
    assert rc == 0, err
    h, r, hh = want(run)
    assert split(body) == (h, r)
    assert hh == h


@pytest.mark.parametrize("run", RUNS)
def test_oracle_gives_sambambas(merge_oracle, run):
    rc, body, err = oracle_merge(merge_oracle, inputs(run))
    assert rc == 0, err
    assert split(body) == want(run)[:2]


def test_the_order_rule_vectors(merge_host, merge_oracle):
    """the equal-key order of sambamba's NWayUnion, stated on three inputs"""
    v1 = "z0 x0 z1 x1 z2 x2 z3 x3 z4 y0 y1 y2 y3 x4 y4 x5 y5 x6 y6 x7 z5 z6 z7".split()
    v2 = "z0 y0 z1 y1 z2 y2 z3 y3 z4 x0 x1 x2 x3 x4 z5 x5 z6 x6 z7 x7 y4 y5 y6".split()
    for run, v in (("ties_012", v1), ("ties_210", v1), ("ties_102", v2)):
        assert names(want(run)[1]) == v, run
        assert names(split(hostsim_merge(merge_host, inputs(run), 1)[1])[1]) == v, run
        assert names(split(oracle_merge(merge_oracle, inputs(run))[1])[1]) == v, run


def test_a_window_end_after_every_record(merge_host, tmp_path):
    """the same records, one BGZF member per record: windows of one member end after every record"""
    for run in ("many_31570246", "unmapped_210", "holes_31024"):
        paths = []
        for k, p in enumerate(inputs(run)):
            t = gzip.open(p).read()
            lt = struct.unpack_from("<i", t, 4)[0]
            _, recs = split(t)
            hdr = t[:len(t) - len(recs)]
            parts, at = [hdr], 0
            while at < len(recs):
                n = 4 + struct.unpack_from("<i", recs, at)[0]
                parts.append(recs[at:at + n])
                at += n
            q = tmp_path / ("%s_%d.bam" % (run, k))
            q.write_bytes(b"".join(member(x) for x in parts) + member(b""))
            paths.append(str(q))
            assert lt >= 0
        rc, body, err = hostsim_merge(merge_host, paths, 1, 64)
        assert rc == 0, err
        assert split(body) == want(run)[:2]


@pytest.mark.skipif(not os.path.exists(T.SSQ_SO), reason="libssq.so is built by build()")
@pytest.mark.parametrize("run", RUNS)
def test_merged_header_on_the_host_is_merge_H(ssq_lib_cpu, run):
    L = ssq_lib_cpu
    L.ssq_merge_header.argtypes = [C.c_void_p, C.c_int, C.c_void_p]
    out = C.c_void_p()
    assert L.ssq_merge_header(cpaths(inputs(run)), len(inputs(run)), C.byref(out)) == 0
    text = C.string_at(out)
    L.ssq_free(out)
    assert text == want(run)[2]


REFS = [("m1", 5000000), ("m2", 300000)]


def refused(d):
    """(name, input paths, code, part of the message)"""
    def f(name, data):
        p = os.path.join(str(d), name + ".bam")
        open(p, "wb").write(data)
        return p
    ok = f("ok", bam([record("o%d" % i, 0, 0, 10 * i) for i in range(20)]))
    yield "one_input", [ok], EINVAL, "at least two inputs"
    yield "plain_gzip", [ok, f("gz", gzip.compress(bam_header(HD + sq())))], EDATA, "not BGZF"
    yield "not_so", [ok, f("noso", bam([], b"@HD\tVN:1.3\n" + sq()))], EFORMAT, "does not say SO:coordinate"
    yield "no_hd", [ok, f("nohd", bam([], sq()))], EFORMAT, "does not say SO:coordinate"
    yield "hd_differs", [ok, f("hd14", bam([], b"@HD\tVN:1.4\tSO:coordinate\n" + sq()))], EFORMAT, "@HD lines"
    yield "sq_differs", [ok, f("sq", bgzf(bam_header(HD + b"@SQ\tSN:m1\tLN:5000000\n", REFS[:1]), 0xff00))], EFORMAT, "@SQ dictionaries"
    rg = b"@RG\tID:g\tSM:a\n"
    yield "id_two_lines", [f("rg1", bam([], HD + sq() + rg)), f("rg2", bam([], HD + sq() + b"@RG\tID:g\tSM:b\n"))], EFORMAT, "two different lines"
    yield "other_line", [ok, f("xx", bam([], HD + sq() + b"@XY\tab\n"))], EFORMAT, "not merged"
    yield "unsorted", [ok, f("uns", bgzf(bam_header(HD + sq()) + record("a", 0, 0, 50) + record("b", 0, 0, 40), 0xff00))], EFORMAT, "not coordinate-sorted"
    yield "unsorted_ref", [ok, f("unsr", bgzf(bam_header(HD + sq()) + record("a", 0, 1, 5) + record("b", 0, 0, 40), 0xff00))], EFORMAT, "not coordinate-sorted"
    yield "nocoor_first", [ok, f("nc", bgzf(bam_header(HD + sq()) + record("a", 4, -1, -1, "*") + record("b", 0, 0, 40), 0xff00))], EFORMAT, "not coordinate-sorted"
    yield "ref_beyond", [ok, f("rb", bgzf(bam_header(HD + sq()) + record("a", 0, 2, 5), 0xff00))], EFORMAT, "not a reference of the header"
    yield "truncated_record", [ok, f("tr", bgzf(bam_header(HD + sq()) + record("a", 0, 0, 5)[:-3], 0xff00))], EFORMAT, "runs past the end of the file"
    yield "bad_block_size", [ok, f("bb", bgzf(bam_header(HD + sq()) + struct.pack("<i", 8) + b"\0" * 8, 0xff00))], EFORMAT, "not a BAM record"
    good = open(ok, "rb").read()
    bad = bytearray(good)
    bad[len(member(bam_header(HD + sq()) + b"".join(record("o%d" % i, 0, 0, 10 * i) for i in range(20)))) // 2] ^= 0x55
    yield "corrupt_member", [ok, f("cm", bytes(bad))], EDATA, "corrupt BGZF member"
    yield "truncated_member", [ok, f("tm", good[:-40])], EDATA, "truncated member"


def test_refusals(merge_host, merge_oracle, tmp_path):
    for name, paths, code, msg in refused(tmp_path):
        for w in (0, 1):
            rc, _, err = hostsim_merge(merge_host, paths, w, 64)
            assert rc == code and msg in err, (name, w, rc, err)
        assert oracle_merge(merge_oracle, paths)[0] != 0, name


@pytest.mark.skipif(not os.path.exists(SHIM), reason="the CLI shims are built by build()")
def test_shim_merge_goes_to_the_real_sambamba(tmp_path):
    """without SSQ_MERGE_GPU=1: the real sambamba, arguments unchanged, nothing on stderr; with it but no GPU: one stderr line,
    then the real sambamba with the same arguments; `merge -H` is answered on the host"""
    real = tmp_path / "real.sh"
    real.write_text("#!/bin/sh\necho \"real $*\"\n")
    real.chmod(0o755)
    run = "ties_012"
    args = ["merge", "-t", "4", str(tmp_path / "out.bam")] + inputs(run)
    env = dict(os.environ, SSQ_SAMBAMBA_REAL=str(real))
    env.pop("SSQ_MERGE_GPU", None)
    r = subprocess.run([SHIM] + args, env=env, capture_output=True, text=True)
    assert r.returncode == 0 and r.stdout.strip() == "real " + " ".join(args) and not r.stderr, r
    env["SSQ_MERGE_GPU"] = "1"
    for a, why in ((["merge", "-F", "mapping_quality > 0", str(tmp_path / "out.bam")] + inputs(run), "option -F"),
                   (["merge", str(tmp_path / "out.bam"), inputs(run)[0]], "at least two inputs")):
        r = subprocess.run([SHIM] + a, env=env, capture_output=True, text=True)
        assert r.returncode == 0 and r.stdout.strip() == "real " + " ".join(a), r
        assert len(r.stderr.strip().splitlines()) == 1 and why in r.stderr, r.stderr
    r = subprocess.run([SHIM, "merge", "-H", str(tmp_path / "out.bam")] + inputs(run), env=env, capture_output=True)
    assert r.returncode == 0 and r.stdout == want(run)[2], r
    if not T.gpu_visible():
        r = subprocess.run([SHIM] + args, env=env, capture_output=True, text=True)
        assert r.returncode == 0 and r.stdout.strip() == "real " + " ".join(args), r
        assert len(r.stderr.strip().splitlines()) == 1 and "no usable GPU" in r.stderr, r.stderr
    assert not os.path.exists(tmp_path / "out.bam") and not glob.glob(str(tmp_path / "out.bam*"))
