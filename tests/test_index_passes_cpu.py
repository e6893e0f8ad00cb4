"""The multi-pass suffix sort of `ssq_index_build_ex` (path 2, speedseq_b200/csrc/ssq_sapass.cuh) run on the host by
tests/hostsim/sapass_host.cpp: the same driver, planners and per-element bodies, host loops and a stable sort in place of the
kernels and CUB; compiled into a temporary directory.  From the .pac the oracle writes, it must give the oracle's .bwt and .sa
(the goldens for the example FASTA) for budgets that make one pass, several passes and one-group chunks, on inputs chosen to
stress short suffixes, long repeats and range boundaries.  Each case asserts the stats it must reach, so that an unlucky input
fails instead of testing less."""
import ctypes as C
import gzip
import hashlib
import json
import math
import os
import subprocess

import numpy as np
import pytest

import ssq_testlib as T

SP_K = 28  # symbols of the first sort: round r (1-based) resolves common prefixes shorter than SP_K * 2^r


class Stats(C.Structure):
    _fields_ = [("path", C.c_int32), ("pad", C.c_int32)] + [(k, C.c_int64) for k in
                ("passes", "rounds", "chunks", "unresolved_first", "largest_group", "oversize_groups", "peak_device_bytes", "ranges")]


def stats_dict(st):
    return {k: getattr(st, k) for k, _ in Stats._fields_ if k != "pad"}


def build_sapass_host(d):
    so = os.path.join(str(d), "libsapass_host.so")
    subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-w", "-I", os.path.join(T.ROOT, "include"), "-o", so,
                    os.path.join(T.ROOT, "tests", "hostsim", "sapass_host.cpp")], check=True)
    lib = C.CDLL(so)
    lib.hostsim_sapass.argtypes = [C.c_char_p, C.c_size_t, C.c_int64, C.c_char_p, C.c_uint64, C.c_uint64, C.POINTER(Stats)]
    lib.hostsim_error.restype = C.c_char_p
    return lib


@pytest.fixture(scope="session")
def sapass_host(tmp_path_factory):
    return build_sapass_host(tmp_path_factory.mktemp("sapass_host"))


def read_pac(path):
    """PREFIX.pac -> (packed bytes, l_pac): the last byte is l_pac % 4, preceded by a 0 byte when that is 0"""
    raw = open(path, "rb").read()
    ct = raw[-1]
    data = raw[:-2] if ct == 0 else raw[:-1]
    l_pac = len(data) * 4 if ct == 0 else (len(data) - 1) * 4 + ct
    return data, l_pac


def host_build(lib, pac_path, prefix, work, chunk_work=0):
    data, l_pac = read_pac(pac_path)
    st = Stats()
    rc = lib.hostsim_sapass(data, len(data), l_pac, prefix.encode(), work, chunk_work, C.byref(st))
    assert rc != 99, "an open member of round h had i + h > n"
    assert rc == 0, (rc, lib.hostsim_error().decode())
    return stats_dict(st)


def budgets(n1):
    """name -> (work bytes, chunk bytes): one pass; several passes; eight or more finalisation ranges; every chunk a single group
    (through the chunk budget alone); and, for genomes of a few kb, a work budget so small that every chunk holds one group and
    every pass one bucket, which the device reaches too"""
    b = {"one_pass": (1 << 30, 0), "passes": (40 * max(64, n1 // 5), 0), "ranges": (11 * max(128, n1 // 8), 0),
         "one_group_chunks": (40 * max(64, n1 // 3), 96)}
    if n1 <= 8200:
        b["tiny"] = (96, 0)
    return b


def fin_rows(work):
    """rows per finalisation range for a work budget (sp_build: SP_FIN_ROW_BYTES = 11, a multiple of 128, at least 128)"""
    return max(128, work // 11) & ~127


def primary_row(prefix):
    return int.from_bytes(open(prefix + ".bwt", "rb").read(8), "little")


def rounds_for(lcp):
    """doubling rounds needed to separate two suffixes with a common prefix of lcp symbols"""
    return max(0, math.ceil(math.log2((lcp + 1) / SP_K))) if lcp >= SP_K else 0


# ------------------------------------------------------------------------------------ corpus ----
def _plant_ambiguity(path, seed):
    txt = open(path).read().split("\n")
    rng = np.random.default_rng(seed)
    for k in rng.integers(1, len(txt) - 1, 6):
        if txt[k] and not txt[k].startswith(">"):
            txt[k] = txt[k][:5] + "NNNNnnRY" + txt[k][13:]
    open(path, "w").write("\n".join(txt))


def corpus():
    """name -> (writer(path), common-prefix length the genome is known to hold, or 0): the synthetic set of test_gpu_index
    (N runs, ambiguity codes, l_pac % 4 in {0,1,2,3}, several contigs), an exact 64 kb duplication, a 20 kb poly-A run, tandem
    arrays of period 1-7, a single-base genome and genomes of 1-4 bp"""
    c = {}
    for n, nc, seed in [(1000, 1, 1), (4097, 3, 2), (250000, 5, 3), (1 << 20, 2, 4), (4098, 2, 5), (4099, 1, 6)]:
        def w(p, n=n, nc=nc, seed=seed):
            g, bounds = T.synth_genome(n, seed, n_contigs=nc)
            T.write_fasta(p, g, bounds)
            _plant_ambiguity(p, seed)
        c["synth_%d_%d" % (n, nc)] = (w, 0)

    def dup(p):
        g, bounds = T.synth_genome(200000, 21, n_contigs=2)
        g[120000:184000] = g[10000:74000]
        T.write_fasta(p, g, bounds)
    c["dup_64kb"] = (dup, 64000)

    def polya(p):
        g, bounds = T.synth_genome(60000, 22)
        g[20000:40000] = 0
        T.write_fasta(p, g, bounds)
    c["polyA_20kb"] = (polya, 19999)
    for per in range(1, 8):
        def tandem(p, per=per):
            rng = np.random.default_rng(30 + per)
            g = rng.integers(0, 4, 12000).astype(np.uint8)
            unit = rng.integers(0, 4, per).astype(np.uint8)
            if per > 1:
                unit[0], unit[1] = 0, 1  # a period-1 unit would make every period the same run
            g[3000:9000] = np.tile(unit, 6000 // per + 1)[:6000]
            T.write_fasta(p, g, np.array([0, 12000]))
        c["tandem_p%d" % per] = (tandem, 6000 - per - 1)

    def single(p):
        T.write_fasta(p, np.zeros(3000, np.uint8), np.array([0, 3000]))
    c["single_base"] = (single, 2998)
    for L in range(1, 5):
        def tiny(p, L=L):
            open(p, "w").write(">t\n" + "ACGT"[:L][::-1] + "\n")
        c["genome_%dbp" % L] = (tiny, 0)
    return c


CORPUS = corpus()


def oracle_index(oracle, writer, d):
    fa = os.path.join(str(d), "ref.fa")
    writer(fa)
    oracle.index_build(fa)
    return fa


def test_host_restatement_gives_the_example_goldens(oracle, sapass_host, tmp_path):
    fa = str(tmp_path / "ex.fa")
    open(fa, "wb").write(gzip.open(os.path.join(T.GOLDEN, "ex_ref.fa.gz")).read())
    oracle.index_build(fa)
    gold = json.load(open(os.path.join(T.GOLDEN, "ex_index.sha256.json")))
    assert hashlib.sha256(open(fa + ".pac", "rb").read()).hexdigest() == gold["pac"]["sha256"]
    n1 = 2 * read_pac(fa + ".pac")[1] + 1
    seen = {}
    for name, (work, cw) in budgets(n1).items():
        pre = str(tmp_path / name)
        seen[name] = host_build(sapass_host, fa + ".pac", pre, work, cw)
        for ext in ("bwt", "sa"):
            data = open(pre + "." + ext, "rb").read()
            assert len(data) == gold[ext]["size"] and hashlib.sha256(data).hexdigest() == gold[ext]["sha256"], (name, ext)
    assert seen["one_pass"]["passes"] == 1 and seen["passes"]["passes"] > 1
    # several finalisation ranges, and the '$' row before the last of them: range boundaries after it see the shifted rows
    assert seen["one_pass"]["ranges"] == 1 and seen["ranges"]["ranges"] >= 8
    assert primary_row(fa) < (seen["ranges"]["ranges"] - 1) * fin_rows(budgets(n1)["ranges"][0])
    assert seen["one_group_chunks"]["oversize_groups"] >= 1
    # one chunk per group: at least as many chunks as the first round has groups, more than with the roomy budget
    assert seen["one_group_chunks"]["chunks"] > seen["one_pass"]["chunks"] >= 1
    for s in seen.values():  # the planners change how the work is cut, never what is found
        assert (s["rounds"], s["unresolved_first"], s["largest_group"]) == (seen["one_pass"]["rounds"], seen["one_pass"]["unresolved_first"], seen["one_pass"]["largest_group"])


@pytest.mark.parametrize("case", sorted(CORPUS))
def test_host_restatement_equals_oracle(oracle, sapass_host, tmp_path, case):
    writer, lcp = CORPUS[case]
    fa = oracle_index(oracle, writer, tmp_path)
    want = {ext: open(fa + "." + ext, "rb").read() for ext in ("bwt", "sa")}
    n1 = 2 * read_pac(fa + ".pac")[1] + 1
    seen = {}
    for name, (work, cw) in budgets(n1).items():
        pre = str(tmp_path / name)
        seen[name] = s = host_build(sapass_host, fa + ".pac", pre, work, cw)
        for ext in ("bwt", "sa"):
            assert open(pre + "." + ext, "rb").read() == want[ext], (name, ext)
        assert s["rounds"] >= rounds_for(lcp), (name, s)
    if n1 > 64 * 5 * 2:
        assert seen["passes"]["passes"] > 1, seen
    if n1 > 128 * 8 * 2:
        assert seen["ranges"]["ranges"] >= 8, seen
    if "tiny" in seen and lcp >= 1000:
        assert seen["tiny"]["oversize_groups"] >= 1 and seen["tiny"]["passes"] > 1, seen
    if lcp >= 1000:
        assert seen["one_group_chunks"]["oversize_groups"] >= 1, seen
    if case == "dup_64kb":
        assert seen["one_pass"]["rounds"] >= 11
