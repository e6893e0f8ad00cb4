"""The one-sector rank query of the seeding (ScalarFm::occ4_pair in speedseq_b200/csrc/ssq_dev.cuh) and the k-mer table in the
phase-split seeding's forward walks, checked on the host: the paired query (tests/hostsim/seed_sector_host.cpp) must give exactly
the counts of two single queries wherever the two rows and the primary ('$') row fall, and the split seeding of the test-only
harness tests/hostsim with the table must give the oracle's intervals."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import ssq_testlib as T


@pytest.fixture(scope="module")
def pair_lib(oracle, tmp_path_factory):
    """tests/hostsim/seed_sector_host.cpp -> a shared library in a temporary directory"""
    so = str(tmp_path_factory.mktemp("seed_sector") / "libseedsector.so")
    odir = os.path.join(T.ROOT, "oracle")
    subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-w", "-o", so, os.path.join(T.ROOT, "tests", "hostsim", "seed_sector_host.cpp"),
                    "-L" + odir, "-lssqo", "-Wl,-rpath," + odir], check=True)
    lib = C.CDLL(so)
    f = lib.seed_sector_pair_check
    f.restype = C.c_longlong
    f.argtypes = [C.c_void_p, C.c_ulonglong, C.c_ulonglong, C.c_ulonglong, C.c_int, C.POINTER(C.c_ulonglong), C.POINTER(C.c_ulonglong)]
    return lib


def _pair_check(lib, idx, primary, lo, hi, span):
    one, two = C.c_ulonglong(), C.c_ulonglong()
    bad = lib.seed_sector_pair_check(C.c_void_p(idx), primary, lo, hi, span, C.byref(one), C.byref(two))
    return bad, one.value, two.value


@pytest.mark.parametrize("pos", [0, 1, 31, 32, 62, 63])
def test_paired_query_equals_two_queries(oracle, pair_lib, syn_index, pos):
    """primary at every position class of its 64-row block (first, second, middle, last rows); every interval [k0, k1] around it
    and across the neighbouring block boundaries, the one starting at row 0 included"""
    fa = syn_index[0]
    idx = oracle.load(fa)
    n = oracle.info(idx, 1)  # rows - 1 (seq_len)
    blk = (n // 2) // 64 * 64
    primary = blk + pos
    bad, one, two = _pair_check(pair_lib, idx, primary, primary - 130, primary + 130, 140)
    assert bad == 0
    assert one > 0 and two > 0
    bad, one, two = _pair_check(pair_lib, idx, primary, 0, 70, 70)  # intervals starting at row 0 (no row before them)
    assert bad == 0


def test_paired_query_real_primary(oracle, pair_lib, syn_index):
    fa = syn_index[0]
    idx = oracle.load(fa)
    p = oracle.info(idx, 2)
    bad, one, two = _pair_check(pair_lib, idx, p, max(0, p - 200), p + 200, 200)
    assert bad == 0 and one > 0 and two > 0


def _corner_reads(g, bounds):
    acgt = "ACGT"
    head = "".join(acgt[x] for x in g[:150])  # the text's first suffix: its row is the primary row
    tail = "".join(acgt[x] for x in g[int(bounds[-1]) - 150:int(bounds[-1])])
    rc = tail[::-1].translate(str.maketrans("ACGT", "TGCA"))
    return [head, head[:40], rc, "", "A", "N" * 30, "N" * 10 + head[10:], head[:70] + "NN" + head[72:], "AC" * 70, "A" * 150, "ACGT" * 37,
            "T" * 100, "AAG" * 50, "CA" * 30 + "G" * 30 + "TTA" * 30]


@pytest.mark.parametrize("kmer", [None, "8", "10"])
def test_split_seeding_with_table(oracle, hostsim, syn_index, monkeypatch, kmer):
    """the phase-split form (k_smem_fwd / k_smem_bwd / k_smem_p3) with the forward walks' short strings from the table"""
    monkeypatch.setenv("HOSTSIM_SPLIT", "1")
    if kmer:
        monkeypatch.setenv("HOSTSIM_KMER", kmer)
    fa, g, bounds = syn_index
    idx = oracle.load(fa)
    names, seqs, quals = T.simulate_pairs(g, bounds, 400, 150, 23, err=0.015, indel=0.003, n_frac=0.004)
    seq, off = T.encode_reads(seqs + _corner_reads(g, bounds))
    hostsim.lib.hostsim_ext_hist_reset()
    a, ao = oracle.smem_batch(idx, seq, off)
    b, bo = hostsim.smem_batch(idx, seq, off)
    assert np.array_equal(ao, bo) and np.array_equal(a, b)
    hostsim.lib.hostsim_table_hits.restype = C.c_ulonglong
    hits = hostsim.lib.hostsim_table_hits()
    assert (hits > 0) == bool(kmer)
