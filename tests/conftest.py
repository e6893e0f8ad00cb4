import gzip
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import ssq_testlib as T  # noqa: E402


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs an H100 (select with -m gpu)")


@pytest.fixture(scope="session")
def oracle():
    return T.Oracle()


@pytest.fixture(scope="session")
def hostsim(oracle):
    return T.HostSim(oracle)


@pytest.fixture(scope="session")
def ex_index(oracle, tmp_path_factory):
    """index of the reference's example FASTA (fixture copy), built by the oracle; returns the prefix"""
    d = tmp_path_factory.mktemp("ex")
    fa = str(d / "ex.fa")
    with open(fa, "wb") as f:
        f.write(gzip.open(os.path.join(T.GOLDEN, "ex_ref.fa.gz")).read())
    oracle.index_build(fa)
    return fa


@pytest.fixture(scope="session")
def ex_reads():
    names, seqs, quals = [], [], []
    with gzip.open(os.path.join(T.GOLDEN, "ex_reads_2k.fq.gz"), "rt") as f:
        for i, l in enumerate(f):
            l = l.rstrip("\n")
            if i % 4 == 0:
                names.append(l[1:].split()[0][:-2])
            elif i % 4 == 1:
                seqs.append(l)
            elif i % 4 == 3:
                quals.append(l)
    return names, seqs, quals


@pytest.fixture(scope="session")
def syn_index(oracle, tmp_path_factory):
    """seeded 3-contig synthetic genome (400 kb, planted repeats) + oracle-built index"""
    d = tmp_path_factory.mktemp("syn")
    g, bounds = T.synth_genome(400000, 7, n_contigs=3)
    fa = str(d / "syn.fa")
    T.write_fasta(fa, g, bounds)
    oracle.index_build(fa)
    return fa, g, bounds


@pytest.fixture(scope="session")
def ssq():
    return T.SSQ()


@pytest.fixture(scope="session")
def ssq_lib_cpu():
    """libssq.so loaded without a GPU: only its pure host helpers (BGZF framing, ABI checks) may be called through this"""
    import ctypes
    lib = ctypes.CDLL(T.SSQ_SO)
    lib.ssq_free.argtypes = [ctypes.c_void_p]
    lib.ssq_bgzf_compress.argtypes = [ctypes.c_char_p, ctypes.c_size_t, ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p]
    return lib
