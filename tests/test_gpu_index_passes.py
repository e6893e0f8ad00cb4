"""The multi-pass device suffix sort (`ssq_index_build_ex` path 2) on the GPU: the corpus of test_index_passes_cpu gives the
oracle's files and the host restatement's stats for the same budgets; the example FASTA gives the goldens with the budget
taken from free memory; an index it built aligns like the oracle; the `bwa` shim names the path it took."""
import gzip
import hashlib
import json
import os
import subprocess

import numpy as np
import pytest

import ssq_testlib as T
from test_index_passes_cpu import CORPUS, budgets, host_build, oracle_index, read_pac, sapass_host  # noqa: F401  (fixture)

pytestmark = pytest.mark.gpu
EXTS = ("amb", "ann", "pac", "bwt", "sa")
SAME = ("passes", "rounds", "chunks", "unresolved_first", "largest_group", "oversize_groups", "ranges")


@pytest.mark.parametrize("case", sorted(CORPUS))
def test_gpu_passes_equal_oracle_and_host_stats(ssq, oracle, sapass_host, tmp_path, case):
    writer, _ = CORPUS[case]
    fa = oracle_index(oracle, writer, tmp_path)
    n1 = 2 * read_pac(fa + ".pac")[1] + 1
    for name, (work, cw) in budgets(n1).items():
        if cw:  # the chunk-only budget is a knob of the host restatement; "tiny" gives the device one-group chunks on small genomes
            continue
        pre = str(tmp_path / ("dev_" + name))
        st = ssq.index_build_ex(fa, pre, path=2, work_bytes=work)
        assert st["path"] == 2
        for ext in EXTS:
            assert open(pre + "." + ext, "rb").read() == open(fa + "." + ext, "rb").read(), (name, ext)
        want = host_build(sapass_host, fa + ".pac", str(tmp_path / ("host_" + name)), work)
        assert {k: st[k] for k in SAME} == {k: want[k] for k in SAME}, (name, st, want)
        assert st["peak_device_bytes"] >= want["peak_device_bytes"]


def test_gpu_passes_golden_with_free_memory_budget(ssq, tmp_path):
    fa = str(tmp_path / "ex.fa")
    open(fa, "wb").write(gzip.open(os.path.join(T.GOLDEN, "ex_ref.fa.gz")).read())
    st = ssq.index_build_ex(fa, path=2, work_bytes=0)
    assert st["path"] == 2 and st["passes"] == 1 and st["peak_device_bytes"] > 0
    gold = json.load(open(os.path.join(T.GOLDEN, "ex_index.sha256.json")))
    for ext, g in gold.items():
        data = open(fa + "." + ext, "rb").read()
        assert len(data) == g["size"] and hashlib.sha256(data).hexdigest() == g["sha256"], ext


def test_gpu_auto_takes_the_device_and_host_path_agrees(ssq, tmp_path):
    g, bounds = T.synth_genome(50000, 9)
    fa = str(tmp_path / "s.fa")
    T.write_fasta(fa, g, bounds)
    assert ssq.index_build_ex(fa)["path"] == 2
    with pytest.raises(RuntimeError):
        ssq.index_build_ex(fa, str(tmp_path / "x"), path=1)
    assert ssq.index_build_ex(fa, str(tmp_path / "h"), path=3)["path"] == 3
    for ext in EXTS:
        assert open(fa + "." + ext, "rb").read() == open(str(tmp_path / "h") + "." + ext, "rb").read(), ext


def test_gpu_passes_index_then_align(ssq, oracle, tmp_path):
    g, bounds = T.synth_genome(300000, 12, n_contigs=2)
    fa = str(tmp_path / "x.fa")
    T.write_fasta(fa, g, bounds)
    st = ssq.index_build_ex(fa, path=2, work_bytes=40 * 150000)
    assert st["passes"] > 1
    h = ssq.index_load(fa)
    oidx = oracle.load(fa)
    names, seqs, quals = T.simulate_pairs(g, bounds, 500, 150, 3)
    seq, off = T.encode_reads(seqs)
    a, ao = oracle.align_batch(oidx, seq, off)
    b, bo = ssq.align_batch(h, seq, off)
    assert np.array_equal(ao, bo) and np.array_equal(a, b)
    ssq.index_free(h)


def test_gpu_bwa_shim_index_names_its_path(tmp_path):
    fa = str(tmp_path / "ex.fa")
    open(fa, "wb").write(gzip.open(os.path.join(T.GOLDEN, "ex_ref.fa.gz")).read())
    r = subprocess.run([os.path.join(T.ROOT, "speedseq_b200", "bin", "bwa"), "index", fa], check=True, timeout=300,
                       stdout=subprocess.PIPE, stderr=subprocess.PIPE)
    assert r.stdout == b""
    assert b"[bwa_index] device suffix sort: 1 passes" in r.stderr, r.stderr
    gold = json.load(open(os.path.join(T.GOLDEN, "ex_index.sha256.json")))
    for ext, g in gold.items():
        assert hashlib.sha256(open(fa + "." + ext, "rb").read()).hexdigest() == g["sha256"], ext
