"""The merge of sorted BAM files on the device (ssq_merge_*, csrc/ssq_merge.cu): every fixture of tests/golden/make_merge_golden.py
(records and header written by the reference's sambamba) at several window sizes, with the output handed back and compressed on
the device; the same refusals and messages as the host restatement (tests/test_merge_cpu.py); seven larger inputs through
windows of a few members against the oracle; the `sambamba` shim's `merge` of tools/merge_bench.py's inputs (bench records split
by a random read group into 2, 3 and 7 files) with host and device BGZF, its .bai against the staged sambamba's index of the same file, and a refused input that leaves the staged sambamba's file and none of the shim's."""
import glob
import gzip
import os
import random
import shutil
import subprocess

import pytest

try:  # before anything loads libssq: torch must bring in its own NCCL first
    import torch
except ImportError:
    torch = None

import ssq_testlib as T
from golden.make_bai_golden import bgzf, record
from golden.make_merge_golden import HD, bam, bam_header, sq
from test_merge_cpu import RUNS, SHIM, hostsim_merge, inputs, merge_host, merge_oracle, oracle_merge, refused, split, want  # noqa: F401  (fixtures)

pytestmark = pytest.mark.gpu
REAL = os.path.join(T.ROOT, "oracle", "_ref", "stage", "src", "sambamba")
need_real = pytest.mark.skipif(not os.access(REAL, os.X_OK), reason="speedseq's own sambamba is not staged under oracle/_ref (build() stages it from a speedseq checkout)")


@pytest.fixture(scope="module")
def merges(ssq):
    h = {w: ssq.merge_create(0, w) for w in (0, 1, 3000)}
    yield h
    for m in h.values():
        ssq.merge_free(m)


def test_device_gives_the_fixtures(ssq, merges):
    for run in RUNS:
        for w, m in merges.items():
            rc, body, n = ssq.merge_run(m, inputs(run))
            assert rc == 0, (run, w, ssq.err())
            assert split(body) == want(run)[:2], (run, w)


def test_device_bgzf_output(ssq, merges):
    z = ssq.bgzf_create(0)
    try:
        for run in RUNS:
            rc, data, n = ssq.merge_run(merges[1], inputs(run), z, 6)
            assert rc == 0, ssq.err()
            assert split(gzip.decompress(data)) == want(run)[:2], run
    finally:
        ssq.bgzf_free(z)


def test_device_refuses_what_the_host_refuses(ssq, merges, merge_host, tmp_path):  # noqa: F811
    for name, paths, code, msg in refused(tmp_path):
        for w, m in merges.items():
            rc, _, _ = ssq.merge_run(m, paths)
            err = ssq.err()
            hrc, _, herr = hostsim_merge(merge_host, paths, w, 0)
            assert rc == code == hrc and msg in err and err.endswith(herr), (name, w, rc, err, herr)


def seven_inputs(d, n_per=40000, seed=3):
    R = random.Random(seed)
    paths = []
    for k in range(7):
        recs = [record("s%d_%d" % (k, i), R.choice([0, 16, 99, 147, 163]), R.choice([0, 0, 0, 1]), R.randrange(0, 300000) // 7 * 7, "%dM" % R.randint(30, 150))
                for i in range(n_per)]
        recs += [record("s%d_u%d" % (k, i), 77, -1, -1, "*") for i in range(R.randint(0, 500))]
        p = os.path.join(str(d), "in%d.bam" % k)
        open(p, "wb").write(bam(recs, size=R.choice([3000, 20000, 0xff00])))
        paths.append(p)
    return paths


def test_seven_inputs_through_small_windows(ssq, merge_oracle, tmp_path):  # noqa: F811
    paths = seven_inputs(tmp_path)
    orc, want_body, err = oracle_merge(merge_oracle, paths)
    assert orc == 0, err
    for w in (1, 100000, 0):
        m = ssq.merge_create(0, w)
        try:
            rc, body, n = ssq.merge_run(m, paths)
            assert rc == 0, ssq.err()
            assert body == want_body, w
            assert all(t >= 0 for t in ssq.merge_times(m))
        finally:
            ssq.merge_free(m)


@pytest.fixture(scope="module")
def split_bench(ssq, tmp_path_factory):
    """tools/merge_bench.py's inputs at a small size: bai_bench's records split by a random read group into 2, 3 and 7 files"""
    import sys
    sys.path.insert(0, os.path.join(T.ROOT, "tools"))
    from merge_bench import split_inputs
    return split_inputs(ssq, tmp_path_factory.mktemp("split"), 0.08)


@need_real
@pytest.mark.parametrize("bgzf_gpu", ["0", "1"])
def test_shim_merge_equals_the_staged_sambamba(split_bench, tmp_path, bgzf_gpu):
    env = dict(os.environ, SSQ_SAMBAMBA_REAL=REAL, SSQ_MERGE_GPU="1", SSQ_BGZF_GPU=bgzf_gpu, SSQ_MERGE_WINDOW="1000000")
    for k, args in split_bench.items():
        ours, theirs = str(tmp_path / "ours.bam"), str(tmp_path / "theirs.bam")
        r = subprocess.run([SHIM, "merge", "-t", "16", ours] + args, env=env, capture_output=True, text=True)
        assert r.returncode == 0 and not r.stderr, r
        subprocess.run([REAL, "merge", "-t", "16", theirs] + args, check=True, capture_output=True)
        assert gzip.open(ours).read() == gzip.open(theirs).read(), k
        shutil.copy(ours, str(tmp_path / "copy.bam"))
        subprocess.run([REAL, "index", str(tmp_path / "copy.bam")], check=True, capture_output=True)
        assert open(ours + ".bai", "rb").read() == open(str(tmp_path / "copy.bam.bai"), "rb").read(), k
        assert not glob.glob(str(tmp_path / "ours.bam.ssq_merge_*"))
        for f in (ours, ours + ".bai", theirs, theirs + ".bai", str(tmp_path / "copy.bam"), str(tmp_path / "copy.bam.bai")):
            os.unlink(f)


@need_real
def test_shim_refused_input_yields_the_real_file(tmp_path):
    paths = seven_inputs(tmp_path, 2000, 4)
    bad = str(tmp_path / "unsorted.bam")
    open(bad, "wb").write(bgzf(bam_header(HD + sq()) + record("a", 0, 0, 500) + record("b", 0, 0, 400), 0xff00))
    out = str(tmp_path / "out.bam")
    env = dict(os.environ, SSQ_SAMBAMBA_REAL=REAL, SSQ_MERGE_GPU="1", SSQ_MERGE_WINDOW="3000")
    r = subprocess.run([SHIM, "merge", out, paths[0], bad], env=env, capture_output=True, text=True)
    assert "not coordinate-sorted" in r.stderr and "running the real sambamba" in r.stderr, r.stderr
    assert not glob.glob(out + ".ssq_merge_*")
    theirs = str(tmp_path / "theirs.bam")
    subprocess.run([REAL, "merge", theirs, paths[0], bad], capture_output=True)
    assert os.path.exists(out) == os.path.exists(theirs)
    if os.path.exists(out):
        assert gzip.open(out).read() == gzip.open(theirs).read()


@pytest.mark.parametrize("bgzf_gpu", ["0", "1"])
def test_shim_write_failure_leaves_nothing(split_bench, tmp_path, bgzf_gpu):
    """the output cannot be written (a 64 KB file size limit): a non-zero exit, one message, no out.bam, no temporary file"""
    real = tmp_path / "real.sh"
    real.write_text("#!/bin/sh\necho \"real $*\"\n")
    real.chmod(0o755)
    env = dict(os.environ, SSQ_SAMBAMBA_REAL=str(real), SSQ_MERGE_GPU="1", SSQ_BGZF_GPU=bgzf_gpu)
    out = str(tmp_path / "out.bam")
    r = subprocess.run(["bash", "-c", 'trap "" XFSZ; ulimit -f 64; exec "$@"', "sh", SHIM, "merge", "-t", "4", out] + split_bench[2], env=env, capture_output=True, text=True)
    assert r.returncode == 1 and "could not be written" in r.stderr and "real" not in r.stdout, r
    assert not glob.glob(out + "*")
