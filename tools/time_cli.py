#!/usr/bin/env python
"""wall-clock throughput of the drop-in executables themselves (speedseq_b200/bin/bwa, .../samblaster) on an interleaved 4-line FASTQ:
`bwa mem -p` alone with 1 and 2 stream lanes, and the fused `bwa mem | samblaster` pipe of speedseq:438-439; checks that every variant
writes the same bytes.  usage: time_cli.py [n_reads] [genome_bp]"""
import hashlib
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench
from speedseq_b200 import capi

n_reads = int(sys.argv[1]) if len(sys.argv) > 1 else 4_000_000
glen = int(sys.argv[2]) if len(sys.argv) > 2 else 63025520
cache = bench.cache_dir()
s = capi.SSQ()
fa, g = bench.ensure_reference(cache, glen, lambda f: s.index_build(f, None, 0))
fq = os.path.join(cache, "cli_%d.fq" % n_reads)
if not os.path.exists(fq):
    codes = bench.fast_pairs(g, n_reads // 2, 150, 4242)
    n = codes.shape[0]
    rec = np.empty((n, 14 + 151 + 2 + 151), np.uint8)
    ids = np.arange(n) // 2
    nm = np.char.add("p", np.char.zfill(ids.astype("U10"), 9)).astype("S10")
    rec[:, 0] = ord("@"); rec[:, 1:11] = np.frombuffer(nm.tobytes(), np.uint8).reshape(n, 10); rec[:, 11] = ord("/"); rec[:, 12] = ord("1") + (np.arange(n) & 1); rec[:, 13] = 10
    rec[:, 14:164] = np.frombuffer(b"ACGT", np.uint8)[codes]; rec[:, 164] = 10; rec[:, 165] = ord("+"); rec[:, 166] = 10
    rec[:, 167:317] = ord("I"); rec[:, 317] = 10
    rec.tofile(fq)
BWA, SB = os.path.join(ROOT, "speedseq_b200", "bin", "bwa"), os.path.join(ROOT, "speedseq_b200", "bin", "samblaster")
RG = r"@RG\tID:x\tSM:x"
sb_args = ["--excludeDups", "--addMateTags", "--maxSplitCount", "2", "--minNonOverlap", "20"]


def md5_of(path):
    h = hashlib.md5()
    with open(path, "rb") as f:
        for l in f:
            if not l.startswith(b"@PG"):
                h.update(l)
    return h.hexdigest()


res = {}
for tag, env in (("bwa mem, 1 lane", {"SSQ_LANES": "1"}), ("bwa mem, 2 lanes", {"SSQ_LANES": "2"}), ("bwa mem, host tokeniser", {"SSQ_HOST_FASTQ": "1"})):
    e = dict(os.environ); e.update(env)
    out = os.path.join(cache, "cli_out.sam")
    t0 = time.time()
    with open(out, "wb") as f:
        subprocess.run([BWA, "mem", "-t", "30", "-p", "-R", RG, fa, fq], stdout=f, stderr=subprocess.DEVNULL, env=e, check=True, timeout=200)
    dt = time.time() - t0
    res[tag] = md5_of(out)
    print("%-28s %6.2f s  %6.2f M reads/s  (%d MB of SAM)" % (tag, dt, n_reads / dt / 1e6, os.path.getsize(out) >> 20))
assert len(set(res.values())) == 1, res
for tag, env in (("unfused bwa | samblaster", {}), ("fused bwa | samblaster", {"SSQ_FUSE_SAMBLASTER": " ".join(sb_args)})):
    e = dict(os.environ); e.update(env)
    outs = [os.path.join(cache, "cli_%s.sam" % k) for k in ("main", "spl", "disc")]
    t0 = time.time()
    p1 = subprocess.Popen([BWA, "mem", "-t", "30", "-p", "-R", RG, fa, fq], stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, env=e)
    with open(outs[0], "wb") as f:
        subprocess.run([SB] + sb_args + ["--splitterFile", outs[1], "--discordantFile", outs[2]], stdin=p1.stdout, stdout=f, stderr=subprocess.DEVNULL, env=e, check=True, timeout=300)
    assert p1.wait(timeout=60) == 0
    dt = time.time() - t0
    res[tag] = tuple(md5_of(o) for o in outs)
    print("%-28s %6.2f s  %6.2f M reads/s" % (tag, dt, n_reads / dt / 1e6))
assert res["unfused bwa | samblaster"] == res["fused bwa | samblaster"], "fused and unfused pipes differ"
print("all variants byte-identical (minus @PG)")
