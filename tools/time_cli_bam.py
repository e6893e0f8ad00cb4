#!/usr/bin/env python
"""The align step's whole chain to a sorted BAM file, wall clock, two ways (speedseq:438-441):
  text : bwa mem | samblaster | sambamba view -S -f bam -l 0 | sambamba sort      — shims for the first two, the REFERENCE'S sambamba
  bam  : the same command line with SSQ_FUSE_BAM and the `sambamba` shim          — the main records never exist as text
and a check that both files hold the same records in the same order (`sambamba view` of both, by the reference's sambamba), i.e. the
device-side encode + sort + the shim's merge against the reference's own tool on a few million reads.
usage: time_cli_bam.py [n_reads] [genome_bp] [path of the real sambamba]"""
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

n_reads = int(sys.argv[1]) if len(sys.argv) > 1 else 2_000_000
glen = int(sys.argv[2]) if len(sys.argv) > 2 else 63025520
REAL = sys.argv[3] if len(sys.argv) > 3 else os.path.join(ROOT, "oracle", "_ref", "stage", "src", "sambamba")
assert os.access(REAL, os.X_OK), "the reference's sambamba is needed (oracle/stage_config1.sh stages it)"
cache = bench.cache_dir()
s = capi.SSQ()
fa, g = bench.ensure_reference(cache, glen, lambda f: s.index_build(f, None, 0))
fq = os.path.join(cache, "cli_%d.fq" % n_reads)
if not os.path.exists(fq):  # same generator and layout as tools/time_cli.py
    codes = bench.fast_pairs(g, n_reads // 2, 150, 4242)
    n = codes.shape[0]
    rec = np.empty((n, 14 + 151 + 2 + 151), np.uint8)
    nm = np.char.add("p", np.char.zfill((np.arange(n) // 2).astype("U10"), 9)).astype("S10")
    rec[:, 0] = ord("@"); rec[:, 1:11] = np.frombuffer(nm.tobytes(), np.uint8).reshape(n, 10); rec[:, 11] = ord("/"); rec[:, 12] = ord("1") + (np.arange(n) & 1); rec[:, 13] = 10
    rec[:, 14:164] = np.frombuffer(b"ACGT", np.uint8)[codes]; rec[:, 164] = 10; rec[:, 165] = ord("+"); rec[:, 166] = 10
    rec[:, 167:317] = ord("I"); rec[:, 317] = 10
    rec.tofile(fq)
B = os.path.join(ROOT, "speedseq_b200", "bin")
RG = r"@RG\tID:x\tSM:x\tLB:l"
sb_args = ["--excludeDups", "--addMateTags", "--maxSplitCount", "2", "--minNonOverlap", "20"]
threads = str(min(32, os.cpu_count() or 4))
for tag, env, with_sb in (("bwa mem (fused, text) > /dev/null", {}, 0), ("bwa mem (BAM runs) > /dev/null", {"SSQ_FUSE_BAM": "1"}, 0), ("bwa mem (BAM runs) | samblaster > /dev/null", {"SSQ_FUSE_BAM": "1"}, 1)):
    e = dict(os.environ, SSQ_FUSE_SAMBLASTER=" ".join(sb_args), **env)  # where the time of the chain goes: its first stages alone
    t0 = time.time()
    with open(os.devnull, "wb") as nul:
        p1 = subprocess.Popen([os.path.join(B, "bwa"), "mem", "-t", "8", "-p", "-R", RG, fa, fq], stdout=subprocess.PIPE if with_sb else nul, stderr=subprocess.DEVNULL, env=e)
        if with_sb:
            subprocess.run([os.path.join(B, "samblaster")] + sb_args + ["--splitterFile", os.devnull, "--discordantFile", os.devnull], stdin=p1.stdout, stdout=nul, stderr=subprocess.DEVNULL, env=e, check=True, timeout=300)
        assert p1.wait(timeout=300) == 0
    print("%-46s %6.2f s" % (tag, time.time() - t0), flush=True)
res = {}
for tag, env, sambamba in (("text + reference sambamba", {}, REAL), ("BAM runs + sambamba shim", {"SSQ_FUSE_BAM": "1"}, os.path.join(B, "sambamba"))):
    e = dict(os.environ, SSQ_FUSE_SAMBLASTER=" ".join(sb_args), SSQ_SAMBAMBA_REAL=REAL, **env)
    out = os.path.join(cache, "cli_%s.bam" % ("text" if not env else "runs"))
    tmp = os.path.join(cache, "sort_tmp"); os.makedirs(tmp, exist_ok=True)
    t0 = time.time()
    p1 = subprocess.Popen([os.path.join(B, "bwa"), "mem", "-t", "8", "-p", "-R", RG, fa, fq], stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, env=e)
    p2 = subprocess.Popen([os.path.join(B, "samblaster")] + sb_args + ["--splitterFile", os.path.join(cache, "cli_spl.sam"), "--discordantFile", os.path.join(cache, "cli_disc.sam")],
                          stdin=p1.stdout, stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, env=e)
    p3 = subprocess.Popen([sambamba, "view", "-S", "-f", "bam", "-l", "0", "/dev/stdin"], stdin=p2.stdout, stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, env=e)
    p4 = subprocess.run([sambamba, "sort", "-t", threads, "-m", "8G", "--tmpdir=" + tmp, "-o", out, "/dev/stdin"], stdin=p3.stdout, stderr=subprocess.DEVNULL, env=e, timeout=400)
    assert p4.returncode == 0 and p3.wait(timeout=60) == 0 and p2.wait(timeout=60) == 0 and p1.wait(timeout=60) == 0, tag
    dt = time.time() - t0
    t1 = time.time()
    h = hashlib.md5()
    v = subprocess.Popen([REAL, "view", "-t", threads, out], stdout=subprocess.PIPE)
    n_rec = 0
    for chunk in iter(lambda: v.stdout.read(1 << 24), b""):
        h.update(chunk); n_rec += chunk.count(b"\n")
    assert v.wait() == 0
    hdr = subprocess.run([REAL, "view", "-H", out], stdout=subprocess.PIPE, check=True).stdout
    res[tag] = (h.hexdigest(), n_rec, b"".join(l for l in hdr.splitlines(True) if not l.startswith(b"@PG")))
    print("%-28s %6.2f s  %6.2f M reads/s to a sorted BAM of %d MB, %d records  (check: %.1f s)" % (tag, dt, n_reads / dt / 1e6, os.path.getsize(out) >> 20, n_rec, time.time() - t1), flush=True)
a, b = res.values()
assert a == b, "the two BAM files differ: %r %r" % (a[:2], b[:2])
print("records (sambamba view of both files) and header minus @PG identical: md5 %s, %d records" % (a[0], a[1]))
