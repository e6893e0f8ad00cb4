#!/usr/bin/env python
"""`ssq_index_build` on a reference beyond the device sort's limit (2^31 - 2 suffixes): the host path (64-bit induced sorting,
csrc/ssq_sais.h).  Builds a seeded synthetic genome (8 contigs, planted repeat family; default 2.2 Gbp = 4.4 G suffixes, more BWT
rows than 2^32; 3100000000 = the size of GRCh37), indexes it without touching a GPU, then checks the result three ways:
  * header: primary row, cumulative base counts = the base composition of forward + reverse-complement strand;
  * order: a million random pairs of consecutive SA samples (32 rows apart) are in lexicographic order, compared on the text;
  * function: the CPU oracle loads the index and places simulated read pairs at their origins.
usage: build_big_index.py [genome_bp] [n_pairs]      (about 15 bytes of host memory per reference base pair)"""
import ctypes as C
import os
import struct
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import bench

glen = int(sys.argv[1]) if len(sys.argv) > 1 else 2_200_000_000
n_pairs = int(sys.argv[2]) if len(sys.argv) > 2 else 2000
cache = bench.cache_dir()
lib = C.CDLL(os.path.join(ROOT, "speedseq_b200", "libssq.so"))
lib.ssq_index_build.argtypes = [C.c_char_p, C.c_char_p, C.c_int]
lib.ssq_last_error.restype = C.c_char_p


def builder(fa):
    t0 = time.time()
    rc = lib.ssq_index_build(fa.encode(), None, 0)
    assert rc == 0, lib.ssq_last_error()
    print("ssq_index_build (host path): %.1f s for %d bp = %d suffixes" % (time.time() - t0, glen, 2 * glen + 1), flush=True)


fa, g = bench.ensure_reference(cache, glen, builder)
n = 2 * glen
# --- header
with open(fa + ".bwt", "rb") as f:
    primary, *L2 = struct.unpack("<5Q", f.read(40))
comp = np.bincount(g, minlength=4).astype(np.int64)
both = comp + comp[::-1]  # the reverse-complement strand holds the complements
want_L2 = np.cumsum(both)
assert list(want_L2) == L2, (list(want_L2), L2)
print("primary row %d, L2 = %s: equal to the base composition of both strands" % (primary, L2), flush=True)
# --- order of consecutive SA samples
with open(fa + ".sa", "rb") as f:
    hdr = struct.unpack("<7Q", f.read(56))
    assert hdr[0] == primary and hdr[5] == 32 and hdr[6] == n
    smp = np.fromfile(f, dtype=np.uint64)
assert smp.size == (n + 32) // 32 - 1
print("%d SA samples, max %d (n = %d, 2^32 = %d)" % (smp.size, int(smp.max()), n, 1 << 32), flush=True)


def sym(pos):  # text symbols at positions pos (int64 array) of forward + reverse complement; n -> sentinel (-1)
    out = np.full(pos.shape, -1, np.int64)
    fw = pos < glen
    rv = (pos >= glen) & (pos < n)
    out[fw] = g[pos[fw]]
    out[rv] = 3 - g[n - 1 - pos[rv]]
    return out


rng = np.random.default_rng(1)
k = rng.integers(0, smp.size - 1, 1_000_000)
a, b = smp[k].astype(np.int64), smp[k + 1].astype(np.int64)
undecided = np.ones(a.size, bool)
ok = np.zeros(a.size, bool)
for d in range(0, 4000):
    idx = np.nonzero(undecided)[0]
    if idx.size == 0:
        break
    sa_, sb_ = sym(a[idx] + d), sym(b[idx] + d)
    lt, gt = sa_ < sb_, sa_ > sb_
    ok[idx[lt]] = True
    undecided[idx[lt | gt]] = False
assert not undecided.any(), "suffix pairs equal over 4000 symbols: %d" % int(undecided.sum())
assert ok.all(), "%d of %d sampled consecutive suffix pairs out of order" % (int((~ok).sum()), ok.size)
print("1,000,000 random pairs of consecutive SA samples are in lexicographic order", flush=True)
# --- function: the oracle aligns reads simulated from known positions
import ssq_testlib as T
rl = 150
pos = rng.integers(0, glen - 1000, n_pairs)
bounds = np.linspace(0, glen, 9).astype(np.int64)
fq = os.path.join(cache, "big_check.fq")
acgt = np.frombuffer(b"ACGT", np.uint8)
comp_t = bytes.maketrans(b"ACGT", b"TGCA")
with open(fq, "wb") as f:
    for i, p in enumerate(pos):
        ins = 400
        r1 = acgt[g[p:p + rl]].tobytes()
        r2 = acgt[g[p + ins - rl:p + ins]].tobytes().translate(comp_t)[::-1]
        f.write(b"@r%d/1\n%s\n+\n%s\n@r%d/2\n%s\n+\n%s\n" % (i, r1, b"I" * rl, i, r2, b"I" * rl))
t0 = time.time()
sam = subprocess.run([T.ORACLE_BIN, "mem", "-t", "8", "-p", fa, fq], check=True, stdout=subprocess.PIPE, stderr=subprocess.DEVNULL).stdout.decode()
good = tot = 0
for l in sam.splitlines():
    if l.startswith("@"):
        continue
    f = l.split("\t")
    flag = int(f[1])
    if flag & 0x900 or not flag & 0x40:
        continue
    i = int(f[0][1:])
    c = int(np.searchsorted(bounds, pos[i], side="right") - 1)
    tot += 1
    if f[2] == "chrS%d" % (c + 1) and abs(int(f[3]) - 1 - (pos[i] - bounds[c])) <= 5 and not flag & 4:
        good += 1
print("oracle `mem` on the index (loaded in %.0f s incl. alignment): %d of %d first reads placed at their origin" % (time.time() - t0, good, tot), flush=True)
assert tot == n_pairs and good >= 0.97 * tot
print("OK")
