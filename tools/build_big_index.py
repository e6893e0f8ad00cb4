#!/usr/bin/env python
"""`ssq_index_build_ex` on a large reference, on the path(s) asked for, then three checks of the result.  Builds a seeded
synthetic genome (8 contigs, planted repeat family; default 2.2 Gbp = 4.4 G suffixes, more BWT rows than 2^32; 3100000000 = the
size of GRCh37), indexes it, then checks:
  * header: primary row, cumulative base counts = the base composition of forward + reverse-complement strand;
  * order: a million random pairs of consecutive SA samples (32 rows apart) are in lexicographic order, compared on the text;
  * function: the CPU oracle loads the index and places simulated read pairs at their origins.
--path: passes (device sort), host, auto, both (= passes,host) or a comma list; the first path builds the index that is
checked (always afresh: index files left in the cache are removed first), every further one builds into its own prefix and must
give the same five files byte for byte.  Each build prints the path that ran (from the stats), its wall time, the device sort's
stats and this process's peak host memory so far.
--repeats: hard repeats on top of the generator's diverged family: 5 % of the genome as exact copies of 10-100 kb segments and
1 % as 171 bp satellite arrays at 2 % divergence, so that many suffixes stay tied for many doubling rounds.
usage: build_big_index.py [genome_bp] [n_pairs] [--path P] [--repeats]    (host path: about 15 bytes of host memory per bp)"""
import argparse
import ctypes as C
import filecmp
import os
import resource
import struct
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import bench
from speedseq_b200 import capi

ap = argparse.ArgumentParser()
ap.add_argument("genome_bp", nargs="?", type=int, default=2_200_000_000)
ap.add_argument("n_pairs", nargs="?", type=int, default=2000)
ap.add_argument("--path", default="passes")
ap.add_argument("--repeats", action="store_true")
args = ap.parse_args()
glen, n_pairs = args.genome_bp, args.n_pairs
PATHS = {"auto": 0, "passes": 2, "host": 3}
NAMES = {2: "device suffix sort", 3: "host suffix sort"}
paths = ["passes", "host"] if args.path == "both" else args.path.split(",")
cache = os.path.join(bench.cache_dir(), "hard") if args.repeats else bench.cache_dir()
ssq = capi.SSQ()
PLANTED = []  # [start, end) of every planted copy, source and target: a read from one of them has no unique origin


def plant(n, seed, g=None):
    """the hard repeats of --repeats (seeded): copies into g when given, their intervals into PLANTED either way"""
    PLANTED.clear()
    rng = np.random.default_rng(seed + 1000)
    done = 0
    while done < 0.05 * n:
        L = int(rng.integers(10000, 100001))
        a, b = (int(x) for x in rng.integers(0, n - L, 2))
        if g is not None:
            g[b:b + L] = g[a:a + L]
        PLANTED.extend([(a, a + L), (b, b + L)])
        done += L
    unit = rng.integers(0, 4, 171).astype(np.uint8)
    done = 0
    while done < 0.01 * n:
        k = int(rng.integers(5, 60))
        arr = np.tile(unit, k)
        m = rng.random(arr.size) < 0.02
        arr[m] = rng.integers(0, 4, int(m.sum())).astype(np.uint8)
        b = int(rng.integers(0, n - arr.size))
        if g is not None:
            g[b:b + arr.size] = arr
        PLANTED.append((b, b + arr.size))
        done += arr.size


if args.repeats:  # the same generator, hard repeats planted on top
    _synth = bench.synth_genome

    def hard(n, seed, repeat_frac=0.08):
        g = _synth(n, seed, repeat_frac)
        plant(n, seed, g)
        return g
    bench.synth_genome = hard


def build_one(fa, prefix, name):
    t0 = time.time()
    st = ssq.index_build_ex(fa, prefix, 0, path=PATHS[name])
    dt = time.time() - t0
    extra = ""
    if st["path"] == 2:
        extra = ": %d passes, %d rounds, %d chunks, %d suffixes open after the first sort (%.3f %%), largest group %d, %d oversize, %d finalisation ranges, peak %.1f GB of device memory" % (
            st["passes"], st["rounds"], st["chunks"], st["unresolved_first"], 100.0 * st["unresolved_first"] / (2 * glen + 1), st["largest_group"], st["oversize_groups"], st["ranges"], st["peak_device_bytes"] / 1e9)
    extra += "; peak host RSS of this process so far %.1f GB" % (resource.getrusage(resource.RUSAGE_SELF).ru_maxrss / 1e6)
    print("ssq_index_build_ex --path %s -> %s: %.1f s for %d bp = %d suffixes%s" % (name, NAMES[st["path"]], dt, glen, 2 * glen + 1, extra), flush=True)
    return dt


def builder(fa):
    build_one(fa, fa, paths[0])


for ext in (".bwt", ".sa", ".pac", ".ann", ".amb"):  # the first path always builds: no check may run on an index some earlier run made
    if os.path.exists(os.path.join(cache, "syn_%d.fa%s" % (glen, ext))):
        os.remove(os.path.join(cache, "syn_%d.fa%s" % (glen, ext)))
fa, g = bench.ensure_reference(cache, glen, builder)
if args.repeats and not PLANTED:  # genome taken from the cache: the same seeded intervals
    plant(glen, 20)
for name in paths[1:]:
    pre = fa + "." + name
    build_one(fa, pre, name)
    for ext in ("amb", "ann", "pac", "bwt", "sa"):
        assert filecmp.cmp(fa + "." + ext, pre + "." + ext, shallow=False), "%s: .%s differs from --path %s" % (name, ext, paths[0])
        os.remove(pre + "." + ext)
    print("--path %s: all five files byte-identical to --path %s" % (name, paths[0]), flush=True)
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
pos = rng.integers(0, glen - 1000, 4 * n_pairs)
if PLANTED:  # only reads with a unique origin can be checked for placement
    iv = np.array(sorted(PLANTED), np.int64)
    reach = np.maximum.accumulate(iv[:, 1])
    k = np.searchsorted(iv[:, 0], pos + 400, side="left")  # planted intervals starting before the fragment ends
    hit = (k > 0) & (reach[np.maximum(k - 1, 0)] > pos)
    print("%d of %d drawn fragments overlap planted copies and are not used" % (int(hit[:n_pairs].sum()), n_pairs), flush=True)
    pos = pos[~hit]
pos = pos[:n_pairs]
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
