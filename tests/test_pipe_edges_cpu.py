"""The stages after extension (insert-size statistics, mate rescue, pairing, CIGAR, samblaster, SAM text) on reads the FR corpus
(ssq_testlib.simulate_pairs) never holds: all four pair orientations and the counts at which an orientation's statistics fail,
fragments at contig ends and across contig borders, reads of mixed lengths from 1 to 255 bases, tiny and degenerate batches, and
read ordinals past 2^31.  tests/hostsim runs the kernels' bodies on the host; every case must give the oracle's `bwa mem` records
and its `bwa mem | samblaster` streams (speedseq's options) byte for byte, and each case asserts that its inputs really reach the
edge it is about.  The same cases through the GPU: tests/test_gpu_pipe_edges.py.

An `-I` override for an orientation other than FR is not covered: `bwa mem -I` only sets the FR statistics, so the oracle has no
way to state one."""
import re

import numpy as np
import pytest

import ssq_testlib as T
from test_hostsim_pipe import oracle_streams, sq_header

ORIENT = ("FF", "FR", "RF", "RR")
SB_TUPLE = (1, 1, 2, 20, 0)  # speedseq's samblaster options: --excludeDups --addMateTags --maxSplitCount 2 --minNonOverlap 20
SB_ARGS = ["--excludeDups", "--addMateTags", "--maxSplitCount", "2", "--minNonOverlap", "20"]
EXACT_LENGTHS = (1, 18, 19, 20, 31, 32, 33, 64, 65, 254, 255)
_COMP = np.array([3, 2, 1, 0, 4], np.uint8)
_ACGTN = np.frombuffer(b"ACGTN", np.uint8)


# ------------------------------------------------------------------------------------------------------------ generator ----
def edge_pairs(g, bounds, n_pairs, seed, orient=(0, 1, 0, 0), ins=(400, 40), lengths=150, edge_frac=0.0, rescue_frac=0.0, err=0.005,
               n_frac=0.001, swap=0.5, all_n=0, prefix="p"):
    """paired reads -> (names, seqs, quals), mates adjacent.

    orient: weight per orientation (FF, FR, RF, RR) as bwa's mem_pestat sees it (strand of read 1, then of read 2 projected onto
    read 1's strand, read 2 downstream or upstream); round(n_pairs * weight / total) pairs get each one, in shuffled order.  Each
    fragment's two ends are forward or reverse-complemented as the orientation says and then swapped with probability `swap`
    (a swapped FF fragment is built as RR, so that the pair still shows the orientation drawn).
    ins: (mean, sd) of the fragment length, or a dict orientation -> (mean, sd); a fragment is never shorter than its two reads + 10.
    lengths: one length; (lo, hi): drawn per read from [lo, hi]; a list: its lengths on the first reads in order, then drawn from it.
    edge_frac: fraction of fragments that start or end within +-20 bases of a contig start or end (a third exactly on it); these
    may cross into the neighbouring contig.  The others lie inside one contig long enough to hold them.
    rescue_frac: fraction of pairs with one mate that has a substitution every 12 bases (reads of 60 bases or more): no exact match
    reaches the 19-base seed length, but local Smith-Waterman in the window the mate's statistics allow places it.
    all_n: that many pairs (spread over the batch) get one all-N mate.
    Names: <prefix><i>_<orientation>[_e (edge fragment)][_x (rescue-only mate)]."""
    rng = np.random.default_rng(seed)
    L = int(bounds[-1])
    w = np.asarray(orient, float)
    cnt = [int(round(n_pairs * x / w.sum())) for x in w]
    dirs = np.repeat(np.arange(4), cnt)
    rng.shuffle(dirs)
    n = len(dirs)
    if isinstance(lengths, int):
        lens = np.full(2 * n, lengths)
    elif isinstance(lengths, tuple):
        lens = rng.integers(lengths[0], lengths[1] + 1, 2 * n)
    else:
        lens = rng.choice(np.asarray(lengths), 2 * n)
        lens[: min(len(lengths), 2 * n)] = lengths[: 2 * n]
    ctg_len = np.diff(bounds)
    allN = set(np.linspace(0, n - 1, all_n).astype(int).tolist()) if all_n else set()
    names, seqs, quals = [], [], []
    for i in range(n):
        d = int(dirs[i])
        l1, l2 = int(lens[2 * i]), int(lens[2 * i + 1])
        sw = rng.random() < swap
        mean, sd = ins[ORIENT[d]] if isinstance(ins, dict) else ins
        size = max(l1 + l2 + 10, int(rng.normal(mean, sd)))
        edge = rng.random() < edge_frac
        if edge:
            off = 0 if rng.random() < 1 / 3 else int(rng.integers(-20, 21))
            c = int(rng.integers(0, len(ctg_len)))
            p = int(bounds[c]) + off if rng.random() < 0.5 else int(bounds[c + 1]) + off - size
            p = min(max(p, 0), L - size)
        else:
            fit = np.where(ctg_len > size + 2)[0]
            c = int(rng.choice(fit, p=ctg_len[fit] / ctg_len[fit].sum()))
            p = int(rng.integers(int(bounds[c]), int(bounds[c + 1]) - size))
        frag = g[p:p + size]
        bd = {0: 3, 3: 0}.get(d, d) if sw else d  # the orientation to build so that swapping the ends gives d
        ll, lr = (l2, l1) if sw else (l1, l2)
        left, right = frag[:ll], frag[size - lr:]
        left = left if "FR"[bd >> 1] == "F" else _COMP[left[::-1]]
        right = right if "FR"[bd & 1] == "F" else _COMP[right[::-1]]
        r = [left.copy(), right.copy()]
        for x in r:
            m = rng.random(len(x)) < err
            x[m] = (x[m] + rng.integers(1, 4, int(m.sum()), dtype=np.uint8)) % 4
            x[rng.random(len(x)) < n_frac] = 4
        if sw:
            r.reverse()
        resc = rng.random() < rescue_frac
        if resc:
            k = int(rng.integers(0, 2))
            if len(r[k]) >= 60:
                x = r[k]
                x[11::12] = np.where(x[11::12] < 4, (x[11::12] + 1 + rng.integers(0, 3, len(x[11::12]))) % 4, 4)
            else:
                resc = False
        if i in allN:
            r[int(rng.integers(0, 2))][:] = 4
        nm = "%s%d_%s%s%s" % (prefix, i, ORIENT[d], "_e" if edge else "", "_x" if resc else "")
        for x in r:
            names.append(nm)
            seqs.append(_ACGTN[x].tobytes().decode())
            quals.append("I" * len(x))
    return names, seqs, quals


def random_pairs(n_pairs, seed, length=100, prefix="u"):
    """pairs of random sequence and all-N reads: nothing in them maps"""
    rng = np.random.default_rng(seed)
    names, seqs = [], []
    for i in range(n_pairs):
        for k in range(2):
            names.append("%s%d" % (prefix, i))
            seqs.append("N" * length if (i + k) % 3 == 0 else "".join("ACGT"[x] for x in rng.integers(0, 4, length)))
    return names, seqs, ["I" * len(s) for s in seqs]


def cat(*parts):
    return tuple(sum((list(p[k]) for p in parts), []) for k in range(3))


# -------------------------------------------------------------------------------------------------------------- genomes ----
EDGE_CONTIGS = (30000, 300, 20000, 120, 25000, 35000)  # one contig shorter than the insert size, one shorter than a read


@pytest.fixture(scope="module")
def edge_index(oracle, tmp_path_factory):
    """six contigs of random sequence (no repeats, so every pair of unique hits counts for the statistics), oracle-built index"""
    d = tmp_path_factory.mktemp("edges")
    rng = np.random.default_rng(2024)
    bounds = np.concatenate([[0], np.cumsum(EDGE_CONTIGS)])
    g = rng.choice(4, size=int(bounds[-1]), p=[0.295, 0.205, 0.205, 0.295]).astype(np.uint8)
    fa = str(d / "edges.fa")
    T.write_fasta(fa, g, bounds)
    oracle.index_build(fa)
    return fa, g, bounds


# ---------------------------------------------------------------------------------------------------------------- cases ----
class Case:
    """inputs of one case and what its coverage asserts expect.  proper: orientations that must have proper pairs; failed: the
    expected failed flag per orientation (None: not asserted); counts: the expected candidate-pair counts of mem_pestat;
    rescue: mates must have been rescued; edges: records at the first and the last base of a contig; lengths: read lengths the
    batch must hold; max_len: the longest read allowed; unmapped: no read maps"""

    def __init__(self, genome, reads, n_processed=0, proper=(), failed=None, counts=None, rescue=False, edges=False, lengths=(), max_len=0, unmapped=False):
        self.genome, (self.names, self.seqs, self.quals) = genome, reads
        self.n_processed, self.proper, self.failed, self.counts = n_processed, proper, failed, counts
        self.rescue, self.edges, self.lengths, self.max_len, self.unmapped = rescue, edges, lengths, max_len, unmapped


def make_case(name, syn, edge):
    sg, sb = syn[1], syn[2]
    eg, eb = edge[1], edge[2]
    S = lambda **kw: edge_pairs(sg, sb, seed=sum(map(ord, name)), **kw)
    if name == "rf_only":  # a mate-pair library: long RF fragments
        return Case("syn", S(n_pairs=600, orient=(0, 0, 1, 0), ins=(2500, 250), lengths=101, rescue_frac=0.1), proper=(2,), rescue=True, failed=(1, 1, 0, 1))
    if name == "fr_and_rf":  # mixed library: short FR and long RF in comparable numbers
        return Case("syn", S(n_pairs=500, orient=(0, 1, 1, 0), ins={"FR": (400, 40), "RF": (2000, 200)}, lengths=150, rescue_frac=0.1), proper=(1, 2), rescue=True,
                    failed=(1, 0, 0, 1))
    if name == "all_four":
        return Case("syn", S(n_pairs=500, orient=(1, 1, 1, 1), ins=(500, 50), lengths=150, rescue_frac=0.1), proper=(0, 1, 2, 3), rescue=True, failed=(0, 0, 0, 0))
    if name == "ff_and_rr":
        return Case("syn", S(n_pairs=600, orient=(1, 0, 0, 1), ins=(600, 60), lengths=125, rescue_frac=0.1), proper=(0, 3), rescue=True, failed=(0, 1, 1, 0))
    # just across the two thresholds of mem_pestat: fewer than 10 pairs, fewer than 5 % of the largest orientation.  The counted pairs
    # carry no rescue-only mate (a pair with an unmapped end is not counted); rescue-only pairs of both orientations come on top
    E = lambda seed, **kw: edge_pairs(eg, eb, seed=seed, err=0.002, n_frac=0, **kw)
    for k, nm in ((9, "ff_9_of_150"), (10, "ff_10_of_150")):
        if name == nm:
            reads = cat(E(1, n_pairs=150 + k, orient=(k, 150, 0, 0), ins=(400, 40), prefix="c"), E(2, n_pairs=24, orient=(1, 1, 0, 0), ins=(400, 40), rescue_frac=1.0, prefix="x"))
            return Case("edge", reads, proper=(1,) + ((0,) if k == 10 else ()), failed=(int(k < 10), 0, 1, 1), counts=(k, 150, 0, 0), rescue=True)
    for k, nm in ((49, "rf_49_of_1000"), (50, "rf_50_of_1000")):
        if name == nm:
            reads = cat(E(3, n_pairs=1000 + k, orient=(0, 1000, k, 0), ins={"FR": (350, 35), "RF": (1000, 50)}, lengths=100, prefix="c"),
                        E(4, n_pairs=24, orient=(0, 1, 1, 0), ins={"FR": (350, 35), "RF": (1000, 50)}, lengths=100, rescue_frac=1.0, prefix="x"))
            return Case("edge", reads, proper=(1,) + ((2,) if k == 50 else ()), failed=(1, 0, int(k < 50), 1), counts=(0, 1000, k, 0), rescue=True)
    # contig ends: fragments from the first base / to the last base of each contig, across contig borders, the tiny contigs
    if name == "ends_fr":
        return Case("edge", edge_pairs(eg, eb, 600, 5, orient=(0, 1, 0, 0), ins=(400, 40), lengths=150, edge_frac=0.5, rescue_frac=0.15), proper=(1,), rescue=True, edges=True)
    if name == "ends_all_four":
        return Case("edge", edge_pairs(eg, eb, 500, 6, orient=(1, 1, 1, 1), ins=(450, 45), lengths=(60, 255), edge_frac=0.4, rescue_frac=0.15), proper=(0, 1, 2, 3), rescue=True, edges=True)
    # read lengths
    if name == "lengths_1_to_255":  # every length from 1 to 255 once, then drawn from 1..255; mates of a pair differ; all-N reads
        return Case("syn", S(n_pairs=450, orient=(1, 3, 1, 1), ins=(600, 60), lengths=list(range(1, 256)), rescue_frac=0.1, all_n=12), proper=(1,), lengths=EXACT_LENGTHS)
    if name == "lengths_255_and_40":
        return Case("syn", S(n_pairs=360, orient=(0, 2, 1, 0), ins={"FR": (450, 45), "RF": (1200, 120)}, lengths=[255, 40, 40, 255], rescue_frac=0.1), proper=(1, 2), rescue=True,
                    lengths=(40, 255))
    if name == "one_long_pair":  # the batch's longest read (what device scratch is sized from) in one pair among short reads
        a = S(n_pairs=400, orient=(0, 1, 0, 0), ins=(300, 30), lengths=(30, 80), rescue_frac=0.1)
        b = edge_pairs(sg, sb, 1, 77, orient=(0, 1, 0, 0), ins=(600, 20), lengths=255, prefix="long")
        reads = cat((a[0][:400], a[1][:400], a[2][:400]), b, (a[0][400:], a[1][400:], a[2][400:]))
        return Case("syn", reads, proper=(1,), rescue=True, lengths=(255,))
    if name == "lengths_up_to_19":  # too short for a 30-point alignment: nothing maps
        return Case("syn", S(n_pairs=300, orient=(1, 1, 1, 1), lengths=(1, 19)), failed=(1, 1, 1, 1), lengths=tuple(range(1, 20)), max_len=19, unmapped=True)
    # degenerate batches
    if name == "one_pair":
        return Case("syn", S(n_pairs=1, lengths=150), failed=(1, 1, 1, 1))
    if name == "two_pairs":
        return Case("syn", S(n_pairs=2, orient=(0, 1, 1, 0), lengths=(100, 150)), failed=(1, 1, 1, 1))
    if name == "all_failed":  # 8 pairs per orientation: every orientation fails, no window, nothing rescued
        reads = cat(S(n_pairs=32, orient=(1, 1, 1, 1), lengths=150, err=0.002), S(n_pairs=8, orient=(1, 1, 1, 1), lengths=150, rescue_frac=1.0, prefix="x"))
        return Case("syn", reads, failed=(1, 1, 1, 1), counts=(8, 8, 8, 8))
    if name == "nothing_maps":
        return Case("syn", random_pairs(60, 9), failed=(1, 1, 1, 1), unmapped=True)
    for np_, nm in ((2 ** 31 - 1, "ordinal_2e31m1"), (2 ** 32 + 5, "ordinal_2e32p5")):  # the read ordinal enters the tie-breaking hash
        if name == nm:
            return Case("syn", S(n_pairs=400, orient=(1, 2, 1, 1), ins=(500, 50), lengths=(90, 150), rescue_frac=0.1), n_processed=np_, proper=(1,), rescue=True)
    raise KeyError(name)


CASES = ("rf_only", "fr_and_rf", "all_four", "ff_and_rr", "ff_9_of_150", "ff_10_of_150", "rf_49_of_1000", "rf_50_of_1000", "ends_fr", "ends_all_four",
         "lengths_1_to_255", "lengths_255_and_40", "one_long_pair", "lengths_up_to_19", "one_pair", "two_pairs", "all_failed", "nothing_maps",
         "ordinal_2e31m1", "ordinal_2e32p5")


# ------------------------------------------------------------------------------------------------------- oracle + checks ----
def pestat_log(err):
    """mem_pestat's stderr lines -> (candidate pair counts (FF, FR, RF, RR), failed flag per orientation)"""
    m = re.findall(r"candidate unique pairs for \(FF, FR, RF, RR\): \((\d+), (\d+), (\d+), (\d+)\)", err)
    assert len(m) == 1, err
    skipped = set(re.findall(r"skip orientation (\w\w)", err))
    return tuple(int(x) for x in m[0]), tuple(int(o in skipped) for o in ORIENT)


def oracle_case(oracle, idx, fa, c, rg, tmp_path, capfd):
    """the oracle's `bwa mem` records, its `bwa mem | samblaster` streams, and mem_pestat's verdict on the batch"""
    capfd.readouterr()
    body, main, spl, disc = oracle_streams(oracle, idx, sq_header(oracle, idx, fa), c.names, c.seqs, c.quals, c.n_processed, rg, SB_ARGS, tmp_path)
    return body, (main, spl, disc), pestat_log(capfd.readouterr().err)


def _span(cigar):
    return sum(int(n) for n, op in re.findall(r"(\d+)([MD])", cigar))


def pair_orient(f1, f2):
    """bwa's mem_infer_dir on the primary records of read 1 and read 2 (one contig) -> 0 FF, 1 FR, 2 RF, 3 RR"""
    L2 = 1 << 41  # any doubled reference length: only differences on one contig matter

    def rb(f):
        b = int(f[3]) - 1
        return (L2 - (b + _span(f[5])), 1) if int(f[1]) & 16 else (b, 0)
    (b1, r1), (b2, r2) = rb(f1), rb(f2)
    p2 = b2 if r1 == r2 else L2 - 1 - b2
    return (0 if r1 == r2 else 1) ^ (0 if p2 > b1 else 3)


def check_coverage(c, body, stats, ctg_len):
    """the case really reaches its edge: proper pairs in each intended orientation, statistics on the intended side of the
    thresholds, rescued mates, records on the first and last base of contigs, the listed read lengths, nothing mapped"""
    counts, failed = stats
    if c.counts is not None:
        assert counts == c.counts
    if c.failed is not None:
        assert failed == tuple(c.failed), counts
    prim = {}
    for l in body.splitlines():
        f = l.split("\t")
        if not int(f[1]) & 0x900:
            prim.setdefault(f[0], []).append(f)
    proper = [0, 0, 0, 0]
    for recs in prim.values():
        if len(recs) == 2 and int(recs[0][1]) & 2 and recs[0][2] == recs[1][2]:
            proper[pair_orient(*recs)] += 1
    for d in c.proper:
        assert proper[d] >= 5, (ORIENT[d], proper)
    if not c.proper and c.failed == (1, 1, 1, 1):
        assert sum(proper) == 0
    # pairs with a rescue-only mate that came out as proper pairs (nothing but mate rescue can place that mate)
    rescued = [n for n, recs in prim.items() if "_x" in n and all(int(f[1]) & 2 and not int(f[1]) & 4 for f in recs)]
    n_rescued = [sum(1 for n in rescued if n.split("_")[1] == o) for o in ORIENT]
    if c.rescue:
        for d in c.proper:
            assert n_rescued[d] >= 1, (ORIENT[d], n_rescued)
    if c.failed is not None:  # an orientation without statistics has no window: nothing is rescued in it
        for d in range(4):
            if c.failed[d] and c.failed[(3, 1, 2, 0)[d]]:  # (read 2 sees an FF pair as RR and an RR pair as FF)
                assert n_rescued[d] == 0, (ORIENT[d], n_rescued)
    if c.edges and c.rescue:  # rescue windows clamped at a contig end
        assert any("_e" in n for n in rescued)
    if c.edges:
        recs = [l.split("\t") for l in body.splitlines()]
        mapped = [f for f in recs if not int(f[1]) & 4]
        starts = {f[2] for f in mapped if f[3] == "1"}
        ends = {(f[2], int(f[1]) & 16) for f in mapped if int(f[3]) - 1 + _span(f[5]) == ctg_len[f[2]]}
        last = "ctg%d" % len(ctg_len)
        assert len(starts) >= 3 and len({e[0] for e in ends}) >= 3, (starts, ends)
        assert "ctg1" in starts and (last, 16) in ends  # position 0 and l_pac - 1, the latter by a reverse-strand read
    if c.lengths:
        assert set(c.lengths) <= {len(s) for s in c.seqs}
    if c.max_len:
        assert max(len(s) for s in c.seqs) <= c.max_len
    if c.unmapped:
        assert all(int(l.split("\t")[1]) & 4 for l in body.splitlines())


@pytest.fixture(scope="module")
def genomes(oracle, syn_index, edge_index):
    """case genome name -> (fasta, oracle index handle, contig lengths by name)"""
    out = {}
    for k, (fa, g, bounds) in (("syn", syn_index), ("edge", edge_index)):
        out[k] = (fa, oracle.load(fa), {"ctg%d" % (i + 1): int(bounds[i + 1] - bounds[i]) for i in range(len(bounds) - 1)})
    return out


@pytest.mark.parametrize("case", CASES)
def test_host_pipe_edge_case(oracle, hostsim, syn_index, edge_index, genomes, tmp_path, capfd, case):
    c = make_case(case, syn_index, edge_index)
    fa, idx, ctg_len = genomes[c.genome]
    body, streams, stats = oracle_case(oracle, idx, fa, c, b"rgE", tmp_path, capfd)
    assert hostsim.mem_pe(idx, c.names, c.seqs, c.quals, c.n_processed, b"rgE") == body
    assert hostsim.pipe(idx, c.names, c.seqs, c.quals, c.n_processed, b"rgE", 1, SB_TUPLE) == streams
    check_coverage(c, body, stats, ctg_len)
