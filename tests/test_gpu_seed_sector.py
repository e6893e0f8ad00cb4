"""GPU parity of the seeding with the one-sector rank query (both interval ends in one 64-row block: one load) and the k-mer table
in the forward walks (built at index load by default): intervals and aligned records equal the oracle's with the table off (SSQ_KMER_K=0: the one-sector step
alone), at the default K and at K = 8, on simulated reads plus reads whose intervals touch the primary row, N runs, homopolymers
and short tandem repeats.  tests/test_seed_sector_cpu.py checks the same routines on the host."""
import numpy as np
import pytest

import ssq_testlib as T

pytestmark = pytest.mark.gpu


def _reads(syn_index, n=1500, seed=47):
    fa, g, bounds = syn_index
    names, seqs, quals = T.simulate_pairs(g, bounds, n, 150, seed, err=0.01, indel=0.002, n_frac=0.003)
    acgt = "ACGT"
    head = "".join(acgt[x] for x in g[:150])  # the text's first suffix: its row is the primary row
    tail = "".join(acgt[x] for x in g[int(bounds[-1]) - 150:int(bounds[-1])])
    rc = tail[::-1].translate(str.maketrans("ACGT", "TGCA"))
    return seqs + [head, head[:40], rc, "", "A", "N" * 30, "N" * 10 + head[10:], head[:70] + "NN" + head[72:], "AC" * 70, "A" * 150,
                   "ACGT" * 37, "T" * 100, "AAG" * 50, "CA" * 30 + "G" * 30 + "TTA" * 30]


@pytest.mark.parametrize("kmer", ["0", None, "8"])
def test_seeding_one_sector_and_table(ssq, oracle, syn_index, monkeypatch, kmer):
    if kmer is not None:
        monkeypatch.setenv("SSQ_KMER_K", kmer)  # read by ssq_index_load
    else:
        monkeypatch.delenv("SSQ_KMER_K", raising=False)
    fa = syn_index[0]
    idx = oracle.load(fa)
    h = ssq.index_load(fa)
    try:
        seq, off = T.encode_reads(_reads(syn_index))
        a, ao = oracle.smem_batch(idx, seq, off)
        b, bo = ssq.smem_batch(h, seq, off)
        assert np.array_equal(ao, bo) and np.array_equal(a, b)
        a, ao = oracle.align_batch(idx, seq, off)
        b, bo = ssq.align_batch(h, seq, off)
        assert np.array_equal(ao, bo) and np.array_equal(a, b)
    finally:
        ssq.index_free(h)
