"""The device Smith-Waterman routines on inputs chosen to break them, against the oracle's ksw_global2 / ksw_align2 / ksw_extend2 with
an explicit matrix and explicit gap penalties, bit-exact, under four scoring sets (problem sets and checks: test_sw_kernels_cpu.py,
which holds the scalar forms to the same problems):
  * sw_global_warp (the CIGAR stage's banded global DP, a warp per problem with lanes = band columns and F as a shuffle scan carried
    from one 32-column chunk to the next) through ssq_sw_global_batch: bands of 1..8 chunks, the end cell on the band edge, tied
    paths, and CIGARs one operation too long for their buffer (-1, never cut short);
  * sw_local_warp (mate rescue) through ssq_sw_local_batch, in both byte-mode forms (SSQ_RESCUE_SPLIT=0: 16 lanes, 1: 32 lanes),
    at every SLEN of their register templates, with saturation, N in the target (shared-memory form) and tlen 0 / 1;
  * sw_extend through ssq_sw_extend_batch with z-drop firing, band 1, end bonus 0 and large, h0 near qlen * a."""
import numpy as np
import pytest

from test_sw_kernels_cpu import (SCORINGS, check_global, extend_coverage, extend_problems, global_coverage, global_problems, local_coverage,
                                 local_problems, oracle_extend, oracle_local)

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def gprob():
    return global_problems()


def test_sw_global_warp_vs_oracle(ssq, oracle, gprob):
    tasks, qbuf, tbuf, kinds = gprob
    need = {}
    for name, sc in SCORINGS.items():
        opts = ssq.make_opts(**sc)
        need[name] = check_global(lambda tk, cig: ssq.sw_global_batch(tk, qbuf, tbuf, cig, opts=opts), oracle, sc, tasks, qbuf, tbuf, kinds)
    global_coverage(tasks, kinds, need)


@pytest.mark.parametrize("split", ["0", "1"])
@pytest.mark.parametrize("name", list(SCORINGS))
def test_sw_local_warp_vs_oracle(ssq, oracle, monkeypatch, name, split):
    monkeypatch.setenv("SSQ_RESCUE_SPLIT", split)
    sc = SCORINGS[name]
    tasks, qbuf, tbuf, tags = local_problems(sc, 5 + list(SCORINGS).index(name))
    ref = oracle_local(oracle, sc, tasks, qbuf, tbuf)
    got = ssq.sw_local_batch(tasks, qbuf, tbuf, opts=ssq.make_opts(**sc))
    bad = np.nonzero(got != ref)[0]
    assert len(bad) == 0, (bad[:5], got[bad[:5]], ref[bad[:5]], tasks[bad[:5]])
    local_coverage(tasks, tags, ref)


@pytest.mark.parametrize("name", list(SCORINGS))
def test_sw_extend_vs_oracle(ssq, oracle, name):
    sc = SCORINGS[name]
    tasks, qbuf, tbuf = extend_problems(sc, 31 + list(SCORINGS).index(name))
    ref = oracle_extend(oracle, sc, tasks, qbuf, tbuf)
    got = ssq.sw_extend_batch(tasks, qbuf, tbuf, opts=ssq.make_opts(**sc))
    bad = np.nonzero(got != ref)[0]
    assert len(bad) == 0, (bad[:5], got[bad[:5]], ref[bad[:5]], tasks[bad[:5]])
    extend_coverage(oracle, sc, tasks, qbuf, tbuf, ref)
