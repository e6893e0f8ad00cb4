"""The three Smith-Waterman routines on inputs chosen to break them, host side: the scalar forms the kernels are checked against
(ssq_dev2.cuh: sw_global, sw_local; ssq_dev.cuh: sw_extend; tests/hostsim/sw_host.cpp runs them on the host) against the oracle's
ksw_global2 / ksw_align2 / ksw_extend2 called directly with an explicit 5x5 matrix and explicit gap penalties, under four scoring
sets.  Every comparison is bit-exact.  The problem sets are built here and shared with tests/test_gpu_sw_kernels.py, which puts the
device routines (the warp forms of ssq_warp.cuh through ssq_sw_global_batch / ssq_sw_local_batch, and ssq_sw_extend_batch) to the
same problems.  What the problem sets reach (band chunks, SLEN cases, saturation, N, tied paths, CIGAR overflow) is asserted."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import ssq_testlib as T
from speedseq_b200.capi import SWGTASK_DT, SWGRES_DT, SWLTASK_DT, SWLRES_DT, SWRES_DT

SCORINGS = {
    "default": dict(a=1, b=4, o_del=6, e_del=1, o_ins=6, e_ins=1),
    "asym_gaps": dict(a=1, b=4, o_del=5, e_del=2, o_ins=8, e_ins=1),
    "a2b3_asym": dict(a=2, b=3, o_del=4, e_del=3, o_ins=7, e_ins=2),
    "cheap_gaps": dict(a=1, b=4, o_del=1, e_del=1, o_ins=1, e_ins=1),
}
XBYTE, XSTOP, XSUBO, XSTART = 0x10000, 0x20000, 0x40000, 0x80000
WG_RCAP = 2048          # longest target of the warp global DP (ssq_warp.cuh)
CIG_CAP_ALN = 62        # operations the pipeline's CIGAR stage leaves to the global DP (CIG_CAP - 2, ssq_dev3.cuh)
QLENS = [1, 2, 31, 32, 33, 63, 64, 65, 127, 128, 129, 200, 250, 255]
# band half-widths: n_col = min(qlen, 2w + 1) covers 1..8 chunks of 32 columns and ends 31 / 33 columns into a chunk
WIDTHS = [0, 1, 2, 15, 16, 31, 32, 47, 48, 63, 64, 79, 80, 95, 96, 111, 112, 126, 127, 300]
GKINDS = ["copy", "subs", "indel_start", "indel_mid", "indel_end", "band_edge", "homopolymer", "str", "n", "random"]


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def seqs_of(k, qbuf, tbuf):
    """query and target of one task record"""
    qo, to = int(k["q_off"]), int(k["t_off"])
    return qbuf[qo:qo + int(k["qlen"])], tbuf[to:to + int(k["tlen"])]


def matrix(sc):
    """the oracle's 5x5 matrix: a on the diagonal, -b off it, -1 against N (ssq_dev2.cuh: score_of)"""
    m = np.full((5, 5), -sc["b"], np.int8)
    np.fill_diagonal(m, sc["a"])
    m[4, :] = -1
    m[:, 4] = -1
    return m.ravel().copy()


def host_scoring(sc):
    """the scoring argument of the sw_host routines: {a, b, o_del, e_del, o_ins, e_ins}"""
    return (C.c_int32 * 6)(*[sc[k] for k in ("a", "b", "o_del", "e_del", "o_ins", "e_ins")])


def build_sw_host(d):
    """tests/hostsim/sw_host.cpp -> a shared library in directory d (the scalar SW routines compiled for the host)"""
    so = os.path.join(str(d), "libsw_host.so")
    subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-w", "-o", so, os.path.join(T.ROOT, "tests", "hostsim", "sw_host.cpp")], check=True)
    return C.CDLL(so)


@pytest.fixture(scope="module")
def sw_host(tmp_path_factory):
    return build_sw_host(tmp_path_factory.mktemp("sw_host"))


# ------------------------------------------------------------------------------------------------ oracle ----
def oracle_global(o, sc, q, t, w):
    """ksw_global2 -> (score, CIGAR words)"""
    mat = matrix(sc)
    n, p = C.c_int(0), C.POINTER(C.c_uint32)()
    s = o.lib.ssqo_ksw_global2(C.c_int(len(q)), _p(q), C.c_int(len(t)), _p(t), C.c_int(5), _p(mat), C.c_int(sc["o_del"]), C.c_int(sc["e_del"]),
                               C.c_int(sc["o_ins"]), C.c_int(sc["e_ins"]), C.c_int(w), C.byref(n), C.byref(p))
    cig = np.array([p[i] for i in range(n.value)], np.uint32)
    o.lib.ssqo_api_free(C.cast(p, C.c_void_p))
    return s, cig


class _KR(C.Structure):
    _fields_ = [(k, C.c_int) for k in SWLRES_DT.names]


def oracle_local(o, sc, tasks, qbuf, tbuf):
    o.lib.ssqo_ksw_align2.restype = _KR
    mat = matrix(sc)
    out = np.zeros(len(tasks), SWLRES_DT)
    for i, k in enumerate(tasks):
        q, t = (x.copy() for x in seqs_of(k, qbuf, tbuf))
        q = q if len(q) else np.zeros(1, np.uint8)
        t = t if len(t) else np.zeros(1, np.uint8)
        r = o.lib.ssqo_ksw_align2(C.c_int(int(k["qlen"])), _p(q), C.c_int(int(k["tlen"])), _p(t), C.c_int(5), _p(mat), C.c_int(sc["o_del"]), C.c_int(sc["e_del"]),
                                  C.c_int(sc["o_ins"]), C.c_int(sc["e_ins"]), C.c_int(int(k["xtra"])))
        out[i] = tuple(getattr(r, f) for f in SWLRES_DT.names)
    return out


def oracle_extend(o, sc, tasks, qbuf, tbuf):
    mat = matrix(sc)
    out = np.zeros(len(tasks), SWRES_DT)
    v = [C.c_int() for _ in range(5)]
    for i, k in enumerate(tasks):
        q, t = seqs_of(k, qbuf, tbuf)
        s = o.lib.ssqo_ksw_extend2(C.c_int(int(k["qlen"])), _p(q), C.c_int(int(k["tlen"])), _p(t), C.c_int(5), _p(mat), C.c_int(sc["o_del"]), C.c_int(sc["e_del"]),
                                   C.c_int(sc["o_ins"]), C.c_int(sc["e_ins"]), C.c_int(int(k["w"])), C.c_int(int(k["end_bonus"])), C.c_int(int(k["zdrop"])),
                                   C.c_int(int(k["h0"])), *[C.byref(x) for x in v])
        out[i] = (s,) + tuple(x.value for x in v)
    return out


# --------------------------------------------------------------------------------------- global DP ----
def _fit(rng, t, tlen, where):
    """insert random bases into / delete bases from t at `where` (start, mid, end, or a position) until it has tlen bases"""
    d = tlen - len(t)
    if d == 0:
        return t
    p = {"start": 0, "mid": len(t) // 2, "end": len(t)}.get(where, where)
    if d > 0:
        return np.concatenate([t[:p], rng.integers(0, 4, d, dtype=np.uint8), t[p:]])
    p = min(p, len(t) + d)
    return np.concatenate([t[:p], t[p - d:]])


def _global_pair(rng, kind, qlen, tlen, w):
    q = rng.integers(0, 4, qlen, dtype=np.uint8)
    if kind == "homopolymer":
        q[:] = rng.integers(0, 4)
        return q, np.full(tlen, q[0], np.uint8)
    if kind == "str":
        unit = rng.integers(0, 4, int(rng.integers(2, 4)), dtype=np.uint8)
        rep = lambda n: np.resize(unit, n)
        return rep(qlen), rep(tlen)
    if kind == "random":
        return q, rng.integers(0, 4, tlen, dtype=np.uint8)
    t = q.copy()
    if kind in ("subs", "n", "indel_start", "indel_mid", "indel_end"):
        m = rng.random(qlen) < 0.04
        t[m] = (t[m] + rng.integers(1, 4, int(m.sum()), dtype=np.uint8)) % 4
    if kind == "n":
        q[rng.integers(0, qlen, 1 + qlen // 50)] = 4
        t[rng.integers(0, qlen, 1 + qlen // 50)] = 4
    where = int(rng.integers(0, qlen + 1))
    if kind.startswith("indel_"):
        where = kind[6:]
        if tlen == qlen and w >= 10 and qlen >= 40:  # a balanced pair of 10-60 bp gaps that stays inside the band
            L = int(rng.integers(10, min(60, w, qlen // 4) + 1))
            p = {"start": 0, "mid": qlen // 2 - L, "end": qlen - 2 * L}[where]
            p = max(0, p)
            t = np.concatenate([t[:p], t[p + L:p + 2 * L], rng.integers(0, 4, L, dtype=np.uint8), t[p + 2 * L:]])[:qlen]
    if kind == "band_edge":
        where = "start" if rng.random() < 0.5 else "end"
    return q, _fit(rng, t, tlen, where)


def global_problems(seed=11):
    """(tasks without CIGAR capacities, qbuf, tbuf, per-task kind): every qlen of QLENS against widths that span 1..8 chunks, length
    differences from -w to +w, and the target kinds of GKINDS; plus targets of the longest length the warp routine takes"""
    rng = np.random.default_rng(seed)
    probs = []
    for qlen in QLENS:
        for w in WIDTHS:
            if w > qlen + 2 and w not in (300,):
                continue
            dls = sorted({-w, -w + 1, -1, 0, 1, w - 1, w})
            for dl in dls:
                tlen = qlen + dl
                if abs(dl) > w or tlen < 1 or tlen > WG_RCAP:
                    continue
                kinds = list(rng.choice(GKINDS, 2, replace=False))
                if abs(dl) == w and w > 0:
                    kinds.append("band_edge")
                if dl != 0 and rng.random() < 0.3:
                    kinds.append("homopolymer" if rng.random() < 0.5 else "str")
                for kind in kinds:
                    probs.append((kind, qlen, tlen, w))
    for qlen, w in ((255, WG_RCAP - 255), (200, WG_RCAP - 200), (64, WG_RCAP)):
        probs.append(("band_edge", qlen, WG_RCAP, w))
    tasks = np.zeros(len(probs), SWGTASK_DT)
    qs, ts, kinds = [], [], []
    qo = to = 0
    for i, (kind, qlen, tlen, w) in enumerate(probs):
        q, t = _global_pair(rng, kind, qlen, tlen, w)
        assert len(q) == qlen and len(t) == tlen, (kind, qlen, tlen, len(q), len(t))
        tasks[i] = (qo, to, qlen, tlen, w, 0, 0)
        qs.append(q); ts.append(t); kinds.append(kind)
        qo += qlen; to += tlen
    return tasks, np.concatenate(qs), np.concatenate(ts), np.array(kinds)


def with_caps(tasks, caps):
    """a copy of the tasks with CIGAR capacities `caps` laid out back to back; returns (tasks, cig buffer)"""
    t = tasks.copy()
    t["cig_cap"] = caps
    t["cig_off"] = np.concatenate([[0], np.cumsum(caps)[:-1]]).astype(np.uint64)
    return t, np.zeros(max(1, int(np.sum(caps))), np.uint32)


def oracle_global_batch(o, sc, tasks, qbuf, tbuf):
    """(scores, list of CIGAR arrays)"""
    sc_, cigs = np.zeros(len(tasks), np.int32), []
    for i, k in enumerate(tasks):
        s, c = oracle_global(o, sc, *seqs_of(k, qbuf, tbuf), int(k["w"]))
        sc_[i] = s
        cigs.append(c)
    return sc_, cigs


def cigar_score(sc, q, t, cig):
    """score of an alignment given by its CIGAR, recomputed from the sequences; also checks that it consumes both exactly"""
    x = y = s = 0
    for c in cig.tolist():
        op, ln = c & 0xf, c >> 4
        assert ln > 0 and op in (0, 1, 2), cig
        if op == 0:
            a, b = q[x:x + ln], t[y:y + ln]
            s += int(np.where((a > 3) | (b > 3), -1, np.where(a == b, sc["a"], -sc["b"])).sum())
            x += ln; y += ln
        elif op == 1:
            s -= sc["o_ins"] + sc["e_ins"] * ln; x += ln
        else:
            s -= sc["o_del"] + sc["e_del"] * ln; y += ln
    assert (x, y) == (len(q), len(t)), (x, y, len(q), len(t))
    return s


def check_global(run, o, sc, tasks, qbuf, tbuf, kinds):
    """run(tasks, cig) -> results, for the exact CIGAR capacity, one below it and zero (score only), against the oracle.  Returns
    the oracle's CIGAR lengths."""
    want_s, want_c = oracle_global_batch(o, sc, tasks, qbuf, tbuf)
    need = np.array([len(c) for c in want_c], np.int32)
    # the oracle's own answers are consistent: CIGARs consume both sequences and re-score to the score
    for i, k in enumerate(tasks):
        q, t = seqs_of(k, qbuf, tbuf)
        assert cigar_score(sc, q, t, want_c[i]) == want_s[i], (i, kinds[i], tasks[i])
    tk, cig = with_caps(tasks, need)
    got = run(tk, cig)
    bad = [i for i in range(len(tasks)) if got["score"][i] != want_s[i] or got["n_cigar"][i] != need[i] or
           not np.array_equal(cig[int(tk["cig_off"][i]):int(tk["cig_off"][i]) + need[i]], want_c[i])]
    assert not bad, [(i, kinds[i], tasks[i], got[i], want_s[i], want_c[i][:8], cig[int(tk["cig_off"][i]):int(tk["cig_off"][i]) + need[i]][:8]) for i in bad[:4]]
    # one operation short: reported as -1, the score is still computed.  (need 1 - 1 = 0 is the score-only case below)
    short = need > 1
    tk, cig = with_caps(tasks, np.where(short, need - 1, 1))
    got = run(tk, cig)
    assert (got["n_cigar"][short] == -1).all() and (got["n_cigar"][~short] == 1).all() and np.array_equal(got["score"], want_s)
    # score only
    tk, cig = with_caps(tasks, np.zeros(len(tasks), np.int32))
    got = run(tk, cig)
    assert (got["n_cigar"] == 0).all() and np.array_equal(got["score"], want_s)
    return need


def global_coverage(tasks, kinds, need_by_scoring):
    """what the global problem sets reach, asserted so that a change to the generator cannot quietly test less"""
    w = tasks["w"].astype(np.int64)
    n_col = np.minimum(tasks["qlen"], 2 * w + 1)
    chunks = (n_col + 31) // 32
    assert set(chunks.tolist()) >= set(range(1, 9)), sorted(set(chunks.tolist()))
    multi = n_col > 32
    assert {31, 0, 1} <= set((n_col[multi] % 32).tolist())
    dl = tasks["tlen"].astype(np.int64) - tasks["qlen"]
    assert ((dl == w) & (w > 0)).sum() >= 50 and ((dl == -w) & (w > 0)).sum() >= 50
    assert (tasks["tlen"] == WG_RCAP).sum() >= 3
    assert set(tasks["qlen"].tolist()) == set(QLENS)
    assert set(kinds.tolist()) == set(GKINDS)
    tied = np.isin(kinds, ["homopolymer", "str"]) & (dl != 0)
    assert tied.sum() >= 100
    assert (np.isin(kinds, ["n"])).sum() >= 20
    for name, need in need_by_scoring.items():
        assert (need > 1).sum() > 0.8 * len(need), name
    assert (need_by_scoring["cheap_gaps"] > CIG_CAP_ALN).sum() >= 20, "no problem needs more operations than the CIGAR stage has room for"


@pytest.fixture(scope="module")
def gprob():
    return global_problems()


def test_sw_global_scalar_vs_oracle(oracle, sw_host, gprob):
    """sw_global (the scalar form; the warp form is held to the same problems in test_gpu_sw_kernels.py) equals ksw_global2 bit for
    bit: score, CIGAR, and -1 when the CIGAR does not fit — under each scoring set"""
    tasks, qbuf, tbuf, kinds = gprob
    need = {}
    for name, sc in SCORINGS.items():
        scv = host_scoring(sc)

        def run(tk, cig):
            res = np.zeros(len(tk), SWGRES_DT)
            assert sw_host.swhost_global_batch(scv, C.c_uint64(len(tk)), _p(tk), _p(qbuf), _p(tbuf), _p(cig), _p(res)) == 0
            return res
        need[name] = check_global(run, oracle, sc, tasks, qbuf, tbuf, kinds)
    global_coverage(tasks, kinds, need)


def test_sw_global_refuses_bad_tasks(sw_host):
    """a task whose end cell lies outside the band (|tlen - qlen| > w), or whose lengths are out of range, is refused before anything
    runs — by the host routine and by ssq_sw_global_batch, which checks its tasks before it looks for a GPU"""
    ssq = T.SSQ()
    q, t = np.zeros(300, np.uint8), np.zeros(WG_RCAP + 8, np.uint8)
    cig = np.zeros(64, np.uint32)
    scv = host_scoring(SCORINGS["default"])
    good = (0, 0, 100, 104, 4, 8, 0)
    for bad in [(0, 0, 100, 105, 4, 8, 0), (0, 0, 100, 95, 4, 8, 0), (0, 0, 0, 1, 4, 8, 0), (0, 0, 256, 256, 4, 8, 0), (0, 0, 10, 0, 10, 8, 0),
                (0, 0, 100, WG_RCAP + 1, WG_RCAP, 8, 0), (0, 0, 10, 10, -1, 8, 0), (0, 0, 10, 10, 1, -1, 0)]:
        tk = np.array([good, bad], SWGTASK_DT)
        res = np.zeros(2, SWGRES_DT)
        assert sw_host.swhost_global_batch(scv, C.c_uint64(2), _p(tk), _p(q), _p(t), _p(cig), _p(res)) == -4, bad
        assert ssq.lib.ssq_sw_global_batch(ssq.opts, C.c_int(0), C.c_uint64(2), _p(tk), _p(q), C.c_uint64(len(q)), _p(t), C.c_uint64(len(t)), _p(cig),
                                           C.c_uint64(len(cig)), _p(res)) == -4, bad
    for bad in [(290, 0, 20, 20, 4, 8, 0), (0, WG_RCAP, 20, 20, 4, 8, 0), (0, 0, 20, 20, 4, 8, 60)]:  # buffers too short for the task
        tk = np.array([good, bad], SWGTASK_DT)
        assert ssq.lib.ssq_sw_global_batch(ssq.opts, C.c_int(0), C.c_uint64(2), _p(tk), _p(q), C.c_uint64(len(q)), _p(t), C.c_uint64(len(t)), _p(cig),
                                           C.c_uint64(len(cig)), _p(np.zeros(2, SWGRES_DT))) == -4, bad


# ---------------------------------------------------------------------------------------- local SW ----
def local_problems(sc, seed):
    """ksw_align2 problems for one scoring set: byte mode at every SLEN (1..16 cells per striped segment) and word mode, planted
    near-exact copies long enough to saturate the byte score, targets holding N, tlen 0 and 1, with and without start coordinates
    and sub-optimal hits.  Returns (tasks, qbuf, tbuf, tags) with tags a dict of boolean arrays."""
    rng = np.random.default_rng(seed)
    a = sc["a"]
    rows = []
    qls = [s * 16 - d for s in range(1, 17) for d in (0, 7, 15)]
    qls = [min(q, 255) for q in qls]
    for rep in range(2):
        for ql in qls:
            for mode in ("byte", "word"):
                rows.append((ql, mode, "plant"))
        for ql in [1, 5, 16, 17, 40, 100, 150, 255]:
            rows += [(ql, "byte", "tgt_n"), (ql, "word", "tgt_n"), (ql, "byte", "tlen0"), (ql, "byte", "tlen1"), (ql, "word", "tlen1")]
    lo = -(-250 // a)  # qlen * a >= 250
    for ql in rng.integers(max(lo, 1), 256, 24).tolist() + [255, 253, 251, lo]:
        if ql <= 255:
            rows.append((int(ql), "byte", "saturate"))
    tasks = np.zeros(len(rows), SWLTASK_DT)
    qs, ts = [], []
    tags = {k: np.zeros(len(rows), bool) for k in ("byte", "tgt_n", "saturate_try", "tlen01")}
    qo = to = 0
    for i, (ql, mode, kind) in enumerate(rows):
        q = rng.integers(0, 4, ql, dtype=np.uint8)
        if kind == "tlen0":
            t = np.zeros(0, np.uint8)
        elif kind == "tlen1":
            t = rng.integers(0, 4, 1, dtype=np.uint8)
        else:
            tl = int(rng.integers(ql, ql + 400))
            t = rng.integers(0, 4, tl, dtype=np.uint8)
            for r in range(1 + (rng.random() < 0.3)):
                c = q.copy()
                if kind != "saturate":
                    m = rng.random(ql) < 0.03
                    c[m] = rng.integers(0, 4, int(m.sum()), dtype=np.uint8)
                    if ql > 30 and rng.random() < 0.3:
                        p = int(rng.integers(5, ql - 5))
                        c = np.concatenate([c[:p], c[p + int(rng.integers(1, 4)):]]) if rng.random() < 0.5 else \
                            np.concatenate([c[:p], rng.integers(0, 4, int(rng.integers(1, 4)), dtype=np.uint8), c[p:]])
                at = int(rng.integers(0, tl - len(c) + 1)) if tl >= len(c) else 0
                t[at:at + len(c)] = c[:tl - at]
            if kind == "tgt_n":
                t[rng.integers(0, tl, 1 + int(rng.integers(0, 3)))] = 4
            elif rng.random() < 0.05:
                q[rng.integers(0, ql)] = 4
        minsc = int(rng.choice([10, 19, 30]))
        xtra = XSUBO | XSTART | minsc
        if i % 9 == 0:
            xtra &= ~XSTART
        if i % 13 == 0:
            xtra &= ~XSUBO
        if mode == "byte":
            xtra |= XBYTE
        tasks[i] = (qo, to, ql, len(t), xtra, 0)
        tags["byte"][i] = mode == "byte"
        tags["tgt_n"][i] = bool((t > 3).any())
        tags["saturate_try"][i] = kind == "saturate"
        tags["tlen01"][i] = len(t) <= 1
        qs.append(q); ts.append(t)
        qo += ql; to += len(t)
    return tasks, np.concatenate(qs), np.concatenate(ts + [np.zeros(1, np.uint8)]), tags


def local_coverage(tasks, tags, ref):
    """what the local problem sets reach"""
    byte, no_n = tags["byte"], ~tags["tgt_n"]
    slen = (tasks["qlen"] + 15) // 16
    assert set(slen[byte & no_n & ~tags["tlen01"]].tolist()) == set(range(1, 17)), "a byte-mode register form (SLEN 1..16) is not reached"
    assert (~byte & ~tags["tlen01"]).sum() >= 50                             # word mode
    assert (byte & tags["tgt_n"]).sum() >= 10                                 # the fallback to the shared-memory form
    assert (tasks["tlen"] == 0).sum() >= 5 and (tasks["tlen"] == 1).sum() >= 5
    assert (ref["score"][byte] == 255).sum() > 0, "byte saturation never reached"
    assert (ref["score2"] >= 0).sum() > 0 and (ref["tb"] >= 0).sum() > 100


@pytest.mark.parametrize("name", list(SCORINGS))
def test_sw_local_scalar_vs_oracle(oracle, sw_host, name):
    """sw_local (the striped kernel's evaluation order, the routine the warp forms are held to) equals ksw_align2 in every field"""
    sc = SCORINGS[name]
    tasks, qbuf, tbuf, tags = local_problems(sc, 5 + list(SCORINGS).index(name))
    ref = oracle_local(oracle, sc, tasks, qbuf, tbuf)
    got = np.zeros(len(tasks), SWLRES_DT)
    assert sw_host.swhost_local_batch(host_scoring(sc), C.c_uint64(len(tasks)), _p(tasks), _p(qbuf), _p(tbuf), _p(got)) == 0
    bad = np.nonzero(got != ref)[0]
    assert len(bad) == 0, (bad[:5], got[bad[:5]], ref[bad[:5]], tasks[bad[:5]])
    local_coverage(tasks, tags, ref)


# --------------------------------------------------------------------------------------- extension ----
def extend_problems(sc, seed, n=600):
    """ksw_extend2 problems: small z-drop (1, 10) so that it fires, end bonus 0 and large, band 1, h0 near qlen * a"""
    rng = np.random.default_rng(seed)
    tasks, qbuf, tbuf = T.extension_tasks(rng, n)
    tasks["zdrop"] = rng.choice([1, 10, 100], n)
    tasks["end_bonus"] = rng.choice([0, 5, 1000], n)
    tasks["w"] = np.where(rng.random(n) < 0.3, 1, tasks["w"])
    near = rng.random(n) < 0.3
    tasks["h0"] = np.where(near, np.maximum(1, tasks["qlen"] * sc["a"] - rng.integers(0, 5, n)), tasks["h0"])
    return tasks, qbuf, tbuf


def extend_coverage(o, sc, tasks, qbuf, tbuf, ref):
    """what the extension problem sets reach; z-drop counts as fired where switching it off changes the oracle's answer"""
    assert (tasks["zdrop"] <= 10).sum() > 100 and (tasks["w"] == 1).sum() > 100 and (tasks["end_bonus"] == 0).sum() > 100
    assert (tasks["end_bonus"] >= 1000).sum() > 100 and (tasks["h0"] >= tasks["qlen"] * sc["a"] - 4).sum() > 100
    no_z = tasks.copy()
    no_z["zdrop"] = 1 << 20
    assert (oracle_extend(o, sc, no_z, qbuf, tbuf) != ref).sum() > 50, "z-drop never changes a result"
    assert (ref["gscore"] > 0).sum() > 50 and (ref["score"] > tasks["h0"]).sum() > 50


@pytest.mark.parametrize("name", list(SCORINGS))
def test_sw_extend_scalar_vs_oracle(oracle, sw_host, name):
    """sw_extend (ssq_dev.cuh, the body of the extension kernels) equals ksw_extend2 in every field under each scoring set"""
    sc = SCORINGS[name]
    tasks, qbuf, tbuf = extend_problems(sc, 31 + list(SCORINGS).index(name))
    ref = oracle_extend(oracle, sc, tasks, qbuf, tbuf)
    got = np.zeros(len(tasks), SWRES_DT)
    assert sw_host.swhost_extend_batch(host_scoring(sc), C.c_uint64(len(tasks)), _p(tasks), _p(qbuf), _p(tbuf), _p(got)) == 0
    bad = np.nonzero(got != ref)[0]
    assert len(bad) == 0, (bad[:5], got[bad[:5]], ref[bad[:5]], tasks[bad[:5]])
    extend_coverage(oracle, sc, tasks, qbuf, tbuf, ref)
