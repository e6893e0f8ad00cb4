"""The edge cases of tests/test_pipe_edges_cpu.py (pair orientations and the statistics' thresholds, contig ends, mixed read lengths,
degenerate batches, read ordinals past 2^31) through the GPU's `bwa mem | samblaster` pipeline (ssq_aligner_* in include/ssq.h,
speedseq_b200/csrc/ssq_pipe.cu): plain records equal to the oracle's `bwa mem`, fused streams equal to its `bwa mem | samblaster`,
byte for byte; the statistics the device paired the batch with fail exactly where mem_pestat's do, and the device's mate rescue ran
where the case needs it and did nothing where no orientation has statistics.  Then several aligner objects, each on its own stream
and host thread, sharing one dup-set and ordered by turns (what bench.py and the CLI's lanes do), against one object and the oracle."""
import ctypes as C
import subprocess
import threading

import numpy as np
import pytest

import ssq_testlib as T
from speedseq_b200 import capi
from test_gpu_pipe import SB_SPEEDSEQ
from test_hostsim_pipe import sq_header
from test_pipe_edges_cpu import SB_ARGS, CASES, cat, check_coverage, edge_index, edge_pairs, genomes, make_case, oracle_case  # noqa: F401 (fixtures)

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def gpu_index(ssq, syn_index, edge_index):
    h = {"syn": ssq.index_load(syn_index[0]), "edge": ssq.index_load(edge_index[0])}
    yield h
    for x in h.values():
        ssq.index_free(x)


def run_gpu(ssq, h, c, sb):
    """one batch through a fresh aligner -> (three streams, info, {counter: value} for the mate-rescue counters)"""
    al = ssq.aligner_create(h, sb, b"rgE")
    try:
        rd, keep = T.pack_reads(c.names, c.seqs, c.quals, None, 1, c.n_processed)
        txt, info = ssq.aligner_run(al, rd)
        cnt = {k: int(ssq.lib.ssq_aligner_counter(al, k)) for k in (105, 107)}
    finally:
        ssq.aligner_free(al)
    return tuple(t.decode() for t in txt), info, cnt


@pytest.mark.parametrize("case", CASES)
def test_gpu_pipe_edge_case(ssq, oracle, syn_index, edge_index, genomes, gpu_index, tmp_path, capfd, case):
    c = make_case(case, syn_index, edge_index)
    fa, idx, ctg_len = genomes[c.genome]
    body, streams, stats = oracle_case(oracle, idx, fa, c, b"rgE", tmp_path, capfd)
    plain, _, _ = run_gpu(ssq, gpu_index[c.genome], c, None)
    assert plain[0] == body
    fused, info, cnt = run_gpu(ssq, gpu_index[c.genome], c, SB_SPEEDSEQ)
    assert fused[0] == streams[0]
    assert fused[1] == streams[1]
    assert fused[2] == streams[2]
    check_coverage(c, body, stats, ctg_len)
    assert tuple(p[2] for p in info["pes"]) == stats[1]  # the device's statistics fail where mem_pestat's do
    if c.rescue:
        assert cnt[105] > 0 and cnt[107] > 0, cnt
    if stats[1] == (1, 1, 1, 1):  # no orientation has statistics: no rescue window, nothing listed, nothing aligned
        assert cnt[105] == 0 and cnt[107] == 0, cnt


# ------------------------------------------------------------------------------------------------ concurrent lanes ----
LANE_PAIRS = (300, 260, 0, 1, 240, 330, 200, 169)  # eight batches of one run: one empty, one of a single pair


def lane_batches(g, bounds):
    """the batches of one run: duplicates of pairs near the end of the batch before open the next one (some with the ends swapped),
    the single-pair batch is a copy of the pair before it -> list of (names, seqs, quals), read offset of each batch"""
    names, seqs, quals = edge_pairs(g, bounds, sum(LANE_PAIRS), 31, orient=(1, 3, 2, 1), ins={"FF": (500, 50), "FR": (400, 40), "RF": (900, 60), "RR": (500, 50)},
                                    lengths=(60, 255), rescue_frac=0.1, prefix="b")
    for k in range(20, len(seqs) - 2, 50):  # improper pairs (discordant records): the mate of another fragment
        seqs[k + 1], quals[k + 1] = seqs[(k + 601) % len(seqs) | 1], quals[(k + 601) % len(seqs) | 1]
    for k in range(10, len(seqs), 40):  # chimeric reads (supplementary records, splitters)
        o = seqs[(k + 300) % len(seqs)]
        seqs[k] = seqs[k][:len(seqs[k]) // 2] + o[len(o) // 2:]  # (at most 127 + 128 bases)
        quals[k] = "I" * len(seqs[k])
    rng = np.random.default_rng(8)
    batches, at = [], 0
    for k, n in enumerate(LANE_PAIRS):
        if n == 1:
            batches.append((["single"] * 2, seqs[2 * at - 2:2 * at], quals[2 * at - 2:2 * at]))
            continue
        b = (names[2 * at:2 * (at + n)], seqs[2 * at:2 * (at + n)], quals[2 * at:2 * (at + n)])
        if at and n:
            d = ([], [], [])
            for i, j in enumerate(int(x) for x in rng.integers(max(0, at - 40), at, 12)):
                e = (2 * j, 2 * j + 1) if i % 3 else (2 * j + 1, 2 * j)
                d[0].extend(["dup%d_%d" % (k, i)] * 2); d[1].extend(seqs[x] for x in e); d[2].extend(quals[x] for x in e)
            b = cat(d, b)
        batches.append(b)
        at += n
    return batches, np.concatenate([[0], np.cumsum([len(b[0]) for b in batches])]).astype(int).tolist()


def oracle_run(oracle, fa, batches, offs, tmp):
    """the oracle's `bwa mem | samblaster` over the whole run: `bwa mem` per batch (its own statistics, global read ordinals)"""
    idx = oracle.load(fa)
    body = "".join(oracle.mem_pe(idx, *b, offs[k], 8, b"lane") for k, b in enumerate(batches) if b[0])
    spl, disc = str(tmp / "o.spl"), str(tmp / "o.disc")
    out = subprocess.run([T.ORACLE_BIN, "samblaster"] + SB_ARGS + ["--splitterFile", spl, "--discordantFile", disc], input=(sq_header(oracle, idx, fa) + body).encode(),
                         check=True, stdout=subprocess.PIPE, stderr=subprocess.DEVNULL).stdout.decode()
    rec = lambda t: "".join(l for l in t.splitlines(True) if not l.startswith("@"))
    return rec(out), rec(open(spl).read()), rec(open(disc).read())


@pytest.fixture(scope="module")
def lane_run(ssq, oracle, syn_index, gpu_index, tmp_path_factory):
    """the batches, the oracle's streams over the run, and the streams of one aligner object running the batches in order"""
    fa, g, bounds = syn_index
    batches, offs = lane_batches(g, bounds)
    want = oracle_run(oracle, fa, batches, offs, tmp_path_factory.mktemp("lanes"))
    al = ssq.aligner_create(gpu_index["syn"], SB_SPEEDSEQ, b"lane")
    one = []
    for k, b in enumerate(batches):
        rd, keep = T.pack_reads(*b, None, 1, offs[k])  # (keep: the buffers rd points into)
        one.append(ssq.aligner_run(al, rd)[0])
    ssq.aligner_free(al)
    return batches, offs, want, tuple("".join(r[i].decode() for r in one) for i in range(3))


def drive_lanes(ssq, h, batches, offs, n_obj):
    """n_obj aligner objects sharing one dup-set; object k runs batches k, k + n_obj, ... on its own host thread and stream with
    turn = batch number, so that the batches overlap on the device and first-seen-wins still follows input order -> per-batch streams"""
    L = ssq.lib
    L.ssq_dupset_create.argtypes = [C.c_int, C.c_void_p]
    L.ssq_dupset_free.argtypes = [C.c_void_p]
    L.ssq_aligner_set_turn.argtypes = [C.c_void_p, C.c_longlong]
    L.ssq_dupset_wait_turn.argtypes = [C.c_void_p, C.c_longlong]
    L.ssq_dupset_end_turn.argtypes = [C.c_void_p, C.c_longlong]
    dset = C.c_void_p()
    ssq.ck(L.ssq_dupset_create(0, C.byref(dset)), "ssq_dupset_create")
    als = [ssq.aligner_create(h, SB_SPEEDSEQ, b"lane") for _ in range(n_obj)]
    for al in als:
        ssq.ck(L.ssq_aligner_share_dupset(al, dset), "ssq_aligner_share_dupset")
    packed = [T.pack_reads(*b, None, 1, offs[k]) for k, b in enumerate(batches)]
    got, errors = [None] * len(batches), []

    def lane(k):
        for b in range(k, len(batches), n_obj):
            computing = False
            try:
                ssq.ck(L.ssq_aligner_set_turn(als[k], b), "ssq_aligner_set_turn")
                ssq.ck(L.ssq_aligner_upload(als[k], C.byref(packed[b][0])), "ssq_aligner_upload")
                computing = True  # ssq_aligner_compute ends the batch's turn whatever happens inside
                ssq.ck(L.ssq_aligner_compute(als[k], None, 0), "ssq_aligner_compute")
                sam = capi.Sam()
                ssq.ck(L.ssq_aligner_fetch(als[k], C.byref(sam)), "ssq_aligner_fetch")
                got[b] = tuple(C.string_at(sam.text[i], sam.len[i]).decode() for i in range(3))
            except Exception as e:  # noqa: BLE001 (reported below, after every lane has finished)
                errors.append((b, e))
            finally:
                if not computing:  # a batch that never reached the duplicate stage still ends its turn: later batches wait for it
                    L.ssq_dupset_wait_turn(dset, b)
                    L.ssq_dupset_end_turn(dset, b)
    threads = [threading.Thread(target=lane, args=(k,)) for k in range(n_obj)]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    for al in als:
        ssq.aligner_free(al)
    L.ssq_dupset_free(dset)
    assert not errors, errors
    return got


@pytest.mark.parametrize("n_obj", [2, 4])
def test_concurrent_lanes_share_the_dup_set(ssq, gpu_index, lane_run, n_obj):
    """run once per configuration: a difference is diffed and explained, not retried"""
    batches, offs, want, one = lane_run
    got = drive_lanes(ssq, gpu_index["syn"], batches, offs, n_obj)
    assert got[2] == ("", "", "")
    run = tuple("".join(g[i] for g in got) for i in range(3))
    for i in range(3):
        assert one[i] == want[i], i  # one object, batches in order
        assert run[i] == want[i], i  # n_obj objects, batches overlapping
    flag = lambda l: int(l.split("\t")[1])
    dup_names = {l.split("\t")[0] for l in run[0].splitlines() if flag(l) & 0x400}
    assert "single" in dup_names and sum(1 for n in dup_names if n.startswith("dup")) >= 40  # first occurrences in earlier batches
    assert len(run[1].splitlines()) > 0 and len(run[2].splitlines()) > 20
