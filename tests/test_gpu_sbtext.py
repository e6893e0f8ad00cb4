"""samblaster over SAM text on the device (ssq_sbtext_*, csrc/ssq_sbtext.cu): byte for byte, counters included, what the host
restatement of its routines gives (tests/test_sbtext_cpu.py holds that against the oracle), in one run and in runs of 7 blocks;
the same refusals; and the `samblaster` shim, whose unfused input now goes through it, against the oracle's samblaster — also on
a stream where one chunk in the middle is refused and goes through the shim's host code."""
import ctypes as C
import os
import subprocess

import pytest

try:  # before anything loads libssq: torch must bring in its own NCCL first
    import torch  # noqa: F401
except ImportError:
    pass

from test_gpu_cli import SAMBLASTER
from test_samblaster_shim_cpu import _fuzz_sam
from test_sbtext_cpu import (OPTION_SETS, REFUSALS, SSQ_EFORMAT, SbOpts, SbtOut, _rec, oracle_run, run_stream, sb_opts, sbt_host,  # noqa: F401  (fixture)
                             split_header, targeted_sam)

pytestmark = pytest.mark.gpu


class DevSbt:
    def __init__(self, lib):
        self.lib = lib
        lib.ssq_sbtext_create.argtypes = [C.c_int, C.POINTER(SbOpts), C.c_char_p, C.c_size_t, C.POINTER(C.c_void_p)]
        lib.ssq_sbtext_run.argtypes = [C.c_void_p, C.c_char_p, C.c_size_t, C.c_int, C.c_uint64, C.POINTER(C.c_size_t), C.POINTER(SbtOut)]
        lib.ssq_sbtext_free.argtypes = [C.c_void_p]
        lib.ssq_last_error.restype = C.c_char_p

    def create(self, header, opts):
        h = C.c_void_p()
        assert self.lib.ssq_sbtext_create(0, C.byref(opts), header, len(header), C.byref(h)) == 0, self.error()
        return h

    def run(self, h, text, final, max_blocks, used, out):
        return self.lib.ssq_sbtext_run(h, text, len(text), final, max_blocks, C.byref(used), C.byref(out))

    def error(self):
        return self.lib.ssq_last_error().decode()

    def free(self, h):
        self.lib.ssq_sbtext_free(h)


@pytest.fixture(scope="module")
def dev(ssq):
    return DevSbt(ssq.lib)


@pytest.fixture(scope="module")
def ex_dup_sam(oracle, ex_index, ex_reads):
    """the oracle's `bwa mem` SAM of the example reads plus 1,000 re-named duplicate pairs"""
    idx = oracle.load(ex_index)
    names, seqs, quals = ex_reads
    body = oracle.mem_pe(idx, names + ["dup_" + n for n in names[:1000]], seqs + seqs[:1000], quals + quals[:1000], 0, 8, b"")
    return ("@SQ\tSN:20_slice\tLN:321635\n" + body).encode()


def corpus(ex_dup_sam):
    items = [("fuzz%d" % s, _fuzz_sam(s, 1500), OPTION_SETS[s - 1] + ["--addMateTags"]) for s in (1, 2, 3, 4)]
    items.append(("targeted_crlf", targeted_sam(crlf=True, final_newline=False), ["--addMateTags", "--removeDups"]))
    items.append(("targeted", targeted_sam(), ["--excludeDups", "--addMateTags"]))
    items.append(("ex_dups", ex_dup_sam, ["--excludeDups", "--addMateTags", "--maxSplitCount", "2", "--minNonOverlap", "20"]))
    return items


def test_device_equals_the_host_restatement(dev, sbt_host, ex_dup_sam):
    for name, sam, args in corpus(ex_dup_sam):
        header, body = split_header(sam)
        for max_blocks in (0, 7):
            want = run_stream(sbt_host, header, body, sb_opts(args), max_blocks)
            got = run_stream(dev, header, body, sb_opts(args), max_blocks)
            assert got == want, (name, max_blocks)
            assert got[1][1] > 0, name  # duplicates were marked
        if name == "fuzz2":  # pieces that cut blocks and lines
            assert run_stream(dev, header, body, sb_opts(args), 0, 4099) == want


def test_device_refuses_what_the_host_restatement_refuses(dev, sbt_host):
    good = [_rec("g%d" % i, flag=f) for i in range(6) for f in ("65", "129")]
    for case, (bad, _) in sorted(REFUSALS.items()):
        text = ("\n".join(good[:7] + [bad] + good[7:]) + "\n").encode()
        msgs = []
        for api in (sbt_host, dev):
            h = api.create(b"@SQ\tSN:c1\tLN:1000\n", sb_opts(["--addMateTags"]))
            used, o = C.c_size_t(99), SbtOut()
            assert api.run(h, text, 1, 0, used, o) == SSQ_EFORMAT and used.value == 0, case
            msgs.append(api.error())
            api.free(h)
        assert msgs[0] == msgs[1] and "line 8 " in msgs[1], (case, msgs)


def _shim(exe, sam, args, tmp_path, env=None):
    spl, disc = str(tmp_path / "x.spl"), str(tmp_path / "x.disc")
    p = subprocess.run([exe] + args + ["--splitterFile", spl, "--discordantFile", disc], input=sam, check=True, stdout=subprocess.PIPE, stderr=subprocess.PIPE,
                       env=dict(os.environ, **(env or {})), timeout=300)
    from test_samblaster_shim_cpu import _strip_pg
    return [_strip_pg(p.stdout), _strip_pg(open(spl, "rb").read()), _strip_pg(open(disc, "rb").read())], p.stderr.decode()


def test_shim_equals_the_oracle(ex_dup_sam, tmp_path):
    for name, sam, args in corpus(ex_dup_sam):
        want, _ = oracle_run(sam, args, tmp_path)
        for env in ({"SSQ_SB_CHUNK": "7"}, {}):
            got, err = _shim(SAMBLASTER, sam, args, tmp_path, env)
            assert got == want, (name, env)
            assert "host code" not in err, name


def test_shim_refused_chunk_in_the_middle(tmp_path):
    """a QNAME block over the device's cap in the middle of the stream: the run of 7 blocks that holds it goes through the shim's host
    code, the runs before and after it through the device, and duplicates whose first occurrence lies on the other side of that chunk
    are still marked as the oracle marks them"""
    header, body = split_header(_fuzz_sam(8, 600))
    lines = body.decode().split("\n")[:-1]
    at, blk, prev = 0, 0, None
    for at, l in enumerate(lines):
        q = l.split("\t")[0]
        if q != prev:
            blk += 1; prev = q
        if blk == 300:
            break
    rec = lambda flag, c, pos, cg: "\t".join(["big", str(flag), c, str(pos), "60", cg, "=", "300", "0", "A" * 100, "I" * 100])
    big = [rec(0x41, "c1", 100, "50M50S")] + [rec(0x841, "c2", 500 + i, "50H50M") for i in range(299)] + [rec(0x81, "c1", 300, "100M")]  # 301 lines
    sam = header + ("\n".join(lines[:at] + big + lines[at:]) + "\n").encode()
    args = ["--addMateTags", "--excludeDups"]
    want, _ = oracle_run(sam, args, tmp_path)
    got, err = _shim(SAMBLASTER, sam, args, tmp_path, {"SSQ_SB_CHUNK": "7"})
    assert got == want
    assert "7 QNAME blocks went through the host code (1 chunks; the first: " in err and "more than 256 lines" in err, err
    # duplicates on both sides of the refused chunk exist in this stream (the corpus reuses few positions: later copies of a
    # signature are marked against first occurrences anywhere before them)
    recs = [l.split(b"\t") for l in want[0].split(b"\n") if l and not l.startswith(b"@")]
    at_big = next(i for i, r in enumerate(recs) if r[0] == b"big")
    dup_at = [i for i, r in enumerate(recs) if int(r[1]) & 0x400]
    assert sum(i < at_big for i in dup_at) > 5 and sum(i > at_big + 300 for i in dup_at) > 5
