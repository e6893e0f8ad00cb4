"""samblaster over SAM text (speedseq_b200/csrc/ssq_sbtext.cuh) run on the host by tests/hostsim/sbtext_host.cpp — the same SSQ_HD
routines in plain loops, compiled into a temporary directory — against the oracle's samblaster: the three streams byte for byte
(minus the @PG line) and its counters, on the fuzz corpus of the shim's CPU test, on targeted inputs (CIGAR ops = X N P H, MC / MQ
already present, CRLF, no final newline, QNAMEs starting with '@', FLAG re-printing, --removeDups, duplicate @SQ names, many
contigs), fed in one call and in blocks of 1, 7 and 64; plus the lines the device refuses."""
import ctypes as C
import os
import re
import subprocess

import pytest

import ssq_testlib as T
from test_samblaster_shim_cpu import _fuzz_sam, _strip_pg

SSQ_EFORMAT = -8
OPTION_SETS = [[], ["--excludeDups"], [], ["--excludeDups", "--maxSplitCount", "3", "--minNonOverlap", "10"]]  # those of the shim's fuzz test


class SbOpts(C.Structure):
    _fields_ = [(n, C.c_int32) for n in ("enabled", "exclude_dups", "add_mate_tags", "max_split_count", "min_non_overlap", "min_indel_size",
                                          "max_unmapped_bases", "remove_dups", "want_split", "want_disc")]


class SbtOut(C.Structure):
    _fields_ = [("text", C.c_void_p * 3), ("len", C.c_size_t * 3), ("n_ids", C.c_uint64), ("n_dup", C.c_uint64), ("n_disc_lines", C.c_uint64), ("n_split_lines", C.c_uint64)]


def sb_opts(args, split=True, disc=True):
    """the options a samblaster command line sets (the shim's defaults otherwise)"""
    o = SbOpts(1, 0, 0, 2, 20, 50, 50, 0, int(split), int(disc))
    it = iter(args)
    for a in it:
        if a == "--excludeDups": o.exclude_dups = 1
        elif a == "--addMateTags": o.add_mate_tags = 1
        elif a == "--removeDups": o.remove_dups = 1
        elif a == "--maxSplitCount": o.max_split_count = int(next(it))
        elif a == "--minNonOverlap": o.min_non_overlap = int(next(it))
        elif a == "--minIndelSize": o.min_indel_size = int(next(it))
        elif a == "--maxUnmappedBases": o.max_unmapped_bases = int(next(it))
        else: raise ValueError(a)
    return o


def split_header(sam):
    i = 0
    while i < len(sam) and sam[i:i + 1] == b"@":
        j = sam.find(b"\n", i)
        i = len(sam) if j < 0 else j + 1
    return sam[:i], sam[i:]


class HostSbt:
    """the host restatement behind the interface of ssq_sbtext_*"""
    def __init__(self, lib):
        self.lib = lib
        lib.hs_sbt_create.restype = C.c_void_p
        lib.hs_sbt_create.argtypes = [C.c_char_p, C.c_size_t, C.POINTER(SbOpts)]
        lib.hs_sbt_run.argtypes = [C.c_void_p, C.c_char_p, C.c_size_t, C.c_int, C.c_uint64, C.POINTER(C.c_size_t), C.POINTER(SbtOut)]
        lib.hs_sbt_free.argtypes = [C.c_void_p]
        lib.hs_sbt_error.restype = C.c_char_p

    def create(self, header, opts):
        return self.lib.hs_sbt_create(header, len(header), C.byref(opts))

    def run(self, h, text, final, max_blocks, used, out):
        return self.lib.hs_sbt_run(h, text, len(text), final, max_blocks, C.byref(used), C.byref(out))

    def error(self):
        return self.lib.hs_sbt_error().decode()

    def free(self, h):
        self.lib.hs_sbt_free(h)


def run_stream(api, header, body, opts, max_blocks=0, piece=None):
    """feed the record text through create/run/free the way the shim does (pieces of `piece` bytes, held-back bytes carried over);
    returns the three streams and the summed counters"""
    h = api.create(header, opts)
    outs, cnt = [b"", b"", b""], [0, 0, 0, 0]
    pending, at = b"", 0
    piece = piece or max(1, len(body))
    try:
        while True:
            if at < len(body) and (not pending or len(pending) < piece):
                pending += body[at:at + piece]; at += piece
            final = int(at >= len(body))
            used, o = C.c_size_t(0), SbtOut()
            rc = api.run(h, pending, final, max_blocks, used, o)
            assert rc == 0, (rc, api.error())
            for k in range(3):
                outs[k] += C.string_at(o.text[k], o.len[k]) if o.len[k] else b""
            cnt = [a + b for a, b in zip(cnt, (o.n_ids, o.n_dup, o.n_disc_lines, o.n_split_lines))]
            if final and used.value == len(pending):
                return outs, cnt
            assert used.value > 0 or not final or not pending
            if used.value == 0 and not final:
                pending += body[at:at + piece]; at += piece
                continue
            pending = pending[used.value:]
    finally:
        api.free(h)


def oracle_run(sam, args, tmp_path):
    spl, disc = str(tmp_path / "o.spl"), str(tmp_path / "o.disc")
    p = subprocess.run([T.ORACLE_BIN, "samblaster"] + args + ["--splitterFile", spl, "--discordantFile", disc], input=sam, check=True, stdout=subprocess.PIPE, stderr=subprocess.PIPE)
    err = p.stderr.decode()
    n_dup, n_ids = map(int, re.search(r"Marked (\d+) of (\d+)", err).groups())
    n_disc = int(re.search(r"Output (\d+) discordant", err).group(1))
    n_split = int(re.search(r"Output (\d+) split", err).group(1))
    return [_strip_pg(p.stdout), _strip_pg(open(spl, "rb").read()), _strip_pg(open(disc, "rb").read())], (n_ids, n_dup, n_disc, n_split)


def check_against_oracle(api, sam, args, tmp_path, max_blocks=0, piece=None):
    header, body = split_header(sam)
    want, wc = oracle_run(sam, args, tmp_path)
    got, cnt = run_stream(api, header, body, sb_opts(args), max_blocks, piece)
    for k, what in enumerate(("main", "splitters", "discordants")):
        assert header + got[k] == want[k], (what, max_blocks, piece)
    assert (cnt[0], cnt[1], cnt[2] // 2, cnt[3] // 2) == wc
    return got, cnt


def targeted_sam(seed=7, n_blocks=600, crlf=False, final_newline=True):
    """the fuzz corpus, rewritten: CIGAR ops = X N P, MC:Z / MQ:i already on some lines, FLAGs with leading zeros, QNAMEs starting with
    '@', contigs renamed into a table of 300 extra @SQ lines, a duplicate SN (first wins), CRLF line ends, no final newline"""
    header, body = split_header(_fuzz_sam(seed, n_blocks))
    hl = header.decode().splitlines()
    hl = hl[:4] + ["@SQ\tSN:x%d\tLN:%d" % (i, 2000 + 37 * i) for i in range(300)] + ["@SQ\tSN:c1\tLN:999", "@SQ\tSN:c2\tLN:77"] + hl[4:]
    lines = body.decode().splitlines()
    out, blk, prev = [], -1, None
    for i, l in enumerate(lines):
        f = l.split("\t")
        if f[0] != prev:
            blk += 1; prev = f[0]
        if blk % 3 == 0 and f[2] == "c3":
            f[2] = "x%d" % (blk % 300)
        if blk % 10 == 5:
            f[0] = "@" + f[0]
        cg = f[5]
        if cg != "*":
            k = i % 7
            if k == 0: cg = cg.replace("M", "=")
            elif k == 1: cg = cg.replace("M", "X", 1)
            elif k == 2: cg = cg.replace("D", "N")
            elif k == 3: cg = re.sub(r"^(\d+[A-Z=])", r"\g<1>2P", cg)
            elif k == 4: cg = re.sub(r"(\d+)M$", lambda m: "%d=1X%dM" % (int(m.group(1)) // 2, int(m.group(1)) - int(m.group(1)) // 2 - 1) if int(m.group(1)) > 3 else m.group(0), cg)
            f[5] = cg
        if i % 11 == 0:
            f.append("MC:Z:7M")
        if i % 13 == 0:
            f.append("MQ:i:5")
        if i % 17 == 0:
            f[1] = "00" + f[1]
        out.append("\t".join(f))
    nl = "\r\n" if crlf else "\n"
    text = nl.join(out) + (nl if final_newline else "")
    return ("\n".join(hl) + "\n").encode() + text.encode()


@pytest.fixture(scope="session")
def sbt_host(tmp_path_factory):
    d = tmp_path_factory.mktemp("sbtext_host")
    so = os.path.join(str(d), "libsbtext_host.so")
    subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-w", "-I", os.path.join(T.ROOT, "include"), "-o", so,
                    os.path.join(T.ROOT, "tests", "hostsim", "sbtext_host.cpp")], check=True)
    return HostSbt(C.CDLL(so))


@pytest.mark.parametrize("seed,max_blocks,extra", [(1, 0, OPTION_SETS[0]), (2, 7, OPTION_SETS[1]), (3, 1, OPTION_SETS[2]), (4, 64, OPTION_SETS[3])])
def test_fuzz_corpus_matches_oracle(sbt_host, tmp_path, seed, max_blocks, extra):
    got, cnt = check_against_oracle(sbt_host, _fuzz_sam(seed, 1500), extra + ["--addMateTags"], tmp_path, max_blocks)
    assert got[2].count(b"\n") > 50 and got[1].count(b"\n") > 20 and cnt[1] > 0


@pytest.mark.parametrize("variant", ["lf", "crlf", "no_final_newline", "crlf_no_final_newline"])
@pytest.mark.parametrize("extra", [["--addMateTags"], ["--addMateTags", "--removeDups"], ["--excludeDups", "--maxSplitCount", "3", "--minNonOverlap", "10"]])
def test_targeted_inputs_match_oracle(sbt_host, tmp_path, variant, extra):
    sam = targeted_sam(crlf="crlf" in variant, final_newline="no_final" not in variant)
    got, cnt = check_against_oracle(sbt_host, sam, extra, tmp_path)
    body = got[0]
    assert b"\n@q5\t" in body and re.search(rb"\t\d+=1X\d+M\t", body) and b"N" in body and b"2P" in body and b"H" in body
    assert cnt[1] > 0 and got[1].count(b"\n") > 10 and got[2].count(b"\n") > 10
    if "--removeDups" in extra:
        assert not any(int(l.split(b"\t")[1]) & 0x400 for l in body.split(b"\n") if l)
    if "--addMateTags" in extra:
        assert body.count(b"MC:Z:") > 100 and body.count(b"\tMC:Z:7M") >= 1
    if "crlf" in variant:
        assert b"\r\tMC:Z:" in body or "--addMateTags" not in extra


@pytest.mark.parametrize("max_blocks", [1, 7, 64])
def test_block_limits_and_pieces_give_one_runs_bytes(sbt_host, tmp_path, max_blocks):
    sam = targeted_sam(seed=9, n_blocks=400)
    header, body = split_header(sam)
    args = ["--addMateTags", "--excludeDups"]
    one, c1 = run_stream(sbt_host, header, body, sb_opts(args))
    for piece in (None, 997, 4096):
        got, c2 = run_stream(sbt_host, header, body, sb_opts(args), max_blocks, piece)
        assert got == one and c2 == c1, piece
    check_against_oracle(sbt_host, sam, args, tmp_path, max_blocks, 1500)


def test_a_block_cut_by_the_chunk_end_is_held_back(sbt_host):
    header, body = split_header(_fuzz_sam(5, 200))
    lines = body.split(b"\n")
    starts, prev, at = [], None, 0
    for l in lines:
        q = l.split(b"\t")[0]
        if q != prev:
            starts.append(at); prev = q
        at += len(l) + 1
    multi = next(i for i in range(10, len(starts) - 1) if body[starts[i]:starts[i + 1]].count(b"\n") >= 2)
    cut = starts[multi] + body[starts[multi]:].index(b"\n") + 1 + 3  # after the first line of a block and 3 bytes into its second
    h = sbt_host.create(header, sb_opts(["--addMateTags"]))
    used, o = C.c_size_t(0), SbtOut()
    assert sbt_host.run(h, body[:cut], 0, 0, used, o) == 0
    assert used.value == starts[multi] and o.n_ids == multi
    assert C.string_at(o.text[0], o.len[0]).count(b"\n") == body[:starts[multi]].count(b"\n")
    # one block in the text, not final: nothing taken yet
    assert sbt_host.run(h, body[starts[multi]:cut], 0, 0, used, o) == 0 and used.value == 0 and o.n_ids == 0
    sbt_host.free(h)


def test_shim_device_path_falls_back_to_the_host_code(oracle, tmp_path):
    """the shim built with its device text path, against a stand-in for ssq_sbtext_* that refuses every chunk: the host code takes
    the chunks over and the streams still equal the oracle's"""
    exe = str(tmp_path / "samblaster_refuse")
    subprocess.check_call(["gcc", "-O1", "-w", "-DSSQ_SB_DEVICE_TEXT", "-I" + os.path.join(T.ROOT, "include"), "-I" + os.path.join(T.ROOT, "speedseq_b200", "cli"), "-o", exe,
                           os.path.join(T.ROOT, "speedseq_b200", "cli", "samblaster_main.c"), os.path.join(T.ROOT, "tests", "stubs", "dupset_stub.c"),
                           os.path.join(T.ROOT, "tests", "stubs", "sbtext_refuse_stub.c")])
    for sam, args, chunk in ((_fuzz_sam(6, 1500), ["--excludeDups", "--addMateTags"], "7"), (targeted_sam(crlf=True, final_newline=False), ["--addMateTags", "--removeDups"], None)):
        want, _ = oracle_run(sam, args, tmp_path)
        spl, disc = str(tmp_path / "s.spl"), str(tmp_path / "s.disc")
        env = dict(os.environ, **({"SSQ_SB_CHUNK": chunk} if chunk else {}))
        p = subprocess.run([exe] + args + ["--splitterFile", spl, "--discordantFile", disc], input=sam, check=True, stdout=subprocess.PIPE, stderr=subprocess.PIPE, env=env)
        assert [_strip_pg(p.stdout), _strip_pg(open(spl, "rb").read()), _strip_pg(open(disc, "rb").read())] == want
        assert b"Marked" in p.stderr


def _rec(name, flag="65", rname="c1", pos="5", cigar="10M", n_extra=0):
    return "\t".join([name, flag, rname, pos, "60", cigar, "=", "9", "0", "A" * 10, "I" * 10] + ["XX:i:%d" % i for i in range(n_extra)])


REFUSALS = {
    "fields": ("\t".join(_rec("bad").split("\t")[:10]), "fewer than 11 fields"),
    "flag_letters": (_rec("bad", flag="6a5"), "FLAG"),
    "flag_empty": (_rec("bad", flag=""), "FLAG"),
    "flag_sign": (_rec("bad", flag="+65"), "FLAG"),
    "flag_long": (_rec("bad", flag="1234567890"), "FLAG"),
    "pos_negative": (_rec("bad", pos="-5"), "POS"),
    "pos_letters": (_rec("bad", pos="5x"), "POS"),
    "cigar_trailing_digits": (_rec("bad", cigar="10M5"), "CIGAR"),
    "cigar_unknown_op": (_rec("bad", cigar="10Q"), "CIGAR"),
    "cigar_no_length": (_rec("bad", cigar="M"), "CIGAR"),
    "cigar_empty": (_rec("bad", cigar=""), "CIGAR"),
    "cigar_huge": (_rec("bad", cigar="268435456M"), "CIGAR"),
    "rname_unknown": (_rec("bad", rname="chrUn"), "RNAME"),
    "rname_star_mapped": (_rec("bad", flag="0", rname="*"), "RNAME '*'"),
    "nul_byte": (_rec("bad").replace("IIII", "II\0I"), "NUL"),
    "block_over_cap": ("\n".join(_rec("bad", flag="2113" if i else "65") for i in range(257)), "QNAME block of more than 256 lines"),
}


@pytest.mark.parametrize("case", sorted(REFUSALS))
def test_refused_lines(sbt_host, case):
    bad, why = REFUSALS[case]
    good = [_rec("g%d" % i, flag=f) for i in range(6) for f in ("65", "129")]
    text = ("\n".join(good[:7] + [bad] + good[7:]) + "\n").encode()
    h = sbt_host.create(b"@SQ\tSN:c1\tLN:1000\n", sb_opts(["--addMateTags"]))
    used, o = C.c_size_t(123), SbtOut()
    assert sbt_host.run(h, text, 1, 0, used, o) == SSQ_EFORMAT
    msg = sbt_host.error()
    assert used.value == 0 and "line 8 " in msg and why in msg, msg
    # the same line inside the held-back last block is not looked at yet
    text2 = ("\n".join(good + [bad.replace("bad", "g5")]) + "\n").encode() if case != "block_over_cap" else None
    if text2 is not None:
        assert sbt_host.run(h, text2, 0, 0, used, o) == 0 and o.n_ids == 5
    sbt_host.free(h)
