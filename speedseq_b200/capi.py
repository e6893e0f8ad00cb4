"""ctypes bindings of the product's C-ABI (include/ssq.h -> speedseq_b200/libssq.so): record dtypes and a thin wrapper class.
No compute happens here and nothing under oracle/ or tests/ is imported: bench.py and the tests bind the library through this
module.  The library has no CPU path; SSQ() raises when it has not been built."""
import ctypes as C
import os

import numpy as np

SSQ_SO = os.path.join(os.path.dirname(os.path.abspath(__file__)), "libssq.so")

SMEM_DT = np.dtype([("k", "<u8"), ("l", "<u8"), ("s", "<u8"), ("qbeg", "<u4"), ("qend", "<u4")])
SEED_DT = np.dtype([("rbeg", "<i8"), ("qbeg", "<i4"), ("len", "<i4")])
SWTASK_DT = np.dtype([("q_off", "<u8"), ("t_off", "<u8"), ("qlen", "<i4"), ("tlen", "<i4"), ("h0", "<i4"), ("w", "<i4"),
                      ("end_bonus", "<i4"), ("zdrop", "<i4")])
SWRES_DT = np.dtype([("score", "<i4"), ("qle", "<i4"), ("tle", "<i4"), ("gtle", "<i4"), ("gscore", "<i4"), ("max_off", "<i4")])
REG_DT = np.dtype([("rb", "<i8"), ("re", "<i8"), ("qb", "<i4"), ("qe", "<i4"), ("rid", "<i4"), ("score", "<i4"), ("truesc", "<i4"),
                   ("w", "<i4"), ("seedcov", "<i4"), ("seedlen0", "<i4"), ("frac_rep", "<f4"), ("read_id", "<i4")])
DUPSIG_DT = np.dtype([("pos1", "<u8"), ("pos2", "<u8"), ("strand1", "u1"), ("strand2", "u1"), ("valid", "u1"), ("pad", "u1", (5,))])
SWLTASK_DT = np.dtype([("q_off", "<u8"), ("t_off", "<u8"), ("qlen", "<i4"), ("tlen", "<i4"), ("xtra", "<i4"), ("pad", "<i4")])
SWLRES_DT = np.dtype([("score", "<i4"), ("te", "<i4"), ("qe", "<i4"), ("score2", "<i4"), ("te2", "<i4"), ("tb", "<i4"), ("qb", "<i4")])
SWGTASK_DT = np.dtype([("q_off", "<u8"), ("t_off", "<u8"), ("qlen", "<i4"), ("tlen", "<i4"), ("w", "<i4"), ("cig_cap", "<i4"), ("cig_off", "<u8")])
SWGRES_DT = np.dtype([("score", "<i4"), ("n_cigar", "<i4")])

assert SMEM_DT.itemsize == 32 and SEED_DT.itemsize == 16 and SWTASK_DT.itemsize == 40 and REG_DT.itemsize == 56 and DUPSIG_DT.itemsize == 24
assert SWLTASK_DT.itemsize == 32 and SWLRES_DT.itemsize == 28 and SWGTASK_DT.itemsize == 40 and SWGRES_DT.itemsize == 8


def _ptr(a):
    return a.ctypes.data_as(C.c_void_p)


class SbOpts(C.Structure):
    """ssq_sb_opts_t"""
    _fields_ = [(n, C.c_int32) for n in ("enabled", "exclude_dups", "add_mate_tags", "max_split_count", "min_non_overlap", "min_indel_size", "max_unmapped_bases",
                                         "remove_dups", "want_split", "want_disc")]


class Reads(C.Structure):
    """ssq_reads_t"""
    _fields_ = [("n_reads", C.c_int32), ("paired", C.c_int32), ("seq", C.c_void_p), ("seq_off", C.c_void_p), ("qual", C.c_void_p), ("name", C.c_void_p), ("name_off", C.c_void_p),
                ("comment", C.c_void_p), ("comment_off", C.c_void_p), ("n_processed", C.c_int64)]


class PeStat(C.Structure):
    """ssq_pestat_t"""
    _fields_ = [("low", C.c_int32), ("high", C.c_int32), ("failed", C.c_int32), ("pad", C.c_int32), ("avg", C.c_double), ("std", C.c_double)]


class Sam(C.Structure):
    """ssq_sam_t"""
    _fields_ = [("text", C.c_void_p * 3), ("len", C.c_size_t * 3), ("read_off", C.c_void_p), ("n_ids", C.c_uint64), ("n_dup", C.c_uint64), ("pes", PeStat * 4)]


def pack_reads(names, seqs, quals=None, comments=None, paired=1, n_processed=0):
    """lists of str/bytes -> (Reads, keepalive): the concatenated layout ssq_aligner_run() takes"""
    b = lambda x: x if isinstance(x, bytes) else x.encode()
    n = len(names)
    seqb = b"".join(b(x) for x in seqs)
    seq_off = np.zeros(n + 1, np.uint64); seq_off[1:] = np.cumsum([len(x) for x in seqs])
    nameb = b"".join(b(x) for x in names)
    name_off = np.zeros(n + 1, np.uint32); name_off[1:] = np.cumsum([len(b(x)) for x in names])
    keep = [np.frombuffer(seqb, np.uint8) if seqb else np.zeros(1, np.uint8), seq_off, np.frombuffer(nameb, np.uint8) if nameb else np.zeros(1, np.uint8), name_off]
    r = Reads()
    r.n_reads, r.paired, r.n_processed = n, paired, n_processed
    r.seq, r.seq_off, r.name, r.name_off = keep[0].ctypes.data, seq_off.ctypes.data, keep[2].ctypes.data, name_off.ctypes.data
    if quals is not None:
        qb = b"".join(b(x) for x in quals)
        keep.append(np.frombuffer(qb, np.uint8) if qb else np.zeros(1, np.uint8))
        r.qual = keep[-1].ctypes.data
    if comments is not None:
        cb = b"".join(b(x or "") for x in comments)
        co = np.zeros(n + 1, np.uint32); co[1:] = np.cumsum([len(b(x or "")) for x in comments])
        keep += [np.frombuffer(cb, np.uint8) if cb else np.zeros(1, np.uint8), co]
        r.comment, r.comment_off = keep[-2].ctypes.data, co.ctypes.data
    return r, keep


class IndexBuildOpts(C.Structure):
    _fields_ = [("path", C.c_int32), ("pad", C.c_int32), ("work_bytes", C.c_uint64)]


class IndexBuildStats(C.Structure):
    _fields_ = [("path", C.c_int32), ("pad", C.c_int32)] + [(k, C.c_int64) for k in
                ("passes", "rounds", "chunks", "unresolved_first", "largest_group", "oversize_groups", "peak_device_bytes", "ranges")]


class SSQ:
    """the product's C-ABI (include/ssq.h); raises when libssq.so is missing — there is no fallback"""
    OPTS_WORDS = 30

    def __init__(self):
        if not os.path.exists(SSQ_SO):
            raise RuntimeError("speedseq_b200/libssq.so is not built; run __graft_entry__.build() — the path has no fallback")
        self.lib = C.CDLL(SSQ_SO)
        L = self.lib
        L.ssq_last_error.restype = C.c_char_p
        L.ssq_index_info.restype = C.c_uint64
        L.ssq_index_info.argtypes = [C.c_void_p, C.c_int]
        L.ssq_batch_counter.restype = C.c_uint64
        L.ssq_batch_counter.argtypes = [C.c_void_p, C.c_int]
        L.ssq_batch_stage_ms.restype = C.c_float
        L.ssq_batch_stage_ms.argtypes = [C.c_void_p, C.c_int]
        L.ssq_batch_stream.restype = C.c_void_p
        L.ssq_batch_stream.argtypes = [C.c_void_p]
        self.opts = (C.c_int32 * self.OPTS_WORDS)()
        L.ssq_opts_default(self.opts)

    def err(self):
        return self.lib.ssq_last_error().decode()

    def ck(self, rc, what):
        if rc != 0:
            raise RuntimeError("%s failed: rc=%d: %s" % (what, rc, self.err()))

    def index_load(self, prefix, device=0):
        h = C.c_void_p()
        self.ck(self.lib.ssq_index_load(prefix.encode(), C.c_int(device), C.byref(h)), "ssq_index_load")
        return h

    def index_build(self, fasta, prefix=None, device=0):
        self.ck(self.lib.ssq_index_build(fasta.encode(), (prefix or fasta).encode(), C.c_int(device)), "ssq_index_build")

    def index_build_ex(self, fasta, prefix=None, device=0, path=0, work_bytes=0):
        """ssq_index_build_ex: path 0 auto, 2 device (multi-pass) sort, 3 host; work_bytes = the
        multi-pass working budget (0: from free device memory).  Returns the stats as a dict ("path" = the path that ran)."""
        opt = IndexBuildOpts(path, 0, work_bytes)
        st = IndexBuildStats()
        self.ck(self.lib.ssq_index_build_ex(fasta.encode(), (prefix or fasta).encode(), C.c_int(device), C.byref(opt), C.byref(st)), "ssq_index_build_ex")
        return {k: getattr(st, k) for k, _ in IndexBuildStats._fields_ if k != "pad"}

    def index_free(self, h):
        self.lib.ssq_index_free(h)

    def smem_batch(self, idx, seq, off):
        n = len(off) - 1
        cap = max(1024, 64 * n)
        while True:
            out = np.zeros(cap, SMEM_DT)
            ooff = np.zeros(n + 1, np.uint64)
            need = C.c_uint64(0)
            rc = self.lib.ssq_smem_batch(idx, self.opts, C.c_int(n), _ptr(seq), _ptr(off), _ptr(out), C.c_uint64(cap), _ptr(ooff), C.byref(need))
            if rc == -5:
                cap = int(need.value) + 16
                continue
            self.ck(rc, "ssq_smem_batch")
            return out[: int(need.value)], ooff

    def sa_lookup_batch(self, idx, rows):
        pos = np.zeros(len(rows), np.uint64)
        self.ck(self.lib.ssq_sa_lookup_batch(idx, C.c_uint64(len(rows)), _ptr(rows), _ptr(pos)), "ssq_sa_lookup_batch")
        return pos

    def make_opts(self, **kw):
        """ssq_opts_t: the defaults with the named scoring fields (a, b, o_del, e_del, o_ins, e_ins) replaced"""
        o = (C.c_int32 * self.OPTS_WORDS)()
        C.memmove(o, self.opts, C.sizeof(o))
        for k, v in kw.items():
            o[("a", "b", "o_del", "e_del", "o_ins", "e_ins").index(k)] = int(v)
        return o

    def sw_extend_batch(self, tasks, qbuf, tbuf, device=0, opts=None):
        res = np.zeros(len(tasks), SWRES_DT)
        self.ck(self.lib.ssq_sw_extend_batch(opts or self.opts, C.c_int(device), C.c_uint64(len(tasks)), _ptr(tasks), _ptr(qbuf), C.c_uint64(len(qbuf)), _ptr(tbuf),
                                             C.c_uint64(len(tbuf)), _ptr(res)), "ssq_sw_extend_batch")
        return res

    def sw_local_batch(self, tasks, qbuf, tbuf, device=0, opts=None):
        """ksw_align2 problems (SWLTASK_DT) -> SWLRES_DT"""
        res = np.zeros(len(tasks), SWLRES_DT)
        self.ck(self.lib.ssq_sw_local_batch(opts or self.opts, C.c_int(device), C.c_uint64(len(tasks)), _ptr(tasks), _ptr(qbuf), C.c_uint64(len(qbuf)), _ptr(tbuf),
                                            C.c_uint64(len(tbuf)), _ptr(res)), "ssq_sw_local_batch")
        return res

    def sw_global_batch(self, tasks, qbuf, tbuf, cig, device=0, opts=None):
        """ksw_global2 problems (SWGTASK_DT) -> SWGRES_DT; the CIGAR of task i is written to cig[cig_off, +n_cigar) (a uint32 array)"""
        res = np.zeros(len(tasks), SWGRES_DT)
        self.ck(self.lib.ssq_sw_global_batch(opts or self.opts, C.c_int(device), C.c_uint64(len(tasks)), _ptr(tasks), _ptr(qbuf), C.c_uint64(len(qbuf)), _ptr(tbuf),
                                             C.c_uint64(len(tbuf)), _ptr(cig), C.c_uint64(len(cig)), _ptr(res)), "ssq_sw_global_batch")
        return res

    def chain_batch(self, idx, seq, off):
        n = len(off) - 1
        scap, ccap = max(4096, 256 * n), max(1024, 64 * n)
        while True:
            seeds = np.zeros(scap, SEED_DT)
            cso = np.zeros(ccap + 1, np.uint64)
            rco = np.zeros(n + 1, np.uint64)
            nc, ns = C.c_uint64(0), C.c_uint64(0)
            rc = self.lib.ssq_chain_batch(idx, self.opts, C.c_int(n), _ptr(seq), _ptr(off), _ptr(seeds), C.c_uint64(scap), _ptr(cso), C.c_uint64(ccap), _ptr(rco),
                                          C.byref(nc), C.byref(ns))
            if rc == -5:
                scap, ccap = int(ns.value) + 16, int(nc.value) + 16
                continue
            self.ck(rc, "ssq_chain_batch")
            return seeds[: int(ns.value)], cso[: int(nc.value) + 1], rco

    def align_batch(self, idx, seq, off):
        n = len(off) - 1
        cap = max(1024, 16 * n)
        while True:
            out = np.zeros(cap, REG_DT)
            ooff = np.zeros(n + 1, np.uint64)
            need = C.c_uint64(0)
            rc = self.lib.ssq_align_batch(idx, self.opts, C.c_int(n), _ptr(seq), _ptr(off), C.c_int(0), _ptr(out), C.c_uint64(cap), _ptr(ooff), C.byref(need))
            if rc == -5:
                cap = int(need.value) + 16
                continue
            self.ck(rc, "ssq_align_batch")
            return out[: int(need.value)], ooff

    def dupmark_batch(self, sig, device=0):
        d = np.zeros(len(sig), np.uint8)
        self.ck(self.lib.ssq_dupmark_batch(C.c_int(device), C.c_uint64(len(sig)), _ptr(sig), _ptr(d)), "ssq_dupmark_batch")
        return d

    # ---- the HBM-resident `bwa mem | samblaster` pipeline ----
    def aligner_create(self, idx, sb=None, rg_id=b""):
        """sb: None (plain `bwa mem`) or dict(exclude_dups=.., add_mate_tags=.., max_split_count=.., min_non_overlap=.., remove_dups=..)"""
        L = self.lib
        L.ssq_aligner_stage_ms.restype = C.c_float
        L.ssq_aligner_stage_ms.argtypes = [C.c_void_p, C.c_int]
        L.ssq_aligner_counter.restype = C.c_uint64
        L.ssq_aligner_counter.argtypes = [C.c_void_p, C.c_int]
        L.ssq_aligner_stream.restype = C.c_void_p
        L.ssq_aligner_stream.argtypes = [C.c_void_p]
        L.ssq_aligner_free.argtypes = [C.c_void_p]
        so = SbOpts()
        L.ssq_sb_opts_default(C.byref(so))
        if sb is not None:
            so.enabled, so.want_split, so.want_disc = 1, 1, 1
            for k, v in sb.items():
                setattr(so, k, int(v))
        h = C.c_void_p()
        self.ck(L.ssq_aligner_create(idx, self.opts, C.byref(so), rg_id if isinstance(rg_id, bytes) else rg_id.encode(), C.byref(h)), "ssq_aligner_create")
        return h

    def aligner_run(self, al, reads, pes=None, verbose=0):
        """reads: Reads (pack_reads) -> ((main, splitters, discordants) as bytes, info dict)"""
        out = Sam()
        pv = None
        if pes is not None:
            pv = (PeStat * 4)()
            for d in range(4):
                pv[d].low, pv[d].high, pv[d].failed, pv[d].avg, pv[d].std = int(pes[d][0]), int(pes[d][1]), int(pes[d][2]), float(pes[d][3]), float(pes[d][4])
        self.ck(self.lib.ssq_aligner_run(al, C.byref(reads), pv, C.c_int(verbose), C.byref(out)), "ssq_aligner_run")
        # everything is copied here: the buffers behind `out` belong to the aligner and are reused by its next run
        info = {"n_ids": int(out.n_ids), "n_dup": int(out.n_dup), "pes": [(p.low, p.high, p.failed, p.avg, p.std) for p in out.pes],
                "read_off": np.ctypeslib.as_array((C.c_uint64 * (reads.n_reads + 1)).from_address(out.read_off)).copy()}
        return tuple(C.string_at(out.text[k], out.len[k]) for k in range(3)), info

    def aligner_free(self, al):
        self.lib.ssq_aligner_free(al)

    # ---- BGZF compression on the device (ssq_bgzf_*) ----
    def bgzf_create(self, device=0):
        L = self.lib
        L.ssq_bgzf_stream.restype = C.c_void_p
        L.ssq_bgzf_stream.argtypes = [C.c_void_p]
        L.ssq_bgzf_free.argtypes = [C.c_void_p]
        L.ssq_free.argtypes = [C.c_void_p]
        h = C.c_void_p()
        self.ck(L.ssq_bgzf_create(C.c_int(device), C.byref(h)), "ssq_bgzf_create")
        return h

    def bgzf_deflate(self, z, data, level=6, with_eof=1):
        """bytes (or a buffer) in host memory -> the BGZF file as bytes"""
        buf = np.frombuffer(data, np.uint8) if len(data) else np.zeros(1, np.uint8)
        out, n = C.c_void_p(), C.c_size_t(0)
        self.ck(self.lib.ssq_bgzf_deflate(z, _ptr(buf), C.c_size_t(len(data)), C.c_int(level), C.c_int(with_eof), C.byref(out), C.byref(n)), "ssq_bgzf_deflate")
        r = C.string_at(out, n.value)
        self.lib.ssq_free(out)
        return r

    def bgzf_deflate_dev(self, z, d_in, n, d_out, out_cap, level=6, with_eof=1):
        """device pointers (ints) -> (rc, out_len, needed); rc is SSQ_ECAP (-5) when out_cap is too small"""
        ln, need = C.c_size_t(0), C.c_size_t(0)
        rc = self.lib.ssq_bgzf_deflate_dev(z, C.c_void_p(d_in), C.c_size_t(n), C.c_int(level), C.c_int(with_eof), C.c_void_p(d_out), C.c_size_t(out_cap), C.byref(ln), C.byref(need))
        if rc not in (0, -5):
            self.ck(rc, "ssq_bgzf_deflate_dev")
        return rc, int(ln.value), int(need.value)

    def bgzf_stream(self, z):
        return self.lib.ssq_bgzf_stream(z)

    def bgzf_free(self, z):
        self.lib.ssq_bgzf_free(z)

    # ---- gzip decoding on the device (ssq_gunzip_*) ----
    def gunzip_create(self, device=0, chunk_bytes=0):
        L = self.lib
        L.ssq_gunzip_stream.restype = C.c_void_p
        L.ssq_gunzip_stream.argtypes = [C.c_void_p]
        L.ssq_gunzip_free.argtypes = [C.c_void_p]
        L.ssq_gunzip_stats.argtypes = [C.c_void_p, C.c_void_p]
        L.ssq_gunzip_inflate.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_int, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p]
        L.ssq_gunzip_inflate_dev.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_void_p]
        h = C.c_void_p()
        self.ck(L.ssq_gunzip_create(C.c_int(device), C.c_size_t(chunk_bytes), C.byref(h)), "ssq_gunzip_create")
        return h

    def gunzip_inflate(self, g, data, final, out):
        """one streaming call into the uint8 array `out`: -> (rc, used, text bytes, done); rc is 0 or SSQ_EDATA (-9)"""
        buf = np.frombuffer(data, np.uint8) if len(data) else np.zeros(1, np.uint8)
        used, ln, done = C.c_size_t(0), C.c_size_t(0), C.c_int(0)
        rc = self.lib.ssq_gunzip_inflate(g, _ptr(buf), C.c_size_t(len(data)), C.c_int(final), C.byref(used), _ptr(out), C.c_size_t(len(out)), C.byref(ln), C.byref(done))
        if rc not in (0, -9):
            self.ck(rc, "ssq_gunzip_inflate")
        return rc, int(used.value), out[:ln.value].tobytes(), bool(done.value)

    def gunzip(self, g, data, piece=1 << 62, out_cap=64 << 20):
        """a whole stream through the streaming call, `piece` more bytes per call after the unconsumed rest: -> (rc, text)"""
        pend, at, text, out = bytearray(), 0, [], np.empty(max(out_cap, 1), np.uint8)
        while True:
            if at < len(data):
                pend += data[at:at + piece]
                at += piece
            rc, used, t, done = self.gunzip_inflate(g, pend, int(at >= len(data)), out[:out_cap])
            if rc:
                return rc, b"".join(text)
            text.append(t)
            del pend[:used]
            if done:
                return 0, b"".join(text)

    def gunzip_inflate_dev(self, g, d_in, n, d_out, out_cap):
        """device pointers (ints) -> (rc, out_len); rc is 0, SSQ_ECAP (-5) or SSQ_EDATA (-9)"""
        ln = C.c_size_t(0)
        rc = self.lib.ssq_gunzip_inflate_dev(g, C.c_void_p(d_in), C.c_size_t(n), C.c_void_p(d_out), C.c_size_t(out_cap), C.byref(ln))
        if rc not in (0, -5, -9):
            self.ck(rc, "ssq_gunzip_inflate_dev")
        return rc, int(ln.value)

    def gunzip_stats(self, g):
        """(chunks decoded, chunks started at a searched sync point, chunks decoded again after a broken link, windows) since create"""
        s = (C.c_int64 * 4)()
        self.ck(self.lib.ssq_gunzip_stats(g, s), "ssq_gunzip_stats")
        return tuple(s)

    def gunzip_stream(self, g):
        return self.lib.ssq_gunzip_stream(g)

    def gunzip_free(self, g):
        self.lib.ssq_gunzip_free(g)
