"""`sambamba merge` on the device against speedseq's sambamba.  Makes the coordinate-sorted record text of tools/bai_bench.py
(about --gb GB: 150-base records over 24 references, 3 % unmapped at their mate's position, 5,000 without coordinates), gives
every record a random read group out of k and writes one BGZF file per group (the header of each names all k read groups, as a
split of one library's BAM does; compressed on the device at level 1), for k = 2, 3 and 7, in a temporary directory.  Then
reports, as one JSON line:
  - the card (name, power limit, SM clock, read in one nvidia-smi call before the runs);
  - per k, a warm ssq_merge_run of the k files: wall clock and ssq_merge_times (windows: read, copy in, inflate, walk, keys; the
    host heap; gathers and output), with the output handed back uncompressed and with it compressed on the device;
  - per k, wall clock of the `sambamba` shim's `merge -t 16` (SSQ_MERGE_GPU=1; host zlib and device BGZF; its .bai included)
    and of the staged sambamba's `merge -t 16` of the same files, and whether the decompressed files are identical.
Exits non-zero when the shim's merged file differs from the staged sambamba's.
usage: python tools/merge_bench.py [--gb 2] [--ks 2,3,7]"""
import argparse
import ctypes as C
import gzip
import hashlib
import json
import os
import struct
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))
from bai_bench import make_text  # noqa: E402
from golden.make_bai_golden import header, record  # noqa: E402
from golden.make_merge_golden import bam_header  # noqa: E402
from speedseq_b200.capi import SSQ  # noqa: E402

SHIM = os.path.join(ROOT, "speedseq_b200", "bin", "sambamba")
REAL = os.path.join(ROOT, "oracle", "_ref", "stage", "src", "sambamba")
REFS = [("chr%d" % (i + 1), 240000000) for i in range(24)]


def split_inputs(s, d, gb, ks=(2, 3, 7), seed=7):
    """{k: [paths of the k files]}: bai_bench's records split by a random read group"""
    text, _ = make_text(gb)
    rec = text[len(header(REFS)):]
    L = len(record("read0000000", 99, 0, 0, "150M"))
    nocoor_at = rec.find(b"nocoor0\0") - 36  # the main records are all L bytes long; those without coordinates follow
    n = nocoor_at // L
    main = np.frombuffer(rec, np.uint8, n * L).reshape(n, L)
    nocoor, at = [], nocoor_at
    while at < len(rec):
        ln = 4 + struct.unpack_from("<i", rec, at)[0]
        nocoor.append(rec[at:at + ln])
        at += ln
    rng = np.random.default_rng(seed)
    z = s.bgzf_create(0)
    out = {}
    try:
        for k in ks:
            rg = b"".join(b"@RG\tID:rg%d\tSM:sample\tLB:lib%d\n" % (g, g) for g in range(k))
            hdr = bam_header(b"@HD\tVN:1.3\tSO:coordinate\n" + b"".join(b"@SQ\tSN:%s\tLN:%d\n" % (a.encode(), b) for a, b in REFS) + rg +
                             b"@PG\tID:bwa\tPN:bwa\tVN:0.7.10\n", REFS)
            grp = rng.integers(0, k, n)
            out[k] = []
            for g in range(k):
                p = os.path.join(str(d), "k%d_rg%d.bam" % (k, g))
                open(p, "wb").write(s.bgzf_deflate(z, hdr + main[grp == g].tobytes() + b"".join(nocoor[g::k]), 1, 1))
                out[k].append(p)
    finally:
        s.bgzf_free(z)
    return out


def digest(path):
    h = hashlib.sha256()
    with gzip.open(path) as f:
        for b in iter(lambda: f.read(64 << 20), b""):
            h.update(b)
    return h.hexdigest()


def wall(args, env=None):
    t0 = time.perf_counter()
    subprocess.run(args, check=True, env=env, stdout=subprocess.DEVNULL)
    return time.perf_counter() - t0


def device_run(s, m, paths, z):
    """one ssq_merge_run into a sink that counts bytes -> (wall s, ms[3], records, output bytes)"""
    got = [0]

    def put(ctx, p, n):
        got[0] += n
        return 0
    sink = s._MERGE_SINK(put)
    arr = (C.c_char_p * len(paths))(*[os.fsencode(p) for p in paths])
    nrec = C.c_uint64(0)
    t0 = time.perf_counter()
    rc = s.lib.ssq_merge_run(m, arr, len(paths), z, C.c_int(1), sink, None, C.byref(nrec))
    w = time.perf_counter() - t0
    assert rc == 0, s.err()
    return w, s.merge_times(m), int(nrec.value), got[0]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gb", type=float, default=2.0)
    ap.add_argument("--ks", default="2,3,7")
    a = ap.parse_args()
    ks = [int(x) for x in a.ks.split(",")]
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    s = SSQ()
    res = {"card": card, "gb": a.gb, "runs": {}}
    ok = True
    with tempfile.TemporaryDirectory() as d:
        files = split_inputs(s, d, a.gb, ks)
        m = s.merge_create(0)
        z = s.bgzf_create(0)
        device_run(s, m, files[ks[0]], None)  # warm: buffers sized, modules loaded
        for k in ks:
            r = {"compressed_bytes": sum(os.path.getsize(p) for p in files[k])}
            for name, zz in (("device_host_out", None), ("device_bgzf_out", z)):
                w, ms, nrec, nout = device_run(s, m, files[k], zz)
                r[name] = {"wall_s": w, "windows_ms": ms[0], "heap_ms": ms[1], "gather_out_ms": ms[2], "records": nrec, "out_bytes": nout}
            ref = os.path.join(d, "ref.bam")
            if os.access(REAL, os.X_OK):
                r["sambamba_merge_t16_s"] = wall([REAL, "merge", "-t", "16", ref] + files[k])
                want = digest(ref)
            for bg in ("0", "1"):
                out = os.path.join(d, "shim%s.bam" % bg)
                env = dict(os.environ, SSQ_MERGE_GPU="1", SSQ_BGZF_GPU=bg, SSQ_SAMBAMBA_REAL=REAL)
                r["shim_merge_t16_bgzf_gpu%s_s" % bg] = wall([SHIM, "merge", "-t", "16", out] + files[k], env)
                if os.access(REAL, os.X_OK):
                    r["identical_bgzf_gpu" + bg] = digest(out) == want
                    ok &= r["identical_bgzf_gpu" + bg]
                for f in (out, out + ".bai"):
                    os.unlink(f)
            for f in (ref, ref + ".bai"):
                if os.path.exists(f):
                    os.unlink(f)
            res["runs"][k] = r
            print(json.dumps({k: r}), file=sys.stderr)
        s.bgzf_free(z)
        s.merge_free(m)
    print(json.dumps(res))
    if not ok:
        sys.exit("the shim's merged file differs from the staged sambamba's")


if __name__ == "__main__":
    main()
