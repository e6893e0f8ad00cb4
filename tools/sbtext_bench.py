#!/usr/bin/env python
"""samblaster over SAM text: GB/s of name-grouped SAM through (1) ssq_sbtext_run from pinned host buffers, copies included, best of
--reps runs, (2) the `samblaster` shim (device text path), (3) the same shim built without SSQ_SB_DEVICE_TEXT (host parsing, GPU
dup-set), compiled into the output directory.  Input: about --gb GB of SAM, made once in the bench cache dir by the `bwa` shim
(`bwa mem -p`, ssq_aligner_*) from bench.fast_pairs reads (10 % planted duplicate pairs) on the bench's 63 Mbp synthetic genome.
Every arm must write the same three streams (compared by SHA-256, @PG lines excluded).  Prints one JSON line and writes it to
OUT/sbtext_bench.json together with the card name, power limit and SM clock read in the same call.
usage: sbtext_bench.py [--gb 2] [--reps 3] [--out DIR]"""
import argparse
import ctypes as C
import hashlib
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import torch  # noqa: E402  (before libssq: torch brings its own NCCL)
import bench  # noqa: E402
from speedseq_b200 import capi  # noqa: E402
from test_sbtext_cpu import SbOpts, SbtOut, sb_opts, split_header  # noqa: E402

GLEN = 63025520
ARGS = ["--excludeDups", "--addMateTags", "--maxSplitCount", "2", "--minNonOverlap", "20"]
SHIM = os.path.join(ROOT, "speedseq_b200", "bin", "samblaster")
BWA = os.path.join(ROOT, "speedseq_b200", "bin", "bwa")


def make_sam(path, fa, g, gb):
    fq = path + ".fq"
    rl, per = 150, 14 + 151 + 2 + 151
    n_pairs = int(gb * (1 << 30) / 420 / 2)  # about 420 B of SAM per read
    with open(fq, "wb") as f:
        done = 0
        while done < n_pairs:
            k = min(1 << 20, n_pairs - done)
            codes = bench.fast_pairs(g, k, rl, 4242 + done)
            n = codes.shape[0]
            rec = np.empty((n, per), np.uint8)
            ids = done + np.arange(n) // 2
            nm = np.char.add("p", np.char.zfill(ids.astype("U10"), 9)).astype("S10")
            rec[:, 0] = ord("@"); rec[:, 1:11] = np.frombuffer(nm.tobytes(), np.uint8).reshape(n, 10); rec[:, 11] = ord("/"); rec[:, 12] = ord("1") + (np.arange(n) & 1); rec[:, 13] = 10
            rec[:, 14:164] = np.frombuffer(b"ACGT", np.uint8)[codes]; rec[:, 164] = 10; rec[:, 165] = ord("+"); rec[:, 166] = 10
            rec[:, 167:317] = (33 + (np.arange(rl)[None, :] * 7 + np.arange(n)[:, None]) % 41).astype(np.uint8); rec[:, 317] = 10
            rec.tofile(f)
            done += k
    with open(path + ".tmp", "wb") as f:
        subprocess.run([BWA, "mem", "-t", "30", "-p", fa, fq], stdout=f, stderr=subprocess.DEVNULL, check=True, timeout=3600)
    os.replace(path + ".tmp", path)
    os.unlink(fq)


def digest(parts):
    h = hashlib.sha256()
    for p in parts:
        for l in p.splitlines(True):
            if not l.startswith(b"@PG"):
                h.update(l)
        h.update(b"|")
    return h.hexdigest()


def run_shim(exe, sam_path, d, tag):
    spl, disc, out = (os.path.join(d, "%s.%s" % (tag, e)) for e in ("spl", "disc", "sam"))
    t0 = time.time()
    with open(sam_path, "rb") as fi, open(out, "wb") as fo:
        p = subprocess.run([exe] + ARGS + ["--splitterFile", spl, "--discordantFile", disc], stdin=fi, stdout=fo, stderr=subprocess.PIPE, check=True, timeout=3600)
    dt = time.time() - t0
    parts = [open(x, "rb").read() for x in (out, spl, disc)]
    for x in (out, spl, disc):
        os.unlink(x)
    return dt, digest(parts), p.stderr.decode()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gb", type=float, default=2.0)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--piece-mb", type=int, default=256)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("sbtext_bench.py measures the device path: no CUDA device")
    out_dir = a.out or tempfile.mkdtemp(prefix="sbtext_bench_")
    os.makedirs(out_dir, exist_ok=True)
    s = capi.SSQ()
    cache = bench.cache_dir()
    fa, g = bench.ensure_reference(cache, GLEN, lambda f: s.index_build(f, None, 0))
    sam_path = os.path.join(cache, "sbtext_%g.sam" % a.gb)
    if not os.path.exists(sam_path):
        make_sam(sam_path, fa, g, a.gb)
    sam = open(sam_path, "rb").read()
    header, body = split_header(sam)
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    res = {"device": smi, "sam_bytes": len(sam), "record_bytes": len(body), "records": body.count(b"\n"), "piece_mb": a.piece_mb}
    # (1) the C-ABI from pinned host buffers
    lib = s.lib
    lib.ssq_sbtext_create.argtypes = [C.c_int, C.POINTER(SbOpts), C.c_char_p, C.c_size_t, C.POINTER(C.c_void_p)]
    lib.ssq_sbtext_run.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_int, C.c_uint64, C.POINTER(C.c_size_t), C.POINTER(SbtOut)]
    lib.ssq_sbtext_free.argtypes = [C.c_void_p]
    pin = torch.frombuffer(bytearray(body), dtype=torch.uint8).pin_memory()
    opts = sb_opts(ARGS)
    times, dig, info = [], None, {}
    for rep in range(a.reps + 1):
        h = C.c_void_p()
        assert lib.ssq_sbtext_create(0, C.byref(opts), header, len(header), C.byref(h)) == 0, s.err()
        parts = [[header], [header], [header]]
        at, busy, ids, dups = 0, 0.0, 0, 0
        while at < len(body):
            n = min(a.piece_mb << 20, len(body) - at)
            used, o = C.c_size_t(0), SbtOut()
            t0 = time.time()
            rc = lib.ssq_sbtext_run(h, C.c_void_p(pin.data_ptr() + at), n, int(at + n == len(body)), 0, C.byref(used), C.byref(o))
            busy += time.time() - t0
            assert rc == 0, s.err()
            if rep == 0:
                for k in range(3):
                    parts[k].append(C.string_at(o.text[k], o.len[k]))
            ids += o.n_ids; dups += o.n_dup
            at += used.value
        lib.ssq_sbtext_free(h)
        if rep == 0:
            dig = digest([b"".join(p) for p in parts]); info = {"qname_blocks": ids, "dup_blocks": dups}
        else:
            times.append(busy)
    res.update(info)
    res["api_pinned_s"] = times
    res["api_pinned_GBps"] = len(body) / min(times) / 1e9
    print(json.dumps({"api_pinned_GBps": res["api_pinned_GBps"]}), file=sys.stderr, flush=True)
    # (2) the shim, device text path; (3) the shim built without it
    host_exe = os.path.join(out_dir, "samblaster_host_text")
    subprocess.check_call(["gcc", "-O2", "-w", "-I" + os.path.join(ROOT, "include"), "-I" + os.path.join(ROOT, "speedseq_b200", "cli"), "-o", host_exe,
                           os.path.join(ROOT, "speedseq_b200", "cli", "samblaster_main.c"), "-L" + os.path.join(ROOT, "speedseq_b200"), "-lssq",
                           "-Wl,-rpath," + os.path.join(ROOT, "speedseq_b200")])
    digs = {"api": dig}
    for tag, exe in (("shim_device", SHIM), ("shim_host_text", host_exe)):
        dt, dg, err = run_shim(exe, sam_path, out_dir, tag)
        assert "host code" not in err, err
        res[tag + "_s"] = dt
        res[tag + "_GBps"] = len(sam) / dt / 1e9
        digs[tag] = dg
        print(json.dumps({tag + "_GBps": res[tag + "_GBps"]}), file=sys.stderr, flush=True)
    res["same_bytes"] = len(set(digs.values())) == 1
    res["sha256"] = digs
    line = json.dumps(res)
    open(os.path.join(out_dir, "sbtext_bench.json"), "w").write(line + "\n")
    print(line)
    assert res["same_bytes"], digs


if __name__ == "__main__":
    main()
