#!/usr/bin/env python
"""gzip decoding of FASTQ: the device decoder (ssq_gunzip_inflate_dev, compressed and decoded data in HBM, CUDA events; and the
streaming ssq_gunzip_inflate from pinned host buffers, copies included) against host zlib on one stream, and `bwa mem -p -t 30`
on the same reads as .fq and as .fq.gz.  Input: about --gb GB of interleaved 2x150 FASTQ, reads from bench.fast_pairs on the
bench's synthetic genome, qualities cycled from the example FASTQ (so the compression ratio is that of real qualities), gzipped as
one member at levels 6 and 1 (kept in the bench cache dir).  Every output is checked against zlib's CRC-32.  Prints one JSON line.
usage: gunzip_bench.py [--gb 2] [--reps 5] [--no-cli]"""
import argparse
import ctypes as C
import gzip
import json
import os
import subprocess
import sys
import time
import zlib

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402  (before libssq: torch brings its own NCCL)
import bench  # noqa: E402
from speedseq_b200 import capi  # noqa: E402

EXAMPLE = os.path.join(ROOT, "oracle", "_ref", "stage", "example", "data", "NA12878.20slice.30X.fastq.gz")
GLEN = 63025520


def make_fastq(path, g, gb):
    quals = [l.rstrip(b"\n") for i, l in enumerate(gzip.open(EXAMPLE)) if i % 4 == 3]
    quals = [q for q in quals if len(q) >= 101]
    qa = np.frombuffer(b"".join(q[:101] for q in quals), np.uint8).reshape(-1, 101)
    qa = np.concatenate([qa, qa[:, :49]], axis=1)  # 150 qualities per read: the example's 101 + its first 49 again
    per = 14 + 151 + 2 + 151
    n_pairs = int(gb * (1 << 30) / per / 2)
    with open(path, "wb") as f:
        done = 0
        while done < n_pairs:
            k = min(1 << 20, n_pairs - done)
            codes = bench.fast_pairs(g, k, 150, 777 + done)
            n = codes.shape[0]
            rec = np.empty((n, per), np.uint8)
            ids = done + np.arange(n) // 2
            nm = np.char.add("p", np.char.zfill(ids.astype("U10"), 9)).astype("S10")
            rec[:, 0] = ord("@"); rec[:, 1:11] = np.frombuffer(nm.tobytes(), np.uint8).reshape(n, 10); rec[:, 11] = ord("/"); rec[:, 12] = ord("1") + (np.arange(n) & 1); rec[:, 13] = 10
            rec[:, 14:164] = np.frombuffer(b"ACGT", np.uint8)[codes]; rec[:, 164] = 10; rec[:, 165] = ord("+"); rec[:, 166] = 10
            rec[:, 167:317] = qa[(2 * done + np.arange(n)) % len(qa)]; rec[:, 317] = 10
            rec.tofile(f)
            done += k


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gb", type=float, default=2.0)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--no-cli", action="store_true")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("gunzip_bench.py measures the device decoder: no CUDA device")
    s = capi.SSQ()
    cache = bench.cache_dir()
    fa, g = bench.ensure_reference(cache, GLEN, lambda f: s.index_build(f, None, 0))
    fq = os.path.join(cache, "gunzip_%g.fq" % a.gb)
    if not os.path.exists(fq):
        make_fastq(fq, g, a.gb)
    text = open(fq, "rb").read()
    crc = zlib.crc32(text)
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    res = {"device": smi, "text_bytes": len(text), "levels": {}}
    g_obj = s.gunzip_create(0, 0)
    d_out = torch.empty(len(text), dtype=torch.uint8, device="cuda")
    for level in (6, 1):
        zpath = fq + ".l%d.gz" % level
        if not os.path.exists(zpath):
            c = zlib.compressobj(level, zlib.DEFLATED, 31)
            with open(zpath, "wb") as f:
                for i in range(0, len(text), 64 << 20):
                    f.write(c.compress(text[i:i + (64 << 20)]))
                f.write(c.flush())
        z = open(zpath, "rb").read()
        r = {"compressed_bytes": len(z), "ratio": len(text) / len(z)}
        t0 = time.time()  # host zlib, one stream
        h = zlib.crc32(zlib.decompress(z, 31))
        r["host_zlib_GBps"] = len(text) / (time.time() - t0) / 1e9
        assert h == crc
        d_in = torch.frombuffer(bytearray(z), dtype=torch.uint8).cuda()
        st = torch.cuda.ExternalStream(s.gunzip_stream(g_obj))
        times = []
        for rep in range(a.reps + 1):
            s0 = s.gunzip_stats(g_obj)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            e0.record(st)
            rc, n = s.gunzip_inflate_dev(g_obj, d_in.data_ptr(), len(z), d_out.data_ptr(), len(text))
            e1.record(st)
            e1.synchronize()
            assert rc == 0 and n == len(text)
            if rep:
                times.append(e0.elapsed_time(e1) / 1e3)
            s1 = s.gunzip_stats(g_obj)
        assert zlib.crc32(d_out.cpu().numpy().tobytes()) == crc
        dec, syn, rep_, win = (b - a_ for a_, b in zip(s0, s1))
        r.update(device_hbm_GBps=len(text) / min(times) / 1e9, device_hbm_s=times, chunks=dec, sync_fraction=syn / max(1, dec - win),
                 repairs_per_chunk=rep_ / max(1, dec), windows=win)
        # streaming from pinned host buffers: the input in pieces of 64 MB, the text into a pinned 512 MB buffer
        pin_in = torch.frombuffer(bytearray(z), dtype=torch.uint8).pin_memory()
        pin_out = torch.empty(512 << 20, dtype=torch.uint8).pin_memory()
        used, ln, done = C.c_size_t(0), C.c_size_t(0), C.c_int(0)
        at, pos, c, busy = 0, 0, 0, 0.0
        while not done.value:
            t0 = time.time()
            rc = s.lib.ssq_gunzip_inflate(g_obj, C.c_void_p(pin_in.data_ptr() + pos), C.c_size_t(len(z) - pos), 1, C.byref(used), C.c_void_p(pin_out.data_ptr()),
                                          C.c_size_t(512 << 20), C.byref(ln), C.byref(done))
            busy += time.time() - t0
            assert rc == 0, s.err()
            c = zlib.crc32(pin_out.numpy()[:ln.value], c)
            at += ln.value; pos += used.value
        r["stream_pinned_GBps"] = len(text) / busy / 1e9
        assert at == len(text) and c == crc
        res["levels"][str(level)] = r
        print(json.dumps({"level": level, **r}), file=sys.stderr, flush=True)
        del d_in
    s.gunzip_free(g_obj)
    del d_out
    torch.cuda.empty_cache()
    if not a.no_cli:
        bwa = os.path.join(ROOT, "speedseq_b200", "bin", "bwa")
        wall = {}
        for tag, path in (("fq", fq), ("fq.gz level 6", fq + ".l6.gz"), ("fq.gz level 1", fq + ".l1.gz")):
            out = os.path.join(cache, "gunzip_cli.sam")
            t0 = time.time()
            with open(out, "wb") as f:
                subprocess.run([bwa, "mem", "-t", "30", "-p", fa, path], stdout=f, stderr=subprocess.DEVNULL, check=True, timeout=1800)
            wall[tag] = time.time() - t0
            h = 0
            with open(out, "rb") as f:
                for l in f:
                    if not l.startswith(b"@PG"):
                        h = zlib.crc32(l, h)
            wall[tag + " sam_crc"] = h
            print(tag, wall[tag], file=sys.stderr, flush=True)
        assert len({v for k, v in wall.items() if k.endswith("sam_crc")}) == 1
        res["bwa_mem_p_t30_s"] = wall
    print(json.dumps(res))


if __name__ == "__main__":
    main()
