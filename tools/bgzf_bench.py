#!/usr/bin/env python
"""BGZF compression of real BAM records: the device encoder (ssq_bgzf_deflate_dev, data in HBM; ssq_bgzf_deflate, from pinned host
buffers with the copies) against host zlib (ssq_bgzf_compress at levels 1 and 6 on all host cores, sliced on block boundaries as the
`sambamba` shim does).  Input: the main-stream BAM records of the config-1 example reads (speedseq's example data: NA12878 qualities),
aligned on the device in BAM mode, copies concatenated to at least --gb GB.  Prints one JSON line.
usage: bgzf_bench.py [--gb 2] [--reps 5] [--zlib-mb 512]"""
import argparse
import ctypes as C
import gzip
import json
import os
import subprocess
import sys
import threading
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
from speedseq_b200 import capi  # noqa: E402

DATA = os.path.join(ROOT, "oracle", "_ref", "stage", "example", "data")
FQ = os.path.join(DATA, "NA12878.20slice.30X.fastq.gz")
FA = os.path.join(DATA, "human_g1k_v37_20_42220611-42542245.fasta")


def example_records(s):
    """main-stream BAM records of the example reads (interleaved pairs, `bwa mem -p` + samblaster as speedseq:438-439 runs them)"""
    d = os.path.join(bench.cache_dir(), "bgzf_example")
    os.makedirs(d, exist_ok=True)
    fa = os.path.join(d, "ref.fa")
    if not os.path.exists(fa + ".sa"):
        open(fa, "wb").write(open(FA, "rb").read())
        s.index_build(fa, None, 0)
    names, seqs, quals = [], [], []
    with gzip.open(FQ, "rt") as f:
        for i, l in enumerate(f):
            l = l.rstrip("\n")
            if i % 4 == 0:
                nm = l[1:].split()[0]
                names.append(nm[:-2] if nm.endswith(("/1", "/2")) else nm)
            elif i % 4 == 1:
                seqs.append(l)
            elif i % 4 == 3:
                quals.append(l)
    h = s.index_load(fa, 0)
    al = s.aligner_create(h, dict(exclude_dups=1, add_mate_tags=1, max_split_count=2, min_non_overlap=20), b"NA12878")
    s.ck(s.lib.ssq_aligner_set_bam(al, C.c_int(1), C.c_int(1)), "ssq_aligner_set_bam")
    rd, keep = capi.pack_reads(names, seqs, quals, None, 1, 0)
    s.aligner_run(al, rd)
    p, n = C.c_void_p(), C.c_size_t(0)
    s.ck(s.lib.ssq_aligner_fetch_bam(al, C.c_int(0), C.byref(p), C.byref(n)), "ssq_aligner_fetch_bam")
    rec = C.string_at(p, n.value)
    s.aligner_free(al)
    s.index_free(h)
    return rec, len(names)


def zlib_rate(lib, data, level, threads):
    """ssq_bgzf_compress over `threads` slices of whole blocks at once -> (GB/s, compressed bytes)"""
    blk = 0xff00
    per = ((len(data) // blk + threads) // threads) * blk
    buf = (C.c_char * len(data)).from_buffer_copy(data)
    outs = [0] * threads

    def one(k):
        lo = k * per
        if lo >= len(data):
            return
        o, n = C.c_void_p(), C.c_size_t(0)
        assert lib.ssq_bgzf_compress(C.byref(buf, lo), C.c_size_t(min(per, len(data) - lo)), level, 0, C.byref(o), C.byref(n)) == 0
        outs[k] = n.value
        lib.ssq_free(o)
    t0 = time.perf_counter()
    th = [threading.Thread(target=one, args=(k,)) for k in range(threads)]
    [t.start() for t in th]
    [t.join() for t in th]
    return len(data) / (time.perf_counter() - t0) / 1e9, sum(outs) + 28


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gb", type=float, default=2.0)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--zlib-mb", type=int, default=512, help="host zlib runs on this leading part of the input (its rate does not depend on the size)")
    a = ap.parse_args()
    if not (os.path.exists(FQ) and os.path.exists(FA)):
        sys.exit("bgzf_bench.py: the example data staged by build() (oracle/_ref/stage/example/data) is missing")
    import torch
    s = capi.SSQ()
    rec, n_reads = example_records(s)
    copies = int(a.gb * 1e9) // len(rec) + 1
    host = torch.empty(copies * len(rec), dtype=torch.uint8, pin_memory=True)
    hv = host.numpy()
    r8 = np.frombuffer(rec, np.uint8)
    for k in range(copies):
        hv[k * len(rec):(k + 1) * len(rec)] = r8
    n = host.numel()
    d_in = host.cuda()
    d_out = torch.empty(n + 31 * (n // 0xff00 + 1) + 64, dtype=torch.uint8, device="cuda")
    z = s.bgzf_create(0)
    st = torch.cuda.ExternalStream(s.bgzf_stream(z))
    rc, dev_len, _ = s.bgzf_deflate_dev(z, d_in.data_ptr(), n, d_out.data_ptr(), d_out.numel(), 6, 1)  # warm-up
    assert rc == 0
    dev_gbs = []
    for _ in range(a.reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(st)
        rc, ln, _ = s.bgzf_deflate_dev(z, d_in.data_ptr(), n, d_out.data_ptr(), d_out.numel(), 6, 1)
        e1.record(st)
        e1.synchronize()
        assert rc == 0 and ln == dev_len
        dev_gbs.append(n / (e0.elapsed_time(e1) / 1e3) / 1e9)
    L = s.lib
    L.ssq_bgzf_deflate.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_int, C.c_int, C.c_void_p, C.c_void_p]
    host_gbs = []
    for _ in range(max(2, a.reps // 2)):
        o, ln = C.c_void_p(), C.c_size_t(0)
        t0 = time.perf_counter()
        s.ck(L.ssq_bgzf_deflate(z, host.data_ptr(), n, 6, 1, C.byref(o), C.byref(ln)), "ssq_bgzf_deflate")
        host_gbs.append(n / (time.perf_counter() - t0) / 1e9)
        if len(host_gbs) == 1:
            first = C.string_at(o, 1 << 20)
            host_len = ln.value
        L.ssq_free(o)
    assert host_len == dev_len and first == bytes(d_out[: 1 << 20].cpu().numpy())
    s.bgzf_free(z)
    L.ssq_bgzf_compress.argtypes = [C.c_void_p, C.c_size_t, C.c_int, C.c_int, C.c_void_p, C.c_void_p]
    L.ssq_free.argtypes = [C.c_void_p]
    cores = os.cpu_count() or 1
    zn = min(n, a.zlib_mb << 20)
    sample = bytes(hv[:zn])
    z1, z1_len = zlib_rate(L, sample, 1, cores)
    z6, z6_len = zlib_rate(L, sample, 6, cores)
    try:  # the card and its clocks, read in the same run

        q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader,nounits"], stdout=subprocess.PIPE, text=True, timeout=30).stdout.strip().split(", ")
    except OSError:
        q = [torch.cuda.get_device_name(0), None, None, None]
    med = lambda v: sorted(v)[len(v) // 2]
    ratio_dev = dev_len / n
    print(json.dumps({
        "input": {"records_bytes": len(rec), "reads": n_reads, "copies": copies, "bytes": n, "source": "config-1 example reads (NA12878 qualities), main-stream BAM records aligned on the device"},
        "device_hbm": {"GB_s_median": med(dev_gbs), "GB_s_min": min(dev_gbs), "GB_s_max": max(dev_gbs), "reps": a.reps, "bytes_out": dev_len, "ratio": ratio_dev},
        "device_from_host": {"GB_s_median": med(host_gbs), "GB_s_min": min(host_gbs), "GB_s_max": max(host_gbs), "bytes_out": host_len},
        "zlib_l1": {"GB_s": z1, "cores": cores, "sample_bytes": zn, "ratio": z1_len / zn},
        "zlib_l6": {"GB_s": z6, "cores": cores, "sample_bytes": zn, "ratio": z6_len / zn},
        "device_ratio_vs_zlib": {"l1": ratio_dev / (z1_len / zn), "l6": ratio_dev / (z6_len / zn)},
        "gpu": {"name": q[0], "power_limit_w": q[1], "sm_mhz": q[2], "sm_max_mhz": q[3]},
    }))


if __name__ == "__main__":
    main()
