"""BAI index of a sorted BAM on the device against speedseq's sambamba.  Makes a coordinate-sorted BAM of about --gb GB of record text
(150-base records over 24 references, 3 % unmapped at their mate's position, a few thousand without coordinates; compressed on
the device at level 1) in a temporary directory, then reports, as one JSON line:
  - the card (name, power limit, SM clock, read in one nvidia-smi call before the runs);
  - wall clock of the `sambamba` shim's `index` and of the staged sambamba's `index -t 16` on the same file (best of --reps; with
    one thread when -t 16 fails), and whether the two .bai files are identical;
  - a warm ssq_bai_build from host memory: wall clock and device time by phase (CUDA events: BGZF inflation with the copy in,
    record walk and checks, index assembly), best of --reps, and GB/s of text.
Exits non-zero when the index differs from the staged sambamba's or from the shim's.
usage: python tools/bai_bench.py [--gb 2] [--reps 3]"""
import argparse
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
from golden.make_bai_golden import header, record  # noqa: E402
from speedseq_b200.capi import SSQ  # noqa: E402

SHIM = os.path.join(ROOT, "speedseq_b200", "bin", "sambamba")
REAL = os.path.join(ROOT, "oracle", "_ref", "stage", "src", "sambamba")


def reg2bin(beg, end):
    end = end - 1
    out = np.zeros(len(beg), np.uint16)
    done = np.zeros(len(beg), bool)
    for shift, base in ((14, 4681), (17, 585), (20, 73), (23, 9), (26, 1)):
        m = ~done & ((beg >> shift) == (end >> shift))
        out[m] = base + (beg[m] >> shift)
        done |= m
    return out


def make_text(gb, seed=1):
    rng = np.random.default_rng(seed)
    tmpl = np.frombuffer(record("read0000000", 99, 0, 0, "150M"), np.uint8)
    L = len(tmpl)
    n = int(gb * 1e9 / L)
    refs = [("chr%d" % (i + 1), 240000000) for i in range(24)]
    recs = np.tile(tmpl, n).reshape(n, L)
    per = n // 24
    ref = np.minimum(np.arange(n) // per, 23).astype(np.int32)
    pos = np.empty(n, np.int64)
    for r in range(24):
        m = ref == r
        pos[m] = np.sort(rng.integers(0, 240000000 - 200, m.sum()))
    unm = rng.random(n) < 0.03
    flag = np.where(unm, 133, 99).astype(np.uint16)
    bins = np.where(unm, reg2bin(pos, pos + 1), reg2bin(pos, pos + 150)).astype(np.uint16)
    body = 36 + 12 + 4  # block_size and fixed fields, the name, one CIGAR op: then 75 bytes of bases and 150 of qualities
    recs[:, body:body + 75] = rng.choice(np.array([0x12, 0x14, 0x18, 0x21, 0x24, 0x28, 0x41, 0x42, 0x48, 0x81, 0x82, 0x84], np.uint8), (n, 75))
    recs[:, body + 75:body + 225] = rng.integers(2, 41, (n, 150), dtype=np.uint8)
    recs[:, 4:8] = ref.view(np.uint8).reshape(n, 4)
    recs[:, 8:12] = pos.astype(np.int32).view(np.uint8).reshape(n, 4)
    recs[:, 14:16] = bins.view(np.uint8).reshape(n, 2)
    recs[:, 18:20] = flag.view(np.uint8).reshape(n, 2)
    nocoor = b"".join(record("nocoor%d" % i, 77, -1, -1, "*", seqlen=150) for i in range(5000))
    return header(refs) + recs.tobytes() + nocoor, n + 5000


def best(f, reps):
    t = []
    for _ in range(reps):
        t0 = time.perf_counter()
        f()
        t.append(time.perf_counter() - t0)
    return min(t)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gb", type=float, default=2.0)
    ap.add_argument("--reps", type=int, default=3)
    a = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    s = SSQ()
    text, n_rec = make_text(a.gb)
    z = s.bgzf_create(0)
    bam = s.bgzf_deflate(z, text, 1, 1)
    s.bgzf_free(z)
    res = {"card": card, "text_bytes": len(text), "bam_bytes": len(bam), "records": n_rec}
    with tempfile.TemporaryDirectory() as d:
        p = os.path.join(d, "big.bam")
        open(p, "wb").write(bam)
        res["shim_index_s"] = best(lambda: subprocess.run([SHIM, "index", p, p + ".gpu.bai"], check=True), a.reps)
        if os.access(REAL, os.X_OK):
            for t in ("16", "1"):  # one thread when -t 16 fails
                if os.path.exists(p + ".ref.bai"):  # sambamba 0.5.9 does not truncate an existing output
                    os.unlink(p + ".ref.bai")
                r = subprocess.run([REAL, "index", "-t", t, p, p + ".ref.bai"], capture_output=True)
                if r.returncode:
                    res["sambamba_index_t%s" % t] = "failed: exit %d" % r.returncode
                    continue
                res["sambamba_index_t%s_s" % t] = best(lambda: subprocess.run([REAL, "index", "-t", t, p, p + ".ref.bai"], check=True), a.reps)
                res["identical"] = open(p + ".gpu.bai", "rb").read() == open(p + ".ref.bai", "rb").read()
                break
        b = s.bai_create(0)
        rc, bai = s.bai_build(b, bam)  # warm: buffers sized
        assert rc == 0, s.err()
        runs = []
        for _ in range(a.reps):
            t0 = time.perf_counter()
            rc, bai2 = s.bai_build(b, bam)
            runs.append((time.perf_counter() - t0, s.bai_times(b)))
            assert rc == 0 and bai2 == bai
        w, ms = min(runs)
        s.bai_free(b)
        res.update({"build_wall_s": w, "device_ms": {"inflate": ms[0], "walk": ms[1], "index": ms[2]}, "text_GBps": len(text) / w / 1e9,
                    "same_as_shim": bai == open(p + ".gpu.bai", "rb").read()})
    print(json.dumps(res))
    if res.get("identical") is False or not res["same_as_shim"]:
        sys.exit("the device index differs from sambamba's or from the shim's")


if __name__ == "__main__":
    main()
