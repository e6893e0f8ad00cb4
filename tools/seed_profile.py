#!/usr/bin/env python
"""Where the seeding stage's time goes on the bench workload (1 Gbp synthetic reference, one 1 M-read batch of bench.py's generator).

Prints one JSON line:
  * stage / kernel times per batch: the seeding stage and the two backward-sweep launches from the library's own CUDA events
    (ssq_aligner_stage_ms 10, ssq_aligner_counter 26); every other seeding launch (forward pass 1 and 2, k_smem_p3, k_smem_p2sel, the
    publish sort) from torch.profiler in a separate run;
  * rank-query classes from the device counters: queries answered from the k-mer table (counter 27), extensions answered from one
    sector (both interval ends in one 64-row block) or two (counter 28 = extensions, counter 0 = sectors loaded), and the sectors of
    the backward sweeps alone (counter 25);
  * index load time and device bytes (the k-mer table is built at load; SSQ_KMER_K=0 turns it off, SSQ_KMER_K=K picks K).
The card's name, power limit and SM clock are read in the same run.

  python tools/seed_profile.py [--genome-len N] [--batch N] [--reps 3] [--cache DIR] [--out FILE]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402

import bench  # noqa: E402
from speedseq_b200 import capi  # noqa: E402


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout
        return q.strip().splitlines()[0]
    except Exception as e:  # the numbers then stand without their card: say so
        return "nvidia-smi unavailable: %s" % e


def seeding_launches(prof_events):
    """per-launch device times (ms) of the seeding stage from a torch.profiler trace of one batch"""
    ev = sorted([e for e in prof_events if e.device_type.name == "CUDA"], key=lambda e: e.time_range.start)
    names = [e.name for e in ev]

    def idx(pred):
        return [i for i, n in enumerate(names) if pred(n)]
    out = {}
    groups = {
        "k_smem_p3": lambda n: "k_smem_p3<" in n,
        "k_smem_fwd pass 1": lambda n: "k_smem_fwd<1" in n,
        "k_smem_fwd pass 2": lambda n: "k_smem_fwd<2" in n,
        "k_smem_bwd (2 launches)": lambda n: "k_smem_bwd<" in n,
        "k_smem_p2sel": lambda n: n.startswith("k_smem_p2sel") or "k_smem_p2sel(" in n,
    }
    for k, f in groups.items():
        out[k] = sum(ev[i].time_range.elapsed_us() for i in idx(f)) / 1000.0
    keys, pub = idx(lambda n: "k_smem_keys" in n), idx(lambda n: "k_smem_publish" in n)
    if keys and pub:  # the publish sort: the CUB radix-sort kernels between the key kernel and the publish kernel
        out["publish sort (CUB radix sort + keys + publish)"] = sum(ev[i].time_range.elapsed_us() for i in range(keys[0], pub[0] + 1)) / 1000.0
    first, last = idx(lambda n: "k_smem_p3<" in n or "k_smem_fwd<1" in n), idx(lambda n: "k_smem_lrep" in n)
    if first and last:
        out["seeding span (first launch start .. k_smem_lrep end)"] = (ev[last[0]].time_range.end - ev[first[0]].time_range.start) / 1000.0
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--genome-len", type=int, default=bench.GENOME_LEN)
    ap.add_argument("--batch", type=int, default=1_000_000)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--cache", default=os.environ.get("SSQ_BENCH_CACHE") or bench.cache_dir())
    ap.add_argument("--out", default=None, help="also append the JSON line to this file")
    ap.add_argument("--label", default="")
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("seed_profile.py: no CUDA device — the seeding kernels have no CPU path")
    torch.cuda.set_device(0)
    s = capi.SSQ()
    L = s.lib
    fa, g = bench.ensure_reference(a.cache, a.genome_len, lambda f: s.index_build(f, None, 0))
    t0 = time.time()
    idx = s.index_load(fa, 0)
    t_load = time.time() - t0
    bt = bench.Batch(torch, bench.fast_pairs(g, a.batch // 2, bench.READ_LEN, 1000), 0)
    al = s.aligner_create(idx, bench.SB, b"seedprof")
    s.ck(L.ssq_aligner_upload(al, C.byref(bt.reads)), "upload")
    dset = C.c_void_p()
    L.ssq_dupset_create.argtypes = [C.c_int, C.c_void_p]
    s.ck(L.ssq_dupset_create(0, C.byref(dset)), "ssq_dupset_create")
    s.ck(L.ssq_aligner_share_dupset(al, dset), "ssq_aligner_share_dupset")

    def one():
        s.ck(L.ssq_dupset_reset(dset), "reset")
        s.ck(L.ssq_aligner_compute(al, None, 0), "compute")
        torch.cuda.synchronize()
    one()
    one()
    rows = []
    for _ in range(a.reps):
        one()
        c = {k: int(L.ssq_aligner_counter(al, k)) for k in (0, 25, 26, 27, 28)}
        rows.append({"seed_ms": float(L.ssq_aligner_stage_ms(al, 10)), "bwd_ms": c[26] / 1000.0, "sectors": c[0], "bwd_sectors": c[25],
                     "table": c[27], "steps": c[28]})
    c = rows[-1]
    one_sector = 2 * c["steps"] - c["sectors"]  # every extension loads one sector or two
    two_sector = c["sectors"] - c["steps"]
    q = c["table"] + c["steps"]
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        one()
    launches = seeding_launches(prof.events())
    s.aligner_free(al)
    L.ssq_dupset_free(dset)
    res = {"label": a.label, "card (name, power limit, SM clock, max SM clock)": card(), "genome_bp": a.genome_len, "batch_reads": a.batch,
           "kmer_k": os.environ.get("SSQ_KMER_K", "default"), "bwd_blocks": os.environ.get("SSQ_SMEM_BWD_BLOCKS", "default"),
           "index_load_s": round(t_load, 2), "index_device_bytes": int(L.ssq_index_info(idx, 6)),
           "seeding_ms": [round(r["seed_ms"], 2) for r in rows], "k_smem_bwd_ms": [round(r["bwd_ms"], 2) for r in rows],
           "rank_queries": q, "from_table": c["table"], "one_sector": one_sector, "two_sector": two_sector,
           "share": {"table": c["table"] / q if q else None, "one_sector": one_sector / q if q else None, "two_sector": two_sector / q if q else None},
           "sectors_loaded": c["sectors"], "bwd_sectors_loaded": c["bwd_sectors"],
           "seeding_GBps": 32.0 * c["sectors"] / (np.median([r["seed_ms"] for r in rows]) * 1e6),
           "k_smem_bwd_GBps": 32.0 * c["bwd_sectors"] / (np.median([r["bwd_ms"] for r in rows]) * 1e6) if c["bwd_sectors"] else None,
           "launches_ms (torch.profiler, one batch)": {k: round(v, 2) for k, v in launches.items()}}
    s.index_free(idx)
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "a") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
