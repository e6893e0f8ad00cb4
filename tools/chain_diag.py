#!/usr/bin/env python
"""diagnostics: cycle counters inside k_chain for one batch (tools only, not part of the bench)"""
import ctypes as C, os, subprocess, sys
import numpy as np
import torch  # before libssq, so that torch's NCCL is the one loaded
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests")); sys.path.insert(0, ROOT)
import ssq_testlib as T, bench
gl = int(sys.argv[1]) if len(sys.argv) > 1 else bench.GENOME_LEN
s = T.SSQ()
fa, g = bench.ensure_reference(bench.cache_dir(), gl, lambda f: s.index_build(f))
idx = s.index_load(fa)
seq, off = bench.fast_pairs(g, 1000000, 150, 1000)
h = C.c_void_p()
s.ck(s.lib.ssq_batch_create(idx, s.opts, C.c_int(len(off) - 1), seq.ctypes.data_as(C.c_void_p), off.ctypes.data_as(C.c_void_p), C.byref(h)), "create")
for _ in range(2):
    s.ck(s.lib.ssq_batch_run(h), "run")
c = [int(s.lib.ssq_batch_counter(h, i)) for i in range(23)]
ms = [s.lib.ssq_batch_stage_ms(h, i) for i in range(5)]
n_sm = torch.cuda.get_device_properties(0).multi_processor_count
ghz = int(subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=clocks.max.sm", "--format=csv,noheader,nounits"], capture_output=True, text=True).stdout.split()[0]) / 1000.0
thr = n_sm * 12 * 128  # k_chain: 12 blocks of 128 threads per SM
print("genome", gl, "stage ms", [round(x, 1) for x in ms], "seeds", c[7])
print("k_chain cycles per thread (avg): add_seed %.1fM finish %.1fM fetch/init %.1fM ; kernel %.1fM cycles" % (c[12] / thr / 1e6, c[13] / thr / 1e6, c[14] / thr / 1e6, ms[2] * ghz * 1e3 / 1e3))
print("slowest single read: %.2fM cycles (%.2f ms) with n_seeds=%d n_chains=%d" % (c[15] / 1e6, c[15] / (ghz * 1e6), c[16] >> 32, c[16] & 0xffffffff))
print("per seed: add %.0f cycles" % (c[12] / max(1, c[7])))
print("tiers: light %.1f ms, heavy %.1f ms, heavy reads %d (of which %d overflowed to the giant tier), cut %d seeds" % (c[17] / 1e3, c[18] / 1e3, c[19], c[21], c[20]))
print("giant tier alone: %.1f ms" % (c[22] / 1e3))
