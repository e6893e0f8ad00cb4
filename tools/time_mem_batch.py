#!/usr/bin/env python
"""times the full `bwa mem` batch path (reads -> SAM text) of libssq against the oracle's on the same reads"""
import ctypes as C, os, sys, time
import numpy as np
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests")); sys.path.insert(0, ROOT)
import ssq_testlib as T
import bench

n_pairs = int(sys.argv[1]) if len(sys.argv) > 1 else 200000
cache = bench.cache_dir()
s = T.SSQ(); o = T.Oracle()
s.opts[29] = bench.usable_cores()  # host threads (opt.n_threads)
fa, g = bench.ensure_reference(cache, bench.GENOME_LEN, lambda f: s.index_build(f))
idx = s.index_load(fa); oidx = o.load(fa)
seq, off = bench.fast_pairs(g, n_pairs, 150, 77)
codes = seq.reshape(-1, 150)
acgt = np.frombuffer(b"ACGTN", np.uint8)
seqs = [acgt[r].tobytes().decode() for r in codes]
names = ["p%d" % (i // 2) for i in range(2 * n_pairs)]
quals = ["I" * 150] * (2 * n_pairs)
n = len(names)
arr = lambda xs: (C.c_char_p * n)(*[x.encode() for x in xs])
an, aq, ql = arr(names), arr(seqs), arr(quals)
for rep in range(2):
    out, ln = C.c_char_p(), C.c_size_t(0)
    t0 = time.time()
    s.ck(s.lib.ssq_mem_batch_sam(idx, s.opts, C.c_int(n), an, aq, ql, None, C.c_int64(0), C.c_int(1), None, b"rg", C.c_int(0), C.byref(out), C.byref(ln), None), "mem")
    dt = time.time() - t0
    sam = C.string_at(out, ln.value); s.lib.ssq_free(out)
    print("libssq ssq_mem_batch_sam: %d reads in %.2f s -> %.0f reads/s (%d SAM bytes)" % (n, dt, n / dt, len(sam)))
m = min(n, 40000)
t0 = time.time(); ref = o.mem_pe(oidx, names[:m], seqs[:m], quals[:m], 0, bench.usable_cores(), b"rg"); dt = time.time() - t0
print("oracle mem_pe (%d threads): %d reads in %.2f s -> %.0f reads/s" % (bench.usable_cores(), m, dt, m / dt))
print("identical on the first %d reads:" % m, sam.decode()[: len(ref)] == ref if n == m else sam.decode().startswith(ref[: 100000]))
