"""speedseq_b200 — H100-native (sm_90a) `speedseq align` hot path (BWA-MEM seed/chain/extend + SAMBLASTER dup-marking).

The product is the C-ABI library speedseq_b200/libssq.so (include/ssq.h) and the two CLI shims under speedseq_b200/bin
that plug into the reference's speedseq.config (BWA=, SAMBLASTER=).  This Python package only locates the library;
there is no Python or CPU implementation of the path behind it."""
import os

LIB = os.path.join(os.path.dirname(os.path.abspath(__file__)), "libssq.so")


def lib_path():
    if not os.path.exists(LIB):
        raise RuntimeError("speedseq_b200/libssq.so is not built (run __graft_entry__.build()); there is no fallback")
    return LIB
