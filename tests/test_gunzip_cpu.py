"""The chunk-parallel gzip decoder (speedseq_b200/csrc/ssq_gunzip.cuh) run on the host by tests/hostsim/gunzip_host.cpp (the same
SSQ_HD phases and window logic, host loops in place of the kernels; compiled into a temporary directory): on a seeded corpus of
gzip streams, at several chunk sizes, the text is zlib's, and each item takes the paths it was made for (sync points, repairs after
false syncs, several windows).  Truncated or corrupted streams are SSQ_EDATA, or exactly what zlib's gzread returns when the damage
lies in bytes gzread ignores."""
import ctypes as C
import ctypes.util
import functools
import gzip
import os
import random
import struct
import subprocess
import zlib

import pytest

import ssq_testlib as T

EDATA = -9
CHUNKS = (4096, 16384, 0)  # 0: the default (32 KB)
DEFAULT_CHUNK = 32768


def fastq_text():
    return b"".join(gzip.open(os.path.join(T.GOLDEN, f)).read() for f in ("ex_reads_2k.fq.gz", "wgsim_r1.fq.gz", "wgsim_r2.fq.gz"))


def gz(data, level=6, strategy=zlib.Z_DEFAULT_STRATEGY):
    c = zlib.compressobj(level, zlib.DEFLATED, 31, 8, strategy)
    return c.compress(data) + c.flush()


def member(data, flags=0, level=6, zdict=None):
    """one gzip member with the header fields `flags` asks for (FHCRC 2, FEXTRA 4, FNAME 8, FCOMMENT 16); zdict: the deflate stream
    may reference zdict as if it came before the member (what a decoder that does not reset its window would accept)"""
    h = b"\x1f\x8b\x08" + bytes([flags]) + b"\x01\x02\x03\x04\x00\xff"
    if flags & 4:
        h += struct.pack("<H", 7) + b"SP\x03\x00abc"
    if flags & 8:
        h += b"reads.fq\0"
    if flags & 16:
        h += b"a comment\0"
    if flags & 2:
        h += struct.pack("<H", zlib.crc32(h) & 0xffff)
    c = zlib.compressobj(level, zlib.DEFLATED, -15, 8, zlib.Z_DEFAULT_STRATEGY, *([zdict] if zdict else []))
    return h + c.compress(data) + c.flush() + struct.pack("<II", zlib.crc32(data), len(data) & 0xffffffff)


@functools.lru_cache(None)
def corpus():
    """name -> gzip stream; seeded"""
    fq = fastq_text()
    rnd = random.Random(7)
    z6 = gz(fq, 6)
    c = {
        "fq_l1": gz(fq, 1), "fq_l6": z6, "fq_l9": gz(fq, 9),
        "fq_fixed": gz(fq, 6, zlib.Z_FIXED), "fq_huffman_only": gz(fq, 6, zlib.Z_HUFFMAN_ONLY), "fq_rle": gz(fq, 6, zlib.Z_RLE),
        "fq_stored": gz(fq, 0),
        "multi_member": member(fq[:1000]) + member(b"", 2) + member(fq[1000:700000], 4, 1) + member(b"", 8 | 16) + member(fq[700000:], 2 | 4 | 8 | 16, 9),
        "zeros_64MB": gz(bytes(64 << 20)),
        "random_l6": gz(rnd.randbytes(1 << 20)),
        "trailing_garbage": z6 + b"not a gzip member\n" * 3,
        "trailing_zeros": z6 + bytes(4096),
        "empty_input": b"",
        "one_empty_member": gz(b""),
        # a gzip stream of FASTQ stored (level 0) inside a gzip stream: its dynamic blocks are false sync points
        "false_sync_bait": gz(z6 + fq[:200000] + gz(fq[100000:], 9), 0),
    }
    return c


def bgzf_file(lib_cpu, data):
    out, n = C.c_void_p(), C.c_size_t(0)
    assert lib_cpu.ssq_bgzf_compress(data, len(data), 6, 1, C.byref(out), C.byref(n)) == 0
    r = C.string_at(out, n.value)
    lib_cpu.ssq_free(out)
    return r


def zlib_text(z):
    """what gzread returns for a stream that decodes: members while they start with 1f 8b, then nothing"""
    out = []
    while z[:2] == b"\x1f\x8b":
        d = zlib.decompressobj(31)
        out.append(d.decompress(z))
        assert d.eof
        z = d.unused_data
    return b"".join(out)


_libz = C.CDLL(ctypes.util.find_library("z"))
_libz.gzopen.restype = C.c_void_p
_libz.gzopen.argtypes = [C.c_char_p, C.c_char_p]
_libz.gzread.argtypes = [C.c_void_p, C.c_void_p, C.c_uint]
_libz.gzclose.argtypes = [C.c_void_p]
_libz.gzerror.argtypes = [C.c_void_p, C.c_void_p]
_libz.gzerror.restype = C.c_char_p


def gzread(path):
    """libz gzread over a file: (text, error); a truncated stream is not a gzread error (it ends the text early), only gzerror
    reports it (Z_BUF_ERROR)"""
    f = _libz.gzopen(path.encode(), b"rb")
    buf, out, err = C.create_string_buffer(1 << 16), [], False
    while True:
        n = _libz.gzread(f, buf, 1 << 16)
        if n < 0:
            err = True
            break
        if n == 0:
            break
        out.append(buf.raw[:n])
    errnum = C.c_int(0)
    _libz.gzerror(f, C.byref(errnum))
    err = err or errnum.value != 0
    _libz.gzclose(f)
    return b"".join(out), err


def build_gunzip_host(d):
    so = os.path.join(str(d), "libgunzip_host.so")
    subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-w", "-I", os.path.join(T.ROOT, "include"), "-o", so,
                    os.path.join(T.ROOT, "tests", "hostsim", "gunzip_host.cpp")], check=True)
    lib = C.CDLL(so)
    lib.hostsim_gunzip.argtypes = [C.c_char_p, C.c_size_t, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    lib.hostsim_free.argtypes = [C.c_void_p]
    return lib


@pytest.fixture(scope="session")
def gunzip_host(tmp_path_factory):
    return build_gunzip_host(tmp_path_factory.mktemp("gunzip_host"))


def hostsim_gunzip(lib, z, chunk=0):
    """-> (rc, text, stats (chunks decoded, sync starts, repairs, windows), error offset)"""
    out, n, st, at = C.c_void_p(), C.c_size_t(0), (C.c_int64 * 4)(), C.c_size_t(0)
    rc = lib.hostsim_gunzip(z, len(z), chunk, C.byref(out), C.byref(n), st, C.byref(at))
    text = C.string_at(out, n.value)
    lib.hostsim_free(out)
    return rc, text, tuple(st), at.value


def expected_paths(name, z, chunk, stats):
    """what each corpus item must exercise, so that a change that makes it test less fails"""
    decoded, syncs, repairs, windows = stats
    grid = max(1, -(-len(z) // (chunk or DEFAULT_CHUNK)))  # chunks the stream is cut into (one window unless stated)
    if name == "fq_l6" and chunk == 0:
        assert syncs >= 0.8 * (grid - 1), stats
    if name in ("fq_l1", "fq_l6", "fq_l9", "fq_huffman_only", "fq_rle"):
        assert syncs >= min(grid - 1, len(z) // 65536) and syncs > 0, stats  # zlib starts a block at least every 64 KB here
    if name in ("fq_stored", "fq_fixed", "random_l6"):
        assert syncs == 0, stats  # no dynamic block to find: sequential decode
    if name == "false_sync_bait":
        assert syncs > 0 and repairs > 0, stats
    if name == "zeros_64MB":
        assert windows > 1 and repairs > 0, stats  # every slot fills: chunks stop inside blocks, windows carry context


@pytest.mark.parametrize("chunk", CHUNKS)
@pytest.mark.parametrize("name", list(corpus()))
def test_host_decoder_gives_zlib_text(gunzip_host, name, chunk):
    z = corpus()[name]
    rc, text, stats, _ = hostsim_gunzip(gunzip_host, z, chunk)
    assert rc == 0
    assert text == zlib_text(z)
    assert stats[3] >= 1 and stats[0] == stats[1] + stats[3]
    expected_paths(name, z, chunk, stats)


@pytest.mark.parametrize("chunk", CHUNKS)
def test_host_decoder_bgzf(gunzip_host, ssq_lib_cpu, chunk):
    fq = fastq_text()
    z = bgzf_file(ssq_lib_cpu, fq)
    rc, text, stats, _ = hostsim_gunzip(gunzip_host, z, chunk)
    assert rc == 0 and text == fq
    assert stats[1] > 0


def test_reference_before_a_member_start_is_corrupt(gunzip_host, tmp_path):
    """a member whose deflate stream reaches back into the member before it (zlib makes such a stream with a preset dictionary; its
    first 20 KB repeat the previous member's tail): gzread fails, and so must the decoder, wherever the member boundary falls in a
    chunk and whether or not the reference crosses a chunk start"""
    fq = fastq_text()
    p = str(tmp_path / "x.gz")
    for n1 in (100000, 170001, 300000):
        z = member(fq[:n1]) + member(fq[n1 - 20000:n1 + 100000], zdict=fq[n1 - 32768:n1])
        open(p, "wb").write(z)
        assert gzread(p)[1]
        for chunk in (1024, 4096, 16384, 0):
            assert hostsim_gunzip(gunzip_host, z, chunk)[0] == EDATA, (n1, chunk)


def damaged():
    """(name, stream) pairs: truncations at many offsets and single-byte corruptions, of a small multi-member stream with trailing
    garbage and of a FASTQ stream"""
    fq = fastq_text()
    rnd = random.Random(3)
    small = member(fq[:3000], 2 | 8) + member(fq[3000:40000], 4) + b"trailing bytes"
    big = gz(fq[:400000])
    out = []
    for base, nm in ((small, "small"), (big, "fq")):
        cuts = sorted(set([2, 3, 9, 10, 11, 20, len(base) - 1, len(base) - 8, len(base) - 9] + [rnd.randrange(2, len(base)) for _ in range(40)]))
        out += [("%s_cut%d" % (nm, k), base[:k]) for k in cuts]
        for _ in range(40):
            k = rnd.randrange(2, len(base))
            b = bytearray(base)
            b[k] ^= 1 << rnd.randrange(8)
            out.append(("%s_flip%d" % (nm, k), bytes(b)))
    return out


def test_truncated_or_corrupt_is_edata_or_gzread(gunzip_host, tmp_path):
    p = str(tmp_path / "d.gz")
    n_err = 0
    for name, z in damaged():
        open(p, "wb").write(z)
        ref, ref_err = gzread(p)
        for chunk in (1024, 0):
            rc, text, _, at = hostsim_gunzip(gunzip_host, z, chunk)
            if ref_err:
                assert rc == EDATA and at <= len(z), (name, chunk)
                n_err += 1
            else:  # damage in bytes gzread ignores (header fields, trailing bytes)
                assert rc == 0 and text == ref, (name, chunk)
    assert n_err > 100


@pytest.mark.skipif(T.gpu_visible(), reason="box has a GPU")
def test_no_gpu_no_device_gunzip(ssq_lib_cpu):
    h = C.c_void_p()
    assert ssq_lib_cpu.ssq_gunzip_create(0, C.c_size_t(0), C.byref(h)) == -1
