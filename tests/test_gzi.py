"""Host index arithmetic (no GPU): .gzi pairs and uncompressed <-> virtual offsets from the scan table, against the
compiled reference — bgzf_index_build_init / bgzf_index_dump when writing, bgzf_index_load + bgzf_useek when
reading (bgzf.c:2336-2621) — and against the reference's own fixture test/bgziptest.txt.gz.gzi."""
import ctypes as C
import os
import random
import struct
import tempfile
import numpy as np
import pytest
import htslib_b200 as H
from _libs import GOLD, ref, stored_reference


def scan(img):
    L = H.lib()
    L.hgpu_bgzf_scan.restype = C.c_long
    a = np.frombuffer(img, dtype=np.uint8)
    n = L.hgpu_bgzf_scan(a.ctypes.data, C.c_uint64(a.size), None, None, None, C.c_long(0))
    assert n > 0
    off = np.zeros(n, dtype=np.uint64); ln = np.zeros(n, dtype=np.uint32); isz = np.zeros(n, dtype=np.uint32)
    assert L.hgpu_bgzf_scan(a.ctypes.data, C.c_uint64(a.size), off.ctypes.data, ln.ctypes.data, isz.ctypes.data, C.c_long(n)) == n
    return off, ln, isz


def gzi(off, isz, terminating):
    L = H.lib()
    L.hgpu_bgzf_gzi_entries.restype = C.c_long
    L.hgpu_bgzf_gzi_dump.restype = C.c_long
    n = len(off)
    k = L.hgpu_bgzf_gzi_entries(off.ctypes.data, isz.ctypes.data, C.c_long(n), terminating, None, None, C.c_long(0))
    ca = np.zeros(max(1, k), dtype=np.uint64); ua = np.zeros(max(1, k), dtype=np.uint64)
    assert L.hgpu_bgzf_gzi_entries(off.ctypes.data, isz.ctypes.data, C.c_long(n), terminating, ca.ctypes.data, ua.ctypes.data, C.c_long(k)) == k
    need = L.hgpu_bgzf_gzi_dump(ca.ctypes.data, ua.ctypes.data, C.c_long(k), None, C.c_size_t(0))
    out = np.zeros(need, dtype=np.uint8)
    assert L.hgpu_bgzf_gzi_dump(ca.ctypes.data, ua.ctypes.data, C.c_long(k), out.ctypes.data, C.c_size_t(need)) == need
    return ca[:k], ua[:k], out.tobytes()


def test_reference_fixture_gzi():
    img = open(os.path.join(GOLD, "htslib", "bgziptest.txt.gz"), "rb").read()
    want = open(os.path.join(GOLD, "htslib", "bgziptest.txt.gz.gzi"), "rb").read()
    off, ln, isz = scan(img)
    _, _, got = gzi(off, isz, 1)                                     # the fixture was made by a reader (one extra record)
    assert got == want


def _bind(r):
    r.bgzf_open.restype = C.c_void_p
    r.bgzf_open.argtypes = [C.c_char_p, C.c_char_p]
    r.bgzf_write.restype = C.c_ssize_t
    r.bgzf_write.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t]
    r.bgzf_read.restype = C.c_ssize_t
    r.bgzf_read.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t]
    r.bgzf_close.argtypes = [C.c_void_p]
    r.bgzf_flush.argtypes = [C.c_void_p]
    r.bgzf_index_build_init.argtypes = [C.c_void_p]
    r.bgzf_index_dump.argtypes = [C.c_void_p, C.c_char_p, C.c_char_p]
    r.bgzf_index_load.argtypes = [C.c_void_p, C.c_char_p, C.c_char_p]
    r.bgzf_useek.argtypes = [C.c_void_p, C.c_int64, C.c_int]
    return r


@stored_reference(limit=20000)
def ref_bgzf_write_indexed(data, chunks):
    """(file, .gzi) of data written by the reference in the given ragged writes (level 6, an explicit flush
    after each 3-byte write) with bgzf_index_build_init / bgzf_index_dump."""
    r = _bind(ref())
    with tempfile.TemporaryDirectory() as td:
        path = os.path.join(td, "t.gz").encode()
        fp = r.bgzf_open(path, b"w6")
        assert fp and r.bgzf_index_build_init(fp) == 0
        p = 0
        for chunk in chunks:
            assert r.bgzf_write(fp, data[p:p + chunk], chunk) == chunk
            p += chunk
            if chunk == 3:
                r.bgzf_flush(fp)
        assert p == len(data)
        assert r.bgzf_index_dump(fp, path, b".gzi") == 0
        r.bgzf_close(fp)
        return open(path, "rb").read(), open(path + b".gzi", "rb").read()


@stored_reference(limit=20000)
def ref_bgzf_useek(img, gzi, offsets):
    """For each uncompressed offset: (block_address, block_offset, next 16 bytes) after the reference's
    bgzf_index_load + bgzf_useek."""
    r = _bind(ref())
    out = []
    with tempfile.TemporaryDirectory() as td:
        path = os.path.join(td, "t.gz").encode()
        open(path, "wb").write(img)
        open(path + b".gzi", "wb").write(gzi)
        fp = r.bgzf_open(path, b"r")
        assert r.bgzf_index_load(fp, path, b".gzi") == 0
        buf = (C.c_uint8 * 32)()
        for u in offsets:
            assert r.bgzf_useek(fp, u, 0) == 0
            raw = C.string_at(fp, 40)                               # BGZF: ... int block_offset @16; int64 block_address @24 (htslib/bgzf.h:68-83)
            block_offset, = struct.unpack_from("<i", raw, 16)
            block_address, = struct.unpack_from("<q", raw, 24)
            n = r.bgzf_read(fp, buf, 16)
            out.append((block_address, block_offset, bytes(buf[:n])))
        r.bgzf_close(fp)
    return out


def test_gzi_and_useek_equal_the_reference():
    rng = random.Random(4)
    data = bytearray(b"ACGTNACGTTGCA\n" * 28572)[:400000]               # compressible, so the stored file is small
    for _ in range(400):
        data[rng.randrange(len(data))] = rng.choice(b"ACGTN\n")
    data = bytes(data)
    img, want = ref_bgzf_write_indexed(data, [1, 70000, 65280, 3, 0, 120000, 144716])   # ragged writes, an explicit flush in the middle
    off, ln, isz = scan(img)
    ca, ua, got = gzi(off, isz, 0)                                   # ... and this one by the writer
    assert got == want
    # random access: the reference seeks by uncompressed offset with the loaded index; ours gives the virtual offset
    L = H.lib()
    L.hgpu_bgzf_useek.restype = C.c_uint64
    L.hgpu_bgzf_utell.restype = C.c_uint64
    us = [0, 1, 65279, 65280, 65281, 70000, 135283, 200000, len(data) - 1] + [rng.randrange(len(data)) for _ in range(40)]
    for u, (block_address, block_offset, after) in zip(us, ref_bgzf_useek(img, want, us)):
        v = L.hgpu_bgzf_useek(ca.ctypes.data, ua.ctypes.data, C.c_long(len(ca)), C.c_uint64(u))
        assert v == (block_address << 16 | block_offset), (u, v, block_address, block_offset)
        assert L.hgpu_bgzf_utell(ca.ctypes.data, ua.ctypes.data, C.c_long(len(ca)), C.c_uint64(v)) == u
        assert after == data[u:u + 16]
    assert L.hgpu_bgzf_utell(ca.ctypes.data, ua.ctypes.data, C.c_long(len(ca)), C.c_uint64((int(off[1]) + 1) << 16)) == 2 ** 64 - 1
