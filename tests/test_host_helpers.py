"""Host-side helpers of the C ABI that need no device: size bounds must equal the reference's own
(callers size their buffers with them), and the tok3 size field reader must follow the block header."""
import ctypes as C
import random
import struct

import pytest

import htslib_b200 as H
from _libs import ref_arith_compress_bounds


def test_tok3_out_bound_reads_the_header():
    L = H.lib()
    blk = struct.pack("<IIB", 12345, 10, 0) + b"\0" * 8
    assert L.hgpu_tok3_out_bound(blk, len(blk)) == 12345 + 1024        # the reference allocates ulen + 1024 (:1808)
    assert L.hgpu_tok3_out_bound(blk[:8], 8) == 0                        # sz < 9 -> NULL there (:1680)
    assert L.hgpu_tok3_out_bound(struct.pack("<IIB", 0x7fffffff, 1, 0), 9) == 0


def test_bounds_equal_the_reference():
    L = H.lib()
    L.hgpu_arith_compress_bound.restype = C.c_uint32
    L.hgpu_arith_compress_bound.argtypes = [C.c_uint32, C.c_int]
    L.hgpu_rans4x8_compress_bound.restype = C.c_uint32
    L.hgpu_rans4x8_compress_bound.argtypes = [C.c_uint32]
    rng = random.Random(3)
    for _ in range(200):
        size = rng.choice([0, 1, 7, 100, 65536, rng.randrange(1, 1 << 24)])
        pairs = [(size, order) for order in (0, 1, 64, 65, 128, 129, 192, 193, 8, 9, 8 | (3 << 8))]
        for (s, order), want in zip(pairs, ref_arith_compress_bounds(pairs)):
            assert L.hgpu_arith_compress_bound(s, order) == want, (s, order)
        # rans_compress_O0/O1 allocate 1.05*in_size + 257*257*3 + 9 (rANS_static.c:77, :401)
        assert L.hgpu_rans4x8_compress_bound(size) == int(1.05 * size) + 257 * 257 * 3 + 9
