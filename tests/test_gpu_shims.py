"""GPU: the reference-named entry points of the libhtscodecs link seam (htslib_b200/csrc/shims.cu) called the
way cram/cram_io.c calls them — malloc'd results, NULL on error — and checked against the compiled reference:
decoders on the reference encoder's output, the byte-identical encoders against the reference's bytes, the
others by the reference decoding what they wrote."""
import ctypes as C
import random

import pytest

import htslib_b200 as H
import _libs as L
from test_oracle_rans import _synth
from test_oracle_tok3 import _names
from test_oracle_fqz import _quals

pytestmark = [pytest.mark.gpu]
libc = C.CDLL(None)
libc.free.argtypes = [C.c_void_p]


def _take(p, n):
    assert p
    b = C.string_at(p, n)
    libc.free(C.c_void_p(p))
    return b


@pytest.fixture(scope="module")
def lib():
    l = H.lib()
    for name in ("rans_uncompress", "rans_compress", "arith_compress_to", "arith_compress", "arith_uncompress_to", "arith_uncompress",
                 "rans_compress_to_4x16", "rans_compress_4x16", "tok3_encode_names", "fqz_compress"):
        getattr(l, name).restype = C.c_void_p
    l.arith_compress_bound.restype = C.c_uint
    l.rans_compress_bound_4x16.restype = C.c_uint
    return l


def test_rans4x8(lib):
    rng = random.Random(1)
    for order in (0, 1):
        raw = _synth(rng, 30001, "q40")
        n = C.c_uint(0)
        comp = _take(lib.rans_compress(L.buf(raw), C.c_uint(len(raw)), C.byref(n), C.c_int(order)), n.value)
        assert comp == L.ref_rans_4x8_encoded(raw, order)
        m = C.c_uint(0)
        assert _take(lib.rans_uncompress(L.buf(comp), C.c_uint(len(comp)), C.byref(m)), m.value) == raw
    assert not lib.rans_uncompress(L.buf(comp[:20]), C.c_uint(20), C.byref(m))


def test_arith(lib):
    rng = random.Random(2)
    for order in (0, 1, 65, 193):
        raw = _synth(rng, 4099, "q4")
        n = C.c_uint(0)
        comp = _take(lib.arith_compress(L.buf(raw), C.c_uint(len(raw)), C.byref(n), C.c_int(order)), n.value)
        assert comp == L.ref_arith_encoded(raw, order)
        assert lib.arith_compress_bound(C.c_uint(len(raw)), C.c_int(order)) == L.ref_arith_compress_bounds([(len(raw), order)])[0]
        m = C.c_uint(0)
        assert _take(lib.arith_uncompress(L.buf(comp), C.c_uint(len(comp)), C.byref(m)), m.value) == raw
        out = (C.c_uint8 * len(raw))(); m = C.c_uint(len(raw))
        assert lib.arith_uncompress_to(L.buf(comp), C.c_uint(len(comp)), out, C.byref(m)) and bytes(out[: m.value]) == raw
    bad = bytearray(comp); bad[1] ^= 0x7f                           # size field no longer matches
    assert not lib.arith_uncompress_to(L.buf(bytes(bad)), C.c_uint(len(bad)), out, C.byref(C.c_uint(len(raw))))


def test_rans_nx16_encode(lib):
    rng = random.Random(3)
    for order in (0, 1, 4, 5, 0x0100 | 5, 0x40 | 1):                # SIMD-hint and RLE bits are accepted and not acted on
        raw = _synth(rng, 70001, "q4")
        n = C.c_uint(0)
        comp = _take(lib.rans_compress_4x16(L.buf(raw), C.c_uint(len(raw)), C.byref(n), C.c_int(order)), n.value)
        assert L.ref_rans_nx16_decode(comp, len(raw)) == raw
        assert len(comp) <= lib.rans_compress_bound_4x16(C.c_uint(len(raw)), C.c_int(order))
    lib.rans_set_cpu(C.c_int(0))


def test_tok3_and_fqz_encode(lib):
    blob = _names(random.Random(4), 600, 0)
    n = C.c_int(0); last = C.c_int(-1)
    src = C.create_string_buffer(blob + b"trailing", len(blob) + 9)
    comp = _take(lib.tok3_encode_names(src, C.c_int(len(blob) + 8), C.c_int(3), C.c_int(0), C.byref(n), C.byref(last)), n.value)
    assert last.value == len(blob)                                  # the unterminated tail is left for the next block
    assert L.ref_tok3_decode(comp) == blob
    q, lens, flags = _quals(random.Random(5), 300, "q40")
    la = (C.c_uint32 * len(lens))(*lens); fa = (C.c_uint32 * len(lens))(*flags)
    sl = L.FqzSlice(len(lens), la, fa)
    m = C.c_size_t(0)
    qb = C.create_string_buffer(q, len(q) + 1)
    comp = _take(lib.fqz_compress(C.c_int(4), C.byref(sl), qb, C.c_size_t(len(q)), C.byref(m), C.c_int(0), None), m.value)
    assert L.ref_fqz_decompress(comp) == q
    assert not lib.fqz_compress(C.c_int(3), C.byref(sl), qb, C.c_size_t(len(q)), C.byref(m), C.c_int(0), None)   # CRAM 3.0 layout: declined
