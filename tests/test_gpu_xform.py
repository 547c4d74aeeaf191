"""GPU parity: the byte transforms of the libhtscodecs seam that cram_codecs.c binds directly — hts_pack / hts_unpack_meta /
hts_unpack (pack.c:56-330) and hts_rle_encode / hts_rle_decode (rle.c:48-190) — against the compiled reference: the
same bytes out of the encoders, the same data (or the same refusal) out of the decoders."""
import ctypes as C
import random
import numpy as np
import pytest
import htslib_b200 as H
from _libs import ref, stored_reference

pytestmark = [pytest.mark.gpu]
u8p = C.POINTER(C.c_uint8)


def bind(L):
    L.hts_pack.restype = C.c_void_p
    L.hts_pack.argtypes = [C.c_void_p, C.c_int64, C.c_void_p, C.POINTER(C.c_int), C.POINTER(C.c_uint64)]
    L.hts_unpack_meta.restype = C.c_uint8
    L.hts_unpack_meta.argtypes = [C.c_void_p, C.c_uint32, C.c_uint64, C.c_void_p, C.POINTER(C.c_int)]
    L.hts_unpack.restype = C.c_void_p
    L.hts_unpack.argtypes = [C.c_void_p, C.c_int64, C.c_void_p, C.c_uint64, C.c_int, C.c_void_p]
    L.hts_rle_encode.restype = C.c_void_p
    L.hts_rle_encode.argtypes = [C.c_void_p, C.c_uint64, C.c_void_p, C.POINTER(C.c_uint64), C.c_void_p, C.POINTER(C.c_int), C.c_void_p, C.POINTER(C.c_uint64)]
    L.hts_rle_decode.restype = C.c_void_p
    L.hts_rle_decode.argtypes = [C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint64, C.c_void_p, C.c_int, C.c_void_p, C.POINTER(C.c_uint64)]
    return L


def pack(L, data):
    meta = (C.c_uint8 * 300)(); ml = C.c_int(0); ol = C.c_uint64(0)
    buf = (C.c_uint8 * max(1, len(data))).from_buffer_copy(data or b"\0")
    p = L.hts_pack(buf, len(data), meta, C.byref(ml), C.byref(ol))
    if not p:
        return None
    out = C.string_at(p, ol.value)
    C.CDLL(None).free(C.c_void_p(p))
    return bytes(meta[:ml.value]), out


def rle_enc(L, data, syms=None):
    run = (C.c_uint8 * (len(data) * 5 + 16))(); rl = C.c_uint64(0); ol = C.c_uint64(0)
    rs = (C.c_uint8 * 256)(); ns = C.c_int(0)
    if syms:
        for i, s in enumerate(syms): rs[i] = s
        ns.value = len(syms)
    out = (C.c_uint8 * (len(data) * 2 + 16))()
    buf = (C.c_uint8 * max(1, len(data))).from_buffer_copy(data or b"\0")
    p = L.hts_rle_encode(buf, len(data), run, C.byref(rl), rs, C.byref(ns), out, C.byref(ol))
    assert p
    return bytes(out[:ol.value]), bytes(run[:rl.value]), bytes(rs[:ns.value])


def rle_dec(L, lit, run, syms, cap):
    out = (C.c_uint8 * max(1, cap))(); ol = C.c_uint64(cap)
    a = (C.c_uint8 * max(1, len(lit))).from_buffer_copy(lit or b"\0"); b = (C.c_uint8 * max(1, len(run))).from_buffer_copy(run or b"\0")
    s = (C.c_uint8 * 256).from_buffer_copy(syms + b"\0" * (256 - len(syms)))
    p = L.hts_rle_decode(a, len(lit), b, len(run), s, len(syms), out, C.byref(ol))
    return bytes(out[:ol.value]) if p else None


@stored_reference(digest=True)
def ref_xform_pack(data):
    return pack(bind(ref()), data)


@stored_reference
def ref_xform_unpack_meta(meta, n):
    """(bytes of meta used, symbol count, map) from the reference's hts_unpack_meta."""
    R = bind(ref())
    mp = (C.c_uint8 * 16)(); ns = C.c_int(-1)
    used = R.hts_unpack_meta((C.c_uint8 * len(meta)).from_buffer_copy(meta), len(meta), n, mp, C.byref(ns))
    return used, ns.value, bytes(mp)


@stored_reference
def ref_xform_unpack_refused(packed, n, ns, mp):
    R = bind(ref())
    out = (C.c_uint8 * max(1, n))()
    pb = (C.c_uint8 * max(1, len(packed))).from_buffer_copy(packed or b"\0")
    return not R.hts_unpack(pb, len(packed), out, n, ns, (C.c_uint8 * 16).from_buffer_copy(mp))


@stored_reference(digest=True)
def ref_xform_rle_encode(data, syms):
    return rle_enc(bind(ref()), data, syms)


@stored_reference(digest=True)
def ref_xform_rle_decode(lit, run, syms, cap):
    return rle_dec(bind(ref()), lit, run, syms, cap)


def test_pack_unpack_equal_the_reference():
    G = bind(H.lib())
    rng = random.Random(12)
    for nsym in (1, 2, 3, 4, 5, 16, 17, 40):
        alphabet = rng.sample(range(256), nsym)
        for n in (0, 1, 2, 3, 7, 8, 9, 15, 16, 17, 1000, 70001):
            data = bytes(rng.choice(alphabet) for _ in range(n))
            want = ref_xform_pack(data); got = pack(G, data)
            assert got == want, (nsym, n)
            if want is None:
                continue
            meta, packed = got
            # meta -> map, then unpack on the device == the input
            mp = (C.c_uint8 * 16)(); ns = C.c_int(-1)
            mb = (C.c_uint8 * len(meta)).from_buffer_copy(meta)
            used = G.hts_unpack_meta(mb, len(meta), n, mp, C.byref(ns))
            assert (used, ns.value, bytes(mp)) == ref_xform_unpack_meta(meta, n)
            out = (C.c_uint8 * max(1, n))()
            pb = (C.c_uint8 * max(1, len(packed))).from_buffer_copy(packed or b"\0")
            assert G.hts_unpack(pb, len(packed), out, n, ns.value, mp)
            assert bytes(out[:n]) == data
            if n > 8 and ns.value > 1:                                   # too little packed data for the claimed output: refused, as the reference does
                assert not G.hts_unpack(pb, max(0, len(packed) - 2), out, n, ns.value, mp)
                assert ref_xform_unpack_refused(packed[:max(0, len(packed) - 2)], n, ns.value, bytes(mp))


def test_rle_equal_the_reference():
    G = bind(H.lib())
    rng = random.Random(13)
    cases = [b"", b"a", b"aa", b"ab", b"a" * 31, b"a" * 32, b"a" * 33, b"a" * 64 + b"b", b"ab" * 100, b"a" * 100000]
    for n in (50, 257, 5000, 70000):
        runs = []
        while sum(map(len, runs)) < n:
            runs.append(bytes([rng.choice(b"ACGT#")]) * rng.choice([1, 1, 1, 2, 3, 9, 40, 300]))
        cases.append(b"".join(runs)[:n])
    for data in cases:
        for syms in (None, [ord("A"), ord("#")]):
            want = ref_xform_rle_encode(data, syms); got = rle_enc(G, data, syms)
            assert got == want, (len(data), syms)
            lit, run, ss = got
            assert rle_dec(G, lit, run, ss, len(data)) == data == (ref_xform_rle_decode(lit, run, ss, len(data)) if data else data)
            if len(data) > 40 and lit != data:                           # an output buffer that is too small: refused
                assert rle_dec(G, lit, run, ss, len(data) - 1) is None and ref_xform_rle_decode(lit, run, ss, len(data) - 1) is None


def test_version_string():
    H.lib().htscodecs_version.restype = C.c_char_p
    assert H.lib().htscodecs_version().startswith(b"1.6")
