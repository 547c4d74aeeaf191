"""hgpu_cram_compress_blocks_host — cram_compress_block2's method trial (cram/cram_io.c:1912-2308) for a batch of blocks: every
winner must be a stream the REFERENCE decoder of that method expands to the block's data, the framing must be cram_write_block's
(CRC-32 over header + payload), and the winning size must be within 3 % (+64 bytes) of the smallest stream the reference's
own encoders produce over the same candidate methods."""
import ctypes as C
import random
import zlib
import numpy as np
import pytest
import htslib_b200 as H
from _libs import ref, ref_rans_nx16_encode, ref_rans_nx16_decode, ref_rans_4x8, ref_arith, stored_reference
from test_oracle_rans import _synth

pytestmark = [pytest.mark.gpu]

RANS_PR = {5: 0, 17: 1, 18: 64, 19: 9, 20: 128, 21: 129, 22: 192, 23: 193}
ARITH_PR = {6: 0, 25: 1, 26: 64, 28: 128, 29: 129, 30: 192, 31: 193}          # 27 (X4 stripe) is not produced
V31_MASK = sum(1 << m for m in RANS_PR)                                          # what a CRAM 3.1 'normal' profile allows for most series
ALL_MASK = V31_MASK | sum(1 << m for m in ARITH_PR) | (1 << 4) | (1 << 16)       # + arith + rANS 4x8


def itf8(buf, p):
    c = buf[p]
    if c < 0x80: return c, p + 1
    if c < 0xc0: return ((c & 0x3f) << 8) | buf[p + 1], p + 2
    if c < 0xe0: return ((c & 0x1f) << 16) | (buf[p + 1] << 8) | buf[p + 2], p + 3
    if c < 0xf0: return ((c & 0x0f) << 24) | (buf[p + 1] << 16) | (buf[p + 2] << 8) | buf[p + 3], p + 4
    return ((c & 0x0f) << 28) | (buf[p + 1] << 20) | (buf[p + 2] << 12) | (buf[p + 3] << 4) | (buf[p + 4] & 0x0f), p + 5


@stored_reference
def ref_size(raw, m):
    """Size of the reference encoder's output for block method m (only the size is stored)."""
    if m in RANS_PR:
        o = RANS_PR[m]
        return len(ref_rans_nx16_encode.__wrapped__(raw, o | (1 << 17)))
    if m in ARITH_PR:
        return len(ref_arith.__wrapped__(raw, ARITH_PR[m]))
    return len(ref_rans_4x8.__wrapped__(raw, 0 if m == 4 else 1))


def ref_decode(method, comp, usize):
    if method == 5: return ref_rans_nx16_decode(comp, usize)
    if method == 6: return ref_arith(comp=comp, cap=usize)
    if method == 4: return ref_rans_4x8(comp=comp)
    raise AssertionError(method)


@pytest.mark.parametrize("mask", [V31_MASK, ALL_MASK])
def test_trial_picks_a_valid_and_small_stream(mask):
    rng = random.Random(9)
    raws = [_synth(rng, n, kind) for kind in ("q4", "q40", "runs", "one", "u32", "rand") for n in (0, 5, 300, 4099, 70001)]
    n = len(raws)
    ctx = H.Context(0)
    L = H.lib()
    keep = [np.frombuffer(r, dtype=np.uint8) if r else np.zeros(1, dtype=np.uint8) for r in raws]
    ptrs = (C.c_void_p * n)(*[k.ctypes.data for k in keep])
    plen = np.array([len(r) for r in raws], dtype=np.uint32)
    masks = np.full(n, mask, dtype=np.uint32)
    cid = np.arange(10, 10 + n, dtype=np.int32)
    ctype = np.full(n, 4, dtype=np.uint8)
    cap = int(plen.sum()) * 2 + 64 * n + 4096
    out = np.zeros(cap, dtype=np.uint8)
    off = np.zeros(n, dtype=np.uint64)
    tot = C.c_uint64(0)
    chosen = np.zeros(n, dtype=np.int32)
    L.hgpu_cram_compress_blocks_host.argtypes = [C.c_void_p] * 6 + [C.c_uint32, C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p, C.c_void_p]
    rc = L.hgpu_cram_compress_blocks_host(ctx.h, ptrs, plen.ctypes.data, masks.ctypes.data, cid.ctypes.data, ctype.ctypes.data, n,
                                          out.ctypes.data, cap, off.ctypes.data, C.byref(tot), chosen.ctypes.data)
    assert rc == 0, H.last_error()
    buf = out[:tot.value].tobytes()
    p = 0
    for i, raw in enumerate(raws):
        assert p == int(off[i])
        start = p
        method, ct = buf[p], buf[p + 1]; p += 2
        assert ct == 4
        v, p = itf8(buf, p); assert v == 10 + i
        csz, p = itf8(buf, p); usz, p = itf8(buf, p)
        assert usz == len(raw)
        comp = buf[p:p + csz]; p += csz
        assert int.from_bytes(buf[p:p + 4], "little") == zlib.crc32(buf[start:p]); p += 4       # cram_write_block :1546-1556
        if method == 0:
            assert comp == raw and chosen[i] == 0
        else:
            assert ref_decode(method, comp, len(raw)) == raw, (i, method, int(chosen[i]))
            assert csz < len(raw)
        if len(raw):
            best_ref = min([ref_size(raw, m) for m in range(32) if mask >> m & 1 and (m in RANS_PR or m in ARITH_PR or m in (4, 16))] + [len(raw)])
            assert csz <= 1.03 * best_ref + 64, (i, len(raw), int(chosen[i]), csz, best_ref)
    assert p == len(buf)
    ctx.close()
