"""Schedules of LZ77 match records in the inflate kernels: records executed 32 per lane group, out of order, in rounds.

Members are written with the raw-DEFLATE writer of test_gpu_bgzf_lz77 (chosen tokens) and shaped so that a schedule of
32 records at a time (a batch, or a rolling window of the oldest pending records) stalls, drains and refills in the ways
that matter: long dependency chains, chains followed by independent records, sources written many rounds earlier, runs
of both kinds with records that read them, match counts around 32 and 64, and small members on the uniform decoder.  Every member goes through bgzf_inflate_kernel (at every output offset
mod 4) and through gzip_inflate_kernel; the expected output is always zlib's inflate of the same stream."""
import ctypes as C
import os
import random
import struct
import zlib
import numpy as np
import pytest
import htslib_b200 as H
from _libs import GOLD
from test_gpu_bgzf_lz77 import Deflate, expand, _bgzf, _inflate

PAR_MIN_BITS = 32 * 96                      # member bits after the block header (footer included) that take the parallel decoder
PAR_MIN_BYTES = PAR_MIN_BITS // 8 + 16


def _fixed(toks, parallel, rng, prefix=b""):
    """one member: an optional stored prefix, then one fixed-Huffman block; `parallel` pads the block with 9-bit
    literals behind the tokens so that the body is long enough for the lane-parallel decoder"""
    d = Deflate()
    if prefix:
        d.stored(prefix)
    if parallel:
        toks = toks + [rng.randrange(144, 256) for _ in range(PAR_MIN_BYTES)]
    d.fixed(toks, final=True)
    return d.raw()


def _chain(rng, n, ln, gap=0):
    """n matches, each copying the previous one (its source is exactly the previous match's destination)"""
    toks = [rng.randrange(256) for _ in range(ln)]
    for i in range(n):
        g = (gap + i) % 4 if gap else 0                                  # literals in front move the destination offset mod 4
        toks += [rng.randrange(256) for _ in range(g)]
        toks.append((ln, ln + g))
    return toks


def _token_sets(rng):
    """(name, tokens, stored prefix); every set is made into a small member (uniform decoder) where it fits, and a
    padded one (lane-parallel decoder)"""
    sets = []
    # serial chains: every round retires one record
    for ln in (3, 4, 5, 8, 33, 100):
        sets.append(("chain%d" % ln, _chain(rng, 120, ln), b""))
    sets.append(("chain_gaps", _chain(rng, 100, 9, gap=1), b""))
    # a long chain, then hundreds of independent records reading a stored prefix: a stalled head, a ready tail
    prefix = bytes(rng.randrange(256) for _ in range(6000))
    toks, o = _chain(rng, 100, 7), 6000 + 7 + 700
    for _ in range(500):
        ln = rng.choice((3, 4, 9, 17, 31, 40))
        toks.append((ln, o - rng.randrange(0, 5000))); o += ln
    sets.append(("chain_then_independent", toks, prefix))
    # independent records interleaved with a chain: each group of 32 holds both
    toks, o = [rng.randrange(256) for _ in range(16)], 6000 + 16
    for i in range(200):
        if i % 3 == 0:
            toks.append((16, 16)); o += 16
        else:
            ln = rng.choice((3, 5, 12, 258)); toks.append((ln, o - rng.randrange(0, 5000))); o += ln
    sets.append(("chain_interleaved", toks, prefix))
    # sources written by records retired many rounds earlier: a match at [64, 114), a 90-record chain at [120, 660),
    # then records reading the first match, the chain's middle and the chain's first record
    toks = [rng.randrange(256) for _ in range(64)] + [(50, 64)] + [rng.randrange(256) for _ in range(6)] + [(6, 6)] * 90
    o = len(expand(toks))
    assert o == 660
    toks += [(40, o - 64), (30, o + 40 - 390), (20, o + 70 - 120), (258, o + 90 - 64), (3, 1)]
    sets.append(("old_sources", toks, b""))
    # runs of period <= 4 (word copy) and > 4 (warp path) inside one window, with records that read them
    toks = [rng.randrange(256) for _ in range(40)]
    for k in range(6):
        toks += [(20 + k, 1), (10, 10), (40, 7 + k), (30, 30), (64, 33), (5, 3), (45, 64 + 5),
                 rng.randrange(256), (9, 2), (100, 40), (12, 4), (31, 31 + 12)]
    sets.append(("runs_mixed", toks, b""))
    # 1, 31, 32, 33, 64 and 65 matches: the last group of records drains at the member's end, independent and chained
    for n in (1, 31, 32, 33, 64, 65):
        toks = [rng.randrange(256) for _ in range(40)] + [(rng.randrange(3, 20), rng.randrange(20, 40)) for _ in range(n)]
        sets.append(("count%d" % n, toks, b""))
        sets.append(("count%d_chain" % n, _chain(rng, n, 11), b""))
    return sets


def _is_parallel(raw):
    """True when a member of one fixed-Huffman block is long enough for the lane-parallel decoder"""
    return (len(raw) + 8) * 8 - 3 >= PAR_MIN_BITS


def _members():
    rng = random.Random(21)
    out = []
    for name, toks, prefix in _token_sets(rng):
        small = _fixed(toks, False, rng, prefix)
        if not prefix and not _is_parallel(small):
            out.append((name, small))
        out.append((name + "_par", _fixed(toks, True, rng, prefix)))
    return out


def test_window_members_inflate_with_zlib():
    """the streams themselves: zlib inflates each to the tokens' expansion, each fits a BGZF block, and the small
    members the other tests rely on take the uniform decoder"""
    rng = random.Random(21)
    for name, toks, prefix in _token_sets(rng):
        raw = _fixed(toks, False, rng, prefix)
        assert zlib.decompress(raw, -15) == expand(toks, prefix), name
    ms = _members()
    names = [n for n, _ in ms]
    assert len(names) == len(set(names))
    for name, raw in ms:
        assert len(zlib.decompress(raw, -15)) <= 65536, name
    small = {n for n in names if not n.endswith("_par")}
    assert {"chain3", "chain_gaps", "runs_mixed", "old_sources", "count1", "count65", "count65_chain"} <= small
    # a chain's records each read exactly the previous record's destination
    toks = _chain(random.Random(0), 120, 8, gap=1)
    dst, prev = 8, None
    for t in toks[8:]:
        if isinstance(t, int):
            dst += 1
            continue
        if prev is not None:
            assert dst - t[1] == prev[0] and t[0] == prev[1] - prev[0]
        prev = (dst, dst + t[0])
        dst += t[0]


@pytest.fixture(scope="module")
def ctx():
    c = H.Context(0)
    yield c
    c.close()


def _check(ctx, raws, shifts=range(4), flip=False):
    blocks, want, sh = [], [], []
    for raw in raws:
        data = zlib.decompress(raw, -15)
        for s in shifts:
            blocks.append(_bgzf(raw, data, flip)); want.append(data); sh.append(s)
    res = _inflate(ctx, blocks, sh, [len(w) for w in want])
    if flip:
        return [(i, st) for i, (st, _) in enumerate(res) if st != H.BGZF_ERR_CRC]
    return [(i, st, len(d), len(w)) for i, ((st, d), w) in enumerate(zip(res, want)) if st != 0 or d != w]


def _gzip(ctx, raws, flip=False):
    """each raw DEFLATE stream as one gzip member through cram_uncompress_blocks (gzip_inflate_kernel)"""
    comps, datas = [], []
    for raw in raws:
        data = zlib.decompress(raw, -15)
        crc = zlib.crc32(data) ^ (1 if flip else 0)
        comps.append(bytes([0x1f, 0x8b, 8, 0, 0, 0, 0, 0, 0, 3]) + raw + struct.pack("<II", crc, len(data)))
        datas.append(data)
    n = len(comps)
    dt = np.dtype([("data_off", "<u8"), ("comp_size", "<u4"), ("uncomp_size", "<u4"), ("content_id", "<i4"), ("method", "u1"),
                   ("content_type", "u1"), ("hdr_len", "<u2"), ("container", "<u4"), ("pad2", "<u4")])
    blocks = np.zeros(n, dtype=dt)
    for i, cb in enumerate(comps):
        blocks[i]["method"] = 1; blocks[i]["content_type"] = 4; blocks[i]["content_id"] = 10 + i
        blocks[i]["comp_size"] = len(cb); blocks[i]["uncomp_size"] = len(datas[i])
    L = H.lib()
    L.hgpu_cram_write_blocks_host.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p]
    bufs = [np.frombuffer(cb, dtype=np.uint8).copy() for cb in comps]
    ptrs = (C.c_void_p * n)(*[b.ctypes.data for b in bufs])
    img = np.zeros(sum(len(cb) for cb in comps) + 32 * n, dtype=np.uint8)
    off = np.zeros(n, dtype=np.uint64); tot = C.c_uint64(0)
    assert L.hgpu_cram_write_blocks_host(ctx.h, blocks.ctypes.data, ptrs, n, img.ctypes.data, img.size, off.ctypes.data, C.byref(tot)) == 0
    img = img[:tot.value].copy()
    scanned = blocks.copy()
    for i in range(n):
        hl = 2 + sum(1 if v < 0x80 else 2 if v < 0x4000 else 3 if v < 0x200000 else 4 if v < 0x10000000 else 5
                     for v in (10 + i, len(comps[i]), len(datas[i])))
        scanned[i]["hdr_len"] = hl; scanned[i]["data_off"] = int(off[i]) + hl
    _, res = H.cram_uncompress_blocks(ctx, img, scanned)
    return res, datas


@pytest.mark.gpu
def test_window_members_bgzf(ctx):
    """every member through bgzf_inflate_kernel at output offsets 0..3 mod 4"""
    ms = _members()
    bad = _check(ctx, [raw for _, raw in ms])
    assert not bad, [(ms[i // 4][0],) + b[1:] for b in bad[:8] for i in [b[0]]]


@pytest.mark.gpu
def test_window_members_flipped_crc(ctx):
    """the CRC cursor absorbs rows behind the match frontier while the records run: a flipped footer CRC still fails"""
    ms = _members()
    bad = _check(ctx, [raw for _, raw in ms], shifts=(1,), flip=True)
    assert not bad, [(ms[i][0], st) for i, st in bad[:8]]


@pytest.mark.gpu
def test_window_members_gzip(ctx):
    """every member as a gzip member (gzip_inflate_kernel), and all of them as the blocks of one large member"""
    ms = _members()
    res, want = _gzip(ctx, [raw for _, raw in ms])
    bad = [(ms[i][0], st, len(d)) for i, ((st, d), w) in enumerate(zip(res, want)) if st != 0 or d != w]
    assert not bad, bad[:8]
    # one member of many non-final blocks: records reach back across deflate blocks
    rng = random.Random(5)
    d = Deflate()
    prefix = bytes(rng.randrange(256) for _ in range(40000))
    d.stored(prefix)
    for name, toks, pre in _token_sets(rng):
        if not pre:
            d.fixed(toks + [(200, 30000), (258, 1)])
    d.stored(b"", final=True)
    raw = d.raw()
    assert len(zlib.decompress(raw, -15)) > 65536
    res, want = _gzip(ctx, [raw])
    assert res[0][0] == 0 and res[0][1] == want[0]
    res, _ = _gzip(ctx, [raw], flip=True)
    assert res[0][0] != 0


@pytest.mark.gpu
def test_window_regress_blocks(ctx):
    """the two regression blocks, every output offset mod 16"""
    d = os.path.join(GOLD, "bgzf_regress")
    raws = [np.load(os.path.join(d, f)).tobytes()[18:-8] for f in sorted(os.listdir(d))]
    assert len(raws) == 2 and not _check(ctx, raws, range(16))
