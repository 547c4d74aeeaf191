"""Run-length (overlapping) LZ77 matches and the re-sync of the lane-parallel Huffman decoder.

Overlapping matches (dist < len) with dist <= 4 are built as whole words from their period inside the coalesced word
copy; longer periods go through a cooperative path.  Re-sync rounds stop where a lane meets the path it decoded in
round 0.  Streams come from the raw-DEFLATE writer of test_gpu_bgzf_lz77 (chosen tokens) and from zlib (dynamic
Huffman); the expected output is always zlib's inflate of the same stream, and a non-zero status or a wrong CRC fails."""
import os
import random
import struct
import zlib
import numpy as np
import pytest
import htslib_b200 as H
from _libs import GOLD
from test_gpu_bgzf_lz77 import Deflate, _bgzf, _inflate

LENS = (3, 4, 5, 31, 32, 33, 127, 258)
PAR_MIN_BITS = 32 * 96                      # member bits after the block header (footer included) that take the parallel decoder
PAR_MIN_BYTES = PAR_MIN_BITS // 8 + 16


def _run_tokens(rng, dists, lit_gap):
    """every (len, dist) pair behind 0..3 literals (destination offset mod 4); a 64-byte prefix holds every period"""
    toks = [rng.randrange(256) for _ in range(64)]
    for dist in dists:
        for ln in LENS:
            toks += [rng.randrange(256) for _ in range(lit_gap)]
            toks.append((ln, dist))
            lit_gap = (lit_gap + 1) % 4
    return toks


def _chain_tokens(rng):
    """back-to-back runs, each reading the previous record's last bytes, and runs whose period is the previous match"""
    toks = [rng.randrange(256) for _ in range(40)]
    toks += [(rng.choice(LENS), 1) for _ in range(40)]                        # dist 1 chained through one batch
    toks += [(rng.choice((5, 9, 33, 100)), d) for d in (2, 3, 4, 1, 3, 2, 4, 4, 1, 2)]
    for dist in (1, 2, 3, 4, 7, 32, 33, 40):
        toks += [rng.randrange(256), (40, 35)] + [(rng.choice((35, 64, 258)), dist)]   # period inside the previous match
    return toks


def _start_tokens(rng, n0, dist, ln):
    """a run at the member's start (dist == bytes so far)"""
    return [rng.randrange(256) for _ in range(n0)] + [(ln, dist)] + [rng.randrange(256) for _ in range(3)]


def _fixed(toks, pad_to_parallel=False, rng=None):
    d = Deflate()
    if pad_to_parallel:                     # a large block: literals behind make the body long enough to split
        toks = toks + [rng.randrange(144, 256) for _ in range(PAR_MIN_BYTES)]
    d.fixed(toks, final=True)
    return d.raw()


def _members():
    rng = random.Random(11)
    out = []
    # every period 1..40 x every length, 0..3 literals in front: large blocks (lane-parallel decoder)
    for g in range(4):
        dists = list(range(1 + 10 * g, 11 + 10 * g))
        for gap in range(4):
            out.append(("runs%d_%d" % (g, gap), _fixed(_run_tokens(rng, dists, gap) * 3, True, rng)))
    # the same pairs a few at a time in small members (uniform decoder), each ending on the member's last byte
    for dist in range(1, 41):
        for gap in range(4):
            toks = _run_tokens(rng, [dist], gap)[64 - max(8, dist):]
            out.append(("small_runs%d_%d" % (dist, gap), _fixed(toks)))
    for name, toks in [("chain", _chain_tokens(rng))] + [
            ("start%d_%d" % (n0, ln), _start_tokens(rng, n0, n0, ln)) for n0 in (1, 2, 3, 4, 5, 7, 32, 33) for ln in (3, 33, 258)]:
        out.append((name, _fixed(toks)))
        out.append((name + "_par", _fixed(toks, True, rng)))
    # a run that ends exactly at the slot's end, in both decoders
    end = [rng.randrange(256) for _ in range(9)] + [(258, 1), 7, (200, 3), 1, 2, (255, 4)]
    out.append(("end", _fixed(end)))
    out.append(("end_par", _fixed([rng.randrange(144, 256) for _ in range(PAR_MIN_BYTES)] + end)))
    return out


def test_run_members_inflate_with_zlib():
    """the streams themselves: every member is what the tests mean (decoder choice, length, zlib's expansion)"""
    for name, raw in _members():
        data = zlib.decompress(raw, -15)
        assert len(data) <= 65536, name
        big = (len(raw) + 8) * 8 - 3 >= PAR_MIN_BITS
        assert big == (name.startswith("runs") or name.endswith("_par")), (name, len(raw))


def _check(ctx, raws, shifts=range(4)):
    blocks, want, sh = [], [], []
    for raw in raws:
        data = zlib.decompress(raw, -15)
        for s in shifts:
            blocks.append(_bgzf(raw, data)); want.append(data); sh.append(s)
    res = _inflate(ctx, blocks, sh, [len(w) for w in want])
    return [(i, st, len(d), len(w)) for i, ((st, d), w) in enumerate(zip(res, want)) if st != 0 or d != w]


@pytest.fixture(scope="module")
def ctx():
    c = H.Context(0)
    yield c
    c.close()


@pytest.mark.gpu
def test_runs_every_period_length_and_offset(ctx):
    """periods 1..40, lengths 3..258, destination offsets mod 4, output slots at offsets 0..3 mod 16 (row edges move)"""
    ms = _members()
    bad = _check(ctx, [raw for _, raw in ms])
    assert not bad, [(ms[i // 4][0], st, got, want) for i, st, got, want in bad[:8]]


@pytest.mark.gpu
def test_runs_flipped_crc(ctx):
    """the CRC of run output is checked: a flipped footer CRC is BGZF_ERR_CRC"""
    ms = _members()[:8]
    blocks = [_bgzf(raw, zlib.decompress(raw, -15), flip=True) for _, raw in ms]
    res = _inflate(ctx, blocks, [0] * len(blocks), [65536] * len(blocks))
    assert [st for st, _ in res] == [H.BGZF_ERR_CRC] * len(blocks)


def _bam_payloads():
    import sys
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    from tools import synth
    out = []
    for quals in ("novaseq", "hiseq"):
        stream, _ = synth.bam_records(7, 900, quals=quals)
        out += [stream[i:i + 65280] for i in range(0, min(len(stream), 3 * 65280), 65280)]
    rng = random.Random(2)
    out.append(bytes(rng.randrange(256) for _ in range(65280)))                       # random: stored or near-stored
    out.append(bytes(rng.choice(b"ACGT") for _ in range(65280)))                       # low entropy
    out.append(bytes(rng.choice(b"AAAAAAAC#") for _ in range(65280)))
    out.append(b"\x2a" * 65280)                                                        # all one byte
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("level", [1, 6, 9])
def test_resync_dynamic_members(ctx, level):
    """zlib dynamic-Huffman members: synthetic BAM (NovaSeq, HiSeq), random, low-entropy and one-byte payloads"""
    raws = []
    for p in _bam_payloads():
        c = zlib.compressobj(level, zlib.DEFLATED, -15, 8)
        raws.append(c.compress(p) + c.flush())
    assert sum((r[0] >> 1) & 3 == 2 for r in raws) >= 6
    assert not _check(ctx, raws)


@pytest.mark.gpu
def test_resync_regress_blocks(ctx):
    """the blocks that once failed in the pre-roll, every output offset mod 16"""
    raws = [np.load(os.path.join(GOLD, "bgzf_regress", f)).tobytes()[18:-8] for f in sorted(os.listdir(os.path.join(GOLD, "bgzf_regress")))]
    assert raws and not _check(ctx, raws, range(16))


@pytest.mark.gpu
def test_resync_without_convergence(ctx):
    """long stretches of 9-bit fixed-code literals: a lane off the true grid needs many tokens to re-join it (or never
    does inside its range), so the re-sync decodes on past its checkpoints"""
    rng = random.Random(4)
    raws = []
    for n in (3000, 20000, 40000):
        toks = [rng.randrange(144, 256) for _ in range(n)]
        for k in range(1000, n, 5000):                              # a few runs and short codes in between
            toks[k:k] = [(rng.choice(LENS), rng.randrange(1, 5)), rng.randrange(0, 144)]
        raws.append(_fixed(toks))
    assert not _check(ctx, raws)


@pytest.mark.gpu
def test_gzip_multiblock_member(ctx):
    """gzip_inflate_kernel: one member of several deflate blocks (fixed runs, zlib dynamic blocks), CRC and ISIZE checked"""
    import ctypes as C
    rng = random.Random(8)
    d = Deflate()
    for g in range(4):
        d.fixed(_run_tokens(rng, range(1 + 10 * g, 11 + 10 * g), g))
    c = zlib.compressobj(6, zlib.DEFLATED, -15, 8)
    tail = b"".join(_bam_payloads()[:4])
    raw = d.raw(c.compress(tail) + c.flush())                       # zlib's blocks follow byte-aligned, the last is final
    data = zlib.decompress(raw, -15)
    assert len(data) > 200000
    comps, pays = [], []
    for flip in (False, True):
        crc = zlib.crc32(data) ^ (1 if flip else 0)
        comps.append(bytes([0x1f, 0x8b, 8, 0, 0, 0, 0, 0, 0, 3]) + raw + struct.pack("<II", crc, len(data)))
        pays.append(None if flip else data)
    n = len(comps)
    dt = np.dtype([("data_off", "<u8"), ("comp_size", "<u4"), ("uncomp_size", "<u4"), ("content_id", "<i4"), ("method", "u1"),
                   ("content_type", "u1"), ("hdr_len", "<u2"), ("container", "<u4"), ("pad2", "<u4")])
    blocks = np.zeros(n, dtype=dt)
    for i, cb in enumerate(comps):
        blocks[i]["method"] = 1; blocks[i]["content_type"] = 4; blocks[i]["content_id"] = 10 + i
        blocks[i]["comp_size"] = len(cb); blocks[i]["uncomp_size"] = len(data)
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
                     for v in (10 + i, len(comps[i]), len(data)))
        scanned[i]["hdr_len"] = hl; scanned[i]["data_off"] = int(off[i]) + hl
    _, res = H.cram_uncompress_blocks(ctx, img, scanned)
    assert res[0][0] == 0 and res[0][1] == data
    assert res[1][0] != 0
