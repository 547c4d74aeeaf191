"""GPU parity of the batching seams a patched htslib calls (INTEGRATION.md B3): hgpu_bgzf_inflate_blocks_host and
hgpu_bgzf_inflate_jobs_host with ragged slots, zero-length blocks in mid-batch and errors in order; untrusted CRAM
size fields; two contexts in one process (per-device function attributes).  bgzf.c:1010-1093, :1373-1384,
:1598-1738; cram/cram_io.c:1576-1754."""
import ctypes as C
import os
import random
import zlib
import numpy as np
import pytest
import htslib_b200 as H
from _libs import GOLD, BGZF_EOF, bgzf_block, orc_bgzf_inflate_block

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    c = H.Context(0)
    yield c
    c.close()


def _mixed_blocks():
    rng = random.Random(11)
    pay = [bytes(rng.choice(b"ACGT\n0123456789=") for _ in range(n)) for n in (65280, 1, 0, 4097, 31000, 0, 300, 65280)]
    blocks = [bgzf_block(p, lv) for p, lv in zip(pay, (6, 1, 6, 0, 9, 0, 6, 2))]
    # a corrupted payload byte (CRC error), a corrupted header, a truncated stream, then good blocks again: errors keep their slots
    bad_crc = bytearray(bgzf_block(pay[4], 6)); bad_crc[40] ^= 0x10
    bad_hdr = bytearray(bgzf_block(pay[6], 6)); bad_hdr[12] = ord("X")
    blocks += [bytes(bad_crc), BGZF_EOF, bytes(bad_hdr), bgzf_block(pay[1], 6)]
    return blocks


def _want(blocks):
    out = []
    for b in blocks:                                         # the oracle (== zlib + htslib's checks): (length or error code, payload)
        rc, data = orc_bgzf_inflate_block(b)
        out.append((0, data) if rc >= 0 else (rc, b""))
    return out


def test_blocks_host_ragged_slots_and_error_order(ctx):
    blocks = _mixed_blocks()
    n = len(blocks)
    in_len = np.array([len(b) for b in blocks], dtype=np.uint32)
    gaps = [(i * 7) % 13 for i in range(n)]                              # blocks are not back to back
    in_off = np.zeros(n, dtype=np.uint64)
    p = 3
    for i in range(n):
        in_off[i] = p; p += len(blocks[i]) + gaps[i]
    blob = np.zeros(p + 8, dtype=np.uint8)
    for i, b in enumerate(blocks):
        blob[int(in_off[i]):int(in_off[i]) + len(b)] = np.frombuffer(b, dtype=np.uint8)
    # ragged output slots, in a different order than the inputs, each with exactly 64 KiB of room (what a bgzf_job has)
    order = list(range(n)); random.Random(5).shuffle(order)
    out_off = np.zeros(n, dtype=np.uint64)
    q = 5
    for i in order:
        out_off[i] = q; q += 65536 + (i % 3)
    out = np.full(q + 8, 0xAA, dtype=np.uint8)
    cap = np.full(n, 65536, dtype=np.uint32)
    got = np.zeros(n, dtype=np.uint32); st = np.full(n, 77, dtype=np.int32)
    L = H.lib()
    rc = L.hgpu_bgzf_inflate_blocks_host(ctx.h, blob.ctypes.data, in_off.ctypes.data, in_len.ctypes.data, n, out.ctypes.data,
                                         out_off.ctypes.data, cap.ctypes.data, got.ctypes.data, st.ctypes.data)
    assert rc == 0, H.last_error()
    for i, (wst, wdata) in enumerate(_want(blocks)):
        assert int(st[i]) == wst, (i, int(st[i]), wst)
        if wst == 0:
            assert int(got[i]) == len(wdata) and out[int(out_off[i]):int(out_off[i]) + len(wdata)].tobytes() == wdata, i
        else:
            assert int(got[i]) == 0
    # nothing was written outside the slots
    mask = np.ones(out.size, dtype=bool)
    for i in range(n):
        mask[int(out_off[i]):int(out_off[i]) + 65536] = False
    assert (out[mask] == 0xAA).all()


def test_jobs_host_like_bgzf_mt_reader(ctx):
    """every block with its own malloc'd comp / uncomp buffers, as bgzf_job has them (bgzf.c:92-101)"""
    blocks = _mixed_blocks() * 3
    n = len(blocks)
    comp = [np.frombuffer(b, dtype=np.uint8).copy() for b in blocks]
    unc = [np.zeros(65536, dtype=np.uint8) for _ in range(n)]
    cp = (C.c_void_p * n)(*[c.ctypes.data for c in comp])
    up = (C.c_void_p * n)(*[u.ctypes.data for u in unc])
    clen = np.array([len(b) for b in blocks], dtype=np.uint32)
    ulen = np.full(n, 65536, dtype=np.uint32)
    st = np.full(n, 77, dtype=np.int32)
    L = H.lib()
    L.hgpu_bgzf_inflate_jobs_host.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    for h in (ctx.h, None):                                              # an explicit context, then the shims' process-wide one
        ulen[:] = 65536; st[:] = 77
        rc = L.hgpu_bgzf_inflate_jobs_host(h, n, cp, clen.ctypes.data, up, ulen.ctypes.data, st.ctypes.data)
        assert rc == 0, H.last_error()
        for i, (wst, wdata) in enumerate(_want(blocks)):
            assert int(st[i]) == wst, i
            if wst == 0:
                assert int(ulen[i]) == len(wdata) and unc[i][:len(wdata)].tobytes() == wdata, i


def test_cram_blocks_with_absurd_size_fields(ctx):
    """size fields are untrusted: a block that claims gigabytes fails on its own, the rest of the file still decodes"""
    cram = np.fromfile(os.path.join(GOLD, "htslib", "ce#1000.v31.cram"), dtype=np.uint8)
    blocks, _ = H.cram_scan_blocks(cram)
    _, base = H.cram_uncompress_blocks(ctx, cram, blocks)
    ok = [i for i, (st, _) in enumerate(base) if st == 0 and int(blocks["method"][i]) in (5, 8) and int(blocks["uncomp_size"][i]) > 64]
    assert len(ok) >= 4
    bad = blocks.copy()
    victims = {ok[0]: 0x7ffffff0, ok[1]: 0x50000000, ok[-1]: 3 << 24}       # over the limit, huge, and a 'big' block that is launched alone
    sizes = bad["uncomp_size"].astype(np.uint64)
    for i, v in victims.items():
        sizes[i] = v
    # lay the output out by the ORIGINAL sizes (the caller's buffer is what it is); only the block table lies
    n = len(bad)
    out_off = np.concatenate([[0], np.cumsum((blocks["uncomp_size"].astype(np.uint64) + 15) // 16 * 16)[:-1]]).astype(np.uint64)
    out = np.zeros(int(out_off[-1]) + int(blocks["uncomp_size"][-1]) + (4 << 24), dtype=np.uint8)
    for i, v in victims.items():
        bad["uncomp_size"][i] = v
    got = np.zeros(n, dtype=np.uint32); st = np.zeros(n, dtype=np.int32)
    L = H.lib()
    L.hgpu_cram_uncompress_blocks_host.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint32, C.c_void_p,
                                                   C.c_void_p, C.c_void_p, C.c_void_p]
    # the lying blocks get their own slots at the end so that a decoder writing 'uncomp_size' bytes stays inside the buffer
    tail = int(out_off[-1]) + int(blocks["uncomp_size"][-1]) + 64
    for i in victims:
        out_off[i] = tail
    barr = np.ascontiguousarray(bad)
    rc = L.hgpu_cram_uncompress_blocks_host(ctx.h, cram.ctypes.data, cram.size, barr.ctypes.data, n, out.ctypes.data,
                                            out_off.ctypes.data, got.ctypes.data, st.ctypes.data)
    assert rc == 0, (rc, H.last_error())
    for i in range(n):
        if i in victims:
            assert int(st[i]) != 0 and int(got[i]) == 0, i              # usize != usize2 -> -1 in the reference (cram_io.c:1709)
        else:
            assert int(st[i]) == base[i][0], i
            if base[i][0] == 0:
                assert out[int(out_off[i]):int(out_off[i]) + int(got[i])].tobytes() == base[i][1], i


def test_two_contexts_in_one_process():
    """function attributes (dynamic shared memory) are per device: a second context on another device must launch too"""
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("one GPU visible")
    rng = random.Random(2)
    p = bytes(rng.choice(b"ACGT") for _ in range(60000))
    img = np.frombuffer(bgzf_block(p, 6) + BGZF_EOF, dtype=np.uint8).copy()
    for dev in (0, 1, 0):
        c = H.Context(dev)
        out = np.zeros(len(p) + 16, dtype=np.uint8)
        rc, n, bad = c.bgzf_inflate_file_host(img, out)
        assert rc == 0 and n == len(p) and out[:n].tobytes() == p, (dev, rc, H.last_error())
        c.close()


def test_cram_write_blocks_reproduce_every_fixture_block(ctx):
    """cram_write_block (cram_io.c:1511-1563) for a batch: rebuilt from (method, content type, content id, sizes, payload),
    every block of every CRAM fixture — reference-written and htsjdk-written — comes out byte for byte, CRC included"""
    import glob
    L = H.lib()
    L.hgpu_cram_write_blocks_host.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p]
    total_blocks = 0
    for path in sorted(glob.glob(os.path.join(GOLD, "htslib", "*.cram"))):
        img = np.fromfile(path, dtype=np.uint8)
        blocks, ver = H.cram_scan_blocks(img)
        n = len(blocks)
        base = img.ctypes.data
        ptrs = (C.c_void_p * n)(*[base + int(b["data_off"]) for b in blocks])
        barr = np.ascontiguousarray(blocks)
        need = C.c_uint64(0)
        rc = L.hgpu_cram_write_blocks_host(ctx.h, barr.ctypes.data, ptrs, n, None, 0, None, C.byref(need))
        assert rc == -103 and need.value > 0                              # HGPU_ERR_NOMEM: the size to come back with
        out = np.zeros(need.value, dtype=np.uint8)
        off = np.zeros(n, dtype=np.uint64)
        got = C.c_uint64(0)
        rc = L.hgpu_cram_write_blocks_host(ctx.h, barr.ctypes.data, ptrs, n, out.ctypes.data, out.size, off.ctypes.data, C.byref(got))
        assert rc == 0, H.last_error()
        for i, b in enumerate(blocks):
            lo = int(b["data_off"]) - int(b["hdr_len"]); hi = int(b["data_off"]) + int(b["comp_size"]) + 4
            end = int(off[i + 1]) if i + 1 < n else got.value
            assert out[int(off[i]):end].tobytes() == img[lo:hi].tobytes(), (os.path.basename(path), i)
        total_blocks += n
    assert total_blocks > 100


def test_cram_gzip_blocks_of_any_size(ctx):
    """cram_uncompress_block's GZIP arm (zlib_mem_inflate, cram_io.c:1068-1157, :1600-1616): whole gzip members larger than a
    BGZF block, with optional header fields, several deflate blocks, stored blocks — and a corrupted one"""
    import gzip as gz
    rng = random.Random(21)
    names = b"".join(b"@HS25_%05d:%d:%d:%d:%d#%d\n" % (rng.randrange(99999), rng.randrange(8), 1100 + rng.randrange(1200), rng.randrange(20000), rng.randrange(200000), rng.randrange(96)) for _ in range(9000))
    pays = [names,                                                         # 300+ KB of read names: several dynamic blocks
            bytes(rng.randrange(256) for _ in range(200000)),              # incompressible: stored blocks
            b"ACGT" * 50000,                                               # long runs: overlapping matches
            b"x"]
    def member(p, level, extra=False):
        c = zlib.compressobj(level, zlib.DEFLATED, -15, 9)
        raw = c.compress(p) + c.flush()
        hdr = bytes([0x1f, 0x8b, 8, 0x18 if extra else 0, 0, 0, 0, 0, 0, 3]) + (b"name.txt\0a comment\0" if extra else b"")
        return hdr + raw + struct.pack("<II", zlib.crc32(p), len(p) & 0xffffffff)
    import struct
    comps = [member(pays[0], 6), member(pays[1], 6, True), member(pays[2], 9), member(pays[3], 1), member(pays[0], 1, True)]
    want = [pays[0], pays[1], pays[2], pays[3], pays[0]]
    bad = bytearray(comps[0]); bad[len(bad) // 2] ^= 0x40
    comps.append(bytes(bad)); want.append(None)
    n = len(comps)
    dt = np.dtype([("data_off", "<u8"), ("comp_size", "<u4"), ("uncomp_size", "<u4"), ("content_id", "<i4"), ("method", "u1"),
                   ("content_type", "u1"), ("hdr_len", "<u2"), ("container", "<u4"), ("pad2", "<u4")])     # hgpu_cram_block: 32 bytes
    assert dt.itemsize == 32
    blocks = np.zeros(n, dtype=dt)
    for i, (c, w) in enumerate(zip(comps, want)):
        blocks[i]["method"] = 1; blocks[i]["content_type"] = 4; blocks[i]["content_id"] = 10 + i
        blocks[i]["comp_size"] = len(c); blocks[i]["uncomp_size"] = len(w if w is not None else pays[0])
    L = H.lib()
    L.hgpu_cram_write_blocks_host.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p]
    bufs = [np.frombuffer(c, dtype=np.uint8).copy() for c in comps]
    ptrs = (C.c_void_p * n)(*[b.ctypes.data for b in bufs])
    img = np.zeros(sum(len(c) for c in comps) + 32 * n, dtype=np.uint8)
    off = np.zeros(n, dtype=np.uint64); tot = C.c_uint64(0)
    assert L.hgpu_cram_write_blocks_host(ctx.h, blocks.ctypes.data, ptrs, n, img.ctypes.data, img.size, off.ctypes.data, C.byref(tot)) == 0
    img = img[:tot.value].copy()
    scanned = blocks.copy()
    for i in range(n):                                                  # where the payloads sit in the image we just wrote
        hl = 2 + sum(1 if v < 0x80 else 2 if v < 0x4000 else 3 if v < 0x200000 else 4 if v < 0x10000000 else 5
                     for v in (10 + i, len(comps[i]), int(blocks[i]["uncomp_size"])))
        scanned[i]["hdr_len"] = hl; scanned[i]["data_off"] = int(off[i]) + hl
    _, res = H.cram_uncompress_blocks(ctx, img, scanned)
    for i, ((st, data), w) in enumerate(zip(res, want)):
        if w is None:
            assert st != 0, i                                           # corrupt: an error or "left to the host", never wrong bytes
        else:
            assert st == 0 and data == w, (i, st, len(data))
