"""LZ77 match execution and the in-line CRC-32 of the inflate kernels, driven by DEFLATE streams with chosen tokens.

A small raw-DEFLATE writer (fixed-Huffman blocks with the tokens the test picks, stored blocks) places matches at
every alignment, length and distance, next to literals and to each other, at the edges of the output, and makes
members of the sizes the CRC cursor cares about.  The expected output is always zlib's inflate of the same stream."""
import ctypes as C
import random
import struct
import zlib
import numpy as np
import pytest
import htslib_b200 as H
from _libs import bgzf_block

LBASE = [3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195, 227, 258]
LXTRA = [0] * 8 + [1] * 4 + [2] * 4 + [3] * 4 + [4] * 4 + [5] * 4 + [0]
DBASE = [1, 2, 3, 4, 5, 7, 9, 13, 17, 25, 33, 49, 65, 97, 129, 193, 257, 385, 513, 769, 1025, 1537, 2049, 3073, 4097, 6145,
         8193, 12289, 16385, 24577]
DXTRA = [0, 0, 0, 0] + [k // 2 for k in range(2, 28)]


class Deflate:
    """LSB-first bit writer for raw DEFLATE.  Tokens: an int is a literal byte, (length, distance) is a match."""

    def __init__(self):
        self.v, self.n = 0, 0

    def bits(self, val, nb):
        self.v |= val << self.n
        self.n += nb

    def code(self, c, nb):                                  # Huffman codes go MSB first
        self.bits(int(format(c, "0%db" % nb)[::-1], 2), nb)

    def stored(self, data, final=False):
        assert len(data) < 65536
        self.bits(int(final), 1); self.bits(0, 2)
        self.n = (self.n + 7) // 8 * 8
        self.bits(len(data), 16); self.bits(len(data) ^ 0xffff, 16)
        for b in data:
            self.bits(b, 8)

    def fixed(self, tokens, final=False):
        self.bits(int(final), 1); self.bits(1, 2)
        for t in tokens:
            if isinstance(t, int):
                self.lit(t)
            else:
                ln, dist = t
                ls = max(i for i in range(29) if LBASE[i] <= ln)
                self.lit(257 + ls); self.bits(ln - LBASE[ls], LXTRA[ls])
                ds = max(i for i in range(30) if DBASE[i] <= dist)
                self.code(ds, 5); self.bits(dist - DBASE[ds], DXTRA[ds])
        self.lit(256)

    def lit(self, s):
        if s < 144: self.code(0x30 + s, 8)
        elif s < 256: self.code(0x190 + s - 144, 9)
        elif s < 280: self.code(s - 256, 7)
        else: self.code(0xc0 + s - 280, 8)

    def raw(self, tail=b""):                                # tail: byte-aligned blocks to append (zlib's own)
        return self.v.to_bytes((self.n + 7) // 8, "little") + tail


def expand(tokens, prefix=b""):
    out = bytearray(prefix)
    for t in tokens:
        if isinstance(t, int):
            out.append(t)
        else:
            for _ in range(t[0]):
                out.append(out[-t[1]])
    return bytes(out)


def random_tokens(rng, out_len, n, dists=None, gaps=(0, 0, 1, 2), lens=None):
    """n matches after out_len bytes of output: every length 3..258 and distance 1..32768 reachable, some overlapping"""
    toks, o = [], out_len
    for _ in range(n):
        for _ in range(rng.choice(gaps)):
            toks.append(rng.randrange(256)); o += 1
        ln = rng.choice(lens) if lens else rng.choice([3, 4, 5, 6, 7, 8, 9, 11, 15, 16, 17, 27, 31, 32, 33, 64, 100, 257, 258])
        dist = rng.choice(dists) if dists else rng.choice([1, 2, 3, 4, 5, 7, 8, ln, ln + 1, ln + 3, rng.randrange(ln, 300), rng.randrange(1, 32769)])
        dist = max(1, min(dist, o))
        toks.append((ln, dist)); o += ln
    return toks


def members(rng):
    """(name, raw deflate) for the cases above"""
    out = []
    # alignment x length x distance: a stored random prefix makes every distance up to 32768 reachable
    for seed in range(6):
        r = random.Random(seed)
        prefix = bytes(r.randrange(256) for _ in range(33000 + seed))
        d = Deflate(); d.stored(prefix); d.fixed(random_tokens(r, len(prefix), 120), final=True)
        out.append(("align%d" % seed, d.raw()))
    # 32 ready matches in one round: each copies from the prefix, none depends on another
    for shift in range(4):
        d = Deflate(); prefix = bytes(rng.randrange(256) for _ in range(5000 + shift))
        d.stored(prefix)
        d.fixed([(rng.randrange(3, 40), rng.randrange(2000, 4500)) for _ in range(32 * 8)], final=True)
        out.append(("wide%d" % shift, d.raw()))
    # matches meeting inside one word, and next to single literals; small blocks take the serial decoder
    for k in range(8):
        toks = [rng.randrange(256) for _ in range(24)]
        for j in range(40):
            toks.append((3 + (j + k) % 6, 1 + (j * 7 + k) % 16 + 8))
            if j % 3 == k % 3:
                toks.append(rng.randrange(256))
        d = Deflate(); d.fixed(toks[:26 + 4 * k], final=True)
        out.append(("serial%d" % k, d.raw()))
        d = Deflate(); d.fixed(toks, final=True)
        out.append(("words%d" % k, d.raw()))
    # overlapping matches, dist 1..8
    toks = [rng.randrange(256) for _ in range(8)]
    for dist in range(1, 9):
        for ln in (max(3, dist + 1), 9, 31, 32, 33, 258):
            toks += [(ln, dist), rng.randrange(256)]
    d = Deflate(); d.fixed(toks, final=True)
    out.append(("overlap", d.raw()))
    # the match's source is byte 0 of the output, and a match ends on the member's last byte
    for n0 in (3, 4, 5, 10, 64):
        toks = [rng.randrange(256) for _ in range(n0)] + [(n0, n0)] + [rng.randrange(256) for _ in range(20)] + [(min(258, n0 + 20), n0 + 20)]
        d = Deflate(); d.fixed(toks, final=True)
        out.append(("edge%d" % n0, d.raw()))
    # member sizes around the CRC rows: 0, 1, 127, 128, 129, 65536 bytes
    for size in (0, 1, 2, 3, 4, 5, 127, 128, 129, 255, 256, 257):
        toks = [rng.randrange(256) for _ in range(min(size, 5))]
        while len(expand(toks)) < size:
            toks.append((min(258, size - len(expand(toks))), 1) if size - len(expand(toks)) >= 3 else rng.randrange(256))
        d = Deflate(); d.fixed(toks, final=True)
        out.append(("size%d" % size, d.raw()))
    d = Deflate(); d.fixed([7] + [(258, 1)] * 254 + [(3, 1)], final=True)
    out.append(("size65536", d.raw()))
    # stored + fixed + dynamic blocks in one member
    text = b"".join(b"read_%05d\tchr1\t%d\t60\t150M\n" % (rng.randrange(99999), rng.randrange(10 ** 6)) for _ in range(600))
    c = zlib.compressobj(9, zlib.DEFLATED, -15)
    dyn = c.compress(text) + c.flush()
    assert (dyn[0] >> 1) & 3 == 2
    d = Deflate(); d.fixed(random_tokens(rng, 0, 0) + [1, 2, 3, (40, 3)]); d.stored(bytes(range(200)))
    out.append(("mixed", d.raw(dyn)))
    return out


def _bgzf(raw, data, flip=False):
    blk = bytearray(bgzf_block(data, raw_deflate=raw))
    if flip:
        blk[-8] ^= 0x01
    return bytes(blk)


def test_writer_streams_inflate_with_zlib():
    """the token writer itself: zlib inflates every stream to the tokens' own expansion"""
    rng = random.Random(5)
    toks = random_tokens(rng, 0, 0) + [rng.randrange(256) for _ in range(9)] + random_tokens(rng, 9, 400)
    d = Deflate(); d.fixed(toks, final=True)
    assert zlib.decompress(d.raw(), -15) == expand(toks)
    pre = bytes(range(256)) * 140
    d = Deflate(); d.stored(pre); d.fixed(random_tokens(rng, len(pre), 300, lens=list(range(3, 259))), final=True)
    assert len(zlib.decompress(d.raw(), -15)) > len(pre)
    for name, raw in members(random.Random(1)):
        data = zlib.decompress(raw, -15)
        assert len(data) <= 65536, name
        blk = _bgzf(raw, data)
        assert zlib.decompress(blk[18:-8], -15) == data, name


def _inflate(ctx, blocks, shifts, caps):
    """BGZF blocks into output slots at the given byte offsets (mod 16 they vary); the last slot ends the buffer"""
    import torch
    dev = torch.device("cuda:0")
    n = len(blocks)
    in_off = np.cumsum([0] + [len(b) + 3 for b in blocks[:-1]]).astype(np.uint64)
    blob = np.zeros(int(in_off[-1]) + len(blocks[-1]), dtype=np.uint8)
    for i, b in enumerate(blocks):
        blob[int(in_off[i]):int(in_off[i]) + len(b)] = np.frombuffer(b, dtype=np.uint8)
    out_off = np.array([i * 65552 + shifts[i] for i in range(n)], dtype=np.uint64)
    total = int(out_off[-1]) + caps[-1]
    t = lambda a: torch.from_numpy(a.view(np.int64) if a.dtype == np.uint64 else a.view(np.int32)).to(dev)
    d_in = torch.from_numpy(blob).to(dev)
    d_out = torch.full((total,), 0x55, dtype=torch.uint8, device=dev)
    d_len = torch.zeros(n, dtype=torch.int32, device=dev)
    d_st = torch.full((n,), 9, dtype=torch.int32, device=dev)
    ctx.bgzf_inflate_dev(d_in, t(in_off), t(np.array([len(b) for b in blocks], dtype=np.uint32)), d_out, t(out_off),
                         t(np.array(caps, dtype=np.uint32)), d_len, d_st, torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    out = d_out.cpu().numpy(); ln = d_len.cpu().numpy(); st = d_st.cpu().numpy()
    return [(int(st[i]), out[int(out_off[i]):int(out_off[i]) + int(ln[i])].tobytes()) for i in range(n)]


@pytest.fixture(scope="module")
def ctx():
    c = H.Context(0)
    yield c
    c.close()


@pytest.mark.gpu
@pytest.mark.parametrize("flip", [False, True])
def test_chosen_tokens_every_offset(ctx, flip):
    """every member at output offsets 0..15 mod 16, each slot exactly the member's size; a flipped CRC is BGZF_ERR_CRC"""
    ms = members(random.Random(1))
    blocks, want, shifts = [], [], []
    for name, raw in ms:
        data = zlib.decompress(raw, -15)
        for sh in range(16):
            blocks.append(_bgzf(raw, data, flip)); want.append(data); shifts.append(sh)
    res = _inflate(ctx, blocks, shifts, [len(w) for w in want])
    for i, ((st, data), w) in enumerate(zip(res, want)):
        tag = (ms[i // 16][0], shifts[i])
        if flip:
            assert st == H.BGZF_ERR_CRC, tag
        else:
            assert st == 0 and data == w, tag


@pytest.mark.gpu
def test_large_gzip_members(ctx):
    """gzip members of several hundred KiB (CRAM GZIP blocks) keep their CRC across many deflate blocks; a flipped CRC fails"""
    rng = random.Random(9)
    prefix = bytes(rng.randrange(256) for _ in range(40000))
    d = Deflate(); d.stored(prefix)
    for _ in range(12):
        d.fixed(random_tokens(rng, 40000, 900))
    d.stored(b"", final=True)
    raw_tok = d.raw()
    names = b"".join(b"@HS25_%05d:%d:%d\n" % (rng.randrange(99999), rng.randrange(8), rng.randrange(20000)) for _ in range(30000))
    raw_z = zlib.compress(names, 6)[2:-4]
    pays, comps = [], []
    for raw in (raw_tok, raw_z):
        data = zlib.decompress(raw, -15)
        assert len(data) > 300000
        for flip in (False, True):
            crc = zlib.crc32(data) ^ (1 if flip else 0)
            comps.append(bytes([0x1f, 0x8b, 8, 0, 0, 0, 0, 0, 0, 3]) + raw + struct.pack("<II", crc, len(data)))
            pays.append(None if flip else data)
    n = len(comps)
    dt = np.dtype([("data_off", "<u8"), ("comp_size", "<u4"), ("uncomp_size", "<u4"), ("content_id", "<i4"), ("method", "u1"),
                   ("content_type", "u1"), ("hdr_len", "<u2"), ("container", "<u4"), ("pad2", "<u4")])
    blocks = np.zeros(n, dtype=dt)
    for i, c in enumerate(comps):
        blocks[i]["method"] = 1; blocks[i]["content_type"] = 4; blocks[i]["content_id"] = 10 + i
        blocks[i]["comp_size"] = len(c); blocks[i]["uncomp_size"] = len(pays[i] if pays[i] is not None else pays[i - 1])
    L = H.lib()
    L.hgpu_cram_write_blocks_host.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p]
    bufs = [np.frombuffer(c, dtype=np.uint8).copy() for c in comps]
    ptrs = (C.c_void_p * n)(*[b.ctypes.data for b in bufs])
    img = np.zeros(sum(len(c) for c in comps) + 32 * n, dtype=np.uint8)
    off = np.zeros(n, dtype=np.uint64); tot = C.c_uint64(0)
    assert L.hgpu_cram_write_blocks_host(ctx.h, blocks.ctypes.data, ptrs, n, img.ctypes.data, img.size, off.ctypes.data, C.byref(tot)) == 0
    img = img[:tot.value].copy()
    scanned = blocks.copy()
    for i in range(n):
        hl = 2 + sum(1 if v < 0x80 else 2 if v < 0x4000 else 3 if v < 0x200000 else 4 if v < 0x10000000 else 5
                     for v in (10 + i, len(comps[i]), int(blocks[i]["uncomp_size"])))
        scanned[i]["hdr_len"] = hl; scanned[i]["data_off"] = int(off[i]) + hl
    _, res = H.cram_uncompress_blocks(ctx, img, scanned)
    for i, ((st, data), w) in enumerate(zip(res, pays)):
        if w is None:
            assert st != 0, i
        else:
            assert st == 0 and data == w, (i, st, len(data))
