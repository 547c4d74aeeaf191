"""Pins the oracle's inflate / CRC32 / BGZF block logic against zlib itself (the library the
reference's bgzf_uncompress calls, bgzf.c:762-804), against the reference's BGZF fixtures and
against the compiled reference's bgzf_read (single- and multi-threaded)."""
import glob, os, random, zlib
import pytest
from _libs import (GOLD, BGZF_EOF, bgzf_block, bgzf_file, orc, orc_inflate_raw, orc_bgzf_inflate_block,
                   orc_bgzf_scan, ref, ref_bgzf_read_all, buf)
import ctypes as C


def payloads(rng):
    yield b""
    yield b"a"
    yield b"hello, hello, hello, hello\n" * 50
    yield bytes(rng.randrange(256) for _ in range(20000))                  # incompressible
    yield bytes(rng.choice(b"ACGT") for _ in range(65280))                 # 2-bit entropy
    yield b"\0" * 65280                                                      # long matches (len 258)
    yield bytes((i * 7 + (i >> 5)) & 0xff for i in range(65280))
    txt = b"".join(b"read%d\t%d\tchr%d\t%d\t60\t150M\t=\t%d\n" % (i, rng.randrange(4096), rng.randrange(24), rng.randrange(1 << 28), rng.randrange(1 << 28)) for i in range(1200))
    yield txt[:65280]


@pytest.mark.parametrize("level", [0, 1, 2, 4, 6, 9])
def test_inflate_vs_zlib(level):
    rng = random.Random(level)
    for p in payloads(rng):
        c = zlib.compressobj(level, zlib.DEFLATED, -15, 8)
        raw = c.compress(p) + c.flush()
        got, used = orc_inflate_raw(raw + b"\x01\x02\x03\x04\x05\x06\x07\x08", 65536)
        assert got == p
        assert used == len(raw)


def test_inflate_fixed_and_multiblock():
    rng = random.Random(3)
    p = bytes(rng.choice(b"abcdefgh ") for _ in range(30000))
    # Z_FIXED strategy -> BTYPE=1 ; Z_FULL_FLUSH every 1000 bytes -> many deflate blocks incl. stored empties
    c = zlib.compressobj(6, zlib.DEFLATED, -15, 8, zlib.Z_FIXED)
    raw = c.compress(p) + c.flush()
    assert orc_inflate_raw(raw)[0] == p
    c = zlib.compressobj(6, zlib.DEFLATED, -15, 8)
    raw = b""
    for i in range(0, len(p), 1000):
        raw += c.compress(p[i:i + 1000]) + c.flush(zlib.Z_FULL_FLUSH)
    raw += c.flush()
    assert orc_inflate_raw(raw)[0] == p


def test_inflate_errors_match_zlib():
    """Bit-flip fuzz: the oracle must fail exactly when zlib's inflate(Z_FINISH) fails, and agree
    byte for byte when both succeed."""
    rng = random.Random(11)
    p = bytes(rng.choice(b"ACGTN\n") for _ in range(9000))
    c = zlib.compressobj(6, zlib.DEFLATED, -15, 8)
    raw = c.compress(p) + c.flush()
    both_ok = both_bad = 0
    for _ in range(600):
        d = bytearray(raw)
        k = rng.randrange(len(d)); d[k] ^= 1 << rng.randrange(8)
        z = zlib.decompressobj(-15)
        try:
            want = z.decompress(bytes(d), 65536)
            ok = z.eof and not z.unconsumed_tail
        except zlib.error:
            ok = False
        got, _ = orc_inflate_raw(bytes(d))
        if ok:
            assert got == want; both_ok += 1
        else:
            assert got is None; both_bad += 1
    assert both_ok > 5 and both_bad > 100


def test_crc32_vs_zlib():
    rng = random.Random(5)
    o = orc(); o.orc_crc32.restype = C.c_uint32
    for n in (0, 1, 2, 3, 7, 8, 9, 255, 256, 4097, 65536):
        b = bytes(rng.randrange(256) for _ in range(n))
        assert o.orc_crc32(C.c_uint32(0), buf(b), C.c_uint64(n)) == zlib.crc32(b)


def test_block_status_codes():
    p = b"the quick brown fox " * 100
    blk = bgzf_block(p)
    assert orc_bgzf_inflate_block(blk) == (len(p), p)
    bad = bytearray(blk); bad[-8] ^= 1                         # CRC field
    assert orc_bgzf_inflate_block(bytes(bad))[0] == -2
    bad = bytearray(blk); bad[30] ^= 0x55                      # deflate payload
    assert orc_bgzf_inflate_block(bytes(bad))[0] in (-1, -2)
    bad = bytearray(blk); bad[12] = ord("X")                   # not BC
    assert orc_bgzf_inflate_block(bytes(bad))[0] == -3
    assert orc_bgzf_inflate_block(BGZF_EOF) == (0, b"")


def test_fixture_bgziptest():
    gz = open(os.path.join(GOLD, "htslib", "bgziptest.txt.gz"), "rb").read()
    txt = open(os.path.join(GOLD, "htslib", "bgziptest.txt"), "rb").read()
    n, blocks = orc_bgzf_scan(gz)
    assert n == len(blocks) and n >= 2
    out = b"".join(orc_bgzf_inflate_block(gz[o:o + l])[1] for o, l in blocks)
    assert out == txt
    assert gz[blocks[-1][0]:] == BGZF_EOF


@pytest.mark.parametrize("path", sorted(glob.glob(os.path.join(GOLD, "htslib", "bgzf_boundaries", "*.bam"))) +
                         [os.path.join(GOLD, "htslib", "range.bam"), os.path.join(GOLD, "htslib", "colons.bam")],
                         ids=os.path.basename)
def test_fixture_bams_vs_zlib_and_reference(path):
    data = open(path, "rb").read()
    n, blocks = orc_bgzf_scan(data)
    assert n > 0
    mine = b"".join(orc_bgzf_inflate_block(data[o:o + l])[1] for o, l in blocks)
    z = b""
    for o, l in blocks:
        z += zlib.decompress(data[o + 18:o + l - 8], -15)
    assert mine == z
    for t in (0, 3):
        got, err = ref_bgzf_read_all(data, t)
        assert err == 0 and got == mine


def test_synthetic_file_vs_reference_reader():
    rng = random.Random(9)
    data = bytes(rng.choice(b"ACGTACGTNN\t\n0123") for _ in range(400000))
    for level in (0, 1, 6):
        img = bgzf_file(data, level)
        n, blocks = orc_bgzf_scan(img)
        mine = b"".join(orc_bgzf_inflate_block(img[o:o + l])[1] for o, l in blocks)
        got, err = ref_bgzf_read_all(img, 2)
        assert err == 0 and got == mine == data


def test_scan_errors():
    img = bgzf_file(b"x" * 1000)
    assert orc_bgzf_scan(img[:-5])[0] == -2          # second block (EOF marker) truncated
    bad = bytearray(img); bad[0] = 0
    assert orc_bgzf_scan(bytes(bad))[0] == -1
