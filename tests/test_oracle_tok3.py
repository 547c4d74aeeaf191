"""Pins the tok3 oracle (oracle/orc_tok3.c) on the reference's own fixtures
(htscodecs/tests/names/tok3/*, driven by tests/tok3.test) and against the compiled reference."""
import glob
import os
import random

import pytest

import _libs as L

TOK3 = sorted(glob.glob(os.path.join(L.GOLD, "htscodecs", "names", "tok3", "*")))


def _plain(path):
    base = os.path.basename(path).rsplit(".", 1)[0]            # 01.names.3 -> 01.names
    return open(os.path.join(L.GOLD, "htscodecs", "names", base), "rb").read().replace(b"\n", b"\0")


@pytest.mark.parametrize("path", TOK3, ids=[os.path.basename(p) for p in TOK3])
def test_golden(path):
    comp = open(path, "rb").read()
    got = L.orc_tok3_decode(comp)
    assert got is not None
    assert got == _plain(path)


def _names(rng, n, style):
    out = []
    x, y, tile = 1000, 2000, 1101
    for i in range(n):
        if style == 0:                                          # Illumina-like
            x += rng.randrange(0, 40); y = rng.randrange(1000, 99999)
            if rng.random() < 0.02: tile += 1
            nm = "A00123:45:HXXXXDSXX:%d:%d:%d:%d" % (1 + i * 4 // max(n, 1), tile, x, y)
        elif style == 1:                                        # leading zeros, dups
            nm = "read_%06d/%d" % (i // 2, 1 + (i & 1)) if rng.random() > 0.1 else (out[-1] if out else "r0")
        else:                                                   # ragged free text
            nm = "".join(rng.choice("abcXYZ019_.:/") for _ in range(rng.randrange(1, 40)))
        out.append(nm)
    return ("\0".join(out) + "\0").encode()


@pytest.mark.parametrize("style", [0, 1, 2])
@pytest.mark.parametrize("level,arith", [(1, 0), (3, 0), (7, 0), (9, 0), (1, 1), (3, 1)])  # level >= 5 with arith wants bzip2 (X_EXT), not compiled into oracle/_ref
def test_vs_reference_seeded(style, level, arith):
    rng = random.Random(100 * style + level + arith)
    blob = _names(rng, rng.choice([1, 2, 37, 600]), style)
    comp = L.ref_tok3_encode(blob, level, arith)
    want = L.ref_tok3_decode(comp)
    assert want == blob
    assert L.orc_tok3_decode(comp) == want


def test_corrupt_agrees_with_reference():
    rng = random.Random(7)
    blob = _names(rng, 200, 0)
    comp = bytearray(L.ref_tok3_encode(blob, 5, 0))
    checked = 0
    for trial in range(150):
        c = bytearray(comp)
        if trial % 3 == 0:
            c = c[: rng.randrange(9, len(c))]
        else:
            for _ in range(rng.randrange(1, 3)):
                c[rng.randrange(8 if trial % 3 == 1 else 0, len(c))] = rng.randrange(256)
        n_reads = int.from_bytes(c[4:8], "little")
        u_len = int.from_bytes(c[0:4], "little")
        if n_reads > 100000 or u_len > 1 << 24:
            continue                                            # keep allocations small
        want = L.ref_tok3_decode(bytes(c))
        got = L.orc_tok3_decode(bytes(c))
        # a failed decode is a failure in both; a success must be byte-identical
        assert (want is None) == (got is None), trial
        if want is not None:
            assert got == want, trial
        checked += 1
    assert checked > 50
