"""Pins the fqzcomp oracle (oracle/orc_fqz.c) on the reference's own fixtures (htscodecs/tests/dat/fqzcomp/*,
driven by tests/fqzcomp.test: the decode must equal column 1 of dat/q*, minus 33) and against the compiled
reference on seeded streams (all strategies, CRAM 3.0 reversed orientation, duplicates) and corrupted ones."""
import glob
import os
import random

import pytest

import _libs as L

FQZ = sorted(glob.glob(os.path.join(L.GOLD, "htscodecs", "dat", "fqzcomp", "*")))


def _column1(name):
    rows = open(os.path.join(L.GOLD, "htscodecs", "dat", name), "rb").read().split(b"\n")
    return b"".join(bytes(c - 33 for c in r.split(b"\t")[0]) for r in rows if r)


def _quals(rng, n_rec, kind):
    lens, recs, flags = [], [], []
    for i in range(n_rec):
        l = 151 if kind != "var" else rng.randrange(1, 400)
        if kind == "q4":
            q = bytes(rng.choice((2, 12, 23, 37)) if rng.random() < 0.1 else 37 for _ in range(l))
        elif kind == "q40":
            q = bytes(max(2, min(41, int(rng.gauss(36 - 10 * k / l, 4)))) for k in range(l))
        else:
            q = bytes(rng.randrange(0, 60) for _ in range(l))
        if recs and rng.random() < 0.1 and len(recs[-1]) == l:
            q = recs[-1]
        recs.append(q); lens.append(l); flags.append(rng.choice((0, 16, 128, 144)))
    return b"".join(recs), lens, flags


@pytest.mark.parametrize("path", FQZ, ids=[os.path.basename(p) for p in FQZ])
def test_golden(path):
    comp = open(path, "rb").read()
    assert L.orc_fqz_decode(comp) == _column1(os.path.basename(path).rsplit(".", 1)[0])


def test_vs_reference_seeded_and_corrupt():
    rng = random.Random(11)
    last = None
    for vers in (4, 3):                                         # 3: qualities stored in read orientation + reverse flag
        for kind in ("q4", "q40", "var"):
            for strat in (0, 1, 2, 3):
                for n_rec in (1, 7, 300):
                    q, lens, flags = _quals(rng, n_rec, kind)
                    last = (q, lens, flags, strat, vers)
                    with L.sampled():
                        c = L.ref_fqz_compress(q, lens, flags, strat, vers)
                        want = L.ref_fqz_decompress(c)
                        assert want is not None
                        assert L.orc_fqz_decode(c) == want, (vers, kind, strat, n_rec)
    last = L.ref_fqz_compress(*last, store_always=True)
    agree = 0
    for _ in range(150):
        c = bytearray(last); c[rng.randrange(2, len(c))] ^= 1 << rng.randrange(8)
        want = L.ref_fqz_decompress(bytes(c)); got = L.orc_fqz_decode(bytes(c))
        assert (want is None) == (got is None)
        if want is not None:
            assert got == want
        agree += 1
    assert agree == 150
