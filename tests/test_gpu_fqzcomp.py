"""GPU parity: fqzcomp quality decode (CRAM 3.1 block method 7).  Checked against the reference's golden
streams (htscodecs/tests/dat/fqzcomp/*: the decode must equal column 1 of dat/q*, minus 33, as
tests/fqzcomp.test does) and against the compiled reference (oracle/_ref) on seeded inputs for every
strategy, with duplicates, reversed records, variable lengths and corrupted streams; oracle/orc_fqz.c is
pinned on the same fixtures in tests/test_oracle_fqz.py."""
import glob
import os
import random

import numpy as np
import pytest

import htslib_b200 as H
import _libs as L

pytestmark = pytest.mark.gpu
FQZ = sorted(glob.glob(os.path.join(L.GOLD, "htscodecs", "dat", "fqzcomp", "*")))


@pytest.fixture(scope="module")
def ctx():
    c = H.Context(0)
    yield c
    c.close()


def _column1(name):
    rows = open(os.path.join(L.GOLD, "htscodecs", "dat", name), "rb").read().split(b"\n")
    rows = [r.split(b"\t")[0] for r in rows if r]
    return b"".join(bytes(c - 33 for c in r) for r in rows)


def test_golden_streams(ctx):
    comps = [open(p, "rb").read() for p in FQZ]
    wants = [_column1(os.path.basename(p).rsplit(".", 1)[0]) for p in FQZ]
    assert len(comps) == 16
    res = H.fqz_decode(ctx, comps, [len(w) for w in wants])
    for p, (st, data), w in zip(FQZ, res, wants):
        assert st == 0, os.path.basename(p)
        assert data == w, os.path.basename(p)


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
            q = recs[-1]                                       # duplicate of the previous record
        recs.append(q); lens.append(l); flags.append(rng.choice((0, 16, 128, 144)))
    return b"".join(recs), lens, flags


def test_seeded_all_strategies_and_corrupt(ctx):
    rng = random.Random(11)
    comps, wants = [], []
    for kind in ("q4", "q40", "var"):
        for strat in (0, 1, 2, 3):
            for n_rec in (1, 7, 300):
                q, lens, flags = _quals(rng, n_rec, kind)
                with L.sampled():                                  # the last case is the base of the corrupt streams below
                    c = L.ref_fqz_compress(q, lens, flags, strat, store_always=(kind, strat, n_rec) == ("var", 3, 300))
                    w = L.ref_fqz_decompress(c)
                    assert w == q
                    comps.append(c); wants.append(w)
    res = H.fqz_decode(ctx, comps, [len(w) for w in wants])
    for i, ((st, data), w) in enumerate(zip(res, wants)):
        assert st == 0 and data == w, i
    base = comps[-1]
    bad = []
    for _ in range(60):
        c = bytearray(base); c[rng.randrange(1, len(c))] ^= 1 << rng.randrange(8); bad.append(bytes(c))
    bad.append(base[: len(base) // 2])
    res = H.fqz_decode(ctx, bad, [len(wants[-1]) + 64] * len(bad))
    cap = len(wants[-1]) + 64
    for c, (st, data) in zip(bad, res):
        w = L.ref_fqz_decompress(c)
        if w is None:
            assert st != 0
        elif len(w) <= cap:                                    # a larger size field does not fit the slot given here
            assert st == 0 and data == w
