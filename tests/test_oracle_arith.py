"""Pins the adaptive-arithmetic oracle (oracle/orc_arith.c) on the reference's own fixtures
(htscodecs/tests/dat/arith/*, driven by tests/arith.test: the decode must equal the raw input) and against
the compiled reference on seeded streams for every flag combination and on corrupted streams."""
import glob
import os
import random

import pytest

import _libs as L
from test_oracle_rans import _synth

ARITH = sorted(glob.glob(os.path.join(L.GOLD, "htscodecs", "dat", "arith", "*")))


@pytest.mark.parametrize("path", ARITH, ids=[os.path.basename(p) for p in ARITH])
def test_golden(path):
    name, order = os.path.basename(path).rsplit(".", 1)
    comp = open(path, "rb").read()
    raw = L.golden_raw(name)
    got = L.orc_arith_decode(comp, len(raw))
    if int(order) & 4:
        assert got is None                                     # X_EXT: bzip2 payload, an error without libbz2
    else:
        assert got == raw


def test_vs_reference_seeded_and_corrupt():
    rng = random.Random(77)
    base = None
    for order in (0, 1, 64, 65, 128, 129, 192, 193, 8, 9, 8 | 64, 32, 8 | (3 << 8)):
        for kind in ("q4", "q40", "runs", "one", "u32", "rand"):
            for n in (1, 3, 32, 100, 1000, 4099, 30001):
                raw = _synth(rng, n, kind)
                if order == 65 and kind == "q40" and n == 4099:
                    base = raw
                with L.sampled():
                    comp = L.ref_arith(raw, order)
                    assert L.ref_arith(comp=comp, cap=len(raw)) == raw
                    assert L.orc_arith_decode(comp, len(raw)) == raw, (order, kind, n)
    comp, cap = L.ref_arith(base, 65, store_always=True), len(base)
    for trial in range(200):
        c = bytearray(comp)
        if trial % 4 == 0: c = c[: rng.randrange(1, len(c))]
        else: c[rng.randrange(0, len(c))] ^= 1 << rng.randrange(8)
        want = L.ref_arith(comp=bytes(c), cap=cap)
        got = L.orc_arith_decode(bytes(c), cap)
        assert (want is None) == (got is None), trial
        if want is not None:
            assert got == want, trial
