"""GPU parity: arith_dynamic (CRAM 3.1 method 6) decode.  Checked against the reference's golden
streams (htscodecs/tests/dat/arith/*: the decode must equal the raw input, as arith.test does) and
against the compiled reference on seeded inputs for every format-byte combination; the checker here
is the unmodified reference itself (oracle/_ref); oracle/orc_arith.c is pinned on the same fixtures in
tests/test_oracle_arith.py."""
import glob, os, random
import pytest
import htslib_b200 as H
from _libs import GOLD, golden_raw, ref, ref_arith, sampled
from test_oracle_rans import _synth

pytestmark = pytest.mark.gpu
ARITH = sorted(glob.glob(os.path.join(GOLD, "htscodecs", "dat", "arith", "*")))


@pytest.fixture(scope="module")
def ctx():
    c = H.Context(0)
    yield c
    c.close()


def test_golden_streams(ctx):
    comps, wants, names = [], [], []
    for path in ARITH:
        name, order = os.path.basename(path).rsplit(".", 1)
        if int(order) & 4:
            continue                                   # X_EXT = bzip2 payload, not supported (nor by the reference here)
        comps.append(open(path, "rb").read()); wants.append(golden_raw(name)); names.append(os.path.basename(path))
    assert len(comps) >= 30
    res = ctx.arith_decode(comps, [len(w) for w in wants])
    for (st, data), w, nm in zip(res, wants, names):
        assert st == 0, nm
        assert data == w, nm


def test_seeded_all_orders_and_corrupt(ctx):
    rng = random.Random(77)
    comps, wants = [], []
    for order in (0, 1, 64, 65, 128, 129, 192, 193, 8, 9, 32):
        for kind in ("q4", "q40", "runs", "one", "u32", "rand"):
            for n in (1, 3, 32, 100, 1000, 4099, 30001):
                raw = _synth(rng, n, kind)
                with sampled():
                    comps.append(ref_arith(raw, order)); wants.append(raw)
    res = ctx.arith_decode(comps, [len(w) for w in wants])
    for i, ((st, data), w) in enumerate(zip(res, wants)):
        assert st == 0 and data == w, (i, comps[i][:4].hex(), len(w))
    base = ref_arith(_synth(rng, 5000, "q40"), 65, store_always=True)
    bad = []
    for _ in range(50):
        c = bytearray(base); k = rng.randrange(8, len(c)); c[k] ^= 1 << rng.randrange(8); bad.append(bytes(c))
    bad.append(base[: len(base) // 2])
    res = ctx.arith_decode(bad, [5000] * len(bad))
    for c, (st, data) in zip(bad, res):
        w = ref_arith(comp=c, cap=5000)
        if w is None: assert st != 0
        else: assert st == 0 and data == w
