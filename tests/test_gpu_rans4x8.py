"""GPU parity: rANS 4x8 (CRAM 3.0) decode against the oracle (pinned to the golden r4x8 streams and
the compiled reference): golden files, the RANS blocks of a reference-written CRAM 3.0 file, seeded
streams from the reference encoder, and bit-flipped streams."""
import glob, os, random
import numpy as np
import pytest
import htslib_b200 as H
from _libs import GOLD, golden_raw, orc_rans_4x8_decode, ref, ref_rans_4x8, sampled
from test_oracle_rans import _synth

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    c = H.Context(0)
    yield c
    c.close()


def test_golden_and_cram30_blocks(ctx):
    comps, wants = [], []
    for path in sorted(glob.glob(os.path.join(GOLD, "htscodecs", "dat", "r4x8", "*"))):
        comps.append(open(path, "rb").read()); wants.append(golden_raw(os.path.basename(path).rsplit(".", 1)[0]))
    img = np.fromfile(os.path.join(GOLD, "htslib", "ce#1000.v30.cram"), dtype=np.uint8)
    blocks, _ = H.cram_scan_blocks(img)
    for b in blocks[blocks["method"] == 4]:
        c = img[int(b["data_off"]):int(b["data_off"]) + int(b["comp_size"])].tobytes()
        comps.append(c); wants.append(orc_rans_4x8_decode(c, int(b["uncomp_size"])))
    res = ctx.rans4x8_decode(comps, [len(w) for w in wants])
    for (st, data), w in zip(res, wants):
        assert st == 0 and data == w


def test_seeded_and_corrupt(ctx):
    rng = random.Random(12)
    comps, wants = [], []
    for order in (0, 1):
        for kind in ("q4", "q40", "runs", "one", "u32", "rand"):
            for n in (1, 3, 4, 5, 31, 100, 1000, 4099, 70001):
                raw = _synth(rng, n, kind)
                with sampled():
                    comps.append(ref_rans_4x8(raw, order)); wants.append(raw)
    res = ctx.rans4x8_decode(comps, [len(w) for w in wants])
    for i, ((st, data), w) in enumerate(zip(res, wants)):
        assert st == 0 and data == w, i
    # damaged payload bytes: same bytes or same failure as the oracle
    base = ref_rans_4x8(_synth(rng, 6000, "q40"), 1, store_always=True)
    bad = []
    for _ in range(60):
        c = bytearray(base); k = rng.randrange(len(c) // 2, len(c)); c[k] ^= 1 << rng.randrange(8); bad.append(bytes(c))
    bad.append(base[:40]); bad.append(base[:-10])
    res = ctx.rans4x8_decode(bad, [6000] * len(bad))
    for c, (st, data) in zip(bad, res):
        w = orc_rans_4x8_decode(c, 6000)
        if w is None: assert st != 0
        else: assert st == 0 and data == w
