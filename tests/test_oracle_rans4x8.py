"""Pins the oracle's rANS 4x8 (CRAM 3.0) decoder: golden streams of htscodecs/tests/dat/r4x8, the
RANS blocks of a reference-written CRAM 3.0 file, and seeded agreement with the compiled reference."""
import glob, os, random
import numpy as np
import pytest
import htslib_b200 as H
from _libs import GOLD, golden_raw, orc_rans_4x8_decode, ref, ref_rans_4x8, sampled
from test_oracle_rans import _synth

R4X8 = sorted(glob.glob(os.path.join(GOLD, "htscodecs", "dat", "r4x8", "*")))


@pytest.mark.parametrize("path", R4X8, ids=[os.path.basename(p) for p in R4X8])
def test_golden_r4x8(path):
    raw = golden_raw(os.path.basename(path).rsplit(".", 1)[0])
    comp = open(path, "rb").read()
    # "-r": one naked stream per file (rans4x8.test:22-28); the 9-byte header carries both sizes
    ulen = int.from_bytes(comp[5:9], "little")
    out = orc_rans_4x8_decode(comp, ulen)
    assert out is not None
    if ref() is not None:
        assert ref_rans_4x8(comp=comp) == out
    assert bytes(out) == raw


def test_cram30_blocks():
    img = np.fromfile(os.path.join(GOLD, "htslib", "ce#1000.v30.cram"), dtype=np.uint8)
    blocks, ver = H.cram_scan_blocks(img)
    rb = blocks[blocks["method"] == 4]
    assert ver == (3, 0) and len(rb) == 9
    for b in rb:
        comp = img[int(b["data_off"]):int(b["data_off"]) + int(b["comp_size"])].tobytes()
        d = orc_rans_4x8_decode(comp, int(b["uncomp_size"]))
        assert d is not None and len(d) == int(b["uncomp_size"])
        if ref() is not None:
            assert ref_rans_4x8(comp=comp) == d


def test_seeded_vs_reference():
    rng = random.Random(8)
    for order in (0, 1):
        for kind in ("q4", "q40", "runs", "one", "u32", "rand"):
            for n in (1, 3, 4, 5, 31, 100, 1000, 4099, 70001):
                raw = _synth(rng, n, kind)
                with sampled():
                    comp = ref_rans_4x8(raw, order)
                    assert comp is not None
                    assert orc_rans_4x8_decode(comp, n) == raw, (order, kind, n)
