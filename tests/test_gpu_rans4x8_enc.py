"""GPU parity: rANS 4x8 ENCODER (CRAM 3.0 method 4).  Deterministic, so the bar is byte equality with the
reference's rans_compress (oracle/_ref) on seeded inputs for both orders, all tail lengths and the
normalisation corner cases (one symbol, near-uniform 256 symbols, tiny inputs); every stream must also
decode back with the oracle's decoder."""
import random

import pytest

import htslib_b200 as H
from _libs import ref, ref_rans_4x8, orc_rans_4x8_decode, ref_rans_4x8_encoded
from test_oracle_rans import _synth

pytestmark = [pytest.mark.gpu]


def test_bytes_equal_reference_encoder():
    ctx = H.Context(0)
    rng = random.Random(9)
    raws, orders = [], []
    for order in (0, 1):
        for kind in ("q4", "q40", "runs", "one", "u32", "rand"):
            for n in (0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 31, 100, 1001, 4099, 30002, 300003):
                raws.append(_synth(rng, n, kind)); orders.append(order)
    got = H.rans4x8_encode(ctx, raws, orders)
    for raw, order, g in zip(raws, orders, got):
        want = ref_rans_4x8_encoded(raw, order)
        assert g is not None, (order, len(raw))
        assert g == want, (order, len(raw), g[:16].hex(), want[:16].hex())
        if raw:
            assert orc_rans_4x8_decode(g, len(raw)) == raw
    ctx.close()
