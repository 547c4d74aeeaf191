"""GPU parity: adaptive arithmetic ENCODER.  The coder is deterministic, so the bar is byte equality with
the reference's arith_compress_to (oracle/_ref) for every flag combination it shares (order 0/1, RLE, PACK,
CAT, NOSZ) on seeded inputs, plus: the reference decodes every stream back to the input."""
import random

import pytest

import htslib_b200 as H
from _libs import ref, ref_arith, ref_arith_encoded
from test_oracle_rans import _synth

pytestmark = [pytest.mark.gpu]


def test_bytes_equal_reference_encoder():
    ctx = H.Context(0)
    rng = random.Random(5)
    raws, orders = [], []
    for order in (0, 1, 64, 65, 128, 129, 192, 193, 32, 16, 17, 80):
        for kind in ("q4", "q40", "runs", "one", "u32", "rand"):
            for n in (0, 1, 5, 9, 100, 4099, 30001):
                raws.append(_synth(rng, n, kind)); orders.append(order)
    got = H.arith_encode(ctx, raws, orders)
    diff = 0
    for raw, order, g in zip(raws, orders, got):
        want = ref_arith_encoded(raw, order)
        assert g is not None, (order, len(raw))
        if g != want:
            diff += 1
        assert g == want, (order, len(raw), g[:8].hex(), want[:8].hex())
        if not order & 16:                                      # NOSZ streams need the size from outside
            assert ref_arith(comp=g, cap=len(raw)) == raw
    # STRIPE is not produced: the flag is dropped, the stream still decodes with the reference
    raw = _synth(rng, 5000, "u32")
    g, = H.arith_encode(ctx, [raw], [8 | 1])
    assert g is not None and not g[0] & 8 and ref_arith(comp=g, cap=len(raw)) == raw
    ctx.close()
