"""GPU rANS Nx16 encoder (hgpu_rans_nx16_encode_batch_dev): its streams must be decoded to the
input by the unmodified reference decoder, by the oracle and by our own decoder (round trip);
size must stay within a stated ratio of the reference encoder's output."""
import random
import numpy as np
import pytest
import htslib_b200 as H
from _libs import orc_rans_nx16_decode, ref, ref_rans_nx16_decode, ref_rans_nx16_encode, ref_rans_nx16_encoded
from test_oracle_rans import _synth
from test_gpu_rans import run_batch

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    c = H.Context(0)
    yield c
    c.close()


STRIPE4 = 8 | (4 << 8)
ALL_ORDERS = [0, 1, 4, 5, 64, 65, 68, 69, 128, 129, 132, 133, 192, 193, 196, 197, 32,
              STRIPE4, STRIPE4 | 1, STRIPE4 | 193, 8 | (3 << 8) | 65, 8 | 1 | (1 << 16)]


@pytest.mark.parametrize("order", ALL_ORDERS)
def test_roundtrip_all_decoders(ctx, order):
    rng = random.Random(40 + order)
    raws = []
    for kind in ("q4", "q40", "runs", "one", "u32", "rand"):
        for n in (0, 1, 3, 31, 32, 33, 100, 1000, 1023, 4099, 70001):
            raws.append(_synth(rng, n, kind) if n else b"")
    comps = ctx.rans_nx16_encode(raws, [order] * len(raws))
    assert all(c is not None for c in comps)
    nz = [(c, r) for c, r in zip(comps, raws) if len(r)]
    for c, r in nz:
        assert orc_rans_nx16_decode(c, len(r)) == r, (order, len(r), c[:8].hex())
        assert ref_rans_nx16_decode(c, len(r)) == r, (order, len(r), c[:8].hex())
    res = run_batch(ctx, [c for c, _ in nz], [len(r) for _, r in nz])
    for (st, data), (_, r) in zip(res, nz):
        assert st == 0 and data == r
    # the transform bits are acted on where the reference acts on them
    for c, r in nz:
        theirs = ref_rans_nx16_encoded(r, order)
        assert (c[0] & 0xc8) == (theirs[0] & 0xc8), (order, len(r), hex(c[0]), hex(theirs[0]))


def test_transform_size_ratio_vs_reference(ctx):
    """PACK / RLE / STRIPE on the data each is for: within 3 % (+64 bytes) of the reference encoder given the same order."""
    rng = random.Random(77)
    cases = [("q4", 128), ("q4", 129), ("q4", 193), ("runs", 64), ("runs", 65), ("runs", 193), ("one", 192),
             ("u32", STRIPE4 | 1), ("u32", STRIPE4 | 193), ("q40", 197)]
    raws = [_synth(rng, 300_000, kind) for kind, _ in cases]
    mine = ctx.rans_nx16_encode(raws, [o for _, o in cases])
    for (kind, order), raw, m in zip(cases, raws, mine):
        assert m is not None, (kind, order)
        theirs = ref_rans_nx16_encoded(raw, order)
        assert ref_rans_nx16_decode(m, len(raw)) == raw, (kind, order)
        assert len(m) <= 1.03 * len(theirs) + 64, (kind, order, len(m), len(theirs))
        plain = ref_rans_nx16_encoded(raw, order & 5)
        if len(theirs) < 0.9 * len(plain):            # the transform pays on this input: it must pay for us too
            assert len(m) < 0.93 * len(plain), (kind, order, len(m), len(plain))


def test_size_ratio_vs_reference(ctx):
    """Stated ratio: within 3 % of the reference encoder on quality-like data (>= 64 KiB)."""
    from tools import synth
    rng = np.random.default_rng(5)
    q4 = (synth.novaseq_quals(rng, 1_500_000) + 33).astype(np.uint8).tobytes()
    q40 = (synth.hiseq_quals(rng, 1_500_000) + 33).astype(np.uint8).tobytes()
    for raw in (q4, q40):
        for order in (4, 5, 0, 1):
            mine = ctx.rans_nx16_encode([raw], [order])[0]
            theirs = ref_rans_nx16_encoded(raw, order)
            assert ref_rans_nx16_decode(mine, len(raw)) == raw
            assert len(mine) <= 1.03 * len(theirs) + 64, (order, len(mine), len(theirs))
