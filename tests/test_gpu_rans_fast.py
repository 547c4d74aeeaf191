"""GPU parity for the two specialised rANS Nx16 kernels (rans_nx16_fast.cuh): the 32-way
small-alphabet symbol loop (fast32) and the eight-streams-per-warp 4-way loop (tile4).
Inputs come from the unmodified reference encoder; outputs must equal the raw input and,
for damaged streams, whatever the oracle produces — bit exact."""
import random
import numpy as np
import pytest
import htslib_b200 as H
from _libs import orc_rans_nx16_decode, ref, ref_rans_nx16_encode, sampled
from test_gpu_rans import run_batch

pytestmark = [pytest.mark.gpu]


@pytest.fixture(scope="module")
def ctx():
    c = H.Context(0)
    yield c
    c.close()


def markov(rng, n, syms, stay=0.9):
    """run-structured bytes over `syms` (NovaSeq-like)"""
    flips = rng.random(n) >= stay
    draw = rng.integers(0, len(syms), size=n)
    idx = np.maximum.accumulate(np.where(flips, np.arange(n), 0))
    return np.asarray(syms, dtype=np.uint8)[draw[idx]].tobytes()


ALPHABETS = [[2, 12, 23, 37], [0, 7, 9, 200], [5, 6], [0, 255, 3], [33], [1, 2, 3, 4, 5, 6, 7, 8], [9, 8, 7, 6, 5]]
SIZES = [2047, 2048, 2049, 2079, 4097, 40000, 65537, 300001, 1500000]


@pytest.mark.parametrize("order", [4, 5])
def test_x32_small_alphabets(ctx, order):
    rng = np.random.default_rng(17 + order)
    comps, raws = [], []
    for a in ALPHABETS:
        for n in SIZES:
            for stay in (0.97, 0.5):
                raw = markov(rng, n, a, stay)
                with sampled():
                    comps.append(ref_rans_nx16_encode(raw, order)); raws.append(raw)
    res = run_batch(ctx, comps, [len(r) for r in raws])
    for i, ((st, data), raw) in enumerate(zip(res, raws)):
        assert st == 0, (order, i, len(raw), comps[i][:4].hex())
        assert data == raw, (order, i, len(raw), comps[i][:4].hex())


def test_x32_nosz_and_shift12(ctx):
    """NOSZ streams (size from the caller) and alphabets whose order-1 table uses 12 bits."""
    rng = np.random.default_rng(3)
    comps, raws = [], []
    for order in (4 | 16, 5 | 16):
        for n in (5000, 123457):
            raw = markov(rng, n, [2, 12, 23, 37], 0.995)          # very skewed -> rans_compute_shift picks 12
            with sampled():
                comps.append(ref_rans_nx16_encode(raw, order)); raws.append(raw)
            raw = markov(rng, n, [40], 1.0)
            with sampled():
                comps.append(ref_rans_nx16_encode(raw, order)); raws.append(raw)
    res = run_batch(ctx, comps, [len(r) for r in raws])
    for i, ((st, data), raw) in enumerate(zip(res, raws)):
        assert st == 0 and data == raw, (i, len(raw), comps[i][:4].hex())


def test_x32_corrupt_matches_oracle(ctx):
    rng = random.Random(8)
    nrng = np.random.default_rng(8)
    comps, ulen = [], []
    for order in (4, 5):
        for a in ([2, 12, 23, 37], [0, 1, 2]):
            raw = markov(nrng, 50001, a, 0.9)
            comp = ref_rans_nx16_encode(raw, order, store_always=True)
            for _ in range(40):
                c = bytearray(comp)
                k = rng.randrange(1, len(c)); c[k] ^= 1 << rng.randrange(8)
                comps.append(bytes(c)); ulen.append(len(raw))
            for cut in (len(comp) // 2, len(comp) - 1, len(comp) - 70, 200):
                comps.append(comp[:cut]); ulen.append(len(raw))
    res = run_batch(ctx, comps, ulen)
    ok = 0
    for i, (c, (st, data)) in enumerate(zip(comps, res)):
        want = orc_rans_nx16_decode(c, ulen[i])
        if want is None:
            assert st != 0, i
        else:
            assert st == 0 and data == want, (i, c[:4].hex())
            ok += 1
    assert ok > 60


def test_n4_many_small_streams(ctx):
    """hundreds of 4-way streams of ragged sizes, both orders: eight per warp in the tile kernel"""
    rng = np.random.default_rng(21)
    comps, raws = [], []
    for i in range(700):
        n = int(rng.choice([1, 2, 3, 4, 5, 7, 8, 15, 16, 17, 63, 100, 999, 1000, 1001, 4096, 10000, 15000, 20011]))
        kind = i % 5
        if kind == 0:   raw = markov(rng, n, [2, 12, 23, 37], 0.8)
        elif kind == 1: raw = rng.integers(0, 256, size=n, dtype=np.uint8).tobytes()
        elif kind == 2: raw = np.clip(rng.normal(60, 25, size=n), 0, 255).astype(np.uint8).tobytes()
        elif kind == 3: raw = markov(rng, n, list(range(0, 40, 3)), 0.6)
        else:           raw = bytes([i & 255]) * n
        with sampled():
            comps.append(ref_rans_nx16_encode(raw, i % 2)); raws.append(raw)
    res = run_batch(ctx, comps, [len(r) for r in raws])
    for i, ((st, data), raw) in enumerate(zip(res, raws)):
        assert st == 0, (i, len(raw), comps[i][:4].hex())
        assert data == raw, (i, len(raw), comps[i][:4].hex())


def test_n4_corrupt_matches_oracle(ctx):
    rng = random.Random(4)
    nrng = np.random.default_rng(4)
    comps, ulen = [], []
    for order in (0, 1):
        for n in (37, 3000, 20000):
            raw = markov(nrng, n, [0, 3, 9, 27, 81], 0.7)
            comp = ref_rans_nx16_encode(raw, order, store_always=True)
            for _ in range(30):
                c = bytearray(comp)
                k = rng.randrange(1, len(c)); c[k] ^= 1 << rng.randrange(8)
                comps.append(bytes(c)); ulen.append(n)
            comps.append(comp[: len(comp) // 2]); ulen.append(n)
    res = run_batch(ctx, comps, ulen)
    ok = 0
    for i, (c, (st, data)) in enumerate(zip(comps, res)):
        want = orc_rans_nx16_decode(c, ulen[i])
        if want is None:
            assert st != 0, i
        else:
            assert st == 0 and data == want, (i, c[:4].hex())
            ok += 1
    assert ok > 60


def test_mixed_batch_every_pass(ctx):
    """one batch that exercises classify -> prep32 / tile4 / fast32 / general together"""
    rng = np.random.default_rng(77)
    comps, raws = [], []
    for i in range(120):
        order = [0, 1, 4, 5, 64, 65, 128, 129, 193, 8, 9, 4 | 64, 5 | 128][i % 13]
        n = int(rng.choice([50, 3000, 70000]))
        a = [[2, 12, 23, 37], list(range(30, 70)), [7]][i % 3]
        raw = markov(rng, n, a, 0.85)
        with sampled():
            comps.append(ref_rans_nx16_encode(raw, order)); raws.append(raw)
    perm = rng.permutation(len(comps))
    comps = [comps[i] for i in perm]; raws = [raws[i] for i in perm]
    res = run_batch(ctx, comps, [len(r) for r in raws])
    for i, ((st, data), raw) in enumerate(zip(res, raws)):
        assert st == 0 and data == raw, (i, len(raw), comps[i][:4].hex())
