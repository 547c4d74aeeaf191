"""Pins the plain references of tests/rans_model.py (no GPU) before they judge the rANS Nx16 encoder kernel.

- trace + core_encode reproduce the reference encoder's streams byte for byte: every order in ORDERS, X32 with order
  0 and 1, STRIPE, and order-1 tables long enough for the reference to code them again.
- rans_model.encode's streams decode to the input with the reference decoder (SIMD and scalar) and the oracle.
- Decisions the data alone fixes (PACK taken, RLE taken, order dropped, X32 dropped) match the reference's stream.
- normalise_opt matches brute force; the restated normalisations keep their invariants."""
import itertools
import math
import random

import numpy as np
import pytest

import rans_model as M
from _libs import orc_rans_nx16_decode, ref_rans_nx16_decode, ref_rans_nx16_decode_scalar, ref_rans_nx16_encode, sampled
from test_oracle_rans import ORDERS, _synth

KINDS = ("q4", "q40", "runs", "one", "u32", "rand")
SMALL = (1, 3, 8, 31, 100, 400)
STRIPE = [8 | 1, 8 | (3 << 8) | 65, 8 | (7 << 8) | 193]


def check_reproduces(stream, n):
    """trace the stream; every entropy core in it, re-encoded from its decoded bytes with its traced tables, gives
    exactly its bytes, and the containers account for every byte.  Returns the trace."""
    t = M.trace(stream, n)
    assert t["end"] == len(stream)
    for where, c in M.cores(t):
        assert c["odd"] == b"", where
        assert M.core_encode(c["data"], c["order"], c["N"], c) == c["bytes"], where
    return t


@pytest.mark.parametrize("order", ORDERS + STRIPE)
def test_trace_reproduces_reference_small(order):
    rng = random.Random(600 + order)
    done = 0
    for kind in KINDS:
        for n in SMALL:
            raw = _synth(rng, n, kind)
            with sampled():
                check_reproduces(ref_rans_nx16_encode(raw, order), n)
                done += 1
    assert done


# larger inputs, stored whatever their size: X32 with order 0 and 1, STRIPE, and long order-1 tables
LARGE = [("q40", 1500, 4), ("q40", 1500, 5), ("u32", 1500, 5), ("runs", 3000, 0x45), ("q4", 2000, 0x85), ("q40", 1200, 8 | 1),
         ("skew", 12000, 1), ("skew", 12000, 5)]


def _input(rng, kind, n):
    """_synth, plus "skew": 200 symbols at Zipf-like frequencies, an order-1 table long enough to be coded again"""
    if kind == "skew":
        return bytes(rng.choices(range(1, 200), weights=[1 / (i + 1) ** 2 for i in range(199)], k=n))
    return _synth(rng, n, kind)


def test_trace_reproduces_reference_large():
    rng = random.Random(601)
    nested = stripe = 0
    for kind, n, order in LARGE:
        raw = _input(rng, kind, n)
        t = check_reproduces(ref_rans_nx16_encode(raw, order, store_always=True), n)
        stripe += bool(t["stripe"])
        nested += any(c.get("nested") is not None for _, c in M.cores(t))
        if order & 4 and not t["stripe"]:
            assert t["fmt"] & 4 and all(c["N"] == 32 for w, c in M.cores(t) if not w.endswith("table"))
    assert nested and stripe


def decisions(stream):
    """The choices of a flat stream that the data alone fixes."""
    f = stream[0]
    return dict(pack=bool(f & M.F_PACK), rle=bool(f & M.F_RLE), x32=bool(f & M.F_X32), order=None if f & M.F_CAT else f & 1)


@pytest.mark.parametrize("order", ORDERS)
def test_model_decodes_and_decides_like_reference(order):
    rng = random.Random(700 + order)
    for kind in KINDS:
        for n in SMALL + (1001, 4099):
            raw = _synth(rng, n, kind)
            s = M.encode(raw, order)
            assert orc_rans_nx16_decode(s, n) == raw, (order, kind, n)
            with sampled():
                assert ref_rans_nx16_decode(s, n) == raw
                assert ref_rans_nx16_decode_scalar(s, n) == raw
            with sampled():
                theirs = ref_rans_nx16_encode(raw, order)
                if order & M.F_STRIPE:
                    continue
                mine, ref_d = decisions(s), decisions(theirs)
                # Intended divergence: the order bit of a CAT stream is cleared by the kernel and kept by the reference,
                # and which side falls back to CAT depends on sizes, not the data alone: compare the order only where
                # neither stream is CAT.
                if mine["order"] is None or ref_d["order"] is None:
                    mine["order"] = ref_d["order"] = None
                assert mine == ref_d, (order, kind, n, s[:4].hex(), theirs[:4].hex())


@pytest.mark.parametrize("flags", [0x41, 0x81, 0xc5, 0x20, 8 | (5 << 8) | 193, 8 | (2 << 8) | 1 | M.F_STRIPE_NO0])
def test_model_encode_decodes_with_transforms(flags):
    rng = random.Random(800 + (flags & 0xffff))
    for kind in KINDS:
        for n in (0, 1, 21, 300, 1001, 5000):
            raw = _synth(rng, n, kind) if n else b""
            s = M.encode(raw, flags)
            if n:
                assert orc_rans_nx16_decode(s, n) == raw, (hex(flags), kind, n)
                with sampled():
                    assert ref_rans_nx16_decode(s, n) == raw
            t = M.trace(s, n)
            assert t["end"] == len(s)


def _brute(counts, M_):
    present = [j for j, c in enumerate(counts) if c]
    best = None
    for f in itertools.product(range(1, M_ + 1), repeat=len(present)):
        if sum(f) != M_:
            continue
        v = sum(counts[j] * math.log(x) for j, x in zip(present, f))
        if best is None or v > best + 1e-12:
            best = v
    return best


def test_normalise_opt_brute_force():
    rng = random.Random(5)
    for _ in range(300):
        k = rng.randrange(1, 5)
        counts = [rng.randrange(0, 30) for _ in range(k)] + [0]
        if not any(counts):
            continue
        Mt = rng.randrange(max(1, sum(1 for c in counts if c)), 17)
        f = M.normalise_opt(counts, Mt)
        assert int(f.sum()) == Mt and all((c > 0) == (x > 0) for c, x in zip(counts, f))
        got = sum(c * math.log(x) for c, x in zip(counts, f) if c)
        assert abs(got - _brute(counts, Mt)) < 1e-9, (counts, Mt, f)


@pytest.mark.parametrize("norm", [M.normalise_row, M.normalise_ref])
def test_normalisations_keep_invariants(norm):
    rng = np.random.default_rng(6)
    for _ in range(300):
        A = int(rng.integers(1, 257))
        c = rng.integers(0, 1 + int(rng.integers(1, 2000)), size=256) * (rng.random(256) < A / 256)
        if not c.any():
            continue
        Mt = int(2 ** rng.integers(max(8, int(np.ceil(np.log2(max(1, (c > 0).sum()))))), 13))
        f = norm(c, Mt)
        assert int(f.sum()) == Mt and ((f > 0) == (c > 0)).all()
        assert M.cost_bits(c, f, Mt) >= M.cost_bits(c, M.normalise_opt(c, Mt), Mt) - 1e-6


def test_row_target_and_shift_rule():
    assert M.shift_rule(128) == 10 and M.shift_rule(129) == 12
    assert M.row_target(0, 0, 12) == (4096, 0)
    assert M.row_target(1, 1, 12) == (1, 12)                 # a single successor: stored as 1, scaled up to 4096
    assert M.row_target(3000, 70, 12) == (2048, 1)
    assert M.row_target(3000, 10, 10) == (1024, 0)
    assert M.row_target(5, 100, 12) == (128, 5)


def test_varints_and_alphabets():
    for v in (0, 1, 127, 128, 16383, 16384, 1 << 21, (1 << 28) + 5, 0xffffffff):
        assert M.vget(M.vput(v) + b"\xff", 0) == (v, len(M.vput(v)))
    rng = random.Random(8)
    for _ in range(200):
        present = [rng.random() < rng.random() for _ in range(256)]
        present[rng.randrange(256)] = True
        syms, p = M.read_alphabet(M.put_alphabet(present) + b"\x07", 0)
        assert syms == [j for j in range(256) if present[j]] and p == len(M.put_alphabet(present))


def test_core_coder_round_trip():
    rng = random.Random(9)
    for order, N in ((0, 4), (0, 32), (1, 4), (1, 32)):
        for n in (1, 7, 33, 1001, 5003):
            raw = _synth(rng, n, "q40")
            c = M.core_encode(raw, order, N)
            core = M._trace_core(c, order, N, n)
            assert M.core_decode(core, n) == raw
            assert orc_rans_nx16_decode(bytes([order | (4 if N == 32 else 0) | M.F_NOSZ]) + c, n) == raw
