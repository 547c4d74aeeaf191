"""Pins the oracle's rANS Nx16 decoder: every golden stream of htscodecs/tests/dat/r4x16 must
decode to the raw input (the same check rans4x16.test:28-30,64-69 performs), and the oracle must
agree with the compiled reference on seeded inputs across every format-byte combination."""
import glob, os, random
import pytest
from _libs import GOLD, golden_raw, orc_rans_nx16_decode, ref, ref_rans_nx16_decode, ref_rans_nx16_decode_scalar, ref_rans_nx16_encode, sampled

R4X16 = sorted(glob.glob(os.path.join(GOLD, "htscodecs", "dat", "r4x16", "*")))


@pytest.mark.parametrize("path", R4X16, ids=[os.path.basename(p) for p in R4X16])
def test_golden_r4x16(path):
    name = os.path.basename(path).rsplit(".", 1)[0]
    raw = golden_raw(name)
    comp = open(path, "rb").read()
    assert orc_rans_nx16_decode(comp, len(raw)) == raw
    if ref() is not None:
        assert ref_rans_nx16_decode(comp, len(raw)) == raw


def _synth(rng, n, kind):
    if kind == "q4":
        syms = b"#-3E"
        out = bytearray(); cur = 3
        for _ in range(n):
            if rng.random() < 0.07: cur = rng.randrange(4)
            out.append(syms[cur])
        return bytes(out)
    if kind == "q40":
        return bytes(33 + min(40, int(abs(rng.gauss(30, 8)))) for _ in range(n))
    if kind == "runs":
        out = bytearray()
        while len(out) < n:
            out += bytes([rng.choice(b"ACGT")]) * rng.randrange(1, 40)
        return bytes(out[:n])
    if kind == "one":
        return b"A" * n
    if kind == "u32":
        out = bytearray(); v = 1000
        while len(out) < n:
            v += rng.randrange(0, 300); out += (v & 0xffffffff).to_bytes(4, "little")
        return bytes(out[:n])
    return bytes(rng.randrange(256) for _ in range(n))


ORDERS = [0, 1, 4, 5, 64, 65, 68, 69, 128, 129, 132, 133, 192, 193, 196, 197, 8, 9, 12, 13, 32]


@pytest.mark.parametrize("order", ORDERS)
def test_oracle_vs_reference_seeded(order):
    rng = random.Random(1234 + order)
    for kind in ("q4", "q40", "runs", "one", "u32", "rand"):
        for n in (0, 1, 3, 31, 32, 33, 100, 1000, 1023, 4099, 70001):
            if n == 0:
                continue
            raw = _synth(rng, n, kind)
            with sampled():
                comp = ref_rans_nx16_encode(raw, order)
                a = ref_rans_nx16_decode(comp, n)
                b = orc_rans_nx16_decode(comp, n)
                assert a == raw
                assert b == raw, (order, kind, n, comp[:8].hex())


def test_oracle_vs_reference_corrupt():
    """Malformed input: wherever the reference succeeds the oracle must give the same bytes."""
    rng = random.Random(7)
    raw = _synth(rng, 5000, "q40")
    agree = 0
    # The reference's SIMD decoders read differently from its scalar ones once a damaged
    # stream runs dry, so pin against the scalar implementation.
    for order in (0, 1, 4, 5, 65, 129, 193):
        comp = bytearray(ref_rans_nx16_encode(raw, order, store_always=True))
        for _ in range(40):
            c = bytearray(comp)
            # leave the header + tables alone: table-level undefined behaviour is not pinned
            k = rng.randrange(len(c) // 2, len(c))
            c[k] ^= 1 << rng.randrange(8)
            a = ref_rans_nx16_decode_scalar(bytes(c), len(raw))
            b = orc_rans_nx16_decode(bytes(c), len(raw))
            if a is not None:
                assert a == b
                agree += 1
    assert agree > 50
