"""GPU parity: tok3 read-name decode (CRAM 3.1 block method 8).  The product path is
hgpu_tok3_decode_batch_host (host framing walk -> rANS/arith batch kernels -> tok3_names_kernel);
checked against the reference's golden blocks (htscodecs/tests/names/tok3/*, tests/tok3.test), the
oracle on seeded blocks written by the reference encoder, the name block of a reference-written
CRAM 3.1 file, and on corrupted blocks (must fail or succeed exactly where the reference does)."""
import ctypes as C
import glob
import os
import random

import numpy as np
import pytest

import htslib_b200 as H
import _libs as L
from test_oracle_tok3 import TOK3, _names, _plain

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    c = H.Context(0)
    yield c
    c.close()


def test_golden_blocks_one_batch(ctx):
    comps = [open(p, "rb").read() for p in TOK3]
    assert len(comps) >= 100
    res = ctx.tok3_decode(comps)
    for p, (st, data) in zip(TOK3, res):
        assert st == 0, os.path.basename(p)
        assert data == _plain(p), os.path.basename(p)


def test_seeded_vs_oracle(ctx):
    comps, wants = [], []
    for style in (0, 1, 2):
        for level, arith in [(1, 0), (3, 0), (5, 0), (7, 0), (9, 0), (1, 1), (3, 1)]:
            for n in (1, 2, 33, 600, 5000):
                rng = random.Random(1000 * style + 10 * level + arith + n)
                blob = _names(rng, n, style)
                with L.sampled():
                    comp = L.ref_tok3_encode(blob, level, arith)
                    want = L.orc_tok3_decode(comp)
                    assert want == blob
                    comps.append(comp); wants.append(want)
    res = ctx.tok3_decode(comps)
    for i, ((st, data), w) in enumerate(zip(res, wants)):
        assert st == 0, i
        assert data == w, i


def test_many_tokens_and_long_names(ctx):
    rng = random.Random(5)
    # > 32 token positions per name (several lane chunks), and names close to the 1024-byte slack
    a = "\0".join(":".join(str(rng.randrange(1, 50) + i // 7) for _ in range(45)) for i in range(300)) + "\0"
    b = "\0".join("x" * rng.randrange(900, 1500) + str(i) for i in range(40)) + "\0"
    comps = [L.ref_tok3_encode(a.encode(), 5, 0, store_always=True), L.ref_tok3_encode(b.encode(), 5, 0, store_always=True)]
    res = ctx.tok3_decode(comps)
    for (st, data), c in zip(res, comps):
        assert st == 0
        assert data == L.orc_tok3_decode(c)


def test_corrupt_blocks_agree(ctx):
    rng = random.Random(7)
    comp = L.ref_tok3_encode(_names(rng, 200, 0), 5, 0)
    bad = []
    for trial in range(200):
        c = bytearray(comp)
        if trial % 3 == 0:
            c = c[: rng.randrange(9, len(c))]
        else:
            for _ in range(rng.randrange(1, 3)):
                c[rng.randrange(8 if trial % 3 == 1 else 0, len(c))] = rng.randrange(256)
        if int.from_bytes(c[4:8], "little") > 100000 or int.from_bytes(c[0:4], "little") > 1 << 20:
            continue
        bad.append(bytes(c))
    res = ctx.tok3_decode(bad)
    refused = 0
    for c, (st, data) in zip(bad, res):
        if st == -5:                  # HGPU_TOK3_ERR_LIMIT: a stream size field beyond what any encoder writes
            refused += 1
            continue
        want = L.orc_tok3_decode(c)
        if want is None:
            assert st != 0
        else:
            assert st == 0 and data == want
    assert len(bad) > 100 and refused < len(bad) // 10


def test_cram31_name_block_and_shim(ctx):
    img = np.fromfile(os.path.join(L.GOLD, "htslib", "ce#1000.v31.cram"), dtype=np.uint8)
    blocks, _ = H.cram_scan_blocks(img)
    nb = blocks[blocks["method"] == 8]
    assert len(nb) == 1
    comp = img[int(nb[0]["data_off"]):int(nb[0]["data_off"]) + int(nb[0]["comp_size"])].tobytes()
    (st, data), = ctx.tok3_decode([comp])
    assert st == 0 and len(data) == int(nb[0]["uncomp_size"])
    assert data == L.orc_tok3_decode(comp)
    assert data.count(b"\0") == 1000
    # the reference-named symbol, as cram_uncompress_block would call it
    lib = H.lib()
    n = C.c_uint32(0)
    p = lib.tok3_decode_names(comp, len(comp), C.byref(n))
    assert p and C.string_at(p, n.value) == data
    C.CDLL(None).free(C.c_void_p(p))
    assert not lib.tok3_decode_names(comp[:40], 40, C.byref(n))
