"""GPU: fqzcomp quality ENCODER.  One parameter block, no selector search, so the bytes are its own; the
bar is the decoder's: the reference's fqz_decompress and this library's decoder return the input, for all
four strategy rows, fixed and variable lengths, duplicate records, tiny and 1.5 MB blocks; and the size
stays close to the reference encoder's."""
import os
import random

import pytest

import htslib_b200 as H
import _libs as L
from test_gpu_fqzcomp import _quals, _column1

pytestmark = pytest.mark.gpu


def test_round_trip_through_reference_and_own_decoder():
    ctx = H.Context(0)
    rng = random.Random(21)
    blocks = []
    for kind in ("q4", "q40", "var"):
        for n_rec in (1, 7, 300):
            q, lens, _ = _quals(rng, n_rec, kind)
            blocks.append((q, lens))
    for name, l in (("q4", 151), ("q40+dir", 100), ("q8", 250)):      # the reference's own test data, whole files
        q = _column1(name)
        rows = open(os.path.join(L.GOLD, "htscodecs", "dat", name), "rb").read().split(b"\n")
        blocks.append((q, [len(r.split(b"\t")[0]) for r in rows if r]))
    q, lens, _ = _quals(rng, 10000, "q4")                              # a CRAM slice worth of NovaSeq-like qualities
    blocks.append((q, lens))
    for strat in (0, 1, 2, 3):
        res = H.fqz_encode(ctx, [b[0] for b in blocks], [b[1] for b in blocks], strat)
        comps = []
        for (q, lens), (st, comp) in zip(blocks, res):
            assert st == 0, (strat, len(q))
            assert L.ref_fqz_decompress(comp) == q, (strat, len(q))
            comps.append(comp)
        back = H.fqz_decode(ctx, comps, [len(b[0]) for b in blocks])
        for (q, _), (st, data) in zip(blocks, back):
            assert st == 0 and data == q
        if strat == 0:                         # size against the reference encoder, same strategy
            ours = sum(len(c) for c in comps[-4:])
            theirs = sum(len(L.ref_fqz_compressed(q, lens, None, 0)) for q, lens in blocks[-4:])
            assert ours < 1.1 * theirs, (ours, theirs)
    # rejected: lengths that do not tile the block
    (st, _), = H.fqz_encode(ctx, [b"\x05" * 100], [[60, 30]])
    assert st != 0
    ctx.close()
