"""GPU: tok3 read-name ENCODER.  Its bytes are its own (names are diffed against the previous name, token
streams coded by this library's rANS encoder), so the bar is: the reference's tok3_decode_names, the oracle
and this library's own decoder all rebuild exactly the input names, and the size stays within a stated
factor of the reference encoder's at the level CRAM uses (3)."""
import glob
import gzip
import os
import random

import pytest

import htslib_b200 as H
import _libs as L
from test_oracle_tok3 import _names

pytestmark = pytest.mark.gpu


def test_round_trip_through_reference_and_own_decoder():
    ctx = H.Context(0)
    blobs = []
    for p in sorted(glob.glob(os.path.join(L.GOLD, "htscodecs", "names", "*.names"))):
        blobs.append(open(p, "rb").read())                              # LF separated, as the reference's tests feed them
    for style in (0, 1, 2):
        for n in (1, 2, 33, 600, 5000):
            blobs.append(_names(random.Random(31 * style + n), n, style))
    for k in range(8):
        blobs.append(gzip.open(os.path.join(L.GOLD, "tok3_slices", "slice%d.names.gz" % k), "rb").read())
    blobs.append(b"0\x0007\x00007:1\x00a1b22c333\x00\x00::\x00" + b"9" * 30 + b"\0")   # zeros, leading zeros, empty name, 9-digit splits
    res = H.tok3_encode(ctx, blobs)
    comps = []
    for blob, (st, comp) in zip(blobs, res):
        assert st == 0
        want = blob.replace(b"\n", b"\0")
        assert L.orc_tok3_decode(comp) == want
        assert L.ref_tok3_decode(comp) == want
        comps.append(comp)
    back = ctx.tok3_decode(comps)
    for blob, (st, data) in zip(blobs, back):
        assert st == 0 and data == blob.replace(b"\n", b"\0")
    # size against the reference encoder at CRAM's level, on the 10 000-name slice fixtures
    ours = sum(len(c) for c in comps[-9:-1])
    theirs = sum(os.path.getsize(os.path.join(L.GOLD, "tok3_slices", "slice%d.tok3" % k)) for k in range(8))
    assert ours < 1.6 * theirs, (ours, theirs)
    # rejected inputs: empty block, more token positions than the format has
    (st0, _), (st1, _) = H.tok3_encode(ctx, [b"", b":".join([b"a"] * 200) + b"\0"])
    assert st0 != 0 and st1 != 0
    ctx.close()
