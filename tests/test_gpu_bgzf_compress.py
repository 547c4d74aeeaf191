"""GPU BGZF compress (hgpu_bgzf_compress_batch_dev): blocks must be valid BGZF that zlib, the
oracle, the compiled reference reader and our own inflate kernel all expand to the input; the
size stays within a stated ratio of zlib level 6."""
import random, sys, zlib
import numpy as np
import pytest
import htslib_b200 as H
from _libs import ROOT, BGZF_EOF, orc_bgzf_inflate_block, ref, ref_bgzf_read_all
from test_oracle_bgzf import payloads
from test_gpu_bgzf import gpu_blocks
sys.path.insert(0, ROOT)
from tools import synth

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    c = H.Context(0)
    yield c
    c.close()


@pytest.mark.parametrize("level", [-1, 0, 1, 2, 3, 4, 5, 6, 7, 8, 9])
def test_roundtrip_every_decoder(ctx, level):
    rng = random.Random(level)
    ps = [p[:65280] for p in payloads(rng)] + [b"x" * 17, bytes(range(256)) * 255]
    blocks = ctx.bgzf_compress(ps, level)
    assert all(b is not None for b in blocks)
    for b, p in zip(blocks, ps):
        assert len(b) <= 65536 and b[:4] == b"\x1f\x8b\x08\x04"
        assert zlib.decompress(b[18:-8], -15) == p
        assert orc_bgzf_inflate_block(b) == (len(p), p)
        if level == 0 and len(p):
            assert len(b) == len(p) + 5 + 26                    # stored block, like bgzf.c:573-580
    res = gpu_blocks(ctx, blocks)
    for (st, data), p in zip(res, ps):
        assert st == 0 and data == p
    got, err = ref_bgzf_read_all(b"".join(blocks) + BGZF_EOF, 2)
    assert err == 0 and got == b"".join(ps)


def test_size_ratio_on_bam(ctx):
    """Stated ratio: <= 1.3x the zlib level-6 size on the synthetic sorted-BAM corpus (dynamic Huffman codes per block,
    single-probe LZ77 with one step of lazy evaluation vs zlib's chained search; measured 1.12x here, 1.39x with fixed
    codes and greedy matching in round 1)."""
    stream, offs = synth.bam_records(11, 6000)
    ps = [stream[i:i + 0xff00] for i in range(0, len(stream), 0xff00)]
    blocks = ctx.bgzf_compress(ps, 6)
    mine = sum(len(b) for b in blocks)
    theirs = sum(len(synth.bgzf_block(p, 6)) for p in ps)
    assert b"".join(zlib.decompress(b[18:-8], -15) for b in blocks) == stream
    assert mine <= 1.3 * theirs, (mine, theirs, len(stream))
    print("deflate ratio: ours %.3f zlib6 %.3f" % (mine / len(stream), theirs / len(stream)))
