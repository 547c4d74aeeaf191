"""GPU BAI / CSI building (hgpu_bam_index_build_host) against the reference's sam_index_build3: the BAI file byte for
byte, the CSI file's inflated content byte for byte, at min_shift 0, 12, 14 and 16; the same bytes however the file is cut
into windows; the same refusals on damaged files."""
import os

import numpy as np
import pytest

import _bam_index_ref as B
import htslib_b200 as H

pytestmark = pytest.mark.gpu
SHIFTS = (0, 12, 14, 16)
WINDOWS = (0xff00, 2 * 0xff00, 3 * 0xff00)


@pytest.fixture(scope="module")
def ctx():
    c = H.Context(0)
    yield c
    c.close()


def gpu_index(ctx, img, min_shift, window_bytes=0):
    out = ctx.bam_index(np.frombuffer(img, dtype=np.uint8), min_shift, window_bytes)
    if min_shift > 0:
        assert out[-28:] == bytes.fromhex("1f8b08040000000000ff0600424302001b0003000000000000000000")
        return B.inflate_bgzf(out)
    return out


def gold(name):
    with open(os.path.join(B.GOLD_HTS, name), "rb") as f:
        return f.read()


def same_as_reference(ctx, img, shifts=SHIFTS, windows=(0,) + WINDOWS):
    for ms in shifts:
        rc, want = B.ref_bam_index(img, ms)
        assert rc == 0, ms
        for w in windows:
            assert gpu_index(ctx, img, ms, w) == want, (ms, w)


def test_index_bam_golden(ctx):
    """index.bam (index.sam through the reference's level-0 writer) gives the reference's own index.bam.bai / .csi."""
    img = B.index_bam()
    same_as_reference(ctx, img)
    assert gpu_index(ctx, img, 0) == gold("index.bam.bai")
    assert gpu_index(ctx, img, 14) == B.inflate_bgzf(gold("index.bam.csi"))


@pytest.mark.parametrize("name,golden,shift", [("range.bam", "range.bam.bai", 0), ("colons.bam", "colons.bam.bai", 0),
                                                ("no_hdr_sq_1.bam", "no_hdr_sq_1.bam.csi", 14)])
def test_reference_fixtures(ctx, name, golden, shift):
    img = gold(name)
    same_as_reference(ctx, img)
    want = gold(golden)
    want = B.inflate_bgzf(want) if shift else want
    if B.ref_bam_index(img, shift)[1] == want:            # a golden file an older htslib wrote may differ: the compiled reference wins
        assert gpu_index(ctx, img, shift) == want


@pytest.mark.parametrize("n", [1, 2, 3])
def test_bgzf_boundaries(ctx, n):
    """Records that straddle blocks."""
    same_as_reference(ctx, gold(os.path.join("bgzf_boundaries", "bgzf_boundaries%d.bam" % n)))


@pytest.mark.parametrize("name", sorted(B.multi_files()))
def test_synthetic_layouts(ctx, name):
    """Several references (one without records), unmapped-placed reads, an unplaced tail, spliced reads over many 16 kb
    windows, a CG-tag CIGAR, blocks ending exactly at record ends, empty blocks, a header ending mid-block, level 0 and
    6 blocks, files with and without the EOF block."""
    same_as_reference(ctx, B.multi_files()[name])


def test_600mbp_reference(ctx):
    img = B.big_ref_file()
    for ms in (12, 14, 16):
        rc, want = B.ref_bam_index(img, ms)
        assert rc == 0
        got = gpu_index(ctx, img, ms)
        assert got == want
        if ms == 14:
            assert got[8:12] == (6).to_bytes(4, "little")          # n_lvls 6
    assert B.ref_bam_index(img, 0)[0] != 0
    with pytest.raises(H.HgpuError) as e:
        ctx.bam_index(np.frombuffer(img, dtype=np.uint8), 0)
    assert (e.value.code, e.value.bad) == (H.IDX_ERR_PUSH, 4)       # the first record that reaches past 2^29


def test_synthetic_corpus(ctx):
    """A few hundred MB of synthetic records: compress_binning merges bins, and the file takes many windows."""
    img = B.synth_file()
    for ms in (0, 14):
        rc, want = B.ref_bam_index(img, ms)
        assert rc == 0
        assert gpu_index(ctx, img, ms) == want
        assert gpu_index(ctx, img, ms, 64 << 20) == want
    assert gpu_index(ctx, img, 0, 3 * 0xff00) == B.ref_bam_index(img, 0)[1]


CODES = {"push": H.IDX_ERR_PUSH, "read": H.IDX_ERR_READ}


@pytest.mark.parametrize("case", sorted(B.refusal_cases()))
def test_refusals(ctx, case):
    """Each refusal injected into a valid file: the right code, and *bad names the injected record or block."""
    img, kind, bad = B.refusal_cases()[case]
    code = CODES.get(kind)
    assert B.ref_bam_index(img, 0)[0] != 0 and B.ref_bam_index(img, 14)[0] != 0
    for ms in (0, 14):
        for w in (0, 0xff00):
            with pytest.raises(H.HgpuError) as e:
                ctx.bam_index(np.frombuffer(img, dtype=np.uint8), ms, w)
            if code is None:
                assert e.value.code in (H.BGZF_ERR_ZLIB, H.BGZF_ERR_CRC), case
            else:
                assert e.value.code == code, case
            assert e.value.bad == bad, case


def test_not_bam(ctx):
    """A BGZF file that is not BAM (SAM text) and a file that is not BGZF are argument errors."""
    sam = B.bgzf(b"@HD\tVN:1.6\n" * 100)
    for img in (sam, b"plain text, not BGZF at all" * 10):
        with pytest.raises(H.HgpuError) as e:
            ctx.bam_index(np.frombuffer(img, dtype=np.uint8), 0)
        assert e.value.code == H.ERR_ARG
