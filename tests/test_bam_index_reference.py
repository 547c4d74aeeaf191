"""The fixtures of the GPU index tests, pinned on the CPU: the reference's sam_index_build3 (its stored results where
oracle/_ref is absent) reproduces its own golden index files, indexes every synthetic layout with the counts the
builders put in, and refuses every damaged file."""
import os

import pytest

import _bam_index_ref as B


def gold(name):
    with open(os.path.join(B.GOLD_HTS, name), "rb") as f:
        return f.read()


def test_index_bam_is_the_reference_fixture():
    img = B.index_bam()
    assert B.ref_bam_index(img, 0) == (0, gold("index.bam.bai"))
    assert B.ref_bam_index(img, 14) == (0, B.inflate_bgzf(gold("index.bam.csi")))


@pytest.mark.parametrize("name", ["range.bam", "colons.bam", "no_hdr_sq_1.bam"] +
                         [os.path.join("bgzf_boundaries", "bgzf_boundaries%d.bam" % n) for n in (1, 2, 3)])
def test_reference_fixtures_index(name):
    for ms in (0, 12, 14, 16):
        assert B.ref_bam_index(gold(name), ms)[0] == 0


@pytest.mark.parametrize("name", sorted(B.multi_files()))
def test_synthetic_layouts_index(name):
    img = B.multi_files()[name]
    for ms in (0, 12, 14, 16):
        assert B.ref_bam_index(img, ms)[0] == 0
        rc, (n_ref, bins, n_no_coor) = B.ref_bam_index_summary(img, ms)
        assert (rc, n_ref, bins[1], n_no_coor) == (0, 3, 0, 30)


def test_600mbp_reference_index():
    img = B.big_ref_file()
    assert B.ref_bam_index(img, 0)[0] != 0
    for ms in (12, 14, 16):
        assert B.ref_bam_index(img, ms)[0] == 0


@pytest.mark.parametrize("case", sorted(B.refusal_cases()))
def test_refusals_refused(case):
    img = B.refusal_cases()[case][0]
    for ms in (0, 14):
        assert B.ref_bam_index(img, ms)[0] != 0
