"""hgpu_cram_index_build_host (Context.cram_index) on the files of test_cram_index_reference.py: the index inflates to the
reference's .crai text, refusals are the reference's, and the file is exactly one gzip member, as the reference's reader
(zlib_mem_inflate, which stops at the end of the first member) needs.  The reference then answers region queries with it."""
import ctypes as C
import os
import zlib
import numpy as np
import pytest
import htslib_b200 as H
from _libs import Bam1, ref
from test_cram_index_reference import (BASE_OF, CASE_NAMES, REF_RC, _sorted_sam, _sq_fasta, cases, hostsim_index, ref_cram_index,
                                       ref_crai_sam_records)
from test_cram_mates import encode

pytestmark = pytest.mark.gpu


def one_member(gz):
    d = zlib.decompressobj(31)
    text = d.decompress(gz)
    assert d.eof and d.unused_data == b""
    return text


@pytest.fixture(scope="module")
def ctx():
    c = H.Context(0)
    yield c
    c.close()


@pytest.mark.parametrize("name", CASE_NAMES)
def test_gpu_index_equals_reference(tmp_path, ctx, name):
    all_cases = dict(cases(tmp_path))
    img = all_cases[name]
    want_rc, want_text = ref_cram_index(img)
    arr = np.frombuffer(img, np.uint8).copy()
    if want_rc == 0:
        assert one_member(ctx.cram_index(arr)) == want_text, name
    else:
        with pytest.raises(H.HgpuError) as e:
            ctx.cram_index(arr)
        assert e.value.code == REF_RC[want_rc], (name, e.value.code, want_rc)
        _, bad, _ = hostsim_index(img, all_cases[BASE_OF[name]] if name in BASE_OF else None)
        assert e.value.bad == bad, (name, e.value.bad, bad)


def _spliced(tmp_path, ctx):
    """A file of 8250 two-record multi-reference slices over 3 references from the device writer's host build: over 3 x 0xff00
    bytes of index text."""
    fa, sam = str(tmp_path / "big.fa"), str(tmp_path / "big.sam")
    _sorted_sam(sam, _sq_fasta(fa, 3, 30000, 11), 5500, 12)
    text, recs = ref_crai_sam_records(sam)
    img, _ = encode(None, text, recs, 2, 1, None, flags=0)
    return img


def test_gpu_index_text_over_several_deflate_payloads(tmp_path, ctx):
    img = _spliced(tmp_path, ctx)
    gz = ctx.cram_index(np.frombuffer(img, np.uint8).copy())
    text = one_member(gz)
    assert len(text) >= 3 * 0xff00
    want_rc, want_text = ref_cram_index(img)
    assert want_rc == 0 and text == want_text
    dev_ms, rest_ms = ctx.cram_index_last_ms()
    assert dev_ms > 0 and rest_ms >= 0


def _query_counts(path, crai, regions):
    r = ref()
    r.hts_open.restype = C.c_void_p
    r.hts_open.argtypes = [C.c_char_p, C.c_char_p]
    r.hts_close.argtypes = [C.c_void_p]
    r.sam_hdr_read.restype = C.c_void_p
    r.sam_hdr_read.argtypes = [C.c_void_p]
    r.sam_hdr_destroy.argtypes = [C.c_void_p]
    r.sam_index_load2.restype = C.c_void_p
    r.sam_index_load2.argtypes = [C.c_void_p, C.c_char_p, C.c_char_p]
    r.sam_itr_querys.restype = C.c_void_p
    r.sam_itr_querys.argtypes = [C.c_void_p, C.c_void_p, C.c_char_p]
    r.hts_itr_next.argtypes = [C.c_void_p, C.c_void_p, C.POINTER(Bam1), C.c_void_p]
    r.hts_itr_destroy.argtypes = [C.c_void_p]
    r.hts_idx_destroy.argtypes = [C.c_void_p]
    r.bam_init1.restype = C.POINTER(Bam1)
    r.bam_destroy1.argtypes = [C.POINTER(Bam1)]
    fp = r.hts_open(path.encode(), b"r")
    hdr = r.sam_hdr_read(fp)
    idx = r.sam_index_load2(fp, path.encode(), crai.encode())
    assert idx
    b = r.bam_init1()
    counts = []
    for reg in regions:
        it = r.sam_itr_querys(idx, hdr, reg)
        assert it, reg
        n = 0
        while r.hts_itr_next(None, it, b, fp) >= 0:          # sam_itr_next on a CRAM file
            n += 1
        counts.append(n)
        r.hts_itr_destroy(it)
    r.bam_destroy1(b)
    r.hts_idx_destroy(idx)
    r.sam_hdr_destroy(hdr)
    r.hts_close(fp)
    return counts


def test_gpu_index_answers_region_queries_in_the_reference(tmp_path, ctx):
    if ref() is None:
        pytest.skip("needs oracle/_ref")
    img = _spliced(tmp_path, ctx)
    path = str(tmp_path / "q.cram")
    open(path, "wb").write(img)
    mine, theirs = str(tmp_path / "mine.crai"), str(tmp_path / "theirs.crai")
    open(mine, "wb").write(ctx.cram_index(np.frombuffer(img, np.uint8).copy()))
    r = ref()
    r.sam_index_build3.argtypes = [C.c_char_p, C.c_char_p, C.c_int, C.c_int]
    assert r.sam_index_build3(path.encode(), theirs.encode(), 0, 0) == 0
    regions = [b"s0:100-500", b"s1", b"s2:29000-30000", b"s1:15000-15100", b"s0:1-1"]
    got = _query_counts(path, mine, regions)
    assert got == _query_counts(path, theirs, regions)
    assert sum(got) > 0
