"""Writes tests/golden/htslib/index.bam: index.sam through the compiled reference's BAM writer at level 0, as the
reference's own test_index makes it (test/test.pl: test_view -l 0 -b).  Needs oracle/_ref built."""
import ctypes as C
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
import _libs  # noqa: E402


def main():
    r = _libs.ref()
    assert r is not None, "oracle/_ref is not built"
    vp = C.c_void_p
    r.hts_open.restype = vp
    r.hts_open.argtypes = [C.c_char_p, C.c_char_p]
    r.hts_close.argtypes = [vp]
    r.sam_hdr_read.restype = vp
    r.sam_hdr_read.argtypes = [vp]
    r.sam_hdr_write.argtypes = [vp, vp]
    r.sam_hdr_destroy.argtypes = [vp]
    r.sam_read1.argtypes = [vp, vp, vp]
    r.sam_write1.argtypes = [vp, vp, vp]
    r.bam_init1.restype = vp
    r.bam_destroy1.argtypes = [vp]
    src = os.path.join(HERE, "htslib", "index.sam")
    dst = os.path.join(HERE, "htslib", "index.bam")
    fi = r.hts_open(src.encode(), b"r")
    fo = r.hts_open(dst.encode(), b"wb0")
    h = r.sam_hdr_read(fi)
    assert fi and fo and h and r.sam_hdr_write(fo, h) == 0
    b = r.bam_init1()
    while r.sam_read1(fi, h, b) >= 0:
        assert r.sam_write1(fo, h, b) >= 0
    r.bam_destroy1(b)
    r.sam_hdr_destroy(h)
    r.hts_close(fi)
    assert r.hts_close(fo) == 0


if __name__ == "__main__":
    main()
