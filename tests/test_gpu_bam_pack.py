"""GPU BAM record pack (hgpu_bam_pack_dev == bam_write1's data movement): unpack -> pack must
reproduce the record stream byte for byte, agree with the oracle's orc_bam_pack1, and the oracle is
pinned to the compiled reference's bam_write1 (uncompressed BGZF mode)."""
import ctypes as C
import os, sys, tempfile, zlib
import numpy as np
import pytest
import htslib_b200 as H
from _libs import ROOT, GOLD, Bam1, BamCore, bam_header, bam_header_len, bgzf_file, orc, orc_bam_unpack_all, orc_bgzf_scan, ref, buf, stored_reference
sys.path.insert(0, ROOT)
from tools import synth


def orc_pack(recs):
    o = orc(); o.orc_bam_pack1.restype = C.c_long
    out = bytearray()
    for st, core, data, _, _ in recs:
        c = BamCore(*core)
        ob = (C.c_uint8 * (len(data) + 64))()
        n = o.orc_bam_pack1(C.byref(c), buf(data), C.c_uint32(len(data)), ob)
        assert n > 0
        out += bytes(ob[:n])
    return bytes(out)


@stored_reference(digest=True)
def ref_bam_write1_all(path):
    """bam_read1 every record of a BAM file and bam_write1 it to an uncompressed ('wu') BGZF file: that file."""
    r = ref()
    r.bgzf_open.restype = C.c_void_p; r.bgzf_open.argtypes = [C.c_char_p, C.c_char_p]
    r.bgzf_close.argtypes = [C.c_void_p]
    r.bam_hdr_read.restype = C.c_void_p; r.bam_hdr_read.argtypes = [C.c_void_p]
    r.bam_init1.restype = C.POINTER(Bam1)
    r.bam_read1.argtypes = [C.c_void_p, C.POINTER(Bam1)]
    r.bam_write1.argtypes = [C.c_void_p, C.POINTER(Bam1)]
    r.bam_destroy1.argtypes = [C.POINTER(Bam1)]
    r.sam_hdr_destroy.argtypes = [C.c_void_p]
    with tempfile.TemporaryDirectory() as td:
        outp = os.path.join(td, "o.raw").encode()
        fin = r.bgzf_open(path.encode(), b"r"); fout = r.bgzf_open(outp, b"wu")
        hdr = r.bam_hdr_read(fin)
        b = r.bam_init1()
        while r.bam_read1(fin, b) >= 0:
            assert r.bam_write1(fout, b) > 0
        r.bam_destroy1(b); r.sam_hdr_destroy(hdr); r.bgzf_close(fin); r.bgzf_close(fout)
        return open(outp, "rb").read()


def test_oracle_pack_matches_reference_bam_write1():
    """reference: bam_read1 every record of a fixture, bam_write1 it to an uncompressed ('wu') BGZF
    file; the file body after the header must equal the oracle's packing of the oracle's unpacking."""
    path = os.path.join(GOLD, "htslib", "range.bam")
    img = open(path, "rb").read()
    _, blocks = orc_bgzf_scan(img)
    stream = b"".join(zlib.decompress(img[o + 18:o + l - 8], -15) for o, l in blocks)
    h = bam_header_len(stream)
    recs, _ = orc_bam_unpack_all(stream[h:])
    want = ref_bam_write1_all(path)
    assert orc_pack(recs) == want
    assert want == stream[h:]            # a read/write round trip reproduces the record stream


@pytest.mark.gpu
def test_gpu_unpack_pack_roundtrip():
    import torch
    ctx = H.Context(0)
    stream, offs = synth.bam_records(21, 4000)
    for body in (stream, open(os.path.join(GOLD, "htslib", "range.bam"), "rb").read()):
        if body[:2] == b"\x1f\x8b":
            _, blocks = orc_bgzf_scan(body)
            s = b"".join(zlib.decompress(body[o + 18:o + l - 8], -15) for o, l in blocks)
            body = s[bam_header_len(s):]
        d = torch.from_numpy(np.frombuffer(body + b"\0" * 8, dtype=np.uint8).copy()).cuda()
        r = ctx.bam_unpack_dev(d, len(body), None, False)
        out, out_off, st = ctx.bam_pack_dev(r["core"], r["data"], r["data_off"], r["n"])
        torch.cuda.synchronize()
        assert int(st.abs().sum()) == 0
        got = out.cpu().numpy().tobytes()
        assert got == body
        recs, _ = orc_bam_unpack_all(body)
        assert got == orc_pack(recs)
    ctx.close()
