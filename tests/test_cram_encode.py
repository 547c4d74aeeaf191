"""CRAM record ENCODE (htslib_b200/csrc/cram_encode.cuh/.cu): bam1_t records -> a CRAM 3.x file that the compiled REFERENCE reads back
(sam_read1) to the input records — field for field and byte for byte, up to what CRAM cannot hold ('=' / 'X' CIGAR ops -> 'M',
MAPQ of unmapped reads -> 0, RNEXT of unpaired reads -> '*'), and that our own record decoder reads back identically.

`-m gpu`: hgpu_cram_encode_records_host (count / scan / write kernels, blocks through the device codecs).  Without a GPU the same
source runs through tests/hostsim (kernels -> loops, blocks stored RAW)."""
import ctypes as C
import os
import struct
import numpy as np
import pytest
import htslib_b200 as H
from _libs import GOLD, ref, ref_read_sam_records, ref_cram_read_all
import test_cram_records as T

HT = os.path.join(GOLD, "htslib")
SAMS = sorted(f[:-4] for f in os.listdir(os.path.join(HT, "sam")) if f.endswith(".sam"))
NAMES = [f for f, _ in H.BAM1_CORE_DT]


def pack(records):
    n = len(records)
    core = np.zeros(max(1, n), dtype=np.dtype(H.BAM1_CORE_DT))
    off = np.zeros(n + 1, dtype=np.uint64)
    for i, (c, d) in enumerate(records):
        core[i] = c
        off[i + 1] = off[i] + len(d)
    data = np.frombuffer(b"".join(d for _, d in records) + b"\0" * 8, dtype=np.uint8).copy()
    return core, data, off


def sq_names(text):
    return [[f[3:] for f in line.split(b"\t") if f.startswith(b"SN:")][0] for line in text.split(b"\n") if line.startswith(b"@SQ\t")]


def encode(entry_ctx, text, records, rps, minor, fasta_path=None):
    core, data, off = pack(records)
    out, ln = C.c_void_p(), C.c_uint64(0)
    refs, keep = None, None
    if fasta_path:
        keep = H.load_fasta_upper(fasta_path, sq_names(text))
        refs = H.CramRefs()
        refs.bases = keep[0].ctypes.data; refs.off = keep[1].ctypes.data; refs.n_ref = len(keep[1]) - 1
    rp = C.byref(refs) if refs is not None else None
    if entry_ctx is None:
        so = T.hostsim()                                    # builds / refreshes the harness
        l = C.CDLL(os.path.join(T.HERE, "hostsim", "_build", "libcramrec_hostsim.so"))
        l.hostsim_cram_encode_records.argtypes = [C.c_char_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint32, C.c_int, C.c_void_p, C.c_void_p]
        l.hostsim_enc_last_error.restype = C.c_char_p
        rc = l.hostsim_cram_encode_records(text, len(text), core.ctypes.data, data.ctypes.data, off.ctypes.data, len(records), rp, rps, minor, C.byref(out), C.byref(ln))
        err = lambda: l.hostsim_enc_last_error().decode()
    else:
        L = H.lib()
        L.hgpu_cram_encode_records_host.argtypes = [C.c_void_p, C.c_char_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint32, C.c_int, C.c_void_p, C.c_void_p]
        rc = L.hgpu_cram_encode_records_host(entry_ctx.h, text, len(text), core.ctypes.data, data.ctypes.data, off.ctypes.data, len(records), rp, rps, minor, C.byref(out), C.byref(ln))
        err = H.last_error
    if rc != 0:
        return rc, err()
    img = C.string_at(out.value, ln.value)
    C.CDLL(None).free(C.c_void_p(out.value))
    return 0, img


def expected(c, d):
    """What CRAM can hold of a record (the documented normalisations)."""
    c = dict(zip(NAMES, c))
    d = bytearray(d)
    lq, nc = c["l_qname"], c["n_cigar"]
    for k in range(nc):
        w = struct.unpack_from("<I", d, lq + 4 * k)[0]
        if (w & 15) in (7, 8):
            struct.pack_into("<I", d, lq + 4 * k, (w & ~15) | 0)
    if c["flag"] & 4:
        c["qual"] = 0
    if not c["flag"] & 1:
        c["mtid"] = -1
    return tuple(c[f] for f in NAMES), bytes(d)


def roundtrip(tmp_path, entry_ctx, sam, rps, minor, with_ref=False):
    text, recs = ref_read_sam_records(os.path.join(HT, "sam", sam + ".sam"))
    fa = os.path.join(HT, sam.split("#")[0] + ".fa") if with_ref else None
    rc, img = encode(entry_ctx, text, recs, rps, minor, fa)
    if rc != 0:
        return rc, img
    out = str(tmp_path / ("%s.%d.%d.%d.cram" % (sam.replace("#", "_"), rps, minor, with_ref)))
    open(out, "wb").write(img)
    back = ref_cram_read_all(out, fa, 0)
    assert len(back) == len(recs), (sam, len(back), len(recs))
    for i, ((gc, gd), (wc, wd)) in enumerate(zip(back, recs)):
        ec, ed = expected(wc, wd)
        assert gc == ec, (sam, i, dict(zip(NAMES, gc)), dict(zip(NAMES, ec)))
        assert gd == ed, (sam, i, gd[:100], ed[:100])
    return 0, img


@pytest.mark.parametrize("rps,minor,with_ref", [(0, 0, False), (3, 1, False), (0, 1, True), (2, 0, True)])
@pytest.mark.parametrize("sam", SAMS)
def test_hostsim_reference_reads_back_what_we_wrote(tmp_path, sam, rps, minor, with_ref):
    rc, img = roundtrip(tmp_path, None, sam, rps, minor, with_ref)
    if rc != 0:
        assert rc == -6, (sam, rc, img)            # HGPU_CRAM_UNSUPPORTED: mapped reads without SEQ etc., by contract
        pytest.skip("left to the host library: " + img)
    if with_ref:
        return
    # and our own record decoder (hostsim) reads the file back to the same records
    arr = np.frombuffer(img, dtype=np.uint8).copy()
    blocks, udata, off = T.cpu_blocks(arr)
    got = H.cram_decode_records(None, arr, blocks, udata, off, None, b"x", 0, _entry=T.hostsim())
    out = str(tmp_path / "again.cram")
    open(out, "wb").write(img)
    want = ref_cram_read_all(out, None, 0)
    assert got["slice_status"].tolist() == [0] * len(got["slice_status"])
    for i, (wc, wd) in enumerate(want):
        assert tuple(int(got["core"][i][f]) for f in NAMES) == wc and got["data"][i] == wd, (sam, i)


@pytest.mark.skipif(ref() is None, reason="the 10 000 synthetic records come from the reference's SAM reader; oracle/_ref not built")
def test_hostsim_synthetic_10000_reads(tmp_path):
    sam = str(tmp_path / "syn.sam")
    n = T._synthetic_sam(sam, n=10000, seed=21)
    text, recs = ref_read_sam_records(sam)
    assert len(recs) == n
    sizes = {}
    for rps, minor, fa in ((0, 1, None), (1500, 0, None), (0, 1, os.path.join(HT, "ce.fa"))):
        rc, img = encode(None, text, recs, rps, minor, fa)
        assert rc == 0, img
        out = str(tmp_path / "syn.cram")
        open(out, "wb").write(img)
        back = ref_cram_read_all(out, fa, 0)
        assert len(back) == n
        for i, ((gc, gd), (wc, wd)) in enumerate(zip(back, recs)):
            ec, ed = expected(wc, wd)
            assert gc == ec and gd == ed, (i, dict(zip(NAMES, gc)), dict(zip(NAMES, ec)))
        sizes[(rps, fa is not None)] = len(img)
    # coded against the reference, the bases all but disappear (blocks are RAW here: ~100 bytes of bases per read become a few)
    assert sizes[(0, True)] < 0.75 * sizes[(0, False)], sizes


@pytest.mark.gpu
@pytest.mark.parametrize("minor", [0, 1])
def test_gpu_reference_reads_back_what_we_wrote(tmp_path, minor):
    ctx = H.Context(0)
    done = 0
    for sam in SAMS:
        for with_ref in (False, True):
            rc, img = roundtrip(tmp_path, ctx, sam, 3 if minor else 0, minor, with_ref)
            assert rc in (0, -6), (sam, rc, img)
            done += rc == 0
    assert done >= 60
    if ref() is None:                                       # the 10 000 synthetic records come from the reference's SAM reader
        ctx.close()
        return
    # a 10 000-read slice: compressed by the device codecs, smaller than the records, read back by the reference
    sam = str(tmp_path / "syn.sam")
    n = T._synthetic_sam(sam, n=10000, seed=21)
    text, recs = ref_read_sam_records(sam)
    raw = sum(len(d) + 32 for _, d in recs)
    for fa, bound in ((None, 0.45), (os.path.join(HT, "ce.fa"), 0.36)):
        rc, img = encode(ctx, text, recs, 0, minor, fa)
        assert rc == 0, img
        out = str(tmp_path / "syn.cram")
        open(out, "wb").write(img)
        back = ref_cram_read_all(out, fa, 0)
        assert len(back) == n
        for i, ((gc, gd), (wc, wd)) in enumerate(zip(back, recs)):
            ec, ed = expected(wc, wd)
            assert gc == ec and gd == ed, i
        assert len(img) < bound * raw, (fa, len(img), raw)
    rc, img = encode(ctx, text, recs, 0, minor, None)
    blocks, _ = H.cram_scan_blocks(np.frombuffer(img, dtype=np.uint8).copy())
    methods = set(int(m) for m in blocks["method"])
    assert (5 in methods and 8 in methods) if minor else (4 in methods), methods
    ctx.close()
