"""CRAI index building (htslib_b200/csrc/cram_index.cu / .cuh) against the compiled reference's sam_index_build3(fn, fnidx, 0, 0):
its return code and the inflated .crai text, on reference-written and device-written CRAM files and on damaged copies.

Without a GPU the index logic runs through tests/hostsim (the walk, the multi-reference record decode and slice_runs built for the
host); test_gpu_cram_index.py runs hgpu_cram_index_build_host on the same files."""
import ctypes as C
import os
import random
import struct
import subprocess
import tempfile
import zlib
import numpy as np
import pytest
import htslib_b200 as H
from _libs import GOLD, _ref_write_cram_to, ref, ref_read_sam_records, stored_reference
import test_cram_records as T
from test_cram_blocks import _expect
from test_cram_mates import encode

HT = os.path.join(GOLD, "htslib")
GOLDEN = ["ce#1000.v30.cram", "ce#1000.v31.cram", "ce#1000.v31arith.cram", "ce#1000.v31fqz.cram", "range.cram", "ce#5b_java.cram",
          "xx#large_aux_java.cram", "auxf#values_java.cram"]
MULTI, SEQS = 10, 3                                   # CRAM_OPT_MULTI_SEQ_PER_SLICE, CRAM_OPT_SEQS_PER_SLICE
REF_RC = {0: H.HGPU_OK, -1: H.IDX_ERR_READ, -2: H.IDX_ERR_PUSH}


@stored_reference(limit=200000)
def ref_cram_index(img):
    """(sam_index_build3 return code, inflated .crai text or None) for a CRAM image."""
    r = ref()
    r.sam_index_build3.argtypes = [C.c_char_p, C.c_char_p, C.c_int, C.c_int]
    with tempfile.TemporaryDirectory() as td:
        fn, fi = os.path.join(td, "x.cram"), os.path.join(td, "x.cram.crai")
        with open(fn, "wb") as f:
            f.write(img)
        rc = r.sam_index_build3(fn.encode(), fi.encode(), 0, 0)
        text = None
        if rc == 0:
            with open(fi, "rb") as f:
                text = zlib.decompressobj(31).decompress(f.read())
        return rc, text


@stored_reference(limit=100000)
def ref_crai_written_cram(sam_path, fasta, version, int_opts):
    """(records written, file image): sam_path written as CRAM by the reference's writer (hts_open "wc", sam_write1)."""
    with tempfile.TemporaryDirectory() as td:
        out = os.path.join(td, "out.cram")
        n = _ref_write_cram_to(sam_path, fasta, out, version, int_opts)
        with open(out, "rb") as f:
            return n, f.read()


@stored_reference(limit=20000)
def ref_crai_sam_records(path):
    """(header text, [(core tuple, data bytes)]) of a generated SAM file through the reference's sam_read1."""
    return ref_read_sam_records.__wrapped__(path)


# ---- the files ----

def _sq_fasta(path, n_sq, length, seed):
    rng = random.Random(seed)
    seqs = ["".join(rng.choice("ACGT") for _ in range(length)) for _ in range(n_sq)]
    with open(path, "w") as f:
        for i, s in enumerate(seqs):
            f.write(">s%d\n%s\n" % (i, s))
    return seqs


def _sorted_sam(path, seqs, per_sq, seed, unmapped=0, unsorted_at=None):
    """Sorted 50 bp reads over every @SQ (mapped, one insertion in some), then `unmapped` unplaced reads."""
    rng = random.Random(seed)
    lines = ["@HD\tVN:1.4\tSO:coordinate"] + ["@SQ\tSN:s%d\tLN:%d" % (i, len(s)) for i, s in enumerate(seqs)]
    k = 0
    for i, s in enumerate(seqs):
        pos = sorted(rng.randrange(1, len(s) - 60) for _ in range(per_sq))
        if unsorted_at is not None and i == 0:
            pos[unsorted_at], pos[unsorted_at + 1] = pos[unsorted_at] + 40, pos[unsorted_at]
        for p in pos:
            cig = "20M2I28M" if rng.random() < 0.2 else "50M"
            seq = s[p - 1:p + 49]
            if cig != "50M":
                seq = seq[:20] + "AC" + seq[20:48]
            lines.append("r%d\t0\ts%d\t%d\t60\t%s\t*\t0\t0\t%s\t%s" % (k, i, p, cig, seq, "I" * 50))
            k += 1
    for _ in range(unmapped):
        lines.append("u%d\t4\t*\t0\t0\t*\t*\t0\t0\t%s\t%s" % (k, "".join(rng.choice("ACGT") for _ in range(50)), "I" * 50))
        k += 1
    with open(path, "w") as f:
        f.write("\n".join(lines) + "\n")


def reference_written(tmp_path, key):
    """CRAM images the reference's writer makes with several references per slice."""
    fa, sam = str(tmp_path / "m.fa"), str(tmp_path / "m.sam")
    if key == "auto_multi":                           # many short @SQ, default options: the writer goes multi-reference by itself
        seqs = _sq_fasta(fa, 60, 400, 1)
        _sorted_sam(sam, seqs, 3, 2)
        opts = []
    elif key == "multi_unmapped":                     # CRAM_OPT_MULTI_SEQ_PER_SLICE = 1 and unplaced reads at the end
        seqs = _sq_fasta(fa, 8, 3000, 3)
        _sorted_sam(sam, seqs, 40, 4, unmapped=30)
        opts = [(MULTI, 1), (SEQS, 100)]
    elif key == "unsorted_containers":                # one container per 20 records, two containers out of order on s0
        seqs = _sq_fasta(fa, 2, 20000, 5)
        _sorted_sam(sam, seqs, 200, 6)
        opts = [(SEQS, 20)]
    _, img = ref_crai_written_cram(sam, fa, "3.1", [list(o) for o in opts])
    if key == "unsorted_containers":
        img = _swap_containers(img, 2, 3)
    return img


def device_written(key, tmp_path=None):
    """CRAM images the device writer's hostsim build makes: every slice multi-reference (ref_seq_id -2)."""
    text, recs = ref_read_sam_records(os.path.join(HT, "sam", "ce#5.sam" if key != "mates" else "xx#pair.sam"))
    if key == "ref":
        img, _ = encode(None, text, recs, 2, 1, os.path.join(HT, "ce.fa"), flags=0)
    elif key == "noref":
        img, _ = encode(None, text, recs, 2, 0, None, flags=0)
    elif key == "mates":
        img, _ = encode(None, text, recs, 0, 1, None)
    elif key == "unsorted_slice":                     # records out of order inside a multi-reference slice
        fa, sam = str(tmp_path / "u.fa"), str(tmp_path / "u.sam")
        _sorted_sam(sam, _sq_fasta(fa, 3, 3000, 7), 30, 8, unsorted_at=10)
        text, recs = ref_crai_sam_records(sam)
        img, _ = encode(None, text, recs, 0, 1, None, flags=0)
    return img


# ---- damage ----

def _itf8(b, p):
    c = b[p]
    n = 0 if c < 0x80 else 1 if c < 0xc0 else 2 if c < 0xe0 else 3 if c < 0xf0 else 4
    if n == 0: v = c
    elif n == 1: v = ((c & 0x3f) << 8) | b[p + 1]
    elif n == 2: v = ((c & 0x1f) << 16) | (b[p + 1] << 8) | b[p + 2]
    elif n == 3: v = ((c & 0x0f) << 24) | (b[p + 1] << 16) | (b[p + 2] << 8) | b[p + 3]
    else: v = ((c & 0x0f) << 28) | (b[p + 1] << 20) | (b[p + 2] << 12) | (b[p + 3] << 4) | (b[p + 4] & 0x0f)
    return v, p + n + 1


def containers(img):
    """[(start, landmark field offsets, crc offset, end)] of every container after the file definition."""
    out, p = [], 26
    while p < len(img):
        s = p
        length = struct.unpack_from("<i", img, p)[0]
        p += 4
        for _ in range(4):
            _, p = _itf8(img, p)
        for _ in range(2):                            # LTF8 record counter, bases
            c, n = img[p], 0
            while n < 8 and (c << n) & 0x80:
                n += 1
            p += n + 1
        _, p = _itf8(img, p)
        nl, p = _itf8(img, p)
        lms = []
        for _ in range(nl):
            lms.append(p)
            _, p = _itf8(img, p)
        out.append((s, lms, p, p + 4 + length))
        p += 4 + length
    return out


def _recrc(b, start, crc_at):
    struct.pack_into("<I", b, crc_at, zlib.crc32(bytes(b[start:crc_at])))


def _swap_containers(img, i, j):
    cs = containers(img)
    a, b = cs[i], cs[j]
    assert b[0] == a[3]
    return img[:a[0]] + img[b[0]:b[3]] + img[a[0]:a[3]] + img[b[3]:]


def wrong_landmark(img):
    b = bytearray(img)
    s, lms, crc_at, _ = containers(img)[1]
    v, q = _itf8(b, lms[0])
    assert q - lms[0] == (1 if v + 1 < 0x80 else 2)
    b[lms[0]:q] = bytes([v + 1]) if v + 1 < 0x80 else bytes([0x80 | ((v + 1) >> 8), (v + 1) & 0xff])
    _recrc(b, s, crc_at)
    return bytes(b)


def wrong_length(img):
    b = bytearray(img)
    s, _, crc_at, _ = containers(img)[1]
    struct.pack_into("<i", b, s, struct.unpack_from("<i", b, s)[0] + 1)
    _recrc(b, s, crc_at)
    return bytes(b)


def bad_crc(img, pick):
    """img with the CRC of the block pick(blocks) chose flipped."""
    blocks, _ = H.cram_scan_blocks(np.frombuffer(img, np.uint8).copy())
    k = pick(blocks)
    b = bytearray(img)
    at = int(blocks[k]["data_off"]) + int(blocks[k]["comp_size"])
    b[at] ^= 0x5a
    return bytes(b)


def _first_core(blocks):
    return [i for i, b in enumerate(blocks) if int(b["content_type"]) == 5][0]


def _single_ref_data_block(blocks):
    """the last external block of the file: a data block only decoding would read"""
    return [i for i, b in enumerate(blocks) if int(b["content_type"]) == 4][-1]


def cases(tmp_path):
    out = [(g, open(os.path.join(HT, g), "rb").read()) for g in GOLDEN]
    for key in ("auto_multi", "multi_unmapped", "unsorted_containers"):
        out.append((key, reference_written(tmp_path, key)))
    for key in ("ref", "noref", "mates", "unsorted_slice"):
        out.append(("device_" + key, device_written(key, tmp_path)))
    dev = device_written("noref")
    v30 = open(os.path.join(HT, "ce#1000.v30.cram"), "rb").read()
    out += [("crc_multiref", bad_crc(dev, _first_core)), ("crc_single_ref_data", bad_crc(v30, _single_ref_data_block)),
            ("wrong_landmark", wrong_landmark(v30)), ("wrong_length", wrong_length(v30)), ("truncated", v30[:len(v30) * 6 // 10]),
            ("wrong_landmark_multiref", wrong_landmark(dev)), ("truncated_multiref", dev[:len(dev) * 7 // 10])]
    return out


CASE_NAMES = GOLDEN + ["auto_multi", "multi_unmapped", "unsorted_containers", "device_ref", "device_noref", "device_mates",
                       "device_unsorted_slice", "crc_multiref", "crc_single_ref_data", "wrong_landmark", "wrong_length", "truncated",
                       "wrong_landmark_multiref", "truncated_multiref"]


# ---- the host build ----

def hostsim_index(img, base=None):
    """(rc, bad, text) of the hostsim index build.  base: the undamaged image the blocks are uncompressed from (same offsets)."""
    srcs = [os.path.join(T.HERE, "..", "htslib_b200", "csrc", f)
            for f in ("cram_index.cu", "cram_index.cuh", "cram_records.cu", "cram_records.cuh", "cram_encode.cu", "cram_encode.cuh")]
    so = os.path.join(T.HERE, "hostsim", "_build", "libcramidx_hostsim.so")
    if not os.path.exists(so) or os.path.getmtime(so) < max(os.path.getmtime(f) for f in srcs):
        subprocess.check_call(["bash", os.path.join(T.HERE, "hostsim", "build_index.sh")], stdout=subprocess.DEVNULL)
    l = C.CDLL(so)
    l.hostsim_cram_index_text.argtypes = [C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p,
                                          C.POINTER(C.c_void_p), C.POINTER(C.c_uint64), C.POINTER(C.c_int64)]
    base = np.frombuffer(base if base is not None else img, np.uint8).copy()
    arr = np.frombuffer(img, np.uint8).copy()
    blocks, _ = H.cram_scan_blocks(base)
    sizes = blocks["uncomp_size"].astype(np.int64)
    off = np.concatenate([[0], np.cumsum((sizes + 15) // 16 * 16)]).astype(np.uint64)
    udata = np.zeros(int(off[-1]) + 16, dtype=np.uint8)
    status = np.zeros(len(blocks) + 1, dtype=np.int32)
    for i, b in enumerate(blocks):
        want = _expect(base, b)
        udata[int(off[i]):int(off[i]) + len(want)] = np.frombuffer(want, dtype=np.uint8)
        h0, e = int(b["data_off"]) - int(b["hdr_len"]), int(b["data_off"]) + int(b["comp_size"])
        if e + 4 <= len(arr) and zlib.crc32(arr[h0:e].tobytes()) != struct.unpack_from("<I", arr, e)[0]:
            status[i] = -2                            # HGPU_CRAM_ERR_CRC
    text, n, bad = C.c_void_p(), C.c_uint64(0), C.c_int64(0)
    rc = l.hostsim_cram_index_text(arr.ctypes.data, len(arr), blocks.ctypes.data, len(blocks), udata.ctypes.data, off.ctypes.data,
                                   status.ctypes.data, C.byref(text), C.byref(n), C.byref(bad))
    t = C.string_at(text.value, n.value)
    C.CDLL(None).free(C.c_void_p(text.value))
    return rc, bad.value, t


BASE_OF = {"crc_multiref": "device_noref", "crc_single_ref_data": "ce#1000.v30.cram", "wrong_landmark": "ce#1000.v30.cram",
           "wrong_length": "ce#1000.v30.cram", "truncated": "ce#1000.v30.cram", "wrong_landmark_multiref": "device_noref",
           "truncated_multiref": "device_noref"}


@pytest.mark.parametrize("name", CASE_NAMES)
def test_hostsim_index_equals_reference(tmp_path, name):
    all_cases = dict(cases(tmp_path))
    img = all_cases[name]
    want_rc, want_text = ref_cram_index(img)
    base = all_cases[BASE_OF[name]] if name in BASE_OF else None
    rc, bad, text = hostsim_index(img, base)
    assert rc == REF_RC[want_rc], (name, rc, bad, want_rc)
    if want_rc == 0:
        assert text == want_text, (name, text[:300], want_text[:300])


def test_the_damage_is_where_it_is_meant_to_be(tmp_path):
    """Each damaged file is refused (or accepted) for the reason it was made for, at the slice it was made at."""
    c = dict(cases(tmp_path))
    expect = {"unsorted_containers": (H.IDX_ERR_PUSH, None), "device_unsorted_slice": (H.IDX_ERR_READ, 0),
              "crc_multiref": (H.IDX_ERR_READ, 0), "crc_single_ref_data": (H.HGPU_OK, None), "wrong_landmark": (H.IDX_ERR_READ, 0),
              "wrong_length": (H.IDX_ERR_READ, 1), "wrong_landmark_multiref": (H.IDX_ERR_READ, 0)}
    for name, (code, at) in expect.items():
        base = c[BASE_OF[name]] if name in BASE_OF else None
        rc, bad, _ = hostsim_index(c[name], base)
        assert rc == code, (name, rc, bad)
        if at is not None:
            assert bad == at, (name, bad)
