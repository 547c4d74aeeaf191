"""The host reader of CRAM compression headers (hgpu_cram_parse_compression_header) against the compiled
reference: for every container of every CRAM fixture the description it prints must be the lines
cram_describe_encodings prints (the reference walks tags in hash order, so lines are compared as sets), and
the external block ids it reports must be the ones in that text."""
import ctypes as C
import os
import re
import zlib

import numpy as np
import pytest

import htslib_b200 as H
import _libs as L

FILES = ["ce#1000.v31.cram", "ce#1000.v30.cram", "ce#1000.v31arith.cram", "ce#1000.v31fqz.cram",
         "auxf#values_java.cram", "ce#5b_java.cram", "xx#large_aux_java.cram", "range.cram"]


class KS(C.Structure):
    _fields_ = [("l", C.c_size_t), ("m", C.c_size_t), ("s", C.c_char_p)]


@L.stored_reference(limit=60000)
def ref_cram_descriptions(path):
    """cram_describe_encodings of every container's compression header."""
    r = L.ref()
    r.cram_open.restype = C.c_void_p; r.cram_open.argtypes = [C.c_char_p, C.c_char_p]
    r.cram_close.argtypes = [C.c_void_p]
    r.cram_read_container.restype = C.c_void_p; r.cram_read_container.argtypes = [C.c_void_p]
    r.cram_read_block.restype = C.c_void_p; r.cram_read_block.argtypes = [C.c_void_p]
    r.cram_uncompress_block.argtypes = [C.c_void_p]
    r.cram_decode_compression_header.restype = C.c_void_p; r.cram_decode_compression_header.argtypes = [C.c_void_p, C.c_void_p]
    r.cram_describe_encodings.argtypes = [C.c_void_p, C.POINTER(KS)]
    r.cram_container_get_num_blocks.restype = C.c_int32; r.cram_container_get_num_blocks.argtypes = [C.c_void_p]
    r.cram_block_get_content_type.argtypes = [C.c_void_p]
    fd = r.cram_open(path.encode(), b"r")
    assert fd
    out = []
    while True:
        c = r.cram_read_container(fd)
        if not c:
            break
        nb = r.cram_container_get_num_blocks(c)
        for k in range(nb):
            b = r.cram_read_block(fd)
            assert b
            if k == 0 and r.cram_block_get_content_type(b) == 1:
                assert r.cram_uncompress_block(b) == 0
                h = r.cram_decode_compression_header(fd, b)
                assert h
                ks = KS(0, 0, None)
                assert r.cram_describe_encodings(h, C.byref(ks)) == 0
                out.append((ks.s or b"").decode())
    r.cram_close(fd)
    return out


@pytest.mark.parametrize("name", FILES)
def test_description_equals_reference(name):
    path = os.path.join(L.GOLD, "htslib", name)
    want = ref_cram_descriptions(path)
    img = np.fromfile(path, dtype=np.uint8)
    blocks, ver = H.cram_scan_blocks(img)
    got = []
    for b in blocks[blocks["content_type"] == 1]:
        comp = img[int(b["data_off"]):int(b["data_off"]) + int(b["comp_size"])].tobytes()
        payload = comp if int(b["method"]) == 0 else zlib.decompress(comp, 31)
        series, text = H.cram_parse_compression_header(payload, ver[0])
        got.append(text)
        ids = [int(x) for x in re.findall(r"id=(-?\d+)", text)]
        assert sorted(i for s in series for i in s["id"].tolist() if i >= 0) == sorted(ids)
        assert len(series) == len(text.splitlines())
    assert len(got) == len(want) and len(got) >= 1
    for g, w in zip(got, want):
        assert sorted(g.splitlines()) == sorted(w.splitlines())
        assert g.splitlines()[:5] == w.splitlines()[:5]          # data series come first, in the reference's order


def test_rejects_garbage():
    img = np.fromfile(os.path.join(L.GOLD, "htslib", "ce#1000.v31.cram"), dtype=np.uint8)
    blocks, _ = H.cram_scan_blocks(img)
    b = blocks[blocks["content_type"] == 1][0]
    comp = img[int(b["data_off"]):int(b["data_off"]) + int(b["comp_size"])].tobytes()
    payload = bytearray(comp if int(b["method"]) == 0 else zlib.decompress(comp, 31))
    import random
    rng = random.Random(3)
    for trial in range(500):
        p = bytearray(payload)
        for _ in range(rng.randrange(1, 4)):
            p[rng.randrange(len(p))] = rng.randrange(256)
        if trial % 3 == 0:
            p = p[: rng.randrange(0, len(p))]
        try:
            H.cram_parse_compression_header(bytes(p))
        except H.HgpuError:
            pass


@pytest.mark.parametrize("name", FILES)
def test_containers_and_slices_equal_reference(name):
    """Every container header field the reference exposes (htslib/cram.h:190-216) and every slice header field
    (:418-441) must match what the host tables report; the block list and the container table must agree."""
    path = os.path.join(L.GOLD, "htslib", name)
    img = np.fromfile(path, dtype=np.uint8)
    cont, lm = H.cram_scan_containers(img)
    blocks, ver = H.cram_scan_blocks(img)
    assert int(cont["n_blocks"].sum()) == len(blocks)
    for i, c in enumerate(cont):
        mine = blocks[blocks["container"] == i]
        assert len(mine) == int(c["n_blocks"])
        if len(mine):
            assert int(np.where(blocks["container"] == i)[0][0]) == int(c["first_block"])
            assert int(mine[0]["data_off"]) - int(mine[0]["hdr_len"]) == int(c["data_off"])
    slices = 0
    ci, bi = 1, int(cont[0]["n_blocks"])
    for length, n_blocks, n_records, bases, landmarks, coords, slice_hdrs in ref_cram_containers(path):
        m = cont[ci]
        assert length == int(m["length"])
        assert n_blocks == int(m["n_blocks"])
        assert n_records == int(m["n_records"])
        assert bases == int(m["bases"])
        assert len(landmarks) == int(m["n_landmarks"])
        assert landmarks == lm[int(m["landmark0"]):int(m["landmark0"]) + len(landmarks)].tolist()
        assert coords == (int(m["ref_id"]), int(m["start"]), int(m["span"]))
        for k in range(int(m["n_blocks"])):
            if k in slice_hdrs:
                h_blocks, h_embed, h_coords = slice_hdrs[k]
                x = blocks[bi]
                comp = img[int(x["data_off"]):int(x["data_off"]) + int(x["comp_size"])].tobytes()
                payload = comp if int(x["method"]) == 0 else zlib.decompress(comp, 31)
                s, ids = H.cram_parse_slice_header(payload, ver[0])
                assert h_blocks == int(s["n_blocks"])
                assert h_embed == int(s["ref_base_id"])
                assert h_coords == (int(s["ref_id"]), int(s["start"]), int(s["span"]))
                # the slice's external blocks carry exactly the content ids its header lists
                follow = blocks[bi + 1: bi + 1 + int(s["n_blocks"])]
                ext = follow[follow["content_type"] == 4]                  # the CORE block (type 5, id 0) is not listed
                assert sorted(int(v) for v in ext["content_id"]) == sorted(ids)
                slices += 1
            bi += 1
        ci += 1
    assert ci == len(cont) and slices >= 1


@L.stored_reference
def ref_cram_containers(path):
    """Per data container: (length, blocks, records, bases, landmarks, (ref id, start, span), {block index of a
    mapped slice header: (blocks, embedded reference id, (ref id, start, span))}) through the reference's accessors."""
    r = L.ref()
    r.cram_open.restype = C.c_void_p; r.cram_open.argtypes = [C.c_char_p, C.c_char_p]
    r.cram_close.argtypes = [C.c_void_p]
    r.cram_read_container.restype = C.c_void_p; r.cram_read_container.argtypes = [C.c_void_p]
    r.cram_read_block.restype = C.c_void_p; r.cram_read_block.argtypes = [C.c_void_p]
    r.cram_uncompress_block.argtypes = [C.c_void_p]
    r.cram_block_get_content_type.argtypes = [C.c_void_p]
    for f in ("cram_container_get_length", "cram_container_get_num_blocks", "cram_container_get_num_records"):
        getattr(r, f).restype = C.c_int32; getattr(r, f).argtypes = [C.c_void_p]
    r.cram_container_get_num_bases.restype = C.c_int64; r.cram_container_get_num_bases.argtypes = [C.c_void_p]
    r.cram_container_get_landmarks.restype = C.POINTER(C.c_int32); r.cram_container_get_landmarks.argtypes = [C.c_void_p, C.POINTER(C.c_int32)]
    r.cram_container_get_coords.argtypes = [C.c_void_p, C.POINTER(C.c_int), C.POINTER(C.c_int64), C.POINTER(C.c_int64)]
    r.cram_decode_slice_header.restype = C.c_void_p; r.cram_decode_slice_header.argtypes = [C.c_void_p, C.c_void_p]
    r.cram_slice_hdr_get_num_blocks.restype = C.c_int32; r.cram_slice_hdr_get_num_blocks.argtypes = [C.c_void_p]
    r.cram_slice_hdr_get_embed_ref_id.argtypes = [C.c_void_p]
    r.cram_slice_hdr_get_coords.argtypes = [C.c_void_p, C.POINTER(C.c_int), C.POINTER(C.c_int64), C.POINTER(C.c_int64)]
    fd = r.cram_open(path.encode(), b"r")                             # consumes container 0, the SAM header container
    out = []
    while True:
        c = r.cram_read_container(fd)
        if not c:
            break
        nl = C.c_int32(0)
        lp = r.cram_container_get_landmarks(c, C.byref(nl))
        rid, st, sp = C.c_int(0), C.c_int64(0), C.c_int64(0)
        r.cram_container_get_coords(c, C.byref(rid), C.byref(st), C.byref(sp))
        nb = r.cram_container_get_num_blocks(c)
        cont = [r.cram_container_get_length(c), nb, r.cram_container_get_num_records(c), r.cram_container_get_num_bases(c),
                [lp[k] for k in range(nl.value)], (rid.value, st.value, sp.value), {}]
        for k in range(nb):
            b = r.cram_read_block(fd)
            assert b
            if r.cram_block_get_content_type(b) == 2:                     # MAPPED_SLICE header
                assert r.cram_uncompress_block(b) == 0
                h = r.cram_decode_slice_header(fd, b)
                assert h
                r.cram_slice_hdr_get_coords(h, C.byref(rid), C.byref(st), C.byref(sp))
                cont[6][k] = (r.cram_slice_hdr_get_num_blocks(h), r.cram_slice_hdr_get_embed_ref_id(h), (rid.value, st.value, sp.value))
        out.append(tuple(cont))
    r.cram_close(fd)
    return out
