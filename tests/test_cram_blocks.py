"""Real CRAM 3.1 blocks written by the reference encoder (tests/golden/make_cram.py): the host
scanner must list the blocks exactly as the reference reads them, and every RANS_PR block must
decode on the GPU to what the reference's / oracle's decoder gives (the per-block work of
cram_uncompress_block inside cram_decode_slice)."""
import collections, os
import numpy as np
import pytest
import htslib_b200 as H
from _libs import GOLD, orc_rans_nx16_decode, ref, ref_rans_nx16_decode

V31 = os.path.join(GOLD, "htslib", "ce#1000.v31.cram")


def test_scan_matches_expected_structure():
    img = np.fromfile(V31, dtype=np.uint8)
    blocks, ver = H.cram_scan_blocks(img)
    assert ver == (3, 1)
    c = collections.Counter(blocks["method"].tolist())
    assert c[5] == 14 and c[8] == 1                       # 14 rANS-Nx16 blocks, 1 tok3 (read names)
    assert int(blocks["container"].max()) == 2            # header, one data container, EOF container
    qs = blocks[(blocks["method"] == 5) & (blocks["uncomp_size"] == 100000)]
    assert len(qs) == 1 and img[int(qs[0]["data_off"])] == 0x45   # QS: 32-way | order-1 | RLE
    # every rANS payload must decode with the oracle to exactly uncomp_size bytes
    for b in blocks[blocks["method"] == 5]:
        comp = img[int(b["data_off"]):int(b["data_off"]) + int(b["comp_size"])].tobytes()
        out = orc_rans_nx16_decode(comp, int(b["uncomp_size"]))
        assert out is not None and len(out) == int(b["uncomp_size"])
        assert ref_rans_nx16_decode(comp, int(b["uncomp_size"])) == out
    bad = img.copy(); bad[0] = ord("X")
    with pytest.raises(H.HgpuError):
        H.cram_scan_blocks(bad)


@pytest.mark.gpu
def test_all_rans_blocks_decode_on_gpu():
    img = np.fromfile(V31, dtype=np.uint8)
    blocks, _ = H.cram_scan_blocks(img)
    rb = blocks[blocks["method"] == 5]
    ctx = H.Context(0)
    in_off = rb["data_off"].astype(np.uint64); in_len = rb["comp_size"].astype(np.uint32)
    out_len = rb["uncomp_size"].astype(np.uint32)
    out_off = np.concatenate([[0], np.cumsum(out_len.astype(np.int64))[:-1]]).astype(np.uint64)
    out = np.zeros(int(out_len.sum()) + 8, dtype=np.uint8)
    got, st = ctx.rans_nx16_decode_host(img, in_off, in_len, out, out_off, out_len)
    assert st.tolist() == [0] * len(rb) and got.tolist() == out_len.tolist()
    for i, b in enumerate(rb):
        comp = img[int(b["data_off"]):int(b["data_off"]) + int(b["comp_size"])].tobytes()
        want = orc_rans_nx16_decode(comp, int(b["uncomp_size"]))
        assert out[int(out_off[i]):int(out_off[i]) + int(out_len[i])].tobytes() == want, i
    ctx.close()


def _expect(img, b):
    """What cram_uncompress_block leaves in b->data, from the per-codec checkers (None = not checked here)."""
    import _libs as L
    comp = img[int(b["data_off"]):int(b["data_off"]) + int(b["comp_size"])].tobytes()
    m, us = int(b["method"]), int(b["uncomp_size"])
    if us == 0: return b""
    if m == 0: return comp[:us]
    if m == 1: return __import__("zlib").decompress(comp, 31)
    if m == 4: return L.orc_rans_4x8_decode(comp, us)
    if m == 5: return L.orc_rans_nx16_decode(comp, us)
    if m == 6:
        out = L.orc_arith_decode(comp, us)
        assert out == L.ref_arith(comp=comp, cap=us)
        return out
    if m == 7:
        out = L.orc_fqz_decode(comp)
        assert out == L.ref_fqz_decompress(comp)
        return out
    if m == 8: return L.orc_tok3_decode(comp)
    return None


FOREIGN = ["auxf#values_java.cram", "ce#5b_java.cram", "xx#large_aux_java.cram", "range.cram"]   # the reference's own test/*.cram


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["ce#1000.v31.cram", "ce#1000.v30.cram", "ce#1000.v31arith.cram", "ce#1000.v31fqz.cram"] + FOREIGN)
def test_uncompress_all_blocks_in_one_call(name):
    img = np.fromfile(os.path.join(GOLD, "htslib", name), dtype=np.uint8)
    ctx = H.Context(0)
    blocks, res = H.cram_uncompress_blocks(ctx, img)
    seen = collections.Counter()
    for b, (st, data) in zip(blocks, res):
        m = int(b["method"])
        if m in (2, 3) or (m == 1 and (int(b["uncomp_size"]) > 65536 or int(b["comp_size"]) + 8 > 65536)):
            assert st == -6                              # HGPU_CRAM_UNSUPPORTED: stays with the host library
            continue
        want = _expect(img, b)
        assert st == 0, (m, int(b["content_id"]))
        if want is not None:
            assert data == want, (m, int(b["content_id"]))
            seen[m] += 1
    if name.endswith("v31.cram"): assert seen[5] == 14 and seen[8] == 1
    if name.endswith("v30.cram"): assert seen[4] == 9
    if name.endswith("arith.cram"): assert seen[6] == 30 and seen[8] == 4
    if name.endswith("fqz.cram"): assert seen[7] == 1
    # one flipped payload bit: that block fails its CRC (cram_io.c:1585-1592), every other block is unaffected
    victim = int(np.argmax(blocks["comp_size"]))
    bad = img.copy(); bad[int(blocks[victim]["data_off"]) + 5] ^= 0x10
    _, res2 = H.cram_uncompress_blocks(ctx, bad, blocks)
    for i, ((st, data), (st0, data0)) in enumerate(zip(res2, res)):
        if i == victim: assert st == -2
        else: assert (st, data) == (st0, data0)
    ctx.close()


@pytest.mark.parametrize("name", FOREIGN)
def test_scan_foreign_writer_files(name):
    """CRAM 3.0 files written by htsjdk (and range.cram), from the reference's test/: the host scanner must walk
    them, every block's stored CRC-32 must match header+payload, and every block must decode with the oracle to
    its uncomp_size (they include empty RANS blocks: comp_size = uncomp_size = 0)."""
    import zlib
    import _libs as L
    img = np.fromfile(os.path.join(GOLD, "htslib", name), dtype=np.uint8)
    blocks, ver = H.cram_scan_blocks(img)
    assert ver == (3, 0) and len(blocks) > 10
    for b in blocks:
        o, cs, us, hl = int(b["data_off"]), int(b["comp_size"]), int(b["uncomp_size"]), int(b["hdr_len"])
        comp = img[o:o + cs].tobytes()
        assert zlib.crc32(img[o - hl:o + cs].tobytes()) == int.from_bytes(img[o + cs:o + cs + 4].tobytes(), "little")
        want = _expect(img, b)
        assert want is not None and len(want) == us, (int(b["method"]), cs, us)
        if int(b["method"]) == 4 and us:         # the oracle agrees with the reference on foreign rANS streams
            assert L.ref_rans_4x8(comp=comp) == want


def test_scanners_survive_corrupt_images():
    """The host scanners read untrusted files: on 3000 corrupted / truncated images they must return a block list
    or raise, never read out of bounds (this test dies with the interpreter if they do)."""
    import random
    from _libs import bgzf_file
    rng = random.Random(99)
    crams = [np.fromfile(os.path.join(GOLD, "htslib", n), dtype=np.uint8) for n in ["ce#1000.v31.cram", "ce#5b_java.cram", "range.cram"]]
    for trial in range(2000):
        img = crams[trial % 3].copy()
        for _ in range(rng.randrange(1, 6)):
            img[rng.randrange(0, min(len(img), 3000) if trial % 2 else len(img))] = rng.randrange(256)
        if trial % 5 == 0:
            img = img[: rng.randrange(1, len(img))].copy()
        try:
            blocks, _ = H.cram_scan_blocks(img)
            for b in blocks:                                     # whatever is listed must lie inside the image
                assert int(b["data_off"]) + int(b["comp_size"]) + 4 <= len(img) and int(b["data_off"]) >= int(b["hdr_len"])
        except H.HgpuError:
            pass
    bg = np.frombuffer(bgzf_file(bytes(rng.randrange(256) for _ in range(100000)), 6, block=9000), dtype=np.uint8)
    for trial in range(1000):
        img = bg.copy()
        for _ in range(rng.randrange(1, 4)):
            img[rng.randrange(len(img))] = rng.randrange(256)
        if trial % 4 == 0:
            img = img[: rng.randrange(1, len(img))].copy()
        try:
            off, ln, _ = H.bgzf_scan(img)
            assert all(int(o) + int(l) <= len(img) for o, l in zip(off, ln))
        except H.HgpuError:
            pass
