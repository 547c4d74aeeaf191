"""CRAM record decode of a field subset (CRAM_OPT_REQUIRED_FIELDS): the block and data-series selection of
cram_dependent_data_series and the gates of the record loop (htslib_b200/csrc/cram_records.cu / .cuh) against the compiled
reference's sam_read1 after hts_set_opt(fp, CRAM_OPT_REQUIRED_FIELDS, mask).

`-m gpu` runs hgpu_cram_decode_records_fields_host and hgpu_cram_decode_file_fields_host; without a GPU the same logic runs
through tests/hostsim (see test_cram_records.py)."""
import ctypes as C
import os
import random
import tempfile
import numpy as np
import pytest
import htslib_b200 as H
from _libs import Bam1, ref, stored_reference, _ref_write_cram_to
from test_cram_records import CASES, HT, SAMS, SHAPES, cpu_blocks, _mutations, _synthetic_sam, _written
from test_cram_records import hostsim as _hostsim_records

ALL = H.SAM_ALL
SINGLE = [1 << i for i in range(13)]
MASKS = SINGLE + [H.SAM_FLAG | H.SAM_MAPQ | H.SAM_RNEXT, H.SAM_RNAME | H.SAM_POS | H.SAM_CIGAR, H.SAM_SEQ | H.SAM_QUAL,
                  H.SAM_QNAME | H.SAM_SEQ | H.SAM_QUAL, ALL & ~H.SAM_QUAL, ALL & ~H.SAM_QNAME, ALL & ~H.SAM_AUX, 0]
REDUCED = [H.SAM_FLAG | H.SAM_MAPQ | H.SAM_RNEXT, H.SAM_RNAME | H.SAM_POS | H.SAM_CIGAR, H.SAM_SEQ | H.SAM_QUAL, ALL & ~H.SAM_QUAL, 0]
CORE_NAMES = [f for f, _ in H.BAM1_CORE_DT]


def _read_fields(path, fasta, decode_md, mask):
    """The records sam_read1 returns with CRAM_OPT_DECODE_MD = decode_md and CRAM_OPT_REQUIRED_FIELDS = mask: [(core, data)]."""
    r = ref()
    r.hts_open.restype = C.c_void_p
    r.hts_open.argtypes = [C.c_char_p, C.c_char_p]
    r.hts_close.argtypes = [C.c_void_p]
    r.sam_hdr_read.restype = C.c_void_p
    r.sam_hdr_read.argtypes = [C.c_void_p]
    r.sam_hdr_destroy.argtypes = [C.c_void_p]
    r.sam_read1.argtypes = [C.c_void_p, C.c_void_p, C.POINTER(Bam1)]
    r.bam_init1.restype = C.POINTER(Bam1)
    r.bam_destroy1.argtypes = [C.POINTER(Bam1)]
    r.hts_set_fai_filename.argtypes = [C.c_void_p, C.c_char_p]
    fp = r.hts_open(path.encode(), b"r")
    assert fp, path
    assert r.hts_set_fai_filename(fp, fasta.encode()) == 0
    r.hts_set_opt.argtypes = [C.c_void_p, C.c_int, C.c_int]
    r.hts_set_opt(fp, 0, int(decode_md))                       # CRAM_OPT_DECODE_MD
    r.hts_set_opt(fp, 18, int(mask))                           # CRAM_OPT_REQUIRED_FIELDS, hts.h:297-318
    hdr = r.sam_hdr_read(fp)
    assert hdr
    b = r.bam_init1()
    out, rc = [], 0
    while True:
        rc = r.sam_read1(fp, hdr, b)
        if rc < 0:
            break
        out.append((b.contents.core.astuple(), bytes(b.contents.data[: b.contents.l_data])))
    r.bam_destroy1(b)
    r.sam_hdr_destroy(hdr)
    r.hts_close(fp)
    return rc, out


def _pack(records):
    return b"".join(b"%r %d\n" % (tuple(core), len(data)) + data for core, data in records)


@stored_reference(digest=True)
def ref_cram_read_fields(path, fasta, decode_md, mask):
    """(sam_read1's last return code, record count, every core and data byte of the file) as _read_fields reads them."""
    rc, out = _read_fields(path, fasta, decode_md, mask)
    return rc, len(out), _pack(out)


def _ours(got):
    return [(tuple(int(got["core"][i][f]) for f in CORE_NAMES), got["data"][i]) for i in range(len(got["data"]))]


def compare(path, fa, got, decode_md, mask):
    want_rc, want_n, want = ref_cram_read_fields(path, os.path.join(HT, fa), decode_md, mask)
    assert want_rc == -1, (path, mask, want_rc)
    assert got["slice_status"].tolist() == [0] * len(got["slice_status"]), (path, mask, got["slice_status"].tolist())
    assert got["rec_status"].tolist() == [0] * len(got["rec_status"])
    mine = _ours(got)
    assert len(mine) == want_n, (path, mask, len(mine), want_n)
    if want != _pack(mine):
        detail = "first difference not known (oracle/_ref not built)"
        if ref() is not None:
            _, live = _read_fields(path, os.path.join(HT, fa), decode_md, mask)
            i = next(k for k in range(len(live)) if live[k] != mine[k])
            detail = "record %d: ours %r, reference %r" % (i, mine[i], live[i])
        raise AssertionError("%s mask %#x decode_md %d: %s" % (path, mask, decode_md, detail))


_hs = None


def hostsim():
    """(records entry, required-blocks entry) of the host build of cram_records.cu."""
    global _hs
    if _hs is None:
        _hostsim_records()                                     # builds tests/hostsim when its sources changed
        so = os.path.join(os.path.dirname(os.path.abspath(__file__)), "hostsim", "_build", "libcramrec_hostsim.so")
        l = C.CDLL(so)
        l.hostsim_cram_decode_records_fields.argtypes = [C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p,
                                                         C.c_char_p, C.c_int, C.c_uint32, C.c_void_p]
        l.hostsim_last_error.restype = C.c_char_p
        err = lambda: l.hostsim_last_error().decode()
        _hs = ((l.hostsim_cram_decode_records_fields, l.hostsim_cram_records_free, err), (l.hostsim_cram_required_blocks, err))
    return _hs


@stored_reference
def ref_synthetic_cram(sam_path, fasta, version, int_opts):
    """(records written, file image) of the reference's writer (hts_open "wc", sam_write1) for the synthetic SAM; stored
    whatever its size, so the synthetic cases run where the reference was never built."""
    with tempfile.TemporaryDirectory() as td:
        out_path = os.path.join(td, "out.cram")
        n = _ref_write_cram_to(sam_path, fasta, out_path, version, int_opts)
        with open(out_path, "rb") as f:
            return n, f.read()


def _synthetic(tmp_path, version, opts):
    sam = str(tmp_path / "syn.sam")
    n = _synthetic_sam(sam)
    out = str(tmp_path / "syn.cram")
    m, img = ref_synthetic_cram(sam, os.path.join(HT, "ce.fa"), version, [list(o) for o in opts], store_always=True)
    assert m == n
    with open(out, "wb") as f:
        f.write(img)
    return out


def _scrambled(blocks, udata, off, used):
    """udata with every block the selection does not use overwritten with 0xA5."""
    u2 = udata.copy()
    for i, b in enumerate(blocks):
        if not used[i]:
            u2[int(off[i]):int(off[i]) + int(b["uncomp_size"])] = 0xA5
    return u2


def _hostsim_case(path, fa, masks, prefix):
    img = np.fromfile(path, dtype=np.uint8)
    blocks, udata, off = cpu_blocks(img)
    fasta = H.load_fasta_upper(os.path.join(HT, fa), H.cram_sq_names(blocks, udata, off))
    rec_entry, blk_entry = hostsim()
    for mask in masks:
        used = H.cram_required_blocks(blocks, udata, off, mask, _entry=blk_entry)
        u2 = _scrambled(blocks, udata, off, used)
        for decode_md in (0, 1):
            got = H.cram_decode_records_fields(None, img, blocks, u2, off, fasta, prefix, decode_md, mask, _entry=rec_entry)
            compare(path, fa, got, decode_md, mask)


@pytest.mark.parametrize("name,fa", CASES)
def test_hostsim_fields_equal_reference(name, fa):
    """Every mask x decode_md on the CASES fixtures, with the blocks the selection leaves out overwritten: the gates never
    read a block the selection did not pick (the Java-written fixtures code their series on CORE)."""
    _hostsim_case(os.path.join(HT, name), fa, MASKS, name.encode())


def test_hostsim_fields_synthetic_10000_read_slice(tmp_path):
    _hostsim_case(_synthetic(tmp_path, "3.1", []), "ce.fa", MASKS, b"syn.cram")


@pytest.mark.parametrize("shape", sorted(SHAPES))
def test_hostsim_fields_written_by_reference(tmp_path, shape):
    for sam in SAMS:
        out, fa, n = _written(tmp_path, sam, shape)
        _hostsim_case(out, fa, REDUCED, os.path.basename(out).encode())


def test_all_fields_mask_reads_every_block():
    img = np.fromfile(os.path.join(HT, "ce#1000.v31.cram"), dtype=np.uint8)
    blocks, udata, off = cpu_blocks(img)
    _, blk_entry = hostsim()
    for mask in (0, ALL):
        assert H.cram_required_blocks(blocks, udata, off, mask, _entry=blk_entry).tolist() == [1] * len(blocks)
    flag = H.cram_required_blocks(blocks, udata, off, H.SAM_FLAG, _entry=blk_entry)
    assert 0 < flag.sum() < len(blocks)
    assert all(flag[i] for i in range(len(blocks)) if int(blocks[i]["content_type"]) in (0, 1, 2, 5))


def test_hostsim_no_reference_without_seq():
    name, fa = "ce#1000.v31.cram", "ce.fa"
    img = np.fromfile(os.path.join(HT, name), dtype=np.uint8)
    blocks, udata, off = cpu_blocks(img)
    rec_entry, _ = hostsim()
    for mask in (ALL & ~H.SAM_SEQ, H.SAM_FLAG | H.SAM_POS | H.SAM_CIGAR, H.SAM_QUAL):
        got = H.cram_decode_records_fields(None, img, blocks, udata, off, None, name.encode(), 1, mask, _entry=rec_entry)
        compare(os.path.join(HT, name), fa, got, 1, mask)
    got = H.cram_decode_records_fields(None, img, blocks, udata, off, None, name.encode(), 1, ALL, _entry=rec_entry)
    assert got["slice_status"].tolist() == [-7]                # with SEQ the slice needs the reference it was not given


@pytest.mark.parametrize("name", ["ce#5b_java.cram", "range.cram"])
def test_hostsim_fields_corrupt_series_never_run_wild(name):
    """The mutation harness of test_cram_records with a random mask per case: a status, never a crash."""
    rec_entry, blk_entry = hostsim()
    rng = random.Random(7)
    seen = set()
    for img, blocks, u2, off, fasta, md in _mutations(name, 60, 9):
        mask = rng.choice(MASKS + [rng.randrange(1 << 13)])
        try:
            H.cram_required_blocks(blocks, u2, off, mask, _entry=blk_entry)
            got = H.cram_decode_records_fields(None, img, blocks, u2, off, fasta, b"x", md, mask, _entry=rec_entry)
            assert set(got["slice_status"].tolist()) <= {0, -1, -4, -6, -7}
            for st, d in zip(got["rec_status"], got["data"]):
                assert st == 0 or d == b""
            seen |= set(got["slice_status"].tolist())
        except H.HgpuError:
            seen.add("call")
    assert 0 in seen and (-1 in seen or "call" in seen)


# ---- on the device ----

def _gpu_case(ctx, path, fa, masks, prefix):
    img = np.fromfile(path, dtype=np.uint8)
    blocks, res = H.cram_uncompress_blocks(ctx, img)
    sizes = blocks["uncomp_size"].astype(np.int64)
    off = np.concatenate([[0], np.cumsum((sizes + 15) // 16 * 16)]).astype(np.uint64)
    udata = np.zeros(int(off[-1]) + 16, dtype=np.uint8)
    for i, (st, data) in enumerate(res):
        assert st == 0, (i, st)
        udata[int(off[i]):int(off[i]) + len(data)] = np.frombuffer(data, dtype=np.uint8)
    off = off[:-1].copy()
    fasta = H.load_fasta_upper(os.path.join(HT, fa), H.cram_sq_names(blocks, udata, off))
    for mask in masks:
        used = H.cram_required_blocks(blocks, udata, off, mask)
        u2 = _scrambled(blocks, udata, off, used)
        for decode_md in (0, 1):
            compare(path, fa, H.cram_decode_records_fields(ctx, img, blocks, u2, off, fasta, prefix, decode_md, mask), decode_md, mask)
            compare(path, fa, H.cram_decode_file_fields(ctx, img, fasta, prefix, decode_md, mask), decode_md, mask)


@pytest.mark.gpu
@pytest.mark.parametrize("name,fa", CASES)
def test_gpu_fields_equal_reference(name, fa):
    ctx = H.Context(0)
    _gpu_case(ctx, os.path.join(HT, name), fa, MASKS, name.encode())
    ctx.close()


@pytest.mark.gpu
def test_gpu_fields_synthetic_10000_read_slice(tmp_path):
    ctx = H.Context(0)
    _gpu_case(ctx, _synthetic(tmp_path, "3.1", []), "ce.fa", MASKS, b"syn.cram")
    ctx.close()


@pytest.mark.gpu
@pytest.mark.parametrize("shape", sorted(SHAPES))
def test_gpu_fields_written_by_reference(tmp_path, shape):
    ctx = H.Context(0)
    for sam in SAMS:
        out, fa, n = _written(tmp_path, sam, shape)
        _gpu_case(ctx, out, fa, REDUCED, os.path.basename(out).encode())
    ctx.close()


@pytest.mark.gpu
def test_gpu_unused_blocks_are_not_uncompressed(tmp_path):
    """The quality block's payload of ce#1000.v31.cram overwritten: a decode without QUAL never uncompresses (or CRC-checks)
    it and equals the reference on that image; the full decode fails with the block's CRC status."""
    name, fa = "ce#1000.v31.cram", "ce.fa"
    img = np.fromfile(os.path.join(HT, name), dtype=np.uint8)
    blocks, udata, off = cpu_blocks(img)
    no_qual = ALL & ~H.SAM_QUAL
    drop = [i for i, u in enumerate(H.cram_required_blocks(blocks, udata, off, no_qual)) if not u]
    assert drop
    qs = max(drop, key=lambda i: int(blocks[i]["uncomp_size"]))            # QS: the largest block of the slice
    bad = img.copy()
    o, n = int(blocks[qs]["data_off"]), int(blocks[qs]["comp_size"])
    bad[o:o + n] = np.frombuffer(random.Random(5).randbytes(n), dtype=np.uint8)
    path = str(tmp_path / "qs_overwritten.cram")
    bad.tofile(path)
    fasta = H.load_fasta_upper(os.path.join(HT, fa), H.cram_sq_names(blocks, udata, off))
    ctx = H.Context(0)
    for decode_md in (0, 1):
        compare(path, fa, H.cram_decode_file_fields(ctx, bad, fasta, name.encode(), decode_md, no_qual), decode_md, no_qual)
    with pytest.raises(H.HgpuError, match="cram_decode_file: -2 "):
        H.cram_decode_file(ctx, bad, fasta, name.encode(), 0)
    ctx.close()


@pytest.mark.gpu
def test_gpu_no_reference_without_seq():
    name, fa = "ce#1000.v31.cram", "ce.fa"
    img = np.fromfile(os.path.join(HT, name), dtype=np.uint8)
    blocks, udata, off = cpu_blocks(img)
    ctx = H.Context(0)
    for mask in (ALL & ~H.SAM_SEQ, H.SAM_FLAG | H.SAM_POS | H.SAM_CIGAR, H.SAM_QUAL):
        compare(os.path.join(HT, name), fa, H.cram_decode_records_fields(ctx, img, blocks, udata, off, None, name.encode(), 1, mask), 1, mask)
        compare(os.path.join(HT, name), fa, H.cram_decode_file_fields(ctx, img, None, name.encode(), 1, mask), 1, mask)
    got = H.cram_decode_file_fields(ctx, img, None, name.encode(), 1, ALL)
    assert got["slice_status"].tolist() == [-7]
    ctx.close()
