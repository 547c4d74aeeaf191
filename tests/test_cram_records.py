"""CRAM record decode (htslib_b200/csrc/cram_records.cuh: the record loop of cram_decode_slice, cram_decode_seq, cram_decode_aux,
cram_decode_slice_xref, cram_to_bam) against the compiled reference's sam_read1 on every CRAM fixture.

Two runs of the same source: `-m gpu` calls hgpu_cram_decode_records_host (the kernels); without a GPU the logic is checked through
tests/hostsim (the same __host__ __device__ code built for the host by g++, kernels replaced by loops — test infrastructure,
never loaded by htslib_b200)."""
import ctypes as C
import os
import subprocess
import numpy as np
import pytest
import htslib_b200 as H
from _libs import GOLD, ref, ref_cram_read_all, ref_write_cram
from test_cram_blocks import _expect

HT = os.path.join(GOLD, "htslib")
HERE = os.path.dirname(os.path.abspath(__file__))
CASES = [("ce#1000.v31.cram", "ce.fa"), ("ce#1000.v30.cram", "ce.fa"), ("ce#1000.v31arith.cram", "ce.fa"), ("ce#1000.v31fqz.cram", "ce.fa"),
         ("ce#5b_java.cram", "ce.fa"), ("auxf#values_java.cram", "auxf.fa"), ("xx#large_aux_java.cram", "xx.fa"), ("range.cram", "ce.fa")]


def hostsim():
    so = os.path.join(HERE, "hostsim", "_build", "libcramrec_hostsim.so")
    srcs = [os.path.join(HERE, "..", "htslib_b200", "csrc", f) for f in ("cram_records.cu", "cram_records.cuh", "cram_encode.cu", "cram_encode.cuh")]
    if not os.path.exists(so) or os.path.getmtime(so) < max(os.path.getmtime(f) for f in srcs):
        subprocess.check_call(["bash", os.path.join(HERE, "hostsim", "build.sh")], stdout=subprocess.DEVNULL)
    l = C.CDLL(so)
    l.hostsim_cram_decode_records.argtypes = [C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_char_p, C.c_int, C.c_void_p]
    l.hostsim_last_error.restype = C.c_char_p
    return (l.hostsim_cram_decode_records, l.hostsim_cram_records_free, lambda: l.hostsim_last_error().decode())


def cpu_blocks(img):
    """The blocks uncompressed by the per-codec checkers (what hgpu_cram_uncompress_blocks_host returns on a GPU box)."""
    blocks, _ = H.cram_scan_blocks(img)
    sizes = blocks["uncomp_size"].astype(np.int64)
    off = np.concatenate([[0], np.cumsum((sizes + 15) // 16 * 16)]).astype(np.uint64)
    udata = np.zeros(int(off[-1]) + 16, dtype=np.uint8)
    for i, b in enumerate(blocks):
        want = _expect(img, b)
        assert want is not None and len(want) == int(b["uncomp_size"]), (i, int(b["method"]))
        udata[int(off[i]):int(off[i]) + len(want)] = np.frombuffer(want, dtype=np.uint8)
    return blocks, udata, off[:-1].copy()


def compare(name, fa, got, decode_md, path=None):
    want = ref_cram_read_all(path or os.path.join(HT, name), os.path.join(HT, fa), decode_md)
    assert got["slice_status"].tolist() == [0] * len(got["slice_status"]), (name, got["slice_status"].tolist())
    assert len(got["data"]) == len(want), (name, len(got["data"]), len(want))
    names = [f for f, _ in H.BAM1_CORE_DT]
    for i, (wc, wd) in enumerate(want):
        gc = tuple(int(got["core"][i][f]) for f in names)
        assert gc == wc, (name, decode_md, i, dict(zip(names, gc)), dict(zip(names, wc)))
        assert got["data"][i] == wd, (name, decode_md, i, got["data"][i][:80], wd[:80])
        assert got["rec_status"][i] == 0


@pytest.mark.parametrize("decode_md", [0, 1])
@pytest.mark.parametrize("name,fa", CASES)
def test_hostsim_records_equal_reference(name, fa, decode_md):
    img = np.fromfile(os.path.join(HT, name), dtype=np.uint8)
    blocks, udata, off = cpu_blocks(img)
    fasta = H.load_fasta_upper(os.path.join(HT, fa), H.cram_sq_names(blocks, udata, off))
    got = H.cram_decode_records(None, img, blocks, udata, off, fasta, name.encode(), decode_md, _entry=hostsim())
    compare(name, fa, got, decode_md)


@pytest.mark.gpu
@pytest.mark.parametrize("decode_md", [0, 1])
@pytest.mark.parametrize("name,fa", CASES)
def test_gpu_records_equal_reference(name, fa, decode_md):
    img = np.fromfile(os.path.join(HT, name), dtype=np.uint8)
    ctx = H.Context(0)
    blocks, res = H.cram_uncompress_blocks(ctx, img)
    sizes = blocks["uncomp_size"].astype(np.int64)
    off = np.concatenate([[0], np.cumsum((sizes + 15) // 16 * 16)]).astype(np.uint64)
    udata = np.zeros(int(off[-1]) + 16, dtype=np.uint8)
    for i, (st, data) in enumerate(res):
        assert st == 0, (i, st)
        udata[int(off[i]):int(off[i]) + len(data)] = np.frombuffer(data, dtype=np.uint8)
    fasta = H.load_fasta_upper(os.path.join(HT, fa), H.cram_sq_names(blocks, udata, off))
    got = H.cram_decode_records(ctx, img, blocks, udata, off[:-1].copy(), fasta, name.encode(), decode_md)
    compare(name, fa, got, decode_md)
    ctx.close()


# the SAM files the reference's own test/test.pl round-trips through CRAM (test/*.sam; the part before '#' names the reference),
# written here by the compiled reference in several shapes: CRAM 3.0 / 3.1, no reference, embedded reference, several references
# per slice with tiny slices, generated read names, stored MD/NM, several slices per container
SAMS = sorted(f[:-4] for f in os.listdir(os.path.join(HT, "sam")) if f.endswith(".sam"))
NO_REF, EMBED_REF, MULTI, SEQS, SLICES, LOSSY, STORE_MD, STORE_NM = 11, 7, 10, 3, 4, 19, 21, 22
SHAPES = {"v30": ("3.0", []), "v31": ("3.1", []), "noref": ("3.0", [(NO_REF, 1)]), "embed": ("3.1", [(EMBED_REF, 1)]),
          "multi": ("3.0", [(MULTI, 1), (SEQS, 3)]), "lossy": ("3.1", [(LOSSY, 1)]), "storemd": ("3.0", [(STORE_MD, 1), (STORE_NM, 1)]),
          "slices": ("3.1", [(SLICES, 2), (SEQS, 2)])}


def _written(tmp_path, sam, shape):
    fa = sam.split("#")[0] + ".fa"
    out = str(tmp_path / ("%s.%s.cram" % (sam.replace("#", "_"), shape)))
    version, opts = SHAPES[shape]
    n = ref_write_cram(os.path.join(HT, "sam", sam + ".sam"), os.path.join(HT, fa), out, version, opts)
    return out, fa, n


@pytest.mark.parametrize("shape", sorted(SHAPES))
@pytest.mark.parametrize("sam", SAMS)
def test_hostsim_written_by_reference(tmp_path, sam, shape):
    out, fa, n = _written(tmp_path, sam, shape)
    img = np.fromfile(out, dtype=np.uint8)
    blocks, udata, off = cpu_blocks(img)
    fasta = H.load_fasta_upper(os.path.join(HT, fa), H.cram_sq_names(blocks, udata, off))
    for decode_md in (0, 1):
        got = H.cram_decode_records(None, img, blocks, udata, off, fasta, os.path.basename(out).encode(), decode_md, _entry=hostsim())
        assert len(got["data"]) == n
        compare(sam, fa, got, decode_md, path=out)


@pytest.mark.gpu
@pytest.mark.parametrize("shape", sorted(SHAPES))
def test_gpu_written_by_reference(tmp_path, shape):
    ctx = H.Context(0)
    for sam in SAMS:
        out, fa, n = _written(tmp_path, sam, shape)
        img = np.fromfile(out, dtype=np.uint8)
        blocks, udata, off = cpu_blocks(img)
        fasta = H.load_fasta_upper(os.path.join(HT, fa), H.cram_sq_names(blocks, udata, off))
        for decode_md in (0, 1):
            got = H.cram_decode_records(ctx, img, blocks, udata, off, fasta, os.path.basename(out).encode(), decode_md)
            assert len(got["data"]) == n
            compare(sam, fa, got, decode_md, path=out)
    ctx.close()


def _synthetic_sam(path, n=10000, seed=3):
    """A coordinate-sorted paired-end SAM over CHROMOSOME_I of ce.fa: matches, substitutions, insertions, deletions, reference skips,
    soft / hard clips, unmapped mates, several read groups and aux tag types — every read feature code the writer emits."""
    import random
    rng = random.Random(seed)
    fa = H.load_fasta_upper(os.path.join(HT, "ce.fa"))
    chrom = fa[0][:int(fa[1][1])].tobytes()
    recs = []
    shapes = [[(100, "M")], [(5, "S"), (95, "M")], [(40, "M"), (2, "I"), (58, "M")], [(50, "M"), (3, "D"), (50, "M")], [(30, "M"), (200, "N"), (70, "M")],
              [(10, "H"), (90, "M"), (10, "S")], [(100, "M")], [(100, "M")], [(60, "M"), (1, "I"), (20, "M"), (1, "D"), (19, "M")]]
    pos = 1000
    for i in range(n // 2):
        pos += rng.randrange(1, max(2, min(150, 1_700_000 // n)))
        ends = []
        for which in (0, 1):
            p = pos + which * rng.randrange(150, 400)
            sh = rng.choice(shapes)
            seq, rp = [], p - 1
            for l, op in sh:
                if op in "M":
                    seq.append(chrom[rp:rp + l].decode()); rp += l
                elif op in "IS":
                    seq.append("".join(rng.choice("ACGT") for _ in range(l)))
                elif op in "DN":
                    rp += l
            s = list("".join(seq))
            for _ in range(rng.choice([0, 0, 1, 2, 5])):
                s[rng.randrange(len(s))] = rng.choice("ACGTN")
            q = "".join(chr(33 + rng.choice([2, 12, 23, 37])) for _ in s)
            ends.append((p, "".join("%d%s" % t for t in sh), "".join(s), q, rp))
        unm = rng.random() < 0.03
        for which in (0, 1):
            p, cig, s, q, rp = ends[which]
            mp = ends[1 - which][0]
            flag = 1 | (64 if which == 0 else 128) | (16 if which else 32)
            if unm and which == 1:
                flag = 1 | 128 | 4 | 32; cig = "*"; p = ends[0][0]
            if unm and which == 0:
                flag |= 8
            lo, hi = min(ends[0][0], ends[1][0]), max(ends[0][4], ends[1][4])
            tlen = 0 if unm else (hi - lo + 1) * (1 if p == lo and which == 0 else -1 if which == 1 else 1)
            tags = ["RG:Z:g%d" % rng.randrange(3), "NH:i:%d" % rng.randrange(1, 300), "XA:A:%s" % rng.choice("xyz")]
            if rng.random() < 0.3: tags.append("XB:B:s,%d,%d,-7" % (rng.randrange(100), rng.randrange(40000) - 20000))
            if rng.random() < 0.2: tags.append("XZ:Z:" + "".join(rng.choice("abc:;") for _ in range(rng.randrange(0, 20))))
            recs.append((p, "r%06d\t%d\tCHROMOSOME_I\t%d\t%d\t%s\t=\t%d\t%d\t%s\t%s\t%s" % (i, flag, p, rng.randrange(0, 61), cig, mp if not (unm and which == 0) else p, tlen, s, q, "\t".join(tags))))
    recs.sort(key=lambda t: t[0])
    with open(path, "w") as f:
        f.write("@HD\tVN:1.4\tSO:coordinate\n@SQ\tSN:CHROMOSOME_I\tLN:1009800\n@RG\tID:g0\tSM:a\n@RG\tID:g1\tSM:a\n@RG\tID:g2\tSM:b\n")
        for _, line in recs:
            f.write(line + "\n")
    return len(recs)


def _synthetic_case(tmp_path, entry_ctx, version, opts):
    sam = str(tmp_path / "syn.sam")
    n = _synthetic_sam(sam)
    out = str(tmp_path / "syn.cram")
    assert ref_write_cram(sam, os.path.join(HT, "ce.fa"), out, version, opts) == n
    img = np.fromfile(out, dtype=np.uint8)
    blocks, udata, off = cpu_blocks(img)
    fasta = H.load_fasta_upper(os.path.join(HT, "ce.fa"), H.cram_sq_names(blocks, udata, off))
    for decode_md in (0, 1):
        if entry_ctx is None:
            got = H.cram_decode_records(None, img, blocks, udata, off, fasta, b"syn.cram", decode_md, _entry=hostsim())
        else:
            got = H.cram_decode_records(entry_ctx, img, blocks, udata, off, fasta, b"syn.cram", decode_md)
        assert len(got["data"]) == n
        compare("syn", "ce.fa", got, decode_md, path=out)
    return len(got["slice_status"])


def test_hostsim_synthetic_10000_read_slice(tmp_path):
    assert _synthetic_case(tmp_path, None, "3.1", []) == 1
    assert _synthetic_case(tmp_path, None, "3.0", [(SEQS, 700), (LOSSY, 1)]) == 15


@pytest.mark.gpu
def test_gpu_synthetic_10000_read_slice(tmp_path):
    ctx = H.Context(0)
    assert _synthetic_case(tmp_path, ctx, "3.1", []) == 1
    assert _synthetic_case(tmp_path, ctx, "3.0", [(SEQS, 700), (LOSSY, 1)]) == 15
    ctx.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name,fa", [("ce#1000.v31.cram", "ce.fa"), ("ce#1000.v31arith.cram", "ce.fa"), ("range.cram", "ce.fa")])
def test_gpu_file_in_records_out(name, fa):
    """hgpu_cram_decode_file_host: the image goes in, every block is uncompressed and every record decoded on the device."""
    img = np.fromfile(os.path.join(HT, name), dtype=np.uint8)
    blocks, udata, off = cpu_blocks(img)                       # only to learn the @SQ order of the header
    fasta = H.load_fasta_upper(os.path.join(HT, fa), H.cram_sq_names(blocks, udata, off))
    ctx = H.Context(0)
    got = H.cram_decode_file(ctx, img, fasta, name.encode(), 1)
    compare(name, fa, got, 1)
    ctx.close()


def _mutations(name, count, seed):
    import random
    rng = random.Random(seed)
    fa = dict(CASES)[name]
    img = np.fromfile(os.path.join(HT, name), dtype=np.uint8)
    blocks, udata, off = cpu_blocks(img)
    fasta = H.load_fasta_upper(os.path.join(HT, fa), H.cram_sq_names(blocks, udata, off))
    for _ in range(count):
        u2 = udata.copy()
        for _ in range(rng.randrange(1, 5)):
            i = rng.randrange(len(blocks))
            if int(blocks[i]["content_type"]) == 0 or int(blocks[i]["uncomp_size"]) == 0:
                continue
            p = int(off[i]) + rng.randrange(int(blocks[i]["uncomp_size"]))
            u2[p] = rng.randrange(256) if rng.random() < 0.7 else (int(u2[p]) ^ (1 << rng.randrange(8)))
        yield img, blocks, u2, off, fasta, rng.randrange(2)


@pytest.mark.parametrize("name", ["ce#5b_java.cram", "range.cram"])
def test_hostsim_corrupt_series_never_run_wild(name):
    """Random bytes flipped in compression headers, slice headers, CORE and external blocks: the decoder must come back with a
    status (a malformed header fails the call; a bad slice is flagged -1; untouched slices still decode), never crash —
    every cursor, bit read and arena append is bounds-checked (the same code runs on the device)."""
    seen = set()
    for img, blocks, u2, off, fasta, md in _mutations(name, 60, 5):
        try:
            got = H.cram_decode_records(None, img, blocks, u2, off, fasta, b"x", md, _entry=hostsim())
            assert set(got["slice_status"].tolist()) <= {0, -1, -4, -6, -7}
            for st, d in zip(got["rec_status"], got["data"]):
                assert st == 0 or d == b""
            seen |= set(got["slice_status"].tolist())
        except H.HgpuError:
            seen.add("call")
    assert 0 in seen and (-1 in seen or "call" in seen)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["ce#5b_java.cram", "range.cram"])
def test_gpu_corrupt_series_never_run_wild(name):
    ctx = H.Context(0)
    for img, blocks, u2, off, fasta, md in _mutations(name, 40, 6):
        try:
            got = H.cram_decode_records(ctx, img, blocks, u2, off, fasta, b"x", md)
            assert set(got["slice_status"].tolist()) <= {0, -1, -4, -6, -7}
        except H.HgpuError as e:
            assert "CUDA" not in str(e) and "illegal" not in str(e), str(e)
    # the context is still healthy: the clean file decodes
    img = np.fromfile(os.path.join(HT, name), dtype=np.uint8)
    blocks, udata, off = cpu_blocks(img)
    fasta = H.load_fasta_upper(os.path.join(HT, dict(CASES)[name]), H.cram_sq_names(blocks, udata, off))
    got = H.cram_decode_records(ctx, img, blocks, udata, off, fasta, name.encode(), 0)
    compare(name, dict(CASES)[name], got, 0)
    ctx.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name,fa", [("ce#1000.v31.cram", "ce.fa"), ("range.cram", "ce.fa"), ("ce#5b_java.cram", "ce.fa")])
def test_gpu_cram_to_sam_text_without_leaving_the_device(name, fa):
    """hgpu_cram_decode_records_dev leaves core / data / data_off in HBM in hgpu_bam_unpack_dev's layout; hgpu_sam_format_dev takes them
    as they are: the SAM text must equal the reference's sam_read1 + sam_format1 on the same CRAM."""
    import ctypes as C
    import torch
    from _libs import ref_cram_sam_text
    img = np.fromfile(os.path.join(HT, name), dtype=np.uint8)
    blocks, udata, off = cpu_blocks(img)
    fasta = H.load_fasta_upper(os.path.join(HT, fa), H.cram_sq_names(blocks, udata, off))
    ctx = H.Context(0)
    dev, sst = H.cram_decode_records_dev(ctx, img, blocks, udata, off, fasta, name.encode(), 1)
    assert sst.tolist() == [0] * len(sst)
    n = int(dev.n_records)

    class Raw:                                        # a device pointer with the two methods the wrapper uses
        def __init__(self, p): self.p = p; self.device = torch.device("cuda", 0)
        def data_ptr(self): return self.p
    names, want = ref_cram_sam_text(os.path.join(HT, name), os.path.join(HT, fa), 1)
    text, out_off, status = ctx.sam_format_dev(Raw(dev.d_core), Raw(dev.d_data), Raw(dev.d_data_off), n, names)
    torch.cuda.synchronize()
    t = text.cpu().numpy().tobytes(); oo = out_off.cpu().numpy(); stt = status.cpu().numpy()
    assert n == len(want)
    for i, w in enumerate(want):
        if stt[i] == 1:
            continue                                  # a floating-point aux value: left to the host by contract
        line = t[int(oo[i]):int(oo[i + 1])]
        assert stt[i] == 0 and line[-1:] == b"\n" and line[:-1] == w, (i, line[:120], w)
    ctx.close()
