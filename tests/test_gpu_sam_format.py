"""GPU parity: SAM text of unpacked BAM records (hgpu_sam_format_dev) against the reference's own sam_format1
(sam.c:4324-4404, htslib/sam.h:1463-1630) — byte for byte, on the reference's BAM fixtures and on records that
carry every aux type; records with floating-point aux values are flagged for the host."""
import glob, os, random, struct, sys, zlib
import numpy as np
import pytest
import htslib_b200 as H
from _libs import GOLD, ROOT, bam_header, bam_header_len, bgzf_file, orc_bgzf_scan, ref, ref_sam_format_all

pytestmark = pytest.mark.gpu
BAMS = sorted(glob.glob(os.path.join(GOLD, "htslib", "bgzf_boundaries", "*.bam"))) + \
    [os.path.join(GOLD, "htslib", "range.bam"), os.path.join(GOLD, "htslib", "colons.bam")]


@pytest.fixture(scope="module")
def ctx():
    c = H.Context(0)
    yield c
    c.close()


def gpu_lines(ctx, img, names):
    import torch
    _, blocks = orc_bgzf_scan(img)
    stream = b"".join(zlib.decompress(img[o + 18:o + l - 8], -15) for o, l in blocks)
    body = stream[bam_header_len(stream):]
    d = torch.from_numpy(np.frombuffer(body + b"\0" * 8, dtype=np.uint8).copy()).to("cuda:0")
    r = ctx.bam_unpack_dev(d, len(body))
    text, off, st = ctx.sam_format_dev(r["core"], r["data"], r["data_off"], r["n"], names)
    torch.cuda.synchronize()
    t = text.cpu().numpy().tobytes(); o = off.cpu().numpy(); s = st.cpu().numpy()
    return [(int(s[i]), t[int(o[i]):int(o[i + 1])]) for i in range(r["n"])]


@pytest.mark.parametrize("path", BAMS, ids=os.path.basename)
def test_fixture_bams_equal_sam_format1(ctx, path):
    img = open(path, "rb").read()
    names, want = ref_sam_format_all(img)
    got = gpu_lines(ctx, img, names)
    assert len(got) == len(want) > 0
    for (st, line), w in zip(got, want):
        assert st == 0 and line[-1:] == b"\n" and line[:-1] == w


def _rec(rng, qname, tid, pos, flag, cigar, seq, qual, aux, mtid=-1, mpos=-1, tlen=0, mapq=30):
    nt16 = {c: i for i, c in enumerate(b"=ACMGRSVTWYHKDBN")}
    l = len(seq)
    pk = bytearray((l + 1) // 2)
    for i, c in enumerate(seq):
        pk[i >> 1] |= nt16[c] << (4 if i % 2 == 0 else 0)
    ops = b"".join(struct.pack("<I", n << 4 | "MIDNSHP=XB".index(o)) for n, o in cigar)
    qn = qname + b"\0"
    body = struct.pack("<iiBBHHHiiii", tid, pos, len(qn), mapq, 4680, len(cigar), flag, l, mtid, mpos, tlen) + qn + ops + bytes(pk) + qual + aux
    return struct.pack("<i", len(body)) + body


def test_every_aux_type_and_odd_records(ctx):
    rng = random.Random(9)
    A = lambda tag, typ, payload: tag + typ + payload
    recs, expect_float = [], []
    hdr_text = b"@HD\tVN:1.6\n@SQ\tSN:chr1\tLN:1000000\n@SQ\tSN:chrUn_KI270442v1\tLN:392061\n"
    hdr = b"BAM\1" + struct.pack("<i", len(hdr_text)) + hdr_text + struct.pack("<i", 2) + \
        struct.pack("<i", 5) + b"chr1\0" + struct.pack("<i", 1000000) + struct.pack("<i", 20) + b"chrUn_KI270442v1\0\0\0\0"[:20] + struct.pack("<i", 392061)
    hdr = b"BAM\1" + struct.pack("<i", len(hdr_text)) + hdr_text + struct.pack("<i", 2) + \
        struct.pack("<i", 5) + b"chr1\0" + struct.pack("<i", 1000000) + struct.pack("<i", 17) + b"chrUn_KI270442v1\0" + struct.pack("<i", 392061)
    auxes = [
        b"",
        A(b"NM", b"C", b"\x07") + A(b"XA", b"A", b"q") + A(b"Xc", b"c", struct.pack("<b", -128)) + A(b"Xs", b"s", struct.pack("<h", -32768)) +
        A(b"XS", b"S", struct.pack("<H", 65535)) + A(b"Xi", b"i", struct.pack("<i", -2147483648)) + A(b"XI", b"I", struct.pack("<I", 4294967295)),
        A(b"MD", b"Z", b"150\0") + A(b"RG", b"Z", b"grp1\0") + A(b"XH", b"H", b"1AE301\0") + A(b"XE", b"Z", b"\0"),
        A(b"Bc", b"B", b"c" + struct.pack("<I", 3) + struct.pack("<3b", -1, 0, 127)) + A(b"BC", b"B", b"C" + struct.pack("<I", 2) + b"\x00\xff") +
        A(b"Bs", b"B", b"s" + struct.pack("<I", 2) + struct.pack("<2h", -300, 300)) + A(b"BS", b"B", b"S" + struct.pack("<I", 1) + struct.pack("<H", 65535)) +
        A(b"Bi", b"B", b"i" + struct.pack("<I", 2) + struct.pack("<2i", -70000, 70000)) + A(b"BI", b"B", b"I" + struct.pack("<I", 0)),
        A(b"Xf", b"f", struct.pack("<f", 3.25)),
        A(b"NM", b"i", struct.pack("<i", 1)) + A(b"Bf", b"B", b"f" + struct.pack("<I", 1) + struct.pack("<f", 0.5)),
        A(b"Xd", b"d", struct.pack("<d", 1e-9)),
    ]
    for k, aux in enumerate(auxes):
        l = rng.choice([0, 1, 2, 7, 150])
        seq = bytes(rng.choice(b"ACGTN=MRWS") for _ in range(l))
        qual = bytes([0xff] * l) if k % 3 == 2 else bytes(rng.randrange(0, 60) for _ in range(l))
        cigar = [] if l == 0 or k == 0 else [(l, "M")] if k % 2 else [(1, "S"), (max(1, l - 1), "M"), (5, "D"), (3, "N")]
        recs.append(_rec(rng, b"read:%d/x" % k if k else b"r", k % 2 if k != 3 else -1, 10 ** k if k < 9 else 5, 99 if k % 2 else 4, cigar, seq, qual, aux,
                         mtid=[-1, 0, 1][k % 3], mpos=k * 1000 - 1, tlen=(-1) ** k * k * 111))
        expect_float.append(any(t in aux for t in (b"Xff", b"Bff", b"Xdd")) or b"Bf" in aux[:0])
    expect_float = [b"Xf" in a or b"Bf" in a or b"Xd" in a for a in auxes]
    img = bgzf_file(hdr + b"".join(recs), 6)
    names, want = ref_sam_format_all(img)
    assert len(want) == len(recs) and names == [b"chr1", b"chrUn_KI270442v1"]
    got = gpu_lines(ctx, img, names)
    for (st, line), w, fl in zip(got, want, expect_float):
        if fl:
            assert st == 1 and line == b""
        else:
            assert st == 0 and line[-1:] == b"\n" and line[:-1] == w, (line, w)
