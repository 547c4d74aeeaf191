"""Pins the oracle's BAM record unpack (orc_bam.c) against the compiled reference's own
bam_read1: every bam1_core_t field and every byte of bam1_t::data, on the reference's BAM
fixtures (including records straddling BGZF blocks) and on seeded synthetic records, plus the
SEQ/QUAL expansion against a direct statement of seq_nt16_str / +33."""
import glob, os, random, struct, sys, zlib
import pytest
from _libs import (GOLD, ROOT, bgzf_file, bam_header, bam_header_len, orc_bam_unpack_all, orc_bgzf_scan, ref,
                   ref_bam_read_all)
sys.path.insert(0, ROOT)
from tools import synth

BAMS = sorted(glob.glob(os.path.join(GOLD, "htslib", "bgzf_boundaries", "*.bam"))) + \
    [os.path.join(GOLD, "htslib", "range.bam"), os.path.join(GOLD, "htslib", "colons.bam")]


def inflate_all(img):
    _, blocks = orc_bgzf_scan(img)
    return b"".join(zlib.decompress(img[o + 18:o + l - 8], -15) for o, l in blocks)


def check_against_reference(img):
    stream = inflate_all(img)
    recs, _ = orc_bam_unpack_all(stream[bam_header_len(stream):])
    want = ref_bam_read_all(img)
    assert len(want) == len(recs) and len(recs) > 0
    for (st, core, data, seq, qual), (wcore, wdata, rc) in zip(recs, want):
        assert rc >= 0 and st == 0
        assert core == wcore
        assert data == wdata
        # SEQ / QUAL expansion (nibble2base, add33)
        lq, lqn, nc = core[8], core[6], core[7]
        nib = data[lqn + 4 * nc: lqn + 4 * nc + (lq + 1) // 2]
        assert seq == bytes(b"=ACMGRSVTWYHKDBN"[(nib[i >> 1] >> (4 if i % 2 == 0 else 0)) & 15] for i in range(lq))
        q = data[lqn + 4 * nc + (lq + 1) // 2:][:lq]
        assert qual == (q if lq and q[0] == 0xff else bytes((x + 33) & 0xff for x in q))
    return len(recs)


@pytest.mark.parametrize("path", BAMS, ids=os.path.basename)
def test_fixture_bams(path):
    check_against_reference(open(path, "rb").read())


def test_synthetic_records_and_odd_cases():
    stream, offs = synth.bam_records(3, 3000)
    rng = random.Random(4)
    extra = bytearray()
    # qname lengths 1..8 (all l_extranul cases), missing NUL terminator, l_qseq 0 / odd, unmapped, no cigar
    for k in range(40):
        name = bytes(rng.choice(b"abcXYZ019") for _ in range(k % 8)) + (b"\0" if k % 5 else b"Q")
        lq = [0, 1, 7, 150, 151][k % 5]
        cig = [] if k % 4 == 0 else [(lq << 4) | 0] if lq else []
        flag = 4 if not cig else 0
        seq = bytes(rng.randrange(256) for _ in range((lq + 1) // 2))
        qual = bytes([0xff] * lq) if k % 7 == 0 else bytes(rng.randrange(42) for _ in range(lq))
        aux = b"XAZ" + b"hi\0" if k % 2 else b""
        body = struct.pack("<iiBBHHHiiii", k % 3 - 1, 1000 + k * 50, len(name), 30, 4681, len(cig), flag, lq, -1, -1, 0)
        body += name + struct.pack("<%dI" % len(cig), *cig) + seq + qual + aux
        extra += struct.pack("<i", len(body)) + body
    full = bam_header() + stream + bytes(extra)
    n = check_against_reference(bgzf_file(full, 6))
    assert n == 3000 + 40
    # tiny blocks: records straddle many BGZF blocks
    check_against_reference(bgzf_file(bam_header() + stream[:offs[200]], 1, block=777))


def test_invalid_records_rejected_like_reference():
    stream, offs = synth.bam_records(5, 20)
    good = bytearray(stream[:offs[5]])
    cases = []
    b = bytearray(good); struct.pack_into("<i", b, offs[4] + 4 + 16, -5); cases.append(bytes(b))          # l_qseq < 0
    b = bytearray(good); b[offs[4] + 4 + 8] = 0; cases.append(bytes(b))                                   # l_qname 0
    b = bytearray(good); struct.pack_into("<i", b, offs[4] + 4 + 16, 100000); cases.append(bytes(b))      # l_qseq too long
    b = bytearray(good); struct.pack_into("<I", b, offs[4] + 36 + good[offs[4] + 12], (149 << 4)); cases.append(bytes(b))  # CIGAR/qlen mismatch
    for c in cases:
        want = ref_bam_read_all(bgzf_file(bam_header() + c, 6))
        recs, _ = orc_bam_unpack_all(c)
        assert want[-1][2] == -4 and len(want) == 5
        assert [r[0] for r in recs] == [0, 0, 0, 0, -4]
