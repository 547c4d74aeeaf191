"""Tag blocks in the CRAM record ENCODE (HGPU_CRAM_ENC_TAG_BLOCKS, htslib_b200/csrc/cram_encode.cuh / .cu): every tag key in a
block of its own, RG:Z naming an @RG line as the RG series, and MD:Z / NM left out where the reader rebuilds them, as the
reference's cram_encode_aux and process_one_read decide (cram/cram_encode.c:2781-3200, :3390-3740).

Checked against a plain restatement of the MD / NM rule (md_nm below), and against the reference's own writer on the same records
with the same slice layout: the reference's reader returns the same records for both files (decode_md 0 and 1), and every tag
block, tag dictionary and RG series value is the same.  Without a GPU the writer runs through tests/hostsim (kernels -> loops,
blocks stored RAW); `-m gpu` runs the device entry point."""
import ctypes as C
import gzip
import hashlib
import json
import os
import random
import struct
import numpy as np
import pytest
import htslib_b200 as H
import _libs
from _libs import GOLD, ref, sampled, stored_reference, bgzf_file
import test_cram_records as T
from test_cram_encode import pack, NAMES
from test_cram_mates import hostsim_lib, fasta_for, raw_series, decode_decisions, reg2bin, SAMS, MULTI, SEQS, NO_REF

TB, ATTACH = H.CRAM_ENC_TAG_BLOCKS, H.CRAM_ENC_ATTACH_MATES
SHAPES = [(minor, with_ref, rps) for minor in (0, 1) for with_ref in (False, True) for rps in (0, 3)]
PARENT_DIGESTS = os.path.join(GOLD, "cram_encode_parent_sha256.json.gz")


# The reference's results for this file's inputs, stored under tests/golden/ref_calls/ref_tags_*.gz (the same calls as the
# _libs helpers they wrap, kept apart from those helpers' stored results).

@stored_reference(limit=20000)
def ref_tags_sam_records(path):
    return _libs.ref_read_sam_records.__wrapped__(path)


@stored_reference(digest=True, limit=200000)
def ref_tags_cram_read_all(path, fasta=None, decode_md=0):
    return _libs.ref_cram_read_all.__wrapped__(path, fasta, decode_md)


@stored_reference(limit=100000)
def ref_tags_write_cram_image(sam_path, fasta, version, int_opts):
    return _libs._ref_write_cram.__wrapped__(sam_path, fasta, version, int_opts)


def ref_tags_write_cram(sam_path, fasta, out_path, version, int_opts):
    n, img = ref_tags_write_cram_image(sam_path, fasta, version, [list(o) for o in int_opts])
    with open(out_path, "wb") as f:
        f.write(img)
    return n


def sam_case(name):
    text, recs = ref_tags_sam_records(os.path.join(T.HT, "sam", name + ".sam"))
    return text, recs, os.path.join(T.HT, name.split("#")[0] + ".fa")


class Refused(Exception):
    def __init__(self, rc, msg):
        super().__init__("%d %s" % (rc, msg))
        self.rc = rc


def encode(ctx, text, recs, rps, minor, fa=None, flags=TB):
    """(file image, per-record (drop bits, RG value) of the hostsim writer, or None on the device)."""
    core, data, off = pack(recs)
    fasta = fasta_for(text, fa) if isinstance(fa, str) else fa
    if ctx is not None:
        try:
            return H.cram_encode_records(ctx, text, core, data, off, len(recs), fasta, rps, minor, flags), None
        except H.HgpuError as e:
            raise Refused(int(str(e).split(":")[1].split()[0]), str(e))
    l = hostsim_lib()
    l.hostsim_cram_enc_tags.restype = C.c_uint64
    l.hostsim_cram_enc_tags.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64]
    refs, keep = H._cram_refs(fasta)
    out, ln = C.c_void_p(), C.c_uint64(0)
    rc = l.hostsim_cram_encode_records_opts(text, len(text), core.ctypes.data, data.ctypes.data, off.ctypes.data, len(recs), refs, rps, minor, flags,
                                            C.byref(out), C.byref(ln))
    if rc != 0:
        raise Refused(rc, l.hostsim_enc_last_error().decode())
    img = C.string_at(out.value, ln.value)
    C.CDLL(None).free(C.c_void_p(out.value))
    drop, rg = np.zeros(max(1, len(recs)), np.uint8), np.zeros(max(1, len(recs)), np.int32)
    got = l.hostsim_cram_enc_tags(drop.ctypes.data, rg.ctypes.data, len(recs))
    return img, list(zip(drop[:got].tolist(), rg[:got].tolist()))


# ---- the rules restated ----

def aux_fields(c, d):
    """[(tag bytes, type, value bytes)] of a record's aux fields."""
    c = dict(zip(NAMES, c))
    p = c["l_qname"] + 4 * c["n_cigar"] + (c["l_qseq"] + 1) // 2 + c["l_qseq"]
    out = []
    while p < len(d):
        tag, t = d[p:p + 2], chr(d[p + 2])
        v = p + 3
        if t in "AcC": n = 1
        elif t in "sS": n = 2
        elif t in "iIf": n = 4
        elif t == "d": n = 8
        elif t in "ZH": n = d.index(0, v) - v + 1
        else:
            st, cnt = chr(d[v]), struct.unpack_from("<I", d, v + 1)[0]
            n = 5 + cnt * {"c": 1, "C": 1, "s": 2, "S": 2, "i": 4, "I": 4, "f": 4}[st]
        out.append((tag, t, d[v:v + n]))
        p = v + n
    return out


def seq_of(c, d):
    c = dict(zip(NAMES, c))
    s = d[c["l_qname"] + 4 * c["n_cigar"]:]
    return "".join("=ACMGRSVTWYHKDBN"[(s[i >> 1] >> (4 * (1 - (i & 1)))) & 15] for i in range(c["l_qseq"]))


def md_nm(c, d, ref):
    """(MD string, NM) process_one_read builds for a mapped record against ref (bytes, base 1 at ref[0]), or None where MD and NM
    are stored verbatim (:3390-3740)."""
    c = dict(zip(NAMES, c))
    if c["flag"] & 4 or c["l_qseq"] <= 0:
        return None
    seq, ref_end = seq_of(tuple(c[f] for f in NAMES), d).encode(), len(ref)
    apos, spos, last, nm, md = c["pos"], 0, c["pos"], 0, ""
    for k in range(c["n_cigar"]):
        w = struct.unpack_from("<I", d, c["l_qname"] + 4 * k)[0]
        op, ln = w & 15, w >> 4
        if op in (0, 7, 8):
            e = ln if ln + apos < ref_end else ref_end - apos
            if e < ln:
                return None
            for l in range(e):
                rb, sb = ref[apos + l], seq[spos + l]
                if rb == sb == ord("N"):
                    return None
                if rb != sb:
                    md += "%d%c" % (apos + l - last, rb); last = apos + l + 1; nm += 1
            apos += ln; spos += ln
        elif op == 2:
            md += "%d" % (apos - last)
            if apos < ref_end:
                md += "^" + ref[apos:apos + min(ref_end - apos, ln)].decode()
            nm += ln; apos += ln; last = apos
        elif op == 3:
            apos += ln; last += ln
        elif op == 1:
            nm += ln; spos += ln
        elif op == 4:
            spos += ln
    return md + "%d" % (apos - last), nm


def nm_value(t, v):
    """bam_aux2i_end (cram_encode.c:1253)."""
    if t in "cCsSiI":
        return struct.unpack("<" + {"c": "b", "C": "B", "s": "h", "S": "H", "i": "i", "I": "i"}[t], v)[0]
    return 0 if t in "Af" else None


def tag_rules(c, d, ref):
    """TAG_DROP_MD (1) | TAG_DROP_NM (2) of a record coded against ref."""
    r = md_nm(c, d, ref)
    if r is None:
        return 0
    md, nm = r
    f = aux_fields(c, d)
    mdf = [x for x in f if x[0] == b"MD"][:1]
    nmf = [x for x in f if x[0] == b"NM"][:1]
    drop = 0
    if mdf and mdf[0][1] == "Z" and mdf[0][2][:-1].lower() == md.lower().encode():
        drop |= 1
    if nmf and nm_value(nmf[0][1], nmf[0][2]) == nm:
        drop |= 2
    return drop


def rg_ids(text):
    ids = {}
    for line in text.split(b"\n"):
        if line.startswith(b"@RG\t"):
            for f in line.split(b"\t")[1:]:
                if f.startswith(b"ID:") and f[3:] not in ids:
                    ids[f[3:]] = len(ids)
    return ids


def rg_rule(text, c, d):
    ids = rg_ids(text)
    for tag, t, v in aux_fields(c, d):
        if tag == b"RG" and t == "Z":
            return ids.get(v[:-1], -1)
    return -1


def predicted(text, recs, fa):
    """Per record (drop bits, RG value) of the rules: MD / NM only against a reference."""
    fasta = fasta_for(text, fa) if fa else None
    out = []
    for c, d in recs:
        drop = 0
        if fasta is not None and not c[5] & 4:
            b, o = fasta
            drop = tag_rules(c, d, b[int(o[c[1]]):int(o[c[1] + 1])].tobytes())
        out.append((drop, rg_rule(text, c, d)))
    return out


# ---- file structure ----

def itf8_get(b, p):
    c = b[p]
    if c < 0x80: return c, p + 1
    if c < 0xc0: return ((c & 0x3f) << 8) | b[p + 1], p + 2
    if c < 0xe0: return ((c & 0x1f) << 16) | (b[p + 1] << 8) | b[p + 2], p + 3
    if c < 0xf0: return ((c & 0x0f) << 24) | (b[p + 1] << 16) | (b[p + 2] << 8) | b[p + 3], p + 4
    v = ((c & 0x0f) << 28) | (b[p + 1] << 20) | (b[p + 2] << 12) | (b[p + 3] << 4) | (b[p + 4] & 0x0f)
    return (v - (1 << 32) if v >= 1 << 31 else v), p + 5


def slices_of(img):
    """Per slice: (tag dictionary lines of its container, {content id: uncompressed bytes} of its external blocks)."""
    arr = np.frombuffer(img, dtype=np.uint8).copy()
    blocks, udata, off = T.cpu_blocks(arr)
    out, td = [], None
    for i, b in enumerate(blocks):
        u = udata[int(off[i]):int(off[i]) + int(b["uncomp_size"])].tobytes()
        ct = int(b["content_type"])
        if ct == 1:                                       # compression header: the preservation map's TD
            _, p = itf8_get(u, 0)
            n, p = itf8_get(u, p)
            for _ in range(n):
                k = u[p:p + 2]; p += 2
                if k == b"TD":
                    ln, p = itf8_get(u, p)
                    td = u[p:p + ln].split(b"\0")[:-1]
                    p += ln
                elif k == b"SM":
                    p += 5
                else:
                    p += 1
        elif ct == 2:
            out.append((td, {}))
        elif ct == 4 and out:
            out[-1][1][int(b["content_id"])] = u
    return out


def rg_series(blk):
    v, p = [], 0
    while p < len(blk):
        x, p = itf8_get(blk, p)
        v.append(x)
    return v


# ---- the reference's writer on the same records ----

def reference_file(tmp_path, path, text, recs, rps, fa, minor):
    """The reference writer's file of the records at path with our slice layout, or None where its layout differs or it declines."""
    r = rps or 10000
    out = str(tmp_path / "ref.cram")
    opts = [(MULTI, 1), (SEQS, r)] + ([] if fa else [(NO_REF, 1)])
    try:
        assert ref_tags_write_cram(path, fa, out, "3.%d" % minor, opts) == len(recs)
    except AssertionError:
        return None
    img = open(out, "rb").read()
    _, _, layout = decode_decisions(img, fa)
    if layout != [min(r, len(recs) - k) for k in range(0, len(recs), r)]:
        return None
    return img


def without_name(r):
    c, d = r
    return c[:4] + c[5:6] + c[7:], d[c[6]:] if isinstance(d, bytes) else d        # a stored digest keeps the whole record


def same_as_reference(tmp_path, path, text, recs, rps, minor, fa, flags=TB, tag="x", names=True):
    """Our file (hostsim) against the reference writer's: records through the reference's reader, tag blocks, dictionaries and RG
    series.  Returns our decisions, or None where the reference declines / lays the slices out differently.  names=False: records
    compare without their names (the reference's writer leaves out the names of unpaired reads after the first in the small
    hand-made files, and its reader makes them up)."""
    img, dec = encode(None, text, recs, rps, minor, fa, flags)
    assert dec == predicted(text, recs, fa), tag
    want = reference_file(tmp_path, path, text, recs, rps, fa, minor)
    if want is None:
        return None
    ours = str(tmp_path / ("%s.cram" % tag))
    theirs = str(tmp_path / "ref.cram")
    open(ours, "wb").write(img)
    for dm in (0, 1):
        with sampled():
            a, b = ref_tags_cram_read_all(ours, fa, dm), ref_tags_cram_read_all(theirs, fa, dm)
            assert (a == b) if names else ([without_name(r) for r in a] == [without_name(r) for r in b]), (tag, dm)
    r = rps or 10000
    mine, refs = slices_of(img), slices_of(want)
    assert len(mine) == len(refs)
    for s, ((td, blk), (rtd, rblk)) in enumerate(zip(mine, refs)):
        assert td == rtd, (tag, s, td, rtd)
        tags = {k: v for k, v in blk.items() if k > 0xffff}
        assert tags == {k: v for k, v in rblk.items() if k > 0xffff}, (tag, s, sorted(tags), sorted(k for k in rblk if k > 0xffff))
        assert rg_series(blk.get(6, b"")) == [g for _, g in dec[s * r:(s + 1) * r]], (tag, s)
    return dec


# ---- 1, 2: every fixture, every shape, against the reference's writer ----

@pytest.mark.parametrize("minor,with_ref,rps", SHAPES)
def test_hostsim_fixtures_same_as_reference_writer(tmp_path, minor, with_ref, rps):
    compared, dropped = 0, 0
    for sam in SAMS:
        text, recs, fa = sam_case(sam)
        if not recs:
            continue
        try:
            dec = same_as_reference(tmp_path, os.path.join(T.HT, "sam", sam + ".sam"), text, recs, rps, minor, fa if with_ref else None, tag=sam)
        except Refused as e:
            assert e.rc == -6, (sam, str(e))
            continue
        if dec is not None:
            compared += 1
            dropped += sum(1 for b, _ in dec if b)
    assert compared >= 20, compared
    assert (dropped > 20) == with_ref, dropped


def test_hostsim_tag_blocks_with_mates_round_trip(tmp_path):
    compared = 0
    for sam in ("xx#pair", "xx#triplet", "xx#rg", "xx#MD", "md#1", "ce#5b", "ce#unmap2"):
        text, recs, fa = sam_case(sam)
        for with_ref in (False, True):
            dec = same_as_reference(tmp_path, os.path.join(T.HT, "sam", sam + ".sam"), text, recs, 0, 1, fa if with_ref else None,
                                    flags=TB | ATTACH, tag=sam)
            compared += dec is not None
    assert compared >= 10, compared


# ---- 3: hand-made records, one per rule ----

def make_ref(n, seed, n_at=()):
    rng = random.Random(seed)
    s = bytearray(rng.choice(b"ACGT") for _ in range(n))
    for i in n_at:
        s[i] = ord("N")
    return bytes(s)


REF1, REF2 = make_ref(400, 1, (200,)), make_ref(70100, 2)
OPS = "MIDNSHP=X"


def rec(name, flag, pos, cigar, seq, tags=b"", tid=0):
    """A bam1_t record (core tuple, data): pos 0-based, cigar [(length, op)], seq '' for '*'."""
    nm = name.encode() + b"\0"
    extra = (4 - len(nm) % 4) % 4
    nm += b"\0" * extra
    cig = b"".join(struct.pack("<I", l << 4 | OPS.index(o)) for l, o in cigar)
    codes = ["=ACMGRSVTWYHKDBN".index(ch) for ch in seq] + [0]
    seq4 = bytes(codes[i] << 4 | codes[i + 1] for i in range(0, len(seq), 2))
    span = sum(l for l, o in cigar if o in "MDN=X")
    b = 4680 if flag & 4 else reg2bin(pos, pos + max(span, 1))
    return (pos, tid, b, 30, extra, flag, len(nm), len(cigar), len(seq), -1, -1, 0), nm + cig + seq4 + bytes([30]) * len(seq) + tags


def tZ(tag, s): return tag.encode() + b"Z" + s.encode() + b"\0"
def tI(tag, t, v): return tag.encode() + t.encode() + struct.pack("<" + {"c": "b", "C": "B", "s": "h", "S": "H", "i": "i", "I": "I"}[t], v)
def tA(tag, ch): return tag.encode() + b"A" + ch.encode()
def tF(tag, v): return tag.encode() + b"f" + struct.pack("<f", v)


def bam_image(text, refs, recs):
    body = b"BAM\1" + struct.pack("<i", len(text)) + text + struct.pack("<i", len(refs))
    for nm, ln in refs:
        body += struct.pack("<i", len(nm) + 1) + nm + b"\0" + struct.pack("<i", ln)
    for c, d in recs:
        pos, tid, bin_, mapq, _, flag, l_qname, n_cigar, l_qseq, mtid, mpos, isize = c
        r = struct.pack("<iiBBHHHiiii", tid, pos, l_qname, mapq, bin_, n_cigar, flag, l_qseq, mtid, mpos, isize) + d
        body += struct.pack("<i", len(r)) + r
    return bgzf_file(body, 6)


def sub(s, i, ch):
    return s[:i] + ch + s[i + 1:]


def r1(a, b): return REF1[a:b].decode()


def hand_cases():
    mm = sub(r1(10, 20), 4, "T" if r1(14, 15) != "T" else "G")        # one substitution at ref 15 (1-based)
    two = sub(sub(r1(10, 20), 2, "A" if r1(12, 13) != "A" else "C"), 7, "A" if r1(17, 18) != "A" else "C")          # two substitutions
    nm2 = lambda t, v=2: [rec("n" + t, 0, 10, [(10, "M")], two, tI("NM", t, v))]
    dl = r1(30, 34) + r1(36, 39) + r1(44, 48)                            # 4M2D3M5N4M at 30
    return {
        "md_equal": [rec("a", 0, 10, [(10, "M")], r1(10, 20), tZ("MD", "10") + tI("NM", "C", 0))],
        "md_equal_up_to_case": [rec("a", 0, 10, [(10, "M")], mm, tZ("MD", "4%s5" % r1(14, 15).lower()) + tI("NM", "C", 1))],
        "md_wrong": [rec("a", 0, 10, [(10, "M")], r1(10, 20), tZ("MD", "9%s0" % r1(19, 20)) + tI("NM", "C", 0))],
        "nm_wrong": [rec("a", 0, 10, [(10, "M")], r1(10, 20), tZ("MD", "10") + tI("NM", "C", 1))],
        "nm_types": nm2("c") + nm2("C") + nm2("s") + nm2("S") + nm2("i") + nm2("I") + nm2("c", -2) + nm2("I", 3),
        "nm_A_and_f": [rec("a", 0, 10, [(10, "M")], r1(10, 20), tA("NM", "x")), rec("b", 0, 10, [(10, "M")], r1(10, 20), tF("NM", 0.0)),
                       rec("c", 0, 10, [(10, "M")], mm, tA("NM", "x"))],
        "md_without_nm": [rec("a", 0, 10, [(10, "M")], mm, tZ("MD", "4%s5" % r1(14, 15)))],
        "nm_without_md": [rec("a", 0, 10, [(10, "M")], mm, tI("NM", "C", 1))],
        "deletion_and_skip": [rec("a", 0, 30, [(4, "M"), (2, "D"), (3, "M"), (5, "N"), (4, "M")], dl,
                                  tZ("MD", "4^%s7" % r1(34, 36)) + tI("NM", "C", 2)),
                              rec("b", 0, 30, [(2, "S"), (4, "M"), (1, "I"), (3, "M")], "GG" + r1(30, 34) + "T" + r1(34, 37),
                                  tZ("MD", "7") + tI("NM", "C", 1))],
        "long_deletion_nm_S": [rec("a", 0, 20, [(5, "M"), (300, "D"), (5, "M")], r1(20, 25) + r1(325, 330),
                                   tZ("MD", "5^%s5" % r1(25, 325)) + tI("NM", "S", 300))],
        "nm_I": [rec("a", 0, 10, [(5, "M"), (70000, "D"), (5, "M")], REF2[10:15].decode() + REF2[70015:70020].decode(),
                     tI("NM", "I", 70000), tid=1)],
        "n_in_read_and_reference": [rec("a", 0, 195, [(10, "M")], sub(r1(195, 205), 5, "N"), tZ("MD", "5N4") + tI("NM", "C", 1)),
                                    rec("b", 0, 195, [(10, "M")], sub(r1(195, 205), 5, "A"), tZ("MD", "5N4") + tI("NM", "C", 1))],
        "match_past_reference_end": [rec("a", 0, 395, [(10, "M")], r1(395, 400) + "ACGTA", tZ("MD", "5") + tI("NM", "C", 0))],
        "seq_star": [rec("a", 0, 10, [(10, "M")], "", tZ("MD", "10") + tI("NM", "C", 0))],
        "unmapped": [rec("a", 4, 10, [], r1(10, 20), tZ("MD", "10") + tI("NM", "C", 0))],
        "rg_second_line": [rec("a", 0, 10, [(10, "M")], r1(10, 20), tI("NH", "C", 1) + tZ("RG", "g2") + tI("AS", "C", 7))],
        "rg_without_line": [rec("a", 0, 10, [(10, "M")], r1(10, 20), tZ("RG", "zz") + tI("NH", "C", 1))],
    }


HAND_HDR = b"@HD\tVN:1.4\n@SQ\tSN:r1\tLN:400\n@SQ\tSN:r2\tLN:70100\n@RG\tID:g1\tSM:a\n@RG\tID:g2\tSM:b\n"
HAND_WANT = {"md_equal": [3], "md_equal_up_to_case": [3], "md_wrong": [2], "nm_wrong": [1], "nm_types": [2] * 6 + [0, 0],
             "nm_A_and_f": [2, 2, 0], "md_without_nm": [1], "nm_without_md": [2], "deletion_and_skip": [3, 3], "long_deletion_nm_S": [3],
             "nm_I": [2], "n_in_read_and_reference": [0, 3], "match_past_reference_end": [0], "seq_star": [0], "unmapped": [0],
             "rg_second_line": [0], "rg_without_line": [0]}


def hand_files(tmp_path, key, recs):
    fa = str(tmp_path / "hand.fa")
    with open(fa, "wb") as f:
        f.write(b">r1\n" + REF1 + b"\n>r2\n" + REF2 + b"\n")
    with open(fa + ".fai", "w") as f:
        f.write("r1\t400\t4\t400\t401\nr2\t70100\t%d\t70100\t70101\n" % (4 + 401 + 4))
    path = str(tmp_path / ("%s.bam" % key))
    with open(path, "wb") as f:
        f.write(bam_image(HAND_HDR, [(b"r1", 400), (b"r2", 70100)], recs))
    return path, fa


@pytest.mark.parametrize("key", sorted(HAND_WANT))
def test_hostsim_hand_made_rules(tmp_path, key):
    path, fa = hand_files(tmp_path, key, hand_cases()[key])
    text, recs = ref_tags_sam_records(path)
    assert [(c, d) for c, d in recs] and len(recs) == len(HAND_WANT[key])
    want_rg = {"rg_second_line": [1]}.get(key, [-1] * len(recs))
    img, dec = encode(None, text, recs, 0, 1, fa)
    assert dec == list(zip(HAND_WANT[key], want_rg)) == predicted(text, recs, fa), (key, dec)
    _, dec0 = encode(None, text, recs, 0, 1, None)                      # without a reference nothing is dropped
    assert dec0 == [(0, g) for g in want_rg]
    for minor in (0, 1):
        for f in (fa, None):
            got = same_as_reference(tmp_path, path, text, recs, 0, minor, f, tag=key, names=False)
            if ref() is not None and key != "match_past_reference_end":
                assert got is not None, (key, minor, f)


def test_hostsim_refusals():
    path_recs = hand_cases()["md_equal"]
    text = HAND_HDR
    d_rec = rec("d", 0, 10, [(10, "M")], r1(10, 20), b"XDd" + struct.pack("<d", 1.5))
    with pytest.raises(Refused) as e:
        encode(None, text, [d_rec], 0, 1, None)
    assert e.value.rc == -6 and "'d'" in str(e.value)
    assert encode(None, text, [d_rec], 0, 1, None, flags=0)[0]          # the shared streams hold it
    keys = [bytes([65 + k // 10, 48 + k % 10]) for k in range(257)]                  # A0 .. Z6: 257 keys of one type
    many = [rec("k%d" % i, 0, 10, [(10, "M")], r1(10, 20), b"".join(k + b"C\1" for k in keys[i::4])) for i in range(4)]
    assert encode(None, text, many[:1] + [rec("k", 0, 10, [(10, "M")], r1(10, 20), b"".join(k + b"C\1" for k in keys[1:256:4]))], 0, 1, None)[0]
    with pytest.raises(Refused) as e:
        encode(None, text, many, 0, 1, None)
    assert e.value.rc == -6
    for dup in (tZ("MD", "10") * 2, tI("NM", "C", 0) + tI("NM", "C", 0), tZ("RG", "g1") + tZ("RG", "g2")):
        with pytest.raises(Refused) as e:
            encode(None, text, [rec("a", 0, 10, [(10, "M")], r1(10, 20), dup)], 0, 1, None)
        assert e.value.rc == -6
    with pytest.raises(Refused) as e:
        encode(None, text, path_recs, 0, 1, None, flags=0x4)
    assert e.value.rc == -102                                            # HGPU_ERR_ARG


# ---- 4: without the bit, the parent commit's bytes ----

def parent_cases():
    for sam in SAMS:
        for minor, with_ref, rps in SHAPES:
            for flags in (0, ATTACH):
                yield sam, minor, with_ref, rps, flags


def test_hostsim_without_the_bit_unchanged():
    """enc_flags 0 and ATTACH_MATES alone give, on every fixture and shape, the bytes the writer gave before tag blocks existed
    (SHA-256 of each file, written by the previous commit's hostsim build)."""
    with gzip.open(PARENT_DIGESTS, "rt") as f:
        want = json.load(f)
    checked = 0
    for sam, minor, with_ref, rps, flags in parent_cases():
        k = "%s|%d|%d|%d|%d" % (sam, minor, with_ref, rps, flags)
        text, recs, fa = sam_case(sam)
        try:
            img, _ = encode(None, text, recs, rps, minor, fa if with_ref else None, flags)
            got = hashlib.sha256(img).hexdigest()
        except Refused as e:
            got = "refused %d" % e.rc
        assert got == want[k], k
        checked += 1
    assert checked == len(want)


# ---- 5: the device ----

def device_blocks(ctx, img):
    """Per slice {content id: bytes} of the external blocks, uncompressed on the device."""
    blocks, res = H.cram_uncompress_blocks(ctx, np.frombuffer(img, dtype=np.uint8).copy())
    out = []
    for b, (st, data) in zip(blocks, res):
        assert st == 0
        if int(b["content_type"]) == 2:
            out.append({})
        elif int(b["content_type"]) == 4 and out:
            out[-1][int(b["content_id"])] = data
    return out


def check_device(tmp_path, ctx, text, recs, rps, minor, fa, flags=TB, tag="x"):
    img, _ = encode(ctx, text, recs, rps, minor, fa, flags)
    sim, dec = encode(None, text, recs, rps, minor, fa, flags)
    assert device_blocks(ctx, img) == raw_series(sim), tag
    return img, dec


@pytest.mark.gpu
@pytest.mark.parametrize("minor", [0, 1])
def test_gpu_fixtures_read_back_as_reference_writer(tmp_path, minor):
    ctx = H.Context(0)
    done = 0
    for sam in SAMS:
        text, recs, fa = sam_case(sam)
        for with_ref in (False, True):
            f = fa if with_ref else None
            rps = 3 if minor else 0
            try:
                img, _ = check_device(tmp_path, ctx, text, recs, rps, minor, f, tag=sam)
            except Refused as e:
                assert e.rc == -6, (sam, str(e))
                continue
            ours = str(tmp_path / "gpu.cram")
            open(ours, "wb").write(img)
            want = reference_file(tmp_path, os.path.join(T.HT, "sam", sam + ".sam"), text, recs, rps, f, minor)
            with sampled():
                mine = ref_tags_cram_read_all(ours, f, 1)
                if want is not None:
                    assert mine == ref_tags_cram_read_all(str(tmp_path / "ref.cram"), f, 1), sam
                # our own device decoder with decode_md 1 returns what the reference's reader returns
                fasta = fasta_for(text, f) if f else None
                got = H.cram_decode_file(ctx, np.frombuffer(img, dtype=np.uint8).copy(), fasta, b"x", 1)
                assert got["slice_status"].tolist() == [0] * len(got["slice_status"])
                assert len(got["data"]) == len(mine)
                for i, (wc, wd) in enumerate(mine):
                    assert tuple(int(got["core"][i][n]) for n in NAMES) == wc and got["data"][i] == wd, (sam, i)
            done += 1
    assert done >= 40, done
    for key, recs in hand_cases().items():
        path, fa = hand_files(tmp_path, key, recs)
        text, rr = ref_tags_sam_records(path)
        check_device(tmp_path, ctx, text, rr, 0, minor, fa, flags=TB | ATTACH, tag=key)
    ctx.close()


def synthetic_tagged(n_pairs, seed=7, wrong=0.05):
    """Coordinate-sorted paired 100 bp reads over CHROMOSOME_I of ce.fa with substitutions, indels and skips, 3 @RG lines, NH / AS /
    XA, and MD / NM as an aligner writes them (a fraction `wrong` deliberately off by one): (header text, records, fasta arrays)."""
    rng = random.Random(seed)
    fa = os.path.join(T.HT, "ce.fa")
    fasta = H.load_fasta_upper(fa, [b"CHROMOSOME_I"])
    chrom = fasta[0][:int(fasta[1][1])].tobytes()
    shapes = [[(100, "M")], [(100, "M")], [(5, "S"), (95, "M")], [(40, "M"), (2, "I"), (58, "M")], [(50, "M"), (3, "D"), (50, "M")],
              [(30, "M"), (200, "N"), (70, "M")]]
    text = b"@HD\tVN:1.4\tSO:coordinate\n@SQ\tSN:CHROMOSOME_I\tLN:%d\n@RG\tID:g0\tSM:a\n@RG\tID:g1\tSM:a\n@RG\tID:g2\tSM:b\n" % len(chrom)
    recs, pos = [], 1000
    for i in range(n_pairs):
        pos += rng.randrange(0, 3)
        p2 = pos + rng.randrange(100, 300)
        for which, p in ((0, pos), (1, p2)):
            cig = rng.choice(shapes)
            s, rp = [], p
            for l, o in cig:
                if o == "M": s.append(chrom[rp:rp + l].decode()); rp += l
                elif o in "IS": s.append("".join(rng.choice("ACGT") for _ in range(l)))
                else: rp += l
            s = list("".join(s))
            for _ in range(rng.choice([0, 0, 1, 2, 4])):
                k = rng.randrange(len(s)); s[k] = rng.choice("ACGT")
            flag = 1 | 2 | (0x40 if which == 0 else 0x80) | (0x10 if which else 0x20)
            c, d = rec("r%07d" % i, flag, p, cig, "".join(s))
            md, nm = md_nm(c, d, chrom)
            if rng.random() < wrong:
                nm += 1
            tags = (tI("NH", "C", 1) + tI("AS", "C", rng.randrange(60, 100)) + tA("XA", rng.choice("xyz")) + tZ("MD", md) + tI("NM", "C", nm) +
                    tZ("RG", "g%d" % rng.randrange(3)))
            c = c[:9] + (0, p2 if which == 0 else pos, (p2 + 100 - pos) * (1 if which == 0 else -1))
            recs.append((c, d + tags))
    recs.sort(key=lambda r: r[0][0])
    return text, recs, fasta


@pytest.mark.gpu
def test_gpu_decisions_equal_hostsim_on_a_million_records():
    text, recs, fasta = synthetic_tagged(500000)
    ctx = H.Context(0)
    img, dec = check_device(None, ctx, text, recs, 9999, 1, fasta, flags=TB | ATTACH)
    assert sum(1 for b, _ in dec if b == 3) > 0.8 * len(recs)
    assert all(g >= 0 for _, g in dec)
    assert H.cram_encode_tags_last_ms() > 0
    plain = encode(ctx, text, recs, 9999, 1, fasta, flags=ATTACH)[0]
    assert len(img) < len(plain), (len(img), len(plain))
    ctx.close()
