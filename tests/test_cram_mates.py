"""Mate attachment in the CRAM record ENCODE (HGPU_CRAM_ENC_ATTACH_MATES, htslib_b200/csrc/cram_encode.cuh / .cu): reads of one
template in the same slice are attached as the reference's process_one_read attaches them (cram/cram_encode.c:3799-4012).

Checked against a plain restatement of that rule (mate_rules below), against the decisions of the reference's own writer on
the same records and slice layout, and by the reference's reader, which must return the input records.  `-m gpu` runs the
device entry point (hgpu_cram_encode_records_opts_host, compressed blocks); without a GPU the same source runs through
tests/hostsim (kernels -> loops, blocks stored RAW)."""
import ctypes as C
import os
import struct
import numpy as np
import pytest
import htslib_b200 as H
from _libs import GOLD, ref, ref_read_sam_records, ref_cram_read_all, ref_write_cram, sampled
import test_cram_records as T
from test_cram_encode import pack, sq_names, expected, NAMES

HT = os.path.join(GOLD, "htslib")
SAMS = sorted(f[:-4] for f in os.listdir(os.path.join(HT, "sam")) if f.endswith(".sam"))
ATTACH = H.CRAM_ENC_ATTACH_MATES
NO_REF, MULTI, SEQS = 11, 10, 3                   # CRAM_OPT_NO_REF, CRAM_OPT_MULTI_SEQ_PER_SLICE, CRAM_OPT_SEQS_PER_SLICE
CF, MF, NS, NP, TS, NF = 2, 8, 9, 10, 11, 32      # content ids of the series (stream index + 1)


def hostsim_lib():
    T.hostsim()                                   # builds / refreshes the harness
    l = C.CDLL(os.path.join(T.HERE, "hostsim", "_build", "libcramrec_hostsim.so"))
    l.hostsim_cram_encode_records_opts.argtypes = [C.c_char_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint32,
                                                   C.c_int, C.c_uint32, C.c_void_p, C.c_void_p]
    l.hostsim_enc_last_error.restype = C.c_char_p
    l.hostsim_cram_enc_mates.restype = C.c_uint64
    l.hostsim_cram_enc_mates.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64]
    l.hostsim_cram_record_mates.restype = C.c_uint64
    l.hostsim_cram_record_mates.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64]
    l.hostsim_cram_enc_hash_mask.argtypes = [C.c_uint64]
    return l


def fasta_for(text, fa):
    return H.load_fasta_upper(fa, sq_names(text)) if fa else None


class Unsupported(Exception):
    """HGPU_CRAM_UNSUPPORTED: records the encoder leaves to the host library, with or without attachment."""


def encode(ctx, text, recs, rps, minor, fa=None, flags=ATTACH):
    """(file image, per-record (cf, nf) decisions of the hostsim pairing pass or None on the device)."""
    core, data, off = pack(recs)
    fasta = fasta_for(text, fa)
    if ctx is not None:
        return H.cram_encode_records(ctx, text, core, data, off, len(recs), fasta, rps, minor, flags), None
    l = hostsim_lib()
    refs, keep = H._cram_refs(fasta)
    out, ln = C.c_void_p(), C.c_uint64(0)
    rc = l.hostsim_cram_encode_records_opts(text, len(text), core.ctypes.data, data.ctypes.data, off.ctypes.data, len(recs), refs, rps, minor, flags,
                                            C.byref(out), C.byref(ln))
    if rc == -6:
        raise Unsupported(l.hostsim_enc_last_error().decode())
    assert rc == 0, (rc, l.hostsim_enc_last_error())
    img = C.string_at(out.value, ln.value)
    C.CDLL(None).free(C.c_void_p(out.value))
    cf, nf = np.zeros(max(1, len(recs)), np.uint8), np.zeros(max(1, len(recs)), np.int32)
    got = l.hostsim_cram_enc_mates(cf.ctypes.data, nf.ctypes.data, len(recs)) if flags & ATTACH else 0
    return img, (list(zip(cf[:got].tolist(), nf[:got].tolist())) if flags & ATTACH else None)


def cram_aend(c, d, no_ref, ref_end):
    """cr->aend of process_one_read (:3718, :3730)."""
    apos = c["pos"] + 1
    if c["flag"] & 4:
        return min(apos, ref_end)
    e = c["pos"]
    for k in range(c["n_cigar"]):
        w = struct.unpack_from("<I", d, c["l_qname"] + 4 * k)[0]
        if (w & 15) in (0, 2, 3, 7, 8):
            e += w >> 4
    return e if no_ref else min(e, max(0, ref_end))


def mate_rules(recs, rps, ref_lens=None):
    """The mate block of process_one_read restated: per record (CRAM_FLAG_DETACHED / CRAM_FLAG_MATE_DOWNSTREAM bits, NF)."""
    n, rps = len(recs), rps or 10000
    out = [(2, 0)] * n
    for a in range(0, n, rps):
        ref_end = 0                               # c->ref_end: 0 without a reference, else the last loaded sequence's length
        tables, state = ({}, {}), {}
        for g in range(a, min(n, a + rps)):
            c, d = dict(zip(NAMES, recs[g][0])), recs[g][1]
            f = c["flag"]
            if ref_lens is not None and 0 <= c["tid"] < len(ref_lens):
                ref_end = ref_lens[c["tid"]]
            apos = c["pos"] + 1
            me = dict(apos=apos, aend=cram_aend(c, d, ref_lens is None, ref_end), ref_id=c["tid"], flags=f,
                      mate_flags=(2 if f & 8 else 0) | (1 if f & 0x20 else 0), mate_pos=max(c["mpos"] + 1, 0), tlen=c["isize"])
            if not f & 1:
                continue
            name = bytes(d[:c["l_qname"]]).split(b"\0")[0]
            bits = (1 if f & 0x40 else 0) | (2 if f & 0x80 else 0)
            t = tables[1 if f & 0x100 else 0]
            if name not in t:
                t[name] = (g, bits)
                state[g] = me
                continue
            pi, r12 = t[name]
            p = state[pi]
            aleft, aright = min(apos, p["apos"]), max(me["aend"], p["aend"])
            sign = 1 if apos < p["apos"] else -1 if apos > p["apos"] else (1 if f & 0x40 else -1)
            span = aright - aleft + 1
            detach = ((r12 & 1 and f & 0x40) or (r12 & 2 and f & 0x80) or max(c["mpos"] + 1, 0) != p["apos"] or
                      bool(f & 8) != bool(p["flags"] & 4) or bool(f & 0x20) != bool(p["flags"] & 0x10) or
                      p["ref_id"] != c["tid"] or p["mate_pos"] != apos or
                      bool(p["flags"] & 8) != bool(p["mate_flags"] & 2) or bool(p["flags"] & 0x20) != bool(p["mate_flags"] & 1) or
                      (f | p["flags"]) & 0x800 or c["isize"] == 0 or c["isize"] != sign * span or p["tlen"] == 0 or p["tlen"] != -sign * span)
            if detach:
                continue
            me.update(mate_pos=p["apos"], tlen=sign * span, mate_flags=(2 if p["flags"] & 8 else 0) | (1 if p["flags"] & 0x20 else 0))
            out[g] = (0, 0)
            out[pi] = (4, g - pi - 1)
            t[name] = (g, r12 | bits)
            state[g] = me
    return out


def decode_decisions(img, fa_pair=None):
    """Decode a file through the hostsim decoder: (records dict, per-record (CF & 6, NF) as the record loop read them)."""
    arr = np.frombuffer(img, dtype=np.uint8).copy()
    blocks, udata, off = T.cpu_blocks(arr)
    fasta = H.load_fasta_upper(fa_pair, H.cram_sq_names(blocks, udata, off)) if fa_pair else None
    got = H.cram_decode_records(None, arr, blocks, udata, off, fasta, b"x", 0, _entry=T.hostsim())
    assert got["slice_status"].tolist() == [0] * len(got["slice_status"])
    l = hostsim_lib()
    n = len(got["data"])
    cf, ml = np.zeros(max(1, n), np.int32), np.zeros(max(1, n), np.int32)
    assert l.hostsim_cram_record_mates(cf.ctypes.data, ml.ctypes.data, n) == n
    rec0 = got["slice_rec0"].tolist()
    dec = []
    for s in range(len(rec0) - 1):
        for g in range(int(rec0[s]), int(rec0[s + 1])):
            b = int(cf[g]) & 6
            dec.append((b, int(ml[g]) - (g - int(rec0[s])) - 1 if b & 4 else 0))
    return got, dec, [int(rec0[s + 1] - rec0[s]) for s in range(len(rec0) - 1)]


def read_back(tmp_path, img, recs, fa, tag):
    """The file decodes to the input records (up to test_cram_encode.expected): through our hostsim decoder always, and
    through the compiled reference's sam_read1 where its result is available.  Returns decode_decisions' result."""
    got, dec, layout = decode_decisions(img, fa)
    want = [expected(c, d) for c, d in recs]
    assert len(got["data"]) == len(recs), (tag, len(got["data"]), len(recs))
    for i, (wc, wd) in enumerate(want):
        gc = tuple(int(got["core"][i][f]) for f in NAMES)
        assert gc == wc, (tag, i, dict(zip(NAMES, gc)), dict(zip(NAMES, wc)))
        assert got["data"][i] == wd, (tag, i)
    out = str(tmp_path / ("%s.cram" % tag))
    open(out, "wb").write(img)
    with sampled():
        back = ref_cram_read_all(out, fa, 0)
        assert len(back) == len(recs), (tag, len(back), len(recs))
        for i, ((gc, gd), (wc, wd)) in enumerate(zip(back, want)):
            assert gc == wc, (tag, i, dict(zip(NAMES, gc)), dict(zip(NAMES, wc)))
            assert gd == wd, (tag, i)
    return got, dec, layout


def ref_lens_of(text, fa):
    if not fa:
        return None
    b, o = fasta_for(text, fa)
    return [int(o[i + 1] - o[i]) for i in range(len(o) - 1)]


def itf8(v):
    v &= 0xffffffff
    if v < 0x80: return bytes([v])
    if v < 0x4000: return bytes([(v >> 8) | 0x80, v & 0xff])
    if v < 0x200000: return bytes([(v >> 16) | 0xc0, (v >> 8) & 0xff, v & 0xff])
    if v < 0x10000000: return bytes([(v >> 24) | 0xe0, (v >> 16) & 0xff, (v >> 8) & 0xff, v & 0xff])
    return bytes([0xf0 | ((v >> 28) & 0xff), (v >> 20) & 0xff, (v >> 12) & 0xff, (v >> 4) & 0xff, v & 0x0f])


def predicted_series(recs, dec):
    """The CF / MF / NS / NP / TS / NF bytes a slice of these records must carry."""
    s = {k: b"" for k in (CF, MF, NS, NP, TS, NF)}
    for (c, d), (b, nf) in zip(recs, dec):
        c = dict(zip(NAMES, c))
        lq, nc, ls = c["l_qname"], c["n_cigar"], c["l_qseq"]
        qual0 = d[lq + 4 * nc + (ls + 1) // 2] if ls > 0 else 0xff
        noseq = not c["flag"] & 4 and ls == 0
        s[CF] += itf8(b | (1 if ls > 0 and qual0 != 0xff else 0) | (8 if noseq else 0))
        if b & 2:
            s[MF] += itf8(0); s[NS] += itf8(c["mtid"]); s[NP] += itf8(c["mpos"] + 1); s[TS] += itf8(c["isize"])
        if b & 4:
            s[NF] += itf8(nf)
    return s


def raw_series(img):
    """Per slice: {content id: payload} of the RAW external blocks."""
    arr = np.frombuffer(img, dtype=np.uint8).copy()
    blocks, _ = H.cram_scan_blocks(arr)
    slices = []
    for b in blocks:
        if int(b["content_type"]) == 2:
            slices.append({})
        elif int(b["content_type"]) == 4 and slices:
            assert int(b["method"]) == 0
            slices[-1][int(b["content_id"])] = arr[int(b["data_off"]):int(b["data_off"]) + int(b["comp_size"])].tobytes()
    return slices


def sam_case(name):
    text, recs = ref_read_sam_records(os.path.join(HT, "sam", name + ".sam"))
    return text, recs, os.path.join(HT, name.split("#")[0] + ".fa")


# ---- 1 and 4: every SAM round trips with attachment; the series bytes are what the rule predicts ----

@pytest.mark.parametrize("rps,minor,with_ref", [(0, 0, False), (0, 1, True), (3, 1, False), (3, 0, True)])
@pytest.mark.parametrize("sam", SAMS)
def test_hostsim_attached_round_trip(tmp_path, sam, rps, minor, with_ref):
    text, recs, fa = sam_case(sam)
    fa = fa if with_ref else None
    try:
        img, dec = encode(None, text, recs, rps, minor, fa)
    except Unsupported as e:
        pytest.skip("left to the host library: %s" % e)
    want = mate_rules(recs, rps, ref_lens_of(text, fa))
    assert dec == want, sam
    _, seen, _ = read_back(tmp_path, img, recs, fa, "rt")
    assert seen == want
    # 4: the mate series of every slice, byte for byte
    r = rps or 10000
    for s, blk in enumerate(raw_series(img)):
        pred = predicted_series(recs[s * r:(s + 1) * r], want[s * r:(s + 1) * r])
        for cid, b in pred.items():
            assert blk.get(cid, b"") == b, (sam, s, cid)


def test_hostsim_without_flag_unchanged():
    """enc_flags = 0: every record detached, no NF series, and the same bytes as the plain entry point."""
    l = hostsim_lib()
    l.hostsim_cram_encode_records.argtypes = [C.c_char_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint32, C.c_int,
                                              C.c_void_p, C.c_void_p]
    for sam in ("xx#pair", "xx#triplet", "ce#unmap2"):
        text, recs, _ = sam_case(sam)
        core, data, off = pack(recs)
        out, ln = C.c_void_p(), C.c_uint64(0)
        assert l.hostsim_cram_encode_records(text, len(text), core.ctypes.data, data.ctypes.data, off.ctypes.data, len(recs), None, 0, 1,
                                             C.byref(out), C.byref(ln)) == 0
        plain = C.string_at(out.value, ln.value)
        img, _ = encode(None, text, recs, 0, 1, flags=0)
        assert img == plain
        assert all(NF not in s for s in raw_series(img))


# ---- 2: the same decisions as the reference's writer, where its slice layout is ours ----

def _reference_decisions(tmp_path, sam_path, text, recs, rps, fa, with_ref, version="3.0"):
    out = str(tmp_path / "ref.cram")
    opts = [(MULTI, 1), (SEQS, rps)] + ([] if with_ref else [(NO_REF, 1)])
    assert ref_write_cram(sam_path, fa, out, version, opts) == len(recs)
    _, dec, layout = decode_decisions(open(out, "rb").read(), fa)
    return dec, layout


@pytest.mark.skipif(ref() is None, reason="writes with the reference's writer; oracle/_ref not built")
@pytest.mark.parametrize("with_ref", [False, True])
def test_hostsim_same_decisions_as_reference_writer(tmp_path, with_ref):
    compared = 0
    for sam in SAMS:
        text, recs, fa = sam_case(sam)
        if not recs:
            continue
        rps = len(recs)
        try:
            dec_ref, layout = _reference_decisions(tmp_path, os.path.join(HT, "sam", sam + ".sam"), text, recs, rps, fa, with_ref)
        except (AssertionError, H.HgpuError):
            continue                                              # the reference declines this input or this shape
        if layout != [rps]:
            continue
        try:
            img, dec = encode(None, text, recs, rps, 0, fa if with_ref else None)
        except Unsupported:
            continue
        assert dec == dec_ref, sam
        compared += 1
    assert compared >= 30, compared


@pytest.mark.skipif(ref() is None, reason="the 10 000 synthetic records come from the reference's SAM reader; oracle/_ref not built")
def test_hostsim_synthetic_same_decisions_as_reference_writer(tmp_path):
    sam = str(tmp_path / "syn.sam")
    n = T._synthetic_sam(sam, n=10000, seed=21)
    text, recs = ref_read_sam_records(sam)
    fa = os.path.join(HT, "ce.fa")
    for rps in (10000, 1500):
        for with_ref in (False, True):
            dec_ref, layout = _reference_decisions(tmp_path, sam, text, recs, rps, fa, with_ref)
            assert layout == [min(rps, n - k) for k in range(0, n, rps)], layout
            img, dec = encode(None, text, recs, rps, 0, fa if with_ref else None)
            assert dec == dec_ref == mate_rules(recs, rps, ref_lens_of(text, fa if with_ref else None))
            assert sum(1 for b, _ in dec if b != 2) > 0.9 * n       # nearly every pair in one slice attaches


# ---- 3: hand-made records, one per `goto detached` test ----

HDR = b"@HD\tVN:1.4\n@SQ\tSN:CHROMOSOME_I\tLN:1009800\n@SQ\tSN:CHROMOSOME_II\tLN:5000\n"
SEQ, QUAL = b"ACGTACGTAC", bytes([40]) * 10


def reg2bin(beg, end):
    """hts_reg2bin(beg, end, 14, 5)."""
    end -= 1
    for shift, first in ((14, 4681), (17, 585), (20, 73), (23, 9), (26, 1)):
        if beg >> shift == end >> shift:
            return first + (beg >> shift)
    return 0


def line(name, flag, pos, pnext, tlen, tid=0, mtid=0):
    """One 10M read as sam_parse1 builds it from 'name flag tid pos 30 10M mtid pnext tlen ACGTACGTAC IIIIIIIIII' (1-based
    positions): the name NUL-padded to a multiple of 4 bytes (l_extranul), bin from the alignment span, 4-bit SEQ."""
    nm = name.encode() + b"\0"
    extra = (4 - len(nm) % 4) % 4
    nm += b"\0" * extra
    seq4 = bytes(("=ACMGRSVTWYHKDBN".index(chr(SEQ[i])) << 4) | "=ACMGRSVTWYHKDBN".index(chr(SEQ[i + 1])) for i in range(0, 10, 2))
    data = nm + struct.pack("<I", 10 << 4) + seq4 + QUAL
    return ((pos - 1, tid, reg2bin(pos - 1, pos + 9), 30, extra, flag, len(nm), 1, 10, mtid, pnext - 1, tlen), data)


def pair(name="p", f1=99, f2=147, p1=100, p2=200, t1=110, t2=-110, pn1=None, pn2=None):
    return [line(name, f1, p1, p2 if pn1 is None else pn1, t1), line(name, f2, p2, p1 if pn2 is None else pn2, t2)]


CASES = {
    "attached": pair(),
    "tlen_off_by_one": pair(t1=111),
    "tlen_zero": pair(t1=0, t2=0),
    "pnext_off_by_one": pair(pn2=101),
    "munmap_disagrees": pair(f2=147 | 8),
    "mreverse_disagrees": pair(f2=147 | 0x20),
    "other_reference": [line("p", 99, 100, 200, 110, 0, 1), line("p", 147, 200, 100, -110, 1, 0)],
    "mate_pos_disagrees": [line("p", 99, 100, 201, 110), line("p", 147, 200, 100, -110)],
    "supplementary": pair(f2=147 | 0x800),
    "third_read1": pair() + pair()[:1],
    "repeated_read2": pair() + pair()[1:],
    "triplet": [line("t", 99, 100, 200, 110), line("t", 147, 200, 100, -110), line("t", 1 | 0x10 | 0x20, 100, 200, 110)],
    "secondary_shares_name": pair() + pair(f1=99 | 0x100, f2=147 | 0x100),
    "two_names": pair("a") + pair("b", p1=150, p2=260, t1=120, t2=-120),
}


def _hand_case(tmp_path, key, ctx=None, minor=1, recs=None):
    recs = recs or CASES[key]
    img, dec = encode(ctx, HDR, recs, 0, minor)
    want = mate_rules(recs, 0)
    _, seen, _ = read_back(tmp_path, img, recs, None, key)
    assert seen == want, (key, seen, want)
    if dec is not None:
        assert dec == want, (key, dec, want)
    return want


@pytest.mark.parametrize("key", sorted(CASES))
def test_hostsim_hand_made_branches(tmp_path, key):
    want = _hand_case(tmp_path, key)
    attached = {"attached", "third_read1", "repeated_read2", "triplet", "secondary_shares_name", "two_names"}
    assert any(b != 2 for b, _ in want) == (key in attached), (key, want)


def test_hostsim_hash_collision_never_pairs_different_names(tmp_path):
    """Every name hashed to 0: only the name comparison keeps the groups of different names apart."""
    l = hostsim_lib()
    l.hostsim_cram_enc_hash_mask(0)
    try:
        for key in ("two_names", "secondary_shares_name", "triplet"):
            _hand_case(tmp_path, key)
        # interleaved pairs that would attach across names if names were not compared
        recs = [line("a", 99, 100, 200, 110), line("b", 99, 100, 200, 110), line("b", 147, 200, 100, -110), line("a", 147, 200, 100, -110)]
        assert _hand_case(tmp_path, "inter", recs=recs) == [(4, 2), (4, 0), (0, 0), (0, 0)]
    finally:
        l.hostsim_cram_enc_hash_mask(0xffffffffffffffff)


# ---- 5-7: the device ----

@pytest.mark.gpu
@pytest.mark.parametrize("minor", [0, 1])
def test_gpu_attached_round_trip(tmp_path, minor):
    ctx = H.Context(0)
    done = 0
    for sam in SAMS:
        text, recs, fa = sam_case(sam)
        for with_ref in (False, True):
            rps = 3 if minor else 0
            f = fa if with_ref else None
            try:
                img, _ = encode(ctx, text, recs, rps, minor, f)
            except H.HgpuError as e:
                assert ": -6 " in str(e), (sam, str(e))
                continue
            _, seen, _ = read_back(tmp_path, img, recs, f, "gpu")
            assert seen == mate_rules(recs, rps, ref_lens_of(text, f)), sam
            done += 1
    assert done >= 60
    for key in sorted(CASES):
        _hand_case(tmp_path, key, ctx, minor)
    ctx.close()


@pytest.mark.gpu
def test_gpu_without_flag_same_bytes_as_plain_entry():
    import test_cram_encode as E
    ctx = H.Context(0)
    for sam in ("xx#pair", "xx#triplet", "ce#unmap2", "ce#1000"):
        if sam not in SAMS:
            continue
        text, recs, fa = sam_case(sam)
        for f in (None, fa):
            rc, plain = E.encode(ctx, text, recs, 0, 1, f)
            assert rc == 0
            assert encode(ctx, text, recs, 0, 1, f, flags=0)[0] == plain
    ctx.close()


@pytest.mark.gpu
@pytest.mark.skipif(ref() is None, reason="the 10 000 synthetic records come from the reference's SAM reader; oracle/_ref not built")
def test_gpu_synthetic_attached_smaller_and_same_decisions(tmp_path):
    ctx = H.Context(0)
    sam = str(tmp_path / "syn.sam")
    n = T._synthetic_sam(sam, n=10000, seed=21)
    text, recs = ref_read_sam_records(sam)
    for rps in (0, 1500):
        for fa in (None, os.path.join(HT, "ce.fa")):
            det, _ = encode(ctx, text, recs, rps, 1, fa, flags=0)
            att, _ = encode(ctx, text, recs, rps, 1, fa)
            assert len(att) < len(det), (rps, fa, len(att), len(det))
            _, seen, _ = read_back(tmp_path, att, recs, fa, "att")
            read_back(tmp_path, det, recs, fa, "det")
            _, sim = encode(None, text, recs, rps, 1, fa)
            assert seen == sim == mate_rules(recs, rps, ref_lens_of(text, fa))
    ctx.close()


def _bench_shaped(n_pairs, seed=5):
    """Paired reads shaped like the bench's (150 bp, coordinate-sorted, ~300 bp inserts, a few unmapped mates), built directly
    as bam1_t records: (header text, records)."""
    import random
    rng = random.Random(seed)
    text = b"@HD\tVN:1.4\tSO:coordinate\n@SQ\tSN:chr1\tLN:250000000\n"
    recs, pos = [], 10000
    for i in range(n_pairs):
        pos += rng.randrange(0, 20)
        p2 = pos + rng.randrange(50, 400)
        name = b"r%09d\0" % i
        unm = rng.random() < 0.02
        for which, p, mp in ((0, pos, p2), (1, p2, pos)):
            flag = 1 | (0x40 if which == 0 else 0x80) | (0x10 if which else 0x20)
            cig = struct.pack("<I", 150 << 4)
            ncig, tl = 1, (p2 + 150 - pos) * (1 if which == 0 else -1)
            if unm and which == 1:
                flag, cig, ncig, p, tl = 1 | 0x80 | 4 | 0x20, b"", 0, pos, 0
            if unm and which == 0:
                flag, mp, tl = flag | 8, pos, 0
            seq = rng.randbytes(75)
            qual = bytes([30]) * 150
            d = name + cig + seq + qual
            recs.append(((p - 1, 0, 0, 60, 0, flag, len(name), ncig, 150, 0, mp - 1, tl), d))
    recs.sort(key=lambda r: r[0][0])
    return text, recs


@pytest.mark.gpu
def test_gpu_decisions_equal_hostsim_on_a_million_records():
    """10^6 bench-shaped records, slices of 9 999 so slice cuts split pairs: the device's decisions (read back from its file)
    equal the hostsim pairing pass's."""
    text, recs = _bench_shaped(500000)
    ctx = H.Context(0)
    img, _ = encode(ctx, text, recs, 9999, 1)
    _, sim = encode(None, text, recs, 9999, 1)
    _, seen, layout = decode_decisions(img)
    assert layout == [min(9999, len(recs) - k) for k in range(0, len(recs), 9999)]
    assert seen == sim
    assert sum(1 for b, _ in sim if b != 2) > 0.9 * len(recs)
    ctx.close()
