"""The reference's sam_index_build3 (through tests/_libs.stored_reference) and the BAM files the index tests feed it.

ref_bam_index(img, min_shift) -> (return code, index content): the BAI file, or the CSI file inflated.
The builders lay records into BGZF blocks at chosen cut points, so a test decides where blocks end (mid-record,
exactly at a record end, an empty block between two records) and whether the EOF block is there.
"""
import ctypes as C
import os
import struct
import tempfile
import zlib

import _libs

GOLD_HTS = os.path.join(_libs.GOLD, "htslib")
CIGAR_OPS = "MIDNSHP=X"


@_libs.stored_reference(digest=True)
def ref_bam_index(img, min_shift):
    """sam_index_build3(fn, fnidx, min_shift, 0) of the compiled reference on a temporary copy of img."""
    r = _libs.ref()
    r.sam_index_build3.argtypes = [C.c_char_p, C.c_char_p, C.c_int, C.c_int]
    r.hts_set_log_level.argtypes = [C.c_int]
    r.hts_set_log_level(0)
    with tempfile.TemporaryDirectory() as td:
        fn, fnidx = os.path.join(td, "in.bam"), os.path.join(td, "in.idx")
        with open(fn, "wb") as f:
            f.write(bytes(img))
        ret = r.sam_index_build3(fn.encode(), fnidx.encode(), min_shift, 0)
        if ret != 0:
            return ret, b""
        with open(fnidx, "rb") as f:
            data = f.read()
    return ret, inflate_bgzf(data) if min_shift > 0 else data


@_libs.stored_reference
def ref_bam_index_summary(img, min_shift):
    """(return code, index_summary of the index) of ref_bam_index: what the CPU tests check of the reference's files."""
    ret, content = ref_bam_index.__wrapped__(img, min_shift)
    return ret, index_summary(content, min_shift > 0) if ret == 0 else None


def inflate_bgzf(data):
    """Concatenated payloads of a BGZF (multi-member gzip) image."""
    out = bytearray()
    while data:
        d = zlib.decompressobj(31)
        out += d.decompress(data)
        data = d.unused_data
    return bytes(out)


def reg2bin(beg, end):
    end -= 1
    for s, first in ((14, 4681), (17, 585), (20, 73), (23, 9), (26, 1)):
        if beg >> s == end >> s:
            return first + (beg >> s)
    return 0


def header(refs, text=b"@HD\tVN:1.6\tSO:coordinate\n"):
    """BAM header (SAM spec 4.2): refs = [(name, length)]."""
    text = text + b"".join(b"@SQ\tSN:%s\tLN:%d\n" % (n, l) for n, l in refs)
    out = b"BAM\1" + struct.pack("<i", len(text)) + text + struct.pack("<i", len(refs))
    for n, l in refs:
        out += struct.pack("<i", len(n) + 1) + n + b"\0" + struct.pack("<I", l)
    return out


def record(tid, pos, cigar=((100, "M"),), flag=0, name=b"r", l_seq=None, mtid=None, mpos=-1, aux=b"", raw_cigar=None):
    """One BAM record (block_size included).  cigar: (length, op) pairs; raw_cigar: uint32 words as they are."""
    words = list(raw_cigar) if raw_cigar is not None else [(n << 4) | CIGAR_OPS.index(o) for n, o in cigar]
    if l_seq is None:
        l_seq = sum(n for n, o in cigar if o in "MIS=X") if raw_cigar is None else 0
    rlen = sum(n for n, o in cigar if o in "MDN=X") if raw_cigar is None else 1
    b = reg2bin(max(pos, 0), max(pos, 0) + max(rlen, 1)) if tid >= 0 else 4680
    body = struct.pack("<iiBBHHHiiii", tid, pos, len(name) + 1, 60, b, len(words), flag, l_seq,
                       tid if mtid is None else mtid, mpos, 0)
    body += name + b"\0" + struct.pack("<%dI" % len(words), *words) + b"\x11" * ((l_seq + 1) // 2) + b"\x1e" * l_seq + aux
    return struct.pack("<i", len(body)) + body


def cg_record(tid, pos, n_pairs, name=b"cg"):
    """A record whose real CIGAR (n_pairs x 1M1N, more ops than n_cigar holds) sits in a CG:B,I tag behind the
    <qlen>S<rlen>N placeholder, as bam_write1 stores long CIGARs (sam.c:899-925)."""
    real = [(1 << 4) | 0, (1 << 4) | 3] * n_pairs
    qlen, rlen = n_pairs, 2 * n_pairs
    fake = [(qlen << 4) | 4, (rlen << 4) | 3]
    aux = b"CGBI" + struct.pack("<I", len(real)) + struct.pack("<%dI" % len(real), *real)
    body = struct.pack("<iiBBHHHiiii", tid, pos, len(name) + 1, 60, reg2bin(pos, pos + rlen), 2, 0, qlen, tid, -1, 0)
    body += name + b"\0" + struct.pack("<2I", *fake) + b"\x11" * ((qlen + 1) // 2) + b"\x1e" * qlen + aux
    return struct.pack("<i", len(body)) + body


def bgzf(stream, cuts=(), level=6, eof=True, empty_at=(), block=0xff00):
    """stream cut into BGZF blocks: a block ends at every position in cuts and wherever a block reaches `block`
    bytes; an empty block is written after each block that ends at a position in empty_at."""
    ends = sorted(set(c for c in cuts if 0 < c < len(stream)) | {len(stream)})
    out, start = bytearray(), 0
    for e in ends:
        while e - start > block:
            out += _libs.bgzf_block(stream[start:start + block], level)
            start += block
        out += _libs.bgzf_block(stream[start:e], level)
        if e in empty_at:
            out += _libs.bgzf_block(b"", level)
        start = e
    if eof:
        out += _libs.BGZF_EOF
    return bytes(out)


REFS = [(b"chr1", 249250621), (b"chr2", 10000000), (b"chr3", 1000000)]


def multi_records():
    """Several references (chr2 without records), unmapped-placed reads, spliced reads whose N ops cross many 16 kb
    windows and reach high-level bins, a CG-tag long CIGAR, and an unplaced tail."""
    recs = []
    pos = 10000
    for i in range(600):
        pos += 37 + (i * 7919) % 400
        if i % 50 == 7:
            recs.append(record(0, pos, ((60, "M"), (3000000 + 1000 * i, "N"), (40, "M")), name=b"splice%d" % i))
        elif i % 40 == 3:
            recs.append(record(0, pos, (), flag=4 | 1, name=b"umap%d" % i, l_seq=100))
        elif i == 300:
            recs.append(cg_record(0, pos, 40000))
        else:
            recs.append(record(0, pos, ((30, "M"), (2, "D"), (70, "M")), name=b"read%d" % i))
    pos = 500
    for i in range(200):
        pos += 11 + (i * 104729) % 3000
        recs.append(record(2, pos, ((100, "M"),), name=b"c3_%d" % i, flag=16 if i & 1 else 0))
    for i in range(30):
        recs.append(record(-1, -1, (), flag=4, name=b"unplaced%d" % i, l_seq=80, mtid=-1))
    return recs


def multi_stream(recs=None):
    recs = multi_records() if recs is None else recs
    hdr = header(REFS)
    ends, p = [], len(hdr)
    for r in recs:
        p += len(r)
        ends.append(p)
    return hdr + b"".join(recs), len(hdr), ends


def multi_files():
    """name -> BGZF image of the multi stream, block layouts that exercise the virtual-offset rules."""
    stream, hlen, ends = multi_stream()
    exact = [ends[i] for i in (5, 40, 41, 250, 601, 799)]              # blocks that end exactly at a record end
    mid = [hlen + 100, ends[100] + 17, ends[400] - 9]                   # header ends mid-block; cuts inside records
    cuts = exact + mid
    return {
        "multi_l6": bgzf(stream, cuts, 6, empty_at=(ends[40],)),
        "multi_l0": bgzf(stream, cuts, 0, empty_at=(ends[40],)),
        "multi_l6_noeof": bgzf(stream, cuts, 6, eof=False),
        "multi_l0_noeof_empty_tail": bgzf(stream, cuts, 0, eof=False, empty_at=(len(stream),)),
        "multi_trailing_empty": bgzf(stream, cuts, 6, empty_at=(ends[250], len(stream))),
    }


def big_ref_file():
    """A 600 Mbp reference: CSI needs 6 levels at min_shift 14, BAI refuses the first record that reaches past 2^29."""
    hdr = header([(b"big", 600000000)])
    recs = [record(0, p, name=b"b%d" % i) for i, p in enumerate((100, 20000, 100000000, 536870000, 536870900, 590000000))]
    return bgzf(hdr + b"".join(recs), (len(hdr) + 5,), 6)


def synth_file(total=256 << 20, n_sq=4, seed=7):
    """About `total` bytes of synthetic 30x-like records (tools/synth.bam_records) over n_sq references, each shard
    on its own stretch of its reference, then a few unplaced reads; BGZF blocks cut as the reference's writer does."""
    import multiprocessing as mp
    per_shard = 20000
    n_shards = max(1, total // (336 * per_shard))
    jobs, seen = [], {}
    for s in range(n_shards):
        t = s * n_sq // n_shards
        k = seen.get(t, 0)
        seen[t] = k + 1
        jobs.append((seed * 1000 + s, per_shard, t, 10000 + k * 120000))     # a shard spans ~100 kbp
    with mp.get_context("spawn").Pool(min(len(jobs), len(os.sched_getaffinity(0)))) as pool:
        parts = pool.map(_synth_shard, jobs, chunksize=1)
    hdr = header([(b"sq%d" % t, 250000000) for t in range(n_sq)])
    tail = b"".join(record(-1, -1, (), flag=4, name=b"u%d" % i, l_seq=150, mtid=-1) for i in range(100))
    return _pack(hdr + b"".join(parts) + tail, len(hdr))


def _synth_shard(job):
    import sys
    sys.path.insert(0, _libs.ROOT)
    from tools import synth
    seed, n, tid, pos0 = job
    return synth.bam_records(seed, n, tid=tid, pos0=pos0)[0]


def _pack(stream, hlen):
    """Blocks of the reference's writer: the header alone, then records packed so that none is split unless it must be."""
    cuts, p, start = [hlen], hlen, hlen
    while p < len(stream):
        n = 4 + struct.unpack_from("<i", stream, p)[0]
        if p + n - start > 0xff00 and p > start:
            cuts.append(p)
            start = p
        p += n
    return bgzf(stream, cuts, 6)


def refusal_cases():
    """name -> (image, "push" | "read" | "block", the record or block the reference stops at): each refusal injected into
    the multi stream."""
    recs = multi_records()

    def with_rec(i, r):
        out = list(recs)
        out[i] = r
        return out

    def image(rs, trim=0):
        stream, hlen, ends = multi_stream(rs)
        return bgzf(stream[:len(stream) - trim], (hlen + 100, ends[250]), 6)

    corrupt = bytearray(multi_files()["multi_l6"])
    starts, p = [], 0
    while p < len(corrupt):
        starts.append(p)
        p += int.from_bytes(corrupt[p + 16:p + 18], "little") + 1
    corrupt[starts[2] + 40] ^= 0x55                     # inside block 2's deflate data
    pos20 = struct.unpack_from("<i", recs[20], 8)[0]
    return {
        "swapped": (image(with_rec(11, record(0, 100, name=b"early"))), "push", 11),
        "tid_returns": (image(with_rec(700, record(0, 5000000, name=b"back"))), "push", 700),
        "placed_after_unplaced": (image(with_rec(805, record(2, 999000, name=b"late"))), "push", 805),
        "tid_out_of_range": (image(with_rec(650, record(3, 1000, name=b"far"))), "read", 650),
        "truncated_last": (image(recs, trim=10), "read", len(recs) - 1),
        "cigar_qlen": (image(with_rec(20, record(0, pos20, ((100, "M"),), l_seq=90))), "read", 20),
        "corrupt_block": (bytes(corrupt), "block", 2),
    }


def index_bam():
    with open(os.path.join(GOLD_HTS, "index.bam"), "rb") as f:
        return f.read()


def index_summary(content, csi):
    """(n_ref, per-reference bin counts, n_no_coor) read back from an index file's content (SAM spec 5.2 / CSI spec)."""
    p = 4
    if csi:
        l_meta = struct.unpack_from("<I", content, 12)[0]
        p = 16 + l_meta
    n_ref = struct.unpack_from("<i", content, p)[0]
    p += 4
    bins = []
    for _ in range(n_ref):
        nb = struct.unpack_from("<i", content, p)[0]
        p += 4
        bins.append(nb)
        for _ in range(nb):
            p += 4 + (8 if csi else 0)
            nc = struct.unpack_from("<i", content, p)[0]
            p += 4 + 16 * nc
        if not csi:
            ni = struct.unpack_from("<i", content, p)[0]
            p += 4 + 8 * ni
    n_no_coor = struct.unpack_from("<Q", content, p)[0]
    assert p + 8 == len(content)
    return n_ref, bins, n_no_coor
