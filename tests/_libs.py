"""ctypes loaders for the three libraries the tests compare.

  orc()  -> oracle/liborc.so          CPU restatement (test infrastructure)
  ref()  -> oracle/_ref/libhts_ref.so unmodified reference (htslib + htscodecs), built by oracle/build_ref.sh
                                      from the reference sources; usually absent
  The product library is loaded through htslib_b200 itself.

Every ref_* helper answers from tests/golden/ref_calls/: what the compiled reference returned for the
same arguments, recorded once.  So the comparisons with the reference run where the reference was never
built.  Only results of up to STORE_LIMIT characters are stored (more for the helpers that read or
write the reference's own fixtures), which keeps the small cases of every test.  Where oracle/_ref is
absent, a case whose result is not stored is passed over (`with sampled():` around one case of a loop)
and a test that needs one outside such a block is skipped; where oracle/_ref is built every case runs.
To store the results of new inputs, build oracle/_ref and run the tests with
HTS_REF_RECORD=tests/golden/ref_calls.
"""
import atexit
import ast
import contextlib
import ctypes as C
import functools
import gzip
import hashlib
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")
REF_CALLS = os.path.join(GOLD, "ref_calls")
STORE_LIMIT = 1500
u8p = C.POINTER(C.c_uint8)
_orc = _ref = None
_stored = {}          # helper name -> {key: repr of the result}
_used = {}            # helper name -> {key: repr of the result} of every call in this process
_limit = {}           # helper name -> longest result stored
_always = set()       # (helper name, key) stored whatever their size: the base streams of the corruption tests


def _canon(x, h):
    """Feed an argument into the key: byte strings and files by content, everything else by repr."""
    if isinstance(x, (bytes, bytearray, memoryview)):
        h.update(b"B%d:" % len(x)); h.update(bytes(x))
    elif isinstance(x, str) and os.path.isfile(x):
        with open(x, "rb") as f:
            data = f.read()
        h.update(b"F%d:" % len(data)); h.update(data)
    elif isinstance(x, (list, tuple)):
        h.update(b"L%d[" % len(x))
        for v in x:
            _canon(v, h)
        h.update(b"]")
    elif hasattr(x, "tolist"):                    # numpy arrays and scalars
        _canon(x.tolist(), h)
    elif isinstance(x, (int, float, str, type(None))):
        h.update(b"V" + repr(x).encode() + b";")
    else:
        raise TypeError("reference call argument of type %s" % type(x).__name__)


def _load(name):
    if name not in _stored:
        d = {}
        p = os.path.join(REF_CALLS, name + ".gz")
        if os.path.exists(p):
            with gzip.open(p, "rt") as f:
                for line in f:
                    k, _, v = line.rstrip("\n").partition("\t")
                    d[k] = v
        _stored[name] = d
    return _stored[name]


def _flush():
    """HTS_REF_RECORD=<dir>: add every result this process used to <dir>/<helper>.gz."""
    out = os.environ.get("HTS_REF_RECORD")
    if not out or not _used:
        return
    os.makedirs(out, exist_ok=True)
    for name, used in _used.items():
        d = {}
        p = os.path.join(out, name + ".gz")
        if os.path.exists(p):
            with gzip.open(p, "rt") as f:
                for line in f:
                    k, _, v = line.rstrip("\n").partition("\t")
                    d[k] = v
        d.update((k, v) for k, v in used.items() if len(v) <= _limit[name] or (name, k) in _always)
        with open(p, "wb") as raw, gzip.GzipFile(fileobj=raw, mode="wb", compresslevel=9, mtime=0) as f:
            f.write("".join("%s\t%s\n" % kv for kv in sorted(d.items())).encode())


atexit.register(_flush)


class Digest:
    """A byte string the reference returned, kept as its length, the first 64 bits of its SHA-256 and its
    first bytes: equal to exactly that string.  Stands for decoder outputs, which the tests only compare;
    strings shorter than MIN (names, short fields) are kept as they are."""
    HEAD = 4
    MIN = 64

    def __init__(self, n, sha, head):
        self.n, self.sha, self.head = n, sha, head

    def __eq__(self, other):
        if isinstance(other, Digest):
            return (self.n, self.sha) == (other.n, other.sha)
        if isinstance(other, (bytes, bytearray, memoryview)):
            return len(other) == self.n and hashlib.sha256(other).hexdigest()[:16] == self.sha
        return NotImplemented

    __hash__ = None

    def __len__(self):
        return self.n

    def __getitem__(self, i):
        if isinstance(i, int) and 0 <= i < len(self.head):
            return self.head[i]
        raise IndexError("only the first %d bytes of a stored decoder output are kept" % self.HEAD)

    def __repr__(self):
        return "<%d bytes, sha256 %s...>" % (self.n, self.sha)


_DIGEST_TAG = "sha256-of-bytes"


def _shrink(v):
    if isinstance(v, (bytes, bytearray)) and len(v) >= Digest.MIN:
        return (_DIGEST_TAG, len(v), hashlib.sha256(v).hexdigest()[:16], bytes(v[:Digest.HEAD]))
    if isinstance(v, (list, tuple)):
        return type(v)(_shrink(x) for x in v)
    return v


def _grow(v):
    if isinstance(v, tuple) and len(v) == 4 and v[0] == _DIGEST_TAG:
        return Digest(v[1], v[2], v[3])
    if isinstance(v, (list, tuple)):
        return type(v)(_grow(x) for x in v)
    return v


class NotStored(pytest.skip.Exception):
    """A reference result that is not among the stored ones, with no compiled reference to compute it."""


@contextlib.contextmanager
def sampled():
    """One case of a loop over inputs: passed over when one of its reference results is not stored."""
    try:
        yield
    except NotStored:
        pass


def stored_reference(fn=None, *, digest=False, limit=STORE_LIMIT):
    """The result of fn (a call into the compiled reference) for these arguments, from the stored results.
    fn must return plain values (bytes, str, numbers, None, tuples, lists) and take content-keyed arguments.
    digest: keep byte strings of the result as Digest (True, or a predicate of the keyword arguments).
    limit: longest result (characters of its repr) that is stored; a call with store_always=True is stored
    whatever its size."""
    if fn is None:
        return functools.partial(stored_reference, digest=digest, limit=limit)
    name = fn.__name__
    _limit[name] = limit

    @functools.wraps(fn)
    def call(*args, store_always=False, **kw):
        h = hashlib.sha256(name.encode())
        _canon(args + tuple(sorted(kw.items())), h)
        key = h.hexdigest()[:16]
        if store_always:
            _always.add((name, key))
        v = _load(name).get(key) or _used.get(name, {}).get(key)
        if v is None:
            if ref() is None:
                raise NotStored("%s%s: no stored reference result and oracle/_ref not built" % (name, _short(args)))
            res = fn(*args, **kw)
            v = repr(_shrink(res) if (digest(kw) if callable(digest) else digest) else res)
        _used.setdefault(name, {})[key] = v
        return _grow(ast.literal_eval(v))
    return call


def _short(args):
    s = repr(tuple(a if not isinstance(a, (bytes, bytearray)) or len(a) < 32 else "<%d bytes>" % len(a) for a in args))
    return s[:300]


def orc():
    global _orc
    if _orc is None:
        so = os.path.join(ROOT, "oracle", "liborc.so")
        srcs = [os.path.join(ROOT, "oracle", f) for f in os.listdir(os.path.join(ROOT, "oracle")) if f.endswith(".c")]
        if not os.path.exists(so) or any(os.path.getmtime(s) > os.path.getmtime(so) for s in srcs):
            subprocess.check_call(["make", "-C", os.path.join(ROOT, "oracle"), "liborc.so"])
        _orc = C.CDLL(so)
    return _orc


def ref():
    """The compiled reference, or None when it was never built."""
    global _ref
    if _ref is None:
        so = os.path.join(ROOT, "oracle", "_ref", "libhts_ref.so")
        if not os.path.exists(so):
            return None
        _ref = C.CDLL(so)
        _ref.rans_uncompress_to_4x16.restype = C.c_void_p
        _ref.rans_compress_to_4x16.restype = C.c_void_p
        _ref.rans_compress_bound_4x16.restype = C.c_uint
    return _ref


def buf(b):
    return (C.c_uint8 * max(1, len(b))).from_buffer_copy(bytes(b) + (b"\0" if len(b) == 0 else b""))


def orc_rans_nx16_decode(data, out_size):
    o = orc()
    out = (C.c_uint8 * max(1, out_size))()
    n = C.c_uint32(out_size)
    rc = o.orc_rans_nx16_decode(buf(data), C.c_uint32(len(data)), out, C.byref(n))
    if rc != 0:
        return None
    return bytes(out[: n.value])


@stored_reference(digest=True)
def ref_rans_nx16_decode(data, out_size):
    r = ref()
    out = (C.c_uint8 * max(1, out_size))()
    n = C.c_uint(out_size)
    p = r.rans_uncompress_to_4x16(buf(data), C.c_uint(len(data)), out, C.byref(n))
    if not p:
        return None
    return bytes(out[: n.value])


@stored_reference
def ref_rans_nx16_encode(data, order):
    r = ref()
    cap = r.rans_compress_bound_4x16(C.c_uint(len(data)), C.c_int(order))
    out = (C.c_uint8 * max(1, cap))()
    n = C.c_uint(cap)
    p = r.rans_compress_to_4x16(buf(data), C.c_uint(len(data)), out, C.byref(n), C.c_int(order))
    assert p, "reference encoder failed"
    return bytes(out[: n.value])


@stored_reference(digest=True)
def ref_rans_nx16_decode_scalar(data, out_size):
    """ref_rans_nx16_decode through the reference's scalar decoders (rans_set_cpu(0), rANS_static4x16pr.c:1191):
    its SIMD decoders read differently once a damaged stream runs dry."""
    r = ref()
    r.rans_set_cpu(0)
    try:
        return ref_rans_nx16_decode.__wrapped__(data, out_size)
    finally:
        r.rans_set_cpu(-1)


@stored_reference(digest=True)
def ref_rans_nx16_encoded(data, order):
    """ref_rans_nx16_encode as a Digest (length, first bytes, hash): for tests that only compare with it."""
    return ref_rans_nx16_encode.__wrapped__(data, order)


@stored_reference(digest=True)
def ref_rans_4x8_encoded(data, order):
    """ref_rans_4x8(data, order) as a Digest."""
    return ref_rans_4x8.__wrapped__(data, order)


@stored_reference(digest=True)
def ref_arith_encoded(data, order):
    """ref_arith(data, order) as a Digest."""
    return ref_arith.__wrapped__(data, order)


@stored_reference(digest=True)
def ref_fqz_compressed(quals, lens, flags=None, strat=0, vers=4):
    """ref_fqz_compress as a Digest."""
    return ref_fqz_compress.__wrapped__(quals, lens, flags, strat, vers)


@stored_reference
def ref_arith_compress_bounds(pairs):
    """arith_compress_bound(size, order) for every (size, order) pair."""
    r = ref()
    r.arith_compress_bound.restype = C.c_uint
    return [r.arith_compress_bound(C.c_uint(s), C.c_int(o)) for s, o in pairs]


def golden_raw(name):
    """The raw input the htscodecs tests feed: first column, newlines removed (rans4x16.test:12)."""
    path = os.path.join(GOLD, "htscodecs", "dat", name)
    if not name.startswith("q"):              # u32 is used verbatim (arith.test:11-18)
        return open(path, "rb").read()
    out = bytearray()
    with open(path, "rb") as f:
        for line in f:
            out += line.rstrip(b"\n").split(b"\t")[0]
    return bytes(out)


# ---------------------------------------------------------------- BGZF helpers
import struct, zlib

BGZF_EOF = bytes.fromhex("1f8b08040000000000ff0600424302001b0003000000000000000000")


def bgzf_block(payload, level=6, raw_deflate=None):
    """One BGZF block the way bgzf_compress's zlib arm writes it (bgzf.c:624-683):
    deflateInit2(level, Z_DEFLATED, -15, 8, Z_DEFAULT_STRATEGY) + header + CRC32 + ISIZE."""
    if raw_deflate is None:
        if level == 0:   # bgzf.c:573-580 stored block
            raw_deflate = b"\x01" + struct.pack("<HH", len(payload), len(payload) ^ 0xffff) + payload
        else:
            c = zlib.compressobj(level, zlib.DEFLATED, -15, 8)
            raw_deflate = c.compress(payload) + c.flush()
    bsize = 18 + len(raw_deflate) + 8
    assert bsize <= 65536
    hdr = b"\x1f\x8b\x08\x04\0\0\0\0\0\xff\x06\0BC\x02\0" + struct.pack("<H", bsize - 1)
    return hdr + raw_deflate + struct.pack("<II", zlib.crc32(payload) & 0xffffffff, len(payload))


def bgzf_file(data, level=6, block=0xff00, eof=True):
    out = bytearray()
    for i in range(0, len(data), block):
        out += bgzf_block(data[i:i + block], level)
    if eof:
        out += BGZF_EOF
    return bytes(out)


def orc_inflate_raw(src, cap=65536):
    o = orc()
    out = (C.c_uint8 * max(1, cap))()
    dl = C.c_uint64(0); used = C.c_uint64(0)
    rc = o.orc_inflate_raw(buf(src), C.c_uint64(len(src)), out, C.c_uint64(cap), C.byref(dl), C.byref(used))
    if rc:
        return None, 0
    return bytes(out[: dl.value]), used.value


class _OrcTrace(C.Structure):
    _fields_ = [("max_blocks", C.c_uint32), ("max_toks", C.c_uint32), ("nblocks", C.c_uint32), ("ntoks", C.c_uint32),
                ("btype", C.POINTER(C.c_uint8)), ("start_bit", C.POINTER(C.c_uint64)), ("body_bit", C.POINTER(C.c_uint64)),
                ("end_bit", C.POINTER(C.c_uint64)), ("first_tok", C.POINTER(C.c_uint32)), ("lens", C.POINTER(C.c_uint8)),
                ("toks", C.POINTER(C.c_uint32))]


def orc_inflate_trace(src, cap=65536, max_blocks=4096):
    """Raw inflate with the oracle's per-block trace.  Returns (output, blocks) or (None, None) on an inflate error.
    Each block is a dict: bfinal, btype, start_bit, body_bit, end_bit, ll (288 lit/len code lengths), dist (32),
    cl (19, indexed by code-length symbol) and toks, a list of literal bytes (int) and (length, distance) tuples."""
    import numpy as np
    o = orc()
    out = (C.c_uint8 * max(1, cap))()
    dl = C.c_uint64(0); used = C.c_uint64(0)
    arrs = dict(btype=(C.c_uint8 * max_blocks)(), start_bit=(C.c_uint64 * max_blocks)(), body_bit=(C.c_uint64 * max_blocks)(),
                end_bit=(C.c_uint64 * max_blocks)(), first_tok=(C.c_uint32 * max_blocks)(), lens=(C.c_uint8 * (max_blocks * 339))(),
                toks=(C.c_uint32 * max(1, cap))())
    t = _OrcTrace(max_blocks, max(1, cap), 0, 0, *(C.cast(arrs[k], C.POINTER(f)) for k, f in
                  (("btype", C.c_uint8), ("start_bit", C.c_uint64), ("body_bit", C.c_uint64), ("end_bit", C.c_uint64),
                   ("first_tok", C.c_uint32), ("lens", C.c_uint8), ("toks", C.c_uint32))))
    rc = o.orc_inflate_trace(buf(src), C.c_uint64(len(src)), out, C.c_uint64(cap), C.byref(dl), C.byref(used), C.byref(t))
    if rc:
        return None, None
    toks = np.frombuffer(arrs["toks"], dtype=np.uint32, count=t.ntoks)
    lens = np.frombuffer(arrs["lens"], dtype=np.uint8, count=t.nblocks * 339).reshape(-1, 339)
    blocks = []
    for k in range(t.nblocks):
        end = arrs["first_tok"][k + 1] if k + 1 < t.nblocks else t.ntoks
        tk = toks[arrs["first_tok"][k]:end]
        blocks.append(dict(bfinal=arrs["btype"][k] & 1, btype=arrs["btype"][k] >> 1, start_bit=arrs["start_bit"][k],
                           body_bit=arrs["body_bit"][k], end_bit=arrs["end_bit"][k], ll=lens[k, :288].tolist(),
                           dist=lens[k, 288:320].tolist(), cl=lens[k, 320:].tolist(),
                           toks=[int(v) if v < 256 else ((int(v) >> 16) & 0x1ff, int(v) & 0xffff) for v in tk]))
    return bytes(out[: dl.value]), blocks


def orc_bgzf_inflate_block(block):
    o = orc()
    out = (C.c_uint8 * 65536)()
    rc = o.orc_bgzf_inflate_block(buf(block), C.c_uint32(len(block)), out)
    return rc, (bytes(out[:rc]) if rc >= 0 else b"")


def orc_bgzf_scan(data):
    o = orc()
    o.orc_bgzf_scan.restype = C.c_long
    cap = len(data) // 26 + 2
    off = (C.c_uint64 * cap)(); ln = (C.c_uint32 * cap)()
    n = o.orc_bgzf_scan(buf(data), C.c_uint64(len(data)), off, ln, C.c_long(cap))
    if n < 0:
        return n, []
    return n, [(off[i], ln[i]) for i in range(n)]


@stored_reference(digest=True)
def ref_bgzf_read_all(data, threads=0):
    """Decompress a whole BGZF file image with the compiled reference: hopen("mem:") ->
    bgzf_hopen -> [bgzf_mt] -> bgzf_read loop.  Returns (bytes, errcode)."""
    r = ref()
    r.hopen.restype = C.c_void_p
    r.hopen.argtypes = [C.c_char_p, C.c_char_p, C.c_void_p, C.c_size_t]
    r.bgzf_hopen.restype = C.c_void_p
    r.bgzf_hopen.argtypes = [C.c_void_p, C.c_char_p]
    r.bgzf_read.restype = C.c_ssize_t
    r.bgzf_read.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t]
    r.bgzf_close.argtypes = [C.c_void_p]
    r.bgzf_mt.argtypes = [C.c_void_p, C.c_int, C.c_int]
    # the mem: backend takes ownership of a malloc'ed buffer and frees it at close (hfile.c:837)
    libc = C.CDLL(None)
    libc.malloc.restype = C.c_void_p
    libc.malloc.argtypes = [C.c_size_t]
    mem = libc.malloc(max(1, len(data)))
    C.memmove(mem, bytes(data), len(data))
    hf = r.hopen(b"mem:", b"r:", mem, len(data))
    assert hf
    fp = r.bgzf_hopen(hf, b"r")
    assert fp
    if threads:
        r.bgzf_mt(fp, threads, 256)
    out = bytearray()
    chunk = (C.c_uint8 * (1 << 20))()
    err = 0
    while True:
        n = r.bgzf_read(fp, chunk, len(chunk))
        if n < 0:
            err = 1
            break
        if n == 0:
            break
        out += bytes(chunk[:n])
    r.bgzf_close(fp)
    return bytes(out), err


# ---------------------------------------------------------------- BAM helpers
class BamCore(C.Structure):
    _fields_ = [("pos", C.c_int64), ("tid", C.c_int32), ("bin", C.c_uint16), ("qual", C.c_uint8),
                ("l_extranul", C.c_uint8), ("flag", C.c_uint16), ("l_qname", C.c_uint16),
                ("n_cigar", C.c_uint32), ("l_qseq", C.c_int32), ("mtid", C.c_int32),
                ("mpos", C.c_int64), ("isize", C.c_int64)]

    def astuple(self):
        return tuple(getattr(self, f) for f, _ in self._fields_)


class Bam1(C.Structure):          # bam1_t, htslib/sam.h:253-260
    _fields_ = [("core", BamCore), ("id", C.c_uint64), ("data", C.POINTER(C.c_uint8)), ("l_data", C.c_int),
                ("m_data", C.c_uint32), ("mempolicy", C.c_uint32)]


def bam_header_len(stream):
    """Length of the BAM header at the start of an inflated BAM stream (SAM spec 4.2)."""
    assert stream[:4] == b"BAM\1"
    l_text = struct.unpack_from("<i", stream, 4)[0]
    p = 8 + l_text
    n_ref = struct.unpack_from("<i", stream, p)[0]
    p += 4
    for _ in range(n_ref):
        l_name = struct.unpack_from("<i", stream, p)[0]
        p += 4 + l_name + 4
    return p


def bam_header(n_ref=1, name=b"chr1", length=250000000):
    text = b"@HD\tVN:1.6\tSO:coordinate\n@SQ\tSN:%s\tLN:%d\n@RG\tID:grp1\n" % (name, length)
    return b"BAM\1" + struct.pack("<i", len(text)) + text + struct.pack("<i", n_ref) + \
        struct.pack("<i", len(name) + 1) + name + b"\0" + struct.pack("<i", length)


@stored_reference(digest=True, limit=400000)
def ref_bam_read_all(img):
    """Every record of a BGZF BAM image through the compiled reference's bam_hdr_read + bam_read1.
    Returns list of (core tuple, data bytes, return code)."""
    r = ref()
    r.hopen.restype = C.c_void_p
    r.hopen.argtypes = [C.c_char_p, C.c_char_p, C.c_void_p, C.c_size_t]
    r.bgzf_hopen.restype = C.c_void_p
    r.bgzf_hopen.argtypes = [C.c_void_p, C.c_char_p]
    r.bgzf_close.argtypes = [C.c_void_p]
    r.bam_hdr_read.restype = C.c_void_p
    r.bam_hdr_read.argtypes = [C.c_void_p]
    r.sam_hdr_destroy.argtypes = [C.c_void_p]
    r.bam_init1.restype = C.POINTER(Bam1)
    r.bam_read1.argtypes = [C.c_void_p, C.POINTER(Bam1)]
    r.bam_destroy1.argtypes = [C.POINTER(Bam1)]
    libc = C.CDLL(None)
    libc.malloc.restype = C.c_void_p
    libc.malloc.argtypes = [C.c_size_t]
    mem = libc.malloc(max(1, len(img)))
    C.memmove(mem, bytes(img), len(img))
    fp = r.bgzf_hopen(r.hopen(b"mem:", b"r:", mem, len(img)), b"r")
    hdr = r.bam_hdr_read(fp)
    assert hdr
    b = r.bam_init1()
    out = []
    while True:
        rc = r.bam_read1(fp, b)
        if rc < 0:
            if rc != -1:
                out.append((None, None, rc))
            break
        out.append((b.contents.core.astuple(), bytes(b.contents.data[: b.contents.l_data]), rc))
    r.bam_destroy1(b)
    r.sam_hdr_destroy(hdr)
    r.bgzf_close(fp)
    return out


class KString(C.Structure):       # kstring_t, htslib/kstring.h
    _fields_ = [("l", C.c_size_t), ("m", C.c_size_t), ("s", C.c_void_p)]


@stored_reference(digest=True, limit=200000)
def ref_sam_format_all(img):
    """Every record of a BGZF BAM image through the compiled reference's bam_read1 + sam_format1.
    Returns (target names, [line bytes or None when sam_format1 fails])."""
    r = ref()
    r.hopen.restype = C.c_void_p
    r.hopen.argtypes = [C.c_char_p, C.c_char_p, C.c_void_p, C.c_size_t]
    r.bgzf_hopen.restype = C.c_void_p
    r.bgzf_hopen.argtypes = [C.c_void_p, C.c_char_p]
    r.bgzf_close.argtypes = [C.c_void_p]
    r.bam_hdr_read.restype = C.c_void_p
    r.bam_hdr_read.argtypes = [C.c_void_p]
    r.sam_hdr_destroy.argtypes = [C.c_void_p]
    r.sam_hdr_nref.argtypes = [C.c_void_p]
    r.sam_hdr_tid2name.restype = C.c_char_p
    r.sam_hdr_tid2name.argtypes = [C.c_void_p, C.c_int]
    r.bam_init1.restype = C.POINTER(Bam1)
    r.bam_read1.argtypes = [C.c_void_p, C.POINTER(Bam1)]
    r.bam_destroy1.argtypes = [C.POINTER(Bam1)]
    r.sam_format1.argtypes = [C.c_void_p, C.POINTER(Bam1), C.POINTER(KString)]
    libc = C.CDLL(None)
    libc.malloc.restype = C.c_void_p
    libc.malloc.argtypes = [C.c_size_t]
    libc.free.argtypes = [C.c_void_p]
    mem = libc.malloc(max(1, len(img)))
    C.memmove(mem, bytes(img), len(img))
    fp = r.bgzf_hopen(r.hopen(b"mem:", b"r:", mem, len(img)), b"r")
    hdr = r.bam_hdr_read(fp)
    assert hdr
    names = [r.sam_hdr_tid2name(hdr, i) for i in range(r.sam_hdr_nref(hdr))]
    b = r.bam_init1()
    ks = KString(0, 0, None)
    lines = []
    while r.bam_read1(fp, b) >= 0:
        n = r.sam_format1(hdr, b, C.byref(ks))
        lines.append(C.string_at(ks.s, ks.l) if n >= 0 else None)
    if ks.s:
        libc.free(ks.s)
    r.bam_destroy1(b)
    r.sam_hdr_destroy(hdr)
    r.bgzf_close(fp)
    return names, lines


def orc_bam_unpack_all(stream):
    """Records of an inflated BAM record stream (header already removed) through the oracle.
    Returns list of (status, core tuple, data, seq, qual) or raises on a broken chain."""
    o = orc()
    o.orc_bam_index.restype = C.c_long
    sb = buf(stream)
    cap = len(stream) // 36 + 1
    offs = (C.c_uint64 * cap)()
    n = o.orc_bam_index(sb, C.c_uint64(len(stream)), offs, C.c_long(cap))
    if n < 0:
        raise ValueError("broken chain at record %d" % (-1 - n))
    res = []
    base = C.addressof(sb)
    for i in range(n):
        ld, lq = C.c_uint32(0), C.c_uint32(0)
        p = C.cast(base + offs[i], C.POINTER(C.c_uint8))
        o.orc_bam_sizes(p, C.byref(ld), C.byref(lq))
        core = BamCore()
        data = (C.c_uint8 * max(1, ld.value))(); seq = (C.c_uint8 * max(1, lq.value))(); qual = (C.c_uint8 * max(1, lq.value))()
        st = o.orc_bam_unpack1(p, C.byref(core), data, seq, qual)
        res.append((st, core.astuple(), bytes(data[: ld.value]), bytes(seq[: lq.value]), bytes(qual[: lq.value])))
    return res, [offs[i] for i in range(n)]


def orc_rans_4x8_decode(data, cap):
    o = orc()
    out = (C.c_uint8 * max(1, cap))()
    n = C.c_uint32(cap)
    rc = o.orc_rans_4x8_decode(buf(data), C.c_uint32(len(data)), out, C.byref(n))
    return None if rc else bytes(out[: n.value])


@stored_reference(digest=lambda kw: "comp" in kw)
def ref_rans_4x8(data=None, order=None, comp=None):
    """reference rans_compress / rans_uncompress (rANS_static.c:829-850)."""
    r = ref()
    r.rans_compress.restype = C.c_void_p; r.rans_uncompress.restype = C.c_void_p
    libc = C.CDLL(None); libc.free.argtypes = [C.c_void_p]
    n = C.c_uint(0)
    if comp is None:
        p = r.rans_compress(buf(data), C.c_uint(len(data)), C.byref(n), C.c_int(order))
    else:
        p = r.rans_uncompress(buf(comp), C.c_uint(len(comp)), C.byref(n))
    if not p:
        return None
    res = C.string_at(p, n.value)
    libc.free(p)
    return res


@stored_reference(digest=lambda kw: "comp" in kw)
def ref_arith(data=None, order=None, comp=None, cap=None):
    """reference arith_compress_to / arith_uncompress_to (arith_dynamic.c:730, :1033)."""
    r = ref()
    r.arith_compress_to.restype = C.c_void_p; r.arith_uncompress_to.restype = C.c_void_p
    r.arith_compress_bound.restype = C.c_uint
    if comp is None:
        capc = r.arith_compress_bound(C.c_uint(len(data)), C.c_int(order))
        out = (C.c_uint8 * max(1, capc))(); n = C.c_uint(capc)
        p = r.arith_compress_to(buf(data), C.c_uint(len(data)), out, C.byref(n), C.c_int(order))
        assert p
        return bytes(out[: n.value])
    out = (C.c_uint8 * max(1, cap))(); n = C.c_uint(cap)
    p = r.arith_uncompress_to(buf(comp), C.c_uint(len(comp)), out, C.byref(n))
    return bytes(out[: n.value]) if p else None


@stored_reference(limit=40000)
def ref_tok3_encode(names, level=3, use_arith=0):
    """reference tok3_encode_names (tokenise_name3.c:1456): names is the NUL- or LF-separated blob."""
    r = ref()
    r.tok3_encode_names.restype = C.c_void_p
    n = C.c_int(0); last = C.c_int(0)
    src = C.create_string_buffer(bytes(names), len(names) + 1)
    p = r.tok3_encode_names(src, C.c_int(len(names)), C.c_int(level), C.c_int(use_arith), C.byref(n), C.byref(last))
    assert p, "reference tok3 encoder failed"
    res = C.string_at(p, n.value)
    C.CDLL(None).free(C.c_void_p(p))
    return res


@stored_reference(digest=True)
def ref_tok3_decode(comp):
    r = ref()
    r.tok3_decode_names.restype = C.c_void_p
    n = C.c_uint(0)
    p = r.tok3_decode_names(buf(comp), C.c_uint(len(comp)), C.byref(n))
    if not p:
        return None
    res = C.string_at(p, n.value)
    C.CDLL(None).free(C.c_void_p(p))
    return res


@C.CFUNCTYPE(C.c_void_p, C.c_void_p, C.c_uint, C.c_void_p, C.POINTER(C.c_uint))
def _orc_arith_uncompress_to(inp, in_size, out, out_size):
    """arith_uncompress_to's contract (out, or NULL on error) over the oracle's own decoder."""
    return out if orc().orc_arith_decode(C.c_void_p(inp), C.c_uint32(in_size), C.c_void_p(out), out_size) == 0 else None


def orc_tok3_decode(comp):
    """oracle tok3 decode; the adaptive arithmetic sub-coder is the oracle's (orc_arith_decode)."""
    o = orc()
    o.orc_tok3_decode.restype = C.c_void_p
    fn = C.cast(_orc_arith_uncompress_to, C.c_void_p)
    n = C.c_uint32(0)
    p = o.orc_tok3_decode(buf(comp), C.c_uint32(len(comp)), C.byref(n), fn)
    if not p:
        return None
    res = C.string_at(p, n.value)
    o.orc_free(C.c_void_p(p))
    return res


class FqzSlice(C.Structure):      # fqz_slice, htscodecs/htscodecs/fqzcomp_qual.h:59-63
    _fields_ = [("num_records", C.c_int), ("len", C.POINTER(C.c_uint32)), ("flags", C.POINTER(C.c_uint32))]


@stored_reference
def ref_fqz_compress(quals, lens, flags=None, strat=0, vers=4):
    """reference fqz_compress (fqzcomp_qual.c:1615): quals = concatenated quality bytes, lens = record lengths."""
    r = ref()
    r.fqz_compress.restype = C.c_void_p
    n = len(lens)
    la = (C.c_uint32 * n)(*lens); fa = (C.c_uint32 * n)(*(flags or [0] * n))
    sl = FqzSlice(n, la, fa)
    src = C.create_string_buffer(bytes(quals), len(quals) + 1)
    m = C.c_size_t(0)
    p = r.fqz_compress(C.c_int(vers), C.byref(sl), src, C.c_size_t(len(quals)), C.byref(m), C.c_int(strat), None)
    assert p, "reference fqz_compress failed"
    res = C.string_at(p, m.value)
    C.CDLL(None).free(C.c_void_p(p))
    return res


@stored_reference(digest=True)
def ref_fqz_decompress(comp):
    r = ref()
    r.fqz_decompress.restype = C.c_void_p
    m = C.c_size_t(0)
    p = r.fqz_decompress(buf(comp), C.c_size_t(len(comp)), C.byref(m), None, C.c_int(0))
    if not p:
        return None
    res = C.string_at(p, m.value)
    C.CDLL(None).free(C.c_void_p(p))
    return res


def orc_fqz_decode(comp):
    """oracle fqzcomp decode (oracle/orc_fqz.c)."""
    o = orc()
    o.orc_fqz_decode.restype = C.c_void_p
    o.orc_fqz_decode.argtypes = [C.c_void_p, C.c_size_t, C.POINTER(C.c_size_t)]
    m = C.c_size_t(0)
    b = buf(comp)
    p = o.orc_fqz_decode(C.cast(b, C.c_void_p), len(comp), C.byref(m))
    if not p:
        return None
    res = C.string_at(p, m.value)
    o.orc_free(C.c_void_p(p))
    return res


def orc_arith_decode(comp, cap):
    """oracle adaptive-arithmetic decode (oracle/orc_arith.c); cap as arith_uncompress_to's *out_size."""
    o = orc()
    out = (C.c_uint8 * max(1, cap))()
    n = C.c_uint32(cap)
    rc = o.orc_arith_decode(buf(comp), C.c_uint32(len(comp)), out, C.byref(n))
    return None if rc != 0 else bytes(out[: n.value])


@stored_reference(digest=True, limit=200000)
def ref_cram_read_all(path, fasta=None, decode_md=0):
    """Every record of a CRAM file through the compiled reference: hts_open + sam_hdr_read + sam_read1 (-> cram_get_bam_seq).
    Returns list of (core tuple, data bytes)."""
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
    fp = r.hts_open(path.encode(), b"r")
    assert fp, path
    if fasta:
        r.hts_set_fai_filename.argtypes = [C.c_void_p, C.c_char_p]
        assert r.hts_set_fai_filename(fp, fasta.encode()) == 0
    r.hts_set_opt.argtypes = [C.c_void_p, C.c_int, C.c_int]
    r.hts_set_opt(fp, 0, int(decode_md))                       # CRAM_OPT_DECODE_MD, hts.h:297
    hdr = r.sam_hdr_read(fp)
    assert hdr
    b = r.bam_init1()
    out = []
    while True:
        rc = r.sam_read1(fp, hdr, b)
        if rc < 0:
            assert rc == -1, rc
            break
        out.append((b.contents.core.astuple(), bytes(b.contents.data[: b.contents.l_data])))
    r.bam_destroy1(b)
    r.sam_hdr_destroy(hdr)
    r.hts_close(fp)
    return out


def ref_write_cram(sam_path, fasta, out_path, version="3.0", int_opts=()):
    """SAM -> CRAM through the compiled reference (hts_open "wc", sam_write1).  int_opts: (hts_fmt_option, int) pairs."""
    n, img = _ref_write_cram(sam_path, fasta, version, [list(o) for o in int_opts])
    with open(out_path, "wb") as f:
        f.write(img)
    return n


@stored_reference(limit=100000)
def _ref_write_cram(sam_path, fasta, version, int_opts):
    """(records written, file image) of ref_write_cram."""
    import tempfile
    with tempfile.TemporaryDirectory() as td:
        out_path = os.path.join(td, "out.cram")
        n = _ref_write_cram_to(sam_path, fasta, out_path, version, int_opts)
        with open(out_path, "rb") as f:
            return n, f.read()


def _ref_write_cram_to(sam_path, fasta, out_path, version, int_opts):
    r = ref()
    r.hts_open.restype = C.c_void_p
    r.hts_open.argtypes = [C.c_char_p, C.c_char_p]
    r.hts_close.argtypes = [C.c_void_p]
    r.sam_hdr_read.restype = C.c_void_p
    r.sam_hdr_read.argtypes = [C.c_void_p]
    r.sam_hdr_write.argtypes = [C.c_void_p, C.c_void_p]
    r.sam_hdr_destroy.argtypes = [C.c_void_p]
    r.sam_read1.argtypes = [C.c_void_p, C.c_void_p, C.POINTER(Bam1)]
    r.sam_write1.argtypes = [C.c_void_p, C.c_void_p, C.POINTER(Bam1)]
    r.bam_init1.restype = C.POINTER(Bam1)
    r.bam_destroy1.argtypes = [C.POINTER(Bam1)]
    fo = r.hts_open(out_path.encode(), b"wc")
    assert fo
    r.hts_set_opt.argtypes = [C.c_void_p, C.c_int, C.c_char_p]
    assert r.hts_set_opt(fo, 6, version.encode()) == 0                 # CRAM_OPT_VERSION
    if fasta:
        assert r.hts_set_opt(fo, 9, fasta.encode()) == 0               # CRAM_OPT_REFERENCE
    r.hts_set_opt.argtypes = [C.c_void_p, C.c_int, C.c_int]
    for opt, val in int_opts:
        assert r.hts_set_opt(fo, opt, val) == 0
    fi = r.hts_open(sam_path.encode(), b"r")
    assert fi
    h = r.sam_hdr_read(fi)
    assert h and r.sam_hdr_write(fo, h) == 0
    b = r.bam_init1()
    n = 0
    while r.sam_read1(fi, h, b) >= 0:
        assert r.sam_write1(fo, h, b) >= 0
        n += 1
    r.bam_destroy1(b)
    r.hts_close(fi)
    assert r.hts_close(fo) == 0
    r.sam_hdr_destroy(h)
    return n


@stored_reference(digest=True, limit=200000)
def ref_cram_sam_text(path, fasta=None, decode_md=0):
    """SAM text of a CRAM file through the compiled reference: sam_read1 + sam_format1.  Returns (target names, [line bytes])."""
    r = ref()
    r.hts_open.restype = C.c_void_p
    r.hts_open.argtypes = [C.c_char_p, C.c_char_p]
    r.hts_close.argtypes = [C.c_void_p]
    r.sam_hdr_read.restype = C.c_void_p
    r.sam_hdr_read.argtypes = [C.c_void_p]
    r.sam_hdr_destroy.argtypes = [C.c_void_p]
    r.sam_hdr_nref.argtypes = [C.c_void_p]
    r.sam_hdr_tid2name.restype = C.c_char_p
    r.sam_hdr_tid2name.argtypes = [C.c_void_p, C.c_int]
    r.sam_read1.argtypes = [C.c_void_p, C.c_void_p, C.POINTER(Bam1)]
    r.sam_format1.argtypes = [C.c_void_p, C.POINTER(Bam1), C.POINTER(KString)]
    r.bam_init1.restype = C.POINTER(Bam1)
    r.bam_destroy1.argtypes = [C.POINTER(Bam1)]
    fp = r.hts_open(path.encode(), b"r")
    assert fp
    if fasta:
        r.hts_set_fai_filename.argtypes = [C.c_void_p, C.c_char_p]
        assert r.hts_set_fai_filename(fp, fasta.encode()) == 0
    r.hts_set_opt.argtypes = [C.c_void_p, C.c_int, C.c_int]
    r.hts_set_opt(fp, 0, int(decode_md))
    hdr = r.sam_hdr_read(fp)
    assert hdr
    names = [r.sam_hdr_tid2name(hdr, i) for i in range(r.sam_hdr_nref(hdr))]
    b = r.bam_init1()
    ks = KString(0, 0, None)
    lines = []
    while r.sam_read1(fp, hdr, b) >= 0:
        n = r.sam_format1(hdr, b, C.byref(ks))
        lines.append(C.string_at(ks.s, ks.l) if n >= 0 else None)
    libc = C.CDLL(None)
    libc.free.argtypes = [C.c_void_p]
    if ks.s:
        libc.free(ks.s)
    r.bam_destroy1(b)
    r.sam_hdr_destroy(hdr)
    r.hts_close(fp)
    return names, lines


@stored_reference(limit=20000)
def ref_read_sam_records(path):
    """(header text, [(core tuple, data bytes)]) of a SAM / BAM / CRAM file through the compiled reference (sam_hdr_read, sam_read1)."""
    r = ref()
    r.hts_open.restype = C.c_void_p
    r.hts_open.argtypes = [C.c_char_p, C.c_char_p]
    r.hts_close.argtypes = [C.c_void_p]
    r.sam_hdr_read.restype = C.c_void_p
    r.sam_hdr_read.argtypes = [C.c_void_p]
    r.sam_hdr_destroy.argtypes = [C.c_void_p]
    r.sam_hdr_str.restype = C.c_char_p
    r.sam_hdr_str.argtypes = [C.c_void_p]
    r.sam_read1.argtypes = [C.c_void_p, C.c_void_p, C.POINTER(Bam1)]
    r.bam_init1.restype = C.POINTER(Bam1)
    r.bam_destroy1.argtypes = [C.POINTER(Bam1)]
    fp = r.hts_open(path.encode(), b"r")
    assert fp, path
    hdr = r.sam_hdr_read(fp)
    assert hdr
    text = r.sam_hdr_str(hdr) or b""
    b = r.bam_init1()
    out = []
    while True:
        rc = r.sam_read1(fp, hdr, b)
        if rc < 0:
            assert rc == -1, rc
            break
        out.append((b.contents.core.astuple(), bytes(b.contents.data[: b.contents.l_data])))
    r.bam_destroy1(b)
    r.sam_hdr_destroy(hdr)
    r.hts_close(fp)
    return bytes(text), out
