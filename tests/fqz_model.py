"""Plain fqzcomp writer (CRAM 3.1 block method 7), no GPU.

The decoders (fqz_decode_kernel in htslib_b200/csrc/fqzcomp.cu, oracle/orc_fqz.c) are checked against streams this
module writes with every field chosen by the caller, so the parts of the format the reference encoder never uses
(several parameter blocks, selector tables, quality tables, 256-symbol alphabets, long records) get exercised too.

- var_put_u32, store_array: the stream's integer and table codings; `raw` replaces any field or table by chosen bytes.
- RangeCoder: RC_Encode / RC_ShiftLowCheck / RC_FinishEncode (c_range_coder.h:51-145).
- SimpleModel: SIMPLE_MODEL(NSYM) in the reference's own layout, all NSYM slots (c_simple_model.h:77-138).
- update_ctx: fqz_update_ctx (fqzcomp_qual.c:344-386).
- store_params / parse_params: fqz_store_parameters(1) (:674-731) / fqz_read_parameters(1) (:1241-1378).
- encode: a stream in the decoder's own terms (uncompress_block_fqz2f :1456-1613, decompress_new_read :1381-1452),
  with the intended output and a trace of the edges the stream reached.
- device_params: the parameter rules of hgpu_fqz_encode_batch_host (htslib_b200/csrc/fqzcomp_enc.cu) restated.

Citations without a file name are to htscodecs/htscodecs/fqzcomp_qual.c."""
import collections
import math

FQZ_VERS = 5
GFLAG_MULTI_PARAM, GFLAG_HAVE_STAB, GFLAG_DO_REV = 1, 2, 4                       # fqzcomp_qual.h:68-70
PFLAG_DO_DEDUP, PFLAG_DO_LEN, PFLAG_DO_SEL, PFLAG_HAVE_QMAP = 2, 4, 8, 16        # fqzcomp_qual.h:72-79
PFLAG_HAVE_PTAB, PFLAG_HAVE_DTAB, PFLAG_HAVE_QTAB = 32, 64, 128
TOP = 1 << 24                                                                    # c_range_coder.h:21-22
THRES = 255 * TOP
MAX_FREQ = (1 << 16) - 17                                                        # c_simple_model.h:63-66
STEP = 16
CTX_SIZE = 1 << 16                                                               # :73-74
M32 = 0xffffffff


# ---------------------------------------------------------------- integer and table codings
def var_put_u32(v):
    """var_put_u32 (varint.h:206): 7-bit groups, most significant first, bit 7 = more follow."""
    out = bytearray()
    for sh in (28, 21, 14, 7):
        if v >= 1 << sh:
            out.append(((v >> sh) & 0x7f) | 0x80)
    out.append(v & 0x7f)
    return bytes(out)


def var_get_u32(b):
    """(value, bytes used) of a well-formed varint."""
    v = i = 0
    while True:
        c = b[i]
        i += 1
        v = (v << 7) | (c & 0x7f)
        if not c & 0x80:
            return v, i


def store_array(array):
    """store_array (:102-144): the length of the run of each value 0, 1, 2, ... (255s continue a run), then a second
    run-length pass over those bytes: a byte equal to the one before it is followed by the count of further copies.
    read_array gives back run indices, so only non-decreasing arrays can be stored."""
    assert all(b >= a for a, b in zip(array, array[1:])), "store_array holds non-decreasing arrays only"
    tmp = []
    i = j = 0
    size = len(array)
    while i < size:
        start = i
        while i < size and array[i] == j:
            i += 1
        run = i - start
        while True:
            r = min(255, run)
            tmp.append(r)
            run -= r
            if r != 255:
                break
        j += 1
    out = bytearray()
    last = -1
    k = 0
    while k < len(tmp):
        out.append(tmp[k])
        k += 1
        if out[-1] == last:
            n = k
            while k < len(tmp) and tmp[k] == last:
                k += 1
            out.append(k - n)
        else:
            last = out[-1]
    return bytes(out)


def read_array(b, size):
    """read_array (:146-190): (array, bytes used), or None where the reference returns -1."""
    size = min(1024, size)
    R = []
    i = z = 0
    last = -1
    while z < size and i < len(b):
        run = b[i]
        R.append(run)
        z += run
        if run == last:
            if i + 1 >= len(b):
                return None
            i += 1
            copy = b[i]
            z += run * copy
            while copy and z <= size and len(R) < 1024:
                copy -= 1
                R.append(run)
        if len(R) >= 1024:
            return None
        last = run
        i += 1
    nb = i
    arr = []
    z = 0
    v = 0
    while len(arr) < size:
        if z >= len(R):
            return None
        run = 0
        while True:
            part = R[z]
            z += 1
            run += part
            if not (part == 255 and z < len(R)):
                break
        if part == 255:
            return None
        take = min(run, size - len(arr))
        arr += [v] * take
        v += 1
    return arr, nb


# ---------------------------------------------------------------- range coder and adaptive model
class Trace:
    """The edges one stream reached while it was written."""

    def __init__(self):
        self.carries = 0          # RC_Encode's low wrapped (Carry += 1)
        self.max_ffnum = 0        # longest run of 0xff bytes held back (FFNum)
        self.carry_over_ff = 0    # a carry that turned a held-back run of 3 or more 0xff bytes into 0x00
        self.normalises = 0       # SIMPLE_MODEL_normalize calls
        self.tot_at_max = 0       # totals that reached MAX_FREQ exactly, which must not normalise ("> MAX_FREQ")
        self.swaps = 0            # "keep approx sorted" swaps
        self.swaps_to_front = 0   # ... of which into slot 0
        self.max_ctx_uses = 0     # most symbols coded in one quality context
        self.p_clamped = 0        # qualities coded at a position p > 1023 (ptab[MIN(1023, p)])
        self.delta_clamped = 0    # ... with delta > 255 (dtab[MIN(255, delta)])
        self.ctx_over_16 = 0      # context sums >= 2^16 before the mask
        self.max_sym = -1         # largest quality symbol coded
        self.max_sel = -1         # largest selector coded
        self.blocks_used = set()  # parameter blocks records selected
        self.records = 0
        self.dups = 0


class RangeCoder:
    """RC_StartEncode / RC_Encode / RC_ShiftLowCheck / RC_FinishEncode (c_range_coder.h:51-145)."""

    def __init__(self, trace):
        self.low, self.range, self.ffnum, self.carry, self.cache = 0, M32, 0, 0, 0
        self.out = bytearray()
        self.t = trace

    def shift_low(self):
        if self.low < THRES or self.carry:
            if self.carry and self.ffnum >= 3:
                self.t.carry_over_ff += 1
            self.out.append((self.cache + self.carry) & 0xff)
            self.out += bytes([(self.carry - 1) & 0xff]) * self.ffnum
            self.ffnum = 0
            self.cache = self.low >> 24
            self.carry = 0
        else:
            self.ffnum += 1
            self.t.max_ffnum = max(self.t.max_ffnum, self.ffnum)
        self.low = (self.low << 8) & M32

    def encode(self, cum, freq, tot):
        tmp = self.low
        self.range //= tot
        self.low = (self.low + cum * self.range) & M32
        self.range = (self.range * freq) & M32
        if self.low < tmp:
            self.carry += 1
            self.t.carries += 1
        while self.range < TOP:
            self.range = (self.range << 8) & M32
            self.shift_low()

    def finish(self):
        for _ in range(5):
            self.shift_low()
        return bytes(self.out)


class SimpleModel:
    """SIMPLE_MODEL(NSYM) (c_simple_model.h:77-138): F[NSYM+1] (Freq, Symbol) approximately sorted by Freq behind a
    MAX_FREQ sentinel; symbols max_sym.. keep frequency 0 and F[NSYM] ends the normalise loop."""

    def __init__(self, nsym_max, max_sym, trace):
        self.F = [1] * max_sym + [0] * (nsym_max + 1 - max_sym)
        self.S = list(range(nsym_max)) + [0]
        self.tot = max_sym
        self.uses = 0
        self.t = trace

    def encode(self, rc, sym):
        i = 0
        acc = 0
        while self.S[i] != sym:
            acc += self.F[i]
            i += 1
        assert self.F[i] > 0, "symbol %d is outside the model's alphabet" % sym
        rc.encode(acc, self.F[i], self.tot)
        self.F[i] += STEP
        self.tot += STEP
        self.t.tot_at_max += self.tot == MAX_FREQ
        if self.tot > MAX_FREQ:                                  # SIMPLE_MODEL_normalize :106-115
            self.t.normalises += 1
            self.tot = 0
            k = 0
            while self.F[k]:
                self.F[k] -= self.F[k] >> 1
                self.tot += self.F[k]
                k += 1
        prev = self.F[i - 1] if i else MAX_FREQ                   # s[-1] of F[0] is the sentinel
        if self.F[i] > prev:
            self.F[i], self.F[i - 1] = self.F[i - 1], self.F[i]
            self.S[i], self.S[i - 1] = self.S[i - 1], self.S[i]
            self.t.swaps += 1
            self.t.swaps_to_front += i == 1
        self.uses += 1
        self.t.max_ctx_uses = max(self.t.max_ctx_uses, self.uses)


# ---------------------------------------------------------------- parameters
def block(**kw):
    """One parameter block (fqz_param as stored).  Every field has a plain default: no flags, max_sym 0, no tables."""
    b = dict(context=0, pflags=0, max_sym=0, qbits=0, qshift=0, qloc=0, sloc=0, ploc=0, dloc=0,
             qmap=None, qtab=None, ptab=None, dtab=None)
    unknown = set(kw) - set(b)
    assert not unknown, unknown
    b.update(kw)
    return b


def gparams(blocks, gflags=None, nparam=None, max_sel=None, stab=None, ulen=None, raw=None, vers=FQZ_VERS):
    """The global parameters (fqz_gparams).  gflags defaults to what the other arguments need; nparam to the number
    of blocks; max_sel to the reader's default.  ulen overrides the size field.  raw maps a field name ("vers",
    "gflags", "nparam", "max_sel", "stab") or (block index, field name) to the bytes written in its place, and
    "tail" to bytes appended after the coded data."""
    if gflags is None:
        gflags = (GFLAG_MULTI_PARAM if len(blocks) > 1 else 0) | (GFLAG_HAVE_STAB if stab is not None else 0)
    return dict(vers=vers, gflags=gflags, nparam=len(blocks) if nparam is None else nparam, max_sel=max_sel,
                stab=stab, blocks=blocks, ulen=ulen, raw=raw or {})


def resolved(gp):
    """(nparam, max_sel, stab[256]) as the reader derives them (:1336-1352)."""
    nparam = gp["nparam"]
    if gp["gflags"] & GFLAG_HAVE_STAB:
        return nparam, gp["max_sel"], list(gp["stab"])
    max_sel = nparam if nparam > 1 else 0
    return nparam, max_sel, [i if i < nparam else nparam - 1 for i in range(256)]


def store_block(pm, raw, b):
    """fqz_store_parameters1 (:674-708), every field as given.  The quality table is written where the reader reads
    it, qbits != 0 and PFLAG_HAVE_QTAB (:1284-1294)."""
    def f(name, data):
        return raw.get((b, name), data)
    fl = pm["pflags"]
    out = bytearray()
    out += f("context", bytes([pm["context"] & 0xff, pm["context"] >> 8]))
    out += f("pflags", bytes([fl]))
    out += f("max_sym", bytes([pm["max_sym"]]))
    out += f("qbits", bytes([pm["qbits"] << 4 | pm["qshift"]]))
    out += f("qloc", bytes([pm["qloc"] << 4 | pm["sloc"]]))
    out += f("ploc", bytes([pm["ploc"] << 4 | pm["dloc"]]))
    if fl & PFLAG_HAVE_QMAP:
        out += f("qmap", bytes(pm["qmap"]))
    if pm["qbits"] and fl & PFLAG_HAVE_QTAB:
        out += f("qtab", store_array(pm["qtab"]))
    if fl & PFLAG_HAVE_PTAB:
        out += f("ptab", store_array(pm["ptab"]))
    if fl & PFLAG_HAVE_DTAB:
        out += f("dtab", store_array(pm["dtab"]))
    return bytes(out)


def store_params(gp):
    """fqz_store_parameters (:710-731)."""
    raw = gp["raw"]
    out = bytearray()
    out += raw.get("vers", bytes([gp["vers"]]))
    out += raw.get("gflags", bytes([gp["gflags"]]))
    if gp["gflags"] & GFLAG_MULTI_PARAM:
        out += raw.get("nparam", bytes([gp["nparam"]]))
    if gp["gflags"] & GFLAG_HAVE_STAB:
        out += raw.get("max_sel", bytes([gp["max_sel"]]))
        out += raw.get("stab", store_array(gp["stab"]))
    for b, pm in enumerate(gp["blocks"]):
        out += store_block(pm, raw, b)
    return bytes(out)


def parse_params(stream):
    """fqz_read_parameters (:1319-1378) on a well-formed stream: (gparams, header length including the size varint)."""
    ulen, k = var_get_u32(stream)
    q = stream[k:]
    j = 2
    vers, gflags = q[0], q[1]
    nparam = 1
    if gflags & GFLAG_MULTI_PARAM:
        nparam = q[j]
        j += 1
    max_sel = stab = None
    if gflags & GFLAG_HAVE_STAB:
        max_sel = q[j]
        stab, used = read_array(q[j + 1:], 256)
        j += 1 + used
    blocks = []
    for _ in range(nparam):
        c = q[j:j + 7]
        fl = c[2]
        pm = block(context=c[0] | c[1] << 8, pflags=fl, max_sym=c[3], qbits=c[4] >> 4, qshift=c[4] & 15,
                   qloc=c[5] >> 4, sloc=c[5] & 15, ploc=c[6] >> 4, dloc=c[6] & 15)
        j += 7
        if fl & PFLAG_HAVE_QMAP:
            pm["qmap"] = list(q[j:j + pm["max_sym"]])
            j += pm["max_sym"]
        for name, flag, size, cond in (("qtab", PFLAG_HAVE_QTAB, 256, pm["qbits"]), ("ptab", PFLAG_HAVE_PTAB, 1024, 1),
                                       ("dtab", PFLAG_HAVE_DTAB, 256, 1)):
            if fl & flag and cond:
                pm[name], used = read_array(q[j:], size)
                j += used
        blocks.append(pm)
    gp = gparams(blocks, gflags=gflags, nparam=nparam, max_sel=max_sel, stab=stab, ulen=ulen, vers=vers)
    return gp, k + j


class Ctx:
    """Block 0's context fields in the form the record loop uses them (the tables shifted as at :1489-1496)."""

    def __init__(self, pm):
        fl = pm["pflags"]
        self.qshift, self.qloc, self.sloc = pm["qshift"], pm["qloc"], pm["sloc"]
        self.qmask = (1 << pm["qbits"]) - 1
        self.qtab = list(pm["qtab"]) if (pm["qbits"] and fl & PFLAG_HAVE_QTAB) else list(range(256))
        self.ptab = [v << pm["ploc"] for v in pm["ptab"]] if fl & PFLAG_HAVE_PTAB else [0] * 1024
        self.dtab = [v << pm["dloc"] for v in pm["dtab"]] if fl & PFLAG_HAVE_DTAB else [0] * 256
        if fl & PFLAG_HAVE_QMAP:                                   # entries past max_sym are INT_MAX: 0xff as a byte
            self.qmap = list(pm["qmap"][:pm["max_sym"]]) + [0xff] * (256 - pm["max_sym"])
        else:
            self.qmap = list(range(256))


def update_ctx(c, st, q, t):
    """fqz_update_ctx (:344-386) with block 0's fields; st = [qctx, p, delta, prevq, sel]."""
    qctx, p, delta, prevq, sel = st
    qctx = ((qctx << c.qshift) + c.qtab[q]) & M32
    last = (qctx & c.qmask) << c.qloc
    t.p_clamped += p > 1023
    t.delta_clamped += delta > 255
    last += c.ptab[min(1023, p)]
    last += c.dtab[min(255, delta)]
    last += sel << c.sloc
    t.ctx_over_16 += last >= CTX_SIZE
    delta += prevq != q
    st[:] = [qctx, p - 1, delta, q, sel]
    return last & (CTX_SIZE - 1)


# ---------------------------------------------------------------- streams
def record(length, sel=0, rev=0, dup=0):
    return dict(length=length, sel=sel, rev=rev, dup=dup)


def encode(symbols, records, gp):
    """The stream the decoder reads as `records` of `symbols`, and what it must return.

    symbols: the quality model symbols of the records that are not duplicates, in stored orientation, concatenated.
    records: record(length, sel, rev, dup) each.  Selectors are coded where block 0 has PFLAG_DO_SEL (:1394); the
    length where the selected block has no PFLAG_DO_LEN or on the first record (:1408); the reverse flag under
    GFLAG_DO_REV; the duplicate flag where the selected block has PFLAG_DO_DEDUP (:1428).  Qualities are coded with
    the selected block's starting context but block 0's context fields and quality map (the record loop keeps
    pm = &gp.p[0], :1532-1560).

    Returns (stream, intended output or None where the decoder must refuse the stream, Trace)."""
    t = Trace()
    nparam, max_sel, stab = resolved(gp)
    blocks = gp["blocks"]
    b0 = blocks[0]
    c = Ctx(b0)
    gmax = max(b["max_sym"] for b in blocks)
    ulen = gp["ulen"] if gp["ulen"] is not None else sum(r["length"] for r in records)
    rc = RangeCoder(t)
    qual = {}
    m_len = [SimpleModel(256, 256, t) for _ in range(4)]
    m_rev, m_dup = SimpleModel(2, 2, t), SimpleModel(2, 2, t)
    m_sel = SimpleModel(256, max_sel + 1, t) if max_sel > 0 else None
    out = bytearray()
    marks = []                                                    # (start, length, rev) of every record
    first_len, last_len = True, 0
    pos = 0
    ok = True
    for r in records:
        sel = 0
        if b0["pflags"] & PFLAG_DO_SEL:
            sel = r["sel"]
            m_sel.encode(rc, sel)
            t.max_sel = max(t.max_sel, sel)
        x = stab[min(255, sel)] if gp["gflags"] & GFLAG_HAVE_STAB else sel
        if x >= nparam:
            ok = False
            break
        pm = blocks[x]
        t.blocks_used.add(x)
        rl = r["length"]
        if not pm["pflags"] & PFLAG_DO_LEN or first_len:
            for k in range(4):
                m_len[k].encode(rc, (rl >> 8 * k) & 0xff)
            first_len, last_len = False, rl
        else:
            assert rl == last_len, "a fixed-length record keeps the last coded length"
        if rl > ulen - len(out) or rl == 0:
            ok = False
            break
        if gp["gflags"] & GFLAG_DO_REV:
            m_rev.encode(rc, r["rev"])
        marks.append((len(out), rl, r["rev"]))
        t.records += 1
        if pm["pflags"] & PFLAG_DO_DEDUP:
            m_dup.encode(rc, r["dup"])
            if r["dup"]:
                t.dups += 1
                if rl > len(out):
                    ok = False
                    break
                out += out[len(out) - rl:]
                continue
        else:
            assert not r["dup"], "a duplicate needs PFLAG_DO_DEDUP in the selected block"
        st = [0, rl, 0, 0, sel]
        last = pm["context"]
        for _ in range(rl):
            q = symbols[pos]
            pos += 1
            m = qual.get(last)
            if m is None:
                m = qual[last] = SimpleModel(256, gmax + 1, t)
            m.encode(rc, q)
            t.max_sym = max(t.max_sym, q)
            last = update_ctx(c, st, q, t)
            out.append(c.qmap[q])
        if len(out) == ulen:
            break
    if ok:
        assert pos == len(symbols), "symbols left over"
        ok = len(out) == ulen
    if ok and gp["gflags"] & GFLAG_DO_REV:
        for a, n, rv in marks:
            if rv:
                out[a:a + n] = out[a:a + n][::-1]
    stream = var_put_u32(ulen) if "ulen" not in gp["raw"] else gp["raw"]["ulen"]
    stream += store_params(gp) + rc.finish() + gp["raw"].get("tail", b"")
    return stream, (bytes(out) if ok else None), t


def dup_flags(quals, lens, do_dedup):
    """Which records the encoders code as duplicates (compress_new_read :982-996): equal in length and bytes to the
    bytes just before them, the last non-duplicate record's length."""
    flags, pos, last_len = [], 0, 0
    for n in lens:
        d = bool(do_dedup and pos and n == last_len and quals[pos - last_len:pos] == quals[pos:pos + n])
        flags.append(d)
        if do_dedup and not d:
            last_len = n
        pos += n
    return flags


# ---------------------------------------------------------------- the device encoder's parameter choice
STRAT_OPTS = [                                                    # strat_opts :195-201 (qb qs pb ps db ds ql sl pl dl r2 qa)
    (10, 5, 4, -1, 2, 1, 0, 14, 10, 14, 0, -1),
    (8, 5, 7, 0, 0, 0, 0, 14, 8, 14, 1, -1),
    (12, 6, 2, 0, 2, 3, 0, 9, 12, 14, 0, 0),
    (12, 6, 0, 0, 0, 0, 0, 12, 0, 0, 0, 0),
]
DSQR = [0, 1, 1, 1, 2, 2, 2, 2, 2, 3, 3, 3, 3, 3, 3, 3, 4, 4, 4, 4, 4, 4, 4, 4, 4, 5, 5, 5, 5, 5, 5, 5,
        5, 5, 5, 5, 6, 6, 6, 6, 6, 6, 6, 6, 6, 6, 6, 6, 6, 7, 7, 7, 7, 7, 7, 7, 7, 7, 7, 7, 7, 7, 7, 7]


def device_params(quals, lens, strat):
    """fqz_pick_parameters (:736-924) as hgpu_fqz_encode_batch_host applies it, without the selector search: one block,
    gflags 0.  Returns (size varint + parameter block as the device writes it, gparams, facts) where facts names the
    rules that fired."""
    strat = max(0, min(3, strat))
    size = len(quals)
    counts = collections.Counter(quals)
    hist = [counts.get(i, 0) for i in range(256)]
    nsym = sum(1 for h in hist if h)
    max_sym = max(i for i in range(256) if hist[i])
    dups, pos = 0, 0                                              # fqz_qual_stats :432-469
    for r, n in enumerate(lens):
        if r and n == lens[r - 1] and quals[pos - lens[r - 1]:pos] == quals[pos:pos + n]:
            dups += 1
        pos += n
    do_dedup = (len(lens) + 1) // (dups + 1) < 500
    fixed_len = all(n == lens[0] for n in lens)
    qb, qs, pb, ps, db, ds, ql, sl, pl, dl, r2, qa = STRAT_OPTS[strat]
    if qa == -1:                                                  # :601-622, whether or not a selector is kept
        if pb > 0 and db > 0:
            sl, pb, db, dl = dl - 1, pb - 1, db - 1, dl + 1
        elif db >= 2:
            sl, db, dl = dl, db - 2, dl + 2
        elif qb >= 2:
            qb, pl, sl = qb - 2, pl - 2, 16 - 2 - r2
            if qb == 6 and qs == 5:
                qb -= 1
    store_qmap = nsym <= 8 and nsym * 2 < max_sym                  # :800
    if ps < 0:                                                    # :814-815
        ps = max(0, int(math.log(lens[0] / (1 << pb)) / math.log(2) + .5))
    if nsym <= 4:                                                 # :817-830
        qs = 2
        if size < 5000000:
            pb, ps = 2, 5
    elif nsym <= 8:
        qb, qs = min(qb, 9), 3
        if size < 5000000:
            qb = 6
    if size < 300000:                                             # :832-835
        qb, db = qs, 2
    dsqr = [min(v, (1 << db) - 1) for v in DSQR]
    ptab = [min((1 << pb) - 1, i >> ps) for i in range(1024)] if pb else None
    dtab = [dsqr[min(63, i >> ds)] for i in range(256)] if db else None
    qmap = [i for i in range(256) if hist[i]] if store_qmap else None
    pflags = ((PFLAG_HAVE_DTAB if db else 0) | (PFLAG_HAVE_PTAB if pb else 0) | (PFLAG_DO_LEN if fixed_len else 0) |
              (PFLAG_DO_DEDUP if do_dedup else 0) | (PFLAG_HAVE_QMAP if store_qmap else 0))
    pm = block(pflags=pflags, max_sym=nsym if store_qmap else max_sym, qbits=qb, qshift=qs, qloc=ql, sloc=sl,
               ploc=pl, dloc=dl, qmap=qmap, ptab=ptab, dtab=dtab)
    gp = gparams([pm], ulen=size)
    facts = dict(nsym=nsym, max_sym=max_sym, store_qmap=store_qmap, fixed_len=fixed_len, do_dedup=do_dedup, dups=dups, pshift=ps,
                 size=size)
    return var_put_u32(size) + store_params(gp), gp, facts


def symbols_of(quals, lens, gp):
    """(symbols, records) that encode() needs to write the device encoder's stream for this block."""
    pm = gp["blocks"][0]
    sym = list(range(256))
    if pm["pflags"] & PFLAG_HAVE_QMAP:
        for j, q in enumerate(pm["qmap"]):
            sym[q] = j
    dup = dup_flags(quals, lens, pm["pflags"] & PFLAG_DO_DEDUP)
    symbols, pos = [], 0
    for n, d in zip(lens, dup):
        if not d:
            symbols += [sym[q] for q in quals[pos:pos + n]]
        pos += n
    return symbols, [record(n, dup=d) for n, d in zip(lens, dup)]
