"""The Huffman half of the inflate kernels, driven by dynamic-Huffman blocks whose code lengths the test picks.

Cases: the worst-case sub-table layouts of both decode tables, 15-bit codes and 48-bit tokens, one- and two-code
tables, header edges (HLIT 286, HDIST 30, HCLEN 4 / 5 / 19, zero runs of 138, repeats across the literal/distance
boundary), block sequences, trailing bytes, an end-of-block code that ends inside the footer, and malformed streams of
every kind zlib names.  The kernel picks its body decoder by the input left after a block header (PAR_MIN_BITS), so
each body-level case comes twice: small (serial decoder) and padded (lane-parallel decoder).  The reference is zlib
itself, called the way bgzf_uncompress calls it."""
import ctypes as C
import random
import struct
import zlib
import numpy as np
import pytest
import htslib_b200 as H
from _libs import orc_bgzf_inflate_block, orc_inflate_trace
from deflate_model import CL_ORDER, build_lengths, canonical_codes, rle_lengths
from test_gpu_bgzf_lz77 import DBASE, DXTRA, LBASE, LXTRA, Deflate, expand, _inflate
from test_gpu_bgzf_inflate_runs import PAR_MIN_BITS

LIT_ROOT, DST_ROOT = 9, 8                  # the kernel's root table bits (zlib's: 9 and 6)
NO_END = "no end of stream"                # zlib stops without an error and without reaching the end of the stream
SLOT = 65536
CRAM_UNSUPPORTED = -6                      # HGPU_CRAM_UNSUPPORTED: the block goes back to the host library


class Writer(Deflate):
    """The raw-DEFLATE writer of test_gpu_bgzf_lz77 and dynamic-Huffman blocks with the code lengths the test picks.
    bodies: the bit position where each Huffman block's body starts (after its header)."""

    def __init__(self):
        super().__init__()
        self.bodies = []

    def stored(self, data, final=False):                    # the same block, its bytes written as one integer
        self.bits(int(final), 1); self.bits(0, 2)
        self.n = (self.n + 7) // 8 * 8
        self.bits(len(data), 16); self.bits(len(data) ^ 0xffff, 16)
        self.bits(int.from_bytes(data, "little"), 8 * len(data))

    def fixed(self, tokens, final=False):
        self.bodies.append(self.n + 3)
        super().fixed(tokens, final)

    def dynamic(self, tokens, ll, dl, final=False, hlit=None, hdist=None, hclen=None, cl=None, seq=None, eob=True):
        """A dynamic-Huffman block: ll for literal/length symbols 0.., dl for distance symbols 0...  The header follows
        from them unless overridden: hlit / hdist / hclen are the raw 5-, 5- and 4-bit fields, cl the 19 code-length-code
        lengths (by symbol), seq the code-length symbols as (symbol, extra value) pairs, 16/17/18 included.  eob=False
        leaves the end-of-block code out."""
        nl = hlit + 257 if hlit is not None else max([257] + [i + 1 for i, l in enumerate(ll) if l])
        nd = hdist + 1 if hdist is not None else max([1] + [i + 1 for i, l in enumerate(dl) if l])
        if seq is None:
            seq = rle_lengths((list(ll) + [0] * nl)[:nl] + (list(dl) + [0] * nd)[:nd])
        if cl is None:
            clf = [0] * 19
            for s, _ in seq:
                clf[s] += 1
            cl = build_lengths(clf, 7)
            if sum(1 for l in cl if l) == 1:                 # a complete code-length code needs two codes
                cl[1 if cl[0] else 0] = 1
        ncl = hclen + 4 if hclen is not None else max([4] + [k + 1 for k in range(4, 19) if cl[CL_ORDER[k]]])
        self.bits(int(final), 1); self.bits(2, 2)
        self.bits(nl - 257, 5); self.bits(nd - 1, 5); self.bits(ncl - 4, 4)
        for k in range(ncl):
            self.bits(cl[CL_ORDER[k]], 3)
        cc = canonical_codes(cl)
        for s, x in seq:
            self.huff(cc[s], cl[s])
            self.bits(x, {16: 2, 17: 3, 18: 7}.get(s, 0))
        self.bodies.append(self.n)
        lc, dc = canonical_codes(list(ll)), canonical_codes(list(dl))
        for t in tokens:
            if isinstance(t, int):
                self.huff(lc[t], ll[t])
            else:
                ln, dist = t
                ls = max(i for i in range(29) if LBASE[i] <= ln)
                self.huff(lc[257 + ls], ll[257 + ls]); self.bits(ln - LBASE[ls], LXTRA[ls])
                ds = max(i for i in range(30) if DBASE[i] <= dist)
                self.huff(dc[ds], dl[ds]); self.bits(dist - DBASE[ds], DXTRA[ds])
        if eob:
            self.huff(lc[256], ll[256])

    def huff(self, c, nb):                                  # a code of a table the test chose (over-subscribed ones too)
        if nb:
            self.code(c & ((1 << nb) - 1), nb)


# ---------------------------------------------------------------- plain references
def zlib_bgzf(raw_with_footer):
    """bgzf_uncompress: raw inflate (wbits -15) of the deflate data and the 8-byte footer behind it, at most 64 KiB of
    output, OK only at the end of the stream.  Returns (status, bytes, zlib's message or NO_END or None)."""
    d = zlib.decompressobj(-15)
    try:
        out = d.decompress(raw_with_footer, SLOT + 1)
    except zlib.error as e:
        return H.BGZF_ERR_ZLIB, b"", str(e).split(": ", 1)[1]
    if not d.eof or len(out) > SLOT:
        return H.BGZF_ERR_ZLIB, out, NO_END
    return 0, out, None


def subtable_slots(lens, root):
    """Sub-table entries a table with `root` root bits allocates for this code laid out canonically: 2^(longest code
    under the prefix - root), summed over the root prefixes of the codes longer than root."""
    deep = {}
    for c, l in zip(canonical_codes(lens), lens):
        if l > root:
            p = c >> (l - root)
            deep[p] = max(deep.get(p, 0), l)
    return sum(1 << (l - root) for l in deep.values())


def worst_case(nsyms, root, maxlen=15):
    """The most sub-table entries a complete code of at most nsyms symbols and maxlen bits can need, and code lengths
    that need them.  g root prefixes lead to sub-tables; the other 2^root - g root slots take at least popcount(2^root - g)
    short codes.  In canonical order each deep prefix holds a complete subtree whose depths run from a to b, a >= the
    previous prefix's b; the fewest leaves for that are 2^a - 1 at depth a, one at each depth a+1..b-1 and two at b
    (2^a + b - a), or 2^a when a == b, and its sub-table has 2^b entries.  Dynamic programming over the prefixes in order,
    state (b of the last prefix, leaves used), maximises the sum of 2^b."""
    D = maxlen - root
    f = [{(1, 0): (0, None)}]                           # f[i][(b, leaves)] = (entries, (previous state, a))
    best = (0, 0, None)
    for g in range(1, (1 << root) + 1):
        nxt = {}
        for (pb, used), (val, _) in f[-1].items():
            for a in range(pb, D + 1):
                for b in range(a, D + 1):
                    u = used + (1 << a) + b - a
                    if u > nsyms:
                        break
                    v = val + (1 << b)
                    if v > nxt.get((b, u), (-1,))[0]:
                        nxt[(b, u)] = (v, ((pb, used), a))
        if not nxt:
            break
        f.append(nxt)
        shallow = bin((1 << root) - g).count("1")
        for (b, u), (v, _) in nxt.items():
            if u + shallow <= nsyms and v > best[0]:
                best = (v, g, (b, u))
    val, g, state = best
    depths = [root - k for k in range(root, -1, -1) if ((1 << root) - g) >> k & 1]     # the short codes
    deep = []
    for i in range(g, 0, -1):
        b = state[0]
        prev, a = f[i][state][1]
        if a == b:
            deep.append([root + a] * (1 << a))
        else:
            deep.append([root + a] * ((1 << a) - 1) + list(range(root + a + 1, root + b)) + [root + b] * 2)
        state = prev
    for sub in reversed(deep):
        depths += sub
    return val, depths


def fill(lens, pool):
    """Complete a code: the symbols of pool, in order, take the code space that lens leaves free, shortest codes first:
    the binary expansion of the free space, its shortest codes split in two until every symbol of pool has one."""
    lens = list(lens)
    free = (1 << 15) - sum(1 << (15 - l) for l in lens if l)
    leaves = sorted(15 - k for k in range(16) if free >> k & 1)
    while leaves[0] == 0 or len(leaves) < len(pool):
        l = leaves.pop(0)
        leaves = sorted(leaves + [l + 1, l + 1])
    assert len(leaves) == len(pool)
    for s, l in zip(pool, leaves):
        assert lens[s] == 0
        lens[s] = l
    return lens


def decoders(d, raw):
    """The body decoder the kernel takes for each Huffman block the writer wrote: lane-parallel when the input after the
    block header, footer included, holds at least PAR_MIN_BITS bits"""
    total = (len(raw) + 8) * 8
    return ["par" if total - b >= PAR_MIN_BITS else "ser" for b in d.bodies]


def footer(data):
    return struct.pack("<II", zlib.crc32(data) & 0xffffffff, len(data) & 0xffffffff)


def repeats(seq):
    """(symbol, first, end) of every 16/17/18 of a code-length sequence, in positions of the lengths it stands for"""
    out, i = [], 0
    for s, x in seq:
        n = {16: 3 + x, 17: 3 + x, 18: 11 + x}.get(s, 1)
        if s >= 16:
            out.append((s, i, i + n))
        i += n
    return out


def match_tokens(rng, lsyms, dsyms, n):
    """n matches that between them use every length symbol of lsyms and every distance symbol of dsyms"""
    out = []
    for i in range(n):
        ls, ds = lsyms[i % len(lsyms)], dsyms[i % len(dsyms)]
        ln = 258 if ls == 285 else LBASE[ls - 257] + rng.randrange(1 << LXTRA[ls - 257])
        if ls == 284:
            ln = min(ln, 257)                               # 258 is symbol 285
        out.append((ln, DBASE[ds] + rng.randrange(1 << DXTRA[ds])))
    return out


def token_bits(toks, ll, dl):
    n = 0
    for t in toks:
        if isinstance(t, int):
            n += ll[t]
        else:
            ls = max(i for i in range(29) if LBASE[i] <= t[0])
            ds = max(i for i in range(30) if DBASE[i] <= t[1])
            n += ll[257 + ls] + LXTRA[ls] + dl[ds] + DXTRA[ds]
    return n


# ---------------------------------------------------------------- the cases
class Case:
    """raw: the deflate data (and any bytes behind it) in front of the 8-byte footer.  dec: the body decoder every
    Huffman block is built for ('ser' / 'par'; None where decoding stops in a header).  want: the output the writer meant
    (valid streams), else None with msg: the zlib message the stream was built to hit, or NO_END."""

    def __init__(self, name, d, raw, foot, dec=None, want=None, msg=None):
        self.name, self.raw, self.foot, self.dec, self.want, self.msg = name, raw, foot, dec, want, msg
        self.decs = decoders(d, raw) if d is not None else []


def both(out, name, build, msg=None):
    """build(npad) -> (writer, raw, expected output): the case as built (small) and with npad grown until every Huffman
    block takes the lane-parallel decoder"""
    d, raw, want = build(0)
    out.append(Case(name + "_ser", d, raw, footer(want) if msg is None else bytes(8), "ser", want if msg is None else None, msg))
    n = 16
    while True:
        d, raw, want = build(n)
        if all(x == "par" for x in decoders(d, raw)):
            break
        n += n // 4 + 16
    out.append(Case(name + "_par", d, raw, footer(want) if msg is None else bytes(8), "par", want if msg is None else None, msg))


def rbytes(rng, n):
    return bytes(rng.randrange(256) for _ in range(n))


def valid_cases():
    rng = random.Random(21)
    out = []
    prefix = rbytes(rng, 33000)                         # every distance up to 32768 can be reached behind it

    # worst-case tables: every symbol with a code used at least once
    _, lw = worst_case(286, LIT_ROOT)
    _, dw = worst_case(30, DST_ROOT)
    lw.sort(); dw.sort()
    ll = [0] * 286
    for s, l in zip([ord("a"), 256] + list(range(257, 286)) + [s for s in range(256) if s != ord("a")], lw):
        ll[s] = l
    dl = [0] * 30
    for s, l in zip(range(30), dw):
        dl[s] = l
    lits = [s for s in range(256) if ll[s]]
    toks = match_tokens(rng, [s for s in range(257, 286) if ll[s]], [s for s in range(30) if dl[s]], 40) + lits
    rng.shuffle(toks)
    chunks, cur = [], []                                # serial: members of fewer than PAR_MIN_BITS body bits
    for t in toks:
        if token_bits(cur + [t], ll, dl) + ll[256] + 64 + 8 >= PAR_MIN_BITS:
            chunks.append(cur); cur = []
        cur.append(t)
    chunks.append(cur)
    for k, ch in enumerate(chunks):
        d = Writer(); d.stored(prefix); d.dynamic(ch, ll, dl, final=True)
        want = expand(ch, prefix)
        out.append(Case("worst_ser%d" % k, d, d.raw(), footer(want), "ser", want))

    def worst(npad):
        t = toks + [ord("a")] * npad
        d = Writer(); d.stored(prefix); d.dynamic(t, ll, dl, final=True)
        return d, d.raw(), expand(t, prefix)
    both(out, "worst", worst)
    out.pop(-2)                                         # worst_ser: the chunks above

    # deep codes: 15-bit literals, length symbols 265..284, distance symbols 26..29
    deep_lits = rng.sample(range(256), 16)
    lens = [0] * 286
    for s in deep_lits + list(range(265, 285)):
        lens[s] = 15
    pad = next(s for s in range(256) if s not in deep_lits)
    ll_deep = fill(lens, [pad, 256, 257, 258, 259] + [s for s in range(256) if s not in deep_lits and s != pad])
    dl_deep = fill([0] * 26 + [15] * 4, list(range(26)))
    deep_toks = deep_lits + match_tokens(rng, list(range(265, 285)), [26, 27, 28, 29], 20)

    def deep(npad):
        t = deep_toks + [pad] * npad
        d = Writer(); d.stored(prefix); d.dynamic(t, ll_deep, dl_deep, final=True)
        return d, d.raw(), expand(t, prefix)
    both(out, "deep_syms", deep)

    def t48(n):                                         # length symbol 284 + 5 bits, distance symbol 29 + 13 bits
        return [(227 + rng.randrange(31), 24577 + rng.randrange(8192)) for _ in range(n)]
    toks48 = t48(40)

    def deep48(npad):
        t = toks48 + t48(npad // 8)
        d = Writer(); d.stored(prefix); d.dynamic(t, ll_deep, dl_deep, final=True)
        return d, d.raw(), expand(t, prefix)
    both(out, "deep48", deep48)

    # a body of 15-bit literal codes only (EOB and a few length codes take the short ones)
    ll15 = fill([15] * 256 + [0] * 30, list(range(256, 286)))
    lit15 = [rng.randrange(256) for _ in range(150)]

    def only15(npad):
        t = lit15 + [rng.randrange(256) for _ in range(npad)]
        d = Writer(); d.dynamic(t, ll15, [], final=True)
        return d, d.raw(), expand(t)
    both(out, "only15", only15)

    # small tables
    def eob_only(npad):                                 # one 1-bit code: end of block; an empty block
        d = Writer(); d.dynamic([], [0] * 256 + [1], [], final=not npad)
        tail = rbytes(random.Random(npad), npad)
        if npad:
            d.stored(tail, final=True)
        return d, d.raw(), tail
    both(out, "eob_only", eob_only)

    def eob_lit(npad):                                  # end of block and one literal, 1 bit each
        t = [0x41] * (20 + npad)
        d = Writer(); d.dynamic(t, [0] * 0x41 + [1] + [0] * 190 + [1], [], final=True)
        return d, d.raw(), expand(t)
    both(out, "eob_lit", eob_lit)

    acgt = b"ACGTN\n"
    ll_small = fill([0] * 286, list(acgt) + [256, 257, 258, 259, 260])
    ll_small_lit = fill([0] * 286, list(acgt) + [256])

    def nodist(npad):                                   # HDIST = 1 with length 0: no distance codes, literals only
        t = [rng.choice(acgt) for _ in range(30 + npad)]
        d = Writer(); d.dynamic(t, ll_small_lit, [0], final=True)
        return d, d.raw(), expand(t)
    both(out, "nodist", nodist)

    def onedist(npad):                                  # one distance code of 1 bit (symbol 3: distance 4)
        t = list(b"ACGT")
        for _ in range(10 + npad // 4):
            t += [(rng.randrange(3, 7), 4), rng.choice(acgt)]
        d = Writer(); d.dynamic(t, ll_small, [0, 0, 0, 1], final=True)
        return d, d.raw(), expand(t)
    both(out, "onedist", onedist)

    ll_full = fill([0] * 285 + [9], list(acgt) + [256] + list(range(257, 285)) + [s for s in range(256) if s not in acgt])
    dl_full = fill([0] * 29 + [5], list(range(29)))

    def full(npad):                                     # HLIT = 286, HDIST = 30: symbols 285 and 29 used
        t = [(258, 30000), (258, 24577)] + match_tokens(rng, [260, 270], [0, 5], 4) + [rng.choice(acgt) for _ in range(npad)]
        d = Writer(); d.stored(prefix); d.dynamic(t, ll_full, dl_full, final=True)
        return d, d.raw(), expand(t, prefix)
    both(out, "hlit286_hdist30", full)

    ll5 = [8] * 255 + [0, 8]                            # HCLEN 5: code-length symbols 16, 17, 18, 0 and 8 only

    def hclen5(npad):
        t = [rng.randrange(255) for _ in range(40 + npad)]
        d = Writer(); d.dynamic(t, ll5, [], final=True)
        return d, d.raw(), expand(t)
    both(out, "hclen5", hclen5)

    def hclen19(npad):                                  # all 19 code-length code lengths sent, the last ones 0
        t = [rng.choice(acgt) for _ in range(30 + npad)]
        d = Writer(); d.dynamic(t, ll_small_lit, [], final=True, hclen=15)
        return d, d.raw(), expand(t)
    both(out, "hclen19", hclen19)

    lens = [0] * 286
    ll138 = fill(lens, list(range(100)) + list(range(238, 256)) + [256])    # literals 100..237: 138 zeros

    def run138(npad):
        t = [rng.choice(list(range(100)) + list(range(238, 256))) for _ in range(30 + npad)]
        d = Writer(); d.dynamic(t, ll138, [], final=True)
        return d, d.raw(), expand(t)
    both(out, "run138", run138)

    # repeats across the literal/distance boundary: a 16 (lengths 6), and a 17 / 18 (zeros, HLIT forced to 286)
    ll16 = fill([0] * 280 + [6] * 6, list(acgt) + [256])
    dl16 = fill([6] * 6 + [0] * 24, list(range(6, 30)))
    ll0 = fill([0] * 286, list(acgt) + [256] + list(range(257, 270)))               # 16 zeros at the end: an 18 crosses
    ll6 = fill([0] * 286, list(acgt) + [256] + list(range(257, 280)))               # 6 zeros at the end: a 17 crosses
    for name, lx, dx, kw in (("rep16_cross", ll16, dl16, {}), ("rep17_cross", ll6, [0] * 3 + [1, 1], dict(hlit=29)),
                             ("rep18_cross", ll0, [0] * 8 + [1, 1], dict(hlit=29))):
        def rep(npad, lx=lx, dx=dx, kw=kw):
            ds = [s for s in range(30) if s < len(dx) and dx[s]]
            ls = [s for s in range(257, 286) if lx[s]]
            t = list(b"ACGTACGTACGTACGTACGTACGTACGTACGT") + match_tokens(rng, ls, [s for s in ds if DBASE[s] <= 32], 8)
            t += [rng.choice(acgt) for _ in range(npad)]
            d = Writer(); d.dynamic(t, lx, dx, final=True, **kw)
            return d, d.raw(), expand(t)
        both(out, name, rep)

    # block sequences: deep, shallow, fixed; shallow, deep; a stored block where a (parallel) block ends; empty stored
    def seq1(npad):
        t1 = lit15[:40]
        t2 = [rng.choice(acgt) for _ in range(30)]
        t3 = [rng.randrange(256) for _ in range(10)] + [(10, 7)] + [rng.randrange(256) for _ in range(npad // 8)]
        d = Writer(); d.dynamic(t1, ll15, []); d.dynamic(t2, ll_small_lit, []); d.fixed(t3, final=True)
        return d, d.raw(), expand(t1 + t2 + t3)
    both(out, "seq_deep_shallow_fixed", seq1)

    def seq2(npad):
        t1 = [rng.choice(acgt) for _ in range(30)]
        t2 = lit15[:30] + [rng.randrange(256) for _ in range(npad // 15)]
        d = Writer(); d.dynamic(t1, ll_small_lit, []); d.dynamic(t2, ll15, [], final=True)
        return d, d.raw(), expand(t1 + t2)
    both(out, "seq_shallow_deep", seq2)

    def seq_stored(npad):
        t1 = [rng.choice(acgt) for _ in range(25 + npad)]
        d = Writer(); d.dynamic(t1, ll_small_lit, [])
        if d.n % 8 == 0:
            t1.append(ord("A")); d = Writer(); d.dynamic(t1, ll_small_lit, [])
        s = rbytes(rng, 100)
        t3 = [rng.choice(acgt) for _ in range(12)] + [(6, 50)] + [rng.choice(acgt) for _ in range(npad)]
        d.stored(s); d.dynamic(t3, ll_small, [0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 1, 1], final=True)
        return d, d.raw(), expand(t1) + s + expand(t3, expand(t1) + s)[len(expand(t1)) + len(s):]
    both(out, "seq_stored_unaligned", seq_stored)

    def seq_empty(npad):
        t1 = [rng.randrange(256) for _ in range(20)]
        t2 = [rng.choice(acgt) for _ in range(20 + npad)]
        d = Writer(); d.fixed(t1); d.stored(b""); d.dynamic(t2, ll_small_lit, []); d.stored(b"", final=True)
        return d, d.raw(), expand(t1 + t2)
    both(out, "seq_stored_empty", seq_empty)

    # bytes behind the final block: the lane that holds the end-of-block code moves
    tj = [rng.choice(acgt) for _ in range(1400)]
    d = Writer(); d.dynamic(tj, ll_small_lit, [], final=True)
    for k in (0, 1, 2, 3, 5, 17, 64, 150, 300, 600, 1200):
        out.append(Case("trailing%d" % k, d, d.raw() + rbytes(rng, k), footer(expand(tj)), "par", expand(tj)))
    d = Writer(); d.dynamic(tj[:40], ll_small_lit, [], final=True)
    for k in (1, 7, 100):
        out.append(Case("trailing_ser%d" % k, d, d.raw() + rbytes(rng, k), footer(expand(tj[:40])), "ser", expand(tj[:40])))

    # the final end-of-block code ends on bit 0 of the footer (the CRC's lowest bit supplies it)
    for name, n0, ll_e in (("eob_in_footer_fixed_ser", 30, None), ("eob_in_footer_fixed_par", 500, None),
                           ("eob_in_footer_dyn_ser", 40, ll_small_lit), ("eob_in_footer_dyn_par", 1400, ll_small_lit)):
        for seed in range(400):
            r = random.Random(seed)
            t = [r.choice(acgt if ll_e else acgt + b"\xc8\xe1") for _ in range(n0 + seed % 8)]
            d = Writer()
            if ll_e is None:
                d.fixed(t, final=True)
            else:
                d.dynamic(t, ll_e, [], final=True)
            want = expand(t)
            if d.n % 8 == 1 and (d.v >> (d.n - 1)) & 1 == zlib.crc32(want) & 1:
                raw = d.raw()[:-1]
                out.append(Case(name, d, raw, footer(want), name[-3:], want))
                break
        else:
            raise AssertionError("no payload puts the end-of-block code into the footer: " + name)
    return out


def malformed_cases():
    """Streams zlib refuses, each built for one message; truncated ones end without an error (NO_END)"""
    rng = random.Random(22)
    out = []
    acgt = b"ACGTN\n"
    ll = fill([0] * 286, list(acgt) + [256, 257, 258, 259, 260])
    toks = [rng.choice(acgt) for _ in range(20)]

    def hdr(name, msg, **kw):
        d = Writer(); d.dynamic(kw.pop("toks", toks), kw.pop("ll", ll), kw.pop("dl", [0, 1, 1]), final=True, **kw)
        out.append(Case(name, d, d.raw(), bytes(8), None, None, msg))

    seq = rle_lengths(ll + [0, 1, 1])
    hdr("cl_incomplete", "invalid code lengths set", cl=[2 if s in (0, 5, 6) else 0 for s in range(19)])
    hdr("cl_over", "invalid code lengths set", cl=[1 if s in (0, 5, 18) else 2 if s == 17 else 0 for s in range(19)])
    hdr("cl_single", "invalid code lengths set", cl=[1 if s == 0 else 0 for s in range(19)])
    hdr("rep16_first", "invalid bit length repeat", seq=[(16, 0)] + seq)
    hdr("rep_past_end", "invalid bit length repeat", seq=seq[:-1] + [(18, 0)])
    for f in (30, 31):
        hdr("hlit_field%d" % f, "too many length or distance symbols", hlit=f)
        hdr("hdist_field%d" % f, "too many length or distance symbols", hdist=f)
    hdr("ll_over", "invalid literal/lengths set", ll=[0] * 65 + [1, 1] + [0] * 189 + [1])
    hdr("ll_incomplete", "invalid literal/lengths set", ll=[0] * 65 + [2] + [0] * 190 + [2])
    hdr("dl_over", "invalid distances set", dl=[1, 1, 1])
    hdr("dl_incomplete", "invalid distances set", dl=[2, 2])
    hdr("no_eob_code", "invalid code -- missing end-of-block", ll=fill([0] * 286, list(acgt)), eob=False)
    hdr("hclen4", "invalid code -- missing end-of-block", hclen=0, ll=[0] * 257, dl=[0], toks=[], eob=False,
        cl=[1 if s in (0, 18) else 0 for s in range(19)], seq=[(18, 127), (18, 109)])       # only zero lengths can be sent

    # body-level errors, in both decoders: the bad token comes after npad good ones
    def fixed_bad(kind):
        def build(npad):
            d = Writer(); d.bits(1, 1); d.bits(1, 2); d.bodies.append(d.n)
            for _ in range(npad + 5):
                d.lit(rng.randrange(144, 256))
            if kind in (286, 287):
                d.lit(kind)
            else:
                d.lit(257); d.code(kind, 5)
            return d, d.raw() + rbytes(rng, 4), b""
        return build
    for s in (286, 287):
        both(out, "fixed_litlen%d" % s, fixed_bad(s), "invalid literal/length code")
    for s in (30, 31):
        both(out, "fixed_dist%d" % s, fixed_bad(s), "invalid distance code")

    def nodist_len(npad):
        t = [rng.choice(acgt) for _ in range(5 + npad)] + [(5, 1)] + [rng.choice(acgt) for _ in range(10)]
        d = Writer(); d.dynamic(t, ll, [0] * 30, final=True)
        return d, d.raw(), b""
    both(out, "nodist_length_code", nodist_len, "invalid distance code")

    for name, pre, dist in (("far_first", 0, 1), ("far_first2", 1, 2), ("far_mid", 100, 101)):
        def far(npad, pre=pre, dist=dist):
            t = [rng.choice(acgt) for _ in range(pre)] + [(3, dist)] + [rng.choice(acgt) for _ in range(10 + npad)]
            d = Writer(); d.dynamic(t, ll, fill([0] * 30, range(16)), final=True)
            return d, d.raw(), b""
        both(out, name, far, "invalid distance too far back")
        both(out, name + "_fixed", lambda npad, pre=pre, dist=dist: _fixed_far(rng, pre, dist, npad), "invalid distance too far back")

    d = Writer(); d.bits(1, 1); d.bits(3, 2); d.bits(0, 13)
    out.append(Case("block_type3", d, d.raw(), bytes(8), None, None, "invalid block type"))
    d = Writer(); d.fixed(toks); d.bits(1, 1); d.bits(0, 2); d.n = (d.n + 7) // 8 * 8; d.bits(5, 16); d.bits(5, 16)
    out.append(Case("stored_nlen", d, d.raw() + bytes(5), bytes(8), None, None, "invalid stored block lengths"))

    # truncation: every cut of a small and a large dynamic member, footer kept
    lt = fill([0] * 286, [ord("e"), 256] + list(b"tao") + list(range(257, 262)) + list(b"insrhldcu"))
    for name, n in (("cut_small", 60), ("cut_large", 900)):
        t = [rng.choice(b"etaoinsrhldcu") for _ in range(8)]
        while len(t) < n:
            t.append((rng.randrange(3, 8), rng.randrange(1, 5)) if rng.random() < 0.2 else rng.choice(b"etaoinsrhldcu"))
        d = Writer(); d.dynamic(t, lt, [1, 2, 3, 3], final=True)
        raw, foot = d.raw(), footer(expand(t))
        for cut in range(1, len(raw)):
            out.append(Case("%s%d" % (name, cut), None, raw[:cut], foot, None, None, None))
    # a three-literal block cut before its end-of-block code, footer zeroed: zlib decodes the zero bits as the literal
    # with the all-zeros code, then runs out of input
    l3 = [0] * 286
    l3[ord("a")], l3[ord("b")], l3[ord("c")], l3[256] = 1, 2, 3, 3

    def cut3(npad):
        t = list(b"abc") + [rng.choice(b"abc") for _ in range(npad)]
        d = Writer(); d.dynamic(t, l3, [], final=True, eob=False)
        return d, d.raw(), b""
    both(out, "cut_zero_footer", cut3, NO_END)
    for zero in (False, True):                          # a last block that is not final
        t = [rng.choice(acgt) for _ in range(30)]
        d = Writer(); d.dynamic(t, ll, [0, 1, 1])
        out.append(Case("not_final%s" % ("_zero_footer" if zero else ""), d, d.raw(),
                        bytes(8) if zero else footer(expand(t)), None, None, None))
    return out


def _fixed_far(rng, pre, dist, npad):
    t = [rng.randrange(256) for _ in range(pre)] + [(3, dist)] + [rng.randrange(144, 256) for _ in range(10 + npad)]
    d = Writer(); d.fixed(t, final=True)
    return d, d.raw(), b""


_CASES = None


def cases():
    global _CASES
    if _CASES is None:
        _CASES = valid_cases() + malformed_cases()
    return _CASES


def expected(c):
    """(status bgzf_uncompress + the CRC check give, output): what the kernel must return for the block"""
    st, data, _ = zlib_bgzf(c.raw + c.foot)
    if st:
        return H.BGZF_ERR_ZLIB, b""
    return (0, data) if zlib.crc32(data) & 0xffffffff == struct.unpack("<I", c.foot[:4])[0] else (H.BGZF_ERR_CRC, b"")


def bgzf(c, flip=False):
    foot = bytearray(c.foot)
    if flip:
        foot[0] ^= 1
    return b"\x1f\x8b\x08\x04\0\0\0\0\0\xff\x06\0BC\x02\0" + struct.pack("<H", 18 + len(c.raw) + 8 - 1) + c.raw + bytes(foot)


# ---------------------------------------------------------------- CPU: the streams are what they are meant to be
def test_worst_case_search_matches_zlib():
    """the search gives zlib's ENOUGH_LENS / ENOUGH_DISTS for zlib's roots (9 and 6 bits), and for the kernel's roots
    (9 and 8) codes that reach it exist; the kernel reserves room for both"""
    assert (1 << 9) + worst_case(286, 9)[0] == 852
    assert (1 << 6) + worst_case(30, 6)[0] == 592
    for n, root, want in ((286, LIT_ROOT, 340), (30, DST_ROOT, 144)):
        val, depths = worst_case(n, root)
        assert val == want and len(depths) <= n and max(depths) == 15
        assert sum(1 << (15 - l) for l in depths) == 1 << 15                     # complete
        assert subtable_slots(sorted(depths), root) == want
        assert subtable_slots(sorted(depths)[::-1], root) == want                # slots depend on the lengths only
    assert (1 << LIT_ROOT) + 340 <= (1 << LIT_ROOT) + 856 and (1 << DST_ROOT) + 144 <= (1 << DST_ROOT) + 512


def test_valid_streams_inflate_with_zlib():
    """every valid case inflates in zlib, as bgzf_uncompress calls it, to what its tokens expand to"""
    for c in valid_cases():
        assert zlib_bgzf(c.raw + c.foot) == (0, c.want, None), c.name
        assert len(c.want) < SLOT, c.name


def test_case_shapes():
    """each case is built for its decoder and has the shape its name says"""
    vc = valid_cases()
    for c in vc + malformed_cases():
        if c.dec is not None:
            assert c.decs and set(c.decs) == {c.dec}, (c.name, c.decs)
    by = {c.name: c for c in vc}
    worst = [c for c in vc if c.name.startswith("worst_ser")]
    assert len(worst) >= 2 and "worst_par" in by
    # the worst-case tables are the ones the members carry, and every coded symbol is used
    _, blocks = orc_inflate_trace(by["worst_par"].raw + by["worst_par"].foot)
    dyn = blocks[-1]
    assert dyn["btype"] == 2
    assert subtable_slots(dyn["ll"][:286], LIT_ROOT) == 340 and subtable_slots(dyn["dist"][:30], DST_ROOT) == 144
    used_l, used_d = set(), set()
    for c in worst:
        for b in orc_inflate_trace(c.raw + c.foot)[1][-1:]:
            for t in b["toks"]:
                if isinstance(t, int):
                    used_l.add(t)
                else:
                    used_l.add(257 + max(i for i in range(29) if LBASE[i] <= t[0]))
                    used_d.add(max(i for i in range(30) if DBASE[i] <= t[1]))
    assert used_l | {256} == {s for s in range(286) if dyn["ll"][s]} and used_d == {s for s in range(30) if dyn["dist"][s]}
    # 15-bit codes for literals, length symbols 265..284 and distance symbols 26..29; 48-bit tokens back to back
    b = orc_inflate_trace(by["deep_syms_ser"].raw + by["deep_syms_ser"].foot)[1][-1]
    assert all(b["ll"][s] == 15 for s in range(265, 285)) and sum(b["ll"][s] == 15 for s in range(256)) == 16
    assert all(b["dist"][s] == 15 for s in range(26, 30)) and b["cl"][15] and b["bfinal"]
    b = orc_inflate_trace(by["deep48_ser"].raw + by["deep48_ser"].foot)[1][-1]
    assert all(not isinstance(t, int) and 227 <= t[0] <= 257 and t[1] > 24576 for t in b["toks"]) and len(b["toks"]) >= 40
    b = orc_inflate_trace(by["only15_par"].raw + by["only15_par"].foot)[1][-1]
    assert all(b["ll"][t] == 15 for t in b["toks"]) and len(b["toks"]) * 15 >= PAR_MIN_BITS
    # header edges
    hdr = lambda name: by[name].raw[0] | by[name].raw[1] << 8 | by[name].raw[2] << 16
    b = orc_inflate_trace(by["hlit286_hdist30_ser"].raw + by["hlit286_hdist30_ser"].foot)[1][-1]
    assert b["ll"][285] and b["dist"][29] and 285 in [257 + max(i for i in range(29) if LBASE[i] <= t[0]) for t in b["toks"]
                                                      if not isinstance(t, int)]
    assert hdr("hclen5_ser") >> 13 & 15 == 1 and hdr("hclen19_ser") >> 13 & 15 == 15
    assert hdr("eob_only_ser") >> 3 & 0x3ff == 0
    ll138 = orc_inflate_trace(by["run138_ser"].raw + by["run138_ser"].foot)[1][-1]["ll"]
    assert (18, 127) in rle_lengths(ll138[:257])
    for name, sym in (("rep16_cross_ser", 16), ("rep17_cross_ser", 17), ("rep18_cross_ser", 18)):
        b = orc_inflate_trace(by[name].raw + by[name].foot)[1][-1]
        nl = 257 + (hdr(name) >> 3 & 31)
        nd = 1 + (hdr(name) >> 8 & 31)
        assert nl == 286
        reps = repeats(rle_lengths(b["ll"][:nl] + b["dist"][:nd]))
        assert any(s == sym and a < nl < e for s, a, e in reps), (name, reps)
    # the stored block starts at an unaligned bit behind a parallel-decoded block
    bl = orc_inflate_trace(by["seq_stored_unaligned_par"].raw + by["seq_stored_unaligned_par"].foot)[1]
    assert [b["btype"] for b in bl] == [2, 0, 2] and bl[1]["start_bit"] % 8
    # trailing bytes move the lane whose range holds the end-of-block code
    lanes = set()
    for c in vc:
        if c.name.startswith("trailing") and not c.name.startswith("trailing_ser"):
            b = orc_inflate_trace(c.raw + c.foot)[1][-1]
            total = (len(c.raw) + 8) * 8
            S = (total - b["body_bit"] + 31) // 32
            lanes.add((b["end_bit"] - 1 - b["body_bit"]) // S)
    assert len(lanes) >= 6, lanes
    # the end-of-block code's last bit is the footer's first
    for c in vc:
        if c.name.startswith("eob_in_footer"):
            b = orc_inflate_trace(c.raw + c.foot)[1][-1]
            assert b["end_bit"] == 8 * len(c.raw) + 1, c.name


def test_malformed_streams_fail_in_zlib_with_their_message():
    """each malformed stream stops zlib with the message it was built for; truncated streams end without end of stream.
    A member cut short with its footer kept reads the footer as deflate data: it fails in zlib, or ends there with the
    wrong CRC"""
    seen = set()
    for c in malformed_cases():
        st, _, msg = zlib_bgzf(c.raw + c.foot)
        if c.msg is not None:
            assert (st, msg) == (H.BGZF_ERR_ZLIB, c.msg), (c.name, msg)
            seen.add(msg)
        else:
            assert expected(c)[0] in (H.BGZF_ERR_ZLIB, H.BGZF_ERR_CRC), c.name
    assert len(seen) == 12


def test_oracle_agrees_with_zlib():
    """orc_bgzf_inflate_block gives bgzf_uncompress's status and bytes on every case (valid, flipped CRC, malformed)"""
    for c in cases():
        for flip in (False, True):
            blk = bgzf(c, flip)
            want = expected(Case(c.name, None, c.raw, blk[-8:]))
            rc, data = orc_bgzf_inflate_block(blk)
            assert (min(rc, 0), data) == want, (c.name, flip, rc)


# ---------------------------------------------------------------- GPU
@pytest.fixture(scope="module")
def ctx():
    c = H.Context(0)
    yield c
    c.close()


@pytest.mark.gpu
@pytest.mark.parametrize("flip", [False, True])
def test_bgzf_inflate_every_case(ctx, flip):
    """every case as a BGZF block at output offsets 0..3 mod 16 in a 64 KiB slot: zlib's bytes where zlib accepts the
    stream, exactly BGZF_ERR_ZLIB where zlib refuses it; with the CRC's lowest bit flipped, every valid stream is
    BGZF_ERR_CRC except those whose end-of-block code ends on that bit (the flip changes their data)"""
    blocks, want, shifts, names = [], [], [], []
    crc_err = 0
    for c in cases():
        if flip and expected(c)[0] != 0:
            continue
        blk = bgzf(c, flip)
        w = expected(Case(c.name, None, c.raw, blk[-8:]))
        crc_err += w[0] == H.BGZF_ERR_CRC
        for sh in range(4):
            blocks.append(blk); want.append(w); shifts.append(sh); names.append(c.name)
    assert not flip or crc_err >= len(blocks) // 4 - 4
    res = _inflate(ctx, blocks, shifts, [SLOT] * len(blocks))
    bad = [(names[i], shifts[i], st, w[0], len(d), len(w[1])) for i, ((st, d), w) in enumerate(zip(res, want)) if (st, d) != w]
    assert not bad, bad[:12]


def _gzip_uncompress(ctx, comps, sizes):
    """gzip members as CRAM GZIP blocks (method 1) of the given uncompressed sizes through gzip_inflate_kernel"""
    n = len(comps)
    dt = np.dtype([("data_off", "<u8"), ("comp_size", "<u4"), ("uncomp_size", "<u4"), ("content_id", "<i4"), ("method", "u1"),
                   ("content_type", "u1"), ("hdr_len", "<u2"), ("container", "<u4"), ("pad2", "<u4")])
    blocks = np.zeros(n, dtype=dt)
    for i, cb in enumerate(comps):
        blocks[i]["method"] = 1; blocks[i]["content_type"] = 4; blocks[i]["content_id"] = 10 + i
        blocks[i]["comp_size"] = len(cb); blocks[i]["uncomp_size"] = sizes[i]
    L = H.lib()
    L.hgpu_cram_write_blocks_host.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p]
    bufs = [np.frombuffer(cb, dtype=np.uint8).copy() for cb in comps]
    ptrs = (C.c_void_p * n)(*[b.ctypes.data for b in bufs])
    img = np.zeros(sum(len(cb) for cb in comps) + 32 * n, dtype=np.uint8)
    off = np.zeros(n, dtype=np.uint64); tot = C.c_uint64(0)
    assert L.hgpu_cram_write_blocks_host(ctx.h, blocks.ctypes.data, ptrs, n, img.ctypes.data, img.size, off.ctypes.data, C.byref(tot)) == 0
    img = img[:tot.value].copy()
    scanned = blocks.copy()
    for i in range(n):
        hl = 2 + sum(1 if v < 0x80 else 2 if v < 0x4000 else 3 if v < 0x200000 else 4 if v < 0x10000000 else 5
                     for v in (10 + i, len(comps[i]), sizes[i]))
        scanned[i]["hdr_len"] = hl; scanned[i]["data_off"] = int(off[i]) + hl
    return H.cram_uncompress_blocks(ctx, img, scanned)[1]


@pytest.mark.gpu
def test_gzip_inflate_every_case(ctx):
    """the same streams as gzip members (CRAM GZIP blocks): zlib's bytes where it accepts them, HGPU_CRAM_UNSUPPORTED
    (back to the host library) where it refuses them.  A refused stream's slot is only a little longer than zlib's
    partial output, so a decoder that runs on past its input stops at the slot"""
    comps, sizes, want, names = [], [], [], []
    for c in cases():
        st, data, _ = zlib_bgzf(c.raw + c.foot)
        ok = st == 0 and zlib.crc32(data) & 0xffffffff == struct.unpack("<I", c.foot[:4])[0] and len(data) == struct.unpack("<I", c.foot[4:])[0]
        comps.append(b"\x1f\x8b\x08\0\0\0\0\0\0\x03" + c.raw + c.foot)
        sizes.append(len(data) if ok else len(data) + 64)
        want.append(data if ok else None if st else False)
        names.append(c.name)
    res = _gzip_uncompress(ctx, comps, sizes)
    bad = []
    for name, (st, data), w in zip(names, res, want):
        if w is None:                                   # zlib refuses it
            good = st == CRAM_UNSUPPORTED
        elif w is False:                                # inflates, but not to its CRC / ISIZE
            good = st not in (0, CRAM_UNSUPPORTED)
        else:
            good = st == 0 and data == w
        if not good:
            bad.append((name, st, len(data)))
    assert not bad, bad[:12]
