"""CPU checks of the fqzcomp writer (tests/fqz_model.py).

- Pinned to the reference encoder: every stored reference stream with one parameter block and no selector, seeded
  as in test_oracle_fqz.py, is what fqz_model.encode writes given that stream's parameters and input.
- decode_cases(): streams over the parts of the format the reference encoder never writes (several parameter blocks,
  selector tables, quality tables, 256-symbol alphabets, long records, duplicates under reversal, malformed headers).
  Each decodes to its intended bytes with oracle/orc_fqz.c, and to the same bytes with the reference's
  fqz_decompress (stored results), and reaches the edge it was built for.  test_gpu_fqzcomp_model.py runs the same
  cases through the device decoder."""
import random

import pytest

import _libs as L
import fqz_model as M
from test_oracle_fqz import _quals

UNKNOWN = object()          # a damaged stream: no intended output, the decoders must only agree


@L.stored_reference(digest=True)
def ref_fqz_model_decompress(comp):
    """L.ref_fqz_decompress for the streams of decode_cases(), stored apart from that helper's own results."""
    return L.ref_fqz_decompress.__wrapped__(comp)


class Case:
    def __init__(self, name, stream, want, trace=None, edge=None):
        self.name, self.stream, self.want, self.trace, self.edge = name, stream, want, trace, edge


def _syms(rng, n, top):
    return [rng.randrange(top + 1) for _ in range(n)]


def _records(rng, gp, n_rec, lens=(1, 300), sel_top=None, dup_rate=0.0, rev_rate=0.0, sym_top=None):
    """(symbols, records) that follow the decoder's rules for gp: a fixed-length block repeats the last coded length,
    a duplicate needs the selected block's PFLAG_DO_DEDUP and enough bytes before it."""
    nparam, max_sel, stab = M.resolved(gp)
    b0 = gp["blocks"][0]
    gmax = max(b["max_sym"] for b in gp["blocks"])
    sym_top = gmax if sym_top is None else sym_top
    syms, recs, first, last_len, total = [], [], True, 0, 0
    for _ in range(n_rec):
        sel = rng.randrange((max_sel if sel_top is None else sel_top) + 1) if b0["pflags"] & M.PFLAG_DO_SEL else 0
        x = stab[min(255, sel)] if gp["gflags"] & M.GFLAG_HAVE_STAB else sel
        pm = gp["blocks"][min(x, nparam - 1)]
        if pm["pflags"] & M.PFLAG_DO_LEN and not first:
            n = last_len
        else:
            n = rng.randrange(lens[0], lens[1] + 1)
            first, last_len = False, n
        dup = bool(pm["pflags"] & M.PFLAG_DO_DEDUP and n <= total and rng.random() < dup_rate)
        if not dup:
            syms += _syms(rng, n, sym_top)
        recs.append(M.record(n, sel=sel, rev=int(rng.random() < rev_rate), dup=int(dup)))
        total += n
    return syms, recs


def _case(name, syms, recs, gp, edge=None):
    stream, want, t = M.encode(syms, recs, gp)
    return Case(name, stream, want, t, edge)


def _multi(rng, nparam, with_stab):
    """nparam blocks that differ in starting context, fixed length, dedup, max_sym and quality map; block 0 selects."""
    blocks = []
    for i in range(nparam):
        fl = (M.PFLAG_DO_SEL if i == 0 else 0) | (M.PFLAG_DO_LEN if i % 3 == 1 else 0) | (M.PFLAG_DO_DEDUP if i % 2 == 0 else 0)
        ms = [40, 12, 63, 7][i % 4]
        qmap = None
        if i % 4 == 1 or i == 0:
            fl |= M.PFLAG_HAVE_QMAP
            qmap = sorted(rng.sample(range(256), ms))
        blocks.append(M.block(context=rng.randrange(65536), pflags=fl | (M.PFLAG_HAVE_PTAB if i == 0 else 0), max_sym=ms,
                              qbits=8, qshift=3, qloc=4, sloc=0, ploc=12, dloc=14, qmap=qmap,
                              ptab=[min(15, k >> 4) for k in range(1024)] if i == 0 else None))
    if with_stab:
        max_sel = min(255, 4 * nparam)
        stab = [min(nparam - 1, s * nparam // (max_sel + 1)) for s in range(256)]
        return M.gparams(blocks, max_sel=max_sel, stab=stab)
    return M.gparams(blocks)


def decode_cases():
    rng = random.Random(7)
    cases = []
    add = cases.append

    # ---- several parameter blocks
    for nparam in (2, 3, 16, 255):
        for with_stab in (False, True):
            gp = _multi(rng, nparam, with_stab)
            nsel = M.resolved(gp)[1]
            syms, recs = _records(rng, gp, 300 if nparam < 255 else 600, lens=(1, 60), dup_rate=0.2,
                                  sel_top=nsel - (0 if with_stab else 1))
            want_blocks = min(nparam, 2 if nparam == 2 else 3)
            add(_case("nparam%d%s" % (nparam, "+stab" if with_stab else ""), syms, recs, gp,
                      lambda t, n=want_blocks: len(t.blocks_used) >= n and t.dups > 0))
    stab = [0] * 128 + [1] * 127 + [2]                             # many selectors -> a few blocks; 255 -> block 2
    gp = M.gparams([M.block(pflags=M.PFLAG_DO_SEL, max_sym=30, qbits=6, qshift=2, sloc=8),
                    M.block(context=77, pflags=M.PFLAG_DO_LEN, max_sym=20), M.block(context=999, max_sym=9)],
                   max_sel=255, stab=stab)
    syms, recs = _records(rng, gp, 200, lens=(1, 40), sym_top=9)
    for r in recs[-3:]:                                            # block 2 has no PFLAG_DO_LEN: lengths stay coded
        r["sel"] = 255
    add(_case("max_sel255", syms, recs, gp, lambda t: t.max_sel == 255 and 2 in t.blocks_used))
    gp = M.gparams([M.block(pflags=M.PFLAG_DO_SEL, max_sym=5)] + [M.block(max_sym=5)] * 2)
    syms, recs = _records(rng, gp, 10, lens=(1, 9), sel_top=2)
    recs.append(M.record(4, sel=3))
    add(_case("sel_eq_nparam", syms, recs, gp, lambda t: t.max_sel == 3))
    gp = M.gparams([M.block(max_sym=20, qbits=4, qshift=2), M.block(pflags=M.PFLAG_DO_SEL, max_sym=20)])
    syms, recs = _records(rng, gp, 30, lens=(1, 50))
    add(_case("do_sel_block1_only", syms, recs, gp, lambda t: t.max_sel == -1 and t.blocks_used == {0}))

    # ---- context fields: every value 0-15 of each, with sums past 16 bits
    for v in range(16):
        pm = M.block(pflags=M.PFLAG_DO_SEL | M.PFLAG_HAVE_PTAB | M.PFLAG_HAVE_DTAB, max_sym=40,
                     qbits=v, qshift=(v * 7 + 3) % 16, qloc=(v * 5 + 1) % 16, sloc=(v * 3 + 2) % 16,
                     ploc=(v * 11 + 5) % 16, dloc=(v * 13 + 7) % 16,
                     ptab=[min(255, k >> 2) for k in range(1024)], dtab=[min(255, k * 4) for k in range(256)])
        gp = M.gparams([pm], max_sel=7, stab=[0] * 256)
        syms, recs = _records(rng, gp, 12, lens=(20, 300))
        top = (((1 << v) - 1) << pm["qloc"]) + (255 << pm["ploc"]) + (255 << pm["dloc"]) + (7 << pm["sloc"])
        add(_case("fields%d" % v, syms, recs, gp, lambda t, big=top >= M.CTX_SIZE: t.max_sel > 0 and (t.ctx_over_16 > 0 or not big)))
    qtab = sorted(rng.randrange(256) for _ in range(256))
    pm = M.block(pflags=M.PFLAG_HAVE_QTAB | M.PFLAG_HAVE_PTAB, max_sym=50, qbits=9, qshift=4, qloc=3, ploc=12,
                 qtab=qtab, ptab=[min(7, k >> 5) for k in range(1024)])
    gp = M.gparams([pm])
    syms, recs = _records(rng, gp, 20, lens=(30, 80))
    c = _case("qtab", syms, recs, gp)
    ident = M.encode(syms, recs, M.gparams([dict(pm, pflags=M.PFLAG_HAVE_PTAB)]))[0]
    c.edge = lambda t, differs=ident[-len(c.stream) // 2:] != c.stream[-len(c.stream) // 2:]: differs   # the table changes contexts
    add(c)
    pm = M.block(pflags=M.PFLAG_HAVE_QTAB | M.PFLAG_HAVE_PTAB | M.PFLAG_HAVE_DTAB, max_sym=30, qbits=0, qshift=3,
                 qtab=list(range(256)), ptab=[min(3, k >> 6) for k in range(1024)], dtab=[min(3, k) for k in range(256)],
                 ploc=8, dloc=10)
    gp = M.gparams([pm])
    syms, recs = _records(rng, gp, 20, lens=(30, 80))
    add(_case("qtab_flag_qbits0", syms, recs, gp, lambda t: True))
    ptab = [0] * 3 + [4] * 100 + [5] * 21 + [9] * 400 + [200] * 500
    dtab = [0, 2, 2, 7] + [8] * 60 + [100] * 192
    gp = M.gparams([M.block(pflags=M.PFLAG_HAVE_PTAB | M.PFLAG_HAVE_DTAB, max_sym=30, qbits=4, qshift=2, ploc=9,
                            dloc=1, ptab=ptab, dtab=dtab)])
    syms, recs = _records(rng, gp, 10, lens=(100, 700))
    add(_case("irregular_tabs", syms, recs, gp, lambda t: t.ctx_over_16 > 0))
    for n in (1023, 1024, 70000):
        gp = M.gparams([M.block(pflags=M.PFLAG_HAVE_PTAB | M.PFLAG_HAVE_DTAB, max_sym=3, qbits=4, qshift=2, ploc=6,
                                dloc=13, ptab=[k >> 4 for k in range(1024)], dtab=[min(7, k >> 5) for k in range(256)])])
        syms = _syms(rng, n, 3)
        add(_case("len%d" % n, syms, [M.record(n)], gp,
                  lambda t, n=n: t.p_clamped == max(0, n - 1023) and t.delta_clamped > (0 if n > 1023 else -1)))
    gp = M.gparams([M.block(pflags=M.PFLAG_HAVE_DTAB, max_sym=1, qbits=2, qshift=1, dloc=8,
                            dtab=[k >> 2 for k in range(256)])])
    add(_case("delta_over_255", [k & 1 for k in range(600)], [M.record(600)], gp, lambda t: t.delta_clamped == 600 - 257))

    # ---- alphabets
    for ms in (0, 1, 255):
        gp = M.gparams([M.block(max_sym=ms, qbits=8, qshift=4)])
        syms, recs = _records(rng, gp, 8, lens=(50, 200))
        add(_case("max_sym%d" % ms, syms, recs, gp, lambda t, ms=ms: t.max_sym == ms))
    gp = M.gparams([M.block(pflags=M.PFLAG_HAVE_QMAP, max_sym=4, qmap=[2, 12, 23, 37], qbits=3, qshift=3)])
    syms, recs = _records(rng, gp, 8, lens=(50, 200))
    add(_case("qmap_max_sym", syms, recs, gp, lambda t: t.max_sym == 4))
    gp = M.gparams([M.block(max_sym=40)])
    syms = [0 if k % 7 else 1 + k % 40 for k in range(6000)]
    syms[:50] = [39] * 50                                          # 39 climbs over 0..38 to the front, then 0 takes over
    add(_case("normalise_swap", syms, [M.record(3000), M.record(3000)], gp,
              lambda t: t.max_ctx_uses > 4096 and t.normalises > 0 and t.swaps_to_front > 1))

    gp = M.gparams([M.block(max_sym=14)])                          # 15 symbols: the total steps onto 65519 exactly
    syms = [k % 3 for k in range(4200)]
    add(_case("normalise_at_max", syms, [M.record(4200)], gp, lambda t: t.tot_at_max > 0 and t.normalises > 0))

    # ---- records
    gp = M.gparams([M.block(max_sym=10)])
    add(_case("ulen0", [], [], gp, lambda t: t.records == 0))
    add(_case("one_byte", [7], [M.record(1)], gp, lambda t: t.records == 1))
    gp = M.gparams([M.block(pflags=M.PFLAG_DO_LEN, max_sym=30, qbits=5, qshift=5)])
    syms, recs = _records(rng, gp, 50, lens=(10, 100))
    add(_case("fixed_len", syms, recs, gp, lambda t: t.records == 50))
    gp = M.gparams([M.block(pflags=M.PFLAG_DO_DEDUP | M.PFLAG_DO_LEN, max_sym=30)])
    add(_case("all_dups", _syms(rng, 75, 30), [M.record(75)] + [M.record(75, dup=1)] * 40, gp, lambda t: t.dups == 40))
    add(_case("dup_first", [], [M.record(5, dup=1)], gp, lambda t: True))
    gp = M.gparams([M.block(pflags=M.PFLAG_DO_DEDUP, max_sym=30, qbits=5, qshift=5)], gflags=M.GFLAG_DO_REV)
    syms, recs = _records(rng, gp, 120, lens=(1, 40), dup_rate=0.3, rev_rate=0.5)
    add(_case("rev_dups", syms, recs, gp,
              lambda t: t.dups > 5 and {r["length"] % 2 for r in recs if r["rev"]} == {0, 1}))
    gp = M.gparams([M.block(max_sym=30)])
    add(_case("len0", _syms(rng, 10, 30), [M.record(10), M.record(0), M.record(5)], gp, lambda t: True))
    gp = M.gparams([M.block(max_sym=30)], ulen=25)
    add(_case("len_past_end", _syms(rng, 10, 30), [M.record(10), M.record(20)], gp, lambda t: True))

    # ---- range coder
    syms = _steer_carry_over_ff()
    gp = M.gparams([M.block(max_sym=255)])
    base = _case("carry_over_ff", syms, [M.record(len(syms))], gp, lambda t: t.carry_over_ff > 0)
    add(base)
    add(Case("trailing_bytes", base.stream + b"\xff\x00\x17", base.want))
    add(Case("last_byte_needed", base.stream[:-1], None))

    # ---- malformed headers and tables: each refused while its parameters are read
    good = M.block(max_sym=30, pflags=M.PFLAG_HAVE_PTAB | M.PFLAG_HAVE_DTAB, ptab=[k >> 8 for k in range(1024)],
                   dtab=[k >> 6 for k in range(256)])
    good_gp = M.gparams([good])
    coded = M.encode(_syms(rng, 40, 30), [M.record(40)], good_gp)[0][len(M.var_put_u32(40) + M.store_params(good_gp)):]
    for name, gp in (
            ("stab_repeat_at_end", M.gparams([good], max_sel=3, stab=[0] * 256, raw={"stab": bytes([2, 3, 4, 5, 6, 7, 7])})),
            ("ptab_too_many_runs", M.gparams([good], raw={(0, "ptab"): bytes([0, 0, 255] + [0, 255] * 4)})),
            ("dtab_short", M.gparams([good], raw={(0, "dtab"): bytes([10, 20])})),
            ("dtab_ends_in_255", M.gparams([good], raw={(0, "dtab"): bytes([255, 255, 0])})),
            ("vers4", M.gparams([good], vers=4)),
            ("nparam0", M.gparams([good], gflags=M.GFLAG_MULTI_PARAM, nparam=0)),
            ("sel_without_max_sel", M.gparams([dict(good, pflags=good["pflags"] | M.PFLAG_DO_SEL)]))):
        cut = name in ("stab_repeat_at_end", "dtab_short")   # these tables must end the stream
        add(Case(name, M.var_put_u32(40) + M.store_params(gp) + (b"" if cut else coded), None))
    qm = M.block(pflags=M.PFLAG_HAVE_QMAP, max_sym=200, qmap=list(range(200)))
    add(Case("qmap_past_end", (M.var_put_u32(40) + M.store_params(M.gparams([qm])))[:60], None))

    # ---- damaged streams
    shorts = []
    gp = _multi(rng, 3, True)
    shorts.append(_case("short_stab", *_records(rng, gp, 6, lens=(1, 9), dup_rate=0.3), gp))
    gp = M.gparams([M.block(pflags=M.PFLAG_DO_DEDUP | M.PFLAG_HAVE_QMAP, max_sym=3, qmap=[9, 20, 30], qbits=2, qshift=1)],
                   gflags=M.GFLAG_DO_REV)
    shorts.append(_case("short_rev", *_records(rng, gp, 6, lens=(1, 9), dup_rate=0.3, rev_rate=0.5), gp))
    gp = M.gparams([dict(pm, max_sym=6)])
    shorts.append(_case("short_qtab", *_records(rng, gp, 4, lens=(1, 12)), gp))
    for c in shorts:
        add(c)
        for k in range(len(c.stream)):
            add(Case("%s_cut%d" % (c.name, k), c.stream[:k], UNKNOWN))
    src = next(c for c in cases if c.name == "nparam16+stab").stream
    hdr = M.parse_params(src)[1]
    for k in range(200):
        b = bytearray(src)
        pos = rng.randrange(1, hdr) if k % 2 else rng.randrange(hdr, len(src))
        b[pos] ^= 1 << rng.randrange(8)
        add(Case("flip%d" % k, bytes(b), UNKNOWN))
    return cases


def _steer_carry_over_ff(limit=4000):
    """Symbols for one 256-symbol context that hold back three or more 0xff bytes and then carry into them: each
    symbol is picked, among those the model offers, for where it puts the coder's low end."""
    t = M.Trace()
    rc = M.RangeCoder(t)
    m = M.SimpleModel(256, 256, t)
    out = []
    while t.carry_over_ff == 0 and len(out) < limit:
        r = rc.range // m.tot
        best = None
        acc = 0
        for i in range(256):
            f = m.F[i]
            low = rc.low + acc * r
            carry = low > M.M32
            low &= M.M32
            rng_ = r * f
            ff, score = rc.ffnum, 0
            while rng_ < M.TOP:                                    # the shifts this symbol would cause
                if low < M.THRES or carry or rc.carry:
                    score = 1000 if (carry or rc.carry) and ff >= 3 else score
                    if not score:
                        ff = 0
                else:
                    ff += 1
                    score += 10
                carry = False
                low = (low << 8) & M.M32
                rng_ <<= 8
            score += ff * 10 + (low >> 24) / 256.0
            if carry:
                score += 1 + (500 if ff >= 3 else 0)
            if best is None or score > best[0]:
                best = (score, m.S[i])
            acc += f
        out.append(best[1])
        m.encode(rc, best[1])
    assert t.carry_over_ff, "no symbol sequence found"
    return out


CASES = decode_cases()


def test_model_pinned_to_reference_encoder():
    """Every stored reference stream of test_oracle_fqz's seeded inputs with gflags 0 (or only GFLAG_DO_REV) is what
    fqz_model.encode writes from the stream's own parameters."""
    rng = random.Random(11)
    pinned = 0
    for vers in (4, 3):
        for kind in ("q4", "q40", "var"):
            for strat in (0, 1, 2, 3):
                for n_rec in (1, 7, 300):
                    q, lens, flags = _quals(rng, n_rec, kind)
                    with L.sampled():
                        c = L.ref_fqz_compress(q, lens, flags, strat, vers)
                        gp, _ = M.parse_params(c)
                        if gp["gflags"] & ~M.GFLAG_DO_REV:
                            continue
                        stored, revs, pos = bytearray(q), [], 0
                        for n, f in zip(lens, flags):
                            rv = int(vers == 3 and bool(f & 16))
                            if rv:
                                stored[pos:pos + n] = stored[pos:pos + n][::-1]
                            revs.append(rv)
                            pos += n
                        syms, recs = M.symbols_of(bytes(stored), lens, gp)
                        for r, rv in zip(recs, revs):
                            r["rev"] = rv
                        s, want, _ = M.encode(syms, recs, gp)
                        assert want == q
                        assert s == c, (vers, kind, strat, n_rec)
                        pinned += 1
    assert pinned >= 20, pinned


def test_store_and_read_array_round_trip():
    """read_array keeps at most 1023 run bytes (:165), so values stay below 900 here."""
    rng = random.Random(5)
    for size in (256, 1024):
        for _ in range(50):
            arr = sorted(rng.choice([rng.randrange(4), rng.randrange(300), rng.randrange(min(size, 900))]) for _ in range(size))
            arr = [a - arr[0] for a in arr] if rng.random() < 0.5 else arr
            b = M.store_array(arr)
            assert M.read_array(b + b"\x00\x09", size) == (arr, len(b))


@pytest.mark.parametrize("c", [c for c in CASES if c.edge], ids=lambda c: c.name)
def test_case_reaches_its_edge(c):
    assert c.edge(c.trace), c.name


def test_cases_against_oracle_and_reference():
    checked = refused = 0
    for c in CASES:
        got = L.orc_fqz_decode(c.stream)
        if c.want is not UNKNOWN:
            assert got == c.want, c.name
        want = ref_fqz_model_decompress(c.stream)                  # stored for every case: raises where it is not
        assert (want is None) == (got is None), c.name
        if got is not None:
            assert want == got, c.name
        checked += 1
        refused += got is None
    assert checked == len(CASES) == 479, len(CASES)
    assert refused > 250, refused
