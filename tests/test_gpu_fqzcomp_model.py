"""GPU: the fqzcomp kernels against the plain writer of tests/fqz_model.py.

Decoder (fqz_decode_kernel): every stream of test_fqz_model.decode_cases() -- several parameter blocks, selector
tables, quality tables, every context field value, long records, 256-symbol alphabets, duplicates under reversal,
malformed parameters, cut and bit-flipped streams -- in one batch and again shuffled: status and bytes equal
oracle/orc_fqz.c's and the intended output.  A batch whose model arenas pass the 6 GiB wave budget decodes as its
streams do one by one.

Encoder (fqz_encode_kernel): for inputs that reach every strategy row, alphabet size class, quality map choice, size
class, fixed and variable lengths, both sides of the dedup ratio and long records, the stream's head equals
fqz_model.device_params and the whole stream equals fqz_model.encode of those parameters; where the reference keeps
no selector the stream equals the reference's byte for byte, and where it keeps one the parameter blocks agree in
every field the selector search leaves alone.  A batch past the wave budget encodes as its blocks do one by one."""
import random

import pytest

import htslib_b200 as H
import _libs as L
import fqz_model as M
from test_fqz_model import CASES, UNKNOWN

pytestmark = pytest.mark.gpu
HGPU_FQZ_ERR = -1


@L.stored_reference
def ref_fqz_model_params(quals, lens, strat):
    """The size field and parameter blocks at the head of the reference's fqz_compress stream: small whatever the
    input's size."""
    comp = L.ref_fqz_compress.__wrapped__(quals, lens, None, strat, 4)
    return comp[:M.parse_params(comp)[1]]


@L.stored_reference(digest=True)
def ref_fqz_model_compressed(quals, lens, strat):
    """The reference's whole fqz_compress stream as a Digest."""
    return L.ref_fqz_compress.__wrapped__(quals, lens, None, strat, 4)


@pytest.fixture(scope="module")
def ctx():
    c = H.Context(0)
    yield c
    c.close()


def _cap(c):
    """The output slot given to the device: the intended length, else the size field where it is sane."""
    if c.want not in (None, UNKNOWN):
        return len(c.want)
    try:
        ulen = M.var_get_u32(c.stream)[0] if c.stream else 0
    except IndexError:
        ulen = 0
    return ulen if ulen <= 1 << 20 else 64


_ORC = {}


def _check(cases, res):
    for c, (st, data) in zip(cases, res):
        if c.stream not in _ORC:
            _ORC[c.stream] = L.orc_fqz_decode(c.stream)
        want = _ORC[c.stream]
        if c.want is not UNKNOWN:
            assert want == c.want, c.name
        if want is None or len(want) > _cap(c):
            assert st == HGPU_FQZ_ERR, c.name
        else:
            assert st == 0 and data == want, c.name


def test_decode_cases_one_batch_and_shuffled(ctx):
    _check(CASES, H.fqz_decode(ctx, [c.stream for c in CASES], [_cap(c) for c in CASES]))
    order = list(range(len(CASES)))
    random.Random(3).shuffle(order)
    shuffled = [CASES[i] for i in order]
    _check(shuffled, H.fqz_decode(ctx, [c.stream for c in shuffled], [_cap(c) for c in shuffled]))


def test_decode_size_field_past_output_slot(ctx):
    good = [c for c in CASES if c.want not in (None, UNKNOWN) and len(c.want) > 0][:20]
    res = H.fqz_decode(ctx, [c.stream for c in good], [len(c.want) - 1 for c in good])
    assert all(st == HGPU_FQZ_ERR for st, _ in res)


def _wide_streams(n):
    """n short streams with 256-symbol models (68 MB of models each)."""
    rng = random.Random(9)
    out = []
    for k in range(n):
        gp = M.gparams([M.block(max_sym=255, qbits=8, qshift=8, pflags=M.PFLAG_DO_DEDUP)])
        syms = [rng.randrange(256) for _ in range(40 + k)]
        recs = [M.record(20 + k), M.record(20), M.record(20, dup=1)]
        stream, want, _ = M.encode(syms, recs, gp)
        out.append((stream, want))
    return out


def _free_bytes():
    import torch
    return torch.cuda.mem_get_info()[0]


def test_decode_waves_match_one_by_one(ctx):
    if _free_bytes() < 10 << 30:
        pytest.skip("needs 10 GB of free device memory")
    streams = _wide_streams(100)                                   # 100 x 68 MB of models: two waves under 6 GiB
    res = H.fqz_decode(ctx, [s for s, _ in streams], [len(w) for _, w in streams])
    for (s, w), (st, data) in zip(streams, res):
        assert st == 0 and data == w
        assert H.fqz_decode(ctx, [s], [len(w)]) == [(0, w)]


# ---------------------------------------------------------------- encoder
def _blocks():
    """(name, quals, lens): inputs chosen to reach each of the device encoder's parameter rules."""
    rng = random.Random(31)

    def iid(alphabet, lens):
        return bytes(rng.choice(alphabet) for _ in range(sum(lens))), list(lens)

    out = [("nsym4_qmap_fixed", *iid((2, 12, 23, 37), [151] * 300)),
           ("nsym7_qmap_var", *iid((2, 7, 13, 20, 27, 33, 40), [rng.randrange(50, 250) for _ in range(300)])),
           ("nsym5_no_qmap", *iid(range(5), [100] * 300)),
           ("nsym4_max8_no_qmap", *iid((0, 3, 6, 8), [100] * 300)),      # nsym * 2 == max_sym: no quality map
           ("nsym40_fixed", *iid(range(2, 42), [100] * 300)),
           ("nsym40_first_small", *iid(range(2, 42), [20] + [rng.randrange(50, 250) for _ in range(600)])),
           ("nsym40_first_large", *iid(range(2, 42), [5000] + [rng.randrange(50, 250) for _ in range(1999)])),
           ("long_records", *iid(range(2, 42), [rng.randrange(1024, 3000) for _ in range(40)])),
           ("sym256", *iid(range(256), [rng.randrange(100, 400) for _ in range(20)]))]
    for name, nrec, ndup in (("dedup_ratio_250", 999, 3), ("dedup_ratio_500", 999, 1)):
        recs = [bytes(rng.randrange(2, 42) for _ in range(20)) for _ in range(nrec)]
        for k in range(ndup):
            recs[100 + 200 * k + 1] = recs[100 + 200 * k]
        out.append((name, b"".join(recs), [20] * nrec))
    return out


def _big_block():
    rng = random.Random(32)
    lens = [151] * 33200
    return "size_5M", bytes(rng.randrange(2, 42) for _ in range(sum(lens))), lens


def _fields(gp):
    """A parameter block's fields as the device writes them: the selector search only adds PFLAG_DO_SEL."""
    pm = dict(gp["blocks"][0])
    pm["pflags"] &= ~M.PFLAG_DO_SEL
    return pm


def test_encode_against_model_and_reference(ctx):
    blocks = _blocks()
    reached = set()
    same_as_ref = with_sel = 0
    for strat in (0, 1, 2, 3):
        res = H.fqz_encode(ctx, [q for _, q, _ in blocks], [lens for _, _, lens in blocks], strat)
        for (name, q, lens), (st, comp) in zip(blocks, res):
            assert st == 0, (name, strat)
            head, gp, facts = M.device_params(q, lens, strat)
            assert comp[:len(head)] == head, (name, strat)
            syms, recs = M.symbols_of(q, lens, gp)
            stream, want, _ = M.encode(syms, recs, gp)
            assert want == q and comp == stream, (name, strat)
            ref_head = ref_fqz_model_params(q, lens, strat)
            rgp, _ = M.parse_params(ref_head)
            if rgp["gflags"] == 0:
                assert ref_fqz_model_compressed(q, lens, strat) == comp, (name, strat)
                same_as_ref += 1
                nsym = facts["nsym"]
                reached |= {"strat%d" % strat, "nsym<=4" if nsym <= 4 else "nsym<=8" if nsym <= 8 else "nsym>8",
                            "qmap" if facts["store_qmap"] else "no_qmap", "fixed" if facts["fixed_len"] else "variable",
                            "dedup" if facts["do_dedup"] else "no_dedup",
                            "size<300k" if len(q) < 300000 else "size<5M", "rec>1023" if max(lens) > 1023 else "rec<=1023",
                            "sym256" if max(q) == 255 else "sym<256"}
                if facts["nsym"] <= 8 and facts["nsym"] * 2 == facts["max_sym"]:
                    reached.add("qmap_boundary")
                if strat == 0 and facts["nsym"] > 4:
                    reached.add("pshift%d" % facts["pshift"])
            else:
                assert rgp["gflags"] == M.GFLAG_HAVE_STAB and rgp["nparam"] == 1, (name, strat)
                assert _fields(rgp) == _fields(gp), (name, strat)
                with_sel += 1
    assert reached >= {"strat0", "strat1", "strat2", "strat3", "nsym<=4", "nsym<=8", "nsym>8", "qmap", "no_qmap",
                       "fixed", "variable", "dedup", "no_dedup", "size<300k", "size<5M", "rec>1023", "sym256", "qmap_boundary",
                       "pshift4", "pshift9"}, reached
    assert same_as_ref >= 30 and with_sel >= 1, (same_as_ref, with_sel)


def test_encode_5mb_block_against_reference(ctx):
    name, q, lens = _big_block()
    for strat in (0,):
        (st, comp), = H.fqz_encode(ctx, [q], [lens], strat)
        assert st == 0
        head, gp, facts = M.device_params(q, lens, strat)
        assert comp[:len(head)] == head and facts["size"] >= 5000000
        assert M.parse_params(ref_fqz_model_params(q, lens, strat))[0]["gflags"] == 0
        assert ref_fqz_model_compressed(q, lens, strat) == comp, strat


def test_encode_waves_match_one_by_one(ctx):
    if _free_bytes() < 10 << 30:
        pytest.skip("needs 10 GB of free device memory")
    rng = random.Random(41)
    quals = [bytes([255]) + bytes(rng.randrange(256) for _ in range(50 + k)) for k in range(100)]
    lens = [[len(q) // 2, len(q) - len(q) // 2] for q in quals]
    batch = H.fqz_encode(ctx, quals, lens, 0)                      # 100 x 68 MB of models: two waves under 6 GiB
    for q, l, got in zip(quals, lens, batch):
        assert got[0] == 0
        assert H.fqz_encode(ctx, [q], [l], 0) == [got]
        assert L.orc_fqz_decode(got[1]) == q
