"""CPU checks of the references the deflate-kernel tests rely on (tests/deflate_model.py, the oracle's
orc_inflate_trace): the trace against zlib's own streams, the pass-2 restatement against zlib's inflater, the Huffman
references against brute force and each other, and the seeded inputs against the edges they are made to reach."""
import itertools
import random
import zlib

import pytest

import deflate_model as M
from _libs import orc_inflate_raw, orc_inflate_trace


def all_tokens(blocks, out):
    """The tokens of a traced stream; a stored block's bytes count as literals."""
    toks, pos = [], 0
    for b in blocks:
        if b["btype"] == 0:
            n = (b["end_bit"] - b["body_bit"]) // 8
            toks += list(out[pos:pos + n])
            pos += n
        else:
            toks += b["toks"]
            pos += sum(1 if isinstance(t, int) else t[0] for t in b["toks"])
    return toks


def expand(toks):
    out = bytearray()
    for t in toks:
        if isinstance(t, int):
            out.append(t)
        else:
            for _ in range(t[0]):
                out.append(out[-t[1]])
    return bytes(out)


def corpus(seed):
    rng = random.Random(seed)
    txt = b"".join(b"read%d\t%d\tchr%d\t%d\t60\t150M\n" % (i, rng.randrange(4096), rng.randrange(24), rng.randrange(1 << 20))
                   for i in range(800))
    return [txt[:40000], bytes(rng.choice(b"ACGT") for _ in range(30000)), b"\0" * 3000 + b"ab" * 2000,
            bytes(rng.randrange(256) for _ in range(3000)), b"x", b""]


STRATEGIES = [(lv, zlib.Z_DEFAULT_STRATEGY) for lv in range(1, 10)] + [(6, zlib.Z_FIXED), (6, zlib.Z_HUFFMAN_ONLY),
                                                                         (6, zlib.Z_RLE)]


def zlib_raw(p, level, strategy):
    c = zlib.compressobj(level, zlib.DEFLATED, -15, 8, strategy)
    return c.compress(p) + c.flush()


@pytest.mark.parametrize("level,strategy", STRATEGIES)
def test_trace_expands_zlib_streams(level, strategy):
    for p in corpus(level):
        raw = zlib_raw(p, level, strategy)
        out, blocks = orc_inflate_trace(raw)
        assert out == p == orc_inflate_raw(raw)[0]
        assert blocks[-1]["bfinal"] == 1 and all(b["bfinal"] == 0 for b in blocks[:-1])
        assert expand(all_tokens(blocks, out)) == p
        assert blocks[0]["start_bit"] == 0 and blocks[-1]["end_bit"] <= 8 * len(raw) < blocks[-1]["end_bit"] + 8
        for a, b in zip(blocks, blocks[1:]):
            assert a["end_bit"] == b["start_bit"]
        for b in blocks:
            toks = b["toks"]
            if strategy == zlib.Z_HUFFMAN_ONLY:
                assert all(isinstance(t, int) for t in toks)
            if strategy == zlib.Z_RLE:
                assert all(isinstance(t, int) or t[1] == 1 for t in toks)
            if strategy == zlib.Z_FIXED and toks:
                assert b["btype"] == 1
            if b["btype"] == 1:
                assert b["ll"] == M.FIXED_LL and b["dist"][:30] == [5] * 30 and b["body_bit"] == b["start_bit"] + 3
            if b["btype"] == 2:
                # the traced lengths are what zlib sent: the code lengths it built are complete (or one 1-bit code)
                assert M.kraft(b["ll"], 15) == 1 << 15
                assert M.kraft(b["dist"], 15) in (1 << 15, 1 << 14)
                assert M.kraft(b["cl"], 7) == 1 << 7
                # and the header is exactly as long as its own fields say
                assert b["body_bit"] - b["start_bit"] >= 17 + 3 * 4
            if b["btype"] == 0:
                assert not toks and b["body_bit"] % 8 == 0


@pytest.mark.parametrize("level,strategy", STRATEGIES)
def test_pass2_reencodes_zlib_tokens(level, strategy):
    """The restatement turns zlib's tokens into a block that zlib inflates back, whose trace gives the same tokens and
    whose code lengths are the ones the restatement says it built."""
    for p in corpus(level + 50):
        raw = zlib_raw(p, level, strategy)
        out, blocks = orc_inflate_trace(raw)
        toks = all_tokens(blocks, out)
        blk, info = M.pass2(toks, p, 6)
        assert len(blk) <= M.SLOT
        assert zlib.decompress(blk[18:-8], -15) == p
        assert zlib.decompress(blk, 31) == p                    # a valid gzip member: header, CRC32, ISIZE
        out, tb = orc_inflate_trace(blk[18:-8])
        assert out == p and len(tb) == 1
        if info["kind"] == "stored":
            assert tb[0]["btype"] == 0 and info["why"] in ("short", "size")
            continue
        assert tb[0]["toks"] == toks
        assert tb[0]["btype"] == (2 if info["kind"] == "dynamic" else 1)
        bits = tb[0]["end_bit"] - tb[0]["start_bit"]
        assert bits == (info["dyn_bits"] if info["kind"] == "dynamic" else info["fixed_bits"])
        assert info["dlen"] == (bits + 7) // 8
        if info["kind"] == "dynamic":
            assert tb[0]["ll"][:286] == info["ll"] and tb[0]["dist"][:30] == info["dist"] and tb[0]["cl"] == info["cl"]
            assert tb[0]["body_bit"] - tb[0]["start_bit"] == info["dyn_bits"] - M.code_cost(info["freq"], info["ll"]) \
                - M.code_cost(info["dfreq"], info["dist"]) - sum(M.LEN_XTRA[M.len_sym(t[0])] + M.DST_XTRA[M.dist_sym(t[1])]
                                                                for t in toks if not isinstance(t, int))
        else:
            assert info["fixed_bits"] <= info["dyn_bits"]


def test_pass2_stored_rules():
    p = bytes(range(15))
    assert M.pass2(list(p), p, 6)[1]["why"] == "short"
    p = b"abc" * 100
    blk, info = M.pass2([97, 98, 99, (258, 3), (39, 3)], p, 0)
    assert info["why"] == "level0" and blk == M.stored_block(p) and len(blk) == len(p) + 5 + 26
    assert M.pass2([97, 98, 99, (258, 3), (39, 3)], p, 1)[1]["kind"] in ("fixed", "dynamic")


def test_limit_fallback_margin():
    """65280 bytes with every byte value equally often go stored because the result is not smaller (dlen >= n + 5),
    well before the token bits reach the end of the slot: the slot-end fallback is a guard, not a size rule."""
    p = M.incompressible_payload()
    _, info = M.pass2(list(p), p, 6)
    assert info["why"] == "size" and 18 * 8 + info["dyn_bits"] < M.LIMIT_BITS


def brute_lengths(freqs, limit):
    """(min cost, min depth at that cost) over every complete prefix code with lengths 1..limit."""
    best = None
    for lens in itertools.product(range(1, limit + 1), repeat=len(freqs)):
        if sum(2.0 ** -l for l in lens) == 1.0:
            c = M.code_cost(freqs, lens)
            if best is None or c < best[0] or (c == best[0] and max(lens) < best[1]):
                best = (c, max(lens))
    return best


def test_huffman_references_vs_brute_force():
    rng = random.Random(7)
    for _ in range(60):
        k = rng.randint(2, 6)
        freqs = [rng.choice([1, 1, 2, 3, 5, 8, 13, 40, 100]) for _ in range(k)]
        opt, depth = M.huffman_opt(freqs)
        assert opt == brute_lengths(freqs, k - 1)[0]
        for limit in range(max(1, (k - 1).bit_length()), k):
            if k <= 1 << limit:
                assert M.package_merge(freqs, limit) == brute_lengths(freqs, limit)[0], (freqs, limit)
        assert M.package_merge(freqs, k - 1) == opt
        assert depth <= k - 1


def test_build_lengths_against_the_optima():
    rng = random.Random(8)
    fib = [1, 1]
    while len(fib) < 25:
        fib.append(fib[-1] + fib[-2])
    cases = [[rng.randrange(0, 1000) for _ in range(286)] for _ in range(20)]
    cases += [fib[:20] + [0] * 10, fib[:24], [rng.choice([0, 1, 2, 1000]) for _ in range(19)], fib[:10] + [0] * 9]
    folded = 0
    for freqs in cases:
        for limit in (7, 15):
            if sum(1 for f in freqs if f) > 1 << limit:
                continue
            lens = M.build_lengths(freqs, limit)
            assert [f > 0 for f in freqs] == [l > 0 for l in lens] and max(lens) <= limit
            if sum(1 for f in freqs if f) > 1:
                assert M.kraft(lens, limit) == 1 << limit
            opt, depth = M.huffman_opt(freqs)
            cost = M.code_cost(freqs, lens)
            if depth <= limit:
                assert cost == opt
            else:
                folded += 1
                pm = M.package_merge(freqs, limit)
                # the fold is zlib's heuristic, not package-merge: 8 % over on 24 Fibonacci weights folded to 7 bits
                assert opt < pm <= cost <= 1.10 * pm
    assert folded >= 4


def test_literal_only_inputs_reach_their_edges():
    """The literal-only generators: no repeated 4-byte string and no byte three times running, so the kernel's tokens
    are the literals and pass2 predicts each block; each reaches the edge it is made for."""
    for p in (M.ll_fold_payload(), M.cl_fold_payload()):
        assert len({p[i:i + 4] for i in range(len(p) - 3)}) == len(p) - 3
        assert all(not (p[i] == p[i + 1] == p[i + 2]) for i in range(len(p) - 2))
    p = M.ll_fold_payload()
    _, info = M.pass2(list(p), p, 6)
    assert info["kind"] == "dynamic" and M.huffman_opt(info["freq"])[1] > 15 and max(info["ll"]) == 15
    p = M.cl_fold_payload()
    _, info = M.pass2(list(p), p, 6)
    assert info["kind"] == "dynamic" and M.huffman_opt(info["clf"])[1] > 7 and max(info["cl"]) == 7
    assert info["dist"] == [1] + [0] * 29


def test_planted_copies_survive_the_kernel_hash():
    for L, cl, d in ((300, 300, 400), (257, 257, 400), (8, 8, 32768), (8, 8, 32769)):
        buf, src, p = M.planted_copy(1, L, cl, d)
        assert p - src == d and buf[p:p + cl] == buf[src:src + cl] and M.hash_survives(buf, src, p)
        assert buf[p + cl] != buf[src + cl]
    p, planted = M.dist_fold_payload()
    assert len(p) <= M.MAX_PAYLOAD and M.huffman_opt(list(planted.values()))[1] == 16
