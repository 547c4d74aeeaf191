"""GPU parity: rANS Nx16 decode (hgpu_rans_nx16_decode_batch_*, rans_uncompress_to_4x16 shim)
against the oracle / compiled reference — bit exact."""
import ctypes as C
import glob, os, random
import numpy as np
import pytest
import htslib_b200 as H
from _libs import GOLD, golden_raw, orc_rans_nx16_decode, ref, ref_rans_nx16_encode, sampled
from test_oracle_rans import _synth, ORDERS

pytestmark = pytest.mark.gpu
R4X16 = sorted(glob.glob(os.path.join(GOLD, "htscodecs", "dat", "r4x16", "*")))


@pytest.fixture(scope="module")
def ctx():
    c = H.Context(0)
    yield c
    c.close()


def run_batch(ctx, comps, ulens):
    n = len(comps)
    in_off = np.zeros(n, dtype=np.uint64); in_len = np.zeros(n, dtype=np.uint32)
    out_off = np.zeros(n, dtype=np.uint64); out_len = np.array(ulens, dtype=np.uint32)
    p = 0; q = 0
    for i, c in enumerate(comps):
        in_off[i] = p; in_len[i] = len(c); p += len(c) + (7 * i) % 5      # ragged, unaligned starts
        out_off[i] = q; q += ulens[i] + (3 * i) % 4
    blob = np.zeros(max(1, p), dtype=np.uint8)
    for i, c in enumerate(comps):
        blob[int(in_off[i]):int(in_off[i]) + len(c)] = np.frombuffer(c, dtype=np.uint8)
    out = np.full(max(1, q), 0xAA, dtype=np.uint8)
    got, st = ctx.rans_nx16_decode_host(blob, in_off, in_len, out, out_off, out_len)
    res = []
    for i in range(n):
        res.append((int(st[i]), out[int(out_off[i]):int(out_off[i]) + int(got[i])].tobytes()))
    return res


def test_golden_vectors_batch(ctx):
    comps, raws = [], []
    for path in R4X16:
        raws.append(golden_raw(os.path.basename(path).rsplit(".", 1)[0]))
        comps.append(open(path, "rb").read())
    res = run_batch(ctx, comps, [len(r) for r in raws])
    for path, (st, data), raw in zip(R4X16, res, raws):
        assert st == 0, path
        assert data == raw, path


@pytest.mark.parametrize("order", ORDERS)
def test_seeded_all_formats(ctx, order):
    rng = random.Random(99 + order)
    comps, raws = [], []
    for kind in ("q4", "q40", "runs", "one", "u32", "rand"):
        for n in (1, 3, 31, 32, 33, 100, 1000, 1023, 4099, 70001):
            raw = _synth(rng, n, kind)
            with sampled():
                comps.append(ref_rans_nx16_encode(raw, order)); raws.append(raw)
    res = run_batch(ctx, comps, [len(r) for r in raws])
    for i, ((st, data), raw) in enumerate(zip(res, raws)):
        assert st == 0, (order, i, len(raw), comps[i][:6].hex())
        assert data == raw, (order, i, len(raw), comps[i][:6].hex())


def test_corrupt_streams_match_oracle(ctx):
    rng = random.Random(5)
    raw = _synth(rng, 6000, "q40")
    comps = []
    for order in (0, 1, 4, 5, 65, 129, 193, 9):
        comp = ref_rans_nx16_encode(raw, order, store_always=True)
        for _ in range(30):
            c = bytearray(comp)
            k = rng.randrange(len(c) // 2, len(c)); c[k] ^= 1 << rng.randrange(8)
            comps.append(bytes(c))
        comps.append(comp[: len(comp) // 2])       # truncated
        comps.append(comp[:3])
    res = run_batch(ctx, comps, [len(raw)] * len(comps))
    ok = 0
    for c, (st, data) in zip(comps, res):
        want = orc_rans_nx16_decode(c, len(raw))
        if want is None:
            assert st != 0
        else:
            assert st == 0 and data == want
            ok += 1
    assert ok > 100


def test_shim_malloc_and_errors(ctx):
    L = H.lib()
    libc = C.CDLL(None)
    rng = random.Random(3)
    raw = _synth(rng, 50000, "q4")
    for order in (1, 5, 193, 8):
        comp = ref_rans_nx16_encode(raw, order, store_always=True)
        buf = (C.c_uint8 * len(comp)).from_buffer_copy(comp)
        n = C.c_uint(0)
        p = L.rans_uncompress_4x16(buf, len(comp), C.byref(n))
        assert p and n.value == len(raw)
        assert C.string_at(p, n.value) == raw
        libc.free(C.c_void_p(p))                          # libc-malloc ownership, like cram_io.c:1675
        small = (C.c_uint8 * 10)(); m = C.c_uint(10)      # capacity too small -> NULL
        assert not L.rans_uncompress_to_4x16(buf, len(comp), small, C.byref(m))
    assert not L.rans_uncompress_4x16(buf, 0, C.byref(n))


def test_device_api_large_qs_blocks(ctx):
    """CRAM-shaped: 1.5 MB 32-way order-1 quality blocks + small 4-way blocks, device pointers."""
    import torch
    rng = np.random.default_rng(11)
    raws, comps = [], []
    for i in range(24):
        n = 1_500_000 if i % 3 == 0 else 15000
        syms = np.array([35, 45, 56, 70], dtype=np.uint8)
        st = np.cumsum(rng.random(n) < 0.15) + i
        raw = syms[(st * 2654435761 >> 7) % 4].astype(np.uint8).tobytes()
        raws.append(raw)
        comps.append(ref_rans_nx16_encode(raw, 5 if n > 100000 else (i % 2)))
    in_len = np.array([len(c) for c in comps], dtype=np.uint32)
    in_off = np.concatenate([[0], np.cumsum((in_len + 15) // 16 * 16)[:-1]]).astype(np.uint64)
    out_len = np.array([len(r) for r in raws], dtype=np.uint32)
    out_off = np.concatenate([[0], np.cumsum(out_len)[:-1]]).astype(np.uint64)
    blob = np.zeros(int(in_off[-1]) + int(in_len[-1]) + 16, dtype=np.uint8)
    for o, c in zip(in_off, comps):
        blob[int(o):int(o) + len(c)] = np.frombuffer(c, dtype=np.uint8)
    dev = torch.device("cuda:0")
    d_in = torch.from_numpy(blob).to(dev)
    d_out = torch.zeros(int(out_len.sum()) + 16, dtype=torch.uint8, device=dev)
    t = lambda a: torch.from_numpy(a.view(np.int64) if a.dtype == np.uint64 else a.view(np.int32)).to(dev)
    d_io, d_il, d_oo, d_ol = t(in_off), t(in_len), t(out_off), t(out_len)
    d_got = torch.zeros(len(comps), dtype=torch.int32, device=dev)
    d_st = torch.full((len(comps),), 7, dtype=torch.int32, device=dev)
    ctx.rans_nx16_decode_dev(d_in, d_io, d_il, d_out, d_oo, d_ol, d_got, d_st, int(out_len.max()),
                             torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    assert d_st.cpu().tolist() == [0] * len(comps)
    assert d_got.cpu().numpy().astype(np.uint32).tolist() == out_len.tolist()
    out = d_out.cpu().numpy()
    for o, r in zip(out_off, raws):
        assert out[int(o):int(o) + len(r)].tobytes() == r
