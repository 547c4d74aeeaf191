"""Plain references for the rANS Nx16 encoder (rans_nx16_encode_kernel, htslib_b200/csrc/rans_nx16_enc.cu), no GPU.

- trace: parse a stream into its whole structure (containers, transforms, every entropy core with its table as stored,
  states and words).  Reads the reference's streams as well as the kernel's.
- core_encode / core_decode: a plain rANS Nx16 entropy coder, vectorised across the N states.  Given the tables of a
  trace, core_encode returns the core's exact bytes.
- histogram, row_target, normalise_row, shift_rule, serialise_o0, serialise_o1: the kernel's table rules restated.
- normalise_opt: the exact optimum max sum c*log f (f >= 1 where c > 0, sum f = M); normalise_ref: the reference's
  normalise_freq (htscodecs rANS_static16_int.h:97-146) restated, for cost comparisons.
- encode: the kernel's container logic (encode_stream / encode_flat / encode_stripe) restated: returns its bytes.

Citations without a file name are to rans_nx16_enc.cu."""
import heapq
import math

import numpy as np

F_ORDER, F_X32, F_STRIPE, F_NOSZ, F_CAT, F_RLE, F_PACK = 1, 4, 8, 0x10, 0x20, 0x40, 0x80
F_STRIPE_NO0 = 1 << 16
RANS_L = 1 << 15
NEST_MAX = 160 * 1024 - 4096          # longest order-1 table text (less its first byte) the kernel tries to code


# ---------------------------------------------------------------- varints and alphabets
def vput(v):
    """var_put_u32 (varint.h:206): 7-bit groups, most significant first, bit 7 = more follow."""
    out = bytearray()
    for sh in (28, 21, 14, 7):
        if v >= 1 << sh:
            out.append(((v >> sh) & 0x7f) | 0x80)
    out.append(v & 0x7f)
    return bytes(out)


def vget(b, p):
    v = 0
    while True:
        c = b[p]
        p += 1
        v = (v << 7) | (c & 0x7f)
        if not c & 0x80:
            return v, p


def put_alphabet(present):
    """encode_alphabet (rANS_static16_int.h:165-189): ascending symbols; one that follows a present symbol is followed by
    the count of further consecutive present symbols, which are then not listed; 0 ends the list."""
    out = bytearray()
    rle = 0
    for j in range(256):
        if not present[j]:
            continue
        if rle:
            rle -= 1
            continue
        out.append(j)
        if j and present[j - 1]:
            r = j + 1
            while r < 256 and present[r]:
                r += 1
            rle = r - (j + 1)
            out.append(rle)
    out.append(0)
    return bytes(out)


def read_alphabet(b, p):
    """decode_alphabet (rANS_static16_int.h:191-238) -> (ascending symbols, next position)."""
    syms = []
    run = 0
    sym = b[p]
    p += 1
    while True:
        syms.append(sym)
        if run == 0 and sym + 1 == b[p]:
            sym = b[p]
            run = b[p + 1]
            p += 2
        elif run:
            run -= 1
            sym += 1
        else:
            sym = b[p]
            p += 1
        if sym == 0:
            return syms, p


# ---------------------------------------------------------------- tables
def shift_rule(A):
    """The kernel's order-1 shift: from the compact alphabet size alone (encode_core)."""
    return 10 if A <= 128 else 12


def histogram(data, order, N):
    """Order 0: 256 counts.  Order 1: 256 x 256 counts [context, symbol]; the context is the previous byte of the same
    state's segment, 0 at each segment start z * (U // N) (encode_freq1; the last segment runs to the end)."""
    d = np.frombuffer(bytes(data), dtype=np.uint8)
    if order == 0:
        return np.bincount(d, minlength=256).astype(np.int64)
    ctx = contexts(d, N)
    return np.bincount(ctx.astype(np.int64) * 256 + d, minlength=65536).reshape(256, 256).astype(np.int64)


def contexts(d, N):
    U = len(d)
    ctx = np.zeros(U, dtype=np.uint8)
    ctx[1:] = d[:-1]
    seg = U // N
    ctx[[z * seg for z in range(N) if z * seg < U]] = 0
    return ctx


def normalise_row(counts, M):
    """The kernel's normalise_row: f = max(1, c * M // total); a shortfall goes to the largest f (lowest index on a tie);
    a surplus is taken back from the largest entries, each down to no less than 1.  None when impossible."""
    c = np.asarray(counts, dtype=np.int64)
    tot = int(c.sum())
    if tot == 0:
        return c.copy()
    if int((c > 0).sum()) > M:
        return None
    f = np.where(c > 0, np.maximum(1, c * M // tot), 0)
    diff = M - int(f.sum())
    if diff > 0:
        f[int(np.argmax(f))] += diff
    while diff < 0:
        bi = int(np.argmax(f))
        b = int(f[bi])
        if b <= 1:
            return None
        take = min(b - 1, -diff)
        f[bi] -= take
        diff += take
    return f


def row_target(trow, ns, shift):
    """The total an order-1 row is stored at, and the scale-up to 2^shift (encode_core, after rans_compute_shift's
    row rule, rANS_static4x16pr.c:376-387): (M, up)."""
    if trow == 0:
        return 1 << shift, 0
    m2 = 1
    while m2 < trow:
        m2 <<= 1
    if ns < 64 and m2 > 128:
        m2 >>= 1
    if m2 > 1024:
        m2 >>= 1
    while m2 < ns:
        m2 <<= 1
    if m2 >= 1 << shift:
        return 1 << shift, 0
    up = 0
    while (m2 << up) < (1 << shift):
        up += 1
    return m2, up


def normalise_opt(counts, M):
    """The exact optimum: f maximising sum c * log f with f >= 1 where c > 0, f = 0 elsewhere, sum f = M.  The
    objective is separable and concave, so handing out units one at a time by largest marginal gain is exact."""
    c = [int(v) for v in counts]
    f = [1 if v else 0 for v in c]
    left = M - sum(f)
    if left < 0:
        return None
    h = [(-(v * math.log(2.0)), j) for j, v in enumerate(c) if v]
    heapq.heapify(h)
    while left > 0 and h:
        _, j = heapq.heappop(h)
        f[j] += 1
        left -= 1
        heapq.heappush(h, (-(c[j] * math.log((f[j] + 1) / f[j])), j))
    return np.array(f, dtype=np.int64)


def normalise_ref(counts, M):
    """The reference's normalise_freq (rANS_static16_int.h:97-146) restated: scale by a rounded reciprocal, bump zeros
    to 1, put the difference on the most frequent symbol; when that cannot absorb a surplus, rescale once, then take
    the surplus from the first entries above 1."""
    F = [int(v) for v in counts]
    size = sum(F)
    if not size:
        return np.array(F, dtype=np.int64)
    loop = 0
    while True:
        tr = ((M << 31) // size) + ((1 << 30) // size)
        m = Mi = size = 0
        for j in range(len(F)):
            if not F[j]:
                continue
            if m < F[j]:
                m, Mi = F[j], j
            F[j] = (F[j] * tr) >> 31
            if F[j] == 0:
                F[j] = 1
            size += F[j]
        adjust = M - size
        if adjust > 0:
            F[Mi] += adjust
        elif adjust < 0:
            if F[Mi] > -adjust and (loop == 1 or F[Mi] // 2 >= -adjust):
                F[Mi] += adjust
            else:
                if loop < 1:
                    loop += 1
                    continue
                adjust += F[Mi] - 1
                F[Mi] = 1
                for j in range(len(F)):
                    if not adjust:
                        break
                    if F[j] < 2:
                        continue
                    d = adjust if F[j] > -adjust else 1 - F[j]
                    F[j] += d
                    adjust -= d
        return np.array(F, dtype=np.int64)


def cost_bits(counts, f, M):
    """sum c * log2(M / f) over the symbols present."""
    c = np.asarray(counts, dtype=np.float64)
    f = np.asarray(f, dtype=np.float64)
    m = c > 0
    return float((c[m] * np.log2(M / f[m])).sum())


def serialise_o0(F):
    """Order-0 table text (encode_freq, rANS_static16_int.h:254-272): alphabet, then a varint per present symbol."""
    return put_alphabet(F) + b"".join(vput(int(v)) for v in F if v)


def serialise_o1(syms, stored, shift):
    """Order-1 table text before any nested coding: the shift byte, the alphabet, then for each context of the
    alphabet its row over the alphabet, a zero followed by the count of further zeros (encode_freq_d, :278-307)."""
    present = [0] * 256
    for s in syms:
        present[s] = 1
    out = bytearray([shift << 4]) + put_alphabet(present)
    for row in stored:
        dz = 0
        for v in row:
            v = int(v)
            if v:
                if dz:
                    out.append(dz - 1)
                dz = 0
                out += vput(v)
            else:
                if not dz:
                    out.append(0)
                dz += 1
        if dz:
            out.append(dz - 1)
    return bytes(out)


def nest_table(text):
    """The order-1 table bytes as written: the text itself, or, when it is over 1000 bytes and an order-0 4-state coding
    of text[1:] plus 6 is shorter, the first byte | 1, the two lengths and that coding (encode_freq1,
    rANS_static16_int.h:397-411)."""
    tlen = len(text)
    if tlen > 1000 and tlen - 1 <= NEST_MAX:
        c = core_encode(text[1:], 0, 4)
        if len(c) + 6 < tlen:
            return bytes([text[0] | 1]) + vput(tlen - 1) + vput(len(c)) + c
    return text


def tables_for(data, order, N):
    """The kernel's tables for one entropy core: dict(shift, syms, stored, up, freq, text).  For order 0, stored / freq
    are 256 entries; for order 1, A x A over the compact alphabet syms (every byte present, plus 0)."""
    h0 = histogram(data, 0, N)
    if order == 0:
        f = normalise_row(h0, 4096)
        return dict(order=0, shift=12, syms=[j for j in range(256) if f[j]], stored=f, up=0, freq=f, text=serialise_o0(f))
    syms = [j for j in range(256) if h0[j] or j == 0]
    A = len(syms)
    shift = shift_rule(A)
    h1 = histogram(data, 1, N)[np.ix_(syms, syms)]
    stored = np.zeros((A, A), dtype=np.int64)
    ups = np.zeros(A, dtype=np.int64)
    for r in range(A):
        M, up = row_target(int(h1[r].sum()), int((h1[r] > 0).sum()), shift)
        stored[r] = normalise_row(h1[r], M)
        ups[r] = up
    text = serialise_o1(syms, stored, shift)
    return dict(order=1, shift=shift, syms=syms, stored=stored, up=ups, freq=stored << ups[:, None],
                text_plain=text, text=nest_table(text))


# ---------------------------------------------------------------- the entropy coder
def _per_symbol(d, order, N, tables):
    """(f, start) of every symbol under the tables."""
    freq = np.asarray(tables["freq"], dtype=np.uint64)
    if order == 0:
        start = np.concatenate([[0], np.cumsum(freq)[:-1]]).astype(np.uint64)
        return freq[d], start[d]
    idx = np.zeros(256, dtype=np.int64)
    idx[tables["syms"]] = np.arange(len(tables["syms"]))
    start = np.concatenate([np.zeros((len(freq), 1), np.uint64), np.cumsum(freq, axis=1)[:, :-1]], axis=1).astype(np.uint64)
    r, k = idx[contexts(d, N)], idx[d]
    return freq[r, k], start[r, k]


def _steps(a, order, N, U, fill):
    """Lay a per-symbol array out as decode steps x states; returns (main [steps, N], tail for the last state)."""
    if order == 0:
        steps = -(-U // N)
        m = np.full(steps * N, fill, dtype=a.dtype)
        m[:U] = a
        return m.reshape(steps, N), a[:0]
    seg = U // N
    return a[:seg * N].reshape(N, seg).T, a[seg * N:]


def core_encode(data, order, N, tables=None):
    """The entropy core's bytes: table text, the N final states (little-endian u32), then the 16-bit words in the
    decoder's read order.  Symbols are coded backwards; a state about to take a symbol of frequency f first sheds its
    low 16 bits while x >= f << (31 - shift).  tables default to tables_for(data, order, N)."""
    d = np.frombuffer(bytes(data), dtype=np.uint8)
    U = len(d)
    if tables is None:
        tables = tables_for(data, order, N)
    shift = tables["shift"]
    f, s = _per_symbol(d, order, N, tables)
    fm, ft = _steps(f, order, N, U, 1 << shift)
    sm, st = _steps(s, order, N, U, 0)
    x = np.full(N, RANS_L, dtype=np.uint64)
    groups = []
    sh = np.uint64(shift)
    top = np.uint64(31 - shift)
    for p in range(len(ft) - 1, -1, -1):                 # order 1: the last state's tail is decoded last
        fr, xs = int(ft[p]), int(x[N - 1])
        if xs >= fr << (31 - shift):
            groups.append(np.array([xs & 0xffff], dtype=np.uint64))
            xs >>= 16
        x[N - 1] = ((xs // fr) << shift) + xs % fr + int(st[p])
    w16 = np.uint64(16)
    for r in range(len(fm) - 1, -1, -1):
        fr = fm[r]
        need = x >= (fr << top)
        if need.any():
            groups.append(x[need] & np.uint64(0xffff))
            x[need] >>= w16
        x = ((x // fr) << sh) + x % fr + sm[r]
    words = np.concatenate(groups[::-1]).astype("<u2") if groups else np.zeros(0, "<u2")
    return bytes(tables["text"]) + x.astype("<u4").tobytes() + words.tobytes()


def core_decode(core, U):
    """Decode a traced entropy core (a dict from trace) to its U symbols, vectorised across the states."""
    order, N, shift = core["order"], core["N"], core["shift"]
    words = core["words"].astype(np.uint64)
    x = core["states"].astype(np.uint64).copy()
    freq = np.asarray(core["freq"], dtype=np.int64)
    if order == 0:
        freq = freq[None, :]
        syms = np.arange(256)
    else:
        syms = np.asarray(core["syms"], dtype=np.int64)
    R, A = freq.shape
    idx = np.zeros(256, dtype=np.int64)
    idx[syms] = np.arange(A)
    # per row: the symbol (compact index) of each slot, and each symbol's f and first slot
    lut = np.zeros((R, 1 << shift), dtype=np.int64)
    first = np.concatenate([np.zeros((R, 1), np.int64), np.cumsum(freq, axis=1)[:, :-1]], axis=1)
    for r in range(R):
        if freq[r].sum() == 1 << shift:
            lut[r] = np.repeat(np.arange(A), freq[r])
    fq = np.maximum(freq, 1).astype(np.uint64)
    mask, L, wp = np.uint64((1 << shift) - 1), np.uint64(RANS_L), 0

    def step(xv, rows):
        nonlocal wp
        slot = (xv & mask).astype(np.int64)
        k = lut[rows, slot]
        xv = fq[rows, k] * (xv >> np.uint64(shift)) + (slot - first[rows, k]).astype(np.uint64)
        need = np.flatnonzero(xv < L)[:len(words) - wp]
        if len(need):
            xv[need] = (xv[need] << np.uint64(16)) | words[wp:wp + len(need)]
            wp += len(need)
        return xv, k
    out = np.zeros(U, dtype=np.uint8)
    if order == 0:
        for i0 in range(0, U, N):
            n = min(N, U - i0)
            x[:n], k = step(x[:n], np.zeros(n, np.int64))
            out[i0:i0 + n] = syms[k]
        return out.tobytes()
    seg = U // N
    rows = np.full(N, idx[0], dtype=np.int64)
    at = np.arange(N) * seg
    for q in range(seg):
        x, rows = step(x, rows)
        out[at + q] = syms[rows]
    for p in range(seg * N, U):
        xv, k = step(x[N - 1:], rows[N - 1:])
        x[N - 1], rows[N - 1] = xv[0], k[0]
        out[p] = syms[k[0]]
    return out.tobytes()


# ---------------------------------------------------------------- trace
def _trace_core(b, order, N, U):
    """One entropy core occupying all of b."""
    core = dict(order=order, N=N, bytes=bytes(b), n=U)
    p = 0
    if order == 0:
        syms, p = read_alphabet(b, 0)
        F = np.zeros(256, dtype=np.int64)
        for s in syms:
            F[s], p = vget(b, p)
        tot = int(F.sum())
        up = 0
        while tot and (tot << up) < 4096:
            up += 1
        core.update(shift=12, syms=syms, stored=F, up=up, freq=F << up, text=bytes(b[:p]), nested=None)
    else:
        shift = b[0] >> 4
        core.update(shift=shift, nested=None)
        if b[0] & 1:
            usz, q = vget(b, 1)
            csz, q = vget(b, q)
            inner = _trace_core(b[q:q + csz], 0, 4, usz)
            inner["data"] = core_decode(inner, usz)
            core["nested"] = inner
            text = bytes([b[0] & ~1]) + inner["data"]
            p = q + csz
        else:
            text = None
        t = text if text is not None else b
        syms, q = read_alphabet(t, 1)
        A = len(syms)
        stored = np.zeros((A, A), dtype=np.int64)
        for r in range(A):
            dz = 0
            for k in range(A):
                if dz:
                    dz -= 1
                    continue
                stored[r, k], q = vget(t, q)
                if stored[r, k] == 0:
                    dz = t[q]
                    q += 1
        ups = np.zeros(A, dtype=np.int64)
        for r in range(A):
            tot = int(stored[r].sum())
            while tot and (tot << int(ups[r])) < (1 << shift):
                ups[r] += 1
        if text is None:
            p = q
        core.update(syms=syms, stored=stored, up=ups, freq=stored << ups[:, None], text=bytes(b[:p]), text_plain=bytes(t[:q]))
    core["states"] = np.frombuffer(bytes(b[p:p + 4 * N]), dtype="<u4").astype(np.uint64)
    rest = bytes(b[p + 4 * N:])
    core["words"] = np.frombuffer(rest[:len(rest) & ~1], dtype="<u2")
    core["odd"] = rest[len(rest) & ~1:]
    return core


def trace(stream, U, decode=True):
    """Parse one stream (U = the length it decodes to; needed when NOSZ is set) into a dict:
    fmt, size (None when NOSZ), and then either stripe = dict(N, lens, parts=[trace of each part]) or
    pack = dict(syms, plen) | None, rle = dict(syms, nlit, meta_len, raw, core | None, meta) | None, cat, n (bytes the
    core stage decodes to), core (entropy core dict) | None, raw (the CAT bytes).  An entropy core holds order, N, shift,
    syms, stored (rows as stored), up (scale-up per row), freq (scaled), text (table bytes as written), nested (the
    traced order-0 coder of an order-1 table) | None, states, words; with decode, also data (what it decodes to)."""
    b = bytes(stream)
    fmt = b[0]
    t = dict(fmt=fmt, size=None, stripe=None, pack=None, rle=None, cat=False, core=None)
    p = 1
    if fmt & F_STRIPE:
        t["size"], p = vget(b, p)
        N = b[p]
        p += 1
        lens = []
        for _ in range(N):
            v, p = vget(b, p)
            lens.append(v)
        parts = []
        for k in range(N):
            uk = U // N + (U % N > k)
            parts.append(trace(b[p:p + lens[k]], uk, decode))
            p += lens[k]
        t["stripe"] = dict(N=N, lens=lens, parts=parts)
        t["end"] = p
        return t
    N = 32 if fmt & F_X32 else 4
    if not fmt & F_NOSZ:
        t["size"], p = vget(b, p)
        U = t["size"]
    n = U
    if fmt & F_PACK:
        ns = b[p] or 256
        syms = list(b[p + 1:p + 1 + ns])
        p += 1 + ns
        n, p = vget(b, p)
        t["pack"] = dict(syms=syms, plen=n)
    if fmt & F_RLE:
        um, p = vget(b, p)
        nlit, p = vget(b, p)
        r = dict(meta_len=um >> 1, nlit=nlit, raw=bool(um & 1), core=None)
        if um & 1:
            r["meta"] = b[p:p + (um >> 1)]
            p += um >> 1
        else:
            c, p = vget(b, p)
            r["core"] = _trace_core(b[p:p + c], 0, N, um >> 1)
            r["meta"] = core_decode(r["core"], um >> 1)
            r["core"]["data"] = r["meta"]
            p += c
        ns = r["meta"][0] or 256
        r["syms"] = list(r["meta"][1:1 + ns])
        t["rle"] = r
        n = nlit
    t["n"] = n
    if fmt & F_CAT:
        t["cat"] = True
        t["raw"] = b[p:p + n]
        t["end"] = p + n
        return t
    if n:
        t["core"] = _trace_core(b[p:], fmt & 1, N, n)
        if decode:
            t["core"]["data"] = core_decode(t["core"], n)
    t["end"] = len(b)
    return t


def cores(t, where=""):
    """Every entropy core of a trace, at any depth: [(where, core)]."""
    out = []
    if t.get("stripe"):
        for k, part in enumerate(t["stripe"]["parts"]):
            out += cores(part, "%sstripe[%d]." % (where, k))
        return out
    if t.get("rle") and t["rle"]["core"] is not None:
        out.append((where + "rle_meta", t["rle"]["core"]))
    if t.get("core") is not None:
        out.append((where + "core", t["core"]))
        if t["core"].get("nested") is not None:
            out.append((where + "core.table", t["core"]["nested"]))
    return out


# ---------------------------------------------------------------- transforms and containers
def pack(data):
    """hts_pack (pack.c:56-150): (symbols, packed bytes), or None over 16 symbols."""
    d = np.frombuffer(bytes(data), dtype=np.uint8)
    syms = np.flatnonzero(np.bincount(d, minlength=256))
    if len(syms) > 16:
        return None
    idx = np.zeros(256, dtype=np.uint8)
    idx[syms] = np.arange(len(syms))
    ns = len(syms)
    per = 2 if ns > 4 else 4 if ns > 2 else 8 if ns > 1 else 0
    if not per:
        return syms.tolist(), b""
    bits = 8 // per
    v = np.zeros(-(-len(d) // per) * per, dtype=np.uint32)
    v[:len(d)] = idx[d]
    v = v.reshape(-1, per) << (bits * np.arange(per, dtype=np.uint32))
    return syms.tolist(), v.sum(axis=1).astype(np.uint8).tobytes()


def rle(data):
    """rle_find_syms (rle.c:48-98) + hts_rle_encode (:100-140): (meta = [nsyms][symbols][run lengths], literals).  A
    symbol carries run lengths when more of its bytes repeat the previous byte than not; a byte is a literal unless it
    repeats the previous byte and is such a symbol."""
    d = np.frombuffer(bytes(data), dtype=np.uint8)
    n = len(d)
    rep = np.zeros(n, dtype=bool)
    rep[1:] = d[1:] == d[:-1]
    saved = np.bincount(d[rep], minlength=256) - np.bincount(d[~rep], minlength=256)
    inset = saved > 0
    syms = np.flatnonzero(inset)
    head = ~(inset[d] & rep)
    heads = np.flatnonzero(head)
    lit = d[heads].tobytes()
    nxt = np.append(heads[1:], n)
    runs = (nxt - heads - 1)[inset[d[heads]]]
    meta = bytearray([len(syms) & 0xff]) + bytes(syms.astype(np.uint8)) + b"".join(vput(int(r)) for r in runs)
    return bytes(meta), lit


def _core_or_fail(data, order, N):
    return core_encode(data, order, N)


def encode_flat(data, want):
    """rans_compress_to_4x16 without STRIPE as the kernel does it (encode_flat)."""
    U = len(data)
    if U <= 1000:
        want &= ~F_X32
    fmt = want & (F_ORDER | F_X32 | F_NOSZ | F_RLE | F_PACK)
    head = b"" if want & F_NOSZ else vput(U)
    if U == 0:
        return bytes([fmt & (F_ORDER | F_X32 | F_NOSZ)]) + head
    cur, n = bytes(data), U
    if fmt & F_PACK:
        pk = pack(cur)
        if pk is None:
            fmt &= ~F_PACK
        else:
            syms, cur = pk
            n = len(cur)
            head += bytes([len(syms)]) + bytes(syms) + vput(n)
            if (fmt & F_X32) and n < 32:
                fmt &= ~F_X32
    if (fmt & F_RLE) and n:
        meta, lit = rle(cur)
        rmeta, nlit = len(meta), len(lit)
        if nlit + rmeta >= 0.99 * n:                         # not worth it (rANS_static4x16pr.c:1467)
            fmt &= ~F_RLE
        else:
            if (fmt & F_X32) and (rmeta < 32 or nlit < 32):
                fmt &= ~F_X32
            c = core_encode(meta, 0, 32 if fmt & F_X32 else 4)
            if len(c) < rmeta:
                head += vput(rmeta * 2) + vput(nlit) + vput(len(c)) + c
            else:                                            # run lengths kept as they are: odd length field
                head += vput(rmeta * 2 + 1) + vput(nlit) + meta
            cur, n = lit, nlit
    else:
        fmt &= ~F_RLE
    order = fmt & F_ORDER
    if order and n < 8:
        fmt &= ~F_ORDER
        order = 0
    c = core_encode(cur, order, 32 if fmt & F_X32 else 4) if n else None
    if c is None or len(c) >= n:                             # CAT fallback (:1539-1553)
        fmt = (fmt & ~3) | F_CAT
        c = cur
    return bytes([fmt]) + head + c


def encode_stripe(data, want):
    """The STRIPE branch (encode_stripe): part j takes data[j::N]; each part keeps the strictly smallest of the
    methods (order 1, RLE, PACK, order 0, tried in that order) the flags admit."""
    U = len(data)
    N = (want >> 8) & 0xff or 4
    N = min(N, U)
    parts = []
    for j in range(N):
        part = bytes(data[j::N])
        best = None
        for m in (1, 64, 128, 0):
            if (want & m) != m or ((want & F_STRIPE_NO0) and not m & 1):
                continue
            c = encode_flat(part, m | F_NOSZ | (want & F_X32))
            if best is None or len(c) < len(best):
                best = c
        parts.append(best)
    return (bytes([want & 0xff & ~F_NOSZ]) + vput(U) + bytes([N]) + b"".join(vput(len(c)) for c in parts)
            + b"".join(parts))


def encode(data, flags):
    """The kernel's stream for data under flags (encode_stream)."""
    U = len(data)
    if U <= 1000:
        flags &= ~F_X32
    if U <= 20:
        flags &= ~F_STRIPE
    if flags & F_STRIPE:
        return encode_stripe(data, flags)
    if flags & F_CAT:
        return bytes([F_CAT]) + vput(U) + bytes(data)
    return encode_flat(data, flags & ~F_NOSZ)
