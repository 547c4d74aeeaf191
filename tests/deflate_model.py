"""Plain references for the BGZF deflate kernel (bgzf_deflate_kernel, DESIGN §4.2c), no GPU.

- huffman_opt: Huffman's algorithm on a heap -> the unconstrained optimal cost sum(freq * len) and depth.
- package_merge: the optimal cost of a prefix code whose lengths are at most `limit` (Larmore-Hirschberg).
- pass2: the kernel's second pass restated from DESIGN §4.2c and RFC 1951 §3.2.5-3.2.7: from an LZ77 token list,
  the payload and the level to the complete BGZF block the kernel writes.  Pass 2 is a deterministic function of the
  tokens, so this is exact; the tokens themselves come from tracing the kernel's output (orc_inflate_trace).

A token is a literal byte (int) or a (length, distance) tuple."""
import heapq
import random
import struct
import zlib

LEN_BASE = [3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195, 227, 258]
LEN_XTRA = [0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 2, 2, 3, 3, 3, 3, 4, 4, 4, 4, 5, 5, 5, 5, 0]
DST_BASE = [1, 2, 3, 4, 5, 7, 9, 13, 17, 25, 33, 49, 65, 97, 129, 193, 257, 385, 513, 769, 1025, 1537, 2049, 3073, 4097,
            6145, 8193, 12289, 16385, 24577]
DST_XTRA = [0, 0, 0, 0, 1, 1, 2, 2, 3, 3, 4, 4, 5, 5, 6, 6, 7, 7, 8, 8, 9, 9, 10, 10, 11, 11, 12, 12, 13, 13]
CL_ORDER = [16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15]
CL_XTRA = {16: 2, 17: 3, 18: 7}
FIXED_LL = [8] * 144 + [9] * 112 + [7] * 24 + [8] * 8
BGZF_HDR = b"\x1f\x8b\x08\x04\0\0\0\0\0\xff\x06\0BC\x02\0"
MAX_PAYLOAD = 65280                       # 0xff00, BGZF_BLOCK_SIZE
SLOT = 65536
LIMIT_BITS = (SLOT - 8 - 4) * 8           # the token stream must end before this absolute bit: room for EOB + footer


def len_sym(length):
    s = 28
    while LEN_BASE[s] > length:
        s -= 1
    return s


def dist_sym(dist):
    s = 29
    while DST_BASE[s] > dist:
        s -= 1
    return s


# ---------------------------------------------------------------- optimal prefix codes
def huffman_opt(freqs):
    """(cost, depth) of an optimal unconstrained prefix code for the nonzero freqs.  One symbol -> (freq, 1)."""
    w = [f for f in freqs if f]
    if not w:
        return 0, 0
    if len(w) == 1:
        return w[0], 1
    heap = [(f, 0, i) for i, f in enumerate(w)]          # (weight, height, tie-break)
    heapq.heapify(heap)
    cost, k = 0, len(w)
    while len(heap) > 1:
        a, ha, _ = heapq.heappop(heap)
        b, hb, _ = heapq.heappop(heap)
        cost += a + b
        heapq.heappush(heap, (a + b, max(ha, hb) + 1, k))
        k += 1
    return cost, heap[0][1]


def package_merge(freqs, limit):
    """Optimal cost sum(freq * len) over complete prefix codes with every length <= limit (nonzero freqs only)."""
    w = sorted(f for f in freqs if f)
    n = len(w)
    if n == 0:
        return 0
    if n == 1:
        return w[0]
    assert n <= 1 << limit, "no code of %d symbols fits %d bits" % (n, limit)
    # the row of the deepest level holds the leaves; each level up packages the row below in pairs and merges the leaves
    # back in.  The cost is the total weight of the 2n-2 cheapest items of the top row.
    items = list(w)
    for _ in range(limit - 1):
        items = sorted(w + [items[i] + items[i + 1] for i in range(0, len(items) - 1, 2)])
    return sum(items[:2 * n - 2])


def code_cost(freqs, lens):
    return sum(f * l for f, l in zip(freqs, lens))


def kraft(lens, limit=15):
    """Kraft sum in units of 2^-limit; a complete code gives 1 << limit."""
    return sum(1 << (limit - l) for l in lens if l)


# ---------------------------------------------------------------- the kernel's length construction
def build_lengths(freq, max_bits):
    """Code lengths for freq (0 = unused), as DESIGN §4.2c builds them: used symbols sorted by count with a stable sort
    (ties in symbol order), Huffman's two-queue merge on the sorted leaves with a leaf taken before an internal node of the
    same weight, leaf depths counted per length class, classes deeper than max_bits clamped and then folded (each step
    drops one max_bits code and splits the deepest shorter code into two one bit longer, until the Kraft sum is exact),
    lengths handed out shortest first from the most frequent symbol.  A lone used symbol gets length 1."""
    n = len(freq)
    lens = [0] * n
    order = sorted((i for i in range(n) if freq[i]), key=lambda i: freq[i])
    used = len(order)
    if used == 0:
        return lens
    if used == 1:
        lens[order[0]] = 1
        return lens
    leaves = [freq[i] for i in order]
    # nodes: leaves 0..used-1, internal nodes appended; parent links give the depths
    weight = list(leaves)
    parent = [None] * used
    li, ii = 0, used
    for _ in range(used - 1):
        pick = []
        for _ in range(2):
            if li < used and (ii >= len(weight) or weight[li] <= weight[ii]):
                pick.append(li); li += 1
            else:
                pick.append(ii); ii += 1
        weight.append(weight[pick[0]] + weight[pick[1]])
        parent.append(None)
        parent[pick[0]] = parent[pick[1]] = len(weight) - 1
    depth = [0] * len(weight)
    for i in range(len(weight) - 2, -1, -1):
        depth[i] = depth[parent[i]] + 1
    cnt = [0] * (max_bits + 1)
    for i in range(used):
        cnt[min(depth[i], max_bits)] += 1
    total = sum(cnt[l] << (max_bits - l) for l in range(1, max_bits + 1))
    while total > 1 << max_bits:
        cnt[max_bits] -= 1
        for l in range(max_bits - 1, 0, -1):
            if cnt[l]:
                cnt[l] -= 1
                cnt[l + 1] += 2
                break
        total -= 1
    k = used - 1
    for l in range(1, max_bits + 1):
        for _ in range(cnt[l]):
            lens[order[k]] = l
            k -= 1
    return lens


def canonical_codes(lens):
    """RFC 1951 §3.2.2 canonical codes (MSB-first values)."""
    mx = max(lens) if lens else 0
    bl = [0] * (mx + 2)
    for l in lens:
        if l:
            bl[l] += 1
    nxt, c = [0] * (mx + 2), 0
    for b in range(1, mx + 1):
        c = (c + bl[b - 1]) << 1
        nxt[b] = c
    codes = [0] * len(lens)
    for i, l in enumerate(lens):
        if l:
            codes[i] = nxt[l]
            nxt[l] += 1
    return codes


def rle_lengths(seq):
    """The code-length sequence as (symbol, extra value) pairs: 18 for zero runs of 11..138, 17 for zero runs of 3..10,
    a length then 16 for each further 3..6 repeats of it, everything shorter sent as itself (RFC 1951 §3.2.7)."""
    out, i = [], 0
    while i < len(seq):
        v, run = seq[i], 1
        while i + run < len(seq) and seq[i + run] == v:
            run += 1
        i += run
        if v == 0:
            while run >= 11:
                r = min(run, 138)
                out.append((18, r - 11)); run -= r
            if run >= 3:
                out.append((17, run - 3)); run = 0
        else:
            out.append((v, 0)); run -= 1
            while run >= 3:
                r = min(run, 6)
                out.append((16, r - 3)); run -= r
        out += [(v, 0)] * run
    return out


class BitWriter:
    def __init__(self):
        self.buf, self.acc, self.nacc, self.n = bytearray(), 0, 0, 0

    def put(self, v, nb):
        """nb bits of v, LSB first."""
        self.acc |= (v & ((1 << nb) - 1)) << self.nacc
        self.nacc += nb
        self.n += nb
        while self.nacc >= 8:
            self.buf.append(self.acc & 0xff)
            self.acc >>= 8
            self.nacc -= 8

    def put_code(self, code, nb):
        """a Huffman code, MSB first."""
        self.put(int(format(code, "0%db" % nb)[::-1], 2) if nb else 0, nb)

    def bytes(self):
        return bytes(self.buf) + (bytes([self.acc]) if self.nacc else b"")


def stored_block(payload):
    n = len(payload)
    return bgzf_wrap(b"\x01" + struct.pack("<HH", n, n ^ 0xffff) + payload, payload)


def bgzf_wrap(deflate, payload):
    total = 18 + len(deflate) + 8
    return BGZF_HDR + struct.pack("<H", total - 1) + deflate + struct.pack("<II", zlib.crc32(payload) & 0xffffffff, len(payload))


def pass2(tokens, payload, level):
    """The BGZF block the kernel writes for these tokens, and a dict saying how it got there:
    kind ('stored' / 'fixed' / 'dynamic'), why a block went stored ('level0', 'short', 'limit', 'size'), the fixed and
    dynamic bit counts, the three length tables, the code-length histogram and HLIT / HDIST / HCLEN."""
    n = len(payload)
    info = dict(kind="stored", why=None)
    if level == 0 or n < 16:
        info["why"] = "level0" if level == 0 else "short"
        return stored_block(payload), info
    freq = [0] * 286
    dfreq = [0] * 30
    xbits = 0
    for t in tokens:
        if isinstance(t, int):
            freq[t] += 1
        else:
            ls, ds = len_sym(t[0]), dist_sym(t[1])
            freq[257 + ls] += 1
            dfreq[ds] += 1
            xbits += LEN_XTRA[ls] + DST_XTRA[ds]
    freq[256] = 1                                          # end of block
    fixed_bits = 3 + xbits + code_cost(freq, FIXED_LL) + 5 * sum(dfreq)
    ll = build_lengths(freq, 15)
    dl = build_lengths(dfreq, 15)
    if not any(dl):
        dl[0] = 1                                          # one distance code of one bit, used by no token
    hlit = max([257] + [i + 1 for i in range(257, 286) if ll[i]])
    hdist = max([1] + [i + 1 for i in range(1, 30) if dl[i]])
    seq = rle_lengths(ll[:hlit] + dl[:hdist])
    clf = [0] * 19
    for s, _ in seq:
        clf[s] += 1
    cl = build_lengths(clf, 7)
    if sum(1 for l in cl if l) == 1:                       # a complete code-length code needs two codes
        cl[1 if cl[0] else 0] = 1
    hclen = max([4] + [k + 1 for k in range(4, 19) if cl[CL_ORDER[k]]])
    dyn_bits = (3 + 14 + 3 * hclen + sum(clf[s] * (cl[s] + CL_XTRA.get(s, 0)) for s in range(19))
                + code_cost(freq, ll) + code_cost(dfreq, dl) + xbits)
    use_dyn = dyn_bits < fixed_bits
    info.update(fixed_bits=fixed_bits, dyn_bits=dyn_bits, ll=ll, dist=dl, cl=cl, freq=freq, dfreq=dfreq, clf=clf,
                hlit=hlit, hdist=hdist, hclen=hclen, seq=seq)
    w = BitWriter()
    if use_dyn:
        lc, dc, cc = canonical_codes(ll), canonical_codes(dl), canonical_codes(cl)
        w.put(1, 1); w.put(2, 2)
        w.put(hlit - 257, 5); w.put(hdist - 1, 5); w.put(hclen - 4, 4)
        for k in range(hclen):
            w.put(cl[CL_ORDER[k]], 3)
        for s, x in seq:
            w.put_code(cc[s], cl[s])
            if s in CL_XTRA:
                w.put(x, CL_XTRA[s])
        lit_lens, dist_lens = ll, dl
    else:
        lc, dc = canonical_codes(FIXED_LL), list(range(30))      # fixed distance codes: the 5-bit symbol itself
        w.put(1, 1); w.put(1, 2)
        lit_lens, dist_lens = FIXED_LL, [5] * 30
    for t in tokens:
        if isinstance(t, int):
            w.put_code(lc[t], lit_lens[t])
        else:
            ls, ds = len_sym(t[0]), dist_sym(t[1])
            w.put_code(lc[257 + ls], lit_lens[257 + ls]); w.put(t[0] - LEN_BASE[ls], LEN_XTRA[ls])
            w.put_code(dc[ds], dist_lens[ds]); w.put(t[1] - DST_BASE[ds], DST_XTRA[ds])
    if 18 * 8 + w.n > LIMIT_BITS:
        info["why"] = "limit"
        return stored_block(payload), info
    w.put_code(lc[256], lit_lens[256])
    info["dlen"] = (w.n + 7) // 8
    if info["dlen"] >= n + 5:
        info["why"] = "size"
        return stored_block(payload), info
    info["kind"] = "dynamic" if use_dyn else "fixed"
    return bgzf_wrap(w.bytes(), payload), info


# ---------------------------------------------------------------- seeded inputs that reach the kernel's edges
def kernel_hash(buf, q):
    """The kernel's 12-bit hash of the 4 bytes at q (multiplicative, 2654435761)."""
    return ((int.from_bytes(buf[q:q + 4], "little") * 2654435761) & 0xffffffff) >> 20


def hash_survives(buf, src, p):
    """True when no other position that the kernel hashes between src's 32-byte step and p shares src's hash: the
    table then still points at src when the lane at p looks (no overwrite, no two lanes of one step storing alike)."""
    h = kernel_hash(buf, src)
    return not any(kernel_hash(buf, q) == h for q in range(src - src % 32, min(p, len(buf) - 3)) if q != src)


def literal_only(rng, counts):
    """Bytes holding counts[b] copies of each byte b in which no 4-byte string occurs twice and no byte three times in a
    row.  Neither of the kernel's match candidates can then fire (a hash match needs 4 equal bytes at some distance, a
    distance-1 match a byte four times in a row), so its tokens are exactly the literals and pass2 predicts the block."""
    seq = [b for b in range(256) for _ in range(counts[b])]
    rng.shuffle(seq)
    seen = set()
    for i in range(len(seq)):
        for _ in range(2000):
            if not (i >= 2 and seq[i] == seq[i - 1] == seq[i - 2]) and (i < 3 or tuple(seq[i - 3:i + 1]) not in seen):
                break
            j = rng.randrange(i, len(seq))
            seq[i], seq[j] = seq[j], seq[i]
        else:
            raise ValueError("no literal-only arrangement found")
        if i >= 3:
            seen.add(tuple(seq[i - 3:i + 1]))
    return bytes(seq)


def ll_fold_payload():
    """Literal-only: 13 bytes with Fibonacci counts 1, 2, 3, 5 .. 377 (EOB is the chain's other 1) under 128 bytes of
    count 300.  The lit/len Huffman tree is a 13-level chain under about 5 levels of bulk: 18 deep, folded to 15."""
    rng = random.Random(15)
    fib = [1, 1]
    while len(fib) < 14:
        fib.append(fib[-1] + fib[-2])
    syms = list(range(256))
    rng.shuffle(syms)
    counts = [0] * 256
    for s, c in zip(syms, fib[1:] + [300] * 128):
        counts[s] = c
    return literal_only(rng, counts)


def cl_fold_payload():
    """Literal-only with a frozen heavy-tailed byte histogram (seed 2370 of an offline search with pass2) whose
    code-length sequence needs a code-length code deeper than 7 bits."""
    rng = random.Random(2370)
    a, b = rng.uniform(4, 14), rng.uniform(0.5, 3)
    counts = [int(2 ** (a * rng.random() ** b)) for _ in range(256)]
    return literal_only(random.Random(7), counts)


def incompressible_payload():
    """65280 literal-only bytes, each byte value 255 times: no code beats 8 bits a byte, so the block goes stored."""
    return literal_only(random.Random(65280), [255] * 256)


def random_counts(rng, n, k):
    syms = rng.sample(range(256), k)
    counts = [0] * 256
    for _ in range(n):
        counts[syms[min(int(rng.expovariate(1.0) * k / 3), k - 1)]] += 1
    return counts


def literal_search(pred, tries=20000):
    """The first seeded literal-only payload (16..400 bytes) whose pass2 result satisfies pred(payload, info)."""
    for seed in range(tries):
        rng = random.Random(seed)
        n = rng.randint(16, 400)
        try:
            p = literal_only(rng, random_counts(rng, n, rng.randint(8, 200)))
        except ValueError:
            continue
        blk, info = pass2(list(p), p, 6)
        if pred(p, info):
            return p
    raise AssertionError("no payload found")


def planted_copy(seed, src_len, copy_len, dist, zeros=64):
    """zeros + SRC (src_len random bytes) + zeros + 4 guard bytes + SRC[:copy_len] + 4 tail bytes, with the copy
    dist bytes after SRC and the byte after the copy differing from the byte after SRC[:copy_len].  Zero filler
    hashes to one bucket, so the table still points at SRC when the copy is reached; the seed is advanced until that
    holds for the kernel's hash."""
    while True:
        rng = random.Random(seed)
        src = bytes(rng.randrange(1, 256) for _ in range(src_len))
        guard = bytes(rng.randrange(1, 256) for _ in range(4))
        after = src[copy_len] if copy_len < src_len else 0
        tail = bytes([(after + 1 + rng.randrange(254)) % 256 or 1]) + bytes(rng.randrange(256) for _ in range(3))
        buf = b"\0" * zeros + src + b"\0" * (dist - src_len - 4) + guard + src[:copy_len] + tail
        p = zeros + dist
        if buf[p - 1] != src[0] and hash_survives(buf, zeros, p):
            return buf, zeros, p
        seed += 1000


def dist_fold_payload(seed=4):
    """Random filler with copies of 4-5 bytes planted at distances whose codes 3..19 (4..1024 bytes) get the counts of a
    Huffman chain (each count 3 % + 2 over the sum of all but the previous one), the rarest at the shortest distance:
    a 17-level chain, 16 deep.  A copy is kept only where hash_survives says the kernel's table still points at its
    source when the lane at the copy looks, and turned back into filler otherwise; a copy closer than 32 bytes starts
    where its source lies in the previous 32-byte step.  A stray match or two still joins the chain; the seed is one
    whose whole parse, strays included, stays deeper than 15.  Returns (payload, planted {code: count})."""
    rng = random.Random(seed)
    codes = list(range(3, 20))
    want = [1, 1]
    while len(want) < len(codes):
        want.append(sum(want[:-1]) * 103 // 100 + 2)
    left = dict(zip(codes, want))
    out = bytearray(rng.randrange(256) for _ in range(1100))
    while any(left.values()):
        c = rng.choices(codes, weights=[left[k] for k in codes])[0]
        out += bytes(rng.randrange(256) for _ in range(rng.randint(1, 2)))
        d = DST_BASE[c] + rng.randrange(1 << DST_XTRA[c])
        while d < 32 and len(out) % 32 >= d:
            out.append(rng.randrange(256))
        p = len(out)
        for k in range(rng.randint(4, 5)):
            out.append(out[p - d + k])
        if hash_survives(out, p - d, p):
            left[c] -= 1
        else:                                      # the kernel may or may not see this one: make it filler
            out[p:] = bytes(rng.randrange(256) for _ in range(len(out) - p))
        assert len(out) < MAX_PAYLOAD - 16, "planted copies do not fit one block"
    out += bytes(rng.randrange(256) for _ in range(4))
    return bytes(out), dict(zip(codes, want))
