"""The shape of the inflate work on a seeded synthetic BAM, modelled on the CPU (no GPU needed).

    python tools/inflate_shape.py [--blocks 40] [--quals novaseq|hiseq] [--level 6]

For each BGZF block it decodes the token stream with a plain Python inflater and prints: tokens, matches,
match batches (32 records); rounds and 32-word copy chunks for two schedules of the match records: batches of 32
run to completion (the kernel's exec_batch) and a rolling window of the 32 oldest pending records refilled every
round (DESIGN.md §6 has its measurement); a round executes every record whose sources are final; the overlapping matches
(dist < len) by distance and length, and the lane-parallel re-sync: the warp maximum of tokens a lane decodes
in round 0, in round 1 when it re-decodes its whole sub-range, and in round 1 when it stops where it meets
its round-0 path (the kernel's checkpoints)."""
import argparse
import bisect
import os
import sys
import zlib
from collections import Counter

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tools import synth  # noqa: E402

LB = [3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195, 227, 258]
LX = [0] * 8 + [1] * 4 + [2] * 4 + [3] * 4 + [4] * 4 + [5] * 4 + [0]
DB = [1, 2, 3, 4, 5, 7, 9, 13, 17, 25, 33, 49, 65, 97, 129, 193, 257, 385, 513, 769, 1025, 1537, 2049, 3073, 4097, 6145,
      8193, 12289, 16385, 24577]
DX = [0, 0, 0, 0] + [k // 2 for k in range(2, 28)]
PAR_MIN_BITS, LANES, RUN_MAX_DIST = 32 * 96, 32, 4


class Bits:
    def __init__(self, v, p=0):
        self.v, self.p = v, p

    def get(self, n):
        r = (self.v >> self.p) & ((1 << n) - 1)
        self.p += n
        return r


def table(lens):
    code, nxt, bl, t = 0, [0] * 16, Counter(l for l in lens if l), {}
    for b in range(1, 16):
        code = (code + bl[b - 1]) << 1
        nxt[b] = code
    for s, l in enumerate(lens):
        if l:
            t[(l, nxt[l])] = s
            nxt[l] += 1
    return t


def sym(br, t):
    c = 0
    for l in range(1, 16):
        c = (c << 1) | br.get(1)
        if (l, c) in t:
            return t[(l, c)]
    return None


def walk(v, start, end, lt, dt):
    """token boundaries from `start` while the position is below `end` (the kernel's lane_decode)"""
    br, pos = Bits(v, start), []
    while br.p < end:
        pos.append(br.p)
        s = sym(br, lt)
        if s is None or s > 285:
            break
        if s == 256:
            break
        if s > 256:
            br.get(LX[s - 257])
            d = sym(br, dt)
            if d is None or d > 29:
                break
            br.get(DX[d])
    return pos


def block_shape(raw):
    v, br, out, toks, bodies = int.from_bytes(raw, "little"), None, 0, [], []
    br = Bits(v)
    while True:
        final, kind = br.get(1), br.get(2)
        if kind == 0:
            br.p = (br.p + 7) // 8 * 8
            n = br.get(16); br.get(16); br.p += 8 * n; out += n
        else:
            if kind == 1:
                lt, dt = table([8] * 144 + [9] * 112 + [7] * 24 + [8] * 8), table([5] * 30)
            else:
                hl, hd, hc = br.get(5) + 257, br.get(5) + 1, br.get(4) + 4
                cl = [0] * 19
                for i in range(hc):
                    cl[[16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15][i]] = br.get(3)
                ct, L = table(cl), []
                while len(L) < hl + hd:
                    s = sym(br, ct)
                    L += [s] if s < 16 else [L[-1]] * (3 + br.get(2)) if s == 16 else [0] * (3 + br.get(3)) if s == 17 else [0] * (11 + br.get(7))
                lt, dt = table(L[:hl]), table(L[hl:])
            bodies.append((br.p, lt, dt))
            while True:
                s = sym(br, lt)
                if s < 256:
                    toks.append((out, 0, 0)); out += 1
                elif s == 256:
                    break
                else:
                    ln = LB[s - 257] + br.get(LX[s - 257]); d = sym(br, dt); di = DB[d] + br.get(DX[d])
                    toks.append((out, ln, di)); out += ln
        if final:
            return v, len(raw) * 8 + 64, toks, bodies          # the kernel's input end includes the 8-byte footer


def deps(ms):
    """per match, the index range [a, b) of the earlier matches whose destination overlaps its source"""
    ds, es = [m[0] for m in ms], [m[0] + m[1] for m in ms]
    out = []
    for d, ln, di in ms:
        s, e = d - di, d if di < ln else d - di + ln
        out.append((bisect.bisect_right(es, s), bisect.bisect_left(ds, e)))
    return out


def words(m):
    """destination words of a match in the round's word copy (output aligned to 4 bytes); long-period runs take none"""
    d, ln, di = m
    return 0 if RUN_MAX_DIST < di < ln else (d + ln + 3) // 4 - d // 4


def rounds(ms):
    """batches of 32 records, each run to completion: (rounds, 32-word copy chunks)"""
    dep, rs, ch = deps(ms), 0, 0
    for i in range(0, len(ms), 32):
        lvl = {}
        for j in range(i, min(i + 32, len(ms))):
            a, b = dep[j]
            lvl[j] = 1 + max([lvl[q] for q in range(max(a, i), b)], default=0)
        for r in range(1, max(lvl.values()) + 1):
            ch += -(-sum(words(ms[j]) for j, v in lvl.items() if v == r) // 32)
        rs += max(lvl.values())
    return rs, ch


def window_rounds(ms, W=32):
    """rolling window of the W oldest pending records, refilled every round: (rounds, 32-word copy chunks)"""
    dep, done, pend, rs, ch = deps(ms), [False] * len(ms), list(range(len(ms))), 0, 0
    while pend:
        ready = [j for j in pend[:W] if all(done[q] for q in range(*dep[j]))]
        for j in ready:
            done[j] = True
        ch += -(-sum(words(ms[j]) for j in ready) // 32)
        pend = [j for j in pend if not done[j]]
        rs += 1
    return rs, ch


def resync(v, total, body, lt, dt):
    """warp maxima of tokens per lane: round 0, round 1 re-decoding the whole sub-range, round 1 stopping on round 0's path"""
    true = set(walk(v, body, total, lt, dt))
    S = (total - body + 31) // 32
    r0, full, conv = [], [], []
    for i in range(LANES):
        st, en = min(total, body + i * S), min(total, body + (i + 1) * S) if i < 31 else total
        p0 = walk(v, st, en, lt, dt)
        r0.append(len(p0))
        if i == 0:
            continue
        p1 = walk(v, min(p for p in true if p >= st) if any(p >= st for p in true) else en, en, lt, dt)
        full.append(len(p1))
        meet = next((k for k, p in enumerate(p1) if p in set(p0)), len(p1))
        conv.append(meet)
    return max(r0), max(full), max(conv)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--blocks", type=int, default=40)
    ap.add_argument("--quals", default="novaseq")
    ap.add_argument("--level", type=int, default=6)
    args = ap.parse_args()
    c = synth.bam_bgzf_corpus(3e6, level=args.level, quals=args.quals, procs=1)
    comp, clen = c["comp"], c["clen"]
    off, rows, ov = 0, [], []
    print("block tokens matches batches rounds chunks window_rounds window_chunks overlapping resync_r0 resync_r1_full resync_r1_converged")
    for k in range(min(args.blocks, len(clen))):
        blk = bytes(comp[off:off + int(clen[k])]); off += int(clen[k])
        v, total, toks, bodies = block_shape(blk[18:-8])
        ms = [t for t in toks if t[1]]
        o = [m for m in ms if m[2] < m[1]]
        ov += o
        body, lt, dt = bodies[0]
        rs = resync(v, total, body, lt, dt) if total - body >= PAR_MIN_BITS else (0, 0, 0)
        rows.append((len(toks), len(ms), (len(ms) + 31) // 32) + rounds(ms) + window_rounds(ms) + (len(o),) + rs)
        print(k, *rows[-1])
    a = np.array(rows, dtype=np.float64).mean(axis=0)
    print("mean", " ".join("%.1f" % x for x in a))
    D, L = Counter(m[2] for m in ov), [m[1] for m in ov]
    print("overlapping by distance:", dict(sorted(D.items())[:12]), "| dist <= 4: %.3f, dist <= 32: %.3f" %
          (sum(n for d, n in D.items() if d <= 4) / max(1, len(ov)), sum(n for d, n in D.items() if d <= 32) / max(1, len(ov))))
    print("overlapping lengths: mean %.1f, percentiles 50/90/99:" % (np.mean(L) if L else 0), np.percentile(L, [50, 90, 99]) if L else [])


if __name__ == "__main__":
    main()
