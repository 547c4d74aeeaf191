// The per-record rules of BAM index building, host/device portable: what sam_index (sam.c:994-1032) learns from one
// record through sam_read1 + bam_endpos + bgzf_tell, and what hts_idx_push (hts.c:2558-2640) makes of it before it
// compares the record with its predecessor.  bam_index.cu runs these one thread per record; a plain C++ build of this
// header gives the same answers on the CPU.
#pragma once
#include <stdint.h>

#ifdef __CUDACC__
#define BIDX_HD __host__ __device__ __forceinline__
#else
#define BIDX_HD inline
#endif

namespace bidx {

enum : int8_t { KEY_OK = 0, KEY_READ = 1, KEY_RANGE = 2 };

BIDX_HD uint32_t ld32(const uint8_t *p)
{
    return p[0] | (uint32_t)p[1] << 8 | (uint32_t)p[2] << 16 | (uint32_t)p[3] << 24;
}

// first bin number of level l: 1 + 8 + ... + 8^(l-1)
BIDX_HD uint32_t level_first(int l) { return ((1u << (3 * l)) - 1) / 7; }

// hts_reg2bin (hts.h:1516): the smallest bin that holds [beg, end), walking up from the bottom level
BIDX_HD uint32_t reg2bin(int64_t beg, int64_t end, int min_shift, int n_lvls)
{
    const int64_t last = end - 1;
    uint32_t first = level_first(n_lvls);
    int s = min_shift;
    for (int l = n_lvls; l > 0; --l, s += 3) {
        if ((beg >> s) == (last >> s)) return first + (uint32_t)(int32_t)(beg >> s);
        first -= 1u << (3 * (l - 1));
    }
    return 0;
}

// bytes an aux value of this type code takes after the code; 'Z'/'H'/'B' stand for themselves, 0 = unknown (aux_type2size)
BIDX_HD int aux_size(uint8_t t)
{
    switch (t) {
    case 'A': case 'c': case 'C': return 1;
    case 's': case 'S': return 2;
    case 'i': case 'I': case 'f': return 4;
    case 'd': return 8;
    case 'Z': case 'H': case 'B': return t;
    default: return 0;
    }
}

// skip_aux (sam.c:4793): s at a value's type code -> just past the value; end when s is already there; nullptr when the
// value is malformed.  The array bound is the 32-bit product the reference computes.
BIDX_HD const uint8_t *aux_skip(const uint8_t *s, const uint8_t *end)
{
    if (s >= end) return end;
    const int size = aux_size(*s++);
    if (size == 'Z' || size == 'H') {
        while (s < end && *s) s++;
        return s < end ? s + 1 : end;
    }
    if (size == 'B') {
        if (end - s < 5) return nullptr;
        const uint32_t es = (uint32_t)aux_size(*s++), n = ld32(s);
        s += 4;
        const uint32_t bytes = es * n;
        if (es == 0 || end - s < (int64_t)bytes) return nullptr;
        return s + bytes;
    }
    if (size == 0) return nullptr;
    return end - s < size ? nullptr : s + size;
}

// bam_aux_get(b, "CG") over [aux, end): 1 found (*val at its type code), 0 absent, -1 corrupt aux (sam.c:4819-4863)
BIDX_HD int aux_find_cg(const uint8_t *aux, const uint8_t *end, const uint8_t **val)
{
    if (end - aux <= 2) return 0;
    const uint8_t *s = aux + 2;
    for (;;) {
        if (s[-2] == 'C' && s[-1] == 'G') {
            const uint8_t *e = aux_skip(s, end);
            if (!e) return -1;
            if ((*s == 'Z' || *s == 'H') && e[-1] != 0) return -1;
            *val = s;
            return 1;
        }
        const uint8_t *next = aux_skip(s, end);
        if (!next) return -1;
        if (end - next <= 2) return 0;
        s = next + 2;
    }
}

// What the index takes from one record.
struct Key {
    int32_t tid;
    uint32_t bin;
    int64_t beg;        // the begin hts_idx_push compares with last_coor: pos, or -1 when unplaced
    int64_t coor;       // last_coor after the push: beg clamped at 0 for a placed record
    int64_t w0, w1;     // linear-index windows the record covers (placed records)
    uint8_t mapped;
    int8_t err;         // KEY_OK, KEY_READ (sam_read1 < -1), KEY_RANGE (hts_idx_check_range)
};

// One complete record: rec -> its block_size field, 4 + block_size bytes readable, block_size >= 32 (the chain walk
// checked both).  bam_read1's validity rules (sam.c:799-857) with the CG-tag CIGAR of bam_tag2cigar (:680-735),
// sam_read1's tid/mtid range (:4135), bam_endpos (:673-678), then hts_idx_push's clamps, range check and bin.
BIDX_HD Key record_key(const uint8_t *rec, int32_t n_targets, int min_shift, int n_lvls)
{
    Key k = {};
    const int32_t bl = (int32_t)ld32(rec);
    k.tid = (int32_t)ld32(rec + 4);
    const int64_t pos = (int32_t)ld32(rec + 8);
    const uint32_t qn = rec[12], x3 = ld32(rec + 16), flag = x3 >> 16;
    uint32_t n_cigar = x3 & 0xffffu;
    const int32_t lq = (int32_t)ld32(rec + 20), mtid = (int32_t)ld32(rec + 24);
    const uint32_t xn = (qn & 3) ? 4 - (qn & 3) : 0;
    const uint64_t l_data = (uint64_t)(uint32_t)(bl - 32) + xn;
    k.mapped = !(flag & 4);
    k.err = KEY_READ;
    if (lq < 0 || qn < 1) return k;
    if (((uint64_t)n_cigar << 2) + qn + xn + (((uint64_t)lq + 1) >> 1) + (uint64_t)lq > l_data) return k;
    if (rec[36 + qn - 1] != 0 && xn == 0 && l_data > 0x7fffffffull - 4) return k;        // fixup_missing_qname_nul
    const uint8_t *cig = rec + 36 + qn, *end = rec + 4 + (uint32_t)bl;
    if (n_cigar > 0 && ld32(cig) == (4u | ((uint32_t)lq << 4)) && k.tid >= 0 && pos >= 0) {
        const uint8_t *aux = cig + 4 * (uint64_t)n_cigar + (((uint64_t)lq + 1) >> 1) + (uint64_t)lq, *cg = nullptr;
        const int f = aux_find_cg(aux, end, &cg);
        if (f < 0) return k;
        if (f > 0 && cg[0] == 'B' && (cg[1] == 'I' || cg[1] == 'i')) {
            const uint32_t len = ld32(cg + 2);
            if (len >= n_cigar && len < (1u << 29)) { cig = cg + 6; n_cigar = len; }
        }
    }
    int64_t rlen = 0, qlen = 0;
    for (uint32_t i = 0; i < n_cigar; i++) {
        const uint32_t op = ld32(cig + 4 * (uint64_t)i), type = (0x3C1A7u >> ((op & 0xf) << 1)) & 3;
        if (type & 1) qlen += op >> 4;
        if (type & 2) rlen += op >> 4;
    }
    if (n_cigar > 0 && lq > 0 && k.mapped && qlen != lq) return k;
    if (k.tid >= n_targets || k.tid < -1 || mtid >= n_targets || mtid < -1) return k;
    k.err = KEY_OK;
    if (!k.mapped) rlen = 0;
    int64_t beg = pos, e = pos + (rlen ? rlen : 1);
    if (k.tid < 0) { beg = -1; e = 0; }
    k.beg = beg;
    const int64_t maxpos = (int64_t)1 << (min_shift + 3 * n_lvls);
    if (k.tid >= 0 && (beg > maxpos || e > maxpos)) { k.err = KEY_RANGE; return k; }
    if (k.tid >= 0) {
        if (beg < 0) beg = 0;
        if (e <= 0) e = 1;
        k.w0 = beg >> min_shift;
        k.w1 = (e - 1) >> min_shift;
    }
    k.coor = beg;
    k.bin = reg2bin(beg, e, min_shift, n_lvls);
    return k;
}

// One BGZF block of a window: [ustart, uend) of the inflated stream (relative to the window's origin), its file address
// and the address of the block that follows it in the file (the file length after the last one).
struct WinBlock {
    int64_t ustart, uend;
    uint64_t caddr, cnext;
};

// bgzf_tell once the bytes before stream position p (> 0) have been read: the block holding byte p-1 and the offset of p
// in it, or, when p is that block's end, the address of the very next block with offset 0, even if that block is empty
// (bgzf_read, bgzf.c:1282-1285).  blk[0..n) ascending; the caller guarantees a block with uend >= p exists.
BIDX_HD uint64_t voff_after(int64_t p, const WinBlock *blk, uint32_t n)
{
    uint32_t lo = 0, hi = n;
    while (lo < hi) {                                   // first block whose end reaches p: empty blocks before it end short of p
        const uint32_t mid = (lo + hi) >> 1;
        if (blk[mid].uend < p) lo = mid + 1; else hi = mid;
    }
    const WinBlock &b = blk[lo];
    return b.uend == p ? b.cnext << 16 : b.caddr << 16 | (uint64_t)(p - b.ustart);
}

} // namespace bidx
