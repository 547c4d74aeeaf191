// CRAM 3.x record ENCODE: bam1_t records -> the data series of a slice (the record loop of cram_encode_slice /
// process_one_read, cram/cram_encode.c:2050-2420, :3490-4010, in the shape the reference writes with no_ref: every base and
// quality explicit, CIGAR as read features, mates detached).
//
// Encoding is parallel where decoding is serial: a record's bytes in every series depend on that record alone, only
// their POSITION depends on the records before it.  So: one thread per record counts what it contributes to each of the
// 30 byte streams (walk<false>), a scan per (slice, stream) turns counts into offsets, one thread per record writes
// (walk<true>).  Same source for both passes, __host__ __device__ (tests/hostsim builds it for the host).
//
// Series layout (all EXTERNAL, ITF8 integers; content id = stream index + 1):
//   BF CF RI RL AP RG | RN (BYTE_ARRAY_STOP 0) | MF NS NP TS | TL | FN, per feature FC FP and DL / RS / HC / PD or
//   BB / SC / IN (BYTE_ARRAY_LEN: length stream + value stream) | BA (unmapped reads) | QS | MQ |
//   tags: every tag value BYTE_ARRAY_LEN over two shared streams (lengths, values), in tag-line order; with tag blocks
//   each tag key is a stream of its own after S_COUNT (see tag_rules / TagRec below).
//   NF (mate distance, only with mate attachment) comes last, content id 32, so the layout without it is unchanged.
// By default every record is written detached (MF NS NP TS explicit, no mate cross references to resolve).  With mate
// attachment the pairing pass below decides per record, as process_one_read does, which reads of a name are attached:
// the earlier read gets MATE_DOWNSTREAM and NF, neither stores MF NS NP TS, the decoder rebuilds them.  RG stays an
// ordinary aux tag (RG series = -1), AP is absolute, RI is per record (multi-reference slice, ref_seq_id -2) and RR = 0
// (no reference needed to decode).  What the reference's decoder returns for such a slice is the input record, except
// what CRAM cannot hold: '=' / 'X' CIGAR ops come back as 'M', the mapping quality of an unmapped read as 0.
#pragma once
#include <stdint.h>
#include <stddef.h>

#ifndef CRAMREC_HD
#ifdef __CUDACC__
#define CRAMREC_HD __host__ __device__
#else
#define CRAMREC_HD
#endif
#endif

namespace cramenc {

enum Stream { S_BF, S_CF, S_RI, S_RL, S_AP, S_RG, S_RN, S_MF, S_NS, S_NP, S_TS, S_TL, S_FN, S_FC, S_FP, S_DL, S_RS, S_HC, S_PD,
              S_BB_LEN, S_BB, S_SC_LEN, S_SC, S_IN_LEN, S_IN, S_BA, S_QS, S_MQ, S_TAG_LEN, S_TAG_VAL, S_BS, S_NF, S_COUNT };

struct Core { int64_t pos; int32_t tid; uint16_t bin; uint8_t qual, l_extranul; uint16_t flag, l_qname; uint32_t n_cigar; int32_t l_qseq, mtid; int64_t mpos, isize; };

enum { ENC_OK = 0, ENC_UNSUPPORTED = -6, ENC_BAD = -1 };

CRAMREC_HD inline int itf8_size(uint32_t v) { return v < 0x80 ? 1 : v < 0x4000 ? 2 : v < 0x200000 ? 3 : v < 0x10000000 ? 4 : 5; }
CRAMREC_HD inline int itf8_put(uint8_t *p, uint32_t v)                    // itf8_put, cram/cram_io.h
{
    if (v < 0x80) { p[0] = (uint8_t)v; return 1; }
    if (v < 0x4000) { p[0] = (uint8_t)((v >> 8) | 0x80); p[1] = (uint8_t)v; return 2; }
    if (v < 0x200000) { p[0] = (uint8_t)((v >> 16) | 0xc0); p[1] = (uint8_t)(v >> 8); p[2] = (uint8_t)v; return 3; }
    if (v < 0x10000000) { p[0] = (uint8_t)((v >> 24) | 0xe0); p[1] = (uint8_t)(v >> 16); p[2] = (uint8_t)(v >> 8); p[3] = (uint8_t)v; return 4; }
    p[0] = (uint8_t)(0xf0 | ((v >> 28) & 0xff)); p[1] = (uint8_t)(v >> 20); p[2] = (uint8_t)(v >> 12); p[3] = (uint8_t)(v >> 4); p[4] = (uint8_t)(v & 0x0f);
    return 5;
}

// one aux field at p: tag[2], type, value length (bytes after the 3-byte id).  Returns false on a malformed field.
CRAMREC_HD inline bool aux_field(const uint8_t *p, const uint8_t *end, uint32_t &vlen)
{
    if (end - p < 3) return false;
    const uint8_t t = p[2];
    const uint8_t *v = p + 3;
    switch (t) {
    case 'A': case 'c': case 'C': vlen = 1; break;
    case 's': case 'S': vlen = 2; break;
    case 'i': case 'I': case 'f': vlen = 4; break;
    case 'd': vlen = 8; break;
    case 'Z': case 'H': { const uint8_t *q = v; while (q < end && *q) q++; if (q >= end) return false; vlen = (uint32_t)(q - v) + 1; break; }
    case 'B': {
        if (end - v < 5) return false;
        const uint8_t st = v[0];
        const uint32_t n = v[1] | v[2] << 8 | v[3] << 16 | (uint32_t)v[4] << 24;
        const uint32_t es = (st == 'c' || st == 'C') ? 1 : (st == 's' || st == 'S') ? 2 : (st == 'i' || st == 'I' || st == 'f') ? 4 : 0;
        if (!es || n > 0x10000000u) return false;
        vlen = 5 + n * es;
        break; }
    default: return false;
    }
    return (uint64_t)(end - v) >= vlen;
}

// WRITE = false: cnt[s] += bytes this record adds to stream s.  WRITE = true: the bytes go to base[s] + off[s] (off advances).
// Streams s >= S_COUNT are the per-tag-key streams of HGPU_CRAM_ENC_TAG_BLOCKS: their counts / offsets stay in the
// global count array (x[(s - S_COUNT) * xs], this record's column) and their bytes go to xarena + xbase[s - S_COUNT].
template <bool WRITE>
struct Emit {
    uint32_t *n;                     // counts or running offsets, S_COUNT entries
    uint8_t *const *base;
    uint32_t *x = nullptr;           // tag-key streams (nullptr: none)
    size_t xs = 0;
    uint8_t *xarena = nullptr;
    const uint64_t *xbase = nullptr;
    CRAMREC_HD uint32_t &at(int s) { return s < S_COUNT ? n[s] : x[(size_t)(s - S_COUNT) * xs]; }
    CRAMREC_HD uint8_t *dst(int s) { return s < S_COUNT ? base[s] + n[s] : xarena + xbase[s - S_COUNT] + x[(size_t)(s - S_COUNT) * xs]; }
    CRAMREC_HD void put_int(int s, int32_t v)
    {
        if (WRITE) at(s) += (uint32_t)itf8_put(dst(s), (uint32_t)v);
        else at(s) += (uint32_t)itf8_size((uint32_t)v);
    }
    CRAMREC_HD void put_byte(int s, uint8_t b) { if (WRITE) *dst(s) = b; at(s) += 1; }
    CRAMREC_HD void put_bytes(int s, const uint8_t *p, uint32_t len) { if (WRITE) { uint8_t *d = dst(s); for (uint32_t i = 0; i < len; i++) d[i] = p[i]; } at(s) += len; }
    CRAMREC_HD void put_fill(int s, uint8_t b, uint32_t len) { if (WRITE) for (uint32_t i = 0; i < len; i++) base[s][n[s] + i] = b; n[s] += len; }
    CRAMREC_HD void put_bases(int s, const uint8_t *seq4, uint32_t from, uint32_t len)          // 4-bit SEQ -> ASCII
    {
        if (WRITE) for (uint32_t i = 0; i < len; i++) { const uint32_t q = from + i; base[s][n[s] + i] = (uint8_t)"=ACMGRSVTWYHKDBN"[(seq4[q >> 1] >> ((~q & 1) << 2)) & 15]; }
        n[s] += len;
    }
};

CRAMREC_HD inline uint8_t base_at(const uint8_t *seq4, uint32_t q) { return (uint8_t)"=ACMGRSVTWYHKDBN"[(seq4[q >> 1] >> ((~q & 1) << 2)) & 15]; }
CRAMREC_HD inline int l1_row(uint8_t c) { return c == 'A' ? 0 : c == 'C' ? 1 : c == 'G' ? 2 : c == 'T' ? 3 : 4; }
// substitution code of read base sb against reference base rb under the default matrix (rows CGTN AGTN ACTN ACGN ACGT): -1 = not expressible
CRAMREC_HD inline int bs_code(uint8_t rb, uint8_t sb)
{
    const char *row = l1_row(rb) == 0 ? "CGTN" : l1_row(rb) == 1 ? "AGTN" : l1_row(rb) == 2 ? "ACTN" : l1_row(rb) == 3 ? "ACGN" : "ACGT";
    for (int k = 0; k < 4; k++) if ((uint8_t)row[k] == sb) return k;
    return -1;
}

// CIGAR (+ SEQ, + reference) -> read features.  EMIT = false only counts them (FN is written before the features).
// ref != nullptr: match operations are compared with the reference (ref[0] = base 1 of the record's reference sequence):
// equal bases leave no feature, a different A/C/G/T/N is a substitution 'X' (BS = its code in the reference base's row),
// anything else a one-base 'b'.  ref == nullptr: every match operation is a 'b' run with its bases.
template <bool WRITE, bool EMIT>
CRAMREC_HD inline int features(const Core &c, const uint8_t *cig, uint32_t nc, const uint8_t *seq4, int32_t ls, bool noseq,
                               const uint8_t *ref, int64_t ref_len, Emit<WRITE> &E, uint32_t &nf)
{
    uint32_t spos = 1, prev = 0, qlen = 0;
    int64_t rpos = c.pos;
    nf = 0;
    for (uint32_t k = 0; k < nc; k++) {
        const uint32_t w = cig[4 * k] | cig[4 * k + 1] << 8 | cig[4 * k + 2] << 16 | (uint32_t)cig[4 * k + 3] << 24;
        const uint32_t op = w & 15, len = w >> 4;
        if (len == 0) return ENC_UNSUPPORTED;                                  // zero-length ops do not survive the feature form
        uint8_t code;
        switch (op) {
        case 0: case 7: case 8: code = 'b'; break;
        case 1: code = 'I'; break;
        case 2: code = 'D'; break;
        case 3: code = 'N'; break;
        case 4: code = 'S'; break;
        case 5: code = 'H'; break;
        default: code = 'P'; break;
        }
        if (code == 'b' && noseq) { spos += len; qlen += len; rpos += len; continue; }       // implicit match
        if (code == 'b' && ref) {
            if ((uint64_t)spos - 1 + len > (uint64_t)ls) return ENC_BAD;
            for (uint32_t i = 0; i < len; i++) {
                const uint8_t rb = rpos + i < ref_len ? ref[rpos + i] : (uint8_t)'N', sb = base_at(seq4, spos - 1 + i);
                if (rb == sb) continue;
                const int bs = bs_code(rb, sb);
                nf++;
                if (EMIT) {
                    E.put_byte(S_FC, bs >= 0 ? 'X' : 'b');
                    E.put_int(S_FP, (int32_t)(spos + i - prev));
                    prev = spos + i;
                    if (bs >= 0) E.put_byte(S_BS, (uint8_t)bs);
                    else { E.put_int(S_BB_LEN, 1); E.put_byte(S_BB, sb); }
                }
            }
            spos += len; qlen += len; rpos += len;
            continue;
        }
        nf++;
        if (EMIT) { E.put_byte(S_FC, code); E.put_int(S_FP, (int32_t)(spos - prev)); prev = spos; }
        if (code == 'b' || code == 'I' || code == 'S') {
            if (!noseq && (uint64_t)spos - 1 + len > (uint64_t)ls) return ENC_BAD;              // CIGAR longer than SEQ
            const int ln = code == 'b' ? S_BB_LEN : code == 'I' ? S_IN_LEN : S_SC_LEN;
            if (EMIT) { E.put_int(ln, (int32_t)len); if (noseq) E.put_fill(ln + 1, 'N', len); else E.put_bases(ln + 1, seq4, spos - 1, len); }
            spos += len; qlen += len;
            if (code == 'b') rpos += len;
        } else {
            if (EMIT) E.put_int(code == 'D' ? S_DL : code == 'N' ? S_RS : code == 'H' ? S_HC : S_PD, (int32_t)len);
            if (code == 'D' || code == 'N') rpos += len;
        }
    }
    if (!noseq && qlen != (uint32_t)ls) return ENC_BAD;                        // bam_set1 would refuse what the decoder rebuilds
    return ENC_OK;
}

// ---- tag blocks (HGPU_CRAM_ENC_TAG_BLOCKS): cram_encode_aux (cram_encode.c:2781-3200) for CRAM 3.x.  Every tag key is
// its own series, content id = its key (tag[0] << 16 | tag[1] << 8 | type), in the byte form of the key's codec:
// A c C s S i I f the value bytes, Z H the value with its NUL and a '\t' stop byte, B an ITF8 length and the bytes from
// the subtype on.  An RG:Z naming an @RG line leaves the tag line, its line index goes to the RG series.  In the
// reference-coded shape a record's MD:Z / NM are left out when the reader rebuilds them exactly (tag_rules).
enum { TAG_DROP_MD = 1, TAG_DROP_NM = 2 };
CRAMREC_HD inline uint32_t aux_key(const uint8_t *p) { return (uint32_t)p[0] << 16 | (uint32_t)p[1] << 8 | p[2]; }
CRAMREC_HD inline uint8_t ascii_lower(uint8_t c) { return c >= 'A' && c <= 'Z' ? (uint8_t)(c + 32) : c; }

// The MD string process_one_read would build, compared with a stored MD:Z value as strncasecmp does (:2852), one
// character at a time as it is produced.  v == nullptr: nothing to compare with.
struct MdCmp {
    const uint8_t *v; uint32_t i; bool ok;
    CRAMREC_HD void ch(uint8_t c) { if (ok && ascii_lower(v[i]) == ascii_lower(c)) i++; else ok = false; }   // v[i] == NUL never matches
    CRAMREC_HD void num(uint64_t x)                                       // kputuw
    {
        uint64_t p = 1;
        while (p <= x / 10) p *= 10;
        for (; p; p /= 10) ch((uint8_t)('0' + x / p % 10));
    }
    CRAMREC_HD bool equal() const { return v && ok && v[i] == 0; }
};

// MD / NM of one record against its reference sequence (ref[0] = base 1, ref_end = its length = c->ref_end of a
// multi-reference container, :2037-2056): process_one_read :3470-3723 and cram_encode_aux :2849-2884.  Returns the
// TAG_DROP_* bits.  Both stay (verbatim) for an unmapped record, SEQ "*", a base 'N' in both read and reference, and a
// match operation running past the reference end (:3512, :3525, :3605-3634); also wherever the reference's writer
// stops with an error (CIGAR and SEQ of different lengths, a mapped read at position 0, an NM of a type it cannot read
// whose value would have to be compared with 0).  NM is read as bam_aux2i_end reads it: c C s S i I by value, A and f
// as 0.  Only the first MD and NM fields are looked at: the host refuses records that repeat them.
CRAMREC_HD inline uint32_t tag_rules(const Core &c, const uint8_t *data, uint32_t l_data, const uint8_t *ref, int64_t ref_end)
{
    const uint32_t lq = c.l_qname, nc = c.n_cigar;
    const int32_t ls = c.l_qseq;
    if ((c.flag & 4) || ls <= 0 || c.pos < 0 || !ref) return 0;
    if ((uint64_t)lq + 4ull * nc + ((uint64_t)ls + 1) / 2 + (uint64_t)ls > l_data) return 0;
    const uint8_t *cig = data + lq, *seq4 = cig + 4 * nc, *aux = seq4 + (ls + 1) / 2 + ls, *end = data + l_data;
    const uint8_t *md = nullptr, *nm = nullptr;
    for (const uint8_t *p = aux; p < end;) {
        uint32_t vlen = 0;
        if (!aux_field(p, end, vlen)) return 0;
        if (p[0] == 'M' && p[1] == 'D' && !md) md = p;
        if (p[0] == 'N' && p[1] == 'M' && !nm) nm = p;
        p += 3 + vlen;
    }
    if (!md && !nm) return 0;
    MdCmp M{md && md[2] == 'Z' ? md + 3 : nullptr, 0, md && md[2] == 'Z'};
    int64_t apos = c.pos, md_last = apos, spos = 0;
    int32_t NM = 0;
    for (uint32_t k = 0; k < nc; k++) {
        const uint32_t w = cig[4 * k] | cig[4 * k + 1] << 8 | cig[4 * k + 2] << 16 | (uint32_t)cig[4 * k + 3] << 24;
        const uint32_t op = w & 15, len = w >> 4;
        switch (op) {
        case 0: case 7: case 8: {
            const int64_t e = (int64_t)len + apos < ref_end ? (int64_t)len : ref_end - apos;
            if (e > ls || spos + (e > 0 ? e : 0) > ls) return 0;                            // the reference's writer refuses the record
            int64_t l = 0;
            for (; l < e; l++) {
                const uint8_t rb = ref[apos + l], sb = base_at(seq4, (uint32_t)(spos + l));
                if (rb == 'N' && sb == 'N') return 0;
                if (rb != sb) { M.num((uint64_t)(apos + l - md_last)); M.ch(rb); md_last = apos + l + 1; NM++; }
            }
            if (l < (int64_t)len) return 0;                                                  // past the reference end
            spos += l; apos += l;
            break; }
        case 2:
            M.num((uint64_t)(apos - md_last));
            if (apos < ref_end) {
                M.ch('^');
                const int64_t d = ref_end - apos < (int64_t)len ? ref_end - apos : (int64_t)len;
                for (int64_t i = 0; i < d; i++) M.ch(ref[apos + i]);
            }
            NM += (int32_t)len; apos += len; md_last = apos;
            break;
        case 3: apos += len; md_last += len; break;
        case 1: NM += (int32_t)len; spos += len; break;
        case 4: spos += len; break;
        case 5: case 6: break;
        default: return 0;
        }
    }
    if (spos != ls) return 0;
    M.num((uint64_t)(apos - md_last));
    uint32_t drop = M.equal() ? TAG_DROP_MD : 0;
    if (nm) {
        const uint8_t *v = nm + 3;
        int32_t x;
        switch (nm[2]) {
        case 'c': x = (int8_t)v[0]; break;
        case 'C': x = v[0]; break;
        case 's': x = (int16_t)(v[0] | v[1] << 8); break;
        case 'S': x = (int32_t)(v[0] | v[1] << 8); break;
        case 'i': case 'I': x = (int32_t)(v[0] | v[1] << 8 | v[2] << 16 | (uint32_t)v[3] << 24); break;
        case 'A': case 'f': x = 0; break;
        default: x = NM == 0 ? -1 : 0; break;                                              // never equal: kept
        }
        if (x == NM) drop |= TAG_DROP_NM;
    }
    return drop;
}

// The tag-block inputs of one record (keys == nullptr: every tag value goes to the two shared streams).
struct TagRec { const uint32_t *keys; uint32_t nkeys; uint32_t drop; int32_t rg; };
CRAMREC_HD inline int key_stream(const TagRec &T, uint32_t key)                 // keys are sorted
{
    uint32_t lo = 0, hi = T.nkeys;
    while (lo < hi) { const uint32_t m = (lo + hi) / 2; if (T.keys[m] < key) lo = m + 1; else hi = m; }
    return lo < T.nkeys && T.keys[lo] == key ? S_COUNT + (int)lo : -1;
}

// One record.  tl = its tag-line index (the host built the dictionary).  ref / ref_len: the record's reference sequence
// (nullptr: none).  mate_cf / mate_nf: the pairing pass's decision (MATE_DETACHED without it).  T: the tag-block inputs.
// Returns ENC_OK or why the slice cannot be written here.
enum { MATE_DETACHED = 2, MATE_DOWNSTREAM = 4 };                               // CRAM_FLAG_DETACHED, CRAM_FLAG_MATE_DOWNSTREAM
template <bool WRITE>
CRAMREC_HD inline int walk(const Core &c, const uint8_t *data, uint32_t l_data, int32_t tl, const uint8_t *ref, int64_t ref_len,
                           uint32_t mate_cf, int32_t mate_nf, const TagRec &T, Emit<WRITE> &E)
{
    const uint32_t lq = c.l_qname, nc = c.n_cigar;
    const int32_t ls = c.l_qseq;
    if (lq == 0 || ls < 0 || (uint64_t)lq + 4ull * nc + ((uint64_t)ls + 1) / 2 + (uint64_t)ls > l_data) return ENC_BAD;
    const uint8_t *cig = data + lq, *seq4 = cig + 4 * nc, *qual = seq4 + (ls + 1) / 2, *aux = qual + ls, *end = data + l_data;
    const bool unmapped = (c.flag & 4) != 0;
    const bool has_qual = ls > 0 && qual[0] != 0xff;
    if (!unmapped && c.pos < 0) return ENC_UNSUPPORTED;                       // the reference's decoder refuses a mapped read at position 0
    if (c.flag >= 0x1000) return ENC_BAD;
    // a mapped read stored without its sequence ("*"): CRAM_FLAG_NO_SEQ, the read length comes from the CIGAR, match
    // operations are implicit (no feature), inserted and clipped bases are placeholders (process_one_read :3845-3870)
    const bool noseq = !unmapped && ls == 0;
    uint32_t cig_q = 0;
    for (uint32_t k = 0; k < nc; k++) {
        const uint32_t w = cig[4 * k] | cig[4 * k + 1] << 8 | cig[4 * k + 2] << 16 | (uint32_t)cig[4 * k + 3] << 24;
        const uint32_t op = w & 15;
        if (op > 8) return ENC_BAD;
        if (op == 0 || op == 1 || op == 4 || op == 7 || op == 8) cig_q += w >> 4;
    }
    if (noseq && nc == 0) return ENC_UNSUPPORTED;
    E.put_int(S_BF, c.flag);
    E.put_int(S_CF, (int32_t)mate_cf | (has_qual ? 1 : 0) | (noseq ? 8 : 0)); // DETACHED / MATE_DOWNSTREAM | PRESERVE_QUAL_SCORES | NO_SEQ
    E.put_int(S_RI, c.tid);
    E.put_int(S_RL, noseq ? (int32_t)cig_q : ls);
    E.put_int(S_AP, (int32_t)(c.pos + 1));
    E.put_int(S_RG, T.keys ? T.rg : -1);
    {   // the name up to its first NUL, then the stop byte
        uint32_t nl = 0;
        while (nl < lq && data[nl]) nl++;
        E.put_bytes(S_RN, data, nl);
        E.put_byte(S_RN, 0);
    }
    if (mate_cf & MATE_DETACHED) {
        E.put_int(S_MF, 0);
        E.put_int(S_NS, c.mtid);
        E.put_int(S_NP, (int32_t)(c.mpos + 1));
        E.put_int(S_TS, (int32_t)c.isize);
    }
    if (mate_cf & MATE_DOWNSTREAM) E.put_int(S_NF, mate_nf);
    E.put_int(S_TL, tl);
    // tags: lengths + values in order over two shared streams, or each value in its key's stream
    for (const uint8_t *p = aux; p < end;) {
        uint32_t vlen = 0;
        if (!aux_field(p, end, vlen)) return ENC_BAD;
        const uint8_t *v = p + 3;
        const uint8_t t = p[2];
        p += 3 + vlen;
        if (!T.keys) {
            E.put_int(S_TAG_LEN, (int32_t)vlen);
            E.put_bytes(S_TAG_VAL, v, vlen);
            continue;
        }
        if (((T.drop & TAG_DROP_MD) && v[-3] == 'M' && v[-2] == 'D' && t == 'Z') || ((T.drop & TAG_DROP_NM) && v[-3] == 'N' && v[-2] == 'M') ||
            (T.rg >= 0 && v[-3] == 'R' && v[-2] == 'G' && t == 'Z')) continue;
        const int s = key_stream(T, aux_key(v - 3));
        if (s < 0 || t == 'd') return ENC_UNSUPPORTED;                        // the host refuses both before the count pass
        if (t == 'B') E.put_int(s, (int32_t)vlen);
        E.put_bytes(s, v, vlen);
        if (t == 'Z' || t == 'H') E.put_byte(s, '\t');
    }
    if (!unmapped) {
        uint32_t nf = 0;
        int rc = features<WRITE, false>(c, cig, nc, seq4, ls, noseq, ref, ref_len, E, nf);
        if (rc != ENC_OK) return rc;
        E.put_int(S_FN, (int32_t)nf);
        rc = features<WRITE, true>(c, cig, nc, seq4, ls, noseq, ref, ref_len, E, nf);
        if (rc != ENC_OK) return rc;
        E.put_int(S_MQ, c.qual);
    } else E.put_bases(S_BA, seq4, 0, (uint32_t)ls);
    if (has_qual) E.put_bytes(S_QS, qual, (uint32_t)ls);
    return ENC_OK;
}

// ---- mate pairing: the mate block of process_one_read (cram_encode.c:3799-4012) for CRAM 3.x with the default options
// (tlen_zero = tlen_approx = 0, names kept).  Per slice, BAM_FPAIRED reads go into one of two name tables, pair[sec]
// (sec = BAM_FSECONDARY set).  The reads of one table entry form a group; groups are independent, a group's rule is
// serial in record order (mate_replay).

// 64-bit FNV-1a of the name (bam_name: up to its NUL) and the table it goes in
CRAMREC_HD inline uint64_t mate_hash(const uint8_t *name, uint32_t len, int sec)
{
    uint64_t h = 0xcbf29ce484222325ull ^ (uint64_t)sec;
    for (uint32_t i = 0; i < len; i++) h = (h ^ name[i]) * 0x100000001b3ull;
    return h;
}
CRAMREC_HD inline uint32_t mate_name_len(const uint8_t *data, uint32_t l_qname) { uint32_t n = 0; while (n < l_qname && data[n]) n++; return n; }

// cr->aend of process_one_read: a mapped read ends at pos + the reference bases its CIGAR spans (M D N = X), clamped to
// the container's reference end when coded against a reference (:3718); an unmapped read "ends" at MIN(apos, ref_end)
// (:3730).  ref_end is c->ref_end: 0 without a reference (the container is calloc'd and never given one), otherwise the
// length of the last reference sequence loaded for the container's records (see mate_ref_end in cram_encode.cu).
CRAMREC_HD inline int64_t mate_aend(const Core &c, const uint8_t *data, uint32_t l_data, bool no_ref, int64_t ref_end)
{
    const int64_t apos = c.pos + 1;
    if (c.flag & 4) return apos < ref_end ? apos : ref_end;
    int64_t e = c.pos;
    const uint32_t nc = c.n_cigar;
    if ((uint64_t)c.l_qname + 4ull * nc > l_data) return apos;                // malformed: the count pass refuses the record
    const uint8_t *cig = data + c.l_qname;
    for (uint32_t k = 0; k < nc; k++) {
        const uint32_t w = cig[4 * k] | cig[4 * k + 1] << 8 | cig[4 * k + 2] << 16 | (uint32_t)cig[4 * k + 3] << 24;
        const uint32_t op = w & 15;
        if (op == 0 || op == 2 || op == 3 || op == 7 || op == 8) e += w >> 4;
    }
    if (no_ref) return e;
    const int64_t re = ref_end > 0 ? ref_end : 0;
    return e < re ? e : re;
}

// The state process_one_read keeps for the record a name table entry points at (cram_record's fields of those names).
struct MateRec { int64_t apos, aend, mate_pos, tlen; int32_t ref_id; uint32_t flags, mate_flags; };

CRAMREC_HD inline MateRec mate_detached(const Core &c, int64_t aend)
{
    MateRec m;
    m.apos = c.pos + 1; m.aend = aend; m.ref_id = c.tid; m.flags = c.flag;
    m.mate_flags = ((c.flag & 8) ? 2u : 0u) | ((c.flag & 0x20) ? 1u : 0u);     // CRAM_M_UNMAP, CRAM_M_REVERSE
    m.mate_pos = c.mpos + 1 > 0 ? c.mpos + 1 : 0;
    m.tlen = c.isize;
    return m;
}

// One group: members[0 .. k) are global record numbers of one slice in increasing order.  cf[] / nf[] arrive as
// MATE_DETACHED / 0 and leave with process_one_read's decisions.
CRAMREC_HD inline void mate_replay(const uint32_t *members, uint32_t k, const Core *core, const int64_t *aend, uint8_t *cf, int32_t *nf)
{
    if (k < 2) return;
    uint32_t pi = members[0];
    MateRec p = mate_detached(core[pi], aend[pi]);
    uint32_t r12 = ((core[pi].flag & 0x40) ? 1u : 0u) | ((core[pi].flag & 0x80) ? 2u : 0u);
    for (uint32_t j = 1; j < k; j++) {
        const uint32_t g = members[j];
        const Core &b = core[g];
        const int64_t apos = b.pos + 1;
        const int64_t aleft = apos < p.apos ? apos : p.apos, aright = aend[g] > p.aend ? aend[g] : p.aend;
        const int64_t sign = apos < p.apos ? 1 : apos > p.apos ? -1 : (b.flag & 0x40) ? 1 : -1;
        const int64_t span = aright - aleft + 1;
        const bool detach =
            ((r12 & 1) && (b.flag & 0x40)) || ((r12 & 2) && (b.flag & 0x80)) ||                 // a repeated READ1 / READ2
            (b.mpos + 1 > 0 ? b.mpos + 1 : 0) != p.apos ||
            ((b.flag & 8) != 0) != ((p.flags & 4) != 0) || ((b.flag & 0x20) != 0) != ((p.flags & 0x10) != 0) ||
            p.ref_id != b.tid || p.mate_pos != apos ||
            ((p.flags & 8) != 0) != ((p.mate_flags & 2) != 0) || ((p.flags & 0x20) != 0) != ((p.mate_flags & 1) != 0) ||
            ((b.flag | p.flags) & 0x800) ||                                                     // supplementary
            b.isize == 0 || b.isize != sign * span || p.tlen == 0 || p.tlen != -sign * span;
        if (detach) continue;                                                                   // cf[g] stays DETACHED, the entry stays at p
        MateRec cr;
        cr.apos = apos; cr.aend = aend[g]; cr.ref_id = b.tid; cr.flags = b.flag;
        cr.mate_pos = p.apos;
        cr.tlen = sign * span;
        cr.mate_flags = ((p.flags & 8) ? 2u : 0u) | ((p.flags & 0x20) ? 1u : 0u);
        cf[g] = 0;
        cf[pi] = MATE_DOWNSTREAM;
        nf[pi] = (int32_t)(g - pi - 1);
        r12 |= ((b.flag & 0x40) ? 1u : 0u) | ((b.flag & 0x80) ? 2u : 0u);
        p = cr; pi = g;
    }
}

}  // namespace cramenc
