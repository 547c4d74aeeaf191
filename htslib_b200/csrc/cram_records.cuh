// CRAM 3.x record decode: the per-record loop of cram_decode_slice (cram/cram_decode.c:2554-2968), cram_decode_seq
// (:1096-1917), cram_decode_aux (:2008-2137), cram_decode_slice_xref (:2140-2304) and cram_to_bam (:3100-3211), with
// the codec readers of cram/cram_codecs.c they call (EXTERNAL :350-437, HUFFMAN :2641-2743, BETA :1072-1129,
// SUBEXP :2452-2499, GAMMA :2546-2572, BYTE_ARRAY_LEN :3371-3400, BYTE_ARRAY_STOP :3586-3672).
//
// One warp owns one slice.  The record loop is a serial chain (every series is a cursor that the previous record
// moved), so the warp runs it as uniform scalar code — all 32 lanes hold the same cursors and take the same branches,
// loads of the same address broadcast — and splits across lanes only where bytes move in bulk: reference bases into
// SEQ, quality runs, names, tag values, the stop-byte search of BYTE_ARRAY_STOP.  The `W` policy supplies those bulk
// operations; tests/hostsim builds this same header for the host with a W made of memcpy/memchr so the logic is
// checked against the reference where no GPU exists (the library itself only ever instantiates the warp policy).
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

#if defined(HGPU_HOSTSIM) && defined(CRAMREC_TRACE_ON)
#include <stdio.h>
#define CRAMREC_TRACE(...) fprintf(stderr, __VA_ARGS__)
#else
#define CRAMREC_TRACE(...) ((void)0)
#endif

namespace cramrec {

enum DS { DS_BF, DS_CF, DS_RI, DS_RL, DS_AP, DS_RG, DS_RN, DS_MF, DS_NS, DS_NP, DS_TS, DS_NF, DS_TL, DS_FN, DS_FC, DS_FP, DS_DL,
          DS_BA, DS_BS, DS_IN, DS_SC, DS_RS, DS_PD, DS_HC, DS_BB, DS_QQ, DS_MQ, DS_QS, DS_COUNT };

// CRAM_OPT_REQUIRED_FIELDS: the SAM_* bits of htslib/hts.h:279-291, and the data-series bits the reference derives from
// them (enum cram_fields, cram/cram_structs.h:890-922).  A slice's `ds` selects which series its record loop reads;
// `req` holds the caller's SAM_* mask for the choices cram_decode_slice / cram_to_bam make on it directly.
enum : int32_t { SAM_QNAME = 0x1, SAM_FLAG = 0x2, SAM_RNAME = 0x4, SAM_POS = 0x8, SAM_MAPQ = 0x10, SAM_CIGAR = 0x20, SAM_RNEXT = 0x40,
                 SAM_PNEXT = 0x80, SAM_TLEN = 0x100, SAM_SEQ = 0x200, SAM_QUAL = 0x400, SAM_AUX = 0x800, SAM_RGAUX = 0x1000,
                 SAM_ALL = 0x7fffffff };
enum : uint32_t { CRAM_BF = 1u << 0, CRAM_AP = 1u << 1, CRAM_FP = 1u << 2, CRAM_RL = 1u << 3, CRAM_DL = 1u << 4, CRAM_NF = 1u << 5,
                  CRAM_BA = 1u << 6, CRAM_QS = 1u << 7, CRAM_FC = 1u << 8, CRAM_FN = 1u << 9, CRAM_BS = 1u << 10, CRAM_IN = 1u << 11,
                  CRAM_RG = 1u << 12, CRAM_MQ = 1u << 13, CRAM_TL = 1u << 14, CRAM_RN = 1u << 15, CRAM_NS = 1u << 16, CRAM_NP = 1u << 17,
                  CRAM_TS = 1u << 18, CRAM_MF = 1u << 19, CRAM_CF = 1u << 20, CRAM_RI = 1u << 21, CRAM_RS = 1u << 22, CRAM_PD = 1u << 23,
                  CRAM_HC = 1u << 24, CRAM_SC = 1u << 25, CRAM_BB = 1u << 26, CRAM_BB_len = 1u << 27, CRAM_QQ = 1u << 28,
                  CRAM_aux = 1u << 30, CRAM_ALL = 0x7fffffffu,
                  CRAM_CIGAR = CRAM_FN | CRAM_FP | CRAM_FC | CRAM_DL | CRAM_IN | CRAM_SC | CRAM_HC | CRAM_PD | CRAM_RS | CRAM_RL | CRAM_BF,
                  CRAM_SEQ = CRAM_CIGAR | CRAM_BA | CRAM_BS | CRAM_RL | CRAM_AP | CRAM_BB,
                  CRAM_QUAL = CRAM_CIGAR | CRAM_RL | CRAM_AP | CRAM_QS | CRAM_QQ };

enum Kind : uint8_t { K_NONE = 0, K_EXTERNAL = 1, K_HUFFMAN = 3, K_BYTE_ARRAY_LEN = 4, K_BYTE_ARRAY_STOP = 5, K_BETA = 6, K_SUBEXP = 7, K_GAMMA = 9 };
enum Type : uint8_t { T_INT = 1, T_BYTE = 2, T_BYTE_ARRAY = 3, T_BYTE_ARRAY_BLOCK = 4 };   // cram_external_type

// EXTERNAL / BYTE_ARRAY_STOP: a = dense external-block index.  HUFFMAN: a = first code in the pool, ncodes.
// BETA: a = offset, b = nbits.  SUBEXP: a = offset, b = k.  GAMMA: a = offset.  BYTE_ARRAY_LEN: a, b = pool indices
// of the length and the value codec.
struct Codec { uint8_t kind, type, stop, pad; int32_t ncodes, a, b; };
struct HuffCode { int32_t symbol, len, code, p; };

struct Table {                       // one per container: cram_block_compression_hdr as the record loop uses it
    Codec ds[DS_COUNT];
    uint32_t n_tags, tag_off;        // tag encoding map: tagkeys[tag_off + i] -> cpool[tag_codec_off + i]
    uint32_t tag_codec_off;
    uint32_t n_tl, tl_off;           // tag dictionary: line i starts at td[tlidx[tl_off + i]], NUL terminated
    uint8_t sub[5][4];               // substitution_matrix
    uint8_t read_names_included, ap_delta, no_ref, qs_seq_orient;
    uint32_t n_ext;
};

struct Ext { uint64_t off; uint32_t size; uint32_t is_tok3; };       // size == 0xffffffff: the slice has no such block

struct Slice {
    int32_t table;
    int32_t ref_seq_id, ref_seq_start, ref_seq_span, n_records, ref_base_ext;    // ref_base_ext: dense index of the embedded reference block, -1 none
    int64_t record_counter;
    uint64_t core_off; uint32_t core_size;
    uint32_t ext_off;                // ext[ext_off .. +n_ext), cursors at the same index
    uint64_t rec0;                   // first record of this slice in the global record arrays
    uint64_t name_off, seq_off, aux_off, cig_off;       // arenas in the scratch buffer (cig_off in bytes, 4-aligned)
    uint32_t name_cap, seq_cap, aux_cap, cig_cap;       // bytes, bytes (seq and qual each), bytes, ops
    uint32_t ds;                     // data series the record loop reads (CRAM_ALL unless a field subset was asked for)
    int32_t req;                     // the SAM_* mask (SAM_ALL when none was given)
    int32_t cont_ref_start;          // the container's ref_seq_start: the position of every record when AP is not read
    int32_t pad;
};

struct Rec {                         // cram_record (cram/cram_structs.h:545-590) as far as cram_to_bam reads it
    int64_t apos, aend, mate_pos, tlen, explicit_tlen;
    int32_t flags, cram_flags, ref_id, len, rg, mate_line, mate_ref_id, mate_flags, mqual;
    uint32_t name, name_len, seq, qual, aux, aux_size, cigar, ncigar;
};

struct Refs {                        // whole reference sequences, upper case, @SQ order; sq_len = the header's LN
    const uint8_t *bases; const uint64_t *off; const int64_t *sq_len; int32_t n_ref;
};

struct Pools {
    const Table *tables; const Codec *cpool; const HuffCode *hpool; const uint32_t *tagkeys; const uint32_t *tlidx; const uint8_t *td;
    const Ext *ext; uint32_t *cur; const uint8_t *udata;
};

enum { ERR_NONE = 0, ERR_DECODE = -1, ERR_SPACE = -4, ERR_NOREF = -7 };
#define CRAMREC_I64_MIN (-9223372036854775807LL - 1)

enum { BAM_FPAIRED = 1, BAM_FUNMAP = 4, BAM_FMUNMAP = 8, BAM_FREVERSE = 16, BAM_FMREVERSE = 32, BAM_FREAD1 = 64 };
enum { CRAM_FLAG_PRESERVE_QUAL_SCORES = 1, CRAM_FLAG_DETACHED = 2, CRAM_FLAG_MATE_DOWNSTREAM = 4, CRAM_FLAG_NO_SEQ = 8,
       CRAM_FLAG_EXPLICIT_TLEN = 16 };
enum { CRAM_M_REVERSE = 1, CRAM_M_UNMAP = 2 };
enum { CIG_M = 0, CIG_I = 1, CIG_D = 2, CIG_N = 3, CIG_S = 4, CIG_H = 5, CIG_P = 6 };

CRAMREC_HD inline int l1_code(uint8_t c)                                 // fd->L1, cram_io.c:5173-5177
{
    switch (c) { case 'A': case 'a': return 0; case 'C': case 'c': return 1; case 'G': case 'g': return 2; case 'T': case 't': return 3; default: return 4; }
}

template <class W>
struct SliceDec {
    Pools P;
    const Table *T;
    const Ext *ext;
    uint32_t *cur;
    const uint8_t *core; uint32_t csize, cbyte; int cbit;
    uint8_t *name; uint32_t name_size, name_cap;
    uint8_t *aux; uint32_t aux_size, aux_cap;
    uint8_t *seqs, *quals; uint32_t sq_size, sq_cap;
    uint32_t *cigar; uint32_t ncigar, cig_cap;
    const uint8_t *ref; int64_t ref_start, ref_end;
    Refs R;
    int decode_md_opt;
    int err;

    // ---- CORE bit stream (MSB first) ----
    CRAMREC_HD bool not_enough_bits(int64_t nbits) const                   // cram_codecs.h:230-238
    {
        if (nbits < 0 || (cbyte >= csize && nbits > 0)) return true;
        return (int64_t)(csize - cbyte) * 8 + cbit - 7 < nbits;
    }
    CRAMREC_HD void get_bit(int32_t &v)
    {
        v = (int32_t)(((uint32_t)v << 1) | ((core[cbyte] >> cbit) & 1u));
        if (--cbit < 0) { cbit = 7; cbyte++; }
    }
    CRAMREC_HD int64_t get_bits(int n) { int64_t v = 0; for (int i = 0; i < n; i++) { v = (v << 1) | ((core[cbyte] >> cbit) & 1u); if (--cbit < 0) { cbit = 7; cbyte++; } } return v; }
    CRAMREC_HD int count_bits(int which)                                   // get_one_bits_MSB / get_zero_bits_MSB :95-131
    {
        int n = 0, b;
        if (cbyte >= csize) return -1;
        do {
            b = core[cbyte] >> cbit;
            if (--cbit == -1) { cbit = 7; cbyte++; if (cbyte == csize && ((b & 1) == which)) return -1; }
            n++;
        } while ((b & 1) == which);
        return n - 1;
    }

    // ---- external blocks ----
    CRAMREC_HD int ext_int(int32_t x, int32_t &out)                        // cram_external_decode_int + safe_itf8_get
    {
        const Ext e = ext[x];
        if (e.size == 0xffffffffu) return -1;
        const uint8_t *p = P.udata + e.off + cur[x];
        const int64_t left = (int64_t)e.size - (int64_t)cur[x];
        if (left < 1) return -1;
        const uint32_t c = p[0];
        const int n = c < 0x80 ? 0 : c < 0xc0 ? 1 : c < 0xe0 ? 2 : c < 0xf0 ? 3 : 4;
        if (left < n + 1) return -1;
        uint32_t v;
        switch (n) {
        case 0: v = c; break;
        case 1: v = ((c & 0x3fu) << 8) | p[1]; break;
        case 2: v = ((c & 0x1fu) << 16) | ((uint32_t)p[1] << 8) | p[2]; break;
        case 3: v = ((c & 0x0fu) << 24) | ((uint32_t)p[1] << 16) | ((uint32_t)p[2] << 8) | p[3]; break;
        default: v = ((c & 0x0fu) << 28) | ((uint32_t)p[1] << 20) | ((uint32_t)p[2] << 12) | ((uint32_t)p[3] << 4) | (p[4] & 0x0fu); break;
        }
        cur[x] += (uint32_t)n + 1;
        out = (int32_t)v;
        return 0;
    }
    CRAMREC_HD const uint8_t *ext_take(int32_t x, int64_t n)               // cram_extract_block :319-326
    {
        const Ext e = ext[x];
        if (e.size == 0xffffffffu) return nullptr;
        const uint8_t *p = P.udata + e.off + cur[x];
        const uint64_t nx = (uint64_t)cur[x] + (uint64_t)n;
        cur[x] = nx > 0xfffffffeull ? 0xfffffffeu : (uint32_t)nx;          // the reference advances before it checks
        if (nx > e.size) return nullptr;
        return p;
    }

    // ---- codecs ----
    CRAMREC_HD int huff_one(const Codec &c, int32_t &sym)                  // cram_huffman_decode_int / _char, one item
    {
        const HuffCode *codes = P.hpool + c.a;
        if (c.ncodes == 0) return -1;                                       // cram_huffman_decode_null
        if (codes[0].len == 0) { sym = codes[0].symbol; return 0; }
        int idx = 0, len = 0, last_len = 0;
        int32_t val = 0;
        for (;;) {
            int dlen = codes[idx].len - last_len;
            if (not_enough_bits(dlen)) return -1;
            last_len = (len += dlen);
            for (; dlen; dlen--) get_bit(val);
            idx = val - codes[idx].p;
            if (idx >= c.ncodes || idx < 0) return -1;
            if (codes[idx].code == val && codes[idx].len == len) { sym = codes[idx].symbol; return 0; }
        }
    }
    CRAMREC_HD int get_int(const Codec &c, int32_t &out)
    {
        switch (c.kind) {
        case K_EXTERNAL: return c.type == T_INT ? ext_int(c.a, out) : -1;
        case K_HUFFMAN: return huff_one(c, out);
        case K_BETA:
            if (c.b) { if (not_enough_bits(c.b)) return -1; out = (int32_t)(get_bits(c.b) - c.a); }
            else out = -c.a;
            return 0;
        case K_SUBEXP: {
            const int k = c.b;
            const int i = count_bits(1);
            if (i < 0 || not_enough_bits(i > 0 ? i + k - 1 : k)) return -1;
            int32_t val = 0;
            if (i) { for (int t = i + k - 1; t; t--) get_bit(val); val += 1 << (i + k - 1); }
            else for (int t = k; t; t--) get_bit(val);
            out = val - c.a;
            return 0; }
        case K_GAMMA: {
            int nz = count_bits(0);
            if (not_enough_bits(nz)) return -1;
            int32_t val = 1;
            while (nz > 0) { get_bit(val); nz--; }
            out = val - c.a;
            return 0; }
        default: return -1;
        }
    }
    // one item of a BYTE series, returned to every lane (FC, BS, single BA / QS)
    CRAMREC_HD int get_byte(const Codec &c, uint8_t &out)
    {
        switch (c.kind) {
        case K_EXTERNAL: {
            if (ext[c.a].size == 0xffffffffu) return -1;
            const uint8_t *p = ext_take(c.a, 1);
            if (!p) return -1;
            out = *p;
            return 0; }
        case K_HUFFMAN: { int32_t s2 = 0; if (huff_one(c, s2)) return -1; out = (uint8_t)s2; return 0; }
        case K_BETA:
            if (c.b) { if (not_enough_bits(c.b)) return -1; out = (uint8_t)(get_bits(c.b) - c.a); }
            else out = (uint8_t)(-c.a);
            return 0;
        default: return -1;
        }
    }
    // type BYTE / BYTE_ARRAY value codecs: n items to out in memory (may be null: consume only)
    CRAMREC_HD int get_bytes(const Codec &c, uint8_t *out, int32_t n)
    {
        switch (c.kind) {
        case K_EXTERNAL: {
            if (ext[c.a].size == 0xffffffffu) return n ? -1 : 0;
            const uint8_t *p = ext_take(c.a, n);
            if (!p) return -1;
            if (out) W::copy(out, p, (uint32_t)n);
            return 0; }
        case K_HUFFMAN: {
            if (c.ncodes == 0) return -1;
            const HuffCode *codes = P.hpool + c.a;
            if (codes[0].len == 0) { if (out) W::fill(out, (uint8_t)codes[0].symbol, (uint32_t)n); return 0; }
            for (int32_t i = 0; i < n; i++) { int32_t s; if (huff_one(c, s)) return -1; if (out) out[i] = (uint8_t)s; }
            W::sync();
            return 0; }
        case K_BETA:
            if (c.b) {
                if (not_enough_bits((int64_t)c.b * n)) return -1;
                for (int32_t i = 0; i < n; i++) { const int64_t v = get_bits(c.b) - c.a; if (out) out[i] = (uint8_t)v; }
                W::sync();
            } else if (out) W::fill(out, (uint8_t)(-c.a), (uint32_t)n);
            return 0;
        default: return -1;
        }
    }
    CRAMREC_HD bool append(uint8_t *&base, uint32_t &size, uint32_t cap, const uint8_t *src, uint32_t n)
    {
        if ((uint64_t)size + n > cap) { CRAMREC_TRACE("append: %u + %u > %u\n", size, n, cap); err = ERR_SPACE; return false; }
        W::copy(base + size, src, n);
        size += n;
        return true;
    }
    // E_BYTE_ARRAY series (IN, SC, BB, QQ): out may be null; out_sz in = room, out = produced
    CRAMREC_HD int get_array_char(const Codec &c, uint8_t *out, int32_t &out_sz)
    {
        if (c.kind == K_BYTE_ARRAY_LEN) {
            int32_t len = 0;
            const int r = get_int(P.cpool[c.a], len);
            if (len < 0 || len > out_sz) return -1;
            if (r) return -1;
            const int r2 = get_bytes(P.cpool[c.b], out, len);
            out_sz = len;
            return r2;
        }
        if (c.kind == K_BYTE_ARRAY_STOP) {                                  // cram_byte_array_stop_decode_char
            const Ext e = ext[c.a];
            if (e.size == 0xffffffffu) return out_sz ? -1 : 0;
            if (cur[c.a] >= e.size) return -1;
            uint32_t term = e.size - cur[c.a];
            const uint8_t *p = P.udata + e.off + cur[c.a];
            if (out && (int64_t)term > (int64_t)out_sz) term = out_sz > 0 ? (uint32_t)out_sz : 0u;
            const uint32_t k = W::find(p, term, c.stop);
            if (cur[c.a] + k >= e.size || p[k] != c.stop) return -1;
            if (out) W::copy(out, p, k);
            out_sz = (int32_t)k;
            cur[c.a] += k + 1;
            return 0;
        }
        return -1;
    }
    // E_BYTE_ARRAY_BLOCK series (RN, tags): appended to an arena
    CRAMREC_HD int block_leaf(const Codec &c, uint8_t *&base, uint32_t &size, uint32_t cap, int32_t &out_sz)
    {
        if (c.kind == K_EXTERNAL) {                                         // cram_external_decode_block
            if (ext[c.a].size == 0xffffffffu) return out_sz ? -1 : 0;
            const uint8_t *p = ext_take(c.a, out_sz);
            if (!p) return -1;
            return append(base, size, cap, p, (uint32_t)out_sz) ? 0 : -1;
        }
        if (c.kind == K_BYTE_ARRAY_STOP) {                                  // cram_byte_array_stop_decode_block
            const Ext e = ext[c.a];
            if (e.size == 0xffffffffu) return out_sz ? -1 : 0;
            if (cur[c.a] >= e.size) return -1;
            const uint8_t stop = e.is_tok3 ? 0 : c.stop;
            const uint8_t *p = P.udata + e.off + cur[c.a];
            const uint32_t k = W::find(p, e.size - cur[c.a], stop);
            if (!append(base, size, cap, p, k)) return -1;
            out_sz = (int32_t)k;
            cur[c.a] += k + 1;
            return 0;
        }
        return -1;
    }
    CRAMREC_HD int get_array_block(const Codec &c, uint8_t *&base, uint32_t &size, uint32_t cap, int32_t &out_sz)
    {
        if (c.kind == K_BYTE_ARRAY_LEN) {
            int32_t len = 0;
            const Codec &vc = P.cpool[c.b];
            const int r = get_int(P.cpool[c.a], len);
            if (len < 0 || (len > out_sz && vc.kind != K_EXTERNAL)) return -1;
            if (r) return -1;
            int32_t l2 = len;
            const int r2 = block_leaf(vc, base, size, cap, l2);            // the tables only admit EXTERNAL / BYTE_ARRAY_STOP here
            out_sz = len;
            return r2;
        }
        return block_leaf(c, base, size, cap, out_sz);
    }

    // ---- small appenders for MD / cigar ----
    CRAMREC_HD bool aux_char(uint8_t c) { if (aux_size >= aux_cap) { CRAMREC_TRACE("aux_char full %u\n", aux_cap); err = ERR_SPACE; return false; } aux[aux_size++] = c; return true; }
    CRAMREC_HD bool aux_uint(uint32_t v)                                    // BLOCK_APPEND_UINT: decimal
    {
        uint8_t tmp[10]; int n = 0;
        do { tmp[n++] = (uint8_t)('0' + v % 10); v /= 10; } while (v);
        if ((uint64_t)aux_size + n > aux_cap) { err = ERR_SPACE; return false; }
        while (n) aux[aux_size++] = tmp[--n];
        return true;
    }
    CRAMREC_HD bool md_char(int decode_md, uint8_t c, int32_t &md_dist)     // add_md_char :1080-1090
    {
        if (decode_md) { if (!aux_uint((uint32_t)md_dist) || !aux_char(c)) return false; md_dist = 0; }
        return true;
    }
    CRAMREC_HD bool cig_push(uint32_t len, uint32_t op)
    {
        if (ncigar >= cig_cap) { CRAMREC_TRACE("cigar full %u\n", cig_cap); err = ERR_SPACE; return false; }
        cigar[ncigar++] = (len << 4) + op;
        return true;
    }
    CRAMREC_HD int64_t sq_len(int32_t id) const { return R.sq_len[id]; }

    // cram_decode_seq :1096-1917.  returns 0 / -1
    // SUBSET: the record loop of a field subset, gated by the slice's data-series mask; the all-fields instantiation
    // (SUBSET false, every gate constant) compiles to the loop without gates
    template <bool SUBSET>
    CRAMREC_HD int decode_seq(Rec &cr, int cf, uint8_t *seq, uint8_t *qual, int has_MD, int has_NM, uint32_t slice_ds)
    {
        const uint32_t ds = SUBSET ? slice_ds : CRAM_ALL;
        int32_t prev_pos = 0, fn = 0, i32 = 0;
        int32_t seq_pos = 1;
        uint32_t cig_len = 0, cig_op = CIG_M;
        int64_t ref_pos = cr.apos;
        uint32_t nm = 0;
        int32_t md_dist = 0;
        uint32_t orig_aux = 0;
        const int do_md = decode_md_opt != 0;
        int decode_md = ref && cr.ref_id >= 0 && ((do_md && !has_MD) || has_MD < 0);
        int decode_nm = ref && cr.ref_id >= 0 && ((do_md && !has_NM) || has_NM < 0);
        const Codec *C = T->ds;
        const int pres_q = cf & CRAM_FLAG_PRESERVE_QUAL_SCORES;

        if ((ds & CRAM_QS) && !pres_q) W::fill(qual, 255, (uint32_t)cr.len);
        if (cr.cram_flags & CRAM_FLAG_NO_SEQ) decode_md = decode_nm = 0;
        if (decode_md) {
            orig_aux = aux_size;
            if (has_MD == 0) { if (!aux_char('M') || !aux_char('D') || !aux_char('Z')) return -1; }
        }
        if (ds & CRAM_FN) {
            if (C[DS_FN].kind == K_NONE) return -1;
            if (get_int(C[DS_FN], fn)) return -1;
        }
        ref_pos--;
        cr.cigar = ncigar;
        // without FC and FP the reference skips the features and the implicit match (goto skip_cigar); the selection
        // makes FP imply FC, so the only partial case is FC alone: the codes are read, nothing else
        if (fn && (ds & (CRAM_FC | CRAM_FP))) {
            if (((ds & CRAM_FC) && C[DS_FC].kind == K_NONE) || ((ds & CRAM_FP) && C[DS_FP].kind == K_NONE)) return -1;
        }

        for (int32_t f = 0; f < fn && (ds & (CRAM_FC | CRAM_FP)); f++) {
            int32_t pos = 0;
            uint8_t op = 0;
            if (ncigar + 2 >= cig_cap) { err = ERR_SPACE; return -1; }
            if ((ds & CRAM_FC) && get_byte(C[DS_FC], op)) return -1;
            if (!(ds & CRAM_FP)) continue;
            if (get_int(C[DS_FP], pos)) return -1;
            pos += prev_pos;
            if (pos <= 0) return -1;
            if (cr.len != 0 && pos > cr.len) {
                const int32_t valid_end = (op == 'N' || op == 'P' || op == 'H' || op == 'D') ? cr.len + 1 : cr.len;
                if (pos > valid_end) return -1;
            }
            if (pos > seq_pos) {
                if (ref && cr.ref_id >= 0) {
                    if (ref_pos + pos - seq_pos > sq_len(cr.ref_id)) {
                        const int64_t rlen = sq_len(cr.ref_id) - ref_pos;
                        if (rlen > 0) {
                            if (ref_pos + rlen > ref_end) return -1;
                            if (cr.len) {
                                W::copy(&seq[seq_pos - 1], &ref[ref_pos - ref_start + 1], (uint32_t)rlen);
                                if ((pos - seq_pos) - rlen > 0) W::fill(&seq[seq_pos - 1 + rlen], 'N', (uint32_t)((pos - seq_pos) - rlen));
                            }
                        } else if (cr.len) W::fill(&seq[seq_pos - 1], 'N', (uint32_t)(cr.len - seq_pos + 1));
                        if (md_dist >= 0) md_dist += pos - seq_pos;
                    } else {
                        if (ref_pos + pos - seq_pos > ref_end) return -1;
                        const uint8_t *refp = ref + (ref_pos - ref_start + 1);
                        const int32_t frag_len = pos - seq_pos;
                        if (decode_md || decode_nm) {
                            if (W::find(refp, (uint32_t)frag_len, 'N') < (uint32_t)frag_len) {
                                for (int32_t i = 0; i < frag_len; i++) {
                                    if (refp[i] == 'N') { if (!md_char(decode_md, 'N', md_dist)) return -1; nm++; }
                                    else md_dist++;
                                }
                            } else md_dist += frag_len;
                        }
                        if (cr.len) W::copy(&seq[seq_pos - 1], refp, (uint32_t)frag_len);
                    }
                }
                if (cig_len && cig_op != CIG_M) { if (!cig_push(cig_len, cig_op)) return -1; cig_len = 0; }
                cig_op = CIG_M;
                cig_len += pos - seq_pos;
                ref_pos += pos - seq_pos;
                seq_pos = pos;
            }
            prev_pos = pos;
            if (!(ds & CRAM_FC)) break;

            switch (op) {
            case 'S': {
                int32_t out_sz2 = cr.len ? cr.len - (pos - 1) : 1;
                if (cig_len) { if (!cig_push(cig_len, cig_op)) return -1; cig_len = 0; }
                if (!(ds & CRAM_SC)) break;
                if (C[DS_SC].kind != K_NONE) { if (get_array_char(C[DS_SC], cr.len ? &seq[pos - 1] : nullptr, out_sz2)) return -1; }
                else { if (cr.len) seq[pos - 1] = 'N'; out_sz2 = 1; }
                if (!cig_push((uint32_t)out_sz2, CIG_S)) return -1;
                cig_op = CIG_S;
                seq_pos += out_sz2;
                break; }
            case 'X': {
                uint8_t base = 0;
                if (cig_len && cig_op != CIG_M) { if (!cig_push(cig_len, cig_op)) return -1; cig_len = 0; }
                if (!(ds & CRAM_BS)) {
                } else if (C[DS_BS].kind == K_NONE || get_byte(C[DS_BS], base)) {
                    return -1;
                } else if (cr.ref_id < 0 || ref_pos >= sq_len(cr.ref_id) || !ref) {
                    if (pos - 1 < cr.len) seq[pos - 1] = T->sub[4][base & 3];
                    if (decode_md || decode_nm) {
                        if (md_dist >= 0 && decode_md) { if (!aux_uint((uint32_t)md_dist)) return -1; }
                        md_dist = -1;
                        nm--;
                    }
                } else {
                    const uint8_t ref_call = ref_pos < ref_end ? ref[ref_pos - ref_start + 1] : (uint8_t)'N';
                    if (pos - 1 < cr.len) seq[pos - 1] = T->sub[l1_code(ref_call)][base & 3];
                    if (!md_char(decode_md, ref_call, md_dist)) return -1;
                }
                cig_op = CIG_M;
                nm++; cig_len++; seq_pos++; ref_pos++;
                break; }
            case 'D': {
                if (cig_len && cig_op != CIG_D) { if (!cig_push(cig_len, cig_op)) return -1; cig_len = 0; }
                if (!(ds & CRAM_DL)) break;
                if (C[DS_DL].kind == K_NONE) return -1;
                if (get_int(C[DS_DL], i32)) return -1;
                if (i32 < 0) return -1;
                if (decode_md || decode_nm) {
                    if (ref_pos + i32 > ref_end) return -1;
                    if (md_dist >= 0 && decode_md) { if (!aux_uint((uint32_t)md_dist)) return -1; }
                    if (ref_pos + i32 <= sq_len(cr.ref_id)) {
                        if (decode_md) {
                            if (!aux_char('^')) return -1;
                            if (!append(aux, aux_size, aux_cap, &ref[ref_pos - ref_start + 1], (uint32_t)i32)) return -1;
                            md_dist = 0;
                        }
                        nm += i32;
                    } else {
                        uint32_t dlen;
                        if (sq_len(cr.ref_id) >= ref_pos) {
                            if (decode_md) {
                                if (!aux_char('^')) return -1;
                                if (!append(aux, aux_size, aux_cap, &ref[ref_pos - ref_start + 1], (uint32_t)(sq_len(cr.ref_id) - ref_pos))) return -1;
                                if (!aux_uint(0)) return -1;
                            }
                            dlen = (uint32_t)(i32 - (sq_len(cr.ref_id) - ref_pos));
                            nm += i32 - dlen;
                        }
                        md_dist = -1;
                    }
                }
                cig_op = CIG_D;
                cig_len += i32;
                ref_pos += i32;
                break; }
            case 'I': {
                int32_t out_sz2 = cr.len ? cr.len - (pos - 1) : 1;
                if (cig_len && cig_op != CIG_I) { if (!cig_push(cig_len, cig_op)) return -1; cig_len = 0; }
                if (!(ds & CRAM_IN)) break;
                if (C[DS_IN].kind == K_NONE) return -1;
                if (get_array_char(C[DS_IN], cr.len ? &seq[pos - 1] : nullptr, out_sz2)) return -1;
                cig_op = CIG_I;
                cig_len += out_sz2; seq_pos += out_sz2; nm += out_sz2;
                break; }
            case 'i': {
                if (cig_len && cig_op != CIG_I) { if (!cig_push(cig_len, cig_op)) return -1; cig_len = 0; }
                if (ds & CRAM_BA) {
                    if (C[DS_BA].kind == K_NONE) return -1;
                    uint8_t b1 = 0; if (get_byte(C[DS_BA], b1)) return -1; if (cr.len) seq[pos - 1] = b1;
                }
                cig_op = CIG_I;
                cig_len++; seq_pos++; nm++;
                break; }
            case 'b': {
                int32_t len = cr.len ? cr.len - (pos - 1) : 1;
                if (cig_len && cig_op != CIG_M) { if (!cig_push(cig_len, cig_op)) return -1; cig_len = 0; }
                if (!(ds & CRAM_BB)) {
                } else if (C[DS_BB].kind == K_NONE || get_array_char(C[DS_BB], cr.len ? &seq[pos - 1] : nullptr, len)) {
                    return -1;
                } else if (decode_md || decode_nm) {
                    int32_t x;
                    if (md_dist >= 0 && decode_md) { if (!aux_uint((uint32_t)md_dist)) return -1; }
                    for (x = 0; x < len; x++) {
                        if (x && decode_md) { if (!aux_uint(0)) return -1; }
                        if (ref_pos + x >= sq_len(cr.ref_id) || !ref) { md_dist = -1; break; }
                        else if (decode_md) {
                            if (ref_pos + x >= ref_end) return -1;
                            if (!aux_char(ref[ref_pos + x - ref_start + 1])) return -1;
                        }
                    }
                    nm += x;
                    md_dist = 0;
                }
                cig_op = CIG_M;
                cig_len += len; seq_pos += len; ref_pos += len;
                break; }
            case 'q': {
                int32_t len = cr.len ? cr.len - (pos - 1) : 1;
                if (cig_len && cig_op != CIG_M) { if (!cig_push(cig_len, cig_op)) return -1; cig_len = 0; }
                if (ds & CRAM_QQ) {
                    if (C[DS_QQ].kind == K_NONE) return -1;
                    if ((ds & CRAM_QS) && !pres_q && cr.len > 0 && qual[0] == 255) W::fill(qual, 30, (uint32_t)cr.len);
                    if (get_array_char(C[DS_QQ], cr.len ? &qual[pos - 1] : nullptr, len)) return -1;
                }
                cig_op = CIG_M;
                break; }
            case 'B': {
                if (cig_len && cig_op != CIG_M) { if (!cig_push(cig_len, cig_op)) return -1; cig_len = 0; }
                uint8_t b1 = 0, q1 = 0;
                int rb = 0, rq = 0;
                if (ds & CRAM_BA) {
                    if (C[DS_BA].kind == K_NONE) return -1;
                    rb = get_byte(C[DS_BA], b1);
                    if (!rb && cr.len) seq[pos - 1] = b1;
                    if (decode_md || decode_nm) {
                        if (md_dist >= 0 && decode_md) { if (!aux_uint((uint32_t)md_dist)) return -1; }
                        if (ref_pos >= sq_len(cr.ref_id) || !ref) md_dist = -1;
                        else {
                            if (decode_md) {
                                if (ref_pos >= ref_end) return -1;
                                if (!aux_char(ref[ref_pos - ref_start + 1])) return -1;
                            }
                            nm++;
                            md_dist = 0;
                        }
                    }
                }
                if (ds & CRAM_QS) {
                    if (C[DS_QS].kind == K_NONE) return -1;
                    if (!pres_q && cr.len > 0 && qual[0] == 255) W::fill(qual, 30, (uint32_t)cr.len);
                    rq = get_byte(C[DS_QS], q1);
                    if (!rq && cr.len) qual[pos - 1] = q1;
                }
                if (rb | rq) return -1;                                    // the reference ORs r and fails the record at the end
                cig_op = CIG_M;
                cig_len++; seq_pos++; ref_pos++;
                break; }
            case 'Q': {
                if (!(ds & CRAM_QS)) break;
                if (C[DS_QS].kind == K_NONE) return -1;
                if (!pres_q && cr.len > 0 && qual[0] == 255) W::fill(qual, 30, (uint32_t)cr.len);
                { uint8_t q1 = 0; if (get_byte(C[DS_QS], q1)) return -1; if (cr.len) qual[pos - 1] = q1; }
                break; }
            case 'H': case 'P': case 'N': {
                const uint32_t cop = op == 'H' ? CIG_H : op == 'P' ? CIG_P : CIG_N;
                const int series = op == 'H' ? DS_HC : op == 'P' ? DS_PD : DS_RS;
                if (cig_len && cig_op != cop) { if (!cig_push(cig_len, cig_op)) return -1; cig_len = 0; }
                if (!(ds & (op == 'H' ? CRAM_HC : op == 'P' ? CRAM_PD : CRAM_RS))) break;
                if (C[series].kind == K_NONE) return -1;
                if (get_int(C[series], i32)) return -1;
                if (i32 < 0) return -1;
                cig_op = cop;
                cig_len += i32;
                if (op == 'N') ref_pos += i32;
                break; }
            default:
                return -1;
            }
            W::sync();
        }

        // implicit match for the bases no feature accounted for
        if ((ds & CRAM_FC) && (ds & CRAM_FN) && cr.len >= seq_pos) {
            if (ref && cr.ref_id >= 0) {
                if (ref_pos + cr.len - seq_pos + 1 > sq_len(cr.ref_id)) {
                    const int64_t rlen = sq_len(cr.ref_id) - ref_pos;
                    if (rlen > 0) {
                        if (ref_pos + rlen > ref_end) return -1;
                        if (seq_pos - 1 + rlen < cr.len) W::copy(&seq[seq_pos - 1], &ref[ref_pos - ref_start + 1], (uint32_t)rlen);
                        if ((cr.len - seq_pos + 1) - rlen > 0) W::fill(&seq[seq_pos - 1 + rlen], 'N', (uint32_t)((cr.len - seq_pos + 1) - rlen));
                    } else if (cr.len - seq_pos + 1 > 0) W::fill(&seq[seq_pos - 1], 'N', (uint32_t)(cr.len - seq_pos + 1));
                    if (md_dist >= 0) md_dist += cr.len - seq_pos + 1;
                } else {
                    if (cr.len - seq_pos + 1 > 0) {
                        if (ref_pos + cr.len - seq_pos + 1 > ref_end) return -1;
                        const int32_t remainder = cr.len - (seq_pos - 1);
                        const int64_t j = ref_pos - ref_start + 1;
                        if (decode_md || decode_nm) {
                            const uint32_t nf = W::find(&ref[j], (uint32_t)remainder, 'N');
                            if (nf >= (uint32_t)remainder) md_dist += cr.len - (seq_pos - 1);
                            else {
                                md_dist += (int32_t)nf;
                                for (int32_t i = (int32_t)nf; i < remainder; i++) {
                                    if (ref[j + i] == 'N') { if (!md_char(decode_md, 'N', md_dist)) return -1; nm++; }
                                    else md_dist++;
                                }
                            }
                        }
                        W::copy(&seq[seq_pos - 1], &ref[j], (uint32_t)remainder);
                    }
                    ref_pos += cr.len - seq_pos + 1;
                }
            } else if (cr.ref_id >= 0) ref_pos += cr.len - seq_pos + 1;
            if (ncigar + 1 >= cig_cap) { err = ERR_SPACE; return -1; }
            if (cig_len && cig_op != CIG_M) { if (!cig_push(cig_len, cig_op)) return -1; cig_len = 0; }
            cig_op = CIG_M;
            cig_len += cr.len - seq_pos + 1;
        }

        if ((ds & CRAM_FN) && decode_md && md_dist >= 0) { if (!aux_uint((uint32_t)md_dist)) return -1; }
        if (cig_len) { if (!cig_push(cig_len, cig_op)) return -1; }
        cr.ncigar = ncigar - cr.cigar;
        cr.aend = ref_pos > cr.apos ? ref_pos : cr.apos;

        int r = 0;
        if (ds & CRAM_MQ) {
            if (C[DS_MQ].kind == K_NONE) return -1;
            r |= get_int(C[DS_MQ], cr.mqual);
        } else cr.mqual = 40;
        if ((ds & CRAM_QS) && pres_q) {
            if (C[DS_QS].kind == K_NONE) return -1;
            r |= get_bytes(C[DS_QS], qual, cr.len);
        }
        if (cr.cram_flags & CRAM_FLAG_NO_SEQ) cr.len = 0;

        if (decode_md) {
            if (!aux_char(0)) return -1;
            const uint32_t sz = aux_size - orig_aux;
            if (has_MD < 0) {
                // the placeholder "MDZ" sits at -has_MD; the text was written at the end: rotate it into place (:1840-1861)
                const uint32_t at = (uint32_t)(-has_MD);
                if ((uint64_t)aux_size + sz > aux_cap) { err = ERR_SPACE; return -1; }
                W::sync();
                for (uint32_t i = 0; i < sz; i++) aux[aux_size + i] = aux[orig_aux + i];              // tmp copy past the end
                for (uint32_t i = orig_aux; i-- > at;) aux[i + sz] = aux[i];
                for (uint32_t i = 0; i < sz; i++) aux[at + i] = aux[aux_size + i];
                W::sync();
                if (-has_NM > -has_MD) has_NM -= (int)sz;
            }
            cr.aux_size += sz;
        }
        if (decode_nm) {
            if (has_NM == 0) {
                if (!aux_char('N') || !aux_char('M')) return -1;
                if (nm <= 0xff) { if (!aux_char('C') || !aux_char((uint8_t)nm)) return -1; cr.aux_size += 4; }
                else if (nm <= 0xffff) { if (!aux_char('S') || !aux_char((uint8_t)nm) || !aux_char((uint8_t)(nm >> 8))) return -1; cr.aux_size += 5; }
                else { if (!aux_char('I') || !aux_char((uint8_t)nm) || !aux_char((uint8_t)(nm >> 8)) || !aux_char((uint8_t)(nm >> 16)) || !aux_char((uint8_t)(nm >> 24))) return -1; cr.aux_size += 7; }
            } else {
                uint8_t *b = aux + (uint32_t)(-has_NM);
                b[0] = (uint8_t)nm; b[1] = (uint8_t)(nm >> 8); b[2] = (uint8_t)(nm >> 16); b[3] = (uint8_t)(nm >> 24);
            }
        }
        W::sync();
        return r ? -1 : 0;
    }

    CRAMREC_HD static int aux_ele_size(uint8_t t)
    {
        switch (t) { case 's': case 'S': return 2; case 'i': case 'I': case 'f': return 4; case 'd': return 8; default: return 1; }
    }

    // cram_decode_aux :2008-2137 (CRAM 3: no '*' placeholders)
    template <bool SUBSET>
    CRAMREC_HD int decode_aux(Rec &cr, int &has_MD, int &has_NM, uint32_t slice_ds)
    {
        const uint32_t ds = SUBSET ? slice_ds : CRAM_ALL;
        int32_t TL = 0;
        if (!(ds & (CRAM_TL | CRAM_aux))) { cr.aux = 0; cr.aux_size = 0; return 0; }
        if (T->ds[DS_TL].kind == K_NONE) return -1;
        if (get_int(T->ds[DS_TL], TL) || TL < 0 || (uint32_t)TL >= T->n_tl) return -1;
        const uint8_t *TN = P.td + P.tlidx[T->tl_off + TL];
        int ntags = 0;
        while (TN[ntags * 3] && TN[ntags * 3 + 1] && TN[ntags * 3 + 2]) ntags++;           // strlen / 3
        cr.aux_size = 0;
        cr.aux = aux_size;
        if (!(ds & CRAM_aux)) return 0;
        for (int i = 0; i < ntags; i++, TN += 3) {
            if (TN[0] == 'M' && TN[1] == 'D') has_MD = (int)(aux_size + 3) * (TN[2] == '*' ? -1 : 1);
            if (TN[0] == 'N' && TN[1] == 'M') has_NM = (int)(aux_size + 3) * (TN[2] == '*' ? -1 : 1);
            const uint32_t id = ((uint32_t)TN[0] << 16) | ((uint32_t)TN[1] << 8) | TN[2];
            int32_t m = -1;
            for (uint32_t k = 0; k < T->n_tags; k++) if (P.tagkeys[T->tag_off + k] == id) { m = (int32_t)k; break; }
            if (m < 0) return -1;
            if (!aux_char(TN[0]) || !aux_char(TN[1]) || !aux_char(TN[2])) return -1;
            const Codec &c = P.cpool[T->tag_codec_off + m];
            int32_t out_sz = 1;
            if (c.kind == K_BYTE_ARRAY_LEN || c.kind == K_BYTE_ARRAY_STOP) out_sz *= aux_ele_size(TN[2]);
            if (get_array_block(c, aux, aux_size, aux_cap, out_sz)) return -1;
            cr.aux_size += out_sz + 3;
            if (TN[0] == 'c' && TN[1] == 'F' && TN[2] == 'C' && out_sz == 1) {
                const uint8_t cF = aux[aux_size - 1];
                aux_size -= out_sz + 3;
                cr.aux_size -= out_sz + 3;
                if ((cF & 1) && has_MD == 0) has_MD = 1;
                if ((cF & 2) && has_NM == 0) has_NM = 1;
            }
            if (aux_size > (1u << 31)) return -1;
        }
        return 0;
    }

    // the record loop of cram_decode_slice :2554-2968.  recs: this slice's records.  returns 0 or an ERR_ code
    template <bool SUBSET>
    CRAMREC_HD int decode_slice(const Slice &S, Rec *recs, int32_t nrg, int32_t unknown_rg)
    {
        const uint32_t ds = SUBSET ? S.ds : CRAM_ALL;
        const int32_t req = SUBSET ? S.req : SAM_ALL;
        const Codec *C = T->ds;
        int64_t last_apos = S.ref_seq_start;                                // s->last_apos = s->hdr->ref_seq_start (cram_decode_slice_header)
        int32_t last_ref_id = -9;
        for (int32_t rec = 0; rec < S.n_records; rec++) {
            Rec cr;
            int32_t bf = 0, cf = 0, v = 0;
            int has_MD = 0, has_NM = 0;
            if (ds & CRAM_BF) {
                if (C[DS_BF].kind == K_NONE) return ERR_DECODE;
                if (get_int(C[DS_BF], bf) || bf < 0 || bf >= 0x1000) return ERR_DECODE;
            } else bf = BAM_FUNMAP;
            cr.flags = bf;
            if (ds & CRAM_CF) {
                if (C[DS_CF].kind == K_NONE) return ERR_DECODE;
                if (get_int(C[DS_CF], cf)) return ERR_DECODE;
            }
            cr.cram_flags = cf;
            cf &= 0xff;                                                     // `unsigned char cf` there
            if (S.ref_seq_id == -2 && !(ds & CRAM_RI)) cr.ref_id = -1;
            else if (S.ref_seq_id == -2) {
                if (C[DS_RI].kind == K_NONE) return ERR_DECODE;
                if (get_int(C[DS_RI], cr.ref_id)) return ERR_DECODE;
                if (cr.ref_id < -1 || cr.ref_id >= R.n_ref) return ERR_DECODE;
                if ((req & (SAM_SEQ | SAM_TLEN)) && cr.ref_id >= 0 && cr.ref_id != last_ref_id) {
                    if (!T->no_ref) {
                        if (!R.bases) return ERR_NOREF;
                        ref = R.bases + R.off[cr.ref_id];
                    }
                    ref_start = 1;
                    ref_end = (int64_t)(R.off ? R.off[cr.ref_id + 1] - R.off[cr.ref_id] : R.sq_len[cr.ref_id]);
                    last_ref_id = cr.ref_id;
                }
            } else cr.ref_id = S.ref_seq_id;
            if (cr.ref_id < -1 || cr.ref_id >= R.n_ref) return ERR_DECODE;

            cr.len = 0;
            if (ds & CRAM_RL) {
                if (C[DS_RL].kind == K_NONE) return ERR_DECODE;
                if (get_int(C[DS_RL], cr.len)) return ERR_DECODE;
                if (cr.len < 0) return ERR_DECODE;
            }

            if (ds & CRAM_AP) {
                if (C[DS_AP].kind == K_NONE) return ERR_DECODE;
                if (get_int(C[DS_AP], v)) return ERR_DECODE;
                cr.apos = v;
                if (T->ap_delta) cr.apos += last_apos;
                last_apos = cr.apos;
                if (S.ref_seq_id >= 0 && cr.apos < S.ref_seq_start) return ERR_DECODE;
            } else cr.apos = S.cont_ref_start;

            cr.rg = -1;
            if (ds & CRAM_RG) {
                if (C[DS_RG].kind == K_NONE) return ERR_DECODE;
                if (get_int(C[DS_RG], cr.rg)) return ERR_DECODE;
                if (cr.rg == unknown_rg) cr.rg = -1;
            }

            cr.name_len = 0;
            cr.name = name_size;
            if (T->read_names_included && (ds & CRAM_RN)) {
                int32_t sz = 1;
                if (C[DS_RN].kind == K_NONE) return ERR_DECODE;
                if (get_array_block(C[DS_RN], name, name_size, name_cap, sz)) return err ? err : ERR_DECODE;
                cr.name_len = (uint32_t)sz;
            }

            cr.mate_pos = 0; cr.mate_line = -1; cr.mate_ref_id = -1; cr.explicit_tlen = CRAMREC_I64_MIN;
            cr.mate_flags = 0; cr.tlen = CRAMREC_I64_MIN;
            // (cf is 0 when CF is not read, so these branches follow the reference's `(ds & CRAM_CF) && (cf & ...)`)
            if (cf & CRAM_FLAG_DETACHED) {
                if (ds & CRAM_MF) {
                    if (C[DS_MF].kind == K_NONE) return ERR_DECODE;
                    if (get_int(C[DS_MF], cr.mate_flags)) return ERR_DECODE;
                }
                if (!T->read_names_included) {
                    int32_t sz = 1;
                    cr.name = name_size;
                    if (ds & CRAM_RN) {
                        if (C[DS_RN].kind == K_NONE) return ERR_DECODE;
                        if (get_array_block(C[DS_RN], name, name_size, name_cap, sz)) return err ? err : ERR_DECODE;
                        cr.name_len = (uint32_t)sz;
                    }
                }
                if (ds & CRAM_NS) {
                    if (C[DS_NS].kind == K_NONE) return ERR_DECODE;
                    if (get_int(C[DS_NS], cr.mate_ref_id)) return ERR_DECODE;
                    if (cr.mate_ref_id < -1 || cr.mate_ref_id >= R.n_ref) return ERR_DECODE;
                }
                if (ds & CRAM_NP) {
                    if (C[DS_NP].kind == K_NONE) return ERR_DECODE;
                    if (get_int(C[DS_NP], v)) return ERR_DECODE;
                    cr.mate_pos = v;
                }
                if (ds & CRAM_TS) {
                    if (C[DS_TS].kind == K_NONE) return ERR_DECODE;
                    if (get_int(C[DS_TS], v)) return ERR_DECODE;
                    cr.tlen = v;
                }
            } else if (cf & CRAM_FLAG_MATE_DOWNSTREAM) {
                if (ds & CRAM_NF) {
                    if (C[DS_NF].kind == K_NONE) return ERR_DECODE;
                    if (get_int(C[DS_NF], cr.mate_line)) return ERR_DECODE;
                    cr.mate_line += rec + 1;
                }
                if ((cf & CRAM_FLAG_EXPLICIT_TLEN) && (ds & CRAM_TS)) {
                    if (C[DS_TS].kind == K_NONE) return ERR_DECODE;
                    if (get_int(C[DS_TS], v)) return ERR_DECODE;
                    cr.explicit_tlen = v;
                }
            } else if ((cf & CRAM_FLAG_EXPLICIT_TLEN) && (ds & CRAM_TS)) {
                if (C[DS_TS].kind == K_NONE) return ERR_DECODE;
                if (get_int(C[DS_TS], v)) return ERR_DECODE;
                cr.explicit_tlen = v;
            }

            cr.aux = aux_size; cr.aux_size = 0;
            if (decode_aux<SUBSET>(cr, has_MD, has_NM, ds)) return err ? err : ERR_DECODE;

            if ((uint64_t)sq_size + (uint32_t)cr.len > sq_cap) { CRAMREC_TRACE("seq full %u + %d > %u\n", sq_size, cr.len, sq_cap); return ERR_SPACE; }
            cr.seq = cr.qual = sq_size;
            uint8_t *seq = seqs + sq_size, *qual = quals + sq_size;
            sq_size += (uint32_t)cr.len;
            if (!ref) W::fill(seq, '=', (uint32_t)cr.len);

            cr.cigar = ncigar; cr.ncigar = 0;
            if (!(bf & BAM_FUNMAP)) {
                if ((ds & CRAM_AP) && cr.apos <= 0) return ERR_DECODE;
                if (ds & (CRAM_SEQ | CRAM_MQ)) {
                    if (decode_seq<SUBSET>(cr, cf, seq, qual, has_MD, has_NM, ds)) return err ? err : ERR_DECODE;
                } else { cr.cigar = 0; cr.ncigar = 0; cr.aend = cr.apos; cr.mqual = 0; }
            } else {
                cr.cigar = 0; cr.ncigar = 0; cr.aend = cr.apos; cr.mqual = 0;
                if ((ds & CRAM_BA) && cr.len) {
                    if (C[DS_BA].kind == K_NONE) return ERR_DECODE;
                    if (get_bytes(C[DS_BA], seq, cr.len)) return ERR_DECODE;
                }
                if (cf & CRAM_FLAG_PRESERVE_QUAL_SCORES) {
                    if (ds & CRAM_QS) {
                        if (C[DS_QS].kind == K_NONE) return ERR_DECODE;
                        if (get_bytes(C[DS_QS], qual, cr.len)) return ERR_DECODE;
                    }
                } else W::fill(qual, 255, (uint32_t)cr.len);
            }
            if (!T->qs_seq_orient && (ds & CRAM_QS) && (cr.flags & BAM_FREVERSE)) {
                W::sync();
                for (int32_t i = 0, j = cr.len - 1; i < j; i++, j--) { const uint8_t c = qual[i]; qual[i] = qual[j]; qual[j] = c; }
                W::sync();
            }
            recs[rec] = cr;
        }
        W::sync();
        return ERR_NONE;
    }
};

// cram_decode_slice_xref :2140-2304.  Serial over the slice's records.
CRAMREC_HD inline int slice_xref(Rec *crecs, int32_t n, int32_t req)
{
    if (!(req & (SAM_RNEXT | SAM_PNEXT | SAM_TLEN))) {
        for (int32_t rec = 0; rec < n; rec++) { crecs[rec].tlen = 0; crecs[rec].mate_pos = 0; crecs[rec].mate_ref_id = -1; }
        return 0;
    }
    for (int32_t rec = 0; rec < n; rec++) {
        Rec *cr = &crecs[rec];
        if (cr->mate_line >= 0) {
            if (cr->mate_line < n) {
                if (cr->tlen == CRAMREC_I64_MIN) {
                    int id1 = rec, id2 = rec;
                    int64_t aleft = cr->apos, aright = cr->aend, tlen;
                    int ref = cr->ref_id;
                    int left_cnt = 0, right_cnt = 0;
                    do {
                        if (aleft > crecs[id2].apos) aleft = crecs[id2].apos, left_cnt = 1;
                        else if (aleft == crecs[id2].apos) left_cnt++;
                        if (aright < crecs[id2].aend) { aright = crecs[id2].aend; right_cnt = 1; }
                        else if (aright == crecs[id2].aend) right_cnt++;
                        if (crecs[id2].mate_line == -1) { crecs[id2].mate_line = rec; break; }
                        if (crecs[id2].mate_line <= id2 || crecs[id2].mate_line >= n) return -1;
                        id2 = crecs[id2].mate_line;
                        if (crecs[id2].ref_id != ref) ref = -1;
                    } while (id2 != id1);
                    if (ref != -1) {
                        tlen = aright - aleft + 1;
                        id1 = id2 = rec;
                        if (crecs[id2].apos == aleft && (crecs[id2].aend < aright || left_cnt <= 1)) { crecs[id2].tlen = tlen; tlen = -tlen; }
                        else if (crecs[id2].apos == aleft && crecs[id2].aend == aright && left_cnt > 1 && right_cnt > 1) {
                            if (crecs[id2].flags & BAM_FREAD1) { crecs[id2].tlen = tlen; tlen = -tlen; }
                            else crecs[id2].tlen = -tlen;
                        } else crecs[id2].tlen = -tlen;
                        id2 = crecs[id2].mate_line;
                        while (id2 != id1) { crecs[id2].tlen = tlen; id2 = crecs[id2].mate_line; }
                    } else {
                        id1 = id2 = rec;
                        crecs[id2].tlen = 0;
                        id2 = crecs[id2].mate_line;
                        while (id2 != id1) { crecs[id2].tlen = 0; id2 = crecs[id2].mate_line; }
                    }
                }
                cr->mate_pos = crecs[cr->mate_line].apos;
                cr->mate_ref_id = crecs[cr->mate_line].ref_id;
                cr->flags |= BAM_FPAIRED;
                if (crecs[cr->mate_line].flags & BAM_FUNMAP) { cr->flags |= BAM_FMUNMAP; cr->tlen = 0; }
                if (cr->flags & BAM_FUNMAP) cr->tlen = 0;
                if (crecs[cr->mate_line].flags & BAM_FREVERSE) cr->flags |= BAM_FMREVERSE;
            }
        } else {
            if (cr->mate_flags & CRAM_M_REVERSE) cr->flags |= BAM_FPAIRED | BAM_FMREVERSE;
            if (cr->mate_flags & CRAM_M_UNMAP) cr->flags |= BAM_FMUNMAP;
            if (!(cr->flags & BAM_FPAIRED)) cr->mate_ref_id = -1;
        }
        if (cr->tlen == CRAMREC_I64_MIN) cr->tlen = 0;
    }
    for (int32_t rec = 0; rec < n; rec++) if (crecs[rec].explicit_tlen != CRAMREC_I64_MIN) crecs[rec].tlen = crecs[rec].explicit_tlen;
    return 0;
}

// ---- cram_to_bam :3100-3211 + bam_set1 sam.c:531-651 ----
struct BamCore { int64_t pos; int32_t tid; uint16_t bin; uint8_t qual, l_extranul; uint16_t flag, l_qname; uint32_t n_cigar; int32_t l_qseq, mtid; int64_t mpos, isize; };

CRAMREC_HD inline int reg2bin(int64_t beg, int64_t end)                   // hts_reg2bin(beg, end, 14, 5), hts.h:1516
{
    int l, s = 14, t = ((1 << 15) - 1) / 7;
    for (--end, l = 5; l > 0; --l, s += 3, t -= 1 << (l * 3))
        if (beg >> s == end >> s) return t + (int)(beg >> s);
    return 0;
}
CRAMREC_HD inline int count_digits(uint64_t v) { int n = 1; while (v >= 10) { v /= 10; n++; } return n; }

struct NameInfo { uint32_t len; int from_mate; uint64_t number; };        // how the QNAME of a record is made (from_mate 3: "?")
CRAMREC_HD inline NameInfo name_info(const Rec *crecs, int32_t n, int32_t rec, uint32_t prefix_len, int64_t record_counter)
{
    const Rec &cr = crecs[rec];
    NameInfo ni; ni.from_mate = 0; ni.number = 0;
    if (cr.name_len) { ni.len = cr.name_len; return ni; }
    if (cr.mate_line >= 0 && cr.mate_line < n && crecs[cr.mate_line].name_len > 0) { ni.from_mate = 1; ni.len = crecs[cr.mate_line].name_len; return ni; }
    ni.from_mate = 2;
    ni.number = (uint64_t)(record_counter + ((cr.mate_line >= 0 && cr.mate_line < rec) ? cr.mate_line : rec) + 1);
    ni.len = prefix_len + 1 + (uint32_t)count_digits(ni.number);
    return ni;
}

// cram_to_bam :3110-3166: QNAME is "?" without SAM_QNAME, SEQ "*" (length 0) without SAM_SEQ and SAM_QUAL
CRAMREC_HD inline uint32_t qname_len(const Rec *crecs, int32_t n, int32_t rec, uint32_t prefix_len, int64_t record_counter, int32_t req)
{
    return (req & SAM_QNAME) ? name_info(crecs, n, rec, prefix_len, record_counter).len : 1;
}
CRAMREC_HD inline int32_t bam_len(const Rec &cr, int32_t req) { return (req & (SAM_SEQ | SAM_QUAL)) ? cr.len : 0; }

// l_data of record `rec`, or -1 where cram_to_bam / bam_set1 fail
CRAMREC_HD inline int64_t bam_size(const Rec *crecs, int32_t n, int32_t rec, uint32_t prefix_len, int64_t record_counter,
                                   const uint32_t *rg_len, int32_t nrg, int32_t req)
{
    const Rec &cr = crecs[rec];
    if (cr.rg < -1 || cr.rg >= nrg) return -1;
    uint32_t lq = qname_len(crecs, n, rec, prefix_len, record_counter, req);
    if (lq == 0) lq = 1;
    if (lq > 254) return -1;
    const uint32_t nuls = 4 - lq % 4;
    const uint32_t rgl = cr.rg != -1 ? rg_len[cr.rg] + 4 : 0;
    const int64_t len = bam_len(cr, req);
    return (int64_t)lq + nuls + (int64_t)cr.ncigar * 4 + (len + 1) / 2 + len + cr.aux_size + rgl;
}

CRAMREC_HD inline uint8_t nt16_of(uint8_t c)                              // seq_nt16_table, hts.c
{
    switch (c) {
    case '=': return 0;
    case 'A': case 'a': case '0': return 1;
    case 'C': case 'c': case '1': return 2;
    case 'M': case 'm': return 3;
    case 'G': case 'g': case '2': return 4;
    case 'R': case 'r': return 5;
    case 'S': case 's': return 6;
    case 'V': case 'v': return 7;
    case 'T': case 't': case 'U': case 'u': case '3': return 8;
    case 'W': case 'w': return 9;
    case 'Y': case 'y': return 10;
    case 'H': case 'h': return 11;
    case 'K': case 'k': return 12;
    case 'D': case 'd': return 13;
    case 'B': case 'b': return 14;
    default: return 15;
    }
}

// Writes bam record `rec` (core + data) — W splits the byte loops across lanes.  Returns 0 / -1 (bam_set1's checks).
template <class W>
CRAMREC_HD inline int bam_fill(const Rec *crecs, int32_t n, int32_t rec, const uint8_t *prefix, uint32_t prefix_len, int64_t record_counter,
                               const uint8_t *name_blk, const uint8_t *seqs, const uint8_t *quals, const uint8_t *aux_blk, const uint32_t *cigars,
                               const uint8_t *rg_names, const uint32_t *rg_off, const uint32_t *rg_len, int32_t req, BamCore &core, uint8_t *data)
{
    const Rec &cr = crecs[rec];
    NameInfo ni = name_info(crecs, n, rec, prefix_len, record_counter);
    if (!(req & SAM_QNAME)) { ni.len = 1; ni.from_mate = 3; }
    const int32_t len = bam_len(cr, req);
    uint32_t lq = ni.len;
    const bool star = lq == 0;
    if (star) lq = 1;
    const uint32_t nuls = 4 - lq % 4;
    const uint32_t *cig = cigars + cr.cigar;
    int64_t rlen = 0, qlen = 0;
    if (!(cr.flags & BAM_FUNMAP)) {
        for (uint32_t k = 0; k < cr.ncigar; k++) {                         // bam_cigar2rqlens
            const uint32_t op = cig[k] & 15, l = cig[k] >> 4;
            const int type = (0x3C1A7 >> (op << 1)) & 3;                   // BAM_CIGAR_TYPE
            if (type & 1) qlen += l;
            if (type & 2) rlen += l;
        }
    }
    if (rlen == 0) rlen = 1;
    if (!(cr.flags & BAM_FUNMAP) && len > 0 && cr.ncigar == 0) return -1;
    if (!(cr.flags & BAM_FUNMAP) && len > 0 && len != qlen) return -1;
    core.pos = cr.apos - 1; core.tid = cr.ref_id; core.bin = (uint16_t)reg2bin(cr.apos - 1, cr.apos - 1 + rlen);
    core.qual = (uint8_t)cr.mqual; core.l_extranul = (uint8_t)(nuls - 1); core.flag = (uint16_t)cr.flags;
    core.l_qname = (uint16_t)(lq + nuls); core.n_cigar = cr.ncigar; core.l_qseq = len;
    core.mtid = cr.mate_ref_id; core.mpos = cr.mate_pos - 1; core.isize = cr.tlen;
    uint8_t *cp = data;
    if (star) cp[0] = '*';
    else if (ni.from_mate == 3) cp[0] = '?';
    else if (ni.from_mate == 0) W::copy(cp, name_blk + cr.name, lq);
    else if (ni.from_mate == 1) W::copy(cp, name_blk + crecs[cr.mate_line].name, lq);
    else {
        W::copy(cp, prefix, prefix_len);
        cp[prefix_len] = ':';
        uint64_t v = ni.number;
        for (uint32_t i = lq; i-- > prefix_len + 1;) { cp[i] = (uint8_t)('0' + v % 10); v /= 10; }
    }
    for (uint32_t i = 0; i < nuls; i++) cp[lq + i] = 0;
    cp += lq + nuls;
    W::copy(cp, reinterpret_cast<const uint8_t *>(cig), cr.ncigar * 4);
    cp += cr.ncigar * 4;
    const uint8_t *sq = seqs + cr.seq;
    W::pack_seq(cp, sq, (uint32_t)len);
    cp += (len + 1) / 2;
    if (req & SAM_QUAL) W::copy(cp, quals + cr.qual, (uint32_t)len);
    else W::fill(cp, 0xff, (uint32_t)len);
    cp += len;
    W::copy(cp, aux_blk + cr.aux, cr.aux_size);
    cp += cr.aux_size;
    if (cr.rg != -1) {
        cp[0] = 'R'; cp[1] = 'G'; cp[2] = 'Z';
        W::copy(cp + 3, rg_names + rg_off[cr.rg], rg_len[cr.rg]);
        cp[3 + rg_len[cr.rg]] = 0;
    }
    W::sync();
    return 0;
}

// ---- for passes of other files over the decoded records (cram_records.cu defines these; host code) ----
}  // namespace cramrec
#include <vector>
struct hgpu_ctx;
struct hgpu_cram_block;
namespace cramrec {

struct SliceRecs {                   // what cram_slice_decode_kernel left, for a pass of the caller's own
    const Rec *recs = nullptr;       // every slice's records, slice after slice: device memory (host memory in the hostsim build),
                                     // valid until the context stages its next call
    std::vector<uint64_t> rec0;      // per slice: its first record; rec0[n_slices] = every record
    std::vector<int32_t> status;     // per slice: 0 or the ERR_* of its decode
    std::vector<uint8_t> image;      // hostsim build: the memory behind recs
    float ms = 0;                    // device time of cram_slice_decode_kernel
};

// cram_slice_decode_kernel with the SAM_* mask req over the slices of a block list (as hgpu_cram_decode_records_fields_host
// takes it), no reference and no bam1_t fill.  HGPU_OK or the error code of the records entry points.
int slice_records(hgpu_ctx *ctx, const uint8_t *file, uint64_t file_len, const hgpu_cram_block *blocks, uint32_t n_blocks,
                  const uint8_t *udata, const uint64_t *udata_off, int32_t req, SliceRecs &out);
// cram_decode_compression_header accepts this uncompressed payload, as the record decoder reads it
bool compression_header_ok(const uint8_t *hdr, uint32_t len);

}  // namespace cramrec
