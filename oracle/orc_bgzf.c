/*
 * ORACLE — TEST INFRASTRUCTURE ONLY (see orc_rans_nx16.c header for the usage rule).
 *
 * CPU restatement of the BGZF block decode path of htslib 1.23.1:
 *   check_header              bgzf.c:896-903
 *   inflate_block             bgzf.c:808-824
 *   bgzf_uncompress (zlib arm) bgzf.c:762-804   raw inflate (window -15), CRC32 of the output
 *   hts_crc32                 bgzf.c:620-622
 * The DEFLATE and CRC-32 arithmetic itself lives in zlib (system 1.3, unpinned by htslib),
 * which is not part of /root/reference; it is restated here from RFC 1951 / RFC 1952.
 * Parity status: PINNED — tests/test_oracle_bgzf.py checks this file against zlib itself on
 * seeded inputs (all block types, levels 0-9), against test/bgziptest.txt.gz and
 * test/bgzf_boundaries/*.bam, and against the compiled reference's bgzf_read.
 *
 * Decoding is done the slow, obviously-correct way: canonical codes walked one bit at a time.
 * orc_inflate_trace runs the same decode loop and also reports each block's type, header extent,
 * code lengths and tokens, so tests can check how an encoder built a block, not only what it holds.
 */
#include <stdint.h>
#include <string.h>

typedef struct {
    const uint8_t *src;
    uint64_t nbits, bitpos;      /* total bits available, next bit to read */
} bitsrc;

static int getbits(bitsrc *b, int n, uint32_t *v)
{
    uint32_t r = 0;
    int i;
    if (b->bitpos + (uint64_t)n > b->nbits) return -1;
    for (i = 0; i < n; i++, b->bitpos++)
        r |= (uint32_t)((b->src[b->bitpos >> 3] >> (b->bitpos & 7)) & 1) << i;
    *v = r;
    return 0;
}

typedef struct { uint16_t count[16], symbol[288]; } canon;

/* lengths -> canonical code description; returns 0 complete, >0 incomplete, <0 over-subscribed */
static int canon_build(canon *h, const uint8_t *len, int n)
{
    uint16_t offs[16];
    int i, left = 1;
    memset(h->count, 0, sizeof(h->count));
    for (i = 0; i < n; i++) h->count[len[i]]++;
    if (h->count[0] == n) return 0;
    for (i = 1; i < 16; i++) {
        left <<= 1;
        left -= h->count[i];
        if (left < 0) return left;
    }
    offs[1] = 0;
    for (i = 1; i < 15; i++) offs[i + 1] = offs[i] + h->count[i];
    for (i = 0; i < n; i++)
        if (len[i]) h->symbol[offs[len[i]]++] = (uint16_t)i;
    return left;
}

static int canon_decode(bitsrc *b, const canon *h)
{
    int code = 0, first = 0, index = 0, l;
    for (l = 1; l < 16; l++) {
        uint32_t bit;
        int cnt = h->count[l];
        if (getbits(b, 1, &bit)) return -1;
        code |= (int)bit;
        if (code - cnt < first) return h->symbol[index + (code - first)];
        index += cnt;
        first += cnt;
        first <<= 1;
        code <<= 1;
    }
    return -2;
}

static const uint16_t LEN_BASE[29] = {3,4,5,6,7,8,9,10,11,13,15,17,19,23,27,31,35,43,51,59,67,83,99,115,131,163,195,227,258};
static const uint8_t  LEN_XTRA[29] = {0,0,0,0,0,0,0,0,1,1,1,1,2,2,2,2,3,3,3,3,4,4,4,4,5,5,5,5,0};
static const uint16_t DST_BASE[30] = {1,2,3,4,5,7,9,13,17,25,33,49,65,97,129,193,257,385,513,769,1025,1537,2049,3073,4097,6145,8193,12289,16385,24577};
static const uint8_t  DST_XTRA[30] = {0,0,0,0,1,1,2,2,3,3,4,4,5,5,6,6,7,7,8,8,9,9,10,10,11,11,12,12,13,13};

/*
 * Optional sink of inflate_stream: what each deflate block said, as decoded.  The caller owns
 * every array; a block or token past max_blocks / max_toks makes the inflate fail.
 *   btype[k]      BFINAL | BTYPE << 1
 *   start_bit[k]  bit position of the block's BFINAL bit
 *   body_bit[k]   first bit after the block header (after LEN/NLEN for a stored block)
 *   end_bit[k]    first bit after the block (after the end-of-block code)
 *   first_tok[k]  index in toks[] of the block's first token (a stored block has none)
 *   lens[k*339..] lit/len[288], distance[32] and code-length[19] code lengths; zero beyond
 *                 HLIT / HDIST, the fixed lengths for BTYPE 1, all zero for a stored block
 *   toks[]        a literal byte, or 1<<31 | length << 16 | distance
 */
typedef struct {
    uint32_t max_blocks, max_toks, nblocks, ntoks;
    uint8_t *btype;
    uint64_t *start_bit, *body_bit, *end_bit;
    uint32_t *first_tok;
    uint8_t *lens;
    uint32_t *toks;
} orc_trace;

enum { TRACE_LENS = 288 + 32 + 19 };

static int trace_tok(orc_trace *t, uint32_t tok)
{
    if (t->ntoks >= t->max_toks) return -1;
    t->toks[t->ntoks++] = tok;
    return 0;
}

static int inflate_stream(const uint8_t *src, uint64_t slen, uint8_t *dst, uint64_t dcap,
                          uint64_t *dlen, uint64_t *consumed, orc_trace *t)
{
    bitsrc b = { src, slen * 8, 0 };
    uint64_t o = 0;
    uint32_t final, type;
    uint8_t *tl = 0;                                   /* this block's traced lengths */
    do {
        if (t) {
            if (t->nblocks >= t->max_blocks) return -1;
            t->start_bit[t->nblocks] = b.bitpos;
        }
        if (getbits(&b, 1, &final) || getbits(&b, 2, &type)) return -1;
        if (t) {
            tl = t->lens + (uint64_t)t->nblocks * TRACE_LENS;
            memset(tl, 0, TRACE_LENS);
            t->btype[t->nblocks] = (uint8_t)(final | type << 1);
            t->first_tok[t->nblocks] = t->ntoks;
        }
        if (type == 0) {
            uint32_t len, nlen;
            b.bitpos = (b.bitpos + 7) & ~7ull;
            if (getbits(&b, 16, &len) || getbits(&b, 16, &nlen)) return -1;
            if ((len ^ 0xffff) != nlen) return -1;
            if (b.bitpos + 8ull * len > b.nbits) return -1;
            if (o + len > dcap) return -1;
            if (t) t->body_bit[t->nblocks] = b.bitpos;
            memcpy(dst + o, src + (b.bitpos >> 3), len);
            o += len;
            b.bitpos += 8ull * len;
        } else if (type == 1 || type == 2) {
            canon lit, dist;
            uint8_t lens[320];
            int i;
            if (type == 1) {
                for (i = 0; i < 144; i++) lens[i] = 8;
                for (; i < 256; i++) lens[i] = 9;
                for (; i < 280; i++) lens[i] = 7;
                for (; i < 288; i++) lens[i] = 8;
                canon_build(&lit, lens, 288);
                for (i = 0; i < 30; i++) lens[i] = 5;
                canon_build(&dist, lens, 30);
            } else {
                static const uint8_t order[19] = {16,17,18,0,8,7,9,6,10,5,11,4,12,3,13,2,14,1,15};
                uint32_t hlit, hdist, hclen, v;
                canon cl;
                int n, err;
                if (getbits(&b, 5, &hlit) || getbits(&b, 5, &hdist) || getbits(&b, 4, &hclen)) return -1;
                hlit += 257; hdist += 1; hclen += 4;
                if (hlit > 286 || hdist > 30) return -1;
                memset(lens, 0, 19);
                for (i = 0; i < (int)hclen; i++) {
                    if (getbits(&b, 3, &v)) return -1;
                    lens[order[i]] = (uint8_t)v;
                }
                if (canon_build(&cl, lens, 19) != 0) return -1;       /* must be complete */
                if (t) memcpy(tl + 320, lens, 19);
                n = 0;
                while (n < (int)(hlit + hdist)) {
                    int sym = canon_decode(&b, &cl);
                    if (sym < 0) return -1;
                    if (sym < 16) lens[n++] = (uint8_t)sym;
                    else {
                        uint32_t rep; uint8_t val = 0;
                        if (sym == 16) {
                            if (n == 0) return -1;
                            val = lens[n - 1];
                            if (getbits(&b, 2, &rep)) return -1;
                            rep += 3;
                        } else if (sym == 17) { if (getbits(&b, 3, &rep)) return -1; rep += 3; }
                        else { if (getbits(&b, 7, &rep)) return -1; rep += 11; }
                        if (n + (int)rep > (int)(hlit + hdist)) return -1;
                        while (rep--) lens[n++] = val;
                    }
                }
                if (lens[256] == 0) return -1;                       /* no end-of-block code */
                {
                    uint8_t dl[32];
                    memcpy(dl, lens + hlit, hdist);
                    err = canon_build(&lit, lens, (int)hlit);
                    /* zlib inftrees.c: an incomplete set is accepted only when the longest
                     * code is 1 bit (a lone 1-bit code); over-subscribed sets never are */
                    if (err < 0 || (err > 0 && !(lit.count[1] == 1 && (int)hlit - lit.count[0] == 1))) return -1;
                    err = canon_build(&dist, dl, (int)hdist);
                    if (err < 0 || (err > 0 && !(dist.count[1] == 1 && (int)hdist - dist.count[0] == 1))) return -1;
                    if (t) { memcpy(tl, lens, hlit); memcpy(tl + 288, dl, hdist); }
                }
            }
            if (t) {
                if (type == 1) {
                    for (i = 0; i < 288; i++) tl[i] = i < 144 ? 8 : i < 256 ? 9 : i < 280 ? 7 : 8;
                    for (i = 0; i < 30; i++) tl[288 + i] = 5;
                }
                t->body_bit[t->nblocks] = b.bitpos;
            }
            for (;;) {
                int sym = canon_decode(&b, &lit);
                if (sym < 0) return -1;
                if (sym < 256) {
                    if (o >= dcap) return -1;
                    if (t && trace_tok(t, (uint32_t)sym)) return -1;
                    dst[o++] = (uint8_t)sym;
                } else if (sym == 256) break;
                else {
                    uint32_t xl, xd, len, d;
                    int ds;
                    sym -= 257;
                    if (sym >= 29) return -1;
                    if (getbits(&b, LEN_XTRA[sym], &xl)) return -1;
                    len = LEN_BASE[sym] + xl;
                    ds = canon_decode(&b, &dist);
                    if (ds < 0 || ds >= 30) return -1;
                    if (getbits(&b, DST_XTRA[ds], &xd)) return -1;
                    d = DST_BASE[ds] + xd;
                    if (d > o) return -1;
                    if (o + len > dcap) return -1;
                    if (t && trace_tok(t, 1u << 31 | len << 16 | d)) return -1;
                    while (len--) { dst[o] = dst[o - d]; o++; }
                }
            }
        } else
            return -1;
        if (t) t->end_bit[t->nblocks++] = b.bitpos;
    } while (!final);
    *dlen = o;
    if (consumed) *consumed = (b.bitpos + 7) >> 3;
    return 0;
}

/*
 * Raw inflate of one complete stream.  Returns 0 and *dlen on success; -1 on any error that
 * makes zlib's inflate(Z_FINISH) return something other than Z_STREAM_END (bad data, input
 * exhausted, output longer than dcap).  *consumed = bytes of src used (rounded up).
 */
int orc_inflate_raw(const uint8_t *src, uint64_t slen, uint8_t *dst, uint64_t dcap,
                    uint64_t *dlen, uint64_t *consumed)
{
    return inflate_stream(src, slen, dst, dcap, dlen, consumed, 0);
}

/* orc_inflate_raw that also reports every block's type, header extent, code lengths and tokens
 * into *t (nblocks / ntoks are reset here).  Same return value; -1 also when t runs out of room. */
int orc_inflate_trace(const uint8_t *src, uint64_t slen, uint8_t *dst, uint64_t dcap,
                      uint64_t *dlen, uint64_t *consumed, orc_trace *t)
{
    t->nblocks = t->ntoks = 0;
    return inflate_stream(src, slen, dst, dcap, dlen, consumed, t);
}

/* CRC-32 (IEEE 802.3, reflected 0xEDB88320), as zlib's crc32() / hts_crc32 (bgzf.c:620). */
uint32_t orc_crc32(uint32_t crc, const uint8_t *p, uint64_t n)
{
    static uint32_t T[256];
    static int ready;
    if (!ready) {
        uint32_t i, k;
        for (i = 0; i < 256; i++) {
            uint32_t c = i;
            for (k = 0; k < 8; k++) c = (c >> 1) ^ (0xEDB88320u & (0u - (c & 1)));
            T[i] = c;
        }
        ready = 1;
    }
    crc = ~crc;
    while (n--) crc = T[(crc ^ *p++) & 0xff] ^ (crc >> 8);
    return ~crc;
}

/* check_header, bgzf.c:896-903: 0 BGZF, -1 other gzip, -2 not gzip */
int orc_bgzf_check_header(const uint8_t *h)
{
    if (h[0] != 31 || h[1] != 139 || h[2] != 8) return -2;
    return ((h[3] & 4) && (h[10] | h[11] << 8) == 6 && h[12] == 'B' && h[13] == 'C'
            && (h[14] | h[15] << 8) == 2) ? 0 : -1;
}

/*
 * One whole BGZF block (header + deflate + footer, block_len = BSIZE+1 bytes) -> out (64 KiB).
 * Mirrors inflate_block: payload = block+18, length block_len-18 (the footer is left for the
 * inflater to ignore), capacity 65536, expected CRC = LE u32 at block_len-8.
 * Returns the inflated length, -1 for an inflate error (BGZF_ERR_ZLIB), -2 for a CRC mismatch
 * (BGZF_ERR_CRC), -3 for a bad header (BGZF_ERR_HEADER).
 */
int orc_bgzf_inflate_block(const uint8_t *block, uint32_t block_len, uint8_t *out)
{
    uint64_t dlen = 0;
    uint32_t want;
    if (block_len < 18 + 8 || orc_bgzf_check_header(block) != 0) return -3;
    if ((uint32_t)(block[16] | block[17] << 8) + 1 != block_len) return -3;
    want = block[block_len - 8] | block[block_len - 7] << 8 | block[block_len - 6] << 16
         | (uint32_t)block[block_len - 5] << 24;
    if (orc_inflate_raw(block + 18, block_len - 18, out, 65536, &dlen, 0)) return -1;
    if (orc_crc32(0, out, dlen) != want) return -2;
    return (int)dlen;
}

/*
 * Walk the BSIZE chain of a BGZF file image (bgzf_read_block's header logic, bgzf.c:1144-1205;
 * bgzf_mt_read_block :1485-1539).  Writes up to cap (offset,length) pairs; returns the number
 * of blocks, or -1 - (index of the bad block) when a header is invalid or a block is truncated.
 */
long orc_bgzf_scan(const uint8_t *file, uint64_t flen, uint64_t *off, uint32_t *len, long cap)
{
    uint64_t p = 0;
    long n = 0;
    while (p < flen) {
        uint32_t bl;
        if (flen - p < 18 || orc_bgzf_check_header(file + p) != 0) return -1 - n;
        bl = (uint32_t)(file[p + 16] | file[p + 17] << 8) + 1;
        if (bl < 18 || p + bl > flen) return -1 - n;
        if (n < cap) { off[n] = p; len[n] = bl; }
        n++;
        p += bl;
    }
    return n;
}
