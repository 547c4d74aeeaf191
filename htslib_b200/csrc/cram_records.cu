// hgpu_cram_decode_records_host: every record of every slice of a CRAM 3.x image as bam1_t (core + data), decoded on
// the device from the uncompressed blocks — cram_decode_slice's record loop, cram_decode_slice_xref and cram_to_bam
// (cram/cram_decode.c:2340-3015, :2140-2304, :3100-3211) for a whole file at once.
//
// Host (framing, the control plane): SAM header text -> @SQ lengths / @RG ids; compression headers -> codec tables
// (cram_decode_compression_header :144-538 and the *_decode_init parsers of cram_codecs.c); slice headers -> block
// lists; arena sizes.  Device: cram_slice_decode_kernel, one warp per slice (cram_records.cuh: uniform scalar record
// loop, lane-parallel byte movement), then cram_bam_fill_kernel, one warp per record (QNAME, CIGAR, 4-bit SEQ, QUAL,
// aux, RG:Z into the bam1_t layout bam_set1 produces).  Slices the kernels cannot take (an encoding this table does
// not model, arena overflow, a reference that was not supplied) come back flagged, records empty, for the host library.
//
// Built a second time by tests/hostsim (g++ -DHGPU_HOSTSIM) with the kernels replaced by loops over the same
// __host__ __device__ code, so the record logic is checked against the reference without a GPU.  libhtsgpu.so never
// contains that variant.
#ifdef HGPU_HOSTSIM
#include "../../include/htsgpu.h"
#include <stdarg.h>
#include <stdio.h>
static char g_sim_err[256];
static void hgpu_set_error(const char *fmt, ...) { va_list ap; va_start(ap, fmt); vsnprintf(g_sim_err, sizeof g_sim_err, fmt, ap); va_end(ap); }
extern "C" const char *hostsim_last_error(void) { return g_sim_err; }
struct hgpu_ctx;
#else
#include "hgpu_internal.h"
#endif
#include "cram_records.cuh"
#include "stage_layout.h"
#include <map>
#include <string>
#include <vector>
#include <algorithm>
#include <stdlib.h>
#include <string.h>

using namespace cramrec;

#ifdef HGPU_HOSTSIM
#define hgpu_cram_records_free hostsim_cram_records_free
extern "C" void hgpu_cram_records_free(hgpu_cram_records *r);
// test hook: every record's cram_flags and mate_line as the record loop read them (before cram_decode_slice_xref
// closes the mate chains), of the last decode; -1 / -1 for records of a slice that failed
static std::vector<int32_t> g_rec_cram_flags, g_rec_mate_line;
extern "C" uint64_t hostsim_cram_record_mates(int32_t *cram_flags, int32_t *mate_line, uint64_t cap)
{
    const uint64_t n = g_rec_cram_flags.size();
    for (uint64_t i = 0; i < n && i < cap; i++) { cram_flags[i] = g_rec_cram_flags[i]; mate_line[i] = g_rec_mate_line[i]; }
    return n;
}
#endif
static_assert(sizeof(BamCore) == 48 && sizeof(hgpu_bam1_core) == 48, "bam1_core_t mirror");

namespace {

struct HRd {
    const uint8_t *p, *e;
    bool err = false;
    int32_t itf8()
    {
        if (p >= e) { err = true; return 0; }
        const uint8_t c = *p;
        const int n = c < 0x80 ? 0 : c < 0xc0 ? 1 : c < 0xe0 ? 2 : c < 0xf0 ? 3 : 4;
        if (e - p < n + 1) { err = true; p = e; return 0; }
        uint32_t v;
        switch (n) {
        case 0: v = c; break;
        case 1: v = ((c & 0x3fu) << 8) | p[1]; break;
        case 2: v = ((c & 0x1fu) << 16) | (p[1] << 8) | p[2]; break;
        case 3: v = ((c & 0x0fu) << 24) | (p[1] << 16) | (p[2] << 8) | p[3]; break;
        default: v = ((c & 0x0fu) << 28) | (p[1] << 20) | (p[2] << 12) | (p[3] << 4) | (p[4] & 0x0f); break;
        }
        p += n + 1;
        return (int32_t)v;
    }
};

// cram_dependent_data_series walks the series in this order (cram/cram_decode.c:559-564); bit i of a slice's data-series
// mask stands for series i here.  Index 27 (QQ) is therefore tested and set as 1 << 27, which is CRAM_BB_len, not CRAM_QQ:
// the reference's quirk, kept, so that exactly its blocks are selected.
const int k_i_to_id[28] = {DS_BF, DS_AP, DS_FP, DS_RL, DS_DL, DS_NF, DS_BA, DS_QS, DS_FC, DS_FN, DS_BS, DS_IN, DS_RG, DS_MQ,
                           DS_TL, DS_RN, DS_NS, DS_NP, DS_TS, DS_MF, DS_CF, DS_RI, DS_RS, DS_PD, DS_HC, DS_SC, DS_BB, DS_QQ};

struct BlockIds { int32_t id[2]; };              // cram_codec_to_id of one codec: -2 no block, -1 CORE, else a content id

struct SeriesBlocks {                            // per table: the blocks every series and tag codec reads
    BlockIds series[28]; uint8_t present[28];
    std::vector<BlockIds> tags;                  // every tag codec, a key defined twice included (the reference walks them all)
};

struct Build {                                   // pools shared by all tables of one call
    std::vector<Table> tables;
    std::vector<Codec> cpool;
    std::vector<HuffCode> hpool;
    std::vector<uint32_t> tagkeys, tlidx;
    std::vector<uint8_t> td;
    std::vector<std::map<int32_t, int32_t>> ext_of;      // per table: content id -> dense index
    std::vector<uint32_t> tl_max;                        // per table: longest tag line
    std::vector<uint8_t> usable;                         // per table: 0 = an encoding the device table does not model
    std::vector<SeriesBlocks> blocks_of;                 // per table
};

int32_t dense_ext(std::map<int32_t, int32_t> &m, int32_t id)
{
    auto it = m.find(id);
    if (it != m.end()) return it->second;
    const int32_t k = (int32_t)m.size();
    m[id] = k;
    return k;
}

// cram_decoder_init for one encoding.  0 ok, -1 the reference would reject the header, 1 not modelled on the device.
int parse_codec(Build &B, std::map<int32_t, int32_t> &ext, int32_t encoding, const uint8_t *data, int32_t size, uint8_t type, int depth, Codec &out)
{
    HRd r{data, data + size};
    memset(&out, 0, sizeof out);
    out.type = type;
    switch (encoding) {
    case 1: {                                                             // EXTERNAL :459-520
        if (size < 1) return -1;
        const int32_t id = r.itf8();
        if (r.err || r.p != r.e) return -1;
        out.kind = K_EXTERNAL; out.a = dense_ext(ext, id);
        return 0; }
    case 3: {                                                             // HUFFMAN :2814-2966
        if (type == T_BYTE_ARRAY_BLOCK) return -1;
        const int32_t n = r.itf8();
        if (r.err || n < 0 || n > size) return -1;
        std::vector<HuffCode> codes((size_t)n);
        for (int32_t i = 0; i < n; i++) codes[(size_t)i].symbol = r.itf8();
        if (r.err || r.itf8() != n) return -1;
        out.kind = K_HUFFMAN; out.ncodes = n; out.a = (int32_t)B.hpool.size();
        if (n == 0) return 0;
        int32_t max_len = 0;
        for (int32_t i = 0; i < n; i++) {
            const int32_t l = r.itf8();
            if (r.err || l < 0) return -1;
            codes[(size_t)i].len = l;
            if (l > max_len) max_len = l;
        }
        if (r.p != r.e || max_len >= n || max_len > 31) return -1;
        std::sort(codes.begin(), codes.end(), [](const HuffCode &x, const HuffCode &y) { return x.len != y.len ? x.len < y.len : x.symbol < y.symbol; });
        int32_t val = -1, last_len = 0;
        uint32_t max_val = 0;
        for (int32_t i = 0; i < n; i++) {                                 // canonical codes
            val++;
            if ((uint32_t)val > max_val) return -1;
            if (codes[(size_t)i].len > last_len) { val <<= (codes[(size_t)i].len - last_len); last_len = codes[(size_t)i].len; max_val = (1u << codes[(size_t)i].len) - 1; }
            codes[(size_t)i].code = val;
        }
        last_len = 0;
        for (int32_t i = 0, j = 0; i < n; i++) {
            if (codes[(size_t)i].len > last_len) { j = codes[(size_t)i].code - i; last_len = codes[(size_t)i].len; }
            codes[(size_t)i].p = j;
        }
        B.hpool.insert(B.hpool.end(), codes.begin(), codes.end());
        return 0; }
    case 4: {                                                             // BYTE_ARRAY_LEN :3428-3477
        if (depth > 4) return -1;
        Codec sub[2];
        for (int k = 0; k < 2; k++) {
            const int32_t enc = r.itf8(), sz = r.itf8();
            if (r.err || sz < 0 || r.e - r.p < sz) return -1;
            const int rc = parse_codec(B, ext, enc, r.p, sz, k == 0 ? (uint8_t)T_INT : type, depth + 1, sub[k]);
            if (rc) return rc;
            r.p += sz;
        }
        if (r.p != r.e) return -1;
        out.kind = K_BYTE_ARRAY_LEN;
        out.a = (int32_t)B.cpool.size(); B.cpool.push_back(sub[0]);
        out.b = (int32_t)B.cpool.size(); B.cpool.push_back(sub[1]);
        if (type == T_BYTE_ARRAY_BLOCK && sub[1].kind != K_EXTERNAL && sub[1].kind != K_BYTE_ARRAY_STOP) return 1;
        return 0; }
    case 5: {                                                             // BYTE_ARRAY_STOP :3682-3727
        if (size < 2) return -1;
        if (type != T_BYTE_ARRAY && type != T_BYTE_ARRAY_BLOCK) return -1;
        out.stop = *r.p++;
        const int32_t id = r.itf8();
        if (r.err || r.p != r.e) return -1;
        out.kind = K_BYTE_ARRAY_STOP; out.a = dense_ext(ext, id);
        return 0; }
    case 6: {                                                             // BETA :1142-1178
        if (type == T_BYTE_ARRAY_BLOCK) return -1;
        const int32_t off = r.itf8();
        const int32_t nbits = r.p < r.e ? r.itf8() : -1;
        if (r.err || r.p != r.e || nbits < 0 || nbits > 32) return -1;
        out.kind = K_BETA; out.a = off; out.b = nbits;
        return 0; }
    case 7: {                                                             // SUBEXP :2508-2540
        if (type != T_INT) return -1;
        const int32_t off = r.itf8(), k = r.itf8();
        if (r.err || r.p != r.e || k < 0) return -1;
        out.kind = K_SUBEXP; out.a = off; out.b = k;
        return k > 30 ? 1 : 0; }
    case 9: {                                                             // GAMMA :2580-2612
        if (type != T_INT) return -1;
        if (size < 1) return -1;
        const int32_t off = r.itf8();
        if (r.err || r.p != r.e) return -1;
        out.kind = K_GAMMA; out.a = off;
        return 0; }
    case 2: case 8:                                                       // GOLOMB / GOLOMB_RICE: the reference has no decoder for them either
        return -1;
    default:
        return -1;
    }
}

struct SeriesKey { const char *key; int ds; uint8_t type; };
const SeriesKey k_series[] = {
    {"BF", DS_BF, T_INT}, {"CF", DS_CF, T_INT}, {"RI", DS_RI, T_INT}, {"RL", DS_RL, T_INT}, {"AP", DS_AP, T_INT}, {"RG", DS_RG, T_INT},
    {"MF", DS_MF, T_INT}, {"NS", DS_NS, T_INT}, {"NP", DS_NP, T_INT}, {"TS", DS_TS, T_INT}, {"NF", DS_NF, T_INT}, {"FN", DS_FN, T_INT},
    {"FC", DS_FC, T_BYTE}, {"FP", DS_FP, T_INT}, {"BS", DS_BS, T_BYTE}, {"IN", DS_IN, T_BYTE_ARRAY}, {"SC", DS_SC, T_BYTE_ARRAY},
    {"DL", DS_DL, T_INT}, {"BA", DS_BA, T_BYTE}, {"BB", DS_BB, T_BYTE_ARRAY}, {"RS", DS_RS, T_INT}, {"PD", DS_PD, T_INT}, {"HC", DS_HC, T_INT},
    {"MQ", DS_MQ, T_INT}, {"RN", DS_RN, T_BYTE_ARRAY_BLOCK}, {"QS", DS_QS, T_BYTE}, {"QQ", DS_QQ, T_BYTE_ARRAY}, {"TL", DS_TL, T_INT}};

// cram_codec_to_id (cram/cram_codecs.c:3968-4016); content_id: dense external index -> content id
int32_t codec_block(const Build &B, const std::vector<int32_t> &content_id, const Codec &c, int32_t *id2)
{
    int32_t b1 = -2, b2 = -2;
    switch (c.kind) {
    case K_HUFFMAN: b1 = c.ncodes == 1 ? -2 : -1; break;
    case K_BETA: case K_SUBEXP: case K_GAMMA: b1 = -1; break;
    case K_EXTERNAL: case K_BYTE_ARRAY_STOP: b1 = content_id[(size_t)c.a]; break;
    case K_BYTE_ARRAY_LEN:
        b1 = codec_block(B, content_id, B.cpool[(size_t)c.a], nullptr);
        b2 = codec_block(B, content_id, B.cpool[(size_t)c.b], nullptr);
        break;
    default: break;
    }
    if (id2) *id2 = b2;
    return b1;
}
BlockIds codec_blocks(const Build &B, const std::vector<int32_t> &content_id, const Codec &c)
{
    BlockIds r;
    r.id[0] = codec_block(B, content_id, c, &r.id[1]);
    return r;
}

// cram_decode_compression_header :144-538.  0 ok (B.usable says whether the device can take it), -1 malformed.
int build_table(Build &B, const uint8_t *hdr, uint32_t len)
{
    Table T;
    std::vector<Codec> tc_all;
    memset(&T, 0, sizeof T);
    std::map<int32_t, int32_t> ext;
    uint8_t usable = 1;
    uint32_t tl_max = 0;
    T.ap_delta = 1; T.qs_seq_orient = 1;
    memcpy(T.sub, "CGTNAGTNACTNACGNACGT", 20);
    HRd r{hdr, hdr + len};
    {   // preservation map :210-344
        const int32_t msz = r.itf8();
        const uint8_t *start = r.p;
        const int32_t cnt = r.itf8();
        if (r.err || msz < 0 || cnt < 0) return -1;
        for (int32_t i = 0; i < cnt; i++) {
            if (r.e - r.p < 3) return -1;
            const uint8_t k0 = r.p[0], k1 = r.p[1];
            r.p += 2;
            if (k0 == 'R' && k1 == 'N') T.read_names_included = *r.p++;
            else if (k0 == 'A' && k1 == 'P') T.ap_delta = *r.p++;
            else if (k0 == 'R' && k1 == 'R') T.no_ref = !*r.p++;
            else if (k0 == 'Q' && k1 == 'O') T.qs_seq_orient = *r.p++;
            else if (k0 == 'S' && k1 == 'M') {
                if (r.e - r.p < 5) return -1;
                static const char order[5][5] = {"CGTN", "AGTN", "ACTN", "ACGN", "ACGT"};
                for (int row = 0; row < 5; row++)
                    for (int k = 0; k < 4; k++) T.sub[row][(r.p[row] >> (6 - 2 * k)) & 3] = (uint8_t)order[row][k];
                r.p += 5;
            } else if (k0 == 'T' && k1 == 'D') {                           // cram_decode_TD :70-137
                const int32_t bs = r.itf8();
                if (r.err || bs < 0 || r.e - r.p < bs) return -1;
                T.n_tl = 0; T.tl_off = (uint32_t)B.tlidx.size();
                if (bs) {
                    const uint32_t base = (uint32_t)B.td.size();
                    B.td.insert(B.td.end(), r.p, r.p + bs);
                    if (B.td.back()) B.td.push_back(0);
                    const uint32_t n = (uint32_t)B.td.size() - base;
                    for (uint32_t i = 0; i < n; i++) {
                        B.tlidx.push_back(base + i);
                        T.n_tl++;
                        const uint32_t s0 = i;
                        while (B.td[base + i]) i++;
                        if (i - s0 > tl_max) tl_max = i - s0;
                    }
                    B.td.push_back(0); B.td.push_back(0); B.td.push_back(0);   // the tag walk reads three bytes at a time
                    r.p += bs;
                }
            } else r.p++;                                                   // MI / UI / PI / unknown: one byte
        }
        if (r.p - start != msz) return -1;
    }
    {   // record encoding map :346-493
        const int32_t msz = r.itf8();
        const uint8_t *start = r.p;
        const int32_t cnt = r.itf8();
        if (r.err || msz < 0 || cnt < 0) return -1;
        for (int32_t i = 0; i < cnt; i++) {
            if (r.e - r.p < 4) return -1;
            const char k0 = (char)r.p[0], k1 = (char)r.p[1];
            r.p += 2;
            const int32_t enc = r.itf8(), sz = r.itf8();
            if (r.err) return -1;
            if (enc == 0) continue;
            if (sz < 0 || r.e - r.p < sz) return -1;
            for (const SeriesKey &s : k_series)
                if (s.key[0] == k0 && s.key[1] == k1) {
                    Codec c;
                    const int rc = parse_codec(B, ext, enc, r.p, sz, s.type, 0, c);
                    if (rc < 0) return -1;
                    if (rc > 0) usable = 0;
                    T.ds[s.ds] = c;
                }
            r.p += sz;
        }
        if (r.p - start != msz) return -1;
    }
    {   // tag encoding map :495-535
        const int32_t msz = r.itf8();
        const uint8_t *start = r.p;
        const int32_t cnt = r.itf8();
        if (r.err || msz < 0 || cnt < 0) return -1;
        T.tag_off = (uint32_t)B.tagkeys.size();
        std::vector<Codec> tc, tc_seen;
        for (int32_t i = 0; i < cnt; i++) {
            if (r.e - r.p < 6) return -1;
            const uint32_t key = (uint32_t)r.itf8();
            const int32_t enc = r.itf8(), sz = r.itf8();
            if (r.err || sz < 0 || r.e - r.p < sz) return -1;
            Codec c;
            const int rc = parse_codec(B, ext, enc, r.p, sz, T_BYTE_ARRAY_BLOCK, 0, c);
            if (rc < 0) return -1;
            if (rc > 0) usable = 0;
            r.p += sz;
            tc_seen.push_back(c);
            // map_find walks a list the parser prepended to: the LAST definition of a key is found first
            bool dup = false;
            for (size_t k = 0; k < tc.size(); k++) if (B.tagkeys[T.tag_off + k] == key) { tc[k] = c; dup = true; }
            if (!dup) { B.tagkeys.push_back(key); tc.push_back(c); }
        }
        if (r.err || r.p - start != msz) return -1;
        tc_all.swap(tc_seen);
        T.n_tags = (uint32_t)tc.size();
        T.tag_codec_off = (uint32_t)B.cpool.size();
        B.cpool.insert(B.cpool.end(), tc.begin(), tc.end());
    }
    T.n_ext = (uint32_t)ext.size();
    {
        std::vector<int32_t> content_id(ext.size());
        for (const auto &kv : ext) content_id[(size_t)kv.second] = kv.first;
        SeriesBlocks Q;
        for (int i = 0; i < 28; i++) {
            const Codec &c = T.ds[k_i_to_id[i]];
            Q.present[i] = c.kind != K_NONE;
            Q.series[i] = codec_blocks(B, content_id, c);
        }
        for (const Codec &c : tc_all) Q.tags.push_back(codec_blocks(B, content_id, c));
        B.blocks_of.push_back(Q);
    }
    B.tables.push_back(T);
    B.ext_of.push_back(ext);
    B.tl_max.push_back(tl_max);
    B.usable.push_back(usable);
    return 0;
}

bool subset_mode(int32_t req) { return req != 0 && req != SAM_ALL; }

// cram_dependent_data_series (cram/cram_decode.c:553-869) for one slice of table `table`: returns the slice's data-series
// mask and sets used[k] for its blocks sb[0 .. nb) (sb[0] is the CORE block, uncompressed whatever the mask, :618-620).  The
// embedded reference block is used too (:2412-2426).  Outside subset mode every block is used and every series read.
uint32_t select_series(const Build &B, int32_t table, int32_t req, const hgpu_cram_block *sb, int32_t nb, int32_t ref_id,
                       int32_t ref_base_id, uint8_t *used)
{
    if (!subset_mode(req)) { memset(used, 1, (size_t)nb); return CRAM_ALL; }
    const Table &T = B.tables[(size_t)table];
    const SeriesBlocks &Q = B.blocks_of[(size_t)table];
    uint32_t ds = 0;                                                        // :574-616
    if (req & SAM_QNAME) ds |= CRAM_RN;
    if (req & SAM_FLAG) ds |= CRAM_BF;
    if (req & SAM_RNAME) ds |= CRAM_RI | CRAM_BF;
    if (req & SAM_POS) ds |= CRAM_AP | CRAM_BF;
    if (req & SAM_MAPQ) ds |= CRAM_MQ;
    if (req & SAM_CIGAR) ds |= CRAM_CIGAR;
    if (req & SAM_RNEXT) ds |= CRAM_CF | CRAM_NF | CRAM_RI | CRAM_NS | CRAM_BF;
    if (req & SAM_PNEXT) ds |= CRAM_CF | CRAM_NF | CRAM_AP | CRAM_NP | CRAM_BF;
    if (req & SAM_TLEN) ds |= CRAM_CF | CRAM_NF | CRAM_AP | CRAM_TS | CRAM_BF | CRAM_MF | CRAM_RI | CRAM_CIGAR;
    if (req & SAM_SEQ) ds |= CRAM_SEQ;
    if (req & SAM_QUAL) ds |= CRAM_QUAL;
    if (req & SAM_AUX) ds |= CRAM_RG | CRAM_TL | CRAM_aux;
    if (req & SAM_RGAUX) ds |= CRAM_RG | CRAM_BF;

    memset(used, 0, (size_t)nb);
    bool core_used = false;
    auto mark = [&](int32_t id) {
        if (id == -1) core_used = true;
        else if (id >= 0) for (int32_t k = 0; k < nb; k++) if (sb[k].content_type == 4 && sb[k].content_id == id) used[k] = 1;
    };
    auto reads_used = [&](int32_t id) {
        if (id == -1) return core_used;
        for (int32_t k = 0; id >= 0 && k < nb; k++) if (sb[k].content_type == 4 && sb[k].content_id == id && used[k]) return true;
        return false;
    };
    // both blocks of a codec, as the reference's `for (;;)` over bnum1 / bnum2 visits them
    auto each = [](const BlockIds &b, auto &&f) { f(b.id[0]); if (b.id[1] != -2 && b.id[1] != b.id[0]) f(b.id[1]); };
    uint32_t orig;
    do {
        const uint32_t feat = CRAM_RS | CRAM_PD | CRAM_HC | CRAM_QS | CRAM_IN | CRAM_SC | CRAM_BS | CRAM_DL | CRAM_BA | CRAM_BB | CRAM_QQ;
        if (ds & feat) ds |= CRAM_FC | CRAM_FP;                            // :645-678
        if (ds & (CRAM_SEQ | CRAM_CIGAR)) ds |= CRAM_RL;
        if (ds & CRAM_FP) ds |= CRAM_FC;
        if (ds & CRAM_FC) ds |= CRAM_FN;
        if (ds & CRAM_aux) ds |= CRAM_TL;
        if (ds & CRAM_MF) ds |= CRAM_CF;
        if (ds & CRAM_MQ) ds |= CRAM_BF;
        if (ds & CRAM_BS) ds |= CRAM_RI;
        if (ds & (CRAM_MF | CRAM_NS | CRAM_NP | CRAM_TS | CRAM_NF)) ds |= CRAM_CF;
        if (!T.read_names_included && (ds & CRAM_RN)) ds |= CRAM_CF | CRAM_NF;
        if (ds & (CRAM_BA | CRAM_QS | CRAM_BB | CRAM_QQ)) ds |= CRAM_BF | CRAM_CF | CRAM_RL;
        if (ds & CRAM_FN) ds |= CRAM_SC | CRAM_IN | CRAM_BB;
        orig = ds;
        for (int i = 0; i < 28; i++)                                        // the blocks the series read (:683-723)
            if (((ds >> i) & 1) && Q.present[i]) each(Q.series[i], mark);
        if ((req & SAM_AUX) || (ds & CRAM_aux))                             // :726-773
            for (const BlockIds &b : Q.tags) each(b, mark);
        for (int i = 0; i < 28; i++)                                        // series sharing a used block join (:777-816)
            if (Q.present[i]) each(Q.series[i], [&](int32_t id) { if (reads_used(id)) ds |= 1u << i; });
        for (const BlockIds &b : Q.tags)                                    // :819-864: a tag on CORE always pulls the tags in
            each(b, [&](int32_t id) { if (id == -1 || reads_used(id)) ds |= CRAM_aux; });
    } while (orig != ds);
    if (nb > 0) used[0] = 1;
    if (ref_id >= 0 && ref_base_id >= 0)
        for (int32_t k = 0; k < nb; k++) if (sb[k].content_type == 4 && sb[k].content_id == ref_base_id) { used[k] = 1; break; }
    return ds;
}

struct HeaderInfo { std::vector<int64_t> sq_len; std::vector<std::string> rg; int32_t unknown_rg = -1; };

void parse_sam_header(const uint8_t *text, size_t len, HeaderInfo &H)
{
    size_t i = 0;
    while (i < len) {
        size_t e = i;
        while (e < len && text[e] != '\n') e++;
        if (e - i > 4 && text[i] == '@' && text[i + 3] == '\t') {
            const bool sq = text[i + 1] == 'S' && text[i + 2] == 'Q', rg = text[i + 1] == 'R' && text[i + 2] == 'G';
            if (sq || rg) {
                int64_t ln = 0; std::string id;
                size_t f = i + 4;
                while (f < e) {
                    size_t g = f;
                    while (g < e && text[g] != '\t') g++;
                    if (g - f > 3 && text[f + 2] == ':') {
                        if (sq && text[f] == 'L' && text[f + 1] == 'N') ln = strtoll(std::string((const char *)text + f + 3, g - f - 3).c_str(), nullptr, 10);
                        if (rg && text[f] == 'I' && text[f + 1] == 'D') id.assign((const char *)text + f + 3, g - f - 3);
                    }
                    f = g + 1;
                }
                if (sq) H.sq_len.push_back(ln); else H.rg.push_back(id);
            }
        }
        i = e + 1;
    }
    if (!H.rg.empty() && H.rg.back() == "UNKNOWN") H.unknown_rg = (int32_t)H.rg.size() - 1;
}

// ---- bulk-operation policies ----
struct HostW {
    static void copy(uint8_t *d, const uint8_t *s, uint32_t n) { if (n) memmove(d, s, n); }
    static void fill(uint8_t *d, uint8_t v, uint32_t n) { if (n) memset(d, v, n); }
    static uint32_t find(const uint8_t *p, uint32_t n, uint8_t stop) { for (uint32_t i = 0; i < n; i++) if (p[i] == stop) return i; return n; }
    static void sync() {}
    static void pack_seq(uint8_t *d, const uint8_t *s, uint32_t n)
    {
        for (uint32_t j = 0; j < (n + 1) / 2; j++) d[j] = (uint8_t)((nt16_of(s[2 * j]) << 4) | (2 * j + 1 < n ? nt16_of(s[2 * j + 1]) : 0));
    }
};

#ifndef HGPU_HOSTSIM
struct WarpW {
    static __device__ __forceinline__ void copy(uint8_t *d, const uint8_t *s, uint32_t n)
    {
        for (uint32_t i = threadIdx.x & 31; i < n; i += 32) d[i] = s[i];
        __syncwarp();
    }
    static __device__ __forceinline__ void fill(uint8_t *d, uint8_t v, uint32_t n)
    {
        for (uint32_t i = threadIdx.x & 31; i < n; i += 32) d[i] = v;
        __syncwarp();
    }
    static __device__ __forceinline__ uint32_t find(const uint8_t *p, uint32_t n, uint8_t stop)
    {
        const uint32_t lane = threadIdx.x & 31;
        for (uint32_t base = 0; base < n; base += 32) {
            const uint32_t i = base + lane;
            const uint32_t bal = __ballot_sync(0xffffffffu, i < n && p[i] == stop);
            if (bal) return base + (uint32_t)__ffs(bal) - 1u;
        }
        return n;
    }
    static __device__ __forceinline__ void sync() { __syncwarp(); }
    static __device__ __forceinline__ void pack_seq(uint8_t *d, const uint8_t *s, uint32_t n)
    {
        for (uint32_t j = threadIdx.x & 31; j < (n + 1) / 2; j += 32)
            d[j] = (uint8_t)((nt16_of(s[2 * j]) << 4) | (2 * j + 1 < n ? nt16_of(s[2 * j + 1]) : 0));
        __syncwarp();
    }
};
#endif

struct Args {                                   // everything the two kernels read, device pointers
    Pools P;
    const Slice *slices; uint32_t n_slices;
    Refs R;
    uint8_t *scratch;                           // arenas
    Rec *recs;
    uint32_t *rec_slice;                        // record -> slice
    uint64_t *local_off;                        // per record: offset of its data inside the slice's output
    uint64_t *slice_bytes;                      // per slice: total data bytes
    int32_t *slice_status;
    const uint8_t *rg_names; const uint32_t *rg_off, *rg_len; int32_t nrg, unknown_rg;
    const uint8_t *prefix; uint32_t prefix_len;
    int decode_md;
    // fill pass
    const uint64_t *slice_base;                 // exclusive prefix of slice_bytes
    BamCore *core; uint8_t *data; uint64_t *data_off; int32_t *rec_status;
    uint64_t n_records;
};

template <class W>
CRAMREC_HD void slice_body(const Args &A, uint32_t si, uint32_t lane, uint32_t nlanes)
{
    const Slice &S = A.slices[si];
    if (S.table < 0) {                                                       // flagged on the host: the records stay empty
        for (int32_t r = (int32_t)lane; r < S.n_records; r += (int32_t)nlanes) { A.local_off[S.rec0 + r] = 0; A.rec_slice[S.rec0 + r] = si; }
        if (lane == 0) { A.slice_bytes[si] = 0; A.slice_status[si] = HGPU_CRAM_UNSUPPORTED; }
        return;
    }
    SliceDec<W> D;
    D.P = A.P;
    D.T = A.P.tables + S.table;
    D.ext = A.P.ext + S.ext_off;
    D.cur = A.P.cur + S.ext_off;
#if defined(__CUDA_ARCH__)
    // every series read is table entry -> block descriptor -> cursor -> bytes, a chain of dependent loads: the first three
    // links live in shared memory (one warp per CTA), only the stream bytes come from L2 / HBM
    constexpr uint32_t SM_EXT = 96;
    __shared__ __align__(16) Table s_T;
    __shared__ __align__(16) Ext s_ext[SM_EXT];
    __shared__ uint32_t s_cur[SM_EXT];
    {
        const uint32_t *src = reinterpret_cast<const uint32_t *>(D.T);
        uint32_t *dst = reinterpret_cast<uint32_t *>(&s_T);
        for (uint32_t i = lane; i < sizeof(Table) / 4; i += 32) dst[i] = src[i];
        const uint32_t ne = D.T->n_ext + 1;
        if (ne <= SM_EXT) {
            for (uint32_t i = lane; i < ne; i += 32) { s_ext[i] = D.ext[i]; s_cur[i] = 0; }
            D.ext = s_ext; D.cur = s_cur;
        }
        __syncwarp();
        D.T = &s_T;
    }
#endif
    D.core = A.P.udata + S.core_off; D.csize = S.core_size; D.cbyte = 0; D.cbit = 7;
    D.name = A.scratch + S.name_off; D.name_size = 0; D.name_cap = S.name_cap;
    D.aux = A.scratch + S.aux_off; D.aux_size = 0; D.aux_cap = S.aux_cap;
    D.seqs = A.scratch + S.seq_off; D.quals = D.seqs + S.seq_cap; D.sq_size = 0; D.sq_cap = S.seq_cap;
    D.cigar = reinterpret_cast<uint32_t *>(A.scratch + S.cig_off); D.ncigar = 0; D.cig_cap = S.cig_cap;
    D.R = A.R;
    D.decode_md_opt = A.decode_md;
    D.err = 0;
    D.ref = nullptr; D.ref_start = 0; D.ref_end = 0;
    int rc = ERR_NONE;
    // reference for this slice (cram_decode_slice :2417-2470)
    if (S.ref_seq_id >= 0) {
        if (S.ref_base_ext >= 0) {
            const Ext e = D.ext[S.ref_base_ext];
            if (e.size == 0xffffffffu || (int64_t)S.ref_seq_span > (int64_t)e.size) rc = ERR_DECODE;
            D.ref = A.P.udata + e.off;
            D.ref_start = S.ref_seq_start;
            D.ref_end = (int64_t)S.ref_seq_start + S.ref_seq_span - 1;
        } else if (!D.T->no_ref && (S.req & SAM_SEQ)) {                  // without SEQ the reference is not fetched (:2439)
            if (!A.R.bases || S.ref_seq_id >= A.R.n_ref) rc = ERR_NOREF;
            else {
                const int64_t flen = (int64_t)(A.R.off[S.ref_seq_id + 1] - A.R.off[S.ref_seq_id]);
                D.ref_start = S.ref_seq_start < 0 ? 0 : S.ref_seq_start;
                D.ref = A.R.bases + A.R.off[S.ref_seq_id] + (D.ref_start - 1);
                D.ref_end = (int64_t)S.ref_seq_start + S.ref_seq_span - 1;
                if (D.ref_end > flen) D.ref_end = flen;
            }
        }
    }
    Rec *recs = A.recs + S.rec0;
    if (rc == ERR_NONE) rc = S.req == SAM_ALL ? D.template decode_slice<false>(S, recs, A.nrg, A.unknown_rg)
                                              : D.template decode_slice<true>(S, recs, A.nrg, A.unknown_rg);
    W::sync();
#ifdef HGPU_HOSTSIM
    if (rc == ERR_NONE)
        for (int32_t r = 0; r < S.n_records; r++) { g_rec_cram_flags[S.rec0 + r] = recs[r].cram_flags; g_rec_mate_line[S.rec0 + r] = recs[r].mate_line; }
#endif
    if (rc == ERR_NONE && slice_xref(recs, S.n_records, S.req)) rc = ERR_DECODE;      // every lane runs it on the same data, same stores
    W::sync();
    // sizes: lanes take records
    uint64_t run = 0;
    for (int32_t base = 0; base < S.n_records; base += (int32_t)nlanes) {
        const int32_t r = base + (int32_t)lane;
        int64_t sz = 0;
        if (r < S.n_records && rc == ERR_NONE) {
            sz = bam_size(recs, S.n_records, r, A.prefix_len, S.record_counter, A.rg_len, A.nrg, S.req);
            if (sz < 0) sz = 0;                                               // cram_to_bam fails on this record: flagged by the fill pass
        }
        uint64_t inc = (uint64_t)sz;
#if defined(__CUDA_ARCH__)
        for (int d = 1; d < 32; d <<= 1) { const uint64_t t = __shfl_up_sync(0xffffffffu, inc, d); if (lane >= (uint32_t)d) inc += t; }
        const uint64_t tot = __shfl_sync(0xffffffffu, inc, 31);
#else
        const uint64_t tot = inc;
#endif
        if (r < S.n_records) { A.local_off[S.rec0 + r] = run + inc - (uint64_t)sz; A.rec_slice[S.rec0 + r] = si; }
        run += tot;
    }
    if (lane == 0) { A.slice_bytes[si] = run; A.slice_status[si] = rc; }
}

template <class W>
CRAMREC_HD void fill_body(const Args &A, uint64_t g)
{
    const uint32_t si = A.rec_slice[g];
    const Slice &S = A.slices[si];
    const uint64_t off = A.slice_base[si] + A.local_off[g];
    A.data_off[g] = off;
    if (g + 1 == A.n_records) A.data_off[g + 1] = A.slice_base[A.n_slices];
    BamCore core;
    memset(&core, 0, sizeof core);
    int st = A.slice_status[si];
    if (st == ERR_NONE) {
        const Rec *recs = A.recs + S.rec0;
        const int32_t r = (int32_t)(g - S.rec0);
        if (bam_size(recs, S.n_records, r, A.prefix_len, S.record_counter, A.rg_len, A.nrg, S.req) < 0) st = ERR_DECODE;
        else if (bam_fill<W>(recs, S.n_records, r, A.prefix, A.prefix_len, S.record_counter, A.scratch + S.name_off, A.scratch + S.seq_off,
                             A.scratch + S.seq_off + S.seq_cap, A.scratch + S.aux_off, reinterpret_cast<const uint32_t *>(A.scratch + S.cig_off),
                             A.rg_names, A.rg_off, A.rg_len, S.req, core, A.data + off)) st = ERR_DECODE;
    }
    A.core[g] = core;
    A.rec_status[g] = st;
}

#ifndef HGPU_HOSTSIM
struct HgpuEvents {                                 // destroyed on every return path
    cudaEvent_t e[2]; int n = 0;
    bool make(int k) { for (; n < k; n++) if (cudaEventCreate(&e[n]) != cudaSuccess) return false; return true; }
    ~HgpuEvents() { for (int k = 0; k < n; k++) cudaEventDestroy(e[k]); }
};
float g_last_ms[2] = {0, 0};                    // device time of the two kernels of the last call (bench.py reads it)
__global__ void __launch_bounds__(32) cram_slice_decode_kernel(Args A)
{
    if (blockIdx.x < A.n_slices) slice_body<WarpW>(A, blockIdx.x, threadIdx.x & 31, 32);
}
__global__ void __launch_bounds__(128) cram_bam_fill_kernel(Args A)
{
    const uint64_t g = (uint64_t)blockIdx.x * 4 + (threadIdx.x >> 5);
    if (g < A.n_records) fill_body<WarpW>(A, g);
}
#endif

struct SliceRun {                                  // what decode_slices leaves for the pass after it
    std::vector<uint8_t> image;                    // HGPU_HOSTSIM: the device image (A points into it)
    Args A;
    std::vector<int32_t> sstat;                    // per slice: the ERR_* of the slice decode
    std::vector<uint64_t> sbytes;                  // per slice: bytes of its bam1_t data
    uint64_t n_records = 0;
    uint32_t ns = 0;
    float ms = 0;                                  // device time of cram_slice_decode_kernel
};

// The framing, the tables, the upload and cram_slice_decode_kernel: every slice's Rec array in device memory (R.A.recs),
// out->slice_status / slice_rec0 filled.  R.n_records == 0 when there is nothing to decode.
int decode_slices(hgpu_ctx *ctx, const uint8_t *file, uint64_t file_len, const hgpu_cram_block *blocks, uint32_t n_blocks,
                  const uint8_t *udata, const uint64_t *udata_off, const hgpu_cram_refs *refs, const char *name_prefix, int decode_md,
                  int32_t req, hgpu_cram_records *out, SliceRun &R)
{
#ifdef HGPU_HOSTSIM
    g_rec_cram_flags.clear(); g_rec_mate_line.clear();
#endif
    if (subset_mode(req) && !(req & SAM_AUX)) decode_md = 0;            // cram_decode.c:605-607
    // req == 0 reads every series like SAM_ALL, but cram_decode_slice_xref and cram_to_bam test the mask itself
    if (!file || !blocks || !udata || !udata_off || !out) { hgpu_set_error("cram records: null argument"); return HGPU_ERR_ARG; }
    memset(out, 0, sizeof *out);
    if (file_len < 26 || memcmp(file, "CRAM", 4) != 0 || file[4] != 3) { hgpu_set_error("cram records: CRAM 3.x only"); return HGPU_ERR_ARG; }
    // containers: bases per container sizes the sequence arenas
    const long nc = hgpu_cram_scan_containers(file, file_len, nullptr, 0, nullptr, 0);
    if (nc < 0) return HGPU_ERR_ARG;
    std::vector<hgpu_cram_container> conts((size_t)nc);
    hgpu_cram_scan_containers(file, file_len, conts.data(), nc, nullptr, 0);

    HeaderInfo H;
    Build B;
    std::vector<Slice> slices;
    std::vector<Ext> ext;
    std::vector<uint8_t> slice_ok;                         // 0: flagged before launch (table not usable)
    int32_t cur_table = -1;
    bool have_header = false;
    uint64_t n_records = 0;
    StageLayout scratch;                                   // per-slice arenas inside the scratch region
    uint64_t udata_end = 0;
    for (uint32_t i = 0; i < n_blocks; i++) udata_end = std::max<uint64_t>(udata_end, udata_off[i] + blocks[i].uncomp_size);
    const uint32_t prefix_len = name_prefix ? (uint32_t)strlen(name_prefix) : 0;
    std::vector<uint8_t> used;

    for (uint32_t i = 0; i < n_blocks; i++) {
        const hgpu_cram_block &b = blocks[i];
        const uint8_t *pay = udata + udata_off[i];
        if (b.content_type == 0 && !have_header) {                          // FILE_HEADER: int32 length + text
            if (b.uncomp_size >= 4) {
                uint32_t tl = pay[0] | pay[1] << 8 | pay[2] << 16 | (uint32_t)pay[3] << 24;
                if (tl > b.uncomp_size - 4) tl = b.uncomp_size - 4;
                parse_sam_header(pay + 4, tl, H);
            }
            have_header = true;
        } else if (b.content_type == 1) {                                    // COMPRESSION_HEADER
            if (build_table(B, pay, b.uncomp_size)) { hgpu_set_error("cram records: malformed compression header (block %u)", i); return HGPU_CRAM_ERR_DECODE; }
            cur_table = (int32_t)B.tables.size() - 1;
        } else if (b.content_type == 2) {                                    // MAPPED_SLICE header
            if (cur_table < 0) { hgpu_set_error("cram records: slice before any compression header"); return HGPU_CRAM_ERR_DECODE; }
            hgpu_cram_slice sh;
            std::vector<int32_t> ids(10000);
            if (hgpu_cram_parse_slice_header(pay, b.uncomp_size, 3, &sh, ids.data(), (long)ids.size()) < 0) return HGPU_CRAM_ERR_DECODE;
            if (sh.n_blocks < 1 || (uint64_t)i + (uint64_t)sh.n_blocks >= (uint64_t)n_blocks + 1 || sh.n_records < 0 || sh.n_records > 50000000) {   // (a slice holds ~10^4 records; the clamp keeps a corrupt count from sizing arrays)
                hgpu_set_error("cram records: slice header block count"); return HGPU_CRAM_ERR_DECODE;
            }
            const Table &T = B.tables[(size_t)cur_table];
            Slice S;
            memset(&S, 0, sizeof S);
            S.table = cur_table;
            S.ref_seq_id = sh.ref_id; S.ref_seq_start = sh.start; S.ref_seq_span = sh.span; S.n_records = sh.n_records;
            S.record_counter = sh.record_counter;
            S.ref_base_ext = -1;
            S.ext_off = (uint32_t)ext.size();
            ext.resize(ext.size() + T.n_ext + 1, Ext{0, 0xffffffffu, 0});
            const hgpu_cram_container &C = conts[b.container < (uint32_t)nc ? b.container : 0];
            used.resize((size_t)sh.n_blocks);
            S.ds = select_series(B, cur_table, req, blocks + i + 1, sh.n_blocks, sh.ref_id, sh.ref_base_id, used.data());
            S.req = req;
            S.cont_ref_start = C.start;
            bool have_core = false;
            uint64_t blk_bytes = 0;
            for (int32_t k = 1; k <= sh.n_blocks; k++) {
                const hgpu_cram_block &sb = blocks[i + (uint32_t)k];
                blk_bytes += sb.uncomp_size;
                if (sb.content_type == 5) {                                  // CORE
                    if (!have_core) { S.core_off = udata_off[i + (uint32_t)k]; S.core_size = sb.uncomp_size; have_core = true; }
                } else if (sb.content_type == 4) {                           // EXTERNAL
                    const Ext e{udata_off[i + (uint32_t)k], sb.uncomp_size, sb.method == 8 ? 1u : 0u};
                    auto it = B.ext_of[(size_t)cur_table].find(sb.content_id);
                    if (it != B.ext_of[(size_t)cur_table].end() && ext[S.ext_off + (uint32_t)it->second].size == 0xffffffffu)
                        ext[S.ext_off + (uint32_t)it->second] = e;          // cram_get_block_by_id: the first block with that id
                    if (sh.ref_base_id >= 0 && sb.content_id == sh.ref_base_id && S.ref_base_ext < 0) {
                        S.ref_base_ext = (int32_t)T.n_ext;
                        ext[S.ext_off + T.n_ext] = e;
                    }
                }
            }
            bool ok = B.usable[(size_t)cur_table] && have_core && blocks[i + 1].content_type == 5;
            if (sh.ref_base_id >= 0 && sh.ref_id >= 0 && S.ref_base_ext < 0) ok = false;
            // arenas
            const uint64_t nr = (uint64_t)S.n_records;
            // total read length of the slice: exact where RL is a byte stream of ITF8 values or a constant (what the writers
            // emit); the container header's base count otherwise (htslib itself miscounts it for multi-reference containers),
            // and when RL is not read (its block may not be uncompressed then)
            uint64_t bases = C.bases > 0 ? 2 * (uint64_t)C.bases + blk_bytes : blk_bytes;
            {
                const Codec &rl = T.ds[DS_RL];
                if (rl.kind == K_EXTERNAL && (S.ds & CRAM_RL) && ext[S.ext_off + (uint32_t)rl.a].size != 0xffffffffu) {
                    const Ext &e = ext[S.ext_off + (uint32_t)rl.a];
                    HRd rr{udata + e.off, udata + e.off + e.size};
                    uint64_t sum = 0;
                    for (uint64_t k = 0; k < nr && !rr.err; k++) { const int32_t v = rr.itf8(); if (v > 0) sum += (uint64_t)v; }
                    bases = sum;
                } else if (rl.kind == K_HUFFMAN && rl.ncodes == 1 && B.hpool[(size_t)rl.a].len == 0 && B.hpool[(size_t)rl.a].symbol >= 0)
                    bases = nr * (uint64_t)B.hpool[(size_t)rl.a].symbol;
            }
            if (bases > (1ull << 31)) { bases = 1ull << 31; }
            const Codec &fc = T.ds[DS_FC], &fp = T.ds[DS_FP];
            uint64_t feat = blk_bytes;
            if (fc.kind == K_EXTERNAL && ext[S.ext_off + (uint32_t)fc.a].size != 0xffffffffu) feat = ext[S.ext_off + (uint32_t)fc.a].size;
            else if (fp.kind == K_EXTERNAL && ext[S.ext_off + (uint32_t)fp.a].size != 0xffffffffu) feat = ext[S.ext_off + (uint32_t)fp.a].size;
            uint64_t name_cap = blk_bytes + 64, seq_cap = bases + 64;
            // MD text: at most two characters per base, plus the deleted reference bases — those lie inside the slice's span
            // (one span's worth per slice is provided for; a slice that needs more comes back HGPU_CRAM_ERR_SPACE)
            const uint64_t del_room = sh.ref_id >= 0 && sh.span > 0 ? 4 * (uint64_t)sh.span : (1u << 20);
            uint64_t aux_cap = blk_bytes + nr * ((uint64_t)B.tl_max[(size_t)cur_table] + 16) + 1024 + (decode_md ? 3 * bases + 64 * nr + del_room : 0);
            uint64_t cig_cap = 2 * feat + 4 * nr + 64;
            if (name_cap > 0xfffffff0ull || seq_cap > 0xfffffff0ull || aux_cap > 0xfffffff0ull || cig_cap > 0x3ffffff0ull) ok = false;
            S.rec0 = n_records;
            n_records += nr;
            if (ok) {
                S.name_off = scratch.seg(name_cap).off; S.name_cap = (uint32_t)name_cap;
                S.seq_off = scratch.seg(2 * seq_cap).off; S.seq_cap = (uint32_t)seq_cap;
                S.aux_off = scratch.seg(aux_cap).off; S.aux_cap = (uint32_t)aux_cap;
                S.cig_off = scratch.seg(4 * cig_cap).off; S.cig_cap = (uint32_t)cig_cap;
            }
            slices.push_back(S);
            slice_ok.push_back(ok ? 1 : 0);
            i += (uint32_t)sh.n_blocks;
        }
    }
    const uint32_t ns = (uint32_t)slices.size();
    const int32_t nref = (int32_t)H.sq_len.size();
    if (refs && refs->bases && refs->n_ref != nref) { hgpu_set_error("cram records: %d reference sequences given, the header has %d @SQ lines", refs->n_ref, nref); return HGPU_ERR_ARG; }
    std::vector<uint32_t> rg_off, rg_len;
    std::vector<uint8_t> rg_names;
    for (const std::string &s : H.rg) { rg_off.push_back((uint32_t)rg_names.size()); rg_len.push_back((uint32_t)s.size()); rg_names.insert(rg_names.end(), s.begin(), s.end()); }
    rg_names.push_back(0);
    if (rg_off.empty()) { rg_off.push_back(0); rg_len.push_back(0); }
    // sanitise_SQ_lines (cram_io.c:2693-2728): where the supplied reference has the sequence, its length replaces the header's LN
    if (refs && refs->bases)
        for (int32_t k = 0; k < nref; k++) { const int64_t fl = (int64_t)(refs->off[k + 1] - refs->off[k]); if (fl && fl != H.sq_len[(size_t)k]) H.sq_len[(size_t)k] = fl; }
    if (H.sq_len.empty()) H.sq_len.push_back(0);

    // host result arrays
    out->n_records = n_records; out->n_slices = ns;
    out->slice_status = (int32_t *)calloc(ns + 1, sizeof(int32_t));
    out->slice_rec0 = (uint64_t *)calloc((size_t)ns + 1, sizeof(uint64_t));
    if (!out->slice_status || !out->slice_rec0) { hgpu_cram_records_free(out); hgpu_set_error("out of host memory"); return HGPU_ERR_NOMEM; }
    for (uint32_t s = 0; s < ns; s++) out->slice_rec0[s] = slices[s].rec0;
    out->slice_rec0[ns] = n_records;
    if (ns == 0 || n_records == 0) return HGPU_OK;

    // one device image: [udata | refs | tables | pools | slices | ext | cur | scratch | recs | per-record arrays]
    const uint64_t ref_bytes = refs && refs->bases ? refs->off[nref] : 0;
    StageLayout L(16);
    const auto s_udata = L.seg(udata_end), s_ref = L.seg(ref_bytes), s_refoff = L.seg((size_t)(nref + 2) * 8), s_sqlen = L.seg((size_t)(nref + 1) * 8),
               s_tab = L.seg(B.tables.size() * sizeof(Table)), s_cp = L.seg(B.cpool.size() * sizeof(Codec)), s_hp = L.seg(B.hpool.size() * sizeof(HuffCode)),
               s_tk = L.seg(B.tagkeys.size() * 4), s_tl = L.seg(B.tlidx.size() * 4), s_td = L.seg(B.td.size() + 8), s_sl = L.seg((size_t)ns * sizeof(Slice)),
               s_ext = L.seg(ext.size() * sizeof(Ext)), s_cur = L.seg(ext.size() * 4), s_rgn = L.seg(rg_names.size()), s_rgo = L.seg(rg_off.size() * 4),
               s_rgl = L.seg(rg_len.size() * 4), s_pre = L.seg(prefix_len + 1), s_scr = L.seg(scratch.total), s_recs = L.seg(n_records * sizeof(Rec)),
               s_rsl = L.seg(n_records * 4), s_loff = L.seg(n_records * 8), s_sby = L.seg((size_t)ns * 8), s_sst = L.seg((size_t)ns * 4), s_sbase = L.seg((size_t)(ns + 1) * 8),
               s_core = L.seg(n_records * sizeof(BamCore)), s_doff = L.seg((n_records + 1) * 8), s_rst = L.seg(n_records * 4);
    for (uint32_t s = 0; s < ns; s++) if (!slice_ok[s]) slices[s].table = -1;      // the kernel skips these

#ifdef HGPU_HOSTSIM
    (void)ctx;
    R.image.assign(L.total, 0);
    L.base = R.image.data();
#define UP(seg, src, n) do { if (n) memcpy(L.at(seg), (src), (n)); } while (0)
#else
    if (!ctx) { hgpu_set_error("null context"); return HGPU_ERR_ARG; }
    if (cudaSetDevice(ctx->device) != cudaSuccess) return HGPU_ERR_CUDA;
    int rc0 = hgpu_stage_ensure(ctx, L);
    if (rc0) return rc0;
    cudaStream_t st = ctx->stream;
#define UP(seg, src, n) do { if (!rc0) rc0 = hgpu_h2d(L.at(seg), (src), (n), st); } while (0)
#endif
    std::vector<uint64_t> refoff((size_t)nref + 2, 0);
    if (ref_bytes) for (int32_t k = 0; k <= nref; k++) refoff[(size_t)k] = refs->off[k];
    UP(s_udata, udata, udata_end);
    UP(s_ref, refs ? refs->bases : nullptr, ref_bytes);
    UP(s_refoff, refoff.data(), refoff.size() * 8);
    UP(s_sqlen, H.sq_len.data(), H.sq_len.size() * 8);
    UP(s_tab, B.tables.data(), B.tables.size() * sizeof(Table));
    UP(s_cp, B.cpool.data(), B.cpool.size() * sizeof(Codec));
    UP(s_hp, B.hpool.data(), B.hpool.size() * sizeof(HuffCode));
    UP(s_tk, B.tagkeys.data(), B.tagkeys.size() * 4);
    UP(s_tl, B.tlidx.data(), B.tlidx.size() * 4);
    UP(s_td, B.td.data(), B.td.size());
    UP(s_sl, slices.data(), (size_t)ns * sizeof(Slice));
    UP(s_ext, ext.data(), ext.size() * sizeof(Ext));
    UP(s_rgn, rg_names.data(), rg_names.size());
    UP(s_rgo, rg_off.data(), rg_off.size() * 4);
    UP(s_rgl, rg_len.data(), rg_len.size() * 4);
    UP(s_pre, name_prefix ? name_prefix : "", prefix_len);

    Args &A = R.A;
    memset(&A, 0, sizeof A);
    A.P.tables = L.at<Table>(s_tab); A.P.cpool = L.at<Codec>(s_cp);
    A.P.hpool = L.at<HuffCode>(s_hp); A.P.tagkeys = L.at<uint32_t>(s_tk);
    A.P.tlidx = L.at<uint32_t>(s_tl); A.P.td = L.at(s_td);
    A.P.ext = L.at<Ext>(s_ext); A.P.cur = L.at<uint32_t>(s_cur); A.P.udata = L.at(s_udata);
    A.slices = L.at<Slice>(s_sl); A.n_slices = ns;
    A.R.bases = ref_bytes ? L.at(s_ref) : nullptr; A.R.off = L.at<uint64_t>(s_refoff);
    A.R.sq_len = L.at<int64_t>(s_sqlen); A.R.n_ref = nref;
    A.scratch = L.at(s_scr); A.recs = L.at<Rec>(s_recs); A.rec_slice = L.at<uint32_t>(s_rsl);
    A.local_off = L.at<uint64_t>(s_loff); A.slice_bytes = L.at<uint64_t>(s_sby);
    A.slice_status = L.at<int32_t>(s_sst);
    A.rg_names = L.at(s_rgn); A.rg_off = L.at<uint32_t>(s_rgo); A.rg_len = L.at<uint32_t>(s_rgl);
    A.nrg = (int32_t)H.rg.size(); A.unknown_rg = H.unknown_rg;
    A.prefix = L.at(s_pre); A.prefix_len = prefix_len;
    A.decode_md = decode_md;
    A.slice_base = L.at<uint64_t>(s_sbase);
    A.core = L.at<BamCore>(s_core); A.data_off = L.at<uint64_t>(s_doff);
    A.rec_status = L.at<int32_t>(s_rst); A.n_records = n_records;

    std::vector<uint64_t> &sbytes = R.sbytes;
    std::vector<int32_t> &sstat = R.sstat;
    sbytes.assign(ns, 0); sstat.assign(ns, 0);
#ifdef HGPU_HOSTSIM
    memset(L.at(s_cur), 0, ext.size() * 4);
    g_rec_cram_flags.assign(n_records, -1); g_rec_mate_line.assign(n_records, -1);
    for (uint32_t s = 0; s < ns; s++) slice_body<HostW>(A, s, 0, 1);
    memcpy(sbytes.data(), A.slice_bytes, (size_t)ns * 8);
    memcpy(sstat.data(), A.slice_status, (size_t)ns * 4);
#else
    if (rc0 || (rc0 = hgpu_memset(L.at(s_cur), 0, ext.size() * 4 + 4, st))) return rc0;
    HgpuEvents evs;
    if (!evs.make(2)) return HGPU_ERR_CUDA;
    cudaEventRecord(evs.e[0], st);
    cram_slice_decode_kernel<<<ns, 32, 0, st>>>(A);
    cudaEventRecord(evs.e[1], st);
    hgpu_count_launch();
    if (hgpu_check(cudaGetLastError(), "cram slice decode launch")) return HGPU_ERR_CUDA;
    if (hgpu_d2h(sbytes.data(), A.slice_bytes, (size_t)ns * 8, st) || hgpu_d2h(sstat.data(), A.slice_status, (size_t)ns * 4, st)) return HGPU_ERR_CUDA;
    if (hgpu_check(cudaStreamSynchronize(st), "cram slice decode")) return HGPU_ERR_CUDA;
    cudaEventElapsedTime(&R.ms, evs.e[0], evs.e[1]);
#endif
    for (uint32_t s = 0; s < ns; s++) out->slice_status[s] = sstat[s] == ERR_SPACE ? HGPU_CRAM_ERR_SPACE : sstat[s] == ERR_NOREF ? HGPU_CRAM_ERR_NOREF : sstat[s];
    R.ns = ns; R.n_records = n_records;
#undef UP
    return HGPU_OK;
}

// decode_slices, then cram_bam_fill_kernel: the records as bam1_t
int decode_impl(hgpu_ctx *ctx, const uint8_t *file, uint64_t file_len, const hgpu_cram_block *blocks, uint32_t n_blocks,
                const uint8_t *udata, const uint64_t *udata_off, const hgpu_cram_refs *refs, const char *name_prefix, int decode_md,
                int32_t req, hgpu_cram_records *out, hgpu_cram_records_dev *dev = nullptr)
{
    if (dev) memset(dev, 0, sizeof *dev);
    SliceRun R;
    int rc = decode_slices(ctx, file, file_len, blocks, n_blocks, udata, udata_off, refs, name_prefix, decode_md, req, out, R);
    if (rc) return rc;
    const uint64_t n_records = out->n_records;
    const uint32_t ns = (uint32_t)out->n_slices;
    if (!dev) {
        out->core = (hgpu_bam1_core *)calloc(n_records + 1, sizeof(hgpu_bam1_core));
        out->data_off = (uint64_t *)calloc(n_records + 1, sizeof(uint64_t));
        out->rec_status = (int32_t *)calloc(n_records + 1, sizeof(int32_t));
        if (!out->core || !out->data_off || !out->rec_status) { hgpu_cram_records_free(out); hgpu_set_error("out of host memory"); return HGPU_ERR_NOMEM; }
    }
    if (ns == 0 || n_records == 0) return HGPU_OK;
    Args &A = R.A;
    std::vector<uint64_t> sbase((size_t)ns + 1, 0);
    for (uint32_t s = 0; s < ns; s++) sbase[s + 1] = sbase[s] + (R.sstat[s] != 0 ? 0 : R.sbytes[s]);
    const uint64_t data_bytes = sbase[ns];
    out->data_bytes = data_bytes;
    if (!dev) out->data = (uint8_t *)malloc(data_bytes + 16);
    if (!dev && !out->data) { hgpu_cram_records_free(out); hgpu_set_error("out of host memory"); return HGPU_ERR_NOMEM; }

#ifdef HGPU_HOSTSIM
    (void)ctx;
    memcpy(const_cast<uint64_t *>(A.slice_base), sbase.data(), sbase.size() * 8);
    std::vector<uint8_t> dbuf(data_bytes + 16);
    A.data = dbuf.data();
    for (uint64_t g = 0; g < n_records; g++) fill_body<HostW>(A, g);
    memcpy(out->core, A.core, n_records * sizeof(BamCore));
    memcpy(out->data_off, A.data_off, (n_records + 1) * 8);
    memcpy(out->rec_status, A.rec_status, n_records * 4);
    memcpy(out->data, dbuf.data(), data_bytes);
#else
    // the record bytes go where the (now dead) uploads of this call's inputs cannot be: a second staging area
    int rc1 = hgpu_ensure_mrec(ctx, data_bytes + 256);            // (not d_bam: hgpu_sam_format_dev / hgpu_bam_pack_dev scan there)
    if (rc1) { hgpu_cram_records_free(out); return rc1; }
    A.data = ctx->d_mrec;
    cudaStream_t st = ctx->stream;
    HgpuEvents evs;
    if (!evs.make(2)) return HGPU_ERR_CUDA;
    if (hgpu_h2d(const_cast<uint64_t *>(A.slice_base), sbase.data(), sbase.size() * 8, st)) return HGPU_ERR_CUDA;
    cudaEventRecord(evs.e[0], st);
    cram_bam_fill_kernel<<<(unsigned)((n_records + 3) / 4), 128, 0, st>>>(A);
    cudaEventRecord(evs.e[1], st);
    hgpu_count_launch();
    if (hgpu_check(cudaGetLastError(), "cram bam fill launch")) return HGPU_ERR_CUDA;
    if (dev) {
        dev->n_records = n_records; dev->data_bytes = data_bytes;
        dev->d_core = reinterpret_cast<hgpu_bam1_core *>(A.core); dev->d_data = A.data; dev->d_data_off = A.data_off; dev->d_rec_status = A.rec_status;
    } else {
        if (hgpu_d2h(out->core, A.core, n_records * sizeof(BamCore), st) || hgpu_d2h(out->data_off, A.data_off, (n_records + 1) * 8, st) ||
            hgpu_d2h(out->rec_status, A.rec_status, n_records * 4, st) || hgpu_d2h(out->data, A.data, data_bytes, st)) return HGPU_ERR_CUDA;
    }
    if (hgpu_check(cudaStreamSynchronize(st), "cram bam fill")) return HGPU_ERR_CUDA;
    g_last_ms[0] = R.ms;
    cudaEventElapsedTime(&g_last_ms[1], evs.e[0], evs.e[1]);
#endif
    return HGPU_OK;
}

// hgpu_cram_required_blocks: the slice walk of decode_impl, header blocks only, with select_series per slice
long required_blocks(const hgpu_cram_block *blocks, uint32_t n_blocks, const uint8_t *udata, const uint64_t *udata_off, int32_t req, uint8_t *used)
{
    if (!blocks || !udata || !udata_off || !used) { hgpu_set_error("cram required blocks: null argument"); return -1; }
    const bool subset = subset_mode(req);
    for (uint32_t i = 0; i < n_blocks; i++) used[i] = !subset || blocks[i].content_type <= 2;
    if (!subset) return (long)n_blocks;
    Build B;
    int32_t cur_table = -1;
    std::vector<int32_t> ids(10000);
    for (uint32_t i = 0; i < n_blocks; i++) {
        const hgpu_cram_block &b = blocks[i];
        const uint8_t *pay = udata + udata_off[i];
        if (b.content_type == 1) {
            if (build_table(B, pay, b.uncomp_size)) { hgpu_set_error("cram required blocks: malformed compression header (block %u)", i); return -1; }
            cur_table = (int32_t)B.tables.size() - 1;
        } else if (b.content_type == 2) {
            hgpu_cram_slice sh;
            if (cur_table < 0 || hgpu_cram_parse_slice_header(pay, b.uncomp_size, 3, &sh, ids.data(), (long)ids.size()) < 0 ||
                sh.n_blocks < 1 || (uint64_t)i + (uint64_t)sh.n_blocks >= (uint64_t)n_blocks + 1) {
                hgpu_set_error("cram required blocks: malformed slice header (block %u)", i); return -1;
            }
            select_series(B, cur_table, req, blocks + i + 1, sh.n_blocks, sh.ref_id, sh.ref_base_id, used + i + 1);
            i += (uint32_t)sh.n_blocks;
        }
    }
    long n = 0;
    for (uint32_t i = 0; i < n_blocks; i++) n += used[i];
    return n;
}

}  // namespace

namespace cramrec {
int slice_records(hgpu_ctx *ctx, const uint8_t *file, uint64_t file_len, const hgpu_cram_block *blocks, uint32_t n_blocks,
                  const uint8_t *udata, const uint64_t *udata_off, int32_t req, SliceRecs &out)
{
    hgpu_cram_records r;
    memset(&r, 0, sizeof r);
    SliceRun R;
    const int rc = decode_slices(ctx, file, file_len, blocks, n_blocks, udata, udata_off, nullptr, nullptr, 0, req, &r, R);
    if (rc == HGPU_OK) {
        out.rec0.assign(r.slice_rec0, r.slice_rec0 + r.n_slices + 1);
        out.status = R.sstat;
        out.status.resize(r.n_slices, 0);
        out.recs = R.A.recs;
        out.image.swap(R.image);
        out.ms = R.ms;
    }
    hgpu_cram_records_free(&r);
    return rc;
}

bool compression_header_ok(const uint8_t *hdr, uint32_t len)
{
    Build B;
    return build_table(B, hdr, len) == 0;
}
}  // namespace cramrec

extern "C" void hgpu_cram_records_free(hgpu_cram_records *r)
{
    if (!r) return;
    free(r->core); free(r->data); free(r->data_off); free(r->rec_status); free(r->slice_status); free(r->slice_rec0);
    memset(r, 0, sizeof *r);
}

#ifdef HGPU_HOSTSIM
extern "C" int hostsim_cram_decode_records(const uint8_t *file, uint64_t file_len, const hgpu_cram_block *blocks, uint32_t n_blocks,
        const uint8_t *udata, const uint64_t *udata_off, const hgpu_cram_refs *refs, const char *name_prefix, int decode_md, hgpu_cram_records *out)
{
    try { return decode_impl(nullptr, file, file_len, blocks, n_blocks, udata, udata_off, refs, name_prefix, decode_md, SAM_ALL, out); }
    catch (...) { hgpu_set_error("internal error"); return HGPU_ERR_NOMEM; }
}
extern "C" int hostsim_cram_decode_records_fields(const uint8_t *file, uint64_t file_len, const hgpu_cram_block *blocks, uint32_t n_blocks,
        const uint8_t *udata, const uint64_t *udata_off, const hgpu_cram_refs *refs, const char *name_prefix, int decode_md,
        uint32_t required_fields, hgpu_cram_records *out)
{
    try { return decode_impl(nullptr, file, file_len, blocks, n_blocks, udata, udata_off, refs, name_prefix, decode_md, (int32_t)required_fields, out); }
    catch (...) { hgpu_set_error("internal error"); return HGPU_ERR_NOMEM; }
}
extern "C" long hostsim_cram_required_blocks(const hgpu_cram_block *blocks, uint32_t n_blocks, const uint8_t *udata, const uint64_t *udata_off,
        uint32_t required_fields, uint8_t *used)
{
    try { return required_blocks(blocks, n_blocks, udata, udata_off, (int32_t)required_fields, used); }
    catch (...) { hgpu_set_error("internal error"); return -1; }
}
#else
// scan + cram_uncompress_block + record decode: a CRAM file image in, bam1_t records out.  With a field subset the header
// blocks are uncompressed first, then only the blocks the selection uses: the others are neither uncompressed nor
// CRC-checked, as in the reference (the CRC check lives in cram_uncompress_block, cram_io.c:1585)
static int decode_file_impl(hgpu_ctx *ctx, const uint8_t *file, uint64_t file_len, const hgpu_cram_refs *refs, const char *name_prefix,
                            int decode_md, int32_t req, hgpu_cram_records *out)
{
    if (!out) { hgpu_set_error("cram file: null argument"); return HGPU_ERR_ARG; }
    memset(out, 0, sizeof *out);
    int maj = 0, mnr = 0;
    const long nb = hgpu_cram_scan_blocks(file, file_len, nullptr, 0, &maj, &mnr);
    if (nb < 0) return HGPU_ERR_ARG;
    std::vector<hgpu_cram_block> blocks((size_t)nb + 1);
    hgpu_cram_scan_blocks(file, file_len, blocks.data(), nb, &maj, &mnr);
    std::vector<uint64_t> off((size_t)nb + 1, 0);
    for (long i = 0; i < nb; i++) off[(size_t)i + 1] = off[(size_t)i] + (((uint64_t)blocks[(size_t)i].uncomp_size + 15) & ~15ull);
    std::vector<uint8_t> udata(off[(size_t)nb] + 16);
    // uncompress the blocks idx[0 .. n) (all of them when idx is null), block i to dst + dst_off[i].  The call writes back the
    // whole span between its first and last slot, so blocks uncompressed by an earlier call must not lie inside it.
    auto uncompress = [&](const uint32_t *idx, uint32_t n, uint8_t *dst, const uint64_t *dst_off) -> int {
        std::vector<hgpu_cram_block> sb;
        std::vector<uint64_t> so;
        if (idx) for (uint32_t k = 0; k < n; k++) { sb.push_back(blocks[idx[k]]); so.push_back(dst_off[idx[k]]); }
        if (n == 0) return HGPU_OK;
        std::vector<uint32_t> got((size_t)n + 1);
        std::vector<int32_t> st((size_t)n + 1);
        int rc = hgpu_cram_uncompress_blocks_host(ctx, file, file_len, idx ? sb.data() : blocks.data(), n, dst, idx ? so.data() : dst_off,
                                                  got.data(), st.data());
        if (rc) return rc;
        for (uint32_t k = 0; k < n; k++) {
            const uint32_t i = idx ? idx[k] : k;
            if (st[k] != HGPU_OK) { hgpu_set_error("cram file: block %u (method %d) did not uncompress: status %d", i, blocks[i].method, st[k]); return st[k]; }
        }
        return HGPU_OK;
    };
    int rc;
    if (!subset_mode(req)) {
        if ((rc = uncompress(nullptr, (uint32_t)nb, udata.data(), off.data()))) return rc;
    } else {
        // the header blocks into a buffer of their own (packed), the used blocks into the file layout, then the headers joined in
        std::vector<uint32_t> idx;
        std::vector<uint64_t> hoff((size_t)nb + 1, 0);
        uint64_t hbytes = 0;
        for (uint32_t i = 0; i < (uint32_t)nb; i++)
            if (blocks[i].content_type <= 2) { idx.push_back(i); hoff[i] = hbytes; hbytes += ((uint64_t)blocks[i].uncomp_size + 15) & ~15ull; }
        std::vector<uint8_t> hdata(hbytes + 16);
        if ((rc = uncompress(idx.data(), (uint32_t)idx.size(), hdata.data(), hoff.data()))) return rc;
        std::vector<uint8_t> used((size_t)nb + 1);
        if (required_blocks(blocks.data(), (uint32_t)nb, hdata.data(), hoff.data(), req, used.data()) < 0) return HGPU_CRAM_ERR_DECODE;
        std::vector<uint32_t> body;
        for (uint32_t i = 0; i < (uint32_t)nb; i++) if (used[i] && blocks[i].content_type > 2) body.push_back(i);
        if ((rc = uncompress(body.data(), (uint32_t)body.size(), udata.data(), off.data()))) return rc;
        for (uint32_t i : idx) memcpy(udata.data() + off[i], hdata.data() + hoff[i], blocks[i].uncomp_size);
    }
    return decode_impl(ctx, file, file_len, blocks.data(), (uint32_t)nb, udata.data(), off.data(), refs, name_prefix, decode_md, req, out);
}

extern "C" int hgpu_cram_decode_records_dev(hgpu_ctx *ctx, const uint8_t *file, uint64_t file_len, const hgpu_cram_block *blocks, uint32_t n_blocks,
        const uint8_t *udata, const uint64_t *udata_off, const hgpu_cram_refs *refs, const char *name_prefix, int decode_md,
        hgpu_cram_records *out, hgpu_cram_records_dev *dev)
{
    if (!dev) { hgpu_set_error("cram records: null argument"); return HGPU_ERR_ARG; }
    return hgpu_abi_call([&] { return decode_impl(ctx, file, file_len, blocks, n_blocks, udata, udata_off, refs, name_prefix, decode_md, SAM_ALL, out, dev); },
                         HGPU_ERR_NOMEM, HGPU_ERR_NOMEM);
}

extern "C" void hgpu_cram_records_last_ms(float *slice_decode_ms, float *bam_fill_ms)
{
    if (slice_decode_ms) *slice_decode_ms = g_last_ms[0];
    if (bam_fill_ms) *bam_fill_ms = g_last_ms[1];
}

extern "C" int hgpu_cram_decode_file_host(hgpu_ctx *ctx, const uint8_t *file, uint64_t file_len, const hgpu_cram_refs *refs,
                                          const char *name_prefix, int decode_md, hgpu_cram_records *out)
{
    return hgpu_abi_call([&] { return decode_file_impl(ctx, file, file_len, refs, name_prefix, decode_md, SAM_ALL, out); }, HGPU_ERR_NOMEM, HGPU_ERR_NOMEM);
}

extern "C" int hgpu_cram_decode_file_fields_host(hgpu_ctx *ctx, const uint8_t *file, uint64_t file_len, const hgpu_cram_refs *refs,
                                                 const char *name_prefix, int decode_md, uint32_t required_fields, hgpu_cram_records *out)
{
    return hgpu_abi_call([&] { return decode_file_impl(ctx, file, file_len, refs, name_prefix, decode_md, (int32_t)required_fields, out); },
                         HGPU_ERR_NOMEM, HGPU_ERR_NOMEM);
}

extern "C" int hgpu_cram_decode_records_host(hgpu_ctx *ctx, const uint8_t *file, uint64_t file_len, const hgpu_cram_block *blocks, uint32_t n_blocks,
        const uint8_t *udata, const uint64_t *udata_off, const hgpu_cram_refs *refs, const char *name_prefix, int decode_md, hgpu_cram_records *out)
{
    return hgpu_abi_call([&] { return decode_impl(ctx, file, file_len, blocks, n_blocks, udata, udata_off, refs, name_prefix, decode_md, SAM_ALL, out); },
                         HGPU_ERR_NOMEM, HGPU_ERR_NOMEM);
}

extern "C" int hgpu_cram_decode_records_fields_host(hgpu_ctx *ctx, const uint8_t *file, uint64_t file_len, const hgpu_cram_block *blocks,
        uint32_t n_blocks, const uint8_t *udata, const uint64_t *udata_off, const hgpu_cram_refs *refs, const char *name_prefix, int decode_md,
        uint32_t required_fields, hgpu_cram_records *out)
{
    return hgpu_abi_call([&] { return decode_impl(ctx, file, file_len, blocks, n_blocks, udata, udata_off, refs, name_prefix, decode_md,
                                                  (int32_t)required_fields, out); }, HGPU_ERR_NOMEM, HGPU_ERR_NOMEM);
}

extern "C" long hgpu_cram_required_blocks(const hgpu_cram_block *blocks, uint32_t n_blocks, const uint8_t *udata, const uint64_t *udata_off,
                                          uint32_t required_fields, uint8_t *used)
{
    return hgpu_abi_call([&] { return required_blocks(blocks, n_blocks, udata, udata_off, (int32_t)required_fields, used); }, -1L, -1L);
}
#endif
