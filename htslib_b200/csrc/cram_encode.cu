// hgpu_cram_encode_records_host: bam1_t records -> a complete CRAM 3.x file image — cram_encode_container /
// cram_encode_slice (cram/cram_encode.c:1950-2420), cram_encode_compression_header (:380-1030), cram_write_container and
// the file framing (cram_io.c:3958-4100, :4694, :4889, :5512), in the no-reference shape described in cram_encode.cuh.
//
// Device: cram_enc_count_kernel (one thread per record: bytes per series), cram_enc_scan_kernel (one warp per
// (slice, series): counts -> offsets), cram_enc_write_kernel (one thread per record: the bytes).  The series blocks are
// then compressed by the existing device encoders — the method trial of hgpu_cram_compress_blocks_host for every series
// (rANS Nx16 family for CRAM 3.1, rANS 4x8 for 3.0) and the tok3 encoder for read names (3.1) — and framed with the
// device CRC-32.  Host: the tag dictionary (one walk over the aux field headers), compression / slice / container headers.
// One slice per container; slices are independent, which is the axis that shards across GPUs.  With mate attachment
// the pairing kernels (cram_mate_key / group / scan / fill / resolve) run first and hand walk() each record's CF bits
// and NF (see cram_encode.cuh).
//
// Built a second time by tests/hostsim (-DHGPU_HOSTSIM): kernels -> loops, blocks stored RAW (the codecs are GPU-only);
// the reference must read that file back to the input records.  libhtsgpu.so never contains that variant.
#ifdef HGPU_HOSTSIM
#include "../../include/htsgpu.h"
#include <stdarg.h>
#include <stdio.h>
static char g_enc_err[256];
static void hgpu_set_error(const char *fmt, ...) { va_list ap; va_start(ap, fmt); vsnprintf(g_enc_err, sizeof g_enc_err, fmt, ap); va_end(ap); }
extern "C" const char *hostsim_enc_last_error(void) { return g_enc_err; }
struct hgpu_ctx;
#else
#include "hgpu_internal.h"
#endif
#include "cram_encode.cuh"
#include "stage_layout.h"
#include <map>
#include <set>
#include <string>
#include <vector>
#ifdef HGPU_HOSTSIM
static std::vector<uint8_t> g_mate_cf;             // the pairing pass's decisions of the last call with mate attachment
static std::vector<int32_t> g_mate_nf;
static std::vector<uint8_t> g_tag_drop;            // the tag pass's drop bits and the RG series values of the last call with tag blocks
static std::vector<int32_t> g_tag_rg;
#endif
#include <stdlib.h>
#include <string.h>

using namespace cramenc;

namespace {

static_assert(sizeof(Core) == 48 && sizeof(hgpu_bam1_core) == 48, "bam1_core_t mirror");
// tag keys (one series each) a call with tag blocks may hold: bounds the per-(slice, series) count array at
// (S_COUNT + 256) * 4 bytes per record
constexpr uint32_t k_max_tag_keys = 256;

uint32_t host_crc32(const uint8_t *p, size_t n, uint32_t crc = 0)         // container headers (a few dozen bytes each)
{
    static uint32_t tab[256];
    static bool init = false;
    if (!init) { for (uint32_t i = 0; i < 256; i++) { uint32_t c = i; for (int k = 0; k < 8; k++) c = (c & 1) ? (c >> 1) ^ 0xEDB88320u : c >> 1; tab[i] = c; } init = true; }
    crc = ~crc;
    for (size_t i = 0; i < n; i++) crc = tab[(crc ^ p[i]) & 0xff] ^ (crc >> 8);
    return ~crc;
}

struct Buf {
    std::vector<uint8_t> v;
    void u8(uint8_t b) { v.push_back(b); }
    void itf8(int32_t x) { uint8_t t[5]; const int n = itf8_put(t, (uint32_t)x); v.insert(v.end(), t, t + n); }
    void ltf8(int64_t x)                                                   // ltf8_put, cram/cram_io.c
    {
        const uint64_t u = (uint64_t)x;
        int n = 0;
        while (n < 8 && (u >> (7 * (n + 1))) != 0) n++;                    // n extra bytes: value < 2^(7 (n + 1)), 9 bytes for 64 bits
        if (n == 8) { v.push_back(0xff); for (int k = 7; k >= 0; k--) v.push_back((uint8_t)(u >> (8 * k))); return; }
        v.push_back((uint8_t)((0xff00u >> n) & 0xff) | (uint8_t)(u >> (8 * n)));
        for (int k = n - 1; k >= 0; k--) v.push_back((uint8_t)(u >> (8 * k)));
    }
    void le32(uint32_t x) { for (int k = 0; k < 4; k++) v.push_back((uint8_t)(x >> (8 * k))); }
    void bytes(const void *p, size_t n) { v.insert(v.end(), (const uint8_t *)p, (const uint8_t *)p + n); }
};

// one block, cram_write_block's layout (cram_io.c:1511-1563); crc = CRC-32 of everything before it
void frame_block(Buf &o, int method, int ctype, int32_t cid, const uint8_t *payload, uint32_t comp, uint32_t uncomp)
{
    const size_t at = o.v.size();
    o.u8((uint8_t)method); o.u8((uint8_t)ctype); o.itf8(cid); o.itf8((int32_t)comp); o.itf8((int32_t)uncomp);
    o.bytes(payload, comp);
    o.le32(host_crc32(o.v.data() + at, o.v.size() - at));
}

const char *const k_keys[S_COUNT] = {"BF", "CF", "RI", "RL", "AP", "RG", "RN", "MF", "NS", "NP", "TS", "TL", "FN", "FC", "FP", "DL", "RS", "HC", "PD",
                                     nullptr, "BB", nullptr, "SC", nullptr, "IN", "BA", "QS", "MQ", nullptr, nullptr, "BS", "NF"};

void enc_external(Buf &o, int id) { o.itf8(1); Buf t; t.itf8(id); o.itf8((int32_t)t.v.size()); o.bytes(t.v.data(), t.v.size()); }
void enc_byte_array_len(Buf &o, int len_id, int val_id)
{
    Buf t;
    enc_external(t, len_id);
    enc_external(t, val_id);
    o.itf8(4); o.itf8((int32_t)t.v.size()); o.bytes(t.v.data(), t.v.size());
}

// cram_encode_compression_header :380-1030 for this writer's fixed layout
void compression_header(Buf &o, const std::vector<std::string> &tag_lines, const std::vector<uint32_t> &tag_keys, bool ref_required, bool attach,
                        bool tag_blocks)
{
    Buf pm;                                                                // preservation map
    pm.itf8(5);
    pm.u8('R'); pm.u8('N'); pm.u8(1);
    pm.u8('A'); pm.u8('P'); pm.u8(0);
    pm.u8('R'); pm.u8('R'); pm.u8(ref_required ? 1 : 0);
    pm.u8('S'); pm.u8('M'); { const uint8_t sm[5] = {0x1b, 0x1b, 0x1b, 0x1b, 0x1b}; pm.bytes(sm, 5); }   // the default matrix (:165): CGTN AGTN ACTN ACGN ACGT
    pm.u8('T'); pm.u8('D');
    { Buf td; for (const std::string &l : tag_lines) { td.bytes(l.data(), l.size()); td.u8(0); } if (tag_lines.empty()) td.u8(0);
      pm.itf8((int32_t)td.v.size()); pm.bytes(td.v.data(), td.v.size()); }
    o.itf8((int32_t)pm.v.size()); o.bytes(pm.v.data(), pm.v.size());
    Buf rm;                                                                // record encoding map
    int cnt = 0;
    Buf body;
    for (int s = 0; s < S_COUNT; s++) {
        if (!k_keys[s] || (s == S_NF && !attach)) continue;
        body.u8((uint8_t)k_keys[s][0]); body.u8((uint8_t)k_keys[s][1]);
        if (s == S_RN) { body.itf8(5); Buf t; t.u8(0); t.itf8(s + 1); body.itf8((int32_t)t.v.size()); body.bytes(t.v.data(), t.v.size()); }
        else if (s == S_BB || s == S_SC || s == S_IN) enc_byte_array_len(body, s, s + 1);              // the length stream sits just before its value stream
        else enc_external(body, s + 1);
        cnt++;
    }
    rm.itf8(cnt); rm.bytes(body.v.data(), body.v.size());
    o.itf8((int32_t)rm.v.size()); o.bytes(rm.v.data(), rm.v.size());
    Buf tm;                                                                // tag encoding map
    tm.itf8((int32_t)tag_keys.size());
    for (uint32_t k : tag_keys) {
        tm.itf8((int32_t)k);
        if (!tag_blocks) { enc_byte_array_len(tm, S_TAG_LEN + 1, S_TAG_VAL + 1); continue; }
        // the codec cram_encode_aux gives each type (:2931-3033, CRAM 3.x); the key is the block's content id
        const uint8_t t = (uint8_t)k;
        if (t == 'Z' || t == 'H') { Buf a; a.u8('\t'); a.itf8((int32_t)k); tm.itf8(5); tm.itf8((int32_t)a.v.size()); tm.bytes(a.v.data(), a.v.size()); }
        else if (t == 'B') enc_byte_array_len(tm, (int)k, (int)k);
        else {                                                             // HUFFMAN with the value size as its only symbol
            Buf h; h.itf8(1); h.itf8(t == 's' || t == 'S' ? 2 : t == 'i' || t == 'I' || t == 'f' ? 4 : 1); h.itf8(1); h.itf8(0);
            Buf a; a.itf8(3); a.itf8((int32_t)h.v.size()); a.bytes(h.v.data(), h.v.size());
            enc_external(a, (int)k);
            tm.itf8(4); tm.itf8((int32_t)a.v.size()); tm.bytes(a.v.data(), a.v.size());
        }
    }
    o.itf8((int32_t)tm.v.size()); o.bytes(tm.v.data(), tm.v.size());
}

struct EArgs {
    const Core *core; const uint8_t *data; const uint64_t *data_off; const int32_t *tl;
    const uint8_t *ref_bases; const uint64_t *ref_off; int32_t n_ref;      // reference sequences (ref_bases == nullptr: the no-reference shape)
    uint64_t n; uint32_t rps;               // records, records per slice
    uint32_t *cnt;                          // [slice][stream][rps]: counts, then exclusive offsets
    uint32_t *tot;                          // [slice][stream]
    const uint64_t *base;                   // [slice][stream] -> byte offset in arena
    uint8_t *arena;
    int32_t *status;                        // per record
    const uint8_t *mate_cf;                 // per record: the pairing pass's CF bits (nullptr: every record detached)
    const int32_t *mate_nf;                 // per record: NF of MATE_DOWNSTREAM records
    uint32_t R;                             // series per slice: S_COUNT, + one per tag key with tag blocks
    const uint32_t *tkeys; uint32_t ntk;    // tag blocks: the call's tag keys, sorted (stream S_COUNT + k); nullptr: shared streams
    const uint8_t *tdrop;                   // per record: the tag pass's TAG_DROP_* bits (nullptr: nothing dropped)
    const int32_t *rg;                      // per record: RG series value, >= 0 when its RG:Z leaves the tag line
};

CRAMREC_HD inline TagRec tag_rec(const EArgs &A, uint64_t g)
{
    TagRec T{A.tkeys, A.ntk, 0u, -1};
    if (A.tkeys) { T.drop = A.tdrop ? A.tdrop[g] : 0u; T.rg = A.rg[g]; }
    return T;
}

// the tag pass: TAG_DROP_* bits of every record, against its own reference sequence (reference-coded shape only)
struct TArgs { const Core *core; const uint8_t *data; const uint64_t *data_off; const uint8_t *ref_bases; const uint64_t *ref_off; int32_t n_ref; uint64_t n; uint8_t *drop; };
CRAMREC_HD inline void tags_body(const TArgs &A, uint64_t g)
{
    const int32_t t = A.core[g].tid;
    const bool has = t >= 0 && t < A.n_ref;
    A.drop[g] = (uint8_t)tag_rules(A.core[g], A.data + A.data_off[g], (uint32_t)(A.data_off[g + 1] - A.data_off[g]),
                                   has ? A.ref_bases + A.ref_off[t] : nullptr, has ? (int64_t)(A.ref_off[t + 1] - A.ref_off[t]) : 0);
}

// the pairing pass: key (hash, aend) -> group (open-addressing name table per slice) -> scan of the group sizes ->
// member lists -> resolve (one thread per group replays process_one_read's rule in record order)
struct PArgs {
    const Core *core; const uint8_t *data; const uint64_t *data_off;
    const uint64_t *ref_off; int32_t n_ref; bool no_ref;
    uint64_t n; uint32_t rps, tsize;        // records, records per slice, table slots per slice (a power of two >= 2 rps)
    uint64_t *hash; int64_t *aend;          // per record
    int32_t *slot;                          // [slice][tsize]: slice-local record number of the slot's first read, -1 = free
    uint32_t *gcnt, *gstart, *gfill;        // [slice][tsize]: reads per slot, their first place in mem, places taken
    int32_t *grp;                           // per record: its slot, -1 = not paired
    uint32_t *mem;                          // [slice][rps]: slice-local record numbers, grouped by slot
    uint8_t *cf; int32_t *nf;               // per record: decisions
    uint64_t hash_mask;
};

#ifdef HGPU_HOSTSIM
static uint64_t g_hash_mask = ~0ull;        // tests force collisions with a narrower mask
#endif
// atomics on the device; the host build runs the kernels as serial loops
CRAMREC_HD inline int32_t at_cas(int32_t *p, int32_t cmp, int32_t v)
{
#ifdef __CUDA_ARCH__
    return atomicCAS(p, cmp, v);
#else
    const int32_t o = *p; if (o == cmp) *p = v; return o;
#endif
}
CRAMREC_HD inline uint32_t at_add(uint32_t *p, uint32_t v)
{
#ifdef __CUDA_ARCH__
    return atomicAdd(p, v);
#else
    const uint32_t o = *p; *p += v; return o;
#endif
}

// c->ref_end when process_one_read sees record g (cram_encode.c:1923-1927, :2037-2056): with a reference, the length of the
// sequence of the last record of the container (= slice here) up to g whose reference id is set; 0 before any, and 0
// throughout without a reference
CRAMREC_HD inline int64_t mate_ref_end(const PArgs &A, uint64_t g)
{
    if (A.no_ref) return 0;
    const uint64_t first = g / A.rps * A.rps;
    for (uint64_t r = g + 1; r-- > first;) {
        const int32_t t = A.core[r].tid;
        if (t >= 0 && t < A.n_ref) return (int64_t)(A.ref_off[t + 1] - A.ref_off[t]);
    }
    return 0;
}

CRAMREC_HD inline uint32_t rec_name_len(const PArgs &A, uint64_t g)
{
    const uint64_t l = A.data_off[g + 1] - A.data_off[g];
    return mate_name_len(A.data + A.data_off[g], A.core[g].l_qname < l ? A.core[g].l_qname : (uint32_t)l);
}

CRAMREC_HD inline void key_body(const PArgs &A, uint64_t g)
{
    const Core &c = A.core[g];
    A.cf[g] = MATE_DETACHED; A.nf[g] = 0;
    // an unmapped read at apos <= 0 ends at apos whatever ref_end is (>= 0): skip the walk back for the unplaced tail
    const int64_t re = (c.flag & 4) && c.pos + 1 <= 0 ? 0 : mate_ref_end(A, g);
    A.aend[g] = mate_aend(c, A.data + A.data_off[g], (uint32_t)(A.data_off[g + 1] - A.data_off[g]), A.no_ref, re);
    A.hash[g] = mate_hash(A.data + A.data_off[g], rec_name_len(A, g), (c.flag & 0x100) != 0) & A.hash_mask;
}

CRAMREC_HD inline bool same_name(const PArgs &A, uint64_t a, uint64_t b)
{
    if (A.hash[a] != A.hash[b] || ((A.core[a].flag ^ A.core[b].flag) & 0x100)) return false;
    const uint32_t la = rec_name_len(A, a), lb = rec_name_len(A, b);
    if (la != lb) return false;
    const uint8_t *pa = A.data + A.data_off[a], *pb = A.data + A.data_off[b];
    for (uint32_t i = 0; i < la; i++) if (pa[i] != pb[i]) return false;
    return true;
}

CRAMREC_HD inline void group_body(const PArgs &A, uint64_t g)
{
    if (!(A.core[g].flag & 1)) { A.grp[g] = -1; return; }
    const uint64_t sl = g / A.rps, g0 = sl * A.rps;
    int32_t *slot = A.slot + sl * A.tsize;
    uint32_t s = (uint32_t)A.hash[g] & (A.tsize - 1);
    for (;;) {                                     // the table has 2 slots per read of the slice: a free one is always found
        const int32_t cur = at_cas(&slot[s], -1, (int32_t)(g - g0));
        if (cur < 0 || same_name(A, g0 + (uint32_t)cur, g)) break;
        s = (s + 1) & (A.tsize - 1);
    }
    A.grp[g] = (int32_t)s;
    at_add(&A.gcnt[sl * A.tsize + s], 1);
}

CRAMREC_HD inline void fill_body(const PArgs &A, uint64_t g)
{
    if (A.grp[g] < 0) return;
    const uint64_t sl = g / A.rps, row = sl * A.tsize + (uint32_t)A.grp[g];
    A.mem[sl * A.rps + A.gstart[row] + at_add(&A.gfill[row], 1)] = (uint32_t)(g - sl * A.rps);
}

CRAMREC_HD inline void resolve_body(const PArgs &A, uint64_t row)
{
    const uint32_t k = A.gcnt[row];
    if (k < 2) return;
    const uint64_t sl = row / A.tsize, g0 = sl * A.rps;
    uint32_t *m = A.mem + g0 + A.gstart[row];
    for (uint32_t i = 1; i < k; i++) {             // record order (the fill pass placed them in any order); groups are tiny
        const uint32_t v = m[i];
        uint32_t j = i;
        for (; j > 0 && m[j - 1] > v; j--) m[j] = m[j - 1];
        m[j] = v;
    }
    mate_replay(m, k, A.core + g0, A.aend + g0, A.cf + g0, A.nf + g0);
}

CRAMREC_HD inline void count_body(const EArgs &A, uint64_t g)
{
    const uint32_t sl = (uint32_t)(g / A.rps), r = (uint32_t)(g % A.rps);
    uint32_t n[S_COUNT];
    for (int s = 0; s < S_COUNT; s++) n[s] = 0;
    Emit<false> E{n, nullptr};
    if (A.tkeys) { E.x = A.cnt + ((size_t)sl * A.R + S_COUNT) * A.rps + r; E.xs = A.rps; }       // zeroed before the count pass
    const uint8_t *ref = nullptr; int64_t rl = 0;
    if (A.ref_bases && A.core[g].tid >= 0 && A.core[g].tid < A.n_ref) { ref = A.ref_bases + A.ref_off[A.core[g].tid]; rl = (int64_t)(A.ref_off[A.core[g].tid + 1] - A.ref_off[A.core[g].tid]); }
    const int rc = walk<false>(A.core[g], A.data + A.data_off[g], (uint32_t)(A.data_off[g + 1] - A.data_off[g]), A.tl[g], ref, rl,
                               A.mate_cf ? A.mate_cf[g] : MATE_DETACHED, A.mate_nf ? A.mate_nf[g] : 0, tag_rec(A, g), E);
    A.status[g] = rc;
    for (int s = 0; s < S_COUNT; s++) A.cnt[((size_t)sl * A.R + s) * A.rps + r] = rc == ENC_OK ? n[s] : 0;
}

CRAMREC_HD inline void write_body(const EArgs &A, uint64_t g)
{
    if (A.status[g] != ENC_OK) return;
    const uint32_t sl = (uint32_t)(g / A.rps), r = (uint32_t)(g % A.rps);
    uint32_t n[S_COUNT];
    uint8_t *base[S_COUNT];
    for (int s = 0; s < S_COUNT; s++) { n[s] = A.cnt[((size_t)sl * A.R + s) * A.rps + r]; base[s] = A.arena + A.base[(size_t)sl * A.R + s]; }
    Emit<true> E{n, base};
    if (A.tkeys) { E.x = A.cnt + ((size_t)sl * A.R + S_COUNT) * A.rps + r; E.xs = A.rps; E.xarena = A.arena; E.xbase = A.base + (size_t)sl * A.R + S_COUNT; }
    const uint8_t *ref = nullptr; int64_t rl = 0;
    if (A.ref_bases && A.core[g].tid >= 0 && A.core[g].tid < A.n_ref) { ref = A.ref_bases + A.ref_off[A.core[g].tid]; rl = (int64_t)(A.ref_off[A.core[g].tid + 1] - A.ref_off[A.core[g].tid]); }
    walk<true>(A.core[g], A.data + A.data_off[g], (uint32_t)(A.data_off[g + 1] - A.data_off[g]), A.tl[g], ref, rl,
               A.mate_cf ? A.mate_cf[g] : MATE_DETACHED, A.mate_nf ? A.mate_nf[g] : 0, tag_rec(A, g), E);
}

#ifndef HGPU_HOSTSIM
__global__ void __launch_bounds__(128) cram_enc_count_kernel(EArgs A)
{
    const uint64_t g = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (g < A.n) count_body(A, g);
}
// one warp per (slice, stream): exclusive scan of that row in place, total to tot[]
__global__ void __launch_bounds__(128) cram_enc_scan_kernel(EArgs A, uint32_t rows)
{
    const uint32_t row = blockIdx.x * 4 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (row >= rows) return;
    const uint32_t sl = row / A.R;
    const uint64_t first = (uint64_t)sl * A.rps;
    const uint32_t nr = (uint32_t)(A.n - first < A.rps ? A.n - first : A.rps);
    uint32_t *p = A.cnt + (size_t)row * A.rps;
    uint32_t run = 0;
    for (uint32_t b = 0; b < nr; b += 32) {
        const uint32_t i = b + lane, v = i < nr ? p[i] : 0;
        uint32_t inc = v;
        for (int d = 1; d < 32; d <<= 1) { const uint32_t t = __shfl_up_sync(0xffffffffu, inc, d); if (lane >= (uint32_t)d) inc += t; }
        if (i < nr) p[i] = run + inc - v;
        run += __shfl_sync(0xffffffffu, inc, 31);
    }
    if (lane == 0) A.tot[row] = run;
}
__global__ void __launch_bounds__(128) cram_enc_write_kernel(EArgs A)
{
    const uint64_t g = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (g < A.n) write_body(A, g);
}

float g_enc_ms[3] = {0, 0, 0};                 // device time of the last call: pairing kernels, count + scan + write kernels, tag pass
// one thread per record: the MD / NM decisions of tag_rules
__global__ void __launch_bounds__(128) cram_enc_tags_kernel(TArgs A)
{
    const uint64_t g = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (g < A.n) tags_body(A, g);
}
__global__ void __launch_bounds__(128) cram_mate_key_kernel(PArgs A)
{
    const uint64_t g = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (g < A.n) key_body(A, g);
}
__global__ void __launch_bounds__(128) cram_mate_group_kernel(PArgs A)
{
    const uint64_t g = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (g < A.n) group_body(A, g);
}
// one warp per slice: exclusive scan of the slot sizes -> each slot's first place in the slice's member list
__global__ void __launch_bounds__(128) cram_mate_scan_kernel(PArgs A, uint32_t ns)
{
    const uint32_t sl = blockIdx.x * 4 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (sl >= ns) return;
    const uint32_t *c = A.gcnt + (size_t)sl * A.tsize;
    uint32_t *o = A.gstart + (size_t)sl * A.tsize;
    uint32_t run = 0;
    for (uint32_t b = 0; b < A.tsize; b += 32) {
        const uint32_t v = c[b + lane];
        uint32_t inc = v;
        for (int d = 1; d < 32; d <<= 1) { const uint32_t t = __shfl_up_sync(0xffffffffu, inc, d); if (lane >= (uint32_t)d) inc += t; }
        o[b + lane] = run + inc - v;
        run += __shfl_sync(0xffffffffu, inc, 31);
    }
}
__global__ void __launch_bounds__(128) cram_mate_fill_kernel(PArgs A)
{
    const uint64_t g = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (g < A.n) fill_body(A, g);
}
__global__ void __launch_bounds__(128) cram_mate_resolve_kernel(PArgs A, uint64_t rows)
{
    const uint64_t row = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (row < rows) resolve_body(A, row);
}
#endif

int encode_impl(hgpu_ctx *ctx, const char *header_text, uint32_t header_len, const hgpu_bam1_core *core, const uint8_t *data,
                const uint64_t *data_off, uint64_t n, const hgpu_cram_refs *refs, uint32_t rps, int minor, uint32_t enc_flags,
                uint8_t **out_file, uint64_t *out_len)
{
    const bool attach = (enc_flags & HGPU_CRAM_ENC_ATTACH_MATES) != 0, tb = (enc_flags & HGPU_CRAM_ENC_TAG_BLOCKS) != 0;
#ifdef HGPU_HOSTSIM
    g_mate_cf.clear(); g_mate_nf.clear(); g_tag_drop.clear(); g_tag_rg.clear();
#endif
    // reference-based shape only when every mapped record's reference sequence was supplied (the reader will need them all)
    bool use_ref = refs && refs->bases && refs->off && refs->n_ref > 0;
    if (use_ref)
        for (uint64_t g = 0; g < n && use_ref; g++) {
            const int32_t t = core[g].tid;
            if (!(core[g].flag & 4) && (t < 0 || t >= refs->n_ref || refs->off[t + 1] == refs->off[t])) use_ref = false;
        }
    const uint64_t ref_bytes = use_ref ? refs->off[refs->n_ref] : 0;
    if (!out_file || !out_len || (n && (!core || !data || !data_off)) || (header_len && !header_text)) { hgpu_set_error("cram encode: null argument"); return HGPU_ERR_ARG; }
    *out_file = nullptr; *out_len = 0;
    if (rps == 0) rps = 10000;
    if (minor != 0 && minor != 1) { hgpu_set_error("cram encode: CRAM 3.0 or 3.1"); return HGPU_ERR_ARG; }
    if (enc_flags & ~(uint32_t)(HGPU_CRAM_ENC_ATTACH_MATES | HGPU_CRAM_ENC_TAG_BLOCKS)) { hgpu_set_error("cram encode: unknown flags 0x%x", enc_flags); return HGPU_ERR_ARG; }
    if (attach && rps > (1u << 29)) { hgpu_set_error("cram encode: records per slice above 2^29 with mate attachment"); return HGPU_ERR_ARG; }
    const uint32_t ns = (uint32_t)((n + rps - 1) / rps);
    // aux fields of record g after SEQ / QUAL (nullptr when the record is too short: the count pass flags it)
    auto aux_of = [&](uint64_t g) -> const uint8_t * {
        const hgpu_bam1_core &c = core[g];
        const uint64_t fixed = (uint64_t)c.l_qname + 4ull * c.n_cigar + ((uint64_t)(c.l_qseq < 0 ? 0 : c.l_qseq) + 1) / 2 + (uint64_t)(c.l_qseq < 0 ? 0 : c.l_qseq);
        return fixed <= data_off[g + 1] - data_off[g] ? data + data_off[g] + fixed : nullptr;
    };
    // ---- tag blocks (host): the header's @RG IDs, each record's RG series value, the call's tag keys ----
    std::vector<int32_t> rgv;
    std::vector<uint32_t> tkeys;
    if (tb) {
        std::map<std::string, int32_t> rg_id;                              // sam_hrecs_find_rg: ID -> line index, the first line of an ID
        for (uint32_t i = 0; i < header_len;) {
            uint32_t e = i;
            while (e < header_len && header_text[e] != '\n') e++;
            if (e - i > 4 && !memcmp(header_text + i, "@RG\t", 4))
                for (uint32_t f = i + 3; f < e; f++)
                    if (header_text[f] == '\t' && f + 3 < e && !memcmp(header_text + f + 1, "ID:", 3)) {
                        uint32_t v = f + 4, ve = v;
                        while (ve < e && header_text[ve] != '\t' && header_text[ve] != '\r') ve++;
                        const std::string id(header_text + v, ve - v);
                        if (!rg_id.count(id)) { const int32_t k = (int32_t)rg_id.size(); rg_id[id] = k; }
                        break;
                    }
            i = e + 1;
        }
        rgv.assign(n ? n : 1, -1);
        std::set<uint32_t> ks;
        for (uint64_t g = 0; g < n; g++) {
            const uint8_t *p = aux_of(g), *end = data + data_off[g + 1];
            int md = 0, nm = 0, rgz = 0;
            for (; p && p < end;) {
                uint32_t vlen = 0;
                if (!aux_field(p, end, vlen)) break;                       // the count pass flags the record
                md += p[0] == 'M' && p[1] == 'D'; nm += p[0] == 'N' && p[1] == 'M';
                if (p[2] == 'd') { hgpu_set_error("cram encode: record %llu has an aux field of type 'd', which CRAM 3 tag blocks cannot hold", (unsigned long long)g); return HGPU_CRAM_UNSUPPORTED; }
                if (p[0] == 'R' && p[1] == 'G' && p[2] == 'Z') {
                    rgz++;
                    auto it = rg_id.find(std::string((const char *)p + 3, vlen - 1));
                    if (it != rg_id.end()) rgv[g] = it->second;
                }
                if (!(p[0] == 'R' && p[1] == 'G' && p[2] == 'Z' && rgv[g] >= 0)) ks.insert(aux_key(p));
                p += 3 + vlen;
            }
            if (md > 1 || nm > 1 || rgz > 1) { hgpu_set_error("cram encode: record %llu repeats an MD, NM or RG tag", (unsigned long long)g); return HGPU_CRAM_UNSUPPORTED; }
        }
        if (ks.size() > k_max_tag_keys) { hgpu_set_error("cram encode: %zu distinct tag keys, above the %u tag blocks a call may hold", ks.size(), k_max_tag_keys); return HGPU_CRAM_UNSUPPORTED; }
        tkeys.assign(ks.begin(), ks.end());
    }
    // ---- tag dictionary per slice (host: one walk over the aux field headers), without what the tag pass dropped ----
    std::vector<int32_t> tl(n ? n : 1, 0);
    std::vector<std::vector<std::string>> lines(ns);
    std::vector<std::vector<uint32_t>> keys(ns);
    auto dictionary = [&](const uint8_t *drop) {
        for (uint32_t sl = 0; sl < ns; sl++) {
            std::map<std::string, int32_t> seen;
            std::map<uint32_t, int> kseen;
            const uint64_t a = (uint64_t)sl * rps, b = a + rps < n ? a + rps : n;
            for (uint64_t g = a; g < b; g++) {
                const uint8_t *aux = aux_of(g), *end = data + data_off[g + 1];
                const uint32_t dr = drop ? drop[g] : 0u;
                std::string line;
                if (aux) {
                    for (const uint8_t *p = aux; p < end;) {
                        uint32_t vlen = 0;
                        if (!aux_field(p, end, vlen)) break;                   // the count pass flags the record
                        if (tb && (((dr & TAG_DROP_MD) && p[0] == 'M' && p[1] == 'D' && p[2] == 'Z') || ((dr & TAG_DROP_NM) && p[0] == 'N' && p[1] == 'M') ||
                                   (rgv[g] >= 0 && p[0] == 'R' && p[1] == 'G' && p[2] == 'Z'))) { p += 3 + vlen; continue; }
                        line.append((const char *)p, 3);
                        const uint32_t key = (uint32_t)p[0] << 16 | (uint32_t)p[1] << 8 | p[2];
                        if (!kseen.count(key)) { kseen[key] = 1; keys[sl].push_back(key); }
                        p += 3 + vlen;
                    }
                }
                auto it = seen.find(line);
                if (it == seen.end()) { const int32_t k = (int32_t)lines[sl].size(); seen[line] = k; lines[sl].push_back(line); tl[g] = k; }
                else tl[g] = it->second;
            }
        }
    };
    // ---- device: the tag pass, count, scan, write ----
    const bool tag_pass = tb && use_ref;
    const uint32_t R = S_COUNT + (uint32_t)tkeys.size();                   // series per slice
    const size_t rows = (size_t)ns * R;
    std::vector<uint32_t> tot(rows ? rows : 1, 0);
    std::vector<uint64_t> base(rows ? rows : 1, 0);
    std::vector<int32_t> status(n ? n : 1, 0);
    std::vector<uint8_t> arena_h;
    const uint64_t data_bytes = n ? data_off[n] : 0;
    if (n) {
        StageLayout L(16);
        const auto s_ref = L.seg(ref_bytes), s_roff = L.seg(use_ref ? ((size_t)refs->n_ref + 1) * 8 : 0);
        const auto s_core = L.seg(n * 48), s_data = L.seg(data_bytes), s_doff = L.seg((n + 1) * 8), s_tl = L.seg(n * 4), s_cnt = L.seg(rows * rps * 4),
                   s_tot = L.seg(rows * 4), s_base = L.seg(rows * 8), s_st = L.seg(n * 4);
        // tag blocks: the sorted key table, per record the tag pass's drop bits and the RG series value
        const auto s_tkeys = L.seg(tkeys.size() * 4), s_tdrop = L.seg(tag_pass ? n : 0), s_rg = L.seg(tb ? n * 4 : 0);
        // every series byte comes from the record data, ITF8 at most 5 bytes per value: bound the arena before the scan
        // (each tag block adds at most its 16-byte alignment)
        const size_t arena_cap = StageLayout::align(2 * data_bytes + 200 * n + 4096 + (tb ? rows * 16 : 0));
        const auto s_arena = L.seg(arena_cap);
        // the pairing pass (mate attachment only): 2 table slots or more per read of a slice
        uint32_t tsize = 0;
        if (attach) { tsize = 32; while (tsize < 2 * rps) tsize <<= 1; }
        const size_t slots = attach ? (size_t)ns * tsize : 0, nm = attach ? n : 0;
        const auto s_hash = L.seg(nm * 8), s_aend = L.seg(nm * 8), s_mcf = L.seg(nm), s_mnf = L.seg(nm * 4), s_grp = L.seg(nm * 4),
                   s_mem = L.seg(attach ? (size_t)ns * rps * 4 : 0), s_slot = L.seg(slots * 4), s_gcnt = L.seg(slots * 4),
                   s_gstart = L.seg(slots * 4), s_gfill = L.seg(slots * 4);
#ifdef HGPU_HOSTSIM
        (void)ctx;
        std::vector<uint8_t> image(L.total);
        L.base = image.data();
        memcpy(L.at(s_core), core, n * 48); memcpy(L.at(s_data), data, data_bytes); memcpy(L.at(s_doff), data_off, (n + 1) * 8);
        if (use_ref) { memcpy(L.at(s_ref), refs->bases, ref_bytes); memcpy(L.at(s_roff), refs->off, ((size_t)refs->n_ref + 1) * 8); }
        if (tb) { memcpy(L.at(s_tkeys), tkeys.data(), tkeys.size() * 4); memcpy(L.at(s_rg), rgv.data(), n * 4); }
#else
        if (!ctx) { hgpu_set_error("null context"); return HGPU_ERR_ARG; }
        if (cudaSetDevice(ctx->device) != cudaSuccess) return HGPU_ERR_CUDA;
        int rc0 = hgpu_stage_ensure(ctx, L);
        if (rc0) return rc0;
        cudaStream_t st = ctx->stream;
        if (hgpu_h2d(L.at(s_core), core, n * 48, st) || hgpu_h2d(L.at(s_data), data, data_bytes, st) ||
            hgpu_h2d(L.at(s_doff), data_off, (n + 1) * 8, st)) return HGPU_ERR_CUDA;
        if (use_ref && (hgpu_h2d(L.at(s_ref), refs->bases, ref_bytes, st) ||
                        hgpu_h2d(L.at(s_roff), refs->off, ((size_t)refs->n_ref + 1) * 8, st))) return HGPU_ERR_CUDA;
        if (tb && (hgpu_h2d(L.at(s_tkeys), tkeys.data(), tkeys.size() * 4, st) || hgpu_h2d(L.at(s_rg), rgv.data(), n * 4, st))) return HGPU_ERR_CUDA;
#endif
        EArgs A;
        A.core = L.at<Core>(s_core); A.data = L.at(s_data); A.data_off = L.at<uint64_t>(s_doff);
        A.tl = L.at<int32_t>(s_tl); A.n = n; A.rps = rps;
        A.ref_bases = use_ref ? L.at(s_ref) : nullptr; A.ref_off = L.at<uint64_t>(s_roff); A.n_ref = use_ref ? refs->n_ref : 0;
        A.cnt = L.at<uint32_t>(s_cnt); A.tot = L.at<uint32_t>(s_tot);
        A.base = L.at<uint64_t>(s_base); A.arena = L.at(s_arena); A.status = L.at<int32_t>(s_st);
        A.mate_cf = attach ? L.at(s_mcf) : nullptr; A.mate_nf = attach ? L.at<int32_t>(s_mnf) : nullptr;
        A.R = R; A.tkeys = tb ? L.at<uint32_t>(s_tkeys) : nullptr; A.ntk = (uint32_t)tkeys.size();
        A.tdrop = tag_pass ? L.at(s_tdrop) : nullptr; A.rg = tb ? L.at<int32_t>(s_rg) : nullptr;
        TArgs TA{A.core, A.data, A.data_off, A.ref_bases, A.ref_off, A.n_ref, n, L.at(s_tdrop)};
        std::vector<uint8_t> tdrop_h;
        PArgs P;
        P.core = A.core; P.data = A.data; P.data_off = A.data_off;
        P.ref_off = A.ref_off; P.n_ref = A.n_ref; P.no_ref = !use_ref;
        P.n = n; P.rps = rps; P.tsize = tsize;
        P.hash = L.at<uint64_t>(s_hash); P.aend = L.at<int64_t>(s_aend); P.slot = L.at<int32_t>(s_slot);
        P.gcnt = L.at<uint32_t>(s_gcnt); P.gstart = L.at<uint32_t>(s_gstart); P.gfill = L.at<uint32_t>(s_gfill);
        P.grp = L.at<int32_t>(s_grp); P.mem = L.at<uint32_t>(s_mem); P.cf = L.at(s_mcf); P.nf = L.at<int32_t>(s_mnf);
        P.hash_mask = ~0ull;
#ifdef HGPU_HOSTSIM
        if (tag_pass) {
            for (uint64_t g = 0; g < n; g++) tags_body(TA, g);
            tdrop_h.assign(TA.drop, TA.drop + n);
        }
        if (tb) { g_tag_drop.assign(n, 0); if (tag_pass) g_tag_drop = tdrop_h; g_tag_rg.assign(rgv.begin(), rgv.begin() + n); }
        dictionary(tag_pass ? tdrop_h.data() : nullptr);
        memcpy(L.at(s_tl), tl.data(), n * 4);
        if (tb) memset(A.cnt, 0, rows * rps * 4);
        if (attach) {
            P.hash_mask = g_hash_mask;
            memset(P.slot, 0xff, slots * 4); memset(P.gcnt, 0, slots * 4); memset(P.gfill, 0, slots * 4);
            for (uint64_t g = 0; g < n; g++) key_body(P, g);
            for (uint64_t g = 0; g < n; g++) group_body(P, g);
            for (uint32_t sl = 0; sl < ns; sl++) {
                uint32_t run = 0;
                for (uint32_t s = 0; s < tsize; s++) { P.gstart[(size_t)sl * tsize + s] = run; run += P.gcnt[(size_t)sl * tsize + s]; }
            }
            for (uint64_t g = 0; g < n; g++) fill_body(P, g);
            for (size_t row = 0; row < slots; row++) resolve_body(P, row);
            g_mate_cf.assign(P.cf, P.cf + n); g_mate_nf.assign(P.nf, P.nf + n);
        }
        for (uint64_t g = 0; g < n; g++) count_body(A, g);
        for (size_t row = 0; row < rows; row++) {
            const uint64_t first = (uint64_t)(row / R) * rps;
            const uint32_t nr = (uint32_t)(n - first < rps ? n - first : rps);
            uint32_t *p = A.cnt + row * rps, run = 0;
            for (uint32_t i = 0; i < nr; i++) { const uint32_t v = p[i]; p[i] = run; run += v; }
            A.tot[row] = run;
        }
        memcpy(tot.data(), A.tot, rows * 4);
        memcpy(status.data(), A.status, n * 4);
#else
        struct Events {                                  // destroyed on every return path
            cudaEvent_t e[8]; int n = 0;
            bool make() { for (; n < 8; n++) if (cudaEventCreate(&e[n]) != cudaSuccess) return false; return true; }
            ~Events() { for (int k = 0; k < n; k++) cudaEventDestroy(e[k]); }
        } evs;
        if (!evs.make()) return HGPU_ERR_CUDA;
        cudaEvent_t *ev = evs.e;
        const unsigned rec_blocks = (unsigned)((n + 127) / 128);
        if (tag_pass) {
            cudaEventRecord(ev[6], st);
            cram_enc_tags_kernel<<<rec_blocks, 128, 0, st>>>(TA);
            cudaEventRecord(ev[7], st);
            hgpu_count_launch();
            if (hgpu_check(cudaGetLastError(), "cram encode tag pass launch")) return HGPU_ERR_CUDA;
            tdrop_h.resize(n);
            if (hgpu_d2h(tdrop_h.data(), TA.drop, n, st) || hgpu_check(cudaStreamSynchronize(st), "cram encode tag pass")) return HGPU_ERR_CUDA;
        }
        dictionary(tag_pass ? tdrop_h.data() : nullptr);
        if (hgpu_h2d(L.at(s_tl), tl.data(), n * 4, st)) return HGPU_ERR_CUDA;
        if (tb && hgpu_memset(A.cnt, 0, rows * rps * 4, st)) return HGPU_ERR_CUDA;
        cudaEventRecord(ev[0], st);
        if (attach) {
            if (hgpu_memset(P.slot, 0xff, slots * 4, st) || hgpu_memset(P.gcnt, 0, slots * 4, st) || hgpu_memset(P.gfill, 0, slots * 4, st)) return HGPU_ERR_CUDA;
            cram_mate_key_kernel<<<rec_blocks, 128, 0, st>>>(P);
            cram_mate_group_kernel<<<rec_blocks, 128, 0, st>>>(P);
            cram_mate_scan_kernel<<<(ns + 3) / 4, 128, 0, st>>>(P, ns);
            cram_mate_fill_kernel<<<rec_blocks, 128, 0, st>>>(P);
            cram_mate_resolve_kernel<<<(unsigned)((slots + 127) / 128), 128, 0, st>>>(P, (uint64_t)slots);
            hgpu_count_launch(5);
            if (hgpu_check(cudaGetLastError(), "cram encode pairing launch")) return HGPU_ERR_CUDA;
        }
        cudaEventRecord(ev[1], st);
        cudaEventRecord(ev[2], st);
        cram_enc_count_kernel<<<rec_blocks, 128, 0, st>>>(A);
        cram_enc_scan_kernel<<<(unsigned)((rows + 3) / 4), 128, 0, st>>>(A, (uint32_t)rows);
        cudaEventRecord(ev[3], st);
        hgpu_count_launch(2);
        if (hgpu_check(cudaGetLastError(), "cram encode launch")) return HGPU_ERR_CUDA;
        if (hgpu_d2h(tot.data(), A.tot, rows * 4, st) || hgpu_d2h(status.data(), A.status, n * 4, st) ||
            hgpu_check(cudaStreamSynchronize(st), "cram encode count")) return HGPU_ERR_CUDA;
#endif
        for (uint64_t g = 0; g < n; g++)
            if (status[g] != ENC_OK) {
                hgpu_set_error("cram encode: record %llu cannot be written by this encoder (%s)", (unsigned long long)g,
                               status[g] == ENC_UNSUPPORTED ? "a mapped read without SEQ / position, or a zero-length CIGAR op: host library" : "malformed bam1_t");
                return status[g] == ENC_UNSUPPORTED ? HGPU_CRAM_UNSUPPORTED : HGPU_CRAM_ERR_DECODE;
            }
        uint64_t at = 0;
        for (size_t row = 0; row < rows; row++) { base[row] = at; at += ((uint64_t)tot[row] + 15) & ~15ull; }
        if (at > arena_cap) { hgpu_set_error("cram encode: series arena bound exceeded"); return HGPU_ERR_NOMEM; }
        arena_h.resize(at + 16);
#ifdef HGPU_HOSTSIM
        memcpy(L.at(s_base), base.data(), rows * 8);
        for (uint64_t g = 0; g < n; g++) write_body(A, g);
        memcpy(arena_h.data(), A.arena, at);
#else
        if (hgpu_h2d(L.at(s_base), base.data(), rows * 8, st)) return HGPU_ERR_CUDA;
        cudaEventRecord(ev[4], st);
        cram_enc_write_kernel<<<(unsigned)((n + 127) / 128), 128, 0, st>>>(A);
        cudaEventRecord(ev[5], st);
        hgpu_count_launch();
        if (hgpu_check(cudaGetLastError(), "cram encode write launch")) return HGPU_ERR_CUDA;
        if (hgpu_d2h(arena_h.data(), A.arena, at, st)) return HGPU_ERR_CUDA;
        if (hgpu_check(cudaStreamSynchronize(st), "cram encode write")) return HGPU_ERR_CUDA;
        float cs = 0, wr = 0;
        cudaEventElapsedTime(&g_enc_ms[0], ev[0], ev[1]);
        cudaEventElapsedTime(&cs, ev[2], ev[3]);
        cudaEventElapsedTime(&wr, ev[4], ev[5]);
        g_enc_ms[1] = cs + wr;
        g_enc_ms[2] = 0;
        if (tag_pass) cudaEventElapsedTime(&g_enc_ms[2], ev[6], ev[7]);
#endif
    }
    // ---- compress the series blocks (device codecs) ----
    struct Blk { uint32_t slice; int stream; int method; std::vector<uint8_t> comp; uint32_t usize; };
    std::vector<Blk> blks;
    for (uint32_t sl = 0; sl < ns; sl++)
        for (int s = 0; s < (int)R; s++)
            if (tot[(size_t)sl * R + s]) blks.push_back({sl, s, 0, {}, tot[(size_t)sl * R + s]});
    // content id: stream index + 1 for the fixed series, the tag key for a tag block
    auto content_id = [&](int s) { return s < S_COUNT ? s + 1 : (int32_t)tkeys[(size_t)(s - S_COUNT)]; };
#ifndef HGPU_HOSTSIM
    if (!blks.empty()) {
        // names through the tok3 encoder (CRAM 3.1); everything through the method trial; the smaller wins
        const uint32_t nb = (uint32_t)blks.size();
        std::vector<const uint8_t *> pay(nb);
        std::vector<uint32_t> plen(nb), mask(nb);
        std::vector<int32_t> cid(nb), chosen(nb);
        std::vector<uint8_t> ctype(nb, 4);
        uint64_t cap = 0;
        const uint32_t m31 = (1u << 5) | (1u << 17) | (1u << 18) | (1u << 20) | (1u << 21) | (1u << 22) | (1u << 23);    // RANS_PR0/1/64/128/129/192/193
        const uint32_t m30 = (1u << 4) | (1u << 16);                                                                  // RANS0 / RANS1
        for (uint32_t i = 0; i < nb; i++) {
            pay[i] = arena_h.data() + base[(size_t)blks[i].slice * R + blks[i].stream];
            plen[i] = blks[i].usize; mask[i] = minor ? m31 : m30; cid[i] = content_id(blks[i].stream);
            cap += (uint64_t)plen[i] + 64;
        }
        std::vector<uint8_t> framed(cap + 4096);
        std::vector<uint64_t> foff(nb);
        uint64_t flen = 0;
        int rc = hgpu_cram_compress_blocks_host(ctx, pay.data(), plen.data(), mask.data(), cid.data(), ctype.data(), nb, framed.data(), framed.size(), foff.data(), &flen, chosen.data());
        if (rc) return rc;
        for (uint32_t i = 0; i < nb; i++) {
            // un-frame: method, type, id, comp size, uncomp size, payload (the CRC is rebuilt when the container is laid out)
            const uint8_t *p = framed.data() + foff[i];
            blks[i].method = p[0];
            const uint8_t *q = p + 2;
            auto rd = [&](void) { uint32_t c = *q; int k = c < 0x80 ? 0 : c < 0xc0 ? 1 : c < 0xe0 ? 2 : c < 0xf0 ? 3 : 4; uint32_t v;
                switch (k) { case 0: v = c; break; case 1: v = ((c & 0x3f) << 8) | q[1]; break; case 2: v = ((c & 0x1f) << 16) | (q[1] << 8) | q[2]; break;
                             case 3: v = ((c & 0x0f) << 24) | (q[1] << 16) | (q[2] << 8) | q[3]; break;
                             default: v = ((c & 0x0f) << 28) | (q[1] << 20) | (q[2] << 12) | (q[3] << 4) | (q[4] & 0x0f); break; }
                q += k + 1; return v; };
            rd();
            const uint32_t csz = rd();
            rd();
            blks[i].comp.assign(q, q + csz);
        }
        if (minor == 1) {
            std::vector<uint32_t> idx;
            for (uint32_t i = 0; i < nb; i++) if (blks[i].stream == S_RN) idx.push_back(i);
            if (!idx.empty()) {
                const uint32_t k = (uint32_t)idx.size();
                std::vector<uint64_t> ioff(k), ooff(k);
                std::vector<uint32_t> ilen(k), ocap(k), olen(k);
                std::vector<int32_t> ost(k);
                uint64_t ipos = 0, opos = 0;
                for (uint32_t j = 0; j < k; j++) { ioff[j] = ipos; ilen[j] = blks[idx[j]].usize; ipos += ((uint64_t)ilen[j] + 15) & ~15ull;
                                                   ooff[j] = opos; ocap[j] = ilen[j] + ilen[j] / 2 + 65536; opos += ((uint64_t)ocap[j] + 15) & ~15ull; }
                std::vector<uint8_t> ibuf(ipos + 16), obuf(opos + 16);
                for (uint32_t j = 0; j < k; j++) memcpy(ibuf.data() + ioff[j], pay[idx[j]], ilen[j]);
                rc = hgpu_tok3_encode_batch_host(ctx, ibuf.data(), ioff.data(), ilen.data(), k, obuf.data(), ooff.data(), ocap.data(), olen.data(), ost.data());
                if (rc == HGPU_OK)
                    for (uint32_t j = 0; j < k; j++) {
                        Blk &b = blks[idx[j]];
                        const size_t cur = b.method == 0 ? b.usize : b.comp.size();
                        if (ost[j] == HGPU_OK && olen[j] && olen[j] < cur) { b.method = 8; b.comp.assign(obuf.data() + ooff[j], obuf.data() + ooff[j] + olen[j]); }
                    }
            }
        }
    }
#endif
    // ---- file image ----
    Buf f;
    { const uint8_t def[6] = {'C', 'R', 'A', 'M', 3, (uint8_t)minor}; f.bytes(def, 6); uint8_t id[20] = "htslib_b200"; f.bytes(id, 20); }
    auto container = [&](int32_t ref_id, int32_t start, int32_t span, int32_t nrec, int64_t counter, int64_t bases, int32_t nblocks,
                         const std::vector<int32_t> &landmarks, const Buf &body) {
        Buf h;
        h.le32((uint32_t)body.v.size());
        h.itf8(ref_id); h.itf8(start); h.itf8(span); h.itf8(nrec); h.ltf8(counter); h.ltf8(bases); h.itf8(nblocks);
        h.itf8((int32_t)landmarks.size());
        for (int32_t l : landmarks) h.itf8(l);
        h.le32(host_crc32(h.v.data(), h.v.size()));
        f.bytes(h.v.data(), h.v.size());
        f.bytes(body.v.data(), body.v.size());
    };
    {   // SAM header container (cram_write_SAM_hdr :4889): one RAW FILE_HEADER block = int32 length + text
        Buf pl; pl.le32(header_len); pl.bytes(header_text, header_len);
        Buf body; frame_block(body, 0, 0, 0, pl.v.data(), (uint32_t)pl.v.size(), (uint32_t)pl.v.size());
        container(0, 0, 0, 0, 0, 0, 1, std::vector<int32_t>{0}, body);
    }
    size_t bi = 0;
    for (uint32_t sl = 0; sl < ns; sl++) {
        const uint64_t a = (uint64_t)sl * rps, b = a + rps < n ? a + rps : n;
        int64_t bases = 0;
        for (uint64_t g = a; g < b; g++) bases += core[g].l_qseq;
        Buf ch; compression_header(ch, lines[sl], keys[sl], use_ref, attach, tb);
        Buf body;
        frame_block(body, 0, 1, 0, ch.v.data(), (uint32_t)ch.v.size(), (uint32_t)ch.v.size());
        const int32_t landmark = (int32_t)body.v.size();
        size_t e = bi;
        while (e < blks.size() && blks[e].slice == sl) e++;
        const int32_t next = (int32_t)(e - bi);
        Buf sh;                                                            // slice header (cram_encode_slice_header :2870)
        sh.itf8(-2); sh.itf8(0); sh.itf8(0); sh.itf8((int32_t)(b - a)); sh.ltf8((int64_t)a); sh.itf8(next + 1); sh.itf8(next + 1);
        sh.itf8(0);                                                        // content ids: the CORE block, then the external blocks
        for (size_t k = bi; k < e; k++) sh.itf8(content_id(blks[k].stream));
        sh.itf8(-1);                                                       // no embedded reference
        { const uint8_t md5[16] = {0}; sh.bytes(md5, 16); }
        frame_block(body, 0, 2, 0, sh.v.data(), (uint32_t)sh.v.size(), (uint32_t)sh.v.size());
        frame_block(body, 0, 5, 0, nullptr, 0, 0);                         // CORE: every series is external
        for (size_t k = bi; k < e; k++) {
            const Blk &bk = blks[k];
            const uint8_t *raw = arena_h.data() + base[(size_t)sl * R + bk.stream];
            if (bk.method == 0) frame_block(body, 0, 4, content_id(bk.stream), raw, bk.usize, bk.usize);
            else frame_block(body, bk.method, 4, content_id(bk.stream), bk.comp.data(), (uint32_t)bk.comp.size(), bk.usize);
        }
        container(-2, 0, 0, (int32_t)(b - a), (int64_t)a, bases, next + 3, std::vector<int32_t>{landmark}, body);
        bi = e;
    }
    { static const uint8_t eof[38] = {0x0f, 0x00, 0x00, 0x00, 0xff, 0xff, 0xff, 0xff, 0x0f, 0xe0, 0x45, 0x4f, 0x46, 0x00, 0x00, 0x00, 0x00, 0x01, 0x00,
                                      0x05, 0xbd, 0xd9, 0x4f, 0x00, 0x01, 0x00, 0x06, 0x06, 0x01, 0x00, 0x01, 0x00, 0x01, 0x00, 0xee, 0x63, 0x01, 0x4b};
      f.bytes(eof, 38); }                                                  // the CRAM 3 end-of-file container (CRAM specification, section 9)
    uint8_t *res = (uint8_t *)malloc(f.v.size() + 1);
    if (!res) { hgpu_set_error("out of host memory"); return HGPU_ERR_NOMEM; }
    memcpy(res, f.v.data(), f.v.size());
    *out_file = res; *out_len = f.v.size();
    return HGPU_OK;
}

}  // namespace

#ifdef HGPU_HOSTSIM
extern "C" int hostsim_cram_encode_records(const char *header_text, uint32_t header_len, const hgpu_bam1_core *core, const uint8_t *data,
        const uint64_t *data_off, uint64_t n, const hgpu_cram_refs *refs, uint32_t rps, int minor, uint8_t **out_file, uint64_t *out_len)
{
    try { return encode_impl(nullptr, header_text, header_len, core, data, data_off, n, refs, rps, minor, 0, out_file, out_len); }
    catch (...) { hgpu_set_error("internal error"); return HGPU_ERR_NOMEM; }
}
extern "C" int hostsim_cram_encode_records_opts(const char *header_text, uint32_t header_len, const hgpu_bam1_core *core, const uint8_t *data,
        const uint64_t *data_off, uint64_t n, const hgpu_cram_refs *refs, uint32_t rps, int minor, uint32_t enc_flags, uint8_t **out_file, uint64_t *out_len)
{
    try { return encode_impl(nullptr, header_text, header_len, core, data, data_off, n, refs, rps, minor, enc_flags, out_file, out_len); }
    catch (...) { hgpu_set_error("internal error"); return HGPU_ERR_NOMEM; }
}
// test hooks: the pairing decisions of the last call with mate attachment (CF bits, NF), and the mask every name hash is
// reduced by (0 makes every name collide, so only the name comparison keeps different names apart)
extern "C" uint64_t hostsim_cram_enc_mates(uint8_t *cf, int32_t *nf, uint64_t cap)
{
    const uint64_t n = g_mate_cf.size();
    for (uint64_t i = 0; i < n && i < cap; i++) { cf[i] = g_mate_cf[i]; nf[i] = g_mate_nf[i]; }
    return n;
}
extern "C" void hostsim_cram_enc_hash_mask(uint64_t mask) { g_hash_mask = mask; }
// test hook: the tag pass's drop bits (0 where it did not run) and the RG series values of the last call with tag blocks
extern "C" uint64_t hostsim_cram_enc_tags(uint8_t *drop, int32_t *rg, uint64_t cap)
{
    const uint64_t n = g_tag_drop.size();
    for (uint64_t i = 0; i < n && i < cap; i++) { drop[i] = g_tag_drop[i]; rg[i] = g_tag_rg[i]; }
    return n;
}
#else
extern "C" int hgpu_cram_encode_records_host(hgpu_ctx *ctx, const char *header_text, uint32_t header_len, const hgpu_bam1_core *core,
        const uint8_t *data, const uint64_t *data_off, uint64_t n, const hgpu_cram_refs *refs, uint32_t records_per_slice, int minor_version,
        uint8_t **out_file, uint64_t *out_len)
{
    return hgpu_abi_call([&] { return encode_impl(ctx, header_text, header_len, core, data, data_off, n, refs, records_per_slice, minor_version, 0,
                                                  out_file, out_len); },
                         HGPU_ERR_NOMEM, HGPU_ERR_NOMEM);
}

extern "C" int hgpu_cram_encode_records_opts_host(hgpu_ctx *ctx, const char *header_text, uint32_t header_len, const hgpu_bam1_core *core,
        const uint8_t *data, const uint64_t *data_off, uint64_t n, const hgpu_cram_refs *refs, uint32_t records_per_slice, int minor_version,
        uint32_t enc_flags, uint8_t **out_file, uint64_t *out_len)
{
    return hgpu_abi_call([&] { return encode_impl(ctx, header_text, header_len, core, data, data_off, n, refs, records_per_slice, minor_version,
                                                  enc_flags, out_file, out_len); },
                         HGPU_ERR_NOMEM, HGPU_ERR_NOMEM);
}

extern "C" void hgpu_cram_encode_last_ms(float *pair_ms, float *count_write_ms)
{
    if (pair_ms) *pair_ms = g_enc_ms[0];
    if (count_write_ms) *count_write_ms = g_enc_ms[1];
}

extern "C" void hgpu_cram_encode_tags_last_ms(float *tag_ms)
{
    if (tag_ms) *tag_ms = g_enc_ms[2];
}
#endif
