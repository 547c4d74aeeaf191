// rANS Nx16 ("RANS_PR", CRAM 3.1 block method 5) decoder for sm_90a.
//
// Replaces rans_uncompress_to_4x16 and the four symbol loops behind it
// (htscodecs rANS_static4x16pr.c:1586-1873, :213-328, :504-800; rANS_static32x16pr.c:254-408,
// :527-754) with ONE warp-per-stream kernel: the N (4 or 32) interleaved rANS states live one
// per lane, and the shared 16-bit renormalisation word stream is indexed with
// __ballot_sync / __popc — lane k takes word  base + popc(ballot(R < 2^15) & lanemask_lt(k)),
// which is exactly the "states renormalise in index order" rule of the scalar code
// (rANS_static32x16pr.c:334-337, :657-666).
//
// Table layout (GPU-first, not the reference's): per context row a BYTE lookup
//   lut[row][m] -> compact symbol index       (1<<shift bytes)
// plus a small per-(row,symbol) record
//   fb[row][k]  -> { f | start<<16 , byte }   (8 bytes)
// so an order-1 table for a 4-symbol NovaSeq alphabet is ~4 KiB (vs 16 KiB for the reference's
// 32-bit s3 table and 1 MiB for its full 256-context array).  Small tables are what lets tens
// of streams be resident per SM, which is where the throughput of a 32-lane-wide serial
// recurrence comes from.  Rows are indexed by compact symbol index, so "next context" is the
// index just looked up.  Tables that do not fit the CTA's shared memory go to a per-CTA slot in
// global memory (L1/L2 resident).
//
// One CTA = one warp.  CTAs pull streams from an atomic work counter (persistent grid sized to
// the SM count), largest streams first if the caller sorted them.
#include "hgpu_internal.h"
#include <stdio.h>

namespace {

constexpr uint32_t RANS_L = 1u << 15;               // RANS_BYTE_L, rANS_word.h:64
constexpr int SM_F      = 0;                        // u32 F[256]          1024 B
constexpr int SM_CUM    = 1024;                     // u32 cum[257]        1028 B -> 1040
constexpr int SM_ROWOF  = 2064;                     // u8 rowof[256]  byte -> compact row / 0xff
constexpr int SM_SYMOF  = 2320;                     // u8 symof[256]  compact index -> byte
constexpr int SM_RING   = 2576;                     // 512 B ring mirroring the compressed word stream
constexpr int SM_TAB    = 3088;                     // table area (16-byte aligned)
constexpr uint32_t GTAB_BYTES = 256u * 4096u + 256u * 256u * 4u;   // worst-case order-1 table
constexpr uint32_t TBLBUF_BYTES = 256u * 1024u;     // decoded (was-compressed) order-1 table text

struct WarpScratch {
    uint8_t *tmp;      // max_out bytes : RLE / PACK intermediate
    uint8_t *planes;   // max_out bytes : STRIPE planes
    uint8_t *meta;     // max_out+1024  : decoded RLE meta
    uint8_t *tblbuf;   // TBLBUF_BYTES  : decoded order-1 table text
    uint8_t *gtab;     // GTAB_BYTES    : table overflow
    uint32_t max_out;
    uint8_t *tab_base;       // shared-memory area tables are placed in ...
    uint32_t tab_cap;        // ... and its size; larger tables go to gtab, or defer the stream when gtab is null
    int pass;                // 0: small-table passes (defer what they cannot hold), 1: everything else
    mutable bool defer;      // set when a small-table pass hands the stream to pass 1
    struct Hook *hook;       // non-null: top-level plain streams stop after the table build (rans_nx16_fast.cuh)
    bool compact = false;    // prefer the compact table form even when the full one would fit (many streams per warp)
};

// What a hooked dec_order0/1 hands back instead of running its symbol loop.
struct Hook {
    int mode;                // HOOK_X32: only 32-way streams stop; HOOK_N4: only 4-way streams stop
    bool taken;
    uint32_t order, N, shift, lb, ncol, ipos, U, R, row0, tab_bytes;
    const uint8_t *in; uint32_t in_len;
    uint8_t *out;
    uint8_t *lut; uint32_t *fb;
    uint16_t *Fcap;          // HOOK_X32: [17][16] normalised frequencies of small alphabets (row 16 = flags), shared memory
};
constexpr int HOOK_X32 = 1, HOOK_N4 = 2;
constexpr int RC_HOOKED = 2;

// ---------------------------------------------------------------------------------------------
// Warp-uniform scalar helpers: every lane runs the same code on the same addresses (loads
// broadcast), so no shuffles are needed and control flow never diverges.
// ---------------------------------------------------------------------------------------------

// 7-bit big-endian varint (var_get_u32, varint.h:267-299)
__device__ int vget(const uint8_t *p, const uint8_t *end, uint32_t &v)
{
    const uint8_t *s = p;
    uint32_t acc = 0;
    uint8_t c;
    if (end - p >= 6) {
        int budget = 5;
        do { c = *p++; acc = (acc << 7) | (c & 0x7f); } while ((c & 0x80) && budget-- > 0);
    } else {
        if (p >= end) { v = 0; return 0; }
        do { c = *p++; acc = (acc << 7) | (c & 0x7f); } while ((c & 0x80) && p < end);
    }
    v = acc;
    return (int)(p - s);
}

// decode_alphabet (rANS_static16_int.h:191-238): marks F[sym] = 1.  F must be zeroed.
__device__ int read_alphabet(const uint8_t *p, const uint8_t *end, uint32_t *F)
{
    const uint8_t *s = p;
    int run = 0, sym;
    if (p >= end) return 0;
    sym = *p++;
    if (sym == 0 && p + 2 >= end) return (int)(p - s);
    for (;;) {
        F[sym] = 1;
        if (p >= end) return 0;
        if (run == 0 && sym + 1 == *p) {
            if (p + 1 >= end) return 0;
            sym = *p++;
            run = *p++;
        } else if (run) {
            run--;
            if (++sym > 255) return 0;
        } else {
            sym = *p++;
        }
        if (sym == 0 || p >= end) break;
    }
    return (int)(p - s);
}

// Two forms of the slot -> symbol map of a row:
//   full     lb == shift: lut[row][m] is the symbol of slot m                      (1 << shift bytes per row)
//   compact  lb <  shift: lut[row][m >> (shift - lb)] is the symbol that owns the FIRST slot of that
//            bucket; the symbol of m is found by walking the row's records forward while m lies behind
//            the record's range (one step in the common case: 64 buckets for at most a few dozen symbols).
//            A 40-symbol order-1 table is 9 KiB instead of 47 KiB (shift 10) / 170 KiB (shift 12), so
//            it stays in shared memory; rows no valid stream enters ("null rows") only exist in full form.
constexpr uint32_t COMPACT_LB = 6, COMPACT_LB_BIG = 8;
struct Table {
    uint8_t *lut;      // [rows][1<<lb]
    uint32_t *fb;      // [rows][ncol]  byte | start<<8 | (f-1)<<20
    uint32_t ncol;     // compact alphabet size
    uint32_t shift;
    uint32_t lb;       // index bits of a lut row
    bool     in_smem;
};

// Inclusive-free cumulative sums of cnt[0..n) (n <= 256) into cum[0..n]; returns the total.
__device__ uint32_t warp_cumsum(const uint32_t *val, uint32_t *cum, int n)
{
    const uint32_t lane = hgpu_lane();
    uint32_t loc[8], sum = 0;
#pragma unroll
    for (int k = 0; k < 8; k++) {
        int j = lane * 8 + k;
        loc[k] = j < n ? val[j] : 0;
        sum += loc[k];
    }
    uint32_t inc = sum;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        uint32_t t = __shfl_up_sync(0xffffffffu, inc, d);
        if (lane >= (uint32_t)d) inc += t;
    }
    uint32_t run = inc - sum;
#pragma unroll
    for (int k = 0; k < 8; k++) {
        int j = lane * 8 + k;
        if (j <= n) cum[j] = run;
        run += loc[k];
    }
    uint32_t total = __shfl_sync(0xffffffffu, inc, 31);
    __syncwarp();
    return total;
}

// Fill one table row from compact frequencies f[0..ncol) whose cumulative sums are cum[].
__device__ void fill_row(const Table &t, uint32_t row, const uint32_t *f, const uint32_t *cum,
                         const uint8_t *symof, bool wrap12)
{
    const uint32_t lane = hgpu_lane();
    uint8_t *lrow = t.lut + ((size_t)row << t.lb);
    uint32_t *frow = t.fb + (size_t)row * t.ncol;
    const uint32_t cs = t.shift - t.lb, rnd = (1u << cs) - 1u;
    for (uint32_t k = 0; k < t.ncol; k++) {
        uint32_t fk = f[k], c0 = cum[k];
        if (!fk) continue;
        // buckets whose first slot lies in [c0, c0 + fk)   (cs == 0: every slot)
        const uint32_t b0 = (c0 + rnd) >> cs, b1 = (c0 + fk + rnd) >> cs;
        for (uint32_t y = b0 + lane; y < b1; y += 32) lrow[y] = (uint8_t)k;
    }
    for (uint32_t k = lane; k < t.ncol; k += 32) {
        uint32_t fk = f[k];
        (void)wrap12;     // F == 4096 only occurs for a one-symbol table, whose output does not depend on the state
        frow[k] = fk ? ((uint32_t)symof[k] | (cum[k] << 8) | ((fk - 1u) << 20)) : 0u;
    }
}

// A row that no valid stream enters: symbol 0, f 0, bias = slot (see oracle/orc_rans_nx16.c).
__device__ void fill_null_row(const Table &t, uint32_t row)
{
    const uint32_t lane = hgpu_lane();
    uint8_t *lrow = t.lut + ((size_t)row << t.lb);       // (only ever called on a full table)
    for (uint32_t y = lane; y < (1u << t.lb); y += 32) lrow[y] = 0;
    if (lane == 0) t.fb[(size_t)row * t.ncol] = 0;     // byte 0, start 0, f 1
}

// ---------------------------------------------------------------------------------------------
// The symbol loops.
//
// Renormalisation words come from a 512-byte ring in shared memory that mirrors the compressed
// stream (refilled 128 bytes at a time with coalesced 32-bit loads, realigned with a funnel
// shift), so the per-step word fetch is one LDS.U16 instead of a global round trip.
// Order-1 output: every lane owns a contiguous segment; bytes are shifted into a 32-bit
// accumulator and stored as aligned words at the step where the lane's address crosses a 4-byte
// boundary (a per-lane phase, constant across the 4-step unrolled loop), so a step costs one
// predicated STG.32 per warp and 8 instead of 32 L2 transactions.
// Table records are 4 bytes (byte | start<<8 | (f-1)<<20): shared-memory bandwidth, not issue, is
// what bounds this loop (24 warps x 3 LDS per step), so the record is as narrow as it can be.
// ---------------------------------------------------------------------------------------------
// Explicit shared-space accesses with 32-bit addresses: the generic pointer of the dynamic shared
// array would otherwise be rebuilt (S2UR/ULEA/IMAD) at every access inside the hot loop.
__device__ __forceinline__ uint32_t lds_u8(uint32_t a) { uint32_t v; asm volatile("ld.shared.u8 %0, [%1];" : "=r"(v) : "r"(a) : "memory"); return v; }
__device__ __forceinline__ uint32_t lds_u16(uint32_t a) { uint32_t v; asm volatile("ld.shared.u16 %0, [%1];" : "=r"(v) : "r"(a) : "memory"); return v; }
__device__ __forceinline__ uint32_t lds_u32(uint32_t a) { uint32_t v; asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(a) : "memory"); return v; }

struct WordRing {
    const uint8_t *in;       // stream start (global)
    uintptr_t lim;           // first aligned word address entirely past the input
    uint32_t ipos0;          // stream offset mirrored at ring offset 0
    uint32_t avail;          // stream bytes [ipos0, avail) have been loaded (multiple of 128 past ipos0)
};

__device__ __forceinline__ void ring_load_chunk(uint8_t *ring, WordRing &wr)
{
    const uint32_t lane = hgpu_lane();
    const uint32_t c = (wr.avail - wr.ipos0) >> 7;                 // chunk index
    uintptr_t g = reinterpret_cast<uintptr_t>(wr.in) + wr.avail + 4u * lane;
    uintptr_t ga = g & ~(uintptr_t)3;
    uint32_t sh = (uint32_t)(g & 3) * 8;
    uint32_t w0 = ga < wr.lim ? *reinterpret_cast<const uint32_t *>(ga) : 0u;
    uint32_t w1 = ga + 4 < wr.lim ? *reinterpret_cast<const uint32_t *>(ga + 4) : 0u;
    reinterpret_cast<uint32_t *>(ring)[(c & 3) * 32 + lane] = __funnelshift_r(w0, w1, sh);
    wr.avail += 128;
}

// make sure the next `margin` bytes past ipos are in the ring (warp-uniform)
__device__ __forceinline__ void ring_ensure(uint8_t *ring, WordRing &wr, uint32_t ipos, uint32_t margin)
{
    if (ipos + margin > wr.avail) {
        __syncwarp();
        while (ipos + margin > wr.avail) ring_load_chunk(ring, wr);
        __syncwarp();
    }
}

__device__ __forceinline__ void ring_init(uint8_t *ring, WordRing &wr, const uint8_t *in, uint32_t in_len, uint32_t ipos)
{
    wr.in = in;
    wr.lim = (reinterpret_cast<uintptr_t>(in) + in_len + 3) & ~(uintptr_t)3;
    wr.ipos0 = ipos;
    wr.avail = ipos;
    ring_ensure(ring, wr, ipos, 256);
}

// renormalise with bounds care (RansDecRenormSafe, rANS_word.h:441): used near the end of input
__device__ __forceinline__ void renorm_safe(uint32_t &R, bool active, const uint8_t *ring, const WordRing &wr,
                                            uint32_t &ipos, uint32_t in_len)
{
    bool need = active && R < RANS_L;
    uint32_t bal = __ballot_sync(0xffffffffu, need);
    if (bal) {
        uint32_t wpos = ipos + 2u * __popc(bal & hgpu_lanemask_lt());
        uint32_t w = *reinterpret_cast<const uint16_t *>(ring + ((wpos - wr.ipos0) & 511u));
        bool ok = need && wpos + 2u <= in_len;
        if (ok) R = (R << 16) | w;
        ipos += 2u * __popc(__ballot_sync(0xffffffffu, ok));
    }
}

// branch-free renormalise; the caller guarantees ipos + 64 <= in_len.  rel = ipos - ipos0.
__device__ __forceinline__ void renorm_fast(uint32_t &R, bool active, const uint8_t *ring, uint32_t &rel)
{
    bool need = active && R < RANS_L;
    uint32_t bal = __ballot_sync(0xffffffffu, need);
    uint32_t rank = __popc(bal & hgpu_lanemask_lt());
    uint32_t w = *reinterpret_cast<const uint16_t *>(ring + ((rel + 2u * rank) & 511u));
    if (need) R = (R << 16) | w;
    rel += 2u * __popc(bal);
}

// record of slot m in one row; COMPACT: start from the bucket's first symbol and walk forward (warp-uniform loop)
template <bool COMPACT>
__device__ __forceinline__ uint32_t row_lookup(const uint8_t *lut, const uint32_t *fb, uint32_t m, uint32_t cs)
{
    uint32_t k = lut[COMPACT ? m >> cs : m];
    uint32_t e = fb[k];
    if (COMPACT) {
        for (;;) {
            const bool go = m >= ((e >> 8) & 0xfffu) + (e >> 20) + 1u;      // m lies behind this record's range
            if (!__any_sync(0xffffffffu, go)) break;
            if (go) e = fb[++k];
        }
    }
    return e;
}

template <bool SMEM, bool COMPACT = false>
__device__ void loop_order0(uint8_t *smem, const Table &t, const uint8_t *in, uint32_t in_len, uint32_t ipos,
                            uint8_t *out, uint32_t U, uint32_t N, uint32_t R)
{
    const uint32_t lane = hgpu_lane();
    const uint32_t mask = (1u << t.shift) - 1, shift = t.shift, cs = t.shift - t.lb;
    const uint8_t *lut = t.lut;
    const uint32_t *fb = t.fb;
    uint8_t *ring = smem + SM_RING;
    WordRing wr;
    ring_init(ring, wr, in, in_len, ipos);
    const bool mine = lane < N;
    uint32_t i = lane;
    // fast rows: every lane of the row active and the input far from its end
    if (N == 32) {
        uint32_t rel = 0;
        while (i + (32u - lane) <= U && ipos + rel + 64u <= in_len) {
            ring_ensure(ring, wr, ipos + rel, 64);
            uint32_t m = R & mask;
            uint32_t e = row_lookup<COMPACT>(lut, fb, m, cs), q = R >> shift;
            R = (e >> 20) * q + q + m - ((e >> 8) & 0xfffu);
            out[i] = (uint8_t)e;
            renorm_fast(R, true, ring, rel);
            i += 32;
        }
        ipos += rel;
    }
    for (; __any_sync(0xffffffffu, mine && i < U); i += N) {
        ring_ensure(ring, wr, ipos, 64);
        bool act = mine && i < U;
        uint32_t m = R & mask;
        uint32_t e = row_lookup<COMPACT>(lut, fb, m, cs), q = R >> shift;
        if (act) {
            R = (e >> 20) * q + q + m - ((e >> 8) & 0xfffu);
            out[i] = (uint8_t)e;
        }
        renorm_safe(R, act, ring, wr, ipos, in_len);
    }
}

// branch-free renormalise on a 32-bit shared address of the ring; caller guarantees the next 64
// input bytes exist.  rel = ipos - ipos0.
__device__ __forceinline__ void renorm_fast_s(uint32_t &R, bool active, uint32_t ring_a, uint32_t &rel)
{
    bool need = active && R < RANS_L;
    uint32_t bal = __ballot_sync(0xffffffffu, need);
    uint32_t rank = __popc(bal & hgpu_lanemask_lt());
    uint32_t w = lds_u16(ring_a + ((rel + 2u * rank) & 511u));
    R = need ? (R << 16) | w : R;
    rel += 2u * __popc(bal);
}

template <bool SMEM, bool FULL, bool COMPACT = false>
__device__ void loop_order1(uint8_t *smem, const Table &t, const uint8_t *in, uint32_t in_len, uint32_t ipos,
                            uint8_t *out, uint32_t U, uint32_t N, uint32_t R, uint32_t row0)
{
    const uint32_t lane = hgpu_lane();
    const uint32_t mask = (1u << t.shift) - 1, shift = t.shift, lb = t.lb, cs = t.shift - t.lb;
    const uint8_t *lut = t.lut;
    const uint8_t *fbb = reinterpret_cast<const uint8_t *>(t.fb);
    const uint32_t sm_base = (uint32_t)__cvta_generic_to_shared(smem);
    const uint32_t lut_a = SMEM ? (uint32_t)__cvta_generic_to_shared(t.lut) : 0u;
    const uint32_t fb_a = SMEM ? (uint32_t)__cvta_generic_to_shared(t.fb) : 0u, ring_a = sm_base + SM_RING;
    uint8_t *ring = smem + SM_RING;
    WordRing wr;
    ring_init(ring, wr, in, in_len, ipos);
    const bool mine = FULL ? true : lane < N;
    const uint32_t seg = U / N;
    uint8_t *op = out + (size_t)(mine ? lane : 0) * seg;
    const uint32_t fstride = t.ncol * 4u;
    uint32_t lrow = row0 << lb, frow = row0 * fstride, acc = 0;

    // one symbol for the lanes in ACTIVE; the record carries the next row's offsets
#define RANS_O1_CORE(ACTIVE)                                                                       \
        uint32_t m = R & mask;                                                                     \
        uint32_t k = SMEM ? lds_u8(lut_a + lrow + (COMPACT ? m >> cs : m)) : (uint32_t)lut[lrow + m]; \
        uint32_t e = SMEM ? lds_u32(fb_a + frow + k * 4u)                                          \
                          : *reinterpret_cast<const uint32_t *>(fbb + frow + k * 4u);              \
        if (COMPACT) {      /* walk forward while m lies behind the record's range */             \
            for (;;) {                                                                             \
                const bool go_ = m >= ((e >> 8) & 0xfffu) + (e >> 20) + 1u;                        \
                if (!__any_sync(0xffffffffu, go_)) break;                                          \
                if (go_) { k++; e = lds_u32(fb_a + frow + k * 4u); }                               \
            }                                                                                      \
        }                                                                                          \
        if (ACTIVE) {                                                                              \
            uint32_t q = R >> shift;                                                               \
            R = (e >> 20) * q + q + m - ((e >> 8) & 0xfffu);                                       \
            acc = __funnelshift_l(acc, e, 24);                                                     \
            lrow = k << lb;                                                                        \
            frow = k * fstride;                                                                    \
        }

    uint32_t s = 0;
    // head: the first word of a segment may be shared with the previous segment -> byte stores
    for (; s < 4 && s < seg; s++) {
        ring_ensure(ring, wr, ipos, 64);
        { RANS_O1_CORE(mine) }
        renorm_safe(R, mine, ring, wr, ipos, in_len);
        if (mine) op[s] = (uint8_t)(acc >> 24);
    }
    if (s == 4) {
        // phase: at unrolled position j the lane's address ends a 4-byte word iff (op+s+j)&3 == 3
        const uint32_t ph = (uint32_t)(reinterpret_cast<uintptr_t>(op) + 4u) & 3u;
        const bool p0 = mine && ph == 3u, p1 = mine && ph == 2u, p2 = mine && ph == 1u, p3 = mine && ph == 0u;
        uint8_t *wp = op + s;                                        // running pointer of the unrolled loop
        uint32_t rel = ipos - wr.ipos0;
        while (s + 4 <= seg && wr.ipos0 + rel + 256u <= in_len) {
            ring_ensure(ring, wr, wr.ipos0 + rel, 256);
            { RANS_O1_CORE(mine) renorm_fast_s(R, mine, ring_a, rel); }
            if (p0) *reinterpret_cast<uint32_t *>(wp - 3) = acc;
            { RANS_O1_CORE(mine) renorm_fast_s(R, mine, ring_a, rel); }
            if (p1) *reinterpret_cast<uint32_t *>(wp - 2) = acc;
            { RANS_O1_CORE(mine) renorm_fast_s(R, mine, ring_a, rel); }
            if (p2) *reinterpret_cast<uint32_t *>(wp - 1) = acc;
            { RANS_O1_CORE(mine) renorm_fast_s(R, mine, ring_a, rel); }
            if (p3) *reinterpret_cast<uint32_t *>(wp) = acc;
            wp += 4;
            s += 4;
        }
        ipos = wr.ipos0 + rel;
        // the last (up to 3) bytes produced by the unrolled loop may not have completed a word
        if (mine) {
            op[s - 1] = (uint8_t)(acc >> 24);
            op[s - 2] = (uint8_t)(acc >> 16);
            op[s - 3] = (uint8_t)(acc >> 8);
        }
        for (; s < seg; s++) {
            ring_ensure(ring, wr, ipos, 64);
            { RANS_O1_CORE(mine) }
            renorm_safe(R, mine, ring, wr, ipos, in_len);
            if (mine) op[s] = (uint8_t)(acc >> 24);
        }
    }
    // the last state also produces the U mod N tail (rANS_static32x16pr.c:669-680)
    const bool last = lane == N - 1;
    for (uint32_t s2 = seg * N; s2 < U; s2++) {
        ring_ensure(ring, wr, ipos, 64);
        { RANS_O1_CORE(last) }
        renorm_safe(R, last, ring, wr, ipos, in_len);
        if (last) out[s2] = (uint8_t)(acc >> 24);
    }
#undef RANS_O1_CORE
}

// Read the N initial states (RansDecInit, rANS_word.h:123) — lane z takes state z.
__device__ int load_states(const uint8_t *p, const uint8_t *end, uint32_t N, uint32_t &R)
{
    const uint32_t lane = hgpu_lane();
    if (end - p < (ptrdiff_t)(4 * N)) return -1;
    R = RANS_L;
    if (lane < N) {
        const uint8_t *q = p + 4 * lane;
        R = q[0] | (uint32_t)q[1] << 8 | (uint32_t)q[2] << 16 | (uint32_t)q[3] << 24;
    }
    return __any_sync(0xffffffffu, R < RANS_L) ? -1 : 0;
}

__device__ __forceinline__ uint32_t table_bytes(uint32_t rows, uint32_t ncol, uint32_t lb)
{ return (((rows << lb) + 15u) & ~15u) + rows * ncol * 4u; }

// full_only: the caller met a row that needs the full form
__device__ Table place_table(uint8_t *smem, const WarpScratch &ws, uint32_t rows, uint32_t ncol, uint32_t shift, bool full_only = false)
{
    Table t;
    (void)smem;
    // compact form: 256 buckets when they fit (the walk is then almost always one step: ncu showed the 64-bucket walk
    // at 40 % of rans_tile4_kernel's instructions on 150-symbol alphabets), else 64
    const uint32_t need_f = table_bytes(rows, ncol, shift);
    uint32_t lb = shift;
    if (!full_only && (ws.compact || need_f > ws.tab_cap)) {
        if (shift > COMPACT_LB_BIG && table_bytes(rows, ncol, COMPACT_LB_BIG) <= ws.tab_cap) lb = COMPACT_LB_BIG;
        else if (table_bytes(rows, ncol, COMPACT_LB) <= ws.tab_cap) lb = COMPACT_LB;
    }
    const uint32_t need = table_bytes(rows, ncol, lb);
    if (need > ws.tab_cap && !ws.gtab) ws.defer = true;                 // caller bails out
    uint8_t *base = need <= ws.tab_cap ? ws.tab_base : ws.gtab;
    t.in_smem = need <= ws.tab_cap;
    t.lut = base;
    t.fb = reinterpret_cast<uint32_t *>(base + (((rows << lb) + 15u) & ~15u));
    t.ncol = ncol;
    t.shift = shift;
    t.lb = lb;
    return t;
}

// order-0 stream: table + states + words  (rans_uncompress_O0_4x16 / _32x16)
__device__ int dec_order0(uint8_t *smem, const WarpScratch &ws, const uint8_t *in, uint32_t in_len,
                          uint8_t *out, uint32_t U, uint32_t N, bool top = false)
{
    uint32_t *F = reinterpret_cast<uint32_t *>(smem + SM_F);
    uint32_t *cum = reinterpret_cast<uint32_t *>(smem + SM_CUM);
    uint8_t *symof = smem + SM_SYMOF;
    const uint32_t lane = hgpu_lane();
    if (in_len < 16) return -1;
    const uint8_t *p = in, *end = in + in_len;
    // the 4-way decoder parses its table against end-8 (rANS_static4x16pr.c:228), the 32-way
    // one against the true end (rANS_static32x16pr.c:272)
    const uint8_t *tend = N == 4 ? end - 8 : end;
    __syncwarp();
    for (int j = lane; j < 256; j += 32) F[j] = 0;
    __syncwarp();
    if (p == tend) return -1;
    p += read_alphabet(p, tend, F);
    __syncwarp();
    // compact alphabet, then one varint per present symbol (decode_freq :254-272)
    uint32_t ncol = 0, tot = 0;
    for (int j = 0; j < 256; j++) {
        if (F[j]) {
            uint32_t f;
            p += vget(p, tend, f);
            tot += f;
            __syncwarp();
            if (lane == 0) { F[ncol] = f; symof[ncol] = (uint8_t)j; }
            __syncwarp();
            ncol++;
        }
    }
    if (p == in) return -1;
    // normalise_freq_shift (:151-162)
    if (tot != 0 && tot != 4096) {
        int sh = 0;
        while (tot < 4096) { tot *= 2; sh++; }
        __syncwarp();
        for (uint32_t k = lane; k < ncol; k += 32) F[k] <<= sh;
        __syncwarp();
    }
    // rans_F_to_s3 (:540-551): every F must fit what is left, and they must sum to 4096
    bool bad = false;
    for (uint32_t k = lane; k < ncol; k += 32) bad |= F[k] > 4096u;
    if (__any_sync(0xffffffffu, bad)) return -1;
    if (warp_cumsum(F, cum, (int)ncol) != 4096u) return -1;
    if (ncol == 0) return -1;
    Table t = place_table(smem, ws, 1, ncol, 12);
    if (ws.defer) return -1;
    fill_row(t, 0, F, cum, symof, N == 32);
    __syncwarp();
    uint32_t R;
    if (load_states(p, end, N, R)) return -1;
    uint32_t ipos = (uint32_t)(p - in) + 4 * N;
    if (top && ws.hook && t.in_smem && ws.hook->mode == (N == 32 ? HOOK_X32 : HOOK_N4)) {
        Hook &h = *ws.hook;
        if (h.Fcap && ncol <= 16) {
            __syncwarp();
            if (lane < 16) h.Fcap[lane] = lane < ncol ? (uint16_t)F[lane] : (uint16_t)0;
            if (lane == 0) h.Fcap[256] = 0;
            __syncwarp();
        }
        h.taken = true; h.order = 0; h.N = N; h.shift = 12; h.ncol = ncol; h.ipos = ipos; h.U = U; h.R = R; h.row0 = 0;
        h.in = in; h.in_len = in_len; h.out = out; h.lut = t.lut; h.fb = t.fb; h.lb = t.lb;
        h.tab_bytes = table_bytes(1, ncol, t.lb);
        return RC_HOOKED;
    }
    if (t.lb != t.shift) loop_order0<true, true>(smem, t, in, in_len, ipos, out, U, N, R);
    else if (t.in_smem)  loop_order0<true>(smem, t, in, in_len, ipos, out, U, N, R);
    else                 loop_order0<false>(smem, t, in, in_len, ipos, out, U, N, R);
    __syncwarp();
    return 0;
}

// order-1 stream (rans_uncompress_O1_4x16 / _32x16; table = decode_freq1, :468-536)
__device__ int dec_order1(uint8_t *smem, const WarpScratch &ws, const uint8_t *in, uint32_t in_len,
                          uint8_t *out, uint32_t U, uint32_t N, bool top = false)
{
    uint32_t *F = reinterpret_cast<uint32_t *>(smem + SM_F);
    uint32_t *cum = reinterpret_cast<uint32_t *>(smem + SM_CUM);
    uint8_t *rowof = smem + SM_ROWOF;
    uint8_t *symof = smem + SM_SYMOF;
    const uint32_t lane = hgpu_lane();
    if (in_len < (N == 4 ? 16u : 4u * N)) return -1;
    const uint8_t *p = in, *end = in + in_len, *tend = end, *after_tab = nullptr;
    const uint32_t shift = *p >> 4;
    if (*p++ & 1) {                       // table is itself order-0 4-way coded (:555-566)
        uint32_t usz, csz;
        p += vget(p, end, usz);
        p += vget(p, end, csz);
        if (csz > (uint32_t)(end - p)) return -1;
        if (usz > TBLBUF_BYTES) return -1;        // documented limit (a real table is < 200 KiB)
        after_tab = p + csz;
        if (dec_order0(smem, ws, p, csz, ws.tblbuf, usz, 4)) return -1;
        __syncwarp();
        __threadfence_block();
        p = ws.tblbuf;
        tend = ws.tblbuf + usz;
    }
    if (shift != 10 && shift != 12) return -1;     // anything else is out of bounds in the reference
    __syncwarp();
    for (int j = lane; j < 256; j += 32) { F[j] = 0; rowof[j] = 0xff; }
    __syncwarp();
    int n = read_alphabet(p, tend, F);
    if (!n) return -1;
    p += n;
    if (p >= tend) return -1;
    __syncwarp();
    // compact alphabet A' = A0 + {0}: byte 0 always owns row/column 0 so the start context
    // exists even in streams that never emit a zero byte.
    uint32_t ncol = 0;
    bool zero_in_a0 = F[0] != 0;
    for (int j = 0; j < 256; j++) {
        if (F[j] || j == 0) {
            __syncwarp();
            if (lane == 0) { rowof[j] = (uint8_t)ncol; symof[ncol] = (uint8_t)j; }
            ncol++;
        }
    }
    __syncwarp();
    Table t = place_table(smem, ws, ncol, ncol, shift);
    if (ws.defer) return -1;
    const uint32_t total = 1u << shift;
    const uint8_t *rows_at = p;
build_rows:
    uint16_t *Fcap = (top && ws.hook && N == 32 && ncol <= 16) ? ws.hook->Fcap : nullptr;
    if (Fcap) {                                   // row 16 = per-row "null row" flags
        __syncwarp();
        for (uint32_t k = lane; k < 17 * 16; k += 32) Fcap[k] = k >= 256 ? (uint16_t)1 : (uint16_t)0;
        __syncwarp();
    }
    for (uint32_t r = 0; r < ncol; r++) {
        if (t.lb != shift && (r == 0 && !zero_in_a0)) goto need_full;
        if (r == 0 && !zero_in_a0) { fill_null_row(t, 0); continue; }
        // decode_freq_d (:425-456): one varint per alphabet symbol, zero followed by a run of zeros
        const uint8_t *q = p;
        uint32_t T = 0;
        int dz = 0;
        if (q == tend) return -1;
        __syncwarp();
        for (uint32_t k = lane; k < ncol; k += 32) F[k] = 0;
        __syncwarp();
        for (uint32_t k = zero_in_a0 ? 0 : 1; k < ncol && q < tend; k++) {
            uint32_t f;
            if (dz) { f = 0; dz--; }
            else {
                q += vget(q, tend, f);
                if (f == 0) { if (q >= tend) return -1; dz = *q++; }
            }
            if (lane == 0) F[k] = f;
            T += f;
        }
        __syncwarp();
        if (q == p) return -1;
        p = q;
        if (!T && t.lb != shift) goto need_full;
        if (!T) { fill_null_row(t, r); continue; }
        if (T != total) {                         // normalise_freq_shift
            int sh = 0; uint32_t tt = T;
            while (tt < total) { tt *= 2; sh++; }
            for (uint32_t k = lane; k < ncol; k += 32) F[k] <<= sh;
            __syncwarp();
        }
        bool bad = false;
        for (uint32_t k = lane; k < ncol; k += 32) bad |= F[k] > total;
        if (__any_sync(0xffffffffu, bad)) return -1;
        if (warp_cumsum(F, cum, (int)ncol) != total) return -1;
        fill_row(t, r, F, cum, symof, false);
        if (Fcap) {
            if (lane < ncol) Fcap[r * 16 + lane] = (uint16_t)F[lane];      // F <= 4096
            if (lane == 0) Fcap[256 + r] = 0;
        }
        __syncwarp();
    }
    if (false) {
need_full:  // a row no valid stream enters exists only in the full form: place the table again and re-read the rows
        __syncwarp();
        t = place_table(smem, ws, ncol, ncol, shift, true);
        if (ws.defer) return -1;
        p = rows_at;
        goto build_rows;
    }
    __syncwarp();
    if (!t.in_smem) __threadfence_block();
    if (after_tab) p = after_tab;
    // p now points into `in` again in every case (an uncompressed table was parsed in place)
    uint32_t R;
    if (load_states(p, end, N, R)) return -1;
    uint32_t ipos = (uint32_t)(p - in) + 4 * N;
    if (top && ws.hook && t.in_smem && ws.hook->mode == (N == 32 ? HOOK_X32 : HOOK_N4)) {
        Hook &h = *ws.hook;
        h.taken = true; h.order = 1; h.N = N; h.shift = shift; h.ncol = ncol; h.ipos = ipos; h.U = U; h.R = R; h.row0 = 0;
        h.in = in; h.in_len = in_len; h.out = out; h.lut = t.lut; h.fb = t.fb; h.lb = t.lb;
        h.tab_bytes = table_bytes(ncol, ncol, t.lb);
        return RC_HOOKED;
    }
    if (t.lb != shift) {
        if (N == 32) loop_order1<true, true, true>(smem, t, in, in_len, ipos, out, U, N, R, 0);
        else         loop_order1<true, false, true>(smem, t, in, in_len, ipos, out, U, N, R, 0);
    } else if (t.in_smem) {
        if (N == 32) loop_order1<true, true>(smem, t, in, in_len, ipos, out, U, N, R, 0);
        else         loop_order1<true, false>(smem, t, in, in_len, ipos, out, U, N, R, 0);
    } else           loop_order1<false, false>(smem, t, in, in_len, ipos, out, U, N, R, 0);
    __syncwarp();
    return 0;
}

// hts_unpack_meta (pack.c:161-196): returns bytes consumed or 0
__device__ int unpack_meta(const uint8_t *d, uint32_t len, uint8_t *map, int &per_byte)
{
    if (!len) return 0;
    uint32_t n = d[0] ? d[0] : 256, j = 1, c = 0;
    if (n <= 1) per_byte = 0;
    else if (n <= 2) per_byte = 8;
    else if (n <= 4) per_byte = 4;
    else if (n <= 16) per_byte = 2;
    else { per_byte = 1; return 1; }
    if (len <= 1) return 0;
    do { map[c++] = d[j++]; } while (c < n && j < len);
    return c < n ? 0 : (int)j;
}

// hts_unpack (pack.c:207-330): out[i] = map[field i of data]; fully parallel.
__device__ int unpack(const uint8_t *d, uint64_t len, uint8_t *out, uint64_t olen, int per_byte,
                      const uint8_t *map)
{
    const uint32_t lane = hgpu_lane();
    if (per_byte == 1) { for (uint64_t i = lane; i < len; i += 32) out[i] = d[i]; return 0; }
    if (per_byte == 0) { for (uint64_t i = lane; i < olen; i += 32) out[i] = map[0]; return 0; }
    int bits = per_byte == 8 ? 1 : per_byte == 4 ? 2 : 4;
    if ((olen + per_byte - 1) / per_byte > len) return -1;
    for (uint64_t i = lane; i < olen; i += 32)
        out[i] = map[(d[i / per_byte] >> (bits * (i % per_byte))) & ((1 << bits) - 1)];
    return 0;
}

// hts_rle_decode (rle.c:142-190).  32 literals per round: ballot which of them carry a run,
// lane 0 walks the run-length varints for those (the only serial part), an exclusive scan of
// the expanded lengths gives every literal its output offset, then all lanes write.
__device__ int unrle(uint8_t *smem, const uint8_t *lit, uint64_t nlit, const uint8_t *run, uint64_t nrun,
                     const uint8_t *syms, int nsyms, uint8_t *out, uint64_t cap, uint64_t &olen)
{
    const uint32_t lane = hgpu_lane();
    uint8_t *flag = smem + SM_ROWOF;                 // 256 B, free outside table building
    uint32_t *rl = reinterpret_cast<uint32_t *>(smem + SM_F);   // 32 run lengths per round
    __syncwarp();
    for (int j = lane; j < 256; j += 32) flag[j] = 0;
    __syncwarp();
    for (int j = lane; j < nsyms; j += 32) flag[syms[j]] = 1;
    __syncwarp();
    const uint8_t *rp = run, *rend = run + nrun;
    uint64_t o = 0;
    for (uint64_t base = 0; base < nlit; base += 32) {
        uint64_t i = base + lane;
        uint8_t b = i < nlit ? lit[i] : 0;
        bool has = i < nlit && flag[b];
        uint32_t bal = __ballot_sync(0xffffffffu, has);
        if (lane == 0) {
            uint32_t mm = bal;
            while (mm) {
                int z = __ffs(mm) - 1;
                mm &= mm - 1;
                uint32_t r;
                rp += vget(rp, rend, r);
                rl[z] = r;
            }
        }
        // every lane must see lane 0's pointer advance
        unsigned long long rp_bits = __shfl_sync(0xffffffffu, (unsigned long long)rp, 0);
        rp = reinterpret_cast<const uint8_t *>(rp_bits);
        __syncwarp();
        uint32_t mylen = i < nlit ? (has ? rl[lane] + 1u : 1u) : 0u;
        // the reference checks literal by literal: a run must leave room for one more byte
        // (outp + rlen >= out_end fails), a plain literal needs outp < out_end
        uint64_t inc = mylen;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            uint64_t tv = __shfl_up_sync(0xffffffffu, inc, d);
            if (lane >= (uint32_t)d) inc += tv;
        }
        uint64_t my_o = o + inc - mylen;
        bool bad = false;
        if (i < nlit) {
            if (my_o >= cap) bad = true;
            else if (has && mylen > 1 && my_o + (mylen - 1) >= cap) bad = true;
        }
        if (__any_sync(0xffffffffu, bad)) return -1;
        if (i < nlit)
            for (uint32_t k = 0; k < mylen; k++) out[my_o + k] = b;
        o += __shfl_sync(0xffffffffu, inc, 31);
        __syncwarp();
    }
    olen = o;
    return 0;
}

// Everything except STRIPE (rans_uncompress_to_4x16, :1675-1873).
__device__ int decode_plain(uint8_t *smem, const WarpScratch &ws, const uint8_t *in, uint32_t in_size,
                            uint8_t *out, uint32_t out_cap, uint32_t &out_size)
{
    const uint32_t lane = hgpu_lane();
    const uint8_t *end = in + in_size;
    uint8_t fmt = *in++; in_size--;
    const uint32_t N = (fmt & 0x04) ? 32 : 4;
    const int order = fmt & 1;
    uint32_t osz;
    if (!(fmt & 0x10)) { int s = vget(in, end, osz); in += s; in_size -= s; }
    else osz = out_cap;
    if (out_cap < osz) return -1;
    if (osz > ws.max_out) return -1;                // scratch was sized from the caller's bound
    out_size = osz;
    uint32_t t1_size = osz;
    uint8_t *t1, *t2, *t3, *tmp = ws.tmp;
    if ((fmt & 0xc0) == 0xc0) { t1 = out; t2 = tmp; t3 = out; }
    else if (fmt & 0x80)      { t1 = tmp; t2 = tmp; t3 = out; }
    else if (fmt & 0x40)      { t1 = tmp; t2 = out; t3 = out; }
    else                      { t1 = t2 = t3 = out; }

    uint8_t map[16];
    for (int k = 0; k < 16; k++) map[k] = 0;
    int per_byte = 0;
    uint64_t unpacked = 0;
    if (fmt & 0x80) {                               // PACK meta (:1748-1767)
        int m = unpack_meta(in, in_size, map, per_byte);
        if (!m) return -1;
        unpacked = osz;
        in += m; in_size -= m;
        uint32_t psz;
        int s = vget(in, end, psz);
        in += s; in_size -= s;
        if (psz > t1_size) return -1;
        t1_size = psz;
    }
    const uint8_t *meta = nullptr;
    uint32_t u_meta = 0;
    if (fmt & 0x40) {                               // RLE meta (:1769-1796)
        uint32_t rle_len, c_meta, s;
        s = vget(in, end, u_meta);
        s += vget(in + s, end, rle_len);
        if (rle_len > t1_size) return -1;
        if (u_meta & 1) {
            meta = in + s;
            u_meta = (u_meta / 2 > (uint32_t)(end - meta)) ? (uint32_t)(end - meta) : u_meta / 2;
            c_meta = u_meta;
        } else {
            s += vget(in + s, end, c_meta);
            u_meta /= 2;
            if (u_meta > ws.max_out + 1024u) return -1;      // documented limit
            if (s > in_size) return -1;
            if (dec_order0(smem, ws, in + s, in_size - s, ws.meta, u_meta, N)) return -1;
            __syncwarp();
            __threadfence_block();
            meta = ws.meta;
        }
        if (c_meta + s > in_size) return -1;
        in += c_meta + s; in_size -= c_meta + s;
        t1_size = rle_len;
    }
    if (in_size) {
        if (fmt & 0x20) {                           // CAT
            if (t1_size > in_size || t1_size > out_size) return -1;
            for (uint32_t i = lane; i < t1_size; i += 32) t1[i] = in[i];
        } else {
            // only a stream with no transform may hand its symbol loop to the hooks (t1 == out then)
            const bool top = !(fmt & 0xc0) && ws.hook != nullptr;
            int rc = order ? dec_order1(smem, ws, in, in_size, t1, t1_size, N, top)
                           : dec_order0(smem, ws, in, in_size, t1, t1_size, N, top);
            if (rc == RC_HOOKED) return RC_HOOKED;
            if (rc) return -1;
        }
    } else
        t1_size = 0;
    __syncwarp();
    __threadfence_block();
    uint64_t t2_size = t1_size, t3_size;
    if (fmt & 0x40) {
        if (u_meta == 0) return -1;
        int ns = meta[0] ? meta[0] : 256;
        if (u_meta < (uint32_t)(1 + ns)) return -1;
        uint64_t got = 0;
        if (unrle(smem, t1, t1_size, meta + 1 + ns, u_meta - (1 + ns), meta + 1, ns, t2, out_size, got)) return -1;
        t2_size = got;
        __syncwarp();
        __threadfence_block();
    }
    t3_size = t2_size;
    if (fmt & 0x80) {
        if (per_byte == 1) unpacked = t2_size;
        if (unpack(t2, t2_size, t3, unpacked, per_byte, map)) return -1;
        t3_size = unpacked;
    }
    out_size = (uint32_t)t3_size;
    return 0;
}

__device__ int decode_stream(uint8_t *smem, const WarpScratch &ws, const uint8_t *in, uint32_t in_size,
                             uint8_t *out, uint32_t out_cap, uint32_t &out_size)
{
    const uint32_t lane = hgpu_lane();
    if (in_size == 0) return -1;
    // pass 0 runs with no transform scratch: PACK / RLE / STRIPE streams go to pass 1
    if (ws.pass == 0 && (in[0] & 0xc8)) { ws.defer = true; return -1; }
    if (!(in[0] & 0x08)) return decode_plain(smem, ws, in, in_size, out, out_cap, out_size);

    // STRIPE (:1594-1673): N sub-streams, byte-plane transposed
    const uint8_t *end = in + in_size;
    uint32_t ulen, off = 1;
    off += vget(in + off, end, ulen);
    if (off >= in_size) return -1;
    uint32_t n = in[off++];
    if (n < 1) return -1;
    if (ulen != out_cap) return -1;
    if (ulen > ws.max_out) return -1;
    // first pass over the length table: validate exactly as the reference does
    uint64_t ctot = 0;
    uint32_t off2 = off;
    for (uint32_t k = 0; k < n; k++) {
        uint32_t cl;
        off2 += vget(in + off2, end, cl);
        ctot += cl;
        if (off2 > in_size || cl > in_size || cl < 1) return -1;
    }
    if (off2 + ctot > in_size) return -1;
    in_size = (uint32_t)(off2 + ctot);
    uint32_t data = off2, idx = 0;
    for (uint32_t k = 0; k < n; k++) {
        uint32_t cl;
        off += vget(in + off, end, cl);
        uint32_t ul = ulen / n + ((ulen % n) > k), got = 0;
        if (in_size < data) return -1;
        if (in_size - data == 0) return -1;
        if (in[data] & 0x08) return -1;             // nested STRIPE: never written by the encoder; unsupported
        if (decode_plain(smem, ws, in + data, in_size - data, ws.planes + idx, ul, got) || got != ul) return -1;
        data += cl;
        idx += ul;
    }
    __syncwarp();
    __threadfence_block();
    // unstripe (utils.h:79-138): out[j] = plane[j % n][j / n]
    const uint32_t q = ulen / n, r = ulen % n;
    for (uint32_t j = lane; j < ulen; j += 32) {
        uint32_t k = j % n, i = j / n;
        uint32_t start = k * q + (k < r ? k : r);
        out[j] = ws.planes[start + i];
    }
    out_size = ulen;
    return 0;
}

constexpr int32_t RANS_DEFERRED = 1;       // internal: written by pass 0, consumed by pass 1

template <int PASS>
__global__ void __launch_bounds__(32, PASS == 0 ? 24 : 10)
rans_nx16_decode_kernel(const uint8_t *__restrict__ in, const uint64_t *__restrict__ in_off,
                        const uint32_t *__restrict__ in_len, uint32_t n, uint8_t *out,
                        const uint64_t *__restrict__ out_off, const uint32_t *__restrict__ out_len,
                        uint32_t *got_len, int32_t *status, uint8_t *scratch, size_t scratch_per_cta,
                        uint32_t max_out, uint32_t smem_tab_bytes, uint32_t *counter)
{
    extern __shared__ __align__(16) uint8_t smem[];
    WarpScratch ws;
    uint8_t *base = scratch + (size_t)blockIdx.x * scratch_per_cta;
    size_t mo = ((size_t)max_out + 255) & ~(size_t)255;
    ws.tmp = base;
    ws.planes = base + mo;
    ws.meta = base + 2 * mo;
    ws.tblbuf = base + 3 * mo + 1024;
    ws.gtab = ws.tblbuf + TBLBUF_BYTES;
    ws.max_out = max_out;
    ws.tab_base = smem + SM_TAB;
    ws.tab_cap = smem_tab_bytes;
    ws.pass = PASS;
    ws.defer = false;
    ws.hook = nullptr;
    if (PASS == 0) { ws.tmp = ws.planes = ws.meta = ws.gtab = nullptr; ws.tblbuf = base; }
    for (;;) {
        uint32_t job = 0;
        if (hgpu_lane() == 0) job = atomicAdd(counter, 1u);
        job = __shfl_sync(0xffffffffu, job, 0);
        if (job >= n) break;
        if (PASS == 1 && status[job] != RANS_DEFERRED) continue;
        uint32_t got = 0;
        int rc = decode_stream(smem, ws, in + in_off[job], in_len[job], out + out_off[job], out_len[job], got);
        __syncwarp();
        if (hgpu_lane() == 0) {
            status[job] = ws.defer ? RANS_DEFERRED : rc ? HGPU_RANS_ERR : HGPU_OK;
            got_len[job] = rc ? 0 : got;
        }
        ws.defer = false;
    }
}


#include "rans_nx16_fast.cuh"

// =============================================================================================
// rANS 4x8 (CRAM 3.0 block method 4, "RANS") — replaces rans_uncompress / rans_uncompress_O0/_O1
// (htscodecs rANS_static.c:840-850, :221-384, :599-827).  One warp per stream, the four states on
// lanes 0-3; renormalisation is byte-wise (L = 2^23, 0-2 bytes per state and step, taken in state
// order: lane z starts at the prefix sum of the lower lanes' byte counts, rANS_byte.h:512-554).
// Tables live in the per-CTA global scratch (a 3.0-era format: correctness first).
// =============================================================================================
constexpr uint32_t L8 = 1u << 23;

__device__ __forceinline__ void renorm8(uint32_t &R, bool active, const uint8_t *in, uint32_t &ipos, uint32_t in_len)
{
    const uint32_t lane = hgpu_lane();
    uint32_t c = !active || R >= L8 ? 0u : (R < (1u << 15) ? 2u : 1u);
    uint32_t b1 = __ballot_sync(0xffffffffu, c >= 1), b2 = __ballot_sync(0xffffffffu, c == 2);
    if (!b1) return;
    uint32_t lt = hgpu_lanemask_lt();
    uint32_t off = __popc(b1 & lt) + __popc(b2 & lt), tot = __popc(b1) + __popc(b2);
    uint32_t avail = in_len - ipos;                                  // ipos <= in_len always
    uint32_t start = off < avail ? off : avail;
    uint32_t n = c < avail - start ? c : avail - start;
    if (n >= 1) R = (R << 8) | in[ipos + start];
    if (n == 2) R = (R << 8) | in[ipos + start + 1];
    ipos += tot < avail ? tot : avail;
    (void)lane;
}

// returns 0 ok / -1 error; out_size = decoded length
__device__ int dec_4x8(uint8_t *gtab, const uint8_t *in, uint32_t in_size, uint8_t *out, uint32_t out_cap, uint32_t &out_size)
{
    const uint32_t lane = hgpu_lane();
    if (in_size < 26) return -1;
    const uint32_t order = in[0];
    if (order > 1) return -1;
    const uint32_t in_sz = in[1] | in[2] << 8 | in[3] << 16 | (uint32_t)in[4] << 24;
    const uint32_t out_sz = in[5] | in[6] << 8 | in[7] << 16 | (uint32_t)in[8] << 24;
    if (in_sz != in_size - 9 || out_sz > out_cap) return -1;
    if (order && in_size < 27) return -1;
    uint8_t *lut = gtab;                                             // [rows][4096]
    uint32_t *fs = reinterpret_cast<uint32_t *>(gtab + 256u * 4096u); // [rows][256]  f | start<<16
    const uint8_t *cp = in + 9, *end = in + in_size;
    uint32_t R = L8;
    if (!order) {
        int j = *cp++, rle = 0;
        uint32_t x = 0, lastF = 0, lastj = 0;
        do {
            if (cp > end - 16) return -1;
            uint32_t F = *cp++;
            if (F >= 128) F = ((F & 127) << 8) | *cp++;
            if (x + F > 4096) return -1;
            for (uint32_t y = lane; y < F; y += 32) lut[x + y] = (uint8_t)j;
            if (lane == 0) fs[j] = F | (x << 16);
            lastF = F; lastj = (uint32_t)j;
            x += F;
            if (!rle && j + 1 == *cp) { j = *cp++; rle = *cp++; }
            else if (rle) { rle--; if (++j > 255) return -1; }
            else j = *cp++;
        } while (j);
        if (x < 4095 || x > 4096) return -1;
        // slot 4095 of a 4095-sum table repeats the last symbol with bias+1 (:299-305): give that
        // symbol one more slot by widening its frequency entry
        if (x != 4096 && lane == 0) lut[4095] = (uint8_t)lastj;      // bias = m - start comes out as sbase[4094]+1
        (void)lastF;
        const bool short_tab = x != 4096;
        if (cp > end - 16) return -1;
        if (lane < 4) { const uint8_t *q = cp + 4 * lane; R = q[0] | q[1] << 8 | q[2] << 16 | (uint32_t)q[3] << 24; }
        if (__any_sync(0xffffffffu, R < L8)) return -1;
        uint32_t ipos = (uint32_t)(cp - in) + 16;
        __syncwarp();
        __threadfence_block();
        const bool mine = lane < 4;
        uint32_t i = 0;
        for (; i + 4 <= out_sz; i += 4) {
            uint32_t m = R & 4095u, sym = lut[m], e = fs[sym];
            if (mine) {
                uint32_t f = e & 0xffffu, st = e >> 16;
                // reference: sfreq[m]*(R>>12) + sbase[m]; for the patched slot sbase = last bias + 1 = m - start
                (void)short_tab;
                R = f * (R >> 12) + m - st;
                out[i + lane] = (uint8_t)sym;
            }
            renorm8(R, mine, in, ipos, in_size);
        }
        if (mine && i + lane < out_sz) out[i + lane] = lut[R & 4095u];
    } else {
        // context rows are numbered in order of first appearance as context or symbol (:636-652)
        uint16_t *map = reinterpret_cast<uint16_t *>(gtab + 256u * 4096u + 256u * 256u * 4u);   // 512 bytes after the tables
        __syncwarp();
        for (uint32_t k = lane; k < 256; k += 32) map[k] = 0xffff;
        for (uint32_t k = lane; k < 256u * 256u; k += 32) fs[k] = 0;
        __syncwarp();
        __threadfence_block();
        uint32_t mi = 0;
        int ci = *cp++, rle_i = 0;
        do {
            if (map[ci] == 0xffff) { __syncwarp(); if (lane == 0) map[ci] = (uint16_t)mi; mi++; __syncwarp(); __threadfence_block(); }
            const uint32_t row = map[ci];
            uint32_t x = 0;
            int j = *cp++, rle_j = 0;
            do {
                if (map[j] == 0xffff) { __syncwarp(); if (lane == 0) map[j] = (uint16_t)mi; mi++; __syncwarp(); __threadfence_block(); }
                if (cp > end - 16) return -1;
                uint32_t F = *cp++;
                if (F >= 128) F = ((F & 127) << 8) | *cp++;
                if (!F) F = 4096;
                if (x + F > 4096) return -1;
                for (uint32_t y = lane; y < F; y += 32) lut[row * 4096u + x + y] = (uint8_t)j;
                if (lane == 0) fs[row * 256u + j] = (F & 0xffffu) | (x << 16);
                x += F;
                if (!rle_j && j + 1 == *cp) { j = *cp++; rle_j = *cp++; }
                else if (rle_j) { rle_j--; if (++j > 255) return -1; }
                else j = *cp++;
            } while (j);
            if (x < 4095 || x > 4096) return -1;
            if (x != 4096 && lane == 0) lut[row * 4096u + 4095u] = 0;   // calloc'd slot in the reference
            if (!rle_i && ci + 1 == *cp) { ci = *cp++; rle_i = *cp++; }
            else if (rle_i) { rle_i--; if (++ci > 255) return -1; }
            else ci = *cp++;
        } while (ci);
        __syncwarp();
        __threadfence_block();
        if (cp > end - 16) return -1;
        if (lane < 4) { const uint8_t *q = cp + 4 * lane; R = q[0] | q[1] << 8 | q[2] << 16 | (uint32_t)q[3] << 24; }
        if (__any_sync(0xffffffffu, R < L8)) return -1;
        uint32_t ipos = (uint32_t)(cp - in) + 16;
        const bool mine = lane < 4;
        const uint32_t q4 = out_sz >> 2;
        uint32_t l = map[0] == 0xffff ? 0u : map[0];
        uint8_t *op = out + (size_t)(mine ? lane : 0) * q4;
        for (uint32_t i = 0; i < q4; i++) {
            uint32_t m = R & 4095u, c = lut[l * 4096u + m], e = fs[l * 256u + c];
            if (mine) {
                uint32_t f = e & 0xffffu;
                R = f * (R >> 12) + m - (e >> 16);
                op[i] = (uint8_t)c;
            }
            renorm8(R, mine, in, ipos, in_size);
            uint16_t ml = map[c];
            if (mine) l = ml == 0xffff ? 0u : ml;
        }
        const bool last = lane == 3;
        for (uint32_t p = 4 * q4; p < out_sz; p++) {
            uint32_t m = R & 4095u, c = lut[l * 4096u + m], e = fs[l * 256u + c];
            if (last) {
                uint32_t f = e & 0xffffu;
                R = f * (R >> 12) + m - (e >> 16);
                out[p] = (uint8_t)c;
            }
            renorm8(R, last, in, ipos, in_size);
            uint16_t ml = map[c];
            if (last) l = ml == 0xffff ? 0u : ml;
        }
    }
    out_size = out_sz;
    return 0;
}

__global__ void __launch_bounds__(32)
rans_4x8_decode_kernel(const uint8_t *__restrict__ in, const uint64_t *__restrict__ in_off,
                       const uint32_t *__restrict__ in_len, uint32_t n, uint8_t *out,
                       const uint64_t *__restrict__ out_off, const uint32_t *__restrict__ out_len,
                       uint32_t *got_len, int32_t *status, uint8_t *scratch, size_t per_cta, uint32_t *counter)
{
    uint8_t *gtab = scratch + (size_t)blockIdx.x * per_cta;
    for (;;) {
        uint32_t job = 0;
        if (hgpu_lane() == 0) job = atomicAdd(counter, 1u);
        job = __shfl_sync(0xffffffffu, job, 0);
        if (job >= n) break;
        uint32_t got = 0;
        int rc = dec_4x8(gtab, in + in_off[job], in_len[job], out + out_off[job], out_len[job], got);
        __syncwarp();
        if (hgpu_lane() == 0) { status[job] = rc ? HGPU_RANS_ERR : HGPU_OK; got_len[job] = rc ? 0 : got; }
    }
}

} // namespace

// 32-way streams the fast kernel keeps resident at once (persistent grid size): callers that can
// choose their batch size should use a multiple of it.
static uint32_t g_f32_smem[64];        // per device: dynamic shared bytes of the fast32 kernel

static uint32_t f32_smem(hgpu_ctx *ctx) { int d = ctx->device; return d >= 0 && d < 64 && g_f32_smem[d] ? g_f32_smem[d] : F32_SMEM + F32_LUT; }

static int rans_attrs(hgpu_ctx *ctx)
{
    // function attributes are per device: set them once per device, not once per process
    static bool done[64];
    int dev = ctx->device;
    if (dev >= 0 && dev < 64 && done[dev]) return 0;
    {   // fast32 wants its LUTs 4 KiB aligned in the shared window: probe where the window starts
        uint32_t *d_o = nullptr, base = 0;
        if (hgpu_check(cudaMalloc(&d_o, 4), "probe alloc")) return -1;
        rans_smem_probe_kernel<<<1, 32, 1024>>>(d_o);
        cudaError_t e = cudaMemcpy(&base, d_o, 4, cudaMemcpyDeviceToHost);
        cudaFree(d_o);
        if (hgpu_check(e, "smem probe")) return -1;
        uint32_t lut0 = (base + F32_WARPS * F32_RING + F32_LUT - 1) & ~(F32_LUT - 1);
        if (dev >= 0 && dev < 64) g_f32_smem[dev] = lut0 + F32_WARPS * (F32_LUT + F32_FB) - base;
    }
    if (hgpu_check(cudaFuncSetAttribute(rans_nx16_decode_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(SM_TAB + 18 * 1024)), "rans smem attr") ||
        hgpu_check(cudaFuncSetAttribute(rans_prep32_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)PREP_SMEM), "rans smem attr") ||
        hgpu_check(cudaFuncSetAttribute(rans_tile4_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)T4_SMEM), "rans smem attr") ||
        hgpu_check(cudaFuncSetAttribute(rans_fast32_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)f32_smem(ctx)), "rans smem attr"))
        return -1;
    if (dev >= 0 && dev < 64) done[dev] = true;
    return 0;
}

extern "C" uint32_t hgpu_rans_nx16_wave_size(hgpu_ctx *ctx)
{
    if (!ctx) return 0;
    if (cudaSetDevice(ctx->device) != cudaSuccess || rans_attrs(ctx)) return 0;
    int per_sm = 0;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, rans_fast32_kernel, F32_WARPS * 32, f32_smem(ctx)) != cudaSuccess) return 0;
    return (uint32_t)ctx->sm_count * (uint32_t)(per_sm < 1 ? 1 : per_sm) * F32_WARPS;
}

int hgpu_launch_rans_nx16(hgpu_ctx *ctx, const uint8_t *d_in, const uint64_t *d_in_off,
                          const uint32_t *d_in_len, uint32_t n, uint8_t *d_out,
                          const uint64_t *d_out_off, const uint32_t *d_out_len,
                          uint32_t *d_got_len, int32_t *d_status, uint32_t max_out_len,
                          cudaStream_t st)
{
    if (n == 0) return HGPU_OK;
    // Five launches over one job list, no host synchronisation in between:
    //  classify  format byte -> ordered lists of plain 32-way and plain 4-way streams; the rest is "deferred"
    //  prep32    32-way plain streams: header + table; small alphabets become fast32 jobs (after 4 head
    //            steps), the others are decoded there with the general loops (table <= 6.5 KiB) or deferred
    //  tile4     4-way plain streams, eight per warp
    //  fast32    the symbol loop of the 32-way jobs, 44 streams per SM
    //  general   everything deferred: PACK / RLE / STRIPE / CAT, big tables (18 KiB shared, else global)
    if (hgpu_check(cudaSetDevice(ctx->device), "cudaSetDevice") || rans_attrs(ctx)) return HGPU_ERR_CUDA;
    const uint32_t smem1 = SM_TAB + 18 * 1024;
    int per_prep = 0, per_t4 = 0, per_f32 = 0, per_gen = 0;
    if (hgpu_check(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_prep, rans_prep32_kernel, 32, PREP_SMEM), "rans occupancy") ||
        hgpu_check(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_t4, rans_tile4_kernel, 32, T4_SMEM), "rans occupancy") ||
        hgpu_check(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_f32, rans_fast32_kernel, F32_WARPS * 32, f32_smem(ctx)), "rans occupancy") ||
        hgpu_check(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_gen, rans_nx16_decode_kernel<1>, 32, smem1), "rans occupancy"))
        return HGPU_ERR_CUDA;
    auto grid_of = [&](int per_sm, uint32_t units) {
        uint32_t g = (uint32_t)ctx->sm_count * (uint32_t)(per_sm < 1 ? 1 : per_sm);
        return g > units ? (units ? units : 1u) : g;
    };
    const uint32_t g_prep = grid_of(per_prep, n), g_t4 = grid_of(per_t4, (n + 7) / 8 + 1);
    const uint32_t g_f32 = grid_of(per_f32, (n + F32_WARPS - 1) / F32_WARPS), g_gen = grid_of(per_gen, n);
    // scratch: [lists 2n u32][counts 4 u32][fast jobs n] | per-CTA areas of the pass that is running
    const size_t lists_b = ((size_t)2 * n * 4 + 255) & ~(size_t)255;
    const size_t jobs_b = (((size_t)n * sizeof(FastJob)) + 255) & ~(size_t)255;
    const size_t fixed = lists_b + 256 + jobs_b;
    const size_t mo = ((size_t)max_out_len + 255) & ~(size_t)255;
    const size_t per_small = TBLBUF_BYTES;
    const size_t per_gen_b = (3 * mo + 1024 + TBLBUF_BYTES + GTAB_BYTES + 255) & ~(size_t)255;
    size_t area = per_small * g_prep;
    if (per_small * g_t4 > area) area = per_small * g_t4;
    if (per_gen_b * g_gen > area) area = per_gen_b * g_gen;
    int rc = hgpu_ensure_scratch(ctx, fixed + area);
    if (rc) return rc;
    uint8_t *sc = ctx->d_scratch;
    uint32_t *list32 = reinterpret_cast<uint32_t *>(sc), *list4 = list32 + n;
    uint32_t *counts = reinterpret_cast<uint32_t *>(sc + lists_b);
    FastJob *jobs = reinterpret_cast<FastJob *>(sc + lists_b + 256);
    uint8_t *percta = sc + fixed;
    uint32_t *c_prep = hgpu_take_counter(ctx, st), *c_t4 = hgpu_take_counter(ctx, st), *c_f32 = hgpu_take_counter(ctx, st);
    uint32_t *c_gen = hgpu_take_counter(ctx, st), *njobs = hgpu_take_counter(ctx, st);
    if (!c_prep || !c_t4 || !c_f32 || !c_gen || !njobs) return HGPU_ERR_CUDA;
    rans_classify_kernel<<<1, 1024, 0, st>>>(d_in, d_in_off, d_in_len, n, d_status, list32, list4, counts);
    rans_prep32_kernel<<<g_prep, 32, PREP_SMEM, st>>>(d_in, d_in_off, d_in_len, list32, counts, d_out, d_out_off, d_out_len,
                                                      d_got_len, d_status, percta, per_small, max_out_len, jobs, njobs, c_prep);
    rans_tile4_kernel<<<g_t4, 32, T4_SMEM, st>>>(d_in, d_in_off, d_in_len, list4, counts, d_out, d_out_off, d_out_len,
                                                 d_got_len, d_status, percta, per_small, max_out_len, c_t4);
    rans_fast32_kernel<<<g_f32, F32_WARPS * 32, f32_smem(ctx), st>>>(jobs, njobs, d_in, d_in_off, d_in_len, d_out, d_out_off, d_out_len,
                                                                     d_status, c_f32, f32_smem(ctx));
    rans_nx16_decode_kernel<1><<<g_gen, 32, smem1, st>>>(d_in, d_in_off, d_in_len, n, d_out, d_out_off, d_out_len,
                                                         d_got_len, d_status, percta, per_gen_b,
                                                         max_out_len, 18 * 1024, c_gen);
    hgpu_count_launch(5);
    return hgpu_check(cudaGetLastError(), "rans launch");
}

// rANS 4x8 batch decode, device pointers (CRAM 3.0 method 4; cram_io.c:1666-1682)
extern "C" int hgpu_rans4x8_decode_batch_dev(hgpu_ctx *ctx, const uint8_t *d_in, const uint64_t *d_in_off,
        const uint32_t *d_in_len, uint32_t n, uint8_t *d_out, const uint64_t *d_out_off, const uint32_t *d_out_len,
        uint32_t *d_got_len, int32_t *d_status, void *stream)
{
    if (!ctx) { hgpu_set_error("null context"); return HGPU_ERR_ARG; }
    if (n == 0) return HGPU_OK;
    cudaStream_t st = stream ? (cudaStream_t)stream : ctx->stream;
    uint32_t grid = (uint32_t)ctx->sm_count * 16u;
    if (grid > n) grid = n;
    size_t per_cta = (GTAB_BYTES + 1024 + 255) & ~(size_t)255;
    int rc = hgpu_ensure_scratch(ctx, per_cta * grid);
    if (rc) return rc;
    uint32_t *counter = hgpu_take_counter(ctx, st);
    if (!counter) return HGPU_ERR_CUDA;
    rans_4x8_decode_kernel<<<grid, 32, 0, st>>>(d_in, d_in_off, d_in_len, n, d_out, d_out_off, d_out_len, d_got_len,
                                                d_status, ctx->d_scratch, per_cta, counter);
    hgpu_count_launch();
    return hgpu_check(cudaGetLastError(), "rans4x8 launch");
}
