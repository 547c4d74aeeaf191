// rANS Nx16 ("RANS_PR", CRAM 3.1 method 5) ENCODER for sm_90a — order 0 / order 1, 4-way or
// 32-way (X32), PACK, RLE, STRIPE (with the per-part method trial) and the CAT fallback; one warp per stream.
//
// Stands where rans_compress_to_4x16 -> rans_compress_O0/O1_4x16 / _32x16 stand in the reference
// (htscodecs rANS_static4x16pr.c:1203-1579, :112-211, :402-497; rANS_static32x16pr.c:67-252,
// :412-525; table writer rANS_static16_int.h:165-421).  Compressed bytes need not equal the
// reference's (SURVEY.md §8c: encoder byte parity is unpinned) — what is pinned is that the
// reference's decoder, the oracle and our own decoder all return the input (tests/test_gpu_rans_enc.py).
//
// The N states live one per lane, mirroring the decoder: symbols are encoded backwards, the lanes
// that must renormalise in a step are found with a ballot, and their 16-bit words are laid down
// below the previous ones in lane order — the exact reverse of the decoder's
// `base + popc(ballot & lanemask_lt)` read order.  Frequencies: warp-aggregated shared/global
// histograms (__match_any_sync), normalised to 2^12 (order 0) or 2^10 / 2^12 per context
// (order 1) so that every present symbol keeps f >= 1.
#include "hgpu_internal.h"
#include "xform_dev.cuh"

namespace {

constexpr uint32_t RANS_L = 1u << 15;
constexpr uint32_t ENC_TAB_SMEM = 16 * 1024;          // {f,start} table: smem when A*A*4 fits
constexpr uint32_t ENC_NEST_TBL = 256 * 256 * 4 + 256 * 1024;   // table text of the nested order-0 coder (compressed order-1 tables)
constexpr uint32_t ENC_NEST_OUT = ENC_NEST_TBL + 2048, ENC_NEST_CAP = 160 * 1024;
constexpr uint32_t ENC_SCRATCH = ENC_NEST_OUT + ENC_NEST_CAP;     // per-warp: full table + table text + nested coder

constexpr uint32_t F_ORDER = 1, F_X32 = 4, F_STRIPE = 8, F_NOSZ = 0x10, F_CAT = 0x20, F_RLE = 0x40, F_PACK = 0x80,
                   F_STRIPE_NO0 = 1u << 16;                            // rANS_static4x16.h:75-100
constexpr uint32_t ENC_FAIL = 0xffffffffu;

// Per-warp transform buffers (global memory, carved by the launcher when a job asks for PACK / RLE / STRIPE):
// P packed bytes, R run-length literals, M run-length meta-data, S the transposed input of a STRIPE job followed by
// its part lengths, B the best candidate of the part being tried.  X = bytes each can take (0: none were carved).
struct XBuf { uint8_t *P, *R, *M, *S, *B; uint32_t X; };
constexpr uint32_t XB_PAD_M = 1024, XB_PAD_S = 2048, XB_PAD_B = 4096;
__host__ __device__ inline size_t xbuf_bytes(uint32_t X) { return X ? 5 * (size_t)X + XB_PAD_M + XB_PAD_S + XB_PAD_B : 0; }

struct EncSmem {
    uint32_t cnt[256];        // order-0 histogram / row scratch
    uint32_t cum[257];
    uint8_t  idxof[256];      // byte -> compact index
    uint8_t  symof[256];      // compact index -> byte
    uint32_t tab[ENC_TAB_SMEM / 4];
};

__device__ int vput(uint8_t *p, uint32_t v)          // var_put_u32, varint.h:206
{
    int n = 0;
    if (v >= (1u << 28)) p[n++] = ((v >> 28) & 0x7f) | 128;
    if (v >= (1u << 21)) p[n++] = ((v >> 21) & 0x7f) | 128;
    if (v >= (1u << 14)) p[n++] = ((v >> 14) & 0x7f) | 128;
    if (v >= (1u << 7))  p[n++] = ((v >> 7) & 0x7f) | 128;
    p[n++] = v & 0x7f;
    return n;
}

// Warp: normalise cnt[0..n) (n <= 256, total > 0) in place to sum exactly M with every non-zero
// count >= 1.  Returns false if impossible (more symbols than M).
__device__ bool normalise_row(uint32_t *cnt, int n, uint32_t M)
{
    const uint32_t lane = hgpu_lane();
    uint64_t tot = 0;
    uint32_t present = 0;
    for (int j = lane; j < n; j += 32) { tot += cnt[j]; present += cnt[j] != 0; }
    for (int d = 16; d > 0; d >>= 1) { tot += __shfl_xor_sync(0xffffffffu, tot, d); present += __shfl_xor_sync(0xffffffffu, present, d); }
    if (tot == 0) return true;
    if (present > M) return false;
    __syncwarp();
    int64_t sum = 0;
    uint32_t best = 0, besti = 0;
    for (int j = lane; j < n; j += 32) {
        uint32_t c = cnt[j];
        if (!c) continue;
        uint32_t f = (uint32_t)(((uint64_t)c * M) / tot);
        if (f == 0) f = 1;
        cnt[j] = f;
        sum += f;
        if (f > best) { best = f; besti = j; }
    }
    for (int d = 16; d > 0; d >>= 1) {
        sum += __shfl_xor_sync(0xffffffffu, sum, d);
        uint32_t ob = __shfl_xor_sync(0xffffffffu, best, d), oi = __shfl_xor_sync(0xffffffffu, besti, d);
        if (ob > best || (ob == best && oi < besti)) { best = ob; besti = oi; }
    }
    __syncwarp();
    int64_t diff = (int64_t)M - sum;
    if (diff > 0) { if (lane == 0) cnt[besti] += (uint32_t)diff; __syncwarp(); return true; }
    // too much (the f>=1 bumps): take it back from the largest entries
    while (diff < 0) {
        uint32_t b = 0, bi = 0;
        for (int j = lane; j < n; j += 32) { uint32_t f = cnt[j]; if (f > b) { b = f; bi = j; } }
        for (int d = 16; d > 0; d >>= 1) {
            uint32_t ob = __shfl_xor_sync(0xffffffffu, b, d), oi = __shfl_xor_sync(0xffffffffu, bi, d);
            if (ob > b || (ob == b && oi < bi)) { b = ob; bi = oi; }
        }
        if (b <= 1) return false;
        uint32_t take = (uint32_t)min((int64_t)(b - 1), -diff);
        __syncwarp();
        if (lane == 0) cnt[bi] -= take;
        __syncwarp();
        diff += take;
    }
    return true;
}

// alphabet writer (encode_alphabet, rANS_static16_int.h:165-189); present[] != 0 marks symbols
__device__ int put_alphabet(uint8_t *cp, const uint32_t *present)
{
    uint8_t *op = cp;
    int rle = 0;
    for (int j = 0; j < 256; j++) {
        if (!present[j]) continue;
        if (rle) { rle--; continue; }
        *cp++ = (uint8_t)j;
        if (j && present[j - 1]) {
            int r = j + 1;
            while (r < 256 && present[r]) r++;
            rle = r - (j + 1);
            *cp++ = (uint8_t)rle;
        }
    }
    *cp++ = 0;
    return (int)(cp - op);
}

__device__ __forceinline__ uint32_t enc_put(uint32_t x, uint32_t f, uint32_t start, uint32_t shift)
{
    return ((x / f) << shift) + (x % f) + start;
}

// The entropy coder proper (rans_enc_func(do_simd, order): rans_compress_O0/O1_4x16, _32x16): frequency table,
// N states, 16-bit words; no format byte, no size.  U > 0.  Returns the bytes written at out, or ENC_FAIL when they
// do not fit in cap.
template <bool nested = false>
__device__ uint32_t encode_core(EncSmem &s, uint8_t *scratch, const uint8_t *in, uint32_t U, uint32_t order, uint32_t N,
                                uint8_t *out, uint32_t cap)
{
    const uint32_t lane = hgpu_lane();
    const uint32_t hdr = 0;
    if (cap < 16) return ENC_FAIL;
    // ---- alphabet (order-0 histogram, warp-aggregated) ----
    __syncwarp();
    for (int j = lane; j < 256; j += 32) s.cnt[j] = 0;
    __syncwarp();
    for (uint32_t base = 0; base < U; base += 32) {
        uint32_t p = base + lane;
        bool act = p < U;
        uint32_t b = act ? in[p] : 0x100;
        uint32_t peers = __match_any_sync(0xffffffffu, b);
        if (act && (peers & hgpu_lanemask_lt()) == 0) atomicAdd(&s.cnt[b], __popc(peers));
    }
    __syncwarp();
    uint8_t *tbl = scratch + (nested ? ENC_NEST_TBL : 256 * 256 * 4);   // table text
    uint32_t tlen = 0;
    uint32_t shift = 12;
    uint32_t *tab = nullptr;
    uint32_t A = 0;
    const uint32_t seg = U / N;
    if (order == 0) {
        if (!normalise_row(s.cnt, 256, 4096)) return ENC_FAIL;
        if (lane == 0) {
            int n = put_alphabet(tbl, s.cnt);
            for (int j = 0; j < 256; j++) if (s.cnt[j]) n += vput(tbl + n, s.cnt[j]);
            tlen = (uint32_t)n;
            uint32_t x = 0;
            for (int j = 0; j < 256; j++) { s.cum[j] = x; x += s.cnt[j]; }
        }
        tlen = __shfl_sync(0xffffffffu, tlen, 0);
        __syncwarp();
    } else {
        // compact alphabet = every byte that occurs, plus 0 (the start context)
        if (lane == 0) {
            uint32_t a = 0;
            for (int j = 0; j < 256; j++) {
                if (s.cnt[j] || j == 0) { s.idxof[j] = (uint8_t)a; s.symof[a] = (uint8_t)j; a++; }
            }
            A = a;
        }
        A = __shfl_sync(0xffffffffu, A, 0);
        shift = A <= 128 ? 10 : 12;
        tab = A * A * 4 <= ENC_TAB_SMEM ? s.tab : reinterpret_cast<uint32_t *>(scratch);
        __syncwarp();
        for (uint32_t j = lane; j < A * A; j += 32) tab[j] = 0;
        __syncwarp();
        // order-1 histogram: context = previous byte of the same segment, 0 at a segment start
        for (uint32_t base = 0; base < U; base += 32) {
            uint32_t p = base + lane;
            bool act = p < U;
            uint32_t key = 0xffffffffu;
            if (act) {
                uint32_t z = seg ? p / seg : N - 1;
                if (z > N - 1) z = N - 1;
                uint32_t c = (p == z * seg) ? 0u : in[p - 1];
                key = (uint32_t)s.idxof[c] * A + s.idxof[in[p]];
            }
            uint32_t peers = __match_any_sync(0xffffffffu, key);
            if (act && (peers & hgpu_lanemask_lt()) == 0) atomicAdd(&tab[key], __popc(peers));
        }
        __syncwarp();
        __threadfence_block();
        // normalise every row; serialise the table (decode_freq1's format)
        if (lane == 0) {
            tbl[0] = (uint8_t)(shift << 4);
            uint32_t pres[256];
            for (int j = 0; j < 256; j++) pres[j] = (s.cnt[j] || j == 0) ? 1 : 0;
            tlen = 1 + put_alphabet(tbl + 1, pres);
        }
        tlen = __shfl_sync(0xffffffffu, tlen, 0);
        for (uint32_t r = 0; r < A; r++) {
            uint32_t *row = tab + r * A;
            // a row that totals well under 2^shift is stored normalised to a smaller power of two and shifted up on both
            // sides (rans_compute_shift :376-387, normalise_freq_shift): smaller varints in the table text
            uint32_t trow = 0, ns = 0;
            for (uint32_t k = lane; k < A; k += 32) { trow += row[k]; ns += row[k] != 0; }
            for (int d = 16; d > 0; d >>= 1) { trow += __shfl_xor_sync(0xffffffffu, trow, d); ns += __shfl_xor_sync(0xffffffffu, ns, d); }
            uint32_t max_val = 1u << shift, up = 0;
            if (trow) {
                uint32_t m2 = 1;
                while (m2 < trow) m2 <<= 1;                          // round2
                if (ns < 64 && m2 > 128) m2 >>= 1;
                if (m2 > 1024) m2 >>= 1;
                while (m2 < ns) m2 <<= 1;
                if (m2 < max_val) { max_val = m2; while ((max_val << up) < (1u << shift)) up++; }
            }
            if (!normalise_row(row, (int)A, max_val)) return ENC_FAIL;
            __syncwarp();
            if (lane == 0) {
                uint8_t *cp = tbl + tlen;
                int dz = 0;
                for (uint32_t k = 0; k < A; k++) {                    // encode_freq_d (:278-307)
                    if (row[k]) {
                        if (dz) { cp -= dz - 1; *cp++ = (uint8_t)(dz - 1); }
                        dz = 0;
                        cp += vput(cp, row[k]);
                    } else { dz++; *cp++ = 0; }
                }
                if (dz) { cp -= dz - 1; *cp++ = (uint8_t)(dz - 1); }
                tlen = (uint32_t)(cp - tbl);
                // row -> {f | start<<16}
                uint32_t x = 0;
                for (uint32_t k = 0; k < A; k++) { uint32_t f = row[k] << up; row[k] = f | (x << 16); x += f; }
            }
            tlen = __shfl_sync(0xffffffffu, tlen, 0);
            __syncwarp();
        }
        __threadfence_block();
        // a long table is itself order-0 coded when that is smaller (encode_freq1, rANS_static16_int.h:397-411)
        if constexpr (!nested) if (tlen > 1000 && tlen - 1 <= ENC_NEST_CAP - 4096) {     // (the nested instantiation has no such call: no recursion)
            __syncwarp();
            uint8_t *tmp = scratch + ENC_NEST_OUT;
            const uint32_t c = encode_core<true>(s, scratch, tbl + 1, tlen - 1, 0, 4, tmp, ENC_NEST_CAP);
            __syncwarp();
            if (c != ENC_FAIL && c + 6 < tlen) {
                uint32_t at = 0;
                if (lane == 0) { tbl[0] |= 1; at = 1 + vput(tbl + 1, tlen - 1); at += vput(tbl + at, c); }
                at = __shfl_sync(0xffffffffu, at, 0);
                for (uint32_t i = lane; i < c; i += 32) tbl[at + i] = tmp[i];
                tlen = at + c;
                __syncwarp();
                __threadfence_block();
            }
        }
    }
    const uint32_t body = hdr + tlen + 4 * N;                         // first byte after the states
    if (body + 2u > cap) return ENC_FAIL;
    // ---- encode backwards; words are laid downwards from the end of the slot ----
    uint32_t wp = cap & ~1u;                                          // byte offset of the lowest word written so far
    uint32_t x = RANS_L;
    const bool mine = lane < N;
    bool overflow = false;
#define ENC_EMIT(ACTIVE, F, START)                                                                 \
    {                                                                                              \
        bool need = (ACTIVE) && x >= ((F) << (31 - shift));                                        \
        uint32_t bal = __ballot_sync(0xffffffffu, need);                                           \
        if (bal) {                                                                                 \
            uint32_t cntw = __popc(bal);                                                           \
            if (wp < body + 2 * cntw) overflow = true;                                             \
            else {                                                                                 \
                wp -= 2 * cntw;                                                                    \
                if (need) {                                                                        \
                    uint32_t o = wp + 2 * __popc(bal & hgpu_lanemask_lt());                        \
                    out[o] = (uint8_t)x; out[o + 1] = (uint8_t)(x >> 8);                           \
                    x >>= 16;                                                                      \
                }                                                                                  \
            }                                                                                      \
        }                                                                                          \
        if (ACTIVE) x = enc_put(x, (F), (START), shift);                                           \
    }
    if (order == 0) {
        // symbol i belongs to state i % N; decode order is i ascending, so encode i descending.
        uint32_t rows = (U + N - 1) / N;
        for (uint32_t rr = rows; rr-- > 0;) {
            uint32_t i = rr * N + lane;
            bool act = mine && i < U;
            uint32_t b = act ? in[i] : 0;
            uint32_t f = act ? s.cnt[b] : 1, st = act ? s.cum[b] : 0;
            ENC_EMIT(act, f, st)
            if (overflow) break;
        }
    } else {
        const bool last = lane == N - 1;
        // the last state's tail first (it is decoded last)
        for (uint32_t p = U; p-- > seg * N;) {
            uint32_t c = (p == (N - 1) * seg) ? 0u : in[p - 1];
            uint32_t e = tab[(uint32_t)s.idxof[c] * A + s.idxof[in[p]]];
            ENC_EMIT(last, e & 0xffffu, e >> 16)
            if (overflow) break;
        }
        const uint8_t *ip = in + (size_t)(mine ? lane : 0) * seg;
        for (uint32_t q = seg; q-- > 0 && !overflow;) {
            uint32_t c = q ? ip[q - 1] : 0u;
            uint32_t e = tab[(uint32_t)s.idxof[c] * A + s.idxof[ip[q]]];
            ENC_EMIT(mine, e & 0xffffu, e >> 16)
        }
    }
#undef ENC_EMIT
    if (overflow) return ENC_FAIL;
    const uint32_t total = body + ((cap & ~1u) - wp);
    // table, states, then the words moved up behind them
    __syncwarp();
    for (uint32_t i = lane; i < tlen; i += 32) out[hdr + i] = tbl[i];
    if (mine) {
        uint8_t *q = out + hdr + tlen + 4 * lane;
        q[0] = (uint8_t)x; q[1] = (uint8_t)(x >> 8); q[2] = (uint8_t)(x >> 16); q[3] = (uint8_t)(x >> 24);
    }
    uint32_t nw = (cap & ~1u) - wp;
    // forward copy in 32-byte strides: destination is below the source, chunks never overtake
    for (uint32_t i0 = 0; i0 < nw; i0 += 32) {
        uint32_t i = i0 + lane;
        uint8_t v = i < nw ? out[wp + i] : 0;
        __syncwarp();
        if (i < nw) out[body + i] = v;
        __syncwarp();
    }
    return total;
}

// Forward copy by the warp; dst may overlap src from below (dst <= src): strides never overtake.
__device__ void warp_move_down(uint8_t *dst, const uint8_t *src, uint32_t n)
{
    const uint32_t lane = hgpu_lane();
    if (dst == src) return;
    for (uint32_t i0 = 0; i0 < n; i0 += 32) {
        const uint32_t i = i0 + lane;
        const uint8_t v = i < n ? src[i] : 0;
        __syncwarp();
        if (i < n) dst[i] = v;
        __syncwarp();
    }
}

// hts_pack (pack.c:56-150) by the warp.  meta gets [nsym][symbols...]; returns nsym (> 16: not packable, nothing
// else written) and the packed length in plen.
__device__ uint32_t warp_pack(EncSmem &s, const uint8_t *in, uint32_t n, uint8_t *meta, uint8_t *packed, uint32_t &plen)
{
    const uint32_t lane = hgpu_lane();
    __syncwarp();
    for (int j = lane; j < 256; j += 32) s.cnt[j] = 0;
    __syncwarp();
    for (uint32_t i = lane; i < n; i += 32) s.cnt[in[i]] = 1;            // same value from every writer
    __syncwarp();
    uint32_t nsym = 0;
#pragma unroll
    for (int k = 0; k < 8; k++) {
        const uint32_t j = k * 32 + lane, pr = s.cnt[j];
        const uint32_t bal = __ballot_sync(0xffffffffu, pr != 0);
        if (pr) { const uint32_t c = nsym + __popc(bal & hgpu_lanemask_lt()); s.idxof[j] = (uint8_t)c; if (c < 16) s.symof[c] = (uint8_t)j; }
        nsym += __popc(bal);
    }
    __syncwarp();
    if (nsym > 16) return nsym;
    if (lane == 0) meta[0] = (uint8_t)nsym;
    if (lane < nsym) meta[1 + lane] = s.symof[lane];
    const uint32_t per = nsym > 4 ? 2 : nsym > 2 ? 4 : nsym > 1 ? 8 : 0, bits = per ? 8 / per : 0;
    plen = per ? (n + per - 1) / per : 0;
    for (uint32_t j = lane; j < plen; j += 32) {
        uint32_t v = 0;
        for (uint32_t k = 0; k < per; k++) {
            const uint32_t i = j * per + k;
            if (i < n) v |= (uint32_t)s.idxof[in[i]] << (bits * k);
        }
        packed[j] = (uint8_t)v;
    }
    __syncwarp();
    return nsym;
}

// rle_find_syms (rle.c:48-98) + hts_rle_encode (:100-140) by the warp.  meta gets [nsyms][symbols...][run lengths...]
// (the layout rans_compress_to_4x16 :1462-1465 assembles), lit the literals.
__device__ void warp_rle(EncSmem &s, const uint8_t *in, uint32_t n, uint8_t *meta, uint8_t *lit, uint32_t &rmeta_len, uint32_t &nlit)
{
    const uint32_t lane = hgpu_lane();
    int *saved = reinterpret_cast<int *>(s.cum);
    __syncwarp();
    for (int j = lane; j < 256; j += 32) saved[j] = 0;
    __syncwarp();
    for (uint32_t base = 0; base < n; base += 32) {
        const uint32_t i = base + lane;
        if (i < n) { const uint8_t b = in[i]; atomicAdd(&saved[b], (i > 0 && in[i - 1] == b) ? 1 : -1); }
    }
    __syncwarp();
    uint32_t nsyms = 0;
#pragma unroll
    for (int k = 0; k < 8; k++) {
        const uint32_t j = k * 32 + lane;
        const bool in_set = saved[j] > 0;
        const uint32_t bal = __ballot_sync(0xffffffffu, in_set);
        s.idxof[j] = in_set ? 1 : 0;
        if (in_set) meta[1 + nsyms + __popc(bal & hgpu_lanemask_lt())] = (uint8_t)j;
        nsyms += __popc(bal);
    }
    if (lane == 0) meta[0] = (uint8_t)nsyms;                              // 256 wraps to 0 like the reference's store
    __syncwarp();
    uint64_t k64, j64;
    warp_rle_encode(in, n, s.idxof, lit, meta + 1 + nsyms, k64, j64);
    __syncwarp();
    nlit = (uint32_t)k64;
    rmeta_len = (uint32_t)j64 + nsyms + 1;
}

// rans_compress_to_4x16 without STRIPE (rANS_static4x16pr.c:1378-1565).  Returns bytes written, 0 on failure.
__device__ uint32_t encode_flat(EncSmem &s, uint8_t *scratch, const XBuf &xb, const uint8_t *in, uint32_t U, uint32_t want,
                                uint8_t *out, uint32_t cap)
{
    const uint32_t lane = hgpu_lane();
    if (cap < 32) return 0;
    if (U <= 1000) want &= ~F_X32;                                        // :1239-1242
    if (U > xb.X) want &= ~(F_PACK | F_RLE);                              // no transform buffers carved for this size
    uint32_t fmt = want & (F_ORDER | F_X32 | F_NOSZ | F_RLE | F_PACK);
    uint32_t cm = 1;
    if (!(want & F_NOSZ)) {
        if (lane == 0) cm += vput(out + 1, U);
        cm = __shfl_sync(0xffffffffu, cm, 0);
    }
    if (U == 0) {
        if (lane == 0) out[0] = (uint8_t)(fmt & (F_ORDER | F_X32 | F_NOSZ));
        return cm;
    }
    const uint8_t *cur = in;
    uint32_t n = U;
    if (fmt & F_PACK) {
        if (cm + 280 > cap) return 0;
        uint32_t plen = 0;
        const uint32_t nsym = warp_pack(s, cur, n, out + cm, xb.P, plen);
        if (nsym > 16) fmt &= ~F_PACK;
        else {
            cm += nsym + 1;
            cur = xb.P; n = plen;
            uint32_t sz = 0;
            if (lane == 0) sz = vput(out + cm, n);
            cm += __shfl_sync(0xffffffffu, sz, 0);
            if ((fmt & F_X32) && n < 32) fmt &= ~F_X32;
        }
    }
    if ((fmt & F_RLE) && n) {
        uint32_t rmeta = 0, nlit = 0;
        warp_rle(s, cur, n, xb.M, xb.R, rmeta, nlit);
        if ((double)nlit + (double)rmeta >= 0.99 * (double)n) fmt &= ~F_RLE;     // not worth it (:1467)
        else {
            uint32_t sz = 0;
            if (lane == 0) { sz = vput(out + cm, rmeta * 2); sz += vput(out + cm + sz, nlit); }
            sz = __shfl_sync(0xffffffffu, sz, 0);
            if ((uint64_t)cm + sz + 5 + 64 > cap) return 0;
            if ((fmt & F_X32) && (rmeta < 32 || nlit < 32)) fmt &= ~F_X32;
            __syncwarp();
            __threadfence_block();
            const uint32_t c = encode_core(s, scratch, xb.M, rmeta, 0, (fmt & F_X32) ? 32 : 4, out + cm + sz + 5, cap - (cm + sz + 5));
            __syncwarp();
            if (c != ENC_FAIL && c < rmeta) {
                uint32_t sz2 = 0;
                if (lane == 0) sz2 = vput(out + cm + sz, c);
                sz2 = __shfl_sync(0xffffffffu, sz2, 0);
                __syncwarp();
                warp_move_down(out + cm + sz + sz2, out + cm + sz + 5, c);
                cm += sz + sz2 + c;
            } else {
                // run lengths kept as they are: odd length field (:1501-1507)
                uint32_t sz2 = 0;
                if (lane == 0) { sz = vput(out + cm, rmeta * 2 + 1); sz2 = vput(out + cm + sz, nlit); }
                sz = __shfl_sync(0xffffffffu, sz, 0);
                sz2 = __shfl_sync(0xffffffffu, sz2, 0);
                if ((uint64_t)cm + sz + sz2 + rmeta > cap) return 0;
                for (uint32_t i = lane; i < rmeta; i += 32) out[cm + sz + sz2 + i] = xb.M[i];
                cm += sz + sz2 + rmeta;
            }
            cur = xb.R; n = nlit;
        }
    } else
        fmt &= ~F_RLE;
    uint32_t order = fmt & F_ORDER;
    if (order && n < 8) { fmt &= ~F_ORDER; order = 0; }                  // :1526-1529
    if (cm + 4 > cap) return 0;
    __syncwarp();
    __threadfence_block();
    uint32_t c = n ? encode_core(s, scratch, cur, n, order, (fmt & F_X32) ? 32 : 4, out + cm, cap - cm) : ENC_FAIL;
    __syncwarp();
    if (c == ENC_FAIL || c >= n) {
        // CAT fallback (:1539-1553): the (possibly transformed) bytes as they are
        if ((uint64_t)cm + n > cap) return 0;
        fmt = (fmt & ~3u) | F_CAT;
        for (uint32_t i = lane; i < n; i += 32) out[cm + i] = cur[i];
        c = n;
    }
    if (lane == 0) out[0] = (uint8_t)fmt;
    __syncwarp();
    return cm + c;
}

// The STRIPE branch (:1244-1376): N interleaved sub-streams, each coded by the smallest of the methods the caller's
// order admits (order 1, RLE, PACK, order 0).
__device__ uint32_t encode_stripe(EncSmem &s, uint8_t *scratch, const XBuf &xb, const uint8_t *in, uint32_t U, uint32_t want,
                                  uint8_t *out, uint32_t cap)
{
    const uint32_t lane = hgpu_lane();
    uint32_t N = (want >> 8) & 0xff;
    if (N == 0) N = 4;
    if (N > U) N = U;
    const uint32_t q = U / N, r = U % N;
    if ((uint64_t)7 + 5 * N + 64 > cap) return 0;
    // transpose: part j takes in[j], in[j + N], ...
    for (uint32_t i = lane; i < U; i += 32) {
        const uint32_t j = i % N, x = i / N;
        xb.S[j * q + min(j, r) + x] = in[i];
    }
    uint32_t *lens = reinterpret_cast<uint32_t *>(xb.S + ((U + 3u) & ~3u));
    uint32_t cm = 0;
    if (lane == 0) {
        out[0] = (uint8_t)(want & 0xff & ~F_NOSZ);
        cm = 1 + vput(out + 1, U);
        out[cm++] = (uint8_t)N;
    }
    cm = __shfl_sync(0xffffffffu, cm, 0);
    __syncwarp();
    __threadfence_block();
    const uint32_t start2 = 7 + 5 * N;
    uint32_t o2 = start2;
    const uint32_t methods[4] = {1, 64, 128, 0};
    XBuf sub = xb;
    sub.S = nullptr; sub.B = nullptr;
    for (uint32_t j = 0; j < N; j++) {
        const uint32_t plen = q + (r > j ? 1u : 0u);
        const uint8_t *part = xb.S + j * q + min(j, r);
        uint32_t best = ENC_FAIL;
        bool in_place = false;
        for (int t = 0; t < 4; t++) {
            const uint32_t m = methods[t];
            if ((want & m) != m) continue;
            if ((want & F_STRIPE_NO0) && !(m & 1)) continue;
            if (o2 >= cap) continue;
            const uint32_t c = encode_flat(s, scratch, sub, part, plen, m | F_NOSZ | (want & F_X32), out + o2, cap - o2);
            __syncwarp();
            if (c && c < best && c <= xb.X + XB_PAD_B) {
                best = c;
                in_place = true;
                for (uint32_t i = lane; i < c; i += 32) xb.B[i] = out[o2 + i];
                __syncwarp();
            } else
                in_place = false;
        }
        if (best == ENC_FAIL) return 0;
        if (!in_place) { for (uint32_t i = lane; i < best; i += 32) out[o2 + i] = xb.B[i]; __syncwarp(); }
        if (lane == 0) lens[j] = best;
        o2 += best;
    }
    __syncwarp();
    if (lane == 0) for (uint32_t j = 0; j < N; j++) cm += vput(out + cm, lens[j]);
    cm = __shfl_sync(0xffffffffu, cm, 0);
    __syncwarp();
    warp_move_down(out + cm, out + start2, o2 - start2);
    return cm + (o2 - start2);
}

__device__ uint32_t encode_stream(EncSmem &s, uint8_t *scratch, const XBuf &xb, const uint8_t *in, uint32_t U, uint32_t want,
                                  uint8_t *out, uint32_t cap)
{
    if (U <= 1000) want &= ~F_X32;
    if (U <= 20 || U > xb.X) want &= ~F_STRIPE;                          // :1237-1238
    if (want & F_STRIPE) return encode_stripe(s, scratch, xb, in, U, want, out, cap);
    if (want & F_CAT) {                                                   // :1378-1392
        if ((uint64_t)6 + U > cap) return 0;
        uint32_t cm = 0;
        if (hgpu_lane() == 0) { out[0] = (uint8_t)F_CAT; cm = 1 + vput(out + 1, U); }
        cm = __shfl_sync(0xffffffffu, cm, 0);
        for (uint32_t i = hgpu_lane(); i < U; i += 32) out[cm + i] = in[i];
        return cm + U;
    }
    return encode_flat(s, scratch, xb, in, U, want & ~F_NOSZ, out, cap);
}

__global__ void __launch_bounds__(32)
rans_nx16_encode_kernel(const uint8_t *__restrict__ in, const uint64_t *__restrict__ in_off,
                        const uint32_t *__restrict__ in_len, const uint32_t *__restrict__ order, uint32_t n,
                        uint8_t *out, const uint64_t *__restrict__ out_off, const uint32_t *__restrict__ out_cap,
                        uint32_t *out_len, int32_t *status, uint8_t *scratch, uint32_t *counter, uint32_t X)
{
    __shared__ EncSmem s;
    const size_t per_warp = ENC_SCRATCH + xbuf_bytes(X);
    uint8_t *my = scratch + (size_t)blockIdx.x * per_warp;
    XBuf xb;
    xb.X = X;
    xb.P = my + ENC_SCRATCH;
    xb.R = xb.P + X;
    xb.M = xb.R + X;
    xb.S = xb.M + X + XB_PAD_M;
    xb.B = xb.S + X + XB_PAD_S;
    for (;;) {
        uint32_t job = 0;
        if (hgpu_lane() == 0) job = atomicAdd(counter, 1u);
        job = __shfl_sync(0xffffffffu, job, 0);
        if (job >= n) break;
        uint32_t got = encode_stream(s, my, xb, in + in_off[job], in_len[job], order[job], out + out_off[job], out_cap[job]);
        __syncwarp();
        if (hgpu_lane() == 0) { out_len[job] = got; status[job] = got ? HGPU_OK : HGPU_RANS_ERR; }
    }
}

// longest input among the jobs that ask for a transform: sizes the per-warp transform buffers
__global__ void rans_nx16_enc_survey_kernel(const uint32_t *__restrict__ in_len, const uint32_t *__restrict__ order, uint32_t n, uint32_t *res)
{
    uint32_t m = 0;
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x)
        if (order[i] & (F_PACK | F_RLE | F_STRIPE)) m = max(m, in_len[i]);
    for (int d = 16; d > 0; d >>= 1) m = max(m, __shfl_xor_sync(0xffffffffu, m, d));
    if ((threadIdx.x & 31) == 0 && m) atomicMax(res, m);
}

} // namespace

extern "C" uint32_t hgpu_rans_nx16_compress_bound(uint32_t size, int order)
{
    // same shape as rans_compress_bound_4x16 (rANS_static4x16pr.c:1203): payload slack + table + states
    uint64_t b = (uint64_t)(1.05 * size) + 257 * 3 + 4 + 64;
    if (order & 0xff) b += 257 * 257 * 3 + 257 * 3 + 4;               // the reference takes this branch for any flag (:98-100)
    b += (order & 4) ? 32 * 4 : 4 * 4;
    if (order & 0x80) b += 1 + 280;
    if (order & 0x40) b += 1 + 257 * 3 + 4 + 64;
    if (order & 0x08) { uint32_t N = (order >> 8) & 0xff; if (!N) N = 4; b += 7 + 5 * N + (uint64_t)N * 1100; }
    b += 20;
    return b > 0xffffffffull ? 0xffffffffu : (uint32_t)b;
}

extern "C" int hgpu_rans_nx16_encode_batch_dev(hgpu_ctx *ctx, const uint8_t *d_in, const uint64_t *d_in_off,
        const uint32_t *d_in_len, const uint32_t *d_order, uint32_t n, uint8_t *d_out, const uint64_t *d_out_off,
        const uint32_t *d_out_cap, uint32_t *d_out_len, int32_t *d_status, void *stream)
{
    if (!ctx) { hgpu_set_error("null context"); return HGPU_ERR_ARG; }
    if (n == 0) return HGPU_OK;
    cudaStream_t st = stream ? (cudaStream_t)stream : ctx->stream;
    int per_sm = 0;
    if (hgpu_check(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, rans_nx16_encode_kernel, 32, 0), "enc occupancy"))
        return HGPU_ERR_CUDA;
    if (per_sm < 1) per_sm = 1;
    uint32_t grid = (uint32_t)ctx->sm_count * (uint32_t)per_sm;
    if (grid > n) grid = n;
    // PACK / RLE / STRIPE need per-warp buffers as long as the longest such input: the job list lives on the device,
    // so one word comes back (the only synchronisation of this call)
    uint32_t *res = hgpu_take_counter(ctx, st);
    if (!res) return HGPU_ERR_CUDA;
    rans_nx16_enc_survey_kernel<<<(n + 255) / 256 < 64u ? (n + 255) / 256 : 64u, 256, 0, st>>>(d_in_len, d_order, n, res);
    hgpu_count_launch();
    uint32_t maxlen = 0;
    if (hgpu_check(cudaMemcpyAsync(&maxlen, res, 4, cudaMemcpyDeviceToHost, st), "enc survey copy")) return HGPU_ERR_CUDA;
    if (hgpu_check(cudaStreamSynchronize(st), "enc survey sync")) return HGPU_ERR_CUDA;
    const uint32_t X = maxlen ? ((maxlen + 255u) & ~255u) + 256u : 0u;
    const size_t per_warp = ENC_SCRATCH + xbuf_bytes(X);
    const size_t budget = (size_t)4 << 30;
    if ((size_t)grid * per_warp > budget) grid = (uint32_t)(budget / per_warp);
    if (grid < 1) grid = 1;
    int rc = hgpu_ensure_scratch(ctx, (size_t)grid * per_warp);
    if (rc) return rc;
    uint32_t *counter = hgpu_take_counter(ctx, st);
    if (!counter) return HGPU_ERR_CUDA;
    rans_nx16_encode_kernel<<<grid, 32, 0, st>>>(d_in, d_in_off, d_in_len, d_order, n, d_out, d_out_off, d_out_cap,
                                                d_out_len, d_status, ctx->d_scratch, counter, X);
    hgpu_count_launch();
    return hgpu_check(cudaGetLastError(), "rans encode launch");
}
