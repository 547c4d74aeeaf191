// CTA-per-block BGZF inflate (included into the anonymous namespace of bgzf_inflate.cu).
//
// The member's whole output (<= 64 KiB) lives in SHARED memory, two CTAs of 256 threads per SM.
// inflate_block -> bgzf_uncompress + CRC check, bgzf.c:762-824.
//
// Why a CTA and a shared window: a sorted-BAM block is ~5000 tokens, ~2300 of them matches whose
// dependency DAG is ~120 levels deep (record n copies from record n-1; forwarding sources through
// earlier matches does not flatten it — measured: 120 -> 104 levels).  With the output in global
// memory every level costs an L2 round trip; in shared memory it costs ~200 cycles.
//
// One block at a time per CTA, software-pipelined over blocks:
//
//   P2  all 256 threads  the body's bit range cut into 256 sub-ranges, speculative Huffman decode
//                        with chained restarts until every sub-range starts where its predecessor
//                        stopped, block-wide prefix sums, then literals straight into the window and
//                        each match parked as a 3-byte record AT its own destination (+ a 16-bit
//                        destination list).  The bit stream was staged into shared memory by TMA.
//   --- barrier ---
//   warp 7               (a) takes the NEXT job, issues its TMA staging copy (the staging buffer is
//                        free now), (b) P1 of the next block: deflate block header, code lengths,
//                        decode tables into the OTHER table buffer.
//   warps 0-6            P3a dependency ranges of all matches (two binary searches each, in parallel)
//                        P3b warp 0: LZ77 resolution, 32 matches per batch, one per lane, out of
//                            order inside the batch; every lane copies its own match with aligned
//                            32-bit shared-memory stores and a funnel-shifted source.
//                        P4  bulk store of the window (TMA, shared -> global) issued FIRST, CRC-32 of
//                            the window computed while it flies: lane-strided Horner form (the data
//                            reads are conflict-free), x^1024 step tables, per-lane / per-warp powers
//                            from precomputed tables.
//   --- barrier ---
//
// Members that are not one big final Huffman block (stored blocks, tiny blocks, several deflate
// blocks) take the same phases without the overlap: warp 0 parses the following headers in place.

constexpr int CTA_T = 256;
constexpr uint32_t P3_T = 224;                      // warps 0..6
constexpr uint32_t WIN_BYTES = 65536 + 32;          // 16 bytes of alignment slack in front, word reads may run past the end
constexpr uint32_t STAGE_BYTES = 18 * 1024;         // compressed blocks up to this size are staged in shared memory (TMA)
constexpr uint32_t SEG_M = 3072;                    // matches resolved per LZ77 segment

struct HdrInfo {             // what P1 leaves for the main phase
    int32_t rc;
    uint32_t type, final_, body;     // body: first body bit (Huffman) / first data byte (stored), member-relative
    uint32_t len;                    // stored: byte count
};

struct CtaCtl {
    HdrInfo h[2];
    uint32_t job, next_job, o, end_pos, E, bad, tot_m, phase, next_staged, emin[2];
    int32_t rc;
    uint32_t crc[8];
    long long t0;            // HGPU_PROFILE: start of the current phase
};

struct CtaSmem {
    uint8_t win[WIN_BYTES];
    uint8_t stage[STAGE_BYTES + 32];
    InflateSmem s[2];                // decode tables (+ their scratch), double-buffered over blocks
    uint16_t D[SEG_M];               // destinations of the segment's matches
    CtaCtl c;
    unsigned long long mbar;         // mbarrier of the staging copy
};
static_assert(sizeof(CtaSmem) <= 115200, "two CTAs per SM: 2 x (size + 1 KiB) must fit 227 KiB");
static_assert(sizeof(InflateSmem) >= 8192 && sizeof(InflateSmem) >= 2 * SEG_M + SEG_M / 8 + 16, "the dependency list + done words (P3), then the CRC tables (P4), overlay a dead table buffer");

#ifdef HGPU_PROFILE
#define CTA_MARK(cs, i) do { if (threadIdx.x == 0) { long long n_ = clock64(); atomicAdd(&g_prof[i], (unsigned long long)(n_ - (cs).c.t0)); (cs).c.t0 = n_; } } while (0)
#else
#define CTA_MARK(cs, i) do { } while (0)
#endif

// ---- TMA (1-D bulk copy) + named-barrier helpers ---------------------------------------------
__device__ __forceinline__ void mbar_init(unsigned long long *mb, uint32_t count)
{
    uint32_t a = (uint32_t)__cvta_generic_to_shared(mb);
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" :: "r"(a), "r"(count) : "memory");
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void tma_load_1d(void *smem_dst, const void *gsrc, uint32_t bytes, unsigned long long *mb)
{
    uint32_t d = (uint32_t)__cvta_generic_to_shared(smem_dst), m = (uint32_t)__cvta_generic_to_shared(mb);
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" :: "r"(m), "r"(bytes) : "memory");
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 :: "r"(d), "l"(gsrc), "r"(bytes), "r"(m) : "memory");
}
__device__ __forceinline__ void mbar_wait(unsigned long long *mb, uint32_t parity)
{
    uint32_t m = (uint32_t)__cvta_generic_to_shared(mb), ok = 0;
    while (!ok) {
        asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                     : "=r"(ok) : "r"(m), "r"(parity) : "memory");
    }
}
__device__ __forceinline__ void bar_p3() { asm volatile("bar.sync 1, 224;" ::: "memory"); }   // warps 0..6

// ---------------------------------------------------------------------------------------------
// P1: one deflate block header, by one warp.  Huffman tables go to s.lit / s.dst.  Nothing but `s`
// and the bit stream is touched (the window belongs to another block while this runs).
// ---------------------------------------------------------------------------------------------
__device__ void parse_block_header(InflateSmem &s, Bits &b, uint32_t slen, uint32_t mis_bits, HdrInfo &hi)
{
    const uint32_t lane = hgpu_lane();
    int rc = HGPU_OK;
    uint32_t final_ = 0, type = 3, body = 0, len = 0;
    do {
        bits_fill(b);
        final_ = bits_get(b, 1);
        type = bits_get(b, 2);
        if (type == 0) {
            bits_drop(b, b.cnt & 7);
            bits_fill(b);
            len = bits_get(b, 16);
            bits_fill(b);
            uint32_t nlen = bits_get(b, 16);
            if (bits_overrun(b) || (len ^ 0xffffu) != nlen) { rc = HGPU_BGZF_ERR_ZLIB; break; }
            body = bits_pos(b) >> 3;
            if ((uint64_t)body + len > slen) { rc = HGPU_BGZF_ERR_ZLIB; break; }
        } else if (type == 1) {
            __syncwarp();
            for (int i = lane; i < 288; i += 32) s.lens[i] = i < 144 ? 8 : i < 256 ? 9 : i < 280 ? 7 : 8;
            __syncwarp();
            if (build_table<LIT_ROOT, LIT_TABLE>(s, s.lit, 288, false, lit_entry)) { rc = HGPU_BGZF_ERR_ZLIB; break; }
            __syncwarp();
            for (int i = lane; i < 32; i += 32) s.lens[i] = 5;
            __syncwarp();
            if (build_table<DST_ROOT, DST_TABLE>(s, s.dst, 32, false, dst_entry)) { rc = HGPU_BGZF_ERR_ZLIB; break; }
            body = mis_bits + bits_pos(b);
        } else if (type == 2) {
            bits_fill(b);
            uint32_t hlit = bits_get(b, 5) + 257, hdist = bits_get(b, 5) + 1, hclen = bits_get(b, 4) + 4;
            if (hlit > 286 || hdist > 30) { rc = HGPU_BGZF_ERR_ZLIB; break; }
            __syncwarp();
            if (lane < 19) s.lens[lane] = 0;
            __syncwarp();
            for (uint32_t i = 0; i < hclen; i++) {
                bits_fill(b);
                uint32_t v = bits_get(b, 3);
                if (lane == 0) s.lens[c_cl_order[i]] = (uint8_t)v;
            }
            if (bits_overrun(b)) { rc = HGPU_BGZF_ERR_ZLIB; break; }
            __syncwarp();
            if (build_table<7, CL_TABLE>(s, s.cl, 19, false, cl_entry)) { rc = HGPU_BGZF_ERR_ZLIB; break; }
            uint32_t nsym = hlit + hdist, i = 0, prev = 0;
            bool badc = false;
            while (i < nsym) {
                bits_fill(b);
                uint32_t e = s.cl[bits_peek(b, 7)];
                if (((e >> 4) & 15) != K_LIT) { badc = true; break; }
                bits_drop(b, e & 15);
                uint32_t sym = e >> 16;
                if (sym < 16) {
                    if (lane == 0) s.code[i] = (uint16_t)sym;
                    prev = sym; i++;
                } else {
                    uint32_t rep, val = 0;
                    if (sym == 16) { if (i == 0) { badc = true; break; } val = prev; rep = 3 + bits_get(b, 2); }
                    else if (sym == 17) rep = 3 + bits_get(b, 3);
                    else rep = 11 + bits_get(b, 7);
                    if (i + rep > nsym) { badc = true; break; }
                    for (uint32_t k = lane; k < rep; k += 32) s.code[i + k] = (uint16_t)val;
                    i += rep;
                    prev = val;
                }
                if (bits_overrun(b)) { badc = true; break; }
            }
            if (badc) { rc = HGPU_BGZF_ERR_ZLIB; break; }
            __syncwarp();
            if (s.code[256] == 0) { rc = HGPU_BGZF_ERR_ZLIB; break; }          // no end-of-block code
            uint32_t dl = lane < hdist ? s.code[hlit + lane] : 0;
            uint32_t ll[9];
#pragma unroll
            for (int k = 0; k < 9; k++) { uint32_t j = lane + 32 * k; ll[k] = j < hlit ? s.code[j] : 0; }
            __syncwarp();
#pragma unroll
            for (int k = 0; k < 9; k++) { uint32_t j = lane + 32 * k; if (j < 288) s.lens[j] = (uint8_t)ll[k]; }
            __syncwarp();
            if (build_table<LIT_ROOT, LIT_TABLE>(s, s.lit, (int)hlit, true, lit_entry)) { rc = HGPU_BGZF_ERR_ZLIB; break; }
            __syncwarp();
            s.lens[lane] = (uint8_t)dl;
            __syncwarp();
            if (build_table<DST_ROOT, DST_TABLE>(s, s.dst, (int)hdist, true, dst_entry)) { rc = HGPU_BGZF_ERR_ZLIB; break; }
            __syncwarp();
            if (bits_overrun(b)) { rc = HGPU_BGZF_ERR_ZLIB; break; }
            body = mis_bits + bits_pos(b);
        } else { rc = HGPU_BGZF_ERR_ZLIB; break; }
    } while (0);
    __syncwarp();
    if (lane == 0) { hi.rc = rc; hi.type = type; hi.final_ = final_; hi.body = body; hi.len = len; }
    __syncwarp();
}

// ---------------------------------------------------------------------------------------------
// P2: all threads.  Returns a CTA-uniform status.
//
// The symbol loop is written without data-dependent branches: one iteration decodes ONE Huffman
// symbol — a literal/length symbol or, right after a length, a distance symbol — for every lane of
// the warp in lock step (a literal takes one iteration, a match two); lanes that are done idle.
// The 32 bits at the lane's bit position are read straight from the (staged) stream; cuts between
// threads sit on word boundaries an ODD number of words apart, so the 32 lanes' stream reads fall
// into different shared-memory banks.  Long codes (second-level table) take a warp-uniform branch.
//
// Speculation: thread t first walks from its cut and RECORDS every token start with the byte / match
// counts in front of it (one word per token, in the still unused window).  When its true start a'
// arrives from its predecessor it walks from a' only until it lands on a recorded token start —
// on sorted BAM a wrong start re-synchronises after 6 tokens in the median, 28 at the 95th
// percentile — and takes the rest of the recorded walk (exit, counts) as it stands; a thread that
// never lands walks its range again.  The last pass writes literals into the window, parks each
// match as a 3-byte record AT its own destination and lists the destinations (16 bits each).
// ---------------------------------------------------------------------------------------------
template <bool SMEM>
__device__ int decode_body_impl(CtaSmem &cs, InflateSmem &s, const uint32_t *wbase, const uint32_t *wend, uint32_t body,
                                uint32_t total, uint32_t wa, uint32_t cap, uint16_t *dglobal)
{
    const uint32_t t = threadIdx.x, lane = t & 31, warp = t >> 5;
    const uint32_t sbase = SMEM ? (uint32_t)__cvta_generic_to_shared(wbase) : 0u;
    // cuts on word boundaries, an odd number of words apart
    const uint32_t w0 = body >> 5, nwords = ((total + 31u) >> 5) - w0;
    const uint32_t Sw = ((nwords + CTA_T - 1) / CTA_T) | 1u;
    const uint32_t cut = t == 0 ? body : min(total, (w0 + t * Sw) << 5);
    uint32_t start = cut;
    const uint32_t end = t == CTA_T - 1 ? total : min(total, (w0 + (t + 1) * Sw) << 5);
    // token records live in the window while it is still empty (the first deflate block of a member: the usual case)
    const bool can_rec = cs.c.o == 0 && Sw * 32u + 64u < 4096u;
    const uint32_t reca = (uint32_t)__cvta_generic_to_shared(cs.win) + 4u * t;
    uint32_t exitp = 0, n = 0, m = 0, st = ST_RUN, rcnt = 0, n0, m0;
    bool dummy = false;
    {
        // pre-roll: start PREROLL bits in front of the cut (never in front of the body), count from the cut on
        const uint32_t pre = t == 0 ? body : max(body, cut - min(cut, PREROLL));
        uint32_t p0 = cut;
        if (can_rec) huff_walk<1, SMEM, false>(s, sbase, wbase, wend, cut, pre, end, cut < end, reca, exitp, n, m, st, rcnt, 0, 0, 0, nullptr, dummy, cut, &p0);
        else         huff_walk<0, SMEM, false>(s, sbase, wbase, wend, cut, pre, end, cut < end, reca, exitp, n, m, st, rcnt, 0, 0, 0, nullptr, dummy, cut, &p0);
        // a pre-roll that never reached the cut leaves no usable state: its start can equal nobody's exit
        if (cut < end) start = p0; else exitp = start;
    }
    n0 = n; m0 = m;
    // Rounds: a thread whose predecessor's exit moved takes it as its new start.  Only threads up to the
    // first one that currently ends in an end-of-block code matter (what lies behind it is not part of
    // this deflate block: the next header, the BGZF footer, cuts past the input), so the others wait —
    // their turn comes if that end-of-block code turns out to be a false one.
    if (t < 2) cs.c.emin[t] = 0xffffffffu;
    __syncthreads();
    for (int round = 0; round < CTA_T + 2; round++) {
        s.x_exit[t] = exitp;
        if (st == ST_EOB) atomicMin(&cs.c.emin[round & 1], t);
        if (t == 0) cs.c.emin[(round + 1) & 1] = 0xffffffffu;
        __syncthreads();
        const uint32_t ns = t == 0 ? start : s.x_exit[t - 1];
        const uint32_t Em = cs.c.emin[round & 1];
        const bool need = ns != start && t <= Em;
        if (need) start = ns;
#ifdef HGPU_PROFILE
        if (t == 0) atomicAdd(&g_prof[8], 1ull);
#endif
        if (!__syncthreads_or(need)) break;
        if (!__any_sync(0xffffffffu, need)) continue;            // nothing moved in this warp
        const bool thru = need && start >= end;                  // the predecessor ran through this whole range
        if (thru) { exitp = start; n = 0; m = 0; st = ST_RUN; rcnt = 0; n0 = 0; m0 = 0; }
        bool landed = false;
        huff_fixup<SMEM>(s, sbase, wbase, wend, cut, start, end, need && !thru, reca, rcnt, n0, m0, n, m, landed);
        const bool again = need && !thru && !landed;
#ifdef HGPU_PROFILE
        if (again) atomicAdd(&g_prof[10], 1ull);
#endif
        if (__any_sync(0xffffffffu, again)) {
            uint32_t e2, n2, m2, s2, r2 = 0;
            const bool rec2 = can_rec;                           // re-record from the new start
            if (rec2) huff_walk<1, SMEM, false>(s, sbase, wbase, wend, cut, start, end, again, reca, e2, n2, m2, s2, r2, 0, 0, 0, nullptr, dummy, start);
            else      huff_walk<0, SMEM, false>(s, sbase, wbase, wend, cut, start, end, again, reca, e2, n2, m2, s2, r2, 0, 0, 0, nullptr, dummy, start);
            if (again) { exitp = e2; n = n2; m = m2; st = s2; rcnt = r2; n0 = n2; m0 = m2; }
        }
    }
    __syncthreads();                                             // the token records are dead: the window is the output again
#ifdef HGPU_PROFILE
    if ((int)cs.c.job == g_dbg_job) { g_dbg[6*t] = start; g_dbg[6*t+1] = exitp; g_dbg[6*t+2] = n; g_dbg[6*t+3] = m; g_dbg[6*t+4] = st; g_dbg[6*t+5] = cut; }
#endif
    CTA_MARK(cs, 1);
    // first end-of-block code, invalid codes at or before it
    if (t == 0) { cs.c.E = 0xffffffffu; cs.c.bad = 0; }
    __syncthreads();
    if (st == ST_EOB) atomicMin(&cs.c.E, t);
    __syncthreads();
    const uint32_t E = cs.c.E;
    if (E == 0xffffffffu) return HGPU_BGZF_ERR_ZLIB;             // input ends without an end-of-block code
    if (st == ST_BAD && t <= E) cs.c.bad = 1;
    if (t == E) cs.c.end_pos = exitp;
    if (t > E) { n = 0; m = 0; }
    // block-wide exclusive prefix sums of bytes and matches
    uint32_t on = n, mn = m;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        uint32_t a = __shfl_up_sync(0xffffffffu, on, d), c = __shfl_up_sync(0xffffffffu, mn, d);
        if (lane >= (uint32_t)d) { on += a; mn += c; }
    }
    __syncthreads();
    if (lane == 31) { s.x_sum[0][warp] = on; s.x_sum[1][warp] = mn; }
    __syncthreads();
    uint32_t tot_out = 0, tot_m = 0, pre_o = 0, pre_m = 0;
#pragma unroll
    for (uint32_t w = 0; w < CTA_T / 32; w++) {
        if (w < warp) { pre_o += s.x_sum[0][w]; pre_m += s.x_sum[1][w]; }
        tot_out += s.x_sum[0][w]; tot_m += s.x_sum[1][w];
    }
    on += pre_o; mn += pre_m;
    if (cs.c.bad) return HGPU_BGZF_ERR_ZLIB;
    if (cs.c.end_pos > total) return HGPU_BGZF_ERR_ZLIB;         // the block ran past the input
    const uint32_t o = cs.c.o;
    if ((uint64_t)o + tot_out > cap) return HGPU_BGZF_ERR_SPACE;
    if (tot_m > MREC_CAP) return HGPU_BGZF_ERR_ZLIB;
    bool bad_dist = false;
    {
        uint32_t e2, n2, m2, st2, r2;
        if (tot_m <= SEG_M) huff_walk<2, SMEM, false>(s, sbase, wbase, wend, cut, start, end, t <= E, 0, e2, n2, m2, st2, r2, wa, o + on - n, mn - m, cs.D, bad_dist);
        else                huff_walk<2, SMEM, true>(s, sbase, wbase, wend, cut, start, end, t <= E, 0, e2, n2, m2, st2, r2, wa, o + on - n, mn - m, dglobal, bad_dist);
    }
    if (__syncthreads_or(bad_dist)) return HGPU_BGZF_ERR_ZLIB;   // distance too far back
    if (t == 0) { cs.c.o = o + tot_out; cs.c.tot_m = tot_m; }
    __threadfence_block();
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");     // the window leaves through the async proxy (bulk store)
    __syncthreads();
    CTA_MARK(cs, 2);
    return HGPU_OK;
}

__device__ int decode_body_cta(CtaSmem &cs, InflateSmem &s, bool staged, const uint32_t *wbase, const uint32_t *wend, uint32_t body,
                               uint32_t total, uint32_t wa, uint32_t cap, uint16_t *dglobal)
{
    return staged ? decode_body_impl<true>(cs, s, wbase, wend, body, total, wa, cap, dglobal)
                  : decode_body_impl<false>(cs, s, wbase, wend, body, total, wa, cap, dglobal);
}

// ---------------------------------------------------------------------------------------------
// P3: LZ77 resolution of the matches parked by P2.  Called by warps 0..6 (224 threads) together.
// wa = shared address of output byte 0.  `deps` overlays a table buffer that is dead by now.
// ---------------------------------------------------------------------------------------------
// One match, one lane: aligned 32-bit stores, funnel-shifted source.  For matches that do not
// overlap their own source (dist >= len): every load of a chunk is issued before its stores, so a
// chunk of up to 32 bytes costs one shared-memory round trip, not one per word.
__device__ __forceinline__ void lz_copy_lane(uint32_t d, uint32_t s, uint32_t n, uint32_t act)
{
    // head (up to the first aligned destination word) and tail bytes: loads up front.
    // act = 0: the lane moves nothing (every access is predicated off; no branches below but the chunk loop)
    if (!act) n = 0;
    uint32_t h = (0u - d) & 3u;
    if (h > n) h = n;
    const uint32_t nw = (n - h) >> 2, tl = (n - h) & 3u;
    const uint32_t ts = s + h + 4u * nw, td = d + h + 4u * nw;
    const uint32_t hb0 = sld8_if(s, h > 0), hb1 = sld8_if(s + 1, h > 1), hb2 = sld8_if(s + 2, h > 2);
    const uint32_t tb0 = sld8_if(ts, tl > 0), tb1 = sld8_if(ts + 1, tl > 1), tb2 = sld8_if(ts + 2, tl > 2);
    uint32_t dw = d + h;
    const uint32_t sw = s + h;
    const uint32_t sh = (sw & 3u) * 8u;
    uint32_t sa = sw & ~3u;
    uint32_t rem = nw;
    uint32_t W0 = sld32_if(sa, rem > 0);
    while (rem) {
        // 8 destination words per chunk; loads past the last needed word stay inside the window's slack
        const uint32_t W1 = sld32(sa + 4), W2 = sld32_if(sa + 8, rem > 1), W3 = sld32_if(sa + 12, rem > 2), W4 = sld32_if(sa + 16, rem > 3);
        const uint32_t W5 = sld32_if(sa + 20, rem > 4), W6 = sld32_if(sa + 24, rem > 5), W7 = sld32_if(sa + 28, rem > 6), W8 = sld32_if(sa + 32, rem > 7);
        sst32(dw, __funnelshift_r(W0, W1, sh));
        sst32_if(dw + 4, __funnelshift_r(W1, W2, sh), rem > 1);
        sst32_if(dw + 8, __funnelshift_r(W2, W3, sh), rem > 2);
        sst32_if(dw + 12, __funnelshift_r(W3, W4, sh), rem > 3);
        sst32_if(dw + 16, __funnelshift_r(W4, W5, sh), rem > 4);
        sst32_if(dw + 20, __funnelshift_r(W5, W6, sh), rem > 5);
        sst32_if(dw + 24, __funnelshift_r(W6, W7, sh), rem > 6);
        sst32_if(dw + 28, __funnelshift_r(W7, W8, sh), rem > 7);
        W0 = W8; sa += 32; dw += 32;
        rem = rem > 8 ? rem - 8 : 0;
    }
    sst8_if(d, hb0, h > 0); sst8_if(d + 1, hb1, h > 1); sst8_if(d + 2, hb2, h > 2);
    sst8_if(td, tb0, tl > 0); sst8_if(td + 1, tb1, tl > 1); sst8_if(td + 2, tb2, tl > 2);
}

__device__ void lz_resolve_cta(CtaSmem &cs, uint16_t *deps, uint32_t wa, uint32_t tot_m, const uint16_t *dglobal)
{
    const uint32_t t = threadIdx.x, lane = t & 31, warp = t >> 5;
    for (uint32_t seg0 = 0; seg0 < tot_m; seg0 += SEG_M) {
        const uint32_t n = min(SEG_M, tot_m - seg0);
        if (tot_m > SEG_M) {                                     // destinations live in the global slot
            bar_p3();
            for (uint32_t i = t; i < n; i += P3_T) cs.D[i] = dglobal[seg0 + i];
        }
        bar_p3();
        for (uint32_t k = t; k < (SEG_M + 31u) / 32u; k += P3_T) reinterpret_cast<uint32_t *>(deps + SEG_M)[k] = 0u;
        // ---- P3a: dependency ranges, every match in parallel ----
        for (uint32_t i = t; i < n; i += P3_T) {
            const uint32_t dst = cs.D[i];
            const uint32_t len = sld8(wa + dst) + 3u, dist = (sld8(wa + dst + 1) | sld8(wa + dst + 2) << 8) + 1u;
            const uint32_t s0 = dst - dist, s1 = dist < len ? dst : s0 + len;
            // ub = #{D <= s0}, lb = #{D < s1}, over D[0..i): fixed 12 steps, both searches interleaved
            uint32_t lo0 = 0, lo1 = 0;
#pragma unroll
            for (uint32_t step = 2048; step; step >>= 1) {
                uint32_t m0 = lo0 + step, m1 = lo1 + step;
                uint32_t v0 = m0 <= i ? cs.D[m0 - 1] : 0xffffffffu, v1 = m1 <= i ? cs.D[m1 - 1] : 0xffffffffu;
                if (v0 <= s0) lo0 = m0;
                if (v1 < s1) lo1 = m1;
            }
            uint32_t first = lo0 ? lo0 - 1 : 0u;
            const uint32_t end = lo1;
            if (first < end) {                                   // does the match that starts at or before s0 reach s0 at all?
                const uint32_t fd = cs.D[first];
                if (fd + sld8(wa + fd) + 3u <= s0) first++;
            }
            const uint32_t cnt = end > first ? end - first : 0u;
            deps[i] = (uint16_t)(first | (cnt < 15u ? cnt : 15u) << 12);       // 15: everything from `first` up to the match itself
        }
        bar_p3();
        CTA_MARK(cs, 9);
        // ---- P3b: the seven warps take the batches of 32 matches round-robin.  Inside a batch a lane runs
        // when the earlier lanes it reads from are done (a register mask); matches of EARLIER batches are
        // checked in the shared done words (only the six batches in front can still be in flight: a warp
        // finishes batch b before it opens b + 7).  So up to 224 matches are in the window at once and a
        // dependency level costs one round of one warp, whichever warp owns the match. ----
        volatile uint32_t *donew = reinterpret_cast<volatile uint32_t *>(deps + SEG_M);
        for (uint32_t B = warp * 32u; B < n; B += P3_T) {
            const uint32_t i = B + lane, bi = B >> 5;
            const bool have = i < n;
            uint32_t dst = 0, len = 0, dist = 1, dep = 0, xlo = 0, xhi = 0;
            if (have) {
                dst = cs.D[i];
                len = sld8(wa + dst) + 3u;
                dist = (sld8(wa + dst + 1) | sld8(wa + dst + 2) << 8) + 1u;
                const uint32_t dp = deps[i];
                const uint32_t first = dp & 0xfffu, cnt = dp >> 12;
                const uint32_t end = cnt == 15u ? i : first + cnt;
                const uint32_t lo = first > B ? first - B : 0u, hi = end > B ? end - B : 0u;      // hi <= lane
                if (hi > lo) dep = low_mask(hi) & ~low_mask(lo);
                if (first < B && first < end) { xlo = first; xhi = end < B ? end : B; }           // the part in earlier batches
            }
            const bool slow = dist < len;                    // the match overlaps its own source: cooperative path
            bool xpend = xlo < xhi;
            const uint32_t k0 = xlo >> 5, k1 = xpend ? (xhi - 1u) >> 5 : k0;
            const uint32_t mk0 = (0xffffffffu << (xlo & 31u)) & (k1 == k0 ? 0xffffffffu >> (31u - ((xhi - 1u) & 31u)) : 0xffffffffu);
            const uint32_t mk1 = 0xffffffffu >> (31u - ((xhi - 1u) & 31u));
            uint32_t done = have ? 0u : 1u;
            done = __ballot_sync(0xffffffffu, done);
            while (done != 0xffffffffu) {
                if (xpend) {                                 // earlier batches: all of [xlo, xhi) done?
                    bool ok = (donew[k0] & mk0) == mk0;
                    if (k1 != k0) {
                        ok = ok && (donew[k1] & mk1) == mk1;
                        for (uint32_t k = k0 + 1; k < k1 && ok; k++) ok = donew[k] == 0xffffffffu;
                    }
                    if (ok) { xpend = false; __threadfence_block(); }    // acquire: the bytes behind those bits
                }
                const bool ready = !((done >> lane) & 1u) && (dep & ~done) == 0u && !xpend;
                const uint32_t R = __ballot_sync(0xffffffffu, ready);
                if (R == 0u) { __nanosleep(64); continue; }
                const uint32_t Rs = __ballot_sync(0xffffffffu, ready && slow);
                lz_copy_lane(wa + dst, wa + dst - dist, len, ready && !slow);
                __syncwarp();
                for (uint32_t mm = Rs; mm; mm &= mm - 1) {
                    // overlapping match: the `di` bytes before the destination, repeated; the warp writes it together
                    const int k = __ffs(mm) - 1;
                    const uint32_t d0 = __shfl_sync(0xffffffffu, dst, k), ln = __shfl_sync(0xffffffffu, len, k);
                    const uint32_t di = __shfl_sync(0xffffffffu, dist, k);
                    const uint32_t stepm = 32u % di;
                    uint32_t r = lane % di;
                    for (uint32_t i2 = lane; i2 < ln; i2 += 32) {
                        sst8(wa + d0 + i2, sld8(wa + d0 - di + r));          // the source bytes lie before d0: never overwritten here
                        r += stepm;
                        if (r >= di) r -= di;
                    }
                }
                __syncwarp();
                done |= R;
                if (lane == 0) { __threadfence_block(); donew[bi] = done; }  // release
            }
        }
    }
    bar_p3();
}

// ---------------------------------------------------------------------------------------------
// P4: CRC-32 of p[0..n) in shared memory by warps 0..6 (called by those 224 threads together).
// Lane-strided Horner form: in round j lane l absorbs word 32j + l of its warp's region, so the
// data reads of a warp are one conflict-free 128-byte row; the step tables advance the state by
// 1024 bits (tabs[4..7]) except in the last round (tabs[0..3], 32 bits); lane l's share is then
// multiplied by x^(32 (31 - l)), a warp's by x^(8 * bytes behind its region).
// crc_std(M) = raw(M with its first four bytes complemented) ^ 0xffffffff.
// ---------------------------------------------------------------------------------------------
__device__ uint32_t g_xpow_lane[32];        // x^(32 (31 - l))

__global__ void crc_init2_kernel()
{
    const uint32_t i = threadIdx.x;
    for (int j = 0; j < 4; j++) {
        uint32_t v = g_crc_tab[j][i];
        for (int k = 0; k < 124; k++) v = g_crc_tab[0][v & 0xff] ^ (v >> 8);
        g_crc_tab2[j][i] = v;
    }
    g_xpow_lo[i] = xpow_bytes(i);
    g_xpow_hi[i] = xpow_bytes(256u * i);
    if (i < 32) g_xpow_lane[i] = xpow_bytes(4u * (31u - i));
    // x^-1 steps: undo one multiplication by x (multmodp's b step), bit 31 = the x^0 coefficient
    uint32_t v = 1u << 31;
    for (uint32_t k = 0; k < 8u * i; k++) v = (v & 0x80000000u) ? ((v ^ 0xEDB88320u) << 1) | 1u : v << 1;
    g_xinv_byte[i] = v;
}

__device__ uint32_t cta_crc32(CtaSmem &cs, uint32_t *tabs /* [8][256], dead table buffer */, uint32_t a0, uint32_t n)
{
    const uint32_t t = threadIdx.x, lane = t & 31, warp = t >> 5;
    constexpr uint32_t NW = P3_T / 32;
    for (uint32_t i = t; i < 1024; i += P3_T) { tabs[i] = (&g_crc_tab[0][0])[i]; tabs[1024 + i] = (&g_crc_tab2[0][0])[i]; }
    bar_p3();
    if (n < 64) {
        uint32_t c = 0xffffffffu;
        for (uint32_t i = 0; i < n; i++) c = tabs[(c ^ sld8(a0 + i)) & 0xff] ^ (c >> 8);
        return ~c;
    }
    const uint32_t mis = a0 & 3u, A0 = a0 - mis, endA = (a0 + n) & ~3u, tail = (a0 + n) & 3u;
    const uint32_t W = (endA - A0) >> 2;
    const uint32_t per = ((W + NW - 1) / NW + 31u) & ~31u;
    const uint32_t rb = warp * per, re = min(W, rb + per);
    uint32_t S = 0;
    if (rb < re) {
        const uint32_t Nw = re - rb, K = (Nw + 31u) >> 5, p = 32u * K - Nw;
        const uint32_t m0 = 0xffffffffu << (8u * mis), m1 = mis ? 0xffffffffu >> (32u - 8u * mis) : 0u;
        uint32_t A = 0;
        int32_t idx = (int32_t)lane - (int32_t)p;
        uint32_t wv = idx >= 0 ? sld32(A0 + 4u * (rb + (uint32_t)idx)) : 0u;
        for (uint32_t j = 0; j < K; j++) {
            uint32_t cur = wv;
            const uint32_t g = rb + (uint32_t)idx;
            if (idx >= 0 && g < 2u) cur = g == 0 ? (cur & m0) ^ m0 : cur ^ m1;      // leading garbage off; first four bytes complemented
            idx += 32;
            if (j + 1 < K) wv = sld32(A0 + 4u * (rb + (uint32_t)idx));               // next word in flight (idx >= 0 from round 1 on)
            A = crc_step4(j + 1 < K ? tabs + 1024 : tabs, A ^ cur);
        }
        S = multmodp(g_xpow_lane[lane], A);
#pragma unroll
        for (int d = 16; d; d >>= 1) S ^= __shfl_xor_sync(0xffffffffu, S, d);
        const uint32_t after = (W - re) * 4u;
        if (after) S = multmodp(multmodp(g_xpow_hi[after >> 8], g_xpow_lo[after & 255u]), S);
    }
    if (lane == 0) cs.c.crc[warp] = S;
    bar_p3();
    uint32_t c = 0;
#pragma unroll
    for (uint32_t w = 0; w < NW; w++) c ^= cs.c.crc[w];
    for (uint32_t i = 0; i < tail; i++) c = tabs[(c ^ sld8(endA + i)) & 0xff] ^ (c >> 8);
    return ~c;
}

// stage the compressed block `blk` (blen bytes, global) at cs.stage so that shared and global
// addresses are congruent mod 16: the 16-byte aligned interior by one bulk copy, the ragged ends
// by plain loads.  Called by ONE warp; its lane 0 issues the copy.
__device__ __forceinline__ void stage_issue_warp(CtaSmem &cs, const uint8_t *blk, uint32_t blen)
{
    const uint32_t lane = hgpu_lane();
    const uint32_t mis = (uint32_t)(reinterpret_cast<uintptr_t>(blk) & 15);
    uint8_t *sp = cs.stage + mis;                                    // byte j of the block -> sp[j]
    uint32_t head = (16u - mis) & 15u;
    if (head > blen) head = blen;
    const uint32_t bulk = (blen - head) & ~15u, tail = blen - head - bulk;
    if (lane < head) sp[lane] = blk[lane];
    if (lane >= 16 && lane - 16 < tail) sp[head + bulk + (lane - 16)] = blk[head + bulk + (lane - 16)];
    __syncwarp();
    if (lane == 0) {
        if (bulk) tma_load_1d(sp + head, blk + head, bulk, &cs.mbar);
        else {
            uint32_t m = (uint32_t)__cvta_generic_to_shared(&cs.mbar);
            asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" :: "r"(m) : "memory");
        }
    }
}

// warp-level: take the next job, stage it, parse its first deflate block header into table buffer `nb`.
// Fills cs.c.next_job / next_staged / h[nb].  The mbarrier phase `parity` is the one this copy completes.
__device__ void prefetch_next(CtaSmem &cs, uint32_t nb, const uint8_t *in, const uint64_t *in_off, const uint32_t *in_len,
                              uint32_t n, uint32_t *counter, uint32_t parity)
{
    const uint32_t lane = hgpu_lane();
#ifdef HGPU_PROFILE
    const long long p1_t0 = clock64();
#endif
    uint32_t job = 0;
    if (lane == 0) job = atomicAdd(counter, 1u);
    job = __shfl_sync(0xffffffffu, job, 0);
    if (lane == 0) cs.c.next_job = job;
    if (job >= n) { if (lane == 0) cs.c.next_staged = 0; __syncwarp(); return; }
    const uint8_t *blk = in + in_off[job];
    const uint32_t blen = in_len[job];
    const bool staged = blen >= 26 && blen <= STAGE_BYTES;
    if (lane == 0) cs.c.next_staged = staged ? 1u : 0u;
    if (staged) {
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");     // earlier generic reads of the staging area vs. the async write
        stage_issue_warp(cs, blk, blen);
        mbar_wait(&cs.mbar, parity);
    }
    __syncwarp();
    const uint8_t *cb = staged ? cs.stage + (uint32_t)(reinterpret_cast<uintptr_t>(blk) & 15) : blk;
    HdrInfo &hi = cs.c.h[nb];
    if (blen < 26 || check_header(cb) != 0 || (uint32_t)(cb[16] | cb[17] << 8) + 1u != blen) {
        if (lane == 0) { hi.rc = HGPU_BGZF_ERR_HEADER; hi.type = 3; hi.final_ = 1; hi.body = 0; hi.len = 0; }
        __syncwarp();
        return;
    }
    Bits b;
    const uint8_t *src = cb + 18;
    bits_init(b, src, 0, blen - 18);
    parse_block_header(cs.s[nb], b, blen - 18, (uint32_t)(reinterpret_cast<uintptr_t>(src) & 3) * 8, hi);
#ifdef HGPU_PROFILE
    if (lane == 0) atomicAdd(&g_prof[7], (unsigned long long)(clock64() - p1_t0));
#endif
}

__global__ void __launch_bounds__(CTA_T, 2)
bgzf_inflate_cta_kernel(const uint8_t *__restrict__ in, const uint64_t *__restrict__ in_off,
                        const uint32_t *__restrict__ in_len, uint32_t n, uint8_t *out,
                        const uint64_t *__restrict__ out_off, const uint32_t *__restrict__ out_cap,
                        uint32_t *out_len, int32_t *status, uint32_t *counter, uint2 *mrec_all)
{
    extern __shared__ __align__(16) uint8_t dyn_smem[];
    CtaSmem &cs = *reinterpret_cast<CtaSmem *>(dyn_smem);
    uint16_t *dglobal = reinterpret_cast<uint16_t *>(mrec_all + (size_t)blockIdx.x * MREC_CAP);
    const uint32_t t = threadIdx.x, lane = t & 31, warp = t >> 5;
    if (t == 0) { mbar_init(&cs.mbar, 1); cs.c.phase = 0; }
    __syncthreads();
    // cold start: warp 7 fetches and parses the first block while the others wait
    uint32_t cur = 0;
    if (warp == 7) prefetch_next(cs, cur, in, in_off, in_len, n, counter, 0);
    __syncthreads();
    uint32_t parity = 0;                                   // mbarrier phase the NEXT staging copy completes
    if (cs.c.next_staged) parity ^= 1u;
    for (;;) {
        const uint32_t job = cs.c.next_job;
        if (job >= n) break;
#ifdef HGPU_PROFILE
        if (t == 0) cs.c.t0 = clock64();
#endif
        const uint8_t *blk = in + in_off[job];
        const uint32_t blen = in_len[job];
        uint8_t *dst = out + out_off[job];
        uint32_t cap = out_cap[job];
        if (cap > 65536u) cap = 65536u;                    // BGZF_MAX_BLOCK_SIZE, bgzf.c:810
        // shared and global addresses congruent mod 16: the payload's byte i sits at win[pad + i]
        const uint32_t pad = (uint32_t)(reinterpret_cast<uintptr_t>(dst) & 15);
        uint8_t *win = cs.win + pad;
        const uint32_t wa = (uint32_t)__cvta_generic_to_shared(win);
        const bool staged = cs.c.next_staged != 0;
        const uint8_t *cb = staged ? cs.stage + (uint32_t)(reinterpret_cast<uintptr_t>(blk) & 15) : blk;
        const uint8_t *src = cb + 18;
        const uint32_t slen = blen >= 18 ? blen - 18 : 0;
        const uintptr_t sa0 = reinterpret_cast<uintptr_t>(src);
        const uint32_t mis_bits = (uint32_t)(sa0 & 3) * 8;
        const uint32_t *wbase = reinterpret_cast<const uint32_t *>(sa0 - (sa0 & 3));
        const uint32_t *wend = reinterpret_cast<const uint32_t *>((sa0 + slen + 3) & ~(uintptr_t)3);
        const uint32_t total = mis_bits + slen * 8;
        HdrInfo hi = cs.c.h[cur];
        int rc = hi.rc;
        uint32_t want = 0;
        if (rc == HGPU_OK) want = cb[blen - 8] | cb[blen - 7] << 8 | cb[blen - 6] << 16 | (uint32_t)cb[blen - 5] << 24;
        if (t == 0) { cs.c.o = 0; cs.c.rc = HGPU_OK; cs.c.job = job; }
        __syncthreads();
        CTA_MARK(cs, 0);
        bool prefetched = false;                           // has warp 7 already taken the next job?
        uint32_t o_final = 0;
        // ---- the member's deflate blocks ----
        while (rc == HGPU_OK) {
            bool last_par = false;
            if (hi.type == 0) {                            // stored
                const uint32_t o = cs.c.o;
                if (o + hi.len > cap) { rc = HGPU_BGZF_ERR_SPACE; break; }
                for (uint32_t i = t; i < hi.len; i += CTA_T) win[o + i] = src[hi.body + i];
                asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
                __syncthreads();
                if (t == 0) cs.c.o = o + hi.len;
                __syncthreads();
            } else if (total - hi.body >= PAR_MIN_BITS) {
                rc = decode_body_cta(cs, cs.s[cur], staged, wbase, wend, hi.body, total, wa, cap, dglobal);
                if (rc) break;
                last_par = true;
            } else {                                       // tiny Huffman block: warp 0 walks it
                if (warp == 0) {
                    Bits b;
                    const uint32_t bp = hi.body - mis_bits;
                    bits_init(b, src, bp >> 3, slen);
                    bits_fill(b);
                    bits_drop(b, bp & 7);
                    uint32_t o = cs.c.o;
                    int r2 = decode_body_uniform<false>(cs.s[cur], b, win, cap, o, nullptr);
                    if (lane == 0) { cs.c.rc = r2; cs.c.o = o; cs.c.end_pos = mis_bits + bits_pos(b); }
                }
                __threadfence_block();
                asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
                __syncthreads();
                rc = cs.c.rc;
                if (rc) break;
            }
            const uint32_t tot_m = last_par ? cs.c.tot_m : 0u;
            // ---- after the last body decode of the member: warp 7 moves on to the next block ----
            if (hi.final_) {
                o_final = cs.c.o;
                if (warp == 7) {
                    prefetch_next(cs, cur ^ 1u, in, in_off, in_len, n, counter, parity);
                    prefetched = true;
                } else {
                    if (tot_m) lz_resolve_cta(cs, reinterpret_cast<uint16_t *>(&cs.s[cur]), wa, tot_m, dglobal);
                    CTA_MARK(cs, 3);
                }
                break;
            }
            // ---- not the final block: resolve, then warp 0 parses the next header in place ----
            if (warp != 7 && tot_m) lz_resolve_cta(cs, reinterpret_cast<uint16_t *>(&cs.s[cur]), wa, tot_m, dglobal);
            __syncthreads();
            if (warp == 0) {
                Bits b;
                uint32_t pos;                              // member-relative bit (Huffman) or byte (stored) where the next header starts
                if (hi.type == 0) pos = (hi.body + hi.len) * 8;
                else pos = cs.c.end_pos - mis_bits;
                bits_init(b, src, pos >> 3, slen);
                bits_fill(b);
                bits_drop(b, pos & 7);
                if (bits_overrun(b)) { if (lane == 0) { cs.c.h[cur].rc = HGPU_BGZF_ERR_ZLIB; } }
                else parse_block_header(cs.s[cur], b, slen, mis_bits, cs.c.h[cur]);
            }
            __threadfence_block();
            __syncthreads();
            hi = cs.c.h[cur];
            rc = hi.rc;
        }
        // an error path leaves warp 7 without its prefetch: do it now (uniform: rc, hi are CTA-uniform)
        if (rc != HGPU_OK) {
            __syncthreads();
            if (warp == 7 && !prefetched) prefetch_next(cs, cur ^ 1u, in, in_off, in_len, n, counter, parity);
        }
        uint32_t got = 0;
        if (rc == HGPU_OK && warp != 7) {
            got = o_final;
            // ---- P4: bulk store first, CRC while it flies ----
            uint32_t head = (16u - pad) & 15u;
            if (head > got) head = got;
            const uint32_t bulk = (got - head) & ~15u, tail = got - head - bulk;
            if (got) {
                if (t < head) dst[t] = win[t];
                if (t >= 32 && t - 32 < tail) dst[head + bulk + (t - 32)] = win[head + bulk + (t - 32)];
                if (bulk) {
                    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");     // generic writes to the window -> async proxy
                    bar_p3();
                    if (t == 0) {
                        uint32_t sa = (uint32_t)__cvta_generic_to_shared(win + head);
                        asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;"
                                     :: "l"(dst + head), "r"(sa), "r"(bulk) : "memory");
                        asm volatile("cp.async.bulk.commit_group;" ::: "memory");
                    }
                }
            }
            const uint32_t crc = cta_crc32(cs, reinterpret_cast<uint32_t *>(&cs.s[cur]), wa, got);
            if (crc != want) rc = HGPU_BGZF_ERR_CRC;
            if (t == 0) {
                asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");       // the window is reused by the next block
                status[job] = rc; out_len[job] = rc == HGPU_OK ? got : 0;
            }
            CTA_MARK(cs, 4);
        } else if (rc != HGPU_OK && t == 0) { status[job] = rc; out_len[job] = 0; }
        __threadfence_block();
        __syncthreads();
        if (cs.c.next_staged) parity ^= 1u;
        cur ^= 1u;
        CTA_MARK(cs, 5);
    }
    if (t == 0) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");   // every bulk store has landed before the CTA retires
}
