// rANS Nx16 decode, the two shapes that carry a CRAM 3.1 slice (SURVEY.md §8a'):
//
//   fast32  32-way streams (RANS_ORDER_X32) with a small alphabet — the 1.5 MB quality blocks.
//           One warp per stream, FOUR such warps per CTA, 11 CTAs per SM (44 streams resident per
//           SM): the kernel holds nothing but the symbol loop (tables are parsed by the prep
//           pass), so it fits 40 registers; per warp 4 KiB byte LUT + 128 B of 8-byte
//           {f - 2^shift, start} records + a 768-byte word ring.
//           Step = lop3 (slot | row) - LDS.U8 - lea - LDS.64 - shf - iadd - imad (R' = (f-2^s)(R>>s) + R - start)
//                  - 2 imad (next row) - shf (symbol nibble) | isetp - vote - lop - popc - lea - LDS.U16
//                  - prmt - popc - lea.   Output bytes are made 4 at a time from symbol nibbles with
//           one PRMT (alphabets <= 8) and leave as aligned 32-bit words.
//   tile4   4-way streams (every small block of a slice, every tok3 token stream): EIGHT streams per
//           warp, one per quad of lanes; a warp-wide ballot serves all eight, each quad ranks its
//           own nibble.  Tables (byte LUT + 4-byte records) are packed into one shared pool.
//
// Both follow rANS_static4x16pr.c:213-328, :504-800 and rANS_static32x16pr.c:254-408, :527-754
// exactly (states renormalise in index order, one 16-bit word each; order-1 segments of U/N
// bytes, the last state owns the U mod N tail).  Table parsing is the shared code of
// rans_nx16.cu (dec_order0 / dec_order1 with a Hook), so header and table semantics — and what
// is an error — are the general decoder's.
//
// Included into the anonymous namespace of rans_nx16.cu.

constexpr int32_t RANS_PENDING = 3;        // internal: table parsed, symbol loop still to run (fast32)

// ---------------------------------------------------------------------------------------------
// classification: one CTA walks the job list in order and writes two ordered index lists
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(1024)
rans_classify_kernel(const uint8_t *__restrict__ in, const uint64_t *__restrict__ in_off,
                     const uint32_t *__restrict__ in_len, uint32_t n, int32_t *status,
                     uint32_t *list32, uint32_t *list4, uint32_t *counts /* [0]=n32 [1]=n4 */)
{
    __shared__ uint32_t wsum[2][32];
    __shared__ uint32_t base[2];
    const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if (tid < 2) base[tid] = 0;
    __syncthreads();
    for (uint32_t i0 = 0; i0 < n; i0 += 1024) {
        uint32_t i = i0 + tid;
        int cls = 0;                                  // 0: general pass, 1: 32-way plain, 2: 4-way plain
        if (i < n) {
            uint32_t len = in_len[i];
            if (len >= 2) {
                uint8_t fmt = in[in_off[i]];
                if (!(fmt & 0xe8)) cls = (fmt & 0x04) ? 1 : 2;      // no STRIPE / CAT / RLE / PACK
            }
            status[i] = cls ? RANS_PENDING : RANS_DEFERRED;
        }
        uint32_t b1 = __ballot_sync(0xffffffffu, cls == 1), b2 = __ballot_sync(0xffffffffu, cls == 2);
        if (lane == 0) { wsum[0][warp] = __popc(b1); wsum[1][warp] = __popc(b2); }
        __syncthreads();
        uint32_t o1 = base[0], o2 = base[1];
        for (uint32_t w = 0; w < warp; w++) { o1 += wsum[0][w]; o2 += wsum[1][w]; }
        if (cls == 1) list32[o1 + __popc(b1 & hgpu_lanemask_lt())] = i;
        if (cls == 2) list4[o2 + __popc(b2 & hgpu_lanemask_lt())] = i;
        __syncthreads();
        if (tid == 0) {
            uint32_t t1 = 0, t2 = 0;
            for (int w = 0; w < 32; w++) { t1 += wsum[0][w]; t2 += wsum[1][w]; }
            base[0] += t1; base[1] += t2;
        }
        __syncthreads();
    }
    if (tid == 0) { counts[0] = base[0]; counts[1] = base[1]; }
}

// ---------------------------------------------------------------------------------------------
// fast32 job record, written by the prep pass
// ---------------------------------------------------------------------------------------------
struct __align__(16) FastJob {
    uint32_t job, ipos, shift, ncol, order, s0, U, hdr;   // hdr: bytes of format byte + size field before the payload
    uint32_t slen, pad[3];      // payload length
    uint8_t  symof[8];          // emit index -> byte
    uint8_t  ctx[32];           // order 1: emit index of every lane's context after the head steps
    uint32_t R[32];             // states (after the head steps for order 1)
    uint32_t prev[32];          // order 1: the lane's last four head bytes, oldest in the low byte
    uint16_t F[64];             // [row][8] normalised frequencies over the emit alphabet
};

constexpr uint32_t F32_WARPS = 4, F32_LUT = 4096, F32_FB = 128, F32_RING = 768;
constexpr uint32_t F32_SMEM = F32_WARPS * (F32_LUT + F32_FB + F32_RING);
constexpr uint32_t F32_HEAD = 4;           // order-1 head steps run by the prep pass
constexpr uint32_t F32_MIN_U = 32 * 64;    // shorter streams stay with the general loops

// The prep pass (one warp per 32-way plain stream): header + table through the general code;
// if the stream fits the fast kernel, run the 4 head steps here (they use the start-context row,
// which the fast kernel never needs again) and write the job, else decode it right here.
__device__ bool fast32_emit(uint8_t *smem, const Hook &h, uint32_t job, uint32_t hdr, FastJob *jobs, uint32_t *njobs)
{
    const uint32_t lane = hgpu_lane();
    const uint16_t *Fc = h.Fcap;
    if (h.ncol > 16 || h.U < F32_MIN_U || h.lb != h.shift) return false;
    // emit alphabet: symbols with a non-zero frequency in any row (order 1: byte 0 may own only the start row)
    uint32_t emit = 0, nullrows = 0;
    const uint32_t rows = h.order ? h.ncol : 1;
    for (uint32_t r = 0; r < rows; r++) {
        if (h.order && Fc[256 + r]) { nullrows |= 1u << r; continue; }
        for (uint32_t k = 0; k < h.ncol; k++) if (Fc[r * 16 + k]) emit |= 1u << k;
    }
    const uint32_t ne = __popc(emit);
    if (ne == 0 || ne > 8) return false;
    if (h.order) {
        if ((ne << h.shift) > F32_LUT || ne > 4) return false;
        if (nullrows & emit) return false;            // a row a valid stream never enters; keep the pinned behaviour of the general loop
    }
    if (h.order && (nullrows & 1u)) return false;     // start-context row must exist
    const uint8_t *symof = smem + SM_SYMOF;
    uint32_t R = h.R, ipos = h.ipos, acc = 0, krow = 0;
    if (h.order) {
        // head: F32_HEAD steps of the general order-1 loop, byte stores (loop_order1's head)
        const uint32_t mask = (1u << h.shift) - 1, seg = h.U / 32;
        uint8_t *op = h.out + (size_t)lane * seg;
        uint8_t *ring = smem + SM_RING;
        WordRing wr;
        ring_init(ring, wr, h.in, h.in_len, ipos);
        uint32_t lrow = h.row0 << h.shift, frow = h.row0 * h.ncol;
        for (uint32_t s = 0; s < F32_HEAD; s++) {
            ring_ensure(ring, wr, ipos, 64);
            uint32_t m = R & mask;
            uint32_t k = h.lut[lrow + m];
            uint32_t e = h.fb[frow + k];
            uint32_t q = R >> h.shift;
            R = (e >> 20) * q + q + m - ((e >> 8) & 0xfffu);
            acc = __funnelshift_l(acc, e, 24);
            lrow = k << h.shift; frow = k * h.ncol; krow = k;
            renorm_safe(R, true, ring, wr, ipos, h.in_len);
            op[s] = (uint8_t)(acc >> 24);
        }
        __syncwarp();
        // every context the fast kernel starts from must be an emit row (always so in a valid stream)
        if (__any_sync(0xffffffffu, !(emit >> krow & 1u))) return false;
    }
    uint32_t slot = 0;
    if (lane == 0) slot = atomicAdd(njobs, 1u);
    slot = __shfl_sync(0xffffffffu, slot, 0);
    FastJob *fj = jobs + slot;
    if (lane == 0) {
        fj->job = job; fj->ipos = ipos; fj->shift = h.shift; fj->ncol = ne; fj->order = h.order;
        fj->s0 = h.order ? F32_HEAD : 0; fj->U = h.U; fj->hdr = hdr; fj->slen = h.in_len;
        uint32_t e = 0;
        for (uint32_t k = 0; k < h.ncol; k++) if (emit >> k & 1) fj->symof[e++] = symof[k];
        for (; e < 8; e++) fj->symof[e] = 0;
    }
    fj->R[lane] = R;
    fj->prev[lane] = acc;
    fj->ctx[lane] = (uint8_t)__popc(emit & ((1u << krow) - 1u));      // every decoded symbol is in the emit set
    // F[re][ke] over emit rows / columns
    for (uint32_t idx = lane; idx < 64; idx += 32) {
        uint32_t re = idx >> 3, ke = idx & 7;
        uint16_t v = 0;
        if (re < (h.order ? ne : 1u) && ke < ne) {
            uint32_t r = h.order ? (uint32_t)__fns(emit, 0, re + 1) : 0u, k = (uint32_t)__fns(emit, 0, ke + 1);
            v = Fc[r * 16 + k];
        }
        fj->F[idx] = v;
    }
    return true;
}

// ---------------------------------------------------------------------------------------------
// fast32 symbol loops
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ void lds_v2(uint32_t a, uint32_t &x, uint32_t &y)
{ asm volatile("ld.shared.v2.u32 {%0, %1}, [%2];" : "=r"(x), "=r"(y) : "r"(a) : "memory"); }
__device__ __forceinline__ void sts_u32(uint32_t a, uint32_t v) { asm volatile("st.shared.u32 [%0], %1;" :: "r"(a), "r"(v) : "memory"); }
__device__ __forceinline__ void sts_v2(uint32_t a, uint32_t x, uint32_t y) { asm volatile("st.shared.v2.u32 [%0], {%1, %2};" :: "r"(a), "r"(x), "r"(y) : "memory"); }

// Word ring of the fast kernel: 512 bytes mirroring the stream from pos0 on, plus a 256-byte
// mirror of its first half so a 4-step group can read linearly past the wrap point.
struct Ring32 {
    const uint8_t *in;
    uintptr_t lim;        // first aligned address entirely past the input
    uint32_t a;           // shared address of the ring
    uint32_t v;           // stream bytes consumed since pos0 ("virtual" position)
    uint32_t loaded;      // virtual position up to which the ring holds data (multiple of 128)
    uint32_t pos0;
};

__device__ __forceinline__ void ring32_load(Ring32 &rg)
{
    const uint32_t lane = hgpu_lane();
    uintptr_t g = reinterpret_cast<uintptr_t>(rg.in) + rg.pos0 + rg.loaded + 4u * lane;
    uintptr_t ga = g & ~(uintptr_t)3;
    uint32_t sh = (uint32_t)(g & 3) * 8;
    uint32_t w0 = ga < rg.lim ? *reinterpret_cast<const uint32_t *>(ga) : 0u;
    uint32_t w1 = ga + 4 < rg.lim ? *reinterpret_cast<const uint32_t *>(ga + 4) : 0u;
    uint32_t w = __funnelshift_r(w0, w1, sh);
    uint32_t off = (rg.loaded & 511u) + 4u * lane;
    sts_u32(rg.a + off, w);
    if (off < 256u) sts_u32(rg.a + 512u + off, w);
    rg.loaded += 128;
}

// keep more than 384 bytes ahead of v (so a 4-step group, <= 256 bytes, never runs dry) without
// overwriting bytes not yet consumed
__device__ __forceinline__ void ring32_fill(Ring32 &rg)
{
    if (rg.loaded - rg.v <= 384u) {
        __syncwarp();
        do ring32_load(rg); while (rg.loaded - rg.v <= 384u);
        __syncwarp();
    }
}

// one bounds-checked renormalisation (RansDecRenormSafe, rANS_word.h:441), ring addressed by v
__device__ __forceinline__ void renorm32_safe(uint32_t &R, bool active, Ring32 &rg, uint32_t in_len)
{
    bool need = active && R < RANS_L;
    uint32_t bal = __ballot_sync(0xffffffffu, need);
    if (bal) {
        uint32_t wv = rg.v + 2u * __popc(bal & hgpu_lanemask_lt());
        uint32_t w = lds_u16(rg.a + (wv & 511u));
        bool ok = need && rg.pos0 + wv + 2u <= in_len;
        if (ok) R = (R << 16) | w;
        rg.v += 2u * __popc(__ballot_sync(0xffffffffu, ok));
    }
}

// prmt with a selector already known to be four 3-bit nibbles (no masking instruction)
__device__ __forceinline__ uint32_t prmt_raw(uint32_t a, uint32_t b, uint32_t sel)
{ uint32_t d; asm("prmt.b32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(sel)); return d; }
__device__ __forceinline__ uint32_t lop3_and_or(uint32_t a, uint32_t b, uint32_t c)      // (a & b) | c
{ uint32_t d; asm("lop3.b32 %0, %1, %2, %3, 0xEA;" : "=r"(d) : "r"(a), "r"(b), "r"(c)); return d; }
__device__ __forceinline__ uint32_t mad_lo(uint32_t a, uint32_t b, uint32_t c)
{ uint32_t d; asm("mad.lo.u32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(c)); return d; }

// SPARSE: streams that renormalise rarely (NovaSeq qualities: 0.015 words per state and step, so
// 6 steps in 10 no lane needs a word) skip the word fetch on a warp-uniform branch.
template <int ORDER, bool SPARSE>
__device__ __forceinline__ void fast32_stream(const FastJob *fj, uint32_t lut_a, uint32_t fb_a, uint32_t ring_a,
                                              const uint8_t *in, uint32_t in_len, uint8_t *out, uint32_t U)
{
    const uint32_t lane = hgpu_lane();
    const uint32_t shift = fj->shift, ncol = fj->ncol;
    const uint32_t total = 1u << shift, mask = total - 1u;
    const uint32_t fstride = ORDER ? 32u : 0u, rowsz = ORDER ? total : 0u;
    // ---- tables: byte LUT rows (emit index per slot) + {f - 2^shift, start} records ----
    __syncwarp();
    {
        const uint32_t rows = ORDER ? ncol : 1u;
        for (uint32_t r = 0; r < rows; r++) {
            uint32_t thr[8], c = 0;
#pragma unroll
            for (int k = 0; k < 8; k++) {
                uint32_t f = fj->F[r * 8 + k];
                if (k == (int)lane && (uint32_t)k < ncol) sts_v2(fb_a + r * 32u + (uint32_t)k * 8u, f - total, c);
                c += f;
                thr[k] = (uint32_t)(k + 1) < ncol ? c : 0xffffffffu;      // thr[k]: first slot of symbol k+1
            }
            for (uint32_t w = lane; w < total / 4; w += 32) {
                uint32_t word = 0;
#pragma unroll
                for (int b = 0; b < 4; b++) {
                    uint32_t y = 4 * w + b, k = 0;
#pragma unroll
                    for (int j = 0; j < 7; j++) k += y >= thr[j];
                    word |= k << (8 * b);
                }
                sts_u32(lut_a + (r << shift) + 4 * w, word);
            }
        }
    }
    const uint32_t mapLo = fj->symof[0] | fj->symof[1] << 8 | fj->symof[2] << 16 | (uint32_t)fj->symof[3] << 24;
    const uint32_t mapHi = fj->symof[4] | fj->symof[5] << 8 | fj->symof[6] << 16 | (uint32_t)fj->symof[7] << 24;
    uint32_t R = fj->R[lane];
    Ring32 rg;
    rg.in = in; rg.lim = (reinterpret_cast<uintptr_t>(in) + in_len + 3) & ~(uintptr_t)3;
    rg.a = ring_a; rg.v = 0; rg.loaded = 0; rg.pos0 = fj->ipos;
    ring32_fill(rg);
    __syncwarp();
    const uint32_t lt = hgpu_lanemask_lt();

#ifdef F32_DEBUG
#define F32_CHECK(A) if ((A) - lut_a >= F32_LUT) { printf("fast32 bad lut addr %x lut_a %x R %x mask %x lrow %x order %d lane %u shift %u ncol %u\n", (A), lut_a, R, mask, lrow, ORDER, lane, shift, ncol); return; }
#else
#define F32_CHECK(A)
#endif
#define F32_SYMBOL(ROWUPD)                                                                         \
        uint32_t a_ = lop3_and_or(R, mask, lrow);                                                  \
        F32_CHECK(a_)                                                                              \
        uint32_t k_ = lds_u8(a_);                                                                  \
        uint32_t x_, y_;                                                                           \
        lds_v2(frow + k_ * 8u, x_, y_);                                                            \
        uint32_t q_ = R >> shift;                                                                  \
        R = x_ * q_ + (R - y_);                                                                    \
        ROWUPD
#define F32_RENORM_FAST                                                                            \
        {                                                                                          \
            bool p_ = R < RANS_L;                                                                  \
            uint32_t bal_ = __ballot_sync(0xffffffffu, p_);                                        \
            if (!SPARSE || bal_) {                                                                 \
                uint32_t w_ = lds_u16(relA + 2u * __popc(bal_ & lt));                              \
                if (p_) R = __byte_perm(w_, R, 0x5410);                                            \
                relA += 2u * __popc(bal_);                                                         \
            }                                                                                      \
        }

    if (ORDER == 0) {
        // out[32 s + lane]; full rows while every lane is active and the input is far from its end
        const uint32_t lrow = lut_a, frow = fb_a;
        const uint32_t nfull = U / 32;
        uint32_t s = 0;
        uint8_t *op = out + lane;
        uint32_t relA = rg.a;
        while (s + 4 <= nfull && rg.pos0 + rg.v + 256u <= in_len) {
            const uint32_t g0 = relA;
#pragma unroll
            for (int j = 0; j < 4; j++) {
                F32_SYMBOL(;)
                op[32 * j] = (uint8_t)prmt_raw(mapLo, mapHi, k_);
                F32_RENORM_FAST
            }
            op += 128; s += 4;
            rg.v += relA - g0;
            if (relA >= rg.a + 512u) relA -= 512u;
            ring32_fill(rg);
        }
        for (uint32_t i = 32 * s + lane; __any_sync(0xffffffffu, i < U); i += 32, op += 32) {
            ring32_fill(rg);
            bool act = i < U;
            uint32_t Rk = R;
            F32_SYMBOL(;)
            if (act) *op = (uint8_t)__byte_perm(mapLo, mapHi, k_); else R = Rk;
            renorm32_safe(R, act, rg, in_len);
        }
    } else {
        const uint32_t seg = U / 32;
        uint8_t *op = out + (size_t)lane * seg;
        uint32_t c0 = fj->ctx[lane];
        uint32_t lrow = lut_a + c0 * rowsz, frow = fb_a + c0 * fstride;
        uint32_t s = fj->s0, acc = 0, prevB = fj->prev[lane];
        // aligned word stores: the word at (op+s) - ph holds ph bytes of the previous group
        const uint32_t ph = (uint32_t)(reinterpret_cast<uintptr_t>(op) + s) & 3u;
        const uint32_t shamt = 32u - 8u * ph;
        uint32_t *wp = reinterpret_cast<uint32_t *>(op + s - ph);
        uint32_t relA = rg.a;
        // one group = 4 steps = one aligned 32-bit word of this lane's segment
#define F32_GROUP(WREG)                                                                            \
        {                                                                                          \
            const uint32_t g0 = relA;                                                              \
            _Pragma("unroll")                                                                      \
            for (int j = 0; j < 4; j++) {                                                          \
                F32_SYMBOL(lrow = mad_lo(k_, rowsz, lut_a); frow = mad_lo(k_, fstride, fb_a);)     \
                acc = __funnelshift_r(acc, k_, 4);                                                 \
                F32_RENORM_FAST                                                                    \
            }                                                                                      \
            uint32_t B = prmt_raw(mapLo, mapHi, acc >> 16);                                        \
            WREG = __funnelshift_rc(prevB, B, shamt);                                              \
            prevB = B;                                                                             \
            rg.v += relA - g0;                                                                     \
            if (relA >= rg.a + 512u) relA -= 512u;                                                 \
            ring32_fill(rg);                                                                       \
        }
        // 16-byte stores: the lanes' segments start at arbitrary addresses, so every lane has its own
        // phase q0 (position of its next word inside a 16-byte line).  The loop body is 4 groups;
        // a line completes after group g for the lanes with (q0 + g) % 4 == 3, and which registers
        // hold its four words is then fixed per g: four predicated STG.128 instead of sixteen
        // 32-bit stores, a quarter of the store transactions (32 lines per STG otherwise).
        if (s + 16 <= seg && rg.pos0 + rg.v + 1024u <= in_len) {
            const uint32_t q0 = (uint32_t)(reinterpret_cast<uintptr_t>(wp) >> 2) & 3u;
            const bool p0 = q0 == 3u, p1 = q0 == 2u, p2 = q0 == 1u, p3 = q0 == 0u;
            uint32_t W0, W1, W2, W3;
            F32_GROUP(W0) wp[0] = W0;
            F32_GROUP(W1) wp[1] = W1;
            F32_GROUP(W2) wp[2] = W2;
            F32_GROUP(W3) wp[3] = W3;
            wp += 4; s += 16;
            while (s + 16 <= seg && rg.pos0 + rg.v + 1024u <= in_len) {
                F32_GROUP(W0) if (p0) *reinterpret_cast<uint4 *>(wp - 3) = make_uint4(W1, W2, W3, W0);
                F32_GROUP(W1) if (p1) *reinterpret_cast<uint4 *>(wp - 2) = make_uint4(W2, W3, W0, W1);
                F32_GROUP(W2) if (p2) *reinterpret_cast<uint4 *>(wp - 1) = make_uint4(W3, W0, W1, W2);
                F32_GROUP(W3) if (p3) *reinterpret_cast<uint4 *>(wp) = make_uint4(W0, W1, W2, W3);
                wp += 4; s += 16;
            }
            wp[-3] = W1; wp[-2] = W2; wp[-1] = W3;       // words of the last body that did not complete a line
        }
        while (s + 4 <= seg && rg.pos0 + rg.v + 256u <= in_len) {
            uint32_t W;
            F32_GROUP(W)
            *wp++ = W;
            s += 4;
        }
#undef F32_GROUP
        // bytes of the last group that have not completed a word (harmless rewrite of the others)
        op[s - 1] = (uint8_t)(prevB >> 24);
        op[s - 2] = (uint8_t)(prevB >> 16);
        op[s - 3] = (uint8_t)(prevB >> 8);
        for (; s < seg; s++) {
            ring32_fill(rg);
            F32_SYMBOL(lrow = k_ * rowsz + lut_a; frow = k_ * fstride + fb_a;)
            op[s] = (uint8_t)__byte_perm(mapLo, mapHi, k_);
            renorm32_safe(R, true, rg, in_len);
        }
        // the last state also produces the U mod 32 tail (rANS_static32x16pr.c:669-680)
        const bool last = lane == 31;
        for (uint32_t s2 = seg * 32; s2 < U; s2++) {
            ring32_fill(rg);
            uint32_t Rk = R, lk = lrow, fk = frow;
            F32_SYMBOL(lrow = k_ * rowsz + lut_a; frow = k_ * fstride + fb_a;)
            if (last) out[s2] = (uint8_t)__byte_perm(mapLo, mapHi, k_);
            else { R = Rk; lrow = lk; frow = fk; }
            renorm32_safe(R, last, rg, in_len);
        }
    }
#undef F32_SYMBOL
#undef F32_RENORM_FAST
    __syncwarp();
}

// where the dynamic shared window of a CTA starts (the system reserves the first KiB of a CTA's shared memory)
__global__ void rans_smem_probe_kernel(uint32_t *o)
{
    extern __shared__ __align__(16) uint8_t smem[];
    if (threadIdx.x == 0) *o = (uint32_t)__cvta_generic_to_shared(smem);
}

__global__ void __launch_bounds__(F32_WARPS * 32, 10)
rans_fast32_kernel(const FastJob *__restrict__ jobs, const uint32_t *__restrict__ njobs,
                   const uint8_t *__restrict__ in, const uint64_t *__restrict__ in_off,
                   const uint32_t *__restrict__ in_len, uint8_t *out, const uint64_t *__restrict__ out_off,
                   const uint32_t *__restrict__ out_len, int32_t *status, uint32_t *counter, uint32_t smem_bytes)
{
    extern __shared__ __align__(16) uint8_t smem[];
    const uint32_t sbase = (uint32_t)__cvta_generic_to_shared(smem);
    const uint32_t warp = threadIdx.x >> 5;
    // LUT rows are addressed with OR, so every warp's LUT sits on a 4 KiB boundary of the shared
    // window: the rings go in front (the window starts 1 KiB in, rings are 3 KiB: no padding then),
    // the records behind.  The host sized the allocation from the probed window start.
    const uint32_t lut0 = (sbase + F32_WARPS * F32_RING + F32_LUT - 1) & ~(F32_LUT - 1);
    if (lut0 + F32_WARPS * (F32_LUT + F32_FB) > sbase + smem_bytes) __trap();
    const uint32_t lut_a = lut0 + warp * F32_LUT;
    const uint32_t fb_a = lut0 + F32_WARPS * F32_LUT + warp * F32_FB;
    const uint32_t ring_a = sbase + warp * F32_RING;
    const uint32_t n = *njobs;
    for (;;) {
        uint32_t j = 0;
        if (hgpu_lane() == 0) j = atomicAdd(counter, 1u);
        j = __shfl_sync(0xffffffffu, j, 0);
        if (j >= n) break;
        const FastJob *fj = jobs + j;
        const uint32_t job = fj->job;
        // the stream's own header was consumed by the prep pass; ipos is relative to the payload
        const uint8_t *sin = in + in_off[job] + fj->hdr;
        const uint32_t slen = fj->slen;
        uint8_t *sout = out + out_off[job];
        const uint32_t U = fj->U;                     // decoded size (the header's, or the caller's for NOSZ)
        (void)out_len; (void)in_len;
        // a job the prep pass could not have written: refuse it rather than index tables with it
        if ((fj->shift != 10 && fj->shift != 12) || fj->ncol == 0 || fj->ncol > 8 || (fj->order && (fj->ncol << fj->shift) > F32_LUT) ||
            (!fj->order && fj->shift != 12) || fj->hdr > in_len[job] || slen > in_len[job] - fj->hdr || fj->ipos > slen) {
            if (hgpu_lane() == 0) {
                printf("fast32: bad job %u: job=%u shift=%u ncol=%u order=%u hdr=%u slen=%u ipos=%u U=%u\n", j, job, fj->shift, fj->ncol,
                       fj->order, fj->hdr, slen, fj->ipos, U);
                status[job] = HGPU_RANS_ERR;
            }
            continue;
        }
        const bool sparse = (uint64_t)slen * 16 < U;      // < 0.5 bit per symbol
        if (fj->order) {
            if (sparse) fast32_stream<1, true>(fj, lut_a, fb_a, ring_a, sin, slen, sout, U);
            else        fast32_stream<1, false>(fj, lut_a, fb_a, ring_a, sin, slen, sout, U);
        } else {
            if (sparse) fast32_stream<0, true>(fj, lut_a, fb_a, ring_a, sin, slen, sout, U);
            else        fast32_stream<0, false>(fj, lut_a, fb_a, ring_a, sin, slen, sout, U);
        }
        if (hgpu_lane() == 0) status[job] = HGPU_OK;
    }
}

// ---------------------------------------------------------------------------------------------
// prep32: one warp per 32-way plain stream (the general pass-0 kernel with a hook)
// ---------------------------------------------------------------------------------------------
constexpr uint32_t PREP_TAB = 6656, PREP_SMEM = SM_TAB + PREP_TAB + 17 * 16 * 2;

__global__ void __launch_bounds__(32, 20)
rans_prep32_kernel(const uint8_t *__restrict__ in, const uint64_t *__restrict__ in_off,
                   const uint32_t *__restrict__ in_len, const uint32_t *__restrict__ list, const uint32_t *__restrict__ counts,
                   uint8_t *out, const uint64_t *__restrict__ out_off, const uint32_t *__restrict__ out_len,
                   uint32_t *got_len, int32_t *status, uint8_t *scratch, size_t scratch_per_cta,
                   uint32_t max_out, FastJob *jobs, uint32_t *njobs, uint32_t *counter)
{
    extern __shared__ __align__(16) uint8_t smem[];
    Hook hook;
    hook.mode = HOOK_X32;
    hook.Fcap = reinterpret_cast<uint16_t *>(smem + SM_TAB + PREP_TAB);
    WarpScratch ws;
    ws.tmp = ws.planes = ws.meta = ws.gtab = nullptr;
    ws.tblbuf = scratch + (size_t)blockIdx.x * scratch_per_cta;
    ws.max_out = max_out;
    ws.tab_base = smem + SM_TAB; ws.tab_cap = PREP_TAB;
    ws.pass = 0; ws.defer = false; ws.hook = &hook;
    const uint32_t n = counts[0];
    for (;;) {
        uint32_t idx = 0;
        if (hgpu_lane() == 0) idx = atomicAdd(counter, 1u);
        idx = __shfl_sync(0xffffffffu, idx, 0);
        if (idx >= n) break;
        const uint32_t job = list[idx];
        const uint8_t *sin = in + in_off[job];
        uint32_t got = 0;
        hook.taken = false;
        int rc = decode_stream(smem, ws, sin, in_len[job], out + out_off[job], out_len[job], got);
        __syncwarp();
        int32_t st;
        if (ws.defer) { st = RANS_DEFERRED; ws.defer = false; }
        else if (rc == RC_HOOKED) {
            if (fast32_emit(smem, hook, job, (uint32_t)(hook.in - sin), jobs, njobs)) st = RANS_PENDING;
            else {
                Table t; t.lut = hook.lut; t.fb = hook.fb; t.ncol = hook.ncol; t.shift = hook.shift; t.lb = hook.lb; t.in_smem = true;
                if (hook.lb != hook.shift) {
                    if (hook.order) loop_order1<true, true, true>(smem, t, hook.in, hook.in_len, hook.ipos, hook.out, hook.U, 32, hook.R, hook.row0);
                    else            loop_order0<true, true>(smem, t, hook.in, hook.in_len, hook.ipos, hook.out, hook.U, 32, hook.R);
                } else if (hook.order) loop_order1<true, true>(smem, t, hook.in, hook.in_len, hook.ipos, hook.out, hook.U, 32, hook.R, hook.row0);
                else            loop_order0<true>(smem, t, hook.in, hook.in_len, hook.ipos, hook.out, hook.U, 32, hook.R);
                __syncwarp();
                st = HGPU_OK;
            }
        } else st = rc ? HGPU_RANS_ERR : HGPU_OK;
        if (hgpu_lane() == 0) { status[job] = st; got_len[job] = (st == HGPU_OK || st == RANS_PENDING) ? got : 0; }
    }
}

// ---------------------------------------------------------------------------------------------
// tile4: eight 4-way streams per warp, one per quad of lanes
// ---------------------------------------------------------------------------------------------
struct Quad {
    uint32_t lut_a, fb_a, mask, shift, cs, rowsz, fstride, ipos, in_len, U, order, job, got;
    const uint8_t *in;
    uint8_t *out;
    uint32_t R[4];
};
constexpr uint32_t T4_POOL = 8192, T4_QUADS = SM_TAB + T4_POOL;                  // compact tables: eight streams' worth
constexpr uint32_t T4_RING = 256;                                                // per quad: a window of its word stream, ring[off & 255] = stream byte off
constexpr uint32_t T4_RINGS = (T4_QUADS + 8 * (uint32_t)sizeof(Quad) + 15u) & ~15u, T4_SMEM = T4_RINGS + 8 * T4_RING;

// The renormalisation words of a quad come from its 256-byte ring (a global round trip per step at 16 warps per SM was
// what bounded this kernel: 9.9 ms for the small blocks of 13 000 slices).  refill: lane z of the quad brings the 16
// stream bytes at loaded + 16 z (aligned words, funnel-shifted), 64 bytes per quad and call.
__device__ __forceinline__ void quad_refill(uint32_t ring_a, const uint8_t *in, uint32_t in_len, uint32_t &loaded, uint32_t z, bool go)
{
    if (go) {
        const uint32_t off = loaded + 16u * z;
        const uintptr_t g = reinterpret_cast<uintptr_t>(in) + off, ga = g & ~(uintptr_t)3;
        const uintptr_t lim = (reinterpret_cast<uintptr_t>(in) + in_len + 3) & ~(uintptr_t)3;
        const uint32_t sh = (uint32_t)(g & 3) * 8u;
        uint32_t w[5];
#pragma unroll
        for (int k = 0; k < 5; k++) w[k] = ga + 4u * k < lim ? *reinterpret_cast<const uint32_t *>(ga + 4u * k) : 0u;
        const uint32_t ra = ring_a + (off & (T4_RING - 1u));
        asm volatile("st.shared.v4.u32 [%0], {%1, %2, %3, %4};" :: "r"(ra), "r"(__funnelshift_r(w[0], w[1], sh)), "r"(__funnelshift_r(w[1], w[2], sh)),
                     "r"(__funnelshift_r(w[2], w[3], sh)), "r"(__funnelshift_r(w[3], w[4], sh)) : "memory");
        loaded += 64u;
    }
}

__device__ __forceinline__ void renorm_quad(uint32_t &R, bool act, uint32_t ring_a, uint32_t &ipos, uint32_t in_len,
                                            uint32_t qsh, uint32_t zlt)
{
    bool need = act && R < RANS_L;
    uint32_t bal = __ballot_sync(0xffffffffu, need);
    if (bal) {
        uint32_t wpos = ipos + 2u * __popc((bal >> qsh) & zlt);
        bool ok = need && wpos + 2u <= in_len;
        // two byte reads: the word stream starts at any byte offset, so a word may wrap around the ring's end
        const uint32_t w = lds_u8(ring_a + (wpos & (T4_RING - 1u))) | lds_u8(ring_a + ((wpos + 1u) & (T4_RING - 1u))) << 8;
        if (ok) R = (R << 16) | w;
        uint32_t bok = __ballot_sync(0xffffffffu, ok);
        ipos += 2u * __popc((bok >> qsh) & 15u);
    }
}

__device__ void tile4_run(const Quad *quads, uint32_t nq, uint32_t idle_a, uint32_t rings_a)
{
    const uint32_t lane = hgpu_lane(), q = lane >> 2, z = lane & 3, qsh = lane & 28u, zlt = (1u << z) - 1u;
    const bool live = q < nq;
    const Quad &Q = quads[live ? q : 0];
    const uint32_t lut_a = live ? Q.lut_a : idle_a, fb_a = live ? Q.fb_a : idle_a;
    const uint32_t mask = live ? Q.mask : 0u, shift = Q.shift, cs = Q.cs, rowsz = live ? Q.rowsz : 0u, fstride = live ? Q.fstride : 0u;
    const uint32_t in_len = Q.in_len, U = live ? Q.U : 0u, order = Q.order;
    const uint8_t *in = Q.in;
    uint32_t ipos = Q.ipos, R = Q.R[z];
    const uint32_t nsteps = U >> 2, rem = U & 3u;
    uint8_t *op = Q.out + (order ? (size_t)z * nsteps : (size_t)z);
    const uint32_t istride = order ? 1u : 4u;
    uint32_t maxsteps = nsteps;
#pragma unroll
    for (int d = 16; d; d >>= 1) maxsteps = max(maxsteps, __shfl_xor_sync(0xffffffffu, maxsteps, d));
    uint32_t lrow = 0, frow = 0;
    const uint32_t ring_a = rings_a + q * T4_RING;
    uint32_t loaded = ipos & ~15u;                           // the ring holds stream bytes [loaded - 256, loaded)
    for (int f = 0; f < 3; f++) quad_refill(ring_a, in, in_len, loaded, z, live);
    __syncwarp();
    for (uint32_t i = 0; i < maxsteps; i++) {
        const bool act = i < nsteps;
        {   // a step takes at most 8 bytes: keep 72 ahead (never more than 136 held)
            const bool fill = live && loaded - ipos < 72u;
            if (__any_sync(0xffffffffu, fill)) { quad_refill(ring_a, in, in_len, loaded, z, fill); __syncwarp(); }
        }
        uint32_t m = R & mask;
        uint32_t k = lds_u8(lut_a + lrow + (m >> cs));
        uint32_t e = lds_u32(fb_a + frow + k * 4u);
        for (;;) {                                           // compact rows: walk forward while m lies behind the record's range
            const bool go = live && m >= ((e >> 8) & 0xfffu) + (e >> 20) + 1u;
            if (!__any_sync(0xffffffffu, go)) break;
            if (go) { k++; e = lds_u32(fb_a + frow + k * 4u); }
        }
        if (act) {
            uint32_t qq = R >> shift;
            R = (e >> 20) * qq + qq + m - ((e >> 8) & 0xfffu);
            op[(size_t)i * istride] = (uint8_t)e;
            lrow = k * rowsz; frow = k * fstride;
        }
        renorm_quad(R, act, ring_a, ipos, in_len, qsh, zlt);
    }
    // tails: order 0 — the first U mod 4 states give one more symbol (rANS_static4x16pr.c:320-327);
    //        order 1 — the last state runs on for U mod 4 symbols (:760-790)
    for (uint32_t t = 0; t < 3; t++) {
        const bool act = order ? (z == 3 && t < rem) : (t == 0 && z < rem);
        if (!__any_sync(0xffffffffu, act)) break;
        uint32_t m = R & mask;
        uint32_t k = lds_u8(lut_a + lrow + (m >> cs));
        uint32_t e = lds_u32(fb_a + frow + k * 4u);
        for (;;) {
            const bool go = live && m >= ((e >> 8) & 0xfffu) + (e >> 20) + 1u;
            if (!__any_sync(0xffffffffu, go)) break;
            if (go) { k++; e = lds_u32(fb_a + frow + k * 4u); }
        }
        if (act) {
            uint32_t qq = R >> shift;
            R = (e >> 20) * qq + qq + m - ((e >> 8) & 0xfffu);
            Q.out[order ? (size_t)4 * nsteps + t : (size_t)4 * nsteps + z] = (uint8_t)e;
            lrow = k * rowsz; frow = k * fstride;
        }
        renorm_quad(R, act, ring_a, ipos, in_len, qsh, zlt);
    }
    __syncwarp();
}

__global__ void __launch_bounds__(32, 16)
rans_tile4_kernel(const uint8_t *__restrict__ in, const uint64_t *__restrict__ in_off,
                  const uint32_t *__restrict__ in_len, const uint32_t *__restrict__ list, const uint32_t *__restrict__ counts,
                  uint8_t *out, const uint64_t *__restrict__ out_off, const uint32_t *__restrict__ out_len,
                  uint32_t *got_len, int32_t *status, uint8_t *scratch, size_t scratch_per_cta,
                  uint32_t max_out, uint32_t *counter)
{
    extern __shared__ __align__(16) uint8_t smem[];
    const uint32_t lane = hgpu_lane();
    Quad *quads = reinterpret_cast<Quad *>(smem + T4_QUADS);
    Hook hook;
    hook.mode = HOOK_N4;
    hook.Fcap = nullptr;
    WarpScratch ws;
    ws.tmp = ws.planes = ws.meta = ws.gtab = nullptr;
    ws.tblbuf = scratch + (size_t)blockIdx.x * scratch_per_cta;
    ws.max_out = max_out;
    ws.pass = 0; ws.defer = false; ws.hook = &hook;
    ws.compact = true;                               // eight streams' tables share the pool
    const uint32_t n = counts[1];
    const uint32_t NONE = 0xffffffffu;
    uint32_t carry = NONE;
    bool exhausted = false;
    for (;;) {
        uint32_t nq = 0, used = 0;
        while (nq < 8) {
            uint32_t job = carry;
            carry = NONE;
            if (job == NONE) {
                if (exhausted) break;
                uint32_t idx = 0;
                if (lane == 0) idx = atomicAdd(counter, 1u);
                idx = __shfl_sync(0xffffffffu, idx, 0);
                if (idx >= n) { exhausted = true; break; }
                job = list[idx];
            }
            ws.tab_base = smem + SM_TAB + used; ws.tab_cap = T4_POOL - used;
            hook.taken = false;
            uint32_t got = 0;
            int rc = decode_stream(smem, ws, in + in_off[job], in_len[job], out + out_off[job], out_len[job], got);
            __syncwarp();
            if (ws.defer) {
                ws.defer = false;
                if (used == 0) { if (lane == 0) { status[job] = RANS_DEFERRED; got_len[job] = 0; } continue; }
                carry = job;                              // does not fit beside the others: first of the next round
                break;
            }
            if (rc == RC_HOOKED) {
                if (lane == 0) {
                    Quad &Q = quads[nq];
                    Q.lut_a = (uint32_t)__cvta_generic_to_shared(hook.lut);
                    Q.fb_a = (uint32_t)__cvta_generic_to_shared(hook.fb);
                    Q.mask = (1u << hook.shift) - 1u; Q.shift = hook.shift; Q.cs = hook.shift - hook.lb;
                    Q.rowsz = hook.order ? 1u << hook.lb : 0u;
                    Q.fstride = hook.order ? hook.ncol * 4u : 0u;
                    Q.ipos = hook.ipos; Q.in_len = hook.in_len; Q.U = hook.U; Q.order = hook.order; Q.job = job; Q.got = got;
                    Q.in = hook.in; Q.out = hook.out;
                }
                if (lane < 4) quads[nq].R[lane] = hook.R;
                used += (hook.tab_bytes + 15u) & ~15u;
                nq++;
            } else if (lane == 0) {
                status[job] = rc ? HGPU_RANS_ERR : HGPU_OK;
                got_len[job] = rc ? 0 : got;
            }
        }
        if (nq == 0) {
            if (exhausted && carry == NONE) break;
            continue;
        }
        __syncwarp();
        tile4_run(quads, nq, (uint32_t)__cvta_generic_to_shared(smem + SM_TAB), (uint32_t)__cvta_generic_to_shared(smem + T4_RINGS));
        if (lane < nq) { status[quads[lane].job] = HGPU_OK; got_len[quads[lane].job] = quads[lane].got; }
        __syncwarp();
    }
}
