// BGZF block inflate for sm_90a: one warp per <=64 KiB BGZF block.
//
// Replaces, for a batch of blocks, what one htslib worker does per job in bgzf_decode_func
// (bgzf.c:1373-1384): check_header (:896-903), inflate_block (:808-824) -> bgzf_uncompress
// (:762-804, raw inflate with a 32 KiB window) and the CRC32 comparison against the footer.
// DEFLATE itself (RFC 1951) and CRC-32 live in zlib/libdeflate for the reference; here they are
// written from the RFC for the GPU.
//
// Kernel structure: the warp parses block headers in lock step and builds the decode tables in
// parallel (canonical code assignment by __match_any_sync ranks) into shared memory:
//   litlen: 9-bit root + sub-tables, dist: 8-bit root + sub-tables, 32-bit entries
//     [31:16] value (literal / length base / distance base / sub-table offset)
//     [15:8]  extra-bit count (or sub-table index bits)
//     [7:4]   kind   [3:0] code bits consumed
// Large deflate block bodies are decoded speculatively, one sub-range per lane; small ones by all
// lanes in lock step.  LZ77 matches are executed 32 at a time, out of order inside a batch, with
// warp-coalesced word copies.  The CRC-32 of the output is computed by the same warp while it
// inflates: a cursor absorbs each 128-byte row of the output as soon as the row is final.
#include "hgpu_internal.h"

namespace {

constexpr int LIT_ROOT = 9, DST_ROOT = 8;
constexpr int LIT_TABLE = (1 << LIT_ROOT) + 856;    // zlib "enough 286 9 15" = 852 sub-table slots
constexpr int DST_TABLE = (1 << DST_ROOT) + 512;    // 30 symbols / 8 root bits: < 4 groups x 128
constexpr int CL_TABLE = 128;

// entry kinds: one bit each for literal / length / distance / end-of-block (so a symbol loop can test them without
// compares); a sub-table link has the literal and length bits both set; no bit set = invalid code
enum : uint32_t { K_BAD = 0, K_LIT = 1, K_LEN = 2, K_SUB = 3, K_DIST = 4, K_EOB = 8 };
#define ENTRY(value, xb, kind, nbits) (((uint32_t)(value) << 16) | ((uint32_t)(xb) << 8) | ((uint32_t)(kind) << 4) | (uint32_t)(nbits))
constexpr uint32_t BAD_ENTRY = ENTRY(0, 0, K_BAD, 0);

// The two areas behind the decode tables are never live at the same time (table building /
// match execution), so they share storage.
struct InflateSmem {
    uint32_t lit[LIT_TABLE];
    uint32_t dst[DST_TABLE];
    union {
        struct {                     // header parse + table construction
            uint32_t cl[CL_TABLE];
            uint16_t code[320];      // canonical code per symbol
            uint8_t  lens[320];
            uint32_t count[16];
            uint32_t next[16];
            uint32_t sub_alloc;
        };
        struct {                     // match execution
            uint2 rbuf[32];          // match records parked by the serial decoder
        };
    };
};
// the dynamic shared memory per CTA (4 KiB + INFLATE_WARPS x this) sets the occupancy: 3 CTAs of 7 warps per SM
static_assert(sizeof(InflateSmem) == 10152, "InflateSmem size sets the inflate kernels' occupancy");

__constant__ uint16_t c_len_base[29] = {3,4,5,6,7,8,9,10,11,13,15,17,19,23,27,31,35,43,51,59,67,83,99,115,131,163,195,227,258};
__constant__ uint8_t  c_len_xtra[29] = {0,0,0,0,0,0,0,0,1,1,1,1,2,2,2,2,3,3,3,3,4,4,4,4,5,5,5,5,0};
__constant__ uint16_t c_dst_base[30] = {1,2,3,4,5,7,9,13,17,25,33,49,65,97,129,193,257,385,513,769,1025,1537,2049,3073,4097,6145,8193,12289,16385,24577};
__constant__ uint8_t  c_dst_xtra[30] = {0,0,0,0,1,1,2,2,3,3,4,4,5,5,6,6,7,7,8,8,9,9,10,10,11,11,12,12,13,13};
__constant__ uint8_t  c_cl_order[19] = {16,17,18,0,8,7,9,6,10,5,11,4,12,3,13,2,14,1,15};

// Optional per-phase cycle accounting (build with -DHGPU_PROFILE; read with hgpu_debug_profile).
#ifdef HGPU_PROFILE
__device__ unsigned long long g_prof[16];
struct Prof {
    long long t;
    __device__ __forceinline__ void start() { t = clock64(); }
    __device__ __forceinline__ void mark(int i) { long long n = clock64(); if (hgpu_lane() == 0) atomicAdd(&g_prof[i], (unsigned long long)(n - t)); t = n; }
};
#else
struct Prof {
    __device__ __forceinline__ void start() {}
    __device__ __forceinline__ void mark(int) {}
};
#endif

__device__ uint32_t g_crc_tab[4][256];      // slice-by-4 tables, filled once by crc_init_kernel
__device__ uint32_t g_xpow_lo[256];         // x^(8 i) mod P            (crc_init2_kernel)
__device__ uint32_t g_xpow_hi[256];         // x^(8 * 256 i) mod P
__device__ uint32_t g_crc_tab2[4][256];     // slice-by-4 tables advanced by 124 more zero bytes (x^1024 per word)
__device__ uint32_t g_xinv_byte[256];       // x^(-8 z) mod P  (x is invertible: P(0) = 1)

// ---------------------------------------------------------------------------------------------
// Bit reader: warp-uniform, 64-bit buffer refilled with aligned 32-bit words.
// ---------------------------------------------------------------------------------------------
struct Bits {
    const uint32_t *w;     // next aligned word to load
    const uint32_t *wend;  // first word entirely past the input
    uint64_t buf;
    int cnt;               // valid bits in buf
    int64_t avail;         // bits of real input not yet moved into buf (may go negative = overrun)
    uint32_t end_bits;     // input length in bits, measured from the member's first byte
};

// Start reading at byte `offset` of a member of `slen` bytes.
__device__ __forceinline__ void bits_init(Bits &b, const uint8_t *src, uint32_t offset, uint32_t slen)
{
    const uint8_t *p = src + offset;
    uint32_t nbytes = slen - offset;
    b.end_bits = slen * 8;
    uintptr_t a = reinterpret_cast<uintptr_t>(p);
    uint32_t mis = (uint32_t)(a & 3);
    b.w = reinterpret_cast<const uint32_t *>(a - mis);
    b.wend = reinterpret_cast<const uint32_t *>((a + nbytes + 3) & ~(uintptr_t)3);
    b.buf = 0; b.cnt = 0;
    b.avail = (int64_t)nbytes * 8;
    if (mis) {
        uint32_t v = b.w < b.wend ? *b.w : 0;
        b.w++;
        b.buf = v >> (8 * mis);
        b.cnt = 32 - 8 * (int)mis;
        b.avail -= b.cnt;
    }
}

// guarantee >= 32 valid bits (zero-padded past the end; overrun is detected via avail)
__device__ __forceinline__ void bits_fill(Bits &b)
{
    if (b.cnt <= 32) {
        uint32_t v = b.w < b.wend ? (*b.w) : 0;
        b.w++;
        b.buf |= (uint64_t)v << b.cnt;
        b.cnt += 32;
        b.avail -= 32;
    }
}
__device__ __forceinline__ uint32_t bits_peek(const Bits &b, int n) { return (uint32_t)b.buf & ((1u << n) - 1u); }
__device__ __forceinline__ void bits_drop(Bits &b, int n) { b.buf >>= n; b.cnt -= n; }
__device__ __forceinline__ uint32_t bits_get(Bits &b, int n) { uint32_t v = bits_peek(b, n); bits_drop(b, n); return v; }
// true once more bits were consumed than the input holds
__device__ __forceinline__ bool bits_overrun(const Bits &b) { return b.avail + b.cnt < 0; }
// bit position of the next unread bit, from the member's first byte
__device__ __forceinline__ uint32_t bits_pos(const Bits &b) { return (uint32_t)((int64_t)b.end_bits - (b.avail + b.cnt)); }

// ---------------------------------------------------------------------------------------------
// Huffman table construction (warp-parallel).  lens[0..n) in shared memory.
// Returns 0 ok, -1 invalid (over-subscribed, or incomplete where zlib refuses it).
// kind_of(sym) supplies the entry payload.
// ---------------------------------------------------------------------------------------------
template <int ROOT, int CAP, typename MakeEntry>
__device__ int build_table(InflateSmem &s, uint32_t *table, int n, bool allow_single, MakeEntry make)
{
    const uint32_t lane = hgpu_lane();
    __syncwarp();
    if (lane < 16) s.count[lane] = 0;
    for (int i = lane; i < CAP; i += 32) table[i] = BAD_ENTRY;
    if (lane == 0) s.sub_alloc = 1u << ROOT;
    __syncwarp();
    for (int i = lane; i < n; i += 32) atomicAdd(&s.count[s.lens[i]], 1u);
    __syncwarp();
    // canonical first codes + Kraft check (zlib inftrees.c: over-subscribed -> error; incomplete
    // only tolerated when the longest code is 1 bit)
    int maxlen = 0;
    int64_t left = 1;
    uint32_t code = 0;
    bool over = false;
    for (int l = 1; l <= 15; l++) {
        uint32_t c = s.count[l];
        left = (left << 1) - (int64_t)c;
        if (left < 0) over = true;
        if (c) maxlen = l;
        code = (code + (l > 1 ? s.count[l - 1] : 0)) << 1;
        if (l == 1) code = 0;
        if (lane == 0) s.next[l] = code;
    }
    if (over) return -1;
    if (maxlen == 0) return allow_single ? 0 : -1;       // no codes at all: every lookup is invalid
    if (left > 0 && !(allow_single && maxlen == 1)) return -1;
    __syncwarp();
    // per-symbol canonical codes, in symbol order: rank within its length class
    for (int base = 0; base < n; base += 32) {
        int i = base + lane;
        uint32_t l = i < n ? s.lens[i] : 0;
        uint32_t peers = __match_any_sync(0xffffffffu, l);
        uint32_t rank = __popc(peers & hgpu_lanemask_lt());
        if (l) s.code[i] = (uint16_t)(s.next[l] + rank);
        __syncwarp();
        if (l && rank + 1 == (uint32_t)__popc(peers)) s.next[l] += __popc(peers);   // last peer bumps the class
        __syncwarp();
    }
    // root entries for short codes; longest length per root prefix for long ones
    for (int i = lane; i < n; i += 32) {
        uint32_t l = s.lens[i];
        if (!l) continue;
        uint32_t rev = __brev((uint32_t)s.code[i]) >> (32 - l);
        if (l <= ROOT) {
            uint32_t e = make(i, l);
            for (uint32_t k = rev; k < (1u << ROOT); k += 1u << l) table[k] = e;
        } else {
            // temporarily keep the max length of the group in the root slot (kind K_SUB, value 0)
            atomicMax(&table[rev & ((1u << ROOT) - 1)], ENTRY(0, l - ROOT, K_SUB, ROOT) | 0x80000000u);
        }
    }
    __syncwarp();
    // allocate sub-tables
    for (uint32_t k = lane; k < (1u << ROOT); k += 32) {
        uint32_t e = table[k];
        if (e & 0x80000000u) {
            uint32_t sub_bits = (e >> 8) & 0xff;
            uint32_t off = atomicAdd(&s.sub_alloc, 1u << sub_bits);
            table[k] = off + (1u << sub_bits) <= (uint32_t)CAP ? ENTRY(off, sub_bits, K_SUB, ROOT) : BAD_ENTRY;
        }
    }
    __syncwarp();
    if (s.sub_alloc > (uint32_t)CAP) return -1;      // cannot happen for a valid code set
    for (int i = lane; i < n; i += 32) {
        uint32_t l = s.lens[i];
        if (l <= ROOT) continue;
        uint32_t rev = __brev((uint32_t)s.code[i]) >> (32 - l);
        uint32_t root = table[rev & ((1u << ROOT) - 1)];
        uint32_t off = root >> 16, sub_bits = (root >> 8) & 0xff;
        uint32_t e = make(i, l - ROOT);
        for (uint32_t k = rev >> ROOT; k < (1u << sub_bits); k += 1u << (l - ROOT)) table[off + k] = e;
    }
    __syncwarp();
    return 0;
}

__device__ __forceinline__ uint32_t lit_entry(int sym, uint32_t nbits)
{
    if (sym < 256) return ENTRY(sym, 0, K_LIT, nbits);
    if (sym == 256) return ENTRY(0, 0, K_EOB, nbits);
    if (sym > 285) return ENTRY(0, 0, K_BAD, nbits);
    return ENTRY(c_len_base[sym - 257], c_len_xtra[sym - 257], K_LEN, nbits);
}
__device__ __forceinline__ uint32_t dst_entry(int sym, uint32_t nbits)
{
    if (sym > 29) return ENTRY(0, 0, K_BAD, nbits);
    return ENTRY(c_dst_base[sym], c_dst_xtra[sym], K_DIST, nbits);
}
__device__ __forceinline__ uint32_t cl_entry(int sym, uint32_t nbits) { return ENTRY(sym, 0, K_LIT, nbits); }

template <int ROOT>
__device__ __forceinline__ uint32_t lookup(const uint32_t *table, Bits &b)
{
    uint32_t e = table[bits_peek(b, ROOT)];
    if (((e >> 4) & 15) == K_SUB) {
        bits_drop(b, ROOT);
        e = table[(e >> 16) + bits_peek(b, (e >> 8) & 0xff)];
    }
    bits_drop(b, e & 15);
    return e;
}

// ---------------------------------------------------------------------------------------------
// CRC-32
// ---------------------------------------------------------------------------------------------
__device__ uint32_t multmodp(uint32_t a, uint32_t b)       // a*b mod P, reflected (zlib crc32.c)
{
    uint32_t p = 0;
    for (uint32_t m = 1u << 31; m; m >>= 1) {
        if (a & m) p ^= b;
        b = (b & 1) ? (b >> 1) ^ 0xEDB88320u : b >> 1;
    }
    return p;
}

// x^(8*nbytes) mod P
__device__ uint32_t xpow_bytes(uint32_t nbytes)
{
    uint32_t p = 1u << 31;            // x^0
    uint32_t sq = 1u << 23;           // x^8  (one byte)
    while (nbytes) {
        if (nbytes & 1) p = multmodp(sq, p);
        sq = multmodp(sq, sq);
        nbytes >>= 1;
    }
    return p;
}

__global__ void crc_init_kernel()
{
    uint32_t i = threadIdx.x;
    uint32_t c = i;
    for (int k = 0; k < 8; k++) c = (c >> 1) ^ (0xEDB88320u & (0u - (c & 1)));
    g_crc_tab[0][i] = c;
    __syncthreads();
    uint32_t c1 = g_crc_tab[0][c & 0xff] ^ (c >> 8);
    g_crc_tab[1][i] = c1;
    uint32_t c2 = g_crc_tab[0][c1 & 0xff] ^ (c1 >> 8);
    g_crc_tab[2][i] = c2;
    uint32_t c3 = g_crc_tab[0][c2 & 0xff] ^ (c2 >> 8);
    g_crc_tab[3][i] = c3;
}

// g_crc_tab2, g_xpow_lo / hi and g_xinv_byte; reads g_crc_tab, so it runs after crc_init_kernel
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
    // x^-1 steps: undo one multiplication by x (multmodp's b step), bit 31 = the x^0 coefficient
    uint32_t v = 1u << 31;
    for (uint32_t k = 0; k < 8u * i; k++) v = (v & 0x80000000u) ? ((v ^ 0xEDB88320u) << 1) | 1u : v << 1;
    g_xinv_byte[i] = v;
}

// CRC-32 of out[0..n) by the whole warp.  Caller must have made the bytes visible.
__device__ uint32_t warp_crc32(const uint32_t (*tab)[256], const uint8_t *out, uint32_t n)
{
    const uint32_t lane = hgpu_lane();
    uint32_t c = n / 32, r = n % 32;
    // lane 0 takes c + r bytes, every other lane c bytes
    uint32_t beg = lane == 0 ? 0 : r + lane * c;
    uint32_t len = lane == 0 ? c + r : c;
    uint32_t crc = 0xffffffffu;
    const uint8_t *p = out + beg, *e = p + len;
    while (p < e && (reinterpret_cast<uintptr_t>(p) & 15)) crc = tab[0][(crc ^ *p++) & 0xff] ^ (crc >> 8);
    if (e - p >= 16) {
        // 16 bytes per load, the next load always in flight (the data sits in L2, ~300 cycles away)
        uint4 nx = *reinterpret_cast<const uint4 *>(p);
        while (e - p >= 16) {
            uint4 cur = nx;
            p += 16;
            if (e - p >= 16) nx = *reinterpret_cast<const uint4 *>(p);
            uint32_t wv[4] = {cur.x, cur.y, cur.z, cur.w};
#pragma unroll
            for (int k = 0; k < 4; k++) {
                crc ^= wv[k];
                crc = tab[3][crc & 0xff] ^ tab[2][(crc >> 8) & 0xff] ^ tab[1][(crc >> 16) & 0xff] ^ tab[0][crc >> 24];
            }
        }
    }
    while (p < e) crc = tab[0][(crc ^ *p++) & 0xff] ^ (crc >> 8);
    crc = ~crc;
    if (c == 0) return __shfl_sync(0xffffffffu, crc, 0);
    // combine: crc(A||B) = crc(A) * x^(8|B|) ^ crc(B)   (crc32_combine).  Level d merges blocks
    // of d lanes; the right-hand block is always d*c bytes long.
    uint32_t xp = c < 65536u ? multmodp(g_xpow_hi[c >> 8], g_xpow_lo[c & 255u]) : xpow_bytes(c);      // x^(8c) mod P
    for (int d = 1; d < 32; d <<= 1) {
        uint32_t right = __shfl_down_sync(0xffffffffu, crc, d);
        if ((lane & (2 * d - 1)) == 0) crc = multmodp(xp, crc) ^ right;
        xp = multmodp(xp, xp);
    }
    return __shfl_sync(0xffffffffu, crc, 0);
}

// predicated global-memory accesses (straight-line code: `if (c) x = *p` would become a divergent branch)
__device__ __forceinline__ uint32_t ld32_if(const uint8_t *a, bool c)
{
    uint32_t v;
    asm volatile("{\n\t.reg .pred q;\n\tsetp.ne.u32 q, %2, 0;\n\tmov.u32 %0, 0;\n\t@q ld.global.u32 %0, [%1];\n\t}" : "=r"(v) : "l"(a), "r"((uint32_t)c) : "memory");
    return v;
}
__device__ __forceinline__ void st32_if(uint8_t *a, uint32_t v, bool c)
{
    asm volatile("{\n\t.reg .pred q;\n\tsetp.ne.u32 q, %2, 0;\n\t@q st.global.u32 [%0], %1;\n\t}" :: "l"(a), "r"(v), "r"((uint32_t)c) : "memory");
}
__device__ __forceinline__ void st8_if(uint8_t *a, uint32_t v, bool c)
{
    asm volatile("{\n\t.reg .pred q;\n\tsetp.ne.u32 q, %2, 0;\n\t@q st.global.u8 [%0], %1;\n\t}" :: "l"(a), "r"(v), "r"((uint32_t)c) : "memory");
}

// ---------------------------------------------------------------------------------------------
// CRC-32 of a member's output, absorbed while it is being written.
//
// The output is read in 128-byte rows aligned to their address (one cache line, one coalesced
// 32-bit load per lane), each row as soon as every byte in it is final and still hot in L1/L2.
// Lane-strided Horner form: lane l absorbs word l of every row and advances its
// sum by x^1024 per row (the tables in shared memory are g_crc_tab2).  The message starts at byte
// m0 of row 0: bytes before it are read as zero (a leading zero does not change a CRC without
// its initial value), and its first four bytes are complemented, which stands for that initial
// value.  At the end the last row is zero-padded by z bytes; lane l's sum times x^(-32 l), summed
// over the lanes, is the register after the padded message, and x^(-8 z) takes the padding out.
// Words at the member's edges are read bytewise: the bytes around a member belong to other warps
// and may lie outside the allocation.
// ---------------------------------------------------------------------------------------------
struct CrcCursor {
    const uint32_t *tab;      // g_crc_tab2 in shared memory
    const uint8_t *row0;      // the member's output rounded down to 128 bytes
    uint32_t m0;              // member start inside row 0
    uint32_t next;            // first row not absorbed yet
    uint32_t acc;             // this lane's Horner sum
};

__device__ __forceinline__ uint32_t crc_step4(const uint32_t *tab, uint32_t v)
{
    return tab[3 * 256 + (v & 0xff)] ^ tab[2 * 256 + ((v >> 8) & 0xff)] ^ tab[256 + ((v >> 16) & 0xff)] ^ tab[v >> 24];
}

__device__ __forceinline__ uint32_t ldg32(const uint8_t *a) { uint32_t v; asm volatile("ld.global.u32 %0, [%1];" : "=r"(v) : "l"(a) : "memory"); return v; }
__device__ __forceinline__ uint32_t ldg8(const uint8_t *a) { uint32_t v; asm volatile("ld.global.u8 %0, [%1];" : "=r"(v) : "l"(a) : "memory"); return v; }

__device__ __forceinline__ void crc_begin(CrcCursor &c, const uint32_t *tab, const uint8_t *out)
{
    const uintptr_t a = reinterpret_cast<uintptr_t>(out);
    c.tab = tab;
    c.row0 = reinterpret_cast<const uint8_t *>(a & ~(uintptr_t)127);
    c.m0 = (uint32_t)(a & 127);
    c.next = 0;
    c.acc = 0;
}

// word at row offset q: member bytes below lim (row coordinates), zero elsewhere, the first four message bytes complemented
__device__ __forceinline__ uint32_t crc_edge_word(const CrcCursor &c, uint32_t q, uint32_t lim)
{
    uint32_t w = 0;
    if (q >= c.m0 && q + 4u <= lim) w = ldg32(c.row0 + q);
    else
        for (uint32_t i = 0; i < 4; i++)
            if (q + i >= c.m0 && q + i < lim) w |= ldg8(c.row0 + q + i) << (8 * i);
    const int32_t rel = (int32_t)c.m0 - (int32_t)q;
    if (rel > -4 && rel < 4) w ^= rel >= 0 ? 0xffffffffu << (8 * rel) : 0xffffffffu >> (-8 * rel);
    return w;
}

// absorb rows [c.next, r_end); lim = end of the member's final bytes in row coordinates
__device__ __forceinline__ void crc_absorb(CrcCursor &c, uint32_t r_end, uint32_t lim)
{
    const uint32_t l4 = 4u * hgpu_lane();
    const uint32_t *tab = c.tab;
    uint32_t r = c.next, acc = c.acc;
    const uint32_t ie = min(r_end, lim >> 7);                  // rows wholly below lim
    for (; r < r_end && r < 2u; r++) acc = crc_step4(tab, acc ^ crc_edge_word(c, 128u * r + l4, lim));
    for (uint32_t r8 = r; r8 < ie; r8 += 8) {                  // interior rows: up to eight loads in flight, one round trip
        const uint8_t *p = c.row0 + 128u * r8 + l4;
        uint32_t w[8];
#pragma unroll
        for (uint32_t k = 0; k < 8; k++) w[k] = ld32_if(p + 128u * k, r8 + k < ie);
#pragma unroll
        for (uint32_t k = 0; k < 8; k++)
            if (r8 + k < ie) acc = crc_step4(tab, acc ^ w[k]);
    }
    r = max(r, ie);
    for (; r < r_end; r++) acc = crc_step4(tab, acc ^ crc_edge_word(c, 128u * r + l4, lim));
    c.acc = acc;
    c.next = r;
}

// the member's bytes [0, f) are final: absorb the whole rows among them.  Warp-uniform; the
// caller has made the bytes visible to the warp (__syncwarp).
__device__ __forceinline__ void crc_advance(CrcCursor &c, uint32_t f)
{
    const uint32_t lim = c.m0 + f;
    if ((lim >> 7) > c.next) crc_absorb(c, lim >> 7, lim);
}

// CRC-32 of the member's n bytes
__device__ uint32_t crc_finish(CrcCursor &c, uint32_t n)
{
    const uint32_t lim = c.m0 + n;
    const uint32_t rows = (max(lim, c.m0 + 4u) + 127u) >> 7;     // the complemented bytes may reach past the data
    crc_absorb(c, rows, lim);
    uint32_t s = multmodp(g_xinv_byte[4u * hgpu_lane()], c.acc);
#pragma unroll
    for (int d = 16; d; d >>= 1) s ^= __shfl_xor_sync(0xffffffffu, s, d);
    return ~multmodp(g_xinv_byte[128u * rows - lim], s);
}

// ---------------------------------------------------------------------------------------------
// LZ77 match execution.
//
// A match is never copied on its own: that would be one round trip to L2 per match for bytes
// this warp wrote a moment ago.  Matches are taken 32 at a time (one record per lane) and
// executed OUT OF ORDER inside the batch.  Destinations inside a batch are ascending and
// disjoint, so the earlier records a match reads from form one index range, found with two
// 5-step binary searches over the lanes (shuffles) and kept as a 32-bit dependency mask.  Then,
// in rounds, every record whose dependencies are done is executed.  The number of L2 round trips
// per batch is the depth of its dependency chain (1-4 for sorted BAM), not the number of matches.
//
// A round's ready matches that do not overlap their own source are laid end to end in one space
// of destination words (4-byte aligned words that hold at least one byte of the match; an
// exclusive scan of the per-match word counts), and the warp walks that space 32 words at a time:
// lane j finds its match by a 5-step search over the inclusive scan, funnel-shifts the word from
// the aligned source words in front of it (the upper one is usually the next lane's lower one)
// and stores it whole, or bytewise where the word is shared with a literal or another match.
// Lanes on one match touch the same one or two cache lines.  The loads of the next 32 words are
// issued before the current ones are first used (load_slot returns with its loads in flight), so a
// round costs about one L2 round trip however many chunks it has: nothing a round stores is read
// in that round.
// Overlapping matches (dist < len, run-length style) are rare and take a separate cooperative
// path with a per-byte modulo.
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t low_mask(uint32_t n) { return n >= 32u ? 0xffffffffu : (1u << n) - 1u; }

struct WordSlot {
    uint32_t d;               // destination word, from the aligned base
    uint32_t lo, hi;          // aligned source words (hi: 0 when the next lane's lo is meant)
    uint32_t f;               // [3:0] bytes of the word that belong to the match (0xf: all), [8:4] source shift,
                              // [9] the upper source word is the next lane's lower one
};

// word `slot` of the round's destination-word space.  inc: inclusive scan of the word counts;
// wb = (first word of the lane's match) - 4 * (words in front of it); u0 = its destination; ld = len | dist << 16
__device__ __forceinline__ WordSlot load_slot(const uint8_t *ob, uint32_t inc, uint32_t wb, uint32_t u0, uint32_t ld,
                                              uint32_t slot, uint32_t T)
{
    const uint32_t lane = hgpu_lane();
    uint32_t k = 0;                                            // owner: the number of matches ending at or before slot
#pragma unroll
    for (int st = 16; st >= 1; st >>= 1)
        if (__shfl_sync(0xffffffffu, inc, k + st - 1) <= slot) k += st;
    const uint32_t D = __shfl_sync(0xffffffffu, wb, k) + 4u * slot;
    const uint32_t a0 = __shfl_sync(0xffffffffu, u0, k), l_d = __shfl_sync(0xffffffffu, ld, k);
    const uint32_t kn = __shfl_down_sync(0xffffffffu, k, 1);
    const bool valid = slot < T;
    const uint32_t dist = l_d >> 16;
    const uint32_t a = max(D, a0), b = min(D + 4u, a0 + (l_d & 0xffffu));     // the match's bytes in this word
    const int32_t S = (int32_t)(D - dist), S0 = S & ~3, sh = (S & 3) * 8;      // S >= -3: the source starts at >= 0
    // only words that hold source bytes [a - dist, b - dist) are touched
    const bool from_next = lane < 31 && kn == k && slot + 1 < T;               // the next lane's lower word is this one's upper
    const bool need_lo = valid && S0 + 4 > (int32_t)(a - dist);
    const bool need_hi = valid && sh != 0 && S0 + 4 < (int32_t)(b - dist) && !from_next;
    WordSlot w;
    w.d = D;
    w.lo = ld32_if(ob + S0, need_lo);
    w.hi = ld32_if(ob + S0 + 4, need_hi);
    const uint32_t m = valid ? ((1u << (b - D)) - 1u) & ~((1u << (a - D)) - 1u) : 0u;
    w.f = m | (uint32_t)sh << 4 | (from_next ? 1u << 9 : 0u);
    return w;
}

// the first use of the loaded words: load_slot returns with its loads in flight
__device__ __forceinline__ void store_slot(uint8_t *ob, const WordSlot &w)
{
    const uint32_t lo_next = __shfl_down_sync(0xffffffffu, w.lo, 1);
    const uint32_t v = __funnelshift_r(w.lo, (w.f >> 9) ? lo_next : w.hi, (w.f >> 4) & 31u);
    const uint32_t m = w.f & 15u;
    const bool part = m != 15u;
    st32_if(ob + w.d, v, !part);
    st8_if(ob + w.d, v, part && (m & 1u));
    st8_if(ob + w.d + 1, v >> 8, part && (m & 2u));
    st8_if(ob + w.d + 2, v >> 16, part && (m & 4u));
    st8_if(ob + w.d + 3, v >> 24, part && (m & 8u));
}

__device__ __forceinline__ void exec_batch(uint8_t *out, uint2 rec, uint32_t nrec)
{
    const uint32_t lane = hgpu_lane();
    const bool have = lane < nrec;
    const uint32_t len = have ? (rec.y & 0xffffu) : 0u, dist = rec.y >> 16;
    const uint32_t dst = have ? rec.x : 0xffffffffu;            // padding lanes keep the arrays sorted
    const uint32_t dst_end = have ? dst + len : 0xffffffffu;
    const bool ov = dist < len;
    const uint32_t src = dst - dist, src_end = ov ? dst : src + len;
    uint32_t dep = 0;
    const uint32_t dst0 = __shfl_sync(0xffffffffu, dst, 0);
    if (__any_sync(0xffffffffu, have && src_end > dst0)) {
        uint32_t j1 = 0, j2 = 0;                                 // #records with dst_end <= src ; #records with dst < src_end
#pragma unroll
        for (int st = 16; st >= 1; st >>= 1) {
            uint32_t e = __shfl_sync(0xffffffffu, dst_end, j1 + st - 1);
            uint32_t d = __shfl_sync(0xffffffffu, dst, j2 + st - 1);
            if (e <= src) j1 += st;
            if (d < src_end) j2 += st;
        }
        if (have && j2 > j1) dep = low_mask(j2) & ~low_mask(j1) & hgpu_lanemask_lt();
    }
    // destination-word space, in coordinates of the 4-byte aligned base ob
    const uint32_t mis = (uint32_t)reinterpret_cast<uintptr_t>(out) & 3u;
    uint8_t *ob = out - mis;
    const uint32_t u0 = dst + mis;
    const uint32_t nw = have && !ov ? ((u0 + len + 3u) >> 2) - (u0 >> 2) : 0u;
    uint32_t done = low_mask(nrec) ^ 0xffffffffu;
#ifdef HGPU_PROFILE
    if (lane == 0) atomicAdd(&g_prof[9], 1ull);
#endif
    while (done != 0xffffffffu) {
        const bool ready = !((done >> lane) & 1u) && (dep & ~done) == 0u;
        const uint32_t R = __ballot_sync(0xffffffffu, ready);
        const uint32_t Rov = __ballot_sync(0xffffffffu, ready && ov);
#ifdef HGPU_PROFILE
        if (lane == 0) { atomicAdd(&g_prof[8], 1ull); atomicAdd(&g_prof[11], (unsigned long long)__popc(Rov)); }
#endif
        // every ready match that does not overlap its own source: coalesced word copies
        const uint32_t cnt = ready ? nw : 0u;
        uint32_t inc = cnt;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const uint32_t t = __shfl_up_sync(0xffffffffu, inc, d);
            if (lane >= (uint32_t)d) inc += t;
        }
        const uint32_t T = __shfl_sync(0xffffffffu, inc, 31);
        const uint32_t wb = (u0 & ~3u) - 4u * (inc - cnt);
        if (T) {
            WordSlot cur = load_slot(ob, inc, wb, u0, rec.y, lane, T);
            for (uint32_t base = 0; base < T; base += 32) {
                WordSlot nxt = {0u, 0u, 0u, 0u};
                if (base + 32 < T) nxt = load_slot(ob, inc, wb, u0, rec.y, base + 32 + lane, T);
                store_slot(ob, cur);
                cur = nxt;
            }
        }
        __syncwarp();
        // overlapping matches of this round: the source is the `dist` bytes before the
        // destination, repeated
        for (uint32_t m = Rov; m; m &= m - 1) {
            const int k = __ffs(m) - 1;
            const uint32_t d0 = __shfl_sync(0xffffffffu, dst, k), ln = __shfl_sync(0xffffffffu, len, k);
            const uint32_t di = __shfl_sync(0xffffffffu, dist, k);
            // i % di for i = lane, lane+32, ...: one division pair, then add-and-wrap.  The source bytes lie in
            // front of the destination and are never overwritten here, so loads and stores need no phases.
            const uint32_t stepm = 32u % di;
            uint32_t r = lane % di;
            for (uint32_t i = lane; i < ln; i += 32) {
                out[d0 + i] = out[d0 - di + r];
                r += stepm;
                if (r >= di) r -= di;
            }
        }
        __syncwarp();                               // next round reads what other lanes just stored
        done |= R;
    }
}

// ---------------------------------------------------------------------------------------------
// Serial ("uniform") body decoder: all lanes walk the same bit stream.  Used for small deflate
// blocks and as the fallback when speculation is not worthwhile.
// ---------------------------------------------------------------------------------------------
__device__ int decode_body_uniform(InflateSmem &s, Bits &b, uint8_t *out, uint32_t cap, uint32_t &o, CrcCursor &crc)
{
    const uint32_t lane = hgpu_lane();
    uint32_t pend = 0;                             // match records parked in s.rbuf
    for (;;) {
        bits_fill(b);
        uint32_t e = lookup<LIT_ROOT>(s.lit, b);
        uint32_t kind = (e >> 4) & 15;
        if (kind == K_LIT) {
            if (o >= cap) return HGPU_BGZF_ERR_SPACE;
            if (lane == 0) out[o] = (uint8_t)(e >> 16);
            o++;
            continue;
        }
        if (kind == K_EOB) break;
        if (kind != K_LEN) return HGPU_BGZF_ERR_ZLIB;
        uint32_t len = (e >> 16) + bits_get(b, (e >> 8) & 0xff);
        bits_fill(b);
        uint32_t d = lookup<DST_ROOT>(s.dst, b);
        if (((d >> 4) & 15) != K_DIST) return HGPU_BGZF_ERR_ZLIB;
        uint32_t dist = (d >> 16) + bits_get(b, (d >> 8) & 0xff);
        if (bits_overrun(b)) return HGPU_BGZF_ERR_ZLIB;
        if (dist > o) return HGPU_BGZF_ERR_ZLIB;
        if (o + len > cap) return HGPU_BGZF_ERR_SPACE;
        __syncwarp();
        if (lane == 0) s.rbuf[pend] = make_uint2(o, len | (dist << 16));
        o += len;
        if (++pend == 32) {
            __syncwarp();
            exec_batch(out, s.rbuf[lane], 32);
            pend = 0;
            crc_advance(crc, o);                           // literals are stored as they are decoded: all of [0, o) is final
        }
    }
    __syncwarp();
    if (pend) exec_batch(out, s.rbuf[lane], pend);
    __syncwarp();
    if (bits_overrun(b)) return HGPU_BGZF_ERR_ZLIB;
    return HGPU_OK;
}

// ---------------------------------------------------------------------------------------------
// Lane-parallel body decoder.
//
// The bit range of the deflate block body is cut into 32 equal sub-ranges.  Lane i decodes tokens
// from a guessed start (the cut itself) to the end of its sub-range; Huffman streams
// self-synchronise, so the position where lane i leaves its range is usually already the true
// token boundary.  Each round lane i+1 restarts from lane i's exit if that moved; lane 0 is exact,
// so after k rounds lanes 0..k are exact, and in practice two or three rounds settle all 32.
// Then output offsets follow from a prefix sum of per-lane byte counts, a last pass writes the
// literals and lists the matches, and the matches are executed in order through the window.
// ---------------------------------------------------------------------------------------------
struct LaneBits {
    const uint32_t *w;      // next word to prefetch
    uint64_t buf;
    uint32_t nxt;           // prefetched word
    int cnt;                // valid bits in buf
    int lim;                // (position < end)  <=>  (cnt > lim)
};

__device__ __forceinline__ void lb_init(LaneBits &b, const uint32_t *wbase, const uint32_t *wend, uint32_t start, uint32_t end)
{
    uint32_t wi = start >> 5, off = start & 31;
    const uint32_t *p = wbase + wi;
    uint32_t w0 = p < wend ? p[0] : 0;
    b.nxt = p + 1 < wend ? p[1] : 0;
    b.w = p + 2;
    b.buf = w0 >> off;
    b.cnt = 32 - (int)off;
    b.lim = (int)((wi + 1) * 32) - (int)end;
}
__device__ __forceinline__ void lb_fill(LaneBits &b, const uint32_t *wend)
{
    if (b.cnt <= 32) {
        b.buf |= (uint64_t)b.nxt << b.cnt;
        b.cnt += 32;
        b.lim += 32;
        b.nxt = b.w < wend ? (*b.w) : 0;
        b.w++;
    }
}
__device__ __forceinline__ uint32_t lb_pos(const LaneBits &b, uint32_t end) { return (uint32_t)(b.lim + (int)end - b.cnt); }

template <int ROOT>
__device__ __forceinline__ uint32_t lb_lookup(const uint32_t *table, LaneBits &b)
{
    uint32_t e = table[(uint32_t)b.buf & ((1u << ROOT) - 1)];
    if (((e >> 4) & 15) == K_SUB) {
        b.buf >>= ROOT; b.cnt -= ROOT;
        e = table[(e >> 16) + ((uint32_t)b.buf & ((1u << ((e >> 8) & 0xff)) - 1))];
    }
    b.buf >>= (e & 15); b.cnt -= (int)(e & 15);
    return e;
}

enum : uint32_t { ST_RUN = 0, ST_EOB = 1, ST_BAD = 2 };

// Decode tokens in [start, end).  EMIT=0: count output bytes / matches.  EMIT=1: write literals at
// out[obase..] and {dst, len | dist<<16} match records at mrec[mbase..]; sets bad_dist on a
// distance that reaches before the start of the output.
template <int EMIT>
__device__ __forceinline__ void lane_decode(const InflateSmem &s, const uint32_t *wbase, const uint32_t *wend,
                                            uint32_t start, uint32_t end, uint32_t &exitp, uint32_t &nout,
                                            uint32_t &nmatch, uint32_t &st, uint8_t *out, uint32_t obase,
                                            uint2 *mrec, uint32_t mbase, bool &bad_dist)
{
    LaneBits b;
    uint32_t n = 0, m = 0, status = ST_RUN;
    if (start >= end) { exitp = start; nout = 0; nmatch = 0; st = ST_RUN; return; }
    lb_init(b, wbase, wend, start, end);
    while (b.cnt > b.lim) {
        lb_fill(b, wend);
        uint32_t e = lb_lookup<LIT_ROOT>(s.lit, b);
        uint32_t kind = (e >> 4) & 15;
        if (kind == K_LIT) {
            if (EMIT) out[obase + n] = (uint8_t)(e >> 16);
            n++;
        } else if (kind == K_LEN) {
            uint32_t xb = (e >> 8) & 0xff;
            uint32_t len = (e >> 16) + ((uint32_t)b.buf & ((1u << xb) - 1));
            b.buf >>= xb; b.cnt -= (int)xb;
            lb_fill(b, wend);
            uint32_t d = lb_lookup<DST_ROOT>(s.dst, b);
            if (((d >> 4) & 15) != K_DIST) { status = ST_BAD; break; }
            uint32_t xd = (d >> 8) & 0xff;
            uint32_t dist = (d >> 16) + ((uint32_t)b.buf & ((1u << xd) - 1));
            b.buf >>= xd; b.cnt -= (int)xd;
            if (EMIT) {
                uint32_t dstpos = obase + n;
                if (dist > dstpos) bad_dist = true;
                mrec[mbase + m] = make_uint2(dstpos, len | (dist << 16));
            }
            n += len; m++;
        } else if (kind == K_EOB) { status = ST_EOB; break; }
        else { status = ST_BAD; break; }
    }
    exitp = lb_pos(b, end);
    nout = n; nmatch = m; st = status;
}

// Execute mrec[0..total) in order through the window.  Records are fetched 32 at a time
// (coalesced) and broadcast with shuffles, so every lane sees the same match.
// After a batch every byte in front of the next batch's first destination is final (literals were
// written by the emit pass, earlier matches are done): the CRC cursor takes it.
__device__ void run_matches(uint8_t *out, const uint2 *mrec, uint32_t total, CrcCursor &crc)
{
    const uint32_t lane = hgpu_lane();
    uint2 nx = lane < total ? mrec[lane] : make_uint2(0, 0);
    for (uint32_t base = 0; base < total; base += 32) {
        uint2 rec = nx;
        nx = base + 32 + lane < total ? mrec[base + 32 + lane] : make_uint2(0, 0);      // next batch in flight
        exec_batch(out, rec, total - base < 32u ? total - base : 32u);
        if (base + 32 < total) crc_advance(crc, __shfl_sync(0xffffffffu, nx.x, 0));
    }
    __syncwarp();
}

constexpr uint32_t PAR_MIN_BITS = 32 * 96;      // below this a deflate block is decoded serially
constexpr uint32_t MREC_CAP = 65536 / 3 + 64;   // a match yields >= 3 bytes of a <= 64 KiB member

// Parallel decode of one Huffman block body starting at bit `body` of the member (bit 0 = first
// bit of word wbase[0], i.e. positions include the alignment offset).  total = end of input.
__device__ int decode_body_parallel(InflateSmem &s, const uint32_t *wbase, const uint32_t *wend, uint32_t body,
                                    uint32_t total, uint8_t *out, uint32_t cap, uint32_t &o, uint2 *mrec,
                                    uint32_t &end_pos, CrcCursor &crc, Prof &pf, uint32_t mcap = MREC_CAP)
{
    const uint32_t lane = hgpu_lane();
    const uint32_t S = (total - body + 31) / 32;
    uint32_t start = body + lane * S;
    uint32_t end = lane == 31 ? total : min(total, body + (lane + 1) * S);
    if (start > total) start = total;
    uint32_t exitp = 0, n = 0, m = 0, st = ST_RUN;
    bool need = true, dummy = false;
    for (int round = 0; round < 34; round++) {
        if (need) lane_decode<0>(s, wbase, wend, start, end, exitp, n, m, st, nullptr, 0, nullptr, 0, dummy);
        uint32_t prev = __shfl_up_sync(0xffffffffu, exitp, 1);
        uint32_t ns = lane == 0 ? start : prev;
        need = ns != start;
        start = ns;
        if (!__any_sync(0xffffffffu, need)) break;
    }
    pf.mark(1);
    // the chain is now consistent: lane i starts where lane i-1 stopped
    uint32_t eob = __ballot_sync(0xffffffffu, st == ST_EOB);
    uint32_t bad = __ballot_sync(0xffffffffu, st == ST_BAD);
    if (!eob) return HGPU_BGZF_ERR_ZLIB;                       // input ends without an end-of-block code
    uint32_t E = __ffs(eob) - 1;
    if (bad & ((2u << E) - 1u)) return HGPU_BGZF_ERR_ZLIB;     // invalid code at or before the end of block
    uint32_t last = __shfl_sync(0xffffffffu, exitp, E);
    if (last > total) return HGPU_BGZF_ERR_ZLIB;               // the block ran past the input
    if (lane > E) { n = 0; m = 0; }
    // exclusive prefix sums of bytes and matches
    uint32_t on = n, mn = m;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        uint32_t a = __shfl_up_sync(0xffffffffu, on, d), c = __shfl_up_sync(0xffffffffu, mn, d);
        if (lane >= (uint32_t)d) { on += a; mn += c; }
    }
    uint32_t tot_out = __shfl_sync(0xffffffffu, on, 31), tot_m = __shfl_sync(0xffffffffu, mn, 31);
    if ((uint64_t)o + tot_out > cap) return HGPU_BGZF_ERR_SPACE;
    if (tot_m > mcap) return HGPU_BGZF_ERR_ZLIB;           // impossible within 64 KiB of output
    bool bad_dist = false;
    if (lane <= E) {
        uint32_t e2, n2, m2, st2;
        lane_decode<1>(s, wbase, wend, start, end, e2, n2, m2, st2, out, o + on - n, mrec, mn - m, bad_dist);
    }
    if (__any_sync(0xffffffffu, bad_dist)) return HGPU_BGZF_ERR_ZLIB;   // distance too far back
    __syncwarp();
    __threadfence_block();
    pf.mark(2);
    run_matches(out, mrec, tot_m, crc);
    pf.mark(3);
    o += tot_out;
    end_pos = last;
    return HGPU_OK;
}

// ---------------------------------------------------------------------------------------------
// One BGZF member: headers + table construction are warp-uniform, bodies go to the lane-parallel
// decoder or, below PAR_MIN_BITS, to the uniform one.
// ---------------------------------------------------------------------------------------------
__device__ int inflate_member(InflateSmem &s, const uint8_t *src, uint32_t slen, uint8_t *out, uint32_t cap,
                              uint32_t &olen, uint2 *mrec, CrcCursor &crc, Prof &pf, uint32_t mcap = MREC_CAP)
{
    const uint32_t lane = hgpu_lane();
    Bits b;
    bits_init(b, src, 0, slen);
    const uintptr_t a0 = reinterpret_cast<uintptr_t>(src);
    const uint32_t mis_bits = (uint32_t)(a0 & 3) * 8;
    const uint32_t *wbase = reinterpret_cast<const uint32_t *>(a0 - (a0 & 3));
    const uint32_t *wend = reinterpret_cast<const uint32_t *>((a0 + slen + 3) & ~(uintptr_t)3);
    const uint32_t total = mis_bits + slen * 8;                // end of input in wbase bit coordinates
    uint32_t o = 0;
    for (;;) {
        bits_fill(b);
        uint32_t final = bits_get(b, 1), type = bits_get(b, 2);
        if (type == 0) {                                       // stored
            bits_drop(b, b.cnt & 7);
            bits_fill(b);
            uint32_t len = bits_get(b, 16);
            bits_fill(b);
            uint32_t nlen = bits_get(b, 16);
            if (bits_overrun(b)) return HGPU_BGZF_ERR_ZLIB;
            if ((len ^ 0xffffu) != nlen) return HGPU_BGZF_ERR_ZLIB;
            uint32_t pos = bits_pos(b) >> 3;
            if ((uint64_t)pos + len > slen) return HGPU_BGZF_ERR_ZLIB;
            if (o + len > cap) return HGPU_BGZF_ERR_SPACE;
            for (uint32_t i = lane; i < len; i += 32) out[o + i] = src[pos + i];
            o += len;
            bits_init(b, src, pos + len, slen);
            __syncwarp();
            crc_advance(crc, o);
        } else if (type == 1 || type == 2) {
            int rc;
            if (type == 1) {
                __syncwarp();
                for (int i = lane; i < 288; i += 32) s.lens[i] = i < 144 ? 8 : i < 256 ? 9 : i < 280 ? 7 : 8;
                __syncwarp();
                rc = build_table<LIT_ROOT, LIT_TABLE>(s, s.lit, 288, false, lit_entry);
                if (rc) return HGPU_BGZF_ERR_ZLIB;
                __syncwarp();
                for (int i = lane; i < 32; i += 32) s.lens[i] = 5;
                __syncwarp();
                rc = build_table<DST_ROOT, DST_TABLE>(s, s.dst, 32, false, dst_entry);
                if (rc) return HGPU_BGZF_ERR_ZLIB;
            } else {
                bits_fill(b);
                uint32_t hlit = bits_get(b, 5) + 257, hdist = bits_get(b, 5) + 1, hclen = bits_get(b, 4) + 4;
                if (hlit > 286 || hdist > 30) return HGPU_BGZF_ERR_ZLIB;
                __syncwarp();
                if (lane < 19) s.lens[lane] = 0;
                __syncwarp();
                for (uint32_t i = 0; i < hclen; i++) {
                    bits_fill(b);
                    uint32_t v = bits_get(b, 3);
                    if (lane == 0) s.lens[c_cl_order[i]] = (uint8_t)v;
                }
                if (bits_overrun(b)) return HGPU_BGZF_ERR_ZLIB;
                __syncwarp();
                rc = build_table<7, CL_TABLE>(s, s.cl, 19, false, cl_entry);
                if (rc) return HGPU_BGZF_ERR_ZLIB;
                uint32_t nsym = hlit + hdist, i = 0, prev = 0;
                while (i < nsym) {
                    bits_fill(b);
                    uint32_t e = s.cl[bits_peek(b, 7)];
                    if (((e >> 4) & 15) != K_LIT) return HGPU_BGZF_ERR_ZLIB;
                    bits_drop(b, e & 15);
                    uint32_t sym = e >> 16;
                    if (sym < 16) {
                        if (lane == 0) s.code[i] = (uint16_t)sym;
                        prev = sym; i++;
                    } else {
                        uint32_t rep, val = 0;
                        if (sym == 16) { if (i == 0) return HGPU_BGZF_ERR_ZLIB; val = prev; rep = 3 + bits_get(b, 2); }
                        else if (sym == 17) rep = 3 + bits_get(b, 3);
                        else rep = 11 + bits_get(b, 7);
                        if (i + rep > nsym) return HGPU_BGZF_ERR_ZLIB;
                        for (uint32_t k = lane; k < rep; k += 32) s.code[i + k] = (uint16_t)val;
                        i += rep;
                        prev = val;
                    }
                    if (bits_overrun(b)) return HGPU_BGZF_ERR_ZLIB;
                }
                __syncwarp();
                if (s.code[256] == 0) return HGPU_BGZF_ERR_ZLIB;         // no end-of-block code
                uint32_t dl = lane < hdist ? s.code[hlit + lane] : 0;
                uint32_t ll[9];
#pragma unroll
                for (int k = 0; k < 9; k++) { uint32_t j = lane + 32 * k; ll[k] = j < hlit ? s.code[j] : 0; }
                __syncwarp();
#pragma unroll
                for (int k = 0; k < 9; k++) { uint32_t j = lane + 32 * k; if (j < 288) s.lens[j] = (uint8_t)ll[k]; }
                __syncwarp();
                rc = build_table<LIT_ROOT, LIT_TABLE>(s, s.lit, (int)hlit, true, lit_entry);
                if (rc) return HGPU_BGZF_ERR_ZLIB;
                __syncwarp();
                s.lens[lane] = (uint8_t)dl;
                __syncwarp();
                rc = build_table<DST_ROOT, DST_TABLE>(s, s.dst, (int)hdist, true, dst_entry);
                if (rc) return HGPU_BGZF_ERR_ZLIB;
            }
            __syncwarp();
            // position of the first body bit, in wbase coordinates
            if (bits_overrun(b)) return HGPU_BGZF_ERR_ZLIB;
            uint32_t body = mis_bits + bits_pos(b);
            pf.mark(0);
            if (total - body >= PAR_MIN_BITS) {
                uint32_t end_pos = 0;
                rc = decode_body_parallel(s, wbase, wend, body, total, out, cap, o, mrec, end_pos, crc, pf, mcap);
                if (rc) return rc;
                // continue the uniform reader right after the end-of-block code
                uint32_t byte = (end_pos - mis_bits) >> 3, bit = (end_pos - mis_bits) & 7;
                bits_init(b, src, byte, slen);
                bits_fill(b);
                bits_drop(b, bit);
            } else {
                rc = decode_body_uniform(s, b, out, cap, o, crc);
                if (rc) return rc;
                pf.mark(5);
            }
            crc_advance(crc, o);
        } else
            return HGPU_BGZF_ERR_ZLIB;
        if (final) break;
    }
    olen = o;
    return HGPU_OK;
}

__device__ int check_header(const uint8_t *h)
{
    if (h[0] != 31 || h[1] != 139 || h[2] != 8) return -2;
    return ((h[3] & 4) && (h[10] | h[11] << 8) == 6 && h[12] == 'B' && h[13] == 'C' && (h[14] | h[15] << 8) == 2) ? 0 : -1;
}

#ifndef HGPU_INFLATE_WARPS
#define HGPU_INFLATE_WARPS 7
#endif
constexpr int INFLATE_WARPS = HGPU_INFLATE_WARPS;      // warps per CTA; they share only the CRC tables (7 x 10 KB + 4 KB per CTA: three CTAs = 21 warps per SM, 80 registers;
                                                       // measured 16 -> 20 -> 21 -> 22 warps/SM: 214 / 229 / 232 / 233 GB/s, shared memory caps it at 22)

#ifndef INFL_LB
#define INFL_LB 3
#endif
__global__ void __launch_bounds__(32 * INFLATE_WARPS, INFL_LB)
bgzf_inflate_kernel(const uint8_t *__restrict__ in, const uint64_t *__restrict__ in_off,
                    const uint32_t *__restrict__ in_len, uint32_t n, uint8_t *out,
                    const uint64_t *__restrict__ out_off, const uint32_t *__restrict__ out_cap,
                    uint32_t *out_len, int32_t *status, uint32_t *counter, uint2 *mrec_all)
{
    extern __shared__ __align__(16) uint8_t dyn_smem[];
    uint32_t *crc_tab = reinterpret_cast<uint32_t *>(dyn_smem);       // g_crc_tab2: the CRC cursor's row step
    InflateSmem *smem_all = reinterpret_cast<InflateSmem *>(dyn_smem + 4096);
    for (int i = threadIdx.x; i < 1024; i += blockDim.x) crc_tab[i] = (&g_crc_tab2[0][0])[i];
    __syncthreads();                                   // the only block-wide barrier: warps are independent below
    InflateSmem &s = smem_all[threadIdx.x >> 5];
    uint2 *mrec = mrec_all + ((size_t)blockIdx.x * INFLATE_WARPS + (threadIdx.x >> 5)) * MREC_CAP;
    const uint32_t lane = hgpu_lane();
    for (;;) {
        uint32_t job = 0;
        if (lane == 0) job = atomicAdd(counter, 1u);
        job = __shfl_sync(0xffffffffu, job, 0);
        if (job >= n) break;
        const uint8_t *blk = in + in_off[job];
        uint32_t blen = in_len[job];
        uint8_t *dst = out + out_off[job];
        uint32_t cap = out_cap[job];
        if (cap > 65536u) cap = 65536u;                    // BGZF_MAX_BLOCK_SIZE, bgzf.c:810
        int rc = HGPU_OK;
        uint32_t got = 0;
        if (blen < 26 || check_header(blk) != 0 || (uint32_t)(blk[16] | blk[17] << 8) + 1u != blen)
            rc = HGPU_BGZF_ERR_HEADER;
        else {
            // inflate_block hands zlib block_length-18 bytes: deflate data plus the 8-byte footer
            Prof pf;
            pf.start();
            CrcCursor cc;
            crc_begin(cc, crc_tab, dst);
            rc = inflate_member(s, blk + 18, blen - 18, dst, cap, got, mrec, cc, pf);
            if (rc == HGPU_OK) {
                uint32_t want = blk[blen - 8] | blk[blen - 7] << 8 | blk[blen - 6] << 16 | (uint32_t)blk[blen - 5] << 24;
                pf.mark(6);
                uint32_t crc = crc_finish(cc, got);
                if (crc != want) rc = HGPU_BGZF_ERR_CRC;
                pf.mark(4);
            }
        }
        __syncwarp();
        if (lane == 0) { status[job] = rc; out_len[job] = rc == HGPU_OK ? got : 0; }
    }
}


// ---------------------------------------------------------------------------------------------
// Plain gzip members of any size — zlib_mem_inflate as cram_uncompress_block uses it for GZIP blocks
// (cram/cram_io.c:1068-1157, :1600-1616): RFC 1952 header (FEXTRA / FNAME / FCOMMENT / FHCRC skipped), raw
// DEFLATE through the same member decoder as a BGZF block, CRC-32 and ISIZE from the trailer.  One warp per
// member.  Limits: a single deflate block with more than GZ_MREC matches is refused (ERR_ZLIB -> the caller's host
// library); CRAM writes its GZIP blocks with memLevel 9 (cram_io.c zlib_mem_deflate): at most 32 767 symbols per block.
// ---------------------------------------------------------------------------------------------
constexpr uint32_t GZ_MREC = 32768 + 64;

__device__ int gzip_header_len(const uint8_t *h, uint32_t n)
{
    if (n < 18 || h[0] != 31 || h[1] != 139 || h[2] != 8 || (h[3] & 0xe0)) return -1;
    const uint32_t flg = h[3];
    uint32_t p = 10;
    if (flg & 4) { if (p + 2 > n) return -1; p += 2u + (h[p] | h[p + 1] << 8); }
    if (flg & 8) { while (p < n && h[p]) p++; p++; }
    if (flg & 16) { while (p < n && h[p]) p++; p++; }
    if (flg & 2) p += 2;
    return p + 8 <= n ? (int)p : -1;
}

__global__ void __launch_bounds__(32 * INFLATE_WARPS, INFL_LB)
gzip_inflate_kernel(const uint8_t *__restrict__ in, const uint64_t *__restrict__ in_off,
                    const uint32_t *__restrict__ in_len, uint32_t n, uint8_t *out,
                    const uint64_t *__restrict__ out_off, const uint32_t *__restrict__ out_cap,
                    uint32_t *out_len, int32_t *status, uint32_t *counter, uint2 *mrec_all)
{
    extern __shared__ __align__(16) uint8_t dyn_smem[];
    uint32_t *crc_tab = reinterpret_cast<uint32_t *>(dyn_smem);       // g_crc_tab2: the CRC cursor's row step
    InflateSmem *smem_all = reinterpret_cast<InflateSmem *>(dyn_smem + 4096);
    for (int i = threadIdx.x; i < 1024; i += blockDim.x) crc_tab[i] = (&g_crc_tab2[0][0])[i];
    __syncthreads();
    InflateSmem &s = smem_all[threadIdx.x >> 5];
    uint2 *mrec = mrec_all + ((size_t)blockIdx.x * INFLATE_WARPS + (threadIdx.x >> 5)) * GZ_MREC;
    const uint32_t lane = hgpu_lane();
    for (;;) {
        uint32_t job = 0;
        if (lane == 0) job = atomicAdd(counter, 1u);
        job = __shfl_sync(0xffffffffu, job, 0);
        if (job >= n) break;
        const uint8_t *blk = in + in_off[job];
        const uint32_t blen = in_len[job];
        uint8_t *dst = out + out_off[job];
        const uint32_t cap = out_cap[job];
        int rc = HGPU_OK;
        uint32_t got = 0;
        const int hl = gzip_header_len(blk, blen);
        if (hl < 0) rc = HGPU_BGZF_ERR_HEADER;
        else {
            Prof pf;
            pf.start();
            CrcCursor cc;
            crc_begin(cc, crc_tab, dst);
            rc = inflate_member(s, blk + hl, blen - (uint32_t)hl, dst, cap, got, mrec, cc, pf, GZ_MREC);
            if (rc == HGPU_OK) {
                const uint8_t *f = blk + blen - 8;
                const uint32_t want = f[0] | f[1] << 8 | f[2] << 16 | (uint32_t)f[3] << 24;
                const uint32_t isize = f[4] | f[5] << 8 | f[6] << 16 | (uint32_t)f[7] << 24;
                const uint32_t crc = crc_finish(cc, got);
                if (crc != want || isize != got) rc = HGPU_BGZF_ERR_CRC;
            }
        }
        __syncwarp();
        if (lane == 0) { status[job] = rc; out_len[job] = rc == HGPU_OK ? got : 0; }
    }
}

__global__ void crc32_chunks_kernel(const uint8_t *buf, size_t len, size_t chunk, uint32_t *partial)
{
    // one warp per chunk
    size_t w = (size_t)blockIdx.x;
    size_t beg = w * chunk;
    if (beg >= len) return;
    size_t n = len - beg < chunk ? len - beg : chunk;
    uint32_t crc = warp_crc32(g_crc_tab, buf + beg, (uint32_t)n);
    if (hgpu_lane() == 0) partial[w] = crc;
}

// one warp per buffer: CRC-32 of n independent byte ranges (CRAM block header+payload, cram_io.c:1428-1433, :1585)
__global__ void crc32_batch_kernel(const uint8_t *buf, const uint64_t *off, const uint32_t *len, uint32_t n, uint32_t *crc_out)
{
    const uint32_t i = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (i >= n) return;
    uint32_t crc = warp_crc32(g_crc_tab, buf + off[i], len[i]);
    if (hgpu_lane() == 0) crc_out[i] = crc;
}

bool g_crc_ready[64];

int ensure_crc_tables(hgpu_ctx *ctx, cudaStream_t st)
{
    if (g_crc_ready[ctx->device & 63]) return HGPU_OK;
    crc_init_kernel<<<1, 256, 0, st>>>();
    crc_init2_kernel<<<1, 256, 0, st>>>();
    hgpu_count_launch();
    if (hgpu_check(cudaGetLastError(), "crc init")) return HGPU_ERR_CUDA;
    if (hgpu_check(cudaStreamSynchronize(st), "crc init sync")) return HGPU_ERR_CUDA;   // once per device
    g_crc_ready[ctx->device & 63] = true;
    return HGPU_OK;
}


// =============================================================================================
// BGZF block COMPRESS — stands where bgzf_compress / deflate_block / bgzf_encode_func stand
// (bgzf.c:624-683, :709, :1330): one warp per <= 0xff00-byte payload, output = a complete BGZF
// block (18-byte header, raw DEFLATE, CRC32, ISIZE).  Compressed bytes need not match zlib's
// (SURVEY.md §8c).  tests/test_gpu_bgzf_compress.py pins that every decoder inflates them back and
// the size ratio to zlib; tests/test_gpu_bgzf_deflate.py pins every block's code construction byte
// for byte against a restatement of pass 2, and the parse and code lengths against plain references.
// A negative level is level 6 (the host entry point maps it).
//
// level 0 or n < 16: stored block, exactly what htslib writes at level 0 (bgzf.c:573-580).
// level >= 1, pass 1 (LZ77): 32 positions per step, one per lane.  Each lane with 4 bytes left
//            hashes them (12-bit hash, 16-bit positions in shared memory; every lane reads before
//            any lane of the step stores), verifies and extends the candidate (>= 4 bytes), and
//            extends the distance-1 candidate (>= 3 bytes, runs), keeping the longer.  Matches stop
//            at n and at 258 bytes.  A greedy in-order walk over the step keeps non-overlapping
//            matches (ballot + ffs over literal stretches); at level >= 4 a match gives way to a
//            match at the next byte that is longer by 2 or more (one step of lazy evaluation).
// pass 2 (codes): token histogram with EOB; lit/len, distance and code-length code lengths by
//            Huffman on sorted leaves, folded to 15 / 15 / 7 bits (build_lengths); the code-length
//            sequence run-length coded with 16 / 17 / 18.  The exact bit counts of the fixed and
//            the dynamic block pick the smaller (fixed on a tie); each lane turns a token into a
//            code of up to 48 bits and ORs it into the slot at its prefix-summed bit offset.
//            A stored block replaces the result when the token bits would pass the slot's end or
//            the result is not smaller than a stored block (the zlib arm does the same,
//            bgzf.c:653-667).
// =============================================================================================
constexpr uint32_t DEFL_HASH_BITS = 12;
constexpr uint32_t DEFL_MAX_IN = 0xff00 + 256;      // htslib never exceeds 0xff00; allow the full 64 KiB - 280
constexpr uint32_t DEFL_TOK_CAP = 65536;

// pass 1 uses the hash table; pass 2 (dynamic Huffman) reuses the same bytes for histograms, code tables and the
// code-length sequence
struct DeflateDyn {
    uint32_t freq[288 + 32];          // lit/len then distance counts; reused as sort keys
    uint16_t code_ll[288], code_d[32];
    uint8_t  len_ll[288], len_d[32];
    uint16_t order[288];              // symbols sorted by count
    uint8_t  cl_sym[320], cl_ext[320];  // code-length alphabet symbols and their extra-bit values
    uint32_t cl_freq[19];
    uint16_t cl_code[19];
    uint8_t  cl_len[19];
    uint32_t n_cl;
    uint32_t w[576];                  // build_lengths work space: node weights, parents, depths
    uint16_t par[576];
    uint8_t  depth[576];
};
union DeflateSmem {
    uint16_t htab[1u << DEFL_HASH_BITS];
    DeflateDyn d;
};
static_assert(sizeof(DeflateDyn) <= (sizeof(uint16_t) << DEFL_HASH_BITS), "pass-2 tables fit the hash table's bytes");

__device__ __forceinline__ uint32_t fixed_lit_code(uint32_t sym, uint32_t &nbits)
{
    // RFC 1951 3.2.6, codes are sent MSB first -> bit-reverse for the LSB-first stream
    uint32_t code;
    if (sym < 144) { code = 0x30 + sym; nbits = 8; }
    else if (sym < 256) { code = 0x190 + (sym - 144); nbits = 9; }
    else if (sym < 280) { code = sym - 256; nbits = 7; }
    else { code = 0xc0 + (sym - 280); nbits = 8; }
    return __brev(code) >> (32 - nbits);
}

// token -> (bits, nbits), fixed Huffman
__device__ __forceinline__ uint32_t token_bits(uint32_t tok, uint32_t &nbits)
{
    if (!(tok >> 31)) return fixed_lit_code(tok & 0xff, nbits);
    uint32_t len = (tok & 0xff) + 3, dist = ((tok >> 8) & 0x7fff) + 1;
    // length symbol
    uint32_t ls = 28;
    while (ls > 0 && c_len_base[ls] > len) ls--;
    uint32_t lx = c_len_xtra[ls], n1;
    uint32_t bits = fixed_lit_code(257 + ls, n1);
    bits |= (len - c_len_base[ls]) << n1; n1 += lx;
    // distance symbol: 5-bit fixed code, MSB first
    uint32_t ds = 29;
    while (ds > 0 && c_dst_base[ds] > dist) ds--;
    uint32_t dx = c_dst_xtra[ds];
    bits |= (__brev(ds) >> 27) << n1; n1 += 5;
    bits |= (dist - c_dst_base[ds]) << n1; n1 += dx;
    nbits = n1;
    return bits;
}

// ---- dynamic Huffman (RFC 1951 3.2.7): code lengths from the token histogram ----
__device__ __forceinline__ uint32_t len_symbol(uint32_t len) { uint32_t ls = 28; while (ls > 0 && c_len_base[ls] > len) ls--; return ls; }
__device__ __forceinline__ uint32_t dist_symbol(uint32_t dist) { uint32_t ds = 29; while (ds > 0 && c_dst_base[ds] > dist) ds--; return ds; }

// One thread: optimal prefix-code lengths for n symbols with counts freq[] (0 = unused), limited to max_bits, into len[].
// order[] is scratch.  Sorted leaves + the two-queue merge give the depths (Huffman's algorithm without a heap); lengths over
// the limit are folded back by moving codes between length classes until the Kraft sum is exact.  A lone used symbol gets
// length 1 (inflaters accept the incomplete one-code set).
__device__ void build_lengths(const uint32_t *freq, int n, int max_bits, uint8_t *len, uint16_t *order, uint32_t *w, uint16_t *par, uint8_t *depth)
{
    int used = 0;
    for (int i = 0; i < n; i++) { len[i] = 0; if (freq[i]) order[used++] = (uint16_t)i; }
    if (used == 0) return;
    if (used == 1) { len[order[0]] = 1; return; }
    // insertion sort by count (ties by symbol): used <= 286
    for (int i = 1; i < used; i++) {
        const uint16_t v = order[i];
        const uint32_t fv = freq[v];
        int j = i - 1;
        while (j >= 0 && (freq[order[j]] > fv)) { order[j + 1] = order[j]; j--; }
        order[j + 1] = v;
    }
    // two-queue Huffman on the sorted leaves: node weights in w[], parent links in par[] (local arrays, 2*286 entries)
    for (int i = 0; i < used; i++) w[i] = freq[order[i]];
    int leaf = 0, inode = used, next = used;            // leaf queue [leaf, used), internal queue [inode, next)
    for (int k = 0; k < used - 1; k++) {
        int a, b;
        if (leaf < used && (inode >= next || w[leaf] <= w[inode])) a = leaf++; else a = inode++;
        if (leaf < used && (inode >= next || w[leaf] <= w[inode])) b = leaf++; else b = inode++;
        w[next] = w[a] + w[b];
        par[a] = par[b] = (uint16_t)next;
        next++;
    }
    const int root = next - 1;
    depth[root] = 0;
    for (int i = root - 1; i >= 0; i--) depth[i] = (uint8_t)(depth[par[i]] + 1);
    // length classes, folded to max_bits
    int cnt[32];
    for (int i = 0; i < 32; i++) cnt[i] = 0;
    for (int i = 0; i < used; i++) cnt[depth[i] > max_bits ? max_bits : depth[i]]++;
    uint32_t total = 0;
    for (int i = 1; i <= max_bits; i++) total += (uint32_t)cnt[i] << (max_bits - i);
    while (total > (1u << max_bits)) {                    // over-subscribed: lengthen the shallowest code that can give way
        cnt[max_bits]--;
        for (int i = max_bits - 1; i > 0; i--) if (cnt[i]) { cnt[i]--; cnt[i + 1] += 2; break; }
        total--;
    }
    // the most frequent symbols get the shortest lengths: walk the sorted order from the back
    int idx = used - 1;
    for (int l = 1; l <= max_bits; l++)
        for (int c = 0; c < cnt[l]; c++) len[order[idx--]] = (uint8_t)l;
}

// canonical codes (RFC 1951 3.2.2), bit-reversed for the LSB-first stream
__device__ void assign_codes(const uint8_t *len, int n, int max_bits, uint16_t *code)
{
    uint32_t bl_count[16], next_code[16];
    for (int i = 0; i < 16; i++) bl_count[i] = 0;
    for (int i = 0; i < n; i++) bl_count[len[i]]++;
    bl_count[0] = 0;
    uint32_t c = 0;
    for (int b = 1; b <= max_bits; b++) { c = (c + bl_count[b - 1]) << 1; next_code[b] = c; }
    for (int i = 0; i < n; i++) if (len[i]) code[i] = (uint16_t)(__brev(next_code[len[i]]++) >> (32 - len[i]));
}

// token -> (bits, nbits <= 48) with the block's own codes
__device__ __forceinline__ uint64_t token_bits_dyn(const DeflateDyn &d, uint32_t tok, uint32_t &nbits)
{
    if (!(tok >> 31)) { const uint32_t sym = tok & 0xff; nbits = d.len_ll[sym]; return d.code_ll[sym]; }
    const uint32_t len = (tok & 0xff) + 3, dist = ((tok >> 8) & 0x7fff) + 1;
    const uint32_t ls = len_symbol(len), ds = dist_symbol(dist);
    uint64_t bits = d.code_ll[257 + ls];
    uint32_t n1 = d.len_ll[257 + ls];
    bits |= (uint64_t)(len - c_len_base[ls]) << n1; n1 += c_len_xtra[ls];
    bits |= (uint64_t)d.code_d[ds] << n1; n1 += d.len_d[ds];
    bits |= (uint64_t)(dist - c_dst_base[ds]) << n1; n1 += c_dst_xtra[ds];
    nbits = n1;
    return bits;
}

__device__ __forceinline__ uint32_t ld4(const uint8_t *p) { return p[0] | (uint32_t)p[1] << 8 | (uint32_t)p[2] << 16 | (uint32_t)p[3] << 24; }

// Returns the BGZF block length written to out (<= 65536), 0 on failure.
__device__ uint32_t deflate_block_warp(DeflateSmem &s, const uint32_t (*crc_tab)[256], const uint8_t *in, uint32_t n,
                                       int level, uint8_t *out, uint32_t *toks)
{
    const uint32_t lane = hgpu_lane();
    if (n > 65280u) return 0;
    const uint32_t crc = warp_crc32(crc_tab, in, n);
    uint32_t dlen = 0;                                   // deflate payload bytes
    bool stored = level == 0 || n < 16;
    if (!stored) {
        // ---- pass 1: LZ77 tokens ----
        __syncwarp();
        for (uint32_t i = lane; i < (1u << DEFL_HASH_BITS); i += 32) s.htab[i] = 0;
        __syncwarp();
        uint32_t ntok = 0, covered = 0;
        for (uint32_t base = 0; base < n; base += 32) {
            const uint32_t p = base + lane;
            uint32_t mlen = 0, mdist = 0;
            const bool can = p + 4 <= n;
            uint32_t cand = 0, h = 0;
            if (can) { h = (ld4(in + p) * 2654435761u) >> (32 - DEFL_HASH_BITS); cand = s.htab[h]; }
            __syncwarp();
            if (can) s.htab[h] = (uint16_t)(p + 1);
            __syncwarp();
            if (can && p >= covered) {
                const uint32_t maxl = n - p < 258u ? n - p : 258u;
                // candidate from the hash table
                if (cand && p + 1 - cand <= 32768u) {
                    const uint8_t *a = in + (cand - 1), *b = in + p;
                    uint32_t l = 0;
                    while (l < maxl && a[l] == b[l]) l++;
                    if (l >= 4) { mlen = l; mdist = p + 1 - cand; }
                }
                // distance-1 candidate (runs)
                if (p >= 1) {
                    const uint8_t *b = in + p, *a1 = in + p - 1;
                    uint32_t l = 0;
                    while (l < maxl && a1[l] == b[l]) l++;
                    if (l >= 3 && l > mlen) { mlen = l; mdist = 1; }
                }
            }
            // greedy in-order selection inside the chunk
            uint32_t cur = covered > base ? covered : base;
            const uint32_t cend = base + 32 < n ? base + 32 : n;
            uint32_t has = __ballot_sync(0xffffffffu, mlen != 0);
            while (cur < cend) {
                uint32_t rel = cur - base;
                uint32_t later = has & ~((1u << rel) - 1u);
                uint32_t nm = later ? (uint32_t)(__ffs(later) - 1) : 32u;       // first match at/after cur
                uint32_t lit_end = base + nm < cend ? base + nm : cend;
                // literals [cur, lit_end)
                uint32_t nl = lit_end - cur;
                if (nl) {
                    if (p >= cur && p < lit_end && ntok + (p - cur) < DEFL_TOK_CAP) toks[ntok + (p - cur)] = in[p];
                    ntok += nl;
                    cur = lit_end;
                }
                if (nm < 32 && base + nm < cend) {
                    uint32_t ml = __shfl_sync(0xffffffffu, mlen, nm), md = __shfl_sync(0xffffffffu, mdist, nm);
                    // lazy evaluation (deflate.c's deflate_slow, one step): a strictly longer match starting at the next byte
                    // wins; this byte goes out as a literal
                    if (level >= 4 && nm < 31 && base + nm + 1 < cend) {
                        const uint32_t ml1 = __shfl_sync(0xffffffffu, mlen, (nm + 1) & 31);
                        if (ml1 > ml + 1) { has &= ~(1u << nm); continue; }
                    }
                    if (lane == 0 && ntok < DEFL_TOK_CAP) toks[ntok] = 0x80000000u | (ml - 3) | ((md - 1) << 8);
                    ntok++;
                    cur = base + nm + ml;
                }
            }
            covered = cur;
        }
        __syncwarp();
        __threadfence_block();
        // ---- pass 2: code construction + bits ----
        // the hash table is dead: its bytes now hold the histograms and code tables (DeflateDyn)
        DeflateDyn &d = s.d;
        bool overflow = ntok > DEFL_TOK_CAP;
        for (uint32_t i = lane; i < 320; i += 32) d.freq[i] = 0;
        __syncwarp();
        uint32_t xbits = 0;                                   // extra bits of all matches (the same under any code)
        for (uint32_t t = lane; t < ntok && !overflow; t += 32) {
            const uint32_t tok = toks[t];
            if (!(tok >> 31)) atomicAdd(&d.freq[tok & 0xff], 1u);
            else {
                const uint32_t ls = len_symbol((tok & 0xff) + 3), ds = dist_symbol(((tok >> 8) & 0x7fff) + 1);
                atomicAdd(&d.freq[257 + ls], 1u);
                atomicAdd(&d.freq[288 + ds], 1u);
                xbits += c_len_xtra[ls] + c_dst_xtra[ds];
            }
        }
        for (int dd = 16; dd > 0; dd >>= 1) xbits += __shfl_xor_sync(0xffffffffu, xbits, dd);
        __syncwarp();
        uint32_t use_dyn = 0, hlit = 257, hdist = 1, hclen = 4;
        if (lane == 0 && !overflow) {
            d.freq[256] = 1;                                  // end of block
            uint64_t fixed_bits = 3 + xbits, dyn_bits = 3 + 14 + xbits;
            for (int i = 0; i < 288; i++) fixed_bits += (uint64_t)d.freq[i] * (i < 144 ? 8 : i < 256 ? 9 : i < 280 ? 7 : 8);
            for (int i = 0; i < 30; i++) fixed_bits += (uint64_t)d.freq[288 + i] * 5;
            build_lengths(d.freq, 286, 15, d.len_ll, d.order, d.w, d.par, d.depth);
            build_lengths(d.freq + 288, 30, 15, d.len_d, d.order, d.w, d.par, d.depth);
            bool any_d = false;
            for (int i = 0; i < 30; i++) any_d |= d.len_d[i] != 0;
            if (!any_d) d.len_d[0] = 1;                       // "one distance code of one bit": a set every inflater accepts
            for (int i = 286; i < 288; i++) d.len_ll[i] = 0;
            d.len_d[30] = d.len_d[31] = 0;
            assign_codes(d.len_ll, 286, 15, d.code_ll);
            assign_codes(d.len_d, 30, 15, d.code_d);
            for (int i = 285; i >= 257; i--) if (d.len_ll[i]) { hlit = (uint32_t)i + 1; break; }
            for (int i = 29; i >= 1; i--) if (d.len_d[i]) { hdist = (uint32_t)i + 1; break; }
            // the code lengths as one sequence, run-length coded with symbols 16 / 17 / 18 (3.2.7)
            for (int i = 0; i < 19; i++) d.cl_freq[i] = 0;
            uint32_t ncl = 0;
            const uint32_t nseq = hlit + hdist;
            uint32_t i = 0;
            while (i < nseq) {
                const uint32_t v = i < hlit ? d.len_ll[i] : d.len_d[i - hlit];
                uint32_t run = 1;
                while (i + run < nseq && (i + run < hlit ? d.len_ll[i + run] : d.len_d[i + run - hlit]) == v) run++;
                i += run;
                if (v == 0) {
                    while (run >= 11) { const uint32_t r = run < 138 ? run : 138; d.cl_sym[ncl] = 18; d.cl_ext[ncl++] = (uint8_t)(r - 11); d.cl_freq[18]++; run -= r; }
                    if (run >= 3) { d.cl_sym[ncl] = 17; d.cl_ext[ncl++] = (uint8_t)(run - 3); d.cl_freq[17]++; run = 0; }
                } else {
                    d.cl_sym[ncl] = (uint8_t)v; d.cl_ext[ncl++] = 0; d.cl_freq[v]++; run--;
                    while (run >= 3) { const uint32_t r = run < 6 ? run : 6; d.cl_sym[ncl] = 16; d.cl_ext[ncl++] = (uint8_t)(r - 3); d.cl_freq[16]++; run -= r; }
                }
                while (run--) { d.cl_sym[ncl] = (uint8_t)v; d.cl_ext[ncl++] = 0; d.cl_freq[v]++; }
            }
            d.n_cl = ncl;
            build_lengths(d.cl_freq, 19, 7, d.cl_len, d.order, d.w, d.par, d.depth);
            {   // the code-length code must be complete (zlib rejects an incomplete CODES set even of one code): pair a lone code
                int used = 0, only = 0;
                for (int k = 0; k < 19; k++) if (d.cl_len[k]) { used++; only = k; }
                if (used == 1) d.cl_len[only == 0 ? 1 : 0] = 1;
            }
            assign_codes(d.cl_len, 19, 7, d.cl_code);
            for (int k = 18; k >= 4; k--) if (d.cl_len[c_cl_order[k]]) { hclen = (uint32_t)k + 1; break; }
            dyn_bits += 3 * hclen;
            for (int k = 0; k < 19; k++) dyn_bits += (uint64_t)d.cl_freq[k] * (d.cl_len[k] + (k == 16 ? 2 : k == 17 ? 3 : k == 18 ? 7 : 0));
            for (int k = 0; k < 286; k++) dyn_bits += (uint64_t)d.freq[k] * d.len_ll[k];
            for (int k = 0; k < 30; k++) dyn_bits += (uint64_t)d.freq[288 + k] * d.len_d[k];
            use_dyn = dyn_bits < fixed_bits ? 1u : 0u;
        }
        use_dyn = __shfl_sync(0xffffffffu, use_dyn, 0);
        hlit = __shfl_sync(0xffffffffu, hlit, 0); hdist = __shfl_sync(0xffffffffu, hdist, 0); hclen = __shfl_sync(0xffffffffu, hclen, 0);
        __syncwarp();
        // zero the slot's deflate area first (bits are ORed in)
        uint32_t *ow = reinterpret_cast<uint32_t *>(out);          // out slots are 64 KiB aligned by contract (>= 4)
        for (uint32_t i = lane; i < 65536 / 4; i += 32) ow[i] = 0;
        __syncwarp();
        __threadfence_block();
        uint64_t bitpos = 18 * 8;
        if (lane == 0) {
            // lane 0 alone writes the block header; the other lanes join after the barrier below
            uint64_t bp = bitpos;
            auto put = [&](uint32_t bits, uint32_t nb) {
                if (!nb) return;
                const uint32_t w = (uint32_t)(bp >> 5), sh = (uint32_t)(bp & 31);
                ow[w] |= bits << sh;
                if (sh + nb > 32) ow[w + 1] |= bits >> (32 - sh);
                bp += nb;
            };
            if (!use_dyn) put(3u, 3);                              // BFINAL=1, BTYPE=01
            else {
                put(5u, 3);                                        // BFINAL=1, BTYPE=10
                put(hlit - 257, 5); put(hdist - 1, 5); put(hclen - 4, 4);
                for (uint32_t k = 0; k < hclen; k++) put(d.cl_len[c_cl_order[k]], 3);
                for (uint32_t k = 0; k < d.n_cl; k++) {
                    const uint32_t sy = d.cl_sym[k];
                    put(d.cl_code[sy], d.cl_len[sy]);
                    if (sy == 16) put(d.cl_ext[k], 2); else if (sy == 17) put(d.cl_ext[k], 3); else if (sy == 18) put(d.cl_ext[k], 7);
                }
            }
            bitpos = bp;
        }
        bitpos = __shfl_sync(0xffffffffu, (unsigned long long)bitpos, 0);
        __syncwarp();
        __threadfence_block();
        const uint64_t limit = (uint64_t)(65536 - 8 - 4) * 8;       // keep room for EOB + footer
        for (uint32_t t0 = 0; t0 < ntok && !overflow; t0 += 32) {
            uint32_t t = t0 + lane, nb = 0;
            uint64_t bits = 0;
            if (t < ntok) { if (use_dyn) bits = token_bits_dyn(d, toks[t], nb); else bits = token_bits(toks[t], nb); }
            uint32_t inc = nb;
#pragma unroll
            for (int dd = 1; dd < 32; dd <<= 1) { uint32_t v = __shfl_up_sync(0xffffffffu, inc, dd); if (lane >= (uint32_t)dd) inc += v; }
            uint32_t tot = __shfl_sync(0xffffffffu, inc, 31);
            if (bitpos + tot > limit) { overflow = true; break; }
            if (nb) {
                uint64_t bp = bitpos + inc - nb;
                uint32_t w = (uint32_t)(bp >> 5), sh = (uint32_t)(bp & 31);
                atomicOr(&ow[w], (uint32_t)(bits << sh));                                   // up to 48 bits at any bit offset: three words
                if (sh + nb > 32) atomicOr(&ow[w + 1], sh ? (uint32_t)(bits >> (32 - sh)) : (uint32_t)(bits >> 32));
                if (sh + nb > 64) atomicOr(&ow[w + 2], (uint32_t)(bits >> (64 - sh)));
            }
            bitpos += tot;
        }
        if (!overflow) {
            // end-of-block code: seven zero bits under the fixed code, the block's own code otherwise
            const uint32_t eob_n = use_dyn ? d.len_ll[256] : 7u;
            if (use_dyn && lane == 0) {
                const uint32_t w = (uint32_t)(bitpos >> 5), sh = (uint32_t)(bitpos & 31);
                const uint32_t bits = d.code_ll[256];
                atomicOr(&ow[w], bits << sh);
                if (sh + eob_n > 32) atomicOr(&ow[w + 1], bits >> (32 - sh));
            }
            bitpos += eob_n;
            dlen = (uint32_t)((bitpos + 7) / 8) - 18;
            if (dlen >= n + 5) overflow = true;                    // stored would be smaller
        }
        __syncwarp();
        __threadfence_block();
        stored = overflow;
    }
    if (stored) {
        dlen = n + 5;
        __syncwarp();
        if (lane == 0) {
            out[18] = 1;                                            // BFINAL=1, BTYPE=00
            out[19] = (uint8_t)n; out[20] = (uint8_t)(n >> 8);
            out[21] = (uint8_t)~n; out[22] = (uint8_t)(~n >> 8);
        }
        for (uint32_t i = lane; i < n; i += 32) out[23 + i] = in[i];
    }
    const uint32_t total = 18 + dlen + 8;
    __syncwarp();
    if (lane == 0) {
        const uint8_t hdr[16] = {0x1f, 0x8b, 8, 4, 0, 0, 0, 0, 0, 0xff, 6, 0, 'B', 'C', 2, 0};
        for (int i = 0; i < 16; i++) out[i] = hdr[i];
        out[16] = (uint8_t)(total - 1); out[17] = (uint8_t)((total - 1) >> 8);
        uint8_t *f = out + 18 + dlen;
        f[0] = (uint8_t)crc; f[1] = (uint8_t)(crc >> 8); f[2] = (uint8_t)(crc >> 16); f[3] = (uint8_t)(crc >> 24);
        f[4] = (uint8_t)n; f[5] = (uint8_t)(n >> 8); f[6] = 0; f[7] = 0;
    }
    __syncwarp();
    return total;
}

__global__ void __launch_bounds__(128)
bgzf_deflate_kernel(const uint8_t *__restrict__ in, const uint64_t *__restrict__ in_off,
                    const uint32_t *__restrict__ in_len, uint32_t n, int level, uint8_t *out,
                    const uint64_t *__restrict__ out_off, uint32_t *out_len, int32_t *status,
                    uint32_t *toks_all, uint32_t *counter)
{
    __shared__ DeflateSmem smem_all[4];
    __shared__ uint32_t crc_tab[4][256];
    for (int i = threadIdx.x; i < 1024; i += blockDim.x) (&crc_tab[0][0])[i] = (&g_crc_tab[0][0])[i];
    __syncthreads();
    const uint32_t w = threadIdx.x >> 5;
    uint32_t *toks = toks_all + ((size_t)blockIdx.x * 4 + w) * DEFL_TOK_CAP;
    for (;;) {
        uint32_t job = 0;
        if (hgpu_lane() == 0) job = atomicAdd(counter, 1u);
        job = __shfl_sync(0xffffffffu, job, 0);
        if (job >= n) break;
        uint32_t got = deflate_block_warp(smem_all[w], crc_tab, in + in_off[job], in_len[job], level, out + out_off[job], toks);
        __syncwarp();
        if (hgpu_lane() == 0) { out_len[job] = got; status[job] = got ? HGPU_OK : HGPU_BGZF_ERR_ZLIB; }
    }
}

} // namespace

int hgpu_launch_bgzf_inflate(hgpu_ctx *ctx, const uint8_t *d_in, const uint64_t *d_in_off,
                             const uint32_t *d_in_len, uint32_t n, uint8_t *d_out,
                             const uint64_t *d_out_off, const uint32_t *d_out_cap,
                             uint32_t *d_out_len, int32_t *d_status, cudaStream_t st)
{
    if (n == 0) return HGPU_OK;
    if (hgpu_check(cudaSetDevice(ctx->device), "cudaSetDevice")) return HGPU_ERR_CUDA;
    int rc = ensure_crc_tables(ctx, st);
    if (rc) return rc;
    // one warp per block, as many blocks in flight per SM as occupancy allows
    static bool attr_set[64];                          // function attributes are per device
    const int dv = ctx->device & 63;
    const size_t dyn_w = 4096 + INFLATE_WARPS * sizeof(InflateSmem);
    if (!attr_set[dv]) {
        if (hgpu_check(cudaFuncSetAttribute(bgzf_inflate_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)dyn_w), "inflate smem attr"))
            return HGPU_ERR_CUDA;
        attr_set[dv] = true;
    }
    int per_sm = 0;
    if (hgpu_check(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, bgzf_inflate_kernel, 32 * INFLATE_WARPS, dyn_w), "inflate occupancy"))
        return HGPU_ERR_CUDA;
    if (per_sm < 1) per_sm = 1;
    const uint32_t units = (n + INFLATE_WARPS - 1) / INFLATE_WARPS;
    uint32_t full_grid = (uint32_t)ctx->sm_count * (uint32_t)per_sm, grid = full_grid;
    if (grid > units) grid = units;
    uint32_t *counter = hgpu_take_counter(ctx, st);
    if (!counter) return HGPU_ERR_CUDA;
    // match-record scratch, one slot per resident warp, sized for the full grid so concurrent
    // launches on other streams (the pipelined host path) can share the same layout
    const uint32_t slots = full_grid * INFLATE_WARPS;
    rc = hgpu_ensure_mrec(ctx, (size_t)slots * MREC_CAP * sizeof(uint2) * 3);
    if (rc) return rc;
    uint2 *mrec = reinterpret_cast<uint2 *>(ctx->d_mrec) + (size_t)(ctx->next_counter % 3) * slots * MREC_CAP;
    bgzf_inflate_kernel<<<grid, 32 * INFLATE_WARPS, dyn_w, st>>>(d_in, d_in_off, d_in_len, n, d_out, d_out_off, d_out_cap,
                                                                 d_out_len, d_status, counter, mrec);
    hgpu_count_launch();
    return hgpu_check(cudaGetLastError(), "inflate launch");
}

// gzip members (device pointers): same calling shape as hgpu_launch_bgzf_inflate, no 64 KiB clamp
int hgpu_launch_gzip_inflate(hgpu_ctx *ctx, const uint8_t *d_in, const uint64_t *d_in_off, const uint32_t *d_in_len, uint32_t n,
                             uint8_t *d_out, const uint64_t *d_out_off, const uint32_t *d_out_cap, uint32_t *d_out_len,
                             int32_t *d_status, cudaStream_t st)
{
    if (n == 0) return HGPU_OK;
    if (hgpu_check(cudaSetDevice(ctx->device), "cudaSetDevice")) return HGPU_ERR_CUDA;
    int rc = ensure_crc_tables(ctx, st);
    if (rc) return rc;
    static bool attr_set[64];
    const int dv = ctx->device & 63;
    const size_t dyn_w = 4096 + INFLATE_WARPS * sizeof(InflateSmem);
    if (!attr_set[dv]) {
        if (hgpu_check(cudaFuncSetAttribute(gzip_inflate_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)dyn_w), "gzip smem attr")) return HGPU_ERR_CUDA;
        attr_set[dv] = true;
    }
    uint32_t grid = (n + INFLATE_WARPS - 1) / INFLATE_WARPS;
    const uint32_t full = (uint32_t)ctx->sm_count;          // CRAM files hold a handful of GZIP blocks: one CTA per SM is plenty
    if (grid > full) grid = full;
    uint32_t *counter = hgpu_take_counter(ctx, st);
    if (!counter) return HGPU_ERR_CUDA;
    // match-record scratch: the BGZF layout (three rotating sets for the pipelined host path) in front, this kernel's slots behind it
    const size_t bgzf_part = (size_t)ctx->sm_count * 4u * INFLATE_WARPS * MREC_CAP * sizeof(uint2) * 3;
    rc = hgpu_ensure_mrec(ctx, bgzf_part + (size_t)full * INFLATE_WARPS * GZ_MREC * sizeof(uint2));
    if (rc) return rc;
    uint2 *mrec = reinterpret_cast<uint2 *>(ctx->d_mrec + bgzf_part);
    gzip_inflate_kernel<<<grid, 32 * INFLATE_WARPS, dyn_w, st>>>(d_in, d_in_off, d_in_len, n, d_out, d_out_off, d_out_cap, d_out_len, d_status, counter, mrec);
    hgpu_count_launch();
    return hgpu_check(cudaGetLastError(), "gzip inflate launch");
}

extern "C" int hgpu_debug_profile(unsigned long long *out8)
{
#ifdef HGPU_PROFILE
    unsigned long long z[16] = {0};
    if (cudaMemcpyFromSymbol(out8, g_prof, sizeof(z)) != cudaSuccess) return -1;
    cudaMemcpyToSymbol(g_prof, z, sizeof(z));
    return 0;
#else
    (void)out8;
    return -1;
#endif
}

// CRC-32 of a device buffer: per-chunk warp CRCs, combined on the host side of the ABI by the
// caller (hgpu_api.cu) with the same x^n arithmetic.
int hgpu_launch_crc32(hgpu_ctx *ctx, const uint8_t *d_buf, size_t len, uint32_t *d_partial,
                      uint32_t *h_result, uint32_t crc0, cudaStream_t st)
{
    (void)h_result; (void)crc0;
    int rc = ensure_crc_tables(ctx, st);
    if (rc) return rc;
    const size_t chunk = 1u << 20;
    size_t nchunk = (len + chunk - 1) / chunk;
    if (nchunk == 0) return HGPU_OK;
    crc32_chunks_kernel<<<(unsigned)nchunk, 32, 0, st>>>(d_buf, len, chunk, d_partial);
    hgpu_count_launch();
    return hgpu_check(cudaGetLastError(), "crc launch");
}

int hgpu_launch_crc32_batch(hgpu_ctx *ctx, const uint8_t *d_buf, const uint64_t *d_off, const uint32_t *d_len, uint32_t n,
                            uint32_t *d_crc, cudaStream_t st)
{
    if (n == 0) return HGPU_OK;
    int rc = ensure_crc_tables(ctx, st);
    if (rc) return rc;
    crc32_batch_kernel<<<(n + 3) / 4, 128, 0, st>>>(d_buf, d_off, d_len, n, d_crc);
    hgpu_count_launch();
    return hgpu_check(cudaGetLastError(), "crc batch launch");
}

// Batch BGZF compress, device pointers.  Every out slot must be 65536 bytes and 4-byte aligned.
extern "C" int hgpu_bgzf_compress_batch_dev(hgpu_ctx *ctx, const uint8_t *d_in, const uint64_t *d_in_off,
        const uint32_t *d_in_len, uint32_t n, int level, uint8_t *d_out, const uint64_t *d_out_off,
        uint32_t *d_out_len, int32_t *d_status, void *stream)
{
    if (!ctx) { hgpu_set_error("null context"); return HGPU_ERR_ARG; }
    if (n == 0) return HGPU_OK;
    if (level < 0) level = 6;                           // Z_DEFAULT_COMPRESSION, as zlib's deflateInit2 reads it
    cudaStream_t st = stream ? (cudaStream_t)stream : ctx->stream;
    int rc = ensure_crc_tables(ctx, st);
    if (rc) return rc;
    int per_sm = 0;
    if (hgpu_check(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, bgzf_deflate_kernel, 128, 0), "deflate occupancy"))
        return HGPU_ERR_CUDA;
    if (per_sm < 1) per_sm = 1;
    uint32_t full = (uint32_t)ctx->sm_count * (uint32_t)per_sm, grid = full;
    if (grid > (n + 3) / 4) grid = (n + 3) / 4;
    rc = hgpu_ensure_mrec(ctx, (size_t)full * 4 * DEFL_TOK_CAP * sizeof(uint32_t));
    if (rc) return rc;
    uint32_t *counter = hgpu_take_counter(ctx, st);
    if (!counter) return HGPU_ERR_CUDA;
    bgzf_deflate_kernel<<<grid, 128, 0, st>>>(d_in, d_in_off, d_in_len, n, level, d_out, d_out_off, d_out_len, d_status,
                                              reinterpret_cast<uint32_t *>(ctx->d_mrec), counter);
    hgpu_count_launch();
    return hgpu_check(cudaGetLastError(), "deflate launch");
}
