// rANS 4x8 ("RANS", CRAM 3.0 block method 4) ENCODER for sm_90a.
//
// Stands where rans_compress stands (htscodecs/htscodecs/rANS_static.c:829-838) with rans_compress_O0
// (:75-214) and rans_compress_O1 (:387-597) behind it.  CRAM 3.0 is the legacy write path, so this is the
// plain mapping: one THREAD per stream runs the reference's steps in the reference's order — histogram
// (hist8 / hist1_4, utils.h:146, :280), the integer (O0) or double-precision (O1) normalisation to 4095+1,
// the run-length coded frequency table, the four interleaved 8-bit-renormalising states written backwards
// from the end of the slot (rANS_byte.h:283-318, :109-122) — and therefore emits the same bytes as the
// reference encoder; tests/test_gpu_rans4x8_enc.py pins byte equality.  The division in the state update
// is exact (x / freq, x % freq) where the reference uses a reciprocal multiply constructed to give the
// same quotient.
#include "hgpu_internal.h"

namespace {

constexpr uint32_t TF_SHIFT = 12, TOTFREQ = 1u << TF_SHIFT, RANS_BYTE_L = 1u << 23;

__device__ __forceinline__ void put_symbol(uint32_t &x, uint8_t *&ptr, uint32_t start, uint32_t freq)
{
    const uint32_t x_max = ((RANS_BYTE_L >> TF_SHIFT) << 8) * freq;
    while (x >= x_max) { *--ptr = (uint8_t)(x & 0xff); x >>= 8; }
    x = ((x / freq) << TF_SHIFT) + (x % freq) + start;
}
__device__ __forceinline__ void flush_state(uint32_t x, uint8_t *&ptr)
{
    ptr -= 4;
    ptr[0] = (uint8_t)x; ptr[1] = (uint8_t)(x >> 8); ptr[2] = (uint8_t)(x >> 16); ptr[3] = (uint8_t)(x >> 24);
}

// the symbol list with runs of consecutive symbols collapsed, shared by both orders (:133-160, :452-489)
struct RunList {
    int rle;
    template <typename Present>
    __device__ void put(uint8_t *&cp, int j, bool prev_present, const Present &present)
    {
        if (rle) { rle--; return; }
        *cp++ = (uint8_t)j;
        if (j && prev_present) {
            int r = j + 1;
            while (r < 256 && present(r)) r++;
            rle = r - (j + 1);
            *cp++ = (uint8_t)rle;
        }
    }
};

__device__ __forceinline__ void put_freq(uint8_t *&cp, uint32_t f)
{
    if (f < 128) *cp++ = (uint8_t)f;
    else { *cp++ = (uint8_t)(128 | (f >> 8)); *cp++ = (uint8_t)(f & 0xff); }
}

__device__ void write_header(uint8_t *out, int order, uint32_t total, uint32_t in_size)
{
    out[0] = (uint8_t)order;
    const uint32_t c = total - 9;
    out[1] = (uint8_t)c; out[2] = (uint8_t)(c >> 8); out[3] = (uint8_t)(c >> 16); out[4] = (uint8_t)(c >> 24);
    out[5] = (uint8_t)in_size; out[6] = (uint8_t)(in_size >> 8); out[7] = (uint8_t)(in_size >> 16); out[8] = (uint8_t)(in_size >> 24);
}

// rans_compress_O0 (:75-214).  F: 256 u32 of scratch.  Returns the stream length.
__device__ uint32_t encode_o0(const uint8_t *in, uint32_t n, uint8_t *out, uint8_t *out_end, uint32_t *F)
{
    for (int j = 0; j < 256; j++) F[j] = 0;
    for (uint32_t i = 0; i < n; i++) F[in[i]]++;
    uint64_t tr = n ? ((uint64_t)TOTFREQ << 31) / n + (1u << 30) / n : 0;
    uint32_t cnt[256];
    for (int j = 0; j < 256; j++) cnt[j] = F[j];
    int M;
    for (;;) {                                                       // normalise_harder
        int fsum = 0, m = 0;
        M = 0;
        for (int j = 0; j < 256; j++) {
            if (!cnt[j]) { F[j] = 0; continue; }
            if (m < (int)cnt[j]) { m = (int)cnt[j]; M = j; }
            uint32_t f = (uint32_t)(((uint64_t)cnt[j] * tr) >> 31);
            if (f == 0) f = 1;
            F[j] = f;
            fsum += (int)f;
        }
        fsum++;
        if (fsum < (int)TOTFREQ) { F[M] += TOTFREQ - fsum; break; }
        if (fsum - (int)TOTFREQ > (int)F[M] / 2) {                   // corner case: scale everything down and redo
            tr = 2104533975;
            for (int j = 0; j < 256; j++) cnt[j] = F[j];             // the reference re-normalises the already scaled values
            continue;
        }
        F[M] -= fsum - TOTFREQ;
        break;
    }
    uint8_t *cp = out + 9;
    uint32_t C[256];
    {
        RunList rl{0};
        uint32_t x = 0;
        for (int j = 0; j < 256; j++) {
            if (!F[j]) continue;
            rl.put(cp, j, j && F[j - 1], [&](int r) { return F[r] != 0; });
            put_freq(cp, F[j]);
            C[j] = x;
            x += F[j];
        }
        *cp++ = 0;
    }
    const uint32_t tab = (uint32_t)(cp - out);
    uint32_t r0 = RANS_BYTE_L, r1 = RANS_BYTE_L, r2 = RANS_BYTE_L, r3 = RANS_BYTE_L;
    uint8_t *ptr = out_end;
    const uint32_t t = n & 3;
    if (t == 3) put_symbol(r2, ptr, C[in[n - 1]], F[in[n - 1]]);
    if (t >= 2) put_symbol(r1, ptr, C[in[n - (t - 1)]], F[in[n - (t - 1)]]);
    if (t >= 1) put_symbol(r0, ptr, C[in[n - t]], F[in[n - t]]);
    for (uint32_t i = n & ~3u; i > 0; i -= 4) {
        put_symbol(r3, ptr, C[in[i - 1]], F[in[i - 1]]);
        put_symbol(r2, ptr, C[in[i - 2]], F[in[i - 2]]);
        put_symbol(r1, ptr, C[in[i - 3]], F[in[i - 3]]);
        put_symbol(r0, ptr, C[in[i - 4]], F[in[i - 4]]);
    }
    flush_state(r3, ptr); flush_state(r2, ptr); flush_state(r1, ptr); flush_state(r0, ptr);
    const uint32_t pay = (uint32_t)(out_end - ptr), total = pay + tab;
    write_header(out, 0, total, n);
    for (uint32_t i = 0; i < pay; i++) out[tab + i] = ptr[i];          // memmove down (tab <= ptr - out)
    return total;
}

// rans_compress_O1 (:387-597).  F: 65536 u32 of scratch (counts, then freq | start << 16).
__device__ uint32_t encode_o1(const uint8_t *in, uint32_t n, uint8_t *out, uint8_t *out_end, uint32_t *F)
{
    if (n < 4) return encode_o0(in, n, out, out_end, F);
    for (uint32_t i = 0; i < 65536; i++) F[i] = 0;
    uint32_t T[256];
    for (int i = 0; i < 256; i++) T[i] = 0;
    {                                                                   // hist1_4 (utils.h:280-355): all adjacent pairs, first has context 0
        uint32_t l = 0;
        for (uint32_t i = 0; i < n; i++) { F[l << 8 | in[i]]++; l = in[i]; }
        T[l]++;
    }
    const uint32_t q4 = n >> 2;
    F[in[1 * q4]]++; F[in[2 * q4]]++; F[in[3 * q4]]++;                  // the other three quarters also start in context 0
    // T[0] += 3 there (:427) is the three increments above, which the row sums below already include
    for (int i = 0; i < 256; i++) { uint32_t tt = 0; for (int j = 0; j < 256; j++) tt += F[i << 8 | j]; T[i] += tt; }

    uint8_t *cp = out + 9;
    RunList ri{0};
    for (int i = 0; i < 256; i++) {
        if (T[i] == 0) continue;
        uint32_t *Fi = F + (i << 8);
        double p = (double)TOTFREQ / T[i];
        int M;
        for (;;) {                                                      // normalise_harder
            int t2 = 0, m = 0;
            M = 0;
            for (int j = 0; j < 256; j++) {
                if (!Fi[j]) continue;
                if (m < (int)Fi[j]) { m = (int)Fi[j]; M = j; }
                int f = (int)((int)Fi[j] * p);
                if (f == 0) f = 1;
                Fi[j] = (uint32_t)f;
                t2 += f;
            }
            t2++;
            if (t2 < (int)TOTFREQ) { Fi[M] += TOTFREQ - t2; break; }
            if (t2 - (int)TOTFREQ >= (int)Fi[M] / 2) { p = .98; continue; }
            Fi[M] -= t2 - TOTFREQ;
            break;
        }
        ri.put(cp, i, i && T[i - 1], [&](int r) { return T[r] != 0; });
        RunList rj{0};
        uint32_t x = 0;
        for (int j = 0; j < 256; j++) {
            if (!Fi[j]) continue;
            rj.put(cp, j, j && (Fi[j - 1] & 0xffff), [&](int r) { return (Fi[r] & 0xffff) != 0; });
            put_freq(cp, Fi[j]);
            const uint32_t f = Fi[j];
            Fi[j] = f | x << 16;                                        // frequency and start for the symbol loop
            x += f;
        }
        *cp++ = 0;
    }
    *cp++ = 0;
    const uint32_t tab = (uint32_t)(cp - out);

    uint32_t r0 = RANS_BYTE_L, r1 = RANS_BYTE_L, r2 = RANS_BYTE_L, r3 = RANS_BYTE_L;
    uint8_t *ptr = out_end;
    int i0 = (int)q4 - 2, i1 = 2 * (int)q4 - 2, i2 = 3 * (int)q4 - 2, i3;
    uint32_t l0 = in[i0 + 1], l1 = in[i1 + 1], l2 = in[i2 + 1], l3 = in[n - 1];
    auto put = [&](uint32_t &r, uint32_t ctx, uint32_t sym) {
        const uint32_t e = F[ctx << 8 | sym];
        put_symbol(r, ptr, e >> 16, e & 0xffff);
    };
    for (i3 = (int)n - 2; i3 > 4 * (int)q4 - 2; i3--) { const uint32_t c3 = in[i3]; put(r3, c3, l3); l3 = c3; }
    for (; i0 >= 0; i0--, i1--, i2--, i3--) {
        const uint32_t c3 = in[i3], c2 = in[i2], c1 = in[i1], c0 = in[i0];
        put(r3, c3, l3); put(r2, c2, l2); put(r1, c1, l1); put(r0, c0, l0);
        l3 = c3; l2 = c2; l1 = c1; l0 = c0;
    }
    put(r3, 0, l3); put(r2, 0, l2); put(r1, 0, l1); put(r0, 0, l0);
    flush_state(r3, ptr); flush_state(r2, ptr); flush_state(r1, ptr); flush_state(r0, ptr);
    const uint32_t pay = (uint32_t)(out_end - ptr), total = pay + tab;
    write_header(out, 1, total, n);
    for (uint32_t i = 0; i < pay; i++) out[tab + i] = ptr[i];
    return total;
}

__global__ void __launch_bounds__(32)
rans4x8_encode_kernel(const uint8_t *__restrict__ in, const uint64_t *__restrict__ in_off, const uint32_t *__restrict__ in_len,
                      const uint32_t *__restrict__ order, uint32_t n, uint8_t *out, const uint64_t *__restrict__ out_off,
                      const uint32_t *__restrict__ out_cap, uint32_t *out_len, int32_t *status, uint32_t *scratch,
                      uint32_t *counter)
{
    const size_t tid = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    uint32_t *F = scratch + tid * 65536;
    for (;;) {
        const uint32_t job = atomicAdd(counter, 1u);
        if (job >= n) break;
        const uint32_t sz = in_len[job];
        const uint32_t need = (uint32_t)(1.05 * sz) + 257 * 257 * 3 + 9;       // the reference's own buffer (:77, :90)
        if (out_cap[job] < need) { status[job] = -1; out_len[job] = 0; continue; }
        uint8_t *o = out + out_off[job];
        const uint32_t got = (order[job] & 1) ? encode_o1(in + in_off[job], sz, o, o + need, F)
                                              : encode_o0(in + in_off[job], sz, o, o + need, F);
        status[job] = 0;
        out_len[job] = got;
    }
}

}  // namespace

extern "C" uint32_t hgpu_rans4x8_compress_bound(uint32_t size) { return (uint32_t)(1.05 * size) + 257 * 257 * 3 + 9; }

extern "C" int hgpu_rans4x8_encode_batch_dev(hgpu_ctx *ctx, const uint8_t *d_in, const uint64_t *d_in_off,
        const uint32_t *d_in_len, const uint32_t *d_order, uint32_t n, uint8_t *d_out, const uint64_t *d_out_off,
        const uint32_t *d_out_cap, uint32_t *d_out_len, int32_t *d_status, void *stream)
{
    if (!ctx) { hgpu_set_error("null context"); return HGPU_ERR_ARG; }
    if (n == 0) return HGPU_OK;
    cudaStream_t st = stream ? (cudaStream_t)stream : ctx->stream;
    const uint32_t threads = n < 2048u ? n : 2048u;
    const uint32_t grid = (threads + 31) / 32;
    int rc = hgpu_ensure_scratch(ctx, (size_t)grid * 32 * 65536 * sizeof(uint32_t));
    if (rc) return rc;
    uint32_t *counter = hgpu_take_counter(ctx, st);
    if (!counter) return HGPU_ERR_CUDA;
    rans4x8_encode_kernel<<<grid, 32, 0, st>>>(d_in, d_in_off, d_in_len, d_order, n, d_out, d_out_off, d_out_cap, d_out_len,
                                               d_status, (uint32_t *)ctx->d_scratch, counter);
    hgpu_count_launch();
    return hgpu_check(cudaGetLastError(), "rans4x8 encode launch");
}
