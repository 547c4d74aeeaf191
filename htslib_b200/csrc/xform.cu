// The byte transforms of the libhtscodecs link seam that cram/cram_codecs.c binds directly (XPACK / XRLE,
// cram_codecs.c:1399, :1520, :2106, :2278) and cram_external.c binds for its version string:
//   hts_pack / hts_unpack_meta / hts_unpack   (htscodecs pack.c:56-150, :161-196, :207-330)
//   hts_rle_encode / hts_rle_decode           (htscodecs rle.c:48-190)
//   htscodecs_version                         (htscodecs.c:42)
// Same signatures, malloc ownership and NULL-on-error as the reference; host pointers; the data goes through
// the device (one stream per call: correct, slow — inside the rANS container the same transforms run fused in
// rans_nx16_decode_kernel).  Output bytes are the format's, so they equal the reference's byte for byte.
#include "hgpu_internal.h"
#include "xform_dev.cuh"
#include <new>
#include <stdlib.h>
#include <string.h>

namespace {

// ---- unpack: out[i] = map[field i of data]; fully parallel
__global__ void xf_unpack_kernel(const uint8_t *d, uint64_t len, uint8_t *out, uint64_t olen, int per_byte, const uint8_t *map)
{
    const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
    const int bits = per_byte == 8 ? 1 : per_byte == 4 ? 2 : 4;
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < olen; i += stride) {
        if (per_byte == 1) out[i] = d[i];
        else if (per_byte == 0) out[i] = map[0];
        else out[i] = map[(d[i / per_byte] >> (bits * (i % per_byte))) & ((1 << bits) - 1)];
    }
    (void)len;
}

// ---- pack, pass 1: which byte values occur
__global__ void xf_present_kernel(const uint8_t *d, uint64_t len, uint32_t *present)
{
    const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < len; i += stride) present[d[i]] = 1;   // benign race
}
// ---- pack, pass 2: one output byte per thread (low fields first, pack.c:97-141)
__global__ void xf_pack_kernel(const uint8_t *d, uint64_t len, uint8_t *out, uint64_t olen, int per_byte, const uint8_t *code)
{
    const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
    const int bits = 8 / per_byte;
    for (uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; j < olen; j += stride) {
        uint32_t v = 0;
        for (int k = 0; k < per_byte; k++) {
            const uint64_t i = j * per_byte + k;
            if (i < len) v |= (uint32_t)code[d[i]] << (bits * k);
        }
        out[j] = (uint8_t)v;
    }
}

// ---- RLE survey (rle_find_syms): saved[s] += 1 when a byte repeats its predecessor, -1 when it does not
__global__ void xf_rle_survey_kernel(const uint8_t *d, uint64_t len, int *saved)
{
    __shared__ int loc[256];
    for (int k = threadIdx.x; k < 256; k += blockDim.x) loc[k] = 0;
    __syncthreads();
    const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < len; i += stride)
        atomicAdd(&loc[d[i]], (i > 0 && d[i] == d[i - 1]) ? 1 : -1);
    __syncthreads();
    for (int k = threadIdx.x; k < 256; k += blockDim.x) if (loc[k]) atomicAdd(&saved[k], loc[k]);
}

// ---- RLE encode (rle.c:100-140), one warp (xform_dev.cuh)
__global__ void xf_rle_encode_kernel(const uint8_t *d, uint64_t len, const uint8_t *inset, uint8_t *lit, uint8_t *run, uint64_t *lens /* [0]=nlit [1]=nrun */)
{
    uint64_t k, j;
    warp_rle_encode(d, len, inset, lit, run, k, j);
    if ((threadIdx.x & 31) == 0) { lens[0] = k; lens[1] = j; }
}

// ---- RLE decode (rle.c:142-190), one warp: 32 literals per round; lane 0 reads the run lengths in order
__device__ __forceinline__ int get_var(const uint8_t *p, const uint8_t *end, uint32_t &v)      // var_get_u32, varint.h:267
{
    const uint8_t *s = p;
    uint32_t acc = 0;
    int budget = 5;
    uint8_t c;
    do {
        if (p >= end) { v = acc; return (int)(p - s); }
        c = *p++;
        acc = (acc << 7) | (c & 0x7f);
    } while ((c & 0x80) && --budget > 0);
    v = acc;
    return (int)(p - s);
}
__global__ void xf_rle_decode_kernel(const uint8_t *lit, uint64_t nlit, const uint8_t *run, uint64_t nrun, const uint8_t *inset,
                                     uint8_t *out, uint64_t cap, uint64_t *res /* [0]=olen or ~0 on error */)
{
    __shared__ uint32_t rl[32];
    const uint32_t lane = threadIdx.x & 31;
    const uint8_t *rp = run, *rend = run + nrun;
    uint64_t o = 0;
    bool bad = false;
    for (uint64_t base = 0; base < nlit && !bad; base += 32) {
        const uint64_t i = base + lane;
        const uint8_t b = i < nlit ? lit[i] : 0;
        const bool has = i < nlit && inset[b];
        const uint32_t bal = __ballot_sync(0xffffffffu, has);
        if (lane == 0) {
            uint32_t mm = bal;
            while (mm) { const int z = __ffs(mm) - 1; mm &= mm - 1; uint32_t r; rp += get_var(rp, rend, r); rl[z] = r; }
        }
        rp = reinterpret_cast<const uint8_t *>(__shfl_sync(0xffffffffu, (unsigned long long)rp, 0));
        __syncwarp();
        const uint32_t mylen = i < nlit ? (has ? rl[lane] + 1u : 1u) : 0u;
        uint64_t inc = mylen;
#pragma unroll
        for (int dd = 1; dd < 32; dd <<= 1) { uint64_t tv = __shfl_up_sync(0xffffffffu, inc, dd); if (lane >= (uint32_t)dd) inc += tv; }
        const uint64_t my_o = o + inc - mylen;
        bool mybad = false;
        if (i < nlit) {                                             // the reference checks literal by literal (rle.c:160-172)
            if (my_o >= cap) mybad = true;
            else if (has && mylen > 1 && my_o + (mylen - 1) >= cap) mybad = true;
        }
        bad = __any_sync(0xffffffffu, mybad);
        if (!bad && i < nlit) for (uint32_t x = 0; x < mylen; x++) out[my_o + x] = b;
        o += __shfl_sync(0xffffffffu, inc, 31);
        __syncwarp();
    }
    if (lane == 0) res[0] = bad ? ~0ull : o;
}

// binds one call's layout to the staging buffer of the process-wide shim context
struct Stage {
    hgpu_ctx *ctx; cudaStream_t s;
    bool ok;
    Stage(StageLayout &L) : ctx(hgpu_shim_ctx()), s(nullptr), ok(false)
    {
        if (!ctx) return;
        if (cudaSetDevice(ctx->device) != cudaSuccess) return;
        if (hgpu_stage_ensure(ctx, L)) return;
        s = ctx->stream; ok = true;
    }
};

}  // namespace

extern "C" {

const char *htscodecs_version(void) { return "1.6.6-htsgpu"; }       // the htscodecs release whose formats this library speaks

uint8_t hts_unpack_meta(uint8_t *data, uint32_t data_len, uint64_t udata_len, uint8_t *map, int *nsym)
{
    // pack.c:161-196: a dozen bytes of framing, read where they lie
    if (data_len == 0) return 0;
    unsigned int n = data[0];
    if (n == 0) n = 256;
    if (n <= 1) *nsym = 0;
    else if (n <= 2) *nsym = 8;
    else if (n <= 4) *nsym = 4;
    else if (n <= 16) *nsym = 2;
    else { *nsym = 1; return 1; }                                     // no packing
    if (data_len <= 1) return 0;
    unsigned int j = 1, c = 0;
    do { map[c++] = data[j++]; } while (c < n && j < data_len);
    (void)udata_len;
    return c < n ? 0 : (uint8_t)j;
}

uint8_t *hts_unpack(uint8_t *data, int64_t len, uint8_t *out, uint64_t out_len, int nsym, uint8_t *map)
{
    if (!out || len < 0 || (len && !data)) return nullptr;
    if (nsym != 0 && nsym != 1 && nsym != 2 && nsym != 4 && nsym != 8) return nullptr;
    if (nsym == 1) { if ((uint64_t)len < out_len) return nullptr; }
    else if (nsym > 1 && (out_len + nsym - 1) / nsym > (uint64_t)len) return nullptr;      // pack.c:226-229, :262, :300
    if (out_len == 0) return out;
    ShimLock lock;
    try {
        StageLayout L;
        const auto s_in = L.seg((size_t)len), s_out = L.seg(out_len), s_map = L.seg(16);
        Stage st(L);
        if (!st.ok) return nullptr;
        uint8_t *d_in = L.at(s_in), *d_out = L.at(s_out), *d_map = L.at(s_map);
        if (hgpu_h2d(d_in, data, (size_t)len, st.s) || hgpu_h2d(d_map, map, 16, st.s)) return nullptr;
        xf_unpack_kernel<<<(unsigned)((out_len + 255) / 256 < 4096 ? (out_len + 255) / 256 : 4096), 256, 0, st.s>>>(d_in, (uint64_t)len, d_out, out_len, nsym, d_map);
        hgpu_count_launch();
        if (hgpu_check(cudaGetLastError(), "xf_unpack") || hgpu_d2h(out, d_out, out_len, st.s) ||
            hgpu_check(cudaStreamSynchronize(st.s), "sync")) return nullptr;
        return out;
    } catch (...) { return nullptr; }
}

uint8_t *hts_pack(uint8_t *data, int64_t len, uint8_t *out_meta, int *out_meta_len, uint64_t *out_len)
{
    if (len < 0 || (len && !data) || !out_meta || !out_meta_len || !out_len) return nullptr;
    ShimLock lock;
    try {
        uint32_t present[256];
        StageLayout L;
        const auto s_in = L.seg((size_t)len), s_out = L.seg((size_t)len + 1), s_code = L.seg(256), s_present = L.seg(sizeof(present));
        Stage st(L);
        if (!st.ok) return nullptr;
        uint8_t *d_in = L.at(s_in), *d_out = L.at(s_out), *d_code = L.at(s_code);
        uint32_t *d_present = L.at<uint32_t>(s_present);
        if (hgpu_h2d(d_in, data, (size_t)len, st.s) || hgpu_memset(d_present, 0, sizeof(present), st.s)) return nullptr;
        if (len) { xf_present_kernel<<<(unsigned)(((uint64_t)len + 255) / 256 < 4096 ? ((uint64_t)len + 255) / 256 : 4096), 256, 0, st.s>>>(d_in, (uint64_t)len, d_present); hgpu_count_launch(); }
        if (hgpu_d2h(present, d_present, sizeof(present), st.s) || hgpu_check(cudaStreamSynchronize(st.s), "sync")) return nullptr;
        uint8_t code[256];
        int n = 0;
        for (int i = 0; i < 256; i++) if (present[i]) { code[i] = (uint8_t)n++; out_meta[n] = (uint8_t)i; } else code[i] = 0;
        out_meta[0] = (uint8_t)n;                                     // 256 wraps to 0
        if (n > 16) return nullptr;
        const int per = n > 4 ? 2 : n > 2 ? 4 : n > 1 ? 8 : 0;
        uint8_t *out = (uint8_t *)malloc((size_t)len + 1);
        if (!out) return nullptr;
        *out_meta_len = n + 1;
        const uint64_t olen = per ? ((uint64_t)len + per - 1) / per : 0;
        if (olen) {
            if (hgpu_h2d(d_code, code, 256, st.s)) { free(out); return nullptr; }
            xf_pack_kernel<<<(unsigned)((olen + 255) / 256 < 4096 ? (olen + 255) / 256 : 4096), 256, 0, st.s>>>(d_in, (uint64_t)len, d_out, olen, per, d_code);
            hgpu_count_launch();
            if (hgpu_check(cudaGetLastError(), "xf_pack") || hgpu_d2h(out, d_out, olen, st.s) ||
                hgpu_check(cudaStreamSynchronize(st.s), "sync")) { free(out); return nullptr; }
        }
        *out_len = olen;
        return out;
    } catch (...) { return nullptr; }
}

uint8_t *hts_rle_encode(uint8_t *data, uint64_t data_len, uint8_t *run, uint64_t *run_len, uint8_t *rle_syms, int *rle_nsyms,
                        uint8_t *out, uint64_t *out_len)
{
    if ((data_len && !data) || !run || !run_len || !rle_syms || !rle_nsyms || !out_len) return nullptr;
    ShimLock lock;
    try {
        // worst cases: literals data_len bytes, run lengths one byte per literal
        StageLayout L;
        const auto s_in = L.seg(data_len), s_lit = L.seg(data_len), s_run = L.seg(data_len), s_set = L.seg(256), s_saved = L.seg(256 * sizeof(int)),
                   s_lens = L.seg(16);
        Stage st(L);
        if (!st.ok) return nullptr;
        uint8_t *d_in = L.at(s_in), *d_lit = L.at(s_lit), *d_run = L.at(s_run), *d_set = L.at(s_set);
        int *d_saved = L.at<int>(s_saved);
        uint64_t *d_lens = L.at<uint64_t>(s_lens);
        if (hgpu_h2d(d_in, data, data_len, st.s)) return nullptr;
        uint8_t inset[256] = {0};
        if (*rle_nsyms) { for (int i = 0; i < *rle_nsyms; i++) inset[rle_syms[i]] = 1; }
        else {
            int saved[256];
            if (hgpu_memset(d_saved, 0, sizeof(saved), st.s)) return nullptr;
            if (data_len) { xf_rle_survey_kernel<<<(unsigned)((data_len + 255) / 256 < 1024 ? (data_len + 255) / 256 : 1024), 256, 0, st.s>>>(d_in, data_len, d_saved); hgpu_count_launch(); }
            if (hgpu_d2h(saved, d_saved, sizeof(saved), st.s) || hgpu_check(cudaStreamSynchronize(st.s), "sync")) return nullptr;
            int n = 0;
            for (int i = 0; i < 256; i++) if (saved[i] > 0) { rle_syms[n++] = (uint8_t)i; inset[i] = 1; }
            *rle_nsyms = n;
        }
        uint64_t lens[2] = {0, 0};
        if (data_len) {
            if (hgpu_h2d(d_set, inset, 256, st.s)) return nullptr;
            xf_rle_encode_kernel<<<1, 32, 0, st.s>>>(d_in, data_len, d_set, d_lit, d_run, d_lens);
            hgpu_count_launch();
            if (hgpu_check(cudaGetLastError(), "xf_rle_encode") || hgpu_d2h(lens, d_lens, sizeof(lens), st.s) ||
                hgpu_check(cudaStreamSynchronize(st.s), "sync")) return nullptr;
        }
        bool mine = false;
        if (!out) { out = (uint8_t *)malloc(data_len * 2 + 1); if (!out) return nullptr; mine = true; }
        if (hgpu_d2h(out, d_lit, lens[0], st.s) || hgpu_d2h(run, d_run, lens[1], st.s) ||
            hgpu_check(cudaStreamSynchronize(st.s), "sync")) { if (mine) free(out); return nullptr; }
        *out_len = lens[0];
        *run_len = lens[1];
        return out;
    } catch (...) { return nullptr; }
}

uint8_t *hts_rle_decode(uint8_t *lit, uint64_t lit_len, uint8_t *run, uint64_t run_len, uint8_t *rle_syms, int rle_nsyms,
                        uint8_t *out, uint64_t *out_len)
{
    if ((lit_len && !lit) || (run_len && !run) || !out || !out_len || rle_nsyms < 0 || (rle_nsyms && !rle_syms)) return nullptr;
    if (lit_len == 0) { *out_len = 0; return out; }
    ShimLock lock;
    try {
        const uint64_t cap = *out_len;
        StageLayout L;
        const auto s_lit = L.seg(lit_len), s_run = L.seg(run_len), s_out = L.seg(cap), s_set = L.seg(256), s_res = L.seg(8);
        Stage st(L);
        if (!st.ok) return nullptr;
        uint8_t *d_lit = L.at(s_lit), *d_run = L.at(s_run), *d_out = L.at(s_out), *d_set = L.at(s_set);
        uint64_t *d_res = L.at<uint64_t>(s_res);
        uint8_t inset[256] = {0};
        for (int i = 0; i < rle_nsyms; i++) inset[rle_syms[i]] = 1;
        if (hgpu_h2d(d_lit, lit, lit_len, st.s) || hgpu_h2d(d_run, run, run_len, st.s) || hgpu_h2d(d_set, inset, 256, st.s)) return nullptr;
        xf_rle_decode_kernel<<<1, 32, 0, st.s>>>(d_lit, lit_len, d_run, run_len, d_set, d_out, cap, d_res);
        hgpu_count_launch();
        uint64_t res = 0;
        if (hgpu_check(cudaGetLastError(), "xf_rle_decode") || hgpu_d2h(&res, d_res, 8, st.s) ||
            hgpu_check(cudaStreamSynchronize(st.s), "sync")) return nullptr;
        if (res == ~0ull || res > cap) return nullptr;
        if (res && (hgpu_d2h(out, d_out, res, st.s) || hgpu_check(cudaStreamSynchronize(st.s), "sync"))) return nullptr;
        *out_len = res;
        return out;
    } catch (...) { return nullptr; }
}

}  // extern "C"
