// C-ABI layer of libhtsgpu.so: context management, the batch entry points declared in
// include/htsgpu.h, the pipelined host-buffer paths and the reference-named shims.
// No CPU fallback anywhere: without a usable CUDA device every entry point fails.
#include "hgpu_internal.h"
#include <algorithm>
#include <atomic>
#include <mutex>
#include <stdarg.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <vector>

static std::mutex g_shim_mu;       // the process-wide context of the reference-named shims: one batch at a time
static hgpu_ctx *shim_ctx();

static thread_local char g_err[512] = "";
static std::atomic<uint64_t> g_launches{0};

void hgpu_set_error(const char *fmt, ...)
{
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}
int hgpu_check(cudaError_t e, const char *what)
{
    if (e == cudaSuccess) return 0;
    hgpu_set_error("%s: %s", what, cudaGetErrorString(e));
    return HGPU_ERR_CUDA;
}
void hgpu_count_launch(int n) { g_launches += (uint64_t)n; }

extern "C" const char *hgpu_last_error(void) { return g_err; }
extern "C" const char *hgpu_version(void) { return "htsgpu 0.1 (sm_90a)"; }
extern "C" uint64_t hgpu_launch_count(void) { return g_launches.load(); }

static int grow(uint8_t **p, size_t *cap, size_t want, bool pinned)
{
    if (*cap >= want) return HGPU_OK;
    size_t ncap = want + want / 8 + 4096;
    if (*p) {
        cudaError_t e = pinned ? cudaFreeHost(*p) : cudaFree(*p);
        *p = nullptr; *cap = 0;
        if (hgpu_check(e, "free")) return HGPU_ERR_CUDA;
    }
    cudaError_t e = pinned ? cudaMallocHost((void **)p, ncap) : cudaMalloc((void **)p, ncap);
    if (e != cudaSuccess) { hgpu_set_error("alloc of %zu bytes failed: %s", ncap, cudaGetErrorString(e)); cudaGetLastError(); return HGPU_ERR_NOMEM; }
    *cap = ncap;
    // HGPU_POISON=1 (tests): fill fresh buffers with a pattern so that a read of bytes nobody wrote shows up as a wrong result
    static const bool poison = getenv("HGPU_POISON") && getenv("HGPU_POISON")[0] == '1';
    if (poison && !pinned) cudaMemset(*p, 0xCD, ncap);
    return HGPU_OK;
}
int hgpu_ensure_scratch(hgpu_ctx *c, size_t b) { return grow(&c->d_scratch, &c->d_scratch_cap, b, false); }
int hgpu_ensure_stage(hgpu_ctx *c, size_t b)   { return grow(&c->d_stage, &c->d_stage_cap, b, false); }
int hgpu_ensure_mrec(hgpu_ctx *c, size_t b)    { return grow(&c->d_mrec, &c->d_mrec_cap, b, false); }
int hgpu_ensure_bam(hgpu_ctx *c, size_t b)     { return grow(&c->d_bam, &c->d_bam_cap, b, false); }
int hgpu_ensure_pinned(hgpu_ctx *c, size_t b)  { return grow(&c->h_pinned, &c->h_pinned_cap, b, true); }
uint32_t *hgpu_take_counter(hgpu_ctx *c, cudaStream_t st)
{
    uint32_t *p = c->d_counter + (c->next_counter++ & 63);
    if (hgpu_check(cudaMemsetAsync(p, 0, sizeof(uint32_t), st), "counter reset")) return nullptr;
    return p;
}

extern "C" hgpu_ctx *hgpu_create(int device)
{
    int ndev = 0;
    cudaError_t e = cudaGetDeviceCount(&ndev);
    if (e != cudaSuccess || ndev == 0) {
        hgpu_set_error("no CUDA device: %s", e == cudaSuccess ? "device count is 0" : cudaGetErrorString(e));
        cudaGetLastError();
        return nullptr;
    }
    if (device < 0) { if (hgpu_check(cudaGetDevice(&device), "cudaGetDevice")) return nullptr; }
    if (device >= ndev) { hgpu_set_error("device %d out of range (%d devices)", device, ndev); return nullptr; }
    if (hgpu_check(cudaSetDevice(device), "cudaSetDevice")) return nullptr;
    hgpu_ctx *c = (hgpu_ctx *)calloc(1, sizeof(hgpu_ctx));
    if (!c) return nullptr;
    c->device = device;
    auto fail = [c]() -> hgpu_ctx * { hgpu_destroy(c); return nullptr; };   // releases what was created so far
    cudaDeviceProp prop;
    if (hgpu_check(cudaGetDeviceProperties(&prop, device), "cudaGetDeviceProperties")) return fail();
    c->sm_count = prop.multiProcessorCount;
    if (hgpu_check(cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking), "stream")) return fail();
    for (int i = 0; i < 2; i++)
        if (hgpu_check(cudaStreamCreateWithFlags(&c->copy_stream[i], cudaStreamNonBlocking), "stream")) return fail();
    for (int i = 0; i < 8; i++)
        if (hgpu_check(cudaEventCreateWithFlags(&c->ev[i], cudaEventDisableTiming), "event")) return fail();
    if (hgpu_check(cudaMalloc((void **)&c->d_counter, 64 * sizeof(uint32_t)), "counter")) return fail();
    cudaMemset(c->d_counter, 0, 64 * sizeof(uint32_t));
    return c;
}

extern "C" void hgpu_destroy(hgpu_ctx *c)
{
    if (!c) return;
    cudaSetDevice(c->device);
    cudaDeviceSynchronize();
    if (c->d_scratch) cudaFree(c->d_scratch);
    if (c->d_stage) cudaFree(c->d_stage);
    if (c->d_mrec) cudaFree(c->d_mrec);
    if (c->d_bam) cudaFree(c->d_bam);
    if (c->h_pinned) cudaFreeHost(c->h_pinned);
    if (c->d_counter) cudaFree(c->d_counter);
    // (a context that hgpu_create gave up on has only some of its streams and events)
    if (c->stream) cudaStreamDestroy(c->stream);
    for (int i = 0; i < 2; i++) if (c->copy_stream[i]) cudaStreamDestroy(c->copy_stream[i]);
    for (int i = 0; i < 8; i++) if (c->ev[i]) cudaEventDestroy(c->ev[i]);
    free(c);
}

// ------------------------------------------------------------------------------------------ BGZF

extern "C" int hgpu_bgzf_inflate_batch_dev(hgpu_ctx *ctx, const uint8_t *d_in, const uint64_t *d_in_off,
        const uint32_t *d_in_len, uint32_t n, uint8_t *d_out, const uint64_t *d_out_off,
        const uint32_t *d_out_cap, uint32_t *d_out_len, int32_t *d_status, void *stream)
{
    if (!ctx) { hgpu_set_error("null context"); return HGPU_ERR_ARG; }
    return hgpu_launch_bgzf_inflate(ctx, d_in, d_in_off, d_in_len, n, d_out, d_out_off, d_out_cap,
                                    d_out_len, d_status, stream ? (cudaStream_t)stream : ctx->stream);
}

static int bgzf_check_header(const uint8_t *h)
{
    if (h[0] != 31 || h[1] != 139 || h[2] != 8) return -2;
    return ((h[3] & 4) && (h[10] | h[11] << 8) == 6 && h[12] == 'B' && h[13] == 'C'
            && (h[14] | h[15] << 8) == 2) ? 0 : -1;
}

extern "C" long hgpu_bgzf_scan(const uint8_t *file, uint64_t flen, uint64_t *off, uint32_t *len,
                               uint32_t *isize, long cap)
{
    uint64_t p = 0;
    long n = 0;
    while (p < flen) {
        if (flen - p < 18 || bgzf_check_header(file + p) != 0) return -1 - n;
        uint32_t bl = (uint32_t)(file[p + 16] | file[p + 17] << 8) + 1;
        if (bl < 26 || p + bl > flen) return -1 - n;
        if (n < cap) {
            if (off) off[n] = p;
            if (len) len[n] = bl;
            if (isize) {
                const uint8_t *f = file + p + bl - 4;
                isize[n] = f[0] | f[1] << 8 | f[2] << 16 | (uint32_t)f[3] << 24;
            }
        }
        n++;
        p += bl;
    }
    return n;
}

// ---- .gzi / uncompressed-offset <-> virtual-offset arithmetic over a scanned file (bgzf.c:2336-2621) ----
// The GPU paths deliver a file's blocks packed back to back, so "where is uncompressed byte u" is index
// arithmetic over the scan table: the same table bgzf_index_build_init / bgzf_index_add_block keep and
// bgzf_index_dump writes (one {compressed address, uncompressed address} pair per block start but the first).
// terminating = 1: the table a READER builds (bgzf_index_build_init + reading to the end, `bgzip -r`): every block start
// but the first, the EOF marker's included ("one extra record when indexing files opened for reading", :2387-2389).
// terminating = 0: the table a WRITER builds (`bgzip -i`, bgzf_flush :1976-1979): one pair per non-empty block it wrote.
extern "C" long hgpu_bgzf_gzi_entries(const uint64_t *off, const uint32_t *isize, long n, int terminating,
                                      uint64_t *caddr, uint64_t *uaddr, long cap)
{
    if (n < 0 || (n && (!off || !isize))) { hgpu_set_error("bad argument"); return -1; }
    uint64_t u = 0;
    long k = 0;
    for (long i = 0; i < n; i++) {
        if (i > 0 && (terminating || isize[i])) { if (k < cap) { if (caddr) caddr[k] = off[i]; if (uaddr) uaddr[k] = u; } k++; }
        u += isize[i];
    }
    return k;
}

// serialised form (bgzf_index_dump_hfile :2385-2415): u64 count, then count x {u64 caddr, u64 uaddr}, little endian
extern "C" long hgpu_bgzf_gzi_dump(const uint64_t *caddr, const uint64_t *uaddr, long n, uint8_t *out, size_t cap)
{
    const size_t need = 8 + (size_t)n * 16;
    if (n < 0 || (n && (!caddr || !uaddr))) { hgpu_set_error("bad argument"); return -1; }
    if (!out || cap < need) return (long)need;
    auto put = [&](size_t at, uint64_t v) { for (int b = 0; b < 8; b++) out[at + b] = (uint8_t)(v >> (8 * b)); };
    put(0, (uint64_t)n);
    for (long i = 0; i < n; i++) { put(8 + (size_t)i * 16, caddr[i]); put(16 + (size_t)i * 16, uaddr[i]); }
    return (long)need;
}

// bgzf_useek (:2540-2608): the virtual offset (block address << 16 | offset in the block) of uncompressed offset u.
// The block is the last one whose uncompressed address is <= u (entry -1 = the first block at {0, 0}).
extern "C" uint64_t hgpu_bgzf_useek(const uint64_t *caddr, const uint64_t *uaddr, long n, uint64_t u)
{
    long lo = 0, hi = n - 1;                                  // first entry with uaddr > u
    while (lo <= hi) { long mid = (lo + hi) / 2; if (u < uaddr[mid]) hi = mid - 1; else lo = mid + 1; }
    const long i = lo - 1;                                    // -1: the first block
    const uint64_t ca = i < 0 ? 0 : caddr[i], ua = i < 0 ? 0 : uaddr[i];
    return ca << 16 | ((u - ua) & 0xffffu);
}

// the inverse: uncompressed offset of a virtual offset, or (uint64)-1 if its block address is not a block start
extern "C" uint64_t hgpu_bgzf_utell(const uint64_t *caddr, const uint64_t *uaddr, long n, uint64_t voffset)
{
    const uint64_t ca = voffset >> 16;
    if (ca == 0) return voffset & 0xffffu;
    long lo = 0, hi = n - 1;
    while (lo <= hi) { long mid = (lo + hi) / 2; if (caddr[mid] < ca) lo = mid + 1; else if (caddr[mid] > ca) hi = mid - 1; else return uaddr[mid] + (voffset & 0xffffu); }
    return ~0ull;
}

// Pipelined whole-file inflate with host buffers.  Chunks of blocks flow through three streams
// (H2D copy, kernel, D2H copy each in stream order) so that transfers of neighbouring chunks
// overlap the kernel.
static int hgpu_bgzf_inflate_file_host_impl(hgpu_ctx *ctx, const uint8_t *file, uint64_t file_len,
                                           uint8_t *out, uint64_t out_cap, uint64_t *out_len, long *bad_block)
{
    if (!ctx || !file || !out_len) { hgpu_set_error("bad argument"); return HGPU_ERR_ARG; }
    if (bad_block) *bad_block = -1;
    if (hgpu_check(cudaSetDevice(ctx->device), "cudaSetDevice")) return HGPU_ERR_CUDA;
    long nb = hgpu_bgzf_scan(file, file_len, nullptr, nullptr, nullptr, 0);
    if (nb < 0) { if (bad_block) *bad_block = -1 - nb; hgpu_set_error("bad BGZF header at block %ld", -1 - nb); return HGPU_BGZF_ERR_HEADER; }
    *out_len = 0;
    if (nb == 0) return HGPU_OK;
    std::vector<uint64_t> off(nb), ooff(nb);
    std::vector<uint32_t> len(nb), isz(nb);
    hgpu_bgzf_scan(file, file_len, off.data(), len.data(), isz.data(), nb);
    uint64_t total = 0;
    for (long i = 0; i < nb; i++) {
        if (isz[i] > 65536u) { if (bad_block) *bad_block = i; hgpu_set_error("ISIZE > 64 KiB at block %ld", i); return HGPU_BGZF_ERR_ZLIB; }
        ooff[i] = total; total += isz[i];
    }
    if (total > out_cap) { hgpu_set_error("output needs %llu bytes, caller gave %llu", (unsigned long long)total, (unsigned long long)out_cap); return HGPU_ERR_ARG; }
    // device layout: [in file (+pad)] [out] [meta arrays]
    StageLayout L;
    const auto s_in = L.seg((size_t)file_len + 4), s_out = L.seg(total), s_off = L.seg(nb * 8), s_ooff = L.seg(nb * 8),
               s_len = L.seg(nb * 4), s_cap = L.seg(nb * 4), s_olen = L.seg(nb * 4), s_st = L.seg(nb * 4);
    int rc = hgpu_stage_ensure(ctx, L);
    if (rc) return rc;
    uint8_t *d_in = L.at(s_in), *d_out = L.at(s_out);
    uint64_t *d_off = L.at<uint64_t>(s_off), *d_ooff = L.at<uint64_t>(s_ooff);
    uint32_t *d_len = L.at<uint32_t>(s_len), *d_cap = L.at<uint32_t>(s_cap), *d_olen = L.at<uint32_t>(s_olen);
    int32_t *d_st = L.at<int32_t>(s_st);
    cudaStream_t s0 = ctx->stream;
    if (hgpu_h2d(d_off, off.data(), nb * 8, s0) || hgpu_h2d(d_ooff, ooff.data(), nb * 8, s0) ||
        hgpu_h2d(d_len, len.data(), nb * 4, s0) || hgpu_h2d(d_cap, isz.data(), nb * 4, s0)) return HGPU_ERR_CUDA;
    if (hgpu_check(cudaEventRecord(ctx->ev[0], s0), "event")) return HGPU_ERR_CUDA;
    // chunking: ~64 MiB of compressed input per chunk
    const uint64_t chunk_bytes = 64ull << 20;
    cudaStream_t st[3] = { ctx->stream, ctx->copy_stream[0], ctx->copy_stream[1] };
    for (int k = 1; k < 3; k++) if (hgpu_check(cudaStreamWaitEvent(st[k], ctx->ev[0], 0), "wait")) return HGPU_ERR_CUDA;
    long b0 = 0;
    int ci = 0;
    while (b0 < nb) {
        long b1 = b0;
        uint64_t start = off[b0], endp = start;
        while (b1 < nb && (endp - start < chunk_bytes)) { endp = off[b1] + len[b1]; b1++; }
        cudaStream_t s = st[ci % 3];
        if (hgpu_h2d(d_in + start, file + start, endp - start, s)) return HGPU_ERR_CUDA;
        rc = hgpu_launch_bgzf_inflate(ctx, d_in, d_off + b0, d_len + b0, (uint32_t)(b1 - b0), d_out, d_ooff + b0,
                                      d_cap + b0, d_olen + b0, d_st + b0, s);
        if (rc) return rc;
        uint64_t o0 = ooff[b0], o1 = (b1 < nb) ? ooff[b1] : total;
        if (out && hgpu_d2h(out + o0, d_out + o0, o1 - o0, s)) return HGPU_ERR_CUDA;
        b0 = b1;
        ci++;
    }
    std::vector<uint32_t> olen(nb);
    std::vector<int32_t> stv(nb);
    for (int k = 0; k < 3; k++) if (hgpu_check(cudaStreamSynchronize(st[k]), "sync")) return HGPU_ERR_CUDA;
    if (hgpu_check(cudaMemcpy(olen.data(), d_olen, nb * 4, cudaMemcpyDeviceToHost), "D2H meta")) return HGPU_ERR_CUDA;
    if (hgpu_check(cudaMemcpy(stv.data(), d_st, nb * 4, cudaMemcpyDeviceToHost), "D2H meta")) return HGPU_ERR_CUDA;
    // errors are reported in block order, like the result queue of bgzf_read_block (bgzf.c:1037-1044)
    bool ragged = false;
    for (long i = 0; i < nb; i++) {
        if (stv[i] != HGPU_OK) { if (bad_block) *bad_block = i; hgpu_set_error("block %ld: status %d", i, stv[i]); return stv[i]; }
        if (olen[i] != isz[i]) ragged = true;
    }
    if (ragged) {
        // a block inflated to fewer bytes than its ISIZE claims (htslib ignores ISIZE): close the gaps
        uint64_t w = 0;
        for (long i = 0; i < nb; i++) {
            if (w != ooff[i]) memmove(out + w, out + ooff[i], olen[i]);
            w += olen[i];
        }
        total = w;
    }
    *out_len = total;
    return HGPU_OK;
}

extern "C" int hgpu_bgzf_inflate_file_host(hgpu_ctx *ctx, const uint8_t *file, uint64_t file_len,
                                           uint8_t *out, uint64_t out_cap, uint64_t *out_len, long *bad_block)
{
    return hgpu_abi_call([&] { return hgpu_bgzf_inflate_file_host_impl(ctx, file, file_len, out, out_cap, out_len, bad_block); });
}

// Multi-GPU sharding rule (SURVEY.md §8e): unit i goes to rank floor(i*world/n), i.e. rank r owns
// the contiguous range [ceil(r*n/world), ceil((r+1)*n/world)), so every rank's output is one
// contiguous byte range of the decompressed stream and no data-path collective is needed.
extern "C" int hgpu_shard_range(uint64_t n_units, const uint32_t *unit_out_len, int world, int rank,
                                uint64_t *first, uint64_t *count, uint64_t *out_base)
{
    if (world < 1 || rank < 0 || rank >= world || !first || !count) { hgpu_set_error("bad shard arguments"); return HGPU_ERR_ARG; }
    uint64_t lo = ((uint64_t)rank * n_units + world - 1) / world, hi = ((uint64_t)(rank + 1) * n_units + world - 1) / world;
    if (hi > n_units) hi = n_units;
    if (lo > hi) lo = hi;
    *first = lo; *count = hi - lo;
    if (out_base) {
        uint64_t b = 0;
        if (unit_out_len) for (uint64_t i = 0; i < lo; i++) b += unit_out_len[i];
        *out_base = b;
    }
    return HGPU_OK;
}

// Downloads the n slots [off[i], off[i] + len[i]) of d_out into out at the same offsets, one copy per run of slots in
// address order.  A slot that starts less than max_gap bytes past the end of the run joins it, and the gap is copied
// too: max_gap = 1 joins only slots that touch or overlap, so nothing of out outside the slots is written.
static int hgpu_d2h_slot_runs(uint8_t *out, const uint8_t *d_out, const uint64_t *off, const uint32_t *len, uint32_t n,
                              uint64_t max_gap, cudaStream_t s)
{
    std::vector<uint32_t> ord(n);
    for (uint32_t i = 0; i < n; i++) ord[i] = i;
    std::sort(ord.begin(), ord.end(), [&](uint32_t a, uint32_t b) { return off[a] < off[b]; });
    uint64_t r0 = off[ord[0]], r1 = r0 + len[ord[0]];
    for (uint32_t k = 1; k <= n; k++) {
        const bool more = k < n;
        if (more && off[ord[k]] < r1 + max_gap) { const uint64_t e = off[ord[k]] + len[ord[k]]; if (e > r1) r1 = e; continue; }
        if (hgpu_d2h(out + r0, d_out + r0, r1 - r0, s)) return HGPU_ERR_CUDA;
        if (more) { r0 = off[ord[k]]; r1 = r0 + len[ord[k]]; }
    }
    return HGPU_OK;
}

// A batch of individual blocks with HOST buffers (the thread-pool job seam, INTEGRATION.md B3):
// H2D of the gathered compressed blocks, one launch, D2H of the slots and the per-block results.
static int hgpu_bgzf_inflate_blocks_host_impl(hgpu_ctx *ctx, const uint8_t *in, const uint64_t *in_off,
        const uint32_t *in_len, uint32_t n, uint8_t *out, const uint64_t *out_off, const uint32_t *out_cap,
        uint32_t *out_len, int32_t *status)
{
    if (!ctx || (n && (!in || !in_off || !in_len || !out || !out_off || !out_cap))) { hgpu_set_error("bad argument"); return HGPU_ERR_ARG; }
    if (n == 0) return HGPU_OK;
    if (hgpu_check(cudaSetDevice(ctx->device), "cudaSetDevice")) return HGPU_ERR_CUDA;
    const uint64_t in_end = hgpu_slots_end(in_off, in_len, n), out_end = hgpu_slots_end(out_off, out_cap, n);
    StageLayout L;
    const auto s_in = L.seg(in_end + 4), s_out = L.seg(out_end), s_ioff = L.seg(n * 8), s_ooff = L.seg(n * 8),
               s_ilen = L.seg(n * 4), s_cap = L.seg(n * 4), s_got = L.seg(n * 4), s_st = L.seg(n * 4);
    int rc = hgpu_stage_ensure(ctx, L);
    if (rc) return rc;
    cudaStream_t s = ctx->stream;
    if (hgpu_h2d(L.at(s_in), in, in_end, s) || hgpu_h2d(L.at(s_ioff), in_off, n * 8, s) || hgpu_h2d(L.at(s_ooff), out_off, n * 8, s) ||
        hgpu_h2d(L.at(s_ilen), in_len, n * 4, s) || hgpu_h2d(L.at(s_cap), out_cap, n * 4, s)) return HGPU_ERR_CUDA;
    rc = hgpu_launch_bgzf_inflate(ctx, L.at(s_in), L.at<uint64_t>(s_ioff), L.at<uint32_t>(s_ilen), n, L.at(s_out), L.at<uint64_t>(s_ooff),
                                  L.at<uint32_t>(s_cap), L.at<uint32_t>(s_got), L.at<int32_t>(s_st), s);
    if (rc) return rc;
    // only the slots come back: runs of slots that touch (the usual 64 KiB stride is one run) are one copy each,
    // and nothing of the caller's buffer outside the slots is written
    if (hgpu_d2h_slot_runs(out, L.at(s_out), out_off, out_cap, n, 1, s)) return HGPU_ERR_CUDA;
    std::vector<uint32_t> got(n);
    std::vector<int32_t> st(n);
    if (hgpu_d2h(got.data(), L.at(s_got), n * 4, s) || hgpu_d2h(st.data(), L.at(s_st), n * 4, s)) return HGPU_ERR_CUDA;
    if (hgpu_check(cudaStreamSynchronize(s), "sync")) return HGPU_ERR_CUDA;
    for (uint32_t i = 0; i < n; i++) { if (out_len) out_len[i] = got[i]; if (status) status[i] = st[i]; }
    return HGPU_OK;
}

extern "C" int hgpu_bgzf_inflate_blocks_host(hgpu_ctx *ctx, const uint8_t *in, const uint64_t *in_off,
        const uint32_t *in_len, uint32_t n, uint8_t *out, const uint64_t *out_off, const uint32_t *out_cap,
        uint32_t *out_len, int32_t *status)
{
    return hgpu_abi_call([&] { return hgpu_bgzf_inflate_blocks_host_impl(ctx, in, in_off, in_len, n, out, out_off, out_cap, out_len, status); });
}

// A batch of bgzf_job-shaped blocks: every block has its OWN host buffers (bgzf.c:92-101 keeps
// comp_data / uncomp_data inside each pooled job).  Gather into pinned staging, one H2D, one
// launch, one D2H, scatter.  ctx == NULL uses the process-wide context of the reference-named
// shims (one batch at a time).  uncomp_len[i]: in = room in uncomp[i], out = inflated length.
static int hgpu_bgzf_inflate_jobs_host_impl(hgpu_ctx *ctx, uint32_t n, const uint8_t *const *comp, const uint32_t *comp_len,
                                           uint8_t *const *uncomp, uint32_t *uncomp_len, int32_t *status)
{
    if (n && (!comp || !comp_len || !uncomp || !uncomp_len || !status)) { hgpu_set_error("bad argument"); return HGPU_ERR_ARG; }
    if (n == 0) return HGPU_OK;
    std::unique_lock<std::mutex> lock(g_shim_mu, std::defer_lock);
    if (!ctx) {
        lock.lock();
        ctx = shim_ctx();
        if (!ctx) return HGPU_ERR_CUDA;
    }
    if (hgpu_check(cudaSetDevice(ctx->device), "cudaSetDevice")) return HGPU_ERR_CUDA;
    std::vector<uint64_t> ioff(n), ooff(n);
    std::vector<uint32_t> cap(n);
    uint64_t in_end = 0, out_end = 0;
    for (uint32_t i = 0; i < n; i++) {
        ioff[i] = in_end; in_end += ((uint64_t)comp_len[i] + 15) & ~(uint64_t)15;
        cap[i] = uncomp_len[i] > 65536u ? 65536u : uncomp_len[i];
        ooff[i] = out_end; out_end += ((uint64_t)cap[i] + 15) & ~(uint64_t)15;
    }
    // one layout for the pinned and the device image; the job arrays travel in one copy each way, so they are in the
    // order the copies need: [ioff ooff ilen cap] up, [got st] down
    StageLayout L;
    const auto s_in = L.seg(in_end + 4), s_out = L.seg(out_end), s_ioff = L.seg(n * 8), s_ooff = L.seg(n * 8),
               s_ilen = L.seg(n * 4), s_cap = L.seg(n * 4), s_got = L.seg(n * 4), s_st = L.seg(n * 4);
    int rc = hgpu_stage_ensure(ctx, L);
    if (rc) return rc;
    rc = hgpu_ensure_pinned(ctx, L.total);
    if (rc) return rc;
    uint8_t *const h = ctx->h_pinned;
    for (uint32_t i = 0; i < n; i++) memcpy(h + s_in.off + ioff[i], comp[i], comp_len[i]);
    memcpy(h + s_ioff.off, ioff.data(), n * 8); memcpy(h + s_ooff.off, ooff.data(), n * 8);
    memcpy(h + s_ilen.off, comp_len, n * 4); memcpy(h + s_cap.off, cap.data(), n * 4);
    const uint32_t *hm_got = (const uint32_t *)(h + s_got.off);
    const int32_t *hm_st = (const int32_t *)(h + s_st.off);
    cudaStream_t s = ctx->stream;
    if (hgpu_h2d(L.at(s_in), h + s_in.off, in_end, s) ||
        hgpu_h2d(L.at(s_ioff), h + s_ioff.off, s_cap.off + s_cap.bytes - s_ioff.off, s)) return HGPU_ERR_CUDA;
    rc = hgpu_launch_bgzf_inflate(ctx, L.at(s_in), L.at<uint64_t>(s_ioff), L.at<uint32_t>(s_ilen), n, L.at(s_out), L.at<uint64_t>(s_ooff),
                                  L.at<uint32_t>(s_cap), L.at<uint32_t>(s_got), L.at<int32_t>(s_st), s);
    if (rc) return rc;
    if (hgpu_d2h(h + s_out.off, L.at(s_out), out_end, s) ||
        hgpu_d2h(h + s_got.off, L.at(s_got), s_st.off + s_st.bytes - s_got.off, s)) return HGPU_ERR_CUDA;
    if (hgpu_check(cudaStreamSynchronize(s), "sync")) return HGPU_ERR_CUDA;
    for (uint32_t i = 0; i < n; i++) {
        status[i] = hm_st[i];
        uncomp_len[i] = hm_st[i] == HGPU_OK ? hm_got[i] : 0;
        if (hm_st[i] == HGPU_OK) memcpy(uncomp[i], h + s_out.off + ooff[i], hm_got[i]);
    }
    return HGPU_OK;
}

extern "C" int hgpu_bgzf_inflate_jobs_host(hgpu_ctx *ctx, uint32_t n, const uint8_t *const *comp, const uint32_t *comp_len,
                                           uint8_t *const *uncomp, uint32_t *uncomp_len, int32_t *status)
{
    return hgpu_abi_call([&] { return hgpu_bgzf_inflate_jobs_host_impl(ctx, n, comp, comp_len, uncomp, uncomp_len, status); });
}

// zlib-compatible combine on the host side of the ABI: crc(A||B) from crc(A), crc(B), |B|
static uint32_t h_multmodp(uint32_t a, uint32_t b)
{
    uint32_t p = 0;
    for (uint32_t m = 1u << 31; m; m >>= 1) {
        if (a & m) p ^= b;
        b = (b & 1) ? (b >> 1) ^ 0xEDB88320u : b >> 1;
    }
    return p;
}
static uint32_t h_xpow_bytes(uint64_t n)
{
    uint32_t p = 1u << 31, sq = 1u << 23;
    while (n) { if (n & 1) p = h_multmodp(sq, p); sq = h_multmodp(sq, sq); n >>= 1; }
    return p;
}

// *status (may be NULL) = HGPU_OK or the error; on error the incoming crc is returned unchanged AND
// hgpu_last_error() is set — a caller that cannot take a status must check hgpu_crc32_failed().
static thread_local int g_crc_failed = 0;
extern "C" int hgpu_crc32_failed(void) { return g_crc_failed; }
static uint32_t crc32_impl(hgpu_ctx *ctx, uint32_t crc, const void *buf, size_t len, int *status)
{
    int dummy;
    if (!status) status = &dummy;
    *status = HGPU_OK;
    if (!ctx) { hgpu_set_error("bad argument"); *status = HGPU_ERR_ARG; return crc; }
    if (len == 0 || !buf) return crc;
    *status = HGPU_ERR_CUDA;
    if (hgpu_check(cudaSetDevice(ctx->device), "cudaSetDevice")) return crc;
    const size_t chunk = 1u << 20;
    size_t nchunk = (len + chunk - 1) / chunk;
    StageLayout L;
    const auto s_data = L.seg(len), s_part = L.seg(nchunk * 4);
    if (hgpu_stage_ensure(ctx, L)) { *status = HGPU_ERR_NOMEM; return crc; }
    uint8_t *d = L.at(s_data);
    uint32_t *d_part = L.at<uint32_t>(s_part);
    if (hgpu_h2d(d, buf, len, ctx->stream)) return crc;
    if (hgpu_launch_crc32(ctx, d, len, d_part, nullptr, 0, ctx->stream)) return crc;
    std::vector<uint32_t> part(nchunk);
    if (hgpu_d2h(part.data(), d_part, nchunk * 4, ctx->stream)) return crc;
    if (hgpu_check(cudaStreamSynchronize(ctx->stream), "sync")) return crc;
    for (size_t i = 0; i < nchunk; i++) {
        size_t n = (i + 1 == nchunk) ? len - i * chunk : chunk;
        crc = h_multmodp(h_xpow_bytes(n), crc) ^ part[i];
    }
    *status = HGPU_OK;
    return crc;
}

extern "C" uint32_t hgpu_crc32(hgpu_ctx *ctx, uint32_t crc, const void *buf, size_t len)
{
    int st = HGPU_OK;
    try { crc = crc32_impl(ctx, crc, buf, len, &st); }
    catch (...) { hgpu_set_error("out of host memory"); st = HGPU_ERR_NOMEM; }
    g_crc_failed = st != HGPU_OK;
    return crc;
}

// ------------------------------------------------------------------------------------------ rANS

extern "C" int hgpu_rans_nx16_decode_batch_dev(hgpu_ctx *ctx, const uint8_t *d_in, const uint64_t *d_in_off,
        const uint32_t *d_in_len, uint32_t n, uint8_t *d_out, const uint64_t *d_out_off,
        const uint32_t *d_out_len, uint32_t *d_got_len, int32_t *d_status, uint32_t max_out_len, void *stream)
{
    if (!ctx) { hgpu_set_error("null context"); return HGPU_ERR_ARG; }
    return hgpu_launch_rans_nx16(ctx, d_in, d_in_off, d_in_len, n, d_out, d_out_off, d_out_len, d_got_len,
                                 d_status, max_out_len, stream ? (cudaStream_t)stream : ctx->stream);
}

static int hgpu_rans_nx16_decode_batch_host_impl(hgpu_ctx *ctx, const uint8_t *in, const uint64_t *in_off,
        const uint32_t *in_len, uint32_t n, uint8_t *out, const uint64_t *out_off, const uint32_t *out_len,
        uint32_t *got_len, int32_t *status)
{
    if (!ctx || (n && (!in || !in_off || !in_len || !out || !out_off || !out_len))) { hgpu_set_error("bad argument"); return HGPU_ERR_ARG; }
    if (n == 0) return HGPU_OK;
    if (hgpu_check(cudaSetDevice(ctx->device), "cudaSetDevice")) return HGPU_ERR_CUDA;
    const uint64_t in_end = hgpu_slots_end(in_off, in_len, n), out_end = hgpu_slots_end(out_off, out_len, n);
    uint32_t max_out = 0;
    for (uint32_t i = 0; i < n; i++) if (out_len[i] > max_out) max_out = out_len[i];
    StageLayout L;
    const auto s_in = L.seg(in_end + 4), s_out = L.seg(out_end), s_ioff = L.seg(n * 8), s_ooff = L.seg(n * 8),
               s_ilen = L.seg(n * 4), s_olen = L.seg(n * 4), s_got = L.seg(n * 4), s_st = L.seg(n * 4);
    int rc = hgpu_stage_ensure(ctx, L);
    if (rc) return rc;
    cudaStream_t s = ctx->stream;
    if (hgpu_h2d(L.at(s_in), in, in_end, s) || hgpu_h2d(L.at(s_ioff), in_off, n * 8, s) || hgpu_h2d(L.at(s_ooff), out_off, n * 8, s) ||
        hgpu_h2d(L.at(s_ilen), in_len, n * 4, s) || hgpu_h2d(L.at(s_olen), out_len, n * 4, s)) return HGPU_ERR_CUDA;
    rc = hgpu_launch_rans_nx16(ctx, L.at(s_in), L.at<uint64_t>(s_ioff), L.at<uint32_t>(s_ilen), n, L.at(s_out), L.at<uint64_t>(s_ooff),
                               L.at<uint32_t>(s_olen), L.at<uint32_t>(s_got), L.at<int32_t>(s_st), max_out, s);
    if (rc) return rc;
    // only the slots come back, in runs: slots that touch, or are separated by alignment padding (< 16 bytes, which
    // may be overwritten), travel in one copy
    if (hgpu_d2h_slot_runs(out, L.at(s_out), out_off, out_len, n, 16, s)) return HGPU_ERR_CUDA;
    std::vector<uint32_t> got(n);
    std::vector<int32_t> st(n);
    if (hgpu_d2h(got.data(), L.at(s_got), n * 4, s) || hgpu_d2h(st.data(), L.at(s_st), n * 4, s)) return HGPU_ERR_CUDA;
    if (hgpu_check(cudaStreamSynchronize(s), "sync")) return HGPU_ERR_CUDA;
    for (uint32_t i = 0; i < n; i++) { if (got_len) got_len[i] = got[i]; if (status) status[i] = st[i]; }
    return HGPU_OK;
}

extern "C" int hgpu_rans_nx16_decode_batch_host(hgpu_ctx *ctx, const uint8_t *in, const uint64_t *in_off,
        const uint32_t *in_len, uint32_t n, uint8_t *out, const uint64_t *out_off, const uint32_t *out_len,
        uint32_t *got_len, int32_t *status)
{
    return hgpu_abi_call([&] { return hgpu_rans_nx16_decode_batch_host_impl(ctx, in, in_off, in_len, n, out, out_off, out_len, got_len, status); });
}

// ------------------------------------------------------------------------------------------ shims

static hgpu_ctx *g_shim_ctx;

static hgpu_ctx *shim_ctx()
{
    if (!g_shim_ctx) g_shim_ctx = hgpu_create(-1);
    return g_shim_ctx;
}
// the same process-wide context and lock for the reference-named shims that live in other files
void hgpu_shim_lock() { g_shim_mu.lock(); }
void hgpu_shim_unlock() { g_shim_mu.unlock(); }
hgpu_ctx *hgpu_shim_ctx() { return shim_ctx(); }

extern "C" unsigned char *rans_uncompress_to_4x16(unsigned char *in, unsigned int in_size,
                                                  unsigned char *out, unsigned int *out_size)
{
    if (!in || in_size == 0 || !out_size) return nullptr;
    // size discovery exactly as the reference does it (rANS_static4x16pr.c:1594-1612, :1684-1711)
    unsigned int ulen = 0;
    bool have = false;
    if (in[0] & 0x08) { hgpu_var_get_u32_bounded(in + 1, in + in_size, &ulen); have = true; }
    else if (!(in[0] & 0x10)) { hgpu_var_get_u32_bounded(in + 1, in + in_size, &ulen); have = true; }
    unsigned char *alloc = nullptr;
    if (!out) {
        if (!have || ulen >= 0x7fffffffu) return nullptr;       // NOSZ needs a caller buffer
        alloc = out = (unsigned char *)malloc(ulen ? ulen : 1);
        if (!out) return nullptr;
        *out_size = ulen;
    }
    if (have) {
        if ((in[0] & 0x08) ? ulen != *out_size : *out_size < ulen) { free(alloc); return nullptr; }
    } else
        ulen = *out_size;
    std::lock_guard<std::mutex> lock(g_shim_mu);
    hgpu_ctx *ctx = shim_ctx();
    if (!ctx) { free(alloc); return nullptr; }
    uint64_t ioff = 0, ooff = 0;
    uint32_t ilen = in_size, olen = ulen, got = 0;
    int32_t st = 0;
    int rc = hgpu_rans_nx16_decode_batch_host(ctx, in, &ioff, &ilen, 1, out, &ooff, &olen, &got, &st);
    if (rc != HGPU_OK || st != HGPU_OK) { free(alloc); return nullptr; }
    *out_size = got;
    return out;
}

extern "C" unsigned char *rans_uncompress_4x16(unsigned char *in, unsigned int in_size, unsigned int *out_size)
{
    return rans_uncompress_to_4x16(in, in_size, nullptr, out_size);
}

extern "C" uint32_t hts_crc32(uint32_t crc, const void *buf, size_t len)
{
    std::lock_guard<std::mutex> lock(g_shim_mu);
    hgpu_ctx *ctx = shim_ctx();
    if (!ctx) { fprintf(stderr, "htsgpu: hts_crc32 without a CUDA device: %s\n", hgpu_last_error()); abort(); }
    // hts_crc32 has no error channel (bgzf.c:620): a checksum that was not computed must not be returned as one
    const uint32_t r = hgpu_crc32(ctx, crc, buf, len);
    if (hgpu_crc32_failed()) { fprintf(stderr, "htsgpu: hts_crc32 failed on the device: %s\n", hgpu_last_error()); abort(); }
    return r;
}

// bgzf_compress (bgzf.c:624-683): one block, host pointers
extern "C" int bgzf_compress(void *dst, size_t *dlen, const void *src, size_t slen, int level)
{
    static const uint8_t eof_block[28] = {0x1f, 0x8b, 8, 4, 0, 0, 0, 0, 0, 0xff, 6, 0, 'B', 'C', 2, 0, 0x1b, 0, 3, 0, 0, 0, 0, 0, 0, 0, 0, 0};
    if (!dst || !dlen || (slen && !src)) return -1;
    if (slen == 0) {                                  // bgzf.c:566: the EOF marker
        if (*dlen < 28) return -1;
        memcpy(dst, eof_block, 28);
        *dlen = 28;
        return 0;
    }
    if (slen > 65280) return -1;
    std::lock_guard<std::mutex> lock(g_shim_mu);
    hgpu_ctx *ctx = shim_ctx();
    if (!ctx) return -1;
    if (cudaSetDevice(ctx->device) != cudaSuccess) return -1;
    StageLayout L;
    const auto s_in = L.seg(slen + 4), s_out = L.seg(65536), s_off = L.seg(16) /* {in_off, out_off} */, s_len = L.seg(4), s_ol = L.seg(4),
               s_st = L.seg(4);
    if (hgpu_stage_ensure(ctx, L)) return -1;
    uint8_t *d_in = L.at(s_in), *d_out = L.at(s_out);
    uint64_t *d_off = L.at<uint64_t>(s_off);
    uint32_t *d_len = L.at<uint32_t>(s_len), *d_ol = L.at<uint32_t>(s_ol);
    int32_t *d_st = L.at<int32_t>(s_st);
    uint64_t offs[2] = {0, 0};
    uint32_t len32 = (uint32_t)slen, got = 0;
    int32_t st = 0;
    cudaStream_t s = ctx->stream;
    if (hgpu_h2d(d_in, src, slen, s) || hgpu_h2d(d_off, offs, 16, s) || hgpu_h2d(d_len, &len32, 4, s)) return -1;
    if (hgpu_bgzf_compress_batch_dev(ctx, d_in, d_off, d_len, 1, level < 0 ? 6 : level, d_out, d_off + 1, d_ol, d_st, s)) return -1;
    if (hgpu_d2h(&got, d_ol, 4, s) || hgpu_d2h(&st, d_st, 4, s)) return -1;
    if (cudaStreamSynchronize(s) != cudaSuccess) return -1;
    if (st != HGPU_OK || got == 0 || got > *dlen) return -1;
    if (cudaMemcpy(dst, d_out, got, cudaMemcpyDeviceToHost) != cudaSuccess) return -1;
    *dlen = got;
    return 0;
}
