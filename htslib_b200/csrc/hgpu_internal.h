// Internal declarations shared by the kernels and the C-ABI layer of libhtsgpu.so.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stddef.h>
#include <new>
#include <type_traits>
#include "../../include/htsgpu.h"
#include "stage_layout.h"

#define HGPU_WARP 32

struct hgpu_ctx {
    int device;
    int sm_count;
    cudaStream_t stream;          // default stream for _host entry points
    cudaStream_t copy_stream[2];  // H2D / D2H overlap in the pipelined host paths
    cudaEvent_t ev[8];
    // device scratch, grown on demand
    uint8_t *d_scratch;  size_t d_scratch_cap;     // rANS per-warp scratch
    uint8_t *d_mrec;     size_t d_mrec_cap;        // inflate match-record scratch
    uint8_t *d_bam;      size_t d_bam_cap;         // BAM index / scan scratch
    uint8_t *d_stage;    size_t d_stage_cap;     // device staging for _host entry points
    uint8_t *h_pinned;   size_t h_pinned_cap;    // pinned host staging
    uint32_t *d_counter;                          // 64 work-queue counters, handed out round-robin
    uint32_t next_counter;
};

// error plumbing (hgpu_api.cu)
void hgpu_set_error(const char *fmt, ...);
int  hgpu_check(cudaError_t e, const char *what);
void hgpu_count_launch(int n = 1);
int  hgpu_ensure_scratch(hgpu_ctx *ctx, size_t bytes);
int  hgpu_ensure_stage(hgpu_ctx *ctx, size_t bytes);
int  hgpu_ensure_mrec(hgpu_ctx *ctx, size_t bytes);
int  hgpu_ensure_bam(hgpu_ctx *ctx, size_t bytes);
int  hgpu_ensure_pinned(hgpu_ctx *ctx, size_t bytes);
// process-wide context of the reference-named shims (one batch at a time); call between lock/unlock
void hgpu_shim_lock();
void hgpu_shim_unlock();
hgpu_ctx *hgpu_shim_ctx();
struct ShimLock { ShimLock() { hgpu_shim_lock(); } ~ShimLock() { hgpu_shim_unlock(); } };
// a zeroed (stream-ordered) work counter; slots rotate so launches in flight on different streams never share one
uint32_t *hgpu_take_counter(hgpu_ctx *ctx, cudaStream_t st);

// Grows ctx->d_stage to L.total and binds L to it.  *moved (may be NULL): the buffer was reallocated, so whatever was
// uploaded into it before this call is gone (a new allocation may land on the old address: capacities are compared).
inline int hgpu_stage_ensure(hgpu_ctx *ctx, StageLayout &L, bool *moved = nullptr)
{
    const size_t cap = ctx->d_stage_cap;
    const int rc = hgpu_ensure_stage(ctx, L.total);
    if (moved) *moved = ctx->d_stage_cap != cap;
    L.base = ctx->d_stage;
    return rc;
}

// Checked stream-ordered copies: HGPU_OK, or HGPU_ERR_CUDA with the error text set.  Zero-byte copies are skipped.
inline int hgpu_h2d(void *dst, const void *src, size_t n, cudaStream_t s)
{
    return n ? hgpu_check(cudaMemcpyAsync(dst, src, n, cudaMemcpyHostToDevice, s), "H2D") : HGPU_OK;
}
inline int hgpu_d2h(void *dst, const void *src, size_t n, cudaStream_t s)
{
    return n ? hgpu_check(cudaMemcpyAsync(dst, src, n, cudaMemcpyDeviceToHost, s), "D2H") : HGPU_OK;
}
inline int hgpu_memset(void *dst, int v, size_t n, cudaStream_t s)
{
    return n ? hgpu_check(cudaMemsetAsync(dst, v, n, s), "memset") : HGPU_OK;
}

// max(off[i] + len[i]): how far into a caller's buffer a batch of slots reaches
inline uint64_t hgpu_slots_end(const uint64_t *off, const uint32_t *len, uint32_t n)
{
    uint64_t e = 0;
    for (uint32_t i = 0; i < n; i++) if (off[i] + len[i] > e) e = off[i] + len[i];
    return e;
}

// No C++ exception may cross the C ABI (host buffers are sized from untrusted input: std::bad_alloc).  Every extern "C"
// entry point that allocates runs its body through this; the codes are what that entry point documents for each case.
template <class F> using hgpu_result_t = std::invoke_result_t<F &>;
template <class F>
hgpu_result_t<F> hgpu_abi_call(F &&f, hgpu_result_t<F> on_nomem = HGPU_ERR_NOMEM, hgpu_result_t<F> on_other = HGPU_ERR_CUDA)
{
    try {
        return f();
    } catch (const std::bad_alloc &) {
        hgpu_set_error("out of host memory");
        return on_nomem;
    } catch (...) {
        hgpu_set_error("internal error");
        return on_other;
    }
}

// The two readers of htscodecs' big-endian 7-bit varints (varint.h).  They differ on truncated and over-long input,
// and each caller keeps the one whose result it has always had.
// var_get_u32 as the reference has it (varint.h:267-299): six or more bytes left -> up to six read without a bound check.
inline int hgpu_var_get_u32(const uint8_t *p, const uint8_t *end, uint32_t *v)
{
    const uint8_t *s = p;
    uint32_t acc = 0;
    uint8_t c;
    if (end - p >= 6) {
        int n = 5;
        do { c = *p++; acc = (acc << 7) | (c & 0x7f); } while ((c & 0x80) && n-- > 0);
    } else {
        if (p >= end) { *v = 0; return 0; }
        if (*p < 128) { *v = *p; return 1; }
        do { c = *p++; acc = (acc << 7) | (c & 0x7f); } while ((c & 0x80) && p < end);
    }
    *v = acc;
    return (int)(p - s);
}
// The groups var_put_u32 writes (varint.h:206), every byte checked against end, at most six read.
inline int hgpu_var_get_u32_bounded(const uint8_t *p, const uint8_t *end, uint32_t *v)
{
    const uint8_t *s = p;
    uint32_t acc = 0, c;
    int n = 0;
    do { if (p >= end) { *v = acc; return (int)(p - s); } c = *p++; acc = (acc << 7) | (c & 0x7f); } while ((c & 0x80) && ++n < 6);
    *v = acc;
    return (int)(p - s);
}

// kernel launchers (one per .cu)
int hgpu_launch_rans_nx16(hgpu_ctx *ctx, const uint8_t *d_in, const uint64_t *d_in_off,
                          const uint32_t *d_in_len, uint32_t n, uint8_t *d_out,
                          const uint64_t *d_out_off, const uint32_t *d_out_len,
                          uint32_t *d_got_len, int32_t *d_status, uint32_t max_out_len,
                          cudaStream_t st);
int hgpu_launch_bgzf_inflate(hgpu_ctx *ctx, const uint8_t *d_in, const uint64_t *d_in_off,
                             const uint32_t *d_in_len, uint32_t n, uint8_t *d_out,
                             const uint64_t *d_out_off, const uint32_t *d_out_cap,
                             uint32_t *d_out_len, int32_t *d_status, cudaStream_t st);
int hgpu_launch_gzip_inflate(hgpu_ctx *ctx, const uint8_t *d_in, const uint64_t *d_in_off, const uint32_t *d_in_len, uint32_t n,
                             uint8_t *d_out, const uint64_t *d_out_off, const uint32_t *d_out_cap, uint32_t *d_out_len,
                             int32_t *d_status, cudaStream_t st);
int hgpu_launch_crc32(hgpu_ctx *ctx, const uint8_t *d_buf, size_t len, uint32_t *d_partial,
                      uint32_t *h_result, uint32_t crc0, cudaStream_t st);
// hgpu_bgzf_compress_batch_dev with, when d_body_bits is not null, the bit length of every job's deflate block (which starts
// at byte 18 of its BGZF block) -- what a caller needs to splice the blocks into one deflate stream
int hgpu_launch_bgzf_deflate(hgpu_ctx *ctx, const uint8_t *d_in, const uint64_t *d_in_off, const uint32_t *d_in_len, uint32_t n,
                             int level, uint8_t *d_out, const uint64_t *d_out_off, uint32_t *d_out_len, int32_t *d_status,
                             uint32_t *d_body_bits, cudaStream_t st);

// hgpu_bam_index_records_dev over a window of a longer record stream (bam_unpack.cu): a record that runs past len ends the
// walk instead of breaking the chain, and *d_tail (device) receives where the walk stopped (len when whole records fill it)
int hgpu_bam_records_window_dev(hgpu_ctx *ctx, const uint8_t *d_stream, uint64_t len, const uint64_t *d_hint_off,
                                uint64_t n_hint, uint64_t *d_rec_off, uint64_t rec_cap, uint64_t *d_n_rec, uint64_t *d_tail,
                                cudaStream_t st);

int hgpu_launch_crc32_batch(hgpu_ctx *ctx, const uint8_t *d_buf, const uint64_t *d_off, const uint32_t *d_len, uint32_t n,
                            uint32_t *d_crc, cudaStream_t st);

#ifdef __CUDACC__
__device__ __forceinline__ uint32_t hgpu_lanemask_lt()
{
    uint32_t m;
    asm("mov.u32 %0, %%lanemask_lt;" : "=r"(m));
    return m;
}
__device__ __forceinline__ uint32_t hgpu_lane() { return threadIdx.x & 31; }
#endif
