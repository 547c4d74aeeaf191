// BAI / CSI index of a BAM image on the device: sam_index_build3 (sam.c:994-1074) — sam_index's record loop of
// sam_read1 + hts_idx_push (hts.c:2558-2640), hts_idx_finish (:2515-2531) and hts_idx_save_as (:2759-2887).
//
// The file goes through in windows of whole BGZF blocks.  Per window, on the device:
//   1. its compressed bytes go up through pinned staging (overlapping the previous window's kernels) and
//      bgzf_inflate_kernel inflates them behind the bytes carried from the previous window;
//   2. the record chain is walked from the block starts (bam_unpack.cu); a record still open at the window's end is
//      carried, with the blocks under it, to the front of the next window;
//   3. bam_index_key_kernel, one thread per record: the record rules of bam_index.cuh (read errors, CG-tag CIGAR,
//      bam_endpos, range, bin), the virtual offset bgzf_tell gives after the record, and the per-reference counts;
//   4. bam_index_push_kernel, one thread per record against its predecessor: the refusals of hts_idx_push, the starts
//      of chunks (a new (tid, bin)), and the linear index (atomicMin of the start offset over the 2^min_shift windows
//      the record covers).
// Only the chunk starts, the window's linear-index entries and a few scalars come back.  The host then replays the
// order in which hts_idx_push would have inserted chunks into its khash tables, runs compress_binning and update_loff,
// and writes the file (index_image below: O(bins)).  CSI output is BGZF-compressed by bgzf_deflate_kernel.
#include "hgpu_internal.h"
#include "bam_index.cuh"
#include <algorithm>
#include <chrono>
#include <stdlib.h>
#include <string.h>
#include <vector>

namespace {

constexpr uint64_t NONE = ~0ull;
constexpr int32_t NO_TID = INT32_MIN;           // "no previous record"

struct WinStat {
    unsigned long long n_rec, tail;             // chain walk: complete records, where the walk stopped
    unsigned long long err;                     // earliest refusal: record << 1 | (1 = hts_idx_push, 0 = sam_read1)
    unsigned long long n_runs;
    int32_t tmin, tmax;                         // placed references of the window
    int32_t last_tid;
    uint32_t last_bin;
    int64_t last_coor;
    uint64_t last_evoff;
};

struct Prev { int32_t tid; uint32_t bin; int64_t coor; uint64_t evoff; };

struct Run { uint64_t rec; int32_t tid; uint32_t bin; uint64_t svoff; };   // a chunk start: record, (tid, bin), start offset

struct Keys {                                   // per-record results of the key kernel (SoA)
    int32_t *tid; uint32_t *bin; int64_t *coor, *beg; int32_t *w0, *w1; uint64_t *evoff; uint8_t *flag;
};
enum : uint8_t { F_BAD = 1, F_MAPPED = 2 };

__global__ void __launch_bounds__(256)
bam_index_key_kernel(const uint8_t *st, const uint64_t *rec_off, uint64_t n, uint64_t rec0, const bidx::WinBlock *blk,
                     uint32_t nblk, int32_t n_targets, int min_shift, int n_lvls, Keys k, WinStat *ws,
                     unsigned long long *first_rec, unsigned long long *n_mapped, unsigned long long *n_unmapped,
                     unsigned long long *n_no_coor, int32_t *lin_lo, int32_t *lin_hi)
{
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint8_t *rec = st + rec_off[i];
    const bidx::Key key = bidx::record_key(rec, n_targets, min_shift, n_lvls);
    const uint64_t evoff = bidx::voff_after((int64_t)(rec_off[i] + 4 + bidx::ld32(rec)), blk, nblk);
    k.tid[i] = key.tid; k.bin[i] = key.bin; k.coor[i] = key.coor; k.beg[i] = key.beg;
    k.w0[i] = (int32_t)key.w0; k.w1[i] = (int32_t)key.w1; k.evoff[i] = evoff;
    k.flag[i] = (key.err ? F_BAD : 0) | (key.mapped ? F_MAPPED : 0);
    const uint64_t g = rec0 + i;
    if (key.err) {
        atomicMin(&ws->err, (unsigned long long)(g << 1 | (key.err == bidx::KEY_RANGE)));
    } else if (key.tid >= 0) {
        atomicMin(first_rec + key.tid, (unsigned long long)g);
        atomicAdd((key.mapped ? n_mapped : n_unmapped) + key.tid, 1ull);
        atomicMin(lin_lo + key.tid, (int32_t)key.w0);
        atomicMax(lin_hi + key.tid, (int32_t)key.w1);
        atomicMin(&ws->tmin, key.tid);
        atomicMax(&ws->tmax, key.tid);
    } else {
        atomicAdd(n_no_coor, 1ull);
    }
    if (i == n - 1) { ws->last_tid = key.tid; ws->last_bin = key.bin; ws->last_coor = key.coor; ws->last_evoff = evoff; }
}

__global__ void __launch_bounds__(256)
bam_index_push_kernel(uint64_t n, uint64_t rec0, Prev prev0, Keys k, const unsigned long long *first_rec, WinStat *ws,
                      Run *runs, unsigned long long *lin, const uint64_t *lin_base, const int32_t *lin_lo, int32_t tmin)
{
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n || (k.flag[i] & F_BAD)) return;
    const Prev p = i ? Prev{k.tid[i - 1], k.bin[i - 1], k.coor[i - 1], k.evoff[i - 1]} : prev0;
    const int32_t tid = k.tid[i];
    const uint64_t g = rec0 + i;
    bool refuse = false;
    if (tid != p.tid) {                          // change of reference (hts.c:2583-2595)
        if (tid >= 0 && p.tid != NO_TID && p.tid < 0) refuse = true;              // placed after unplaced
        if (tid >= 0 && first_rec[tid] < g) refuse = true;                        // a reference that returns
    } else if (tid >= 0 && p.coor > k.beg[i]) {
        refuse = true;                                                            // unsorted positions
    }
    if (refuse) { atomicMin(&ws->err, (unsigned long long)(g << 1 | 1)); return; }
    const uint32_t bin = k.bin[i];
    if (tid != p.tid || bin != p.bin) {
        const unsigned long long slot = atomicAdd(&ws->n_runs, 1ull);
        runs[slot] = Run{g, tid, bin, p.evoff};
    }
    if (tid >= 0) {
        const uint64_t b = lin_base[tid - tmin];
        const int32_t lo = lin_lo[tid];
        for (int32_t w = k.w0[i]; w <= k.w1[i]; w++) atomicMin(lin + b + (uint32_t)(w - lo), (unsigned long long)p.evoff);
    }
}

// the chain of a window is broken (a block_size < 32): how many records precede the bad one, and where it starts
__global__ void bam_index_chain_error_kernel(const uint8_t *st, uint64_t len, unsigned long long *out)
{
    uint64_t pos = 0, c = 0;
    while (len - pos >= 4) {
        const int32_t bl = (int32_t)bidx::ld32(st + pos);
        if (bl < 32 || pos + 4 + (uint64_t)bl > len) break;
        pos += 4 + (uint64_t)bl;
        c++;
    }
    out[0] = c;
    out[1] = pos;
}

// ------------------------------------------------------------------------------------------ host finishing

// khash's integer-key map (open addressing over a power-of-two table, probe steps 1, 2, 3, ..., grown at a 0.77 load,
// deletions left as tombstones) restated for the bin tables of one reference.  hts_idx_save writes bins in bucket
// order, so a byte-identical index needs the same buckets: same puts, same rehashes, same deletions.
struct BinList { std::vector<std::pair<uint64_t, uint64_t>> c; uint64_t loff = 0; };

class BinHash {
public:
    enum : uint8_t { LIVE = 0, DEL = 1, EMPTY = 2 };
    uint32_t nb = 0, size = 0;
    std::vector<uint32_t> key;
    std::vector<uint8_t> st;
    std::vector<BinList> val;

    bool live(uint32_t i) const { return st[i] == LIVE; }

    uint32_t get(uint32_t k) const
    {
        if (!nb) return 0;
        const uint32_t mask = nb - 1, first = k & mask;
        uint32_t i = first, step = 0;
        while (st[i] != EMPTY && (st[i] == DEL || key[i] != k)) {
            i = (i + ++step) & mask;
            if (i == first) return nb;
        }
        return st[i] == LIVE ? i : nb;
    }

    // slot of k, created empty if absent
    BinList &put(uint32_t k)
    {
        if (occupied >= upper) resize(nb > (size << 1) ? nb - 1 : nb + 1);
        const uint32_t mask = nb - 1, first = k & mask;
        uint32_t i = first, x = nb, site = nb, step = 0;
        if (st[i] == EMPTY) x = i;
        else {
            while (st[i] != EMPTY && (st[i] == DEL || key[i] != k)) {
                if (st[i] == DEL) site = i;
                i = (i + ++step) & mask;
                if (i == first) { x = site; break; }
            }
            if (x == nb) x = (st[i] == EMPTY && site != nb) ? site : i;
        }
        if (st[x] != LIVE) {
            if (st[x] == EMPTY) occupied++;
            key[x] = k; st[x] = LIVE; size++;
            val[x] = BinList();
        }
        return val[x];
    }

    void del(uint32_t i) { if (i != nb && st[i] == LIVE) { st[i] = DEL; size--; } }

private:
    uint32_t occupied = 0, upper = 0;

    void resize(uint32_t want)
    {
        uint32_t n = 4;
        while (n < want) n <<= 1;
        if (size >= (uint32_t)(n * 0.77 + 0.5)) return;
        std::vector<uint8_t> nst(n, EMPTY);
        if (n > nb) { key.resize(n); val.resize(n); st.resize(n, EMPTY); }
        const uint32_t mask = n - 1;
        for (uint32_t j = 0; j < nb; j++) {
            if (st[j] != LIVE) continue;
            uint32_t k = key[j];
            BinList v = std::move(val[j]);
            st[j] = DEL;
            for (;;) {                          // place, displacing a not-yet-moved element of the old table
                uint32_t i = k & mask, step = 0;
                while (nst[i] != EMPTY) i = (i + ++step) & mask;
                nst[i] = LIVE;
                if (i < nb && st[i] == LIVE) {
                    std::swap(k, key[i]);
                    std::swap(v, val[i]);
                    st[i] = DEL;
                } else {
                    key[i] = k;
                    val[i] = std::move(v);
                    break;
                }
            }
        }
        if (n < nb) { key.resize(n); val.resize(n); }
        st = std::move(nst);
        nb = n;
        occupied = size;
        upper = (uint32_t)(nb * 0.77 + 0.5);
    }
};

struct IndexParts {
    bool csi;
    int min_shift, n_lvls;
    int32_t n_ref;
    const std::vector<Run> *runs;                       // chunk starts in file order
    uint64_t final_off;
    std::vector<uint64_t> n_mapped, n_unmapped;         // per reference
    std::vector<std::vector<uint64_t>> lin;             // per reference: linear index (~0 = no record starts there)
    uint64_t n_no_coor;
};

int bin_level(uint32_t b) { int l = 0; while (b) { b = (b - 1) >> 3; l++; } return l; }

// hts_idx_push's chunk inserts (replayed from the chunk starts), hts_idx_finish (update_loff, compress_binning) and
// idx_save_core: the index file's bytes before any BGZF framing.
std::vector<uint8_t> index_image(IndexParts &P)
{
    const uint32_t n_bins = bidx::level_first(P.n_lvls + 1), meta = n_bins + 1;
    std::vector<BinHash> bh(P.n_ref > 0 ? P.n_ref : 0);
    std::vector<uint8_t> have(bh.size(), 0);
    auto insert = [&](int32_t tid, uint32_t bin, uint64_t u, uint64_t v) {
        have[tid] = 1;
        bh[tid].put(bin).c.emplace_back(u, v);
    };
    const std::vector<Run> &R = *P.runs;
    uint64_t off_beg = R.empty() ? 0 : R[0].svoff;
    for (size_t r = 1; r < R.size(); r++) {
        const Run &q = R[r - 1];
        insert(q.tid, q.bin, q.svoff, R[r].svoff);
        if (R[r].tid != q.tid) {
            insert(q.tid, meta, off_beg, R[r].svoff);
            insert(q.tid, meta, P.n_mapped[q.tid], P.n_unmapped[q.tid]);
            off_beg = R[r].svoff;
        }
    }
    if (!R.empty() && R.back().tid >= 0) {
        const Run &q = R.back();
        insert(q.tid, q.bin, q.svoff, P.final_off);
        insert(q.tid, meta, off_beg, P.final_off);
        insert(q.tid, meta, P.n_mapped[q.tid], P.n_unmapped[q.tid]);
    }
    for (int32_t t = 0; t < P.n_ref; t++) {
        std::vector<uint64_t> &L = P.lin[t];
        for (int64_t l = (int64_t)L.size() - 2; l >= 0; l--) if (L[l] == NONE) L[l] = L[l + 1];
        if (!have[t]) continue;
        BinHash &h = bh[t];
        for (uint32_t k = 0; k < h.nb; k++) {                       // update_loff
            if (!h.live(k)) continue;
            const uint32_t b = h.key[k];
            if (b < n_bins) {
                const int l = bin_level(b);
                const uint64_t bot = (uint64_t)(b - bidx::level_first(l)) << (3 * (P.n_lvls - l));
                h.val[k].loff = bot < L.size() ? L[bot] : 0;
            } else h.val[k].loff = 0;
        }
        auto by_u = [](const std::pair<uint64_t, uint64_t> &a, const std::pair<uint64_t, uint64_t> &b) { return a.first < b.first; };
        for (int l = P.n_lvls; l > 0; --l) {                        // compress_binning
            const uint32_t start = bidx::level_first(l);
            for (uint32_t k = 0; k < h.nb; k++) {
                if (!h.live(k) || h.key[k] >= n_bins || h.key[k] < start) continue;
                std::vector<std::pair<uint64_t, uint64_t>> &c = h.val[k].c;
                if (l < P.n_lvls && c.size() > 1) std::sort(c.begin(), c.end(), by_u);
                if ((c.back().second >> 16) - (c.front().first >> 16) < 0x10000) {
                    const uint32_t kp = h.get((h.key[k] - 1) >> 3);
                    if (kp == h.nb) continue;
                    std::vector<std::pair<uint64_t, uint64_t>> &q = h.val[kp].c;
                    q.insert(q.end(), c.begin(), c.end());
                    c.clear();
                    h.del(k);
                }
            }
        }
        const uint32_t k0 = h.get(0);
        if (k0 != h.nb) std::sort(h.val[k0].c.begin(), h.val[k0].c.end(), by_u);
        for (uint32_t k = 0; k < h.nb; k++) {                       // merge chunks that start in the same block
            if (!h.live(k) || h.key[k] >= n_bins) continue;
            std::vector<std::pair<uint64_t, uint64_t>> &c = h.val[k].c;
            size_t m = 0;
            for (size_t l = 1; l < c.size(); l++) {
                if ((c[m].second >> 16) >= (c[l].first >> 16)) { if (c[m].second < c[l].second) c[m].second = c[l].second; }
                else c[++m] = c[l];
            }
            c.resize(m + 1);
        }
    }
    std::vector<uint8_t> out;
    auto put = [&](uint64_t v, int bytes) { for (int b = 0; b < bytes; b++) out.push_back((uint8_t)(v >> (8 * b))); };
    if (P.csi) {
        out.insert(out.end(), {'C', 'S', 'I', 1});
        put((uint32_t)P.min_shift, 4); put((uint32_t)P.n_lvls, 4); put(0, 4);
    } else {
        out.insert(out.end(), {'B', 'A', 'I', 1});
    }
    put((uint32_t)P.n_ref, 4);
    for (int32_t t = 0; t < P.n_ref; t++) {
        const BinHash &h = bh[t];
        put(have[t] ? h.size : 0, 4);
        if (have[t])
            for (uint32_t k = 0; k < h.nb; k++) {
                if (!h.live(k)) continue;
                const BinList &b = h.val[k];
                put(h.key[k], 4);
                if (P.csi) put(b.loff, 8);
                put((uint32_t)b.c.size(), 4);
                for (const auto &ch : b.c) { put(ch.first, 8); put(ch.second, 8); }
            }
        if (!P.csi) {
            put((uint32_t)P.lin[t].size(), 4);
            for (uint64_t v : P.lin[t]) put(v, 8);
        }
    }
    put(P.n_no_coor, 8);
    return out;
}

// hts_adjust_csi_settings (hts.c:2372): enough levels, or failing that a coarser min_shift, for the longest reference
void csi_settings(int64_t max_len, int &min_shift, int &n_lvls)
{
    const int64_t need = max_len + 256;
    auto maxpos = [](int s, int l) { return (int64_t)1 << (s + 3 * l); };
    if (need <= maxpos(min_shift, 9)) {
        for (n_lvls = 0; need > maxpos(min_shift, n_lvls); n_lvls++) {}
    } else {
        n_lvls = 9;
        while (need > maxpos(min_shift, n_lvls)) min_shift++;
    }
}

struct DevBuf {
    void *p = nullptr;
    size_t cap = 0;
    ~DevBuf() { if (p) cudaFree(p); }
    // room for `bytes`; with `keep` bytes of the old contents preserved (stream-ordered copy on st)
    int ensure(size_t bytes, size_t keep = 0, cudaStream_t st = 0)
    {
        if (bytes <= cap) return HGPU_OK;
        const size_t ncap = bytes + bytes / 8 + 4096;
        void *q = nullptr;
        if (cudaMalloc(&q, ncap) != cudaSuccess) {
            cudaGetLastError();
            hgpu_set_error("device alloc of %zu bytes failed", ncap);
            return HGPU_ERR_NOMEM;
        }
        if (keep && hgpu_check(cudaMemcpyAsync(q, p, keep, cudaMemcpyDeviceToDevice, st), "D2D")) { cudaFree(q); return HGPU_ERR_CUDA; }
        if (keep && hgpu_check(cudaStreamSynchronize(st), "sync")) { cudaFree(q); return HGPU_ERR_CUDA; }
        if (p) cudaFree(p);
        p = q;
        cap = ncap;
        return HGPU_OK;
    }
    template <class T = uint8_t> T *at(size_t off = 0) const { return reinterpret_cast<T *>((uint8_t *)p + off); }
};

struct HostPinned {
    uint8_t *p = nullptr;
    ~HostPinned() { if (p) cudaFreeHost(p); }
};

// CSI files are BGZF: 0xff00-byte payloads through bgzf_deflate_kernel at the default level, then the EOF block
int bgzf_frame(hgpu_ctx *ctx, const std::vector<uint8_t> &raw, std::vector<uint8_t> &out)
{
    static const uint8_t eof_block[28] = {0x1f, 0x8b, 8, 4, 0, 0, 0, 0, 0, 0xff, 6, 0, 'B', 'C', 2, 0, 0x1b, 0, 3, 0, 0, 0, 0, 0, 0, 0, 0, 0};
    const uint32_t n = (uint32_t)((raw.size() + 0xff00 - 1) / 0xff00);
    out.clear();
    if (n) {
        std::vector<uint64_t> off(2 * (size_t)n);
        std::vector<uint32_t> len(n), olen(n);
        std::vector<int32_t> st(n);
        for (uint32_t i = 0; i < n; i++) {
            off[i] = (uint64_t)i * 0xff00;
            len[i] = (uint32_t)std::min<uint64_t>(0xff00, raw.size() - off[i]);
            off[n + i] = (uint64_t)i * 65536;
        }
        StageLayout L;
        const auto s_in = L.seg(raw.size() + 4), s_off = L.seg(16 * (size_t)n), s_len = L.seg(4 * (size_t)n),
                   s_out = L.seg(65536 * (size_t)n), s_olen = L.seg(4 * (size_t)n), s_st = L.seg(4 * (size_t)n);
        int rc = hgpu_stage_ensure(ctx, L);
        if (rc) return rc;
        cudaStream_t s = ctx->stream;
        if (hgpu_h2d(L.at(s_in), raw.data(), raw.size(), s) || hgpu_h2d(L.at(s_off), off.data(), 16 * (size_t)n, s) ||
            hgpu_h2d(L.at(s_len), len.data(), 4 * (size_t)n, s)) return HGPU_ERR_CUDA;
        rc = hgpu_bgzf_compress_batch_dev(ctx, L.at(s_in), L.at<uint64_t>(s_off), L.at<uint32_t>(s_len), n, -1, L.at(s_out),
                                          L.at<uint64_t>(s_off) + n, L.at<uint32_t>(s_olen), L.at<int32_t>(s_st), s);
        if (rc) return rc;
        std::vector<uint8_t> blocks(65536 * (size_t)n);
        if (hgpu_d2h(blocks.data(), L.at(s_out), blocks.size(), s) || hgpu_d2h(olen.data(), L.at(s_olen), 4 * (size_t)n, s) ||
            hgpu_d2h(st.data(), L.at(s_st), 4 * (size_t)n, s) || hgpu_check(cudaStreamSynchronize(s), "sync")) return HGPU_ERR_CUDA;
        for (uint32_t i = 0; i < n; i++) {
            if (st[i] != HGPU_OK) { hgpu_set_error("index BGZF block %u: status %d", i, st[i]); return HGPU_ERR_CUDA; }
            out.insert(out.end(), blocks.begin() + (size_t)i * 65536, blocks.begin() + (size_t)i * 65536 + olen[i]);
        }
    }
    out.insert(out.end(), eof_block, eof_block + 28);
    return HGPU_OK;
}

float g_last_ms[2];

} // namespace

extern "C" void hgpu_bam_index_last_ms(float *ms2)
{
    if (ms2) { ms2[0] = g_last_ms[0]; ms2[1] = g_last_ms[1]; }
}

static int bam_index_build_impl(hgpu_ctx *ctx, const uint8_t *file, uint64_t file_len, int min_shift, uint64_t window_bytes,
                                uint8_t **out, uint64_t *out_len, int64_t *bad)
{
    if (!ctx || !file || !out || !out_len) { hgpu_set_error("bad argument"); return HGPU_ERR_ARG; }
    *out = nullptr; *out_len = 0;
    int64_t bad_dummy;
    if (!bad) bad = &bad_dummy;
    *bad = -1;
    g_last_ms[0] = g_last_ms[1] = 0;
    if (hgpu_check(cudaSetDevice(ctx->device), "cudaSetDevice")) return HGPU_ERR_CUDA;
    // ---- block table (hgpu_bgzf_scan) ----
    if (file_len < 18 || file[0] != 31 || file[1] != 139) { hgpu_set_error("not a BGZF file"); return HGPU_ERR_ARG; }
    long nb = hgpu_bgzf_scan(file, file_len, nullptr, nullptr, nullptr, 0);
    if (nb == -1) { hgpu_set_error("not a BGZF file"); return HGPU_ERR_ARG; }
    if (nb < 0) { *bad = -1 - nb; hgpu_set_error("bad BGZF header at block %ld", -1 - nb); return HGPU_BGZF_ERR_HEADER; }
    std::vector<uint64_t> off(nb + 1);
    std::vector<uint32_t> clen(nb), isz(nb);
    hgpu_bgzf_scan(file, file_len, off.data(), clen.data(), isz.data(), nb);
    off[nb] = file_len;
    std::vector<int64_t> ustart(nb + 1, 0);
    for (long i = 0; i < nb; i++) {
        if (isz[i] > 65536u) { *bad = i; hgpu_set_error("ISIZE > 64 KiB at block %ld", i); return HGPU_BGZF_ERR_ZLIB; }
        ustart[i + 1] = ustart[i] + isz[i];
    }
    auto gblock = [&](long i) { return bidx::WinBlock{ustart[i], ustart[i + 1], off[i], off[i + 1]}; };
    // ---- windows of new blocks: [wb[k], wb[k+1]) ----
    if (window_bytes == 0) {
        size_t fr = 0, tot = 0;
        if (hgpu_check(cudaMemGetInfo(&fr, &tot), "cudaMemGetInfo")) return HGPU_ERR_CUDA;
        // resident per uncompressed byte: the stream, two compressed buffers (at most ~1 byte each), ~1.2 bytes of
        // per-record arrays (41 bytes per record of >= 36 bytes)
        const uint64_t spare = fr > (1ull << 30) ? fr - (1ull << 30) : fr / 2;
        window_bytes = std::max<uint64_t>(spare / 5, 64ull << 20);
    }
    std::vector<long> wb{0};
    for (long i = 0; i < nb;) {
        uint64_t u = 0;
        long j = i;
        while (j < nb && (j == i || u + isz[j] <= window_bytes)) u += isz[j++];
        wb.push_back(j);
        i = j;
    }
    const long nw = (long)wb.size() - 1;
    uint64_t max_comp = 0, max_new = 0, max_nblk = 0;
    for (long k = 0; k < nw; k++) {
        max_comp = std::max<uint64_t>(max_comp, off[wb[k + 1]] - off[wb[k]]);
        max_new = std::max<uint64_t>(max_new, (uint64_t)(ustart[wb[k + 1]] - ustart[wb[k]]));
        max_nblk = std::max<uint64_t>(max_nblk, (uint64_t)(wb[k + 1] - wb[k]));
    }
    // ---- buffers ----
    cudaStream_t s = ctx->stream, up = ctx->copy_stream[0];
    DevBuf dcomp[2], dmeta[2], dout, drec, dkeys, dtid, dws, dwin, dlin, druns;
    // per-window inflate job arrays, one image uploaded with the compressed bytes
    StageLayout M;
    const auto m_ioff = M.seg(max_nblk * 8), m_ooff = M.seg(max_nblk * 8), m_ilen = M.seg(max_nblk * 4), m_cap = M.seg(max_nblk * 4),
               m_olen = M.seg(max_nblk * 4), m_st = M.seg(max_nblk * 4);
    for (int b = 0; b < 2; b++)
        if (dcomp[b].ensure(max_comp + 4) || dmeta[b].ensure(M.total)) return HGPU_ERR_NOMEM;
    const size_t chunk = 16u << 20;
    HostPinned pin;
    if (hgpu_check(cudaMallocHost((void **)&pin.p, 2 * chunk + M.total), "pinned staging")) return HGPU_ERR_NOMEM;
    cudaEvent_t ev_chunk[2] = {ctx->ev[4], ctx->ev[5]}, ev_up[2] = {ctx->ev[2], ctx->ev[3]}, t0, t1;
    if (hgpu_check(cudaEventCreate(&t0), "event") || hgpu_check(cudaEventCreate(&t1), "event")) return HGPU_ERR_CUDA;
    struct EvGuard { cudaEvent_t a, b; ~EvGuard() { cudaEventDestroy(a); cudaEventDestroy(b); } } evg{t0, t1};
    int chunk_i = 0;
    // window k's compressed bytes and job arrays through pinned staging on the copy stream
    auto upload = [&](long k) -> int {
        const long b0 = wb[k], b1 = wb[k + 1];
        const uint64_t c0 = off[b0], cn = off[b1] - c0;
        for (uint64_t p = 0; p < cn; p += chunk) {
            const int h = chunk_i++ & 1;
            const uint64_t m = std::min<uint64_t>(chunk, cn - p);
            if (hgpu_check(cudaEventSynchronize(ev_chunk[h]), "staging wait")) return HGPU_ERR_CUDA;
            memcpy(pin.p + h * chunk, file + c0 + p, m);
            if (hgpu_h2d(dcomp[k & 1].at(p), pin.p + h * chunk, m, up) || hgpu_check(cudaEventRecord(ev_chunk[h], up), "event"))
                return HGPU_ERR_CUDA;
        }
        uint8_t *hm = pin.p + 2 * chunk;
        if (hgpu_check(cudaStreamSynchronize(up), "staging wait")) return HGPU_ERR_CUDA;   // hm is reused per window
        uint64_t *ioff = (uint64_t *)(hm + m_ioff.off), *ooff = (uint64_t *)(hm + m_ooff.off);
        uint32_t *ilen = (uint32_t *)(hm + m_ilen.off), *cap = (uint32_t *)(hm + m_cap.off);
        for (long i = b0; i < b1; i++) {
            ioff[i - b0] = off[i] - c0; ooff[i - b0] = (uint64_t)(ustart[i] - ustart[b0]);
            ilen[i - b0] = clen[i]; cap[i - b0] = isz[i];
        }
        if (hgpu_h2d(dmeta[k & 1].p, hm, m_olen.off, up)) return HGPU_ERR_CUDA;
        return hgpu_check(cudaEventRecord(ev_up[k & 1], up), "event");
    };
    // ---- per-reference state (sized once the header is read) ----
    bool hdr_done = false;
    int32_t n_ref = 0;
    int64_t max_len = 0, hdr_len = 0;
    int ms = 14, nl = 5;
    const bool csi = min_shift > 0;
    uint64_t offset0 = 0, n_total = 0;
    Prev prev{NO_TID, 0, 0, 0};
    std::vector<Run> runs;
    std::vector<std::vector<uint64_t>> lin;
    unsigned long long *first_rec = nullptr, *n_mapped = nullptr, *n_unmapped = nullptr, *n_no_coor = nullptr;
    int32_t *lin_lo = nullptr, *lin_hi = nullptr;
    uint64_t *lin_base = nullptr;
    WinStat *ws = nullptr;
    if (dws.ensure(256)) return HGPU_ERR_NOMEM;
    ws = dws.at<WinStat>();
    n_no_coor = dws.at<unsigned long long>(128);
    if (hgpu_memset(dws.p, 0, 256, s)) return HGPU_ERR_CUDA;
    float dev_ms = 0;
    int64_t o_glob = 0;                                  // stream position of dout[0]
    uint64_t carry = 0;                                  // bytes at the front of dout carried from the previous window
    int rc = upload(0);
    if (rc) return rc;
    for (long k = 0; k < nw; k++) {
        const long b0 = wb[k], b1 = wb[k + 1], nnew = b1 - b0;
        const uint64_t new_len = (uint64_t)(ustart[b1] - ustart[b0]), len = carry + new_len;
        if ((rc = dout.ensure(len + 16, carry, s))) return rc;
        if (hgpu_check(cudaStreamWaitEvent(s, ev_up[k & 1], 0), "wait") || hgpu_check(cudaEventRecord(t0, s), "event")) return HGPU_ERR_CUDA;
        const DevBuf &mb = dmeta[k & 1];
        rc = hgpu_launch_bgzf_inflate(ctx, dcomp[k & 1].at(), mb.at<uint64_t>(m_ioff.off), mb.at<uint32_t>(m_ilen.off), (uint32_t)nnew,
                                      dout.at(carry), mb.at<uint64_t>(m_ooff.off), mb.at<uint32_t>(m_cap.off),
                                      mb.at<uint32_t>(m_olen.off), mb.at<int32_t>(m_st.off), s);
        if (rc) return rc;
        // the next window goes up while this one inflates (its buffers were last read by window k-1, already synchronised)
        if (k + 1 < nw && (rc = upload(k + 1))) return rc;
        std::vector<uint32_t> olen(nnew);
        std::vector<int32_t> bst(nnew);
        if (hgpu_d2h(olen.data(), mb.at(m_olen.off), 4 * nnew, s) || hgpu_d2h(bst.data(), mb.at(m_st.off), 4 * nnew, s) ||
            hgpu_check(cudaStreamSynchronize(s), "sync")) return HGPU_ERR_CUDA;
        for (long i = 0; i < nnew; i++) {
            if (bst[i] != HGPU_OK) { *bad = b0 + i; hgpu_set_error("block %ld: status %d", b0 + i, bst[i]); return bst[i]; }
            if (olen[i] != isz[b0 + i]) { *bad = b0 + i; hgpu_set_error("block %ld: inflated size differs from ISIZE", b0 + i); return HGPU_BGZF_ERR_ZLIB; }
        }
        const bool last = k + 1 == nw;
        int64_t rs = 0;                                  // where this window's records start in dout
        if (!hdr_done) {
            // bam_hdr_read (sam.c:229-319): only the header's fixed fields, n_ref and the @SQ lengths come down
            std::vector<uint8_t> cache;
            int64_t cpos = 0;
            auto need = [&](int64_t p, int64_t n, uint8_t *dst) -> int {       // 1 ok, 0 not in this window yet
                if (p + n > (int64_t)len) return 0;
                if (p < cpos || p + n > cpos + (int64_t)cache.size()) {
                    cpos = p;
                    cache.resize((size_t)std::min<int64_t>(std::max<int64_t>(n, 1 << 20), (int64_t)len - p));
                    if (hgpu_d2h(cache.data(), dout.at(p), cache.size(), s) || hgpu_check(cudaStreamSynchronize(s), "sync")) return -1;
                }
                memcpy(dst, cache.data() + (p - cpos), n);
                return 1;
            };
            uint8_t b8[8];
            int64_t p = 0;
            const int magic = need(0, 4, b8);
            if (magic < 0) return HGPU_ERR_CUDA;
            if ((magic > 0 && memcmp(b8, "BAM\1", 4) != 0) || (magic == 0 && last)) { hgpu_set_error("not a BAM file"); return HGPU_ERR_ARG; }
            int got = magic > 0 ? need(0, 8, b8) : 0;
            bool invalid = false;
            if (got > 0) {
                p = 8 + (int64_t)bidx::ld32(b8 + 4);
                got = need(p, 4, b8);
                if (got > 0) {
                    n_ref = (int32_t)bidx::ld32(b8);
                    p += 4;
                    if (n_ref < 0) invalid = true;
                    max_len = 0;
                    for (int32_t t = 0; got > 0 && !invalid && t < n_ref; t++) {
                        if ((got = need(p, 4, b8)) <= 0) break;
                        const int32_t l_name = (int32_t)bidx::ld32(b8);
                        if (l_name <= 0) { invalid = true; break; }
                        p += 4 + (int64_t)l_name;
                        if ((got = need(p, 4, b8)) <= 0) break;
                        max_len = std::max<int64_t>(max_len, (int64_t)bidx::ld32(b8));
                        p += 4;
                    }
                }
            }
            if (got < 0) return HGPU_ERR_CUDA;
            if (invalid || (got == 0 && last)) { hgpu_set_error("invalid or truncated BAM header"); return HGPU_IDX_ERR_READ; }
            if (got == 0) { carry = len; continue; }     // the header runs on into the next window
            hdr_done = true;
            hdr_len = p;
            rs = p;
            if (csi) { ms = min_shift; nl = 0; csi_settings(max_len, ms, nl); }
            // offset0: bgzf_tell after the header
            {
                std::vector<bidx::WinBlock> g(nb);
                for (long i = 0; i < nb; i++) g[i] = gblock(i);
                offset0 = bidx::voff_after(hdr_len, g.data(), (uint32_t)nb);
            }
            prev.evoff = offset0;
            lin.assign(n_ref, {});
            const size_t nr = (size_t)std::max(n_ref, 1);
            if (dtid.ensure(nr * 8 * 3 + nr * 4 * 2 + (nr + 1) * 8 + 1024)) return HGPU_ERR_NOMEM;
            first_rec = dtid.at<unsigned long long>();
            n_mapped = first_rec + nr; n_unmapped = n_mapped + nr;
            lin_lo = (int32_t *)(n_unmapped + nr); lin_hi = lin_lo + nr;
            lin_base = (uint64_t *)(((uintptr_t)(lin_hi + nr) + 255) & ~(uintptr_t)255);
            if (hgpu_memset(first_rec, 0xff, nr * 8, s) || hgpu_memset(n_mapped, 0, nr * 16, s)) return HGPU_ERR_CUDA;
        }
        // ---- records of this window: stream [origin, origin + slen) ----
        const int64_t origin = o_glob + rs;
        const uint64_t slen = len - (uint64_t)rs;
        const uint8_t *d_st = dout.at(rs);
        std::vector<bidx::WinBlock> wblk;
        std::vector<uint64_t> hints{0};
        const long first = (long)(std::upper_bound(ustart.begin() + 1, ustart.end(), origin) - (ustart.begin() + 1));
        for (long i = first; i < b1; i++) {              // the blocks under the carried bytes, then the new ones
            bidx::WinBlock g = gblock(i);
            g.ustart -= origin; g.uend -= origin;
            wblk.push_back(g);
            if (g.ustart > 0 && g.uend > g.ustart) hints.push_back((uint64_t)g.ustart);
        }
        const size_t nwb = wblk.size(), rec_cap = slen / 36 + 1;
        StageLayout W;
        const auto w_blk = W.seg(nwb * sizeof(bidx::WinBlock)), w_hint = W.seg(hints.size() * 8);
        if (dwin.ensure(W.total)) return HGPU_ERR_NOMEM;
        W.base = dwin.at();
        WinStat init{};
        init.err = NONE; init.tmin = INT32_MAX; init.tmax = INT32_MIN;
        if (hgpu_h2d(W.at(w_blk), wblk.data(), nwb * sizeof(bidx::WinBlock), s) || hgpu_h2d(W.at(w_hint), hints.data(), hints.size() * 8, s) ||
            hgpu_h2d(ws, &init, sizeof(init), s)) return HGPU_ERR_CUDA;
        if (drec.ensure(rec_cap * 8)) return HGPU_ERR_NOMEM;
        uint64_t *rec_off = drec.at<uint64_t>();
        if ((rc = hgpu_bam_records_window_dev(ctx, d_st, slen, W.at<uint64_t>(w_hint), hints.size(), rec_off, rec_cap, (uint64_t *)&ws->n_rec, (uint64_t *)&ws->tail, s)))
            return rc;
        WinStat hs;
        if (hgpu_d2h(&hs, ws, sizeof(hs), s) || hgpu_check(cudaStreamSynchronize(s), "sync")) return HGPU_ERR_CUDA;
        uint64_t n = hs.n_rec, tail = hs.tail;
        bool broken = false;
        if (n == NONE) {
            // a block_size < 32: the records before it are indexed as usual (an earlier refusal wins), then it is the error
            unsigned long long ce[2];
            bam_index_chain_error_kernel<<<1, 1, 0, s>>>(d_st, slen, dws.at<unsigned long long>(192));
            hgpu_count_launch();
            if (hgpu_d2h(ce, dws.at(192), 16, s) || hgpu_check(cudaStreamSynchronize(s), "sync")) return HGPU_ERR_CUDA;
            if (hgpu_h2d(ws, &init, sizeof(init), s)) return HGPU_ERR_CUDA;
            if ((rc = hgpu_bam_records_window_dev(ctx, d_st, ce[1], W.at<uint64_t>(w_hint), hints.size(), rec_off, rec_cap, (uint64_t *)&ws->n_rec, (uint64_t *)&ws->tail, s)))
                return rc;
            if (hgpu_d2h(&hs, ws, sizeof(hs), s) || hgpu_check(cudaStreamSynchronize(s), "sync")) return HGPU_ERR_CUDA;
            n = hs.n_rec;
            broken = true;
        }
        if (n > 0) {
            StageLayout K;
            const auto k_tid = K.seg(n * 4), k_bin = K.seg(n * 4), k_coor = K.seg(n * 8), k_beg = K.seg(n * 8), k_w0 = K.seg(n * 4),
                       k_w1 = K.seg(n * 4), k_ev = K.seg(n * 8), k_fl = K.seg(n);
            if (dkeys.ensure(K.total)) return HGPU_ERR_NOMEM;
            K.base = dkeys.at();
            Keys keys{K.at<int32_t>(k_tid), K.at<uint32_t>(k_bin), K.at<int64_t>(k_coor), K.at<int64_t>(k_beg), K.at<int32_t>(k_w0),
                      K.at<int32_t>(k_w1), K.at<uint64_t>(k_ev), K.at<uint8_t>(k_fl)};
            if (n_ref > 0 && (hgpu_memset(lin_lo, 0x7f, (size_t)n_ref * 4, s) || hgpu_memset(lin_hi, 0xff, (size_t)n_ref * 4, s))) return HGPU_ERR_CUDA;
            const unsigned grid = (unsigned)((n + 255) / 256);
            bam_index_key_kernel<<<grid, 256, 0, s>>>(d_st, rec_off, n, n_total, W.at<bidx::WinBlock>(w_blk), (uint32_t)nwb, n_ref, ms, nl, keys,
                                                      ws, first_rec, n_mapped, n_unmapped, n_no_coor, lin_lo, lin_hi);
            hgpu_count_launch();
            if (hgpu_check(cudaGetLastError(), "bam_index_key_kernel") || hgpu_d2h(&hs, ws, sizeof(hs), s) ||
                hgpu_check(cudaStreamSynchronize(s), "sync")) return HGPU_ERR_CUDA;
            // this window's slice of the linear index: per placed reference, the windows its records cover
            const int32_t tmin = hs.tmin, tmax = hs.tmax, nt = tmax >= tmin ? tmax - tmin + 1 : 0;
            std::vector<int32_t> lo(nt), hi(nt);
            std::vector<uint64_t> base(nt + 1, 0);
            if (nt) {
                if (hgpu_d2h(lo.data(), lin_lo + tmin, nt * 4, s) || hgpu_d2h(hi.data(), lin_hi + tmin, nt * 4, s) ||
                    hgpu_check(cudaStreamSynchronize(s), "sync")) return HGPU_ERR_CUDA;
                for (int32_t t = 0; t < nt; t++) base[t + 1] = base[t] + (hi[t] >= lo[t] ? (uint64_t)(hi[t] - lo[t] + 1) : 0);
                if (hgpu_h2d(lin_base, base.data(), nt * 8, s)) return HGPU_ERR_CUDA;
            }
            if (dlin.ensure(base[nt] * 8 + 8) || druns.ensure(n * sizeof(Run))) return HGPU_ERR_NOMEM;
            if (hgpu_memset(dlin.p, 0xff, base[nt] * 8, s)) return HGPU_ERR_CUDA;
            bam_index_push_kernel<<<grid, 256, 0, s>>>(n, n_total, prev, keys, first_rec, ws, druns.at<Run>(), dlin.at<unsigned long long>(),
                                                       lin_base, lin_lo, tmin);
            hgpu_count_launch();
            if (hgpu_check(cudaGetLastError(), "bam_index_push_kernel") || hgpu_d2h(&hs, ws, sizeof(hs), s) ||
                hgpu_check(cudaEventRecord(t1, s), "event") || hgpu_check(cudaStreamSynchronize(s), "sync")) return HGPU_ERR_CUDA;
            float wms = 0;
            cudaEventElapsedTime(&wms, t0, t1);
            dev_ms += wms;
            if (hs.err != NONE) {
                *bad = (int64_t)(hs.err >> 1);
                hgpu_set_error("record %lld: %s", (long long)*bad, (hs.err & 1) ? "refused by hts_idx_push" : "sam_read1 fails");
                return (hs.err & 1) ? HGPU_IDX_ERR_PUSH : HGPU_IDX_ERR_READ;
            }
            const size_t r0 = runs.size();
            runs.resize(r0 + hs.n_runs);
            std::vector<uint64_t> lw(base[nt]);
            if (hgpu_d2h(runs.data() + r0, druns.p, hs.n_runs * sizeof(Run), s) || hgpu_d2h(lw.data(), dlin.p, lw.size() * 8, s) ||
                hgpu_check(cudaStreamSynchronize(s), "sync")) return HGPU_ERR_CUDA;
            std::sort(runs.begin() + r0, runs.end(), [](const Run &a, const Run &b) { return a.rec < b.rec; });
            for (int32_t t = 0; t < nt; t++) {
                if (hi[t] < lo[t]) continue;
                std::vector<uint64_t> &L = lin[tmin + t];
                if (L.size() < (size_t)hi[t] + 1) L.resize((size_t)hi[t] + 1, NONE);
                for (int32_t w = lo[t]; w <= hi[t]; w++) L[w] = std::min(L[w], lw[base[t] + (w - lo[t])]);
            }
            prev = Prev{hs.last_tid, hs.last_bin, hs.last_coor, hs.last_evoff};
            n_total += n;
        }
        if (broken) {
            *bad = (int64_t)n_total;
            hgpu_set_error("record %lld: broken record chain", (long long)*bad);
            return HGPU_IDX_ERR_READ;
        }
        if (last) {
            if (tail != slen) {
                *bad = (int64_t)n_total;
                hgpu_set_error("record %lld: truncated", (long long)*bad);
                return HGPU_IDX_ERR_READ;
            }
            break;
        }
        // carry the open record to the front of the buffer, in pieces that never overlap
        carry = slen - tail;
        const uint64_t from = (uint64_t)rs + tail;
        for (uint64_t p = 0; p < carry && from; p += from) {
            const uint64_t m = std::min<uint64_t>(from, carry - p);
            if (hgpu_check(cudaMemcpyAsync(dout.at(p), dout.at(from + p), m, cudaMemcpyDeviceToDevice, s), "carry")) return HGPU_ERR_CUDA;
        }
        o_glob = origin + (int64_t)tail;
    }
    if (!hdr_done) { hgpu_set_error("truncated BAM header"); return HGPU_IDX_ERR_READ; }
    // ---- finish on the host ----
    const auto h0 = std::chrono::steady_clock::now();
    IndexParts P;
    P.csi = csi; P.min_shift = ms; P.n_lvls = nl; P.n_ref = n_ref; P.runs = &runs;
    P.final_off = n_total ? prev.evoff : offset0;
    P.n_mapped.assign(n_ref, 0); P.n_unmapped.assign(n_ref, 0);
    unsigned long long nnc = 0;
    if (n_ref && (hgpu_d2h(P.n_mapped.data(), n_mapped, (size_t)n_ref * 8, s) || hgpu_d2h(P.n_unmapped.data(), n_unmapped, (size_t)n_ref * 8, s)))
        return HGPU_ERR_CUDA;
    if (hgpu_d2h(&nnc, n_no_coor, 8, s) || hgpu_check(cudaStreamSynchronize(s), "sync")) return HGPU_ERR_CUDA;
    P.n_no_coor = nnc;
    P.lin = std::move(lin);
    std::vector<uint8_t> img = index_image(P), framed;
    const std::vector<uint8_t> *res = &img;
    if (csi) {
        if ((rc = bgzf_frame(ctx, img, framed))) return rc;
        res = &framed;
    }
    uint8_t *o = (uint8_t *)malloc(res->size() ? res->size() : 1);
    if (!o) { hgpu_set_error("out of host memory"); return HGPU_ERR_NOMEM; }
    memcpy(o, res->data(), res->size());
    *out = o;
    *out_len = res->size();
    g_last_ms[0] = dev_ms;
    g_last_ms[1] = std::chrono::duration<float, std::milli>(std::chrono::steady_clock::now() - h0).count();
    return HGPU_OK;
}

extern "C" int hgpu_bam_index_build_host(hgpu_ctx *ctx, const uint8_t *file, uint64_t file_len, int min_shift, uint64_t window_bytes,
                                         uint8_t **out, uint64_t *out_len, int64_t *bad)
{
    return hgpu_abi_call([&] { return bam_index_build_impl(ctx, file, file_len, min_shift, window_bytes, out, out_len, bad); });
}
