// hgpu_cram_index_build_host: the .crai of a CRAM 3.x image -- cram_index_build (cram/cram_index.c:779-848) as
// sam_index_build3 (sam.c:1047) runs it, for a whole file image at once.
//
// Host (O(containers + slices)): the walk of cram_index_build / cram_index_container / cram_index_slice over container, block
// and slice headers, with their refusals.  A slice with ref_seq_id != -2 gives its line straight from its header.
// Device: the multi-reference slices (the device writer makes every slice one).  Their blocks that
// CRAM_OPT_REQUIRED_FIELDS = SAM_RNAME | SAM_POS | SAM_CIGAR reads are uncompressed in one batch, cram_slice_decode_kernel
// decodes those slices only (cram_records.cu: slice_records, no bam1_t fill), and cram_index_runs_kernel, a warp per slice,
// reduces each slice's records to its runs of equal ref_id (cram_index.cuh).  Only the runs (24 bytes each) and the first
// record out of order come back.  The text is then deflated on the device into one gzip member (gzip_member below).
//
// Built a second time by tests/hostsim (g++ -DHGPU_HOSTSIM), the kernels replaced by slice_runs, the block uncompress by the
// blocks the caller hands in.
#ifdef HGPU_HOSTSIM
#include "../../include/htsgpu.h"
#include <stdarg.h>
#include <stdio.h>
static char g_idx_err[256];
static void hgpu_set_error(const char *fmt, ...) { va_list ap; va_start(ap, fmt); vsnprintf(g_idx_err, sizeof g_idx_err, fmt, ap); va_end(ap); }
extern "C" const char *hostsim_index_last_error(void) { return g_idx_err; }
#else
#include "hgpu_internal.h"
#include <chrono>
#endif
#include "cram_index.cuh"
#include "stage_layout.h"
#include <algorithm>
#include <climits>
#include <functional>
#include <map>
#include <string>
#include <vector>
#include <inttypes.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

using cramrec::Rec;
using crai::Run;

namespace {

uint32_t crc32_host(const uint8_t *p, size_t n)             // container headers only: a few dozen bytes per container
{
    uint32_t c = 0xffffffffu;
    for (size_t i = 0; i < n; i++) {
        c ^= p[i];
        for (int k = 0; k < 8; k++) c = (c >> 1) ^ (0xedb88320u & (0u - (c & 1)));
    }
    return ~c;
}

struct Cur {                                                // the file position (htell) and the reads cram_io.c makes there
    const uint8_t *file; uint64_t len, pos;
    bool itf8(int32_t &v)
    {
        if (pos >= len) return false;
        const uint8_t *p = file + pos;
        const uint8_t c = p[0];
        const int n = c < 0x80 ? 0 : c < 0xc0 ? 1 : c < 0xe0 ? 2 : c < 0xf0 ? 3 : 4;
        if (len - pos < (uint64_t)n + 1) return false;
        uint32_t u;
        switch (n) {
        case 0: u = c; break;
        case 1: u = ((c & 0x3fu) << 8) | p[1]; break;
        case 2: u = ((c & 0x1fu) << 16) | (p[1] << 8) | p[2]; break;
        case 3: u = ((c & 0x0fu) << 24) | (p[1] << 16) | (p[2] << 8) | p[3]; break;
        default: u = ((c & 0x0fu) << 28) | (p[1] << 20) | (p[2] << 12) | (p[3] << 4) | (p[4] & 0x0f); break;
        }
        pos += (uint64_t)n + 1;
        v = (int32_t)u;
        return true;
    }
    bool ltf8()
    {
        if (pos >= len) return false;
        const uint8_t c = file[pos];
        int n = 0;
        while (n < 8 && (c << n) & 0x80) n++;
        if (len - pos < (uint64_t)n + 1) return false;
        pos += (uint64_t)n + 1;
        return true;
    }
    bool i32(uint32_t &v)
    {
        if (len - pos < 4) return false;
        const uint8_t *p = file + pos;
        v = p[0] | p[1] << 8 | p[2] << 16 | (uint32_t)p[3] << 24;
        pos += 4;
        return true;
    }
    // cram_read_container (cram_io.c:3760-3945), CRAM 3.x: false where it returns NULL
    bool container(hgpu_cram_container &c, std::vector<int32_t> &landmarks)
    {
        const uint64_t start = pos;
        uint32_t u, crc;
        memset(&c, 0, sizeof c);
        if (!i32(u)) return false;
        c.length = (int32_t)u;
        if (!itf8(c.ref_id) || !itf8(c.start) || !itf8(c.span) || !itf8(c.n_records) || !ltf8() || !ltf8() || !itf8(c.n_blocks) ||
            !itf8(c.n_landmarks) || c.n_landmarks < 0)
            return false;
        landmarks.clear();
        for (int32_t k = 0; k < c.n_landmarks; k++) {
            int32_t v;
            if (!itf8(v)) return false;
            landmarks.push_back(v);
        }
        const uint64_t hdr_end = pos;
        if (!i32(crc) || crc != crc32_host(file + start, hdr_end - start)) return false;
        c.offset = start; c.data_off = pos;
        return true;
    }
    // cram_read_block (cram_io.c:1414-1483): false where it returns NULL.  The CRC is checked where the block is uncompressed.
    bool block(hgpu_cram_block &b, uint32_t container)
    {
        const uint64_t start = pos;
        int32_t cs, us;
        if (len - pos < 2) return false;
        b.method = file[pos]; b.content_type = file[pos + 1];
        pos += 2;
        if (!itf8(b.content_id) || !itf8(cs) || !itf8(us)) return false;
        if (b.method == 0 ? (us < 0 || cs != us) : (cs < 0 || us < 0)) return false;
        if (len - pos < (uint64_t)cs + 4) return false;
        b.data_off = pos; b.hdr_len = (uint16_t)(pos - start); b.comp_size = (uint32_t)cs; b.uncomp_size = (uint32_t)us;
        b.container = container;
        pos += (uint64_t)cs + 4;
        return true;
    }
};

// Where cram_index_build stops: slice index (the slices indexed before it), then the step of cram_index_build it fails in.
// The earliest of the walk's own stop and the refusals found later (block CRCs, multi-reference decodes) is the answer.
enum Step { ST_LENGTH = 0, ST_COMP_HDR = 1, ST_SORT = 2, ST_SLICE = 3, ST_MULTIREF = 4 };
struct Stop {
    int64_t slice = INT64_MAX; int step = 0; int code = HGPU_OK;
    void at(int64_t k, int s, int c) { if (k < slice || (k == slice && s < step)) { slice = k; step = s; code = c; } }
};

struct IdxSlice {                                           // one slice as cram_index_slice sees it
    int64_t cpos; int32_t landmark, sz;
    int32_t ref, start, span;                               // from the slice header
    uint32_t hdr_block, n_blocks;                           // in Walk::blocks
    uint32_t comp_block;                                    // its container's compression header
};

struct Walk {
    std::vector<hgpu_cram_block> blocks;                    // every block read, in file order
    std::vector<IdxSlice> slices;
    std::vector<std::pair<uint32_t, int64_t>> comp_blocks;  // compression header block -> first slice of its container
    int64_t sam_header = -1;                                // the SAM header block (@SQ lines: the decoder checks ref_id with them)
    uint64_t whole = 0;                                     // the file up to the end of the last container that lies in it whole
    Stop stop;
};

// header_payload(block, status) -> the uncompressed payload of a compression / slice header block, nullptr when it will not
// uncompress (the walk then stops there, as cram_uncompress_block fails there).  Its CRC is checked by the caller afterwards.
using Payload = std::function<const uint8_t *(const hgpu_cram_block &)>;

void walk(const uint8_t *file, uint64_t len, const Payload &payload, Walk &W)
{
    Cur c{file, len, 26};
    hgpu_cram_container C;
    std::vector<int32_t> lm;
    // the file header container (cram_read_SAM_hdr): cpos starts past it, padding included
    if (!c.container(C, lm) || C.length < 0 || len - c.pos < (uint64_t)C.length) { W.stop.at(-1, 0, HGPU_IDX_ERR_READ); return; }
    {
        Cur t = c;
        hgpu_cram_block b;
        if (C.n_blocks > 0 && t.block(b, 0) && b.content_type == 0) { W.sam_header = (int64_t)W.blocks.size(); W.blocks.push_back(b); }
    }
    c.pos += (uint64_t)C.length;
    W.whole = c.pos;
    int64_t last_ref = -9, last_start = -9;
    uint32_t ci = 1;                                        // container numbers as hgpu_cram_scan_containers counts them
    std::vector<int32_t> ids(10000);
    while (c.pos < len) {
        const int64_t k0 = (int64_t)W.slices.size();
        const uint64_t cpos = c.pos;
        if (!c.container(C, lm)) return;                    // cram_read_container returns NULL without fd->err: the index ends here
        const uint64_t hpos = c.pos;
        if (C.length >= 0 && len - hpos >= (uint64_t)C.length) W.whole = hpos + (uint64_t)C.length;
        hgpu_cram_block b;
        if (!c.block(b, ci)) { W.stop.at(k0, ST_COMP_HDR, HGPU_IDX_ERR_READ); return; }
        const uint32_t comp = (uint32_t)W.blocks.size();
        W.blocks.push_back(b);
        W.comp_blocks.push_back({comp, k0});
        const uint8_t *ch = payload(b);
        if (!ch || !cramrec::compression_header_ok(ch, b.uncomp_size)) { W.stop.at(k0, ST_COMP_HDR, HGPU_IDX_ERR_READ); return; }
        if (C.ref_id == last_ref && C.start < last_start) { W.stop.at(k0, ST_SORT, HGPU_IDX_ERR_PUSH); return; }
        last_ref = C.ref_id; last_start = C.start;
        for (int32_t j = 0; j < C.n_landmarks; j++) {       // cram_index_container
            const int64_t k = (int64_t)W.slices.size();
            const uint64_t spos = c.pos;
            if ((int64_t)(spos - cpos) - (int64_t)(hpos - cpos) != lm[(size_t)j]) { W.stop.at(k, ST_SLICE, HGPU_IDX_ERR_READ); return; }
            IdxSlice S;
            S.cpos = (int64_t)cpos; S.landmark = lm[(size_t)j]; S.comp_block = comp;
            S.hdr_block = (uint32_t)W.blocks.size();
            hgpu_cram_slice sh;                             // cram_read_slice (cram_io.c:4566-4638)
            if (!c.block(b, ci) || b.content_type != 2) { W.stop.at(k, ST_SLICE, HGPU_IDX_ERR_READ); return; }
            W.blocks.push_back(b);
            const uint8_t *sp = payload(b);
            if (!sp || hgpu_cram_parse_slice_header(sp, b.uncomp_size, 3, &sh, ids.data(), (long)ids.size()) < 0 || sh.n_blocks < 1) {
                W.stop.at(k, ST_SLICE, HGPU_IDX_ERR_READ); return;
            }
            for (int32_t q = 0; q < sh.n_blocks; q++) {
                if (!c.block(b, ci)) { W.stop.at(k, ST_SLICE, HGPU_IDX_ERR_READ); return; }
                W.blocks.push_back(b);
            }
            const uint64_t sz = c.pos - spos;
            if (sz > (uint64_t)INT_MAX) { W.stop.at(k, ST_SLICE, HGPU_IDX_ERR_READ); return; }
            S.sz = (int32_t)sz; S.ref = sh.ref_id; S.start = sh.start; S.span = sh.span; S.n_blocks = (uint32_t)sh.n_blocks;
            W.slices.push_back(S);
        }
        if (C.length < 0 || c.pos != hpos + (uint64_t)C.length) { W.stop.at((int64_t)W.slices.size(), ST_LENGTH, HGPU_IDX_ERR_READ); return; }
        ci++;
    }
}

void line(std::string &t, int32_t ref, int64_t start, int64_t span, int64_t cpos, int32_t landmark, int32_t sz)
{
    char buf[128];
    const int n = snprintf(buf, sizeof buf, "%d\t%" PRId64 "\t%" PRId64 "\t%" PRId64 "\t%d\t%d\n", ref, start, span, cpos, landmark, sz);
    t.append(buf, (size_t)n);
}

// The blocks of the multi-reference slices before the stop, as the record decoder takes them: each container's compression
// header, then every multi-reference slice's header and blocks.  mr[s] = the Walk slice of decoder slice s.
struct MultiRef {
    std::vector<hgpu_cram_block> blocks;
    std::vector<uint32_t> from;                             // Walk block of each
    std::vector<uint64_t> off;                              // udata offset of each
    std::vector<int64_t> mr;
    uint64_t bytes = 0;
};

void multiref_blocks(const Walk &W, MultiRef &M)
{
    int64_t last_comp = -1;
    auto add = [&](uint32_t wb) {
        M.blocks.push_back(W.blocks[wb]); M.from.push_back(wb); M.off.push_back(M.bytes);
        M.bytes += ((uint64_t)W.blocks[wb].uncomp_size + 15) & ~15ull;
    };
    for (size_t k = 0; k < W.slices.size() && (int64_t)k < W.stop.slice; k++) {
        const IdxSlice &S = W.slices[k];
        if (S.ref != -2) continue;
        if (M.mr.empty() && W.sam_header >= 0) add((uint32_t)W.sam_header);
        if ((int64_t)S.comp_block != last_comp) { add(S.comp_block); last_comp = S.comp_block; }
        for (uint32_t q = 0; q <= S.n_blocks; q++) add(S.hdr_block + q);
        M.mr.push_back((int64_t)k);
    }
}

// The text of the index, or the stop.  uncompress(blocks, n, dst, dst_off, status) fills dst + dst_off[i] with block i's
// payload and status[i] with its cram_uncompress_block result; runs(R, runs_of_slice, bad_record) reduces the decoded records.
struct Device {
    std::function<int(const hgpu_cram_block *, uint32_t, uint8_t *, const uint64_t *, int32_t *)> uncompress;
    std::function<int(const cramrec::SliceRecs &, std::vector<std::vector<Run>> &, int64_t &)> runs;
    hgpu_ctx *ctx = nullptr;
};

int index_text(const uint8_t *file, uint64_t len, const Payload &payload, Device &D, std::string &text, int64_t *bad)
{
    *bad = 0;
    text.clear();
    if (!file || len < 26 || memcmp(file, "CRAM", 4) != 0 || file[4] != 3) { hgpu_set_error("cram index: CRAM 3.x only"); return HGPU_ERR_ARG; }
    Walk W;
    walk(file, len, payload, W);
    // CRCs of the header blocks the walk read (cram_uncompress_block checks them before the header is decoded)
    {
        std::vector<hgpu_cram_block> hb;
        std::vector<uint64_t> hoff;
        std::vector<int64_t> at_slice;
        std::vector<int> at_step;
        uint64_t bytes = 0;
        size_t ic = 0;
        for (size_t k = 0; k <= W.slices.size(); k++) {
            for (; ic < W.comp_blocks.size() && W.comp_blocks[ic].second <= (int64_t)k; ic++) {
                hb.push_back(W.blocks[W.comp_blocks[ic].first]); at_slice.push_back(W.comp_blocks[ic].second); at_step.push_back(ST_COMP_HDR);
                hoff.push_back(bytes); bytes += ((uint64_t)hb.back().uncomp_size + 15) & ~15ull;
            }
            if (k < W.slices.size()) {
                hb.push_back(W.blocks[W.slices[k].hdr_block]); at_slice.push_back((int64_t)k); at_step.push_back(ST_SLICE);
                hoff.push_back(bytes); bytes += ((uint64_t)hb.back().uncomp_size + 15) & ~15ull;
            }
        }
        std::vector<uint8_t> hdata(bytes + 16);
        std::vector<int32_t> st(hb.size() + 1);
        int rc = D.uncompress(hb.data(), (uint32_t)hb.size(), hdata.data(), hoff.data(), st.data());
        if (rc) return rc;
        for (size_t i = 0; i < hb.size(); i++) if (st[i]) W.stop.at(at_slice[i], at_step[i], HGPU_IDX_ERR_READ);
    }
    // the multi-reference slices: their used blocks, the record decode and the runs
    MultiRef M;
    multiref_blocks(W, M);
    std::vector<std::vector<Run>> runs;
    if (!M.mr.empty()) {
        const uint32_t n = (uint32_t)M.blocks.size();
        std::vector<uint8_t> udata(M.bytes + 16);
        std::vector<int32_t> st(n + 1);
        std::vector<uint32_t> hdr;
        for (uint32_t i = 0; i < n; i++) if (M.blocks[i].content_type <= 2) hdr.push_back(i);   // the SAM header too
        // the header blocks into a buffer of their own, joined in before each use: an uncompress call writes back the whole span
        // between its first and last slot
        std::vector<uint64_t> ho;
        uint64_t hbytes = 0;
        for (uint32_t i : hdr) { ho.push_back(hbytes); hbytes += ((uint64_t)M.blocks[i].uncomp_size + 15) & ~15ull; }
        std::vector<uint8_t> hdata(hbytes + 16);
        auto join_headers = [&] { for (size_t q = 0; q < hdr.size(); q++) memcpy(udata.data() + M.off[hdr[q]], hdata.data() + ho[q], M.blocks[hdr[q]].uncomp_size); };
        {
            std::vector<hgpu_cram_block> hb;
            for (uint32_t i : hdr) hb.push_back(M.blocks[i]);
            int rc = D.uncompress(hb.data(), (uint32_t)hb.size(), hdata.data(), ho.data(), st.data());
            if (rc) return rc;
            for (size_t q = 0; q < hdr.size(); q++) if (st[q]) { hgpu_set_error("cram index: header block did not uncompress"); return HGPU_IDX_ERR_READ; }
            join_headers();
        }
        std::vector<uint8_t> used(n + 1);
        const int32_t req = cramrec::SAM_RNAME | cramrec::SAM_POS | cramrec::SAM_CIGAR;
        if (hgpu_cram_required_blocks(M.blocks.data(), n, udata.data(), M.off.data(), (uint32_t)req, used.data()) < 0) {
            W.stop.at(M.mr[0], ST_MULTIREF, HGPU_IDX_ERR_READ);
        } else {
            std::vector<uint32_t> body;
            for (uint32_t i = 0; i < n; i++) if (used[i] && M.blocks[i].content_type > 2) body.push_back(i);
            std::vector<hgpu_cram_block> bb;
            std::vector<uint64_t> bo;
            for (uint32_t i : body) { bb.push_back(M.blocks[i]); bo.push_back(M.off[i]); }
            std::vector<int32_t> bst(body.size() + 1);
            int rc = D.uncompress(bb.data(), (uint32_t)bb.size(), udata.data(), bo.data(), bst.data());
            if (rc) return rc;
            join_headers();
            // a block that fails its CRC or its codec fails the slice that owns it
            std::vector<uint8_t> slice_bad(M.mr.size(), 0);
            {
                size_t s = 0;
                int64_t cur = -1;
                std::vector<int64_t> owner(n, -1);
                for (uint32_t i = 0; i < n; i++) {
                    if (M.blocks[i].content_type == 2) cur = (int64_t)s++;
                    else if (M.blocks[i].content_type == 1) cur = -1;
                    owner[i] = cur;
                }
                for (size_t q = 0; q < body.size(); q++) if (bst[q] && owner[body[q]] >= 0) slice_bad[(size_t)owner[body[q]]] = 1;
            }
            cramrec::SliceRecs R;
            rc = cramrec::slice_records(D.ctx, file, W.whole, M.blocks.data(), n, udata.data(), M.off.data(), req, R);
            if (rc == HGPU_CRAM_ERR_DECODE) W.stop.at(M.mr[0], ST_MULTIREF, HGPU_IDX_ERR_READ);
            else if (rc) return rc;
            else {
                int64_t bad_rec = -1;
                if ((rc = D.runs(R, runs, bad_rec))) return rc;
                for (size_t s = 0; s < M.mr.size(); s++) if (slice_bad[s] || R.status[s]) W.stop.at(M.mr[s], ST_MULTIREF, HGPU_IDX_ERR_READ);
                if (bad_rec >= 0) {
                    const size_t s = (size_t)(std::upper_bound(R.rec0.begin(), R.rec0.end(), (uint64_t)bad_rec) - R.rec0.begin()) - 1;
                    W.stop.at(M.mr[s], ST_MULTIREF, HGPU_IDX_ERR_READ);   // -2 of cram_index_slice, -1 once cram_index_container returns it
                }
            }
        }
    }
    if (W.stop.code != HGPU_OK) {
        *bad = W.stop.slice;
        hgpu_set_error("cram index: %s at slice %" PRId64 " (step %d)", W.stop.code == HGPU_IDX_ERR_PUSH ? "containers out of order" : "read failure", W.stop.slice, W.stop.step);
        return W.stop.code;
    }
    size_t m = 0;
    for (size_t k = 0; k < W.slices.size(); k++) {
        const IdxSlice &S = W.slices[k];
        if (S.ref != -2) { line(text, S.ref, S.start, S.span, S.cpos, S.landmark, S.sz); continue; }
        for (const Run &r : runs[m]) line(text, r.ref, r.start, r.end - r.start + 1, S.cpos, S.landmark, S.sz);
        m++;
    }
    return HGPU_OK;
}

#ifndef HGPU_HOSTSIM
// ---- device ----
// A warp per multi-reference slice.  Pass 1 (WRITE = false) counts each slice's runs and finds the first record out of order
// (one atomicMin of its record index); pass 2 writes the runs at the slice's offset of the scanned counts.  Run starts are a
// ballot of run_start; a run's largest aend is a segmented max scan inside the 32-record chunk, carried across chunks.
template <bool WRITE>
__global__ void __launch_bounds__(32) cram_index_runs_kernel(const Rec *__restrict__ recs, const uint64_t *__restrict__ rec0, uint32_t ns,
        uint32_t *count, const uint32_t *__restrict__ run_off, Run *out, unsigned long long *first_bad)
{
    const uint32_t s = blockIdx.x;
    if (s >= ns) return;
    const uint32_t lane = threadIdx.x & 31;
    const Rec *r = recs + rec0[s];
    const int32_t n = (int32_t)(rec0[s + 1] - rec0[s]);
    uint32_t runs = 0;                                      // runs opened before this chunk
    int32_t c_ref = 0;                                      // the run open at the end of the previous chunk
    int64_t c_start = 0, c_end = 0;
    Run *o = WRITE ? out + run_off[s] : nullptr;
    for (int32_t base = 0; base < n; base += 32) {
        const int32_t i = base + (int32_t)lane;
        const bool valid = i < n;
        const uint32_t starts = __ballot_sync(0xffffffffu, valid && crai::run_start(r, i));
        if (!WRITE) {
            const uint32_t back = __ballot_sync(0xffffffffu, valid && crai::unsorted(r, i));
            if (back) { if (lane == 0) atomicMin(first_bad, (unsigned long long)(rec0[s] + (uint64_t)base + (uint64_t)(__ffs(back) - 1))); return; }
            runs += (uint32_t)__popc(starts);
            continue;
        }
        const int32_t last = (n - base < 32 ? n - base : 32) - 1;
        const uint32_t mine = starts & (lane == 31 ? 0xffffffffu : (2u << lane) - 1u);
        const int32_t seg = mine ? 31 - __clz(mine) : -1;   // the lane that opened this lane's run, -1: the carried run
        const int32_t ref = valid ? r[i].ref_id : 0;
        long long v = valid ? (long long)r[i].aend : LLONG_MIN;
        for (int d = 1; d < 32; d <<= 1) {
            const long long t = __shfl_up_sync(0xffffffffu, v, d);
            if ((int32_t)lane >= d && (int32_t)lane - d >= seg) v = t > v ? t : v;
        }
        const long long apos = __shfl_sync(0xffffffffu, valid ? (long long)r[i].apos : 0LL, seg < 0 ? 0 : seg);
        const long long start = seg < 0 ? (long long)c_start : apos;
        if (seg < 0 && (long long)c_end > v) v = (long long)c_end;
        if ((starts & 1u) && runs > 0 && lane == 0) o[runs - 1] = Run{c_ref, 0, c_start, c_end};   // the carried run ended with the chunk before
        if (valid && (int32_t)lane < last && ((starts >> (lane + 1)) & 1u))
            o[seg < 0 ? runs - 1 : runs + (uint32_t)__popc(mine) - 1] = Run{ref, 0, (int64_t)start, (int64_t)v};
        c_ref = __shfl_sync(0xffffffffu, ref, last);
        c_start = (int64_t)__shfl_sync(0xffffffffu, start, last);
        c_end = (int64_t)__shfl_sync(0xffffffffu, v, last);
        runs += (uint32_t)__popc(starts);
    }
    if (WRITE) { if (runs > 0 && lane == 0) o[runs - 1] = Run{c_ref, 0, c_start, c_end}; }
    else if (lane == 0) count[s] = runs;
}

float g_last_ms[2];
float g_dev_ms;                                             // device time of the current call, summed

int device_runs(hgpu_ctx *ctx, const cramrec::SliceRecs &R, std::vector<std::vector<Run>> &runs, int64_t &bad_rec)
{
    const uint32_t ns = (uint32_t)R.status.size();
    runs.assign(ns, {});
    bad_rec = -1;
    if (ns == 0) return HGPU_OK;
    cudaStream_t st = ctx->stream;
    // the records stay where slice_records left them (the staging area); the runs go to the second staging area
    const uint64_t n_rec = R.rec0[ns];
    StageLayout L;
    const auto s_rec0 = L.seg(8 * ((size_t)ns + 1)), s_cnt = L.seg(4 * (size_t)ns), s_off = L.seg(4 * (size_t)ns), s_bad = L.seg(8);
    int rc = hgpu_ensure_mrec(ctx, L.total + (n_rec + 1) * sizeof(Run) + 256);
    if (rc) return rc;
    L.base = ctx->d_mrec;
    Run *d_runs = reinterpret_cast<Run *>(ctx->d_mrec + StageLayout::align(L.total));
    const unsigned long long none = ~0ull;
    std::vector<uint32_t> cnt(ns), off(ns);
    cudaEvent_t ev[4];
    int ne = 0;
    for (; ne < 4; ne++) if (cudaEventCreate(&ev[ne]) != cudaSuccess) break;
    struct Free { cudaEvent_t *e; int n; ~Free() { for (int k = 0; k < n; k++) cudaEventDestroy(e[k]); } } fr{ev, ne};
    if (ne < 4) return HGPU_ERR_CUDA;
    if (hgpu_h2d(L.at(s_rec0), R.rec0.data(), 8 * ((size_t)ns + 1), st) || hgpu_memset(L.at(s_cnt), 0, 4 * (size_t)ns, st) ||
        hgpu_h2d(L.at(s_bad), &none, 8, st)) return HGPU_ERR_CUDA;
    cudaEventRecord(ev[0], st);
    cram_index_runs_kernel<false><<<ns, 32, 0, st>>>(R.recs, L.at<uint64_t>(s_rec0), ns, L.at<uint32_t>(s_cnt), nullptr, nullptr,
                                                     L.at<unsigned long long>(s_bad));
    cudaEventRecord(ev[1], st);
    hgpu_count_launch();
    if (hgpu_check(cudaGetLastError(), "cram index runs launch")) return HGPU_ERR_CUDA;
    unsigned long long b = none;
    if (hgpu_d2h(cnt.data(), L.at(s_cnt), 4 * (size_t)ns, st) || hgpu_d2h(&b, L.at(s_bad), 8, st) ||
        hgpu_check(cudaStreamSynchronize(st), "cram index runs")) return HGPU_ERR_CUDA;
    float ms = 0;
    cudaEventElapsedTime(&ms, ev[0], ev[1]);
    g_dev_ms += ms;
    if (b != none) { bad_rec = (int64_t)b; return HGPU_OK; }
    uint64_t total = 0;
    for (uint32_t s = 0; s < ns; s++) { off[s] = (uint32_t)total; total += cnt[s]; }
    if (hgpu_h2d(L.at(s_off), off.data(), 4 * (size_t)ns, st)) return HGPU_ERR_CUDA;
    cudaEventRecord(ev[2], st);
    cram_index_runs_kernel<true><<<ns, 32, 0, st>>>(R.recs, L.at<uint64_t>(s_rec0), ns, nullptr, L.at<uint32_t>(s_off), d_runs, nullptr);
    cudaEventRecord(ev[3], st);
    hgpu_count_launch();
    if (hgpu_check(cudaGetLastError(), "cram index runs launch")) return HGPU_ERR_CUDA;
    std::vector<Run> all(total + 1);
    if (hgpu_d2h(all.data(), d_runs, total * sizeof(Run), st) || hgpu_check(cudaStreamSynchronize(st), "cram index runs")) return HGPU_ERR_CUDA;
    cudaEventElapsedTime(&ms, ev[2], ev[3]);
    g_dev_ms += ms;
    for (uint32_t s = 0; s < ns; s++) runs[s].assign(all.begin() + off[s], all.begin() + off[s] + cnt[s]);
    return HGPU_OK;
}

// One gzip member (RFC 1952) of text, as bgzf_open(fn, "wg") writes the index: 0xff00-byte payloads through
// bgzf_deflate_kernel, one deflate block each, spliced into one stream.  Each block but the last gets BFINAL cleared and an
// empty stored block after it, which brings the next block to a byte boundary: its 3 header bits (zero) and the padding to
// the byte go into the block's last byte when at least 3 of its bits are free (then LEN / NLEN: 00 00 FF FF), into one more
// zero byte otherwise (00 00 00 FF FF).  Then the CRC-32 of the text and ISIZE.
int gzip_member(hgpu_ctx *ctx, const std::string &text, std::vector<uint8_t> &out)
{
    static const uint8_t hdr[10] = {0x1f, 0x8b, 8, 0, 0, 0, 0, 0, 0, 0xff};
    out.assign(hdr, hdr + 10);
    const uint32_t n = (uint32_t)((text.size() + 0xff00 - 1) / 0xff00);
    if (n == 0) {
        static const uint8_t empty[2] = {0x03, 0x00};       // one empty fixed-Huffman block, final
        out.insert(out.end(), empty, empty + 2);
    } else {
        std::vector<uint64_t> off(2 * (size_t)n);
        std::vector<uint32_t> len(n), olen(n), bits(n);
        std::vector<int32_t> st(n);
        for (uint32_t i = 0; i < n; i++) {
            off[i] = (uint64_t)i * 0xff00;
            len[i] = (uint32_t)std::min<uint64_t>(0xff00, text.size() - off[i]);
            off[n + i] = (uint64_t)i * 65536;
        }
        StageLayout L;
        const auto s_in = L.seg(text.size() + 4), s_off = L.seg(16 * (size_t)n), s_len = L.seg(4 * (size_t)n),
                   s_out = L.seg(65536 * (size_t)n), s_olen = L.seg(4 * (size_t)n), s_st = L.seg(4 * (size_t)n), s_bits = L.seg(4 * (size_t)n);
        int rc = hgpu_stage_ensure(ctx, L);
        if (rc) return rc;
        cudaStream_t s = ctx->stream;
        if (hgpu_h2d(L.at(s_in), text.data(), text.size(), s) || hgpu_h2d(L.at(s_off), off.data(), 16 * (size_t)n, s) ||
            hgpu_h2d(L.at(s_len), len.data(), 4 * (size_t)n, s)) return HGPU_ERR_CUDA;
        rc = hgpu_launch_bgzf_deflate(ctx, L.at(s_in), L.at<uint64_t>(s_off), L.at<uint32_t>(s_len), n, -1, L.at(s_out),
                                      L.at<uint64_t>(s_off) + n, L.at<uint32_t>(s_olen), L.at<int32_t>(s_st), L.at<uint32_t>(s_bits), s);
        if (rc) return rc;
        std::vector<uint8_t> blocks(65536 * (size_t)n);
        if (hgpu_d2h(blocks.data(), L.at(s_out), blocks.size(), s) || hgpu_d2h(olen.data(), L.at(s_olen), 4 * (size_t)n, s) ||
            hgpu_d2h(st.data(), L.at(s_st), 4 * (size_t)n, s) || hgpu_d2h(bits.data(), L.at(s_bits), 4 * (size_t)n, s) ||
            hgpu_check(cudaStreamSynchronize(s), "sync")) return HGPU_ERR_CUDA;
        for (uint32_t i = 0; i < n; i++) {
            if (st[i] != HGPU_OK) { hgpu_set_error("index deflate block %u: status %d", i, st[i]); return HGPU_ERR_CUDA; }
            const uint8_t *body = blocks.data() + (size_t)i * 65536 + 18;
            const uint32_t nbytes = (bits[i] + 7) / 8, spare = 8 * nbytes - bits[i];
            const size_t at = out.size();
            out.insert(out.end(), body, body + nbytes);
            if (i + 1 == n) break;
            out[at] &= 0xfe;                                // BFINAL
            static const uint8_t sync4[4] = {0, 0, 0xff, 0xff}, sync5[5] = {0, 0, 0, 0xff, 0xff};
            if (spare >= 3) out.insert(out.end(), sync4, sync4 + 4);
            else out.insert(out.end(), sync5, sync5 + 5);
        }
    }
    const uint32_t crc = text.empty() ? 0 : hgpu_crc32(ctx, 0, text.data(), text.size());
    if (hgpu_crc32_failed()) return HGPU_ERR_CUDA;
    const uint32_t isize = (uint32_t)text.size();
    for (int k = 0; k < 4; k++) out.push_back((uint8_t)(crc >> (8 * k)));
    for (int k = 0; k < 4; k++) out.push_back((uint8_t)(isize >> (8 * k)));
    return HGPU_OK;
}

int cram_index_build_impl(hgpu_ctx *ctx, const uint8_t *file, uint64_t file_len, uint8_t **out, uint64_t *out_len, int64_t *bad)
{
    g_last_ms[0] = g_last_ms[1] = 0;
    g_dev_ms = 0;
    if (!ctx || !out || !out_len || !bad) { hgpu_set_error("cram index: null argument"); return HGPU_ERR_ARG; }
    *out = nullptr; *out_len = 0; *bad = 0;
    if (cudaSetDevice(ctx->device) != cudaSuccess) return HGPU_ERR_CUDA;
    const auto h0 = std::chrono::steady_clock::now();
    // a header block that is not RAW (no writer makes one) is uncompressed on its own as the walk reaches it
    std::vector<std::vector<uint8_t>> kept;
    Payload payload = [&](const hgpu_cram_block &b) -> const uint8_t * {
        if (b.method == 0) return file + b.data_off;
        kept.emplace_back((size_t)b.uncomp_size + 16);
        const uint64_t o = 0;
        uint32_t got = 0;
        int32_t st = 0;
        if (hgpu_cram_uncompress_blocks_host(ctx, file, file_len, &b, 1, kept.back().data(), &o, &got, &st) || st) return nullptr;
        return kept.back().data();
    };
    Device D;
    D.ctx = ctx;
    D.uncompress = [&](const hgpu_cram_block *b, uint32_t n, uint8_t *dst, const uint64_t *dst_off, int32_t *st) -> int {
        if (n == 0) return HGPU_OK;
        std::vector<uint32_t> got(n + 1);
        return hgpu_cram_uncompress_blocks_host(ctx, file, file_len, b, n, dst, dst_off, got.data(), st);
    };
    D.runs = [&](const cramrec::SliceRecs &R, std::vector<std::vector<Run>> &runs, int64_t &bad_rec) -> int {
        g_dev_ms += R.ms;
        return device_runs(ctx, R, runs, bad_rec);
    };
    std::string text;
    int rc = index_text(file, file_len, payload, D, text, bad);
    if (rc) return rc;
    std::vector<uint8_t> gz;
    if ((rc = gzip_member(ctx, text, gz))) return rc;
    *out = (uint8_t *)malloc(gz.size());
    if (!*out) { hgpu_set_error("out of host memory"); return HGPU_ERR_NOMEM; }
    memcpy(*out, gz.data(), gz.size());
    *out_len = gz.size();
    g_last_ms[0] = g_dev_ms;
    g_last_ms[1] = std::chrono::duration<float, std::milli>(std::chrono::steady_clock::now() - h0).count() - g_dev_ms;
    return HGPU_OK;
}
#endif

}  // namespace

#ifdef HGPU_HOSTSIM
// The index text of a CRAM image, the multi-reference slices through slice_records and slice_runs on the host.  blocks /
// udata / udata_off / status: what the per-codec checkers made of the blocks of this image (or of a longer one it is a prefix
// of), status[i] != 0 where block i fails its CRC or its codec.  *text (malloc'd) and *text_len: the index text on HGPU_OK.
extern "C" int hostsim_cram_index_text(const uint8_t *file, uint64_t file_len, const hgpu_cram_block *blocks, uint32_t n_blocks,
        const uint8_t *udata, const uint64_t *udata_off, const int32_t *status, char **text, uint64_t *text_len, int64_t *bad)
{
    try {
        std::map<uint64_t, uint32_t> at;
        for (uint32_t i = 0; i < n_blocks; i++) at[blocks[i].data_off] = i;
        auto find = [&](const hgpu_cram_block &b) -> int64_t { auto it = at.find(b.data_off); return it == at.end() ? -1 : (int64_t)it->second; };
        Payload payload = [&](const hgpu_cram_block &b) -> const uint8_t * { const int64_t i = find(b); return i < 0 ? nullptr : udata + udata_off[i]; };
        Device D;
        D.uncompress = [&](const hgpu_cram_block *b, uint32_t n, uint8_t *dst, const uint64_t *dst_off, int32_t *st) -> int {
            for (uint32_t k = 0; k < n; k++) {
                const int64_t i = find(b[k]);
                st[k] = i < 0 ? HGPU_CRAM_ERR_DECODE : status[i];
                if (i >= 0) memcpy(dst + dst_off[k], udata + udata_off[i], b[k].uncomp_size);
            }
            return HGPU_OK;
        };
        D.runs = [&](const cramrec::SliceRecs &R, std::vector<std::vector<Run>> &runs, int64_t &bad_rec) -> int {
            const size_t ns = R.status.size();
            runs.assign(ns, {});
            bad_rec = -1;
            for (size_t s = 0; s < ns; s++) {
                const Rec *r = R.recs + R.rec0[s];
                const int32_t n = (int32_t)(R.rec0[s + 1] - R.rec0[s]);
                int32_t b;
                runs[s].resize((size_t)n);
                runs[s].resize((size_t)crai::slice_runs(r, n, runs[s].data(), &b));
                if (b >= 0 && bad_rec < 0) bad_rec = (int64_t)(R.rec0[s] + (uint64_t)b);
            }
            return HGPU_OK;
        };
        std::string t;
        const int rc = index_text(file, file_len, payload, D, t, bad);
        *text = (char *)malloc(t.size() + 1);
        memcpy(*text, t.data(), t.size());
        *text_len = t.size();
        return rc;
    } catch (...) { hgpu_set_error("internal error"); return HGPU_ERR_NOMEM; }
}
#else
extern "C" int hgpu_cram_index_build_host(hgpu_ctx *ctx, const uint8_t *file, uint64_t file_len, uint8_t **out, uint64_t *out_len, int64_t *bad)
{
    return hgpu_abi_call([&] { return cram_index_build_impl(ctx, file, file_len, out, out_len, bad); });
}

extern "C" void hgpu_cram_index_last_ms(float *ms2)
{
    if (ms2) { ms2[0] = g_last_ms[0]; ms2[1] = g_last_ms[1]; }
}
#endif
