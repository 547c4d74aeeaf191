// The CRAI lines of a multi-reference slice, host/device portable: cram_index_build_multiref (cram/cram_index.c:632-690) over
// the records cram_decode_slice leaves with CRAM_OPT_REQUIRED_FIELDS = SAM_RNAME | SAM_POS | SAM_CIGAR.  One line per run of
// records with equal ref_id: the run's first apos and its largest aend.  cram_index.cu runs these predicates a warp per slice
// (cram_index_runs_kernel); slice_runs below is the same rule as one loop, which the host-only test build runs.
#pragma once
#include <stdint.h>
#include "cram_records.cuh"

#ifdef __CUDACC__
#define CRAI_HD __host__ __device__ __forceinline__
#else
#define CRAI_HD inline
#endif

namespace crai {

struct Run { int32_t ref, pad; int64_t start, end; };      // one index line: ref, start, end (span = end - start + 1)

// record i opens a run: the first record, or a ref_id other than its predecessor's (`ref` starts at -2, which no record has)
CRAI_HD bool run_start(const cramrec::Rec *r, int32_t i) { return i == 0 || r[i].ref_id != r[i - 1].ref_id; }

// record i goes backwards: the reference compares apos with the predecessor's apos held in an int32_t `last_pos` (:653-656)
CRAI_HD bool unsorted(const cramrec::Rec *r, int32_t i)
{
    return i > 0 && r[i].ref_id == r[i - 1].ref_id && r[i].apos < (int64_t)(int32_t)r[i - 1].apos;
}

// the whole rule for one slice of n records: returns the number of runs (written to out when not null) and sets *bad to the
// first record that goes backwards, -1 when none does (the reference writes nothing for a slice it refuses)
CRAI_HD int32_t slice_runs(const cramrec::Rec *r, int32_t n, Run *out, int32_t *bad)
{
    int32_t k = -1;
    *bad = -1;
    for (int32_t i = 0; i < n; i++) {
        if (unsorted(r, i)) { *bad = i; return 0; }
        if (run_start(r, i)) {
            k++;
            if (out) { out[k].ref = r[i].ref_id; out[k].pad = 0; out[k].start = r[i].apos; out[k].end = r[i].aend; }
        } else if (out && out[k].end < r[i].aend) out[k].end = r[i].aend;
    }
    return k + 1;
}

}  // namespace crai
