#!/usr/bin/env python
"""Tag blocks in the device CRAM writer (HGPU_CRAM_ENC_TAG_BLOCKS): file bytes per record, compressed bytes per tag block, device time
of the tag pass and of the count / write kernels, and end-to-end records/s, for {bit off, on} x {no reference, reference} x
{mates off, on}; beside it the reference's writer (oracle/_ref) on the same records with the same records per slice.

Records: tests/test_cram_tags.synthetic_tagged — sorted paired 100 bp reads over CHROMOSOME_I of ce.fa with substitutions, indels and
skips, 3 @RG lines, NH / AS / XA, MD / NM as an aligner writes them (5 % of NM deliberately wrong).

  python tools/cram_tags_bench.py [pairs (100 000)] [records_per_slice] [out.json] [--skip-reference-writer]
"""
import json
import os
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from cram_mates_bench import gpu_info                                     # noqa: E402


def tag_blocks(H, img):
    """Compressed bytes per tag key (content id >= 2^16, as 'XX:t'), and of the two shared tag streams, summed over slices."""
    blocks, _ = H.cram_scan_blocks(np.frombuffer(img, dtype=np.uint8).copy())
    ext = blocks[blocks["content_type"] == 4]
    out = {}
    for cid, cs in zip(ext["content_id"].tolist(), ext["comp_size"].tolist()):
        k = "%c%c:%c" % (cid >> 16, (cid >> 8) & 255, cid & 255) if cid > 0xffff else {29: "shared_len", 30: "shared_val", 6: "RG"}.get(cid)
        if k:
            out[k] = out.get(k, 0) + int(cs)
    return out


def run(ctx, pairs=100000, rps=10000, reps=3, reference_writer=True):
    import htslib_b200 as H
    from _libs import ref, _ref_write_cram_to
    from test_cram_encode import pack
    import test_cram_tags as TT
    t0 = time.perf_counter()
    text, recs, fasta = TT.synthetic_tagged(pairs)
    print("records built in %.1f s" % (time.perf_counter() - t0), flush=True)
    n = len(recs)
    core, data, off = pack(recs)
    res = {"gpu": gpu_info(), "records": n, "records_per_slice": rps,
           "workload": "%d synthetic paired 100 bp reads with MD/NM/RG/NH/AS/XA (tests/test_cram_tags.synthetic_tagged), CRAM 3.1" % n}
    for shape, fz in (("no_reference", None), ("reference", fasta)):
        out = {}
        for mates in (False, True):
            for tb in (False, True):
                flags = (H.CRAM_ENC_ATTACH_MATES if mates else 0) | (H.CRAM_ENC_TAG_BLOCKS if tb else 0)
                H.cram_encode_records(ctx, text, core, data, off, n, fz, rps, 1, flags)          # warm-up
                walls, tag, cw = [], [], []
                for _ in range(reps):
                    t0 = time.perf_counter()
                    img = H.cram_encode_records(ctx, text, core, data, off, n, fz, rps, 1, flags)
                    walls.append(time.perf_counter() - t0)
                    tag.append(H.cram_encode_tags_last_ms())
                    cw.append(H.cram_encode_last_ms()[1])
                wall = sorted(walls)[len(walls) // 2]
                out["tags_%s_mates_%s" % ("on" if tb else "off", "on" if mates else "off")] = {
                    "file_bytes": len(img), "bytes_per_record": len(img) / n, "tag_block_comp_bytes": tag_blocks(H, img),
                    "tag_pass_ms_median": sorted(tag)[len(tag) // 2], "count_write_kernels_ms_median": sorted(cw)[len(cw) // 2],
                    "e2e_wall_s_median": wall, "records_per_s_e2e": n / wall}
                print(shape, "mates", mates, "tags", tb, len(img), flush=True)
        if reference_writer and ref() is not None:                              # the reference's writer, same records per slice
            tmp = tempfile.mkdtemp()
            bam = os.path.join(tmp, "syn.bam")
            with open(bam, "wb") as f:
                f.write(TT.bam_image(text, [(b"CHROMOSOME_I", int(fasta[1][1]))], recs))
            rout = os.path.join(tmp, "ref.cram")
            opts = [(TT.MULTI, 1), (TT.SEQS, rps)] + ([(TT.NO_REF, 1)] if fz is None else [])
            t0 = time.perf_counter()
            assert _ref_write_cram_to(bam, os.path.join(TT.T.HT, "ce.fa"), rout, "3.1", opts) == n
            ref_img = open(rout, "rb").read()
            print(shape, "reference writer", len(ref_img), flush=True)
            out["reference_writer"] = {"file_bytes": len(ref_img), "bytes_per_record": len(ref_img) / n,
                                       "wall_s_1core": time.perf_counter() - t0}
            for k in list(out):
                if k.startswith("tags_"):
                    out[k]["over_reference_writer"] = out[k]["file_bytes"] / len(ref_img)
        res[shape] = out
    return res


if __name__ == "__main__":
    import torch
    import htslib_b200 as H
    torch.cuda.set_device(0)
    ctx = H.Context(0)
    pairs = int(sys.argv[1]) if len(sys.argv) > 1 else 100000
    rps = int(sys.argv[2]) if len(sys.argv) > 2 else 10000
    r = run(ctx, pairs, rps, reference_writer="--skip-reference-writer" not in sys.argv)
    print(json.dumps(r))
    if len(sys.argv) > 3:
        with open(sys.argv[3], "w") as f:
            json.dump(r, f, indent=1)
    ctx.close()
