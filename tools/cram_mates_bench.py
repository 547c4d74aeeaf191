#!/usr/bin/env python
"""Mate attachment in the device CRAM writer (HGPU_CRAM_ENC_ATTACH_MATES): file size, mate series sizes, attached fraction and
times, with and without the flag, on bench-shaped paired records; beside it the reference's writer (oracle/_ref) on the same
records with the same records per slice.

Records: the synthetic coordinate-sorted paired-end SAM of tests/test_cram_records.py over CHROMOSOME_I of ce.fa (100 bp reads,
every read-feature code, 3 read groups, 3% unmapped mates), read by the reference's SAM reader, tiled K times (records per slice
divide the tile, so no slice holds two copies of a name).

  python tools/cram_mates_bench.py [reads_per_tile] [tiles] [records_per_slice] [out.json]
"""
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

SERIES = {"CF": 2, "MF": 8, "NS": 9, "NP": 10, "TS": 11, "NF": 32}


def series_bytes(H, img):
    """Compressed and uncompressed bytes per mate series (content id), summed over slices."""
    blocks, _ = H.cram_scan_blocks(np.frombuffer(img, dtype=np.uint8).copy())
    ext = blocks[blocks["content_type"] == 4]
    comp = {k: int(ext["comp_size"][ext["content_id"] == cid].astype(np.int64).sum()) for k, cid in SERIES.items()}
    raw = {k: int(ext["uncomp_size"][ext["content_id"] == cid].astype(np.int64).sum()) for k, cid in SERIES.items()}
    return comp, raw


def gpu_info():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as ex:
        return repr(ex)


def run(ctx, reads=100000, tiles=10, rps=10000, reps=3):
    import htslib_b200 as H
    from _libs import ref, ref_read_sam_records, ref_cram_read_all, _ref_write_cram_to
    import test_cram_records as T
    from test_cram_encode import pack, expected
    if ref() is None:
        return {"error": "oracle/_ref not built (the records come from the reference's SAM reader)"}
    assert reads % rps == 0, "records per slice must divide the tile"
    tmp = tempfile.mkdtemp()
    sam = os.path.join(tmp, "syn.sam")
    n1 = T._synthetic_sam(sam, n=reads, seed=11)
    text, recs1 = ref_read_sam_records.__wrapped__(sam)
    assert len(recs1) == n1
    recs = recs1 * tiles
    n = len(recs)
    core, data, off = pack(recs)
    fa = os.path.join(T.HT, "ce.fa")
    fasta = H.load_fasta_upper(fa, [b"CHROMOSOME_I"])
    res = {"gpu": gpu_info(), "records": n, "records_per_slice": rps,
           "workload": "%d synthetic 100 bp paired reads (tests/test_cram_records._synthetic_sam, seed 11) tiled %dx, CRAM 3.1" % (n1, tiles)}
    for shape, fz in (("no_reference", None), ("reference", fasta)):
        out = {}
        for label, flags in (("detached", 0), ("attached", H.CRAM_ENC_ATTACH_MATES)):
            H.cram_encode_records(ctx, text, core, data, off, n, fz, rps, 1, flags)          # warm-up
            walls, pair, cw = [], [], []
            for _ in range(reps):
                t0 = time.perf_counter()
                img = H.cram_encode_records(ctx, text, core, data, off, n, fz, rps, 1, flags)
                walls.append(time.perf_counter() - t0)
                a, b = H.cram_encode_last_ms()
                pair.append(a); cw.append(b)
            comp, raw = series_bytes(H, img)
            wall = sorted(walls)[len(walls) // 2]
            out[label] = {"file_bytes": len(img), "bytes_per_record": len(img) / n, "series_comp_bytes": comp,
                          "attached_fraction": 1.0 - raw["MF"] / n,          # one MF byte (value 0) per detached record
                          "e2e_wall_s_median": wall, "records_per_s_e2e": n / wall,
                          "pair_kernels_ms_median": sorted(pair)[len(pair) // 2], "count_write_kernels_ms_median": sorted(cw)[len(cw) // 2]}
            if label == "attached":                                            # the reference reads the first tile back
                path = os.path.join(tmp, "att.cram")
                open(path, "wb").write(img)
                back = ref_cram_read_all.__wrapped__(path, fa if fz is not None else None, 0)
                assert len(back) == n
                for i in list(range(0, n1, max(1, n1 // 2000))) + [n - 1]:
                    assert back[i] == expected(*recs[i]), i
        # the reference's writer on the same records: SAM text tiled the same way, same records per slice
        tiled = os.path.join(tmp, "tiled.sam")
        with open(sam, "rb") as f:
            lines = f.read().split(b"\n")
        hdr = [l for l in lines if l.startswith(b"@")]
        body = [l for l in lines if l and not l.startswith(b"@")]
        with open(tiled, "wb") as f:
            f.write(b"\n".join(hdr + body * tiles) + b"\n")
        rout = os.path.join(tmp, "ref.cram")
        opts = [(3, rps)] + ([(11, 1)] if fz is None else [])                 # CRAM_OPT_SEQS_PER_SLICE, CRAM_OPT_NO_REF
        t0 = time.perf_counter()
        assert _ref_write_cram_to(tiled, fa, rout, "3.1", opts) == n
        # (its content ids are not ours, so only the file size compares)
        out["reference_writer"] = {"file_bytes": os.path.getsize(rout), "bytes_per_record": os.path.getsize(rout) / n,
                                   "wall_s_1core": time.perf_counter() - t0}
        out["attached_over_detached"] = out["attached"]["file_bytes"] / out["detached"]["file_bytes"]
        out["attached_over_reference"] = out["attached"]["file_bytes"] / out["reference_writer"]["file_bytes"]
        res[shape] = out
    return res


if __name__ == "__main__":
    import torch
    import htslib_b200 as H
    torch.cuda.set_device(0)
    ctx = H.Context(0)
    reads = int(sys.argv[1]) if len(sys.argv) > 1 else 100000
    tiles = int(sys.argv[2]) if len(sys.argv) > 2 else 10
    rps = int(sys.argv[3]) if len(sys.argv) > 3 else 10000
    r = run(ctx, reads, tiles, rps)
    print(json.dumps(r))
    if len(sys.argv) > 4:
        with open(sys.argv[4], "w") as f:
            json.dump(r, f, indent=1)
    ctx.close()
