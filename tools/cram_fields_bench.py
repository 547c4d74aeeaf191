#!/usr/bin/env python
"""Field-subset CRAM decode (CRAM_OPT_REQUIRED_FIELDS) on the tiled synthetic CRAM 3.1 file of tools/cram_records_bench.py.
For each mask: end-to-end wall time of hgpu_cram_decode_file_fields_host (scan + uncompress of the used blocks + record decode,
best of 3), device time of cram_slice_decode_kernel and cram_bam_fill_kernel, the uncompressed bytes of the blocks the
selection uses, and the reference's single-core sam_read1 rate with the same option.  The first and last tile are checked
against the reference's records on sampled reads.  Needs oracle/_ref (the reference writes the file and is the CPU baseline).

  python tools/cram_fields_bench.py [reads_per_unique_file] [tiles]
"""
import ctypes as C
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
sys.path.insert(0, os.path.join(ROOT, "tools"))


def masks(H):
    return {"all": H.SAM_ALL, "FLAG|MAPQ|RNEXT": H.SAM_FLAG | H.SAM_MAPQ | H.SAM_RNEXT,
            "RNAME|POS|CIGAR": H.SAM_RNAME | H.SAM_POS | H.SAM_CIGAR, "all but QUAL": H.SAM_ALL & ~H.SAM_QUAL}


def cpu_rate(path, fasta, mask, limit=500000):
    """Records per second of the reference's sam_read1 loop on one core with CRAM_OPT_REQUIRED_FIELDS = mask."""
    from _libs import Bam1, ref
    r = ref()
    r.hts_open.restype = C.c_void_p
    r.hts_open.argtypes = [C.c_char_p, C.c_char_p]
    r.hts_close.argtypes = [C.c_void_p]
    r.hts_set_fai_filename.argtypes = [C.c_void_p, C.c_char_p]
    r.hts_set_opt.argtypes = [C.c_void_p, C.c_int, C.c_int]
    r.sam_hdr_read.restype = C.c_void_p
    r.sam_hdr_read.argtypes = [C.c_void_p]
    r.sam_hdr_destroy.argtypes = [C.c_void_p]
    r.bam_init1.restype = C.POINTER(Bam1)
    r.bam_destroy1.argtypes = [C.POINTER(Bam1)]
    r.sam_read1.argtypes = [C.c_void_p, C.c_void_p, C.POINTER(Bam1)]
    fp = r.hts_open(path.encode(), b"r")
    r.hts_set_fai_filename(fp, fasta.encode())
    r.hts_set_opt(fp, 18, int(mask))                                  # CRAM_OPT_REQUIRED_FIELDS
    hdr = r.sam_hdr_read(fp)
    b = r.bam_init1()
    k = 0
    t0 = time.perf_counter()
    while k < limit and r.sam_read1(fp, hdr, b) >= 0:
        k += 1
    sec = time.perf_counter() - t0
    r.bam_destroy1(b)
    r.sam_hdr_destroy(hdr)
    r.hts_close(fp)
    return {"records": k, "records_per_s": k / sec}


def run(ctx, reads=100000, tiles=20, decode_md=0, cpu=True):
    import htslib_b200 as H
    import test_cram_records as T
    from _libs import ref, ref_write_cram
    from cram_records_bench import scan_containers, tile_containers
    from test_cram_required_fields import _read_fields
    if ref() is None:
        return {"error": "oracle/_ref not built"}
    HT = T.HT
    fa = os.path.join(HT, "ce.fa")
    tmp = tempfile.mkdtemp()
    sam = os.path.join(tmp, "syn.sam")
    n = T._synthetic_sam(sam, n=reads, seed=11)
    one = os.path.join(tmp, "syn.cram")
    ref_write_cram(sam, fa, one, "3.1", [])
    img1 = np.fromfile(one, dtype=np.uint8)
    blocks1, _ = H.cram_scan_blocks(img1)
    img = tile_containers(img1, blocks1, scan_containers(H, img1), tiles)
    tiled = os.path.join(tmp, "tiled.cram")
    img.tofile(tiled)
    blocks, res = H.cram_uncompress_blocks(ctx, img)
    sizes = blocks["uncomp_size"].astype(np.int64)
    off = np.concatenate([[0], np.cumsum((sizes + 15) // 16 * 16)]).astype(np.uint64)
    udata = np.zeros(int(off[-1]) + 16, dtype=np.uint8)
    for i, (st, data) in enumerate(res):
        if int(blocks[i]["content_type"]) <= 2:
            udata[int(off[i]):int(off[i]) + len(data)] = np.frombuffer(data, dtype=np.uint8)
    del res
    fasta = H.load_fasta_upper(fa, [b"CHROMOSOME_I"])
    L = H.lib()
    L.hgpu_cram_records_last_ms.argtypes = [C.POINTER(C.c_float), C.POINTER(C.c_float)]
    L.hgpu_cram_decode_file_fields_host.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.c_char_p, C.c_int, C.c_uint32, C.c_void_p]
    L.hgpu_cram_records_free.argtypes = [C.c_void_p]
    refs = H.CramRefs()
    refs.bases = fasta[0].ctypes.data; refs.off = fasta[1].ctypes.data; refs.n_ref = 1
    names = [f for f, _ in H.BAM1_CORE_DT]
    view = lambda ptr, count, dt: np.frombuffer((C.c_uint8 * (count * np.dtype(dt).itemsize)).from_address(ptr), dtype=dt)
    out = {"workload": "CRAM 3.1 written by the reference from %d synthetic 100 bp paired reads over CHROMOSOME_I, data containers tiled %dx: "
                       "%d records" % (n, tiles, n * tiles),
           "records": n * tiles, "file_bytes": int(img.size), "decode_md": decode_md, "masks": {}}
    for label, mask in masks(H).items():
        used = H.cram_required_blocks(blocks, udata, off[:-1].copy(), mask)
        best, rec = None, None
        for it in range(3):
            if rec is not None:
                L.hgpu_cram_records_free(C.byref(rec))
            rec = H.CramRecords()
            t0 = time.perf_counter()
            rc = L.hgpu_cram_decode_file_fields_host(ctx.h, img.ctypes.data, img.size, C.byref(refs), b"tiled.cram", decode_md, mask, C.byref(rec))
            wall = time.perf_counter() - t0
            assert rc == 0, H.last_error()
            a, b = C.c_float(0), C.c_float(0)
            L.hgpu_cram_records_last_ms(C.byref(a), C.byref(b))
            if best is None or wall < best[0]:
                best = (wall, a.value, b.value)
        nrec, nsl = int(rec.n_records), int(rec.n_slices)
        assert nrec == n * tiles and view(rec.slice_status, nsl, np.int32).tolist() == [0] * nsl
        core = view(rec.core, nrec, np.dtype(H.BAM1_CORE_DT))
        doff = view(rec.data_off, nrec + 1, np.uint64)
        blob = view(rec.data, int(rec.data_bytes), np.uint8)
        _, want = _read_fields(one, fa, decode_md, mask)
        for i in list(range(0, n, max(1, n // 500))) + [n - 1]:
            for t in (0, tiles - 1):
                g = t * n + i
                assert (tuple(int(core[g][f]) for f in names), blob[int(doff[g]):int(doff[g + 1])].tobytes()) == want[i], (label, i, t)
        L.hgpu_cram_records_free(C.byref(rec))
        m = {"mask": "%#x" % mask, "used_blocks": int(used.sum()), "blocks": len(blocks),
             "uncompressed_bytes": int(sizes[used.astype(bool)].sum()), "e2e_wall_s": best[0], "records_per_s_e2e": nrec / best[0],
             "slice_decode_ms": best[1], "bam_fill_ms": best[2], "records_per_s_device": nrec / ((best[1] + best[2]) / 1e3)}
        if cpu:
            m["cpu_reference_1core"] = cpu_rate(tiled, fa, mask)
        out["masks"][label] = m
    out["checked"] = "per mask: first and last tile equal the reference's sam_read1 with the same CRAM_OPT_REQUIRED_FIELDS on sampled records"
    return out


if __name__ == "__main__":
    import torch
    import htslib_b200 as H
    torch.cuda.set_device(0)
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    ctx = H.Context(0)
    reads = int(sys.argv[1]) if len(sys.argv) > 1 else 100000
    tiles = int(sys.argv[2]) if len(sys.argv) > 2 else 20
    res = run(ctx, reads, tiles)
    res["gpu"] = gpu
    print(json.dumps(res))
