#!/usr/bin/env python
"""CRAM record decode leg of bench.py (extra.cram_records): a CRAM 3.1 file written on the box by the unmodified reference
(oracle/_ref) from a synthetic coordinate-sorted paired-end SAM over CHROMOSOME_I of tests/golden/htslib/ce.fa, its data
containers tiled K times so there are enough slices to fill the GPU; decoded by hgpu_cram_decode_file_host (block
uncompress + record decode, host buffers) and, beside it, by the reference's own sam_read1 loop on one core.

  python tools/cram_records_bench.py [reads_per_unique_file] [tiles]
"""
import ctypes as C
import json
import os
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def tile_containers(img, blocks, conts, k):
    """The file image with its data containers repeated k times (between the header container and the EOF container).
    Containers are self-contained, so every copy decodes to the same records."""
    first = int(conts[1]["offset"])
    last = int(conts[-1]["offset"])
    body = img[first:last]
    return np.concatenate([img[:first]] + [body] * k + [img[last:]])


def scan_containers(H, img):
    L = H.lib()
    dt = np.dtype([("offset", "<u8"), ("data_off", "<u8"), ("record_counter", "<i8"), ("bases", "<i8"), ("length", "<i4"), ("ref_id", "<i4"),
                   ("start", "<i4"), ("span", "<i4"), ("n_records", "<i4"), ("n_blocks", "<i4"), ("n_landmarks", "<i4"), ("landmark0", "<u4"),
                   ("first_block", "<u4"), ("crc32", "<u4")])
    L.hgpu_cram_scan_containers.restype = C.c_long
    L.hgpu_cram_scan_containers.argtypes = [C.c_void_p, C.c_uint64, C.c_void_p, C.c_long, C.c_void_p, C.c_long]
    n = L.hgpu_cram_scan_containers(img.ctypes.data, img.size, None, 0, None, 0)
    a = np.zeros(n, dtype=dt)
    L.hgpu_cram_scan_containers(img.ctypes.data, img.size, a.ctypes.data, n, None, 0)
    return a


def run(ctx, reads=100000, tiles=20, cpu=True, decode_md=0):
    import htslib_b200 as H
    from _libs import ref, ref_write_cram, ref_cram_read_all
    ref_cram_read_all = ref_cram_read_all.__wrapped__              # the live reference: the checks below slice its records
    import test_cram_records as T
    if ref() is None:
        return {"error": "oracle/_ref not built"}
    HT = T.HT
    tmp = tempfile.mkdtemp()
    sam = os.path.join(tmp, "syn.sam")
    t0 = time.perf_counter()
    n = T._synthetic_sam(sam, n=reads, seed=11)
    out = os.path.join(tmp, "syn.cram")
    ref_write_cram(sam, os.path.join(HT, "ce.fa"), out, "3.1", [])
    gen_s = time.perf_counter() - t0
    img1 = np.fromfile(out, dtype=np.uint8)
    blocks1, _ = H.cram_scan_blocks(img1)
    conts = scan_containers(H, img1)
    img = tile_containers(img1, blocks1, conts, tiles)
    tiled = os.path.join(tmp, "tiled.cram")
    img.tofile(tiled)
    blocks, _ = H.cram_scan_blocks(img)
    # @SQ order for the reference bases
    fasta = H.load_fasta_upper(os.path.join(HT, "ce.fa"), [b"CHROMOSOME_I"])
    L = H.lib()
    L.hgpu_cram_records_last_ms.argtypes = [C.POINTER(C.c_float), C.POINTER(C.c_float)]
    L.hgpu_cram_decode_file_host.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.c_char_p, C.c_int, C.c_void_p]
    L.hgpu_cram_records_free.argtypes = [C.c_void_p]
    refs = H.CramRefs()
    refs.bases = fasta[0].ctypes.data; refs.off = fasta[1].ctypes.data; refs.n_ref = 1
    best = None
    out_s = None
    for it in range(3):
        if out_s is not None:
            L.hgpu_cram_records_free(C.byref(out_s))
        out_s = H.CramRecords()
        t0 = time.perf_counter()
        rc = L.hgpu_cram_decode_file_host(ctx.h, img.ctypes.data, img.size, C.byref(refs), b"tiled.cram", decode_md, C.byref(out_s))
        wall = time.perf_counter() - t0
        assert rc == 0, H.last_error()
        a, b = C.c_float(0), C.c_float(0)
        L.hgpu_cram_records_last_ms(C.byref(a), C.byref(b))
        if best is None or wall < best[0]:
            best = (wall, a.value, b.value)
    nrec, nsl = int(out_s.n_records), int(out_s.n_slices)
    view = lambda ptr, count, dt: np.frombuffer((C.c_uint8 * (count * np.dtype(dt).itemsize)).from_address(ptr), dtype=dt)
    sst = view(out_s.slice_status, nsl, np.int32)
    assert sst.tolist() == [0] * nsl, sst.tolist()[:8]
    assert nrec == n * tiles
    core = view(out_s.core, nrec, np.dtype(H.BAM1_CORE_DT))
    doff = view(out_s.data_off, nrec + 1, np.uint64)
    blob = view(out_s.data, int(out_s.data_bytes), np.uint8)
    # every tile equals the first; the first equals the reference
    want = ref_cram_read_all(out, os.path.join(HT, "ce.fa"), decode_md)
    names = [f for f, _ in H.BAM1_CORE_DT]
    for i in list(range(0, n, max(1, n // 500))) + [n - 1]:
        for t in (0, tiles - 1):
            g = t * n + i
            assert tuple(int(core[g][f]) for f in names) == want[i][0] and blob[int(doff[g]):int(doff[g + 1])].tobytes() == want[i][1], (i, t)
    data_bytes = int(out_s.data_bytes)
    got = {"slice_status": sst}
    usize = int(blocks["uncomp_size"].astype(np.int64).sum())
    res = {"workload": "CRAM 3.1 written by the reference from %d synthetic 100 bp paired reads over CHROMOSOME_I (all read-feature codes, 3 read groups, "
                       "aux tags), data containers tiled %dx: %d slices, %d records" % (n, tiles, len(got["slice_status"]), nrec),
           "records": nrec, "slices": len(got["slice_status"]), "file_bytes": int(img.size), "uncompressed_block_bytes": usize,
           "bam_bytes_out": data_bytes + 48 * nrec, "gen_s": round(gen_s, 1),
           "slice_decode_ms": best[1], "bam_fill_ms": best[2],
           "records_per_s_device": nrec / ((best[1] + best[2]) / 1e3),
           "e2e_wall_s": best[0], "records_per_s_e2e": nrec / best[0],
           "api": "hgpu_cram_decode_file_host (scan + block uncompress + record decode, host buffers)",
           "roofline": {"bound": "hbm", "achieved": (usize + data_bytes + 48 * nrec) / ((best[1] + best[2]) / 1e3) / 1e9, "unit": "GB/s",
                        "note": "algorithmic bytes = uncompressed blocks read + bam1_t written; the slice kernel is a latency-bound scalar "
                                "chain per warp (one warp per slice), not a bandwidth kernel"},
           "checked": "first and last tile equal the reference's sam_read1 on sampled records; all slices status 0"}
    # ---- the write side (BASELINE config 4 shape): the decoded records of the first tiles back into a CRAM 3.1 file ----
    try:
        header = b"".join(l for l in open(sam, "rb") if l.startswith(b"@"))
        ne = min(nrec, n * 10)
        L.hgpu_cram_encode_records_host.argtypes = [C.c_void_p, C.c_char_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint32, C.c_int, C.c_void_p, C.c_void_p]
        best_e = None
        for it in range(2):
            eo, el = C.c_void_p(), C.c_uint64(0)
            t0 = time.perf_counter()
            rc = L.hgpu_cram_encode_records_host(ctx.h, header, len(header), out_s.core, out_s.data, out_s.data_off, ne, C.byref(refs), 10000, 1, C.byref(eo), C.byref(el))
            sec = time.perf_counter() - t0
            assert rc == 0, H.last_error()
            img_e = C.string_at(eo.value, el.value)
            C.CDLL(None).free(C.c_void_p(eo.value))
            if best_e is None or sec < best_e:
                best_e = sec
        enc_path = os.path.join(tmp, "enc.cram")
        open(enc_path, "wb").write(img_e)
        back = ref_cram_read_all(enc_path, os.path.join(HT, "ce.fa"), 0)
        assert len(back) == ne
        for i in (0, 1, ne // 2, ne - 1):
            lqn = int(core[i]["l_qname"])
            assert back[i][0][:3] == tuple(int(core[i][f]) for f in names[:3]) and back[i][1][:lqn] == blob[int(doff[i]):int(doff[i]) + lqn].tobytes(), i
        in_bytes = int(doff[ne]) + 48 * ne
        res["encode"] = {"workload": "the first %d decoded records back into a CRAM 3.1 file (coded against the reference: substitution features), 10 000 records per slice" % ne,
                         "records": ne, "bam_bytes_in": in_bytes, "cram_bytes_out": len(img_e), "ratio": len(img_e) / in_bytes,
                         "wall_s": best_e, "records_per_s_e2e": ne / best_e,
                         "api": "hgpu_cram_encode_records_host (host buffers; series split + rANS Nx16 trial + tok3 names on the device)",
                         "checked": "the reference's sam_read1 reads the file back: record count and sampled records equal"}
    except Exception as ex:
        res["encode"] = {"error": repr(ex)}
    L.hgpu_cram_records_free(C.byref(out_s))
    if cpu:
        r = ref()
        r.hts_open.restype = C.c_void_p
        r.hts_open.argtypes = [C.c_char_p, C.c_char_p]
        fp = r.hts_open(tiled.encode(), b"r")
        r.hts_set_fai_filename.argtypes = [C.c_void_p, C.c_char_p]
        r.hts_set_fai_filename(fp, os.path.join(HT, "ce.fa").encode())
        r.hts_set_opt.argtypes = [C.c_void_p, C.c_int, C.c_int]
        r.hts_set_opt(fp, 0, decode_md)
        r.sam_hdr_read.restype = C.c_void_p
        r.sam_hdr_read.argtypes = [C.c_void_p]
        hdr = r.sam_hdr_read(fp)
        from _libs import Bam1
        r.bam_init1.restype = C.POINTER(Bam1)
        r.sam_read1.argtypes = [C.c_void_p, C.c_void_p, C.POINTER(Bam1)]
        b = r.bam_init1()
        k = 0
        t0 = time.perf_counter()
        while r.sam_read1(fp, hdr, b) >= 0:
            k += 1
            if k >= 2_000_000:
                break
        sec = time.perf_counter() - t0
        res["cpu_reference_1core"] = {"records": k, "records_per_s": k / sec, "sample": "sam_read1 loop over the same tiled file, first %d records" % k}
    return res


if __name__ == "__main__":
    import torch
    import htslib_b200 as H
    torch.cuda.set_device(0)
    ctx = H.Context(0)
    reads = int(sys.argv[1]) if len(sys.argv) > 1 else 100000
    tiles = int(sys.argv[2]) if len(sys.argv) > 2 else 120
    print(json.dumps(run(ctx, reads, tiles)))
