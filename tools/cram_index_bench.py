#!/usr/bin/env python
"""CRAI index building: hgpu_cram_index_build_host against the reference's sam_index_build3 (cram_index_build) on two corpora of
the same synthetic sorted 150 bp records over several @SQ:
  device  -- written by the device writer, records_per_slice 10 000: every slice multi-reference, the decode path;
  ref     -- the same records written by the reference with default options: single-reference slices, the header path.
One JSON line per corpus: device_ms (CUDA events over the slice decode and runs kernels), e2e_ms (the whole call from host
memory, best of 3), ref_ms at 0 threads and at every host core, same (the device index inflates to the reference's text),
and the card's name, power limit and sampled SM clock.  Needs oracle/_ref.

  python tools/cram_index_bench.py [records]
"""
import ctypes as C
import json
import os
import sys
import tempfile
import time
import zlib

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

READ_LEN, N_SQ, SQ_LEN = 150, 8, 60_000_000


def records(n, seed=7):
    """n unmapped-free sorted records, 150M, no aux: BAM1_CORE_DT core, data, data_off."""
    import htslib_b200 as H
    rng = np.random.default_rng(seed)
    per = n // N_SQ
    tid = np.minimum(np.arange(n) // per, N_SQ - 1).astype(np.int32)
    pos = np.zeros(n, np.int64)
    for t in range(N_SQ):
        m = tid == t
        pos[m] = 1000 + np.cumsum(rng.integers(0, 12, size=int(m.sum())))
    core = np.zeros(n, dtype=np.dtype(H.BAM1_CORE_DT))
    core["pos"], core["tid"], core["qual"], core["l_qname"], core["l_extranul"] = pos, tid, 60, 12, 1
    core["n_cigar"], core["l_qseq"], core["mtid"], core["mpos"] = 1, READ_LEN, -1, -1
    b = pos >> 14                                            # hts_reg2bin for a 150 bp read inside one 16 kbp bin
    core["bin"] = np.where((pos >> 14) == ((pos + READ_LEN - 1) >> 14), 4681 + b, 585 + (pos >> 17))
    rec = 12 + 4 + READ_LEN // 2 + READ_LEN
    data = np.zeros((n, rec), np.uint8)
    names = np.char.encode(np.char.add("r", np.char.zfill(np.arange(n).astype(str), 9)))
    data[:, :10] = np.frombuffer(names.astype("S10").tobytes(), np.uint8).reshape(n, 10)
    data[:, 12:16] = np.frombuffer(np.uint32(READ_LEN << 4).tobytes(), np.uint8)
    nib = np.array([1, 2, 4, 8], np.uint8)[rng.integers(0, 4, size=(n, READ_LEN), dtype=np.uint8)]
    data[:, 16:16 + READ_LEN // 2] = (nib[:, 0::2] << 4) | nib[:, 1::2]
    data[:, 16 + READ_LEN // 2:] = rng.integers(2, 40, size=(n, READ_LEN), dtype=np.uint8)
    off = np.arange(n + 1, dtype=np.uint64) * rec
    return core, np.concatenate([data.reshape(-1), np.zeros(8, np.uint8)]), off


def header():
    return b"@HD\tVN:1.6\tSO:coordinate\n" + b"".join(b"@SQ\tSN:c%d\tLN:%d\n" % (t, SQ_LEN) for t in range(N_SQ))


def ref_rewrite(src, dst):
    """dst: src read by the reference and written back as CRAM 3.1 with its default options (no reference: RR=0)."""
    from _libs import Bam1, ref
    r = ref()
    r.hts_open.restype = C.c_void_p
    r.hts_open.argtypes = [C.c_char_p, C.c_char_p]
    r.hts_close.argtypes = [C.c_void_p]
    r.sam_hdr_read.restype = C.c_void_p
    r.sam_hdr_read.argtypes = [C.c_void_p]
    r.sam_hdr_write.argtypes = [C.c_void_p, C.c_void_p]
    r.sam_read1.argtypes = [C.c_void_p, C.c_void_p, C.POINTER(Bam1)]
    r.sam_write1.argtypes = [C.c_void_p, C.c_void_p, C.POINTER(Bam1)]
    r.bam_init1.restype = C.POINTER(Bam1)
    r.hts_set_opt.argtypes = [C.c_void_p, C.c_int, C.c_int]
    fi, fo = r.hts_open(src.encode(), b"r"), r.hts_open(dst.encode(), b"wc")
    r.hts_set_opt.argtypes = [C.c_void_p, C.c_int, C.c_char_p]
    r.hts_set_opt(fo, 6, b"3.1")                             # CRAM_OPT_VERSION
    r.hts_set_opt.argtypes = [C.c_void_p, C.c_int, C.c_int]
    r.hts_set_opt(fo, 11, 1)                                 # CRAM_OPT_NO_REF: no reference sequence to look up
    h = r.sam_hdr_read(fi)
    assert r.sam_hdr_write(fo, h) == 0
    b = r.bam_init1()
    while r.sam_read1(fi, h, b) >= 0:
        assert r.sam_write1(fo, h, b) >= 0
    r.hts_close(fi)
    assert r.hts_close(fo) == 0


def ref_index(path, threads):
    from _libs import ref
    r = ref()
    r.sam_index_build3.argtypes = [C.c_char_p, C.c_char_p, C.c_int, C.c_int]
    out = path + ".crai"
    t = time.perf_counter()
    rc = r.sam_index_build3(path.encode(), out.encode(), 0, threads)
    ms = (time.perf_counter() - t) * 1e3
    assert rc == 0, rc
    return ms, zlib.decompressobj(31).decompress(open(out, "rb").read())


def main():
    import htslib_b200 as H
    from bam_index_bench import ClockSampler, gpu_info
    n = int(sys.argv[1]) if len(sys.argv) > 1 else 10_000_000
    ctx = H.Context(0)
    core, data, off = records(n)
    with tempfile.TemporaryDirectory() as td:
        dev_path, ref_path = os.path.join(td, "device.cram"), os.path.join(td, "ref.cram")
        img = H.cram_encode_records(ctx, header(), core, data, off, n, None, 10000, 1, 0)
        del core, data, off
        open(dev_path, "wb").write(img)
        ref_rewrite(dev_path, ref_path)
        for name, path in (("device", dev_path), ("ref", ref_path)):
            arr = np.fromfile(path, dtype=np.uint8)
            ctx.cram_index(arr)                               # warm-up
            best, dev_ms = None, None
            with ClockSampler() as clk:
                for _ in range(3):
                    t = time.perf_counter()
                    crai = ctx.cram_index(arr)
                    e2e = (time.perf_counter() - t) * 1e3
                    if best is None or e2e < best:
                        best, dev_ms = e2e, ctx.cram_index_last_ms()[0]
            d = zlib.decompressobj(31)
            text = d.decompress(crai)
            one_member = d.eof and d.unused_data == b""
            ref0, want = ref_index(path, 0)
            refn, _ = ref_index(path, os.cpu_count())
            print(json.dumps({"corpus": name, "records": n, "file_bytes": int(arr.size), "crai_lines": text.count(b"\n"),
                              "device_ms": round(dev_ms, 2), "e2e_ms": round(best, 1), "ref_ms_0_threads": round(ref0, 1),
                              "ref_ms_threads": {"threads": os.cpu_count(), "ms": round(refn, 1)},
                              "same": text == want and one_member, "gpu": gpu_info(clk.samples)}), flush=True)
    ctx.close()


if __name__ == "__main__":
    main()
