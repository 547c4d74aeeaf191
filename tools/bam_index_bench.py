"""BAI / CSI building on the device against the reference's sam_index_build3, on one synthetic BAM.

Corpus: tools/synth.bam_records over several @SQ (each shard on its own stretch of its reference), a BAM header block
in front, an unplaced tail; blocks cut as the reference's writer cuts them, level 6.  Reports, from one run:
  device_ms    hgpu_bam_index_build_host's windows from compressed bytes in HBM to the index kernels' end (CUDA events)
  e2e_ms       hgpu_bam_index_build_host from the host image to the finished file (host clock; warm-up run first)
  ref_ms       the reference's sam_index_build3 at 0 threads and at every host core, the file in page cache
  same         the device index equals the reference's, BAI bytes and CSI inflated
  gpu          card name, power limit, SM clock sampled during the device runs
One JSON line per min_shift.  Needs a GPU; oracle/_ref for the reference columns (left out without it).

  python tools/bam_index_bench.py [--gb 10] [--window-mb 0,1024] [--shifts 0,14] [--reps 3]
"""
import argparse
import ctypes as C
import json
import multiprocessing as mp
import os
import subprocess
import sys
import tempfile
import threading
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def _shard(job):
    """One shard's records, cut into BGZF blocks the way the reference's writer cuts them: (compressed, uncompressed bytes)."""
    from tools import synth
    seed, n, tid, pos0 = job
    stream, offs = synth.bam_records(seed, n, tid=tid, pos0=pos0)
    return b"".join(b for b, _ in synth.bgzf_pack_records(stream, offs, 6)), len(stream)


def corpus(total, n_sq=8, seed=11):
    """(BGZF image, uncompressed bytes): header block, shards compressed in parallel, an unplaced tail, the EOF block."""
    import _bam_index_ref as B
    import _libs
    per_shard = 60000
    n_shards = max(1, total // (336 * per_shard))
    jobs, seen = [], {}
    for s in range(n_shards):
        t = s * n_sq // n_shards
        k = seen.get(t, 0)
        seen[t] = k + 1
        jobs.append((seed * 100003 + s, per_shard, t, 10000 + k * 320000))     # a shard spans ~300 kbp
    with mp.get_context("spawn").Pool(min(len(jobs), len(os.sched_getaffinity(0)))) as pool:
        parts = pool.map(_shard, jobs, chunksize=1)
    hdr = B.header([(b"chr%d" % (t + 1), 250000000) for t in range(n_sq)])
    tail = b"".join(B.record(-1, -1, (), flag=4, name=b"u%d" % i, l_seq=150, mtid=-1) for i in range(10000))
    img = _libs.bgzf_block(hdr) + b"".join(c for c, _ in parts) + B.bgzf(tail)
    return img, len(hdr) + sum(u for _, u in parts) + len(tail)


def gpu_info(samples):
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    name, plim = [x.strip() for x in q.stdout.strip().split("\n")[0].split(",")]
    clk = [s for s in samples if s]
    return {"name": name, "power_limit": plim, "sm_clock_mhz": {"min": min(clk), "max": max(clk)} if clk else None}


class ClockSampler:
    """SM clock of GPU 0 every 50 ms while the device runs (a read-only nvidia-smi query)."""

    def __init__(self):
        self.samples, self.stop = [], threading.Event()
        self.t = threading.Thread(target=self.run, daemon=True)

    def run(self):
        while not self.stop.is_set():
            q = subprocess.run(["nvidia-smi", "--query-gpu=clocks.sm", "--format=csv,noheader,nounits", "-i", "0"],
                               capture_output=True, text=True)
            try:
                self.samples.append(int(q.stdout.strip()))
            except ValueError:
                pass
            time.sleep(0.05)

    def __enter__(self):
        self.t.start()
        return self

    def __exit__(self, *a):
        self.stop.set()
        self.t.join()


def ref_index(path, min_shift, threads):
    import _libs
    r = _libs.ref()
    r.sam_index_build3.argtypes = [C.c_char_p, C.c_char_p, C.c_int, C.c_int]
    out = path + (".csi" if min_shift > 0 else ".bai")
    t = time.perf_counter()
    rc = r.sam_index_build3(path.encode(), out.encode(), min_shift, threads)
    ms = (time.perf_counter() - t) * 1e3
    with open(out, "rb") as f:
        return rc, ms, f.read()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gb", type=float, default=10.0, help="uncompressed size of the corpus")
    ap.add_argument("--window-mb", default="0", help="window_bytes in MiB, comma-separated (0: from free device memory)")
    ap.add_argument("--shifts", default="0,14")
    ap.add_argument("--reps", type=int, default=3)
    a = ap.parse_args()
    import _bam_index_ref as B
    import _libs
    import htslib_b200 as H
    t = time.perf_counter()
    img, ulen = corpus(int(a.gb * 1e9))
    build_s = time.perf_counter() - t
    arr = np.frombuffer(img, dtype=np.uint8)
    ctx = H.Context(0)
    have_ref = _libs.ref() is not None
    with tempfile.TemporaryDirectory() as td:
        path = os.path.join(td, "corpus.bam")
        if have_ref:
            with open(path, "wb") as f:
                f.write(img)
            with open(path, "rb") as f:                        # into page cache
                while f.read(1 << 26):
                    pass
        first = {}
        for ms, wmb in [(int(x), int(w)) for w in a.window_mb.split(",") for x in a.shifts.split(",")]:
            ctx.bam_index(arr, ms, wmb << 20)                  # warm-up: module load, allocations
            e2e, dev = [], []
            with ClockSampler() as cs:
                for _ in range(a.reps):
                    t = time.perf_counter()
                    out = ctx.bam_index(arr, ms, wmb << 20)
                    e2e.append((time.perf_counter() - t) * 1e3)
                    dev.append(ctx.bam_index_last_ms()[0])
            res = {"min_shift": ms, "file_bytes": len(img), "uncompressed_bytes": ulen, "window_mb": wmb,
                   "corpus_build_s": round(build_s, 1), "index_bytes": len(out),
                   "device_ms": round(min(dev), 1), "e2e_ms": round(min(e2e), 1),
                   "e2e_GBps_compressed": round(len(img) / min(e2e) / 1e6, 2),
                   "e2e_GBps_uncompressed": round(ulen / min(e2e) / 1e6, 2), "gpu": gpu_info(cs.samples)}
            if ms in first:
                res["same_as_window_mb_%d" % first[ms][0]] = out == first[ms][1]
            else:
                first[ms] = (wmb, out)
            if have_ref and first[ms][0] == wmb:
                got = B.inflate_bgzf(out) if ms > 0 else out
                for th in (0, len(os.sched_getaffinity(0))):
                    rc, rms, rdata = ref_index(path, ms, th)
                    res["ref_threads_%d_ms" % th] = round(rms, 1)
                    res["same_threads_%d" % th] = rc == 0 and got == (B.inflate_bgzf(rdata) if ms > 0 else rdata)
            elif not have_ref:
                res["ref"] = "not measured (oracle/_ref not built)"
            print(json.dumps(res), flush=True)
    ctx.close()


if __name__ == "__main__":
    main()
