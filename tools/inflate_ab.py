"""A/B of two or more builds of bgzf_inflate_kernel in one process, on the bench corpus.

    python tools/inflate_ab.py A.so B.so [C.so ...] [--gb 10] [--runs 3] [--steps 10] [--warmup 2] [--out DIR]

Build the libraries side by side first (HGPU_OUT names the output, HGPU_BUILD_DIR the object directory):
    HGPU_OUT=libhtsgpu_a.so HGPU_BUILD_DIR=build_a python -m htslib_b200.build
Every library inflates the same synthetic BAM (tools/synth.py, the corpus bench.py times) into its own output
buffer; the runs alternate A, B, C, A, B, C, ... at `--steps` launches each, timed with CUDA events, and the card's
name, power limit and SM clock are read around them.  Every build's whole output, per-block lengths and statuses are
compared on the device with the first build's.  Prints one JSON line; `--out DIR` also writes it to DIR/inflate_ab.json."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tools import synth  # noqa: E402


def smi(q):
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader", "-i", "0"],
                              capture_output=True, text=True, timeout=20).stdout.strip()
    except Exception as e:          # the numbers are reported as missing, the run goes on
        return "unavailable (%s)" % e


class Build:
    def __init__(self, path):
        self.path = path
        self.L = C.CDLL(os.path.abspath(path))
        vp, u32 = C.c_void_p, C.c_uint32
        self.L.hgpu_create.restype = vp
        self.L.hgpu_create.argtypes = [C.c_int]
        self.L.hgpu_destroy.argtypes = [vp]
        self.L.hgpu_bgzf_inflate_batch_dev.argtypes = [vp, vp, vp, vp, u32, vp, vp, vp, vp, vp, vp]
        self.h = self.L.hgpu_create(0)
        if not self.h:
            raise RuntimeError("hgpu_create failed for %s" % path)

    def launch(self, a, stream):
        rc = self.L.hgpu_bgzf_inflate_batch_dev(self.h, a["in"].data_ptr(), a["in_off"].data_ptr(), a["in_len"].data_ptr(),
                                                a["n"], a["out"].data_ptr(), a["out_off"].data_ptr(), a["cap"].data_ptr(),
                                                a["len"].data_ptr(), a["st"].data_ptr(), stream)
        if rc != 0:
            raise RuntimeError("inflate launch failed in %s: rc=%d" % (self.path, rc))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("builds", nargs="+")
    ap.add_argument("--gb", type=float, default=10.0)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--out")
    args = ap.parse_args()

    corpus = synth.bam_bgzf_corpus(args.gb * 1e9)
    comp, clen, ulen = corpus["comp"], corpus["clen"], corpus["ulen"]
    n = len(clen)
    dev = torch.device("cuda:0")
    t = lambda x: torch.from_numpy(x.view(np.int64) if x.dtype == np.uint64 else x.view(np.int32)).to(dev)
    in_off = np.concatenate([[0], np.cumsum(clen.astype(np.int64))[:-1]]).astype(np.uint64)
    out_off = np.concatenate([[0], np.cumsum(ulen.astype(np.int64))[:-1]]).astype(np.uint64)
    d_in = torch.zeros(comp.size + 64, dtype=torch.uint8, device=dev)
    d_in[:comp.size].copy_(torch.from_numpy(comp.copy()))
    shared = dict(n=n, **{"in": d_in}, in_off=t(in_off), in_len=t(clen), out_off=t(out_off), cap=t(ulen))
    if len(args.builds) < 2:
        ap.error("at least two builds")
    builds = [Build(p) for p in args.builds]
    bufs = [dict(shared, out=torch.zeros(int(ulen.sum()) + 64, dtype=torch.uint8, device=dev),
                 len=torch.zeros(n, dtype=torch.int32, device=dev), st=torch.full((n,), 9, dtype=torch.int32, device=dev))
            for _ in builds]
    s = torch.cuda.Stream()
    for b, a in zip(builds, bufs):
        for _ in range(args.warmup):
            b.launch(a, s.cuda_stream)
    torch.cuda.synchronize()
    card = dict(name=smi("name"), power_limit=smi("power.limit"), clocks_max_sm=smi("clocks.max.sm"))
    runs = {p: [] for p in args.builds}
    clocks = []
    for _ in range(args.runs):
        for b, a in zip(builds, bufs):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            with torch.cuda.stream(s):
                e0.record(s)
                for _ in range(args.steps):
                    b.launch(a, s.cuda_stream)
                e1.record(s)
            clocks.append(smi("clocks.sm"))                # sampled while the launches run
            torch.cuda.synchronize()
            runs[b.path].append(round(e0.elapsed_time(e1) / args.steps, 3))
    same_out = all(bool(torch.equal(bufs[0]["out"], a["out"])) for a in bufs[1:])
    same_len = all(bool(torch.equal(bufs[0]["len"], a["len"])) for a in bufs[1:])
    same_st = all(bool(torch.equal(bufs[0]["st"], a["st"])) for a in bufs[1:])
    errors = [int((a["st"] != 0).sum()) for a in bufs]
    res = dict(blocks=n, bytes=int(ulen.sum()), card=card, clocks_sm_sampled=clocks,
               ms_per_step={k: v for k, v in runs.items()},
               gbs={k: [round(float(ulen.sum()) / ms / 1e6, 1) for ms in v] for k, v in runs.items()},
               identical_output=same_out, identical_block_len=same_len, identical_block_status=same_st, blocks_not_ok=errors)
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "inflate_ab.json"), "w") as f:
            f.write(line + "\n")
    for b in builds:
        b.L.hgpu_destroy(b.h)
    if not (same_out and same_len and same_st):
        sys.exit(1)


if __name__ == "__main__":
    main()
